"""CPU checks of the Hopper SageSLA block family (BLKQ=64, BLKK=128): argument validation of the block sizes and head-major
shapes in tdb200_sla_quant_qk / tdb200_sla_attn_fwd, the served-arch switch and the sequence-parallel refusal under "sm90"."""
import ctypes

import pytest


def _p(v=4096):
    return ctypes.c_void_p(v)          # non-null, 16-byte aligned, never dereferenced: validation runs before any CUDA call


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


def _quant(lib, d=128, blkq=64, blkk=128):
    return lib.tdb200_sla_quant_qk(_p(), _p(), 0, 1, 256, 256, 2, d, _p(), _p(), _p(), _p(), _p(), _p(), _p(), blkq, blkk, None)


def _attn(lib, d=128, blkq=64, blkk=128, topk=1, q_i8=None, dtype=0):
    return lib.tdb200_sla_attn_fwd(_p() if q_i8 is None else q_i8, _p(), _p(), _p(), _p(), _p(), dtype, _p(), topk, _p(), _p(), _p(),
                                   _p(), 1, 256, 256, 2, d, 0.088, 0, blkq, blkk, 0, None)


def test_argument_validation_of_the_block_entry_points(lib):
    INVALID, UNSUPPORTED = -1, -2
    cases = [
        ("quant block pair", lambda: _quant(lib, blkq=64, blkk=64), UNSUPPORTED, b"block"),
        ("quant block pair 128x128", lambda: _quant(lib, blkq=128, blkk=128), UNSUPPORTED, b"block"),
        ("quant head dim", lambda: _quant(lib, d=96), UNSUPPORTED, b"head dim"),
        ("quant null", lambda: lib.tdb200_sla_quant_qk(None, None, 0, 1, 256, 256, 2, 128, _p(), _p(), _p(), _p(), _p(), _p(), _p(),
                                                        64, 128, None), INVALID, b"null"),
        ("attn block pair", lambda: _attn(lib, blkq=32, blkk=128), UNSUPPORTED, b"block"),
        ("attn head dim", lambda: _attn(lib, d=96), UNSUPPORTED, b"head dim"),
        ("attn head dim 128x64", lambda: _attn(lib, d=96, blkq=128, blkk=64), UNSUPPORTED, b"head dim"),
        ("attn null", lambda: _attn(lib, q_i8=ctypes.c_void_p(0)), INVALID, b"null"),
        # lk = 256: nblk = 2 for 128-row key blocks, so topk = 3 is out of range ...
        ("attn topk follows blkk", lambda: _attn(lib, topk=3), INVALID, b"topk"),
        # ... but not for 64-row key blocks (nblk = 4): that call gets past the topk check and stops at the dtype tag
        ("attn topk 128x64", lambda: _attn(lib, topk=3, blkq=128, blkk=64, dtype=7), UNSUPPORTED, b"dtype"),
    ]
    for name, call, code, needle in cases:
        rc = call()
        msg = lib.tdb200_last_error() or b""
        assert rc == code, (name, rc, msg)
        assert needle in msg, (name, msg)


def test_served_arch_switch():
    from turbodiffusion_b200.SLA import utils
    assert utils.SERVED_ARCH == "sm100"
    with pytest.raises(ValueError):
        utils.set_served_arch("sm80")
    assert utils.SERVED_ARCH == "sm100"
    prev = utils.set_served_arch("sm90")
    try:
        assert prev == "sm100" and utils.SERVED_ARCH == "sm90"
    finally:
        assert utils.set_served_arch(prev) == "sm90"
    assert utils.SERVED_ARCH == "sm100"


def test_install_forwards_sage_arch():
    import sys
    import turbodiffusion_b200
    from turbodiffusion_b200.SLA import utils
    saved = {n: sys.modules.get(n) for n in ("turbo_diffusion_ops", "ops", "SLA", "turbodiffusion.ops", "turbodiffusion.SLA")}
    try:
        turbodiffusion_b200.install(sage_arch="sm90")
        assert utils.SERVED_ARCH == "sm90"
        with pytest.raises(ValueError):
            turbodiffusion_b200.install(sage_arch="sm86")
        turbodiffusion_b200.install()
        assert utils.SERVED_ARCH == "sm100"
    finally:
        utils.set_served_arch("sm100")
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m


def test_sequence_parallel_refuses_the_hopper_family():
    from turbodiffusion_b200.dist import SequenceParallel
    from turbodiffusion_b200.SLA import utils
    sp = SequenceParallel(1024, world=2, rank=0)
    prev = utils.set_served_arch("sm90")
    try:
        with pytest.raises(NotImplementedError, match="sm100"):
            sp.install(None)
    finally:
        utils.set_served_arch(prev)


def test_sequence_parallel_hooks_refuse_a_switch_made_after_install():
    """Hooks installed under "sm100" must not go on running 128/64 blocks once "sm90" is selected."""
    from turbodiffusion_b200.dist import SequenceParallel, SPAttention, UlyssesAttention, UnevenUlyssesAttention
    from turbodiffusion_b200.SLA import utils
    sp = SequenceParallel(1024, world=2, rank=0)
    hooks = [SPAttention(sp, None), UlyssesAttention(sp, None), UnevenUlyssesAttention(sp, None, heads=3)]
    prev = utils.set_served_arch("sm90")
    try:
        for hook in hooks:
            with pytest.raises(NotImplementedError, match="sm100"):
                hook(None, None, None)
    finally:
        utils.set_served_arch(prev)
