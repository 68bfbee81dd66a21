"""CPU checks of the SLA modules' per-entry lengths: the five _vl entry points return their codes before any CUDA call (a null
or misaligned seq_lens or topks, head dim 64, l != lk), topk_i follows Python's int(ratio * nblk) rule exactly, and
SparseLinearAttention / SageSparseLinearAttention.forward reach today's entry points without seq_lens, the _vl ones with it, and
refuse the calls it does not serve before any library call (checked with a recording stand-in for the library).  The numbers
are checked on the GPU in tests/test_gpu_sla_seq_lens.py."""
import ctypes

import pytest
import torch

INVALID, UNSUPPORTED = -1, -2
BF16 = 0
NULL = ctypes.c_void_p(0)


def _p(v=4096):
    return ctypes.c_void_p(v)          # non-null, 16-byte aligned, never dereferenced: validation runs before any CUDA call


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


def _quant(lib, d=128, seq_lens=None):
    return lib.tdb200_sla_quant_qk_vl(_p(), _p(), BF16, 2, 256, 2, d, _p() if seq_lens is None else seq_lens, _p(), _p(), _p(),
                                      _p(), _p(), _p(), _p(), 128, 64, None)


def _bmap(lib, d=128, seq_lens=None, topks=None):
    return lib.tdb200_sla_block_map_vl(_p(), _p(), BF16, 2, 2, 2, 4, d, 1, _p() if seq_lens is None else seq_lens,
                                       _p() if topks is None else topks, 128, 64, _p(), _p(), None)


def _mom(lib, d=128, seq_lens=None):
    return lib.tdb200_sla_linear_moments_vl(_p(), _p(), BF16, 2, 256, 2, d, _p() if seq_lens is None else seq_lens, 0, _p(), _p(),
                                            None)


def _attn(lib, d=128, lk=256, seq_lens=None, topks=None):
    return lib.tdb200_sla_attn_fwd_vl(_p(), _p(), _p(), _p(), _p(), _p(), BF16, _p(), 1, _p(), _p(), _p(), _p(), 2, 256, lk, 2, d,
                                      _p() if seq_lens is None else seq_lens, _p() if topks is None else topks, 0.088, 0, 128, 64,
                                      None)


def _attn16(lib, d=128, lk=256, seq_lens=None, topks=None):
    return lib.tdb200_sla_attn16_fwd_vl(_p(), _p(), _p(), BF16, _p(), 1, _p(), _p(), _p(), _p(), 2, 256, lk, 2, d,
                                        _p() if seq_lens is None else seq_lens, _p() if topks is None else topks, 0.088, 0, 128,
                                        64, None)


CASES = [
    ("quant", _quant, dict(seq_lens=NULL), INVALID, "seq_lens"),
    ("quant", _quant, dict(seq_lens=_p(4098)), INVALID, "seq_lens"),
    ("quant", _quant, dict(d=64), UNSUPPORTED, "head dim"),
    ("bmap", _bmap, dict(seq_lens=NULL), INVALID, "seq_lens"),
    ("bmap", _bmap, dict(topks=_p(4098)), INVALID, "topks"),
    ("bmap", _bmap, dict(d=64), UNSUPPORTED, "head dim"),
    ("mom", _mom, dict(seq_lens=NULL), INVALID, "seq_lens"),
    ("mom", _mom, dict(seq_lens=_p(4097)), INVALID, "seq_lens"),
    ("mom", _mom, dict(d=64), UNSUPPORTED, "head dim"),
    ("attn", _attn, dict(seq_lens=NULL), INVALID, "seq_lens"),
    ("attn", _attn, dict(topks=NULL), INVALID, "topks"),
    ("attn", _attn, dict(lk=128), INVALID, "lk"),
    ("attn", _attn, dict(d=64), UNSUPPORTED, "head dim"),
    ("attn16", _attn16, dict(seq_lens=_p(4098)), INVALID, "seq_lens"),
    ("attn16", _attn16, dict(topks=NULL), INVALID, "topks"),
    ("attn16", _attn16, dict(lk=128), INVALID, "lk"),
    ("attn16", _attn16, dict(d=64), UNSUPPORTED, "head dim"),
]


@pytest.mark.parametrize("name,fn,kw,code,needle", CASES, ids=[f"{c[0]}-{i}" for i, c in enumerate(CASES)])
def test_argument_checks_return_codes(lib, name, fn, kw, code, needle):
    assert fn(lib, **kw) == code
    assert needle in lib.tdb200_last_error().decode()


@pytest.mark.parametrize("ratio", [0.0, 0.05, 0.1, 0.15, 0.2, 0.3, 1 / 3, 0.5, 0.7, 0.99, 1.0, 1.5, 7])
@pytest.mark.parametrize("blkk", [64, 128])
def test_topks_follow_the_modules_rule(ratio, blkk):
    from turbodiffusion_b200.SLA.utils import seq_topks
    lens = torch.tensor([0, 1, 63, 64, 65, 127, 128, 129, 1000, 20280, 32759, 32760, 75600], dtype=torch.int32)
    got = seq_topks(lens, ratio, blkk)
    for n, t in zip(lens.tolist(), got.tolist()):
        nblk = (n + blkk - 1) // blkk
        assert t == max(1, min(nblk, int(ratio * nblk))), (n, ratio)


class _Recorder:
    """Stands in for the library: records the entry points called and returns 0."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append(name)
            return 0
        return fn


@pytest.fixture
def recorder(monkeypatch):
    from turbodiffusion_b200 import _lib
    from turbodiffusion_b200.SLA import core, utils
    rec = _Recorder()
    for mod in (core, utils):
        monkeypatch.setattr(mod, "lib", lambda: rec)
    for mod in (core, utils):
        monkeypatch.setattr(mod, "require_cuda", lambda *t: None)
        monkeypatch.setattr(mod, "stream_ptr", lambda dev: None)
    monkeypatch.setattr(_lib, "stream_ptr", lambda dev: None)
    monkeypatch.setattr(core, "get_cuda_arch", lambda device_index: "sm100")
    return rec


def _mod(kind):
    from turbodiffusion_b200.SLA import core
    if kind == "sage":
        return core.SageSparseLinearAttention(128, 0.3)
    return core.SparseLinearAttention(128, 0.3, BLKQ=128, BLKK=64)


@pytest.mark.parametrize("kind", ["sage", "sla"])
def test_seq_lens_reach_the_vl_entry_points(recorder, monkeypatch, kind):
    from turbodiffusion_b200.SLA import core
    monkeypatch.setattr(core, "project_moments", lambda w, kv, dtype: torch.empty(kv.shape, dtype=dtype))
    q = torch.zeros(2, 256, 2, 128, dtype=torch.bfloat16)
    m = _mod(kind)
    m._keep_selection = {}
    with torch.no_grad():
        m(q, q, q, seq_lens=torch.tensor([256, 100]))
    assert m._keep_selection["topk"] == 1 and isinstance(m._keep_selection["topk"], int)   # the LUT stride: max(1, int(0.3 * 4))
    assert m._keep_selection["topks"].tolist() == [1, 1]
    want = ["tdb200_sla_quant_qk_vl", "tdb200_sla_block_map_vl", "tdb200_sla_linear_moments_vl",
            "tdb200_sla_attn_fwd_vl" if kind == "sage" else "tdb200_sla_attn16_fwd_vl"]
    assert recorder.calls == want


@pytest.mark.parametrize("kind", ["sage", "sla"])
@pytest.mark.parametrize("what", ["grad", "head dim", "tangent", "fp8"])
def test_refusals_come_before_any_library_call(recorder, kind, what, monkeypatch):
    import torch.autograd.forward_ad as fwAD
    from turbodiffusion_b200.SLA import utils
    m = _mod(kind)
    q = torch.zeros(1, 64, 1, 128)
    lens = torch.tensor([10])
    if what == "fp8":
        if kind != "sage":
            pytest.skip("FP8 P.V is a SageSparseLinearAttention setting")
        monkeypatch.setattr(utils, "SAGE_PV", "fp8")
    with pytest.raises(NotImplementedError):
        if what == "grad":
            m(q.clone().requires_grad_(), q, q, seq_lens=lens)
        elif what == "head dim":
            m(torch.zeros(1, 64, 1, 64), torch.zeros(1, 64, 1, 64), torch.zeros(1, 64, 1, 64), seq_lens=lens)
        elif what == "tangent":
            with fwAD.dual_level():
                m(fwAD.make_dual(q, torch.ones_like(q)), q, q, seq_lens=lens)
        else:
            m(q, q, q, seq_lens=lens)
    assert recorder.calls == []


def test_lengths_outside_the_sequence_are_refused_before_any_library_call(recorder):
    from turbodiffusion_b200.SLA import core
    q = torch.zeros(2, 64, 1, 128, dtype=torch.bfloat16)
    with torch.no_grad(), pytest.raises(ValueError, match="seq_lens"):
        core._SLABase._forward_vl(_mod("sla"), q, q, q, False, torch.tensor([65, 3]))
    with torch.no_grad(), pytest.raises(ValueError, match="prefix"):
        core._SLABase._forward_vl(_mod("sla"), q, q, q, False, torch.tensor([[True] * 63 + [False]] * 1 + [[False] + [True] * 63]))
    assert recorder.calls == []


def test_no_seq_lens_runs_todays_path(monkeypatch):
    """forward without seq_lens does not enter _forward_vl."""
    from turbodiffusion_b200.SLA import core
    monkeypatch.setattr(core._SLABase, "_forward_vl", lambda *a: pytest.fail("_forward_vl reached without seq_lens"))
    monkeypatch.setattr(core, "require_cuda", lambda *t: (_ for _ in ()).throw(RuntimeError("stop")))
    with torch.no_grad(), pytest.raises(RuntimeError, match="stop"):
        _mod("sage")(torch.zeros(1, 64, 1, 128), torch.zeros(1, 64, 1, 128), torch.zeros(1, 64, 1, 128))
