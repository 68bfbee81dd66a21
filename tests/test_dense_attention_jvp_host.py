"""CPU checks of the dense attention JVP entry point (tdb200_attn_dense_jvp) and its Python function: every argument check
returns its code and a message naming the entry point before any CUDA call, a well-formed call on a host without a GPU comes
back with an error code, and ops.dense_attention_jvp refuses CPU tensors and tangents whose shape is not their primal's."""
import ctypes
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, UNSUPPORTED = -1, -2
BF16, FP16 = 0, 1


def _p(v=4096):
    return ctypes.c_void_p(v)          # non-null, 16-byte aligned, never dereferenced: validation runs before any CUDA call


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


POINTERS = ("q", "k", "v", "q_t", "k_t", "v_t", "out", "out_t")


def _call(lib, dtype=BF16, b=1, lq=256, lk=77, h=2, d=128, sm_scale=0.088, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in POINTERS}
    return lib.tdb200_attn_dense_jvp(a["q"], a["k"], a["v"], a["q_t"], a["k_t"], a["v_t"], dtype, a["out"], a["out_t"], b, lq,
                                     lk, h, d, sm_scale, None)


NULL = ctypes.c_void_p(0)
CASES = ([(f"null {n}", {n: NULL}, INVALID, b"null") for n in POINTERS] +
         [(f"misaligned {n}", {n: _p(4100)}, INVALID, b"aligned") for n in POINTERS] + [
    ("b = 0", dict(b=0), INVALID, b"shape"),
    ("lq = 0", dict(lq=0), INVALID, b"shape"),
    ("lk < 0", dict(lk=-5), INVALID, b"shape"),
    ("h = 0", dict(h=0), INVALID, b"shape"),
    ("d = 0", dict(d=0), INVALID, b"shape"),
    ("dtype tag", dict(dtype=7), UNSUPPORTED, b"dtype"),
    ("head dim 64", dict(d=64), UNSUPPORTED, b"head dim"),
    ("head dim 96", dict(d=96), UNSUPPORTED, b"head dim"),
    ("heads beyond the grid", dict(h=70000), UNSUPPORTED, b"too large"),
    ("batch beyond the grid", dict(b=70000), UNSUPPORTED, b"too large"),
    ("lq beyond the tensor map", dict(lq=1 << 33), UNSUPPORTED, b"too large"),
    ("lk * h * d beyond the tensor map's stride", dict(lk=1 << 30, h=1024), UNSUPPORTED, b"too large"),
])


@pytest.mark.parametrize("name,kw,code,needle", [pytest.param(*c, id=c[0].replace(" ", "-")) for c in CASES])
def test_argument_checks_return_codes(lib, name, kw, code, needle):
    rc = _call(lib, **kw)
    msg = lib.tdb200_last_error() or b""
    assert rc == code, (name, rc, msg)
    assert msg.startswith(b"attn_dense_jvp:") and needle in msg, (name, msg)


def test_valid_call_without_a_gpu_reports_an_error_code(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    for dtype in (BF16, FP16):
        rc = _call(lib, dtype=dtype)
        assert rc in (-3, -4) and lib.tdb200_last_error()


def test_dense_attention_jvp_refuses_cpu_tensors(lib):
    import torch
    from turbodiffusion_b200 import _lib, ops
    q, kv = torch.zeros(1, 4, 2, 128, dtype=torch.bfloat16), torch.zeros(1, 3, 2, 128, dtype=torch.bfloat16)
    with pytest.raises(_lib.Tdb200Error, match="CUDA tensors only"):
        ops.dense_attention_jvp(q, kv, kv, q, kv, kv)


@pytest.mark.parametrize("which", [0, 1, 2], ids=["q_t", "k_t", "v_t"])
def test_dense_attention_jvp_refuses_tangents_of_another_shape(lib, which, monkeypatch):
    import torch
    from turbodiffusion_b200 import ops
    from turbodiffusion_b200.ops import core
    monkeypatch.setattr(core, "require_cuda", lambda *t: None)    # reach the shape check on CPU tensors
    q, kv = torch.zeros(1, 4, 2, 128, dtype=torch.bfloat16), torch.zeros(1, 3, 2, 128, dtype=torch.bfloat16)
    tangents = [q, kv, kv]
    tangents[which] = torch.zeros(1, 5, 2, 128, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match=["q_t", "k_t", "v_t"][which]):
        ops.dense_attention_jvp(q, kv, kv, *tangents)


def test_abi_version_and_export(lib):
    from turbodiffusion_b200 import _lib
    assert "tdb200_attn_dense_jvp" in _lib.exported_names()
    assert lib.tdb200_abi_version() == 2          # an added symbol breaks no caller
