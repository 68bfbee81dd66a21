"""CPU checks of the dense attention entry point (tdb200_attn_dense_fwd) and its Python function: every argument check returns
its code and a message naming the entry point before any CUDA call, a well-formed call on a host without a GPU comes back
with an error code, and ops.dense_attention refuses CPU tensors."""
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


def _call(lib, q=None, k=None, v=None, dtype=BF16, out=None, b=1, lq=256, lk=77, h=2, d=128, sm_scale=0.088):
    args = [_p() if t is None else t for t in (q, k, v)]
    return lib.tdb200_attn_dense_fwd(*args, dtype, _p() if out is None else out, b, lq, lk, h, d, sm_scale, None)


NULL = ctypes.c_void_p(0)
CASES = [
    ("null q", dict(q=NULL), INVALID, b"null"),
    ("null k", dict(k=NULL), INVALID, b"null"),
    ("null v", dict(v=NULL), INVALID, b"null"),
    ("null out", dict(out=NULL), INVALID, b"null"),
    ("b = 0", dict(b=0), INVALID, b"shape"),
    ("lq = 0", dict(lq=0), INVALID, b"shape"),
    ("lk < 0", dict(lk=-5), INVALID, b"shape"),
    ("h = 0", dict(h=0), INVALID, b"shape"),
    ("d = 0", dict(d=0), INVALID, b"shape"),
    ("misaligned k", dict(k=_p(4100)), INVALID, b"aligned"),
    ("dtype tag", dict(dtype=7), UNSUPPORTED, b"dtype"),
    ("head dim 64", dict(d=64), UNSUPPORTED, b"head dim"),
    ("head dim 96", dict(d=96), UNSUPPORTED, b"head dim"),
    ("heads beyond the grid", dict(h=70000), UNSUPPORTED, b"too large"),
    ("batch beyond the grid", dict(b=70000), UNSUPPORTED, b"too large"),
    ("lq beyond the tensor map", dict(lq=1 << 33), UNSUPPORTED, b"too large"),
    ("lk * h * d beyond the tensor map's stride", dict(lk=1 << 30, h=1024), UNSUPPORTED, b"too large"),
]


@pytest.mark.parametrize("name,kw,code,needle", [pytest.param(*c, id=c[0].replace(" ", "-")) for c in CASES])
def test_argument_checks_return_codes(lib, name, kw, code, needle):
    rc = _call(lib, **kw)
    msg = lib.tdb200_last_error() or b""
    assert rc == code, (name, rc, msg)
    assert msg.startswith(b"attn_dense_fwd:") and needle in msg, (name, msg)


def test_valid_call_without_a_gpu_reports_an_error_code(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    for dtype in (BF16, FP16):
        rc = _call(lib, dtype=dtype)
        assert rc in (-3, -4) and lib.tdb200_last_error()


def test_dense_attention_refuses_cpu_tensors(lib):
    import torch
    from turbodiffusion_b200 import _lib, ops
    q, kv = torch.zeros(1, 4, 2, 128, dtype=torch.bfloat16), torch.zeros(1, 3, 2, 128, dtype=torch.bfloat16)
    with pytest.raises(_lib.Tdb200Error, match="CUDA tensors only"):
        ops.dense_attention(q, kv, kv)


def test_abi_version_and_export(lib):
    from turbodiffusion_b200 import _lib
    assert "tdb200_attn_dense_fwd" in _lib.exported_names()
    assert lib.tdb200_abi_version() == 2          # an added symbol breaks no caller


def test_product_does_not_import_the_oracle():
    for name in ("ops/core.py", "csrc/dense_attn.cu"):
        text = open(os.path.join(ROOT, "turbodiffusion_b200", name)).read()
        assert "td_oracle" not in text and "from oracle" not in text and "import oracle" not in text, name
