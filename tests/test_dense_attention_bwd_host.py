"""CPU checks of the dense attention training path: the argument checks of tdb200_attn_dense_fwd_lse, tdb200_attn_dense_jvp_lse,
tdb200_attn_dense_bwd and tdb200_attn_dense_bwd_workspace_bytes return their codes and a message naming the entry point before
any CUDA call, well-formed calls on a host without a GPU come back with an error code, and ops.dense_attention /
ops.dense_attention_jvp pick their path by grad mode and requires_grad (checked with a recording stand-in for the library)."""
import ctypes

import pytest

INVALID, UNSUPPORTED, WORKSPACE = -1, -2, -5
BF16, FP16 = 0, 1
NULL = ctypes.c_void_p(0)


def _p(v=4096):
    return ctypes.c_void_p(v)          # non-null, 16-byte aligned, never dereferenced: validation runs before any CUDA call


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


SHAPE_CASES = [
    ("b = 0", dict(b=0), INVALID, b"shape"),
    ("lq = 0", dict(lq=0), INVALID, b"shape"),
    ("lk < 0", dict(lk=-5), INVALID, b"shape"),
    ("h = 0", dict(h=0), INVALID, b"shape"),
    ("d = 0", dict(d=0), INVALID, b"shape"),
    ("dtype tag", dict(dtype=7), UNSUPPORTED, b"dtype"),
    ("head dim 64", dict(d=64), UNSUPPORTED, b"head dim"),
    ("heads beyond the grid", dict(h=70000), UNSUPPORTED, b"too large"),
    ("batch beyond the grid", dict(b=70000), UNSUPPORTED, b"too large"),
    ("lq * h * d of 2^39 elements", dict(lq=1 << 30, h=4), UNSUPPORTED, b"too large"),
    ("lk * h * d of 2^39 elements", dict(lk=1 << 30, h=4), UNSUPPORTED, b"too large"),
]


def _pointer_cases(names, misaligned):
    return ([(f"null {n}", {n: NULL}, INVALID, b"null") for n in names] +
            [(f"misaligned {n}", {n: _p(misaligned.get(n, 4100))}, INVALID, b"aligned") for n in names])


# ------------------------------------------------------------------------------------------------ the two lse forwards
FWD_PTRS = ("q", "k", "v", "out", "lse")
JVP_PTRS = ("q", "k", "v", "q_t", "k_t", "v_t", "out", "out_t", "lse")
LSE_MISALIGNED = {"lse": 4098}          # fp32: 4-byte alignment is all lse needs


def _fwd_lse(lib, dtype=BF16, b=1, lq=256, lk=77, h=2, d=128, sm_scale=0.088, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in FWD_PTRS}
    return lib.tdb200_attn_dense_fwd_lse(a["q"], a["k"], a["v"], dtype, a["out"], a["lse"], b, lq, lk, h, d, sm_scale, None)


def _jvp_lse(lib, dtype=BF16, b=1, lq=256, lk=77, h=2, d=128, sm_scale=0.088, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in JVP_PTRS}
    return lib.tdb200_attn_dense_jvp_lse(a["q"], a["k"], a["v"], a["q_t"], a["k_t"], a["v_t"], dtype, a["out"], a["out_t"],
                                         a["lse"], b, lq, lk, h, d, sm_scale, None)


FWD_CASES = [("fwd_lse", _fwd_lse, b"attn_dense_fwd_lse:", *c) for c in _pointer_cases(FWD_PTRS, LSE_MISALIGNED) + SHAPE_CASES]
JVP_CASES = [("jvp_lse", _jvp_lse, b"attn_dense_jvp_lse:", *c) for c in _pointer_cases(JVP_PTRS, LSE_MISALIGNED) + SHAPE_CASES]


# ------------------------------------------------------------------------------------------------ the backward
BWD_PTRS = ("q", "k", "v", "out", "d_out", "lse", "dq", "dk", "dv", "workspace")
BWD_MISALIGNED = {"lse": 4098, "workspace": 4098}


def _ws(lib, b, h, lq):
    return lib.tdb200_attn_dense_bwd_workspace_bytes(b, h, lq)


def _bwd(lib, dtype=BF16, b=1, lq=256, lk=77, h=2, d=128, sm_scale=0.088, workspace_bytes=None, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in BWD_PTRS}
    if workspace_bytes is None:
        workspace_bytes = 1 << 40
    return lib.tdb200_attn_dense_bwd(a["q"], a["k"], a["v"], a["out"], a["d_out"], a["lse"], dtype, a["dq"], a["dk"], a["dv"],
                                     a["workspace"], workspace_bytes, b, lq, lk, h, d, sm_scale, None)


BWD_CASES = [("bwd", _bwd, b"attn_dense_bwd:", *c) for c in _pointer_cases(BWD_PTRS, BWD_MISALIGNED) + SHAPE_CASES + [
    # lq * h * d stays below 2^39, but b * lq * h rows exceed what the delta kernel's grid covers
    ("b * lq * h beyond the delta kernel's grid", dict(b=65535, lq=1 << 20, h=1), UNSUPPORTED, b"too large"),
]]

ALL = FWD_CASES + JVP_CASES + BWD_CASES


@pytest.mark.parametrize("entry,fn,prefix,name,kw,code,needle",
                         [pytest.param(*c, id=f"{c[0]}-{c[3]}".replace(" ", "-")) for c in ALL])
def test_argument_checks_return_codes(lib, entry, fn, prefix, name, kw, code, needle):
    rc = fn(lib, **kw)
    msg = lib.tdb200_last_error() or b""
    assert rc == code, (entry, name, rc, msg)
    assert msg.startswith(prefix) and needle in msg, (entry, name, msg)


@pytest.mark.parametrize("b,h,lq", [(1, 2, 256), (2, 12, 32760), (3, 40, 75600), (1, 1, 1)])
def test_workspace_holds_delta(lib, b, h, lq):
    assert _ws(lib, b, h, lq) == 4 * b * h * lq


def test_a_workspace_one_byte_short_is_refused(lib):
    need = _ws(lib, 2, 3, 333)
    rc = _bwd(lib, b=2, h=3, lq=333, workspace_bytes=need - 1)
    msg = lib.tdb200_last_error() or b""
    assert rc == WORKSPACE and msg.startswith(b"attn_dense_bwd:") and b"workspace" in msg, (rc, msg)


@pytest.mark.parametrize("b,h,lq,code", [(0, 2, 256, INVALID), (1, 0, 256, INVALID), (1, 2, 0, INVALID), (-1, 2, 256, INVALID),
                                         (1, 2, -7, INVALID), (70000, 2, 256, UNSUPPORTED), (1, 70000, 256, UNSUPPORTED),
                                         (1, 1, 1 << 31, UNSUPPORTED), (65535, 1, 1 << 20, UNSUPPORTED)],
                         ids=["b0", "h0", "lq0", "b-neg", "lq-neg", "b-grid", "h-grid", "lq-int32", "rows"])
def test_workspace_size_query_refuses_bad_shapes(lib, b, h, lq, code):
    assert _ws(lib, b, h, lq) == code
    assert (lib.tdb200_last_error() or b"").startswith(b"attn_dense_bwd_workspace_bytes:")


def test_valid_calls_without_a_gpu_report_an_error_code(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    for dtype in (BF16, FP16):
        for fn in (_fwd_lse, _jvp_lse, _bwd):
            rc = fn(lib, dtype=dtype)
            assert rc in (-3, -4) and lib.tdb200_last_error(), (fn.__name__, rc)


def test_abi_version_and_exports(lib):
    from turbodiffusion_b200 import _lib
    names = set(_lib.exported_names())
    assert {"tdb200_attn_dense_fwd_lse", "tdb200_attn_dense_jvp_lse", "tdb200_attn_dense_bwd",
            "tdb200_attn_dense_bwd_workspace_bytes"} <= names
    assert lib.tdb200_abi_version() == 2          # added symbols break no caller


# ------------------------------------------------------------------------------------------------ path selection
class _Recorder:
    """Stands in for the library: records which entry points are called and reports success."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append(name)
            return 256 if name.endswith("_workspace_bytes") else 0
        return fn


@pytest.fixture
def recorder(monkeypatch):
    from turbodiffusion_b200.ops import core
    rec = _Recorder()
    monkeypatch.setattr(core, "lib", lambda: rec)
    monkeypatch.setattr(core, "require_cuda", lambda *t: None)      # CPU tensors stand in for device tensors
    monkeypatch.setattr(core, "stream_ptr", lambda device=None: 0)
    return rec


def _qkv(dtype=None, grad=()):
    import torch
    dtype = dtype or torch.bfloat16
    q, k, v = torch.zeros(1, 5, 2, 128, dtype=dtype), torch.zeros(1, 3, 2, 128, dtype=dtype), torch.zeros(1, 3, 2, 128, dtype=dtype)
    for i in grad:
        (q, k, v)[i].requires_grad_()
    return q, k, v


def test_no_grad_calls_take_the_inference_entry_points(recorder):
    import torch
    from turbodiffusion_b200 import ops
    q, k, v = _qkv()
    ops.dense_attention(q, k, v)
    ops.dense_attention_jvp(q, k, v, q, k, v)
    q, k, v = _qkv(grad=(0, 1, 2))
    with torch.no_grad():
        out = ops.dense_attention(q, k, v)
        out2, _ = ops.dense_attention_jvp(q, k, v, q, k, v)
    assert not out.requires_grad and not out2.requires_grad
    assert recorder.calls == ["tdb200_attn_dense_fwd", "tdb200_attn_dense_jvp"] * 2


@pytest.mark.parametrize("which", [0, 1, 2], ids=["q", "k", "v"])
def test_grad_calls_take_the_lse_forward_and_the_dense_backward(recorder, which):
    from turbodiffusion_b200 import ops
    q, k, v = _qkv(grad=(which,))
    out = ops.dense_attention(q, k, v)
    assert recorder.calls == ["tdb200_attn_dense_fwd_lse"] and out.requires_grad
    out.float().sum().backward()
    assert recorder.calls[1:] == ["tdb200_attn_dense_bwd_workspace_bytes", "tdb200_attn_dense_bwd"]
    grad = (q, k, v)[which].grad
    assert grad is not None and grad.shape == (q, k, v)[which].shape and grad.dtype == (q, k, v)[which].dtype


@pytest.mark.parametrize("which", [0, 1, 2], ids=["q", "k", "v"])
def test_jvp_grad_calls_differentiate_out_and_not_out_t(recorder, which):
    import torch
    from turbodiffusion_b200 import ops
    q, k, v = _qkv(grad=(which,))
    q_t, k_t, v_t = (torch.zeros_like(t).requires_grad_() for t in (q, k, v))
    out, out_t = ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t)
    assert recorder.calls == ["tdb200_attn_dense_jvp_lse"]
    assert out.requires_grad and not out_t.requires_grad
    out.float().sum().backward()
    assert recorder.calls[1:] == ["tdb200_attn_dense_bwd_workspace_bytes", "tdb200_attn_dense_bwd"]
    assert (q, k, v)[which].grad is not None
    assert q_t.grad is None and k_t.grad is None and v_t.grad is None


def test_tangents_that_require_grad_do_not_select_the_training_path(recorder):
    import torch
    from turbodiffusion_b200 import ops
    q, k, v = _qkv()
    q_t, k_t, v_t = (torch.zeros_like(t).requires_grad_() for t in (q, k, v))
    out, out_t = ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t)
    assert recorder.calls == ["tdb200_attn_dense_jvp"] and not out.requires_grad and not out_t.requires_grad


def test_float32_inputs_get_float32_gradients(recorder):
    import torch
    from turbodiffusion_b200 import ops
    q, k, v = _qkv(dtype=torch.float32, grad=(0, 1, 2))
    out = ops.dense_attention(q, k, v)
    assert out.dtype == torch.float32
    out.sum().backward()
    assert all(t.grad.dtype == torch.float32 for t in (q, k, v))


@pytest.mark.parametrize("grad", [False, True], ids=["no-grad", "grad"])
def test_cpu_tensors_are_refused_on_both_paths(lib, grad):
    from turbodiffusion_b200 import _lib, ops
    q, k, v = _qkv(grad=(0, 1, 2) if grad else ())
    with pytest.raises(_lib.Tdb200Error, match="CUDA tensors only"):
        ops.dense_attention(q, k, v)
    with pytest.raises(_lib.Tdb200Error, match="CUDA tensors only"):
        ops.dense_attention_jvp(q, k, v, q.detach(), k.detach(), v.detach())
