"""CPU checks of the attention operators' forward-AD rules: the argument checks of tdb200_attn_dense_tangent and
tdb200_sla_attn16_tangent return their codes and a message naming the entry point before any CUDA call, and (with a recording
stand-in for the library) ops.dense_attention and SparseLinearAttention.forward with a forward-mode tangent call the lse forward
and then the tangent entry with that lse, never a JVP entry; calls without tangents make exactly the calls they made before;
refusals come before any library call."""
import ctypes

import pytest
import torch
import torch.autograd.forward_ad as fwAD

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


DENSE_PTRS = ("q", "k", "v", "q_t", "k_t", "v_t", "out", "lse", "out_t")
SLA_PTRS = ("q", "k", "v", "q_t", "k_t", "v_t", "o_s", "lse", "lut", "o_s_t")
MISALIGNED = {"lut": 4098, "lse": 4098}       # int32 / fp32: 4-byte alignment is all they need


def _dense(lib, dtype=BF16, b=1, lq=300, lk=200, h=2, d=128, sm_scale=0.088, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in DENSE_PTRS}
    return lib.tdb200_attn_dense_tangent(a["q"], a["k"], a["v"], a["q_t"], a["k_t"], a["v_t"], a["out"], a["lse"], dtype,
                                         a["out_t"], b, lq, lk, h, d, sm_scale, None)


def _sla(lib, dtype=BF16, topk=3, b=1, l=300, h=2, d=128, sm_scale=0.088, blkq=128, blkk=64, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in SLA_PTRS}
    return lib.tdb200_sla_attn16_tangent(a["q"], a["k"], a["v"], a["q_t"], a["k_t"], a["v_t"], a["o_s"], a["lse"], dtype, a["lut"],
                                         topk, a["o_s_t"], b, l, h, d, sm_scale, blkq, blkk, None)


def _pointer_cases(names):
    return ([(f"null {n}", {n: NULL}, INVALID, b"null") for n in names] +
            [(f"misaligned {n}", {n: _p(MISALIGNED.get(n, 4100))}, INVALID, b"aligned") for n in names])


DENSE_SHAPES = [
    ("b = 0", dict(b=0), INVALID, b"shape"),
    ("lq = 0", dict(lq=0), INVALID, b"shape"),
    ("lk < 0", dict(lk=-64), INVALID, b"shape"),
    ("h = 0", dict(h=0), INVALID, b"shape"),
    ("dtype tag", dict(dtype=7), UNSUPPORTED, b"dtype"),
    ("head dim 64", dict(d=64), UNSUPPORTED, b"head dim"),
    ("heads beyond the grid", dict(h=70000), UNSUPPORTED, b"too large"),
    ("batch beyond the grid", dict(b=70000), UNSUPPORTED, b"too large"),
    ("lq * h * d beyond the tensor map's stride", dict(lq=1 << 30, h=1024), UNSUPPORTED, b"too large"),
]
SLA_SHAPES = [
    ("b = 0", dict(b=0), INVALID, b"shape"),
    ("l = 0", dict(l=0), INVALID, b"shape"),
    ("h = 0", dict(h=0), INVALID, b"shape"),
    ("topk = 0", dict(topk=0), INVALID, b"topk"),
    ("topk > nblk", dict(topk=6), INVALID, b"topk"),          # l = 300: nblk = 5
    ("blocks (64, 64)", dict(blkq=64, blkk=64), UNSUPPORTED, b"block sizes"),
    ("blocks (64, 128)", dict(blkq=64, blkk=128), UNSUPPORTED, b"block sizes"),
    ("dtype tag", dict(dtype=7), UNSUPPORTED, b"dtype"),
    ("head dim 64", dict(d=64), UNSUPPORTED, b"head dim"),
    ("heads beyond the grid", dict(h=70000), UNSUPPORTED, b"too large"),
    ("topk beyond the on-chip LUT", dict(l=8641 * 64, topk=8641), UNSUPPORTED, b"LUT"),
]
CASES = ([("dense", _dense, b"attn_dense_tangent:", *c) for c in _pointer_cases(DENSE_PTRS) + DENSE_SHAPES] +
         [("sla", _sla, b"sla_attn16_tangent:", *c) for c in _pointer_cases(SLA_PTRS) + SLA_SHAPES])


@pytest.mark.parametrize("entry,fn,prefix,name,kw,code,needle",
                         [pytest.param(*c, id=f"{c[0]}-{c[3]}".replace(" ", "-")) for c in CASES])
def test_argument_checks_return_codes(lib, entry, fn, prefix, name, kw, code, needle):
    rc = fn(lib, **kw)
    msg = lib.tdb200_last_error() or b""
    assert rc == code, (entry, name, rc, msg)
    assert msg.startswith(prefix) and needle in msg, (entry, name, msg)


def test_the_largest_staged_lut_passes_validation(lib):
    """The sparse tangent at topk = 8640 ids (the LUT row fills the shared memory the kernel may use, jvp::kMaxLutIds) gets
    past validation; 8641 is refused (SLA_SHAPES)."""
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    rc = _sla(lib, l=8640 * 64, topk=8640)
    assert rc in (-3, -4) and lib.tdb200_last_error()


def test_valid_calls_without_a_gpu_report_an_error_code(lib):
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    for fn in (_dense, _sla):
        for dtype in (0, 1):
            rc = fn(lib, dtype=dtype)
            assert rc in (-3, -4) and lib.tdb200_last_error(), (fn.__name__, rc)


def test_abi_version_and_exports(lib):
    from turbodiffusion_b200 import _lib
    assert {"tdb200_attn_dense_tangent", "tdb200_sla_attn16_tangent"} <= set(_lib.exported_names())
    assert lib.tdb200_abi_version() == 2


# ------------------------------------------------------------------------------------------------ path selection
class _Recorder:
    """Stands in for the library: records the entry points called and their arguments, and reports success."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 0
        return fn

    def names(self):
        return [n for n, _ in self.calls]


L, H, D = 300, 2, 128          # nblk = 5 key blocks, mblk = 3 query blocks


class _Prep:
    nblk = (L + 63) // 64
    q_pool = k_pool = None


@pytest.fixture
def recorder(monkeypatch):
    """The library, the device checks and the block selection replaced by stand-ins, so both operators run on CPU tensors;
    the SLA lse forward and backward ops record themselves under their entry points' names, with the lse pointer."""
    from turbodiffusion_b200 import _ops
    from turbodiffusion_b200.ops import core as ops_core
    from turbodiffusion_b200.SLA import core
    rec = _Recorder()
    for mod in (core, ops_core):
        monkeypatch.setattr(mod, "lib", lambda: rec)
        monkeypatch.setattr(mod, "require_cuda", lambda *t: None)
        monkeypatch.setattr(mod, "stream_ptr", lambda device=None: 0)
    monkeypatch.setattr(core, "select_prep", lambda q, k, blkq, blkk: _Prep())

    def block_map(q_pool, k_pool, topk):
        lut = torch.arange(topk, dtype=torch.int32).expand(1, H, 3, topk).contiguous()
        return torch.zeros(1, H, 3, _Prep.nblk, dtype=torch.int8), lut
    monkeypatch.setattr(core, "block_map_from_pools", block_map)

    def sla_fwd_lse(q, k, v, lut, topk, sm_scale, blkq):
        lse = torch.zeros(q.shape[0], q.shape[2], q.shape[1])
        rec.calls.append(("tdb200_sla_attn16_fwd_lse", (lse.data_ptr(), topk, blkq)))
        return torch.zeros_like(q), lse
    monkeypatch.setattr(_ops, "sla_attn16_fwd_lse", sla_fwd_lse)

    def sla_bwd(q, k, v, o_s, d_o, lse, lut, topk, sm_scale, blkq):
        rec.calls.append(("tdb200_sla_attn16_bwd", (lse.data_ptr(), topk, blkq)))
        return torch.ones_like(q), torch.ones_like(k), torch.ones_like(v)
    monkeypatch.setattr(_ops, "sla_attn16_bwd", sla_bwd)
    return rec


def _module(**kw):
    from turbodiffusion_b200.SLA import SparseLinearAttention
    return SparseLinearAttention(D, 0.5, **{"BLKQ": 128, "BLKK": 64, **kw})


def _qkv(lq=L, lk=L, d=D, grad=()):
    q, k, v = (torch.randn(1, n, H, d, dtype=torch.bfloat16) for n in (lq, lk, lk))
    for i in grad:
        (q, k, v)[i].requires_grad_()
    return q, k, v


def _dense_attention(q, k, v):
    from turbodiffusion_b200 import ops
    return ops.dense_attention(q, k, v)


def _lse_arg(rec, name, index):
    return next(args[index] for n, args in rec.calls if n == name)


@pytest.mark.parametrize("how", ["forward_ad", "func.jvp"])
def test_dense_tangent_calls_fwd_lse_then_the_tangent_entry_with_its_lse(recorder, how):
    q, k, v = _qkv(lq=200)
    if how == "forward_ad":
        with fwAD.dual_level():
            out = _dense_attention(fwAD.make_dual(q, torch.randn_like(q)), k, v)
            out, out_t = fwAD.unpack_dual(out)
    else:
        out, out_t = torch.func.jvp(_dense_attention, (q, k, v), (torch.randn_like(q), torch.randn_like(k), torch.randn_like(v)))
    assert recorder.names() == ["tdb200_attn_dense_fwd_lse", "tdb200_attn_dense_tangent"]
    lse = _lse_arg(recorder, "tdb200_attn_dense_fwd_lse", 5)
    out_ptr = _lse_arg(recorder, "tdb200_attn_dense_fwd_lse", 4)
    args = recorder.calls[1][1]
    assert args[6] == out_ptr and args[7] == lse           # the forward's out and lse
    assert args[10:15] == (1, 200, L, H, D)
    assert out_t is not None and out_t.shape == out.shape == q.shape and out_t.dtype == q.dtype


def test_dense_missing_tangents_are_zeros(recorder):
    q, k, v = _qkv()
    with fwAD.dual_level():
        out = _dense_attention(q, fwAD.make_dual(k, torch.randn_like(k)), v)
        assert fwAD.unpack_dual(out).tangent is not None
    assert recorder.names() == ["tdb200_attn_dense_fwd_lse", "tdb200_attn_dense_tangent"]


def test_dense_under_forward_ad_with_grad_uses_the_dense_backward(recorder, monkeypatch):
    from turbodiffusion_b200.ops import core as ops_core
    monkeypatch.setattr(ops_core, "_dense_bwd", lambda ctx, d: (recorder.calls.append(("tdb200_attn_dense_bwd", ())),
                                                                *(torch.ones_like(t) for t in ctx.saved_tensors[:3]))[1:])
    q, k, v = _qkv(grad=(0,))
    with fwAD.dual_level():
        out = _dense_attention(fwAD.make_dual(q, torch.randn_like(q)), k, v)
        primal, tangent = fwAD.unpack_dual(out)
        assert primal.requires_grad and not tangent.requires_grad
        primal.float().sum().backward()
    assert recorder.names() == ["tdb200_attn_dense_fwd_lse", "tdb200_attn_dense_tangent", "tdb200_attn_dense_bwd"]
    assert q.grad is not None


def test_dense_without_tangents_makes_todays_calls(recorder):
    q, k, v = _qkv()
    _dense_attention(q, k, v)
    with fwAD.dual_level():                                 # a level with no dual input is no tangent
        _dense_attention(q, k, v)
    q.requires_grad_()
    _dense_attention(q, k, v)
    assert recorder.names() == ["tdb200_attn_dense_fwd", "tdb200_attn_dense_fwd", "tdb200_attn_dense_fwd_lse"]


@pytest.mark.parametrize("how", ["forward_ad", "func.jvp"])
def test_sla_tangent_calls_fwd_lse_then_the_tangent_entry_with_its_lse(recorder, how):
    mod = _module()
    q, k, v = _qkv()
    if how == "forward_ad":
        with fwAD.dual_level():
            o = mod(fwAD.make_dual(q, torch.randn_like(q)), k, v)
            o, o_t = fwAD.unpack_dual(o)
    else:
        o, o_t = torch.func.jvp(mod, (q, k, v), (torch.randn_like(q), torch.randn_like(k), torch.randn_like(v)))
    assert recorder.names() == ["tdb200_sla_attn16_fwd_lse", "tdb200_sla_attn16_tangent"]
    lse = _lse_arg(recorder, "tdb200_sla_attn16_fwd_lse", 0)
    args = recorder.calls[1][1]
    assert args[7] == lse and args[10] == 2 and args[17:19] == (128, 64)   # the forward's lse, topk = int(0.5 * 5), blocks
    assert o_t is not None and o_t.shape == o.shape == q.shape and o_t.dtype == q.dtype


def test_sla_under_forward_ad_with_grad_uses_the_sla_backward_with_the_forwards_lse(recorder):
    mod = _module()
    q, k, v = _qkv(grad=(0, 1, 2))
    with fwAD.dual_level():
        o = mod(fwAD.make_dual(q, torch.randn_like(q)), k, v)
        primal, tangent = fwAD.unpack_dual(o)
        assert primal.requires_grad        # (the linear branch's tangent is torch's own, with its graph through proj_l)
        primal.float().sum().backward()
    assert recorder.names() == ["tdb200_sla_attn16_fwd_lse", "tdb200_sla_attn16_tangent", "tdb200_sla_attn16_bwd"]
    assert recorder.calls[2][1] == (_lse_arg(recorder, "tdb200_sla_attn16_fwd_lse", 0), 2, 128)
    assert q.grad is not None and mod.proj_l.weight.grad is not None


def test_sla_without_tangents_makes_todays_calls(recorder, monkeypatch):
    from turbodiffusion_b200.SLA import core
    monkeypatch.setattr(core, "attn_fwd_qk16", lambda *a, **kw: (recorder.calls.append(("tdb200_sla_attn16_fwd", ())),
                                                                 torch.zeros_like(a[0]))[1])
    monkeypatch.setattr(core, "linear_moments", lambda k, v, f: (None, None))
    monkeypatch.setattr(core, "project_moments", lambda w, kv, dtype: None)
    mod = _module()
    q, k, v = _qkv()
    mod(q, k, v)
    q.requires_grad_()
    mod(q, k, v)
    assert recorder.names() == ["tdb200_sla_attn16_fwd", "tdb200_sla_attn16_fwd_lse"]


@pytest.mark.parametrize("how", ["forward_ad", "func.jvp"])
def test_sla_keeps_the_selection_and_returns_the_sparsity(recorder, how):
    mod = _module()
    q, k, v = _qkv()
    mod._keep_selection = {}
    if how == "forward_ad":
        with fwAD.dual_level():
            o, sparsity = mod(fwAD.make_dual(q, torch.randn_like(q)), k, v, return_sparsity=True)
    else:
        out = {}
        torch.func.jvp(lambda x: out.setdefault("o", mod(x, k, v, return_sparsity=True))[0], (q,), (torch.randn_like(q),))
        sparsity = out["o"][1]
    assert sparsity == 2 / 5 and mod._keep_selection["topk"] == 2 and mod._keep_selection["lut"].shape == (1, H, 3, 2)


@pytest.mark.parametrize("case", ["head dim 64", "blocks (64, 64)", "blocks (64, 128)", "sage"])
def test_refusals_come_before_any_library_call(recorder, monkeypatch, case):
    from turbodiffusion_b200.SLA import SageSparseLinearAttention, SparseLinearAttention, core
    calls = []
    for name in ("select_prep", "block_map_from_pools", "require_cuda"):
        monkeypatch.setattr(core, name, lambda *a, _n=name, **kw: calls.append(_n))
    d = 64 if case == "head dim 64" else D
    if case == "sage":
        mod = SageSparseLinearAttention(D, 0.5)
    elif case == "head dim 64":
        mod = SparseLinearAttention(64, 0.5, BLKQ=128, BLKK=64)
    else:
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mod = _module(BLKQ=64, BLKK=64 if case == "blocks (64, 64)" else 128)
    q, k, v = _qkv(d=d)
    with pytest.raises(NotImplementedError, match="forward-mode tangent"):
        torch.func.jvp(mod, (q, k, v), (torch.randn_like(q), torch.randn_like(k), torch.randn_like(v)))
    with fwAD.dual_level(), pytest.raises(NotImplementedError, match="forward-mode tangent"):
        mod(q, k, fwAD.make_dual(v, torch.randn_like(v)))
    assert recorder.calls == [] and calls == []
