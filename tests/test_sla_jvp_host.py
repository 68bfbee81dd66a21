"""CPU checks of the sparse attention JVP: the argument checks of tdb200_sla_attn16_jvp and tdb200_sla_attn16_jvp_lse return
their codes and a message naming the entry point before any CUDA call, a well-formed call on a host without a GPU comes back
with an error code, and SparseLinearAttention.forward_jvp picks its entry point by grad mode and requires_grad, sends the
gradient of o through the SLA backward with the lse of the JVP's forward, and refuses what it does not serve before any library
call (checked with a recording stand-in for the library)."""
import ctypes

import pytest
import torch

INVALID, UNSUPPORTED = -1, -2
BF16, FP16 = 0, 1
NULL = ctypes.c_void_p(0)


def _p(v=4096):
    return ctypes.c_void_p(v)          # non-null, 16-byte aligned, never dereferenced: validation runs before any CUDA call


@pytest.fixture(scope="module")
def lib():
    from turbodiffusion_b200 import _build, _lib
    _build.build()
    return _lib.lib()


PTRS = ("q", "k", "v", "q_t", "k_t", "v_t", "lut", "o_s", "o_s_t")
LSE_PTRS = PTRS + ("lse",)
MISALIGNED = {"lut": 4098, "lse": 4098}       # int32 / fp32: 4-byte alignment is all they need


def _jvp(lib, dtype=BF16, topk=3, b=1, l=300, h=2, d=128, sm_scale=0.088, blkq=128, blkk=64, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in PTRS}
    return lib.tdb200_sla_attn16_jvp(a["q"], a["k"], a["v"], a["q_t"], a["k_t"], a["v_t"], dtype, a["lut"], topk, a["o_s"],
                                     a["o_s_t"], b, l, h, d, sm_scale, blkq, blkk, None)


def _jvp_lse(lib, dtype=BF16, topk=3, b=1, l=300, h=2, d=128, sm_scale=0.088, blkq=128, blkk=64, **ptrs):
    a = {n: ptrs.get(n, _p()) for n in LSE_PTRS}
    return lib.tdb200_sla_attn16_jvp_lse(a["q"], a["k"], a["v"], a["q_t"], a["k_t"], a["v_t"], dtype, a["lut"], topk, a["o_s"],
                                         a["o_s_t"], a["lse"], b, l, h, d, sm_scale, blkq, blkk, None)


def _pointer_cases(names):
    return ([(f"null {n}", {n: NULL}, INVALID, b"null") for n in names] +
            [(f"misaligned {n}", {n: _p(MISALIGNED.get(n, 4100))}, INVALID, b"aligned") for n in names])


SHAPE_CASES = [
    ("b = 0", dict(b=0), INVALID, b"shape"),
    ("l = 0", dict(l=0), INVALID, b"shape"),
    ("l < 0", dict(l=-64), INVALID, b"shape"),
    ("h = 0", dict(h=0), INVALID, b"shape"),
    ("d = 0", dict(d=0), INVALID, b"shape"),
    ("topk = 0", dict(topk=0), INVALID, b"topk"),
    ("topk < 0", dict(topk=-1), INVALID, b"topk"),
    ("topk > nblk", dict(topk=6), INVALID, b"topk"),          # l = 300: nblk = 5
    ("blocks (64, 64)", dict(blkq=64, blkk=64), UNSUPPORTED, b"block sizes"),
    ("blocks (64, 128)", dict(blkq=64, blkk=128), UNSUPPORTED, b"block sizes"),
    ("blocks (128, 128)", dict(blkq=128, blkk=128), UNSUPPORTED, b"block sizes"),
    ("dtype tag", dict(dtype=7), UNSUPPORTED, b"dtype"),
    ("head dim 64", dict(d=64), UNSUPPORTED, b"head dim"),
    ("heads beyond the grid", dict(h=70000), UNSUPPORTED, b"too large"),
    ("batch beyond the grid", dict(b=70000), UNSUPPORTED, b"too large"),
    ("l * h * d beyond the tensor map's stride", dict(l=1 << 30, h=1024), UNSUPPORTED, b"too large"),
    ("topk beyond the on-chip LUT", dict(l=8641 * 64, topk=8641), UNSUPPORTED, b"LUT"),
]

CASES = ([("jvp", _jvp, b"sla_attn16_jvp:", *c) for c in _pointer_cases(PTRS) + SHAPE_CASES] +
         [("jvp_lse", _jvp_lse, b"sla_attn16_jvp_lse:", *c) for c in _pointer_cases(LSE_PTRS) + SHAPE_CASES])


@pytest.mark.parametrize("entry,fn,prefix,name,kw,code,needle",
                         [pytest.param(*c, id=f"{c[0]}-{c[3]}".replace(" ", "-")) for c in CASES])
def test_argument_checks_return_codes(lib, entry, fn, prefix, name, kw, code, needle):
    rc = fn(lib, **kw)
    msg = lib.tdb200_last_error() or b""
    assert rc == code, (entry, name, rc, msg)
    assert msg.startswith(prefix) and needle in msg, (entry, name, msg)


def test_the_largest_staged_lut_passes_validation(lib):
    """topk = 8640 ids (the LUT row fills the shared memory the kernel may use) gets past validation."""
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    rc = _jvp(lib, l=8640 * 64, topk=8640)
    assert rc in (-3, -4) and lib.tdb200_last_error()


def test_valid_calls_without_a_gpu_report_an_error_code(lib):
    if torch.cuda.is_available():
        pytest.skip("this check is for hosts without a GPU")
    for dtype in (BF16, FP16):
        for fn in (_jvp, _jvp_lse):
            rc = fn(lib, dtype=dtype)
            assert rc in (-3, -4) and lib.tdb200_last_error(), (fn.__name__, rc)


def test_abi_version_and_exports(lib):
    from turbodiffusion_b200 import _lib
    assert {"tdb200_sla_attn16_jvp", "tdb200_sla_attn16_jvp_lse"} <= set(_lib.exported_names())
    assert lib.tdb200_abi_version() == 2          # added symbols break no caller


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
    """The library, the device checks and the block selection replaced by stand-ins, so forward_jvp runs on CPU tensors;
    the SLA backward op records itself under its entry point's name with the lse it was handed."""
    from turbodiffusion_b200 import _ops
    from turbodiffusion_b200.SLA import core
    rec = _Recorder()
    monkeypatch.setattr(core, "lib", lambda: rec)
    monkeypatch.setattr(core, "require_cuda", lambda *t: None)
    monkeypatch.setattr(core, "stream_ptr", lambda device=None: 0)
    monkeypatch.setattr(core, "select_prep", lambda q, k, blkq, blkk: _Prep())

    def block_map(q_pool, k_pool, topk):
        lut = torch.arange(topk, dtype=torch.int32).expand(1, H, 3, topk).contiguous()
        return torch.zeros(1, H, 3, _Prep.nblk, dtype=torch.int8), lut
    monkeypatch.setattr(core, "block_map_from_pools", block_map)

    def sla_bwd(q, k, v, o_s, d_o, lse, lut, topk, sm_scale, blkq):
        rec.calls.append(("tdb200_sla_attn16_bwd", (lse.data_ptr(), topk, blkq)))
        return torch.ones_like(q), torch.ones_like(k), torch.ones_like(v)
    monkeypatch.setattr(_ops, "sla_attn16_bwd", sla_bwd)
    return rec


def _module(**kw):
    from turbodiffusion_b200.SLA import SparseLinearAttention
    return SparseLinearAttention(D, 0.5, **{"BLKQ": 128, "BLKK": 64, **kw})


def _qkv(grad=(), d=D):
    q, k, v = (torch.randn(1, L, H, d, dtype=torch.bfloat16) for _ in range(3))
    for i in grad:
        (q, k, v)[i].requires_grad_()
    return q, k, v


def _tangents(q, k, v, grad=False):
    return tuple(torch.randn_like(t).requires_grad_(grad) for t in (q, k, v))


def test_without_grad_forward_jvp_calls_the_jvp_entry_point(recorder):
    mod = _module()
    q, k, v = _qkv()
    o, o_t = mod.forward_jvp(q, k, v, *_tangents(q, k, v))
    q, k, v = _qkv(grad=(0, 1, 2))
    with torch.no_grad():
        o2, o2_t = mod.forward_jvp(q, k, v, *_tangents(q, k, v))
    assert recorder.names() == ["tdb200_sla_attn16_jvp"] * 2
    assert not o2.requires_grad and not o2_t.requires_grad and not o_t.requires_grad
    assert o.shape == o_t.shape == q.shape and o.dtype == o_t.dtype == q.dtype
    name, args = recorder.calls[0]
    assert args[8] == 2 and args[16:18] == (128, 64)       # topk = int(0.5 * 5), (blkq, blkk)


def test_tangents_that_require_grad_do_not_select_the_training_path(recorder):
    mod = _module()
    q, k, v = _qkv()
    o, o_t = mod.forward_jvp(q, k, v, *_tangents(q, k, v, grad=True))
    assert recorder.names() == ["tdb200_sla_attn16_jvp"] and not o_t.requires_grad


@pytest.mark.parametrize("which", [0, 1, 2], ids=["q", "k", "v"])
def test_with_grad_forward_jvp_calls_the_lse_entry_and_the_sla_backward_with_its_lse(recorder, which):
    mod = _module()
    q, k, v = _qkv(grad=(which,))
    q_t, k_t, v_t = _tangents(q, k, v, grad=True)
    o, o_t = mod.forward_jvp(q, k, v, q_t, k_t, v_t)
    assert recorder.names() == ["tdb200_sla_attn16_jvp_lse"]
    assert o.requires_grad and not o_t.requires_grad and o_t.grad_fn is None
    lse_ptr = recorder.calls[0][1][11]
    o.float().sum().backward()
    assert recorder.names()[1:] == ["tdb200_sla_attn16_bwd"]
    assert recorder.calls[1][1] == (lse_ptr, 2, 128)       # the lse the JVP's forward wrote
    grad = (q, k, v)[which].grad
    assert grad is not None and grad.shape == q.shape and grad.dtype == q.dtype
    assert q_t.grad is None and k_t.grad is None and v_t.grad is None
    assert mod.proj_l.weight.grad is not None and mod.proj_l.bias.grad is not None


def test_o_t_carries_no_gradient_and_its_loss_reaches_no_backward(recorder):
    mod = _module()
    q, k, v = _qkv(grad=(0, 1, 2))
    o, o_t = mod.forward_jvp(q, k, v, *_tangents(q, k, v))
    assert not o_t.requires_grad
    (o.float() * o_t.float()).sum().backward()                # o_t enters as a constant
    assert recorder.names() == ["tdb200_sla_attn16_jvp_lse", "tdb200_sla_attn16_bwd"]


def test_sparse_attention16_jvp_marks_o_s_t_non_differentiable(recorder):
    from turbodiffusion_b200.SLA import core
    q, k, v = _qkv(grad=(0,))
    lut = torch.zeros(1, H, 3, 1, dtype=torch.int32)
    o_s, o_s_t = core.sparse_attention16_jvp(q, k, v, q.detach(), k, v, lut, 1, D ** -0.5)
    assert o_s.requires_grad and not o_s_t.requires_grad
    assert recorder.names() == ["tdb200_sla_attn16_jvp_lse"]


def test_return_sparsity(recorder):
    q, k, v = _qkv()
    o, o_t, sparsity = _module().forward_jvp(q, k, v, *_tangents(q, k, v), return_sparsity=True)
    assert sparsity == 2 / 5


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
    q, k, v = _qkv(grad=(0,), d=d)
    with pytest.raises(NotImplementedError):
        mod.forward_jvp(q, k, v, *_tangents(q, k, v))
    assert recorder.calls == [] and calls == []


@pytest.mark.parametrize("which", [0, 1, 2], ids=["q_t", "k_t", "v_t"])
def test_tangents_of_another_shape_are_refused(recorder, which):
    q, k, v = _qkv()
    tangents = list(_tangents(q, k, v))
    tangents[which] = torch.zeros(1, L + 1, H, D, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match=["q_t", "k_t", "v_t"][which]):
        _module().forward_jvp(q, k, v, *tangents)
    assert recorder.calls == []


def test_forward_jvp_refuses_cpu_tensors(lib):
    from turbodiffusion_b200 import _lib
    q, k, v = _qkv()
    with pytest.raises(_lib.Tdb200Error, match="CUDA tensors only"):
        _module().forward_jvp(q, k, v, q, k, v)


def test_the_training_forward_is_unchanged_by_the_shared_linear_branch():
    """_linear_branch is _forward_train's linear branch; on float64 CPU tensors it is the reference formula of SLA/core.py."""
    torch.manual_seed(0)
    mod = _module()
    with torch.no_grad():
        mod.proj_l.weight.normal_()
        mod.proj_l.bias.normal_()
    mod.dtype = torch.float64
    q, k, v = (torch.randn(1, 40, H, D, dtype=torch.float64) for _ in range(3))
    qh, kh, vh = (t.transpose(1, 2) for t in (q, k, v))
    c_q, c_k = torch.softmax(qh, -1), torch.softmax(kh, -1)
    want = (c_q @ (c_k.transpose(-1, -2) @ vh)) / (1e-5 + (c_q * c_k.sum(-2, keepdim=True)).sum(-1, keepdim=True))
    want = torch.nn.functional.linear(want, mod.proj_l.weight.double(), mod.proj_l.bias.double()).transpose(1, 2)
    torch.testing.assert_close(mod._linear_branch(q, k, v), want, rtol=1e-12, atol=1e-12)
