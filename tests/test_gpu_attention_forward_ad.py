"""GPU checks of the attention operators' forward-AD rules (torch.func.jvp and torch.autograd.forward_ad through
ops.dense_attention and SparseLinearAttention.forward), and of the tangent kernels behind them (tdb200_attn_dense_tangent,
tdb200_sla_attn16_tangent), which compute the tangent from the lse forward's saved output and lse.

Bars are those of tests/test_gpu_dense_attention_jvp.py and tests/test_gpu_sla_jvp.py: the tangent's rel-L2 against float64
torch.func.jvp at most 1.5x that of the float32 restatement of the fused JVP kernel's rounding, plus 1e-7.  The primal is
bit-identical to the operator's ordinary output (dense) or to the training forward's (sparse)."""
import pytest
import torch
import torch.autograd.forward_ad as fwAD

import test_gpu_dense_attention_jvp as DJ
import test_gpu_sla_jvp as SJ

pytestmark = pytest.mark.gpu
D, BQ, BK = 128, 128, 64
SM = D ** -0.5
BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]


def SJ_core():
    from turbodiffusion_b200.SLA import core
    return core


def _dense(q, k, v):
    from turbodiffusion_b200 import ops
    return ops.dense_attention(q, k, v)


def _func_jvp(fn, ins):
    return torch.func.jvp(fn, tuple(ins[:3]), tuple(ins[3:]))


def _forward_ad(fn, ins):
    with fwAD.dual_level():
        out = fn(*(fwAD.make_dual(p, t) for p, t in zip(ins[:3], ins[3:])))
        return fwAD.unpack_dual(out)


def _dense_tangent(ins, out, lse, sm_scale=SM, out_t=None):
    """tdb200_attn_dense_tangent on the C ABI"""
    from turbodiffusion_b200 import _lib
    q, k = ins[0], ins[1]
    out_t = torch.empty_like(q) if out_t is None else out_t
    _lib.check(_lib.lib().tdb200_attn_dense_tangent(*(t.data_ptr() for t in ins), out.data_ptr(), lse.data_ptr(),
                                                    _lib.DTYPE_TAG[q.dtype], out_t.data_ptr(), q.shape[0], q.shape[1], k.shape[1],
                                                    q.shape[2], D, sm_scale, _lib.stream_ptr(q.device)), "attn_dense_tangent")
    return out_t


def _dense_fwd_lse(q, k, v, sm_scale=SM):
    from turbodiffusion_b200 import _lib
    b, lq, h, _ = q.shape
    out, lse = torch.empty_like(q), torch.empty(b, h, lq, dtype=torch.float32, device=q.device)
    _lib.check(_lib.lib().tdb200_attn_dense_fwd_lse(q.data_ptr(), k.data_ptr(), v.data_ptr(), _lib.DTYPE_TAG[q.dtype], out.data_ptr(),
                                                    lse.data_ptr(), b, lq, k.shape[1], h, D, sm_scale, _lib.stream_ptr(q.device)),
               "attn_dense_fwd_lse")
    return out, lse


def _sla_tangent(ins, o_s, lse, lut, o_s_t=None):
    from turbodiffusion_b200 import _lib
    q = ins[0]
    b, l, h, _ = q.shape
    o_s_t = torch.empty_like(q) if o_s_t is None else o_s_t
    _lib.check(_lib.lib().tdb200_sla_attn16_tangent(*(t.data_ptr() for t in ins), o_s.data_ptr(), lse.data_ptr(),
                                                    _lib.DTYPE_TAG[q.dtype], lut.data_ptr(), lut.shape[-1], o_s_t.data_ptr(), b, l, h,
                                                    D, SM, BQ, BK, _lib.stream_ptr(q.device)), "sla_attn16_tangent")
    return o_s_t


# ------------------------------------------------------------------------------------------------ dense: float64
LENGTHS = (1, 77, 226, 512, 1000)
DENSE_CASES = [(1 + i % 2, 1 + i % 3, lq, lk) for i, (lq, lk) in enumerate((lq, lk) for lq in LENGTHS for lk in LENGTHS)]


@pytest.mark.parametrize("how", ["func.jvp", "forward_ad"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,lq,lk", [pytest.param(*c, id="b{}h{}-{}x{}".format(*c)) for c in DENSE_CASES])
def test_dense_primal_bits_and_tangent_against_float64(cuda, b, h, lq, lk, dtype, how):
    ins = DJ._inputs(b, lq, lk, h, dtype, seed=1000 * lq + lk + 7)
    out, out_t = (_func_jvp if how == "func.jvp" else _forward_ad)(_dense, ins)
    assert out.shape == out_t.shape == ins[0].shape and out.dtype == out_t.dtype == dtype
    assert torch.equal(out, _dense(*ins[:3]))
    DJ._check_tangent(out_t, ins, f"({b}, {h}, {lq}, {lk}) {dtype} {how}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_partial_tangent_cross_attention(cuda, dtype):
    """q_t only (k_t = v_t = 0: the text keys of cross-attention carry no tangent), through torch.func.jvp of q alone."""
    q, k, v, q_t, _, _ = DJ._inputs(2, 1000, 512, 3, dtype, seed=5)
    out, out_t = torch.func.jvp(lambda x: _dense(x, k, v), (q,), (q_t,))
    assert torch.equal(out, _dense(q, k, v))
    DJ._check_tangent(out_t, [q, k, v, q_t, torch.zeros_like(k), torch.zeros_like(v)], f"q_t only {dtype}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_large_scores(cuda, dtype):
    """Rows whose log2-domain scores reach 300 and more, so lse is far from 0 (DJ's large-score construction)."""
    import math
    lq, lk, h = 700, 1000, 2
    g = torch.Generator().manual_seed(11)
    u = torch.ones(D) / D ** 0.5
    q, k, v = torch.randn(1, lq, h, D, generator=g), torch.randn(1, lk, h, D, generator=g), torch.randn(1, lk, h, D, generator=g)
    q = 8.0 * (q - (q @ u)[..., None] * u) + 4.0 * u
    k = k + (30.0 * (torch.arange(lk) // BK) / (4.0 * SM / math.log(2.0)))[None, :, None, None] * u
    q_t = torch.randn(1, lq, h, D, generator=g)
    q_t = q_t - (q_t @ u)[..., None] * u
    k_t, v_t = 0.125 * torch.randn(1, lk, h, D, generator=g), torch.randn(1, lk, h, D, generator=g)
    ins = [t.to(dtype).cuda() for t in (q, k, v, q_t, k_t, v_t)]
    out, out_t = _func_jvp(_dense, ins)
    assert _dense_fwd_lse(*ins[:3])[1].amin() > 300
    ours, _ = DJ._check_tangent(out_t, ins, f"large scores {dtype}")
    assert ours <= DJ.REL


# ------------------------------------------------------------------------------------------------ dense: memory, bits, graphs
@pytest.mark.parametrize("poison", [float("nan"), 1e4], ids=["nan", "1e4"])
def test_dense_memory_beyond_lk_and_rows_beyond_lq(cuda, poison):
    """k, v, k_t, v_t as the first lk rows of poisoned allocations give the bits of tight copies; out_t rows >= lq keep their
    sentinel, and lse entries past lq (never read) may hold anything."""
    lq, lk, h, extra = 333, 130, 2, 120
    ins = DJ._inputs(1, lq, lk, h, BF16, seed=lk)
    views = list(ins)
    for i in (1, 2, 4, 5):
        big = torch.full((1, 256, h, D), poison, dtype=BF16, device="cuda")
        big[:, :lk] = ins[i]
        views[i] = big[:, :lk]
    out, lse = _dense_fwd_lse(*ins[:3])
    want = _dense_tangent(ins, out, lse)
    big_t = torch.full((1, lq + extra, h, D), 7.0, dtype=BF16, device="cuda")
    _dense_tangent(views, out, lse, out_t=big_t)
    assert torch.equal(big_t[:, :lq], want) and (big_t[:, lq:] == 7.0).all() and torch.isfinite(want).all()
    assert torch.equal(want, _func_jvp(_dense, ins)[1])


@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_bits_reproducible_and_independent_of_the_other_heads(cuda, dtype):
    ins = DJ._inputs(2, 700, 300, 3, dtype, seed=31)
    out, out_t = _func_jvp(_dense, ins)
    again, again_t = _func_jvp(_dense, ins)
    assert torch.equal(out, again) and torch.equal(out_t, again_t)
    one, one_t = _func_jvp(_dense, [t[1:2, :, 2:3].contiguous() for t in ins])
    assert torch.equal(one, out[1:2, :, 2:3]) and torch.equal(one_t, out_t[1:2, :, 2:3])


def test_dense_cuda_graph_replay_of_forward_lse_and_tangent(cuda):
    ins = DJ._inputs(1, 900, 512, 2, BF16, seed=41)
    out, lse = _dense_fwd_lse(*ins[:3])
    eager_t = _dense_tangent(ins, out, lse)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out, g_lse = _dense_fwd_lse(*ins[:3])
        g_t = _dense_tangent(ins, g_out, g_lse)
    g_out.zero_(), g_lse.zero_(), g_t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g_out, out) and torch.equal(g_lse, lse) and torch.equal(g_t, eager_t)


@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_gradients_under_forward_ad_equal_the_training_path(cuda, dtype):
    ins = DJ._inputs(1, 500, 300, 2, dtype, seed=61)
    gout = torch.randn(ins[0].shape, generator=torch.Generator().manual_seed(62)).to(dtype).cuda()
    leaves = [t.clone().requires_grad_() for t in ins[:3]]
    with fwAD.dual_level():
        out = _dense(*(fwAD.make_dual(p, t) for p, t in zip(leaves, ins[3:])))
        primal, tangent = fwAD.unpack_dual(out)
        assert not tangent.requires_grad
        primal.backward(gout)
    plain = [t.clone().requires_grad_() for t in ins[:3]]
    _dense(*plain).backward(gout)
    for a, b in zip(leaves, plain):
        assert torch.equal(a.grad, b.grad)


def test_dense_shape_a_on_sampled_rows(cuda):
    """Shape A's cross-attention: 32760 queries, 12 heads, 512 keys; 64 sampled rows per head against float64."""
    lq, lk, h, n = 32760, 512, 12, 64
    g = torch.Generator(device="cuda").manual_seed(51)
    q, q_t = (torch.randn(1, lq, h, D, generator=g, device="cuda").bfloat16() for _ in range(2))
    k, v, k_t, v_t = (torch.randn(1, lk, h, D, generator=g, device="cuda").bfloat16() for _ in range(4))
    out, out_t = _func_jvp(_dense, [q, k, v, q_t, k_t, v_t])
    assert torch.isfinite(out_t).all()
    rows = torch.stack([torch.randperm(lq, generator=torch.Generator().manual_seed(60 + i))[:n] for i in range(h)]).cuda()
    rows[:, 0], rows[:, 1] = 0, lq - 1
    heads = torch.arange(h, device="cuda")[:, None]
    pick = lambda t: t[0][rows, heads].transpose(0, 1)[None]
    DJ._check_tangent(pick(out_t), [pick(q), k, v, pick(q_t), k_t, v_t], "shape A cross, sampled rows")


# ------------------------------------------------------------------------------------------------ sparse: the kernel
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,l,topk,tail", SJ.RANDOM_CASES)
def test_sla_tangent_kernel_against_float64(cuda, b, h, l, topk, tail, dtype):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    ins = SJ._inputs(b, l, h, dtype, seed=7 * l + topk + 1)
    lut = SJ._random_lut(b, h, l, topk, seed=l + topk + 1, tail=tail)
    o_s, lse = attn_fwd_qk16_lse(*ins[:3], lut, topk, SM)
    o_s_t = _sla_tangent(ins, o_s, lse, lut)
    SJ._check(o_s, o_s_t, ins, SJ._mask(lut, l), f"({b}, {h}, {l}) topk {topk} tail {tail} {dtype}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_sla_tangent_kernel_large_scores(cuda, dtype):
    import math
    l, h, topk = 1000, 2, 9
    g = torch.Generator().manual_seed(11)
    u = torch.ones(D) / D ** 0.5
    q, k, v = (torch.randn(1, l, h, D, generator=g) for _ in range(3))
    q = 8.0 * (q - (q @ u)[..., None] * u) + 4.0 * u
    k = k + (30.0 * (torch.arange(l) // BK) / (4.0 * SM / math.log(2.0)))[None, :, None, None] * u
    q_t = torch.randn(1, l, h, D, generator=g)
    q_t = q_t - (q_t @ u)[..., None] * u
    k_t, v_t = 0.125 * torch.randn(1, l, h, D, generator=g), torch.randn(1, l, h, D, generator=g)
    ins = [t.to(dtype).cuda() for t in (q, k, v, q_t, k_t, v_t)]
    lut = SJ._random_lut(1, h, l, topk, seed=12, ascending=True)
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    o_s, lse = attn_fwd_qk16_lse(*ins[:3], lut, topk, SM)
    assert lse.amin() > 100
    ours = SJ._check(o_s, _sla_tangent(ins, o_s, lse, lut), ins, SJ._mask(lut, l), f"large scores {dtype}")
    assert ours <= SJ.REL


@pytest.mark.parametrize("poison", [float("nan"), 1e4], ids=["nan", "1e4"])
def test_sla_memory_beyond_l_and_rows_beyond_l(cuda, poison):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    l, h, topk, extra = 300, 2, 3, 100
    ins = SJ._inputs(1, l, h, BF16, seed=l)
    lut = SJ._random_lut(1, h, l, topk, seed=3, tail=True)
    o_s, lse = attn_fwd_qk16_lse(*ins[:3], lut, topk, SM)
    want = _sla_tangent(ins, o_s, lse, lut)
    views = list(ins)
    for i in (1, 2, 4, 5):
        big = torch.full((1, 384, h, D), poison, dtype=BF16, device="cuda")
        big[:, :l] = ins[i]
        views[i] = big[:, :l]
    big_t = torch.full((1, l + extra, h, D), 7.0, dtype=BF16, device="cuda")
    _sla_tangent(views, o_s, lse, lut, o_s_t=big_t)
    assert torch.equal(big_t[:, :l], want) and (big_t[:, l:] == 7.0).all() and torch.isfinite(want).all()


@pytest.mark.parametrize("dtype", DTYPES)
def test_sla_bits_reproducible_and_independent_of_the_other_heads(cuda, dtype):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    l, topk = 700, 4
    ins = SJ._inputs(2, l, 3, dtype, seed=31)
    lut = SJ._random_lut(2, 3, l, topk, seed=32)
    o_s, lse = attn_fwd_qk16_lse(*ins[:3], lut, topk, SM)
    t1, t2 = _sla_tangent(ins, o_s, lse, lut), _sla_tangent(ins, o_s, lse, lut)
    assert torch.equal(t1, t2)
    one = [t[1:2, :, 2:3].contiguous() for t in ins]
    o1, lse1 = attn_fwd_qk16_lse(*one[:3], lut[1:2, 2:3].contiguous(), topk, SM)
    assert torch.equal(_sla_tangent(one, o1, lse1, lut[1:2, 2:3].contiguous()), t1[1:2, :, 2:3])


def test_sla_cuda_graph_replay_of_forward_lse_and_tangent(cuda):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    l, topk = 1000, 5
    ins = SJ._inputs(1, l, 2, BF16, seed=41)
    lut = SJ._random_lut(1, 2, l, topk, seed=42)
    o_s, lse = attn_fwd_qk16_lse(*ins[:3], lut, topk, SM)
    eager_t = _sla_tangent(ins, o_s, lse, lut)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_o, g_lse = attn_fwd_qk16_lse(*ins[:3], lut, topk, SM)
        g_t = _sla_tangent(ins, g_o, g_lse, lut)
    g_o.zero_(), g_t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g_o, o_s) and torch.equal(g_t, eager_t)


# ------------------------------------------------------------------------------------------------ sparse: the module
@pytest.mark.parametrize("how", ["func.jvp", "forward_ad"])
@pytest.mark.parametrize("b,l,h,ratio,dtype,feature", SJ.MODULE_CASES)
def test_sla_module_o_and_o_t(cuda, b, l, h, ratio, dtype, feature, how):
    """o and o_t against float64 torch.func.jvp of the module's formula with the selection held fixed (test_gpu_sla_jvp.py's
    bars for forward_jvp); o_t close to forward_jvp's.  The sparse branch's primal is the lse forward's bits either way; under
    forward_ad o is the training forward's bits, while under torch.func.jvp torch runs the linear branch's matmuls and proj_l
    through its own jvp rules, whose last bits may differ from the plain ops'."""
    ins = SJ._module_qkv(b, l, h, dtype, seed=300 + l)
    mod = SJ._module(ratio, feature, dtype)
    mod._keep_selection = {}
    o, o_t = (_func_jvp if how == "func.jvp" else _forward_ad)(mod, ins)
    lut = mod._keep_selection["lut"]
    mod._keep_selection = None
    assert o.dtype == o_t.dtype == dtype and o.shape == o_t.shape == ins[0].shape
    train = mod(*(t.clone().requires_grad_() for t in ins[:3])).detach()
    if how == "forward_ad":
        assert torch.equal(o, train)
    else:
        print(f"  o vs the training forward: rel-L2 {SJ._rel(o, train):.2e}")
        assert SJ._rel(o, train) <= 1e-2 and SJ._cos(o, train) >= 0.9999
    from turbodiffusion_b200.SLA.core import _SparseAttention16AD, attn_fwd_qk16_lse
    o_s, _ = (_func_jvp if how == "func.jvp" else _forward_ad)(
        lambda a, b_, c: _SparseAttention16AD.apply(a, b_, c, lut.shape[-1], SM, None)[0], ins)
    assert torch.equal(o_s, attn_fwd_qk16_lse(*ins[:3], lut, lut.shape[-1], SM)[0])
    mask = SJ._mask(lut, l)
    w, bias = mod.proj_l.weight.detach().to(SJ.F64), mod.proj_l.bias.detach().to(SJ.F64)
    prim, tan = tuple(t.to(SJ.F64) for t in ins[:3]), tuple(t.to(SJ.F64) for t in ins[3:])
    want, want_t = torch.func.jvp(lambda a, b_, c: SJ._reference(a, b_, c, w, bias, mask, feature), prim, tan)
    for name, got, ref in (("o", o, want), ("o_t", o_t, want_t)):
        rel, cos = SJ._rel(got, ref), SJ._cos(got, ref)
        print(f"({b}, {l}, {h}, {ratio}, {dtype}, {feature}) {how} {name}: rel-L2 {rel:.2e} cos {cos:.6f}")
        assert torch.isfinite(got).all() and cos >= 0.9999 and rel <= 5e-3, (name, rel, cos)
    with torch.no_grad():
        _, fj_t = mod.forward_jvp(*ins)
    rel = SJ._rel(o_t, fj_t)
    print(f"  o_t vs forward_jvp: rel-L2 {rel:.2e}")
    assert rel <= 5e-3


def test_sla_gradients_under_forward_ad_equal_the_training_path(cuda):
    """The sparse branch's gradients under forward_ad are the training op's (sparse_attention16) bit for bit; the module's,
    whose linear branch runs torch's own ops with dual inputs, within rounding of the training path's."""
    from turbodiffusion_b200.SLA.core import _SparseAttention16AD, sparse_attention16
    ins = SJ._module_qkv(1, 600, 2, BF16, seed=71)
    lut = SJ._random_lut(1, 2, 600, 3, seed=73, ascending=True)
    gout = torch.randn(ins[0].shape, generator=torch.Generator().manual_seed(74)).bfloat16().cuda()
    leaves = [t.clone().requires_grad_() for t in ins[:3]]
    select, block_map = SJ_core().select_prep, SJ_core().block_map_from_pools

    class _Prep:
        q_pool = k_pool = None
    try:
        SJ_core().select_prep, SJ_core().block_map_from_pools = (lambda *a: _Prep()), (lambda *a: (None, lut))
        with fwAD.dual_level():
            o_s = _SparseAttention16AD.apply(*(fwAD.make_dual(p, t) for p, t in zip(leaves, ins[3:])), 3, SM, None)[0]
            fwAD.unpack_dual(o_s).primal.backward(gout)
    finally:
        SJ_core().select_prep, SJ_core().block_map_from_pools = select, block_map
    plain = [t.clone().requires_grad_() for t in ins[:3]]
    sparse_attention16(*plain, lut, 3, SM).backward(gout)
    for a, b in zip(leaves, plain):
        assert torch.equal(a.grad, b.grad)

    mod = SJ._module(0.25)
    gout = torch.randn(ins[0].shape, generator=torch.Generator().manual_seed(72)).bfloat16().cuda()
    leaves = [t.clone().requires_grad_() for t in ins[:3]]
    with fwAD.dual_level():
        primal, _ = fwAD.unpack_dual(mod(*(fwAD.make_dual(p, t) for p, t in zip(leaves, ins[3:]))))
        primal.backward(gout)
    grads = [t.grad for t in leaves] + [mod.proj_l.weight.grad.clone(), mod.proj_l.bias.grad.clone()]
    mod.zero_grad()
    plain = [t.clone().requires_grad_() for t in ins[:3]]
    mod(*plain).backward(gout)
    for a, b in zip(grads, [t.grad for t in plain] + [mod.proj_l.weight.grad, mod.proj_l.bias.grad]):
        print(f"  module gradient: rel-L2 to the training path {SJ._rel(a, b):.2e}")
        assert SJ._rel(a, b) <= 1e-2


def test_sla_shape_a_on_sampled_rows(cuda):
    """Shape A self-attention through SparseLinearAttention under torch.func.jvp, top-k 0.1: o_t against forward_jvp's
    (the same selection) and, on 32 sampled rows per head, against float64 of the sparse branch."""
    l, h = 32760, 12
    mod = SJ._module(0.1)
    g = torch.Generator(device="cuda").manual_seed(81)
    ins = [torch.randn(1, l, h, D, generator=g, device="cuda").bfloat16() for _ in range(6)]
    mod._keep_selection = {}
    o, o_t = _func_jvp(mod, ins)
    lut = mod._keep_selection["lut"]
    mod._keep_selection = None
    with torch.no_grad():
        fj, fj_t = mod.forward_jvp(*ins)
    assert torch.isfinite(o_t).all()
    print(f"shape A: o_t vs forward_jvp rel-L2 {SJ._rel(o_t, fj_t):.2e}")
    assert SJ._rel(o_t, fj_t) <= 5e-3
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    o_s, lse = attn_fwd_qk16_lse(*ins[:3], lut, lut.shape[-1], SM)
    o_s_t = _sla_tangent(ins, o_s, lse, lut)
    n = 32
    rows = torch.stack([torch.randperm(l, generator=torch.Generator().manual_seed(90 + i))[:n] for i in range(h)]).cuda()
    heads = torch.arange(h, device="cuda")[:, None]
    pick = lambda t: t[0][rows, heads].transpose(0, 1)[None]
    mask = SJ._mask(lut, l, rows)
    sub = [pick(ins[0]), ins[1], ins[2], pick(ins[3]), ins[4], ins[5]]
    _, want_t = SJ.exact_f64(*sub, mask)
    ours, ref = SJ._rel(pick(o_s_t), want_t), SJ._rel(SJ.restated(*sub, mask), want_t)
    print(f"shape A sampled rows: o_s_t rel-L2 {ours:.2e}, restatement {ref:.2e}")
    assert ours <= 1.5 * ref + 1e-7


# ------------------------------------------------------------------------------------------------ a toy network
class _Block(torch.nn.Module):
    """LayerNorm, q/k/v projections, sparse self-attention, dense cross-attention over a context, GELU MLP, residuals"""

    def __init__(self, dim, heads, g):
        super().__init__()
        from turbodiffusion_b200.SLA import SparseLinearAttention
        self.h = heads
        self.norm = torch.nn.LayerNorm(dim)
        self.qkv, self.q2, self.kv2, self.mlp = (torch.nn.Linear(dim, n) for n in (3 * dim, dim, 2 * dim, dim))
        for lin in (self.qkv, self.q2, self.kv2, self.mlp):
            torch.nn.init.normal_(lin.weight, std=dim ** -0.5, generator=g)
        self.sla = SparseLinearAttention(D, 0.25, BLKQ=128, BLKK=64)
        torch.nn.init.normal_(self.sla.proj_l.weight, std=0.05, generator=g)

    def pre_self(self, x):
        return self.qkv(self.norm(x)).bfloat16().view(*x.shape[:2], 3, self.h, D).unbind(2)

    def pre_cross(self, x):
        return self.q2(x).bfloat16().view(*x.shape[:2], self.h, D)

    def kv_cross(self, ctx):
        return self.kv2(ctx).bfloat16().view(*ctx.shape[:2], 2, self.h, D).unbind(2)

    def mlp_res(self, x):
        return x + torch.nn.functional.gelu(self.mlp(x))

    def forward(self, x, ctx):
        from turbodiffusion_b200 import ops
        x = x + self.sla(*self.pre_self(x)).reshape(x.shape).float()
        x = x + ops.dense_attention(self.pre_cross(x), *self.kv_cross(ctx)).reshape(x.shape).float()
        return self.mlp_res(x)

    def forward_explicit(self, x, x_t, ctx):
        """(forward(x), its tangent along x_t): forward_jvp and dense_attention_jvp for the attention, torch.func.jvp of the
        segments between them"""
        from turbodiffusion_b200 import ops
        (q, k, v), (q_t, k_t, v_t) = torch.func.jvp(self.pre_self, (x,), (x_t,))
        o, o_t = self.sla.forward_jvp(q, k, v, q_t, k_t, v_t)
        x, x_t = x + o.reshape(x.shape).float(), x_t + o_t.reshape(x.shape).float()
        q2, q2_t = torch.func.jvp(self.pre_cross, (x,), (x_t,))
        k2, v2 = self.kv_cross(ctx)
        o, o_t = ops.dense_attention_jvp(q2, k2, v2, q2_t, torch.zeros_like(k2), torch.zeros_like(v2))
        x, x_t = x + o.reshape(x.shape).float(), x_t + o_t.reshape(x.shape).float()
        return torch.func.jvp(self.mlp_res, (x,), (x_t,))


def test_two_block_network_under_func_jvp_matches_the_explicit_jvp_network(cuda):
    """torch.func.jvp through two blocks of torch ops, SparseLinearAttention and ops.dense_attention, against the same network
    with its tangent carried by hand through forward_jvp and dense_attention_jvp."""
    g = torch.Generator().manual_seed(3)
    heads, l, lc = 2, 700, 226
    dim = heads * D
    blocks = torch.nn.ModuleList(_Block(dim, heads, g) for _ in range(2)).cuda()
    x, x_t = (torch.randn(1, l, dim, generator=g).cuda() for _ in range(2))
    ctx = torch.randn(1, lc, dim, generator=g).cuda()

    def net(x):
        for blk in blocks:
            x = blk(x, ctx)
        return x

    with torch.no_grad():
        y, y_t = torch.func.jvp(net, (x,), (x_t,))
        ref, ref_t = x, x_t
        for blk in blocks:
            ref, ref_t = blk.forward_explicit(ref, ref_t, ctx)
    rel, rel_t = SJ._rel(y, ref), SJ._rel(y_t, ref_t)
    print(f"two blocks: y rel-L2 {rel:.2e}, y_t rel-L2 {rel_t:.2e} to the explicit-JVP network")
    assert torch.isfinite(y_t).all() and rel <= 5e-3 and rel_t <= 5e-3
