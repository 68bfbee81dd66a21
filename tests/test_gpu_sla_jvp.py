"""GPU checks of the sparse attention JVP (tdb200_sla_attn16_jvp, SLA.core.sparse_attention16_jvp and
SparseLinearAttention.forward_jvp): bit-equality with the dense JVP on a LUT listing every key block, o_s and o_s_t against
float64 on random LUTs and at large score magnitudes, o_s against the SLA forward, the module's o, o_t and gradients against
float64, exact cases, masking, reproducibility, CUDA-graph capture, and shape A on sampled rows.

Bars.  o_s: cos >= 0.999 and rel-L2 <= 5e-3 against float64, and o_s_t: rel-L2 against float64 at most 1.5x that of a float32
torch restatement that rounds p and p * S_t to the 16-bit type where the kernel does, plus 1e-7 (the bars of
tests/test_gpu_dense_attention_jvp.py).  o_s against tdb200_sla_attn16_fwd_lse: cos >= 0.9999, rel-L2 <= 5e-3, lse within 1e-3
(the SLA forward's bars).  Module: o and o_t cos >= 0.9999, rel-L2 <= 5e-3 (the training path's output bars,
tests/test_gpu_sla_backward.py); gradients cos >= 0.999, rel-L2 <= 2e-2 (proj_l: rel-L2 <= 2e-2), that file's bars."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import td_oracle as O

pytestmark = pytest.mark.gpu
D, BQ, BK = 128, 128, 64
SM = D ** -0.5
LOG2E = 1.0 / math.log(2.0)
F64 = torch.float64
BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]
COS, REL = 0.999, 5e-3


def _rel(got, want):
    a, b = got.to(F64).flatten(), want.to(F64).flatten().to(got.device)
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _cos(got, want):
    a, b = got.to(F64).flatten(), want.to(F64).flatten().to(got.device)
    return (torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-300)).item()


def _inputs(b, l, h, dtype, seed):
    """q, k, v, q_t, k_t, v_t [b, l, h, D] on the GPU"""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(b, l, h, D, generator=g).to(dtype).cuda() for _ in range(6)]


def _nblk(l):
    return (l + BK - 1) // BK


def _full_lut(b, h, l):
    mblk, nblk = (l + BQ - 1) // BQ, _nblk(l)
    return torch.arange(nblk, dtype=torch.int32).expand(b, h, mblk, nblk).contiguous().cuda()


def _random_lut(b, h, l, topk, seed, tail=None, ascending=False):
    """distinct random key blocks per query block, in random order unless `ascending`; tail True / False forces the last
    (ragged) key block into / out of every row"""
    g = torch.Generator().manual_seed(seed)
    mblk, nblk = (l + BQ - 1) // BQ, _nblk(l)
    lut = torch.empty(b, h, mblk, topk, dtype=torch.int32)
    for i in range(b * h * mblk):
        pool = torch.randperm(nblk - 1, generator=g) if tail is not None else torch.randperm(nblk, generator=g)
        ids = pool[: topk - 1] if tail else pool[:topk]
        if tail:
            ids = torch.cat([ids, torch.tensor([nblk - 1])])[torch.randperm(topk, generator=g)]
        lut.view(-1, topk)[i] = ids.sort().values if ascending else ids
    return lut.cuda()


def _jvp(q, k, v, q_t, k_t, v_t, lut, sm_scale=SM):
    from turbodiffusion_b200.SLA.core import attn_jvp_qk16
    return attn_jvp_qk16(q, k, v, q_t, k_t, v_t, lut, lut.shape[-1], sm_scale)


def _jvp_lse(q, k, v, q_t, k_t, v_t, lut, sm_scale=SM):
    from turbodiffusion_b200 import _lib
    b, l, h, d = q.shape
    o_s, o_s_t = torch.empty_like(q), torch.empty_like(q)
    lse = torch.empty(b, h, l, dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().tdb200_sla_attn16_jvp_lse(*(t.data_ptr() for t in (q, k, v, q_t, k_t, v_t)), _lib.DTYPE_TAG[q.dtype],
                                                    lut.data_ptr(), lut.shape[-1], o_s.data_ptr(), o_s_t.data_ptr(),
                                                    lse.data_ptr(), b, l, h, d, sm_scale, BQ, BK, _lib.stream_ptr(q.device)),
               "sla_attn16_jvp_lse")
    return o_s, o_s_t, lse


def _mask(lut, l, rows=None):
    """[B, H, n, l] bool: key j is listed for query row i (rows [H, n] per head, or every row)"""
    b, h, _, _ = lut.shape
    if rows is None:
        rows = torch.arange(l, device=lut.device).expand(h, l)
    blocks = lut[:, torch.arange(h, device=lut.device)[:, None], rows // BQ]            # [B, H, n, topk]
    sel = torch.zeros(*blocks.shape[:3], _nblk(l), dtype=torch.bool, device=lut.device)
    sel.scatter_(-1, blocks.long(), True)
    return sel[..., torch.arange(l, device=lut.device) // BK]


def _attn(q, k, v, mask, sm_scale):
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * sm_scale
    s = s.masked_fill(~mask, -math.inf)
    return torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v)


def exact_f64(q, k, v, q_t, k_t, v_t, mask, sm_scale=SM):
    """(o_s, o_s_t) of float64 torch.func.jvp of the softmax over the listed keys, the selection held fixed"""
    prim, tan = (tuple(t.to(F64) for t in ts) for ts in ((q, k, v), (q_t, k_t, v_t)))
    return torch.func.jvp(lambda a, b, c: _attn(a, b, c, mask, sm_scale), prim, tan)


def restated(q, k, v, q_t, k_t, v_t, mask, sm_scale=SM):
    """The kernel's tangent arithmetic in float32 torch over the listed keys (tests/test_gpu_dense_attention_jvp.py's)"""
    f = [t.float() for t in (q, k, v, q_t, k_t, v_t)]
    s = (torch.einsum("bqhd,bkhd->bhqk", f[0], f[1]) * sm_scale).masked_fill(~mask, -math.inf)
    st = (torch.einsum("bqhd,bkhd->bhqk", f[3], f[1]) + torch.einsum("bqhd,bkhd->bhqk", f[0], f[4])) * sm_scale
    p = torch.exp(s - s.amax(-1, keepdim=True))
    pst = p * st
    l, mu = p.sum(-1), pst.sum(-1)
    p_r, pst_r = (t.to(q.dtype).float() for t in (p, pst))
    o = torch.einsum("bhqk,bkhd->bqhd", p_r, f[2])
    a = torch.einsum("bhqk,bkhd->bqhd", pst_r, f[2]) + torch.einsum("bhqk,bkhd->bqhd", p_r, f[5])
    l, mu = l.transpose(1, 2)[..., None], mu.transpose(1, 2)[..., None]
    return ((a - mu / l * o) / l).to(q.dtype)


def _check(o_s, o_s_t, ins, mask, what):
    want, want_t = exact_f64(*ins, mask)
    rel, cos = _rel(o_s, want), _cos(o_s, want)
    ours, ref = _rel(o_s_t, want_t), _rel(restated(*ins, mask), want_t)
    print(f"{what}: o_s rel-L2 {rel:.2e} cos {cos:.6f}; o_s_t rel-L2 {ours:.2e}, restatement {ref:.2e}")
    assert torch.isfinite(o_s).all() and cos >= COS and rel <= REL, (what, rel, cos)
    assert torch.isfinite(o_s_t).all() and ours <= 1.5 * ref + 1e-7, (what, ours, ref)
    return ours


# ------------------------------------------------------------------------------------------------ the dense JVP's bits
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,l", [(2, 3, 64), (2, 3, 1000), (2, 2, 1182), (1, 1, 300)])
def test_full_ascending_lut_gives_the_dense_jvp_bits(cuda, b, h, l, dtype):
    from turbodiffusion_b200 import _lib
    ins = _inputs(b, l, h, dtype, seed=l + b)
    o_s, o_s_t, lse = _jvp_lse(*ins, _full_lut(b, h, l))
    out, out_t = torch.empty_like(o_s), torch.empty_like(o_s)
    lse_d = torch.empty_like(lse)
    _lib.check(_lib.lib().tdb200_attn_dense_jvp_lse(*(t.data_ptr() for t in ins), _lib.DTYPE_TAG[dtype], out.data_ptr(),
                                                    out_t.data_ptr(), lse_d.data_ptr(), b, l, l, h, D, SM,
                                                    _lib.stream_ptr(ins[0].device)), "attn_dense_jvp_lse")
    assert torch.equal(o_s, out) and torch.equal(o_s_t, out_t) and torch.equal(lse, lse_d)
    no_lse = _jvp(*ins, _full_lut(b, h, l))
    assert torch.equal(no_lse[0], o_s) and torch.equal(no_lse[1], o_s_t)


# ------------------------------------------------------------------------------------------------ float64
RANDOM_CASES = [
    # b, h, l, topk, tail (True: in every row, False: never, None: as drawn)
    (1, 2, 1000, 1, None),
    (1, 2, 1000, 1, True),
    (2, 3, 1000, 5, True),
    (2, 3, 1000, 5, False),
    (1, 2, 1000, 16, None),          # topk = nblk, in random order
    (1, 3, 1182, 7, True),
    (2, 1, 333, 3, False),
    (1, 1, 64, 1, None),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,l,topk,tail", RANDOM_CASES)
def test_random_luts_against_float64(cuda, b, h, l, topk, tail, dtype):
    ins = _inputs(b, l, h, dtype, seed=7 * l + topk)
    lut = _random_lut(b, h, l, topk, seed=l + topk, tail=tail)
    o_s, o_s_t = _jvp(*ins, lut)
    assert o_s.shape == o_s_t.shape == ins[0].shape and o_s.dtype == o_s_t.dtype == dtype
    _check(o_s, o_s_t, ins, _mask(lut, l), f"({b}, {h}, {l}) topk {topk} tail {tail} {dtype}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_large_scores_rescale_every_accumulator(cuda, dtype):
    """log2-domain scores climb by about 30 per key block and the LUT lists blocks in ascending order, so the running maximum of
    most rows grows by more than 2^8 between tiles and the kernel rescales O, A, l and mu (as in the dense JVP's test)."""
    l, h, topk = 1000, 2, 9
    g = torch.Generator().manual_seed(11)
    u = torch.ones(D) / D ** 0.5
    q, k, v = (torch.randn(1, l, h, D, generator=g) for _ in range(3))
    a = 4.0
    q = 8.0 * (q - (q @ u)[..., None] * u) + a * u
    k = k + (30.0 * (torch.arange(l) // BK) / (a * SM * LOG2E))[None, :, None, None] * u
    q_t = torch.randn(1, l, h, D, generator=g)
    q_t = q_t - (q_t @ u)[..., None] * u
    k_t, v_t = 0.125 * torch.randn(1, l, h, D, generator=g), torch.randn(1, l, h, D, generator=g)
    ins = [t.to(dtype).cuda() for t in (q, k, v, q_t, k_t, v_t)]
    lut = _random_lut(1, h, l, topk, seed=12, ascending=True)
    o_s, o_s_t = _jvp(*ins, lut)
    ours = _check(o_s, o_s_t, ins, _mask(lut, l), f"large scores {dtype}")
    assert ours <= REL, ours


# ------------------------------------------------------------------------------------------------ the SLA forward
@pytest.mark.parametrize("dtype", DTYPES)
def test_o_s_matches_the_sla_forward(cuda, dtype):
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    b, h, l, topk = 2, 3, 1182, 8
    ins = _inputs(b, l, h, dtype, seed=21)
    lut = _random_lut(b, h, l, topk, seed=22, ascending=True)
    o_s, _, lse = _jvp_lse(*ins, lut)
    fwd, fwd_lse = attn_fwd_qk16_lse(*ins[:3], lut, topk, SM)
    s = O.stats(o_s.float().cpu(), fwd.float().cpu())
    print(f"o_s vs tdb200_sla_attn16_fwd_lse {dtype}: bit-equal {torch.equal(o_s, fwd)}, rel-L2 {s['rel_l2']:.2e}, "
          f"lse bit-equal {torch.equal(lse, fwd_lse)}, max |d lse| {(lse - fwd_lse).abs().max().item():.2e}")
    assert s["cos"] >= 0.9999 and s["rel_l2"] <= 5e-3, s
    assert (lse - fwd_lse).abs().max().item() <= 1e-3


# ------------------------------------------------------------------------------------------------ the module
def _module(ratio, feature="softmax", dtype=BF16, seed=5):
    from turbodiffusion_b200.SLA import SparseLinearAttention
    mod = SparseLinearAttention(D, ratio, feature_map=feature, BLKQ=128, BLKK=64, use_bf16=dtype == BF16).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        mod.proj_l.weight.copy_(torch.randn(D, D, generator=g) * 0.05)
        mod.proj_l.bias.copy_(torch.randn(D, generator=g) * 0.05)
    return mod


def _module_qkv(b, l, h, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(b, l, h, D, generator=g)
    k = torch.randn(b, l, h, D, generator=g) + torch.randn(1, 1, h, D, generator=g) * 2.0
    v, q_t, k_t, v_t = (torch.randn(b, l, h, D, generator=g) for _ in range(4))
    return [t.to(dtype).cuda() for t in (q, k, v, q_t, k_t, v_t)]


def _reference(q, k, v, w, bias, mask, feature):
    """the module's formula in the inputs' precision: masked softmax attention plus proj_l of the linear branch"""
    fq, fk = O.feature_maps(feature)
    o_s = _attn(q, k, v, mask, SM)
    qh, kh, vh = (t.transpose(1, 2) for t in (q, k, v))
    pq, pk = fq(qh), fk(kh)
    o_l = (pq @ (pk.transpose(-1, -2) @ vh)) / (1e-5 + (pq * pk.sum(-2, keepdim=True)).sum(-1, keepdim=True))
    return o_s + F.linear(o_l, w, bias).transpose(1, 2)


MODULE_CASES = [
    # b, l, h, ratio, dtype, feature
    (1, 1000, 2, 0.25, BF16, "softmax"),
    (2, 333, 3, 0.5, BF16, "softmax"),
    (1, 1280, 2, 0.1, BF16, "softmax"),
    (1, 600, 2, 0.25, FP16, "softmax"),
    (1, 600, 2, 0.25, BF16, "elu"),
    (1, 600, 2, 0.25, BF16, "relu"),
]


@pytest.mark.parametrize("b,l,h,ratio,dtype,feature", MODULE_CASES)
def test_forward_jvp_o_o_t_and_gradients_against_float64(cuda, b, l, h, ratio, dtype, feature):
    ins = _module_qkv(b, l, h, dtype, seed=300 + l)
    mod = _module(ratio, feature, dtype)
    mod._keep_selection = {}
    qg, kg, vg = (t.clone().requires_grad_() for t in ins[:3])
    o, o_t = mod.forward_jvp(qg, kg, vg, *ins[3:])
    lut = mod._keep_selection["lut"]
    mod._keep_selection = None
    assert o.requires_grad and not o_t.requires_grad and o.dtype == o_t.dtype == dtype
    train = mod(*(t.clone().requires_grad_() for t in ins[:3])).detach()          # the training path of forward
    mask = _mask(lut, l)
    w, bias = mod.proj_l.weight.detach().to(F64), mod.proj_l.bias.detach().to(F64)
    prim, tan = tuple(t.to(F64) for t in ins[:3]), tuple(t.to(F64) for t in ins[3:])
    want, want_t = torch.func.jvp(lambda a, b_, c: _reference(a, b_, c, w, bias, mask, feature), prim, tan)
    for name, got, ref in (("o", o, want), ("o_t", o_t, want_t)):
        s = O.stats(got.double().cpu(), ref.cpu())
        print(f"({b}, {l}, {h}, {ratio}, {dtype}, {feature}) {name}: rel-L2 {s['rel_l2']:.2e} cos {s['cos']:.6f}")
        assert torch.isfinite(got).all() and s["cos"] >= 0.9999 and s["rel_l2"] <= 5e-3, (name, s)
    print(f"  o vs the training forward: bit-equal {torch.equal(o, train)}, rel-L2 {_rel(o, train):.2e}")
    assert _rel(o, train) <= REL and _cos(o, train) >= 0.9999

    gout = torch.randn(o.shape, generator=torch.Generator().manual_seed(9)).to(dtype).cuda()
    o.backward(gout)
    leaves = [t.to(F64).requires_grad_() for t in ins[:3]] + [w.clone().requires_grad_(), bias.clone().requires_grad_()]
    (_reference(*leaves, mask, feature) * gout.to(F64)).sum().backward()
    got = [qg.grad, kg.grad, vg.grad, mod.proj_l.weight.grad, mod.proj_l.bias.grad]
    for name, gt, lf in zip(("dq", "dk", "dv", "dW", "db"), got, leaves):
        s = O.stats(gt.double().cpu(), lf.grad.cpu())
        print(f"  {name}: rel-L2 {s['rel_l2']:.2e} cos {s['cos']:.6f}")
        assert s["rel_l2"] <= 2e-2 and (name in ("dW", "db") or s["cos"] >= 0.999), (name, s)


def test_forward_jvp_without_grad_gives_the_same_bits(cuda):
    ins = _module_qkv(1, 700, 2, BF16, seed=77)
    mod = _module(0.3)
    with torch.no_grad():
        o, o_t = mod.forward_jvp(*ins)
    og, og_t = mod.forward_jvp(*(t.clone().requires_grad_() for t in ins[:3]), *ins[3:])
    assert torch.equal(o, og.detach()) and torch.equal(o_t, og_t)


# ------------------------------------------------------------------------------------------------ properties
@pytest.mark.parametrize("dtype", DTYPES)
def test_zero_tangents_give_a_zero_tangent_and_the_same_output(cuda, dtype):
    q, k, v, q_t, k_t, v_t = _inputs(2, 700, 3, dtype, seed=7)
    lut = _random_lut(2, 3, 700, 4, seed=8, tail=True)
    o_s, o_s_t = _jvp(q, k, v, *(torch.zeros_like(t) for t in (q_t, k_t, v_t)), lut)
    assert torch.equal(o_s_t, torch.zeros_like(o_s_t))
    assert torch.equal(o_s, _jvp(q, k, v, q_t, k_t, v_t, lut)[0])


@pytest.mark.parametrize("poison", [float("nan"), 1e4], ids=["nan", "1e4"])
@pytest.mark.parametrize("l", [77, 300])
def test_memory_beyond_l_is_never_used(cuda, l, poison):
    """every input is the first l rows of a larger allocation whose other rows hold NaN or 1e4, and the LUT lists the ragged
    tail block: both outputs equal, bit for bit, those of tight copies."""
    ins = _inputs(1, l, 2, BF16, seed=l)
    views = []
    for t in ins:
        big = torch.full((1, 512, 2, D), poison, dtype=BF16, device="cuda")
        big[:, :l] = t
        views.append(big[:, :l])
        assert views[-1].is_contiguous() and views[-1].data_ptr() == big.data_ptr()
    lut = _random_lut(1, 2, l, _nblk(l), seed=3)
    o_s, o_s_t = _jvp(*views, lut)
    ref, ref_t = _jvp(*ins, lut)
    assert torch.isfinite(o_s).all() and torch.isfinite(o_s_t).all()
    assert torch.equal(o_s, ref) and torch.equal(o_s_t, ref_t)


def test_rows_beyond_l_are_not_stored(cuda):
    from turbodiffusion_b200 import _lib
    l, h, extra = 333, 2, 120
    ins = _inputs(1, l, h, BF16, seed=9)
    lut = _random_lut(1, h, l, 3, seed=10, tail=True)
    big, big_t = (torch.full((1, l + extra, h, D), 7.0, dtype=BF16, device="cuda") for _ in range(2))
    lse = torch.full((1, h, l + extra), 7.0, device="cuda")
    _lib.check(_lib.lib().tdb200_sla_attn16_jvp_lse(*(t.data_ptr() for t in ins), _lib.DTYPE_TAG[BF16], lut.data_ptr(), 3,
                                                    big.data_ptr(), big_t.data_ptr(), lse.data_ptr(), 1, l, h, D, SM, BQ, BK,
                                                    _lib.stream_ptr(ins[0].device)), "sla_attn16_jvp_lse")
    o_s, o_s_t = _jvp(*ins, lut)
    assert torch.equal(big[:, :l], o_s) and torch.equal(big_t[:, :l], o_s_t)
    assert (big[:, l:] == 7.0).all() and (big_t[:, l:] == 7.0).all()


@pytest.mark.parametrize("dtype", DTYPES)
def test_bits_are_reproducible_and_independent_of_the_other_heads(cuda, dtype):
    ins = _inputs(2, 700, 3, dtype, seed=31)
    lut = _random_lut(2, 3, 700, 5, seed=32)
    o_s, o_s_t = _jvp(*ins, lut)
    again, again_t = _jvp(*ins, lut)
    assert torch.equal(o_s, again) and torch.equal(o_s_t, again_t)
    one, one_t = _jvp(*(t[1:2, :, 2:3].contiguous() for t in ins), lut[1:2, 2:3].contiguous())
    assert torch.equal(one, o_s[1:2, :, 2:3]) and torch.equal(one_t, o_s_t[1:2, :, 2:3])


def test_cuda_graph_replay_matches_eager(cuda):
    ins = _inputs(1, 900, 2, BF16, seed=41)
    lut = _random_lut(1, 2, 900, 6, seed=42)
    eager, eager_t, eager_lse = _jvp_lse(*ins, lut)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured, captured_t, captured_lse = _jvp_lse(*ins, lut)
    for t in (captured, captured_t, captured_lse):
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured, eager) and torch.equal(captured_t, eager_t) and torch.equal(captured_lse, eager_lse)


def test_shape_a_on_sampled_rows(cuda):
    """Wan2.1-1.3B at 480p: 32760 tokens, 12 heads of 128, topk 51 of 512 key blocks (SparseLinearAttention at 0.1); 64 sampled
    query rows per head against float64 rows over their listed keys."""
    l, h, n, topk = 32760, 12, 64, 51
    g = torch.Generator(device="cuda").manual_seed(51)
    ins = [torch.randn(1, l, h, D, generator=g, device="cuda").bfloat16() for _ in range(6)]
    mblk, nblk = (l + BQ - 1) // BQ, _nblk(l)
    lut = torch.stack([torch.randperm(nblk, generator=torch.Generator().manual_seed(i))[:topk] for i in range(h * mblk)])
    lut = lut.view(1, h, mblk, topk).int().cuda()
    o_s, o_s_t = _jvp(*ins, lut)
    assert torch.isfinite(o_s).all() and torch.isfinite(o_s_t).all()
    rows = torch.stack([torch.randperm(l, generator=torch.Generator().manual_seed(60 + i))[:n] for i in range(h)]).cuda()
    rows[:, 0], rows[:, 1] = 0, l - 1
    heads = torch.arange(h, device="cuda")[:, None]
    pick = lambda t: t[0][rows, heads].transpose(0, 1)[None]                    # [1, n, h, D]
    sub = [pick(ins[0]), ins[1], ins[2], pick(ins[3]), ins[4], ins[5]]
    mask = _mask(lut, l, rows)
    _check(pick(o_s), pick(o_s_t), sub, mask, f"shape A, topk {topk}, {n} rows x {h} heads")
