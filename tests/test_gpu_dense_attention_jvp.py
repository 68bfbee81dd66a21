"""GPU checks of the dense attention JVP operator (ops.dense_attention_jvp, tdb200_attn_dense_jvp): the tangent against float64
torch.func.jvp of explicit-softmax attention, the primal output against the oracle, exact cases (zero and v-only tangents),
large score magnitudes (the lazy rescale of all four accumulators), masking of the ragged tails, the [l, h*d] layout,
reproducibility, CUDA-graph capture, and shape A at full size on sampled rows.

Bars.  Primal output: those of tests/test_gpu_dense_attention.py, cos >= 0.999 and rel-L2 <= 5e-3 against the oracle.  Tangent:
rel-L2 against float64 at most 1.5x that of a float32 torch restatement that rounds p and p * S_t to the 16-bit type where the
kernel does (p relative to the row's final maximum, l and mu from the unrounded values, one rounding of out_t), plus 1e-7."""
import math

import pytest
import torch

from oracle import td_oracle as O

pytestmark = pytest.mark.gpu
D, BK = 128, 64                                   # head dim; the JVP kernel's key tile
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


def _inputs(b, lq, lk, h, dtype, seed):
    """q, k, v, q_t, k_t, v_t on the GPU"""
    g = torch.Generator().manual_seed(seed)
    shapes = [(b, lq, h, D), (b, lk, h, D), (b, lk, h, D)] * 2
    return [torch.randn(*s, generator=g).to(dtype).cuda() for s in shapes]


def _jvp(q, k, v, q_t, k_t, v_t, sm_scale=None):
    from turbodiffusion_b200 import ops
    return ops.dense_attention_jvp(q, k, v, q_t, k_t, v_t, sm_scale)


def _attn(q, k, v, sm_scale):
    """explicit-softmax attention of [B, L, H, D] tensors"""
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * sm_scale
    return torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v)


def exact_f64(q, k, v, q_t, k_t, v_t, sm_scale=SM):
    """(out, out_t) of float64 torch.func.jvp, on the inputs' device"""
    prim, tan = (tuple(t.to(F64) for t in ts) for ts in ((q, k, v), (q_t, k_t, v_t)))
    return torch.func.jvp(lambda a, b, c: _attn(a, b, c, sm_scale), prim, tan)


def restated(q, k, v, q_t, k_t, v_t, sm_scale=SM):
    """The kernel's tangent arithmetic in float32 torch: p = exp(s - max) and p * S_t rounded to q's dtype as the operands of
    the products, l and mu summed from the unrounded values, out_t = (A - (mu / l) O) / l rounded to q's dtype."""
    f = [t.float() for t in (q, k, v, q_t, k_t, v_t)]
    s = torch.einsum("bqhd,bkhd->bhqk", f[0], f[1]) * sm_scale
    st = (torch.einsum("bqhd,bkhd->bhqk", f[3], f[1]) + torch.einsum("bqhd,bkhd->bhqk", f[0], f[4])) * sm_scale
    p = torch.exp(s - s.amax(-1, keepdim=True))
    pst = p * st
    l, mu = p.sum(-1), pst.sum(-1)
    p_r, pst_r = (t.to(q.dtype).float() for t in (p, pst))
    o = torch.einsum("bhqk,bkhd->bqhd", p_r, f[2])
    a = torch.einsum("bhqk,bkhd->bqhd", pst_r, f[2]) + torch.einsum("bhqk,bkhd->bqhd", p_r, f[5])
    l, mu = l.transpose(1, 2)[..., None], mu.transpose(1, 2)[..., None]
    return ((a - mu / l * o) / l).to(q.dtype)


def _oracle(q, k, v, sm_scale=SM):
    qh, kh, vh = (t.float().cpu().transpose(1, 2) for t in (q, k, v))
    return O.dense_attention(qh, kh, vh, sm_scale).transpose(1, 2)


def _check_tangent(out_t, ins, what, sm_scale=SM):
    _, want_t = exact_f64(*ins, sm_scale=sm_scale)
    ours, ref = _rel(out_t, want_t), _rel(restated(*ins, sm_scale=sm_scale), want_t)
    print(f"{what}: tangent rel-L2 {ours:.2e}, restatement {ref:.2e}")
    assert torch.isfinite(out_t).all() and ours <= 1.5 * ref + 1e-7, (what, ours, ref)
    return ours, ref


def _check_primal(out, want, what):
    rel, cos = _rel(out, want), _cos(out, want)
    assert torch.isfinite(out).all() and cos >= COS and rel <= REL, (what, rel, cos)


# ------------------------------------------------------------------------------------------------------------ accuracy
LENGTHS = (1, 77, 128, 129, 512, 700)
BH = [(1, 1), (1, 3), (2, 1), (2, 3)]
CASES = [(*BH[i % 4], lq, lk) for i, (lq, lk) in enumerate((lq, lk) for lq in LENGTHS for lk in LENGTHS)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,h,lq,lk", [pytest.param(*c, id="b{}h{}-{}x{}".format(*c)) for c in CASES])
def test_tangent_and_output_against_float64(cuda, b, h, lq, lk, dtype):
    ins = _inputs(b, lq, lk, h, dtype, seed=1000 * lq + lk)
    out, out_t = _jvp(*ins)
    assert out.shape == out_t.shape == ins[0].shape and out.dtype == out_t.dtype == dtype
    assert out.is_contiguous() and out_t.is_contiguous()
    _check_primal(out, _oracle(*ins[:3]), (b, h, lq, lk, dtype))
    _check_tangent(out_t, ins, f"({b}, {h}, {lq}, {lk}) {dtype}")


def test_float32_inputs_run_in_bf16_and_sm_scale_is_passed_on(cuda):
    ins = [t.float() for t in _inputs(1, 200, 300, 2, BF16, seed=3)]
    out, out_t = _jvp(*ins, sm_scale=0.5 * SM)
    assert out.dtype == out_t.dtype == torch.float32
    out16, out_t16 = _jvp(*(t.bfloat16() for t in ins), sm_scale=0.5 * SM)
    assert torch.equal(out, out16.float()) and torch.equal(out_t, out_t16.float())
    _check_tangent(out_t16, [t.bfloat16() for t in ins], "sm_scale", sm_scale=0.5 * SM)


# ------------------------------------------------------------------------------------------------------------ exact cases
@pytest.mark.parametrize("dtype", DTYPES)
def test_zero_tangents_give_a_zero_tangent_and_the_same_output(cuda, dtype):
    q, k, v, q_t, k_t, v_t = _inputs(2, 333, 700, 3, dtype, seed=7)
    out, out_t = _jvp(q, k, v, *(torch.zeros_like(t) for t in (q_t, k_t, v_t)))
    assert torch.equal(out_t, torch.zeros_like(out_t))
    assert torch.equal(out, _jvp(q, k, v, q_t, k_t, v_t)[0])     # the primal does not depend on the tangents


@pytest.mark.parametrize("dtype", DTYPES)
def test_v_only_tangent_is_attention_of_the_tangent(cuda, dtype):
    """S_t = 0: out_t = P.v_t, the same arithmetic as the output with v_t for v, so bit-equal to the JVP kernel's own output
    on (q, k, v_t), and within rounding (different key tiles) of ops.dense_attention(q, k, v_t)."""
    from turbodiffusion_b200 import ops
    q, k, v, _, _, v_t = _inputs(1, 500, 600, 2, dtype, seed=8)
    z_q, z_k = torch.zeros_like(q), torch.zeros_like(k)
    _, out_t = _jvp(q, k, v, z_q, z_k, v_t)
    assert torch.equal(out_t, _jvp(q, k, v_t, z_q, z_k, v)[0])
    fwd = ops.dense_attention(q, k, v_t)
    print(f"v-only tangent {dtype}: rel-L2 to dense_attention(q, k, v_t) {_rel(out_t, fwd):.2e}")
    assert _rel(out_t, fwd) <= REL and _cos(out_t, fwd) >= COS


# ------------------------------------------------------------------------------------------------------------ large scores
@pytest.mark.parametrize("dtype", DTYPES)
def test_large_scores_rescale_every_accumulator(cuda, dtype):
    """log2-domain scores climb by about 30 per 64-key tile, so the running maximum of most rows grows by more than 2^8
    between tiles and the kernel rescales O, A, l and mu; a missed rescale of A or mu leaves out_t off by a factor 2^-30 or more
    in a term.  q_t is orthogonal to the ramp direction and k_t is small, so S_t stays moderate."""
    lq, lk, h = 700, 1000, 2
    g = torch.Generator().manual_seed(11)
    u = torch.ones(D) / D ** 0.5
    q, k, v = torch.randn(1, lq, h, D, generator=g), torch.randn(1, lk, h, D, generator=g), torch.randn(1, lk, h, D, generator=g)
    a = 4.0
    q = 8.0 * (q - (q @ u)[..., None] * u) + a * u
    k = k + (30.0 * (torch.arange(lk) // BK) / (a * SM * LOG2E))[None, :, None, None] * u
    q_t = torch.randn(1, lq, h, D, generator=g)
    q_t = q_t - (q_t @ u)[..., None] * u
    k_t, v_t = 0.125 * torch.randn(1, lk, h, D, generator=g), torch.randn(1, lk, h, D, generator=g)
    ins = [t.to(dtype).cuda() for t in (q, k, v, q_t, k_t, v_t)]
    s = torch.einsum("bqhd,bkhd->bhqk", ins[0].to(F64), ins[1].to(F64))[0] * (SM * LOG2E)
    tiles = torch.nn.functional.pad(s, (0, -lk % BK), value=-math.inf).view(h, lq, -1, BK).amax(-1)
    run = torch.cummax(tiles, -1).values
    rescaled = ((run[..., 1:] - run[..., :-1]) > 8).any(-1).float().mean().item()
    assert tiles.amax(-1).min() > 300 and rescaled > 0.9, (tiles.amax(-1).min(), rescaled)
    out, out_t = _jvp(*ins)
    want, _ = exact_f64(*ins)
    _check_primal(out, want, ("large scores", dtype))
    ours, ref = _check_tangent(out_t, ins, f"large scores {dtype} (rescaling rows {rescaled:.3f})")
    assert ours <= REL, ours


# ------------------------------------------------------------------------------------------------------------ masking
@pytest.mark.parametrize("poison", [float("nan"), 1e4], ids=["nan", "1e4"])
@pytest.mark.parametrize("lk", [77, 130])
def test_memory_beyond_lk_is_never_used(cuda, lk, poison):
    """k, v, k_t and v_t are the first lk rows of larger allocations whose other rows hold NaN or 1e4: both outputs equal,
    bit for bit, those of tight copies."""
    ins = _inputs(1, 300, lk, 2, BF16, seed=lk)
    views = list(ins)
    for i in (1, 2, 4, 5):
        big = torch.full((1, 256, 2, D), poison, dtype=BF16, device="cuda")
        big[:, :lk] = ins[i]
        views[i] = big[:, :lk]
        assert views[i].is_contiguous() and views[i].data_ptr() == big.data_ptr()
    out, out_t = _jvp(*views)
    ref, ref_t = _jvp(*ins)
    assert torch.isfinite(out).all() and torch.isfinite(out_t).all()
    assert torch.equal(out, ref) and torch.equal(out_t, ref_t)


def test_rows_beyond_lq_are_not_stored(cuda):
    """The C entry point on output buffers longer than lq: rows >= lq of both keep their sentinel."""
    from turbodiffusion_b200 import _lib
    lq, lk, h, extra = 333, 226, 2, 120
    ins = _inputs(1, lq, lk, h, BF16, seed=9)
    big, big_t = (torch.full((1, lq + extra, h, D), 7.0, dtype=BF16, device="cuda") for _ in range(2))
    _lib.check(_lib.lib().tdb200_attn_dense_jvp(*(t.data_ptr() for t in ins), _lib.DTYPE_TAG[BF16], big.data_ptr(),
                                                big_t.data_ptr(), 1, lq, lk, h, D, SM, _lib.stream_ptr(ins[0].device)),
               "attn_dense_jvp")
    out, out_t = _jvp(*ins)
    assert torch.equal(big[:, :lq], out) and torch.equal(big_t[:, :lq], out_t)
    assert (big[:, lq:] == 7.0).all() and (big_t[:, lq:] == 7.0).all()


# ------------------------------------------------------------------------------------------------------------ layout, bits
def test_views_of_projection_outputs_give_the_bits_of_contiguous_copies(cuda):
    """q, k, v and their tangents as [l, h*d] matrices (GEMM outputs); their .view(1, l, h, d) is consumed in place."""
    lq, lk, h = 500, 226, 3
    g = torch.Generator().manual_seed(5)
    mats = [torch.randn(l, h * D, generator=g).bfloat16().cuda() for l in (lq, lk, lk, lq, lk, lk)]
    views = [m.view(1, m.shape[0], h, D) for m in mats]
    assert all(t.is_contiguous() and t.data_ptr() == m.data_ptr() for t, m in zip(views, mats))
    out, out_t = _jvp(*views)
    ref, ref_t = _jvp(*(t.clone() for t in views))
    assert torch.equal(out, ref) and torch.equal(out_t, ref_t)
    _check_tangent(out_t, views, "views")


@pytest.mark.parametrize("dtype", DTYPES)
def test_bits_are_reproducible_and_independent_of_the_other_heads(cuda, dtype):
    ins = _inputs(2, 700, 300, 3, dtype, seed=31)
    out, out_t = _jvp(*ins)
    again, again_t = _jvp(*ins)
    assert torch.equal(out, again) and torch.equal(out_t, again_t)
    one, one_t = _jvp(*(t[1:2, :, 2:3].contiguous() for t in ins))
    assert torch.equal(one, out[1:2, :, 2:3]) and torch.equal(one_t, out_t[1:2, :, 2:3])


def test_cuda_graph_replay_matches_eager(cuda):
    ins = _inputs(1, 900, 512, 2, BF16, seed=41)
    eager, eager_t = _jvp(*ins)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured, captured_t = _jvp(*ins)
    captured.zero_()
    captured_t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured, eager) and torch.equal(captured_t, eager_t)


# ------------------------------------------------------------------------------------------------------------ full size
@pytest.mark.parametrize("lk", [512, 32760], ids=["cross", "self"])
def test_shape_a_on_sampled_rows(cuda, lk):
    """Wan2.1-1.3B at 480p: 32760 queries, 12 heads of 128, over 512 text keys or all 32760 tokens; 64 sampled query rows per
    head against exact float64 rows (a row's output and tangent depend only on its own q and q_t)."""
    lq, h, n = 32760, 12, 64
    g = torch.Generator(device="cuda").manual_seed(51)
    q, q_t = (torch.randn(1, lq, h, D, generator=g, device="cuda").bfloat16() for _ in range(2))
    k, v, k_t, v_t = (torch.randn(1, lk, h, D, generator=g, device="cuda").bfloat16() for _ in range(4))
    out, out_t = _jvp(q, k, v, q_t, k_t, v_t)
    assert torch.isfinite(out).all() and torch.isfinite(out_t).all()
    rows = torch.stack([torch.randperm(lq, generator=torch.Generator().manual_seed(60 + i))[:n] for i in range(h)]).cuda()
    rows[:, 0], rows[:, 1] = 0, lq - 1
    heads = torch.arange(h, device="cuda")[:, None]
    pick = lambda t: t[0][rows, heads].transpose(0, 1)[None]                    # [1, n, h, D]
    ins = [pick(q), k, v, pick(q_t), k_t, v_t]
    want, _ = exact_f64(*ins)
    _check_primal(pick(out), want, ("shape A", lk))
    _check_tangent(pick(out_t), ins, f"shape A, {lk} keys, {n} rows x {h} heads")
