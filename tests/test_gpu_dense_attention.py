"""GPU checks of the dense attention operator (ops.dense_attention, tdb200_attn_dense_fwd): parity with the oracle and with
F.scaled_dot_product_attention, masking of the ragged tails, large score magnitudes (the lazy rescale), agreement with the
sparse 16-bit kernel on a full block list, the [l, h*d] layout, reproducibility, CUDA-graph capture, and shape A's
cross-attention at full size on sampled rows.

Bars: cos >= 0.999 and rel-L2 <= 5e-3 against the oracle (fp32 attention of the same 16-bit inputs), and the kernel's
rel-L2 at most 1.5x that of F.scaled_dot_product_attention on the GPU for the same inputs."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import td_oracle as O

pytestmark = pytest.mark.gpu
D, BK = 128, 128                                  # head dim; the kernel's key tile
SM = D ** -0.5
LOG2E = 1.0 / math.log(2.0)
F64 = torch.float64
BF16, FP16 = torch.bfloat16, torch.float16
DTYPES = [pytest.param(BF16, id="bf16"), pytest.param(FP16, id="fp16")]
COS, REL = 0.999, 5e-3


def _stats(got, want):
    a, b = got.to(F64).flatten().cpu(), want.to(F64).flatten().cpu()
    return {"rel_l2": ((a - b).norm() / b.norm().clamp_min(1e-300)).item(),
            "cos": (torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-300)).item()}


def _inputs(b, lq, lk, h, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(b, lq, h, D, generator=g)
    k, v = torch.randn(b, lk, h, D, generator=g), torch.randn(b, lk, h, D, generator=g)
    return [t.to(dtype).cuda() for t in (q, k, v)]


def _oracle(q, k, v, sm_scale=SM):
    """oracle.dense_attention on fp32 CPU copies of the 16-bit inputs; [B, L, H, D] in and out."""
    qh, kh, vh = (t.float().cpu().transpose(1, 2) for t in (q, k, v))
    return O.dense_attention(qh, kh, vh, sm_scale).transpose(1, 2)


def _sdpa(q, k, v, sm_scale=SM):
    """torch's SDPA on the GPU, fed the transposed views block.py feeds it."""
    return F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), scale=sm_scale).transpose(1, 2)


def _dense(q, k, v, sm_scale=None):
    from turbodiffusion_b200 import ops
    return ops.dense_attention(q, k, v, sm_scale)


def _check(out, want, what):
    s = _stats(out, want)
    assert s["cos"] >= COS and s["rel_l2"] <= REL, (what, s)
    return s


# ------------------------------------------------------------------------------------------------------------ parity
SHAPES = [(1, 1000, 512, 3), (2, 700, 77, 2), (1, 130, 1, 1), (1, 1, 226, 2), (1, 1182, 1182, 2)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b,lq,lk,h", [pytest.param(*s, id="x".join(map(str, s))) for s in SHAPES])
def test_parity_with_the_oracle_and_sdpa(cuda, b, lq, lk, h, dtype):
    q, k, v = _inputs(b, lq, lk, h, dtype, seed=lq + lk)
    out = _dense(q, k, v)
    assert out.shape == q.shape and out.dtype == dtype and out.is_contiguous() and torch.isfinite(out).all()
    want = _oracle(q, k, v)
    s = _check(out, want, (b, lq, lk, h, dtype))
    r = _stats(_sdpa(q, k, v), want)
    print(f"({b}, {lq}, {lk}, {h}) {dtype}: kernel rel-L2 {s['rel_l2']:.2e} cos {s['cos']:.7f} | SDPA rel-L2 {r['rel_l2']:.2e}")
    assert s["rel_l2"] <= 1.5 * r["rel_l2"] + 1e-7, ("kernel", s, "SDPA", r)
    if lk == 1:                                   # softmax over one key is 1: the output is that key's value row
        assert torch.equal(out, v.expand(b, lq, h, D))


def test_float32_inputs_run_in_bf16_and_sm_scale_is_passed_on(cuda):
    q, k, v = (t.float() for t in _inputs(1, 200, 300, 2, BF16, seed=3))
    out = _dense(q, k, v, sm_scale=0.5 * SM)
    assert out.dtype == torch.float32
    assert torch.equal(out, _dense(q.bfloat16(), k.bfloat16(), v.bfloat16(), sm_scale=0.5 * SM).float())
    _check(out, _oracle(q, k, v, 0.5 * SM), "sm_scale")


# ------------------------------------------------------------------------------------------------------------ masking
@pytest.mark.parametrize("poison", [float("nan"), 1e4], ids=["nan", "1e4"])
@pytest.mark.parametrize("lk", [77, 130])
def test_memory_beyond_lk_is_never_used(cuda, lk, poison):
    """k and v are the first lk rows of a larger allocation whose other rows hold NaN or 1e4: the key tiles that reach past lk
    must come back zero-filled and masked, so the output equals, bit for bit, that of tight copies."""
    q, k, v = _inputs(1, 300, lk, 2, BF16, seed=lk)
    big_k, big_v = (torch.full((1, 256, 2, D), poison, dtype=BF16, device="cuda") for _ in range(2))
    big_k[:, :lk], big_v[:, :lk] = k, v
    kk, vv = big_k[:, :lk], big_v[:, :lk]
    assert kk.is_contiguous() and kk.data_ptr() == big_k.data_ptr() and vv.data_ptr() == big_v.data_ptr()
    out = _dense(q, kk, vv)
    assert torch.isfinite(out).all() and torch.equal(out, _dense(q, k, v))


def test_rows_beyond_lq_are_not_stored(cuda):
    """The C entry point on an output buffer longer than lq: rows >= lq keep their sentinel."""
    from turbodiffusion_b200 import _lib
    lq, lk, h, extra = 333, 226, 2, 120
    q, k, v = _inputs(1, lq, lk, h, BF16, seed=9)
    big = torch.full((1, lq + extra, h, D), 7.0, dtype=BF16, device="cuda")
    _lib.check(_lib.lib().tdb200_attn_dense_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), _lib.DTYPE_TAG[BF16], big.data_ptr(),
                                                1, lq, lk, h, D, SM, _lib.stream_ptr(q.device)), "attn_dense_fwd")
    assert torch.equal(big[:, :lq], _dense(q, k, v))
    assert (big[:, lq:] == 7.0).all()


# ------------------------------------------------------------------------------------------------------------ large scores
def large_score_inputs(lq, lk, h, seed):
    """fp32 q, k, v [1, l, h, D] whose log2-domain scores climb by about 60 per 128-key tile (a ramp on k along a direction
    q has a fixed component on), with q's other components scaled by 8 so that one key per row stands well above the rest."""
    g = torch.Generator().manual_seed(seed)
    u = torch.ones(D) / D ** 0.5
    q, k, v = torch.randn(1, lq, h, D, generator=g), torch.randn(1, lk, h, D, generator=g), torch.randn(1, lk, h, D, generator=g)
    a = 4.0
    q = 8.0 * (q - (q @ u)[..., None] * u) + a * u
    ramp = 60.0 * (torch.arange(lk) // BK)
    k = k + (ramp / (a * SM * LOG2E))[None, :, None, None] * u
    return q, k, v


def reference_f64(q, k, v, sm_scale=SM):
    """Float64 attention of [1, L, H, D] tensors: (out, per-tile maxima of the log2-domain scores [H, Lq, tiles], softmax
    weight of each row's heaviest key [H, Lq])."""
    qh, kh, vh = (t[0].to(F64).transpose(0, 1) for t in (q, k, v))
    s = (qh @ kh.transpose(-1, -2)) * (sm_scale * LOG2E)
    lk = s.shape[-1]
    tiles = F.pad(s, (0, -lk % BK), value=-math.inf).view(*s.shape[:-1], -1, BK).amax(-1)
    p = torch.softmax(s * math.log(2.0), -1)
    return (p @ vh).transpose(0, 1)[None], tiles, p.amax(-1)


@pytest.mark.parametrize("dtype", DTYPES)
def test_large_scores_take_the_lazy_rescale(cuda, dtype):
    q, k, v = (t.to(dtype).cuda() for t in large_score_inputs(700, 1000, 2, seed=11))
    want, tiles, top = reference_f64(q, k, v)
    run = torch.cummax(tiles, -1).values
    rescaled = ((run[..., 1:] - run[..., :-1]) > 8).any(-1).float().mean().item()   # the kernel's threshold: 2^8
    assert tiles.amax(-1).min() > 300 and rescaled > 0.9 and top.median() > 0.5, (tiles.amax(-1).min(), rescaled, top.median())
    out = _dense(q, k, v)
    assert torch.isfinite(out).all()
    s = _check(out, want, ("large scores", dtype))
    print(f"large scores {dtype}: row maxima {tiles.amax(-1).min().item():.0f}..{tiles.amax().item():.0f} (log2), rescaling rows "
          f"{rescaled:.3f}, median top weight {top.median().item():.3f}, rel-L2 {s['rel_l2']:.2e}")


# ------------------------------------------------------------------------------------------------------------ sparse kernel
@pytest.mark.parametrize("blkq", [128, 64])
def test_agrees_with_the_sparse_16bit_kernel_on_a_full_block_list(cuda, blkq):
    """Same per-tile arithmetic, different tiles: 64-key tiles from a LUT that lists every key block, against 128-key tiles.
    The tile width decides the running maximum P is rounded to T against, so the two kernels round P differently and are
    not bit-equal: on these inputs they sit 2.3e-3 (128-row blocks) and 2.5e-3 (64-row blocks) apart in bf16, the distance
    each has from the oracle (2.3e-3).  The bar: no further from each other than 1.5x the larger of those two distances
    (independent errors of that size would be 1.41x apart), and inside the oracle bar."""
    from turbodiffusion_b200.SLA.core import attn_fwd_qk16_lse
    l, h = 1000, 2
    q, k, v = _inputs(1, l, l, h, BF16, seed=21)
    mblk, nblk = -(-l // blkq), -(-l // 64)
    lut = torch.arange(nblk, dtype=torch.int32, device="cuda").expand(1, h, mblk, nblk).contiguous()
    o_s, _ = attn_fwd_qk16_lse(q, k, v, lut, nblk, SM, blkq=blkq)
    out, want = _dense(q, k, v), _oracle(q, k, v)
    s, d, r = _stats(out, o_s), _check(out, want, "dense"), _check(o_s, want, "sparse")
    print(f"dense vs sparse 16-bit (blkq {blkq}): rel-L2 {s['rel_l2']:.2e}; vs the oracle: dense {d['rel_l2']:.2e}, sparse "
          f"{r['rel_l2']:.2e}")
    assert s["rel_l2"] <= min(REL, 1.5 * max(d["rel_l2"], r["rel_l2"])), (s, d, r)


# ------------------------------------------------------------------------------------------------------------ layout, bits
def test_views_of_projection_outputs_give_the_bits_of_contiguous_copies(cuda):
    """block.py holds q, k, v as [l, h*d] matrices (GEMM outputs); their .view(1, l, h, d) is consumed as it is."""
    lq, lk, h = 500, 226, 3
    g = torch.Generator().manual_seed(5)
    mq, mk, mv = (torch.randn(l, h * D, generator=g).bfloat16().cuda() for l in (lq, lk, lk))
    views = [m.view(1, m.shape[0], h, D) for m in (mq, mk, mv)]
    assert all(t.is_contiguous() and t.data_ptr() == m.data_ptr() for t, m in zip(views, (mq, mk, mv)))
    out = _dense(*views)
    assert torch.equal(out, _dense(*(t.clone() for t in views)))
    _check(out, _oracle(*views), "views")
    # a head-major tensor seen as [b, l, h, d] is not in the kernel's layout: the function copies it, the values are the same
    qt = views[0].transpose(1, 2).contiguous().transpose(1, 2)
    assert not qt.is_contiguous() and torch.equal(_dense(qt, views[1], views[2]), out)


@pytest.mark.parametrize("dtype", DTYPES)
def test_bits_are_reproducible_and_independent_of_the_other_heads(cuda, dtype):
    q, k, v = _inputs(2, 700, 300, 3, dtype, seed=31)
    out = _dense(q, k, v)
    assert torch.equal(out, _dense(q, k, v))
    one = _dense(*(t[1:2, :, 2:3].contiguous() for t in (q, k, v)))
    assert torch.equal(one, out[1:2, :, 2:3])


def test_cuda_graph_replay_matches_eager(cuda):
    q, k, v = _inputs(1, 900, 512, 2, BF16, seed=41)
    eager = _dense(q, k, v)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = _dense(q, k, v)
    captured.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured, eager)


# ------------------------------------------------------------------------------------------------------------ full size
def test_shape_a_cross_attention_on_sampled_rows(cuda):
    """Wan2.1-1.3B at 480p: 32760 queries, 512 text keys, 12 heads of 128; 256 sampled query rows per head against the oracle."""
    lq, lk, h, n = 32760, 512, 12, 256
    g = torch.Generator(device="cuda").manual_seed(51)
    q = torch.randn(1, lq, h, D, generator=g, device="cuda").bfloat16()
    k, v = (torch.randn(1, lk, h, D, generator=g, device="cuda").bfloat16() for _ in range(2))
    out = _dense(q, k, v)
    assert torch.isfinite(out).all()
    rows = torch.stack([torch.randperm(lq, generator=torch.Generator().manual_seed(60 + i))[:n] for i in range(h)]).cuda()   # [h, n]
    rows[:, 0], rows[:, 1] = 0, lq - 1
    heads = torch.arange(h, device="cuda")[:, None]
    q_s = q[0][rows, heads].transpose(0, 1)[None]                              # [1, n, h, D]
    want = _oracle(q_s, k, v)
    s = _check(out[0][rows, heads].transpose(0, 1)[None], want, "shape A sampled")
    r = _stats(_sdpa(q, k, v)[0][rows, heads].transpose(0, 1)[None], want)
    print(f"shape A cross-attention, {n} rows x {h} heads: kernel rel-L2 {s['rel_l2']:.2e} cos {s['cos']:.7f} | SDPA rel-L2 "
          f"{r['rel_l2']:.2e}")
    assert s["rel_l2"] <= 1.5 * r["rel_l2"], ("kernel", s, "SDPA", r)
