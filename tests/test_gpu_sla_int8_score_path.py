"""The INT8 SageSLA forward kernels (both block families, bf16 and fp16, 128- and 64-wide heads) against the fp32
block-sparse oracle on the kernel's own block map: the score-to-P path (row maxima on the int32 accumulator, the ragged last
key block on its own code path), and the linear-branch epilogue that reads the 16-bit query rows from shared memory and
stores the output through a TMA box that clips rows >= l.

Bars: every query block at cosine >= 0.999 and rel-L2 <= 2e-2 against the fp32 oracle (test_gpu_sla.py); the inputs with
large scores, whose INT8 quantisation error is itself larger, against the INT8 emulation at rel-L2 <= 3e-2 and the fp32 oracle
at cosine >= 0.99 (test_gpu_sla.py's lazy-rescale test).
"""
import pytest
import torch

from oracle import td_oracle as O

pytestmark = pytest.mark.gpu

FAMILIES = {"sm100": (128, 64), "sm90": (64, 128)}
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
FEATURES = {"softmax": 0, "elu": 1, "relu": 2}
PAD_ROWS = 37          # rows of the buffer after the output tensor, which the kernel must leave alone
SENTINEL = -1234.0     # exact in bf16 and fp16


def _qkv(l, h, d, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(1, l, h, d, generator=g)
    k = torch.randn(1, l, h, d, generator=g) + torch.randn(1, 1, h, d, generator=g) * 2.0
    v = torch.randn(1, l, h, d, generator=g)
    return q, k, v


def _attn(q, k, v, w, bias, blkq, blkk, topk, feature, cuda):
    """One call of tdb200_sla_attn_fwd on q, k, v [1, l, h, d] (CPU, 16-bit), into a buffer PAD_ROWS rows longer than the
    output and filled with SENTINEL.  Returns (out [1, l, h, d] on the CPU, the pad rows, the LUT on the CPU)."""
    from turbodiffusion_b200._lib import DTYPE_TAG, check, lib, ptr, stream_ptr
    from turbodiffusion_b200.SLA.core import linear_moments, project_moments
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, quant_qk
    b, l, h, d = q.shape
    qc, kc, vc = q.to(cuda), k.to(cuda), v.to(cuda)
    prep = quant_qk(qc, kc, blkq=blkq, blkk=blkk)
    topk = min(prep.nblk, topk)
    _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    kv, ksum = linear_moments(kc, vc, feature)
    kvw = project_moments(w.to(cuda), kv, q.dtype)
    pb = bias.float().to(cuda).contiguous()
    buf = torch.full(((l + PAD_ROWS) * h * d,), SENTINEL, dtype=q.dtype, device=cuda)
    check(lib().tdb200_sla_attn_fwd(ptr(prep.q_i8), ptr(prep.q_scale), ptr(prep.k_i8), ptr(prep.k_scale), ptr(vc), ptr(qc),
                                    DTYPE_TAG[q.dtype], ptr(lut), topk, ptr(kvw), ptr(ksum), ptr(pb), ptr(buf), b, l, l, h, d,
                                    d ** -0.5, feature, blkq, blkk, 0, stream_ptr(cuda)), "sla_attn_fwd")
    torch.cuda.synchronize()
    buf = buf.cpu()
    return buf[: l * h * d].view(1, l, h, d), buf[l * h * d:], lut.cpu()


def _weights(d, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(d, d, generator=g) * 0.05, torch.randn(d, generator=g) * 0.05


@pytest.mark.parametrize("feature", sorted(FEATURES))
@pytest.mark.parametrize("d", [128, 64])
@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_int8_forward_ragged_blocks_feature_maps_and_clipped_store(cuda, family, dtype, d, feature):
    """l = 1000: the last key block is ragged (40 valid keys of 64, 104 of 128), and the last query block ends inside the
    TMA box (104 of 128 rows, 40 of 64), so the output store must clip rows >= l: the buffer's pad rows keep the sentinel.
    Every query block selects all key blocks but one, so the ragged block is read."""
    blkq, blkk = FAMILIES[family]
    l, h = 1000, 2
    q, k, v = _qkv(l, h, d, 7000 + d + FEATURES[feature], torch.float32)
    if feature != "softmax":
        q = q * 0.5          # keep elu / relu features in a range where the linear branch matters
    q, k, v = (t.to(DTYPES[dtype]) for t in (q, k, v))
    w, bias = _weights(d, 9)
    nblk = (l + blkk - 1) // blkk
    out, pad, lut = _attn(q, k, v, w, bias, blkq, blkk, nblk - 1, FEATURES[feature], cuda)
    assert torch.equal(pad, torch.full_like(pad, SENTINEL)), "the kernel wrote past row l"
    assert torch.isfinite(out.float()).all()
    assert (lut == nblk - 1).any(), "no query block reads the ragged block"
    for head in range(h):
        for m in range((l + blkq - 1) // blkq):
            ref = O.sla_forward_block(q, k, v, w, bias, head, m, lut[0, head, m], blkq, blkk, dtype=q.dtype, mode="exact",
                                      feature_map=feature)
            got = out[0, m * blkq:min(l, (m + 1) * blkq), head]
            s = O.stats(got, ref)
            assert s["cos"] >= 0.999 and s["rel_l2"] <= 2e-2, (family, dtype, d, feature, head, m, s)


@pytest.mark.parametrize("d", [128, 64])
@pytest.mark.parametrize("dtype", sorted(DTYPES))
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_int8_forward_negative_first_block_then_lazy_rescale(cuda, family, dtype, d):
    """Dense selection, so every row walks the key blocks in order.  Every query has a common component along u; the keys of
    key block 0 point against u, so each row's first entry holds only negative scores (a negative integer row maximum), and
    the keys of the middle block point along u, so the running maximum grows there by far more than 2^8 (the lazy rescale of
    l and O), with the ragged last block after it."""
    blkq, blkk = FAMILIES[family]
    l, h = 1000, 2
    q, k, v = _qkv(l, h, d, 8000 + d, torch.float32)
    u = torch.ones(d) / d ** 0.5
    q = q * 0.25 + 6.0 * u
    mid = (l // blkk) // 2 * blkk
    k[:, :blkk] -= 6.0 * u
    k[:, mid:mid + blkk] += 16.0 * u
    q, k, v = (t.to(DTYPES[dtype]) for t in (q, k, v))
    w, bias = _weights(d, 10)
    nblk = (l + blkk - 1) // blkk
    out, pad, lut = _attn(q, k, v, w, bias, blkq, blkk, nblk, 0, cuda)
    assert torch.equal(pad, torch.full_like(pad, SENTINEL)), "the kernel wrote past row l"
    assert torch.isfinite(out.float()).all()

    # the kernel's scores (smoothed keys, log2 domain): block 0 all negative, the middle block's maximum more than 2^8 above
    qh, kh = q.transpose(1, 2).float(), k.transpose(1, 2).float()
    s = (qh @ (kh - kh.mean(-2, keepdim=True)).transpose(-1, -2)) * d ** -0.5 * 1.4426950408889634
    first, before, at = s[..., :blkk].amax(-1), s[..., :mid].amax(-1), s[..., mid:mid + blkk].amax(-1)
    assert (first < 0).float().mean() > 0.9, (first < 0).float().mean()
    assert (at - before > 8).float().mean() > 0.5, (at - before > 8).float().mean()

    sage = O.sla_forward(q, k, v, w, bias, 1.0, blkq, blkk, dtype=q.dtype, mode="sage", lut=lut)
    exact = O.sla_forward(q, k, v, w, bias, 1.0, blkq, blkk, dtype=q.dtype, mode="exact", lut=lut)
    s_sage, s_exact = O.stats(out, sage), O.stats(out, exact)
    assert s_sage["rel_l2"] <= 3e-2 and s_exact["cos"] >= 0.99, (family, dtype, d, s_sage, s_exact)
