"""Seeded inputs, float64 statistics and references for the linear-branch operand of the fused SLA forwards.

Every fused inference forward ends in linear_branch_store (csrc/sla_attn.cu), which adds A . KVW^T to the softmax
accumulator with one more MMA, A_j = T(phi_j * l / den), den = 1e-5 + sum_j phi_j ksum_j, l the unnormalised softmax row sum
(>= 1, and up to 2^8 x the number of selected keys under the lazy rescale).  bf16 holds A whatever its magnitude; fp16
overflows above 65504 and goes subnormal below 2^-14.  The builders here reach each regime in the module's [B, L, H, D]
layout (tests/test_sla_linear_branch_range_host.py on the CPU, tests/test_gpu_sla_linear_branch_range.py on the kernels):

  dead_relu_*      relu map, d/8 channels J on which every key is negative (ksum_J = 0, kv[:, J] = 0) and the dead query
                   rows positive only on J: den = 1e-5 and A_J ~ 1e5 l, against a KVW column of zeros.  The exact linear
                   branch of those rows is 0.  Row patterns: every other row; the first 16 rows of every 64-row group (one
                   warp); the rows of the ragged last 128-row query block
  partial_dead     dead_relu_alternate with a few keys slightly positive on J: den small but not 1e-5, A above 65504 and an
                   exact linear branch of order one
  softmax_outlier  softmax map, k_c set to a constant a and q_c lowered by a in one channel c: a per-row constant shift of the
                   scores (the attention part and the key smoothing are unchanged), while phi(k) concentrates on c and phi(q)
                   avoids it, so den is small and max A passes 65504
  peaked_*         elu or relu map, q x 8 (l of 1 to 2) over 32760 keys (75600 for peaked_elu_75600): den grows with L and
                   every A falls below 2^-14.  v carries a per-channel mean and proj_l has weights of scale 1/sqrt(d), so the
                   linear branch is comparable to the softmax part; the mean is scaled to put max |KVW| in [2^14, 2^15)
  ordinary         randn inputs and the softmax map (max A near 1): the control

KVW's own fp16 range is not this regime's subject: KVW = T(proj_w . kv) grows with L * E[phi] * mean(v), and the training
path and the reference round kvsum at the same place, so every builder keeps max |KVW| < 2^15.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

F64 = torch.float64
LOG2E = 1.0 / math.log(2.0)
FEATURE = {"softmax": 0, "elu": 1, "relu": 2}
FP16_MAX, FP16_MIN_NORMAL = 65504.0, 2.0 ** -14
# a row whose max A lies outside [2^-6, 2^15) is rescaled in fp16 so that its max A lands in [2^14, 2^15)
SCALE_LO, SCALE_HI, SCALE_TARGET = -6, 15, 14


def cdiv(a, b):
    return (a + b - 1) // b


# ------------------------------------------------------------------------------------------------------------ builders
# name: (feature map, L, batch, heads, topk ratio, allowed head dims)
CASES = {
    "dead_relu_alternate": ("relu", 2000, 2, 2, 0.5, (128, 64)),
    "dead_relu_warp": ("relu", 2000, 2, 2, 0.5, (128, 64)),
    "dead_relu_ragged": ("relu", 2000, 2, 2, 0.5, (128, 64)),
    "partial_dead": ("relu", 2000, 2, 2, 0.5, (128, 64)),
    "softmax_outlier": ("softmax", 4040, 2, 2, 0.5, (128, 64)),
    "peaked_elu": ("elu", 32760, 1, 2, 0.2, (128, 64)),
    "peaked_relu": ("relu", 32760, 1, 2, 0.2, (128, 64)),
    "peaked_elu_75600": ("elu", 75600, 1, 1, 0.1, (128,)),
    "ordinary": ("softmax", 2000, 2, 2, 0.5, (128, 64)),
}
OUTLIER_A = 20.0
PARTIAL_EPS, PARTIAL_KEYS = 2.0 ** -16, 4
KVW_TARGET = 1.5 * 2.0 ** 14


def dead_channels(d):
    return torch.arange(3, d, 8)


def dead_rows(name, l):
    """bool [L]: the rows built dead (q positive only on the dead channels), or None."""
    r = torch.arange(l)
    if name in ("dead_relu_alternate", "partial_dead"):
        return r % 2 == 0
    if name == "dead_relu_warp":
        return r % 64 < 16
    if name == "dead_relu_ragged":
        return r >= (l // 128) * 128
    return None


def phi_k(k, feature):
    """phi(k) as the moments use it: evaluated in fp32 from T-rounded k and rounded to T (the reference module's rounding
    point, SLA/core.py), then widened to float64.  In fp16 small phi(k) entries flush to zero, in kv and ksum alike."""
    return phi(k.float(), feature).to(k.dtype).to(F64)


def kvw_exact(k, v, w, feature):
    """float64 proj_w . kv [B, H, D_out, D_k] from T-rounded k, v and T(phi(k)) (CPU or GPU)."""
    pk = phi_k(k, feature)
    kv = torch.einsum("blhj,blhc->bhcj", pk, v.to(F64))
    return torch.einsum("oc,bhcj->bhoj", w.to(F64), kv)


def build(name, d, dtype, seed=0):
    """(q, k, v in dtype [B, L, H, D] on the CPU, proj_w [D, D] fp32, proj_b [D] fp32, info dict)."""
    feature, l, b, h, ratio, dims = CASES[name]
    assert d in dims, (name, d)
    g = torch.Generator().manual_seed(1000 * d + seed + sum(map(ord, name)))
    q, k, v = (torch.randn(b, l, h, d, generator=g) for _ in range(3))
    w = torch.randn(d, d, generator=g) * 0.05
    bias = torch.randn(d, generator=g) * 0.05
    info = {"feature": feature, "ratio": ratio, "dead": dead_rows(name, l)}
    if name.startswith("dead_relu") or name == "partial_dead":
        j = dead_channels(d)
        k[..., j] = -(k[..., j].abs() + 0.5)
        rows = info["dead"]
        qd = -(q[:, rows].abs() + 0.01)
        qd[..., j] = q[:, rows][..., j].abs() + 1.0
        q[:, rows] = qd
        if name == "partial_dead":
            keys = torch.randperm(l, generator=g)[:PARTIAL_KEYS]
            k[:, keys.unsqueeze(-1), :, j] = PARTIAL_EPS
            v[:, keys] = v[:, keys] + 4.0
    elif name == "softmax_outlier":
        c = d // 2 + 1
        k[..., c] = OUTLIER_A
        q[..., c] -= OUTLIER_A
    elif name.startswith("peaked"):
        q = q * 8.0
        w = torch.randn(d, d, generator=g) / math.sqrt(d)
        mu = torch.randn(d, generator=g)
        noise = v
        for _ in range(3):   # KVW is affine in the mean: two steps put max |KVW| on the target
            v = noise + mu
            kq, vq = k.to(dtype), v.to(dtype)
            mx = kvw_exact(kq, vq, w, feature).abs().max().item()
            mu = mu * (KVW_TARGET / mx)
        v = noise + mu
    return q.to(dtype), k.to(dtype), v.to(dtype), w, bias, info


# ------------------------------------------------------------------------------------------------------------ float64 pieces
def phi(x, feature):
    """The feature map of the linear branch, in the precision of x."""
    if feature == "softmax":
        return torch.softmax(x, -1)
    if feature == "elu":
        return F.elu(x) + 1.0
    return torch.relu(x)


def pooled_lut(q, k, blkq, blkk, ratio):
    """The module's block selection restated: top int(ratio * nblk) key blocks per query block by the score of the block
    means (the key mean the kernels subtract shifts a row's block scores by a constant).  Ascending int32 [B, H, Mblk, topk].
    Near-ties may order differently from the kernel; the GPU tests use the kernel's own selection."""
    b, l, h, d = q.shape
    lk = k.shape[1]
    mblk, nblk = cdiv(l, blkq), cdiv(lk, blkk)
    qp = F.pad(q.to(F64), (0, 0, 0, 0, 0, mblk * blkq - l)).view(b, mblk, blkq, h, d).sum(2)
    qp = qp / torch.tensor([min(blkq, l - i * blkq) for i in range(mblk)], dtype=F64, device=q.device)[None, :, None, None]
    kp = F.pad(k.to(F64), (0, 0, 0, 0, 0, nblk * blkk - lk)).view(b, nblk, blkk, h, d).sum(2)
    kp = kp / torch.tensor([min(blkk, lk - i * blkk) for i in range(nblk)], dtype=F64, device=q.device)[None, :, None, None]
    s = torch.einsum("bmhd,bnhd->bhmn", qp, kp)
    topk = max(1, min(nblk, int(ratio * nblk)))
    return s.topk(topk, -1).indices.sort(-1).values.to(torch.int32)


def _rows_mask(lut, rows, blkq, blkk, lk):
    """bool [len(rows), Lk]: the keys the query rows `rows` attend to under `lut` [Mblk, topk] (one batch entry and head)."""
    nblk = cdiv(lk, blkk)
    bm = torch.zeros(lut.shape[0], nblk, dtype=torch.bool, device=lut.device).scatter_(-1, lut.long(), True)
    return bm[rows // blkq][:, torch.arange(lk, device=lut.device) // blkk]


def head_terms(q, k, feature, bi, hi, rows):
    """float64 (phi(q) [R, D], ksum [D] of T(phi(k)), den [R]) of rows `rows` of batch entry bi, head hi."""
    pq = phi(q[bi, rows, hi].to(F64), feature)
    ksum = phi_k(k[bi, :, hi], feature).sum(0)
    return pq, ksum, 1e-5 + pq @ ksum


def row_l(q, k, lut, blkq, blkk, bi, hi, rows, sm_scale):
    """float64 l_min = sum exp2(s - max s) over each row's selected keys (scores from q, k)."""
    s = (q[bi, rows, hi].to(F64) @ k[bi, :, hi].to(F64).t()) * (sm_scale * LOG2E)
    s = s.masked_fill(~_rows_mask(lut[bi, hi], rows, blkq, blkk, k.shape[1]), -math.inf)
    return torch.exp2(s - s.amax(-1, keepdim=True)).sum(-1)


def stats(q, k, v, w, bias, info, lut, blkq, blkk, kvw=None, rows=None, dtype=None):
    """float64 statistics of the linear-branch operand over every (batch, head) and the rows `rows` (all by default):
    max_a [B, H, R] = max_j phi_j l_min / den; sub_frac = fraction of the significant A_j (within 2^24 of their row's max)
    below 2^-14; kvw_max = max |KVW| (KVW as given, else T(proj_w . kv) in float64); out_max = max |exact
    output| of the rows (float64 attention + phi(q) KVW^T / den + b)."""
    b, l, h, d = q.shape
    sm = d ** -0.5
    feature = info["feature"]
    rows = torch.arange(l, device=q.device) if rows is None else rows.to(q.device)
    kvw = kvw_exact(k, v, w, feature).to(dtype or q.dtype) if kvw is None else kvw
    max_a = torch.empty(b, h, len(rows), dtype=F64, device=q.device)
    n_sig = n_sub = 0
    out_max = 0.0
    for bi in range(b):
        for hi in range(h):
            pq, ksum, den = head_terms(q, k, feature, bi, hi, rows)
            lm = row_l(q, k, lut, blkq, blkk, bi, hi, rows, sm)
            a = pq * (lm / den)[:, None]
            am = a.amax(-1)
            max_a[bi, hi] = am
            sig = a >= am[:, None] * 2.0 ** -24
            n_sig += int(sig.sum())
            n_sub += int((sig & (a < FP16_MIN_NORMAL)).sum())
            o = attention_rows(q, k, v, lut, blkq, blkk, bi, hi, rows, sm) + (pq @ kvw[bi, hi].to(F64).t()) / den[:, None]
            out_max = max(out_max, (o + bias.to(F64).to(q.device)).abs().max().item())
    return {"max_a": max_a, "sub_frac": n_sub / max(1, n_sig),
            "kvw_max": kvw.to(F64).abs().max().item(), "out_max": out_max}


def attention_rows(q, k, v, lut, blkq, blkk, bi, hi, rows, sm_scale):
    """float64 block-sparse softmax attention of rows `rows` of (bi, hi) over `lut`."""
    s = (q[bi, rows, hi].to(F64) @ k[bi, :, hi].to(F64).t()) * sm_scale
    s = s.masked_fill(~_rows_mask(lut[bi, hi], rows, blkq, blkk, k.shape[1]), -math.inf)
    return torch.softmax(s, -1) @ v[bi, :, hi].to(F64)


# ------------------------------------------------------------------------------------------------------------ emulation
def fp16_row_shift(amax):
    """The power-of-two exponent linear_branch_store's fp16 instantiations scale a row's A by: 0 inside [2^-6, 2^15),
    else the one that puts max A in [2^14, 2^15), within [-64, 64]."""
    e = torch.floor(torch.log2(amax.clamp_min(1e-300)))
    out = (e >= SCALE_HI) | ((amax > 0) & (e < SCALE_LO))
    return torch.where(out, (SCALE_TARGET - e).clamp(-64, 64), torch.zeros_like(e))


def emulate_linear_branch(pq, ksum, l, kvw, dtype, rescale=False):
    """linear_branch_store's operand arithmetic for rows with phi(q) pq [R, D] (from T-rounded q), ksum [D] and row sums
    l [R]: A = T(phi * (l / den)) in fp32, and with `rescale` the fp16 row scaling; returns the linear branch
    (A . KVW^T) / l [R, D_out] in float64 (the MMA's products and sum taken exactly)."""
    pq32, ks32 = pq.float(), ksum.float()
    den = 1e-5 + pq32 @ ks32
    cscale = l.float() / den
    sc = torch.zeros_like(cscale)
    if rescale:
        sc = fp16_row_shift((pq32.amax(-1) * cscale).to(F64)).float()
    a = (pq32 * (cscale * torch.exp2(sc))[:, None]).to(dtype)
    return (a.to(F64) @ kvw.to(F64).t()) * (torch.exp2(-sc.to(F64)) / l.to(F64))[:, None]
