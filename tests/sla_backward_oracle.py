"""Closed-form backward of the block-sparse softmax attention (oracle/td_oracle.py `sparse_attention`), in float64: the
reference for the SparseLinearAttention backward kernels (csrc/sla_attn_bwd.cu).  FlashAttention-2's formulation with the
row statistics of the forward: lse (log2 units) and delta = rowsum(dO * O).  Test infrastructure only.  Tensors are
[B, H, L, D] like td_oracle.sparse_attention; lut [B, H, Mblk, topk] key-block ids.

The second half holds what the GPU float64 tests of the attention kernels share, on the module layout [B, L, H, D] and on
whatever device the tensors live: the large-score and entry-split input builders, the long-list inputs, the closed-form
dQ / dK / dV of one block given float64 (or any) lse and delta, the module's block selection, sentinel-filled output
buffers, seeded GPU inputs, the linear branch's feature maps, the library's last error, and two rounding points of the
forward kernels' restatements (the lazily rescaled running maximum and the fp16 linear-branch operand)."""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

D, BK = 128, 64
SM = D ** -0.5
LOG2E = 1.0 / math.log(2.0)
F64 = torch.float64
U = torch.ones(D) / D ** 0.5                      # the direction the magnitude ramps of the input builders live on


def cdiv(a: int, b: int) -> int:
    return (a + b - 1) // b


def _block_cols(lut_row, blkk: int, lk: int):
    ids = lut_row.long()
    cols = (ids[:, None] * blkk + torch.arange(blkk)[None, :]).reshape(-1)
    return cols.clamp_max(lk - 1), cols < lk


def sparse_attention_lse(q, k, lut, blkq: int = 128, blkk: int = 64, sm_scale: Optional[float] = None) -> torch.Tensor:
    """Row log-sum-exp of the block-sparse scores in log2 units (scores scaled by sm_scale * log2(e)), float64 [B,H,L]: the
    statistic the training-path forward saves (SLA/kernel.py:33-82 keeps the same quantity for its backward)."""
    b, h, l, d = q.shape
    sm_scale = d ** -0.5 if sm_scale is None else sm_scale
    out = torch.empty(b, h, l, dtype=torch.float64)
    for bi in range(b):
        for hi in range(h):
            for mi in range(cdiv(l, blkq)):
                r0, r1 = mi * blkq, min(l, (mi + 1) * blkq)
                cidx, valid = _block_cols(lut[bi, hi, mi], blkk, k.shape[2])
                s = (q[bi, hi, r0:r1].double() @ k[bi, hi, cidx].double().t()) * (sm_scale * math.log2(math.e))
                s = s.masked_fill(~valid[None, :], float("-inf"))
                out[bi, hi, r0:r1] = torch.logsumexp(s * math.log(2.0), -1) / math.log(2.0)
    return out


def sparse_attention_bwd_dq(q, k, v, d_o, lut, lse, delta, bi: int, hi: int, mi: int, blkq: int = 128, blkk: int = 64,
                            sm_scale: Optional[float] = None) -> torch.Tensor:
    """Closed-form dQ of one query block of sparse_attention (FlashAttention-2's backward, in float64), given the row
    statistics lse (log2 units, sparse_attention_lse) and delta = rowsum(dO * O), both [B,H,L]:
        P = 2^(S sm_scale log2(e) - lse),  dS = P * (dO V^T - delta),  dQ = sm_scale dS K.   q,k,v,d_o [B,H,L,D]."""
    l, d = q.shape[2], q.shape[3]
    sm_scale = d ** -0.5 if sm_scale is None else sm_scale
    r0, r1 = mi * blkq, min(l, (mi + 1) * blkq)
    cidx, valid = _block_cols(lut[bi, hi, mi], blkk, k.shape[2])
    kb, vb = k[bi, hi, cidx].double() * valid[:, None], v[bi, hi, cidx].double() * valid[:, None]
    s = (q[bi, hi, r0:r1].double() @ kb.t()) * (sm_scale * math.log2(math.e))
    p = torch.exp2(s - lse[bi, hi, r0:r1].double()[:, None]).masked_fill(~valid[None, :], 0.0)
    ds = p * (d_o[bi, hi, r0:r1].double() @ vb.t() - delta[bi, hi, r0:r1].double()[:, None])
    return sm_scale * ds @ kb


def sparse_attention_bwd_dkdv(q, k, v, d_o, lut, lse, delta, bi: int, hi: int, ni: int, blkq: int = 128, blkk: int = 64,
                              sm_scale: Optional[float] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Closed-form (dK, dV) of key block `ni` (its valid rows), float64: the sum over every query block whose LUT row selects
    it (each selection counted) of dV = P^T dO and dK = sm_scale dS^T Q, with P, dS as in sparse_attention_bwd_dq.  A key
    block that no query block selects gets zeros."""
    l, d = q.shape[2], q.shape[3]
    lk = k.shape[2]
    sm_scale = d ** -0.5 if sm_scale is None else sm_scale
    c0, c1 = ni * blkk, min(lk, (ni + 1) * blkk)
    kb, vb = k[bi, hi, c0:c1].double(), v[bi, hi, c0:c1].double()
    dk = torch.zeros(c1 - c0, d, dtype=torch.float64)
    dv = torch.zeros(c1 - c0, d, dtype=torch.float64)
    for mi in range(cdiv(l, blkq)):
        times = int((lut[bi, hi, mi].long() == ni).sum())
        if times == 0:
            continue
        r0, r1 = mi * blkq, min(l, (mi + 1) * blkq)
        qb, gb = q[bi, hi, r0:r1].double(), d_o[bi, hi, r0:r1].double()
        p = torch.exp2((qb @ kb.t()) * (sm_scale * math.log2(math.e)) - lse[bi, hi, r0:r1].double()[:, None])
        ds = p * (gb @ vb.t() - delta[bi, hi, r0:r1].double()[:, None])
        dv += times * (p.t() @ gb)
        dk += times * sm_scale * (ds.t() @ qb)
    return dk, dv


# ------------------------------------------------------------------------------------------------------------ [B, L, H, D]
def block_mask(lut, nblk):
    """[B,H,Mblk,topk] LUT -> bool [B,H,Mblk,Nblk].  Every LUT here lists a key block at most once per row."""
    b, h, m, _ = lut.shape
    return torch.zeros(b, h, m, nblk, dtype=torch.bool, device=lut.device).scatter_(-1, lut.long(), True)


def ref_dq(q, k, v, d_o, bm, blkq, ref, b, hi, mi, sm_scale=SM):
    """Closed-form float64 dQ of query block mi (its valid rows), given ref["lse"] and ref["delta"] [B,H,L]."""
    l = q.shape[1]
    r0, r1 = mi * blkq, min(l, (mi + 1) * blkq)
    cols = bm[b, hi, mi][torch.arange(k.shape[1], device=q.device) // BK].nonzero().squeeze(-1)
    kc, vc = k[b, cols, hi].to(F64), v[b, cols, hi].to(F64)
    s = (q[b, r0:r1, hi].to(F64) @ kc.t()) * (sm_scale * LOG2E)
    p = torch.exp2(s - ref["lse"][b, hi, r0:r1, None].to(F64))
    ds = p * (d_o[b, r0:r1, hi].to(F64) @ vc.t() - ref["delta"][b, hi, r0:r1, None].to(F64))
    return sm_scale * ds @ kc


def ref_dkdv(q, k, v, d_o, bm, blkq, ref, b, hi, ni, sm_scale=SM):
    """Closed-form float64 (dK, dV) of key block ni (its valid rows): the sum over every query row whose block selects it."""
    l = q.shape[1]
    c0, c1 = ni * BK, min(k.shape[1], (ni + 1) * BK)
    rows = bm[b, hi, :, ni][torch.arange(l, device=q.device) // blkq].nonzero().squeeze(-1)
    qr, gr = q[b, rows, hi].to(F64), d_o[b, rows, hi].to(F64)
    kc, vc = k[b, c0:c1, hi].to(F64), v[b, c0:c1, hi].to(F64)
    p = torch.exp2((qr @ kc.t()) * (sm_scale * LOG2E) - ref["lse"][b, hi, rows, None].to(F64))
    ds = p * (gr @ vc.t() - ref["delta"][b, hi, rows, None].to(F64))
    return sm_scale * ds.t() @ qr, p.t() @ gr


# Large-score patterns.  The q-scaling ones are the INT8 lazy-rescale tests' (test_gpu_sla.py): pattern, q scale, L, ratio.
#   all          every row scaled: log2-domain scores spread over tens of units, running maxima jump by more than 8
#   half_warp    rows r with r % 16 < 8: one of the two rows each thread of a 16-row warp slice holds
#   one_warp     the first 16 rows of every query block: one warp (of warpgroup 0 on 128-row blocks)
#   ragged_last  the maximum of many rows sits in the ragged last key block
# Entry-split patterns (hand-made LUTs; on 64-row blocks warpgroup g takes the entries j = g mod 2).  Every LUT row lists
# pairs (2i, 2i + 1) of key blocks in ascending order, so odd LUT positions always hold odd key blocks, and a magnitude ramp
# on K per key block places the scores:
#   split_dominant  odd blocks 140 + 12 i above the even ones: the row maximum lies in warpgroup 1's entries, more than 128
#                   log2 units above all warpgroup 0 sees (exp2 of the difference taken the wrong way round overflows fp32)
#   split_merge     even blocks at 10 i, odd ones at 10 i + 14, times a per-row factor in [1, 4]: both warpgroups rescale,
#                   and warpgroup 1 ends about 14 to 56 units above warpgroup 0, so both states enter the merge
SCALED = {"all_x8": ("all", 8.0, 1280, 0.5), "all_x16": ("all", 16.0, 700, 1.0), "half_warp": ("half_warp", 16.0, 640, 1.0),
          "one_warp": ("one_warp", 16.0, 640, 1.0), "ragged_last": ("ragged_last", 12.0, 1000, 1.0)}
SPLIT = ("split_dominant", "split_merge")


def randn_qkv(l, h, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(1, l, h, D, generator=g) for _ in range(3)]


def scaled_case(name, blkq, h=2, seed=0):
    """(q, k, v [1, L, H, D] float32 on the CPU, the module's top-k ratio) of a SCALED pattern."""
    pattern, qscale, l, ratio = SCALED[name]
    q, k, v = randn_qkv(l, h, 4000 + l + seed)
    rows = torch.arange(l)
    if pattern in ("all", "ragged_last"):
        q = q * qscale
    elif pattern == "half_warp":
        q[:, (rows % 16) < 8] *= qscale
    elif pattern == "one_warp":
        q[:, (rows % blkq) < 16] *= qscale
    if pattern == "ragged_last":
        q = q + 2.0 * qscale * U
        k[:, -(l % BK):] += 6.0 * U
    return q, k, v, ratio


def pair_lut(h, mblk, npairs, keep, seed):
    """[1,h,mblk,2*keep] int32: per row `keep` of the `npairs` pairs (2i, 2i+1), ascending."""
    g = torch.Generator().manual_seed(seed)
    lut = torch.empty(1, h, mblk, 2 * keep, dtype=torch.int32)
    for hi in range(h):
        for mi in range(mblk):
            pairs = torch.randperm(npairs, generator=g)[:keep].sort().values
            lut[0, hi, mi] = torch.stack([2 * pairs, 2 * pairs + 1], -1).flatten()
    return lut


def split_case(name, blkq, h=2, seed=0):
    """(q, k, v [1, L, H, D] float32 on the CPU, lut) of a SPLIT pattern.  L = 1240: 20 key blocks (the last one 24 keys, odd:
    in warpgroup 1's entries), ragged last query block."""
    l, a = 1240, 4.0
    q, k, v = randn_qkv(l, h, 7000 + seed)
    q = q - (q @ U)[..., None] * U                           # q orthogonal to U, then a chosen component along it
    g = torch.Generator().manual_seed(8000 + seed)
    alpha = torch.ones(1, l, h, 1) if name == "split_dominant" else 1.0 + 3.0 * torch.rand(1, l, h, 1, generator=g)
    q = q + a * alpha * U
    n = torch.arange(cdiv(l, BK))
    if name == "split_dominant":
        offset = torch.where(n % 2 == 1, 140.0 + 12.0 * (n // 2), torch.zeros(()))
    else:
        offset = 10.0 * (n // 2) + 14.0 * (n % 2)
    c = (offset / (a * SM * LOG2E)).repeat_interleave(BK)[:l]    # score offset of key block n = alpha * offset[n]
    k = k + c[None, :, None, None] * U
    return q, k, v, pair_lut(h, cdiv(l, blkq), 10, 7, 9000 + seed + blkq)


def long_inputs(l, h, dtype, seed):
    """randn q, k, v on the GPU plus a ramp of 6 log2 units over the key blocks (later blocks weigh up to 64x more), so that
    every part of a long LUT row, its last entries included, carries a visible share of each row's softmax mass."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v = (torch.randn(1, l, h, D, generator=g, device="cuda") for _ in range(3))
    a, u = 4.0, U.cuda()
    q = q - (q @ u)[..., None] * u + a * u
    ramp = 6.0 * (torch.arange(l, device="cuda") // BK) / (cdiv(l, BK) - 1)
    k = k + (ramp / (a * SM * LOG2E))[None, :, None, None] * u
    return [t.to(dtype) for t in (q, k, v)]


def block_map_lut(q, k, blkq, topk, blkk=BK):
    """The module's block selection (mean pooling over blocks, top-k of the pooled scores), ascending [B,H,Mblk,topk], of
    16-bit q, k [B, L, H, D] on the GPU."""
    from turbodiffusion_b200.SLA.utils import block_map_from_pools, mean_pool
    qh, kh = (t.transpose(1, 2).contiguous() for t in (q, k))
    return block_map_from_pools(mean_pool(qh, blkq), mean_pool(kh, blkk), topk)[1].contiguous()


def sentinel_buffers(dtype, dev, pad_rows, sentinel, *shapes):
    """Flat buffers filled with `sentinel`, pad_rows rows longer than each [..., l, h, d] shape (a row: h * d values):
    (views of the shapes, the pads after them)."""
    views, pads = [], []
    for shape in shapes:
        n = math.prod(shape)
        buf = torch.full((n + pad_rows * shape[-2] * shape[-1],), sentinel, dtype=dtype, device=dev)
        views.append(buf[:n].view(*shape))
        pads.append(buf[n:])
    return views, pads


def running_max(ent_max, two_warpgroups):
    """The row maximum each entry's P is formed against in the SLA forward kernels ([R, entries] float32, in list order):
    the first entry of a warpgroup sets it, and it moves only when an entry's maximum exceeds it by more than 2^8 (the lazy
    rescale).  The 64-row kernels run one such sequence per warpgroup, over alternate entries."""
    m = ent_max.clone()
    for j in range(2 if two_warpgroups else 1, ent_max.shape[1]):
        prev = m[:, j - 2] if two_warpgroups else m[:, j - 1]
        m[:, j] = torch.where(ent_max[:, j] > prev + 8.0, ent_max[:, j], prev)
    return m


def round_operand(a, dtype):
    """T(a) as the fused forwards form the linear branch's MMA operand: in fp16 a row whose max lies outside [2^-6, 2^15) is
    rounded as a * 2^sc with sc = clamp(14 - floor(log2 max), -64, 64), and the power of two divided out again (sla_attn.cu)."""
    if dtype == torch.bfloat16:
        return a.to(dtype).double()
    amax = a.amax(-1, keepdim=True)
    e = torch.frexp(amax.clamp_min(1e-300)).exponent - 1          # floor(log2 amax)
    sc = (14 - e).clamp(-64, 64).double()
    sc = torch.where(((amax > 0) & (amax < 2.0 ** -6)) | (amax >= 2.0 ** 15), sc, torch.zeros_like(sc))
    return (a * torch.exp2(sc)).to(dtype).double() * torch.exp2(-sc)


def randn(shape, dtype, seed, scale=1.0):
    """randn * scale in `dtype` on the GPU, from its own seeded generator."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def phi(x, feature):
    """The linear branch's feature map (SLA/core.py:57-73): 0 softmax over the channels, 1 elu + 1, 2 relu."""
    if feature == 0:
        return torch.softmax(x, -1)
    if feature == 1:
        return torch.nn.functional.elu(x) + 1
    return torch.relu(x)


def last_error():
    """The library's message for its last failed call."""
    from turbodiffusion_b200._lib import lib
    msg = lib().tdb200_last_error()
    return msg.decode() if msg else ""
