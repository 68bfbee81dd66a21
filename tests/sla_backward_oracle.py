"""Closed-form backward of the block-sparse softmax attention (oracle/td_oracle.py `sparse_attention`), in float64: the
reference for the SparseLinearAttention backward kernels (csrc/sla_attn_bwd.cu).  FlashAttention-2's formulation with the
row statistics of the forward: lse (log2 units) and delta = rowsum(dO * O).  Test infrastructure only.  Tensors are
[B, H, L, D] like td_oracle.sparse_attention; lut [B, H, Mblk, topk] key-block ids."""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch


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
