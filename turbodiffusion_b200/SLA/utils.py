"""Mirror of turbodiffusion/SLA/utils.py: mean_pool, get_block_map, get_cuda_arch (H100 implementation)."""
from __future__ import annotations

import os

import torch

from .. import _ops
from .._lib import DTYPE_TAG, check, lib, ptr, require_cuda, stream_ptr


def cdiv(a, b):
    return (a + b - 1) // b


# The SpargeAttn kernel family this package serves (see get_cuda_arch); changed with set_served_arch().
SERVED_ARCH = "sm100"
SAGE_BLOCKS = {"sm100": (128, 64), "sm90": (64, 128)}   # (BLKQ, BLKK) of each family, SLA/core.py:191-193


def set_served_arch(arch: str) -> str:
    """Select the SpargeAttn kernel family get_cuda_arch reports, and with it SageSLA's block sizes: "sm100" (the default,
    the Sage2++ family, BLKQ=128 / BLKK=64) or "sm90" (the Hopper family the reference picks on an H100, BLKQ=64 /
    BLKK=128).  Returns the previous value.  Both families run on the H100.  Sequence parallelism (dist.py) serves both:
    its hooks are built for one family (`SequenceParallel.install(model, mode, sage_arch=...)`, "sm100" by default) and
    raise NotImplementedError, at install and at every call, while the served arch names the other."""
    global SERVED_ARCH
    if arch not in SAGE_BLOCKS:
        raise ValueError(f"served arch must be one of {sorted(SAGE_BLOCKS)}, got {arch!r}")
    prev, SERVED_ARCH = SERVED_ARCH, arch
    return prev


# SparseLinearAttention's linear branch in training (see set_linear_branch).
LINEAR_BRANCH = "reference"
LINEAR_BRANCHES = ("reference", "fused")


def set_linear_branch(name: str) -> str:
    """Select how SparseLinearAttention's training forward computes the linear branch and proj_l: "reference" (the default,
    torch ops at the reference's rounding points, SLA/core.py:104-117) or "fused" (SLA.core.linear_branch: the CUDA forward
    and backward of tdb200_sla_linear_fwd / _bwd).  Read at every call; returns the previous value.  Calls that carry a
    forward-mode tangent (forward_jvp, torch.func.jvp, forward_ad) take the reference branch under either setting."""
    global LINEAR_BRANCH
    if name not in LINEAR_BRANCHES:
        raise ValueError(f"linear branch must be one of {list(LINEAR_BRANCHES)}, got {name!r}")
    prev, LINEAR_BRANCH = LINEAR_BRANCH, name
    return prev


# SageSparseLinearAttention's P.V arithmetic (see set_sage_pv).
SAGE_PV_MODES = ("bf16", "fp8")


def _sage_pv_default():
    mode = os.environ.get("TDB200_SAGE_PV") or "bf16"
    if mode not in SAGE_PV_MODES:
        raise ValueError(f"TDB200_SAGE_PV must be one of {list(SAGE_PV_MODES)}, got {mode!r}")
    return mode


SAGE_PV = _sage_pv_default()


def set_sage_pv(mode: str) -> str:
    """Select SageSparseLinearAttention's P.V: "bf16" (16-bit P and V, the default unless the environment variable
    TDB200_SAGE_PV names the other) or "fp8" (SageAttention2's arithmetic: e4m3 P and V with per-channel V scales,
    tdb200_sla_quant_v_fp8 + tdb200_sla_attn_fwd_fp8v; both block families, d = 128 only).  Read at every call, by the module
    and by the LTX adapters in SLA.core; returns the previous value.  Under "fp8", 64-wide heads raise NotImplementedError, and
    so do sequence parallelism's install and hooks (dist.py)."""
    global SAGE_PV
    if mode not in SAGE_PV_MODES:
        raise ValueError(f"sage P.V must be one of {list(SAGE_PV_MODES)}, got {mode!r}")
    prev, SAGE_PV = SAGE_PV, mode
    return prev


def get_cuda_arch(device_index):
    """SLA/utils.py:70-71.  The reference (SLA/core.py:191-193, 211-235) and the LTX client (acceleration.py:286-378) use this
    value only to choose a SpargeAttn kernel family and its block sizes: sm80/86/87 -> fp16-V kernels, sm90 -> the
    BLKQ=64 / BLKK=128 Hopper kernels, anything else -> the Sage2++ entry with BLKQ=128 / BLKK=64.  This package implements
    the last two (as the fused kernel) on every GPU, H100 included, and reports the one chosen with set_served_arch()
    ("sm100" unless changed), so callers take a branch whose entry points exist here.  The device's compute capability is
    torch.cuda.get_device_capability()."""
    torch.cuda.get_device_capability(device_index)   # an invalid device index raises like the reference's call
    return SERVED_ARCH


class QKPrep:
    """Outputs of tdb200_sla_quant_qk for q,k in the module layout [B, L, H, D]."""
    __slots__ = ("kmean", "q_i8", "q_scale", "k_i8", "k_scale", "q_pool", "k_pool", "mblk", "nblk", "k_seq_major")


def quant_qk(q: torch.Tensor, k: torch.Tensor, lk: int = None, blkq: int = 128, blkk: int = 64) -> QKPrep:
    """One pass over q, two over k: key mean, pooled block means (SLA/utils.py:21-52), Sage INT8 Q / smoothed-K
    (SLA/core.py:197-203).  q [B, Lq, H, D], k [B, >=lk, H, D] contiguous bf16/fp16; only the first `lk` key rows are
    used (sequence-parallel callers pass the gathered, tail-padded key slab).  (blkq, blkk): (128, 64) or (64, 128)."""
    require_cuda(q, k)
    b, lq, h, d = q.shape
    lk = k.shape[1] if lk is None else lk
    assert k.shape[0] == b and k.shape[2:] == q.shape[2:] and lk <= k.shape[1]
    assert q.is_contiguous() and k.is_contiguous() and (b == 1 or lk == k.shape[1])
    o = QKPrep()
    o.mblk, o.nblk, o.k_seq_major = cdiv(lq, blkq), cdiv(lk, blkk), False
    o.kmean, o.q_i8, o.q_scale, o.k_i8, o.k_scale, o.q_pool, o.k_pool = _ops.sla_quant_qk(q, k, lk, blkq, blkk)
    return o


def quant_q_only(q: torch.Tensor, blkq: int = 128) -> QKPrep:
    """The query half of quant_qk (pooled means + Sage INT8 of q); fill in the key half later with quant_k_into()."""
    require_cuda(q)
    o = QKPrep()
    o.mblk, o.k_seq_major = cdiv(q.shape[1], blkq), False
    o.q_i8, o.q_scale, o.q_pool = _ops.sla_quant_q(q, blkq)
    return o


def quant_k_into(o: QKPrep, k: torch.Tensor, lk: int, blkk: int = 64) -> QKPrep:
    """The key half of quant_qk on the first `lk` rows of k [B, >=lk, H, D]."""
    require_cuda(k)
    o.nblk = cdiv(lk, blkk)
    o.kmean, o.k_i8, o.k_scale, o.k_pool = _ops.sla_quant_k(k, lk, blkk)
    return o


def kmean_partials(k: torch.Tensor) -> torch.Tensor:
    """Column sums of each 128-row chunk of k [B, rows, H, D] -> [B, H, ceil(rows/128), D] fp32: stage one of the key mean
    (the partials tdb200_sla_quant_qk forms internally; a sequence-parallel rank computes those of its own rows)."""
    require_cuda(k)
    b, rows, h, d = k.shape
    out = torch.empty(b, h, cdiv(rows, 128), d, dtype=torch.float32, device=k.device)
    check(lib().tdb200_sla_kmean_partial(ptr(k), DTYPE_TAG[k.dtype], b, rows, h, d, ptr(out), stream_ptr(k.device)),
          "sla_kmean_partial")
    return out


def kmean_from_partials(partials: torch.Tensor, l_total: int) -> torch.Tensor:
    """Stage two: partials [B, H, chunks, D] fp32 (contiguous, in global chunk order) -> kmean [B, H, D] fp32."""
    require_cuda(partials)
    b, h, chunks, d = partials.shape
    assert partials.is_contiguous() and partials.dtype == torch.float32
    out = torch.empty(b, h, d, dtype=torch.float32, device=partials.device)
    check(lib().tdb200_sla_kmean_final(ptr(partials), b, h, chunks, d, l_total, ptr(out), stream_ptr(partials.device)),
          "sla_kmean_final")
    return out


def quant_k_seq(k: torch.Tensor, kmean: torch.Tensor, k_i8=None, blkk: int = 64):
    """Smoothed Sage INT8 of the rows of k [B, rows, H, D] against a given key mean, per `blkk` (64 or 128) rows: (k_i8
    [B, rows, H, D] int8 -- the input layout --, k_scale [B, H, ceil(rows/blkk)] fp32, k_pool [B, H, ceil(rows/blkk), D])."""
    require_cuda(k, kmean)
    b, rows, h, d = k.shape
    nb = cdiv(rows, blkk)
    k_i8 = torch.empty(b, rows, h, d, dtype=torch.int8, device=k.device) if k_i8 is None else k_i8
    k_scale = torch.empty(b, h, nb, dtype=torch.float32, device=k.device)
    k_pool = torch.empty(b, h, nb, d, dtype=k.dtype, device=k.device)
    check(lib().tdb200_sla_quant_k_seq(ptr(k), ptr(kmean), DTYPE_TAG[k.dtype], b, rows, h, d, ptr(k_i8), ptr(k_scale),
                                       ptr(k_pool), blkk, stream_ptr(k.device)), "sla_quant_k_seq")
    return k_i8, k_scale, k_pool


def seq_topks(seq_lens: torch.Tensor, ratio, blkk: int) -> torch.Tensor:
    """Per-entry blocks per row for lengths seq_lens (int32 [B]): topk_i = max(1, min(nblk_i, int(ratio * nblk_i))) with
    nblk_i = ceil(n_i / blkk), the modules' rule on each entry's own key-block count, evaluated on the lengths' device in float64
    (Python's int(ratio * nblk) truncates the same float64 product), so device lengths are never read on the host."""
    nblk = torch.div(seq_lens + (blkk - 1), blkk, rounding_mode="floor")    # lengths are in [0, L]: no int32 overflow
    nb = nblk.to(torch.float64)
    # min(nblk, int(x)) == int(min(nblk, x)) for an integer nblk; the conversion truncates toward zero, as int() does
    return torch.clamp(torch.minimum(nb * float(ratio), nb).to(torch.int32), min=1)


def quant_qk_vl(q: torch.Tensor, k: torch.Tensor, seq_lens: torch.Tensor, blkq: int, blkk: int) -> QKPrep:
    """quant_qk (or, at (64, 64), quant_q_only + quant_k_into) of a padded batch q, k [B, L, H, 128] whose entry i owns its
    first seq_lens[i] rows (int32 [B] on q's device): tdb200_sla_quant_qk_vl, one call per half where the pair is not a SageSLA
    family.  Entry i's codes, scales and pools over its rows are those of the call on entry i alone."""
    require_cuda(q, k, seq_lens)
    b, l, h, d = q.shape
    o = QKPrep()
    o.mblk, o.nblk, o.k_seq_major = cdiv(l, blkq), cdiv(l, blkk), False
    o.q_i8, o.q_scale, o.q_pool = _ops._q_half(q, blkq)
    o.kmean, o.k_i8, o.k_scale, o.k_pool = _ops._k_half(k, l, blkk)
    other = {128: 64, 64: 128}
    if (blkq, blkk) in SAGE_BLOCKS.values():
        halves = ((q, k, blkq, blkk),)
    else:   # the key block size only matters to the key half and the query block size to the query half
        halves = ((q, None, blkq, other[blkq]), (None, k, other[blkk], blkk))
    for qq, kk, bq, bk in halves:
        qh, kh = qq is not None, kk is not None
        check(lib().tdb200_sla_quant_qk_vl(ptr(qq) if qh else None, ptr(kk) if kh else None, DTYPE_TAG[q.dtype], b, l, h, d,
                                           ptr(seq_lens), ptr(o.kmean) if kh else None, ptr(o.q_i8) if qh else None,
                                           ptr(o.q_scale) if qh else None, ptr(o.k_i8) if kh else None,
                                           ptr(o.k_scale) if kh else None, ptr(o.q_pool) if qh else None,
                                           ptr(o.k_pool) if kh else None, bq, bk, stream_ptr(q.device)),
              "sla_quant_qk_vl", launches=(1 if qh else 0) + (3 if kh else 0))
    return o


def block_map_vl(q_pool: torch.Tensor, k_pool: torch.Tensor, topk: int, seq_lens: torch.Tensor, topks: torch.Tensor,
                 blkq: int, blkk: int):
    """block_map_from_pools per entry (tdb200_sla_block_map_vl): entry i selects topks[i] of its own ceil(n_i / blkk) key blocks
    for each of its ceil(n_i / blkq) query blocks.  Returns (sparse_map int8 [B,H,Mblk,Nblk], lut int32 [B,H,Mblk,topk]); LUT
    entries past topks[i] and rows past entry i's query blocks are -1, the map 0 there."""
    b, h, mblk, d = q_pool.shape
    nblk = k_pool.shape[2]
    sparse_map = torch.empty(b, h, mblk, nblk, dtype=torch.int8, device=q_pool.device)
    lut = torch.empty(b, h, mblk, topk, dtype=torch.int32, device=q_pool.device)
    check(lib().tdb200_sla_block_map_vl(ptr(q_pool), ptr(k_pool), DTYPE_TAG[q_pool.dtype], b, h, mblk, nblk, d, topk,
                                        ptr(seq_lens), ptr(topks), blkq, blkk, ptr(sparse_map), ptr(lut),
                                        stream_ptr(q_pool.device)), "sla_block_map_vl")
    return sparse_map, lut


def block_map_from_pools(q_pool: torch.Tensor, k_pool: torch.Tensor, topk: int):
    """Pooled score + top-k (SLA/utils.py:59-66).  Returns (sparse_map int8 [B,H,Mblk,Nblk], lut int32 ascending)."""
    return _ops.sla_block_map(q_pool, k_pool, topk)


def mean_pool(x: torch.Tensor, BLK: int) -> torch.Tensor:
    """SLA/utils.py:44-52 for x [B, H, L, D]; BLK in {64, 128}.  (Uses the fused prepass on a [B,L,H,D] view.)"""
    assert x.is_contiguous() and BLK in (64, 128)
    xt = x.transpose(1, 2).contiguous()
    if BLK == 128:
        return quant_q_only(xt).q_pool
    # 64-row blocks: the key half of the prepass pools (k - mean_L k); adding the T-rounded mean back gives the plain
    # block means up to one rounding of T (the reference pools the tensor it is handed, SLA/utils.py:44-52)
    prep = quant_k_into(QKPrep(), xt, xt.shape[1])
    return (prep.k_pool.float() + prep.kmean.to(x.dtype).float()[:, :, None, :]).to(x.dtype)


def get_block_map(q: torch.Tensor, k: torch.Tensor, topk_ratio: float, BLKQ: int = 128, BLKK: int = 64):
    """SLA/utils.py:55-67.  q,k [B, H, L, D].  Returns (sparse_map int8, lut int32 [B,H,Mblk,topk] ascending, topk).
    NOTE the reference returns the unsorted torch.topk indices (int64) as `lut`; only the SET is defined
    (sorted=False), and SageSLA rebuilds an ascending LUT from the map anyway (SLA/core.py:204).  (BLKQ, BLKK) is one of the
    two SageSLA families, (128, 64) or (64, 128) (SLA/core.py:191-193)."""
    assert (BLKQ, BLKK) in SAGE_BLOCKS.values(), f"block sizes BLKQ={BLKQ}, BLKK={BLKK}: this implementation serves (128, 64) and (64, 128)"
    prep = quant_qk(q.transpose(1, 2).contiguous(), k.transpose(1, 2).contiguous(), blkq=BLKQ, blkk=BLKK)
    nblk = prep.nblk
    topk = min(nblk, int(topk_ratio * nblk))
    sparse_map, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
    sparse_map._tdb200_lut = lut   # SLA.core.block_map_lut_triton hands this back instead of rebuilding it from the map
    return sparse_map, lut, topk
