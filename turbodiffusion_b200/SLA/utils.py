"""Mirror of turbodiffusion/SLA/utils.py: mean_pool, get_block_map, get_cuda_arch (H100 implementation)."""
from __future__ import annotations

import torch

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
    dev = q.device
    mblk, nblk = cdiv(lq, blkq), cdiv(lk, blkk)
    o = QKPrep()
    o.mblk, o.nblk = mblk, nblk
    o.kmean = torch.empty(b, h, d, dtype=torch.float32, device=dev)
    o.q_i8 = torch.empty(b, h, lq, d, dtype=torch.int8, device=dev)
    o.k_i8 = torch.empty(b, h, lk, d, dtype=torch.int8, device=dev)
    o.q_scale = torch.empty(b, h, mblk, dtype=torch.float32, device=dev)
    o.k_scale = torch.empty(b, h, nblk, dtype=torch.float32, device=dev)
    o.q_pool = torch.empty(b, h, mblk, d, dtype=q.dtype, device=dev)
    o.k_pool = torch.empty(b, h, nblk, d, dtype=q.dtype, device=dev)
    check(lib().tdb200_sla_quant_qk_blocks(ptr(q), ptr(k), DTYPE_TAG[q.dtype], b, lq, lk, h, d, ptr(o.kmean), ptr(o.q_i8),
                                           ptr(o.q_scale), ptr(o.k_i8), ptr(o.k_scale), ptr(o.q_pool), ptr(o.k_pool), blkq, blkk,
                                           stream_ptr(dev)), "sla_quant_qk_blocks")
    return o


def quant_q_only(q: torch.Tensor, blkq: int = 128) -> QKPrep:
    """The query half of quant_qk (pooled means + Sage INT8 of q); fill in the key half later with quant_k_into()."""
    require_cuda(q)
    b, lq, h, d = q.shape
    dev = q.device
    o = QKPrep()
    o.mblk = cdiv(lq, blkq)
    o.q_i8 = torch.empty(b, h, lq, d, dtype=torch.int8, device=dev)
    o.q_scale = torch.empty(b, h, o.mblk, dtype=torch.float32, device=dev)
    o.q_pool = torch.empty(b, h, o.mblk, d, dtype=q.dtype, device=dev)
    # the key block size only matters to the key half; any valid pair with this blkq serves
    check(lib().tdb200_sla_quant_qk_blocks(ptr(q), None, DTYPE_TAG[q.dtype], b, lq, lq, h, d, None, ptr(o.q_i8), ptr(o.q_scale),
                                           None, None, ptr(o.q_pool), None, blkq, 64 if blkq == 128 else 128, stream_ptr(dev)),
          "sla_quant_qk_blocks", launches=1)
    return o


def quant_k_into(o: QKPrep, k: torch.Tensor, lk: int, blkk: int = 64) -> QKPrep:
    """The key half of quant_qk on the first `lk` rows of k [B, >=lk, H, D]."""
    require_cuda(k)
    b, _, h, d = k.shape
    dev = k.device
    o.nblk = cdiv(lk, blkk)
    o.kmean = torch.empty(b, h, d, dtype=torch.float32, device=dev)
    o.k_i8 = torch.empty(b, h, lk, d, dtype=torch.int8, device=dev)
    o.k_scale = torch.empty(b, h, o.nblk, dtype=torch.float32, device=dev)
    o.k_pool = torch.empty(b, h, o.nblk, d, dtype=k.dtype, device=dev)
    check(lib().tdb200_sla_quant_qk_blocks(None, ptr(k), DTYPE_TAG[k.dtype], b, lk, lk, h, d, ptr(o.kmean), None, None,
                                           ptr(o.k_i8), ptr(o.k_scale), None, ptr(o.k_pool), 128 if blkk == 64 else 64, blkk,
                                           stream_ptr(dev)), "sla_quant_qk_blocks", launches=3)
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
    check(lib().tdb200_sla_quant_k_seq_blocks(ptr(k), ptr(kmean), DTYPE_TAG[k.dtype], b, rows, h, d, ptr(k_i8), ptr(k_scale),
                                              ptr(k_pool), blkk, stream_ptr(k.device)), "sla_quant_k_seq")
    return k_i8, k_scale, k_pool


def block_map_from_pools(q_pool: torch.Tensor, k_pool: torch.Tensor, topk: int):
    """Pooled score + top-k (SLA/utils.py:59-66).  Returns (sparse_map int8 [B,H,Mblk,Nblk], lut int32 ascending)."""
    b, h, mblk, d = q_pool.shape
    nblk = k_pool.shape[2]
    sparse_map = torch.empty(b, h, mblk, nblk, dtype=torch.int8, device=q_pool.device)
    lut = torch.empty(b, h, mblk, topk, dtype=torch.int32, device=q_pool.device)
    check(lib().tdb200_sla_block_map(ptr(q_pool), ptr(k_pool), DTYPE_TAG[q_pool.dtype], b, h, mblk, nblk, d, topk,
                                     ptr(sparse_map), ptr(lut), stream_ptr(q_pool.device)), "sla_block_map")
    return sparse_map, lut


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
