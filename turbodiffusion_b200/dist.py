"""Sequence (video-token) parallelism for the hot path: one process per GPU, torch.distributed for the plumbing.

Every GEMM / norm / modulation / RoPE / FFN in the block is row-independent, so rank r simply owns the token rows
[row_begin, row_end).  Only self-attention needs an exchange (SURVEY 8e / BASELINE north star):

    1. all-gather of the local V slab (16-bit, [rows, H, D]) and of the local K rows -- as INT8 (Sage-quantised by the owning
       rank against the global key mean, whose 128-row partial sums are all-gathered first) plus per-block scales and pooled
       means, or as the 16-bit slab for the shapes the INT8 kernel does not serve -- into one [L_pad, H, D] slab per tensor;
    2. all-reduce (sum) of the linear-attention moments  phi(K)^T V  [H,D,D]  and  sum phi(K)  [H,D], which
       tdb200_sla_linear_moments accumulates over the LOCAL rows only;
    3. the block map over all key blocks and the fused attention over the gathered K/V run locally for this rank's query rows
       (with the 16-bit K exchange also the key mean / INT8 / pooling of the WHOLE key sequence, repeated on every rank).

Shard boundaries are multiples of 128 rows, so 128x128 quant blocks and the SageSLA blocks of either family (128-row query
and 64-row key blocks for "sm100", 64-row query and 128-row key blocks for "sm90"; 128 = max(BLKQ, BLKK) in both) never
straddle ranks and the result equals the single-GPU computation block for block.  The key mean is built from 128-row
partial sums in both families, so the gathered mean is the single-GPU one bit for bit.  Only the last rank may be short; the
all-gather pads it with zero rows at the very END of the sequence, so the gathered slab is simply the full tensor followed
by < 128*world padding rows that the kernels never read (lk = L).

The hooks run the SageSLA block family they were built for (`sage_arch`, "sm100" by default): a sequence-parallel model
under SLA.utils.set_served_arch("sm90") is installed with `SequenceParallel.install(model, mode, sage_arch="sm90")`.
Installing, or calling a hook, while the served arch names the other family raises NotImplementedError, since the
single-GPU module would then run one block geometry and the hooks the other.

The reference's own scheme is Ulysses all-to-all (rcm/utils/a2a_cp.py:66-182; heads <-> sequence), which needs
H % world == 0 (12 heads do not split 8 ways).  UlyssesAttention below implements it as the second mode: three all-to-alls
turn the local [rows, H, D] slabs of q, k, v into [L, H/world, D] (all rows, this rank's heads), the unchanged single-GPU SLA
forward runs on those heads, and a fourth all-to-all brings the output back to [rows, H, D].  Per rank and layer it moves
4*(N-1)/N^2 * L*dim*2 bytes instead of 2*(N-1)/N * L*dim*2 for the K/V all-gather (4x less at N = 8) and no rank repeats
the K-side preparation of the full sequence; `SequenceParallel.install(mode="auto")` picks it from four GPUs up
(see pick_mode).
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.distributed as dist

from .SLA import utils as sla_utils


def cdiv(a: int, b: int) -> int:
    return (a + b - 1) // b


def sage_blocks(sage_arch: str):
    """(BLKQ, BLKK) of a SageSLA family, "sm100" or "sm90" (SLA.utils.SAGE_BLOCKS)."""
    if sage_arch not in sla_utils.SAGE_BLOCKS:
        raise ValueError(f"sage_arch must be one of {sorted(sla_utils.SAGE_BLOCKS)}, got {sage_arch!r}")
    return sla_utils.SAGE_BLOCKS[sage_arch]


def require_served_arch(sage_arch: str) -> None:
    """Refuse, at install and at every hook call, to run `sage_arch`'s block sizes while a single GPU would run the other
    family's (SLA.utils.set_served_arch)."""
    served = sla_utils.SERVED_ARCH
    if served != sage_arch:
        bq, bk = sla_utils.SAGE_BLOCKS[sage_arch]
        sq, sk = sla_utils.SAGE_BLOCKS[served]
        raise NotImplementedError(f"sequence parallelism built for the {sage_arch} SageSLA family (BLKQ={bq}, BLKK={bk}) "
                                  f"while the served arch is {served!r} (BLKQ={sq}, BLKK={sk}); install it with "
                                  f"sage_arch={served!r} or select {sage_arch!r} with SLA.utils.set_served_arch")


def shard_rows(total_rows: int, world: int, rank: int, align: int = 128):
    """128-aligned contiguous shards; returns (row_begin, row_end, rows_per_rank_padded)."""
    blocks = cdiv(total_rows, align)
    per_rank = cdiv(blocks, world) * align
    begin = min(total_rows, rank * per_rank)
    end = min(total_rows, (rank + 1) * per_rank)
    return begin, end, per_rank


class GpuPrimitives:
    """The C-ABI kernels (default).  The CPU test injects oracle implementations with the same signatures.

    `int8_k`: the rank quantises its OWN key rows and the exchange carries INT8 K (+ per-block scales and pooled means) instead
    of 16-bit K; the key mean stays global and bit-identical to the single-GPU one because the ranks all-gather the 128-row
    partial sums the single-GPU reduction is built from (tdb200_sla_kmean_partial / _final).  Served by the 128-wide softmax
    kernels of both block families; other head dims / feature maps keep the 16-bit exchange.  `sage_arch` selects the block
    family (BLKQ, BLKK) every method works on."""

    def __init__(self, sla_module, sage_arch: str = "sm100"):
        self.sla = sla_module
        self.sage_arch = sage_arch
        self.blkq, self.blkk = sage_blocks(sage_arch)
        self.int8_k = (getattr(sla_module, "quantised_qk", True) and getattr(sla_module, "feature", 0) == 0
                       and os.environ.get("TDB200_SP_INT8_K", "1") != "0")       # "0": the 16-bit K exchange, for A/B timing

    def prepare_q(self, q):
        from .SLA.utils import quant_q_only
        return quant_q_only(q, self.blkq)

    def attention(self, q, k_full, v_full, lk, kv, ksum, qprep=None):
        from .SLA.core import attn_fwd, project_moments
        from .SLA.utils import block_map_from_pools, quant_k_into, quant_q_only
        sla = self.sla
        d = q.shape[-1]
        prep = quant_k_into(qprep if qprep is not None else quant_q_only(q, self.blkq), k_full, lk, self.blkk)
        topk = min(prep.nblk, int(sla.topk * prep.nblk))
        _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
        kvw = project_moments(sla.proj_l.weight, kv, q.dtype)
        return attn_fwd(prep, v_full, q, lut, topk, kvw, ksum, sla.proj_l.bias.float().contiguous(), d ** -0.5, lk=lk,
                        blkq=self.blkq, blkk=self.blkk)

    def moments(self, k_local, v_local):
        from .SLA.core import linear_moments
        return linear_moments(k_local, v_local)

    # ---- INT8-K exchange ------------------------------------------------------------------------------------------------
    def k_partials(self, k_local):
        from .SLA.utils import kmean_partials
        return kmean_partials(k_local)

    def k_mean(self, partials, l_total):
        from .SLA.utils import kmean_from_partials
        return kmean_from_partials(partials, l_total)

    def k_quant(self, k_local, kmean, k_i8_out=None):
        from .SLA.utils import quant_k_seq
        return quant_k_seq(k_local, kmean, k_i8_out, blkk=self.blkk)

    def attention_i8(self, q, qprep, k_i8_full, k_scale, k_pool, kmean, v_full, lk, kv, ksum):
        from .SLA.core import attn_fwd, project_moments
        from .SLA.utils import block_map_from_pools, quant_q_only
        sla = self.sla
        d = q.shape[-1]
        prep = qprep if qprep is not None else quant_q_only(q, self.blkq)
        prep.kmean, prep.k_i8, prep.k_scale, prep.k_pool = kmean, k_i8_full, k_scale, k_pool
        prep.nblk, prep.k_seq_major = cdiv(lk, self.blkk), True
        topk = min(prep.nblk, int(sla.topk * prep.nblk))
        _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
        kvw = project_moments(sla.proj_l.weight, kv, q.dtype)
        return attn_fwd(prep, v_full, q, lut, topk, kvw, ksum, sla.proj_l.bias.float().contiguous(), d ** -0.5, lk=lk,
                        blkq=self.blkq, blkk=self.blkk)


class SPAttention:
    """Drop-in for the block's attention callable: (q, k, v) local [1, rows, H, D] -> [1, rows, H, D].

    The block calls start_k(k) / start_kv(k, v) as soon as K and V exist: the exchanges are issued asynchronously (NCCL
    stream) and overlap with the V and Q projections, Q RMSNorm+RoPE and the Q-side quantisation that the block and __call__
    run before waiting on them.  With `prims.int8_k` the K exchange is: all-gather of the key-mean partials (tiny) -> global
    mean -> local smoothing / INT8 / pooling -> all-gather of INT8 K [rows, H, D], k_scale and k_pool; otherwise the 16-bit K
    slab is gathered and every rank prepares the whole key sequence.  `sage_arch` is the block family of `prims`; the scales
    and pooled means travel per BLKK-row key block."""

    def __init__(self, sp: "SequenceParallel", prims, sage_arch: str = "sm100"):
        self.sp, self.prims = sp, prims
        self.sage_arch = sage_arch
        self.blocks = sage_blocks(sage_arch)
        self._bufs = {}
        self._pending = None
        self._pending_k = None

    def _buf(self, name, shape, dtype, device, zero=False):
        key = (name, tuple(shape), dtype, device)
        if key not in self._bufs:
            self._bufs[key] = (torch.zeros if zero else torch.empty)(*shape, dtype=dtype, device=device)
        return self._bufs[key]

    def _gather_async(self, name: str, t: torch.Tensor, pad_rows: int, copy: bool = True):
        """t [rows, ...] -> ([world*pad_rows, ...] buffer, NCCL work handle); rows beyond t's stay zero (last rank).  With
        copy=False `t` already IS the first rows of the send buffer (see send_buffer)."""
        sp = self.sp
        send = self.send_buffer(name, t.shape[1:], pad_rows, t.dtype, t.device)
        if copy:
            send[: t.shape[0]].copy_(t)
        recv = self._buf(name + ".r", (sp.world * pad_rows, *t.shape[1:]), t.dtype, t.device)
        work = dist.all_gather_into_tensor(recv, send, group=sp.group, async_op=True)
        return recv, work

    def send_buffer(self, name, tail_shape, pad_rows, dtype, device):
        return self._buf(name + ".s", (pad_rows, *tail_shape), dtype, device, zero=True)

    def _cdt(self, t):
        return self.prims.sla.dtype if hasattr(self.prims, "sla") else t.dtype

    def _use_int8(self, k):
        return getattr(self.prims, "int8_k", False) and k.shape[-1] == 128

    def start_k(self, k):
        """K exists (projected, normalised, rotated): start its exchange; the V and Q projections run under it."""
        sp = self.sp
        k = k.to(self._cdt(k)).contiguous()
        if not self._use_int8(k):
            k_full, wk = self._gather_async("k", k[0], sp.rows_pad)
            self._pending_k = (k, ("bf16", k_full.unsqueeze(0)), [wk])
            return
        _, rows, h, d = k.shape
        w, cp, nbp = sp.world, sp.rows_pad // 128, sp.rows_pad // self.blocks[1]
        part = self.prims.k_partials(k)                                        # [1, H, ceil(rows/128), D]
        recv, wp = self._gather_async("kpart", part[0].transpose(0, 1), cp)     # rows = chunks: [w*cp, H, D]
        wp.wait()
        chunks = cdiv(sp.total_rows, 128)
        partials = recv[:chunks].transpose(0, 1).contiguous().unsqueeze(0)      # [1, H, chunks, D], global chunk order
        kmean = self.prims.k_mean(partials, sp.total_rows)
        send_k = self.send_buffer("k8", (h, d), sp.rows_pad, torch.int8, k.device)
        k_i8, k_scale, k_pool = self.prims.k_quant(k, kmean, send_k[:rows].unsqueeze(0))
        if k_i8.data_ptr() != send_k.data_ptr():                               # primitives that allocate their own output
            send_k[:rows].copy_(k_i8[0])
        k8_full, w1 = self._gather_async("k8", send_k[:rows], sp.rows_pad, copy=False)
        ks_full, w2 = self._gather_async("kscale", k_scale[0].transpose(0, 1), nbp)          # [w*nbp, H]
        kp_full, w3 = self._gather_async("kpool", k_pool[0].transpose(0, 1), nbp)            # [w*nbp, H, D]
        self._pending_k = (k, ("int8", k8_full.unsqueeze(0), ks_full, kp_full, kmean), [w1, w2, w3])

    def start_kv(self, k, v):
        sp = self.sp
        cdt = self._cdt(k)
        if self._pending_k is None:
            self.start_k(k)
        k, kx, works = self._pending_k
        self._pending_k = None
        v = v.to(cdt).contiguous()
        v_full, wv = self._gather_async("v", v[0], sp.rows_pad)
        kv, ksum = self.prims.moments(k, v)
        base = kv._base
        if base is not None and ksum._base is base and base.is_contiguous() and base.numel() == kv.numel() + ksum.numel():
            red = [dist.all_reduce(base, group=sp.group, async_op=True)]      # both accumulators live in one buffer: one collective
        else:
            red = [dist.all_reduce(kv, group=sp.group, async_op=True), dist.all_reduce(ksum, group=sp.group, async_op=True)]
        self._pending = (kx, v_full.unsqueeze(0), kv, ksum, works + [wv] + red)

    def __call__(self, q, k, v):
        require_served_arch(self.sage_arch)
        sp = self.sp
        dtype = q.dtype
        q = q.to(self._cdt(q)).contiguous()
        if self._pending is None:
            self.start_kv(k, v)
        kx, v_full, kv, ksum, works = self._pending
        self._pending = None
        qprep = self.prims.prepare_q(q) if hasattr(self.prims, "prepare_q") else None  # overlaps with the collectives
        for w in works:
            w.wait()
        if kx[0] == "bf16":
            out = self.prims.attention(q, kx[1], v_full, sp.total_rows, kv, ksum, qprep)
        else:
            _, k8_full, ks_full, kp_full, kmean = kx
            nblk = cdiv(sp.total_rows, self.blocks[1])
            k_scale = ks_full[:nblk].transpose(0, 1).contiguous().unsqueeze(0)             # [1, H, nblk]
            k_pool = kp_full[:nblk].transpose(0, 1).contiguous().unsqueeze(0)              # [1, H, nblk, D]
            out = self.prims.attention_i8(q, qprep, k8_full, k_scale, k_pool, kmean, v_full, sp.total_rows, kv, ksum)
        return out.to(dtype)


class UlyssesGpuPrims:
    """Per-rank attention for the head<->sequence mode: the single-GPU SLA pipeline on this rank's heads, split so that each
    stage starts as soon as the tensor it needs has arrived (K: key mean + INT8 + pooled means; Q: INT8 + pooled means +
    block map; V: linear moments + fused attention) on the blocks of `sage_arch`."""

    def __init__(self, sla_module, sage_arch: str = "sm100"):
        self.sla = sla_module
        self.sage_arch = sage_arch
        self.blkq, self.blkk = sage_blocks(sage_arch)

    def attend(self, get_q, get_k, get_v):
        from .SLA.core import attn_fwd, linear_moments, project_moments
        from .SLA.utils import QKPrep, block_map_from_pools, quant_k_into, quant_q_only
        sla = self.sla
        k = get_k()
        d = k.shape[-1]
        if d != 128:
            return sla(get_q(), k, get_v())
        kp = quant_k_into(QKPrep(), k, k.shape[1], self.blkk)
        q = get_q()
        prep = quant_q_only(q, self.blkq)
        for f in ("kmean", "k_i8", "k_scale", "k_pool", "nblk"):
            setattr(prep, f, getattr(kp, f))
        topk = min(prep.nblk, int(sla.topk * prep.nblk))
        _, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
        v = get_v()
        kv, ksum = linear_moments(k, v)
        kvw = project_moments(sla.proj_l.weight, kv, q.dtype)
        return attn_fwd(prep, v, q, lut, topk, kvw, ksum, sla.proj_l.bias.float().contiguous(), d ** -0.5,
                        blkq=self.blkq, blkk=self.blkk)


class UlyssesAttention:
    """Head <-> sequence exchange (a2a_cp.py:66-182 semantics).  `q_first` asks the block to project Q before K and V and to
    call start_q / start_k / start_kv as each tensor appears: the Q exchange then runs under the K and V projections, the K
    exchange under the V projection, and the V exchange under the K- and Q-side preparation inside `prims.attend`, which
    receives three callables that wait for and return the full-sequence [1, L, H/world, D] tensors.  The output goes back
    to its rows with a fourth all-to-all.  Uneven shards use all_to_all_single's split sizes: no padding rows move.
    `sage_arch` is the block family of `prims`; the exchange itself does not depend on it."""

    q_first = True

    def __init__(self, sp: "SequenceParallel", prims, compute_dtype=None, sage_arch: str = "sm100"):
        self.sp, self.prims, self.cdt = sp, prims, compute_dtype
        self.sage_arch = sage_arch
        self.blocks = sage_blocks(sage_arch)
        self.rows_of = [shard_rows(sp.total_rows, sp.world, r)[1] - shard_rows(sp.total_rows, sp.world, r)[0]
                        for r in range(sp.world)]
        self._bufs = {}
        self._pending = {}

    def _buf(self, name, shape, like):
        key = (name, tuple(shape), like.dtype, like.device)
        if key not in self._bufs:
            self._bufs[key] = torch.empty(*shape, dtype=like.dtype, device=like.device)
        return self._bufs[key]

    def _to_heads_async(self, name: str, t: torch.Tensor):
        """t [1, rows, H, D] -> ([L, H/world, D] buffer, work handle)."""
        sp, w = self.sp, self.sp.world
        t = (t if self.cdt is None else t.to(self.cdt)).contiguous()
        _, rows, h, d = t.shape
        if h % w:
            raise ValueError(f"Ulysses exchange needs heads % world == 0 (heads={h}, world={w})")
        hl = h // w
        send = self._buf(name + ".s", (w, rows, hl, d), t)
        send.copy_(t[0].view(rows, w, hl, d).permute(1, 0, 2, 3))          # chunk j = head group j of my rows
        recv = self._buf(name + ".r", (sp.total_rows, hl, d), t)
        work = dist.all_to_all_single(recv, send.view(w * rows, hl, d), output_split_sizes=self.rows_of,
                                      input_split_sizes=[rows] * w, group=sp.group, async_op=True)
        self._pending[name] = (recv, work)

    def start_q(self, q):
        self._to_heads_async("q", q)

    def start_k(self, k):
        self._to_heads_async("k", k)

    def start_kv(self, k, v):
        if "k" not in self._pending:
            self.start_k(k)
        self._to_heads_async("v", v)

    def _getter(self, name):
        def get():
            recv, work = self._pending.pop(name)
            work.wait()
            return recv.unsqueeze(0)
        return get

    def __call__(self, q, k, v):
        require_served_arch(self.sage_arch)
        sp, w = self.sp, self.sp.world
        dtype = q.dtype
        for name, t in (("q", q), ("k", k), ("v", v)):
            if name not in self._pending:
                self._to_heads_async(name, t)
        o = self.prims.attend(self._getter("q"), self._getter("k"), self._getter("v"))       # [1, L, hl, D]
        o = o[0].contiguous()
        rows, hl, d = sp.local_rows, o.shape[1], o.shape[2]
        recv = self._buf("o.r", (w, rows, hl, d), o)
        dist.all_to_all_single(recv.view(w * rows, hl, d), o, output_split_sizes=[rows] * w,
                               input_split_sizes=self.rows_of, group=sp.group)
        return recv.permute(1, 0, 2, 3).reshape(1, rows, w * hl, d).to(dtype)            # chunk i = head group i of my rows


def split_heads(heads: int, world: int):
    """Contiguous head ranges per rank, the first heads % world ranks get one more: returns (counts, offsets)."""
    counts = [heads // world + (1 if r < heads % world else 0) for r in range(world)]
    offsets = [sum(counts[:r]) for r in range(world)]
    return counts, offsets


class UnevenUlyssesAttention(UlyssesAttention):
    """The same exchange when heads % world != 0 (e.g. the 12 heads of Wan-1.3B on 8 GPUs -> 2,2,2,2,1,1,1,1): rank r takes
    the contiguous head range split_heads() assigns it; every all-to-all uses per-peer split sizes in units of one
    [D]-row (rows * heads_of_peer).  The slab <-> per-peer-chunk reordering is ONE gather kernel each way (a precomputed row
    permutation), not one copy per peer."""

    def __init__(self, sp: "SequenceParallel", prims, heads: int, compute_dtype=None, sage_arch: str = "sm100"):
        super().__init__(sp, prims, compute_dtype, sage_arch)
        if heads < sp.world:
            raise ValueError(f"Ulysses exchange needs at least one head per rank (heads={heads}, world={sp.world})")
        self.heads = heads
        self.heads_of, self.head_off = split_heads(heads, sp.world)
        self._perm = {}

    def _perms(self, device):
        """send position p (chunk j = rank j's heads of my rows, laid out [rows, heads_of[j]]) <-> slab row r*H + head."""
        if device not in self._perm:
            rows, h = self.sp.local_rows, self.heads
            r = torch.arange(rows).view(rows, 1)
            perm = torch.cat([(r * h + torch.arange(self.head_off[j], self.head_off[j] + self.heads_of[j]).view(1, -1)).reshape(-1)
                              for j in range(self.sp.world)])
            self._perm[device] = (perm.to(device), torch.argsort(perm).to(device))
        return self._perm[device]

    def _to_heads_async(self, name: str, t: torch.Tensor):
        """t [1, rows, H, D] -> ([L, heads_of[rank], D] buffer, work handle)."""
        sp = self.sp
        t = (t if self.cdt is None else t.to(self.cdt)).contiguous()
        _, rows, h, d = t.shape
        if h != self.heads:
            raise ValueError(f"expected {self.heads} heads, got {h}")
        send = self._buf(name + ".s", (rows * h, d), t)
        torch.index_select(t.view(rows * h, d), 0, self._perms(t.device)[0], out=send)
        mine = self.heads_of[sp.rank]
        recv = self._buf(name + ".r", (sp.total_rows * mine, d), t)
        work = dist.all_to_all_single(recv, send, output_split_sizes=[r * mine for r in self.rows_of],
                                      input_split_sizes=[rows * c for c in self.heads_of], group=sp.group, async_op=True)
        self._pending[name] = (recv.view(sp.total_rows, mine, d), work)

    def __call__(self, q, k, v):
        require_served_arch(self.sage_arch)
        sp = self.sp
        dtype = q.dtype
        for name, t in (("q", q), ("k", k), ("v", v)):
            if name not in self._pending:
                self._to_heads_async(name, t)
        o = self.prims.attend(self._getter("q"), self._getter("k"), self._getter("v"))       # [1, L, mine, D]
        o = o[0].contiguous()
        rows, mine, d = sp.local_rows, o.shape[1], o.shape[2]
        recv = self._buf("o.r", (rows * self.heads, d), o)
        dist.all_to_all_single(recv, o.view(sp.total_rows * mine, d), output_split_sizes=[rows * c for c in self.heads_of],
                               input_split_sizes=[r * mine for r in self.rows_of], group=sp.group)
        out = torch.index_select(recv, 0, self._perms(o.device)[1])      # chunk order -> [rows, H] order
        return out.view(1, rows, self.heads, d).to(dtype)


class SequenceParallel:
    def __init__(self, total_rows: int, world: Optional[int] = None, rank: Optional[int] = None, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if world is None else world
        self.rank = dist.get_rank(group) if rank is None else rank
        self.total_rows = total_rows
        self.row_begin, self.row_end, self.rows_pad = shard_rows(total_rows, self.world, self.rank)
        self.local_rows = self.row_end - self.row_begin
        if self.local_rows <= 0:
            raise ValueError(f"rank {self.rank} owns no rows: L={total_rows} is too short for {self.world} ranks of 128-row blocks")

    def pick_mode(self, heads: int, mode: str = "auto") -> str:
        if mode not in ("auto", "allgather", "ulysses"):
            raise ValueError(f"unknown sequence-parallel mode {mode!r}")
        if mode == "auto":
            # at N=2 the all-gather's exchanges hide under the V / Q projections, while the all-to-all has the output exchange
            # and the slab permutes on the critical path; from N=4 up the all-to-all moves N/2 times fewer bytes and has no
            # per-rank work that grows with the full sequence (12 heads at N=8 -> uneven split 2,2,2,2,1,1,1,1).  Not measured
            # on H100.
            return "ulysses" if self.world >= 4 and heads >= self.world else "allgather"
        if mode == "ulysses" and heads < self.world:
            raise ValueError(f"mode 'ulysses' needs at least one head per rank (heads={heads}, world={self.world})")
        return mode

    def install(self, model, mode: str = "auto", sage_arch: str = "sm100") -> str:
        """Replace every block's attention callable by the sequence-parallel one (the reference seam is
        `WanSelfAttention.attn_op.local_attn`, inference/modify_model.py:48-52).  Returns the mode used:
        "allgather" (K/V all-gather + moment all-reduce, any head count) or "ulysses" (head<->sequence all-to-all; with
        heads % world != 0 the uneven-split variant).  `sage_arch` is the SageSLA block family the hooks run, "sm100"
        (BLKQ=128, BLKK=64) or "sm90" (BLKQ=64, BLKK=128); it must be the served arch (SLA.utils.set_served_arch), which
        the single-GPU module follows."""
        sage_blocks(sage_arch)
        require_served_arch(sage_arch)
        used = None
        for blk in model.blocks:
            used = self.pick_mode(blk.heads, mode)
            prims = UlyssesGpuPrims(blk.sla, sage_arch) if used == "ulysses" else GpuPrimitives(blk.sla, sage_arch)
            if used == "ulysses" and blk.heads % self.world:
                blk.attn_hook = UnevenUlyssesAttention(self, prims, blk.heads, compute_dtype=blk.sla.dtype, sage_arch=sage_arch)
            elif used == "ulysses":
                blk.attn_hook = UlyssesAttention(self, prims, compute_dtype=blk.sla.dtype, sage_arch=sage_arch)
            else:
                blk.attn_hook = SPAttention(self, prims, sage_arch)
        self.mode = used
        return used

    def scatter(self, full: torch.Tensor) -> torch.Tensor:
        return full[self.row_begin:self.row_end].contiguous()

    def gather_rows(self, local: torch.Tensor) -> torch.Tensor:
        """All-gather of the step output rows (context_parallel.py:60-91 equivalent); local [rows, C] -> [L, C]."""
        send = torch.zeros(self.rows_pad, *local.shape[1:], dtype=local.dtype, device=local.device)
        send[: local.shape[0]].copy_(local)
        recv = torch.empty(self.world * self.rows_pad, *local.shape[1:], dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(recv, send, group=self.group)
        return recv[: self.total_rows]
