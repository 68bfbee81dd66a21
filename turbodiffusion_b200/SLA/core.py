"""Mirror of turbodiffusion/SLA/core.py: SparseLinearAttention / SageSparseLinearAttention on H100.

Same constructor arguments, parameters (`proj_l`, fp32, zero-init) and call convention (q,k,v in [B, L, H, D], result in
the same layout and dtype; SLA/core.py:181-183,253).  The forward is five kernel launches:
  quant_qk (key mean, pooled means, INT8 Q / smoothed K)  ->  block_map (pooled score, top-k, LUT)
  -> linear_moments (phi(K)^T V, sum phi(K))  ->  [tiny cuBLAS bmm: proj_l folded into the moment matrix]
  -> attn_fwd (sparse INT8 QK^T, softmax, PV, linear branch, merge).
Inputs are consumed in place in their [B, L, H, D] layout; no transposed copies of q/k/v are made.
"""
from __future__ import annotations


import torch
import torch.autograd.forward_ad as fwAD
import torch.nn as nn
import torch.nn.functional as F

from .. import _ops
from . import utils as _utils
from .._lib import DTYPE_TAG, check, has_tangent, lib, plain, ptr, require_cuda, stream_ptr
from .utils import (SAGE_BLOCKS, QKPrep, block_map_from_pools, get_block_map, get_cuda_arch, quant_k_into,  # noqa: F401
                    quant_q_only, quant_qk)

SAGESLA_ENABLED = True   # the INT8 path is built in (no SpargeAttn dependency)
SAGE2PP_ENABLED = True


FEATURE_TAG = {"softmax": 0, "elu": 1, "relu": 2}   # SLA/core.py:57-73


def linear_moments(k: torch.Tensor, v: torch.Tensor, feature: int = 0):
    """kv [B,H,D(v),D(k)] fp32, ksum [B,H,D] fp32 of the local keys (accumulated: add shards / all-reduce).  D in {64, 128};
    `feature`: 0 softmax over D, 1 elu+1, 2 relu."""
    b, l, h, d = k.shape
    buf = _ops.sla_linear_moments(k, v, feature)        # both accumulators in one buffer: one fill
    return buf[: b * h * d * d].view(b, h, d, d), buf[b * h * d * d:].view(b, h, d)


def linear_moments_vl(k: torch.Tensor, v: torch.Tensor, seq_lens: torch.Tensor, feature: int = 0):
    """linear_moments per entry of a padded batch (tdb200_sla_linear_moments_vl): entry i's kv [H,D,D] and ksum [H,D] over its
    first seq_lens[i] rows, the bits of linear_moments on entry i alone cut to those rows.  D = 128."""
    b, l, h, d = k.shape
    buf = torch.zeros(b * h * d * (d + 1), dtype=torch.float32, device=k.device)
    check(lib().tdb200_sla_linear_moments_vl(ptr(k), ptr(v), DTYPE_TAG[k.dtype], b, l, h, d, ptr(seq_lens), feature, ptr(buf),
                                             ptr(buf) + 4 * b * h * d * d, stream_ptr(k.device)), "sla_linear_moments_vl")
    return buf[: b * h * d * d].view(b, h, d, d), buf[b * h * d * d:].view(b, h, d)


def project_moments(proj_w: torch.Tensor, kv: torch.Tensor, dtype) -> torch.Tensor:
    """kvw [B,H,D_out,D_k] = T(proj_w . kv): proj_l's weight folded into the moment matrix (the fused kernel's last MMA)."""
    b, h, d, _ = kv.shape
    w = proj_w if (proj_w.dtype == torch.float32 and proj_w.is_contiguous()) else proj_w.float().contiguous()
    assert kv.dtype == torch.float32 and kv.is_contiguous() and w.shape == (d, d)
    return _ops.sla_project_moments(w, kv, dtype)


ATTN_TIMER = None  # bench.py installs a callable(h, mblk, topk, d) -> context manager to time the fused-attention launches


def attn_fwd(prep, v, q, lut, topk, kvw, ksum, proj_b, sm_scale, lk=None, feature=0, blkq=128, blkk=64, fp8_v=False):
    """(blkq, blkk): the block sizes `prep` and `lut` were built with, (128, 64) or (64, 128).  fp8_v: P.V on e4m3 P and V
    (tdb200_sla_quant_v_fp8 of the first lk rows of v, then tdb200_sla_attn_fwd_fp8v; d = 128)."""
    if ATTN_TIMER is not None:
        # bench.py counts H*Mblk*topk*4*128*64*D FLOPs: exact for both families, BLKQ*BLKK = 8192 in each
        with ATTN_TIMER(q.shape[2] * q.shape[0], (q.shape[1] + blkq - 1) // blkq, topk, q.shape[3]):
            return _attn_fwd(prep, v, q, lut, topk, kvw, ksum, proj_b, sm_scale, lk, feature, blkq, blkk, fp8_v)
    return _attn_fwd(prep, v, q, lut, topk, kvw, ksum, proj_b, sm_scale, lk, feature, blkq, blkk, fp8_v)


def _attn_fwd(prep, v, q, lut, topk, kvw, ksum, proj_b, sm_scale, lk=None, feature=0, blkq=128, blkk=64, fp8_v=False):
    d = q.shape[3]
    lk = v.shape[1] if lk is None else lk
    k_seq_major = bool(getattr(prep, "k_seq_major", False))   # INT8 K in the gathered [B, Lk, H, D] layout (dist.py)
    if k_seq_major and (d != 128 or feature != 0):
        raise NotImplementedError("sequence-major INT8 K is served by the 128-wide softmax kernels only")
    if fp8_v:
        if d != 128:
            raise NotImplementedError(f"FP8 P.V (SLA.utils.set_sage_pv('fp8')): head dim {d}; it is served for d = 128")
        assert v.is_contiguous() and (v.shape[0] == 1 or v.shape[1] == lk)
        v_fp8, v_scale = _ops.sla_quant_v_fp8(v, lk, blkk)
        return _ops.sla_attn_fwd_fp8v(prep.q_i8, prep.q_scale, prep.k_i8, prep.k_scale, v_fp8, v_scale, q, lut, topk, kvw, ksum,
                                      proj_b, float(sm_scale), lk, feature, blkq, blkk, k_seq_major)
    return _ops.sla_attn_fwd(prep.q_i8, prep.q_scale, prep.k_i8, prep.k_scale, v, q, lut, topk, kvw, ksum, proj_b,
                             float(sm_scale), lk, feature, blkq, blkk, k_seq_major)


# The 16-bit attention serves 64-row key blocks (_ops.BLKK16) with 128- or 64-row query blocks; `blkq` below is the query
# block size `lut` was built with.


def attn_fwd_qk16(q, k, v, lut, topk, kvw, ksum, proj_b, sm_scale, lk=None, feature=0, blkq=128):
    """The non-quantised sparse attention (a9', SLA/kernel.py:33-82): 16-bit Q.K^T on the tensor cores, fp32 scores, and the
    linear branch with feature map `feature`."""
    lk = v.shape[1] if lk is None else lk
    return _ops.sla_attn16_fwd(q, k, v, lut, topk, kvw, ksum, proj_b, float(sm_scale), lk, feature, blkq)


def attn_fwd_qk16_lse(q, k, v, lut, topk, sm_scale, blkq=128):
    """Sparse branch of attn_fwd_qk16 alone, for the training path: (o_s [B,L,H,D] in q.dtype, lse [B,H,L] fp32), lse being
    the row log-sum-exp of the scores in log2 units (scores scaled by sm_scale * log2(e)).  `lut` [B,H,Mblk,topk] int32.
    Differentiable in q, k and v through o_s (the backward is attn_bwd_qk16)."""
    return _ops.sla_attn16_fwd_lse(q, k, v, lut, topk, float(sm_scale), blkq)


def attn_bwd_qk16(q, k, v, o_s, d_o, lse, lut, topk, sm_scale, blkq=128):
    """(dq, dk, dv) of attn_fwd_qk16_lse's o_s for the incoming gradient d_o; all [B,L,H,D] contiguous in q.dtype."""
    return _ops.sla_attn16_bwd(q, k, v, o_s, d_o, lse, lut, topk, float(sm_scale), blkq)


def sparse_attention16(q, k, v, lut, topk, sm_scale, blkq=128):
    """o_s = block-sparse softmax attention of q, k, v ([B,L,H,D], 16-bit, d = 128) over `lut`'s key blocks (`blkq`-row query
    blocks, 64-row key blocks), differentiable in q, k and v (the reference's `_attention`, SLA/kernel.py:240-319)."""
    return attn_fwd_qk16_lse(q, k, v, lut, topk, sm_scale, blkq)[0]


def _jvp_call(q, k, v, q_t, k_t, v_t, lut, topk, sm_scale, blkq, with_lse):
    b, l, h, d = q.shape
    o_s, o_s_t = torch.empty_like(q), torch.empty_like(q)
    if not with_lse:
        check(lib().tdb200_sla_attn16_jvp(ptr(q), ptr(k), ptr(v), ptr(q_t), ptr(k_t), ptr(v_t), DTYPE_TAG[q.dtype], ptr(lut), topk,
                                          ptr(o_s), ptr(o_s_t), b, l, h, d, sm_scale, blkq, _ops.BLKK16, stream_ptr(q.device)),
              "sla_attn16_jvp")
        return o_s, o_s_t, None
    lse = torch.empty(b, h, l, dtype=torch.float32, device=q.device)
    check(lib().tdb200_sla_attn16_jvp_lse(ptr(q), ptr(k), ptr(v), ptr(q_t), ptr(k_t), ptr(v_t), DTYPE_TAG[q.dtype], ptr(lut), topk,
                                          ptr(o_s), ptr(o_s_t), ptr(lse), b, l, h, d, sm_scale, blkq, _ops.BLKK16,
                                          stream_ptr(q.device)),
          "sla_attn16_jvp_lse")
    return o_s, o_s_t, lse


def attn_jvp_qk16(q, k, v, q_t, k_t, v_t, lut, topk, sm_scale, blkq=128):
    """(o_s, o_s_t): attn_fwd_qk16_lse's o_s and its forward-mode derivative along the tangents (q_t, k_t, v_t), the softmax
    restricted to `lut`'s key blocks held fixed (tdb200_sla_attn16_jvp, one kernel).  All [B,L,H,D] contiguous in q.dtype,
    d = 128, (blkq, blkk) = (128, 64).  Eager: not a `tdb200::` operator, no autograd."""
    return _jvp_call(q, k, v, q_t, k_t, v_t, lut, topk, float(sm_scale), blkq, False)[:2]


class _SparseAttention16Jvp(torch.autograd.Function):
    """sparse_attention16_jvp's training path: o_s differentiable in q, k and v through the SLA backward (attn_bwd_qk16, fed
    the lse of tdb200_sla_attn16_jvp_lse); o_s_t, and the tangents, carry no gradient."""

    @staticmethod
    def forward(ctx, q, k, v, q_t, k_t, v_t, lut, topk, sm_scale, blkq):
        o_s, o_s_t, lse = _jvp_call(q, k, v, q_t, k_t, v_t, lut, topk, sm_scale, blkq, True)
        ctx.mark_non_differentiable(o_s_t)
        ctx.set_materialize_grads(False)    # o_s_t's gradient is never used: no zero tensor for it
        ctx.save_for_backward(q, k, v, o_s, lse, lut)
        ctx.topk, ctx.sm_scale, ctx.blkq = topk, sm_scale, blkq
        return o_s, o_s_t

    @staticmethod
    def backward(ctx, d_o, d_o_t):
        if d_o is None:
            return (None,) * 10
        q, k, v, o_s, lse, lut = ctx.saved_tensors
        dq, dk, dv = attn_bwd_qk16(q, k, v, o_s, d_o.to(q.dtype).contiguous(), lse, lut, ctx.topk, ctx.sm_scale, ctx.blkq)
        return dq, dk, dv, None, None, None, None, None, None, None


def sparse_attention16_jvp(q, k, v, q_t, k_t, v_t, lut, topk, sm_scale, blkq=128):
    """(o_s, o_s_t): sparse_attention16's o_s and its tangent along (q_t, k_t, v_t) with the block selection `lut` held fixed
    (it is piecewise constant in q, k).  q, k, v and the tangents [B,L,H,D] contiguous 16-bit of one dtype, d = 128, blkq = 128.
    With grad enabled and any of q, k, v requiring grad, o_s is differentiable in q, k and v (the same bits, plus the row lse the
    SLA backward reads); o_s_t never carries a gradient (a stop-gradient target) and the tangents get none."""
    sm_scale = float(sm_scale)
    q_t, k_t, v_t = q_t.detach(), k_t.detach(), v_t.detach()
    if torch.is_grad_enabled() and any(t.requires_grad for t in (q, k, v)):
        return _SparseAttention16Jvp.apply(q, k, v, q_t, k_t, v_t, lut, topk, sm_scale, blkq)
    return attn_jvp_qk16(q, k, v, q_t, k_t, v_t, lut, topk, sm_scale, blkq)


class _SparseAttention16AD(torch.autograd.Function):
    """SparseLinearAttention.forward's sparse branch for q, k, v of which one carries a forward-mode tangent: the block
    selection from the primal q, k ((BLKQ, BLKK) = (128, 64), `topk` blocks per row; `module`'s _keep_selection, if set,
    receives it: passed as the module, since torch.func rebuilds a dict argument), then
    attn_fwd_qk16_lse once; jvp = tdb200_sla_attn16_tangent from the saved o_s and lse with the selection held fixed (missing
    tangents are zeros); backward = attn_bwd_qk16.  lse and lut are outputs only so that setup_context can save them.  The
    tangent carries no gradient."""

    @staticmethod
    def forward(q, k, v, topk, sm_scale, module):
        prep = select_prep(q, k, 128, _ops.BLKK16)
        sparse_map, lut = block_map_from_pools(prep.q_pool, prep.k_pool, topk)
        keep = getattr(module, "_keep_selection", None)
        if keep is not None:
            keep.update(lut=lut, sparse_map=sparse_map, topk=topk)
        o_s, lse = attn_fwd_qk16_lse(q, k, v, lut, topk, sm_scale, 128)
        return o_s, lse, lut

    @staticmethod
    def setup_context(ctx, inputs, output):
        q, k, v, topk, sm_scale, _ = inputs
        o_s, lse, lut = output
        ctx.mark_non_differentiable(lse, lut)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(q, k, v, o_s, lse, lut)
        ctx.save_for_forward(q, k, v, o_s, lse, lut)
        ctx.topk, ctx.sm_scale = topk, sm_scale

    @staticmethod
    def jvp(ctx, q_t, k_t, v_t, *_):
        with torch._C._DisableFuncTorch():
            q, k, v, o_s, lse, lut = (plain(t) for t in ctx.saved_tensors)
            q_t, k_t, v_t = (torch.zeros_like(p) if t is None else plain(t).detach().to(p.dtype).contiguous()
                             for t, p in ((q_t, q), (k_t, k), (v_t, v)))
            b, l, h, d = q.shape
            o_s_t = torch.empty_like(q)
            check(lib().tdb200_sla_attn16_tangent(ptr(q), ptr(k), ptr(v), ptr(q_t), ptr(k_t), ptr(v_t), ptr(o_s), ptr(lse),
                                                  DTYPE_TAG[q.dtype], ptr(lut), ctx.topk, ptr(o_s_t), b, l, h, d, ctx.sm_scale, 128,
                                                  _ops.BLKK16, stream_ptr(q.device)),
                  "sla_attn16_tangent")
        return o_s_t, None, None

    @staticmethod
    def backward(ctx, d_o, d_lse, d_lut):
        if d_o is None:
            return (None,) * 6
        q, k, v, o_s, lse, lut = ctx.saved_tensors
        dq, dk, dv = attn_bwd_qk16(q, k, v, o_s, d_o.to(q.dtype).contiguous(), lse, lut, ctx.topk, ctx.sm_scale, 128)
        return dq, dk, dv, None, None, None


def _linear_args(q, k, v, proj_w, proj_b, feature, what):
    feature = FEATURE_TAG[feature] if isinstance(feature, str) else int(feature)
    if q.shape[-1] != 128:
        raise NotImplementedError(f"{what}: head dim {q.shape[-1]}; the linear-branch kernels serve d = 128")
    if not (q.dtype == k.dtype == v.dtype and q.dtype in (torch.bfloat16, torch.float16)):
        raise ValueError(f"{what}: q, k, v must share one 16-bit dtype, got {q.dtype}, {k.dtype}, {v.dtype}")
    if not (q.shape == k.shape == v.shape):
        raise ValueError(f"{what}: q, k, v shapes differ: {tuple(q.shape)}, {tuple(k.shape)}, {tuple(v.shape)}")
    if has_tangent(proj_w, proj_b):
        raise NotImplementedError(f"{what}: proj_w / proj_b carry a forward-mode tangent; the tangent kernels hold them "
                                  "fixed (SparseLinearAttention takes its torch branch for such calls)")
    require_cuda(q, k, v, proj_w, proj_b)
    return feature, proj_w.float().contiguous(), proj_b.float().contiguous()


def _linear_tangent(q, k, v, q_t, k_t, v_t, mom, w, feature):
    q_t, k_t, v_t = (torch.zeros_like(p) if t is None else t.detach().to(p.dtype).contiguous()
                     for t, p in ((q_t, q), (k_t, k), (v_t, v)))
    return _ops.sla_linear_tangent(q, k, v, q_t, k_t, v_t, mom, w, feature)


class _LinearBranchAD(torch.autograd.Function):
    """linear_branch for q, k, v of which one carries a forward-mode tangent: the forward operator once (its bits), jvp =
    tdb200_sla_linear_tangent from the saved moments (missing tangents are zeros), backward = tdb200_sla_linear_bwd."""

    @staticmethod
    def forward(q, k, v, w, b, feature):
        return _ops.sla_linear_fwd(q, k, v, w, b, feature)

    @staticmethod
    def setup_context(ctx, inputs, output):
        q, k, v, w, b, feature = inputs
        ctx.mark_non_differentiable(output[1])
        ctx.save_for_backward(q, k, v, w, output[1])
        ctx.save_for_forward(q, k, v, w, output[1])
        ctx.feature = feature

    @staticmethod
    def jvp(ctx, q_t, k_t, v_t, *_):
        with torch._C._DisableFuncTorch():
            q, k, v, w, mom = (plain(t) for t in ctx.saved_tensors)
            o_t = _linear_tangent(q, k, v, plain(q_t), plain(k_t), plain(v_t), mom, w, ctx.feature)
        return o_t, None

    @staticmethod
    def backward(ctx, d_o, d_mom):
        q, k, v, w, mom = ctx.saved_tensors
        dq, dk, dv, dw, db = _ops.sla_linear_bwd(q, k, v, d_o.to(q.dtype).contiguous(), mom, w, ctx.feature)
        return dq, dk, dv, dw, db, None


def linear_branch(q, k, v, proj_w, proj_b, feature="softmax"):
    """SparseLinearAttention's linear branch and proj_l as CUDA kernels: o_l [B, L, H, D] in q.dtype,
    o_l,i = T(u_i proj_w^T + proj_b) with u_i = phi(q_i) M / (1e-5 + phi(q_i).s), M = sum_j phi(k_j)^T v_j, s = sum_j phi(k_j).
    q, k, v [B, L, H, 128] of one 16-bit dtype; proj_w [128, 128], proj_b [128] (fp32: proj_l's parameters); `feature` is
    "softmax", "elu" or "relu" (or its tag 0, 1, 2).  Differentiable in all five inputs (tdb200_sla_linear_bwd; the gradients
    of proj_w and proj_b are fp32 sums over batch, heads and rows, in a fixed order).  When q, k or v carries a forward-mode
    tangent (torch.func.jvp, forward_ad) the output carries its tangent from tdb200_sla_linear_tangent; proj_w and proj_b
    must carry none (NotImplementedError).  Rounding points: include/tdb200.h."""
    feature, w, b = _linear_args(q, k, v, proj_w, proj_b, feature, "linear_branch")
    if has_tangent(q, k, v):
        return _LinearBranchAD.apply(q.contiguous(), k.contiguous(), v.contiguous(), w, b, feature)[0]
    q, k, v = (t.contiguous() for t in (q, k, v))
    return _ops.sla_linear_fwd(q, k, v, w, b, feature)[0]


def linear_branch_jvp(q, k, v, q_t, k_t, v_t, proj_w, proj_b, feature="softmax"):
    """(o_l, o_l_t): linear_branch and its forward-mode derivative along (q_t, k_t, v_t), proj_w and proj_b held fixed.
    o_l is differentiable as linear_branch's is (the same forward kernel, so the same bits with and without grad); o_l_t
    carries no gradient and the tangents get none."""
    feature, w, b = _linear_args(q, k, v, proj_w, proj_b, feature, "linear_branch_jvp")
    q, k, v = (t.contiguous() for t in (q, k, v))
    o_l, mom = _ops.sla_linear_fwd(q, k, v, w, b, feature)
    with torch.no_grad():
        o_t = _linear_tangent(q, k, v, q_t, k_t, v_t, mom.detach(), w.detach(), feature)
    return o_l, o_t


def select_prep(q, k, blkq, blkk):
    """The pooled means (and Sage INT8 codes) block selection reads, for q, k [B, L, H, D]: quant_qk for the SageSLA families;
    (64, 64), a pair tdb200_sla_quant_qk does not take, from its query half at blkq = 64 and its key half at blkk = 64."""
    if (blkq, blkk) == (64, 64):
        return quant_k_into(quant_q_only(q, blkq), k, k.shape[1], blkk)
    return quant_qk(q, k, blkq=blkq, blkk=blkk)


class _SLABase(nn.Module):
    quantised_qk = True   # SageSparseLinearAttention: INT8 Q.K^T; SparseLinearAttention: 16-bit Q.K^T (128-wide heads)

    def block_sizes(self, device_index):
        """(BLKQ, BLKK) of this call."""
        return 128, 64

    def __init__(self, head_dim, topk, feature_map="softmax", use_bf16=True, tie_feature_map_qk=True):
        super().__init__()
        self.dtype = torch.bfloat16 if use_bf16 else torch.float16
        self.topk = topk
        self.proj_l = nn.Linear(head_dim, head_dim, dtype=torch.float32)
        if feature_map == "elu":            # SLA/core.py:57-61
            self.feature_map_q = self.feature_map_k = lambda x: F.elu(x) + 1
        elif feature_map == "relu":         # :62-64
            self.feature_map_q = self.feature_map_k = nn.ReLU()
        elif feature_map == "softmax":      # :65-69
            self.feature_map_q = self.feature_map_k = lambda x: F.softmax(x, dim=-1)
        else:
            raise NotImplementedError(f"Not supported feature map {feature_map}.")
        self.feature = FEATURE_TAG[feature_map]   # evaluated inside the fused kernels (moments + attention epilogue)
        self.init_weights_()

    def init_weights_(self):
        with torch.no_grad():
            nn.init.zeros_(self.proj_l.weight)
            nn.init.zeros_(self.proj_l.bias)

    def forward(self, q, k, v, return_sparsity=False, seq_lens=None):
        """q,k,v [B, L, H, D] (any float dtype), D in {64, 128} (SLA/core.py:207) -> [B, L, H, D] in q.dtype.
        SparseLinearAttention with grad enabled and any of q, k, v requiring grad takes the differentiable training path
        (_forward_train); every other call runs the fused forward-only kernels.  When any of q, k, v carries a forward-mode
        tangent (torch.func.jvp, torch.autograd.forward_ad), the call takes _forward_ad, whose output carries the tangent.

        seq_lens: per-entry lengths of a padded batch (clips of different token counts packed to one L), an integer tensor [B]
        or a boolean prefix mask [B, L], as dense_attention's q_lens (ops.core._lengths: CPU lengths are checked, GPU lengths
        clamped to [0, L] on the device, without a synchronisation).  Entry i's rows below n_i = seq_lens[i] are bit-identical
        to this module on entry i alone with q, k and v cut to n_i rows: its own key mean, block selection (topk_i = max(1,
        min(nblk_i, int(topk * nblk_i))) of its own nblk_i key blocks), moments and key mask.  Rows past n_i are 0, and what q, k
        and v hold there, NaN and inf included, reaches no output.  return_sparsity then gives a float64 [B] tensor of
        topk_i / nblk_i (0 for an empty entry).  The _keep_selection record (forward_with_lut) keeps "topk" an int, the LUT's
        row stride, and adds "topks", the int32 [B] topk_i on the device; LUT entries past topk_i are -1.  Inference only, eager only (the _vl entry points are called through ctypes,
        not `tdb200::` operators), d = 128, 16-bit P.V: grad-requiring inputs, forward-mode tangents, head dim 64 and
        set_sage_pv("fp8") raise NotImplementedError before any CUDA work."""
        if seq_lens is not None:
            return self._forward_vl(q, k, v, return_sparsity, seq_lens)
        if has_tangent(q, k, v):
            return self._forward_ad(q, k, v, return_sparsity)
        if not self.quantised_qk and torch.is_grad_enabled() and any(t.requires_grad for t in (q, k, v)):
            return self._forward_train(q, k, v, return_sparsity)
        fp8_v = self.quantised_qk and _utils.SAGE_PV == "fp8"   # SageSparseLinearAttention under SLA.utils.set_sage_pv("fp8")
        if fp8_v and q.shape[-1] != 128:
            raise NotImplementedError(f"SageSparseLinearAttention with FP8 P.V (SLA.utils.set_sage_pv('fp8')): head dim "
                                      f"{q.shape[-1]}; FP8 P.V is served for d = 128")
        require_cuda(q, k, v)
        dtype = q.dtype
        q, k, v = (t if (t.dtype == self.dtype and t.is_contiguous()) else t.to(self.dtype).contiguous() for t in (q, k, v))
        b, l, h, d = q.shape
        if d not in (64, 128):
            raise AssertionError("headdim should be in [64, 128].")  # SLA/core.py:207
        blkq, blkk = self.block_sizes(q.device.index)
        prep = select_prep(q, k, blkq, blkk)
        nblk = prep.nblk
        real_topk = min(nblk, int(self.topk * nblk))
        if real_topk < 1:
            # the reference would select zero key blocks here (an empty softmax); short sequences get one block instead
            real_topk = 1
        sparse_map, lut = block_map_from_pools(prep.q_pool, prep.k_pool, real_topk)
        if getattr(self, "_keep_selection", None) is not None:
            self._keep_selection.update(lut=lut, sparse_map=sparse_map, topk=real_topk)
        kv, ksum = linear_moments(k, v, self.feature)
        # proj_l folded into the moments: (phi(q) KV / den) W^T + b == phi(q) (W KV^T)^T / den + b ; kv is [dv, dk]
        # forward-only kernels: proj_l enters as data (detached), so the output carries no autograd history
        kvw = project_moments(self.proj_l.weight.detach(), kv, self.dtype)  # [B,H,d_out,d_k]
        proj_b = self.proj_l.bias.detach().float().contiguous()
        if not self.quantised_qk and d == 128 and (self.feature == 0 or blkq == 64):
            o = attn_fwd_qk16(q, k, v, lut, real_topk, kvw, ksum, proj_b, d ** -0.5, feature=self.feature, blkq=blkq)
        else:
            o = attn_fwd(prep, v, q, lut, real_topk, kvw, ksum, proj_b, d ** -0.5, feature=self.feature, blkq=blkq, blkk=blkk,
                         fp8_v=fp8_v)
        o = o if o.dtype == dtype else o.to(dtype)
        return (o, real_topk / nblk) if return_sparsity else o

    def _forward_vl(self, q, k, v, return_sparsity, seq_lens):
        """forward() with per-entry lengths: tdb200_sla_quant_qk_vl, _block_map_vl, _linear_moments_vl, then
        tdb200_sla_attn16_fwd_vl or tdb200_sla_attn_fwd_vl, in the branch forward() takes without lengths."""
        what = f"{type(self).__name__}.forward with seq_lens"
        if has_tangent(q, k, v):
            raise NotImplementedError(f"{what}: inputs carry a forward-mode tangent; per-entry lengths serve inference only")
        if torch.is_grad_enabled() and any(t.requires_grad for t in (q, k, v)):
            raise NotImplementedError(f"{what}: inputs require grad; per-entry lengths serve inference only (use torch.no_grad())")
        if q.shape[-1] != 128:
            raise NotImplementedError(f"{what}: head dim {q.shape[-1]}; per-entry lengths serve d = 128")
        if self.quantised_qk and _utils.SAGE_PV == "fp8":
            raise NotImplementedError(f"{what}: FP8 P.V (SLA.utils.set_sage_pv('fp8')); per-entry lengths serve 16-bit P.V")
        if not (q.dim() == 4 and q.shape == k.shape == v.shape):
            raise ValueError(f"{what}: q, k, v [B, L, H, D] of one shape, got {tuple(q.shape)}, {tuple(k.shape)}, {tuple(v.shape)}")
        require_cuda(q, k, v)
        from ..ops.core import _lengths
        dtype = q.dtype
        q, k, v = (t if (t.dtype == self.dtype and t.is_contiguous()) else t.to(self.dtype).contiguous() for t in (q, k, v))
        b, l, h, d = q.shape
        # clamped here too (int32 device lengths reach the kernels unclamped): topk_i and the sparsity then count the n_i the
        # kernels use, on the device, without a synchronisation
        lens = _lengths(what, seq_lens, b, l, q.device, "seq_lens", "sequence", "L").clamp(0, l)
        blkq, blkk = self.block_sizes(q.device.index)
        nblk = _utils.cdiv(l, blkk)
        topk = max(1, min(nblk, int(self.topk * nblk)))   # the LUT's row stride: no entry keeps more
        prep = _utils.quant_qk_vl(q, k, lens, blkq, blkk)
        topks = _utils.seq_topks(lens, self.topk, blkk)   # after the prep launches: its small ops then run under them
        sparse_map, lut = _utils.block_map_vl(prep.q_pool, prep.k_pool, topk, lens, topks, blkq, blkk)
        if getattr(self, "_keep_selection", None) is not None:
            self._keep_selection.update(lut=lut, sparse_map=sparse_map, topk=topk, topks=topks)
        kv, ksum = linear_moments_vl(k, v, lens, self.feature)
        kvw = project_moments(self.proj_l.weight.detach(), kv, self.dtype)
        proj_b = self.proj_l.bias.detach().float().contiguous()
        out = torch.empty_like(q)
        sm_scale = d ** -0.5
        if not self.quantised_qk and (self.feature == 0 or blkq == 64):
            check(lib().tdb200_sla_attn16_fwd_vl(ptr(q), ptr(k), ptr(v), DTYPE_TAG[q.dtype], ptr(lut), topk, ptr(kvw), ptr(ksum),
                                                 ptr(proj_b), ptr(out), b, l, l, h, d, ptr(lens), ptr(topks), sm_scale,
                                                 self.feature, blkq, blkk, stream_ptr(q.device)), "sla_attn16_fwd_vl")
        else:
            check(lib().tdb200_sla_attn_fwd_vl(ptr(prep.q_i8), ptr(prep.q_scale), ptr(prep.k_i8), ptr(prep.k_scale), ptr(v), ptr(q),
                                               DTYPE_TAG[q.dtype], ptr(lut), topk, ptr(kvw), ptr(ksum), ptr(proj_b), ptr(out), b, l, l,
                                               h, d, ptr(lens), ptr(topks), sm_scale, self.feature, blkq, blkk,
                                               stream_ptr(q.device)), "sla_attn_fwd_vl")
        o = out if out.dtype == dtype else out.to(dtype)
        if not return_sparsity:
            return o
        nblk_i = (lens.to(torch.int64) + blkk - 1) // blkk
        return o, torch.where(nblk_i > 0, topks.to(torch.float64) / nblk_i.clamp(min=1).to(torch.float64), 0.0)

    def _forward_train(self, q, k, v, return_sparsity):
        """The reference's SparseLinearAttention.forward (SLA/core.py:81-119) with autograd: the same block selection as the
        fused path, the sparse branch through sparse_attention16, the linear branch and proj_l in torch at the reference's
        rounding points (feature maps -> dtype, bmm in dtype, proj_l evaluated in dtype as under its autocast), or, with
        SLA.utils.set_linear_branch("fused"), through linear_branch's CUDA kernels."""
        if q.shape[-1] != 128:
            raise NotImplementedError(f"SparseLinearAttention backward: head dim {q.shape[-1]}; gradients are served for d = 128")
        require_cuda(q, k, v)
        dtype = q.dtype
        q, k, v = (t if (t.dtype == self.dtype and t.is_contiguous()) else t.to(self.dtype).contiguous() for t in (q, k, v))
        d = q.shape[-1]
        blkq, blkk = self.block_sizes(q.device.index)
        with torch.no_grad():
            prep = select_prep(q.detach(), k.detach(), blkq, blkk)
            nblk = prep.nblk
            real_topk = max(1, min(nblk, int(self.topk * nblk)))
            sparse_map, lut = block_map_from_pools(prep.q_pool, prep.k_pool, real_topk)
        if getattr(self, "_keep_selection", None) is not None:
            self._keep_selection.update(lut=lut, sparse_map=sparse_map, topk=real_topk)
        o_s = sparse_attention16(q, k, v, lut, real_topk, d ** -0.5, blkq)
        o_l = linear_branch(q, k, v, *self._proj, self.feature) if self._fused_linear() else self._linear_branch(q, k, v)
        o = (o_s + o_l).to(dtype).contiguous()
        return (o, real_topk / nblk) if return_sparsity else o

    def _forward_ad(self, q, k, v, return_sparsity):
        """forward() with a forward-AD rule: _forward_train's composition, the sparse branch through _SparseAttention16AD
        (one primal forward with the training op's bits; its tangent by tdb200_sla_attn16_tangent with the block selection
        held fixed; its backward the training op's) and the linear branch and proj_l in torch, whose forward AD gives their
        tangent (under torch.func.jvp torch's jvp rules for those ops may round differently from the plain ops).  Served
        where forward_jvp is; other calls raise NotImplementedError before any CUDA work."""
        self._refuse_unserved_jvp("forward with a forward-mode tangent", q.shape[-1])
        require_cuda(q, k, v)
        dtype = q.dtype
        q, k, v = (t if (t.dtype == self.dtype and t.is_contiguous()) else t.to(self.dtype).contiguous() for t in (q, k, v))
        b, l, h, d = q.shape
        nblk = (l + _ops.BLKK16 - 1) // _ops.BLKK16
        real_topk = max(1, min(nblk, int(self.topk * nblk)))
        o_s = _SparseAttention16AD.apply(q, k, v, real_topk, d ** -0.5, self)[0]
        o_l = linear_branch(q, k, v, *self._proj, self.feature) if self._fused_linear() else self._linear_branch(q, k, v)
        o = (o_s + o_l).to(dtype).contiguous()
        return (o, real_topk / nblk) if return_sparsity else o

    def _refuse_unserved_jvp(self, what, d):
        """NotImplementedError for the calls the sparse attention JVP and tangent kernels do not serve"""
        if self.quantised_qk:
            raise NotImplementedError(f"{what}: SageSparseLinearAttention is inference-only (as in the reference); "
                                      "use SparseLinearAttention")
        if d != 128:
            raise NotImplementedError(f"{what}: head dim {d}; the sparse attention JVP is served for d = 128")
        if (self.BLKQ, self.BLKK) != (128, 64):
            raise NotImplementedError(f"{what}: block sizes (BLKQ, BLKK) = ({self.BLKQ}, {self.BLKK}); the sparse attention "
                                      "JVP is served for (128, 64)")

    @property
    def _proj(self):
        return self.proj_l.weight, self.proj_l.bias

    def _fused_linear(self):
        """The linear branch of this call runs on the CUDA kernels: "fused" is selected (SLA.utils.set_linear_branch) and
        proj_l's parameters carry no forward-mode tangent (those calls take the torch branch, whose forward AD covers them)."""
        return _utils.LINEAR_BRANCH == "fused" and not has_tangent(*self._proj)

    def _linear_branch(self, q, k, v):
        """proj_l(phi(q) (phi(k)^T v) / (1e-5 + phi(q).sum phi(k))) as [B, L, H, D] in self.dtype, in torch at the reference's
        rounding points (SLA/core.py:104-117): feature maps -> dtype, bmm in dtype, proj_l evaluated in dtype as under its
        autocast."""
        qh, kh, vh = (t.transpose(1, 2) for t in (q, k, v))                       # [B, H, L, D] views
        c_q = self.feature_map_q(qh).contiguous().to(self.dtype)
        c_k = self.feature_map_k(kh).contiguous().to(self.dtype)
        kvsum = c_k.transpose(-1, -2) @ vh
        ksum = torch.sum(c_k, dim=-2, keepdim=True)
        o_l = (c_q @ kvsum) / (1e-5 + (c_q * ksum).sum(dim=-1, keepdim=True))
        o_l = F.linear(o_l.to(self.dtype), self.proj_l.weight.to(self.dtype), self.proj_l.bias.to(self.dtype))
        return o_l.transpose(1, 2)

    def forward_jvp(self, q, k, v, q_t, k_t, v_t, return_sparsity=False):
        """forward(q, k, v) and its forward-mode derivative along the tangents (q_t, k_t, v_t): (o, o_t), both [B, L, H, D] in
        q.dtype (plus the sparsity with return_sparsity), for the tangent pass of rCM / sCM consistency distillation.
        The block selection is forward's, computed from the primal q, k; the tangent holds it fixed (it is piecewise constant).
        The sparse branch is one kernel (sparse_attention16_jvp); the linear branch and proj_l are _forward_train's torch ops,
        their tangent by torch forward-mode AD.  o is differentiable in q, k, v and proj_l as _forward_train's output is; o_t
        never carries a gradient and the tangents get none.  Served for SparseLinearAttention with d = 128 and
        (BLKQ, BLKK) = (128, 64); every other call raises NotImplementedError before any CUDA work.  Eager only: under
        torch.compile it is a graph break.  The same tangent is what forward() carries under torch.func.jvp / forward_ad
        (_forward_ad); this is the explicit-tangent form of it."""
        self._refuse_unserved_jvp("forward_jvp", q.shape[-1])
        for name, t, primal in (("q_t", q_t, q), ("k_t", k_t, k), ("v_t", v_t, v)):
            if t.shape != primal.shape:
                raise ValueError(f"forward_jvp: {name} {tuple(t.shape)} must have its primal's shape {tuple(primal.shape)}")
        require_cuda(q, k, v, q_t, k_t, v_t)
        dtype = q.dtype
        q, k, v = (t if (t.dtype == self.dtype and t.is_contiguous()) else t.to(self.dtype).contiguous() for t in (q, k, v))
        q_t, k_t, v_t = (t.detach().to(self.dtype).contiguous() for t in (q_t, k_t, v_t))
        d = q.shape[-1]
        blkq, blkk = 128, 64
        with torch.no_grad():
            prep = select_prep(q.detach(), k.detach(), blkq, blkk)
            nblk = prep.nblk
            real_topk = max(1, min(nblk, int(self.topk * nblk)))
            sparse_map, lut = block_map_from_pools(prep.q_pool, prep.k_pool, real_topk)
        if getattr(self, "_keep_selection", None) is not None:
            self._keep_selection.update(lut=lut, sparse_map=sparse_map, topk=real_topk)
        o_s, o_s_t = sparse_attention16_jvp(q, k, v, q_t, k_t, v_t, lut, real_topk, d ** -0.5, blkq)
        if self._fused_linear():
            o_l, o_l_t = linear_branch_jvp(q, k, v, q_t, k_t, v_t, *self._proj, self.feature)
            o = (o_s + o_l).to(dtype).contiguous()
            o_t = (o_s_t + o_l_t).to(dtype).contiguous()
            return (o, o_t, real_topk / nblk) if return_sparsity else (o, o_t)
        with fwAD.dual_level():
            o_l = self._linear_branch(fwAD.make_dual(q, q_t), fwAD.make_dual(k, k_t), fwAD.make_dual(v, v_t))
            o_l, o_l_t = fwAD.unpack_dual(o_l)
        o = (o_s + o_l).to(dtype).contiguous()
        o_t = (o_s_t + o_l_t.detach()).to(dtype).contiguous()
        return (o, o_t, real_topk / nblk) if return_sparsity else (o, o_t)

    def forward_with_lut(self, q, k, v):
        """forward() that also returns the block selection it used: (o, {"lut": int32 [B,H,Mblk,topk] ascending key-block
        ids, "sparse_map": int8 [B,H,Mblk,Nblk], "topk": int}).  Test/diagnostic entry point (sampled oracle parity at
        full shapes needs the kernel's own selection)."""
        self._keep_selection = {}
        try:
            o = self.forward(q, k, v)
            return o, self._keep_selection
        finally:
            self._keep_selection = None


class SparseLinearAttention(_SLABase):
    """SLA/core.py:38-119: the non-quantised variant (`--attention_type sla`).  Block sizes (BLKQ, BLKK) = (128, 64) (the
    configuration modify_model.py:50 requests) and, for 128-wide heads, the constructor's default (64, 64) are served as
    the reference computes them.  128-wide heads run the fused kernel with a 16-bit Q.K^T (the arithmetic of the reference's
    Triton _attn_fwd, SLA/kernel.py:21-82); at (128, 64) the elu / relu maps and 64-wide heads are served by the INT8-QK
    kernel.  Other block sizes are accepted for signature compatibility with a warning and run as (128, 64)."""
    quantised_qk = False

    def block_sizes(self, device_index):
        """(BLKQ, BLKK) of this call: the constructor's pair where it is served, else (128, 64)."""
        return (self.BLKQ, self.BLKK) if self._served else (128, 64)

    def __init__(self, head_dim, topk, feature_map="softmax", BLKQ=64, BLKK=64, use_bf16=True, tie_feature_map_qk=True):
        super().__init__(head_dim, topk, feature_map, use_bf16, tie_feature_map_qk)
        self.BLKQ, self.BLKK = BLKQ, BLKK
        self._served = (BLKQ, BLKK) == (128, 64) or ((BLKQ, BLKK) == (64, 64) and head_dim == 128)
        if not self._served:
            import warnings
            warnings.warn(f"SparseLinearAttention(BLKQ={BLKQ}, BLKK={BLKK}): these kernels use 128-row query blocks and "
                          "64-row key blocks (the configuration TurboDiffusion's modify_model.py:50 requests); block "
                          "selection differs from the reference for other sizes", stacklevel=2)


class SageSparseLinearAttention(_SLABase):
    """SLA/core.py:122-257."""

    def __init__(self, head_dim, topk, feature_map="softmax", use_bf16=True, tie_feature_map_qk=True):
        super().__init__(head_dim, topk, feature_map, use_bf16, tie_feature_map_qk)

    def block_sizes(self, device_index):
        """The reference's choice (SLA/core.py:191-193): BLKQ=64 / BLKK=128 where get_cuda_arch reports sm90, else 128 / 64."""
        return SAGE_BLOCKS["sm90"] if get_cuda_arch(device_index) == "sm90" else SAGE_BLOCKS["sm100"]


# ------------------------------------------------------------------------------------------------------------------------
# Names the LTX-2 client reaches for inside `SLA.core` (TurboT2AV ltx_distillation/acceleration.py:260-383,
# LTXSageSLAAttention._sparse_only_forward, the default path while proj_l is still zero): SpargeAttn's quantiser, LUT
# builder, V preparation and the Sage2++ kernel entry.  Here they are thin adapters onto the same C-ABI kernels the modules
# use; the tensors SpargeAttn would transform (transposed / padded / fp8 V) are carried by reference instead, because the
# fused kernel consumes 16-bit V in its original layout.
# ------------------------------------------------------------------------------------------------------------------------
def get_vanilla_qk_quant(q, k, km=None, BLKQ=128, BLKK=64):
    """q,k [B,H,L,D] -> (q_int8 [B,H,L,D], q_scale [B,H,Mblk], k_int8 of (k - mean_L k), k_scale [B,H,Nblk]); call site
    SLA/core.py:200-203.  `km` is accepted for signature compatibility (the key mean is recomputed by the fused prepass).
    (BLKQ, BLKK) is (128, 64) or the Hopper family's (64, 128)."""
    if (BLKQ, BLKK) not in SAGE_BLOCKS.values():
        raise NotImplementedError(f"block sizes BLKQ={BLKQ}, BLKK={BLKK}: this implementation serves (128, 64) and (64, 128)")
    prep = quant_qk(q.transpose(1, 2).contiguous(), k.transpose(1, 2).contiguous(), blkq=BLKQ, blkk=BLKK)
    return prep.q_i8, prep.q_scale, prep.k_i8, prep.k_scale


def block_map_lut_triton(sparse_map):
    """sparse_map int8 [B,H,Mblk,Nblk] -> (lut int32 [B,H,Mblk,topk] ascending block ids, valid_block_num int32 [B,H,Mblk]).
    Maps produced by this package's get_block_map carry their LUT; others are rebuilt from the map (every row must select the
    same number of blocks, as get_block_map guarantees)."""
    valid = sparse_map.sum(-1, dtype=torch.int32)
    lut = getattr(sparse_map, "_tdb200_lut", None)
    if lut is None:
        b, h, m, n = sparse_map.shape
        topk = int(valid.reshape(-1)[0].item())
        lut = sparse_map.bool().nonzero()[:, -1].view(b, h, m, topk).to(torch.int32).contiguous()
    return lut, valid


class _FusedShim:
    """SpargeAttn `fused` namespace: V transposition / fp8 quantisation are not materialised; the outputs remember their source."""

    @staticmethod
    def transpose_pad_permute_cuda(v, out, tensor_layout=1):
        out._tdb200_src = v

    @staticmethod
    def scale_fuse_quant_cuda(v_in, v_fp8, v_scale, kv_len, scale_max=2.25, tensor_layout=1):
        v_fp8._tdb200_src = getattr(v_in, "_tdb200_src", v_in)


fused = _FusedShim()


def _sparse_only_attn(q_int8, k_int8, v_fp8, o, lut, q_scale, k_scale, sm_scale, blkq, blkk):
    """Sparse (softmax) branch only: o [B,H,L,D] <- block-sparse INT8-QK attention over the LUT's key blocks, the linear
    branch switched off (zero moments, zero bias).  Same kernel as SageSparseLinearAttention.forward, with its P.V setting
    (SLA.utils.set_sage_pv): under "fp8" the 16-bit V is quantised by tdb200_sla_quant_v_fp8 (d = 128 only)."""
    fp8_v = _utils.SAGE_PV == "fp8"
    if fp8_v and q_int8.shape[-1] != 128:
        raise NotImplementedError(f"FP8 P.V (SLA.utils.set_sage_pv('fp8')): head dim {q_int8.shape[-1]}; it is served for d = 128")
    v = getattr(v_fp8, "_tdb200_src", None)
    if v is None:
        raise RuntimeError("this adapter needs the 16-bit V that SLA.core.fused.* was called with")
    b, h, lq, d = q_int8.shape
    lk = k_int8.shape[2]
    prep = QKPrep()
    prep.q_i8, prep.q_scale, prep.k_i8, prep.k_scale = q_int8, q_scale, k_int8, k_scale
    prep.mblk, prep.nblk = (lq + blkq - 1) // blkq, (lk + blkk - 1) // blkk
    vt = v.transpose(1, 2).contiguous()                       # [B,L,H,D]
    qz = torch.zeros(b, lq, h, d, dtype=v.dtype, device=v.device)
    kvw = torch.zeros(b, h, d, d, dtype=v.dtype, device=v.device)
    ksum = torch.ones(b, h, d, dtype=torch.float32, device=v.device)
    pb = torch.zeros(d, dtype=torch.float32, device=v.device)
    out = attn_fwd(prep, vt, qz, lut, lut.shape[-1], kvw, ksum, pb, sm_scale if sm_scale is not None else d ** -0.5, lk=lk,
                   blkq=blkq, blkk=blkk, fp8_v=fp8_v)
    o.copy_(out.transpose(1, 2))
    return o


def qk_int8_sv_f8_accum_f16_block_sparse_attn_inst_buf_fuse_v_scale_with_pv_threshold(
        q_int8, k_int8, v_fp8, o, lut, valid_block_num, pvthreshold, q_scale, k_scale, v_scale, tensor_layout=1,
        is_causal=False, qk_quant_gran=1, sm_scale=None, return_lse=0):
    """The Sage2++ entry (BLKQ=128, BLKK=64): see _sparse_only_attn."""
    return _sparse_only_attn(q_int8, k_int8, v_fp8, o, lut, q_scale, k_scale, sm_scale, *SAGE_BLOCKS["sm100"])


class _QattnShim:
    """SpargeAttn's `qattn` extension module holds its sm80 / sm90 kernels.  The sm90 entry (BLKQ=64, BLKK=128) runs the fused
    kernel on those blocks; the sm80 kernels have no counterpart here."""

    @staticmethod
    def qk_int8_sv_f8_accum_f32_block_sparse_attn_inst_buf_fuse_v_scale_with_pv_threshold_sm90(
            q_int8, k_int8, v_fp8, o, lut, valid_block_num, pvthreshold, q_scale, k_scale, v_scale, tensor_layout=1,
            is_causal=False, qk_quant_gran=1, sm_scale=None, return_lse=0):
        """The Hopper entry (SLA/core.py:226-229), BLKQ=64 / BLKK=128: see _sparse_only_attn.  The argument list is taken to
        be the Sage2++ entry's, as recorded in SURVEY.md section 2.2; the SpargeAttn sources are not in this tree, so that
        signature is unverified."""
        return _sparse_only_attn(q_int8, k_int8, v_fp8, o, lut, q_scale, k_scale, sm_scale, *SAGE_BLOCKS["sm90"])

    def __getattr__(self, name):
        raise NotImplementedError(f"SLA.core.qattn.{name}: the sm80 SpargeAttn kernels have no counterpart here; "
                                  "call the Sage2++ entry or qattn's sm90 entry, which run the fused kernel")


qattn = _QattnShim()
