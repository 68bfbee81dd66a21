"""The Wan DiT block hot path composed from the H100 operators: a fused restatement of
`WanAttentionBlock.forward` (turbodiffusion/rcm/networks/wan2pt1.py:390-417) as TurboDiffusion runs it after model
surgery (inference/modify_model.py:40-81): Int8Linear everywhere in the block, FastLayerNorm / FastRMSNorm,
SageSLA self-attention, dense SDPA cross-attention over the text tokens.

Per block and per call the reference launches ~60 kernels and re-quantises the same activation three times for q/k/v;
here the sequence is
  LN+modulate+quant -> q/k/v GEMMs (shared int8 input) -> RMSNorm+RoPE (q,k) -> SLA (5 launches) -> quant+o GEMM
  -> gate/residual -> LN(affine) -> cross-attention (q/k/v/o GEMMs, library SDPA on 512 keys) -> residual
  -> LN+modulate+quant -> FFN-up GEMM (+bias+GELU+block-quant fused, int8 out) -> FFN-down GEMM -> gate/residual.
Weights use the reference's checkpoint format (Int8Linear buffers `int8_weight`, `scale`, `bias`).
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import ops
from .SLA.core import SageSparseLinearAttention, SparseLinearAttention
from .turbo_diffusion_ops import (gelu_quant_cuda, gemm_cuda_bias_gelu, gemm_cuda_quant_out, gemm_cuda_split,
                                  gemm_cuda_swizzle_bias, quant_cuda)

# FFN activation between the two W8A8 GEMMs:
#   "fused": bias + GELU (one-MUFU tanh) + quantisation in the up-projection's epilogue: no 16-bit intermediate in HBM; the
#            epilogue runs on the warps that dequantise;
#   "split": up-projection writes T(acc + bias); one HBM pass applies GELU(tanh) and the 128x128-block quantisation
#            (tdb200_gelu_quant_int8_block128), no activation on the GEMM's dequant warps.
# fused is the default: it saves the 16-bit intermediate's round trip through HBM.
FFN_ACT_MODE = os.environ.get("TDB200_FFN_ACT", "fused")

# Self-attention q/k/v as ONE GEMM against the row-concatenated weights (the packing of the LTX client's fused to_qkv,
# acceleration.py:836-860), outputs written as three contiguous matrices: bit-identical to the three GEMMs (scales are per
# 128 weight rows), fewer partial tile waves and two launches fewer.
#   "1": always, "0": never, "auto": single GPU yes; under a sequence-parallel hook no (the separate K projection lets the
#   K exchange start under the V and Q projections).  Unless "0" the cross-attention k/v of the text tokens are one GEMM too
#   (M = 512 rows: 12 tiles per projection on 132 SMs, so the fused launch costs what one of the two did).
FUSE_QKV = os.environ.get("TDB200_FUSE_QKV", "auto")

LINEARS = ("self_attn.q", "self_attn.k", "self_attn.v", "self_attn.o", "cross_attn.q", "cross_attn.k", "cross_attn.v",
           "cross_attn.o", "ffn.0", "ffn.2")


def random_block_state(dim: int, ffn_dim: int, heads: int, seed: int, device, dtype=torch.bfloat16) -> Dict[str, torch.Tensor]:
    """Random-init weights of one block in the reference's quantised state-dict layout (modify_model.py:156-183:
    Int8Linear.from_linear quantises nn.Linear weights with int8_quant)."""
    gdev = torch.device(device)
    g = torch.Generator(device=gdev).manual_seed(seed)  # generated on the target device (14B-parameter shapes)
    sd: Dict[str, torch.Tensor] = {}
    shapes = {"self_attn.q": (dim, dim), "self_attn.k": (dim, dim), "self_attn.v": (dim, dim), "self_attn.o": (dim, dim),
              "cross_attn.q": (dim, dim), "cross_attn.k": (dim, dim), "cross_attn.v": (dim, dim),
              "cross_attn.o": (dim, dim), "ffn.0": (ffn_dim, dim), "ffn.2": (dim, ffn_dim)}
    for name, (n, k) in shapes.items():
        w = (torch.randn(n, k, generator=g, device=gdev) * (k ** -0.5)).to(dtype)
        q, s = ops.int8_quant(w)
        sd[name + ".int8_weight"], sd[name + ".scale"] = q, s
        sd[name + ".bias"] = (torch.randn(n, generator=g, device=gdev) * 0.02).to(dtype)
    for name in ("self_attn.norm_q", "self_attn.norm_k", "cross_attn.norm_q", "cross_attn.norm_k"):
        sd[name + ".weight"] = (1.0 + 0.1 * torch.randn(dim, generator=g, device=gdev)).float()
    sd["norm3.weight"] = (1.0 + 0.1 * torch.randn(dim, generator=g, device=gdev)).float()
    sd["norm3.bias"] = (0.05 * torch.randn(dim, generator=g, device=gdev)).float()
    sd["modulation"] = (torch.randn(1, 6, dim, generator=g, device=gdev) / dim ** 0.5).float()
    d = dim // heads
    sd["self_attn.attn_op.local_attn.proj_l.weight"] = (torch.randn(d, d, generator=g, device=gdev) * 0.05).float()
    sd["self_attn.attn_op.local_attn.proj_l.bias"] = (torch.randn(d, generator=g, device=gdev) * 0.05).float()
    return sd


class WanBlockB200:
    """One DiT block on the H100 operators.  `sd` uses the reference state-dict keys relative to `blocks.<i>.`."""

    def __init__(self, sd: Dict[str, torch.Tensor], dim: int, heads: int, eps: float = 1e-6, topk: float = 0.1,
                 attention: str = "sagesla"):
        # norm weights / modulation are read by the fused kernels through fp32 pointers: a checkpoint loaded with
        # load_state_dict(assign=True) may hold them in bf16, so normalise them ONCE here (no per-call casts)
        sd = dict(sd)
        for key in ("self_attn.norm_q.weight", "self_attn.norm_k.weight", "cross_attn.norm_q.weight", "cross_attn.norm_k.weight",
                    "norm3.weight", "norm3.bias", "modulation"):
            if key in sd and (sd[key].dtype != torch.float32 or not sd[key].is_contiguous()):
                sd[key] = sd[key].float().contiguous()
        self.sd, self.dim, self.heads, self.eps = sd, dim, heads, eps
        self.head_dim = dim // heads
        dev = sd["modulation"].device
        # modify_model.py:48-52: "sagesla" -> SageSparseLinearAttention (INT8 Q.K^T), "sla" -> SparseLinearAttention(BLKQ=128, BLKK=64)
        self.sla = (SageSparseLinearAttention(self.head_dim, topk) if attention == "sagesla"
                    else SparseLinearAttention(self.head_dim, topk, BLKQ=128, BLKK=64)).to(dev)
        with torch.no_grad():
            self.sla.proj_l.weight.copy_(sd["self_attn.attn_op.local_attn.proj_l.weight"])
            self.sla.proj_l.bias.copy_(sd["self_attn.attn_op.local_attn.proj_l.bias"])
        self.attn_hook = None  # sequence-parallel wrapper installs its own attention callable here
        self._packed = {}      # fused projection weights (int8_weight, scale, bias), built on first use

    def _fused(self, *names):
        """Row-concatenated weights of projections that share their input (self-attention q/k/v, cross-attention k/v)."""
        if names not in self._packed:
            sd = self.sd
            if any(sd[n + ".int8_weight"].shape[0] % 256 for n in names):
                raise ValueError("fused projections need out_features % 256 == 0")
            self._packed[names] = tuple(torch.cat([sd[n + suffix] for n in names], dim=0).contiguous()
                                        for suffix in (".int8_weight", ".scale", ".bias"))
        return self._packed[names]

    # -- helpers -----------------------------------------------------------------------------------------------
    def _gemm(self, xq, xs, name, dtype, gelu=False):
        sd = self.sd
        w_q, w_s, bias = sd[name + ".int8_weight"], sd[name + ".scale"], sd[name + ".bias"]
        y = torch.empty(xq.shape[0], w_q.shape[0], dtype=dtype, device=xq.device)
        (gemm_cuda_bias_gelu if gelu else gemm_cuda_swizzle_bias)(xq, xs, w_q, w_s, y, bias)
        return y

    def _linear(self, x, name, gelu=False):
        xq, xs = quant_cuda(x)
        return self._gemm(xq, xs, name, x.dtype, gelu)

    # -- forward -------------------------------------------------------------------------------------------------
    def forward(self, x: torch.Tensor, e0: torch.Tensor, angles: torch.Tensor, context: torch.Tensor,
                stats: Optional[torch.Tensor] = None, want_stats: bool = False, e: Optional[torch.Tensor] = None):
        """x [L, dim] 16-bit, e0 [6, dim] fp32 (time modulation), angles [L, head_dim/2] fp32, context [Lc, dim].
        `stats`: LayerNorm row statistics of x if the producer of x already computed them (the previous block's last
        residual kernel does); with want_stats=True returns (x_out, stats_of_x_out) for the next block.  `e`: this block's
        `modulation + e0` [6, dim] fp32 if the caller already formed it (WanHotPath adds all blocks' tables in one launch)."""
        sd, dim, h, d, eps = self.sd, self.dim, self.heads, self.head_dim, self.eps
        l = x.shape[0]
        if e is None:
            e = (sd["modulation"][0] + e0).contiguous()  # [6, dim] fp32 (wan2pt1.py:400)

        # ---- self-attention (wan2pt1.py:404, 251-274)
        if stats is None:
            xq, xs = ops.layernorm_modulate_quant(x, e[1], e[0], eps)
        else:
            xq, xs = ops.layernorm_modulate_quant_from_stats(x, stats, e[1], e[0])
        # K and V first: the all-gather hook starts their exchange while Q is still being produced.  The head<->sequence
        # hook asks for Q first instead (its last exchange is hidden by the K/Q-side preparation, see dist.py).
        attn = self.attn_hook or self.sla
        fuse = FUSE_QKV == "1" or (FUSE_QKV == "auto" and self.attn_hook is None and dim % 256 == 0)
        if fuse:
            wq, ws, wb = self._fused("self_attn.q", "self_attn.k", "self_attn.v")
            q_raw, k_raw, v = gemm_cuda_split(xq, xs, wq, ws, wb, x.dtype, 3).unbind(0)
            proj = {"q": lambda: q_raw, "k": lambda: k_raw, "v": lambda: v}
        else:
            proj = {n: (lambda n=n: self._gemm(xq, xs, "self_attn." + n, x.dtype)) for n in ("q", "k", "v")}
        q = None
        if getattr(attn, "q_first", False):
            q = ops.rmsnorm_rope(proj["q"](), sd["self_attn.norm_q.weight"], angles, eps, h)
            attn.start_q(q.view(1, l, h, d))
        k = ops.rmsnorm_rope(proj["k"](), sd["self_attn.norm_k.weight"], angles, eps, h)
        if hasattr(attn, "start_k"):
            attn.start_k(k.view(1, l, h, d))
        v = proj["v"]()
        if hasattr(attn, "start_kv"):
            attn.start_kv(k.view(1, l, h, d), v.view(1, l, h, d))
        if q is None:
            q = ops.rmsnorm_rope(proj["q"](), sd["self_attn.norm_q.weight"], angles, eps, h)
        a = attn(q.view(1, l, h, d), k.view(1, l, h, d), v.view(1, l, h, d)).reshape(l, dim)
        y = self._linear(a, "self_attn.o")
        x = ops.gate_residual(x, y, e[2])  # x + y * e[2] (:405-406)

        # ---- cross-attention over the text tokens (:410, 277-298); dense SDPA stays a library call (512 keys)
        hn = ops.fast_layernorm(x, sd["norm3.weight"], sd["norm3.bias"], eps)
        cq = ops.fast_rmsnorm(self._linear(hn, "cross_attn.q"), sd["cross_attn.norm_q.weight"], eps)
        cxq, cxs = quant_cuda(context)      # one quantisation of the text tokens for both projections
        if FUSE_QKV != "0" and dim % 256 == 0:
            ck, cv = gemm_cuda_split(cxq, cxs, *self._fused("cross_attn.k", "cross_attn.v"), x.dtype, 2).unbind(0)
        else:
            ck, cv = self._gemm(cxq, cxs, "cross_attn.k", x.dtype), self._gemm(cxq, cxs, "cross_attn.v", x.dtype)
        ck = ops.fast_rmsnorm(ck, sd["cross_attn.norm_k.weight"], eps)
        lc = context.shape[0]
        ca = F.scaled_dot_product_attention(cq.view(1, l, h, d).transpose(1, 2), ck.view(1, lc, h, d).transpose(1, 2),
                                            cv.view(1, lc, h, d).transpose(1, 2))
        ca = ca.transpose(1, 2).reshape(l, dim)
        # x + cross_attn(...) and, in the same pass, the row statistics the FFN's LayerNorm needs
        x, st2 = ops.gate_residual_stats(x, self._linear(ca, "cross_attn.o"), None, eps)

        # ---- FFN (:411-413)
        hq, hs = ops.layernorm_modulate_quant_from_stats(x, st2, e[4], e[3])
        # Linear -> GELU(tanh) -> quant for the down projection, all in the up-projection's epilogue
        if FFN_ACT_MODE == "fused":
            uq, us = gemm_cuda_quant_out(hq, hs, sd["ffn.0.int8_weight"], sd["ffn.0.scale"], sd["ffn.0.bias"], x.dtype, gelu=True)
        else:
            uq, us = gelu_quant_cuda(self._gemm(hq, hs, "ffn.0", x.dtype))
        y = self._gemm(uq, us, "ffn.2", x.dtype)
        if want_stats:
            return ops.gate_residual_stats(x, y, e[5], eps)
        return ops.gate_residual(x, y, e[5])

    __call__ = forward


class WanHotPath:
    """`num_layers` distinct blocks = the per-denoise-step loop of WanModel.forward (wan2pt1.py:697-698)."""

    def __init__(self, dim: int, ffn_dim: int, heads: int, num_layers: int, device, topk: float = 0.1, seed: int = 0,
                 dtype=torch.bfloat16):
        self.dim, self.heads, self.dtype = dim, heads, dtype
        self.blocks = [WanBlockB200(random_block_state(dim, ffn_dim, heads, seed + i, device, dtype), dim, heads, topk=topk)
                       for i in range(num_layers)]
        self._mods = None

    def step(self, x, e0, angles, context):
        stats = None
        last = len(self.blocks) - 1
        if self._mods is None:   # every block's modulation table, stacked once: `modulation + e0` is then one launch per step
            self._mods = torch.stack([blk.sd["modulation"][0] for blk in self.blocks]).contiguous()
        e_all = self._mods + e0
        for i, blk in enumerate(self.blocks):
            if i < last:  # the block's final residual kernel also emits the next block's LayerNorm statistics
                x, stats = blk(x, e0, angles, context, stats, want_stats=True, e=e_all[i])
            else:
                x = blk(x, e0, angles, context, stats, e=e_all[i])
        return x
