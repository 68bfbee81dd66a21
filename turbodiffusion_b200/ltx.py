"""LTX-2 (TurboT2AV) prologue operators on H100 — the second client of the operator API (SURVEY 8a row a12).

Same signatures as the fused helpers in ltx_core/model/transformer/transformer.py:46-94 and the Triton fast path
(ltx_distillation/fast_norm_kernels.py): x [B, T, N] bf16/fp16, scale_shift_table [num_ada, N], timestep [B, Tt, num_ada*N]
with Tt in {1, T}."""
from __future__ import annotations

import torch

from . import _ops
from ._lib import DTYPE_TAG, require_cuda


def _prep(x, table, timestep, num_ada):
    require_cuda(x, table, timestep)
    assert x.dim() == 3 and x.dtype in DTYPE_TAG
    b, t, n = x.shape
    ts = timestep.reshape(b, -1, num_ada * n).to(x.dtype).contiguous()
    return x.contiguous(), table.float().contiguous(), ts


def modulated_rms_norm_from_ada(x, scale_shift_table, timestep, scale_index, shift_index, num_ada_params, eps):
    x, tab, ts = _prep(x, scale_shift_table, timestep, num_ada_params)
    return _ops.ltx_modulated_rms_norm_ada(x, tab, ts, scale_index, shift_index, num_ada_params, float(eps))


def modulate_from_ada(x, scale_shift_table, timestep, scale_index, shift_index, num_ada_params):
    x, tab, ts = _prep(x, scale_shift_table, timestep, num_ada_params)
    return _ops.ltx_modulate_ada(x, tab, ts, scale_index, shift_index, num_ada_params)


def gated_residual_from_ada(x, residual, scale_shift_table, timestep, gate_index, num_ada_params):
    x, tab, ts = _prep(x, scale_shift_table, timestep, num_ada_params)
    return _ops.ltx_gated_residual_ada(x, residual.to(x.dtype).contiguous(), tab, ts, gate_index, num_ada_params)


def apply_split_rotary_emb(x, cos_freqs, sin_freqs):
    """x [B, T, H*D] (or [B, T, H, D]); cos/sin [B, H, T, D/2]  (ltx_core/model/transformer/rope.py:42-60)."""
    require_cuda(x, cos_freqs, sin_freqs)
    return _ops.ltx_split_rope(x.contiguous(), cos_freqs.to(x.dtype).contiguous(), sin_freqs.to(x.dtype).contiguous())


# ------------------------------------------------------------------------------------------------ per-row post-scale W8A8
def row_quant_int8(x: torch.Tensor, out_q: torch.Tensor = None, out_s: torch.Tensor = None):
    """ltx_distillation/tilelang_w8a8.py:39-75: x [M,K] bf16/fp16 -> (int8 [M,K], fp32 scale [M])."""
    require_cuda(x)
    assert x.dim() == 2 and x.is_contiguous() and x.dtype in DTYPE_TAG
    if out_q is None and out_s is None:
        return _ops.quant_int8_rowwise(x)
    m, k = x.shape
    q = torch.empty((m, k), dtype=torch.int8, device=x.device) if out_q is None else out_q
    s = torch.empty((m,), dtype=torch.float32, device=x.device) if out_s is None else out_s
    _ops.quant_int8_rowwise_out(x, q, s)
    return q, s


def gemm_int8_post_scale_bias(x_q, x_s, w_q, w_s, bias, out_dtype=torch.bfloat16):
    """_tl_gemm_int8_post_scale_bias (tilelang_w8a8.py:78-117): C = acc_int32 * sA[i] * sB[j] + bias[j], evaluated as the
    reference's compiled kernel does: fma(float(acc) * sA[i], sB[j], bias[j]) (see tools/tilelang_epilogue_probe.py)."""
    require_cuda(x_q, x_s, w_q, w_s, bias)
    if bias is not None and bias.dtype != out_dtype:
        bias = bias.to(out_dtype)
    return _ops.gemm_w8a8_rowwise(x_q, x_s, w_q, w_s, bias, out_dtype)


class PostScaleInt8Linear(torch.nn.Module):
    """Mirror of TileLangPostScaleInt8Linear (tilelang_w8a8.py:120-258): buffers int8_weight [N,K], scale [N], bias [N]."""

    def __init__(self, in_features, out_features, bias=True, dtype=torch.bfloat16):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.register_buffer("int8_weight", torch.empty((out_features, in_features), dtype=torch.int8))
        self.register_buffer("scale", torch.empty((out_features,), dtype=torch.float32))
        self.register_buffer("bias", torch.zeros(out_features, dtype=dtype))
        self._had_bias = bias

    def forward(self, x):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1]).contiguous()
        x_q, x_s = row_quant_int8(x2)
        y = gemm_int8_post_scale_bias(x_q, x_s, self.int8_weight, self.scale, self.bias, x.dtype)
        return y.reshape(*shape[:-1], self.out_features)

    @classmethod
    def from_linear(cls, lin: torch.nn.Linear):
        layer = cls(lin.in_features, lin.out_features, bias=lin.bias is not None, dtype=torch.bfloat16).to(lin.weight.device)
        w_q, w_s = row_quant_int8(lin.weight.detach().to(torch.bfloat16).contiguous())
        layer.int8_weight.copy_(w_q)
        layer.scale.copy_(w_s)
        if lin.bias is not None:
            layer.bias.copy_(lin.bias.detach().to(torch.bfloat16))
        return layer

    @classmethod
    def from_tilelang_linears(cls, linears):
        """tilelang_w8a8.py:229-258: one layer for projections that share their input (to_q/to_k/to_v -> to_qkv, to_k/to_v ->
        to_kv): INT8 weights, per-output-channel scales and biases concatenated along the output dimension.  The scales are
        per channel, so `fused(x).split(...)` equals the separate layers' outputs bit for bit."""
        if not linears:
            raise ValueError("Expected at least one PostScaleInt8Linear")
        k = linears[0].in_features
        if any(lin.in_features != k for lin in linears):
            raise ValueError("Fused W8A8 linears must share in_features")
        dev = linears[0].int8_weight.device
        if any(lin.int8_weight.device != dev for lin in linears):
            raise ValueError("Fused W8A8 linears must share a device")
        fused = cls(k, sum(lin.out_features for lin in linears), bias=any(lin._had_bias for lin in linears),
                    dtype=linears[0].bias.dtype).to(dev)
        fused.int8_weight.copy_(torch.cat([lin.int8_weight for lin in linears], dim=0))
        fused.scale.copy_(torch.cat([lin.scale for lin in linears], dim=0))
        fused.bias.copy_(torch.cat([lin.bias if lin._had_bias else torch.zeros_like(lin.bias) for lin in linears], dim=0))
        return fused


def fuse_attention_projections(model: torch.nn.Module) -> int:
    """fuse_tilelang_attention_projections (acceleration.py:836-860): every module whose to_q/to_k/to_v are PostScaleInt8Linear
    with equal in_features gains `to_qkv`; equal to_k/to_v in_features gains `to_kv` (what ltx_core's Attention.forward looks
    up, attention.py:186-193).  Returns the number of fused layers added."""
    fused = 0
    for module in model.modules():
        if not all(isinstance(getattr(module, a, None), PostScaleInt8Linear) for a in ("to_k", "to_v")):
            continue
        if isinstance(getattr(module, "to_q", None), PostScaleInt8Linear) and (
                module.to_q.in_features == module.to_k.in_features == module.to_v.in_features):
            module.to_qkv = PostScaleInt8Linear.from_tilelang_linears((module.to_q, module.to_k, module.to_v))
            fused += 1
        if module.to_k.in_features == module.to_v.in_features:
            module.to_kv = PostScaleInt8Linear.from_tilelang_linears((module.to_k, module.to_v))
            fused += 1
    return fused
