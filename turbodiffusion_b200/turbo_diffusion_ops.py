"""Drop-in for the reference's pybind module `turbo_diffusion_ops` (turbodiffusion/ops/bindings.cpp:11-16).

Same function names, argument order and return values as the reference extension; the work is done by
libtdb200.so through its C ABI on the current CUDA stream.  Extra exports `gemm_cuda_swizzle` and
`gemm_cuda_swizzle_bias` are the ones TurboT2AV's acceleration.py looks up with getattr
(ltx_distillation/acceleration.py:695-701); the swizzle arguments are accepted and ignored (tile order is
an implementation detail of the GEMM kernel).
"""
from __future__ import annotations

import contextlib

from typing import Optional, Tuple

import torch

from . import _ops
from ._lib import DTYPE_TAG, require_cuda


def _cdiv(a, b):
    return (a + b - 1) // b


def quant_cuda(x: torch.Tensor, out_q: Optional[torch.Tensor] = None,
               out_s: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """quant.cu:28-71.  x [M,K] bf16/fp16 CUDA contiguous -> (q int8 [M,K], s fp32 [ceil(M/128), ceil(K/128)]).
    Allocates the outputs when None (common.hpp:65-84), else writes in place."""
    require_cuda(x)
    if x.dtype not in DTYPE_TAG:
        raise RuntimeError("Unsupported input data type for quant_cuda (bf16/fp16 only).")  # quant.cu:64-67
    if x.dim() != 2 or not x.is_contiguous():
        raise RuntimeError("quant_cuda expects a contiguous 2-D tensor")
    if out_q is None and out_s is None:
        return _ops.quant_int8_block128(x)
    m, k = x.shape
    if out_q is None:
        out_q = torch.empty((m, k), dtype=torch.int8, device=x.device)
    if out_s is None:
        out_s = torch.empty((_cdiv(m, 128), _cdiv(k, 128)), dtype=torch.float32, device=x.device)
    _ops.quant_int8_block128_out(x, out_q, out_s)
    return out_q, out_s


def gelu_quant_cuda(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """quant_cuda(gelu_tanh(x)) in one pass over x [M,K] bf16/fp16 (the FFN activation feeding the down projection)."""
    require_cuda(x)
    if x.dtype not in DTYPE_TAG or x.dim() != 2 or not x.is_contiguous():
        raise RuntimeError("gelu_quant_cuda expects a contiguous 2-D bf16/fp16 tensor")
    return _ops.gelu_quant_int8_block128(x)


GEMM_TIMER = None  # bench.py installs a callable(m, n, k) -> context manager to time GEMM launches with CUDA events


def _gemm(a_q, a_s, b_q, b_s, c, bias, epilogue: int = 0):
    if GEMM_TIMER is not None:
        with GEMM_TIMER(a_q.size(0), b_q.size(0), b_q.size(1)):
            return _gemm_impl(a_q, a_s, b_q, b_s, c, bias, epilogue)
    return _gemm_impl(a_q, a_s, b_q, b_s, c, bias, epilogue)


def _gemm_impl(a_q, a_s, b_q, b_s, c, bias, epilogue: int = 0):
    require_cuda(a_q, a_s, b_q, b_s, c, bias)
    if c.dtype not in DTYPE_TAG:
        raise RuntimeError("Unsupported output data type for int8 gemm.")  # gemm.cu:62-65
    for t in (a_q, a_s, b_q, b_s, c):
        if not t.is_contiguous():
            raise RuntimeError("gemm_cuda expects contiguous tensors")
    if bias is not None and bias.dtype != c.dtype:
        bias = bias.to(c.dtype)
    _ops.gemm_w8a8(a_q, a_s, b_q, b_s, bias, epilogue, c)   # M, N, K = a_q.size(0), b_q.size(0), b_q.size(1) (gemm.cu:37-39)


def gemm_cuda(a_q, a_s, b_q, b_s, c) -> None:
    """gemm.cu:27-68: writes C[M,N] (bf16/fp16) in place.  Shapes the reference silently skips (k % 128 != 0,
    launch.hpp:34-35) raise here instead of leaving zeros behind."""
    _gemm(a_q, a_s, b_q, b_s, c, None)


def gemm_cuda_swizzle(a_q, a_s, b_q, b_s, c, swizzle_dir: int = 1, swizzle_log: int = 5) -> None:
    _gemm(a_q, a_s, b_q, b_s, c, None)


def gemm_cuda_swizzle_bias(a_q, a_s, b_q, b_s, c, bias, swizzle_dir: int = 1, swizzle_log: int = 5) -> None:
    """Bias fused into the GEMM epilogue: c = T(T(acc) + bias)."""
    _gemm(a_q, a_s, b_q, b_s, c, bias)


def gemm_cuda_bias_gelu(a_q, a_s, b_q, b_s, c, bias) -> None:
    """c = T(gelu_tanh(T(T(acc) + bias))): Linear + nn.GELU(approximate="tanh") of the Wan FFN in one kernel."""
    _gemm(a_q, a_s, b_q, b_s, c, bias, epilogue=1)


def gemm_cuda_split(a_q, a_s, b_q, b_s, bias, out_dtype, parts: int):
    """One GEMM against `parts` row-concatenated projection weights (b_q [parts*n, k], b_s, bias); returns the outputs as a
    [parts, m, n] tensor of separate contiguous matrices (each bit-identical to its own gemm_cuda_swizzle_bias call)."""
    require_cuda(a_q, a_s, b_q, b_s, bias)
    if bias is not None and bias.dtype != out_dtype:
        bias = bias.to(out_dtype)
    with (GEMM_TIMER(a_q.size(0), b_q.size(0), b_q.size(1)) if GEMM_TIMER is not None else contextlib.nullcontext()):
        return _ops.gemm_w8a8_split(a_q, a_s, b_q, b_s, bias, out_dtype, parts)


def gemm_cuda_quant_out(a_q, a_s, b_q, b_s, bias, mid_dtype, gelu: bool = False):
    """(q, s) = quant_cuda(act(gemm + bias)) in one kernel; the 16-bit activation never reaches HBM."""
    require_cuda(a_q, a_s, b_q, b_s, bias)
    if bias is not None and bias.dtype != mid_dtype:
        bias = bias.to(mid_dtype)
    with (GEMM_TIMER(a_q.size(0), b_q.size(0), b_q.size(1)) if GEMM_TIMER is not None else contextlib.nullcontext()):
        return _ops.gemm_w8a8_quant_out(a_q, a_s, b_q, b_s, bias, mid_dtype, bool(gelu))


def rms_norm_cuda(x: torch.Tensor, eps: float, w: Optional[torch.Tensor] = None,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """rmsnorm.cu:57-59: fp32 [M,N] in, fp32 out."""
    require_cuda(x, w, out)
    if x.dtype != torch.float32 or x.dim() != 2 or not x.is_contiguous():
        raise RuntimeError("rms_norm_cuda expects a contiguous fp32 [M,N] tensor")
    if out is None:
        out = torch.empty_like(x)
    _ops.rms_norm_f32(x, w, float(eps), out)
    return out


def layer_norm_cuda(x: torch.Tensor, eps: float, w: Optional[torch.Tensor] = None, b: Optional[torch.Tensor] = None,
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """layernorm.cu:60-62: fp32 [M,N] in, fp32 out, optional affine."""
    require_cuda(x, w, b, out)
    if x.dtype != torch.float32 or x.dim() != 2 or not x.is_contiguous():
        raise RuntimeError("layer_norm_cuda expects a contiguous fp32 [M,N] tensor")
    if out is None:
        out = torch.empty_like(x)
    _ops.layer_norm_f32(x, w, b, float(eps), out)
    return out
