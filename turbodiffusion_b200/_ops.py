"""The `tdb200::` PyTorch operators: every C-ABI entry point the public functions launch work through, registered with
torch.library so that torch.compile (fullgraph=True included) and torch.export trace them as single graph nodes.

Each op has two implementations:
  CUDA  the ctypes call into libtdb200.so (include/tdb200.h) on the current stream of the tensors' device, exactly as the
        public functions made it before; outputs are allocated here, in PyTorch;
  fake  output shapes, dtypes and strides (all contiguous) derived from the inputs, for FakeTensor tracing.
Validation, dtype coercion and defaults stay in the public functions (turbo_diffusion_ops, ops.core, ltx, SLA), which call
the op handles below.  Ops that write into caller-provided tensors declare them mutated (`Tensor(a!)`) and return nothing.
The block-sparse attention forward with row log-sum-exp carries an autograd formula whose backward is the sparse backward
kernel.
"""
from __future__ import annotations

import torch

from ._lib import DTYPE_TAG, check, lib, ptr, stream_ptr

LIB = torch.library.Library("tdb200", "DEF")


def _cdiv(a, b):
    return (a + b - 1) // b


def _op(schema: str, cuda, fake, lib=LIB, ns="tdb200"):
    name = schema.split("(", 1)[0]
    lib.define(schema)
    lib.impl(name, cuda, "CUDA")
    torch.library.register_fake(f"{ns}::{name}", fake, lib=lib)
    return getattr(getattr(torch.ops, ns), name).default


def _like(x, shape=None, dtype=None):
    return torch.empty(x.shape if shape is None else shape, dtype=x.dtype if dtype is None else dtype, device=x.device)


def _block_scales(x, m, k):
    return torch.empty((_cdiv(m, 128), _cdiv(k, 128)), dtype=torch.float32, device=x.device)


# ------------------------------------------------------------------------------------------------ 128x128-block INT8 quantisation
def _quant_out_cuda(x, out_q, out_s):
    m, k = x.shape
    if m == 0 or k == 0:         # empty batch: nothing to launch (an empty tensor has no data pointer to hand to the C ABI)
        return
    check(lib().tdb200_quant_int8_block128(ptr(x), DTYPE_TAG[x.dtype], m, k, ptr(out_q), ptr(out_s), stream_ptr(x.device)),
          "quant_cuda")


def _quant_cuda(x):
    q, s = _like(x, dtype=torch.int8), _block_scales(x, *x.shape)
    _quant_out_cuda(x, q, s)
    return q, s


def _quant_fake(x):
    return _like(x, dtype=torch.int8), _block_scales(x, *x.shape)


quant_int8_block128 = _op("quant_int8_block128(Tensor x) -> (Tensor, Tensor)", _quant_cuda, _quant_fake)
quant_int8_block128_out = _op("quant_int8_block128_out(Tensor x, Tensor(a!) out_q, Tensor(b!) out_s) -> ()",
                              _quant_out_cuda, lambda x, out_q, out_s: None)


def _gelu_quant_cuda(x):
    m, k = x.shape
    q, s = _quant_fake(x)
    check(lib().tdb200_gelu_quant_int8_block128(ptr(x), DTYPE_TAG[x.dtype], m, k, ptr(q), ptr(s), stream_ptr(x.device)),
          "gelu_quant_cuda")
    return q, s


gelu_quant_int8_block128 = _op("gelu_quant_int8_block128(Tensor x) -> (Tensor, Tensor)", _gelu_quant_cuda, _quant_fake)


# ------------------------------------------------------------------------------------------------ W8A8 GEMM family
def _gemm_cuda(a_q, a_s, b_q, b_s, bias, epilogue, c):
    m, n, k = a_q.size(0), b_q.size(0), b_q.size(1)
    if m == 0 or n == 0:
        return
    check(lib().tdb200_gemm_w8a8_ex(ptr(a_q), ptr(a_s), ptr(b_q), ptr(b_s), ptr(bias), ptr(c), DTYPE_TAG[c.dtype], m, n, k,
                                    epilogue, stream_ptr(c.device)), "gemm_cuda")


gemm_w8a8 = _op("gemm_w8a8(Tensor a_q, Tensor a_s, Tensor b_q, Tensor b_s, Tensor? bias, int epilogue, Tensor(a!) c) -> ()",
                _gemm_cuda, lambda a_q, a_s, b_q, b_s, bias, epilogue, c: None)


def _gemm_split_fake(a_q, a_s, b_q, b_s, bias, out_dtype, parts):
    return torch.empty((parts, a_q.size(0), b_q.size(0) // parts), dtype=out_dtype, device=a_q.device)


def _gemm_split_cuda(a_q, a_s, b_q, b_s, bias, out_dtype, parts):
    m, n, k = a_q.size(0), b_q.size(0), b_q.size(1)
    c = _gemm_split_fake(a_q, a_s, b_q, b_s, bias, out_dtype, parts)
    check(lib().tdb200_gemm_w8a8_split(ptr(a_q), ptr(a_s), ptr(b_q), ptr(b_s), ptr(bias), ptr(c), DTYPE_TAG[out_dtype], m, n,
                                       k, parts, stream_ptr(a_q.device)), "gemm_cuda_split")
    return c


gemm_w8a8_split = _op("gemm_w8a8_split(Tensor a_q, Tensor a_s, Tensor b_q, Tensor b_s, Tensor? bias, ScalarType out_dtype, "
                      "int parts) -> Tensor", _gemm_split_cuda, _gemm_split_fake)


def _gemm_quant_out_fake(a_q, a_s, b_q, b_s, bias, mid_dtype, gelu):
    m, n = a_q.size(0), b_q.size(0)
    return torch.empty((m, n), dtype=torch.int8, device=a_q.device), _block_scales(a_q, m, n)


def _gemm_quant_out_cuda(a_q, a_s, b_q, b_s, bias, mid_dtype, gelu):
    m, n, k = a_q.size(0), b_q.size(0), b_q.size(1)
    q, s = _gemm_quant_out_fake(a_q, a_s, b_q, b_s, bias, mid_dtype, gelu)
    check(lib().tdb200_gemm_w8a8_quant_out(ptr(a_q), ptr(a_s), ptr(b_q), ptr(b_s), ptr(bias), ptr(q), ptr(s),
                                           DTYPE_TAG[mid_dtype], m, n, k, 1 if gelu else 0, stream_ptr(a_q.device)),
          "gemm_cuda_quant_out")
    return q, s


gemm_w8a8_quant_out = _op("gemm_w8a8_quant_out(Tensor a_q, Tensor a_s, Tensor b_q, Tensor b_s, Tensor? bias, "
                          "ScalarType mid_dtype, bool gelu) -> (Tensor, Tensor)", _gemm_quant_out_cuda, _gemm_quant_out_fake)


# ------------------------------------------------------------------------------------------------ norms
def _rms_norm_f32_cuda(x, w, eps, out):
    check(lib().tdb200_rms_norm_f32(ptr(x), ptr(w), ptr(out), x.shape[0], x.shape[1], eps, stream_ptr(x.device)),
          "rms_norm_cuda")


def _layer_norm_f32_cuda(x, w, b, eps, out):
    check(lib().tdb200_layer_norm_f32(ptr(x), ptr(w), ptr(b), ptr(out), x.shape[0], x.shape[1], eps, stream_ptr(x.device)),
          "layer_norm_cuda")


rms_norm_f32 = _op("rms_norm_f32(Tensor x, Tensor? w, float eps, Tensor(a!) out) -> ()", _rms_norm_f32_cuda,
                   lambda x, w, eps, out: None)
layer_norm_f32 = _op("layer_norm_f32(Tensor x, Tensor? w, Tensor? b, float eps, Tensor(a!) out) -> ()", _layer_norm_f32_cuda,
                     lambda x, w, b, eps, out: None)


def _rms_norm_cuda(x, w, eps):
    y = _like(x)
    if x.numel():
        check(lib().tdb200_rms_norm(ptr(x), DTYPE_TAG[x.dtype], ptr(w), ptr(y), x.shape[0], x.shape[1], eps,
                                    stream_ptr(x.device)), "fast_rmsnorm")
    return y


def _layer_norm_cuda(x, w, b, eps):
    y = _like(x)
    if x.numel():
        check(lib().tdb200_layer_norm(ptr(x), DTYPE_TAG[x.dtype], ptr(w), ptr(b), ptr(y), x.shape[0], x.shape[1], eps,
                                      stream_ptr(x.device)), "fast_layernorm")
    return y


rms_norm = _op("rms_norm(Tensor x, Tensor? w, float eps) -> Tensor", _rms_norm_cuda, lambda x, w, eps: _like(x))
layer_norm = _op("layer_norm(Tensor x, Tensor? w, Tensor? b, float eps) -> Tensor", _layer_norm_cuda,
                 lambda x, w, b, eps: _like(x))


# ------------------------------------------------------------------------------------------------ fused prologues / epilogues
def _ln_mod_cuda(x, scale, shift, eps):
    y = _like(x)
    check(lib().tdb200_layer_norm_modulate(ptr(x), DTYPE_TAG[x.dtype], ptr(scale), ptr(shift), ptr(y), x.shape[0], x.shape[1],
                                           eps, stream_ptr(x.device)), "layernorm_modulate")
    return y


layer_norm_modulate = _op("layer_norm_modulate(Tensor x, Tensor scale, Tensor shift, float eps) -> Tensor", _ln_mod_cuda,
                          lambda x, scale, shift, eps: _like(x))


def _ln_mod_quant_cuda(x, scale, shift, eps):
    m, n = x.shape
    q, s = _quant_fake(x)
    stats = torch.empty((2 * m,), dtype=torch.float32, device=x.device)
    check(lib().tdb200_layer_norm_modulate_quant(ptr(x), DTYPE_TAG[x.dtype], ptr(scale), ptr(shift), ptr(q), ptr(s), ptr(stats),
                                                 m, n, eps, stream_ptr(x.device)), "layernorm_modulate_quant")
    return q, s


layer_norm_modulate_quant = _op("layer_norm_modulate_quant(Tensor x, Tensor scale, Tensor shift, float eps) -> (Tensor, Tensor)",
                                _ln_mod_quant_cuda, lambda x, scale, shift, eps: _quant_fake(x))


def _ln_mod_quant_stats_cuda(x, stats, scale, shift):
    m, n = x.shape
    q, s = _quant_fake(x)
    check(lib().tdb200_layer_norm_modulate_quant_stats(ptr(x), DTYPE_TAG[x.dtype], ptr(stats), ptr(scale), ptr(shift), ptr(q),
                                                       ptr(s), m, n, stream_ptr(x.device)), "layernorm_modulate_quant_from_stats")
    return q, s


layer_norm_modulate_quant_stats = _op("layer_norm_modulate_quant_stats(Tensor x, Tensor stats, Tensor scale, Tensor shift) "
                                      "-> (Tensor, Tensor)", _ln_mod_quant_stats_cuda,
                                      lambda x, stats, scale, shift: _quant_fake(x))


def _gate_residual_cuda(x, y, gate):
    out = _like(x)
    check(lib().tdb200_gate_residual(ptr(x), ptr(y), ptr(gate), ptr(out), DTYPE_TAG[x.dtype], x.shape[0], x.shape[1],
                                     stream_ptr(x.device)), "gate_residual")
    return out


gate_residual = _op("gate_residual(Tensor x, Tensor y, Tensor? gate) -> Tensor", _gate_residual_cuda,
                    lambda x, y, gate: _like(x))


def _gate_residual_stats_fake(x, y, gate, eps):
    return _like(x), torch.empty((2 * x.shape[0],), dtype=torch.float32, device=x.device)


def _gate_residual_stats_cuda(x, y, gate, eps):
    out, stats = _gate_residual_stats_fake(x, y, gate, eps)
    check(lib().tdb200_gate_residual_stats(ptr(x), ptr(y), ptr(gate), ptr(out), ptr(stats), DTYPE_TAG[x.dtype], x.shape[0],
                                           x.shape[1], eps, stream_ptr(x.device)), "gate_residual_stats")
    return out, stats


gate_residual_stats = _op("gate_residual_stats(Tensor x, Tensor y, Tensor? gate, float eps) -> (Tensor, Tensor)",
                          _gate_residual_stats_cuda, _gate_residual_stats_fake)


def _rope_interleaved_cuda(x, angles):
    h, d = x.shape[-2:]
    y = _like(x)
    check(lib().tdb200_rope_interleaved(ptr(x), DTYPE_TAG[x.dtype], ptr(angles), ptr(y), x.numel() // (h * d), h, d,
                                        stream_ptr(x.device)), "rope_interleaved")
    return y


rope_interleaved = _op("rope_interleaved(Tensor x, Tensor angles) -> Tensor", _rope_interleaved_cuda,
                       lambda x, angles: _like(x))


def _rms_norm_rope_cuda(x, w, angles, eps, heads):
    l, hd = x.shape
    y = _like(x)
    check(lib().tdb200_rms_norm_rope(ptr(x), DTYPE_TAG[x.dtype], ptr(w), ptr(angles), ptr(y), l, heads, hd // heads, eps,
                                     stream_ptr(x.device)), "rmsnorm_rope")
    return y


def _rms_norm_rope_table_cuda(x, w, table, eps, heads):
    l, hd = x.shape
    y = _like(x)
    check(lib().tdb200_rms_norm_rope_table(ptr(x), DTYPE_TAG[x.dtype], ptr(w), ptr(table), ptr(y), l, heads, hd // heads, eps,
                                           stream_ptr(x.device)), "rmsnorm_rope")
    return y


rms_norm_rope = _op("rms_norm_rope(Tensor x, Tensor w, Tensor angles, float eps, int heads) -> Tensor", _rms_norm_rope_cuda,
                    lambda x, w, angles, eps, heads: _like(x))
rms_norm_rope_table = _op("rms_norm_rope_table(Tensor x, Tensor w, Tensor table, float eps, int heads) -> Tensor",
                          _rms_norm_rope_table_cuda, lambda x, w, table, eps, heads: _like(x))


# ------------------------------------------------------------------------------------------------ LTX-2 prologue operators
def _ltx_rms_ada_cuda(x, table, timestep, scale_index, shift_index, num_ada, eps):
    b, t, n = x.shape
    y = _like(x)
    check(lib().tdb200_ltx_modulated_rms_norm_ada(ptr(x), DTYPE_TAG[x.dtype], ptr(table), ptr(timestep), scale_index,
                                                  shift_index, num_ada, ptr(y), b, t, timestep.shape[1], n, eps,
                                                  stream_ptr(x.device)), "ltx_modulated_rms_norm_ada")
    return y


def _ltx_mod_ada_cuda(x, table, timestep, scale_index, shift_index, num_ada):
    b, t, n = x.shape
    y = _like(x)
    check(lib().tdb200_ltx_modulate_ada(ptr(x), DTYPE_TAG[x.dtype], ptr(table), ptr(timestep), scale_index, shift_index,
                                        num_ada, ptr(y), b, t, timestep.shape[1], n, stream_ptr(x.device)), "ltx_modulate_ada")
    return y


def _ltx_gate_ada_cuda(x, residual, table, timestep, gate_index, num_ada):
    b, t, n = x.shape
    y = _like(x)
    check(lib().tdb200_ltx_gated_residual_ada(ptr(x), ptr(residual), DTYPE_TAG[x.dtype], ptr(table), ptr(timestep), gate_index,
                                              num_ada, ptr(y), b, t, timestep.shape[1], n, stream_ptr(x.device)),
          "ltx_gated_residual_ada")
    return y


ltx_modulated_rms_norm_ada = _op("ltx_modulated_rms_norm_ada(Tensor x, Tensor table, Tensor timestep, int scale_index, "
                                 "int shift_index, int num_ada, float eps) -> Tensor", _ltx_rms_ada_cuda,
                                 lambda x, table, timestep, scale_index, shift_index, num_ada, eps: _like(x))
ltx_modulate_ada = _op("ltx_modulate_ada(Tensor x, Tensor table, Tensor timestep, int scale_index, int shift_index, "
                       "int num_ada) -> Tensor", _ltx_mod_ada_cuda,
                       lambda x, table, timestep, scale_index, shift_index, num_ada: _like(x))
ltx_gated_residual_ada = _op("ltx_gated_residual_ada(Tensor x, Tensor residual, Tensor table, Tensor timestep, int gate_index, "
                             "int num_ada) -> Tensor", _ltx_gate_ada_cuda,
                             lambda x, residual, table, timestep, gate_index, num_ada: _like(x))


def _ltx_split_rope_cuda(x, cos, sin):
    b, h, t, half = cos.shape
    y = _like(x)
    check(lib().tdb200_ltx_split_rope(ptr(x), ptr(cos), ptr(sin), DTYPE_TAG[x.dtype], ptr(y), b, t, h, 2 * half,
                                      stream_ptr(x.device)), "ltx_split_rope")
    return y


ltx_split_rope = _op("ltx_split_rope(Tensor x, Tensor cos, Tensor sin) -> Tensor", _ltx_split_rope_cuda,
                     lambda x, cos, sin: _like(x))


def _row_quant_out_cuda(x, out_q, out_s):
    m, k = x.shape
    check(lib().tdb200_quant_int8_rowwise(ptr(x), DTYPE_TAG[x.dtype], m, k, ptr(out_q), ptr(out_s), stream_ptr(x.device)),
          "quant_int8_rowwise")


def _row_quant_fake(x):
    return _like(x, dtype=torch.int8), torch.empty((x.shape[0],), dtype=torch.float32, device=x.device)


def _row_quant_cuda(x):
    q, s = _row_quant_fake(x)
    _row_quant_out_cuda(x, q, s)
    return q, s


quant_int8_rowwise = _op("quant_int8_rowwise(Tensor x) -> (Tensor, Tensor)", _row_quant_cuda, _row_quant_fake)
quant_int8_rowwise_out = _op("quant_int8_rowwise_out(Tensor x, Tensor(a!) out_q, Tensor(b!) out_s) -> ()", _row_quant_out_cuda,
                             lambda x, out_q, out_s: None)


def _gemm_rowwise_fake(x_q, x_s, w_q, w_s, bias, out_dtype):
    return torch.empty((x_q.shape[0], w_q.shape[0]), dtype=out_dtype, device=x_q.device)


def _gemm_rowwise_cuda(x_q, x_s, w_q, w_s, bias, out_dtype):
    m, k = x_q.shape
    y = _gemm_rowwise_fake(x_q, x_s, w_q, w_s, bias, out_dtype)
    check(lib().tdb200_gemm_w8a8_rowwise(ptr(x_q), ptr(x_s), ptr(w_q), ptr(w_s), ptr(bias), ptr(y), DTYPE_TAG[out_dtype], m,
                                         w_q.shape[0], k, stream_ptr(x_q.device)), "gemm_w8a8_rowwise")
    return y


gemm_w8a8_rowwise = _op("gemm_w8a8_rowwise(Tensor x_q, Tensor x_s, Tensor w_q, Tensor w_s, Tensor? bias, "
                        "ScalarType out_dtype) -> Tensor", _gemm_rowwise_cuda, _gemm_rowwise_fake)


# ------------------------------------------------------------------------------------------------ SparseLinearAttention
def _q_half(q, blkq):
    b, lq, h, d = q.shape
    mblk = _cdiv(lq, blkq)
    dev = q.device
    return (torch.empty(b, h, lq, d, dtype=torch.int8, device=dev), torch.empty(b, h, mblk, dtype=torch.float32, device=dev),
            torch.empty(b, h, mblk, d, dtype=q.dtype, device=dev))


def _k_half(k, lk, blkk):
    b, _, h, d = k.shape
    nblk = _cdiv(lk, blkk)
    dev = k.device
    return (torch.empty(b, h, d, dtype=torch.float32, device=dev), torch.empty(b, h, lk, d, dtype=torch.int8, device=dev),
            torch.empty(b, h, nblk, dtype=torch.float32, device=dev), torch.empty(b, h, nblk, d, dtype=k.dtype, device=dev))


def _quant_qk_fake(q, k, lk, blkq, blkk):
    q_i8, q_scale, q_pool = _q_half(q, blkq)
    kmean, k_i8, k_scale, k_pool = _k_half(k, lk, blkk)
    return kmean, q_i8, q_scale, k_i8, k_scale, q_pool, k_pool


def _quant_qk_cuda(q, k, lk, blkq, blkk):
    b, lq, h, d = q.shape
    out = _quant_qk_fake(q, k, lk, blkq, blkk)
    check(lib().tdb200_sla_quant_qk(ptr(q), ptr(k), DTYPE_TAG[q.dtype], b, lq, lk, h, d, *map(ptr, out), blkq, blkk,
                                    stream_ptr(q.device)), "sla_quant_qk")
    return out


def _quant_q_cuda(q, blkq):
    b, lq, h, d = q.shape
    q_i8, q_scale, q_pool = out = _q_half(q, blkq)
    # the key block size only matters to the key half; any valid pair with this blkq serves
    check(lib().tdb200_sla_quant_qk(ptr(q), None, DTYPE_TAG[q.dtype], b, lq, lq, h, d, None, ptr(q_i8), ptr(q_scale), None,
                                    None, ptr(q_pool), None, blkq, 64 if blkq == 128 else 128, stream_ptr(q.device)),
          "sla_quant_qk", launches=1)
    return out


def _quant_k_cuda(k, lk, blkk):
    b, _, h, d = k.shape
    kmean, k_i8, k_scale, k_pool = out = _k_half(k, lk, blkk)
    check(lib().tdb200_sla_quant_qk(None, ptr(k), DTYPE_TAG[k.dtype], b, lk, lk, h, d, ptr(kmean), None, None, ptr(k_i8),
                                    ptr(k_scale), None, ptr(k_pool), 128 if blkk == 64 else 64, blkk, stream_ptr(k.device)),
          "sla_quant_qk", launches=3)
    return out


sla_quant_qk = _op("sla_quant_qk(Tensor q, Tensor k, int lk, int blkq, int blkk) -> "
                   "(Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor)", _quant_qk_cuda, _quant_qk_fake)
sla_quant_q = _op("sla_quant_q(Tensor q, int blkq) -> (Tensor, Tensor, Tensor)", _quant_q_cuda, _q_half)
sla_quant_k = _op("sla_quant_k(Tensor k, int lk, int blkk) -> (Tensor, Tensor, Tensor, Tensor)", _quant_k_cuda, _k_half)


def _block_map_fake(q_pool, k_pool, topk):
    b, h, mblk, _ = q_pool.shape
    dev = q_pool.device
    return (torch.empty(b, h, mblk, k_pool.shape[2], dtype=torch.int8, device=dev),
            torch.empty(b, h, mblk, topk, dtype=torch.int32, device=dev))


def _block_map_cuda(q_pool, k_pool, topk):
    b, h, mblk, d = q_pool.shape
    sparse_map, lut = _block_map_fake(q_pool, k_pool, topk)
    check(lib().tdb200_sla_block_map(ptr(q_pool), ptr(k_pool), DTYPE_TAG[q_pool.dtype], b, h, mblk, k_pool.shape[2], d, topk,
                                     ptr(sparse_map), ptr(lut), stream_ptr(q_pool.device)), "sla_block_map")
    return sparse_map, lut


sla_block_map = _op("sla_block_map(Tensor q_pool, Tensor k_pool, int topk) -> (Tensor, Tensor)", _block_map_cuda,
                    _block_map_fake)


def _moments_fake(k, v, feature):
    b, l, h, d = k.shape
    return torch.empty(b * h * d * (d + 1), dtype=torch.float32, device=k.device)


def _moments_cuda(k, v, feature):
    """kv [B,H,D,D] followed by ksum [B,H,D] in one flat fp32 buffer, zero-filled once: the kernel accumulates into both."""
    b, l, h, d = k.shape
    buf = torch.zeros(b * h * d * (d + 1), dtype=torch.float32, device=k.device)
    check(lib().tdb200_sla_linear_moments(ptr(k), ptr(v), DTYPE_TAG[k.dtype], b, l, h, d, feature, ptr(buf),
                                          ptr(buf) + 4 * b * h * d * d, stream_ptr(k.device)), "sla_linear_moments")
    return buf


sla_linear_moments = _op("sla_linear_moments(Tensor k, Tensor v, int feature) -> Tensor", _moments_cuda, _moments_fake)


def _project_fake(w, kv, dtype):
    return torch.empty(kv.shape, dtype=dtype, device=kv.device)


def _project_cuda(w, kv, dtype):
    b, h, d, _ = kv.shape
    out = _project_fake(w, kv, dtype)
    check(lib().tdb200_sla_project_moments(ptr(w), ptr(kv), DTYPE_TAG[dtype], b * h, d, ptr(out), stream_ptr(kv.device)),
          "sla_project_moments")
    return out


sla_project_moments = _op("sla_project_moments(Tensor w, Tensor kv, ScalarType dtype) -> Tensor", _project_cuda, _project_fake)


def _attn_fwd_cuda(q_i8, q_scale, k_i8, k_scale, v, q, lut, topk, kvw, ksum, proj_b, sm_scale, lk, feature, blkq, blkk,
                   k_seq_major):
    b, l, h, d = q.shape
    out = _like(q)
    check(lib().tdb200_sla_attn_fwd(ptr(q_i8), ptr(q_scale), ptr(k_i8), ptr(k_scale), ptr(v), ptr(q), DTYPE_TAG[q.dtype], ptr(lut),
                                    topk, ptr(kvw), ptr(ksum), ptr(proj_b), ptr(out), b, l, lk, h, d, sm_scale, feature, blkq, blkk,
                                    int(k_seq_major), stream_ptr(q.device)), "sla_attn_fwd")
    return out


sla_attn_fwd = _op("sla_attn_fwd(Tensor q_i8, Tensor q_scale, Tensor k_i8, Tensor k_scale, Tensor v, Tensor q, Tensor lut, "
                   "int topk, Tensor kvw, Tensor ksum, Tensor proj_b, float sm_scale, int lk, int feature, int blkq, int blkk, "
                   "bool k_seq_major) -> Tensor", _attn_fwd_cuda, lambda q_i8, q_scale, k_i8, k_scale, v, q, *rest: _like(q))

BLKK16 = 64   # key block of the 16-bit attention kernels (query blocks: 128 or 64 rows)


def _attn16_fwd_cuda(q, k, v, lut, topk, kvw, ksum, proj_b, sm_scale, lk, feature, blkq):
    b, l, h, d = q.shape
    out = _like(q)
    check(lib().tdb200_sla_attn16_fwd(ptr(q), ptr(k), ptr(v), DTYPE_TAG[q.dtype], ptr(lut), topk, ptr(kvw), ptr(ksum), ptr(proj_b),
                                      ptr(out), b, l, lk, h, d, sm_scale, feature, blkq, BLKK16, stream_ptr(q.device)),
          "sla_attn16_fwd")
    return out


sla_attn16_fwd = _op("sla_attn16_fwd(Tensor q, Tensor k, Tensor v, Tensor lut, int topk, Tensor kvw, Tensor ksum, "
                     "Tensor proj_b, float sm_scale, int lk, int feature, int blkq) -> Tensor", _attn16_fwd_cuda,
                     lambda q, *rest: _like(q))


def _attn16_lse_fake(q, k, v, lut, topk, sm_scale, blkq):
    b, l, h, d = q.shape
    return _like(q), torch.empty(b, h, l, dtype=torch.float32, device=q.device)


def _attn16_lse_cuda(q, k, v, lut, topk, sm_scale, blkq):
    b, l, h, d = q.shape
    o_s, lse = _attn16_lse_fake(q, k, v, lut, topk, sm_scale, blkq)
    check(lib().tdb200_sla_attn16_fwd_lse(ptr(q), ptr(k), ptr(v), DTYPE_TAG[q.dtype], ptr(lut), topk, ptr(o_s), ptr(lse), b, l, h,
                                          d, sm_scale, blkq, BLKK16, stream_ptr(q.device)), "sla_attn16_fwd_lse")
    return o_s, lse


sla_attn16_fwd_lse = _op("sla_attn16_fwd_lse(Tensor q, Tensor k, Tensor v, Tensor lut, int topk, float sm_scale, int blkq) "
                         "-> (Tensor, Tensor)", _attn16_lse_cuda, _attn16_lse_fake)


def _attn16_bwd_cuda(q, k, v, o_s, d_o, lse, lut, topk, sm_scale, blkq):
    b, l, h, d = q.shape
    dq, dk, dv = _like(q), _like(q), _like(q)
    nbytes = lib().tdb200_sla_attn16_bwd_workspace_bytes(b, h, l, topk, blkq)
    check(0 if nbytes >= 0 else nbytes, "sla_attn16_bwd_workspace_bytes", launches=0)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=q.device)
    check(lib().tdb200_sla_attn16_bwd(ptr(q), ptr(k), ptr(v), ptr(o_s), ptr(d_o), ptr(lse), DTYPE_TAG[q.dtype], ptr(lut), topk,
                                      ptr(dq), ptr(dk), ptr(dv), ptr(ws), nbytes, b, l, h, d, sm_scale, blkq, BLKK16,
                                      stream_ptr(q.device)), "sla_attn16_bwd")
    return dq, dk, dv


sla_attn16_bwd = _op("sla_attn16_bwd(Tensor q, Tensor k, Tensor v, Tensor o_s, Tensor d_o, Tensor lse, Tensor lut, int topk, "
                     "float sm_scale, int blkq) -> (Tensor, Tensor, Tensor)", _attn16_bwd_cuda,
                     lambda q, *rest: (_like(q), _like(q), _like(q)))


def _attn16_setup_context(ctx, inputs, output):
    q, k, v, lut, topk, sm_scale, blkq = inputs
    o_s, lse = output
    ctx.save_for_backward(q, k, v, o_s, lse, lut)
    ctx.topk, ctx.sm_scale, ctx.blkq = topk, sm_scale, blkq


def _attn16_backward(ctx, d_o, d_lse):
    """Gradients of o_s in q, k, v; lse is a by-product (row statistics for the backward), not differentiated."""
    q, k, v, o_s, lse, lut = ctx.saved_tensors
    dq, dk, dv = sla_attn16_bwd(q, k, v, o_s, d_o.to(q.dtype).contiguous(), lse, lut, ctx.topk, ctx.sm_scale, ctx.blkq)
    return dq, dk, dv, None, None, None, None


torch.library.register_autograd("tdb200::sla_attn16_fwd_lse", _attn16_backward, setup_context=_attn16_setup_context, lib=LIB)


# ------------------------------------------------------------------------------------------------ SLA linear branch (training)
# In a namespace of their own: the tdb200:: set is the one tests/test_compile_host.py pairs one-to-one with its fake-kernel
# cases; these two have theirs in tests/test_sla_linear_branch_host.py.
LIB_LINEAR = torch.library.Library("tdb200_linear", "DEF")
def _linear_fwd_fake(q, k, v, w, bias, feature):
    return _like(q), _moments_fake(k, v, feature)


def _linear_fwd_cuda(q, k, v, w, bias, feature):
    """(o_l, the moments buffer of sla_linear_moments): the buffer (kv, ksum) is what the backward reads."""
    b, l, h, d = q.shape
    mom = _moments_cuda(k, v, feature)
    o_l = _like(q)
    check(lib().tdb200_sla_linear_fwd(ptr(q), ptr(mom), ptr(mom) + 4 * b * h * d * d, ptr(w), ptr(bias), DTYPE_TAG[q.dtype],
                                      feature, ptr(o_l), b, l, h, d, stream_ptr(q.device)), "sla_linear_fwd")
    return o_l, mom


sla_linear_fwd = _op("sla_linear_fwd(Tensor q, Tensor k, Tensor v, Tensor w, Tensor bias, int feature) -> (Tensor, Tensor)",
                     _linear_fwd_cuda, _linear_fwd_fake, LIB_LINEAR, "tdb200_linear")


def _linear_bwd_fake(q, k, v, d_o, mom, w, feature):
    return _like(q), _like(q), _like(q), _like(w), _like(w, shape=(w.shape[0],))


def _linear_bwd_cuda(q, k, v, d_o, mom, w, feature):
    b, l, h, d = q.shape
    dq, dk, dv, dw, db = _linear_bwd_fake(q, k, v, d_o, mom, w, feature)
    nbytes = lib().tdb200_sla_linear_bwd_workspace_bytes(b, h, l, d)
    check(0 if nbytes >= 0 else nbytes, "sla_linear_bwd_workspace_bytes", launches=0)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=q.device)
    check(lib().tdb200_sla_linear_bwd(ptr(q), ptr(k), ptr(v), ptr(d_o), ptr(mom), ptr(mom) + 4 * b * h * d * d, ptr(w),
                                      DTYPE_TAG[q.dtype], feature, ptr(dq), ptr(dk), ptr(dv), ptr(dw), ptr(db), ptr(ws), nbytes,
                                      b, l, h, d, stream_ptr(q.device)), "sla_linear_bwd")
    return dq, dk, dv, dw, db


sla_linear_bwd = _op("sla_linear_bwd(Tensor q, Tensor k, Tensor v, Tensor d_o, Tensor mom, Tensor w, int feature) "
                     "-> (Tensor, Tensor, Tensor, Tensor, Tensor)", _linear_bwd_cuda, _linear_bwd_fake, LIB_LINEAR,
                     "tdb200_linear")


def _linear_tangent_cuda(q, k, v, q_t, k_t, v_t, mom, w, feature):
    b, l, h, d = q.shape
    o_t = _like(q)
    nbytes = lib().tdb200_sla_linear_tangent_workspace_bytes(b, h, l, d)
    check(0 if nbytes >= 0 else nbytes, "sla_linear_tangent_workspace_bytes", launches=0)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=q.device)
    check(lib().tdb200_sla_linear_tangent(ptr(q), ptr(k), ptr(v), ptr(q_t), ptr(k_t), ptr(v_t), ptr(mom),
                                          ptr(mom) + 4 * b * h * d * d, ptr(w), DTYPE_TAG[q.dtype], feature, ptr(o_t), ptr(ws),
                                          nbytes, b, l, h, d, stream_ptr(q.device)), "sla_linear_tangent")
    return o_t


sla_linear_tangent = _op("sla_linear_tangent(Tensor q, Tensor k, Tensor v, Tensor q_t, Tensor k_t, Tensor v_t, Tensor mom, "
                         "Tensor w, int feature) -> Tensor", _linear_tangent_cuda, lambda q, *rest: _like(q), LIB_LINEAR,
                         "tdb200_linear")


def _linear_setup_context(ctx, inputs, output):
    q, k, v, w, bias, feature = inputs
    ctx.save_for_backward(q, k, v, w, output[1])
    ctx.feature = feature


def _linear_backward(ctx, d_o, d_mom):
    """Gradients of o_l in q, k, v, proj_w and proj_b; the moments buffer is a by-product, not differentiated."""
    q, k, v, w, mom = ctx.saved_tensors
    dq, dk, dv, dw, db = sla_linear_bwd(q, k, v, d_o.to(q.dtype).contiguous(), mom, w, ctx.feature)
    return dq, dk, dv, dw, db, None


torch.library.register_autograd("tdb200_linear::sla_linear_fwd", _linear_backward, setup_context=_linear_setup_context,
                                lib=LIB_LINEAR)


# ------------------------------------------------------------------------------------------------ SageSLA with FP8 P.V
# In a namespace of their own, like tdb200_linear::; their fake-kernel cases are in tests/test_sla_fp8_pv_host.py.
LIB_FP8 = torch.library.Library("tdb200_fp8", "DEF")


def _quant_v_fp8_fake(v, lk, blkk):
    b, _, h, d = v.shape
    return (torch.empty(b, h, d, _cdiv(lk, blkk) * blkk, dtype=torch.uint8, device=v.device),
            torch.empty(b, h, d, dtype=torch.float32, device=v.device))


def _quant_v_fp8_cuda(v, lk, blkk):
    b, _, h, d = v.shape
    v_fp8, v_scale = _quant_v_fp8_fake(v, lk, blkk)
    check(lib().tdb200_sla_quant_v_fp8(ptr(v), DTYPE_TAG[v.dtype], b, lk, h, d, blkk, ptr(v_fp8), ptr(v_scale),
                                       stream_ptr(v.device)), "sla_quant_v_fp8")
    return v_fp8, v_scale


sla_quant_v_fp8 = _op("sla_quant_v_fp8(Tensor v, int lk, int blkk) -> (Tensor, Tensor)", _quant_v_fp8_cuda, _quant_v_fp8_fake,
                      LIB_FP8, "tdb200_fp8")


def _attn_fwd_fp8v_cuda(q_i8, q_scale, k_i8, k_scale, v_fp8, v_scale, q, lut, topk, kvw, ksum, proj_b, sm_scale, lk, feature,
                        blkq, blkk, k_seq_major):
    b, l, h, d = q.shape
    out = _like(q)
    check(lib().tdb200_sla_attn_fwd_fp8v(ptr(q_i8), ptr(q_scale), ptr(k_i8), ptr(k_scale), ptr(v_fp8), ptr(v_scale), ptr(q),
                                         DTYPE_TAG[q.dtype], ptr(lut), topk, ptr(kvw), ptr(ksum), ptr(proj_b), ptr(out), b, l, lk, h,
                                         d, sm_scale, feature, blkq, blkk, int(k_seq_major), stream_ptr(q.device)),
          "sla_attn_fwd_fp8v")
    return out


sla_attn_fwd_fp8v = _op("sla_attn_fwd_fp8v(Tensor q_i8, Tensor q_scale, Tensor k_i8, Tensor k_scale, Tensor v_fp8, "
                        "Tensor v_scale, Tensor q, Tensor lut, int topk, Tensor kvw, Tensor ksum, Tensor proj_b, float sm_scale, "
                        "int lk, int feature, int blkq, int blkk, bool k_seq_major) -> Tensor", _attn_fwd_fp8v_cuda,
                        lambda q_i8, q_scale, k_i8, k_scale, v_fp8, v_scale, q, *rest: _like(q), LIB_FP8, "tdb200_fp8")
