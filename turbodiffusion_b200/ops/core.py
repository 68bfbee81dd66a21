"""Mirror of the reference operator API `turbodiffusion.ops` (turbodiffusion/ops/core.py), backed by libtdb200.so.

Same function / class names, constructor arguments, buffers and state-dict keys as the reference, so
`inference/modify_model.py:56-81` (replace_linear_norm) and checkpoints with `int8_weight / scale / bias` keys work
unchanged.  Additional fused entry points (one HBM pass instead of several) sit below the mirrored ones.
"""
from __future__ import annotations

import os
import weakref
from typing import Optional, Tuple

import torch
import torch.nn as nn

from .. import _ops
from .._lib import DTYPE_TAG, check, has_tangent, lib, plain, ptr, require_cuda, stream_ptr
from ..turbo_diffusion_ops import quant_cuda, gemm_cuda, gemm_cuda_swizzle_bias


# ------------------------------------------------------------------------------------------------ mirrored API
def int8_quant(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """ops/core.py:12-25."""
    return quant_cuda(x, None, None)


def int8_linear(x: torch.Tensor, w_q: torch.Tensor, w_s: torch.Tensor, bias: Optional[torch.Tensor] = None,
                **kwargs) -> torch.Tensor:
    """ops/core.py:28-57 (+ optional fused bias: T(T(acc)+bias), the value Int8Linear.forward :408-412 produces)."""
    assert w_q.dtype == torch.int8, "Weight tensor must be int8."
    shape = x.shape
    x = x.reshape(-1, shape[-1])
    if not x.is_contiguous():
        x = x.contiguous()
    m, n = x.shape[0], w_q.shape[0]
    y = torch.empty(m, n, dtype=x.dtype, device=x.device)  # the reference pre-zeroes (:53); every element is written here
    x_q, x_s = int8_quant(x)
    if bias is None:
        gemm_cuda(x_q, x_s, w_q, w_s, y)
    else:
        gemm_cuda_swizzle_bias(x_q, x_s, w_q, w_s, y, bias)
    return y.reshape(*shape[:-1], n)


def int8_linear_prequant(x_q: torch.Tensor, x_s: torch.Tensor, w_q: torch.Tensor, w_s: torch.Tensor,
                         bias: Optional[torch.Tensor], out_dtype: torch.dtype) -> torch.Tensor:
    """GEMM on an already-quantised activation (lets q/k/v share one quantisation of the same input)."""
    y = torch.empty(x_q.shape[0], w_q.shape[0], dtype=out_dtype, device=x_q.device)
    if bias is None:
        gemm_cuda(x_q, x_s, w_q, w_s, y)
    else:
        gemm_cuda_swizzle_bias(x_q, x_s, w_q, w_s, y, bias)
    return y


def _flatten_rows(x: torch.Tensor):
    assert x.is_contiguous(), "Input must be contiguous"
    assert x.dim() in (2, 3), "Input tensors must be batched (3D) or not batched (2D)"
    return x.reshape(-1, x.shape[-1])


def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    """ops/core.py:139-191: fp32 [M,N] or [B,M,N] in, fp32 out."""
    require_cuda(x, w)
    x2 = _flatten_rows(x)
    if x2.dtype != torch.float32:
        raise RuntimeError("rmsnorm expects an fp32 input (the module casts with x.float())")
    y = torch.empty_like(x2)
    _ops.rms_norm_f32(x2, w.float(), float(eps), y)
    return y.reshape(x.shape)


def layernorm(x, w, b, eps, elementwise_affine=True):
    """ops/core.py:380-386."""
    if elementwise_affine:
        assert w is not None and b is not None
    else:
        assert w is None and b is None
    require_cuda(x, w, b)
    x2 = _flatten_rows(x)
    if x2.dtype != torch.float32:
        raise RuntimeError("layernorm expects an fp32 input (the module casts with x.float())")
    y = torch.empty_like(x2)
    _ops.layer_norm_f32(x2, None if w is None else w.float(), None if b is None else b.float(), float(eps), y)
    return y.reshape(x.shape)


def cdiv(a: int, b: int):
    return (a + b - 1) // b


class Int8Linear(nn.Module):
    """ops/core.py:391-432.  Buffers: int8_weight [N,K] int8, scale [ceil(N/128), ceil(K/128)] fp32, bias [N]."""

    def __init__(self, in_features, out_features, bias=True, dtype=torch.bfloat16):
        super().__init__()
        self.in_features = in_features
        self.out_features = out_features
        row_blocks = cdiv(out_features, b=128)
        col_blocks = cdiv(in_features, b=128)
        self.register_buffer("int8_weight", torch.empty((out_features, in_features), dtype=torch.int8))
        self.register_buffer("scale", torch.empty((row_blocks, col_blocks), dtype=torch.float32))
        if bias:
            self.register_buffer("bias", torch.empty(out_features, dtype=dtype))
        else:
            self.bias = None

    def forward(self, x):
        # quant + wgmma GEMM with the bias add fused into the epilogue (same value as `out + self.bias`)
        return int8_linear(x, self.int8_weight, self.scale, self.bias)

    @classmethod
    def from_linear(cls, original_linear: nn.Linear, quantize: bool = True):
        int8_layer = cls(original_linear.in_features, original_linear.out_features,
                         bias=original_linear.bias is not None, dtype=original_linear.weight.dtype)
        if quantize:
            w_data = original_linear.weight.data.cuda()
            int8_w, scale = int8_quant(w_data.contiguous())
            int8_layer.int8_weight = int8_layer.int8_weight.to(int8_w.device)
            int8_layer.scale = int8_layer.scale.to(int8_w.device)
            int8_layer.int8_weight.copy_(int8_w)
            int8_layer.scale.copy_(scale)
            if original_linear.bias is not None:
                int8_layer.bias = int8_layer.bias.to(int8_w.device)
                int8_layer.bias.data.copy_(original_linear.bias.data.cuda())
        return int8_layer


class FastRMSNorm(nn.Module):
    """ops/core.py:434-452.  forward == rmsnorm(x.float(), w, eps).to(x.dtype), done in ONE pass for 16-bit x."""

    def __init__(self, dim: int, eps: float = 1e-5):
        super().__init__()
        self.dim = dim
        self.eps = eps
        self.register_buffer("weight", torch.ones(dim))

    def forward(self, x):
        return fast_rmsnorm(x, self.weight, self.eps)

    @classmethod
    def from_rmsnorm(cls, original_rmsnorm):
        layer = cls(dim=original_rmsnorm.dim, eps=original_rmsnorm.eps)
        if original_rmsnorm.weight.device != torch.device("meta"):
            layer.weight.data.copy_(original_rmsnorm.weight.float().data)
        return layer


class FastLayerNorm(nn.Module):
    """ops/core.py:454-491."""

    def __init__(self, dim: int, eps: float = 1e-5, elementwise_affine: bool = False, bias: bool = True):
        super().__init__()
        self.dim = dim
        self.eps = eps
        self.elementwise_affine = elementwise_affine
        if self.elementwise_affine:
            self.register_buffer("weight", torch.empty(self.dim))
            if bias:
                self.register_buffer("bias", torch.empty(self.dim))
            else:
                self.bias = None
        else:
            self.register_parameter("weight", None)
            self.register_parameter("bias", None)

    def forward(self, x):
        return fast_layernorm(x, self.weight, self.bias, self.eps)

    @classmethod
    def from_layernorm(cls, original_layernorm):
        layer = cls(dim=original_layernorm.normalized_shape[0], eps=original_layernorm.eps,
                    elementwise_affine=False if original_layernorm.weight is None else True,
                    bias=original_layernorm.bias is not None)
        if original_layernorm.weight is not None and original_layernorm.weight.device != torch.device("meta"):
            layer.weight.data.copy_(original_layernorm.weight.data)
        if original_layernorm.bias is not None and original_layernorm.bias.device != torch.device("meta"):
            layer.bias.data.copy_(original_layernorm.bias.data)
        return layer


# ------------------------------------------------------------------------------------------------ fused entry points
def _f32(t: Optional[torch.Tensor], n: int, what: str) -> Optional[torch.Tensor]:
    """Side inputs of the fused kernels (norm weights, modulation vectors, gates, angle tables) are read through raw fp32
    pointers.  Checkpoints loaded with load_state_dict(assign=True) keep the checkpoint dtype (often bf16), so coerce to
    contiguous fp32 here (a no-op for fp32 contiguous tensors) and check the element count."""
    if t is None:
        return None
    require_cuda(t)
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.float().contiguous()
    if t.numel() != n:
        raise ValueError(f"{what}: expected {n} elements, got {tuple(t.shape)}")
    return t


def _rows16(x: torch.Tensor):
    require_cuda(x)
    if x.dtype not in DTYPE_TAG:
        return None
    x2 = x.reshape(-1, x.shape[-1])
    if not x2.is_contiguous():
        x2 = x2.contiguous()
    return x2


def fast_rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    """FastRMSNorm.forward (ops/core.py:441-442) in one pass: T(float(x) * rstd * w)."""
    x2 = _rows16(x)
    if x2 is None:  # fp32 input: the reference entry point
        return rmsnorm(x.float().contiguous(), w, eps).to(x.dtype)
    if x2.numel() == 0:          # empty batch: nothing to launch (an empty tensor has no data pointer to hand to the C ABI)
        return torch.empty_like(x2).reshape(x.shape)
    w = _f32(w, x2.shape[1], "fast_rmsnorm weight")
    return _ops.rms_norm(x2, w, float(eps)).reshape(x.shape)


def fast_layernorm(x, w, b, eps) -> torch.Tensor:
    """FastLayerNorm.forward (ops/core.py:477-478) in one pass."""
    x2 = _rows16(x)
    if x2 is None:
        return layernorm(x.float().contiguous(), w, b, eps, w is not None).to(x.dtype)
    if x2.numel() == 0:
        return torch.empty_like(x2).reshape(x.shape)
    w, b = _f32(w, x2.shape[1], "fast_layernorm weight"), _f32(b, x2.shape[1], "fast_layernorm bias")
    return _ops.layer_norm(x2, w, b, float(eps)).reshape(x.shape)


def layernorm_modulate(x: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, eps: float) -> torch.Tensor:
    """(norm(x).float() * (1 + scale) + shift).type_as(x)  — rcm/networks/wan2pt1.py:404, scale/shift fp32 [dim]."""
    x2 = _rows16(x)
    assert x2 is not None, "layernorm_modulate expects a bf16/fp16 input"
    scale, shift = _f32(scale, x2.shape[1], "layernorm_modulate scale"), _f32(shift, x2.shape[1], "layernorm_modulate shift")
    return _ops.layer_norm_modulate(x2, scale, shift, float(eps)).reshape(x.shape)


def layernorm_modulate_quant(x: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, eps: float):
    """int8_quant(layernorm_modulate(x)) without materialising the 16-bit intermediate.  Returns (q, s)."""
    x2 = _rows16(x)
    assert x2 is not None
    m, n = x2.shape
    scale, shift = _f32(scale, n, "layernorm_modulate_quant scale"), _f32(shift, n, "layernorm_modulate_quant shift")
    return _ops.layer_norm_modulate_quant(x2, scale, shift, float(eps))


def gate_residual(x: torch.Tensor, y: torch.Tensor, gate: torch.Tensor) -> torch.Tensor:
    """x + y * gate.type_as(x)  — rcm/networks/wan2pt1.py:405-406, gate fp32 [dim]."""
    x2, y2 = _rows16(x), _rows16(y)
    gate = _f32(gate, x2.shape[1], "gate_residual gate")
    return _ops.gate_residual(x2, y2, gate).reshape(x.shape)


def gate_residual_stats(x: torch.Tensor, y: torch.Tensor, gate: Optional[torch.Tensor], eps: float):
    """(x + y * gate.type_as(x)  [gate None: x + y],  row statistics of that result for the next LayerNorm)."""
    x2, y2 = _rows16(x), _rows16(y)
    gate = _f32(gate, x2.shape[1], "gate_residual_stats gate")
    out, stats = _ops.gate_residual_stats(x2, y2, gate, float(eps))
    return out.reshape(x.shape), stats


def layernorm_modulate_quant_from_stats(x: torch.Tensor, stats: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor):
    """The tile pass of layernorm_modulate_quant with precomputed row statistics (from gate_residual_stats)."""
    x2 = _rows16(x)
    m, n = x2.shape
    scale, shift = _f32(scale, n, "layernorm_modulate_quant_from_stats scale"), _f32(shift, n, "layernorm_modulate_quant_from_stats shift")
    stats = _f32(stats, 2 * m, "layernorm_modulate_quant_from_stats stats")
    return _ops.layer_norm_modulate_quant_stats(x2, stats, scale, shift)


def rope_interleaved(x: torch.Tensor, angles: torch.Tensor) -> torch.Tensor:
    """rope_apply (wan2pt1.py:156-178).  x [..., L, H, D] with leading batch folded into L by the caller; angles [L, D/2]."""
    require_cuda(x, angles)
    l, h, d = x.shape[-3:]
    xc = x.contiguous()
    rows = xc.numel() // (h * d)
    assert rows == angles.shape[0], "one angle row per token row"
    angles = _f32(angles, rows * (d // 2), "rope_interleaved angles")
    return _ops.rope_interleaved(xc, angles)


_ROPE_TABLES = {}   # id(angles) -> (weakref to the angle tensor, its _version, (cos, sin) table [L, D/2, 2] fp32)
ROPE_TABLE = os.environ.get("TDB200_ROPE_TABLE", "1") != "0"   # "0": evaluate sin/cos inside the kernel (A/B timing)


def rope_cos_sin(angles: torch.Tensor) -> torch.Tensor:
    """(cos, sin) of an angle tensor [L, D/2] as one fp32 table [L, D/2, 2], built once per tensor (and per in-place version of
    it) and reused by every rmsnorm_rope call that is handed the same angles: all heads, q and k, every layer of a step.
    Under torch.compile the table is computed from the traced angles instead (the identity/version cache cannot be traced);
    the compiler folds the identical computations of one graph into one."""
    if torch.compiler.is_compiling():
        return _cos_sin(angles)
    key = id(angles)
    hit = _ROPE_TABLES.get(key)
    if hit is not None and hit[0]() is angles and hit[1] == angles._version:
        return hit[2]
    if len(_ROPE_TABLES) >= 16:
        _ROPE_TABLES.clear()
    table = _cos_sin(angles)
    _ROPE_TABLES[key] = (weakref.ref(angles), angles._version, table)
    return table


def _cos_sin(angles: torch.Tensor) -> torch.Tensor:
    a = angles.detach().float()
    return torch.stack((torch.cos(a), torch.sin(a)), dim=-1).contiguous()


def rmsnorm_rope(x: torch.Tensor, w: torch.Tensor, angles: torch.Tensor, eps: float, heads: int) -> torch.Tensor:
    """rope_apply(norm_q(x).view(L, H, D), freqs) in one pass; x [L, H*D]."""
    require_cuda(x, w, angles)
    xc = x.contiguous()
    l, hd = xc.shape
    w = _f32(w, hd, "rmsnorm_rope weight")
    if ROPE_TABLE:
        if angles.numel() != l * (hd // heads // 2):
            raise ValueError("rmsnorm_rope angles: expected [L, head_dim/2]")
        return _ops.rms_norm_rope_table(xc, w, rope_cos_sin(angles), float(eps), heads)
    angles = _f32(angles, l * (hd // heads // 2), "rmsnorm_rope angles")
    return _ops.rms_norm_rope(xc, w, angles, float(eps), heads)


def wan_rope_angles(t: int, h: int, w: int, head_dim: int, device=None) -> torch.Tensor:
    """Angle table [t*h*w, head_dim/2] fp32 of Wan's 3-D RoPE (VideoRopePosition3DEmb.generate_embeddings,
    rcm/networks/wan2pt1.py:111-137): bands d_h = d_w = 2*(head_dim//6), d_t = head_dim - 2*d_h, theta 10000."""
    dh = dw = head_dim // 6 * 2
    dt = head_dim - 2 * dh

    def freqs(dim):
        return 1.0 / (10000.0 ** (torch.arange(0, dim, 2)[: dim // 2].float() / dim))

    seq = torch.arange(max(t, h, w)).float()
    ft, fh, fw = torch.outer(seq[:t], freqs(dt)), torch.outer(seq[:h], freqs(dh)), torch.outer(seq[:w], freqs(dw))
    out = torch.cat([ft[:, None, None, :].expand(t, h, w, -1), fh[None, :, None, :].expand(t, h, w, -1),
                     fw[None, None, :, :].expand(t, h, w, -1)], dim=-1).reshape(t * h * w, head_dim // 2).float().contiguous()
    return out if device is None else out.to(device)


def _dense_args(what, q, k, v):
    if q.dim() != 4 or k.shape != v.shape or k.dim() != 4 or (q.shape[0], *q.shape[2:]) != (k.shape[0], *k.shape[2:]):
        raise ValueError(f"{what}: q [B, Lq, H, D] and k, v [B, Lk, H, D] expected, got {tuple(q.shape)}, "
                         f"{tuple(k.shape)}, {tuple(v.shape)}")
    return q.dtype if q.dtype in DTYPE_TAG else torch.bfloat16


def _lengths(what, lens, b: int, l: int, device, name: str, side: str, dim: str) -> Optional[torch.Tensor]:
    """A per-sample length argument of dense_attention / dense_attention_jvp (`name`: k_lens or q_lens, over the `side` rows,
    key or query, of length `dim` = l) as the int32 [b] device tensor the _kl / _vl entry points read, or None.  An integer [b]
    tensor holds the lengths; a boolean [b, l] padding mask (True = keep) is turned into them and refused unless each row is a
    run of Trues followed by Falses (for a CUDA mask that check synchronises once).  Lengths the caller hands in on the CPU are
    checked against [0, l]; CUDA lengths are not read on the host (no synchronisation): wider integer types are clamped to
    [0, l] on their device before they are narrowed to int32, and the kernels clamp int32 lengths to [0, l]."""
    if lens is None:
        return None
    if not isinstance(lens, torch.Tensor):
        raise TypeError(f"{what}: {name} must be a tensor, got {type(lens).__name__}")
    if lens.dtype == torch.bool:
        if tuple(lens.shape) != (b, l):
            raise ValueError(f"{what}: a boolean {name} is a {side}-padding mask [B, {dim}] = {(b, l)}, got {tuple(lens.shape)}")
        n = lens.sum(dim=1)
        if not torch.equal(torch.arange(l, device=lens.device) < n[:, None], lens):
            raise ValueError(f"{what}: the {side}-padding mask must keep a prefix of every row (Trues, then Falses)")
        lens = n
    elif lens.is_floating_point() or lens.is_complex() or tuple(lens.shape) != (b,):
        raise ValueError(f"{what}: {name} must be an integer tensor [B] = [{b}] or a boolean mask [B, {dim}], got "
                         f"{lens.dtype} {tuple(lens.shape)}")
    elif not lens.is_cuda and b and (int(lens.min()) < 0 or int(lens.max()) > l):
        raise ValueError(f"{what}: {name} {lens.tolist()} outside [0, {dim} = {l}]")
    if lens.dtype != torch.int32:   # widen, then clamp, then narrow: no length wraps around into [0, l]
        lens = lens.to(torch.int64).clamp(0, l)
    return lens.to(device=device, dtype=torch.int32).contiguous()


def _key_lens(what, k_lens, b: int, lk: int, device) -> Optional[torch.Tensor]:
    """The k_lens argument (key lengths, or a [b, lk] key-padding mask) as _lengths returns it."""
    return _lengths(what, k_lens, b, lk, device, "k_lens", "key", "Lk")


def _query_lens(what, q_lens, b: int, lq: int, device) -> Optional[torch.Tensor]:
    """The q_lens argument (query lengths, or a [b, lq] query-padding mask) as _lengths returns it."""
    return _lengths(what, q_lens, b, lq, device, "q_lens", "query", "Lq")


def _seq_lens(what, q_lens, k_lens, b: int, lq: int, lk: int, device):
    """(q_lens, k_lens) as the entry points take them: (None, None) or (None, k) for the plain and _kl entry points, and with
    query lengths (q, k) for the _vl ones, k filled with lk when the caller gave query lengths only."""
    kl = _key_lens(what, k_lens, b, lk, device)
    ql = _query_lens(what, q_lens, b, lq, device)
    if ql is not None and kl is None:
        kl = torch.full((b,), lk, dtype=torch.int32, device=device)
    return ql, kl


def _needs_grad(*tensors) -> bool:
    """The training path's rule, the SLA modules' too: grad mode on and a primal input that requires grad."""
    return torch.is_grad_enabled() and any(t.requires_grad for t in tensors)


def _dense_fwd_lse(q, k, v, sm_scale, k_lens, q_lens):
    """(out, lse) of tdb200_attn_dense_fwd_lse, or with k_lens of tdb200_attn_dense_fwd_lse_kl, or with q_lens (and k_lens) of
    tdb200_attn_dense_fwd_lse_vl."""
    b, lq, h, d = q.shape
    out = torch.empty_like(q)
    lse = torch.empty(b, h, lq, dtype=torch.float32, device=q.device)
    if q_lens is not None:
        check(lib().tdb200_attn_dense_fwd_lse_vl(ptr(q), ptr(k), ptr(v), DTYPE_TAG[q.dtype], ptr(out), ptr(lse), b, lq, k.shape[1],
                                                 ptr(q_lens), ptr(k_lens), h, d, sm_scale, stream_ptr(q.device)),
              "attn_dense_fwd_lse_vl")
    elif k_lens is None:
        check(lib().tdb200_attn_dense_fwd_lse(ptr(q), ptr(k), ptr(v), DTYPE_TAG[q.dtype], ptr(out), ptr(lse), b, lq, k.shape[1], h, d,
                                              sm_scale, stream_ptr(q.device)), "attn_dense_fwd_lse")
    else:
        check(lib().tdb200_attn_dense_fwd_lse_kl(ptr(q), ptr(k), ptr(v), DTYPE_TAG[q.dtype], ptr(out), ptr(lse), b, lq, k.shape[1],
                                                 ptr(k_lens), h, d, sm_scale, stream_ptr(q.device)), "attn_dense_fwd_lse_kl")
    return out, lse


def _dense_bwd(ctx, d_out):
    """(dq, dk, dv) from tdb200_attn_dense_bwd (or, with the k_lens the forward saved, tdb200_attn_dense_bwd_kl, and with its
    q_lens tdb200_attn_dense_bwd_vl), for the tensors the lse forward saved."""
    q, k, v, out, lse, k_lens, q_lens = ctx.saved_tensors
    b, lq, h, d = q.shape
    lk = k.shape[1]
    d_out = d_out.to(q.dtype).contiguous()
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    nbytes = lib().tdb200_attn_dense_bwd_workspace_bytes(b, h, lq)
    check(0 if nbytes >= 0 else nbytes, "attn_dense_bwd_workspace_bytes", launches=0)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=q.device)
    if q_lens is not None:
        check(lib().tdb200_attn_dense_bwd_vl(ptr(q), ptr(k), ptr(v), ptr(out), ptr(d_out), ptr(lse), DTYPE_TAG[q.dtype], ptr(dq),
                                             ptr(dk), ptr(dv), ptr(ws), nbytes, b, lq, lk, ptr(q_lens), ptr(k_lens), h, d, ctx.sm_scale,
                                             stream_ptr(q.device)),
              "attn_dense_bwd_vl")
    elif k_lens is None:
        check(lib().tdb200_attn_dense_bwd(ptr(q), ptr(k), ptr(v), ptr(out), ptr(d_out), ptr(lse), DTYPE_TAG[q.dtype], ptr(dq), ptr(dk),
                                          ptr(dv), ptr(ws), nbytes, b, lq, lk, h, d, ctx.sm_scale, stream_ptr(q.device)),
              "attn_dense_bwd")
    else:
        check(lib().tdb200_attn_dense_bwd_kl(ptr(q), ptr(k), ptr(v), ptr(out), ptr(d_out), ptr(lse), DTYPE_TAG[q.dtype], ptr(dq),
                                             ptr(dk), ptr(dv), ptr(ws), nbytes, b, lq, lk, ptr(k_lens), h, d, ctx.sm_scale,
                                             stream_ptr(q.device)),
              "attn_dense_bwd_kl")
    return dq, dk, dv


class _DenseAttention(torch.autograd.Function):
    """dense_attention's training path on 16-bit contiguous q, k, v: the lse forward, and the dense backward.  k_lens and q_lens
    (int32 [b] on the device, or None) are not differentiable; with k_lens alone both run their _kl twins, with q_lens (and
    k_lens) their _vl twins."""

    @staticmethod
    def forward(ctx, q, k, v, sm_scale, k_lens, q_lens):
        out, lse = _dense_fwd_lse(q, k, v, sm_scale, k_lens, q_lens)
        ctx.save_for_backward(q, k, v, out, lse, k_lens, q_lens)
        ctx.sm_scale = sm_scale
        return out

    @staticmethod
    def backward(ctx, d_out):
        return (*_dense_bwd(ctx, d_out), None, None, None)


class _DenseAttentionJvp(torch.autograd.Function):
    """dense_attention_jvp's training path: out differentiable in q, k and v; out_t, and the tangents, carry no gradient."""

    @staticmethod
    def forward(ctx, q, k, v, q_t, k_t, v_t, sm_scale, k_lens, q_lens):
        b, lq, h, d = q.shape
        out, out_t = torch.empty_like(q), torch.empty_like(q)
        lse = torch.empty(b, h, lq, dtype=torch.float32, device=q.device)
        if q_lens is not None:
            check(lib().tdb200_attn_dense_jvp_lse_vl(ptr(q), ptr(k), ptr(v), ptr(q_t), ptr(k_t), ptr(v_t), DTYPE_TAG[q.dtype],
                                                     ptr(out), ptr(out_t), ptr(lse), b, lq, k.shape[1], ptr(q_lens), ptr(k_lens), h,
                                                     d, sm_scale, stream_ptr(q.device)),
                  "attn_dense_jvp_lse_vl")
        elif k_lens is None:
            check(lib().tdb200_attn_dense_jvp_lse(ptr(q), ptr(k), ptr(v), ptr(q_t), ptr(k_t), ptr(v_t), DTYPE_TAG[q.dtype], ptr(out),
                                                  ptr(out_t), ptr(lse), b, lq, k.shape[1], h, d, sm_scale, stream_ptr(q.device)),
                  "attn_dense_jvp_lse")
        else:
            check(lib().tdb200_attn_dense_jvp_lse_kl(ptr(q), ptr(k), ptr(v), ptr(q_t), ptr(k_t), ptr(v_t), DTYPE_TAG[q.dtype],
                                                     ptr(out), ptr(out_t), ptr(lse), b, lq, k.shape[1], ptr(k_lens), h, d, sm_scale,
                                                     stream_ptr(q.device)),
                  "attn_dense_jvp_lse_kl")
        ctx.mark_non_differentiable(out_t)
        ctx.set_materialize_grads(False)    # out_t's gradient is never used: no zero tensor for it
        ctx.save_for_backward(q, k, v, out, lse, k_lens, q_lens)
        ctx.sm_scale = sm_scale
        return out, out_t

    @staticmethod
    def backward(ctx, d_out, d_out_t):
        if d_out is None:
            return (None,) * 9
        return (*_dense_bwd(ctx, d_out), None, None, None, None, None, None)


class _DenseAttentionAD(torch.autograd.Function):
    """dense_attention with a forward-AD rule, for q, k, v of which one carries a tangent (torch.func.jvp, forward_ad): the lse
    forward once; jvp = tdb200_attn_dense_tangent from the saved out and lse (missing tangents are zeros); backward = the dense
    backward.  lse is an output only so that setup_context can save it.  The tangent carries no gradient."""

    @staticmethod
    def forward(q, k, v, sm_scale, k_lens, q_lens):
        return _dense_fwd_lse(q, k, v, sm_scale, k_lens, q_lens)

    @staticmethod
    def setup_context(ctx, inputs, output):
        q, k, v, sm_scale, k_lens, q_lens = inputs
        out, lse = output
        ctx.mark_non_differentiable(lse)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(q, k, v, out, lse, k_lens, q_lens)
        ctx.save_for_forward(q, k, v, out, lse, k_lens, q_lens)
        ctx.sm_scale = sm_scale

    @staticmethod
    def jvp(ctx, q_t, k_t, v_t, *_):
        with torch._C._DisableFuncTorch():
            q, k, v, out, lse, k_lens, q_lens = (plain(t) for t in ctx.saved_tensors)
            q_t, k_t, v_t = (torch.zeros_like(p) if t is None else plain(t).detach().to(p.dtype).contiguous()
                             for t, p in ((q_t, q), (k_t, k), (v_t, v)))
            b, lq, h, d = q.shape
            out_t = torch.empty_like(q)
            if q_lens is not None:
                check(lib().tdb200_attn_dense_tangent_vl(ptr(q), ptr(k), ptr(v), ptr(q_t), ptr(k_t), ptr(v_t), ptr(out), ptr(lse),
                                                         DTYPE_TAG[q.dtype], ptr(out_t), b, lq, k.shape[1], ptr(q_lens),
                                                         ptr(k_lens), h, d, ctx.sm_scale, stream_ptr(q.device)),
                      "attn_dense_tangent_vl")
            elif k_lens is None:
                check(lib().tdb200_attn_dense_tangent(ptr(q), ptr(k), ptr(v), ptr(q_t), ptr(k_t), ptr(v_t), ptr(out), ptr(lse),
                                                      DTYPE_TAG[q.dtype], ptr(out_t), b, lq, k.shape[1], h, d, ctx.sm_scale,
                                                      stream_ptr(q.device)), "attn_dense_tangent")
            else:
                check(lib().tdb200_attn_dense_tangent_kl(ptr(q), ptr(k), ptr(v), ptr(q_t), ptr(k_t), ptr(v_t), ptr(out), ptr(lse),
                                                         DTYPE_TAG[q.dtype], ptr(out_t), b, lq, k.shape[1], ptr(k_lens), h, d,
                                                         ctx.sm_scale, stream_ptr(q.device)), "attn_dense_tangent_kl")
        return out_t, None

    @staticmethod
    def backward(ctx, d_out, d_lse):
        if d_out is None:
            return None, None, None, None, None, None
        return (*_dense_bwd(ctx, d_out), None, None, None)


def dense_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, sm_scale: Optional[float] = None,
                    k_lens: Optional[torch.Tensor] = None, q_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(q.k^T * sm_scale).v per (batch, head), the reference's dense attention (rcm/utils/attention.py:120-167):
    q [B, Lq, H, D], k and v [B, Lk, H, D], D = 128, any Lq and Lk; returns [B, Lq, H, D] in q's dtype.  bf16 / fp16 inputs run
    in their own type, any other float type in bf16.  sm_scale defaults to D ** -0.5.  One kernel on the current stream
    (tdb200_attn_dense_fwd), the arithmetic of the 16-bit SLA kernel.  With grad enabled and any of q, k, v requiring grad the
    output is differentiable: the forward also stores the row lse (tdb200_attn_dense_fwd_lse, the same output bits) and the
    backward is tdb200_attn_dense_bwd.  Forward-mode AD (torch.func.jvp, torch.autograd.forward_ad): when any of q, k, v
    carries a tangent, the output carries out_t = dense_attention_jvp's tangent, computed by tdb200_attn_dense_tangent from the
    lse forward's out and lse, so the primal runs once and has these bits; out_t carries no gradient.  Not a `tdb200::`
    operator: eager use.

    k_lens: a key-padding mask, for a batch whose key sequences have different lengths (text prompts that tokenise to different
    lengths).  An integer tensor [B] on any device, batch entry i attending to keys 0 .. k_lens[i] - 1 of its own Lk, or a
    boolean mask [B, Lk] (True = keep) whose rows are a run of Trues followed by Falses.  Entry i then gets the bits of this
    operator called on entry i alone with k and v cut to their first k_lens[i] rows, in the forward, the backward and the
    tangent alike; the gradients of keys and values past k_lens[i] are zero, and an entry with no keys gets out = 0.  What the
    rows of k and v (and of their tangents) past k_lens[i] hold, inf and NaN included, does not reach any output: the kernels
    do not load whole key tiles past it, and zero the rows past it in the tile they do load.  Lengths on the CPU are checked
    against [0, Lk]; lengths on a CUDA device are used without a synchronisation, clamped to [0, Lk].

    q_lens: a query-padding mask, for self-attention over a padded batch (clips of different token counts packed to one Lq):
    an integer tensor [B] on any device, batch entry i owning query rows 0 .. q_lens[i] - 1 of its own Lq, or a boolean mask
    [B, Lq] (True = keep) whose rows keep a prefix; lengths are checked or clamped to [0, Lq] as k_lens are.  Entry i's rows
    below q_lens[i] get the bits of this operator called on entry i alone with q cut to those rows (and k, v cut by k_lens when
    given), in the forward, the backward and the tangent alike, and so do its key and value gradients; rows past q_lens[i] get
    out = 0 (and out_t = 0, and a zero gradient), and add nothing to the key and value gradients.  What the rows of q, of its
    tangent and of the output gradient past q_lens[i] hold, inf and NaN included, does not reach any output: query blocks wholly
    past it are not computed, and the backward zeroes the rows past it on chip in the block it loads.  With q_lens the calls
    run the _vl entry points (tdb200_attn_dense_fwd_vl and its twins), given k_lens filled with Lk when k_lens is None."""
    require_cuda(q, k, v)
    dtype = _dense_args("dense_attention", q, k, v)
    qc, kc, vc = (t.to(dtype).contiguous() for t in (q, k, v))
    b, lq, h, d = qc.shape
    sm_scale = float(d ** -0.5 if sm_scale is None else sm_scale)
    ql, kl = _seq_lens("dense_attention", q_lens, k_lens, b, lq, kc.shape[1], qc.device)
    if has_tangent(q, k, v):
        return _DenseAttentionAD.apply(qc, kc, vc, sm_scale, kl, ql)[0].to(q.dtype)
    if _needs_grad(q, k, v):
        return _DenseAttention.apply(qc, kc, vc, sm_scale, kl, ql).to(q.dtype)
    out = torch.empty_like(qc)
    if ql is not None:
        check(lib().tdb200_attn_dense_fwd_vl(ptr(qc), ptr(kc), ptr(vc), DTYPE_TAG[dtype], ptr(out), b, lq, kc.shape[1], ptr(ql),
                                             ptr(kl), h, d, sm_scale, stream_ptr(qc.device)),
              "attn_dense_fwd_vl")
    elif kl is None:
        check(lib().tdb200_attn_dense_fwd(ptr(qc), ptr(kc), ptr(vc), DTYPE_TAG[dtype], ptr(out), b, lq, kc.shape[1], h, d, sm_scale,
                                          stream_ptr(qc.device)),
              "attn_dense_fwd")
    else:
        check(lib().tdb200_attn_dense_fwd_kl(ptr(qc), ptr(kc), ptr(vc), DTYPE_TAG[dtype], ptr(out), b, lq, kc.shape[1], ptr(kl), h, d,
                                             sm_scale, stream_ptr(qc.device)),
              "attn_dense_fwd_kl")
    return out.to(q.dtype)


def dense_attention_jvp(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, q_t: torch.Tensor, k_t: torch.Tensor,
                        v_t: torch.Tensor, sm_scale: Optional[float] = None,
                        k_lens: Optional[torch.Tensor] = None,
                        q_lens: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """dense_attention(q, k, v) and its forward-mode derivative along the tangents (q_t, k_t, v_t), from one kernel
    (tdb200_attn_dense_jvp): (out, out_t) with out_t = sum_j P_j S_t,j v_j - (sum_j P_j S_t,j) out + P.v_t, S_t =
    sm_scale (q_t.k^T + q.k_t^T).  Shapes and dtype rules as dense_attention; each tangent has its primal's shape and runs in
    the primal's 16-bit type.  Both outputs are [B, Lq, H, D] in q's dtype.  With grad enabled and any of q, k, v requiring
    grad, out is differentiable in q, k and v (tdb200_attn_dense_jvp_lse, the same bits, then tdb200_attn_dense_bwd), as a
    consistency-distillation loss needs; out_t never carries a gradient (a stop-gradient target) and the tangents get none.
    k_lens: per-sample key lengths or a prefix key-padding mask, as for dense_attention (tdb200_attn_dense_jvp_kl).  q_lens:
    per-sample query lengths or a prefix query-padding mask, as for dense_attention (tdb200_attn_dense_jvp_vl); rows past
    q_lens[i] get out = out_t = 0.  Not a `tdb200::` operator: eager use."""
    require_cuda(q, k, v, q_t, k_t, v_t)
    dtype = _dense_args("dense_attention_jvp", q, k, v)
    for name, t, primal in (("q_t", q_t, q), ("k_t", k_t, k), ("v_t", v_t, v)):
        if t.shape != primal.shape:
            raise ValueError(f"dense_attention_jvp: {name} {tuple(t.shape)} must have its primal's shape {tuple(primal.shape)}")
    qc, kc, vc, qtc, ktc, vtc = (t.to(dtype).contiguous() for t in (q, k, v, q_t, k_t, v_t))
    b, lq, h, d = qc.shape
    sm_scale = float(d ** -0.5 if sm_scale is None else sm_scale)
    ql, kl = _seq_lens("dense_attention_jvp", q_lens, k_lens, b, lq, kc.shape[1], qc.device)
    if _needs_grad(q, k, v):
        out, out_t = _DenseAttentionJvp.apply(qc, kc, vc, qtc, ktc, vtc, sm_scale, kl, ql)
        return out.to(q.dtype), out_t.to(q.dtype)
    out, out_t = torch.empty_like(qc), torch.empty_like(qc)
    if ql is not None:
        check(lib().tdb200_attn_dense_jvp_vl(ptr(qc), ptr(kc), ptr(vc), ptr(qtc), ptr(ktc), ptr(vtc), DTYPE_TAG[dtype], ptr(out),
                                             ptr(out_t), b, lq, kc.shape[1], ptr(ql), ptr(kl), h, d, sm_scale, stream_ptr(qc.device)),
              "attn_dense_jvp_vl")
    elif kl is None:
        check(lib().tdb200_attn_dense_jvp(ptr(qc), ptr(kc), ptr(vc), ptr(qtc), ptr(ktc), ptr(vtc), DTYPE_TAG[dtype], ptr(out),
                                          ptr(out_t), b, lq, kc.shape[1], h, d, sm_scale, stream_ptr(qc.device)),
              "attn_dense_jvp")
    else:
        check(lib().tdb200_attn_dense_jvp_kl(ptr(qc), ptr(kc), ptr(vc), ptr(qtc), ptr(ktc), ptr(vtc), DTYPE_TAG[dtype], ptr(out),
                                             ptr(out_t), b, lq, kc.shape[1], ptr(kl), h, d, sm_scale, stream_ptr(qc.device)),
              "attn_dense_jvp_kl")
    return out.to(q.dtype), out_t.to(q.dtype)
