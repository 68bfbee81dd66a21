"""ctypes binding of libtdb200.so (the C ABI declared in include/tdb200.h).

The product path has NO fallback: if the library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_void_p

import torch
import torch.autograd.forward_ad as fwAD

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG_DIR, "libtdb200.so")
if os.environ.get("TDB200_LIB"):   # kernel-variant experiments: a differently compiled build of the same ABI
    LIB_PATH = os.environ["TDB200_LIB"]

DTYPE_TAG = {torch.bfloat16: 0, torch.float16: 1}

_P, _I64, _F, _I = c_void_p, c_int64, c_float, c_int

# name -> argtypes (restype is int unless listed in _RESTYPES)
_PROTOS = {
    "tdb200_abi_version": [],
    "tdb200_last_error": [],
    "tdb200_quant_int8_block128": [_P, _I, _I64, _I64, _P, _P, _P],
    "tdb200_gelu_quant_int8_block128": [_P, _I, _I64, _I64, _P, _P, _P],
    "tdb200_gemm_w8a8": [_P, _P, _P, _P, _P, _P, _I, _I64, _I64, _I64, _P],
    "tdb200_gemm_w8a8_ex": [_P, _P, _P, _P, _P, _P, _I, _I64, _I64, _I64, _I, _P],
    "tdb200_gemm_w8a8_split": [_P, _P, _P, _P, _P, _P, _I, _I64, _I64, _I64, _I64, _P],
    "tdb200_gemm_w8a8_quant_out": [_P, _P, _P, _P, _P, _P, _P, _I, _I64, _I64, _I64, _I, _P],
    "tdb200_rms_norm_f32": [_P, _P, _P, _I64, _I64, _F, _P],
    "tdb200_layer_norm_f32": [_P, _P, _P, _P, _I64, _I64, _F, _P],
    "tdb200_rms_norm": [_P, _I, _P, _P, _I64, _I64, _F, _P],
    "tdb200_layer_norm": [_P, _I, _P, _P, _P, _I64, _I64, _F, _P],
    "tdb200_layer_norm_modulate": [_P, _I, _P, _P, _P, _I64, _I64, _F, _P],
    "tdb200_layer_norm_modulate_quant": [_P, _I, _P, _P, _P, _P, _P, _I64, _I64, _F, _P],
    "tdb200_gate_residual": [_P, _P, _P, _P, _I, _I64, _I64, _P],
    "tdb200_gate_residual_stats": [_P, _P, _P, _P, _P, _I, _I64, _I64, _F, _P],
    "tdb200_layer_norm_modulate_quant_stats": [_P, _I, _P, _P, _P, _P, _P, _I64, _I64, _P],
    "tdb200_rope_interleaved": [_P, _I, _P, _P, _I64, _I64, _I64, _P],
    "tdb200_rms_norm_rope": [_P, _I, _P, _P, _P, _I64, _I64, _I64, _F, _P],
    "tdb200_rms_norm_rope_table": [_P, _I, _P, _P, _P, _I64, _I64, _I64, _F, _P],
    "tdb200_sla_quant_qk": [_P, _P, _I, _I64, _I64, _I64, _I64, _I64, _P, _P, _P, _P, _P, _P, _P, _I64, _I64, _P],
    "tdb200_sla_block_map": [_P, _P, _I, _I64, _I64, _I64, _I64, _I64, _I64, _P, _P, _P],
    "tdb200_sla_linear_moments": [_P, _P, _I, _I64, _I64, _I64, _I64, _I, _P, _P, _P],
    "tdb200_sla_attn_fwd": [_P, _P, _P, _P, _P, _P, _I, _P, _I64, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _F,
                            _I, _I64, _I64, _I, _P],
    "tdb200_sla_quant_v_fp8": [_P, _I, _I64, _I64, _I64, _I64, _I64, _P, _P, _P],
    "tdb200_sla_attn_fwd_fp8v": [_P, _P, _P, _P, _P, _P, _P, _I, _P, _I64, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _F,
                                 _I, _I64, _I64, _I, _P],
    "tdb200_sla_project_moments": [_P, _P, _I, _I64, _I64, _P, _P],
    "tdb200_sla_linear_fwd": [_P, _P, _P, _P, _P, _I, _I, _P, _I64, _I64, _I64, _I64, _P],
    "tdb200_sla_linear_bwd": [_P, _P, _P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _P],
    "tdb200_sla_linear_bwd_workspace_bytes": [_I64, _I64, _I64, _I64],
    "tdb200_sla_linear_tangent": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _P, _P, _I64, _I64, _I64, _I64, _I64, _P],
    "tdb200_sla_linear_tangent_workspace_bytes": [_I64, _I64, _I64, _I64],
    "tdb200_sla_kmean_partial": [_P, _I, _I64, _I64, _I64, _I64, _P, _P],
    "tdb200_sla_kmean_final": [_P, _I64, _I64, _I64, _I64, _I64, _P, _P],
    "tdb200_sla_quant_k_seq": [_P, _P, _I, _I64, _I64, _I64, _I64, _P, _P, _P, _I64, _P],
    "tdb200_sla_attn_fwd_qk16": [_P, _P, _P, _I, _P, _I64, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _F, _P],
    "tdb200_sla_attn_fwd_qk16_lse": [_P, _P, _P, _I, _P, _I64, _P, _P, _I64, _I64, _I64, _I64, _F, _P],
    "tdb200_sla_attn_bwd_qk16": [_P, _P, _P, _P, _P, _P, _I, _P, _I64, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _F, _P],
    "tdb200_sla_attn_bwd_workspace_bytes": [_I64, _I64, _I64, _I64],
    "tdb200_sla_attn16_fwd": [_P, _P, _P, _I, _P, _I64, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _F, _I, _I64, _I64, _P],
    "tdb200_sla_attn16_fwd_lse": [_P, _P, _P, _I, _P, _I64, _P, _P, _I64, _I64, _I64, _I64, _F, _I64, _I64, _P],
    "tdb200_sla_attn16_bwd": [_P, _P, _P, _P, _P, _P, _I, _P, _I64, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _F, _I64, _I64,
                              _P],
    "tdb200_sla_attn16_bwd_workspace_bytes": [_I64, _I64, _I64, _I64, _I64],
    "tdb200_attn_dense_fwd": [_P, _P, _P, _I, _P, _I64, _I64, _I64, _I64, _I64, _F, _P],
    "tdb200_attn_dense_jvp": [_P, _P, _P, _P, _P, _P, _I, _P, _P, _I64, _I64, _I64, _I64, _I64, _F, _P],
    "tdb200_attn_dense_fwd_lse": [_P, _P, _P, _I, _P, _P, _I64, _I64, _I64, _I64, _I64, _F, _P],
    "tdb200_attn_dense_jvp_lse": [_P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _F, _P],
    "tdb200_attn_dense_bwd": [_P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _I64, _F, _P],
    "tdb200_attn_dense_bwd_workspace_bytes": [_I64, _I64, _I64],
    "tdb200_sla_attn16_jvp": [_P, _P, _P, _P, _P, _P, _I, _P, _I64, _P, _P, _I64, _I64, _I64, _I64, _F, _I64, _I64, _P],
    "tdb200_sla_attn16_jvp_lse": [_P, _P, _P, _P, _P, _P, _I, _P, _I64, _P, _P, _P, _I64, _I64, _I64, _I64, _F, _I64, _I64, _P],
    "tdb200_attn_dense_tangent": [_P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _I64, _I64, _I64, _I64, _I64, _F, _P],
    "tdb200_attn_dense_fwd_kl": [_P, _P, _P, _I, _P, _I64, _I64, _I64, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_fwd_lse_kl": [_P, _P, _P, _I, _P, _P, _I64, _I64, _I64, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_jvp_kl": [_P, _P, _P, _P, _P, _P, _I, _P, _P, _I64, _I64, _I64, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_jvp_lse_kl": [_P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _I64, _I64, _I64, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_tangent_kl": [_P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _I64, _I64, _I64, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_bwd_kl": [_P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_fwd_vl": [_P, _P, _P, _I, _P, _I64, _I64, _I64, _P, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_fwd_lse_vl": [_P, _P, _P, _I, _P, _P, _I64, _I64, _I64, _P, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_jvp_vl": [_P, _P, _P, _P, _P, _P, _I, _P, _P, _I64, _I64, _I64, _P, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_jvp_lse_vl": [_P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _I64, _I64, _I64, _P, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_tangent_vl": [_P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _I64, _I64, _I64, _P, _P, _I64, _I64, _F, _P],
    "tdb200_attn_dense_bwd_vl": [_P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _P, _P, _I64, _I64, _F, _P],
    "tdb200_sla_quant_qk_vl": [_P, _P, _I, _I64, _I64, _I64, _I64, _P, _P, _P, _P, _P, _P, _P, _P, _I64, _I64, _P],
    "tdb200_sla_block_map_vl": [_P, _P, _I, _I64, _I64, _I64, _I64, _I64, _I64, _P, _P, _I64, _I64, _P, _P, _P],
    "tdb200_sla_linear_moments_vl": [_P, _P, _I, _I64, _I64, _I64, _I64, _P, _I, _P, _P, _P],
    "tdb200_sla_attn_fwd_vl": [_P, _P, _P, _P, _P, _P, _I, _P, _I64, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _P, _P, _F, _I,
                               _I64, _I64, _P],
    "tdb200_sla_attn16_fwd_vl": [_P, _P, _P, _I, _P, _I64, _P, _P, _P, _P, _I64, _I64, _I64, _I64, _I64, _P, _P, _F, _I, _I64,
                                 _I64, _P],
    "tdb200_sla_attn16_tangent": [_P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _I64, _P, _I64, _I64, _I64, _I64, _F, _I64, _I64, _P],
    "tdb200_ltx_modulated_rms_norm_ada": [_P, _I, _P, _P, _I, _I, _I, _P, _I64, _I64, _I64, _I64, _F, _P],
    "tdb200_ltx_modulate_ada": [_P, _I, _P, _P, _I, _I, _I, _P, _I64, _I64, _I64, _I64, _P],
    "tdb200_ltx_gated_residual_ada": [_P, _P, _I, _P, _P, _I, _I, _P, _I64, _I64, _I64, _I64, _P],
    "tdb200_ltx_split_rope": [_P, _P, _P, _I, _P, _I64, _I64, _I64, _I64, _P],
    "tdb200_quant_int8_rowwise": [_P, _I, _I64, _I64, _P, _P, _P],
    "tdb200_gemm_w8a8_rowwise": [_P, _P, _P, _P, _P, _P, _I, _I64, _I64, _I64, _P],
}
_RESTYPES = {"tdb200_last_error": c_char_p, "tdb200_sla_attn_bwd_workspace_bytes": c_int64,
             "tdb200_sla_attn16_bwd_workspace_bytes": c_int64, "tdb200_attn_dense_bwd_workspace_bytes": c_int64,
             "tdb200_sla_linear_bwd_workspace_bytes": c_int64, "tdb200_sla_linear_tangent_workspace_bytes": c_int64}
ABI_VERSION = 2   # TDB200_ABI_VERSION of include/tdb200.h, whose prototypes _PROTOS mirrors

_lib = None


class Tdb200Error(RuntimeError):
    pass


def exported_names():
    return list(_PROTOS.keys())


def lib() -> ctypes.CDLL:
    """Load libtdb200.so (once).  Raises if it has not been built: there is no CPU or eager fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Tdb200Error(
                f"{LIB_PATH} not found. Build it with `python -m turbodiffusion_b200._build` "
                "(or __graft_entry__.build()). turbodiffusion_b200 has no fallback path.")
        handle = ctypes.CDLL(LIB_PATH)
        for name, argtypes in _PROTOS.items():
            fn = getattr(handle, name)  # AttributeError if the library does not export a declared symbol
            fn.argtypes = argtypes
            fn.restype = _RESTYPES.get(name, c_int)
        if handle.tdb200_abi_version() != ABI_VERSION:
            raise Tdb200Error("libtdb200.so ABI version mismatch")
        _lib = _DeviceGuarded(handle)
    return _lib


_CALL_DEVICE = None  # device index of the tensors of the call being assembled (set by stream_ptr)


class _DeviceGuarded:
    """The C side works on the CUDA runtime's *current* device (cudaGetDevice) with the stream handed in.  Every Python
    wrapper evaluates stream_ptr(tensor.device) while building its argument list; if that device is not the current one,
    the call is made under torch.cuda.device(...) so tensors on a non-current GPU work like they do for torch ops."""

    def __init__(self, handle):
        self._handle = handle
        self._cache = {}

    def __getattr__(self, name):
        fn = self._cache.get(name)
        if fn is None:
            raw = getattr(self._handle, name)

            def fn(*args, _raw=raw):
                global _CALL_DEVICE
                dev, _CALL_DEVICE = _CALL_DEVICE, None
                if dev is not None and dev != torch.cuda.current_device():
                    with torch.cuda.device(dev):
                        return _raw(*args)
                return _raw(*args)

            self._cache[name] = fn
        return fn


LAUNCHES = 0  # kernels launched through the C ABI (each entry point documents how many it enqueues)
_KERNELS_PER_CALL = {"sla_quant_qk": 4, "layernorm_modulate_quant": 2, "sla_attn16_bwd": 4, "attn_dense_bwd": 3, "attn_dense_bwd_kl": 3, "attn_dense_bwd_vl": 3,
                     "sla_linear_bwd": 8, "sla_linear_tangent": 5, "sla_quant_v_fp8": 4,
                     "sla_quant_qk_vl": 4}  # upper bounds per entry point


def check(rc: int, what: str, launches: int = None) -> None:
    global LAUNCHES
    LAUNCHES += _KERNELS_PER_CALL.get(what, 1) if launches is None else launches
    if rc != 0:
        msg = lib().tdb200_last_error()
        raise Tdb200Error(f"{what} failed (code {rc}): {msg.decode() if msg else ''}")


def stream_ptr(device=None) -> int:
    global _CALL_DEVICE
    if device is not None:
        dev = torch.device(device)
        _CALL_DEVICE = dev.index if dev.index is not None else torch.cuda.current_device()
    return torch.cuda.current_stream(device).cuda_stream


def ptr(t):
    return 0 if t is None else t.data_ptr()


def has_tangent(*tensors) -> bool:
    """Any of the tensors carries a forward-mode tangent: a dual tensor at the current torch.autograd.forward_ad level, or an
    input of torch.func.jvp (which runs on a forward_ad level of its own).  False while torch.compile traces."""
    if torch.compiler.is_compiling():
        return False
    return any(t is not None and fwAD.unpack_dual(t).tangent is not None for t in tensors)


def plain(t):
    """The tensor under any torch.func wrappers: the same values, with a data pointer for the C ABI.  A forward-AD rule's jvp
    sees its saved tensors and tangents wrapped at the torch.func.jvp level; it reads them through this, under
    torch._C._DisableFuncTorch() so that the tensors it allocates are plain as well."""
    while t is not None and torch._C._functorch.is_functorch_wrapped_tensor(t):
        t = torch._C._functorch.get_unwrapped(t)
    return t


def require_cuda(*tensors) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise Tdb200Error("turbodiffusion_b200 ops take CUDA tensors only (no CPU fallback)")
