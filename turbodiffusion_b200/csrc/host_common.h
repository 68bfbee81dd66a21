// Host-side helpers shared by the C-ABI entry points: error reporting (never exit()),
// TMA tensor-map encoding via the driver entry point (no libcuda link dependency), device queries.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tdb200.h"

namespace tdb {

// Records a thread-local message retrievable through tdb200_last_error(); returns `code`.
int fail(int code, const char* fmt, ...);

// Converts a CUDA runtime error into TDB200_ERR_CUDA (+ message). Returns 0 on cudaSuccess.
int check_cuda(cudaError_t e, const char* what);

// Checks the last launch (cudaGetLastError) without synchronising.
int check_launch(const char* kernel_name);

// Number of SMs of the current device (cached per device).
int sm_count();

// Verifies the current device is compute capability 9.x; the kernels are sm_90a-only.
int require_sm90();

// Rank-2 tiled tensor map over a row-major [outer, inner] matrix of `elem_bytes`-sized elements.
// `row_stride_bytes` is the distance between consecutive outer indices (multiple of 16).
// Swizzle is always 128B: box_inner * elem_bytes must be <= 128.
int make_tmap_2d(CUtensorMap* out, const void* base, CUtensorMapDataType dtype, uint32_t elem_bytes, uint64_t inner,
                 uint64_t outer, uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer);

// Rank-4 tiled tensor map; dims/strides listed innermost first (strides for dims 1..3, in bytes).
// swizzle_bytes: 128 (default) or 64 (tiles whose rows are 64 bytes: int8 Q/K of 64-wide heads).
int make_tmap_4d(CUtensorMap* out, const void* base, CUtensorMapDataType dtype, uint32_t elem_bytes,
                 const uint64_t dims[4], const uint64_t strides_bytes[3], const uint32_t box[4], int swizzle_bytes = 128);

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per device (`done_per_device`: a static bool[64] owned by the
// caller, one per kernel instantiation, for kernels whose dynamic shared memory size is a compile-time constant).
int set_max_dynamic_smem_once(const void* func, size_t bytes, bool* done_per_device, const char* what);

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// The size checks the dense attention entry points share (dense_attn.cu, sla_attn_bwd.cu), messages prefixed with `what`.
// dense_attn_shape: non-positive b, lq, lk, h or d -> TDB200_ERR_INVALID_ARG.  dense_attn_limits: a bad dtype tag, d != 128,
// b or h above 65535 (grid y and z), lq or lk above 2^31 - 1 (int32 TMA coordinates), lq*h*d or lk*h*d of 2^39 elements or
// more (tensor-map strides below 2^40 bytes) -> TDB200_ERR_UNSUPPORTED.
int dense_attn_shape(const char* what, int64_t b, int64_t lq, int64_t lk, int64_t h, int64_t d);
int dense_attn_limits(const char* what, int dtype, int64_t b, int64_t lq, int64_t lk, int64_t h, int64_t d);

}  // namespace tdb
