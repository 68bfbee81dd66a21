// a1. Per-128x128-block symmetric INT8 quantisation (reference: turbodiffusion/ops/quant/quant.hpp:86-99,122-164;
// scale layout common/store.hpp:46).  HBM-bound: 2 B read + 1 B written per element.
//
// One CTA (256 threads) per 128x128 tile.  A warp-wide load instruction covers two full 256-byte row
// segments (lane -> 16-byte chunk), so every global access is a fully used 128-byte line; each thread keeps
// 8 independent 16-byte loads in flight (8 rows x 8 elements) before the first use.
#include "common.cuh"
#include "host_common.h"

namespace {

using namespace tdb;

constexpr int kBlk = 128;
constexpr int kThreads = 256;
constexpr int kRowsPerPass = kThreads / 16;      // 16 rows per pass (16 lanes x 16 B cover one 256-byte row segment)
constexpr int kPasses = kBlk / kRowsPerPass;     // 8

// kGelu: the input is the FFN's pre-activation; y = T(gelu_tanh(x)) (nn.GELU(approximate="tanh") on a 16-bit tensor: fp32
// math, one rounding, rcm/networks/wan2pt1.py:375) is quantised instead of x.  gelu_tanh(x) = x * sigmoid(2u),
// u = sqrt(2/pi)(x + 0.044715 x^3), evaluated as x / (1 + 2^z) with ex2.approx + rcp.approx (relative error ~2^-21 everywhere,
// including the negative tail where 1 + tanh(u) cancels).
template <typename T>
__global__ void __launch_bounds__(kThreads) quant_int8_block128_kernel(const T* __restrict__ x, int8_t* __restrict__ q,
                                                                       float* __restrict__ s, int64_t m, int64_t k,
                                                                       int k_blocks) {
  __shared__ float warp_amax[kThreads / 32];
  const int tid = threadIdx.x;
  const int blk_n = blockIdx.x, blk_m = blockIdx.y;
  const int col = blk_n * kBlk + (tid & 15) * 8;  // first of this thread's 8 consecutive columns
  const int row0 = blk_m * kBlk + (tid >> 4);
  const bool col_ok = col < k;  // k % 8 == 0, so a chunk is entirely in or out

  uint4 raw[kPasses];
#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    const int64_t row = row0 + p * kRowsPerPass;
    raw[p] = make_uint4(0u, 0u, 0u, 0u);
    if (col_ok && row < m) raw[p] = ldg_nc_v4(x + row * k + col);
  }

  float v[kPasses][8];
  float amax = 1e-8f;
#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    const uint32_t w[4] = {raw[p].x, raw[p].y, raw[p].z, raw[p].w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = F16Traits<T>::lo(w[j]), b = F16Traits<T>::hi(w[j]);
      v[p][2 * j] = a;
      v[p][2 * j + 1] = b;
      amax = fmaxf(amax, fmaxf(fabsf(a), fabsf(b)));
    }
  }
  amax = warp_max(amax);
  if ((tid & 31) == 0) warp_amax[tid >> 5] = amax;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) amax = fmaxf(amax, warp_amax[w]);

  const float r = __fdiv_rn(128.0f, amax);  // IEEE division: codes reproduce on any host (the reference's
                                            // --use_fast_math div.approx differs from this only at .5 ties)
  if (tid == 0) s[static_cast<int64_t>(blk_m) * k_blocks + blk_n] = amax * 0.0078125f;  // amax / 128, exact

#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    const int64_t row = row0 + p * kRowsPerPass;
    const uint32_t lo = pack4_s8_rne(__fmul_rn(v[p][0], r), __fmul_rn(v[p][1], r), __fmul_rn(v[p][2], r), __fmul_rn(v[p][3], r));
    const uint32_t hi = pack4_s8_rne(__fmul_rn(v[p][4], r), __fmul_rn(v[p][5], r), __fmul_rn(v[p][6], r), __fmul_rn(v[p][7], r));
    if (col_ok && row < m) *reinterpret_cast<uint2*>(q + row * k + col) = make_uint2(lo, hi);
  }
}


// ---- FFN activation + quantisation in one HBM pass:  (q, s) = quant_int8_block128( T( gelu_tanh(x) ) ) ----------------------
// gelu_tanh(x) = 0.5 x (1 + tanh(u)), u = sqrt(2/pi) (x + 0.044715 x^3) (nn.GELU(approximate="tanh"), rcm/networks/wan2pt1.py:375),
// tanh by MUFU (tanh.approx.f32, absolute error <= 2^-11): the same evaluation as the GEMM's fused quantised-output epilogue, whose
// int8 codes it reproduces; against torch's fp32 GELU the codes differ by one on ~1 % of the elements (the error is ~2 % of an
// int8 step).  The per-element work is kept to one MUFU tanh and a few FP32 multiply-adds (lane-wise f32x2 helpers of
// common.cuh, one FMUL/FFMA per lane on sm_90) plus packed bf16x2 max for the block amax, so that the kernel stays close to
// its 3 bytes of HBM traffic per element.
template <typename T>
__global__ void __launch_bounds__(kThreads) gelu_quant_int8_block128_kernel(const T* __restrict__ x, int8_t* __restrict__ q,
                                                                            float* __restrict__ s, int64_t m, int64_t k,
                                                                            int k_blocks) {
  __shared__ float warp_amax[kThreads / 32];
  const int tid = threadIdx.x;
  const int blk_n = blockIdx.x, blk_m = blockIdx.y;
  const int col = blk_n * kBlk + (tid & 15) * 8;
  const int row0 = blk_m * kBlk + (tid >> 4);
  const bool col_ok = col < k;

  uint4 raw[kPasses];
#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    const int64_t row = row0 + p * kRowsPerPass;
    raw[p] = make_uint4(0u, 0u, 0u, 0u);
    if (col_ok && row < m) raw[p] = ldg_nc_v4(x + row * k + col);
  }
  uint32_t g[kPasses][4];            // T( gelu(x) ), packed pairs
  uint32_t amax2 = 0u;               // running |.| maximum of both halves (16-bit lanes)
  const float2 c1 = make_float2(0.7978845608028654f, 0.7978845608028654f);
  const float2 c3 = make_float2(0.7978845608028654f * 0.044715f, 0.7978845608028654f * 0.044715f);
  const float2 half2v = make_float2(0.5f, 0.5f);
#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    const uint32_t w[4] = {raw[p].x, raw[p].y, raw[p].z, raw[p].w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 xv = make_float2(F16Traits<T>::lo(w[j]), F16Traits<T>::hi(w[j]));
      const float2 u = fmul2_rn(ffma2_rn(fmul2_rn(xv, xv), c3, c1), xv);
      float2 t;
      asm("tanh.approx.f32 %0, %1;" : "=f"(t.x) : "f"(u.x));
      asm("tanh.approx.f32 %0, %1;" : "=f"(t.y) : "f"(u.y));
      const float2 hx = fmul2_rn(xv, half2v);
      const float2 y = ffma2_rn(hx, t, hx);
      g[p][j] = F16Traits<T>::pack(y.x, y.y);
      amax2 = F16Traits<T>::absmax2(amax2, g[p][j]);
    }
  }
  float amax = fmaxf(1e-8f, fmaxf(F16Traits<T>::lo(amax2), F16Traits<T>::hi(amax2)));
  amax = warp_max(amax);
  if ((tid & 31) == 0) warp_amax[tid >> 5] = amax;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) amax = fmaxf(amax, warp_amax[w]);
  const float r = __fdiv_rn(128.0f, amax);
  if (tid == 0) s[static_cast<int64_t>(blk_m) * k_blocks + blk_n] = amax * 0.0078125f;
  const float2 r2 = make_float2(r, r);
#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    const int64_t row = row0 + p * kRowsPerPass;
    uint32_t word[2];
#pragma unroll
    for (int j = 0; j < 4; j += 2) {
      const float2 v0 = fmul2_rn(make_float2(F16Traits<T>::lo(g[p][j]), F16Traits<T>::hi(g[p][j])), r2);
      const float2 v1 = fmul2_rn(make_float2(F16Traits<T>::lo(g[p][j + 1]), F16Traits<T>::hi(g[p][j + 1])), r2);
      word[j >> 1] = pack4_s8_rne(v0.x, v0.y, v1.x, v1.y);
    }
    if (col_ok && row < m) *reinterpret_cast<uint2*>(q + row * k + col) = make_uint2(word[0], word[1]);
  }
}

}  // namespace

static int quant_impl(const void* x, int x_dtype, int64_t m, int64_t k, int8_t* q, float* s, bool gelu, void* stream) {
  using namespace tdb;
  if (!x || !q || !s) return fail(TDB200_ERR_INVALID_ARG, "quant_int8_block128: null pointer");
  if (m < 0 || k < 0) return fail(TDB200_ERR_INVALID_ARG, "quant_int8_block128: negative size");
  if (m == 0 || k == 0) return TDB200_OK;
  if (k % 8 != 0) return fail(TDB200_ERR_UNSUPPORTED, "quant_int8_block128: k=%lld must be a multiple of 8", (long long)k);
  if (!aligned16(x) || (reinterpret_cast<uintptr_t>(q) & 7u))
    return fail(TDB200_ERR_INVALID_ARG, "quant_int8_block128: x must be 16-byte and q 8-byte aligned");
  if (int rc = require_sm90()) return rc;
  const int64_t kb = cdiv64(k, kBlk), mb = cdiv64(m, kBlk);
  if (mb > 65535) return fail(TDB200_ERR_UNSUPPORTED, "quant_int8_block128: m too large (%lld)", (long long)m);
  dim3 grid(static_cast<unsigned>(kb), static_cast<unsigned>(mb));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (x_dtype == TDB200_DTYPE_BF16 && !gelu)
    quant_int8_block128_kernel<__nv_bfloat16>
        <<<grid, kThreads, 0, st>>>(static_cast<const __nv_bfloat16*>(x), q, s, m, k, static_cast<int>(kb));
  else if (x_dtype == TDB200_DTYPE_FP16 && !gelu)
    quant_int8_block128_kernel<__half><<<grid, kThreads, 0, st>>>(static_cast<const __half*>(x), q, s, m, k,
                                                                  static_cast<int>(kb));
  else if (x_dtype == TDB200_DTYPE_BF16)
    gelu_quant_int8_block128_kernel<__nv_bfloat16>
        <<<grid, kThreads, 0, st>>>(static_cast<const __nv_bfloat16*>(x), q, s, m, k, static_cast<int>(kb));
  else if (x_dtype == TDB200_DTYPE_FP16)
    gelu_quant_int8_block128_kernel<__half><<<grid, kThreads, 0, st>>>(static_cast<const __half*>(x), q, s, m, k,
                                                                       static_cast<int>(kb));
  else
    return fail(TDB200_ERR_UNSUPPORTED, "quant_int8_block128: dtype tag %d (only bf16/fp16, like quant.cu:64-67)", x_dtype);
  return check_launch("quant_int8_block128_kernel");
}

extern "C" int tdb200_quant_int8_block128(const void* x, int x_dtype, int64_t m, int64_t k, int8_t* q, float* s,
                                          void* stream) {
  return quant_impl(x, x_dtype, m, k, q, s, false, stream);
}

extern "C" int tdb200_gelu_quant_int8_block128(const void* x, int x_dtype, int64_t m, int64_t k, int8_t* q, float* s,
                                               void* stream) {
  return quant_impl(x, x_dtype, m, k, q, s, true, stream);
}
