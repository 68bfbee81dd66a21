// a12. LTX-2 (TurboT2AV) prologue variants: the `*_ada` fused row kernels and split-half RoPE.
//   semantics: TurboT2AV/LTX-2/packages/ltx-core/src/ltx_core/model/transformer/transformer.py:21-94
//     modulated_rms_norm_from_ada : rms_norm(x) * (1 + s) + t,  s/t = table[i] + timestep[b, tok, i, :]
//     modulate_from_ada           : x * (1 + s) + t
//     gated_residual_from_ada     : x + residual * g
//   rms_norm = F.rms_norm without weight (ltx_core/utils.py:7-12); split RoPE ltx_core/model/transformer/rope.py:42-60;
//   the reference's fast path are the Triton kernels in ltx_distillation/fast_norm_kernels.py:388-473 (fp32 math, one
//   rounding to the io dtype), which is what these kernels reproduce.  HBM-bound, one CTA per row, 16-byte accesses.
#include "common.cuh"
#include "host_common.h"

namespace {
using namespace tdb;

enum LtxOp { kModRms = 0, kModulate = 1, kGatedRes = 2 };

struct LtxParams {
  const void* x;
  const void* res;      // residual (kGatedRes)
  const float* table;   // [num_ada, n] fp32
  const void* ts;       // timestep [b, ts_tokens, num_ada*n] in T, ts_tokens == 1 (broadcast) or == tokens
  void* y;
  int64_t rows;         // b * tokens
  int tokens, ts_tokens, n, num_ada, idx0, idx1;
  float eps;
};

template <typename T, int kOp, int kThreads, int kChunks>
__global__ void __launch_bounds__(kThreads) ltx_row_kernel(LtxParams p) {
  __shared__ float red[kThreads / 32];
  const int64_t row = blockIdx.x;
  const int nchunks = p.n / 8;
  const int64_t b = row / p.tokens, tok = row % p.tokens;
  const T* xr = static_cast<const T*>(p.x) + row * p.n;
  const T* tsr = static_cast<const T*>(p.ts) + (b * p.ts_tokens + (p.ts_tokens == 1 ? 0 : tok)) * int64_t(p.num_ada) * p.n;
  uint4 raw[kChunks];
#pragma unroll
  for (int i = 0; i < kChunks; ++i) {
    const int c = threadIdx.x + i * kThreads;
    raw[i] = make_uint4(0u, 0u, 0u, 0u);
    if (c < nchunks) raw[i] = ldg_nc_v4(xr + c * 8);
  }
  float rstd = 1.0f;
  if (kOp == kModRms) {
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kChunks; ++i) {
      const uint32_t w[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float a = F16Traits<T>::lo(w[j]), c2 = F16Traits<T>::hi(w[j]);
        ss = fmaf(a, a, fmaf(c2, c2, ss));
      }
    }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];
    rstd = rsqrtf(t / static_cast<float>(p.n) + p.eps);
  }
  T* yr = static_cast<T*>(p.y) + row * p.n;
#pragma unroll
  for (int i = 0; i < kChunks; ++i) {
    const int c = threadIdx.x + i * kThreads;
    if (c >= nchunks) continue;
    const int col = c * 8;
    const uint32_t w[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
    float xf[8], a0[8], a1[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      xf[2 * j] = F16Traits<T>::lo(w[j]);
      xf[2 * j + 1] = F16Traits<T>::hi(w[j]);
    }
    auto ada = [&](int idx, float* out) {  // table[idx] + timestep[.., idx, :]
      const float4 t0 = __ldg(reinterpret_cast<const float4*>(p.table + int64_t(idx) * p.n + col));
      const float4 t1 = __ldg(reinterpret_cast<const float4*>(p.table + int64_t(idx) * p.n + col) + 1);
      const uint4 tv = ldg_nc_v4(tsr + int64_t(idx) * p.n + col);
      const uint32_t tw[4] = {tv.x, tv.y, tv.z, tv.w};
      const float tb[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        out[2 * j] = tb[2 * j] + F16Traits<T>::lo(tw[j]);
        out[2 * j + 1] = tb[2 * j + 1] + F16Traits<T>::hi(tw[j]);
      }
    };
    ada(p.idx0, a0);
    if (kOp != kGatedRes) ada(p.idx1, a1);
    float o[8];
    if (kOp == kGatedRes) {
      const uint4 rv = ldg_nc_v4(static_cast<const T*>(p.res) + row * p.n + col);
      const uint32_t rw[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        o[2 * j] = fmaf(F16Traits<T>::lo(rw[j]), a0[2 * j], xf[2 * j]);
        o[2 * j + 1] = fmaf(F16Traits<T>::hi(rw[j]), a0[2 * j + 1], xf[2 * j + 1]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = fmaf(xf[j] * rstd, 1.0f + a0[j], a1[j]);  // idx0 = scale, idx1 = shift
    }
    stg_v4(yr + col, make_uint4(F16Traits<T>::pack(o[0], o[1]), F16Traits<T>::pack(o[2], o[3]),
                                F16Traits<T>::pack(o[4], o[5]), F16Traits<T>::pack(o[6], o[7])));
  }
}

// split-half RoPE: x viewed [b, t, h, d]; cos/sin [b, h, t, d/2] fp32-or-T given as T; out[:d/2] = x1*c - x2*s, out[d/2:] = x2*c + x1*s
template <typename T>
__global__ void __launch_bounds__(256) ltx_split_rope_kernel(const T* __restrict__ x, const T* __restrict__ cs,
                                                             const T* __restrict__ sn, T* __restrict__ y, int64_t chunks,
                                                             int t, int h, int d) {
  const int half = d / 2, cph = half / 8;  // 16-byte chunks per half head
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t c = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; c < chunks; c += stride) {
    const int ci = static_cast<int>(c % cph);
    int64_t r = c / cph;
    const int hh = static_cast<int>(r % h);
    r /= h;
    const int tok = static_cast<int>(r % t);
    const int64_t b = r / t;
    const T* xp = x + ((b * t + tok) * h + hh) * d + ci * 8;
    const int64_t fo = ((b * h + hh) * t + tok) * half + ci * 8;
    const uint4 x1 = ldg_nc_v4(xp), x2 = ldg_nc_v4(xp + half), cv = ldg_nc_v4(cs + fo), sv = ldg_nc_v4(sn + fo);
    const uint32_t a[4] = {x1.x, x1.y, x1.z, x1.w}, bq[4] = {x2.x, x2.y, x2.z, x2.w};
    const uint32_t cw[4] = {cv.x, cv.y, cv.z, cv.w}, sw[4] = {sv.x, sv.y, sv.z, sv.w};
    uint32_t o1[4], o2[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a0 = F16Traits<T>::lo(a[j]), a1 = F16Traits<T>::hi(a[j]);
      const float b0 = F16Traits<T>::lo(bq[j]), b1 = F16Traits<T>::hi(bq[j]);
      const float c0 = F16Traits<T>::lo(cw[j]), c1 = F16Traits<T>::hi(cw[j]);
      const float s0 = F16Traits<T>::lo(sw[j]), s1 = F16Traits<T>::hi(sw[j]);
      o1[j] = F16Traits<T>::pack(fmaf(-s0, b0, a0 * c0), fmaf(-s1, b1, a1 * c1));
      o2[j] = F16Traits<T>::pack(fmaf(s0, a0, b0 * c0), fmaf(s1, a1, b1 * c1));
    }
    T* yp = y + ((b * t + tok) * h + hh) * d + ci * 8;
    stg_v4(yp, make_uint4(o1[0], o1[1], o1[2], o1[3]));
    stg_v4(yp + half, make_uint4(o2[0], o2[1], o2[2], o2[3]));
  }
}

template <typename T, int kOp>
int launch(const LtxParams& p, cudaStream_t st) {
  const int nchunks = p.n / 8;
  const unsigned grid = static_cast<unsigned>(p.rows);
#define TDB_L(TH, CH)                                        \
  ltx_row_kernel<T, kOp, TH, CH><<<grid, TH, 0, st>>>(p);    \
  return check_launch("ltx_row_kernel")
  if (nchunks <= 128) { TDB_L(128, 1); }
  if (nchunks <= 256) { TDB_L(128, 2); }
  if (nchunks <= 512) { TDB_L(256, 2); }
  if (nchunks <= 1024) { TDB_L(256, 4); }
  if (nchunks <= 2048) { TDB_L(256, 8); }
#undef TDB_L
  return fail(TDB200_ERR_UNSUPPORTED, "ltx row kernel: n=%d too large", p.n);
}

template <int kOp>
int run(const char* name, const void* x, const void* res, int dtype, const float* table, const void* ts, int idx0, int idx1,
        int num_ada, void* y, int64_t b, int64_t tokens, int64_t ts_tokens, int64_t n, float eps, void* stream) {
  if (!x || !table || !ts || !y || (kOp == kGatedRes && !res)) return fail(TDB200_ERR_INVALID_ARG, "%s: null pointer", name);
  if (b <= 0 || tokens <= 0 || n <= 0 || n % 8 != 0) return fail(TDB200_ERR_INVALID_ARG, "%s: bad shape (n %% 8 == 0)", name);
  if (ts_tokens != 1 && ts_tokens != tokens) return fail(TDB200_ERR_INVALID_ARG, "%s: timestep tokens must be 1 or %lld", name, (long long)tokens);
  if (idx0 < 0 || idx0 >= num_ada || (kOp != kGatedRes && (idx1 < 0 || idx1 >= num_ada)))
    return fail(TDB200_ERR_INVALID_ARG, "%s: ada index out of range", name);
  if (!aligned16(x) || !aligned16(y) || !aligned16(table) || !aligned16(ts) || (res && !aligned16(res)))
    return fail(TDB200_ERR_INVALID_ARG, "%s: buffers must be 16-byte aligned", name);
  if (b * tokens > 0x7FFFFFFFll) return fail(TDB200_ERR_UNSUPPORTED, "%s: too many rows", name);
  if (int rc = require_sm90()) return rc;
  LtxParams p{x, res, table, ts, y, b * tokens, int(tokens), int(ts_tokens), int(n), num_ada, idx0, idx1, eps};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == TDB200_DTYPE_BF16) return launch<__nv_bfloat16, kOp>(p, st);
  if (dtype == TDB200_DTYPE_FP16) return launch<__half, kOp>(p, st);
  return fail(TDB200_ERR_UNSUPPORTED, "%s: dtype tag %d", name, dtype);
}
}  // namespace

extern "C" int tdb200_ltx_modulated_rms_norm_ada(const void* x, int dtype, const float* table, const void* timestep,
                                                 int scale_index, int shift_index, int num_ada, void* y, int64_t b,
                                                 int64_t tokens, int64_t ts_tokens, int64_t n, float eps, void* stream) {
  return run<kModRms>("ltx_modulated_rms_norm_ada", x, nullptr, dtype, table, timestep, scale_index, shift_index, num_ada,
                      y, b, tokens, ts_tokens, n, eps, stream);
}
extern "C" int tdb200_ltx_modulate_ada(const void* x, int dtype, const float* table, const void* timestep, int scale_index,
                                       int shift_index, int num_ada, void* y, int64_t b, int64_t tokens, int64_t ts_tokens,
                                       int64_t n, void* stream) {
  return run<kModulate>("ltx_modulate_ada", x, nullptr, dtype, table, timestep, scale_index, shift_index, num_ada, y, b,
                        tokens, ts_tokens, n, 0.f, stream);
}
extern "C" int tdb200_ltx_gated_residual_ada(const void* x, const void* residual, int dtype, const float* table,
                                             const void* timestep, int gate_index, int num_ada, void* y, int64_t b,
                                             int64_t tokens, int64_t ts_tokens, int64_t n, void* stream) {
  return run<kGatedRes>("ltx_gated_residual_ada", x, residual, dtype, table, timestep, gate_index, 0, num_ada, y, b, tokens,
                        ts_tokens, n, 0.f, stream);
}
extern "C" int tdb200_ltx_split_rope(const void* x, const void* cos_freqs, const void* sin_freqs, int dtype, void* y,
                                     int64_t b, int64_t t, int64_t h, int64_t d, void* stream) {
  using namespace tdb;
  if (!x || !cos_freqs || !sin_freqs || !y) return fail(TDB200_ERR_INVALID_ARG, "ltx_split_rope: null pointer");
  if (b <= 0 || t <= 0 || h <= 0 || d <= 0 || d % 16 != 0) return fail(TDB200_ERR_INVALID_ARG, "ltx_split_rope: bad shape (d %% 16 == 0)");
  if (int rc = require_sm90()) return rc;
  const int64_t chunks = b * t * h * (d / 16);
  int64_t grid = (chunks + 255) / 256;
  const int64_t cap = int64_t(sm_count()) * 16;
  if (grid > cap) grid = cap;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == TDB200_DTYPE_BF16)
    ltx_split_rope_kernel<__nv_bfloat16><<<static_cast<unsigned>(grid), 256, 0, st>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(cos_freqs),
        static_cast<const __nv_bfloat16*>(sin_freqs), static_cast<__nv_bfloat16*>(y), chunks, int(t), int(h), int(d));
  else if (dtype == TDB200_DTYPE_FP16)
    ltx_split_rope_kernel<__half><<<static_cast<unsigned>(grid), 256, 0, st>>>(
        static_cast<const __half*>(x), static_cast<const __half*>(cos_freqs), static_cast<const __half*>(sin_freqs),
        static_cast<__half*>(y), chunks, int(t), int(h), int(d));
  else
    return fail(TDB200_ERR_UNSUPPORTED, "ltx_split_rope: dtype tag %d", dtype);
  return check_launch("ltx_split_rope_kernel");
}

// ---------------------------------------------------------------------------------------------------------------
// Per-row symmetric INT8 quantisation of the LTX W8A8 path (ltx_distillation/tilelang_w8a8.py:16-36):
//   scale = max(amax, 1e-4) / 127;  q = clip(round_half_away(x / scale), -128, 127).   One CTA per row.
// ---------------------------------------------------------------------------------------------------------------
namespace {
using namespace tdb;
template <typename T, int kThreads, int kChunks>
__global__ void __launch_bounds__(kThreads) row_quant_kernel(const T* __restrict__ x, int8_t* __restrict__ q,
                                                             float* __restrict__ s, int n) {
  __shared__ float red[kThreads / 32];
  const int64_t row = blockIdx.x;
  const int nchunks = n / 8;
  uint4 raw[kChunks];
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < kChunks; ++i) {
    const int c = threadIdx.x + i * kThreads;
    raw[i] = make_uint4(0u, 0u, 0u, 0u);
    if (c < nchunks) raw[i] = ldg_nc_v4(x + row * n + c * 8);
    const uint32_t w[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
#pragma unroll
    for (int j = 0; j < 4; ++j) amax = fmaxf(amax, fmaxf(fabsf(F16Traits<T>::lo(w[j])), fabsf(F16Traits<T>::hi(w[j]))));
  }
  amax = warp_max(amax);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) amax = fmaxf(amax, red[w]);
  const float scale = fmaxf(amax, 1.0e-4f) / 127.0f;
  if (threadIdx.x == 0) s[row] = scale;
#pragma unroll
  for (int i = 0; i < kChunks; ++i) {
    const int c = threadIdx.x + i * kThreads;
    if (c >= nchunks) continue;
    const uint32_t w[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = (j & 1) ? F16Traits<T>::hi(w[j >> 1]) : F16Traits<T>::lo(w[j >> 1]);
      const float sc = __fdiv_rn(v, scale);
      float r = sc >= 0.f ? floorf(__fadd_rn(sc, 0.5f)) : ceilf(__fsub_rn(sc, 0.5f));
      r = fminf(fmaxf(r, -128.f), 127.f);
      const uint32_t b = static_cast<uint32_t>(static_cast<int>(r)) & 0xFFu;
      if (j < 4) lo |= b << (8 * j); else hi |= b << (8 * (j - 4));
    }
    *reinterpret_cast<uint2*>(q + row * n + c * 8) = make_uint2(lo, hi);
  }
}
}  // namespace

extern "C" int tdb200_quant_int8_rowwise(const void* x, int dtype, int64_t m, int64_t k, int8_t* q, float* s, void* stream) {
  using namespace tdb;
  if (!x || !q || !s) return fail(TDB200_ERR_INVALID_ARG, "quant_int8_rowwise: null pointer");
  if (m < 0 || k <= 0 || k % 8 != 0) return fail(TDB200_ERR_INVALID_ARG, "quant_int8_rowwise: bad shape (k %% 8 == 0)");
  if (m == 0) return TDB200_OK;
  if (!aligned16(x) || (reinterpret_cast<uintptr_t>(q) & 7u)) return fail(TDB200_ERR_INVALID_ARG, "quant_int8_rowwise: misaligned buffer");
  if (m > 0x7FFFFFFFll) return fail(TDB200_ERR_UNSUPPORTED, "quant_int8_rowwise: too many rows");
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nchunks = static_cast<int>(k / 8);
  const unsigned grid = static_cast<unsigned>(m);
#define TDB_RQ(T, TH, CH) row_quant_kernel<T, TH, CH><<<grid, TH, 0, st>>>(static_cast<const T*>(x), q, s, static_cast<int>(k))
#define TDB_RQ_DISPATCH(T)                         \
  if (nchunks <= 128) TDB_RQ(T, 128, 1);           \
  else if (nchunks <= 256) TDB_RQ(T, 128, 2);      \
  else if (nchunks <= 512) TDB_RQ(T, 256, 2);      \
  else if (nchunks <= 1024) TDB_RQ(T, 256, 4);     \
  else if (nchunks <= 2048) TDB_RQ(T, 256, 8);     \
  else return fail(TDB200_ERR_UNSUPPORTED, "quant_int8_rowwise: k too large")
  if (dtype == TDB200_DTYPE_BF16) { TDB_RQ_DISPATCH(__nv_bfloat16); }
  else if (dtype == TDB200_DTYPE_FP16) { TDB_RQ_DISPATCH(__half); }
  else return fail(TDB200_ERR_UNSUPPORTED, "quant_int8_rowwise: dtype tag %d", dtype);
#undef TDB_RQ_DISPATCH
#undef TDB_RQ
  return check_launch("row_quant_kernel");
}
