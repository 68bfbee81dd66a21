// a3-a6. FastNorm family, AdaLN modulation / gate, RoPE — all HBM-bound row kernels.
//   reference semantics: turbodiffusion/ops/core.py:96-136 (RMS), :193-243 / :293-335 (LayerNorm, incl. the unmasked
//   variance padding term, see below), call-site casts :441-442 / :477-478; modulation rcm/networks/wan2pt1.py:398-417;
//   RoPE wan2pt1.py:156-178.
//
// One CTA per row; the row lives in registers (16-byte chunks, lane -> consecutive chunk, so every warp-wide access
// is a contiguous 512-byte segment).  Reductions: warp shuffle + one smem exchange.  Arithmetic mirrors the
// reference's op order with explicit (non-contracted) fp32 multiplies/adds where the reference runs separate ops.
//
// LayerNorm variance quirk (reproduced on purpose): the Triton kernels pad the row to N2 = next_pow2(N) with zeros and
// do not mask (x - mean)^2, so var = (sum_{j<N}(x_j-mean)^2 + (N2-N)*mean^2) / N   (ops/core.py:217-224, 315-322).
#include "common.cuh"
#include "host_common.h"

namespace {
using namespace tdb;


template <int kThreads>
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();  // protect `red` from the previous use
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) t += red[w];
  return t;
}

__device__ __forceinline__ int next_pow2_dev(int n) { return n <= 1 ? 1 : 1 << (32 - __clz(n - 1)); }

// ---- element access: a "chunk" is 8 elements for 16-bit types and 4 elements for fp32 (both 16 bytes) ----------
template <typename T>
struct Chunk;
template <>
struct Chunk<float> {
  static constexpr int kElems = 4;
  static __device__ __forceinline__ void unpack(const uint4& r, float* f) {
    f[0] = __uint_as_float(r.x); f[1] = __uint_as_float(r.y); f[2] = __uint_as_float(r.z); f[3] = __uint_as_float(r.w);
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
  }
  static __device__ __forceinline__ float round(float a) { return a; }
};
template <typename T16>
struct Chunk16 {
  static constexpr int kElems = 8;
  static __device__ __forceinline__ void unpack(const uint4& r, float* f) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      f[2 * j] = F16Traits<T16>::lo(w[j]);
      f[2 * j + 1] = F16Traits<T16>::hi(w[j]);
    }
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    return make_uint4(F16Traits<T16>::pack(f[0], f[1]), F16Traits<T16>::pack(f[2], f[3]),
                      F16Traits<T16>::pack(f[4], f[5]), F16Traits<T16>::pack(f[6], f[7]));
  }
  static __device__ __forceinline__ float round(float a) { return F16Traits<T16>::round(a); }
};
template <>
struct Chunk<__nv_bfloat16> : Chunk16<__nv_bfloat16> {};
template <>
struct Chunk<__half> : Chunk16<__half> {};

// E consecutive fp32 parameters (E = 4 or 8, 16-byte aligned) with 128-bit loads
template <int E>
__device__ __forceinline__ void load_params(const float* __restrict__ p, float* out) {
#pragma unroll
  for (int i = 0; i < E / 4; ++i) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(p) + i);
    out[4 * i] = v.x; out[4 * i + 1] = v.y; out[4 * i + 2] = v.z; out[4 * i + 3] = v.w;
  }
}

// sin/cos of a RoPE angle (|x| up to a few thousand rad): two-term Cody-Waite reduction to [-pi, pi] followed by the
// MUFU approximations (abs error ~2^-21 there).  The reference calls torch.cos/torch.sin (wan2pt1.py:170-171); the
// difference (< 1e-6 abs) moves a bf16 result by one ulp in ~1e-4 of the elements, inside the stated RoPE tolerance,
// and keeps this kernel HBM-bound instead of bound by the ~40-instruction accurate sincosf.
__device__ __forceinline__ void rope_sincos(float x, float* sn, float* cs) {
  const float n = rintf(x * 0.15915494309189535f);
  float r = fmaf(n, -6.2831854820251465f, x);
  r = fmaf(n, 1.7484555e-7f, r);
  *sn = __sinf(r);
  *cs = __cosf(r);
}

enum NormKind { kRms = 0, kLayer = 1 };
enum PostKind { kPostNone = 0, kPostModulate = 1, kPostRope = 2, kPostStatsOnly = 3, kPostRopeTable = 4 };

struct RowParams {
  const void* x;
  void* y;
  const float* w;       // affine weight or NULL
  const float* b;       // affine bias or NULL
  const float* scale;   // modulation scale (1 + scale applied) or NULL
  const float* shift;   // modulation shift
  const float* angles;  // RoPE angles [rows, d/2]; kPostRopeTable: (cos, sin) pairs [rows, d/2, 2]
  float* stats;         // [2*m] mean, rstd (kPostStatsOnly)
  int64_t m;
  int n;
  int d;                // head dim for RoPE
  float eps;
  const void* res_y;    // kResidIn: x <- T(x + T(res_y * T(gate)))  (gate NULL: plain x + res_y), written to `y` first
  const float* gate;
};

// T: element type of x and y.  kChunks: 16-byte chunks per thread.
// kWarpRow = false: one CTA per row (reductions through shared memory, two __syncthreads each).
// kWarpRow = true : one WARP per row, kThreads/32 rows per CTA: the reductions are shuffles only, no CTA barrier, and a
//   lane keeps kChunks independent 16-byte loads in flight (6 for dim 1536, 20 for dim 5120), which is what an HBM-bound
//   row kernel needs.  The CTA-per-row form serves longer rows.
template <typename T, int kNorm, int kPost, int kThreads, int kChunks, bool kResidIn = false, bool kWarpRow = false>
__global__ void __launch_bounds__(kThreads) row_norm_kernel(RowParams p) {
  __shared__ float red[kThreads / 32];
  constexpr int E = Chunk<T>::kElems;
  constexpr int kStride = kWarpRow ? 32 : kThreads;
  const int tix = kWarpRow ? int(threadIdx.x & 31) : int(threadIdx.x);
  const int64_t row = kWarpRow ? int64_t(blockIdx.x) * (kThreads / 32) + (threadIdx.x >> 5) : int64_t(blockIdx.x);
  if (kWarpRow && row >= p.m) return;  // whole warp leaves; there is no CTA-wide barrier in this form
  const int nchunks = p.n / E;
  const T* xr = static_cast<const T*>(p.x) + row * p.n;

  uint4 raw[kChunks];
#pragma unroll
  for (int i = 0; i < kChunks; ++i) {
    const int c = tix + i * kStride;
    raw[i] = make_uint4(0u, 0u, 0u, 0u);
    if (c < nchunks) raw[i] = ldg_nc_v4(xr + c * E);
  }
  if (kResidIn) {
    // fused gate/residual update (wan2pt1.py:405-406): the updated row is stored and becomes the LayerNorm input
    const T* yr_in = static_cast<const T*>(p.res_y) + row * p.n;
    T* out = static_cast<T*>(p.y) + row * p.n;
#pragma unroll
    for (int i = 0; i < kChunks; ++i) {
      const int c = tix + i * kStride;
      if (c < nchunks) {
        float xf[E], yf[E], gv[E];
        Chunk<T>::unpack(raw[i], xf);
        Chunk<T>::unpack(ldg_nc_v4(yr_in + c * E), yf);
        if (p.gate != nullptr) load_params<E>(p.gate + c * E, gv);
#pragma unroll
        for (int j = 0; j < E; ++j) {
          const float t = (p.gate != nullptr) ? Chunk<T>::round(__fmul_rn(yf[j], Chunk<T>::round(gv[j]))) : yf[j];
          xf[j] = __fadd_rn(xf[j], t);
        }
        raw[i] = Chunk<T>::pack(xf);  // rounded to T: exactly what a separate LayerNorm pass would read back
        stg_v4(out + c * E, raw[i]);
      }
    }
  }

  const float inv_n = 1.0f / static_cast<float>(p.n);
  float mean = 0.f, rstd;
  if (kNorm == kRms) {
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kChunks; ++i) {
      float f[E];
      Chunk<T>::unpack(raw[i], f);
#pragma unroll
      for (int j = 0; j < E; ++j) ss = fmaf(f[j], f[j], ss);
    }
    ss = kWarpRow ? warp_sum(ss) : block_sum<kThreads>(ss, red);
    rstd = 1.0f / sqrtf(__fadd_rn(ss / static_cast<float>(p.n), p.eps));
  } else {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kChunks; ++i) {
      float f[E];
      Chunk<T>::unpack(raw[i], f);
#pragma unroll
      for (int j = 0; j < E; ++j) s += f[j];
    }
    s = kWarpRow ? warp_sum(s) : block_sum<kThreads>(s, red);
    mean = s / static_cast<float>(p.n);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kChunks; ++i) {
      const int c = tix + i * kStride;
      if (c < nchunks) {
        float f[E];
        Chunk<T>::unpack(raw[i], f);
#pragma unroll
        for (int j = 0; j < E; ++j) {
          const float dlt = f[j] - mean;
          ss = fmaf(dlt, dlt, ss);
        }
      }
    }
    ss = kWarpRow ? warp_sum(ss) : block_sum<kThreads>(ss, red);
    // the reference's unmasked padding columns: (N2 - N) * mean^2
    ss = __fadd_rn(ss, __fmul_rn(static_cast<float>(next_pow2_dev(p.n) - p.n), __fmul_rn(mean, mean)));
    rstd = 1.0f / sqrtf(__fadd_rn(ss / static_cast<float>(p.n), p.eps));
  }
  (void)inv_n;

  if (kPost == kPostStatsOnly) {
    if (tix == 0) {
      p.stats[2 * row] = mean;
      p.stats[2 * row + 1] = rstd;
    }
    return;
  }

  T* yr = static_cast<T*>(p.y) + row * p.n;
#pragma unroll
  for (int i = 0; i < kChunks; ++i) {
    const int c = tix + i * kStride;
    if (c < nchunks) {
      float f[E];
      Chunk<T>::unpack(raw[i], f);
      const int col = c * E;
      float wv[E], bv[E], scv[E], shv[E];
      if (p.w != nullptr) load_params<E>(p.w + col, wv);
      if (p.w != nullptr && p.b != nullptr) load_params<E>(p.b + col, bv);
      if (kPost == kPostModulate) {
        load_params<E>(p.scale + col, scv);
        load_params<E>(p.shift + col, shv);
      }
#pragma unroll
      for (int j = 0; j < E; ++j) {
        float v = (kNorm == kRms) ? __fmul_rn(f[j], rstd) : __fmul_rn(f[j] - mean, rstd);
        if (p.w != nullptr) {
          v = __fmul_rn(v, wv[j]);
          if (p.b != nullptr) v = __fadd_rn(v, bv[j]);
        }
        if (kPost == kPostModulate) {
          v = Chunk<T>::round(v);  // norm output is cast to T before the modulation (wan2pt1.py:404)
          v = __fadd_rn(__fmul_rn(v, __fadd_rn(1.0f, scv[j])), shv[j]);
        }
        f[j] = v;
      }
      if (kPost == kPostRope) {
        // pairs (2i, 2i+1) inside a head of width d; angle index = row * d/2 + (col % d)/2 + i
        float ang[E / 2];
        load_params<E / 2>(p.angles + row * (p.d >> 1) + ((col % p.d) >> 1), ang);
#pragma unroll
        for (int j = 0; j < E; j += 2) {
          float sn, cs;
          rope_sincos(ang[j >> 1], &sn, &cs);
          const float x0 = Chunk<T>::round(f[j]), x1 = Chunk<T>::round(f[j + 1]);  // rope input is the T-cast norm
          f[j] = __fsub_rn(__fmul_rn(x0, cs), __fmul_rn(x1, sn));
          f[j + 1] = __fadd_rn(__fmul_rn(x0, sn), __fmul_rn(x1, cs));
        }
      }
      if (kPost == kPostRopeTable) {
        // the same rotation with (cos, sin) read from a table built once per angle tensor: every head of a row and every
        // layer / projection of a step reuse the same 64 pairs, so the table lines stay in L1/L2 and the kernel keeps no
        // range reduction or MUFU work (the in-kernel sincos form spends issue slots on both)
        float cs[E];
        load_params<E>(p.angles + (row * (p.d >> 1) + ((col % p.d) >> 1)) * 2, cs);
#pragma unroll
        for (int j = 0; j < E; j += 2) {
          const float x0 = Chunk<T>::round(f[j]), x1 = Chunk<T>::round(f[j + 1]);
          f[j] = __fsub_rn(__fmul_rn(x0, cs[j]), __fmul_rn(x1, cs[j + 1]));
          f[j + 1] = __fadd_rn(__fmul_rn(x0, cs[j + 1]), __fmul_rn(x1, cs[j]));
        }
      }
      stg_v4(yr + col, Chunk<T>::pack(f));
    }
  }
}

template <typename T, int kNorm, int kPost, bool kResidIn = false>
int launch_rows(const RowParams& p, cudaStream_t st) {
  constexpr int E = Chunk<T>::kElems;
  const int nchunks = p.n / E;
  if (p.m > 0x7FFFFFFFll) return fail(TDB200_ERR_UNSUPPORTED, "row kernel: too many rows");
  // warp-per-row form for rows of up to 24 chunks per lane (n <= 6144 16-bit elements); 8 rows per 256-thread CTA
  {
    const unsigned wgrid = static_cast<unsigned>((p.m + 7) / 8);
#define TDB_LAUNCH_W(CH)                                                                   \
  row_norm_kernel<T, kNorm, kPost, 256, CH, kResidIn, true><<<wgrid, 256, 0, st>>>(p);    \
  return check_launch("row_norm_kernel(warp)")
    // used up to 8 chunks per lane (n <= 2048 16-bit elements, e.g. dim 1536): more chunks per lane hold more registers and cut
    // the occupancy the shuffle-only form relies on, so longer rows (dim 5120) take the CTA-per-row form.  The threshold has not
    // been re-measured on H100.
    if (nchunks <= 32 * 2) { TDB_LAUNCH_W(2); }
    if (nchunks <= 32 * 4) { TDB_LAUNCH_W(4); }
    if (nchunks <= 32 * 6) { TDB_LAUNCH_W(6); }
    if (nchunks <= 32 * 8) { TDB_LAUNCH_W(8); }
#undef TDB_LAUNCH_W
  }
  const unsigned grid = static_cast<unsigned>(p.m);
#define TDB_LAUNCH(TH, CH)                                                         \
  row_norm_kernel<T, kNorm, kPost, TH, CH, kResidIn><<<grid, TH, 0, st>>>(p);      \
  return check_launch("row_norm_kernel")
  if (nchunks <= 128) { TDB_LAUNCH(128, 1); }
  if (nchunks <= 256) { TDB_LAUNCH(128, 2); }
  if (nchunks <= 512) { TDB_LAUNCH(256, 2); }
  if (nchunks <= 1024) { TDB_LAUNCH(256, 4); }
  if (nchunks <= 2048) { TDB_LAUNCH(256, 8); }
#undef TDB_LAUNCH
  return fail(TDB200_ERR_UNSUPPORTED, "row kernel: n=%d too large (max %d)", p.n, 2048 * E);
}

int check_rows(const char* name, const void* x, const void* y, int64_t m, int64_t n, int elems_per_chunk) {
  if (!x || !y) return fail(TDB200_ERR_INVALID_ARG, "%s: null pointer", name);
  if (m < 0 || n <= 0) return fail(TDB200_ERR_INVALID_ARG, "%s: bad shape", name);
  if (n % elems_per_chunk != 0)
    return fail(TDB200_ERR_UNSUPPORTED, "%s: n=%lld must be a multiple of %d", name, (long long)n, elems_per_chunk);
  if (!aligned16(x) || !aligned16(y)) return fail(TDB200_ERR_INVALID_ARG, "%s: buffers must be 16-byte aligned", name);
  return require_sm90();
}

template <int kNorm, int kPost>
int dispatch16(int dtype, const RowParams& p, cudaStream_t st, const char* name) {
  if (dtype == TDB200_DTYPE_BF16) return launch_rows<__nv_bfloat16, kNorm, kPost>(p, st);
  if (dtype == TDB200_DTYPE_FP16) return launch_rows<__half, kNorm, kPost>(p, st);
  return fail(TDB200_ERR_UNSUPPORTED, "%s: dtype tag %d", name, dtype);
}

// ---- elementwise: out = T(x + T(y * T(gate[j]))) ------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) gate_residual_kernel(const T* __restrict__ x, const T* __restrict__ y,
                                                            const float* __restrict__ gate, T* __restrict__ out,
                                                            int64_t total_chunks, int n) {
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t c = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; c < total_chunks; c += stride) {
    const int64_t e = c * 8;
    const int col = static_cast<int>(e % n);
    const uint4 xr = ldg_nc_v4(x + e), yr = ldg_nc_v4(y + e);
    float xf[8], yf[8];
    Chunk<T>::unpack(xr, xf);
    Chunk<T>::unpack(yr, yf);
    float gv[8];
    load_params<8>(gate + col, gv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float g = Chunk<T>::round(gv[j]);
      xf[j] = __fadd_rn(xf[j], Chunk<T>::round(__fmul_rn(yf[j], g)));
    }
    stg_v4(out + e, Chunk<T>::pack(xf));
  }
}

// ---- standalone RoPE: y = T(rotate(float(x))) ------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) rope_kernel(const T* __restrict__ x, const float* __restrict__ angles,
                                                   T* __restrict__ y, int64_t total_chunks, int hd, int d) {
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t c = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; c < total_chunks; c += stride) {
    const int64_t e = c * 8;
    const int64_t row = e / hd;
    const int col = static_cast<int>(e % hd);
    float ang[4];
    load_params<4>(angles + row * (d >> 1) + ((col % d) >> 1), ang);
    float f[8];
    Chunk<T>::unpack(ldg_nc_v4(x + e), f);
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      float sn, cs;
      rope_sincos(ang[j >> 1], &sn, &cs);
      const float x0 = f[j], x1 = f[j + 1];
      f[j] = __fsub_rn(__fmul_rn(x0, cs), __fmul_rn(x1, sn));
      f[j + 1] = __fadd_rn(__fmul_rn(x0, sn), __fmul_rn(x1, cs));
    }
    stg_v4(y + e, Chunk<T>::pack(f));
  }
}

// ---- LN + modulate + 128x128-block int8 quant (tile pass; row statistics come from the stats pass) ---------------
template <typename T>
__global__ void __launch_bounds__(256) ln_modulate_quant_tile_kernel(const T* __restrict__ x,
                                                                     const float* __restrict__ stats,
                                                                     const float* __restrict__ scale,
                                                                     const float* __restrict__ shift,
                                                                     int8_t* __restrict__ q, float* __restrict__ s,
                                                                     int64_t m, int64_t n, int n_blocks) {
  __shared__ float warp_amax[8];
  const int tid = threadIdx.x;
  const int blk_n = blockIdx.x, blk_m = blockIdx.y;
  const int col = blk_n * 128 + (tid & 15) * 8;
  const int row0 = blk_m * 128 + (tid >> 4);
  const bool col_ok = col < n;

  uint4 raw[8];
  float mu[8], rs[8];
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int64_t row = row0 + p * 16;
    raw[p] = make_uint4(0u, 0u, 0u, 0u);
    mu[p] = 0.f;
    rs[p] = 0.f;
    if (col_ok && row < m) {
      raw[p] = ldg_nc_v4(x + row * n + col);
      const float2 st = __ldg(reinterpret_cast<const float2*>(stats) + row);
      mu[p] = st.x;
      rs[p] = st.y;
    }
  }
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) sc[j] = sh[j] = 0.f;
  if (col_ok) {
    load_params<8>(scale + col, sc);
    load_params<8>(shift + col, sh);
#pragma unroll
    for (int j = 0; j < 8; ++j) sc[j] = __fadd_rn(1.0f, sc[j]);
  }
  float v[8][8];
  float amax = 1e-8f;
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int64_t row = row0 + p * 16;
    const bool ok = col_ok && row < m;
    float f[8];
    Chunk<T>::unpack(raw[p], f);
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      // both roundings to T are done on PAIRS (one pack instruction per two values instead of one conversion each)
      const uint32_t n2 = F16Traits<T>::pack(__fmul_rn(f[j] - mu[p], rs[p]), __fmul_rn(f[j + 1] - mu[p], rs[p]));
      const uint32_t m2 = F16Traits<T>::pack(__fadd_rn(__fmul_rn(F16Traits<T>::lo(n2), sc[j]), sh[j]),
                                             __fadd_rn(__fmul_rn(F16Traits<T>::hi(n2), sc[j + 1]), sh[j + 1]));  // the modulated activation in T, as quant_cuda sees it
      v[p][j] = ok ? F16Traits<T>::lo(m2) : 0.f;
      v[p][j + 1] = ok ? F16Traits<T>::hi(m2) : 0.f;
      amax = fmaxf(amax, fmaxf(fabsf(v[p][j]), fabsf(v[p][j + 1])));
    }
  }
  amax = warp_max(amax);
  if ((tid & 31) == 0) warp_amax[tid >> 5] = amax;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < 8; ++w) amax = fmaxf(amax, warp_amax[w]);
  const float r = __fdiv_rn(128.0f, amax);
  if (tid == 0) s[int64_t(blk_m) * n_blocks + blk_n] = amax * 0.0078125f;
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int64_t row = row0 + p * 16;
    const uint32_t lo = pack4_s8_rne(__fmul_rn(v[p][0], r), __fmul_rn(v[p][1], r), __fmul_rn(v[p][2], r), __fmul_rn(v[p][3], r));
    const uint32_t hi = pack4_s8_rne(__fmul_rn(v[p][4], r), __fmul_rn(v[p][5], r), __fmul_rn(v[p][6], r), __fmul_rn(v[p][7], r));
    if (col_ok && row < m) *reinterpret_cast<uint2*>(q + row * n + col) = make_uint2(lo, hi);
  }
}

int elementwise_grid(int64_t chunks) {
  const int64_t want = (chunks + 255) / 256;
  const int64_t cap = int64_t(sm_count()) * 16;
  return static_cast<int>(want < cap ? (want > 0 ? want : 1) : cap);
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
extern "C" int tdb200_rms_norm_f32(const float* x, const float* w, float* y, int64_t m, int64_t n, float eps,
                                   void* stream) {
  if (int rc = check_rows("rms_norm_f32", x, y, m, n, 4)) return rc;
  if (m == 0) return TDB200_OK;
  RowParams p{x, y, w, nullptr, nullptr, nullptr, nullptr, nullptr, m, static_cast<int>(n), 0, eps, nullptr, nullptr};
  return launch_rows<float, kRms, kPostNone>(p, static_cast<cudaStream_t>(stream));
}

extern "C" int tdb200_layer_norm_f32(const float* x, const float* w, const float* b, float* y, int64_t m, int64_t n,
                                     float eps, void* stream) {
  if (int rc = check_rows("layer_norm_f32", x, y, m, n, 4)) return rc;
  if (m == 0) return TDB200_OK;
  RowParams p{x, y, w, b, nullptr, nullptr, nullptr, nullptr, m, static_cast<int>(n), 0, eps, nullptr, nullptr};
  return launch_rows<float, kLayer, kPostNone>(p, static_cast<cudaStream_t>(stream));
}

extern "C" int tdb200_rms_norm(const void* x, int dtype, const float* w, void* y, int64_t m, int64_t n, float eps,
                               void* stream) {
  if (int rc = check_rows("rms_norm", x, y, m, n, 8)) return rc;
  if (m == 0) return TDB200_OK;
  RowParams p{x, y, w, nullptr, nullptr, nullptr, nullptr, nullptr, m, static_cast<int>(n), 0, eps, nullptr, nullptr};
  return dispatch16<kRms, kPostNone>(dtype, p, static_cast<cudaStream_t>(stream), "rms_norm");
}

extern "C" int tdb200_layer_norm(const void* x, int dtype, const float* w, const float* b, void* y, int64_t m,
                                 int64_t n, float eps, void* stream) {
  if (int rc = check_rows("layer_norm", x, y, m, n, 8)) return rc;
  if (m == 0) return TDB200_OK;
  RowParams p{x, y, w, b, nullptr, nullptr, nullptr, nullptr, m, static_cast<int>(n), 0, eps, nullptr, nullptr};
  return dispatch16<kLayer, kPostNone>(dtype, p, static_cast<cudaStream_t>(stream), "layer_norm");
}

extern "C" int tdb200_layer_norm_modulate(const void* x, int dtype, const float* scale, const float* shift, void* y,
                                          int64_t m, int64_t n, float eps, void* stream) {
  if (int rc = check_rows("layer_norm_modulate", x, y, m, n, 8)) return rc;
  if (!scale || !shift) return tdb::fail(TDB200_ERR_INVALID_ARG, "layer_norm_modulate: null scale/shift");
  if (m == 0) return TDB200_OK;
  RowParams p{x, y, nullptr, nullptr, scale, shift, nullptr, nullptr, m, static_cast<int>(n), 0, eps, nullptr, nullptr};
  return dispatch16<kLayer, kPostModulate>(dtype, p, static_cast<cudaStream_t>(stream), "layer_norm_modulate");
}

extern "C" int tdb200_layer_norm_modulate_quant(const void* x, int dtype, const float* scale, const float* shift,
                                                int8_t* q, float* s, float* row_stats, int64_t m, int64_t n,
                                                float eps, void* stream) {
  using namespace tdb;
  if (int rc = check_rows("layer_norm_modulate_quant", x, q, m, n, 8)) return rc;
  if (!scale || !shift || !s || !row_stats)
    return fail(TDB200_ERR_INVALID_ARG, "layer_norm_modulate_quant: null pointer");
  if (m == 0) return TDB200_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RowParams p{x, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, row_stats, m, static_cast<int>(n), 0, eps, nullptr, nullptr};
  if (int rc = dispatch16<kLayer, kPostStatsOnly>(dtype, p, st, "layer_norm_modulate_quant(stats)")) return rc;
  const int64_t nb = cdiv64(n, 128), mb = cdiv64(m, 128);
  if (mb > 65535) return fail(TDB200_ERR_UNSUPPORTED, "layer_norm_modulate_quant: m too large");
  dim3 grid(static_cast<unsigned>(nb), static_cast<unsigned>(mb));
  if (dtype == TDB200_DTYPE_BF16)
    ln_modulate_quant_tile_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(x), row_stats,
                                                                      scale, shift, q, s, m, n, static_cast<int>(nb));
  else
    ln_modulate_quant_tile_kernel<__half><<<grid, 256, 0, st>>>(static_cast<const __half*>(x), row_stats, scale, shift,
                                                               q, s, m, n, static_cast<int>(nb));
  return check_launch("ln_modulate_quant_tile_kernel");
}

extern "C" int tdb200_gate_residual(const void* x, const void* y, const float* gate, void* out, int dtype, int64_t m,
                                    int64_t n, void* stream) {
  using namespace tdb;
  if (int rc = check_rows("gate_residual", x, out, m, n, 8)) return rc;
  if (!y || !gate || !aligned16(y)) return fail(TDB200_ERR_INVALID_ARG, "gate_residual: bad y/gate pointer");
  if (m == 0) return TDB200_OK;
  const int64_t chunks = m * n / 8;
  const int grid = elementwise_grid(chunks);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == TDB200_DTYPE_BF16)
    gate_residual_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(x),
                                                             static_cast<const __nv_bfloat16*>(y), gate,
                                                             static_cast<__nv_bfloat16*>(out), chunks, static_cast<int>(n));
  else if (dtype == TDB200_DTYPE_FP16)
    gate_residual_kernel<__half><<<grid, 256, 0, st>>>(static_cast<const __half*>(x), static_cast<const __half*>(y),
                                                      gate, static_cast<__half*>(out), chunks, static_cast<int>(n));
  else
    return fail(TDB200_ERR_UNSUPPORTED, "gate_residual: dtype tag %d", dtype);
  return check_launch("gate_residual_kernel");
}

extern "C" int tdb200_rope_interleaved(const void* x, int dtype, const float* angles, void* y, int64_t l, int64_t h,
                                       int64_t d, void* stream) {
  using namespace tdb;
  if (int rc = check_rows("rope_interleaved", x, y, l, h * d, 8)) return rc;
  if (!angles || d % 8 != 0) return fail(TDB200_ERR_INVALID_ARG, "rope_interleaved: null angles or d %% 8 != 0");
  if (l == 0) return TDB200_OK;
  const int64_t chunks = l * h * d / 8;
  const int grid = elementwise_grid(chunks);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == TDB200_DTYPE_BF16)
    rope_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(x), angles,
                                                    static_cast<__nv_bfloat16*>(y), chunks, static_cast<int>(h * d),
                                                    static_cast<int>(d));
  else if (dtype == TDB200_DTYPE_FP16)
    rope_kernel<__half><<<grid, 256, 0, st>>>(static_cast<const __half*>(x), angles, static_cast<__half*>(y), chunks,
                                             static_cast<int>(h * d), static_cast<int>(d));
  else
    return fail(TDB200_ERR_UNSUPPORTED, "rope_interleaved: dtype tag %d", dtype);
  return check_launch("rope_kernel");
}

extern "C" int tdb200_rms_norm_rope(const void* x, int dtype, const float* w, const float* angles, void* y, int64_t l,
                                    int64_t h, int64_t d, float eps, void* stream) {
  using namespace tdb;
  if (int rc = check_rows("rms_norm_rope", x, y, l, h * d, 8)) return rc;
  if (!angles || !w || d % 8 != 0) return fail(TDB200_ERR_INVALID_ARG, "rms_norm_rope: null pointer or d %% 8 != 0");
  if (l == 0) return TDB200_OK;
  RowParams p{x, y, w, nullptr, nullptr, nullptr, angles, nullptr, l, static_cast<int>(h * d), static_cast<int>(d), eps, nullptr, nullptr};
  return dispatch16<kRms, kPostRope>(dtype, p, static_cast<cudaStream_t>(stream), "rms_norm_rope");
}

extern "C" int tdb200_rms_norm_rope_table(const void* x, int dtype, const float* w, const float* cos_sin, void* y, int64_t l,
                                          int64_t h, int64_t d, float eps, void* stream) {
  using namespace tdb;
  if (int rc = check_rows("rms_norm_rope_table", x, y, l, h * d, 8)) return rc;
  if (!cos_sin || !w || d % 8 != 0 || !aligned16(cos_sin))
    return fail(TDB200_ERR_INVALID_ARG, "rms_norm_rope_table: null / misaligned pointer or d %% 8 != 0");
  if (l == 0) return TDB200_OK;
  RowParams p{x, y, w, nullptr, nullptr, nullptr, cos_sin, nullptr, l, static_cast<int>(h * d), static_cast<int>(d), eps, nullptr, nullptr};
  return dispatch16<kRms, kPostRopeTable>(dtype, p, static_cast<cudaStream_t>(stream), "rms_norm_rope_table");
}

extern "C" int tdb200_gate_residual_stats(const void* x, const void* y, const float* gate, void* out, float* row_stats,
                                          int dtype, int64_t m, int64_t n, float eps, void* stream) {
  using namespace tdb;
  if (int rc = check_rows("gate_residual_stats", x, out, m, n, 8)) return rc;
  if (!y || !row_stats || !aligned16(y)) return fail(TDB200_ERR_INVALID_ARG, "gate_residual_stats: bad y/stats pointer");
  if (m == 0) return TDB200_OK;
  RowParams p{x, out, nullptr, nullptr, nullptr, nullptr, nullptr, row_stats, m, static_cast<int>(n), 0, eps, y, gate};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == TDB200_DTYPE_BF16) return launch_rows<__nv_bfloat16, kLayer, kPostStatsOnly, true>(p, st);
  if (dtype == TDB200_DTYPE_FP16) return launch_rows<__half, kLayer, kPostStatsOnly, true>(p, st);
  return fail(TDB200_ERR_UNSUPPORTED, "gate_residual_stats: dtype tag %d", dtype);
}

extern "C" int tdb200_layer_norm_modulate_quant_stats(const void* x, int dtype, const float* row_stats, const float* scale,
                                                      const float* shift, int8_t* q, float* s, int64_t m, int64_t n,
                                                      void* stream) {
  using namespace tdb;
  if (int rc = check_rows("layer_norm_modulate_quant_stats", x, q, m, n, 8)) return rc;
  if (!scale || !shift || !s || !row_stats)
    return fail(TDB200_ERR_INVALID_ARG, "layer_norm_modulate_quant_stats: null pointer");
  if (m == 0) return TDB200_OK;
  const int64_t nb = cdiv64(n, 128), mb = cdiv64(m, 128);
  if (mb > 65535) return fail(TDB200_ERR_UNSUPPORTED, "layer_norm_modulate_quant_stats: m too large");
  dim3 grid(static_cast<unsigned>(nb), static_cast<unsigned>(mb));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == TDB200_DTYPE_BF16)
    ln_modulate_quant_tile_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(x), row_stats,
                                                                      scale, shift, q, s, m, n, static_cast<int>(nb));
  else if (dtype == TDB200_DTYPE_FP16)
    ln_modulate_quant_tile_kernel<__half><<<grid, 256, 0, st>>>(static_cast<const __half*>(x), row_stats, scale, shift,
                                                               q, s, m, n, static_cast<int>(nb));
  else
    return fail(TDB200_ERR_UNSUPPORTED, "layer_norm_modulate_quant_stats: dtype tag %d", dtype);
  return check_launch("ln_modulate_quant_tile_kernel");
}
