// a7/a8 producers for SLA: key mean, block mean-pooling, Sage INT8 per-block quantisation of Q and smoothed K.
//   reference: mean_pool turbodiffusion/SLA/utils.py:21-52; smooth-K :56; Sage quant = SpargeAttn get_vanilla_qk_quant
//   (third party, call site SLA/core.py:200-203): scale = amax/127 + 1e-7, round half away from zero.
//
// Inputs are read in the module's own [B, L, H, D] layout (row stride H*D), outputs are head-major [B, H, L, D] int8
// so the attention kernel's TMA tiles are dense 128-byte rows.  HBM-bound: q is read once (2 B -> 1 B), k twice
// (mean pass + quant pass; the second read of a <=126 MB tensor largely hits L2).
//
// Tile = ROWS x D elements held in registers by ROWS*D/64 threads (8 x 16-byte chunks per thread, warp-contiguous
// 256-byte row segments).  Column sums for the pooled mean go through shared memory in a fixed order, so results are
// run-to-run deterministic; the key mean uses a deterministic two-stage reduction (partials live in the not-yet-
// written k_i8 buffer).
#include "common.cuh"
#include "host_common.h"

namespace {
using namespace tdb;

constexpr int kMeanRows = 128;  // rows per partial in the key-mean pass (= the sequence-parallel shard alignment, so a rank's
                                // partials are exactly the single-GPU partials of its rows)

// ---- stage 1 of the key mean: partial column sums over kMeanRows rows ---------------------------------------
template <typename T, int D>
__global__ void __launch_bounds__(256) kmean_partial_kernel(const T* __restrict__ k, float* __restrict__ partial,
                                                            int64_t l, int h, int chunks) {
  constexpr int CPR = D / 8;          // 16-byte chunks per row
  constexpr int RPP = 256 / CPR;      // rows per pass
  __shared__ float red[RPP][D];
  const int hh = blockIdx.x, chunk = blockIdx.y, b = blockIdx.z;  // heads fastest: concurrent CTAs read whole [row, H*D] lines
  const int c = threadIdx.x % CPR, r = threadIdx.x / CPR;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const int64_t row_begin = int64_t(chunk) * kMeanRows;
#pragma unroll 4
  for (int p = 0; p < kMeanRows / RPP; ++p) {
    const int64_t row = row_begin + p * RPP + r;
    if (row < l) {
      const uint4 raw = ldg_nc_v4(k + ((int64_t(b) * l + row) * h + hh) * D + c * 8);
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[2 * j] += F16Traits<T>::lo(w[j]);
        acc[2 * j + 1] += F16Traits<T>::hi(w[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[r][c * 8 + j] = acc[j];
  __syncthreads();
  if (threadIdx.x < D) {
    float s = 0.f;
#pragma unroll 4
    for (int rr = 0; rr < RPP; ++rr) s += red[rr][threadIdx.x];
    partial[((int64_t(b) * h + hh) * chunks + chunk) * D + threadIdx.x] = s;
  }
}

// ---- stage 2: fixed-order reduction of the partials -> kmean [b,h,d] fp32 -------------------------------------
// 1024 threads per (b,h): thread = (group g, column); group g adds chunks g, g+G, g+2G, ... in order, the G group sums are
// combined in index order through shared memory (deterministic).  One CTA per head used to walk all chunks serially: 14 us of
// pure load latency per call.
__global__ void __launch_bounds__(1024) kmean_final_kernel(const float* __restrict__ partial, float* __restrict__ kmean, int64_t l,
                                                           int chunks, int d) {
  __shared__ float red[1024];
  const int bh = blockIdx.x;
  const int groups = 1024 / d;                 // 8 for d = 128, 16 for d = 64
  const int col = threadIdx.x % d, g = threadIdx.x / d;
  float s = 0.f;
  for (int ch = g; ch < chunks; ch += groups) s += partial[(int64_t(bh) * chunks + ch) * d + col];
  red[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x < d) {
    float t = 0.f;
    for (int gg = 0; gg < groups; ++gg) t += red[gg * d + threadIdx.x];
    kmean[int64_t(bh) * d + threadIdx.x] = t / static_cast<float>(l);
  }
}

// ---- block pass: pooled mean + Sage int8 quant of one ROWS x D tile ---------------------------------------------
template <typename T, int D, int ROWS, bool kSubMean>
__global__ void __launch_bounds__(ROWS* D / 64) pool_quant_kernel(const T* __restrict__ x,
                                                                   const float* __restrict__ kmean,
                                                                   int8_t* __restrict__ x_i8, float* __restrict__ scale,
                                                                   T* __restrict__ pool, int64_t l, int h, int nblk,
                                                                   int64_t out_row_stride, int64_t out_head_stride) {
  constexpr int THREADS = ROWS * D / 64;
  constexpr int CPR = D / 8;
  constexpr int RPP = THREADS / CPR;
  static_assert(ROWS / RPP == 8, "8 passes per thread");
  __shared__ float red[RPP][D];
  __shared__ float warp_amax[THREADS / 32];
  const int hh = blockIdx.x, blk = blockIdx.y, b = blockIdx.z;  // heads fastest: concurrent CTAs read whole [row, H*D] lines
  const int c = threadIdx.x % CPR, r = threadIdx.x / CPR;
  const int64_t bh = int64_t(b) * h + hh;

  float km[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) km[j] = kSubMean ? F16Traits<T>::round(__ldg(kmean + bh * D + c * 8 + j)) : 0.f;

  uint4 raw[8];
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int64_t row = int64_t(blk) * ROWS + p * RPP + r;
    raw[p] = make_uint4(0u, 0u, 0u, 0u);
    if (row < l) raw[p] = ldg_nc_v4(x + ((int64_t(b) * l + row) * h + hh) * D + c * 8);
  }
  float v[8][8];
  float colsum[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  float amax = 0.f;
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int64_t row = int64_t(blk) * ROWS + p * RPP + r;
    const bool ok = row < l;
    const uint32_t w[4] = {raw[p].x, raw[p].y, raw[p].z, raw[p].w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float f = (j & 1) ? F16Traits<T>::hi(w[j >> 1]) : F16Traits<T>::lo(w[j >> 1]);
      if (kSubMean) f = F16Traits<T>::round(__fsub_rn(f, km[j]));  // arg_k = k - mean, evaluated in T (utils.py:56)
      f = ok ? f : 0.f;
      v[p][j] = f;
      colsum[j] += f;
      amax = fmaxf(amax, fabsf(f));
    }
  }
  // ---- pooled mean: fixed-order column reduction, divided by the ACTUAL row count (utils.py:38-40)
#pragma unroll
  for (int j = 0; j < 8; ++j) red[r][c * 8 + j] = colsum[j];
  amax = warp_max(amax);
  if ((threadIdx.x & 31) == 0) warp_amax[threadIdx.x >> 5] = amax;
  __syncthreads();
  if (threadIdx.x < D) {
    float s = 0.f;
#pragma unroll 4
    for (int rr = 0; rr < RPP; ++rr) s += red[rr][threadIdx.x];
    const int64_t rem = l - int64_t(blk) * ROWS;
    const float cnt = static_cast<float>(rem < ROWS ? rem : ROWS);
    pool[(bh * nblk + blk) * D + threadIdx.x] = static_cast<T>(s / cnt);
  }
#pragma unroll
  for (int w = 0; w < THREADS / 32; ++w) amax = fmaxf(amax, warp_amax[w]);
  const float sc = __fadd_rn(amax / 127.0f, 1e-7f);
  const float rinv = __frcp_rn(sc);
  if (threadIdx.x == 0) scale[bh * nblk + blk] = sc;

#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int64_t row = int64_t(blk) * ROWS + p * RPP + r;
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      // x / sc, correctly rounded, without the per-element division sequence: one reciprocal per block and Markstein's
      // correction (q0 = x*r; q = q0 + (x - q0*sc)*r with fused multiply-adds equals RN(x/sc) for these magnitudes)
      const float q0 = __fmul_rn(v[p][j], rinv);
      float y = __fmaf_rn(__fmaf_rn(-q0, sc, v[p][j]), rinv, q0);
      y = __fadd_rn(y, y >= 0.f ? 0.5f : -0.5f);
      int qi = __float2int_rz(y);  // truncation toward zero == round half away after the +-0.5
      qi = max(-128, min(127, qi));
      if (j < 4)
        lo |= (static_cast<uint32_t>(qi) & 0xFFu) << (8 * j);
      else
        hi |= (static_cast<uint32_t>(qi) & 0xFFu) << (8 * (j - 4));
    }
    if (row < l)
      *reinterpret_cast<uint2*>(x_i8 + int64_t(b) * h * l * D + hh * out_head_stride + row * out_row_stride + c * 8) = make_uint2(lo, hi);
  }
}

// BQ / BK: query / key block rows, (128, 64) or (64, 128)
template <typename T, int D, int BQ>
int run_q(const void* q, int64_t b, int64_t lq, int64_t h, int8_t* q_i8, float* q_scale, void* q_pool, cudaStream_t st) {
  const int mblk = static_cast<int>(cdiv64(lq, BQ));
  dim3 gq(static_cast<unsigned>(h), mblk, static_cast<unsigned>(b));
  pool_quant_kernel<T, D, BQ, false><<<gq, BQ * D / 64, 0, st>>>(static_cast<const T*>(q), nullptr, q_i8, q_scale,
                                                                 static_cast<T*>(q_pool), lq, static_cast<int>(h), mblk, D, lq * D);
  return check_launch("pool_quant_kernel<q>");
}

template <typename T, int D>
int run_kmean_partial(const void* k, int64_t b, int64_t l, int64_t h, float* partial, cudaStream_t st) {
  const int chunks = static_cast<int>(cdiv64(l, kMeanRows));
  dim3 g1(static_cast<unsigned>(h), chunks, static_cast<unsigned>(b));
  kmean_partial_kernel<T, D><<<g1, 256, 0, st>>>(static_cast<const T*>(k), partial, l, static_cast<int>(h), chunks);
  return check_launch("kmean_partial_kernel");
}

// seq_major: k_i8 keeps the input's [b, l, h, d] layout (what a sequence-parallel rank all-gathers) instead of [b, h, l, d]
template <typename T, int D, int BK = 64>
int run_k_quant(const void* k, int64_t b, int64_t l, int64_t h, const float* kmean, int8_t* k_i8, float* k_scale, void* k_pool,
                bool seq_major, cudaStream_t st) {
  const int nblk = static_cast<int>(cdiv64(l, BK));
  dim3 gk(static_cast<unsigned>(h), nblk, static_cast<unsigned>(b));
  pool_quant_kernel<T, D, BK, true><<<gk, BK * D / 64, 0, st>>>(static_cast<const T*>(k), kmean, k_i8, k_scale,
                                                                static_cast<T*>(k_pool), l, static_cast<int>(h), nblk,
                                                                seq_major ? h * D : D, seq_major ? D : l * D);
  return check_launch("pool_quant_kernel<k>");
}

template <typename T, int D, int BK>
int run_k(const void* k, int64_t b, int64_t l, int64_t h, float* kmean, int8_t* k_i8, float* k_scale, void* k_pool,
          cudaStream_t st) {
  const int chunks = static_cast<int>(cdiv64(l, kMeanRows));
  // scratch for the partial column sums: chunks*D floats per head.  They fit in the not-yet-written k_i8 buffer (l*D bytes
  // per head) whenever 4*chunks <= l, i.e. l >= 4; a single chunk (l <= 128) reduces in place in the kmean output itself.
  float* partial = chunks == 1 ? kmean : reinterpret_cast<float*>(k_i8);
  if (int rc = run_kmean_partial<T, D>(k, b, l, h, partial, st)) return rc;
  kmean_final_kernel<<<static_cast<unsigned>(b * h), 1024, 0, st>>>(partial, kmean, l, chunks, D);
  if (int rc = check_launch("kmean_final_kernel")) return rc;
  return run_k_quant<T, D, BK>(k, b, l, h, kmean, k_i8, k_scale, k_pool, false, st);
}

template <typename T, int D, int BQ, int BK>
int run(const void* q, const void* k, int64_t b, int64_t lq, int64_t l, int64_t h, float* kmean, int8_t* q_i8,
        float* q_scale, int8_t* k_i8, float* k_scale, void* q_pool, void* k_pool, cudaStream_t st) {
  if (q != nullptr)
    if (int rc = run_q<T, D, BQ>(q, b, lq, h, q_i8, q_scale, q_pool, st)) return rc;
  if (k != nullptr)
    if (int rc = run_k<T, D, BK>(k, b, l, h, kmean, k_i8, k_scale, k_pool, st)) return rc;
  return TDB200_OK;
}

// (blkq, blkk) is (128, 64) or (64, 128); the callers check it
int quant_qk(const void* q, const void* k, int dtype, int64_t b, int64_t lq, int64_t l, int64_t h, int64_t d, float* kmean,
             int8_t* q_i8, float* q_scale, int8_t* k_i8, float* k_scale, void* q_pool, void* k_pool, int64_t blkq, int64_t blkk,
             void* stream) {
  if ((!q && !k) || (q && (!q_i8 || !q_scale || !q_pool)) || (k && (!kmean || !k_i8 || !k_scale || !k_pool)))
    return fail(TDB200_ERR_INVALID_ARG, "sla_quant_qk: null pointer");
  if (b <= 0 || l <= 0 || lq <= 0 || h <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_quant_qk: bad shape");
  if (d != 64 && d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_qk: head dim %lld (64 or 128, SLA/core.py:207)", (long long)d);
  if (h > 65535 || b > 65535 || cdiv64(l, blkk) > 65535 || cdiv64(lq, blkq) > 65535)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_qk: h, b or sequence length too large");
  if ((q && (!aligned16(q) || !aligned16(q_i8))) || (k && (!aligned16(k) || !aligned16(k_i8))))
    return fail(TDB200_ERR_INVALID_ARG, "sla_quant_qk: buffers must be 16-byte aligned");
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define TDB_RUN(T, D)                                                                                                    \
  return blkq == 128 ? run<T, D, 128, 64>(q, k, b, lq, l, h, kmean, q_i8, q_scale, k_i8, k_scale, q_pool, k_pool, st)    \
                     : run<T, D, 64, 128>(q, k, b, lq, l, h, kmean, q_i8, q_scale, k_i8, k_scale, q_pool, k_pool, st)
  if (dtype == TDB200_DTYPE_BF16) {
    if (d == 128) TDB_RUN(__nv_bfloat16, 128);
    TDB_RUN(__nv_bfloat16, 64);
  } else if (dtype == TDB200_DTYPE_FP16) {
    if (d == 128) TDB_RUN(__half, 128);
    TDB_RUN(__half, 64);
  }
#undef TDB_RUN
  return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_qk: dtype tag %d", dtype);
}

}  // namespace

extern "C" int tdb200_sla_quant_qk(const void* q, const void* k, int dtype, int64_t b, int64_t lq, int64_t l, int64_t h,
                                   int64_t d, float* kmean, int8_t* q_i8, float* q_scale, int8_t* k_i8, float* k_scale,
                                   void* q_pool, void* k_pool, void* stream) {
  return quant_qk(q, k, dtype, b, lq, l, h, d, kmean, q_i8, q_scale, k_i8, k_scale, q_pool, k_pool, 128, 64, stream);
}

// tdb200_sla_quant_qk with the block geometry chosen by the caller: Q pooled / quantised per blkq rows, smoothed K per blkk rows,
// (blkq, blkk) = (128, 64) or (64, 128).  The key mean is the same (its 128-row partials do not depend on the block size).
extern "C" int tdb200_sla_quant_qk_blocks(const void* q, const void* k, int dtype, int64_t b, int64_t lq, int64_t l, int64_t h,
                                          int64_t d, float* kmean, int8_t* q_i8, float* q_scale, int8_t* k_i8, float* k_scale,
                                          void* q_pool, void* k_pool, int64_t blkq, int64_t blkk, void* stream) {
  using namespace tdb;
  if (!((blkq == 128 && blkk == 64) || (blkq == 64 && blkk == 128)))
    return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_qk_blocks: block sizes (%lld, %lld) (BLKQ x BLKK = 128 x 64 or 64 x 128)",
                (long long)blkq, (long long)blkk);
  return quant_qk(q, k, dtype, b, lq, l, h, d, kmean, q_i8, q_scale, k_i8, k_scale, q_pool, k_pool, blkq, blkk, stream);
}

// ---- the key half split in three, for sequence-parallel ranks (dist.py): each rank reduces ITS rows to 128-row partial sums,
// the partials are all-gathered (they are exactly the single-GPU partials, so the mean is bit-identical), every rank finishes
// the mean and quantises / pools only its own key rows; INT8 K travels in the [b, l, h, d] layout it is gathered in. -------------
extern "C" int tdb200_sla_kmean_partial(const void* k, int dtype, int64_t b, int64_t l, int64_t h, int64_t d, float* partial,
                                        void* stream) {
  using namespace tdb;
  if (!k || !partial) return fail(TDB200_ERR_INVALID_ARG, "sla_kmean_partial: null pointer");
  if (b <= 0 || l <= 0 || h <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_kmean_partial: bad shape");
  if (d != 64 && d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_kmean_partial: head dim %lld (64 or 128)", (long long)d);
  if (h > 65535 || b > 65535 || cdiv64(l, kMeanRows) > 65535) return fail(TDB200_ERR_UNSUPPORTED, "sla_kmean_partial: dimension too large");
  if (!aligned16(k)) return fail(TDB200_ERR_INVALID_ARG, "sla_kmean_partial: k must be 16-byte aligned");
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == TDB200_DTYPE_BF16) return d == 128 ? run_kmean_partial<__nv_bfloat16, 128>(k, b, l, h, partial, st) : run_kmean_partial<__nv_bfloat16, 64>(k, b, l, h, partial, st);
  if (dtype == TDB200_DTYPE_FP16) return d == 128 ? run_kmean_partial<__half, 128>(k, b, l, h, partial, st) : run_kmean_partial<__half, 64>(k, b, l, h, partial, st);
  return fail(TDB200_ERR_UNSUPPORTED, "sla_kmean_partial: dtype tag %d", dtype);
}

extern "C" int tdb200_sla_kmean_final(const float* partial, int64_t b, int64_t h, int64_t chunks, int64_t d, int64_t l_total,
                                      float* kmean, void* stream) {
  using namespace tdb;
  if (!partial || !kmean) return fail(TDB200_ERR_INVALID_ARG, "sla_kmean_final: null pointer");
  if (b <= 0 || h <= 0 || chunks <= 0 || l_total <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_kmean_final: bad shape");
  if (d != 64 && d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_kmean_final: head dim %lld (64 or 128)", (long long)d);
  if (int rc = require_sm90()) return rc;
  kmean_final_kernel<<<static_cast<unsigned>(b * h), 1024, 0, static_cast<cudaStream_t>(stream)>>>(partial, kmean, l_total,
                                                                                                  static_cast<int>(chunks), static_cast<int>(d));
  return check_launch("kmean_final_kernel");
}

extern "C" int tdb200_sla_quant_k_seq_blocks(const void* k, const float* kmean, int dtype, int64_t b, int64_t l, int64_t h,
                                             int64_t d, int8_t* k_i8, float* k_scale, void* k_pool, int64_t blkk, void* stream) {
  using namespace tdb;
  if (blkk != 64 && blkk != 128)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_k_seq_blocks: key block size %lld (BLKK = 64 or 128)", (long long)blkk);
  if (!k || !kmean || !k_i8 || !k_scale || !k_pool) return fail(TDB200_ERR_INVALID_ARG, "sla_quant_k_seq: null pointer");
  if (b <= 0 || l <= 0 || h <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_quant_k_seq: bad shape");
  if (d != 64 && d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_k_seq: head dim %lld (64 or 128)", (long long)d);
  if (h > 65535 || b > 65535 || cdiv64(l, blkk) > 65535) return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_k_seq: dimension too large");
  if (!aligned16(k) || !aligned16(k_i8)) return fail(TDB200_ERR_INVALID_ARG, "sla_quant_k_seq: buffers must be 16-byte aligned");
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define TDB_RUN(T, D)                                                                                 \
  return blkk == 64 ? run_k_quant<T, D, 64>(k, b, l, h, kmean, k_i8, k_scale, k_pool, true, st)      \
                    : run_k_quant<T, D, 128>(k, b, l, h, kmean, k_i8, k_scale, k_pool, true, st)
  if (dtype == TDB200_DTYPE_BF16) {
    if (d == 128) TDB_RUN(__nv_bfloat16, 128);
    TDB_RUN(__nv_bfloat16, 64);
  } else if (dtype == TDB200_DTYPE_FP16) {
    if (d == 128) TDB_RUN(__half, 128);
    TDB_RUN(__half, 64);
  }
#undef TDB_RUN
  return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_k_seq: dtype tag %d", dtype);
}

extern "C" int tdb200_sla_quant_k_seq(const void* k, const float* kmean, int dtype, int64_t b, int64_t l, int64_t h, int64_t d,
                                      int8_t* k_i8, float* k_scale, void* k_pool, void* stream) {
  return tdb200_sla_quant_k_seq_blocks(k, kmean, dtype, b, l, h, d, k_i8, k_scale, k_pool, 64, stream);
}
