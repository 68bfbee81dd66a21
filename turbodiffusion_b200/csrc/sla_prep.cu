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

// kVL (tdb200_sla_quant_qk_vl): batch entry b owns its first seq_lens[b] rows, clamped to [0, l] on the device; l stays the row
// stride of the padded buffers.  Every row test below then masks at that length, as a call on the entry alone masks at its l.
template <bool kVL>
__device__ __forceinline__ int64_t rows_of(const int32_t* seq_lens, int64_t l, int b) {
  if constexpr (kVL) return min(max(int64_t(__ldg(seq_lens + b)), int64_t(0)), l);
  return l;
}

// ---- stage 1 of the key mean: partial column sums over kMeanRows rows ---------------------------------------
template <typename T, int D, bool kVL = false>
__global__ void __launch_bounds__(256) kmean_partial_kernel(const T* __restrict__ k, float* __restrict__ partial,
                                                            int64_t l, int h, int chunks, const int32_t* seq_lens = nullptr) {
  constexpr int CPR = D / 8;          // 16-byte chunks per row
  constexpr int RPP = 256 / CPR;      // rows per pass
  __shared__ float red[RPP][D];
  const int hh = blockIdx.x, chunk = blockIdx.y, b = blockIdx.z;  // heads fastest: concurrent CTAs read whole [row, H*D] lines
  const int c = threadIdx.x % CPR, r = threadIdx.x / CPR;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const int64_t row_begin = int64_t(chunk) * kMeanRows;
  const int64_t n = rows_of<kVL>(seq_lens, l, b);
#pragma unroll 4
  for (int p = 0; p < kMeanRows / RPP; ++p) {
    const int64_t row = row_begin + p * RPP + r;
    if (row < n) {
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
// pure load latency per call.  kVL: entry b reduces its own ceil(n / 128) chunks (the partials a call on the entry alone forms,
// in the same order) and divides by its n; an entry with no rows gets a zero mean.
template <bool kVL = false>
__global__ void __launch_bounds__(1024) kmean_final_kernel(const float* __restrict__ partial, float* __restrict__ kmean, int64_t l,
                                                           int chunks, int d, const int32_t* seq_lens = nullptr, int h = 1) {
  __shared__ float red[1024];
  const int bh = blockIdx.x;
  const int groups = 1024 / d;                 // 8 for d = 128, 16 for d = 64
  const int col = threadIdx.x % d, g = threadIdx.x / d;
  const int64_t n = rows_of<kVL>(seq_lens, l, kVL ? bh / h : 0);
  const int my_chunks = kVL ? static_cast<int>(cdiv64(n, kMeanRows)) : chunks;
  float s = 0.f;
  for (int ch = g; ch < my_chunks; ch += groups) s += partial[(int64_t(bh) * chunks + ch) * d + col];
  red[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x < d) {
    float t = 0.f;
    for (int gg = 0; gg < groups; ++gg) t += red[gg * d + threadIdx.x];
    kmean[int64_t(bh) * d + threadIdx.x] = (kVL && n == 0) ? 0.f : t / static_cast<float>(n);
  }
}

// ---- block pass: pooled mean + Sage int8 quant of one ROWS x D tile ---------------------------------------------
// kVL: rows past the entry's length are masked as rows past l are; a block wholly past it pools to zero.
template <typename T, int D, int ROWS, bool kSubMean, bool kVL = false>
__global__ void __launch_bounds__(ROWS* D / 64) pool_quant_kernel(const T* __restrict__ x,
                                                                   const float* __restrict__ kmean,
                                                                   int8_t* __restrict__ x_i8, float* __restrict__ scale,
                                                                   T* __restrict__ pool, int64_t l, int h, int nblk,
                                                                   int64_t out_row_stride, int64_t out_head_stride,
                                                                   const int32_t* seq_lens = nullptr) {
  constexpr int THREADS = ROWS * D / 64;
  constexpr int CPR = D / 8;
  constexpr int RPP = THREADS / CPR;
  static_assert(ROWS / RPP == 8, "8 passes per thread");
  __shared__ float red[RPP][D];
  __shared__ float warp_amax[THREADS / 32];
  const int hh = blockIdx.x, blk = blockIdx.y, b = blockIdx.z;  // heads fastest: concurrent CTAs read whole [row, H*D] lines
  const int c = threadIdx.x % CPR, r = threadIdx.x / CPR;
  const int64_t bh = int64_t(b) * h + hh;
  const int64_t n = rows_of<kVL>(seq_lens, l, b);

  float km[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) km[j] = kSubMean ? F16Traits<T>::round(__ldg(kmean + bh * D + c * 8 + j)) : 0.f;

  uint4 raw[8];
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int64_t row = int64_t(blk) * ROWS + p * RPP + r;
    raw[p] = make_uint4(0u, 0u, 0u, 0u);
    if (row < n) raw[p] = ldg_nc_v4(x + ((int64_t(b) * l + row) * h + hh) * D + c * 8);
  }
  float v[8][8];
  float colsum[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  float amax = 0.f;
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int64_t row = int64_t(blk) * ROWS + p * RPP + r;
    const bool ok = row < n;
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
    const int64_t rem = n - int64_t(blk) * ROWS;
    const float cnt = static_cast<float>(rem < ROWS ? rem : ROWS);
    pool[(bh * nblk + blk) * D + threadIdx.x] = (kVL && rem <= 0) ? static_cast<T>(0.f) : static_cast<T>(s / cnt);
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
    if (row < n)
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
  kmean_final_kernel<><<<static_cast<unsigned>(b * h), 1024, 0, st>>>(partial, kmean, l, chunks, D);
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

}  // namespace

// Q pooled / quantised per blkq rows, smoothed K per blkk rows, (blkq, blkk) = (128, 64) or (64, 128).  The key mean is the same
// for both (its 128-row partials do not depend on the block size).
extern "C" int tdb200_sla_quant_qk(const void* q, const void* k, int dtype, int64_t b, int64_t lq, int64_t l, int64_t h,
                                   int64_t d, float* kmean, int8_t* q_i8, float* q_scale, int8_t* k_i8, float* k_scale,
                                   void* q_pool, void* k_pool, int64_t blkq, int64_t blkk, void* stream) {
  using namespace tdb;
  if (!((blkq == 128 && blkk == 64) || (blkq == 64 && blkk == 128)))
    return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_qk: block sizes (%lld, %lld) (BLKQ x BLKK = 128 x 64 or 64 x 128)",
                (long long)blkq, (long long)blkk);
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
  kmean_final_kernel<><<<static_cast<unsigned>(b * h), 1024, 0, static_cast<cudaStream_t>(stream)>>>(partial, kmean, l_total,
                                                                                                  static_cast<int>(chunks), static_cast<int>(d));
  return check_launch("kmean_final_kernel");
}

extern "C" int tdb200_sla_quant_k_seq(const void* k, const float* kmean, int dtype, int64_t b, int64_t l, int64_t h, int64_t d,
                                      int8_t* k_i8, float* k_scale, void* k_pool, int64_t blkk, void* stream) {
  using namespace tdb;
  if (blkk != 64 && blkk != 128)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_k_seq: key block size %lld (BLKK = 64 or 128)", (long long)blkk);
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

// ---- e4m3 V for the SageSLA kernels' FP8 P.V (tdb200_sla_attn_fwd_fp8v) ----------------------------------------------------
// Two passes over v [b, l, h, d]: the per-channel amax over all l rows (order-independent, so the scales are reproducible),
// then codes of v / v_scale, transposed to [b, h, d, l_pad] with each 32-key group in the order the attention kernel's e4m3
// A fragment needs (sla_attn.cuh, PvOps): the permutation costs nothing here, since this pass gathers every output byte from a
// staged tile anyway, and saves the kernel a byte exchange between lanes for every P.V.
namespace {
constexpr int kVAmaxRows = 256;             // rows per CTA of the amax pass
constexpr float kE4m3Max = 448.0f;
constexpr float kVAmaxFloor = 0x1p-64f;     // an all-zero channel gets a finite, normal scale (and zero codes)

// amax[b, h, d] (fp32 bits, non-negative, so integer max is float max) over rows [kVAmaxRows * blockIdx.x, +kVAmaxRows)
template <typename T>
__global__ void __launch_bounds__(256) v_amax_kernel(const T* __restrict__ v, unsigned int* __restrict__ amax, int64_t l, int hd) {
  const int b = blockIdx.y;
  const int64_t row0 = int64_t(blockIdx.x) * kVAmaxRows;
  const int rows = l - row0 < kVAmaxRows ? static_cast<int>(l - row0) : kVAmaxRows;
  for (int cv = threadIdx.x; cv < hd / 8; cv += 256) {
    uint32_t m[4] = {0u, 0u, 0u, 0u};
    const T* src = v + (int64_t(b) * l + row0) * hd + cv * 8;
#pragma unroll 8
    for (int r = 0; r < rows; ++r) {
      const uint4 raw = ldg_nc_v4(src + int64_t(r) * hd);
      m[0] = F16Traits<T>::absmax2(m[0], raw.x);
      m[1] = F16Traits<T>::absmax2(m[1], raw.y);
      m[2] = F16Traits<T>::absmax2(m[2], raw.z);
      m[3] = F16Traits<T>::absmax2(m[3], raw.w);
    }
    unsigned int* dst = amax + int64_t(b) * hd + cv * 8;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      atomicMax(dst + 2 * j, __float_as_uint(F16Traits<T>::lo(m[j])));
      atomicMax(dst + 2 * j + 1, __float_as_uint(F16Traits<T>::hi(m[j])));
    }
  }
}

// in place: amax -> v_scale = max(amax, floor) / 448
__global__ void v_scale_kernel(float* __restrict__ scale, int64_t n) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) scale[i] = __fdiv_rn(fmaxf(scale[i], kVAmaxFloor), kE4m3Max);
}

// one [BK keys x 128 channels] tile of one (b, h): rows >= l are zero.  Position 16 u + 4 t + j of every 32-key group holds key
// 16 u + 8 (j >> 1) + 2 t + (j & 1).
template <typename T, int BK>
__global__ void __launch_bounds__(256) v_quant_fp8_kernel(const T* __restrict__ v, const float* __restrict__ scale,
                                                          uint8_t* __restrict__ v_fp8, int64_t l, int h, int64_t l_pad) {
  constexpr int D = 128;
  __shared__ __align__(16) uint16_t tile[BK][D];
  const int blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  for (int c = threadIdx.x; c < BK * D / 8; c += 256) {   // 16 chunks of 16 bytes per key row
    const int r = c / (D / 8), cc = c % (D / 8);
    const int64_t row = int64_t(blk) * BK + r;
    uint4 raw = make_uint4(0u, 0u, 0u, 0u);
    if (row < l) raw = ldg_nc_v4(v + ((int64_t(b) * l + row) * h + hh) * D + cc * 8);
    *reinterpret_cast<uint4*>(&tile[r][cc * 8]) = raw;
  }
  __syncthreads();
  const int dch = threadIdx.x & (D - 1);                   // a warp reads 32 channels of one key row: no bank conflict
  const float s = __ldg(scale + (int64_t(b) * h + hh) * D + dch);
  uint8_t* dst = v_fp8 + ((int64_t(b) * h + hh) * D + dch) * l_pad + int64_t(blk) * BK;
  for (int g = threadIdx.x >> 7; g < BK / 16; g += 2) {     // 16 output positions per store
    float x[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int pos = 16 * g + i;
      const int key = (pos & ~15) | (((pos >> 1) & 1) << 3) | (((pos >> 2) & 3) << 1) | (pos & 1);
      uint16_t bits = tile[key][dch];
      x[i] = __fdiv_rn(F16Traits<T>::lo(bits), s);
    }
    uint4 out;
    out.x = pack4_e4m3(x[0], x[1], x[2], x[3]);
    out.y = pack4_e4m3(x[4], x[5], x[6], x[7]);
    out.z = pack4_e4m3(x[8], x[9], x[10], x[11]);
    out.w = pack4_e4m3(x[12], x[13], x[14], x[15]);
    *reinterpret_cast<uint4*>(dst + 16 * g) = out;
  }
}

template <typename T>
int run_quant_v_fp8(const void* v, int64_t b, int64_t l, int64_t h, int64_t blkk, uint8_t* v_fp8, float* v_scale, cudaStream_t st) {
  const int64_t nblk = cdiv64(l, blkk), n = b * h * 128;
  if (int rc = check_cuda(cudaMemsetAsync(v_scale, 0, size_t(n) * 4, st), "cudaMemsetAsync(v_scale)")) return rc;
  v_amax_kernel<T><<<dim3(static_cast<unsigned>(cdiv64(l, kVAmaxRows)), static_cast<unsigned>(b)), 256, 0, st>>>(
      static_cast<const T*>(v), reinterpret_cast<unsigned int*>(v_scale), l, static_cast<int>(h * 128));
  if (int rc = check_launch("v_amax_kernel")) return rc;
  v_scale_kernel<<<static_cast<unsigned>(cdiv64(n, 256)), 256, 0, st>>>(v_scale, n);
  if (int rc = check_launch("v_scale_kernel")) return rc;
  const dim3 grid(static_cast<unsigned>(nblk), static_cast<unsigned>(h), static_cast<unsigned>(b));
  if (blkk == 128)
    v_quant_fp8_kernel<T, 128><<<grid, 256, 0, st>>>(static_cast<const T*>(v), v_scale, v_fp8, l, static_cast<int>(h), nblk * 128);
  else
    v_quant_fp8_kernel<T, 64><<<grid, 256, 0, st>>>(static_cast<const T*>(v), v_scale, v_fp8, l, static_cast<int>(h), nblk * 64);
  return check_launch("v_quant_fp8_kernel");
}
}  // namespace

extern "C" int tdb200_sla_quant_v_fp8(const void* v, int dtype, int64_t b, int64_t l, int64_t h, int64_t d, int64_t blkk,
                                      uint8_t* v_fp8, float* v_scale, void* stream) {
  using namespace tdb;
  if (blkk != 64 && blkk != 128)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_v_fp8: key block size %lld (BLKK = 64 or 128)", (long long)blkk);
  if (!v || !v_fp8 || !v_scale) return fail(TDB200_ERR_INVALID_ARG, "sla_quant_v_fp8: null pointer");
  if (b <= 0 || l <= 0 || h <= 0 || d <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_quant_v_fp8: bad shape");
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_v_fp8: head dim %lld (FP8 P.V is implemented for d=128)", (long long)d);
  if (dtype != TDB200_DTYPE_BF16 && dtype != TDB200_DTYPE_FP16) return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_v_fp8: dtype tag %d", dtype);
  if (h > 65535 || b > 65535 || cdiv64(l, blkk) > 0x7FFFFFFF || int64_t(1) * l * h * d * 2 >= (int64_t(1) << 40))
    return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_v_fp8: dimension too large (b, h <= 65535; l * h * d below 2^39)");
  if (!aligned16(v) || !aligned16(v_fp8) || !aligned16(v_scale))
    return fail(TDB200_ERR_INVALID_ARG, "sla_quant_v_fp8: buffers must be 16-byte aligned");
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == TDB200_DTYPE_BF16) return run_quant_v_fp8<__nv_bfloat16>(v, b, l, h, blkk, v_fp8, v_scale, st);
  return run_quant_v_fp8<__half>(v, b, l, h, blkk, v_fp8, v_scale, st);
}

// ---- per-entry lengths (tdb200_sla_quant_qk_vl): the kVL instantiations, after every existing one -------------------------
namespace {
template <typename T, int BQ, int BK>
int run_vl(const void* q, const void* k, int64_t b, int64_t l, int64_t h, const int32_t* seq_lens, float* kmean, int8_t* q_i8,
           float* q_scale, int8_t* k_i8, float* k_scale, void* q_pool, void* k_pool, cudaStream_t st) {
  constexpr int D = 128;
  if (q != nullptr) {
    const int mblk = static_cast<int>(cdiv64(l, BQ));
    pool_quant_kernel<T, D, BQ, false, true><<<dim3(static_cast<unsigned>(h), mblk, static_cast<unsigned>(b)), BQ * D / 64, 0, st>>>(
        static_cast<const T*>(q), nullptr, q_i8, q_scale, static_cast<T*>(q_pool), l, static_cast<int>(h), mblk, D, l * D, seq_lens);
    if (int rc = check_launch("pool_quant_kernel<q, vl>")) return rc;
  }
  if (k != nullptr) {
    const int chunks = static_cast<int>(cdiv64(l, kMeanRows));
    float* partial = chunks == 1 ? kmean : reinterpret_cast<float*>(k_i8);   // as run_k
    kmean_partial_kernel<T, D, true><<<dim3(static_cast<unsigned>(h), chunks, static_cast<unsigned>(b)), 256, 0, st>>>(
        static_cast<const T*>(k), partial, l, static_cast<int>(h), chunks, seq_lens);
    if (int rc = check_launch("kmean_partial_kernel<vl>")) return rc;
    kmean_final_kernel<true><<<static_cast<unsigned>(b * h), 1024, 0, st>>>(partial, kmean, l, chunks, D, seq_lens,
                                                                             static_cast<int>(h));
    if (int rc = check_launch("kmean_final_kernel<vl>")) return rc;
    const int nblk = static_cast<int>(cdiv64(l, BK));
    pool_quant_kernel<T, D, BK, true, true><<<dim3(static_cast<unsigned>(h), nblk, static_cast<unsigned>(b)), BK * D / 64, 0, st>>>(
        static_cast<const T*>(k), kmean, k_i8, k_scale, static_cast<T*>(k_pool), l, static_cast<int>(h), nblk, D, l * D, seq_lens);
    if (int rc = check_launch("pool_quant_kernel<k, vl>")) return rc;
  }
  return TDB200_OK;
}
}  // namespace

// tdb200_sla_quant_qk for a padded batch: q and k [b, l, h, 128] share one length per entry, seq_lens [b] (device int32, clamped
// to [0, l]).  Entry b's rows below its length get the bits tdb200_sla_quant_qk gives on that entry alone cut to those rows: its
// own key mean, pooled means and scales.  Rows past it are not written; blocks wholly past it pool to zero.  Either half may be
// NULL, as for tdb200_sla_quant_qk.
extern "C" int tdb200_sla_quant_qk_vl(const void* q, const void* k, int dtype, int64_t b, int64_t l, int64_t h, int64_t d,
                                      const int32_t* seq_lens, float* kmean, int8_t* q_i8, float* q_scale, int8_t* k_i8,
                                      float* k_scale, void* q_pool, void* k_pool, int64_t blkq, int64_t blkk, void* stream) {
  using namespace tdb;
  if (!((blkq == 128 && blkk == 64) || (blkq == 64 && blkk == 128)))
    return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_qk_vl: block sizes (%lld, %lld) (BLKQ x BLKK = 128 x 64 or 64 x 128)",
                (long long)blkq, (long long)blkk);
  if ((!q && !k) || (q && (!q_i8 || !q_scale || !q_pool)) || (k && (!kmean || !k_i8 || !k_scale || !k_pool)))
    return fail(TDB200_ERR_INVALID_ARG, "sla_quant_qk_vl: null pointer");
  if (!seq_lens || (reinterpret_cast<uintptr_t>(seq_lens) & 3u))
    return fail(TDB200_ERR_INVALID_ARG, "sla_quant_qk_vl: seq_lens must be a non-null, 4-byte aligned int32 [b]");
  if (b <= 0 || l <= 0 || h <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_quant_qk_vl: bad shape");
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_qk_vl: head dim %lld (per-entry lengths serve d = 128)", (long long)d);
  if (h > 65535 || b > 65535 || cdiv64(l, 64) > 65535) return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_qk_vl: h, b or sequence length too large");
  if ((q && (!aligned16(q) || !aligned16(q_i8))) || (k && (!aligned16(k) || !aligned16(k_i8))))
    return fail(TDB200_ERR_INVALID_ARG, "sla_quant_qk_vl: buffers must be 16-byte aligned");
  if (dtype != TDB200_DTYPE_BF16 && dtype != TDB200_DTYPE_FP16) return fail(TDB200_ERR_UNSUPPORTED, "sla_quant_qk_vl: dtype tag %d", dtype);
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define TDB_RUN(T)                                                                                                         \
  return blkq == 128 ? run_vl<T, 128, 64>(q, k, b, l, h, seq_lens, kmean, q_i8, q_scale, k_i8, k_scale, q_pool, k_pool, st) \
                     : run_vl<T, 64, 128>(q, k, b, l, h, seq_lens, kmean, q_i8, q_scale, k_i8, k_scale, q_pool, k_pool, st)
  if (dtype == TDB200_DTYPE_BF16) TDB_RUN(__nv_bfloat16);
  TDB_RUN(__half);
#undef TDB_RUN
}
