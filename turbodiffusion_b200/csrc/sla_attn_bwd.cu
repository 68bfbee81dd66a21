// Backward of the block-sparse 16-bit attention (the sparse branch of SparseLinearAttention; reference: the autograd function
// `_attention`, SLA/kernel.py:240-319, whose backward runs _attn_bwd_preprocess / _attn_bwd_dq / _attn_bwd_dkdv, :85-237).
// Block geometry of the forward: BLKQ = 128 (or 64) query rows, BLKK = 64 key rows, 128-wide
// heads, q/k/v/o/dO/dq/dk/dv in the module layout [b, l, h, d].  The forward (sla_attn.cu, kLse) leaves o_s = T(O / l) and
// lse = m + log2(l) in the log2 domain, so that P = exp2(S * sm_scale * log2e - lse) is recomputed exactly as the forward
// normalised it.
//
//   sla_bwd_delta_kernel      delta[b,h,row] = sum_d T(dO) * T(o_s), fp32
//   sla_bwd_kmajor_index_kernel  the LUT transposed: for every (b, h, key block) the ascending list of the query blocks that
//                                selected it (CSR offsets + entries), built on the device without a host synchronisation
//   sla_bwd_dq_kernel         one CTA per (query block, head, batch): Q_i and dO_i resident, K_j / V_j streamed over the LUT row;
//                             S = Q.K^T, dP = dO.V^T, dS = P o (dP - delta), dQ += dS.K  (K tile as the MN-major operand)
//   sla_bwd_dq_q64_kernel     the same on 64-row query blocks, on the entry-split schedule of sla_attn.cuh
//   sla_bwd_dkdv_kernel       one CTA per (key block, head, batch): K_j and V_j resident, (Q_i, dO_i) streamed over the key
//                             block's list; S^T = K.Q^T, dP^T = V.dO^T, dV += P^T.dO, dK += dS^T.Q  (Q / dO tiles MN-major);
//                             one template for both query-block heights
//
// Dense attention (tdb200_attn_dense_bwd, the backward of dense_attn.cu's kLse forwards, lq != lk allowed) runs the delta
// kernel and the 128-row dQ and dK/dV kernels with kDense: the dQ CTA visits every 64-key tile and the dK/dV CTA every 128-row
// query block, in ascending order, with no LUT staging, no index read and no index kernel.  kDense is a compile-time choice
// that only replaces where a block id comes from; the per-tile arithmetic is the same instructions.  kKeyLens (with kDense,
// tdb200_attn_dense_bwd_kl): batch entry b has lk_b = k_lens[b] keys; the dQ CTA visits tiles 0 .. ceil(lk_b / 64) - 1 with
// columns >= lk_b masked and the last tile's K and V rows >= lk_b zeroed (zero_key_rows), a dK/dV CTA whose key block starts
// at or past lk_b stores zeros, and rows >= lk_b of a block that straddles lk_b are stored as zeros.  kQueryLens (with kDense
// and kKeyLens, tdb200_attn_dense_bwd_vl): batch entry b has lq_b = q_lens[b] query rows; the delta kernel writes delta = 0 for
// rows >= lq_b without reading them, a dQ CTA whose block starts at or past lq_b loads nothing and stores zeros, rows >= lq_b
// of the dQ block that straddles lq_b are stored as zeros, and the dK/dV CTA visits query blocks 0 .. ceil(lq_b / 128) - 1 with
// the straddling block's Q and dO rows >= lq_b zeroed on chip (zero_query_rows) and their lse / delta staged as +inf / 0.
//
// Rounding points (FlashAttention-2's): P and dS are formed in fp32 and rounded to T only as MMA operands; dQ, dK, dV accumulate
// in fp32 registers and are rounded to T once.  No floating-point atomics: every output element is written by one thread in a
// fixed order, so the gradients are bit-for-bit reproducible.  Key columns >= lk are masked to -inf; query rows >= lq get
// lse = +inf (P = 0) and delta = 0 explicitly, because TMA zero-fill gives their scores, not their statistics.
//
// fp16 only: dS = P o (dP - delta) is small where P is (peaked softmax) or dO is (loss-scaled training), and below fp16's
// normal range (2^-14) rounding it keeps only a few bits although dq and dk themselves are normal fp16 values.  So the dS
// operand is rounded as dS * 2^e, e per accumulator row (a query row of dQ, a key row of dK) and chosen from the largest |dS|
// that row has seen (its top bit at 2^14); when a later tile needs a smaller e the row's fp32 accumulator is rescaled by the
// power of two, and it is divided by 2^e before the store.  Every rescale is exact.  bf16 has fp32's exponent range and takes
// none of this: its instructions are unchanged.
#include <type_traits>

#include "sla_attn.cuh"
#include "host_common.h"

namespace {
using namespace tdb;

constexpr int HD = 128, BLKQ = 128, BLKQ64 = 64, BLKK = 64;

struct BwdParams {
  const float* lse;        // [b,h,lq]
  const float* delta;      // [b,h,lq]
  const int32_t* lut;      // [b,h,mblk,topk]       (dQ; not read by the dense kernels)
  const int32_t* kv_off;   // [b*h, nblk+1]          (dK/dV: CSR offsets into kv_idx; not read by the dense kernels)
  const int32_t* kv_idx;   // [b*h, mblk*topk]
  void* dq;                // [b,lq,h,d] T
  void* dk;                // [b,lk,h,d] T
  void* dv;
  int lq, lk;              // query and key lengths (lq = lk = l for SLA)
  int h, mblk, nblk;       // mblk / nblk: query / key blocks
  int topk;                // key blocks per query block (dense: nblk)
  float sm_scale;
  const int32_t* k_lens = nullptr;   // [b] int32 (kKeyLens only)
  const int32_t* q_lens = nullptr;   // [b] int32 (kQueryLens only)
};

// ------------------------------------------------------------------------------------------------ preprocessing
// One warp per (b, row, head); lanes take 4 consecutive columns, then a butterfly sum (fixed order).  kQueryLens: a row past its
// entry's q_lens[b] gets delta = 0 and reads neither o nor d_o.
template <typename T, bool kQueryLens = false>
__global__ void __launch_bounds__(256) sla_bwd_delta_kernel(const T* o, const T* d_o, float* delta, int64_t rows, int l, int h,
                                                            const int32_t* q_lens) {
  const int64_t r = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  if constexpr (kQueryLens) {
    const int64_t bl = r / h;           // b * l + row
    const int hh = int(r - bl * h);
    const int64_t b = bl / l, row = bl - b * l;
    if (row >= queries_of<true>(q_lens, l, int(b))) {
      if (lane == 0) delta[(b * h + hh) * l + row] = 0.f;
      return;
    }
  }
  const uint2 ov = *reinterpret_cast<const uint2*>(o + r * HD + lane * 4);
  const uint2 gv = *reinterpret_cast<const uint2*>(d_o + r * HD + lane * 4);
  float acc = F16Traits<T>::lo(ov.x) * F16Traits<T>::lo(gv.x);
  acc = fmaf(F16Traits<T>::hi(ov.x), F16Traits<T>::hi(gv.x), acc);
  acc = fmaf(F16Traits<T>::lo(ov.y), F16Traits<T>::lo(gv.y), acc);
  acc = fmaf(F16Traits<T>::hi(ov.y), F16Traits<T>::hi(gv.y), acc);
  acc = warp_sum(acc);
  if (lane == 0) {
    const int64_t bl = r / h;           // b * l + row
    const int hh = int(r - bl * h);
    const int64_t b = bl / l, row = bl - b * l;
    delta[(b * h + hh) * l + row] = acc;
  }
}

// One CTA per (b, h): count the selections of every key block, exclusive scan into offsets, then fill the lists taking query
// blocks in ascending order (one LUT row per step).  The integer atomics only hand out slots; within a step every slot of one
// key block receives the same query-block id, so the index does not depend on their order.
constexpr int kIndexThreads = 256;
__global__ void __launch_bounds__(kIndexThreads) sla_bwd_kmajor_index_kernel(const int32_t* lut, int mblk, int nblk, int topk,
                                                                             int32_t* kv_off, int32_t* cursor, int32_t* kv_idx) {
  __shared__ int32_t scan[kIndexThreads];
  const int bh = blockIdx.x, t = threadIdx.x;
  const int64_t n_sel = int64_t(mblk) * topk;
  const int32_t* lt = lut + bh * n_sel;
  int32_t* off = kv_off + int64_t(bh) * (nblk + 1);
  int32_t* cur = cursor + int64_t(bh) * nblk;
  int32_t* idx = kv_idx + bh * n_sel;
  for (int k = t; k < nblk; k += kIndexThreads) cur[k] = 0;
  __syncthreads();
  for (int64_t e = t; e < n_sel; e += kIndexThreads) atomicAdd(&cur[__ldg(lt + e)], 1);
  __syncthreads();
  int32_t carry = 0;
  for (int k0 = 0; k0 < nblk; k0 += kIndexThreads) {
    const int32_t c = k0 + t < nblk ? cur[k0 + t] : 0;
    scan[t] = c;
    __syncthreads();
    for (int s = 1; s < kIndexThreads; s <<= 1) {  // inclusive Hillis-Steele scan
      const int32_t v = t >= s ? scan[t - s] : 0;
      __syncthreads();
      scan[t] += v;
      __syncthreads();
    }
    if (k0 + t < nblk) {
      off[k0 + t] = carry + scan[t] - c;
      cur[k0 + t] = 0;
    }
    carry += scan[kIndexThreads - 1];
    __syncthreads();
  }
  if (t == 0) off[nblk] = carry;
  __syncthreads();
  for (int i = 0; i < mblk; ++i) {
    for (int e = t; e < topk; e += kIndexThreads) {
      const int k = __ldg(lt + int64_t(i) * topk + e);
      idx[off[k] + atomicAdd(&cur[k], 1)] = i;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ fp16 dS operand scale
// e[hf] is the exponent of rows hf = 0, 1 (r0, r0 + 8) of this thread's accumulator fragment; kDsUnset until the row has seen a
// nonzero |dS|.  Clamped to [-60, 60], so 2^e, 2^-e and every rescale ratio are normal fp32 powers of two.
constexpr int kDsUnset = 1 << 30, kDsMaxExp = 60;

__device__ __forceinline__ float pow2f(int e) { return __int_as_float((e + 127) << 23); }

// The fragment's four lanes of a row share the row maximum m[hf] of |dS| in this tile (butterfly over lanes ^1, ^2); e[hf]
// drops to 14 - floor(log2 m) when that is below it, and acc's row is rescaled to the new exponent.
__device__ __forceinline__ void ds_exponent(int (&e)[2], float (&m)[2], float (&acc)[HD / 2]) {
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    float mm = fmaxf(m[hf], __shfl_xor_sync(0xffffffffu, m[hf], 1));
    mm = fmaxf(mm, __shfl_xor_sync(0xffffffffu, mm, 2));
    if (mm > 0.f) {
      const int want = min(max(14 - (((__float_as_int(mm) >> 23) & 0xff) - 127), -kDsMaxExp), kDsMaxExp);
      if (want < e[hf]) {
        if (e[hf] != kDsUnset) {
          const float r = pow2f(want - e[hf]);
#pragma unroll
          for (int c = 0; c < HD / 8; ++c) {
            acc[4 * c + 2 * hf] *= r;
            acc[4 * c + 2 * hf + 1] *= r;
          }
        }
        e[hf] = want;
      }
    }
  }
}

// the accumulator rows back to the unscaled sum: acc row hf *= 2^-e[hf]
__device__ __forceinline__ void ds_unscale(const int (&e)[2], float (&acc)[HD / 2]) {
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const float r = pow2f(-min(e[hf], kDsMaxExp));
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      acc[4 * c + 2 * hf] *= r;
      acc[4 * c + 2 * hf + 1] *= r;
    }
  }
}

// dS of a 64 x 64 tile (fp32, fragment layout: element i in row (i >> 1) & 1) -> the T operand fragments.  fp16: scaled by
// 2^e of its row after ds_exponent has settled e (and rescaled acc) for this tile.
template <typename T>
__device__ __forceinline__ void pack_ds(float (&ds)[32], uint32_t (&da)[4][4], int (&e)[2], float (&acc)[HD / 2]) {
  if constexpr (std::is_same<T, __half>::value) {
    float m[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 32; ++i) m[(i >> 1) & 1] = fmaxf(m[(i >> 1) & 1], fabsf(ds[i]));
    ds_exponent(e, m, acc);
    const float sc[2] = {pow2f(min(e[0], kDsMaxExp)), pow2f(min(e[1], kDsMaxExp))};
#pragma unroll
    for (int i = 0; i < 32; i += 2) da[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(ds[i] * sc[(i >> 1) & 1], ds[i + 1] * sc[(i >> 1) & 1]);
  } else {
#pragma unroll
    for (int i = 0; i < 32; i += 2) da[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(ds[i], ds[i + 1]);
  }
}

// Rows r0 and r0 + 8 of an m64n128 fp32 accumulator (fragment layout, common.cuh) -> T(acc * scale) at rows [row0, row0 + 8].
template <typename T>
__device__ __forceinline__ void store_rows(const float (&acc)[HD / 2], float scale, void* out, int64_t row0, int l, int h, int hh,
                                           int b, int cq) {
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int64_t r = row0 + 8 * hf;
    if (r >= l) continue;
    T* orow = static_cast<T*>(out) + ((int64_t(b) * l + r) * h + hh) * HD;
#pragma unroll
    for (int c = 0; c < HD / 8; ++c)
      *reinterpret_cast<uint32_t*>(orow + 8 * c + cq) = F16Traits<T>::pack(acc[4 * c + 2 * hf] * scale, acc[4 * c + 2 * hf + 1] * scale);
  }
}

// ------------------------------------------------------------------------------------------------ dQ
// CTA = 2 consumer warpgroups (64 query rows each, like sla_attn_fwd_kernel) + 1 TMA warp.  Per thread: dQ 64, S 32, dP 32 fp32
// registers and the dS A fragments.  Shared memory: Q | dO (resident) | K ring | V ring (3 stages); V is released as soon as
// dP has retired, K after dQ += dS.K.
namespace dq {
constexpr int kConsumerWarps = 8, kThreads = kConsumerWarps * 32 + 32, kStages = 3;
constexpr uint32_t kTileQ = BLKQ * HD * 2, kTileK = BLKK * HD * 2;   // 32 KB, 16 KB
constexpr uint32_t kOffQ = 0, kOffDO = kTileQ, kOffK = 2 * kTileQ, kOffV = kOffK + kStages * kTileK;
constexpr uint32_t kOffBars = kOffV + kStages * kTileK, kOffLut = kOffBars + 256;
enum Bar { kQFull = 0, kKFull = 1, kKEmpty = 4, kVFull = 7, kVEmpty = 10 };
}  // namespace dq

template <typename T, bool kDense = false, bool kKeyLens = false, bool kQueryLens = false>
__global__ void __launch_bounds__(dq::kThreads, 1)
sla_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_do,
                  const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v, BwdParams p) {
  using namespace dq;
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, stays a shared-space pointer
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBars);
  uint16_t* s_lut = reinterpret_cast<uint16_t*>(smem + kOffLut);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  const int bh = b * p.h + hh;
  const int lk = keys_of<kKeyLens>(p.k_lens, p.lk, b);
  const int lq = queries_of<kQueryLens>(p.q_lens, p.lq, b);
  const bool idle = kQueryLens && m_blk * BLKQ >= lq;   // the block lies wholly past the entry's queries
  const int n_tiles = idle ? 0 : kKeyLens ? (lk + BLKK - 1) / BLKK : p.topk;

  if (threadIdx.x == 0) {
    mbar_init(&bars[kQFull], 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&bars[kKFull + i], 1);
      mbar_init(&bars[kKEmpty + i], kConsumerWarps);
      mbar_init(&bars[kVFull + i], 1);
      mbar_init(&bars[kVEmpty + i], kConsumerWarps);
    }
    mbar_fence_init();
  }
  if constexpr (!kDense) {
    const int32_t* lut_row = p.lut + (int64_t(bh) * p.mblk + m_blk) * p.topk;
    for (int i = threadIdx.x; i < p.topk; i += kThreads) s_lut[i] = static_cast<uint16_t>(__ldg(lut_row + i));
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // =============================================================== TMA producer
    if (lane == 0 && !idle) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_do);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
      mbar_expect_tx(&bars[kQFull], 2 * kTileQ);
#pragma unroll
      for (int c = 0; c < HD / 64; ++c) {
        tma_load_4d(smem + kOffQ + c * (BLKQ * 128), &tmap_q, &bars[kQFull], c * 64, hh, m_blk * BLKQ, b);
        tma_load_4d(smem + kOffDO + c * (BLKQ * 128), &tmap_do, &bars[kQFull], c * 64, hh, m_blk * BLKQ, b);
      }
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j % kStages;
        const uint32_t ph = ((j / kStages) & 1) ^ 1;
        const int blk = kDense ? j : s_lut[j];
        mbar_wait(&bars[kKEmpty + st], ph);
        mbar_expect_tx(&bars[kKFull + st], kTileK);
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(smem + kOffK + st * kTileK + c * (BLKK * 128), &tmap_k, &bars[kKFull + st], c * 64, hh, blk * BLKK, b);
        mbar_wait(&bars[kVEmpty + st], ph);
        mbar_expect_tx(&bars[kVFull + st], kTileK);
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(smem + kOffV + st * kTileK + c * (BLKK * 128), &tmap_v, &bars[kVFull + st], c * 64, hh, blk * BLKK, b);
      }
    }
    return;
  }

  // =============================================================== consumer warpgroups
  const int wg = warp >> 2, w4 = warp & 3;
  const int r_lo = wg * 64 + w4 * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t sbase = smem_u32(smem);
  const float sc = p.sm_scale * kLog2e;
  float lse[2], dlt[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int64_t r = int64_t(m_blk) * BLKQ + r_lo + 8 * hf;
    lse[hf] = r < lq ? __ldg(p.lse + int64_t(bh) * p.lq + r) : INFINITY;
    dlt[hf] = r < lq ? __ldg(p.delta + int64_t(bh) * p.lq + r) : 0.f;
  }
  float acc[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) acc[i] = 0.f;
  int ds_e[2] = {kDsUnset, kDsUnset};   // per query row (fp16)

  if (!idle) mbar_wait(&bars[kQFull], 0);
  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % kStages;
    const uint32_t ph = (j / kStages) & 1;
    const int valid = lk - (kDense ? j : s_lut[j]) * BLKK;
    const uint32_t sk = sbase + kOffK + st * kTileK, sv = sbase + kOffV + st * kTileK;

    // ---- S = Q.K^T and dP = dO.V^T for this warpgroup's 64 rows (all operands K-major over d)
    float s[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = dp[i] = 0.f;
    mbar_wait(&bars[kKFull + st], ph);
    if constexpr (kKeyLens)
      if (valid < BLKK && lk < p.lk) {   // the last tile, with rows past the entry's keys inside the buffer
        mbar_wait(&bars[kVFull + st], ph);
        zero_key_rows(smem + kOffK + st * kTileK, BLKK, HD / 64, valid, threadIdx.x);
        zero_key_rows(smem + kOffV + st * kTileK, BLKK, HD / 64, valid, threadIdx.x);
        fence_proxy_async_smem();
        named_bar_sync(1, kConsumerWarps * 32);
      }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      const uint64_t qd = make_desc_kmajor_sw128(sbase + kOffQ + (ks >> 2) * (BLKQ * 128) + wg * (64 * 128)) + uint64_t((ks & 3) * 2);
      const uint64_t kd = make_desc_kmajor_sw128(sk + (ks >> 2) * (BLKK * 128)) + uint64_t((ks & 3) * 2);
      wgmma_f16_ss<64, kBF16>(s, qd, kd, ks > 0 ? 1u : 0u);
    }
    wgmma_commit();
    mbar_wait(&bars[kVFull + st], ph);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      const uint64_t gd = make_desc_kmajor_sw128(sbase + kOffDO + (ks >> 2) * (BLKQ * 128) + wg * (64 * 128)) + uint64_t((ks & 3) * 2);
      const uint64_t vd = make_desc_kmajor_sw128(sv + (ks >> 2) * (BLKK * 128)) + uint64_t((ks & 3) * 2);
      wgmma_f16_ss<64, kBF16>(dp, gd, vd, ks > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    reg_fence(dp);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[kVEmpty + st]);

    // ---- P = exp2(S sc - lse) (columns past l masked), dS = P o (dP - delta), rounded to T into the A fragments
    uint32_t da[BLKK / 16][4];
    if constexpr (kBF16) {
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int hf = (i >> 1) & 1, col = 8 * (i >> 2) + cq;
        const float p0 = col < valid ? fast_exp2(fmaf(s[i], sc, -lse[hf])) : 0.f;
        const float p1 = col + 1 < valid ? fast_exp2(fmaf(s[i + 1], sc, -lse[hf])) : 0.f;
        da[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(p0 * (dp[i] - dlt[hf]), p1 * (dp[i + 1] - dlt[hf]));
      }
    } else {
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int hf = (i >> 1) & 1, col = 8 * (i >> 2) + cq;
        const float p0 = col < valid ? fast_exp2(fmaf(s[i], sc, -lse[hf])) : 0.f;
        const float p1 = col + 1 < valid ? fast_exp2(fmaf(s[i + 1], sc, -lse[hf])) : 0.f;
        s[i] = p0 * (dp[i] - dlt[hf]);
        s[i + 1] = p1 * (dp[i + 1] - dlt[hf]);
      }
      pack_ds<T>(s, da, ds_e, acc);
    }
    // ---- dQ += dS.K  (K: [64 keys x HD], the MN-major operand; +16 keys = +2048 B per K step)
    const uint64_t kmn = make_desc_mnmajor_sw128(sk, BLKK * 128);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BLKK / 16; ++kk) wgmma_f16_rs<HD, kBF16, 1>(acc, da[kk], kmn + uint64_t(kk * 128));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(acc);
#pragma unroll
    for (int kk = 0; kk < BLKK / 16; ++kk) reg_fence(da[kk]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[kKEmpty + st]);
  }
  if constexpr (!kBF16) ds_unscale(ds_e, acc);
  if constexpr (kQueryLens) {
    // rows past the entry's queries are zero (assigned, not scaled: their q and d_out rows may hold inf or NaN)
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
      if (int64_t(m_blk) * BLKQ + r_lo + 8 * hf >= lq) zero_o_row(acc, hf);
  }
  store_rows<T>(acc, p.sm_scale, p.dq, int64_t(m_blk) * BLKQ + r_lo, p.lq, p.h, hh, b, cq);
}

// ------------------------------------------------------------------------------------------------ dK / dV
// CTA = a producer warpgroup (one warp issues TMA; setmaxnreg hands its registers to the consumers) + 2 consumer warpgroups, both
// on the same 64 key rows; K_j and V_j resident, (Q_i, dO_i) streamed over the key block's list.  Per streamed 64-row query slab
// S^T and dP^T are 64 x 64 tiles (32 registers each); the partial dK and dV are 64 x 128 (64 + 64).  The lse / delta values of
// a slab are staged in shared memory per warpgroup (double-buffered, one named barrier per step).  At the end warpgroup 1 hands
// its partials to warpgroup 0, which adds them (fixed order) and stores.
//   kBQ = 128: warpgroup g takes query rows [64g, 64g + 64) of every list entry through a 2-stage ring whose stages both
//              warpgroups read.
//   kBQ = 64:  each list entry is one 64-row query block, taken by warpgroup j % 2.  With four ring stages slot j % 4 is only
//              ever used by warpgroup j % 2, so every slot's barriers are consumed by one warpgroup, in order, and each
//              warpgroup has its next (Q_i, dO_i) pair in flight while it computes.
template <int kBQ>
struct Dkv {
  static constexpr bool kSplit = kBQ == BLKQ64;
  static constexpr int kStages = kSplit ? 4 : 2;
  static constexpr uint32_t kTileQ = kBQ * HD * 2, kTileK = BLKK * HD * 2;
  static constexpr uint32_t kOffK = 0, kOffV = kTileK, kOffQ = 2 * kTileK, kOffDO = kOffQ + kStages * kTileQ;
  static constexpr uint32_t kOffStats = kOffDO + kStages * kTileQ;             // [warpgroup][buffer][lse 64 | delta 64] fp32
  static constexpr uint32_t kOffBars = kOffStats + 2 * 2 * 128 * 4;
  static constexpr uint32_t kSmem = kOffBars + (kSplit ? 128 : 64);
  enum Bar { kKVFull = 0, kFull = 1 /*kStages*/, kEmpty = 1 + kStages /*kStages*/ };
  static_assert((kEmpty + kStages) * 8 <= kSmem - kOffBars, "barriers exceed their shared-memory slot");
  static_assert(HD * 128 * 4 <= 2 * kStages * kTileQ, "partial dK / dV do not fit in the ring");
};

template <typename T, int kBQ, bool kDense = false, bool kKeyLens = false, bool kQueryLens = false>
__global__ void __launch_bounds__(split::kThreads, 1)
sla_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_do,
                    const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v, BwdParams p) {
  using L = Dkv<kBQ>;
  constexpr int kStages = L::kStages;
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBars);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  const int bh = b * p.h + hh;
  const int32_t* list = nullptr;   // the query blocks of this key block: list[j], or (kDense) j for every j < mblk
  int n_list = p.mblk;
  if constexpr (!kDense) {
    const int32_t* kv_off = p.kv_off + int64_t(bh) * (p.nblk + 1);
    list = p.kv_idx + int64_t(bh) * p.mblk * p.topk + __ldg(kv_off + n_blk);
    n_list = __ldg(kv_off + n_blk + 1) - __ldg(kv_off + n_blk);
  }
  const int lk = keys_of<kKeyLens>(p.k_lens, p.lk, b);
  const int lq = queries_of<kQueryLens>(p.q_lens, p.lq, b);
  if (kQueryLens) n_list = (lq + kBQ - 1) / kBQ;     // (kDense) only the query blocks below this entry's queries
  if (kKeyLens && n_blk * BLKK >= lk) n_list = 0;   // a key block past this entry's keys

  if (n_list == 0) {  // no query block selected this key block: its gradients are zero (the outputs are not pre-zeroed)
    for (int e = threadIdx.x; e < BLKK * HD / 8; e += split::kThreads) {
      const int64_t r = int64_t(n_blk) * BLKK + e / (HD / 8);
      if (r >= p.lk) break;
      const int64_t o = ((int64_t(b) * p.lk + r) * p.h + hh) * HD + (e % (HD / 8)) * 8;
      stg_v4(static_cast<T*>(p.dk) + o, make_uint4(0, 0, 0, 0));
      stg_v4(static_cast<T*>(p.dv) + o, make_uint4(0, 0, 0, 0));
    }
    return;
  }
  if (threadIdx.x == 0) {
    mbar_init(&bars[L::kKVFull], 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&bars[L::kFull + i], 1);
      mbar_init(&bars[L::kEmpty + i], L::kSplit ? 4 : 8);   // the four warps of warpgroup i % 2, or both warpgroups
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // =============================================================== TMA producer
    reg_dealloc<split::kProducerRegs>();
    if (warp == 8 && lane == 0) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_do);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
      mbar_expect_tx(&bars[L::kKVFull], 2 * L::kTileK);
#pragma unroll
      for (int c = 0; c < HD / 64; ++c) {
        tma_load_4d(smem + L::kOffK + c * (BLKK * 128), &tmap_k, &bars[L::kKVFull], c * 64, hh, n_blk * BLKK, b);
        tma_load_4d(smem + L::kOffV + c * (BLKK * 128), &tmap_v, &bars[L::kKVFull], c * 64, hh, n_blk * BLKK, b);
      }
      for (int j = 0; j < n_list; ++j) {
        const int st = j % kStages;
        const uint32_t ph = ((j / kStages) & 1) ^ 1;
        const int qb = kDense ? j : __ldg(list + j);
        mbar_wait(&bars[L::kEmpty + st], ph);
        mbar_expect_tx(&bars[L::kFull + st], 2 * L::kTileQ);
#pragma unroll
        for (int c = 0; c < HD / 64; ++c) {
          tma_load_4d(smem + L::kOffQ + st * L::kTileQ + c * (kBQ * 128), &tmap_q, &bars[L::kFull + st], c * 64, hh, qb * kBQ, b);
          tma_load_4d(smem + L::kOffDO + st * L::kTileQ + c * (kBQ * 128), &tmap_do, &bars[L::kFull + st], c * 64, hh, qb * kBQ, b);
        }
      }
    }
    return;
  }

  // =============================================================== consumer warpgroups
  reg_alloc<split::kConsumerRegs>();
  const int wg = warp >> 2, w4 = warp & 3, t = threadIdx.x & 127;
  const int kr_lo = w4 * 16 + (lane >> 2);   // key rows kr_lo, kr_lo + 8 of the block
  const int cq = 2 * (lane & 3);
  const uint32_t sbase = smem_u32(smem);
  const float sc = p.sm_scale * kLog2e;
  const int q0 = L::kSplit ? 0 : wg * 64;    // this warpgroup's first row of a streamed query block
  float* stats = reinterpret_cast<float*>(smem + L::kOffStats) + wg * 256;
  float dk[HD / 2], dv[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) dk[i] = dv[i] = 0.f;
  int ds_e[2] = {kDsUnset, kDsUnset};   // per key row of dk (fp16)

  mbar_wait(&bars[L::kKVFull], 0);
  for (int j = L::kSplit ? wg : 0, it = 0; j < n_list; j += L::kSplit ? 2 : 1, ++it) {
    const int st = j % kStages;
    const uint32_t ph = (j / kStages) & 1;
    const int qb = kDense ? j : __ldg(list + j);
    // ---- lse / delta of this warpgroup's 64 query rows; query rows >= lq: P = 0 and delta = 0
    float* sb = stats + ((L::kSplit ? it : j) & 1) * 128;
    {
      const int64_t r = int64_t(qb) * kBQ + q0 + (t & 63);
      const bool in = r < lq;
      sb[t] = t < 64 ? (in ? __ldg(p.lse + int64_t(bh) * p.lq + r) : INFINITY) : (in ? __ldg(p.delta + int64_t(bh) * p.lq + r) : 0.f);
    }
    named_bar_sync(1 + wg, 128);

    // ---- S^T = K.Q^T and dP^T = V.dO^T over this warpgroup's 64 query rows (all operands K-major over d)
    const uint32_t sq = sbase + L::kOffQ + st * L::kTileQ + q0 * 128, sg = sbase + L::kOffDO + st * L::kTileQ + q0 * 128;
    float s[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = dp[i] = 0.f;
    mbar_wait(&bars[L::kFull + st], ph);
    if constexpr (kQueryLens) {
      // this warpgroup's rows of the block that straddles lq lie past the entry's queries but inside the buffer: zeroed (and
      // their lse / delta staged as +inf / 0 above), as a trimmed call's TMA zero fill leaves them, so that no inf or NaN
      // there reaches dK or dV through P^T = 0.  Only this warpgroup reads its 64 rows of the slot.
      const int lo = lq - qb * kBQ - q0;
      if (lo < 64 && lq < p.lq) {
        zero_query_rows(smem + L::kOffQ + st * L::kTileQ + q0 * 128, kBQ, HD / 64, max(lo, 0), 64, t);
        zero_query_rows(smem + L::kOffDO + st * L::kTileQ + q0 * 128, kBQ, HD / 64, max(lo, 0), 64, t);
        fence_proxy_async_smem();
        named_bar_sync(1 + wg, 128);
      }
    }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      const uint64_t kd = make_desc_kmajor_sw128(sbase + L::kOffK + (ks >> 2) * (BLKK * 128)) + uint64_t((ks & 3) * 2);
      const uint64_t qd = make_desc_kmajor_sw128(sq + (ks >> 2) * (kBQ * 128)) + uint64_t((ks & 3) * 2);
      wgmma_f16_ss<64, kBF16>(s, kd, qd, ks > 0 ? 1u : 0u);
    }
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      const uint64_t vd = make_desc_kmajor_sw128(sbase + L::kOffV + (ks >> 2) * (BLKK * 128)) + uint64_t((ks & 3) * 2);
      const uint64_t gd = make_desc_kmajor_sw128(sg + (ks >> 2) * (kBQ * 128)) + uint64_t((ks & 3) * 2);
      wgmma_f16_ss<64, kBF16>(dp, vd, gd, ks > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    reg_fence(dp);

    // ---- P^T (columns = query rows) rounded to T; dV += P^T.dO with dO as the MN-major operand (+16 rows = +2048 B per K step).
    //      Key rows >= lk only reach dK / dV rows that are never stored, so they need no mask.
    uint32_t pa[4][4], da[4][4];
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const float2 ls = *reinterpret_cast<const float2*>(sb + 8 * (i >> 2) + cq);
      s[i] = fast_exp2(fmaf(s[i], sc, -ls.x));
      s[i + 1] = fast_exp2(fmaf(s[i + 1], sc, -ls.y));
      pa[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(s[i], s[i + 1]);
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_f16_rs<HD, kBF16, 1>(dv, pa[kk], make_desc_mnmajor_sw128(sg, kBQ * 128) + uint64_t(kk * 128));
    wgmma_commit();
    // ---- dS^T = P^T o (dP^T - delta) rounded to T; dK += dS^T.Q
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const float2 dl = *reinterpret_cast<const float2*>(sb + 64 + 8 * (i >> 2) + cq);
      dp[i] = s[i] * (dp[i] - dl.x);
      dp[i + 1] = s[i + 1] * (dp[i + 1] - dl.y);
    }
    pack_ds<T>(dp, da, ds_e, dk);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_f16_rs<HD, kBF16, 1>(dk, da[kk], make_desc_mnmajor_sw128(sq, kBQ * 128) + uint64_t(kk * 128));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dv);
    reg_fence(dk);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      reg_fence(pa[kk]);
      reg_fence(da[kk]);
    }
    warp_release(&bars[L::kEmpty + st], lane);
  }

  // ---- warpgroup 1's partials -> warpgroup 0 through the Q / dO ring, which both warpgroups have drained (dk unscaled first)
  if constexpr (!kBF16) ds_unscale(ds_e, dk);
  const Handoff x = handoff_wg1_to_wg0(smem + L::kOffQ, wg, 3, [&](const Handoff& x) {
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) {
      x[i] = dk[i];
      x[HD / 2 + i] = dv[i];
    }
  });
  if (wg == 1) return;
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) {
    dk[i] += x[i];
    dv[i] += x[HD / 2 + i];
  }
  const int64_t row0 = int64_t(n_blk) * BLKK + kr_lo;
  if constexpr (kKeyLens) {
    // key rows >= lk of the block that straddles lk saw keys the entry does not have: their rows are zero (assigned, not
    // scaled, since such a row may hold inf or NaN from whatever its keys' memory holds)
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
      if (row0 + 8 * hf >= lk) {
#pragma unroll
        for (int c = 0; c < HD / 8; ++c) dk[4 * c + 2 * hf] = dk[4 * c + 2 * hf + 1] = dv[4 * c + 2 * hf] = dv[4 * c + 2 * hf + 1] = 0.f;
      }
  }
  store_rows<T>(dk, p.sm_scale, p.dk, row0, p.lk, p.h, hh, b, cq);
  store_rows<T>(dv, 1.0f, p.dv, row0, p.lk, p.h, hh, b, cq);
}

// ------------------------------------------------------------------------------------------------ dQ on 64-row query blocks
// The backward of the 64 x 64 forward, on the entry-split schedule (sla_attn.cuh): one CTA per (64-row query block, head,
// batch); Q_i and dO_i resident, K_j / V_j streamed over the LUT row, the two consumer warpgroups take alternate entries with
// the per-entry arithmetic of sla_bwd_dq_kernel.  Each keeps its own fp32 partial, and warpgroup 0 adds warpgroup 1's in a
// fixed order before storing.
namespace dq64 {
constexpr uint32_t kTileQ = BLKQ64 * HD * 2, kTileK = BLKK * HD * 2;   // 16 KB each
constexpr uint32_t kOffQ = 0, kOffDO = kTileQ, kOffK = 2 * kTileQ, kOffV = kOffK + split::kStages * kTileK;
constexpr uint32_t kOffBars = kOffV + split::kStages * kTileK, kOffLut = kOffBars + 256;
static_assert(split::kNumBars * 8 <= 256, "barriers exceed their shared-memory slot");
static_assert(HD / 2 * 128 * 4 <= split::kStages * kTileK, "partial dQ does not fit in the K ring");
}  // namespace dq64

template <typename T>
__global__ void __launch_bounds__(split::kThreads, 1)
sla_bwd_dq_q64_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_do,
                      const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v, BwdParams p) {
  using namespace dq64;
  using namespace split;
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBars);
  uint16_t* s_lut = reinterpret_cast<uint16_t*>(smem + kOffLut);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  const int bh = b * p.h + hh;

  if (threadIdx.x == 0) init_barriers(bars);
  {
    const int32_t* lut_row = p.lut + (int64_t(bh) * p.mblk + m_blk) * p.topk;
    for (int i = threadIdx.x; i < p.topk; i += split::kThreads) s_lut[i] = static_cast<uint16_t>(__ldg(lut_row + i));
  }
  __syncthreads();

  if (warp >= 8) {
    // =============================================================== TMA producer
    reg_dealloc<kProducerRegs>();
    if (warp == 8 && lane == 0) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_do);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
      mbar_expect_tx(&bars[kQFull], 2 * kTileQ);
#pragma unroll
      for (int c = 0; c < HD / 64; ++c) {
        tma_load_4d(smem + kOffQ + c * (BLKQ64 * 128), &tmap_q, &bars[kQFull], c * 64, hh, m_blk * BLKQ64, b);
        tma_load_4d(smem + kOffDO + c * (BLKQ64 * 128), &tmap_do, &bars[kQFull], c * 64, hh, m_blk * BLKQ64, b);
      }
      for (int j = 0; j < p.topk; ++j) {
        const int st = j % kStages;
        const uint32_t ph = ((j / kStages) & 1) ^ 1;
        const int blk = s_lut[j];
        uint64_t* kfull = &bars[full(kKFull, j)];
        uint64_t* vfull = &bars[full(kVFull, j)];
        mbar_wait(&bars[kKEmpty + st], ph);
        mbar_expect_tx(kfull, kTileK);
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(smem + kOffK + st * kTileK + c * (BLKK * 128), &tmap_k, kfull, c * 64, hh, blk * BLKK, b);
        mbar_wait(&bars[kVEmpty + st], ph);
        mbar_expect_tx(vfull, kTileK);
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(smem + kOffV + st * kTileK + c * (BLKK * 128), &tmap_v, vfull, c * 64, hh, blk * BLKK, b);
      }
    }
    return;
  }

  // =============================================================== consumer warpgroups (same 64 rows, alternate LUT entries)
  reg_alloc<kConsumerRegs>();
  const int wg = warp >> 2, w4 = warp & 3;
  const int r_lo = w4 * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t sbase = smem_u32(smem);
  const float sc = p.sm_scale * kLog2e;
  float lse[2], dlt[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int64_t r = int64_t(m_blk) * BLKQ64 + r_lo + 8 * hf;
    lse[hf] = r < p.lq ? __ldg(p.lse + int64_t(bh) * p.lq + r) : INFINITY;
    dlt[hf] = r < p.lq ? __ldg(p.delta + int64_t(bh) * p.lq + r) : 0.f;
  }
  float acc[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) acc[i] = 0.f;
  int ds_e[2] = {kDsUnset, kDsUnset};   // per query row (fp16)

  mbar_wait(&bars[kQFull], 0);
  for (int j = wg; j < p.topk; j += 2) {
    const int st = j % kStages;
    const uint32_t ph = full_phase(j);
    const int valid = p.lk - s_lut[j] * BLKK;
    const uint32_t sk = sbase + kOffK + st * kTileK, sv = sbase + kOffV + st * kTileK;

    // ---- S = Q.K^T and dP = dO.V^T (all operands K-major over d)
    float s[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = dp[i] = 0.f;
    mbar_wait(&bars[full(kKFull, j)], ph);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      const uint64_t qd = make_desc_kmajor_sw128(sbase + kOffQ + (ks >> 2) * (BLKQ64 * 128)) + uint64_t((ks & 3) * 2);
      const uint64_t kd = make_desc_kmajor_sw128(sk + (ks >> 2) * (BLKK * 128)) + uint64_t((ks & 3) * 2);
      wgmma_f16_ss<64, kBF16>(s, qd, kd, ks > 0 ? 1u : 0u);
    }
    wgmma_commit();
    mbar_wait(&bars[full(kVFull, j)], ph);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      const uint64_t gd = make_desc_kmajor_sw128(sbase + kOffDO + (ks >> 2) * (BLKQ64 * 128)) + uint64_t((ks & 3) * 2);
      const uint64_t vd = make_desc_kmajor_sw128(sv + (ks >> 2) * (BLKK * 128)) + uint64_t((ks & 3) * 2);
      wgmma_f16_ss<64, kBF16>(dp, gd, vd, ks > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    reg_fence(dp);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[kVEmpty + st]);

    // ---- P = exp2(S sc - lse) (columns past l masked), dS = P o (dP - delta), rounded to T into the A fragments
    uint32_t da[BLKK / 16][4];
    if constexpr (kBF16) {
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int hf = (i >> 1) & 1, col = 8 * (i >> 2) + cq;
        const float p0 = col < valid ? fast_exp2(fmaf(s[i], sc, -lse[hf])) : 0.f;
        const float p1 = col + 1 < valid ? fast_exp2(fmaf(s[i + 1], sc, -lse[hf])) : 0.f;
        da[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(p0 * (dp[i] - dlt[hf]), p1 * (dp[i + 1] - dlt[hf]));
      }
    } else {
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int hf = (i >> 1) & 1, col = 8 * (i >> 2) + cq;
        const float p0 = col < valid ? fast_exp2(fmaf(s[i], sc, -lse[hf])) : 0.f;
        const float p1 = col + 1 < valid ? fast_exp2(fmaf(s[i + 1], sc, -lse[hf])) : 0.f;
        s[i] = p0 * (dp[i] - dlt[hf]);
        s[i + 1] = p1 * (dp[i + 1] - dlt[hf]);
      }
      pack_ds<T>(s, da, ds_e, acc);
    }
    // ---- dQ += dS.K  (K as the MN-major operand; +16 keys = +2048 B per K step)
    const uint64_t kmn = make_desc_mnmajor_sw128(sk, BLKK * 128);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BLKK / 16; ++kk) wgmma_f16_rs<HD, kBF16, 1>(acc, da[kk], kmn + uint64_t(kk * 128));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(acc);
#pragma unroll
    for (int kk = 0; kk < BLKK / 16; ++kk) reg_fence(da[kk]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[kKEmpty + st]);
  }

  // ---- dQ = partial of warpgroup 0 + partial of warpgroup 1, through the drained K ring (each unscaled first)
  if constexpr (!kBF16) ds_unscale(ds_e, acc);
  const Handoff x = handoff_wg1_to_wg0(smem + kOffK, wg, 1, [&](const Handoff& x) {
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) x[i] = acc[i];
  });
  if (wg == 1) return;
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) acc[i] += x[i];
  store_rows<T>(acc, p.sm_scale, p.dq, int64_t(m_blk) * BLKQ64 + r_lo, p.lq, p.h, hh, b, cq);
}

// ------------------------------------------------------------------------------------------------ host
struct WsLayout {
  size_t delta, kv_off, cursor, kv_idx, total;
};
size_t align256(size_t x) { return (x + 255) & ~size_t(255); }
WsLayout ws_layout(int64_t b, int64_t h, int64_t l, int64_t topk, int64_t blkq) {
  const int64_t mblk = cdiv64(l, blkq), nblk = cdiv64(l, BLKK), bh = b * h;
  WsLayout w;
  w.delta = 0;
  w.kv_off = w.delta + align256(size_t(bh * l) * 4);
  w.cursor = w.kv_off + align256(size_t(bh * (nblk + 1)) * 4);
  w.kv_idx = w.cursor + align256(size_t(bh * nblk) * 4);
  w.total = w.kv_idx + align256(size_t(bh * mblk * topk) * 4);
  return w;
}

// [b, l, h, d] 16-bit tensor, boxes of 64 columns x `rows` sequence rows of one head
int tmap_rows(CUtensorMap* m, const void* base, CUtensorMapDataType t16, int64_t b, int64_t l, int64_t h, uint32_t rows) {
  const uint64_t dims[4] = {uint64_t(HD), uint64_t(h), uint64_t(l), uint64_t(b)};
  const uint64_t str[3] = {uint64_t(HD * 2), uint64_t(h * HD * 2), uint64_t(l * h * HD * 2)};
  const uint32_t box[4] = {64, 1, rows, 1};
  return make_tmap_4d(m, base, t16, 2, dims, str, box);
}

template <typename T, int kBQ>
int launch_bwd(const void* q, const void* k, const void* v, const void* o_s, const void* d_o, const float* lse, const int32_t* lut,
               int64_t topk, void* dq, void* dk, void* dv, uint8_t* ws, int64_t b, int64_t l, int64_t h, float sm_scale,
               cudaStream_t st) {
  const int64_t mblk = cdiv64(l, kBQ), nblk = cdiv64(l, BLKK);
  const WsLayout w = ws_layout(b, h, l, topk, kBQ);
  float* delta = reinterpret_cast<float*>(ws + w.delta);
  int32_t* kv_off = reinterpret_cast<int32_t*>(ws + w.kv_off);
  int32_t* cursor = reinterpret_cast<int32_t*>(ws + w.cursor);
  int32_t* kv_idx = reinterpret_cast<int32_t*>(ws + w.kv_idx);
  const CUtensorMapDataType t16 = std::is_same<T, __nv_bfloat16>::value ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                                        : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap tq, tdo, tk, tv;
  if (int rc = tmap_rows(&tq, q, t16, b, l, h, kBQ)) return rc;
  if (int rc = tmap_rows(&tdo, d_o, t16, b, l, h, kBQ)) return rc;
  if (int rc = tmap_rows(&tk, k, t16, b, l, h, BLKK)) return rc;
  if (int rc = tmap_rows(&tv, v, t16, b, l, h, BLKK)) return rc;

  const int64_t rows = b * l * h;
  sla_bwd_delta_kernel<T><<<unsigned(cdiv64(rows, 8)), 256, 0, st>>>(static_cast<const T*>(o_s), static_cast<const T*>(d_o), delta,
                                                                       rows, int(l), int(h), nullptr);
  if (int rc = check_launch("sla_bwd_delta_kernel")) return rc;
  sla_bwd_kmajor_index_kernel<<<unsigned(b * h), kIndexThreads, 0, st>>>(lut, int(mblk), int(nblk), int(topk), kv_off, cursor, kv_idx);
  if (int rc = check_launch("sla_bwd_kmajor_index_kernel")) return rc;

  BwdParams p;
  p.lse = lse;
  p.delta = delta;
  p.lut = lut;
  p.kv_off = kv_off;
  p.kv_idx = kv_idx;
  p.dq = dq;
  p.dk = dk;
  p.dv = dv;
  p.lq = p.lk = int(l);
  p.h = int(h);
  p.mblk = int(mblk);
  p.nblk = int(nblk);
  p.topk = int(topk);
  p.sm_scale = sm_scale;

  constexpr bool kQ64 = kBQ == BLKQ64;
  const auto dq_kern = kQ64 ? sla_bwd_dq_q64_kernel<T> : sla_bwd_dq_kernel<T>;
  const auto dkdv_kern = sla_bwd_dkdv_kernel<T, kBQ>;
  const int threads_dq = kQ64 ? split::kThreads : dq::kThreads;
  const size_t smem_dq = 1024 + (kQ64 ? dq64::kOffLut : dq::kOffLut) + ((size_t(topk) * 2 + 15) & ~size_t(15));
  if (int rc = check_cuda(cudaFuncSetAttribute(dq_kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem_dq)),
                          "cudaFuncSetAttribute(sla_bwd_dq)"))
    return rc;
  dq_kern<<<dim3(unsigned(mblk), unsigned(h), unsigned(b)), threads_dq, smem_dq, st>>>(tq, tdo, tk, tv, p);
  if (int rc = check_launch("sla_bwd_dq_kernel")) return rc;

  const size_t smem_kv = 1024 + Dkv<kBQ>::kSmem;
  if (int rc = check_cuda(cudaFuncSetAttribute(dkdv_kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem_kv)),
                          "cudaFuncSetAttribute(sla_bwd_dkdv)"))
    return rc;
  dkdv_kern<<<dim3(unsigned(nblk), unsigned(h), unsigned(b)), split::kThreads, smem_kv, st>>>(tq, tdo, tk, tv, p);
  return check_launch("sla_bwd_dkdv_kernel");
}

int check_blkq(const char* what, int64_t blkq, int64_t blkk) {
  if ((blkq == BLKQ || blkq == BLKQ64) && blkk == BLKK) return 0;
  return fail(TDB200_ERR_UNSUPPORTED, "%s: block sizes (%lld, %lld) (BLKQ x BLKK = 128 x 64 or 64 x 64)", what, (long long)blkq,
              (long long)blkk);
}

}  // namespace

extern "C" int64_t tdb200_sla_attn16_bwd_workspace_bytes(int64_t b, int64_t h, int64_t l, int64_t topk, int64_t blkq) {
  if (int rc = check_blkq("sla_attn16_bwd_workspace_bytes", blkq, BLKK)) return rc;
  if (b <= 0 || h <= 0 || l <= 0 || topk <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_bwd_workspace_bytes: bad shape");
  return int64_t(ws_layout(b, h, l, topk, blkq).total);
}

// (blkq, blkk) = (128, 64) runs sla_bwd_dq_kernel / sla_bwd_dkdv_kernel<T, 128>, (64, 64) sla_bwd_dq_q64_kernel /
// sla_bwd_dkdv_kernel<T, 64>.
extern "C" int tdb200_sla_attn16_bwd(const void* q, const void* k, const void* v, const void* o_s, const void* d_o, const float* lse,
                                     int dtype, const int32_t* lut, int64_t topk, void* dq, void* dk, void* dv, void* workspace,
                                     int64_t workspace_bytes, int64_t b, int64_t l, int64_t h, int64_t d, float sm_scale,
                                     int64_t blkq, int64_t blkk, void* stream) {
  if (int rc = check_blkq("sla_attn16_bwd", blkq, blkk)) return rc;
  if (!q || !k || !v || !o_s || !d_o || !lse || !lut || !dq || !dk || !dv || !workspace)
    return fail(TDB200_ERR_INVALID_ARG, "sla_attn16_bwd: null pointer");
  if (b <= 0 || l <= 0 || h <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_attn16_bwd: bad shape");
  const int64_t mblk = cdiv64(l, blkq), nblk = cdiv64(l, BLKK);
  if (topk <= 0 || topk > nblk)
    return fail(TDB200_ERR_INVALID_ARG, "sla_attn16_bwd: topk=%lld outside [1, %lld]", (long long)topk, (long long)nblk);
  if (d != HD) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn16_bwd: head dim %lld (this kernel implements d=128)", (long long)d);
  if (dtype != TDB200_DTYPE_BF16 && dtype != TDB200_DTYPE_FP16)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn16_bwd: dtype tag %d", dtype);
  if (nblk > 65535 || h > 65535 || b > 65535 || b * h * mblk * topk > 0x7FFFFFFF)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn16_bwd: dimension too large");
  if (1024 + (blkq == BLKQ ? dq::kOffLut : dq64::kOffLut) + ((size_t(topk) * 2 + 15) & ~size_t(15)) > 227 * 1024)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn16_bwd: topk=%lld too large for on-chip LUT", (long long)topk);
  const int64_t need = int64_t(ws_layout(b, h, l, topk, blkq).total);
  if (workspace_bytes < need)
    return fail(TDB200_ERR_WORKSPACE, "sla_attn16_bwd: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
                (long long)need);
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  // the (128, 64) kernels are instantiated first: nvcc's output for them depends on the order
  if (blkq == BLKQ) {
    if (dtype == TDB200_DTYPE_BF16)
      return launch_bwd<__nv_bfloat16, BLKQ>(q, k, v, o_s, d_o, lse, lut, topk, dq, dk, dv, ws, b, l, h, sm_scale, st);
    return launch_bwd<__half, BLKQ>(q, k, v, o_s, d_o, lse, lut, topk, dq, dk, dv, ws, b, l, h, sm_scale, st);
  }
  if (dtype == TDB200_DTYPE_BF16)
    return launch_bwd<__nv_bfloat16, BLKQ64>(q, k, v, o_s, d_o, lse, lut, topk, dq, dk, dv, ws, b, l, h, sm_scale, st);
  return launch_bwd<__half, BLKQ64>(q, k, v, o_s, d_o, lse, lut, topk, dq, dk, dv, ws, b, l, h, sm_scale, st);
}

extern "C" int64_t tdb200_sla_attn_bwd_workspace_bytes(int64_t b, int64_t h, int64_t l, int64_t topk) {
  return tdb200_sla_attn16_bwd_workspace_bytes(b, h, l, topk, BLKQ);
}

extern "C" int tdb200_sla_attn_bwd_qk16(const void* q, const void* k, const void* v, const void* o_s, const void* d_o, const float* lse,
                                        int dtype, const int32_t* lut, int64_t topk, void* dq, void* dk, void* dv, void* workspace,
                                        int64_t workspace_bytes, int64_t b, int64_t l, int64_t h, int64_t d, float sm_scale,
                                        void* stream) {
  return tdb200_sla_attn16_bwd(q, k, v, o_s, d_o, lse, dtype, lut, topk, dq, dk, dv, workspace, workspace_bytes, b, l, h, d, sm_scale,
                               BLKQ, BLKK, stream);
}

// ------------------------------------------------------------------------------------------------ dense attention
namespace {

// The delta kernel's grid has one 8-row CTA per 8 rows of [b, lq, h], and grid.x stops at 2^31 - 1.
constexpr int64_t kMaxDenseRows = int64_t(8) * 0x7FFFFFFF;

bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }

// delta kernel, then dQ over every key tile and dK / dV over every 128-row query block (no index kernel); kKeyLens: over the
// tiles and key blocks below k_lens[b]; kQueryLens: also over the query rows and blocks below q_lens[b]
template <typename T, bool kKeyLens, bool kQueryLens = false>
int launch_dense_bwd(const void* q, const void* k, const void* v, const void* out, const void* d_out, const float* lse, void* dq,
                     void* dk, void* dv, float* delta, int64_t b, int64_t lq, int64_t lk, const int32_t* q_lens,
                     const int32_t* k_lens, int64_t h, float sm_scale, cudaStream_t st) {
  const CUtensorMapDataType t16 = std::is_same<T, __nv_bfloat16>::value ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                                        : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap tq, tdo, tk, tv;
  if (int rc = tmap_rows(&tq, q, t16, b, lq, h, BLKQ)) return rc;
  if (int rc = tmap_rows(&tdo, d_out, t16, b, lq, h, BLKQ)) return rc;
  if (int rc = tmap_rows(&tk, k, t16, b, lk, h, BLKK)) return rc;
  if (int rc = tmap_rows(&tv, v, t16, b, lk, h, BLKK)) return rc;

  const int64_t rows = b * lq * h;
  sla_bwd_delta_kernel<T, kQueryLens><<<unsigned(cdiv64(rows, 8)), 256, 0, st>>>(
      static_cast<const T*>(out), static_cast<const T*>(d_out), delta, rows, int(lq), int(h), q_lens);
  if (int rc = check_launch("sla_bwd_delta_kernel")) return rc;

  BwdParams p = {};
  p.lse = lse;
  p.delta = delta;
  p.dq = dq;
  p.dk = dk;
  p.dv = dv;
  p.lq = int(lq);
  p.lk = int(lk);
  p.h = int(h);
  p.mblk = int(cdiv64(lq, BLKQ));
  p.nblk = int(cdiv64(lk, BLKK));
  p.topk = p.nblk;
  p.sm_scale = sm_scale;
  p.k_lens = k_lens;
  p.q_lens = q_lens;

  static bool smem_set_dq[64], smem_set_kv[64];
  const auto dq_kern = sla_bwd_dq_kernel<T, true, kKeyLens, kQueryLens>;
  const auto dkdv_kern = sla_bwd_dkdv_kernel<T, BLKQ, true, kKeyLens, kQueryLens>;
  const size_t smem_dq = 1024 + dq::kOffLut, smem_kv = 1024 + Dkv<BLKQ>::kSmem;
  if (int rc = set_max_dynamic_smem_once(reinterpret_cast<const void*>(dq_kern), smem_dq, smem_set_dq, "cudaFuncSetAttribute(dense_bwd_dq)"))
    return rc;
  dq_kern<<<dim3(unsigned(p.mblk), unsigned(h), unsigned(b)), dq::kThreads, smem_dq, st>>>(tq, tdo, tk, tv, p);
  if (int rc = check_launch("sla_bwd_dq_kernel")) return rc;
  if (int rc = set_max_dynamic_smem_once(reinterpret_cast<const void*>(dkdv_kern), smem_kv, smem_set_kv, "cudaFuncSetAttribute(dense_bwd_dkdv)"))
    return rc;
  dkdv_kern<<<dim3(unsigned(p.nblk), unsigned(h), unsigned(b)), split::kThreads, smem_kv, st>>>(tq, tdo, tk, tv, p);
  return check_launch("sla_bwd_dkdv_kernel");
}

}  // namespace

extern "C" int64_t tdb200_attn_dense_bwd_workspace_bytes(int64_t b, int64_t h, int64_t lq) {
  if (b <= 0 || h <= 0 || lq <= 0)
    return fail(TDB200_ERR_INVALID_ARG, "attn_dense_bwd_workspace_bytes: bad shape (b=%lld, h=%lld, lq=%lld)", (long long)b,
                (long long)h, (long long)lq);
  if (b > 65535 || h > 65535 || lq > 0x7FFFFFFF || b * h * lq > kMaxDenseRows)
    return fail(TDB200_ERR_UNSUPPORTED, "attn_dense_bwd_workspace_bytes: dimension too large (b, h <= 65535; b * lq * h <= 8 * (2^31 - 1))");
  return b * h * lq * int64_t(sizeof(float));
}

namespace {

// tdb200_attn_dense_bwd and, key_lens, its _kl twin, and, query_lens (with key_lens), its _vl twin
int dense_bwd(const char* what, const void* q, const void* k, const void* v, const void* out, const void* d_out, const float* lse,
              int dtype, void* dq, void* dk, void* dv, void* workspace, int64_t workspace_bytes, int64_t b, int64_t lq, int64_t lk,
              const int32_t* q_lens, bool query_lens, const int32_t* k_lens, bool key_lens, int64_t h, int64_t d, float sm_scale,
              void* stream) {
  if (!q || !k || !v || !out || !d_out || !lse || !dq || !dk || !dv || !workspace || (key_lens && !k_lens) || (query_lens && !q_lens))
    return fail(TDB200_ERR_INVALID_ARG, "%s: null pointer", what);
  if (int rc = dense_attn_shape(what, b, lq, lk, h, d)) return rc;
  if (!aligned16(q) || !aligned16(k) || !aligned16(v) || !aligned16(out) || !aligned16(d_out) || !aligned16(dq) || !aligned16(dk) ||
      !aligned16(dv))
    return fail(TDB200_ERR_INVALID_ARG, "%s: q, k, v, out, d_out, dq, dk and dv must be 16-byte aligned", what);
  if (!aligned4(lse) || !aligned4(workspace)) return fail(TDB200_ERR_INVALID_ARG, "%s: lse and workspace must be 4-byte aligned", what);
  if (key_lens && !aligned4(k_lens)) return fail(TDB200_ERR_INVALID_ARG, "%s: k_lens must be 4-byte aligned", what);
  if (query_lens && !aligned4(q_lens)) return fail(TDB200_ERR_INVALID_ARG, "%s: q_lens must be 4-byte aligned", what);
  if (int rc = dense_attn_limits(what, dtype, b, lq, lk, h, d)) return rc;
  if (b * lq * h > kMaxDenseRows)
    return fail(TDB200_ERR_UNSUPPORTED, "%s: dimension too large (b * lq * h above 8 * (2^31 - 1), the delta kernel's grid)", what);
  const int64_t need = tdb200_attn_dense_bwd_workspace_bytes(b, h, lq);
  if (workspace_bytes < need)
    return fail(TDB200_ERR_WORKSPACE, "%s: workspace of %lld bytes, %lld needed", what, (long long)workspace_bytes, (long long)need);
  if (int rc = require_sm90()) return rc;
  // Autograd calls a backward from a worker thread of its own, on which no runtime call may yet have made the device's
  // primary context current; the tensor maps are encoded through the driver API, which needs one.
  int dev = 0;
  if (int rc = check_cuda(cudaGetDevice(&dev), "cudaGetDevice")) return rc;
  if (int rc = check_cuda(cudaSetDevice(dev), "cudaSetDevice")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* delta = static_cast<float*>(workspace);
  if (query_lens) {
    if (dtype == TDB200_DTYPE_BF16)
      return launch_dense_bwd<__nv_bfloat16, true, true>(q, k, v, out, d_out, lse, dq, dk, dv, delta, b, lq, lk, q_lens, k_lens, h,
                                                         sm_scale, st);
    return launch_dense_bwd<__half, true, true>(q, k, v, out, d_out, lse, dq, dk, dv, delta, b, lq, lk, q_lens, k_lens, h, sm_scale,
                                                st);
  }
  if (!key_lens) {
    if (dtype == TDB200_DTYPE_BF16)
      return launch_dense_bwd<__nv_bfloat16, false>(q, k, v, out, d_out, lse, dq, dk, dv, delta, b, lq, lk, nullptr, nullptr, h,
                                                    sm_scale, st);
    return launch_dense_bwd<__half, false>(q, k, v, out, d_out, lse, dq, dk, dv, delta, b, lq, lk, nullptr, nullptr, h, sm_scale, st);
  }
  if (dtype == TDB200_DTYPE_BF16)
    return launch_dense_bwd<__nv_bfloat16, true>(q, k, v, out, d_out, lse, dq, dk, dv, delta, b, lq, lk, nullptr, k_lens, h, sm_scale,
                                                 st);
  return launch_dense_bwd<__half, true>(q, k, v, out, d_out, lse, dq, dk, dv, delta, b, lq, lk, nullptr, k_lens, h, sm_scale, st);
}

}  // namespace

extern "C" int tdb200_attn_dense_bwd(const void* q, const void* k, const void* v, const void* out, const void* d_out, const float* lse,
                                     int dtype, void* dq, void* dk, void* dv, void* workspace, int64_t workspace_bytes, int64_t b,
                                     int64_t lq, int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream) {
  return dense_bwd("attn_dense_bwd", q, k, v, out, d_out, lse, dtype, dq, dk, dv, workspace, workspace_bytes, b, lq, lk, nullptr, false,
                   nullptr, false, h, d, sm_scale, stream);
}

extern "C" int tdb200_attn_dense_bwd_kl(const void* q, const void* k, const void* v, const void* out, const void* d_out,
                                        const float* lse, int dtype, void* dq, void* dk, void* dv, void* workspace,
                                        int64_t workspace_bytes, int64_t b, int64_t lq, int64_t lk, const int32_t* k_lens, int64_t h,
                                        int64_t d, float sm_scale, void* stream) {
  return dense_bwd("attn_dense_bwd_kl", q, k, v, out, d_out, lse, dtype, dq, dk, dv, workspace, workspace_bytes, b, lq, lk, nullptr,
                   false, k_lens, true, h, d, sm_scale, stream);
}

extern "C" int tdb200_attn_dense_bwd_vl(const void* q, const void* k, const void* v, const void* out, const void* d_out,
                                        const float* lse, int dtype, void* dq, void* dk, void* dv, void* workspace,
                                        int64_t workspace_bytes, int64_t b, int64_t lq, int64_t lk, const int32_t* q_lens,
                                        const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream) {
  return dense_bwd("attn_dense_bwd_vl", q, k, v, out, d_out, lse, dtype, dq, dk, dv, workspace, workspace_bytes, b, lq, lk, q_lens,
                   true, k_lens, true, h, d, sm_scale, stream);
}
