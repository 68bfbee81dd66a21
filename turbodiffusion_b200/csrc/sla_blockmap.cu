// a7. Block-sparsity map construction (reference: get_block_map, turbodiffusion/SLA/utils.py:55-67).
//   S = T(Qpool . Kpool^T)  (fp32 accumulate, rounded to the 16-bit type like the bf16 matmul at :59)
//   per row keep the `topk` largest scores (torch.topk(sorted=False) semantics as a SET; ties broken towards the lowest
//   block index), emit the 0/1 int8 map (:64-66) and the ascending int32 LUT the attention kernel walks.
//
// One CTA handles kRows pooled query rows: their Q vectors sit in shared memory, every thread streams whole 256-byte
// Kpool rows (L2-resident) and produces kRows scores per key block.  Selection is an exact bitwise radix search on the
// order-preserving 16-bit key of the rounded score (one warp per row, ballot + popc), followed by an index-ordered
// compaction, so the result is deterministic and independent of thread scheduling.
#include "common.cuh"
#include "host_common.h"

namespace {
using namespace tdb;

constexpr int kRows = 8;      // pooled query rows per CTA == warps per CTA
constexpr int kThreads = 256;

template <typename T>
__device__ __forceinline__ uint32_t order_key(float score) {
  // round to T, then map the 16-bit pattern to an unsigned key whose order matches the float order
  const T t = static_cast<T>(score);
  const uint32_t u = *reinterpret_cast<const unsigned short*>(&t);
  return (u & 0x8000u) ? (~u & 0xFFFFu) : (u | 0x8000u);
}

// kVL (tdb200_sla_block_map_vl): batch entry b = bh / h has seq_lens[b] rows (clamped to [0, mblk * blkq], which holds l), so mb = its query
// blocks, nb = its key blocks and tk = topks[b] (clamped to [1, min(nb, topk)], 0 when nb = 0) blocks per row; the score, selection and
// compaction run over those alone, as on the entry by itself.  LUT entries past tk and LUT rows past mb are -1, the map is 0
// past nb and on rows past mb.
template <typename T, int D, bool kVL = false>
__global__ void __launch_bounds__(kThreads) block_map_kernel(const T* __restrict__ q_pool, const T* __restrict__ k_pool,
                                                             int mblk, int nblk, int topk,
                                                             int8_t* __restrict__ sparse_map, int32_t* __restrict__ lut,
                                                             const int32_t* seq_lens = nullptr, const int32_t* topks = nullptr,
                                                             int h = 1, int blkq = 1, int blkk = 1) {
  extern __shared__ uint8_t smem_raw[];
  float* sq = reinterpret_cast<float*>(smem_raw);                          // [kRows][D]
  uint16_t* keys = reinterpret_cast<uint16_t*>(smem_raw + kRows * D * 4);  // [kRows][nblk]
  const int bh = blockIdx.y;
  const int m0 = blockIdx.x * kRows;
  int mb = mblk, nb = nblk, tk = topk;
  if constexpr (kVL) {
    const int len = min(max(__ldg(seq_lens + bh / h), 0), mblk * blkq);
    mb = min(mblk, (len + blkq - 1) / blkq);
    nb = min(nblk, (len + blkk - 1) / blkk);
    tk = min(max(__ldg(topks + bh / h), 1), min(nb, topk));
  }
  const int rows = min(kRows, mb - m0);

  for (int i = threadIdx.x; i < kRows * D; i += kThreads) {
    const int r = i / D, c = i % D;
    sq[i] = (r < rows) ? static_cast<float>(q_pool[(int64_t(bh) * mblk + m0 + r) * D + c]) : 0.f;
  }
  __syncthreads();

  // ---- scores: thread n handles key blocks n, n+256, ...
  for (int n = threadIdx.x; n < nb; n += kThreads) {
    const T* kr = k_pool + (int64_t(bh) * nblk + n) * D;
    float acc[kRows];
#pragma unroll
    for (int r = 0; r < kRows; ++r) acc[r] = 0.f;
#pragma unroll 4
    for (int c = 0; c < D; c += 8) {
      const uint4 raw = *reinterpret_cast<const uint4*>(kr + c);
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
      float kf[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        kf[2 * j] = F16Traits<T>::lo(w[j]);
        kf[2 * j + 1] = F16Traits<T>::hi(w[j]);
      }
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[r] = fmaf(sq[r * D + c + j], kf[j], acc[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < kRows; ++r) keys[r * nblk + n] = static_cast<uint16_t>(order_key<T>(acc[r]));
  }
  __syncthreads();

  // ---- selection: warp w owns row w
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if constexpr (kVL)
    if (w >= rows && w < mblk - m0) {   // a row past the entry's query blocks: an empty selection
      for (int i = lane; i < topk; i += 32) lut[(int64_t(bh) * mblk + m0 + w) * topk + i] = -1;
      for (int n = lane; n < nblk; n += 32) sparse_map[(int64_t(bh) * mblk + m0 + w) * nblk + n] = 0;
      return;
    }
  if (w >= rows) return;
  const uint16_t* kk = keys + w * nblk;
  // largest threshold t such that count(key >= t) >= topk  == the topk-th largest key
  uint32_t thr = 0;
  for (int bit = 15; bit >= 0; --bit) {
    const uint32_t cand = thr | (1u << bit);
    int cnt = 0;
    for (int n = lane; n < nb; n += 32) cnt += (kk[n] >= cand) ? 1 : 0;
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if (cnt >= tk) thr = cand;
  }
  int cnt_gt = 0;
  for (int n = lane; n < nb; n += 32) cnt_gt += (kk[n] > thr) ? 1 : 0;
  cnt_gt = __reduce_add_sync(0xffffffffu, cnt_gt);
  const int need_eq = tk - cnt_gt;  // how many of the threshold-valued blocks to take, lowest index first

  int8_t* map_row = sparse_map + (int64_t(bh) * mblk + m0 + w) * nblk;
  int32_t* lut_row = lut + (int64_t(bh) * mblk + m0 + w) * topk;
  int run_sel = 0, run_eq = 0;
  const uint32_t lt_mask = (1u << lane) - 1u;
  for (int base = 0; base < nb; base += 32) {
    const int n = base + lane;
    const uint32_t key = (n < nb) ? kk[n] : 0u;
    const bool gt = (n < nb) && key > thr;
    const bool eq = (n < nb) && key == thr;
    const uint32_t eq_ballot = __ballot_sync(0xffffffffu, eq);
    const int eq_rank = run_eq + __popc(eq_ballot & lt_mask);
    const bool sel = gt || (eq && eq_rank < need_eq);
    const uint32_t sel_ballot = __ballot_sync(0xffffffffu, sel);
    if (sel) lut_row[run_sel + __popc(sel_ballot & lt_mask)] = n;
    if (n < nb) map_row[n] = sel ? 1 : 0;
    run_sel += __popc(sel_ballot);
    run_eq += __popc(eq_ballot);
  }
  if constexpr (kVL) {
    for (int i = tk + lane; i < topk; i += 32) lut_row[i] = -1;
    for (int n = nb + lane; n < nblk; n += 32) map_row[n] = 0;
  }
}

}  // namespace

extern "C" int tdb200_sla_block_map(const void* q_pool, const void* k_pool, int dtype, int64_t b, int64_t h,
                                    int64_t mblk, int64_t nblk, int64_t d, int64_t topk, int8_t* sparse_map,
                                    int32_t* lut, void* stream) {
  using namespace tdb;
  if (!q_pool || !k_pool || !sparse_map || !lut) return fail(TDB200_ERR_INVALID_ARG, "sla_block_map: null pointer");
  if (b <= 0 || h <= 0 || mblk <= 0 || nblk <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_block_map: bad shape");
  if (topk <= 0 || topk > nblk) return fail(TDB200_ERR_INVALID_ARG, "sla_block_map: topk=%lld outside [1, nblk=%lld]", (long long)topk, (long long)nblk);
  if (d != 64 && d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_block_map: head dim %lld", (long long)d);
  if (b * h > 65535) return fail(TDB200_ERR_UNSUPPORTED, "sla_block_map: b*h too large");
  const size_t smem = size_t(kRows) * d * 4 + size_t(kRows) * nblk * 2;
  if (smem > 200 * 1024) return fail(TDB200_ERR_UNSUPPORTED, "sla_block_map: nblk=%lld too large for the on-chip score rows", (long long)nblk);
  if (!aligned16(k_pool)) return fail(TDB200_ERR_INVALID_ARG, "sla_block_map: k_pool must be 16-byte aligned");
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(static_cast<unsigned>(cdiv64(mblk, kRows)), static_cast<unsigned>(b * h));
#define TDB_BM(T, D)                                                                                             \
  do {                                                                                                           \
    if (smem > 48 * 1024)                                                                                        \
      if (int rc = check_cuda(cudaFuncSetAttribute(block_map_kernel<T, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                                   static_cast<int>(smem)), "cudaFuncSetAttribute(block_map)")) \
        return rc;                                                                                               \
    block_map_kernel<T, D><<<grid, kThreads, smem, st>>>(static_cast<const T*>(q_pool), static_cast<const T*>(k_pool), \
                                                        static_cast<int>(mblk), static_cast<int>(nblk),         \
                                                        static_cast<int>(topk), sparse_map, lut);                \
    return check_launch("block_map_kernel");                                                                     \
  } while (0)
  if (dtype == TDB200_DTYPE_BF16) {
    if (d == 128) TDB_BM(__nv_bfloat16, 128);
    TDB_BM(__nv_bfloat16, 64);
  } else if (dtype == TDB200_DTYPE_FP16) {
    if (d == 128) TDB_BM(__half, 128);
    TDB_BM(__half, 64);
  }
#undef TDB_BM
  return fail(TDB200_ERR_UNSUPPORTED, "sla_block_map: dtype tag %d", dtype);
}

// tdb200_sla_block_map for a padded batch: q_pool [b, h, mblk, d] and k_pool [b, h, nblk, d] of tdb200_sla_quant_qk_vl with the
// same blkq, blkk and seq_lens [b]; topks [b] (device int32) the blocks each of entry b's rows keeps.  Entry b's rows get the
// map and LUT tdb200_sla_block_map gives on that entry alone; the LUT keeps its row stride `topk` (the largest topks[b]).
extern "C" int tdb200_sla_block_map_vl(const void* q_pool, const void* k_pool, int dtype, int64_t b, int64_t h, int64_t mblk,
                                       int64_t nblk, int64_t d, int64_t topk, const int32_t* seq_lens, const int32_t* topks,
                                       int64_t blkq, int64_t blkk, int8_t* sparse_map, int32_t* lut, void* stream) {
  using namespace tdb;
  if (!q_pool || !k_pool || !sparse_map || !lut) return fail(TDB200_ERR_INVALID_ARG, "sla_block_map_vl: null pointer");
  if (!seq_lens || !topks || (reinterpret_cast<uintptr_t>(seq_lens) & 3u) || (reinterpret_cast<uintptr_t>(topks) & 3u))
    return fail(TDB200_ERR_INVALID_ARG, "sla_block_map_vl: seq_lens and topks must be non-null, 4-byte aligned int32 [b]");
  if (b <= 0 || h <= 0 || mblk <= 0 || nblk <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_block_map_vl: bad shape");
  if (!((blkq == 128 && blkk == 64) || (blkq == 64 && (blkk == 64 || blkk == 128))))
    return fail(TDB200_ERR_UNSUPPORTED, "sla_block_map_vl: block sizes (%lld, %lld)", (long long)blkq, (long long)blkk);
  if (topk <= 0 || topk > nblk) return fail(TDB200_ERR_INVALID_ARG, "sla_block_map_vl: topk=%lld outside [1, nblk=%lld]", (long long)topk, (long long)nblk);
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_block_map_vl: head dim %lld (per-entry lengths serve d = 128)", (long long)d);
  if (b * h > 65535) return fail(TDB200_ERR_UNSUPPORTED, "sla_block_map_vl: b*h too large");
  const size_t smem = size_t(kRows) * d * 4 + size_t(kRows) * nblk * 2;
  if (smem > 200 * 1024) return fail(TDB200_ERR_UNSUPPORTED, "sla_block_map_vl: nblk=%lld too large for the on-chip score rows", (long long)nblk);
  if (!aligned16(k_pool)) return fail(TDB200_ERR_INVALID_ARG, "sla_block_map_vl: k_pool must be 16-byte aligned");
  if (dtype != TDB200_DTYPE_BF16 && dtype != TDB200_DTYPE_FP16) return fail(TDB200_ERR_UNSUPPORTED, "sla_block_map_vl: dtype tag %d", dtype);
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(static_cast<unsigned>(cdiv64(mblk, kRows)), static_cast<unsigned>(b * h));
#define TDB_BM(T)                                                                                                  \
  do {                                                                                                             \
    if (smem > 48 * 1024)                                                                                          \
      if (int rc = check_cuda(cudaFuncSetAttribute(block_map_kernel<T, 128, true>,                                 \
                                                   cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)), \
                              "cudaFuncSetAttribute(block_map_vl)"))                                               \
        return rc;                                                                                                 \
    block_map_kernel<T, 128, true><<<grid, kThreads, smem, st>>>(                                                 \
        static_cast<const T*>(q_pool), static_cast<const T*>(k_pool), static_cast<int>(mblk), static_cast<int>(nblk), \
        static_cast<int>(topk), sparse_map, lut, seq_lens, topks, static_cast<int>(h), static_cast<int>(blkq),     \
        static_cast<int>(blkk));                                                                                   \
    return check_launch("block_map_kernel<vl>");                                                                   \
  } while (0)
  if (dtype == TDB200_DTYPE_BF16) TDB_BM(__nv_bfloat16);
  TDB_BM(__half);
#undef TDB_BM
}
