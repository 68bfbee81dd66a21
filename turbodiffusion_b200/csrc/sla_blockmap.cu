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

template <typename T, int D>
__global__ void __launch_bounds__(kThreads) block_map_kernel(const T* __restrict__ q_pool, const T* __restrict__ k_pool,
                                                             int mblk, int nblk, int topk,
                                                             int8_t* __restrict__ sparse_map, int32_t* __restrict__ lut) {
  extern __shared__ uint8_t smem_raw[];
  float* sq = reinterpret_cast<float*>(smem_raw);                          // [kRows][D]
  uint16_t* keys = reinterpret_cast<uint16_t*>(smem_raw + kRows * D * 4);  // [kRows][nblk]
  const int bh = blockIdx.y;
  const int m0 = blockIdx.x * kRows;
  const int rows = min(kRows, mblk - m0);

  for (int i = threadIdx.x; i < kRows * D; i += kThreads) {
    const int r = i / D, c = i % D;
    sq[i] = (r < rows) ? static_cast<float>(q_pool[(int64_t(bh) * mblk + m0 + r) * D + c]) : 0.f;
  }
  __syncthreads();

  // ---- scores: thread n handles key blocks n, n+256, ...
  for (int n = threadIdx.x; n < nblk; n += kThreads) {
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
  if (w >= rows) return;
  const uint16_t* kk = keys + w * nblk;
  // largest threshold t such that count(key >= t) >= topk  == the topk-th largest key
  uint32_t thr = 0;
  for (int bit = 15; bit >= 0; --bit) {
    const uint32_t cand = thr | (1u << bit);
    int cnt = 0;
    for (int n = lane; n < nblk; n += 32) cnt += (kk[n] >= cand) ? 1 : 0;
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if (cnt >= topk) thr = cand;
  }
  int cnt_gt = 0;
  for (int n = lane; n < nblk; n += 32) cnt_gt += (kk[n] > thr) ? 1 : 0;
  cnt_gt = __reduce_add_sync(0xffffffffu, cnt_gt);
  const int need_eq = topk - cnt_gt;  // how many of the threshold-valued blocks to take, lowest index first

  int8_t* map_row = sparse_map + (int64_t(bh) * mblk + m0 + w) * nblk;
  int32_t* lut_row = lut + (int64_t(bh) * mblk + m0 + w) * topk;
  int run_sel = 0, run_eq = 0;
  const uint32_t lt_mask = (1u << lane) - 1u;
  for (int base = 0; base < nblk; base += 32) {
    const int n = base + lane;
    const uint32_t key = (n < nblk) ? kk[n] : 0u;
    const bool gt = (n < nblk) && key > thr;
    const bool eq = (n < nblk) && key == thr;
    const uint32_t eq_ballot = __ballot_sync(0xffffffffu, eq);
    const int eq_rank = run_eq + __popc(eq_ballot & lt_mask);
    const bool sel = gt || (eq && eq_rank < need_eq);
    const uint32_t sel_ballot = __ballot_sync(0xffffffffu, sel);
    if (sel) lut_row[run_sel + __popc(sel_ballot & lt_mask)] = n;
    if (n < nblk) map_row[n] = sel ? 1 : 0;
    run_sel += __popc(sel_ballot);
    run_eq += __popc(eq_ballot);
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
