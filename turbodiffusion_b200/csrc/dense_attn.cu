// Dense softmax attention forward, out = softmax(q.k^T * sm_scale).v, for 16-bit q [b, lq, h, d] and k, v [b, lk, h, d] read
// in place through 4-D TMA tensor maps (the cross-attention over the text tokens, and the dense baseline of the SLA kernels).
//   reference: the 'original' attention of rcm/utils/attention.py:120-167 (F.scaled_dot_product_attention / FlashAttention).
// The arithmetic is the 16-bit SLA kernel's, step for step (sla_attn.cuh): S by wgmma into fp32, scores scaled by
// sm_scale * log2e, exp2 online softmax with the lazy rescale, the row sum from the unrounded P, P rounded to T as the register
// A operand of P.V, fp32 accumulation, out = T(O / l).
//
// One CTA per (128-row query block, head, batch): a producer warpgroup (one thread issues the TMA loads; setmaxnreg hands its
// registers to the consumers) and two consumer warpgroups, warpgroup g owning query rows [64g, 64g + 64) of the block.  What the
// sparse kernels carry and dense attention does not need is gone: key blocks are visited in order, so there is no LUT in shared
// memory and no LUT read in the producer, no KVW tile and no linear-branch epilogue.  The shared memory that frees goes to
// 128-row key tiles (wgmma.m64n128k16 scores: half the softmax rounds and barrier trips of a 64-row tile, which needs the
// 232 registers setmaxnreg gives a consumer thread: O 64 + S 64 + P 32) on a 3-stage K ring and a 3-stage V ring:
// Q 32 KB + 3 x (K 32 KB + V 32 KB) = 224 KB.  128 query rows per CTA, not 64: K and V do not fit on chip next to Q
// (128 KB each per head at lk = 512), so every CTA streams all of K and V from L2, and 128 rows halve that traffic per FLOP.
// Key columns >= lk are masked to -inf (their K and V rows are TMA zero fill, whatever memory holds there) and query rows >= lq
// are not stored, so lq and lk need not be multiples of anything.  Every output row is written by one warpgroup that visits the
// key tiles in ascending order: no atomics, and the bits of a (batch, head) depend only on its own q, k, v.
#include <type_traits>

#include "sla_attn.cuh"
#include "host_common.h"

namespace {
using namespace tdb;

constexpr int HD = 128, BQ = 128, BK = 128;
constexpr int kStages = 3;
constexpr int kConsumerWarps = 8;
constexpr uint32_t kQBytes = BQ * HD * 2;      // HD/64 chunks of [BQ rows x 128 B]
constexpr uint32_t kTileBytes = BK * HD * 2;   // K and V alike: HD/64 chunks of [BK keys x 128 B]
constexpr uint32_t kOffQ = 0;
constexpr uint32_t kOffK = kOffQ + kQBytes;
constexpr uint32_t kOffV = kOffK + kStages * kTileBytes;
constexpr uint32_t kOffBars = kOffV + kStages * kTileBytes;
constexpr size_t kSmemBytes = 1024 + kOffBars + 256;   // 1024: the tiles are aligned inside the dynamic allocation
static_assert(kSmemBytes <= 227 * 1024, "shared memory of the dense attention kernel");

// both warpgroups consume every tile, so a slot has one full barrier and its empty barrier counts their eight warps
enum Bar { kQFull = 0, kKFull = 1, kKEmpty = kKFull + kStages, kVFull = kKEmpty + kStages, kVEmpty = kVFull + kStages,
           kNumBars = kVEmpty + kStages };
static_assert(kNumBars * 8 <= 256, "barriers exceed their shared-memory slot");

struct DenseParams {
  void* out;    // [b, lq, h, d] T
  float* lse;   // [b, h, lq] fp32, log2 domain (kLse only)
  int lq, lk, h;
  float sm_scale;
  const int32_t* k_lens = nullptr;   // [b] int32 (kKeyLens only)
  const int32_t* q_lens = nullptr;   // [b] int32 (kQueryLens only)
};

// kLse: also lse[b, h, row] = m_used + log2(l), the row log-sum-exp of the scores in the log2 domain with m_used the maximum the
// lazy rescale last used (tdb200_sla_attn16_fwd_lse's convention), for the backward (sla_attn_bwd.cu) to recompute P from.
// kKeyLens: batch entry b attends to its first lk_b = keys_of(k_lens, lk, b) keys only; tiles past them are neither loaded nor
// visited, the last tile's rows past them are zeroed (zero_key_rows), and a row with no keys (lk_b = 0) stores out = 0 and
// lse = +inf, the convention of rows past lq.
// kQueryLens: batch entry b owns its first lq_b = queries_of(q_lens, lq, b) query rows only; rows past them store out = 0 and
// lse = +inf (assigned, not scaled: their q rows may hold inf or NaN), and a CTA whose block lies wholly past lq_b loads
// nothing and only stores those rows.  Rows do not mix in the forward, so the straddling block needs nothing more.
template <typename T, bool kLse, bool kKeyLens = false, bool kQueryLens = false>
__global__ void __launch_bounds__(split::kThreads, 1)
dense_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                      const __grid_constant__ CUtensorMap tmap_v, DenseParams p) {
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, stays a shared-space pointer
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBars);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  const int lk = keys_of<kKeyLens>(p.k_lens, p.lk, b);
  const int lq = queries_of<kQueryLens>(p.q_lens, p.lq, b);
  const bool idle = kQueryLens && m_blk * BQ >= lq;   // the block lies wholly past the entry's queries
  const int n_tiles = idle ? 0 : (lk + BK - 1) / BK;

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
  __syncthreads();

  if (warp >= kConsumerWarps) {
    // =============================================================== TMA producer
    reg_dealloc<split::kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0 && !idle) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
      mbar_expect_tx(&bars[kQFull], kQBytes);
#pragma unroll
      for (int c = 0; c < HD / 64; ++c)
        tma_load_4d(smem + kOffQ + c * (BQ * 128), &tmap_q, &bars[kQFull], c * 64, hh, m_blk * BQ, b);
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j % kStages;
        const uint32_t ph = ((j / kStages) & 1) ^ 1;
        mbar_wait(&bars[kKEmpty + st], ph);
        mbar_expect_tx(&bars[kKFull + st], kTileBytes);
        uint8_t* sk = smem + kOffK + st * kTileBytes;
#pragma unroll
        for (int c = 0; c < HD / 64; ++c) tma_load_4d(sk + c * (BK * 128), &tmap_k, &bars[kKFull + st], c * 64, hh, j * BK, b);
        mbar_wait(&bars[kVEmpty + st], ph);
        mbar_expect_tx(&bars[kVFull + st], kTileBytes);
        uint8_t* sv = smem + kOffV + st * kTileBytes;
#pragma unroll
        for (int c = 0; c < HD / 64; ++c) tma_load_4d(sv + c * (BK * 128), &tmap_v, &bars[kVFull + st], c * 64, hh, j * BK, b);
      }
    }
    return;
  }

  // =============================================================== consumer warpgroups (64 query rows each, every key tile)
  reg_alloc<split::kConsumerRegs>();
  const int wg = warp >> 2, w4 = warp & 3;
  const int r_lo = wg * 64 + w4 * 16 + (lane >> 2);   // rows r_lo and r_lo + 8 of the block (fragment layout, common.cuh)
  const int cq = 2 * (lane & 3);                       // column pair offset inside every 8-column slice
  const uint32_t sbase = smem_u32(smem);
  const float sc = p.sm_scale * kLog2e;

  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_used[2] = {-INFINITY, -INFINITY}, l_part[2] = {0.f, 0.f};  // l_part: this thread's columns of the row sum

  if (!idle) mbar_wait(&bars[kQFull], 0);
  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % kStages;
    const uint32_t ph = (j / kStages) & 1;

    float s[BK / 2];
    mbar_wait(&bars[kKFull + st], ph);
    if constexpr (kKeyLens)
      if (lk - j * BK < BK && lk < p.lk) {   // the last tile, with rows past the entry's keys inside the buffer
        mbar_wait(&bars[kVFull + st], ph);
        zero_key_rows(smem + kOffK + st * kTileBytes, BK, HD / 64, lk - j * BK, threadIdx.x);
        zero_key_rows(smem + kOffV + st * kTileBytes, BK, HD / 64, lk - j * BK, threadIdx.x);
        fence_proxy_async_smem();
        named_bar_sync(1, kConsumerWarps * 32);
      }
    score_tile<true, HD, BK, kBF16>(s, sbase + kOffQ + wg * (64 * 128), BQ * 128, sbase + kOffK + st * kTileBytes, sc);
    warp_release(&bars[kKEmpty + st], lane);
    uint32_t pa[BK / 16][4];
    softmax_step<T, HD, BK>(s, o, m_used, l_part, pa, lk - j * BK, cq, j == 0);   // valid < BK only in the ragged last tile
    mbar_wait(&bars[kVFull + st], ph);
    pv_step<HD, BK, kBF16>(o, pa, sbase + kOffV + st * kTileBytes);
    warp_release(&bars[kVEmpty + st], lane);
  }

#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float l_tot = quad_sum(l_part[h]);   // all four lanes of a row take part, stored or not
    const int64_t qr = int64_t(m_blk) * BQ + r_lo + 8 * h;
    if (qr >= p.lq) continue;
    const bool pad = kQueryLens && qr >= lq;   // a row past the entry's queries
    if (pad) zero_o_row(o, h);
    const bool empty = (kKeyLens && lk == 0) || pad;   // o = 0 and l = 0: store 0 * 0 and lse = +inf
    if constexpr (kLse)
      if (cq == 0) p.lse[(int64_t(b) * p.h + hh) * p.lq + qr] = empty ? INFINITY : m_used[h] + __log2f(l_tot);
    store_o_row<T, HD>(static_cast<T*>(p.out) + ((int64_t(b) * p.lq + qr) * p.h + hh) * HD, o, h, empty ? 0.f : 1.0f / l_tot, cq);
  }
}

template <typename T, bool kLse, bool kKeyLens, bool kQueryLens = false>
int launch(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const DenseParams& p, dim3 grid, cudaStream_t st) {
  static bool smem_set[64];
  const auto kern = dense_attn_fwd_kernel<T, kLse, kKeyLens, kQueryLens>;
  if (int rc = set_max_dynamic_smem_once(reinterpret_cast<const void*>(kern), kSmemBytes, smem_set, "cudaFuncSetAttribute(dense_attn)"))
    return rc;
  kern<<<grid, split::kThreads, kSmemBytes, st>>>(tq, tk, tv, p);
  return check_launch("dense_attn_fwd_kernel");
}

// ---------------------------------------------------------------------------------------------------------------------------
// Forward-mode derivative (JVP): o = softmax(S).v and its tangent od for tangents qd, kd, vd of q, k, v, with S = c q.k^T and
// Sd = c (qd.k^T + q.kd^T), c = sm_scale:
//   od = sum_j P_j Sd_j v_j - (sum_j P_j Sd_j) o + P.vd.
// With the online softmax and p = exp2(s - m) unnormalised, each warpgroup row keeps l = sum p and O = sum p v as the forward
// does, plus A = sum p (Sd v + vd) and mu = sum p Sd; the lazy rescale scales all four, and at the end o = O / l and
// od = (A - (mu / l) O) / l.  Per 64-key tile: S by wgmma and the softmax, which leaves p in fp32 in S's registers; then Sd as
// one commit group (O 64 + A 64 + p 32 + Sd 32 fp32 registers per thread at the peak; issuing S and Sd together so that the
// softmax overlaps Sd's MMAs spilled); l and mu sum the unrounded p and p Sd, the tensor core gets p and
// p Sd rounded to T; then O += P.V, A += (P Sd).V and A += P.Vd as one commit group.
// CTA per (128-row query block, head, batch), the forward's warp roles.  Shared memory: Q and Qd resident (64 KB), a 2-stage
// (K, Kd) ring and a 2-stage (V, Vd) ring of 32 KB per stage: 192 KB.  A third stage of both rings would need 256 KB.
// kSparse (tdb200_sla_attn16_jvp): the same kernel over the key blocks lut[b, h, m, :] lists, in list order, instead of tiles
// 0 .. ceil(lk / 64) - 1; the 64-key tile is the SLA key block (BLKK = 64), the 128-row query block its BLKQ = 128.  The LUT row
// is staged in shared memory behind the barriers (4 * topk bytes) and the producer and the consumers read the same ids from it;
// keys are masked by their absolute column, blk * 64 + c >= lk.  Only the source of the tile index changes, so on an ascending
// LUT listing every key block the sparse kernel computes the dense one's bits.
namespace jvp {
constexpr int BK = 64;
constexpr int kStages = 2;
constexpr uint32_t kQBytes = BQ * HD * 2;           // Q and Qd alike
constexpr uint32_t kHalfBytes = BK * HD * 2;        // one of K, Kd, V, Vd: HD/64 chunks of [BK keys x 128 B]
constexpr uint32_t kStageBytes = 2 * kHalfBytes;    // (K, Kd) or (V, Vd)
constexpr uint32_t kOffQ = 0, kOffQd = kQBytes;
constexpr uint32_t kOffK = 2 * kQBytes;
constexpr uint32_t kOffV = kOffK + kStages * kStageBytes;
constexpr uint32_t kOffBars = kOffV + kStages * kStageBytes;
constexpr size_t kSmemBytes = 1024 + kOffBars + 256;
static_assert(kSmemBytes <= 227 * 1024, "shared memory of the dense attention JVP kernel");
constexpr uint32_t kOffLut = kOffBars + 256;                        // kSparse: the CTA's LUT row, int32 [topk]
constexpr size_t kSparseSmemMax = 227 * 1024;
constexpr int64_t kMaxLutIds = (kSparseSmemMax - kSmemBytes) / 4;   // 8640 ids: topk of any l up to 552,960 keys

enum Bar { kQFull = 0, kKFull = 1, kKEmpty = kKFull + kStages, kVFull = kKEmpty + kStages, kVEmpty = kVFull + kStages,
           kNumBars = kVEmpty + kStages };
static_assert(kNumBars * 8 <= 256, "barriers exceed their shared-memory slot");

struct Params {
  void* out;     // [b, lq, h, d] T
  void* out_t;   // [b, lq, h, d] T
  float* lse;    // [b, h, lq] fp32, log2 domain (kLse only)
  int lq, lk, h;
  float sm_scale;
  const int32_t* lut;   // [b, h, mblk, topk] key-block ids (kSparse only)
  int topk, mblk;
  const int32_t* k_lens = nullptr;   // [b] int32 (kKeyLens only)
  const int32_t* q_lens = nullptr;   // [b] int32 (kQueryLens only)
};

// d (+)= Q.K^T over one 64-key tile: Q rows at sq (HD/64 chunks kQBytes/2 apart), K at sk (chunks BK * 128 bytes apart)
template <bool kBF16>
__device__ __forceinline__ void qk_mmas(float (&d)[BK / 2], uint32_t sq, uint32_t sk, bool accumulate) {
#pragma unroll
  for (int ks = 0; ks < HD / 16; ++ks) {
    const uint64_t qd = make_desc_kmajor_sw128(sq + (ks >> 2) * (BQ * 128)) + uint64_t((ks & 3) * 2);
    const uint64_t kd = make_desc_kmajor_sw128(sk + (ks >> 2) * (BK * 128)) + uint64_t((ks & 3) * 2);
    wgmma_f16_ss<BK, kBF16>(d, qd, kd, (accumulate || ks > 0) ? 1u : 0u);
  }
}

// softmax_step's masking, maxima and lazy rescale, with A and mu rescaled beside O and l; leaves p = exp2(s - m_used) in s.
// kRunMax (fp16): also m_run, the row's running maximum, for the overflow rescale of dense_attn_jvp_kernel.
template <bool kRunMax>
__device__ __forceinline__ void softmax_step_jvp(float (&s)[BK / 2], float (&o)[HD / 2], float (&a)[HD / 2], float (&m_used)[2],
                                                 float (&m_run)[2], float (&l_part)[2], float (&mu_part)[2], int valid, int cq,
                                                 bool first) {
  if (valid < BK) {
#pragma unroll
    for (int i = 0; i < BK / 2; ++i)
      if (8 * (i >> 2) + cq + (i & 1) >= valid) s[i] = -INFINITY;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < BK / 2; ++i)
      if (((i >> 1) & 1) == h) mx = fmaxf(mx, s[i]);
    mx = quad_max(mx);
    if (first) {
      m_used[h] = mx;
    } else if (mx > m_used[h] + kRescaleThreshold) {
      const float alpha = fast_exp2(m_used[h] - mx);
#pragma unroll
      for (int i = 0; i < HD / 2; ++i)
        if (((i >> 1) & 1) == h) {
          o[i] *= alpha;
          a[i] *= alpha;
        }
      l_part[h] *= alpha;
      mu_part[h] *= alpha;
      m_used[h] = mx;
    }
    if constexpr (kRunMax) m_run[h] = first ? mx : fmaxf(m_run[h], mx);
  }
#pragma unroll
  for (int i = 0; i < BK / 2; i += 2) {
    const int h = (i >> 1) & 1;
    s[i] = fast_exp2(s[i] - m_used[h]);
    s[i + 1] = fast_exp2(s[i + 1] - m_used[h]);
    l_part[h] += s[i] + s[i + 1];
  }
}

// kLse: also the row lse of the primal, as dense_attn_fwd_kernel<T, true> stores it.  kKeyLens (dense only): the forward's, so
// a row with no keys also stores out_t = 0, and the ragged last tile's rows past the entry's keys (K, K_t, V and V_t) are zeroed.
// kQueryLens (dense only): the forward's, so a row past the entry's queries also stores out_t = 0.
template <typename T, bool kLse, bool kSparse = false, bool kKeyLens = false, bool kQueryLens = false>
__global__ void __launch_bounds__(split::kThreads, 1)
dense_attn_jvp_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                      const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_qt,
                      const __grid_constant__ CUtensorMap tmap_kt, const __grid_constant__ CUtensorMap tmap_vt, Params p) {
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBars);
  int32_t* s_lut = reinterpret_cast<int32_t*>(smem + kOffLut);   // kSparse only

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  const int lk = keys_of<kKeyLens>(p.k_lens, p.lk, b);
  // the block lies wholly past the entry's queries (the epilogue reads the length again rather than hold it in a register)
  const bool idle = kQueryLens && m_blk * BQ >= queries_of<kQueryLens>(p.q_lens, p.lq, b);
  const int n_tiles = idle ? 0 : kSparse ? p.topk : (lk + BK - 1) / BK;

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
  if constexpr (kSparse) {
    const int32_t* lut_row = p.lut + ((int64_t(b) * p.h + hh) * p.mblk + m_blk) * p.topk;
    for (int i = threadIdx.x; i < p.topk; i += split::kThreads) s_lut[i] = __ldg(lut_row + i);
  }
  __syncthreads();

  if (warp >= kConsumerWarps) {
    // =============================================================== TMA producer
    reg_dealloc<split::kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0 && !idle) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_qt);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_kt);
      tma_prefetch_desc(&tmap_v);
      tma_prefetch_desc(&tmap_vt);
      mbar_expect_tx(&bars[kQFull], 2 * kQBytes);
#pragma unroll
      for (int c = 0; c < HD / 64; ++c) {
        tma_load_4d(smem + kOffQ + c * (BQ * 128), &tmap_q, &bars[kQFull], c * 64, hh, m_blk * BQ, b);
        tma_load_4d(smem + kOffQd + c * (BQ * 128), &tmap_qt, &bars[kQFull], c * 64, hh, m_blk * BQ, b);
      }
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j % kStages;
        const uint32_t ph = ((j / kStages) & 1) ^ 1;
        const int key0 = (kSparse ? s_lut[j] : j) * BK;
        mbar_wait(&bars[kKEmpty + st], ph);
        mbar_expect_tx(&bars[kKFull + st], kStageBytes);
        uint8_t* sk = smem + kOffK + st * kStageBytes;
#pragma unroll
        for (int c = 0; c < HD / 64; ++c) {
          tma_load_4d(sk + c * (BK * 128), &tmap_k, &bars[kKFull + st], c * 64, hh, key0, b);
          tma_load_4d(sk + kHalfBytes + c * (BK * 128), &tmap_kt, &bars[kKFull + st], c * 64, hh, key0, b);
        }
        mbar_wait(&bars[kVEmpty + st], ph);
        mbar_expect_tx(&bars[kVFull + st], kStageBytes);
        uint8_t* sv = smem + kOffV + st * kStageBytes;
#pragma unroll
        for (int c = 0; c < HD / 64; ++c) {
          tma_load_4d(sv + c * (BK * 128), &tmap_v, &bars[kVFull + st], c * 64, hh, key0, b);
          tma_load_4d(sv + kHalfBytes + c * (BK * 128), &tmap_vt, &bars[kVFull + st], c * 64, hh, key0, b);
        }
      }
    }
    return;
  }

  // =============================================================== consumer warpgroups (64 query rows each, every key tile)
  reg_alloc<split::kConsumerRegs>();
  const int wg = warp >> 2, w4 = warp & 3;
  const int r_lo = wg * 64 + w4 * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sq = sbase + kOffQ + wg * (64 * 128), sqd = sbase + kOffQd + wg * (64 * 128);
  const float sc = p.sm_scale * kLog2e;

  float o[HD / 2], a[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = a[i] = 0.f;
  float m_used[2] = {-INFINITY, -INFINITY}, m_run[2], l_part[2] = {0.f, 0.f}, mu_part[2] = {0.f, 0.f};

  if (!idle) mbar_wait(&bars[kQFull], 0);
  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % kStages;
    const uint32_t ph = (j / kStages) & 1;
    const uint32_t sk = sbase + kOffK + st * kStageBytes, sv = sbase + kOffV + st * kStageBytes;

    float s[BK / 2], sd[BK / 2];
    mbar_wait(&bars[kKFull + st], ph);
    if constexpr (kKeyLens)
      if (lk - j * BK < BK && lk < p.lk) {   // the last tile, with rows past the entry's keys inside the buffer
        mbar_wait(&bars[kVFull + st], ph);
        uint8_t* const tiles[4] = {smem + kOffK + st * kStageBytes, smem + kOffK + st * kStageBytes + kHalfBytes,
                                   smem + kOffV + st * kStageBytes, smem + kOffV + st * kStageBytes + kHalfBytes};
#pragma unroll
        for (uint8_t* t : tiles) zero_key_rows(t, BK, HD / 64, lk - j * BK, threadIdx.x);
        fence_proxy_async_smem();
        named_bar_sync(1, kConsumerWarps * 32);
      }
    score_tile<true, HD, BK, kBF16>(s, sq, BQ * 128, sk, sc);
    softmax_step_jvp<!kBF16>(s, o, a, m_used, m_run, l_part, mu_part, lk - (kSparse ? s_lut[j] : j) * BK, cq,
                             j == 0);   // s := p
#pragma unroll
    for (int i = 0; i < BK / 2; ++i) sd[i] = 0.f;
    wgmma_fence();
    qk_mmas<kBF16>(sd, sqd, sk, false);               // Sd / c = Qd.K^T + Q.Kd^T
    qk_mmas<kBF16>(sd, sq, sk + kHalfBytes, true);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(sd);
    warp_release(&bars[kKEmpty + st], lane);

    // fp16: p reaches 2^kRescaleThreshold between lazy rescales, so p * Sd rounded to fp16 overflows from |Sd| ~ 256 on, where
    // the normalised P * Sd is still far inside fp16's range.  In a row where some |p * Sd| of the tile would round to inf, the
    // kernel rescales O, A, l and mu onto the running maximum first (a rescale the lazy rule skipped): then p <= 1 and
    // |p * Sd| <= |Sd|, P * Sd's range.  Other rows, and every row of an input whose tangent did not overflow, keep their bits.
    if constexpr (!kBF16) {
#pragma unroll
      for (int i = 0; i < BK / 2; ++i) sd[i] = s[i] * (sd[i] * p.sm_scale);   // sd := p * Sd, Sd in natural-log units
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float xm = 0.f;
#pragma unroll
        for (int i = 0; i < BK / 2; ++i)
          if (((i >> 1) & 1) == h) xm = fmaxf(xm, fabsf(sd[i]));
        if (quad_max(xm) > 65504.0f) {
          const float alpha = fast_exp2(m_used[h] - m_run[h]);
#pragma unroll
          for (int i = 0; i < HD / 2; ++i)
            if (((i >> 1) & 1) == h) {
              o[i] *= alpha;
              a[i] *= alpha;
            }
#pragma unroll
          for (int i = 0; i < BK / 2; ++i)
            if (((i >> 1) & 1) == h) {
              s[i] *= alpha;
              sd[i] *= alpha;
            }
          l_part[h] *= alpha;   // this tile's p are already in it
          mu_part[h] *= alpha;
          m_used[h] = m_run[h];
        }
      }
    }
    uint32_t pa[BK / 16][4], pda[BK / 16][4];        // P and P * Sd rounded to T: the A operands of the products
#pragma unroll
    for (int i = 0; i < BK / 2; i += 2) {
      const int h = (i >> 1) & 1;
      const float x0 = kBF16 ? s[i] * (sd[i] * p.sm_scale) : sd[i];   // Sd in natural-log units
      const float x1 = kBF16 ? s[i + 1] * (sd[i + 1] * p.sm_scale) : sd[i + 1];
      mu_part[h] += x0 + x1;
      pa[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(s[i], s[i + 1]);
      pda[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(x0, x1);
    }

    mbar_wait(&bars[kVFull + st], ph);
    const uint64_t vdesc = make_desc_mnmajor_sw128(sv, BK * 128), vddesc = make_desc_mnmajor_sw128(sv + kHalfBytes, BK * 128);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) wgmma_f16_rs<HD, kBF16, 1>(o, pa[kk], vdesc + uint64_t(kk * 128));
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) wgmma_f16_rs<HD, kBF16, 1>(a, pda[kk], vdesc + uint64_t(kk * 128));
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) wgmma_f16_rs<HD, kBF16, 1>(a, pa[kk], vddesc + uint64_t(kk * 128));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    reg_fence(a);
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) {
      reg_fence(pa[kk]);
      reg_fence(pda[kk]);
    }
    warp_release(&bars[kVEmpty + st], lane);
  }

  const int lq = queries_of<kQueryLens>(p.q_lens, p.lq, b);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float l_tot = quad_sum(l_part[h]), mu_tot = quad_sum(mu_part[h]);   // all four lanes of a row take part
    const int64_t qr = int64_t(m_blk) * BQ + r_lo + 8 * h;
    if (qr >= p.lq) continue;
    const int64_t row = ((int64_t(b) * p.lq + qr) * p.h + hh) * HD;
    const bool pad = kQueryLens && qr >= lq;   // a row past the entry's queries: o = a = mu = 0, assigned
    if (pad) {
      zero_o_row(o, h);
      zero_o_row(a, h);
    }
    const bool empty = (kKeyLens && lk == 0) || pad;   // o = a = 0 and l = mu = 0: store zeros and lse = +inf
    if constexpr (kLse)
      if (cq == 0) p.lse[(int64_t(b) * p.h + hh) * p.lq + qr] = empty ? INFINITY : m_used[h] + __log2f(l_tot);
    const float inv_l = empty ? 0.f : 1.0f / l_tot, mu_l = pad ? 0.f : mu_tot * inv_l;
    store_o_row<T, HD>(static_cast<T*>(p.out) + row, o, h, inv_l, cq);
    T* trow = static_cast<T*>(p.out_t) + row;
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      const int i = 4 * c + 2 * h;
      *reinterpret_cast<uint32_t*>(trow + 8 * c + cq) =
          F16Traits<T>::pack(fmaf(-mu_l, o[i], a[i]) * inv_l, fmaf(-mu_l, o[i + 1], a[i + 1]) * inv_l);
    }
  }
}

template <typename T, bool kLse, bool kKeyLens, bool kQueryLens = false>
int launch(const CUtensorMap (&tm)[6], const Params& p, dim3 grid, cudaStream_t st) {
  static bool smem_set[64];
  const auto kern = dense_attn_jvp_kernel<T, kLse, false, kKeyLens, kQueryLens>;
  if (int rc = set_max_dynamic_smem_once(reinterpret_cast<const void*>(kern), kSmemBytes, smem_set, "cudaFuncSetAttribute(dense_attn_jvp)"))
    return rc;
  kern<<<grid, split::kThreads, kSmemBytes, st>>>(tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], p);
  return check_launch("dense_attn_jvp_kernel");
}

// kSparse: the dynamic shared memory grows by the LUT row, so the attribute is set once to the largest size any topk may use
template <typename T, bool kLse>
int launch_sparse(const CUtensorMap (&tm)[6], const Params& p, dim3 grid, cudaStream_t st) {
  static bool smem_set[64];
  const auto kern = dense_attn_jvp_kernel<T, kLse, true>;
  if (int rc = set_max_dynamic_smem_once(reinterpret_cast<const void*>(kern), kSparseSmemMax, smem_set,
                                         "cudaFuncSetAttribute(sla_attn16_jvp)"))
    return rc;
  kern<<<grid, split::kThreads, kSmemBytes + 4 * size_t(p.topk), st>>>(tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], p);
  return check_launch("sla_attn16_jvp_kernel");
}

// ---------------------------------------------------------------------------------------------------------------------------
// Tangent alone, from the primal's saved out and lse (tdb200_attn_dense_tangent, tdb200_sla_attn16_tangent): the forward-AD rule
// of the attention operators, whose primal the lse forward has already computed.  lse being the row's log-sum-exp of the
// log2-domain scores, P = exp2(s - lse) is the normalised softmax itself, so there is no online softmax and no rescale:
//   od = (P o Sd).V + P.Vd - rowsum(P o Sd) out.
// Per 64-key tile: S, P (keys >= lk masked), Sd as one commit group; mu sums the unrounded P Sd, the tensor core gets P and
// P Sd rounded to T; then A += (P Sd).V + P.Vd as one commit group.  The epilogue reads the forward's rounded out for the last
// term, which saves the product O = P.V.  Five products per tile against the JVP kernel's six; warp roles, shared memory,
// the rings and kSparse as dense_attn_jvp_kernel's.  Query rows >= lq read no lse and store nothing (their P is 0).
// p.out and p.lse are inputs here.  The set-up and the producer are dense_attn_jvp_kernel's, written out again: moved into a
// shared function they changed that kernel's register allocation.  kKeyLens (dense only): tiles past k_lens[b] are neither
// loaded nor visited, the last tile's rows past them are zeroed as in dense_attn_jvp_kernel, and a row with no keys has A = 0
// and mu = 0, so it stores out_t = 0.  kQueryLens (dense only): a row past the entry's queries reads no lse and no out and
// stores out_t = 0, and a CTA whose block lies wholly past them loads nothing.
template <typename T, bool kSparse, bool kKeyLens = false, bool kQueryLens = false>
__global__ void __launch_bounds__(split::kThreads, 1)
attn_tangent_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                    const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_qt,
                    const __grid_constant__ CUtensorMap tmap_kt, const __grid_constant__ CUtensorMap tmap_vt, Params p) {
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBars);
  int32_t* s_lut = reinterpret_cast<int32_t*>(smem + kOffLut);   // kSparse only

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  const int lk = keys_of<kKeyLens>(p.k_lens, p.lk, b);
  const int lq = queries_of<kQueryLens>(p.q_lens, p.lq, b);
  const bool idle = kQueryLens && m_blk * BQ >= lq;   // the block lies wholly past the entry's queries
  const int n_tiles = idle ? 0 : kSparse ? p.topk : (lk + BK - 1) / BK;

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
  if constexpr (kSparse) {
    const int32_t* lut_row = p.lut + ((int64_t(b) * p.h + hh) * p.mblk + m_blk) * p.topk;
    for (int i = threadIdx.x; i < p.topk; i += split::kThreads) s_lut[i] = __ldg(lut_row + i);
  }
  __syncthreads();

  if (warp >= kConsumerWarps) {
    // =============================================================== TMA producer (dense_attn_jvp_kernel's)
    reg_dealloc<split::kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0 && !idle) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_qt);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_kt);
      tma_prefetch_desc(&tmap_v);
      tma_prefetch_desc(&tmap_vt);
      mbar_expect_tx(&bars[kQFull], 2 * kQBytes);
#pragma unroll
      for (int c = 0; c < HD / 64; ++c) {
        tma_load_4d(smem + kOffQ + c * (BQ * 128), &tmap_q, &bars[kQFull], c * 64, hh, m_blk * BQ, b);
        tma_load_4d(smem + kOffQd + c * (BQ * 128), &tmap_qt, &bars[kQFull], c * 64, hh, m_blk * BQ, b);
      }
      for (int j = 0; j < n_tiles; ++j) {
        const int st = j % kStages;
        const uint32_t ph = ((j / kStages) & 1) ^ 1;
        const int key0 = (kSparse ? s_lut[j] : j) * BK;
        mbar_wait(&bars[kKEmpty + st], ph);
        mbar_expect_tx(&bars[kKFull + st], kStageBytes);
        uint8_t* sk = smem + kOffK + st * kStageBytes;
#pragma unroll
        for (int c = 0; c < HD / 64; ++c) {
          tma_load_4d(sk + c * (BK * 128), &tmap_k, &bars[kKFull + st], c * 64, hh, key0, b);
          tma_load_4d(sk + kHalfBytes + c * (BK * 128), &tmap_kt, &bars[kKFull + st], c * 64, hh, key0, b);
        }
        mbar_wait(&bars[kVEmpty + st], ph);
        mbar_expect_tx(&bars[kVFull + st], kStageBytes);
        uint8_t* sv = smem + kOffV + st * kStageBytes;
#pragma unroll
        for (int c = 0; c < HD / 64; ++c) {
          tma_load_4d(sv + c * (BK * 128), &tmap_v, &bars[kVFull + st], c * 64, hh, key0, b);
          tma_load_4d(sv + kHalfBytes + c * (BK * 128), &tmap_vt, &bars[kVFull + st], c * 64, hh, key0, b);
        }
      }
    }
    return;
  }

  reg_alloc<split::kConsumerRegs>();
  const int wg = warp >> 2, w4 = warp & 3;
  const int r_lo = wg * 64 + w4 * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sq = sbase + kOffQ + wg * (64 * 128), sqd = sbase + kOffQd + wg * (64 * 128);
  const float sc = p.sm_scale * kLog2e;

  float lse[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t qr = int64_t(m_blk) * BQ + r_lo + 8 * h;
    lse[h] = qr < lq ? p.lse[(int64_t(b) * p.h + hh) * p.lq + qr] : INFINITY;
  }
  float a[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) a[i] = 0.f;
  float mu_part[2] = {0.f, 0.f};

  if (!idle) mbar_wait(&bars[kQFull], 0);
  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % kStages;
    const uint32_t ph = (j / kStages) & 1;
    const uint32_t sk = sbase + kOffK + st * kStageBytes, sv = sbase + kOffV + st * kStageBytes;

    float s[BK / 2], sd[BK / 2];
    mbar_wait(&bars[kKFull + st], ph);
    if constexpr (kKeyLens)
      if (lk - j * BK < BK && lk < p.lk) {   // the last tile, with rows past the entry's keys inside the buffer
        mbar_wait(&bars[kVFull + st], ph);
        uint8_t* const tiles[4] = {smem + kOffK + st * kStageBytes, smem + kOffK + st * kStageBytes + kHalfBytes,
                                   smem + kOffV + st * kStageBytes, smem + kOffV + st * kStageBytes + kHalfBytes};
#pragma unroll
        for (uint8_t* t : tiles) zero_key_rows(t, BK, HD / 64, lk - j * BK, threadIdx.x);
        fence_proxy_async_smem();
        named_bar_sync(1, kConsumerWarps * 32);
      }
    score_tile<true, HD, BK, kBF16>(s, sq, BQ * 128, sk, sc);
    const int valid = lk - (kSparse ? s_lut[j] : j) * BK;
#pragma unroll
    for (int i = 0; i < BK / 2; ++i) {
      const float x = s[i] - lse[(i >> 1) & 1];
      s[i] = valid < BK && 8 * (i >> 2) + cq + (i & 1) >= valid ? 0.f : fast_exp2(x);   // s := P
    }
#pragma unroll
    for (int i = 0; i < BK / 2; ++i) sd[i] = 0.f;
    wgmma_fence();
    qk_mmas<kBF16>(sd, sqd, sk, false);               // Sd / c = Qd.K^T + Q.Kd^T
    qk_mmas<kBF16>(sd, sq, sk + kHalfBytes, true);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(sd);
    warp_release(&bars[kKEmpty + st], lane);

    uint32_t pa[BK / 16][4], pda[BK / 16][4];        // P and P * Sd rounded to T: the A operands of the products
#pragma unroll
    for (int i = 0; i < BK / 2; i += 2) {
      const int h = (i >> 1) & 1;
      const float x0 = s[i] * (sd[i] * p.sm_scale), x1 = s[i + 1] * (sd[i + 1] * p.sm_scale);
      mu_part[h] += x0 + x1;
      pa[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(s[i], s[i + 1]);
      pda[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(x0, x1);
    }

    mbar_wait(&bars[kVFull + st], ph);
    const uint64_t vdesc = make_desc_mnmajor_sw128(sv, BK * 128), vddesc = make_desc_mnmajor_sw128(sv + kHalfBytes, BK * 128);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) wgmma_f16_rs<HD, kBF16, 1>(a, pda[kk], vdesc + uint64_t(kk * 128));
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) wgmma_f16_rs<HD, kBF16, 1>(a, pa[kk], vddesc + uint64_t(kk * 128));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(a);
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) {
      reg_fence(pa[kk]);
      reg_fence(pda[kk]);
    }
    warp_release(&bars[kVEmpty + st], lane);
  }

#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float mu = quad_sum(mu_part[h]);   // all four lanes of a row take part
    const int64_t qr = int64_t(m_blk) * BQ + r_lo + 8 * h;
    if (qr >= p.lq) continue;
    const int64_t row = ((int64_t(b) * p.lq + qr) * p.h + hh) * HD;
    const T* orow = static_cast<const T*>(p.out) + row;
    T* trow = static_cast<T*>(p.out_t) + row;
    if (kQueryLens && qr >= lq) {   // a row past the entry's queries
#pragma unroll
      for (int c = 0; c < HD / 8; ++c) *reinterpret_cast<uint32_t*>(trow + 8 * c + cq) = 0u;
      continue;
    }
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      const int i = 4 * c + 2 * h;
      const uint32_t ow = *reinterpret_cast<const uint32_t*>(orow + 8 * c + cq);
      *reinterpret_cast<uint32_t*>(trow + 8 * c + cq) =
          F16Traits<T>::pack(fmaf(-mu, F16Traits<T>::lo(ow), a[i]), fmaf(-mu, F16Traits<T>::hi(ow), a[i + 1]));
    }
  }
}

// kSparse: the dynamic shared memory grows by the LUT row, as for launch_sparse
template <typename T, bool kSparse, bool kKeyLens = false, bool kQueryLens = false>
int launch_tangent(const CUtensorMap (&tm)[6], const Params& p, dim3 grid, cudaStream_t st) {
  static bool smem_set[64];
  const auto kern = attn_tangent_kernel<T, kSparse, kKeyLens, kQueryLens>;
  const size_t smem_max = kSparse ? kSparseSmemMax : kSmemBytes;
  if (int rc = set_max_dynamic_smem_once(reinterpret_cast<const void*>(kern), smem_max, smem_set,
                                         kSparse ? "cudaFuncSetAttribute(sla_attn16_tangent)" : "cudaFuncSetAttribute(attn_dense_tangent)"))
    return rc;
  kern<<<grid, split::kThreads, kSmemBytes + (kSparse ? 4 * size_t(p.topk) : 0), st>>>(tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], p);
  return check_launch(kSparse ? "sla_attn16_tangent_kernel" : "attn_dense_tangent_kernel");
}
}  // namespace jvp

// [b, l, h, HD] 16-bit tensor, boxes of 64 columns x `rows` sequence rows of one head
int tmap16(CUtensorMap* m, const void* base, int dtype, int64_t b, int64_t l, int64_t h, uint32_t rows) {
  const CUtensorMapDataType t16 = dtype == TDB200_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const uint64_t dims[4] = {uint64_t(HD), uint64_t(h), uint64_t(l), uint64_t(b)};
  const uint64_t str[3] = {uint64_t(HD * 2), uint64_t(h * HD * 2), uint64_t(l * h * HD * 2)};
  const uint32_t box[4] = {64, 1, rows, 1};
  return make_tmap_4d(m, base, t16, 2, dims, str, box);
}

bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }

// tdb200_attn_dense_fwd (lse null) and tdb200_attn_dense_fwd_lse; `what` prefixes the messages.  key_lens: their _kl twins,
// which take k_lens [b] and launch the kKeyLens kernels; query_lens (with key_lens): their _vl twins, which also take q_lens [b]
// and launch the kernels with both flags set.
int dense_fwd(const char* what, const void* q, const void* k, const void* v, int dtype, void* out, float* lse, bool with_lse,
              int64_t b, int64_t lq, int64_t lk, const int32_t* q_lens, bool query_lens, const int32_t* k_lens, bool key_lens,
              int64_t h, int64_t d, float sm_scale, void* stream) {
  if (!q || !k || !v || !out || (with_lse && !lse) || (key_lens && !k_lens) || (query_lens && !q_lens))
    return fail(TDB200_ERR_INVALID_ARG, "%s: null pointer", what);
  if (int rc = dense_attn_shape(what, b, lq, lk, h, d)) return rc;
  if (!aligned16(q) || !aligned16(k) || !aligned16(v) || !aligned16(out))
    return fail(TDB200_ERR_INVALID_ARG, "%s: q, k, v and out must be 16-byte aligned", what);
  if (with_lse && !aligned4(lse)) return fail(TDB200_ERR_INVALID_ARG, "%s: lse must be 4-byte aligned", what);
  if (key_lens && !aligned4(k_lens)) return fail(TDB200_ERR_INVALID_ARG, "%s: k_lens must be 4-byte aligned", what);
  if (query_lens && !aligned4(q_lens)) return fail(TDB200_ERR_INVALID_ARG, "%s: q_lens must be 4-byte aligned", what);
  if (int rc = dense_attn_limits(what, dtype, b, lq, lk, h, d)) return rc;
  if (int rc = require_sm90()) return rc;

  CUtensorMap tq, tk, tv;
  if (int rc = tmap16(&tq, q, dtype, b, lq, h, BQ)) return rc;
  if (int rc = tmap16(&tk, k, dtype, b, lk, h, BK)) return rc;
  if (int rc = tmap16(&tv, v, dtype, b, lk, h, BK)) return rc;
  DenseParams p;
  p.out = out;
  p.lse = lse;
  p.lq = int(lq);
  p.lk = int(lk);
  p.h = int(h);
  p.sm_scale = sm_scale;
  p.k_lens = k_lens;
  p.q_lens = q_lens;
  const dim3 grid(static_cast<unsigned>(cdiv64(lq, BQ)), static_cast<unsigned>(h), static_cast<unsigned>(b));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool bf16 = dtype == TDB200_DTYPE_BF16;
  if (query_lens) {
    if (!with_lse)
      return bf16 ? launch<__nv_bfloat16, false, true, true>(tq, tk, tv, p, grid, st)
                  : launch<__half, false, true, true>(tq, tk, tv, p, grid, st);
    return bf16 ? launch<__nv_bfloat16, true, true, true>(tq, tk, tv, p, grid, st) : launch<__half, true, true, true>(tq, tk, tv, p, grid, st);
  }
  if (!key_lens) {
    if (!with_lse)
      return bf16 ? launch<__nv_bfloat16, false, false>(tq, tk, tv, p, grid, st) : launch<__half, false, false>(tq, tk, tv, p, grid, st);
    return bf16 ? launch<__nv_bfloat16, true, false>(tq, tk, tv, p, grid, st) : launch<__half, true, false>(tq, tk, tv, p, grid, st);
  }
  if (!with_lse)
    return bf16 ? launch<__nv_bfloat16, false, true>(tq, tk, tv, p, grid, st) : launch<__half, false, true>(tq, tk, tv, p, grid, st);
  return bf16 ? launch<__nv_bfloat16, true, true>(tq, tk, tv, p, grid, st) : launch<__half, true, true>(tq, tk, tv, p, grid, st);
}

// tdb200_attn_dense_jvp (lse null), tdb200_attn_dense_jvp_lse and, `tangent`, tdb200_attn_dense_tangent (out and lse inputs);
// key_lens: their _kl twins, query_lens: their _vl twins, as for dense_fwd
int dense_jvp(const char* what, const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
              int dtype, void* out, void* out_t, float* lse, bool with_lse, int64_t b, int64_t lq, int64_t lk, const int32_t* q_lens,
              bool query_lens, const int32_t* k_lens, bool key_lens, int64_t h, int64_t d, float sm_scale, void* stream,
              bool tangent = false) {
  if (!q || !k || !v || !q_t || !k_t || !v_t || !out || !out_t || (with_lse && !lse) || (key_lens && !k_lens) ||
      (query_lens && !q_lens))
    return fail(TDB200_ERR_INVALID_ARG, "%s: null pointer", what);
  if (int rc = dense_attn_shape(what, b, lq, lk, h, d)) return rc;
  if (!aligned16(q) || !aligned16(k) || !aligned16(v) || !aligned16(q_t) || !aligned16(k_t) || !aligned16(v_t) ||
      !aligned16(out) || !aligned16(out_t))
    return fail(TDB200_ERR_INVALID_ARG, "%s: q, k, v, their tangents, out and out_t must be 16-byte aligned", what);
  if (with_lse && !aligned4(lse)) return fail(TDB200_ERR_INVALID_ARG, "%s: lse must be 4-byte aligned", what);
  if (key_lens && !aligned4(k_lens)) return fail(TDB200_ERR_INVALID_ARG, "%s: k_lens must be 4-byte aligned", what);
  if (query_lens && !aligned4(q_lens)) return fail(TDB200_ERR_INVALID_ARG, "%s: q_lens must be 4-byte aligned", what);
  if (int rc = dense_attn_limits(what, dtype, b, lq, lk, h, d)) return rc;
  if (int rc = require_sm90()) return rc;

  CUtensorMap tm[6];   // q, k, v, q_t, k_t, v_t
  if (int rc = tmap16(&tm[0], q, dtype, b, lq, h, BQ)) return rc;
  if (int rc = tmap16(&tm[3], q_t, dtype, b, lq, h, BQ)) return rc;
  if (int rc = tmap16(&tm[1], k, dtype, b, lk, h, jvp::BK)) return rc;
  if (int rc = tmap16(&tm[2], v, dtype, b, lk, h, jvp::BK)) return rc;
  if (int rc = tmap16(&tm[4], k_t, dtype, b, lk, h, jvp::BK)) return rc;
  if (int rc = tmap16(&tm[5], v_t, dtype, b, lk, h, jvp::BK)) return rc;
  jvp::Params p;
  p.out = out;
  p.out_t = out_t;
  p.lse = lse;
  p.lq = int(lq);
  p.lk = int(lk);
  p.h = int(h);
  p.sm_scale = sm_scale;
  p.k_lens = k_lens;
  p.q_lens = q_lens;
  const dim3 grid(static_cast<unsigned>(cdiv64(lq, BQ)), static_cast<unsigned>(h), static_cast<unsigned>(b));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool bf16 = dtype == TDB200_DTYPE_BF16;
  if (query_lens) {
    if (tangent)
      return bf16 ? jvp::launch_tangent<__nv_bfloat16, false, true, true>(tm, p, grid, st)
                  : jvp::launch_tangent<__half, false, true, true>(tm, p, grid, st);
    if (!with_lse)
      return bf16 ? jvp::launch<__nv_bfloat16, false, true, true>(tm, p, grid, st) : jvp::launch<__half, false, true, true>(tm, p, grid, st);
    return bf16 ? jvp::launch<__nv_bfloat16, true, true, true>(tm, p, grid, st) : jvp::launch<__half, true, true, true>(tm, p, grid, st);
  }
  if (!key_lens) {
    if (tangent)
      return bf16 ? jvp::launch_tangent<__nv_bfloat16, false>(tm, p, grid, st) : jvp::launch_tangent<__half, false>(tm, p, grid, st);
    if (!with_lse)
      return bf16 ? jvp::launch<__nv_bfloat16, false, false>(tm, p, grid, st) : jvp::launch<__half, false, false>(tm, p, grid, st);
    return bf16 ? jvp::launch<__nv_bfloat16, true, false>(tm, p, grid, st) : jvp::launch<__half, true, false>(tm, p, grid, st);
  }
  if (tangent)
    return bf16 ? jvp::launch_tangent<__nv_bfloat16, false, true>(tm, p, grid, st)
                : jvp::launch_tangent<__half, false, true>(tm, p, grid, st);
  if (!with_lse)
    return bf16 ? jvp::launch<__nv_bfloat16, false, true>(tm, p, grid, st) : jvp::launch<__half, false, true>(tm, p, grid, st);
  return bf16 ? jvp::launch<__nv_bfloat16, true, true>(tm, p, grid, st) : jvp::launch<__half, true, true>(tm, p, grid, st);
}

// tdb200_sla_attn16_jvp (lse null) and tdb200_sla_attn16_jvp_lse: the JVP kernel over the LUT's key blocks, lq = lk = l;
// `tangent`: tdb200_sla_attn16_tangent, the tangent kernel over them (o_s and lse inputs)
int sla_jvp(const char* what, const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
            int dtype, const int32_t* lut, int64_t topk, void* o_s, void* o_s_t, float* lse, bool with_lse, int64_t b, int64_t l,
            int64_t h, int64_t d, float sm_scale, int64_t blkq, int64_t blkk, void* stream, bool tangent = false) {
  if (blkq != BQ || blkk != jvp::BK)
    return fail(TDB200_ERR_UNSUPPORTED, "%s: block sizes (%lld, %lld) (the JVP serves BLKQ x BLKK = 128 x 64)", what,
                (long long)blkq, (long long)blkk);
  if (!q || !k || !v || !q_t || !k_t || !v_t || !lut || !o_s || !o_s_t || (with_lse && !lse))
    return fail(TDB200_ERR_INVALID_ARG, "%s: null pointer", what);
  if (int rc = dense_attn_shape(what, b, l, l, h, d)) return rc;
  if (!aligned16(q) || !aligned16(k) || !aligned16(v) || !aligned16(q_t) || !aligned16(k_t) || !aligned16(v_t) ||
      !aligned16(o_s) || !aligned16(o_s_t))
    return fail(TDB200_ERR_INVALID_ARG, "%s: q, k, v, their tangents, o_s and o_s_t must be 16-byte aligned", what);
  if (!aligned4(lut) || (with_lse && !aligned4(lse))) return fail(TDB200_ERR_INVALID_ARG, "%s: lut and lse must be 4-byte aligned", what);
  const int64_t nblk = cdiv64(l, jvp::BK);
  if (topk <= 0 || topk > nblk)
    return fail(TDB200_ERR_INVALID_ARG, "%s: topk=%lld outside [1, %lld]", what, (long long)topk, (long long)nblk);
  if (int rc = dense_attn_limits(what, dtype, b, l, l, h, d)) return rc;
  if (topk > jvp::kMaxLutIds)
    return fail(TDB200_ERR_UNSUPPORTED, "%s: topk=%lld too large for the on-chip LUT (at most %lld)", what, (long long)topk,
                (long long)jvp::kMaxLutIds);
  if (int rc = require_sm90()) return rc;

  CUtensorMap tm[6];   // q, k, v, q_t, k_t, v_t
  if (int rc = tmap16(&tm[0], q, dtype, b, l, h, BQ)) return rc;
  if (int rc = tmap16(&tm[3], q_t, dtype, b, l, h, BQ)) return rc;
  if (int rc = tmap16(&tm[1], k, dtype, b, l, h, jvp::BK)) return rc;
  if (int rc = tmap16(&tm[2], v, dtype, b, l, h, jvp::BK)) return rc;
  if (int rc = tmap16(&tm[4], k_t, dtype, b, l, h, jvp::BK)) return rc;
  if (int rc = tmap16(&tm[5], v_t, dtype, b, l, h, jvp::BK)) return rc;
  jvp::Params p;
  p.out = o_s;
  p.out_t = o_s_t;
  p.lse = lse;
  p.lq = int(l);
  p.lk = int(l);
  p.h = int(h);
  p.sm_scale = sm_scale;
  p.lut = lut;
  p.topk = int(topk);
  p.mblk = int(cdiv64(l, BQ));
  const dim3 grid(static_cast<unsigned>(p.mblk), static_cast<unsigned>(h), static_cast<unsigned>(b));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool bf16 = dtype == TDB200_DTYPE_BF16;
  if (tangent)
    return bf16 ? jvp::launch_tangent<__nv_bfloat16, true>(tm, p, grid, st) : jvp::launch_tangent<__half, true>(tm, p, grid, st);
  if (!with_lse)
    return bf16 ? jvp::launch_sparse<__nv_bfloat16, false>(tm, p, grid, st) : jvp::launch_sparse<__half, false>(tm, p, grid, st);
  return bf16 ? jvp::launch_sparse<__nv_bfloat16, true>(tm, p, grid, st) : jvp::launch_sparse<__half, true>(tm, p, grid, st);
}

}  // namespace

extern "C" int tdb200_attn_dense_fwd(const void* q, const void* k, const void* v, int dtype, void* out, int64_t b, int64_t lq,
                                     int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream) {
  return dense_fwd("attn_dense_fwd", q, k, v, dtype, out, nullptr, false, b, lq, lk, nullptr, false, nullptr, false, h, d, sm_scale, stream);
}

extern "C" int tdb200_attn_dense_fwd_lse(const void* q, const void* k, const void* v, int dtype, void* out, float* lse, int64_t b,
                                         int64_t lq, int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream) {
  return dense_fwd("attn_dense_fwd_lse", q, k, v, dtype, out, lse, true, b, lq, lk, nullptr, false, nullptr, false, h, d, sm_scale, stream);
}

extern "C" int tdb200_attn_dense_jvp(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                     const void* v_t, int dtype, void* out, void* out_t, int64_t b, int64_t lq, int64_t lk,
                                     int64_t h, int64_t d, float sm_scale, void* stream) {
  return dense_jvp("attn_dense_jvp", q, k, v, q_t, k_t, v_t, dtype, out, out_t, nullptr, false, b, lq, lk, nullptr, false, nullptr, false, h, d,
                   sm_scale, stream);
}

extern "C" int tdb200_attn_dense_jvp_lse(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                         const void* v_t, int dtype, void* out, void* out_t, float* lse, int64_t b, int64_t lq,
                                         int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream) {
  return dense_jvp("attn_dense_jvp_lse", q, k, v, q_t, k_t, v_t, dtype, out, out_t, lse, true, b, lq, lk, nullptr, false, nullptr, false, h, d,
                   sm_scale, stream);
}

extern "C" int tdb200_sla_attn16_jvp(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                                     int dtype, const int32_t* lut, int64_t topk, void* o_s, void* o_s_t, int64_t b, int64_t l,
                                     int64_t h, int64_t d, float sm_scale, int64_t blkq, int64_t blkk, void* stream) {
  return sla_jvp("sla_attn16_jvp", q, k, v, q_t, k_t, v_t, dtype, lut, topk, o_s, o_s_t, nullptr, false, b, l, h, d, sm_scale, blkq,
                 blkk, stream);
}

extern "C" int tdb200_sla_attn16_jvp_lse(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                         const void* v_t, int dtype, const int32_t* lut, int64_t topk, void* o_s, void* o_s_t,
                                         float* lse, int64_t b, int64_t l, int64_t h, int64_t d, float sm_scale, int64_t blkq,
                                         int64_t blkk, void* stream) {
  return sla_jvp("sla_attn16_jvp_lse", q, k, v, q_t, k_t, v_t, dtype, lut, topk, o_s, o_s_t, lse, true, b, l, h, d, sm_scale, blkq,
                 blkk, stream);
}

extern "C" int tdb200_attn_dense_tangent(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                         const void* v_t, const void* out, const float* lse, int dtype, void* out_t, int64_t b,
                                         int64_t lq, int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream) {
  return dense_jvp("attn_dense_tangent", q, k, v, q_t, k_t, v_t, dtype, const_cast<void*>(out), out_t, const_cast<float*>(lse), true,
                   b, lq, lk, nullptr, false, nullptr, false, h, d, sm_scale, stream, true);
}

extern "C" int tdb200_sla_attn16_tangent(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                         const void* v_t, const void* o_s, const float* lse, int dtype, const int32_t* lut,
                                         int64_t topk, void* o_s_t, int64_t b, int64_t l, int64_t h, int64_t d, float sm_scale,
                                         int64_t blkq, int64_t blkk, void* stream) {
  return sla_jvp("sla_attn16_tangent", q, k, v, q_t, k_t, v_t, dtype, lut, topk, const_cast<void*>(o_s), o_s_t, const_cast<float*>(lse),
                 true, b, l, h, d, sm_scale, blkq, blkk, stream, true);
}

// ---------------------------------------------------------------------------------------------------------------------------
// The _kl twins: the entry points above with per-sample key lengths k_lens [b] (the kKeyLens kernels)
extern "C" int tdb200_attn_dense_fwd_kl(const void* q, const void* k, const void* v, int dtype, void* out, int64_t b, int64_t lq,
                                        int64_t lk, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream) {
  return dense_fwd("attn_dense_fwd_kl", q, k, v, dtype, out, nullptr, false, b, lq, lk, nullptr, false, k_lens, true, h, d, sm_scale, stream);
}

extern "C" int tdb200_attn_dense_fwd_lse_kl(const void* q, const void* k, const void* v, int dtype, void* out, float* lse, int64_t b,
                                            int64_t lq, int64_t lk, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale,
                                            void* stream) {
  return dense_fwd("attn_dense_fwd_lse_kl", q, k, v, dtype, out, lse, true, b, lq, lk, nullptr, false, k_lens, true, h, d, sm_scale, stream);
}

extern "C" int tdb200_attn_dense_jvp_kl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                        const void* v_t, int dtype, void* out, void* out_t, int64_t b, int64_t lq, int64_t lk,
                                        const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream) {
  return dense_jvp("attn_dense_jvp_kl", q, k, v, q_t, k_t, v_t, dtype, out, out_t, nullptr, false, b, lq, lk, nullptr, false, k_lens, true, h, d,
                   sm_scale, stream);
}

extern "C" int tdb200_attn_dense_jvp_lse_kl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                            const void* v_t, int dtype, void* out, void* out_t, float* lse, int64_t b, int64_t lq,
                                            int64_t lk, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream) {
  return dense_jvp("attn_dense_jvp_lse_kl", q, k, v, q_t, k_t, v_t, dtype, out, out_t, lse, true, b, lq, lk, nullptr, false, k_lens, true, h, d,
                   sm_scale, stream);
}

extern "C" int tdb200_attn_dense_tangent_kl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                            const void* v_t, const void* out, const float* lse, int dtype, void* out_t, int64_t b,
                                            int64_t lq, int64_t lk, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale,
                                            void* stream) {
  return dense_jvp("attn_dense_tangent_kl", q, k, v, q_t, k_t, v_t, dtype, const_cast<void*>(out), out_t, const_cast<float*>(lse),
                   true, b, lq, lk, nullptr, false, k_lens, true, h, d, sm_scale, stream, true);
}

// ---------------------------------------------------------------------------------------------------------------------------
// The _vl twins: per-sample query lengths q_lens [b] and key lengths k_lens [b] (the kernels with kQueryLens and kKeyLens)
extern "C" int tdb200_attn_dense_fwd_vl(const void* q, const void* k, const void* v, int dtype, void* out, int64_t b, int64_t lq,
                                        int64_t lk, const int32_t* q_lens, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale,
                                        void* stream) {
  return dense_fwd("attn_dense_fwd_vl", q, k, v, dtype, out, nullptr, false, b, lq, lk, q_lens, true, k_lens, true, h, d, sm_scale,
                   stream);
}

extern "C" int tdb200_attn_dense_fwd_lse_vl(const void* q, const void* k, const void* v, int dtype, void* out, float* lse, int64_t b,
                                            int64_t lq, int64_t lk, const int32_t* q_lens, const int32_t* k_lens, int64_t h, int64_t d,
                                            float sm_scale, void* stream) {
  return dense_fwd("attn_dense_fwd_lse_vl", q, k, v, dtype, out, lse, true, b, lq, lk, q_lens, true, k_lens, true, h, d, sm_scale,
                   stream);
}

extern "C" int tdb200_attn_dense_jvp_vl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                        const void* v_t, int dtype, void* out, void* out_t, int64_t b, int64_t lq, int64_t lk,
                                        const int32_t* q_lens, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale,
                                        void* stream) {
  return dense_jvp("attn_dense_jvp_vl", q, k, v, q_t, k_t, v_t, dtype, out, out_t, nullptr, false, b, lq, lk, q_lens, true, k_lens,
                   true, h, d, sm_scale, stream);
}

extern "C" int tdb200_attn_dense_jvp_lse_vl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                            const void* v_t, int dtype, void* out, void* out_t, float* lse, int64_t b, int64_t lq,
                                            int64_t lk, const int32_t* q_lens, const int32_t* k_lens, int64_t h, int64_t d,
                                            float sm_scale, void* stream) {
  return dense_jvp("attn_dense_jvp_lse_vl", q, k, v, q_t, k_t, v_t, dtype, out, out_t, lse, true, b, lq, lk, q_lens, true, k_lens,
                   true, h, d, sm_scale, stream);
}

extern "C" int tdb200_attn_dense_tangent_vl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                            const void* v_t, const void* out, const float* lse, int dtype, void* out_t, int64_t b,
                                            int64_t lq, int64_t lk, const int32_t* q_lens, const int32_t* k_lens, int64_t h,
                                            int64_t d, float sm_scale, void* stream) {
  return dense_jvp("attn_dense_tangent_vl", q, k, v, q_t, k_t, v_t, dtype, const_cast<void*>(out), out_t, const_cast<float*>(lse),
                   true, b, lq, lk, q_lens, true, k_lens, true, h, d, sm_scale, stream, true);
}
