// a9 + a10. Fused SageSLA attention forward for one (query block, head, batch) per CTA:
//   block-sparse INT8 Q.K^T -> online softmax (exp2) -> 16-bit P.V, then the linear branch phi(Q).KVW / (eps + phi(Q).ksum)
//   folded into the same accumulator, all in one wgmma kernel.
//   reference: Sage call site turbodiffusion/SLA/core.py:231-235 (arithmetic in third-party SpargeAttn, unpinned);
//   the in-tree statement of the same attention is the Triton kernel SLA/kernel.py:33-82 (tail masking :57-62, exp2 with
//   qk_scale*log2e :60, row sum from unrounded P :71, P cast before P.V :73); linear branch + merge SLA/core.py:243-253.
//
// Two kernels: sla_attn_fwd_kernel on 128-row query blocks (2 consumer warpgroups + 1 TMA warp; warpgroup g owns query rows
//   [64g, 64g+64) of the block), and sla_attn_fwd_q64_kernel on 64-row query blocks (the entry-split CTA of sla_attn.cuh).
//   Both run the same per-entry steps on a warpgroup's 64 rows, and every thread holds two rows of the fragments
//   (common.cuh): S[64 x BK] in BK/2 registers (wgmma m64nBK, A = Q and B = K from shared memory),
//   P converted in registers straight into the A fragments of P.V (wgmma m64nHD, A from registers, B = V MN-major from
//   shared memory, so no transposed copy of V is ever materialised), and the O accumulator [64 x HD] in HD/2 registers.
//   Row maxima / sums are reduced across the four lanes that share a row.
//   After the last key block the linear branch adds A.KVW^T to O with A = phi(q) * l / den in registers, so that
//   O / l = softmax part + phi(q).KVW^T / den, and out = O / l + proj_b.
// Shared memory: Q | K ring | V ring (3 stages each; K and V released per warp as soon as their MMA retired) | KVW, and for
//   INT8 Q/K the 16-bit query rows, loaded with Q and read by the linear branch, whose rows each warp then overwrites with
//   its 16 output rows for a TMA store.  Q/K/KVW are K-major swizzled (128B rows, or 64B rows for 64-wide int8 heads).
// The O accumulator is only rescaled when a row maximum grows by more than 2^8 (lazy rescale): P stays <= 256, which
// bf16/fp32 hold exactly as well as P <= 1, and the final O / l normalisation is unchanged.
// Entry points: tdb200_sla_attn_fwd (INT8 Q/K, head dims 64 and 128, feature maps of the linear branch, K head-major or in
// [b, lk, h, d], 128 x 64 blocks or 64 x 128 blocks), tdb200_sla_attn16_fwd (16-bit Q/K read from the module layout
// [b, l, h, d], fp32 scores; 128 x 64 or 64 x 64 blocks) and tdb200_sla_attn16_fwd_lse (its sparse branch and row
// log-sum-exp, for the backward).
#include <type_traits>

#include "sla_attn.cuh"
#include "host_common.h"

namespace {
using namespace tdb;

constexpr int BLKQ = 128, BLKK = 64;
constexpr int kBlkQ64 = 64, kHopperBlkK = 128;   // the 64-row query blocks; 128-row key blocks of the INT8 Hopper family
constexpr int kConsumerWarps = 8;
constexpr int kThreads = kConsumerWarps * 32 + 32;
constexpr int kStages = 3;
static_assert(kStages == split::kStages, "the 64-row kernel uses the entry-split rings");

template <int HD, bool kQK16, int kBQ = BLKQ, int kBK = BLKK, bool kF8V = false>
struct Lay {
  static constexpr uint32_t kQBytes = kQK16 ? kBQ * HD * 2 : kBQ * HD;     // 16-bit: HD/64 chunks of [kBQ rows x 128 B]
  static constexpr uint32_t kKBytes = kQK16 ? kBK * HD * 2 : kBK * HD;
  static constexpr uint32_t kVBytes = kF8V ? kBK * HD : kBK * HD * 2;      // HD/64 boxes of [kBK keys x 128 B]; e4m3: [HD x kBK B]
  static constexpr uint32_t kWBytes = HD * HD * 2;                         // HD/64 d_k chunks of [HD rows x 128 B]
  // INT8 only: the 16-bit query rows for phi(q), HD/64 chunks of [kBQ rows x 128 B], then the output rows staged for TMA
  static constexpr uint32_t kQ16Bytes = kQK16 ? 0 : kBQ * HD * 2;
  static constexpr uint32_t kOffQ = 0;
  static constexpr uint32_t kOffK = kOffQ + kQBytes;
  static constexpr uint32_t kOffV = kOffK + kStages * kKBytes;
  static constexpr uint32_t kOffW = kOffV + kStages * kVBytes;
  static constexpr uint32_t kOffQ16 = kOffW + kWBytes;
  static constexpr uint32_t kOffBars = kOffQ16 + kQ16Bytes;
  static constexpr uint32_t kOffLut = kOffBars + 256;
};
static_assert(split::kNumBars * 8 <= 256, "barriers exceed their shared-memory slot");

struct AttnParams {
  const float* q_scale;   // [b,h,mblk]
  const float* k_scale;   // [b,h,nblk]
  const void* q;          // [b,l,h,d] T (linear branch)
  const int32_t* lut;     // [b,h,mblk,topk]
  const float* ksum;      // [b,h,d]
  const float* proj_b;    // [d]
  void* out;              // [b,l,h,d] T
  int l, lk, h, mblk, nblk, topk, feature;  // feature: 0 softmax, 1 elu+1, 2 relu (SLA/core.py:57-73)
  float sm_scale;
  float* lse;             // [b,h,l] fp32, log2 domain (kLse kernels only)
  const float* v_scale;   // [b,h,d] fp32 (kF8V kernels only)
  const int32_t* seq_lens;   // [b] int32 (kVL kernels only): entry b's rows, lq = lk
  const int32_t* topks;      // [b] int32 (kVL kernels only): the LUT entries each of entry b's rows walks
  const void* v;             // [b,l,h,d] T (kVL 128-row kernels only: the producer's straddling V block)
};

// kVL (the _vl entry points): entry b owns its first n = seq_lens[b] query and key rows (clamped to [0, l], read once before the
// first barrier) and walks topks[b] LUT entries, clamped to [1, min(ceil(n / BK), topk)] as the block map clamps them.  Rows past
// n are stored as zeros; a query block wholly past n stores its zero rows and exits (vl_store_zero_block).  Keys past n are masked
// as keys past lk are, and the V rows past n of the straddling key block are zero in shared memory before the P.V reads them (TMA
// would load the padding there, where a call on the entry alone gets zero fill, and 0 * NaN is NaN): in the 128-row kernel the
// producer warp loads that block itself (vl_load_v_block), in the 64-row kernel its warpgroup zeroes the rows.
__device__ __forceinline__ int vl_topk(const AttnParams& p, int b, int n, int bk) {
  return min(max(__ldg(p.topks + b), 1), min((n + bk - 1) / bk, p.topk));
}

// The 128-row kVL kernel's straddling V block: rows [0, valid) of key block blk of head hh of entry b, the rest zero, written by
// the producer warp in the layout TMA gives (HD/64 chunks of [BK rows x 128 B], 16-byte units swizzled by row & 7).  The caller
// then fences the async proxy and arrives on the V-full barrier.
template <typename T, int HD, int BK>
__device__ __forceinline__ void vl_load_v_block(uint8_t* sv, const AttnParams& p, int b, int hh, int blk, int valid, int lane) {
  for (int e = lane; e < BK * (HD / 8); e += 32) {
    const int r = e / (HD / 8), cu = e % (HD / 8);
    uint4 x = make_uint4(0u, 0u, 0u, 0u);
    if (r < valid) x = ldg_nc_v4(static_cast<const T*>(p.v) + ((int64_t(b) * p.l + int64_t(blk) * BK + r) * p.h + hh) * HD + cu * 8);
    *reinterpret_cast<uint4*>(sv + (cu >> 3) * (BK * 128) + r * 128 + (((cu & 7) ^ (r & 7)) << 4)) = x;
  }
}

// rows [row0, min(row0 + rows, l)) of head hh of entry b of the output are zero; every thread of the CTA takes part
template <int HD>
__device__ __forceinline__ void vl_store_zero_block(const AttnParams& p, int row0, int rows, int b, int hh) {
  const int n_rows = min(rows, p.l - row0);
  uint8_t* base = static_cast<uint8_t*>(p.out);
  for (int e = threadIdx.x; e < n_rows * (HD / 8); e += blockDim.x) {
    const int r = e / (HD / 8), c = e % (HD / 8);
    *reinterpret_cast<uint4*>(base + (((int64_t(b) * p.l + row0 + r) * p.h + hh) * HD + c * 8) * 2) = make_uint4(0u, 0u, 0u, 0u);
  }
}

enum Bar { kQFull = 0, kKFull = 1 /*3*/, kKEmpty = 4 /*3*/, kVFull = 7 /*3*/, kVEmpty = 10 /*3*/, kNumBars = 13 };

__device__ __forceinline__ float feat(float x, float off_log2, int feature) {
  // softmax numerator exp(x - max) | elu(x)+1 | relu(x)
  if (feature == 0) return fast_exp2(fmaf(x, kLog2e, -off_log2));
  if (feature == 1) return x > 0.f ? x + 1.0f : fast_exp2(x * kLog2e);
  return fmaxf(x, 0.f);
}

// kLse epilogue: out = T(O / l) and lse[b,h,row] = m_used + log2(l), the row log-sum-exp of the scores in the kernel's log2
// domain, for rows qrow0 + {0, 8}.
template <typename T, int HD>
__device__ __forceinline__ void store_o_lse(const float (&o)[HD / 2], const float (&m_used)[2], const float (&l_part)[2],
                                            const AttnParams& p, int64_t qrow0, int cq, int b, int hh, int bh) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t qr = qrow0 + 8 * h;
    if (qr >= p.l) continue;
    const float l_tot = quad_sum(l_part[h]), inv_l = 1.0f / l_tot;
    if (cq == 0) p.lse[int64_t(bh) * p.l + qr] = m_used[h] + __log2f(l_tot);
    store_o_row<T, HD>(static_cast<T*>(p.out) + ((int64_t(b) * p.l + qr) * p.h + hh) * HD, o, h, inv_l, cq);
  }
}

// The INT8 kernels' 16 query rows of one warp in shared memory: the 16-bit query rows TMA loaded with the Q barrier, HD/64
// chunks of [16 rows x 128 B] `chunk` bytes apart in the 128-byte swizzle, which the output rows overwrite and a TMA store
// (map `tmap_out`, boxes of 64 columns x 16 rows at query row `row`) writes out.
struct RowTile {
  uint8_t* smem;
  uint32_t chunk;
  const CUtensorMap* tmap_out;
  int32_t row;
};

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// volatile: read where it is used, so that the value does not hold a register across the loop that uses it
__device__ __forceinline__ int lds_s32(uint32_t addr) {
  int v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

// After the last key block, for the 64 query rows of one warpgroup (rows qrow0 + {0, 8} for this thread): the linear branch
// adds A.KVW^T to O, then out = T( O / l + proj_b ).  kvw_smem: the KVW tile (K-major, swizzled like Q).
// kTile (the INT8 kernels): the query rows are read from and the output rows written through the warp's RowTile, and rows
// >= l are clipped by the tensor map; otherwise the query rows are read from and the output rows stored to global memory.
// kVL: rows >= n (the entry's length) are stored as zeros.
template <typename T, int HD, bool kTile = false, bool kVL = false>
__device__ __forceinline__ void linear_branch_store(float (&o)[HD / 2], const float (&l_part)[2], const AttnParams& p,
                                                    uint32_t kvw_smem, int64_t qrow0, int cq, int b, int hh, int bh,
                                                    const RowTile& tile = RowTile{}, int n = 0) {
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  const float l_tot[2] = {quad_sum(l_part[0]), quad_sum(l_part[1])};
  const int lane = threadIdx.x & 31;
  const uint32_t tile_s = smem_u32(tile.smem);

  // ---- linear branch operand (SLA/core.py:243).  f_j = feature map numerator of the query row:
  //      E = sum f_j, F = sum f_j * ksum_j;  phi_j = f_j / E (softmax) or f_j;  den = 1e-5 + sum_j phi_j ksum_j;
  //      A_j = T(phi_j * l / den), so that O + A.KVW^T = l * (O/l + phi.KVW^T/den).
  //      This thread holds, for each K=16 step kk, the column pairs 16 kk + cq and 16 kk + 8 + cq of its two rows.
  uint32_t qa[HD / 16][4];
  if constexpr (kTile) {   // lane i addresses row (i & 7) + 8 ((i >> 3) & 1), 16-byte column unit i >> 4 of each K = 16 step
    const int r = (lane & 7) + 8 * ((lane >> 3) & 1);
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
      ldsm_x4(qa[kk], tile_s + (kk >> 2) * tile.chunk + r * 128 + ((((kk & 3) * 2 + (lane >> 4)) ^ (lane & 7)) << 4));
  } else {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t qr = qrow0 + 8 * h;
      const T* qrow = static_cast<const T*>(p.q) + ((int64_t(b) * p.l + (qr < p.l ? qr : p.l - 1)) * p.h + hh) * HD;
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) {
        qa[kk][h] = __ldg(reinterpret_cast<const unsigned int*>(qrow + 16 * kk + cq));
        qa[kk][2 + h] = __ldg(reinterpret_cast<const unsigned int*>(qrow + 16 * kk + 8 + cq));
      }
    }
  }
  const float* ks = p.ksum + int64_t(bh) * HD;
  // fp16: A is rounded to T only as the MMA operand, and its range follows l / den, not the output's: a relu channel dead on
  // every key (ksum_j = 0, den = 1e-5) puts A_j near 1e5 * l, inf against a KVW column of zeros (inf * 0 = NaN), a large
  // shared channel lifts max A past 65504, and peaked rows over long sequences make every A subnormal (below 2^-14).  A row
  // whose max A lies outside [2^-6, 2^15) runs the product on A * 2^sc, O * 2^sc and stores with 1 / l * 2^-sc, sc chosen
  // to put max A near 2^14.  |sc| <= 64, so the three scalings are exact in fp32: O <= l max|v| < 2^42 times 2^64 stays
  // finite, 1/l in [2^-27, 1] stays normal, and O elements that 2^-64 would take below fp32's normal range are < 2^-62, far
  // under fp16's last subnormal after the division by l >= 1.  Other rows keep sc = 0 and their bits.
  float out_scale[2] = {1.f, 1.f};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float off = 0.f;
    if (p.feature == 0) {
      float qm = -INFINITY;
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk)
#pragma unroll
        for (int u = 0; u < 2; ++u)
          qm = fmaxf(qm, fmaxf(F16Traits<T>::lo(qa[kk][h + 2 * u]), F16Traits<T>::hi(qa[kk][h + 2 * u])));
      off = quad_max(qm) * kLog2e;
    }
    float e = 0.f, f = 0.f, fm = 0.f;
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const uint32_t w = qa[kk][h + 2 * u];
        const float2 k2 = __ldg(reinterpret_cast<const float2*>(ks + 16 * kk + 8 * u + cq));
        const float a0 = feat(F16Traits<T>::lo(w), off, p.feature), a1 = feat(F16Traits<T>::hi(w), off, p.feature);
        e += a0 + a1;
        f = fmaf(a0, k2.x, fmaf(a1, k2.y, f));
        if constexpr (!kBF16) fm = fmaxf(fm, fmaxf(a0, a1));   // every feature map is >= 0
      }
    const float E = quad_sum(e), F = quad_sum(f);
    const float inv_e = p.feature == 0 ? 1.0f / E : 1.0f;
    const float den = 1e-5f + F * inv_e;
    float cscale = inv_e * l_tot[h] / den;
    if constexpr (!kBF16) {
      const float amax = quad_max(fm) * cscale;   // = max_j A_j before rounding (rounding is monotone)
      if ((amax > 0.f && amax < 0x1p-6f) || amax >= 0x1p15f) {
        const int sc = min(64, max(-64, 14 - ((__float_as_int(amax) >> 23) - 127)));
        const float up = __int_as_float((127 + sc) << 23);
        cscale *= up;
#pragma unroll
        for (int i = 0; i < HD / 2; ++i)
          if (((i >> 1) & 1) == h) o[i] *= up;
        out_scale[h] = __int_as_float((127 - sc) << 23);
      }
    }
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const uint32_t w = qa[kk][h + 2 * u];
        qa[kk][h + 2 * u] = F16Traits<T>::pack(feat(F16Traits<T>::lo(w), off, p.feature) * cscale,
                                               feat(F16Traits<T>::hi(w), off, p.feature) * cscale);
      }
  }
  // ---- O += A . KVW^T  (KVW: [d_out rows x d_k] K-major, d_k chunk kk/4, +32 bytes per K=16 step inside the chunk)
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < HD / 16; ++kk)
    wgmma_f16_rs<HD, kBF16, 0>(o, qa[kk], make_desc_kmajor_sw128(kvw_smem + (kk >> 2) * (HD * 128)) + uint64_t((kk & 3) * 2));
  wgmma_commit();
  wgmma_wait<0>();
  reg_fence(o);
#pragma unroll
  for (int kk = 0; kk < HD / 16; ++kk) reg_fence(qa[kk]);

  // ---- out = T( O / l + proj_b )
  if constexpr (kTile) {   // this thread's rows lane / 4 + {0, 8} of the tile, over the query rows it was read from
    __syncwarp();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float inv_l = kBF16 ? 1.0f / l_tot[h] : 1.0f / l_tot[h] * out_scale[h];
      const uint32_t row_s = tile_s + ((lane >> 2) + 8 * h) * 128 + 2 * cq;
#pragma unroll
      for (int c = 0; c < HD / 8; ++c) {
        const float2 pb = __ldg(reinterpret_cast<const float2*>(p.proj_b + 8 * c + cq));
        if constexpr (kVL)
          sts_u32(row_s + (c >> 3) * tile.chunk + (((c & 7) ^ (lane >> 2)) << 4),
                  qrow0 + 8 * h < n ? F16Traits<T>::pack(fmaf(o[4 * c + 2 * h], inv_l, pb.x), fmaf(o[4 * c + 2 * h + 1], inv_l, pb.y))
                                    : 0u);
        else
          sts_u32(row_s + (c >> 3) * tile.chunk + (((c & 7) ^ (lane >> 2)) << 4),
                  F16Traits<T>::pack(fmaf(o[4 * c + 2 * h], inv_l, pb.x), fmaf(o[4 * c + 2 * h + 1], inv_l, pb.y)));
      }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
#pragma unroll
      for (int c = 0; c < HD / 64; ++c) tma_store_4d(tile.tmap_out, tile.smem + c * tile.chunk, c * 64, hh, tile.row, b);
      tma_store_commit();
      tma_store_wait_read<0>();   // the shared memory stays the CTA's until the copy has read it
    }
  } else {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t qr = qrow0 + 8 * h;
      if (qr >= p.l) continue;
      const float inv_l = kBF16 ? 1.0f / l_tot[h] : 1.0f / l_tot[h] * out_scale[h];
      T* orow = static_cast<T*>(p.out) + ((int64_t(b) * p.l + qr) * p.h + hh) * HD;
#pragma unroll
      for (int c = 0; c < HD / 8; ++c) {
        const float2 pb = __ldg(reinterpret_cast<const float2*>(p.proj_b + 8 * c + cq));
        uint32_t packed = F16Traits<T>::pack(fmaf(o[4 * c + 2 * h], inv_l, pb.x), fmaf(o[4 * c + 2 * h + 1], inv_l, pb.y));
        if constexpr (kVL) packed = qr < n ? packed : 0u;
        *reinterpret_cast<uint32_t*>(orow + 8 * c + cq) = packed;
      }
    }
  }
}

// 128-row query blocks.  CTA = 2 consumer warpgroups + 1 TMA warp; warpgroup g owns query rows [64g, 64g+64) of the block.
// kLse: the sparse branch alone for the training path (sla_attn_bwd.cu): store_o_lse instead of the KVW load and the linear branch.
// kF8V (INT8 Q/K, HD = 128): e4m3 P.V on the [b, h, d, lk_pad] codes of tdb200_sla_quant_v_fp8 (PvOps), unscaled by v_scale.
template <typename T, int HD, bool kQK16, bool kLse = false, bool kF8V = false, bool kVL = false>
__global__ void __launch_bounds__(kThreads, 1)
sla_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                    const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_kvw, AttnParams p,
                    const __grid_constant__ CUtensorMap tmap_q16, const __grid_constant__ CUtensorMap tmap_out) {
  static_assert(!(kVL && (kLse || kF8V)), "per-entry lengths serve the inference kernels with 16-bit P.V");
  using L = Lay<HD, kQK16, BLKQ, BLKK, kF8V>;
  using PV = PvOps<T, HD, BLKK, kF8V>;
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, stays a shared-space pointer
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBars);
  uint16_t* s_lut = reinterpret_cast<uint16_t*>(smem + L::kOffLut);                 // [topk] key-block ids
  float* s_ksc = reinterpret_cast<float*>(smem + L::kOffLut + ((p.topk * 2 + 15) & ~15));  // [topk] k_scale of those blocks

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  const int bh = b * p.h + hh;
  const int n = kVL ? keys_of<true>(p.seq_lens, p.l, b) : p.l;   // kVL: the entry's rows, queries and keys alike
  if constexpr (kVL)
    if (m_blk * BLKQ >= n) {   // the block lies wholly past the entry's rows
      vl_store_zero_block<HD>(p, m_blk * BLKQ, BLKQ, b, hh);
      return;
    }
  const int T_blocks = kVL ? vl_topk(p, b, n, BLKK) : p.topk;
  // kVL: the consumers read the entry's length and LUT entry count from shared memory where they use them (beside the
  // barriers, 13 of the slot's 32), so that neither holds a register across the LUT walk: at 168 registers that spills.
  const uint32_t s_vl = smem_u32(smem + L::kOffBars + 128);
  auto keys_n = [&]() { return kVL ? lds_s32(s_vl) : p.lk; };
  auto n_blocks = [&]() { return kVL ? lds_s32(s_vl + 4) : p.topk; };

  if (threadIdx.x == 0) {
    if constexpr (kVL) {
      sts_u32(s_vl, uint32_t(n));
      sts_u32(s_vl + 4, uint32_t(T_blocks));
    }
    mbar_init(&bars[kQFull], 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&bars[kKFull + i], 1);
      mbar_init(&bars[kKEmpty + i], kConsumerWarps);
      mbar_init(&bars[kVFull + i], 1);
      mbar_init(&bars[kVEmpty + i], kConsumerWarps);
    }
    mbar_fence_init();
  }
  {
    const int32_t* lut_row = p.lut + (int64_t(bh) * p.mblk + m_blk) * p.topk;
    const float* ksc_row = p.k_scale + int64_t(bh) * p.nblk;
    for (int i = threadIdx.x; i < T_blocks; i += kThreads) {
      const int blk = __ldg(lut_row + i);
      s_lut[i] = static_cast<uint16_t>(blk);
      s_ksc[i] = kQK16 ? 1.0f : __ldg(ksc_row + blk);
    }
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // =============================================================== TMA producer
    if constexpr (kVL) {   // the loads of the code below, but the straddling V block from vl_load_v_block, by the whole warp
      if (lane == 0) {
        tma_prefetch_desc(&tmap_q);
        tma_prefetch_desc(&tmap_k);
        tma_prefetch_desc(&tmap_v);
        tma_prefetch_desc(&tmap_kvw);
        mbar_expect_tx(&bars[kQFull], L::kQBytes + L::kWBytes + L::kQ16Bytes);
        if constexpr (kQK16) {
#pragma unroll
          for (int c = 0; c < HD / 64; ++c)
            tma_load_4d(smem + L::kOffQ + c * (BLKQ * 128), &tmap_q, &bars[kQFull], c * 64, hh, m_blk * BLKQ, b);
        } else {
          tma_prefetch_desc(&tmap_q16);
          tma_prefetch_desc(&tmap_out);
          tma_load_4d(smem + L::kOffQ, &tmap_q, &bars[kQFull], 0, m_blk * BLKQ, bh, 0);
#pragma unroll
          for (int c = 0; c < HD / 64; ++c)
            tma_load_4d(smem + L::kOffQ16 + c * (BLKQ * 128), &tmap_q16, &bars[kQFull], c * 64, hh, m_blk * BLKQ, b);
        }
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(smem + L::kOffW + c * (HD * 128), &tmap_kvw, &bars[kQFull], c * 64, 0, bh, 0);
      }
      for (int j = 0; j < T_blocks; ++j) {
        const int st = j % kStages;
        const uint32_t ph = ((j / kStages) & 1) ^ 1;
        const int blk = s_lut[j];
        uint8_t* sk = smem + L::kOffK + st * L::kKBytes;
        uint8_t* sv = smem + L::kOffV + st * L::kVBytes;
        const int valid = n - blk * BLKK;
        if (lane == 0) {
          mbar_wait(&bars[kKEmpty + st], ph);
          mbar_expect_tx(&bars[kKFull + st], L::kKBytes);
          if constexpr (kQK16) {
#pragma unroll
            for (int c = 0; c < HD / 64; ++c)
              tma_load_4d(sk + c * (BLKK * 128), &tmap_k, &bars[kKFull + st], c * 64, hh, blk * BLKK, b);
          } else {
            tma_load_4d(sk, &tmap_k, &bars[kKFull + st], 0, blk * BLKK, hh, b);
          }
          mbar_wait(&bars[kVEmpty + st], ph);
          if (valid >= BLKK) {
            mbar_expect_tx(&bars[kVFull + st], L::kVBytes);
#pragma unroll
            for (int c = 0; c < HD / 64; ++c)
              tma_load_4d(sv + c * (BLKK * 128), &tmap_v, &bars[kVFull + st], c * 64, hh, blk * BLKK, b);
          }
        }
        if (valid < BLKK) {
          __syncwarp();   // lane 0 saw the stage empty
          vl_load_v_block<T, HD, BLKK>(sv, p, b, hh, blk, valid, lane);
          fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) mbar_arrive(&bars[kVFull + st]);
        }
      }
      return;
    }
    // The producer of the kernels without kVL.  The kVL branch above is a copy of its load schedule (it differs only in the
    // straddling V block): a change to one belongs in both.  The copy keeps these instantiations' code as it was.
    if (lane == 0) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
      if constexpr (!kLse) tma_prefetch_desc(&tmap_kvw);
      mbar_expect_tx(&bars[kQFull], L::kQBytes + (kLse ? 0 : L::kWBytes) + L::kQ16Bytes);
      if constexpr (kQK16) {  // 16-bit Q rows from [B,L,H,D]: HD/64 chunks of 128 rows x 128 B
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(smem + L::kOffQ + c * (BLKQ * 128), &tmap_q, &bars[kQFull], c * 64, hh, m_blk * BLKQ, b);
      } else {
        tma_prefetch_desc(&tmap_q16);
        tma_prefetch_desc(&tmap_out);
        tma_load_4d(smem + L::kOffQ, &tmap_q, &bars[kQFull], 0, m_blk * BLKQ, bh, 0);
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)  // the same rows in 16 bits, for phi(q)
          tma_load_4d(smem + L::kOffQ16 + c * (BLKQ * 128), &tmap_q16, &bars[kQFull], c * 64, hh, m_blk * BLKQ, b);
      }
      if constexpr (!kLse) {
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)  // KVW: d_k chunk c of the [d_out, d_k] matrix of this head
          tma_load_4d(smem + L::kOffW + c * (HD * 128), &tmap_kvw, &bars[kQFull], c * 64, 0, bh, 0);
      }
      for (int j = 0; j < T_blocks; ++j) {
        const int st = j % kStages;
        const uint32_t ph = ((j / kStages) & 1) ^ 1;
        const int blk = s_lut[j];
        mbar_wait(&bars[kKEmpty + st], ph);
        mbar_expect_tx(&bars[kKFull + st], L::kKBytes);
        uint8_t* sk = smem + L::kOffK + st * L::kKBytes;
        if constexpr (kQK16) {
#pragma unroll
          for (int c = 0; c < HD / 64; ++c)
            tma_load_4d(sk + c * (BLKK * 128), &tmap_k, &bars[kKFull + st], c * 64, hh, blk * BLKK, b);
        } else {
          tma_load_4d(sk, &tmap_k, &bars[kKFull + st], 0, blk * BLKK, hh, b);
        }
        mbar_wait(&bars[kVEmpty + st], ph);
        mbar_expect_tx(&bars[kVFull + st], L::kVBytes);
        uint8_t* sv = smem + L::kOffV + st * L::kVBytes;
        if constexpr (kF8V) {
          tma_load_4d(sv, &tmap_v, &bars[kVFull + st], blk * BLKK, 0, hh, b);
        } else {
#pragma unroll
          for (int c = 0; c < HD / 64; ++c)
            tma_load_4d(sv + c * (BLKK * 128), &tmap_v, &bars[kVFull + st], c * 64, hh, blk * BLKK, b);
        }
      }
    }
    return;
  }

  // =============================================================== consumer warpgroups
  const int wg = warp >> 2, w4 = warp & 3;
  const int r_lo = wg * 64 + w4 * 16 + (lane >> 2);   // rows r_lo and r_lo + 8 of the block (fragment layout, common.cuh)
  const int cq = 2 * (lane & 3);                       // column pair offset inside every 8-column slice
  const uint32_t sbase = smem_u32(smem);
  const float qsc = (kQK16 ? 1.0f : __ldg(p.q_scale + int64_t(bh) * p.mblk + m_blk)) * p.sm_scale * kLog2e;

  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_used[2] = {-INFINITY, -INFINITY}, l_part[2] = {0.f, 0.f};  // l_part: this thread's columns of the row sum

  // Software pipeline, per warpgroup (the FA3 order): S_{j+1} = Q.K_{j+1}^T and O += P_j.V_j are issued back to back as two
  // commit groups, and the softmax of S_{j+1} runs while P_j.V_j is still on the tensor core.  Per element the steps and their
  // order are those of softmax_step and pv_step: l is scaled before it adds an entry's P, O is scaled after the previous P.V
  // retired and before this one, and the entries accumulate in LUT order.  Every P.V retires inside its own iteration: with one
  // still in flight across the loop's back edge, ptxas no longer proves which group a wait retires and serialises every wgmma
  // of the kernel (C7514).
  const uint32_t sq = sbase + L::kOffQ + wg * (64 * HD);
  ScoreAcc<kQK16> sacc[BLKK / 2];   // S_{j+1} in flight
  float s[BLKK / 2];                // S_j, then P_j
  typename PV::Frag pa;             // P_j, read by the P.V in flight
  typename PV::Acc pacc;            // kF8V: P_j.V_j alone, added to O once retired
  bool rescale[2];
  float alpha[2];
  mbar_wait(&bars[kQFull], 0);
  if constexpr (kF8V) {
    // e4m3 P.V gives each block's P.V an accumulator of its own (PvOps), and that beside O, S_{j+1} and P_j does not fit in
    // this kernel's 168 registers: the steps of an entry run one after the other, as in the 64-row kernel.
    for (int j = 0; j < n_blocks(); ++j) {
      const int st = j % kStages;
      mbar_wait(&bars[kKFull + st], (j / kStages) & 1);
      score_issue<kQK16, HD, BLKK, kBF16>(sacc, sq, BLKQ * 128, sbase + L::kOffK + st * L::kKBytes);
      wgmma_wait<0>();
      warp_release(&bars[kKEmpty + st], lane);
      softmax_p_i8<BLKK>(sacc, s, qsc * s_ksc[j], m_used, l_part, rescale, alpha, keys_n() - int(s_lut[j]) * BLKK, cq, j == 0);
      rescale_o<HD>(o, rescale, alpha);
      PV::pack(s, pa);
      mbar_wait(&bars[kVFull + st], (j / kStages) & 1);
      PV::step(o, pacc, pa, sbase + L::kOffV + st * L::kVBytes);
      warp_release(&bars[kVEmpty + st], lane);
    }
  } else {
    mbar_wait(&bars[kKFull], 0);
    score_issue<kQK16, HD, BLKK, kBF16>(sacc, sq, BLKQ * 128, sbase + L::kOffK);
    wgmma_wait<0>();
    // valid < 64 only in the ragged last key block
    if constexpr (kQK16) {
      score_finish<kQK16, BLKK>(sacc, s, qsc * s_ksc[0]);
      warp_release(&bars[kKEmpty], lane);
      softmax_p<BLKK>(s, m_used, l_part, rescale, alpha, keys_n() - int(s_lut[0]) * BLKK, cq, true);
    } else {
      warp_release(&bars[kKEmpty], lane);
      softmax_p_i8<BLKK>(sacc, s, qsc * s_ksc[0], m_used, l_part, rescale, alpha, keys_n() - int(s_lut[0]) * BLKK, cq, true);
    }
    for (int j = 0; j < n_blocks(); ++j) {
      const int st = j % kStages, st1 = (j + 1) % kStages;
      const bool next = j + 1 < n_blocks();
      if (next) {
        mbar_wait(&bars[kKFull + st1], ((j + 1) / kStages) & 1);
        score_issue<kQK16, HD, BLKK, kBF16>(sacc, sq, BLKQ * 128, sbase + L::kOffK + st1 * L::kKBytes);
      }
      rescale_o<HD>(o, rescale, alpha);
      PV::pack(s, pa);
      mbar_wait(&bars[kVFull + st], (j / kStages) & 1);
      PV::issue(o, pacc, pa, sbase + L::kOffV + st * L::kVBytes);
      wgmma_wait<1>();                                    // S_{j+1} retired, P_j.V_j may still run
      if (next) {
        if constexpr (kQK16) {
          score_finish<kQK16, BLKK>(sacc, s, qsc * s_ksc[j + 1]);
          warp_release(&bars[kKEmpty + st1], lane);
          softmax_p<BLKK>(s, m_used, l_part, rescale, alpha, keys_n() - int(s_lut[j + 1]) * BLKK, cq, false);
        } else {
          warp_release(&bars[kKEmpty + st1], lane);
          softmax_p_i8<BLKK>(sacc, s, qsc * s_ksc[j + 1], m_used, l_part, rescale, alpha, keys_n() - int(s_lut[j + 1]) * BLKK, cq,
                             false);
        }
      }
      wgmma_wait<0>();
      PV::fence(o, pacc, pa);
      warp_release(&bars[kVEmpty + st], lane);
    }
  }
  if constexpr (kF8V) unscale_o_f8v<HD>(o, p.v_scale + int64_t(bh) * HD, cq);
  if constexpr (kLse) {
    store_o_lse<T, HD>(o, m_used, l_part, p, int64_t(m_blk) * BLKQ + r_lo, cq, b, hh, bh);
  } else if constexpr (kQK16) {
    linear_branch_store<T, HD, false, kVL>(o, l_part, p, sbase + L::kOffW, int64_t(m_blk) * BLKQ + r_lo, cq, b, hh, bh, RowTile{}, keys_n());
  } else {
    const int row16 = wg * 64 + w4 * 16;   // this warp's 16 rows of the block
    const RowTile tile{smem + L::kOffQ16 + row16 * 128, BLKQ * 128, &tmap_out, m_blk * BLKQ + row16};
    linear_branch_store<T, HD, true, kVL>(o, l_part, p, sbase + L::kOffW, int64_t(m_blk) * BLKQ + r_lo, cq, b, hh, bh, tile, keys_n());
  }
}

// 64-row query blocks, on the entry-split schedule (sla_attn.cuh): both consumer warpgroups work on the same 64 query rows and
// take alternate LUT entries, each running its own online softmax, so one warpgroup's softmax overlaps the other's MMAs.  The
// producer is a whole warpgroup so that setmaxnreg can move registers to the consumers: at BK = 128, O (64) + S (64) + P (32)
// fp32 registers per thread do not fit in the 168 a 384-thread CTA starts with.  Two block families:
//   INT8 Q/K, BK = 128: SpargeAttn's Hopper block geometry (SLA/core.py:191-193, 226-229 on sm90); wgmma m64n128k32.
//   16-bit Q/K, BK = 64: SparseLinearAttention's default geometry (the reference's BLOCK_M = 64, BLOCK_N = 64 configuration
//   of SLA/kernel.py:21-82); wgmma m64n64k16 into fp32.
// After both loops warpgroup 1 hands its (m, l, O) to warpgroup 0, which merges the two states and then runs the linear
// branch and the output (linear_branch_store), or with kLse stores o_s and the row lse.
template <typename T, int HD, bool kQK16, int BK, bool kLse, bool kF8V = false, bool kVL = false>
__global__ void __launch_bounds__(split::kThreads, 1)
sla_attn_fwd_q64_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                        const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_kvw, AttnParams p,
                        const __grid_constant__ CUtensorMap tmap_q16, const __grid_constant__ CUtensorMap tmap_out) {
  constexpr int BQ = kBlkQ64;
  using L = Lay<HD, kQK16, BQ, BK, kF8V>;
  using PV = PvOps<T, HD, BK, kF8V>;
  // hand-off of warpgroup 1's state: HD/2 accumulator registers + m_used[2] + l_part[2] per thread, over the K and V rings
  static_assert((HD / 2 + 4) * 128 * 4 <= kStages * (L::kKBytes + L::kVBytes), "merge buffer does not fit in the ring");
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBars);
  uint16_t* s_lut = reinterpret_cast<uint16_t*>(smem + L::kOffLut);
  float* s_ksc = reinterpret_cast<float*>(smem + L::kOffLut + ((p.topk * 2 + 15) & ~15));  // INT8 only
  static_assert(!(kVL && (kLse || kF8V)), "per-entry lengths serve the inference kernels with 16-bit P.V");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  const int bh = b * p.h + hh;
  const int n = kVL ? keys_of<true>(p.seq_lens, p.l, b) : p.l;   // kVL: the entry's rows, queries and keys alike
  if constexpr (kVL)
    if (m_blk * BQ >= n) {   // the block lies wholly past the entry's rows
      vl_store_zero_block<HD>(p, m_blk * BQ, BQ, b, hh);
      return;
    }
  const int T_blocks = kVL ? vl_topk(p, b, n, BK) : p.topk;

  if (threadIdx.x == 0) split::init_barriers(bars);
  {
    const int32_t* lut_row = p.lut + (int64_t(bh) * p.mblk + m_blk) * p.topk;
    const float* ksc_row = p.k_scale + int64_t(bh) * p.nblk;
    for (int i = threadIdx.x; i < T_blocks; i += split::kThreads) {
      const int blk = __ldg(lut_row + i);
      s_lut[i] = static_cast<uint16_t>(blk);
      if constexpr (!kQK16) s_ksc[i] = __ldg(ksc_row + blk);
    }
  }
  __syncthreads();

  if (warp >= kConsumerWarps) {
    // =============================================================== TMA producer
    reg_dealloc<split::kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
      if constexpr (!kLse) tma_prefetch_desc(&tmap_kvw);
      mbar_expect_tx(&bars[split::kQFull], L::kQBytes + (kLse ? 0 : L::kWBytes) + L::kQ16Bytes);
      if constexpr (kQK16) {
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(smem + L::kOffQ + c * (BQ * 128), &tmap_q, &bars[split::kQFull], c * 64, hh, m_blk * BQ, b);
      } else {
        tma_prefetch_desc(&tmap_q16);
        tma_prefetch_desc(&tmap_out);
        tma_load_4d(smem + L::kOffQ, &tmap_q, &bars[split::kQFull], 0, m_blk * BQ, bh, 0);
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(smem + L::kOffQ16 + c * (BQ * 128), &tmap_q16, &bars[split::kQFull], c * 64, hh, m_blk * BQ, b);
      }
      if constexpr (!kLse) {
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(smem + L::kOffW + c * (HD * 128), &tmap_kvw, &bars[split::kQFull], c * 64, 0, bh, 0);
      }
      for (int j = 0; j < T_blocks; ++j) {
        const int st = j % kStages;
        const uint32_t ph = ((j / kStages) & 1) ^ 1;
        const int blk = s_lut[j];
        uint64_t* kfull = &bars[split::full(split::kKFull, j)];
        uint64_t* vfull = &bars[split::full(split::kVFull, j)];
        mbar_wait(&bars[split::kKEmpty + st], ph);
        mbar_expect_tx(kfull, L::kKBytes);
        uint8_t* sk = smem + L::kOffK + st * L::kKBytes;
        if constexpr (kQK16) {
#pragma unroll
          for (int c = 0; c < HD / 64; ++c) tma_load_4d(sk + c * (BK * 128), &tmap_k, kfull, c * 64, hh, blk * BK, b);
        } else {
          tma_load_4d(sk, &tmap_k, kfull, 0, blk * BK, hh, b);
        }
        mbar_wait(&bars[split::kVEmpty + st], ph);
        mbar_expect_tx(vfull, L::kVBytes);
        uint8_t* sv = smem + L::kOffV + st * L::kVBytes;
        if constexpr (kF8V) {
          tma_load_4d(sv, &tmap_v, vfull, blk * BK, 0, hh, b);
        } else {
#pragma unroll
          for (int c = 0; c < HD / 64; ++c) tma_load_4d(sv + c * (BK * 128), &tmap_v, vfull, c * 64, hh, blk * BK, b);
        }
      }
    }
    return;
  }

  // =============================================================== consumer warpgroups (same 64 rows, alternate LUT entries)
  reg_alloc<split::kConsumerRegs>();
  const int wg = warp >> 2, w4 = warp & 3;
  const int r_lo = w4 * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t sbase = smem_u32(smem);
  const float qsc = kQK16 ? p.sm_scale * kLog2e : __ldg(p.q_scale + int64_t(bh) * p.mblk + m_blk) * p.sm_scale * kLog2e;

  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_used[2] = {-INFINITY, -INFINITY}, l_part[2] = {0.f, 0.f};  // a warpgroup without entries keeps m = -inf, l = 0

  mbar_wait(&bars[split::kQFull], 0);
  for (int j = wg; j < T_blocks; j += 2) {
    const int st = j % kStages;
    const uint32_t ph = split::full_phase(j);
    const int blk = s_lut[j];
    const float sc = kQK16 ? qsc : qsc * s_ksc[j];
    const int valid = (kVL ? n : p.lk) - blk * BK;      // < BK only in the ragged last key block

    float s[BK / 2];
    typename PV::Frag pa;
    typename PV::Acc pacc;
    mbar_wait(&bars[split::full(split::kKFull, j)], ph);
    if constexpr (kQK16) {
      score_tile<kQK16, HD, BK, kBF16>(s, sbase + L::kOffQ, BQ * 128, sbase + L::kOffK + st * L::kKBytes, sc);
      warp_release(&bars[split::kKEmpty + st], lane);
      softmax_step<T, HD, BK>(s, o, m_used, l_part, pa, valid, cq, j == wg);
    } else {
      uint32_t si[BK / 2];
      score_issue<kQK16, HD, BK, kBF16>(si, sbase + L::kOffQ, BQ * 128, sbase + L::kOffK + st * L::kKBytes);
      wgmma_wait<0>();
      warp_release(&bars[split::kKEmpty + st], lane);
      bool rescale[2];
      float alpha[2];
      softmax_p_i8<BK>(si, s, sc, m_used, l_part, rescale, alpha, valid, cq, j == wg);
      rescale_o<HD>(o, rescale, alpha);
      PV::pack(s, pa);
    }
    mbar_wait(&bars[split::full(split::kVFull, j)], ph);
    if constexpr (kVL)
      if (valid < BK) {   // the straddling key block, this warpgroup's alone: V rows past the entry's keys are padding
        zero_query_rows(smem + L::kOffV + st * L::kVBytes, BK, HD / 64, valid, BK, threadIdx.x & 127);
        fence_proxy_async_smem();
        named_bar_sync(2 + wg, 128);
      }
    PV::step(o, pacc, pa, sbase + L::kOffV + st * L::kVBytes);
    warp_release(&bars[split::kVEmpty + st], lane);
  }

  const Handoff x = handoff_wg1_to_wg0(smem + L::kOffK, wg, 1, [&](const Handoff& x) {
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) x[i] = o[i];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      x[HD / 2 + h] = m_used[h];
      x[HD / 2 + 2 + h] = l_part[h];
    }
  });
  if (wg == 1) return;
  float a0[2], a1[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {  // warpgroup 0 always has entry 0, so its maximum is finite and exp2(-inf - m) = 0 drops an empty state
    const float m1 = x[HD / 2 + h], l1 = x[HD / 2 + 2 + h];
    const float mx = fmaxf(m_used[h], m1);
    a0[h] = fast_exp2(m_used[h] - mx);
    a1[h] = fast_exp2(m1 - mx);
    l_part[h] = fmaf(l_part[h], a0[h], l1 * a1[h]);
    m_used[h] = mx;
  }
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) {
    const int h = (i >> 1) & 1;
    o[i] = fmaf(o[i], a0[h], x[i] * a1[h]);
  }
  if constexpr (kF8V) unscale_o_f8v<HD>(o, p.v_scale + int64_t(bh) * HD, cq);
  const int64_t qrow0 = int64_t(m_blk) * BQ + r_lo;
  if constexpr (kLse) {
    store_o_lse<T, HD>(o, m_used, l_part, p, qrow0, cq, b, hh, bh);
  } else if constexpr (kQK16) {
    linear_branch_store<T, HD, false, kVL>(o, l_part, p, sbase + L::kOffW, qrow0, cq, b, hh, bh, RowTile{}, n);
  } else {
    const RowTile tile{smem + L::kOffQ16 + w4 * 16 * 128, BQ * 128, &tmap_out, m_blk * BQ + w4 * 16};
    linear_branch_store<T, HD, true, kVL>(o, l_part, p, sbase + L::kOffW, qrow0, cq, b, hh, bh, tile, n);
  }
}

template <typename T, int HD, bool kQK16, int kBQ, int kBK, bool kLse, bool kF8V, bool kVL = false>
constexpr auto attn_kernel() {
  if constexpr (kVL) {
    if constexpr (kBQ == kBlkQ64) return sla_attn_fwd_q64_kernel<T, HD, kQK16, kBK, false, false, true>;
    else return sla_attn_fwd_kernel<T, HD, kQK16, false, false, true>;
  } else if constexpr (kF8V) {
    if constexpr (kBQ == kBlkQ64) return sla_attn_fwd_q64_kernel<T, HD, kQK16, kBK, kLse, true>;
    else return sla_attn_fwd_kernel<T, HD, kQK16, kLse, true>;
  } else {
    if constexpr (kBQ == kBlkQ64) return sla_attn_fwd_q64_kernel<T, HD, kQK16, kBK, kLse>;
    else return sla_attn_fwd_kernel<T, HD, kQK16, kLse>;
  }
}

// kQK16: 16-bit Q and K in [b, l, h, d]; otherwise INT8 Q [b*h, l, d] and INT8 K [b, h, lk, d] (or [b, lk, h, d] when k_seq_major).
// kBQ x kBK: the block geometry, 128 x 64 (sla_attn_fwd_kernel), or with sla_attn_fwd_q64_kernel 64 x 128 (INT8 Q/K only)
// or 64 x 64 (16-bit Q/K only).
// kLse (16-bit only): sparse branch and row log-sum-exp into `lse`; kvw, ksum and proj_b are not read.
// kF8V (INT8 only, HD = 128): v is tdb200_sla_quant_v_fp8's e4m3 [b, h, d, lk_pad] with lk_pad = ceil(lk / kBK) * kBK, and
// v_scale its [b, h, d] channel scales.
template <int HD, bool kQK16, int kBQ = BLKQ, int kBK = BLKK, bool kLse = false, bool kF8V = false, bool kVL = false>
int launch(const void* q_op, const float* q_scale, const void* k_op, const float* k_scale, const void* v, const void* q, int dtype,
           const int32_t* lut, int64_t topk, const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
           int64_t l, int64_t lk, int64_t h, float sm_scale, int feature, bool k_seq_major, void* stream, float* lse = nullptr,
           const float* v_scale = nullptr, const int32_t* seq_lens = nullptr, const int32_t* topks = nullptr) {
  using L = Lay<HD, kQK16, kBQ, kBK, kF8V>;
  const int64_t d = HD;
  const int64_t mblk = cdiv64(l, kBQ), nblk = cdiv64(lk, kBK);
  if (topk <= 0 || topk > nblk) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: topk=%lld outside [1, %lld]", (long long)topk, (long long)nblk);
  if (nblk > 65535 || h > 65535 || b > 65535 || mblk > 0x7FFFFFFF) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: dimension too large");
  const size_t lut_bytes = ((size_t(topk) * 2 + 15) & ~size_t(15)) + size_t(topk) * 4;
  const size_t smem = 1024 + L::kOffLut + lut_bytes;
  if (smem > 227 * 1024) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: topk=%lld too large for on-chip LUT", (long long)topk);
  if (dtype != TDB200_DTYPE_BF16 && dtype != TDB200_DTYPE_FP16) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: dtype tag %d", dtype);
  if (int rc = require_sm90()) return rc;

  const CUtensorMapDataType t16 = dtype == TDB200_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const int sw8 = HD == 128 ? 128 : 64;
  CUtensorMap tq, tk, tv, tw, tq16, tout;
  if (kQK16) {  // 16-bit Q / K rows in the module layout [b, l, h, d]
    const uint64_t dq[4] = {uint64_t(d), uint64_t(h), uint64_t(l), uint64_t(b)};
    const uint64_t sq[3] = {uint64_t(d * 2), uint64_t(h * d * 2), uint64_t(l * h * d * 2)};
    const uint32_t bq[4] = {64, 1, kBQ, 1};
    if (int rc = make_tmap_4d(&tq, q_op, t16, 2, dq, sq, bq)) return rc;
    const uint64_t dk[4] = {uint64_t(d), uint64_t(h), uint64_t(lk), uint64_t(b)};
    const uint64_t sk[3] = {uint64_t(d * 2), uint64_t(h * d * 2), uint64_t(lk * h * d * 2)};
    const uint32_t bk[4] = {64, 1, kBK, 1};
    if (int rc = make_tmap_4d(&tk, k_op, t16, 2, dk, sk, bk)) return rc;
  } else {
    {
      const uint64_t dims[4] = {uint64_t(d), uint64_t(l), uint64_t(b * h), 1};
      const uint64_t str[3] = {uint64_t(d), uint64_t(l * d), uint64_t(b * h * l * d)};
      const uint32_t box[4] = {uint32_t(HD), kBQ, 1, 1};
      if (int rc = make_tmap_4d(&tq, q_op, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, dims, str, box, sw8)) return rc;
    }
    {
      // INT8 K: head-major [b, h, lk, d] (tdb200_sla_quant_qk) or, for sequence-parallel callers, the gathered [b, lk, h, d]
      const uint64_t dims[4] = {uint64_t(d), uint64_t(lk), uint64_t(h), uint64_t(b)};
      const uint64_t str[3] = {uint64_t(k_seq_major ? h * d : d), uint64_t(k_seq_major ? d : lk * d), uint64_t(h * lk * d)};
      const uint32_t box[4] = {uint32_t(HD), kBK, 1, 1};
      if (int rc = make_tmap_4d(&tk, k_op, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, dims, str, box, sw8)) return rc;
    }
  }
  if (kF8V) {   // [kBK keys x HD channels] boxes of the transposed codes, key-block rows of kBK bytes
    const uint64_t lk_pad = uint64_t(nblk * kBK);
    const uint64_t dims[4] = {lk_pad, uint64_t(d), uint64_t(h), uint64_t(b)};
    const uint64_t str[3] = {lk_pad, uint64_t(d) * lk_pad, uint64_t(h * d) * lk_pad};
    const uint32_t box[4] = {uint32_t(kBK), uint32_t(HD), 1, 1};
    if (int rc = make_tmap_4d(&tv, v, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, dims, str, box, kBK)) return rc;
  } else {
    const uint64_t dims[4] = {uint64_t(d), uint64_t(h), uint64_t(lk), uint64_t(b)};
    const uint64_t str[3] = {uint64_t(d * 2), uint64_t(h * d * 2), uint64_t(lk * h * d * 2)};
    const uint32_t box[4] = {64, 1, kBK, 1};
    if (int rc = make_tmap_4d(&tv, v, t16, 2, dims, str, box)) return rc;
  }
  if (kQK16) {
    tq16 = tout = tv;  // not read
  } else {  // INT8: the 16-bit query rows for phi(q), and the output, both [b, l, h, d] in 16-bit boxes of 64 columns
    const uint64_t dims[4] = {uint64_t(d), uint64_t(h), uint64_t(l), uint64_t(b)};
    const uint64_t str[3] = {uint64_t(d * 2), uint64_t(h * d * 2), uint64_t(l * h * d * 2)};
    const uint32_t bq[4] = {64, 1, kBQ, 1}, bo[4] = {64, 1, 16, 1};
    if (int rc = make_tmap_4d(&tq16, q, t16, 2, dims, str, bq)) return rc;
    if (int rc = make_tmap_4d(&tout, out, t16, 2, dims, str, bo)) return rc;
  }
  if (kLse) {
    tw = tv;  // not read
  } else {
    const uint64_t dims[4] = {uint64_t(d), uint64_t(d), uint64_t(b * h), 1};
    const uint64_t str[3] = {uint64_t(d * 2), uint64_t(d * d * 2), uint64_t(b * h * d * d * 2)};
    const uint32_t box[4] = {64, uint32_t(HD), 1, 1};
    if (int rc = make_tmap_4d(&tw, kvw, t16, 2, dims, str, box)) return rc;
  }
  AttnParams p;
  p.q_scale = q_scale;
  p.k_scale = k_scale;
  p.q = q;
  p.lut = lut;
  p.ksum = ksum;
  p.proj_b = proj_b;
  p.out = out;
  p.l = int(l);
  p.lk = int(lk);
  p.h = int(h);
  p.mblk = int(mblk);
  p.nblk = int(nblk);
  p.topk = int(topk);
  p.feature = feature;
  p.sm_scale = sm_scale;
  p.lse = lse;
  p.v_scale = v_scale;
  p.seq_lens = seq_lens;
  p.topks = topks;
  p.v = v;
  dim3 grid(static_cast<unsigned>(mblk), static_cast<unsigned>(h), static_cast<unsigned>(b));
  const int threads = kBQ == kBlkQ64 ? split::kThreads : kThreads;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define TDB_ATTN(T)                                                                                                   \
  do {                                                                                                                \
    const auto kern = attn_kernel<T, HD, kQK16, kBQ, kBK, kLse, kF8V, kVL>();                                                    \
    if (int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)), \
                            "cudaFuncSetAttribute(sla_attn)"))                                                        \
      return rc;                                                                                                      \
    kern<<<grid, threads, smem, st>>>(tq, tk, tv, tw, p, tq16, tout);                                                 \
    return check_launch("sla_attn_fwd_kernel");                                                                       \
  } while (0)
  if (dtype == TDB200_DTYPE_BF16) TDB_ATTN(__nv_bfloat16);
  TDB_ATTN(__half);
#undef TDB_ATTN
}

int check_common(const void* q_op, const void* k_op, const void* v, const void* q, const int32_t* lut, const void* kvw,
                 const float* ksum, const float* proj_b, void* out, int64_t b, int64_t l, int64_t lk, int64_t h) {
  if (!q_op || !k_op || !v || !q || !lut || !kvw || !ksum || !proj_b || !out)
    return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: null pointer");
  if (b <= 0 || l <= 0 || lk <= 0 || h <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: bad shape");
  return 0;
}

}  // namespace

// INT8 Q [b*h, l, d]; INT8 K head-major [b, h, lk, d] or, with k_seq_major, the [1, lk, h, d] slab sequence-parallel ranks
// all-gather.  Both producers load K at (0, blk*BK, head, b) over the dims (d, lk, h, b), so the sequence-major layout is only a
// different set of tensor-map strides.  (blkq, blkk) = (128, 64) runs sla_attn_fwd_kernel, (64, 128) sla_attn_fwd_q64_kernel.
extern "C" int tdb200_sla_attn_fwd(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                                   const void* v, const void* q, int dtype, const int32_t* lut, int64_t topk,
                                   const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
                                   int64_t l, int64_t lk, int64_t h, int64_t d, float sm_scale, int feature, int64_t blkq,
                                   int64_t blkk, int k_seq_major, void* stream) {
  const bool hopper = blkq == kBlkQ64 && blkk == kHopperBlkK;
  if (!hopper && !(blkq == BLKQ && blkk == BLKK))
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: block sizes (%lld, %lld) (BLKQ x BLKK = 128 x 64 or 64 x 128)",
                (long long)blkq, (long long)blkk);
  if (int rc = check_common(q_i8, k_i8, v, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (!q_scale || !k_scale) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: null pointer");
  if (k_seq_major) {
    if (d != 128)
      return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: head dim %lld (sequence-major K is implemented for d=128)", (long long)d);
    if (feature != 0)
      return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: feature map tag %d (sequence-major K is implemented for softmax)", feature);
    if (b != 1)
      return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: batch %lld (the gathered [lk_pad, h, d] key slab is one sequence)", (long long)b);
  } else {
    if (d != 64 && d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: head dim %lld (64 or 128, SLA/core.py:207)", (long long)d);
    if (feature < 0 || feature > 2) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: feature map tag %d", feature);
  }
#define TDB_LAUNCH(HD, BQ, BK)                                                                                             \
  return launch<HD, false, BQ, BK>(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum, proj_b, out, b, l, lk, h, \
                                   sm_scale, feature, k_seq_major != 0, stream)
  // the order of these instantiations is the order nvcc compiles the kernels in, which changes the code it emits for them
  if (d == 128) {
    if (!hopper) TDB_LAUNCH(128, BLKQ, BLKK);
    TDB_LAUNCH(128, kBlkQ64, kHopperBlkK);
  }
  if (!hopper) TDB_LAUNCH(64, BLKQ, BLKK);
  TDB_LAUNCH(64, kBlkQ64, kHopperBlkK);
#undef TDB_LAUNCH
}

namespace {
int check_blocks16(const char* what, int64_t blkq, int64_t blkk) {
  if ((blkq == BLKQ || blkq == kBlkQ64) && blkk == BLKK) return 0;
  return fail(TDB200_ERR_UNSUPPORTED, "%s: block sizes (%lld, %lld) (BLKQ x BLKK = 128 x 64 or 64 x 64)", what, (long long)blkq,
              (long long)blkk);
}

// The four 16-bit kernels, instantiated in this order: the (128, 64) ones first, because nvcc's output depends on the order.
int launch16(bool with_lse, int64_t blkq, const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
             const void* kvw, const float* ksum, const float* proj_b, void* out, float* lse, int64_t b, int64_t l, int64_t lk,
             int64_t h, float sm_scale, int feature, void* stream) {
#define TDB_LAUNCH16(BQ, LSE)                                                                                                  \
  return launch<128, true, BQ, BLKK, LSE>(q, nullptr, k, nullptr, v, q, dtype, lut, topk, kvw, ksum, proj_b, out, b, l, lk, h, \
                                          sm_scale, feature, false, stream, lse)
  if (blkq == BLKQ) {
    if (!with_lse) TDB_LAUNCH16(BLKQ, false);
    TDB_LAUNCH16(BLKQ, true);
  }
  if (!with_lse) TDB_LAUNCH16(kBlkQ64, false);
  TDB_LAUNCH16(kBlkQ64, true);
#undef TDB_LAUNCH16
}
}  // namespace

// 16-bit Q/K read from the module layout: (blkq, blkk) = (128, 64) runs sla_attn_fwd_kernel, (64, 64) sla_attn_fwd_q64_kernel.
extern "C" int tdb200_sla_attn16_fwd(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
                                     const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b, int64_t l,
                                     int64_t lk, int64_t h, int64_t d, float sm_scale, int feature, int64_t blkq, int64_t blkk,
                                     void* stream) {
  if (int rc = check_blocks16("sla_attn16_fwd", blkq, blkk)) return rc;
  if (int rc = check_common(q, k, v, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: head dim %lld (this kernel implements d=128)", (long long)d);
  if (feature < 0 || feature > 2) return fail(TDB200_ERR_INVALID_ARG, "sla_attn16_fwd: feature map tag %d", feature);
  return launch16(false, blkq, q, k, v, dtype, lut, topk, kvw, ksum, proj_b, out, nullptr, b, l, lk, h, sm_scale, feature, stream);
}

// The sparse branch of tdb200_sla_attn16_fwd with its row log-sum-exp, the forward half of the training path.
extern "C" int tdb200_sla_attn16_fwd_lse(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
                                         void* o_s, float* lse, int64_t b, int64_t l, int64_t h, int64_t d, float sm_scale,
                                         int64_t blkq, int64_t blkk, void* stream) {
  if (int rc = check_blocks16("sla_attn16_fwd_lse", blkq, blkk)) return rc;
  if (!q || !k || !v || !lut || !o_s || !lse) return fail(TDB200_ERR_INVALID_ARG, "sla_attn16_fwd_lse: null pointer");
  if (b <= 0 || l <= 0 || h <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_attn16_fwd_lse: bad shape");
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn16_fwd_lse: head dim %lld (this kernel implements d=128)", (long long)d);
  return launch16(true, blkq, q, k, v, dtype, lut, topk, nullptr, nullptr, nullptr, o_s, lse, b, l, l, h, sm_scale, 0, stream);
}

extern "C" int tdb200_sla_attn_fwd_qk16(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
                                        const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
                                        int64_t l, int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream) {
  return tdb200_sla_attn16_fwd(q, k, v, dtype, lut, topk, kvw, ksum, proj_b, out, b, l, lk, h, d, sm_scale, 0, BLKQ, BLKK, stream);
}

extern "C" int tdb200_sla_attn_fwd_qk16_lse(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
                                            void* o_s, float* lse, int64_t b, int64_t l, int64_t h, int64_t d, float sm_scale,
                                            void* stream) {
  return tdb200_sla_attn16_fwd_lse(q, k, v, dtype, lut, topk, o_s, lse, b, l, h, d, sm_scale, BLKQ, BLKK, stream);
}

// tdb200_sla_attn_fwd with e4m3 P.V: v_fp8 / v_scale from tdb200_sla_quant_v_fp8 with the same blkk.  Its kernels are instantiated
// here, after every 16-bit-V kernel of this file, so that those compile as they did without them.
extern "C" int tdb200_sla_attn_fwd_fp8v(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                                        const uint8_t* v_fp8, const float* v_scale, const void* q, int dtype, const int32_t* lut,
                                        int64_t topk, const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
                                        int64_t l, int64_t lk, int64_t h, int64_t d, float sm_scale, int feature, int64_t blkq,
                                        int64_t blkk, int k_seq_major, void* stream) {
  const bool hopper = blkq == kBlkQ64 && blkk == kHopperBlkK;
  if (!hopper && !(blkq == BLKQ && blkk == BLKK))
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd_fp8v: block sizes (%lld, %lld) (BLKQ x BLKK = 128 x 64 or 64 x 128)",
                (long long)blkq, (long long)blkk);
  if (int rc = check_common(q_i8, k_i8, v_fp8, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (!q_scale || !k_scale || !v_scale) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd_fp8v: null pointer");
  if (!aligned16(v_fp8) || !aligned16(v_scale))
    return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd_fp8v: v_fp8 and v_scale must be 16-byte aligned");
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd_fp8v: head dim %lld (FP8 P.V is implemented for d=128)", (long long)d);
  if (feature < 0 || feature > 2) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd_fp8v: feature map tag %d", feature);
  if (k_seq_major && feature != 0)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd_fp8v: feature map tag %d (sequence-major K is implemented for softmax)", feature);
  if (k_seq_major && b != 1)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd_fp8v: batch %lld (the gathered [lk_pad, h, d] key slab is one sequence)",
                (long long)b);
  if (!hopper)
    return launch<128, false, BLKQ, BLKK, false, true>(q_i8, q_scale, k_i8, k_scale, v_fp8, q, dtype, lut, topk, kvw, ksum, proj_b,
                                                       out, b, l, lk, h, sm_scale, feature, k_seq_major != 0, stream, nullptr, v_scale);
  return launch<128, false, kBlkQ64, kHopperBlkK, false, true>(q_i8, q_scale, k_i8, k_scale, v_fp8, q, dtype, lut, topk, kvw, ksum,
                                                               proj_b, out, b, l, lk, h, sm_scale, feature, k_seq_major != 0, stream,
                                                               nullptr, v_scale);
}

// ---- per-entry lengths: the _vl twins of tdb200_sla_attn_fwd (INT8 Q/K, K head-major) and tdb200_sla_attn16_fwd, d = 128, l = lk.
// seq_lens [b] and topks [b] are device int32: entry b's rows below seq_lens[b] get the bits of the entry point without lengths
// called on entry b alone, cut to those rows, with its own LUT, topk, moments and scales; its rows past the length are zero.
// Their kernels are instantiated here, after every other kernel of this file.
namespace {
int check_vl(const char* what, const int32_t* seq_lens, const int32_t* topks, int64_t l, int64_t lk, int64_t d) {
  if (!seq_lens || !topks || (reinterpret_cast<uintptr_t>(seq_lens) & 3u) || (reinterpret_cast<uintptr_t>(topks) & 3u))
    return fail(TDB200_ERR_INVALID_ARG, "%s: seq_lens and topks must be non-null, 4-byte aligned int32 [b]", what);
  if (l != lk) return fail(TDB200_ERR_INVALID_ARG, "%s: l = %lld and lk = %lld (one length per entry: self-attention)", what,
                           (long long)l, (long long)lk);
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "%s: head dim %lld (per-entry lengths serve d = 128)", what, (long long)d);
  return 0;
}
}  // namespace

extern "C" int tdb200_sla_attn_fwd_vl(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                                      const void* v, const void* q, int dtype, const int32_t* lut, int64_t topk, const void* kvw,
                                      const float* ksum, const float* proj_b, void* out, int64_t b, int64_t l, int64_t lk,
                                      int64_t h, int64_t d, const int32_t* seq_lens, const int32_t* topks, float sm_scale,
                                      int feature, int64_t blkq, int64_t blkk, void* stream) {
  const bool hopper = blkq == kBlkQ64 && blkk == kHopperBlkK;
  if (!hopper && !(blkq == BLKQ && blkk == BLKK))
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd_vl: block sizes (%lld, %lld) (BLKQ x BLKK = 128 x 64 or 64 x 128)",
                (long long)blkq, (long long)blkk);
  if (int rc = check_common(q_i8, k_i8, v, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (!q_scale || !k_scale) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd_vl: null pointer");
  if (int rc = check_vl("sla_attn_fwd_vl", seq_lens, topks, l, lk, d)) return rc;
  if (feature < 0 || feature > 2) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd_vl: feature map tag %d", feature);
  if (!hopper)
    return launch<128, false, BLKQ, BLKK, false, false, true>(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum,
                                                              proj_b, out, b, l, lk, h, sm_scale, feature, false, stream, nullptr,
                                                              nullptr, seq_lens, topks);
  return launch<128, false, kBlkQ64, kHopperBlkK, false, false, true>(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw,
                                                                      ksum, proj_b, out, b, l, lk, h, sm_scale, feature, false,
                                                                      stream, nullptr, nullptr, seq_lens, topks);
}

extern "C" int tdb200_sla_attn16_fwd_vl(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
                                        const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b, int64_t l,
                                        int64_t lk, int64_t h, int64_t d, const int32_t* seq_lens, const int32_t* topks,
                                        float sm_scale, int feature, int64_t blkq, int64_t blkk, void* stream) {
  if (int rc = check_blocks16("sla_attn16_fwd_vl", blkq, blkk)) return rc;
  if (int rc = check_common(q, k, v, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (int rc = check_vl("sla_attn16_fwd_vl", seq_lens, topks, l, lk, d)) return rc;
  if (feature < 0 || feature > 2) return fail(TDB200_ERR_INVALID_ARG, "sla_attn16_fwd_vl: feature map tag %d", feature);
  if (blkq == BLKQ)
    return launch<128, true, BLKQ, BLKK, false, false, true>(q, nullptr, k, nullptr, v, q, dtype, lut, topk, kvw, ksum, proj_b, out,
                                                             b, l, lk, h, sm_scale, feature, false, stream, nullptr, nullptr,
                                                             seq_lens, topks);
  return launch<128, true, kBlkQ64, BLKK, false, false, true>(q, nullptr, k, nullptr, v, q, dtype, lut, topk, kvw, ksum, proj_b, out,
                                                              b, l, lk, h, sm_scale, feature, false, stream, nullptr, nullptr,
                                                              seq_lens, topks);
}
