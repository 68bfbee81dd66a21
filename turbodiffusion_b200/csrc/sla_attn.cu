// a9 + a10. Fused SageSLA attention forward for one (128-row query block, head, batch) per CTA:
//   block-sparse INT8 Q.K^T -> online softmax (exp2) -> 16-bit P.V, then the linear branch phi(Q).KVW / (eps + phi(Q).ksum)
//   folded into the same accumulator, all in one wgmma kernel.
//   reference: Sage call site turbodiffusion/SLA/core.py:231-235 (arithmetic in third-party SpargeAttn, unpinned);
//   the in-tree statement of the same attention is the Triton kernel SLA/kernel.py:33-82 (tail masking :57-62, exp2 with
//   qk_scale*log2e :60, row sum from unrounded P :71, P cast before P.V :73); linear branch + merge SLA/core.py:243-253.
//
// CTA = 2 consumer warpgroups + 1 TMA warp.  Warpgroup g owns query rows [64g, 64g+64) of the block; every thread holds two
//   rows of the fragments (common.cuh): S[64 x 64] in 32 registers (wgmma m64n64, A = Q and B = K from shared memory),
//   P converted in registers straight into the A fragments of P.V (wgmma m64nHD, A from registers, B = V MN-major from
//   shared memory, so no transposed copy of V is ever materialised), and the O accumulator [64 x HD] in HD/2 registers.
//   Row maxima / sums are reduced across the four lanes that share a row.
//   After the last key block the linear branch adds A.KVW^T to O with A = phi(q) * l / den in registers, so that
//   O / l = softmax part + phi(q).KVW^T / den, and out = O / l + proj_b.
// Shared memory: Q | K ring | V ring (3 stages each; K and V released per warp as soon as their MMA retired) | KVW.
//   Q/K/KVW are K-major swizzled (128B rows, or 64B rows for 64-wide int8 heads).
// The O accumulator is only rescaled when a row maximum grows by more than 2^8 (lazy rescale): P stays <= 256, which
// bf16/fp32 hold exactly as well as P <= 1, and the final O / l normalisation is unchanged.
// Entry points: tdb200_sla_attn_fwd (INT8 Q/K, head-major K), _kseq (INT8 K in [b, lk, h, d]), _qk16 (16-bit Q/K read from
// the module layout [b, l, h, d], fp32 scores), _v2 (INT8, head dims 64 and 128, feature maps of the linear branch) and
// _blocks (_v2 with the block geometry as an argument; 64 x 128 blocks run sla_attn_fwd_q64_kernel, further down).
#include <type_traits>

#include "common.cuh"
#include "host_common.h"

namespace {
using namespace tdb;

constexpr int BLKQ = 128, BLKK = 64;
constexpr int kConsumerWarps = 8;
constexpr int kThreads = kConsumerWarps * 32 + 32;
constexpr int kStages = 3;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kRescaleThreshold = 8.0f;  // log2 domain

template <int HD, bool kQK16, int kBQ = BLKQ, int kBK = BLKK>
struct Lay {
  static constexpr uint32_t kQBytes = kQK16 ? kBQ * HD * 2 : kBQ * HD;     // 16-bit: HD/64 chunks of [128 rows x 128 B]
  static constexpr uint32_t kKBytes = kQK16 ? kBK * HD * 2 : kBK * HD;
  static constexpr uint32_t kVBytes = kBK * HD * 2;                        // HD/64 boxes of [kBK keys x 128 B]
  static constexpr uint32_t kWBytes = HD * HD * 2;                         // HD/64 d_k chunks of [HD rows x 128 B]
  static constexpr uint32_t kOffQ = 0;
  static constexpr uint32_t kOffK = kOffQ + kQBytes;
  static constexpr uint32_t kOffV = kOffK + kStages * kKBytes;
  static constexpr uint32_t kOffW = kOffV + kStages * kVBytes;
  static constexpr uint32_t kOffBars = kOffW + kWBytes;
  static constexpr uint32_t kOffLut = kOffBars + 256;
};

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
};

enum Bar { kQFull = 0, kKFull = 1 /*3*/, kKEmpty = 4 /*3*/, kVFull = 7 /*3*/, kVEmpty = 10 /*3*/, kNumBars = 13 };

__device__ __forceinline__ float feat(float x, float off_log2, int feature) {
  // softmax numerator exp(x - max) | elu(x)+1 | relu(x)
  if (feature == 0) return fast_exp2(fmaf(x, kLog2e, -off_log2));
  if (feature == 1) return x > 0.f ? x + 1.0f : fast_exp2(x * kLog2e);
  return fmaxf(x, 0.f);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// After the last key block, for the 64 query rows of one warpgroup (rows qrow0 + {0, 8} for this thread): the linear branch
// adds A.KVW^T to O, then out = T( O / l + proj_b ).  kvw_smem: the KVW tile (K-major, swizzled like Q).
template <typename T, int HD>
__device__ __forceinline__ void linear_branch_store(float (&o)[HD / 2], const float (&l_part)[2], const AttnParams& p,
                                                    uint32_t kvw_smem, int64_t qrow0, int cq, int b, int hh, int bh) {
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  const float l_tot[2] = {quad_sum(l_part[0]), quad_sum(l_part[1])};

  // ---- linear branch operand (SLA/core.py:243).  f_j = feature map numerator of the query row:
  //      E = sum f_j, F = sum f_j * ksum_j;  phi_j = f_j / E (softmax) or f_j;  den = 1e-5 + sum_j phi_j ksum_j;
  //      A_j = T(phi_j * l / den), so that O + A.KVW^T = l * (O/l + phi.KVW^T/den).
  //      This thread holds, for each K=16 step kk, the column pairs 16 kk + cq and 16 kk + 8 + cq of its two rows.
  uint32_t qa[HD / 16][4];
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
  const float* ks = p.ksum + int64_t(bh) * HD;
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
    float e = 0.f, f = 0.f;
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const uint32_t w = qa[kk][h + 2 * u];
        const float2 k2 = __ldg(reinterpret_cast<const float2*>(ks + 16 * kk + 8 * u + cq));
        const float a0 = feat(F16Traits<T>::lo(w), off, p.feature), a1 = feat(F16Traits<T>::hi(w), off, p.feature);
        e += a0 + a1;
        f = fmaf(a0, k2.x, fmaf(a1, k2.y, f));
      }
    const float E = quad_sum(e), F = quad_sum(f);
    const float inv_e = p.feature == 0 ? 1.0f / E : 1.0f;
    const float den = 1e-5f + F * inv_e;
    const float cscale = inv_e * l_tot[h] / den;
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
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t qr = qrow0 + 8 * h;
    if (qr >= p.l) continue;
    const float inv_l = 1.0f / l_tot[h];
    T* orow = static_cast<T*>(p.out) + ((int64_t(b) * p.l + qr) * p.h + hh) * HD;
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      const float2 pb = __ldg(reinterpret_cast<const float2*>(p.proj_b + 8 * c + cq));
      *reinterpret_cast<uint32_t*>(orow + 8 * c + cq) =
          F16Traits<T>::pack(fmaf(o[4 * c + 2 * h], inv_l, pb.x), fmaf(o[4 * c + 2 * h + 1], inv_l, pb.y));
    }
  }
}

template <typename T, int HD, bool kQK16>
__global__ void __launch_bounds__(kThreads, 1)
sla_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                    const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_kvw, AttnParams p) {
  using L = Lay<HD, kQK16>;
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, stays a shared-space pointer
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBars);
  uint16_t* s_lut = reinterpret_cast<uint16_t*>(smem + L::kOffLut);                 // [topk] key-block ids
  float* s_ksc = reinterpret_cast<float*>(smem + L::kOffLut + ((p.topk * 2 + 15) & ~15));  // [topk] k_scale of those blocks

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  const int bh = b * p.h + hh;
  const int T_blocks = p.topk;

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
    if (lane == 0) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
      tma_prefetch_desc(&tmap_kvw);
      mbar_expect_tx(&bars[kQFull], L::kQBytes + L::kWBytes);
      if constexpr (kQK16) {  // 16-bit Q rows from [B,L,H,D]: HD/64 chunks of 128 rows x 128 B
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(smem + L::kOffQ + c * (BLKQ * 128), &tmap_q, &bars[kQFull], c * 64, hh, m_blk * BLKQ, b);
      } else {
        tma_load_4d(smem + L::kOffQ, &tmap_q, &bars[kQFull], 0, m_blk * BLKQ, bh, 0);
      }
#pragma unroll
      for (int c = 0; c < HD / 64; ++c)  // KVW: d_k chunk c of the [d_out, d_k] matrix of this head
        tma_load_4d(smem + L::kOffW + c * (HD * 128), &tmap_kvw, &bars[kQFull], c * 64, 0, bh, 0);
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
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(sv + c * (BLKK * 128), &tmap_v, &bars[kVFull + st], c * 64, hh, blk * BLKK, b);
      }
    }
    return;
  }

  // =============================================================== consumer warpgroups
  const int wg = warp >> 2, w4 = warp & 3;
  const int r_lo = wg * 64 + w4 * 16 + (lane >> 2);   // rows r_lo and r_lo + 8 of the block (fragment layout, common.cuh)
  const int cq = 2 * (lane & 3);                       // column pair offset inside every 8-column slice
  const uint32_t sbase = smem_u32(smem);
  // INT8 path: scores are int32 dot products scaled by q_scale * k_scale; 16-bit path: fp32 scores.  Both in the log2 domain.
  const float qsc = (kQK16 ? 1.0f : __ldg(p.q_scale + int64_t(bh) * p.mblk + m_blk)) * p.sm_scale * kLog2e;

  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_used[2] = {-INFINITY, -INFINITY}, l_part[2] = {0.f, 0.f};  // l_part: this thread's columns of the row sum

  mbar_wait(&bars[kQFull], 0);
  for (int j = 0; j < T_blocks; ++j) {
    const int st = j % kStages;
    const uint32_t ph = (j / kStages) & 1;
    const int blk = s_lut[j];
    const float sc = qsc * s_ksc[j];
    const int valid = p.lk - blk * BLKK;                // < 64 only in the ragged last key block

    // ---- S = Q.K^T for this warpgroup's 64 rows
    float s[32];
    mbar_wait(&bars[kKFull + st], ph);
    const uint32_t sk = sbase + L::kOffK + st * L::kKBytes;
    if constexpr (kQK16) {
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < HD / 16; ++ks) {  // K = 16 elements per MMA: chunk ks/4, +32 bytes per step inside the chunk
        const uint64_t qd = make_desc_kmajor_sw128(sbase + L::kOffQ + (ks >> 2) * (BLKQ * 128) + wg * (64 * 128)) + uint64_t((ks & 3) * 2);
        const uint64_t kd = make_desc_kmajor_sw128(sk + (ks >> 2) * (BLKK * 128)) + uint64_t((ks & 3) * 2);
        wgmma_f16_ss<64, kBF16>(s, qd, kd, ks > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] *= sc;
    } else {
      uint32_t si[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) si[i] = 0u;
      // int8 rows are HD bytes: 128-byte swizzle for 128-wide heads, 64-byte swizzle for 64-wide heads
      const uint32_t qa = sbase + L::kOffQ + wg * (64 * HD);
      const uint64_t qdesc = HD == 128 ? make_desc_kmajor_sw128(qa) : make_desc_kmajor_sw64(qa);
      const uint64_t kdesc = HD == 128 ? make_desc_kmajor_sw128(sk) : make_desc_kmajor_sw64(sk);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < HD / 32; ++ks)
        wgmma_i8_ss<64>(si, qdesc + uint64_t(ks * 2), kdesc + uint64_t(ks * 2), ks > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(si);
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] = static_cast<float>(static_cast<int>(si[i])) * sc;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[kKEmpty + st]);

    // ---- ragged last key block: columns past lk do not exist
    if (valid < BLKK) {
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (8 * (i >> 2) + cq + (i & 1) >= valid) s[i] = -INFINITY;
    }
    // ---- row maxima and the lazy rescale of the O accumulator (per row: alpha == 1 exactly where the maximum is kept)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (((i >> 1) & 1) == h) mx = fmaxf(mx, s[i]);
      mx = quad_max(mx);
      if (j == 0) {
        m_used[h] = mx;
      } else if (mx > m_used[h] + kRescaleThreshold) {
        const float alpha = fast_exp2(m_used[h] - mx);
#pragma unroll
        for (int i = 0; i < HD / 2; ++i)
          if (((i >> 1) & 1) == h) o[i] *= alpha;
        l_part[h] *= alpha;
        m_used[h] = mx;
      }
    }
    // ---- P = exp2(s - m_used); the row sum is taken from the unrounded P, the tensor core gets P rounded to T
    uint32_t pa[BLKK / 16][4];
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int h = (i >> 1) & 1;
      const float p0 = fast_exp2(s[i] - m_used[h]), p1 = fast_exp2(s[i + 1] - m_used[h]);
      l_part[h] += p0 + p1;
      pa[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(p0, p1);
    }

    // ---- O += P.V  (V: [64 keys x HD] rows, MN-major operand; +16 keys = +2048 B per K step)
    mbar_wait(&bars[kVFull + st], ph);
    const uint64_t vdesc = make_desc_mnmajor_sw128(sbase + L::kOffV + st * L::kVBytes, BLKK * 128);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BLKK / 16; ++kk) wgmma_f16_rs<HD, kBF16, 1>(o, pa[kk], vdesc + uint64_t(kk * 128));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
#pragma unroll
    for (int kk = 0; kk < BLKK / 16; ++kk) reg_fence(pa[kk]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[kVEmpty + st]);
  }
  linear_branch_store<T, HD>(o, l_part, p, sbase + L::kOffW, int64_t(m_blk) * BLKQ + r_lo, cq, b, hh, bh);
}

// SpargeAttn's Hopper block geometry (SLA/core.py:191-193, 226-229 on sm90): BLKQ = 64 query rows, BLKK = 128 key rows.
// CTA = (64-row query block, head, batch); both consumer warpgroups work on the SAME 64 query rows and split the block's LUT
// entries (warpgroup g takes entries j = g mod 2, the producer streams all of them through one ring), each running its own
// online softmax on a 64 x 128 score tile (wgmma m64n128k32: 64 int32 / fp32 registers), so one warpgroup's softmax overlaps
// the other's MMAs.  After both loops warpgroup 1 hands its (m, l, O) to warpgroup 0 through the drained K/V ring; warpgroup 0
// merges the two states and runs the linear branch and the output once (linear_branch_store).
// The producer is a whole warpgroup (one warp issues the TMA loads) so that setmaxnreg can move registers to the consumers:
// O (64) + S (64) + P (32) fp32 registers per thread do not fit in the 168 a 384-thread CTA starts with.
constexpr int kHopperBlkQ = 64, kHopperBlkK = 128;
constexpr int kThreadsQ64 = 3 * 128;
constexpr uint32_t kProducerRegsQ64 = 40, kConsumerRegsQ64 = 232;   // 128 * 40 + 256 * 232 <= 65536

// Ring slot st serves entries st, st+3, st+6, ..., which alternate between the two warpgroups.  One full barrier per slot would
// let a warpgroup skip a phase (the other warpgroup's entry), and try_wait.parity cannot tell phase n from phase n-2, so the
// wait could pass while the skipped entry's load is still landing.  Each slot therefore has one full barrier per warpgroup:
// entry j completes phase j / 6 of barrier (j % 3, j % 2), and warpgroup j % 2 consumes that barrier's phases in order.  The
// empty barriers stay per slot: the producer waits on every phase in order, and the four warps of the entry's warpgroup
// arrive only after its load, i.e. after the previous phase completed.
enum BarQ64 { kQ64QFull = 0, kQ64KFull = 1 /*3 x 2*/, kQ64KEmpty = 7 /*3*/, kQ64VFull = 10 /*3 x 2*/, kQ64VEmpty = 16 /*3*/ };
__device__ __forceinline__ int q64_full(int base, int j) { return base + 2 * (j % kStages) + (j & 1); }

template <typename T, int HD>
__global__ void __launch_bounds__(kThreadsQ64, 1)
sla_attn_fwd_q64_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                        const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_kvw, AttnParams p) {
  constexpr int BQ = kHopperBlkQ, BK = kHopperBlkK;
  using L = Lay<HD, false, BQ, BK>;
  // exchange of warpgroup 1's state: HD/2 accumulator registers + m_used[2] + l_part[2] per thread, over the K and V rings
  static_assert((HD / 2 + 4) * 128 * 4 <= kStages * (L::kKBytes + L::kVBytes), "merge buffer does not fit in the ring");
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBars);
  uint16_t* s_lut = reinterpret_cast<uint16_t*>(smem + L::kOffLut);
  float* s_ksc = reinterpret_cast<float*>(smem + L::kOffLut + ((p.topk * 2 + 15) & ~15));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blk = blockIdx.x, hh = blockIdx.y, b = blockIdx.z;
  const int bh = b * p.h + hh;
  const int T_blocks = p.topk;

  static_assert((kQ64VEmpty + kStages) * 8 <= 256, "barriers exceed their shared-memory slot");
  if (threadIdx.x == 0) {
    mbar_init(&bars[kQ64QFull], 1);
    for (int i = 0; i < kStages; ++i) {  // each use of a ring slot is consumed by the four warps of one warpgroup
      for (int g = 0; g < 2; ++g) {
        mbar_init(&bars[kQ64KFull + 2 * i + g], 1);
        mbar_init(&bars[kQ64VFull + 2 * i + g], 1);
      }
      mbar_init(&bars[kQ64KEmpty + i], 4);
      mbar_init(&bars[kQ64VEmpty + i], 4);
    }
    mbar_fence_init();
  }
  {
    const int32_t* lut_row = p.lut + (int64_t(bh) * p.mblk + m_blk) * p.topk;
    const float* ksc_row = p.k_scale + int64_t(bh) * p.nblk;
    for (int i = threadIdx.x; i < T_blocks; i += kThreadsQ64) {
      const int blk = __ldg(lut_row + i);
      s_lut[i] = static_cast<uint16_t>(blk);
      s_ksc[i] = __ldg(ksc_row + blk);
    }
  }
  __syncthreads();

  if (warp >= kConsumerWarps) {
    // =============================================================== TMA producer
    reg_dealloc<kProducerRegsQ64>();
    if (warp == kConsumerWarps && lane == 0) {
      tma_prefetch_desc(&tmap_q);
      tma_prefetch_desc(&tmap_k);
      tma_prefetch_desc(&tmap_v);
      tma_prefetch_desc(&tmap_kvw);
      mbar_expect_tx(&bars[kQ64QFull], L::kQBytes + L::kWBytes);
      tma_load_4d(smem + L::kOffQ, &tmap_q, &bars[kQ64QFull], 0, m_blk * BQ, bh, 0);
#pragma unroll
      for (int c = 0; c < HD / 64; ++c)
        tma_load_4d(smem + L::kOffW + c * (HD * 128), &tmap_kvw, &bars[kQ64QFull], c * 64, 0, bh, 0);
      for (int j = 0; j < T_blocks; ++j) {
        const int st = j % kStages;
        const uint32_t ph = ((j / kStages) & 1) ^ 1;
        const int blk = s_lut[j];
        uint64_t* kfull = &bars[q64_full(kQ64KFull, j)];
        uint64_t* vfull = &bars[q64_full(kQ64VFull, j)];
        mbar_wait(&bars[kQ64KEmpty + st], ph);
        mbar_expect_tx(kfull, L::kKBytes);
        tma_load_4d(smem + L::kOffK + st * L::kKBytes, &tmap_k, kfull, 0, blk * BK, hh, b);
        mbar_wait(&bars[kQ64VEmpty + st], ph);
        mbar_expect_tx(vfull, L::kVBytes);
        uint8_t* sv = smem + L::kOffV + st * L::kVBytes;
#pragma unroll
        for (int c = 0; c < HD / 64; ++c)
          tma_load_4d(sv + c * (BK * 128), &tmap_v, vfull, c * 64, hh, blk * BK, b);
      }
    }
    return;
  }

  // =============================================================== consumer warpgroups (same 64 rows, alternate LUT entries)
  reg_alloc<kConsumerRegsQ64>();
  const int wg = warp >> 2, w4 = warp & 3;
  const int r_lo = w4 * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t sbase = smem_u32(smem);
  const float qsc = __ldg(p.q_scale + int64_t(bh) * p.mblk + m_blk) * p.sm_scale * kLog2e;
  const uint64_t qdesc = HD == 128 ? make_desc_kmajor_sw128(sbase + L::kOffQ) : make_desc_kmajor_sw64(sbase + L::kOffQ);

  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_used[2] = {-INFINITY, -INFINITY}, l_part[2] = {0.f, 0.f};  // a warpgroup without entries keeps m = -inf, l = 0

  mbar_wait(&bars[kQ64QFull], 0);
  for (int j = wg; j < T_blocks; j += 2) {
    const int st = j % kStages;
    const uint32_t ph = (j / (2 * kStages)) & 1;        // phase j / 6 of this warpgroup's full barriers of slot st
    const int blk = s_lut[j];
    const float sc = qsc * s_ksc[j];
    const int valid = p.lk - blk * BK;                  // < 128 only in the ragged last key block

    // ---- S = Q.K^T over this entry's 128 keys
    float s[64];
    {
      uint32_t si[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) si[i] = 0u;
      mbar_wait(&bars[q64_full(kQ64KFull, j)], ph);
      const uint32_t sk = sbase + L::kOffK + st * L::kKBytes;
      const uint64_t kdesc = HD == 128 ? make_desc_kmajor_sw128(sk) : make_desc_kmajor_sw64(sk);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < HD / 32; ++ks)
        wgmma_i8_ss<128>(si, qdesc + uint64_t(ks * 2), kdesc + uint64_t(ks * 2), ks > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(si);
#pragma unroll
      for (int i = 0; i < 64; ++i) s[i] = static_cast<float>(static_cast<int>(si[i])) * sc;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[kQ64KEmpty + st]);

    // ---- ragged last key block (fewer than 64 valid keys masks a whole half of the tile)
    if (valid < BK) {
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (8 * (i >> 2) + cq + (i & 1) >= valid) s[i] = -INFINITY;
    }
    // ---- row maxima and the lazy rescale, as in sla_attn_fwd_kernel
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (((i >> 1) & 1) == h) mx = fmaxf(mx, s[i]);
      mx = quad_max(mx);
      if (j == wg) {
        m_used[h] = mx;
      } else if (mx > m_used[h] + kRescaleThreshold) {
        const float alpha = fast_exp2(m_used[h] - mx);
#pragma unroll
        for (int i = 0; i < HD / 2; ++i)
          if (((i >> 1) & 1) == h) o[i] *= alpha;
        l_part[h] *= alpha;
        m_used[h] = mx;
      }
    }
    uint32_t pa[BK / 16][4];
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int h = (i >> 1) & 1;
      const float p0 = fast_exp2(s[i] - m_used[h]), p1 = fast_exp2(s[i + 1] - m_used[h]);
      l_part[h] += p0 + p1;
      pa[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(p0, p1);
    }

    // ---- O += P.V  (V: [128 keys x HD], HD/64 MN-major chunks of 128 x 128 B; +16 keys = +2048 B per K step)
    mbar_wait(&bars[q64_full(kQ64VFull, j)], ph);
    const uint64_t vdesc = make_desc_mnmajor_sw128(sbase + L::kOffV + st * L::kVBytes, BK * 128);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) wgmma_f16_rs<HD, kBF16, 1>(o, pa[kk], vdesc + uint64_t(kk * 128));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) reg_fence(pa[kk]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[kQ64VEmpty + st]);
  }

  // ---- merge: every ring slot has been consumed once both loops are done, so the ring holds warpgroup 1's state.  Thread t of
  //      warpgroup 0 and thread t of warpgroup 1 own the same fragment positions; the buffer is [value][thread], conflict-free.
  float* xchg = reinterpret_cast<float*>(smem + L::kOffK) + (threadIdx.x & 127);
  named_bar_sync(1, 256);
  if (wg == 1) {
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) xchg[i * 128] = o[i];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      xchg[(HD / 2 + h) * 128] = m_used[h];
      xchg[(HD / 2 + 2 + h) * 128] = l_part[h];
    }
  }
  named_bar_sync(1, 256);
  if (wg == 1) return;
  float a0[2], a1[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {  // warpgroup 0 always has entry 0, so its maximum is finite and exp2(-inf - m) = 0 drops an empty state
    const float m1 = xchg[(HD / 2 + h) * 128], l1 = xchg[(HD / 2 + 2 + h) * 128];
    const float mx = fmaxf(m_used[h], m1);
    a0[h] = fast_exp2(m_used[h] - mx);
    a1[h] = fast_exp2(m1 - mx);
    l_part[h] = fmaf(l_part[h], a0[h], l1 * a1[h]);
  }
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) {
    const int h = (i >> 1) & 1;
    o[i] = fmaf(o[i], a0[h], xchg[i * 128] * a1[h]);
  }
  linear_branch_store<T, HD>(o, l_part, p, sbase + L::kOffW, int64_t(m_blk) * BQ + r_lo, cq, b, hh, bh);
}

template <typename T, int HD, bool kQK16, int kBQ>
constexpr auto attn_kernel() {
  if constexpr (kBQ == kHopperBlkQ) return sla_attn_fwd_q64_kernel<T, HD>;
  else return sla_attn_fwd_kernel<T, HD, kQK16>;
}

// kQK16: 16-bit Q and K in [b, l, h, d]; otherwise INT8 Q [b*h, l, d] and INT8 K [b, h, lk, d] (or [b, lk, h, d] when k_seq_major).
// kBQ x kBK: the block geometry, 128 x 64 (sla_attn_fwd_kernel) or 64 x 128 (sla_attn_fwd_q64_kernel, INT8 head-major K only).
template <int HD, bool kQK16, int kBQ = BLKQ, int kBK = BLKK>
int launch(const void* q_op, const float* q_scale, const void* k_op, const float* k_scale, const void* v, const void* q, int dtype,
           const int32_t* lut, int64_t topk, const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
           int64_t l, int64_t lk, int64_t h, float sm_scale, int feature, bool k_seq_major, void* stream) {
  using L = Lay<HD, kQK16, kBQ, kBK>;
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
  CUtensorMap tq, tk, tv, tw;
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
  {
    const uint64_t dims[4] = {uint64_t(d), uint64_t(h), uint64_t(lk), uint64_t(b)};
    const uint64_t str[3] = {uint64_t(d * 2), uint64_t(h * d * 2), uint64_t(lk * h * d * 2)};
    const uint32_t box[4] = {64, 1, kBK, 1};
    if (int rc = make_tmap_4d(&tv, v, t16, 2, dims, str, box)) return rc;
  }
  {
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
  dim3 grid(static_cast<unsigned>(mblk), static_cast<unsigned>(h), static_cast<unsigned>(b));
  const int threads = kBQ == kHopperBlkQ ? kThreadsQ64 : kThreads;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define TDB_ATTN(T)                                                                                                   \
  do {                                                                                                                \
    const auto kern = attn_kernel<T, HD, kQK16, kBQ>();                                                               \
    if (int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)), \
                            "cudaFuncSetAttribute(sla_attn)"))                                                        \
      return rc;                                                                                                      \
    kern<<<grid, threads, smem, st>>>(tq, tk, tv, tw, p);                                                             \
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

extern "C" int tdb200_sla_attn_fwd(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                                   const void* v, const void* q, int dtype, const int32_t* lut, int64_t topk,
                                   const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
                                   int64_t l, int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream) {
  if (int rc = check_common(q_i8, k_i8, v, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (!q_scale || !k_scale) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: null pointer");
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: head dim %lld (this kernel implements d=128)", (long long)d);
  return launch<128, false>(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum, proj_b, out, b, l, lk, h, sm_scale, 0,
                            false, stream);
}

// the same kernel reading INT8 K in the [b, lk, h, d] layout (tdb200_sla_quant_k_seq; what sequence-parallel ranks all-gather)
extern "C" int tdb200_sla_attn_fwd_kseq(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                                        const void* v, const void* q, int dtype, const int32_t* lut, int64_t topk,
                                        const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
                                        int64_t l, int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream) {
  if (int rc = check_common(q_i8, k_i8, v, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (!q_scale || !k_scale) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: null pointer");
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: head dim %lld (this kernel implements d=128)", (long long)d);
  if (b != 1)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd_kseq: batch %lld (the gathered [lk_pad, h, d] key slab is one sequence)", (long long)b);
  return launch<128, false>(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum, proj_b, out, b, l, lk, h, sm_scale, 0,
                            true, stream);
}

// tdb200_sla_attn_fwd_kseq with the block geometry chosen by the caller: (128, 64) is tdb200_sla_attn_fwd_kseq itself, (64, 128)
// runs sla_attn_fwd_q64_kernel.  Its producer loads K at (0, blk*BK, head, b) over the dims (d, lk, h, b), so the sequence-major
// layout is only a different set of tensor-map strides.
extern "C" int tdb200_sla_attn_fwd_kseq_blocks(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                                               const void* v, const void* q, int dtype, const int32_t* lut, int64_t topk,
                                               const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
                                               int64_t l, int64_t lk, int64_t h, int64_t d, float sm_scale, int64_t blkq,
                                               int64_t blkk, void* stream) {
  const bool hopper = blkq == kHopperBlkQ && blkk == kHopperBlkK;
  if (!hopper && !(blkq == BLKQ && blkk == BLKK))
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd_kseq_blocks: block sizes (%lld, %lld) (BLKQ x BLKK = 128 x 64 or 64 x 128)",
                (long long)blkq, (long long)blkk);
  if (!hopper)
    return tdb200_sla_attn_fwd_kseq(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum, proj_b, out, b, l, lk, h, d,
                                    sm_scale, stream);
  if (int rc = check_common(q_i8, k_i8, v, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (!q_scale || !k_scale) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: null pointer");
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: head dim %lld (this kernel implements d=128)", (long long)d);
  if (b != 1)
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd_kseq: batch %lld (the gathered [lk_pad, h, d] key slab is one sequence)", (long long)b);
  return launch<128, false, kHopperBlkQ, kHopperBlkK>(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum, proj_b, out,
                                                      b, l, lk, h, sm_scale, 0, true, stream);
}

extern "C" int tdb200_sla_attn_fwd_qk16(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
                                        const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
                                        int64_t l, int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream) {
  if (int rc = check_common(q, k, v, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: head dim %lld (this kernel implements d=128)", (long long)d);
  return launch<128, true>(q, nullptr, k, nullptr, v, q, dtype, lut, topk, kvw, ksum, proj_b, out, b, l, lk, h, sm_scale, 0, false,
                           stream);
}

extern "C" int tdb200_sla_attn_fwd_v2(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                                      const void* v, const void* q, int dtype, const int32_t* lut, int64_t topk,
                                      const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
                                      int64_t l, int64_t lk, int64_t h, int64_t d, float sm_scale, int feature,
                                      void* stream) {
  if (int rc = check_common(q_i8, k_i8, v, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (!q_scale || !k_scale) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: null pointer");
  if (d != 64 && d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: head dim %lld (64 or 128, SLA/core.py:207)", (long long)d);
  if (feature < 0 || feature > 2) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: feature map tag %d", feature);
  if (d == 128)
    return launch<128, false>(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum, proj_b, out, b, l, lk, h, sm_scale,
                              feature, false, stream);
  return launch<64, false>(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum, proj_b, out, b, l, lk, h, sm_scale,
                           feature, false, stream);
}

// tdb200_sla_attn_fwd_v2 with the block geometry chosen by the caller: (blkq, blkk) = (128, 64) is tdb200_sla_attn_fwd_v2 itself,
// (64, 128) runs sla_attn_fwd_q64_kernel (mblk = ceil(l/64), nblk = ceil(lk/128)).
extern "C" int tdb200_sla_attn_fwd_blocks(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                                          const void* v, const void* q, int dtype, const int32_t* lut, int64_t topk,
                                          const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
                                          int64_t l, int64_t lk, int64_t h, int64_t d, float sm_scale, int feature,
                                          int64_t blkq, int64_t blkk, void* stream) {
  const bool hopper = blkq == kHopperBlkQ && blkk == kHopperBlkK;
  if (!hopper && !(blkq == BLKQ && blkk == BLKK))
    return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd_blocks: block sizes (%lld, %lld) (BLKQ x BLKK = 128 x 64 or 64 x 128)",
                (long long)blkq, (long long)blkk);
  if (!hopper)
    return tdb200_sla_attn_fwd_v2(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum, proj_b, out, b, l, lk, h, d,
                                  sm_scale, feature, stream);
  if (int rc = check_common(q_i8, k_i8, v, q, lut, kvw, ksum, proj_b, out, b, l, lk, h)) return rc;
  if (!q_scale || !k_scale) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: null pointer");
  if (d != 64 && d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_attn_fwd: head dim %lld (64 or 128, SLA/core.py:207)", (long long)d);
  if (feature < 0 || feature > 2) return fail(TDB200_ERR_INVALID_ARG, "sla_attn_fwd: feature map tag %d", feature);
  if (d == 128)
    return launch<128, false, kHopperBlkQ, kHopperBlkK>(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum, proj_b,
                                                        out, b, l, lk, h, sm_scale, feature, false, stream);
  return launch<64, false, kHopperBlkQ, kHopperBlkK>(q_i8, q_scale, k_i8, k_scale, v, q, dtype, lut, topk, kvw, ksum, proj_b, out,
                                                     b, l, lk, h, sm_scale, feature, false, stream);
}
