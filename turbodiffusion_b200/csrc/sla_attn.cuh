// Shared by the attention kernels (sla_attn.cu, sla_attn_bwd.cu, dense_attn.cu): the release of a ring slot, the per-tile steps
// of the forward kernels (scores, online softmax with the lazy rescale, register-A P.V, output rows), and the entry-split
// schedule of the 64-row-query-block kernels with the hand-off between their two consumer warpgroups.
//
// Entry split.  CTA = a producer warpgroup (one warp issues the TMA loads; setmaxnreg gives its registers to the consumers) and
// two consumer warpgroups on the same 64 query rows, which take alternate LUT entries: warpgroup g consumes entries j = g mod 2,
// while the producer streams every entry through one K ring and one V ring of kStages slots.
// Ring slot st serves entries st, st + 3, st + 6, ..., which alternate between the two warpgroups.  One full barrier per slot
// would let a warpgroup skip a phase (the other warpgroup's entry), and try_wait.parity cannot tell phase n from phase n - 2, so
// the wait could pass while the skipped entry's load is still landing.  Each slot therefore has one full barrier per warpgroup:
// entry j completes phase j / 6 of barrier (j % 3, j % 2), and warpgroup j % 2 consumes that barrier's phases in order.  The
// empty barriers stay per slot: the producer waits on every phase in order, and the four warps of the entry's warpgroup arrive
// only after its load, i.e. after the previous phase completed.
#pragma once
#include "common.cuh"

namespace tdb {

// the calling warp is done reading a ring slot: one arrival on the slot's empty barrier, after every lane's reads
__device__ __forceinline__ void warp_release(uint64_t* empty, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(empty);
}

// The keys batch entry b of a dense attention kernel attends to: lk, or (kKeyLens, the _kl entry points) k_lens[b] clamped to
// [0, lk].  Read once per CTA before its first barrier, so that the producer and the consumers derive the same tile count.
template <bool kKeyLens>
__device__ __forceinline__ int keys_of(const int32_t* k_lens, int lk, int b) {
  if constexpr (kKeyLens) return min(max(__ldg(k_lens + b), 0), lk);
  return lk;
}

// kKeyLens: key rows [valid, rows) of a streamed tile lie past the entry's keys but inside the buffer, so TMA loaded whatever
// memory holds there rather than zero fill.  Their score columns are masked, but an MMA multiplies the masked zeros by the
// rows themselves (P.V, the tangent's S_t = q_t.k^T + q.k_t^T, dP = dO.V^T, dS.K), and 0 * inf is NaN: so the consumers zero
// those rows, as TMA's zero fill would.  Whole 128-byte rows: the 128-byte swizzle permutes 16-byte units within a row.  A
// tile of `chunks` column chunks of rows x 128 B at `tile`; the 256 consumer threads share the work (tid = threadIdx.x).
// The caller then runs fence_proxy_async_smem() and a barrier over the consumers, before any MMA reads the tile.
__device__ __forceinline__ void zero_key_rows(uint8_t* tile, int rows, int chunks, int valid, int tid) {
  const int per_chunk = (rows - valid) * 8;   // 16-byte units
  for (int e = tid; e < chunks * per_chunk; e += 256) {
    const int c = e / per_chunk, u = e - c * per_chunk;
    *reinterpret_cast<uint4*>(tile + c * rows * 128 + valid * 128 + u * 16) = make_uint4(0u, 0u, 0u, 0u);
  }
}

// The query rows batch entry b of a dense attention kernel owns: lq, or (kQueryLens, the _vl entry points) q_lens[b] clamped
// to [0, lq].  Read once per CTA before its first barrier, as keys_of.
template <bool kQueryLens>
__device__ __forceinline__ int queries_of(const int32_t* q_lens, int lq, int b) {
  return keys_of<kQueryLens>(q_lens, lq, b);
}

// kQueryLens: query rows [lo, hi) of a streamed Q or dO tile (`chunks` column chunks of rows x 128 B at `tile`) lie past the
// entry's queries but inside the buffer.  Where one query row's values reach a sum over query rows (the dK / dV kernel's
// P^T.dO and dS^T.Q), 0 * inf would be NaN: so the warpgroup that reads those rows zeroes them, as TMA's zero fill would.
// The 128 threads of that warpgroup share the work (t = threadIdx.x & 127); whole 128-byte rows, as zero_key_rows.  The caller
// then runs fence_proxy_async_smem() and a barrier over the warpgroup, before any MMA reads the tile.
__device__ __forceinline__ void zero_query_rows(uint8_t* tile, int rows, int chunks, int lo, int hi, int t) {
  const int per_chunk = (hi - lo) * 8;   // 16-byte units
  for (int e = t; e < chunks * per_chunk; e += 128) {
    const int c = e / per_chunk, u = e - c * per_chunk;
    *reinterpret_cast<uint4*>(tile + c * rows * 128 + lo * 128 + u * 16) = make_uint4(0u, 0u, 0u, 0u);
  }
}

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kRescaleThreshold = 8.0f;  // log2 domain

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// ---- The per-entry steps of every forward kernel (sla_attn.cu, dense_attn.cu), on one warpgroup's 64 query rows.  Each thread
//      holds rows r and r + 8 of the tiles (fragment layout, common.cuh); cq is its column pair offset inside every 8-column slice.

// The raw score accumulator of S = Q.K^T: int32 dot products for INT8 Q/K, fp32 for 16-bit Q/K.
template <bool kQK16>
using ScoreAcc = std::conditional_t<kQK16, float, uint32_t>;

// Issue S = Q.K^T over the BK keys of one ring slot into acc, as one commit group.  INT8: Q and K rows of HD bytes with a
// 128-byte swizzle for 128-wide heads and a 64-byte one for 64-wide heads.  16-bit: Q and K in HD/64 chunks of 128-byte rows,
// q_chunk bytes apart for Q.  acc must not be touched until the group has retired and score_finish has fenced it.
template <bool kQK16, int HD, int BK, bool kBF16>
__device__ __forceinline__ void score_issue(ScoreAcc<kQK16> (&acc)[BK / 2], uint32_t sq, uint32_t q_chunk, uint32_t sk) {
#pragma unroll
  for (int i = 0; i < BK / 2; ++i) acc[i] = 0;
  if constexpr (kQK16) {
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {  // K = 16 elements per MMA: chunk ks/4, +32 bytes per step inside the chunk
      const uint64_t qd = make_desc_kmajor_sw128(sq + (ks >> 2) * q_chunk) + uint64_t((ks & 3) * 2);
      const uint64_t kd = make_desc_kmajor_sw128(sk + (ks >> 2) * (BK * 128)) + uint64_t((ks & 3) * 2);
      wgmma_f16_ss<BK, kBF16>(acc, qd, kd, ks > 0 ? 1u : 0u);
    }
  } else {
    const uint64_t qdesc = HD == 128 ? make_desc_kmajor_sw128(sq) : make_desc_kmajor_sw64(sq);
    const uint64_t kdesc = HD == 128 ? make_desc_kmajor_sw128(sk) : make_desc_kmajor_sw64(sk);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 32; ++ks)
      wgmma_i8_ss<BK>(acc, qdesc + uint64_t(ks * 2), kdesc + uint64_t(ks * 2), ks > 0 ? 1u : 0u);
  }
  wgmma_commit();
}

// Once score_issue's group has retired: s = acc scaled by sc into the log2 domain (INT8: sc folds in q_scale * k_scale).
template <bool kQK16, int BK>
__device__ __forceinline__ void score_finish(ScoreAcc<kQK16> (&acc)[BK / 2], float (&s)[BK / 2], float sc) {
  reg_fence(acc);
#pragma unroll
  for (int i = 0; i < BK / 2; ++i) {
    if constexpr (kQK16) s[i] = acc[i] * sc;
    else s[i] = static_cast<float>(static_cast<int>(acc[i])) * sc;
  }
}

// S = Q.K^T over the BK keys of one ring slot, scaled by sc into the log2 domain, with nothing else in flight.
template <bool kQK16, int HD, int BK, bool kBF16>
__device__ __forceinline__ void score_tile(float (&s)[BK / 2], uint32_t sq, uint32_t q_chunk, uint32_t sk, float sc) {
  if constexpr (kQK16) {   // the fp32 accumulator is s itself
    score_issue<kQK16, HD, BK, kBF16>(s, sq, q_chunk, sk);
    wgmma_wait<0>();
    score_finish<kQK16, BK>(s, s, sc);
  } else {
    uint32_t si[BK / 2];
    score_issue<kQK16, HD, BK, kBF16>(si, sq, q_chunk, sk);
    wgmma_wait<0>();
    score_finish<kQK16, BK>(si, s, sc);
  }
}

// The part of one online-softmax step that does not touch O: key columns from `valid` on do not exist (the ragged last key
// block), then the row maxima, the lazy rescale of the row sums (per row half h: rescale[h] where the maximum grew by more than
// the threshold, O to be scaled by alpha[h]; elsewhere the maximum is kept and O stays as it is), then P = exp2(s - m_used),
// left unrounded in s, and its row sums.  `first`: the first entry of this warpgroup, which sets the maxima.
template <int BK>
__device__ __forceinline__ void softmax_p(float (&s)[BK / 2], float (&m_used)[2], float (&l_part)[2], bool (&rescale)[2],
                                          float (&alpha)[2], int valid, int cq, bool first) {
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
    rescale[h] = false;
    alpha[h] = 1.0f;
    if (first) {
      m_used[h] = mx;
    } else if (mx > m_used[h] + kRescaleThreshold) {
      alpha[h] = fast_exp2(m_used[h] - mx);
      rescale[h] = true;
      l_part[h] *= alpha[h];
      m_used[h] = mx;
    }
  }
#pragma unroll
  for (int i = 0; i < BK / 2; i += 2) {
    const int h = (i >> 1) & 1;
    s[i] = fast_exp2(s[i] - m_used[h]);
    s[i + 1] = fast_exp2(s[i + 1] - m_used[h]);
    l_part[h] += s[i] + s[i + 1];
  }
}

// softmax_p for INT8 Q/K, straight from score_issue's int32 accumulator once its group has retired: p = P, unrounded, for the
// scores s = float(acc) * sc.  sc >= 0 and rounding is monotone, so the row maxima are taken on the integers (IMNMX) and
// float(max) * sc is the maximum softmax_p finds.  Each exponent argument keeps softmax_p's two roundings, s and then s - m,
// so every bit of P, l and O is softmax_p's (one FFMA instead is faster, but its last-bit changes do not stay last-bit
// after the INT8 quantisation of the next layer's input; DESIGN.md).  The ragged last key block masks the float argument to
// -inf as softmax_p does (an INT_MIN score times a small sc minus m would not underflow exp2).  kRagged: the block has columns
// from `valid` on.  Full blocks run their own instantiation without the per-column test: written as one path, ptxas
// predicates the test into every element of every block.
template <int BK, bool kRagged>
__device__ __forceinline__ void softmax_p_i8_cols(uint32_t (&acc)[BK / 2], float (&p)[BK / 2], float sc, float (&m_used)[2],
                                                  float (&l_part)[2], bool (&rescale)[2], float (&alpha)[2], int valid, int cq,
                                                  bool first) {
  auto dead = [&](int i) { return kRagged && 8 * (i >> 2) + cq + (i & 1) >= valid; };
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    int imx = INT_MIN;   // every row has a valid column in its quad
#pragma unroll
    for (int i = 0; i < BK / 2; ++i)
      if (((i >> 1) & 1) == h && !dead(i)) imx = max(imx, static_cast<int>(acc[i]));
    imx = max(imx, __shfl_xor_sync(0xffffffffu, imx, 1));
    imx = max(imx, __shfl_xor_sync(0xffffffffu, imx, 2));
    const float mx = static_cast<float>(imx) * sc;
    rescale[h] = false;
    alpha[h] = 1.0f;
    if (first) {
      m_used[h] = mx;
    } else if (mx > m_used[h] + kRescaleThreshold) {
      alpha[h] = fast_exp2(m_used[h] - mx);
      rescale[h] = true;
      l_part[h] *= alpha[h];
      m_used[h] = mx;
    }
  }
#pragma unroll
  for (int i = 0; i < BK / 2; i += 2) {
    const int h = (i >> 1) & 1;
    const float x0 = __fsub_rn(__fmul_rn(static_cast<float>(static_cast<int>(acc[i])), sc), m_used[h]);
    const float x1 = __fsub_rn(__fmul_rn(static_cast<float>(static_cast<int>(acc[i + 1])), sc), m_used[h]);
    p[i] = fast_exp2(dead(i) ? -INFINITY : x0);
    p[i + 1] = fast_exp2(dead(i + 1) ? -INFINITY : x1);
    l_part[h] += p[i] + p[i + 1];
  }
}
template <int BK>
__device__ __forceinline__ void softmax_p_i8(uint32_t (&acc)[BK / 2], float (&p)[BK / 2], float sc, float (&m_used)[2],
                                             float (&l_part)[2], bool (&rescale)[2], float (&alpha)[2], int valid, int cq,
                                             bool first) {
  reg_fence(acc);
  if (valid < BK) softmax_p_i8_cols<BK, true>(acc, p, sc, m_used, l_part, rescale, alpha, valid, cq, first);
  else softmax_p_i8_cols<BK, false>(acc, p, sc, m_used, l_part, rescale, alpha, valid, cq, first);
}

// The O part of the step: the lazy rescale softmax_p decided.  O must hold every earlier entry's P.V.
template <int HD>
__device__ __forceinline__ void rescale_o(float (&o)[HD / 2], const bool (&rescale)[2], const float (&alpha)[2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (rescale[h]) {
#pragma unroll
      for (int i = 0; i < HD / 2; ++i)
        if (((i >> 1) & 1) == h) o[i] *= alpha[h];
    }
  }
}

// P rounded to T into the A fragments of P.V (the row sums were taken from the unrounded P)
template <typename T, int BK>
__device__ __forceinline__ void pack_p(const float (&p)[BK / 2], uint32_t (&pa)[BK / 16][4]) {
#pragma unroll
  for (int i = 0; i < BK / 2; i += 2) pa[i >> 3][(i >> 1) & 3] = F16Traits<T>::pack(p[i], p[i + 1]);
}

// One online-softmax step, with no P.V in flight: softmax_p, the rescale of O, and P into the A fragments of P.V.
template <typename T, int HD, int BK>
__device__ __forceinline__ void softmax_step(float (&s)[BK / 2], float (&o)[HD / 2], float (&m_used)[2], float (&l_part)[2],
                                             uint32_t (&pa)[BK / 16][4], int valid, int cq, bool first) {
  bool rescale[2];
  float alpha[2];
  softmax_p<BK>(s, m_used, l_part, rescale, alpha, valid, cq, first);
  rescale_o<HD>(o, rescale, alpha);
  pack_p<T, BK>(s, pa);
}

// Issue O += P.V as one commit group (V: [BK keys x HD], HD/64 MN-major chunks of BK x 128 B, so no transposed copy of V;
// +16 keys = +2048 B per K step).  o and pa must not be touched until the group has retired and pv_fence has run.
template <int HD, int BK, bool kBF16>
__device__ __forceinline__ void pv_issue(float (&o)[HD / 2], uint32_t (&pa)[BK / 16][4], uint32_t sv) {
  const uint64_t vdesc = make_desc_mnmajor_sw128(sv, BK * 128);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < BK / 16; ++kk) wgmma_f16_rs<HD, kBF16, 1>(o, pa[kk], vdesc + uint64_t(kk * 128));
  wgmma_commit();
}
template <int HD, int BK>
__device__ __forceinline__ void pv_fence(float (&o)[HD / 2], uint32_t (&pa)[BK / 16][4]) {
  reg_fence(o);
#pragma unroll
  for (int kk = 0; kk < BK / 16; ++kk) reg_fence(pa[kk]);
}

// O += P.V, waited for
template <int HD, int BK, bool kBF16>
__device__ __forceinline__ void pv_step(float (&o)[HD / 2], uint32_t (&pa)[BK / 16][4], uint32_t sv) {
  pv_issue<HD, BK, kBF16>(o, pa, sv);
  wgmma_wait<0>();
  pv_fence<HD, BK>(o, pa);
}

// ---- P.V with e4m3 P and V (the SageSLA kernels' FP8 option, tdb200_sla_attn_fwd_fp8v).  V arrives as codes of V / v_scale
//      in tiles of [HD channels x BK keys], K-major (the only B layout e4m3 wgmma takes), rows of BK bytes in the 128-byte
//      (BK = 128) or 64-byte (BK = 64) swizzle.  The A fragment of one K = 32 step holds, per row, the 4-byte groups k 4 (l%4)
//      + {0..3} (a[0], a[1]: rows l/4, l/4 + 8) and 16 + 4 (l%4) + {0..3} (a[2], a[3]); the score accumulator holds keys
//      8 c + 2 (l%4) + {0, 1}.  tdb200_sla_quant_v_fp8 stores the keys of every 32-key group in the order that makes the two
//      agree (position 16 u + 4 t + j holds key 16 u + 8 (j >> 1) + 2 t + (j & 1)), so P packs into the fragment in registers
//      without any exchange between lanes.
// P is rounded to e4m3 times kF8PScale: p <= 2^8 under the lazy rescale, and 2^0 is the largest power of two that keeps
// 2^8 s <= 448 (e4m3's largest finite value); a larger one would saturate the p in (224, 256], a smaller one would only push
// more small p below e4m3's smallest normal, 2^-6.
constexpr float kF8PScale = 1.0f;

// The P.V step of one key block, for 16-bit P and V (kF8V = false: pack_p / pv_issue / pv_fence, straight into O) or e4m3 P
// and V.  issue starts the block's P.V, fence (once it has retired) leaves O holding it; Acc is the block's own accumulator.
template <typename T, int HD, int BK, bool kF8V>
struct PvOps {
  static constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  static constexpr int kSteps = BK / 16;   // A fragments: one per K = 16 step
  using Frag = uint32_t[kSteps][4];
  struct Acc {};
  static __device__ __forceinline__ void pack(const float (&p)[BK / 2], Frag& pa) { pack_p<T, BK>(p, pa); }
  static __device__ __forceinline__ void issue(float (&o)[HD / 2], Acc&, Frag& pa, uint32_t sv) { pv_issue<HD, BK, kBF16>(o, pa, sv); }
  static __device__ __forceinline__ void fence(float (&o)[HD / 2], Acc&, Frag& pa) { pv_fence<HD, BK>(o, pa); }
  static __device__ __forceinline__ void step(float (&o)[HD / 2], Acc&, Frag& pa, uint32_t sv) { pv_step<HD, BK, kBF16>(o, pa, sv); }
};
template <typename T, int HD, int BK>
struct PvOps<T, HD, BK, true> {
  static_assert(HD == 128 && (BK == 64 || BK == 128), "e4m3 P.V: 128 channels, 64- or 128-key blocks");
  static constexpr int kSteps = BK / 32;   // one per K = 32 step
  using Frag = uint32_t[kSteps][4];
  // The e4m3 wgmma accumulates at less than fp32 precision, so over a whole key list O would lose the small terms of every
  // block (the rel-L2 error grew with the list: 5-12 % against float64 at 50-120 blocks).  Each block's P.V therefore
  // starts a fresh accumulator of BK / 32 MMAs, added to O in fp32 once it has retired (SageAttention2's two-level
  // accumulation).
  using Acc = float[HD / 2];
  static __device__ __forceinline__ void pack(const float (&p)[BK / 2], Frag& pa) {
#pragma unroll
    for (int kk = 0; kk < kSteps; ++kk)
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = 4 * (4 * kk + 2 * u) + 2 * h;   // accumulator slices 4 kk + 2 u and + 1, row half h
          pa[kk][2 * u + h] = pack4_e4m3(p[i] * kF8PScale, p[i + 1] * kF8PScale, p[i + 4] * kF8PScale, p[i + 5] * kF8PScale);
        }
  }
  static __device__ __forceinline__ void issue(float (&)[HD / 2], Acc& acc, Frag& pa, uint32_t sv) {
    const uint64_t vdesc = BK == 128 ? make_desc_kmajor_sw128(sv) : make_desc_kmajor_sw64(sv);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kSteps; ++kk)   // +32 bytes per K step; the first one overwrites acc
      wgmma_e4m3_rs<HD>(acc, pa[kk], vdesc + uint64_t(kk * 2), kk > 0 ? 1u : 0u);
    wgmma_commit();
  }
  static __device__ __forceinline__ void fence(float (&o)[HD / 2], Acc& acc, Frag& pa) {
    reg_fence(acc);
#pragma unroll
    for (int kk = 0; kk < kSteps; ++kk) reg_fence(pa[kk]);
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] += acc[i];
  }
  static __device__ __forceinline__ void step(float (&o)[HD / 2], Acc& acc, Frag& pa, uint32_t sv) {
    issue(o, acc, pa, sv);
    wgmma_wait<0>();
    fence(o, acc, pa);
  }
};

// After the last e4m3 P.V: O = sum e4m3(p kF8PScale) e4m3(v / v_scale) back in the units of P.V, column by column
// (v_scale: this head's [HD] channel scales).
template <int HD>
__device__ __forceinline__ void unscale_o_f8v(float (&o)[HD / 2], const float* v_scale, int cq) {
#pragma unroll
  for (int c = 0; c < HD / 8; ++c) {
    const float2 s = __ldg(reinterpret_cast<const float2*>(v_scale + 8 * c + cq));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      o[4 * c + 2 * h] *= s.x * (1.0f / kF8PScale);
      o[4 * c + 2 * h + 1] *= s.y * (1.0f / kF8PScale);
    }
  }
}

// columns 8 c + cq + {0, 1} of one output row = T(O / l), from row half h (rows r and r + 8) of this thread's O fragment
template <typename T, int HD>
__device__ __forceinline__ void store_o_row(T* orow, const float (&o)[HD / 2], int h, float inv_l, int cq) {
#pragma unroll
  for (int c = 0; c < HD / 8; ++c)
    *reinterpret_cast<uint32_t*>(orow + 8 * c + cq) = F16Traits<T>::pack(o[4 * c + 2 * h] * inv_l, o[4 * c + 2 * h + 1] * inv_l);
}

// Row h (0: r_lo, 1: r_lo + 8) of this thread's m64 accumulator fragment set to zero: a query row past its entry's queries
// (kQueryLens) stores zeros whatever its q held, where scaling by zero would keep inf or NaN
template <int N>
__device__ __forceinline__ void zero_o_row(float (&o)[N], int h) {
#pragma unroll
  for (int c = 0; c < N / 4; ++c) o[4 * c + 2 * h] = o[4 * c + 2 * h + 1] = 0.f;
}

namespace split {
constexpr int kThreads = 3 * 128;
constexpr uint32_t kProducerRegs = 40, kConsumerRegs = 232;   // 128 * 40 + 256 * 232 <= 65536
constexpr int kStages = 3;
// the resident tiles' barrier, then per ring the full barriers [slot][warpgroup] and the empty barriers [slot]
enum Bar { kQFull = 0, kKFull = 1 /*3 x 2*/, kKEmpty = 7 /*3*/, kVFull = 10 /*3 x 2*/, kVEmpty = 16 /*3*/, kNumBars = 19 };

// the full barrier of entry j in the ring whose full barriers start at `base`, and the phase the consumer waits for
__device__ __forceinline__ int full(int base, int j) { return base + 2 * (j % kStages) + (j & 1); }
__device__ __forceinline__ uint32_t full_phase(int j) { return (j / (2 * kStages)) & 1; }

__device__ __forceinline__ void init_barriers(uint64_t* bars) {
  mbar_init(&bars[kQFull], 1);
  for (int i = 0; i < kStages; ++i) {  // each use of a ring slot is consumed by the four warps of one warpgroup
    for (int g = 0; g < 2; ++g) {
      mbar_init(&bars[kKFull + 2 * i + g], 1);
      mbar_init(&bars[kVFull + 2 * i + g], 1);
    }
    mbar_init(&bars[kKEmpty + i], 4);
    mbar_init(&bars[kVEmpty + i], 4);
  }
  mbar_fence_init();
}
}  // namespace split

// Hand-off from consumer warpgroup 1 to consumer warpgroup 0 once both have drained the ring, so that `ring` (shared memory the
// ring's tiles occupied) is free.  Thread t of warpgroup 1 stores value v at x[v], which is float v * 128 + t: thread t of
// warpgroup 0 holds the same fragment positions, and the [value][thread] layout is conflict-free.  `put` runs on warpgroup 1
// only; after the call warpgroup 1 is done and warpgroup 0 reads x[v].  `bar` is a named barrier the kernel uses for nothing else.
struct Handoff {
  float* base;
  __device__ __forceinline__ float& operator[](int v) const { return base[v * 128]; }
};
template <typename Put>
__device__ __forceinline__ Handoff handoff_wg1_to_wg0(uint8_t* ring, int wg, uint32_t bar, Put&& put) {
  const Handoff x{reinterpret_cast<float*>(ring) + (threadIdx.x & 127)};
  named_bar_sync(bar, 256);
  if (wg == 1) put(x);
  named_bar_sync(bar, 256);
  return x;
}

}  // namespace tdb
