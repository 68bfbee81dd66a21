// a2. W8A8 GEMM with per-128-K-block rescale on wgmma (reference semantics: turbodiffusion/ops/gemm/kernel.hpp:391-427,
// utils.hpp:116-121, output cast kernel.hpp:471-477; bias add ops/core.py:410-411).
//
//   c[i,j] = T( fma-chain over kb of  float(int32 dot of K-block kb) * (a_s[i/128,kb]*b_s[j/128,kb]) )  [+ bias]
//
// Design (128x256 output tiles, 128-deep K-blocks; a tile is one 128-row block of the activation scale grid and two
// 128-column blocks ("halves") of the weight scale grid).  The kernel is persistent: min(tiles, SMs) CTAs, one per SM, and
// CTA b works through tiles b, b + grid, b + 2 grid, ... with tile id = m_tile * n_tiles + n_tile, so the CTAs running
// together share A rows and a few B tiles in L2.  Producer and consumers derive that sequence on their own (no scheduler,
// no atomics); barriers, the register split and the tensor-map prefetch are paid once per CTA.  A GEMM with fewer tiles
// than SMs is one tile per CTA.
//   warpgroup 2  TMA producer (one thread of warp 8; setmaxnreg gives its registers to the consumers, whose two fp32
//            accumulators and int32 staging accumulator do not fit in the 168 a 384-thread CTA starts with): A tile
//            [128 rows x 128 B] and B tile [256 rows x 128 B] per K-block, 128B-swizzled, 4-stage ring, mbarrier
//            complete_tx.  The wide tile does twice the MMA work of a 128x128 one for 1.5x the operand bytes pulled from
//            L2.  Ring slot and phase come from one K-block counter that runs on across tiles, so the next tile's first
//            loads are issued as soon as slots free up: during the consumers' last K-blocks and their epilogue.
//   warpgroups 0-1  MMA + dequant + epilogue; warpgroup g owns output rows [64g, 64g+64) of the tile.  Per K-block and
//            half: four wgmma.m64n128k32.s32.s8.s8 into one 64-register int32 staging accumulator, then the int -> float
//            conversion and the FFMA with that half's block scale into the half's 64 fp32 registers.  Both warpgroups
//            issue off the same full barrier; ordering them to alternate (ping-pong) was measured slower (DESIGN.md,
//            a2).  The accumulate flag is reset at every K-block because the reference rescales per K-block.  After the
//            last K-block, per half: round to T, (+bias), (GELU), store.  A half that lies entirely past n is not stored,
//            and in the block-scale variant not multiplied either.  Each warpgroup loops over the tiles on its own with
//            the same running K-block counter; only the quantised epilogue's amax exchange makes the two meet, so
//            otherwise one warpgroup's epilogue overlaps the other's MMAs once they drift apart.
//   The store: each consumer warpgroup writes its 64 rows of a half into its own 16 KB shared-memory buffer (after the
//            ring: 4 x 48 KB + 2 x 16 KB + barriers = 230,656 B of the 232,448 B opt-in), in the 128B-swizzled layout of
//            a TMA box, and one of its threads stores the boxes with cp.async.bulk.tensor: whole 128-byte lines instead
//            of 4,096 partial-sector STGs per tile, issued asynchronously, so the warpgroup goes on to its next tile's
//            MMAs while they drain.  The buffer is waited on (wait_group.read) only before it is written again.  The
//            output tensor maps clip rows >= m, columns >= n and a split output's parts, so the epilogue has no
//            per-element predicates.
// Integer accumulation is exact and the fp32 FMA chain runs in ascending kb order, so the result is bit-identical
// to the reference restatement (oracle.int8_linear) on the same int8 inputs.
#include "common.cuh"
#include "host_common.h"

namespace {

using namespace tdb;

constexpr int BM = 128, BN = 256, BK = 128;
constexpr int BH = 128;                              // one half of the tile: one weight-scale block, one MMA N
constexpr int kStages = 4;
constexpr int kConsumerWarps = 8;                    // warpgroups 0-1
constexpr int kThreads = kConsumerWarps * 32 + 128;  // + the TMA warpgroup
constexpr uint32_t kProducerRegs = 40, kConsumerRegs = 232;   // 128 * 40 + 256 * 232 <= 65536
constexpr uint32_t kATile = BM * BK;                 // 16 KB
constexpr uint32_t kBTile = BN * BK;                 // 32 KB: half h at +16 KB h
constexpr uint32_t kStageBytes = kATile + kBTile;
constexpr uint32_t kOutBox = 64 * 128;               // one 128B-swizzled TMA store box: 64 rows x 128 B
constexpr uint32_t kOutWg = 2 * kOutBox;             // a warpgroup's staging buffer: 64 rows x one half in 16 bits
constexpr size_t kSmemBytes =
    1024 + size_t(kStages) * kStageBytes + 2 * kOutWg + 256 /*barriers 64 B + amax exchange 128 B*/;   // 230,656 B
static_assert(kSmemBytes <= 232448, "over the sm_90 opt-in shared memory per block");

struct GemmParams {
  const float* a_s;
  const float* b_s;
  const void* bias;
  void* c;
  int64_t m, n, k;
  int k_blocks;
  int n_tiles;    // 256-column tiles per 128-row tile
  int tiles;      // ceil(m / 128) * n_tiles
  int act;        // 0 none, 1 GELU(tanh) applied to the T-rounded (acc [+ bias]) value, result rounded to T again
  int8_t* out_q;  // when non-NULL: emit quant_int8_block128(T output) instead of the T output itself
  float* out_s;   // [ceil(m/128), n/128]
  int n_part;     // 16-bit output: columns per output matrix; c is [n / n_part, m, n_part] (n_part == n: the plain [m, n])
};

// Two evaluations of gelu_tanh(x) = 0.5 x (1 + tanh(u)),  u = sqrt(2/pi) (x + 0.044715 x^3):
//  * quantised output (the FFN hot path): tanh.approx (one MUFU, ABSOLUTE error <= 2^-11 on tanh, i.e. <= 2.5e-4 |x| on
//    the result): far below the int8 step amax/128 the value is rounded to next; compared with the oracle's exact
//    GELU the codes differ by one on ~1 % of the elements (tests/test_gpu_quant_gemm.py);
//  * 16-bit output: x * sigmoid(2u) with ex2 + rcp (two MUFU, relative error ~2^-21 everywhere, including the negative
//    tail where 1 + tanh(u) cancels): within one ulp of torch's fp32 GELU after rounding to T.
__device__ __forceinline__ float gelu_tanh_approx(float x) {
  const float u = __fmul_rn(__fmaf_rn(__fmul_rn(x, x), 0.7978845608028654f * 0.044715f, 0.7978845608028654f), x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  const float hx = __fmul_rn(x, 0.5f);
  return __fmaf_rn(hx, t, hx);
}
__device__ __forceinline__ float gelu_precise(float x) {
  // -2u*log2(e) = x * (c1 + c3 x^2);  x * 1/(1 + 2^z);  z -> +inf gives x*0 = 0 (sign kept), z -> -inf gives x
  const float z = x * fmaf(-0.10294324f, x * x, -2.3022082f);
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + fast_exp2(z)));
  return x * r;
}

// kRowScale: the LTX-2 client's variant (TurboT2AV ltx_distillation/tilelang_w8a8.py:78-117): a_s [m] per activation row,
// b_s [n] per output channel, int32 accumulation over ALL of K in the wgmma accumulator and ONE epilogue per tile
// c = T(float(acc) * a_s[i] * b_s[j] + bias[j]).
template <typename T, bool kRowScale>
__global__ void __launch_bounds__(kThreads, 1)
gemm_w8a8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_c, GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, stays a shared-space pointer
  uint8_t* out_stage = smem + size_t(kStages) * kStageBytes;                      // [2 warpgroups][kOutWg]
  uint64_t* bars = reinterpret_cast<uint64_t*>(out_stage + 2 * kOutWg);
  uint64_t* full_bar = bars;                // [kStages]  TMA -> MMA
  uint64_t* empty_bar = bars + kStages;     // [kStages]  MMA -> TMA (one arrival per consumer warp)
  float* amax_x = reinterpret_cast<float*>(bars + 2 * kStages);  // [2][2][kConsumerWarps] block-amax exchange: tile parity, half

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kConsumerWarps);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= kConsumerWarps) {
    // ------------------------------------------------------------------ TMA producer
    reg_dealloc<kProducerRegs>();
    if (warp == kConsumerWarps && lane == 0) {
      tma_prefetch_desc(&tmap_a);
      tma_prefetch_desc(&tmap_b);
      uint32_t it = 0;   // K-blocks loaded so far, over all tiles; only it % (2 kStages) matters, so wrap-around is harmless
      for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        const int n_tile = tile % p.n_tiles, m_tile = tile / p.n_tiles;
        for (int kb = 0; kb < p.k_blocks; ++kb, ++it) {
          const uint32_t stage = it % kStages, phase = (it / kStages) & 1u;
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + size_t(stage) * kStageBytes;
          mbar_expect_tx(&full_bar[stage], kStageBytes);
          tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BK, m_tile * BM);
          tma_load_2d(sa + kATile, &tmap_b, &full_bar[stage], kb * BK, n_tile * BN);
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ MMA + dequant + epilogue warpgroups
  reg_alloc<kConsumerRegs>();
  const int wg = warp >> 2, w4 = warp & 3;
  const uint32_t sbase = smem_u32(smem);
  // `it` below counts this CTA's K-blocks over all its tiles, as the producer does: it names the ring slot and its phase.
  // The four K=32 steps of K-block `it` against half `h` of the B tile into `d` (onto its contents when `acc_in`); the
  // caller has waited on the stage's full barrier and commits the group
  auto issue = [&](uint32_t (&d)[64], uint32_t it, int h, bool acc_in) {
    const uint32_t sa = sbase + (it % kStages) * kStageBytes;
    const uint64_t adesc = make_desc_kmajor_sw128(sa + wg * (64 * 128));
    const uint64_t bdesc = make_desc_kmajor_sw128(sa + kATile + h * (BH * BK));
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < BK / 32; ++ks)  // +32 bytes (one K=32 int8 slice) inside the 128B swizzle row: +2 in 16-byte units
      wgmma_i8_ss<BH>(d, adesc + uint64_t(ks * 2), bdesc + uint64_t(ks * 2), (ks > 0 || acc_in) ? 1u : 0u);
  };
  auto wait_full = [&](uint32_t it) { mbar_wait(&full_bar[it % kStages], (it / kStages) & 1u); };
  auto release = [&](uint32_t it) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[it % kStages]);
  };

  // fragment coordinates (common.cuh): register i holds row r_lo + 8 ((i >> 1) & 1), column 8 (i >> 2) + cq + (i & 1)
  const int r_lo = wg * 64 + w4 * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const T* bias = static_cast<const T*>(p.bias);
  const bool act_gelu = p.act == 1;

  // Output staging.  Warpgroup wg's buffer holds its 64 rows of one half: two {64 columns x 64 rows} boxes of T, or for
  // the int8 output one {128 B x 64 rows} box per half, each in the 128B-swizzled layout of the TMA map: row r at 128 r,
  // its 16-byte chunk c at chunk c ^ (r & 7).  A warp's store of one register covers 8 rows x 16 bytes that land in 8
  // different chunks, so it is free of bank conflicts.  One thread per warpgroup issues the TMA stores; the bulk groups it
  // commits are its own, so it alone can wait for them, and the warpgroup's named barrier passes that on.
  uint8_t* const stage_wg = out_stage + wg * kOutWg;
  const bool issuer = (threadIdx.x & 127) == 0;
  const uint32_t wg_bar = 2 + wg;   // barrier 0 is __syncthreads, 1 the amax exchange of both warpgroups
  const int32_t row_wg = wg * 64;   // + m_tile * BM: the first output row of this warpgroup's boxes
  // byte offset of (row 8 h + the thread's fragment row, byte column bc < 128) inside a box
  auto box_off = [&](int h, int bc) -> uint32_t {
    return uint32_t(w4 * 16 + 8 * h + (lane >> 2)) * 128u + ((((bc >> 4) ^ (lane >> 2)) << 4) | (bc & 15));
  };
  if (issuer) tma_prefetch_desc(&tmap_c);
  // one half of 16-bit output, yw[2 j + h] = the T pair at fragment row h, columns 8 j + cq (+1), stored at column `col`
  // of output part `part`; the map clips rows >= m and columns >= n_part
  auto store16 = [&](const uint32_t (&yw)[BH / 4], int32_t col, int32_t row, int32_t part) {
    if (issuer) tma_store_wait_read<0>();   // the previous half's boxes have left the buffer
    named_bar_sync(wg_bar, 128);
#pragma unroll
    for (int j = 0; j < BH / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *reinterpret_cast<uint32_t*>(stage_wg + (j >> 3) * kOutBox + box_off(h, 16 * (j & 7) + 2 * cq)) = yw[2 * j + h];
    fence_proxy_async_smem();
    named_bar_sync(wg_bar, 128);
    if (issuer) {
      tma_store_4d(&tmap_c, stage_wg, col, row, part, 0);
      tma_store_4d(&tmap_c, stage_wg + kOutBox, col + 64, row, part, 0);
      tma_store_commit();
    }
  };

  uint32_t it0 = 0;       // the running K-block count at the start of the tile
  uint32_t parity = 0;    // of this CTA's tile count: selects the amax exchange slots
  for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x, it0 += p.k_blocks, parity ^= 1u) {
    const int n_tile = tile % p.n_tiles, m_tile = tile / p.n_tiles;
    const int64_t row0 = int64_t(m_tile) * BM + r_lo, row1 = row0 + 8;
    // the second half holds at least one column < n (CTA-uniform)
    const bool has_hi = int64_t(n_tile) * BN + BH < p.n;

    if constexpr (kRowScale) {
      uint32_t ia0[64], ia1[64];
      // K-block kb's MMAs chain onto kb-1's in flight (same accumulators, in order): wait only for kb-1 to free its slot,
      // so the tensor pipe does not drain at every K-block of a long K
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        wait_full(it0 + kb);
        issue(ia0, it0 + kb, 0, kb > 0);
        issue(ia1, it0 + kb, 1, kb > 0);   // unconditional: a wgmma under a branch costs an injected warpgroup.arrive per K-block
        wgmma_commit();
        if (kb > 0) {
          wgmma_wait<1>();
          release(it0 + kb - 1);
        }
      }
      wgmma_wait<0>();
      release(it0 + p.k_blocks - 1);   // the producer refills the last slot for the next tile during this epilogue
      reg_fence(ia0);
      reg_fence(ia1);
      // c = T(fma(float(acc) * a_s[row], b_s[col], bias[col])): the reference's TileLang epilogue compiles (nvcc default
      // -fmad) to I2FP, FMUL, FFMA per element (tools/tilelang_epilogue_probe.py)
      const float sa0 = row0 < p.m ? __ldg(p.a_s + row0) : 0.f, sa1 = row1 < p.m ? __ldg(p.a_s + row1) : 0.f;
      auto store = [&](const uint32_t (&ia)[64], int hf) {
        const int64_t col_base = int64_t(n_tile) * BN + hf * BH + cq;
        uint32_t yw[BH / 4];
#pragma unroll
        for (int j = 0; j < BH / 8; ++j) {
          const int64_t col = col_base + 8 * j;
          const bool in = col < p.n;   // columns >= n are clipped by the store
          const float sb0 = in ? __ldg(p.b_s + col) : 0.f, sb1 = in ? __ldg(p.b_s + col + 1) : 0.f;
          const uint32_t bw = bias != nullptr && in ? __ldg(reinterpret_cast<const unsigned int*>(bias + col)) : 0u;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float sa = h ? sa1 : sa0;
            const float y0 = __fmaf_rn(__fmul_rn(__int2float_rn(static_cast<int>(ia[4 * j + 2 * h])), sa), sb0, F16Traits<T>::lo(bw));
            const float y1 = __fmaf_rn(__fmul_rn(__int2float_rn(static_cast<int>(ia[4 * j + 2 * h + 1])), sa), sb1, F16Traits<T>::hi(bw));
            yw[2 * j + h] = F16Traits<T>::pack(y0, y1);
          }
        }
        store16(yw, n_tile * BN + hf * BH, m_tile * BM + row_wg, 0);
      };
      store(ia0, 0);
      if (has_hi) store(ia1, 1);
      continue;
    }

    // block scales: a_s [m/128, k_blocks] row m_tile, b_s [ceil(n/128), k_blocks] rows 2 n_tile (+1 only when has_hi)
    const float* as_row = p.a_s + int64_t(m_tile) * p.k_blocks;
    const float* bs_row0 = p.b_s + int64_t(2 * n_tile) * p.k_blocks;
    const float* bs_row1 = bs_row0 + p.k_blocks;
    float acc0[64], acc1[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc0[i] = acc1[i] = 0.0f;
    uint32_t ia[64];
    // float(s) is exact (a K-block sum is at most 128^3 = 2^21 in magnitude).  I2FP + FFMA is two instructions per value
    // against three for the magic-number conversion (IADD, FADD, FFMA), and measured faster on the H100 (DESIGN.md, a2).
    auto dequant = [&](float (&acc)[64], float scale) {
      wgmma_wait<0>();
      reg_fence(ia);
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = __fmaf_rn(__int2float_rn(static_cast<int>(ia[i])), scale, acc[i]);
    };
    for (int kb = 0; kb < p.k_blocks; ++kb) {
      wait_full(it0 + kb);
      const float as = __ldg(as_row + kb);
      issue(ia, it0 + kb, 0, false);
      wgmma_commit();
      dequant(acc0, as * __ldg(bs_row0 + kb));
      if (has_hi) {
        issue(ia, it0 + kb, 1, false);
        wgmma_commit();
        dequant(acc1, as * __ldg(bs_row1 + kb));
      }
      release(it0 + kb);
    }

    if (p.out_q != nullptr) {
      // ---- fused a1: each half is one 128x128 quant block (m_tile, 2 n_tile + hf).  y = the T-rounded value the plain
      //      epilogue would store (rows >= m count as 0); amax over the block; q = sat_s8(rint(y*128/amax)).
      auto store_q = [&](const float (&acc)[64], int hf) {
        const int64_t col_base = int64_t(n_tile) * BN + hf * BH + cq;
        uint32_t yw[32];
        uint32_t amax2 = 0u;
#pragma unroll
        for (int j = 0; j < BH / 8; ++j) {
          const int64_t col = col_base + 8 * j;
          const uint32_t bw = bias != nullptr ? *reinterpret_cast<const uint32_t*>(bias + col) : 0u;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t y = F16Traits<T>::pack(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);   // T(acc)
            if (bias != nullptr) y = F16Traits<T>::add2(y, bw);                            // T(T(acc) + bias)
            if (act_gelu) y = F16Traits<T>::pack(gelu_tanh_approx(F16Traits<T>::lo(y)), gelu_tanh_approx(F16Traits<T>::hi(y)));
            if ((h ? row1 : row0) >= p.m) y = 0u;
            yw[2 * j + h] = y;
            amax2 = F16Traits<T>::absmax2(amax2, y);
          }
        }
        float amax = fmaxf(1e-8f, fmaxf(F16Traits<T>::lo(amax2), F16Traits<T>::hi(amax2)));
        amax = warp_max(amax);
        // One slot set per (tile parity, half).  A set is rewritten two tiles later, and every warp passes the barrier of
        // the tile in between, after its reads here, before any warp can get there.  One set per half alone would not
        // do: a tile without a second half has a single barrier, so a warp still reading its slots could be overtaken
        // by the next tile's write to the same ones.  The parity bit costs 64 bytes and no extra barrier.
        float* xch = amax_x + (parity * 2 + hf) * kConsumerWarps;
        if (lane == 0) xch[warp] = amax;
        // Both halves' codes fit in the buffer (8 KB each), so only the first half waits, for the previous tile's boxes,
        // and the exchange barrier tells the warpgroup.
        if (issuer && hf == 0) tma_store_wait_read<0>();
        named_bar_sync(1, kConsumerWarps * 32);
#pragma unroll
        for (int w = 0; w < kConsumerWarps; ++w) amax = fmaxf(amax, xch[w]);
        const float r = __fdiv_rn(128.0f, amax);
        if (threadIdx.x == 0) p.out_s[int64_t(m_tile) * (p.n >> 7) + 2 * n_tile + hf] = amax * 0.0078125f;
        uint8_t* const box = stage_wg + hf * kOutBox;
#pragma unroll
        for (int j = 0; j < BH / 8; ++j) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t y = yw[2 * j + h];
            const int q0 = __float2int_rn(fminf(__fmul_rn(F16Traits<T>::lo(y), r), 127.0f));
            const int q1 = __float2int_rn(fminf(__fmul_rn(F16Traits<T>::hi(y), r), 127.0f));
            *reinterpret_cast<uint16_t*>(box + box_off(h, 8 * j + cq)) = static_cast<uint16_t>((q0 & 0xFF) | ((q1 & 0xFF) << 8));
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(wg_bar, 128);
        if (issuer) {   // rows >= m are clipped by the map
          tma_store_2d(&tmap_c, box, n_tile * BN + hf * BH, m_tile * BM + row_wg);
          tma_store_commit();
        }
      };
      store_q(acc0, 0);
      if (has_hi) store_q(acc1, 1);
      continue;
    }
    // a tile lies inside one output part (n_part is n itself or a multiple of 256): one division per tile, not per column
    const int part = n_tile * BN / p.n_part;
    auto store = [&](const float (&acc)[64], int hf) {
      const int64_t col_base = int64_t(n_tile) * BN + hf * BH + cq;
      // all of the half's bias words are loaded before any value is staged
      uint32_t bw[BH / 8];
#pragma unroll
      for (int j = 0; j < BH / 8; ++j) {
        const int64_t col = col_base + 8 * j;
        bw[j] = bias != nullptr && col < p.n ? __ldg(reinterpret_cast<const unsigned int*>(bias + col)) : 0u;
      }
      uint32_t yw[BH / 4];
#pragma unroll
      for (int j = 0; j < BH / 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // T(acc) then the packed 16-bit add: one rounding each, exactly the module's `out + bias` on 16-bit tensors
          uint32_t y = F16Traits<T>::pack(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          if (bias != nullptr) y = F16Traits<T>::add2(y, bw[j]);
          if (act_gelu) y = F16Traits<T>::pack(gelu_precise(F16Traits<T>::lo(y)), gelu_precise(F16Traits<T>::hi(y)));
          yw[2 * j + h] = y;
        }
      }
      store16(yw, n_tile * BN + hf * BH - part * p.n_part, m_tile * BM + row_wg, part);
    };
    store(acc0, 0);
    if (has_hi) store(acc1, 1);
  }
  if (issuer) tma_store_wait<0>();   // the staging buffers must outlive the stores that read them
}

template <typename T, bool kRowScale>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const GemmParams& p, cudaStream_t st) {
  auto kern = gemm_w8a8_kernel<T, kRowScale>;
  static bool attr_done[64] = {false};
  if (int rc = set_max_dynamic_smem_once(reinterpret_cast<const void*>(kern), kSmemBytes, attr_done,
                                         "cudaFuncSetAttribute(gemm_w8a8)"))
    return rc;
  kern<<<std::min(p.tiles, sm_count()), kThreads, kSmemBytes, st>>>(ta, tb, tc, p);
  return check_launch("gemm_w8a8_kernel");
}

}  // namespace

extern "C" int tdb200_gemm_w8a8(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s,
                                const void* bias, void* c, int c_dtype, int64_t m, int64_t n, int64_t k,
                                void* stream) {
  return tdb200_gemm_w8a8_ex(a_q, a_s, b_q, b_s, bias, c, c_dtype, m, n, k, TDB200_EPILOGUE_NONE, stream);
}

static int gemm_impl(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s, const void* bias, void* c,
                     int8_t* out_q, float* out_s, int c_dtype, int64_t m, int64_t n, int64_t k, int epilogue, void* stream,
                     bool row_scale = false, int64_t parts = 1);

extern "C" int tdb200_gemm_w8a8_ex(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s,
                                   const void* bias, void* c, int c_dtype, int64_t m, int64_t n, int64_t k,
                                   int epilogue, void* stream) {
  if (!c) return tdb::fail(TDB200_ERR_INVALID_ARG, "gemm_w8a8: null pointer");
  return gemm_impl(a_q, a_s, b_q, b_s, bias, c, nullptr, nullptr, c_dtype, m, n, k, epilogue, stream);
}

extern "C" int tdb200_gemm_w8a8_quant_out(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s,
                                          const void* bias, int8_t* out_q, float* out_s, int mid_dtype, int64_t m,
                                          int64_t n, int64_t k, int epilogue, void* stream) {
  if (!out_q || !out_s) return tdb::fail(TDB200_ERR_INVALID_ARG, "gemm_w8a8_quant_out: null pointer");
  if (n % 128 != 0) return tdb::fail(TDB200_ERR_UNSUPPORTED, "gemm_w8a8_quant_out: n=%lld must be a multiple of 128", (long long)n);
  return gemm_impl(a_q, a_s, b_q, b_s, bias, out_q, out_q, out_s, mid_dtype, m, n, k, epilogue, stream);
}

extern "C" int tdb200_gemm_w8a8_rowwise(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s,
                                        const void* bias, void* c, int c_dtype, int64_t m, int64_t n, int64_t k,
                                        void* stream) {
  if (!c) return tdb::fail(TDB200_ERR_INVALID_ARG, "gemm_w8a8_rowwise: null pointer");
  return gemm_impl(a_q, a_s, b_q, b_s, bias, c, nullptr, nullptr, c_dtype, m, n, k, TDB200_EPILOGUE_NONE, stream, true);
}

// one GEMM for several projections that share their input (q/k/v): b_q / b_s / bias are the row-wise concatenation of the
// projections' weights (n = parts * n_part, n_part a multiple of 256), the outputs are written as `parts` separate contiguous
// [m, n_part] matrices c[0..parts).  Block scales are per 128 weight rows, so each output equals its own GEMM bit for bit.
extern "C" int tdb200_gemm_w8a8_split(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s,
                                      const void* bias, void* c, int c_dtype, int64_t m, int64_t n, int64_t k,
                                      int64_t parts, void* stream) {
  if (!c) return tdb::fail(TDB200_ERR_INVALID_ARG, "gemm_w8a8_split: null pointer");
  return gemm_impl(a_q, a_s, b_q, b_s, bias, c, nullptr, nullptr, c_dtype, m, n, k, TDB200_EPILOGUE_NONE, stream, false, parts);
}

static int gemm_impl(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s, const void* bias, void* c,
                     int8_t* out_q, float* out_s, int c_dtype, int64_t m, int64_t n, int64_t k, int epilogue, void* stream,
                     bool row_scale, int64_t parts) {
  using namespace tdb;
  if (parts < 1 || n % parts != 0 || (parts > 1 && (n / parts) % 256 != 0))
    return fail(TDB200_ERR_UNSUPPORTED, "gemm_w8a8_split: n=%lld must split into %lld parts of a multiple of 256 columns",
                (long long)n, (long long)parts);
  if (epilogue != TDB200_EPILOGUE_NONE && epilogue != TDB200_EPILOGUE_GELU_TANH)
    return fail(TDB200_ERR_INVALID_ARG, "gemm_w8a8_ex: unknown epilogue %d", epilogue);
  if (!a_q || !a_s || !b_q || !b_s || !c) return fail(TDB200_ERR_INVALID_ARG, "gemm_w8a8: null pointer");
  if (m < 0 || n < 0 || k < 0) return fail(TDB200_ERR_INVALID_ARG, "gemm_w8a8: negative size");
  if (m == 0 || n == 0) return TDB200_OK;
  if (k == 0 || k % BK != 0)
    return fail(TDB200_ERR_UNSUPPORTED, "gemm_w8a8: k=%lld must be a positive multiple of 128 (gemm/launch.hpp:181-186)",
                (long long)k);
  if (n % 8 != 0) return fail(TDB200_ERR_UNSUPPORTED, "gemm_w8a8: n=%lld must be a multiple of 8", (long long)n);
  if (!aligned16(a_q) || !aligned16(b_q) || !aligned16(c) || (bias && !aligned16(bias)))
    return fail(TDB200_ERR_INVALID_ARG, "gemm_w8a8: a_q, b_q, c and bias must be 16-byte aligned");
  if (m > (int64_t(1) << 31) - 256 || n > (int64_t(1) << 31) - 256 || k > (int64_t(1) << 31) - 256)
    return fail(TDB200_ERR_UNSUPPORTED, "gemm_w8a8: dimension exceeds int32 TMA coordinates");
  if (int rc = require_sm90()) return rc;

  const int64_t m_tiles = cdiv64(m, BM), n_tiles = cdiv64(n, BN);
  if (m_tiles * n_tiles > (int64_t(1) << 30))   // int tile ids, with room for the grid stride past the last one
    return fail(TDB200_ERR_UNSUPPORTED, "gemm_w8a8: m=%lld x n=%lld exceeds 2^30 output tiles", (long long)m, (long long)n);
  if (c_dtype != TDB200_DTYPE_BF16 && c_dtype != TDB200_DTYPE_FP16)
    return fail(TDB200_ERR_UNSUPPORTED, "gemm_w8a8: output dtype tag %d (bf16/fp16 only, gemm.cu:41-65)", c_dtype);
  CUtensorMap ta, tb;
  if (int rc = make_tmap_2d(&ta, a_q, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, uint64_t(k), uint64_t(m), uint64_t(k), BK, BM))
    return rc;
  if (int rc = make_tmap_2d(&tb, b_q, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, uint64_t(k), uint64_t(n), uint64_t(k), BK, BN))
    return rc;
  // the output, stored from 64-row boxes: int8 codes [m, n] in 128-byte boxes, or the 16-bit c as (n_part, m, parts) in
  // 64-column boxes, so that a part's last rows and the columns past n are clipped rather than written into the next
  CUtensorMap tc;
  if (out_q) {
    if (int rc = make_tmap_2d(&tc, out_q, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, uint64_t(n), uint64_t(m), uint64_t(n), 128, 64))
      return rc;
  } else {
    const uint64_t np = uint64_t(n / parts);
    const uint64_t dims[4] = {np, uint64_t(m), uint64_t(parts), 1};
    const uint64_t strides[3] = {2 * np, 2 * np * uint64_t(m), 2 * uint64_t(n) * uint64_t(m)};
    const uint32_t box[4] = {64, 64, 1, 1};
    const CUtensorMapDataType t16 = c_dtype == TDB200_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    if (int rc = make_tmap_4d(&tc, c, t16, 2, dims, strides, box)) return rc;
  }

  GemmParams p;
  p.a_s = a_s;
  p.b_s = b_s;
  p.bias = bias;
  p.c = c;
  p.m = m;
  p.n = n;
  p.k = k;
  p.act = epilogue;
  p.out_q = out_q;
  p.out_s = out_s;
  p.n_part = static_cast<int>(n / parts);
  p.k_blocks = static_cast<int>(k / BK);
  p.n_tiles = static_cast<int>(n_tiles);
  p.tiles = static_cast<int>(m_tiles * n_tiles);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (row_scale) {
    if (k > 16384 * 8) return fail(TDB200_ERR_UNSUPPORTED, "gemm_w8a8_rowwise: k too large for int32 accumulation");
    if (c_dtype == TDB200_DTYPE_BF16) return launch<__nv_bfloat16, true>(ta, tb, tc, p, st);
    return launch<__half, true>(ta, tb, tc, p, st);
  }
  if (c_dtype == TDB200_DTYPE_BF16) return launch<__nv_bfloat16, false>(ta, tb, tc, p, st);
  return launch<__half, false>(ta, tb, tc, p, st);
}
