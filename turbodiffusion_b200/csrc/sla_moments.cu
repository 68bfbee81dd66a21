// a10 (first half). Linear-attention moments of the keys (reference: turbodiffusion/SLA/core.py:243-247):
//   phi = softmax over the head dim (rounded to the 16-bit type),
//   kv[b,h,dv,dk] += sum_l v[l,dv] * phi(k)[l,dk]        (stored transposed: rows = value channel, cols = key channel)
//   ksum[b,h,dk]  += sum_l phi(k)[l,dk]
// Both outputs are ACCUMULATED in fp32 (caller zeroes them): every element receives exactly one plain add of this call's
// total, so sequence shards combine by plain addition (and one all-reduce across GPUs), and two launches into the same
// buffer give exactly fp32(t + t).
//
// Reproducibility: the bits of kv and ksum of one (b, h) depend only on that head's k, v, l, d, feature map and dtype.
// They do not depend on the run, the GPU's SM count, the number of heads or batch entries in the call, or other work on
// the device.  There are no floating-point atomics.  The tiles ceil(l/128) are split over S = min(tiles, kMaxSplits) CTAs
// (split s owns tiles s, s+S, s+2S, ...), a function of the tile count alone.  Those S CTAs form one thread-block cluster
// along grid.y.  After the last tile each CTA stages its fp32 partial kv (and its two ksum row halves, folded lower half
// first) in its own shared memory, in the V ring that is free by then.  After a cluster barrier, CTA r reduces its slice
// of the elements over distributed shared memory in split order 0, 1, ..., S-1 and adds the total to global memory, so
// each element has one writer and one summation order.
//
// CTA = 2 warpgroups, 128 key rows per tile.  Two threads per key row (each owns 64 of its 128 channels): load the row,
// feature map (softmax over D with MUFU ex2), write phi(k) into shared memory in the MN-major 128B-swizzled operand layout;
// thread 0 streams the V tiles in by TMA (3-stage ring).  Warpgroup g then issues wgmma (16-bit inputs, fp32 accumulator in
// registers across all tiles of this CTA): D[64 (dv rows 64g..) x 128 (dk)] += V^T . phi(K), both operands MN-major, and
// column-sums the tile for ksum while the MMAs run.
// 64-wide heads (SLA/core.py:207) run through the same 128-row tile as PAIRS of adjacent heads: in the [L, H, 64] layout two
// heads are 128 contiguous columns, i.e. exactly one 128-wide row of V and of K.  Warpgroup g computes only the diagonal
// 64x64 block of head 2*pair+g (N = 64), and phi is evaluated per 64-wide half.
// Feature maps (SLA/core.py:57-73): 0 softmax over the head dim, 1 elu(x)+1, 2 relu(x).
#include <type_traits>

#include "common.cuh"
#include "host_common.h"

namespace {
using namespace tdb;

constexpr int D = 128;
constexpr int kRowsPerTile = 128;
constexpr int kThreads = 256;
constexpr int kVStages = 3;
constexpr uint32_t kOperandBytes = kRowsPerTile * D * 2;  // 32 KB: two 64-channel blocks of 128 rows x 128 B
constexpr uint32_t kBlockBytes = kOperandBytes / 2;       // 16 KB
constexpr uint32_t kOffV = 0;                             // kVStages stages
constexpr uint32_t kOffPhi = kVStages * kOperandBytes;
constexpr uint32_t kOffBars = kOffPhi + kOperandBytes;    // 128 KB
constexpr size_t kSmemBytes = 1024 + kOffBars + 128;
constexpr float kLog2e = 1.4426950408889634f;
// Split CTAs per (head or head pair, b): the cluster size, at most 8 (portable).  12 heads x 8 = 96 CTAs fill one wave
// on an H100 (two 8-CTA clusters per GPC).
constexpr int kMaxSplits = 8;
// Partials staged after the last tile, in the V ring: kv [D*D] fp32 (a pair uses the first 2*64*64), then ksum [2][128]
constexpr uint32_t kOffPartKsum = D * D * 4;
static_assert(kOffPartKsum + 2 * 128 * 4 <= kOffPhi - kOffV, "the staged partials must fit in the V ring");

struct MomParams {
  const void* k;
  float* kv;
  float* ksum;
  int l, h, tiles, splits;
  int hd;        // 128, or 64 (two heads per 128-wide row; `h` is then the number of REAL heads, grid.x = ceil(h/2) pairs)
  int feature;   // 0 softmax, 1 elu+1, 2 relu
  const int32_t* seq_lens;   // [b] int32 (kVL only)
};

// kVL (tdb200_sla_linear_moments_vl): batch entry b has n = seq_lens[b] rows (clamped to [0, l]; l stays the row stride), so
// ceil(n / 128) tiles over S_b = min(tiles, kMaxSplits) splits: the tiles, splits and summation order of a call on the entry
// alone.  The launch's cluster is sized for l; its CTAs past S_b load nothing, and the reduction sums splits 0 .. S_b - 1 only.
// V rows past n in the straddling tile are zeroed in shared memory before the MMAs read them (TMA loads the padding there,
// where a call on the entry alone gets zero fill, and 0 * NaN is NaN).
template <typename T, bool kPair, bool kVL = false>
__global__ void __launch_bounds__(kThreads, 1)
sla_moments_kernel(const __grid_constant__ CUtensorMap tmap_v, MomParams p) {
  constexpr int N = kPair ? 64 : 128;          // key channels of this warpgroup's accumulator
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // 1024-aligned, stays a shared-space pointer
  uint64_t* vfull = reinterpret_cast<uint64_t*>(smem + kOffBars);                 // [kVStages]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int hh = blockIdx.x, split = blockIdx.y, b = blockIdx.z;  // heads (or head pairs) fastest: DRAM page locality of [L, H, D]
  const int head0 = kPair ? 2 * hh : hh;                           // first real head of this CTA
  const bool second_ok = !kPair || head0 + 1 < p.h;                // odd head count: the last pair has one real head
  const int64_t row_elems = int64_t(p.h) * p.hd;                   // elements per token row of k / v
  const int n = kVL ? min(max(__ldg(p.seq_lens + b), 0), p.l) : p.l;   // rows of this entry
  const int tiles = kVL ? (n + kRowsPerTile - 1) / kRowsPerTile : p.tiles;
  const int splits = kVL ? min(tiles, kMaxSplits) : p.splits;
  // tiles split, split+splits, ...; >= 1 (splits <= tiles), or with kVL 0 on the CTAs past the entry's splits
  const int my_tiles = kVL ? (split < splits ? (tiles - split + splits - 1) / splits : 0) : (p.tiles - split + p.splits - 1) / p.splits;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kVStages; ++i) mbar_init(&vfull[i], 1);
    mbar_fence_init();
  }
  __syncthreads();
  auto load_v = [&](int i) {   // thread 0: V tile i -> stage i % kVStages
    const int st = i % kVStages, tile = split + i * splits;
    uint8_t* sv = smem + kOffV + st * kOperandBytes;
    mbar_expect_tx(&vfull[st], kOperandBytes);
    // 128-wide head: columns [0,64) and [64,128) of head hh; 64-wide heads: heads 2hh and 2hh+1 (a missing second
    // head is out of range in the head dimension, which TMA fills with zeros)
    tma_load_4d(sv, &tmap_v, &vfull[st], 0, head0, tile * kRowsPerTile, b);
    tma_load_4d(sv + kBlockBytes, &tmap_v, &vfull[st], kPair ? 0 : 64, kPair ? head0 + 1 : head0, tile * kRowsPerTile, b);
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_v);
    for (int i = 0; i < kVStages - 1 && i < my_tiles; ++i) load_v(i);
  }

  const int r = threadIdx.x >> 1, half = threadIdx.x & 1;   // key row inside the tile, which 64 of its 128 channels
  const int wg = warp >> 2;
  const uint32_t sbase = smem_u32(smem);
  uint8_t* const sphi = smem + kOffPhi;
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  float ksum_acc = 0.f;
  // The key rows of tile i+1 are requested before tile i is transformed (eight independent 16-byte loads per thread in
  // flight under the exponentials), and phi needs ONE exponential per element: e_j is kept in fp32 registers until the
  // row sum is known.
  auto load_row = [&](int i, uint4 (&dst)[8]) {
    const int64_t row = int64_t(split + i * splits) * kRowsPerTile + r;
    const bool ok = i < my_tiles && row < n && (half == 0 || second_ok);   // missing second head: zeros
    const uint4* src = reinterpret_cast<const uint4*>(static_cast<const T*>(p.k) + (int64_t(b) * p.l + (ok ? row : 0)) * row_elems +
                                                      int64_t(head0) * p.hd + half * 64);
#pragma unroll
    for (int c = 0; c < 8; ++c) dst[c] = ok ? ldg_nc_v4(src + c) : make_uint4(0u, 0u, 0u, 0u);
  };
  uint4 cur[8];
  load_row(0, cur);
  for (int i = 0; i < my_tiles; ++i) {
    const int tile = split + i * splits;
    const int64_t row = int64_t(tile) * kRowsPerTile + r;
    uint4 nxt[8];
    load_row(i + 1, nxt);
    uint32_t w[32];
#pragma unroll
    for (int c = 0; c < 8; ++c) { w[4 * c] = cur[c].x; w[4 * c + 1] = cur[c].y; w[4 * c + 2] = cur[c].z; w[4 * c + 3] = cur[c].w; }
    const bool live = row < n && (half == 0 || second_ok);
    if (p.feature == 0) {
      // softmax over the head: my 64 channels, combined with the partner thread's for a 128-wide head
      float m = -INFINITY;
#pragma unroll
      for (int q = 0; q < 32; ++q) m = fmaxf(m, fmaxf(F16Traits<T>::lo(w[q]), F16Traits<T>::hi(w[q])));
      if (!kPair) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
      const float off = m * kLog2e;
      float e[64];
      float sa = 0.f, sb = 0.f;
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        e[2 * q] = fast_exp2(fmaf(F16Traits<T>::lo(w[q]), kLog2e, -off));
        e[2 * q + 1] = fast_exp2(fmaf(F16Traits<T>::hi(w[q]), kLog2e, -off));
        sa += e[2 * q];
        sb += e[2 * q + 1];
      }
      float sum = sa + sb;
      if (!kPair) sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      const float inv = 1.0f / sum;
#pragma unroll
      for (int q = 0; q < 32; ++q) w[q] = F16Traits<T>::pack(e[2 * q] * inv, e[2 * q + 1] * inv);
    } else {
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        const float a = F16Traits<T>::lo(w[q]), c = F16Traits<T>::hi(w[q]);
        const float fa = p.feature == 1 ? (a > 0.f ? a + 1.0f : fast_exp2(a * kLog2e)) : fmaxf(a, 0.f);
        const float fc = p.feature == 1 ? (c > 0.f ? c + 1.0f : fast_exp2(c * kLog2e)) : fmaxf(c, 0.f);
        w[q] = F16Traits<T>::pack(fa, fc);
      }
    }
    if (!live) {
#pragma unroll
      for (int q = 0; q < 32; ++q) w[q] = 0u;
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) cur[c] = nxt[c];
    // every warpgroup's MMAs of tile i-1 have retired (they read the phi buffer and V stage (i-1) % kVStages)
    wgmma_wait<0>();
    __syncthreads();
    if (threadIdx.x == 0 && i + kVStages - 1 < my_tiles) load_v(i + kVStages - 1);
#pragma unroll
    for (int c = 0; c < 8; ++c)
      *reinterpret_cast<uint4*>(sphi + half * kBlockBytes + r * 128 + ((c ^ (r & 7)) << 4)) =
          make_uint4(w[4 * c], w[4 * c + 1], w[4 * c + 2], w[4 * c + 3]);
    fence_proxy_async_smem();
    __syncthreads();   // all 128 rows of phi are written (also orders the ksum reads below)
    {
      const int st = i % kVStages;
      mbar_wait(&vfull[st], (i / kVStages) & 1);
      if constexpr (kVL)
        if ((tile + 1) * kRowsPerTile > n) {   // whole 128-byte rows of both 64-channel blocks (the swizzle stays in a row)
          const int valid = n - tile * kRowsPerTile, per_block = (kRowsPerTile - valid) * 8;
          uint8_t* sv = smem + kOffV + st * kOperandBytes;
          for (int e = threadIdx.x; e < 2 * per_block; e += kThreads) {
            const int c = e / per_block, u = e - c * per_block;
            *reinterpret_cast<uint4*>(sv + c * kBlockBytes + valid * 128 + u * 16) = make_uint4(0u, 0u, 0u, 0u);
          }
          fence_proxy_async_smem();
          __syncthreads();
        }
      // A = V^T (dv rows of block wg), B = phi (key channels; a pair's warpgroup takes its own 64-channel block): both MN-major,
      // K = 16 key rows per MMA: +2048 B in both operands
      const uint64_t adesc = make_desc_mnmajor_sw128(sbase + kOffV + st * kOperandBytes + wg * kBlockBytes, kBlockBytes);
      const uint64_t bdesc = make_desc_mnmajor_sw128(sbase + kOffPhi + (kPair ? wg * kBlockBytes : 0), kBlockBytes);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < kRowsPerTile / 16; ++ks)
        wgmma_f16_ss_mn<N, kBF16>(acc, adesc + uint64_t(ks * 128), bdesc + uint64_t(ks * 128), 1u);
      wgmma_commit();
    }
    // ---- ksum: thread t sums key channel t % 128 over half of the 128 rows of the tile
    {
      const int col = threadIdx.x & 127, r0 = (threadIdx.x >> 7) * 64;
      const uint8_t* colbase = sphi + (col >> 6) * kBlockBytes + (col & 7) * 2;
      const int chunk = (col & 63) >> 3;
      float s4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
      for (int rr = r0; rr < r0 + 64; rr += 4) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const unsigned short raw =
              *reinterpret_cast<const unsigned short*>(colbase + (rr + u) * 128 + ((chunk ^ ((rr + u) & 7)) << 4));
          s4[u] += F16Traits<T>::lo(static_cast<uint32_t>(raw));
        }
      }
      ksum_acc += (s4[0] + s4[1]) + (s4[2] + s4[3]);
    }
  }
  wgmma_wait<0>();
  reg_fence(acc);
  __syncthreads();   // both warpgroups' MMAs have retired: the V ring is free for the partials
  // ---- stage this CTA's partials.  kv in the layout of its global block: a 128-wide head's [dv][dk] rows 64wg.., or a
  // pair's two [64][64] blocks one after the other (accumulator rows = value channels, fragment layout in common.cuh).
  // ksum: thread t's sum over key rows 64(t/128).. of channel t % 128 (head0's channel, or a pair's channel c-64 of head0+1).
  float* const part = reinterpret_cast<float*>(smem + kOffV);
  {
    const int w4 = warp & 3;
    const int dv_lo = w4 * 16 + (lane >> 2), cq = 2 * (lane & 3);
    float* const mine = part + wg * 64 * N;
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2)
        *reinterpret_cast<float2*>(mine + (dv_lo + 8 * h2) * N + 8 * j + cq) =
            make_float2(acc[4 * j + 2 * h2], acc[4 * j + 2 * h2 + 1]);
    part[kOffPartKsum / 4 + threadIdx.x] = ksum_acc;
  }
  cluster_sync_all();   // every split's partials are staged and visible across the cluster
  // ---- reduce: CTA `rank` owns every S-th run of kThreads float4 chunks; each element is summed over splits 0..S-1
  {
    const uint32_t rank = cluster_ctarank(), S = p.splits;
    const uint32_t SS = kVL ? uint32_t(splits) : S;   // the splits summed (kVL: the entry's; 0 for an entry with no rows)
    const uint32_t spart = smem_u32(part);
    const int64_t bh0 = int64_t(b) * p.h + head0;
    constexpr int kChunks = (kPair ? 2 * 64 * 64 : D * D) / 4;
    const int live_chunks = second_ok ? kChunks : kChunks / 2;   // odd head count: the last pair's second head is absent
    float4* const dst = reinterpret_cast<float4*>(p.kv + bh0 * (kPair ? 64 * 64 : D * D));
    // all S loads of an element are issued before the first add, so the remote reads overlap
    for (int c = int(rank) * kThreads + threadIdx.x; (!kVL || SS > 0) && c < live_chunks; c += S * kThreads) {
      float4 g = dst[c];
      float4 u[kMaxSplits];
#pragma unroll
      for (uint32_t s = 0; s < kMaxSplits; ++s)
        if (s < SS) u[s] = ld_dsmem_v4(spart + c * 16, s);
      float4 t = u[0];
#pragma unroll
      for (uint32_t s = 1; s < kMaxSplits; ++s)
        if (s < SS) { t.x += u[s].x; t.y += u[s].y; t.z += u[s].z; t.w += u[s].w; }
      g.x += t.x; g.y += t.y; g.z += t.z; g.w += t.w;
      dst[c] = g;
    }
    const int live_cols = second_ok ? 128 : 64;
    for (int c = int(rank) * kThreads + threadIdx.x; (!kVL || SS > 0) && c < live_cols; c += S * kThreads) {
      const uint32_t a = spart + kOffPartKsum + c * 4;
      float u[kMaxSplits][2];
#pragma unroll
      for (uint32_t s = 0; s < kMaxSplits; ++s)
        if (s < SS) { u[s][0] = ld_dsmem_f32(a, s); u[s][1] = ld_dsmem_f32(a + 128 * 4, s); }
      float t = u[0][0] + u[0][1];
#pragma unroll
      for (uint32_t s = 1; s < kMaxSplits; ++s)
        if (s < SS) t += u[s][0] + u[s][1];
      p.ksum[bh0 * p.hd + c] += t;   // a pair's channels 64.. are head0+1's, which follow head0's 64 in ksum
    }
  }
  cluster_sync_all();   // no CTA leaves while another still reads its shared memory
}

}  // namespace

extern "C" int tdb200_sla_linear_moments(const void* k, const void* v, int dtype, int64_t b, int64_t l, int64_t h,
                                         int64_t d, int feature, float* kv, float* ksum, void* stream) {
  using namespace tdb;
  if (!k || !v || !kv || !ksum) return fail(TDB200_ERR_INVALID_ARG, "sla_linear_moments: null pointer");
  if (b <= 0 || l <= 0 || h <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_linear_moments: bad shape");
  if (d != 64 && d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_linear_moments: head dim %lld (64 or 128, SLA/core.py:207)", (long long)d);
  if (feature < 0 || feature > 2) return fail(TDB200_ERR_INVALID_ARG, "sla_linear_moments: feature map tag %d", feature);
  if (h > 65535 || b > 65535) return fail(TDB200_ERR_UNSUPPORTED, "sla_linear_moments: h or b too large");
  if (!aligned16(k) || !aligned16(kv)) return fail(TDB200_ERR_INVALID_ARG, "sla_linear_moments: buffers must be 16-byte aligned");
  if (int rc = require_sm90()) return rc;
  const CUtensorMapDataType t16 = dtype == TDB200_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap tv;
  {
    const uint64_t dims[4] = {uint64_t(d), uint64_t(h), uint64_t(l), uint64_t(b)};
    const uint64_t str[3] = {uint64_t(d * 2), uint64_t(h * d * 2), uint64_t(l * h * d * 2)};
    const uint32_t box[4] = {64, 1, kRowsPerTile, 1};
    if (int rc = make_tmap_4d(&tv, v, t16, 2, dims, str, box)) return rc;
  }
  const int64_t units = d == 128 ? h : cdiv64(h, 2);   // CTAs along x: heads, or pairs of 64-wide heads
  MomParams p;
  p.k = k;
  p.kv = kv;
  p.ksum = ksum;
  p.l = int(l);
  p.h = int(h);
  p.hd = int(d);
  p.feature = feature;
  p.seq_lens = nullptr;
  p.tiles = int(cdiv64(l, kRowsPerTile));
  p.splits = p.tiles < kMaxSplits ? p.tiles : kMaxSplits;   // the tile count alone decides the summation order
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(units), static_cast<unsigned>(p.splits), static_cast<unsigned>(b));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = kSmemBytes;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute cluster;
  cluster.id = cudaLaunchAttributeClusterDimension;
  cluster.val.clusterDim.x = 1;
  cluster.val.clusterDim.y = static_cast<unsigned>(p.splits);   // the split CTAs of one (head or pair, b)
  cluster.val.clusterDim.z = 1;
  cfg.attrs = &cluster;
  cfg.numAttrs = 1;
#define TDB_MOM2(T, PAIR)                                                                                          \
  do {                                                                                                              \
    static bool attr_done[64] = {false};                                                                            \
    if (int rc = set_max_dynamic_smem_once(reinterpret_cast<const void*>(sla_moments_kernel<T, PAIR>), kSmemBytes, attr_done, \
                                           "cudaFuncSetAttribute(sla_moments)"))                                   \
      return rc;                                                                                                    \
    return check_cuda(cudaLaunchKernelEx(&cfg, sla_moments_kernel<T, PAIR>, tv, p), "sla_moments_kernel");          \
  } while (0)
#define TDB_MOM(T) do { if (d == 64) { TDB_MOM2(T, true); } else { TDB_MOM2(T, false); } } while (0)
  if (dtype == TDB200_DTYPE_BF16) TDB_MOM(__nv_bfloat16);
  if (dtype == TDB200_DTYPE_FP16) TDB_MOM(__half);
#undef TDB_MOM2
#undef TDB_MOM
  return fail(TDB200_ERR_UNSUPPORTED, "sla_linear_moments: dtype tag %d", dtype);
}

// ---- kvw = T(proj_w . kv): the linear branch's output projection folded into the moment matrix (SLA/core.py:243-253:
// proj_l(phi(q) kv / den) == phi(q) (proj_w kv)^T / den + b), one launch instead of a library sgemm plus casts.
//   proj_w [d_out, d_v] fp32, kv [bh, d_v, d_k] fp32  ->  kvw [bh, d_out, d_k] T;  fp32 FMA chain over d_v in ascending order.
namespace {
template <typename T, int D>
__global__ void __launch_bounds__(D) project_moments_kernel(const float* __restrict__ w, const float* __restrict__ kv,
                                                            T* __restrict__ out) {
  constexpr int kRows = 32;                      // output rows (d_out) per CTA
  __shared__ float ws[kRows][D];
  const int bh = blockIdx.x, o0 = blockIdx.y * kRows, k = threadIdx.x;
  for (int i = threadIdx.x; i < kRows * D; i += D) ws[i / D][i % D] = __ldg(w + int64_t(o0 + i / D) * D + (i % D));
  __syncthreads();
  float acc[kRows];
#pragma unroll
  for (int i = 0; i < kRows; ++i) acc[i] = 0.f;
  const float* kvp = kv + int64_t(bh) * D * D + k;
#pragma unroll 4
  for (int v = 0; v < D; ++v) {
    const float x = __ldg(kvp + int64_t(v) * D);
#pragma unroll
    for (int i = 0; i < kRows; ++i) acc[i] = fmaf(ws[i][v], x, acc[i]);
  }
  T* op = out + (int64_t(bh) * D + o0) * D + k;
#pragma unroll
  for (int i = 0; i < kRows; ++i) op[int64_t(i) * D] = static_cast<T>(acc[i]);
}
}  // namespace

extern "C" int tdb200_sla_project_moments(const float* proj_w, const float* kv, int dtype, int64_t bh, int64_t d, void* kvw,
                                          void* stream) {
  using namespace tdb;
  if (!proj_w || !kv || !kvw) return fail(TDB200_ERR_INVALID_ARG, "sla_project_moments: null pointer");
  if (bh <= 0 || bh > 0x7FFFFFFF) return fail(TDB200_ERR_INVALID_ARG, "sla_project_moments: bad shape");
  if (d != 64 && d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_project_moments: head dim %lld (64 or 128)", (long long)d);
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(static_cast<unsigned>(bh), static_cast<unsigned>(d / 32));
#define TDB_PM(T, D) project_moments_kernel<T, D><<<grid, D, 0, st>>>(proj_w, kv, static_cast<T*>(kvw)); return check_launch("project_moments_kernel")
  if (dtype == TDB200_DTYPE_BF16) {
    if (d == 128) { TDB_PM(__nv_bfloat16, 128); }
    TDB_PM(__nv_bfloat16, 64);
  }
  if (dtype == TDB200_DTYPE_FP16) {
    if (d == 128) { TDB_PM(__half, 128); }
    TDB_PM(__half, 64);
  }
#undef TDB_PM
  return fail(TDB200_ERR_UNSUPPORTED, "sla_project_moments: dtype tag %d", dtype);
}

// tdb200_sla_linear_moments for a padded batch: k and v [b, l, h, 128], seq_lens [b] (device int32, clamped to [0, l]).  Entry b's
// kv and ksum get the bits tdb200_sla_linear_moments gives on that entry alone cut to its first seq_lens[b] rows; what the rows
// past it hold, inf and NaN included, does not reach them.  Accumulated like tdb200_sla_linear_moments (the caller zeroes).
extern "C" int tdb200_sla_linear_moments_vl(const void* k, const void* v, int dtype, int64_t b, int64_t l, int64_t h, int64_t d,
                                            const int32_t* seq_lens, int feature, float* kv, float* ksum, void* stream) {
  using namespace tdb;
  if (!k || !v || !kv || !ksum) return fail(TDB200_ERR_INVALID_ARG, "sla_linear_moments_vl: null pointer");
  if (!seq_lens || (reinterpret_cast<uintptr_t>(seq_lens) & 3u))
    return fail(TDB200_ERR_INVALID_ARG, "sla_linear_moments_vl: seq_lens must be a non-null, 4-byte aligned int32 [b]");
  if (b <= 0 || l <= 0 || h <= 0) return fail(TDB200_ERR_INVALID_ARG, "sla_linear_moments_vl: bad shape");
  if (d != 128) return fail(TDB200_ERR_UNSUPPORTED, "sla_linear_moments_vl: head dim %lld (per-entry lengths serve d = 128)", (long long)d);
  if (feature < 0 || feature > 2) return fail(TDB200_ERR_INVALID_ARG, "sla_linear_moments_vl: feature map tag %d", feature);
  if (h > 65535 || b > 65535 || l > 0x7FFFFFFF) return fail(TDB200_ERR_UNSUPPORTED, "sla_linear_moments_vl: dimension too large");
  if (!aligned16(k) || !aligned16(kv)) return fail(TDB200_ERR_INVALID_ARG, "sla_linear_moments_vl: buffers must be 16-byte aligned");
  if (dtype != TDB200_DTYPE_BF16 && dtype != TDB200_DTYPE_FP16) return fail(TDB200_ERR_UNSUPPORTED, "sla_linear_moments_vl: dtype tag %d", dtype);
  if (int rc = require_sm90()) return rc;
  const CUtensorMapDataType t16 = dtype == TDB200_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap tv;
  {
    const uint64_t dims[4] = {uint64_t(d), uint64_t(h), uint64_t(l), uint64_t(b)};
    const uint64_t str[3] = {uint64_t(d * 2), uint64_t(h * d * 2), uint64_t(l * h * d * 2)};
    const uint32_t box[4] = {64, 1, kRowsPerTile, 1};
    if (int rc = make_tmap_4d(&tv, v, t16, 2, dims, str, box)) return rc;
  }
  MomParams p;
  p.k = k;
  p.kv = kv;
  p.ksum = ksum;
  p.l = int(l);
  p.h = int(h);
  p.hd = int(d);
  p.feature = feature;
  p.seq_lens = seq_lens;
  p.tiles = int(cdiv64(l, kRowsPerTile));
  p.splits = p.tiles < kMaxSplits ? p.tiles : kMaxSplits;   // the cluster size; each entry sums its own splits
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(h), static_cast<unsigned>(p.splits), static_cast<unsigned>(b));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = kSmemBytes;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute cluster;
  cluster.id = cudaLaunchAttributeClusterDimension;
  cluster.val.clusterDim.x = 1;
  cluster.val.clusterDim.y = static_cast<unsigned>(p.splits);
  cluster.val.clusterDim.z = 1;
  cfg.attrs = &cluster;
  cfg.numAttrs = 1;
#define TDB_MOM(T)                                                                                                  \
  do {                                                                                                              \
    static bool attr_done[64] = {false};                                                                            \
    if (int rc = set_max_dynamic_smem_once(reinterpret_cast<const void*>(sla_moments_kernel<T, false, true>), kSmemBytes, \
                                           attr_done, "cudaFuncSetAttribute(sla_moments_vl)"))                      \
      return rc;                                                                                                    \
    return check_cuda(cudaLaunchKernelEx(&cfg, sla_moments_kernel<T, false, true>, tv, p), "sla_moments_kernel<vl>"); \
  } while (0)
  if (dtype == TDB200_DTYPE_BF16) TDB_MOM(__nv_bfloat16);
  TDB_MOM(__half);
#undef TDB_MOM
}
