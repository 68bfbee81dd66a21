// a10 for training: SparseLinearAttention's linear branch and proj_l, forward and backward (reference: turbodiffusion/SLA/core.py:
// 104-117).  Per (batch, head), with phi the feature map, c_q = phi(q), c_k = phi(k) rounded to T, M = sum_j c_k,j^T v_j and
// s = sum_j c_k,j (tdb200_sla_linear_moments: kv = M^T and ksum in fp32):
//   den_i = 1e-5 + c_q,i . s     u_i = c_q,i M / den_i     o_l,i = T(u_i W^T + b)
// Backward, g = dL/do_l:
//   du = g W   e = du.u / den   dc_q = du M^T / den - e s   dM = sum_i c_q,i^T du_i / den_i   ds = -sum_i e_i c_q,i
//   dc_k = v dM^T + ds   dv = c_k dM   dq = J_phi(q)^T dc_q   dk = J_phi(k)^T dc_k   dW = sum g^T u   db = sum g
//
// Every product is a 16-bit tensor-core MMA (mma.sync m16n8k16, fp32 accumulation) on a warp's 16 rows.  Row kernels: one CTA
// of 4 warps per 64 rows of one (b, h); the 128 x 128 right-hand matrices (M, W, dM and their transposes) are staged once per
// CTA in shared memory as T, [n][k] with a 136-element row pitch (conflict-free fragment loads).  Reductions over rows (dM,
// dW) are a separate X^T.Y kernel over row-major operands the query pass writes to the workspace, summed in a fixed order:
// each (b, h) splits its 64-row tiles over min(tiles, kSplits) CTAs (split s owns tiles s, s + S, ...), and one more kernel
// adds the split partials (and, for dW and db, the (b, h) partials) in ascending order.  No floating-point atomics: the bits
// depend only on the inputs, and a (b, h)'s dq, dk, dv and o_l only on that head's inputs.
//
// Operand range.  M and dM grow with L, and 1/den reaches 1e5 on rows whose features sit on channels every key leaves at 0.
// M and dM are fp32 and enter the MMA scaled by a power of two per (b, h) that puts their largest magnitude in [2^14, 2^15)
// (undone in fp32 on the accumulator, exactly).  The dM reduction's operands c_q,i and du_i / den_i share a per-row power of
// two: c_q,i 2^e and (du_i / den_i) 2^-e, e balancing the two rows' largest exponents, so neither leaves T's range where
// their product fits.  u (a convex combination of v rows scaled by < 1) and du need no scaling.  The same scalings run in
// both dtypes (in bf16 they change no bit unless a value would otherwise be subnormal).
#include <type_traits>

#include "common.cuh"
#include "host_common.h"

namespace {
using namespace tdb;

constexpr int D = 128;
constexpr int kRows = 64;          // rows per row-kernel CTA (4 warps x 16) and per X^T.Y tile
constexpr int kPitch = 136;        // shared-memory row pitch of a staged matrix, in 16-bit elements (272 B)
constexpr int kMatBytes = D * kPitch * 2;
constexpr int kSplits = 16;        // X^T.Y CTAs per (b, h) at most; the tile count alone decides the split
constexpr float kLog2e = 1.4426950408889634f;

template <typename T>
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (std::is_same<T, __nv_bfloat16>::value) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

// A warp's 16 x 128 block of rows in the MMA accumulator layout: x[j][0..1] = row g, columns 8j + 2t, +1; x[j][2..3] = row
// g + 8 (g = lane / 4, t = lane % 4).  Row data are loaded into it, and per-row sums reduce over j and the lane quad.
using Rows = float[16][4];

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// rows r0 (x[j][0..1]) and r0 + 8 (x[j][2..3]) of a [*, h, 128] 16-bit tensor at `base` (row stride `rs` elements); rows at
// or past `l` read as zeros and are not touched
template <typename T>
__device__ __forceinline__ void load_rows(Rows& x, const T* base, int64_t rs, int64_t r0, int64_t l) {
  const int t = threadIdx.x & 3;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int64_t r = r0 + 8 * hh;
    const uint32_t* p = reinterpret_cast<const uint32_t*>(base + (r < l ? r : 0) * rs + 2 * t);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const uint32_t w = r < l ? __ldg(p + 4 * j) : 0u;
      x[j][2 * hh] = F16Traits<T>::lo(w);
      x[j][2 * hh + 1] = F16Traits<T>::hi(w);
    }
  }
}

template <typename T>
__device__ __forceinline__ void store_rows(const Rows& x, T* base, int64_t rs, int64_t r0, int64_t l) {
  const int t = threadIdx.x & 3;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int64_t r = r0 + 8 * hh;
    if (r >= l) continue;
    uint32_t* p = reinterpret_cast<uint32_t*>(base + r * rs + 2 * t);
#pragma unroll
    for (int j = 0; j < 16; ++j) p[4 * j] = F16Traits<T>::pack(x[j][2 * hh], x[j][2 * hh + 1]);
  }
}

// x rounded to T as the A operand of a 16 x 128 (K) MMA row block
template <typename T>
__device__ __forceinline__ void to_afrag(uint32_t (&a)[8][4], const Rows& x) {
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    a[kk][0] = F16Traits<T>::pack(x[2 * kk][0], x[2 * kk][1]);
    a[kk][1] = F16Traits<T>::pack(x[2 * kk][2], x[2 * kk][3]);
    a[kk][2] = F16Traits<T>::pack(x[2 * kk + 1][0], x[2 * kk + 1][1]);
    a[kk][3] = F16Traits<T>::pack(x[2 * kk + 1][2], x[2 * kk + 1][3]);
  }
}

// c = A . B (kAcc: c += A . B) for the warp's 16 rows, B[k][n] staged as S[n][k] (pitch kPitch)
template <typename T, bool kAcc = false>
__device__ __forceinline__ void rows_times(Rows& c, const uint32_t (&a)[8][4], const T* s) {
  const int g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
  if (!kAcc) {
#pragma unroll
    for (int j = 0; j < 16; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.f;
  }
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const T* p = s + (8 * j + g) * kPitch + 16 * kk + 2 * t;
      mma16816<T>(c[j], a[kk], *reinterpret_cast<const uint32_t*>(p), *reinterpret_cast<const uint32_t*>(p + 8));
    }
}

// phi of the rows in x (in place, fp32) for feature map F: 0 softmax over the head, 1 elu + 1, 2 relu
template <int F>
__device__ __forceinline__ void feature_map(Rows& x) {
  if constexpr (F == 0) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float m = -INFINITY;
#pragma unroll
      for (int j = 0; j < 16; ++j) m = fmaxf(m, fmaxf(x[j][2 * hh], x[j][2 * hh + 1]));
      m = quad_max(m);
      const float off = m * kLog2e;
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          x[j][2 * hh + u] = fast_exp2(fmaf(x[j][2 * hh + u], kLog2e, -off));
          sum += x[j][2 * hh + u];
        }
      const float inv = 1.0f / quad_sum(sum);
#pragma unroll
      for (int j = 0; j < 16; ++j) { x[j][2 * hh] *= inv; x[j][2 * hh + 1] *= inv; }
    }
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float a = x[j][u];
        x[j][u] = F == 1 ? (a > 0.f ? a + 1.0f : fast_exp2(a * kLog2e)) : fmaxf(a, 0.f);
      }
  }
}

// dx = J_phi(x)^T dc in place in dc, x the pre-feature rows (overwritten)
template <int F>
__device__ __forceinline__ void feature_vjp(Rows& dc, Rows& x) {
  if constexpr (F == 0) {
    feature_map<0>(x);   // c
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float dot = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) dot += x[j][2 * hh] * dc[j][2 * hh] + x[j][2 * hh + 1] * dc[j][2 * hh + 1];
      dot = quad_sum(dot);
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int u = 0; u < 2; ++u) dc[j][2 * hh + u] = x[j][2 * hh + u] * (dc[j][2 * hh + u] - dot);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float a = x[j][u];
        dc[j][u] *= F == 1 ? (a > 0.f ? 1.0f : fast_exp2(a * kLog2e)) : (a > 0.f ? 1.0f : 0.f);
      }
  }
}

// dc = J_phi(x) . dx in place in dx, from c = phi(x) in fp32 (elu+1: phi' = 1 where c > 1, else c; relu: phi' = 1 where c > 0)
template <int F>
__device__ __forceinline__ void feature_jvp(Rows& dx, const Rows& c) {
  if constexpr (F == 0) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float dot = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) dot += c[j][2 * hh] * dx[j][2 * hh] + c[j][2 * hh + 1] * dx[j][2 * hh + 1];
      dot = quad_sum(dot);
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int u = 0; u < 2; ++u) dx[j][2 * hh + u] = c[j][2 * hh + u] * (dx[j][2 * hh + u] - dot);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float cc = c[j][u];
        dx[j][u] *= F == 1 ? (cc > 1.0f ? 1.0f : cc) : (cc > 0.f ? 1.0f : 0.f);
      }
  }
}

// c rounded to T (what the moments kernel and the reference multiply with)
template <typename T>
__device__ __forceinline__ void round_rows(Rows& x) {
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int u = 0; u < 4; ++u) x[j][u] = F16Traits<T>::round(x[j][u]);
}

// den_i = 1e-5 + c_i . s for the lane's two rows
__device__ __forceinline__ void row_den(float (&den)[2], const Rows& c, const float* s) {
  const int t = threadIdx.x & 3;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float a = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) a += c[j][2 * hh] * s[8 * j + 2 * t] + c[j][2 * hh + 1] * s[8 * j + 2 * t + 1];
    den[hh] = 1e-5f + quad_sum(a);
  }
}

// 2^-e with max|src| 2^-e in [2^14, 2^15) (1 for an all-zero matrix), for src [128 x 128] fp32; all threads of the CTA call it
__device__ float range_scale(const float* src, float* red) {
  float m = 0.f;
  for (int i = threadIdx.x; i < D * D; i += blockDim.x) m = fmaxf(m, fabsf(src[i]));
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = 0.f;
  for (int w = 0; w < int(blockDim.x >> 5); ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  if (!(m > 0.f) || m > 3.0e38f) return 1.0f;
  int e;
  frexpf(m, &e);                 // m in [2^(e-1), 2^e)
  e = min(max(e - 15, -60), 60);   // two such scales stay within fp32 as a ratio
  return ldexpf(1.0f, -e);
}

// S[n][k] = T(src[n][k] * sc), or T(src[k][n] * sc) with kTrans, for src [128 x 128] fp32
template <typename T, bool kTrans>
__device__ void stage_mat(T* s, const float* src, float sc) {
  for (int i = threadIdx.x; i < D * D; i += blockDim.x) {
    const int r = i >> 7, c = i & 127;   // src row r, column c (coalesced reads)
    const T v = static_cast<T>(src[i] * sc);
    if (kTrans) s[c * kPitch + r] = v; else s[r * kPitch + c] = v;
  }
}

struct RowParams {
  int64_t l;
  int h;
};

// ---- forward: o_l = T(u W^T + b)
template <typename T, int F>
__global__ void __launch_bounds__(128) lin_fwd_kernel(const T* __restrict__ q, const float* __restrict__ kv,
                                                      const float* __restrict__ ksum, const float* __restrict__ w,
                                                      const float* __restrict__ bias, T* __restrict__ o, RowParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  T* s_kv = reinterpret_cast<T*>(smem);
  T* s_w = reinterpret_cast<T*>(smem + kMatBytes);
  float* s_s = reinterpret_cast<float*>(smem + 2 * kMatBytes);
  float* s_b = s_s + D;
  float* red = s_b + D;
  const int b = blockIdx.z, h = blockIdx.y;
  const int64_t bh = int64_t(b) * p.h + h;
  const float* kvp = kv + bh * D * D;
  const float sc = range_scale(kvp, red);
  stage_mat<T, false>(s_kv, kvp, sc);    // B[k = dk][n = dv] = M[dk][dv] = kv[dv][dk]
  stage_mat<T, false>(s_w, w, 1.0f);     // B[k = dv][n = out] = W[out][dv]
  for (int i = threadIdx.x; i < D; i += blockDim.x) { s_s[i] = ksum[bh * D + i]; s_b[i] = bias[i]; }
  __syncthreads();
  const int warp = threadIdx.x >> 5, g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
  const int64_t rs = int64_t(p.h) * D, r0 = int64_t(blockIdx.x) * kRows + 16 * warp + g;
  const T* qb = q + int64_t(b) * p.l * rs + int64_t(h) * D;
  Rows x, acc;
  uint32_t a[8][4];
  float den[2];
  load_rows<T>(x, qb, rs, r0, p.l);
  feature_map<F>(x);
  round_rows<T>(x);
  row_den(den, x, s_s);
  to_afrag<T>(a, x);
  rows_times<T>(acc, a, s_kv);
  const float un = 1.0f / sc;
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int u = 0; u < 4; ++u) acc[j][u] = acc[j][u] * un / den[u >> 1];
  to_afrag<T>(a, acc);
  rows_times<T>(x, a, s_w);
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int u = 0; u < 4; ++u) x[j][u] += s_b[8 * j + 2 * t + (u & 1)];
  store_rows<T>(x, o + int64_t(b) * p.l * rs + int64_t(h) * D, rs, r0, p.l);
}

// column sums of the warp's 16 rows of x into red[warp][128] (fixed order: lane rows, then g = 0..7 by butterfly)
__device__ __forceinline__ void warp_colsum(const Rows& x, const float (&wt)[2], float* red) {
  const int warp = threadIdx.x >> 5, g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      float v = x[j][u] * wt[0] + x[j][2 + u] * wt[1];
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if (g == 0) red[warp * D + 8 * j + 2 * t + u] = v;
    }
}

struct BwdQParams {
  int64_t l;
  int h, tiles;
};

// ---- backward, query rows: dq, the per-tile partials of ds and db, and the row-major operands of dM (c_q 2^e, du / den 2^-e)
// and of dW (u) in the workspace
template <typename T, int F>
__global__ void __launch_bounds__(128) lin_bwd_q_kernel(const T* __restrict__ q, const T* __restrict__ gin,
                                                        const float* __restrict__ kv, const float* __restrict__ ksum,
                                                        const float* __restrict__ w, T* __restrict__ dq, T* __restrict__ cw,
                                                        T* __restrict__ pw, T* __restrict__ uw, float* __restrict__ dsp,
                                                        float* __restrict__ dbp, BwdQParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  T* s_kv = reinterpret_cast<T*>(smem);
  T* s_kvt = reinterpret_cast<T*>(smem + kMatBytes);
  T* s_wt = reinterpret_cast<T*>(smem + 2 * kMatBytes);
  float* s_s = reinterpret_cast<float*>(smem + 3 * kMatBytes);
  float* red = s_s + D;   // [2][4][128]
  const int b = blockIdx.z, h = blockIdx.y;
  const int64_t bh = int64_t(b) * p.h + h;
  const float* kvp = kv + bh * D * D;
  const float sc = range_scale(kvp, red);
  stage_mat<T, false>(s_kv, kvp, sc);    // c_q M:   B[k = dk][n = dv] = kv[dv][dk]
  stage_mat<T, true>(s_kvt, kvp, sc);    // du M^T:  B[k = dv][n = dk] = kv[dv][dk]
  stage_mat<T, true>(s_wt, w, 1.0f);     // g W:     B[k = out][n = dv] = W[out][dv]
  for (int i = threadIdx.x; i < D; i += blockDim.x) s_s[i] = ksum[bh * D + i];
  __syncthreads();
  const int warp = threadIdx.x >> 5;
  const int g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
  const int64_t rs = int64_t(p.h) * D, r0 = int64_t(blockIdx.x) * kRows + 16 * warp + g;
  const int64_t off = int64_t(b) * p.l * rs + int64_t(h) * D;
  const float un = 1.0f / sc;
  Rows x, du, acc;
  uint32_t a[8][4];
  float den[2];
  const float one[2] = {1.0f, 1.0f};
  // du = g W, and g's column sums (db)
  load_rows<T>(x, gin + off, rs, r0, p.l);
  warp_colsum(x, one, red + 4 * D);
  to_afrag<T>(a, x);
  rows_times<T>(du, a, s_wt);
  // c_q, den, u = c_q M / den
  load_rows<T>(x, q + off, rs, r0, p.l);
  feature_map<F>(x);
  round_rows<T>(x);
  row_den(den, x, s_s);
  float cmax[2], e[2], up[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float m = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) m = fmaxf(m, fmaxf(fabsf(x[j][2 * hh]), fabsf(x[j][2 * hh + 1])));
    cmax[hh] = quad_max(m);
  }
  to_afrag<T>(a, x);     // c_q: kept as the operand below (exact: x is rounded to T)
  rows_times<T>(acc, a, s_kv);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        acc[j][2 * hh + u] = acc[j][2 * hh + u] * un / den[hh];
        dot += du[j][2 * hh + u] * acc[j][2 * hh + u];
      }
    e[hh] = quad_sum(dot) / den[hh];
  }
  store_rows<T>(acc, uw + off, rs, r0, p.l);   // u (dW's right operand)
  // dM's operands: c_q 2^sh and du / den 2^-sh, sh splitting the two rows' largest exponents
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float m = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        acc[j][2 * hh + u] = du[j][2 * hh + u] / den[hh];
        m = fmaxf(m, fabsf(acc[j][2 * hh + u]));
      }
    m = quad_max(m);
    int sh = 0;
    if (m > 0.f && cmax[hh] > 0.f && m < 3.0e38f) {
      int pe, ce;
      frexpf(m, &pe);
      frexpf(cmax[hh], &ce);
      sh = min(max((pe - ce) >> 1, -60), 60);
    }
    up[hh] = ldexpf(1.0f, sh);
    const float dn = ldexpf(1.0f, -sh);
#pragma unroll
    for (int j = 0; j < 16; ++j) { acc[j][2 * hh] *= dn; acc[j][2 * hh + 1] *= dn; }
  }
  store_rows<T>(acc, pw + off, rs, r0, p.l);
  // c_q back from its operand copy (exact): ds partial -sum_i e_i c_q,i, then dM's left operand c_q 2^sh
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      x[2 * kk + (r & 2 ? 1 : 0)][(r & 1) * 2] = F16Traits<T>::lo(a[kk][r]);
      x[2 * kk + (r & 2 ? 1 : 0)][(r & 1) * 2 + 1] = F16Traits<T>::hi(a[kk][r]);
    }
  const float ne[2] = {-e[0], -e[1]};
  warp_colsum(x, ne, red);
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int u = 0; u < 4; ++u) x[j][u] *= up[u >> 1];
  store_rows<T>(x, cw + off, rs, r0, p.l);
  // dc_q = du M^T / den - e s, dq = J^T dc_q
  to_afrag<T>(a, du);
  rows_times<T>(acc, a, s_kvt);
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int u = 0; u < 4; ++u) acc[j][u] = acc[j][u] * un / den[u >> 1] - e[u >> 1] * s_s[8 * j + 2 * t + (u & 1)];
  load_rows<T>(x, q + off, rs, r0, p.l);
  feature_vjp<F>(acc, x);
  store_rows<T>(acc, dq + off, rs, r0, p.l);
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * D; c += blockDim.x) {
    const float* r = red + (c >= D ? 4 * D : 0) + (c & (D - 1));
    const float s = ((r[0] + r[D]) + r[2 * D]) + r[3 * D];
    (c >= D ? dbp : dsp)[(bh * p.tiles + blockIdx.x) * D + (c & (D - 1))] = s;
  }
}

// ---- backward, key rows: dv = c_k dM, dk = J^T (v dM^T + ds)
template <typename T, int F>
__global__ void __launch_bounds__(128) lin_bwd_k_kernel(const T* __restrict__ k, const T* __restrict__ v,
                                                        const float* __restrict__ dm, const float* __restrict__ ds,
                                                        T* __restrict__ dk, T* __restrict__ dv, RowParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  T* s_dm = reinterpret_cast<T*>(smem);
  T* s_dmt = reinterpret_cast<T*>(smem + kMatBytes);
  float* s_ds = reinterpret_cast<float*>(smem + 2 * kMatBytes);
  float* red = s_ds + D;
  const int b = blockIdx.z, h = blockIdx.y;
  const int64_t bh = int64_t(b) * p.h + h;
  const float* dmp = dm + bh * D * D;    // dM [dk][dv]
  const float sc = range_scale(dmp, red);
  stage_mat<T, false>(s_dm, dmp, sc);    // v dM^T: B[k = dv][n = dk] = dM[dk][dv]
  stage_mat<T, true>(s_dmt, dmp, sc);    // c_k dM: B[k = dk][n = dv] = dM[dk][dv]
  for (int i = threadIdx.x; i < D; i += blockDim.x) s_ds[i] = ds[bh * D + i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
  const int64_t rs = int64_t(p.h) * D, r0 = int64_t(blockIdx.x) * kRows + 16 * warp + g;
  const int64_t off = int64_t(b) * p.l * rs + int64_t(h) * D;
  const float un = 1.0f / sc;
  Rows x, acc;
  uint32_t a[8][4];
  load_rows<T>(x, k + off, rs, r0, p.l);
  feature_map<F>(x);
  to_afrag<T>(a, x);
  rows_times<T>(acc, a, s_dmt);
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int u = 0; u < 4; ++u) acc[j][u] *= un;
  store_rows<T>(acc, dv + off, rs, r0, p.l);
  load_rows<T>(x, v + off, rs, r0, p.l);
  to_afrag<T>(a, x);
  rows_times<T>(acc, a, s_dm);
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int u = 0; u < 4; ++u) acc[j][u] = acc[j][u] * un + s_ds[8 * j + 2 * t + (u & 1)];
  load_rows<T>(x, k + off, rs, r0, p.l);
  feature_vjp<F>(acc, x);
  store_rows<T>(acc, dk + off, rs, r0, p.l);
}

// ---- tangent, key rows: C = T(c_k), Cdot = T(J_phi(k) k_t) (the row operands of Mdot^T = V^T Cdot + V_t^T C) and the
// per-tile partials of sdot = sum_j J_phi(k_j) k_t,j (fp32)
template <typename T, int F>
__global__ void __launch_bounds__(128) lin_tan_k_kernel(const T* __restrict__ k, const T* __restrict__ k_t, T* __restrict__ cw,
                                                        T* __restrict__ ctw, float* __restrict__ sdp, BwdQParams p) {
  __shared__ float red[4 * D];
  const int b = blockIdx.z, h = blockIdx.y;
  const int64_t bh = int64_t(b) * p.h + h;
  const int warp = threadIdx.x >> 5, g = (threadIdx.x & 31) >> 2;
  const int64_t rs = int64_t(p.h) * D, r0 = int64_t(blockIdx.x) * kRows + 16 * warp + g;
  const int64_t off = int64_t(b) * p.l * rs + int64_t(h) * D;
  Rows c, ct;
  load_rows<T>(c, k + off, rs, r0, p.l);
  feature_map<F>(c);
  load_rows<T>(ct, k_t + off, rs, r0, p.l);
  feature_jvp<F>(ct, c);
  const float one[2] = {1.0f, 1.0f};
  warp_colsum(ct, one, red);   // rows past l read zero tangents: their cdot is 0
  store_rows<T>(c, cw + off, rs, r0, p.l);
  store_rows<T>(ct, ctw + off, rs, r0, p.l);
  __syncthreads();
  for (int c0 = threadIdx.x; c0 < D; c0 += blockDim.x)
    sdp[(bh * p.tiles + blockIdx.x) * D + c0] = ((red[c0] + red[D + c0]) + red[2 * D + c0]) + red[3 * D + c0];
}

// ---- tangent, query rows: o_l_t = T(udot W^T), udot = (cdot M + c Mdot) / den - u (cdot.s + c.sdot) / den
template <typename T, int F>
__global__ void __launch_bounds__(128) lin_tan_q_kernel(const T* __restrict__ q, const T* __restrict__ q_t,
                                                        const float* __restrict__ kv, const float* __restrict__ ksum,
                                                        const float* __restrict__ kvd, const float* __restrict__ sd,
                                                        const float* __restrict__ w, T* __restrict__ ot, RowParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  T* s_kv = reinterpret_cast<T*>(smem);
  T* s_kvd = reinterpret_cast<T*>(smem + kMatBytes);
  T* s_w = reinterpret_cast<T*>(smem + 2 * kMatBytes);
  float* s_s = reinterpret_cast<float*>(smem + 3 * kMatBytes);
  float* s_sd = s_s + D;
  float* red = s_sd + D;
  const int b = blockIdx.z, h = blockIdx.y;
  const int64_t bh = int64_t(b) * p.h + h;
  const float sc = range_scale(kv + bh * D * D, red);
  const float scd = range_scale(kvd + bh * D * D, red);
  stage_mat<T, false>(s_kv, kv + bh * D * D, sc);
  stage_mat<T, false>(s_kvd, kvd + bh * D * D, scd);
  stage_mat<T, false>(s_w, w, 1.0f);
  for (int i = threadIdx.x; i < D; i += blockDim.x) { s_s[i] = ksum[bh * D + i]; s_sd[i] = sd[bh * D + i]; }
  __syncthreads();
  const int warp = threadIdx.x >> 5, g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
  const int64_t rs = int64_t(p.h) * D, r0 = int64_t(blockIdx.x) * kRows + 16 * warp + g;
  const int64_t off = int64_t(b) * p.l * rs + int64_t(h) * D;
  Rows x, xt;
  uint32_t ca[8][4], cta[8][4];
  float den[2], dden[2];
  load_rows<T>(x, q + off, rs, r0, p.l);
  feature_map<F>(x);
  load_rows<T>(xt, q_t + off, rs, r0, p.l);
  feature_jvp<F>(xt, x);
  round_rows<T>(x);
  row_den(den, x, s_s);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float a = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int col = 8 * j + 2 * t + u;
        a += xt[j][2 * hh + u] * s_s[col] + x[j][2 * hh + u] * s_sd[col];
      }
    dden[hh] = quad_sum(a);
  }
  to_afrag<T>(ca, x);
  to_afrag<T>(cta, xt);
  // xt <- (cdot M + c Mdot) scd: cdot (M sc) rescaled by scd / sc, then c (Mdot scd) added by the tensor core
  rows_times<T>(xt, cta, s_kv);
  const float r = scd / sc;
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int u = 0; u < 4; ++u) xt[j][u] *= r;
  rows_times<T, true>(xt, ca, s_kvd);
  rows_times<T>(x, ca, s_kv);          // u sc den
  const float un = 1.0f / sc, und = 1.0f / scd;
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float uu = x[j][u] * un / den[u >> 1];
      xt[j][u] = (xt[j][u] * und - uu * dden[u >> 1]) / den[u >> 1];
    }
  to_afrag<T>(ca, xt);
  rows_times<T>(x, ca, s_w);
  store_rows<T>(x, ot + off, rs, r0, p.l);
}

struct XtyParams {
  int64_t l;
  int h, tiles, splits;
};

// ---- part[b, h, split] = sum over the split's 64-row tiles of X^T Y, X and Y [b, l, h, 128] 16-bit: [128 (X col)][128 (Y col)] fp32
template <typename T>
__global__ void __launch_bounds__(256) xty_kernel(const T* __restrict__ xg, const T* __restrict__ yg, const T* __restrict__ xg2,
                                                  const T* __restrict__ yg2, float* __restrict__ part, XtyParams p) {
  __shared__ __align__(16) uint16_t sx_raw[kRows * kPitch];
  __shared__ __align__(16) uint16_t sy_raw[kRows * kPitch];
  T* const sx = reinterpret_cast<T*>(sx_raw);
  T* const sy = reinterpret_cast<T*>(sy_raw);
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int64_t rs = int64_t(p.h) * D, off = int64_t(b) * p.l * rs + int64_t(h) * D;
  Rows acc;
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  const int m0 = 16 * warp;
  const int mi = lane >> 3, mr = lane & 7;
  const uint32_t ax = smem_u32(sx) + 2 * (((mi >> 1) * 8 + mr) * kPitch + m0 + (mi & 1) * 8);   // A = X^T: k rows, m columns
  const uint32_t by = smem_u32(sy) + 2 * (((mi & 1) * 8 + mr) * kPitch + (mi >> 1) * 8);         // B = Y: k rows, n columns
  // with a second pair (xg2, yg2 non-null), each tile adds X^T Y and then X2^T Y2
  const int npairs = xg2 ? 2 : 1;
  for (int tile = split; tile < p.tiles; tile += p.splits)
  for (int pr = 0; pr < npairs; ++pr) {
    const T* const xs = pr ? xg2 : xg;
    const T* const ys = pr ? yg2 : yg;
    __syncthreads();
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int r = (threadIdx.x >> 4) + 16 * it, ch = threadIdx.x & 15;
      const int64_t row = int64_t(tile) * kRows + r;
      uint4 vx = make_uint4(0u, 0u, 0u, 0u), vy = vx;
      if (row < p.l) {
        vx = ldg_nc_v4(xs + off + row * rs + 8 * ch);
        vy = ldg_nc_v4(ys + off + row * rs + 8 * ch);
      }
      *reinterpret_cast<uint4*>(sx + r * kPitch + 8 * ch) = vx;
      *reinterpret_cast<uint4*>(sy + r * kPitch + 8 * ch) = vy;
    }
    __syncthreads();
#pragma unroll
    for (int kc = 0; kc < kRows / 16; ++kc) {
      uint32_t a[4];
      ldsm_x4_trans(a, ax + 2 * 16 * kc * kPitch);
#pragma unroll
      for (int j = 0; j < 16; j += 2) {
        uint32_t bb[4];
        ldsm_x4_trans(bb, by + 2 * (16 * kc * kPitch + 8 * j));
        mma16816<T>(acc[j], a, bb[0], bb[1]);
        mma16816<T>(acc[j + 1], a, bb[2], bb[3]);
      }
    }
  }
  float* dst = part + ((int64_t(b) * p.h + h) * p.splits + split) * D * D;
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
      *reinterpret_cast<float2*>(dst + (m0 + g + 8 * hh) * D + 8 * j + 2 * t) = make_float2(acc[j][2 * hh], acc[j][2 * hh + 1]);
}

// ---- out[o][i] = sum_{p < np} in[o][p][i], p ascending
__global__ void __launch_bounds__(256) sum_parts_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t np,
                                                        int64_t n) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x, o = blockIdx.y;
  if (i >= n) return;
  const float* src = in + o * np * n + i;
  float s = 0.f;
  for (int64_t q = 0; q < np; ++q) s += src[q * n];
  out[o * n + i] = s;
}

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

struct BwdLayout {
  size_t rows16, tile_part, split_part, mats, vecs, total;
  int tiles, splits;
};

BwdLayout bwd_layout(int64_t b, int64_t h, int64_t l) {
  BwdLayout w;
  w.tiles = int(cdiv64(l, kRows));
  w.splits = w.tiles < kSplits ? w.tiles : kSplits;
  w.rows16 = align256(size_t(b * l * h) * D * 2);
  w.tile_part = align256(size_t(b * h) * w.tiles * D * 4);
  w.split_part = align256(size_t(b * h) * w.splits * D * D * 4);
  w.mats = align256(size_t(b * h) * D * D * 4);
  w.vecs = align256(size_t(b * h) * D * 4);
  w.total = 3 * w.rows16 + 2 * w.tile_part + w.split_part + w.mats + w.vecs;
  return w;
}

// the checks every entry point shares; `what` prefixes the messages
int check_shape(const char* what, int dtype, int feature, int64_t b, int64_t l, int64_t h, int64_t d) {
  if (b <= 0 || l <= 0 || h <= 0 || d <= 0) return fail(TDB200_ERR_INVALID_ARG, "%s: bad shape", what);
  if (d != D) return fail(TDB200_ERR_UNSUPPORTED, "%s: head dim %lld (the linear-branch kernels serve 128)", what, (long long)d);
  if (dtype != TDB200_DTYPE_BF16 && dtype != TDB200_DTYPE_FP16) return fail(TDB200_ERR_UNSUPPORTED, "%s: dtype tag %d", what, dtype);
  if (feature < 0 || feature > 2) return fail(TDB200_ERR_UNSUPPORTED, "%s: feature map tag %d", what, feature);
  if (b * h > 65535) return fail(TDB200_ERR_UNSUPPORTED, "%s: b * h above 65535", what);
  if (l * h * d >= (int64_t(1) << 39) || cdiv64(l, kRows) > 0x7FFFFFFF)
    return fail(TDB200_ERR_UNSUPPORTED, "%s: l * h * d of 2^39 elements or more", what);
  return 0;
}

bool all_aligned(std::initializer_list<const void*> ps) {
  for (const void* p : ps)
    if (!aligned16(p)) return false;
  return true;
}

bool any_null(std::initializer_list<const void*> ps) {
  for (const void* p : ps)
    if (!p) return true;
  return false;
}

template <typename K, typename... A>
int launch_rows(K kernel, size_t smem, bool* done, const char* name, int64_t b, int64_t l, int64_t h, cudaStream_t st,
                A... args) {
  if (int rc = set_max_dynamic_smem_once(reinterpret_cast<const void*>(kernel), smem, done, name)) return rc;
  kernel<<<dim3(unsigned(cdiv64(l, kRows)), unsigned(h), unsigned(b)), 128, smem, st>>>(args...);
  return check_launch(name);
}

constexpr size_t kFwdSmem = 2 * kMatBytes + (2 * D + 8) * 4;
constexpr size_t kBwdQSmem = 3 * kMatBytes + (D + 8 * D) * 4;
constexpr size_t kBwdKSmem = 2 * kMatBytes + (D + 8) * 4;

template <typename T>
int fwd_dispatch(int feature, const void* q, const float* kv, const float* ksum, const float* w, const float* bias, void* o,
                 int64_t b, int64_t l, int64_t h, cudaStream_t st) {
  RowParams p{l, int(h)};
  static bool done[3][64] = {};
#define TDB_LF(F)                                                                                                          \
  if (feature == F)                                                                                                        \
    return launch_rows(lin_fwd_kernel<T, F>, kFwdSmem, done[F], "lin_fwd_kernel", b, l, h, st, static_cast<const T*>(q), kv, \
                       ksum, w, bias, static_cast<T*>(o), p);
  TDB_LF(0) TDB_LF(1) TDB_LF(2)
#undef TDB_LF
  return fail(TDB200_ERR_UNSUPPORTED, "sla_linear_fwd: feature map tag %d", feature);
}

template <typename T>
int bwd_dispatch(int feature, const T* q, const T* k, const T* v, const T* g, const float* kv, const float* ksum,
                 const float* w, T* dq, T* dk, T* dv, float* dw, float* db, uint8_t* ws, int64_t b, int64_t l, int64_t h,
                 cudaStream_t st) {
  const BwdLayout L = bwd_layout(b, h, l);
  T* cw = reinterpret_cast<T*>(ws);
  T* pw = reinterpret_cast<T*>(ws + L.rows16);
  T* uw = reinterpret_cast<T*>(ws + 2 * L.rows16);
  float* dsp = reinterpret_cast<float*>(ws + 3 * L.rows16);
  float* dbp = reinterpret_cast<float*>(ws + 3 * L.rows16 + L.tile_part);
  float* part = reinterpret_cast<float*>(ws + 3 * L.rows16 + 2 * L.tile_part);
  float* dm = reinterpret_cast<float*>(ws + 3 * L.rows16 + 2 * L.tile_part + L.split_part);
  float* ds = reinterpret_cast<float*>(ws + 3 * L.rows16 + 2 * L.tile_part + L.split_part + L.mats);
  const unsigned bh = unsigned(b * h);
  static bool done_q[3][64] = {}, done_k[3][64] = {};
  int rc = 0;
#define TDB_LQ(F)                                                                                                                 \
  if (feature == F)                                                                                                               \
    rc = launch_rows(lin_bwd_q_kernel<T, F>, kBwdQSmem, done_q[F], "lin_bwd_q_kernel", b, l, h, st, q, g, kv, ksum, w, dq, cw, pw, \
                     uw, dsp, dbp, BwdQParams{l, int(h), L.tiles});
  TDB_LQ(0) TDB_LQ(1) TDB_LQ(2)
#undef TDB_LQ
  if (rc) return rc;
  const XtyParams xp{l, int(h), L.tiles, L.splits};
  const dim3 xgrid(unsigned(L.splits), unsigned(h), unsigned(b));
  xty_kernel<T><<<xgrid, 256, 0, st>>>(cw, pw, nullptr, nullptr, part, xp);   // dM [dk][dv]
  if ((rc = check_launch("xty_kernel"))) return rc;
  sum_parts_kernel<<<dim3(D * D / 256, bh), 256, 0, st>>>(part, dm, L.splits, D * D);
  if ((rc = check_launch("sum_parts_kernel"))) return rc;
  sum_parts_kernel<<<dim3(1, bh), 256, 0, st>>>(dsp, ds, L.tiles, D);
  if ((rc = check_launch("sum_parts_kernel"))) return rc;
#define TDB_LK(F)                                                                                                          \
  if (feature == F)                                                                                                        \
    rc = launch_rows(lin_bwd_k_kernel<T, F>, kBwdKSmem, done_k[F], "lin_bwd_k_kernel", b, l, h, st, k, v, dm, ds, dk, dv, \
                     RowParams{l, int(h)});
  TDB_LK(0) TDB_LK(1) TDB_LK(2)
#undef TDB_LK
  if (rc) return rc;
  xty_kernel<T><<<xgrid, 256, 0, st>>>(g, uw, nullptr, nullptr, part, xp);    // dW [out][dv]
  if ((rc = check_launch("xty_kernel"))) return rc;
  sum_parts_kernel<<<dim3(D * D / 256, 1), 256, 0, st>>>(part, dw, int64_t(bh) * L.splits, D * D);
  if ((rc = check_launch("sum_parts_kernel"))) return rc;
  sum_parts_kernel<<<dim3(1, 1), 256, 0, st>>>(dbp, db, int64_t(bh) * L.tiles, D);
  return check_launch("sum_parts_kernel");
}

constexpr size_t kTanQSmem = 3 * kMatBytes + (2 * D + 8) * 4;

// tangent workspace: C, Cdot [b, l, h, d] 16-bit, sdot per-tile partials, Mdot split partials, Mdot, sdot
size_t tangent_bytes(const BwdLayout& L) { return 2 * L.rows16 + L.tile_part + L.split_part + L.mats + L.vecs; }

template <typename T>
int tan_dispatch(int feature, const T* q, const T* k, const T* v, const T* q_t, const T* k_t, const T* v_t, const float* kv,
                 const float* ksum, const float* w, T* ot, uint8_t* ws, int64_t b, int64_t l, int64_t h, cudaStream_t st) {
  const BwdLayout L = bwd_layout(b, h, l);
  T* cw = reinterpret_cast<T*>(ws);
  T* ctw = reinterpret_cast<T*>(ws + L.rows16);
  float* sdp = reinterpret_cast<float*>(ws + 2 * L.rows16);
  float* part = reinterpret_cast<float*>(ws + 2 * L.rows16 + L.tile_part);
  float* kvd = reinterpret_cast<float*>(ws + 2 * L.rows16 + L.tile_part + L.split_part);
  float* sd = reinterpret_cast<float*>(ws + 2 * L.rows16 + L.tile_part + L.split_part + L.mats);
  const unsigned bh = unsigned(b * h);
  const dim3 rgrid(unsigned(L.tiles), unsigned(h), unsigned(b));
  int rc = 0;
#define TDB_TK(F)                                                                                                         \
  if (feature == F) {                                                                                                     \
    lin_tan_k_kernel<T, F><<<rgrid, 128, 0, st>>>(k, k_t, cw, ctw, sdp, BwdQParams{l, int(h), L.tiles});                 \
    rc = check_launch("lin_tan_k_kernel");                                                                                \
  }
  TDB_TK(0) TDB_TK(1) TDB_TK(2)
#undef TDB_TK
  if (rc) return rc;
  xty_kernel<T><<<dim3(unsigned(L.splits), unsigned(h), unsigned(b)), 256, 0, st>>>(v, ctw, v_t, cw, part,
                                                                                     XtyParams{l, int(h), L.tiles, L.splits});
  if ((rc = check_launch("xty_kernel"))) return rc;   // Mdot^T [dv][dk], the layout of kv
  sum_parts_kernel<<<dim3(D * D / 256, bh), 256, 0, st>>>(part, kvd, L.splits, D * D);
  if ((rc = check_launch("sum_parts_kernel"))) return rc;
  sum_parts_kernel<<<dim3(1, bh), 256, 0, st>>>(sdp, sd, L.tiles, D);
  if ((rc = check_launch("sum_parts_kernel"))) return rc;
  static bool done[3][64] = {};
#define TDB_TQ(F)                                                                                                              \
  if (feature == F)                                                                                                            \
    return launch_rows(lin_tan_q_kernel<T, F>, kTanQSmem, done[F], "lin_tan_q_kernel", b, l, h, st, q, q_t, kv, ksum,      \
                       static_cast<const float*>(kvd), static_cast<const float*>(sd), w, ot, RowParams{l, int(h)});
  TDB_TQ(0) TDB_TQ(1) TDB_TQ(2)
#undef TDB_TQ
  return fail(TDB200_ERR_UNSUPPORTED, "sla_linear_tangent: feature map tag %d", feature);
}

}  // namespace

extern "C" int64_t tdb200_sla_linear_tangent_workspace_bytes(int64_t b, int64_t h, int64_t l, int64_t d) {
  using namespace tdb;
  if (int rc = check_shape("sla_linear_tangent_workspace_bytes", TDB200_DTYPE_BF16, 0, b, l, h, d)) return rc;
  return int64_t(tangent_bytes(bwd_layout(b, h, l)));
}

extern "C" int tdb200_sla_linear_tangent(const void* q, const void* k, const void* v, const void* q_t, const void* k_t,
                                         const void* v_t, const float* kv, const float* ksum, const float* proj_w, int dtype,
                                         int feature, void* o_l_t, void* workspace, int64_t workspace_bytes, int64_t b,
                                         int64_t l, int64_t h, int64_t d, void* stream) {
  using namespace tdb;
  if (any_null({q, k, v, q_t, k_t, v_t, kv, ksum, proj_w, o_l_t, workspace}))
    return fail(TDB200_ERR_INVALID_ARG, "sla_linear_tangent: null pointer");
  if (!all_aligned({q, k, v, q_t, k_t, v_t, kv, ksum, proj_w, o_l_t, workspace}))
    return fail(TDB200_ERR_INVALID_ARG, "sla_linear_tangent: buffers must be 16-byte aligned");
  if (int rc = check_shape("sla_linear_tangent", dtype, feature, b, l, h, d)) return rc;
  const size_t need = tangent_bytes(bwd_layout(b, h, l));
  if (workspace_bytes < int64_t(need))
    return fail(TDB200_ERR_WORKSPACE, "sla_linear_tangent: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
                (long long)need);
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
#define TDB_LT(T)                                                                                                          \
  return tan_dispatch<T>(feature, static_cast<const T*>(q), static_cast<const T*>(k), static_cast<const T*>(v),           \
                         static_cast<const T*>(q_t), static_cast<const T*>(k_t), static_cast<const T*>(v_t), kv, ksum,    \
                         proj_w, static_cast<T*>(o_l_t), ws, b, l, h, st)
  if (dtype == TDB200_DTYPE_BF16) TDB_LT(__nv_bfloat16);
  TDB_LT(__half);
#undef TDB_LT
}

extern "C" int tdb200_sla_linear_fwd(const void* q, const float* kv, const float* ksum, const float* proj_w,
                                     const float* proj_b, int dtype, int feature, void* o_l, int64_t b, int64_t l, int64_t h,
                                     int64_t d, void* stream) {
  using namespace tdb;
  if (any_null({q, kv, ksum, proj_w, proj_b, o_l})) return fail(TDB200_ERR_INVALID_ARG, "sla_linear_fwd: null pointer");
  if (!all_aligned({q, kv, ksum, proj_w, proj_b, o_l}))
    return fail(TDB200_ERR_INVALID_ARG, "sla_linear_fwd: buffers must be 16-byte aligned");
  if (int rc = check_shape("sla_linear_fwd", dtype, feature, b, l, h, d)) return rc;
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == TDB200_DTYPE_BF16) return fwd_dispatch<__nv_bfloat16>(feature, q, kv, ksum, proj_w, proj_b, o_l, b, l, h, st);
  return fwd_dispatch<__half>(feature, q, kv, ksum, proj_w, proj_b, o_l, b, l, h, st);
}

extern "C" int64_t tdb200_sla_linear_bwd_workspace_bytes(int64_t b, int64_t h, int64_t l, int64_t d) {
  using namespace tdb;
  if (int rc = check_shape("sla_linear_bwd_workspace_bytes", TDB200_DTYPE_BF16, 0, b, l, h, d)) return rc;
  return int64_t(bwd_layout(b, h, l).total);
}

extern "C" int tdb200_sla_linear_bwd(const void* q, const void* k, const void* v, const void* d_o, const float* kv,
                                     const float* ksum, const float* proj_w, int dtype, int feature, void* dq, void* dk,
                                     void* dv, float* dproj_w, float* dproj_b, void* workspace, int64_t workspace_bytes,
                                     int64_t b, int64_t l, int64_t h, int64_t d, void* stream) {
  using namespace tdb;
  if (any_null({q, k, v, d_o, kv, ksum, proj_w, dq, dk, dv, dproj_w, dproj_b, workspace}))
    return fail(TDB200_ERR_INVALID_ARG, "sla_linear_bwd: null pointer");
  if (!all_aligned({q, k, v, d_o, kv, ksum, proj_w, dq, dk, dv, dproj_w, dproj_b, workspace}))
    return fail(TDB200_ERR_INVALID_ARG, "sla_linear_bwd: buffers must be 16-byte aligned");
  if (int rc = check_shape("sla_linear_bwd", dtype, feature, b, l, h, d)) return rc;
  if (workspace_bytes < int64_t(bwd_layout(b, h, l).total))
    return fail(TDB200_ERR_WORKSPACE, "sla_linear_bwd: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
                (long long)bwd_layout(b, h, l).total);
  if (int rc = require_sm90()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
#define TDB_LB(T)                                                                                                         \
  return bwd_dispatch<T>(feature, static_cast<const T*>(q), static_cast<const T*>(k), static_cast<const T*>(v),          \
                         static_cast<const T*>(d_o), kv, ksum, proj_w, static_cast<T*>(dq), static_cast<T*>(dk),         \
                         static_cast<T*>(dv), dproj_w, dproj_b, ws, b, l, h, st)
  if (dtype == TDB200_DTYPE_BF16) TDB_LB(__nv_bfloat16);
  TDB_LB(__half);
#undef TDB_LB
}
