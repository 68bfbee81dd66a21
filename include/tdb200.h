/*
 * tdb200.h — C ABI of libtdb200.so: the H100 (sm_90a) implementation of TurboDiffusion's denoise hot path.
 *
 * This is the drop-in boundary.  Every entry point replaces one interface of the reference
 * (thu-ml/TurboDiffusion; citations are file:line inside that repository):
 *
 *   turbo_diffusion_ops.quant_cuda        turbodiffusion/ops/quant/quant.cu:28-71     -> tdb200_quant_int8_block128
 *   turbo_diffusion_ops.gemm_cuda         turbodiffusion/ops/gemm/gemm.cu:27-68       -> tdb200_gemm_w8a8
 *   turbo_diffusion_ops.rms_norm_cuda     turbodiffusion/ops/norm/rmsnorm.cu:57-59    -> tdb200_rms_norm_f32
 *   turbo_diffusion_ops.layer_norm_cuda   turbodiffusion/ops/norm/layernorm.cu:60-62  -> tdb200_layer_norm_f32
 *   ops.FastRMSNorm / FastLayerNorm fwd   turbodiffusion/ops/core.py:441-442,477-478  -> tdb200_rms_norm / tdb200_layer_norm
 *   AdaLN modulate / gate (caller math)   turbodiffusion/rcm/networks/wan2pt1.py:398-417 -> tdb200_layer_norm_modulate[_quant], tdb200_gate_residual
 *   rope_apply                            turbodiffusion/rcm/networks/wan2pt1.py:156-178 -> tdb200_rope_interleaved, tdb200_rms_norm_rope
 *   SLA.utils.get_block_map               turbodiffusion/SLA/utils.py:55-67           -> tdb200_sla_block_map
 *   spas_sage_attn get_vanilla_qk_quant   call site turbodiffusion/SLA/core.py:200-203 -> tdb200_sla_quant_qk
 *   Sage block-sparse attention + linear  turbodiffusion/SLA/core.py:231-253          -> tdb200_sla_linear_moments, tdb200_sla_attn_fwd
 *   attention (dense SDPA / FlashAttention) turbodiffusion/rcm/utils/attention.py:120-167 -> tdb200_attn_dense_fwd
 *   JVP flash attention (rCM distillation) turbodiffusion/rcm/networks/wan2pt1_jvp.py -> tdb200_attn_dense_jvp
 *   backward of the dense attention and of the JVP's primal                          -> tdb200_attn_dense_bwd
 *
 * Conventions
 *   - plain pointers and sizes; all pointers are DEVICE pointers unless stated; no allocation inside;
 *   - every call enqueues work on `stream` (a cudaStream_t passed as void*) and returns without synchronising;
 *   - return value: TDB200_OK or a negative TDB200_ERR_* code; the library never calls exit();
 *     tdb200_last_error() returns a thread-local description of the last failure;
 *   - reentrant per stream; no internal threads, no global mutable state besides per-device caches;
 *   - 16-bit floating tensors are described by a TDB200_DTYPE_* tag.
 */
#ifndef TDB200_H_
#define TDB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TDB200_ABI_VERSION 2

#define TDB200_OK 0
#define TDB200_ERR_INVALID_ARG (-1)  /* null pointer, bad size, misaligned buffer            */
#define TDB200_ERR_UNSUPPORTED (-2)  /* shape/dtype outside what the kernels implement        */
#define TDB200_ERR_CUDA (-3)         /* a CUDA runtime/driver call failed (see last_error)    */
#define TDB200_ERR_ARCH (-4)         /* current device is not compute capability 9.x          */
#define TDB200_ERR_WORKSPACE (-5)    /* caller-provided workspace too small                   */

#define TDB200_DTYPE_BF16 0
#define TDB200_DTYPE_FP16 1

/* ABI version of the loaded library (== TDB200_ABI_VERSION it was built with). */
int tdb200_abi_version(void);
/* Thread-local, NUL-terminated description of the most recent error on this thread ("" if none). */
const char* tdb200_last_error(void);

/* ---------------------------------------------------------------------------------------------
 * a1. per-128x128-block symmetric INT8 quantisation   (ops/quant/quant.hpp:86-99,122-164)
 *   x [m,k] row-major contiguous 16-bit float; q [m,k] int8; s [ceil(m/128), ceil(k/128)] fp32 row-major.
 *   per block: amax = max(1e-8, max|x|); s = amax/128; q = sat_s8(rint(x * (128/amax))).
 *   k must be a multiple of 8.  x and q 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
int tdb200_quant_int8_block128(const void* x, int x_dtype, int64_t m, int64_t k, int8_t* q, float* s, void* stream);
/* (q, s) = quant_int8_block128( T( gelu_tanh(x) ) ): the FFN activation (nn.GELU(approximate="tanh"),
 * rcm/networks/wan2pt1.py:375) and the quantisation of the down-projection's input in one HBM pass (2 B read, 1 B written
 * per element).  gelu in fp32 with one rounding to T, like torch on a 16-bit tensor. */
int tdb200_gelu_quant_int8_block128(const void* x, int x_dtype, int64_t m, int64_t k, int8_t* q, float* s, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a2. W8A8 GEMM with per-128-K-block rescale   (ops/gemm/kernel.hpp:391-427, utils.hpp:116-121)
 *   c[i,j] = T( sum_kb float(sum_{t in kb} a_q[i,t]*b_q[j,t]) * (a_s[i/128,kb]*b_s[j/128,kb]) )   fp32 FMA, kb ascending
 *   then, if bias != NULL,  c[i,j] = T(float(c[i,j]) + float(bias[j]))      (ops/core.py:410-411)
 *   a_q [m,k] int8, a_s [ceil(m/128), k/128]; b_q [n,k] int8 ("TN": both K-major), b_s [ceil(n/128), k/128];
 *   bias [n] of dtype c_dtype or NULL; c [m,n] row-major of dtype c_dtype.
 *   Requires k % 128 == 0 and n % 8 == 0 (the reference silently skips such shapes, gemm/launch.hpp:34-35;
 *   here they return TDB200_ERR_UNSUPPORTED).  wgmma int8, TMA-staged tiles, accumulators in registers.
 * ------------------------------------------------------------------------------------------- */
int tdb200_gemm_w8a8(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s, const void* bias,
                     void* c, int c_dtype, int64_t m, int64_t n, int64_t k, void* stream);
/* Same GEMM with a fused activation on the output:  TDB200_EPILOGUE_GELU_TANH computes
 * c = T(gelu_tanh(float(c_plain))) where c_plain is the value tdb200_gemm_w8a8 would store
 * (nn.GELU(approximate="tanh") after the FFN up-projection, rcm/networks/wan2pt1.py:375). */
#define TDB200_EPILOGUE_NONE 0
#define TDB200_EPILOGUE_GELU_TANH 1
int tdb200_gemm_w8a8_ex(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s, const void* bias,
                        void* c, int c_dtype, int64_t m, int64_t n, int64_t k, int epilogue, void* stream);
/* One W8A8 GEMM for projections that share their input (the q/k/v of a self-attention; reference: the fused to_qkv / to_kv
 * packing of TurboT2AV ltx_distillation/acceleration.py:836-860): b_q [n,k], b_s and bias are the row-wise concatenation of
 * `parts` equal projections (n = parts * n_part, n_part a multiple of 256); c receives `parts` separate contiguous
 * [m, n_part] matrices.  Scales are per 128 weight rows, so every output equals tdb200_gemm_w8a8 on its own weights. */
int tdb200_gemm_w8a8_split(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s, const void* bias,
                           void* c, int c_dtype, int64_t m, int64_t n, int64_t k, int64_t parts, void* stream);
/* GEMM whose output is emitted already block-quantised for the next W8A8 GEMM:
 *   (out_q, out_s) == tdb200_quant_int8_block128( output of tdb200_gemm_w8a8_ex in dtype `mid_dtype` )   bit for bit,
 * without the 16-bit tensor ever reaching HBM (FFN: Linear -> GELU -> Int8Linear, ops/core.py:28-57 called twice).
 * out_q [m,n] int8, out_s [ceil(m/128), n/128] fp32; n % 128 == 0. */
int tdb200_gemm_w8a8_quant_out(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s,
                               const void* bias, int8_t* out_q, float* out_s, int mid_dtype, int64_t m, int64_t n,
                               int64_t k, int epilogue, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a3/a4. FastNorm
 *   *_f32 : the registered-but-unused reference entry points (fp32 in, fp32 out), 1 CTA per row.
 *   16-bit variants: the whole FastRMSNorm.forward / FastLayerNorm.forward including the caller-side
 *   casts (x.float() in, .to(x.dtype) out) in ONE pass: y = T(float(x) * rstd * w), etc.
 *   w / b are fp32 [n] or NULL (no affine).  n % 8 == 0 (16-bit) / n % 4 == 0 (fp32), n <= 16384.
 * ------------------------------------------------------------------------------------------- */
int tdb200_rms_norm_f32(const float* x, const float* w, float* y, int64_t m, int64_t n, float eps, void* stream);
int tdb200_layer_norm_f32(const float* x, const float* w, const float* b, float* y, int64_t m, int64_t n, float eps,
                          void* stream);
int tdb200_rms_norm(const void* x, int dtype, const float* w, void* y, int64_t m, int64_t n, float eps, void* stream);
int tdb200_layer_norm(const void* x, int dtype, const float* w, const float* b, void* y, int64_t m, int64_t n,
                      float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a5. AdaLN prologue / epilogue   (rcm/networks/wan2pt1.py:398-417)
 *   layer_norm_modulate:        y = T( float(T(LN(x))) * (1 + scale[j]) + shift[j] )
 *   layer_norm_modulate_quant:  same value, emitted directly as a1-format int8 + block scales
 *                               (one stats pass + one tile pass instead of LN, 2 casts, modulate, quant).
 *                               row_stats: workspace of 2*m floats (mean, rstd per row).
 *   gate_residual:              out = T( x + T( y * T(gate[j]) ) )          (x + y*e under bf16 tensors)
 *   scale/shift/gate: fp32 [n] (one modulation vector: batch 1 per call).
 * ------------------------------------------------------------------------------------------- */
int tdb200_layer_norm_modulate(const void* x, int dtype, const float* scale, const float* shift, void* y, int64_t m,
                               int64_t n, float eps, void* stream);
int tdb200_layer_norm_modulate_quant(const void* x, int dtype, const float* scale, const float* shift, int8_t* q,
                                     float* s, float* row_stats, int64_t m, int64_t n, float eps, void* stream);
int tdb200_gate_residual(const void* x, const void* y, const float* gate, void* out, int dtype, int64_t m, int64_t n,
                         void* stream);
/* Cross-kernel fusion of the two above: the gate/residual update (gate == NULL: plain x + y) also emits the row
 * statistics (mean, rstd incl. the reference's variance padding term) of its OUTPUT, i.e. of the next LayerNorm's input,
 * and layer_norm_modulate_quant_stats is the tile pass alone, consuming them.  Results are bit-identical to
 * gate_residual followed by layer_norm_modulate_quant; one full read of the activation per LayerNorm is saved. */
int tdb200_gate_residual_stats(const void* x, const void* y, const float* gate, void* out, float* row_stats, int dtype,
                               int64_t m, int64_t n, float eps, void* stream);
int tdb200_layer_norm_modulate_quant_stats(const void* x, int dtype, const float* row_stats, const float* scale,
                                           const float* shift, int8_t* q, float* s, int64_t m, int64_t n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a6. RoPE, interleaved pairs   (rcm/networks/wan2pt1.py:156-178; flash_attn interleaved=True)
 *   x, y [l, h, d] contiguous 16-bit; angles [l, d/2] fp32 (radians).
 *   y[2i] = T(x[2i]*cos - x[2i+1]*sin), y[2i+1] = T(x[2i]*sin + x[2i+1]*cos), math in fp32.
 *   rms_norm_rope: y = rope( T( rmsnorm_{over h*d}(x) * w ) ) in one pass (norm_q/norm_k + rope_apply).
 * ------------------------------------------------------------------------------------------- */
int tdb200_rope_interleaved(const void* x, int dtype, const float* angles, void* y, int64_t l, int64_t h, int64_t d,
                            void* stream);
int tdb200_rms_norm_rope(const void* x, int dtype, const float* w, const float* angles, void* y, int64_t l, int64_t h,
                         int64_t d, float eps, void* stream);
/* rms_norm_rope with the rotation read from a table cos_sin [l, d/2, 2] fp32 = (cos a, sin a) of the same angles (the reference
 * precomputes its complex `freqs` once per call as well, wan2pt1.py:111-137,156-178): one table serves every head, projection
 * and layer of a denoise step, and the kernel carries no range reduction / sin / cos work. */
int tdb200_rms_norm_rope_table(const void* x, int dtype, const float* w, const float* cos_sin, void* y, int64_t l, int64_t h,
                               int64_t d, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a7-a10. SLA / SageSLA.  q, k, v, out are [b, l, h, d] contiguous 16-bit (the layout the module is
 * called with, SLA/core.py:181-183), d in {64, 128}.
 * Block families (blkq, blkk): (128, 64), the non-sm90 branch of SLA/core.py:191-193, or (64, 128), SpargeAttn's Hopper family
 * (SLA/core.py:191-193, 226-229); any other pair returns TDB200_ERR_UNSUPPORTED.
 * mblk = ceil(query rows / blkq), nblk = ceil(key rows / blkk).
 * INT8 K layouts: head-major [b,h,lk,d] (tdb200_sla_quant_qk), or sequence-major [b,lk,h,d] (tdb200_sla_quant_k_seq), the layout
 * in which sequence-parallel ranks all-gather their key rows.
 *
 * tdb200_sla_quant_qk   one pass over q [b,lq,h,d] and two over k [b,lk,h,d] (lq != lk when the query rows are one rank's
 *     sequence shard and k is the gathered key slab):
 *     kmean  [b,h,d]  fp32   = sum_l k / l  (T-rounded copy is what is subtracted, SLA/utils.py:56)
 *     q_i8   [b,h,lq,d] int8 per blkq rows, q_scale [b,h,mblk];  k_i8 [b,h,lk,d] int8 of T(k - T(kmean)) per blkk rows,
 *     k_scale [b,h,nblk]      scale = amax/127 + 1e-7, round half away from zero (SpargeAttn get_vanilla_qk_quant)
 *     q_pool [b,h,mblk,d] T,  k_pool [b,h,nblk,d] T   block means (SLA/utils.py:21-52; actual row count in the tail)
 *     q == NULL or k == NULL runs only the other half (the sequence-parallel path prepares Q while the K/V all-gather
 *     is still in flight); the pair (blkq, blkk) must still be one of the two families.
 * tdb200_sla_block_map  pooled score T(q_pool . k_pool^T), top-`topk` per row (ties -> lowest index),
 *     sparse_map [b,h,mblk,nblk] int8 0/1 (SLA/utils.py:64-66) and lut [b,h,mblk,topk] int32 ascending block ids.
 * tdb200_sla_linear_moments   phi = feature map of the keys: 0 softmax over d, 1 elu+1, 2 relu (SLA/core.py:57-73);
 *     kv [b,h,d(v),d(k)] fp32 = sum_l v[l,:]^T phi(k)[l,:], ksum [b,h,d] fp32 = sum_l phi(k)[l,:]   (SLA/core.py:243-247).
 *     Both must be zeroed by the caller (they are accumulated, so sequence shards can be summed with one all-reduce);
 *     each element receives one plain add of the call's total, so a second launch into the same buffer gives fp32(t + t).
 *     Reproducible: the bits of one (b, h) depend only on that head's k, v, l, d, feature map and dtype, not on the run,
 *     the GPU's SM count, the number of heads or batch entries in the call, or other work on the device.  The 128-row
 *     tiles are split over min(ceil(l/128), 8) CTAs of one thread-block cluster, whose partials are summed in split order
 *     without floating-point atomics.
 * tdb200_sla_project_moments  kvw [bh,d,d] T = T(proj_w [d,d] . kv [bh,d,d]): folds proj_l's weight (SLA/core.py:246
 *     `self.proj_l(o_l)`) into the moment matrix so the fused kernel applies it with its last MMA; fp32 FMA chain over d_v.
 * tdb200_sla_attn_fwd   o = T( sparse_softmax_attention(q_i8,k_i8,v; lut) + proj( phi(q) kv / (1e-5 + phi(q).ksum) ) )
 *     q_i8 / q_scale / k_scale as tdb200_sla_quant_qk made them, lut [b,h,mblk,topk] of blkk-row key blocks (1 <= topk <= nblk),
 *     kvw [b,h,d(out),d(k)] T = (proj_w . kv) so that proj is folded into the moment matrix, proj_b [d] fp32; `feature` is the
 *     map the moments were built with.  The int8 QK^T, online softmax (exp2), PV, linear branch and merge run in one wgmma
 *     kernel; with (64, 128) one CTA per 64-row query block runs two consumer warpgroups on alternate key blocks and merges
 *     their softmax states.  k_seq_major != 0 reads k_i8 in the sequence-major layout [1,lk,h,d] (rows past lk may follow);
 *     it is implemented for d = 128, the softmax map and b = 1, other calls return TDB200_ERR_UNSUPPORTED.
 *     Range: the linear branch enters as one more MMA whose 16-bit operand is A = phi(q) * l / den (l the unnormalised
 *     softmax row sum).  In fp16 a row whose max A lies outside [2^-6, 2^15) runs that MMA on A and the accumulator scaled by
 *     one power of two (and divides it out in the store), so dead relu channels (den = 1e-5), outlier channels and long
 *     peaked rows neither overflow nor go subnormal; other rows, and every bf16 call, are unchanged.  kvw itself must fit in T:
 *     proj_w . kv grows with l * E[phi(k)] * mean(v), and in fp16 it overflows first (for example relu at l = 75600 with a
 *     modest mean in v); the caller's T(proj_w . kv) is what the kernel multiplies.
 * ------------------------------------------------------------------------------------------- */
int tdb200_sla_quant_qk(const void* q, const void* k, int dtype, int64_t b, int64_t lq, int64_t lk, int64_t h, int64_t d,
                        float* kmean, int8_t* q_i8, float* q_scale, int8_t* k_i8, float* k_scale, void* q_pool,
                        void* k_pool, int64_t blkq, int64_t blkk, void* stream);
int tdb200_sla_block_map(const void* q_pool, const void* k_pool, int dtype, int64_t b, int64_t h, int64_t mblk,
                         int64_t nblk, int64_t d, int64_t topk, int8_t* sparse_map, int32_t* lut, void* stream);
int tdb200_sla_linear_moments(const void* k, const void* v, int dtype, int64_t b, int64_t l, int64_t h, int64_t d,
                              int feature, float* kv, float* ksum, void* stream);
int tdb200_sla_project_moments(const float* proj_w, const float* kv, int dtype, int64_t bh, int64_t d, void* kvw, void* stream);
int tdb200_sla_attn_fwd(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                        const void* v, const void* q, int dtype, const int32_t* lut, int64_t topk, const void* kvw,
                        const float* ksum, const float* proj_b, void* out, int64_t b, int64_t l, int64_t lk,
                        int64_t h, int64_t d, float sm_scale, int feature, int64_t blkq, int64_t blkk,
                        int k_seq_major, void* stream);
/* Per-entry lengths (the _vl twins; inference only, d = 128, lq = lk = l): a padded batch whose entry i owns its first
 * seq_lens[i] rows of q, k and v (seq_lens [b] device int32, clamped to [0, l] on the device).  Entry i's results over those
 * rows are the bits of the entry point without `_vl` called on entry i alone, cut to those rows: its own key mean, pooled means
 * and scales, its own mblk_i = ceil(n_i / blkq), nblk_i = ceil(n_i / blkk) and topks[i] blocks per row (device int32, clamped to
 * [1, min(nblk_i, topk)]), its own moments (the split count and summation order tdb200_sla_linear_moments picks for n_i rows),
 * and keys masked at n_i.  Output rows past n_i are 0; what q, k and v hold past n_i, inf and NaN included, reaches no result.
 * tdb200_sla_quant_qk_vl       one length for both halves; either half may be NULL as for tdb200_sla_quant_qk.  Rows past n_i
 *                              of the INT8 codes are not written; blocks wholly past n_i pool to 0.
 * tdb200_sla_block_map_vl      blkq, blkk: the block sizes of the pools.  LUT [b,h,mblk,topk] keeps the row stride `topk`, the
 *                              largest topks[i]; LUT entries past topks[i] and rows past mblk_i are -1, sparse_map is 0 there.
 * tdb200_sla_linear_moments_vl accumulated like tdb200_sla_linear_moments (the caller zeroes kv and ksum).
 * tdb200_sla_attn_fwd_vl       INT8 Q/K with head-major K, (blkq, blkk) = (128, 64) or (64, 128), 16-bit P.V.
 * tdb200_sla_attn16_fwd_vl     (blkq, blkk) = (128, 64) or (64, 64).
 * Errors as their twins; a null or misaligned seq_lens or topks is TDB200_ERR_INVALID_ARG, d != 128 TDB200_ERR_UNSUPPORTED,
 * l != lk (attention) TDB200_ERR_INVALID_ARG, all before any CUDA call. */
int tdb200_sla_quant_qk_vl(const void* q, const void* k, int dtype, int64_t b, int64_t l, int64_t h, int64_t d,
                           const int32_t* seq_lens, float* kmean, int8_t* q_i8, float* q_scale, int8_t* k_i8, float* k_scale,
                           void* q_pool, void* k_pool, int64_t blkq, int64_t blkk, void* stream);
int tdb200_sla_block_map_vl(const void* q_pool, const void* k_pool, int dtype, int64_t b, int64_t h, int64_t mblk, int64_t nblk,
                            int64_t d, int64_t topk, const int32_t* seq_lens, const int32_t* topks, int64_t blkq, int64_t blkk,
                            int8_t* sparse_map, int32_t* lut, void* stream);
int tdb200_sla_linear_moments_vl(const void* k, const void* v, int dtype, int64_t b, int64_t l, int64_t h, int64_t d,
                                 const int32_t* seq_lens, int feature, float* kv, float* ksum, void* stream);
int tdb200_sla_attn_fwd_vl(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                           const void* v, const void* q, int dtype, const int32_t* lut, int64_t topk, const void* kvw,
                           const float* ksum, const float* proj_b, void* out, int64_t b, int64_t l, int64_t lk, int64_t h,
                           int64_t d, const int32_t* seq_lens, const int32_t* topks, float sm_scale, int feature, int64_t blkq,
                           int64_t blkk, void* stream);
/* SageSLA with FP8 P.V (SageAttention2's arithmetic: e4m3 P and V, per-channel V scales), an option beside the 16-bit P.V of
 * tdb200_sla_attn_fwd; d = 128 only.
 * tdb200_sla_quant_v_fp8  v [b,l,h,d] 16-bit (`dtype`) -> v_scale [b,h,d] fp32 and v_fp8 [b,h,d,l_pad] e4m3 codes, l_pad =
 *     ceil(l / blkk) * blkk (blkk = 64 or 128, the key block of the attention call).  v_scale = max(amax over all l rows of the
 *     channel, 2^-64) / 448, an IEEE division; codes = e4m3(v / v_scale), IEEE division then round to nearest even, saturated to
 *     +-448 (what torch's float32 -> float8_e4m3fn cast gives for these values).  Keys l..l_pad-1 are zero codes.  Inside every
 *     32-key group the keys are stored permuted for the kernel's register fragment: position 16 u + 4 t + j holds key
 *     16 u + 8 (j >> 1) + 2 t + (j & 1).  A memset and three kernels on `stream`; the scales are order-independent (a max), so
 *     both outputs are bit-reproducible.
 * tdb200_sla_attn_fwd_fp8v  tdb200_sla_attn_fwd with `v` replaced by v_fp8 / v_scale from tdb200_sla_quant_v_fp8 over the lk keys
 *     with the same blkk.  P (fp32, unrounded, <= 2^8 under the lazy rescale) is rounded to e4m3 as the MMA operand with the
 *     scale 2^0; the row sum l is taken from the unrounded P as in tdb200_sla_attn_fwd.  Each key block's P.V is one chain of
 *     e4m3 x e4m3 wgmma (whose accumulation is narrower than fp32), added to O in fp32; the softmax part is O * v_scale[d] / l; the linear branch, its fp16 range scaling and the output store
 *     are tdb200_sla_attn_fwd's.  Both block families and k_seq_major as there.
 * Errors, all before any CUDA call: null pointer, non-positive b, l, lk, h or d, or (tdb200_sla_quant_v_fp8: any buffer,
 * tdb200_sla_attn_fwd_fp8v: v_fp8, v_scale) not 16-byte aligned -> TDB200_ERR_INVALID_ARG, as are a bad feature tag and topk
 * outside [1, nblk]; d != 128, block sizes other than (128, 64) and (64, 128) (blkk other than 64 and 128), a bad dtype tag,
 * b or h above 65535, sequence-major K with another feature map than softmax or b != 1 -> TDB200_ERR_UNSUPPORTED. */
int tdb200_sla_quant_v_fp8(const void* v, int dtype, int64_t b, int64_t l, int64_t h, int64_t d, int64_t blkk, uint8_t* v_fp8,
                           float* v_scale, void* stream);
int tdb200_sla_attn_fwd_fp8v(const int8_t* q_i8, const float* q_scale, const int8_t* k_i8, const float* k_scale,
                             const uint8_t* v_fp8, const float* v_scale, const void* q, int dtype, const int32_t* lut,
                             int64_t topk, const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b,
                             int64_t l, int64_t lk, int64_t h, int64_t d, float sm_scale, int feature, int64_t blkq,
                             int64_t blkk, int k_seq_major, void* stream);
/* SparseLinearAttention's linear branch and proj_l for training (reference SLA/core.py:104-117), per (batch, head), phi the
 * feature map `feature` (0 softmax over d, 1 elu+1, 2 relu), c = T(phi(x)), kv = M^T [b,h,d(v),d(k)] and ksum = s [b,h,d] fp32
 * from tdb200_sla_linear_moments of the same k, v and feature:
 *   tdb200_sla_linear_fwd   den_i = 1e-5 + c_q,i . s,  u_i = c_q,i M / den_i,  o_l,i = T(u_i proj_w^T + proj_b)
 *   tdb200_sla_linear_bwd   for d_o = dL/do_l: dq, dk, dv (T) and dproj_w [d,d], dproj_b [d] (fp32, summed over b, h and l) of
 *                           the forward above, from q, k, v, kv and ksum (nothing of l's size is saved by the forward)
 *   tdb200_sla_linear_bwd_workspace_bytes  host-only size of the backward's workspace (or a negative error code): three
 *                           [b,l,h,d] 16-bit operands, per-64-row partials of ds and dproj_b, split partials of dM and dproj_w,
 *                           dM and ds, each 256-byte aligned.
 *   tdb200_sla_linear_tangent  o_l_t = T(udot proj_w^T), the forward's tangent along q_t, k_t, v_t (proj_w, proj_b fixed):
 *                           Mdot = sum_j (cdot_k,j^T v_j + c_k,j^T v_t,j), sdot = sum_j cdot_k,j with cdot = J_phi . x_t,
 *                           udot_i = (cdot_q,i M + c_q,i Mdot) / den_i - u_i (cdot_q,i . s + c_q,i . sdot) / den_i.
 *                           J_phi: softmax c (x_t - c . x_t); elu+1 1 where x > 0, else e^x; relu 1[x > 0].  Five launches.
 *   tdb200_sla_linear_tangent_workspace_bytes  its workspace: c_k and cdot_k [b,l,h,d] 16-bit, per-64-row partials of sdot,
 *                           split partials of Mdot, Mdot and sdot, each 256-byte aligned.
 * q, k, v, d_o, o_l, dq, dk, dv [b,l,h,d] contiguous 16-bit of type `dtype`; proj_w [d(out),d(in)] and proj_b [d] fp32.
 * Rounding points: c_q and c_k to T; cdot (fp32) to T as MMA operands, sdot from the fp32 cdot; M, Mdot and dM (fp32) to
 * T as MMA operands after a power-of-two scale per (b, h) that puts their largest magnitude in [2^14, 2^15); udot,
 * proj_w, u, g and du to T as MMA operands; dM's row operands c_q,i 2^e and du_i/den_i 2^-e
 * to T with e splitting the two rows' exponents; everything else, den, e_i, s and ds included, fp32.  Products are 16-bit
 * tensor-core MMAs with fp32 accumulation.  Every reduction over rows, heads and batch entries is summed in a fixed order
 * without atomics: the results are bit-reproducible, and a (batch, head)'s o_l, dq, dk and dv depend only on its own inputs.
 * The forward is one launch, the backward eight, the tangent five; neither synchronises the host, so both can be captured in a CUDA graph.
 * Errors, all before any CUDA call: null or misaligned (16 B) pointer, non-positive b, l, h or d -> TDB200_ERR_INVALID_ARG;
 * d != 128, bad dtype or feature tag, b*h above 65535, l*h*d of 2^39 elements or more -> TDB200_ERR_UNSUPPORTED;
 * workspace_bytes below the size query -> TDB200_ERR_WORKSPACE. */
int tdb200_sla_linear_fwd(const void* q, const float* kv, const float* ksum, const float* proj_w, const float* proj_b, int dtype,
                          int feature, void* o_l, int64_t b, int64_t l, int64_t h, int64_t d, void* stream);
int tdb200_sla_linear_bwd(const void* q, const void* k, const void* v, const void* d_o, const float* kv, const float* ksum,
                          const float* proj_w, int dtype, int feature, void* dq, void* dk, void* dv, float* dproj_w,
                          float* dproj_b, void* workspace, int64_t workspace_bytes, int64_t b, int64_t l, int64_t h, int64_t d,
                          void* stream);
int64_t tdb200_sla_linear_bwd_workspace_bytes(int64_t b, int64_t h, int64_t l, int64_t d);
int tdb200_sla_linear_tangent(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                              const float* kv, const float* ksum, const float* proj_w, int dtype, int feature, void* o_l_t,
                              void* workspace, int64_t workspace_bytes, int64_t b, int64_t l, int64_t h, int64_t d, void* stream);
int64_t tdb200_sla_linear_tangent_workspace_bytes(int64_t b, int64_t h, int64_t l, int64_t d);
/* Sequence-parallel form of the key half of tdb200_sla_quant_qk (reference: the context-parallel attention of
 * rcm/utils/a2a_cp.py:66-182 exchanges 16-bit K; here each rank quantises its own key rows and the INT8 tensor travels).
 *   tdb200_sla_kmean_partial  partial [b,h,ceil(l/128),d] fp32 = column sums of each 128-row chunk of k [b,l,h,d];
 *   tdb200_sla_kmean_final    kmean [b,h,d] = (fixed-order sum of `chunks` partials) / l_total  -- the reduction
 *                             tdb200_sla_quant_qk runs, so gathering every rank's partials reproduces its mean bit for bit
 *                             (the 128-row partials serve both block families);
 *   tdb200_sla_quant_k_seq    smoothed Sage INT8 of k's rows per blkk rows, blkk = 64 or 128: k_i8 in the sequence-major
 *                             layout [b,l,h,d], k_scale [b,h,ceil(l/blkk)], k_pool [b,h,ceil(l/blkk),d]. */
int tdb200_sla_kmean_partial(const void* k, int dtype, int64_t b, int64_t l, int64_t h, int64_t d, float* partial, void* stream);
int tdb200_sla_kmean_final(const float* partial, int64_t b, int64_t h, int64_t chunks, int64_t d, int64_t l_total, float* kmean,
                           void* stream);
int tdb200_sla_quant_k_seq(const void* k, const float* kmean, int dtype, int64_t b, int64_t l, int64_t h, int64_t d,
                           int8_t* k_i8, float* k_scale, void* k_pool, int64_t blkk, void* stream);
/* ---------------------------------------------------------------------------------------------
 * a9'. The non-quantised SLA path (SparseLinearAttention, --attention_type sla; reference: the Triton _attn_fwd, its autograd
 * function `_attention` and its backward, turbodiffusion/SLA/kernel.py:21-319).  Q.K^T is a 16-bit tensor-core product on the
 * un-quantised q, k (fp32 scores, exp2 softmax, P rounded to T before P.V, :60-73); no q/k scales, no key smoothing.
 * d = 128; q, k, v, out, o_s, d_o, dq, dk, dv are [b, l, h, d] contiguous 16-bit; lut [b,h,mblk,topk] int32 of distinct
 * blkk-row key-block ids per row (1 <= topk <= nblk).
 * Block sizes (blkq, blkk): (128, 64), the configuration TurboDiffusion's modify_model.py requests, or (64, 64), the module's
 * default (the reference's BLOCK_M = 64 kernels); any other pair returns TDB200_ERR_UNSUPPORTED.  With (64, 64) one CTA per
 * 64-row query block runs two consumer warpgroups on alternate key blocks and merges their softmax states (forward) or adds
 * their dQ / dK / dV partials in a fixed order (backward).
 *   tdb200_sla_attn16_fwd      o = T( sparse_softmax_attention(q,k,v; lut) + proj( phi(q) kv / (1e-5 + phi(q).ksum) ) ), with
 *                              kvw, ksum, proj_b and `feature` as for tdb200_sla_attn_fwd (0 softmax, 1 elu+1, 2 relu), and
 *                              the same fp16 range of the linear-branch operand and limit on kvw.
 *   tdb200_sla_attn16_fwd_lse  o_s = T(the softmax part alone) (no linear branch, no proj_b; lk = l) and lse [b,h,l] fp32 =
 *                              m + log2(l) of the scores in the log2 domain (S * sm_scale * log2e): the training forward.
 *   tdb200_sla_attn16_bwd      dq, dk, dv of o_s w.r.t. q, k, v for the incoming gradient d_o, given the forward's o_s and lse.
 *                              P and dS are rounded to T only as MMA operands, accumulation is fp32, no atomics (bit-for-bit
 *                              reproducible); key blocks no query block selected get zero dk / dv.  Four kernel launches and
 *                              no host synchronisation, so the call can be captured in a CUDA graph.
 *   tdb200_sla_attn16_bwd_workspace_bytes  host-only size of the workspace the backward needs (or a negative error code):
 *                              delta [b,h,l] fp32, then the key-major index of the LUT: offsets [b*h, nblk+1], cursors
 *                              [b*h, nblk] and entries [b*h, mblk*topk] int32, each 256-byte aligned (mblk = ceil(l / blkq)).
 * Errors, all before any CUDA call: an unsupported block pair, d != 128 or a bad dtype tag -> TDB200_ERR_UNSUPPORTED; null pointer,
 * bad shape, bad feature tag or topk outside [1, nblk] -> TDB200_ERR_INVALID_ARG; workspace_bytes below the size query ->
 * TDB200_ERR_WORKSPACE.
 * The four older names below are the same operations at (blkq, blkk) = (128, 64) (and the softmax map for the fused forward):
 * each is one call of its general form, kept because existing callers link against them.
 * ------------------------------------------------------------------------------------------- */
int tdb200_sla_attn16_fwd(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
                          const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b, int64_t l, int64_t lk,
                          int64_t h, int64_t d, float sm_scale, int feature, int64_t blkq, int64_t blkk, void* stream);
/* tdb200_sla_attn16_fwd with per-entry lengths: see tdb200_sla_attn_fwd_vl above. */
int tdb200_sla_attn16_fwd_vl(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
                             const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b, int64_t l, int64_t lk,
                             int64_t h, int64_t d, const int32_t* seq_lens, const int32_t* topks, float sm_scale, int feature,
                             int64_t blkq, int64_t blkk, void* stream);
int tdb200_sla_attn16_fwd_lse(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk, void* o_s,
                              float* lse, int64_t b, int64_t l, int64_t h, int64_t d, float sm_scale, int64_t blkq, int64_t blkk,
                              void* stream);
int tdb200_sla_attn16_bwd(const void* q, const void* k, const void* v, const void* o_s, const void* d_o, const float* lse,
                          int dtype, const int32_t* lut, int64_t topk, void* dq, void* dk, void* dv, void* workspace,
                          int64_t workspace_bytes, int64_t b, int64_t l, int64_t h, int64_t d, float sm_scale, int64_t blkq,
                          int64_t blkk, void* stream);
int64_t tdb200_sla_attn16_bwd_workspace_bytes(int64_t b, int64_t h, int64_t l, int64_t topk, int64_t blkq);
int tdb200_sla_attn_fwd_qk16(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
                             const void* kvw, const float* ksum, const float* proj_b, void* out, int64_t b, int64_t l,
                             int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_sla_attn_fwd_qk16_lse(const void* q, const void* k, const void* v, int dtype, const int32_t* lut, int64_t topk,
                                 void* o_s, float* lse, int64_t b, int64_t l, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_sla_attn_bwd_qk16(const void* q, const void* k, const void* v, const void* o_s, const void* d_o, const float* lse,
                             int dtype, const int32_t* lut, int64_t topk, void* dq, void* dk, void* dv, void* workspace,
                             int64_t workspace_bytes, int64_t b, int64_t l, int64_t h, int64_t d, float sm_scale, void* stream);
int64_t tdb200_sla_attn_bwd_workspace_bytes(int64_t b, int64_t h, int64_t l, int64_t topk);

/* ---------------------------------------------------------------------------------------------
 * f1. Dense softmax attention, forward only: the block's cross-attention over the text tokens and `--attention_type original`
 * (reference: the `attention` wrapper over FlashAttention / F.scaled_dot_product_attention, turbodiffusion/rcm/utils/attention.py:120-167,
 * without its dropout, causal and window arguments, which the denoise path leaves at their defaults; its variable-length
 * arguments are the _kl (key lengths) and _vl (query and key lengths) twins below).
 *   out = T( softmax(q . k^T * sm_scale) . v )   per (batch, head)
 * q, out [b, lq, h, d] and k, v [b, lk, h, d], contiguous 16-bit of type `dtype`, 16-byte aligned, read and written in place
 * (row stride h*d: the [l, h*d] output of a projection GEMM is consumed as it is, no transposed copies).  lq and lk are
 * independent and need not be multiples of anything: key columns >= lk are masked to -inf and query rows >= lq are not stored.
 * Arithmetic, that of tdb200_sla_attn16_fwd's softmax part: S by wgmma into fp32, scores scaled by sm_scale * log2(e), online
 * softmax with exp2 over 128-key tiles in ascending order, the row sum from the unrounded P, P rounded to T as the operand of
 * P.V, fp32 accumulation, one rounding of O / l to T.  No atomics: the bits of a (batch, head) depend only on its own q, k, v.
 * d = 128 only (d = 64 returns TDB200_ERR_UNSUPPORTED).  One kernel launch, no host synchronisation (capturable in a CUDA graph).
 * Errors, all before any CUDA call: null or misaligned pointer, non-positive b, lq, lk, h or d -> TDB200_ERR_INVALID_ARG; bad
 * dtype tag, d != 128, b or h above 65535, lq*h*d or lk*h*d of 2^39 elements or more -> TDB200_ERR_UNSUPPORTED.
 * ------------------------------------------------------------------------------------------- */
int tdb200_attn_dense_fwd(const void* q, const void* k, const void* v, int dtype, void* out, int64_t b, int64_t lq, int64_t lk,
                          int64_t h, int64_t d, float sm_scale, void* stream);

/* ---------------------------------------------------------------------------------------------
 * f1 key lengths. Key-padding masks as per-sample key lengths (a batched text cross-attention whose prompts tokenise to different
 * lengths): each entry point of the f1 family has a twin, suffixed _kl, that takes k_lens right after lk and is otherwise the
 * same call.
 *   k_lens [b] int32, device memory, 4-byte aligned: batch entry i attends to keys 0 .. lk_i - 1 of its own [lk, h, d] slab,
 *   lk_i = min(max(k_lens[i], 0), lk).  The values are device data and are clamped by the kernels, never read by the host.
 * Batch entry i computes the bits the entry point without _kl computes on entry i alone with k and v (and k_t, v_t) cut to
 * their first lk_i rows: its key tiles past lk_i are neither loaded nor visited, columns >= lk_i are masked, and in the tile
 * that straddles lk_i the rows >= lk_i of k, v (and k_t, v_t) are zeroed in shared memory after the load, as the load's zero
 * fill past lk would be.  So what those rows hold in memory, inf and NaN included, never reaches a result.  An entry with lk_i = 0 has no keys: out = 0, out_t = 0 and lse = +inf (the
 * convention of rows >= lq), so its dq is 0.  The backward stores dk = dv = 0 in rows lk_i .. lk - 1.
 *   tdb200_attn_dense_fwd_kl, tdb200_attn_dense_fwd_lse_kl, tdb200_attn_dense_jvp_kl, tdb200_attn_dense_jvp_lse_kl,
 *   tdb200_attn_dense_tangent_kl, tdb200_attn_dense_bwd_kl (its workspace: tdb200_attn_dense_bwd_workspace_bytes).
 * Errors: those of the twin without _kl, plus k_lens null or not 4-byte aligned -> TDB200_ERR_INVALID_ARG, all before any CUDA
 * call.  Launches, synchronisation and graph capture as the twin without _kl.
 * ------------------------------------------------------------------------------------------- */
int tdb200_attn_dense_fwd_kl(const void* q, const void* k, const void* v, int dtype, void* out, int64_t b, int64_t lq, int64_t lk,
                             const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_fwd_lse_kl(const void* q, const void* k, const void* v, int dtype, void* out, float* lse, int64_t b,
                                 int64_t lq, int64_t lk, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_jvp_kl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                             int dtype, void* out, void* out_t, int64_t b, int64_t lq, int64_t lk, const int32_t* k_lens, int64_t h,
                             int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_jvp_lse_kl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                                 int dtype, void* out, void* out_t, float* lse, int64_t b, int64_t lq, int64_t lk,
                                 const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_tangent_kl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                                 const void* out, const float* lse, int dtype, void* out_t, int64_t b, int64_t lq, int64_t lk,
                                 const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_bwd_kl(const void* q, const void* k, const void* v, const void* out, const void* d_out, const float* lse,
                             int dtype, void* dq, void* dk, void* dv, void* workspace, int64_t workspace_bytes, int64_t b, int64_t lq,
                             int64_t lk, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream);

/* ---------------------------------------------------------------------------------------------
 * f1 query lengths. Self-attention over a padded batch (clips of different token counts packed to one lq, queries and keys both
 * padded): each entry point of the f1 family has a twin, suffixed _vl (variable length), that takes q_lens and k_lens right after
 * lk and is otherwise the same call.  Both are required: self-attention passes the same pointer twice, and a caller with query
 * lengths only passes k_lens filled with lk.
 *   q_lens [b] int32, device memory, 4-byte aligned: batch entry i owns query rows 0 .. lq_i - 1 of its own [lq, h, d] slab,
 *   lq_i = min(max(q_lens[i], 0), lq).  k_lens as for the _kl twins.  The values are device data, clamped by the kernels and
 *   never read by the host.
 * Batch entry i's results in rows < lq_i are bit-identical to the entry point without lengths called on entry i alone with q (and
 * q_t, out and d_out where the call reads them) cut to its first lq_i rows and k, v (and k_t, v_t) cut to their first lk_i rows;
 * dk and dv of entry i are bit-identical to that trimmed call's.  Rows lq_i .. lq - 1 store out = 0, out_t = 0, dq = 0 and
 * lse = +inf (the convention of rows >= lq), and contribute nothing to dk and dv; an entry with lq_i = 0 also gets dk = dv = 0.
 * What the rows past lq_i of q, q_t, out and d_out hold, inf and NaN included, never reaches an output: query tiles wholly past
 * lq_i are neither loaded nor visited (their CTAs store the zero rows and exit, in the forward, JVP, tangent and dQ kernels; the
 * dK/dV kernel walks only the query blocks below lq_i), the dK/dV kernel zeroes the straddling block's Q and dO rows past lq_i on
 * chip after the load and stages their lse / delta as +inf / 0, and the delta kernel writes delta = 0 for them without reading.
 *   tdb200_attn_dense_fwd_vl, tdb200_attn_dense_fwd_lse_vl, tdb200_attn_dense_jvp_vl, tdb200_attn_dense_jvp_lse_vl,
 *   tdb200_attn_dense_tangent_vl, tdb200_attn_dense_bwd_vl (its workspace: tdb200_attn_dense_bwd_workspace_bytes).
 * Errors: those of the _kl twin, plus q_lens null or not 4-byte aligned -> TDB200_ERR_INVALID_ARG, all before any CUDA call.
 * Launches, synchronisation and graph capture as the twin without _vl.
 * ------------------------------------------------------------------------------------------- */
int tdb200_attn_dense_fwd_vl(const void* q, const void* k, const void* v, int dtype, void* out, int64_t b, int64_t lq, int64_t lk,
                             const int32_t* q_lens, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_fwd_lse_vl(const void* q, const void* k, const void* v, int dtype, void* out, float* lse, int64_t b,
                                 int64_t lq, int64_t lk, const int32_t* q_lens, const int32_t* k_lens, int64_t h, int64_t d,
                                 float sm_scale, void* stream);
int tdb200_attn_dense_jvp_vl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                             int dtype, void* out, void* out_t, int64_t b, int64_t lq, int64_t lk, const int32_t* q_lens,
                             const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_jvp_lse_vl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                                 int dtype, void* out, void* out_t, float* lse, int64_t b, int64_t lq, int64_t lk,
                                 const int32_t* q_lens, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_tangent_vl(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                                 const void* out, const float* lse, int dtype, void* out_t, int64_t b, int64_t lq, int64_t lk,
                                 const int32_t* q_lens, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_bwd_vl(const void* q, const void* k, const void* v, const void* out, const void* d_out, const float* lse,
                             int dtype, void* dq, void* dk, void* dv, void* workspace, int64_t workspace_bytes, int64_t b, int64_t lq,
                             int64_t lk, const int32_t* q_lens, const int32_t* k_lens, int64_t h, int64_t d, float sm_scale,
                             void* stream);

/* ---------------------------------------------------------------------------------------------
 * f1 JVP. Forward-mode derivative of the dense attention above (rCM distillation's tangent pass, reference
 * turbodiffusion/rcm/networks/wan2pt1_jvp.py): the attention output and its tangent for tangents q_t, k_t, v_t, in one kernel.
 *   S = sm_scale q.k^T,  S_t = sm_scale (q_t.k^T + q.k_t^T),  P = softmax(S),  out = T(P.v)
 *   out_t = T( sum_j P_j S_t,j v_j - (sum_j P_j S_t,j) out + P.v_t )   per (batch, head) and query row
 * q, q_t, out, out_t [b, lq, h, d] and k, v, k_t, v_t [b, lk, h, d], contiguous 16-bit of type `dtype` (tangents included),
 * 16-byte aligned, read and written in place; key columns >= lk are masked and query rows >= lq are stored to neither output.
 * Arithmetic: the online softmax of tdb200_attn_dense_fwd over 64-key tiles, with two more accumulators per row,
 * A = sum p (S_t v + v_t) and mu = sum p S_t, rescaled with O and l; l and mu sum the unrounded p and p S_t, the tensor core
 * gets p and p S_t rounded to T; out = T(O / l), out_t = T((A - (mu / l) O) / l).  No atomics: the bits of a (batch, head)
 * depend only on its own inputs.  d = 128 only.  One kernel launch, no workspace, no host synchronisation.
 * Errors, all before any CUDA call: any of the eight pointers null or misaligned, non-positive b, lq, lk, h or d ->
 * TDB200_ERR_INVALID_ARG; bad dtype tag, d != 128, b or h above 65535, lq*h*d or lk*h*d of 2^39 elements or more ->
 * TDB200_ERR_UNSUPPORTED.
 * ------------------------------------------------------------------------------------------- */
int tdb200_attn_dense_jvp(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                          int dtype, void* out, void* out_t, int64_t b, int64_t lq, int64_t lk, int64_t h, int64_t d,
                          float sm_scale, void* stream);

/* ---------------------------------------------------------------------------------------------
 * f1 backward. Gradients of the dense attention above, for training through tdb200_attn_dense_fwd or the primal output of
 * tdb200_attn_dense_jvp (rCM / sCM distillation differentiates through out; out_t is a stop-gradient target).
 *   tdb200_attn_dense_fwd_lse  tdb200_attn_dense_fwd, plus lse [b, h, lq] fp32 = m + log2(l): the row log-sum-exp of the scores
 *                              in the log2 domain (S * sm_scale * log2e), m the row maximum the lazy rescale last used.
 *   tdb200_attn_dense_jvp_lse  tdb200_attn_dense_jvp, plus the same lse of the primal.
 *                              out (and out_t) are bit-identical to those of the entry points without lse: the arithmetic is
 *                              the same, only the store of lse is added.  Argument checks as theirs, plus lse null or not
 *                              4-byte aligned -> TDB200_ERR_INVALID_ARG.
 *   tdb200_attn_dense_bwd      dq [b, lq, h, d], dk and dv [b, lk, h, d] of out for the incoming gradient d_out [b, lq, h, d],
 *                              given q, k, v, the forward's out and lse.  FlashAttention-2's backward on 128-row query and
 *                              64-row key tiles: P = exp2(S * sm_scale * log2e - lse) and dS = P o (dO.V^T - delta) with
 *                              delta = rowsum(dO o out) in fp32, rounded to T only as MMA operands; fp32 accumulation, dq, dk
 *                              and dv rounded to T once.  Key columns >= lk are masked; rows >= lq of dq and rows >= lk of dk
 *                              and dv are not written.  No atomics: every output row is written by one thread in a fixed
 *                              order, so the gradients are bit-for-bit reproducible.  Three kernel launches (delta, dq,
 *                              dk/dv), no host synchronisation, so the call can be captured in a CUDA graph.
 *   tdb200_attn_dense_bwd_workspace_bytes  host-only size of the workspace the backward needs, delta [b, h, lq] fp32 (or a
 *                              negative error code: non-positive sizes -> TDB200_ERR_INVALID_ARG, sizes past the limits
 *                              below -> TDB200_ERR_UNSUPPORTED).
 * All tensors contiguous 16-bit of type `dtype` except lse (fp32); d = 128 only.
 * Errors of tdb200_attn_dense_bwd, all before any CUDA call: any pointer null, q, k, v, out, d_out, dq, dk or dv not 16-byte
 * aligned, lse or workspace not 4-byte aligned, non-positive b, lq, lk, h or d -> TDB200_ERR_INVALID_ARG; bad dtype tag,
 * d != 128, b or h above 65535, lq*h*d or lk*h*d of 2^39 elements or more, or b*lq*h above 8 * (2^31 - 1) rows (the delta
 * kernel's grid: a tighter limit than the forward's) -> TDB200_ERR_UNSUPPORTED; workspace_bytes below the size query ->
 * TDB200_ERR_WORKSPACE.
 * ------------------------------------------------------------------------------------------- */
int tdb200_attn_dense_fwd_lse(const void* q, const void* k, const void* v, int dtype, void* out, float* lse, int64_t b, int64_t lq,
                              int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_jvp_lse(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                              int dtype, void* out, void* out_t, float* lse, int64_t b, int64_t lq, int64_t lk, int64_t h,
                              int64_t d, float sm_scale, void* stream);
int tdb200_attn_dense_bwd(const void* q, const void* k, const void* v, const void* out, const void* d_out, const float* lse,
                          int dtype, void* dq, void* dk, void* dv, void* workspace, int64_t workspace_bytes, int64_t b, int64_t lq,
                          int64_t lk, int64_t h, int64_t d, float sm_scale, void* stream);
int64_t tdb200_attn_dense_bwd_workspace_bytes(int64_t b, int64_t h, int64_t lq);

/* ---------------------------------------------------------------------------------------------
 * a9' JVP. Forward-mode derivative of the sparse softmax branch of a9' (SparseLinearAttention.forward_jvp, the tangent pass of
 * rCM / sCM distillation through sparse attention): the f1 JVP restricted to the key blocks lut[b, h, m, :] lists.
 *   o_s   = T( softmax over the listed keys of S ) . v                      (tdb200_sla_attn16_fwd_lse's o_s: no linear branch)
 *   o_s_t = T( sum_j P_j S_t,j v_j - (sum_j P_j S_t,j) o_s + P.v_t )          j over the listed keys, S_t as for f1 JVP
 * q, k, v, their tangents, o_s and o_s_t [b, l, h, d] contiguous 16-bit of type `dtype`, 16-byte aligned, read and written in
 * place; lut [b, h, ceil(l / blkq), topk] int32 of distinct key-block ids (1 <= topk <= nblk = ceil(l / blkk)), 4-byte aligned.
 * (blkq, blkk) = (128, 64) only: the f1 JVP kernel's 128-row query block over 64-key tiles, its tile ids read from the LUT in list
 * order.  Keys >= l are masked, rows >= l are stored to neither output.  The arithmetic is tdb200_attn_dense_jvp's, step for step,
 * so on an ascending LUT listing every key block the outputs are its bits.  d = 128.  One kernel launch, no workspace, no host
 * synchronisation; no atomics, so the bits of a (batch, head) depend only on its own inputs.
 *   tdb200_sla_attn16_jvp_lse  also lse [b, h, l] fp32 = m + log2(l) in log2 units, the convention tdb200_sla_attn16_bwd reads,
 *                              so the gradient of o_s goes through the existing SLA backward.
 * Errors, all before any CUDA call: (blkq, blkk) other than (128, 64) -> TDB200_ERR_UNSUPPORTED ((64, 64) included: its CTA holds
 * one 64-row query block); any pointer null, a 16-bit tensor not 16-byte aligned, lut or lse not 4-byte aligned, non-positive b,
 * l, h or d, topk outside [1, nblk] -> TDB200_ERR_INVALID_ARG; bad dtype tag, d != 128, the size limits of f1, topk above 8640
 * (the LUT row is staged in shared memory) -> TDB200_ERR_UNSUPPORTED.
 * ------------------------------------------------------------------------------------------- */
int tdb200_sla_attn16_jvp(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                          int dtype, const int32_t* lut, int64_t topk, void* o_s, void* o_s_t, int64_t b, int64_t l, int64_t h,
                          int64_t d, float sm_scale, int64_t blkq, int64_t blkk, void* stream);
int tdb200_sla_attn16_jvp_lse(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                              int dtype, const int32_t* lut, int64_t topk, void* o_s, void* o_s_t, float* lse, int64_t b, int64_t l,
                              int64_t h, int64_t d, float sm_scale, int64_t blkq, int64_t blkk, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Tangents alone, from a saved primal: the forward-mode rules of ops.dense_attention and SparseLinearAttention.forward
 * (torch.func.jvp / torch.autograd.forward_ad), whose primal the lse forward has already computed.
 *   tdb200_attn_dense_tangent  out_t of f1 JVP for tangents q_t, k_t, v_t, given out and lse of tdb200_attn_dense_fwd_lse on the
 *                              same q, k, v.  Shapes, layouts and argument checks as tdb200_attn_dense_jvp_lse, with out and lse
 *                              read instead of written.
 *   tdb200_sla_attn16_tangent  o_s_t of a9' JVP over the same lut, given o_s and lse of tdb200_sla_attn16_fwd_lse (blkq = 128).
 *                              Shapes, layouts and argument checks as tdb200_sla_attn16_jvp_lse, with o_s and lse read.
 * lse [b, h, lq] is the log2-domain row log-sum-exp, so P = exp2(S * sm_scale * log2e - lse) is the softmax without an online
 * pass or a rescale:
 *   out_t = T( (P o S_t).v + P.v_t - rowsum(P o S_t) out ),   S_t = sm_scale (q_t.k^T + q.k_t^T)
 * The tensor core gets P and P o S_t rounded to T; the row sum is of the unrounded P o S_t; the last term reads the rounded out.
 * f1 JVP's CTA and rings, 64-key tiles, keys >= lk masked; rows >= lq read no lse and are not stored.  No atomics, one kernel
 * launch, no workspace, no host synchronisation.
 * ------------------------------------------------------------------------------------------- */
int tdb200_attn_dense_tangent(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                              const void* out, const float* lse, int dtype, void* out_t, int64_t b, int64_t lq, int64_t lk,
                              int64_t h, int64_t d, float sm_scale, void* stream);
int tdb200_sla_attn16_tangent(const void* q, const void* k, const void* v, const void* q_t, const void* k_t, const void* v_t,
                              const void* o_s, const float* lse, int dtype, const int32_t* lut, int64_t topk, void* o_s_t, int64_t b,
                              int64_t l, int64_t h, int64_t d, float sm_scale, int64_t blkq, int64_t blkk, void* stream);

/* ---------------------------------------------------------------------------------------------
 * a12. LTX-2 (TurboT2AV) prologue variants   (ltx_core/model/transformer/transformer.py:21-94; Triton fast path
 *      ltx_distillation/fast_norm_kernels.py:388-473).  x, y, residual [b, tokens, n] 16-bit; table [num_ada, n] fp32;
 *      timestep [b, ts_tokens, num_ada*n] 16-bit with ts_tokens in {1, tokens}; ada value i = table[i] + timestep[.., i, :].
 *      fp32 math, one rounding to the io dtype.
 *   modulated_rms_norm_ada:  y = rms_norm(x, eps) * (1 + ada[scale_index]) + ada[shift_index]
 *   modulate_ada:            y = x * (1 + ada[scale_index]) + ada[shift_index]
 *   gated_residual_ada:      y = x + residual * ada[gate_index]
 *   split_rope:              x [b,t,h,d], cos/sin [b,h,t,d/2]:  y[:d/2] = x1*cos - x2*sin,  y[d/2:] = x2*cos + x1*sin
 *                            (ltx_core/model/transformer/rope.py:42-60)
 * ------------------------------------------------------------------------------------------- */
int tdb200_ltx_modulated_rms_norm_ada(const void* x, int dtype, const float* table, const void* timestep, int scale_index,
                                      int shift_index, int num_ada, void* y, int64_t b, int64_t tokens, int64_t ts_tokens,
                                      int64_t n, float eps, void* stream);
int tdb200_ltx_modulate_ada(const void* x, int dtype, const float* table, const void* timestep, int scale_index,
                            int shift_index, int num_ada, void* y, int64_t b, int64_t tokens, int64_t ts_tokens, int64_t n,
                            void* stream);
int tdb200_ltx_gated_residual_ada(const void* x, const void* residual, int dtype, const float* table, const void* timestep,
                                  int gate_index, int num_ada, void* y, int64_t b, int64_t tokens, int64_t ts_tokens,
                                  int64_t n, void* stream);
int tdb200_ltx_split_rope(const void* x, const void* cos_freqs, const void* sin_freqs, int dtype, void* y, int64_t b,
                          int64_t t, int64_t h, int64_t d, void* stream);

/* LTX-2 W8A8 with per-row post-scale (ltx_distillation/tilelang_w8a8.py:16-36, 78-117):
 *   quant_int8_rowwise: x [m,k] 16-bit -> q int8 [m,k], s [m] fp32; scale = max(amax,1e-4)/127, round half away, clip.
 *                       (IEEE division here; the reference's Triton `/` is div.full.f32, so exact .5 ties may differ)
 *   gemm_w8a8_rowwise:  c[i,j] = T( fma( float(sum_k a_q[i,k]*b_q[j,k]) * a_s[i], b_s[j], bias[j] ) ) -- the arithmetic the
 *                       reference's TileLang epilogue executes (I2FP, FMUL, FFMA under nvcc's default -fmad; see
 *                       tools/tilelang_epilogue_probe.py); int32 accumulation over all of K in registers, one epilogue per
 *                       tile (no per-K-block dequant).  bias may be NULL (= 0).  k % 128 == 0, n % 8 == 0. */
int tdb200_quant_int8_rowwise(const void* x, int dtype, int64_t m, int64_t k, int8_t* q, float* s, void* stream);
int tdb200_gemm_w8a8_rowwise(const int8_t* a_q, const float* a_s, const int8_t* b_q, const float* b_s, const void* bias,
                             void* c, int c_dtype, int64_t m, int64_t n, int64_t k, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TDB200_H_ */
