/*
 * pww_b200.h -- C ABI of the H100-native Paint-with-Words attention path (libpww_b200.so).
 *
 * The reference (cloneofsimo/paint-with-words-sd) has no FFI: its boundary is the Python callable
 * `inj_forward(self, hidden_states, context=None, mask=None)` that it monkey-patches over
 * diffusers' `CrossAttention.__call__` (paint_with_words/paint_with_words.py:60-125, 193-195).
 * These entry points replace the region of that function BETWEEN the q/k/v projections and the
 * output projection (paint_with_words.py:83-118); the Python shim
 * `paint_with_words_sd_b200.attention.inj_forward` keeps the reference calling convention and calls
 * them through ctypes (INTEGRATION.md shows the binding).
 *
 * Conventions: plain pointers and sizes, no torch types.  Every pointer is a DEVICE pointer owned by
 * the caller.  Calls enqueue work on `stream` (a cudaStream_t passed as void*) and return without
 * synchronising; they allocate nothing and are CUDA-graph capturable.  Return value: PWW_OK (0) or a
 * negative pww_status_t; nothing throws.  Unsupported (D, T) combinations return
 * PWW_ERR_UNSUPPORTED -- there is no fallback path inside or outside the library.
 *
 * Element types: every activation entry point exists as an `_f16` (IEEE binary16) and a `_bf16` (bfloat16) twin with
 * the same arguments, validation and return codes; q, k, v, out, x, y, ... are of the twin's type.  Everything else
 * keeps its type in both: weight maps, statistics and G(sigma) are fp32, the packed map `mpack` is fp16 (it is a
 * host-built encoding of the fp32 map, not an activation) and `cidx` is int8.
 *
 * Tensor layouts (elem = fp16 or bf16):
 *   q, out : [B, N, H*D] elem, element (b,n,h,d) at  b*q_batch_stride + n*q_row_stride + h*D + d
 *   k, v   : [B, T, H*D] elem, element (b,t,h,d) at  b*k_batch_stride + t*k_row_stride + h*D + d
 *            (strides in ELEMENTS; the head slice of a row is contiguous -- no head permute/copy,
 *             unlike paint_with_words.py:83-85,118)
 *   wmap   : [Bw, N, T] fp32 dense weight maps, the reference's CROSS_ATTENTION_WEIGHT_{N} tensors
 *            (paint_with_words.py:255-268, 370-377) stacked along dim 0
 *   wmap_index : [B] int32, image b uses wmap[wmap_index[b]]; -1 = no bias for that image (the
 *            reference's uncond dict / tensor context, paint_with_words.py:107-110, 379-386, 493)
 *
 * Key lengths: T <= 80 (Stable Diffusion's 77-token context), or a long prompt of k = 2 or 3 CLIP chunks
 * concatenated along tokens (T = 154 or 231; each chunk is [BOS] + up to 75 tokens + [EOS] + padding, encoded
 * on its own).  Any other T returns PWW_ERR_UNSUPPORTED.  Workspace sizes do not depend on T.
 */
#ifndef PWW_B200_H_
#define PWW_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  PWW_OK = 0,
  PWW_ERR_BAD_ARG = -1,      /* null pointer, non-positive size, misaligned pointer/stride        */
  PWW_ERR_UNSUPPORTED = -2,  /* (D, T, H) outside the compiled kernel family                        */
  PWW_ERR_CUDA = -3,         /* a CUDA runtime/driver call failed; see pww_last_cuda_error()        */
  PWW_ERR_WORKSPACE = -4     /* workspace_bytes smaller than pww_xattn_workspace_bytes()            */
} pww_status_t;

#define PWW_STAT_MAX 0 /* qk.max()                       (paint_with_words.py:405) */
#define PWW_STAT_STD 1 /* qk.std(), unbiased (Bessel)    (README.md:129-152)       */

/* Library version: major*10000 + minor*100 + patch. */
int pww_version(void);

/* Static string for a status code. */
const char* pww_status_str(int status);

/* cudaGetErrorString of the last CUDA failure seen by this library on the calling thread ("" if none). */
const char* pww_last_cuda_error(void);

/* 1 if the running device is compute capability 9.x (H100, the only target), 0 otherwise, <0 on error. */
int pww_device_supported(void);

/* Bytes of scratch `pww_xattn_stats_f16` needs for this problem size.  The scratch must be zero-filled
 * ONCE after allocation (cudaMemset); calls leave it zeroed again (self-cleaning arrival counters). */
size_t pww_xattn_workspace_bytes(int B, int H, int N, int T, int D);

/*
 * Per-image statistic of the UNSCALED score tensor S[b] = Q_h K_h^T over all heads, pixels and tokens
 * (one scalar per image per call -- what `qk.max()` / `qk.std()` evaluate to inside the reference's
 * weight_function, paint_with_words.py:87,106,402-405).  S is rounded to the element type before the std sums, as
 * the reference's autocast matmul does; the maximum is taken over S and rounded once (rounding is monotonic); the
 * result is rounded to the element type and stored as float.  For bf16 this is what qk.max() / qk.std() return when the
 * reference's op sequence runs under a bf16 autocast; bf16 has fp32's exponent range, so a statistic above 65504
 * (inf in fp16) stays finite.
 * _bf16: the same with bf16 q / k.
 * Images with wmap_index[b] < 0 are skipped (stats[b] = 0).  wmap_index may be NULL (= all images).
 */
int pww_xattn_stats_f16(const void* q, const void* k,
                        int B, int H, int N, int T, int D,
                        int64_t q_batch_stride, int64_t q_row_stride,
                        int64_t k_batch_stride, int64_t k_row_stride,
                        int stat, const int32_t* wmap_index,
                        float* stats /* [B] out */,
                        void* workspace, size_t workspace_bytes, void* stream);
int pww_xattn_stats_bf16(const void* q, const void* k,
                         int B, int H, int N, int T, int D,
                         int64_t q_batch_stride, int64_t q_row_stride,
                         int64_t k_batch_stride, int64_t k_row_stride,
                         int stat, const int32_t* wmap_index,
                         float* stats /* [B] out */,
                         void* workspace, size_t workspace_bytes, void* stream);

/*
 * Fused cross-attention with the Paint-with-Words bias (paint_with_words.py:87-118):
 *   P[b,h,n,:] = softmax_t( scale * ( S[b,h,n,t] + g_sigma[0] * stats[b] * wmap[wmap_index[b]][n,t] ) )
 *   out[b,n,h,:] = sum_t P[b,h,n,t] * V[b,t,h,:]
 * `g_sigma` is a 1-element device array holding G(sigma) = coef*ln(1+sigma^p) for this step (a device
 * scalar so a captured CUDA graph can be replayed with a new sigma).  wmap/wmap_index/stats/g_sigma may
 * all be NULL: plain cross-attention (tensor context, paint_with_words.py:67-69,107-108).
 * Requires T <= 80 or T = 154 / 231 (see "Key lengths" above; wmap stays [Bw, N, T], no padding columns).
 * P is rounded to the element type before P.V and the row sum is the sum of the rounded P; out is stored in it.
 */
int pww_xattn_fwd_f16(const void* q, const void* k, const void* v, void* out,
                      int B, int H, int N, int T, int D,
                      int64_t q_batch_stride, int64_t q_row_stride,
                      int64_t k_batch_stride, int64_t k_row_stride,
                      int64_t o_batch_stride, int64_t o_row_stride,
                      const float* wmap, int64_t wmap_batch_stride, const int32_t* wmap_index,
                      const float* stats, const float* g_sigma, float scale, void* stream);
int pww_xattn_fwd_bf16(const void* q, const void* k, const void* v, void* out,
                       int B, int H, int N, int T, int D,
                       int64_t q_batch_stride, int64_t q_row_stride,
                       int64_t k_batch_stride, int64_t k_row_stride,
                       int64_t o_batch_stride, int64_t o_row_stride,
                       const float* wmap, int64_t wmap_batch_stride, const int32_t* wmap_index,
                       const float* stats, const float* g_sigma, float scale, void* stream);

/*
 * ONE-LAUNCH Paint-with-Words cross-attention: statistic + bias + softmax + P.V (paint_with_words.py:87-118 with the
 * weight function of paint_with_words.py:402-405 inlined).  Replaces the pww_xattn_stats_f16 + pww_xattn_fwd_f16 pair:
 * the per-image statistic is reduced inside the kernel (cooperative launch, deterministic fixed-order reduction of
 * per-CTA partials) and the bias is rebuilt from the packed map in shared memory.
 *
 * The weight map is passed in PACKED form (SURVEY 8f-4).  The reference's dense [N, T] fp32 map
 * (paint_with_words.py:255-272) has one distinct non-zero column per painted region, so it is a column dictionary
 *     W[n, t] = Mu[n, cidx[t]]       Mu [N, R] fp32, R <= 10 distinct columns; cidx[t] = -1 for an all-zero column
 *   mpack : [Bw, N, 32] fp16, row n = [ hi(Mu[n,0..9]) | lo(Mu[n,0..9]) | hi(Mu[n,0..9]) | 0 0 ] with
 *           hi(x) = fp16(x), lo(x) = fp16(x - hi(x));  64 bytes per pixel instead of 308
 *           (element (w,n,c) at w*mpack_batch_stride + n*32 + c; 16-byte aligned)
 *   cidx  : [Bw, 80 k] int8, k = 1 for T <= 80, else T / 77: dictionary column (0..9) or -1 of token 77 c + j at
 *           column 80 c + j (for k = 1: token t at column t, -1 for t >= T; for k > 1 the columns 80 c + 77 .. 80 c + 79
 *           of every chunk are -1)
 * `paint_with_words_sd_b200.conditioning.pack_weight_map` builds both, bit-exactly reversible to the dense map.
 * Maps with more than 10 distinct columns use the two-launch dense path above.
 *
 *   stats [B] out : the per-image statistic (rounded to the element type as for pww_xattn_stats_f16 / _bf16, as
 *                   float; 0 for images without a map); may be NULL
 *   workspace     : pww_xattn_fused_workspace_bytes() bytes, zero-filled ONCE after allocation (self-cleaning)
 * mpack == NULL (or every wmap_index[b] < 0): plain cross-attention, workspace may be NULL.
 * Requires T <= 80 or T = 154 / 231, B <= 32 per launch (larger batches are split internally), 16-byte aligned `out`
 * strides.  _bf16: bf16 q / k / v / out; mpack stays fp16.
 */
size_t pww_xattn_fused_workspace_bytes(void);
int pww_xattn_fused_f16(const void* q, const void* k, const void* v, void* out,
                        int B, int H, int N, int T, int D,
                        int64_t q_batch_stride, int64_t q_row_stride,
                        int64_t k_batch_stride, int64_t k_row_stride,
                        int64_t o_batch_stride, int64_t o_row_stride,
                        const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
                        const int32_t* wmap_index, int stat, const float* g_sigma, float scale,
                        float* stats, void* workspace, size_t workspace_bytes, void* stream);
int pww_xattn_fused_bf16(const void* q, const void* k, const void* v, void* out,
                         int B, int H, int N, int T, int D,
                         int64_t q_batch_stride, int64_t q_row_stride,
                         int64_t k_batch_stride, int64_t k_row_stride,
                         int64_t o_batch_stride, int64_t o_row_stride,
                         const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
                         const int32_t* wmap_index, int stat, const float* g_sigma, float scale,
                         float* stats, void* workspace, size_t workspace_bytes, void* stream);

/*
 * Per-image settings: the three calls above with a statistic kind and a G(sigma) for EACH image, so one launch serves a
 * batch of images made with different weight functions (max / std, different strengths or sigma exponents).  Same
 * arguments and rules as the twin without `_multi` (key lengths, head dims, batch splits, workspace), except:
 *   stat    : [B] int32 device array instead of one int; entry b is image b's kind.  PWW_STAT_STD means std, any
 *             other value means max.
 *   g_sigma : [B] fp32 device array instead of one element; entry b is image b's G(sigma).
 * Entry b belongs to image b of the call; entries of images with wmap_index[b] < 0 are ignored.  A NULL `stat` or
 * `g_sigma` array where a map is given returns PWW_ERR_BAD_ARG (pww_xattn_stats_multi_f16 always needs `stat`).
 * With every kind equal and every G equal, the results are bit-identical to the twin's.  The _multi_bf16 calls are the
 * same with bf16 activations.
 */
int pww_xattn_stats_multi_f16(const void* q, const void* k,
                              int B, int H, int N, int T, int D,
                              int64_t q_batch_stride, int64_t q_row_stride,
                              int64_t k_batch_stride, int64_t k_row_stride,
                              const int32_t* stat, const int32_t* wmap_index,
                              float* stats /* [B] out */,
                              void* workspace, size_t workspace_bytes, void* stream);
int pww_xattn_fwd_multi_f16(const void* q, const void* k, const void* v, void* out,
                            int B, int H, int N, int T, int D,
                            int64_t q_batch_stride, int64_t q_row_stride,
                            int64_t k_batch_stride, int64_t k_row_stride,
                            int64_t o_batch_stride, int64_t o_row_stride,
                            const float* wmap, int64_t wmap_batch_stride, const int32_t* wmap_index,
                            const float* stats, const float* g_sigma, float scale, void* stream);
int pww_xattn_fused_multi_f16(const void* q, const void* k, const void* v, void* out,
                              int B, int H, int N, int T, int D,
                              int64_t q_batch_stride, int64_t q_row_stride,
                              int64_t k_batch_stride, int64_t k_row_stride,
                              int64_t o_batch_stride, int64_t o_row_stride,
                              const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
                              const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale,
                              float* stats, void* workspace, size_t workspace_bytes, void* stream);
int pww_xattn_stats_multi_bf16(const void* q, const void* k,
                               int B, int H, int N, int T, int D,
                               int64_t q_batch_stride, int64_t q_row_stride,
                               int64_t k_batch_stride, int64_t k_row_stride,
                               const int32_t* stat, const int32_t* wmap_index,
                               float* stats /* [B] out */,
                               void* workspace, size_t workspace_bytes, void* stream);
int pww_xattn_fwd_multi_bf16(const void* q, const void* k, const void* v, void* out,
                             int B, int H, int N, int T, int D,
                             int64_t q_batch_stride, int64_t q_row_stride,
                             int64_t k_batch_stride, int64_t k_row_stride,
                             int64_t o_batch_stride, int64_t o_row_stride,
                             const float* wmap, int64_t wmap_batch_stride, const int32_t* wmap_index,
                             const float* stats, const float* g_sigma, float scale, void* stream);
int pww_xattn_fused_multi_bf16(const void* q, const void* k, const void* v, void* out,
                               int B, int H, int N, int T, int D,
                               int64_t q_batch_stride, int64_t q_row_stride,
                               int64_t k_batch_stride, int64_t k_row_stride,
                               int64_t o_batch_stride, int64_t o_row_stride,
                               const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
                               const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale,
                               float* stats, void* workspace, size_t workspace_bytes, void* stream);

/*
 * Attention recording: pww_xattn_fused_multi_f16 / _bf16 that also ACCUMULATES, for every recorded image, head and
 * query row, the softmax mass each painted region's tokens receive.  `out` (and `stats`) are bit-identical to the
 * _multi call's on the same inputs.  Extra arguments, after `stream`:
 *   ridx      [Br, 80 k] int8 : region slot (0 .. 15) of each token, in the cidx column layout (token 77 c + j of chunk
 *               c at column 80 c + j, k key chunks as for cidx); -1 = the token belongs to no region
 *   rec_index [B] int32        : image b's record (row of ridx and of rec_acc), -1 = image b is not recorded.  The
 *               recorded images of one call must have distinct records.
 *   rec_acc   [Br, H, N, 16] fp32, 16-byte aligned, record i at rec_acc + i * rec_batch_stride:
 *               rec_acc[i, h, n, r] += sum_{t : ridx[t] = r} P[n, t] / sum_t P[n, t]
 *               with P the softmax probabilities of head h (after the bias, for biased images).  Slots no token maps to
 *               get 0; when every real token has a slot, the slots sum to 1 up to fp32 rounding.  A plain read-add-write
 *               in stream order (no atomics): zero the buffer before the first call, and calls on one stream add up.
 *   rec_batch_stride : elements between records, >= H * N * 16
 * Recording covers biased and unbiased images alike; mpack == NULL (no image biased) records plain attention.  A NULL
 * ridx / rec_index / rec_acc, a misaligned rec_acc or a too small rec_batch_stride returns PWW_ERR_BAD_ARG before any
 * CUDA call.  Batch splits offset rec_index with the images, as they do wmap_index.
 */
int pww_xattn_fused_rec_f16(const void* q, const void* k, const void* v, void* out,
                            int B, int H, int N, int T, int D,
                            int64_t q_batch_stride, int64_t q_row_stride,
                            int64_t k_batch_stride, int64_t k_row_stride,
                            int64_t o_batch_stride, int64_t o_row_stride,
                            const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
                            const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale,
                            float* stats, void* workspace, size_t workspace_bytes, void* stream,
                            const int8_t* ridx, const int32_t* rec_index, float* rec_acc, int64_t rec_batch_stride);
int pww_xattn_fused_rec_bf16(const void* q, const void* k, const void* v, void* out,
                             int B, int H, int N, int T, int D,
                             int64_t q_batch_stride, int64_t q_row_stride,
                             int64_t k_batch_stride, int64_t k_row_stride,
                             int64_t o_batch_stride, int64_t o_row_stride,
                             const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
                             const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale,
                             float* stats, void* workspace, size_t workspace_bytes, void* stream,
                             const int8_t* ridx, const int32_t* rec_index, float* rec_acc, int64_t rec_batch_stride);

/*
 * Self-attention through the same patched function (context=None, paint_with_words.py:71-72):
 *   out = softmax(scale * Q_h K_h^T) V_h  with keys/values [B, N, H*D]; no bias; online softmax.
 */
int pww_attn_fwd_f16(const void* q, const void* k, const void* v, void* out,
                     int B, int H, int N, int D,
                     int64_t qkv_batch_stride, int64_t qkv_row_stride,
                     int64_t o_batch_stride, int64_t o_row_stride,
                     float scale, void* stream);
int pww_attn_fwd_bf16(const void* q, const void* k, const void* v, void* out,
                      int B, int H, int N, int D,
                      int64_t qkv_batch_stride, int64_t qkv_row_stride,
                      int64_t o_batch_stride, int64_t o_row_stride,
                      float scale, void* stream);

/*
 * Fused memory-bound ops of the UNet that calls the attention path (the reference gets them from diffusers/ATen as
 * separate eager launches): channels-last fp16 (_f16) or bf16 (_bf16) activations, parameters and `add` of the same
 * type, fp32 arithmetic, deterministic reductions.
 *
 * GroupNorm over [B, HW, C] (channels last) with G groups:  y = act((x + add[b,c] - mean) * rstd * gamma + beta),
 * `add` ([B, C] with row stride `add_batch_stride`, may be NULL) is the ResNet block's time-embedding term (added before normalisation), act = SiLU when
 * `silu` != 0.  Needs C % 8 == 0, C % G == 0, G <= 64 and pww_groupnorm_workspace_bytes() of scratch (any
 * contents: the statistics launch writes every partial the apply launch reads).  The apply launch is a programmatic
 * dependent of the statistics launch on `stream`.
 */
size_t pww_groupnorm_workspace_bytes(int B, int HW, int G);
int pww_groupnorm_nhwc_f16(const void* x, const void* add, int64_t add_batch_stride /* elements */,
                           const void* gamma, const void* beta, void* y,
                           int B, int HW, int C, int G, float eps, int silu,
                           void* workspace, size_t workspace_bytes, void* stream);
int pww_groupnorm_nhwc_bf16(const void* x, const void* add, int64_t add_batch_stride /* elements */,
                            const void* gamma, const void* beta, void* y,
                            int B, int HW, int C, int G, float eps, int silu,
                            void* workspace, size_t workspace_bytes, void* stream);

/* GEGLU: out[m, i] = in[m, i] * gelu(in[m, I + i]) for in [M, 2*I], out [M, I] (exact erf GELU); I % 8 == 0. */
int pww_geglu_f16(const void* in, void* out, int64_t M, int I, void* stream);
int pww_geglu_bf16(const void* in, void* out, int64_t M, int I, void* stream);

/* Residual add + LayerNorm over the last dim of [M, C]:  s = x + res (res may be NULL);  sum_out = s (may be NULL);
 * y = LayerNorm(s) * gamma + beta.  The transformer block's "x = attn(...) + x; h = norm(x)" pair in one pass.
 * C % 8 == 0, C <= 2048. */
int pww_add_layernorm_f16(const void* x, const void* res, const void* gamma, const void* beta, void* sum_out, void* y,
                          int64_t M, int C, float eps, void* stream);
int pww_add_layernorm_bf16(const void* x, const void* res, const void* gamma, const void* beta, void* sum_out, void* y,
                           int64_t M, int C, float eps, void* stream);

/* ResNet-block residual epilogue over [rows, C] channels-last activations:
 *   out[r, c] = E( a[r, c] + h[r, c] + bias[c] )
 * a is the block input (identity shortcut) or the bias-free shortcut conv output, h the bias-free conv2 output, bias an
 * fp32 [C] array (conv2's bias plus the shortcut's).  fp32 arithmetic with one rounding.  out may be h (in place); it
 * must not otherwise overlap a or h.  Returns PWW_ERR_BAD_ARG, before any CUDA call, for a null pointer, rows <= 0,
 * C <= 0, C % 8 != 0 or a pointer that is not 16-byte aligned. */
int pww_resnet_residual_f16(const void* a, const void* h, const float* bias, void* out, int64_t rows, int C,
                            void* stream);
int pww_resnet_residual_bf16(const void* a, const void* h, const float* bias, void* out, int64_t rows, int C,
                             void* stream);

/* T2I-Adapter feature add fused into a residual epilogue, over [rows, pixels, C] channels-last activations:
 *   s = E( a + b [+ bias[c]] )                               every row
 *   out = E( s + feat )  for rows r < feat_rows,  out = s  otherwise
 * a and b are the two residual operands (a transformer's projection and its input, or a ResNet block's shortcut and its
 * bias-free conv2 output), bias an fp32 [C] array or NULL (no bias term), feat a [feat_rows, pixels, C] adapter
 * feature (NULL when feat_rows == 0).  fp32 arithmetic, rounded to E after each add: with feat_rows == 0 and a bias
 * this is bitwise pww_resnet_residual, without a bias torch's `a + b`.  out may be a or b (in place); it must not
 * otherwise overlap a, b or feat.  Returns PWW_ERR_BAD_ARG, before any CUDA call, for a null a, b or out, rows <= 0,
 * pixels <= 0, C <= 0, C % 8 != 0, feat_rows outside 0..rows, a null feat with feat_rows > 0, or a pointer that is not
 * 16-byte aligned. */
int pww_adapter_residual_f16(const void* a, const void* b, const float* bias, const void* feat, void* out, int rows,
                             int64_t pixels, int C, int feat_rows, void* stream);
int pww_adapter_residual_bf16(const void* a, const void* b, const float* bias, const void* feat, void* out, int rows,
                              int64_t pixels, int C, int feat_rows, void* stream);

/*
 * The sampler step around the UNet (LMS, Euler, Euler ancestral, DPM++ 2M), two launches per denoising step.
 * Latents are [m, 4, h, w] fp32 contiguous; dtype codes name the UNet's input / output type.
 *
 * pww_sampler_input: the UNet input [2m, channels, h, w] (contiguous, `out_dtype`): rows i and m + i both get
 *   round(latents[i] * scale[0]) in channels 0..3 and, for channels == 9, round(extra[i]) in channels 4..8 (extra is
 *   [m, 5, h, w] fp32: the inpaint mask and masked-image latents; NULL for channels == 4).  `scale` is a device scalar.
 *
 * pww_sampler_update: classifier-free guidance and one step of the linear step form, latents updated in place:
 *   eps    = eps_u + guidance[i] (eps_c - eps_u)         eps_c = eps[i], eps_u = eps[m + i] ([2m, 4, h, w], any strides)
 *   q      = a x + b eps                                 written to history entry `slot`
 *   x_next = alpha x + (beta[0] q + beta[1] h1 + ... + beta[L-1] h_{L-1}) + gamma z
 * h_k is history entry (slot - k) mod L, L = history_len (1..4); history is [L, m, 4, h, w] fp32.  z is noise row
 * `row` of noise [n, m, 4, h, w] fp32 (noise may be NULL; the term is skipped when gamma == 0).  beta is a [4] and
 * form a [6] device array: form = {alpha, a, b, gamma, slot, row}.  All arithmetic is fp32, rounded after every
 * operation in the order written; a == 0 gives q = b eps and alpha == 1 gives x + (...).
 * Both return PWW_ERR_BAD_ARG for null pointers or bad sizes and PWW_ERR_UNSUPPORTED for other dtypes, before any
 * CUDA call.  Dtype codes: 0 fp32, 1 fp16, 4 bf16.  Codes 2 and 3 are not assigned: releases up to 0.3.0 returned
 * PWW_ERR_UNSUPPORTED for them, and they keep doing so, so a caller that relied on that answer sees no change.
 */
#define PWW_DTYPE_F32 0
#define PWW_DTYPE_F16 1
#define PWW_DTYPE_BF16 4
int pww_sampler_input(const float* latents, const float* scale, const float* extra, void* out, int out_dtype,
                      int m, int channels, int height, int width, void* stream);
int pww_sampler_update(const void* eps, int eps_dtype, int64_t eps_batch_stride, int64_t eps_channel_stride,
                       int64_t eps_row_stride, int64_t eps_col_stride,
                       float* latents, float* history, int history_len, const float* noise,
                       const float* guidance, const float* beta, const float* form,
                       int m, int height, int width, void* stream);

/*
 * ControlNet residual injection: n (1..16) residuals added in place into n activations, in one launch.
 *   dst_k[b] = E( dst_k[b] + E( s[k, b] * res_k[b] ) )        k < n, b < rows
 * dst[k] points at a [B, elems_per_image[k]] tensor and res[k] at a [rows, elems_per_image[k]] one, both dense (a
 * channels-last activation is); only the first `rows` images of each dst are touched (rows = B is the ordinary case,
 * rows = B / 2 guess mode, where only the cond half gets the residuals).  `scales` is a device fp32 [n, rows] array, or
 * NULL for a scale of 1.  The arithmetic is fp32, the product rounded to E before the add, so the result is bitwise
 * torch's `skip + (r * s)` with the product in E.  dst, res and elems_per_image are HOST arrays of n entries; the
 * table travels in the kernel parameters, so a captured CUDA graph carries it.
 * Returns PWW_ERR_BAD_ARG, before any CUDA call, for n outside 1..16, rows < 1, an elems_per_image entry that is not a
 * positive multiple of 8, or a null or not 16-byte-aligned pointer.
 */
int pww_control_inject_f16(int n, void* const* dst, const void* const* res, const int64_t* elems_per_image, int rows,
                           const float* scales, void* stream);
int pww_control_inject_bf16(int n, void* const* dst, const void* const* res, const int64_t* elems_per_image, int rows,
                            const float* scales, void* stream);

/*
 * Multi-ControlNet residual combine: the n (1..16) residuals of each of `units` (1..10) ControlNets, scaled and summed
 * level by level in unit order, in one launch.
 *   out_k[b] = E( ... E( E(s[0,k,b] * res_{0,k}[b]) + E(s[1,k,b] * res_{1,k}[b]) ) ... + E(s[U-1,k,b] * res_{U-1,k}[b]) )
 *                                                                                             k < n, b < rows
 * out[k] and res[u * n + k] (unit-major, units * n entries) point at dense [rows, elems_per_image[k]] tensors.  out[k]
 * may be the same buffer as any res[u * n + k] (in place into one unit's residuals); partial overlaps are undefined.
 * `scales` is a device fp32 [units, n, rows] array.  Every product and partial sum is rounded to E, so the result is
 * bitwise torch's left-to-right sum of `(r * s).to(E)` in E; passing it to pww_control_inject with a NULL scale then
 * adds it unchanged.  out, res and elems_per_image are HOST arrays; the table travels in the kernel parameters, so a
 * captured CUDA graph carries it.
 * Returns PWW_ERR_BAD_ARG, before any CUDA call, for units outside 1..10, n outside 1..16, rows < 1, a NULL scales, an
 * elems_per_image entry that is not a positive multiple of 8, or a null or not 16-byte-aligned pointer.
 */
int pww_control_combine_f16(int units, int n, void* const* out, const void* const* res,
                            const int64_t* elems_per_image, int rows, const float* scales, void* stream);
int pww_control_combine_bf16(int units, int n, void* const* out, const void* const* res,
                             const int64_t* elems_per_image, int rows, const float* scales, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PWW_B200_H_ */
