/*
 * unispeech_b200 -- C ABI of the H100 (sm_90a) WavLM / UniSpeech-SAT encoder hot path.
 *
 * Every entry point enqueues hand-written sm_90a kernels on the given CUDA stream and returns without
 * synchronising.  All pointers are DEVICE pointers owned by the caller (PyTorch tensors); the library never
 * allocates or frees caller memory on the hot path.  Return value: 0 on success, negative on error (message via
 * b200s_last_error(), thread-local).  There is no CPU fallback: on a device that is not compute capability 9.0
 * b200s_check_device() fails and so does every kernel launch.
 *
 * The reference (microsoft/UniSpeech) has no FFI for this path: it is plain PyTorch module code.  Each function
 * below cites the reference lines whose library calls (cuDNN conv, cuBLAS GEMM, F.multi_head_attention_forward,
 * F.layer_norm, F.group_norm, F.gelu, autograd) it replaces.  Paths are relative to /root/reference.
 * Conventions: activations bf16, accumulation fp32, parameters / gradients fp32 masters in the reference
 * state_dict layout.  "bs" = batch stride, "rs"/"ld" = row stride, always in ELEMENTS.  Gradient outputs marked
 * (+=) are accumulated with fp32 atomics: the caller zeroes them once per optimisation step.
 */
#ifndef UNISPEECH_B200_H_
#define UNISPEECH_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* b200s_stream; /* cudaStream_t */

int b200s_version(void);
const char* b200s_last_error(void);
/* 0 if the current device can run the kernels (sm_90), negative otherwise */
int b200s_check_device(void);
/* number of kernels launched by this library so far (bench.py reports the per-step count) */
long long b200s_launch_count(void);
/* zero `bytes` bytes of device memory on the stream (cudaMemsetAsync): the per-step reset of the flat gradient buffer that the
 * backward kernels accumulate into (the reference's `optimizer.zero_grad()`, src/fairseq/trainer.py:627) */
int b200s_memset_zero(void* p, unsigned long long bytes, b200s_stream stream);

/* ---- fused GEMM epilogue description (all tensors optional) ------------------------------------------------
 * value = acc (+ bias[col]);  if gelu: out_pre <- value (gelu = 1) or gelu'(value) (gelu = 2) (optional), value = gelu_erf(value)
 *         if dgelu: value *= gelu'(gelu_aux[row,col]) (dgelu = 1) or gelu_aux[row,col] (dgelu = 2, aux written by a gelu = 2
 *         forward: the backward epilogue is then a plain multiply);  value += res1 + res2;  out <- value
 * colsum (fp32[N], +=) accumulates column sums of the stored values (bias gradients). */
typedef struct {
  const float* bias;
  const void* res1; long long res1_bs, res1_ld;
  const void* res2; long long res2_bs, res2_ld;
  const void* gelu_aux; long long aux_bs, aux_ld;
  void* out_pre; long long pre_bs, pre_ld;
  float* colsum;
  int gelu;
  int dgelu;
} b200s_epilogue;

/* ============================ wgmma GEMM family (csrc/gemm.cuh, gemm.cu) ============================== */

/* out[b, r, 0:N] = epilogue( A[b, r, 0:K] . W[N,K]^T ),  bf16 in / bf16 out, fp32 accumulate.
 * A rows live at a + b*a_bs + r*a_rs and may OVERLAP (a_rs < K): this is how the strided Conv1d layers 1-6 of
 * ConvFeatureExtractionModel (WavLM/WavLM.py:400-403,485-504) and their input gradients become GEMMs on
 * channels-last [B,T,C] activations (row = k*C window, row stride = stride*C).  Also every nn.Linear forward /
 * input-gradient: q,k,v,out_proj (WavLM/modules.py:540-563), fc1/fc2 (WavLM/WavLM.py:706-739),
 * post_extract_proj (WavLM/WavLM.py:347-348).  K % 64 == 0, N % 8 == 0. */
int b200s_gemm_rows(const void* a, long long a_bs, long long a_rs, int rows, int batches, int K,
                    const void* w, int N, void* out, long long out_bs, long long out_ld,
                    const b200s_epilogue* epi, b200s_stream stream);

/* dW[n, k] (+=) sum_{b,r} Y[b,r,n] * X[b,r,k]   (fp32, row stride dw_ld): the weight gradient of the GEMMs above
 * (autograd of nn.Linear / nn.Conv1d).  Both operands are read MN-major by wgmma; X rows may overlap
 * (conv im2col view).  The reduction over (batch, 64-row) blocks is split across CTAs and summed with fp32 atomics (K >= 256:
 * stream-K over 128 x 256 tiles; narrower: split-K over 128 x 64 tiles).  N % 8 == 0, K % 8 == 0. */
int b200s_gemm_wgrad(const void* y, long long y_bs, long long y_rs, const void* x, long long x_bs,
                     long long x_rs, int rows, int batches, int N, int K, float* dw, long long dw_ld,
                     b200s_stream stream);
/* Ragged batches (utterances of different lengths, zero-padded to the longest: BASELINE.json configs[4]).  Same contracts as
 * b200s_gemm_rows / b200s_gemm_wgrad with batches = utterances and rows = padded frames per utterance, plus a DEVICE int32 array
 * `valid[batches]` = frames of each utterance that hold real audio (padding is a suffix).  gemm_rows_ragged: an M tile that
 * starts at or beyond valid[b] is not computed; its output rows (and the saved pre-activation) are written as ZEROS (padded rows
 * must stay finite).  gemm_wgrad_ragged: 64-row blocks that start at or beyond valid[b] are neither loaded nor multiplied --
 * exact whenever the loss does not read padded frames (their gradient rows are then zero; the reference computes them anyway,
 * WavLM/WavLM.py:574-575 zeroes the inputs but every row-wise op still runs on them).  Small shapes that take the single-CTA
 * kernel ignore `valid` (they compute every row). */
int b200s_gemm_rows_ragged(const void* a, long long a_bs, long long a_rs, int rows, int batches, int K, const void* w, int N,
                           void* out, long long out_bs, long long out_ld, const b200s_epilogue* epi, const int* valid,
                           b200s_stream stream);
int b200s_gemm_wgrad_ragged(const void* y, long long y_bs, long long y_rs, const void* x, long long x_bs, long long x_rs,
                            int rows, int batches, int N, int K, float* dw, long long dw_ld, const int* valid,
                            b200s_stream stream);

/* ---- FP8 (e4m3) inference path of the encoder projections (csrc/fp8.cu, csrc/fp8.cuh) ----------------------------------
 * Quantisation rule (activations per row, weights per output channel), amax = max |x| of the row in fp32:
 *   q = e4m3_satfinite(x * (448 / amax)),  s = amax / 448  (IEEE divisions);  amax == 0 gives q = 0, s = 0.
 * A bf16 input is quantised from its bf16 value.  `valid` (int32 [batches], device) may be NULL (every row counts).
 *
 * out[b, r, n] = epilogue( a_scale[b*rows + r] * w_scale[n] * sum_k a8[b, r, k] w8[n, k] ): e4m3 K-major operands (A rows at
 * a8 + b*a_bs + r*a_rs bytes, W [N, K] contiguous), fp32 accumulation, bf16 out.  The epilogue takes `bias`, `gelu` (the value,
 * no out_pre) and `res1`, applied after the scales; anything else is an error.  Ragged batches as b200s_gemm_rows_ragged: an M
 * tile at or past valid[b] is written as zeros.  K % 128 == 0, N % 8 == 0, 16-byte-aligned rows. */
int b200s_gemm_rows_fp8(const void* a8, const float* a_scale, long long a_bs, long long a_rs, int rows, int batches, int K,
                        const void* w8, const float* w_scale, int N, void* out, long long out_bs, long long out_ld,
                        const b200s_epilogue* epi, const int* valid, b200s_stream stream);
/* bf16 rows [batches, rows, D] (element strides x_bs, x_rs) -> e4m3 rows (byte strides q_bs, q_rs) and scale[b*rows + r]: the
 * GEMM inputs that no LayerNorm produces (attention output, GELU output).  Rows at or past valid[b] are not read; they are
 * written as zeros with s = 0.  D % 8 == 0, D <= 8192. */
int b200s_quantize_rows_fp8(const void* x, long long x_bs, long long x_rs, int rows, int batches, int D, void* q, long long q_bs,
                            long long q_rs, float* scale, const int* valid, b200s_stream stream);
/* Every e4m3 weight of the encoder in one launch.  descs: device array of n_descs records
 *   { const float* src; void* dst; float* scale; int N; int K; }   (32 bytes, K % 8 == 0)
 * dst[n, k] = e4m3 of the fp32 master src[n, k] with scale[n] per output channel; max_rows = the largest N. */
int b200s_prep_linear_fp8_batched(const void* descs, int n_descs, int max_rows, b200s_stream stream);

/* Grouped positional convolution as an implicit GEMM (TransformerEncoder.pos_conv, WavLM/WavLM.py:514-527,577-579;
 * SamePad WavLM/modules.py:72-83), also used for its input gradient with flipped/transposed taps:
 *   out[b,t,g*Cg+n] = epilogue( sum_{j<taps} sum_{c<Cg} xpad[b, t+j, g*Cg+c] * wp[g*Cgp+n, j*Cgp+c] )
 * xpad: [B, Tpad, D] bf16 (row stride D) with zero rows around the T valid frames, pointer offset so that tap j of
 * output frame t reads row t+j;  wp: [G*Cgp, taps*Cgp] bf16 zero padded (b200s_posconv_prep).  Cg = D/G <= 128, a multiple
 * of 8; Cgp = 64 if Cg <= 64, else 128 (then taps <= 129). */
int b200s_posconv_gemm(const void* xpad, long long xpad_bs, int T, int B, int D, int G, int taps,
                       const void* wp, void* out, long long out_bs, long long out_ld,
                       const b200s_epilogue* epi, b200s_stream stream);

/* dwp[g, n, j, c] (+=) sum_{b,t} dy[b,t,g*Cg+n] * xpad[b,t+j,g*Cg+c];  dwp fp32 [G, Cg, taps, Cgp], only c < Cg is
 * meaningful. */
int b200s_posconv_wgrad(const void* dy, long long dy_bs, long long dy_rs, const void* xpad, long long xpad_bs,
                        int T, int B, int D, int G, int taps, float* dwp, b200s_stream stream);

/* ============================ attention (csrc/attn_fwd.cu, attn_bwd2.cu) =========================== */

/* out[b,t,h*HD+d] = sum_j softmax_j(scale q_i.k_j + gate[b,h,i]*tab[h,j-i+T-1], -inf at padded keys) v_j
 * Replaces compute_bias + gate multiply + F.multi_head_attention_forward (WavLM/modules.py:417-455,504-563); the
 * [B*H,T,T] bias is never materialised (it is Toeplitz).  qkv: bf16 [B,T,3D] fused projection output; gate: fp32
 * [B,H,T] or NULL (=1); tab: fp32 [H,2T-1] or NULL (no bias); key_pad: uint8 [B,T] or NULL; out: bf16 [B,T,D];
 * lse: fp32 [B,H,T] log2-domain log-sum-exp (saved for backward).  head_dim HD = 64, or 80 / 120 with tab = NULL (D = H * HD;
 * any other value is an error); any T >= 1 with B*H*T < 2^32 (the kernel stages the bias window and key mask per key tile:
 * its shared memory does not depend on T).  The same head_dim argument ends every attention entry point below. */
int b200s_attn_fwd(const void* qkv, const float* gate, const float* tab, const uint8_t* key_pad, void* out,
                   float* lse, int B, int T, int H, float scale, int head_dim, b200s_stream stream);

/* Backward of b200s_attn_fwd (autograd of the same lines).  delta: fp32 [B,H,T] workspace; dqkv: bf16 [B,T,3D];
 * dgate: fp32 [B,H,T] (written); dtab: fp32 [H,2T-1] (+=, shared by all layers: WavLM/WavLM.py:549,594-599).  Any T >= 1;
 * runs the fused kernel below with an fp32 dQ buffer allocated on the stream for the call. */
int b200s_attn_bwd(const void* qkv, const void* out, const void* dout, const float* gate, const float* tab,
                   const uint8_t* key_pad, const float* lse, float* delta, void* dqkv, float* dgate, float* dtab,
                   int B, int T, int H, float scale, int head_dim, b200s_stream stream);

/* Same contract as b200s_attn_bwd, computed by ONE fused tensor-core kernel (csrc/attn_bwd2.cu: probabilities recomputed
 * once, dK/dV accumulated in registers, dQ reduced across key tiles in fp32).  dq_acc: fp32 [B,T,D] workspace that must be ZERO
 * on entry and is zero again on return.  Any T >= 1 (constant shared memory). */
int b200s_attn_bwd_fused(const void* qkv, const void* out, const void* dout, const float* gate, const float* tab,
                         const uint8_t* key_pad, const float* lse, float* delta, float* dq_acc, void* dqkv,
                         float* dgate, float* dtab, int B, int T, int H, float scale, int head_dim,
                         b200s_stream stream);

/* Attention with dropout on the probabilities (attention_dropout; the dropout_p argument of
 * F.multi_head_attention_forward, WavLM/modules.py:551): O = (softmax(..) o M) V / (1 - p).  M comes from the counter-based
 * hash of csrc/dropout.cuh keyed by (key0, key1, (b*H+h)*T + i, j); the forward kernel also records it as a bit mask
 * (drop_mask: b200s_attn_dropout_mask_words(B,T,H) uint32 words) which the fused backward re-reads, so the backward needs
 * no key.  drop_p = 0 is exactly b200s_attn_fwd / b200s_attn_bwd_fused (drop_mask may be NULL).  B*H*T < 2^32 (the row
 * counter of the hash); the mask takes B*H*T^2/8 bytes (134 MB per layer for one utterance of T = 8192 with 16 heads). */
int b200s_attn_fwd_dropout(const void* qkv, const float* gate, const float* tab, const uint8_t* key_pad, void* out,
                           float* lse, int B, int T, int H, float scale, float drop_p, uint32_t key0, uint32_t key1,
                           uint32_t* drop_mask, int head_dim, b200s_stream stream);
int b200s_attn_bwd_fused_dropout(const void* qkv, const void* out, const void* dout, const float* gate,
                                 const float* tab, const uint8_t* key_pad, const float* lse, float* delta,
                                 float* dq_acc, void* dqkv, float* dgate, float* dtab, int B, int T, int H, float scale,
                                 float drop_p, const uint32_t* drop_mask, int head_dim, b200s_stream stream);
long long b200s_attn_dropout_mask_words(int B, int T, int H);

/* Deprecated, kept for callers of the earlier ABI: validates 0 <= sms < SM count and has no effect.  It reserved SMs of the persistent
 * GEMM grid for a concurrent collective; the GEMMs now launch one CTA per tile, so NCCL's CTAs take SMs as tiles retire. */
int b200s_reserve_sms(int sms);

/* ============================ row kernels (csrc/rowops.cu) ============================ */

/* y = LayerNorm(x) * gamma + beta [then exact GELU]; saves mean / rstd (fp32 [rows]).  nn.LayerNorm / Fp32LayerNorm
 * (WavLM/WavLM.py:342,559,666,675; WavLM/modules.py:30-42) and the LN+GELU of the layer_norm extractor
 * (WavLM/WavLM.py:409-419).  D in {64,128,256,512,768,1024}. */
int b200s_layer_norm_fwd(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta,
                         void* y, long long y_bs, long long y_rs, float* mean, float* rstd, int rows_per_batch,
                         int batches, int D, int gelu, b200s_stream stream);

/* LayerNorm forward fused with the gru_rel_pos gate of the attention that consumes y (b200s_gate_fwd semantics on the stored
 * bf16 y): saves one pass over y per layer.  D = H * 64; gate: fp32 [B, H, T]; rows = B * T with the usual views. */
int b200s_layer_norm_gate_fwd(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta,
                              void* y, long long y_bs, long long y_rs, float* mean, float* rstd, int T, int B, int D,
                              const float* grep_w, const float* grep_b, const float* grep_a, int H, float* gate,
                              b200s_stream stream);

/* LayerNorm forward with an e4m3 output for the fp8 GEMMs: q / scale (b200s_quantize_rows_fp8 layout and rule) are taken from
 * the bf16-rounded normalised row, so they equal the quantisation of the bf16 y.  y (bf16), mean and rstd are optional (NULL);
 * y, when written, is bit-identical to b200s_layer_norm_fwd.  gate != NULL also writes the gru_rel_pos gate of the attention
 * that consumes the row (b200s_layer_norm_gate_fwd semantics; D = H * 64 in 256..1280).  Rows at or past valid[b] (valid may be
 * NULL): zeros, s = 0, mean = rstd = 0, gate = 1.  D as b200s_layer_norm_fwd. */
int b200s_layer_norm_fwd_fp8(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta, void* y,
                             long long y_bs, long long y_rs, float* mean, float* rstd, void* q, long long q_bs, long long q_rs,
                             float* scale, int rows_per_batch, int batches, int D, const float* grep_w, const float* grep_b,
                             const float* grep_a, int H, float* gate, const int* valid, b200s_stream stream);

/* dx = LN-backward(dy) [+ dres];  dgamma, dbeta (+=);  colsum (+=) = column sums of dx (bias gradient of x's producer). */
int b200s_layer_norm_bwd(const void* dy, long long dy_bs, long long dy_rs, const void* x, long long x_bs,
                         long long x_rs, const float* mean, const float* rstd, const float* gamma,
                         const float* beta, const void* dres, long long dres_bs, long long dres_rs, void* dx,
                         long long dx_bs, long long dx_rs, float* dgamma, float* dbeta, float* colsum,
                         int rows_per_batch, int batches, int D, int gelu, b200s_stream stream);

/* Ragged-batch forms of the row kernels (BASELINE configs[4]; the reference pads and computes every frame, WavLM.py:574-575).
 * valid[b] (int32, device): rows of batch b that hold real frames.  Rows at or beyond it are PADDING: the forward kernels write
 * zeros (mean = rstd = 0, gate = 1) without reading x, the backward kernels write a zero gradient row (nothing downstream of a
 * padded frame reaches the loss), the column sum skips them.  valid == NULL: identical to the plain entry point. */
int b200s_layer_norm_fwd_ragged(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta,
                                void* y, long long y_bs, long long y_rs, float* mean, float* rstd, int rows_per_batch,
                                int batches, int D, int gelu, const int* valid, b200s_stream stream);
int b200s_layer_norm_gate_fwd_ragged(const void* x, long long x_bs, long long x_rs, const float* gamma, const float* beta,
                                     void* y, long long y_bs, long long y_rs, float* mean, float* rstd, int T, int B, int D,
                                     const float* grep_w, const float* grep_b, const float* grep_a, int H, float* gate,
                                     const int* valid, b200s_stream stream);
int b200s_layer_norm_bwd_ragged(const void* dy, long long dy_bs, long long dy_rs, const void* x, long long x_bs,
                                long long x_rs, const float* mean, const float* rstd, const float* gamma,
                                const float* beta, const void* dres, long long dres_bs, long long dres_rs, void* dx,
                                long long dx_bs, long long dx_rs, float* dgamma, float* dbeta, float* colsum,
                                int rows_per_batch, int batches, int D, int gelu, const int* valid, b200s_stream stream);
int b200s_colsum_ragged(const void* x, long long x_bs, long long x_rs, int rows_per_batch, int batches, int N, float* out,
                        const int* valid, b200s_stream stream);
int b200s_gate_bwd_ragged(const void* x, long long x_bs, long long x_rs, int T, int B, int H, const float* grep_w,
                          const float* grep_b, const float* grep_a, const float* dgate, void* dxg, long long dx_bs,
                          long long dx_rs, float* dgrep_w, float* dgrep_b, float* dgrep_a, const int* valid,
                          b200s_stream stream);

/* out[c] (+=) sum_rows x[r,c]  -- nn.Linear bias gradients */
int b200s_colsum(const void* x, long long x_bs, long long x_rs, int rows_per_batch, int batches, int N, float* out,
                 b200s_stream stream);

/* out = dy * gelu'(pre); colsum (+=) optional.  Backward of x + gelu(pos_conv(x)) (WavLM/WavLM.py:577-579) and of the
 * last conv layer's GELU. */
int b200s_dgelu_mul(const void* dy, long long dy_bs, long long dy_rs, const void* pre, long long pre_bs,
                    long long pre_rs, void* out, long long out_bs, long long out_rs, int rows_per_batch, int batches,
                    int N, float* colsum, b200s_stream stream);
/* Same; pre_is_grad != 0: `pre` already holds gelu'(pre-activation) (written by a gelu = 2 epilogue), out = dy * pre. */
int b200s_dgelu_mul_ex(const void* dy, long long dy_bs, long long dy_rs, const void* pre, long long pre_bs,
                       long long pre_rs, void* out, long long out_bs, long long out_rs, int rows_per_batch, int batches,
                       int N, float* colsum, int pre_is_grad, b200s_stream stream);

/* *out += sum of x^2 over a bf16 rows view (fp64 accumulator, caller zeroes it): numerator of the feature penalty
 * `features.float().pow(2).mean()` (src/fairseq/models/wavlm/wavlm.py:484).  N % 8 == 0. */
int b200s_sumsq_rows(const void* x, long long x_bs, long long x_rs, int rows_per_batch, int batches, int N, double* out,
                     b200s_stream stream);
/* Backward of GradMultiply.apply(features, scale) (WavLM/modules.py:60-69, WavLM/WavLM.py:333-336) fused with the gradient of
 * the feature penalty taken on its output (fairseq wavlm.py:477-484), in place on the bf16 gradient rows g:
 *   g <- scale * (g + (*pen_grad * pen_mul) * x);   pen_grad = DEVICE float (upstream gradient of the penalty scalar) or NULL. */
int b200s_grad_multiply(void* g, long long g_bs, long long g_rs, const void* x, long long x_bs, long long x_rs,
                        int rows_per_batch, int batches, int N, float scale, const float* pen_grad, float pen_mul,
                        b200s_stream stream);
/* y = [res +] dropout(x), y may alias x.  nn.Dropout / F.dropout of the transformer stack (WavLM/WavLM.py:350,584,659-661,
 * 702-738): keep(row, col) is a pure function of (key0, key1, logical row = b*rows_per_batch + r, col) (csrc/dropout.cuh),
 * kept values are scaled by 1/(1-p).  The backward pass is the same call on the incoming gradient with the same key and
 * res = NULL.  N % 8 == 0, 0 <= p < 1. */
int b200s_dropout_rows(const void* x, long long x_bs, long long x_rs, const void* res, long long res_bs,
                       long long res_rs, void* y, long long y_bs, long long y_rs, int rows_per_batch, int batches,
                       int N, float p, uint32_t key0, uint32_t key1, b200s_stream stream);

/* Host-side evaluation of the mask formulas (csrc/dropout.cuh), no device involved: bits word of counter `ctr`; per-row key
 * of the attention mask (which = 0 / 1 for key0 / key1); 16-bit keep threshold of probability p. */
uint32_t b200s_dropout_bits(uint32_t key0, uint32_t key1, uint32_t ctr);
uint32_t b200s_dropout_row_key(uint32_t key, uint32_t row, int which);
uint32_t b200s_dropout_threshold16(float p);

/* x[b,t,:] = mask_emb where mask[b,t]; = 0 where pad[b,t]   (apply_mask WavLM/WavLM.py:285-286; x[padding_mask]=0 :574-575);
 * then x[b,:,c] = 0 where chan_mask[b,c] (uint8 [B, D], the channel mask of apply_mask :288-307, or NULL).  Backward: dx = 0
 * wherever the forward overwrote x; dmask_emb[c] (+=) sums dx over masked, unpadded frames whose channel c is not masked.
 * mask, pad and chan_mask may each be NULL. */
int b200s_frame_mask_fwd(void* x, long long x_bs, long long x_rs, int T, int B, int D, const uint8_t* mask,
                         const uint8_t* pad, const float* mask_emb, const uint8_t* chan_mask, b200s_stream stream);
int b200s_frame_mask_bwd(void* dx, long long x_bs, long long x_rs, int T, int B, int D, const uint8_t* mask,
                         const uint8_t* pad, float* dmask_emb, const uint8_t* chan_mask, b200s_stream stream);

/* gate[b,h,t] of gru_rel_pos from the RAW layer input (WavLM/modules.py:523-533) and its backward */
int b200s_gate_fwd(const void* x, long long x_bs, long long x_rs, int T, int B, int H, const float* grep_w,
                   const float* grep_b, const float* grep_a, float* gate, b200s_stream stream);
int b200s_gate_bwd(const void* x, long long x_bs, long long x_rs, int T, int B, int H, const float* grep_w,
                   const float* grep_b, const float* grep_a, const float* dgate, void* dxg, long long dx_bs,
                   long long dx_rs, float* dgrep_w, float* dgrep_b, float* dgrep_a, b200s_stream stream);

/* tab[h, i] = emb[lut[i], h]  (Toeplitz form of compute_bias, WavLM/modules.py:445-455) and the scatter-add backward */
int b200s_relpos_table_fwd(const float* emb, const int* lut, int n, int H, float* tab, b200s_stream stream);
int b200s_relpos_table_bwd(const float* dtab, const int* lut, int n, int H, float* demb, b200s_stream stream);

/* ============================ conv layer 0 (csrc/conv0.cu) ============================ */

/* Conv1d(1,C,k,stride s, optional bias) + GroupNorm(C,C) (mode 0) or LayerNorm over channels (mode 1) + GELU on the raw
 * waveform (WavLM/WavLM.py:400-426).  wav fp32 [B,L]; w fp32 [C,1,k]; out bf16 channels-last.  stats: fp64 [B,C,2]
 * (mode 0);  fmean/frstd: fp32 [B,T] (mode 1).  C in {64, 512}.  bias fp32 [C] or NULL (conv_bias=True): added before the
 * LayerNorm in mode 1; in mode 0 the per-(utterance, channel) GroupNorm removes a per-channel constant exactly, so the bias is
 * not applied there and its gradient is zero.  Backward: dbias (+=, mode 1, needs bias) = sum over (b, t) of the gradient at
 * the raw convolution output; mode 0 leaves it untouched. */
int b200s_conv0_fwd(const float* wav, long long L, int B, int T, int C, int k, int s, const float* w,
                    const float* gamma, const float* beta, int mode, double* stats, float* fmean, float* frstd,
                    void* out, long long out_bs, const float* bias, b200s_stream stream);
int b200s_conv0_bwd(const float* wav, long long L, int B, int T, int C, int k, int s, const float* w,
                    const float* gamma, const float* beta, int mode, const double* stats, float* bstats,
                    const float* fmean, const float* frstd, const void* da, long long da_bs, float* dw,
                    float* dgamma, float* dbeta, const float* bias, float* dbias, b200s_stream stream);
/* Same, with a bf16 workspace [B, ws_bs/C rows >= T, C] for the gradient w.r.t. the raw convolution output (mode 1 only; may
 * alias `da`, which is then consumed): the LayerNorm-mode backward becomes one pass over the frames plus one streaming
 * weight-gradient reduction instead of two full recomputing passes. */
int b200s_conv0_bwd_ws(const float* wav, long long L, int B, int T, int C, int k, int s, const float* w,
                       const float* gamma, const float* beta, int mode, const double* stats, float* bstats,
                       const float* fmean, const float* frstd, const void* da, long long da_bs, void* dconv_ws,
                       long long ws_bs, float* dw, float* dgamma, float* dbeta, const float* bias, float* dbias,
                       b200s_stream stream);

/* ============================ parameter preparation (csrc/prep.cu) ============================ */

int b200s_scale_copy_f32(const float* src, float* dst, long long n, float scale, b200s_stream stream);
/* fp32 [N,K] -> bf16 dst[n*ld+k] and/or its transpose dstT[k*ldT+n] */
int b200s_prep_linear(const float* src, int N, int K, float scale, void* dst, long long ld, void* dstT,
                      long long ldT, b200s_stream stream);
/* all nn.Linear operands of the model in ONE launch: descs = device array of n_descs 56-byte records
 * {const float* src; bf16* dst; bf16* dstT; int64 ld, ldT; int32 N, K, tile_begin, tiles_k} (64x64 tiles: tiles_k = ceil(K/64),
 * tile_begin = prefix sum of ceil(N/64)*ceil(K/64)) */
int b200s_prep_linear_batched(const void* descs, int n_descs, int total_tiles, b200s_stream stream);
/* nn.Conv1d weight [Co,Ci,k] -> forward operand [Co, k*Ci] / per-phase input-gradient operand / gradient un-layout */
int b200s_prep_conv_fwd(const float* src, int Co, int Ci, int k, void* dst, b200s_stream stream);
int b200s_prep_conv_dgrad(const float* src, int Co, int Ci, int k, int s, int rho, void* dst, b200s_stream stream);
int b200s_unprep_conv_wgrad(const float* dwk, int Co, int Ci, int k, float* dw, b200s_stream stream);
/* weight_norm(dim=2) of pos_conv (WavLM/WavLM.py:526) -> padded per-group operands wp_fwd / wp_dgrad bf16 [G, Cgp, taps, Cgp]
 * (Cgp as for b200s_posconv_gemm); and its backward from dwp [G, Cg, taps, Cgp].  Workspaces (8-byte aligned,
 * zeroed inside): norm2 = 2 * taps floats, work = 4 * taps floats -- the per-tap sums are accumulated in fp64 so that the norm, and
 * with it every bf16 pos_conv weight, is the same value on every run (the forward pass is bit-reproducible). */
int b200s_posconv_prep(const float* weight_v, const float* weight_g, int D, int G, int taps, float* norm2,
                       void* wp_fwd, void* wp_dgrad, b200s_stream stream);
int b200s_posconv_unprep(const float* weight_v, const float* weight_g, const float* dwp, int D, int G, int taps,
                         float* work, float* dweight_v, float* dweight_g, b200s_stream stream);

/* ============================ optimizer step on the flat gradient buffer (csrc/optim.cu) ============================ */

/* *out += sum_i g[i]^2 (fp64 accumulator on the device; the caller zeroes it).  With the flat gradient buffer this is the global
 * gradient norm of utils.clip_grad_norm_ (src/fairseq/utils.py:338-377) in one launch and without a host round trip. */
int b200s_sumsq_f32(const float* g, long long n, double* out, b200s_stream stream);

/* Same sum restricted to the tensors of an optimizer descriptor table (the layout b200s_adam_step takes): gradients of
 * parameters the optimizer does not own (excluded / frozen) are not counted -- fairseq's clip_grad_norm_ only sees
 * parameters whose .grad exists (src/fairseq/utils.py:338-345). */
int b200s_sumsq_table(const void* table, int n_tensors, long long total_chunks, const float* g, double* out,
                      b200s_stream stream);

/* Fused fairseq Adam update (src/fairseq/optim/adam.py:150-228) of n_tensors fp32 master tensors whose gradients (g) and
 * moments (m = exp_avg, v = exp_avg_sq) live in flat buffers:
 *   g' = g * grad_scale * clip,   clip = max_norm > 0 ? min(1, max_norm / (|grad_scale| * sqrt(*sumsq) + 1e-6)) : 1
 *        (multiply_grads + clip_grad_norm, src/fairseq/optim/fp16_optimizer.py:176-214, utils.py:378-381)
 *   m = beta1 m + (1-beta1) g';  v = beta2 v + (1-beta2) g'^2;  p -= weight_decay*lr*p;
 *   p -= lr*sqrt(1-beta2^step)/(1-beta1^step) * m / (sqrt(v) + eps);   g = 0 if zero_grad.
 * table: DEVICE array of n_tensors records {float* param; int64 goff; int64 numel; int64 chunk0} (32 bytes; goff = element
 * offset in g/m/v, multiple of 4; chunk0 = prefix sum of ceil(numel/2048)); total_chunks = sum of all chunks; step >= 1. */
int b200s_adam_step(const void* table, int n_tensors, long long total_chunks, float* g, float* m, float* v,
                    const double* sumsq, float grad_scale, float max_norm, float lr, float beta1, float beta2,
                    float eps, float weight_decay, int step, int zero_grad, b200s_stream stream);

/* ============================ masked-prediction loss head (csrc/nce.cu) ============================ */
/* final_proj + cosine-similarity NCE logits + sum-reduced cross entropy of the pre-training models
 * (src/fairseq/models/wavlm/wavlm.py:426-438,525-576; src/fairseq/criterions/wavlm_criterion.py:63-87), built around the
 * wgmma GEMMs above: z[s,c] = cos(proj_s, E_c)/temp = (proj En^T)[s,c] / (|proj_s| temp), loss = w * sum_s CE(z[s,:], target_s)
 * (the reference's {positive} U {negatives != positive} softmax IS the softmax over the C classes). */

/* out[s,:] = x[idx[s],:]  (x[masked_indices], wavlm.py:541,558) and its autograd dx[idx[s],:] += src[s,:] (distinct rows) */
int b200s_gather_rows(const void* x, long long x_rs, const int* idx, int S, int D, void* out, long long out_rs,
                      b200s_stream stream);
int b200s_scatter_add_rows(const void* src, long long src_rs, const int* idx, int S, int D, void* dx, long long dx_rs,
                           b200s_stream stream);
/* en[c,:] = bf16(E_c / max(|E_c|,1e-8)) for c < C, zero rows up to Cpad; en_t = its transpose [Dp, Cpad]; invn[c] = 1/max(|E_c|,1e-8) */
int b200s_nce_prep(const float* label_embs, int C, int Cpad, int Dp, void* en, void* en_t, float* invn,
                   b200s_stream stream);
/* zraw = proj En^T (bf16 [S,Cpad], from b200s_gemm_rows).  Writes g[s,c] = weight (softmax(z)_c - [c==target_s]) / (|proj_s| temp)
 * (bf16 [S,Cpad], zero in the padded columns), pn[s] = 1/|proj_s|, rvec[s] = sum_c g[s,c] cos[s,c]; adds weight * sum_s CE to
 * *loss_sum (fp64) and the number of frames whose target has the largest logit to *correct (compute_correct,
 * wavlm_criterion.py:116-126; may be NULL). */
int b200s_nce_ce(const void* proj, long long proj_rs, int Dp, const void* zraw, long long z_rs, const int* target, int S,
                 int C, int Cpad, float logit_temp, float weight, void* g, long long g_rs, float* pn, float* rvec,
                 double* loss_sum, int* correct, b200s_stream stream);
/* dproj[s,:] -= rvec[s] * pn[s] * proj[s,:]   (dproj holds g En on entry: the gradient through 1/|proj_s|) */
int b200s_nce_dproj(void* dproj, long long d_rs, const void* proj, long long p_rs, int S, int Dp, const float* pn,
                    const float* rvec, b200s_stream stream);
/* d_label_embs[c,:] += (d_en_c - (d_en_c . En_c) En_c) / |E_c|,  d_en = g^T proj (fp32 [>=C, Dp], from b200s_gemm_wgrad) */
int b200s_nce_dlabel(const float* d_en, const float* label_embs, const float* invn, int C, int Dp, float* d_label_embs,
                     b200s_stream stream);

/* ============================ UniSpeech-SAT utterance-contrastive head (csrc/sat.cu) ============================ */
/* Utterance-contrastive loss of src/fairseq/models/unispeech_sat/unispeech_sat.py:699-758 (compute_pred_spk, compute_nce with
 * replace_inf=False :545-557, F.binary_cross_entropy_with_logits(...).mean() :736) without the [N+1, S, Dp] gathered instances:
 *   logit[s,0] = cos(proj_s, y_s)/temp, logit[s,1+n] = cos(proj_s, y[idx[n*S+s]])/temp; target[s,0] = 1, target[s,1+n] = same[n*S+s].
 * proj, y: bf16 [S, Dp] rows; idx: int32 [N, S] (host-drawn like sample_instances :487-543); same: uint8 [N, S].
 * Outputs: g fp32 [S, N+1] = d loss / d logit; *loss_sum (fp64, +=) the mean loss; stats[0] += #{(logit >= 0) == target},
 * stats[1] += #{target == 1} (contrastive_acc and mean_targets are these / (S (N+1))).  Dp % 4 == 0, Dp <= 1024. */
int b200s_sat_nce_fwd(const void* proj, long long proj_rs, const void* y, long long y_rs, const int* idx, const uint8_t* same,
                      int S, int N, int Dp, float logit_temp, float* g, double* loss_sum, int* stats, b200s_stream stream);
/* Backward: dproj_acc[s,:] += d loss/d proj_s, dy_acc[r,:] += d loss/d y_r (fp32 [S, Dp], vector reductions; pass the SAME buffer
 * for both when y IS proj, i.e. no quantizer); upstream = DEVICE float, the gradient of the loss scalar. */
/* wav2vec 2.0 InfoNCE (src/fairseq/models/wav2vec/wav2vec2.py:533-553 compute_preds; criterions/wav2vec_criterion.py:57-62,103-118) on
 * the same operands: logit[s,0] = cos(x_s, y_s)/temp, logit[s,1+n] = cos(x_s, y[idx[n*S+s]])/temp, a negative equal to the positive
 * is masked with -inf; *loss_sum += sum_s cross_entropy(logit[s,:], 0); g fp32 [S, N+1] = softmax - onehot(0) (consumed by
 * b200s_sat_nce_bwd); stats[0] += correct (argmax == 0, not also argmin == 0), stats[1] += S.  Dp % 4 == 0, Dp <= 1024. */
int b200s_w2v_nce_fwd(const void* proj, long long proj_rs, const void* y, long long y_rs, const int* idx, int S, int N, int Dp,
                      float logit_temp, float* g, double* loss_sum, int* stats, b200s_stream stream);
int b200s_sat_nce_bwd(const void* proj, long long proj_rs, const void* y, long long y_rs, const int* idx, int S, int N, int Dp,
                      float logit_temp, const float* g, const float* upstream, float* dproj_acc, float* dy_acc,
                      b200s_stream stream);
/* dst (bf16 rows) = src (fp32 rows); N and the row strides multiples of 4 elements */
int b200s_f32_to_bf16_rows(const float* src, long long src_rs, void* dst, long long dst_rs, long long rows, int N,
                           b200s_stream stream);
/* GumbelVectorQuantizer.forward with hard codes (src/fairseq/modules/gumbel_vector_quantizer.py:141-201; time_first,
 * combine_groups = False): logits bf16 [S, G*V] = weight_proj(x); codes[s*G+g] = argmax_v logits (eval) or argmax_v (logits +
 * Gumbel noise from the counter hash with (key0, key1)) (training: the hard sample of F.gumbel_softmax);
 * q[s, g*dv ..] = vars[g*V + code, :] (bf16; vars fp32 [G*V, dv]); counts[g*V+v] += [v == argmax of the NOISE-FREE logits], probs[g*V+v] += softmax(logits)_v
 * (fp32, the caller zeroes them: hard_probs / avg_probs of :152-170 are these / S). */
int b200s_vq_hard(const void* logits, long long logits_rs, const float* vars, int S, int G, int V, int dv, int* codes, void* q,
                  long long q_rs, float* counts, float* probs, int gumbel, uint32_t key0, uint32_t key1, b200s_stream stream);
/* d loss / d logits (bf16 [S, G*V], fully written) = p (c - <c, p>) / S  [c: fp32 [G*V] = d loss / d avg_probs, or NULL]
 *   + ys (h - <h, ys>) / tau  [h: bf16 [S, G*V] = dq . vars^T, or NULL: straight-through gradient of F.gumbel_softmax(hard=True),
 *     ys = softmax((logits + the same noise) / tau)]. */
int b200s_vq_logits_bwd(const void* logits, long long logits_rs, int S, int G, int V, const float* c, const void* h, long long h_rs,
                        float tau, uint32_t key0, uint32_t key1, void* dlogits, long long dlogits_rs, b200s_stream stream);
/* dvars[g*V + codes[s*G+g], :] += dq[s, g*dv ..]   (backward of the codebook lookup) */
int b200s_vq_dvars(const void* dq, long long dq_rs, const int* codes, int S, int G, int V, int dv, float* dvars,
                   b200s_stream stream);

/* ============================ CTC fine-tuning loss (csrc/ctc.cu) ============================ */
/* log-softmax + connectionist temporal classification (Graves et al. 2006; the loss of the fairseq `ctc` criterion) on the bf16
 * logits of the fine-tuning wrappers' `proj` head, without ever materialising log-probabilities: lp[t,c] = logit[t,c] - lse[t].
 * logits: element (t, b, c) at logits[b * batch_stride + t * frame_stride + c] (strides in elements, unit class stride), so the
 * T x B x V view of a [B*T, Vp] buffer is (frame_stride = Vp, batch_stride = T * Vp) and a contiguous T x B x V tensor is
 * (B * V, V).  input_len: int32 [B] valid frames (clamped to [0, T]); frames t >= input_len[b] are NEVER read (they may hold
 * anything) and get an exactly zero gradient.  targets: int32 [B, Smax] padded; target_len: int32 [B].  All device memory.
 * Limits: 1 <= V <= 1024, 0 <= blank < V, Smax <= B200S_CTC_MAX_TARGET (one thread per position of the extended label
 * sequence blank, l_1, blank, ..., l_S, blank); calls beyond them fail, nothing is truncated.
 * An utterance is INFEASIBLE when input_len is too short for its target (with one blank per repeat), or when target_len is
 * outside [0, Smax] or a label outside [0, V): nll = +inf and its whole gradient is written as zeros (with and without
 * zero_infinity). */
#define B200S_CTC_MAX_TARGET 511
/* One warp per valid frame: lse[b*T + t] = logsumexp_c logit[t,b,c] (fp32), argmax[b*T + t] = first class with the largest
 * logit (int32; NULL to skip).  Entries of padded frames are left untouched. */
int b200s_ctc_stats(const void* logits, long long frame_stride, long long batch_stride, const int* input_len, int B, int T, int V,
                    float* lse, int* argmax, b200s_stream stream);
/* Alpha recursion, one CTA per utterance, fp32 log space.  log_alpha: fp32 [B, T, 2*Smax+1] workspace (written for valid frames
 * and positions only; read back by b200s_ctc_beta_grad).  nll[b] = -log p(target_b | logits_b), +inf when infeasible.
 * *loss_sum (fp64, may be NULL) += sum_b nll[b]; with zero_infinity the infeasible utterances are left out of that sum. */
int b200s_ctc_alpha(const void* logits, long long frame_stride, long long batch_stride, const float* lse, const int* input_len,
                    const int* targets, int Smax, const int* target_len, int B, int T, int V, int blank, int zero_infinity,
                    float* log_alpha, float* nll, double* loss_sum, b200s_stream stream);
/* Beta recursion with the gradient through CTC AND the log-softmax fused in (log_beta is never stored):
 *   grad[t,b,c] = upstream[b] * (softmax(logit[t,b,:])_c - sum_{s: l'_s = c} gamma_t(s)),   gamma = exp(alpha + beta - lp + nll),
 * as bf16 at grad[b * grad_batch_stride + t * grad_frame_stride + c] for c < Vpad (columns V..Vpad and every padded frame are
 * zeros).  upstream: DEVICE fp32 [B] = d loss / d nll[b].  The per-class sums run over positions bucketed by class in a fixed
 * order (no floating-point atomics): two calls give bit-identical gradients. */
int b200s_ctc_beta_grad(const void* logits, long long frame_stride, long long batch_stride, const float* lse, const int* input_len,
                        const int* targets, int Smax, const int* target_len, int B, int T, int V, int blank, const float* log_alpha,
                        const float* nll, const float* upstream, void* grad, long long grad_frame_stride,
                        long long grad_batch_stride, int Vpad, b200s_stream stream);

/* ============================ CTC forced alignment (csrc/ctc_align.cu) ============================ */
/* The most probable CTC path of each utterance's known transcript (torchaudio.functional.forced_align, batched): Viterbi over
 * the extended sequence l' = (blank, l_1, blank, ..., l_S, blank) with lp[t,c] = float(logit[t,c]) - lse[t] in fp32, lse from
 * b200s_ctc_stats.  Logits, input_len, targets and target_len are addressed as in the CTC loss entry points above (frames
 * t >= input_len[b] are never read).
 * Tie rule (torchaudio's CPU implementation, reproduced bit for bit): at each (frame, position) the predecessor is skip (s-2)
 * if skip > advance && skip > stay, else advance (s-1) if advance > stay && advance > skip, else stay (s) -- strict
 * comparisons, so exact ties go to stay, and advance == skip > stay takes stay.  The path ends at the final blank if its alpha
 * is strictly larger than the last label's, else at the last label.
 * Outputs: labels int32 [B, T] (class per frame on the path), frame_scores fp32 [B, T] (lp at that class), score fp32 [B]
 * (alpha at the end position: the sum of frame_scores up to fp32 reassociation).  Frames t >= input_len[b] get (-1, 0).  An
 * INFEASIBLE utterance (input_len < S + number of equal adjacent labels, target_len outside [0, Smax], a label outside [0, V)
 * or equal to blank) gets labels -1 and frame_scores 0 on every frame and score -inf; the others are unaffected.  S = 0 aligns
 * every valid frame to blank (score 0 when input_len = 0).
 * workspace: caller-allocated 2-bit backpointers, b200s_ctc_align_workspace_bytes(B, T, Smax) =
 *   B * T * ceil((2 * Smax + 1) / 16) * 4 bytes (one 32-bit word per 16 positions per frame).
 * Limits, checked before any launch: 1 <= V <= 1024, 0 <= blank < V, 0 <= Smax <= B200S_CTC_ALIGN_MAX_TARGET, workspace_bytes
 * at least the size above.  Two launches (Viterbi, backtrack), no floating-point atomics: results are bit-identical from call
 * to call and do not depend on the other utterances of the batch. */
#define B200S_CTC_ALIGN_MAX_TARGET 8191
long long b200s_ctc_align_workspace_bytes(int B, int T, int Smax); /* -1 for bad sizes */
int b200s_ctc_align(const void* logits, long long frame_stride, long long batch_stride, const float* lse, const int* input_len,
                    const int* targets, int Smax, const int* target_len, int B, int T, int V, int blank, void* workspace,
                    long long workspace_bytes, int* labels, float* frame_scores, float* score, b200s_stream stream);

/* ============================ CTC beam-search decoding (csrc/ctc_decode.cu) ============================ */
/* CTC prefix beam search (Hannun et al. 2014) with optional word n-gram LM scoring, batched over utterances; the definition is
 * oracle/decode_oracle.py.  Logits and input_len are addressed as in b200s_ctc_align (frames t >= input_len[b] are never read),
 * lp[t,c] = float(logit[t,c]) - lse[t] in fp32, lse from b200s_ctc_stats.  lae(a, b) = max + log1p(exp(-|a - b|)) in fp32.
 *
 * Hash: h' = splitmix64(h ^ (x + 1)) from h = 0 (splitmix64: z += 0x9E3779B97F4A7C15; z = (z ^ z >> 30) * 0xBF58476D1CE4E5B9;
 * z = (z ^ z >> 27) * 0x94D049BB133111EB; z ^ z >> 31).  A prefix is identified by the hash of its class ids, a spelling by the
 * hash of its class ids, an n-gram by the hash of its word ids (oldest first).
 * Beam state: pb, pnb (log-probabilities of the prefix ending in blank / in its last class), lm (LM part), the prefix hash, the
 * partial word's hash (0 when empty), the last class, the last order - 1 words (starting at <s>).  Start: the empty prefix,
 * pb = 0, pnb = -inf, lm = 0.  Per frame, with T_K = the beam_token non-blank classes of highest lp (ties to the smaller id):
 *   stay of every beam:           pb' = lae(pb, pnb) + lp[blank];  pnb' = pnb + lp[last] (-inf for the empty prefix);
 *   extension of beam j by c in T_K: prefix + c receives (c == last_j ? pb_j : lae(pb_j, pnb_j)) + lp[c] into pnb.
 *   An extension reaching a prefix that is already a beam is merged into its stay (pnb' = lae(pnb', ext)); stays first, then
 *   extensions by parent rank, then class id.  Ranking score = lae(pb, pnb) + lm, order by (score desc, prefix hash asc), keep the
 *   best `beam` after every frame.
 * LM (word level, KenLM's ARPA semantics): appending word_boundary after a non-empty partial word ends the word:
 *   lm += lm_weight * ln P(word | context) + word_score (in that fp32 order), and the word joins the context.  ln P = ln 10 * (the
 *   backoffs, log10, of the longer contexts that matched no n-gram, summed from the longest down, then the log10 p of the
 *   longest n-gram that exists).  The spelling table maps the class ids of each LM word's spelling to its id, each character
 *   spelled by the FIRST class whose symbol is that single character (the boundary excluded): a partial word is a known word
 *   only if its class ids are exactly that spelling, so a later class with a repeated symbol, or a multi-character symbol,
 *   spells no known word.  A spelling that is not in the spelling table is the word `unk`: it adds unk_score after
 *   word_score, and its LM term is 0 when has_unk is 0 (the ARPA file has no <unk>).  An empty word (a leading boundary, or
 *   boundary blank boundary) scores nothing.  After the last frame a non-empty partial word is scored the same way, then
 *   lm += lm_weight * ln P(</s> | context); score = lae(pb, pnb) + lm.  With order = 0 there is no LM and word_boundary is unused.
 * Candidate pruning: each beam is extended only by the min(beam_token, beam + 2) classes of T_K with the highest lp and the
 * boundary class; this can differ from the full candidate set only where exact score ties straddle the beam cutoff.
 * Outputs: tokens int32 [B, nbest, T] (class ids, blanks removed and repeats collapsed, -1 after the end), lengths int32
 * [B, nbest], scores fp32 [B, nbest], best first.  Entries past the number of surviving beams have length 0 and score -inf.
 * workspace: (parent slot | (appended class + 1) << 8) per (b, t, slot), b200s_ctc_decode_workspace_bytes(B, T, beam) =
 * B * T * beam * 4 bytes.
 * Limits, checked before any launch: 2 <= V <= 1024, 0 <= blank < V, 1 <= beam <= B200S_CTC_DECODE_MAX_BEAM,
 * 1 <= nbest <= beam, 1 <= beam_token <= V - 1, 0 <= order <= B200S_CTC_LM_MAX_ORDER, word_boundary in [0, V) and != blank
 * with an LM, table capacities powers of two, workspace_bytes at least the size above.  Two launches (search, backtrack), no
 * floating-point atomics: results are bit-identical from call to call and do not depend on the other utterances.
 *
 * b200s_ctc_lm_table_build: inserts n entries into an open-addressing table (keys uint64 [capacity], zero-filled by the caller;
 * vals two uint32 per slot): key = the hash of seqs[i, :] (width ints, ended by the first negative one), value = (v0[i], v1[i]
 * or 0).  capacity: a power of two above n.  *status |= 1 when a key is 0 or already present (a 64-bit collision: the caller
 * passes no duplicate sequences), |= 2 when the table is full.  n-gram table: (log10 p, log10 backoff) as fp32 bits; spelling
 * table: (word id, 0). */
#define B200S_CTC_DECODE_MAX_BEAM 128
#define B200S_CTC_LM_MAX_ORDER 5
long long b200s_ctc_decode_workspace_bytes(int B, int T, int beam); /* -1 for bad sizes */
int b200s_ctc_lm_table_build(const int* seqs, int n, int width, const uint32_t* v0, const uint32_t* v1, void* keys, void* vals,
                             long long capacity, int* status, b200s_stream stream);
int b200s_ctc_decode(const void* logits, long long frame_stride, long long batch_stride, const float* lse, const int* input_len,
                     int B, int T, int V, int blank, int beam, int nbest, int beam_token, int word_boundary, const void* lm_keys,
                     const void* lm_vals, long long lm_capacity, const void* spell_keys, const void* spell_vals,
                     long long spell_capacity, int order, int bos, int eos, int unk, int has_unk, float lm_weight,
                     float word_score, float unk_score, void* workspace, long long workspace_bytes, int* tokens, int* lengths,
                     float* scores, b200s_stream stream);

/* ============================ Lexicon-constrained CTC beam search (csrc/ctc_decode_lex.cu) ============================ */
/* b200s_ctc_decode with every word held to a lexicon (flashlight's LexiconDecoder), and the LM look-ahead of partial words in the
 * ranking; the definition is oracle/lexicon_oracle.py.  Everything of b200s_ctc_decode above holds (lp, lae, prefix hash, stays,
 * merges and their order, ranking ties, the backoff LM term, fp32 order of operations, outputs, workspace, limits), with these
 * changes.
 * Lexicon: each word has one or more spellings, sequences of non-blank classes other than word_boundary; the first word in file
 * order keeps a spelling that several words share.  The spellings form a trie whose root (node 0) is the empty partial word.
 * Beam state: the trie node of the partial word in place of its hash (the node is a function of the prefix).
 * Extension of beam j by c in T_K:
 *   c != word_boundary: allowed only if node_j has a child by c, which becomes the beam's node (also for the repeat extension
 *   from pb; the stay pnb + lp[last] keeps the node);
 *   c == word_boundary at the root: the empty word, allowed, scores nothing;
 *   c == word_boundary at a node that ends word w: lm += lm_weight * ln P(w | ctx) + word_score (+ unk_score when w is not in
 *   the LM, whose LM term is then <unk>'s, or 0 without <unk>), the node returns to the root and w (or <unk>) joins the
 *   context.  Without an LM (order = 0) only word_score is added;
 *   c == word_boundary at a node that ends no word: not allowed.
 * Every allowed extension of every beam by every class of T_K is a candidate, with the stays (no min(beam_token, beam + 2)
 * pruning).  Merges: an extension reaching an existing beam's prefix is merged into that beam's stay, as in b200s_ctc_decode.
 * Look-ahead: smear[n] fp32 per node, 0 at the root (trie_smear null: 0 everywhere).  Ranking score =
 * lae(pb, pnb) + (lm + lm_weight * smear[node]), each operation rounded to fp32 in that order; lm holds completed words only.
 * unispeech_b200.lexicon computes smear[n] = max over the words w ending at n or below it of ln P(w | <s>) (w as <unk>, or 0
 * without <unk>, when not in the LM), with ln_prob's order (log10 terms summed in fp32, then * ln 10); 0 without an LM.
 * End of utterance: at a node that ends a word, that word is scored as at a boundary, then lm += lm_weight * ln P(</s> | ctx);
 * at the root only </s>; at a node that ends no word the hypothesis is dropped.  The n-best are the survivors by (score desc,
 * hash asc); entries past them have length 0 and score -inf.
 * Trie arrays (device, nodes in BFS order, the children of a node contiguous and in class order):
 *   trie_mask uint32 [nodes, ceil(V / 32)]  bit c of node n: n has a child by class c;
 *   trie_first_child int32 [nodes]          index of n's first child; its child by c is first_child + (mask bits below c);
 *   trie_word int32 [nodes]                 -1: n ends no word, -2: a word the LM does not know, else the LM word id (any
 *                                           value >= 0 without an LM);
 *   trie_smear fp32 [nodes] or null.
 * b200s_ctc_trie_bytes(nodes, V) = nodes * (4 * ceil(V / 32) + 12).  The kernel trusts the arrays' contents
 * (unispeech_b200.lexicon builds and checks them); null arrays and a node count outside [1, B200S_CTC_TRIE_MAX_NODES] are
 * rejected before any launch, with the checks of b200s_ctc_decode (word_boundary is required).  Candidates per frame:
 * at most beam * (beam_token + 1) <= 128 * 1024, enumerated by index and not stored, so no further limit applies.  Dynamic
 * shared memory: beam * ceil(V / 32) * 10 bytes. */
#define B200S_CTC_TRIE_MAX_NODES (1 << 30)
long long b200s_ctc_trie_bytes(long long nodes, int V); /* -1 for bad sizes */
int b200s_ctc_decode_lexicon(const void* logits, long long frame_stride, long long batch_stride, const float* lse,
                             const int* input_len, int B, int T, int V, int blank, int beam, int nbest, int beam_token,
                             int word_boundary, const void* lm_keys, const void* lm_vals, long long lm_capacity, int order, int bos,
                             int eos, int unk, int has_unk, float lm_weight, float word_score, float unk_score,
                             const uint32_t* trie_mask, const int* trie_first_child, const int* trie_word,
                             const float* trie_smear, long long trie_nodes, void* workspace, long long workspace_bytes,
                             int* tokens, int* lengths, float* scores, b200s_stream stream);

/* ============================ k-means pseudo-labels (csrc/kmeans.cu) ============================ */
/* Nearest-centroid labels, Lloyd updates and k-means++ seeding over bf16 features (the label stage of HuBERT-style pre-training).
 * Centres: fp32 master [K, D]; the bf16 copy the assignment multiplies, [Kp, D] with Kp = K rounded up to a multiple of 256 (rows
 * K..Kp are zeros); cnorm fp32 [Kp] = |bf16 copy|^2.  Limits, checked before any launch: 1 <= K <= B200S_KMEANS_MAX_K, D a
 * positive multiple of 64 (zero-pad narrower features: distances do not change).  No floating-point atomics: every result is
 * bit-identical from call to call.  All pointers are device memory. */
#define B200S_KMEANS_MAX_K 1024
/* labels[b*rows + t] = argmin_k (cnorm[k] - 2 x[b,t] . c_k) (ties to the lowest k), score[...] = that minimum (fp32, NULL to
 * skip), for t < valid[b] (valid: int32 [batches] or NULL = all rows); rows t >= valid[b] get label -1 and no score, and a
 * 128-row band that starts at or past valid[b] is not read.  x: bf16, element (b, t, d) at x[b*x_bs + t*x_rs + d] (x_bs, x_rs
 * multiples of 8, 16-byte aligned base).  prev_labels / changed (both or neither): *changed += number of valid rows whose label
 * differs from prev_labels (int32 atomics; the caller zeroes it). */
int b200s_kmeans_assign(const void* x, long long x_bs, long long x_rs, int rows, int batches, int D, const int* valid,
                        const void* centers, const float* cnorm, int K, int* labels, float* score, const int* prev_labels,
                        int* changed, b200s_stream stream);
/* Bytes of workspace b200s_kmeans_update needs (-1 for bad sizes). */
long long b200s_kmeans_update_workspace(long long n, int K, int D);
/* Per-cluster statistics of n labelled rows (x: bf16 [n, D], row stride x_rs; labels outside [0, K) are skipped):
 * counts[k] (int32), sums[k, :] (fp32, summed in fp64 across fixed pieces), *inertia = sum over labelled rows of |x|^2 + score
 * (fp64; with the scores of b200s_kmeans_assign that is the sum of squared distances to the assigned centres). */
int b200s_kmeans_update(const void* x, long long x_rs, int n, int D, const int* labels, const float* score, int K, void* workspace,
                        long long workspace_bytes, int* counts, float* sums, double* inertia, b200s_stream stream);
/* centers[k] = sums[k] / counts[k] where counts[k] > 0; an empty cluster keeps its centre (sums = counts = NULL: no update).
 * Then writes the bf16 copy centers_bf16 [Kp, D] and cnorm [Kp]. */
int b200s_kmeans_centers(const float* sums, const int* counts, int K, int D, float* centers, void* centers_bf16, float* cnorm,
                         b200s_stream stream);
/* k-means++ seeding over n rows (x: bf16 [n, D], row stride x_rs): centre 0 uniform, centre j drawn with probability
 * d2[i] / sum d2 (fp64 prefix sums, counter-based hash keyed by (seed0, seed1)), d2[i] = min over chosen centres of
 * |x_i - c|^2 (fp32 workspace [n]).  centers: fp32 [K, D] out (copies of the chosen bf16 rows).  *inertia (fp64, may be NULL) =
 * sum d2 with all K centres chosen.  2K + 1 launches, no read-back. */
int b200s_kmeanspp_init(const void* x, long long x_rs, int n, int D, int K, uint32_t seed0, uint32_t seed1, float* d2,
                        float* centers, double* inertia, b200s_stream stream);

/* ============================ on-device data path (csrc/datapath.cu) ============================ */
/* Span masking of compute_mask_indices (WavLM/WavLM.py:35-159; static span length, overlapping spans) on the device, with the
 * library's counter-based RNG instead of numpy's (statistical parity): per row count = max(min_masks, floor(mask_prob sz / L + u)),
 * `count` distinct uniform starts in [0, sz - L), union of the spans, every row trimmed to the batch-minimum number of masked
 * frames.  valid_len: int32 [B] unpadded frames per row, or NULL (all T).  mask: uint8 [B, T] out; counts: int32 [B] workspace.
 * T <= 4096. */
int b200s_span_mask(const int* valid_len, int B, int T, float mask_prob, int mask_length, int min_masks, uint32_t key0,
                    uint32_t key1, uint8_t* mask, int* counts, b200s_stream stream);
/* power[b] += sum_t x[b,t]^2 (fp32 waveforms [B, L], batch stride x_bs; fp64 accumulators zeroed by the caller) */
int b200s_row_power(const float* x, long long x_bs, int B, int L, double* power, b200s_stream stream);
/* Utterance mixing (src/fairseq/data/audio/utterance_mixing_dataset.py:415-432): plan = DEVICE array of B records
 * {int32 c (-1: not mixed), int32 len, int32 c_start, int32 s_start, float snr_db} drawn by the caller;
 * dst[b, s_start + t] += src[c, c_start + t] * sqrt(P_b / (P_c 10^(snr/10))), P = power / L (from b200s_row_power of src). */
int b200s_mix_apply(const float* src, long long bs, int B, int L, const void* plan, const double* power, float* dst,
                    b200s_stream stream);
/* x[b, :n_b] = (x - mean) / sqrt(var + 1e-5) over the row's n_b = valid_len[b] (or L) samples (F.layer_norm(wav, wav.shape),
 * utterance_mixing_dataset.py:433-435,571-573); stats: fp64 [B, 2] zeroed by the caller; plan != NULL: only rows with c >= 0. */
int b200s_row_normalize(float* x, long long bs, int B, int L, const int* valid_len, double* stats, const void* plan,
                        b200s_stream stream);

/* ============================ MFCC features of HuBERT's first iteration (csrc/mfcc.cu) ============================ */
/* torchaudio.compliance.kaldi.mfcc(wav, sample_frequency=16000, use_energy=False) with every other argument at its default,
 * then compute_deltas twice (win_length 5, replicate padding): 13 cepstra, 13 deltas, 13 delta-deltas per 10 ms frame, fp32.
 * wav: fp32 [B, L] (batch stride wav_bs >= L).  n_samples: int32 [B] device, valid samples per utterance, clamped to [0, L];
 * utterance b has Tm_b = 1 + (n - 400) / 160 frames when n >= 400, else none; frame t covers samples [160 t, 160 t + 400).
 * Deltas clamp frame indices to the utterance's own [0, Tm_b - 1] in each pass.  feats: fp32 [B, Tm, 39] (batch stride
 * feats_bs, rows of 39).  rows_bf16: bf16 [B, Tm, 64] (batch stride rows_bs, a multiple of 8; 16-byte aligned) or NULL --
 * columns 0..38 = feats rounded to bf16, 39..63 = 0: the operand b200s_kmeans_assign multiplies.  Frames t >= Tm_b are written
 * as zeros in both outputs.  Tm must equal the frame count of L (Tm = 0, L < 400: nothing is launched).  Two launches, no
 * floating-point atomics: results are bit-identical from call to call and do not depend on the other utterances. */
int b200s_mfcc(const float* wav, long long wav_bs, int L, const int* n_samples, int B, int Tm, float* feats, long long feats_bs,
               void* rows_bf16, long long rows_bs, b200s_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* UNISPEECH_B200_H_ */
