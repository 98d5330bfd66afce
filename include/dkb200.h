/* dkb200 — C ABI of the H100-native denoise + decode engine behind DiffusionKit's
 * `diffusionkit.mlx` DiffusionPipeline / FluxPipeline API.
 *
 * The reference (argmaxinc/DiffusionKit @ 498e5dba) has no FFI boundary: its hot path sits behind a
 * Python class API and bottoms out in MLX library calls.  This header is the boundary a maintainer
 * would bind instead (ctypes stub in INTEGRATION.md).  Each entry point cites the reference code it
 * replaces (paths relative to python/src/diffusionkit/mlx/).
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; dk_last_error() gives the message
 *     (thread-local).  No C++ exception crosses this boundary.
 *   - all pointers are DEVICE pointers unless a name ends in _host; buffers are caller-owned
 *     (torch tensors on the Python side); the library borrows them for the duration of a call
 *     (weights: until the model handle is destroyed).
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous on it.
 *   - dtype: DK_BF16 (FLUX: __init__.py:610) or DK_FP16 (SD3: __init__.py:76) for weights and
 *     activations; sampler state is fp32 (__init__.py:761-788).
 *   - layouts follow the reference: latents/images NHWC (mmdit.py:188-266, vae.py:386-401),
 *     Linear weights (out,in) (mlx nn.Linear), conv weights (O,kh,kw,I) (mlx nn.Conv2d).
 *
 * Why the boundary is at the OPERATOR level (and not dk_mmdit_forward / dk_vae_decode)
 *   The reference's own boundary to its accelerator library is the operator level: mmdit.py / vae.py are
 *   Python modules that call mx.fast.scaled_dot_product_attention, mx.fast.layer_norm, nn.Linear,
 *   nn.Conv2d, nn.GroupNorm one by one; model structure (block lists, which stream skips its post-attention
 *   path, the modulation cache keyed by timestep, the img2img branch) lives in Python and is what its
 *   maintainers edit.  This header replaces exactly that layer — every MLX call on the path has one entry
 *   point here, with the fusions expressed as epilogue/prologue arguments of those calls — so a binding keeps
 *   the reference's module code and swaps its library calls.  A model-level entry point would have to freeze
 *   the parameter-tree naming, six model configurations, the modulation cache and the quirk flags of
 *   SURVEY.md App. A.4 into a C struct.  The cost of staying at the operator level is launch overhead, which
 *   the host layer removes by capturing each forward / decode in a CUDA graph (one cudaGraphLaunch per
 *   MMDiT forward or VAE decode: diffusionkit_b200/mmdit.py, vae.py); a non-Python host does the same with
 *   cudaStreamBeginCapture around its own sequence of dk_* calls — every entry point is capture-safe (no
 *   allocation, no synchronisation, no host-side state beyond the launch counter).
 */
#ifndef DKB200_H
#define DKB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DK_BF16 0
#define DK_FP16 1
#define DK_F32 2 /* dk_resample's fp32 input / output only */

#define DK_ACT_NONE 0
#define DK_ACT_GELU_ERF 1 /* mlx nn.GELU() exact erf — mmdit.py:421,835 */
#define DK_ACT_SILU 2
#define DK_ACT_QUICK_GELU 3 /* x * sigmoid(1.702 x): mlx nn.gelu_fast_approx, CLIP-L "quick_gelu" — clip.py:11 */
#define DK_ACT_GELU_TANH 4  /* 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))), accurate tanhf: SigLIP's
                               "gelu_pytorch_tanh" (FLUX.1 Redux image encoder, DESIGN.md §15) */

typedef struct dk_ctx dk_ctx;

const char* dk_version(void);
const char* dk_last_error(void);
int dk_ctx_create(int device, dk_ctx** out);
void dk_ctx_destroy(dk_ctx* ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
long long dk_ctx_launch_count(dk_ctx* ctx);

/* ---------------------------------------------------------------------------------------------
 * K1  wgmma GEMM with fused epilogue — replaces every nn.Linear on the path
 *     (mmdit.py:471-473 q/k/v, :532 o_proj, :830-835 FFN, :430-435 adaLN, :56-59 context_embedder,
 *      :357-361/:372-376 embedders, :771-774 final linear; vae.py:36-39 attention projections).
 *     out[row(m), n] = res[rrow(m), n] + gate[m / rows_per_batch, n] * act(sum_k A[m,k] W[n,k] + bias[n])
 *     row(m)  = (m / rows_per_batch) * out_batch_rows + out_row_off + m % rows_per_batch
 *     rrow(m) = (m / rows_per_batch) * res_batch_rows + res_row_off + m % rows_per_batch
 *     (the row maps let a stream's GEMM write straight into the joint [text|image] sequence buffer,
 *      mmdit.py:594-625, and let a per-position table broadcast over the batch, mmdit.py:334-349.)
 * ------------------------------------------------------------------------------------------- */
typedef struct dk_gemm_args {
  int dtype;
  int M, N, K;
  const void* A; /* [M, K] row-major, leading dim lda (elements) */
  long long lda;
  const void* W; /* [N, K] row-major (nn.Linear weight), leading dim ldw; if w_n_major: [K, N] */
  long long ldw;
  void* out; /* 16-bit output */
  long long ldc;
  const void* bias; /* [N] or NULL */
  const void* gate; /* [batches, gate_ld] or NULL */
  long long gate_ld;
  const void* res; /* residual or NULL (may alias out) */
  long long ldres;
  int rows_per_batch; /* 0 => M */
  int out_batch_rows, out_row_off;
  int res_batch_rows, res_row_off;
  int act;       /* DK_ACT_* applied to (acc + bias) */
  int w_n_major; /* 1: W is [K, N] row-major (exercises the MN-major operand path used for V) */
  /* fused epilogue for a packed [q | k | v] projection (N = 3 * qk_heads * qk_head_dim), qk_head_dim = 0 disables:
   * per head of the q and k thirds  x = RMSNorm(x; weight, qk_eps)  (mmdit.py:754-764; NULL weight = no norm)
   * then RoPE with table qk_rope[pos][pair] = (cos, sin), pos = out_row_off + m % rows_per_batch (mmdit.py:934-942;
   * NULL = no RoPE).  Replaces a separate dk_qk_norm_rope pass over the QKV buffer. */
  const void* qk_q_weight;
  const void* qk_k_weight;
  const float* qk_rope;
  int qk_heads, qk_head_dim;
  float qk_eps;
} dk_gemm_args;
int dk_gemm(dk_ctx* ctx, const dk_gemm_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K1 with e4m3 operands — the opt-in FP8 form of the MMDiT block linears (mmdit.py:471-473 q/k/v, :532 o_proj,
 *     :830-835 FFN; the reference has no 8-bit path, this trades accuracy for tensor-core rate).
 *     args->A [M, K] and args->W [N, K] hold e4m3 bytes (lda / ldw in elements), quantised per row:
 *     A[m,k] ~ a_scale[m] * e4m3(A)[m,k], W[n,k] ~ w_scale[n] * e4m3(W)[n,k].  args->dtype is the 16-bit type of
 *     out / bias / gate / residual / norm weights.  The epilogue is dk_gemm's with the accumulator replaced by
 *     a_scale[m] * w_scale[n] * sum_k e4m3(A)[m,k] e4m3(W)[n,k]   (a_scale indexed by the A row, before any row map).
 *     K, lda, ldw multiples of 16; w_n_major is not supported; both scale vectors required, 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
int dk_gemm_fp8(dk_ctx* ctx, const dk_gemm_args* args, const float* a_scale, const float* w_scale, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Row quantiser to e4m3 for dk_gemm_fp8 (weights by output feature — the nn.Linear weights of mmdit.py:471-473,
 *     :532, :830-835 — and activations by token).  x: [rows, cols] 16-bit, row stride ldx (elements);
 *     q: [rows, cols] e4m3 bytes, contiguous; q_scale: [rows] fp32.
 *     q_scale[r] = max_c |x[r,c]| / 448 (1 if the row is all zero); q[r,c] = e4m3_rn_satfinite(x[r,c] / q_scale[r]),
 *     evaluated in fp32.  cols, ldx multiples of 8.
 * ------------------------------------------------------------------------------------------- */
int dk_quantize_rows_e4m3(dk_ctx* ctx, int dtype, const void* x, long long ldx, void* q, float* q_scale, int rows,
                          int cols, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K2  LayerNorm (no affine, eps) + adaLN modulate: y = LN(x) * (1 + scale[b]) + shift[b]
 *     replaces affine_transform / mx.fast.layer_norm — mmdit.py:958-972, :838-849.
 *     x, y: [B*rows_per_batch, h]; shift/scale: row b at ptr + b*mod_ld (16-bit).
 * ------------------------------------------------------------------------------------------- */
int dk_ln_modulate(dk_ctx* ctx, int dtype, const void* x, void* y, const void* shift, const void* scale,
                   long long mod_ld, int rows, int rows_per_batch, int h, float eps, void* stream);
/* K2 feeding dk_gemm_fp8 (mmdit.py:958-972 ahead of the q/k/v and fc1 linears): the modulated fp32 row is not rounded
 * to 16 bits but quantised like dk_quantize_rows_e4m3: q [rows, h] e4m3 bytes, q_scale [rows] fp32. */
int dk_ln_modulate_fp8(dk_ctx* ctx, int dtype, const void* x, void* q, float* q_scale, const void* shift,
                       const void* scale, long long mod_ld, int rows, int rows_per_batch, int h, float eps,
                       void* stream);

/* ---------------------------------------------------------------------------------------------
 * QK-RMSNorm (mmdit.py:754-764, eps 1e-6, learned weight) + FLUX RoPE (mmdit.py:934-942) applied
 * in place to the q and k thirds of a packed [rows, 3h] QKV buffer.
 *   rows = B * S; row r -> sequence position r % S.
 *   q_w/k_w: norm weights [d] for positions < split, q_w2/k_w2 for positions >= split (the text and
 *   image streams of a MultiModalTransformerBlock own separate QKNorm modules); NULL => no norm.
 *   rope: fp32 [S, d/2, 2] (cos, sin) or NULL (SD3: no RoPE).
 * ------------------------------------------------------------------------------------------- */
int dk_qk_norm_rope(dk_ctx* ctx, int dtype, void* qkv, int rows, int S, int heads, int d, int split, const void* q_w,
                    const void* k_w, const void* q_w2, const void* k_w2, const float* rope, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K3  attention forward: softmax(scale * Q K^T) V, no mask — replaces
 *     mx.fast.scaled_dot_product_attention (mmdit.py:562-563,643,687-688,736).
 *     qkv: packed [B*S, 3*heads*d] (q | k | v thirds, head-major inside a third).
 *     output row (b, s): s < split -> out0[(b*split + s) * ld0 + head*d ...]
 *                        else      -> out1[(b*(S-split) + s-split) * ld1 + head*d ...]
 *     (split = S with out1 = NULL writes one [B*S, ld0] buffer.)  d in {64, 128}.
 * ------------------------------------------------------------------------------------------- */
int dk_attention_fwd(dk_ctx* ctx, int dtype, const void* qkv, int B, int S, int heads, int d, float scale, int split,
                     void* out0, long long ld0, void* out1, long long ld1, void* stream);

/* ---------------------------------------------------------------------------------------------
 * elementwise / layout kernels on the MMDiT path
 * ------------------------------------------------------------------------------------------- */
/* c[t*B + b, :] = silu(y[b, :] + temb[t, :])  — input of every adaLN Linear (mmdit.py:94-96, :430-431) */
int dk_silu_add(dk_ctx* ctx, int dtype, const void* y, const void* temb, void* c, int n_t, int B, int h, void* stream);
/* act(x) elementwise, 16-bit (MLP embedders: mmdit.py:357-361, :372-376) */
int dk_act(dk_ctx* ctx, int dtype, const void* x, void* y, long long n, int act, void* stream);
/* latent NHWC (B,H,W,C) 16-bit -> patch rows [B*(H/2)*(W/2), 4C].
 * order 0: (c, ph, pw)  FLUX reshape patchify (mmdit.py:292-302)
 * order 1: (ph, pw, c)  SD3 conv k2 s2 im2col, matches weight (O,kh,kw,I) (mmdit.py:285-290) */
int dk_patchify(dk_ctx* ctx, int dtype, const void* latent, void* rows, int B, int H, int W, int C, int order,
                void* stream);
/* rows [B*(H/2)*(W/2), 4C] 16-bit -> NHWC (B,H,W,C) 16-bit.  order 0: FLUX unpack (mmdit.py:304-321);
 * order 1: SD3 unpatchify (p, q, c) (mmdit.py:975-988) */
int dk_unpatchify(dk_ctx* ctx, int dtype, const void* rows, void* latent, int B, int H, int W, int C, int order,
                  void* stream);
/* crop of the learned position table (mmdit.py:334-349): table [max_hw*max_hw, h] -> out [hp*wp, h] */
int dk_pos_embed_crop(dk_ctx* ctx, int dtype, const void* table, void* out, int max_hw, int hp, int wp, int h,
                      void* stream);
/* copy [B, rows, h] blocks into a wider sequence buffer: dst[b, dst_off + r, :] = src[b, r, :] */
int dk_copy_rows(dk_ctx* ctx, int dtype, const void* src, void* dst, int B, int rows, int h, int dst_rows, int dst_off,
                 int src_rows, int src_off, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K6  sampler step (fp32 state) — CFGDenoiser + Euler update, __init__.py:691-719, :775-782,
 *     sampler.py:37-39.
 *   dk_sampler_prepare: xin[(k*B + b)] = cast16(x[b]) for k in 0..reps-1  (reps = 2 when cfg > 0, :700-706)
 *   dk_sampler_step:    den = float(xin) - float(out) * sigma; if cfg: den = den_neg + w (den_text - den_neg)
 *                       x += ((x - den) / sigma) * (sigma_next - sigma)
 *   Higher-order solvers of the same ODE dx/dsigma = (x - D(x, sigma)) / sigma, D = den above (DESIGN.md §11):
 *   dk_sampler_heun_predict: d = (x - D(x, sigma)) / sigma; x2 = x + d * (sigma_next - sigma)   (x unchanged)
 *   dk_sampler_heun_correct: xin / out = forward at (x2, sigma_next), sigma_next != 0:
 *                            d2 = (x2 - D(x2, sigma_next)) / sigma_next; x += (d + d2) / 2 * (sigma_next - sigma)
 *   dk_sampler_dpmpp_2m:     x = a x + b D + c d_prev; d_prev = D   (d_prev not read when c == 0; a, b, c from
 *                            sampler.dpmpp_2m_coefficients)
 *   *_slg: the same updates with skip-layer guidance (DESIGN.md §13); xin / out hold [pos | neg | pos skipping joint
 *          blocks] (reps = 3 in dk_sampler_prepare) and D = D_neg + w (D_pos - D_neg) + slg (D_pos - D_skip).
 *          cfg_weight must be > 0 and slg finite.
 * ------------------------------------------------------------------------------------------- */
int dk_sampler_prepare(dk_ctx* ctx, int dtype, const float* x, void* xin, long long n_per_rep, int reps, void* stream);
int dk_sampler_step(dk_ctx* ctx, int dtype, float* x, const void* xin, const void* out, long long n, float sigma,
                    float sigma_next, float cfg_weight, void* stream);
int dk_sampler_heun_predict(dk_ctx* ctx, int dtype, const float* x, const void* xin, const void* out, float* d,
                            float* x2, long long n, float sigma, float sigma_next, float cfg_weight, void* stream);
int dk_sampler_heun_correct(dk_ctx* ctx, int dtype, float* x, const float* d, const float* x2, const void* xin,
                            const void* out, long long n, float sigma, float sigma_next, float cfg_weight, void* stream);
int dk_sampler_dpmpp_2m(dk_ctx* ctx, int dtype, float* x, float* d_prev, const void* xin, const void* out, long long n,
                        float sigma, float a, float b, float c, float cfg_weight, void* stream);
int dk_sampler_step_slg(dk_ctx* ctx, int dtype, float* x, const void* xin, const void* out, long long n, float sigma,
                        float sigma_next, float cfg_weight, float slg, void* stream);
int dk_sampler_heun_predict_slg(dk_ctx* ctx, int dtype, const float* x, const void* xin, const void* out, float* d,
                                float* x2, long long n, float sigma, float sigma_next, float cfg_weight, float slg,
                                void* stream);
int dk_sampler_heun_correct_slg(dk_ctx* ctx, int dtype, float* x, const float* d, const float* x2, const void* xin,
                                const void* out, long long n, float sigma, float sigma_next, float cfg_weight, float slg,
                                void* stream);
int dk_sampler_dpmpp_2m_slg(dk_ctx* ctx, int dtype, float* x, float* d_prev, const void* xin, const void* out,
                            long long n, float sigma, float a, float b, float c, float cfg_weight, float slg,
                            void* stream);
/* Stochastic samplers (Euler ancestral, DPM-Solver++(2M) SDE; DESIGN.md §16), one step of B images of n_per_image
 * elements each: x = a x + b D + c d_prev + noise z, then d_prev = D.  a, b, c, noise from
 * sampler.euler_ancestral_coefficients / dpmpp_2m_sde_coefficients (Lu et al. 2022, data-prediction SDE solver; the
 * rectified-flow ancestral step).  reps 1 (no CFG), 2 (CFG) or 3 (CFG + skip-layer guidance, slg the scale): D as in the
 * updates above.  d_prev NULL: neither read nor written (then c must be 0); d_prev is not read when c == 0.
 * z of element e of image b at solver step `step`: (v0..v3) = Philox4x32-10(counter (e / 4, step, 0, 0),
 * key (lo32(seeds[b]), hi32(seeds[b]))), u_j = ((v_j >> 9) + 0.5) 2^-23, Box-Muller (sqrtf(-2 logf u), sincospif(2 u'))
 * on (u0, u1) for e % 4 in {0, 1} and on (u2, u3) for {2, 3}: independent of B, the image's batch position and reps.
 * noise == 0 draws nothing (seeds may be NULL) and computes what dk_sampler_dpmpp_2m computes, bit for bit.
 * n_per_image % 4 == 0; x, d_prev, xin, out 16-byte aligned; seeds a device array of B values. */
int dk_sampler_sde_step(dk_ctx* ctx, int dtype, float* x, float* d_prev, const void* xin, const void* out,
                        long long n_per_image, int B, int reps, float sigma, float a, float b, float c, float noise,
                        float cfg_weight, float slg, const uint64_t* seeds, int step, void* stream);
/* Masked inpainting (DESIGN.md §17), run after each solver step to sigma: at every position hw whose mask[hw] == 0
 * (kept), x[b, hw, :] = a * eps[b, hw, :] + b * x0[b, hw, :] with a = sigma, b = 1 - sigma, rounded as dk_axpby_f32
 * rounds it (fma(a, eps, b * x0)); positions with mask[hw] != 0 (repainted) are neither read nor written.
 * x, eps, x0 fp32 (B, HW, C), 16-byte aligned, C % 4 == 0; mask uint8 (HW), shared by the B images. */
int dk_inpaint_blend(dk_ctx* ctx, float* x, const float* eps, const float* x0, const uint8_t* mask, int B, long long HW,
                     int C, float a, float b, void* stream);
/* y = x * a + b (fp32): latent_format.process_out (__init__.py:732-733) and noise scaling (sampler.py:41-42) */
int dk_axpb_f32(dk_ctx* ctx, const float* x, float* y, long long n, float a, float b, void* stream);
/* ---- text encoders (SURVEY.md §8 row f2): CLIP-L/G (mlx/clip.py) and the T5-XXL encoder (mlx/t5.py) ------------- */
/* out[i] = table[ids[i]] (+ pos[i % pos_len]); table [vocab, d], pos [pos_len, d] or NULL   (clip.py:97-98, t5.py:322) */
int dk_embedding(dk_ctx* ctx, int dtype, const void* table, const int* ids, const void* pos, void* out, long long n,
                 int d, int vocab, int pos_len, void* stream);
/* y = LN(x) * weight + bias, biased variance, fp32 statistics (mlx nn.LayerNorm; clip.py:32-33,78) */
int dk_layernorm(dk_ctx* ctx, int dtype, const void* x, void* y, const void* weight, const void* bias, int rows, int h,
                 float eps, void* stream);
/* T5 RMSNorm over the fp32 residual stream: y = (dtype)(weight * x * rsqrt(mean(x^2) + eps))   (t5.py:150-170) */
int dk_rmsnorm_f32(dk_ctx* ctx, int dtype, const float* x, const void* weight, void* y, int rows, int d, float eps,
                   void* stream);
/* x (fp32) += y (16-bit): T5 keeps the residual stream in fp32 (t5.py:214-221) */
int dk_add_f32_16(dk_ctx* ctx, int dtype, float* x, const void* y, long long n, void* stream);
/* out[r, f] = gelu_erf(h[r, f]) * h[r, F + f], h [rows, 2F] = x @ [wi_0 | wi_1]^T   (t5.py:195-199) */
int dk_glu_gelu(dk_ctx* ctx, int dtype, const void* h, void* out, long long rows, int F, void* stream);
/* short-sequence attention (S <= 512, head dim 64) over a packed (q | k | v) projection [B*S, 3*heads*64]:
 * out = softmax(scale * q k^T + rel_bias[head][j - i + S - 1] + (causal ? -6e4 * [j > i] : 0)) v
 * rel_bias [heads, 2S-1] 16-bit or NULL (T5 relative-position bias, t5.py:21-102); causal: CLIP mask (clip.py:84-90) */
int dk_attention_small(dk_ctx* ctx, int dtype, const void* qkv, const void* rel_bias, void* out, int B, int S, int heads,
                       int head_dim, float scale, int causal, void* stream);
/* MLX affine 4-bit Linear weights -> dense 16-bit (the `*-4bit-quantized` model versions, reference
 * mlx/model_io.py:728-734, 772-775: nn.quantize with MLX defaults group_size 64, bits 4).
 * wq [N, K/8] uint32 (8 nibbles per word, element 0 in the low bits); scales, biases [N, K/group_size] 16-bit;
 * out[n, k] = scales[n, k/group] * q[n, k] + biases[n, k/group]  (one fp32 FMA, rounded once to `dtype`) */
int dk_dequant_q4(dk_ctx* ctx, int dtype, const uint32_t* wq, const void* scales, const void* biases, void* out,
                  long long N, int K, int group_size, void* stream);
/* read_image (__init__.py:536-551): uint8 [pixels, src_channels >= 3] -> 16-bit [pixels, cpad]; channels 0..2 =
 * u8 / 255 * 2 - 1, the padding channels are zero */
int dk_image_pre(dk_ctx* ctx, int dtype, const uint8_t* img, void* out, long long pixels, int src_channels, int cpad,
                 void* stream);
/* FLUX.1 Fill's masked image (DESIGN.md §18): dk_image_pre of one uint8 (H, W, src_channels >= 3) image into 16-bit
 * (H, W, cpad), except that every pixel with mask[p] != 0 (uint8 (H, W)) is +0 in every channel.  Kept pixels round
 * exactly as dk_image_pre rounds them.  H, W positive multiples of 16; out 16-byte aligned; cpad % 8 == 0. */
int dk_image_pre_masked(dk_ctx* ctx, int dtype, const uint8_t* img, const uint8_t* mask, void* out, int H, int W,
                        int src_channels, int cpad, void* stream);
/* FLUX.1 Fill's conditioning rows (DESIGN.md §18): lat (N, 64) 16-bit packed masked-image latent rows, N = (H/16)(W/16)
 * tokens, and the uint8 (H, W) pixel mask -> out (N, 320) = [lat | mask channels].  Mask channel c * 4 + ph * 2 + pw,
 * c = ph1 * 8 + pw1, of token (h, w) is 1 when mask[(2h + ph) * 8 + ph1, (2w + pw) * 8 + pw1] != 0, else 0.
 * H, W positive multiples of 16; lat and out 16-byte aligned and contiguous. */
int dk_fill_cond_rows(dk_ctx* ctx, int dtype, const void* lat, const uint8_t* mask, void* out, int H, int W,
                      void* stream);
/* FLUX.1 Canny's edge map (DESIGN.md §19): OpenCV's cv2.Canny(lut[img], low, high) (L1 gradient, 3 x 3 Sobel,
 * replicated borders, the channel of largest |dx| + |dy|, exact 8-connected hysteresis) of channels 0-2 of a uint8
 * (H, W, src_channels >= 3) image, each value first mapped through the 256-entry uint8 table lut -> out uint8 (H, W, 3),
 * 255 on edges and 0 elsewhere in all three channels.  A candidate has magnitude > low, a strong pixel > high;
 * 0 <= low <= high.  ws: DK_CANNY_WS_BYTES_PER_PIXEL * H * W bytes, 16-byte aligned.  H * W < 2^31.  Five launches. */
#define DK_CANNY_WS_BYTES_PER_PIXEL 10
int dk_canny(dk_ctx* ctx, const uint8_t* img, const uint8_t* lut, uint8_t* out, void* ws, int H, int W,
             int src_channels, int low, int high, void* stream);
/* FLUX.1 Redux's SigLIP patch embedding (DESIGN.md §15): uint8 NHWC [B, H, W, src_channels >= 3] -> 16-bit patch rows
 * [B * (H/p) * (W/p), kp] of the stride-p, p x p convolution without padding (the last H % p rows and W % p columns are
 * dropped).  Column k < 3p^2 holds channel k % 3 of pixel (k / 3p, (k / 3) % p) of the patch, normalised like
 * dk_image_pre (u8 / 255 * 2 - 1, SigLIP's (x / 255 - 0.5) / 0.5); columns 3p^2 .. kp are zero.  kp % 8 == 0, so the
 * rows feed dk_gemm with the conv weight permuted to (O, kh, kw, c) and zero-padded to kp. */
int dk_image_patches(dk_ctx* ctx, int dtype, const uint8_t* img, void* out, int B, int H, int W, int src_channels,
                     int p, int kp, void* stream);
/* FLUX.1 Depth's depth estimator (DESIGN.md §20, csrc/depth.cu).
 * dk_resample: separable linear resampling of an NHWC map in [Hi, Wi, C] -> out [Ho, Wo, C] through per-axis tap tables:
 *   out(y, x, c) = sum_t wy[y * ty + t] * sum_u wx[x * tx + u] * in(y0[y] + t, x0[x] + u, c), in fp32.  y0 int32 [Ho],
 *   wy fp32 [Ho * ty], x0 int32 [Wo], wx fp32 [Wo * tx] (device), every index y0[y] + t in [0, Hi) (x likewise).
 *   in_dtype / out_dtype: DK_BF16, DK_FP16 or DK_F32.  mode 0 writes the map; mode 1 (C == 1) writes BFL's
 *   v / 127.5 - 1 to all three channels of out [Ho, Wo, 3].  1 <= ty, tx <= 64.  One launch. */
int dk_resample(dk_ctx* ctx, int in_dtype, int out_dtype, const void* in, void* out, int Hi, int Wi, int C, int Ho,
                int Wo, const int* y0, const float* wy, int ty, const int* x0, const float* wx, int tx, int mode,
                void* stream);
/* sum = a + b (b null: a) rounded to 16 bits, relu = max(sum, 0); sum or relu may be null, either may alias a.  n
 * elements.  The DPT residual units' pre-activations and fusion sums.  One launch. */
int dk_depth_add_relu(dk_ctx* ctx, int dtype, const void* a, const void* b, void* sum, void* relu, long long n,
                      void* stream);
/* Depth Anything's head tail: out[p] = max(sum_k w[k] * max(x[p, k], 0) + b, 0) in fp32, summed in channel order with
 * every product and sum rounded; x 16-bit [pixels, C], w fp32 [C] (device), out fp32 [pixels].  One launch. */
int dk_depth_head(dk_ctx* ctx, int dtype, const void* x, const float* w, float b, float* out, long long pixels, int C,
                  void* stream);
/* out = a * x + b * y (fp32): img2img noise scaling sigma * noise + (1 - sigma) * latent (sampler.py:41-42) */
int dk_axpby_f32(dk_ctx* ctx, const float* x, const float* y, float* out, long long n, float a, float b, void* stream);
/* VAE-encoder posterior sample + process_in: hidden [pixels, 2C] 16-bit = (mean | logvar);
 * out = ((mean + exp(0.5 * clip(logvar, -30, 20)) * noise) - shift) * scale   (__init__.py:586-594, :729-730) */
int dk_vae_sample_latent(dk_ctx* ctx, int dtype, const void* hidden, const float* noise, float* out, long long pixels,
                         int C, float shift, float scale, void* stream);
/* fp32 <-> 16-bit casts */
int dk_cast_f32_to_16(dk_ctx* ctx, int dtype, const float* x, void* y, long long n, void* stream);
int dk_cast_16_to_f32(dk_ctx* ctx, int dtype, const void* x, float* y, long long n, void* stream);
/* First-block step cache (opt-in, MMDiT.set_step_cache).  Over nseq sequences of `rows` rows of width h:
 *     r = fp32(x) - fp32(base), row r of sequence s at x + (s * x_seq_rows + r) * ldx (base likewise);
 * r_out [nseq * rows, h] fp32 or NULL receives r; with prev [nseq * rows, h] fp32, sums [nseq, 2] fp32 receives
 * (sum |r - prev|, sum |prev|) per sequence, reduced in a fixed order without atomics (two launches are bit-identical);
 * ws is scratch of nseq * 512 floats.  prev NULL: no sums (store only).  16-byte aligned x, base, r_out, prev. */
int dk_residual_delta(dk_ctx* ctx, int dtype, const void* x, long long ldx, int x_seq_rows, const void* base,
                      long long ldb, int b_seq_rows, float* r_out, const float* prev, float* sums, float* ws, int nseq,
                      int rows, int h, void* stream);
/* out = round16(x + r), x and out 16-bit, r fp32, n elements (one fp32 add, one rounding); out may alias x */
int dk_residual_apply(dk_ctx* ctx, int dtype, const void* x, const float* r, void* out, long long n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * VAE decoder kernels (vae.py:20-149, 336-401)
 * ------------------------------------------------------------------------------------------- */
/* K7a GroupNorm statistics (nn.GroupNorm(32, C, pytorch_compatible=True), eps 1e-5; vae.py:34,72,78):
 *     stats[(b*G + g)*2 + {0,1}] = mean, rstd over (H*W, C/G); x NHWC 16-bit.
 *     ws: scratch of dk_groupnorm_ws_floats(B, G) floats (two-stage deterministic reduction, no atomics). */
int dk_groupnorm_ws_floats(int B, int G);
int dk_groupnorm_stats(dk_ctx* ctx, int dtype, const void* x, float* stats, float* ws, int B, int HW, int C, int G,
                       float eps, void* stream);
/* GroupNorm apply (+ optional SiLU): y = act((x - mean) * rstd * gamma[c] + beta[c]) */
int dk_groupnorm_apply(dk_ctx* ctx, int dtype, const void* x, void* y, const float* stats, const void* gamma,
                       const void* beta, int B, int HW, int C, int G, int silu, void* stream);
/* K7  conv 3x3, stride 1, zero pad 1, NHWC, as an im2col-free implicit GEMM: the 9 taps are 9 shifted TMA
 *     boxes of the input (out-of-bounds = zero fill = the padding), accumulated in registers (wgmma).
 *     x [B,H,W,Cin] (Cin % 64 == 0), w [Cout,3,3,Cin] (Cout % 8 == 0), bias [Cout], res NHWC [B,H,W,Cout] or NULL
 *     (the ResnetBlock2D skip, vae.py:99).  replaces nn.Conv2d 3x3 (vae.py:73-81,134-136,349-351,384) */
int dk_conv3x3(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, const void* res, void* out,
               int B, int H, int W, int Cin, int Cout, void* stream);
/* 3x3 convolution with stride 2 and mlx's (0,1),(0,1) bottom/right zero padding — the VAE encoder's downsample
 * (vae.py:130-132,142-144).  x [B,H,W,Cin] (H, W even) -> out [B,H/2,W/2,Cout].  Same TMA implicit GEMM; the tap tile is
 * a 4-D box traversed with element stride 2. */
int dk_conv3x3_s2(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, void* out, int B, int H, int W,
                  int Cin, int Cout, void* stream);
/* 3x3 convolution with stride 2 and one pixel of zero padding on every side (PyTorch's Conv2d(3, stride=2, padding=1),
 * Depth Anything's DPT downsample, DESIGN.md §20).  x [B,H,W,Cin] (any H, W) -> out [B,ceil(H/2),ceil(W/2),Cout]: output
 * pixel (y, x) reads input rows 2y - 1 .. 2y + 1; the TMA unit zero-fills the taps outside the image. */
int dk_conv3x3_s2_p1(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, void* out, int B, int H,
                     int W, int Cin, int Cout, void* stream);
/* K7f fused ResNet-path convolution (csrc/conv_fused.cu): [GroupNorm-apply + SiLU on the input] -> [nearest 2x] ->
 *     conv 3x3 (+ bias, + skip) -> output AND the GroupNorm partial statistics of the output, in ONE kernel.
 *     replaces nn.GroupNorm + nn.SiLU + nn.Conv2d (+ skip) of ResnetBlock2D (vae.py:60-101) and
 *     upsample_nearest + nn.Conv2d of the upsample stages (vae.py:20-25,146-147).
 *     x NHWC [B,H,W,Cin] RAW (pre-norm); gn_stats [B,G,2] (mean, rstd) + gamma/beta [Cin] normalise it on the fly while
 *     the 64-channel halo tile sits in shared memory (NULL: no norm); silu != 0 applies x*sigmoid(x) after the affine.
 *     up == 0: w [Cout,3,3,Cin], out [B,H,W,Cout].   up == 1: conv3x3(nearest2x(x)) by sub-pixel phases,
 *     w = the phase weights made by dk_conv_up_weights [4*Cout, 4*Cin], out [B,2H,2W,Cout].  res like out, or NULL.
 *     out_partial [B, slots, out_G, 2], slots = output pixels / 128: (sum, sum of squares) of the STORED output per
 *     128-pixel row segment and channel group, folded by dk_groupnorm_finalize (NULL: not wanted).
 *     Shapes: W % 128 == 0, H % 4 == 0, Cin % 64 == 0 (<= 512), Cout % 128 == 0 — dk_conv_fused_supported says. */
int dk_conv_fused_supported(int H, int W, int Cin, int Cout);
int dk_conv3x3_fused(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, const void* res, void* out,
                     int B, int H, int W, int Cin, int Cout, int up, const float* gn_stats, const void* gamma,
                     const void* beta, int G, int silu, float* out_partial, int out_G, void* stream);
/* Phase weights of conv3x3(nearest2x(.)): w [Cout,3,3,Cin] -> wp [4][Cout][2x2][Cin]; the 3x3 taps that fall on the
 * same source pixel are added in fp32 and rounded once (2.25x fewer FLOPs than convolving the upsampled tensor). */
int dk_conv_up_weights(dk_ctx* ctx, int dtype, const void* w, void* wp, int Cout, int Cin, void* stream);
/* Second stage of the GroupNorm statistics: partial [B, slots, G, 2] (sum, sumsq) -> stats [B, G, 2] (mean, rstd);
 * count = elements per (image, group).  Deterministic (fixed order, double accumulation). */
int dk_groupnorm_finalize(dk_ctx* ctx, const float* partial, float* stats, int B, int G, int slots, double count,
                          float eps, void* stream);
/* nearest 2x upsample NHWC (vae.py:20-25) */
int dk_upsample_nearest2x(dk_ctx* ctx, int dtype, const void* x, void* y, int B, int H, int W, int C, void* stream);
/* row softmax in place: x[r, :n] = softmax(scale * x[r, :n]); fp32 math, 16-bit storage (vae.py:49-52) */
int dk_softmax_rows(dk_ctx* ctx, int dtype, void* x, long long rows, int n, long long ld, float scale, void* stream);
/* clip(x/2 + 0.5, 0, 1) (and optional trunc(x*255) -> uint8): __init__.py:583, :526.
 * x NHWC [.., C_in_stride] 16-bit, takes the first 3 channels. */
int dk_image_post(dk_ctx* ctx, int dtype, const void* x, int c_stride, float* img_f32, uint8_t* img_u8, long long pixels,
                  void* stream);
/* Inpainting paste-back (DESIGN.md §17): img uint8 (B, pixels, 3) in place; every pixel p with mask[p] == 0 becomes
 * src[p] (uint8 (pixels, 3)), bit for bit; the others are not touched.  pixels % 4 == 0; img, src, mask 4-byte aligned. */
int dk_inpaint_paste(dk_ctx* ctx, uint8_t* img, const uint8_t* src, const uint8_t* mask, int B, long long pixels,
                     void* stream);

/* ---------------------------------------------------------------------------------------------
 * one-time weight broadcast for multi-GPU batch sharding (no per-step collective).
 * The Python host uses torch.distributed (NCCL) for the rendezvous; these are thin NCCL wrappers
 * for hosts without torch.
 * ------------------------------------------------------------------------------------------- */
int dk_comm_unique_id(uint8_t id_host[128]);
int dk_comm_init(dk_ctx* ctx, int rank, int world, const uint8_t id_host[128]);
int dk_comm_broadcast(dk_ctx* ctx, void* ptr, size_t bytes, int root, void* stream);
int dk_comm_destroy(dk_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* DKB200_H */
