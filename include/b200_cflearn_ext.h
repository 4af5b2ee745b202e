/* b200_cflearn_ext.h -- entry points of libb200_cflearn.so added after version 4 of include/b200_cflearn.h.
 *
 * The same library exports them, under the conventions of b200_cflearn.h: C99, plain device pointers plus sizes plus a stream,
 * 0 or a negative B200_ERR_* status, b200_last_error() for the reason of a refusal, every argument checked before anything is
 * launched or a tensor map is encoded.  Include b200_cflearn.h first.
 */
#ifndef B200_CFLEARN_EXT_H_
#define B200_CFLEARN_EXT_H_

#include "b200_cflearn.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------------------
 * Resampling convolutions of the SD-v1.5 UNet (cflearn/modules/core/convs/residual.py:86-151 with use_conv, 2-D signals,
 * padding 1), on channels-last bf16 activations, as implicit GEMMs on the main loop of b200_conv3x3_nhwc_bf16: every
 * (tap, 64-channel) k-block is one TMA box of the activation, its halo zero-filled by the TMA unit.  Weights are packed
 * [Cout, 9 * Cin], k = (ky * 3 + kx) * Cin + ci, as for b200_conv3x3_nhwc_bf16.
 *
 * Geometry: H and W are the sizes of the lower-resolution side (the input of the stride-2 convolution is H x W and its output
 * H/2 x W/2; the upsampling convolution's input is H x W and its output 2H x 2W).  Write h x w for the grid the GEMM tiles:
 * H/2 x W/2 for the stride-2 convolution and its input gradient, H x W for the upsampling convolution.  Then w divides 128 and
 * h is a multiple of 128 / w (or h * w divides 128), the rule of b200_conv3x3_nhwc_bf16; the upsampling convolution also takes
 * a w of 128 times a power of 2, as that entry does (the KL-f8 decoder's 128 -> 256 and 256 -> 512).  The weight gradient needs, on its
 * h x w grid, w dividing 64 and h * w a multiple of 64.  Channel counts: the reduction's channels (Cin of a forward, Cout of an
 * input gradient) are a multiple of 64, the output's a multiple of 8.  Sizes are positive; H and W of the stride-2 entries
 * are even.  The six resampling layers of SD-v1.5 at 512 px (H x W, Cin = Cout: 64 x 64 / 320, 32 x 32 / 640, 16 x 16 / 1280
 * down; 8 x 8 / 1280, 16 x 16 / 1280, 32 x 32 / 640 up) fit at every batch size.
 * --------------------------------------------------------------------------------------------------------- */

/* ResDownsample: 3x3 convolution with stride 2, zero padding 1.  x [B, H, W, Cin]; out0 / aux rows [B * H/2 * W/2, ldo].
 * Each k-block is one box of x with element strides 2, shifted by its tap.  epilogue and bias as b200_conv3x3_nhwc_bf16:
 * B200_EPI_BIAS_BF16, B200_EPI_BIAS_RESID_F32, B200_EPI_BIAS_ADD_PER_IMAGE_BF16 (aux bf16 [B, ldo]; with bias NULL and every
 * row of aux the bias this is eager's bf16(bf16(conv) + bias)) or B200_EPI_BIAS_RESID_CLAMP_BF16. */
int b200_conv3x3_s2_nhwc_bf16(const void* x, const void* w_packed, const void* bias, void* out0, const void* aux, long long ldo,
                              int B, int H, int W, int Cin, int Cout, int epilogue, cudaStream_t stream);

/* Its input gradient: dx [B, H, W, Cin] (dense) from dy [B, H/2, W/2, Cout] (dense).  No zero insertion: the pixels of dx fall
 * into four (row, column) parity classes, and class (py, px) is a stride-1 implicit GEMM over dy with 1, 2, 2 or 4 taps whose
 * output rows go to that class's pixels; the MMAs are those of the forward.  w_dgrad: bf16 [Cin, 9 * Cout], for the classes
 * (0, 0), (0, 1), (1, 0), (1, 1) in turn, each of its taps (ky, kx) in row-major order -- ky in {1} for py = 0 and {0, 2} for
 * py = 1, kx likewise with px -- as Cout columns w[co][ci][ky][kx]. */
int b200_conv3x3_s2_dgrad_nhwc_bf16(const void* dy, const void* w_dgrad, void* dx, int B, int H, int W, int Cin, int Cout,
                                    cudaStream_t stream);

/* Its weight gradient: ONE split-K GEMM with M = Cout, N = 9 * Cin, K = B * H/2 * W/2 (dy MN-major, x read through the
 * per-tap boxes with element strides 2).  dy: bf16 rows [B * H/2 * W/2, ld_dy]; partials: f32 [splits][Cout][9 * Cin] in the
 * packed weight layout (finish with b200_splitk_reduce). */
int b200_conv3x3_s2_wgrad_nhwc_bf16(const void* dy, long long ld_dy, const void* x, void* partials, int B, int H, int W, int Cin,
                                    int Cout, int splits, cudaStream_t stream);

/* ResUpsample: nearest 2x upsampling and a 3x3 / padding 1 convolution in one GEMM, no upsampled copy written.  x [B, H, W, Cin];
 * out0 / aux rows [B * 2H * 2W, ldo].  Output parity class (py, px) reads, for tap (ky, kx), x shifted by
 * (floor((py + ky - 1) / 2), floor((px + kx - 1) / 2)), so the products are those of the convolution of the upsampled image.
 * epilogue and bias as b200_conv3x3_s2_nhwc_bf16 (aux of B200_EPI_BIAS_ADD_PER_IMAGE_BF16: bf16 [B, ldo]). */
int b200_conv3x3_up2_nhwc_bf16(const void* x, const void* w_packed, const void* bias, void* out0, const void* aux, long long ldo,
                               int B, int H, int W, int Cin, int Cout, int epilogue, cudaStream_t stream);

/* Nearest 2x upsampling, an exact copy: out [B, 2H, 2W, C] (dense) from x [B, H, W, C] (dense); C % 8 == 0. */
int b200_upsample_nearest2x_bf16(const void* x, void* out, int B, int H, int W, int C, cudaStream_t stream);

/* Its backward: out[b, y, x, c] = bf16(the fp32 sum of x[b, 2y + i, 2x + j, c] over (i, j) = (0, 0), (0, 1), (1, 0), (1, 1)),
 * out [B, H, W, C] (dense) from x [B, 2H, 2W, C] (dense); C % 8 == 0. */
int b200_sum2x2_bf16(const void* x, void* out, int B, int H, int W, int C, cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The two ends of the SD-v1.5 UNet's training step (cflearn/modules/multimodal/diffusion/unet.py:215-275 and
 * cflearn/models/cv/diffusion.py:44-94).
 * --------------------------------------------------------------------------------------------------------- */

/* Channel padding: out [B, H, W, Cp] bf16 (dense, channels-last) from x [B, C, H, W], channels >= C set to +0.  x is fp32
 * (x_f32 = 1, rounded to nearest even) or bf16 (copied bit for bit), dense NCHW (x_channels_last = 0) or dense channels-last
 * (1).  0 < C <= Cp, Cp % 8 == 0, H * W < 2^31, B * H * W * Cp <= 2^38.  The 4-channel stem and head run on the 64-channel
 * convolutions through it. */
int b200_pad_channels_bf16(const void* x, int x_f32, int x_channels_last, void* out, int B, int C, int H, int W, int Cp,
                           cudaStream_t stream);

/* The DDPM noise-prediction loss at DDPMStep's defaults (l2, eps parameterization, l_simple_weight 1, log_var 0, no ELBO
 * term): mean over b of (mean over the N = C H W elements of image b of (pred - noise)^2).  pred: bf16, noise: fp32
 * (noise_f32 = 1) or bf16, both [B, N] rows (the images of NCHW and of channels-last tensors alike), in the same layout.  Give
 * exactly one of
 *   loss (fp32 [1]): the loss, in a fixed order (one CTA: per-image partials, then their mean), bit-identical run to run;
 *   dpred (bf16 [B, N], pred's layout) with grad_out (fp32 [1] on the device, the loss's upstream gradient): the gradient with
 *   eager's fp32 operations, bf16(fl(2 fl(pred - noise)) fl(fl(grad_out fl(1/B)) fl(1/N))).
 * B * N <= 2^38.  Each call is one launch. */
int b200_noise_prediction_loss_bf16(const void* pred, const void* noise, int noise_f32, float* loss, void* dpred,
                                    const float* grad_out, int B, long long N, cudaStream_t stream);

/* DDPM noising fused into the stem's input (q_sample, cflearn/modules/multimodal/diffusion/samplers/schema.py:94-108, before the
 * stem's autocast cast): out [B, H, W, Cp] bf16 (dense, channels-last) with, for channel c < C of image b and t = timesteps[b],
 * bf16(fl(fl(sqrt_alphas_cumprod[t] x0) + fl(sqrt_one_minus_alphas_cumprod[t] noise))) -- two fp32 products and their fp32 sum,
 * no contraction -- and channels >= C set to +0.  x0, noise: fp32 [B, C, H, W], both dense NCHW (channels_last = 0) or both
 * dense channels-last (1); timesteps: int64 [B]; the two tables: fp32 [T].  A timestep outside [0, T) reads no table entry: it
 * sets *bad_flag = 1 (int32, never cleared here) and the image's channels < C are NaN.  0 < C <= Cp, Cp % 8 == 0, H * W < 2^31,
 * B * H * W * Cp <= 2^38.  One launch, on the pad_channels kernel. */
int b200_q_sample_pad_bf16(const float* x0, const float* noise, int channels_last, const long long* timesteps,
                           const float* sqrt_alphas_cumprod, const float* sqrt_one_minus_alphas_cumprod, long long T, int* bad_flag,
                           void* out, int B, int C, int H, int W, int Cp, cudaStream_t stream);

/* One DDIM denoising step (DDIMSampler, cflearn/modules/multimodal/diffusion/samplers/ddim.py:195-239, with the classifier-free
 * guidance of samplers/schema.py:215-255), which also writes the stem's input for the next step.  step = *step_dev (int32, only
 * read by the step) picks coef[step] = {s1m, sqrt_a, sqrt_ap, c_dir, sigma} (fp32 [S, 5]) and for every element, with e the
 * bf16 eps (dense channels-last [B, H, W, C], UNetDiffuserB200's output layout):
 *   guided (eps_uncond, the same layout, given and guidance_scale != 1):  e = bf16(u + bf16(scale bf16(e - u))), u = eps_uncond;
 *   x <- ((sqrt_ap ((x - s1m e) / sqrt_a)) + c_dir e) + (sigma noise) temperature
 * in fp32, every operation rounded, no contraction.  x and noise: fp32 [B, C, H, W], dense NCHW; x is updated in place.  When
 * step + 1 < S: next_in (bf16 [copies B, H, W, Cp], dense) gets bf16(x) in channels < C and +0 in channels C..Cp of each of its
 * copies (1 or 2; 2 needs eps_uncond), and next_ts (int64 [copies B]) gets ts_table[step + 1] (ts_table: int64 [S]).  A counter
 * outside [0, S) reads no table entry: it sets *bad_flag = 1 (never cleared here), x becomes NaN and nothing else is written.
 * increment = 1 then adds 1 to *step_dev in a second, one-thread launch.  0 < C <= Cp, Cp % 8 == 0, H * W < 2^31,
 * 2 B * H * W * Cp <= 2^38. */
int b200_ddim_step_bf16(const void* eps, const void* eps_uncond, float guidance_scale, float* x, const float* noise, const float* coef,
                        const long long* ts_table, int S, float temperature, int* step_dev, int increment, int* bad_flag,
                        void* next_in, long long* next_ts, int copies, int B, int C, int H, int W, int Cp, cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * AdamW on the flat fp32 arenas (torch.optim.AdamW without amsgrad; the zoo's DDPM trains with "adamw",
 * cflearn/optimizers.py:31): b200_adam_step / b200_adam_step_dev with decoupled weight decay, in torch.optim.AdamW's order:
 * p <- p (1 - lr weight_decay) first, then the Adam update with no L2 term in the gradient.  Same arguments, rules and device
 * hyper block {lr, beta1, beta2, eps, weight_decay, grad_scale} (grad_scale multiplies the gradient) as the Adam entries.
 * --------------------------------------------------------------------------------------------------------- */
int b200_adamw_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n, float lr, float beta1,
                    float beta2, float eps, float weight_decay, int step, int* step_dev, cudaStream_t stream);
int b200_adamw_step_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n, const float* hyper_dev,
                        int* step_dev, int increment, cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Row softmax of the KL-f8 autoencoder's single-head SpatialAttention (cflearn/modules/core/attentions.py:330-370, sdp_attn
 * with one head of width C over the H * W pixels), between the GEMMs S = Q K^T (fp32 out) and O = P V:
 *   p[r][c] = bf16( exp(scale (s[r][c] - m_r)) / l_r ),  m_r = max_c s[r][c],  l_r = sum_c exp(scale (s[r][c] - m_r))
 * in fp32, every row reduced in a fixed order (bit-identical run to run).  s: fp32 [rows, lds]; p: bf16 [rows, ldp];
 * rows, cols > 0, lds >= cols, ldp >= cols, scale > 0 and finite.  One launch.
 * --------------------------------------------------------------------------------------------------------- */
int b200_softmax_rows_bf16(const float* s, long long lds, void* p, long long ldp, int rows, int cols, float scale,
                           cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200_CFLEARN_EXT_H_ */
