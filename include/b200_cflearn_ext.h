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
 * h is a multiple of 128 / w (or h * w divides 128), the rule of b200_conv3x3_nhwc_bf16.  The weight gradient needs, on its
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

#ifdef __cplusplus
}
#endif
#endif /* B200_CFLEARN_EXT_H_ */
