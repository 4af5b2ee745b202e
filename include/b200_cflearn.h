/* b200_cflearn.h -- C-ABI of the native (sm_90a, H100) transformer-block training-step kernels.
 *
 * The reference (carefree-learn @ ca5ced1) has NO native code and no FFI: its plug-in surface is a Python
 * registry of nn.Module classes (cflearn/modules/common.py:30-53) whose forward()s call torch.nn.functional.
 * This header is therefore the boundary a maintainer would bind from Python (ctypes stub in INTEGRATION.md);
 * each entry point names the reference call site (file:line under cflearn/) whose arithmetic it replaces.
 *
 * Conventions (all entry points):
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless stated otherwise, caller-owned,
 *     16-byte aligned, dense row-major with the documented leading dimension;
 *   - asynchronous on `stream`; never allocates, never synchronises, never falls back to the CPU;
 *   - returns 0 on success or a negative B200_ERR_* code; b200_last_error() describes the last failure
 *     on the calling thread;
 *   - bf16 = IEEE bfloat16 (round-to-nearest-even), f32 = IEEE binary32;
 *   - every argument is checked before anything is launched.  A refused call returns B200_ERR_ARG for a size outside the
 *     entry's range, a NULL required pointer or a leading dimension smaller than the row width, and B200_ERR_ALIGN for a
 *     misaligned pointer or a leading dimension that is not a multiple of the kernel's vector width;
 *   - every non-NULL device pointer is 16-byte aligned, except the ones an entry's comment names as ELEMENT-WISE: its
 *     kernels access them one element at a time, so they need only their natural alignment (2 bytes for bf16, 4 for f32
 *     and int32, 8 for int64);
 *   - sizes whose products a kernel indexes in 32-bit int are refused when the product would overflow.
 */
#ifndef B200_CFLEARN_H_
#define B200_CFLEARN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef __CUDA_RUNTIME_H__
typedef struct CUstream_st* cudaStream_t;
#endif

#define B200_ABI_VERSION 4

enum {
    B200_OK = 0,
    B200_ERR_ARG = -1,    /* invalid argument (shape, null pointer, unsupported combination) */
    B200_ERR_ALIGN = -2,  /* pointer / stride alignment requirement violated */
    B200_ERR_DRIVER = -3, /* CUDA driver entry point missing or tensor-map encode failed */
    B200_ERR_LAUNCH = -4, /* kernel launch failed (cudaGetLastError) */
    B200_ERR_NO_DEVICE = -5
};

/* GEMM epilogues (b200_gemm_bf16) */
enum {
    B200_EPI_BIAS_BF16 = 0,      /* out0[bf16] = bf16(acc + bias)                                               */
    B200_EPI_BIAS_GELU_BF16 = 1, /* out0 = h = bf16(acc + bias); out1 = bf16(gelu_erf(h))                        */
    B200_EPI_BIAS_RESID_F32 = 2, /* out0[f32] = aux[f32] + float(bf16(acc + bias))   (aux may alias out0)         */
    B200_EPI_DGELU_BF16 = 3,     /* out0[bf16] = bf16(float(bf16(acc)) * gelu_erf'(aux[bf16]))                   */
    B200_EPI_PARTIAL_F32 = 4,    /* out0[f32][split, M, N] = partial accumulators (split-K)                      */
    B200_EPI_BIAS_QGELU_BF16 = 5, /* like 1 with QuickGELU x * sigmoid(1.702 x) (CLIP, activations.py:151-153), rounded to
                                    bf16 after each of eager's three elementwise ops                              */
    B200_EPI_DQGELU_BF16 = 6,     /* like 3: autograd of those three ops with eager's bf16 rounding after each kernel */
    /* GEGLU (cflearn/modules/core/activations.py:157-164): N = 2F, the rows of W1 = [h rows 0..F-1 ; gate rows F..2F-1]
     * (the reference layout), F % 8 == 0.  out0 = hg = bf16(acc + bias) [M, ldo] (2F columns, the reference's column order);
     * out1 = a = bf16(float(h) * float(bf16(gelu_erf(gate)))), DENSE [M, F] (row stride F).  bias bf16 [2F], required.
     * A and B K-major. */
    B200_EPI_BIAS_GEGLU_BF16 = 7,
    /* its backward through the FF2 dgrad: the GEMM is da = dy . W2 with W2 MN-major [K, ldb] of F columns, but N = 2F as
     * above; aux = hg [M, ldo], out0 = dhg [M, ldo]:  dh = bf16(float(bf16(da)) * g), dg = bf16(float(bf16(da)) * h),
     * dgate = bf16(gelu_erf'(gate) * float(dg)), g = bf16(gelu_erf(gate)) -- eager's three roundings.  No bias. */
    B200_EPI_DGEGLU_BF16 = 8,
    /* out0[bf16] = bf16(float(bf16(acc + bias)) + float(aux[bf16]))   (aux may alias out0): the bf16 residual stream */
    B200_EPI_BIAS_RESID_BF16 = 9,
    /* The two 3x3-convolution epilogues of the UNet's ResBlock (b200_conv3x3_nhwc_bf16 only; b200_gemm_bf16 refuses them).
     * Variants of 9, with eager's two bf16 roundings (cflearn/modules/core/convs/residual.py:232-249):
     *   10: out0 = bf16(float(bf16(acc + bias)) + float(aux[row / (H * W), col])), aux = bf16 [B, ldo], one row per image:
     *       conv1 plus the time embedding t[b, c].
     *   11: as 9, then +-inf becomes +-bf16 max and NaN stays NaN (safe_clip_, toolkit.py:1236-1255): conv2 plus the shortcut.
     * aux is required and 16-byte aligned. */
    B200_EPI_BIAS_ADD_PER_IMAGE_BF16 = 10,
    B200_EPI_BIAS_RESID_CLAMP_BF16 = 11
};

int b200_abi_version(void);
const char* b200_last_error(void);
/* number of kernels this library has launched on the calling process so far (bench.py's gpu_launches) */
long long b200_launch_count(void);

/* ---------------------------------------------------------------------------------------------------------
 * Dense layers: C[M,N] = A[M,K] . B[N,K]^T on the tensor cores (wgmma: bf16 in, fp32 accumulate in registers).
 *   a_mn_major = 0: A is row-major [M, lda] (K contiguous);  1: A is row-major [K, lda] (M contiguous).
 *   b_mn_major = 0: B is row-major [N, ldb] (K contiguous);  1: B is row-major [K, ldb] (N contiguous).
 *   bias: bf16 [N] or NULL, read in 16-byte groups up to roundup(N, 8) elements (the values past N never reach an output).
 *   ldo: leading dimension (elements) of out0/out1/aux (but see the GEGLU epilogues: their out1 is dense).  Any N >= 1;
 *   columns >= N of out0 / out1 are never written.  out0 / out1 / aux 16-byte aligned.
 *   splits > 1 only with B200_EPI_PARTIAL_F32 (out0 is f32 [s, M, ldo] with s = min(splits, ceil(K / 64)): one split per
 *   64-deep k-block at most; planes s .. splits - 1 are not written).  max_ctas <= 0: all SMs.
 *   ldo >= N.  out1 is required by the GELU epilogues (1, 5, 7), aux by 2, 3, 6, 8 and 9; bias is ignored by 3, 4 and 6.
 *   Operand majors (a_mn_major, b_mn_major): any with BIAS_BF16, (0, 1) with 3, 6 and 8, (1, 1) with PARTIAL_F32, else (0, 0).
 *   Every argument is checked before any tensor map is encoded.
 * Replaces F.linear at cflearn/modules/core/customs.py:85-89 (Linear.forward), the packed-QKV projection at
 * cflearn/modules/core/attentions.py:214, FeedForward's Linear->GELU->Linear at
 * cflearn/modules/core/mixed_stacks/channel_mixers.py:29-36, the k=s=16 patch-embed F.conv2d at
 * cflearn/modules/core/convs/basic.py:155-174, and autograd's dgrad/wgrad of all of them.
 * --------------------------------------------------------------------------------------------------------- */
int b200_gemm_bf16(const void* A, long long lda, int a_mn_major, const void* B, long long ldb, int b_mn_major,
                   int M, int N, int K, int epilogue, const void* bias, void* out0, void* out1, const void* aux,
                   long long ldo, int splits, int max_ctas, cudaStream_t stream);
/* split count that fills the 132 SMs of an H100 SXM best for an [M,N] output with reduction length K */
int b200_gemm_pick_splits(int M, int N, int K);
/* GEMM cluster mode (0, 1 or 2), kept for ABI compatibility: the sm_90a GEMM runs one CTA per 128x256 tile in every
 * mode, so the setting is only recorded.  Returns the previous setting. */
int b200_set_gemm_multicast(int enable);
/* out[f32][n] (+)= round( sum_s partial[s][n] ); round_bf16 mirrors autocast (the weight grad of a bf16 matmul
 * is produced in bf16, cf. cflearn/schema.py:1266-1276 autocast + :980 backward). accumulate: 0 overwrite.
 * n % 4 == 0; partial and out required. */
int b200_splitk_reduce(const float* partial, int splits, long long n, float* out, int round_bf16, int accumulate,
                       cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * LayerNorm over the last dim (fp32 statistics), replaces nn.LayerNorm built by NormFactory("layer")
 * (cflearn/modules/core/norms.py:88-89,118-124; used at mixed_stacks/api.py:141,155,397-402).
 *   x: f32 [rows, ld_x] (first `dim` columns are normalised; ld_x lets the head LN read only token 0 of each
 *   image -- api.py:365).  y: bf16 [rows, dim] (the value autocast hands to the next F.linear).
 *   mean, rstd: f32 [rows], saved for backward.  Required: x, gamma, beta, y_bf16, mean, rstd; ld_x >= dim, ld_x % 4 == 0.
 *   Element-wise: mean, rstd.
 * --------------------------------------------------------------------------------------------------------- */
int b200_layernorm_fwd(const float* x, long long ld_x, const float* gamma, const float* beta, void* y_bf16,
                       float* y_f32 /* optional [rows, dim]: the un-rounded fp32 result */, float* mean, float* rstd,
                       int rows, int dim, float eps, cudaStream_t stream);
/* dx_out[f32] = (dres ? dres : 0) + LN'(dy); dx_out and dres (f32, optional) both have row stride ld_dx (so the head LN
 * can scatter into token 0).
 * dy: bf16 [rows, dim].  dx_bf16 (optional) receives bf16(dx_out) -- the gradient the preceding bf16 matmul
 * output sees under autocast.  dgb_part: f32 [nparts, 2*dim] workspace ([.., 0:dim] dgamma partials, [.., dim:2dim]
 * dbeta partials), reduced by b200_colsum_finish.  Returns nparts through *nparts_out (host int).
 * dy is bf16 [rows, dim], or fp32 when dy_is_f32 != 0 (a LayerNorm whose output is the fp32 residual stream itself:
 * CLIP's embedding_norm, mixed_stacks/api.py:433-434).  dx_colsum != 0 (needs dx_bf16, bf16 dy): the part rows are 3*dim wide and columns [2*dim, 3*dim) hold the column sums of
 * the bf16-rounded dx rows, i.e. the bias gradient of the Linear layer whose output gradient this dx is (the
 * separate b200_colsum_bf16 pass over dx_bf16 is then not needed).  Required: dy, x, gamma, mean, rstd, dx_out, dgb_part;
 * optional: dres, dx_bf16, nparts_out; ld_x, ld_dx >= dim and multiples of 4; max_parts >= 1.  Element-wise: mean, rstd,
 * dgb_part. */
int b200_layernorm_bwd(const void* dy, int dy_is_f32, const float* x, long long ld_x, const float* gamma, const float* mean,
                       const float* rstd, const float* dres, float* dx_out, long long ld_dx, void* dx_bf16,
                       float* dgb_part, int max_parts, int* nparts_out, int rows, int dim, int dx_colsum,
                       cudaStream_t stream);

/* LayerNorm over BF16 rows: the SD-v1.5 UNet's SpatialTransformerBlock norms (mixed_stacks/api.py:800-812), whose residual
 * stream is bf16 under autocast.  x, y, dy, dres, dx: bf16 [rows, dim] dense; gamma, beta f32 [dim]; 0 < dim <= 2048,
 * dim % 8 == 0; dres is optional, every other pointer required.  Element-wise: mean, rstd, dgb_part.
 *   forward : y = bf16(LN_fp32(x)); mean, rstd f32 [rows].
 *   backward: dx = bf16(float(dres) + float(bf16(LN'(dy))))  (dres NULL: dx = bf16(LN'(dy))) -- eager's cast back to the bf16
 *             input followed by the bf16 accumulation of the residual branch.  dgb_part: f32 [nparts, 2 * dim] ([.., 0:dim]
 *             dgamma, [.., dim:2 dim] dbeta partials; finish with b200_colsum_finish, unrounded).  Deterministic. */
int b200_layernorm_bf16_fwd(const void* x_bf16, const float* gamma, const float* beta, void* y_bf16, float* mean, float* rstd,
                            int rows, int dim, float eps, cudaStream_t stream);
int b200_layernorm_bf16_bwd(const void* dy_bf16, const void* x_bf16, const float* gamma, const float* mean, const float* rstd,
                            const void* dres_bf16, void* dx_bf16, float* dgb_part, int max_parts, int* nparts_out, int rows, int dim,
                            cudaStream_t stream);

/* column sums: part[p][c] = sum over a slice of rows of x[r][c]  (x bf16 or f32), then finish() reduces the
 * parts.  Bias gradients of every Linear (autograd of customs.py:89) and LN gamma/beta gradients.
 * b200_colsum_bf16: ld % 8 == 0 and ld >= roundup(cols, 8); each row is read in 16-byte groups up to roundup(cols, 8)
 * elements (the values past cols never reach a part); part is [nparts, cols] dense, nparts <= max_parts.  x and part are
 * required, nparts_out optional; part is element-wise.
 * b200_colsum_finish / _finish2: part_ld >= cols (cols0 + cols1); part and out (out0, out1) required and element-wise, so
 * part may point into a row (e.g. at a column offset). */
int b200_colsum_bf16(const void* x_bf16, long long ld, int rows, int cols, float* part, int max_parts,
                     int* nparts_out, cudaStream_t stream);
int b200_colsum_finish(const float* part, long long part_ld, int nparts, int cols, float* out, int round_bf16,
                       int accumulate, cudaStream_t stream);
/* the same reduction with two destinations: columns [0, cols0) -> out0, [cols0, cols0 + cols1) -> out1 */
int b200_colsum_finish2(const float* part, long long part_ld, int nparts, int cols0, float* out0, int round0, int cols1,
                        float* out1, int round1, int accumulate, cudaStream_t stream);
/* Per-image column sums of x bf16 [B, HW, C] (dense, C % 8 == 0, x 16-byte aligned), one pass over x, no atomics:
 *   per_image bf16 [B, C] = bf16(sum over the HW rows of image b)  (the gradient of a [B, C] table broadcast over the pixels:
 *                           the ResBlock's time embedding, cflearn/modules/core/convs/residual.py:240-244)
 *   total f32 [C] = float(bf16(sum over b of the unrounded per-image sums))  (the bias gradient of the conv that wrote x)
 * workspace: b200_colsum_per_image_workspace_floats(B, HW, C) floats.  Deterministic.  All pointers required;
 * element-wise: per_image, total, workspace. */
long long b200_colsum_per_image_workspace_floats(int B, int HW, int C);
int b200_colsum_per_image_bf16(const void* x_bf16, int B, int HW, int C, void* per_image_bf16, float* total, float* workspace,
                               cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Fused multi-head self-attention on the PACKED qkv tensor, replaces the split/permute/contiguous copies at
 * cflearn/modules/core/attentions.py:216,180-185,245,270 and F.scaled_dot_product_attention reached through
 * cflearn/toolkit.py:911-974 (sdp_attn).  qkv: bf16 [B, T, 3*H*Dh] laid out [q | k | v], heads contiguous
 * inside each third (chunk(3, dim=-1) then view(B,T,H,Dh)).  out: bf16 [B, T, H*Dh].  lse: f32 [B, H, T]
 * (natural-log sum-exp of the scaled scores), saved for backward.  causal != 0 applies the lower-triangular
 * mask of cflearn/modules/nlp/encoder/transformer.py:42-48.  Dh must be 64, T <= 256.
 * Pointers, for every attention entry point below: qkv (q, k, v), out, lse and, in the backward, dout and dqkv (dq, dk, dv)
 * are required; dbias_part is optional; the streamed backward entries (long and cross) require their workspace.  Every
 * non-NULL pointer is 16-byte aligned (TMA bases, and the backward reads out / dout in 16-byte groups).  All arguments are
 * checked before any tensor map is encoded: a size outside the entry's range, a NULL required pointer or a missing workspace
 * is B200_ERR_ARG, a misaligned pointer or leading dim B200_ERR_ALIGN.
 * --------------------------------------------------------------------------------------------------------- */
int b200_attention_fwd(const void* qkv_bf16, void* out_bf16, float* lse, int B, int T, int H, int Dh, float scale,
                       int causal, cudaStream_t stream);
/* kernel version switches (forward 0-2, backward 0-3) and the L2-prefetch switch, kept for ABI compatibility: the sm_90a
 * build has one forward and one backward kernel, so these settings are only recorded.  Each returns the previous setting. */
int b200_set_attention_fwd_version(int version);
int b200_set_attention_bwd_version(int version);
int b200_set_attention_prefetch(int enable);
/* dbias_part (optional, f32 [B, 3*H*Dh]): per-image column sums of the bf16 dqkv rows written; summed over the batch
 * (b200_colsum_finish, nparts = B) they are the gradient of the packed qkv bias (attentions.py:112-119). */
int b200_attention_bwd(const void* qkv_bf16, const void* out_bf16, const void* dout_bf16, const float* lse,
                       void* dqkv_bf16, int B, int T, int H, int Dh, float scale, int causal, float* dbias_part,
                       cudaStream_t stream);
/* The same attention for long sequences: 1 <= T <= 16384, Dh = 64, the same layouts, outputs and causal flag as
 * b200_attention_fwd / _bwd.  These kernels stream K / V (forward, dQ) or Q / dO (dK / dV) through shared memory in
 * 64-row blocks with an online softmax, so no head has to fit in shared memory at once.  Deterministic (no atomics).
 * workspace (backward): b200_attention_long_bwd_workspace_floats(B, T, H) floats of device scratch.
 * dbias_part (optional): the same per-image column sums as b200_attention_bwd writes. */
int b200_attention_long_fwd(const void* qkv_bf16, void* out_bf16, float* lse, int B, int T, int H, int Dh, float scale,
                            int causal, cudaStream_t stream);
long long b200_attention_long_bwd_workspace_floats(int B, int T, int H);
int b200_attention_long_bwd(const void* qkv_bf16, const void* out_bf16, const void* dout_bf16, const float* lse,
                            void* dqkv_bf16, int B, int T, int H, int Dh, float scale, int causal, float* dbias_part,
                            float* workspace, cudaStream_t stream);
/* Attention with separate Q / K / V and head dims 8 ... 160 (multiple of 8) on the same streamed kernels: the SD-v1.5 UNet's
 * CrossAttention, cflearn/modules/core/attentions.py:534-569 (heads folded into the batch, then sdp_attn ->
 * F.scaled_dot_product_attention at cflearn/toolkit.py:959-963).  q: bf16 [B, Tq, ldq], k / v: bf16 [B, Tk, ldkv], head h at
 * columns [h * Dh, h * Dh + Dh); out: bf16 [B, Tq, ldo]; lse: f32 [B, H, Tq].  1 <= Tq, Tk <= 16384; causal only with Tq == Tk.
 * Leading dims are multiples of 8 and >= H * Dh, so q / k / v may be column slices of one packed
 * projection output (self-attention: q = qkv, k = qkv + H * Dh, v = qkv + 2 * H * Dh, ld = 3 * H * Dh).
 * Backward: dout uses ldo, dq uses ldq, dk / dv use ldkv (so dq / dk / dv may be views of one packed gradient buffer).
 * workspace (backward): b200_cross_attention_bwd_workspace_floats(B, Tq, Tk, H, Dh) floats.  Deterministic (no atomics). */
int b200_cross_attention_fwd(const void* q, long long ldq, const void* k, const void* v, long long ldkv, void* out, long long ldo,
                             float* lse, int B, int Tq, int Tk, int H, int Dh, float scale, int causal, cudaStream_t stream);
long long b200_cross_attention_bwd_workspace_floats(int B, int Tq, int Tk, int H, int Dh);
int b200_cross_attention_bwd(const void* q, long long ldq, const void* k, const void* v, long long ldkv, const void* out,
                             long long ldo, const void* dout, const float* lse, void* dq, void* dk, void* dv, int B, int Tq, int Tk,
                             int H, int Dh, float scale, int causal, float* workspace, cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * FCNN (cflearn/modules/ml/fcnn.py:12-59: Mapping(Linear + ReLU) x n, then nn.Linear) -- one launch per training
 * step, fp32, for networks whose parameters + activations of 128 samples fit in shared memory (BASELINE.json
 * configs[0]: 10 -> 32 -> 32 -> 1).  dims[0..n_layers] are the widths (host array); W_l ([dims[l+1], dims[l]],
 * row-major like nn.Linear.weight) and b_l live at w_offsets[l] / b_offsets[l] (floats, -1 = no bias) inside the flat
 * fp32 `params` arena of arena_len floats.  pred (optional): [M, dims[n]].  part == NULL: inference only.  Otherwise
 * part[nblocks, arena_len + 1] receives per-128-sample gradient partials in arena layout (b200_colsum_finish sums
 * them) and, in column arena_len, the loss partial.  loss_mode 1: w_mae * mean|p - y| + w_mse * mean (p - y)^2
 * ("multi_task" of "mae" + "mse", losses/basic.py:45-61, losses/common.py:72-88); loss_mode 0: dpred [M, dims[n]] is
 * the gradient of the output (autograd's backward).  *nblocks_out (host int) = number of partial rows written.
 * Required: x, params and the host arrays dims, w_offsets, b_offsets (and y with loss_mode 1, dpred with loss_mode 0 when
 * part != NULL); optional: y, dpred, pred, part, nblocks_out.  Element-wise: every device pointer. */
int b200_fcnn_step(const float* x, const float* y, const float* dpred, const float* params, float* pred, float* part,
                   int M, int n_layers, const int* dims, const int* w_offsets, const int* b_offsets, int arena_len,
                   int loss_mode, float w_mae, float w_mse, int* nblocks_out, cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Patch embedding glue (cflearn/modules/core/high_level.py:143-149,181-188, mixed_stacks/api.py:419-438):
 *   im2col : x f32 [B, C, IMG, IMG] (NCHW) -> cols bf16 [B*(IMG/P)^2, C*P*P]  (k index = (c, ky, kx))
 *   assemble: net f32 [B, 1+np, D] = cat(cls, float(patch bf16 [B*np, D])) + pos[1+np, D]
 *   assemble_bwd: dpatch bf16 [B*np, D] = bf16(dnet[:,1:,:]); dpos f32 [1+np, D] = sum_b dnet; dcls f32 [D]
 * Every device pointer is required (conv_bias_bf16 optional); assemble_bwd needs (np + 1) * D / 4 to fit in int.
 * --------------------------------------------------------------------------------------------------------- */
int b200_patch_im2col(const float* x, void* cols_bf16, int B, int C, int img, int patch, cudaStream_t stream);
/* The same matrix straight from the RAW batch: x = uint8 [B, img, img, C] (HWC, C <= 4), value = ((x / division) - mean[c])
 * / std[c] evaluated in float64, rounded to float32, then to bf16 -- the reference's rounding chain.  Replaces the host-side
 * runtime blocks static_normalize / imagenet_normalize / hwc_to_chw (cflearn/data/blocks/cv/normalize.py:11-67,
 * hwc_to_chw.py:9-15), TensorBatcher's float32 conversion + host->device copy of 4 bytes per value
 * (cflearn/data/utils.py:255-283) and autocast's bf16 cast.  mean / std: HOST pointers to C doubles (NULL: 0 / 1). */
int b200_patch_im2col_u8(const void* x_u8_hwc, void* cols_bf16, int B, int C, int img, int patch, double division,
                         const double* mean_host, const double* std_host, cudaStream_t stream);
/* conv_bias_bf16 (bf16 [D] or NULL): the patch rows first become bf16(patch + bias) -- eager's F.conv2d with a bias on CUDA
 * rounds the convolution output to bf16 and then adds the bias in a second bf16 op (ATen cuDNN path: `output.add_(bias)`). */
int b200_assemble_tokens(const void* patch_bf16, const float* cls, const float* pos, float* net, int B, int np,
                         int D, const void* conv_bias_bf16, cudaStream_t stream);
int b200_assemble_tokens_bwd(const float* dnet, void* dpatch_bf16, float* dpos, float* dcls, int B, int np, int D,
                             int accumulate, cudaStream_t stream);
/* Text-tower input stage (TeTEncoder, cflearn/modules/nlp/encoder/transformer.py:92 -> mixed_stacks/api.py:419-438 without
 * a head token): net f32 [B, T, D] = x f32 [B, T, D] + pos f32 [T, D];  backward: dpos = sum over the batch of dnet.
 * D % 4 == 0, T * D / 4 fits in int; every pointer required. */
int b200_add_pos(const float* x, const float* pos, float* net, int B, int T, int D, cudaStream_t stream);
int b200_add_pos_bwd(const float* dnet, float* dpos, int B, int T, int D, int accumulate, cudaStream_t stream);

/* CLIP text glue (cflearn/modules/multimodal/clip.py:235,248-250): integer-indexed row moves, bit-exact.
 *   embedding_fwd : out f32 [n, D] = weight f32 [V, D][ids[n]]; ids outside [0, V) set *bad_index_flag (device int)
 *   embedding_bwd : dweight[ids[n]] += dnet[n] for ids[n] != padding_idx (dweight zeroed by the caller; fp32 atomics)
 *   argmax_gather : pos[b] = first arg-max of ids[b, :]; out f32 [B, D] = x f32 [B, T, D][b, pos[b]]
 *   scatter_rows  : dx[b, pos[b], :] = dout[b, :]   (dx zero-filled by the caller)
 * Every pointer is required.  Element-wise: ids and bad_index_flag of embedding_fwd (weight and out are read in 16-byte
 * groups, D % 4 == 0), every pointer of the other three. */
int b200_embedding_fwd(const long long* ids, const float* weight, float* out, long long n, int D, int V, int* bad_index_flag,
                       cudaStream_t stream);
int b200_embedding_bwd(const long long* ids, const float* dnet, float* dweight, long long n, int D, int V, int padding_idx,
                       cudaStream_t stream);
int b200_argmax_gather_rows(const long long* ids, const float* x, float* out, int* pos, int B, int T, int D, cudaStream_t stream);
int b200_scatter_rows(const float* dout, const int* pos, float* dx, int B, int T, int D, cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Cross entropy with integer labels (cflearn/losses/basic.py:137-141: -log_softmax(logits,1).gather(1,labels),
 * mean over the batch via ILoss._reduce, cflearn/schema.py:767-810).  logits bf16 [B, C] (ld = ldl),
 * labels int64 [B].  loss_rows f32 [B], loss_mean f32 [1].  dlogits bf16 [B, C] = bf16((softmax - onehot) *
 * grad_scale * (grad_scale_dev ? *grad_scale_dev : 1) / B) -- grad_scale_dev is the upstream gradient of the mean
 * loss living on the device (autograd's grad_output), so backward needs no host synchronisation.
 * The label gather is integer-exact; out-of-range labels set *bad_label_flag (device int).
 * Required: logits, labels, loss_rows, bad_label_flag; optional: loss_mean, dlogits, grad_scale_dev; ldl >= C.
 * Element-wise: every pointer of both cross entropies.
 * --------------------------------------------------------------------------------------------------------- */
int b200_softmax_xent_fwd_bwd(const void* logits_bf16, long long ldl, const long long* labels, float* loss_rows,
                              float* loss_mean, void* dlogits_bf16, int* bad_label_flag, int B, int C,
                              float grad_scale, const float* grad_scale_dev, cudaStream_t stream);
/* Symmetric (contrastive) cross entropy of a square bf16 logits matrix L [B, B] (leading dimension ldl) with targets
 * arange(B): loss[0] = (CE(L) + CE(L^T)) / 2, dlogits = bf16 of the fp32 gradient scaled by grad_scale (* grad_scale_dev[0]).
 * The training objective of CLIP (cflearn/modules/multimodal/clip.py:209-256 produce L; the reference ships no loss for
 * it, SURVEY.md 8d -- the definition is oracle/clip_oracle.py::symmetric_cross_entropy).  lse_ws: 2*B floats of scratch.
 * Required: logits, loss, lse_ws; optional: dlogits, grad_scale_dev; ldl >= B. */
int b200_symmetric_xent_fwd_bwd(const void* logits_bf16, long long ldl, float* loss, void* dlogits_bf16, float* lse_ws, int B,
                                float grad_scale, const float* grad_scale_dev, cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Optimizer step on the flat fp32 arenas (torch.optim.Adam semantics without amsgrad; the reference's default
 * optimizer "adam", cflearn/optimizers.py:29-32, stepped at cflearn/schema.py:983).  n % 4 == 0.
 * step_dev == NULL: `step` (>= 1) is the host-side step count.  step_dev != NULL: a device int that is incremented
 * (on the stream) and then used as the step count, so the call can be replayed from a CUDA graph.
 * The four arenas are required; element-wise: step_dev (and hyper_dev below).
 * --------------------------------------------------------------------------------------------------------- */
int b200_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n, float lr,
                   float beta1, float beta2, float eps, float weight_decay, int step, int* step_dev,
                   cudaStream_t stream);
/* The same update with every hyper-parameter in DEVICE memory: hyper_dev = {lr, beta1, beta2, eps, weight_decay,
 * grad_scale} (6 floats; grad_scale multiplies the gradient first: 1/world after a SUM all-reduce, or the clip
 * coefficient of cflearn/schema.py:981-982).  A captured CUDA graph therefore follows an LR scheduler
 * (cflearn/pipeline/blocks/basic.py:334-352 "warmup" is the reference's default) without being re-captured.
 * increment != 0: *step_dev += 1 first (pass 0 for all but the first slice when one step updates several slices).
 * hyper_dev and step_dev are required. */
int b200_adam_step_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                       const float* hyper_dev, int* step_dev, int increment, cudaStream_t stream);

/* element-wise helpers (every pointer required and 16-byte aligned) */
int b200_cast_f32_to_bf16(const float* src, void* dst_bf16, long long n, cudaStream_t stream);
int b200_fill_f32(float* dst, float value, long long n, cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * 3x3 convolution (stride 1, zero padding 1) on channels-last bf16 activations as an IMPLICIT GEMM on the wgmma main
 * loop: x [B, H, W, Cin], w_packed [Cout, 9 * Cin] (k = (ky * 3 + kx) * Cin + ci), bias bf16 [Cout] or NULL,
 * out0 / aux [B*H*W, ldo].  Cin % 64 == 0; W divides 128 and H is a multiple of 128 / W (or H * W divides 128), or W is 128
 * times a power of 2 (256, 512, ...; each 128-pixel tile is then part of one image row).
 * epilogue: B200_EPI_BIAS_BF16, B200_EPI_BIAS_RESID_F32, B200_EPI_BIAS_RESID_CLAMP_BF16 (aux bf16 [B*H*W, ldo]) or
 * B200_EPI_BIAS_ADD_PER_IMAGE_BF16 (aux bf16 [B, ldo]).  No im2col matrix exists: each (tap, 64-channel) k-block is ONE
 * TMA box of the activation shifted by the tap, its halo zero-filled by the TMA unit.
 * Replaces F.conv2d at cflearn/modules/core/convs/basic.py:155-174 for the UNet's 3x3 convolutions
 * (convs/residual.py:179-186,199-205; multimodal/diffusion/unet.py:213-217,269-272); the input gradient is the same
 * call with flipped, transposed weights.
 * --------------------------------------------------------------------------------------------------------- */
int b200_conv3x3_nhwc_bf16(const void* x, const void* w_packed, const void* bias, void* out0, const void* aux, long long ldo,
                           int B, int H, int W, int Cin, int Cout, int epilogue, cudaStream_t stream);
/* weight gradient of that convolution: ONE split-K GEMM with M = Cout, N = 9 * Cin, K = B * H * W (dy MN-major, x behind the
 * 4-D map, each 64-channel box shifted by its own tap).  dy: bf16 [B*H*W, ld_dy]; partials: f32 [splits][Cout][9 * Cin]
 * (finish with b200_splitk_reduce; the plane layout is the packed forward weight layout).  Cin % 64 == 0, W divides 64,
 * H * W % 64 == 0.  Replaces the weight half of conv2d's backward for cflearn/modules/core/convs/basic.py:155-174. */
int b200_conv3x3_wgrad_nhwc_bf16(const void* dy, long long ld_dy, const void* x, void* partials, int B, int H, int W, int Cin,
                                 int Cout, int splits, cudaStream_t stream);

/* Upper bound on the grid of every persistent kernel of this library (the GEMMs); 0 = all SMs (default);
 * launches > 0: the bound lapses by itself after that many persistent launches.  Returns the previous value.  For co-scheduling with other kernels that must hold SMs (an NCCL all-reduce in flight): tiles are
 * assigned to CTAs statically, so a CTA that has to wait for an SM stretches its kernel.  The package's data-parallel step
 * does not use this bound: it shrinks only the GEMM launched right behind a bucket (max_ctas of b200_gemm_bf16).  (DistributedDataParallel's overlap,
 * accelerate.prepare, cflearn/schema.py:1174-1180, has no such knob: eager kernels are not persistent.) */
int b200_set_persistent_ctas(int n, int launches);

/* ---------------------------------------------------------------------------------------------------------
 * GroupNorm(32) (+ SiLU) on channels-last bf16 activations x [B, HW, C] (C contiguous, C % 32 == 0, C <= 2560): the
 * normalisation in front of every 3x3 convolution of the SD-v1.5 UNet (BASELINE.json configs[4]).
 *   y = bf16( act( (x - mean_g) * rstd_g * gamma_c + beta_c ) ),  act = SiLU if silu != 0 else identity
 * with fp32 statistics per (image, group of C / 32 channels) and ONE rounding at the end, i.e. what
 * F.group_norm -> F.silu -> autocast's bf16 cast at the following conv amount to
 * (cflearn/modules/core/convs/residual.py:176-178,197-198,221,241; multimodal/diffusion/unet.py:264-268;
 * SpatialTransformer.norm without activation, mixed_stacks/api.py:866-870).  mean / rstd: f32 [B, 32], kept for backward.
 * Backward: dx = bf16 of the fp32 GroupNorm (o SiLU) gradient, dgamma / dbeta f32 [C] (accumulate != 0: added).
 * workspace: b200_groupnorm_workspace_floats(B, HW, C) floats.  Deterministic (no atomics).  Every pointer is required,
 * gamma and beta included.  Element-wise: every pointer but x, y, dy and dx.
 * --------------------------------------------------------------------------------------------------------- */
long long b200_groupnorm_workspace_floats(int B, int HW, int C);
int b200_groupnorm_silu_fwd(const void* x_bf16, const float* gamma, const float* beta, void* y_bf16, float* mean, float* rstd,
                            float* workspace, int B, int HW, int C, float eps, int silu, cudaStream_t stream);
int b200_groupnorm_silu_bwd(const void* x_bf16, const void* dy_bf16, const float* gamma, const float* beta, const float* mean,
                            const float* rstd, void* dx_bf16, float* dgamma, float* dbeta, float* workspace, int B, int HW, int C,
                            int silu, int accumulate, cudaStream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Data-parallel gradient exchange (replaces the DDP wrap of `accelerator.prepare`, cflearn/trainer.py:226-229,
 * 266-273; the all-reduce sits between backward and optimizer.step, cflearn/schema.py:980-984).  One communicator per
 * process / GPU over NCCL (libnccl.so.2 is dlopen'ed at first use).  b200_comm_unique_id: rank 0 creates the 128-byte
 * id (HOST pointer) and ships it to the other ranks by any means; b200_comm_init is collective over all ranks and
 * binds to the CURRENT device (max_ctas > 0: ncclConfig_t.maxCTAs of THIS communicator -- its kernels share the SMs with the
 * backward's persistent kernels, see b200_set_persistent_ctas; 0: NCCL's default); b200_comm_allreduce_bucket enqueues an in-place fp32 all-reduce (average != 0: mean
 * over ranks, else sum) of buf[0..n) on `stream` -- an ordinary stream operation, capturable in a CUDA graph;
 * b200_comm_async_error polls the communicator (0 healthy, negative: abort the job); b200_comm_finalize destroys
 * (abort != 0: ncclCommAbort) the communicator -- every CUDA graph that captured it must have been destroyed first (NCCL waits).
 * --------------------------------------------------------------------------------------------------------- */
int b200_comm_unique_id(void* id_out_128);
int b200_comm_init(const void* id_128, int rank, int world, int max_ctas, void** comm_out);
int b200_comm_allreduce_bucket(void* comm, float* buf, long long n, int average, cudaStream_t stream);
int b200_comm_async_error(void* comm);
int b200_comm_finalize(void* comm, int abort);
int b200_comm_nccl_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_CFLEARN_H_ */
