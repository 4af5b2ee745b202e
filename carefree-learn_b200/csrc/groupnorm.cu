// GroupNorm(32) + SiLU, forward and backward, on channels-last (NHWC) bf16 activations: the normalisation that precedes every
// 3x3 convolution of the SD-v1.5 UNet (BASELINE.json configs[4]; SURVEY.md 8f row N3).
//
// Replaces, per ResBlock / head of the reference (under bf16 autocast):
//   F.group_norm(net, 32, w, b, eps)   cflearn/modules/core/convs/residual.py:221,241 (norm1 / norm2, built :176-177,197),
//                                      cflearn/modules/multimodal/diffusion/unet.py:264-268 (head)      -- autocast runs it in fp32
//   F.silu(...)                        the "SiLU" activation between norm and conv (residual.py:178,198) -- fp32 in, fp32 out
//   the bf16 cast of the conv input    autocast's cast at F.conv2d
// i.e. y = bf16( silu( (x - mean_g) * rstd_g * gamma_c + beta_c ) ) with fp32 statistics over (H, W, C / 32) per (image, group),
// ONE rounding at the end -- exactly eager's.  activation == 0 gives the plain GroupNorm (SpatialTransformer.norm, eps 1e-6,
// mixed_stacks/api.py:866-870).  HBM-bound: forward 6 bytes / element (x twice, y once), backward 10 (x, dy twice; dx once).
//
// Layout: x [B, HW, C] with C contiguous.  A block owns one image and a slab of pixels and reads whole pixel rows (coalesced,
// 16 bytes per thread); per-channel partial sums meet in shared memory and leave as per-(image, slab, group) partials in a
// FIXED order (no atomics: results are run-to-run identical).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200_internal.h"
#include "ptx.cuh"

namespace b200 {

constexpr int GN_GROUPS = 32;
constexpr int GN_THREADS = 256;
constexpr int GN_MAX_C = 2560;  // SD-v1.5: 320 .. 2560 channels (skip concatenations); per-channel scratch lives in smem

__device__ __forceinline__ float silu_f(float z) { return z * fast_rcp(1.0f + fast_ex2(-1.4426950408889634f * z)); }
// d/dz silu(z) = s + z s (1 - s),  s = sigmoid(z)
__device__ __forceinline__ float silu_grad_f(float z) {
    const float sg = fast_rcp(1.0f + fast_ex2(-1.4426950408889634f * z));
    return sg * (1.0f + z * (1.0f - sg));
}

// ---- pass 1 (forward): per-(image, slab, group) count, mean and M2 (sum of squared deviations from that mean) -------------
// The variance is never formed as E[x^2] - E[x]^2: in fp32 that loses (mean / std)^2 * eps_fp32 of it, i.e. every bit once a
// group's mean is a few thousand of its standard deviations.  Each pixel lane sums (x - K) and (x - K)^2 about its own first
// value K instead, which keeps the sums at the scale of the spread (K is one of the values, so it contributes to M2 whatever
// it is); the lane partials then meet as (count, mean, M2) through Chan's pairwise update, in a FIXED order (no atomics).
// grid (nslab, B); part[((b * nslab + slab) * 32 + g) * 3 + {n, mean, M2}].  Thread -> (16-byte vector v of a pixel row,
// pixel lane pl): consecutive threads read consecutive vectors; the per-lane, per-channel mean and M2 meet in dynamic shared
// memory s[pl][2][C].
__device__ __forceinline__ int gn_lanes(int C) {  // pixel lanes a 256-thread block runs side by side
    const int cv = C / 8;
    return cv >= GN_THREADS ? 1 : GN_THREADS / cv;
}
// Fold the partial (nb, mb, m2b) into (n, m, m2) (Chan, Golub & LeVeque): exact algebra, no cancellation between large terms.
__device__ __forceinline__ void gn_chan_merge(float& n, float& m, float& m2, float nb, float mb, float m2b) {
    if (nb == 0.f) return;
    if (n == 0.f) { n = nb; m = mb; m2 = m2b; return; }
    const float nn = n + nb, d = mb - m, r = nb * fast_rcp(nn);
    m = fmaf(d, r, m);
    m2 += fmaf(d * d * n, r, m2b);
    n = nn;
}
__global__ void __launch_bounds__(GN_THREADS) gn_stats_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ part, int HW, int C,
                                                              int pix_per_slab) {
    extern __shared__ float gn_smem[];
    const int b = blockIdx.y, slab = blockIdx.x, nslab = gridDim.x;
    const int cv = C / 8;
    const int lanes = gn_lanes(C);
    const int p0 = slab * pix_per_slab;
    const int p1 = min(HW, p0 + pix_per_slab);  // p1 <= p0 for an empty trailing slab: every lane count is then 0
    const long long base = static_cast<long long>(b) * HW * C;
    for (int v0 = 0; v0 < cv; v0 += GN_THREADS) {  // (one pass unless a pixel row has more than 256 vectors: C > 2048)
        const int cvb = min(GN_THREADS, cv - v0);
        const int v = v0 + static_cast<int>(threadIdx.x) % cvb, pl = static_cast<int>(threadIdx.x) / cvb;
        if (pl < lanes) {
            float K[8] = {0, 0, 0, 0, 0, 0, 0, 0}, a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            const int first = p0 + pl;
            if (first < p1) {  // the lane's first pixel is its shift K (and contributes x - K = 0 to the sums)
                const uint4 t = *reinterpret_cast<const uint4*>(x + base + static_cast<long long>(first) * C + v * 8);
                K[0] = bf16lo(t.x); K[1] = bf16hi(t.x); K[2] = bf16lo(t.y); K[3] = bf16hi(t.y);
                K[4] = bf16lo(t.z); K[5] = bf16hi(t.z); K[6] = bf16lo(t.w); K[7] = bf16hi(t.w);
            }
            for (int pix = first + lanes; pix < p1; pix += lanes) {
                const uint4 t = *reinterpret_cast<const uint4*>(x + base + static_cast<long long>(pix) * C + v * 8);
                const float f[8] = {bf16lo(t.x), bf16hi(t.x), bf16lo(t.y), bf16hi(t.y), bf16lo(t.z), bf16hi(t.z), bf16lo(t.w), bf16hi(t.w)};
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float d = f[k] - K[k];
                    a[k] += d;
                    q[k] = fmaf(d, d, q[k]);
                }
            }
            const float rn = first < p1 ? 1.0f / static_cast<float>((p1 - first + lanes - 1) / lanes) : 0.f;
            float* dst = gn_smem + static_cast<long long>(pl) * 2 * C + v * 8;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                dst[k] = fmaf(a[k], rn, K[k]);                     // lane mean
                dst[C + k] = fmaxf(fmaf(-a[k] * a[k], rn, q[k]), 0.f);  // lane M2 = sum (x - K)^2 - (sum (x - K))^2 / n
            }
        }
    }
    __syncthreads();
    const int cpg = C / GN_GROUPS;
    if (threadIdx.x < GN_GROUPS) {
        float n = 0.f, m = 0.f, m2 = 0.f;
        for (int pl = 0; pl < lanes; ++pl) {
            const int first = p0 + pl;
            const float nl = first < p1 ? static_cast<float>((p1 - first + lanes - 1) / lanes) : 0.f;
            for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c)
                gn_chan_merge(n, m, m2, nl, gn_smem[pl * 2 * C + c], gn_smem[pl * 2 * C + C + c]);
        }
        float* o = part + ((static_cast<long long>(b) * nslab + slab) * GN_GROUPS + threadIdx.x) * 3;
        o[0] = n;
        o[1] = m;
        o[2] = m2;
    }
}

// ---- pass 1b: slab partials -> mean / rstd per (image, group), merged in slab order -----------------------------------
__global__ void gn_finish_stats_kernel(const float* __restrict__ part, int nslab, float inv_n, float eps, float* __restrict__ mean,
                                       float* __restrict__ rstd, int total) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (b, g)
    if (i >= total) return;
    const int b = i / GN_GROUPS, g = i % GN_GROUPS;
    float n = 0.f, m = 0.f, m2 = 0.f;
    for (int s = 0; s < nslab; ++s) {
        const float* o = part + ((static_cast<long long>(b) * nslab + s) * GN_GROUPS + g) * 3;
        gn_chan_merge(n, m, m2, o[0], o[1], o[2]);
    }
    mean[i] = m;
    rstd[i] = rsqrtf(m2 * inv_n + eps);
}

// ---- pass 2 (forward): y = bf16(act(x_hat * gamma + beta)) --------------------------------------------------------
__global__ void __launch_bounds__(GN_THREADS) gn_apply_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, const float* __restrict__ mean,
                                                              const float* __restrict__ rstd, __nv_bfloat16* __restrict__ y, int HW, int C,
                                                              long long total_vec, int silu) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total_vec) return;
    const int cv = C / 8, cpg = C / GN_GROUPS;
    const int v = static_cast<int>(i % cv);
    const long long pix = i / cv;
    const int b = static_cast<int>(pix / HW);
    const uint4 t = *reinterpret_cast<const uint4*>(x + i * 8);
    const float f[8] = {bf16lo(t.x), bf16hi(t.x), bf16lo(t.y), bf16hi(t.y), bf16lo(t.z), bf16hi(t.z), bf16lo(t.w), bf16hi(t.w)};
    float o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int c = v * 8 + k;
        const int g = c / cpg;
        const float z = (f[k] - mean[b * GN_GROUPS + g]) * rstd[b * GN_GROUPS + g] * __ldg(gamma + c) + __ldg(beta + c);
        o[k] = silu ? silu_f(z) : z;
    }
    uint4 w;
    w.x = pack_bf16x2(o[0], o[1]); w.y = pack_bf16x2(o[2], o[3]); w.z = pack_bf16x2(o[4], o[5]); w.w = pack_bf16x2(o[6], o[7]);
    *reinterpret_cast<uint4*>(y + i * 8) = w;
}

// ---- backward pass 1: per-(image, slab) group sums of h = g * gamma and h * x_hat, and per-channel sums of g, g * x_hat -----
// g = dy * act'(z).  part_g[((b*nslab+slab)*32+grp)*2], part_c[((b*nslab+slab)*C + c)*2] = {sum g, sum g x_hat}
__global__ void __launch_bounds__(GN_THREADS) gn_bwd_stats_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                                                  const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                  const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                  float* __restrict__ part_g, float* __restrict__ part_c, int HW, int C,
                                                                  int pix_per_slab, int silu) {
    extern __shared__ float gn_smem[];
    const int b = blockIdx.y, slab = blockIdx.x, nslab = gridDim.x;
    const int cv = C / 8, cpg = C / GN_GROUPS;
    const int lanes = gn_lanes(C);
    const int p0 = slab * pix_per_slab;
    const int p1 = min(HW, p0 + pix_per_slab);
    const long long base = static_cast<long long>(b) * HW * C;
    for (int v0 = 0; v0 < cv; v0 += GN_THREADS) {
        const int cvb = min(GN_THREADS, cv - v0);
        const int v = v0 + static_cast<int>(threadIdx.x) % cvb, pl = static_cast<int>(threadIdx.x) / cvb;
        if (pl < lanes) {
            float ga[8], be[8], mu[8], rs[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int c = v * 8 + k;
                ga[k] = __ldg(gamma + c); be[k] = __ldg(beta + c);
                mu[k] = mean[b * GN_GROUPS + c / cpg]; rs[k] = rstd[b * GN_GROUPS + c / cpg];
            }
            float a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            for (int pix = p0 + pl; pix < p1; pix += lanes) {
                const uint4 t = *reinterpret_cast<const uint4*>(x + base + static_cast<long long>(pix) * C + v * 8);
                const uint4 d = *reinterpret_cast<const uint4*>(dy + base + static_cast<long long>(pix) * C + v * 8);
                const float f[8] = {bf16lo(t.x), bf16hi(t.x), bf16lo(t.y), bf16hi(t.y), bf16lo(t.z), bf16hi(t.z), bf16lo(t.w), bf16hi(t.w)};
                const float e[8] = {bf16lo(d.x), bf16hi(d.x), bf16lo(d.y), bf16hi(d.y), bf16lo(d.z), bf16hi(d.z), bf16lo(d.w), bf16hi(d.w)};
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float xh = (f[k] - mu[k]) * rs[k];
                    const float gg = silu ? e[k] * silu_grad_f(fmaf(xh, ga[k], be[k])) : e[k];
                    a[k] += gg;
                    q[k] = fmaf(gg, xh, q[k]);
                }
            }
            float* dst = gn_smem + static_cast<long long>(pl) * 2 * C + v * 8;
#pragma unroll
            for (int k = 0; k < 8; ++k) { dst[k] = a[k]; dst[C + k] = q[k]; }
        }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += GN_THREADS) {  // lanes -> lane 0 (fixed order), then out
        float a = 0.f, q = 0.f;
        for (int pl = 0; pl < lanes; ++pl) { a += gn_smem[pl * 2 * C + c]; q += gn_smem[pl * 2 * C + C + c]; }
        gn_smem[c] = a;
        gn_smem[C + c] = q;
        float* o = part_c + ((static_cast<long long>(b) * nslab + slab) * C + c) * 2;
        o[0] = a;
        o[1] = q;
    }
    __syncthreads();
    if (threadIdx.x < GN_GROUPS) {
        float a = 0.f, q = 0.f;
        for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c) {
            const float gmm = __ldg(gamma + c);
            a = fmaf(gn_smem[c], gmm, a);
            q = fmaf(gn_smem[C + c], gmm, q);
        }
        float* o = part_g + ((static_cast<long long>(b) * nslab + slab) * GN_GROUPS + threadIdx.x) * 2;
        o[0] = a;
        o[1] = q;
    }
}

// group sums over slabs -> c1 = mean(h), c2 = mean(h x_hat) per (image, group); per-channel sums over images and slabs -> dgamma, dbeta
__global__ void gn_bwd_finish_kernel(const float* __restrict__ part_g, const float* __restrict__ part_c, int B, int nslab, int C, float inv_n,
                                     float* __restrict__ c1, float* __restrict__ c2, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                     int accumulate) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B * GN_GROUPS) {
        const int b = i / GN_GROUPS, g = i % GN_GROUPS;
        float a = 0.f, q = 0.f;
        for (int s = 0; s < nslab; ++s) {
            const float* o = part_g + ((static_cast<long long>(b) * nslab + s) * GN_GROUPS + g) * 2;
            a += o[0];
            q += o[1];
        }
        c1[i] = a * inv_n;
        c2[i] = q * inv_n;
    }
    if (i < C) {
        float a = 0.f, q = 0.f;
        for (int bs = 0; bs < B * nslab; ++bs) {
            const float* o = part_c + (static_cast<long long>(bs) * C + i) * 2;
            a += o[0];
            q += o[1];
        }
        dbeta[i] = accumulate ? dbeta[i] + a : a;
        dgamma[i] = accumulate ? dgamma[i] + q : q;
    }
}

// ---- backward pass 2: dx = bf16( rstd * (h - c1 - x_hat * c2) ),  h = dy * act'(z) * gamma -------------------------------
__global__ void __launch_bounds__(GN_THREADS) gn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                                                  const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                  const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                  const float* __restrict__ c1, const float* __restrict__ c2,
                                                                  __nv_bfloat16* __restrict__ dx, int HW, int C, long long total_vec, int silu) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total_vec) return;
    const int cv = C / 8, cpg = C / GN_GROUPS;
    const int v = static_cast<int>(i % cv);
    const long long pix = i / cv;
    const int b = static_cast<int>(pix / HW);
    const uint4 t = *reinterpret_cast<const uint4*>(x + i * 8);
    const uint4 d = *reinterpret_cast<const uint4*>(dy + i * 8);
    const float f[8] = {bf16lo(t.x), bf16hi(t.x), bf16lo(t.y), bf16hi(t.y), bf16lo(t.z), bf16hi(t.z), bf16lo(t.w), bf16hi(t.w)};
    const float e[8] = {bf16lo(d.x), bf16hi(d.x), bf16lo(d.y), bf16hi(d.y), bf16lo(d.z), bf16hi(d.z), bf16lo(d.w), bf16hi(d.w)};
    float o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int c = v * 8 + k;
        const int gi = b * GN_GROUPS + c / cpg;
        const float rs = rstd[gi];
        const float xh = (f[k] - mean[gi]) * rs;
        const float gm = __ldg(gamma + c);
        const float gg = silu ? e[k] * silu_grad_f(fmaf(xh, gm, __ldg(beta + c))) : e[k];
        o[k] = rs * (gg * gm - c1[gi] - xh * c2[gi]);
    }
    uint4 w;
    w.x = pack_bf16x2(o[0], o[1]); w.y = pack_bf16x2(o[2], o[3]); w.z = pack_bf16x2(o[4], o[5]); w.w = pack_bf16x2(o[6], o[7]);
    *reinterpret_cast<uint4*>(dx + i * 8) = w;
}

static int gn_check(const char* entry, int B, int HW, int C) {
    if (B <= 0 || HW <= 0 || C <= 0) return refuse(B200_ERR_ARG, entry, "non-positive size");
    if (C % 8 != 0 || C % GN_GROUPS != 0 || C > GN_MAX_C) return refuse(B200_ERR_ARG, entry, "need C % 32 == 0 and C <= 2560");
    return 0;
}

static int gn_smem_bytes(int C) {  // s[lanes][2][C] floats: <= 20 KB for every supported width
    const int cv = C / 8;
    const int lanes = cv >= GN_THREADS ? 1 : GN_THREADS / cv;
    return lanes * 2 * C * 4;
}

static int gn_slabs(int B, int HW) {
    // enough blocks to fill the 132 SMs of an H100 a few times over, at least 64 pixels per slab
    int nslab = (4 * 132 + B - 1) / B;
    const int max_slab = (HW + 63) / 64;
    if (nslab > max_slab) nslab = max_slab;
    if (nslab < 1) nslab = 1;
    return nslab;
}

}  // namespace b200

using namespace b200;

extern "C" long long b200_groupnorm_workspace_floats(int B, int HW, int C) {
    const int nslab = gn_slabs(B, HW);
    // backward: B*nslab*32*2 + B*nslab*C*2 + 2*B*32; the forward's B*nslab*32*3 fits in that because C >= 32
    return static_cast<long long>(B) * nslab * GN_GROUPS * 2 + static_cast<long long>(B) * nslab * C * 2 + 2ll * B * GN_GROUPS;
}

extern "C" int b200_groupnorm_silu_fwd(const void* x_bf16, const float* gamma, const float* beta, void* y_bf16, float* mean, float* rstd,
                                       float* workspace, int B, int HW, int C, float eps, int silu, cudaStream_t stream) {
    const char* E = "groupnorm_fwd";
    int rc = gn_check(E, B, HW, C);
    if (rc) return rc;
    if (!x_bf16 || !gamma || !beta || !y_bf16 || !mean || !rstd || !workspace) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {x_bf16, y_bf16})) return refuse(B200_ERR_ALIGN, E, "x / y not 16-byte aligned");
    if (!aligned(4, {gamma, beta, mean, rstd, workspace})) return refuse(B200_ERR_ALIGN, E, "gamma / beta / mean / rstd / workspace not 4-byte aligned");
    const int nslab = gn_slabs(B, HW);
    const int pps = (HW + nslab - 1) / nslab;
    const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(x_bf16);
    gn_stats_kernel<<<dim3(nslab, B), GN_THREADS, gn_smem_bytes(C), stream>>>(x, workspace, HW, C, pps);
    if ((rc = check_launch("groupnorm_stats")) != 0) return rc;
    const float inv_n = 1.0f / (static_cast<float>(HW) * static_cast<float>(C / GN_GROUPS));
    gn_finish_stats_kernel<<<(B * GN_GROUPS + 127) / 128, 128, 0, stream>>>(workspace, nslab, inv_n, eps, mean, rstd, B * GN_GROUPS);
    if ((rc = check_launch("groupnorm_finish_stats")) != 0) return rc;
    const long long total_vec = static_cast<long long>(B) * HW * (C / 8);
    gn_apply_kernel<<<static_cast<unsigned>((total_vec + GN_THREADS - 1) / GN_THREADS), GN_THREADS, 0, stream>>>(
        x, gamma, beta, mean, rstd, reinterpret_cast<__nv_bfloat16*>(y_bf16), HW, C, total_vec, silu);
    return check_launch("groupnorm_apply");
}

extern "C" int b200_groupnorm_silu_bwd(const void* x_bf16, const void* dy_bf16, const float* gamma, const float* beta, const float* mean,
                                       const float* rstd, void* dx_bf16, float* dgamma, float* dbeta, float* workspace, int B, int HW, int C,
                                       int silu, int accumulate, cudaStream_t stream) {
    const char* E = "groupnorm_bwd";
    int rc = gn_check(E, B, HW, C);
    if (rc) return rc;
    if (!x_bf16 || !dy_bf16 || !gamma || !beta || !mean || !rstd || !dx_bf16 || !dgamma || !dbeta || !workspace)
        return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {x_bf16, dy_bf16, dx_bf16})) return refuse(B200_ERR_ALIGN, E, "x / dy / dx not 16-byte aligned");
    if (!aligned(4, {gamma, beta, mean, rstd, dgamma, dbeta, workspace}))
        return refuse(B200_ERR_ALIGN, E, "gamma / beta / mean / rstd / dgamma / dbeta / workspace not 4-byte aligned");
    const int nslab = gn_slabs(B, HW);
    const int pps = (HW + nslab - 1) / nslab;
    float* part_g = workspace;
    float* part_c = part_g + static_cast<long long>(B) * nslab * GN_GROUPS * 2;
    float* c1 = part_c + static_cast<long long>(B) * nslab * C * 2;
    float* c2 = c1 + B * GN_GROUPS;
    const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(x_bf16);
    const __nv_bfloat16* dy = reinterpret_cast<const __nv_bfloat16*>(dy_bf16);
    gn_bwd_stats_kernel<<<dim3(nslab, B), GN_THREADS, gn_smem_bytes(C), stream>>>(x, dy, gamma, beta, mean, rstd, part_g, part_c, HW, C, pps, silu);
    if ((rc = check_launch("groupnorm_bwd_stats")) != 0) return rc;
    const float inv_n = 1.0f / (static_cast<float>(HW) * static_cast<float>(C / GN_GROUPS));
    const int n = (B * GN_GROUPS > C ? B * GN_GROUPS : C);
    gn_bwd_finish_kernel<<<(n + 127) / 128, 128, 0, stream>>>(part_g, part_c, B, nslab, C, inv_n, c1, c2, dgamma, dbeta, accumulate);
    if ((rc = check_launch("groupnorm_bwd_finish")) != 0) return rc;
    const long long total_vec = static_cast<long long>(B) * HW * (C / 8);
    gn_bwd_apply_kernel<<<static_cast<unsigned>((total_vec + GN_THREADS - 1) / GN_THREADS), GN_THREADS, 0, stream>>>(
        x, dy, gamma, beta, mean, rstd, c1, c2, reinterpret_cast<__nv_bfloat16*>(dx_bf16), HW, C, total_vec, silu);
    return check_launch("groupnorm_bwd_apply");
}
