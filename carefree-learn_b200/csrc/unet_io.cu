// The two ends of the SD-v1.5 UNet's training step (include/b200_cflearn_ext.h): the channel padding that lets the 4-channel
// stem and head run on the 64-channel implicit-GEMM convolutions, and the DDPM noise-prediction loss with its gradient.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200_internal.h"
#include "../../include/b200_cflearn_ext.h"

namespace b200 {

// ---- channel padding -------------------------------------------------------------------------------------------------------------
// One thread per 8 output channels of one pixel: a 16-byte store.  Source element (b, c, pixel p of HW): NCHW at (b C + c) HW + p,
// channels-last at (b HW + p) C + c.  fp32 is rounded to nearest even (__float2bfloat16_rn, the cast torch's CUDA kernels make);
// a bf16 source is copied bit for bit.
__device__ __forceinline__ uint16_t to_bf16_bits(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }
__device__ __forceinline__ uint16_t to_bf16_bits(uint16_t v) { return v; }

template <typename T, bool kChannelsLast>
__global__ void pad_channels_kernel(const T* __restrict__ x, uint4* __restrict__ out, long long groups, int C, int HW, int Cp8) {
    const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (g >= groups) return;
    const int c0 = static_cast<int>(g % Cp8) * 8;
    const long long pix = g / Cp8;  // b HW + p
    const long long b = pix / HW;
    const long long p = pix - b * HW;
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        uint32_t lo = 0, hi = 0;
        const int c = c0 + 2 * k;
        if (c < C) lo = to_bf16_bits(kChannelsLast ? x[pix * C + c] : x[(b * C + c) * HW + p]);
        if (c + 1 < C) hi = to_bf16_bits(kChannelsLast ? x[pix * C + c + 1] : x[(b * C + c + 1) * HW + p]);
        w[k] = lo | (hi << 16);
    }
    out[g] = make_uint4(w[0], w[1], w[2], w[3]);
}

// ---- the noise-prediction loss ---------------------------------------------------------------------------------------------------
// Each image's N elements are contiguous in NCHW and in channels-last alike, so both layouts are rows [B, N] here.
constexpr int kLossThreads = 1024;
// Largest element count either entry takes (2^38, more than a GPU holds): the 1-D grids of 256 threads stay below 2^31 blocks.
constexpr long long kMaxElements = 1ll << 38;

__device__ __forceinline__ float load_f32(const float* p, long long i) { return p[i]; }
__device__ __forceinline__ float load_f32(const __nv_bfloat16* p, long long i) { return __bfloat162float(p[i]); }

// loss = (sum over b of (sum over i of (pred - noise)^2) / N) / B in one CTA, in a fixed order: each thread's strided fp32 sum,
// the warp's xor tree, then the warps in index order, image after image.  No atomics: reruns are bit-identical.
template <typename TN>
__global__ void __launch_bounds__(kLossThreads) noise_loss_kernel(const __nv_bfloat16* __restrict__ pred, const TN* __restrict__ noise,
                                                                  int B, long long N, float* __restrict__ loss) {
    __shared__ float warp_sums[kLossThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float total = 0.f;  // thread 0's
    for (int b = 0; b < B; ++b) {
        const long long base = static_cast<long long>(b) * N;
        float s = 0.f;
        for (long long i = threadIdx.x; i < N; i += kLossThreads) {
            const float d = __fsub_rn(__bfloat162float(pred[base + i]), load_f32(noise, base + i));
            s = __fmaf_rn(d, d, s);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
        if (lane == 0) warp_sums[warp] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            float img = 0.f;
            for (int k = 0; k < kLossThreads / 32; ++k) img = __fadd_rn(img, warp_sums[k]);
            total = __fadd_rn(total, __fdiv_rn(img, static_cast<float>(N)));
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *loss = __fdiv_rn(total, static_cast<float>(B));
}

// d loss / d pred with eager's fp32 operations on CUDA (DESIGN.md section 2, tools/probe_noise_loss_rounding.py): the two means'
// backward multiply by the reciprocal of their counts, g = (g0 * fl(1/B)) * fl(1/N); mse_loss's backward is (2 (pred - noise)) g;
// then the bf16 cast of autocast's backward.
template <typename TN>
__global__ void noise_loss_grad_kernel(const __nv_bfloat16* __restrict__ pred, const TN* __restrict__ noise, long long total,
                                       float inv_b, float inv_n, const float* __restrict__ grad_out, __nv_bfloat16* __restrict__ dpred) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const float g = __fmul_rn(__fmul_rn(*grad_out, inv_b), inv_n);
    const float d = __fsub_rn(__bfloat162float(pred[i]), load_f32(noise, i));
    dpred[i] = __float2bfloat16_rn(__fmul_rn(__fmul_rn(2.0f, d), g));
}

}  // namespace b200

using namespace b200;

extern "C" int b200_pad_channels_bf16(const void* x, int x_f32, int x_channels_last, void* out, int B, int C, int H, int W, int Cp,
                                      cudaStream_t stream) {
    const char* E = "pad_channels";
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || Cp <= 0) return refuse(B200_ERR_ARG, E, "non-positive size");
    if (Cp % 8 != 0) return refuse(B200_ERR_ARG, E, "Cp must be a multiple of 8");
    if (C > Cp) return refuse(B200_ERR_ARG, E, "C must be at most Cp");
    if ((x_f32 != 0 && x_f32 != 1) || (x_channels_last != 0 && x_channels_last != 1)) return refuse(B200_ERR_ARG, E, "flags must be 0 or 1");
    if (static_cast<long long>(H) * W > 0x7fffffffll) return refuse(B200_ERR_ARG, E, "H * W must be at most 2^31 - 1");
    if (static_cast<long long>(B) * H * W > kMaxElements / Cp) return refuse(B200_ERR_ARG, E, "too many elements");
    if (x == nullptr || out == nullptr) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(x_f32 ? 4 : 2, {x})) return refuse(B200_ERR_ALIGN, E, "x not aligned to its element size");
    if (!aligned(16, {out})) return refuse(B200_ERR_ALIGN, E, "out not 16-byte aligned");
    const long long groups = static_cast<long long>(B) * H * W * (Cp / 8);
    const unsigned grid = static_cast<unsigned>((groups + 255) / 256);
    uint4* o = reinterpret_cast<uint4*>(out);
    const int HW = H * W;
    if (x_f32 && x_channels_last) pad_channels_kernel<float, true><<<grid, 256, 0, stream>>>(static_cast<const float*>(x), o, groups, C, HW, Cp / 8);
    else if (x_f32) pad_channels_kernel<float, false><<<grid, 256, 0, stream>>>(static_cast<const float*>(x), o, groups, C, HW, Cp / 8);
    else if (x_channels_last) pad_channels_kernel<uint16_t, true><<<grid, 256, 0, stream>>>(static_cast<const uint16_t*>(x), o, groups, C, HW, Cp / 8);
    else pad_channels_kernel<uint16_t, false><<<grid, 256, 0, stream>>>(static_cast<const uint16_t*>(x), o, groups, C, HW, Cp / 8);
    return check_launch("pad_channels");
}

extern "C" int b200_noise_prediction_loss_bf16(const void* pred, const void* noise, int noise_f32, float* loss, void* dpred,
                                               const float* grad_out, int B, long long N, cudaStream_t stream) {
    const char* E = "noise_prediction_loss";
    if (B <= 0 || N <= 0) return refuse(B200_ERR_ARG, E, "non-positive size");
    if (N > kMaxElements / B) return refuse(B200_ERR_ARG, E, "too many elements");
    if (noise_f32 != 0 && noise_f32 != 1) return refuse(B200_ERR_ARG, E, "noise_f32 must be 0 or 1");
    if (pred == nullptr || noise == nullptr) return refuse(B200_ERR_ARG, E, "null pointer");
    if ((loss == nullptr) == (dpred == nullptr)) return refuse(B200_ERR_ARG, E, "give exactly one of loss and dpred");
    if (dpred != nullptr && grad_out == nullptr) return refuse(B200_ERR_ARG, E, "dpred needs grad_out");
    if (!aligned(2, {pred, dpred}) || !aligned(noise_f32 ? 4 : 2, {noise}) || !aligned(4, {loss, grad_out}))
        return refuse(B200_ERR_ALIGN, E, "pointers not aligned to their element size");
    const __nv_bfloat16* p = static_cast<const __nv_bfloat16*>(pred);
    const float* nf = static_cast<const float*>(noise);
    const __nv_bfloat16* nb = static_cast<const __nv_bfloat16*>(noise);
    if (loss != nullptr) {
        if (noise_f32) noise_loss_kernel<<<1, kLossThreads, 0, stream>>>(p, nf, B, N, loss);
        else noise_loss_kernel<<<1, kLossThreads, 0, stream>>>(p, nb, B, N, loss);
        return check_launch("noise_prediction_loss");
    }
    const long long total = static_cast<long long>(B) * N;
    const unsigned grid = static_cast<unsigned>((total + 255) / 256);
    const float inv_b = 1.0f / static_cast<float>(B), inv_n = 1.0f / static_cast<float>(N);
    __nv_bfloat16* d = static_cast<__nv_bfloat16*>(dpred);
    if (noise_f32) noise_loss_grad_kernel<<<grid, 256, 0, stream>>>(p, nf, total, inv_b, inv_n, grad_out, d);
    else noise_loss_grad_kernel<<<grid, 256, 0, stream>>>(p, nb, total, inv_b, inv_n, grad_out, d);
    return check_launch("noise_prediction_loss_grad");
}
