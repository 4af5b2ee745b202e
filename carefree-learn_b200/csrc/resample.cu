// Nearest 2x upsampling of channels-last bf16 activations and its backward, the 2x2 sum (include/b200_cflearn_ext.h).
// One thread per 8 channels of one low-resolution pixel: 16-byte loads and stores.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200_internal.h"
#include "../../include/b200_cflearn_ext.h"

namespace b200 {

// offset (in 8-channel groups) of high-resolution pixel (2y + i, 2x + j) of low-resolution group g = ((b H + y) W + x) C8 + c8
__device__ __forceinline__ long long hi_group(long long g, int H, int W, int C8, int i, int j) {
    const int c8 = static_cast<int>(g % C8);
    const long long pix = g / C8;
    const int x = static_cast<int>(pix % W);
    const long long t = pix / W;
    const int y = static_cast<int>(t % H);
    const long long b = t / H;
    return ((b * 2 * H + 2 * y + i) * (2ll * W) + 2 * x + j) * C8 + c8;
}

__global__ void upsample_nearest2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, long long groups, int H, int W, int C8) {
    const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (g >= groups) return;
    const uint4 v = x[g];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) out[hi_group(g, H, W, C8, i, j)] = v;
}

__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

__global__ void sum2x2_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, long long groups, int H, int W, int C8) {
    const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (g >= groups) return;
    float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const uint4 v = x[hi_group(g, H, W, C8, i, j)];
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                s[2 * k] += bf_lo(w[k]);
                s[2 * k + 1] += bf_hi(w[k]);
            }
        }
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const __nv_bfloat162 p = __floats2bfloat162_rn(s[2 * k], s[2 * k + 1]);
        o[k] = *reinterpret_cast<const uint32_t*>(&p);
    }
    out[g] = make_uint4(o[0], o[1], o[2], o[3]);
}

static int check_copy(const char* entry, const void* x, const void* out, int B, int H, int W, int C) {
    if (B <= 0 || H <= 0 || W <= 0 || C <= 0) return refuse(B200_ERR_ARG, entry, "non-positive size");
    if (C % 8 != 0) return refuse(B200_ERR_ARG, entry, "C must be a multiple of 8");
    if (4ll * B * H * W * C > 0x7fffffffffffll) return refuse(B200_ERR_ARG, entry, "too many elements");
    if (x == nullptr || out == nullptr) return refuse(B200_ERR_ARG, entry, "null pointer");
    if (!aligned(16, {x, out})) return refuse(B200_ERR_ALIGN, entry, "x / out not 16-byte aligned");
    return 0;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_upsample_nearest2x_bf16(const void* x, void* out, int B, int H, int W, int C, cudaStream_t stream) {
    if (const int rc = check_copy("upsample_nearest2x", x, out, B, H, W, C)) return rc;
    const long long groups = static_cast<long long>(B) * H * W * (C / 8);
    upsample_nearest2x_kernel<<<static_cast<unsigned>((groups + 255) / 256), 256, 0, stream>>>(
        reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), groups, H, W, C / 8);
    return check_launch("upsample_nearest2x");
}

extern "C" int b200_sum2x2_bf16(const void* x, void* out, int B, int H, int W, int C, cudaStream_t stream) {
    if (const int rc = check_copy("sum2x2", x, out, B, H, W, C)) return rc;
    const long long groups = static_cast<long long>(B) * H * W * (C / 8);
    sum2x2_kernel<<<static_cast<unsigned>((groups + 255) / 256), 256, 0, stream>>>(
        reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), groups, H, W, C / 8);
    return check_launch("sum2x2");
}
