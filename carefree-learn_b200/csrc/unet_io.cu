// The two ends of the SD-v1.5 UNet's training step (include/b200_cflearn_ext.h): the channel padding that lets the 4-channel
// stem and head run on the 64-channel implicit-GEMM convolutions (plain, or fused with the DDPM noising of the latent), and the
// DDPM noise-prediction loss with its gradient.
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

// The element reads are a Source's: src(i, b) returns the bf16 bits of element i (of image b) of the real channels.
template <typename T>
struct CastSource {
    const T* x;
    __device__ __forceinline__ uint16_t operator()(long long i, long long) const { return to_bf16_bits(x[i]); }
};

template <bool kChannelsLast, typename Source>
__global__ void pad_channels_kernel(Source src, uint4* __restrict__ out, long long groups, int C, int HW, int Cp8) {
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
        if (c < C) lo = src(kChannelsLast ? pix * C + c : (b * C + c) * HW + p, b);
        if (c + 1 < C) hi = src(kChannelsLast ? pix * C + c + 1 : (b * C + c + 1) * HW + p, b);
        w[k] = lo | (hi << 16);
    }
    out[g] = make_uint4(w[0], w[1], w[2], w[3]);
}

// ---- DDPM noising ----------------------------------------------------------------------------------------------------------------
// bf16(fl(fl(a[t_b] x0) + fl(s[t_b] noise))): q_sample's `w_net * net + w_noise * noise` in fp32 with no contraction, then autocast's
// cast at the stem.  A timestep outside [0, T) reads no table entry: it sets *bad and the image's elements become NaN.
struct QSampleSource {
    const float* x0;
    const float* noise;
    const long long* t;
    const float* a;
    const float* s;
    long long T;
    int* bad;
    __device__ __forceinline__ uint16_t operator()(long long i, long long b) const {
        const long long tb = t[b];
        if (tb < 0 || tb >= T) {
            atomicExch(bad, 1);
            return 0x7fc0u;  // bf16 NaN
        }
        return to_bf16_bits(__fadd_rn(__fmul_rn(a[tb], x0[i]), __fmul_rn(s[tb], noise[i])));
    }
};

template <typename Source>
static void launch_pad(Source src, bool channels_last, uint4* out, int B, int C, int H, int W, int Cp, cudaStream_t stream) {
    const long long groups = static_cast<long long>(B) * H * W * (Cp / 8);
    const unsigned grid = static_cast<unsigned>((groups + 255) / 256);
    if (channels_last) pad_channels_kernel<true><<<grid, 256, 0, stream>>>(src, out, groups, C, H * W, Cp / 8);
    else pad_channels_kernel<false><<<grid, 256, 0, stream>>>(src, out, groups, C, H * W, Cp / 8);
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

// ---- one DDIM denoising step ---------------------------------------------------------------------------------------------------
// The reference's DDIMSampler update (samplers/ddim.py:195-239, schema.py:255) with its rounding points: classifier-free guidance
// as eager's three bf16 tensor ops, then the fp32 update, each operation rounded, in the reference's order.  The per-step scalars
// come from coef[step] = {s1m, sqrt_a, sqrt_ap, c_dir, sigma} (fp32, computed on the host as the reference computes them).
constexpr int kDdimCoefs = 5;

__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

struct DdimArgs {
    const __nv_bfloat16* eps;     // [B, H, W, C]
    const __nv_bfloat16* eps_u;   // [B, H, W, C] or nullptr
    float scale;
    int guided;                   // eps_u given and scale != 1
    float* x;                     // [B, C, H, W]
    const float* noise;           // [B, C, H, W]
    const float* coef;            // [S, kDdimCoefs]
    const long long* ts_table;    // [S]
    int S;
    float temperature;
    const int* step_dev;
    int* bad;
    uint4* next_in;               // [copies B, H, W, Cp]
    long long* next_ts;           // [copies B]
    int copies, B, C, HW, Cp8;
    long long groups;             // B HW Cp8
};

// One thread per 8 channels of one pixel of next_in, as pad_channels_kernel: the threads whose group holds real channels also
// advance x for those channels.  Reads of the counter and the table are uniform across the grid.
__global__ void ddim_step_kernel(DdimArgs a) {
    const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int step = *a.step_dev;
    const bool ok = step >= 0 && step < a.S;
    const bool has_next = ok && step + 1 < a.S;
    if (has_next && g < static_cast<long long>(a.copies) * a.B) a.next_ts[g] = a.ts_table[step + 1];
    if (g >= a.groups) return;
    const int c0 = static_cast<int>(g % a.Cp8) * 8;
    const long long pix = g / a.Cp8;  // b HW + p
    const long long b = pix / a.HW;
    const long long p = pix - b * a.HW;
    if (!ok) {
        if (g == 0) atomicExch(a.bad, 1);
        for (int c = c0; c < c0 + 8 && c < a.C; ++c) a.x[(b * a.C + c) * a.HW + p] = __int_as_float(0x7fc00000);
        return;
    }
    float s1m = 0.f, sqrt_a = 1.f, sqrt_ap = 0.f, c_dir = 0.f, sigma = 0.f;
    if (c0 < a.C) {
        const float* k = a.coef + static_cast<long long>(step) * kDdimCoefs;
        s1m = k[0], sqrt_a = k[1], sqrt_ap = k[2], c_dir = k[3], sigma = k[4];
    }
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        uint32_t half[2] = {0u, 0u};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = c0 + 2 * j + h;
            if (c >= a.C) continue;
            float e = __bfloat162float(a.eps[pix * a.C + c]);
            if (a.guided) {  // eps_uncond + scale * (eps - eps_uncond), three bf16 tensor ops
                const float u = __bfloat162float(a.eps_u[pix * a.C + c]);
                const float d = bf16_round(__fsub_rn(e, u));
                const float m = bf16_round(__fmul_rn(a.scale, d));
                e = bf16_round(__fadd_rn(u, m));
            }
            const long long i = (b * a.C + c) * a.HW + p;
            const float x0 = __fdiv_rn(__fsub_rn(a.x[i], __fmul_rn(s1m, e)), sqrt_a);
            const float dir = __fmul_rn(c_dir, e);
            const float nz = __fmul_rn(__fmul_rn(sigma, a.noise[i]), a.temperature);
            const float out = __fadd_rn(__fadd_rn(__fmul_rn(sqrt_ap, x0), dir), nz);
            a.x[i] = out;
            half[h] = to_bf16_bits(out);
        }
        w[j] = half[0] | (half[1] << 16);
    }
    if (!has_next) return;
    const uint4 v = make_uint4(w[0], w[1], w[2], w[3]);
    for (int k = 0; k < a.copies; ++k) a.next_in[g + k * a.groups] = v;
}

__global__ void ddim_increment_kernel(int* counter) { counter[0] += 1; }

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
    uint4* o = reinterpret_cast<uint4*>(out);
    if (x_f32) launch_pad(CastSource<float>{static_cast<const float*>(x)}, x_channels_last != 0, o, B, C, H, W, Cp, stream);
    else launch_pad(CastSource<uint16_t>{static_cast<const uint16_t*>(x)}, x_channels_last != 0, o, B, C, H, W, Cp, stream);
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

extern "C" int b200_q_sample_pad_bf16(const float* x0, const float* noise, int channels_last, const long long* timesteps,
                                      const float* sqrt_alphas_cumprod, const float* sqrt_one_minus_alphas_cumprod, long long T,
                                      int* bad_flag, void* out, int B, int C, int H, int W, int Cp, cudaStream_t stream) {
    const char* E = "q_sample_pad";
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || Cp <= 0 || T <= 0) return refuse(B200_ERR_ARG, E, "non-positive size");
    if (Cp % 8 != 0) return refuse(B200_ERR_ARG, E, "Cp must be a multiple of 8");
    if (C > Cp) return refuse(B200_ERR_ARG, E, "C must be at most Cp");
    if (channels_last != 0 && channels_last != 1) return refuse(B200_ERR_ARG, E, "flags must be 0 or 1");
    if (static_cast<long long>(H) * W > 0x7fffffffll) return refuse(B200_ERR_ARG, E, "H * W must be at most 2^31 - 1");
    if (static_cast<long long>(B) * H * W > kMaxElements / Cp) return refuse(B200_ERR_ARG, E, "too many elements");
    if (x0 == nullptr || noise == nullptr || timesteps == nullptr || sqrt_alphas_cumprod == nullptr ||
        sqrt_one_minus_alphas_cumprod == nullptr || bad_flag == nullptr || out == nullptr)
        return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(4, {x0, noise, sqrt_alphas_cumprod, sqrt_one_minus_alphas_cumprod, bad_flag}) || !aligned(8, {timesteps}))
        return refuse(B200_ERR_ALIGN, E, "pointers not aligned to their element size");
    if (!aligned(16, {out})) return refuse(B200_ERR_ALIGN, E, "out not 16-byte aligned");
    launch_pad(QSampleSource{x0, noise, timesteps, sqrt_alphas_cumprod, sqrt_one_minus_alphas_cumprod, T, bad_flag}, channels_last != 0,
               reinterpret_cast<uint4*>(out), B, C, H, W, Cp, stream);
    return check_launch("q_sample_pad");
}

extern "C" int b200_ddim_step_bf16(const void* eps, const void* eps_uncond, float guidance_scale, float* x, const float* noise,
                                   const float* coef, const long long* ts_table, int S, float temperature,
                                   int* step_dev, int increment, int* bad_flag, void* next_in, long long* next_ts, int copies,
                                   int B, int C, int H, int W, int Cp, cudaStream_t stream) {
    const char* E = "ddim_step";
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || Cp <= 0 || S <= 0) return refuse(B200_ERR_ARG, E, "non-positive size");
    if (Cp % 8 != 0) return refuse(B200_ERR_ARG, E, "Cp must be a multiple of 8");
    if (C > Cp) return refuse(B200_ERR_ARG, E, "C must be at most Cp");
    if (copies != 1 && copies != 2) return refuse(B200_ERR_ARG, E, "copies must be 1 or 2");
    if (increment != 0 && increment != 1) return refuse(B200_ERR_ARG, E, "increment must be 0 or 1");
    if (copies == 2 && eps_uncond == nullptr) return refuse(B200_ERR_ARG, E, "copies = 2 needs eps_uncond");
    if (static_cast<long long>(H) * W > 0x7fffffffll) return refuse(B200_ERR_ARG, E, "H * W must be at most 2^31 - 1");
    if (static_cast<long long>(B) * H * W > kMaxElements / (2 * Cp)) return refuse(B200_ERR_ARG, E, "too many elements");
    if (eps == nullptr || x == nullptr || noise == nullptr || coef == nullptr || ts_table == nullptr || step_dev == nullptr ||
        bad_flag == nullptr || next_in == nullptr || next_ts == nullptr)
        return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(2, {eps, eps_uncond}) || !aligned(4, {x, noise, coef, step_dev, bad_flag}) || !aligned(8, {ts_table, next_ts}))
        return refuse(B200_ERR_ALIGN, E, "pointers not aligned to their element size");
    if (!aligned(16, {next_in})) return refuse(B200_ERR_ALIGN, E, "next_in not 16-byte aligned");
    DdimArgs a;
    a.eps = static_cast<const __nv_bfloat16*>(eps);
    a.eps_u = static_cast<const __nv_bfloat16*>(eps_uncond);
    a.scale = guidance_scale;
    a.guided = eps_uncond != nullptr && guidance_scale != 1.0f;
    a.x = x, a.noise = noise, a.coef = coef, a.ts_table = ts_table, a.S = S, a.temperature = temperature;
    a.step_dev = step_dev, a.bad = bad_flag;
    a.next_in = static_cast<uint4*>(next_in), a.next_ts = next_ts;
    a.copies = copies, a.B = B, a.C = C, a.HW = H * W, a.Cp8 = Cp / 8;
    a.groups = static_cast<long long>(B) * H * W * (Cp / 8);
    const long long threads = a.groups > 2ll * B ? a.groups : 2ll * B;
    ddim_step_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, stream>>>(a);
    int rc = check_launch("ddim_step");
    if (rc || !increment) return rc;
    ddim_increment_kernel<<<1, 1, 0, stream>>>(step_dev);  // after the step: the kernel above only reads the counter
    return check_launch("ddim_step_increment");
}
