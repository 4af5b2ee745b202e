// HBM-bound row kernels of the transformer-block training step: LayerNorm fwd/bwd, column sums (bias / gamma /
// beta grads), split-K reduction, patch-embed glue, softmax cross-entropy, casts.  All are coalesced 16-byte
// vector streams with warp-shuffle reductions; none of them re-reads a tensor.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <type_traits>

#include "b200_internal.h"
#include "ptx.cuh"
#include "../../include/b200_cflearn_ext.h"

namespace b200 {

// ------------------------------------------------------------------------------------------------
// error / bookkeeping
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

int set_error(int code, const char* msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg ? msg : "");
    return code;
}
int refuse(int code, const char* entry, const char* rule) {
    char msg[256];
    snprintf(msg, sizeof(msg), "%s: %s", entry, rule);
    return set_error(code, msg);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        char buf[256];
        snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
        return set_error(B200_ERR_LAUNCH, buf);
    }
    count_launch(1);
    return 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm forward: one warp per row, row held in registers (dim <= 1024, dim % 4 == 0)
// ------------------------------------------------------------------------------------------------
constexpr int LN_MAX_V4 = 8;  // float4 per lane

template <int NV>
__global__ void __launch_bounds__(256) layernorm_fwd_kernel(const float* __restrict__ x, long long ld_x,
                                                            const float* __restrict__ gamma,
                                                            const float* __restrict__ beta,
                                                            __nv_bfloat16* __restrict__ y, float* __restrict__ y32,
                                                            float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                            int rows, int dim, float eps) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const float* xr = x + static_cast<long long>(warp) * ld_x;
    float4 v[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = (lane + 32 * i) * 4;
        if (c < dim) {
            v[i] = *reinterpret_cast<const float4*>(xr + c);
            s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        } else {
            v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    const float inv_n = 1.0f / static_cast<float>(dim);
    const float mean = warp_sum(s) * inv_n;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = (lane + 32 * i) * 4;
        if (c < dim) {
            const float a = v[i].x - mean, b = v[i].y - mean, cc = v[i].z - mean, d = v[i].w - mean;
            ss += (a * a + b * b) + (cc * cc + d * d);
        }
    }
    const float var = warp_sum(ss) * inv_n;
    const float rstd = rsqrtf(var + eps);
    if (lane == 0) {
        mean_out[warp] = mean;
        rstd_out[warp] = rstd;
    }
    __nv_bfloat16* yr = y + static_cast<long long>(warp) * dim;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = (lane + 32 * i) * 4;
        if (c < dim) {
            const float4 g = *reinterpret_cast<const float4*>(gamma + c);
            const float4 b = *reinterpret_cast<const float4*>(beta + c);
            const float4 r = make_float4((v[i].x - mean) * rstd * g.x + b.x, (v[i].y - mean) * rstd * g.y + b.y,
                                         (v[i].z - mean) * rstd * g.z + b.z, (v[i].w - mean) * rstd * g.w + b.w);
            uint2 o;
            o.x = pack_bf16x2(r.x, r.y);
            o.y = pack_bf16x2(r.z, r.w);
            *reinterpret_cast<uint2*>(yr + c) = o;
            if (y32 != nullptr) *reinterpret_cast<float4*>(y32 + static_cast<long long>(warp) * dim + c) = r;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward: warps stride over rows.  Everything a row needs (x, dy, upstream residual grad) is requested
// up front -- 18 independent 8/16-byte loads per lane -- and the kernel is held to 128 registers so two 256-thread
// blocks fit per SM (a version at 148 registers with dres loaded after the reductions was latency-bound).
// Per-lane dgamma/dbeta partials live in registers and are reduced across the block's warps through shared memory
// -> part[blockIdx][0:dim] (dgamma) and part[blockIdx][dim:2*dim] (dbeta).
// DXSUM: additionally part[blockIdx][2*dim:3*dim] = column sums of the bf16-ROUNDED dx rows this block wrote, i.e. the
// bias gradient of the Linear whose dY this dx is (it used to be a separate pass over dx_bf16).  These partials are
// accumulated in each warp's private shared-memory row: 24 more accumulator registers would break the 128 budget.
// ------------------------------------------------------------------------------------------------
// DYF32: dy is fp32 (a LayerNorm whose output is the fp32 residual stream itself, e.g. CLIP's embedding_norm) instead of bf16.
template <int NV, bool DXSUM, bool DYF32>
__global__ void __launch_bounds__(256, 2) layernorm_bwd_kernel(const void* __restrict__ dy_any,
                                                               const float* __restrict__ x, long long ld_x,
                                                               const float* __restrict__ gamma,
                                                               const float* __restrict__ mean_in,
                                                               const float* __restrict__ rstd_in,
                                                               const float* __restrict__ dres, float* __restrict__ dx_out,
                                                               long long ld_dx, __nv_bfloat16* __restrict__ dx_bf16,
                                                               float* __restrict__ part, int rows, int dim) {
    extern __shared__ float sred[];  // [8 warps][2][dim] (+ [8 warps][dim] with DXSUM)
    const int wib = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int warps_per_block = blockDim.x >> 5;
    constexpr int NP = DXSUM ? 3 : 2;
    float* sx = sred + (warps_per_block * 2 + wib) * dim;  // this warp's running column sums of bf16(dx)
    if constexpr (DXSUM) {
        for (int c = lane * 4; c < dim; c += 128) *reinterpret_cast<float4*>(sx + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float4 dg[NV], db[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        dg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        db[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float fn = static_cast<float>(dim);
    for (int row = blockIdx.x * warps_per_block + wib; row < rows; row += gridDim.x * warps_per_block) {
        const float* xr = x + static_cast<long long>(row) * ld_x;
        const __nv_bfloat16* dyr = reinterpret_cast<const __nv_bfloat16*>(dy_any) + static_cast<long long>(row) * dim;
        const float* dyr32 = reinterpret_cast<const float*>(dy_any) + static_cast<long long>(row) * dim;
        const float* rr = dres != nullptr ? dres + static_cast<long long>(row) * ld_dx : nullptr;
        float4 xv[NV], rv[NV];
        uint2 dv[NV];
        float4 dv32[DYF32 ? NV : 1];
#pragma unroll
        for (int i = 0; i < NV; ++i) {  // issue every load of this row before touching any of them
            const int c = (lane + 32 * i) * 4;
            if (c < dim) {
                xv[i] = *reinterpret_cast<const float4*>(xr + c);
                if constexpr (DYF32) dv32[i] = *reinterpret_cast<const float4*>(dyr32 + c);
                else dv[i] = *reinterpret_cast<const uint2*>(dyr + c);
                rv[i] = rr != nullptr ? *reinterpret_cast<const float4*>(rr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        const float mean = mean_in[row];
        const float rstd = rstd_in[row];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int c = (lane + 32 * i) * 4;
            if (c < dim) {
                const float4 g = *reinterpret_cast<const float4*>(gamma + c);  // L1-resident
                float d0, d1, d2, d3;
                if constexpr (DYF32) { d0 = dv32[i].x; d1 = dv32[i].y; d2 = dv32[i].z; d3 = dv32[i].w; }
                else { d0 = bf16lo(dv[i].x); d1 = bf16hi(dv[i].x); d2 = bf16lo(dv[i].y); d3 = bf16hi(dv[i].y); }
                xv[i] = make_float4((xv[i].x - mean) * rstd, (xv[i].y - mean) * rstd, (xv[i].z - mean) * rstd, (xv[i].w - mean) * rstd);
                const float g0 = d0 * g.x, g1 = d1 * g.y, g2 = d2 * g.z, g3 = d3 * g.w;
                s1 += (g0 + g1) + (g2 + g3);
                s2 += (g0 * xv[i].x + g1 * xv[i].y) + (g2 * xv[i].z + g3 * xv[i].w);
                dg[i].x += d0 * xv[i].x; dg[i].y += d1 * xv[i].y; dg[i].z += d2 * xv[i].z; dg[i].w += d3 * xv[i].w;
                db[i].x += d0; db[i].y += d1; db[i].z += d2; db[i].w += d3;
            }
        }
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        const float term = rstd / fn;
        float* dxr = dx_out + static_cast<long long>(row) * ld_dx;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int c = (lane + 32 * i) * 4;
            if (c < dim) {
                const float4 g = *reinterpret_cast<const float4*>(gamma + c);
                float d0, d1, d2, d3;
                if constexpr (DYF32) { d0 = dv32[i].x; d1 = dv32[i].y; d2 = dv32[i].z; d3 = dv32[i].w; }
                else { d0 = bf16lo(dv[i].x); d1 = bf16hi(dv[i].x); d2 = bf16lo(dv[i].y); d3 = bf16hi(dv[i].y); }
                float4 o;
                o.x = (fn * (d0 * g.x) - s1 - xv[i].x * s2) * term + rv[i].x;
                o.y = (fn * (d1 * g.y) - s1 - xv[i].y * s2) * term + rv[i].y;
                o.z = (fn * (d2 * g.z) - s1 - xv[i].z * s2) * term + rv[i].z;
                o.w = (fn * (d3 * g.w) - s1 - xv[i].w * s2) * term + rv[i].w;
                *reinterpret_cast<float4*>(dxr + c) = o;
                if (dx_bf16 != nullptr) {
                    uint2 p;
                    p.x = pack_bf16x2(o.x, o.y);
                    p.y = pack_bf16x2(o.z, o.w);
                    *reinterpret_cast<uint2*>(dx_bf16 + static_cast<long long>(row) * dim + c) = p;
                    if constexpr (DXSUM) {  // (lane-private columns: no synchronisation)
                        float4 a = *reinterpret_cast<float4*>(sx + c);
                        a.x += bf16lo(p.x); a.y += bf16hi(p.x); a.z += bf16lo(p.y); a.w += bf16hi(p.y);
                        *reinterpret_cast<float4*>(sx + c) = a;
                    }
                }
            }
        }
    }
    // block reduce of dgamma / dbeta partials
    float* sg = sred + (wib * 2 + 0) * dim;
    float* sb = sred + (wib * 2 + 1) * dim;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = (lane + 32 * i) * 4;
        if (c < dim) {
            *reinterpret_cast<float4*>(sg + c) = dg[i];
            *reinterpret_cast<float4*>(sb + c) = db[i];
        }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < dim; c += blockDim.x) {
        float a = 0.f, b = 0.f;
        for (int w = 0; w < warps_per_block; ++w) {
            a += sred[(w * 2 + 0) * dim + c];
            b += sred[(w * 2 + 1) * dim + c];
        }
        part[static_cast<long long>(blockIdx.x) * NP * dim + c] = a;
        part[static_cast<long long>(blockIdx.x) * NP * dim + dim + c] = b;
        if constexpr (DXSUM) {
            float d = 0.f;
            for (int w = 0; w < warps_per_block; ++w) d += sred[(warps_per_block * 2 + w) * dim + c];
            part[static_cast<long long>(blockIdx.x) * NP * dim + 2 * dim + c] = d;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over bf16 rows (the SD-UNet SpatialTransformer's residual stream is bf16 under autocast): one warp per row,
// 8 bf16 (16 bytes) per lane access, the row kept packed in registers; dim % 8 == 0, dim <= 256 * NV.
// Forward: y = bf16(LN_fp32(x)), fp32 mean / rstd.
// ------------------------------------------------------------------------------------------------
constexpr int LNB_MAX_V8 = 8;  // 16-byte chunks per lane: dim <= 2048

template <int NV>
__global__ void __launch_bounds__(256) layernorm_bf16_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                                                                 const float* __restrict__ beta, __nv_bfloat16* __restrict__ y,
                                                                 float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows,
                                                                 int dim, float eps) {
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const __nv_bfloat16* xr = x + static_cast<long long>(row) * dim;
    uint4 v[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = (lane + 32 * i) * 8;
        v[i] = c < dim ? *reinterpret_cast<const uint4*>(xr + c) : make_uint4(0u, 0u, 0u, 0u);
        const uint32_t w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) s += bf16lo(w[k]) + bf16hi(w[k]);
    }
    const float inv_n = 1.0f / static_cast<float>(dim);
    const float mean = warp_sum(s) * inv_n;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = (lane + 32 * i) * 8;
        if (c < dim) {
            const uint32_t w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float a = bf16lo(w[k]) - mean, b = bf16hi(w[k]) - mean;
                ss += a * a + b * b;
            }
        }
    }
    const float rstd = rsqrtf(warp_sum(ss) * inv_n + eps);
    if (lane == 0) {
        mean_out[row] = mean;
        rstd_out[row] = rstd;
    }
    __nv_bfloat16* yr = y + static_cast<long long>(row) * dim;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = (lane + 32 * i) * 8;
        if (c < dim) {
            const float4 g0 = *reinterpret_cast<const float4*>(gamma + c), g1 = *reinterpret_cast<const float4*>(gamma + c + 4);
            const float4 b0 = *reinterpret_cast<const float4*>(beta + c), b1 = *reinterpret_cast<const float4*>(beta + c + 4);
            const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
            const uint32_t w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
            uint32_t o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k)
                o[k] = pack_bf16x2((bf16lo(w[k]) - mean) * rstd * g[2 * k] + b[2 * k], (bf16hi(w[k]) - mean) * rstd * g[2 * k + 1] + b[2 * k + 1]);
            *reinterpret_cast<uint4*>(yr + c) = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
}

// Backward: dx = bf16(float(dres) + float(bf16(LN'(dy)))) -- eager's cast back to the bf16 input, then the bf16 addition of
// the residual branch's gradient (dres == nullptr: no addition).  Warps stride over rows; each warp keeps running dgamma /
// dbeta sums of its rows in its own shared-memory rows (lane-private columns: no synchronisation, and no accumulator
// registers), which the block reduces in warp order into part[blockIdx][0:dim] / [dim:2 dim].  A fixed grid and fixed
// summation orders make the result deterministic.
template <int NV>
__global__ void __launch_bounds__(256) layernorm_bf16_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                                                 const float* __restrict__ gamma, const float* __restrict__ mean_in,
                                                                 const float* __restrict__ rstd_in, const __nv_bfloat16* __restrict__ dres,
                                                                 __nv_bfloat16* __restrict__ dx, float* __restrict__ part, int rows, int dim) {
    extern __shared__ float sred[];  // [8 warps][2][dim]
    const int wib = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int warps_per_block = blockDim.x >> 5;
    float* sg = sred + wib * 2 * dim;
    float* sb = sg + dim;
    for (int c = lane * 4; c < dim; c += 128) {
        *reinterpret_cast<float4*>(sg + c) = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(sb + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncwarp();
    const float fn = static_cast<float>(dim);
    for (int row = blockIdx.x * warps_per_block + wib; row < rows; row += gridDim.x * warps_per_block) {
        const long long off = static_cast<long long>(row) * dim;
        uint4 xv[NV], dv[NV], rv[NV];
#pragma unroll
        for (int i = 0; i < NV; ++i) {  // every load of the row in flight before any is used
            const int c = (lane + 32 * i) * 8;
            if (c < dim) {
                xv[i] = *reinterpret_cast<const uint4*>(x + off + c);
                dv[i] = *reinterpret_cast<const uint4*>(dy + off + c);
                rv[i] = dres != nullptr ? *reinterpret_cast<const uint4*>(dres + off + c) : make_uint4(0u, 0u, 0u, 0u);
            }
        }
        const float mean = mean_in[row];
        const float rstd = rstd_in[row];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int c = (lane + 32 * i) * 8;
            if (c < dim) {
                const uint32_t xw[4] = {xv[i].x, xv[i].y, xv[i].z, xv[i].w};
                const uint32_t dw[4] = {dv[i].x, dv[i].y, dv[i].z, dv[i].w};
                float4 ag[2], ab[2];
                ag[0] = *reinterpret_cast<float4*>(sg + c); ag[1] = *reinterpret_cast<float4*>(sg + c + 4);
                ab[0] = *reinterpret_cast<float4*>(sb + c); ab[1] = *reinterpret_cast<float4*>(sb + c + 4);
                float* pg = reinterpret_cast<float*>(ag);
                float* pb = reinterpret_cast<float*>(ab);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const uint32_t xk = xw[k >> 1], dk = dw[k >> 1];
                    const float xh = ((k & 1) ? bf16hi(xk) : bf16lo(xk)) - mean;
                    const float d = (k & 1) ? bf16hi(dk) : bf16lo(dk);
                    const float xn = xh * rstd;
                    const float gd = d * gamma[c + k];
                    s1 += gd;
                    s2 += gd * xn;
                    pg[k] += d * xn;
                    pb[k] += d;
                }
                *reinterpret_cast<float4*>(sg + c) = ag[0]; *reinterpret_cast<float4*>(sg + c + 4) = ag[1];
                *reinterpret_cast<float4*>(sb + c) = ab[0]; *reinterpret_cast<float4*>(sb + c + 4) = ab[1];
            }
        }
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        const float term = rstd / fn;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int c = (lane + 32 * i) * 8;
            if (c < dim) {
                const uint32_t xw[4] = {xv[i].x, xv[i].y, xv[i].z, xv[i].w};
                const uint32_t dw[4] = {dv[i].x, dv[i].y, dv[i].z, dv[i].w};
                const uint32_t rw[4] = {rv[i].x, rv[i].y, rv[i].z, rv[i].w};
                float o[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const uint32_t xk = xw[k >> 1], dk = dw[k >> 1], rk = rw[k >> 1];
                    const float xn = (((k & 1) ? bf16hi(xk) : bf16lo(xk)) - mean) * rstd;
                    const float d = (k & 1) ? bf16hi(dk) : bf16lo(dk);
                    const float g = bf16_round((fn * (d * gamma[c + k]) - s1 - xn * s2) * term);  // bf16(LN'(dy))
                    o[k] = dres != nullptr ? g + ((k & 1) ? bf16hi(rk) : bf16lo(rk)) : g;
                }
                *reinterpret_cast<uint4*>(dx + off + c) =
                    make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
            }
        }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < dim; c += blockDim.x) {
        float a = 0.f, b = 0.f;
        for (int w = 0; w < warps_per_block; ++w) {
            a += sred[(w * 2 + 0) * dim + c];
            b += sred[(w * 2 + 1) * dim + c];
        }
        part[static_cast<long long>(blockIdx.x) * 2 * dim + c] = a;
        part[static_cast<long long>(blockIdx.x) * 2 * dim + dim + c] = b;
    }
}

// ------------------------------------------------------------------------------------------------
// column sums of a bf16 matrix: grid (col chunks of 256, row slices); block (32, 8)
// ------------------------------------------------------------------------------------------------
// one block's share: part_row[c] = sum of x[r][c] over rows [r_begin, r_end), for the 256 columns of blockIdx.x
__device__ __forceinline__ void colsum_slice(const __nv_bfloat16* __restrict__ x, long long ld, int r_begin, int r_end, int cols,
                                             float* __restrict__ part_row) {
    __shared__ float sm[8][256 + 8];
    const int c0 = blockIdx.x * 256 + threadIdx.x * 8;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (c0 < cols) {
        int r = r_begin + threadIdx.y;
        for (; r + 24 < r_end; r += 32) {  // 4 independent loads in flight per thread
            uint4 t[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) t[k] = *reinterpret_cast<const uint4*>(x + static_cast<long long>(r + 8 * k) * ld + c0);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                acc[0] += bf16lo(t[k].x); acc[1] += bf16hi(t[k].x); acc[2] += bf16lo(t[k].y); acc[3] += bf16hi(t[k].y);
                acc[4] += bf16lo(t[k].z); acc[5] += bf16hi(t[k].z); acc[6] += bf16lo(t[k].w); acc[7] += bf16hi(t[k].w);
            }
        }
        for (; r < r_end; r += 8) {
            const uint4 t = *reinterpret_cast<const uint4*>(x + static_cast<long long>(r) * ld + c0);
            acc[0] += bf16lo(t.x); acc[1] += bf16hi(t.x); acc[2] += bf16lo(t.y); acc[3] += bf16hi(t.y);
            acc[4] += bf16lo(t.z); acc[5] += bf16hi(t.z); acc[6] += bf16lo(t.w); acc[7] += bf16hi(t.w);
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) sm[threadIdx.y][threadIdx.x * 8 + k] = acc[k];
    __syncthreads();
    const int t = threadIdx.y * 32 + threadIdx.x;  // 0..255 -> one column each
    const int c = blockIdx.x * 256 + t;
    if (c < cols) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += sm[w][t];
        part_row[c] = s;
    }
}

__global__ void __launch_bounds__(256) colsum_bf16_kernel(const __nv_bfloat16* __restrict__ x, long long ld, int rows,
                                                          int cols, float* __restrict__ part) {
    const int nslices = gridDim.y;
    const int r_begin = static_cast<int>((static_cast<long long>(rows) * blockIdx.y) / nslices);
    const int r_end = static_cast<int>((static_cast<long long>(rows) * (blockIdx.y + 1)) / nslices);
    colsum_slice(x, ld, r_begin, r_end, cols, part + static_cast<long long>(blockIdx.y) * cols);
}

// per-image column sums: grid (column chunks of 256, slices per image, images); x dense [B, hw, cols]; the partial row of
// (image b, slice s) is b * gridDim.y + s
__global__ void __launch_bounds__(256) colsum_per_image_kernel(const __nv_bfloat16* __restrict__ x, int hw, int cols,
                                                               float* __restrict__ part) {
    const int nslices = gridDim.y;
    const int r_begin = static_cast<int>((static_cast<long long>(hw) * blockIdx.y) / nslices);
    const int r_end = static_cast<int>((static_cast<long long>(hw) * (blockIdx.y + 1)) / nslices);
    colsum_slice(x + static_cast<long long>(blockIdx.z) * hw * cols, cols, r_begin, r_end, cols,
                 part + (static_cast<long long>(blockIdx.z) * nslices + blockIdx.y) * cols);
}

// per_image[b][c] = bf16(sum_s part[b][s][c]); total[c] = bf16_round(sum_b of those unrounded sums), all in a fixed order
__global__ void __launch_bounds__(256) colsum_per_image_finish_kernel(const float* __restrict__ part, int B, int nslices, int cols,
                                                                      __nv_bfloat16* __restrict__ per_image, float* __restrict__ total) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    float tot = 0.f;
    for (int b = 0; b < B; ++b) {
        float s = 0.f;
        for (int j = 0; j < nslices; ++j) s += part[(static_cast<long long>(b) * nslices + j) * cols + c];
        per_image[static_cast<long long>(b) * cols + c] = __float2bfloat16_rn(s);
        tot += s;
    }
    total[c] = bf16_round(tot);
}

// out[c] (+)= sum_p part[p * part_ld + c]: block = 32 columns x 8 part lanes (a loop over up to 592 parts serially per
// thread made this reduction latency-bound at ~100 calls per step)
__global__ void __launch_bounds__(256) colsum_finish_kernel(const float* __restrict__ part, long long part_ld, int nparts,
                                                            int cols, float* __restrict__ out, int round_bf16,
                                                            int accumulate) {
    __shared__ float sm[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    float s = 0.f;
    if (c < cols)
        for (int p = threadIdx.y; p < nparts; p += 8) s += part[static_cast<long long>(p) * part_ld + c];
    sm[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && c < cols) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += sm[w][threadIdx.x];
        if (round_bf16) t = bf16_round(t);
        out[c] = accumulate ? out[c] + t : t;
    }
}

// two destinations in one launch: columns [0, cols0) -> out0, [cols0, cols0 + cols1) -> out1 (own rounding flag each)
__global__ void __launch_bounds__(256) colsum_finish2_kernel(const float* __restrict__ part, long long part_ld, int nparts,
                                                             int cols0, float* __restrict__ out0, int round0, int cols1,
                                                             float* __restrict__ out1, int round1, int accumulate) {
    __shared__ float sm[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int cols = cols0 + cols1;
    float s = 0.f;
    if (c < cols)
        for (int p = threadIdx.y; p < nparts; p += 8) s += part[static_cast<long long>(p) * part_ld + c];
    sm[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && c < cols) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += sm[w][threadIdx.x];
        float* o = c < cols0 ? out0 + c : out1 + (c - cols0);
        if (c < cols0 ? round0 : round1) t = bf16_round(t);
        *o = accumulate ? *o + t : t;
    }
}

__global__ void splitk_reduce_kernel(const float* __restrict__ partial, int splits, long long n4,
                                     float* __restrict__ out, int round_bf16, int accumulate) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    float4 s = reinterpret_cast<const float4*>(partial)[i];
    for (int k = 1; k < splits; ++k) {
        const float4 t = reinterpret_cast<const float4*>(partial)[static_cast<long long>(k) * n4 + i];
        s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
    }
    if (round_bf16) { s.x = bf16_round(s.x); s.y = bf16_round(s.y); s.z = bf16_round(s.z); s.w = bf16_round(s.w); }
    if (accumulate) {
        const float4 o = reinterpret_cast<const float4*>(out)[i];
        s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
    }
    reinterpret_cast<float4*>(out)[i] = s;
}

// ------------------------------------------------------------------------------------------------
// patch-embed glue
// ------------------------------------------------------------------------------------------------
// thread = (b, c, y, x16): 16 consecutive pixels of one image row -> 16 consecutive k of one patch row
__global__ void patch_im2col_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ cols, int B, int C,
                                    int img, int P) {
    const int segs = img / 16;
    const long long total = static_cast<long long>(B) * C * img * segs;
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int x16 = static_cast<int>(i % segs);
    long long r = i / segs;
    const int y = static_cast<int>(r % img);
    r /= img;
    const int c = static_cast<int>(r % C);
    const int b = static_cast<int>(r / C);
    const float4* src = reinterpret_cast<const float4*>(x + ((static_cast<long long>(b) * C + c) * img + y) * img + x16 * 16);
    const float4 a0 = src[0], a1 = src[1], a2 = src[2], a3 = src[3];
    const int side = img / P;
    const int py = y / P, ky = y % P;
    const int px = (x16 * 16) / P, kx0 = (x16 * 16) % P;
    const long long row = (static_cast<long long>(b) * side + py) * side + px;
    __nv_bfloat16* dst = cols + row * (static_cast<long long>(C) * P * P) + (static_cast<long long>(c) * P + ky) * P + kx0;
    uint4 o0, o1;
    o0.x = pack_bf16x2(a0.x, a0.y); o0.y = pack_bf16x2(a0.z, a0.w); o0.z = pack_bf16x2(a1.x, a1.y); o0.w = pack_bf16x2(a1.z, a1.w);
    o1.x = pack_bf16x2(a2.x, a2.y); o1.y = pack_bf16x2(a2.z, a2.w); o1.z = pack_bf16x2(a3.x, a3.y); o1.w = pack_bf16x2(a3.z, a3.w);
    reinterpret_cast<uint4*>(dst)[0] = o0;
    reinterpret_cast<uint4*>(dst)[1] = o1;
}

// The same gather straight from the RAW batch: uint8 [B, S, S, C] (HWC, what the reference's loader holds before its runtime
// blocks) -> normalise -> bf16 im2col matrix.  Replaces, per step, the numpy passes static_normalize (x.astype(float64) /
// division, cflearn/data/blocks/cv/normalize.py:11-24), imagenet / affine normalisation ((x - mean) / std in float64,
// :27-67), hwc_to_chw (hwc_to_chw.py:9-15), the float32 tensor conversion + host->device copy of TensorBatcher
// (cflearn/data/utils.py:255-283) and autocast's bf16 cast of the conv input: the GPU receives 1 byte per value instead
// of 4, and the 154 MB fp32 image tensor is never materialised.  Arithmetic follows the reference's rounding chain:
// float64 -> float32 -> bf16.  thread = (b, y, x16): 16 consecutive pixels (16 * C bytes) -> 16 k of one patch row per channel.
struct NormParams {
    double division;
    double mean[4];
    double stdv[4];
};
template <int C>
__global__ void patch_im2col_u8_kernel(const uint8_t* __restrict__ x, __nv_bfloat16* __restrict__ cols, int B, int img, int P,
                                       const NormParams np_) {
    const int segs = img / 16;
    const long long total = static_cast<long long>(B) * img * segs;
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int x16 = static_cast<int>(i % segs);
    const long long r = i / segs;
    const int y = static_cast<int>(r % img);
    const int b = static_cast<int>(r / img);
    const uint4* src = reinterpret_cast<const uint4*>(x + ((static_cast<long long>(b) * img + y) * img + x16 * 16) * C);
    uint32_t w[4 * C];
#pragma unroll
    for (int k = 0; k < C; ++k) {
        const uint4 t = __ldg(src + k);
        w[4 * k + 0] = t.x; w[4 * k + 1] = t.y; w[4 * k + 2] = t.z; w[4 * k + 3] = t.w;
    }
    const int side = img / P;
    const int py = y / P, ky = y % P;
    const int px = (x16 * 16) / P, kx0 = (x16 * 16) % P;
    const long long row = (static_cast<long long>(b) * side + py) * side + px;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        float v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const int byte = k * C + c;  // pixel k, channel c inside the 16 * C bytes
            const double raw = static_cast<double>((w[byte >> 2] >> ((byte & 3) * 8)) & 0xffu);
            v[k] = static_cast<float>((raw / np_.division - np_.mean[c]) / np_.stdv[c]);
        }
        __nv_bfloat16* dst = cols + row * (static_cast<long long>(C) * P * P) + (static_cast<long long>(c) * P + ky) * P + kx0;
        uint4 o0, o1;
        o0.x = pack_bf16x2(v[0], v[1]); o0.y = pack_bf16x2(v[2], v[3]); o0.z = pack_bf16x2(v[4], v[5]); o0.w = pack_bf16x2(v[6], v[7]);
        o1.x = pack_bf16x2(v[8], v[9]); o1.y = pack_bf16x2(v[10], v[11]); o1.z = pack_bf16x2(v[12], v[13]); o1.w = pack_bf16x2(v[14], v[15]);
        reinterpret_cast<uint4*>(dst)[0] = o0;
        reinterpret_cast<uint4*>(dst)[1] = o1;
    }
}

// net[b, t, d..d+7] = (t == 0 ? cls : float(patch[b*np + t-1])) + pos[t]
// conv_bias != nullptr: the patch rows first take eager's separate bias add, bf16(patch + bias), i.e. the SECOND rounding of
// `F.conv2d(x, w, bias)` on CUDA (the convolution output is rounded to bf16, then `output.add_(bias)` rounds again)
__global__ void assemble_tokens_kernel(const __nv_bfloat16* __restrict__ patch, const float* __restrict__ cls,
                                       const float* __restrict__ pos, float* __restrict__ net, int B, int np, int D,
                                       const __nv_bfloat16* __restrict__ conv_bias) {
    const int d8 = D / 8;
    const long long total = static_cast<long long>(B) * (np + 1) * d8;
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int dc = static_cast<int>(i % d8) * 8;
    const long long bt = i / d8;
    const int t = static_cast<int>(bt % (np + 1));
    const int b = static_cast<int>(bt / (np + 1));
    float v[8];
    if (t == 0) {
        const float4 a = *reinterpret_cast<const float4*>(cls + dc);
        const float4 c = *reinterpret_cast<const float4*>(cls + dc + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
    } else {
        const uint4 p = *reinterpret_cast<const uint4*>(patch + (static_cast<long long>(b) * np + (t - 1)) * D + dc);
        v[0] = bf16lo(p.x); v[1] = bf16hi(p.x); v[2] = bf16lo(p.y); v[3] = bf16hi(p.y);
        v[4] = bf16lo(p.z); v[5] = bf16hi(p.z); v[6] = bf16lo(p.w); v[7] = bf16hi(p.w);
        if (conv_bias != nullptr) {
            const uint4 cb = *reinterpret_cast<const uint4*>(conv_bias + dc);
            v[0] = bf16_round(v[0] + bf16lo(cb.x)); v[1] = bf16_round(v[1] + bf16hi(cb.x));
            v[2] = bf16_round(v[2] + bf16lo(cb.y)); v[3] = bf16_round(v[3] + bf16hi(cb.y));
            v[4] = bf16_round(v[4] + bf16lo(cb.z)); v[5] = bf16_round(v[5] + bf16hi(cb.z));
            v[6] = bf16_round(v[6] + bf16lo(cb.w)); v[7] = bf16_round(v[7] + bf16hi(cb.w));
        }
    }
    const float4 p0 = *reinterpret_cast<const float4*>(pos + static_cast<long long>(t) * D + dc);
    const float4 p1 = *reinterpret_cast<const float4*>(pos + static_cast<long long>(t) * D + dc + 4);
    float* o = net + bt * D + dc;
    *reinterpret_cast<float4*>(o) = make_float4(v[0] + p0.x, v[1] + p0.y, v[2] + p0.z, v[3] + p0.w);
    *reinterpret_cast<float4*>(o + 4) = make_float4(v[4] + p1.x, v[5] + p1.y, v[6] + p1.z, v[7] + p1.w);
}

// text tower input stage (TeTEncoder: no head token): net[b, t, :] = x[b, t, :] + pos[t, :], fp32
__global__ void add_pos_kernel(const float* __restrict__ x, const float* __restrict__ pos, float* __restrict__ net, long long n4,
                               int td4) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 a = reinterpret_cast<const float4*>(x)[i];
    const float4 p = reinterpret_cast<const float4*>(pos)[i % td4];
    reinterpret_cast<float4*>(net)[i] = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
}
// dpos[t, :] = sum_b dnet[b, t, :] (thread = 4 columns of (t, d), loops over the batch in a fixed order)
__global__ void add_pos_bwd_kernel(const float* __restrict__ dnet, float* __restrict__ dpos, int B, int td4, int accumulate) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= td4) return;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int b = 0; b < B; ++b) {
        const float4 v = reinterpret_cast<const float4*>(dnet)[static_cast<long long>(b) * td4 + i];
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    float4* o = reinterpret_cast<float4*>(dpos) + i;
    if (accumulate) { const float4 old = *o; s.x += old.x; s.y += old.y; s.z += old.z; s.w += old.w; }
    *o = s;
}

// ---- CLIP text glue: integer-indexed row moves (bit-exact copies) ------------------------------------------------------
// out[n, :] = W[ids[n], :]   (nn.Embedding forward, clip.py:235); ids outside [0, V) raise the flag and read row 0
__global__ void embedding_fwd_kernel(const long long* __restrict__ ids, const float* __restrict__ W, float* __restrict__ out,
                                     long long n4_total, int d4, int V, int* __restrict__ bad) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n4_total) return;
    const long long n = i / d4;
    const int c = static_cast<int>(i % d4);
    long long id = ids[n];
    if (id < 0 || id >= V) { if (c == 0) atomicExch(bad, 1); id = 0; }
    reinterpret_cast<float4*>(out)[i] = reinterpret_cast<const float4*>(W)[id * d4 + c];
}
// dW[ids[n], :] += dnet[n, :] for ids[n] != padding_idx (embedding_dense_backward; fp32 atomics: the summation order over
// repeated tokens is not fixed, the set of rows touched is exact)
__global__ void embedding_bwd_kernel(const long long* __restrict__ ids, const float* __restrict__ dnet, float* __restrict__ dW,
                                     long long n_total, int D, int V, int padding_idx) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n_total) return;
    const long long n = i / D;
    const int c = static_cast<int>(i % D);
    const long long id = ids[n];
    if (id < 0 || id >= V || id == padding_idx) return;
    const float v = dnet[i];
    if (v != 0.f) atomicAdd(dW + id * D + c, v);
}
// pos[b] = first arg-max of ids[b, :] (clip.py:250); out[b, :] = x[b, pos[b], :].  One block per sample.
__global__ void argmax_gather_kernel(const long long* __restrict__ ids, const float* __restrict__ x, float* __restrict__ out,
                                     int* __restrict__ pos_out, int T, int D) {
    __shared__ int spos;
    const int b = blockIdx.x;
    if (threadIdx.x == 0) {
        long long best = ids[static_cast<long long>(b) * T];
        int bp = 0;
        for (int t = 1; t < T; ++t) {
            const long long v = ids[static_cast<long long>(b) * T + t];
            if (v > best) { best = v; bp = t; }
        }
        spos = bp;
        pos_out[b] = bp;
    }
    __syncthreads();
    const float* src = x + (static_cast<long long>(b) * T + spos) * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) out[static_cast<long long>(b) * D + c] = src[c];
}
// dx[b, pos[b], :] = dout[b, :] (dx zero-filled by the caller)
__global__ void scatter_rows_kernel(const float* __restrict__ dout, const int* __restrict__ pos, float* __restrict__ dx, int T, int D) {
    const int b = blockIdx.x;
    float* dst = dx + (static_cast<long long>(b) * T + pos[b]) * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) dst[c] = dout[static_cast<long long>(b) * D + c];
}

// thread = (t, d4): loops over the batch; dpos[t] = sum_b dnet[b,t]; dpatch = bf16(dnet[:,1:]); dcls = dpos[0]
__global__ void assemble_tokens_bwd_kernel(const float* __restrict__ dnet, __nv_bfloat16* __restrict__ dpatch,
                                           float* __restrict__ dpos, float* __restrict__ dcls, int B, int np, int D,
                                           int accumulate) {
    const int d4 = D / 4;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (np + 1) * d4) return;
    const int dc = (i % d4) * 4;
    const int t = i / d4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    const long long bstride = static_cast<long long>(np + 1) * D;
    const float* src = dnet + static_cast<long long>(t) * D + dc;
#pragma unroll 4
    for (int b = 0; b < B; ++b) {
        const float4 v = *reinterpret_cast<const float4*>(src + b * bstride);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        if (t > 0) {
            uint2 p;
            p.x = pack_bf16x2(v.x, v.y);
            p.y = pack_bf16x2(v.z, v.w);
            *reinterpret_cast<uint2*>(dpatch + (static_cast<long long>(b) * np + (t - 1)) * D + dc) = p;
        }
    }
    float* pp = dpos + static_cast<long long>(t) * D + dc;
    if (accumulate) { const float4 o = *reinterpret_cast<const float4*>(pp); *reinterpret_cast<float4*>(pp) = make_float4(o.x + s.x, o.y + s.y, o.z + s.z, o.w + s.w); }
    else *reinterpret_cast<float4*>(pp) = s;
    if (t == 0) {
        float* pc = dcls + dc;
        if (accumulate) { const float4 o = *reinterpret_cast<const float4*>(pc); *reinterpret_cast<float4*>(pc) = make_float4(o.x + s.x, o.y + s.y, o.z + s.z, o.w + s.w); }
        else *reinterpret_cast<float4*>(pc) = s;
    }
}

// ------------------------------------------------------------------------------------------------
// softmax cross entropy: one block per row
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) softmax_xent_kernel(const __nv_bfloat16* __restrict__ logits, long long ldl,
                                                           const long long* __restrict__ labels,
                                                           float* __restrict__ loss_rows,
                                                           __nv_bfloat16* __restrict__ dlogits, int* bad_flag, int B,
                                                           int C, float gscale, const float* __restrict__ gscale_dev) {
    __shared__ float sred[8];
    __shared__ float sbc;
    const int row = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const __nv_bfloat16* lr = logits + static_cast<long long>(row) * ldl;
    float m = -INFINITY;
    for (int c = tid; c < C; c += 256) m = fmaxf(m, __bfloat162float(lr[c]));
    m = warp_max(m);
    if (lane == 0) sred[wid] = m;
    __syncthreads();
    if (tid == 0) { float t = sred[0]; for (int w = 1; w < 8; ++w) t = fmaxf(t, sred[w]); sbc = t; }
    __syncthreads();
    m = sbc;
    float s = 0.f;
    for (int c = tid; c < C; c += 256) s += expf(__bfloat162float(lr[c]) - m);
    s = warp_sum(s);
    __syncthreads();
    if (lane == 0) sred[wid] = s;
    __syncthreads();
    if (tid == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += sred[w]; sbc = t; }
    __syncthreads();
    const float lse = m + logf(sbc);
    long long lab = labels[row];
    if (lab < 0 || lab >= C) {  // torch's gather would raise; flag it and clamp so we stay in bounds
        if (tid == 0) atomicExch(bad_flag, 1);
        lab = lab < 0 ? 0 : C - 1;
    }
    if (tid == 0) loss_rows[row] = lse - __bfloat162float(lr[lab]);
    if (dlogits != nullptr) {
        __nv_bfloat16* dr = dlogits + static_cast<long long>(row) * ldl;  // same row stride as the logits
        const float sc = gscale * (gscale_dev != nullptr ? gscale_dev[0] : 1.0f) / static_cast<float>(B);
        for (int c = tid; c < C; c += 256) {
            float p = expf(__bfloat162float(lr[c]) - lse);
            if (c == lab) p -= 1.0f;
            dr[c] = __float2bfloat16_rn(p * sc);
        }
    }
}
// ------------------------------------------------------------------------------------------------
// symmetric (contrastive) cross entropy over a square bf16 logits matrix L [B, B] with targets arange(B):
//   loss = (CE(L, arange) + CE(L^T, arange)) / 2        -- the usual CLIP objective.  The reference defines none
//   (SURVEY.md 8d); the product-side definition follows oracle/clip_oracle.py::symmetric_cross_entropy: fp32 maths on the
//   bf16 logits (autocast runs cross_entropy in fp32), and ONE rounding of the summed gradient to bf16.
// stats kernel: warp w < B -> log-sum-exp of row w; warp w >= B -> of column w - B.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sym_xent_stats_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int B,
                                                             float* __restrict__ lse /* [2B] */) {
    const int w = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (w >= 2 * B) return;
    const bool col = w >= B;
    const int k = col ? w - B : w;
    const long long base = col ? k : static_cast<long long>(k) * ld;
    const long long stride = col ? ld : 1;
    float m = -INFINITY;
    for (int j = lane; j < B; j += 32) m = fmaxf(m, __bfloat162float(logits[base + j * stride]));
    m = warp_max(m);
    float sacc = 0.f;
    for (int j = lane; j < B; j += 32) sacc += expf(__bfloat162float(logits[base + j * stride]) - m);
    sacc = warp_sum(sacc);
    if (lane == 0) lse[w] = m + logf(sacc);
}
// loss (deterministic single-block sum) = mean_i( (lse_row[i] - L_ii) + (lse_col[i] - L_ii) ) / 2
__global__ void sym_xent_loss_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int B, const float* __restrict__ lse,
                                     float* __restrict__ loss) {
    __shared__ float sred[8];
    float sacc = 0.f;
    for (int i = threadIdx.x; i < B; i += 256) sacc += lse[i] + lse[B + i] - 2.0f * __bfloat162float(logits[static_cast<long long>(i) * ld + i]);
    sacc = warp_sum(sacc);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = sacc;
    __syncthreads();
    if (threadIdx.x == 0) { float t = 0.f; for (int k = 0; k < 8; ++k) t += sred[k]; loss[0] = 0.5f * t / static_cast<float>(B); }
}
// dL_ij = bf16( sc / (2B) * ( softmax_row(i)_j + softmax_col(j)_i - 2 [i == j] ) )
__global__ void sym_xent_grad_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int B, const float* __restrict__ lse,
                                     __nv_bfloat16* __restrict__ dlogits, float gscale, const float* __restrict__ gscale_dev) {
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= static_cast<long long>(B) * B) return;
    const int i = static_cast<int>(idx / B), j = static_cast<int>(idx % B);
    const float l = __bfloat162float(logits[static_cast<long long>(i) * ld + j]);
    const float sc = gscale * (gscale_dev != nullptr ? gscale_dev[0] : 1.0f) * 0.5f / static_cast<float>(B);
    float g = expf(l - lse[i]) + expf(l - lse[B + j]);
    if (i == j) g -= 2.0f;
    dlogits[static_cast<long long>(i) * ld + j] = __float2bfloat16_rn(g * sc);
}

__global__ void mean_kernel(const float* __restrict__ v, int n, float* __restrict__ out) {
    __shared__ float sred[8];
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += 256) s += v[i];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += sred[w]; out[0] = t / static_cast<float>(n); }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
    const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
    if (i + 8 <= n) {
        const float4 a = *reinterpret_cast<const float4*>(src + i);
        const float4 b = *reinterpret_cast<const float4*>(src + i + 4);
        uint4 o;
        o.x = pack_bf16x2(a.x, a.y); o.y = pack_bf16x2(a.z, a.w); o.z = pack_bf16x2(b.x, b.y); o.w = pack_bf16x2(b.z, b.w);
        *reinterpret_cast<uint4*>(dst + i) = o;
    } else {
        for (long long k = i; k < n; ++k) dst[k] = __float2bfloat16_rn(src[k]);
    }
}
__global__ void fill_f32_kernel(float* __restrict__ dst, float v, long long n) {
    const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
    if (i + 4 <= n) *reinterpret_cast<float4*>(dst + i) = make_float4(v, v, v, v);
    else for (long long k = i; k < n; ++k) dst[k] = v;
}

// Adam over the flat parameter arena (torch.optim.Adam semantics, no amsgrad; L2 weight decay added to the grad).
// kDecoupled: AdamW (torch.optim.AdamW's order): p <- p (1 - lr wd) first, then the Adam update with no L2 term.
template <bool kDecoupled>
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, long long n4, float lr, float b1, float b2, float eps, float wd,
                            float bc1, float bc2_sqrt, const int* __restrict__ step_dev) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    if (step_dev != nullptr) {  // step counter lives on the device (CUDA-graph replay): derive the bias corrections here
        const float t = static_cast<float>(step_dev[0]);
        bc1 = 1.0f - powf(b1, t);
        bc2_sqrt = sqrtf(1.0f - powf(b2, t));
    }
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    float4 mm = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    const float step = lr / bc1;
    const float keep = 1.0f - lr * wd;
    auto upd = [&](float& pw, float gw, float& mw, float& vw) {
        if (kDecoupled) pw *= keep;
        else gw += wd * pw;
        mw += (gw - mw) * (1.0f - b1);
        vw = vw * b2 + (1.0f - b2) * gw * gw;
        const float denom = sqrtf(vw) / bc2_sqrt + eps;
        pw -= step * (mw / denom);
    };
    upd(pp.x, gg.x, mm.x, vv.x);
    upd(pp.y, gg.y, mm.y, vv.y);
    upd(pp.z, gg.z, mm.z, vv.z);
    upd(pp.w, gg.w, mm.w, vv.w);
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
}

__global__ void increment_kernel(int* counter) { counter[0] += 1; }

// Same update with EVERY hyper-parameter read from device memory (hyper = {lr, beta1, beta2, eps, weight_decay, grad_scale}):
// a captured CUDA graph then follows a learning-rate schedule (the reference's default scheduler is "warmup",
// cflearn/pipeline/blocks/basic.py:334-352) by rewriting 24 bytes between replays.  grad_scale multiplies the gradient
// first (1 / world_size after a SUM all-reduce, or a clip coefficient, cflearn/schema.py:981-982).  kDecoupled as adam_kernel.
template <bool kDecoupled>
__global__ void adam_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                float* __restrict__ v, long long n4, const float* __restrict__ hyper,
                                const int* __restrict__ step_dev) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float lr = hyper[0], b1 = hyper[1], b2 = hyper[2], eps = hyper[3], wd = hyper[4], gs = hyper[5];
    const float t = static_cast<float>(step_dev[0]);
    const float bc1 = 1.0f - powf(b1, t);
    const float bc2_sqrt = sqrtf(1.0f - powf(b2, t));
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    float4 mm = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    const float step = lr / bc1;
    const float keep = 1.0f - lr * wd;
    auto upd = [&](float& pw, float gw, float& mw, float& vw) {
        if (kDecoupled) {
            pw *= keep;
            gw *= gs;
        } else {
            gw = gw * gs + wd * pw;
        }
        mw += (gw - mw) * (1.0f - b1);
        vw = vw * b2 + (1.0f - b2) * gw * gw;
        const float denom = sqrtf(vw) / bc2_sqrt + eps;
        pw -= step * (mw / denom);
    };
    upd(pp.x, gg.x, mm.x, vv.x);
    upd(pp.y, gg.y, mm.y, vv.y);
    upd(pp.z, gg.z, mm.z, vv.z);
    upd(pp.w, gg.w, mm.w, vv.w);
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
}

// The row-width ladders of the two LayerNorm families: launch(std::integral_constant<int, NV>) with the fewest 16-byte chunks per
// lane that hold a row (fp32 rows: dim <= 128 * NV; bf16 rows: dim <= 256 * NV)
template <typename Launch>
static int ln_dispatch(int dim, Launch launch) {
    const int nv = (dim + 127) / 128;
    if (nv <= 4) return launch(std::integral_constant<int, 4>());
    if (nv <= 6) return launch(std::integral_constant<int, 6>());
    return launch(std::integral_constant<int, 8>());
}
template <typename Launch>
static int lnb_dispatch(int dim, Launch launch) {
    const int nv = (dim + 255) / 256;
    if (nv <= 2) return launch(std::integral_constant<int, 2>());
    if (nv <= 4) return launch(std::integral_constant<int, 4>());
    if (nv <= 5) return launch(std::integral_constant<int, 5>());
    return launch(std::integral_constant<int, 8>());
}

// grid of the LayerNorm backwards (= partial rows written): two resident 256-thread blocks per SM (one wave), at most one block per
// 8 rows and at most max_parts
static int ln_bwd_parts(int rows, int max_parts) {
    int nparts = num_sms() * 2;
    if (nparts > (rows + 7) / 8) nparts = (rows + 7) / 8;
    return nparts < max_parts ? nparts : max_parts;
}

template <int NV, bool DXSUM, bool DYF32>
static int ln_bwd_launch(const void* dy, const float* x, long long ld_x, const float* gamma, const float* mean, const float* rstd,
                         const float* dres, float* dx_out, long long ld_dx, void* dx_bf16, float* part, int nparts, int rows, int dim,
                         cudaStream_t st) {
    constexpr int NP = DXSUM ? 3 : 2;
    static bool configured[64] = {};
    if (const int rc = configure_smem(layernorm_bwd_kernel<NV, DXSUM, DYF32>, 8 * NP * 128 * NV * 4, configured)) return rc;
    layernorm_bwd_kernel<NV, DXSUM, DYF32><<<nparts, 256, static_cast<size_t>(8) * NP * dim * sizeof(float), st>>>(
        dy, x, ld_x, gamma, mean, rstd, dres, dx_out, ld_dx, reinterpret_cast<__nv_bfloat16*>(dx_bf16), part, rows, dim);
    return check_launch("layernorm_bwd");
}

// products of sizes that a kernel indexes in 32-bit int
static bool int_overflow(long long a, long long b) { return a * b > 0x7fffffffll; }

}  // namespace b200

using namespace b200;

extern "C" int b200_abi_version(void) { return B200_ABI_VERSION; }
extern "C" const char* b200_last_error(void) { return g_err; }
extern "C" long long b200_launch_count(void) { return g_launches.load(); }

extern "C" int b200_layernorm_bf16_fwd(const void* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd, int rows,
                                       int dim, float eps, cudaStream_t stream) {
    const char* E = "layernorm_bf16_fwd";
    if (rows <= 0 || dim <= 0 || dim % 8 != 0 || dim > 256 * LNB_MAX_V8) return refuse(B200_ERR_ARG, E, "need rows > 0, 0 < dim <= 2048, dim % 8 == 0");
    if (!x || !gamma || !beta || !y || !mean || !rstd) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {x, gamma, beta, y})) return refuse(B200_ERR_ALIGN, E, "x / gamma / beta / y not 16-byte aligned");
    if (!aligned(4, {mean, rstd})) return refuse(B200_ERR_ALIGN, E, "mean / rstd not 4-byte aligned");
    return lnb_dispatch(dim, [&](auto nv) {
        layernorm_bf16_fwd_kernel<decltype(nv)::value><<<(rows + 7) / 8, 256, 0, stream>>>(
            reinterpret_cast<const __nv_bfloat16*>(x), gamma, beta, reinterpret_cast<__nv_bfloat16*>(y), mean, rstd, rows, dim, eps);
        return check_launch("layernorm_bf16_fwd");
    });
}

extern "C" int b200_layernorm_bf16_bwd(const void* dy, const void* x, const float* gamma, const float* mean, const float* rstd,
                                       const void* dres, void* dx, float* dgb_part, int max_parts, int* nparts_out, int rows, int dim,
                                       cudaStream_t stream) {
    const char* E = "layernorm_bf16_bwd";
    if (rows <= 0 || dim <= 0 || dim % 8 != 0 || dim > 256 * LNB_MAX_V8) return refuse(B200_ERR_ARG, E, "need rows > 0, 0 < dim <= 2048, dim % 8 == 0");
    if (max_parts < 1) return refuse(B200_ERR_ARG, E, "max_parts < 1");
    if (!dy || !x || !gamma || !mean || !rstd || !dx || !dgb_part) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {dy, x, gamma, dres, dx})) return refuse(B200_ERR_ALIGN, E, "dy / x / gamma / dres / dx not 16-byte aligned");
    if (!aligned(4, {mean, rstd, dgb_part})) return refuse(B200_ERR_ALIGN, E, "mean / rstd / dgb_part not 4-byte aligned");
    const int nparts = ln_bwd_parts(rows, max_parts);
    if (nparts_out) *nparts_out = nparts;
    return lnb_dispatch(dim, [&](auto nv) {
        constexpr int NV = decltype(nv)::value;
        static bool configured[64] = {};
        if (const int rc = configure_smem(layernorm_bf16_bwd_kernel<NV>, 8 * 2 * 256 * NV * 4, configured)) return rc;
        layernorm_bf16_bwd_kernel<NV><<<nparts, 256, static_cast<size_t>(8) * 2 * dim * sizeof(float), stream>>>(
            reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(x), gamma, mean, rstd,
            reinterpret_cast<const __nv_bfloat16*>(dres), reinterpret_cast<__nv_bfloat16*>(dx), dgb_part, rows, dim);
        return check_launch("layernorm_bf16_bwd");
    });
}

extern "C" int b200_layernorm_fwd(const float* x, long long ld_x, const float* gamma, const float* beta, void* y_bf16,
                                  float* y_f32, float* mean, float* rstd, int rows, int dim, float eps,
                                  cudaStream_t stream) {
    const char* E = "layernorm_fwd";
    if (rows <= 0 || dim <= 0 || dim % 4 != 0 || dim > 128 * LN_MAX_V4) return refuse(B200_ERR_ARG, E, "need rows > 0, 0 < dim <= 1024, dim % 4 == 0");
    if (!x || !gamma || !beta || !y_bf16 || !mean || !rstd) return refuse(B200_ERR_ARG, E, "null pointer");
    if (ld_x < dim) return refuse(B200_ERR_ARG, E, "ld_x < dim");
    if (ld_x % 4 != 0) return refuse(B200_ERR_ALIGN, E, "ld_x % 4 != 0");
    if (!aligned(16, {x, gamma, beta, y_bf16, y_f32})) return refuse(B200_ERR_ALIGN, E, "x / gamma / beta / y_bf16 / y_f32 not 16-byte aligned");
    if (!aligned(4, {mean, rstd})) return refuse(B200_ERR_ALIGN, E, "mean / rstd not 4-byte aligned");
    return ln_dispatch(dim, [&](auto nv) {
        layernorm_fwd_kernel<decltype(nv)::value><<<(rows + 7) / 8, 256, 0, stream>>>(
            x, ld_x, gamma, beta, reinterpret_cast<__nv_bfloat16*>(y_bf16), y_f32, mean, rstd, rows, dim, eps);
        return check_launch("layernorm_fwd");
    });
}

extern "C" int b200_layernorm_bwd(const void* dy, int dy_is_f32, const float* x, long long ld_x, const float* gamma,
                                  const float* mean, const float* rstd, const float* dres, float* dx_out,
                                  long long ld_dx, void* dx_bf16, float* dgb_part, int max_parts, int* nparts_out,
                                  int rows, int dim, int dx_colsum, cudaStream_t stream) {
    const char* E = "layernorm_bwd";
    if (rows <= 0 || dim <= 0 || dim % 4 != 0 || dim > 128 * LN_MAX_V4) return refuse(B200_ERR_ARG, E, "need rows > 0, 0 < dim <= 1024, dim % 4 == 0");
    if (max_parts < 1) return refuse(B200_ERR_ARG, E, "max_parts < 1");
    if (dx_colsum && dy_is_f32) return refuse(B200_ERR_ARG, E, "dx_colsum is not offered with an fp32 dy");
    if (!dy || !x || !gamma || !mean || !rstd || !dx_out || !dgb_part) return refuse(B200_ERR_ARG, E, "null pointer");
    if (dx_colsum && dx_bf16 == nullptr) return refuse(B200_ERR_ARG, E, "dx_colsum needs dx_bf16 (null pointer)");
    if (ld_x < dim || ld_dx < dim) return refuse(B200_ERR_ARG, E, "ld_x / ld_dx < dim");
    if (ld_x % 4 != 0 || ld_dx % 4 != 0) return refuse(B200_ERR_ALIGN, E, "ld % 4 != 0");
    if (!aligned(16, {dy, x, gamma, dres, dx_out, dx_bf16})) return refuse(B200_ERR_ALIGN, E, "dy / x / gamma / dres / dx_out / dx_bf16 not 16-byte aligned");
    if (!aligned(4, {mean, rstd, dgb_part})) return refuse(B200_ERR_ALIGN, E, "mean / rstd / dgb_part not 4-byte aligned");
    const int nparts = ln_bwd_parts(rows, max_parts);
    if (nparts_out) *nparts_out = nparts;
    return ln_dispatch(dim, [&](auto nv) {
        constexpr int NV = decltype(nv)::value;
        if (dy_is_f32) return ln_bwd_launch<NV, false, true>(dy, x, ld_x, gamma, mean, rstd, dres, dx_out, ld_dx, dx_bf16, dgb_part, nparts, rows, dim, stream);
        if (dx_colsum) return ln_bwd_launch<NV, true, false>(dy, x, ld_x, gamma, mean, rstd, dres, dx_out, ld_dx, dx_bf16, dgb_part, nparts, rows, dim, stream);
        return ln_bwd_launch<NV, false, false>(dy, x, ld_x, gamma, mean, rstd, dres, dx_out, ld_dx, dx_bf16, dgb_part, nparts, rows, dim, stream);
    });
}

extern "C" int b200_colsum_bf16(const void* x_bf16, long long ld, int rows, int cols, float* part, int max_parts,
                                int* nparts_out, cudaStream_t stream) {
    const char* E = "colsum";
    if (rows <= 0 || cols <= 0 || max_parts < 1) return refuse(B200_ERR_ARG, E, "need rows, cols > 0 and max_parts >= 1");
    if (!x_bf16 || !part) return refuse(B200_ERR_ARG, E, "null pointer");
    if (ld < (cols + 7) / 8 * 8) return refuse(B200_ERR_ARG, E, "ld must be >= roundup(cols, 8)");
    if (ld % 8 != 0) return refuse(B200_ERR_ALIGN, E, "ld must be a multiple of 8");
    if (!aligned(16, {x_bf16})) return refuse(B200_ERR_ALIGN, E, "x not 16-byte aligned");
    if (!aligned(4, {part})) return refuse(B200_ERR_ALIGN, E, "part not 4-byte aligned");
    const int chunks = (cols + 255) / 256;
    int slices = (num_sms() * 4) / chunks;
    if (slices < 1) slices = 1;
    if (slices > (rows + 7) / 8) slices = (rows + 7) / 8;
    if (slices > max_parts) slices = max_parts;
    if (nparts_out) *nparts_out = slices;
    colsum_bf16_kernel<<<dim3(chunks, slices), dim3(32, 8), 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x_bf16), ld, rows, cols, part);
    return check_launch("colsum_bf16");
}

extern "C" int b200_colsum_finish(const float* part, long long part_ld, int nparts, int cols, float* out, int round_bf16,
                                  int accumulate, cudaStream_t stream) {
    const char* E = "colsum_finish";
    if (nparts <= 0 || cols <= 0) return refuse(B200_ERR_ARG, E, "bad size");
    if (!part || !out) return refuse(B200_ERR_ARG, E, "null pointer");
    if (part_ld < cols) return refuse(B200_ERR_ARG, E, "part_ld < cols");
    if (!aligned(4, {part, out})) return refuse(B200_ERR_ALIGN, E, "part / out not 4-byte aligned");
    colsum_finish_kernel<<<(cols + 31) / 32, dim3(32, 8), 0, stream>>>(part, part_ld, nparts, cols, out, round_bf16, accumulate);
    return check_launch("colsum_finish");
}

extern "C" int b200_colsum_finish2(const float* part, long long part_ld, int nparts, int cols0, float* out0, int round0,
                                   int cols1, float* out1, int round1, int accumulate, cudaStream_t stream) {
    const char* E = "colsum_finish2";
    if (nparts <= 0 || cols0 <= 0 || cols1 <= 0) return refuse(B200_ERR_ARG, E, "bad size");
    if (!part || !out0 || !out1) return refuse(B200_ERR_ARG, E, "null pointer");
    if (part_ld < static_cast<long long>(cols0) + cols1) return refuse(B200_ERR_ARG, E, "part_ld < cols0 + cols1");
    if (!aligned(4, {part, out0, out1})) return refuse(B200_ERR_ALIGN, E, "part / out0 / out1 not 4-byte aligned");
    colsum_finish2_kernel<<<(cols0 + cols1 + 31) / 32, dim3(32, 8), 0, stream>>>(part, part_ld, nparts, cols0, out0, round0, cols1, out1, round1, accumulate);
    return check_launch("colsum_finish2");
}

// slices per image: about four blocks per SM of an H100 SXM over the whole grid, at most 32, at least 8 rows each
static int colsum_per_image_slices(int B, int HW, int C) {
    const int chunks = (C + 255) / 256;
    int s = (132 * 4) / (chunks * B);
    const int cap = (HW + 7) / 8 < 32 ? (HW + 7) / 8 : 32;
    if (s > cap) s = cap;
    return s < 1 ? 1 : s;
}

extern "C" long long b200_colsum_per_image_workspace_floats(int B, int HW, int C) {
    if (B <= 0 || HW <= 0 || C <= 0) return 0;
    return static_cast<long long>(B) * colsum_per_image_slices(B, HW, C) * C;
}

extern "C" int b200_colsum_per_image_bf16(const void* x_bf16, int B, int HW, int C, void* per_image_bf16, float* total, float* workspace,
                                          cudaStream_t stream) {
    const char* E = "colsum_per_image";
    if (B <= 0 || HW <= 0 || C <= 0 || C % 8 != 0) return refuse(B200_ERR_ARG, E, "need B, HW > 0 and C a positive multiple of 8");
    if (int_overflow(B, HW)) return refuse(B200_ERR_ARG, E, "too many rows");
    if (!x_bf16 || !per_image_bf16 || !total || !workspace) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {x_bf16})) return refuse(B200_ERR_ALIGN, E, "x not 16-byte aligned");
    if (!aligned(4, {per_image_bf16, total, workspace})) return refuse(B200_ERR_ALIGN, E, "per_image / total / workspace not 4-byte aligned");
    const int slices = colsum_per_image_slices(B, HW, C);
    colsum_per_image_kernel<<<dim3((C + 255) / 256, slices, B), dim3(32, 8), 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x_bf16), HW, C,
                                                                                         workspace);
    if (const int rc = check_launch("colsum_per_image")) return rc;
    colsum_per_image_finish_kernel<<<(C + 127) / 128, 128, 0, stream>>>(workspace, B, slices, C, reinterpret_cast<__nv_bfloat16*>(per_image_bf16),
                                                                        total);
    return check_launch("colsum_per_image_finish");
}

extern "C" int b200_splitk_reduce(const float* partial, int splits, long long n, float* out, int round_bf16,
                                  int accumulate, cudaStream_t stream) {
    const char* E = "splitk_reduce";
    if (splits < 1 || n <= 0 || n % 4 != 0) return refuse(B200_ERR_ARG, E, "need splits >= 1 and n a positive multiple of 4");
    if (!partial || !out) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {partial, out})) return refuse(B200_ERR_ALIGN, E, "partial / out not 16-byte aligned");
    const long long n4 = n / 4;
    splitk_reduce_kernel<<<static_cast<unsigned>((n4 + 255) / 256), 256, 0, stream>>>(partial, splits, n4, out, round_bf16, accumulate);
    return check_launch("splitk_reduce");
}

extern "C" int b200_patch_im2col(const float* x, void* cols_bf16, int B, int C, int img, int patch, cudaStream_t stream) {
    const char* E = "patch_im2col";
    if (B <= 0 || C <= 0 || img <= 0 || patch <= 0 || patch % 16 != 0 || img % patch != 0) return refuse(B200_ERR_ARG, E, "need patch % 16 == 0 and img % patch == 0");
    if (!x || !cols_bf16) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {x, cols_bf16})) return refuse(B200_ERR_ALIGN, E, "x / cols not 16-byte aligned");
    const long long total = static_cast<long long>(B) * C * img * (img / 16);
    patch_im2col_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(x, reinterpret_cast<__nv_bfloat16*>(cols_bf16), B, C, img, patch);
    return check_launch("patch_im2col");
}

extern "C" int b200_patch_im2col_u8(const void* x_u8_hwc, void* cols_bf16, int B, int C, int img, int patch, double division,
                                    const double* mean_host, const double* std_host, cudaStream_t stream) {
    const char* E = "patch_im2col_u8";
    if (B <= 0 || img <= 0 || patch <= 0 || patch % 16 != 0 || img % patch != 0) return refuse(B200_ERR_ARG, E, "need patch % 16 == 0 and img % patch == 0");
    if (C < 1 || C > 4) return refuse(B200_ERR_ARG, E, "1 <= channels <= 4");
    if (division == 0.0) return refuse(B200_ERR_ARG, E, "division == 0");
    NormParams np_;
    np_.division = division;
    for (int c = 0; c < 4; ++c) {
        np_.mean[c] = (mean_host != nullptr && c < C) ? mean_host[c] : 0.0;
        np_.stdv[c] = (std_host != nullptr && c < C) ? std_host[c] : 1.0;
        if (np_.stdv[c] == 0.0) return refuse(B200_ERR_ARG, E, "std == 0");
    }
    if (!x_u8_hwc || !cols_bf16) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {x_u8_hwc, cols_bf16})) return refuse(B200_ERR_ALIGN, E, "input / cols not 16-byte aligned");
    const long long total = static_cast<long long>(B) * img * (img / 16);
    const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
    const uint8_t* x = reinterpret_cast<const uint8_t*>(x_u8_hwc);
    __nv_bfloat16* cols = reinterpret_cast<__nv_bfloat16*>(cols_bf16);
    switch (C) {
        case 1: patch_im2col_u8_kernel<1><<<blocks, 256, 0, stream>>>(x, cols, B, img, patch, np_); break;
        case 2: patch_im2col_u8_kernel<2><<<blocks, 256, 0, stream>>>(x, cols, B, img, patch, np_); break;
        case 3: patch_im2col_u8_kernel<3><<<blocks, 256, 0, stream>>>(x, cols, B, img, patch, np_); break;
        default: patch_im2col_u8_kernel<4><<<blocks, 256, 0, stream>>>(x, cols, B, img, patch, np_); break;
    }
    return check_launch("patch_im2col_u8");
}

extern "C" int b200_assemble_tokens(const void* patch_bf16, const float* cls, const float* pos, float* net, int B, int np,
                                    int D, const void* conv_bias_bf16, cudaStream_t stream) {
    const char* E = "assemble_tokens";
    if (B <= 0 || np <= 0 || D <= 0 || D % 8 != 0) return refuse(B200_ERR_ARG, E, "need B, np > 0 and D a positive multiple of 8");
    if (!patch_bf16 || !cls || !pos || !net) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {patch_bf16, cls, pos, net, conv_bias_bf16})) return refuse(B200_ERR_ALIGN, E, "pointers must be 16-byte aligned");
    const long long total = static_cast<long long>(B) * (np + 1) * (D / 8);
    assemble_tokens_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(patch_bf16), cls, pos, net, B, np, D,
                                                                                       reinterpret_cast<const __nv_bfloat16*>(conv_bias_bf16));
    return check_launch("assemble_tokens");
}

extern "C" int b200_assemble_tokens_bwd(const float* dnet, void* dpatch_bf16, float* dpos, float* dcls, int B, int np,
                                        int D, int accumulate, cudaStream_t stream) {
    const char* E = "assemble_tokens_bwd";
    if (B <= 0 || np <= 0 || D <= 0 || D % 4 != 0) return refuse(B200_ERR_ARG, E, "need B, np > 0 and D a positive multiple of 4");
    if (int_overflow(np + 1ll, D / 4)) return refuse(B200_ERR_ARG, E, "(np + 1) * D / 4 overflows int");
    if (!dnet || !dpatch_bf16 || !dpos || !dcls) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {dnet, dpatch_bf16, dpos, dcls})) return refuse(B200_ERR_ALIGN, E, "pointers must be 16-byte aligned");
    const int total = (np + 1) * (D / 4);
    assemble_tokens_bwd_kernel<<<(total + 127) / 128, 128, 0, stream>>>(dnet, reinterpret_cast<__nv_bfloat16*>(dpatch_bf16), dpos, dcls, B, np, D, accumulate);
    return check_launch("assemble_tokens_bwd");
}

extern "C" int b200_embedding_fwd(const long long* ids, const float* weight, float* out, long long n, int D, int V,
                                  int* bad_index_flag, cudaStream_t stream) {
    const char* E = "embedding_fwd";
    if (n <= 0 || D <= 0 || D % 4 != 0 || V <= 0) return refuse(B200_ERR_ARG, E, "need n, V > 0 and D a positive multiple of 4");
    if (!ids || !weight || !out || !bad_index_flag) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {weight, out})) return refuse(B200_ERR_ALIGN, E, "weight / out not 16-byte aligned");
    if (!aligned(8, {ids}) || !aligned(4, {bad_index_flag})) return refuse(B200_ERR_ALIGN, E, "ids / flag not naturally aligned");
    const long long total = n * (D / 4);
    embedding_fwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(ids, weight, out, total, D / 4, V, bad_index_flag);
    return check_launch("embedding_fwd");
}

extern "C" int b200_embedding_bwd(const long long* ids, const float* dnet, float* dweight, long long n, int D, int V,
                                  int padding_idx, cudaStream_t stream) {
    const char* E = "embedding_bwd";
    if (n <= 0 || D <= 0 || V <= 0) return refuse(B200_ERR_ARG, E, "bad size");
    if (!ids || !dnet || !dweight) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(8, {ids}) || !aligned(4, {dnet, dweight})) return refuse(B200_ERR_ALIGN, E, "pointers not naturally aligned");
    const long long total = n * D;
    embedding_bwd_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(ids, dnet, dweight, total, D, V, padding_idx);
    return check_launch("embedding_bwd");
}

extern "C" int b200_argmax_gather_rows(const long long* ids, const float* x, float* out, int* pos, int B, int T, int D,
                                       cudaStream_t stream) {
    const char* E = "argmax_gather_rows";
    if (B <= 0 || T <= 0 || D <= 0) return refuse(B200_ERR_ARG, E, "bad size");
    if (!ids || !x || !out || !pos) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(8, {ids}) || !aligned(4, {x, out, pos})) return refuse(B200_ERR_ALIGN, E, "pointers not naturally aligned");
    argmax_gather_kernel<<<B, 128, 0, stream>>>(ids, x, out, pos, T, D);
    return check_launch("argmax_gather_rows");
}

extern "C" int b200_scatter_rows(const float* dout, const int* pos, float* dx, int B, int T, int D, cudaStream_t stream) {
    const char* E = "scatter_rows";
    if (B <= 0 || T <= 0 || D <= 0) return refuse(B200_ERR_ARG, E, "bad size");
    if (!dout || !pos || !dx) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(4, {dout, pos, dx})) return refuse(B200_ERR_ALIGN, E, "pointers not 4-byte aligned");
    scatter_rows_kernel<<<B, 128, 0, stream>>>(dout, pos, dx, T, D);
    return check_launch("scatter_rows");
}

extern "C" int b200_add_pos(const float* x, const float* pos, float* net, int B, int T, int D, cudaStream_t stream) {
    const char* E = "add_pos";
    if (B <= 0 || T <= 0 || D <= 0 || D % 4 != 0) return refuse(B200_ERR_ARG, E, "need B, T > 0 and D a positive multiple of 4");
    if (int_overflow(T, D / 4)) return refuse(B200_ERR_ARG, E, "T * D / 4 overflows int");
    if (!x || !pos || !net) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {x, pos, net})) return refuse(B200_ERR_ALIGN, E, "pointers must be 16-byte aligned");
    const long long n4 = static_cast<long long>(B) * T * (D / 4);
    add_pos_kernel<<<static_cast<unsigned>((n4 + 255) / 256), 256, 0, stream>>>(x, pos, net, n4, T * (D / 4));
    return check_launch("add_pos");
}

extern "C" int b200_add_pos_bwd(const float* dnet, float* dpos, int B, int T, int D, int accumulate, cudaStream_t stream) {
    const char* E = "add_pos_bwd";
    if (B <= 0 || T <= 0 || D <= 0 || D % 4 != 0) return refuse(B200_ERR_ARG, E, "need B, T > 0 and D a positive multiple of 4");
    if (int_overflow(T, D / 4)) return refuse(B200_ERR_ARG, E, "T * D / 4 overflows int");
    if (!dnet || !dpos) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {dnet, dpos})) return refuse(B200_ERR_ALIGN, E, "pointers must be 16-byte aligned");
    const int td4 = T * (D / 4);
    add_pos_bwd_kernel<<<(td4 + 127) / 128, 128, 0, stream>>>(dnet, dpos, B, td4, accumulate);
    return check_launch("add_pos_bwd");
}

extern "C" int b200_softmax_xent_fwd_bwd(const void* logits_bf16, long long ldl, const long long* labels,
                                         float* loss_rows, float* loss_mean, void* dlogits_bf16, int* bad_label_flag,
                                         int B, int C, float grad_scale, const float* grad_scale_dev,
                                         cudaStream_t stream) {
    const char* E = "softmax_xent";
    if (B <= 0 || C <= 0) return refuse(B200_ERR_ARG, E, "bad size");
    if (!logits_bf16 || !labels || !loss_rows || !bad_label_flag) return refuse(B200_ERR_ARG, E, "null pointer");
    if (ldl < C) return refuse(B200_ERR_ARG, E, "ldl < C");
    if (!aligned(2, {logits_bf16, dlogits_bf16}) || !aligned(8, {labels}) || !aligned(4, {loss_rows, loss_mean, bad_label_flag, grad_scale_dev}))
        return refuse(B200_ERR_ALIGN, E, "pointers not naturally aligned");
    softmax_xent_kernel<<<B, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(logits_bf16), ldl, labels, loss_rows,
                                               reinterpret_cast<__nv_bfloat16*>(dlogits_bf16), bad_label_flag, B, C, grad_scale, grad_scale_dev);
    int rc = check_launch("softmax_xent");
    if (rc) return rc;
    if (loss_mean != nullptr) {
        mean_kernel<<<1, 256, 0, stream>>>(loss_rows, B, loss_mean);
        rc = check_launch("loss_mean");
    }
    return rc;
}

extern "C" int b200_symmetric_xent_fwd_bwd(const void* logits_bf16, long long ldl, float* loss, void* dlogits_bf16, float* lse_ws, int B,
                                           float grad_scale, const float* grad_scale_dev, cudaStream_t stream) {
    const char* E = "symmetric_xent";
    if (B <= 0) return refuse(B200_ERR_ARG, E, "bad size");
    if (!logits_bf16 || !loss || !lse_ws) return refuse(B200_ERR_ARG, E, "null pointer");
    if (ldl < B) return refuse(B200_ERR_ARG, E, "ldl < B");
    if (!aligned(2, {logits_bf16, dlogits_bf16}) || !aligned(4, {loss, lse_ws, grad_scale_dev}))
        return refuse(B200_ERR_ALIGN, E, "pointers not naturally aligned");
    const __nv_bfloat16* lg = reinterpret_cast<const __nv_bfloat16*>(logits_bf16);
    sym_xent_stats_kernel<<<(2 * B + 7) / 8, 256, 0, stream>>>(lg, ldl, B, lse_ws);
    int rc = check_launch("symmetric_xent_stats");
    if (rc) return rc;
    sym_xent_loss_kernel<<<1, 256, 0, stream>>>(lg, ldl, B, lse_ws, loss);
    if ((rc = check_launch("symmetric_xent_loss")) != 0) return rc;
    if (dlogits_bf16 != nullptr) {
        const long long n = static_cast<long long>(B) * B;
        sym_xent_grad_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(lg, ldl, B, lse_ws, reinterpret_cast<__nv_bfloat16*>(dlogits_bf16),
                                                                                        grad_scale, grad_scale_dev);
        rc = check_launch("symmetric_xent_grad");
    }
    return rc;
}

extern "C" int b200_cast_f32_to_bf16(const float* src, void* dst_bf16, long long n, cudaStream_t stream) {
    const char* E = "cast";
    if (n <= 0) return refuse(B200_ERR_ARG, E, "n <= 0");
    if (!src || !dst_bf16) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {src, dst_bf16})) return refuse(B200_ERR_ALIGN, E, "src / dst not 16-byte aligned");
    const long long thr = (n + 7) / 8;
    cast_f32_bf16_kernel<<<static_cast<unsigned>((thr + 255) / 256), 256, 0, stream>>>(src, reinterpret_cast<__nv_bfloat16*>(dst_bf16), n);
    return check_launch("cast_f32_bf16");
}
template <bool kDecoupled>
static int adam_step_host(const char* E, float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n, float lr,
                          float beta1, float beta2, float eps, float weight_decay, int step, int* step_dev, cudaStream_t stream) {
    if (n <= 0 || n % 4 != 0) return refuse(B200_ERR_ARG, E, "n must be a positive multiple of 4");
    if (step_dev == nullptr && step < 1) return refuse(B200_ERR_ARG, E, "step >= 1 (or pass step_dev)");
    if (!params || !grads || !exp_avg || !exp_avg_sq) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {params, grads, exp_avg, exp_avg_sq})) return refuse(B200_ERR_ALIGN, E, "arenas not 16-byte aligned");
    if (!aligned(4, {step_dev})) return refuse(B200_ERR_ALIGN, E, "step_dev not 4-byte aligned");
    if (step_dev != nullptr) {
        increment_kernel<<<1, 1, 0, stream>>>(step_dev);
        int rc = check_launch("adam_step_increment");
        if (rc) return rc;
    }
    const float t = static_cast<float>(step < 1 ? 1 : step);
    const float bc1 = 1.0f - powf(beta1, t);
    const float bc2_sqrt = sqrtf(1.0f - powf(beta2, t));
    const long long n4 = n / 4;
    adam_kernel<kDecoupled><<<static_cast<unsigned>((n4 + 255) / 256), 256, 0, stream>>>(params, grads, exp_avg, exp_avg_sq, n4, lr,
                                                                                      beta1, beta2, eps, weight_decay, bc1, bc2_sqrt,
                                                                                      step_dev);
    return check_launch(E);
}
template <bool kDecoupled>
static int adam_step_dev_host(const char* E, float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                              const float* hyper_dev, int* step_dev, int increment, cudaStream_t stream) {
    if (n <= 0 || n % 4 != 0) return refuse(B200_ERR_ARG, E, "n must be a positive multiple of 4");
    if (!params || !grads || !exp_avg || !exp_avg_sq || !hyper_dev || !step_dev) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {params, grads, exp_avg, exp_avg_sq})) return refuse(B200_ERR_ALIGN, E, "arenas not 16-byte aligned");
    if (!aligned(4, {hyper_dev, step_dev})) return refuse(B200_ERR_ALIGN, E, "hyper_dev / step_dev not 4-byte aligned");
    if (increment) {
        increment_kernel<<<1, 1, 0, stream>>>(step_dev);
        int rc = check_launch("adam_step_increment");
        if (rc) return rc;
    }
    const long long n4 = n / 4;
    adam_dev_kernel<kDecoupled><<<static_cast<unsigned>((n4 + 255) / 256), 256, 0, stream>>>(params, grads, exp_avg, exp_avg_sq, n4,
                                                                                          hyper_dev, step_dev);
    return check_launch(E);
}
extern "C" int b200_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                              float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                              int* step_dev, cudaStream_t stream) {
    return adam_step_host<false>("adam_step", params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step,
                                 step_dev, stream);
}
extern "C" int b200_adam_step_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                                  const float* hyper_dev, int* step_dev, int increment, cudaStream_t stream) {
    return adam_step_dev_host<false>("adam_step_dev", params, grads, exp_avg, exp_avg_sq, n, hyper_dev, step_dev, increment, stream);
}
extern "C" int b200_adamw_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                               float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                               int* step_dev, cudaStream_t stream) {
    return adam_step_host<true>("adamw_step", params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step,
                                step_dev, stream);
}
extern "C" int b200_adamw_step_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n,
                                   const float* hyper_dev, int* step_dev, int increment, cudaStream_t stream) {
    return adam_step_dev_host<true>("adamw_step_dev", params, grads, exp_avg, exp_avg_sq, n, hyper_dev, step_dev, increment, stream);
}
extern "C" int b200_fill_f32(float* dst, float value, long long n, cudaStream_t stream) {
    const char* E = "fill";
    if (n <= 0) return refuse(B200_ERR_ARG, E, "n <= 0");
    if (!dst) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(16, {dst})) return refuse(B200_ERR_ALIGN, E, "dst not 16-byte aligned");
    const long long thr = (n + 3) / 4;
    fill_f32_kernel<<<static_cast<unsigned>((thr + 255) / 256), 256, 0, stream>>>(dst, value, n);
    return check_launch("fill_f32");
}

// ------------------------------------------------------------------------------------------------
// row softmax of the KL decoder's single-head spatial attention (include/b200_cflearn_ext.h)
// ------------------------------------------------------------------------------------------------
namespace b200 {

constexpr int SOFTMAX_THREADS = 256;

// the block's max or sum of v (every thread gets it), reduced in a fixed order
template <bool kMax>
__device__ __forceinline__ float softmax_block_reduce(float v, float* red) {
    v = kMax ? warp_max(v) : warp_sum(v);
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    v = lane < SOFTMAX_THREADS / 32 ? red[lane] : (kMax ? -INFINITY : 0.f);
    v = kMax ? warp_max(v) : warp_sum(v);
    __syncthreads();  // red is reused by the next reduction
    return v;
}

// One block per row: m = max_c s[c], l = sum_c exp(scale (s[c] - m)), p[c] = bf16(exp(scale (s[c] - m)) / l).  Two reads of the
// fp32 row (the second mostly from L2), one bf16 write.
__global__ void __launch_bounds__(SOFTMAX_THREADS) softmax_rows_kernel(const float* __restrict__ s, long long lds, __nv_bfloat16* __restrict__ p,
                                                                       long long ldp, int cols, float scale) {
    __shared__ float red[SOFTMAX_THREADS / 32];
    const float* row = s + static_cast<long long>(blockIdx.x) * lds;
    __nv_bfloat16* out = p + static_cast<long long>(blockIdx.x) * ldp;
    float m = -INFINITY;
    for (int c = threadIdx.x; c < cols; c += SOFTMAX_THREADS) m = fmaxf(m, row[c]);
    m = softmax_block_reduce<true>(m, red);
    float l = 0.f;
    for (int c = threadIdx.x; c < cols; c += SOFTMAX_THREADS) l += expf(scale * (row[c] - m));
    l = softmax_block_reduce<false>(l, red);
    for (int c = threadIdx.x; c < cols; c += SOFTMAX_THREADS) out[c] = __float2bfloat16_rn(expf(scale * (row[c] - m)) / l);
}

}  // namespace b200

extern "C" int b200_softmax_rows_bf16(const float* s, long long lds, void* p_bf16, long long ldp, int rows, int cols, float scale,
                                      cudaStream_t stream) {
    const char* E = "softmax_rows";
    if (rows <= 0 || cols <= 0) return refuse(B200_ERR_ARG, E, "non-positive size");
    if (!(scale > 0.f) || isinf(scale)) return refuse(B200_ERR_ARG, E, "scale must be positive and finite");
    if (lds < cols || ldp < cols) return refuse(B200_ERR_ARG, E, "lds / ldp < cols");
    if (!s || !p_bf16) return refuse(B200_ERR_ARG, E, "null pointer");
    if (!aligned(4, {s}) || !aligned(2, {p_bf16})) return refuse(B200_ERR_ALIGN, E, "s not 4-byte / p not 2-byte aligned");
    softmax_rows_kernel<<<rows, SOFTMAX_THREADS, 0, stream>>>(s, lds, reinterpret_cast<__nv_bfloat16*>(p_bf16), ldp, cols, scale);
    return check_launch(E);
}
