// Fused multi-head self-attention forward / backward for sm_90a on the PACKED qkv tensor [B, T, 3*H*64].
//
// Replaces, per transformer block of the reference:
//   qkv.chunk(3) + _to_heads permutes + .contiguous() copies   cflearn/modules/core/attentions.py:216,180-185,245
//   F.scaled_dot_product_attention (via sdp_attn)               cflearn/toolkit.py:911-974
//   output.transpose(1,2).contiguous()                          cflearn/modules/core/attentions.py:270
// and their autograd.  T <= 256 (197 for ViT-B/16, 50 / 77 for CLIP) so every K / V tile of a head fits in shared memory
// at once: no online-softmax rescaling is needed and a warpgroup holds whole score rows in registers.  Longer sequences (up
// to 16384) go to the streamed kernels at the end of this file (attn_long_*), which reuse these helpers.
//
// Every product is a warpgroup MMA (wgmma m64n64k16, fp32 accumulators in registers).  Operands that come from memory are
// TMA-loaded 128B-swizzled tiles (a 3-D tensor map over qkv: rows >= T are zero-filled); operands that were just computed
// (P, P^T, dS, dS^T) go from the accumulator registers straight into the A-operand registers of the next wgmma -- the
// accumulator fragment of a 64 x 16 column slice IS the A fragment of a k16 step -- so they never touch shared memory.
//
// Forward, one CTA per (batch, head, 128-query tile), 2 warpgroups of 64 queries:
//   S = Q K^T (64 x Tp per warpgroup), softmax in registers (a row lives in the 4 lanes of a quad), O = P V, O / rowsum.
// Backward, one CTA per (batch, head), Q / K / V / dO of the head resident in shared memory:
//   phase 1, warpgroup = 64-key tile:   S^T = K Q^T, dP^T = V dO^T -> P^T, dS^T -> dV += P^T dO, dK += dS^T Q
//   phase 2, warpgroup = 64-query tile: S = Q K^T,   dP = dO V^T   -> P, dS     -> dQ += dS K
// (phase 2 recomputes S and dP instead of exchanging dS through shared memory or fp32 atomics: deterministic, and the
// attention's share of the step's FLOPs is small).
// Numerics mirror the flash kernels torch dispatches to: fp32 scores / softmax / row sums, P and dS rounded to
// bf16 only as MMA operands, softmax scale folded into exp2, dQ / dK scaled in fp32 at the end.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <initializer_list>

#include "b200_internal.h"
#include "ptx.cuh"

namespace b200 {

constexpr float kLog2e = 1.4426950408889634f;
constexpr int ATT_THREADS = 256;   // two warpgroups
constexpr int TILE_BYTES = 8192;   // 64 rows x 64 bf16, 128B-swizzled

struct AttnParams {
    int B, T, H, D;   // D = H * 64
    int tp;           // T rounded up to a multiple of 64 (<= 256)
    float scale;
    int causal;
};

__device__ __forceinline__ uint64_t kmajor_desc(uint32_t addr) { return make_smem_desc(addr, 16, 1024, kSwz128); }
__device__ __forceinline__ uint64_t mnmajor_desc(uint32_t addr) { return make_smem_desc(addr, TILE_BYTES, 1024, kSwz128); }

// acc (+)= A[64 x 64] * B[64 x 64]^T, both K-major tiles in shared memory (K = 64 = head dim)
__device__ __forceinline__ void mma_tile_kk(float (&acc)[32], uint32_t a_base, uint32_t b_base) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_ss(acc, kmajor_desc(a_base + kk * 32), kmajor_desc(b_base + kk * 32), kk > 0 ? 1u : 0u);
}
// A fragment of k16 step s from a 64 x 64 accumulator-layout array of probabilities (n8 blocks 2s, 2s + 1), rounded to bf16
__device__ __forceinline__ void a_frag(const float (&v)[32], int s, uint32_t (&a)[4]) {
    a[0] = pack_bf16x2(v[8 * s + 0], v[8 * s + 1]);
    a[1] = pack_bf16x2(v[8 * s + 2], v[8 * s + 3]);
    a[2] = pack_bf16x2(v[8 * s + 4], v[8 * s + 5]);
    a[3] = pack_bf16x2(v[8 * s + 6], v[8 * s + 7]);
}
// Stores a warpgroup's 64 x 64 accumulator (rows row0 + {0, 8} per thread, see ptx.cuh) times `sc` as bf16 at g0 + row *
// stride; rows >= nrows are skipped.  csum (optional): this warp's fp32 column sums of the bf16 values written, 64 floats.
// kCols: columns >= ncols are skipped as well (a head dim padded to whole 64-column boxes).
template <bool kCols = false>
__device__ __forceinline__ void store_tile(const float (&v)[32], float sc, __nv_bfloat16* g0, long long stride, int row0, int nrows,
                                           int lane, float* csum, int ncols = 64) {
    const int c0 = (lane & 3) * 2;
    float cs[16];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = row0 + h * 8;
            const uint32_t t = pack_bf16x2(v[4 * j + 2 * h] * sc, v[4 * j + 2 * h + 1] * sc);
            const bool ok = row < nrows && (!kCols || j * 8 + c0 < ncols);
            if (ok) *reinterpret_cast<uint32_t*>(g0 + row * stride + j * 8 + c0) = t;
            if (h == 0) { cs[2 * j] = 0.f; cs[2 * j + 1] = 0.f; }
            if (ok) { cs[2 * j] += bf16lo(t); cs[2 * j + 1] += bf16hi(t); }
        }
    }
    if (csum == nullptr) return;
#pragma unroll
    for (int k = 0; k < 16; ++k) {  // lanes with the same lane % 4 hold the same columns of different rows
        cs[k] += __shfl_xor_sync(0xffffffffu, cs[k], 4);
        cs[k] += __shfl_xor_sync(0xffffffffu, cs[k], 8);
        cs[k] += __shfl_xor_sync(0xffffffffu, cs[k], 16);
    }
    if (lane < 4) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            csum[j * 8 + lane * 2] = cs[2 * j];
            csum[j * 8 + lane * 2 + 1] = cs[2 * j + 1];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
constexpr int AF_SQ = 0;            // 16 KB: the 128-query tile
constexpr int AF_SK = 16384;        // up to 32 KB
constexpr int AF_SV = 49152;        // up to 32 KB
constexpr int AF_BAR = 81920;
constexpr int AF_SMEM = AF_BAR + 64 + 1024;

__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                __nv_bfloat16* __restrict__ out, float* __restrict__ lse_out, const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* bar_load = reinterpret_cast<uint64_t*>(smem + AF_BAR);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_mt = (p.T + 127) / 128;
    const int mt = blockIdx.x % n_mt;
    const int bh = blockIdx.x / n_mt;
    const int h = bh % p.H;
    const int b = bh / p.H;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmKV);
        mbar_init(bar_load, 1);
        fence_mbar_init();
        mbar_expect_tx(bar_load, 16384u + 2u * static_cast<uint32_t>(p.tp) * 128u);
        tma_load_3d(smem + AF_SQ, &tmQ, bar_load, h * 64, mt * 128, b);
        tma_load_3d(smem + AF_SK, &tmKV, bar_load, p.D + h * 64, 0, b);
        tma_load_3d(smem + AF_SV, &tmKV, bar_load, 2 * p.D + h * 64, 0, b);
    }
    __syncthreads();
    const int g = warp >> 2;  // warpgroup: queries [64 g, 64 g + 64) of the tile
    const int rl = (warp & 3) * 16 + (lane >> 2);
    const int i0 = mt * 128 + g * 64 + rl;  // this thread's query rows: i0 and i0 + 8
    if (mt * 128 + g * 64 >= p.T) return;   // (a warpgroup of padding rows only)
    const int nkc = p.tp / 64;
    const float sl2 = p.scale * kLog2e;
    const uint32_t q_base = smem_u32(smem + AF_SQ) + g * TILE_BYTES;
    const uint32_t k_base = smem_u32(smem + AF_SK), v_base = smem_u32(smem + AF_SV);
    mbar_wait(bar_load, 0);

    float s[4][32];
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 4; ++c)
        if (c < nkc) mma_tile_kk(s[c], q_base, k_base + c * TILE_BYTES);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < 4; ++c)
        if (c < nkc) reg_fence(s[c]);

    // row max (masked), combined over the quad that shares a row
    float m[2] = {-INFINITY, -INFINITY};
    const int jq = (lane & 3) * 2;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (c >= nkc) continue;
#pragma unroll
        for (int e = 0; e < 32; ++e) {
            const int hr = (e >> 1) & 1;
            const int j = c * 64 + (e >> 2) * 8 + jq + (e & 1);
            const bool ok = j < p.T && (!p.causal || j <= i0 + 8 * hr);
            if (!ok) s[c][e] = -INFINITY;
            m[hr] = fmaxf(m[hr], s[c][e]);
        }
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        m[hr] = fmaxf(m[hr], __shfl_xor_sync(0xffffffffu, m[hr], 1));
        m[hr] = fmaxf(m[hr], __shfl_xor_sync(0xffffffffu, m[hr], 2));
    }
    const float m2[2] = {m[0] * sl2, m[1] * sl2};
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (c >= nkc) continue;
#pragma unroll
        for (int e = 0; e < 32; ++e) {
            const int hr = (e >> 1) & 1;
            const float pv = fast_ex2(fmaf(s[c][e], sl2, -m2[hr]));  // exp2(-inf) = 0 for masked keys
            s[c][e] = pv;
            sum[hr] += pv;
        }
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        sum[hr] += __shfl_xor_sync(0xffffffffu, sum[hr], 1);
        sum[hr] += __shfl_xor_sync(0xffffffffu, sum[hr], 2);
    }
    // O = P V: P from registers (bf16), V MN-major from shared memory
    float o[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) o[e] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (c >= nkc) continue;
#pragma unroll
        for (int st = 0; st < 4; ++st) {
            uint32_t a[4];
            a_frag(s[c], st, a);
            wgmma_m64n64k16_rs_tb(o, a, mnmajor_desc(v_base + c * TILE_BYTES + st * 2048), 1u);
        }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    const float inv[2] = {1.0f / sum[0], 1.0f / sum[1]};
#pragma unroll
    for (int e = 0; e < 32; ++e) o[e] *= inv[(e >> 1) & 1];
    __nv_bfloat16* g0 = out + (static_cast<long long>(b) * p.T) * p.D + h * 64;
    store_tile(o, 1.0f, g0, p.D, i0, p.T, lane, nullptr);
    if ((lane & 3) == 0) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int i = i0 + 8 * hr;
            if (i < p.T) lse_out[(static_cast<long long>(b) * p.H + h) * p.T + i] = m[hr] * p.scale + logf(sum[hr]);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
constexpr int AB_SQ = 0;          // up to 32 KB each: Q, dO, K, V of the head
constexpr int AB_SDO = 32768;
constexpr int AB_SK = 65536;
constexpr int AB_SV = 98304;
constexpr int AB_LSE = 131072;    // 256 floats: lse * log2(e) (+inf on padded rows)
constexpr int AB_DELTA = AB_LSE + 1024;
constexpr int AB_CSUM = AB_DELTA + 1024;  // [3][4 tiles][4 warps][64] column sums of dQ / dK / dV
constexpr int AB_BAR = AB_CSUM + 3 * 16 * 64 * 4;
constexpr int AB_SMEM = AB_BAR + 64 + 1024;

__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO,
                const __nv_bfloat16* __restrict__ o_in, const __nv_bfloat16* __restrict__ do_in,
                const float* __restrict__ lse_in, __nv_bfloat16* __restrict__ dqkv, float* __restrict__ dbias_part,
                const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    float* lse_s = reinterpret_cast<float*>(smem + AB_LSE);
    float* delta_s = reinterpret_cast<float*>(smem + AB_DELTA);
    float* csum = reinterpret_cast<float*>(smem + AB_CSUM);
    uint64_t* bar_load = reinterpret_cast<uint64_t*>(smem + AB_BAR);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int h = blockIdx.x % p.H;
    const int b = blockIdx.x / p.H;
    const long long D3 = 3ll * p.D;
    const int nt = p.tp / 64;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQKV);
        tma_prefetch_desc(&tmDO);
        mbar_init(bar_load, 1);
        fence_mbar_init();
        mbar_expect_tx(bar_load, 4u * static_cast<uint32_t>(p.tp) * 128u);
        tma_load_3d(smem + AB_SQ, &tmQKV, bar_load, h * 64, 0, b);
        tma_load_3d(smem + AB_SK, &tmQKV, bar_load, p.D + h * 64, 0, b);
        tma_load_3d(smem + AB_SV, &tmQKV, bar_load, 2 * p.D + h * 64, 0, b);
        tma_load_3d(smem + AB_SDO, &tmDO, bar_load, h * 64, 0, b);
    }
    {
        // delta_i = sum_d dO[i,d] O[i,d] and the log2-domain lse, one query row per thread (overlaps the TMA loads)
        const int i = threadIdx.x;
        float dl = 0.f, l2 = INFINITY;  // padded query rows: exp2(s - inf) = 0 -> P = dS = 0 for free
        if (i < p.T) {
            const uint4* po = reinterpret_cast<const uint4*>(o_in + (static_cast<long long>(b) * p.T + i) * p.D + h * 64);
            const uint4* pd = reinterpret_cast<const uint4*>(do_in + (static_cast<long long>(b) * p.T + i) * p.D + h * 64);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint4 a = __ldg(po + k), gg = __ldg(pd + k);
                dl += bf16lo(a.x) * bf16lo(gg.x) + bf16hi(a.x) * bf16hi(gg.x) + bf16lo(a.y) * bf16lo(gg.y) + bf16hi(a.y) * bf16hi(gg.y) +
                      bf16lo(a.z) * bf16lo(gg.z) + bf16hi(a.z) * bf16hi(gg.z) + bf16lo(a.w) * bf16lo(gg.w) + bf16hi(a.w) * bf16hi(gg.w);
            }
            l2 = __ldg(lse_in + (static_cast<long long>(b) * p.H + h) * p.T + i) * kLog2e;
        }
        lse_s[i] = l2;
        delta_s[i] = dl;
        for (int k = threadIdx.x; k < 3 * 16 * 64; k += ATT_THREADS) csum[k] = 0.f;
    }
    __syncthreads();
    mbar_wait(bar_load, 0);

    const int g = warp >> 2;
    const int wq = warp & 3;
    const int rl = wq * 16 + (lane >> 2);   // accumulator rows rl, rl + 8 of a 64-row tile
    const int jq = (lane & 3) * 2;          // accumulator columns 8 n + jq (+ 1)
    const float sl2 = p.scale * kLog2e;
    const uint32_t q_base = smem_u32(smem + AB_SQ), do_base = smem_u32(smem + AB_SDO);
    const uint32_t k_base = smem_u32(smem + AB_SK), v_base = smem_u32(smem + AB_SV);

    // ---- phase 1: warpgroup g owns key tiles g, g + 2: dV = P^T dO, dK = dS^T Q ----
    for (int kt = g; kt < nt; kt += 2) {
        float dv[32], dk[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) { dv[e] = 0.f; dk[e] = 0.f; }
        const int key0 = kt * 64 + rl;
        for (int qc = 0; qc < nt; ++qc) {
            if (p.causal && qc * 64 + 63 < kt * 64) continue;  // every query of the chunk precedes every key of the tile
            float st[32], dpt[32];
            wgmma_fence();
            mma_tile_kk(st, k_base + kt * TILE_BYTES, q_base + qc * TILE_BYTES);
            mma_tile_kk(dpt, v_base + kt * TILE_BYTES, do_base + qc * TILE_BYTES);
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(st);
            reg_fence(dpt);
#pragma unroll
            for (int e = 0; e < 32; ++e) {
                const int key = key0 + ((e >> 1) & 1) * 8;
                const int i = qc * 64 + (e >> 2) * 8 + jq + (e & 1);
                const bool ok = key < p.T && (!p.causal || key <= i);
                const float pv = ok ? fast_ex2(fmaf(st[e], sl2, -lse_s[i])) : 0.f;
                st[e] = pv;
                dpt[e] = pv * (dpt[e] - delta_s[i]);
            }
            wgmma_fence();
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                uint32_t a[4];
                a_frag(st, s, a);
                wgmma_m64n64k16_rs_tb(dv, a, mnmajor_desc(do_base + qc * TILE_BYTES + s * 2048), 1u);
                a_frag(dpt, s, a);
                wgmma_m64n64k16_rs_tb(dk, a, mnmajor_desc(q_base + qc * TILE_BYTES + s * 2048), 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(dv);
            reg_fence(dk);
        }
        __nv_bfloat16* g0 = dqkv + (static_cast<long long>(b) * p.T) * D3 + h * 64;
        store_tile(dk, p.scale, g0 + p.D, D3, key0, p.T, lane, csum + ((1 * 4 + kt) * 4 + wq) * 64);
        store_tile(dv, 1.0f, g0 + 2 * p.D, D3, key0, p.T, lane, csum + ((2 * 4 + kt) * 4 + wq) * 64);
    }

    // ---- phase 2: warpgroup g owns query tiles g, g + 2: dQ = dS K ----
    for (int qt = g; qt < nt; qt += 2) {
        float dq[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) dq[e] = 0.f;
        const int i0 = qt * 64 + rl;
        const float l2[2] = {lse_s[i0], lse_s[i0 + 8]};
        const float de[2] = {delta_s[i0], delta_s[i0 + 8]};
        for (int kt = 0; kt < nt; ++kt) {
            if (p.causal && kt * 64 > qt * 64 + 63) continue;  // every key of the tile follows every query of the chunk
            float sc[32], dp[32];
            wgmma_fence();
            mma_tile_kk(sc, q_base + qt * TILE_BYTES, k_base + kt * TILE_BYTES);
            mma_tile_kk(dp, do_base + qt * TILE_BYTES, v_base + kt * TILE_BYTES);
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(sc);
            reg_fence(dp);
#pragma unroll
            for (int e = 0; e < 32; ++e) {
                const int hr = (e >> 1) & 1;
                const int j = kt * 64 + (e >> 2) * 8 + jq + (e & 1);
                const bool ok = j < p.T && (!p.causal || j <= i0 + 8 * hr);
                const float pv = ok ? fast_ex2(fmaf(sc[e], sl2, -l2[hr])) : 0.f;
                dp[e] = pv * (dp[e] - de[hr]);
            }
            wgmma_fence();
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                uint32_t a[4];
                a_frag(dp, s, a);
                wgmma_m64n64k16_rs_tb(dq, a, mnmajor_desc(k_base + kt * TILE_BYTES + s * 2048), 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(dq);
        }
        __nv_bfloat16* g0 = dqkv + (static_cast<long long>(b) * p.T) * D3 + h * 64;
        store_tile(dq, p.scale, g0, D3, i0, p.T, lane, csum + ((0 * 4 + qt) * 4 + wq) * 64);
    }

    if (dbias_part != nullptr) {
        // per-(batch, head) column sums of dq | dk | dv in a fixed order: the qkv-bias gradient is their sum over the batch
        __syncthreads();
        if (threadIdx.x < 192) {
            const int sec = threadIdx.x >> 6, c = threadIdx.x & 63;
            float t = 0.f;
            for (int k = 0; k < 16; ++k) t += csum[(sec * 16 + k) * 64 + c];
            dbias_part[static_cast<long long>(b) * D3 + sec * p.D + h * 64 + c] = t;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// streamed kernels (1 <= Tq, Tk <= 16384, head dim Dh <= 160, separate Q / K / V operands)
// ------------------------------------------------------------------------------------------------
// The kernels above hold a head's whole K / V (or Q / dO) in shared memory, loaded as ONE TMA box of tp <= 256 rows.
// The kernels below keep one side of the product resident and stream the other through a ring of 64-row TMA blocks with
// full / empty mbarriers (FlashAttention-2 scheme, the pipeline of the GEMM in gemm_sm90.cu):
//   forward   one CTA per (image, head, 128-query tile): Q resident, K / V streamed, online softmax in fp32
//   delta     delta = rowsum(dO o O) in fp32, one value per (image, head, query), into the workspace
//   dK / dV   one CTA per (image, head, key tile[, query chunk]): K / V resident, Q / dO streamed with their lse / delta rows
//   dQ        one CTA per (image, head, 128-query tile): Q / dO / lse / delta resident, K / V streamed
//   dbias     per-64-row-tile column sums of the stored dq | dk | dv, summed per image in a fixed order (packed layout only)
// Q is [B, Tq, ldq] with head h at column h * Dh, K / V are [B, Tk, ldkv]; the packed qkv tensor is q = qkv, k = qkv + D,
// v = qkv + 2 D with ld = 3 D.  Every operand is read through a 4-D tensor map {Dh, H, T, B} with 64 x 64 boxes, so columns
// >= Dh and rows >= T arrive as zeros.  The kernels are instantiated per k16-step count KS of S = Q K^T and dP = dO V^T
// (attn_long_ksteps: ceil(Dh / 16) up to Dh 80, then 8 and 10), the head dim is padded to NB = ceil(KS / 4) whole 64-column
// boxes, and outputs skip the padding.
// Warp 8 is the TMA producer; warpgroup g in {0, 1} owns rows [64 g, 64 g + 64) of the CTA's tile (the NB > 1 dK / dV kernel
// splits its work differently, see there).  Causal CTAs (Tq == Tk) stop at the diagonal.  Nothing is accumulated with
// atomics: two runs give bit-identical results.
constexpr int LA_THREADS = 288;  // two consumer warpgroups + the producer warp
constexpr int LA_MAX_T = 16384;
constexpr int LA_MAX_DH = 160;
constexpr int LA_SMS = 132;  // H100 SXM: a dK / dV grid smaller than this is split over the queries

struct LongParams {
    int B, Tq, Tk, H, Dh;
    long long ldq, ldkv, ldo;  // leading dims (elements) of q / dq, k / v / dk / dv, out / dout
    float scale;
    int causal;
    int qb_chunk;  // dK / dV: 64-query blocks per chunk
    int nchunk;    // dK / dV: query chunks; > 1 writes fp32 partials that attn_long_dkdv_reduce_kernel sums in chunk order
};

// Shared-memory layouts per padded head dim.  Stage counts keep every kernel <= 227 KB; NB = 1 fits two forward CTAs per SM.
template <int NB>
struct LongCfg {
    static constexpr int BOX = NB * TILE_BYTES;  // one 64-row block over the padded head dim
    // forward: 128-query tile, per stage a K block and a V block
    static constexpr int F_STAGES = NB == 3 ? 3 : 4;
    static constexpr int F_Q = 0;
    static constexpr int F_KV = 2 * BOX;
    static constexpr int F_BAR = F_KV + F_STAGES * 2 * BOX;  // full[S], empty[S], q
    static constexpr int F_SMEM = F_BAR + 128 + 1024;
    // dK / dV: NB = 1 keeps a 128-key tile, a warpgroup per 64 keys, each accumulating dK and dV.  For NB > 1 those two
    // accumulators (2 x 32 NB fp32 per thread) plus S^T and dP^T exceed the register budget, so both warpgroups share a 64-key
    // tile: warpgroup 0 computes P^T and dV += P^T dO, warpgroup 1 dP^T, dS^T and dK += dS^T Q, and P^T is handed from 0 to 1
    // through shared memory in fp32 (K_PB) -- two GEMMs per warpgroup, nothing recomputed.
    static constexpr int K_ROWS = NB == 1 ? 128 : 64;
    static constexpr int K_STAGES = NB == 3 ? 3 : 4;
    static constexpr int K_K = 0;
    static constexpr int K_V = K_ROWS / 64 * BOX;
    static constexpr int K_QD = 2 * K_V;                          // per stage: Q block, dO block
    static constexpr int K_ROW = K_QD + K_STAGES * 2 * BOX;       // per stage: lse * log2(e) [64], delta [64]
    static constexpr int K_CS = K_ROW + K_STAGES * 512;           // NB = 1: [dk | dv][warpgroup][warp][64] column sums
    static constexpr int K_PB = K_CS + (NB == 1 ? 2 * 8 * 64 * 4 : 0);  // NB > 1: P^T, [32 values][128 threads] fp32
    static constexpr int K_BAR = K_PB + (NB == 1 ? 0 : 32 * 128 * 4);
    static constexpr int K_SMEM = K_BAR + 128 + 1024;
    // dQ: 128-query tile of Q and dO, per stage a K block and a V block
    static constexpr int Q_STAGES = NB == 3 ? 2 : 4;
    static constexpr int Q_Q = 0;
    static constexpr int Q_DO = 2 * BOX;
    static constexpr int Q_KV = 4 * BOX;
    static constexpr int Q_CS = Q_KV + Q_STAGES * 2 * BOX;  // [warpgroup][warp][64] column sums
    static constexpr int Q_BAR = Q_CS + 8 * 64 * 4;
    static constexpr int Q_SMEM = Q_BAR + 128 + 1024;
};
static_assert(LongCfg<1>::F_SMEM == 83072 && LongCfg<1>::K_SMEM == 105600 && LongCfg<1>::Q_SMEM == 101504, "Dh 64 layouts");
static_assert(LongCfg<3>::F_SMEM <= 232448 && LongCfg<3>::K_SMEM <= 232448 && LongCfg<3>::Q_SMEM <= 232448, "227 KB");
static_assert(LongCfg<2>::F_SMEM <= 232448 && LongCfg<2>::K_SMEM <= 232448 && LongCfg<2>::Q_SMEM <= 232448, "227 KB");

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// acc = A B^T over the first KS k16 steps of the padded head dim: A and B are 64-row blocks of K-major 64-column boxes
template <int KS>
__device__ __forceinline__ void mma_rows_kk(float (&acc)[32], uint32_t a_base, uint32_t b_base) {
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
        const uint32_t off = (kk >> 2) * TILE_BYTES + (kk & 3) * 32;
        wgmma_m64n64k16_ss(acc, kmajor_desc(a_base + off), kmajor_desc(b_base + off), kk > 0 ? 1u : 0u);
    }
}

// fp32 copy of a warpgroup's 64 x 64 accumulator: rows < nrows, columns < ncols, at p0 + row * ld
__device__ __forceinline__ void store_part(const float (&v)[32], float* p0, int ld, int row0, int nrows, int ncols, int lane) {
    const int c0 = (lane & 3) * 2;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = row0 + h * 8;
            if (row < nrows && j * 8 + c0 < ncols)
                *reinterpret_cast<float2*>(p0 + static_cast<long long>(row) * ld + j * 8 + c0) = make_float2(v[4 * j + 2 * h], v[4 * j + 2 * h + 1]);
        }
    }
}

template <int KS>
__global__ void __launch_bounds__(LA_THREADS, KS <= 4 ? 2 : 1)
attn_long_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                     __nv_bfloat16* __restrict__ out, float* __restrict__ lse_out, const LongParams p) {
    constexpr int NB = (KS + 3) / 4;
    using C = LongCfg<NB>;
    constexpr int S = C::F_STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::F_BAR);
    uint64_t* empty = full + S;
    uint64_t* bar_q = empty + S;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_mt = (p.Tq + 127) / 128;
    const int mt = blockIdx.x % n_mt;
    const int bh = blockIdx.x / n_mt;
    const int h = bh % p.H;
    const int b = bh / p.H;
    const int n_cons = mt * 128 + 64 < p.Tq ? 2 : 1;  // warpgroups with at least one query row < Tq
    const int nkb_all = (p.Tk + 63) / 64;
    const int nkb = p.causal ? min(nkb_all, 2 * mt + n_cons) : nkb_all;  // key blocks this CTA streams
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 4 * n_cons);  // one arrival per consumer warp
        }
        mbar_init(bar_q, 1);
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ---- producer: Q once, then the K / V blocks through the ring ----
        if (lane == 0) {
            tma_prefetch_desc(&tmQ);
            tma_prefetch_desc(&tmK);
            tma_prefetch_desc(&tmV);
            mbar_expect_tx(bar_q, static_cast<uint32_t>(n_cons) * C::BOX);
            for (int g = 0; g < n_cons; ++g)
                for (int c = 0; c < NB; ++c)
                    tma_load_4d(smem + C::F_Q + (g * NB + c) * TILE_BYTES, &tmQ, bar_q, c * 64, h, mt * 128 + g * 64, b);
            for (int kb = 0; kb < nkb; ++kb) {
                const int s = kb % S;
                mbar_wait(&empty[s], ((kb / S) & 1) ^ 1u);
                uint8_t* dst = smem + C::F_KV + s * 2 * C::BOX;
                mbar_expect_tx(&full[s], 2u * C::BOX);
                for (int c = 0; c < NB; ++c) {
                    tma_load_4d(dst + c * TILE_BYTES, &tmK, &full[s], c * 64, h, kb * 64, b);
                    tma_load_4d(dst + C::BOX + c * TILE_BYTES, &tmV, &full[s], c * 64, h, kb * 64, b);
                }
            }
        }
        return;
    }
    const int g = warp >> 2;
    if (g >= n_cons) return;  // (a warpgroup of padding rows only)
    const int rl = (warp & 3) * 16 + (lane >> 2);
    const int jq = (lane & 3) * 2;
    const int q0 = mt * 128 + g * 64;
    const int i0 = q0 + rl;  // this thread's query rows: i0 and i0 + 8
    const int diag = q0 / 64;  // the key block on the diagonal of this warpgroup's queries
    const int nkb_g = p.causal ? min(nkb, diag + 1) : nkb;
    const float sl2 = p.scale * kLog2e;
    const uint32_t q_base = smem_u32(smem + C::F_Q) + g * C::BOX;

    float o[NB][32];
#pragma unroll
    for (int c = 0; c < NB; ++c)
#pragma unroll
        for (int e = 0; e < 32; ++e) o[c][e] = 0.f;
    // running row max (raw scores) and this thread's share of the row sum; every row has a valid key in block 0, so m is
    // finite from the first block on
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    mbar_wait(bar_q, 0);
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % S;
        mbar_wait(&full[s], (kb / S) & 1);
        if (kb < nkb_g) {
            const uint32_t k_base = smem_u32(smem + C::F_KV + s * 2 * C::BOX);
            float sc[32];
            wgmma_fence();
            mma_rows_kk<KS>(sc, q_base, k_base);
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(sc);
            if (kb * 64 + 64 > p.Tk || (p.causal && kb == diag)) {
                // keys >= Tk were zero-filled by TMA and score 0, not -inf; causal: keys after the query
#pragma unroll
                for (int e = 0; e < 32; ++e) {
                    const int hr = (e >> 1) & 1;
                    const int j = kb * 64 + (e >> 2) * 8 + jq + (e & 1);
                    if (!(j < p.Tk && (!p.causal || j <= i0 + 8 * hr))) sc[e] = -INFINITY;
                }
            }
            float mn[2] = {m[0], m[1]};
#pragma unroll
            for (int e = 0; e < 32; ++e) mn[(e >> 1) & 1] = fmaxf(mn[(e >> 1) & 1], sc[e]);
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
                mn[hr] = fmaxf(mn[hr], __shfl_xor_sync(0xffffffffu, mn[hr], 1));
                mn[hr] = fmaxf(mn[hr], __shfl_xor_sync(0xffffffffu, mn[hr], 2));
            }
            const float alpha[2] = {fast_ex2((m[0] - mn[0]) * sl2), fast_ex2((m[1] - mn[1]) * sl2)};  // 0 on the first block
            const float m2[2] = {mn[0] * sl2, mn[1] * sl2};
            float rs[2] = {0.f, 0.f};
#pragma unroll
            for (int e = 0; e < 32; ++e) {
                const int hr = (e >> 1) & 1;
                const float pv = fast_ex2(fmaf(sc[e], sl2, -m2[hr]));  // exp2(-inf) = 0 for masked keys
                sc[e] = pv;
                rs[hr] += pv;
            }
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
                l[hr] = fmaf(l[hr], alpha[hr], rs[hr]);
                m[hr] = mn[hr];
            }
#pragma unroll
            for (int c = 0; c < NB; ++c)
#pragma unroll
                for (int e = 0; e < 32; ++e) o[c][e] *= alpha[(e >> 1) & 1];
            // O += P V: P from registers (bf16), V MN-major from the stage
            wgmma_fence();
#pragma unroll
            for (int st = 0; st < 4; ++st) {
                uint32_t a[4];
                a_frag(sc, st, a);
#pragma unroll
                for (int c = 0; c < NB; ++c) wgmma_m64n64k16_rs_tb(o[c], a, mnmajor_desc(k_base + C::BOX + c * TILE_BYTES + st * 2048), 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int c = 0; c < NB; ++c) reg_fence(o[c]);
        }
        if (lane == 0) mbar_arrive(&empty[s]);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        l[hr] += __shfl_xor_sync(0xffffffffu, l[hr], 1);
        l[hr] += __shfl_xor_sync(0xffffffffu, l[hr], 2);
    }
    const float inv[2] = {1.0f / l[0], 1.0f / l[1]};
    __nv_bfloat16* g0 = out + static_cast<long long>(b) * p.Tq * p.ldo + h * p.Dh;
#pragma unroll
    for (int c = 0; c < NB; ++c) {
#pragma unroll
        for (int e = 0; e < 32; ++e) o[c][e] *= inv[(e >> 1) & 1];
        store_tile<true>(o[c], 1.0f, g0 + c * 64, p.ldo, i0, p.Tq, lane, nullptr, p.Dh - c * 64);
    }
    if ((lane & 3) == 0) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int i = i0 + 8 * hr;
            if (i < p.Tq) lse_out[static_cast<long long>(bh) * p.Tq + i] = m[hr] * p.scale + logf(l[hr]);
        }
    }
}

// delta[b, h, i] = sum_d dO[b, i, h, d] O[b, i, h, d] in fp32: one (row, head) per thread, 2 Dh contiguous bytes of each
__global__ void attn_long_delta_kernel(const __nv_bfloat16* __restrict__ o_in, const __nv_bfloat16* __restrict__ do_in,
                                       float* __restrict__ delta, int B, int T, int H, int Dh, long long ldo) {
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= static_cast<long long>(B) * T * H) return;
    const int h = static_cast<int>(idx % H);
    const long long row = idx / H;
    const int b = static_cast<int>(row / T), i = static_cast<int>(row % T);
    const uint4* po = reinterpret_cast<const uint4*>(o_in + row * ldo + h * Dh);
    const uint4* pd = reinterpret_cast<const uint4*>(do_in + row * ldo + h * Dh);
    float dl = 0.f;
    for (int k = 0; k < Dh / 8; ++k) {
        const uint4 a = __ldg(po + k), gg = __ldg(pd + k);
        dl += bf16lo(a.x) * bf16lo(gg.x) + bf16hi(a.x) * bf16hi(gg.x) + bf16lo(a.y) * bf16lo(gg.y) + bf16hi(a.y) * bf16hi(gg.y) +
              bf16lo(a.z) * bf16lo(gg.z) + bf16hi(a.z) * bf16hi(gg.z) + bf16lo(a.w) * bf16lo(gg.w) + bf16hi(a.w) * bf16hi(gg.w);
    }
    delta[(static_cast<long long>(b) * H + h) * T + i] = dl;
}

// Column-sum partials: [B * H][ceil(T / 64) row tiles][dq | dk | dv][64], each slot written by exactly one warpgroup.
// Sums the 64-column partials of the 4 warps of warpgroup g (cs: [4][64], written by store_tile) in a fixed order.
__device__ __forceinline__ float wg_colsum(const float* cs, int c) { return ((cs[c] + cs[64 + c]) + cs[128 + c]) + cs[192 + c]; }

// dK / dV.  CTA = (query chunk, key tile, image, head) with the chunk fastest.  With one chunk dK / dV are stored as bf16; with
// several, chunk c writes its fp32 sums to part[dk | dv][c][B * H][Tk][Dh] and attn_long_dkdv_reduce_kernel finishes them.
template <int KS>
__global__ void __launch_bounds__(LA_THREADS, 1)
attn_long_dkdv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                      const __grid_constant__ CUtensorMap tmDO, const float* __restrict__ lse_in, const float* __restrict__ delta_in,
                      __nv_bfloat16* __restrict__ dk_out, __nv_bfloat16* __restrict__ dv_out, float* __restrict__ part,
                      float* __restrict__ csum_part, const LongParams p) {
    constexpr int NB = (KS + 3) / 4;
    using C = LongCfg<NB>;
    constexpr int S = C::K_STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::K_BAR);
    uint64_t* empty = full + S;
    uint64_t* bar_kv = empty + S;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_kt = (p.Tk + C::K_ROWS - 1) / C::K_ROWS;
    const int chunk = blockIdx.x % p.nchunk;
    const int kt = (blockIdx.x / p.nchunk) % n_kt;
    const int bh = blockIdx.x / p.nchunk / n_kt;
    const int h = bh % p.H;
    const int b = bh / p.H;
    const int n_kb = (NB == 1 && kt * 128 + 64 < p.Tk) ? 2 : 1;  // resident 64-key blocks
    const int nqb = (p.Tq + 63) / 64;
    // causal: query blocks wholly before the key tile contribute nothing
    const int qb_lo = max(chunk * p.qb_chunk, p.causal ? kt * (C::K_ROWS / 64) : 0);
    const int qb_hi = min(nqb, (chunk + 1) * p.qb_chunk);
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full[s], 1 + 32);  // the producer's expect_tx + one arrival per producer lane after its lse / delta stores
            mbar_init(&empty[s], NB == 1 ? 4 * n_kb : 8);
        }
        mbar_init(bar_kv, 1);
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ---- producer: K / V once, then Q / dO blocks (TMA) and their lse / delta rows (lanes) through the ring ----
        if (lane == 0) {
            tma_prefetch_desc(&tmQ);
            tma_prefetch_desc(&tmK);
            tma_prefetch_desc(&tmV);
            tma_prefetch_desc(&tmDO);
            mbar_expect_tx(bar_kv, 2u * n_kb * C::BOX);
            for (int g = 0; g < n_kb; ++g)
                for (int c = 0; c < NB; ++c) {
                    tma_load_4d(smem + C::K_K + (g * NB + c) * TILE_BYTES, &tmK, bar_kv, c * 64, h, kt * C::K_ROWS + g * 64, b);
                    tma_load_4d(smem + C::K_V + (g * NB + c) * TILE_BYTES, &tmV, bar_kv, c * 64, h, kt * C::K_ROWS + g * 64, b);
                }
        }
        const float* lse_bh = lse_in + static_cast<long long>(bh) * p.Tq;
        const float* delta_bh = delta_in + static_cast<long long>(bh) * p.Tq;
        for (int qb = qb_lo, it = 0; qb < qb_hi; ++qb, ++it) {
            const int s = it % S;
            mbar_wait(&empty[s], ((it / S) & 1) ^ 1u);
            if (lane == 0) {
                uint8_t* dst = smem + C::K_QD + s * 2 * C::BOX;
                mbar_expect_tx(&full[s], 2u * C::BOX);
                for (int c = 0; c < NB; ++c) {
                    tma_load_4d(dst + c * TILE_BYTES, &tmQ, &full[s], c * 64, h, qb * 64, b);
                    tma_load_4d(dst + C::BOX + c * TILE_BYTES, &tmDO, &full[s], c * 64, h, qb * 64, b);
                }
            }
            float* row = reinterpret_cast<float*>(smem + C::K_ROW + s * 512);
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int r = lane + 32 * k, i = qb * 64 + r;
                // padded query rows: lse = +inf makes P = dS = 0 (their Q / dO rows are zero-filled as well)
                row[r] = i < p.Tq ? __ldg(lse_bh + i) * kLog2e : INFINITY;
                row[64 + r] = i < p.Tq ? __ldg(delta_bh + i) : 0.f;
            }
            mbar_arrive(&full[s]);
        }
        return;
    }
    const int g = warp >> 2;
    const int wq = warp & 3;
    const int rl = wq * 16 + (lane >> 2);  // accumulator rows rl, rl + 8: keys
    const int jq = (lane & 3) * 2;         // accumulator columns 8 n + jq (+ 1): queries
    const float sl2 = p.scale * kLog2e;
    const long long n_part = static_cast<long long>(p.nchunk) * p.B * p.H * p.Tk * p.Dh;  // floats per dk / dv partial set
    const long long kv_row0 = static_cast<long long>(b) * p.Tk;

    if constexpr (NB == 1) {
        if (g >= n_kb) return;
        const int k0 = kt * 128 + g * 64;
        const int key0 = k0 + rl;
        const int diag = k0 / 64;
        const int qb_g = p.causal ? diag : 0;
        const uint32_t k_base = smem_u32(smem + C::K_K) + g * TILE_BYTES, v_base = smem_u32(smem + C::K_V) + g * TILE_BYTES;
        const bool key_edge = k0 + 64 > p.Tk;

        float dv[32], dk[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) { dv[e] = 0.f; dk[e] = 0.f; }
        mbar_wait(bar_kv, 0);
        for (int qb = qb_lo, it = 0; qb < qb_hi; ++qb, ++it) {
            const int s = it % S;
            mbar_wait(&full[s], (it / S) & 1);
            if (qb >= qb_g) {
                const uint32_t q_st = smem_u32(smem + C::K_QD + s * 2 * C::BOX), do_st = q_st + C::BOX;
                const float* row = reinterpret_cast<const float*>(smem + C::K_ROW + s * 512);
                float st[32], dpt[32];
                wgmma_fence();
                mma_rows_kk<KS>(st, k_base, q_st);    // S^T = K Q^T
                mma_rows_kk<KS>(dpt, v_base, do_st);  // dP^T = V dO^T
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(st);
                reg_fence(dpt);
                const bool edge = key_edge || (p.causal && qb == diag);
#pragma unroll
                for (int e = 0; e < 32; ++e) {
                    const int key = key0 + ((e >> 1) & 1) * 8;
                    const int ii = (e >> 2) * 8 + jq + (e & 1);
                    float pv = fast_ex2(fmaf(st[e], sl2, -row[ii]));
                    if (edge && !(key < p.Tk && (!p.causal || key <= qb * 64 + ii))) pv = 0.f;
                    st[e] = pv;
                    asm volatile("" ::: "memory");  // keeps ptxas' schedule (and register count, 164) of the Dh-64 kernel
                    dpt[e] = pv * (dpt[e] - row[64 + ii]);
                }
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    uint32_t a[4];
                    a_frag(st, k, a);
                    wgmma_m64n64k16_rs_tb(dv, a, mnmajor_desc(do_st + k * 2048), 1u);  // dV += P^T dO
                    a_frag(dpt, k, a);
                    wgmma_m64n64k16_rs_tb(dk, a, mnmajor_desc(q_st + k * 2048), 1u);   // dK += dS^T Q
                }
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(dv);
                reg_fence(dk);
            }
            if (lane == 0) mbar_arrive(&empty[s]);
        }
        if (p.nchunk > 1) {
            const long long at = ((static_cast<long long>(chunk) * p.B * p.H + bh) * p.Tk) * p.Dh;
            store_part(dk, part + at, p.Dh, key0, p.Tk, p.Dh, lane);
            store_part(dv, part + n_part + at, p.Dh, key0, p.Tk, p.Dh, lane);
            return;
        }
        float* cs = reinterpret_cast<float*>(smem + C::K_CS);
        const bool sums = csum_part != nullptr;
        const long long off = kv_row0 * p.ldkv + h * p.Dh;
        store_tile<true>(dk, p.scale, dk_out + off, p.ldkv, key0, p.Tk, lane, sums ? cs + ((0 * 2 + g) * 4 + wq) * 64 : nullptr, p.Dh);
        store_tile<true>(dv, 1.0f, dv_out + off, p.ldkv, key0, p.Tk, lane, sums ? cs + ((1 * 2 + g) * 4 + wq) * 64 : nullptr, p.Dh);
        if (sums) {
            named_bar_sync(1 + g, 128);
            const int t = threadIdx.x & 127, sec = t >> 6, c = t & 63;
            float* dst = csum_part + (static_cast<long long>(bh) * ((p.Tq + 63) / 64) + diag) * 192;
            dst[(1 + sec) * 64 + c] = wg_colsum(cs + (sec * 2 + g) * 4 * 64, c);
        }
    } else {
        // both warpgroups on keys [64 kt, 64 kt + 64): 0 -> P^T, dV;  1 -> dP^T, dS^T, dK.  P^T goes through K_PB, guarded by
        // named barriers 3 (P^T written) and 4 (P^T read, the buffer may be overwritten)
        const int key0 = kt * 64 + rl;
        const uint32_t k_base = smem_u32(smem + C::K_K), v_base = smem_u32(smem + C::K_V);
        const bool key_edge = kt * 64 + 64 > p.Tk;
        float* pb = reinterpret_cast<float*>(smem + C::K_PB) + (threadIdx.x & 127);
        float acc[NB][32];
#pragma unroll
        for (int c = 0; c < NB; ++c)
#pragma unroll
            for (int e = 0; e < 32; ++e) acc[c][e] = 0.f;
        mbar_wait(bar_kv, 0);
        for (int qb = qb_lo, it = 0; qb < qb_hi; ++qb, ++it) {
            const int s = it % S;
            mbar_wait(&full[s], (it / S) & 1);
            const uint32_t q_st = smem_u32(smem + C::K_QD + s * 2 * C::BOX), do_st = q_st + C::BOX;
            const float* row = reinterpret_cast<const float*>(smem + C::K_ROW + s * 512);
            float x[32];
            wgmma_fence();
            if (g == 0)
                mma_rows_kk<KS>(x, k_base, q_st);   // S^T = K Q^T
            else
                mma_rows_kk<KS>(x, v_base, do_st);  // dP^T = V dO^T
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(x);
            if (g == 0) {
                const bool edge = key_edge || (p.causal && qb == kt);
#pragma unroll
                for (int e = 0; e < 32; ++e) {
                    const int key = key0 + ((e >> 1) & 1) * 8;
                    const int ii = (e >> 2) * 8 + jq + (e & 1);
                    float pv = fast_ex2(fmaf(x[e], sl2, -row[ii]));
                    if (edge && !(key < p.Tk && (!p.causal || key <= qb * 64 + ii))) pv = 0.f;
                    x[e] = pv;
                }
                if (qb > qb_lo) named_bar_sync(4, 256);
#pragma unroll
                for (int e = 0; e < 32; ++e) pb[e * 128] = x[e];
                named_bar_arrive(3, 256);
            } else {
                named_bar_sync(3, 256);
#pragma unroll
                for (int e = 0; e < 32; ++e) x[e] = pb[e * 128] * (x[e] - row[64 + (e >> 2) * 8 + jq + (e & 1)]);
                if (qb + 1 < qb_hi) named_bar_arrive(4, 256);
            }
            const uint32_t b_st = g == 0 ? do_st : q_st;  // dV += P^T dO  |  dK += dS^T Q
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                uint32_t a[4];
                a_frag(x, k, a);
#pragma unroll
                for (int c = 0; c < NB; ++c) wgmma_m64n64k16_rs_tb(acc[c], a, mnmajor_desc(b_st + c * TILE_BYTES + k * 2048), 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int c = 0; c < NB; ++c) reg_fence(acc[c]);
            if (lane == 0) mbar_arrive(&empty[s]);
        }
        if (p.nchunk > 1) {
            float* dst = part + (g == 0 ? n_part : 0) + ((static_cast<long long>(chunk) * p.B * p.H + bh) * p.Tk) * p.Dh;
#pragma unroll
            for (int c = 0; c < NB; ++c) store_part(acc[c], dst + c * 64, p.Dh, key0, p.Tk, p.Dh - c * 64, lane);
            return;
        }
        __nv_bfloat16* dst = (g == 0 ? dv_out : dk_out) + kv_row0 * p.ldkv + h * p.Dh;
        const float sc = g == 0 ? 1.0f : p.scale;
#pragma unroll
        for (int c = 0; c < NB; ++c) store_tile<true>(acc[c], sc, dst + c * 64, p.ldkv, key0, p.Tk, lane, nullptr, p.Dh - c * 64);
    }
}

// dK / dV of a query-split grid: the chunk partials summed in chunk order, dK scaled, rounded to bf16 once
__global__ void attn_long_dkdv_reduce_kernel(const float* __restrict__ part, __nv_bfloat16* __restrict__ dk, __nv_bfloat16* __restrict__ dv,
                                             int B, int H, int Tk, int Dh, long long ldkv, int nchunk, float scale) {
    const long long n = static_cast<long long>(B) * H * Tk * Dh;
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= 2 * n) return;
    const int which = idx >= n ? 1 : 0;
    const long long r = idx - which * n;
    const int d = static_cast<int>(r % Dh);
    const long long key_row = r / Dh;  // (b * H + h) * Tk + key
    const int key = static_cast<int>(key_row % Tk);
    const int bh = static_cast<int>(key_row / Tk);
    const float* src = part + which * nchunk * n + r;
    float t = 0.f;
    for (int c = 0; c < nchunk; ++c) t += src[c * n];
    __nv_bfloat16* dst = which ? dv : dk;
    dst[(static_cast<long long>(bh / H) * Tk + key) * ldkv + (bh % H) * Dh + d] = __float2bfloat16_rn(which ? t : t * scale);
}

// dQ.  For Dh > 64 the dQ accumulators (32 NB fp32) plus S and dP do not fit the 168 registers per thread that 288 threads
// leave, so those instances run 256 threads without the producer warp: thread 0 issues the loads, each K / V block as soon as
// every consumer warp has released the stage it goes into.
template <int KS>
constexpr int dq_threads() { return KS <= 4 ? LA_THREADS : 256; }

template <int KS>
__global__ void __launch_bounds__(dq_threads<KS>(), 1)
attn_long_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const __grid_constant__ CUtensorMap tmDO, const float* __restrict__ lse_in, const float* __restrict__ delta_in,
                    __nv_bfloat16* __restrict__ dq_out, float* __restrict__ csum_part, const LongParams p) {
    constexpr int NB = (KS + 3) / 4;
    using C = LongCfg<NB>;
    constexpr int S = C::Q_STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::Q_BAR);
    uint64_t* empty = full + S;
    uint64_t* bar_q = empty + S;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_qt = (p.Tq + 127) / 128;
    const int qt = blockIdx.x % n_qt;
    const int bh = blockIdx.x / n_qt;
    const int h = bh % p.H;
    const int b = bh / p.H;
    const int n_cons = qt * 128 + 64 < p.Tq ? 2 : 1;
    const int nkb_all = (p.Tk + 63) / 64;
    const int nkb = p.causal ? min(nkb_all, 2 * qt + n_cons) : nkb_all;
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 4 * n_cons);
        }
        mbar_init(bar_q, 1);
        fence_mbar_init();
    }
    __syncthreads();

    auto load_kv = [&](int kb) {  // K / V block kb into stage kb % S (its empty barrier already waited on)
        const int s = kb % S;
        uint8_t* dst = smem + C::Q_KV + s * 2 * C::BOX;
        mbar_expect_tx(&full[s], 2u * C::BOX);
        for (int c = 0; c < NB; ++c) {
            tma_load_4d(dst + c * TILE_BYTES, &tmK, &full[s], c * 64, h, kb * 64, b);
            tma_load_4d(dst + C::BOX + c * TILE_BYTES, &tmV, &full[s], c * 64, h, kb * 64, b);
        }
    };
    const bool issuer = dq_threads<KS>() == LA_THREADS ? (warp == 8 && lane == 0) : threadIdx.x == 0;
    if (issuer) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmV);
        tma_prefetch_desc(&tmDO);
        mbar_expect_tx(bar_q, 2u * n_cons * C::BOX);
        for (int g = 0; g < n_cons; ++g)
            for (int c = 0; c < NB; ++c) {
                tma_load_4d(smem + C::Q_Q + (g * NB + c) * TILE_BYTES, &tmQ, bar_q, c * 64, h, qt * 128 + g * 64, b);
                tma_load_4d(smem + C::Q_DO + (g * NB + c) * TILE_BYTES, &tmDO, bar_q, c * 64, h, qt * 128 + g * 64, b);
            }
        if constexpr (dq_threads<KS>() == LA_THREADS) {  // the producer warp streams every block through the ring
            for (int kb = 0; kb < nkb; ++kb) {
                mbar_wait(&empty[kb % S], ((kb / S) & 1) ^ 1u);
                load_kv(kb);
            }
        } else {
            for (int kb = 0; kb < min(nkb, S); ++kb) load_kv(kb);  // the ring starts empty
        }
    }
    if (warp == 8) return;
    const int g = warp >> 2;
    if (g >= n_cons) return;
    const int wq = warp & 3;
    const int rl = wq * 16 + (lane >> 2);
    const int jq = (lane & 3) * 2;
    const int q0 = qt * 128 + g * 64;
    const int i0 = q0 + rl;
    const int diag = q0 / 64;
    const int nkb_g = p.causal ? min(nkb, diag + 1) : nkb;
    const float sl2 = p.scale * kLog2e;
    const uint32_t q_base = smem_u32(smem + C::Q_Q) + g * C::BOX, do_base = smem_u32(smem + C::Q_DO) + g * C::BOX;
    float l2[2], de[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const int i = i0 + 8 * hr;
        const long long at = static_cast<long long>(bh) * p.Tq + i;
        l2[hr] = i < p.Tq ? __ldg(lse_in + at) * kLog2e : INFINITY;  // padded query rows: P = dS = 0
        de[hr] = i < p.Tq ? __ldg(delta_in + at) : 0.f;
    }

    float dq[NB][32];
#pragma unroll
    for (int c = 0; c < NB; ++c)
#pragma unroll
        for (int e = 0; e < 32; ++e) dq[c][e] = 0.f;
    mbar_wait(bar_q, 0);
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % S;
        mbar_wait(&full[s], (kb / S) & 1);
        if (kb < nkb_g) {
            const uint32_t k_st = smem_u32(smem + C::Q_KV + s * 2 * C::BOX), v_st = k_st + C::BOX;
            float sc[32], dp[32];
            wgmma_fence();
            mma_rows_kk<KS>(sc, q_base, k_st);   // S = Q K^T
            mma_rows_kk<KS>(dp, do_base, v_st);  // dP = dO V^T
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(sc);
            reg_fence(dp);
            const bool edge = kb * 64 + 64 > p.Tk || (p.causal && kb == diag);
#pragma unroll
            for (int e = 0; e < 32; ++e) {
                const int hr = (e >> 1) & 1;
                const int j = kb * 64 + (e >> 2) * 8 + jq + (e & 1);
                float pv = fast_ex2(fmaf(sc[e], sl2, -l2[hr]));
                if (edge && !(j < p.Tk && (!p.causal || j <= i0 + 8 * hr))) pv = 0.f;
                dp[e] = pv * (dp[e] - de[hr]);
            }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                uint32_t a[4];
                a_frag(dp, k, a);
#pragma unroll
                for (int c = 0; c < NB; ++c) wgmma_m64n64k16_rs_tb(dq[c], a, mnmajor_desc(k_st + c * TILE_BYTES + k * 2048), 1u);  // dQ += dS K
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int c = 0; c < NB; ++c) reg_fence(dq[c]);
        }
        if (lane == 0) mbar_arrive(&empty[s]);
        if (dq_threads<KS>() != LA_THREADS && threadIdx.x == 0 && kb + S < nkb) {
            mbar_wait(&empty[s], (kb / S) & 1);
            load_kv(kb + S);
        }
    }
    float* cs = reinterpret_cast<float*>(smem + C::Q_CS);
    const bool sums = csum_part != nullptr;
    __nv_bfloat16* g0 = dq_out + static_cast<long long>(b) * p.Tq * p.ldq + h * p.Dh;
#pragma unroll
    for (int c = 0; c < NB; ++c)
        store_tile<true>(dq[c], p.scale, g0 + c * 64, p.ldq, i0, p.Tq, lane, sums && c == 0 ? cs + (g * 4 + wq) * 64 : nullptr, p.Dh - c * 64);
    if (sums) {
        named_bar_sync(1 + g, 128);
        const int t = threadIdx.x & 127;
        if (t < 64) csum_part[(static_cast<long long>(bh) * ((p.Tq + 63) / 64) + diag) * 192 + t] = wg_colsum(cs + g * 4 * 64, t);
    }
}

// dbias_part[b, sec * D + h * 64 + c] = sum over the 64-row tiles of (b, h), in tile order
__global__ void attn_long_dbias_kernel(const float* __restrict__ csum_part, float* __restrict__ dbias_part, int B, int H, int n64) {
    const int D = H * 64;
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= 3ll * B * D) return;
    const int b = static_cast<int>(idx / (3 * D));
    const int r = static_cast<int>(idx % (3 * D));
    const int sec = r / D, h = (r % D) / 64, c = r & 63;
    const float* src = csum_part + (static_cast<long long>(b) * H + h) * n64 * 192 + sec * 64 + c;
    float t = 0.f;
    for (int k = 0; k < n64; ++k) t += src[k * 192];
    dbias_part[idx] = t;
}

}  // namespace b200

using namespace b200;

// One kernel per direction on sm_90; the version switches of the C-ABI are recorded and returned (A/B timing hooks of
// other builds), they do not change the computation.
static int g_attn_fwd_version = 0;
static int g_attn_bwd_version = 0;
static int g_attn_prefetch = 0;

// packed qkv with T <= 256 (resident kernels), packed qkv with T <= 16384 (streamed kernels), separate Q / K / V (streamed)
enum AttnFamily { ATTN_RESIDENT, ATTN_LONG, ATTN_CROSS };

// One call of an attention entry point, as check_attn_args sees it.  The packed entries pass qkv as q, k and v, dqkv as dq, dk
// and dv, and the leading dims of their layout; the forward entries leave the backward's pointers null.
struct AttnCall {
    const char* entry;
    AttnFamily family;
    bool bwd;
    int B, Tq, Tk, H, Dh, causal;
    long long ldq, ldkv, ldo;
    const void *q, *k, *v, *out, *lse;
    const void *dout, *dq, *dk, *dv;  // required by the backward entries
    const void* dbias_part;           // optional
    const void* workspace;            // required by the streamed backward entries
};

// Every argument check of the attention entries, before any tensor map is encoded: a call is refused the same way with or
// without a device.
static int check_attn_args(const AttnCall& c) {
    const bool packed = c.family != ATTN_CROSS, resident = c.family == ATTN_RESIDENT;
    if (c.B <= 0 || c.H <= 0 || c.Tq <= 0 || c.Tk <= 0) return refuse(B200_ERR_ARG, c.entry, "non-positive size");
    const int max_t = resident ? 256 : LA_MAX_T;
    if (c.Tq > max_t || c.Tk > max_t) return refuse(B200_ERR_ARG, c.entry, resident ? "T must be <= 256" : "T must be <= 16384");
    if (packed && c.Dh != 64) return refuse(B200_ERR_ARG, c.entry, "head dim must be 64");
    if (c.Dh < 8 || c.Dh > LA_MAX_DH || c.Dh % 8 != 0) return refuse(B200_ERR_ARG, c.entry, "head dim must be a multiple of 8 in [8, 160]");
    if (c.causal && c.Tq != c.Tk) return refuse(B200_ERR_ARG, c.entry, "causal needs Tq == Tk");
    const long long width = static_cast<long long>(c.H) * c.Dh;
    if (c.ldq < width || c.ldkv < width || c.ldo < width) return refuse(B200_ERR_ARG, c.entry, "leading dim < H * Dh");
    if (c.ldq % 8 != 0 || c.ldkv % 8 != 0 || c.ldo % 8 != 0) return refuse(B200_ERR_ALIGN, c.entry, "leading dims must be multiples of 8");
    if (!(c.q && c.k && c.v && c.out && c.lse) || (c.bwd && !(c.dout && c.dq && c.dk && c.dv)))
        return refuse(B200_ERR_ARG, c.entry, "null pointer");
    if (c.bwd && !resident && c.workspace == nullptr) return refuse(B200_ERR_ARG, c.entry, "workspace is required");
    // TMA bases, and the backward's 16-byte reads of out / dout
    if (!aligned(16, {c.q, c.k, c.v, c.out, c.lse, c.dout, c.dq, c.dk, c.dv, c.dbias_part, c.workspace}))
        return refuse(B200_ERR_ALIGN, c.entry, "pointers must be 16-byte aligned");
    return 0;
}

// {width, T, B} over a packed [B, T, width] bf16 tensor; boxes of 64 columns x `rows` rows (128B-swizzled): rows >= T of an
// image are zero-filled
static int packed_tmap(CUtensorMap* tm, const void* base, int width, int T, int B, int rows) {
    uint64_t dims[3] = {static_cast<uint64_t>(width), static_cast<uint64_t>(T), static_cast<uint64_t>(B)};
    uint64_t strides[2] = {static_cast<uint64_t>(width) * 2, static_cast<uint64_t>(width) * 2 * static_cast<uint64_t>(T)};
    uint32_t box[3] = {64, static_cast<uint32_t>(rows), 1};
    return make_tmap(tm, base, 2, 3, dims, strides, box, 128);
}

extern "C" int b200_attention_fwd(const void* qkv_bf16, void* out_bf16, float* lse, int B, int T, int H, int Dh,
                                  float scale, int causal, cudaStream_t stream) {
    const long long ld = 64ll * H;
    int rc = check_attn_args({"attention_fwd", ATTN_RESIDENT, false, B, T, T, H, Dh, causal, 3 * ld, 3 * ld, ld, qkv_bf16, qkv_bf16,
                              qkv_bf16, out_bf16, lse});
    if (rc) return rc;
    const int D = H * 64;
    const int tp = (T + 63) / 64 * 64;
    CUtensorMap tmQ, tmKV;
    if ((rc = packed_tmap(&tmQ, qkv_bf16, 3 * D, T, B, 128)) != 0) return rc;
    if ((rc = packed_tmap(&tmKV, qkv_bf16, 3 * D, T, B, tp)) != 0) return rc;
    static bool configured[64] = {};
    if ((rc = configure_smem(attn_fwd_kernel, AF_SMEM, configured)) != 0) return rc;
    AttnParams p;
    p.B = B; p.T = T; p.H = H; p.D = D; p.tp = tp; p.scale = scale; p.causal = causal;
    const int n_mt = (T + 127) / 128;
    attn_fwd_kernel<<<B * H * n_mt, ATT_THREADS, AF_SMEM, stream>>>(tmQ, tmKV, reinterpret_cast<__nv_bfloat16*>(out_bf16), lse, p);
    return check_launch("attention_fwd");
}

extern "C" int b200_set_attention_fwd_version(int version) {
    const int old = g_attn_fwd_version;
    g_attn_fwd_version = (version == 1 || version == 2) ? version : 0;
    return old;
}

extern "C" int b200_attention_bwd(const void* qkv_bf16, const void* out_bf16, const void* dout_bf16, const float* lse,
                                  void* dqkv_bf16, int B, int T, int H, int Dh, float scale, int causal,
                                  float* dbias_part, cudaStream_t stream) {
    const long long ld = 64ll * H;
    int rc = check_attn_args({"attention_bwd", ATTN_RESIDENT, true, B, T, T, H, Dh, causal, 3 * ld, 3 * ld, ld, qkv_bf16, qkv_bf16,
                              qkv_bf16, out_bf16, lse, dout_bf16, dqkv_bf16, dqkv_bf16, dqkv_bf16, dbias_part, nullptr});
    if (rc) return rc;
    const int D = H * 64;
    const int tp = (T + 63) / 64 * 64;
    CUtensorMap tmQKV, tmDO;
    if ((rc = packed_tmap(&tmQKV, qkv_bf16, 3 * D, T, B, tp)) != 0) return rc;
    if ((rc = packed_tmap(&tmDO, dout_bf16, D, T, B, tp)) != 0) return rc;
    static bool configured[64] = {};
    if ((rc = configure_smem(attn_bwd_kernel, AB_SMEM, configured)) != 0) return rc;
    AttnParams p;
    p.B = B; p.T = T; p.H = H; p.D = D; p.tp = tp; p.scale = scale; p.causal = causal;
    attn_bwd_kernel<<<B * H, ATT_THREADS, AB_SMEM, stream>>>(tmQKV, tmDO, reinterpret_cast<const __nv_bfloat16*>(out_bf16),
                                                             reinterpret_cast<const __nv_bfloat16*>(dout_bf16), lse,
                                                             reinterpret_cast<__nv_bfloat16*>(dqkv_bf16), dbias_part, p);
    return check_launch("attention_bwd");
}

extern "C" int b200_set_attention_prefetch(int enable) {
    const int old = g_attn_prefetch;
    g_attn_prefetch = enable ? 1 : 0;
    return old;
}

extern "C" int b200_set_attention_bwd_version(int version) {
    const int old = g_attn_bwd_version;
    g_attn_bwd_version = (version >= 1 && version <= 3) ? version : 0;
    return old;
}

// ---- streamed kernels: any 1 <= Tq, Tk <= 16384, Dh <= 160 ----
// {Dh, H, T, B} over a [B, T, ld] bf16 tensor whose head h starts at column h * Dh; 64 x 64 boxes (128B-swizzled): columns
// >= Dh and rows >= T of an image are zero-filled
static int attn_long_tmap(CUtensorMap* tm, const void* base, long long ld, int Dh, int H, int T, int B) {
    uint64_t dims[4] = {static_cast<uint64_t>(Dh), static_cast<uint64_t>(H), static_cast<uint64_t>(T), static_cast<uint64_t>(B)};
    uint64_t strides[3] = {static_cast<uint64_t>(Dh) * 2, static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(ld) * 2 * static_cast<uint64_t>(T)};
    uint32_t box[4] = {64, 1, 64, 1};
    return make_tmap(tm, base, 2, 4, dims, strides, box, 128);
}

// A dK / dV CTA walks every query block of its (image, head).  When B * H * (key tiles) cannot fill the SMs -- cross-attention
// on a 77-token context -- the queries are split into chunks of whole 64-row blocks instead.  Returns the chunk count.
static int attn_long_dkdv_chunks(int B, int Tq, int Tk, int H, int Dh, int* qb_chunk) {
    const int rows = Dh <= 64 ? LongCfg<1>::K_ROWS : LongCfg<2>::K_ROWS;
    const long long ctas = static_cast<long long>(B) * H * ((Tk + rows - 1) / rows);
    const int nqb = (Tq + 63) / 64;
    const int want = static_cast<int>(min(static_cast<long long>(nqb), ctas >= LA_SMS ? 1ll : LA_SMS / ctas));
    *qb_chunk = (nqb + want - 1) / want;
    return (nqb + *qb_chunk - 1) / *qb_chunk;
}

static LongParams attn_long_params(int B, int Tq, int Tk, int H, int Dh, long long ldq, long long ldkv, long long ldo, float scale, int causal) {
    LongParams p;
    p.B = B; p.Tq = Tq; p.Tk = Tk; p.H = H; p.Dh = Dh;
    p.ldq = ldq; p.ldkv = ldkv; p.ldo = ldo; p.scale = scale; p.causal = causal;
    p.qb_chunk = (Tq + 63) / 64; p.nchunk = 1;
    return p;
}

// k16 steps of S = Q K^T / dP = dO V^T per head dim: exact up to Dh 80 (the SD UNet's 40, ViT's 64, 80), then Dh 128 and 160
static int attn_long_ksteps(int Dh) {
    const int ks = (Dh + 15) / 16;
    return ks <= 2 ? 2 : ks <= 5 ? ks : ks <= 8 ? 8 : 10;
}

template <int KS>
static int attn_long_fwd_launch(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, void* out, float* lse,
                                const LongParams& p, cudaStream_t stream) {
    constexpr int NB = (KS + 3) / 4;
    static bool configured[64] = {};
    int rc = configure_smem(attn_long_fwd_kernel<KS>, LongCfg<NB>::F_SMEM, configured);
    if (rc) return rc;
    const int n_mt = (p.Tq + 127) / 128;
    attn_long_fwd_kernel<KS><<<p.B * p.H * n_mt, LA_THREADS, LongCfg<NB>::F_SMEM, stream>>>(tmQ, tmK, tmV, reinterpret_cast<__nv_bfloat16*>(out), lse, p);
    return check_launch("attention_long_fwd");
}

template <int KS>
static int attn_long_bwd_launch(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const CUtensorMap& tmDO, const float* lse,
                                const float* delta, void* dq, void* dk, void* dv, float* part, float* csum_part, const LongParams& p,
                                cudaStream_t stream) {
    using C = LongCfg<(KS + 3) / 4>;
    static bool configured_kv[64] = {}, configured_q[64] = {};
    int rc;
    if ((rc = configure_smem(attn_long_dkdv_kernel<KS>, C::K_SMEM, configured_kv)) != 0) return rc;
    if ((rc = configure_smem(attn_long_dq_kernel<KS>, C::Q_SMEM, configured_q)) != 0) return rc;
    const int n_kt = (p.Tk + C::K_ROWS - 1) / C::K_ROWS;
    attn_long_dkdv_kernel<KS><<<p.B * p.H * n_kt * p.nchunk, LA_THREADS, C::K_SMEM, stream>>>(
        tmQ, tmK, tmV, tmDO, lse, delta, reinterpret_cast<__nv_bfloat16*>(dk), reinterpret_cast<__nv_bfloat16*>(dv), part, csum_part, p);
    if ((rc = check_launch("attention_long_bwd (dk, dv)")) != 0) return rc;
    const int n_qt = (p.Tq + 127) / 128;
    attn_long_dq_kernel<KS><<<p.B * p.H * n_qt, dq_threads<KS>(), C::Q_SMEM, stream>>>(tmQ, tmK, tmV, tmDO, lse, delta,
                                                                                reinterpret_cast<__nv_bfloat16*>(dq), csum_part, p);
    return check_launch("attention_long_bwd (dq)");
}

static int attn_long_fwd_run(const void* q, long long ldq, const void* k, const void* v, long long ldkv, void* out, long long ldo, float* lse,
                             int B, int Tq, int Tk, int H, int Dh, float scale, int causal, cudaStream_t stream) {
    CUtensorMap tmQ, tmK, tmV;
    int rc;
    if ((rc = attn_long_tmap(&tmQ, q, ldq, Dh, H, Tq, B)) != 0) return rc;
    if ((rc = attn_long_tmap(&tmK, k, ldkv, Dh, H, Tk, B)) != 0) return rc;
    if ((rc = attn_long_tmap(&tmV, v, ldkv, Dh, H, Tk, B)) != 0) return rc;
    const LongParams p = attn_long_params(B, Tq, Tk, H, Dh, ldq, ldkv, ldo, scale, causal);
    switch (attn_long_ksteps(Dh)) {
        case 2: return attn_long_fwd_launch<2>(tmQ, tmK, tmV, out, lse, p, stream);
        case 3: return attn_long_fwd_launch<3>(tmQ, tmK, tmV, out, lse, p, stream);
        case 4: return attn_long_fwd_launch<4>(tmQ, tmK, tmV, out, lse, p, stream);
        case 5: return attn_long_fwd_launch<5>(tmQ, tmK, tmV, out, lse, p, stream);
        case 8: return attn_long_fwd_launch<8>(tmQ, tmK, tmV, out, lse, p, stream);
        default: return attn_long_fwd_launch<10>(tmQ, tmK, tmV, out, lse, p, stream);
    }
}

// workspace: delta [B, H, Tq] (rounded up to 4 floats), then either the packed layout's column-sum partials (dbias_part) or,
// for a query-split dK / dV grid (split != 0 only), the fp32 partials [dk | dv][chunk][B, H, Tk, Dh]
static int attn_long_bwd_run(const void* q, long long ldq, const void* k, const void* v, long long ldkv, const void* out, long long ldo,
                             const void* dout, const float* lse, void* dq, void* dk, void* dv, int B, int Tq, int Tk, int H, int Dh, float scale,
                             int causal, float* dbias_part, float* workspace, bool split, cudaStream_t stream) {
    CUtensorMap tmQ, tmK, tmV, tmDO;
    int rc;
    if ((rc = attn_long_tmap(&tmQ, q, ldq, Dh, H, Tq, B)) != 0) return rc;
    if ((rc = attn_long_tmap(&tmK, k, ldkv, Dh, H, Tk, B)) != 0) return rc;
    if ((rc = attn_long_tmap(&tmV, v, ldkv, Dh, H, Tk, B)) != 0) return rc;
    if ((rc = attn_long_tmap(&tmDO, dout, ldo, Dh, H, Tq, B)) != 0) return rc;
    LongParams p = attn_long_params(B, Tq, Tk, H, Dh, ldq, ldkv, ldo, scale, causal);
    if (split) p.nchunk = attn_long_dkdv_chunks(B, Tq, Tk, H, Dh, &p.qb_chunk);
    float* delta = workspace;
    float* csum_part = dbias_part != nullptr ? workspace + static_cast<long long>(B) * H * Tq : nullptr;
    float* part = p.nchunk > 1 ? workspace + (static_cast<long long>(B) * H * Tq + 3) / 4 * 4 : nullptr;
    const long long rows = static_cast<long long>(B) * Tq * H;
    attn_long_delta_kernel<<<static_cast<unsigned>((rows + 255) / 256), 256, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(out), reinterpret_cast<const __nv_bfloat16*>(dout), delta, B, Tq, H, Dh, ldo);
    if ((rc = check_launch("attention_long_bwd (delta)")) != 0) return rc;
    switch (attn_long_ksteps(Dh)) {
        case 2: rc = attn_long_bwd_launch<2>(tmQ, tmK, tmV, tmDO, lse, delta, dq, dk, dv, part, csum_part, p, stream); break;
        case 3: rc = attn_long_bwd_launch<3>(tmQ, tmK, tmV, tmDO, lse, delta, dq, dk, dv, part, csum_part, p, stream); break;
        case 4: rc = attn_long_bwd_launch<4>(tmQ, tmK, tmV, tmDO, lse, delta, dq, dk, dv, part, csum_part, p, stream); break;
        case 5: rc = attn_long_bwd_launch<5>(tmQ, tmK, tmV, tmDO, lse, delta, dq, dk, dv, part, csum_part, p, stream); break;
        case 8: rc = attn_long_bwd_launch<8>(tmQ, tmK, tmV, tmDO, lse, delta, dq, dk, dv, part, csum_part, p, stream); break;
        default: rc = attn_long_bwd_launch<10>(tmQ, tmK, tmV, tmDO, lse, delta, dq, dk, dv, part, csum_part, p, stream); break;
    }
    if (rc) return rc;
    if (p.nchunk > 1) {
        const long long n = 2ll * B * H * Tk * Dh;
        attn_long_dkdv_reduce_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(
            part, reinterpret_cast<__nv_bfloat16*>(dk), reinterpret_cast<__nv_bfloat16*>(dv), B, H, Tk, Dh, ldkv, p.nchunk, scale);
        if ((rc = check_launch("attention_long_bwd (dk, dv reduce)")) != 0) return rc;
    }
    if (dbias_part != nullptr) {
        const long long n = 3ll * B * H * 64;
        attn_long_dbias_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(csum_part, dbias_part, B, H, (Tq + 63) / 64);
        if ((rc = check_launch("attention_long_bwd (dbias)")) != 0) return rc;
    }
    return 0;
}

extern "C" int b200_attention_long_fwd(const void* qkv_bf16, void* out_bf16, float* lse, int B, int T, int H, int Dh,
                                       float scale, int causal, cudaStream_t stream) {
    const long long D = 64ll * H;
    if (const int rc = check_attn_args({"attention_long_fwd", ATTN_LONG, false, B, T, T, H, Dh, causal, 3 * D, 3 * D, D, qkv_bf16, qkv_bf16,
                                        qkv_bf16, out_bf16, lse}))
        return rc;
    const __nv_bfloat16* qkv = reinterpret_cast<const __nv_bfloat16*>(qkv_bf16);
    return attn_long_fwd_run(qkv, 3 * D, qkv + D, qkv + 2 * D, 3 * D, out_bf16, D, lse, B, T, T, H, 64, scale, causal, stream);
}

extern "C" long long b200_attention_long_bwd_workspace_floats(int B, int T, int H) {
    if (B <= 0 || T <= 0 || H <= 0) return 0;
    // delta [B, H, T] + column-sum partials [B, H, ceil(T / 64)][3][64]
    return static_cast<long long>(B) * H * (static_cast<long long>(T) + (T + 63) / 64 * 192ll);
}

extern "C" int b200_attention_long_bwd(const void* qkv_bf16, const void* out_bf16, const void* dout_bf16, const float* lse,
                                       void* dqkv_bf16, int B, int T, int H, int Dh, float scale, int causal,
                                       float* dbias_part, float* workspace, cudaStream_t stream) {
    const long long D = 64ll * H;
    if (const int rc = check_attn_args({"attention_long_bwd", ATTN_LONG, true, B, T, T, H, Dh, causal, 3 * D, 3 * D, D, qkv_bf16, qkv_bf16,
                                        qkv_bf16, out_bf16, lse, dout_bf16, dqkv_bf16, dqkv_bf16, dqkv_bf16, dbias_part, workspace}))
        return rc;
    const __nv_bfloat16* qkv = reinterpret_cast<const __nv_bfloat16*>(qkv_bf16);
    __nv_bfloat16* dqkv = reinterpret_cast<__nv_bfloat16*>(dqkv_bf16);
    return attn_long_bwd_run(qkv, 3 * D, qkv + D, qkv + 2 * D, 3 * D, out_bf16, D, dout_bf16, lse, dqkv, dqkv + D, dqkv + 2 * D, B, T, T, H, 64,
                             scale, causal, dbias_part, workspace, false, stream);
}

// ---- separate Q / K / V (cross-attention, head dims 8 ... 160) on the same streamed kernels ----
extern "C" int b200_cross_attention_fwd(const void* q, long long ldq, const void* k, const void* v, long long ldkv, void* out, long long ldo,
                                        float* lse, int B, int Tq, int Tk, int H, int Dh, float scale, int causal, cudaStream_t stream) {
    if (const int rc = check_attn_args({"cross_attention_fwd", ATTN_CROSS, false, B, Tq, Tk, H, Dh, causal, ldq, ldkv, ldo, q, k, v, out, lse}))
        return rc;
    return attn_long_fwd_run(q, ldq, k, v, ldkv, out, ldo, lse, B, Tq, Tk, H, Dh, scale, causal, stream);
}

extern "C" long long b200_cross_attention_bwd_workspace_floats(int B, int Tq, int Tk, int H, int Dh) {
    if (B <= 0 || Tq <= 0 || Tk <= 0 || H <= 0 || Dh <= 0) return 0;
    int qb_chunk;
    const int nchunk = attn_long_dkdv_chunks(B, Tq, Tk, H, Dh, &qb_chunk);
    // delta [B, H, Tq] rounded up to 4 floats, then the fp32 dk | dv partials of a query-split grid
    const long long delta = (static_cast<long long>(B) * H * Tq + 3) / 4 * 4;
    return delta + (nchunk > 1 ? 2ll * nchunk * B * H * Tk * Dh : 0ll);
}

extern "C" int b200_cross_attention_bwd(const void* q, long long ldq, const void* k, const void* v, long long ldkv, const void* out,
                                        long long ldo, const void* dout, const float* lse, void* dq, void* dk, void* dv, int B, int Tq, int Tk,
                                        int H, int Dh, float scale, int causal, float* workspace, cudaStream_t stream) {
    if (const int rc = check_attn_args({"cross_attention_bwd", ATTN_CROSS, true, B, Tq, Tk, H, Dh, causal, ldq, ldkv, ldo, q, k, v, out, lse,
                                        dout, dq, dk, dv, nullptr, workspace}))
        return rc;
    return attn_long_bwd_run(q, ldq, k, v, ldkv, out, ldo, dout, lse, dq, dk, dv, B, Tq, Tk, H, Dh, scale, causal, nullptr, workspace, true,
                             stream);
}
