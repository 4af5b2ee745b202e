// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,N] = A[M,K] * B[N,K]^T  (fp32 accumulate in registers)
//
//   warpgroups 0, 1 : MMA.  Warpgroup c owns rows [64 c, 64 c + 64) of the 128 x 256 tile: wgmma m64n256k16 straight
//                     from the smem ring (one k-block = 4 instructions); the accumulator (128 fp32 per thread) stays in
//                     registers.
//   TMA producer    : one thread; cp.async.bulk.tensor -> 128B-swizzled smem ring of STAGES x (A 16 KB + B 32 KB).
//
// Fused epilogues (every variant but the split-K partials) run on their own warpgroup, overlapped with the next tile's
// MMAs: at the end of a tile the MMA warpgroups write t = bf16(acc + bias) -- the first thing every such variant computes --
// into a 64 KB staging tile in shared memory and go straight on to the next tile's k-loop; the epilogue warpgroup reads
// t back row by row and does the rest (GELU / dual output, fp32 or bf16 residual, dGELU on h, GEGLU / dGEGLU, M / N edges)
// with 16-byte global accesses.  Roles (384 threads):
//   warps 0-7   the two MMA warpgroups
//   warp 8      the TMA producer (lane 0)
//   warps 9-11  the epilogue
// ptxas compiles the whole kernel under one register cap (launch bounds: 65536 / 384 -> 168), which the 128-register
// accumulator plus the wgmma operands need; setmaxnreg cannot raise it, so a 512-thread layout (cap 128) with a full
// fourth warpgroup does not compile, and at 384 threads every role already fits in the 64K register file.
// Shared memory: 3 stages (144 KB) + staging (64 KB) + barriers.  The split-K partial variant (wgrad: K per unit is in
// the thousands, its epilogue a small share) keeps the epilogue in the MMA warpgroups, 4 stages and 288 threads.
//
// One wgmma group stays in flight: the stage of k-block i is handed back to the producer once the MMAs of k-block i + 1
// have been issued and those of k-block i have retired.  Both operands may be K-major (row-major [rows, K]) or MN-major
// (row-major [K, rows]); the latter is what the backward GEMMs need (dgrad reads W[N,K] with the reduction over N, wgrad
// reads dY and X with the reduction over tokens) -- wgmma reads either layout through its transpose bits, so no
// transposed copies are ever materialised.  The majors are template parameters: a runtime choice inside the k-loop
// makes ptxas fence the accumulator around every branch.
//
// This one kernel serves every dense layer on the hot path of the reference's transformer block
// (SURVEY.md section 2b, K1/K4/K8/K10/K11/K12/K14):
//   F.linear call sites  cflearn/modules/core/customs.py:85-89, attentions.py:214,277, channel_mixers.py:29-33
//   conv-as-GEMM         cflearn/modules/core/convs/basic.py:155-174 (patch embed, k = s = 16)
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#include <array>
#include <utility>

#include "b200_internal.h"
#include "../../include/b200_cflearn_ext.h"
#include "ptx.cuh"

namespace b200 {

constexpr int BM = 128;
constexpr int BN = 256;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int B_STAGE_BYTES = BN * BK * 2;  // 32 KB
constexpr int MN_BOX_BYTES = 64 * BK * 2;   // one MN-major TMA box: 64 (MN) x 64 (K) bf16 = 8 KB
constexpr int STAGING_ROW_BYTES = BN * 2;   // one bf16 row of the staging tile
constexpr int STAGING_BYTES = BM * STAGING_ROW_BYTES;  // 64 KB

// What each public epilogue of include/b200_cflearn.h is, in one place: the kernel, the argument check and the launcher table
// read these fields instead of listing epilogues.  The arithmetic of an epilogue is its branch of epi_chunk / epi_geglu.
enum EpiBias : int { BIAS_OPTIONAL, BIAS_PAIR, BIAS_IGNORED, BIAS_REFUSED };
enum EpiAux : int { AUX_NONE, AUX_ROWS_BF16, AUX_ROWS_F32, AUX_IMAGE_BF16, AUX_HG_BF16 };
enum EpiCols : int { COLS_N, COLS_F, COLS_F_PAIRED };
enum : int { ENTRY_GEMM = 1, ENTRY_CONV3X3 = 2 };
enum : int { MAJORS_00 = 1, MAJORS_01 = 2, MAJORS_11 = 8, MAJORS_ALL = 15 };

struct EpiTraits {
    int kernel;    // EPI of the kernel that runs it
    bool quick;    // QuickGELU x * sigmoid(1.702 x) instead of the exact erf GELU
    bool partial;  // split-K fp32 partials: no staging tile, the epilogue in the MMA warpgroups (288 threads, 4 stages)
    bool out_f32;  // out0 is fp32, else bf16
    int bias;      // OPTIONAL bf16 [N] or NULL; PAIR required [2F], 4-byte aligned, read as (h, gate) pairs; IGNORED; REFUSED: must be NULL
    int aux;       // ROWS [M, ldo]; IMAGE bf16 [B, ldo], one row per image of the convolution; HG hg [M, ldo], h at c, the gate at F + c
    bool out1;     // required: bf16 at ldo (GELU) or dense [M, F] (GEGLU)
    int cols;      // N: the GEMM is N wide; F: N = 2F and the GEMM is F wide; F_PAIRED: N = 2F and a 256-column tile is 128 h
                   // columns and their 128 gate columns (B behind a 3-D map)
    int majors;    // (TA, TB) pairs compiled: bit 2 TA + TB
    int entries;   // the entry points that accept it
};

// Indexed by the public enum value.  Operand majors: (0,0) forward and conv, (0,1) dgrad, (1,1) wgrad, conv wgrad and CLIP's
// db; the plain bias epilogue takes all four (ops.gemm's general form).
constexpr EpiTraits kEpi[] = {
    // kernel                     quick  partial f32    bias           aux             out1   cols           majors      entries
    {EPI_BIAS_BF16,               false, false,  false, BIAS_OPTIONAL, AUX_NONE,       false, COLS_N,        MAJORS_ALL, ENTRY_GEMM | ENTRY_CONV3X3},
    {EPI_BIAS_GELU_BF16,          false, false,  false, BIAS_OPTIONAL, AUX_NONE,       true,  COLS_N,        MAJORS_00,  ENTRY_GEMM},
    {EPI_BIAS_RESID_F32,          false, false,  true,  BIAS_OPTIONAL, AUX_ROWS_F32,   false, COLS_N,        MAJORS_00,  ENTRY_GEMM | ENTRY_CONV3X3},
    {EPI_DGELU_BF16,              false, false,  false, BIAS_IGNORED,  AUX_ROWS_BF16,  false, COLS_N,        MAJORS_01,  ENTRY_GEMM},
    {EPI_PARTIAL_F32,             false, true,   true,  BIAS_IGNORED,  AUX_NONE,       false, COLS_N,        MAJORS_11,  ENTRY_GEMM},
    {EPI_BIAS_GELU_BF16,          true,  false,  false, BIAS_OPTIONAL, AUX_NONE,       true,  COLS_N,        MAJORS_00,  ENTRY_GEMM},
    {EPI_DGELU_BF16,              true,  false,  false, BIAS_IGNORED,  AUX_ROWS_BF16,  false, COLS_N,        MAJORS_01,  ENTRY_GEMM},
    {EPI_BIAS_GEGLU_BF16,         false, false,  false, BIAS_PAIR,     AUX_NONE,       true,  COLS_F_PAIRED, MAJORS_00,  ENTRY_GEMM},
    {EPI_DGEGLU_BF16,             false, false,  false, BIAS_REFUSED,  AUX_HG_BF16,    false, COLS_F,        MAJORS_01,  ENTRY_GEMM},
    {EPI_BIAS_RESID_BF16,         false, false,  false, BIAS_OPTIONAL, AUX_ROWS_BF16,  false, COLS_N,        MAJORS_00,  ENTRY_GEMM},
    {EPI_BIAS_ADD_PER_IMAGE_BF16, false, false,  false, BIAS_OPTIONAL, AUX_IMAGE_BF16, false, COLS_N,        MAJORS_00,  ENTRY_CONV3X3},
    {EPI_BIAS_RESID_CLAMP_BF16,   false, false,  false, BIAS_OPTIONAL, AUX_ROWS_BF16,  false, COLS_N,        MAJORS_00,  ENTRY_CONV3X3},
};
constexpr int kNumEpi = sizeof(kEpi) / sizeof(kEpi[0]);
static_assert(kNumEpi == B200_EPI_BIAS_RESID_CLAMP_BF16 + 1, "one kEpi row per public epilogue");

// Kernel layout by epilogue: OVERLAP = separate epilogue warpgroup (everything but the split-K partials).
template <int EPI>
struct GemmCfg {
    static constexpr bool OVERLAP = !kEpi[EPI].partial;
    static constexpr int STAGES = OVERLAP ? 3 : 4;
    static constexpr int THREADS = OVERLAP ? 384 : 288;
    static constexpr int EPI_WARPS = 3;  // warps 9-11
    static constexpr int B_OFF = STAGES * A_STAGE_BYTES;
    static constexpr int STAGING_OFF = B_OFF + STAGES * B_STAGE_BYTES;
    static constexpr int BAR_OFF = STAGING_OFF + (OVERLAP ? STAGING_BYTES : 0);
    static constexpr int SMEM_BYTES = BAR_OFF + 128 + 1024;  // + the manual 1 KB alignment of the base
    static_assert(SMEM_BYTES <= 232448, "GEMM shared-memory layout does not fit the 227 KB of an H100 SM");
};

struct GemmParams {
    int M, N, K;
    int num_m_tiles, num_n_tiles, splits, num_kb;
    const __nv_bfloat16* bias;  // [N] bf16 or nullptr
    void* out0;                 // epilogue outputs / aux operand: plain pointers, leading dimension ldo (elements)
    void* out1;
    const void* aux;
    long long ldo;
    // 3x3 convolution as implicit GEMM (conv != 0): A is a channels-last activation [B, H, W, Cin] behind a 4-D tensor map;
    // an M tile is 128 consecutive pixels (whole image rows), k-block kb = (tap, 64-channel block), and the A tile of a tap is
    // the SAME box shifted by (kx - 1, ky - 1) -- TMA zero-fills what falls outside the image: the padding costs nothing
    int conv, conv_h, conv_w, conv_cin;
    // The tap-to-box mapping and the output addressing of the convolution, by kind (CONV_*).  Its GEMM rows are one grid, or four
    // parity classes of [B, conv_h, conv_w] pixels, class c at rows [c class_stride, c class_stride + class_rows) (class_stride:
    // class_rows rounded up to whole tiles).  k-block (tap j, 64 channels) of class c loads the activation box at (x, y conv_ys)
    // shifted by conv_tap(); a parity class writes grid pixel (b, m, n) of class c = (py, px) to output pixel (b, 2m + py, 2n + px)
    // of a 2 conv_h x 2 conv_w image.  (Three ints: a larger parameter block costs the plain GEMMs' staging loop its unrolling.)
    int conv_kind, class_rows, class_stride;
};

// CONV_S1 / CONV_S2: the nine taps of a 3x3 / padding 1 convolution at stride 1 / 2 (the activation map is then 2 conv_h x
// 2 conv_w with element strides 2); CONV_UP2: the nearest-2x upsampling convolution, four classes of nine taps;
// CONV_S2_DGRAD: the stride-2 input gradient, four classes of 1, 2, 2, 4 taps.
enum : int { CONV_S1 = 1, CONV_S2 = 2, CONV_UP2 = 3, CONV_S2_DGRAD = 4 };

__host__ __device__ __forceinline__ int conv_classes(int kind) { return kind >= CONV_UP2 ? 4 : 1; }
__host__ __device__ __forceinline__ int conv_ys(int kind) { return kind == CONV_S2 ? 2 : 1; }
// taps of class c, and the taps of the classes before it (the class's first B column in taps)
__host__ __device__ __forceinline__ int conv_class_taps(int kind, int c) {
    return kind == CONV_S2_DGRAD ? ((c >> 1) + 1) * ((c & 1) + 1) : 9;
}
__host__ __device__ __forceinline__ int conv_class_tap0(int kind, int c) { return kind == CONV_S2_DGRAD ? 2 * c - (c > 0) : 0; }

// box offset (dx, dy) of tap j of class c
__device__ __forceinline__ void conv_tap(int kind, int c, int j, int& dx, int& dy) {
    const int py = c >> 1, px = c & 1;
    if (kind == CONV_UP2) {  // upsampled row 2m + py + ky - 1 is x row m + floor((py + ky - 1) / 2); columns alike
        dy = (py + j / 3 + 1) / 2 - 1;
        dx = (px + j % 3 + 1) / 2 - 1;
    } else if (kind == CONV_S2_DGRAD) {
        // dx row 2m + py takes ky = 1 from dy row m (py = 0), or ky = 0 from row m + 1 and ky = 2 from row m (py = 1); columns
        // alike.  Taps in row-major (ky, kx) order.
        const int nx = px + 1, jy = j / nx, jx = j - jy * nx;
        dy = py && jy == 0 ? 1 : 0;
        dx = px && jx == 0 ? 1 : 0;
    } else {
        dy = j / 3 - 1;
        dx = j % 3 - 1;
    }
}

// Output row of GEMM row `row`: itself, or its pixel of the 2x-sized image under a parity-class scatter.
__device__ __forceinline__ long long conv_out_row(const GemmParams& p, int row) {
    if (conv_classes(p.conv_kind) == 1) return row;
    const int c = row / p.class_stride, q = row - c * p.class_stride;
    const int n = q % p.conv_w, t = q / p.conv_w, m = t % p.conv_h, b = t / p.conv_h;
    return (static_cast<long long>(b) * 2 * p.conv_h + 2 * m + (c >> 1)) * (2 * p.conv_w) + 2 * n + (c & 1);
}

// Rows of m tile m_t the epilogue writes (a parity class ends inside its last tile).
__device__ __forceinline__ int tile_rows(const GemmParams& p, int m_t) {
    const int m0 = m_t * BM;
    if (conv_classes(p.conv_kind) == 1) return min(BM, p.M - m0);
    return min(BM, p.class_rows - (m0 - (m0 / p.class_stride) * p.class_stride));
}

// Work unit u -> (m tile, n tile, split, k-block range).  Consecutive units share the m tile (A stays in L2).
template <bool CONV>
__device__ __forceinline__ void decode_unit(const GemmParams& p, int u, int& m_t, int& n_t, int& sp, int& kb0, int& kb1) {
    n_t = u % p.num_n_tiles;
    int r = u / p.num_n_tiles;
    sp = r % p.splits;
    m_t = r / p.splits;
    kb0 = static_cast<int>((static_cast<long long>(p.num_kb) * sp) / p.splits);
    kb1 = static_cast<int>((static_cast<long long>(p.num_kb) * (sp + 1)) / p.splits);
    if constexpr (CONV) {
        if (conv_classes(p.conv_kind) > 1) kb1 = conv_class_taps(p.conv_kind, (m_t * BM) / p.class_stride) * (p.conv_cin / BK);  // (one split)
    }
}

// one k-block (BK = 64 = four k16 steps) of this warpgroup's 64 x 256 accumulator; scale_d = 0 on a unit's first k-block
// starts the accumulator from zero (no register zeroing between the wgmma groups)
template <int TA, int TB>
__device__ __forceinline__ void mma_kblock(float (&acc)[128], uint32_t a_base, uint32_t b_base, uint32_t scale_d) {
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) {
        const uint64_t ad = TA ? make_smem_desc(a_base + kk * 2048, MN_BOX_BYTES, 1024, kSwz128) : make_smem_desc(a_base + kk * 32, 16, 1024, kSwz128);
        const uint64_t bd = TB ? make_smem_desc(b_base + kk * 2048, MN_BOX_BYTES, 1024, kSwz128) : make_smem_desc(b_base + kk * 32, 16, 1024, kSwz128);
        const uint32_t sd = kk == 0 ? scale_d : 1u;
        if constexpr (TA == 0 && TB == 0) wgmma_m64n256k16_ss_t00(acc, ad, bd, sd);
        if constexpr (TA == 0 && TB == 1) wgmma_m64n256k16_ss_t01(acc, ad, bd, sd);
        if constexpr (TA == 1 && TB == 0) wgmma_m64n256k16_ss_t10(acc, ad, bd, sd);
        if constexpr (TA == 1 && TB == 1) wgmma_m64n256k16_ss_t11(acc, ad, bd, sd);
    }
}

// split-K partial of two horizontally adjacent accumulator elements (row, col), (row, col + 1).  ok0 / ok1: inside [M, N].
__device__ __forceinline__ void store_partial_pair(const GemmParams& p, int sp, int row, int col, float v0, float v1, bool ok0, bool ok1) {
    float* dst = reinterpret_cast<float*>(p.out0) + (static_cast<long long>(sp) * p.M + row) * p.ldo + col;
    if (ok1) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
    else if (ok0) dst[0] = v0;
}

// Fused epilogue of 8 consecutive elements (row, col .. col + 7) of one output row; t = bf16(acc + bias) as 4 bf16 pairs.
// n_ok: how many of the 8 columns are inside N (8 on every interior chunk).  Element for element the same arithmetic as
// the per-pair epilogue it replaces, so results are bit-identical.  h8 (dGELU / dQuickGELU only): the chunk's h when n_ok == 8,
// loaded by the caller rows ahead (see the epilogue loop).
template <int EPI, bool QUICK, bool CONV>
__device__ __forceinline__ void epi_chunk(const GemmParams& p, int row, int col, const uint32_t (&t)[4], int n_ok, const uint4& h8) {
    const long long off = (CONV ? conv_out_row(p, row) : row) * p.ldo + col;
    uint32_t o[4];  // the bf16 output (out0) of the bf16 variants
    if constexpr (EPI == EPI_BIAS_BF16) {
#pragma unroll
        for (int i = 0; i < 4; ++i) o[i] = t[i];
    } else if constexpr (EPI == EPI_BIAS_GELU_BF16) {
        // out0 = h (rounded pre-activation), out1 = bf16(gelu(h)): GELU sees the ROUNDED h, like eager
        uint32_t g[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float g0, g1;
            if constexpr (!QUICK) {
                gelu_erf2(bf16lo(t[i]), bf16hi(t[i]), g0, g1);
            } else {
                g0 = quick_gelu_bf16(bf16lo(t[i]));
                g1 = quick_gelu_bf16(bf16hi(t[i]));
            }
            g[i] = pack_bf16x2(g0, g1);
            o[i] = t[i];
        }
        __nv_bfloat16* d1 = reinterpret_cast<__nv_bfloat16*>(p.out1) + off;
        if (n_ok == 8) {
            *reinterpret_cast<uint4*>(d1) = make_uint4(g[0], g[1], g[2], g[3]);
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (e < n_ok) d1[e] = __ushort_as_bfloat16(static_cast<unsigned short>(g[e >> 1] >> (16 * (e & 1))));
        }
    } else if constexpr (EPI == EPI_BIAS_RESID_F32) {
        // out0(fp32) = aux(fp32) + float(bf16(acc + bias))     (aux may alias out0)
        const float* src = reinterpret_cast<const float*>(p.aux) + off;
        float* dst = reinterpret_cast<float*>(p.out0) + off;
        if (n_ok == 8) {
            float4 a = reinterpret_cast<const float4*>(src)[0];
            float4 b = reinterpret_cast<const float4*>(src)[1];
            a.x += bf16lo(t[0]); a.y += bf16hi(t[0]); a.z += bf16lo(t[1]); a.w += bf16hi(t[1]);
            b.x += bf16lo(t[2]); b.y += bf16hi(t[2]); b.z += bf16lo(t[3]); b.w += bf16hi(t[3]);
            reinterpret_cast<float4*>(dst)[0] = a;
            reinterpret_cast<float4*>(dst)[1] = b;
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (e < n_ok) dst[e] = src[e] + ((e & 1) ? bf16hi(t[e >> 1]) : bf16lo(t[e >> 1]));
        }
    } else if constexpr (EPI == EPI_BIAS_RESID_BF16 || EPI == EPI_BIAS_ADD_PER_IMAGE_BF16 || EPI == EPI_BIAS_RESID_CLAMP_BF16) {
        // out0(bf16) = bf16(float(bf16(acc + bias)) + float(aux(bf16)))     (aux may alias out0)
        // per image: aux is a [B, ldo] table, one row per image of the convolution (a 128-row tile may hold two images)
        const int grid_row = CONV && conv_classes(p.conv_kind) > 1 ? row % p.class_stride : row;
        const long long aux_off = EPI == EPI_BIAS_ADD_PER_IMAGE_BF16 ? static_cast<long long>(grid_row / (p.conv_h * p.conv_w)) * p.ldo + col : off;
        const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(p.aux) + aux_off;
        uint32_t rw[4] = {0u, 0u, 0u, 0u};
        if (n_ok == 8) {
            const uint4 r = *reinterpret_cast<const uint4*>(src);
            rw[0] = r.x; rw[1] = r.y; rw[2] = r.z; rw[3] = r.w;
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (e < n_ok) rw[e >> 1] |= static_cast<uint32_t>(__bfloat16_as_ushort(src[e])) << (16 * (e & 1));
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) o[i] = pack_bf16x2(bf16lo(t[i]) + bf16lo(rw[i]), bf16hi(t[i]) + bf16hi(rw[i]));
        if constexpr (EPI == EPI_BIAS_RESID_CLAMP_BF16) {
            // torch.clamp to bf16's finite range on the rounded sum: +-inf (0x7f80 / 0xff80) -> +-max (0x7f7f / 0xff7f), NaN kept
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if ((o[i] & 0x7fffu) == 0x7f80u) o[i] = (o[i] & 0xffff8000u) | 0x7f7fu;
                if ((o[i] & 0x7fff0000u) == 0x7f800000u) o[i] = (o[i] & 0x8000ffffu) | 0x7f7f0000u;
            }
        }
    } else if constexpr (EPI == EPI_DGEGLU_BF16) {
        // t = bf16(da) at columns col.. of F; aux = hg [M, 2F]: h at col, gate at F + col.  out0 = dhg: dh at col, dgate at F + col.
        // (F % 8 == 0, so a chunk is either whole or outside: the caller only passes n_ok == 8.)
        const int F = p.N >> 1;
        const __nv_bfloat16* hg = reinterpret_cast<const __nv_bfloat16*>(p.aux) + off;
        const uint4 hv = *reinterpret_cast<const uint4*>(hg);
        const uint4 gv = *reinterpret_cast<const uint4*>(hg + F);
        const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w};
        const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w};
        uint32_t dgate[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float d0 = bf16lo(t[i]), d1 = bf16hi(t[i]);
            float g0, g1, q0, q1;
            gelu_erf2(bf16lo(gw[i]), bf16hi(gw[i]), g0, g1);
            o[i] = pack_bf16x2(d0 * bf16_round(g0), d1 * bf16_round(g1));              // dh = bf16(da * g)
            const float dg0 = bf16_round(d0 * bf16lo(hw[i])), dg1 = bf16_round(d1 * bf16hi(hw[i]));  // dg = bf16(da * h)
            gelu_erf_grad2(bf16lo(gw[i]), bf16hi(gw[i]), q0, q1);
            dgate[i] = pack_bf16x2(dg0 * q0, dg1 * q1);                                  // dgate = bf16(gelu'(gate) * dg)
        }
        *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out0) + off + F) = make_uint4(dgate[0], dgate[1], dgate[2], dgate[3]);
    } else {  // EPI_DGELU_BF16: out0 = bf16( float(bf16(acc)) * gelu'(h) ),  h = aux (bf16)
        const __nv_bfloat16* hsrc = reinterpret_cast<const __nv_bfloat16*>(p.aux) + off;
        uint32_t hw[4] = {0u, 0u, 0u, 0u};
        if (n_ok == 8) {
            hw[0] = h8.x; hw[1] = h8.y; hw[2] = h8.z; hw[3] = h8.w;
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (e < n_ok) hw[e >> 1] |= static_cast<uint32_t>(__bfloat16_as_ushort(hsrc[e])) << (16 * (e & 1));
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if constexpr (!QUICK) {
                float g0, g1;
                gelu_erf_grad2(bf16lo(hw[i]), bf16hi(hw[i]), g0, g1);
                o[i] = pack_bf16x2(bf16lo(t[i]) * g0, bf16hi(t[i]) * g1);
            } else {
                o[i] = pack_bf16x2(quick_gelu_bf16_grad(bf16lo(hw[i]), bf16lo(t[i])), quick_gelu_bf16_grad(bf16hi(hw[i]), bf16hi(t[i])));
            }
        }
    }
    if constexpr (!kEpi[EPI].out_f32) {
        __nv_bfloat16* d0 = reinterpret_cast<__nv_bfloat16*>(p.out0) + off;
        if (n_ok == 8) {
            *reinterpret_cast<uint4*>(d0) = make_uint4(o[0], o[1], o[2], o[3]);
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (e < n_ok) d0[e] = __ushort_as_bfloat16(static_cast<unsigned short>(o[e >> 1] >> (16 * (e & 1))));
        }
    }
}

// GEGLU forward of 8 consecutive columns f .. f + 7 of F: th = bf16(acc + bias) of h, tg that of the gate.  out0 = hg in the
// reference's column order (h at f, gate at F + f), out1 = a = bf16(h * bf16(gelu(gate))) (dense [M, F]).
__device__ __forceinline__ void epi_geglu(const GemmParams& p, int row, int f, const uint4& th, const uint4& tg) {
    const int F = p.N >> 1;
    const uint32_t hw[4] = {th.x, th.y, th.z, th.w};
    const uint32_t gw[4] = {tg.x, tg.y, tg.z, tg.w};
    uint32_t a[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float g0, g1;
        gelu_erf2(bf16lo(gw[i]), bf16hi(gw[i]), g0, g1);
        a[i] = pack_bf16x2(bf16lo(hw[i]) * bf16_round(g0), bf16hi(hw[i]) * bf16_round(g1));
    }
    __nv_bfloat16* d0 = reinterpret_cast<__nv_bfloat16*>(p.out0) + static_cast<long long>(row) * p.ldo + f;
    *reinterpret_cast<uint4*>(d0) = th;
    *reinterpret_cast<uint4*>(d0 + F) = tg;
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out1) + static_cast<long long>(row) * F + f) = make_uint4(a[0], a[1], a[2], a[3]);
}

// Staging tile: 128 rows x 256 bf16, 512 B per row; the 16-byte chunk c of row r sits at chunk c ^ (r & 7) of that row.
// The MMA warpgroups' 4-byte writes (8 rows x 4 lanes per chunk column) and the epilogue's 16-byte row reads (a warp reads
// one whole row) are both free of bank conflicts.
__device__ __forceinline__ uint32_t staging_offset(int r, int chunk) {
    return static_cast<uint32_t>(r) * STAGING_ROW_BYTES + (static_cast<uint32_t>(chunk ^ (r & 7)) << 4);
}

// QUICK (GELU / dGELU variants only): QuickGELU instead of the exact erf GELU.  A template parameter, not a runtime flag,
// so the other variants carry none of its registers.
// TA / TB: 1 = that operand is MN-major.
// CONV: the forward / input-gradient convolution entries (A behind the 4-D tap map, parity classes, scattered output rows); a
// separate instantiation, so the plain GEMMs carry none of its addressing.
template <int EPI, bool QUICK, int TA, int TB, bool CONV>
__global__ void __launch_bounds__(GemmCfg<EPI>::THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
    using Cfg = GemmCfg<EPI>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    // 1 KB alignment (the 128B swizzle pattern repeats every 1024 bytes) as an OFFSET from the __shared__ array
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sA = smem;
    uint8_t* sB = smem + Cfg::B_OFF;
    uint8_t* staging = smem + Cfg::STAGING_OFF;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFF);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* staging_full = empty_bar + STAGES;  // the MMA warpgroups have written a tile's t
    uint64_t* staging_empty = staging_full + 1;   // the epilogue warpgroup has read it

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int total_units = p.num_m_tiles * p.num_n_tiles * p.splits;

    if (threadIdx.x == 0) {
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 2);  // one arrival per consumer warpgroup
        }
        if constexpr (Cfg::OVERLAP) {
            mbar_init(staging_full, 256);  // every MMA thread, after its own staging writes
            mbar_init(staging_empty, 32 * Cfg::EPI_WARPS);  // every epilogue thread, after its last staging read of the tile
        }
        fence_mbar_init();
    }
    __syncthreads();

    if constexpr (Cfg::OVERLAP) {
        if (warp > 8) {
            // ===================================== epilogue warps =====================================
            uint32_t sphase = 0;
            for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
                int m_t, n_t, sp, kb0, kb1;
                decode_unit<CONV>(p, u, m_t, n_t, sp, kb0, kb1);
                const int col = n_t * BN + lane * 8;
                const int n_ok = min(8, max(0, (kEpi[EPI].cols == COLS_F ? p.N >> 1 : p.N) - col));
                const int rows = CONV ? tile_rows(p, m_t) : min(BM, p.M - m_t * BM);
                if constexpr (kEpi[EPI].aux == AUX_ROWS_BF16 || kEpi[EPI].aux == AUX_ROWS_F32) {
                    // pull the tile's aux rows into L2 while its MMAs still run: three warps cannot hide HBM latency alone.
                    // Rows are 16-byte aligned and padded to ldo >= the 16-byte-rounded width, so no byte past a row is named.
                    constexpr int eb = kEpi[EPI].aux == AUX_ROWS_F32 ? 4 : 2;
                    const int n0 = n_t * BN;
                    const uint32_t bytes = static_cast<uint32_t>((min(BN, p.N - n0) * eb + 15) & ~15);
                    const uint8_t* aux = reinterpret_cast<const uint8_t*>(p.aux);
                    for (int r = threadIdx.x - 9 * 32; r < rows; r += 32 * Cfg::EPI_WARPS)
                        bulk_prefetch_l2(aux + ((CONV ? conv_out_row(p, m_t * BM + r) : m_t * BM + r) * p.ldo + n0) * eb, bytes);
                }
                if constexpr (kEpi[EPI].aux == AUX_IMAGE_BF16) {  // the table has one row per image: prefetch the tile's images
                    const int hw = p.conv_h * p.conv_w, n0 = n_t * BN, q0 = CONV ? (m_t * BM) % p.class_stride : m_t * BM;
                    const int img0 = q0 / hw, img1 = (q0 + rows - 1) / hw;
                    const uint32_t bytes = static_cast<uint32_t>((min(BN, p.N - n0) * 2 + 15) & ~15);
                    const uint8_t* aux = reinterpret_cast<const uint8_t*>(p.aux);
                    for (int b = img0 + threadIdx.x - 9 * 32; b <= img1; b += 32 * Cfg::EPI_WARPS)
                        bulk_prefetch_l2(aux + (static_cast<long long>(b) * p.ldo + n0) * 2, bytes);
                }
                if constexpr (kEpi[EPI].aux == AUX_HG_BF16) {  // the same for both halves of hg: h at n0, the gate at F + n0
                    const int F = p.N >> 1, n0 = n_t * BN;
                    const uint32_t bytes = static_cast<uint32_t>(min(BN, F - n0) * 2);
                    const __nv_bfloat16* aux = reinterpret_cast<const __nv_bfloat16*>(p.aux);
                    for (int r = threadIdx.x - 9 * 32; r < rows; r += 32 * Cfg::EPI_WARPS) {
                        const __nv_bfloat16* src = aux + static_cast<long long>(m_t * BM + r) * p.ldo + n0;
                        bulk_prefetch_l2(src, bytes);
                        bulk_prefetch_l2(src + F, bytes);
                    }
                }
                mbar_wait(staging_full, sphase);
                if constexpr (kEpi[EPI].cols == COLS_F_PAIRED) {
                    // the tile's 256 columns are 128 h columns and the matching 128 gate columns: a half-warp takes one row,
                    // lane l & 15 the h chunk l & 15 and the gate chunk 16 + (l & 15) -- one 8-column piece of out0's two
                    // halves and of out1 each
                    const int hl = lane & 15;
                    const int f = n_t * (BN / 2) + hl * 8;
                    const bool ok = f < (p.N >> 1);
#pragma unroll 2
                    for (int r = 2 * (warp - 9) + (lane >> 4); r < rows; r += 2 * Cfg::EPI_WARPS) {
                        const uint4 th = *reinterpret_cast<const uint4*>(staging + staging_offset(r, hl));
                        const uint4 tg = *reinterpret_cast<const uint4*>(staging + staging_offset(r, 16 + hl));
                        if (ok) epi_geglu(p, m_t * BM + r, f, th, tg);
                    }
                } else if constexpr (EPI == EPI_DGELU_BF16) {
                    // as below, with the warp's h chunks loaded HQ rows ahead: the compiler cannot move a row's h load above
                    // the previous row's store (they might alias), so loading it in place waits one L2 round trip per row
                    constexpr int HQ = 4;
                    const __nv_bfloat16* hrows = reinterpret_cast<const __nv_bfloat16*>(p.aux) + static_cast<long long>(m_t * BM) * p.ldo + col;
                    const int r0 = warp - 9;
                    uint4 hq[HQ] = {};
#pragma unroll
                    for (int i = 0; i < HQ; ++i) {
                        const int r = r0 + i * Cfg::EPI_WARPS;
                        if (n_ok == 8 && r < rows) hq[i] = *reinterpret_cast<const uint4*>(hrows + static_cast<long long>(r) * p.ldo);
                    }
                    for (int rb = r0; rb < rows; rb += HQ * Cfg::EPI_WARPS) {
#pragma unroll
                        for (int i = 0; i < HQ; ++i) {
                            const int r = rb + i * Cfg::EPI_WARPS;
                            if (r < rows) {
                                const uint4 h8 = hq[i];
                                const int rn = r + HQ * Cfg::EPI_WARPS;
                                if (n_ok == 8 && rn < rows) hq[i] = *reinterpret_cast<const uint4*>(hrows + static_cast<long long>(rn) * p.ldo);
                                const uint4 v = *reinterpret_cast<const uint4*>(staging + staging_offset(r, lane));
                                const uint32_t t[4] = {v.x, v.y, v.z, v.w};
                                if (n_ok > 0) epi_chunk<EPI, QUICK, CONV>(p, m_t * BM + r, col, t, n_ok, h8);
                            }
                        }
                    }
                } else {
                    // epilogue warp w takes rows w, w + 3, ...: one 512-byte row per warp access, 16 bytes per lane
#pragma unroll 4
                    for (int r = warp - 9; r < rows; r += Cfg::EPI_WARPS) {
                        const uint4 v = *reinterpret_cast<const uint4*>(staging + staging_offset(r, lane));
                        const uint32_t t[4] = {v.x, v.y, v.z, v.w};
                        if (n_ok > 0) epi_chunk<EPI, QUICK, CONV>(p, m_t * BM + r, col, t, n_ok, make_uint4(0u, 0u, 0u, 0u));
                    }
                }
                mbar_arrive(staging_empty);
                sphase ^= 1u;
            }
            return;
        }
    }

    if (warp == 8) {
        // ===================================== TMA producer =====================================
        if (lane == 0) {
            tma_prefetch_desc(&tmA);
            tma_prefetch_desc(&tmB);
            int stage = 0;
            uint32_t phase = 0;
            for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
                int m_t, n_t, sp, kb0, kb1;
                decode_unit<CONV>(p, u, m_t, n_t, sp, kb0, kb1);
                const int m0 = m_t * BM, n0 = n_t * BN;
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1u);
                    uint8_t* a_dst = sA + stage * A_STAGE_BYTES;
                    uint8_t* b_dst = sB + stage * B_STAGE_BYTES;
                    mbar_expect_tx(&full_bar[stage], A_STAGE_BYTES + B_STAGE_BYTES);
                    const int cls = CONV ? m0 / p.class_stride : 0;
                    if constexpr (CONV) {
                        const int cpb = p.conv_cin / BK;
                        const int tap = kb / cpb, c0 = (kb - tap * cpb) * BK;
                        const int hw = p.conv_h * p.conv_w, q0 = m0 - cls * p.class_stride;
                        const int bimg = q0 / hw, q = q0 - bimg * hw, y0 = q / p.conv_w;
                        const int x0 = q - y0 * p.conv_w;  // 0 unless a row is wider than a tile (then a multiple of 128)
                        int dx, dy;
                        conv_tap(p.conv_kind, cls, tap, dx, dy);
                        tma_load_4d(a_dst, &tmA, &full_bar[stage], c0, x0 * conv_ys(p.conv_kind) + dx, y0 * conv_ys(p.conv_kind) + dy, bimg);
                    } else if constexpr (!TA) {
                        tma_load_2d(a_dst, &tmA, &full_bar[stage], kb * BK, m0);
                    } else {
#pragma unroll
                        for (int i = 0; i < BM / 64; ++i)
                            tma_load_2d(a_dst + i * MN_BOX_BYTES, &tmA, &full_bar[stage], m0 + i * 64, kb * BK);
                    }
                    if (p.conv == 2) {
                        // weight gradient of the 3x3 convolution: B = the activation behind a 4-D map, k-block = 64 consecutive
                        // pixels, every 64-channel box of the N tile shifted by ITS tap (n = tap * Cin + c)
                        const int hw = p.conv_h * p.conv_w, p0 = kb * BK;
                        const int bimg = p0 / hw, y0 = (p0 - bimg * hw) / p.conv_w;
#pragma unroll
                        for (int i = 0; i < BN / 64; ++i) {
                            const int n = n0 + i * 64;
                            const int tap = n / p.conv_cin, c0 = n - tap * p.conv_cin;
                            const int ky = tap / 3, kx = tap - ky * 3;
                            // (boxes past N = 9 Cin: tap >= 9 lands outside the image -> zero fill, bytes still credited)
                            tma_load_4d(b_dst + i * MN_BOX_BYTES, &tmB, &full_bar[stage], c0, kx - 1, tap < 9 ? y0 * conv_ys(p.conv_kind) + ky - 1 : -65536, bimg);
                        }
                    } else if constexpr (kEpi[EPI].cols == COLS_F_PAIRED) {
                        // W1 behind a 3-D map {K, F, 2}: one box = 128 h rows then the matching 128 gate rows (rows past F
                        // zero-filled), so the B tile holds [h | gate] of the same 128 columns
                        tma_load_3d(b_dst, &tmB, &full_bar[stage], kb * BK, n_t * (BN / 2), 0);
                    } else if constexpr (!TB) {
                        tma_load_2d(b_dst, &tmB, &full_bar[stage], ((CONV ? conv_class_tap0(p.conv_kind, cls) * (p.conv_cin / BK) : 0) + kb) * BK, n0);
                    } else {
#pragma unroll
                        for (int i = 0; i < BN / 64; ++i)
                            tma_load_2d(b_dst + i * MN_BOX_BYTES, &tmB, &full_bar[stage], n0 + i * 64, kb * BK);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1u; }
                }
            }
        }
        return;
    }

    // ===================================== MMA warpgroups ==================================
    const int wg = warp >> 2;        // 0 / 1: which 64-row half of the tile
    const int wq = warp & 3;         // warp inside the warpgroup: 16 accumulator rows each
    const bool leader = (threadIdx.x & 127) == 0;
    // a K-major A tile is 128 rows of 128 B, an MN-major one two 8 KB boxes of 64 rows: the half starts 8 KB in either way
    const uint32_t a_half = static_cast<uint32_t>(wg) * 8192u;
    int stage = 0;
    uint32_t phase = 0, sphase = 0;
    for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
        int m_t, n_t, sp, kb0, kb1;
        decode_unit<CONV>(p, u, m_t, n_t, sp, kb0, kb1);
        float acc[128];
        int prev = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t a_base = smem_u32(sA + stage * A_STAGE_BYTES) + a_half;
            const uint32_t b_base = smem_u32(sB + stage * B_STAGE_BYTES);
            wgmma_fence();
            mma_kblock<TA, TB>(acc, a_base, b_base, kb == kb0 ? 0u : 1u);
            wgmma_commit();
            wgmma_wait<1>();  // the k-block before this one has been read completely: its stage goes back to the producer
            if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        reg_fence(acc);
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);

        const int rl = wg * 64 + wq * 16 + (lane >> 2);  // accumulator rows rl, rl + 8 of the tile
        const int colq = n_t * BN + (lane & 3) * 2;
        if constexpr (Cfg::OVERLAP) {
            // ---- handoff: t = bf16(acc + bias) into the staging tile, the rest on the epilogue warpgroup ----
            mbar_wait(staging_empty, sphase ^ 1u);
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const int col = colq + j * 8;
                float b0 = 0.f, b1 = 0.f;
                if constexpr (kEpi[EPI].bias == BIAS_PAIR) {
                    // tile column c < 128: h column n_t * 128 + c; c >= 128: gate column F + n_t * 128 + c - 128
                    // (the bias is required; f is even and F % 8 == 0, so f < F covers f + 1 too: one 4-byte load of the pair)
                    const int f = colq - n_t * (BN / 2) + (j & 15) * 8;  // colq = n_t * BN + (lane & 3) * 2
                    if (f < (p.N >> 1)) {
                        const uint32_t bp = *reinterpret_cast<const uint32_t*>(p.bias + (j < 16 ? f : f + (p.N >> 1)));
                        b0 = bf16lo(bp);
                        b1 = bf16hi(bp);
                    }
                } else if constexpr (kEpi[EPI].bias == BIAS_OPTIONAL) {
                    if (p.bias != nullptr) {
                        if (col < p.N) b0 = __bfloat162float(p.bias[col]);
                        if (col + 1 < p.N) b1 = __bfloat162float(p.bias[col + 1]);
                    }
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint32_t t = pack_bf16x2(acc[4 * j + 2 * h] + b0, acc[4 * j + 2 * h + 1] + b1);
                    *reinterpret_cast<uint32_t*>(staging + staging_offset(rl + h * 8, j) + (lane & 3) * 4) = t;
                }
            }
            mbar_arrive(staging_full);
            sphase ^= 1u;
        } else {
            // ---- split-K partials straight from the accumulator fragment ----
            const int row0 = m_t * BM + rl;
            const bool interior = (m_t * BM + BM <= p.M) && (n_t * BN + BN <= p.N);
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const int col = colq + j * 8;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = row0 + h * 8;
                    const bool rok = interior || row < p.M;
                    store_partial_pair(p, sp, row, col, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], rok && (interior || col < p.N),
                                       rok && (interior || col + 1 < p.N));
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || p == nullptr) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
    return fn;
}

// The tensor-map encode is a driver call and needs a current context.  A host thread that has not yet made a runtime call
// that binds one has none -- autograd's device thread, for example, when one of our GEMMs is the first CUDA work of a
// backward.  cudaSetDevice on the runtime's current device makes that device's primary context current; it is skipped
// whenever a context already is.
typedef CUresult (*PFN_ctxGetCurrent)(CUcontext*);

static int ensure_current_context() {
    static PFN_ctxGetCurrent get = nullptr;
    if (get == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuCtxGetCurrent", &p, cudaEnableDefault, &q);
        if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || p == nullptr)
            return set_error(B200_ERR_DRIVER, "cuCtxGetCurrent entry point unavailable");
        get = reinterpret_cast<PFN_ctxGetCurrent>(p);
    }
    CUcontext c = nullptr;
    if (get(&c) == CUDA_SUCCESS && c != nullptr) return 0;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaSetDevice(dev);
    if (e != cudaSuccess) return set_error(B200_ERR_DRIVER, cudaGetErrorString(e));
    return 0;
}

// rank-2/3 tiled map; dims/box innermost first; strides in BYTES for dims 1.. (rank-1 entries)
int make_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes, const uint32_t* elem_strides) {
    PFN_encodeTiled fn = get_encode_fn();
    if (!fn) return set_error(B200_ERR_DRIVER, "cuTensorMapEncodeTiled entry point unavailable");
    CUtensorMapDataType dt = elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    CUtensorMapSwizzle sw = swizzle_bytes == 128  ? CU_TENSOR_MAP_SWIZZLE_128B
                            : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                            : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                  : CU_TENSOR_MAP_SWIZZLE_NONE;
    cuuint64_t gdim[5];
    cuuint64_t gstr[5];
    cuuint32_t bx[5];
    cuuint32_t es[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bx[i] = box[i];
        es[i] = elem_strides != nullptr ? elem_strides[i] : 1;
    }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
    if (!aligned(16, {base})) return set_error(B200_ERR_ALIGN, "tensor base not 16 B aligned");
    for (int i = 0; i + 1 < rank; ++i)
        if (gstr[i] % 16 != 0) return set_error(B200_ERR_ALIGN, "tensor stride not a multiple of 16 B");
    if (const int rc = ensure_current_context()) return rc;
    CUresult r = fn(out, dt, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim, gstr, bx, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char msg[160];
        snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled failed: CUresult %d (rank %d dims %llu %llu box %u %u)",
                 static_cast<int>(r), rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
        return set_error(B200_ERR_DRIVER, msg);
    }
    return 0;
}

int current_device_slot() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev < 0 || dev >= 64) ? 0 : dev;
}

int num_sms() {
    static int cached[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (cached[dev] == 0) {
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        cached[dev] = n > 0 ? n : 132;
    }
    return cached[dev];
}

// Upper bound on the grid of every persistent kernel (GEMM, attention version 2), 0 = all SMs.  The data-parallel step lowers it
// by the communicator's CTA count while gradient buckets are in flight: these kernels assign their tiles to CTAs statically, and
// a CTA whose SM is held by an NCCL kernel starts only when that all-reduce is over -- with its full share of tiles still to do.
static int g_persistent_ctas = 0;
static int g_persistent_window = 0;  // > 0: the limit lapses after that many more persistent launches
int persistent_ctas() {  // (called exactly once per persistent launch)
    const int n = num_sms();
    const int r = (g_persistent_ctas > 0 && g_persistent_ctas < n) ? g_persistent_ctas : n;
    if (g_persistent_window > 0 && --g_persistent_window == 0) g_persistent_ctas = 0;
    return r;
}
extern "C" int b200_set_persistent_ctas(int n, int launches) {
    const int old = g_persistent_ctas;
    g_persistent_ctas = n > 0 ? n : 0;
    g_persistent_window = (n > 0 && launches > 0) ? launches : 0;
    return old;
}

// Kept for the C-ABI (b200_set_gemm_multicast): the sm_90 kernel runs one CTA per tile in every mode, so the setting is
// only recorded and returned.
static int g_gemm_multicast = 0;

template <int EPI, bool QUICK, int TA, int TB, bool CONV = false>
static int launch_gemm_impl(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int grid, cudaStream_t stream) {
    using Cfg = GemmCfg<EPI>;
    static bool configured[64] = {};
    if (const int rc = configure_smem(gemm_bf16_kernel<EPI, QUICK, TA, TB, CONV>, Cfg::SMEM_BYTES, configured)) return rc;
    gemm_bf16_kernel<EPI, QUICK, TA, TB, CONV><<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, p);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(B200_ERR_LAUNCH, cudaGetErrorString(e));
    count_launch(1);
    return 0;
}

typedef int (*GemmLauncher)(const CUtensorMap&, const CUtensorMap&, const GemmParams&, int, cudaStream_t);

// public epilogue P with majors (TA, TB): its kernel instance, or nullptr where kEpi[P] does not compile those majors
template <int P, int TA, int TB>
constexpr GemmLauncher launcher() {
    if constexpr (((kEpi[P].majors >> (2 * TA + TB)) & 1) != 0) return &launch_gemm_impl<kEpi[P].kernel, kEpi[P].quick, TA, TB>;
    else return nullptr;
}

template <int... P>
constexpr std::array<std::array<GemmLauncher, 4>, sizeof...(P)> launcher_table(std::integer_sequence<int, P...>) {
    return {{{launcher<P, 0, 0>(), launcher<P, 0, 1>(), launcher<P, 1, 0>(), launcher<P, 1, 1>()}...}};
}

// indexed by (public epilogue, 2 TA + TB)
static constexpr auto kLaunch = launcher_table(std::make_integer_sequence<int, kNumEpi>{});

// the convolution-forward instance of public epilogue P (operands (0, 0)), or nullptr where the convolutions do not offer it
template <int P>
constexpr GemmLauncher conv_launcher() {
    if constexpr ((kEpi[P].entries & ENTRY_CONV3X3) != 0) return &launch_gemm_impl<kEpi[P].kernel, kEpi[P].quick, 0, 0, true>;
    else return nullptr;
}

template <int... P>
constexpr std::array<GemmLauncher, sizeof...(P)> conv_launcher_table(std::integer_sequence<int, P...>) {
    return {{conv_launcher<P>()...}};
}

static constexpr auto kLaunchConv = conv_launcher_table(std::make_integer_sequence<int, kNumEpi>{});

}  // namespace b200

using namespace b200;

extern "C" int b200_set_gemm_multicast(int enable) {
    const int old = g_gemm_multicast;
    g_gemm_multicast = enable < 0 ? 0 : (enable > 2 ? 2 : enable);
    return old;
}

extern "C" int b200_gemm_pick_splits(int M, int N, int K) {
    const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
    const int num_kb = (K + BK - 1) / BK;
    const int sms = 132;  // H100 SXM
    int best = 1;
    double best_score = -1.0;
    for (int s = 1; s <= 16 && s <= num_kb; ++s) {
        const int units = tiles * s;
        const int waves = (units + sms - 1) / sms;
        double eff = static_cast<double>(units) / (static_cast<double>(waves) * sms);
        // each split costs a pipeline fill/drain (~ 8 k-blocks worth) and an extra fp32 partial
        const double kb_per = static_cast<double>(num_kb) / s;
        eff *= kb_per / (kb_per + 8.0);
        if (eff > best_score + 1e-9) {
            best_score = eff;
            best = s;
        }
    }
    return best;
}

// mode 1: forward / input gradient (A behind the 4-D map); 2: weight gradient (B).  B, H, W: the grid of the GEMM rows (mode 1) or
// of the reduction's pixels (mode 2); kind: CONV_* (the activation is 2H x 2W for CONV_S2).
struct ConvGeom { int B, H, W, Cin, mode, kind; };

// Every argument check of the GEMM entries, before any tensor map is encoded: a call is refused the same way with or without
// a device.  conv_fwd: the call comes from b200_conv3x3_nhwc_bf16.
static int check_gemm_args(const void* A, int a_mn, const void* B, int b_mn, int M, int N, int K, int epilogue, const void* bias,
                           const void* out0, const void* out1, const void* aux, long long ldo, int splits, bool conv_fwd) {
    if (epilogue < 0 || epilogue >= kNumEpi) return refuse(B200_ERR_ARG, "gemm", "unknown epilogue");
    const EpiTraits& e = kEpi[epilogue];
    if (conv_fwd && !(e.entries & ENTRY_CONV3X3)) return refuse(B200_ERR_ARG, "conv3x3", "epilogue not offered for convolutions");
    if (!conv_fwd && !(e.entries & ENTRY_GEMM)) return refuse(B200_ERR_ARG, "gemm", "epilogue offered by conv3x3 only");
    if (M <= 0 || N <= 0 || K <= 0) return refuse(B200_ERR_ARG, "gemm", "non-positive dimension");
    // N need not be a multiple of 8: the bias is read in 16-byte groups (readable up to roundup(N, 8) elements) and the
    // epilogue clips columns >= N
    if (A == nullptr || B == nullptr || out0 == nullptr) return refuse(B200_ERR_ARG, "gemm", "null pointer");
    if (!e.partial && splits != 1) return refuse(B200_ERR_ARG, "gemm", "split-K needs EPI_PARTIAL_F32");
    if (kLaunch[epilogue][2 * a_mn + b_mn] == nullptr) return refuse(B200_ERR_ARG, "gemm", "operand majors not supported by this epilogue");
    if (e.cols != COLS_N && N % 16 != 0) return refuse(B200_ERR_ARG, "gemm", "GEGLU epilogues need N = 2F with F % 8 == 0");
    if (ldo < N) return refuse(B200_ERR_ARG, "gemm", "ldo < N");
    if (e.out1 && out1 == nullptr) return refuse(B200_ERR_ARG, "gemm", "epilogue needs out1");
    if (e.aux != AUX_NONE && aux == nullptr) return refuse(B200_ERR_ARG, "gemm", "epilogue needs aux");
    if (e.bias == BIAS_REFUSED && bias != nullptr) return refuse(B200_ERR_ARG, "gemm", "epilogue takes no bias");
    if (e.bias == BIAS_PAIR && (bias == nullptr || !aligned(4, {bias})))
        return refuse(B200_ERR_ARG, "gemm", "epilogue needs a 4-byte aligned bias [2F]");
    // the epilogue writes and reads with plain 16-byte global accesses: rows must start 16-byte aligned
    if ((static_cast<unsigned long long>(ldo) * (e.out_f32 ? 4 : 2)) % 16 != 0) return refuse(B200_ERR_ALIGN, "gemm", "ldo rows must be 16-byte aligned");
    if (!aligned(16, {out0, out1, aux})) return refuse(B200_ERR_ALIGN, "gemm", "out0 / out1 / aux not 16-byte aligned");
    return 0;
}

static int gemm_dispatch(const void* A, long long lda, int a_mn_major, const void* B, long long ldb,
                         int b_mn_major, int M, int N, int K, int epilogue, const void* bias, void* out0,
                         void* out1, const void* aux, long long ldo, int splits, int max_ctas,
                         cudaStream_t stream, const ConvGeom* cg) {
    const int a_mn = a_mn_major ? 1 : 0, b_mn = b_mn_major ? 1 : 0;
    if (splits < 1) splits = 1;
    if (const int rc = check_gemm_args(A, a_mn, B, b_mn, M, N, K, epilogue, bias, out0, out1, aux, ldo, splits, cg != nullptr && cg->mode == 1))
        return rc;
    const EpiTraits& e = kEpi[epilogue];
    const int num_kb = (K + BK - 1) / BK;
    if (splits > num_kb) splits = num_kb;
    const int n_cols = e.cols == COLS_N ? N : N / 2;  // the width of the GEMM itself

    CUtensorMap tmA, tmB;
    int rc;
    {
        // A: K-major [M, lda] -> dims {K, M}, box {64, 128};  MN-major [K, lda] -> dims {M, K}, box {64, 64}
        uint64_t d[2], s[1];
        uint32_t bx[2];
        if (cg != nullptr && cg->mode == 1) {
            // channels-last activation [B, H, W, Cin]: dims {Cin, W, H, B}; box = 64 channels x 128 consecutive pixels: whole
            // rows when W divides 128, else (W = 128 times a power of 2) 128 pixels of one row
            const int wb = cg->W < BM ? cg->W : BM;                                         // pixels of a row per tile
            const int hb = cg->W >= BM ? 1 : (cg->H < BM / cg->W ? cg->H : BM / cg->W);      // image rows per tile
            const int nb = BM / (wb * hb);                                // images per tile (> 1 only when H * W < 128)
            const uint32_t st = conv_ys(cg->kind);
            const uint64_t sw = st * static_cast<uint64_t>(cg->W), sh = st * static_cast<uint64_t>(cg->H);
            uint64_t d4[4] = {static_cast<uint64_t>(cg->Cin), sw, sh, static_cast<uint64_t>(cg->B)};
            uint64_t s4[3] = {static_cast<uint64_t>(cg->Cin) * 2, sw * cg->Cin * 2, sh * sw * cg->Cin * 2};
            uint32_t b4[4] = {BK, st * wb, st * hb, static_cast<uint32_t>(nb)};
            const uint32_t es[4] = {1, st, st, 1};
            if ((rc = make_tmap(&tmA, A, 2, 4, d4, s4, b4, 128, es)) != 0) return rc;
        } else {
        if (!a_mn) { d[0] = K; d[1] = M; bx[0] = BK; bx[1] = BM; }
        else       { d[0] = M; d[1] = K; bx[0] = 64; bx[1] = BK; }
        s[0] = static_cast<uint64_t>(lda) * 2;
        if ((rc = make_tmap(&tmA, A, 2, 2, d, s, bx, 128)) != 0) return rc;
        }
        if (cg != nullptr && cg->mode == 2) {
            // weight gradient: the activation as the MN-major B operand, box = 64 channels x 64 consecutive pixels (one k-block)
            const int hb = BK / cg->W;
            const uint32_t st = conv_ys(cg->kind);
            const uint64_t sw = st * static_cast<uint64_t>(cg->W), sh = st * static_cast<uint64_t>(cg->H);
            uint64_t d4[4] = {static_cast<uint64_t>(cg->Cin), sw, sh, static_cast<uint64_t>(cg->B)};
            uint64_t s4[3] = {static_cast<uint64_t>(cg->Cin) * 2, sw * cg->Cin * 2, sh * sw * cg->Cin * 2};
            uint32_t b4[4] = {64, static_cast<uint32_t>(sw), st * hb, 1};
            const uint32_t es[4] = {1, st, st, 1};
            if ((rc = make_tmap(&tmB, B, 2, 4, d4, s4, b4, 128, es)) != 0) return rc;
        } else if (e.cols == COLS_F_PAIRED) {
            // W1 [2F, ldb] as {K, F, 2}: one box is 128 rows of the h half and the same 128 rows of the gate half
            const uint64_t F = static_cast<uint64_t>(n_cols);
            uint64_t d3[3] = {static_cast<uint64_t>(K), F, 2};
            uint64_t s3[2] = {static_cast<uint64_t>(ldb) * 2, F * static_cast<uint64_t>(ldb) * 2};
            uint32_t b3[3] = {BK, BN / 2, 2};
            if ((rc = make_tmap(&tmB, B, 2, 3, d3, s3, b3, 128)) != 0) return rc;
        } else {
        if (!b_mn) { d[0] = K; d[1] = n_cols; bx[0] = BK; bx[1] = BN; }
        else       { d[0] = n_cols; d[1] = K; bx[0] = 64; bx[1] = BK; }
        s[0] = static_cast<uint64_t>(ldb) * 2;
        if ((rc = make_tmap(&tmB, B, 2, 2, d, s, bx, 128)) != 0) return rc;
        }
    }
    GemmParams p{};
    p.conv = cg != nullptr ? cg->mode : 0;
    p.conv_h = cg != nullptr ? cg->H : 0;
    p.conv_w = cg != nullptr ? cg->W : 0;
    p.conv_cin = cg != nullptr ? cg->Cin : 0;
    p.M = M; p.N = N; p.K = K;
    p.num_m_tiles = (M + BM - 1) / BM;
    p.conv_kind = cg != nullptr ? cg->kind : 0;
    p.class_rows = M;
    p.class_stride = p.num_m_tiles * BM;
    if (cg != nullptr && conv_classes(cg->kind) > 1) {  // M = 4 class_stride
        p.class_rows = cg->B * cg->H * cg->W;
        p.class_stride = M / 4;
    }
    const int tile_n = e.cols == COLS_F_PAIRED ? BN / 2 : BN;
    p.num_n_tiles = (n_cols + tile_n - 1) / tile_n;
    p.splits = splits;
    p.num_kb = num_kb;
    p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
    p.out0 = out0;
    p.out1 = out1;
    p.aux = aux;
    p.ldo = ldo;
    const long long units = static_cast<long long>(p.num_m_tiles) * p.num_n_tiles * splits;
    int grid = persistent_ctas();
    if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
    if (units < grid) grid = static_cast<int>(units);
    if (cg != nullptr && cg->mode == 1) return kLaunchConv[epilogue](tmA, tmB, p, grid, stream);  // (admitted by check_gemm_args)
    return kLaunch[epilogue][2 * a_mn + b_mn](tmA, tmB, p, grid, stream);
}

extern "C" int b200_gemm_bf16(const void* A, long long lda, int a_mn_major, const void* B, long long ldb,
                              int b_mn_major, int M, int N, int K, int epilogue, const void* bias, void* out0,
                              void* out1, const void* aux, long long ldo, int splits, int max_ctas,
                              cudaStream_t stream) {
    return gemm_dispatch(A, lda, a_mn_major, B, ldb, b_mn_major, M, N, K, epilogue, bias, out0, out1, aux, ldo, splits, max_ctas, stream, nullptr);
}

// Widths of 128 times a power of 2 (256, 512, ...: the KL decoder's wide images) take tiles of 128 pixels of one row; the
// narrower widths that divide 128 keep tiles of whole rows.  The power of 2 is a policy, not a correctness condition: any
// multiple of 128 keeps every tile inside one row and would tile the same way.  It keeps the admitted widths to those the
// decoder's levels produce (W = 384, a 768 px image's, stays refused with the rest of that geometry).
static bool wide_rows(int W) { return W > BM && W % BM == 0 && ((W / BM) & (W / BM - 1)) == 0; }

// 3x3 convolution, stride 1, zero padding 1, on channels-last bf16 activations, as an implicit GEMM on the wgmma main loop:
//   out[b, y, x, co] = epilogue( sum_{ky,kx,ci} x[b, y+ky-1, x+kx-1, ci] * w[co, ky, kx, ci] )
// x: [B, H, W, Cin]; w_packed: [Cout, 9 * Cin] (tap-major: k = (ky * 3 + kx) * Cin + ci); out / aux: [B*H*W, ldo].
// M = B*H*W pixels, N = Cout, K = 9 * Cin; the im2col matrix is never materialised -- every (tap, 64-channel) k-block is one
// TMA box of the activation shifted by the tap, with the halo zero-filled by the TMA unit.
// Replaces Conv2d.forward -> F.conv2d (cflearn/modules/core/convs/basic.py:155-174) as the SD-v1.5 UNet uses it
// (convs/residual.py:179-186,199-205 conv1 / conv2; multimodal/diffusion/unet.py:213-217,269-272).  Its input gradient is the
// same call with the weights flipped and transposed ([Cin, 9 * Cout], tap (2-ky, 2-kx)).
extern "C" int b200_conv3x3_nhwc_bf16(const void* x, const void* w_packed, const void* bias, void* out0, const void* aux, long long ldo,
                                      int B, int H, int W, int Cin, int Cout, int epilogue, cudaStream_t stream) {
    if (B <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return refuse(B200_ERR_ARG, "conv3x3", "non-positive size");
    if (Cin % BK != 0) return refuse(B200_ERR_ARG, "conv3x3", "Cin must be a multiple of 64");
    if (!wide_rows(W)) {
        if (W > BM || BM % W != 0) return refuse(B200_ERR_ARG, "conv3x3", "the image width must divide 128 or be 128 times a power of 2");
        const int hb = H < BM / W ? H : BM / W;
        if (H % hb != 0 || BM % (W * hb) != 0) return refuse(B200_ERR_ARG, "conv3x3", "H must be a multiple of 128 / W (or H * W must divide 128)");
    }
    const ConvGeom cg{B, H, W, Cin, 1, CONV_S1};
    const long long M = static_cast<long long>(B) * H * W;
    if (M > 0x7fffffffll) return refuse(B200_ERR_ARG, "conv3x3", "too many pixels");
    return gemm_dispatch(x, Cin, 0, w_packed, 9ll * Cin, 0, static_cast<int>(M), Cout, 9 * Cin, epilogue, bias, out0, nullptr, aux, ldo, 1, 0,
                         stream, &cg);
}

// Weight gradient of the same convolution: dW[co][tap][ci] = sum over pixels of dy[pixel, co] * x[pixel shifted by tap, ci], as ONE
// split-K GEMM with M = Cout, N = 9 * Cin, K = B * H * W: A = dy MN-major (plain 2-D map), B = x MN-major behind the 4-D map, every
// 64-channel box of an N tile shifted by its own tap (halo zero-filled by TMA).  Writes `splits` fp32 partial planes
// [splits][Cout][9 * Cin] (b200_splitk_reduce finishes them); the plane layout IS the packed forward weight layout.
// Replaces the weight half of torch's conv2d backward for convs/basic.py:155-174 under the UNet blocks (convs/residual.py:179-205).
extern "C" int b200_conv3x3_wgrad_nhwc_bf16(const void* dy, long long ld_dy, const void* x, void* partials, int B, int H, int W, int Cin,
                                            int Cout, int splits, cudaStream_t stream) {
    if (B <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return refuse(B200_ERR_ARG, "conv3x3 wgrad", "non-positive size");
    if (Cin % 64 != 0) return refuse(B200_ERR_ARG, "conv3x3 wgrad", "Cin must be a multiple of 64");
    if (W > BK || BK % W != 0) return refuse(B200_ERR_ARG, "conv3x3 wgrad", "the image width must divide 64");
    if ((static_cast<long long>(H) * W) % BK != 0) return refuse(B200_ERR_ARG, "conv3x3 wgrad", "H * W must be a multiple of 64");
    const long long K = static_cast<long long>(B) * H * W;
    if (K > 0x7fffffffll) return refuse(B200_ERR_ARG, "conv3x3 wgrad", "too many pixels");
    const ConvGeom cg{B, H, W, Cin, 2, CONV_S1};
    return gemm_dispatch(dy, ld_dy, 1, x, Cin, 1, Cout, 9 * Cin, static_cast<int>(K), EPI_PARTIAL_F32, nullptr, partials, nullptr, nullptr,
                         9ll * Cin, splits, 0, stream, &cg);
}

// ------------------------------------------------------------------------------------------------
// resampling convolutions (include/b200_cflearn_ext.h): the same main loop with other tap tables and output addressing
// ------------------------------------------------------------------------------------------------
// The size checks every resampling entry shares.  (H, W) is the lower-resolution side; (h, w) the grid the GEMM tiles;
// red / outc: the reduction's and the output's channels.  wide: the grid may also be 128 times a power of 2 wide (forward entries
// whose tiles need no whole rows).
static int check_resample(const char* entry, int B, int H, int W, int red, int outc, bool even, int h, int w, bool wide = false) {
    if (B <= 0 || H <= 0 || W <= 0 || red <= 0 || outc <= 0) return refuse(B200_ERR_ARG, entry, "non-positive size");
    if (even && (H % 2 != 0 || W % 2 != 0)) return refuse(B200_ERR_ARG, entry, "H and W must be even");
    if (red % BK != 0) return refuse(B200_ERR_ARG, entry, "the reduction's channel count must be a multiple of 64");
    if (outc % 8 != 0) return refuse(B200_ERR_ARG, entry, "the output's channel count must be a multiple of 8");
    if (!(wide && wide_rows(w))) {
        if (w > BM || BM % w != 0)
            return refuse(B200_ERR_ARG, entry, wide ? "the grid width must divide 128 or be 128 times a power of 2" : "the grid width must divide 128");
        const int hb = h < BM / w ? h : BM / w;
        if (h % hb != 0 || BM % (w * hb) != 0) return refuse(B200_ERR_ARG, entry, "the grid height must be a multiple of 128 / width (or height * width must divide 128)");
    }
    if (4ll * B * (2 * H) * (2 * W) > 0x7fffffffll) return refuse(B200_ERR_ARG, entry, "too many pixels");
    return 0;
}

// four parity classes of a [B, h, w] grid, each padded to whole tiles: the GEMM's M
static int class_m(const ConvGeom& g) {
    const long long rows = static_cast<long long>(g.B) * g.H * g.W;
    return static_cast<int>(4 * ((rows + BM - 1) / BM) * BM);
}

extern "C" int b200_conv3x3_s2_nhwc_bf16(const void* x, const void* w_packed, const void* bias, void* out0, const void* aux, long long ldo,
                                         int B, int H, int W, int Cin, int Cout, int epilogue, cudaStream_t stream) {
    if (const int rc = check_resample("conv3x3_s2", B, H, W, Cin, Cout, true, H / 2, W / 2)) return rc;
    const ConvGeom cg{B, H / 2, W / 2, Cin, 1, CONV_S2};
    return gemm_dispatch(x, Cin, 0, w_packed, 9ll * Cin, 0, B * (H / 2) * (W / 2), Cout, 9 * Cin, epilogue, bias, out0, nullptr, aux, ldo,
                         1, 0, stream, &cg);
}

extern "C" int b200_conv3x3_s2_dgrad_nhwc_bf16(const void* dy, const void* w_dgrad, void* dx, int B, int H, int W, int Cin, int Cout,
                                               cudaStream_t stream) {
    if (const int rc = check_resample("conv3x3_s2 dgrad", B, H, W, Cout, Cin, true, H / 2, W / 2)) return rc;
    const ConvGeom cg{B, H / 2, W / 2, Cout, 1, CONV_S2_DGRAD};
    return gemm_dispatch(dy, Cout, 0, w_dgrad, 9ll * Cout, 0, class_m(cg), Cin, 9 * Cout, EPI_BIAS_BF16, nullptr, dx, nullptr, nullptr, Cin,
                         1, 0, stream, &cg);
}

extern "C" int b200_conv3x3_s2_wgrad_nhwc_bf16(const void* dy, long long ld_dy, const void* x, void* partials, int B, int H, int W, int Cin,
                                               int Cout, int splits, cudaStream_t stream) {
    const char* what = "conv3x3_s2 wgrad";
    if (const int rc = check_resample(what, B, H, W, Cin, Cout, true, H / 2, W / 2)) return rc;
    const int h = H / 2, w = W / 2;
    if (w > BK || BK % w != 0) return refuse(B200_ERR_ARG, what, "the grid width must divide 64");
    if ((h * w) % BK != 0) return refuse(B200_ERR_ARG, what, "the grid's height * width must be a multiple of 64");
    const ConvGeom cg{B, h, w, Cin, 2, CONV_S2};
    return gemm_dispatch(dy, ld_dy, 1, x, Cin, 1, Cout, 9 * Cin, B * h * w, EPI_PARTIAL_F32, nullptr, partials, nullptr, nullptr, 9ll * Cin,
                         splits, 0, stream, &cg);
}

extern "C" int b200_conv3x3_up2_nhwc_bf16(const void* x, const void* w_packed, const void* bias, void* out0, const void* aux, long long ldo,
                                          int B, int H, int W, int Cin, int Cout, int epilogue, cudaStream_t stream) {
    if (const int rc = check_resample("conv3x3_up2", B, H, W, Cin, Cout, false, H, W, true)) return rc;
    const ConvGeom cg{B, H, W, Cin, 1, CONV_UP2};
    return gemm_dispatch(x, Cin, 0, w_packed, 9ll * Cin, 0, class_m(cg), Cout, 9 * Cin, epilogue, bias, out0, nullptr, aux, ldo, 1, 0,
                         stream, &cg);
}
