// Fused fp32 training step of a small fully-connected network (Linear -> ReLU -> ... -> Linear) for sm_90a.
//
// Replaces, for BASELINE.json configs[0] (FCNN on 10-feature tabular data, batch 128):
//   FCNN.forward                      cflearn/modules/ml/fcnn.py:58-59
//   Mapping.forward (Linear + ReLU)   cflearn/modules/core/mappings.py:74-83, core/customs.py:81-100
//   MAELoss / MSELoss + mean + merge  cflearn/losses/basic.py:45-61, schema.py:767-771, losses/common.py:72-79
//   and their autograd.
// The reference runs this configuration on the CPU and is bound by per-op Python / dispatch overhead (1,441
// parameters).  Here the whole step -- forward, loss, backward, per-block gradient partials -- is ONE launch: the
// parameters and every activation live in shared memory, one thread owns one sample (activations stored
// [unit][sample], row stride 129 floats, so both the per-sample and the per-weight passes are bank-conflict free).
// fp32 FFMA throughout (no tensor cores: a 32x32 layer has nothing to tile); sums run in a fixed order, so results are
// deterministic run to run.  Blocks of 128 samples write gradient partials part[block][P + 1] (column P = loss), which
// b200_colsum_finish reduces.
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200_internal.h"

namespace b200 {

constexpr int MLP_ROWS = 128;
constexpr int MLP_LD = MLP_ROWS + 1;
constexpr int MLP_MAX_L = 8;

struct MlpParams {
    int M, L, P;                  // samples, Linear layers, parameter-arena length (floats)
    int dims[MLP_MAX_L + 1];      // widths: input, hidden..., output
    int woff[MLP_MAX_L];          // arena offset of W_l [dims[l+1], dims[l]] (row-major, like nn.Linear.weight)
    int boff[MLP_MAX_L];          // arena offset of b_l [dims[l+1]], -1 without bias
    int aoff[MLP_MAX_L + 1];      // smem offset (floats) of activation buffer l
    int loss_mode;                // 0: gradient of the output given (dpred) ; 1: w_mae * mean|p-y| + w_mse * mean (p-y)^2
    float w_mae, w_mse;
};

__global__ void __launch_bounds__(MLP_ROWS)
mlp_step_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dpred,
                const float* __restrict__ params, float* __restrict__ pred, float* __restrict__ part, const MlpParams p) {
    extern __shared__ float sm[];
    float* sp = sm;            // parameters, arena layout
    float* sa = sm + p.P;      // activation buffers
    __shared__ float sred[MLP_ROWS / 32];
    const int s = threadIdx.x;
    const int row = blockIdx.x * MLP_ROWS + s;
    const bool valid = row < p.M;
    for (int i = s; i < p.P; i += MLP_ROWS) sp[i] = params[i];
    {
        float* a0 = sa + p.aoff[0];
        const int in = p.dims[0];
        for (int k = 0; k < in; ++k) a0[k * MLP_LD + s] = valid ? x[static_cast<long long>(row) * in + k] : 0.f;
    }
    __syncthreads();
    // ---- forward: thread-private sample column, weights broadcast from shared memory ----
    for (int l = 0; l < p.L; ++l) {
        const int in = p.dims[l], out = p.dims[l + 1];
        const float* a = sa + p.aoff[l];
        float* o = sa + p.aoff[l + 1];
        const float* W = sp + p.woff[l];
        for (int j = 0; j < out; ++j) {
            float z = p.boff[l] >= 0 ? sp[p.boff[l] + j] : 0.f;
            const float* wr = W + j * in;
            for (int k = 0; k < in; ++k) z = fmaf(wr[k], a[k * MLP_LD + s], z);
            if (l + 1 < p.L) z = fmaxf(z, 0.f);  // ReLU on every Mapping, none on the output Linear (fcnn.py:54)
            o[j * MLP_LD + s] = z;
        }
    }
    const int nout = p.dims[p.L];
    float* aL = sa + p.aoff[p.L];
    if (pred != nullptr && valid)
        for (int j = 0; j < nout; ++j) pred[static_cast<long long>(row) * nout + j] = aL[j * MLP_LD + s];
    if (part == nullptr) return;  // inference
    // ---- output gradient (and the loss) ----
    float lsum = 0.f;
    const float inv = 1.0f / (static_cast<float>(p.M) * static_cast<float>(nout));  // mean over every element
    for (int j = 0; j < nout; ++j) {
        float g = 0.f;
        if (valid) {
            if (p.loss_mode == 1) {
                const float d = aL[j * MLP_LD + s] - y[static_cast<long long>(row) * nout + j];
                lsum += p.w_mae * fabsf(d) + p.w_mse * d * d;
                const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);  // torch's l1 backward: sign(d), 0 at 0
                g = (p.w_mae * sg + p.w_mse * 2.f * d) * inv;
            } else {
                g = dpred[static_cast<long long>(row) * nout + j];
            }
        }
        aL[j * MLP_LD + s] = g;
    }
    float* prow = part + static_cast<long long>(blockIdx.x) * (p.P + 1);
    {
        for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
        if ((s & 31) == 0) sred[s >> 5] = lsum;
    }
    for (int i = s; i < p.P; i += MLP_ROWS) prow[i] = 0.f;  // alignment gaps of the arena
    __syncthreads();
    if (s == 0) prow[p.P] = ((sred[0] + sred[1]) + (sred[2] + sred[3])) * inv;
    // ---- backward ----
    for (int l = p.L - 1; l >= 0; --l) {
        const int in = p.dims[l], out = p.dims[l + 1];
        float* a = sa + p.aoff[l];              // input of layer l (post-ReLU for l > 0)
        const float* d = sa + p.aoff[l + 1];    // gradient of layer l's output
        const int nw = out * in;
        for (int e = s; e < nw + out; e += MLP_ROWS) {  // one weight (or bias) per thread: sum over the block's samples
            float acc = 0.f;
            if (e < nw) {
                const float* dj = d + (e / in) * MLP_LD;
                const float* ak = a + (e % in) * MLP_LD;
                for (int r = 0; r < MLP_ROWS; ++r) acc = fmaf(dj[r], ak[r], acc);
                prow[p.woff[l] + e] = acc;
            } else if (p.boff[l] >= 0) {
                const float* dj = d + (e - nw) * MLP_LD;
                for (int r = 0; r < MLP_ROWS; ++r) acc += dj[r];
                prow[p.boff[l] + (e - nw)] = acc;
            }
        }
        __syncthreads();
        if (l > 0) {  // gradient of layer l's input, through the ReLU that produced it; in place over the activation
            const float* W = sp + p.woff[l];
            for (int k = 0; k < in; ++k) {
                float t = 0.f;
                for (int j = 0; j < out; ++j) t = fmaf(d[j * MLP_LD + s], W[j * in + k], t);
                a[k * MLP_LD + s] = a[k * MLP_LD + s] > 0.f ? t : 0.f;
            }
            __syncthreads();
        }
    }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_fcnn_step(const float* x, const float* y, const float* dpred, const float* params, float* pred,
                              float* part, int M, int n_layers, const int* dims, const int* w_offsets,
                              const int* b_offsets, int arena_len, int loss_mode, float w_mae, float w_mse,
                              int* nblocks_out, cudaStream_t stream) {
    const char* E = "fcnn_step";
    if (M <= 0 || n_layers < 1 || n_layers > MLP_MAX_L || arena_len <= 0) return refuse(B200_ERR_ARG, E, "need 1 <= layers <= 8 and M > 0");
    if (!x || !params || !dims || !w_offsets || !b_offsets) return refuse(B200_ERR_ARG, E, "null pointer");
    if (part != nullptr && loss_mode == 0 && dpred == nullptr) return refuse(B200_ERR_ARG, E, "backward without a loss needs dpred (null pointer)");
    if (part != nullptr && loss_mode == 1 && y == nullptr) return refuse(B200_ERR_ARG, E, "the fused loss needs labels (null pointer)");
    if (!aligned(4, {x, y, dpred, params, pred, part})) return refuse(B200_ERR_ALIGN, E, "pointers not 4-byte aligned");
    MlpParams p;
    p.M = M; p.L = n_layers; p.P = arena_len; p.loss_mode = loss_mode; p.w_mae = w_mae; p.w_mse = w_mse;
    int aoff = 0;
    for (int l = 0; l <= n_layers; ++l) {
        if (dims[l] <= 0) return refuse(B200_ERR_ARG, E, "non-positive layer width");
        p.dims[l] = dims[l];
        p.aoff[l] = aoff;
        aoff += dims[l] * MLP_LD;
    }
    for (int l = 0; l < n_layers; ++l) {
        p.woff[l] = w_offsets[l];
        p.boff[l] = b_offsets[l];
        if (p.woff[l] < 0 || p.woff[l] + dims[l] * dims[l + 1] > arena_len || (p.boff[l] >= 0 && p.boff[l] + dims[l + 1] > arena_len))
            return refuse(B200_ERR_ARG, E, "parameter offsets outside the arena");
    }
    const size_t smem = (static_cast<size_t>(arena_len) + aoff) * sizeof(float);
    if (smem > 220 * 1024) return refuse(B200_ERR_ARG, E, "network too wide for the fused shared-memory kernel (parameters + activations > 220 KB)");
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(mlp_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
        if (e != cudaSuccess) return set_error(B200_ERR_LAUNCH, cudaGetErrorString(e));
    }
    const int nblk = (M + MLP_ROWS - 1) / MLP_ROWS;
    if (nblocks_out) *nblocks_out = nblk;
    mlp_step_kernel<<<nblk, MLP_ROWS, smem, stream>>>(x, y, dpred, params, pred, part, p);
    return check_launch("fcnn_step");
}
