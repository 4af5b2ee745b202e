// Internal declarations shared by the .cu files of libb200_cflearn.so
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <initializer_list>

#include "../../include/b200_cflearn.h"

namespace b200 {

enum : int {
    EPI_BIAS_BF16 = B200_EPI_BIAS_BF16,
    EPI_BIAS_GELU_BF16 = B200_EPI_BIAS_GELU_BF16,
    EPI_BIAS_RESID_F32 = B200_EPI_BIAS_RESID_F32,
    EPI_DGELU_BF16 = B200_EPI_DGELU_BF16,
    EPI_PARTIAL_F32 = B200_EPI_PARTIAL_F32,
    EPI_BIAS_GEGLU_BF16 = B200_EPI_BIAS_GEGLU_BF16,
    EPI_DGEGLU_BF16 = B200_EPI_DGEGLU_BF16,
    EPI_BIAS_RESID_BF16 = B200_EPI_BIAS_RESID_BF16,
    EPI_BIAS_ADD_PER_IMAGE_BF16 = B200_EPI_BIAS_ADD_PER_IMAGE_BF16,
    EPI_BIAS_RESID_CLAMP_BF16 = B200_EPI_BIAS_RESID_CLAMP_BF16,
};

int set_error(int code, const char* msg);  // records msg (thread-local) and returns code
int refuse(int code, const char* entry, const char* rule);  // set_error(code, "<entry>: <rule>")
void count_launch(int n = 1);
int check_launch(const char* what);  // cudaGetLastError -> set_error

// every non-NULL pointer of ps is aligned to n bytes (a power of two)
inline bool aligned(uintptr_t n, std::initializer_list<const void*> ps) {
    uintptr_t any = 0;
    for (const void* p : ps) any |= reinterpret_cast<uintptr_t>(p);
    return (any & (n - 1)) == 0;
}

int num_sms();
int persistent_ctas();  // grid of the persistent kernels: num_sms() unless b200_set_persistent_ctas() lowered it (gemm_sm90.cu)
int current_device_slot();  // cudaGetDevice() clamped to [0, 64): index of per-device caches

// The dynamic shared-memory limit belongs to the (function, device) pair: raised to smem bytes once per device, and checked.
template <typename Kernel>
int configure_smem(Kernel kernel, int smem, bool (&configured)[64]) {
    const int dev = current_device_slot();
    if (configured[dev]) return 0;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return set_error(B200_ERR_LAUNCH, cudaGetErrorString(e));
    configured[dev] = true;
    return 0;
}

int make_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes, const uint32_t* elem_strides = nullptr);

}  // namespace b200
