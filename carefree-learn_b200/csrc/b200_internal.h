// Internal declarations shared by the .cu files of libb200_cflearn.so
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

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
void count_launch(int n = 1);
int check_launch(const char* what);  // cudaGetLastError -> set_error

int num_sms();
int persistent_ctas();  // grid of the persistent kernels: num_sms() unless b200_set_persistent_ctas() lowered it (gemm_sm90.cu)
int current_device_slot();  // cudaGetDevice() clamped to [0, 64): index of per-device caches
int make_tmap(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes);

}  // namespace b200
