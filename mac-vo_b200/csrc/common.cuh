// Shared helpers for the macvo_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/macvo_b200.h"

#define MACVO_CUDA_TRY(expr)                         \
    do {                                             \
        cudaError_t _e = (expr);                     \
        if (_e != cudaSuccess) return (int)_e;       \
    } while (0)

#define MACVO_LAUNCH_CHECK()                         \
    do {                                             \
        cudaError_t _e = cudaGetLastError();         \
        if (_e != cudaSuccess) return (int)_e;       \
    } while (0)

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

__host__ __device__ static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// exact (erf) GELU, the default of torch.nn.functional.gelu
__device__ __forceinline__ static float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
