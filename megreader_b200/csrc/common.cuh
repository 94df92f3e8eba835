// Shared helpers for the megreader_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cublas_v2.h>
#include <stdint.h>
#include <atomic>
#include "../../include/megreader_b200.h"

namespace mr {

extern std::atomic<int64_t> g_launch_count;
void set_cuda_error(cudaError_t e, const char *where);

inline int check_launch(const char *where) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_cuda_error(e, where); return MR_ERR_CUDA; }
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    return MR_OK;
}

#define MR_CUDA_TRY(expr, where)                                            \
    do { cudaError_t _e = (expr);                                           \
         if (_e != cudaSuccess) { ::mr::set_cuda_error(_e, where); return MR_ERR_CUDA; } } while (0)

// cuBLAS handle, one per device, created on first use (cuBLAS allocates its own workspace then); bound to `st`.
int blas_handle(cublasHandle_t *h, cudaStream_t st);
#define MR_BLAS_TRY(expr, where)                                                                        \
    do { if ((expr) != CUBLAS_STATUS_SUCCESS) { ::mr::set_cuda_error(cudaErrorUnknown, where); return MR_ERR_CUDA; } } while (0)

// Per-DEVICE caches (a process may drive several GPUs): opt a kernel into `bytes` of dynamic shared memory once per
// (kernel, device) -- cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute -- and the SM count.
int ensure_dyn_smem(const void *func, size_t bytes, const char *where);
int sm_count();

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline int64_t round_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// ---- async copy (LDGSTS) ----
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async8(void *smem, const void *gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void *smem, const void *gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

}  // namespace mr
