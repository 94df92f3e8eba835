#include "common.cuh"
#include <map>
#include <mutex>
#include <utility>
#include <string>

namespace mr {
std::atomic<int64_t> g_launch_count{0};
static std::mutex g_err_mu;
static std::string g_err;
void set_cuda_error(cudaError_t e, const char *where) {
    std::lock_guard<std::mutex> lk(g_err_mu);
    g_err = std::string(where) + ": " + cudaGetErrorName(e) + ": " + cudaGetErrorString(e);
}
static std::mutex g_attr_mu;
static std::map<std::pair<const void *, int>, size_t> g_attr;
int ensure_dyn_smem(const void *func, size_t bytes, const char *where) {
    int dev = 0;
    MR_CUDA_TRY(cudaGetDevice(&dev), "cudaGetDevice");
    std::lock_guard<std::mutex> lk(g_attr_mu);
    size_t &have = g_attr[std::make_pair(func, dev)];
    if (bytes > have) {
        MR_CUDA_TRY(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes), where);
        have = bytes;
    }
    return MR_OK;
}
int sm_count() {
    static std::atomic<int> cache[16];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return 132;
    int v = cache[dev].load(std::memory_order_relaxed);
    if (v <= 0) {
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        cache[dev].store(v, std::memory_order_relaxed);
    }
    return v;
}
static std::mutex g_blas_mu;
static cublasHandle_t g_blas[16] = {nullptr};
int blas_handle(cublasHandle_t *h, cudaStream_t st) {
    int dev = 0;
    MR_CUDA_TRY(cudaGetDevice(&dev), "cudaGetDevice");
    if (dev < 0 || dev >= 16) return MR_ERR_NO_DEVICE;
    std::lock_guard<std::mutex> lk(g_blas_mu);
    if (!g_blas[dev]) {
        if (cublasCreate(&g_blas[dev]) != CUBLAS_STATUS_SUCCESS) { set_cuda_error(cudaErrorUnknown, "cublasCreate"); return MR_ERR_CUDA; }
        cublasSetMathMode(g_blas[dev], CUBLAS_DEFAULT_MATH);  // fp32 GEMMs stay plain fp32 (no TF32)
    }
    if (cublasSetStream(g_blas[dev], st) != CUBLAS_STATUS_SUCCESS) { set_cuda_error(cudaErrorUnknown, "cublasSetStream"); return MR_ERR_CUDA; }
    *h = g_blas[dev];
    return MR_OK;
}
}  // namespace mr

extern "C" {
const char *mr_status_string(int s) {
    switch (s) {
        case MR_OK: return "ok";
        case MR_ERR_NULL_POINTER: return "null pointer argument";
        case MR_ERR_BLANK_RANGE: return "blank must be in label range";
        case MR_ERR_TARGET_TOO_LONG: return "max target length out of range (2*S+1 must be <= 1024)";
        case MR_ERR_BAD_SHAPE: return "bad shape / size argument";
        case MR_ERR_UNSUPPORTED: return "shape not supported by this build (on-chip staging does not fit)";
        case MR_ERR_CUDA: return "CUDA runtime error (see mr_last_cuda_error)";
        case MR_ERR_NO_DEVICE: return "no CUDA device";
        default: return "unknown status";
    }
}
const char *mr_last_cuda_error(void) {
    static thread_local std::string copy;
    std::lock_guard<std::mutex> lk(mr::g_err_mu);
    copy = mr::g_err;
    return copy.c_str();
}
int mr_abi_version(void) { return 1; }
int64_t mr_launch_count(void) { return mr::g_launch_count.load(); }
void mr_launch_count_reset(void) { mr::g_launch_count.store(0); }
}
