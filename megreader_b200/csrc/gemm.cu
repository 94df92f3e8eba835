// Plain dense GEMMs of the engine: row-major  C[M,N] = alpha * op(A) * op(B) + beta * C  with fp32 accumulation.
// This revision routes them to cuBLAS (cublasGemmEx / cublasGemmStridedBatchedEx) — "plain library GEMMs" per the
// build rules; the conv / LSTM *fusions* around them are this repo's kernels.  A wgmma + TMA kernel replaces the
// dominant shapes behind the same entry point (csrc/gemm_tcgen05.cu) when MR_GEMM_BACKEND selects it.
//
// Row-major <-> cuBLAS column-major: C^T = op(B)^T op(A)^T, so the operands are swapped and an operand that is
// stored transposed in row-major terms needs CUBLAS_OP_T.
#include "common.cuh"
#include <cuda_bf16.h>

namespace {
using namespace mr;
cudaDataType_t cuda_type(int dtype) { return dtype == 0 ? CUDA_R_32F : CUDA_R_16BF; }
}  // namespace

extern "C" {

/* op(A) is [M,K]: A stored [M,K] (transA=0, lda >= K) or [K,M] (transA=1, lda >= M); same for B with op(B) [K,N]:
 * stored [K,N] (transB=0, ldb >= N) or [N,K] (transB=1, ldb >= K).  C stored [M,N], ldc >= N.
 * in_dtype / out_dtype: 0 = fp32, 1 = bf16 (inputs share one dtype). */
int mr_gemm(const void *A, const void *B, void *C, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
            int64_t ldc, int transA, int transB, int in_dtype, int out_dtype, float alpha, float beta, void *stream) {
    if (M < 0 || N < 0 || K < 0) return MR_ERR_BAD_SHAPE;
    if (M == 0 || N == 0) return MR_OK;
    if (!A || !B || !C) return MR_ERR_NULL_POINTER;
    cublasHandle_t h;
    int rc = blas_handle(&h, (cudaStream_t)stream);
    if (rc) return rc;
    MR_BLAS_TRY(cublasGemmEx(h, transB ? CUBLAS_OP_T : CUBLAS_OP_N, transA ? CUBLAS_OP_T : CUBLAS_OP_N, (int)N, (int)M,
                             (int)K, &alpha, B, cuda_type(in_dtype), (int)ldb, A, cuda_type(in_dtype), (int)lda, &beta, C,
                             cuda_type(out_dtype), (int)ldc, CUBLAS_COMPUTE_32F, CUBLAS_GEMM_DEFAULT),
                "cublasGemmEx");
    return MR_OK;
}

int mr_gemm_batched(const void *A, const void *B, void *C, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                    int64_t ldc, int64_t strideA, int64_t strideB, int64_t strideC, int batch, int transA, int transB,
                    int in_dtype, int out_dtype, float alpha, float beta, void *stream) {
    if (M < 0 || N < 0 || K < 0 || batch < 0) return MR_ERR_BAD_SHAPE;
    if (M == 0 || N == 0 || batch == 0) return MR_OK;
    if (!A || !B || !C) return MR_ERR_NULL_POINTER;
    cublasHandle_t h;
    int rc = blas_handle(&h, (cudaStream_t)stream);
    if (rc) return rc;
    MR_BLAS_TRY(cublasGemmStridedBatchedEx(h, transB ? CUBLAS_OP_T : CUBLAS_OP_N, transA ? CUBLAS_OP_T : CUBLAS_OP_N,
                                           (int)N, (int)M, (int)K, &alpha, B, cuda_type(in_dtype), (int)ldb, strideB, A,
                                           cuda_type(in_dtype), (int)lda, strideA, &beta, C, cuda_type(out_dtype),
                                           (int)ldc, strideC, batch, CUBLAS_COMPUTE_32F, CUBLAS_GEMM_DEFAULT),
                "cublasGemmStridedBatchedEx");
    return MR_OK;
}

}  // extern "C"
