// Generic tensor-core Linear (csrc/tc_linear.cu): drop-in for sgemm() of field_simt.cu when the field runs at a tensor-core precision
// but its shape is outside the fused kernel's family.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sdfb200 {

enum { TCL_NONE = 0, TCL_SOFTPLUS = 1, TCL_RELU = 2, TCL_MUL_DSOFTPLUS = 3 };   // same numbering as EPI_* in field_simt.cu
constexpr size_t kTcGemmScratchBytes = 2ull * 256 * 256 * 2;                    // packed weight planes of one (N, K) chunk

// Y[M, Np] = epi(X[M, Kp] W[Np, Kp]^T + bias);  planes: 1 = bf16, 2 = bf16x3.  Y must not alias X.
int tc_gemm(int planes, int epi, const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy, int64_t M, int Np, int Kp,
            const float* aux, int ldaux, int aux_cols, void* scratch, cudaStream_t st);

int tc_gemm_ex(int planes, int epi, const float* X, int ldx, const float* W, int ldw, int trans_w, int Nw, int Kw, const float* bias, float* Y, int ldy,
               int64_t M, int Np, int Kp, const float* aux, int ldaux, int aux_cols, void* scratch, cudaStream_t st);

// weight-gradient GEMM (csrc/tc_wgrad.cu): C[N, K] = A[P, N]^T B[P, K]
size_t tc_wgrad_workspace_bytes();
int tc_wgrad(int planes, const float* A, long long lda, const float* B, long long ldb, float* C, long long ldc, int64_t P, int N, int K, void* workspace,
             size_t workspace_bytes, cudaStream_t st);

}  // namespace sdfb200
