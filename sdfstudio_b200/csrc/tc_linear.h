// Generic tensor-core Linear (csrc/tc_linear.cu): drop-in for sgemm() of field_simt.cu when the field runs at a tensor-core precision
// but its shape is outside the fused kernel's family.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sdfb200 {

enum { TCL_NONE = 0, TCL_SOFTPLUS = 1, TCL_RELU = 2, TCL_MUL_DSOFTPLUS = 3 };   // same numbering as EPI_* in field_simt.cu
constexpr size_t kTcGemmScratchBytes = 2ull * 256 * 256 * 2;                    // packed weight planes of one (N, K) chunk

// packed index -> source index (-1 = zero) of the fused kernel's 96-wide small-K operands (field_tc.h kInK)
struct TcIdxMap { short src[96]; };

// fp32 W -> bf16 split planes (w = w0 + w1, `planes` of them) in the wgmma B-operand layout of the tensor-core kernels (tc_common.cuh):
//     [K-block of kblk][plane][k/8][row n < Np][8 bf16],   nblocks K-blocks, zero padded
// Element (n, k) is W[n * ldw + k], or W[k * ldw + n] when trans != 0.  Without a map, rows n >= N and columns k >= K are zero; with
// one, packed row n / column k takes source index rowmap->src[n] / colmap->src[k] (and N / K are not used).  One kernel launch.
int tc_pack(const float* W, int ldw, int trans, int N, int K, int Np, int kblk, int nblocks, int planes, const TcIdxMap* rowmap,
            const TcIdxMap* colmap, void* out, cudaStream_t st);

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
