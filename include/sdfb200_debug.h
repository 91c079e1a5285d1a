/*
 * sdfb200_debug.h -- validation hooks of the tensor-core (wgmma) building blocks.  NOT part of the product library: these entry points are
 * compiled into libsdfb200_dbg.so only (sdfstudio_b200/build.py build_debug), which the -m gpu building-block tests load.
 */
#ifndef SDFB200_DEBUG_H_
#define SDFB200_DEBUG_H_
#include "sdfb200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------------------------
 * Debug / validation hook (no reference counterpart): one CTA computes D[128,Np] = A[128,K] W[N,K]^T with the wgmma
 * machinery of the tensor-core kernels (bf16 split planes, A operand in shared memory (mode_ts = 0) or in registers
 * (mode_ts = 1), bulk-copy weight ring).  K % 32 == 0, K <= 256, N <= 256, Np = N rounded up to 16.
 * scratch: >= (K/32)*planes*Np64*64 bytes, Np64 = N rounded up to 64.
 * ------------------------------------------------------------------------------------------------------------- */
int sdfb200_debug_tc_gemm(const float* A, const float* W, int32_t K, int32_t N, int32_t mode_ts, int32_t planes, float* D,
                          void* scratch, void* stream);

/* Building-block test of the generic tensor-core Linear (csrc/tc_linear.cu): Y[M, Np] = epi(X[M, Kp] W[Np, Kp]^T + bias) with
 * epi 0 none / 1 softplus(beta 100) / 2 relu / 3 multiply by softplus'(aux) (no bias); planes 1 = bf16, 2 = bf16x3.
 * All dims padded to 16; scratch >= 256 KiB. */
int sdfb200_debug_tc_linear(int32_t planes, int32_t epi, const float* X, int32_t ldx, const float* W, const float* bias, float* Y,
                            int32_t ldy, int64_t M, int32_t Np, int32_t Kp, const float* aux, int32_t ldaux, int32_t aux_cols,
                            void* scratch, void* stream);

/* debug: copies the 16x32 clock64 phase stamps recorded by the fused tensor-core kernel (CTA 0, first 16 tiles) into a HOST buffer
 * of 512 int64.  The stamps come from the debug library's own build of the bf16x3 / torch-layout instantiation, compiled with
 * -DSDFB200_TC_TIMING (sdfstudio_b200/build.py); the product library records none. */
int sdfb200_debug_tc_timing(long long* host_out_512);

#ifdef __cplusplus
}
#endif
#endif /* SDFB200_DEBUG_H_ */
