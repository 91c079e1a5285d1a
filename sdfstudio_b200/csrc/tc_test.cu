// Building-block test of the wgmma path (sdfb200_debug_tc_gemm): one CTA computes D[128,N] = A[128,K] * W[N,K]^T with
// the machinery of the tensor-core kernels -- bf16 split planes, canonical no-swizzle K-major operands, A either in shared memory
// (SS) or in registers (RS), weights streamed through a 2-stage ring by 1-D bulk copies, accumulator in registers (two warpgroups
// of 64 rows).  Lets the descriptors / layouts be validated in isolation on the GPU.
#include "tc_common.cuh"
#include "tc_linear.h"
#include "../../include/sdfb200_debug.h"

namespace sdfb200 {
using namespace tc;

constexpr int kKB = 32;  // K elements per streamed weight block

template <int P, bool RS>
__global__ void __launch_bounds__(288, 1) k_tc_gemm_test(const float* __restrict__ A, const __nv_bfloat16* __restrict__ Wp, int K, int Np, int Np64,
                                                         float* __restrict__ D) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ Handoff<2> bars;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nblocks = K / kKB;
  const uint32_t stage_bytes = (uint32_t)P * Np64 * kKB * 2;
  uint8_t* a_smem = smem;                                        // [P][K/8][128][16 B]   (SS mode only)
  uint8_t* w_smem = smem + (RS ? 0 : (size_t)P * K * 256);       // 2 stages
  if (tid == 0) {
    bars.init(1, 2);
    fence_barrier_init();
  }
  if (!RS && tid < 256) {
    // ---- stage A as bf16 planes: thread (r, half) converts half of row r ----
    const int r = tid & 127;
    for (int k0 = (tid >> 7) * 16; k0 < K; k0 += 32) {
      uint32_t hi[8], lo[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) split2(A[(size_t)r * K + k0 + 2 * j], A[(size_t)r * K + k0 + 2 * j + 1], hi[j], lo[j]);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const uint32_t off = (uint32_t)((k0 / 8 + c) * kAChunk + r * 16);
        *reinterpret_cast<uint4*>(a_smem + off) = make_uint4(hi[4 * c], hi[4 * c + 1], hi[4 * c + 2], hi[4 * c + 3]);
        if (P > 1) *reinterpret_cast<uint4*>(a_smem + (size_t)K * 256 + off) = make_uint4(lo[4 * c], lo[4 * c + 1], lo[4 * c + 2], lo[4 * c + 3]);
      }
    }
    fence_async_smem();
  }
  __syncthreads();

  if (warp == 8) {
    // ---- weight producer ----
    if (lane == 0) {
      for (int b = 0; b < nblocks; ++b) ring_fill(bars, w_smem, b, reinterpret_cast<const uint8_t*>(Wp), b, stage_bytes);
    }
  } else {
    // ---- two warpgroups, 64 rows each ----
    const int wg = warp >> 2, t = tid & 127;
    const int r0 = frag_row0(wg * 64, t), c2 = frag_cq(t);
    const int nch = Np64 / 64;
    float acc[4][32];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
    const uint32_t lbo_b = (uint32_t)Np64 * 16, plane_b = (uint32_t)Np64 * kKB * 2;
    const uint32_t abase = smem_u32(a_smem) + wg * 64 * 16;
    for (int b = 0; b < nblocks; ++b) {
      bars.wait_full(b);
      const uint32_t wbase = smem_u32(w_smem + (size_t)bars.slot(b) * stage_bytes);
      uint32_t afr[kKB / 16][2][4];
      if (RS) {
        // A fragments straight from global memory: rows r0 / r0 + 8, columns 2c, 2c + 1 (+8) of each K step
#pragma unroll
        for (int j = 0; j < kKB / 16; ++j) {
          const int k = b * kKB + j * 16 + c2;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float* src = A + (size_t)(r0 + 8 * (q & 1)) * K + k + 8 * (q >> 1);
            split2(src[0], src[1], afr[j][0][q], afr[j][1][q]);
          }
        }
      }
      wg_fence_acc(acc[0]); wg_fence_acc(acc[1]); wg_fence_acc(acc[2]); wg_fence_acc(acc[3]);
      wg_arrive();
#pragma unroll
      for (int j = 0; j < kKB / 16; ++j) {
        const int kstep = b * (kKB / 16) + j;  // global 16-wide K step
        const uint32_t baddr = wbase + j * 2 * lbo_b;
        if (RS) {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            if (c < nch) {
              const uint64_t b0 = make_smem_desc(baddr + c * 1024, lbo_b, 128);
              wgmma64_rs(acc[c], afr[j][0], b0);
              if (P > 1) {
                wgmma64_rs(acc[c], afr[j][1], b0);
                wgmma64_rs(acc[c], afr[j][0], make_smem_desc(baddr + plane_b + c * 1024, lbo_b, 128));
              }
            }
          }
        } else {
          wgmma_kstep_ss<P, 4>(acc, a_desc(abase, kstep), a_desc(abase + (uint32_t)K * 256, kstep), baddr, plane_b, lbo_b, nch);
        }
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(acc[0]); wg_fence_acc(acc[1]); wg_fence_acc(acc[2]); wg_fence_acc(acc[3]);
      if (t == 0) bars.arrive_empty(b);
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int col = frag_col(c2, c, i), row = frag_row(r0, i);
        if (c < nch && col < Np) D[(size_t)row * Np + col] = acc[c][i];
      }
    }
  }
}

}  // namespace sdfb200

using namespace sdfb200;

// D[128,Np] = A[128,K] W[N,K]^T ; K % 32 == 0, K <= 256, Np = N rounded up to 16 <= 256.  scratch: >= K/32*planes*Np64*64 B
// (Np64 = N rounded up to 64: the weights are packed in whole n64 blocks)
extern "C" int sdfb200_debug_tc_gemm(const float* A, const float* W, int32_t K, int32_t N, int32_t mode_ts, int32_t planes, float* D, void* scratch,
                                     void* stream) {
  SDFB_REQUIRE(A && W && D && scratch, "NULL pointer");
  SDFB_REQUIRE(K % 32 == 0 && K >= 32 && K <= 256 && N >= 1 && N <= 256 && (planes == 1 || planes == 2), "unsupported test shape");
  const int Np = (N + 15) / 16 * 16, Np64 = (N + 63) / 64 * 64;
  const int nblocks = K / kKB;
  cudaStream_t st = (cudaStream_t)stream;
  if (int r = tc_pack(W, K, 0, N, K, Np64, kKB, nblocks, planes, nullptr, nullptr, scratch, st)) return r;
  const size_t smem = (mode_ts ? 0 : (size_t)planes * K * 256) + 2 * (size_t)planes * Np64 * kKB * 2 + 1024;
#define LAUNCH(P_, TS_)                                                                                              \
  do {                                                                                                               \
    SDFB_CUDA(cudaFuncSetAttribute(k_tc_gemm_test<P_, TS_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    k_tc_gemm_test<P_, TS_><<<1, 288, smem, st>>>(A, (const __nv_bfloat16*)scratch, K, Np, Np64, D);                        \
  } while (0)
  if (planes == 1 && !mode_ts) LAUNCH(1, false);
  else if (planes == 1 && mode_ts) LAUNCH(1, true);
  else if (planes == 2 && !mode_ts) LAUNCH(2, false);
  else LAUNCH(2, true);
#undef LAUNCH
  SDFB_LAUNCHED("k_tc_gemm_test");
  return 0;
}

// building-block test of the generic tensor-core Linear (tc_linear.cu) against a reference GEMM: same arguments as the internal sgemm()
extern "C" int sdfb200_debug_tc_linear(int32_t planes, int32_t epi, const float* X, int32_t ldx, const float* W, const float* bias, float* Y,
                                       int32_t ldy, int64_t M, int32_t Np, int32_t Kp, const float* aux, int32_t ldaux, int32_t aux_cols,
                                       void* scratch, void* stream) {
  SDFB_REQUIRE(X && W && Y && scratch && M >= 0, "NULL pointer");
  return tc_gemm(planes, epi, X, ldx, W, bias, Y, ldy, M, Np, Kp, aux, ldaux, aux_cols, scratch, (cudaStream_t)stream);
}
