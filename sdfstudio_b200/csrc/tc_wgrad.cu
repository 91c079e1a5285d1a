// Weight-gradient GEMM of the training path on wgmma:  C[N, K] = A[P, N]^T B[P, K]   (dW = dY^T X, reduction over the P points)
// (what autograd's mm backward computes for every nn.Linear of the reference's SDFField, nerfstudio/fields/sdf_field.py:400-409,
// trained through engine/trainer.py:319-323).
//
// Persistent CTAs, each accumulating its share of the points in registers: both operands are "long" in the reduction dimension, so both
// are staged TRANSPOSED into shared memory as bf16 split planes in the canonical K-major (here: point-major) no-swizzle layout
//     element (row r, point m) -> (m/8) * LBO + r * 16 + (m%8) * 2,   LBO = rows * 16
// (global reads coalesced along the row index: 32 lanes = 32 consecutive columns of one point's row; each thread gathers 8 consecutive
// points of ONE column and writes one 16-byte unit per plane), double buffered so that the loads of the next 32 points run under the
// MMAs of the current ones.  Two warpgroups: D[n, k] += sum_m A[m, n] B[m, k] with warpgroup w owning the rows n in [64 w, 64 w + 64)
// of a 128-row chunk, N = K columns in n64 blocks, K = 16 points per instruction; bf16x3 = a0 b0 + a1 b0 + a0 b1.  The per-CTA
// partial sums go to a workspace and are reduced by a second kernel in a fixed order (deterministic, unlike atomics).
#include "tc_common.cuh"

namespace sdfb200 {
using namespace tc;

namespace {
constexpr int kWgThreads = 256;     // two warpgroups: staging + MMAs
constexpr int kWgPts = 32;          // points per stage
constexpr int kWgRowsA = 128;       // rows of the A operand tile (N chunk, zero padded): the 128-row A layout of tc_common.cuh
constexpr int kWgRowsB = 256;       // rows of the B operand tile (K chunk, zero padded)
constexpr uint32_t kWgPlaneA = (kWgPts / 8) * kWgRowsA * 16;          // 8 KB
constexpr uint32_t kWgPlaneB = (kWgPts / 8) * kWgRowsB * 16;          // 16 KB
constexpr uint32_t kWgStageBytes = 2 * (kWgPlaneA + kWgPlaneB);       // both operands, both planes

struct WgArgs {
  const float* A; long long lda;    // [P, >= n0 + Nc]
  const float* B; long long ldb;    // [P, >= k0 + Kc]
  long long P;
  int Nc, Kc;                       // rows of this (n, k) chunk: Nc <= 128, Kc <= 256
  float* partial;                   // [gridDim.x][256][256]
};

template <int PL>
__global__ void __launch_bounds__(kWgThreads, 1) k_tc_wgrad(const WgArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5;
  const long long nblk = (a.P + kWgPts - 1) / kWgPts;
  const int nch = (a.Kc + 63) / 64;
  const int wg = warp >> 2, t = tid & 127;
  const bool mma_rows = wg * 64 < a.Nc;          // warpgroup-uniform: this warpgroup's 64 rows hold live columns of A

  // thread (op, col) gathers 8 consecutive points of one column: 128 A columns + 256 B columns, 4 groups of 8 points per stage
  auto stage = [&](long long blk, uint8_t* dst) {
    const long long m0 = blk * kWgPts;
    for (int u = tid; u < (kWgRowsA + kWgRowsB) * (kWgPts / 8); u += kWgThreads) {
      const int cc = u % (kWgRowsA + kWgRowsB), g = u / (kWgRowsA + kWgRowsB);
      const bool isA = cc < kWgRowsA;
      const int col = isA ? cc : cc - kWgRowsA;
      const float* src = isA ? a.A : a.B;
      const long long ld = isA ? a.lda : a.ldb;
      const bool live = col < (isA ? a.Nc : a.Kc);
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const long long m = m0 + g * 8 + i;
        v[i] = (live && m < a.P) ? __ldg(src + m * ld + col) : 0.f;
      }
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) split2(v[2 * e], v[2 * e + 1], hi[e], lo[e]);
      const int rows = isA ? kWgRowsA : kWgRowsB;
      uint8_t* base = dst + (isA ? 0 : PL * kWgPlaneA) + (size_t)g * rows * 16 + col * 16;
      *reinterpret_cast<uint4*>(base) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
      if (PL > 1) *reinterpret_cast<uint4*>(base + (isA ? kWgPlaneA : kWgPlaneB)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
    fence_async_smem();
  };

  float acc[4][32];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
  int it = 0;
  if (blockIdx.x < nblk) stage(blockIdx.x, smem);
  __syncthreads();
  for (long long blk = blockIdx.x; blk < nblk; blk += gridDim.x, ++it) {
    uint8_t* cur = smem + (size_t)(it & 1) * kWgStageBytes;
    if (mma_rows) {
      const uint32_t abase = smem_u32(cur) + wg * 64 * 16, bbase = smem_u32(cur + PL * kWgPlaneA);
      wg_fence_acc(acc[0]); wg_fence_acc(acc[1]); wg_fence_acc(acc[2]); wg_fence_acc(acc[3]);
      wg_arrive();
#pragma unroll
      for (int j = 0; j < kWgPts / 16; ++j) {
        wgmma_kstep_ss<PL, 4>(acc, a_desc(abase, j), a_desc(abase + kWgPlaneA, j), bbase + j * 2 * kWgRowsB * 16, kWgPlaneB, kWgRowsB * 16, nch);
      }
      wg_commit();
    }
    if (blk + gridDim.x < nblk) stage(blk + gridDim.x, smem + (size_t)((it + 1) & 1) * kWgStageBytes);
    if (mma_rows) {
      wg_wait<0>();
      wg_fence_acc(acc[0]); wg_fence_acc(acc[1]); wg_fence_acc(acc[2]); wg_fence_acc(acc[3]);
    }
    __syncthreads();
  }
  // ---------------- partial sums of this CTA -> workspace (zeros for a CTA without points) ----------------
  float* out = a.partial + (size_t)blockIdx.x * 256 * 256;
  const int r0 = frag_row0(wg * 64, t), c2 = frag_cq(t);
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int n = frag_row(r0, i), k = frag_col(c2, c, i);
      if (c < nch) *reinterpret_cast<float2*>(out + (size_t)n * 256 + k) = make_float2(acc[c][i], acc[c][i + 1]);
    }
  }
}

// C[n0 + n, k0 + k] (+)= sum_g partial[g][n][k]   in a fixed order
__global__ void k_wgrad_reduce(const float* __restrict__ partial, int G, int Nc, int Kc, float* __restrict__ C, long long ldc, int accumulate) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= Nc * Kc) return;
  const int n = idx / Kc, k = idx - n * Kc;
  float acc = 0.f;
  for (int g = 0; g < G; ++g) acc += partial[(size_t)g * 65536 + n * 256 + k];
  float* c = C + (long long)n * ldc + k;
  *c = accumulate ? *c + acc : acc;
}
}  // namespace

size_t tc_wgrad_workspace_bytes() { return (size_t)kNumSMs * 256 * 256 * sizeof(float); }

// C[N, K] = A[P, N]^T B[P, K]; planes 1 = bf16, 2 = bf16x3
int tc_wgrad(int planes, const float* A, long long lda, const float* B, long long ldb, float* C, long long ldc, int64_t P, int N, int K, void* workspace,
             size_t workspace_bytes, cudaStream_t st) {
  SDFB_REQUIRE(planes == 1 || planes == 2, "tc_wgrad: planes");
  SDFB_REQUIRE(A && B && C && workspace, "tc_wgrad: NULL pointer");
  SDFB_REQUIRE(workspace_bytes >= tc_wgrad_workspace_bytes(), "tc_wgrad: workspace too small");
  SDFB_REQUIRE(N >= 1 && K >= 1 && P >= 0, "tc_wgrad: bad sizes");
  const long long nblk = (P + kWgPts - 1) / kWgPts;
  const int ctas = persistent_ctas();
  const int grid = (int)(nblk < ctas ? (nblk > 0 ? nblk : 1) : ctas);
  const size_t smem = 2 * (size_t)kWgStageBytes + 1024;
  for (int n0 = 0; n0 < N; n0 += kWgRowsA) {
    for (int k0 = 0; k0 < K; k0 += 256) {
      WgArgs a;
      a.A = A + n0; a.lda = lda; a.B = B + k0; a.ldb = ldb; a.P = P; a.Nc = N - n0 < kWgRowsA ? N - n0 : kWgRowsA; a.Kc = K - k0 < 256 ? K - k0 : 256;
      a.partial = (float*)workspace;
      if (planes == 2) {
        SDFB_CUDA(cudaFuncSetAttribute(k_tc_wgrad<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_tc_wgrad<2><<<grid, kWgThreads, smem, st>>>(a);
      } else {
        SDFB_CUDA(cudaFuncSetAttribute(k_tc_wgrad<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_tc_wgrad<1><<<grid, kWgThreads, smem, st>>>(a);
      }
      SDFB_LAUNCHED("k_tc_wgrad");
      k_wgrad_reduce<<<(a.Nc * a.Kc + 255) / 256, 256, 0, st>>>(a.partial, grid, a.Nc, a.Kc, C + (long long)n0 * ldc + k0, ldc, 0);
      SDFB_LAUNCHED("k_wgrad_reduce");
    }
  }
  return 0;
}

}  // namespace sdfb200
