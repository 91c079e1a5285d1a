// Generic tensor-core Linear for the field shapes the fused kernel does not cover (bakedsdf / angelo / stock volsdf ...):
//   Y[M, n0:n0+Nc] = epi( X[M, k0:k0+Kc] * W[n0:n0+Nc, k0:k0+Kc]^T (+ partial sums) + bias )
// One CTA per 128-row tile: two warpgroups (64 rows each) stage the fp32 activations as bf16 split planes in shared memory, one warp
// streams the pre-packed weight K-blocks through a 2-stage shared-memory ring with 1-D bulk copies, and each warpgroup runs wgmma
// m64n64k16 over its rows (bf16x3 = a0 w0 + a1 w0 + a0 w1, fp32 accumulate in registers), then applies the epilogue of k_sgemm
// (field_simt.cu) straight from the accumulator registers.
// K > 256 / N > 256 are chunked by the host wrapper (partial sums round-trip through Y).
#include "tc_common.cuh"
#include "tc_linear.h"

namespace sdfb200 {
using namespace tc;

namespace {
constexpr int kKBL = 32;          // K per streamed weight block
constexpr int kStagesL = 2;
constexpr int kThreadsL = 288;    // two MMA / epilogue warpgroups + weight producer
constexpr uint32_t kAPlaneL = 32 * 2048;                          // one plane of the A operand: [K/8 (<= 32)][128 rows][16 B]
constexpr uint32_t kRingBytesL = kStagesL * 2 * 256 * kKBL * 2;   // weight ring at its largest (2 planes, N = 256)

// one thread per packed element of every plane; see tc_pack (tc_linear.h)
__global__ void k_tc_pack(const float* __restrict__ W, int ldw, int trans, int N, int K, int Np, int kblk, int nblocks, int planes, int use_rowmap,
                          const TcIdxMap rowmap, int use_colmap, const TcIdxMap colmap, __nv_bfloat16* __restrict__ out) {
  constexpr int kMap = (int)(sizeof(TcIdxMap) / sizeof(short));
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nblocks * Np * kblk) return;
  const int kk = idx % kblk;
  const int n = (idx / kblk) % Np;
  const int b = idx / (kblk * Np);
  const int k = b * kblk + kk;
  const int ks = use_colmap ? (k < kMap ? colmap.src[k] : -1) : (k < K ? k : -1);
  const int ns = use_rowmap ? (n < kMap ? rowmap.src[n] : -1) : (n < N ? n : -1);
  const float w = (ns >= 0 && ks >= 0) ? (trans ? W[(size_t)ks * ldw + ns] : W[(size_t)ns * ldw + ks]) : 0.f;
  const __nv_bfloat16 hi = __float2bfloat16_rn(w);
  const size_t plane_elems = (size_t)Np * kblk;
  const size_t off = (size_t)b * planes * plane_elems + (size_t)(kk / 8) * (Np * 8) + (size_t)n * 8 + (kk % 8);
  out[off] = hi;
  if (planes > 1) out[off + plane_elems] = __float2bfloat16_rn(w - __bfloat162float(hi));
}

struct LinArgs {
  const float* X; int ldx; long long M;
  int Kc32, Kvalid;                 // K of this chunk rounded up to 32 / columns of X actually present
  const __nv_bfloat16* Wp; int Ncp, Np64;   // packed weights of this chunk (Np64 rows), N of this chunk (multiple of 16, <= 256)
  const float* bias;                // already offset by n0 (may be NULL)
  float* Y; int ldy; int n0;
  int accumulate, final_chunk;      // add the partial sums already in Y / apply bias + activation
  const float* aux; int ldaux, aux_cols;
};

template <int P, int EPI>
__global__ void __launch_bounds__(kThreadsL, 1) k_tc_linear(const LinArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ Handoff<kStagesL> bars;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nblocks = a.Kc32 / kKBL;
  const uint32_t stage_bytes = (uint32_t)P * a.Np64 * kKBL * 2;
  uint8_t* a_smem = smem;                               // [P][K/8][128][16 B]
  uint8_t* ring = smem + P * kAPlaneL;
  const long long m0 = (long long)blockIdx.x * 128;
  if (tid == 0) {
    bars.init(1, 2);
    fence_barrier_init();
  }
  if (tid < 256) {
    // stage A: thread (row, chunk) converts 8 consecutive columns of one row (rows fastest: conflict-free 16-byte smem stores)
    const int chunks = a.Kc32 / 8;
    for (int u = tid; u < chunks * 128; u += 256) {
      const int r = u & 127, ch = u >> 7, k = ch * 8;
      const long long m = m0 + r;
      float v[8];
      if (m < a.M && k + 8 <= a.Kvalid) {
        const float4 x0 = __ldg(reinterpret_cast<const float4*>(a.X + m * (long long)a.ldx + k));
        const float4 x1 = __ldg(reinterpret_cast<const float4*>(a.X + m * (long long)a.ldx + k + 4));
        v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w; v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = (m < a.M && k + e < a.Kvalid) ? __ldg(a.X + m * (long long)a.ldx + k + e) : 0.f;
      }
      uint32_t hi[4], lo[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) split2(v[2 * e], v[2 * e + 1], hi[e], lo[e]);
      *reinterpret_cast<uint4*>(a_smem + (size_t)ch * kAChunk + r * 16) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
      if (P > 1) *reinterpret_cast<uint4*>(a_smem + kAPlaneL + (size_t)ch * kAChunk + r * 16) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
    fence_async_smem();
  }
  __syncthreads();

  if (warp == 8) {
    // ---------------- weight producer ----------------
    if (lane == 0) {
      for (int b = 0; b < nblocks; ++b)
        ring_fill(bars, ring, b, reinterpret_cast<const uint8_t*>(a.Wp), b, stage_bytes);
    }
    return;
  }
  // ---------------- two warpgroups: MMAs over 64 rows each, then the epilogue from the accumulator registers ----------------
  const int wg = warp >> 2, t = tid & 127;
  const int rw = frag_row0(wg * 64, t), c2 = frag_cq(t);
  const int nch = a.Np64 / 64;
  float acc[4][32];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
  const uint32_t lbo_b = (uint32_t)a.Np64 * 16, plane_b = (uint32_t)a.Np64 * kKBL * 2;
  const uint32_t abase = smem_u32(a_smem) + wg * 64 * 16;
  for (int b = 0; b < nblocks; ++b) {
    bars.wait_full(b);
    const uint32_t wbase = smem_u32(ring + (size_t)bars.slot(b) * stage_bytes);
    wg_fence_acc(acc[0]); wg_fence_acc(acc[1]); wg_fence_acc(acc[2]); wg_fence_acc(acc[3]);
    wg_arrive();
#pragma unroll
    for (int j = 0; j < kKBL / 16; ++j) {
      const int kstep = b * (kKBL / 16) + j;
      wgmma_kstep_ss<P, 4>(acc, a_desc(abase, kstep), a_desc(abase + kAPlaneL, kstep), wbase + j * 2 * lbo_b, plane_b, lbo_b, nch);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(acc[0]); wg_fence_acc(acc[1]); wg_fence_acc(acc[2]); wg_fence_acc(acc[3]);
    if (t == 0) bars.arrive_empty(b);
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int n = frag_col(c2, c, i);                  // column inside this N chunk (even; n + 1 < Ncp when n < Ncp)
      const long long m = frag_row(m0 + rw, i);
      if (c < nch && n < a.Ncp && m < a.M) {
        float y[2] = {acc[c][i], acc[c][i + 1]};
        float2* yp = reinterpret_cast<float2*>(a.Y + m * (long long)a.ldy + a.n0 + n);
        if (a.accumulate) { const float2 pv = *yp; y[0] += pv.x; y[1] += pv.y; }
        if (a.final_chunk) {
          if (EPI == TCL_MUL_DSOFTPLUS) {
#pragma unroll
            for (int j = 0; j < 2; ++j)
              if (a.n0 + n + j < a.aux_cols) y[j] *= dsoftplus100_fast_from_h(__ldg(a.aux + m * (long long)a.ldaux + a.n0 + n + j));
          } else {
            const float2 bv = a.bias != nullptr ? __ldg(reinterpret_cast<const float2*>(a.bias + n)) : make_float2(0.f, 0.f);
            const float b2[2] = {bv.x, bv.y};
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              y[j] += b2[j];
              if (EPI == TCL_SOFTPLUS) y[j] = softplus100_fast(y[j]);
              if (EPI == TCL_RELU) y[j] = fmaxf(y[j], 0.f);
            }
          }
        }
        *yp = make_float2(y[0], y[1]);
      }
    }
  }
}

template <int P>
int launch_linear(int epi, const LinArgs& a, size_t smem, unsigned grid, cudaStream_t st) {
#define SDFB_TCL(E)                                                                                                  \
  do {                                                                                                               \
    SDFB_CUDA(cudaFuncSetAttribute(k_tc_linear<P, E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));      \
    k_tc_linear<P, E><<<grid, kThreadsL, smem, st>>>(a);                                                             \
  } while (0)
  switch (epi) {
    case TCL_NONE: SDFB_TCL(TCL_NONE); break;
    case TCL_SOFTPLUS: SDFB_TCL(TCL_SOFTPLUS); break;
    case TCL_RELU: SDFB_TCL(TCL_RELU); break;
    default: SDFB_TCL(TCL_MUL_DSOFTPLUS); break;
  }
#undef SDFB_TCL
  SDFB_LAUNCHED("k_tc_linear");
  return 0;
}
}  // namespace

int tc_pack(const float* W, int ldw, int trans, int N, int K, int Np, int kblk, int nblocks, int planes, const TcIdxMap* rowmap,
            const TcIdxMap* colmap, void* out, cudaStream_t st) {
  const TcIdxMap none{};
  const int tot = nblocks * Np * kblk;
  k_tc_pack<<<(tot + 255) / 256, 256, 0, st>>>(W, ldw, trans, N, K, Np, kblk, nblocks, planes, rowmap != nullptr, rowmap ? *rowmap : none,
                                               colmap != nullptr, colmap ? *colmap : none, (__nv_bfloat16*)out);
  SDFB_LAUNCHED("k_tc_pack");
  return 0;
}

int tc_gemm(int planes, int epi, const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy, int64_t M, int Np, int Kp,
            const float* aux, int ldaux, int aux_cols, void* scratch, cudaStream_t st) {
  return tc_gemm_ex(planes, epi, X, ldx, W, Kp, 0, Np, Kp, bias, Y, ldy, M, Np, Kp, aux, ldaux, aux_cols, scratch, st);
}

// general form: W is [Nw, Kw] with row stride ldw (or its transpose when trans_w), zero padded on the fly to (Np, Kp); bias may be NULL for
// TCL_NONE (no bias added)
int tc_gemm_ex(int planes, int epi, const float* X, int ldx, const float* W, int ldw, int trans_w, int Nw, int Kw, const float* bias, float* Y, int ldy,
               int64_t M, int Np, int Kp, const float* aux, int ldaux, int aux_cols, void* scratch, cudaStream_t st) {
  SDFB_REQUIRE(planes == 1 || planes == 2, "tc_gemm: planes");
  SDFB_REQUIRE(Np % 16 == 0 && Kp % 16 == 0 && ldx % 4 == 0 && ldy % 4 == 0, "tc_gemm: dims must be padded to 16");
  SDFB_REQUIRE(scratch != nullptr, "tc_gemm: scratch is NULL");
  if (M == 0) return 0;
  const unsigned grid = (unsigned)ceil_div(M, 128);
  for (int n0 = 0; n0 < Np; n0 += 256) {
    const int Nc = Np - n0 < 256 ? Np - n0 : 256;
    for (int k0 = 0; k0 < Kp; k0 += 256) {
      const int Kc = Kp - k0 < 256 ? Kp - k0 : 256;
      const int Kc32 = (Kc + 31) / 32 * 32, nblocks = Kc32 / kKBL;
      const int Np64 = (Nc + 63) / 64 * 64;
      const float* wsrc = trans_w ? W + (size_t)k0 * ldw + n0 : W + (size_t)n0 * ldw + k0;
      const int nv = Nw - n0 < Nc ? (Nw - n0 > 0 ? Nw - n0 : 0) : Nc, kv = Kw - k0 < Kc ? (Kw - k0 > 0 ? Kw - k0 : 0) : Kc;
      if (int r = tc_pack(wsrc, ldw, trans_w, nv, kv, Np64, kKBL, nblocks, planes, nullptr, nullptr, scratch, st)) return r;
      LinArgs a;
      a.X = X + k0; a.ldx = ldx; a.M = M; a.Kc32 = Kc32; a.Kvalid = kv; a.Wp = (const __nv_bfloat16*)scratch; a.Ncp = Nc; a.Np64 = Np64;
      a.bias = bias ? bias + n0 : nullptr; a.Y = Y; a.ldy = ldy; a.n0 = n0; a.accumulate = k0 > 0; a.final_chunk = k0 + 256 >= Kp;
      a.aux = aux; a.ldaux = ldaux; a.aux_cols = aux_cols;
      if (epi != TCL_MUL_DSOFTPLUS && epi != TCL_NONE) SDFB_REQUIRE(bias != nullptr, "tc_gemm: bias is NULL");
      const size_t smem = (size_t)planes * kAPlaneL + kRingBytesL + 1024;
      const int r = planes == 2 ? launch_linear<2>(epi, a, smem, grid, st) : launch_linear<1>(epi, a, smem, grid, st);
      if (r) return r;
    }
  }
  return 0;
}

}  // namespace sdfb200
