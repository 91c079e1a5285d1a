// Generic fp32 (CUDA-core) evaluation of the SDF field: any layer count / skip connection / head combination of
// SDFFieldConfig.  This is the exact-fp32 path (SDFB200_PRECISION_FP32) and the reference for the tensor-core path.
//
// Stages (each a kernel; activations live in the caller's workspace, chunked so they stay L2-resident):
//   k_field_inputs   positions (o + d*t), SceneContraction, NeRF PE           sdf_field.py:623-631, encodings.py:167-208
//   k_grid_encode    hash features (+ d feat / d x)                           sdf_field.py:384-388
//   k_sgemm<EPI>     weight-normed Linear + Softplus(beta=100) / ReLU         sdf_field.py:400-410, 586-592
//   reverse sweep    d sdf / d x by explicit back-substitution (what torch.autograd.grad computes at :647-654)
//   k_color_inputs / k_field_post   get_colors :532-612, LaplaceDensity :57-66, get_alpha :476-525
#include "field_plan.h"
#include "grid.cuh"
#include "tc_linear.h"

namespace sdfb200 {

int grid_encode(const sdfb200_grid_t& g, const void* table, const float* x01, int64_t n, float* out, int64_t out_ld,
                float* dout_dx, cudaStream_t st);
int validate_grid(const sdfb200_grid_t* g);

__constant__ float c_offaxis[3][21] = {
    {0.8506508f, 0.809017f, 0.5257311f, 1.f, 0.809017f, 0.8506508f, 0.309017f, 0.f, 0.5f, 0.f, -0.5257311f, -0.309017f, 0.f, -0.309017f, 0.309017f, 0.5f, 0.5f, 0.f, -0.5f, -0.809017f, -0.809017f},
    {0.f, 0.5f, 0.8506508f, 0.f, 0.5f, 0.f, 0.809017f, 0.5257311f, 0.309017f, 1.f, 0.8506508f, 0.809017f, 0.5257311f, 0.809017f, 0.809017f, 0.309017f, -0.309017f, 0.f, 0.309017f, 0.5f, 0.5f},
    {0.5257311f, 0.309017f, 0.f, 0.f, -0.309017f, -0.5257311f, -0.5f, -0.8506508f, -0.809017f, 0.f, 0.f, -0.5f, 0.8506508f, 0.5f, 0.5f, 0.809017f, 0.809017f, 1.f, 0.809017f, 0.309017f, -0.309017f}};

constexpr float kHalfPi = 1.5707963267948966f;

// x @ P[:, b] of the off-axis encoding -- one fixed evaluation order shared by the forward and the jacobian
__device__ __forceinline__ float offaxis_dot(float px, float py, float pz, int b) {
  return fmaf(pz, c_offaxis[2][b], fmaf(py, c_offaxis[1][b], px * c_offaxis[0][b]));
}

// -----------------------------------------------------------------------------------------------------------------
// weight packing: W = v * (g / ||v||_row)   (nn.utils.weight_norm dim=0, sdf_field.py:312-313,360-361)
// one block per output row; writes the padded [Np,Kp] matrix, its transpose [Kp,Np] and the padded bias.
// -----------------------------------------------------------------------------------------------------------------
__global__ void k_pack_layer(const float* __restrict__ v, const float* __restrict__ g, const float* __restrict__ b, int N, int K,
                             int Np, int Kp, float post_scale, float* __restrict__ W, float* __restrict__ Wt, float* __restrict__ bias) {
  const int o = blockIdx.x;  // 0..Np-1
  __shared__ float red[32];
  float scale = 0.f;
  if (o < N) {
    if (g != nullptr) {
      float ss = 0.f;
      for (int k = threadIdx.x; k < K; k += blockDim.x) {
        const float t = v[(size_t)o * K + k];
        ss = fmaf(t, t, ss);
      }
      for (int s = 16; s > 0; s >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, s);
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
      __syncthreads();
      if (threadIdx.x < 32) {
        float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        for (int s = 16; s > 0; s >>= 1) t += __shfl_xor_sync(0xffffffffu, t, s);
        if (threadIdx.x == 0) red[0] = t;
      }
      __syncthreads();
      scale = g[o] / sqrtf(red[0]);
    } else {
      scale = 1.f;
    }
  }
  for (int k = threadIdx.x; k < Kp; k += blockDim.x) {
    float w = 0.f;
    if (o < N && k < K) w = v[(size_t)o * K + k] * scale * post_scale;
    W[(size_t)o * Kp + k] = w;
    if (Wt) Wt[(size_t)k * Np + o] = w;
  }
  if (threadIdx.x == 0) bias[o] = (o < N) ? b[o] : 0.f;
}

__global__ void k_pack_heads(const float* dw, const float* db, const float* tw, const float* tb, int gf, float* out) {
  // layout: diffuse W[3*gf], b[4], tint W[3*gf], b[4]
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int per = 3 * gf + 4;
  if (i >= 2 * per) return;
  const int which = i / per, j = i % per;
  const float* w = which ? tw : dw;
  const float* b = which ? tb : db;
  float val = 0.f;
  if (w != nullptr) {
    if (j < 3 * gf) val = w[j];
    else if (j - 3 * gf < 3) val = b[j - 3 * gf];
  }
  out[i] = val;
}

// -----------------------------------------------------------------------------------------------------------------
// inputs: positions, contraction, PE.
// -----------------------------------------------------------------------------------------------------------------
struct InputArgs {
  const float* origins; const float* directions; const float* bins;
  int64_t point0, n_points; int n_samples;
  int contraction, pe_degree, use_pe, off_axis, in_pad, pe_dim, grid_dim;
  float dx, dy, dz;                 // constant offset added after contraction (numerical gradients), usually 0
  float* x; float* x01; float* in; float* points_norm; float* points_out;
};

// One WARP per point (8 points per block): lane l writes columns l, l+32, ... of the point's input row, so the 1.5 KB row leaves the
// SM as coalesced 128-byte stores (a thread-per-point layout strides the lanes by the row length: 32 L1 wavefronts per store
// instruction, and all of a row's sinf evaluations serialised in one thread).
__global__ void __launch_bounds__(256) k_field_inputs(const InputArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= a.n_points) return;
  const int64_t gi = a.point0 + i;
  float px, py, pz;
  if (a.bins != nullptr) {
    const int64_t r = gi / a.n_samples;
    const int s = (int)(gi - r * a.n_samples);
    const float t = __ldg(a.bins + r * (a.n_samples + 1) + s);
    px = __fadd_rn(__ldg(a.origins + r * 3 + 0), __fmul_rn(__ldg(a.directions + r * 3 + 0), t));
    py = __fadd_rn(__ldg(a.origins + r * 3 + 1), __fmul_rn(__ldg(a.directions + r * 3 + 1), t));
    pz = __fadd_rn(__ldg(a.origins + r * 3 + 2), __fmul_rn(__ldg(a.directions + r * 3 + 2), t));
  } else {
    px = __ldg(a.origins + gi * 3 + 0); py = __ldg(a.origins + gi * 3 + 1); pz = __ldg(a.origins + gi * 3 + 2);
  }
  if (a.contraction != SDFB200_CONTRACT_NONE) {
    // spatial_distortions.py:66-73: x <- (2 - 1/|x|) * (x/|x|) where |x| >= 1
    float mag = a.contraction == SDFB200_CONTRACT_LINF ? fmaxf(fabsf(px), fmaxf(fabsf(py), fabsf(pz)))
                                                        : sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)), __fmul_rn(pz, pz)));
    if (mag >= 1.f) {
      const float k = __fsub_rn(2.f, __fdiv_rn(1.f, mag));
      px = __fmul_rn(k, __fdiv_rn(px, mag)); py = __fmul_rn(k, __fdiv_rn(py, mag)); pz = __fmul_rn(k, __fdiv_rn(pz, mag));
    }
  }
  if (lane == 0) {
    if (a.points_norm) a.points_norm[gi] = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)), __fmul_rn(pz, pz)));
    if (a.points_out) { a.points_out[gi * 3] = px; a.points_out[gi * 3 + 1] = py; a.points_out[gi * 3 + 2] = pz; }
  }
  px += a.dx; py += a.dy; pz += a.dz;
  if (lane < 3) {
    const float v = lane == 0 ? px : (lane == 1 ? py : pz);
    a.x[i * 3 + lane] = v;
    a.x01[i * 3 + lane] = (v + 2.0f) * 0.25f;
  }
  float* row = a.in + i * a.in_pad;
  const int nb = a.off_axis ? 21 : 3;
  const int half = nb * a.pe_degree;
  for (int c = lane; c < a.in_pad; c += 32) {
    float val = 0.f;                                       // grid block (overwritten by k_grid_encode) + padding
    if (c < 3) val = c == 0 ? px : (c == 1 ? py : pz);
    else if (c < 3 + a.pe_dim) {
      const int j = c - 3;
      const int jj = j >= half ? j - half : j;
      const int b2 = jj / a.pe_degree, k = jj - b2 * a.pe_degree;
      const float v = a.off_axis ? offaxis_dot(px, py, pz, b2) : (b2 == 0 ? px : (b2 == 1 ? py : pz));
      const float sarg = v * (float)(1 << k);
      val = a.use_pe ? sinf(j >= half ? sarg + kHalfPi : sarg) : 0.f;
    }
    row[c] = val;
  }
}

// -----------------------------------------------------------------------------------------------------------------
// fp32 tile GEMM:  Y[M, Np] = epi( X[M, Kp] * W[Np, Kp]^T + bias )        128x128x16 tiles, 8x8 per thread
// -----------------------------------------------------------------------------------------------------------------
enum { EPI_NONE = 0, EPI_SOFTPLUS = 1, EPI_RELU = 2, EPI_MUL_DSOFTPLUS = 3 };

template <int EPI>
__global__ void __launch_bounds__(256) k_sgemm(const float* __restrict__ X, int ldx, const float* __restrict__ W, const float* __restrict__ bias,
                                               float* __restrict__ Y, int ldy, int64_t M, int Np, int Kp, const float* __restrict__ aux,
                                               int ldaux, int aux_cols) {
  constexpr int BM = 128, BN = 128, BK = 16, PADS = 4;
  __shared__ __align__(16) float Xs[BK][BM + PADS];
  __shared__ __align__(16) float Ws[BK][BN + PADS];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < Kp; k0 += BK) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int id = t + j * 256, row = id >> 2, kq = id & 3;
      float4 xv = make_float4(0.f, 0.f, 0.f, 0.f), wv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m0 + row < M) xv = __ldg(reinterpret_cast<const float4*>(X + (m0 + row) * ldx + k0 + kq * 4));
      if (n0 + row < Np) wv = __ldg(reinterpret_cast<const float4*>(W + (size_t)(n0 + row) * Kp + k0 + kq * 4));
      Xs[kq * 4 + 0][row] = xv.x; Xs[kq * 4 + 1][row] = xv.y; Xs[kq * 4 + 2][row] = xv.z; Xs[kq * 4 + 3][row] = xv.w;
      Ws[kq * 4 + 0][row] = wv.x; Ws[kq * 4 + 1][row] = wv.y; Ws[kq * 4 + 2][row] = wv.z; Ws[kq * 4 + 3][row] = wv.w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&Xs[k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&Xs[k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Ws[k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Ws[k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int n = n0 + jh * 64 + tx * 4;
      if (n >= Np) continue;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float y = acc[i][jh * 4 + j];
        if (EPI != EPI_MUL_DSOFTPLUS) y += __ldg(bias + n + j);
        if (EPI == EPI_SOFTPLUS) y = softplus100(y);
        if (EPI == EPI_RELU) y = fmaxf(y, 0.f);
        if (EPI == EPI_MUL_DSOFTPLUS) {
          if (n + j < aux_cols) y *= dsoftplus100_from_h(__ldg(aux + m * ldaux + n + j));
        }
        v[j] = y;
      }
      *reinterpret_cast<float4*>(Y + m * ldy + n) = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
}

// GEMM engine of the current field call: 0 planes = the exact-fp32 CUDA-core kernel below; 1 / 2 = the generic tensor-core Linear
// (bf16 / bf16x3, csrc/tc_linear.cu) with `scratch` for its packed weight chunk.  Set by field_forward_fp32 for the duration of a call.
struct GemmEngine { int planes; void* scratch; };
static thread_local GemmEngine g_gemm = {0, nullptr};

static int sgemm(int epi, const float* X, int ldx, const float* W, const float* bias, float* Y, int ldy, int64_t M, int Np, int Kp,
                 const float* aux, int ldaux, int aux_cols, cudaStream_t st) {
  if (g_gemm.planes > 0) return tc_gemm(g_gemm.planes, epi, X, ldx, W, bias, Y, ldy, M, Np, Kp, aux, ldaux, aux_cols, g_gemm.scratch, st);
  dim3 grid((unsigned)ceil_div(M, 128), (unsigned)ceil_div(Np, 128));
  switch (epi) {
    case EPI_NONE: k_sgemm<EPI_NONE><<<grid, 256, 0, st>>>(X, ldx, W, bias, Y, ldy, M, Np, Kp, aux, ldaux, aux_cols); break;
    case EPI_SOFTPLUS: k_sgemm<EPI_SOFTPLUS><<<grid, 256, 0, st>>>(X, ldx, W, bias, Y, ldy, M, Np, Kp, aux, ldaux, aux_cols); break;
    case EPI_RELU: k_sgemm<EPI_RELU><<<grid, 256, 0, st>>>(X, ldx, W, bias, Y, ldy, M, Np, Kp, aux, ldaux, aux_cols); break;
    default: k_sgemm<EPI_MUL_DSOFTPLUS><<<grid, 256, 0, st>>>(X, ldx, W, bias, Y, ldy, M, Np, Kp, aux, ldaux, aux_cols); break;
  }
  SDFB_LAUNCHED("k_sgemm");
  return 0;
}

// copy `ncols` columns (src[:, src_col0:]) into dst[:, dst_col0:], zero dst[:, dst_col0+ncols : dst_ld)
__global__ void k_copy_cols(const float* __restrict__ src, int src_ld, int src_col0, float* __restrict__ dst, int dst_ld, int dst_col0,
                            int ncols, int64_t M, int zero_tail) {
  const int64_t m = blockIdx.x;
  for (int c = threadIdx.x; c < dst_ld - dst_col0; c += blockDim.x) {
    if (c < ncols) dst[m * dst_ld + dst_col0 + c] = src[m * src_ld + src_col0 + c];
    else if (zero_tail) dst[m * dst_ld + dst_col0 + c] = 0.f;
  }
}
// dst[:, :ncols] += src[:, src_col0 : src_col0+ncols]
__global__ void k_add_cols(const float* __restrict__ src, int src_ld, int src_col0, float* __restrict__ dst, int dst_ld, int ncols, int64_t M) {
  const int64_t m = blockIdx.x;
  for (int c = threadIdx.x; c < ncols; c += blockDim.x) dst[m * dst_ld + c] += src[m * src_ld + src_col0 + c];
}

// seed of the reverse sweep: dz_{n-2}[m][j] = W_last[0][j] * softplus'(z_{n-2})   (d sdf / d a_{n-1} = row 0 of W_last)
__global__ void k_grad_seed(const float* __restrict__ w_row0, const float* __restrict__ H, int ldh, int ncols, int aux_cols, float* __restrict__ G,
                            int ldg, int64_t M) {
  const int64_t m = blockIdx.x;
  for (int c = threadIdx.x; c < ldg; c += blockDim.x) {
    float v = 0.f;
    if (c < ncols) {
      v = w_row0[c];
      if (c < aux_cols) v *= dsoftplus100_from_h(H[m * ldh + c]);
    }
    G[m * ldg + c] = v;
  }
}

// -----------------------------------------------------------------------------------------------------------------
// d sdf/dx from d sdf/d(inputs):  x part + PE jacobian + grid jacobian / 4
// -----------------------------------------------------------------------------------------------------------------
struct GradArgs {
  const float* gin; const float* in; const float* jac; int in_pad, pe_degree, use_pe, off_axis, pe_dim, grid_dim, use_grid;
  int64_t n; float* grad;
};
// one warp per point: lane l owns input columns l, l+32, ...; three warp reductions at the end
__global__ void __launch_bounds__(256) k_grad_finish(const GradArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= a.n) return;
  const float* g = a.gin + i * a.in_pad;
  const float* in = a.in + i * a.in_pad;
  const float x0 = in[0], x1 = in[1], x2 = in[2];
  float gx = 0.f, gy = 0.f, gz = 0.f;
  if (lane < 3) { const float v = g[lane]; gx = lane == 0 ? v : 0.f; gy = lane == 1 ? v : 0.f; gz = lane == 2 ? v : 0.f; }
  if (a.use_pe) {
    const int nb = a.off_axis ? 21 : 3;
    const int half = nb * a.pe_degree;
    for (int j = lane; j < a.pe_dim; j += 32) {
      const int jj = j >= half ? j - half : j;
      const int b = jj / a.pe_degree, k = jj - b * a.pe_degree;
      const float v = a.off_axis ? offaxis_dot(x0, x1, x2, b) : (b == 0 ? x0 : (b == 1 ? x1 : x2));
      const float fr = (float)(1 << k);
      const float sarg = v * fr;
      // autograd of sin(s) and sin(u), u = fl(s + pi/2): cos evaluated on the SAME fp32 arguments as the forward
      const float t = fr * g[3 + j] * cosf(j >= half ? sarg + kHalfPi : sarg);
      if (a.off_axis) { gx = fmaf(t, c_offaxis[0][b], gx); gy = fmaf(t, c_offaxis[1][b], gy); gz = fmaf(t, c_offaxis[2][b], gz); }
      else if (b == 0) gx += t; else if (b == 1) gy += t; else gz += t;
    }
  }
  if (a.use_grid) {
    const float* J = a.jac + i * (int64_t)a.grid_dim * 3;
    float jx = 0.f, jy = 0.f, jz = 0.f;
    for (int c = lane; c < a.grid_dim; c += 32) {
      const float gv = g[3 + a.pe_dim + c];
      jx = fmaf(gv, J[c * 3], jx); jy = fmaf(gv, J[c * 3 + 1], jy); jz = fmaf(gv, J[c * 3 + 2], jz);
    }
    gx += 0.25f * jx; gy += 0.25f * jy; gz += 0.25f * jz;  // positions = (x + 2) / 4   (sdf_field.py:384)
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    gx += __shfl_xor_sync(0xffffffffu, gx, d); gy += __shfl_xor_sync(0xffffffffu, gy, d); gz += __shfl_xor_sync(0xffffffffu, gz, d);
  }
  if (lane == 0) { a.grad[i * 3] = gx; a.grad[i * 3 + 1] = gy; a.grad[i * 3 + 2] = gz; }
}

// numerical gradient from the 6 offset SDFs (sdf_field.py:446-453)
__global__ void k_numgrad(const float* __restrict__ nsdf, float delta, int64_t n, float* __restrict__ grad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* s = nsdf + i * 6;
  grad[i * 3 + 0] = __fdiv_rn(__fmul_rn(0.5f, __fsub_rn(s[0], s[1])), delta);
  grad[i * 3 + 1] = __fdiv_rn(__fmul_rn(0.5f, __fsub_rn(s[2], s[3])), delta);
  grad[i * 3 + 2] = __fdiv_rn(__fmul_rn(0.5f, __fsub_rn(s[4], s[5])), delta);
}
__global__ void k_store_col(const float* __restrict__ src, int ld, int64_t n, float* __restrict__ dst, int dst_ld, int dst_col) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i * dst_ld + dst_col] = src[i * ld];
}

// -----------------------------------------------------------------------------------------------------------------
// colour-network input (sdf_field.py:541-584)
// -----------------------------------------------------------------------------------------------------------------
struct ColorInArgs {
  const float* x; const float* directions; const float* grad; const float* outg; int ldoutg; const float* appearance;
  int64_t point0, n; int n_samples; int has_bins; int geo_feat, app_dim, use_diffuse, use_reflections, use_n_dot_v, cin_pad;
  float* cin;
};
// one warp per point: lane l writes columns l, l+32, ... of the colour-network input row (coalesced; the 256-wide geo feature copy
// is a row-to-row copy)
__global__ void __launch_bounds__(256) k_color_inputs(const ColorInArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= a.n) return;
  const int64_t gi = a.point0 + i;
  const int64_t r = a.has_bins ? gi / a.n_samples : gi;
  const float dx = __ldg(a.directions + r * 3), dy = __ldg(a.directions + r * 3 + 1), dz = __ldg(a.directions + r * 3 + 2);
  const float gx = a.grad[i * 3], gy = a.grad[i * 3 + 1], gz = a.grad[i * 3 + 2];
  // F.normalize(p=2, eps=1e-12)
  const float nrm = fmaxf(sqrtf(gx * gx + gy * gy + gz * gz), 1e-12f);
  const float nx = gx / nrm, ny = gy / nrm, nz = gz / nrm;
  float ex = dx, ey = dy, ez = dz;
  if (a.use_reflections) {
    const float dot = 2.0f * (nx * -dx + ny * -dy + nz * -dz);
    ex = dot * nx + dx; ey = dot * ny + dy; ez = dot * nz + dz;
  }
  float* row = a.cin + i * a.cin_pad;
  const int c_enc = a.use_diffuse ? 0 : 3;                  // x(3) first unless the diffuse head is on
  const int c_grad = c_enc + 27;                            // gradient(3) unless the diffuse head is on
  const int c_gf = c_grad + (a.use_diffuse ? 0 : 3);
  const int c_app = c_gf + a.geo_feat;
  const int c_ndv = c_app + a.app_dim;
  const float* gf = a.outg + i * a.ldoutg + 1;
  for (int c = lane; c < a.cin_pad; c += 32) {
    float val = 0.f;
    if (c < c_enc) val = a.x[i * 3 + c];
    else if (c < c_enc + 24) {
      const int j = c - c_enc;
      const int jj = j >= 12 ? j - 12 : j;
      const int b = jj >> 2, k = jj & 3;
      const float e = b == 0 ? ex : (b == 1 ? ey : ez);
      const float arg = e * (float)(1 << k);
      val = sinf(j >= 12 ? arg + kHalfPi : arg);
    } else if (c < c_enc + 27) { const int j = c - c_enc - 24; val = j == 0 ? ex : (j == 1 ? ey : ez); }
    else if (c < c_gf) { const int j = c - c_grad; val = j == 0 ? gx : (j == 1 ? gy : gz); }
    else if (c < c_app) val = gf[c - c_gf];
    else if (c < c_ndv) val = a.appearance ? __ldg(a.appearance + r * a.app_dim + (c - c_app)) : 0.f;
    else if (c == c_ndv && a.use_n_dot_v) val = nx * dx + ny * dy + nz * dz;
    row[c] = val;
  }
}

// -----------------------------------------------------------------------------------------------------------------
// per-point heads: rgb, density, alpha, occupancy, normals
// -----------------------------------------------------------------------------------------------------------------
struct PostArgs {
  const float* outg; int ldoutg; const float* grad; const float* craw; int ldc; const float* heads; const float* directions; const float* bins;
  int64_t point0, n; int n_samples; int geo_feat, use_diffuse, use_tint; float rgb_padding;
  const float* variance; const float* beta; const float* beta_min; float cos_anneal;
  float *sdf, *geo_feature, *gradients, *normals, *rgb, *density, *alpha, *occupancy;
};
// one warp per point: the geo-feature copy and the six 256-wide head dot products (diffuse / tint, sdf_field.py:596-607) are split over
// the lanes; the scalar heads are finished by lane 0
__global__ void __launch_bounds__(256) k_field_post(const PostArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= a.n) return;
  const int64_t gi = a.point0 + i;
  const float sdf = a.outg[i * a.ldoutg];
  const float* gf = a.outg + i * a.ldoutg + 1;
  if (a.geo_feature)
    for (int k = lane; k < a.geo_feat; k += 32) a.geo_feature[gi * a.geo_feat + k] = gf[k];
  float hd[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (a.rgb && a.use_diffuse) {
    const int per = 3 * a.geo_feat + 4;
    for (int k = lane; k < a.geo_feat; k += 32) {
      const float f = gf[k];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        hd[c] = fmaf(__ldg(a.heads + c * a.geo_feat + k), f, hd[c]);
        if (a.use_tint) hd[3 + c] = fmaf(__ldg(a.heads + per + c * a.geo_feat + k), f, hd[3 + c]);
      }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1)
#pragma unroll
      for (int c = 0; c < 6; ++c) hd[c] += __shfl_xor_sync(0xffffffffu, hd[c], d);
  }
  if (lane != 0) return;
  if (a.sdf) a.sdf[gi] = sdf;
  float gx = 0.f, gy = 0.f, gz = 0.f;
  if (a.grad) { gx = a.grad[i * 3]; gy = a.grad[i * 3 + 1]; gz = a.grad[i * 3 + 2]; }
  if (a.gradients) { a.gradients[gi * 3] = gx; a.gradients[gi * 3 + 1] = gy; a.gradients[gi * 3 + 2] = gz; }
  if (a.normals) {
    const float nrm = fmaxf(sqrtf(gx * gx + gy * gy + gz * gz), 1e-12f);
    a.normals[gi * 3] = gx / nrm; a.normals[gi * 3 + 1] = gy / nrm; a.normals[gi * 3 + 2] = gz / nrm;
  }
  if (a.rgb) {
    float rgb[3];
    for (int c = 0; c < 3; ++c) rgb[c] = sigmoidf_(a.craw[i * a.ldc + c]);
    if (a.use_diffuse) {
      // sdf_field.py:596-607
      const int per = 3 * a.geo_feat + 4;
      for (int c = 0; c < 3; ++c) {
        const float rd = hd[c] + a.heads[3 * a.geo_feat + c];
        const float diffuse = sigmoidf_(rd - 1.0986122886681098f);  // log(3)
        const float spec = a.use_tint ? sigmoidf_(hd[3 + c] + a.heads[per + 3 * a.geo_feat + c]) * rgb[c] : 0.5f * rgb[c];
        rgb[c] = fminf(fmaxf(spec + diffuse, 0.f), 1.f);
      }
    }
    for (int c = 0; c < 3; ++c) a.rgb[gi * 3 + c] = rgb[c] * (1.f + 2.f * a.rgb_padding) - a.rgb_padding;
  }
  if (a.density) {
    // LaplaceDensity.forward, sdf_field.py:57-71
    const float beta = fabsf(__ldg(a.beta)) + __ldg(a.beta_min);
    const float al = 1.0f / beta;
    const float sg = sdf > 0.f ? 1.f : (sdf < 0.f ? -1.f : 0.f);
    a.density[gi] = al * (0.5f + 0.5f * sg * expm1f(-fabsf(sdf) / beta));
  }
  if (a.occupancy) a.occupancy[gi] = sigmoidf_(-10.0f * sdf);
  if (a.alpha) {
    // get_alpha, sdf_field.py:494-517
    const int64_t r = gi / a.n_samples;
    const int s = (int)(gi - r * a.n_samples);
    const float dxr = __ldg(a.directions + r * 3), dyr = __ldg(a.directions + r * 3 + 1), dzr = __ldg(a.directions + r * 3 + 2);
    const float delta = __fsub_rn(__ldg(a.bins + r * (a.n_samples + 1) + s + 1), __ldg(a.bins + r * (a.n_samples + 1) + s));
    const float inv_s = fminf(fmaxf(expf(__ldg(a.variance) * 10.0f), 1e-6f), 1e6f);
    const float true_cos = dxr * gx + dyr * gy + dzr * gz;
    const float ratio = a.cos_anneal;
    const float iter_cos = -(fmaxf(-true_cos * 0.5f + 0.5f, 0.f) * (1.0f - ratio) + fmaxf(-true_cos, 0.f) * ratio);
    const float est_next = sdf + iter_cos * delta * 0.5f;
    const float est_prev = sdf - iter_cos * delta * 0.5f;
    const float prev_cdf = sigmoidf_(est_prev * inv_s), next_cdf = sigmoidf_(est_next * inv_s);
    const float p = prev_cdf - next_cdf, c = prev_cdf;
    a.alpha[gi] = fminf(fmaxf((p + 1e-5f) / (c + 1e-5f), 0.f), 1.f);
  }
}

// -----------------------------------------------------------------------------------------------------------------
// host orchestration
// -----------------------------------------------------------------------------------------------------------------
int field_pack_fp32(const sdfb200_field_t& f, const FieldPlan& p, const sdfb200_field_params_t& prm, char* blob, cudaStream_t st) {
  for (int l = 0; l < p.n_geo; ++l) {
    const LayerPlan& L = p.geo[l];
    SDFB_REQUIRE(prm.geo_weight_v[l] && prm.geo_bias[l], "geo layer parameter pointer is NULL");
    const float post = (l == f.geo_skip_layer) ? 0.70710678118654752440f : 1.f;
    k_pack_layer<<<L.Np, 128, 0, st>>>(prm.geo_weight_v[l], prm.geo_weight_g[l], prm.geo_bias[l], L.N, L.K, L.Np, L.Kp, post,
                                       (float*)(blob + L.w_off), (float*)(blob + L.wt_off), (float*)(blob + L.b_off));
    SDFB_LAUNCHED("k_pack_layer");
  }
  for (int l = 0; l < p.n_col; ++l) {
    const LayerPlan& L = p.col[l];
    SDFB_REQUIRE(prm.color_weight_v[l] && prm.color_bias[l], "colour layer parameter pointer is NULL");
    k_pack_layer<<<L.Np, 128, 0, st>>>(prm.color_weight_v[l], prm.color_weight_g[l], prm.color_bias[l], L.N, L.K, L.Np, L.Kp, 1.f,
                                       (float*)(blob + L.w_off), nullptr, (float*)(blob + L.b_off));
    SDFB_LAUNCHED("k_pack_layer");
  }
  if (p.head_off != (size_t)-1) {
    if (f.use_diffuse_color) SDFB_REQUIRE(prm.diffuse_weight && prm.diffuse_bias, "diffuse head parameters are NULL");
    if (f.use_specular_tint) SDFB_REQUIRE(prm.tint_weight && prm.tint_bias, "tint head parameters are NULL");
    const int tot = 2 * (3 * p.geo_feat + 4);
    k_pack_heads<<<(tot + 255) / 256, 256, 0, st>>>(prm.diffuse_weight, prm.diffuse_bias, prm.tint_weight, prm.tint_bias, p.geo_feat,
                                                    (float*)(blob + p.head_off));
    SDFB_LAUNCHED("k_pack_heads");
  }
  return 0;
}

// geo network forward on `n` points whose inputs are already in ws.in; keeps hidden activations in ws.h[].
static int geo_forward(const sdfb200_field_t& f, const FieldPlan& p, const FieldWorkspace& w, float* ws, const char* blob, int64_t n,
                       cudaStream_t st) {
  const float* X = ws + w.in;
  int ldx = p.in_pad;
  for (int l = 0; l < p.n_geo; ++l) {
    const LayerPlan& L = p.geo[l];
    const bool last = l == p.n_geo - 1;
    float* Y = last ? ws + w.outg : ws + w.h[l];
    const int ldy = last ? L.Np : ((l + 1 == f.geo_skip_layer) ? p.geo[l + 1].Kp : L.Np);
    int r = sgemm(last ? EPI_NONE : EPI_SOFTPLUS, X, ldx, (const float*)(blob + L.w_off), (const float*)(blob + L.b_off), Y, ldy, n, L.Np, L.Kp,
                  nullptr, 0, 0, st);
    if (r) return r;
    if (l + 1 == f.geo_skip_layer) {
      // x = cat([x, inputs], 1) / sqrt(2)  (sdf_field.py:403-404; the 1/sqrt(2) is folded into the next weight)
      k_copy_cols<<<(unsigned)n, 64, 0, st>>>(ws + w.in, p.in_pad, 0, Y, ldy, L.N, p.in_dim, n, 1);
      SDFB_LAUNCHED("k_copy_cols");
    }
    X = Y;
    ldx = ldy;
  }
  return 0;
}

// reverse sweep: d sdf / d inputs -> ws.gin
static int geo_backward_inputs(const sdfb200_field_t& f, const FieldPlan& p, const FieldWorkspace& w, float* ws, const char* blob, int64_t n,
                               cudaStream_t st) {
  const int nl = p.n_geo;
  float* G = ws + w.g0;
  float* G2 = ws + w.g1;
  float* skipgrad = ws + w.c1;  // colour buffers are idle during the sweep
  bool have_skip = false;
  if (nl == 1) {
    // sdf = W0[0,:] . inputs + b : gradient w.r.t. inputs is row 0 of W0
    k_grad_seed<<<(unsigned)n, 64, 0, st>>>((const float*)(blob + p.geo[0].w_off), nullptr, 0, p.geo[0].K, 0, ws + w.gin, p.in_pad, n);
    SDFB_LAUNCHED("k_grad_seed");
    return 0;
  }
  // delta a_{nl-1} = row 0 of W_{nl-1}; it is the (possibly concatenated) input of the last layer
  {
    const LayerPlan& L = p.geo[nl - 1];
    const int l = nl - 1;
    const bool skip = l == f.geo_skip_layer;
    const int hcols = p.geo[l - 1].N;  // softplus outputs feeding this layer
    const int ldh = skip ? L.Kp : p.geo[l - 1].Np;
    k_grad_seed<<<(unsigned)n, 128, 0, st>>>((const float*)(blob + L.w_off), ws + w.h[l - 1], ldh, L.K, hcols, G, L.Kp, n);
    SDFB_LAUNCHED("k_grad_seed");
    if (skip) {
      k_copy_cols<<<(unsigned)n, 64, 0, st>>>(G, L.Kp, hcols, skipgrad, p.in_pad, 0, p.in_dim, n, 1);
      SDFB_LAUNCHED("k_copy_cols");
      have_skip = true;
    }
  }
  int ldg = p.geo[nl - 1].Kp;
  for (int l = nl - 2; l >= 1; --l) {
    // G holds dz_l (first N_l columns meaningful, K dim = Np_l); da_l = W_l^T dz_l ; dz_{l-1} = da_l[:N_{l-1}] * softplus'(h_{l-1})
    const LayerPlan& L = p.geo[l];
    const bool skip = l == f.geo_skip_layer;
    const int hcols = p.geo[l - 1].N;
    const int ldh = skip ? L.Kp : p.geo[l - 1].Np;
    int r = sgemm(EPI_MUL_DSOFTPLUS, G, ldg, (const float*)(blob + L.wt_off), nullptr, G2, L.Kp, n, L.Kp, L.Np, ws + w.h[l - 1], ldh, hcols, st);
    if (r) return r;
    if (skip) {
      k_copy_cols<<<(unsigned)n, 64, 0, st>>>(G2, L.Kp, hcols, skipgrad, p.in_pad, 0, p.in_dim, n, 1);
      SDFB_LAUNCHED("k_copy_cols");
      have_skip = true;
    }
    float* t = G; G = G2; G2 = t;
    ldg = L.Kp;
  }
  {
    const LayerPlan& L = p.geo[0];
    int r = sgemm(EPI_MUL_DSOFTPLUS, G, ldg, (const float*)(blob + L.wt_off), nullptr, ws + w.gin, p.in_pad, n, L.Kp, L.Np, nullptr, 0, 0, st);
    if (r) return r;
  }
  if (have_skip) {
    k_add_cols<<<(unsigned)n, 64, 0, st>>>(skipgrad, p.in_pad, 0, ws + w.gin, p.in_pad, p.in_dim, n);
    SDFB_LAUNCHED("k_add_cols");
  }
  return 0;
}

int field_forward_fp32(const sdfb200_field_t& f, const FieldPlan& p, const char* blob, const void* table, const sdfb200_field_in_t& in,
                       const sdfb200_field_out_t& out, float* ws, size_t ws_floats, cudaStream_t st, int gemm_planes) {
  const int64_t N = in.n_rays * (int64_t)in.n_samples;
  if (N == 0) return 0;
  struct EngineScope {   // restores the exact-fp32 engine on every exit path
    ~EngineScope() { g_gemm = {0, nullptr}; }
  } engine_scope;
  const int64_t chunk = N < kChunkPoints ? N : kChunkPoints;
  FieldWorkspace w;
  make_workspace_plan(f, p, chunk, w);
  if (ws_floats < w.floats_per_chunk) return fail(SDFB200_EWORKSPACE, "workspace too small%s (need %lld floats)", "", (long long)w.floats_per_chunk);
  g_gemm = {gemm_planes, ws + w.tcw};

  const bool want_color = out.rgb != nullptr;
  const bool want_grad = want_color || out.gradients || out.normals || out.alpha;
  const bool numerical = f.use_numerical_gradients != 0;
  if (want_color || out.alpha) SDFB_REQUIRE(in.directions != nullptr, "directions required for rgb / alpha");
  if (out.alpha) SDFB_REQUIRE(in.bins != nullptr && in.variance != nullptr, "alpha needs bins and the variance parameter");
  if (out.density) SDFB_REQUIRE(in.beta != nullptr && in.beta_min != nullptr, "density needs beta and beta_min");
  if (out.sampled_sdf) SDFB_REQUIRE(numerical, "sampled_sdf is only produced with use_numerical_gradients");
  const int use_grid = f.use_grid_feature;

  for (int64_t p0 = 0; p0 < N; p0 += chunk) {
    const int64_t n = (N - p0) < chunk ? (N - p0) : chunk;
    const unsigned pb = (unsigned)ceil_div(n, 256);
    const unsigned wb = (unsigned)ceil_div(n, 8);     // warp-per-point kernels: 8 points per 256-thread block
    InputArgs ia;
    ia.origins = in.origins; ia.directions = in.directions; ia.bins = in.bins; ia.point0 = p0; ia.n_points = n; ia.n_samples = in.n_samples;
    ia.contraction = in.apply_contraction ? f.contraction : SDFB200_CONTRACT_NONE;
    ia.pe_degree = f.pe_degree; ia.use_pe = f.use_position_encoding; ia.off_axis = f.off_axis; ia.in_pad = p.in_pad; ia.pe_dim = p.pe_dim;
    ia.grid_dim = p.grid_dim; ia.dx = ia.dy = ia.dz = 0.f;
    ia.x = ws + w.x; ia.x01 = ws + w.x01; ia.in = ws + w.in; ia.points_norm = out.points_norm; ia.points_out = out.points;

    if (numerical && want_grad) {
      // sdf_field.py:430-453: six offset evaluations in contracted space
      const float d = in.numerical_delta;
      const float offs[6][3] = {{d, 0, 0}, {-d, 0, 0}, {0, d, 0}, {0, -d, 0}, {0, 0, d}, {0, 0, -d}};
      for (int k = 0; k < 6; ++k) {
        InputArgs ib = ia;
        ib.dx = offs[k][0]; ib.dy = offs[k][1]; ib.dz = offs[k][2];
        ib.points_norm = nullptr; ib.points_out = nullptr;
        k_field_inputs<<<wb, 256, 0, st>>>(ib);
        SDFB_LAUNCHED("k_field_inputs");
        if (use_grid) {
          int r = grid_encode(f.grid, table, ws + w.x01, n, ws + w.in + 3 + p.pe_dim, p.in_pad, nullptr, st);
          if (r) return r;
        }
        int r = geo_forward(f, p, w, ws, blob, n, st);
        if (r) return r;
        k_store_col<<<pb, 256, 0, st>>>(ws + w.outg, p.geo[p.n_geo - 1].Np, n, ws + w.nsdf, 6, k);
        SDFB_LAUNCHED("k_store_col");
      }
      k_numgrad<<<pb, 256, 0, st>>>(ws + w.nsdf, d, n, ws + w.grad);
      SDFB_LAUNCHED("k_numgrad");
      if (out.sampled_sdf) SDFB_CUDA(cudaMemcpyAsync(out.sampled_sdf + p0 * 6, ws + w.nsdf, (size_t)n * 6 * 4, cudaMemcpyDeviceToDevice, st));
    }
    k_field_inputs<<<wb, 256, 0, st>>>(ia);
    SDFB_LAUNCHED("k_field_inputs");
    const bool analytic = want_grad && !numerical;
    if (use_grid) {
      int r = grid_encode(f.grid, table, ws + w.x01, n, ws + w.in + 3 + p.pe_dim, p.in_pad, analytic ? ws + w.jac : nullptr, st);
      if (r) return r;
    }
    int r = geo_forward(f, p, w, ws, blob, n, st);
    if (r) return r;
    if (analytic) {
      r = geo_backward_inputs(f, p, w, ws, blob, n, st);
      if (r) return r;
      GradArgs ga;
      ga.gin = ws + w.gin; ga.in = ws + w.in; ga.jac = ws + w.jac; ga.in_pad = p.in_pad; ga.pe_degree = f.pe_degree; ga.use_pe = f.use_position_encoding;
      ga.off_axis = f.off_axis; ga.pe_dim = p.pe_dim; ga.grid_dim = p.grid_dim; ga.use_grid = use_grid; ga.n = n; ga.grad = ws + w.grad;
      k_grad_finish<<<wb, 256, 0, st>>>(ga);
      SDFB_LAUNCHED("k_grad_finish");
    }
    const float* craw = nullptr;
    int ldc = 0;
    if (want_color) {
      ColorInArgs ca;
      ca.x = ws + w.x; ca.directions = in.directions; ca.grad = ws + w.grad; ca.outg = ws + w.outg; ca.ldoutg = p.geo[p.n_geo - 1].Np;
      ca.appearance = in.appearance; ca.point0 = p0; ca.n = n; ca.n_samples = in.n_samples; ca.has_bins = in.bins != nullptr; ca.geo_feat = p.geo_feat;
      ca.app_dim = f.appearance_dim; ca.use_diffuse = f.use_diffuse_color; ca.use_reflections = f.use_reflections; ca.use_n_dot_v = f.use_n_dot_v;
      ca.cin_pad = p.cin_pad; ca.cin = ws + w.cin;
      k_color_inputs<<<wb, 256, 0, st>>>(ca);
      SDFB_LAUNCHED("k_color_inputs");
      const float* X = ws + w.cin;
      int ldx = p.cin_pad;
      float* bufs[2] = {ws + w.c0, ws + w.c1};
      for (int l = 0; l < p.n_col; ++l) {
        const LayerPlan& L = p.col[l];
        const bool last = l == p.n_col - 1;
        float* Y = bufs[l & 1];
        r = sgemm(last ? EPI_NONE : EPI_RELU, X, ldx, (const float*)(blob + L.w_off), (const float*)(blob + L.b_off), Y, L.Np, n, L.Np, L.Kp, nullptr, 0, 0, st);
        if (r) return r;
        X = Y; ldx = L.Np;
      }
      craw = X; ldc = ldx;
    }
    PostArgs pa;
    pa.outg = ws + w.outg; pa.ldoutg = p.geo[p.n_geo - 1].Np; pa.grad = want_grad ? ws + w.grad : nullptr; pa.craw = craw; pa.ldc = ldc;
    pa.heads = p.head_off != (size_t)-1 ? (const float*)(blob + p.head_off) : nullptr; pa.directions = in.directions; pa.bins = in.bins;
    pa.point0 = p0; pa.n = n; pa.n_samples = in.n_samples; pa.geo_feat = p.geo_feat; pa.use_diffuse = f.use_diffuse_color; pa.use_tint = f.use_specular_tint;
    pa.rgb_padding = f.rgb_padding; pa.variance = in.variance; pa.beta = in.beta; pa.beta_min = in.beta_min; pa.cos_anneal = in.cos_anneal_ratio;
    pa.sdf = out.sdf; pa.geo_feature = out.geo_feature; pa.gradients = out.gradients; pa.normals = out.normals; pa.rgb = out.rgb; pa.density = out.density;
    pa.alpha = out.alpha; pa.occupancy = out.occupancy;
    k_field_post<<<wb, 256, 0, st>>>(pa);
    SDFB_LAUNCHED("k_field_post");
  }
  return 0;
}

}  // namespace sdfb200
