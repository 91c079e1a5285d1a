// Background field of neus-facto-angelo / bakedangelo: TCNNNerfactoField.forward (nerfstudio/fields/nerfacto_field.py:223-318 through
// Field.forward, fields/base_field.py:104-123) for one sample per thread.
//   density half: the proposal network's body (hash_mlp.cuh), output 1 + geo_feat_dim (padded to 16 rows), density = exp(out[0]);
//   colour half:  tcnn SphericalHarmonics degree 4 of the direction, cat([SH 16, geo, appearance]) -> ReLU MLP -> 3 outputs -> sigmoid.
// Both weight sets are broadcast from shared memory; the geometry feature and every hidden layer stay in registers.  Blocks stride
// over the samples so that each block loads the weights once.  Instantiated per table type (nerfacto_field.cu: fp32 and the ABI,
// nerfacto_field_f16.cu: fp16) so that the two halves compile in parallel.
#pragma once
#include <algorithm>

#include "field.h"
#include "hash_mlp.cuh"

namespace sdfb200 {

constexpr int kNerfactoThreads = 256;
constexpr int kOutRows = 16;   // tcnn pads an output layer to 16 neurons

struct NerfactoArgs {
  sdfb200_grid_t grid;
  const void* table;
  const float* base_w;      // [H, in_pad] | (n_base-1) x [H, H] | [16, H]
  const float* head_w;      // [HC, head_pad] | (n_head-1) x [HC, HC] | [16, HC]
  const float* aabb;        // [2,3] or NULL
  const float* origins;     // ray mode [R,3]; point mode: positions [N,3]
  const float* directions;  // ray mode [R,3]; point mode [N,3]; NULL when rgb is not wanted
  const float* bins;        // ray mode [R,S+1] euclidean bin edges; point mode NULL
  const float* appearance;  // row r at appearance + r * app_stride, or NULL (= zeros)
  long long app_stride;
  int contraction, n_base, n_head, in_pad, head_pad, geo_dim, app_dim, S;   // S = 0: point mode
  long long n;
  float *density, *rgb, *pre_activation, *geo_feature;
};

// tiny-cuda-nn SphericalHarmonics, degree 4, of x in [-1,1]^3 (the encoding maps its [0,1] input back with 2x - 1)
__device__ __forceinline__ void sh4(float x, float y, float z, float (&s)[16]) {
  const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
  s[0] = 0.28209479177387814f;
  s[1] = -0.48860251190291987f * y;
  s[2] = 0.48860251190291987f * z;
  s[3] = -0.48860251190291987f * x;
  s[4] = 1.0925484305920792f * xy;
  s[5] = -1.0925484305920792f * yz;
  s[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
  s[7] = -1.0925484305920792f * xz;
  s[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
  s[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
  s[10] = 2.8906114426405538f * xy * z;
  s[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
  s[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
  s[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
  s[14] = 1.4453057213202769f * z * (x2 - y2);
  s[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

template <int H>
__device__ __forceinline__ float dot_row(const float* w, const float (&h)[H]) {
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < H; ++k) acc = fmaf(w[k], h[k], acc);
  return acc;
}

template <typename T, int F, int H, int HC>
__global__ void __launch_bounds__(kNerfactoThreads) k_nerfacto_field(const __grid_constant__ NerfactoArgs a) {
  extern __shared__ float w_s[];
  const int n_bw = H * a.in_pad + (a.n_base - 1) * H * H + kOutRows * H;
  const int n_hw = a.rgb ? HC * a.head_pad + (a.n_head - 1) * HC * HC + kOutRows * HC : 0;
  float* hw_s = w_s + n_bw;
  for (int i = threadIdx.x; i < n_bw; i += blockDim.x) w_s[i] = __ldg(a.base_w + i);
  for (int i = threadIdx.x; i < n_hw; i += blockDim.x) hw_s[i] = __ldg(a.head_w + i);
  __syncthreads();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (long long)gridDim.x * blockDim.x) {
    const long long row = a.S ? i / a.S : i;   // ray (ray mode) or point: the row of origins, directions and appearance
    float p[3];
    if (a.S) {
      ray_midpoint(a.origins, a.directions, a.bins, row, a.S, i - row * a.S, p);
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) p[c] = __ldg(a.origins + i * 3 + c);
    }
    float x01, y01, z01;
    normalize_position(a.aabb, a.contraction, p[0], p[1], p[2], x01, y01, z01);
    float geo[15];
    {
      float h[H];
      const float* wo = hash_mlp_hidden<T, F, H>(a.grid, a.table, w_s, a.in_pad, a.n_base, x01, y01, z01, h);
      const float out = dot_row<H>(wo, h);
      if (a.pre_activation) a.pre_activation[i] = out;
      a.density[i] = expf(out);   // trunc_exp forward = exp
#pragma unroll
      for (int j = 0; j < 15; ++j) geo[j] = j < a.geo_dim ? dot_row<H>(wo + (1 + j) * H, h) : 0.f;
    }
    if (a.geo_feature) {
#pragma unroll
      for (int j = 0; j < 15; ++j)
        if (j < a.geo_dim) a.geo_feature[i * a.geo_dim + j] = geo[j];
    }
    if (!a.rgb) continue;
    // get_normalized_directions (nerfacto_field.py:58-64) then tcnn's 2x - 1: both steps in fp32 like the reference
    float s[16];
    {
      const float* d = a.directions + row * 3;
      float x[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) x[c] = __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(__ldg(d + c), 1.f), 0.5f), 2.f), 1.f);
      sh4(x[0], x[1], x[2], s);
    }
    // colour layer 0, input cat([SH, geo, appearance]) (nerfacto_field.py:307-314) applied column by column
    float c[HC];
#pragma unroll
    for (int o = 0; o < HC; ++o) c[o] = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) accumulate_column<HC>(hw_s + k, a.head_pad, s[k], c);
#pragma unroll
    for (int k = 0; k < 15; ++k)
      if (k < a.geo_dim) accumulate_column<HC>(hw_s + 16 + k, a.head_pad, geo[k], c);
    if (a.appearance) {
      const float* app = a.appearance + row * a.app_stride;
      for (int k = 0; k < a.app_dim; ++k) accumulate_column<HC>(hw_s + 16 + a.geo_dim + k, a.head_pad, __ldg(app + k), c);
    }
    relu_<HC>(c);
    const float* wo = relu_layers<HC>(hw_s + HC * a.head_pad, a.n_head - 1, c);
#pragma unroll
    for (int j = 0; j < 3; ++j) a.rgb[i * 3 + j] = sigmoidf_(dot_row<HC>(wo + j * HC, c));
  }
}

template <typename T, int H, int HC>
static int launch_nerfacto(const NerfactoArgs& a, cudaStream_t st) {
  const int n_bw = H * a.in_pad + (a.n_base - 1) * H * H + kOutRows * H;
  const int n_hw = a.rgb ? HC * a.head_pad + (a.n_head - 1) * HC * HC + kOutRows * HC : 0;
  const size_t smem = (size_t)(n_bw + n_hw) * sizeof(float);
  if (smem > 48 * 1024) SDFB_CUDA(cudaFuncSetAttribute(k_nerfacto_field<T, 2, H, HC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // a few resident blocks per SM, each loading the weights once and striding over the samples
  const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(a.n, kNerfactoThreads), (int64_t)persistent_ctas() * 4);
  k_nerfacto_field<T, 2, H, HC><<<blocks, kNerfactoThreads, smem, st>>>(a);
  SDFB_LAUNCHED("k_nerfacto_field");
  return 0;
}

template <typename T, int H>
static int launch_nerfacto_hc(const NerfactoArgs& a, int hc, cudaStream_t st) {
  switch (hc) {
    case 16: return launch_nerfacto<T, H, 16>(a, st);
    case 32: return launch_nerfacto<T, H, 32>(a, st);
    default: return launch_nerfacto<T, H, 64>(a, st);
  }
}

template <typename T>
int launch_nerfacto_h(const NerfactoArgs& a, int h, int hc, cudaStream_t st) {
  switch (h) {
    case 16: return launch_nerfacto_hc<T, 16>(a, hc, st);
    case 32: return launch_nerfacto_hc<T, 32>(a, hc, st);
    default: return launch_nerfacto_hc<T, 64>(a, hc, st);
  }
}

int launch_nerfacto_f32(const NerfactoArgs& a, int h, int hc, cudaStream_t st);
int launch_nerfacto_f16(const NerfactoArgs& a, int h, int hc, cudaStream_t st);

}  // namespace sdfb200
