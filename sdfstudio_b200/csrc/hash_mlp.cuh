// The tiny-cuda-nn NetworkWithInputEncoding fields on one kernel, k_hash_mlp_field<T, F, H, HC>, one thread per point:
//   density half: normalisation into the grid's unit cube, HashGrid -> ReLU MLP without biases (FullyFusedMLP semantics), output row 0
//     -> density = exp (trunc_exp forward);
//   colour half (HC > 0, the nerfacto background field TCNNNerfactoField.forward, nerfstudio/fields/nerfacto_field.py:223-318): output
//     rows 1..geo_dim are the geometry feature; tcnn SphericalHarmonics degree 4 of the direction, cat([SH 16, geo, appearance]) -> ReLU
//     MLP -> 3 outputs -> sigmoid.
// HC = 0 is the proposal density field (HashMLPDensityField, nerfstudio/fields/density_fields.py:40-121): density only, point mode.
// The weights are broadcast from shared memory (every thread of a warp reads the same word); the geometry feature and every hidden layer
// stay in registers.  With the colour half, blocks stride over the points, so each block loads the weights once.  hash_mlp_field.cu
// holds the fp32-table instantiations and the C-ABI entry points, hash_mlp_field_f16.cu the fp16-table ones, so that the two halves
// compile in parallel.
#pragma once
#include <algorithm>
#include <atomic>

#include "field.h"
#include "grid.cuh"

namespace sdfb200 {

// aabb != NULL: SceneBox.get_normalized_positions (data/scene_box.py:67-76); else SceneContraction (spatial_distortions.py:66-73,
// `contraction`) followed by (x + 2) / 4
__device__ __forceinline__ void normalize_position(const float* aabb, int contraction, float px, float py, float pz, float& x01, float& y01,
                                                   float& z01) {
  if (aabb != nullptr) {
    const float lx = __ldg(aabb + 3) - __ldg(aabb), ly = __ldg(aabb + 4) - __ldg(aabb + 1), lz = __ldg(aabb + 5) - __ldg(aabb + 2);
    x01 = (px - __ldg(aabb)) / lx; y01 = (py - __ldg(aabb + 1)) / ly; z01 = (pz - __ldg(aabb + 2)) / lz;
  } else {
    if (contraction != SDFB200_CONTRACT_NONE) {
      const float mag = contraction == SDFB200_CONTRACT_LINF ? fmaxf(fabsf(px), fmaxf(fabsf(py), fabsf(pz))) : sqrtf(px * px + py * py + pz * pz);
      if (mag >= 1.f) {
        const float k = 2.f - 1.f / mag;
        px = k * (px / mag); py = k * (py / mag); pz = k * (pz / mag);
      }
    }
    x01 = (px + 2.0f) * 0.25f; y01 = (py + 2.0f) * 0.25f; z01 = (pz + 2.0f) * 0.25f;
  }
}

// h += column `wc` (stride ld) x v: one input of a layer applied to all H outputs
template <int H>
__device__ __forceinline__ void accumulate_column(const float* wc, int ld, float v, float (&h)[H]) {
#pragma unroll
  for (int o = 0; o < H; ++o) h[o] = fmaf(wc[o * ld], v, h[o]);
}

template <int H>
__device__ __forceinline__ void relu_(float (&h)[H]) {
#pragma unroll
  for (int o = 0; o < H; ++o) h[o] = fmaxf(h[o], 0.f);
}

template <int H>
__device__ __forceinline__ float dot_row(const float* w, const float (&h)[H]) {
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < H; ++k) acc = fmaf(w[k], h[k], acc);
  return acc;
}

// n_layers ReLU layers [H, H] (row-major, starting at w) applied to h in place; returns the weights that follow them
template <int H>
__device__ __forceinline__ const float* relu_layers(const float* w, int n_layers, float (&h)[H]) {
  for (int layer = 0; layer < n_layers; ++layer, w += H * H) {
    float g[H];
#pragma unroll
    for (int o = 0; o < H; ++o) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < H; ++k) acc = fmaf(w[o * H + k], h[k], acc);
      g[o] = fmaxf(acc, 0.f);
    }
#pragma unroll
    for (int o = 0; o < H; ++o) h[o] = g[o];
  }
  return w;
}

// w: [H, in_pad] | (n_hidden - 1) x [H, H] | output rows.  h = the last hidden layer's activations; returns the output rows.
// Layer 0 is accumulated level by level (the encoded vector is never materialised); levels >= active_levels contribute zeros.
template <typename T, int F, int H>
__device__ __forceinline__ const float* hash_mlp_hidden(const sdfb200_grid_t& g, const void* table, const float* w, int in_pad, int n_hidden,
                                                        float x01, float y01, float z01, float (&h)[H]) {
#pragma unroll
  for (int o = 0; o < H; ++o) h[o] = 0.f;
  for (int l = 0; l < g.n_levels; ++l) {
    float f[F];
    float d[F][3];
    if (l < g.active_levels) encode_level<T, F>(g, table, l, x01, y01, z01, f, d);
    else
      for (int k = 0; k < F; ++k) f[k] = 0.f;
#pragma unroll
    for (int k = 0; k < F; ++k) accumulate_column<H>(w + (l * F + k), in_pad, f[k], h);
  }
  relu_<H>(h);
  return relu_layers<H>(w + H * in_pad, n_hidden - 1, h);
}

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

// Threads per block: 256 with the colour half, 128 for the density half alone (launch_hash_mlp says why)
template <int HC>
constexpr int kHashMlpThreads = HC > 0 ? 256 : 128;
constexpr int kOutRows = 16;   // tcnn pads an output layer to 16 neurons
constexpr int kRgbRows = 3;

struct HashMlpArgs {
  sdfb200_grid_t grid;
  const void* table;
  const float* base_w;      // [H, in_pad] | (n_base-1) x [H, H] | output rows (rows 0..geo_dim read)
  const float* head_w;      // [HC, head_pad] | (n_head-1) x [HC, HC] | output rows (rows 0..2 read); may be NULL when rgb is
  const float* aabb;        // [2,3] or NULL
  const float* origins;     // ray mode [R,3]; point mode: positions [N,3]
  const float* directions;  // ray mode [R,3]; point mode [N,3]; NULL when rgb is not wanted
  const float* bins;        // ray mode [R,S+1] euclidean bin edges; point mode NULL
  const float* appearance;  // row r at appearance + r * app_stride, or NULL (= zeros)
  long long app_stride;
  int contraction, n_base, n_head, in_pad, head_pad, geo_dim, app_dim, S;   // S = 0: point mode
  long long n;
  float *density, *rgb, *pre_activation, *geo_feature;   // rgb and geo_feature NULL when HC = 0
};

// Shared memory holds the base weights, then (colour half) the head weights.  Only the output rows the kernel reads are loaded: base rows
// 0..geo_dim (the density ABI's last block is the one row [H]) and head rows 0..2.  The head weights start where the nerfacto ABI's
// 16-row base block ends, so base rows geo_dim + 1..15 are reserved but not loaded: with the head right after row geo_dim, ptxas gives
// the colour instantiations up to 255 registers.
template <int H>
__host__ __device__ __forceinline__ int base_weight_floats(const HashMlpArgs& a, int out_rows) {
  return H * a.in_pad + (a.n_base - 1) * H * H + out_rows * H;
}
template <int H, int HC>
__host__ __device__ __forceinline__ int head_weight_offset(const HashMlpArgs& a) { return base_weight_floats<H>(a, HC > 0 ? kOutRows : 1); }
template <int HC>
__host__ __device__ __forceinline__ int head_weight_floats(const HashMlpArgs& a) {
  return HC > 0 && a.rgb ? HC * a.head_pad + (a.n_head - 1) * HC * HC + kRgbRows * HC : 0;
}

template <typename T, int F, int H, int HC>
__global__ void __launch_bounds__(kHashMlpThreads<HC>) k_hash_mlp_field(const __grid_constant__ HashMlpArgs a) {
  extern __shared__ float w_s[];
  const int n_bw = base_weight_floats<H>(a, 1 + a.geo_dim);
  for (int i = threadIdx.x; i < n_bw; i += blockDim.x) w_s[i] = __ldg(a.base_w + i);
  float* hw_s = w_s + head_weight_offset<H, HC>(a);
  if constexpr (HC > 0) {
    const int n_hw = head_weight_floats<HC>(a);
    for (int i = threadIdx.x; i < n_hw; i += blockDim.x) hw_s[i] = __ldg(a.head_w + i);
  }
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
      if constexpr (HC > 0) {
#pragma unroll
        for (int j = 0; j < 15; ++j) geo[j] = j < a.geo_dim ? dot_row<H>(wo + (1 + j) * H, h) : 0.f;
      }
    }
    if constexpr (HC > 0) {
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
      for (int j = 0; j < kRgbRows; ++j) a.rgb[i * 3 + j] = sigmoidf_(dot_row<HC>(wo + j * HC, c));
    } else {
      break;   // the density half alone: one point per thread (launch_hash_mlp)
    }
  }
}

// The grid.  With the colour half: no more blocks than can be resident at once (the occupancy of this instantiation at this shared-memory
// size, times the SM count), each loading its weights (up to 48 KB) once and striding over the points.  The density half alone: one point
// per thread, one block per 128 points.  Its weights are a few KB, and the stride loop would cost its instantiations up to 24 more
// registers (ptxas -v), i.e. fewer resident warps to hide the L2 latency of the hash gathers that bound it.
template <typename T, int F, int H, int HC>
static int launch_hash_mlp(const HashMlpArgs& a, cudaStream_t st) {
  const auto kernel = k_hash_mlp_field<T, F, H, HC>;
  constexpr int threads = kHashMlpThreads<HC>;
  const size_t smem = (size_t)(head_weight_offset<H, HC>(a) + head_weight_floats<HC>(a)) * sizeof(float);
  if (smem > 48 * 1024) SDFB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t blocks = ceil_div(a.n, threads);
  if constexpr (HC > 0) {
    // blocks per SM, cached per device ordinal as smem << 8 | blocks for the shared-memory size of the last query; a call at another size
    // (rgb on or off, another appearance width) queries again
    static std::atomic<long long> resident[64];
    int dev = 0;
    SDFB_CUDA(cudaGetDevice(&dev));
    long long r = dev >= 0 && dev < 64 ? resident[dev].load(std::memory_order_relaxed) : 0;
    if ((r & 0xff) == 0 || (size_t)(r >> 8) != smem) {
      int per_sm = 0;
      SDFB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
      if (per_sm < 1)
        return fail(SDFB200_EUNSUPPORTED, "nerfacto field: no block fits on an SM with %s%lld bytes of weights in shared memory", "", (long long)smem);
      r = (long long)smem << 8 | per_sm;
      if (dev >= 0 && dev < 64) resident[dev].store(r, std::memory_order_relaxed);
    }
    blocks = std::min<int64_t>(blocks, (r & 0xff) * persistent_ctas());
  }
  kernel<<<(unsigned)blocks, threads, smem, st>>>(a);
  SDFB_LAUNCHED("k_hash_mlp_field");
  return 0;
}

// hc = 0: the density half alone; hc = 16, 32 or 64 (colour widths) only with 2 features per level, the nerfacto field's grid
template <typename T, int F, int H>
static int launch_hash_mlp_hc(const HashMlpArgs& a, int hc, cudaStream_t st) {
  if constexpr (F == 2) {
    switch (hc) {
      case 16: return launch_hash_mlp<T, F, H, 16>(a, st);
      case 32: return launch_hash_mlp<T, F, H, 32>(a, st);
      case 64: return launch_hash_mlp<T, F, H, 64>(a, st);
    }
  }
  return launch_hash_mlp<T, F, H, 0>(a, st);
}

template <typename T, int F>
static int launch_hash_mlp_h(const HashMlpArgs& a, int h, int hc, cudaStream_t st) {
  switch (h) {
    case 16: return launch_hash_mlp_hc<T, F, 16>(a, hc, st);
    case 32: return launch_hash_mlp_hc<T, F, 32>(a, hc, st);
    default: return launch_hash_mlp_hc<T, F, 64>(a, hc, st);
  }
}

// widths h (base) and hc (colour, 0 = density only), checked by the entry points; the feature count is the grid's
template <typename T>
int launch_hash_mlp_t(const HashMlpArgs& a, int h, int hc, cudaStream_t st) {
  switch (a.grid.n_features) {
    case 1: return launch_hash_mlp_h<T, 1>(a, h, hc, st);
    case 2: return launch_hash_mlp_h<T, 2>(a, h, hc, st);
    case 4: return launch_hash_mlp_h<T, 4>(a, h, hc, st);
    default: return launch_hash_mlp_h<T, 8>(a, h, hc, st);
  }
}

int launch_hash_mlp_f16(const HashMlpArgs& a, int h, int hc, cudaStream_t st);

}  // namespace sdfb200
