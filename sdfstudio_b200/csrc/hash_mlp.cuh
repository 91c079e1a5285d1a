// The body shared by the tiny-cuda-nn NetworkWithInputEncoding fields (proposal density field, nerfacto background field): a point's
// normalisation into the grid's unit cube, then HashGrid -> ReLU MLP without biases (FullyFusedMLP semantics) up to the last hidden
// layer.  One thread per point; the weights are read from shared memory (every thread of a warp reads the same word: a broadcast).
#pragma once
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

}  // namespace sdfb200
