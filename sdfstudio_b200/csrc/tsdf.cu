// TSDF fusion (nerfstudio/exporter/tsdf_utils.py:168-270 of the reference, TSDF.integrate_tsdf) for B images in one launch.
//   k_tsdf_integrate: one thread per voxel.  The cameras are staged in shared memory in tiles of kCamTile; each thread visits the
//                     images in order with the voxel's value, weight and colour held in registers, so the volume is read once and
//                     written once and nothing per (voxel, image) reaches memory.  No atomics: a voxel's result depends only on the
//                     order of the images, not on how they are batched.
// Every float operation is rounded on its own (no FMA contraction, IEEE division and square root) in the op order documented in
// include/sdfb200.h, which restates the reference's separately rounded ATen ops.
#include "common.cuh"

namespace sdfb200 {
namespace {

constexpr int kTsdfThreads = 256;
constexpr int kCamTile = 128;
constexpr int kCamFloats = 18;   // rows 0-2 of inverse(c2w), rows 0-1 of K

__device__ __forceinline__ float dot4(const float* m, float x, float y, float z) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fmul_rn(m[1], y)), __fmul_rn(m[2], z)), m[3]);
}

// grid_sample(mode="nearest", padding_mode="zeros", align_corners=False)'s pixel along an axis of `size` pixels for the pixel
// coordinate p: g = 2 p / size - 1 (tsdf_utils.py:227), ATen's CUDA unnormalisation ((g + 1) size - 1) / 2, then nearbyint (half to
// even).  Returns -1 when the pixel lies outside the image or the coordinate is not finite.
__device__ __forceinline__ int pixel_index(float p, int32_t size) {
  const float s = (float)size;
  const float g = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, p), s), 1.f);
  const float f = nearbyintf(__fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(g, 1.f), s), 1.f), 2.f));
  return (f >= 0.f && f < s) ? (int)f : -1;   // false for NaN
}

__global__ void __launch_bounds__(kTsdfThreads)
    k_tsdf_integrate(const float* __restrict__ voxel_coords, int64_t N, const float* __restrict__ cams, int32_t B,
                     const float* __restrict__ depth, const float* __restrict__ color, int32_t H, int32_t W,
                     const float* __restrict__ truncation, float* __restrict__ values, float* __restrict__ weights,
                     float* __restrict__ colors) {
  __shared__ float tile[kCamTile * kCamFloats];
  const int64_t i = (int64_t)blockIdx.x * kTsdfThreads + threadIdx.x;
  const int64_t q = i < N ? i : N - 1;
  const float x = __ldg(voxel_coords + q), y = __ldg(voxel_coords + N + q), z = __ldg(voxel_coords + 2 * N + q);
  const float trunc = __ldg(truncation), neg_trunc = -trunc;
  float value = values[q], weight = weights[q];
  float c0 = 0.f, c1 = 0.f, c2 = 0.f;
  if (color) {
    c0 = colors[q * 3];
    c1 = colors[q * 3 + 1];
    c2 = colors[q * 3 + 2];
  }
  const int64_t plane = (int64_t)H * W;
  for (int32_t b0 = 0; b0 < B; b0 += kCamTile) {
    const int nt = B - b0 < kCamTile ? B - b0 : kCamTile;
    __syncthreads();
    for (int k = threadIdx.x; k < nt * kCamFloats; k += kTsdfThreads) tile[k] = __ldg(cams + (int64_t)b0 * kCamFloats + k);
    __syncthreads();
    for (int c = 0; c < nt; ++c) {
      const float* m = tile + c * kCamFloats;
      const float cx = dot4(m, x, y, z);
      const float cy = -dot4(m + 4, x, y, z);
      const float cz = -dot4(m + 8, x, y, z);
      const float vd = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), __fmul_rn(cz, cz)));
      const float u = __fdiv_rn(cx, cz), v = __fdiv_rn(cy, cz), w = __fdiv_rn(cz, cz);
      const float* k = m + 12;
      const float px = __fadd_rn(__fadd_rn(__fmul_rn(k[0], u), __fmul_rn(k[1], v)), __fmul_rn(k[2], w));
      const float py = __fadd_rn(__fadd_rn(__fmul_rn(k[3], u), __fmul_rn(k[4], v)), __fmul_rn(k[5], w));
      const int ix = pixel_index(px, W), iy = pixel_index(py, H);
      const bool inside = ix >= 0 && iy >= 0;
      const int64_t pix = (int64_t)iy * W + ix;
      const int64_t img = (int64_t)(b0 + c);
      const float sd = inside ? __ldg(depth + img * plane + pix) : 0.f;
      const float dist = __fsub_rn(sd, vd);
      if (!(vd > 0.f && sd > 0.f && dist > neg_trunc)) continue;
      float t = __fdiv_rn(dist, trunc);
      t = t < -1.f ? -1.f : (t > 1.f ? 1.f : t);
      const float total = __fadd_rn(weight, 1.f);
      value = __fdiv_rn(__fadd_rn(__fmul_rn(value, weight), t), total);
      if (color) {
        const float* cimg = color + img * 3 * plane + pix;   // inside: sd > 0 only where the pixel lies in the image
        c0 = __fdiv_rn(__fadd_rn(__fmul_rn(c0, weight), __ldg(cimg)), total);
        c1 = __fdiv_rn(__fadd_rn(__fmul_rn(c1, weight), __ldg(cimg + plane)), total);
        c2 = __fdiv_rn(__fadd_rn(__fmul_rn(c2, weight), __ldg(cimg + 2 * plane)), total);
      }
      weight = total > 1.f ? 1.f : total;
    }
  }
  if (i < N) {
    values[i] = value;
    weights[i] = weight;
    if (color) {
      colors[i * 3] = c0;
      colors[i * 3 + 1] = c1;
      colors[i * 3 + 2] = c2;
    }
  }
}

}  // namespace
}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_tsdf_integrate(const float* voxel_coords, int64_t n_voxels, const float* cams, int32_t n_cams, const float* depth,
                                      const float* color, int32_t height, int32_t width, const float* truncation, float* values,
                                      float* weights, float* colors, void* stream) {
  SDFB_REQUIRE(n_voxels >= 0 && n_cams >= 0 && height >= 0 && width >= 0, "bad sizes");
  SDFB_REQUIRE(n_cams == 0 || (height >= 1 && width >= 1), "images need height and width >= 1");
  SDFB_REQUIRE(n_voxels == 0 || (voxel_coords && values && weights && truncation), "NULL pointer");
  SDFB_REQUIRE(n_cams == 0 || (cams && depth), "NULL pointer");
  SDFB_REQUIRE(color == nullptr || n_voxels == 0 || colors, "NULL pointer");
  if (n_voxels == 0 || n_cams == 0) return 0;
  k_tsdf_integrate<<<(unsigned)ceil_div(n_voxels, kTsdfThreads), kTsdfThreads, 0, (cudaStream_t)stream>>>(
      voxel_coords, n_voxels, cams, n_cams, depth, color, height, width, truncation, values, weights, colors);
  SDFB_LAUNCHED("k_tsdf_integrate");
  return 0;
}
