// Texture export (nerfstudio/exporter/texture_utils.py of the reference): which face every texel of a UV texture lies on, its
// barycentric weights, and the ray that colours it.
//   k_uv_rasterize:  the xatlas path's brute-force search (:265-301), one thread per texel, faces staged through shared memory in
//                    ascending tiles.  The reference's chunking is kept: a chunk of c faces yields the face with the smallest
//                    |w0|+|w1|+|w2| (lowest index on ties), a chunk with a NaN for the texel yields nothing (torch.min propagates NaN
//                    and NaN < best is false), and a chunk only replaces the running best with a strictly smaller value.
//   k_uv_unwrap_grid: the custom unwrap (:100-192), two triangles per rectangle of a regular grid.
//   k_uv_texel_rays:  the interpolated origin and the negated, normalised interpolated normal of each texel (:194-205, :303-321),
//                     shifted back by half the ray length (:391).
// Every float operation of the weights and the origins is rounded on its own (no FMA contraction, IEEE division) in the reference's
// operand order, so face, weights and unshifted origins are bit-identical to the reference's separately rounded ATen ops.
#include <float.h>

#include "common.cuh"

namespace sdfb200 {
namespace {

constexpr int kRasterThreads = 256;
constexpr int kFaceTile = 256;

// get_parallelogram_area(p, a, b) (:43-56) with the edge terms (b - a) given
__device__ __forceinline__ float par_area(float px, float py, float ax, float ay, float ebx, float eby) {
  return __fsub_rn(__fmul_rn(__fsub_rn(px, ax), eby), __fmul_rn(__fsub_rn(py, ay), ebx));
}

// one face as the texel loop reads it: the three corners, the three edges and the doubled area
struct FaceUV {
  float4 v;     // v0x, v0y, v1x, v1y
  float4 w;     // v2x, v2y, area, -
  float4 e0;    // (v2 - v1).x, (v2 - v1).y, (v0 - v2).x, (v0 - v2).y
  float2 e1;    // (v1 - v0).x, (v1 - v0).y
};

__device__ __forceinline__ FaceUV load_face(const float* __restrict__ uv, int64_t f) {
  const float* t = uv + f * 6;
  FaceUV s;
  const float v0x = t[0], v0y = t[1], v1x = t[2], v1y = t[3], v2x = t[4], v2y = t[5];
  s.v = make_float4(v0x, v0y, v1x, v1y);
  s.e0 = make_float4(__fsub_rn(v2x, v1x), __fsub_rn(v2y, v1y), __fsub_rn(v0x, v2x), __fsub_rn(v0y, v2y));
  s.e1 = make_float2(__fsub_rn(v1x, v0x), __fsub_rn(v1y, v0y));
  s.w = make_float4(v2x, v2y, par_area(v2x, v2y, v0x, v0y, s.e1.x, s.e1.y), 0.f);   // area = par(v2, v0, v1)
  return s;
}

// w0 = par(p, v1, v2) / area, w1 = par(p, v2, v0) / area, w2 = par(p, v0, v1) / area
__device__ __forceinline__ void face_weights(const FaceUV& s, float px, float py, float& w0, float& w1, float& w2) {
  const float area = s.w.z;
  w0 = __fdiv_rn(par_area(px, py, s.v.z, s.v.w, s.e0.x, s.e0.y), area);
  w1 = __fdiv_rn(par_area(px, py, s.w.x, s.w.y, s.e0.z, s.e0.w), area);
  w2 = __fdiv_rn(par_area(px, py, s.v.x, s.v.y, s.e1.x, s.e1.y), area);
}

__global__ void __launch_bounds__(kRasterThreads) k_uv_rasterize(const float* __restrict__ uv, int64_t n_used, int32_t chunk,
                                                                 const float* __restrict__ lin_w, int32_t W, const float* __restrict__ lin_h,
                                                                 int64_t P, int32_t* __restrict__ face, float* __restrict__ bary) {
  __shared__ FaceUV tile[kFaceTile];
  const int64_t p = (int64_t)blockIdx.x * kRasterThreads + threadIdx.x;
  const int64_t q = p < P ? p : P - 1;
  const float px = __ldg(lin_w + q % W), py = __ldg(lin_h + q / W);
  float best = FLT_MAX, b0 = 0.f, b1 = 0.f, b2 = 0.f;
  int32_t best_f = 0;
  float cd = INFINITY, c0 = 0.f, c1 = 0.f, c2 = 0.f;   // the current chunk's minimum so far
  int32_t cf = 0, pos = 0;
  bool cnan = false;
  for (int64_t t0 = 0; t0 < n_used; t0 += kFaceTile) {
    const int nt = n_used - t0 < kFaceTile ? (int)(n_used - t0) : kFaceTile;
    __syncthreads();
    if ((int)threadIdx.x < nt) tile[threadIdx.x] = load_face(uv, t0 + threadIdx.x);
    __syncthreads();
#pragma unroll 2
    for (int k = 0; k < nt; ++k) {
      float w0, w1, w2;
      face_weights(tile[k], px, py, w0, w1, w2);
      const float d = __fadd_rn(__fadd_rn(fabsf(w0), fabsf(w1)), fabsf(w2));
      cnan |= isnan(d);
      if (d < cd) {
        cd = d; cf = (int32_t)(t0 + k); c0 = w0; c1 = w1; c2 = w2;
      }
      if (++pos == chunk) {   // the same face for every thread: a uniform branch
        if (!cnan && cd < best) {
          best = cd; best_f = cf; b0 = c0; b1 = c1; b2 = c2;
        }
        cd = INFINITY; cnan = false; pos = 0;
      }
    }
  }
  if (p < P) {
    face[p] = best_f;
    bary[p * 3 + 0] = b0;
    bary[p * 3 + 1] = b1;
    bary[p * 3 + 2] = b2;
  }
}

// custom unwrap: rectangle s = f / 2 of the grid (row s / sw, column s % sw) holds faces 2s (upper left) and 2s + 1 (lower right);
// corner k of face f is square_uv[f % 2][k] + (column, row) * lr, as the reference's broadcast add computes it
__device__ __forceinline__ float2 grid_corner(const float* __restrict__ square_uv, const float* __restrict__ lr, int64_t f, int k, int32_t sw) {
  const int64_t s = f >> 1;
  const float* c = square_uv + ((f & 1) * 3 + k) * 2;
  return make_float2(__fadd_rn(__ldg(c), __fmul_rn((float)(s % sw), __ldg(lr))), __fadd_rn(__ldg(c + 1), __fmul_rn((float)(s / sw), __ldg(lr + 1))));
}

__global__ void k_uv_unwrap_grid(const float* __restrict__ square_uv, const float* __restrict__ lr, int64_t F, int32_t sw, int32_t px_tri,
                                 const float* __restrict__ lin_w, int32_t W, const float* __restrict__ lin_h, int64_t P,
                                 float* __restrict__ texture_coordinates, int32_t* __restrict__ face, float* __restrict__ bary) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < F) {
    for (int k = 0; k < 3; ++k) {
      const float2 c = grid_corner(square_uv, lr, p, k, sw);
      texture_coordinates[p * 6 + k * 2] = c.x;
      texture_coordinates[p * 6 + k * 2 + 1] = c.y;
    }
  }
  if (p >= P) return;
  const int64_t j = p % W, i = p / W;
  const int32_t sqw = px_tri + 3;   // rectangle width: the triangle plus a 3-texel gap
  const int64_t square = (i / px_tri) * sw + j / sqw;
  const bool lower_right = (j % sqw) + (i % px_tri) >= sqw - 2;
  int64_t f = square * 2 + (lower_right ? 1 : 0);
  f = f < 0 ? 0 : (f > F - 1 ? F - 1 : f);
  FaceUV s;
  {
    const float2 a = grid_corner(square_uv, lr, f, 0, sw), b = grid_corner(square_uv, lr, f, 1, sw), c = grid_corner(square_uv, lr, f, 2, sw);
    s.v = make_float4(a.x, a.y, b.x, b.y);
    s.e0 = make_float4(__fsub_rn(c.x, b.x), __fsub_rn(c.y, b.y), __fsub_rn(a.x, c.x), __fsub_rn(a.y, c.y));
    s.e1 = make_float2(__fsub_rn(b.x, a.x), __fsub_rn(b.y, a.y));
    s.w = make_float4(c.x, c.y, par_area(c.x, c.y, a.x, a.y, s.e1.x, s.e1.y), 0.f);
  }
  float w0, w1, w2;
  face_weights(s, __ldg(lin_w + j), __ldg(lin_h + i), w0, w1, w2);
  face[p] = (int32_t)f;
  bary[p * 3 + 0] = w0;
  bary[p * 3 + 1] = w1;
  bary[p * 3 + 2] = w2;
}

__global__ void k_uv_texel_rays(const float* __restrict__ vertices, const float* __restrict__ normals, const int64_t* __restrict__ faces,
                                const int32_t* __restrict__ face, const float* __restrict__ bary, const float* __restrict__ raylen, int64_t P,
                                float* __restrict__ origins, float* __restrict__ directions, float* __restrict__ fars) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int64_t f = __ldg(face + p);
  const int64_t i0 = __ldg(faces + f * 3), i1 = __ldg(faces + f * 3 + 1), i2 = __ldg(faces + f * 3 + 2);
  const float w0 = __ldg(bary + p * 3), w1 = __ldg(bary + p * 3 + 1), w2 = __ldg(bary + p * 3 + 2);
  float o[3], d[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    o[c] = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(vertices + i0 * 3 + c), w0), __fmul_rn(__ldg(vertices + i1 * 3 + c), w1)),
                     __fmul_rn(__ldg(vertices + i2 * 3 + c), w2));
    d[c] = -__fadd_rn(__fadd_rn(__fmul_rn(__ldg(normals + i0 * 3 + c), w0), __fmul_rn(__ldg(normals + i1 * 3 + c), w1)),
                      __fmul_rn(__ldg(normals + i2 * 3 + c), w2));
  }
  // F.normalize: x / max(||x||, 1e-12)
  const float norm = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2]))), 1e-12f);
  const float len = raylen ? __ldg(raylen) : 0.f, half = __fmul_rn(0.5f, len);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float dc = __fdiv_rn(d[c], norm);
    directions[p * 3 + c] = dc;
    origins[p * 3 + c] = raylen ? __fsub_rn(o[c], __fmul_rn(half, dc)) : o[c];
  }
  if (raylen) fars[p] = len;
}

}  // namespace
}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_uv_rasterize(const float* texture_coordinates, int64_t n_faces, int32_t chunk, const float* linspace_w, int32_t width,
                                    const float* linspace_h, int32_t height, int32_t* face, float* bary, void* stream) {
  SDFB_REQUIRE(n_faces >= 0 && n_faces <= INT32_MAX && chunk >= 1 && width >= 0 && height >= 0, "bad sizes");
  const int64_t P = (int64_t)width * height;
  if (P == 0) return 0;
  SDFB_REQUIRE(linspace_w && linspace_h && face && bary, "NULL pointer");
  const int64_t n_used = n_faces / chunk * chunk;   // range(num_faces // chunk): the tail chunk takes no part
  SDFB_REQUIRE(n_used == 0 || texture_coordinates, "NULL pointer");
  k_uv_rasterize<<<(unsigned)ceil_div(P, kRasterThreads), kRasterThreads, 0, (cudaStream_t)stream>>>(texture_coordinates, n_used, chunk, linspace_w,
                                                                                                      width, linspace_h, P, face, bary);
  SDFB_LAUNCHED("k_uv_rasterize");
  return 0;
}

extern "C" int sdfb200_uv_unwrap_grid(const float* square_uv, const float* lr, int64_t n_faces, int32_t squares_per_side_w,
                                      int32_t px_per_uv_triangle, const float* linspace_w, int32_t width, const float* linspace_h, int32_t height,
                                      float* texture_coordinates, int32_t* face, float* bary, void* stream) {
  SDFB_REQUIRE(n_faces >= 1 && n_faces <= INT32_MAX && squares_per_side_w >= 1 && px_per_uv_triangle >= 1 && width >= 0 && height >= 0,
               "bad sizes");
  const int64_t P = (int64_t)width * height;
  const int64_t n = P > n_faces ? P : n_faces;
  SDFB_REQUIRE(square_uv && lr && texture_coordinates, "NULL pointer");
  SDFB_REQUIRE(P == 0 || (linspace_w && linspace_h && face && bary), "NULL pointer");
  k_uv_unwrap_grid<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(square_uv, lr, n_faces, squares_per_side_w, px_per_uv_triangle,
                                                                                 linspace_w, width, linspace_h, P, texture_coordinates, face, bary);
  SDFB_LAUNCHED("k_uv_unwrap_grid");
  return 0;
}

extern "C" int sdfb200_uv_texel_rays(const float* vertices, const float* vertex_normals, const int64_t* faces, const int32_t* face,
                                     const float* bary, const float* raylen, int64_t n_texels, float* origins, float* directions, float* fars,
                                     void* stream) {
  SDFB_REQUIRE(n_texels >= 0, "bad sizes");
  if (n_texels == 0) return 0;
  SDFB_REQUIRE(vertices && vertex_normals && faces && face && bary && origins && directions && (raylen == nullptr || fars), "NULL pointer");
  k_uv_texel_rays<<<(unsigned)ceil_div(n_texels, 256), 256, 0, (cudaStream_t)stream>>>(vertices, vertex_normals, faces, face, bary, raylen,
                                                                                        n_texels, origins, directions, fars);
  SDFB_LAUNCHED("k_uv_texel_rays");
  return 0;
}
