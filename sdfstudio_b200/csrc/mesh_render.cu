// Mesh rendering (scripts/render_mesh.py of the reference, drawn there by open3d's OpenGL visualizer) for B frames of one mesh.
//   k_mesh_rasterize: one thread per (frame, face).  The thread sets up the face in camera space and walks the pixels of its box with the
//                     homogeneous edge test; a face whose box holds more than SDFB200_MESH_LARGE_TRIANGLE_PIXELS pixels is queued in
//                     shared memory instead, and the whole block walks each queued box, one pixel per thread.  Every covering
//                     (pixel, face) pair does atomicMin on the pixel's 64-bit (depth, face) key.
//   k_mesh_shade:     one thread per pixel: the key's face, the same setup and edge products, then barycentrics and the shading.
// Every double operation is rounded on its own (no FMA contraction), in the op order documented in include/sdfb200.h, so the keys are
// bit-identical to a brute-force fp64 restatement over every (pixel, face) pair.
#include <math.h>

#include "common.cuh"

namespace sdfb200 {
namespace {

constexpr int kRasterThreads = 256;
constexpr int kShadeThreads = 256;
constexpr int kCamFloats = 18;   // rows 0-2 of inverse(c2w), rows 0-1 of K
constexpr unsigned long long kBackground = ~0ull;

struct V3 {
  double x, y, z;
};

__device__ __forceinline__ V3 cross(const V3& a, const V3& b) {
  return {__dsub_rn(__dmul_rn(a.y, b.z), __dmul_rn(a.z, b.y)), __dsub_rn(__dmul_rn(a.z, b.x), __dmul_rn(a.x, b.z)),
          __dsub_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x))};
}
__device__ __forceinline__ double dot(const V3& a, const V3& b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}
__device__ __forceinline__ V3 neg(const V3& a) { return {-a.x, -a.y, -a.z}; }

// row r of inverse(c2w) applied to (x, y, z, 1)
__device__ __forceinline__ double row(const float* m, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)__ldg(m), x), __dmul_rn((double)__ldg(m + 1), y)), __dmul_rn((double)__ldg(m + 2), z)),
                   (double)__ldg(m + 3));
}
__device__ __forceinline__ V3 to_camera(const float* cam, const float* vertices, int64_t v) {
  const double x = __ldg(vertices + v * 3), y = __ldg(vertices + v * 3 + 1), z = __ldg(vertices + v * 3 + 2);
  return {row(cam, x, y, z), row(cam + 4, x, y, z), row(cam + 8, x, y, z)};
}

// A front-facing face in camera space: oriented edge normals e_k (every w_k >= 0 inside), num = -det > 0, the pixel box, the frame's
// intrinsics and the key's face id.
struct Tri {
  V3 e[3];
  double num, fx, cx, fy, cy;
  int32_t x0, x1, y0, y1, frame;
  uint32_t face;
};

// The face's vertices in camera space and its Tri; false when it is back-facing or degenerate (det >= 0 or NaN).
__device__ __forceinline__ bool setup(const float* cam, const float* vertices, const int64_t* faces, int64_t f, V3 (&v)[3], Tri& t) {
#pragma unroll
  for (int k = 0; k < 3; ++k) v[k] = to_camera(cam, vertices, __ldg(faces + f * 3 + k));
  const V3 E0 = cross(v[1], v[2]), E1 = cross(v[2], v[0]), E2 = cross(v[0], v[1]);
  const double det = dot(v[0], E0);
  if (!(det < 0.0)) return false;
  t.e[0] = neg(E0);
  t.e[1] = neg(E1);
  t.e[2] = neg(E2);
  t.num = -det;
  t.fx = __ldg(cam + 12);
  t.cx = __ldg(cam + 14);
  t.fy = __ldg(cam + 16);
  t.cy = __ldg(cam + 17);
  t.face = (uint32_t)f;
  return true;
}

// w_k of the ray through pixel (i, j); returns the depth, or a negative value when the face does not cover the pixel
__device__ __forceinline__ double edge_test(const Tri& t, int32_t i, int32_t j, double z_near, double (&w)[3], V3& d) {
  d.x = __ddiv_rn(__dsub_rn((double)i + 0.5, t.cx), t.fx);
  d.y = -__ddiv_rn(__dsub_rn((double)j + 0.5, t.cy), t.fy);
  d.z = -1.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) w[k] = __dsub_rn(__dadd_rn(__dmul_rn(d.x, t.e[k].x), __dmul_rn(d.y, t.e[k].y)), t.e[k].z);
  const double S = __dadd_rn(__dadd_rn(w[0], w[1]), w[2]);
  if (!(w[0] >= 0.0 && w[1] >= 0.0 && w[2] >= 0.0 && S > 0.0)) return -1.0;
  const double depth = __ddiv_rn(t.num, S);
  return depth >= z_near ? depth : -1.0;
}

__device__ __forceinline__ void cover(const Tri& t, int32_t i, int32_t j, double z_near, unsigned long long* keys, int32_t W) {
  double w[3];
  V3 d;
  const double depth = edge_test(t, i, j, z_near, w, d);
  if (depth < 0.0) return;
  const unsigned long long key = ((unsigned long long)__float_as_uint(__double2float_rn(depth)) << 32) | t.face;
  atomicMin(keys + (int64_t)j * W + i, key);
}

// widen the projected box by the projection of the camera-space point (x, y, -depth), depth > 0
__device__ __forceinline__ void extend_box(double (&box)[4], const Tri& t, double x, double y, double depth) {
  const double px = t.cx + t.fx * (x / depth), py = t.cy - t.fy * (y / depth);
  box[0] = fmin(box[0], px);
  box[1] = fmax(box[1], px);
  box[2] = fmin(box[2], py);
  box[3] = fmax(box[3], py);
}

// clamp a projected pixel coordinate to [-1, n] before the integer conversion (it may be huge, or infinite)
__device__ __forceinline__ int32_t clamp_px(double p, int32_t n) { return (int32_t)fmin(fmax(p, -1.0), (double)n); }

__global__ void __launch_bounds__(kRasterThreads)
    k_mesh_rasterize(const float* __restrict__ vertices, const int64_t* __restrict__ faces, int64_t F, const float* __restrict__ cams, int32_t B,
                     int32_t H, int32_t W, double z_near, int64_t large_pixels, unsigned long long* __restrict__ keys) {
  __shared__ Tri queue[kRasterThreads];
  __shared__ int n_queued;
  if (threadIdx.x == 0) n_queued = 0;
  __syncthreads();
  const int64_t tid = (int64_t)blockIdx.x * kRasterThreads + threadIdx.x;
  Tri t;
  bool live = false;
  int64_t pixels = 0;
  if (tid < (int64_t)B * F) {
    const int32_t b = (int32_t)(tid / F);
    const int64_t f = tid - (int64_t)b * F;
    const float* cam = cams + (int64_t)b * kCamFloats;
    V3 v[3];
    live = setup(cam, vertices, faces, f, v, t);
    if (live) {
      const double z0 = -v[0].z, z1 = -v[1].z, z2 = -v[2].z;
      live = fmax(fmax(z0, z1), z2) >= 0.5 * z_near;
    }
    if (live) {
      t.frame = b;
      // Every hit that can cover a pixel has view depth >= z_near, so it lies in the part of the face at depth >= z_near / 2: the
      // face clipped by that plane (at most four corners, all in front of the camera).  A covered pixel centre lies in the hull of
      // the clipped corners' projections.
      const double c = 0.5 * z_near;
      double box[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};   // projected x min, max, y min, max
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const V3& a = v[k];
        const V3& e = v[k == 2 ? 0 : k + 1];
        const double da = -a.z, de = -e.z;
        if (da >= c) extend_box(box, t, a.x, a.y, da);
        if ((da >= c) != (de >= c)) {
          const double s = (c - da) / (de - da);
          extend_box(box, t, a.x + (e.x - a.x) * s, a.y + (e.y - a.y) * s, c);
        }
      }
      const double pxmin = box[0], pxmax = box[1], pymin = box[2], pymax = box[3];
      t.x0 = max(clamp_px(ceil(pxmin - 0.5), W) - 1, 0);
      t.x1 = min(clamp_px(floor(pxmax - 0.5), W) + 1, W - 1);
      t.y0 = max(clamp_px(ceil(pymin - 0.5), H) - 1, 0);
      t.y1 = min(clamp_px(floor(pymax - 0.5), H) + 1, H - 1);
      live = t.x0 <= t.x1 && t.y0 <= t.y1;
      pixels = (int64_t)(t.x1 - t.x0 + 1) * (t.y1 - t.y0 + 1);
    }
    if (live && pixels > large_pixels) {
      queue[atomicAdd(&n_queued, 1)] = t;
      live = false;
    }
  }
  if (live) {
    unsigned long long* fk = keys + (int64_t)t.frame * H * W;
    for (int32_t j = t.y0; j <= t.y1; ++j)
      for (int32_t i = t.x0; i <= t.x1; ++i) cover(t, i, j, z_near, fk, W);
  }
  __syncthreads();
  const int nq = n_queued;
  for (int q = 0; q < nq; ++q) {
    const Tri& s = queue[q];
    const int32_t bw = s.x1 - s.x0 + 1;
    const int64_t n = (int64_t)bw * (s.y1 - s.y0 + 1);
    unsigned long long* fk = keys + (int64_t)s.frame * H * W;
    for (int64_t p = threadIdx.x; p < n; p += kRasterThreads) cover(s, s.x0 + (int32_t)(p % bw), s.y0 + (int32_t)(p / bw), z_near, fk, W);
  }
}

struct Lights {
  double colour[4][3], diffuse[4], specular[4], shininess[4], ambient[3];
};

__device__ __forceinline__ V3 normalized(const V3& a) {
  const double n = __dsqrt_rn(dot(a, a));
  return n > 0.0 ? V3{__ddiv_rn(a.x, n), __ddiv_rn(a.y, n), __ddiv_rn(a.z, n)} : a;
}
__device__ __forceinline__ V3 blend(const double (&b)[3], const V3 (&n)[3]) {
  return {__dadd_rn(__dadd_rn(__dmul_rn(b[0], n[0].x), __dmul_rn(b[1], n[1].x)), __dmul_rn(b[2], n[2].x)),
          __dadd_rn(__dadd_rn(__dmul_rn(b[0], n[0].y), __dmul_rn(b[1], n[1].y)), __dmul_rn(b[2], n[2].y)),
          __dadd_rn(__dadd_rn(__dmul_rn(b[0], n[0].z), __dmul_rn(b[1], n[1].z)), __dmul_rn(b[2], n[2].z))};
}
__device__ __forceinline__ uint8_t quantise(double c) {
  return (uint8_t)floor(__dadd_rn(__dmul_rn(fmin(fmax(c, 0.0), 1.0), 255.0), 0.5));
}

__global__ void __launch_bounds__(kShadeThreads)
    k_mesh_shade(const unsigned long long* __restrict__ keys, int32_t B, int32_t H, int32_t W, const float* __restrict__ vertices,
                 const float* __restrict__ vertex_normals, const int64_t* __restrict__ faces, const float* __restrict__ cams,
                 const float* __restrict__ light_positions, Lights L, uint8_t* __restrict__ rgb, uint8_t* __restrict__ normal) {
  const int64_t p = (int64_t)blockIdx.x * kShadeThreads + threadIdx.x;
  const int64_t plane = (int64_t)H * W;
  if (p >= (int64_t)B * plane) return;
  const unsigned long long key = __ldg(keys + p);
  if (key == kBackground) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (rgb) rgb[p * 3 + c] = 255;
      if (normal) normal[p * 3 + c] = 255;
    }
    return;
  }
  const int32_t b = (int32_t)(p / plane), j = (int32_t)((p - (int64_t)b * plane) / W), i = (int32_t)(p - (int64_t)b * plane - (int64_t)j * W);
  const int64_t f = (int64_t)(key & 0xffffffffull);
  const float* cam = cams + (int64_t)b * kCamFloats;
  V3 v[3];
  Tri t;
  setup(cam, vertices, faces, f, v, t);   // the key came from this face, so it is front-facing
  double w[3];
  V3 d;
  const double depth = edge_test(t, i, j, -INFINITY, w, d);   // the rasterizer's depth: this pixel passed its test
  const double S = __dadd_rn(__dadd_rn(w[0], w[1]), w[2]);
  const double bc[3] = {__ddiv_rn(w[0], S), __ddiv_rn(w[1], S), __ddiv_rn(w[2], S)};
  V3 n[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int64_t vi = __ldg(faces + f * 3 + k);
    const double nx = __ldg(vertex_normals + vi * 3), ny = __ldg(vertex_normals + vi * 3 + 1), nz = __ldg(vertex_normals + vi * 3 + 2);
    n[k] = {__dadd_rn(__dadd_rn(__dmul_rn((double)__ldg(cam), nx), __dmul_rn((double)__ldg(cam + 1), ny)), __dmul_rn((double)__ldg(cam + 2), nz)),
            __dadd_rn(__dadd_rn(__dmul_rn((double)__ldg(cam + 4), nx), __dmul_rn((double)__ldg(cam + 5), ny)), __dmul_rn((double)__ldg(cam + 6), nz)),
            __dadd_rn(__dadd_rn(__dmul_rn((double)__ldg(cam + 8), nx), __dmul_rn((double)__ldg(cam + 9), ny)), __dmul_rn((double)__ldg(cam + 10), nz))};
  }
  if (normal) {
    const V3 nn = normalized(blend(bc, n));
    normal[p * 3] = quantise(__dadd_rn(__dmul_rn(nn.x, 0.5), 0.5));
    normal[p * 3 + 1] = quantise(__dadd_rn(__dmul_rn(nn.y, 0.5), 0.5));
    normal[p * 3 + 2] = quantise(__dadd_rn(__dmul_rn(nn.z, 0.5), 0.5));
  }
  if (rgb) {
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (dot(n[k], neg(v[k])) < 0.0) n[k] = neg(n[k]);
    const V3 nn = normalized(blend(bc, n));
    const V3 hit = {__dmul_rn(depth, d.x), __dmul_rn(depth, d.y), __dmul_rn(depth, d.z)};
    const V3 e = normalized(neg(hit));
    double c[3] = {L.ambient[0], L.ambient[1], L.ambient[2]};
    const float* lp = light_positions + (int64_t)b * 12;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const V3 l = normalized({__dsub_rn((double)__ldg(lp + 3 * k), hit.x), __dsub_rn((double)__ldg(lp + 3 * k + 1), hit.y),
                               __dsub_rn((double)__ldg(lp + 3 * k + 2), hit.z)});
      const double ndl = dot(nn, l), two = __dmul_rn(2.0, ndl);
      const V3 r = {__dsub_rn(__dmul_rn(two, nn.x), l.x), __dsub_rn(__dmul_rn(two, nn.y), l.y), __dsub_rn(__dmul_rn(two, nn.z), l.z)};
      const double edr = dot(e, r);
      const double spec = edr > 0.0 ? pow(edr, L.shininess[k]) : 0.0;
      const double s = __dadd_rn(__dmul_rn(L.diffuse[k], fmax(ndl, 0.0)), __dmul_rn(L.specular[k], spec));
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) c[ch] = __dadd_rn(c[ch], __dmul_rn(L.colour[k][ch], s));
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) rgb[p * 3 + ch] = quantise(c[ch]);
  }
}

bool aligned(const void* p, size_t a) { return ((uintptr_t)p % a) == 0; }

int check_frames(const float* vertices, const int64_t* faces, int64_t n_faces, const float* cams, int32_t n_frames, int32_t height, int32_t width,
                 float z_near) {
  SDFB_REQUIRE(n_frames >= 0, "n_frames must be >= 0");
  SDFB_REQUIRE(height >= 1 && height <= SDFB200_MESH_MAX_SIDE && width >= 1 && width <= SDFB200_MESH_MAX_SIDE,
               "height and width must lie in [1, SDFB200_MESH_MAX_SIDE]");
  SDFB_REQUIRE(n_faces >= 0 && n_faces < INT32_MAX, "n_faces must lie in [0, 2^31 - 1)");
  SDFB_REQUIRE(isfinite(z_near) && z_near > 0.f, "z_near must be finite and > 0");
  if (n_frames == 0) return 0;
  SDFB_REQUIRE(cams && aligned(cams, 4), "cams NULL or misaligned");
  SDFB_REQUIRE(n_faces == 0 || (vertices && faces && aligned(vertices, 4) && aligned(faces, 8)), "vertices or faces NULL or misaligned");
  return 0;
}

}  // namespace

// the rasterizer with the large-box threshold as a parameter: the product entry passes SDFB200_MESH_LARGE_TRIANGLE_PIXELS, the debug
// library's hook any value (tools/render_mesh_bench.py times each path on its own)
int mesh_rasterize(const float* vertices, const int64_t* faces, int64_t n_faces, const float* cams, int32_t n_frames, int32_t height, int32_t width,
                   float z_near, uint64_t* keys, int64_t large_pixels, void* stream) {
  const int rc = check_frames(vertices, faces, n_faces, cams, n_frames, height, width, z_near);
  if (rc) return rc;
  if (n_frames == 0) return 0;
  SDFB_REQUIRE(keys && aligned(keys, 8), "keys NULL or misaligned");
  const cudaStream_t st = (cudaStream_t)stream;
  SDFB_CUDA(cudaMemsetAsync(keys, 0xff, (size_t)n_frames * height * width * sizeof(uint64_t), st));
  if (n_faces == 0) return 0;
  const int64_t pairs = (int64_t)n_frames * n_faces;
  SDFB_REQUIRE(ceil_div(pairs, kRasterThreads) < INT32_MAX, "n_frames * n_faces too large for one launch");
  k_mesh_rasterize<<<(unsigned)ceil_div(pairs, kRasterThreads), kRasterThreads, 0, st>>>(
      vertices, faces, n_faces, cams, n_frames, height, width, (double)z_near, large_pixels, reinterpret_cast<unsigned long long*>(keys));
  SDFB_LAUNCHED("k_mesh_rasterize");
  return 0;
}

}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_mesh_rasterize(const float* vertices, const int64_t* faces, int64_t n_faces, const float* cams, int32_t n_frames,
                                      int32_t height, int32_t width, float z_near, uint64_t* keys, void* stream) {
  return mesh_rasterize(vertices, faces, n_faces, cams, n_frames, height, width, z_near, keys, SDFB200_MESH_LARGE_TRIANGLE_PIXELS, stream);
}

extern "C" int sdfb200_mesh_shade(const uint64_t* keys, int32_t n_frames, int32_t height, int32_t width, const float* vertices,
                                  const float* vertex_normals, const int64_t* faces, int64_t n_faces, const float* cams,
                                  const float* light_positions, const float* light_params, uint8_t* rgb, uint8_t* normal, void* stream) {
  const int rc = check_frames(vertices, faces, n_faces, cams, n_frames, height, width, 1.f);
  if (rc) return rc;
  SDFB_REQUIRE(rgb || normal, "neither output given");
  SDFB_REQUIRE(light_params, "light_params NULL");
  if (n_frames == 0) return 0;
  SDFB_REQUIRE(keys && aligned(keys, 8), "keys NULL or misaligned");
  SDFB_REQUIRE(n_faces == 0 || (vertex_normals && aligned(vertex_normals, 4)), "vertex_normals NULL or misaligned");
  SDFB_REQUIRE(!rgb || (light_positions && aligned(light_positions, 4)), "light_positions NULL or misaligned");
  Lights L;
  for (int k = 0; k < 4; ++k) {
    for (int c = 0; c < 3; ++c) L.colour[k][c] = light_params[6 * k + c];
    L.diffuse[k] = light_params[6 * k + 3];
    L.specular[k] = light_params[6 * k + 4];
    L.shininess[k] = light_params[6 * k + 5];
  }
  for (int c = 0; c < 3; ++c) L.ambient[c] = light_params[24 + c];
  const int64_t n = (int64_t)n_frames * height * width;
  SDFB_REQUIRE(ceil_div(n, kShadeThreads) < INT32_MAX, "too many pixels for one launch");
  k_mesh_shade<<<(unsigned)ceil_div(n, kShadeThreads), kShadeThreads, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const unsigned long long*>(keys), n_frames, height, width, vertices, vertex_normals, faces, cams, light_positions, L, rgb,
      normal);
  SDFB_LAUNCHED("k_mesh_shade");
  return 0;
}
