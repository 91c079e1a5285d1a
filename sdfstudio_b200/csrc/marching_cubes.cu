// Marching cubes on a dense fp32 volume (what skimage.measure.marching_cubes does on the host for utils/marching_cubes.py:133-142 /
// :201-209 / :305-314 of the reference).  One warp per (i, j) row of nz lattice points; lane l of a 32-point chunk handles point k and
// the cube whose lowest corner it is.  Two passes on the same inputs:
//   count: per row, the vertices its points own (each point owns its +x, +y, +z edges) and the triangles of its cubes;
//   emit:  with the exclusive cumsum of those counts, vertices / normals / faces are written in place.  A cube's edges owned by the
//          three neighbouring rows are ranked by recomputing those rows' edge flags, so no atomics decide a position.
// The cube conventions and the triangle table (mc_tables.h) come from the face rule restated in the oracle; every float operation of
// the vertices, normals and face decisions is rounded on its own (no FMA contraction) so that the oracle reproduces them bit for bit.
#include "common.cuh"
#include "mc_tables.h"

namespace sdfb200 {
namespace {

struct McArgs {
  const float* vol;
  const uint8_t* mask;
  int64_t nx, ny, nz;
  float level;
  float org[3], sp[3];
  const int32_t* counts;   // [2, nx*ny]: vertex counts then face counts
  int32_t* counts_out;
  const int64_t* offsets;  // [2, nx*ny] exclusive cumsum of counts
  float* verts;
  float* normals;
  int32_t* faces;
};

// corner m = (0,0), (1,0), (1,1), (0,1) of face f = A * 2 + side, over the two other axes U < V; corner n = dx | dy << 1 | dz << 2
__host__ __device__ constexpr int face_corner(int f, int m) {
  return ((f & 1) << (f >> 1)) | ((m == 1 || m == 2) << ((f >> 1) == 0 ? 1 : 0)) | ((m >= 2) << ((f >> 1) == 2 ? 1 : 2));
}
static_assert(face_corner(0, 2) == 6 && face_corner(3, 3) == 6 && face_corner(5, 1) == 5, "face corners");

__device__ __forceinline__ bool cube_on(const McArgs& a, int64_t i, int64_t j, int64_t k) {
  if (i < 0 || j < 0 || k < 0 || i > a.nx - 2 || j > a.ny - 2 || k > a.nz - 2) return false;
  return a.mask == nullptr || __ldg(a.mask + (i * a.ny + j) * a.nz + k) != 0;
}

__device__ __forceinline__ bool inside(const McArgs& a, int64_t p) { return __ldg(a.vol + p) < a.level; }

// bit `axis` set: the edge of point (i, j, k) along +axis is cut and belongs to a processed cube
__device__ unsigned edge_flags(const McArgs& a, int64_t i, int64_t j, int64_t k) {
  if (i >= a.nx || j >= a.ny || k >= a.nz) return 0u;
  const int64_t p = (i * a.ny + j) * a.nz + k;
  const bool in0 = inside(a, p);
  unsigned f = 0u;
  if (i + 1 < a.nx && inside(a, p + a.ny * a.nz) != in0 &&
      (cube_on(a, i, j, k) || cube_on(a, i, j - 1, k) || cube_on(a, i, j, k - 1) || cube_on(a, i, j - 1, k - 1)))
    f |= 1u;
  if (j + 1 < a.ny && inside(a, p + a.nz) != in0 &&
      (cube_on(a, i, j, k) || cube_on(a, i - 1, j, k) || cube_on(a, i, j, k - 1) || cube_on(a, i - 1, j, k - 1)))
    f |= 2u;
  if (k + 1 < a.nz && inside(a, p + 1) != in0 &&
      (cube_on(a, i, j, k) || cube_on(a, i - 1, j, k) || cube_on(a, i, j - 1, k) || cube_on(a, i - 1, j - 1, k)))
    f |= 4u;
  return f;
}

// table entry of the processed cube at (i, j, k), or -1 when it has no cut edge
__device__ int cube_entry(const McArgs& a, int64_t i, int64_t j, int64_t k) {
  const int64_t p0 = (i * a.ny + j) * a.nz + k;
  float rel[8];
  unsigned cas = 0u;
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    const float v = __ldg(a.vol + p0 + ((n & 1) ? a.ny * a.nz : 0) + ((n & 2) ? a.nz : 0) + ((n & 4) ? 1 : 0));
    rel[n] = __fsub_rn(v, a.level);
    cas |= (v < a.level ? 1u : 0u) << n;
  }
  if (cas == 0u || cas == 255u) return -1;
  const unsigned amb = mc::kAmbiguousFaces[cas];
  int bits = 0, r = 0;
#pragma unroll
  for (int f = 0; f < 6; ++f) {
    if ((amb >> f) & 1u) {
      // a, c: the outside diagonal pair; b, d: the inside pair, each in face order.  The denominator is > 0.
      const float a0 = rel[face_corner(f, 0)], b0 = rel[face_corner(f, 1)], c0 = rel[face_corner(f, 2)], d0 = rel[face_corner(f, 3)];
      const bool first_out = ((cas >> face_corner(f, 0)) & 1u) == 0u;
      const float av = first_out ? a0 : b0, cv = first_out ? c0 : d0, bv = first_out ? b0 : a0, dv = first_out ? d0 : c0;
      const float s = __fdiv_rn(__fsub_rn(__fmul_rn(av, cv), __fmul_rn(bv, dv)), __fsub_rn(__fsub_rn(__fadd_rn(av, cv), bv), dv));
      if (s < 0.f) bits |= 1 << r;
      ++r;
    }
  }
  return mc::kCaseEntry[cas] + bits;
}

__device__ __forceinline__ float corner_gradient(const McArgs& a, int64_t p, const int64_t (&idx)[3], int c) {
  const int64_t n = c == 0 ? a.nx : (c == 1 ? a.ny : a.nz);
  const int64_t stride = c == 0 ? a.ny * a.nz : (c == 1 ? a.nz : 1);
  const int64_t hi = idx[c] + 1 < n ? p + stride : p, lo = idx[c] > 0 ? p - stride : p;
  float d = __fsub_rn(__ldg(a.vol + hi), __ldg(a.vol + lo));
  if (idx[c] > 0 && idx[c] + 1 < n) d = __fmul_rn(d, 0.5f);
  return __fdiv_rn(d, a.sp[c]);
}

// vertex on the edge of point (i, j, k) along +axis
__device__ void emit_vertex(const McArgs& a, int64_t i, int64_t j, int64_t k, int axis, int64_t out) {
  const int64_t stride = axis == 0 ? a.ny * a.nz : (axis == 1 ? a.nz : 1);
  const int64_t p = (i * a.ny + j) * a.nz + k;
  const float v0 = __ldg(a.vol + p), v1 = __ldg(a.vol + p + stride);
  const float t = __fdiv_rn(__fsub_rn(a.level, v0), __fsub_rn(v1, v0));
  const int64_t idx0[3] = {i, j, k};
  const int64_t idx1[3] = {i + (axis == 0), j + (axis == 1), k + (axis == 2)};
  float g[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float pos = __fadd_rn(a.org[c], __fmul_rn(a.sp[c], __fadd_rn((float)idx0[c], c == axis ? t : 0.f)));
    a.verts[out * 3 + c] = pos;
    const float g0 = corner_gradient(a, p, idx0, c), g1 = corner_gradient(a, p + stride, idx1, c);
    g[c] = __fadd_rn(g0, __fmul_rn(t, __fsub_rn(g1, g0)));
  }
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(g[0], g[0]), __fmul_rn(g[1], g[1])), __fmul_rn(g[2], g[2])));
  const float inv = len > 0.f ? __fdiv_rn(1.f, len) : 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) a.normals[out * 3 + c] = -__fmul_rn(g[c], inv);
}

__device__ __forceinline__ int warp_excl_scan(int v, int lane, int& total) {
  const int x = warp_scan_incl(v, lane);
  total = __shfl_sync(0xffffffffu, x, 31);
  return x - v;
}

template <class T>
__device__ __forceinline__ T pick(const T (&v)[4], int r) {
  return r == 0 ? v[0] : (r == 1 ? v[1] : (r == 2 ? v[2] : v[3]));
}

__global__ void __launch_bounds__(256) k_mc_count(McArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t U = a.nx * a.ny;
  if (u >= U) return;
  const int64_t i = u / a.ny, j = u % a.ny;
  int nv = 0, nf = 0;
  for (int64_t k = lane; k < a.nz; k += 32) {
    nv += __popc(edge_flags(a, i, j, k));
    if (cube_on(a, i, j, k)) {
      const int e = cube_entry(a, i, j, k);
      if (e >= 0) nf += mc::kTriStart[e + 1] - mc::kTriStart[e];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    nv += __shfl_down_sync(0xffffffffu, nv, o);
    nf += __shfl_down_sync(0xffffffffu, nf, o);
  }
  if (lane == 0) {
    a.counts_out[u] = nv;
    a.counts_out[U + u] = nf;
  }
}

__global__ void __launch_bounds__(256) k_mc_emit(McArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t U = a.nx * a.ny;
  if (u >= U) return;
  if (__ldg(a.counts + u) == 0 && __ldg(a.counts + U + u) == 0) return;
  const int64_t i = u / a.ny, j = u % a.ny;
  const bool cube_row = i <= a.nx - 2 && j <= a.ny - 2;
  // rows r = dx | dy << 1: (i + dx, j + dy); the three neighbours only matter for the cubes of this row
  int64_t base[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) base[r] = (r == 0 || cube_row) ? __ldg(a.offsets + (i + (r & 1)) * a.ny + j + (r >> 1)) : 0;
  int64_t fbase = __ldg(a.offsets + U + u);
  for (int64_t k0 = 0; k0 < a.nz; k0 += 32) {
    const int64_t k = k0 + lane;
    unsigned fl[4];
    int excl[4], cnt[4], tot[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      fl[r] = (r == 0 || cube_row) ? edge_flags(a, i + (r & 1), j + (r >> 1), k) : 0u;
      cnt[r] = __popc(fl[r]);
      excl[r] = warp_excl_scan(cnt[r], lane, tot[r]);
    }
    // this row's vertices, by point then axis
    int64_t v = base[0] + excl[0];
#pragma unroll
    for (int ax = 0; ax < 3; ++ax)
      if ((fl[0] >> ax) & 1u) emit_vertex(a, i, j, k, ax, v++);
    // this row's cubes
    const int e = cube_row && cube_on(a, i, j, k) ? cube_entry(a, i, j, k) : -1;
    const int t0 = e >= 0 ? mc::kTriStart[e] : 0;
    const int ntri = e >= 0 ? mc::kTriStart[e + 1] - t0 : 0;
    int ftot;
    const int fexcl = warp_excl_scan(ntri, lane, ftot);
    // x flags of rows 0 and 1 at k + 1: rank of the y edges the cube's upper corners own
    unsigned xn[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      xn[r] = __shfl_down_sync(0xffffffffu, fl[r] & 1u, 1);
      if (lane == 31 && ntri > 0) xn[r] = edge_flags(a, i + r, j, k + 1) & 1u;
    }
    for (int t = 0; t < ntri; ++t) {
      int32_t tri[3];
#pragma unroll
      for (int m = 0; m < 3; ++m) {
        const int ed = mc::kTriEdges[(t0 + t) * 3 + m];
        const int axis = ed >> 2, b = ed & 3;
        const int row = axis == 0 ? (b & 1) << 1 : (axis == 1 ? (b & 1) : b);
        const int up = axis == 2 ? 0 : b >> 1;   // owner at k + 1
        int64_t id = pick(base, row) + pick(excl, row);
        if (up) id += pick(cnt, row) + (axis == 1 ? (int)(row == 0 ? xn[0] : xn[1]) : 0);
        else id += __popc(pick(fl, row) & ((1u << axis) - 1u));
        tri[m] = (int32_t)id;
      }
      const int64_t out = fbase + fexcl + t;
#pragma unroll
      for (int m = 0; m < 3; ++m) a.faces[out * 3 + m] = tri[m];
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) base[r] += tot[r];
    fbase += ftot;
  }
}

}  // namespace
}  // namespace sdfb200

using namespace sdfb200;

extern "C" size_t sdfb200_marching_cubes_workspace_bytes(const int64_t* dims) {
  if (dims == nullptr || dims[0] < 0 || dims[1] < 0 || dims[2] < 0) return 0;
  return (size_t)(2 * dims[0] * dims[1]) * sizeof(int32_t);
}

extern "C" int sdfb200_marching_cubes(const float* volume, const int64_t* dims, float level, const uint8_t* mask, const float* origin,
                                      const float* spacing, const int64_t* offsets, int32_t* counts, float* verts, float* normals,
                                      int32_t* faces, void* stream) {
  SDFB_REQUIRE(dims && origin && spacing, "NULL pointer");
  SDFB_REQUIRE(dims[0] >= 0 && dims[1] >= 0 && dims[2] >= 0, "bad sizes");
  SDFB_REQUIRE(dims[0] <= INT32_MAX && dims[1] <= INT32_MAX && dims[0] * dims[1] / 8 < INT32_MAX, "too many rows");
  const int64_t U = dims[0] * dims[1];
  if (U == 0 || dims[2] == 0) return 0;
  SDFB_REQUIRE(volume && counts, "NULL pointer");
  McArgs a;
  a.vol = volume; a.mask = mask; a.nx = dims[0]; a.ny = dims[1]; a.nz = dims[2]; a.level = level;
  for (int c = 0; c < 3; ++c) { a.org[c] = origin[c]; a.sp[c] = spacing[c]; }   // HOST arrays
  a.counts = counts; a.counts_out = counts; a.offsets = offsets; a.verts = verts; a.normals = normals; a.faces = faces;
  const unsigned blocks = (unsigned)ceil_div(U * 32, 256);
  if (offsets == nullptr) {
    k_mc_count<<<blocks, 256, 0, (cudaStream_t)stream>>>(a);
    SDFB_LAUNCHED("k_mc_count");
    return 0;
  }
  SDFB_REQUIRE(verts && normals && faces, "NULL pointer");
  k_mc_emit<<<blocks, 256, 0, (cudaStream_t)stream>>>(a);
  SDFB_LAUNCHED("k_mc_emit");
  return 0;
}
