// Point-cloud cleaning and normals (open3d's RemoveStatisticalOutliers and EstimateNormals, as the reference's
// exporter_utils.generate_point_cloud calls them) on a uniform grid of the cloud.
//   k_knn:           exact k nearest neighbours, one thread per point, the threads in cell order.  Each thread searches Chebyshev
//                    shells of cells around its own and keeps the k best (squared distance, original index) pairs in registers,
//                    sorted, until the k-th is no farther than every cell not yet visited.
//   k_point_normals: per point, the covariance of its neighbour list in open3d's cumulant form and the eigenvector of its smallest
//                    eigenvalue (cyclic Jacobi, double).
// The cell size is a power of two 2^e and the cell of a coordinate x is floor(x 2^-e) - cell_min: both scalings are exact in double,
// so the cell is exactly the one whose walls [j 2^e, (j + 1) 2^e) hold x, and the distance to a wall is computed from exact
// operands.  The op order is documented in include/sdfb200.h.
#include <math.h>

#include "common.cuh"

namespace sdfb200 {
namespace {

constexpr int kKnnThreads = 128;
constexpr int kNormalThreads = 128;

struct KnnGrid {
  int32_t dims[3];
  int64_t cmin[3];
  double inv_h, h;   // 2^-e, 2^e
};

__device__ __forceinline__ double sq_dist(float ax, float ay, float az, float bx, float by, float bz) {
  const double dx = __dsub_rn((double)ax, (double)bx), dy = __dsub_rn((double)ay, (double)by), dz = __dsub_rn((double)az, (double)bz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// (d, i) before (e, j): ascending squared distance, then ascending original index
__device__ __forceinline__ bool before(double d, int32_t i, double e, int32_t j) { return d < e || (d == e && i < j); }

// The k best pairs, sorted, in slots KB-k..KB-1 of a list of KB; slots below KB-k hold sentinels that sort before every pair and never
// move.  So the k-th entry is always slot KB-1 and every slot index is known at compile time: the list stays in registers.
template <int KB>
struct TopK {
  double d[KB];
  int32_t i[KB];

  __device__ __forceinline__ void init(int k) {
#pragma unroll
    for (int j = 0; j < KB; ++j) {
      const bool sentinel = j < KB - k;
      d[j] = sentinel ? -INFINITY : INFINITY;
      i[j] = sentinel ? INT32_MIN : INT32_MAX;
    }
  }
  __device__ __forceinline__ bool passes(double dn, int32_t in) const { return before(dn, in, d[KB - 1], i[KB - 1]); }
  __device__ __forceinline__ void insert(double dn, int32_t in) {
#pragma unroll
    for (int j = KB - 1; j >= 0; --j) {
      if (j > 0 && before(dn, in, d[j > 0 ? j - 1 : 0], i[j > 0 ? j - 1 : 0])) {
        d[j] = d[j > 0 ? j - 1 : 0];
        i[j] = i[j > 0 ? j - 1 : 0];
      } else if (before(dn, in, d[j], i[j])) {
        d[j] = dn;
        i[j] = in;
      }
    }
  }
};

// cell of coordinate x along axis a: floor(x 2^-e) - cmin[a], clamped to the grid (a no-op for a coordinate inside the box)
__device__ __forceinline__ int32_t cell_of(float x, const KnnGrid& g, int a) {
  const int64_t c = (int64_t)floor(__dmul_rn((double)x, g.inv_h)) - g.cmin[a];
  return (int32_t)(c < 0 ? 0 : (c >= g.dims[a] ? g.dims[a] - 1 : c));
}

template <int KB>
__global__ void __launch_bounds__(kKnnThreads)
    k_knn(const float* __restrict__ pts, const int32_t* __restrict__ order, int64_t n, const int32_t* __restrict__ cell_start, KnnGrid g,
          int k, double* __restrict__ mean_dist, int32_t* __restrict__ indices) {
  const int64_t s = (int64_t)blockIdx.x * kKnnThreads + threadIdx.x;
  if (s >= n) return;
  const float qx = __ldg(pts + s * 3), qy = __ldg(pts + s * 3 + 1), qz = __ldg(pts + s * 3 + 2);
  const float q[3] = {qx, qy, qz};
  int32_t c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = cell_of(q[a], g, a);
  const int k_eff = (int64_t)k < n ? k : (int)n;
  int32_t rmax = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int32_t m = c[a] > g.dims[a] - 1 - c[a] ? c[a] : g.dims[a] - 1 - c[a];
    rmax = m > rmax ? m : rmax;
  }
  TopK<KB> top;
  top.init(k);
  int held = 0;
  const int64_t row = g.dims[0], plane = (int64_t)g.dims[0] * g.dims[1];
  for (int32_t r = 0; r <= rmax; ++r) {
    const int32_t z0 = c[2] - r < 0 ? 0 : c[2] - r, z1 = c[2] + r >= g.dims[2] ? g.dims[2] - 1 : c[2] + r;
    const int32_t y0 = c[1] - r < 0 ? 0 : c[1] - r, y1 = c[1] + r >= g.dims[1] ? g.dims[1] - 1 : c[1] + r;
    const int32_t x0 = c[0] - r < 0 ? 0 : c[0] - r, x1 = c[0] + r >= g.dims[0] ? g.dims[0] - 1 : c[0] + r;
    for (int32_t z = z0; z <= z1; ++z) {
      for (int32_t y = y0; y <= y1; ++y) {
        const bool face = z == c[2] - r || z == c[2] + r || y == c[1] - r || y == c[1] + r;
        // on a face of the shell the whole clipped row is new; inside it only the two end cells are
        for (int part = 0; part < (face ? 1 : 2); ++part) {
          int32_t xa = x0, xb = x1;
          if (!face) {
            xa = xb = part == 0 ? c[0] - r : c[0] + r;
            if (xa < 0 || xa >= g.dims[0]) continue;
          }
          const int64_t base = z * plane + y * row;
          const int32_t j0 = __ldg(cell_start + base + xa), j1 = __ldg(cell_start + base + xb + 1);
          for (int32_t j = j0; j < j1; ++j) {
            const double d = sq_dist(__ldg(pts + (int64_t)j * 3), __ldg(pts + (int64_t)j * 3 + 1), __ldg(pts + (int64_t)j * 3 + 2), qx, qy, qz);
            const int32_t id = __ldg(order + j);
            if (top.passes(d, id)) {
              top.insert(d, id);
              held += held < k;
            }
          }
        }
      }
    }
    if (held < k_eff) continue;
    // squared distance to the nearest cell not yet visited: the nearest wall of the visited cube that has cells beyond it
    double g2 = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double qa = (double)q[a];
      if (c[a] - r > 0) {
        const double gap = __dsub_rn(qa, __dmul_rn((double)(g.cmin[a] + c[a] - r), g.h));
        g2 = fmin(g2, __dmul_rn(gap, gap));
      }
      if (c[a] + r + 1 < g.dims[a]) {
        const double gap = __dsub_rn(__dmul_rn((double)(g.cmin[a] + c[a] + r + 1), g.h), qa);
        g2 = fmin(g2, __dmul_rn(gap, gap));
      }
    }
    // (1 - 2^-48) absorbs the rounding of both sides, so a point beyond the wall is strictly farther than the k-th
    if (top.d[KB - 1] <= __dmul_rn(g2, 0x1.fffffffffffcp-1)) break;
  }
  const int64_t orig = __ldg(order + s);
  if (mean_dist) {
    double sum = 0.0;
#pragma unroll
    for (int j = 0; j < KB; ++j)
      if (j >= KB - k && j < KB - k + k_eff) sum = __dadd_rn(sum, __dsqrt_rn(top.d[j]));
    mean_dist[orig] = __ddiv_rn(sum, (double)k_eff);
  }
  if (indices) {
    const int64_t row0 = orig * k - (KB - k);   // slot j goes to column j - (KB - k)
#pragma unroll
    for (int j = 0; j < KB; ++j)
      if (j >= KB - k) indices[row0 + j] = j < KB - k + k_eff ? top.i[j] : -1;
  }
}

// one Jacobi rotation zeroing a[p][q] of the symmetric a, accumulated into the columns of v
template <int P, int Q>
__device__ __forceinline__ void jacobi_rotate(double (&a)[3][3], double (&v)[3][3]) {
  constexpr int R = 3 - P - Q;
  const double apq = a[P][Q];
  if (apq == 0.0) return;
  const double app = a[P][P], aqq = a[Q][Q];
  // negligible against both diagonal entries: set it to zero
  const double g = __dmul_rn(100.0, fabs(apq));
  if (__dadd_rn(fabs(app), g) == fabs(app) && __dadd_rn(fabs(aqq), g) == fabs(aqq)) {
    a[P][Q] = a[Q][P] = 0.0;
    return;
  }
  const double theta = __ddiv_rn(__dsub_rn(aqq, app), __dmul_rn(2.0, apq));
  double t;
  if (fabs(theta) > 1e150) {
    t = __ddiv_rn(0.5, theta);
  } else {
    t = __ddiv_rn(1.0, __dadd_rn(fabs(theta), __dsqrt_rn(__dadd_rn(__dmul_rn(theta, theta), 1.0))));
    if (theta < 0.0) t = -t;
  }
  const double cs = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(__dmul_rn(t, t), 1.0))), sn = __dmul_rn(t, cs);
  a[P][P] = __dsub_rn(app, __dmul_rn(t, apq));
  a[Q][Q] = __dadd_rn(aqq, __dmul_rn(t, apq));
  a[P][Q] = a[Q][P] = 0.0;
  const double arp = a[R][P], arq = a[R][Q];
  a[R][P] = a[P][R] = __dsub_rn(__dmul_rn(cs, arp), __dmul_rn(sn, arq));
  a[R][Q] = a[Q][R] = __dadd_rn(__dmul_rn(sn, arp), __dmul_rn(cs, arq));
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double vp = v[r][P], vq = v[r][Q];
    v[r][P] = __dsub_rn(__dmul_rn(cs, vp), __dmul_rn(sn, vq));
    v[r][Q] = __dadd_rn(__dmul_rn(sn, vp), __dmul_rn(cs, vq));
  }
}

__global__ void __launch_bounds__(kNormalThreads)
    k_point_normals(const float* __restrict__ pts, int64_t n, const int32_t* __restrict__ indices, int k, float* __restrict__ normals) {
  const int64_t i = (int64_t)blockIdx.x * kNormalThreads + threadIdx.x;
  if (i >= n) return;
  double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};   // x, y, z, xx, xy, xz, yy, yz, zz
  int cnt = 0;
  for (int j = 0; j < k; ++j) {
    const int32_t id = __ldg(indices + i * k + j);
    if (id < 0) continue;
    const double x = __ldg(pts + (int64_t)id * 3), y = __ldg(pts + (int64_t)id * 3 + 1), z = __ldg(pts + (int64_t)id * 3 + 2);
    m[0] = __dadd_rn(m[0], x);
    m[1] = __dadd_rn(m[1], y);
    m[2] = __dadd_rn(m[2], z);
    m[3] = __dadd_rn(m[3], __dmul_rn(x, x));
    m[4] = __dadd_rn(m[4], __dmul_rn(x, y));
    m[5] = __dadd_rn(m[5], __dmul_rn(x, z));
    m[6] = __dadd_rn(m[6], __dmul_rn(y, y));
    m[7] = __dadd_rn(m[7], __dmul_rn(y, z));
    m[8] = __dadd_rn(m[8], __dmul_rn(z, z));
    ++cnt;
  }
  float3 out = make_float3(0.f, 0.f, 1.f);
  if (cnt > 0) {
#pragma unroll
    for (int t = 0; t < 9; ++t) m[t] = __ddiv_rn(m[t], (double)cnt);
    double a[3][3];
    a[0][0] = __dsub_rn(m[3], __dmul_rn(m[0], m[0]));
    a[0][1] = a[1][0] = __dsub_rn(m[4], __dmul_rn(m[0], m[1]));
    a[0][2] = a[2][0] = __dsub_rn(m[5], __dmul_rn(m[0], m[2]));
    a[1][1] = __dsub_rn(m[6], __dmul_rn(m[1], m[1]));
    a[1][2] = a[2][1] = __dsub_rn(m[7], __dmul_rn(m[1], m[2]));
    a[2][2] = __dsub_rn(m[8], __dmul_rn(m[2], m[2]));
    const bool zero = a[0][0] == 0.0 && a[0][1] == 0.0 && a[0][2] == 0.0 && a[1][1] == 0.0 && a[1][2] == 0.0 && a[2][2] == 0.0;
    if (!zero) {
      double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
      for (int sweep = 0; sweep < 32 && (a[0][1] != 0.0 || a[0][2] != 0.0 || a[1][2] != 0.0); ++sweep) {
        jacobi_rotate<0, 1>(a, v);
        jacobi_rotate<0, 2>(a, v);
        jacobi_rotate<1, 2>(a, v);
      }
      // the smallest eigenvalue, the first axis on ties
      int e = 0;
      if (a[1][1] < a[e][e]) e = 1;
      if (a[2][2] < (e == 0 ? a[0][0] : a[1][1])) e = 2;
      double nv[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) nv[r] = e == 0 ? v[r][0] : (e == 1 ? v[r][1] : v[r][2]);
      // sign, on the fp32 vector that is written: the component of largest magnitude is positive, the first axis on ties
      const float f0 = (float)nv[0], f1 = (float)nv[1], f2 = (float)nv[2];
      float big = f0;
      if (fabsf(f1) > fabsf(big)) big = f1;
      if (fabsf(f2) > fabsf(big)) big = f2;
      out = big < 0.f ? make_float3(-f0, -f1, -f2) : make_float3(f0, f1, f2);
    }
  }
  normals[i * 3] = out.x;
  normals[i * 3 + 1] = out.y;
  normals[i * 3 + 2] = out.z;
}

template <int KB>
void launch_knn(const float* pts, const int32_t* order, int64_t n, const int32_t* cell_start, const KnnGrid& g, int k, double* mean_dist,
                int32_t* indices, cudaStream_t st) {
  k_knn<KB><<<(unsigned)ceil_div(n, kKnnThreads), kKnnThreads, 0, st>>>(pts, order, n, cell_start, g, k, mean_dist, indices);
}

}  // namespace
}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_knn(const float* points, const int32_t* order, int64_t n_points, const int32_t* cell_start, const float* box,
                           int32_t log2_cell, int32_t k, double* mean_dist, int32_t* indices, void* stream) {
  SDFB_REQUIRE(k >= 1 && k <= 32, "k must lie in [1, 32]");
  SDFB_REQUIRE(n_points >= 0 && n_points <= INT32_MAX, "n_points must lie in [0, 2^31)");
  SDFB_REQUIRE(mean_dist || indices, "neither output given");
  if (n_points == 0) return 0;
  SDFB_REQUIRE(points && order && cell_start && box, "NULL pointer");
  SDFB_REQUIRE(log2_cell >= -160 && log2_cell <= 140, "log2_cell must lie in [-160, 140]");
  KnnGrid g;
  g.h = ldexp(1.0, log2_cell);
  g.inv_h = ldexp(1.0, -log2_cell);
  int64_t cells = 1;
  for (int a = 0; a < 3; ++a) {
    SDFB_REQUIRE(isfinite(box[a]) && isfinite(box[a + 3]), "non-finite point (the box of the cloud is not finite)");
    SDFB_REQUIRE(box[a] <= box[a + 3], "box min > box max");
    const double lo = floor(ldexp((double)box[a], -log2_cell)), hi = floor(ldexp((double)box[a + 3], -log2_cell));
    SDFB_REQUIRE(fabs(lo) < 0x1p52 && fabs(hi) < 0x1p52 && hi - lo < 0x1p31, "cell size too small for the box");
    g.cmin[a] = (int64_t)lo;
    g.dims[a] = (int32_t)(hi - lo) + 1;
    cells *= g.dims[a];
    SDFB_REQUIRE(cells < INT32_MAX, "more than 2^31 - 2 cells");
  }
  const cudaStream_t st = (cudaStream_t)stream;
  if (k <= 8) launch_knn<8>(points, order, n_points, cell_start, g, k, mean_dist, indices, st);
  else if (k <= 16) launch_knn<16>(points, order, n_points, cell_start, g, k, mean_dist, indices, st);
  else if (k <= 24) launch_knn<24>(points, order, n_points, cell_start, g, k, mean_dist, indices, st);
  else launch_knn<32>(points, order, n_points, cell_start, g, k, mean_dist, indices, st);
  SDFB_LAUNCHED("k_knn");
  return 0;
}

extern "C" int sdfb200_point_normals(const float* points, int64_t n_points, const int32_t* indices, int32_t k, float* normals, void* stream) {
  SDFB_REQUIRE(k >= 1 && k <= 32, "k must lie in [1, 32]");
  SDFB_REQUIRE(n_points >= 0 && n_points <= INT32_MAX, "n_points must lie in [0, 2^31)");
  if (n_points == 0) return 0;
  SDFB_REQUIRE(points && indices && normals, "NULL pointer");
  k_point_normals<<<(unsigned)ceil_div(n_points, kNormalThreads), kNormalThreads, 0, (cudaStream_t)stream>>>(points, n_points, indices, k, normals);
  SDFB_LAUNCHED("k_point_normals");
  return 0;
}
