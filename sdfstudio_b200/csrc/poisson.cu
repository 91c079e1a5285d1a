// Screened Poisson surface reconstruction on a dense grid (the discretisation of include/sdfb200.h, "Poisson").
//   k_cells:      per occupied cell, its points in bucket order: the 8x8 screening block M_c = sum phi phi^T, the 8 right-hand-side
//                 terms sum n.grad(phi), or the 8 splat weights sum phi with the colour sums sum phi rgb.  Double accumulation.
//   k_coarsen:    M_C = sum over the 8 children c of Q_c^T M_c Q_c.  Q_c interpolates the coarse hats on the child cell, so this is the
//                 coarse hats' screening matrix (the same sum over the same points), built without a pass over the points.
//   k_gather:     per node, the corner entries of its <= 8 adjacent occupied cells, in a fixed order.
//   k_sample:     trilinear interpolation of node values at points.
//   k_operator:   y = A x, r = f - A x or one damped l1-Jacobi sweep, A = L + alpha a S, one thread per node.  L is the Q1 stiffness
//                 with natural boundaries (analytic per node), S is read from the blocks of the adjacent cells.
//   k_restrict / k_prolong_add: the Q1 transfer operators (P^T and P).
// The solve is conjugate gradients preconditioned by one symmetric V-cycle per iteration; all reductions are in double over a fixed
// partition, so reruns are bit-identical.
#include <math.h>

#include "common.cuh"

namespace sdfb200 {
namespace {

constexpr int kThreads = 256;
constexpr int kDotBlocks = 1024;
constexpr int kCoarsest = 1;          // 2 cells per side, 27 nodes: solved by a dense Cholesky factor
constexpr int kCoarseNodes = 27;
constexpr double kOmega = 1.4;        // l1-Jacobi weight: l1-Jacobi converges for any weight < 2
constexpr int kSweeps = 2;

struct Grid {
  int32_t n;   // cells per side
  double o[3], h;
};

struct Level {
  int32_t n;
  double h;
  const int32_t* slot;   // [n^3] occupied-cell slot or -1
  const float* mat;      // [slots, 8, 8]
};

__host__ __device__ __forceinline__ int64_t node_count(int32_t n) { return (int64_t)(n + 1) * (n + 1) * (n + 1); }

// t = (p - o) / h, the cell floor(t) clamped to [0, n-1] and u = t - cell
__device__ __forceinline__ void locate(const float* p, const Grid& g, int32_t c[3], double u[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double t = __ddiv_rn(__dsub_rn((double)p[a], g.o[a]), g.h);
    double f = floor(t);
    f = f < 0.0 ? 0.0 : (f > (double)(g.n - 1) ? (double)(g.n - 1) : f);
    c[a] = (int32_t)f;
    u[a] = __dsub_rn(t, f);
  }
}

// hat of corner l = (lx, ly, lz), l = 4 lx + 2 ly + lz
__device__ __forceinline__ double hat(const double u[3], int l) {
  const double wx = (l & 4) ? u[0] : __dsub_rn(1.0, u[0]);
  const double wy = (l & 2) ? u[1] : __dsub_rn(1.0, u[1]);
  const double wz = (l & 1) ? u[2] : __dsub_rn(1.0, u[2]);
  return __dmul_rn(__dmul_rn(wx, wy), wz);
}

// MODE_SCREEN: mat + rhs (needs normals).  MODE_SPLAT: weight + colour sums into splat [slots, 8, 4].
enum { MODE_SCREEN = 0, MODE_SPLAT = 1 };

template <int MODE>
__global__ void __launch_bounds__(kThreads)
    k_cells(const float* __restrict__ pts, const float* __restrict__ aux, int64_t n_cells, const int64_t* __restrict__ key,
            const int64_t* __restrict__ start, Grid g, float* __restrict__ mat, float* __restrict__ rhs, float* __restrict__ splat) {
  const int64_t s = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (s >= n_cells) return;
  const int64_t p0 = start[s], p1 = start[s + 1];
  if constexpr (MODE == MODE_SCREEN) {
    double m[36], b[8];
#pragma unroll
    for (int t = 0; t < 36; ++t) m[t] = 0.0;
#pragma unroll
    for (int t = 0; t < 8; ++t) b[t] = 0.0;
    const double inv_h = __ddiv_rn(1.0, g.h);
    for (int64_t p = p0; p < p1; ++p) {
      int32_t c[3];
      double u[3], w[8];
      locate(pts + p * 3, g, c, u);
      const double nx = aux[p * 3], ny = aux[p * 3 + 1], nz = aux[p * 3 + 2];
      const double len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz)));
      const double n3[3] = {__ddiv_rn(nx, len), __ddiv_rn(ny, len), __ddiv_rn(nz, len)};
      const double v0[3] = {__dsub_rn(1.0, u[0]), __dsub_rn(1.0, u[1]), __dsub_rn(1.0, u[2])};
#pragma unroll
      for (int l = 0; l < 8; ++l) {
        w[l] = hat(u, l);
        const double wx = (l & 4) ? u[0] : v0[0], wy = (l & 2) ? u[1] : v0[1], wz = (l & 1) ? u[2] : v0[2];
        // n . grad(phi_l), grad(phi_l) = (sx wy wz, wx sy wz, wx wy sz) / h with s = +1 on the far corner, -1 on the near one
        const double gx = (l & 4) ? __dmul_rn(wy, wz) : -__dmul_rn(wy, wz);
        const double gy = (l & 2) ? __dmul_rn(wx, wz) : -__dmul_rn(wx, wz);
        const double gz = (l & 1) ? __dmul_rn(wx, wy) : -__dmul_rn(wx, wy);
        const double dn = __dadd_rn(__dadd_rn(__dmul_rn(n3[0], gx), __dmul_rn(n3[1], gy)), __dmul_rn(n3[2], gz));
        b[l] = __dadd_rn(b[l], __dmul_rn(dn, inv_h));
      }
      int t = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int l = k; l < 8; ++l, ++t) m[t] = __dadd_rn(m[t], __dmul_rn(w[k], w[l]));
    }
    int t = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
      for (int l = k; l < 8; ++l, ++t) {
        mat[s * 64 + k * 8 + l] = (float)m[t];
        mat[s * 64 + l * 8 + k] = (float)m[t];
      }
#pragma unroll
    for (int l = 0; l < 8; ++l) rhs[s * 8 + l] = (float)b[l];
  } else {
    double acc[32];
#pragma unroll
    for (int t = 0; t < 32; ++t) acc[t] = 0.0;
    for (int64_t p = p0; p < p1; ++p) {
      int32_t c[3];
      double u[3];
      locate(pts + p * 3, g, c, u);
      const double r = aux[p * 3], gr = aux[p * 3 + 1], bl = aux[p * 3 + 2];
#pragma unroll
      for (int l = 0; l < 8; ++l) {
        const double w = hat(u, l);
        acc[l * 4] = __dadd_rn(acc[l * 4], w);
        acc[l * 4 + 1] = __dadd_rn(acc[l * 4 + 1], __dmul_rn(w, r));
        acc[l * 4 + 2] = __dadd_rn(acc[l * 4 + 2], __dmul_rn(w, gr));
        acc[l * 4 + 3] = __dadd_rn(acc[l * 4 + 3], __dmul_rn(w, bl));
      }
    }
#pragma unroll
    for (int t = 0; t < 32; ++t) splat[s * 32 + t] = (float)acc[t];
  }
  (void)key;
}

// coarse hat K on child cell o (offsets 0/1 per axis) at the child's corner k: prod over axes of (K_a ? t : 1 - t), t = (o_a + k_a) / 2
__device__ __forceinline__ double q_entry(int o, int k, int K) {
  double q = 1.0;
#pragma unroll
  for (int a = 2; a >= 0; --a) {
    const double t = 0.5 * (double)(((o >> a) & 1) + ((k >> a) & 1));
    q *= ((K >> a) & 1) ? t : 1.0 - t;   // exact: t is 0, 1/2 or 1
  }
  return q;
}

// one thread per (coarse cell, row K)
__global__ void __launch_bounds__(kThreads)
    k_coarsen(int32_t nf, const int32_t* __restrict__ fine_slot, const float* __restrict__ fine_mat, int64_t n_cells,
              const int64_t* __restrict__ key, int32_t nc, float* __restrict__ mat) {
  const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (t >= n_cells * 8) return;
  const int64_t s = t >> 3;
  const int K = (int)(t & 7);
  const int64_t kk = key[s];
  const int64_t cz = kk % nc, cy = (kk / nc) % nc, cx = kk / ((int64_t)nc * nc);
  double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int o = 0; o < 8; ++o) {
    const int64_t fx = 2 * cx + ((o >> 2) & 1), fy = 2 * cy + ((o >> 1) & 1), fz = 2 * cz + (o & 1);
    const int32_t fs = fine_slot[(fx * nf + fy) * nf + fz];
    if (fs < 0) continue;
    const float* m = fine_mat + (int64_t)fs * 64;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const double qk = q_entry(o, k, K);
      if (qk == 0.0) continue;
      double row[8];
#pragma unroll
      for (int L = 0; L < 8; ++L) row[L] = 0.0;
#pragma unroll
      for (int l = 0; l < 8; ++l) {
        const double mkl = (double)m[k * 8 + l];
#pragma unroll
        for (int L = 0; L < 8; ++L) row[L] = fma(mkl, q_entry(o, l, L), row[L]);
      }
#pragma unroll
      for (int L = 0; L < 8; ++L) acc[L] = fma(qk, row[L], acc[L]);
    }
  }
#pragma unroll
  for (int L = 0; L < 8; ++L) mat[s * 64 + K * 8 + L] = (float)acc[L];
}

__device__ __forceinline__ void node_ijk(int64_t id, int32_t n, int32_t& i, int32_t& j, int32_t& k) {
  const int64_t m = n + 1;
  k = (int32_t)(id % m);
  j = (int32_t)((id / m) % m);
  i = (int32_t)(id / (m * m));
}

// per node, sum over the adjacent occupied cells (x, then y, then z offset, low first) of vals[slot * cs + corner * ks + ch]
__global__ void __launch_bounds__(kThreads)
    k_gather(int32_t n, const int32_t* __restrict__ slot, const float* __restrict__ vals, int cs, int ks, int channels,
             float* __restrict__ out) {
  const int64_t id = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (id >= node_count(n)) return;
  int32_t i, j, k;
  node_ijk(id, n, i, j, k);
  double acc[4] = {0, 0, 0, 0};
#pragma unroll
  for (int o = 0; o < 8; ++o) {
    const int32_t cx = i - 1 + ((o >> 2) & 1), cy = j - 1 + ((o >> 1) & 1), cz = k - 1 + (o & 1);
    if (cx < 0 || cy < 0 || cz < 0 || cx >= n || cy >= n || cz >= n) continue;
    const int32_t sl = slot[((int64_t)cx * n + cy) * n + cz];
    if (sl < 0) continue;
    const float* v = vals + (int64_t)sl * cs + (7 - o) * ks;
    for (int ch = 0; ch < channels; ++ch) acc[ch] += (double)v[ch];
  }
  for (int ch = 0; ch < channels; ++ch) out[id * channels + ch] = (float)acc[ch];
}

__global__ void __launch_bounds__(kThreads)
    k_sample(const float* __restrict__ pts, int64_t n_points, Grid g, const float* __restrict__ vals, int channels, double* __restrict__ out) {
  const int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (p >= n_points) return;
  int32_t c[3];
  double u[3];
  locate(pts + p * 3, g, c, u);
  const int64_t m = g.n + 1;
  double acc[4] = {0, 0, 0, 0};
#pragma unroll
  for (int l = 0; l < 8; ++l) {
    const double w = hat(u, l);
    const int64_t id = ((int64_t)(c[0] + ((l >> 2) & 1)) * m + (c[1] + ((l >> 1) & 1))) * m + (c[2] + (l & 1));
    for (int ch = 0; ch < channels; ++ch) acc[ch] = __dadd_rn(acc[ch], __dmul_rn(w, (double)vals[id * channels + ch]));
  }
  for (int ch = 0; ch < channels; ++ch) out[p * channels + ch] = acc[ch];
}

// the 27 coefficients of row (i, j, k) of L + alpha_a S, neighbour (dx, dy, dz) at (dx + 1) * 9 + (dy + 1) * 3 + dz + 1
__device__ __forceinline__ void row_coeffs(const Level& L, int32_t i, int32_t j, int32_t k, double alpha_a, double c[27]) {
  const int32_t n = L.n;
  const int32_t v[3] = {i, j, k};
  double cnt[3][3];   // cells shared with the neighbour along each axis, for d = -1, 0, +1
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    cnt[a][0] = v[a] > 0 ? 1.0 : 0.0;
    cnt[a][2] = v[a] < n ? 1.0 : 0.0;
    cnt[a][1] = cnt[a][0] + cnt[a][2];
  }
  const double kd[4] = {L.h / 3.0, 0.0, -L.h / 12.0, -L.h / 12.0};   // Q1 element stiffness by the number of differing axes
#pragma unroll
  for (int dx = 0; dx < 3; ++dx)
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dz = 0; dz < 3; ++dz) {
        const int nz = (dx != 1) + (dy != 1) + (dz != 1);
        c[dx * 9 + dy * 3 + dz] = cnt[0][dx] * cnt[1][dy] * cnt[2][dz] * kd[nz];
      }
#pragma unroll
  for (int o = 0; o < 8; ++o) {
    const int ox = (o >> 2) & 1, oy = (o >> 1) & 1, oz = o & 1;
    const int32_t cx = i - 1 + ox, cy = j - 1 + oy, cz = k - 1 + oz;
    if (cx < 0 || cy < 0 || cz < 0 || cx >= n || cy >= n || cz >= n) continue;
    const int32_t sl = __ldg(L.slot + ((int64_t)cx * n + cy) * n + cz);
    if (sl < 0) continue;
    const float* m = L.mat + (int64_t)sl * 64 + (7 - o) * 8;   // the node is corner (1 - ox, 1 - oy, 1 - oz) of the cell
#pragma unroll
    for (int l = 0; l < 8; ++l) {
      const int d = (ox + ((l >> 2) & 1)) * 9 + (oy + ((l >> 1) & 1)) * 3 + (oz + (l & 1));
      c[d] = fma(alpha_a, (double)__ldg(m + l), c[d]);
    }
  }
}

enum { OP_APPLY = 0, OP_RESIDUAL = 1, OP_JACOBI = 2, OP_L1 = 3 };

// OP_APPLY: y = A x.  OP_RESIDUAL: y = f - A x.  OP_JACOBI: y = x + omega (f - A x) / d.  OP_L1: y = sum |row|.
template <int OP>
__global__ void __launch_bounds__(kThreads)
    k_operator(Level L, double alpha_a, const float* __restrict__ x, const float* __restrict__ f, const float* __restrict__ d,
               float* __restrict__ y) {
  const int64_t id = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (id >= node_count(L.n)) return;
  int32_t i, j, k;
  node_ijk(id, L.n, i, j, k);
  double c[27];
  row_coeffs(L, i, j, k, alpha_a, c);
  double acc = 0.0;
  if constexpr (OP == OP_L1) {
#pragma unroll
    for (int t = 0; t < 27; ++t) acc += fabs(c[t]);
    y[id] = (float)acc;
    return;
  } else {
    const int64_t m = L.n + 1;
#pragma unroll
    for (int dx = 0; dx < 3; ++dx)
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dz = 0; dz < 3; ++dz) {
          const double ct = c[dx * 9 + dy * 3 + dz];
          if (ct != 0.0) acc = fma(ct, (double)__ldg(x + id + ((dx - 1) * m + (dy - 1)) * m + (dz - 1)), acc);
        }
    if constexpr (OP == OP_APPLY) y[id] = (float)acc;
    else if constexpr (OP == OP_RESIDUAL) y[id] = (float)((double)f[id] - acc);
    else y[id] = (float)((double)x[id] + kOmega * ((double)f[id] - acc) / (double)d[id]);
  }
}

// first sweep from x = 0: y = omega f / d
__global__ void __launch_bounds__(kThreads) k_jacobi0(int64_t n, const float* __restrict__ f, const float* __restrict__ d, float* __restrict__ y) {
  const int64_t id = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (id < n) y[id] = (float)(kOmega * (double)f[id] / (double)d[id]);
}

__device__ __forceinline__ double transfer_w(int d) { return d == 0 ? 1.0 : 0.5; }

// coarse f[I] = sum over fine nodes 2 I + d, d in {-1, 0, 1}^3, of prod w(d) r
__global__ void __launch_bounds__(kThreads) k_restrict(int32_t nc, const float* __restrict__ r, float* __restrict__ f) {
  const int64_t id = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (id >= node_count(nc)) return;
  int32_t I, J, K;
  node_ijk(id, nc, I, J, K);
  const int32_t nf = 2 * nc;
  const int64_t m = nf + 1;
  double acc = 0.0;
#pragma unroll
  for (int dx = -1; dx <= 1; ++dx)
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
      for (int dz = -1; dz <= 1; ++dz) {
        const int32_t a = 2 * I + dx, b = 2 * J + dy, c = 2 * K + dz;
        if (a < 0 || b < 0 || c < 0 || a > nf || b > nf || c > nf) continue;
        acc = fma(transfer_w(dx) * transfer_w(dy) * transfer_w(dz), (double)__ldg(r + ((int64_t)a * m + b) * m + c), acc);
      }
  f[id] = (float)acc;
}

// fine x[i] += sum over the coarse nodes of its cell of the trilinear weights times e
__global__ void __launch_bounds__(kThreads) k_prolong_add(int32_t nf, const float* __restrict__ e, float* __restrict__ x) {
  const int64_t id = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (id >= node_count(nf)) return;
  int32_t i, j, k;
  node_ijk(id, nf, i, j, k);
  const int64_t m = nf / 2 + 1;
  const int32_t v[3] = {i, j, k};
  int32_t lo[3], hi[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = v[a] >> 1;
    hi[a] = (v[a] + 1) >> 1;
  }
  double acc = 0.0;
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const int bx = (t >> 2) & 1, by = (t >> 1) & 1, bz = t & 1;
    // an even index has lo == hi: take it once with weight 1
    if ((bx && lo[0] == hi[0]) || (by && lo[1] == hi[1]) || (bz && lo[2] == hi[2])) continue;
    const double w = (lo[0] == hi[0] ? 1.0 : 0.5) * (lo[1] == hi[1] ? 1.0 : 0.5) * (lo[2] == hi[2] ? 1.0 : 0.5);
    const int64_t cid = ((int64_t)(bx ? hi[0] : lo[0]) * m + (by ? hi[1] : lo[1])) * m + (bz ? hi[2] : lo[2]);
    acc = fma(w, (double)__ldg(e + cid), acc);
  }
  x[id] = (float)((double)x[id] + acc);
}

// partial[b] = sum over i = b * kThreads + t (mod grid stride) of a[i] b[i] in double, fixed tree per block
template <typename T>
__global__ void __launch_bounds__(kThreads) k_dot(int64_t n, const T* __restrict__ a, const T* __restrict__ b, double* __restrict__ partial) {
  __shared__ double sh[kThreads];
  double acc = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)kDotBlocks * kThreads)
    acc += b ? (double)a[i] * (double)b[i] : (double)a[i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = sh[0];
}

__global__ void __launch_bounds__(kDotBlocks) k_dot_final(const double* __restrict__ partial, double* __restrict__ out) {
  __shared__ double sh[kDotBlocks];
  sh[threadIdx.x] = partial[threadIdx.x];
  __syncthreads();
  for (int s = kDotBlocks / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sh[0];
}

// x += alpha p; r -= alpha q
__global__ void __launch_bounds__(kThreads)
    k_cg_update(int64_t n, double alpha, const float* __restrict__ p, const float* __restrict__ q, float* __restrict__ x, float* __restrict__ r) {
  const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  x[i] = (float)fma(alpha, (double)p[i], (double)x[i]);
  r[i] = (float)fma(-alpha, (double)q[i], (double)r[i]);
}

// p = z + beta p
__global__ void __launch_bounds__(kThreads) k_cg_direction(int64_t n, double beta, const float* __restrict__ z, float* __restrict__ p) {
  const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i < n) p[i] = (float)fma(beta, (double)p[i], (double)z[i]);
}

// the dense 27 x 27 matrix of the coarsest level, then its Cholesky factor (one thread, double)
__global__ void k_coarse_factor(Level L, double alpha_a, double* __restrict__ A) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int m = L.n + 1;
  for (int r = 0; r < kCoarseNodes * kCoarseNodes; ++r) A[r] = 0.0;
  for (int id = 0; id < kCoarseNodes; ++id) {
    const int i = id / (m * m), j = (id / m) % m, k = id % m;
    double c[27];
    row_coeffs(L, i, j, k, alpha_a, c);
    for (int t = 0; t < 27; ++t) {
      const int a = i + t / 9 - 1, b = j + (t / 3) % 3 - 1, cc = k + t % 3 - 1;
      if (a < 0 || b < 0 || cc < 0 || a >= m || b >= m || cc >= m) continue;
      A[id * kCoarseNodes + (a * m + b) * m + cc] += c[t];
    }
  }
  for (int c = 0; c < kCoarseNodes; ++c) {
    double s = A[c * kCoarseNodes + c];
    for (int t = 0; t < c; ++t) s -= A[c * kCoarseNodes + t] * A[c * kCoarseNodes + t];
    const double dgl = sqrt(fmax(s, 1e-300));
    A[c * kCoarseNodes + c] = dgl;
    for (int r = c + 1; r < kCoarseNodes; ++r) {
      double v = A[r * kCoarseNodes + c];
      for (int t = 0; t < c; ++t) v -= A[r * kCoarseNodes + t] * A[c * kCoarseNodes + t];
      A[r * kCoarseNodes + c] = v / dgl;
    }
  }
}

__global__ void k_coarse_solve(const double* __restrict__ F, const float* __restrict__ f, float* __restrict__ x) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double y[kCoarseNodes];
  for (int r = 0; r < kCoarseNodes; ++r) {
    double v = f[r];
    for (int t = 0; t < r; ++t) v -= F[r * kCoarseNodes + t] * y[t];
    y[r] = v / F[r * kCoarseNodes + r];
  }
  for (int r = kCoarseNodes - 1; r >= 0; --r) {
    double v = y[r];
    for (int t = r + 1; t < kCoarseNodes; ++t) v -= F[t * kCoarseNodes + r] * y[t];
    y[r] = v / F[r * kCoarseNodes + r];
  }
  for (int r = 0; r < kCoarseNodes; ++r) x[r] = (float)y[r];
}

unsigned blocks(int64_t n) { return (unsigned)ceil_div(n, kThreads); }

int64_t nodes_of(int level) {
  const int64_t m = ((int64_t)1 << level) + 1;
  return m * m * m;
}

// workspace layout: per level 1..depth the vectors d, f, x, t (f and x of the finest level are the solver's r and z), then p and q of the
// finest level, then the dense coarse factor and the reduction scratch
struct Workspace {
  float* d[11];
  float* f[11];
  float* x[11];
  float* t[11];
  float* p;
  float* q;
  double* coarse;
  double* partial;
  double* scalar;
  size_t bytes;
};

Workspace carve(int depth, void* base) {
  Workspace w{};
  char* c = (char*)base;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    void* p = c ? c + off : nullptr;
    off += (bytes + 255) & ~(size_t)255;
    return p;
  };
  for (int l = kCoarsest; l <= depth; ++l) {
    const size_t nb = (size_t)nodes_of(l) * sizeof(float);
    w.d[l] = (float*)take(nb);
    w.f[l] = (float*)take(nb);
    w.x[l] = (float*)take(nb);
    w.t[l] = (float*)take(nb);
  }
  const size_t nb = (size_t)nodes_of(depth) * sizeof(float);
  w.p = (float*)take(nb);
  w.q = (float*)take(nb);
  w.coarse = (double*)take(sizeof(double) * kCoarseNodes * kCoarseNodes);
  w.partial = (double*)take(sizeof(double) * kDotBlocks);
  w.scalar = (double*)take(sizeof(double) * 4);
  w.bytes = off;
  return w;
}

template <typename T>
int dot(int64_t n, const T* a, const T* b, const Workspace& w, cudaStream_t st, double* host) {
  k_dot<T><<<kDotBlocks, kThreads, 0, st>>>(n, a, b, w.partial);
  SDFB_LAUNCHED("k_dot");
  k_dot_final<<<1, kDotBlocks, 0, st>>>(w.partial, w.scalar);
  SDFB_LAUNCHED("k_dot_final");
  SDFB_CUDA(cudaMemcpyAsync(host, w.scalar, sizeof(double), cudaMemcpyDeviceToHost, st));
  SDFB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

template <int OP>
int op(const Level& L, double alpha_a, const float* x, const float* f, const float* d, float* y, cudaStream_t st) {
  k_operator<OP><<<blocks(node_count(L.n)), kThreads, 0, st>>>(L, alpha_a, x, f, d, y);
  SDFB_LAUNCHED("k_operator");
  return 0;
}

// x[l] = V-cycle applied to f[l]
int vcycle(const Level* lv, int l, double alpha_a, const Workspace& w, cudaStream_t st) {
  const Level& L = lv[l];
  if (l == kCoarsest) {
    k_coarse_solve<<<1, 32, 0, st>>>(w.coarse, w.f[l], w.x[l]);
    SDFB_LAUNCHED("k_coarse_solve");
    return 0;
  }
  const int64_t nn = node_count(L.n);
  k_jacobi0<<<blocks(nn), kThreads, 0, st>>>(nn, w.f[l], w.d[l], w.t[l]);
  SDFB_LAUNCHED("k_jacobi0");
  if (int r = op<OP_JACOBI>(L, alpha_a, w.t[l], w.f[l], w.d[l], w.x[l], st)) return r;
  if (int r = op<OP_RESIDUAL>(L, alpha_a, w.x[l], w.f[l], nullptr, w.t[l], st)) return r;
  k_restrict<<<blocks(node_count(lv[l - 1].n)), kThreads, 0, st>>>(lv[l - 1].n, w.t[l], w.f[l - 1]);
  SDFB_LAUNCHED("k_restrict");
  if (int r = vcycle(lv, l - 1, alpha_a, w, st)) return r;
  k_prolong_add<<<blocks(nn), kThreads, 0, st>>>(L.n, w.x[l - 1], w.x[l]);
  SDFB_LAUNCHED("k_prolong_add");
  for (int s = 0; s < kSweeps / 2; ++s) {
    if (int r = op<OP_JACOBI>(L, alpha_a, w.x[l], w.f[l], w.d[l], w.t[l], st)) return r;
    if (int r = op<OP_JACOBI>(L, alpha_a, w.t[l], w.f[l], w.d[l], w.x[l], st)) return r;
  }
  return 0;
}

bool grid_ok(const double* origin, double h) {
  return origin && isfinite(origin[0]) && isfinite(origin[1]) && isfinite(origin[2]) && isfinite(h) && h > 0.0;
}

}  // namespace
}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_poisson_cells(const float* points, const float* normals, const float* colors, int64_t n_cells, const int64_t* cell_key,
                                     const int64_t* cell_start, int32_t level, const double* origin, double h, float* mat, float* rhs,
                                     float* splat, void* stream) {
  SDFB_REQUIRE(level >= 0 && level <= 10, "level must lie in [0, 10]");
  SDFB_REQUIRE(n_cells >= 0 && n_cells <= ((int64_t)1 << (3 * level)), "n_cells must lie in [0, 8^level]");
  SDFB_REQUIRE(grid_ok(origin, h), "origin and h must be finite, h > 0");
  SDFB_REQUIRE((normals != nullptr) != (colors != nullptr), "give normals (screening blocks) or colors (splat), not both");
  SDFB_REQUIRE(normals ? (mat && rhs) : splat != nullptr, "NULL output");
  if (n_cells == 0) return 0;
  SDFB_REQUIRE(points && cell_key && cell_start, "NULL pointer");
  Grid g{1 << level, {origin[0], origin[1], origin[2]}, h};
  const cudaStream_t st = (cudaStream_t)stream;
  if (normals) k_cells<MODE_SCREEN><<<blocks(n_cells), kThreads, 0, st>>>(points, normals, n_cells, cell_key, cell_start, g, mat, rhs, nullptr);
  else k_cells<MODE_SPLAT><<<blocks(n_cells), kThreads, 0, st>>>(points, colors, n_cells, cell_key, cell_start, g, nullptr, nullptr, splat);
  SDFB_LAUNCHED("k_cells");
  return 0;
}

extern "C" int sdfb200_poisson_coarsen(int32_t level, const int32_t* fine_slot, const float* fine_mat, int64_t n_cells, const int64_t* cell_key,
                                       float* mat, void* stream) {
  SDFB_REQUIRE(level >= 0 && level <= 9, "level must lie in [0, 9]");
  SDFB_REQUIRE(n_cells >= 0 && n_cells <= ((int64_t)1 << (3 * level)), "n_cells must lie in [0, 8^level]");
  if (n_cells == 0) return 0;
  SDFB_REQUIRE(fine_slot && fine_mat && cell_key && mat, "NULL pointer");
  k_coarsen<<<blocks(n_cells * 8), kThreads, 0, (cudaStream_t)stream>>>(2 << level, fine_slot, fine_mat, n_cells, cell_key, 1 << level, mat);
  SDFB_LAUNCHED("k_coarsen");
  return 0;
}

extern "C" int sdfb200_poisson_gather(int32_t level, const int32_t* cell_slot, const float* cell_vals, int32_t cell_stride, int32_t corner_stride,
                                      int32_t channels, float* node_vals, void* stream) {
  SDFB_REQUIRE(level >= 0 && level <= 10, "level must lie in [0, 10]");
  SDFB_REQUIRE(channels >= 1 && channels <= 4, "channels must lie in [1, 4]");
  SDFB_REQUIRE(corner_stride >= channels && cell_stride >= 8 * corner_stride - corner_stride + channels, "strides too small");
  SDFB_REQUIRE(cell_slot && cell_vals && node_vals, "NULL pointer");
  k_gather<<<blocks(nodes_of(level)), kThreads, 0, (cudaStream_t)stream>>>(1 << level, cell_slot, cell_vals, cell_stride, corner_stride,
                                                                         channels, node_vals);
  SDFB_LAUNCHED("k_gather");
  return 0;
}

extern "C" int sdfb200_poisson_sample(const float* points, int64_t n_points, int32_t level, const double* origin, double h,
                                      const float* node_vals, int32_t channels, double* out, void* stream) {
  SDFB_REQUIRE(level >= 0 && level <= 10, "level must lie in [0, 10]");
  SDFB_REQUIRE(channels >= 1 && channels <= 4, "channels must lie in [1, 4]");
  SDFB_REQUIRE(n_points >= 0, "n_points must be >= 0");
  SDFB_REQUIRE(grid_ok(origin, h), "origin and h must be finite, h > 0");
  if (n_points == 0) return 0;
  SDFB_REQUIRE(points && node_vals && out, "NULL pointer");
  Grid g{1 << level, {origin[0], origin[1], origin[2]}, h};
  k_sample<<<blocks(n_points), kThreads, 0, (cudaStream_t)stream>>>(points, n_points, g, node_vals, channels, out);
  SDFB_LAUNCHED("k_sample");
  return 0;
}

extern "C" int sdfb200_poisson_apply(int32_t level, double h, const int32_t* cell_slot, const float* mat, double alpha_a, const float* x,
                                     float* y, void* stream) {
  SDFB_REQUIRE(level >= 0 && level <= 10, "level must lie in [0, 10]");
  SDFB_REQUIRE(isfinite(h) && h > 0.0 && isfinite(alpha_a) && alpha_a >= 0.0, "h must be finite and > 0, alpha_a finite and >= 0");
  SDFB_REQUIRE(cell_slot && mat && x && y, "NULL pointer");
  Level L{1 << level, h, cell_slot, mat};
  return op<OP_APPLY>(L, alpha_a, x, nullptr, nullptr, y, (cudaStream_t)stream);
}

extern "C" size_t sdfb200_poisson_workspace_bytes(int32_t depth) {
  if (depth < 1 || depth > 10) return 0;
  return carve(depth, nullptr).bytes;
}

extern "C" int sdfb200_poisson_solve(int32_t depth, double h, const int32_t* const* cell_slot, const float* const* mat, double alpha_a,
                                     const float* rhs, float* x, int32_t max_cycles, double tol, void* workspace, size_t workspace_bytes,
                                     int32_t* cycles, double* rel_residual, void* stream) {
  SDFB_REQUIRE(depth >= 1 && depth <= 10, "depth must lie in [1, 10]");
  SDFB_REQUIRE(isfinite(h) && h > 0.0 && isfinite(alpha_a) && alpha_a > 0.0, "h and alpha_a must be finite and > 0");
  SDFB_REQUIRE(max_cycles >= 1 && max_cycles <= 1000, "max_cycles must lie in [1, 1000]");
  SDFB_REQUIRE(isfinite(tol) && tol > 0.0, "tol must be finite and > 0");
  SDFB_REQUIRE(cell_slot && mat && rhs && x && workspace && cycles && rel_residual, "NULL pointer");
  for (int l = kCoarsest; l <= depth; ++l) SDFB_REQUIRE(cell_slot[l] && mat[l], "NULL level pointer");
  const Workspace w = carve(depth, workspace);
  SDFB_REQUIRE(workspace_bytes >= w.bytes, "workspace smaller than sdfb200_poisson_workspace_bytes(depth)");
  const cudaStream_t st = (cudaStream_t)stream;
  Level lv[11];
  for (int l = kCoarsest; l <= depth; ++l) lv[l] = Level{1 << l, ldexp(h, depth - l), cell_slot[l], mat[l]};
  for (int l = kCoarsest + 1; l <= depth; ++l)
    if (int r = op<OP_L1>(lv[l], alpha_a, nullptr, nullptr, nullptr, w.d[l], st)) return r;
  k_coarse_factor<<<1, 32, 0, st>>>(lv[kCoarsest], alpha_a, w.coarse);
  SDFB_LAUNCHED("k_coarse_factor");

  const int64_t n = node_count(lv[depth].n);
  float *r = w.f[depth], *z = w.x[depth], *t = w.t[depth];
  SDFB_CUDA(cudaMemsetAsync(x, 0, n * sizeof(float), st));
  SDFB_CUDA(cudaMemcpyAsync(r, rhs, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  double bb, rz, pq, rr, tt;
  if (int e = dot<float>(n, rhs, rhs, w, st, &bb)) return e;
  const double bn = sqrt(bb);
  *cycles = 0;
  *rel_residual = 0.0;
  if (bn == 0.0) return 0;
  bool restart = true;
  for (int it = 1; it <= max_cycles; ++it) {
    if (int e = vcycle(lv, depth, alpha_a, w, st)) return e;
    double rz_new;
    if (int e = dot<float>(n, r, z, w, st, &rz_new)) return e;
    if (restart) {
      SDFB_CUDA(cudaMemcpyAsync(w.p, z, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
      restart = false;
    } else {
      k_cg_direction<<<blocks(n), kThreads, 0, st>>>(n, rz_new / rz, z, w.p);
      SDFB_LAUNCHED("k_cg_direction");
    }
    rz = rz_new;
    if (int e = op<OP_APPLY>(lv[depth], alpha_a, w.p, nullptr, nullptr, w.q, st)) return e;
    if (int e = dot<float>(n, w.p, w.q, w, st, &pq)) return e;
    k_cg_update<<<blocks(n), kThreads, 0, st>>>(n, rz / pq, w.p, w.q, x, r);
    SDFB_LAUNCHED("k_cg_update");
    *cycles = it;
    if (int e = dot<float>(n, r, r, w, st, &rr)) return e;
    if (sqrt(rr) > tol * bn) continue;
    // the recurrence says converged: check the true residual, and restart from it when it does not agree
    if (int e = op<OP_RESIDUAL>(lv[depth], alpha_a, x, rhs, nullptr, t, st)) return e;
    if (int e = dot<float>(n, t, t, w, st, &tt)) return e;
    if (sqrt(tt) <= tol * bn) break;
    SDFB_CUDA(cudaMemcpyAsync(r, t, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    restart = true;
  }
  if (int e = op<OP_RESIDUAL>(lv[depth], alpha_a, x, rhs, nullptr, t, st)) return e;
  if (int e = dot<float>(n, t, t, w, st, &tt)) return e;
  *rel_residual = sqrt(tt) / bn;
  return 0;
}

extern "C" int sdfb200_poisson_sum(const double* values, int64_t n, double* partial, double* out, void* stream) {
  SDFB_REQUIRE(n >= 0, "n must be >= 0");
  SDFB_REQUIRE(values && partial && out, "NULL pointer");
  const cudaStream_t st = (cudaStream_t)stream;
  k_dot<double><<<kDotBlocks, kThreads, 0, st>>>(n, values, nullptr, partial);
  SDFB_LAUNCHED("k_dot");
  k_dot_final<<<1, kDotBlocks, 0, st>>>(partial, out);
  SDFB_LAUNCHED("k_dot_final");
  return 0;
}
