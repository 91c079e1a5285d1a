// Stand-alone grid encode / backward kernels behind sdfb200_grid_encode{,_backward} (the tcnn.Encoding operator
// boundary, nerfstudio/fields/sdf_field.py:230-241,386).  HBM/L2-gather bound: one thread per (point, level) so that
// a warp covers 2 points x 16 levels and its F-wide outputs are written to consecutive addresses.
#include "field.h"
#include "grid.cuh"

namespace sdfb200 {

template <typename T, int F, bool GRAD>
__global__ void __launch_bounds__(256) k_grid_encode(const __grid_constant__ sdfb200_grid_t g, const void* __restrict__ table,
                                                     const float* __restrict__ x01, int64_t n, float* __restrict__ out,
                                                     int64_t out_ld, float* __restrict__ dout_dx) {
  const int L = g.n_levels;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * L) return;
  const int64_t p = idx / L;
  const int l = (int)(idx - p * L);
  float o[F];
  float d[F][3];
  if (l < g.active_levels) {
    const float x = __ldg(x01 + p * 3), y = __ldg(x01 + p * 3 + 1), z = __ldg(x01 + p * 3 + 2);
    encode_level<T, F>(g, table, l, x, y, z, o, d);
  } else {
#pragma unroll
    for (int f = 0; f < F; ++f) {
      o[f] = 0.f;
      d[f][0] = d[f][1] = d[f][2] = 0.f;
    }
  }
  float* op = out + p * out_ld + l * F;
#pragma unroll
  for (int f = 0; f < F; ++f) op[f] = o[f];
  if (GRAD) {
    float* dp = dout_dx + (p * L * F + l * F) * 3;
#pragma unroll
    for (int f = 0; f < F; ++f) {
      dp[f * 3 + 0] = d[f][0]; dp[f * 3 + 1] = d[f][1]; dp[f * 3 + 2] = d[f][2];
    }
  }
}

// vector atomics (sm_90+: red.global.add.v2.f32 / .v4.f32): one L2 atomic per 8 / 16 bytes of a table row instead of one per float
template <int F>
__device__ __forceinline__ void atomic_add_row(float* dst, const float (&v)[F]) {
  if constexpr (F % 4 == 0) {
#pragma unroll
    for (int f = 0; f < F; f += 4) atomicAdd(reinterpret_cast<float4*>(dst + f), make_float4(v[f], v[f + 1], v[f + 2], v[f + 3]));
  } else if constexpr (F == 2) {
    atomicAdd(reinterpret_cast<float2*>(dst), make_float2(v[0], v[1]));
  } else {
#pragma unroll
    for (int f = 0; f < F; ++f) atomicAdd(dst + f, v[f]);
  }
}

// backward: scatter dout into the table gradient, optional dx01.
template <typename T, int F>
__global__ void __launch_bounds__(256) k_grid_encode_bwd(const __grid_constant__ sdfb200_grid_t g, const void* __restrict__ table,
                                                         const float* __restrict__ x01, const float* __restrict__ dout, int64_t n,
                                                         float* __restrict__ dtable, float* __restrict__ dx01) {
  const int L = g.n_levels;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * L) return;
  const int64_t p = idx / L;
  const int l = (int)(idx - p * L);
  if (l >= g.active_levels) return;
  const float x = __ldg(x01 + p * 3), y = __ldg(x01 + p * 3 + 1), z = __ldg(x01 + p * 3 + 2);
  float go[F];
#pragma unroll
  for (int f = 0; f < F; ++f) go[f] = __ldg(dout + p * L * F + l * F + f);
  LevelCtx c;
  level_prepare(g, l, x, y, z, c);
  // dtable == NULL: input gradient only (autograd.grad(sdf, x) of the eikonal / normal path), no scatter
  if (dtable != nullptr) {
    float w[8];
    corner_weights(c, w);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float wv[F];
#pragma unroll
      for (int f = 0; f < F; ++f) wv[f] = w[k] * go[f];
      atomic_add_row<F>(dtable + (c.base + c.idx[k]) * F, wv);
    }
  }
  if (dx01 != nullptr) {
    float v[8][F], o[F], d[F][3];
    level_fetch<T, F>(table, c, v);
    level_finish<F>(g, c, v, o, d);
    float ax = 0.f, ay = 0.f, az = 0.f;
#pragma unroll
    for (int f = 0; f < F; ++f) {
      ax = fmaf(go[f], d[f][0], ax); ay = fmaf(go[f], d[f][1], ay); az = fmaf(go[f], d[f][2], az);
    }
    atomicAdd(dx01 + p * 3 + 0, ax); atomicAdd(dx01 + p * 3 + 1, ay); atomicAdd(dx01 + p * 3 + 2, az);
  }
}

// -----------------------------------------------------------------------------------------------------------------
// Grouped variants for numerical-gradient fields (sdf_field.py:424-452): the batch holds `group` points per sample -- the sample and
// its +-delta taps, point gi of sample n at row gi * n_samples + n -- that almost always fall into the SAME cell of a level (delta is the
// finest level's cell size, the active levels are coarser).  One thread walks the taps of a (sample, level): while the 8 table rows
// stay the same it gathers them once (forward) / accumulates the 8 row gradients in registers and issues ONE set of atomics
// (backward) instead of `group` of them.  Arithmetic per point is the ungrouped kernels'.
// -----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool same_rows(const LevelCtx& a, const LevelCtx& b) {
  bool same = true;
#pragma unroll
  for (int k = 0; k < 8; ++k) same = same && (a.idx[k] == b.idx[k]);
  return same;
}

template <typename T, int F>
__global__ void __launch_bounds__(256) k_grid_encode_grouped(const __grid_constant__ sdfb200_grid_t g, const void* __restrict__ table,
                                                             const float* __restrict__ x01, int64_t n_samples, int group, float* __restrict__ out,
                                                             int64_t out_ld) {
  const int L = g.n_levels;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_samples * L) return;
  const int64_t n = idx / L;
  const int l = (int)(idx - n * L);
  LevelCtx cur;
  float tv[8][F];
  bool have = false;
  for (int gi = 0; gi < group; ++gi) {
    const int64_t p = (int64_t)gi * n_samples + n;
    float o[F];
    if (l < g.active_levels) {
      LevelCtx c;
      level_prepare(g, l, __ldg(x01 + p * 3), __ldg(x01 + p * 3 + 1), __ldg(x01 + p * 3 + 2), c);
      if (!have || !same_rows(c, cur)) {
        level_fetch<T, F>(table, c, tv);
        have = true;
      }
      cur = c;
      float dj[F][3];
      level_finish<F>(g, c, tv, o, dj);
    } else {
#pragma unroll
      for (int f = 0; f < F; ++f) o[f] = 0.f;
    }
    float* op = out + p * out_ld + l * F;
#pragma unroll
    for (int f = 0; f < F; ++f) op[f] = o[f];
  }
}

template <int F>
__global__ void __launch_bounds__(256) k_grid_encode_bwd_grouped(const __grid_constant__ sdfb200_grid_t g, const float* __restrict__ x01,
                                                                 const float* __restrict__ dout, int64_t n_samples, int group,
                                                                 float* __restrict__ dtable) {
  const int L = g.n_levels;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_samples * L) return;
  const int64_t n = idx / L;
  const int l = (int)(idx - n * L);
  if (l >= g.active_levels) return;
  LevelCtx cur;
  float acc[8][F];
  bool have = false;
  auto flush = [&]() {
#pragma unroll
    for (int k = 0; k < 8; ++k) atomic_add_row<F>(dtable + (cur.base + cur.idx[k]) * F, acc[k]);
  };
  for (int gi = 0; gi < group; ++gi) {
    const int64_t p = (int64_t)gi * n_samples + n;
    LevelCtx c;
    level_prepare(g, l, __ldg(x01 + p * 3), __ldg(x01 + p * 3 + 1), __ldg(x01 + p * 3 + 2), c);
    if (have && !same_rows(c, cur)) {
      flush();
      have = false;
    }
    if (!have) {
      cur = c;
#pragma unroll
      for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int f = 0; f < F; ++f) acc[k][f] = 0.f;
      have = true;
    }
    float w[8], go[F];
    corner_weights(c, w);
#pragma unroll
    for (int f = 0; f < F; ++f) go[f] = __ldg(dout + p * L * F + l * F + f);
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
      for (int f = 0; f < F; ++f) acc[k][f] = fmaf(w[k], go[f], acc[k][f]);
  }
  if (have) flush();
}

// second-order backward (the backward of k_grid_encode_bwd's dx01 output), needed by the eikonal loss
// (models/base_surface_model.py:358-362 differentiates |grad sdf| w.r.t. the parameters):
//   first backward:  dx[c] = sum_lf dout[lf] * J[lf][c](x, table)
//   given g_dx = dLoss/d(dx):  g_dout[lf] = sum_c g_dx[c] J[lf][c];   g_table[corner][f] += dout[lf] * sum_c g_dx[c] dW_corner/dx_c;
//                              g_x[c'] += sum_lf dout[lf] sum_c g_dx[c] d2 feat_lf / dx_c dx_c'
template <typename T, int F>
__global__ void __launch_bounds__(256) k_grid_encode_bwd2(const __grid_constant__ sdfb200_grid_t g, const void* __restrict__ table,
                                                          const float* __restrict__ x01, const float* __restrict__ dout,
                                                          const float* __restrict__ g_dx, int64_t n, float* __restrict__ g_dout,
                                                          float* __restrict__ g_table, float* __restrict__ g_x) {
  const int L = g.n_levels;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * L) return;
  const int64_t p = idx / L;
  const int l = (int)(idx - p * L);
  float* gdo = g_dout ? g_dout + p * L * F + l * F : nullptr;
  if (l >= g.active_levels) {
    if (gdo)
#pragma unroll
      for (int f = 0; f < F; ++f) gdo[f] = 0.f;
    return;
  }
  const float gx[3] = {__ldg(g_dx + p * 3), __ldg(g_dx + p * 3 + 1), __ldg(g_dx + p * 3 + 2)};
  float go[F];
#pragma unroll
  for (int f = 0; f < F; ++f) go[f] = __ldg(dout + p * L * F + l * F + f);
  LevelCtx q;
  level_prepare(g, l, __ldg(x01 + p * 3), __ldg(x01 + p * 3 + 1), __ldg(x01 + p * 3 + 2), q);
  const float dw[3] = {q.dw[0] * q.s, q.dw[1] * q.s, q.dw[2] * q.s};   // d w / d x01
  float acc_do[F];
#pragma unroll
  for (int f = 0; f < F; ++f) acc_do[f] = 0.f;
  float acc_x[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int b[3] = {c & 1, (c >> 1) & 1, (c >> 2) & 1};
    float A[3], sg[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      A[d] = b[d] ? q.w[d] : 1.f - q.w[d];
      sg[d] = b[d] ? 1.f : -1.f;
    }
    const uint64_t row = q.base + q.idx[c];
    float v[F];
    load_row<T, F>(table, row, v);
    // first derivatives of the corner weight
    const float d0 = sg[0] * dw[0], d1 = sg[1] * dw[1], d2 = sg[2] * dw[2];
    const float gW = gx[0] * d0 * A[1] * A[2] + gx[1] * A[0] * d1 * A[2] + gx[2] * A[0] * A[1] * d2;
    float dot = 0.f;
#pragma unroll
    for (int f = 0; f < F; ++f) {
      acc_do[f] = fmaf(gW, v[f], acc_do[f]);
      dot = fmaf(go[f], v[f], dot);
    }
    if (g_table) {
      float wv[F];
#pragma unroll
      for (int f = 0; f < F; ++f) wv[f] = gW * go[f];
      atomic_add_row<F>(g_table + row * F, wv);
    }
    if (g_x) {
      const float h00 = sg[0] * q.d2w[0] * A[1] * A[2], h11 = A[0] * sg[1] * q.d2w[1] * A[2], h22 = A[0] * A[1] * sg[2] * q.d2w[2];
      const float h01 = d0 * d1 * A[2], h02 = d0 * A[1] * d2, h12 = A[0] * d1 * d2;
      acc_x[0] = fmaf(dot, gx[0] * h00 + gx[1] * h01 + gx[2] * h02, acc_x[0]);
      acc_x[1] = fmaf(dot, gx[0] * h01 + gx[1] * h11 + gx[2] * h12, acc_x[1]);
      acc_x[2] = fmaf(dot, gx[0] * h02 + gx[1] * h12 + gx[2] * h22, acc_x[2]);
    }
  }
  if (gdo)
#pragma unroll
    for (int f = 0; f < F; ++f) gdo[f] = acc_do[f];
  if (g_x) {
    atomicAdd(g_x + p * 3 + 0, acc_x[0]); atomicAdd(g_x + p * 3 + 1, acc_x[1]); atomicAdd(g_x + p * 3 + 2, acc_x[2]);
  }
}

int validate_grid(const sdfb200_grid_t* g) {
  SDFB_REQUIRE(g != nullptr, "grid descriptor is NULL");
  SDFB_REQUIRE(g->n_levels >= 1 && g->n_levels <= SDFB200_MAX_LEVELS, "grid.n_levels out of range");
  SDFB_REQUIRE(g->n_features == 1 || g->n_features == 2 || g->n_features == 4 || g->n_features == 8, "grid.n_features must be 1,2,4,8");
  SDFB_REQUIRE(g->layout == SDFB200_GRID_TORCH || g->layout == SDFB200_GRID_TCNN, "grid.layout");
  SDFB_REQUIRE(g->table_dtype == SDFB200_DT_F32 || g->table_dtype == SDFB200_DT_F16, "grid.table_dtype");
  SDFB_REQUIRE(g->log2_hashmap_size >= 1 && g->log2_hashmap_size <= 31, "grid.log2_hashmap_size");
  SDFB_REQUIRE(g->active_levels >= 0 && g->active_levels <= g->n_levels, "grid.active_levels");
  return 0;
}

// load_row reads a row with one vector load per 16 bytes (F * sizeof(T), capped at 16); atomic_add_row adds 16 (F % 4 == 0), 8 (F == 2)
// or 4 bytes at once.  A pointer those instructions cannot take is refused before anything launches.  NULL pointers pass.
int validate_grid_pointers(const sdfb200_grid_t* g, const void* table, const float* grad) {
  const long long row = (long long)g->n_features * (g->table_dtype == SDFB200_DT_F16 ? 2 : 4);
  const long long load = row < 16 ? row : 16;
  const long long add = g->n_features % 4 == 0 ? 16 : g->n_features == 2 ? 8 : 4;
  if ((uintptr_t)table % load) return fail(SDFB200_EINVAL, "grid table%s must be aligned to %lld bytes (its row loads)", "", load);
  if ((uintptr_t)grad % add) return fail(SDFB200_EINVAL, "grid gradient%s must be aligned to %lld bytes (its vector atomics)", "", add);
  return 0;
}

template <typename T, int F>
static int launch_encode(const sdfb200_grid_t& g, const void* table, const float* x01, int64_t n, float* out, int64_t out_ld,
                         float* dout_dx, cudaStream_t st) {
  const int64_t total = n * g.n_levels;
  const unsigned blocks = (unsigned)ceil_div(total, 256);
  if (dout_dx)
    k_grid_encode<T, F, true><<<blocks, 256, 0, st>>>(g, table, x01, n, out, out_ld, dout_dx);
  else
    k_grid_encode<T, F, false><<<blocks, 256, 0, st>>>(g, table, x01, n, out, out_ld, nullptr);
  SDFB_LAUNCHED("k_grid_encode");
  return 0;
}

template <typename T, int F>
static int launch_encode_bwd(const sdfb200_grid_t& g, const void* table, const float* x01, const float* dout, int64_t n,
                             float* dtable, float* dx01, cudaStream_t st) {
  const int64_t total = n * g.n_levels;
  k_grid_encode_bwd<T, F><<<(unsigned)ceil_div(total, 256), 256, 0, st>>>(g, table, x01, dout, n, dtable, dx01);
  SDFB_LAUNCHED("k_grid_encode_bwd");
  return 0;
}

template <typename T, int F>
static int launch_encode_bwd2(const sdfb200_grid_t& g, const void* table, const float* x01, const float* dout, const float* g_dx, int64_t n,
                              float* g_dout, float* g_table, float* g_x, cudaStream_t st) {
  const int64_t total = n * g.n_levels;
  k_grid_encode_bwd2<T, F><<<(unsigned)ceil_div(total, 256), 256, 0, st>>>(g, table, x01, dout, g_dx, n, g_dout, g_table, g_x);
  SDFB_LAUNCHED("k_grid_encode_bwd2");
  return 0;
}

template <typename T, int F>
static int launch_encode_grouped(const sdfb200_grid_t& g, const void* table, const float* x01, int64_t n_samples, int group, float* out, int64_t out_ld,
                                 cudaStream_t st) {
  const int64_t total = n_samples * g.n_levels;
  k_grid_encode_grouped<T, F><<<(unsigned)ceil_div(total, 256), 256, 0, st>>>(g, table, x01, n_samples, group, out, out_ld);
  SDFB_LAUNCHED("k_grid_encode_grouped");
  return 0;
}

template <typename T, int F>
static int launch_encode_bwd_grouped(const sdfb200_grid_t& g, const float* x01, const float* dout, int64_t n_samples, int group, float* dtable,
                                     cudaStream_t st) {
  const int64_t total = n_samples * g.n_levels;
  k_grid_encode_bwd_grouped<F><<<(unsigned)ceil_div(total, 256), 256, 0, st>>>(g, x01, dout, n_samples, group, dtable);
  SDFB_LAUNCHED("k_grid_encode_bwd_grouped");
  return 0;
}

#define SDFB_DISPATCH_GRID(g, FN, ...)                                                      \
  do {                                                                                      \
    const bool h__ = (g).table_dtype == SDFB200_DT_F16;                                     \
    switch ((g).n_features) {                                                               \
      case 1: return h__ ? FN<__half, 1>(__VA_ARGS__) : FN<float, 1>(__VA_ARGS__);          \
      case 2: return h__ ? FN<__half, 2>(__VA_ARGS__) : FN<float, 2>(__VA_ARGS__);          \
      case 4: return h__ ? FN<__half, 4>(__VA_ARGS__) : FN<float, 4>(__VA_ARGS__);          \
      default: return h__ ? FN<__half, 8>(__VA_ARGS__) : FN<float, 8>(__VA_ARGS__);         \
    }                                                                                       \
  } while (0)

int grid_encode(const sdfb200_grid_t& g, const void* table, const float* x01, int64_t n, float* out, int64_t out_ld,
                float* dout_dx, cudaStream_t st) {
  if (n == 0) return 0;
  SDFB_DISPATCH_GRID(g, launch_encode, g, table, x01, n, out, out_ld, dout_dx, st);
}

}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_grid_encode(const sdfb200_grid_t* grid, const void* table, const float* x01, int64_t n, float* out,
                                   int64_t out_ld, float* dout_dx, void* stream) {
  int r = validate_grid(grid);
  if (r) return r;
  SDFB_REQUIRE(n >= 0, "n < 0");
  if (n == 0) return 0;
  SDFB_REQUIRE(table && x01 && out, "NULL pointer");
  SDFB_REQUIRE(out_ld >= (int64_t)grid->n_levels * grid->n_features, "out_ld too small");
  r = validate_grid_pointers(grid, table, nullptr);
  if (r) return r;
  return grid_encode(*grid, table, x01, n, out, out_ld, dout_dx, (cudaStream_t)stream);
}

extern "C" int sdfb200_grid_encode_backward(const sdfb200_grid_t* grid, const void* table, const float* x01, const float* dout,
                                            int64_t n, float* dtable, float* dx01, void* stream) {
  int r = validate_grid(grid);
  if (r) return r;
  SDFB_REQUIRE(n >= 0, "n < 0");
  if (n == 0) return 0;
  SDFB_REQUIRE(table && x01 && dout && (dtable || dx01), "NULL pointer");
  r = validate_grid_pointers(grid, table, dtable);
  if (r) return r;
  SDFB_DISPATCH_GRID(*grid, launch_encode_bwd, *grid, table, x01, dout, n, dtable, dx01, (cudaStream_t)stream);
}

extern "C" int sdfb200_grid_encode_backward_backward(const sdfb200_grid_t* grid, const void* table, const float* x01, const float* dout,
                                                     const float* g_dx01, int64_t n, float* g_dout, float* g_table, float* g_x01, void* stream) {
  int r = validate_grid(grid);
  if (r) return r;
  SDFB_REQUIRE(n >= 0, "n < 0");
  if (n == 0) return 0;
  SDFB_REQUIRE(table && x01 && dout && g_dx01, "NULL pointer");
  r = validate_grid_pointers(grid, table, g_table);
  if (r) return r;
  SDFB_DISPATCH_GRID(*grid, launch_encode_bwd2, *grid, table, x01, dout, g_dx01, n, g_dout, g_table, g_x01, (cudaStream_t)stream);
}

extern "C" int sdfb200_grid_encode_grouped(const sdfb200_grid_t* grid, const void* table, const float* x01, int64_t n, int32_t group, float* out,
                                           int64_t out_ld, void* stream) {
  int r = validate_grid(grid);
  if (r) return r;
  SDFB_REQUIRE(n >= 0 && group >= 1 && n % group == 0, "n must be a non-negative multiple of group");
  if (n == 0) return 0;
  SDFB_REQUIRE(table && x01 && out, "NULL pointer");
  SDFB_REQUIRE(out_ld >= (int64_t)grid->n_levels * grid->n_features, "out_ld too small");
  r = validate_grid_pointers(grid, table, nullptr);
  if (r) return r;
  SDFB_DISPATCH_GRID(*grid, launch_encode_grouped, *grid, table, x01, n / group, group, out, out_ld, (cudaStream_t)stream);
}

extern "C" int sdfb200_grid_encode_backward_grouped(const sdfb200_grid_t* grid, const float* x01, const float* dout, int64_t n, int32_t group,
                                                    float* dtable, void* stream) {
  int r = validate_grid(grid);
  if (r) return r;
  SDFB_REQUIRE(n >= 0 && group >= 1 && n % group == 0, "n must be a non-negative multiple of group");
  if (n == 0) return 0;
  SDFB_REQUIRE(x01 && dout && dtable, "NULL pointer");
  r = validate_grid_pointers(grid, nullptr, dtable);
  if (r) return r;
  SDFB_DISPATCH_GRID(*grid, launch_encode_bwd_grouped, *grid, x01, dout, n / group, group, dtable, (cudaStream_t)stream);
}
