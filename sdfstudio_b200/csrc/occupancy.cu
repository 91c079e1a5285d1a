// Occupancy grid of the neus-acc sampler (NeuSAccSampler, model_components/ray_samplers.py:1315-1503):
//   k_occupancy_prune : update_binary_grid's alpha test on the occupied voxel centres (:1384-1433); clears the voxels that fail
//   k_occupancy_march : nerfacc 0.3.5 ray_marching for the AABB contraction with cone_angle = 0 (called at :1473-1483), as a count
//                       pass and a write pass at the caller's exclusive-cumsum offsets
// Every float operation is written out non-contracted (__fadd_rn / __fmul_rn / __fdiv_rn / __frcp_rn, fminf / fmaxf for the NaNs of
// 0 * inf on axis-aligned directions) so that a numpy float32 restatement of the loop reproduces the march bit for bit.
// The march is latency-bound: one thread per ray walking a chain of dependent byte reads of the grid (L2-resident at 128^3).
#include "common.cuh"

namespace sdfb200 {

// s = max(|sdf| - bound, 0);  prev / next cdf = sigmoid((s +/- half_step) * inv_s);  alpha = ((p + 1e-5) / (c + 1e-5)).clip(0, 1)
__global__ void __launch_bounds__(256) k_occupancy_prune(const float* __restrict__ sdf, const int64_t* __restrict__ voxel, int64_t n, float bound,
                                                         float half_step, const float* __restrict__ inv_s_ptr, float alpha_thres,
                                                         uint8_t* __restrict__ binary) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float inv_s = inv_s_ptr[0];
  const float s = fmaxf(__fsub_rn(fabsf(sdf[i]), bound), 0.0f);
  const float next_sdf = __fsub_rn(s, half_step);
  const float prev_sdf = __fadd_rn(s, half_step);
  const float prev_cdf = __frcp_rn(__fadd_rn(1.0f, expf(-__fmul_rn(prev_sdf, inv_s))));
  const float next_cdf = __frcp_rn(__fadd_rn(1.0f, expf(-__fmul_rn(next_sdf, inv_s))));
  const float p = __fsub_rn(prev_cdf, next_cdf);
  const float alpha = fminf(fmaxf(__fdiv_rn(__fadd_rn(p, 1e-5f), __fadd_rn(prev_cdf, 1e-5f)), 0.0f), 1.0f);
  if (!(alpha > alpha_thres)) binary[voxel[i]] = 0;   // voxels are only ever removed (a NaN alpha removes, like `alpha > thres`)
}

// Loop iterations of one ray (outer steps plus the steps inside empty-space skips) after which the march stops regardless.
constexpr int64_t kMarchMaxIters = int64_t(1) << 26;

struct MarchArgs {
  const float *o, *d, *nears, *fars;
  const uint8_t* grid;
  int64_t R;
  int res;
  float roi_min[3], roi_max[3], extent[3];
  float step;
  const int64_t* offsets;   // NULL: count pass
  int32_t* counts;
  int64_t* ray_indices;
  float *t_starts, *t_ends;
};

__global__ void __launch_bounds__(128) k_occupancy_march(const MarchArgs a) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.R) return;
  float o[3], d[3], inv_d[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    o[c] = a.o[r * 3 + c];
    d[c] = a.d[r * 3 + c];
    inv_d[c] = __frcp_rn(d[c]);
  }
  const float far = a.fars[r];
  const float res_f = (float)a.res;
  const float dt = a.step;
  const float half_dt = __fmul_rn(dt, 0.5f);
  const bool write = a.offsets != nullptr;
  const int64_t base = write ? a.offsets[r] : 0;
  int64_t j = 0, iters = 0;

  float t0 = a.nears[r];
  float t1 = __fadd_rn(t0, dt);
  float t_mid = __fmul_rn(__fadd_rn(t0, t1), 0.5f);
  // Deliberate deviation from nerfacc: the march stops as soon as a step no longer advances t (fp32 absorption of dt at a large t,
  // where nerfacc would loop forever), and after kMarchMaxIters iterations in all.
  bool alive = t1 > t0;
  while (alive && t_mid < far) {
    float x[3], u[3];
    bool inside = true;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      x[c] = __fadd_rn(o[c], __fmul_rn(t_mid, d[c]));
      inside = inside && !(x[c] < a.roi_min[c] || x[c] > a.roi_max[c]);
      u[c] = __fmul_rn(__fdiv_rn(__fsub_rn(x[c], a.roi_min[c]), a.extent[c]), res_f);   // roi_to_unit(x) * res
    }
    bool occupied = false;
    if (inside) {
      int64_t idx = 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        int v = __float2int_rz(u[c]);
        v = v < 0 ? 0 : (v > a.res - 1 ? a.res - 1 : v);
        idx = idx * a.res + v;
      }
      occupied = a.grid[idx] != 0;
    }
    if (occupied) {
      if (write) {
        a.ray_indices[base + j] = r;
        a.t_starts[base + j] = t0;
        a.t_ends[base + j] = t1;
      }
      ++j;
      t0 = t1;
      t1 = __fadd_rn(t0, dt);
      t_mid = __fmul_rn(__fadd_rn(t0, t1), 0.5f);
      alive = t1 > t0;
    } else {
      // advance_to_next_voxel: distance to the next voxel boundary, then `do t += dt while t < target`
      float dist = INFINITY;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float sgn = copysignf(1.0f, d[c]);
        const float edge = floorf(__fadd_rn(__fadd_rn(u[c], 0.5f), __fmul_rn(0.5f, sgn)));
        const float tc = __fmul_rn(__fdiv_rn(__fmul_rn(__fsub_rn(edge, u[c]), inv_d[c]), res_f), a.extent[c]);
        dist = c == 0 ? tc : fminf(dist, tc);
      }
      dist = fmaxf(dist, 0.0f);
      const float target = __fadd_rn(t_mid, dist);
      float t = t_mid;
      do {
        const float nt = __fadd_rn(t, dt);
        if (!(nt > t)) { alive = false; break; }
        t = nt;
        ++iters;
      } while (t < target && iters < kMarchMaxIters);
      t_mid = t;
      t0 = __fsub_rn(t_mid, half_dt);
      t1 = __fadd_rn(t_mid, half_dt);
      alive = alive && t1 > t0;
    }
    if (++iters >= kMarchMaxIters) alive = false;
  }
  if (!write) a.counts[r] = (int32_t)j;
}

}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_occupancy_prune(const float* sdf, const int64_t* voxel_indices, int64_t n, float bound, float half_step, const float* inv_s,
                                       float alpha_thres, uint8_t* binary, void* stream) {
  SDFB_REQUIRE(n >= 0, "bad sizes");
  if (n == 0) return 0;
  SDFB_REQUIRE(sdf && voxel_indices && inv_s && binary, "NULL pointer");
  k_occupancy_prune<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(sdf, voxel_indices, n, bound, half_step, inv_s, alpha_thres, binary);
  SDFB_LAUNCHED("k_occupancy_prune");
  return 0;
}

extern "C" int sdfb200_occupancy_march(const float* origins, const float* directions, const float* nears, const float* fars, int64_t n_rays,
                                       const float* roi_aabb, const uint8_t* binary, int32_t resolution, float step_size, const int64_t* offsets,
                                       int32_t* counts, int64_t* ray_indices, float* t_starts, float* t_ends, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && resolution >= 1 && resolution <= 2048, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(origins && directions && nears && fars && roi_aabb && binary, "NULL pointer");
  SDFB_REQUIRE(step_size > 0.0f, "step_size must be positive");
  if (offsets) SDFB_REQUIRE(ray_indices && t_starts && t_ends, "the write pass needs ray_indices, t_starts and t_ends");
  else SDFB_REQUIRE(counts != nullptr, "the count pass needs counts");
  MarchArgs a;
  a.o = origins; a.d = directions; a.nears = nears; a.fars = fars; a.grid = binary; a.R = n_rays; a.res = resolution; a.step = step_size;
  for (int c = 0; c < 3; ++c) {
    a.roi_min[c] = roi_aabb[c];
    a.roi_max[c] = roi_aabb[3 + c];
    a.extent[c] = roi_aabb[3 + c] - roi_aabb[c];
    SDFB_REQUIRE(a.extent[c] > 0.0f, "roi_aabb must have max > min");
  }
  a.offsets = offsets; a.counts = counts; a.ray_indices = ray_indices; a.t_starts = t_starts; a.t_ends = t_ends;
  k_occupancy_march<<<(unsigned)ceil_div(n_rays, 128), 128, 0, (cudaStream_t)stream>>>(a);
  SDFB_LAUNCHED("k_occupancy_march");
  return 0;
}
