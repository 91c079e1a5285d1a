// Weights + per-ray compositing (nerfstudio/cameras/rays.py:131-230, model_components/renderers.py dense branch).
// HBM-bound streaming reductions: one thread per ray walks its S samples front to back; transmittance prefixes are
// accumulated in double and rounded per prefix (torch-CPU cumsum / cumprod semantics).
#include "common.cuh"

namespace sdfb200 {

__global__ void __launch_bounds__(128) k_weights_from_alphas(const float* __restrict__ alphas, int64_t R, int S, float* __restrict__ weights,
                                                             float* __restrict__ trans) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  double T = 1.0;
  for (int i = 0; i < S; ++i) {
    const float a = alphas[r * S + i];
    const float Tf = (float)T;
    if (trans) trans[r * (S + 1) + i] = Tf;
    weights[r * S + i] = __fmul_rn(a, Tf);
    T *= (double)neus_trans_factor(a);
  }
  if (trans) trans[r * (S + 1) + S] = (float)T;
}

__global__ void __launch_bounds__(128) k_weights_from_density(const float* __restrict__ density, const float* __restrict__ eu, int64_t R, int S,
                                                              float* __restrict__ weights, float* __restrict__ trans) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* e = eu + r * (S + 1);
  double integ = 0.0;
  for (int i = 0; i < S; ++i) {
    const float dd = __fmul_rn(__fsub_rn(e[i + 1], e[i]), density[r * S + i]);
    const float T = expf(-(float)integ);
    if (trans) trans[r * S + i] = T;
    weights[r * S + i] = __fmul_rn(__fsub_rn(1.0f, expf(-dd)), T);
    integ += (double)dd;
  }
}

struct RenderArgs {
  const float* weights; const float* rgb; const float* normals; const float* eu; const float* bg;
  int bg_mode, clamp01, depth_median; int64_t R; int S;
  float *o_rgb, *o_depth, *o_normal, *o_acc, *o_minmax;
};

__global__ void __launch_bounds__(128) k_render(const RenderArgs a) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  float smin = INFINITY, smax = -INFINITY;
  if (r < a.R) {
    const int S = a.S;
    const float* w = a.weights + r * S;
    float cr = 0.f, cg = 0.f, cb = 0.f, acc = 0.f, dsum = 0.f, nx = 0.f, ny = 0.f, nz = 0.f;
    double cum = 0.0;
    int median_idx = -1;
    for (int i = 0; i < S; ++i) {
      const float wi = w[i];
      acc += wi;
      if (a.rgb) {
        const float* c = a.rgb + (r * S + i) * 3;
        cr = __fadd_rn(cr, __fmul_rn(wi, c[0])); cg = __fadd_rn(cg, __fmul_rn(wi, c[1])); cb = __fadd_rn(cb, __fmul_rn(wi, c[2]));
      }
      if (a.normals && a.o_normal) {
        const float* n = a.normals + (r * S + i) * 3;
        nx = __fadd_rn(nx, __fmul_rn(wi, n[0])); ny = __fadd_rn(ny, __fmul_rn(wi, n[1])); nz = __fadd_rn(nz, __fmul_rn(wi, n[2]));
      }
      if (a.eu && a.o_depth) {
        const float step = __fdiv_rn(__fadd_rn(a.eu[r * (S + 1) + i], a.eu[r * (S + 1) + i + 1]), 2.0f);
        dsum = __fadd_rn(dsum, __fmul_rn(wi, step));
        smin = fminf(smin, step); smax = fmaxf(smax, step);
        if (a.depth_median) {
          cum += (double)wi;
          if (median_idx < 0 && (float)cum >= 0.5f) median_idx = i;  // searchsorted(side="left")
        }
      }
    }
    if (a.o_rgb && a.rgb) {
      float bgc[3];
      ray_background(a.bg_mode, a.bg, r, a.rgb + (r * S + S - 1) * 3, bgc);
      const float rem = __fsub_rn(1.0f, acc);
      float o[3] = {__fadd_rn(cr, __fmul_rn(bgc[0], rem)), __fadd_rn(cg, __fmul_rn(bgc[1], rem)), __fadd_rn(cb, __fmul_rn(bgc[2], rem))};
      for (int c = 0; c < 3; ++c) a.o_rgb[r * 3 + c] = a.clamp01 ? fminf(fmaxf(o[c], 0.f), 1.f) : o[c];
    }
    if (a.o_acc) a.o_acc[r] = acc;
    if (a.o_normal && a.normals) { a.o_normal[r * 3] = nx; a.o_normal[r * 3 + 1] = ny; a.o_normal[r * 3 + 2] = nz; }
    if (a.o_depth && a.eu) {
      if (a.depth_median) {
        int idx = median_idx < 0 ? S : median_idx;
        idx = idx > S - 1 ? S - 1 : idx;
        a.o_depth[r] = __fdiv_rn(__fadd_rn(a.eu[r * (S + 1) + idx], a.eu[r * (S + 1) + idx + 1]), 2.0f);
      } else {
        a.o_depth[r] = __fdiv_rn(dsum, __fadd_rn(acc, 1e-10f));
      }
    }
  }
  if (a.o_minmax && a.eu && a.o_depth) {
    // batch-global steps.min()/max() for the clip at renderers.py:257
    for (int s = 16; s > 0; s >>= 1) {
      smin = fminf(smin, __shfl_xor_sync(0xffffffffu, smin, s));
      smax = fmaxf(smax, __shfl_xor_sync(0xffffffffu, smax, s));
    }
    if ((threadIdx.x & 31) == 0 && smin <= smax) {
      atomic_min_float(a.o_minmax, smin);
      atomic_max_float(a.o_minmax + 1, smax);
    }
  }
}

// -----------------------------------------------------------------------------------------------------------------
// fused alpha -> transmittance -> weights -> composite, ONE WARP PER RAY (coalesced: lane = sample % 32; the running
// transmittance is a warp-level prefix product in double, carried across 32-sample rows).  What SurfaceModel.get_outputs does
// with get_weights_and_transmittance_from_alphas + four renderers (models/neus.py:100-103, base_surface_model.py:300-310).
// -----------------------------------------------------------------------------------------------------------------
struct RenderAlphaArgs {
  const float* alphas; const float* rgb; const float* normals; const float* eu; const float* bg;
  int bg_mode, clamp01; int64_t R; int S;
  float *o_weights, *o_rgb, *o_depth, *o_normal, *o_acc, *o_bgT, *o_minmax;
};
__global__ void __launch_bounds__(256) k_render_alphas(const RenderAlphaArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= a.R) return;  // whole warp
  const int S = a.S;
  double carry = 1.0;
  float cr = 0.f, cg = 0.f, cb = 0.f, acc = 0.f, dsum = 0.f, nx = 0.f, ny = 0.f, nz = 0.f, smin = INFINITY, smax = -INFINITY;
  for (int s0 = 0; s0 < S; s0 += 32) {
    const int s = s0 + lane;
    const bool on = s < S;
    const float al = on ? a.alphas[r * S + s] : 0.f;
    const double incl = warp_scan_incl(on ? (double)neus_trans_factor(al) : 1.0, lane, ScanMul());
    const double excl = warp_scan_excl(incl, lane, 1.0);
    const float T = (float)(carry * excl);
    carry *= __shfl_sync(0xffffffffu, incl, 31);
    const float w = __fmul_rn(al, T);
    if (on) {
      if (a.o_weights) a.o_weights[r * S + s] = w;
      acc += w;
      if (a.rgb) { const float* c = a.rgb + (r * S + s) * 3; cr = fmaf(w, c[0], cr); cg = fmaf(w, c[1], cg); cb = fmaf(w, c[2], cb); }
      if (a.normals) { const float* n = a.normals + (r * S + s) * 3; nx = fmaf(w, n[0], nx); ny = fmaf(w, n[1], ny); nz = fmaf(w, n[2], nz); }
      if (a.eu) {
        const float step = __fdiv_rn(__fadd_rn(a.eu[r * (S + 1) + s], a.eu[r * (S + 1) + s + 1]), 2.0f);
        dsum = fmaf(w, step, dsum);
        smin = fminf(smin, step); smax = fmaxf(smax, step);
      }
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    cr += __shfl_xor_sync(0xffffffffu, cr, d); cg += __shfl_xor_sync(0xffffffffu, cg, d); cb += __shfl_xor_sync(0xffffffffu, cb, d);
    nx += __shfl_xor_sync(0xffffffffu, nx, d); ny += __shfl_xor_sync(0xffffffffu, ny, d); nz += __shfl_xor_sync(0xffffffffu, nz, d);
    acc += __shfl_xor_sync(0xffffffffu, acc, d); dsum += __shfl_xor_sync(0xffffffffu, dsum, d);
    smin = fminf(smin, __shfl_xor_sync(0xffffffffu, smin, d)); smax = fmaxf(smax, __shfl_xor_sync(0xffffffffu, smax, d));
  }
  if (lane == 0) {
    finish_ray(r, acc, {cr, cg, cb}, {nx, ny, nz}, dsum, a.bg_mode, a.bg, a.rgb + (r * S + S - 1) * 3, a.clamp01, a.rgb ? a.o_rgb : nullptr, a.o_acc,
               a.normals ? a.o_normal : nullptr, a.eu ? a.o_depth : nullptr);
    if (a.o_bgT) a.o_bgT[r] = (float)carry;                               // transmittance[:, -1] (bg_transmittance)
    if (a.o_minmax && a.eu && smin <= smax) { atomic_min_float(a.o_minmax, smin); atomic_max_float(a.o_minmax + 1, smax); }
  }
}

// -----------------------------------------------------------------------------------------------------------------
// packed samples (the nerfacc branch of the renderers: renderers.py:74-79,192-194,249-253): samples of all rays in one flat
// list with a ray index each; nerfacc.accumulate_along_rays == scatter-add per ray.  Pass 1 accumulates, pass 2 finalises.
// -----------------------------------------------------------------------------------------------------------------
struct PackedArgs {
  const float* weights; const float* rgb; const float* normals; const float* starts; const float* ends; const int64_t* ray_indices;
  int64_t N, R;
  float* acc;  // [R][8]: sum w, sum w rgb (3), sum w step, sum w n (3)
  float* o_minmax;
};
__global__ void __launch_bounds__(256) k_render_packed_accumulate(const PackedArgs a) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  float smin = INFINITY, smax = -INFINITY;
  if (i < a.N) {
    const int64_t r = a.ray_indices[i];
    if (r >= 0 && r < a.R) {
      const float w = a.weights[i];
      float* o = a.acc + r * 8;
      atomicAdd(o, w);
      if (a.rgb) { atomicAdd(o + 1, w * a.rgb[i * 3]); atomicAdd(o + 2, w * a.rgb[i * 3 + 1]); atomicAdd(o + 3, w * a.rgb[i * 3 + 2]); }
      if (a.starts) {
        const float step = __fdiv_rn(__fadd_rn(a.starts[i], a.ends[i]), 2.0f);
        atomicAdd(o + 4, w * step);
        smin = smax = step;
      }
      if (a.normals) { atomicAdd(o + 5, w * a.normals[i * 3]); atomicAdd(o + 6, w * a.normals[i * 3 + 1]); atomicAdd(o + 7, w * a.normals[i * 3 + 2]); }
    }
  }
  if (a.o_minmax && a.starts) {
    for (int s = 16; s > 0; s >>= 1) {
      smin = fminf(smin, __shfl_xor_sync(0xffffffffu, smin, s));
      smax = fmaxf(smax, __shfl_xor_sync(0xffffffffu, smax, s));
    }
    if ((threadIdx.x & 31) == 0 && smin <= smax) { atomic_min_float(a.o_minmax, smin); atomic_max_float(a.o_minmax + 1, smax); }
  }
}
__global__ void k_render_packed_finish(const float* __restrict__ acc, int64_t R, const float* __restrict__ bg, int bg_mode, int clamp01, float* o_rgb,
                                       float* o_depth, float* o_normal, float* o_acc) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* a = acc + r * 8;
  const float w = a[0];
  // not finish_ray: packed samples have no last-sample background, and its three-way background select costs 20 % more instructions here
  if (o_rgb) {
    const float* b = bg_mode == SDFB200_BG_PER_RAY ? bg + r * 3 : bg;
    const float rem = 1.0f - w;
    for (int c = 0; c < 3; ++c) {
      const float v = a[1 + c] + b[c] * rem;
      o_rgb[r * 3 + c] = clamp01 ? fminf(fmaxf(v, 0.f), 1.f) : v;
    }
  }
  if (o_acc) o_acc[r] = w;
  if (o_depth) o_depth[r] = a[4] / (w + 1e-10f);
  if (o_normal) { o_normal[r * 3] = a[5]; o_normal[r * 3 + 1] = a[6]; o_normal[r * 3 + 2] = a[7]; }
}

// -----------------------------------------------------------------------------------------------------------------
// segmented packed samples (nerfacc 0.3.5 render_weight_from_alpha / accumulate_along_rays, models/neus_acc.py:102-120): the samples of
// ray r are the contiguous segment [offsets[r], offsets[r+1]).  ONE WARP PER RAY streams its segment (lane = sample % 32); every sum and
// product runs in double in a fixed order, so the results are deterministic and need no atomics.
// -----------------------------------------------------------------------------------------------------------------
// w = alpha T, T = exclusive product of (1 - alpha) over the segment (no +1e-7, unlike the dense rays.py:204)
__global__ void __launch_bounds__(256) k_packed_weights(const float* __restrict__ alphas, const int64_t* __restrict__ offsets, int64_t R,
                                                        float* __restrict__ weights) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= R) return;  // whole warp
  const int64_t b = offsets[r], e = offsets[r + 1];
  double carry = 1.0;
  for (int64_t s0 = b; s0 < e; s0 += 32) {
    const int64_t s = s0 + lane;
    const bool on = s < e;
    const float al = on ? alphas[s] : 0.f;
    const double incl = warp_scan_incl(1.0 - (double)al, lane, ScanMul());
    const double excl = warp_scan_excl(incl, lane, 1.0);
    if (on) weights[s] = (float)((double)al * (carry * excl));
    carry *= __shfl_sync(0xffffffffu, incl, 31);
  }
}

// out[r, c] = sum over the segment of w * values[:, c]  (values == NULL: sum of w, C = 1)
__global__ void __launch_bounds__(256) k_packed_accumulate(const float* __restrict__ weights, const float* __restrict__ values,
                                                           const int64_t* __restrict__ offsets, int64_t R, int C, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= R) return;  // whole warp
  const int64_t b = offsets[r], e = offsets[r + 1];
  for (int c0 = 0; c0 < C; c0 += 4) {
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int64_t s = b + lane; s < e; s += 32) {
      const double w = (double)weights[s];
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (c0 + k < C) acc[k] += values ? w * (double)values[s * C + c0 + k] : w;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], d);
      if (lane == 0 && c0 + k < C) out[r * C + c0 + k] = (float)acc[k];
    }
  }
}

__global__ void k_depth_clip(float* __restrict__ depth, const float* __restrict__ mm, int64_t R) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < R) depth[r] = fminf(fmaxf(depth[r], mm[0]), mm[1]);
}

}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_weights_from_alphas(const float* alphas, int64_t n_rays, int32_t n_samples, float* weights, float* transmittance, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(alphas && weights, "NULL pointer");
  k_weights_from_alphas<<<(unsigned)ceil_div(n_rays, 128), 128, 0, (cudaStream_t)stream>>>(alphas, n_rays, n_samples, weights, transmittance);
  SDFB_LAUNCHED("k_weights_from_alphas");
  return 0;
}

extern "C" int sdfb200_weights_from_density(const float* density, const float* euclid_bins, int64_t n_rays, int32_t n_samples, float* weights,
                                            float* transmittance, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(density && euclid_bins && weights, "NULL pointer");
  k_weights_from_density<<<(unsigned)ceil_div(n_rays, 128), 128, 0, (cudaStream_t)stream>>>(density, euclid_bins, n_rays, n_samples, weights, transmittance);
  SDFB_LAUNCHED("k_weights_from_density");
  return 0;
}

extern "C" int sdfb200_render(const float* weights, const float* rgb, const float* normals, const float* euclid_bins, const float* bg, int32_t bg_mode,
                              int32_t clamp01, int32_t depth_median, int64_t n_rays, int32_t n_samples, const sdfb200_render_out_t* out, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sizes");
  SDFB_REQUIRE(out != nullptr && weights != nullptr, "NULL pointer");
  if (n_rays == 0) return 0;
  if (out->rgb) SDFB_REQUIRE(rgb != nullptr && (bg_mode == SDFB200_BG_LAST_SAMPLE || bg != nullptr), "rgb output needs rgb and background");
  if (out->depth) SDFB_REQUIRE(euclid_bins != nullptr, "depth output needs bins");
  if (out->normal) SDFB_REQUIRE(normals != nullptr, "normal output needs normals");
  RenderArgs a;
  a.weights = weights; a.rgb = rgb; a.normals = normals; a.eu = euclid_bins; a.bg = bg; a.bg_mode = bg_mode; a.clamp01 = clamp01;
  a.depth_median = depth_median; a.R = n_rays; a.S = n_samples; a.o_rgb = out->rgb; a.o_depth = out->depth; a.o_normal = out->normal;
  a.o_acc = out->accumulation; a.o_minmax = out->steps_minmax;
  k_render<<<(unsigned)ceil_div(n_rays, 128), 128, 0, (cudaStream_t)stream>>>(a);
  SDFB_LAUNCHED("k_render");
  return 0;
}

extern "C" int sdfb200_depth_clip(float* depth, const float* steps_minmax, int64_t n_rays, void* stream) {
  SDFB_REQUIRE(n_rays >= 0, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(depth && steps_minmax, "NULL pointer");
  k_depth_clip<<<(unsigned)ceil_div(n_rays, 256), 256, 0, (cudaStream_t)stream>>>(depth, steps_minmax, n_rays);
  SDFB_LAUNCHED("k_depth_clip");
  return 0;
}


extern "C" int sdfb200_render_alphas(const float* alphas, const float* rgb, const float* normals, const float* euclid_bins, const float* bg,
                                     int32_t bg_mode, int32_t clamp01, int64_t n_rays, int32_t n_samples, float* weights, float* bg_transmittance,
                                     const sdfb200_render_out_t* out, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sizes");
  SDFB_REQUIRE(out != nullptr && alphas != nullptr, "NULL pointer");
  if (n_rays == 0) return 0;
  if (out->rgb) SDFB_REQUIRE(rgb != nullptr && (bg_mode == SDFB200_BG_LAST_SAMPLE || bg != nullptr), "rgb output needs rgb and background");
  if (out->depth) SDFB_REQUIRE(euclid_bins != nullptr, "depth output needs bins");
  if (out->normal) SDFB_REQUIRE(normals != nullptr, "normal output needs normals");
  RenderAlphaArgs a;
  a.alphas = alphas; a.rgb = rgb; a.normals = out->normal ? normals : nullptr; a.eu = out->depth ? euclid_bins : nullptr; a.bg = bg; a.bg_mode = bg_mode;
  a.clamp01 = clamp01; a.R = n_rays; a.S = n_samples; a.o_weights = weights; a.o_rgb = out->rgb; a.o_depth = out->depth; a.o_normal = out->normal;
  a.o_acc = out->accumulation; a.o_bgT = bg_transmittance; a.o_minmax = out->steps_minmax;
  k_render_alphas<<<(unsigned)ceil_div(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(a);
  SDFB_LAUNCHED("k_render_alphas");
  return 0;
}

extern "C" int sdfb200_render_packed(const float* weights, const float* rgb, const float* normals, const float* starts, const float* ends,
                                     const int64_t* ray_indices, int64_t n_samples_total, int64_t n_rays, const float* bg, int32_t bg_mode, int32_t clamp01,
                                     const sdfb200_render_out_t* out, void* workspace, size_t workspace_bytes, void* stream) {
  SDFB_REQUIRE(n_samples_total >= 0 && n_rays >= 0, "bad sizes");
  SDFB_REQUIRE(out != nullptr, "NULL pointer");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(workspace != nullptr && workspace_bytes >= (size_t)n_rays * 8 * sizeof(float), "render_packed: workspace must hold 8 floats per ray");
  SDFB_REQUIRE(n_samples_total == 0 || (weights && ray_indices), "NULL pointer");
  SDFB_REQUIRE(bg_mode != SDFB200_BG_LAST_SAMPLE, "background 'last_sample' is not defined for packed samples (renderers.py:76-77)");
  if (out->rgb) SDFB_REQUIRE(rgb != nullptr && bg != nullptr, "rgb output needs rgb and background");
  if (out->depth) SDFB_REQUIRE(starts != nullptr && ends != nullptr, "depth output needs starts and ends");
  if (out->normal) SDFB_REQUIRE(normals != nullptr, "normal output needs normals");
  SDFB_CUDA(cudaMemsetAsync(workspace, 0, (size_t)n_rays * 8 * sizeof(float), (cudaStream_t)stream));
  PackedArgs a;
  a.weights = weights; a.rgb = out->rgb ? rgb : nullptr; a.normals = out->normal ? normals : nullptr; a.starts = out->depth ? starts : nullptr; a.ends = ends;
  a.ray_indices = ray_indices; a.N = n_samples_total; a.R = n_rays; a.acc = (float*)workspace; a.o_minmax = out->steps_minmax;
  if (n_samples_total > 0) {
    k_render_packed_accumulate<<<(unsigned)ceil_div(n_samples_total, 256), 256, 0, (cudaStream_t)stream>>>(a);
    SDFB_LAUNCHED("k_render_packed_accumulate");
  }
  k_render_packed_finish<<<(unsigned)ceil_div(n_rays, 256), 256, 0, (cudaStream_t)stream>>>((const float*)workspace, n_rays, bg, bg_mode, clamp01, out->rgb,
                                                                                             out->depth, out->normal, out->accumulation);
  SDFB_LAUNCHED("k_render_packed_finish");
  return 0;
}

extern "C" int sdfb200_packed_weights(const float* alphas, const int64_t* offsets, int64_t n_rays, float* weights, void* stream) {
  SDFB_REQUIRE(n_rays >= 0, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(alphas && offsets && weights, "NULL pointer");
  k_packed_weights<<<(unsigned)ceil_div(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(alphas, offsets, n_rays, weights);
  SDFB_LAUNCHED("k_packed_weights");
  return 0;
}

extern "C" int sdfb200_packed_accumulate(const float* weights, const float* values, int32_t n_channels, const int64_t* offsets, int64_t n_rays,
                                         float* out, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_channels >= 1, "bad sizes");
  SDFB_REQUIRE(values != nullptr || n_channels == 1, "values == NULL accumulates the weights: n_channels must be 1");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(weights && offsets && out, "NULL pointer");
  k_packed_accumulate<<<(unsigned)ceil_div(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(weights, values, offsets, n_rays, n_channels, out);
  SDFB_LAUNCHED("k_packed_accumulate");
  return 0;
}
