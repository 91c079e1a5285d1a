// Backward of the weights / compositing operators (training path).  The reference gets these from autograd over
// rays.py:131-230 and renderers.py:42-295; here they are two explicit kernels:
//   k_render_bwd   : d(per-ray outputs)/d(weights, rgb samples, normal samples)    -- elementwise given per-ray scalars
//   k_weights_bwd  : d(weights, last transmittance)/d(alphas | density)            -- one warp per ray, prefix scans in double
#include "common.cuh"

namespace sdfb200 {

struct RenderBwdArgs {
  const float *weights, *rgb, *normals, *eu, *bg;
  int bg_mode; int64_t R; int S;
  const float *acc, *depth;
  const float *g_rgb, *g_depth, *g_normal, *g_acc, *g_weights_in;
  float *g_weights, *g_rgb_s, *g_normal_s;
};

__global__ void __launch_bounds__(256) k_render_bwd(const RenderBwdArgs a) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.R * a.S) return;
  const int64_t r = i / a.S;
  const int s = (int)(i - r * a.S);
  const int S = a.S;
  const float w = a.weights[i];
  float gw = a.g_weights_in ? a.g_weights_in[i] : 0.f;
  if (a.g_rgb) {
    const float g0 = a.g_rgb[r * 3], g1 = a.g_rgb[r * 3 + 1], g2 = a.g_rgb[r * 3 + 2];
    const float* c = a.rgb + i * 3;
    float b[3];
    ray_background(a.bg_mode, a.bg, r, a.rgb + (r * S + S - 1) * 3, b);
    gw += g0 * (c[0] - b[0]) + g1 * (c[1] - b[1]) + g2 * (c[2] - b[2]);   // out = sum w c + bg (1 - sum w)
    if (a.g_rgb_s) {
      float e0 = g0 * w, e1 = g1 * w, e2 = g2 * w;
      if (a.bg_mode == SDFB200_BG_LAST_SAMPLE && s == S - 1) {
        const float rem = 1.0f - a.acc[r];
        e0 += g0 * rem; e1 += g1 * rem; e2 += g2 * rem;
      }
      a.g_rgb_s[i * 3] = e0; a.g_rgb_s[i * 3 + 1] = e1; a.g_rgb_s[i * 3 + 2] = e2;
    }
  } else if (a.g_rgb_s) {
    a.g_rgb_s[i * 3] = 0.f; a.g_rgb_s[i * 3 + 1] = 0.f; a.g_rgb_s[i * 3 + 2] = 0.f;
  }
  if (a.g_normal) {
    const float g0 = a.g_normal[r * 3], g1 = a.g_normal[r * 3 + 1], g2 = a.g_normal[r * 3 + 2];
    const float* n = a.normals + i * 3;
    gw += g0 * n[0] + g1 * n[1] + g2 * n[2];
    if (a.g_normal_s) { a.g_normal_s[i * 3] = g0 * w; a.g_normal_s[i * 3 + 1] = g1 * w; a.g_normal_s[i * 3 + 2] = g2 * w; }
  } else if (a.g_normal_s) {
    a.g_normal_s[i * 3] = 0.f; a.g_normal_s[i * 3 + 1] = 0.f; a.g_normal_s[i * 3 + 2] = 0.f;
  }
  if (a.g_acc) gw += a.g_acc[r];
  if (a.g_depth) {
    // depth = sum(w step) / (acc + 1e-10)   (renderers.py:249-252, before the global clip)
    const float step = (a.eu[r * (S + 1) + s] + a.eu[r * (S + 1) + s + 1]) * 0.5f;
    gw += a.g_depth[r] * (step - a.depth[r]) / (a.acc[r] + 1e-10f);
  }
  a.g_weights[i] = gw;
}

// weights_i = alpha_i T_i,  T_i = prod_{j<i} f_j,  f_j = 1 - alpha_j + 1e-7 (rays.py:204-206)     [mode 0]
// weights_i = (1 - f_i) T_i, f_i = exp(-delta_i sigma_i), T_i = exp(-sum_{j<i} delta_j sigma_j) (rays.py:131-180)  [mode 1]
//   dL/dalpha_i = gw_i T_i - (sum_{k>i} (gw_k w_k + gT_k T_k) + gT_S T_S) / f_i ;      dL/dsigma_i = delta_i f_i dL/dalpha_i
// g_T: gradient of the returned transmittance, gt_cols = 0 (none), 1 (only the last column, [R]: bg_transmittance of
// models/neus.py:101) or the full width ([R,S+1] for alphas, [R,S] for densities: volsdf.py:67-68 reads transmittance[:, -1],
// the transmittance BEFORE the last sample).
__global__ void __launch_bounds__(256) k_weights_bwd(const float* __restrict__ in, const float* __restrict__ eu, int from_density, int64_t R, int S,
                                                     const float* __restrict__ g_weights, const float* __restrict__ g_T, int gt_cols,
                                                     float* __restrict__ g_in) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= R) return;
  double U = 0.0, TS = 1.0;
  for (int pass = 0; pass < 2; ++pass) {
    double carryT = 1.0, carryI = 0.0, carryU = 0.0;
    for (int s0 = 0; s0 < S; s0 += 32) {
      const int s = s0 + lane;
      const bool on = s < S;
      float f = 1.f, al = 0.f, delta = 0.f, T;
      if (!from_density) {
        al = on ? in[r * S + s] : 0.f;
        f = on ? neus_trans_factor(al) : 1.f;
        const double incl = warp_scan_incl((double)f, lane, ScanMul());
        T = (float)(carryT * warp_scan_excl(incl, lane, 1.0));
        carryT *= __shfl_sync(0xffffffffu, incl, 31);
      } else {
        delta = on ? __fsub_rn(eu[r * (S + 1) + s + 1], eu[r * (S + 1) + s]) : 0.f;
        const float dd = on ? __fmul_rn(delta, in[r * S + s]) : 0.f;
        const double incl = warp_scan_incl((double)dd, lane);
        T = expf(-(float)(carryI + warp_scan_excl(incl, lane, 0.0)));
        carryI += __shfl_sync(0xffffffffu, incl, 31);
        f = expf(-dd);
        al = 1.0f - f;
      }
      const float gw = on ? g_weights[r * S + s] : 0.f;
      const float gt = (on && (from_density ? gt_cols >= 1 : gt_cols > 1)) ? g_T[r * gt_cols + s] : 0.f;
      const double u = (double)gw * (double)(al * T) + (double)gt * (double)T;
      const double uincl = warp_scan_incl(u, lane);
      if (pass == 1 && on) {
        const double suffix = U - (carryU + uincl);                       // sum_{k>s} gw_k w_k
        const double tail = suffix + ((!from_density && gt_cols >= 1) ? (double)g_T[r * gt_cols + (gt_cols - 1)] * TS : 0.0);
        if (!from_density) g_in[r * S + s] = (float)((double)gw * (double)T - tail / (double)f);
        else g_in[r * S + s] = (float)((double)delta * ((double)gw * (double)T * (double)f - tail));
      }
      carryU += __shfl_sync(0xffffffffu, uincl, 31);
    }
    if (pass == 0) { U = carryU; TS = from_density ? 1.0 : carryT; }
  }
}

// backward of k_packed_weights (w_k = alpha_k T_k over a segment), one warp per ray, without division (finite at alpha = 1):
//   dL/dalpha_k = T_k (g_k - S_k),  S_k = g_{k+1} alpha_{k+1} + (1 - alpha_{k+1}) S_{k+1},  S_last = 0.
// A forward pass stages T_k in g_alpha; a reverse pass scans R_k = g_k alpha_k + (1 - alpha_k) R_{k+1} (S_k = R_{k+1}) as a suffix
// composition of affine maps in double and overwrites g_alpha.
__global__ void __launch_bounds__(256) k_packed_weights_bwd(const float* __restrict__ alphas, const int64_t* __restrict__ offsets, int64_t R,
                                                            const float* __restrict__ g_w, float* __restrict__ g_alpha) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= R) return;  // whole warp
  const int64_t b = offsets[r], e = offsets[r + 1];
  if (e <= b) return;
  double carry = 1.0;
  for (int64_t s0 = b; s0 < e; s0 += 32) {
    const int64_t s = s0 + lane;
    const bool on = s < e;
    const double incl = warp_scan_incl(on ? 1.0 - (double)alphas[s] : 1.0, lane, ScanMul());
    const double excl = warp_scan_excl(incl, lane, 1.0);
    if (on) g_alpha[s] = (float)(carry * excl);
    carry *= __shfl_sync(0xffffffffu, incl, 31);
  }
  double carry_r = 0.0;   // R of the first sample after this chunk
  for (int64_t s0 = b + (e - 1 - b) / 32 * 32; s0 >= b; s0 -= 32) {
    const int64_t s = s0 + lane;
    const bool on = s < e;
    const double al = on ? (double)alphas[s] : 0.0;
    const double g = on ? (double)g_w[s] : 0.0;
    double A = g * al, B = 1.0 - al;   // R_s = A + B R_{s+1}
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const double Ao = __shfl_down_sync(0xffffffffu, A, d);
      const double Bo = __shfl_down_sync(0xffffffffu, B, d);
      if (lane + d < 32) { A += B * Ao; B *= Bo; }
    }
    const double Rk = A + B * carry_r;
    double S = __shfl_down_sync(0xffffffffu, Rk, 1);
    if (lane == 31) S = carry_r;
    if (on) g_alpha[s] = (float)((double)g_alpha[s] * (g - S));
    carry_r = __shfl_sync(0xffffffffu, Rk, 0);
  }
}

// backward of sdfb200_render_packed (the ray_indices branch of the renderers), one thread per sample; any sample order, like the
// forward's atomics.  Same per-sample terms as k_render_bwd with r = ray_indices[i] and step = (starts + ends) / 2; a sample whose ray
// index lies outside [0, R) does not reach the forward and gets zero gradients.  g_steps [N]: d/d step_i = g_depth[r] w_i / (acc_r + 1e-10).
struct PackedRenderBwdArgs {
  const float *weights, *rgb, *normals, *starts, *ends, *bg;
  const int64_t* ray_indices;
  int bg_mode; int64_t N, R;
  const float *acc, *depth;
  const float *g_rgb, *g_depth, *g_normal, *g_acc;
  float *g_weights, *g_rgb_s, *g_normal_s, *g_steps;
};

__global__ void __launch_bounds__(256) k_render_packed_bwd(const PackedRenderBwdArgs a) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.N) return;
  const int64_t r = a.ray_indices[i];
  const bool in = r >= 0 && r < a.R;
  const float w = a.weights[i];
  float gw = 0.f, e[3] = {0.f, 0.f, 0.f}, m[3] = {0.f, 0.f, 0.f}, gs = 0.f;
  if (in && a.g_rgb) {
    // not ray_background: packed samples have no last-sample background, and the pointer select here takes 2 registers fewer
    const float* b = a.bg_mode == SDFB200_BG_PER_RAY ? a.bg + r * 3 : a.bg;
    for (int c = 0; c < 3; ++c) {
      const float g = a.g_rgb[r * 3 + c];
      gw += g * (a.rgb[i * 3 + c] - b[c]);   // out = sum w c + bg (1 - sum w)
      e[c] = g * w;
    }
  }
  if (in && a.g_normal) {
    for (int c = 0; c < 3; ++c) {
      const float g = a.g_normal[r * 3 + c];
      gw += g * a.normals[i * 3 + c];
      m[c] = g * w;
    }
  }
  if (in && a.g_acc) gw += a.g_acc[r];
  if (in && a.g_depth) {
    // depth = sum(w step) / (acc + 1e-10)   (renderers.py:249-252, before the global clip)
    const float step = (a.starts[i] + a.ends[i]) * 0.5f;
    const float q = a.g_depth[r] / (a.acc[r] + 1e-10f);
    gw += q * (step - a.depth[r]);
    gs = q * w;
  }
  a.g_weights[i] = gw;
  if (a.g_rgb_s) for (int c = 0; c < 3; ++c) a.g_rgb_s[i * 3 + c] = e[c];
  if (a.g_normal_s) for (int c = 0; c < 3; ++c) a.g_normal_s[i * 3 + c] = m[c];
  if (a.g_steps) a.g_steps[i] = gs;
}

// backward of k_packed_accumulate, one thread per sample: dv[i, c] = w_i g[r_i, c],  dw_i = sum_c g[r_i, c] v[i, c]  (or g[r_i])
__global__ void __launch_bounds__(256) k_packed_accumulate_bwd(const float* __restrict__ weights, const float* __restrict__ values,
                                                               const int64_t* __restrict__ ray_indices, int64_t N, int C,
                                                               const float* __restrict__ g_out, float* __restrict__ g_w, float* __restrict__ g_v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float* g = g_out + ray_indices[i] * C;
  if (g_w) {
    double s = 0.0;
    for (int c = 0; c < C; ++c) s += (double)g[c] * (values ? (double)values[i * C + c] : 1.0);
    g_w[i] = (float)s;
  }
  if (g_v) {
    const float w = weights[i];
    for (int c = 0; c < C; ++c) g_v[i * C + c] = __fmul_rn(w, g[c]);
  }
}

}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_packed_weights_backward(const float* alphas, const int64_t* offsets, int64_t n_rays, const float* g_weights, float* g_alphas,
                                               void* stream) {
  SDFB_REQUIRE(n_rays >= 0, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(alphas && offsets && g_weights && g_alphas, "NULL pointer");
  k_packed_weights_bwd<<<(unsigned)ceil_div(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(alphas, offsets, n_rays, g_weights, g_alphas);
  SDFB_LAUNCHED("k_packed_weights_bwd");
  return 0;
}

extern "C" int sdfb200_packed_accumulate_backward(const float* weights, const float* values, int32_t n_channels, const int64_t* ray_indices,
                                                  int64_t n_samples_total, const float* g_out, float* g_weights, float* g_values, void* stream) {
  SDFB_REQUIRE(n_samples_total >= 0 && n_channels >= 1, "bad sizes");
  SDFB_REQUIRE(values != nullptr || n_channels == 1, "values == NULL accumulates the weights: n_channels must be 1");
  if (n_samples_total == 0) return 0;
  SDFB_REQUIRE(ray_indices && g_out, "NULL pointer");
  if (g_values) SDFB_REQUIRE(values != nullptr && weights != nullptr, "g_values needs values and weights");
  k_packed_accumulate_bwd<<<(unsigned)ceil_div(n_samples_total, 256), 256, 0, (cudaStream_t)stream>>>(weights, values, ray_indices, n_samples_total,
                                                                                                     n_channels, g_out, g_weights, g_values);
  SDFB_LAUNCHED("k_packed_accumulate_bwd");
  return 0;
}

extern "C" int sdfb200_render_backward(const float* weights, const float* rgb, const float* normals, const float* euclid_bins, const float* bg,
                                       int32_t bg_mode, int64_t n_rays, int32_t n_samples, const float* accumulation, const float* depth,
                                       const float* g_rgb, const float* g_depth, const float* g_normal, const float* g_accumulation,
                                       const float* g_weights_in, float* g_weights, float* g_rgb_samples, float* g_normal_samples, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(weights && g_weights, "NULL pointer");
  if (g_rgb) SDFB_REQUIRE(rgb != nullptr && (bg_mode == SDFB200_BG_LAST_SAMPLE || bg != nullptr) && accumulation != nullptr, "g_rgb needs rgb, background, accumulation");
  if (g_normal) SDFB_REQUIRE(normals != nullptr, "g_normal needs normals");
  if (g_depth) SDFB_REQUIRE(euclid_bins != nullptr && depth != nullptr && accumulation != nullptr, "g_depth needs bins, depth, accumulation");
  RenderBwdArgs a;
  a.weights = weights; a.rgb = rgb; a.normals = normals; a.eu = euclid_bins; a.bg = bg; a.bg_mode = bg_mode; a.R = n_rays; a.S = n_samples;
  a.acc = accumulation; a.depth = depth; a.g_rgb = g_rgb; a.g_depth = g_depth; a.g_normal = g_normal; a.g_acc = g_accumulation;
  a.g_weights_in = g_weights_in; a.g_weights = g_weights; a.g_rgb_s = g_rgb_samples; a.g_normal_s = g_normal_samples;
  k_render_bwd<<<(unsigned)ceil_div(n_rays * n_samples, 256), 256, 0, (cudaStream_t)stream>>>(a);
  SDFB_LAUNCHED("k_render_bwd");
  return 0;
}

extern "C" int sdfb200_render_packed_backward(const float* weights, const float* rgb, const float* normals, const float* starts, const float* ends,
                                              const int64_t* ray_indices, int64_t n_samples_total, int64_t n_rays, const float* bg, int32_t bg_mode,
                                              const float* accumulation, const float* depth, const float* g_rgb, const float* g_depth,
                                              const float* g_normal, const float* g_accumulation, float* g_weights, float* g_rgb_samples,
                                              float* g_normal_samples, float* g_steps, void* stream) {
  SDFB_REQUIRE(n_samples_total >= 0 && n_rays >= 0, "bad sizes");
  if (n_samples_total == 0) return 0;
  SDFB_REQUIRE(weights && ray_indices && g_weights, "NULL pointer");
  SDFB_REQUIRE(bg_mode != SDFB200_BG_LAST_SAMPLE, "background 'last_sample' is not defined for packed samples (renderers.py:76-77)");
  if (g_rgb) SDFB_REQUIRE(rgb != nullptr && bg != nullptr, "g_rgb needs rgb and background");
  if (g_normal) SDFB_REQUIRE(normals != nullptr, "g_normal needs normals");
  if (g_depth) SDFB_REQUIRE(starts != nullptr && ends != nullptr && depth != nullptr && accumulation != nullptr, "g_depth needs starts, ends, depth, accumulation");
  PackedRenderBwdArgs a;
  a.weights = weights; a.rgb = rgb; a.normals = normals; a.starts = starts; a.ends = ends; a.bg = bg; a.ray_indices = ray_indices; a.bg_mode = bg_mode;
  a.N = n_samples_total; a.R = n_rays; a.acc = accumulation; a.depth = depth; a.g_rgb = g_rgb; a.g_depth = g_depth; a.g_normal = g_normal;
  a.g_acc = g_accumulation; a.g_weights = g_weights; a.g_rgb_s = g_rgb_samples; a.g_normal_s = g_normal_samples; a.g_steps = g_steps;
  k_render_packed_bwd<<<(unsigned)ceil_div(n_samples_total, 256), 256, 0, (cudaStream_t)stream>>>(a);
  SDFB_LAUNCHED("k_render_packed_bwd");
  return 0;
}

extern "C" int sdfb200_weights_backward(const float* alphas_or_density, const float* euclid_bins, int32_t from_density, int64_t n_rays,
                                        int32_t n_samples, const float* g_weights, const float* g_transmittance, int32_t g_transmittance_cols,
                                        float* g_in, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(alphas_or_density && g_weights && g_in, "NULL pointer");
  if (from_density) SDFB_REQUIRE(euclid_bins != nullptr, "density mode needs bins");
  const int gt_cols = g_transmittance ? g_transmittance_cols : 0;
  SDFB_REQUIRE(gt_cols == 0 || (gt_cols == 1 && !from_density) || gt_cols == n_samples + (from_density ? 0 : 1),
               "g_transmittance_cols must be 1 (alphas: last column only) or the width of the transmittance output");
  k_weights_bwd<<<(unsigned)ceil_div(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(alphas_or_density, euclid_bins, from_density, n_rays, n_samples,
                                                                                 g_weights, g_transmittance, gt_cols, g_in);
  SDFB_LAUNCHED("k_weights_bwd");
  return 0;
}
