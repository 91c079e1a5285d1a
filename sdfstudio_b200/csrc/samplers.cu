// Per-ray sampler kernels (nerfstudio/model_components/ray_samplers.py).  These are latency-bound scans over
// S <= ~640 samples per ray; the arithmetic follows the reference's op order (fp32, prefix sums accumulated in
// double and rounded per prefix exactly like torch-CPU's cumsum/cumprod) so that searchsorted / sort indices are
// bit-identical to the reference on identical inputs.
#include "common.cuh"

namespace sdfb200 {

// ---- spacing functions (ray_samplers.py:130-247) -----------------------------------------------------------------
__device__ __forceinline__ float spacing_fn(int kind, float x) {
  switch (kind) {
    case SDFB200_SPACING_LINDISP: return __fdiv_rn(1.f, x);
    case SDFB200_SPACING_SQRT: return sqrtf(x);
    case SDFB200_SPACING_LOG: return logf(x);
    case SDFB200_SPACING_PIECEWISE: return x < 1.f ? __fdiv_rn(x, 2.f) : __fsub_rn(1.f, __fdiv_rn(1.f, __fmul_rn(2.f, x)));
    default: return x;
  }
}
__device__ __forceinline__ float spacing_fn_inv(int kind, float x) {
  switch (kind) {
    case SDFB200_SPACING_LINDISP: return __fdiv_rn(1.f, x);
    case SDFB200_SPACING_SQRT: return __fmul_rn(x, x);
    case SDFB200_SPACING_LOG: return expf(x);
    case SDFB200_SPACING_PIECEWISE: return x < 0.5f ? __fmul_rn(2.f, x) : __fdiv_rn(1.f, __fsub_rn(2.f, __fmul_rn(2.f, x)));
    default: return x;
  }
}
// spacing_to_euclidean_fn = spacing_fn_inv(x * s_far + (1 - x) * s_near)   (:115-116)
__device__ __forceinline__ float to_euclid(int kind, float x, float s_near, float s_far) {
  if (kind == SDFB200_SPACING_IDENTITY) return x;
  return spacing_fn_inv(kind, __fadd_rn(__fmul_rn(x, s_far), __fmul_rn(__fsub_rn(1.f, x), s_near)));
}

__global__ void k_spaced_bins(const float* __restrict__ nears, const float* __restrict__ fars, const float* __restrict__ base,
                              const float* __restrict__ jitter, int jitter_per_bin, int64_t R, int S, int kind, float* __restrict__ sp,
                              float* __restrict__ eu) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int nb = S + 1;
  if (idx >= R * nb) return;
  const int64_t r = idx / nb;
  const int j = (int)(idx - r * nb);
  float b = base[j];
  if (jitter != nullptr) {
    // :105-113 stratified jitter
    const float lower = j == 0 ? base[0] : __fdiv_rn(__fadd_rn(base[j], base[j - 1]), 2.0f);
    const float upper = j == S ? base[S] : __fdiv_rn(__fadd_rn(base[j + 1], base[j]), 2.0f);
    const float t = jitter_per_bin ? jitter[r * nb + j] : jitter[r];
    b = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), t));
  }
  sp[idx] = b;
  eu[idx] = to_euclid(kind, b, spacing_fn(kind, nears[r]), spacing_fn(kind, fars[r]));
}

__global__ void k_bins_to_euclid(const float* __restrict__ sp, const float* __restrict__ nears, const float* __restrict__ fars, int64_t R, int nb,
                                 int kind, float* __restrict__ eu) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= R * nb) return;
  const int64_t r = idx / nb;
  eu[idx] = to_euclid(kind, sp[idx], spacing_fn(kind, nears[r]), spacing_fn(kind, fars[r]));
}

// ---- PDFSampler (:275-370).  One thread per ray; u is ascending, so searchsorted(side="right") is a merge walk over
// the incrementally-built cdf (no per-ray scratch). ---------------------------------------------------------------
__global__ void __launch_bounds__(128) k_pdf_sample(const float* __restrict__ weights, const float* __restrict__ ebins, const float* __restrict__ ugrid,
                                                    const float* __restrict__ jitter, int jitter_per_bin, int64_t R, int s_in, int s_out,
                                                    float hist_pad, float eps, int include_original, float* __restrict__ out,
                                                    int64_t* __restrict__ inds_out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* w = weights + r * s_in;
  const float* eb = ebins + r * (s_in + 1);
  const int nb = s_out + 1;
  // weights_sum (torch.sum: order unspecified in the reference; accumulated in double here)
  double acc = 0.0;
  for (int i = 0; i < s_in; ++i) acc += (double)__fadd_rn(w[i], hist_pad);
  float w_sum = (float)acc;
  const float padding = fmaxf(__fsub_rn(eps, w_sum), 0.f);
  const float pad_each = __fdiv_rn(padding, (float)s_in);
  w_sum = __fadd_rn(w_sum, padding);

  // walk state: `k` = number of cdf entries <= u so far (cdf has s_in+1 entries, cdf[0] = 0)
  int k = 1;                       // cdf[0] = 0 <= u always
  double run = 0.0;                // double prefix of pdf
  float c_lo = 0.f;                // cdf[k-1]
  float c_hi;                      // cdf[k] (valid while k <= s_in)
  {
    const float pdf0 = __fdiv_rn(__fadd_rn(__fadd_rn(w[0], hist_pad), pad_each), w_sum);
    run = (double)pdf0;
    c_hi = fminf(1.0f, (float)run);
  }
  // optional merge with the original bins (include_original): both sequences ascending
  int eo = 0;                      // next original bin to emit
  int64_t o = 0;
  float* dst = out + r * (include_original ? (int64_t)(s_in + 1 + nb) : (int64_t)nb);
  for (int j = 0; j < nb; ++j) {
    float u = ugrid[j];
    if (jitter != nullptr) u = __fadd_rn(u, __fdiv_rn(jitter_per_bin ? jitter[r * nb + j] : jitter[r], (float)nb));
    while (k <= s_in && c_hi <= u) {
      c_lo = c_hi;
      ++k;
      if (k <= s_in) {
        const float pdfk = __fdiv_rn(__fadd_rn(__fadd_rn(w[k - 1], hist_pad), pad_each), w_sum);
        run += (double)pdfk;
        c_hi = fminf(1.0f, (float)run);
      }
    }
    // inds = k; below = clamp(k-1), above = clamp(k) into [0, s_in]
    const int below = k - 1;                         // k >= 1  ->  0..s_in
    const int above = k <= s_in ? k : s_in;
    const float cdf_g0 = c_lo;
    const float cdf_g1 = k <= s_in ? c_hi : c_lo;
    const float b0 = eb[below], b1 = eb[above];
    float t = __fdiv_rn(__fsub_rn(u, cdf_g0), __fsub_rn(cdf_g1, cdf_g0));
    if (isnan(t)) t = 0.f;                           // nan_to_num(nan=0) then clip(0,1) (inf -> 1, -inf -> 0)
    t = fminf(fmaxf(t, 0.f), 1.f);
    const float nbin = __fadd_rn(b0, __fmul_rn(t, __fsub_rn(b1, b0)));
    if (inds_out) inds_out[r * nb + j] = k;
    if (include_original) {
      while (eo <= s_in && eb[eo] <= nbin) dst[o++] = eb[eo++];
      dst[o++] = nbin;
    } else {
      dst[j] = nbin;
    }
  }
  if (include_original)
    while (eo <= s_in) dst[o++] = eb[eo++];
}

// ---- merge_ray_samples (:758-788): stable two-way merge of the starts, ends = max of the last edges ----------------
__global__ void __launch_bounds__(128) k_merge_bins(const float* __restrict__ a, const float* __restrict__ b, int64_t R, int sa, int sb,
                                                    float* __restrict__ merged, int64_t* __restrict__ sidx) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* pa = a + r * (sa + 1);
  const float* pb = b + r * (sb + 1);
  float* m = merged + r * (sa + sb + 1);
  int64_t* si = sidx ? sidx + r * (sa + sb) : nullptr;
  int i = 0, j = 0;
  for (int o = 0; o < sa + sb; ++o) {
    const bool take_a = j >= sb || (i < sa && pa[i] <= pb[j]);
    if (take_a) { m[o] = pa[i]; if (si) si[o] = i; ++i; }
    else { m[o] = pb[j]; if (si) si[o] = sa + j; ++j; }
  }
  m[sa + sb] = fmaxf(pa[sa], pb[sb]);
}

__global__ void k_merge_gather(const float* __restrict__ a, const float* __restrict__ b, const int64_t* __restrict__ sidx, int64_t R, int sa, int sb,
                               float* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int s = sa + sb;
  if (idx >= R * s) return;
  const int64_t r = idx / s;
  const int64_t k = sidx[idx];
  out[idx] = k < sa ? a[r * sa + k] : b[r * sb + (k - sa)];
}

// ---- NeuS up-sampling weights (:909-944 + rays.py:194-210 + zero pad :885) ---------------------------------------
__global__ void __launch_bounds__(128) k_neus_weights(const float* __restrict__ eu, const float* __restrict__ sdf, int64_t R, int S, float inv_s,
                                                      float* __restrict__ weights) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* e = eu + r * (S + 1);
  const float* sd = sdf + r * S;
  float* w = weights + r * S;
  double T = 1.0;           // cumprod accumulated in double (torch-CPU semantics), rounded per prefix
  float prev_cos = 0.f;
  for (int i = 0; i < S - 1; ++i) {
    const float prev_sdf = sd[i], next_sdf = sd[i + 1];
    const float delta = __fsub_rn(e[i + 1], e[i]);
    const float mid = __fmul_rn(__fadd_rn(prev_sdf, next_sdf), 0.5f);
    const float cosv = __fdiv_rn(__fsub_rn(next_sdf, prev_sdf), __fadd_rn(delta, 1e-5f));
    float c = fminf(prev_cos, cosv);
    prev_cos = cosv;
    c = fminf(fmaxf(c, -1e3f), 0.0f);
    const float half = __fmul_rn(__fmul_rn(c, delta), 0.5f);
    const float prev_cdf = sigmoidf_(__fmul_rn(__fsub_rn(mid, half), inv_s));
    const float next_cdf = sigmoidf_(__fmul_rn(__fadd_rn(mid, half), inv_s));
    const float alpha = __fdiv_rn(__fadd_rn(__fsub_rn(prev_cdf, next_cdf), 1e-5f), __fadd_rn(prev_cdf, 1e-5f));
    w[i] = __fmul_rn(alpha, (float)T);
    T *= (double)neus_trans_factor(alpha);
  }
  w[S - 1] = 0.f;
}

// ---- VolSDF error-bounded sampler ---------------------------------------------------------------------------------
__device__ __forceinline__ float laplace_density(float sdf, float beta) {
  // sdf_field.py:65-66: alpha * (0.5 + 0.5 * sign(sdf) * expm1(-|sdf| / beta)), alpha = 1/beta
  const float al = __fdiv_rn(1.0f, beta);
  const float sg = sdf > 0.f ? 1.f : (sdf < 0.f ? -1.f : 0.f);
  return __fmul_rn(al, __fadd_rn(0.5f, __fmul_rn(__fmul_rn(0.5f, sg), expm1f(__fdiv_rn(-fabsf(sdf), beta)))));
}

__global__ void k_volsdf_init_beta(const float* __restrict__ eu, int64_t R, int S, float eps, float* __restrict__ beta) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* e = eu + r * (S + 1);
  double acc = 0.0;
  for (int i = 0; i < S; ++i) {
    const float d = __fsub_rn(e[i + 1], e[i]);
    acc += (double)__fmul_rn(d, d);
  }
  const float coef = __fdiv_rn(1.0f, __fmul_rn(4.0f, logf(__fadd_rn(eps, 1.0f))));
  beta[r] = sqrtf(__fmul_rn(coef, (float)acc));
}

// d* of section i (get_dstar :704-726); i in [0, S-2], the last section repeats S-2
__device__ __forceinline__ float volsdf_dstar(const float* e, const float* sd, int i) {
  const float a = __fsub_rn(e[i + 1], e[i]);
  const float d0 = sd[i], d1 = sd[i + 1];
  const float b = fabsf(d0), c = fabsf(d1);
  const float a2 = __fmul_rn(a, a), b2 = __fmul_rn(b, b), c2 = __fmul_rn(c, c);
  const bool first = __fadd_rn(a2, b2) <= c2;
  const bool second = __fadd_rn(a2, c2) <= b2;
  float ds = 0.f;
  if (first) ds = b;
  if (second) ds = c;
  if (!first && !second && (__fsub_rn(__fadd_rn(b, c), a) > 0.f)) {
    const float s = __fdiv_rn(__fadd_rn(__fadd_rn(a, b), c), 2.0f);
    const float area = __fmul_rn(__fmul_rn(__fmul_rn(s, __fsub_rn(s, a)), __fsub_rn(s, b)), __fsub_rn(s, c));
    ds = __fdiv_rn(__fmul_rn(2.0f, sqrtf(area)), a);
  }
  const float sg0 = d0 > 0.f ? 1.f : (d0 < 0.f ? -1.f : 0.f), sg1 = d1 > 0.f ? 1.f : (d1 < 0.f ? -1.f : 0.f);
  return (sg1 * sg0 == 1.f) ? ds : 0.f;
}

// ONE WARP PER RAY.  get_error_bound (:740-756) at one beta:  max_i (clamp(exp(E_i), 1e6) - 1) * exp(-I_i) with the inclusive prefix
// sum E_i of the section errors and the exclusive prefix sum I_i of delta * sigma -- both as warp scans in double carried across
// 32-sample rows (not the sequential order of torch.cumsum: agreement at the 1e-7 level, like the compositing kernels).  Per-sample
// quantities that do not depend on beta (delta, d*, sdf) are cached in shared memory once per ray.
// torch.clamp and .max(-1) propagate NaN: fminf / fmaxf would drop it, so it is carried explicitly -- a NaN bound leaves beta untouched,
// as in the reference.  The NaN comes through I: a NaN sdf sample (or bin) makes delta * sigma NaN from that sample on.  d* itself is
// not NaN for finite inputs: the Heron branch runs only when neither squared test fires and b + c - a > 0, and there the rounded area is
// not negative (tests/test_oracle_samplers_train.py searches near-degenerate triangles of every orientation and magnitude for one).  So E
// is NaN only where I is NaN too, and the NaN-keeping clamp of exp(E) below and the plain fminf of the err weights in k_volsdf_step give
// the same results.
constexpr int kVolsdfMaxS = 1000;   // 4 rays x 3 x S floats of dynamic shared memory stay under the 48 KB default
__device__ float volsdf_error_bound_warp(const float* delta_s, const float* dstar_s, const float* sdf_s, int S, float beta, int lane) {
  double carryE = 0.0, carryI = 0.0;
  float best = -INFINITY;
  bool saw_nan = false;
  const float b2 = __fmul_rn(4.0f, __fmul_rn(beta, beta));
  for (int s0 = 0; s0 < S; s0 += 32) {
    const int i = s0 + lane;
    const bool on = i < S;
    const float delta = on ? delta_s[i] : 0.f;
    const float err_sec = on ? __fdiv_rn(__fmul_rn(expf(__fdiv_rn(-dstar_s[i], beta)), __fmul_rn(delta, delta)), b2) : 0.f;
    const float dd = on ? __fmul_rn(delta, laplace_density(sdf_s[i], beta)) : 0.f;
    const double einc = warp_scan_incl((double)err_sec, lane);
    const double iinc = warp_scan_incl((double)dd, lane);
    const float E = (float)(carryE + einc), I = (float)(carryI + iinc - (double)dd);
    const float ef = expf(E);
    const float bound = __fmul_rn(__fsub_rn(ef != ef ? ef : fminf(ef, 1.0e6f), 1.0f), expf(-I));
    if (on) {
      if (bound != bound) saw_nan = true;
      else best = fmaxf(best, bound);
    }
    carryE += __shfl_sync(0xffffffffu, einc, 31);
    carryI += __shfl_sync(0xffffffffu, iinc, 31);
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, d));
  saw_nan = __any_sync(0xffffffffu, saw_nan);
  return saw_nan ? __int_as_float(0x7fc00000) : best;
}

__global__ void __launch_bounds__(128) k_volsdf_step(const float* __restrict__ eu, const float* __restrict__ sdf, const float* __restrict__ beta0p,
                                                     float* __restrict__ beta_io, int64_t R, int S, float eps, int beta_iters,
                                                     float* __restrict__ weights, float* __restrict__ err_weights) {
  extern __shared__ float vs_smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + wib;
  if (r >= R) return;                                     // whole warp
  float* delta_s = vs_smem + (size_t)wib * 3 * S;
  float* dstar_s = delta_s + S;
  float* sdf_s = dstar_s + S;
  const float* e = eu + r * (S + 1);
  const float* sd = sdf + r * S;
  for (int i = lane; i < S; i += 32) {
    delta_s[i] = __fsub_rn(e[i + 1], e[i]);
    dstar_s[i] = volsdf_dstar(e, sd, i < S - 1 ? i : S - 2);
    sdf_s[i] = sd[i];
  }
  __syncwarp();
  const float beta0 = *beta0p;
  float beta = beta_io[r];
  // get_updated_beta (:728-738)
  if (volsdf_error_bound_warp(delta_s, dstar_s, sdf_s, S, beta0, lane) <= eps) beta = beta0;
  float bmin = beta0, bmax = beta;
  for (int j = 0; j < beta_iters; ++j) {
    const float mid = __fdiv_rn(__fadd_rn(bmin, bmax), 2.0f);
    const float err = volsdf_error_bound_warp(delta_s, dstar_s, sdf_s, S, mid, lane);
    if (err <= eps) bmax = mid;
    if (err > eps) bmin = mid;
  }
  beta = bmax;
  if (lane == 0) beta_io[r] = beta;
  // density weights + transmittance (rays.py:167-192) and the error-bound pdf (:664-671)
  double carryE = 0.0, carryI = 0.0;
  const float b2 = __fmul_rn(4.0f, __fmul_rn(beta, beta));
  for (int s0 = 0; s0 < S; s0 += 32) {
    const int i = s0 + lane;
    const bool on = i < S;
    const float delta = on ? delta_s[i] : 0.f;
    const float dd = on ? __fmul_rn(delta, laplace_density(sdf_s[i], beta)) : 0.f;
    const float err_sec = on ? __fdiv_rn(__fmul_rn(expf(__fdiv_rn(-dstar_s[i], beta)), __fmul_rn(delta, delta)), b2) : 0.f;
    const double einc = warp_scan_incl((double)err_sec, lane);
    const double iinc = warp_scan_incl((double)dd, lane);
    const float trans = expf(-(float)(carryI + iinc - (double)dd));
    if (on) {
      weights[r * S + i] = __fmul_rn(__fsub_rn(1.0f, expf(-dd)), trans);
      err_weights[r * S + i] = __fmul_rn(__fsub_rn(fminf(expf((float)(carryE + einc)), 1.0e6f), 1.0f), trans);
    }
    carryE += __shfl_sync(0xffffffffu, einc, 31);
    carryI += __shfl_sync(0xffffffffu, iinc, 31);
  }
}

// ---- UniSurf surface interval (:1027-1077) ------------------------------------------------------------------------
__global__ void k_unisurf_interval(const float* __restrict__ eu, const float* __restrict__ sdf, const float* __restrict__ nears,
                                   const float* __restrict__ fars, int64_t R, int S, float delta, float* __restrict__ z_out, uint8_t* __restrict__ hit,
                                   float* __restrict__ nn, float* __restrict__ nf) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float* e = eu + r * (S + 1);
  const float* sd = sdf + r * S;
  int idx = -1;
  for (int i = 0; i < S - 1; ++i) {
    if (__fmul_rn(sd[i], sd[i + 1]) < 0.f) { idx = i; break; }
  }
  const float near = nears[r], far = fars[r];
  bool ok = idx >= 0 && sd[idx] > 0.f;
  float z = NAN, n2 = near, f2 = far;
  if (ok) {
    const int i2 = idx + 1 < S - 1 ? idx + 1 : S - 1;
    const float d_low = e[idx], v_low = sd[idx], d_high = e[i2], v_high = sd[i2];
    z = __fdiv_rn(__fsub_rn(__fmul_rn(v_low, d_high), __fmul_rn(v_high, d_low)), __fsub_rn(v_low, v_high));
    const float dist = __fsub_rn(far, near);
    n2 = fmaxf(__fsub_rn(z, __fmul_rn(dist, delta)), near);
    f2 = fminf(__fadd_rn(z, __fmul_rn(dist, delta)), far);
  }
  z_out[r] = z;
  hit[r] = ok ? 1 : 0;
  nn[r] = n2;
  nf[r] = f2;
}

}  // namespace sdfb200

using namespace sdfb200;

#define ST(s) ((cudaStream_t)(s))

extern "C" int sdfb200_spaced_bins(const float* nears, const float* fars, const float* base_bins, const float* jitter, int32_t jitter_per_bin,
                                   int64_t n_rays, int32_t n_samples, int32_t spacing, float* spacing_bins, float* euclid_bins, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(nears && fars && base_bins && spacing_bins && euclid_bins, "NULL pointer");
  SDFB_REQUIRE(spacing >= 0 && spacing <= SDFB200_SPACING_IDENTITY, "unknown spacing");
  const int64_t tot = n_rays * (n_samples + 1);
  k_spaced_bins<<<(unsigned)ceil_div(tot, 256), 256, 0, ST(stream)>>>(nears, fars, base_bins, jitter, jitter_per_bin, n_rays, n_samples, spacing,
                                                                      spacing_bins, euclid_bins);
  SDFB_LAUNCHED("k_spaced_bins");
  return 0;
}

extern "C" int sdfb200_bins_to_euclid(const float* spacing_bins, const float* nears, const float* fars, int64_t n_rays, int32_t n_bins,
                                      int32_t spacing, float* euclid_bins, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_bins >= 1, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(spacing_bins && nears && fars && euclid_bins, "NULL pointer");
  SDFB_REQUIRE(spacing >= 0 && spacing <= SDFB200_SPACING_IDENTITY, "unknown spacing");
  k_bins_to_euclid<<<(unsigned)ceil_div(n_rays * n_bins, 256), 256, 0, ST(stream)>>>(spacing_bins, nears, fars, n_rays, n_bins, spacing, euclid_bins);
  SDFB_LAUNCHED("k_bins_to_euclid");
  return 0;
}

extern "C" int sdfb200_pdf_sample(const float* weights, const float* existing_bins, const float* u, const float* jitter, int32_t jitter_per_bin,
                                  int64_t n_rays, int32_t s_in, int32_t s_out, float histogram_padding, float eps, int32_t include_original,
                                  float* new_bins, int64_t* inds, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && s_in >= 1 && s_out >= 1, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(weights && existing_bins && u && new_bins, "NULL pointer");
  k_pdf_sample<<<(unsigned)ceil_div(n_rays, 128), 128, 0, ST(stream)>>>(weights, existing_bins, u, jitter, jitter_per_bin, n_rays, s_in, s_out,
                                                                        histogram_padding, eps, include_original, new_bins, inds);
  SDFB_LAUNCHED("k_pdf_sample");
  return 0;
}

extern "C" int sdfb200_merge_bins(const float* bins_a, const float* bins_b, int64_t n_rays, int32_t sa, int32_t sb, float* merged,
                                  int64_t* sorted_index, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && sa >= 1 && sb >= 1, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(bins_a && bins_b && merged, "NULL pointer");
  k_merge_bins<<<(unsigned)ceil_div(n_rays, 128), 128, 0, ST(stream)>>>(bins_a, bins_b, n_rays, sa, sb, merged, sorted_index);
  SDFB_LAUNCHED("k_merge_bins");
  return 0;
}

extern "C" int sdfb200_merge_gather(const float* a, const float* b, const int64_t* sorted_index, int64_t n_rays, int32_t sa, int32_t sb, float* out,
                                    void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && sa >= 1 && sb >= 1, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(a && b && sorted_index && out, "NULL pointer");
  k_merge_gather<<<(unsigned)ceil_div(n_rays * (sa + sb), 256), 256, 0, ST(stream)>>>(a, b, sorted_index, n_rays, sa, sb, out);
  SDFB_LAUNCHED("k_merge_gather");
  return 0;
}

extern "C" int sdfb200_neus_upsample_weights(const float* euclid_bins, const float* sdf, int64_t n_rays, int32_t n_samples, float inv_s,
                                             float* weights, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 2, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(euclid_bins && sdf && weights, "NULL pointer");
  k_neus_weights<<<(unsigned)ceil_div(n_rays, 128), 128, 0, ST(stream)>>>(euclid_bins, sdf, n_rays, n_samples, inv_s, weights);
  SDFB_LAUNCHED("k_neus_weights");
  return 0;
}

extern "C" int sdfb200_volsdf_init_beta(const float* euclid_bins, int64_t n_rays, int32_t n_samples, float eps, float* beta, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 1, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(euclid_bins && beta, "NULL pointer");
  k_volsdf_init_beta<<<(unsigned)ceil_div(n_rays, 128), 128, 0, ST(stream)>>>(euclid_bins, n_rays, n_samples, eps, beta);
  SDFB_LAUNCHED("k_volsdf_init_beta");
  return 0;
}

extern "C" int sdfb200_volsdf_step(const float* euclid_bins, const float* sdf, const float* beta0, float* beta, int64_t n_rays, int32_t n_samples,
                                   float eps, int32_t beta_iters, float* weights, float* err_weights, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 2 && beta_iters >= 0, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(euclid_bins && sdf && beta0 && beta && weights && err_weights, "NULL pointer");
  SDFB_REQUIRE(n_samples <= kVolsdfMaxS, "volsdf_step: n_samples > 1000");
  // one warp per ray, 4 rays per block; per-ray cache of delta / d* / sdf in shared memory
  const size_t smem = (size_t)4 * 3 * n_samples * sizeof(float);
  k_volsdf_step<<<(unsigned)ceil_div(n_rays, 4), 128, smem, ST(stream)>>>(euclid_bins, sdf, beta0, beta, n_rays, n_samples, eps, beta_iters, weights,
                                                                          err_weights);
  SDFB_LAUNCHED("k_volsdf_step");
  return 0;
}

extern "C" int sdfb200_unisurf_interval(const float* euclid_bins, const float* sdf, const float* nears, const float* fars, int64_t n_rays,
                                        int32_t n_samples, float delta, float* z, uint8_t* hit, float* new_nears, float* new_fars, void* stream) {
  SDFB_REQUIRE(n_rays >= 0 && n_samples >= 2, "bad sizes");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(euclid_bins && sdf && nears && fars && z && hit && new_nears && new_fars, "NULL pointer");
  k_unisurf_interval<<<(unsigned)ceil_div(n_rays, 128), 128, 0, ST(stream)>>>(euclid_bins, sdf, nears, fars, n_rays, n_samples, delta, z, hit,
                                                                              new_nears, new_fars);
  SDFB_LAUNCHED("k_unisurf_interval");
  return 0;
}
