// Interlevel (proposal) losses of nerfstudio/model_components/losses.py: the mip-NeRF 360 outer-measure form (:38-112) and the Zip-NeRF
// blurred-histogram form (:116-172), each with d loss / d proposal weights written by the same launch.
//
// One warp per ray.  A ray is a few hundred floats and every step after the loads is a dependent scan or search, so a CTA per ray would
// leave most of its threads idle between barriers; a warp keeps the ray's arrays in its own slice of shared memory and synchronises
// with __syncwarp only.  A CTA holds up to four such warps (fewer when the sample counts grow, so that the slices stay under 48 KiB).
// Prefix sums are accumulated in double and rounded to fp32 per prefix, like torch-CPU's cumsum, as in samplers.cu.
#include "common.cuh"

namespace sdfb200 {

constexpr int kInterlevelMaxSamples = 1024;
constexpr int kInterlevelMaxWarps = 4;
constexpr size_t kInterlevelSmemBudget = 48 * 1024;

constexpr unsigned kFullWarp = 0xffffffffu;

// butterfly sum: every lane ends with the same value, added in the same order on every call
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(kFullWarp, v, d);
  return v;
}

// torch.searchsorted(a[0..n), v, side="right"): the number of entries <= v
__device__ __forceinline__ int count_le(const float* a, int n, float v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] <= v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// torch.clip(x, min=0): unlike fmaxf, a NaN stays a NaN (a fine bin of zero width must poison its ray as it does in the reference)
__device__ __forceinline__ float clip0(float x) { return x < 0.f ? 0.f : x; }

// nan_to_num(x, 0) followed by clip(0, 1) (losses.py:164): NaN -> 0, +inf -> 1, -inf -> 0
__device__ __forceinline__ float unit_clip(float t) {
  if (isnan(t)) t = 0.f;
  return fminf(fmaxf(t, 0.f), 1.f);
}

// shared-memory floats of one warp's slice
__host__ __device__ inline size_t zip_slice_floats(int sf, int sp) { return 3 * (size_t)(2 * sf + 2) + (size_t)(sp + 1); }
__host__ __device__ inline size_t outer_slice_floats(int sf, int sp) {
  // prefix of g [sf+1] doubles | cp, cy [sp+1] | c [sf+1] | lo, hi [sf]; an even count, so that every slice's doubles are 8-byte aligned
  const size_t n = 2 * (size_t)(sf + 1) + 2 * (size_t)(sp + 1) + (size_t)(sf + 1) + 2 * (size_t)sf;
  return (n + 1) & ~(size_t)1;
}

// ---- Zip-NeRF form (blur_stepfun + interlevel_loss_zip, :116-172) -------------------------------------------------------------------
// The 2(Sf+1) knots c - r and c + r are two ascending sequences: every knot finds its place in the sorted order with one binary search
// in the other sequence (a merge; ties between a c_i - r and a c_j + r put the former first, and the interval between them has zero
// width, so the blurred function does not depend on it).  Then one pass over the knots in tiles of 32 carries the three dependent
// prefix sums (slope, blurred value, its integral), and the proposal edges look the integral up.
__global__ void __launch_bounds__(32 * kInterlevelMaxWarps)
k_interlevel_zip(const float* __restrict__ c_all, const float* __restrict__ w_all, int sf, const float* __restrict__ cp_all,
                 const float* __restrict__ wp_all, int sp, int64_t R, float r, float* __restrict__ loss_per_ray, float* __restrict__ grad_wp) {
  extern __shared__ __align__(8) float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ray = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (ray >= R) return;
  const int nk = 2 * sf + 2;                       // knots
  float* x = smem + warp * zip_slice_floats(sf, sp);   // sorted knots [nk]
  float* slope = x + nk;                           // slope change at each sorted knot [nk] (the last one is not used)
  float* ycum = slope + nk;                        // integral of the blurred function at each knot [nk]; first holds the fine edges
  float* bins = ycum + nk;                         // that integral at the proposal edges [sp+1]
  const float* c = c_all + ray * (sf + 1);
  const float* w = w_all + ray * sf;
  const float* cp = cp_all + ray * (sp + 1);
  const float* wp = wp_all + ray * sp;

  float* cs = ycum;
  for (int i = lane; i <= sf; i += 32) cs[i] = c[i];
  __syncwarp();
  const float two_r = __fmul_rn(2.f, r);
  for (int i = lane; i <= sf; i += 32) {
    // y_1 of blur_stepfun: (w_n[i] - w_n[i-1]) / 2r with w_n = w / (c[1:] - c[:-1]) and zeros past both ends
    const float wn_hi = i < sf ? __fdiv_rn(w[i], __fsub_rn(cs[i + 1], cs[i])) : 0.f;
    const float wn_lo = i > 0 ? __fdiv_rn(w[i - 1], __fsub_rn(cs[i], cs[i - 1])) : 0.f;
    const float y1 = __fdiv_rn(__fsub_rn(wn_hi, wn_lo), two_r);
    const float a = __fsub_rn(cs[i], r), b = __fadd_rn(cs[i], r);
    // place of a = c_i - r: after the i knots c_k - r before it and the knots c_j + r < a; of b = c_i + r: after those <= b
    int lo = 0, hi = i;                            // c_j + r < c_i - r needs j < i
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (__fadd_rn(cs[mid], r) < a) lo = mid + 1; else hi = mid;
    }
    const int pa = i + lo;
    lo = i; hi = sf + 1;                           // c_j - r <= c_i + r holds for every j <= i
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (__fsub_rn(cs[mid], r) <= b) lo = mid + 1; else hi = mid;
    }
    const int pb = i + lo;
    x[pa] = a; slope[pa] = y1;
    x[pb] = b; slope[pb] = -y1;
  }
  __syncwarp();

  // over the intervals k = 0 .. nk-2 between sorted knots: inner = cumsum(slope), y_r = [0, cumsum(dx * inner)] clipped at 0,
  // y_cum = [0, cumsum((y_r[k+1] + y_r[k]) / 2 * dx)]
  double carry_inner = 0.0, carry_yr = 0.0, carry_cum = 0.0;
  float prev_yr = 0.f;                             // clipped y_r at the tile's first knot
  for (int base = 0; base < nk - 1; base += 32) {
    const int k = base + lane;
    const bool live = k < nk - 1;
    const float dx = live ? __fsub_rn(x[k + 1], x[k]) : 0.f;
    const double inner_d = carry_inner + warp_scan_incl(live ? (double)slope[k] : 0.0, lane);
    const float inner = (float)inner_d;
    const double yr_d = carry_yr + warp_scan_incl(live ? (double)__fmul_rn(dx, inner) : 0.0, lane);
    const float yr_hi = clip0((float)yr_d);   // y_r[k+1]
    float yr_lo = __shfl_up_sync(kFullWarp, yr_hi, 1);
    if (lane == 0) yr_lo = prev_yr;
    const float area = __fmul_rn(__fmul_rn(__fadd_rn(yr_hi, yr_lo), 0.5f), dx);
    const double cum_d = carry_cum + warp_scan_incl(live ? (double)area : 0.0, lane);
    if (live) ycum[k + 1] = (float)cum_d;
    // the running sums stay in double across tiles: only what is stored or multiplied is rounded to fp32, as in one long cumsum
    carry_inner = __shfl_sync(kFullWarp, inner_d, 31);
    carry_yr = __shfl_sync(kFullWarp, yr_d, 31);
    carry_cum = __shfl_sync(kFullWarp, cum_d, 31);
    prev_yr = __shfl_sync(kFullWarp, yr_hi, 31);
  }
  if (lane == 0) ycum[0] = 0.f;
  __syncwarp();

  // resample the integral at the proposal edges (:156-165)
  for (int j = lane; j <= sp; j += 32) {
    const float v = cp[j];
    const int inds = count_le(x, nk, v);
    const int below = min(max(inds - 1, 0), nk - 1), above = min(inds, nk - 1);
    const float t = unit_clip(__fdiv_rn(__fsub_rn(v, x[below]), __fsub_rn(x[above], x[below])));
    bins[j] = __fadd_rn(ycum[below], __fmul_rn(t, __fsub_rn(ycum[above], ycum[below])));
  }
  __syncwarp();

  double sum = 0.0;
  for (int j = lane; j < sp; j += 32) {
    const float w_gt = __fsub_rn(bins[j + 1], bins[j]);
    const float p = wp[j];
    const float m = clip0(__fsub_rn(w_gt, p));
    const float den = __fadd_rn(p, 1e-5f);
    const float q = __fdiv_rn(m, den);
    sum += (double)__fmul_rn(m, q);                // m^2 / (wp + eps)
    // d/d wp of max(w_gt - wp, 0)^2 / (wp + eps): -2 m / (wp + eps) - m^2 / (wp + eps)^2
    if (grad_wp) grad_wp[ray * sp + j] = -(2.f * q + q * q);
  }
  sum = warp_sum(sum);
  if (lane == 0) loss_per_ray[ray] = (float)sum;
}

// ---- mip-NeRF 360 form (outer + lossfun_outer, :38-87) ------------------------------------------------------------------------------
// w_outer_i = cy[hi_i + 1] - cy[lo_i] with cy = [0, cumsum(wp)], so d w_outer_i / d wp_j = [j <= hi_i] - [j < lo_i].  lo and hi do not
// decrease along the ray: the fine intervals with hi_i >= j are those from some first index on, and likewise lo_i > j.  With
// G(n) = sum of g_i over i < n (g_i = d element_i / d w_outer_i), d / d wp_j = G(first i with lo_i > j) - G(first i with hi_i >= j):
// two binary searches and two reads per proposal sample, no atomics, the same bits on every call.
__global__ void __launch_bounds__(32 * kInterlevelMaxWarps)
k_interlevel_outer(const float* __restrict__ c_all, const float* __restrict__ w_all, int sf, const float* __restrict__ cp_all,
                   const float* __restrict__ wp_all, int sp, int64_t R, float* __restrict__ loss_per_ray, float* __restrict__ grad_wp) {
  extern __shared__ __align__(8) float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ray = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (ray >= R) return;
  float* slice = smem + warp * outer_slice_floats(sf, sp);   // an even number of floats: every slice starts 8-byte aligned
  double* gsum = reinterpret_cast<double*>(slice);           // G [sf+1]
  float* cps = slice + 2 * (sf + 1);                         // proposal edges [sp+1]
  float* cy = cps + (sp + 1);                                // [0, cumsum(wp)] [sp+1]
  float* cs = cy + (sp + 1);                                 // fine edges [sf+1]
  int* lo_s = reinterpret_cast<int*>(cs + (sf + 1));         // [sf]
  int* hi_s = lo_s + sf;                                     // [sf]
  const float* c = c_all + ray * (sf + 1);
  const float* w = w_all + ray * sf;
  const float* cp = cp_all + ray * (sp + 1);
  const float* wp = wp_all + ray * sp;

  for (int i = lane; i <= sf; i += 32) cs[i] = c[i];
  for (int j = lane; j <= sp; j += 32) cps[j] = cp[j];
  double carry = 0.0;
  for (int base = 0; base < sp; base += 32) {
    const int j = base + lane;
    const double s = carry + warp_scan_incl(j < sp ? (double)wp[j] : 0.0, lane);
    if (j < sp) cy[j + 1] = (float)s;
    carry = __shfl_sync(kFullWarp, s, 31);
  }
  if (lane == 0) { cy[0] = 0.f; gsum[0] = 0.0; }
  __syncwarp();

  double sum = 0.0;
  carry = 0.0;
  for (int base = 0; base < sf; base += 32) {
    const int i = base + lane;
    double g = 0.0;
    if (i < sf) {
      const int lo = min(max(count_le(cps, sp, cs[i]) - 1, 0), sp - 1);          // starts = cp[:-1]
      const int hi = min(count_le(cps + 1, sp, cs[i + 1]), sp - 1);              // ends = cp[1:]
      lo_s[i] = lo; hi_s[i] = hi;
      const float wi = w[i];
      const float m = clip0(__fsub_rn(wi, __fsub_rn(cy[hi + 1], cy[lo])));
      const float q = __fdiv_rn(m, __fadd_rn(wi, 1e-7f));
      sum += (double)__fmul_rn(m, q);              // m^2 / (w + eps)
      g = -2.0 * (double)q;
    }
    const double s = carry + warp_scan_incl(g, lane);
    if (i < sf) gsum[i + 1] = s;
    carry = __shfl_sync(kFullWarp, s, 31);
  }
  sum = warp_sum(sum);
  if (lane == 0) loss_per_ray[ray] = (float)sum;
  if (grad_wp == nullptr) return;
  __syncwarp();
  for (int j = lane; j < sp; j += 32) {
    int a = 0, b = sf;                             // first i with hi_i >= j
    while (a < b) {
      const int mid = (a + b) >> 1;
      if (hi_s[mid] >= j) b = mid; else a = mid + 1;
    }
    const int first_hi = a;
    a = 0; b = sf;                                 // first i with lo_i > j
    while (a < b) {
      const int mid = (a + b) >> 1;
      if (lo_s[mid] > j) b = mid; else a = mid + 1;
    }
    grad_wp[ray * sp + j] = (float)(gsum[a] - gsum[first_hi]);
  }
}

// mean over all elements: the per-ray sums added in one fixed order by a single CTA
__global__ void __launch_bounds__(256) k_interlevel_mean(const float* __restrict__ loss_per_ray, int64_t R, double inv_count, float* __restrict__ loss) {
  __shared__ double part[256];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < R; i += 256) s += (double)loss_per_ray[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int d = 128; d > 0; d >>= 1) {
    if ((int)threadIdx.x < d) part[threadIdx.x] += part[threadIdx.x + d];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = (float)(part[0] * inv_count);
}

}  // namespace sdfb200

using namespace sdfb200;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int sdfb200_interlevel_loss(const float* fine_bins, const float* fine_weights, int32_t n_fine, const float* proposal_bins,
                                       const float* proposal_weights, int32_t n_proposal, int64_t n_rays, int32_t form, float blur_radius,
                                       float* loss_per_ray, float* loss, float* grad_proposal_weights, void* stream) {
  SDFB_REQUIRE(n_rays >= 0, "n_rays must not be negative");
  SDFB_REQUIRE(n_fine >= 1 && n_fine <= kInterlevelMaxSamples, "n_fine must be 1..1024");
  SDFB_REQUIRE(n_proposal >= 1 && n_proposal <= kInterlevelMaxSamples, "n_proposal must be 1..1024");
  SDFB_REQUIRE(form == SDFB200_INTERLEVEL_OUTER || form == SDFB200_INTERLEVEL_ZIP, "form must be SDFB200_INTERLEVEL_OUTER or SDFB200_INTERLEVEL_ZIP");
  SDFB_REQUIRE(form != SDFB200_INTERLEVEL_ZIP || blur_radius > 0.f, "the Zip-NeRF form needs blur_radius > 0");
  if (n_rays == 0) return 0;
  SDFB_REQUIRE(fine_bins && fine_weights && proposal_bins && proposal_weights && loss_per_ray, "NULL pointer");
  const bool zip = form == SDFB200_INTERLEVEL_ZIP;
  const size_t slice = sizeof(float) * (zip ? zip_slice_floats(n_fine, n_proposal) : outer_slice_floats(n_fine, n_proposal));
  size_t warps = kInterlevelSmemBudget / slice;
  warps = warps < 1 ? 1 : (warps > kInterlevelMaxWarps ? kInterlevelMaxWarps : warps);
  const unsigned blocks = (unsigned)ceil_div(n_rays, (int64_t)warps);
  if (zip) {
    k_interlevel_zip<<<blocks, 32 * (unsigned)warps, warps * slice, ST(stream)>>>(fine_bins, fine_weights, n_fine, proposal_bins, proposal_weights,
                                                                                  n_proposal, n_rays, blur_radius, loss_per_ray, grad_proposal_weights);
    SDFB_LAUNCHED("k_interlevel_zip");
  } else {
    k_interlevel_outer<<<blocks, 32 * (unsigned)warps, warps * slice, ST(stream)>>>(fine_bins, fine_weights, n_fine, proposal_bins, proposal_weights,
                                                                                    n_proposal, n_rays, loss_per_ray, grad_proposal_weights);
    SDFB_LAUNCHED("k_interlevel_outer");
  }
  if (loss != nullptr) {
    const double count = (double)n_rays * (double)(zip ? n_proposal : n_fine);
    k_interlevel_mean<<<1, 256, 0, ST(stream)>>>(loss_per_ray, n_rays, 1.0 / count, loss);
    SDFB_LAUNCHED("k_interlevel_mean");
  }
  return 0;
}
