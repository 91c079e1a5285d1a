// Shared helpers for the sdfb200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/sdfb200.h"

namespace sdfb200 {

extern thread_local char g_err[512];
extern std::atomic<long long> g_launches;

inline int fail(int code, const char* fmt, const char* a = "", long long b = 0) {
  snprintf(g_err, sizeof(g_err), fmt, a, b);
  return code;
}

#define SDFB_REQUIRE(cond, msg)                                                  \
  do {                                                                           \
    if (!(cond)) return ::sdfb200::fail(SDFB200_EINVAL, "%s (%lld)", msg, 0LL);  \
  } while (0)

// after a kernel launch: count it and surface launch-configuration errors without synchronising
inline int launched(const char* name) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    snprintf(g_err, sizeof(g_err), "%s: %s", name, cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}
#define SDFB_LAUNCHED(name)                   \
  do {                                        \
    int r__ = ::sdfb200::launched(name);      \
    if (r__) return r__;                      \
  } while (0)

#define SDFB_CUDA(call)                                                                             \
  do {                                                                                              \
    cudaError_t e__ = (call);                                                                       \
    if (e__ != cudaSuccess) {                                                                       \
      snprintf(::sdfb200::g_err, sizeof(::sdfb200::g_err), "%s: %s", #call, cudaGetErrorString(e__)); \
      return (int)e__;                                                                              \
    }                                                                                               \
  } while (0)

constexpr int kNumSMs = 132;   // H100 SXM: sizes the per-CTA workspaces of the persistent kernels

// CTAs of a persistent launch: the SM count of the current device (114 on the H100 PCIe part), at most kNumSMs (the workspace bound).
// Queried once per device: the samplers launch the field kernel many times per step and the attribute query is not free.
inline int persistent_ctas() {
  static std::atomic<int> cached[64];   // per device ordinal, 0 = not queried yet
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    cudaGetLastError();   // do not leave the failed query behind for the next launch check
    return kNumSMs;
  }
  if (dev >= 0 && dev < 64 && (n = cached[dev].load(std::memory_order_relaxed)) > 0) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    return kNumSMs;
  }
  n = n < kNumSMs ? n : kNumSMs;
  if (dev >= 0 && dev < 64) cached[dev].store(n, std::memory_order_relaxed);
  return n;
}

__host__ __device__ inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// nn.Softplus(beta=100), threshold 20 (sdf_field.py:365)
__device__ __forceinline__ float softplus100(float z) {
  float t = z * 100.0f;
  return t > 20.0f ? z : log1pf(expf(t)) * 0.01f;
}
// d softplus100 / dz expressed through h = softplus100(z):  sigma(100 z) = 1 - exp(-100 h)
__device__ __forceinline__ float dsoftplus100_from_h(float h) { return -expm1f(-100.0f * h); }

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// ---- SDFField heads (sdf_field.py), shared by the generic engine (field_simt.cu) and the fused kernel (field_tc_kernel.cuh).  The
// expressions are contractible, so both engines get the same fused multiply-adds.

// LaplaceDensity.forward (sdf_field.py:57-71) with beta = |beta| + beta_min
__device__ __forceinline__ float sdf_density(float sdf, float beta_param, float beta_min) {
  const float beta = fabsf(beta_param) + beta_min;
  const float sg = sdf > 0.f ? 1.f : (sdf < 0.f ? -1.f : 0.f);
  return (1.0f / beta) * (0.5f + 0.5f * sg * expm1f(-fabsf(sdf) / beta));
}

// get_alpha (sdf_field.py:494-517): true_cos = direction . gradient, delta the sample's length, inv_s = exp(10 variance) clamped
__device__ __forceinline__ float neus_alpha(float sdf, float true_cos, float delta, float variance, float cos_anneal) {
  const float inv_s = fminf(fmaxf(expf(variance * 10.0f), 1e-6f), 1e6f);
  const float iter_cos = -(fmaxf(-true_cos * 0.5f + 0.5f, 0.f) * (1.0f - cos_anneal) + fmaxf(-true_cos, 0.f) * cos_anneal);
  const float prev_cdf = sigmoidf_((sdf - iter_cos * delta * 0.5f) * inv_s), next_cdf = sigmoidf_((sdf + iter_cos * delta * 0.5f) * inv_s);
  return fminf(fmaxf((prev_cdf - next_cdf + 1e-5f) / (prev_cdf + 1e-5f), 0.f), 1.f);
}

// F.normalize(g, p=2, eps=1e-12)
__device__ __forceinline__ float3 normalize_eps(float x, float y, float z) {
  const float n = fmaxf(sqrtf(x * x + y * y + z * z), 1e-12f);
  return make_float3(x / n, y / n, z / n);
}

// rgb * (1 + 2 padding) - padding (sdf_field.py:610)
__device__ __forceinline__ float padded_rgb(float rgb, float padding) { return rgb * (1.f + 2.f * padding) - padding; }

// sigmoid(-10 sdf) (sdf_field.py:529)
__device__ __forceinline__ float occupancy(float sdf) { return sigmoidf_(-10.0f * sdf); }

// ---- transmittance and compositing (cameras/rays.py:131-230, model_components/renderers.py:42-261)

struct ScanAdd {
  template <class T> __device__ __forceinline__ T operator()(T a, T b) const { return a + b; }
};
struct ScanMul {
  template <class T> __device__ __forceinline__ T operator()(T a, T b) const { return a * b; }
};

// inclusive scan of v over the 32 lanes of a full warp (Hillis-Steele: log2(32) shuffle steps, every lane in the same order)
template <class T, class Op = ScanAdd>
__device__ __forceinline__ T warp_scan_incl(T v, int lane, Op op = Op()) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const T o = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v = op(v, o);
  }
  return v;
}
// the exclusive scan from the inclusive one: shifted up by one lane, the identity on lane 0
template <class T>
__device__ __forceinline__ T warp_scan_excl(T incl, int lane, T identity) {
  const T e = __shfl_up_sync(0xffffffffu, incl, 1);
  return lane == 0 ? identity : e;
}

// the factor by which a NeuS alpha lowers the transmittance: 1 - alpha + 1e-7 (rays.py:204-206)
__device__ __forceinline__ float neus_trans_factor(float alpha) { return __fadd_rn(__fsub_rn(1.0f, alpha), 1e-7f); }

// background colour of ray r (renderers.py:97-118): one colour, one per ray, or the ray's last sample colour `last`
__device__ __forceinline__ void ray_background(int bg_mode, const float* bg, int64_t r, const float* last, float (&c)[3]) {
  if (bg_mode == SDFB200_BG_COLOR) { c[0] = bg[0]; c[1] = bg[1]; c[2] = bg[2]; }
  else if (bg_mode == SDFB200_BG_PER_RAY) { c[0] = bg[r * 3]; c[1] = bg[r * 3 + 1]; c[2] = bg[r * 3 + 2]; }
  else { c[0] = last[0]; c[1] = last[1]; c[2] = last[2]; }
}

// The end of the compositing of ray r from its sums of w, w rgb, w normal and w step: rgb over the background (clamped to [0, 1] when
// clamp01), accumulation, normal and expected depth (renderers.py:97-118, 190-197, 249-252).  Contractible: `sum + bg * (1 - acc)` becomes
// one fma per channel.  A NULL output is not written; the background is read only for the rgb.
__device__ __forceinline__ void finish_ray(int64_t r, float acc, const float (&wrgb)[3], const float (&wn)[3], float wstep, int bg_mode, const float* bg,
                                           const float* last, int clamp01, float* o_rgb, float* o_acc, float* o_normal, float* o_depth) {
  if (o_rgb) {
    float bgc[3];
    ray_background(bg_mode, bg, r, last, bgc);
    const float rem = 1.0f - acc;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = wrgb[c] + bgc[c] * rem;
      o_rgb[r * 3 + c] = clamp01 ? fminf(fmaxf(v, 0.f), 1.f) : v;
    }
  }
  if (o_acc) o_acc[r] = acc;
  if (o_normal) { o_normal[r * 3] = wn[0]; o_normal[r * 3 + 1] = wn[1]; o_normal[r * 3 + 2] = wn[2]; }
  if (o_depth) o_depth[r] = wstep / (acc + 1e-10f);
}

// SceneContraction (spatial_distortions.py:66-73): x <- (2 - 1/|x|) * (x/|x|) where |x| >= 1, |x| the L-inf or L2 norm.  Every
// operation is rounded on its own (no FMA contraction), so the result is the reference's fp32 one.
__device__ __forceinline__ void scene_contract(int contraction, float& px, float& py, float& pz) {
  if (contraction == SDFB200_CONTRACT_NONE) return;
  const float mag = contraction == SDFB200_CONTRACT_LINF ? fmaxf(fabsf(px), fmaxf(fabsf(py), fabsf(pz)))
                                                         : sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)), __fmul_rn(pz, pz)));
  if (mag >= 1.f) {
    const float k = __fsub_rn(2.f, __fdiv_rn(1.f, mag));
    px = __fmul_rn(k, __fdiv_rn(px, mag)); py = __fmul_rn(k, __fdiv_rn(py, mag)); pz = __fmul_rn(k, __fdiv_rn(pz, mag));
  }
}

// Frustums.get_positions (cameras/rays.py) of sample s of ray r, bins [R, S+1]: origins + directions * (starts + ends) / 2 in the
// reference's operation order, each operation rounded on its own (no FMA), so the positions are the reference's fp32 ones
__device__ __forceinline__ void ray_midpoint(const float* origins, const float* directions, const float* bins, long long r, int S, long long s,
                                             float (&x)[3]) {
  const float* b = bins + r * (S + 1) + s;
  const float se = __fadd_rn(__ldg(b), __ldg(b + 1));
#pragma unroll
  for (int c = 0; c < 3; ++c) x[c] = __fadd_rn(__ldg(origins + r * 3 + c), __fmul_rn(__fmul_rn(__ldg(directions + r * 3 + c), se), 0.5f));
}

// float atomic min / max by compare-and-swap (used for the batch-global steps.min()/max() of DepthRenderer, renderers.py:257)
__device__ __forceinline__ void atomic_min_float(float* addr, float v) {
  int* ia = reinterpret_cast<int*>(addr);
  int old = *ia;
  while (__int_as_float(old) > v) {
    const int assumed = old;
    old = atomicCAS(ia, assumed, __float_as_int(v));
    if (old == assumed) break;
  }
}
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  int* ia = reinterpret_cast<int*>(addr);
  int old = *ia;
  while (__int_as_float(old) < v) {
    const int assumed = old;
    old = atomicCAS(ia, assumed, __float_as_int(v));
    if (old == assumed) break;
  }
}

}  // namespace sdfb200
