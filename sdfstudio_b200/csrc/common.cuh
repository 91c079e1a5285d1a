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
