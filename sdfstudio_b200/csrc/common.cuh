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
