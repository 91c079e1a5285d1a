// Multi-resolution hash-grid lookup (device side).  One (point, level) is prepared once (level_prepare: the 8 corner rows, the blend
// weights and their derivatives); every grid kernel builds on that: the forward fetches the rows and blends them (level_finish), the
// backward scatters with the blend's corner weights (corner_weights), the double backward takes rows and per-axis weights from it.
//
// torch layout restates HashEncoding.pytorch_fwd (nerfstudio/field_components/encodings.py:357-398 and the
// smoothstep remap :700-701): corners = ceil/floor(x*scale), weight `offset` on the CEIL corner, blend order x,y,z.
// tcnn layout follows tiny-cuda-nn's GridEncoding conventions (SURVEY.md appendix A.3).
#pragma once
#include "common.cuh"

namespace sdfb200 {

constexpr uint32_t kPrimeY = 2654435761u;
constexpr uint32_t kPrimeZ = 805459861u;

// L2 eviction-priority policy (createpolicy): the hash table is re-read by every tile of the fused kernel -> evict_last
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// One table row (F features of type T) as fp32.  HINT: an L2 cache-hinted load under policy `pol` (F = 2, the fused kernel's).
template <typename T, int F, bool HINT = false>
__device__ __forceinline__ void load_row(const void* table, uint64_t row, float (&v)[F], uint64_t pol = 0) {
  const T* p = reinterpret_cast<const T*>(table) + row * F;
  if constexpr (HINT) {
    static_assert(F == 2, "hinted loads are only used by the F=2 fused kernel");
    if constexpr (sizeof(T) == 4) {
      asm volatile("ld.global.nc.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;" : "=f"(v[0]), "=f"(v[1]) : "l"(p), "l"(pol));
    } else {
      uint32_t raw;
      asm volatile("ld.global.nc.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(raw) : "l"(p), "l"(pol));
      const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&raw));
      v[0] = t.x; v[1] = t.y;
    }
  } else if constexpr (sizeof(T) == 4) {
    if constexpr (F == 1) {
      v[0] = __ldg(p);
    } else if constexpr (F == 2) {
      float2 t = __ldg(reinterpret_cast<const float2*>(p));
      v[0] = t.x; v[1] = t.y;
    } else {
#pragma unroll
      for (int i = 0; i < F; i += 4) {
        float4 t = __ldg(reinterpret_cast<const float4*>(p + i));
        v[i] = t.x; v[i + 1] = t.y; v[i + 2] = t.z; v[i + 3] = t.w;
      }
    }
  } else {
    if constexpr (F == 1) {
      v[0] = __half2float(p[0]);
    } else if constexpr (F == 2) {
      float2 t = __half22float2(__ldg(reinterpret_cast<const __half2*>(p)));
      v[0] = t.x; v[1] = t.y;
    } else if constexpr (F == 4) {
      uint2 raw = __ldg(reinterpret_cast<const uint2*>(p));
      float2 a = __half22float2(*reinterpret_cast<__half2*>(&raw.x));
      float2 b = __half22float2(*reinterpret_cast<__half2*>(&raw.y));
      v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
    } else {
#pragma unroll
      for (int i = 0; i < F; i += 8) {
        uint4 raw = __ldg(reinterpret_cast<const uint4*>(p + i));
        const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 a = __half22float2(h[j]);
          v[i + 2 * j] = a.x; v[i + 2 * j + 1] = a.y;
        }
      }
    }
  }
}

// LAYOUT < 0: decided at run time from g.layout; otherwise compile-time (the dead branch is dropped: code size matters for the
// warp-specialised fused kernel, whose roles compete for the instruction cache)
template <int LAYOUT>
__device__ __forceinline__ bool torch_layout(const sdfb200_grid_t& g) {
  return LAYOUT < 0 ? g.layout == SDFB200_GRID_TORCH : LAYOUT == SDFB200_GRID_TORCH;
}

// One prepared (point, level).  Corner k sits at bit 0 = x, bit 1 = y, bit 2 = z; a set bit is the corner that carries the per-axis
// weight w (torch: the ceil corner, tcnn: cell + 1), a clear bit carries 1 - w.  Per axis, dw = dw/d(x*scale) and
// d2w = d2w/dx01^2 = (6 - 12t) scale^2 (floor / ceil are treated as constants).
struct LevelCtx {
  uint32_t idx[8];   // table row of corner k, relative to `base`
  uint64_t base;
  float w[3], dw[3], d2w[3], s;
};

template <int LAYOUT = -1>
__device__ __forceinline__ void level_prepare(const sdfb200_grid_t& g, int l, float x, float y, float z, LevelCtx& c) {
  if constexpr (LAYOUT < 0) {   // one branch per level, not a select per step
    if (g.layout == SDFB200_GRID_TORCH) level_prepare<SDFB200_GRID_TORCH>(g, l, x, y, z, c);
    else level_prepare<SDFB200_GRID_TCNN>(g, l, x, y, z, c);
    return;
  }
  constexpr bool torch = LAYOUT == SDFB200_GRID_TORCH;
  const float s = g.scale[l];
  const float xs[3] = {x, y, z};
  uint32_t lo[3], hi[3];   // per axis the corner coordinate of a clear / set bit
  c.s = s;
  c.base = g.offset[l];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float p = torch ? __fmul_rn(xs[d], s) : fmaf(xs[d], s, 0.5f);
    const float fl = floorf(p);
    lo[d] = (uint32_t)(int)fl;
    hi[d] = torch ? (uint32_t)(int)ceilf(p) : lo[d] + 1u;
    const float t = __fsub_rn(p, fl);
    if (g.smoothstep) {
      // rounded step by step as the reference's remap; 2t is exact, so this is also tcnn's t*t*(3-2t)
      c.w[d] = __fmul_rn(__fmul_rn(t, t), __fsub_rn(3.0f, __fmul_rn(2.0f, t)));
      c.dw[d] = 6.f * t * (1.f - t);
      c.d2w[d] = (6.f - 12.f * t) * s * s;
    } else {
      c.w[d] = t; c.dw[d] = 1.f; c.d2w[d] = 0.f;
    }
  }
  const uint32_t mask = (1u << g.log2_hashmap_size) - 1u;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t ix = (k & 1) ? hi[0] : lo[0], iy = (k & 2) ? hi[1] : lo[1], iz = (k & 4) ? hi[2] : lo[2];
    // hash = x ^ y*P1 ^ z*P2 (int64 in the torch reference; the low log2T bits equal the uint32 product's low bits)
    const uint32_t h = ix ^ (iy * kPrimeY) ^ (iz * kPrimeZ);
    if (torch) {
      c.idx[k] = h & mask;
    } else {
      const uint32_t res = g.resolution[l];
      c.idx[k] = (g.hashed[l] ? h : ix + iy * res + iz * res * res) % g.size[l];
    }
  }
}

template <typename T, int F, bool HINT = false>
__device__ __forceinline__ void level_fetch(const void* table, const LevelCtx& c, float (&v)[8][F], uint64_t pol = 0) {
#pragma unroll
  for (int k = 0; k < 8; ++k) load_row<T, F, HINT>(table, c.base + c.idx[k], v[k], pol);
}

// the same rows requested into L2 (evict_last, the fused kernel's table policy) without waiting for them or holding registers
template <typename T, int F>
__device__ __forceinline__ void level_prefetch_l2(const void* table, const LevelCtx& c) {
#pragma unroll
  for (int k = 0; k < 8; ++k)
    asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(reinterpret_cast<const T*>(table) + (c.base + c.idx[k]) * F));
}

// out[f] and dout[f][c] = d out[f] / d x01[c].  torch: the reference's expression tree (no FMA contraction on the value path).
template <int F, int LAYOUT = -1>
__device__ __forceinline__ void level_finish(const sdfb200_grid_t& g, const LevelCtx& c, const float (&v)[8][F], float (&out)[F], float (&dout)[F][3]) {
  if (torch_layout<LAYOUT>(g)) {
    // the reference's corners f0..f7 = (c,c,c)(c,f,c)(f,f,c)(f,c,c)(c,c,f)(c,f,f)(f,f,f)(f,c,f) in x,y,z (c = ceil = set bit)
    const float(&f0)[F] = v[7], (&f1)[F] = v[5], (&f2)[F] = v[4], (&f3)[F] = v[6], (&f4)[F] = v[3], (&f5)[F] = v[1], (&f6)[F] = v[0], (&f7)[F] = v[2];
    const float ox = c.w[0], oy = c.w[1], oz = c.w[2];
    const float nx = __fsub_rn(1.f, ox), ny = __fsub_rn(1.f, oy), nz = __fsub_rn(1.f, oz);
#pragma unroll
    for (int f = 0; f < F; ++f) {
      const float f03 = __fadd_rn(__fmul_rn(f0[f], ox), __fmul_rn(f3[f], nx));
      const float f12 = __fadd_rn(__fmul_rn(f1[f], ox), __fmul_rn(f2[f], nx));
      const float f56 = __fadd_rn(__fmul_rn(f5[f], ox), __fmul_rn(f6[f], nx));
      const float f47 = __fadd_rn(__fmul_rn(f4[f], ox), __fmul_rn(f7[f], nx));
      const float f0312 = __fadd_rn(__fmul_rn(f03, oy), __fmul_rn(f12, ny));
      const float f4756 = __fadd_rn(__fmul_rn(f47, oy), __fmul_rn(f56, ny));
      out[f] = __fadd_rn(__fmul_rn(f0312, oz), __fmul_rn(f4756, nz));
      const float gx = ((f0[f] - f3[f]) * oy + (f1[f] - f2[f]) * ny) * oz + ((f4[f] - f7[f]) * oy + (f5[f] - f6[f]) * ny) * nz;
      const float gy = (f03 - f12) * oz + (f47 - f56) * nz;
      const float gz = f0312 - f4756;
      dout[f][0] = gx * c.dw[0] * c.s; dout[f][1] = gy * c.dw[1] * c.s; dout[f][2] = gz * c.dw[2] * c.s;
    }
  } else {
#pragma unroll
    for (int f = 0; f < F; ++f) { out[f] = 0.f; dout[f][0] = dout[f][1] = dout[f][2] = 0.f; }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float wx = (k & 1) ? c.w[0] : 1.f - c.w[0], wy = (k & 2) ? c.w[1] : 1.f - c.w[1], wz = (k & 4) ? c.w[2] : 1.f - c.w[2];
      const float wt = wx * wy * wz;
#pragma unroll
      for (int f = 0; f < F; ++f) {
        out[f] = fmaf(wt, v[k][f], out[f]);
        dout[f][0] += ((k & 1) ? 1.f : -1.f) * wy * wz * v[k][f];
        dout[f][1] += ((k & 2) ? 1.f : -1.f) * wx * wz * v[k][f];
        dout[f][2] += ((k & 4) ? 1.f : -1.f) * wx * wy * v[k][f];
      }
    }
#pragma unroll
    for (int f = 0; f < F; ++f) { dout[f][0] *= c.dw[0] * c.s; dout[f][1] *= c.dw[1] * c.s; dout[f][2] *= c.dw[2] * c.s; }
  }
}

// the whole lookup of one (point, level)
template <typename T, int F>
__device__ __forceinline__ void encode_level(const sdfb200_grid_t& g, const void* table, int l, float x, float y, float z,
                                             float (&out)[F], float (&dout)[F][3]) {
  LevelCtx c;
  float v[8][F];
  level_prepare(g, l, x, y, z, c);
  level_fetch<T, F>(table, c, v);
  level_finish<F>(g, c, v, out, dout);
}

// weight of corner k in the blend of level_finish: the backward scatters d out / d row with it
__device__ __forceinline__ void corner_weights(const LevelCtx& c, float (&w)[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k)
    w[k] = ((k & 1) ? c.w[0] : 1.f - c.w[0]) * ((k & 2) ? c.w[1] : 1.f - c.w[1]) * ((k & 4) ? c.w[2] : 1.f - c.w[2]);
}

}  // namespace sdfb200
