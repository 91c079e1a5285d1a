// Multi-resolution hash-grid lookup (device side).  One call = one (point, level): 8 corner gathers + tri-linear /
// smoothstep blend, optionally with d(out)/d(x01).
//
// torch layout restates HashEncoding.pytorch_fwd (nerfstudio/field_components/encodings.py:357-398 and the
// smoothstep remap :700-701): corners = ceil/floor(x*scale), weight `offset` on the CEIL corner, blend order x,y,z.
// tcnn layout follows tiny-cuda-nn's GridEncoding conventions (SURVEY.md appendix A.3).
#pragma once
#include "common.cuh"

namespace sdfb200 {

constexpr uint32_t kPrimeY = 2654435761u;
constexpr uint32_t kPrimeZ = 805459861u;

template <typename T, int F>
struct TableLoad;
template <int F>
struct TableLoad<float, F> {
  __device__ static __forceinline__ void load(const void* table, uint64_t row, float (&v)[F]) {
    const float* p = reinterpret_cast<const float*>(table) + row * F;
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
  }
};
template <int F>
struct TableLoad<__half, F> {
  __device__ static __forceinline__ void load(const void* table, uint64_t row, float (&v)[F]) {
    const __half* p = reinterpret_cast<const __half*>(table) + row * F;
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
};

// L2 eviction-priority policies (createpolicy): the hash table is re-read by every tile -> evict_last; streaming
// scratch -> evict_first, so that it pushes as little of the table out of L2 as possible.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_normal() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// hinted F=2 table loads (fp32: 8 bytes, fp16: 4 bytes) used by the fused kernel
template <typename T, int F>
__device__ __forceinline__ void table_load_hint(const void* table, uint64_t row, float (&v)[F], uint64_t pol) {
  static_assert(F == 2, "hinted loads are only used by the F=2 fused kernel");
  if constexpr (sizeof(T) == 4) {
    const float* p = reinterpret_cast<const float*>(table) + row * F;
    asm volatile("ld.global.nc.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;" : "=f"(v[0]), "=f"(v[1]) : "l"(p), "l"(pol));
  } else {
    const __half* p = reinterpret_cast<const __half*>(table) + row * F;
    uint32_t raw;
    asm volatile("ld.global.nc.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(raw) : "l"(p), "l"(pol));
    const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&raw));
    v[0] = t.x; v[1] = t.y;
  }
}

// -----------------------------------------------------------------------------------------------------------------
// torch layout.  out[f] and (optionally) dout[f][c] = d out[f] / d x01[c].
// Rounding follows the reference expression tree (no FMA contraction on the value path).
// -----------------------------------------------------------------------------------------------------------------
template <typename T, int F, bool GRAD, bool HINT = false>
__device__ __forceinline__ void encode_level_torch(const sdfb200_grid_t& g, const void* table, int l, float x, float y, float z,
                                                   float (&out)[F], float (&dout)[F][3], uint64_t pol = 0) {
  const float s = g.scale[l];
  const float sx = __fmul_rn(x, s), sy = __fmul_rn(y, s), sz = __fmul_rn(z, s);
  const float fxf = floorf(sx), fyf = floorf(sy), fzf = floorf(sz);
  const uint32_t fx = (uint32_t)(int)fxf, fy = (uint32_t)(int)fyf, fz = (uint32_t)(int)fzf;
  const uint32_t cx = (uint32_t)(int)ceilf(sx), cy = (uint32_t)(int)ceilf(sy), cz = (uint32_t)(int)ceilf(sz);
  float ox = __fsub_rn(sx, fxf), oy = __fsub_rn(sy, fyf), oz = __fsub_rn(sz, fzf);
  float dx = 1.f, dy = 1.f, dz = 1.f;  // d(blend weight)/d(scaled coordinate)
  if (g.smoothstep) {
    if (GRAD) {
      dx = 6.f * ox * (1.f - ox); dy = 6.f * oy * (1.f - oy); dz = 6.f * oz * (1.f - oz);
    }
    ox = __fmul_rn(__fmul_rn(ox, ox), __fsub_rn(3.0f, __fmul_rn(2.0f, ox)));
    oy = __fmul_rn(__fmul_rn(oy, oy), __fsub_rn(3.0f, __fmul_rn(2.0f, oy)));
    oz = __fmul_rn(__fmul_rn(oz, oz), __fsub_rn(3.0f, __fmul_rn(2.0f, oz)));
  }
  const uint32_t mask = (1u << g.log2_hashmap_size) - 1u;
  const uint64_t base = g.offset[l];
  // hash = x ^ y*P1 ^ z*P2 (int64 in the reference; the low log2T bits equal the uint32 product's low bits)
  const uint32_t hyc = cy * kPrimeY, hyf = fy * kPrimeY, hzc = cz * kPrimeZ, hzf = fz * kPrimeZ;
  float f0[F], f1[F], f2[F], f3[F], f4[F], f5[F], f6[F], f7[F];
  if constexpr (HINT) table_load_hint<T, F>(table, base + ((cx ^ hyc ^ hzc) & mask), f0, pol); else TableLoad<T, F>::load(table, base + ((cx ^ hyc ^ hzc) & mask), f0);  // (c,c,c)
  if constexpr (HINT) table_load_hint<T, F>(table, base + ((cx ^ hyf ^ hzc) & mask), f1, pol); else TableLoad<T, F>::load(table, base + ((cx ^ hyf ^ hzc) & mask), f1);  // (c,f,c)
  if constexpr (HINT) table_load_hint<T, F>(table, base + ((fx ^ hyf ^ hzc) & mask), f2, pol); else TableLoad<T, F>::load(table, base + ((fx ^ hyf ^ hzc) & mask), f2);  // (f,f,c)
  if constexpr (HINT) table_load_hint<T, F>(table, base + ((fx ^ hyc ^ hzc) & mask), f3, pol); else TableLoad<T, F>::load(table, base + ((fx ^ hyc ^ hzc) & mask), f3);  // (f,c,c)
  if constexpr (HINT) table_load_hint<T, F>(table, base + ((cx ^ hyc ^ hzf) & mask), f4, pol); else TableLoad<T, F>::load(table, base + ((cx ^ hyc ^ hzf) & mask), f4);  // (c,c,f)
  if constexpr (HINT) table_load_hint<T, F>(table, base + ((cx ^ hyf ^ hzf) & mask), f5, pol); else TableLoad<T, F>::load(table, base + ((cx ^ hyf ^ hzf) & mask), f5);  // (c,f,f)
  if constexpr (HINT) table_load_hint<T, F>(table, base + ((fx ^ hyf ^ hzf) & mask), f6, pol); else TableLoad<T, F>::load(table, base + ((fx ^ hyf ^ hzf) & mask), f6);  // (f,f,f)
  if constexpr (HINT) table_load_hint<T, F>(table, base + ((fx ^ hyc ^ hzf) & mask), f7, pol); else TableLoad<T, F>::load(table, base + ((fx ^ hyc ^ hzf) & mask), f7);  // (f,c,f)
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
    if (GRAD) {
      const float gx = ((f0[f] - f3[f]) * oy + (f1[f] - f2[f]) * ny) * oz + ((f4[f] - f7[f]) * oy + (f5[f] - f6[f]) * ny) * nz;
      const float gy = (f03 - f12) * oz + (f47 - f56) * nz;
      const float gz = f0312 - f4756;
      dout[f][0] = gx * dx * s; dout[f][1] = gy * dy * s; dout[f][2] = gz * dz * s;
    }
  }
}

// -----------------------------------------------------------------------------------------------------------------
// tcnn layout
// -----------------------------------------------------------------------------------------------------------------
template <typename T, int F, bool GRAD, bool HINT = false>
__device__ __forceinline__ void encode_level_tcnn(const sdfb200_grid_t& g, const void* table, int l, float x, float y, float z,
                                                  float (&out)[F], float (&dout)[F][3], uint64_t pol = 0) {
  const float s = g.scale[l];
  const uint32_t res = g.resolution[l], size = g.size[l];
  const bool hashed = g.hashed[l];
  const uint64_t base = g.offset[l];
  float p[3] = {fmaf(x, s, 0.5f), fmaf(y, s, 0.5f), fmaf(z, s, 0.5f)};
  uint32_t cell[3];
  float w[3], dw[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float fl = floorf(p[d]);
    cell[d] = (uint32_t)(int)fl;
    const float t = p[d] - fl;
    if (g.smoothstep) {
      w[d] = t * t * (3.f - 2.f * t);
      dw[d] = 6.f * t * (1.f - t);
    } else {
      w[d] = t;
      dw[d] = 1.f;
    }
  }
#pragma unroll
  for (int f = 0; f < F; ++f) {
    out[f] = 0.f;
    if (GRAD) dout[f][0] = dout[f][1] = dout[f][2] = 0.f;
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const uint32_t ix = cell[0] + (c & 1), iy = cell[1] + ((c >> 1) & 1), iz = cell[2] + ((c >> 2) & 1);
    const float wx = (c & 1) ? w[0] : 1.f - w[0], wy = (c & 2) ? w[1] : 1.f - w[1], wz = (c & 4) ? w[2] : 1.f - w[2];
    uint32_t idx = hashed ? (ix ^ (iy * kPrimeY) ^ (iz * kPrimeZ)) : (ix + iy * res + iz * res * res);
    idx %= size;
    float v[F];
    if constexpr (HINT) table_load_hint<T, F>(table, base + idx, v, pol); else TableLoad<T, F>::load(table, base + idx, v);
    const float wt = wx * wy * wz;
#pragma unroll
    for (int f = 0; f < F; ++f) {
      out[f] = fmaf(wt, v[f], out[f]);
      if (GRAD) {
        dout[f][0] += ((c & 1) ? 1.f : -1.f) * wy * wz * v[f];
        dout[f][1] += ((c & 2) ? 1.f : -1.f) * wx * wz * v[f];
        dout[f][2] += ((c & 4) ? 1.f : -1.f) * wx * wy * v[f];
      }
    }
  }
  if (GRAD) {
#pragma unroll
    for (int f = 0; f < F; ++f) {
      dout[f][0] *= dw[0] * s; dout[f][1] *= dw[1] * s; dout[f][2] *= dw[2] * s;
    }
  }
}

// LAYOUT < 0: decided at run time from g.layout; otherwise compile-time (the dead branch is dropped: code size matters for the
// warp-specialised fused kernel, whose roles compete for the instruction cache)
template <typename T, int F, bool GRAD, bool HINT = false, int LAYOUT = -1>
__device__ __forceinline__ void encode_level(const sdfb200_grid_t& g, const void* table, int l, float x, float y, float z,
                                             float (&out)[F], float (&dout)[F][3], uint64_t pol = 0) {
  if (LAYOUT < 0 ? g.layout == SDFB200_GRID_TORCH : LAYOUT == SDFB200_GRID_TORCH)
    encode_level_torch<T, F, GRAD, HINT>(g, table, l, x, y, z, out, dout, pol);
  else
    encode_level_tcnn<T, F, GRAD, HINT>(g, table, l, x, y, z, out, dout, pol);
}


// -----------------------------------------------------------------------------------------------------------------
// Split form of encode_level for software-pipelined gathers: prepare (indices + weights), fetch (8 loads), finish (blend).
// prepare + fetch + finish computes exactly what encode_level computes (same expression trees), so several levels can have
// their 8 gathers in flight together.
// -----------------------------------------------------------------------------------------------------------------
struct LevelCtx {
  uint32_t idx[8];   // table rows relative to `base`; torch corner order (c,c,c)(c,f,c)(f,f,c)(f,c,c)(c,c,f)(c,f,f)(f,f,f)(f,c,f), tcnn: bit0=x bit1=y bit2=z
  uint64_t base;
  float w[3], dw[3], s;
};

template <int LAYOUT = -1>
__device__ __forceinline__ void level_prepare(const sdfb200_grid_t& g, int l, float x, float y, float z, LevelCtx& c) {
  const float s = g.scale[l];
  c.s = s;
  c.base = g.offset[l];
  if (LAYOUT < 0 ? g.layout == SDFB200_GRID_TORCH : LAYOUT == SDFB200_GRID_TORCH) {
    const float sx = __fmul_rn(x, s), sy = __fmul_rn(y, s), sz = __fmul_rn(z, s);
    const float fxf = floorf(sx), fyf = floorf(sy), fzf = floorf(sz);
    const uint32_t fx = (uint32_t)(int)fxf, fy = (uint32_t)(int)fyf, fz = (uint32_t)(int)fzf;
    const uint32_t cx = (uint32_t)(int)ceilf(sx), cy = (uint32_t)(int)ceilf(sy), cz = (uint32_t)(int)ceilf(sz);
    float ox = __fsub_rn(sx, fxf), oy = __fsub_rn(sy, fyf), oz = __fsub_rn(sz, fzf);
    c.dw[0] = c.dw[1] = c.dw[2] = 1.f;
    if (g.smoothstep) {
      c.dw[0] = 6.f * ox * (1.f - ox); c.dw[1] = 6.f * oy * (1.f - oy); c.dw[2] = 6.f * oz * (1.f - oz);
      ox = __fmul_rn(__fmul_rn(ox, ox), __fsub_rn(3.0f, __fmul_rn(2.0f, ox)));
      oy = __fmul_rn(__fmul_rn(oy, oy), __fsub_rn(3.0f, __fmul_rn(2.0f, oy)));
      oz = __fmul_rn(__fmul_rn(oz, oz), __fsub_rn(3.0f, __fmul_rn(2.0f, oz)));
    }
    c.w[0] = ox; c.w[1] = oy; c.w[2] = oz;
    const uint32_t mask = (1u << g.log2_hashmap_size) - 1u;
    const uint32_t hyc = cy * kPrimeY, hyf = fy * kPrimeY, hzc = cz * kPrimeZ, hzf = fz * kPrimeZ;
    c.idx[0] = (cx ^ hyc ^ hzc) & mask; c.idx[1] = (cx ^ hyf ^ hzc) & mask; c.idx[2] = (fx ^ hyf ^ hzc) & mask; c.idx[3] = (fx ^ hyc ^ hzc) & mask;
    c.idx[4] = (cx ^ hyc ^ hzf) & mask; c.idx[5] = (cx ^ hyf ^ hzf) & mask; c.idx[6] = (fx ^ hyf ^ hzf) & mask; c.idx[7] = (fx ^ hyc ^ hzf) & mask;
  } else {
    const uint32_t res = g.resolution[l], size = g.size[l];
    const bool hashed = g.hashed[l];
    const float p[3] = {fmaf(x, s, 0.5f), fmaf(y, s, 0.5f), fmaf(z, s, 0.5f)};
    uint32_t cell[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const float fl = floorf(p[d]);
      cell[d] = (uint32_t)(int)fl;
      const float t = p[d] - fl;
      if (g.smoothstep) { c.w[d] = t * t * (3.f - 2.f * t); c.dw[d] = 6.f * t * (1.f - t); }
      else { c.w[d] = t; c.dw[d] = 1.f; }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t ix = cell[0] + (k & 1), iy = cell[1] + ((k >> 1) & 1), iz = cell[2] + ((k >> 2) & 1);
      const uint32_t idx = hashed ? (ix ^ (iy * kPrimeY) ^ (iz * kPrimeZ)) : (ix + iy * res + iz * res * res);
      c.idx[k] = idx % size;
    }
  }
}

template <typename T, int F>
__device__ __forceinline__ void level_fetch(const void* table, const LevelCtx& c, float (&v)[8][F], uint64_t pol) {
#pragma unroll
  for (int k = 0; k < 8; ++k) table_load_hint<T, F>(table, c.base + c.idx[k], v[k], pol);
}

// F = 2 table entries whose element type is only known at run time (g.table_dtype)
__device__ __forceinline__ void level_fetch_rt2(const sdfb200_grid_t& g, const void* table, const LevelCtx& c, float (&v)[8][2], uint64_t pol) {
  if (g.table_dtype == SDFB200_DT_F16) {
#pragma unroll
    for (int k = 0; k < 8; ++k) table_load_hint<__half, 2>(table, c.base + c.idx[k], v[k], pol);
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) table_load_hint<float, 2>(table, c.base + c.idx[k], v[k], pol);
  }
}

template <int F, int LAYOUT = -1>
__device__ __forceinline__ void level_finish(const sdfb200_grid_t& g, const LevelCtx& c, const float (&v)[8][F], float (&out)[F], float (&dout)[F][3]) {
  if (LAYOUT < 0 ? g.layout == SDFB200_GRID_TORCH : LAYOUT == SDFB200_GRID_TORCH) {
    const float ox = c.w[0], oy = c.w[1], oz = c.w[2];
    const float nx = __fsub_rn(1.f, ox), ny = __fsub_rn(1.f, oy), nz = __fsub_rn(1.f, oz);
#pragma unroll
    for (int f = 0; f < F; ++f) {
      const float f03 = __fadd_rn(__fmul_rn(v[0][f], ox), __fmul_rn(v[3][f], nx));
      const float f12 = __fadd_rn(__fmul_rn(v[1][f], ox), __fmul_rn(v[2][f], nx));
      const float f56 = __fadd_rn(__fmul_rn(v[5][f], ox), __fmul_rn(v[6][f], nx));
      const float f47 = __fadd_rn(__fmul_rn(v[4][f], ox), __fmul_rn(v[7][f], nx));
      const float f0312 = __fadd_rn(__fmul_rn(f03, oy), __fmul_rn(f12, ny));
      const float f4756 = __fadd_rn(__fmul_rn(f47, oy), __fmul_rn(f56, ny));
      out[f] = __fadd_rn(__fmul_rn(f0312, oz), __fmul_rn(f4756, nz));
      const float gx = ((v[0][f] - v[3][f]) * oy + (v[1][f] - v[2][f]) * ny) * oz + ((v[4][f] - v[7][f]) * oy + (v[5][f] - v[6][f]) * ny) * nz;
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

// -----------------------------------------------------------------------------------------------------------------
// Layout-independent per-level geometry for the derivative kernels: per axis the two corner coordinates (c[d][1] carries
// weight w[d], c[d][0] carries 1-w[d]) and w, dw/dx01, d2w/dx01^2 (piecewise: floor/ceil are treated as constants).
// -----------------------------------------------------------------------------------------------------------------
struct LevelGeom {
  uint32_t c[3][2];
  float w[3], dw[3], d2w[3];
};

__device__ __forceinline__ void level_geom(const sdfb200_grid_t& g, int l, const float (&x)[3], LevelGeom& q) {
  const float s = g.scale[l];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    float t;
    if (g.layout == SDFB200_GRID_TORCH) {
      const float sx = __fmul_rn(x[d], s);
      const float fl = floorf(sx);
      q.c[d][0] = (uint32_t)(int)fl;
      q.c[d][1] = (uint32_t)(int)ceilf(sx);
      t = sx - fl;
    } else {
      const float p = fmaf(x[d], s, 0.5f);
      const float fl = floorf(p);
      q.c[d][0] = (uint32_t)(int)fl;
      q.c[d][1] = q.c[d][0] + 1u;
      t = p - fl;
    }
    if (g.smoothstep) {
      q.w[d] = t * t * (3.f - 2.f * t);
      q.dw[d] = 6.f * t * (1.f - t) * s;
      q.d2w[d] = (6.f - 12.f * t) * s * s;
    } else {
      q.w[d] = t;
      q.dw[d] = s;
      q.d2w[d] = 0.f;
    }
  }
}

__device__ __forceinline__ uint64_t corner_row(const sdfb200_grid_t& g, int l, uint32_t ix, uint32_t iy, uint32_t iz) {
  if (g.layout == SDFB200_GRID_TORCH) {
    const uint32_t mask = (1u << g.log2_hashmap_size) - 1u;
    return g.offset[l] + ((ix ^ (iy * kPrimeY) ^ (iz * kPrimeZ)) & mask);
  }
  const uint32_t res = g.resolution[l];
  uint32_t idx = g.hashed[l] ? (ix ^ (iy * kPrimeY) ^ (iz * kPrimeZ)) : (ix + iy * res + iz * res * res);
  return g.offset[l] + idx % g.size[l];
}

}  // namespace sdfb200
