// Host-side layout plan of the packed-weight blob and of the per-chunk workspace of the SDF field.
// Everything is derived deterministically from the sdfb200_field_t descriptor so that sdfb200_field_pack and
// sdfb200_field_forward agree without exchanging any state.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/sdfb200.h"

namespace sdfb200 {

constexpr int kPad = 16;               // every K / N dimension is padded to a multiple of 16 (zero filled)
constexpr int64_t kChunkPoints = 132 * 4 * 128;  // points per pass of the generic path (bounds the workspace): 4 full waves of 128-row tiles on 132 SMs

inline int pad16(int v) { return (v + kPad - 1) / kPad * kPad; }

struct LayerPlan {
  int K, N, Kp, Np;     // logical / padded dims
  size_t w_off;         // [Np, Kp] fp32   (folded weight; skip layer pre-scaled by 1/sqrt(2))
  size_t b_off;         // [Np]     fp32
  size_t wt_off;        // [Kp, Np] fp32   (transposed copy for the reverse sweep; geo layers only, (size_t)-1 if absent)
};

struct FieldPlan {
  int n_geo, n_col;
  LayerPlan geo[SDFB200_MAX_LAYERS], col[SDFB200_MAX_LAYERS];
  int pe_dim, grid_dim, in_dim, in_pad;  // geo input: [x(3) | PE | grid | pad]
  int dir_dim;                           // 27
  int cin_dim, cin_pad;                  // colour input
  int geo_feat;                          // geo_dims[n] - 1
  size_t head_off;                       // diffuse W[3,gf] b[3] tint W[3,gf] b[3] (fp32), (size_t)-1 if neither
  size_t fp32_bytes;                     // size of the fp32 section
  size_t tc_off, tc_bytes;               // tensor-core (bf16 split-plane) section, 0 bytes for PRECISION_FP32
  size_t total_bytes;
};

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// returns 0 on success, negative on an unsupported descriptor
inline int make_field_plan(const sdfb200_field_t& f, FieldPlan& p) {
  if (f.n_geo_linear < 1 || f.n_geo_linear > SDFB200_MAX_LAYERS) return -1;
  if (f.n_color_linear < 1 || f.n_color_linear > SDFB200_MAX_LAYERS) return -1;
  p.n_geo = f.n_geo_linear;
  p.n_col = f.n_color_linear;
  p.pe_dim = (f.off_axis ? 21 : 3) * f.pe_degree * 2;
  p.grid_dim = f.grid.n_levels * f.grid.n_features;
  p.in_dim = 3 + p.pe_dim + p.grid_dim;
  if (f.geo_dims[0] != p.in_dim) return -2;
  p.in_pad = pad16(p.in_dim);
  p.dir_dim = 27;
  p.geo_feat = f.geo_dims[p.n_geo] - 1;
  if (p.geo_feat < 1) return -3;
  int cin = f.use_diffuse_color ? (p.dir_dim + p.geo_feat + f.appearance_dim) : (3 + p.dir_dim + 3 + p.geo_feat + f.appearance_dim);
  if (f.use_n_dot_v) cin += 1;
  if (f.color_dims[0] != cin) return -4;
  p.cin_dim = cin;
  p.cin_pad = pad16(cin);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return o;
  };
  for (int l = 0; l < p.n_geo; ++l) {
    LayerPlan& L = p.geo[l];
    // logical output width of layer l: the layer feeding the skip concat is narrower (sdf_field.py:285-288)
    L.N = (l + 1 == f.geo_skip_layer) ? f.geo_dims[l + 1] - f.geo_dims[0] : f.geo_dims[l + 1];
    L.K = f.geo_dims[l];
    if (l > 0 && l != f.geo_skip_layer && L.K != p.geo[l - 1].N) return -5;
    if (l == f.geo_skip_layer && (l == 0 || L.K != p.geo[l - 1].N + p.in_dim)) return -6;
    if (L.N < 1) return -7;
    L.Kp = pad16(L.K);
    L.Np = pad16(L.N);
    L.w_off = take((size_t)L.Np * L.Kp * 4);
    L.b_off = take((size_t)L.Np * 4);
    L.wt_off = take((size_t)L.Kp * L.Np * 4);
  }
  for (int l = 0; l < p.n_col; ++l) {
    LayerPlan& L = p.col[l];
    L.K = f.color_dims[l];
    L.N = f.color_dims[l + 1];
    L.Kp = pad16(L.K);
    L.Np = pad16(L.N);
    L.w_off = take((size_t)L.Np * L.Kp * 4);
    L.b_off = take((size_t)L.Np * 4);
    L.wt_off = (size_t)-1;
  }
  if (p.col[p.n_col - 1].N != 3) return -8;
  p.head_off = (size_t)-1;
  if (f.use_diffuse_color || f.use_specular_tint) p.head_off = take((size_t)(2 * (3 * p.geo_feat + 4)) * 4);
  p.fp32_bytes = off;
  p.tc_off = off;
  p.tc_bytes = 0;
  p.total_bytes = off;
  return 0;
}

// ---- per-chunk workspace (floats), generic fp32 path ----
struct FieldWorkspace {
  size_t x, x01, in, jac, h[SDFB200_MAX_LAYERS], outg, g0, g1, gin, cin, c0, c1, sdf, grad, nsdf;
  size_t tcw;            // packed weight planes of one tensor-core GEMM chunk (fixed size, csrc/tc_linear.h)
  size_t floats_per_chunk;
};

inline void make_workspace_plan(const sdfb200_field_t& f, const FieldPlan& p, int64_t chunk, FieldWorkspace& w) {
  size_t off = 0;
  auto take = [&](size_t per_point) {
    size_t o = off;
    off = align_up(off + per_point * (size_t)chunk, 64);
    return o;
  };
  int maxw = p.in_pad;
  for (int l = 0; l < p.n_geo; ++l) {
    if (p.geo[l].Np > maxw) maxw = p.geo[l].Np;
    if (p.geo[l].Kp > maxw) maxw = p.geo[l].Kp;
  }
  int maxc = p.cin_pad;
  for (int l = 0; l < p.n_col; ++l) maxc = p.col[l].Np > maxc ? p.col[l].Np : maxc;
  w.x = take(3);
  w.x01 = take(3);
  w.in = take(p.in_pad);
  w.jac = take((size_t)p.grid_dim * 3);
  for (int l = 0; l < p.n_geo - 1; ++l) w.h[l] = take(l + 1 == f.geo_skip_layer ? p.geo[l + 1].Kp : p.geo[l].Np);
  w.outg = take(p.geo[p.n_geo - 1].Np);
  w.g0 = take(maxw);
  w.g1 = take(maxw);
  w.gin = take(p.in_pad);
  w.cin = take(p.cin_pad);
  w.c0 = take(maxc);
  w.c1 = take(maxc);
  w.sdf = take(1);
  w.grad = take(3);
  w.nsdf = take(6);
  w.tcw = off;
  off = align_up(off + 65536, 64);   // kTcGemmScratchBytes / 4
  w.floats_per_chunk = off;
}

}  // namespace sdfb200
