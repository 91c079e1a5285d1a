// Host side of the fused tensor-core field kernel (csrc/field_tc_kernel.cuh): which descriptors it runs and its part of the packed-weight
// plan, weight packing (tc_pack, tc_linear.cu), launch dispatch.  See field_tc_kernel.cuh for the kernel itself.
#include "field.h"
#include "field_tc.h"
#include "tc_common.cuh"
#include "tc_linear.h"

namespace sdfb200 {
using namespace tc;
static_assert(sizeof(TcIdxMap) == kInK * sizeof(short), "one index map entry per column of the small-K operands");

// colour layer 0 pre-multiplied with the (activation-free) last geo layer: Wc[o][k] = sum_j Wc0[o][33+j] W2[1+j][k],
// bias[o] = bc0[o] + sum_j Wc0[o][33+j] b2[1+j]        (sdf_field.py:406-410 feeds :576-592)
__global__ void k_fuse_c0(const float* __restrict__ Wc0, int ldc0, const float* __restrict__ bc0, const float* __restrict__ W2, int ld2,
                          const float* __restrict__ b2, float* __restrict__ Wc, float* __restrict__ bc) {
  __shared__ float wrow[256];
  const int o = blockIdx.x, k = threadIdx.x;
  wrow[k] = Wc0[(size_t)o * ldc0 + 33 + k];
  __syncthreads();
  float acc = 0.f;
  for (int j = 0; j < 256; ++j) acc = fmaf(wrow[j], W2[(size_t)(1 + j) * ld2 + k], acc);
  Wc[o * 256 + k] = acc;
  if (k == 0) {
    float b = bc0[o];
    for (int j = 0; j < 256; ++j) b = fmaf(wrow[j], b2[1 + j], b);
    bc[o] = b;
  }
}

// -----------------------------------------------------------------------------------------------------------------
// host side
// -----------------------------------------------------------------------------------------------------------------
// the neus-facto shape family at a tensor-core precision; everything else runs the generic kernels
static bool fused_family(const sdfb200_field_t& f, const FieldPlan& p) {
  if (f.precision != SDFB200_PRECISION_BF16X3 && f.precision != SDFB200_PRECISION_BF16) return false;
  if (p.n_geo != 3 || p.n_col != 3) return false;
  if (p.geo[0].N != 256 || p.geo[1].N != 256 || p.geo_feat != 256 || p.col[0].N != 256 || p.col[1].N != 256) return false;
  if (f.use_numerical_gradients || f.off_axis || f.use_diffuse_color || f.use_specular_tint || f.use_reflections) return false;
  if (p.grid_dim > kMaxGridDim || p.pe_dim > kMaxPe || 32 + p.pe_dim + 3 > kInK) return false;
  if (f.pe_degree < 1) return false;
  if (f.use_grid_feature && f.grid.n_features != 2) return false;
  if (38 + f.appearance_dim > kInK) return false;
  return true;
}

void plan_tc_section(const sdfb200_field_t& f, FieldPlan& p) {
  p.fused = fused_family(f, p);
  p.tc_bytes = 0;
  if (!p.fused) return;
  const int planes = tc_planes(f.precision);
  size_t off = p.tc_off;
  for (int l = 0; l < L_COUNT; ++l) {
    p.tc_w_off[l] = off;
    off = align_up(off + (size_t)tc_layer_nkb(l) * tc_stage_bytes(planes), 256);
  }
  p.tc_wc_off = off;
  off = align_up(off + 256 * 256 * 4, 256);
  p.tc_bc_off = off;
  off = align_up(off + 256 * 4, 256);
  p.tc_bytes = off - p.tc_off;
}

size_t field_tc_workspace_floats(const sdfb200_field_t& f) { return kNumSMs * kScratchPerCta(tc_planes(f.precision)) / sizeof(float); }

int field_tc_pack(const sdfb200_field_t& f, const FieldPlan& p, char* blob, cudaStream_t st) {
  const int planes = tc_planes(f.precision);
  auto pack = [&](int L, const float* W, int ldw, int N, int K, const TcIdxMap* colmap, const TcIdxMap* rowmap) -> int {
    return tc_pack(W, ldw, 0, N, K, tc_layer_np(L), tc_layer_kblk(L), tc_layer_nkb(L), planes, rowmap, colmap, blob + p.tc_w_off[L], st);
  };
  const LayerPlan &g0 = p.geo[0], &g1 = p.geo[1], &g2 = p.geo[2], &c0 = p.col[0], &c1 = p.col[1];
  // geo input, kernel column order [grid(32) | PE | x | 0]  <-  reference order [x(3) | PE | grid]  (sdf_field.py:391-396)
  TcIdxMap gin;
  for (int i = 0; i < kInK; ++i) gin.src[i] = -1;
  for (int i = 0; i < p.grid_dim; ++i) gin.src[i] = (short)(3 + p.pe_dim + i);
  for (int i = 0; i < p.pe_dim; ++i) gin.src[32 + i] = (short)(3 + i);
  for (int i = 0; i < 3; ++i) gin.src[32 + p.pe_dim + i] = (short)i;
  int r;
  if ((r = pack(L_G0, (const float*)(blob + g0.w_off), g0.Kp, 256, g0.K, &gin, nullptr))) return r;
  if ((r = pack(L_G1, (const float*)(blob + g1.w_off), g1.Kp, 256, 256, nullptr, nullptr))) return r;
  if ((r = pack(L_B1, (const float*)(blob + g1.wt_off), g1.Np, 256, 256, nullptr, nullptr))) return r;          // W1^T: [in][out]
  if ((r = pack(L_B0, (const float*)(blob + g0.wt_off), g0.Np, g0.K, 256, nullptr, &gin))) return r;            // W0^T: rows = input index (kernel order)
  // colour layer 0 (sdf_field.py:572-584): reference input = [x(3) dir(27) grad(3) | geo feature(256) | appearance | n.v]
  k_fuse_c0<<<256, 256, 0, st>>>((const float*)(blob + c0.w_off), c0.Kp, (const float*)(blob + c0.b_off), (const float*)(blob + g2.w_off), g2.Kp,
                                 (const float*)(blob + g2.b_off), (float*)(blob + p.tc_wc_off), (float*)(blob + p.tc_bc_off));
  SDFB_LAUNCHED("k_fuse_c0");
  if ((r = pack(L_C0H, (const float*)(blob + p.tc_wc_off), 256, 256, 256, nullptr, nullptr))) return r;
  // misc operand, kernel order: chunk 0 = [grad(3), n.v, 0 x4] (written per tile by the epilogue), then the static part
  // [x(3), dir-enc(27), appearance] prepared by the gather warps
  TcIdxMap cm;
  for (int i = 0; i < kInK; ++i) cm.src[i] = -1;
  cm.src[0] = 30; cm.src[1] = 31; cm.src[2] = 32;
  if (f.use_n_dot_v) cm.src[3] = (short)(289 + f.appearance_dim);
  for (int i = 0; i < 30; ++i) cm.src[8 + i] = (short)i;
  for (int i = 0; i < f.appearance_dim; ++i) cm.src[38 + i] = (short)(289 + i);
  if ((r = pack(L_C0MISC, (const float*)(blob + c0.w_off), c0.Kp, 256, kInK, &cm, nullptr))) return r;
  if ((r = pack(L_C1, (const float*)(blob + c1.w_off), c1.Kp, 256, 256, nullptr, nullptr))) return r;
  return 0;
}

int field_tc_forward(const sdfb200_field_t& f, const FieldPlan& p, const char* blob, const void* table, const sdfb200_field_in_t& in,
                     const sdfb200_field_out_t& out, const sdfb200_field_render_t* rnd, float* ws, cudaStream_t st) {
  const int64_t N = in.n_rays * (int64_t)in.n_samples;
  const int planes = tc_planes(f.precision);
  const bool render = rnd != nullptr;
  const bool sdf_only = !render && out.sdf && !out.gradients && !out.normals && !out.rgb && !out.density && !out.alpha && !out.occupancy;
  TcArgs a;
  a.grid = f.grid;
  for (int l = 0; l < L_COUNT; ++l) a.layer[l].w_off = p.tc_w_off[l];
  a.use_grid = f.use_grid_feature; a.pe_degree = f.pe_degree; a.use_pe = f.use_position_encoding;
  a.contraction = in.apply_contraction ? f.contraction : SDFB200_CONTRACT_NONE;
  a.pe_dim = p.pe_dim; a.grid_dim = p.grid_dim; a.app_dim = f.appearance_dim; a.use_n_dot_v = f.use_n_dot_v;
  a.mode = sdf_only ? 0 : 1;
  a.n_samples = in.n_samples; a.has_bins = in.bins != nullptr; a.n_points = N; a.n_tiles = (int)ceil_div(N, 128);
  a.rgb_padding = f.rgb_padding; a.cos_anneal = in.cos_anneal_ratio;
  a.origins = in.origins; a.directions = in.directions; a.bins = in.bins; a.appearance = in.appearance; a.variance = in.variance; a.beta = in.beta;
  a.beta_min = in.beta_min; a.table = table; a.blob = blob;
  a.b_g0 = p.geo[0].b_off; a.b_g1 = p.geo[1].b_off; a.b_g2 = p.geo[2].b_off; a.w_g2 = p.geo[2].w_off;
  a.b_c0 = p.tc_bc_off; a.b_c1 = p.col[1].b_off; a.w_c2 = p.col[2].w_off; a.b_c2 = p.col[2].b_off;
  a.scratch = reinterpret_cast<char*>(ws); a.out = out;
  a.render = render;
  a.rnd = render ? *rnd : sdfb200_field_render_t{};
  // persistent CTAs, one per SM (the static tile loop needs no co-residency, but more CTAs than SMs would only add a tail wave)
  const int ctas = persistent_ctas();
  const int grid = a.n_tiles < ctas ? a.n_tiles : ctas;
  const size_t smem = tc_smem(planes).bytes;
  const bool torch_layout = f.grid.layout == SDFB200_GRID_TORCH;
  if (planes == 2) return torch_layout ? launch_field_tc_p2_torch(a, grid, smem, st) : launch_field_tc_p2_tcnn(a, grid, smem, st);
  return torch_layout ? launch_field_tc_p1_torch(a, grid, smem, st) : launch_field_tc_p1_tcnn(a, grid, smem, st);
}

}  // namespace sdfb200
