// Host side of the fused tensor-core field kernel (csrc/field_tc_kernel.cuh): packed-weight plan, weight packing (tc_pack,
// tc_linear.cu), launch dispatch.  See field_tc_kernel.cuh for the kernel itself.
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
struct TcPlan {
  int planes;
  TcLayer layer[L_COUNT];
  size_t total, wc_off, bc_off;
};

static void make_tc_plan(const sdfb200_field_t& f, const FieldPlan& p, TcPlan& t) {
  t.planes = f.precision == SDFB200_PRECISION_BF16X3 ? 2 : 1;
  size_t off = p.tc_off;
  for (int l = 0; l < L_COUNT; ++l) {
    t.layer[l].w_off = off;
    off = align_up(off + (size_t)tc_layer_nkb(l) * tc_stage_bytes(t.planes), 256);
  }
  t.wc_off = off;                       // fp32 [256][256]: Wgf * W2[1:,:]   (colour layer 0 applied to h2 directly)
  off = align_up(off + 256 * 256 * 4, 256);
  t.bc_off = off;                       // fp32 [256]: bc0 + Wgf * b2[1:]
  off = align_up(off + 256 * 4, 256);
  t.total = off - p.tc_off;
}

bool field_tc_supported(const sdfb200_field_t& f, const FieldPlan& p) {
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

// fused compositing needs whole rays inside a 128-point tile
bool field_tc_render_supported(const sdfb200_field_t& f, const FieldPlan& p, int n_samples) {
  return field_tc_supported(f, p) && n_samples >= 1 && n_samples <= 128 && (128 % n_samples) == 0;
}

size_t field_tc_packed_bytes(const sdfb200_field_t& f, const FieldPlan& p) {
  TcPlan t;
  make_tc_plan(f, p, t);
  return t.total;
}

size_t field_tc_workspace_floats(const sdfb200_field_t& f, const FieldPlan&, int64_t) {
  const int planes = f.precision == SDFB200_PRECISION_BF16X3 ? 2 : 1;
  return kNumSMs * kScratchPerCta(planes) / sizeof(float) + 64;
}

int field_tc_pack(const sdfb200_field_t& f, const FieldPlan& p, char* blob, cudaStream_t st) {
  TcPlan t;
  make_tc_plan(f, p, t);
  auto pack = [&](int L, const float* W, int ldw, int N, int K, const TcIdxMap* colmap, const TcIdxMap* rowmap) -> int {
    return tc_pack(W, ldw, 0, N, K, tc_layer_np(L), tc_layer_kblk(L), tc_layer_nkb(L), t.planes, rowmap, colmap, blob + t.layer[L].w_off, st);
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
                                 (const float*)(blob + g2.b_off), (float*)(blob + t.wc_off), (float*)(blob + t.bc_off));
  SDFB_LAUNCHED("k_fuse_c0");
  if ((r = pack(L_C0H, (const float*)(blob + t.wc_off), 256, 256, 256, nullptr, nullptr))) return r;
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
                     const sdfb200_field_out_t& out, const sdfb200_field_render_t* rnd, float* ws, size_t ws_floats, cudaStream_t st) {
  const int64_t N = in.n_rays * (int64_t)in.n_samples;
  if (N == 0) return 0;
  TcPlan t;
  make_tc_plan(f, p, t);
  const size_t per_cta = kScratchPerCta(t.planes);
  if (ws_floats * sizeof(float) < (size_t)kNumSMs * per_cta) return fail(SDFB200_EWORKSPACE, "workspace too small for the tensor-core path%s", "", 0);
  SDFB_REQUIRE(out.geo_feature == nullptr, "geo_feature is not produced by the tensor-core path (use precision fp32)");
  const bool render = rnd != nullptr;
  const bool sdf_only = !render && out.sdf && !out.gradients && !out.normals && !out.rgb && !out.density && !out.alpha && !out.occupancy;
  if (!sdf_only) {
    if (out.rgb || out.alpha || render) SDFB_REQUIRE(in.directions != nullptr, "directions required for rgb / alpha");
    if (out.alpha || (render && !rnd->from_density)) SDFB_REQUIRE(in.bins != nullptr && in.variance != nullptr, "alpha needs bins and the variance parameter");
    if (out.density || (render && rnd->from_density)) SDFB_REQUIRE(in.beta != nullptr && in.beta_min != nullptr, "density needs beta and beta_min");
  }
  if (render) SDFB_REQUIRE(in.bins != nullptr && (128 % in.n_samples) == 0, "fused compositing needs bins and 128 % n_samples == 0");
  SDFB_REQUIRE(out.sampled_sdf == nullptr, "sampled_sdf is only produced with use_numerical_gradients");
  TcArgs a;
  a.grid = f.grid;
  for (int l = 0; l < L_COUNT; ++l) a.layer[l] = t.layer[l];
  a.use_grid = f.use_grid_feature; a.pe_degree = f.pe_degree; a.use_pe = f.use_position_encoding;
  a.contraction = in.apply_contraction ? f.contraction : SDFB200_CONTRACT_NONE;
  a.pe_dim = p.pe_dim; a.grid_dim = p.grid_dim; a.app_dim = f.appearance_dim; a.use_n_dot_v = f.use_n_dot_v;
  a.mode = sdf_only ? 0 : 1;
  a.n_samples = in.n_samples; a.has_bins = in.bins != nullptr; a.n_points = N; a.n_tiles = (int)ceil_div(N, 128);
  a.rgb_padding = f.rgb_padding; a.cos_anneal = in.cos_anneal_ratio;
  a.origins = in.origins; a.directions = in.directions; a.bins = in.bins; a.appearance = in.appearance; a.variance = in.variance; a.beta = in.beta;
  a.beta_min = in.beta_min; a.table = table; a.blob = blob;
  a.b_g0 = p.geo[0].b_off; a.b_g1 = p.geo[1].b_off; a.b_g2 = p.geo[2].b_off; a.w_g2 = p.geo[2].w_off;
  a.b_c0 = t.bc_off; a.b_c1 = p.col[1].b_off; a.w_c2 = p.col[2].w_off; a.b_c2 = p.col[2].b_off;
  a.scratch = reinterpret_cast<char*>(ws); a.out = out;
  a.render = render;
  a.rnd = render ? *rnd : sdfb200_field_render_t{};
  // persistent CTAs, one per SM (the static tile loop needs no co-residency, but more CTAs than SMs would only add a tail wave)
  const int ctas = persistent_ctas();
  const int grid = a.n_tiles < ctas ? a.n_tiles : ctas;
  const size_t smem = tc_smem(t.planes).bytes;
  const bool torch_layout = f.grid.layout == SDFB200_GRID_TORCH;
  if (t.planes == 2) return torch_layout ? launch_field_tc_p2_torch(a, grid, smem, st) : launch_field_tc_p2_tcnn(a, grid, smem, st);
  return torch_layout ? launch_field_tc_p1_torch(a, grid, smem, st) : launch_field_tc_p1_tcnn(a, grid, smem, st);
}

}  // namespace sdfb200
