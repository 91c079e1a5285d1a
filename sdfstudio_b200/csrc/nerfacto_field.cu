// Nerfacto background field: the C-ABI entry point and the fp32-table instantiation of k_nerfacto_field (nerfacto_field.cuh).
#include "nerfacto_field.cuh"

namespace sdfb200 {

int launch_nerfacto_f32(const NerfactoArgs& a, int h, int hc, cudaStream_t st) { return launch_nerfacto_h<float>(a, h, hc, st); }

static bool width_ok(int w) { return w == 16 || w == 32 || w == 64; }

}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_nerfacto_field_forward(const sdfb200_grid_t* grid, const sdfb200_nerfacto_t* f, const void* table, const float* base_weights,
                                              const float* head_weights, const float* aabb, const float* origins, const float* directions,
                                              const float* bins, int64_t n_rays, const float* appearance, int64_t appearance_stride, float* density,
                                              float* rgb, float* pre_activation, float* geo_feature, void* stream) {
  SDFB_REQUIRE(grid && f, "NULL descriptor");
  int r = validate_grid(grid);
  if (r) return r;
  if (grid->layout != SDFB200_GRID_TCNN || grid->n_features != 2)
    return fail(SDFB200_EUNSUPPORTED, "nerfacto field: the grid must be tcnn layout with 2 features per level%s", "", 0);
  if (!width_ok(f->hidden_dim) || !width_ok(f->hidden_dim_color))
    return fail(SDFB200_EUNSUPPORTED, "nerfacto field: hidden_dim and hidden_dim_color must be 16, 32 or 64%s", "", 0);
  if (f->n_hidden_layers < 1 || f->n_hidden_layers > 3 || f->n_hidden_layers_color < 1 || f->n_hidden_layers_color > 3)
    return fail(SDFB200_EUNSUPPORTED, "nerfacto field: num_layers and num_layers_color must be 2, 3 or 4%s", "", 0);
  if (f->geo_feat_dim < 0 || f->geo_feat_dim > 15 || f->appearance_dim < 0 || 16 + f->geo_feat_dim + f->appearance_dim > 64)
    return fail(SDFB200_EUNSUPPORTED, "nerfacto field: needs geo_feat_dim <= 15 and 16 + geo_feat_dim + appearance_dim <= 64%s", "", 0);
  SDFB_REQUIRE(f->contraction >= SDFB200_CONTRACT_NONE && f->contraction <= SDFB200_CONTRACT_L2, "contraction");
  SDFB_REQUIRE(f->n_samples >= 0 && n_rays >= 0 && appearance_stride >= 0, "bad sizes");
  const int64_t n = f->n_samples ? n_rays * f->n_samples : n_rays;
  if (n == 0) return 0;
  SDFB_REQUIRE(table && base_weights && origins && density, "NULL pointer");
  r = validate_grid_pointers(grid, table, nullptr);
  if (r) return r;
  SDFB_REQUIRE(f->n_samples == 0 || (bins != nullptr && directions != nullptr), "ray mode needs bins and directions (the midpoints use them)");
  if (rgb) SDFB_REQUIRE(head_weights != nullptr && directions != nullptr, "rgb needs head_weights and directions");
  NerfactoArgs a;
  a.grid = *grid; a.table = table; a.base_w = base_weights; a.head_w = head_weights; a.aabb = aabb;
  a.origins = origins; a.directions = directions; a.bins = f->n_samples ? bins : nullptr;
  a.appearance = f->appearance_dim > 0 ? appearance : nullptr; a.app_stride = appearance_stride;
  a.contraction = f->contraction; a.n_base = f->n_hidden_layers; a.n_head = f->n_hidden_layers_color;
  a.in_pad = (grid->n_levels * grid->n_features + 15) / 16 * 16;
  a.head_pad = (16 + f->geo_feat_dim + f->appearance_dim + 15) / 16 * 16;
  a.geo_dim = f->geo_feat_dim; a.app_dim = f->appearance_dim; a.S = f->n_samples; a.n = n;
  a.density = density; a.rgb = rgb; a.pre_activation = pre_activation; a.geo_feature = geo_feature;
  cudaStream_t st = (cudaStream_t)stream;
  return grid->table_dtype == SDFB200_DT_F16 ? launch_nerfacto_f16(a, f->hidden_dim, f->hidden_dim_color, st)
                                             : launch_nerfacto_f32(a, f->hidden_dim, f->hidden_dim_color, st);
}
