// The C-ABI entry points of the tiny-cuda-nn NetworkWithInputEncoding fields and the fp32-table instantiations of k_hash_mlp_field
// (hash_mlp.cuh):
//   sdfb200_density_field_forward: the proposal density field (HashMLPDensityField.get_density / density_fn,
//     nerfstudio/fields/density_fields.py:40-121, fields/base_field.py:48-65), the density half alone in point mode;
//   sdfb200_nerfacto_field_forward: the grid background field (TCNNNerfactoField.forward, nerfstudio/fields/nerfacto_field.py:223-318
//     through fields/base_field.py:104-123), both halves in ray or point mode.
#include "hash_mlp.cuh"

namespace sdfb200 {

static bool width_ok(int w) { return w == 16 || w == 32 || w == 64; }

static int launch_field(const HashMlpArgs& a, int h, int hc, cudaStream_t st) {
  return a.grid.table_dtype == SDFB200_DT_F16 ? launch_hash_mlp_f16(a, h, hc, st) : launch_hash_mlp_t<float>(a, h, hc, st);
}

}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_density_field_forward(const sdfb200_grid_t* grid, const void* table, const float* weights, int32_t hidden_dim,
                                             int32_t n_hidden_layers, int32_t contraction, const float* aabb, const float* positions, int64_t n,
                                             float* density, float* pre_activation, void* stream) {
  int r = validate_grid(grid);
  if (r) return r;
  SDFB_REQUIRE(n >= 0, "n < 0");
  if (n == 0) return 0;
  SDFB_REQUIRE(table && weights && positions && density, "NULL pointer");
  SDFB_REQUIRE(n_hidden_layers >= 1 && n_hidden_layers <= 4, "n_hidden_layers out of range");
  SDFB_REQUIRE(grid->n_features == 2 || grid->n_features == 4 || grid->n_features == 1 || grid->n_features == 8, "n_features");
  r = validate_grid_pointers(grid, table, nullptr);
  if (r) return r;
  if (!width_ok(hidden_dim)) return fail(SDFB200_EUNSUPPORTED, "density field hidden_dim must be 16, 32 or 64%s", "", 0);
  HashMlpArgs a{};
  a.grid = *grid; a.table = table; a.base_w = weights; a.aabb = aabb; a.origins = positions;
  a.contraction = contraction; a.n_base = n_hidden_layers; a.in_pad = (grid->n_levels * grid->n_features + 15) / 16 * 16; a.n = n;
  a.density = density; a.pre_activation = pre_activation;
  return launch_field(a, hidden_dim, 0, (cudaStream_t)stream);
}

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
  HashMlpArgs a;
  a.grid = *grid; a.table = table; a.base_w = base_weights; a.head_w = head_weights; a.aabb = aabb;
  a.origins = origins; a.directions = directions; a.bins = f->n_samples ? bins : nullptr;
  a.appearance = f->appearance_dim > 0 ? appearance : nullptr; a.app_stride = appearance_stride;
  a.contraction = f->contraction; a.n_base = f->n_hidden_layers; a.n_head = f->n_hidden_layers_color;
  a.in_pad = (grid->n_levels * grid->n_features + 15) / 16 * 16;
  a.head_pad = (16 + f->geo_feat_dim + f->appearance_dim + 15) / 16 * 16;
  a.geo_dim = f->geo_feat_dim; a.app_dim = f->appearance_dim; a.S = f->n_samples; a.n = n;
  a.density = density; a.rgb = rgb; a.pre_activation = pre_activation; a.geo_feature = geo_feature;
  return launch_field(a, f->hidden_dim, f->hidden_dim_color, (cudaStream_t)stream);
}
