// extern "C" entry points of the field (pack / forward) + library bookkeeping.  See include/sdfb200.h.
#include "common.cuh"
#include "field_plan.h"
#include "tc_linear.h"

#include <string.h>

namespace sdfb200 {
thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

int validate_grid(const sdfb200_grid_t* g);
int field_pack_fp32(const sdfb200_field_t& f, const FieldPlan& p, const sdfb200_field_params_t& prm, char* blob, cudaStream_t st);
int field_forward_fp32(const sdfb200_field_t& f, const FieldPlan& p, const char* blob, const void* table, const sdfb200_field_in_t& in,
                       const sdfb200_field_out_t& out, float* ws, size_t ws_floats, cudaStream_t st, int gemm_planes);
// tensor-core path (field_tc.cu)
size_t field_tc_packed_bytes(const sdfb200_field_t& f, const FieldPlan& p);
bool field_tc_supported(const sdfb200_field_t& f, const FieldPlan& p);
int field_tc_pack(const sdfb200_field_t& f, const FieldPlan& p, char* blob, cudaStream_t st);
bool field_tc_render_supported(const sdfb200_field_t& f, const FieldPlan& p, int n_samples);
int field_tc_forward(const sdfb200_field_t& f, const FieldPlan& p, const char* blob, const void* table, const sdfb200_field_in_t& in,
                     const sdfb200_field_out_t& out, const sdfb200_field_render_t* rnd, float* ws, size_t ws_floats, cudaStream_t st);
size_t field_tc_workspace_floats(const sdfb200_field_t& f, const FieldPlan& p, int64_t n_points);

static int plan_or_fail(const sdfb200_field_t* f, FieldPlan& p) {
  SDFB_REQUIRE(f != nullptr, "field descriptor is NULL");
  if (f->use_grid_feature) {
    int r = validate_grid(&f->grid);
    if (r) return r;
  } else {
    SDFB_REQUIRE(f->grid.n_levels >= 1 && f->grid.n_levels <= SDFB200_MAX_LEVELS && f->grid.n_features >= 1, "grid dims (needed for the zero feature block)");
  }
  SDFB_REQUIRE(f->pe_degree >= 0 && f->pe_degree <= 16, "pe_degree out of range");
  SDFB_REQUIRE(f->appearance_dim >= 0 && f->appearance_dim <= 256, "appearance_dim out of range");
  const int rc = make_field_plan(*f, p);
  if (rc) return fail(SDFB200_EINVAL, "inconsistent field descriptor%s (plan error %lld)", "", (long long)rc);
  // tensor-core precisions: the fused kernel (field_tc.cu) for the neus-facto shape family, otherwise the generic kernels with the
  // tensor-core Linear (tc_linear.cu) as their GEMM engine -- no extra packed section for the latter
  if (f->precision != SDFB200_PRECISION_FP32 && field_tc_supported(*f, p)) {
    p.tc_bytes = field_tc_packed_bytes(*f, p);
    p.total_bytes = p.tc_off + p.tc_bytes;
  }
  return 0;
}
}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_version(void) { return SDFB200_VERSION; }
extern "C" const char* sdfb200_last_error_string(void) { return g_err; }
extern "C" int64_t sdfb200_launch_count(void) { return (int64_t)g_launches.load(); }
extern "C" size_t sdfb200_struct_size(int32_t which) {
  switch (which) {
    case 0: return sizeof(sdfb200_grid_t);
    case 1: return sizeof(sdfb200_field_t);
    case 2: return sizeof(sdfb200_field_params_t);
    case 3: return sizeof(sdfb200_field_in_t);
    case 4: return sizeof(sdfb200_field_out_t);
    case 5: return sizeof(sdfb200_render_out_t);
    case 6: return sizeof(sdfb200_field_render_t);
    default: return 0;
  }
}

extern "C" size_t sdfb200_field_packed_bytes(const sdfb200_field_t* f) {
  FieldPlan p;
  if (plan_or_fail(f, p)) return 0;
  return p.total_bytes;
}

extern "C" int sdfb200_field_pack(const sdfb200_field_t* f, const sdfb200_field_params_t* prm, void* packed, void* stream) {
  FieldPlan p;
  int r = plan_or_fail(f, p);
  if (r) return r;
  SDFB_REQUIRE(prm != nullptr && packed != nullptr, "NULL pointer");
  r = field_pack_fp32(*f, p, *prm, (char*)packed, (cudaStream_t)stream);
  if (r) return r;
  if (f->precision != SDFB200_PRECISION_FP32 && p.tc_bytes > 0) return field_tc_pack(*f, p, (char*)packed, (cudaStream_t)stream);
  return 0;
}

extern "C" size_t sdfb200_field_workspace_bytes(const sdfb200_field_t* f, int64_t n_points) {
  FieldPlan p;
  if (plan_or_fail(f, p) || n_points < 0) return 0;
  if (n_points == 0) return 256;
  FieldWorkspace w;
  make_workspace_plan(*f, p, n_points < kChunkPoints ? n_points : kChunkPoints, w);
  size_t floats = w.floats_per_chunk;
  if (f->precision != SDFB200_PRECISION_FP32 && p.tc_bytes > 0) {
    const size_t t = field_tc_workspace_floats(*f, p, n_points);
    floats = t > floats ? t : floats;
  }
  return floats * sizeof(float) + 256;
}

extern "C" int sdfb200_field_forward(const sdfb200_field_t* f, const void* packed, const void* table, const sdfb200_field_in_t* in,
                                     const sdfb200_field_out_t* out, void* workspace, size_t workspace_bytes, void* stream) {
  FieldPlan p;
  int r = plan_or_fail(f, p);
  if (r) return r;
  SDFB_REQUIRE(packed && in && out, "NULL pointer");
  SDFB_REQUIRE(in->n_rays >= 0 && in->n_samples >= 1, "bad sizes");
  if (in->n_rays == 0) return 0;
  SDFB_REQUIRE(in->origins != nullptr, "origins is NULL");
  SDFB_REQUIRE(in->bins != nullptr || in->n_samples == 1, "point mode requires n_samples == 1");
  SDFB_REQUIRE(in->bins == nullptr || in->directions != nullptr, "ray mode requires directions");
  SDFB_REQUIRE(!f->use_grid_feature || table != nullptr, "grid table is NULL");
  SDFB_REQUIRE(workspace != nullptr, "workspace is NULL");
  uintptr_t wsp = ((uintptr_t)workspace + 255) & ~(uintptr_t)255;
  const size_t lost = wsp - (uintptr_t)workspace;
  SDFB_REQUIRE(workspace_bytes > lost, "workspace too small");
  const size_t ws_floats = (workspace_bytes - lost) / sizeof(float);
  // the tensor-core kernel never materialises the geo feature (colour layer 0 is pre-multiplied with the last geo layer);
  // the rare callers that want it (forward_geonetwork) take the exact-fp32 kernels, which read the same packed blob
  const bool fused = p.tc_bytes > 0;
  if (f->precision != SDFB200_PRECISION_FP32 && fused && out->geo_feature == nullptr)
    return field_tc_forward(*f, p, (const char*)packed, table, *in, *out, nullptr, (float*)wsp, ws_floats, (cudaStream_t)stream);
  // shapes outside the fused family run the generic kernels with tensor-core GEMMs; the fused family's geo-feature requests keep
  // the exact-fp32 engine (unchanged behaviour)
  // numerical gradients divide sdf differences by 2 delta (~1e-3): they need the sdf to fp32 accuracy, which 2^-16-relative GEMMs do not
  // give (measured: gradient error 6e-3 vs 5e-4 of fp32 noise on the angelo-shaped case) -> those fields keep the exact engine
  const int gemm_planes = (f->precision != SDFB200_PRECISION_FP32 && !fused && !f->use_numerical_gradients)
                              ? (f->precision == SDFB200_PRECISION_BF16 ? 1 : 2) : 0;
  return field_forward_fp32(*f, p, (const char*)packed, table, *in, *out, (float*)wsp, ws_floats, (cudaStream_t)stream, gemm_planes);
}

// ---------------------------------------------------------------------------------------------------------------------
// field + compositing in one call.  Fused into the tensor-core kernel when every 128-point tile holds whole rays; otherwise the
// same result is composed from sdfb200_field_forward + the compositing kernels (per-sample heads staged in the workspace).
// ---------------------------------------------------------------------------------------------------------------------
static size_t render_stage_floats(int64_t n_points) { return (size_t)n_points * 9 + 64; }   // alpha|density, rgb(3), normals(3), weights, transmittance

extern "C" size_t sdfb200_field_render_workspace_bytes(const sdfb200_field_t* f, int64_t n_rays, int32_t n_samples) {
  if (n_rays < 0 || n_samples < 1) return 0;
  const int64_t n = n_rays * (int64_t)n_samples;
  const size_t base = sdfb200_field_workspace_bytes(f, n);
  if (base == 0) return 0;
  FieldPlan p;
  if (plan_or_fail(f, p)) return 0;
  const bool fused = f->precision != SDFB200_PRECISION_FP32 && p.tc_bytes > 0 && field_tc_render_supported(*f, p, n_samples);
  return base + (fused ? 0 : render_stage_floats(n) * sizeof(float)) + 256;
}

extern "C" int sdfb200_field_render(const sdfb200_field_t* f, const void* packed, const void* table, const sdfb200_field_in_t* in,
                                    const sdfb200_field_out_t* sample_out, const sdfb200_field_render_t* rnd, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  FieldPlan p;
  int r = plan_or_fail(f, p);
  if (r) return r;
  SDFB_REQUIRE(packed && in && rnd, "NULL pointer");
  SDFB_REQUIRE(in->n_rays >= 0 && in->n_samples >= 1, "bad sizes");
  if (in->n_rays == 0) return 0;
  SDFB_REQUIRE(in->origins && in->directions && in->bins, "field_render needs origins, directions and bins");
  SDFB_REQUIRE(!f->use_grid_feature || table != nullptr, "grid table is NULL");
  SDFB_REQUIRE(workspace != nullptr, "workspace is NULL");
  if (rnd->out.rgb) SDFB_REQUIRE(rnd->bg_mode == SDFB200_BG_LAST_SAMPLE || rnd->bg != nullptr, "rgb output needs a background");
  if (rnd->out.depth) SDFB_REQUIRE(rnd->out.steps_minmax != nullptr, "depth output needs steps_minmax (pre-set to {+inf,-inf})");
  sdfb200_field_out_t so;
  if (sample_out) so = *sample_out; else memset(&so, 0, sizeof(so));
  uintptr_t wsp = ((uintptr_t)workspace + 255) & ~(uintptr_t)255;
  const size_t lost = wsp - (uintptr_t)workspace;
  SDFB_REQUIRE(workspace_bytes > lost, "workspace too small");
  const size_t ws_floats = (workspace_bytes - lost) / sizeof(float);
  const int64_t N = in->n_rays * (int64_t)in->n_samples;
  const bool fused = f->precision != SDFB200_PRECISION_FP32 && p.tc_bytes > 0 && so.geo_feature == nullptr &&
                     field_tc_render_supported(*f, p, in->n_samples);
  if (fused) {
    r = field_tc_forward(*f, p, (const char*)packed, table, *in, so, rnd, (float*)wsp, ws_floats, (cudaStream_t)stream);
    if (r) return r;
  } else {
    const size_t stage = render_stage_floats(N);
    SDFB_REQUIRE(ws_floats > stage, "workspace too small (use sdfb200_field_render_workspace_bytes)");
    float* st = (float*)wsp + (ws_floats - stage);
    float* s_a = st;                 // alpha or density [N]
    float* s_rgb = s_a + N;          // [N,3]
    float* s_nrm = s_rgb + 3 * N;    // [N,3]
    float* s_w = s_nrm + 3 * N;      // [N]
    if (rnd->from_density) { if (!so.density) so.density = s_a; } else { if (!so.alpha) so.alpha = s_a; }
    if (!so.rgb) so.rgb = s_rgb;
    if (!so.normals) so.normals = s_nrm;
    r = sdfb200_field_forward(f, packed, table, in, &so, (void*)wsp, (ws_floats - stage) * sizeof(float), stream);
    if (r) return r;
    float* w = rnd->weights ? rnd->weights : s_w;
    if (rnd->from_density) {
      // transmittance[:, -1] (the transmittance BEFORE the last sample) is VolSDF's bg_transmittance (models/volsdf.py:67-68)
      float* Tbuf = rnd->bg_transmittance ? s_w + N : nullptr;
      r = sdfb200_weights_from_density(so.density, in->bins, in->n_rays, in->n_samples, w, Tbuf, stream);
      if (r) return r;
      if (Tbuf)
        SDFB_CUDA(cudaMemcpy2DAsync(rnd->bg_transmittance, sizeof(float), Tbuf + (in->n_samples - 1), (size_t)in->n_samples * sizeof(float),
                                    sizeof(float), (size_t)in->n_rays, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
      r = sdfb200_render(w, so.rgb, so.normals, in->bins, rnd->bg, rnd->bg_mode, rnd->clamp01, 0, in->n_rays, in->n_samples, &rnd->out, stream);
      if (r) return r;
    } else {
      r = sdfb200_render_alphas(so.alpha, so.rgb, so.normals, in->bins, rnd->bg, rnd->bg_mode, rnd->clamp01, in->n_rays, in->n_samples,
                                rnd->weights, rnd->bg_transmittance, &rnd->out, stream);
      if (r) return r;
    }
  }
  if (rnd->out.depth && rnd->clip_depth) return sdfb200_depth_clip(rnd->out.depth, rnd->out.steps_minmax, in->n_rays, stream);
  return 0;
}


// ---------------------------------------------------------------------------------------------------------------------
// Training path: the three GEMMs autograd needs for a Linear layer (forward / input gradient / weight gradient), closed under
// differentiation (the backward of each is made of the other two), on the tensor-core kernels of tc_linear.cu / tc_wgrad.cu.
// ---------------------------------------------------------------------------------------------------------------------
static int gemm_planes(int32_t precision) { return precision == SDFB200_PRECISION_BF16 ? 1 : 2; }

extern "C" size_t sdfb200_gemm_workspace_bytes(void) { return tc_wgrad_workspace_bytes() + kTcGemmScratchBytes + 256; }

extern "C" int sdfb200_gemm_nt(int32_t precision, const float* X, int64_t ldx, const float* W, int64_t ldw, int32_t N, int32_t K, const float* bias,
                               int32_t epilogue, float* Y, int64_t ldy, int64_t P, void* workspace, size_t workspace_bytes, void* stream) {
  SDFB_REQUIRE(precision == SDFB200_PRECISION_BF16X3 || precision == SDFB200_PRECISION_BF16, "gemm: precision must be bf16x3 or bf16");
  SDFB_REQUIRE(X && W && Y && workspace && workspace_bytes >= kTcGemmScratchBytes, "gemm_nt: NULL pointer / workspace too small");
  SDFB_REQUIRE(epilogue == TCL_NONE || epilogue == TCL_SOFTPLUS || epilogue == TCL_RELU, "gemm_nt: epilogue");
  SDFB_REQUIRE(N >= 1 && K >= 1 && ldx >= pad16(K) && ldy >= pad16(N) && ldx % 4 == 0 && ldy % 4 == 0, "gemm_nt: X / Y must hold the dims padded to 16");
  return tc_gemm_ex(gemm_planes(precision), epilogue, X, (int)ldx, W, (int)ldw, 0, N, K, bias, Y, (int)ldy, P, pad16(N), pad16(K), nullptr, 0, 0, workspace,
                    (cudaStream_t)stream);
}

extern "C" int sdfb200_gemm_nn(int32_t precision, const float* X, int64_t ldx, const float* W, int64_t ldw, int32_t N, int32_t K, float* Y, int64_t ldy,
                               int64_t P, void* workspace, size_t workspace_bytes, void* stream) {
  SDFB_REQUIRE(precision == SDFB200_PRECISION_BF16X3 || precision == SDFB200_PRECISION_BF16, "gemm: precision must be bf16x3 or bf16");
  SDFB_REQUIRE(X && W && Y && workspace && workspace_bytes >= kTcGemmScratchBytes, "gemm_nn: NULL pointer / workspace too small");
  SDFB_REQUIRE(N >= 1 && K >= 1 && ldx >= pad16(N) && ldy >= pad16(K) && ldx % 4 == 0 && ldy % 4 == 0, "gemm_nn: X / Y must hold the dims padded to 16");
  // Y[P, K] = X[P, N] W[N, K]  ==  X (W^T)^T : the weight tile is packed from the transposed view
  return tc_gemm_ex(gemm_planes(precision), TCL_NONE, X, (int)ldx, W, (int)ldw, 1, K, N, nullptr, Y, (int)ldy, P, pad16(K), pad16(N), nullptr, 0, 0, workspace,
                    (cudaStream_t)stream);
}

extern "C" int sdfb200_gemm_tn(int32_t precision, const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int64_t P, int32_t N,
                               int32_t K, void* workspace, size_t workspace_bytes, void* stream) {
  SDFB_REQUIRE(precision == SDFB200_PRECISION_BF16X3 || precision == SDFB200_PRECISION_BF16, "gemm: precision must be bf16x3 or bf16");
  return tc_wgrad(gemm_planes(precision), A, lda, B, ldb, C, ldc, P, N, K, workspace, workspace_bytes, (cudaStream_t)stream);
}
