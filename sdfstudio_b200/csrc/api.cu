// extern "C" entry points of the field (pack / forward / render) + library bookkeeping.  See include/sdfb200.h.
#include "common.cuh"
#include "field.h"
#include "tc_linear.h"

#include <string.h>

namespace sdfb200 {
thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

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
  return 0;
}

// The kernels that run one field call; the rules are in DESIGN §3.
struct FieldEngine {
  bool fused;          // the fused kernel (k_field_tc) runs the field
  bool fused_render;   // a render composites in the same launch; otherwise it runs the field as chosen here, then the compositing kernels
  int gemm_planes;     // the generic kernels' GEMMs: 0 = exact fp32, 1 / 2 = tensor-core bf16 / bf16x3
};

static FieldEngine field_engine(const sdfb200_field_t& f, const FieldPlan& p, bool geo_feature, int32_t n_samples) {
  FieldEngine e;
  e.fused = p.fused && !geo_feature;
  e.fused_render = e.fused && n_samples <= 128 && 128 % n_samples == 0;
  e.gemm_planes = f.precision != SDFB200_PRECISION_FP32 && !p.fused && !f.use_numerical_gradients ? tc_planes(f.precision) : 0;
  return e;
}

// A size query cannot see the outputs: it returns the larger of the two engines a descriptor of the fused family can take.
static size_t field_workspace_bytes(const sdfb200_field_t& f, const FieldPlan& p, int64_t n_points) {
  if (n_points == 0) return 256;
  size_t floats = field_generic_workspace_floats(f, p, n_points);
  if (field_engine(f, p, false, 1).fused) {
    const size_t t = field_tc_workspace_floats(f) + 64;
    floats = t > floats ? t : floats;
  }
  return floats * sizeof(float) + 256;
}

// per-sample heads a composed render stages at the end of the workspace
static size_t render_stage_floats(int64_t n_points) { return (size_t)n_points * 9 + 64; }   // alpha|density, rgb(3), normals(3), weights, transmittance

// A field call that passed check_field_call.  n_points == 0: nothing to do.
struct FieldCall {
  const sdfb200_field_t* f;
  FieldPlan p;
  FieldEngine e;
  const char* blob;
  const void* table;
  const sdfb200_field_in_t* in;
  sdfb200_field_out_t out;   // the per-sample outputs (all NULL when a render asks for none)
  int64_t n_points;
  float* ws;                 // the 256-byte aligned part of the caller's workspace
  size_t ws_floats;
};

// Every check of a forward (rnd == NULL) or render call, before any device work: the entry checks (descriptor, NULLs, sizes, mode,
// table, render descriptor, workspace pointer), then the workspace size, then what each requested output needs.  A render's sample
// outputs are optional.
static int check_field_call(const sdfb200_field_t* f, const void* packed, const void* table, const sdfb200_field_in_t* in, const sdfb200_field_out_t* out,
                            const sdfb200_field_render_t* rnd, void* workspace, size_t workspace_bytes, FieldCall& c) {
  int r = plan_or_fail(f, c.p);
  if (r) return r;
  SDFB_REQUIRE(packed && in && (out || rnd), "NULL pointer");
  SDFB_REQUIRE(in->n_rays >= 0 && in->n_samples >= 1, "bad sizes");
  c.n_points = in->n_rays * (int64_t)in->n_samples;
  if (c.n_points == 0) return 0;
  SDFB_REQUIRE(in->origins != nullptr, "origins is NULL");
  if (rnd) SDFB_REQUIRE(in->directions && in->bins, "field_render needs origins, directions and bins");
  SDFB_REQUIRE(in->bins != nullptr || in->n_samples == 1, "point mode requires n_samples == 1");
  SDFB_REQUIRE(in->bins == nullptr || in->directions != nullptr, "ray mode requires directions");
  SDFB_REQUIRE(!f->use_grid_feature || table != nullptr, "grid table is NULL");
  if (f->use_grid_feature) {
    r = validate_grid_pointers(&f->grid, table, nullptr);
    if (r) return r;
  }
  SDFB_REQUIRE(workspace != nullptr, "workspace is NULL");
  if (rnd && rnd->out.rgb) SDFB_REQUIRE(rnd->bg_mode == SDFB200_BG_LAST_SAMPLE || rnd->bg != nullptr, "rgb output needs a background");
  if (rnd && rnd->out.depth) SDFB_REQUIRE(rnd->out.steps_minmax != nullptr, "depth output needs steps_minmax (pre-set to {+inf,-inf})");
  const uintptr_t aligned = ((uintptr_t)workspace + 255) & ~(uintptr_t)255;
  SDFB_REQUIRE(workspace_bytes > aligned - (uintptr_t)workspace, "workspace too small");
  c.ws = (float*)aligned;
  c.ws_floats = (workspace_bytes - (aligned - (uintptr_t)workspace)) / sizeof(float);
  c.f = f;
  c.blob = (const char*)packed;
  c.table = table;
  c.in = in;
  if (out) c.out = *out; else memset(&c.out, 0, sizeof(c.out));
  c.e = field_engine(*f, c.p, c.out.geo_feature != nullptr, in->n_samples);

  size_t field_floats = c.ws_floats;
  if (rnd && !c.e.fused_render) {
    const size_t stage = render_stage_floats(c.n_points);
    SDFB_REQUIRE(field_floats > stage, "workspace too small (use sdfb200_field_render_workspace_bytes)");
    field_floats -= stage;
  }
  const size_t need = c.e.fused ? field_tc_workspace_floats(*f) : field_generic_workspace_floats(*f, c.p, c.n_points);
  if (field_floats < need) return fail(SDFB200_EWORKSPACE, "workspace too small%s (need %lld floats)", "", (long long)need);

  // a render also needs what its compositing reads: alpha (NeuS) or density (VolSDF), and rgb
  const bool alpha = c.out.alpha || (rnd && !rnd->from_density);
  const bool density = c.out.density || (rnd && rnd->from_density);
  if (c.out.rgb || alpha) SDFB_REQUIRE(in->directions != nullptr, "directions required for rgb / alpha");
  if (alpha) SDFB_REQUIRE(in->bins != nullptr && in->variance != nullptr, "alpha needs bins and the variance parameter");
  if (density) SDFB_REQUIRE(in->beta != nullptr && in->beta_min != nullptr, "density needs beta and beta_min");
  if (c.out.sampled_sdf) SDFB_REQUIRE(f->use_numerical_gradients, "sampled_sdf is only produced with use_numerical_gradients");
  return 0;
}

// the field part of a checked call on its engine, writing `out`; rnd != NULL composites in the same launch (e.fused_render)
static int run_field(const FieldCall& c, const sdfb200_field_out_t& out, const sdfb200_field_render_t* rnd, cudaStream_t st) {
  if (c.e.fused) return field_tc_forward(*c.f, c.p, c.blob, c.table, *c.in, out, rnd, c.ws, st);
  return field_forward_generic(*c.f, c.p, c.blob, c.table, *c.in, out, c.ws, c.e.gemm_planes, st);
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
    case 7: return sizeof(sdfb200_nerfacto_t);
    case 8: return sizeof(sdfb200_nerf_field_t);
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
  if (p.fused) return field_tc_pack(*f, p, (char*)packed, (cudaStream_t)stream);
  return 0;
}

extern "C" size_t sdfb200_field_workspace_bytes(const sdfb200_field_t* f, int64_t n_points) {
  FieldPlan p;
  if (plan_or_fail(f, p) || n_points < 0) return 0;
  return field_workspace_bytes(*f, p, n_points);
}

extern "C" int sdfb200_field_forward(const sdfb200_field_t* f, const void* packed, const void* table, const sdfb200_field_in_t* in,
                                     const sdfb200_field_out_t* out, void* workspace, size_t workspace_bytes, void* stream) {
  FieldCall c;
  int r = check_field_call(f, packed, table, in, out, nullptr, workspace, workspace_bytes, c);
  if (r || c.n_points == 0) return r;
  return run_field(c, c.out, nullptr, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// field + compositing in one call: fused into the tensor-core kernel, or composed from the field call and the compositing kernels
// with the per-sample heads staged at the end of the workspace.
// ---------------------------------------------------------------------------------------------------------------------
extern "C" size_t sdfb200_field_render_workspace_bytes(const sdfb200_field_t* f, int64_t n_rays, int32_t n_samples) {
  if (n_rays < 0 || n_samples < 1) return 0;
  FieldPlan p;
  if (plan_or_fail(f, p)) return 0;
  const int64_t n = n_rays * (int64_t)n_samples;
  const bool fused = field_engine(*f, p, false, n_samples).fused_render;
  return field_workspace_bytes(*f, p, n) + (fused ? 0 : render_stage_floats(n) * sizeof(float)) + 256;
}

extern "C" int sdfb200_field_render(const sdfb200_field_t* f, const void* packed, const void* table, const sdfb200_field_in_t* in,
                                    const sdfb200_field_out_t* sample_out, const sdfb200_field_render_t* rnd, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  SDFB_REQUIRE(rnd != nullptr, "NULL pointer");
  FieldCall c;
  int r = check_field_call(f, packed, table, in, sample_out, rnd, workspace, workspace_bytes, c);
  if (r || c.n_points == 0) return r;
  if (c.e.fused_render) {
    r = run_field(c, c.out, rnd, (cudaStream_t)stream);
    if (r) return r;
  } else {
    const int64_t N = c.n_points;
    sdfb200_field_out_t so = c.out;
    float* st = c.ws + (c.ws_floats - render_stage_floats(N));
    float* s_a = st;                 // alpha or density [N]
    float* s_rgb = s_a + N;          // [N,3]
    float* s_nrm = s_rgb + 3 * N;    // [N,3]
    float* s_w = s_nrm + 3 * N;      // [N]
    if (rnd->from_density) { if (!so.density) so.density = s_a; } else { if (!so.alpha) so.alpha = s_a; }
    if (!so.rgb) so.rgb = s_rgb;
    if (!so.normals) so.normals = s_nrm;
    r = run_field(c, so, nullptr, (cudaStream_t)stream);
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
extern "C" size_t sdfb200_gemm_workspace_bytes(void) { return tc_wgrad_workspace_bytes() + kTcGemmScratchBytes + 256; }

// What k_tc_linear's memory accesses need of the caller's buffers: X rows are read 16 bytes at a time (float4), bias and Y 8 bytes at a
// time (float2), and the packed weights are bulk-copied out of the workspace, which needs 16-byte alignment.  Checked before any launch.
static int check_gemm_buffers(const char* name, const float* X, const float* bias, const float* Y, const void* workspace, int64_t P) {
  if (P < 0) return fail(SDFB200_EINVAL, "%s: negative point count P (%lld)", name, (long long)P);
  if ((uintptr_t)X % 16) return fail(SDFB200_EINVAL, "%s: X must be aligned to %lld bytes (its float4 loads)", name, 16);
  if ((uintptr_t)Y % 8) return fail(SDFB200_EINVAL, "%s: Y must be aligned to %lld bytes (its float2 loads and stores)", name, 8);
  if ((uintptr_t)bias % 8) return fail(SDFB200_EINVAL, "%s: bias must be aligned to %lld bytes (its float2 loads)", name, 8);
  if ((uintptr_t)workspace % 16) return fail(SDFB200_EINVAL, "%s: workspace must be aligned to %lld bytes (bulk copies of the packed weights)", name, 16);
  return 0;
}

extern "C" int sdfb200_gemm_nt(int32_t precision, const float* X, int64_t ldx, const float* W, int64_t ldw, int32_t N, int32_t K, const float* bias,
                               int32_t epilogue, float* Y, int64_t ldy, int64_t P, void* workspace, size_t workspace_bytes, void* stream) {
  SDFB_REQUIRE(precision == SDFB200_PRECISION_BF16X3 || precision == SDFB200_PRECISION_BF16, "gemm: precision must be bf16x3 or bf16");
  SDFB_REQUIRE(X && W && Y && workspace && workspace_bytes >= kTcGemmScratchBytes, "gemm_nt: NULL pointer / workspace too small");
  SDFB_REQUIRE(epilogue == TCL_NONE || epilogue == TCL_SOFTPLUS || epilogue == TCL_RELU, "gemm_nt: epilogue");
  SDFB_REQUIRE(N >= 1 && K >= 1 && ldx >= pad16(K) && ldy >= pad16(N) && ldx % 4 == 0 && ldy % 4 == 0, "gemm_nt: X / Y must hold the dims padded to 16");
  SDFB_REQUIRE(ldw >= K, "gemm_nt: W rows must hold K (ldw >= K)");
  if (int r = check_gemm_buffers("gemm_nt", X, bias, Y, workspace, P)) return r;
  return tc_gemm_ex(tc_planes(precision), epilogue, X, (int)ldx, W, (int)ldw, 0, N, K, bias, Y, (int)ldy, P, pad16(N), pad16(K), nullptr, 0, 0, workspace,
                    (cudaStream_t)stream);
}

extern "C" int sdfb200_gemm_nn(int32_t precision, const float* X, int64_t ldx, const float* W, int64_t ldw, int32_t N, int32_t K, float* Y, int64_t ldy,
                               int64_t P, void* workspace, size_t workspace_bytes, void* stream) {
  SDFB_REQUIRE(precision == SDFB200_PRECISION_BF16X3 || precision == SDFB200_PRECISION_BF16, "gemm: precision must be bf16x3 or bf16");
  SDFB_REQUIRE(X && W && Y && workspace && workspace_bytes >= kTcGemmScratchBytes, "gemm_nn: NULL pointer / workspace too small");
  SDFB_REQUIRE(N >= 1 && K >= 1 && ldx >= pad16(N) && ldy >= pad16(K) && ldx % 4 == 0 && ldy % 4 == 0, "gemm_nn: X / Y must hold the dims padded to 16");
  SDFB_REQUIRE(ldw >= K, "gemm_nn: W rows must hold K (ldw >= K)");
  if (int r = check_gemm_buffers("gemm_nn", X, nullptr, Y, workspace, P)) return r;
  // Y[P, K] = X[P, N] W[N, K]  ==  X (W^T)^T : the weight tile is packed from the transposed view
  return tc_gemm_ex(tc_planes(precision), TCL_NONE, X, (int)ldx, W, (int)ldw, 1, K, N, nullptr, Y, (int)ldy, P, pad16(K), pad16(N), nullptr, 0, 0, workspace,
                    (cudaStream_t)stream);
}

extern "C" int sdfb200_gemm_tn(int32_t precision, const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int64_t P, int32_t N,
                               int32_t K, void* workspace, size_t workspace_bytes, void* stream) {
  SDFB_REQUIRE(precision == SDFB200_PRECISION_BF16X3 || precision == SDFB200_PRECISION_BF16, "gemm: precision must be bf16x3 or bf16");
  return tc_wgrad(tc_planes(precision), A, lda, B, ldb, C, ldc, P, N, K, workspace, workspace_bytes, (cudaStream_t)stream);
}
