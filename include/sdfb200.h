/*
 * sdfb200.h -- C ABI of the H100-native SDF volume-rendering hot path (sdfstudio drop-in).
 *
 * The reference (autonomousvision/sdfstudio) has NO native/FFI boundary on this path: its plug points are Python
 * nn.Modules (SURVEY.md section 8b).  This header is the C-ABI *underneath* those modules; every entry point names the
 * reference function it replaces (paths relative to the reference root).  The Python host side
 * (sdfstudio_b200/*.py) mirrors the reference classes and binds these symbols with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - plain pointers + sizes; no torch / C++ types cross the boundary.  All pointers are DEVICE pointers unless a
 *     parameter is documented as host.  Tensors are dense row-major fp32 unless stated.
 *   - ownership: the caller allocates every buffer including workspace (size-query functions are provided); the
 *     library never allocates, frees or retains a pointer past the call.
 *   - every call only enqueues work on `stream` (a cudaStream_t passed as void*); no hidden synchronisation.
 *   - return value: 0 = ok, <0 = invalid argument (SDFB200_E*), >0 = cudaError_t.  No exceptions, no abort.
 *     sdfb200_last_error_string() returns a thread-local description of the last failure.
 *   - re-entrant and stateless apart from immutable per-device kernel attributes set once.
 */
#ifndef SDFB200_H_
#define SDFB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SDFB200_VERSION 100
#define SDFB200_MAX_LEVELS 32
#define SDFB200_MAX_LAYERS 12

enum {
  SDFB200_OK = 0,
  SDFB200_EINVAL = -1,      /* bad argument / unsupported configuration */
  SDFB200_EWORKSPACE = -2,  /* workspace too small */
  SDFB200_EUNSUPPORTED = -3
};

enum { SDFB200_GRID_TORCH = 0, SDFB200_GRID_TCNN = 1 };      /* table layout */
enum { SDFB200_DT_F32 = 0, SDFB200_DT_F16 = 1 };             /* table element type */
enum { SDFB200_CONTRACT_NONE = 0, SDFB200_CONTRACT_LINF = 1, SDFB200_CONTRACT_L2 = 2 };
enum { SDFB200_SPACING_UNIFORM = 0, SDFB200_SPACING_LINDISP = 1, SDFB200_SPACING_SQRT = 2, SDFB200_SPACING_LOG = 3,
       SDFB200_SPACING_PIECEWISE = 4, SDFB200_SPACING_IDENTITY = 5 /* bins already euclidean */ };
enum { SDFB200_BG_COLOR = 0, SDFB200_BG_LAST_SAMPLE = 1, SDFB200_BG_PER_RAY = 2 };
enum { SDFB200_PRECISION_FP32 = 0,      /* CUDA-core fp32 FMA (exact-fp32 reference numerics)            */
       SDFB200_PRECISION_BF16X3 = 1,    /* wgmma bf16 split a0*w0 + a1*w0 + a0*w1, fp32 accumulate        */
       SDFB200_PRECISION_BF16 = 2 };    /* wgmma single bf16 pass (fast mode; reported with PSNR-vs-ref)   */

/* ---------------------------------------------------------------------------------------------------------------
 * Multi-resolution grid.  Replaces tinycudann.Encoding(HashGrid) as configured at
 * nerfstudio/fields/sdf_field.py:230-241 and HashEncoding.pytorch_fwd (field_components/encodings.py:357-398).
 * Filled by the host (sdfstudio_b200/encoding.py).  `scale`: per-level coordinate scale; torch layout: corner =
 * ceil/floor(x*scale), every level hashed, offset = l*2^log2_hashmap_size; tcnn layout: pos = x*scale+0.5,
 * `resolution`/`size`/`hashed` per level.  `offset` counts table ENTRIES (rows of n_features values).
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct sdfb200_grid {
  int32_t layout;            /* SDFB200_GRID_* */
  int32_t n_levels;          /* <= SDFB200_MAX_LEVELS */
  int32_t n_features;        /* 1, 2, 4 or 8 */
  int32_t log2_hashmap_size;
  int32_t smoothstep;        /* 0 linear, 1 smoothstep (t*t*(3-2t)) */
  int32_t active_levels;     /* levels >= this are zeroed: SDFField.update_mask (sdf_field.py:376-378) */
  int32_t table_dtype;       /* SDFB200_DT_* */
  int32_t reserved;
  float scale[SDFB200_MAX_LEVELS];
  uint32_t resolution[SDFB200_MAX_LEVELS];
  uint32_t size[SDFB200_MAX_LEVELS];
  uint64_t offset[SDFB200_MAX_LEVELS];
  uint8_t hashed[SDFB200_MAX_LEVELS];
} sdfb200_grid_t;

/* tcnn.Encoding.forward / HashEncoding.pytorch_fwd: x01 [n,3] in [0,1] -> out [n, L*F] (masked levels = 0).
 * dout_dx (optional, may be NULL): [n, L*F, 3] = d out / d x01.  out_ld = row stride of `out` in floats. */
int sdfb200_grid_encode(const sdfb200_grid_t* grid, const void* table, const float* x01, int64_t n, float* out,
                        int64_t out_ld, float* dout_dx, void* stream);

/* backward of the above w.r.t. the table (atomic scatter-add into dtable, fp32, same row layout as the table) and,
 * optionally, w.r.t. x01 (dx01 [n,3], may be NULL).  dout [n, L*F].  dtable may be NULL when only dx01 is wanted. */
int sdfb200_grid_encode_backward(const sdfb200_grid_t* grid, const void* table, const float* x01, const float* dout,
                                 int64_t n, float* dtable, float* dx01, void* stream);

/* backward of sdfb200_grid_encode_backward's dx01 output (second order; what autograd's create_graph=True gives the
 * reference for the eikonal loss, models/base_surface_model.py:358-362 through sdf_field.py:655-662).
 * g_dx01 [n,3] = dLoss/d(dx01).  Outputs (each may be NULL): g_dout [n, L*F] (overwritten), g_table (fp32, table row
 * layout, atomically ACCUMULATED -- zero it first), g_x01 [n,3] (ACCUMULATED). */
int sdfb200_grid_encode_backward_backward(const sdfb200_grid_t* grid, const void* table, const float* x01, const float* dout,
                                          const float* g_dx01, int64_t n, float* g_dout, float* g_table, float* g_x01, void* stream);

/* Grouped forms of the two calls above for numerical-gradient fields (SDFField.gradient with use_numerical_gradients,
 * sdf_field.py:424-452: the network is evaluated at x and at x +- delta e_i).  The batch holds `group` taps per sample, tap gi of
 * sample s at row gi * (n / group) + s; taps that hit the same 8 table rows of a level share one set of gathers / one set of atomic
 * adds.  Results equal the ungrouped calls on the same n points (forward: bit for bit; backward: up to the order of the atomic sums).
 * The backward produces the table gradient only (numerical-gradient fields never differentiate the encoding w.r.t. its input). */
int sdfb200_grid_encode_grouped(const sdfb200_grid_t* grid, const void* table, const float* x01, int64_t n, int32_t group, float* out,
                                int64_t out_ld, void* stream);
int sdfb200_grid_encode_backward_grouped(const sdfb200_grid_t* grid, const float* x01, const float* dout, int64_t n, int32_t group,
                                         float* dtable, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * SDFField.  Replaces nerfstudio/fields/sdf_field.py: forward_geonetwork :380-410, gradient :424-465, get_alpha
 * :476-525, get_colors :532-612, get_outputs :614-689, LaplaceDensity :57-66, get_occupancy :527-530,
 * NeRFEncoding.forward (encodings.py:167-208) and SceneContraction.forward (spatial_distortions.py:66-73).
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct sdfb200_field {
  sdfb200_grid_t grid;
  int32_t use_grid_feature;
  int32_t pe_degree;              /* position_encoding_max_degree */
  int32_t use_position_encoding;  /* 0 => PE block is zeros (sdf_field.py:393-394) */
  int32_t off_axis;               /* 21-direction off-axis PE (encodings.py:129-153,191-192) */
  int32_t contraction;            /* SDFB200_CONTRACT_* (spatial_distortion passed to SDFField) */
  int32_t n_geo_linear;           /* num_layers + 1 */
  int32_t geo_dims[SDFB200_MAX_LAYERS + 1]; /* dims[0..n_geo_linear]; dims[0] = 3+pe+grid */
  int32_t geo_skip_layer;         /* index l whose input is cat(h, inputs)/sqrt(2) (skip_in=[4]); -1 = none */
  int32_t n_color_linear;         /* num_layers_color + 1 */
  int32_t color_dims[SDFB200_MAX_LAYERS + 1];
  int32_t appearance_dim;
  int32_t use_diffuse_color, use_specular_tint, use_reflections, use_n_dot_v;
  int32_t use_numerical_gradients;
  float rgb_padding;
  int32_t precision;              /* SDFB200_PRECISION_* */
} sdfb200_field_t;

/* raw (un-packed) parameter pointers, fp32, reference layout (nn.Linear weight [out,in] row-major).
 * weight_g may be NULL for a layer without weight-norm (then weight_v is the plain weight). */
typedef struct sdfb200_field_params {
  const float* geo_weight_v[SDFB200_MAX_LAYERS];
  const float* geo_weight_g[SDFB200_MAX_LAYERS];
  const float* geo_bias[SDFB200_MAX_LAYERS];
  const float* color_weight_v[SDFB200_MAX_LAYERS];
  const float* color_weight_g[SDFB200_MAX_LAYERS];
  const float* color_bias[SDFB200_MAX_LAYERS];
  const float* diffuse_weight;  const float* diffuse_bias;   /* [3,geo_feat], [3] or NULL */
  const float* tint_weight;     const float* tint_bias;
} sdfb200_field_params_t;

/* bytes of the packed-weight blob for this field (weight-norm folded, padded, bf16 split planes when a tensor-core
 * precision is selected). */
size_t sdfb200_field_packed_bytes(const sdfb200_field_t* f);
/* fold weight-norm (W = g*v/||v||, sdf_field.py:312-313,360-361) and write the packed blob.  Call again whenever the
 * parameters change. */
int sdfb200_field_pack(const sdfb200_field_t* f, const sdfb200_field_params_t* p, void* packed, void* stream);

typedef struct sdfb200_field_in {
  int64_t n_rays;
  int32_t n_samples;             /* samples per ray; N = n_rays*n_samples.  Point mode: n_samples=1, bins=NULL */
  int32_t apply_contraction;     /* get_outputs contracts (:629-630); get_sdf / get_density do not (:412-418) */
  const float* origins;          /* [R,3] (point mode: the points)                         */
  const float* directions;       /* [R,3] or NULL when no colour/alpha output is requested */
  const float* bins;             /* [R, S+1] euclidean bin edges; starts=bins[:, :-1], deltas=bins[:,1:]-bins[:,:-1] */
  const float* appearance;       /* [R, appearance_dim] embedded appearance per ray, or NULL (= zeros)  */
  const float* variance;         /* device ptr to deviation_network.variance (1 float) or NULL           */
  const float* beta;             /* device ptr to laplace_density.beta (1 float) or NULL                 */
  const float* beta_min;         /* device ptr to laplace_density.beta_min                               */
  float cos_anneal_ratio;        /* SDFField._cos_anneal_ratio                                           */
  float numerical_delta;         /* SDFField.numerical_gradients_delta                                   */
} sdfb200_field_in_t;

/* any NULL output is skipped, and stages nobody consumes are not run (e.g. only `sdf` => geo forward only). */
typedef struct sdfb200_field_out {
  float* sdf;          /* [N]      FieldHeadNames.SDF        */
  float* geo_feature;  /* [N, geo_feat_dim]  (forward_geonetwork()[:,1:]) */
  float* gradients;    /* [N,3]    FieldHeadNames.GRADIENT   */
  float* normals;      /* [N,3]    FieldHeadNames.NORMAL     */
  float* rgb;          /* [N,3]    FieldHeadNames.RGB        */
  float* density;      /* [N]      FieldHeadNames.DENSITY    */
  float* alpha;        /* [N]      FieldHeadNames.ALPHA      */
  float* occupancy;    /* [N]      FieldHeadNames.OCCUPANCY  */
  float* points_norm;  /* [N]      "points_norm"             */
  float* sampled_sdf;  /* [N,6]    "sampled_sdf" (numerical gradients only) */
  float* points;       /* [N,3]    the (contracted) sample positions  */
} sdfb200_field_out_t;

size_t sdfb200_field_workspace_bytes(const sdfb200_field_t* f, int64_t n_points);
int sdfb200_field_forward(const sdfb200_field_t* f, const void* packed, const void* table, const sdfb200_field_in_t* in,
                          const sdfb200_field_out_t* out, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Proposal density field.  Replaces HashMLPDensityField.get_density / density_fn (nerfstudio/fields/density_fields.py:40-121,
 * fields/base_field.py:48-65): tcnn.NetworkWithInputEncoding (HashGrid -> FullyFusedMLP, ReLU, no biases) + trunc_exp
 * (field_components/activations.py:24-42).  positions [n,3]; normalisation: aabb != NULL -> (x - aabb[0]) / (aabb[1] - aabb[0])
 * (data/scene_box.py:67-76), else SceneContraction (`contraction`) followed by (x + 2) / 4.
 * weights (fp32, row-major): [hidden, in_pad] | (n_hidden_layers-1) x [hidden, hidden] | [hidden]; in_pad = L*F rounded up to 16.
 * density [n] = exp(pre-activation); pre_activation [n] optional.
 * ------------------------------------------------------------------------------------------------------------- */
int sdfb200_density_field_forward(const sdfb200_grid_t* grid, const void* table, const float* weights, int32_t hidden_dim,
                                  int32_t n_hidden_layers, int32_t contraction, const float* aabb, const float* positions,
                                  int64_t n, float* density, float* pre_activation, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Ray samplers.  Replace nerfstudio/model_components/ray_samplers.py.  A sample set is a pair of bin-edge buffers
 * [R, S+1]: `spacing` (normalised) and `euclid` (distance along the ray), cf. cameras/rays.py:295-339.
 * ------------------------------------------------------------------------------------------------------------- */
/* SpacedSampler.generate_ray_samples :80-127.  base_bins [S+1] = linspace(0,1,S+1) (host computes it so that the
 * values are bit-identical to torch.linspace); jitter: NULL (eval) or [R,1] / [R,S+1] uniform randoms (training). */
int sdfb200_spaced_bins(const float* nears, const float* fars, const float* base_bins, const float* jitter,
                        int32_t jitter_per_bin, int64_t n_rays, int32_t n_samples, int32_t spacing, float* spacing_bins,
                        float* euclid_bins, void* stream);

/* spacing -> euclidean map of an existing bin buffer: spacing_fn_inv(x*s_far + (1-x)*s_near)  (:115-117) */
int sdfb200_bins_to_euclid(const float* spacing_bins, const float* nears, const float* fars, int64_t n_rays,
                           int32_t n_bins, int32_t spacing, float* euclid_bins, void* stream);

/* PDFSampler.generate_ray_samples :275-370.  weights [R,S_in] (the [...,0] slice), existing spacing bins [R,S_in+1],
 * u [S_out+1] = the eval-mode u grid (host: torch.linspace(...)+1/(2*nb)) or the stratified base; jitter NULL or
 * [R,1] / [R,S_out+1] (already divided by num_bins by the host: u + rand/num_bins).  Outputs: new spacing bins
 * [R,S_out+1] (sorted-merged with the originals when include_original: [R, S_in+S_out+2]) and, optionally, the
 * searchsorted indices `inds` [R,S_out+1] (int64, side="right"; may be NULL). */
int sdfb200_pdf_sample(const float* weights, const float* existing_bins, const float* u, const float* jitter,
                       int32_t jitter_per_bin, int64_t n_rays, int32_t s_in, int32_t s_out, float histogram_padding,
                       float eps, int32_t include_original, float* new_bins, int64_t* inds, void* stream);

/* ErrorBoundedSampler.merge_ray_samples :758-788: stable merge of the starts of two sample sets (spacing domain).
 * bins_a [R,Sa+1], bins_b [R,Sb+1] -> merged [R,Sa+Sb+1], sorted_index [R,Sa+Sb] (int64; indices into cat(a,b)). */
int sdfb200_merge_bins(const float* bins_a, const float* bins_b, int64_t n_rays, int32_t sa, int32_t sb, float* merged,
                       int64_t* sorted_index, void* stream);
/* torch.gather(cat([sdf_a, sdf_b], -1), 1, sorted_index) (:872-874, :646-648) */
int sdfb200_merge_gather(const float* a, const float* b, const int64_t* sorted_index, int64_t n_rays, int32_t sa,
                         int32_t sb, float* out, void* stream);

/* NeuSSampler.rendering_sdf_with_fixed_inv_s :909-944 fused with RaySamples.get_weights_from_alphas
 * (cameras/rays.py:194-210) and the zero pad (:885): euclid bins [R,S+1], sdf [R,S] -> weights [R,S] (last = 0). */
int sdfb200_neus_upsample_weights(const float* euclid_bins, const float* sdf, int64_t n_rays, int32_t n_samples,
                                  float inv_s, float* weights, void* stream);

/* ErrorBoundedSampler inner step (:650-676): get_dstar :704-726, get_updated_beta :728-738 (beta_iters bisection
 * steps of get_error_bound :740-756), LaplaceDensity with per-ray beta, weights/transmittance, and the error-bound
 * upsampling weights.  beta [R] in/out.  beta0: device ptr (1 float, already |beta|+beta_min).
 * Outputs weights [R,S] (density weights), err_weights [R,S] (error-bound pdf). */
int sdfb200_volsdf_step(const float* euclid_bins, const float* sdf, const float* beta0, float* beta, int64_t n_rays,
                        int32_t n_samples, float eps, int32_t beta_iters, float* weights, float* err_weights,
                        void* stream);
/* initial beta from Lemma 2 (:629-633): sqrt( sum(deltas^2) / (4 log(1+eps)) ) */
int sdfb200_volsdf_init_beta(const float* euclid_bins, int64_t n_rays, int32_t n_samples, float eps, float* beta,
                             void* stream);

/* UniSurfSampler surface search (:1027-1077): first +->- sign change along the marching samples, linear root, and
 * the shrunk [near, far] interval.  Outputs: z [R] (NaN when no hit), hit [R] (uint8), new nears/fars [R]. */
int sdfb200_unisurf_interval(const float* euclid_bins, const float* sdf, const float* nears, const float* fars,
                             int64_t n_rays, int32_t n_samples, float delta, float* z, uint8_t* hit, float* new_nears,
                             float* new_fars, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Weights + renderers.  Replace cameras/rays.py:131-230 and model_components/renderers.py (dense branch).
 * ------------------------------------------------------------------------------------------------------------- */
/* RaySamples.get_weights_and_transmittance_from_alphas: alphas [R,S] -> weights [R,S], transmittance [R,S+1] (NULL ok) */
int sdfb200_weights_from_alphas(const float* alphas, int64_t n_rays, int32_t n_samples, float* weights,
                                float* transmittance, void* stream);
/* RaySamples.get_weights_and_transmittance: density [R,S], euclid bins [R,S+1] -> weights, transmittance [R,S] */
int sdfb200_weights_from_density(const float* density, const float* euclid_bins, int64_t n_rays, int32_t n_samples,
                                 float* weights, float* transmittance, void* stream);

typedef struct sdfb200_render_out {
  float* rgb;           /* [R,3]  RGBRenderer.forward :98-118                       */
  float* depth;         /* [R]    DepthRenderer 'expected' :246-259 (before the global clip) or 'median' :233-245 */
  float* normal;        /* [R,3]  SemanticRenderer :284-295                         */
  float* accumulation;  /* [R]    AccumulationRenderer :171-197                     */
  float* steps_minmax;  /* [2]    global min / max of steps (for the clip at :257); must be pre-set to {+inf,-inf} */
} sdfb200_render_out_t;
/* composites rgb [R,S,3] / normals [R,S,3] with weights [R,S] along each ray.  background: bg_mode COLOR -> bg [3];
 * PER_RAY -> bg [R,3] (the "random" draw); LAST_SAMPLE.  clamp01: eval-mode clamp (:116-117).
 * depth_median != 0 selects the median method. */
int sdfb200_render(const float* weights, const float* rgb, const float* normals, const float* euclid_bins,
                   const float* bg, int32_t bg_mode, int32_t clamp01, int32_t depth_median, int64_t n_rays,
                   int32_t n_samples, const sdfb200_render_out_t* out, void* stream);
/* fused form of what SurfaceModel.get_outputs does after the field (models/neus.py:100-103 +
 * models/base_surface_model.py:300-310): alphas [R,S] -> transmittance (rays.py:194-230) -> weights [R,S] (optional out) ->
 * rgb / expected depth / normal / accumulation, one warp per ray.  bg_transmittance [R] (optional) = transmittance[:, -1].
 * The prefix product is a warp scan in double (not the sequential order of torch.cumprod): results agree with
 * sdfb200_weights_from_alphas + sdfb200_render to ~1e-7 relative, not bit-exactly. */
int sdfb200_render_alphas(const float* alphas, const float* rgb, const float* normals, const float* euclid_bins,
                          const float* bg, int32_t bg_mode, int32_t clamp01, int64_t n_rays, int32_t n_samples,
                          float* weights, float* bg_transmittance, const sdfb200_render_out_t* out, void* stream);
/* SDFField.get_outputs + weights + the four renderers in ONE call: what SurfaceModel.get_outputs does between the sampler and
 * the losses (models/base_surface_model.py:292-365 with models/neus.py:85-116 or models/volsdf.py:62-87).  from_density = 0:
 * NeuS alphas -> get_weights_and_transmittance_from_alphas (rays.py:194-230); 1: Laplace density -> get_weights_and_transmittance
 * (rays.py:131-192).  The neus-facto shape family at a tensor-core precision with 128 % n_samples == 0 runs as one fused
 * kernel (compositing in registers, no per-sample round trip through HBM); every other case is composed inside the
 * library from sdfb200_field_forward + the compositing kernels, with identical results.  `sample_out` (may be NULL) selects
 * per-sample heads to materialise as well (weights_list / eikonal consumers); `weights` [R,S], `bg_transmittance` [R] optional.
 * out.depth is the 'expected' depth; with clip_depth != 0 it is clipped to the batch-global [steps.min(), steps.max()]
 * (renderers.py:257) at the end of the call; out.steps_minmax [2] must be pre-set to {+inf, -inf}. */
typedef struct sdfb200_field_render {
  int32_t from_density;
  int32_t bg_mode;            /* SDFB200_BG_* */
  int32_t clamp01;            /* eval-mode clamp of rgb (renderers.py:116-117) */
  int32_t clip_depth;
  const float* bg;            /* [3] (BG_COLOR) or [R,3] (BG_PER_RAY); unused for BG_LAST_SAMPLE */
  float* weights;             /* [R,S] or NULL */
  float* bg_transmittance;    /* [R]   or NULL: transmittance[:, -1] */
  sdfb200_render_out_t out;
} sdfb200_field_render_t;
size_t sdfb200_field_render_workspace_bytes(const sdfb200_field_t* f, int64_t n_rays, int32_t n_samples);
int sdfb200_field_render(const sdfb200_field_t* f, const void* packed, const void* table, const sdfb200_field_in_t* in,
                         const sdfb200_field_out_t* sample_out, const sdfb200_field_render_t* render, void* workspace,
                         size_t workspace_bytes, void* stream);

/* packed samples (the `ray_indices` / `num_rays` branch of the renderers, fed by nerfacc-style samplers: renderers.py:74-79 RGB,
 * :192-194 accumulation, :249-253 expected depth; nerfacc.accumulate_along_rays == per-ray scatter-add): weights [N], rgb / normals
 * [N,3], starts / ends [N] (frustum bin edges, for the depth), ray_indices [N] int64 in [0, n_rays).  Background COLOR or PER_RAY
 * ('last_sample' is rejected like the reference does).  workspace >= n_rays * 8 floats.  out.depth is the un-clipped expected depth;
 * out.steps_minmax (optional, pre-set to {+inf,-inf}) receives steps.min()/max() for sdfb200_depth_clip. */
int sdfb200_render_packed(const float* weights, const float* rgb, const float* normals, const float* starts, const float* ends,
                          const int64_t* ray_indices, int64_t n_samples_total, int64_t n_rays, const float* bg, int32_t bg_mode, int32_t clamp01,
                          const sdfb200_render_out_t* out, void* workspace, size_t workspace_bytes, void* stream);
/* torch.clip(depth, steps.min(), steps.max()) (:257) using the min/max accumulated by sdfb200_render. */
int sdfb200_depth_clip(float* depth, const float* steps_minmax, int64_t n_rays, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * The step before the path (SURVEY.md section 8f rows 2-3): camera rays, colliders, meshing lattice.
 * ------------------------------------------------------------------------------------------------------------- */
#define SDFB200_CAMERA_PERSPECTIVE 1 /* CameraType.PERSPECTIVE.value, cameras/cameras.py:38-43 */
#define SDFB200_CAMERA_FISHEYE 2
#define SDFB200_COLLIDER_AABB 0
#define SDFB200_COLLIDER_NEAR_FAR 1
#define SDFB200_COLLIDER_SPHERE 2

/* Cameras._generate_rays_from_coords (cameras/cameras.py:459-695) for perspective / fisheye cameras without distortion
 * parameters.  Per-camera arrays fx, fy, cx, cy [C], camera_type [C] (NULL = all perspective), camera_to_worlds [C,3,4];
 * per-ray camera_indices [N] (int32) and coords [N,2] = (y, x) pixel coordinates (already offset by 0.5 by the caller, like
 * the reference).  Outputs: origins, directions [N,3]; pixel_area, directions_norm [N] (may be NULL). */
int sdfb200_generate_rays(const float* fx, const float* fy, const float* cx, const float* cy, const int32_t* camera_type,
                          const float* camera_to_worlds, int32_t n_cameras, const int32_t* camera_indices, const float* coords,
                          int64_t n_rays, float* origins, float* directions, float* pixel_area, float* directions_norm, void* stream);

/* scene_colliders.py:47-163.  `params` is a HOST array: AABB = {min x,y,z, max x,y,z} (:56-98, near_plane clamp :92-94),
 * NEAR_FAR = {near, far} (:116-134), SPHERE = {radius, soft_intersection != 0, radius**2} (:137-163).  nears / fars [N]. */
int sdfb200_collide(const float* origins, const float* directions, int64_t n_rays, int32_t collider_type, const float* params,
                    float near_plane, float* nears, float* fars, void* stream);

/* points [n,3] = entries [start, start+n) of np.meshgrid(np.linspace(min, max, res) x3, indexing="ij") flattened
 * (utils/marching_cubes.py:49-56): the lattice is generated on the device chunk by chunk instead of being materialised.
 * bbox_min / bbox_max (double[3]) and resolution (int32[3]) are HOST arrays. */
int sdfb200_lattice_points(const double* bbox_min, const double* bbox_max, const int32_t* resolution, int64_t start, int64_t n,
                           float* points, void* stream);

/* Training path: backward of sdfb200_render (expected depth) / sdfb200_render_alphas' compositing w.r.t. the per-sample
 * inputs (autograd over renderers.py:42-295 in the reference).  `accumulation`, `depth` = forward outputs (depth BEFORE the
 * global clip).  g_rgb [R,3], g_depth [R], g_normal [R,3], g_accumulation [R], g_weights_in [R,S]: incoming gradients, each
 * may be NULL.  Outputs: g_weights [R,S] (required), g_rgb_samples / g_normal_samples [R,S,3] (may be NULL). */
int sdfb200_render_backward(const float* weights, const float* rgb, const float* normals, const float* euclid_bins, const float* bg,
                            int32_t bg_mode, int64_t n_rays, int32_t n_samples, const float* accumulation, const float* depth,
                            const float* g_rgb, const float* g_depth, const float* g_normal, const float* g_accumulation,
                            const float* g_weights_in, float* g_weights, float* g_rgb_samples, float* g_normal_samples, void* stream);

/* backward of sdfb200_weights_from_alphas (from_density = 0) or sdfb200_weights_from_density (from_density = 1):
 * g_weights [R,S] (+ the gradient of the returned transmittance) -> g_in [R,S].  g_transmittance may be NULL; otherwise
 * g_transmittance_cols = 1 (alphas only: [R], gradient of transmittance[:, -1] = bg_transmittance, models/neus.py:101) or the
 * full width of the transmittance output ([R,S+1] for alphas, [R,S] for densities; models/volsdf.py:67-68 back-propagates
 * through transmittance[:, -1] of the density form). */
int sdfb200_weights_backward(const float* alphas_or_density, const float* euclid_bins, int32_t from_density, int64_t n_rays,
                             int32_t n_samples, const float* g_weights, const float* g_transmittance, int32_t g_transmittance_cols,
                             float* g_in, void* stream);


/* ---------------------------------------------------------------------------------------------------------------
 * Training path: dense-layer GEMMs on wgmma (bf16x3 = parity grade, bf16 = fast), fp32 row-major in / out.  They replace the ATen /
 * cuBLAS matmuls autograd runs for every nn.Linear of SDFField when the reference trains (sdf_field.py:400-409 through
 * engine/trainer.py:319-323): forward Y = X W^T (+ bias, activation), input gradient dX = dY W, weight gradient dW = dY^T X.  The set is
 * closed under differentiation (each one's backward is the other two), which is what the eikonal term's double backward needs
 * (sdf_field.py:646-655, create_graph=True).  P = number of points (the long dimension); N, K = layer widths.  Buffers of width N / K
 * must be allocated with their row padded to a multiple of 16 floats (ld >= pad16(width)); padding columns of outputs are written
 * (zeros for epilogue 0), padding columns of inputs are ignored.  workspace >= sdfb200_gemm_workspace_bytes().
 * epilogue: 0 none, 1 softplus(beta = 100), 2 relu.  bias [pad16(N)] or NULL.
 * ------------------------------------------------------------------------------------------------------------- */
size_t sdfb200_gemm_workspace_bytes(void);
/* Y[P, N] = epilogue(X[P, K] W[N, K]^T + bias) */
int sdfb200_gemm_nt(int32_t precision, const float* X, int64_t ldx, const float* W, int64_t ldw, int32_t N, int32_t K, const float* bias,
                    int32_t epilogue, float* Y, int64_t ldy, int64_t P, void* workspace, size_t workspace_bytes, void* stream);
/* Y[P, K] = X[P, N] W[N, K] */
int sdfb200_gemm_nn(int32_t precision, const float* X, int64_t ldx, const float* W, int64_t ldw, int32_t N, int32_t K, float* Y, int64_t ldy,
                    int64_t P, void* workspace, size_t workspace_bytes, void* stream);
/* C[N, K] = A[P, N]^T B[P, K]  (reduction over the points; per-SM partial sums reduced in a fixed order: deterministic) */
int sdfb200_gemm_tn(int32_t precision, const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int64_t P, int32_t N,
                    int32_t K, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------------*/
int sdfb200_version(void);
const char* sdfb200_last_error_string(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches). */
int64_t sdfb200_launch_count(void);
/* sizeof() of the ABI structs (0 grid, 1 field, 2 field_params, 3 field_in, 4 field_out, 5 render_out, 6 field_render): lets a binding
 * verify its struct mirrors before the first call. */
size_t sdfb200_struct_size(int32_t which);

#ifdef __cplusplus
}
#endif
#endif /* SDFB200_H_ */
