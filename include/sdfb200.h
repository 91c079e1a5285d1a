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
 * Nerfacto background field (background_model="grid" of neus-facto-angelo / bakedangelo).  Replaces TCNNNerfactoField.forward
 * (nerfstudio/fields/nerfacto_field.py:223-318 through fields/base_field.py:104-123) without normals, transients, semantics or
 * predicted normals.  grid: tcnn layout, 2 features per level.  Normalisation as sdfb200_density_field_forward (aabb != NULL selects
 * the SceneBox, else `contraction` then (x + 2) / 4).
 * Geometry: ray mode (n_samples = S > 0): origins / directions [n_rays,3], bins [n_rays,S+1] euclidean edges, positions = midpoints
 * origins + directions * (start + end) / 2 (rounded like the reference, no FMA), N = n_rays * S.  Point mode (n_samples = 0):
 * origins = positions [n_rays,3], directions [n_rays,3], bins unused, N = n_rays.
 * base_weights (fp32, row-major): [hidden_dim, in_pad] | (n_hidden_layers-1) x [hidden_dim, hidden_dim] | [16, hidden_dim], rows
 * 0..geo_feat_dim live; in_pad = 2 L rounded up to 16.  head_weights: [hidden_dim_color, head_pad] | (n_hidden_layers_color-1) x
 * [hidden_dim_color, hidden_dim_color] | [16, hidden_dim_color], rows 0..2 live; head input = cat(SH4 16, geo, appearance),
 * head_pad = its width rounded up to 16.
 * appearance: row r (the ray in ray mode, the point in point mode) at appearance + r * appearance_stride (stride 0 broadcasts one
 * vector), or NULL for zeros.
 * Outputs [N] / [N,3] / [N] / [N,geo_feat_dim]: density = exp(pre-activation), rgb = sigmoid(head) (NULL: the colour half is skipped and
 * head_weights may be NULL; so may directions, in point mode only), pre_activation and geo_feature optional.  One launch, no workspace.
 * Unsupported shapes return SDFB200_EUNSUPPORTED.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct sdfb200_nerfacto {
  int32_t hidden_dim;             /* base MLP width: 16, 32 or 64 */
  int32_t n_hidden_layers;        /* num_layers - 1: 1, 2 or 3 */
  int32_t hidden_dim_color;       /* colour MLP width: 16, 32 or 64 */
  int32_t n_hidden_layers_color;  /* num_layers_color - 1: 1, 2 or 3 */
  int32_t geo_feat_dim;           /* <= 15 */
  int32_t appearance_dim;         /* 16 + geo_feat_dim + appearance_dim <= 64 */
  int32_t contraction;            /* SDFB200_CONTRACT_* (used when aabb == NULL) */
  int32_t n_samples;              /* samples per ray (ray mode), 0 = point mode */
} sdfb200_nerfacto_t;

int sdfb200_nerfacto_field_forward(const sdfb200_grid_t* grid, const sdfb200_nerfacto_t* f, const void* table, const float* base_weights,
                                   const float* head_weights, const float* aabb, const float* origins, const float* directions,
                                   const float* bins, int64_t n_rays, const float* appearance, int64_t appearance_stride, float* density,
                                   float* rgb, float* pre_activation, float* geo_feature, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Vanilla NeRF background field (background_model="mlp" of the surface presets, models/base_surface_model.py:188-201): the eval
 * forward of NeRFField (nerfstudio/fields/vanilla_nerf_field.py:91-114 through fields/base_field.py:104-123) as ONE launch of the
 * fused tensor-core kernel k_nerf_field_tc (precision bf16x3 or bf16).
 * Family: base MLP 8 x 256 ReLU with the skip at layer 4, head MLP 2 x 128 ReLU, NeRFEncoding position / direction encodings with
 * 0..10 frequencies (the host passes the frequencies 2**linspace(min, max, n) as torch computes them), with or without the input,
 * positional encoding 1..63 columns wide.  sdfb200_nerf_field_in_family tells whether a descriptor is in it; the other entry points
 * return SDFB200_EUNSUPPORTED (packed_bytes: 0) for one that is not.
 * Geometry: ray mode (n_samples = S > 0): origins / directions [n_rows,3], bins [n_rows,S+1] euclidean edges, positions = midpoints
 * origins + directions * (start + end) / 2, N = n_rows * S.  Point mode (n_samples = 0): origins = positions [n_rows,3], directions
 * [n_rows,3], N = n_rows.  Then `contraction`.
 * Pack: weights[12] / biases[12] = nn.Linear weight [out, in] / bias [out] of mlp_base.layers.0..7, mlp_head.layers.0..1,
 * field_output_density.net, field_heads.0.net (fp32 device pointers), into `packed` (sdfb200_nerf_field_packed_bytes).
 * Forward: density [N] = softplus(.), rgb [N,3] = sigmoid(.).  One launch, no workspace.
 * ------------------------------------------------------------------------------------------------------------- */
#define SDFB200_NERF_MAX_FREQS 10
typedef struct sdfb200_nerf_field {
  int32_t base_layers;            /* mlp_base: number of Linear layers (8) */
  int32_t base_width;             /* 256 */
  int32_t skip_layer;             /* the layer that takes cat([encoding, x]): 4 */
  int32_t head_layers;            /* mlp_head: number of Linear layers (2) */
  int32_t head_width;             /* 128 */
  int32_t pe_frequencies;         /* position NeRFEncoding: num_frequencies (0..10) */
  int32_t pe_include_input;
  float pe_freqs[SDFB200_NERF_MAX_FREQS];
  int32_t dir_frequencies;        /* direction NeRFEncoding */
  int32_t dir_include_input;
  float dir_freqs[SDFB200_NERF_MAX_FREQS];
  int32_t contraction;            /* SDFB200_CONTRACT_* */
  int32_t n_samples;              /* samples per ray (ray mode), 0 = point mode */
  int32_t precision;              /* SDFB200_PRECISION_BF16X3 or _BF16 */
} sdfb200_nerf_field_t;

int sdfb200_nerf_field_in_family(const sdfb200_nerf_field_t* f);
size_t sdfb200_nerf_field_packed_bytes(const sdfb200_nerf_field_t* f);
int sdfb200_nerf_field_pack(const sdfb200_nerf_field_t* f, const float* const* weights, const float* const* biases, void* packed, void* stream);
int sdfb200_nerf_field_forward(const sdfb200_nerf_field_t* f, const void* packed, const float* origins, const float* directions, const float* bins,
                               int64_t n_rows, float* density, float* rgb, void* stream);

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

/* Segmented packed samples (nerfacc 0.3.5 render_weight_from_alpha / accumulate_along_rays as models/neus_acc.py:102-120 calls them):
 * the samples of ray r are [offsets[r], offsets[r+1]) of the flat list; offsets [n_rays+1] int64, offsets[0] = 0, non-decreasing.
 * Deterministic (fixed-order double sums, no atomics).
 * weights[i] = alphas[i] * prod_{j in segment, j < i} (1 - alphas[j])   (no +1e-7, unlike sdfb200_weights_from_alphas). */
int sdfb200_packed_weights(const float* alphas, const int64_t* offsets, int64_t n_rays, float* weights, void* stream);
/* out [n_rays, n_channels] = per-segment sum of weights * values ([N, n_channels]); values == NULL (n_channels = 1): sum of weights.
 * An empty segment gives 0. */
int sdfb200_packed_accumulate(const float* weights, const float* values, int32_t n_channels, const int64_t* offsets, int64_t n_rays,
                              float* out, void* stream);
/* g_weights [N] -> g_alphas [N]: T_k (g_k - S_k), S_k = g_{k+1} alpha_{k+1} + (1 - alpha_{k+1}) S_{k+1}; no division (finite at alpha = 1). */
int sdfb200_packed_weights_backward(const float* alphas, const int64_t* offsets, int64_t n_rays, const float* g_weights, float* g_alphas,
                                    void* stream);
/* g_out [n_rays, n_channels] -> g_weights [N] = sum_c g_out[r_i, c] values[i, c] (or g_out[r_i]), g_values [N, n_channels] =
 * weights[i] g_out[r_i, c]; either output may be NULL.  ray_indices [N] int64 in [0, n_rays). */
int sdfb200_packed_accumulate_backward(const float* weights, const float* values, int32_t n_channels, const int64_t* ray_indices,
                                       int64_t n_samples_total, const float* g_out, float* g_weights, float* g_values, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Occupancy grid of the neus-acc sampler (NeuSAccSampler, model_components/ray_samplers.py:1315-1503).  binary: the [res,res,res] bool
 * grid (1 byte per voxel), voxel (x, y, z) at x*res^2 + y*res + z.
 * ------------------------------------------------------------------------------------------------------------- */
/* update_binary_grid's test (:1405-1424) on the n occupied voxels: sdf [n] at their centres, voxel_indices [n] int64 flat indices.
 * alpha = ((p + 1e-5) / (c + 1e-5)).clip(0, 1) with c / p from sigmoid((max(|sdf| - bound, 0) +/- half_step) * inv_s[0]); voxels with
 * !(alpha > alpha_thres) are cleared, no voxel is set. */
int sdfb200_occupancy_prune(const float* sdf, const int64_t* voxel_indices, int64_t n, float bound, float half_step, const float* inv_s,
                            float alpha_thres, uint8_t* binary, void* stream);
/* nerfacc 0.3.5 ray_marching, AABB contraction, cone_angle = 0, dt = step_size: a sample (t0, t1) is kept where the midpoint lies in an
 * occupied voxel of roi_aabb (HOST float[6] = min xyz, max xyz); empty voxels are skipped to the next voxel boundary in whole steps.
 * Rays stop at t_mid >= far, when a step no longer advances t (fp32 absorption; nerfacc would not terminate), or after 2^26 loop
 * iterations.  Two passes on the same inputs: offsets == NULL counts the samples of each ray into counts [n_rays] int32; otherwise
 * offsets [n_rays] int64 (exclusive cumsum of the counts) places ray_indices [N] int64, t_starts / t_ends [N]. */
int sdfb200_occupancy_march(const float* origins, const float* directions, const float* nears, const float* fars, int64_t n_rays,
                            const float* roi_aabb, const uint8_t* binary, int32_t resolution, float step_size, const int64_t* offsets,
                            int32_t* counts, int64_t* ray_indices, float* t_starts, float* t_ends, void* stream);

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

/* Marching cubes on volume [nx, ny, nz] fp32 ('ij' order, z fastest), in place of skimage.measure.marching_cubes
 * (utils/marching_cubes.py:133-142, :201-209, :305-314).  dims (int64[3]), origin and spacing (float[3]) are HOST arrays.  A corner is
 * inside when v < level; an ambiguous face is resolved by the asymptotic decider on its four values, so a closed surface comes out
 * closed; no interior vertex.  mask [nx, ny, nz] uint8 or NULL: cube (i, j, k) is processed when mask[i, j, k] != 0.  One vertex per
 * cut edge used by a processed cube, at origin + spacing * (idx + t) with t = (level - v0) / (v1 - v0) along the edge; vertices ordered
 * by the linear index of the point that owns the edge (its +x, +y, +z edges), then by axis; faces by cube, then table order; triangles
 * wind so that their normal and the vertex normals (central-difference gradients, negated, normalised) point down the values.
 * Two passes over the same inputs, one warp per (i, j) row: offsets == NULL counts into counts (workspace of
 * sdfb200_marching_cubes_workspace_bytes(dims): int32 [2, nx*ny], each row's vertices then its faces); otherwise, with the same counts
 * and offsets [2, nx*ny] int64 = their exclusive cumsum, verts / normals [V,3] fp32 and faces [F,3] int32 are written.
 * Deterministic (no atomics). */
size_t sdfb200_marching_cubes_workspace_bytes(const int64_t* dims);
int sdfb200_marching_cubes(const float* volume, const int64_t* dims, float level, const uint8_t* mask, const float* origin,
                           const float* spacing, const int64_t* offsets, int32_t* counts, float* verts, float* normals, int32_t* faces,
                           void* stream);

/* Texture export (nerfstudio/exporter/texture_utils.py).  A texel grid is [height, width] in row-major order; its centres are
 * (linspace_w[j], linspace_h[i]) with the two vectors of get_texture_image (:59-75) on the device.  face [P] int32 and bary [P,3] fp32
 * (w0, w1, w2), P = width * height, are each texel's face and barycentric weights; the weights are rounded op by op as the reference's
 * ATen ops round them (IEEE division, no FMA contraction), so face and bary are bit-identical to the reference's.
 *
 * sdfb200_uv_rasterize: unwrap_mesh_with_xatlas' search (:265-301) over texture_coordinates [n_faces,3,2] fp32 in chunks of `chunk`
 * faces; only faces 0 .. floor(n_faces / chunk) * chunk - 1 take part.  In a chunk, the face with the smallest |w0|+|w1|+|w2| wins (lowest
 * index on ties), and a chunk that gives the texel a NaN contributes nothing; a chunk replaces the texel's face only with a strictly
 * smaller value, starting from FLT_MAX.  Texels no chunk claims keep face 0 and weights 0.  Deterministic (no atomics). */
int sdfb200_uv_rasterize(const float* texture_coordinates, int64_t n_faces, int32_t chunk, const float* linspace_w, int32_t width,
                         const float* linspace_h, int32_t height, int32_t* face, float* bary, void* stream);
/* sdfb200_uv_unwrap_grid: unwrap_mesh_per_uv_triangle (:100-192).  square_uv [6,2] fp32 = the two triangles of the first rectangle,
 * lr [2] fp32 = the rectangle's extent in UV; rectangle s holds faces 2s and 2s + 1 at column s % squares_per_side_w and row
 * s / squares_per_side_w, each (px_per_uv_triangle + 3) x px_per_uv_triangle texels.  Writes texture_coordinates [n_faces,3,2] and each
 * texel's face (clamped to n_faces - 1, so padding texels extrapolate from the last face) and bary. */
int sdfb200_uv_unwrap_grid(const float* square_uv, const float* lr, int64_t n_faces, int32_t squares_per_side_w, int32_t px_per_uv_triangle,
                           const float* linspace_w, int32_t width, const float* linspace_h, int32_t height, float* texture_coordinates,
                           int32_t* face, float* bary, void* stream);
/* sdfb200_uv_texel_rays (:194-205, :303-321, :391): per texel, origin = v0 w0 + v1 w1 + v2 w2 and direction = -normalize(n0 w0 + n1 w1 +
 * n2 w2) (F.normalize's eps) over the corners faces[face] (int64 [F,3]) of vertices / vertex_normals [V,3] fp32, then origin -= 0.5 raylen
 * direction.  raylen is a DEVICE fp32 scalar; origins / directions [P,3] and fars [P] = raylen are written.  With raylen NULL the origins
 * are not shifted and fars is not written. */
int sdfb200_uv_texel_rays(const float* vertices, const float* vertex_normals, const int64_t* faces, const int32_t* face, const float* bary,
                          const float* raylen, int64_t n_texels, float* origins, float* directions, float* fars, void* stream);

/* TSDF fusion: TSDF.integrate_tsdf (nerfstudio/exporter/tsdf_utils.py:168-270) of n_cams images, in order, into n_voxels voxels.
 * voxel_coords [3,N] fp32 (world x, y, z planes); cams [B,18] fp32 = rows 0-2 of inverse(c2w) (12 floats, row-major), then rows 0-1 of
 * K (6 floats; K's third row is never used); depth [B,H,W]; color [B,3,H,W] or NULL; truncation is a DEVICE fp32 scalar.  values,
 * weights [N] and colors [N,3] (untouched when color is NULL) are read once and written once.  Per voxel and image, every operation
 * rounded on its own (no FMA contraction, IEEE division and square root):
 *   x, y, z = ((m0 x + m1 y) + m2 z) + m3 for rows 0, 1, 2 of inverse(c2w); then y = -y, z = -z
 *   voxel_depth = sqrt((x^2 + y^2) + z^2);  u = x / z, v = y / z, w = z / z
 *   px = (k00 u + k01 v) + k02 w, py = (k10 u + k11 v) + k12 w
 *   g = (2 px) / W - 1;  ix = nearbyint(((g + 1) W - 1) / 2)   (ATen's CUDA unnormalisation; half to even), likewise iy from py and H
 *   sampled = depth[b, iy, ix], or 0 when the pixel lies outside the image or the coordinate is not finite (the reference's result for
 *             a non-finite coordinate depends on the grid_sample backend; here such a voxel is outside)
 *   dist = sampled - voxel_depth;  valid = voxel_depth > 0 && sampled > 0 && dist > -truncation   (a NaN depth is never valid)
 *   if valid: total = weight + 1;  value = (value weight + clamp(dist / truncation, -1, 1)) / total;
 *             color_c = (color_c weight + color[b, c, iy, ix]) / total;  weight = min(total, 1)
 * Kept from the reference: voxels behind a camera (z < 0) project through the mirrored point and fuse when they land in the image; the
 * depth images are compared with the Euclidean voxel_depth.  One thread per voxel, no atomics: the result depends only on the order
 * of the images, not on how they are split into calls, and reruns are bit-identical. */
int sdfb200_tsdf_integrate(const float* voxel_coords, int64_t n_voxels, const float* cams, int32_t n_cams, const float* depth,
                           const float* color, int32_t height, int32_t width, const float* truncation, float* values, float* weights,
                           float* colors, void* stream);

/* Exact k nearest neighbours of every point of a cloud among all its points, itself included at distance 0 (open3d's SearchKNN, as
 * PointCloud::RemoveStatisticalOutliers and EstimateNormals call it from exporter_utils.generate_point_cloud,
 * nerfstudio/exporter/exporter_utils.py:86-205).  The caller buckets the cloud on a grid of cells of edge h = 2^log2_cell:
 *   box [6] (HOST fp32) = min x, y, z, max x, y, z of the cloud, read back by the caller (the box sets the grid dimensions)
 *   cell_min_a = floor(box_min_a 2^-log2_cell), dims_a = floor(box_max_a 2^-log2_cell) - cell_min_a + 1 (computed in double; exact)
 *   cell of p: c_a = floor(double(p_a) 2^-log2_cell) - cell_min_a;  key = (c_z dims_y + c_y) dims_x + c_x
 *   points [N,3] fp32 = the cloud sorted by key; order [N] int32 = the original index of each sorted point;
 *   cell_start [cells + 1] int32 = the first sorted position of each key (cell_start[cells] = N)
 * Per pair, in double (fp32 converted as open3d's Vector3dVector does), every operation rounded on its own:
 *   dx = double(a_x) - double(b_x) (likewise dy, dz);  d2 = (dx dx + dy dy) + dz dz
 * The neighbours of a point are the k_eff = min(k, N) smallest (d2, original index) pairs, in that order: ties in d2 go to the lower
 * index, so the lists are fully defined and do not depend on the bucketing.  The search visits Chebyshev shells of cells around the
 * point's cell and stops once k_eff are held and the k-th d2 is at most (1 - 2^-48) times the squared distance to the nearest wall with
 * unvisited cells beyond it (the factor covers the rounding of both sides, so the result is exact).
 * Outputs, indexed by original index, either may be NULL (not both):
 *   mean_dist [N] double = (sqrt(d2_0) + sqrt(d2_1) + ... + sqrt(d2_{k_eff-1})) / k_eff, added in ascending order (__dsqrt_rn,
 *                          __dadd_rn, __ddiv_rn)
 *   indices [N,k] int32 = the neighbour list; entries k_eff..k-1 (only when N < k) are -1.  Offsets are int64.
 * Refused with SDFB200_EINVAL before any launch: k outside [1, 32], N outside [0, 2^31), both outputs NULL, a NULL input (N > 0), a
 * non-finite box (any non-finite point makes the box non-finite), box min > max, more than 2^31 - 2 cells. */
int sdfb200_knn(const float* points, const int32_t* order, int64_t n_points, const int32_t* cell_start, const float* box, int32_t log2_cell,
                int32_t k, double* mean_dist, int32_t* indices, void* stream);

/* Normals by PCA over given neighbour lists (open3d's EstimateNormals without its orientation step).  points [N,3] fp32 in original
 * order, indices [N,k] int32 (entries < 0 are skipped), normals [N,3] fp32.  Per point, in double, every operation rounded on its own:
 *   cumulants x, y, z, xx, xy, xz, yy, yz, zz summed over the list in list order, each divided by the count n;
 *   cov_ab = E[ab] - E[a] E[b]   (open3d's cumulant form)
 * then cyclic Jacobi rotations on (0,1), (0,2), (1,2) until the off-diagonal is zero, and the eigenvector of the smallest eigenvalue
 * (the first axis on ties), written as fp32.  Sign (the package's own rule; open3d's is not pinned): the component of largest
 * magnitude of the fp32 vector is positive, the first axis on ties.  A zero covariance, or an empty list, gives (0, 0, 1).
 * Refused with SDFB200_EINVAL: k outside [1, 32], N outside [0, 2^31), a NULL pointer (N > 0). */
int sdfb200_point_normals(const float* points, int64_t n_points, const int32_t* indices, int32_t k, float* normals, void* stream);

/* Mesh rendering (scripts/render_mesh.py of the reference, which draws with open3d's OpenGL visualizer): a triangle rasterizer and a
 * shader for B frames of one mesh.
 *   vertices [V,3] fp32, faces [F,3] int64 (indices in [0, V); the caller checks them), cams [B,18] fp32 = rows 0-2 of inverse(c2w)
 *   (12 floats, row-major; c2w in nerfstudio's OpenGL axes: x right, y up, looking along -z), then rows 0-1 of K (6 floats: fx at 0,
 *   cx at 2, fy at 4, cy at 5; the skew and K's third row are not read).  keys [B,H,W] uint64.
 * Per (frame, face), in double from the fp32 inputs, every operation rounded on its own (__dmul_rn, __dadd_rn, __dsub_rn, __ddiv_rn):
 *   v_k = ((m0 x + m1 y) + m2 z) + m3 for rows 0, 1, 2 of inverse(c2w)     (camera space of vertex k = 0, 1, 2)
 *   a x b = (a_y b_z - a_z b_y, a_z b_x - a_x b_z, a_x b_y - a_y b_x);  a . b = (a_x b_x + a_y b_y) + a_z b_z
 *   E_0 = v_1 x v_2, E_1 = v_2 x v_0, E_2 = v_0 x v_1;  det = v_0 . E_0
 *   the face is front-facing (counter-clockwise as seen from the camera) and non-degenerate iff det < 0; only then may it cover a
 *   pixel.  Then e_k = -E_k and num = -det (exact negations).
 * Per pixel (i, j), the ray through its centre, d = ((i + 0.5 - cx) / fx, -((j + 0.5 - cy) / fy), -1):
 *   w_k = (d_x e_k.x + d_y e_k.y) - e_k.z;  S = (w_0 + w_1) + w_2;  depth = num / S   (the view depth, -z, of the hit on the plane)
 *   the face covers the pixel iff w_0 >= 0, w_1 >= 0, w_2 >= 0, S > 0 and depth >= z_near  (edges and vertices included; NaN never
 *   covers).  key = (bits of (float)depth << 32) | face; depth > 0, so the keys order like the depths.
 * The homogeneous test needs no clipping: a face across the camera plane covers exactly the pixels whose rays meet it in front of the
 * camera, and one wholly behind it covers none.  Adjacent faces share their edge's E with opposite signs, exactly, so a closed mesh
 * leaves no holes.  keys is set to all ones (background) and every covering pair does atomicMin: the result does not depend on the
 * schedule, the binning, the order of faces of equal depth or how frames are batched, and ties go to the smaller face id.
 * Per (frame, face), a pixel box bounds the work: faces whose largest vertex depth is below z_near / 2 are skipped, and the others
 * walk the box of the projected corners of the face clipped at view depth z_near / 2 (every hit that may cover lies in that part),
 * widened by one pixel (a margin that dwarfs the rounding of the test and of the clipping).  One thread walks a box of at most SDFB200_MESH_LARGE_TRIANGLE_PIXELS pixels; a larger box is queued in
 * shared memory and walked by the whole block, one pixel per thread.
 * Refused with SDFB200_EINVAL before any launch: n_frames < 0, height or width outside [1, SDFB200_MESH_MAX_SIDE], F outside
 * [0, 2^31 - 1), z_near not finite and > 0, a NULL or misaligned pointer (vertices and cams 4 bytes, faces and keys 8) when
 * n_frames > 0 (vertices and faces may be NULL when F = 0). */
#define SDFB200_MESH_LARGE_TRIANGLE_PIXELS 256
#define SDFB200_MESH_MAX_SIDE 32768
int sdfb200_mesh_rasterize(const float* vertices, const int64_t* faces, int64_t n_faces, const float* cams, int32_t n_frames, int32_t height,
                           int32_t width, float z_near, uint64_t* keys, void* stream);
/* Shading of the keys of sdfb200_mesh_rasterize (same vertices, faces and cams) into rgb and / or normal [B,H,W,3] uint8 (either may
 * be NULL, not both).  vertex_normals [V,3] fp32 (world space).  light_positions [B,4,3] fp32 (DEVICE): each frame's four lights in
 * its camera space.  light_params [27] fp32 (HOST): per light k = 0..3 colour r, g, b, diffuse, specular, shininess, then the ambient
 * colour r, g, b.  Background pixels are white (255).  Per covered pixel, in double: the face's v_k, e_k, w_k, S and depth exactly as
 * the rasterizer computes them, barycentrics b_k = w_k / S, hit p = depth d, and the vertex normals in camera space n_k = R n (R the
 * rotation rows of inverse(c2w)).
 *   normal: n = normalize((b_0 n_0 + b_1 n_1) + b_2 n_2), colour n / 2 + 1/2
 *   rgb:    each n_k with n_k . (-v_k) < 0 is negated first; n as above, e = normalize(-p); per light, l = normalize(L_k - p),
 *           r = 2 (n . l) n - l, colour = ambient + sum_k colour_k (diffuse_k max(0, n . l) + specular_k max(0, e . r)^shininess_k)
 *   byte = floor(clamp(colour, 0, 1) 255 + 0.5).
 * Refused as sdfb200_mesh_rasterize, and when both outputs are NULL. */
int sdfb200_mesh_shade(const uint64_t* keys, int32_t n_frames, int32_t height, int32_t width, const float* vertices, const float* vertex_normals,
                       const int64_t* faces, int64_t n_faces, const float* cams, const float* light_positions, const float* light_params,
                       uint8_t* rgb, uint8_t* normal, void* stream);

/* Poisson surface reconstruction (the mesh of open3d's TriangleMesh.create_from_point_cloud_poisson, which the reference's
 * ns-export poisson calls), as a screened Poisson problem on a dense grid.  The discretisation:
 *   cube   c = the centre of the box of the points that take part, W = scale * (largest box extent), scale = 1.1; n = 2^depth cells per
 *          side, h = W / n, origin o = c - W / 2, (n+1)^3 nodes at o + h (i, j, k), depth in [1, 10].  Node (i, j, k) has linear index
 *          (i (n+1) + j) (n+1) + k and cell (x, y, z) key (x n + y) n + z (z fastest, the layout of sdfb200_marching_cubes).
 *   point  t = (p - o) / h in double, cell = clamp(floor(t), 0, n-1), u = t - cell; corner l = (lx, ly, lz) = 4 lx + 2 ly + lz of the
 *          cell has hat phi_l = prod (l_a ? u_a : 1 - u_a).  Points with a zero or non-finite normal take no part in anything; normals
 *          are normalised before use.
 *   system (L + alpha a S) x = a b, chi = sum x_i phi_i (Q1 hats):
 *          L   the Q1 stiffness matrix with natural boundaries: element entries h/3 (same node), 0 (differ in one axis), -h/12 (two or
 *              three); interior stencil 8h/3 centre, 0 face, -h/6 edge, -h/12 corner neighbours; zero row sums.
 *          b_i = sum_p n_p . grad(phi_i)(p)          S_ij = sum_p phi_i(p) phi_j(p)
 *          alpha = SDFB200_POISSON_POINT_WEIGHT,  a = h^2 (cells holding a point) / N, N the points that take part.
 *   iso    the mean over the points of chi(p), summed in double in a fixed order.
 *   density / colour: the hats' sums sum_p phi_i(p) and sum_p phi_i(p) rgb_p on the grid of depth max(depth - 2, 0), interpolated at the
 *          mesh vertices; colour = colour sum / density, 0 where the density is 0.
 * S enters as per-cell 8x8 blocks M_c = sum_{p in c} phi phi^T (row = corner).  Every sum runs over the points of one cell in the
 * caller's bucket order (a stable sort by cell key), then over a node's <= 8 adjacent cells in the order x, then y, then z offset, low
 * first; accumulation is in double, results are stored as fp32.  No floating-point atomics anywhere: reruns are bit-identical.
 *
 * sdfb200_poisson_cells: for the n_cells occupied cells of the grid 2^level (keys cell_key [n_cells] int64, points of cell s at
 * cell_start[s] .. cell_start[s+1]-1 of points [*,3] fp32), with normals [*,3]: mat [n_cells,8,8] = M_c and rhs [n_cells,8] = the cell's
 * part of b; with colors [*,3] instead: splat [n_cells,8,4] = per corner (sum phi, sum phi r, sum phi g, sum phi b).  origin (double[3])
 * and h are the level's, on the host.
 * sdfb200_poisson_coarsen: mat of the occupied cells of level `level` (cell_key) from the blocks of level + 1 (fine_slot [(2n)^3] int32,
 * -1 for an empty cell, fine_mat): M_C = sum over the 8 children (x, y, z offset order) of Q^T M_c Q, Q the coarse hats on the child.
 * This is S evaluated with the coarse hats; the coarse L is the stiffness at the coarse h.
 * sdfb200_poisson_gather: node_vals [(n+1)^3, channels] fp32 = per node the sum over its adjacent occupied cells (cell_slot [n^3]) of
 * cell_vals[slot * cell_stride + corner * corner_stride + ch], corner the node's corner of that cell.
 * sdfb200_poisson_sample: out [n_points, channels] double = the trilinear interpolation of node_vals at the points.
 * sdfb200_poisson_apply: y = (L + alpha_a S) x at level `level` with cell size h.
 * sdfb200_poisson_solve: x = the solution of (L + alpha_a S) x = rhs at `depth` (rhs = a b, caller-owned; x written).  cell_slot[l] and
 * mat[l], l = 1 .. depth (host arrays of device pointers, index l), are each level's slots and blocks.  Conjugate gradients
 * preconditioned by one V-cycle per iteration: two l1-Jacobi sweeps x += 1.4 (f - A x) / (l1 row sum of A) before and after, the Q1
 * transfer operators, a dense Cholesky solve on the 3^3 nodes of level 1.  Stops when ||rhs - A x||_2 <= tol ||rhs||_2 (the true
 * residual, recomputed whenever the recurrence says so) or after max_cycles; *cycles and *rel_residual (host) report the iterations and
 * the final true relative residual.  Synchronises `stream` once per reduction.  workspace: sdfb200_poisson_workspace_bytes(depth) bytes.
 * sdfb200_poisson_sum: *out (device) = the sum of values [n] double over a fixed partition (partial: 1024 doubles of scratch).
 * All refuse bad arguments with SDFB200_EINVAL before any launch. */
#define SDFB200_POISSON_POINT_WEIGHT 4.0
int sdfb200_poisson_cells(const float* points, const float* normals, const float* colors, int64_t n_cells, const int64_t* cell_key,
                          const int64_t* cell_start, int32_t level, const double* origin, double h, float* mat, float* rhs, float* splat,
                          void* stream);
int sdfb200_poisson_coarsen(int32_t level, const int32_t* fine_slot, const float* fine_mat, int64_t n_cells, const int64_t* cell_key,
                            float* mat, void* stream);
int sdfb200_poisson_gather(int32_t level, const int32_t* cell_slot, const float* cell_vals, int32_t cell_stride, int32_t corner_stride,
                           int32_t channels, float* node_vals, void* stream);
int sdfb200_poisson_sample(const float* points, int64_t n_points, int32_t level, const double* origin, double h, const float* node_vals,
                           int32_t channels, double* out, void* stream);
int sdfb200_poisson_apply(int32_t level, double h, const int32_t* cell_slot, const float* mat, double alpha_a, const float* x, float* y,
                          void* stream);
size_t sdfb200_poisson_workspace_bytes(int32_t depth);
int sdfb200_poisson_solve(int32_t depth, double h, const int32_t* const* cell_slot, const float* const* mat, double alpha_a,
                          const float* rhs, float* x, int32_t max_cycles, double tol, void* workspace, size_t workspace_bytes,
                          int32_t* cycles, double* rel_residual, void* stream);
int sdfb200_poisson_sum(const double* values, int64_t n, double* partial, double* out, void* stream);

/* Training path: backward of sdfb200_render (expected depth) / sdfb200_render_alphas' compositing w.r.t. the per-sample
 * inputs (autograd over renderers.py:42-295 in the reference).  `accumulation`, `depth` = forward outputs (depth BEFORE the
 * global clip).  g_rgb [R,3], g_depth [R], g_normal [R,3], g_accumulation [R], g_weights_in [R,S]: incoming gradients, each
 * may be NULL.  Outputs: g_weights [R,S] (required), g_rgb_samples / g_normal_samples [R,S,3] (may be NULL). */
int sdfb200_render_backward(const float* weights, const float* rgb, const float* normals, const float* euclid_bins, const float* bg,
                            int32_t bg_mode, int64_t n_rays, int32_t n_samples, const float* accumulation, const float* depth,
                            const float* g_rgb, const float* g_depth, const float* g_normal, const float* g_accumulation,
                            const float* g_weights_in, float* g_weights, float* g_rgb_samples, float* g_normal_samples, void* stream);

/* backward of sdfb200_render_packed (before its depth clip) w.r.t. the per-sample inputs, in any sample order; nerfacc's
 * accumulate_along_rays is differentiable in the reference (renderers.py:78-79, 194, 251-252).  `accumulation`, `depth` [n_rays] = forward
 * outputs; g_rgb [R,3], g_depth [R], g_normal [R,3], g_accumulation [R] may each be NULL.  Outputs: g_weights [N] (required),
 * g_rgb_samples / g_normal_samples [N,3] and g_steps [N] (d/d (starts + ends) / 2) may be NULL; each is zero where its incoming gradient
 * is NULL or the sample's ray index lies outside [0, n_rays).  bg_mode: SDFB200_BG_COLOR or SDFB200_BG_PER_RAY. */
int sdfb200_render_packed_backward(const float* weights, const float* rgb, const float* normals, const float* starts, const float* ends,
                                   const int64_t* ray_indices, int64_t n_samples_total, int64_t n_rays, const float* bg, int32_t bg_mode,
                                   const float* accumulation, const float* depth, const float* g_rgb, const float* g_depth,
                                   const float* g_normal, const float* g_accumulation, float* g_weights, float* g_rgb_samples,
                                   float* g_normal_samples, float* g_steps, void* stream);

/* backward of sdfb200_weights_from_alphas (from_density = 0) or sdfb200_weights_from_density (from_density = 1):
 * g_weights [R,S] (+ the gradient of the returned transmittance) -> g_in [R,S].  g_transmittance may be NULL; otherwise
 * g_transmittance_cols = 1 (alphas only: [R], gradient of transmittance[:, -1] = bg_transmittance, models/neus.py:101) or the
 * full width of the transmittance output ([R,S+1] for alphas, [R,S] for densities; models/volsdf.py:67-68 back-propagates
 * through transmittance[:, -1] of the density form). */
int sdfb200_weights_backward(const float* alphas_or_density, const float* euclid_bins, int32_t from_density, int64_t n_rays,
                             int32_t n_samples, const float* g_weights, const float* g_transmittance, int32_t g_transmittance_cols,
                             float* g_in, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Training path: the interlevel loss that trains the proposal networks.  Replaces interlevel_loss (mip-NeRF 360,
 * model_components/losses.py:38-112) and interlevel_loss_zip (Zip-NeRF, :116-172) for one proposal level.
 * fine_bins [R,Sf+1], fine_weights [R,Sf]: the final level's spacing bin edges and weights (constants);
 * proposal_bins [R,Sp+1], proposal_weights [R,Sp]: the proposal level's.  1 <= Sf, Sp <= 1024.
 * form OUTER: elements max(w - w_outer, 0)^2 / (w + 1e-7) over the R*Sf fine samples; form ZIP: the fine histogram blurred
 * with radius blur_radius (> 0) and resampled on the proposal edges, elements max(w_gt - wp, 0)^2 / (wp + 1e-5) over the R*Sp
 * proposal samples.  Outputs: loss_per_ray [R] (required; the sum of a ray's elements), loss [1] (the mean over all elements,
 * the per-ray sums added in a fixed order; NULL: not computed) and grad_proposal_weights [R,Sp] =
 * d loss_per_ray[r] / d proposal_weights[r, :] (NULL: not computed).  No atomics: the same inputs give the same bits.
 * One launch, two with `loss`.  n_rays = 0 launches nothing and writes nothing.
 * ------------------------------------------------------------------------------------------------------------- */
enum { SDFB200_INTERLEVEL_OUTER = 0, SDFB200_INTERLEVEL_ZIP = 1 };
int sdfb200_interlevel_loss(const float* fine_bins, const float* fine_weights, int32_t n_fine, const float* proposal_bins,
                            const float* proposal_weights, int32_t n_proposal, int64_t n_rays, int32_t form, float blur_radius,
                            float* loss_per_ray, float* loss, float* grad_proposal_weights, void* stream);


/* ---------------------------------------------------------------------------------------------------------------
 * Training path: dense-layer GEMMs on wgmma (bf16x3 = parity grade, bf16 = fast), fp32 row-major in / out.  They replace the ATen /
 * cuBLAS matmuls autograd runs for every nn.Linear of SDFField when the reference trains (sdf_field.py:400-409 through
 * engine/trainer.py:319-323): forward Y = X W^T (+ bias, activation), input gradient dX = dY W, weight gradient dW = dY^T X.  The set is
 * closed under differentiation (each one's backward is the other two), which is what the eikonal term's double backward needs
 * (sdf_field.py:646-655, create_graph=True).  P = number of points (the long dimension); N, K = layer widths.  Buffers of width N / K
 * must be allocated with their row padded to a multiple of 16 floats (ld >= pad16(width)); padding columns of outputs are written
 * (zeros for epilogue 0 without bias, epilogue(bias) otherwise), padding columns of inputs are ignored.
 * workspace >= sdfb200_gemm_workspace_bytes(), aligned to 16 bytes.  W is [N, K] with ldw >= K in all three; tn needs lda >= N,
 * ldb >= K and ldc >= K.  nt / nn read X 16 bytes at a time and bias / Y 8 bytes at a time: X must be aligned to 16 bytes, Y and bias
 * to 8 (ldx, ldy multiples of 4 keep every row so).  A call that breaks one of these, or has P < 0, returns -1 before any launch.
 * epilogue: 0 none, 1 softplus(beta = 100), 2 relu.  bias [pad16(N)] or NULL (NULL only with epilogue 0).
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
/* sizeof() of the ABI structs (0 grid, 1 field, 2 field_params, 3 field_in, 4 field_out, 5 render_out, 6 field_render,
 * 7 nerfacto, 8 nerf_field): lets a binding
 * verify its struct mirrors before the first call. */
size_t sdfb200_struct_size(int32_t which);

#ifdef __cplusplus
}
#endif
#endif /* SDFB200_H_ */
