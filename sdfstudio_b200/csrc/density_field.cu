// Proposal density field: HashGrid (tcnn layout) -> narrow ReLU MLP (no biases, tiny-cuda-nn FullyFusedMLP semantics) -> exp.
// Replaces HashMLPDensityField.get_density / density_fn (nerfstudio/fields/density_fields.py:40-121, fields/base_field.py:48-65),
// i.e. tcnn.NetworkWithInputEncoding + trunc_exp (field_components/activations.py:24-42).  One thread per point: the L2-gather-bound
// grid lookup dominates (8 L corners), the <= 64-wide MLP runs in registers with the weights broadcast from shared memory.
#include "field.h"
#include "hash_mlp.cuh"

namespace sdfb200 {

struct DensityArgs {
  sdfb200_grid_t grid;
  const void* table;
  const float* weights;   // [H, in_pad] | (n_hidden-1) x [H, H] | [H]   (row-major, fp32)
  const float* positions; // [N,3]
  const float* aabb;      // [2,3] device pointer or NULL (then contraction mode)
  int contraction, n_hidden, in_dim, in_pad;
  long long n;
  float* density;         // [N]
  float* pre_activation;  // [N] or NULL
};

template <typename T, int F, int H>
__global__ void __launch_bounds__(128) k_density_field(const __grid_constant__ DensityArgs a) {
  extern __shared__ float w_s[];
  const int n_w = H * a.in_pad + (a.n_hidden - 1) * H * H + H;
  for (int i = threadIdx.x; i < n_w; i += blockDim.x) w_s[i] = __ldg(a.weights + i);
  __syncthreads();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  float x01, y01, z01;
  normalize_position(a.aabb, a.contraction, __ldg(a.positions + i * 3), __ldg(a.positions + i * 3 + 1), __ldg(a.positions + i * 3 + 2), x01, y01, z01);
  float h[H];
  const float* w = hash_mlp_hidden<T, F, H>(a.grid, a.table, w_s, a.in_pad, a.n_hidden, x01, y01, z01, h);
  float out = 0.f;
#pragma unroll
  for (int k = 0; k < H; ++k) out = fmaf(w[k], h[k], out);
  if (a.pre_activation) a.pre_activation[i] = out;
  a.density[i] = expf(out);  // trunc_exp forward = exp
}

template <typename T, int F>
static int launch_density(const DensityArgs& a, int hidden, cudaStream_t st) {
  const unsigned blocks = (unsigned)ceil_div(a.n, 128);
  const size_t smem = (size_t)(hidden * a.in_pad + (a.n_hidden - 1) * hidden * hidden + hidden) * sizeof(float);
  switch (hidden) {
    case 16: k_density_field<T, F, 16><<<blocks, 128, smem, st>>>(a); break;
    case 32: k_density_field<T, F, 32><<<blocks, 128, smem, st>>>(a); break;
    case 64:
      SDFB_CUDA(cudaFuncSetAttribute(k_density_field<T, F, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      k_density_field<T, F, 64><<<blocks, 128, smem, st>>>(a);
      break;
    default: return fail(SDFB200_EUNSUPPORTED, "density field hidden_dim must be 16, 32 or 64%s", "", 0);
  }
  SDFB_LAUNCHED("k_density_field");
  return 0;
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
  DensityArgs a;
  a.grid = *grid; a.table = table; a.weights = weights; a.positions = positions; a.aabb = aabb; a.contraction = contraction; a.n_hidden = n_hidden_layers;
  a.in_dim = grid->n_levels * grid->n_features; a.in_pad = (a.in_dim + 15) / 16 * 16; a.n = n; a.density = density; a.pre_activation = pre_activation;
  cudaStream_t st = (cudaStream_t)stream;
  const bool h16 = grid->table_dtype == SDFB200_DT_F16;
  switch (grid->n_features) {
    case 1: return h16 ? launch_density<__half, 1>(a, hidden_dim, st) : launch_density<float, 1>(a, hidden_dim, st);
    case 2: return h16 ? launch_density<__half, 2>(a, hidden_dim, st) : launch_density<float, 2>(a, hidden_dim, st);
    case 4: return h16 ? launch_density<__half, 4>(a, hidden_dim, st) : launch_density<float, 4>(a, hidden_dim, st);
    default: return h16 ? launch_density<__half, 8>(a, hidden_dim, st) : launch_density<float, 8>(a, hidden_dim, st);
  }
}
