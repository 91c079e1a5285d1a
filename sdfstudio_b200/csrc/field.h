// Internal cross-file declarations of the SDF field: the grid encoder (grid_encode.cu), the generic kernels (field_simt.cu) and the
// host side of the fused tensor-core kernel (field_tc.cu).  api.cu chooses between the two engines and checks every call before
// either runs, so neither re-checks its inputs.
#pragma once
#include <cuda_runtime.h>

#include "field_plan.h"

namespace sdfb200 {

// grid_encode.cu
int validate_grid(const sdfb200_grid_t* g);
int validate_grid_pointers(const sdfb200_grid_t* g, const void* table, const float* grad);   // grad: the table gradient, or NULL
int grid_encode(const sdfb200_grid_t& g, const void* table, const float* x01, int64_t n, float* out, int64_t out_ld, float* dout_dx,
                cudaStream_t st);

// field_simt.cu: the fp32 section of the packed blob, and the generic kernels (any SDFFieldConfig shape) with GEMM engine
// gemm_planes: 0 = exact fp32 (k_sgemm), 1 / 2 = tensor-core bf16 / bf16x3 (k_tc_linear)
int field_pack_fp32(const sdfb200_field_t& f, const FieldPlan& p, const sdfb200_field_params_t& prm, char* blob, cudaStream_t st);
size_t field_generic_workspace_floats(const sdfb200_field_t& f, const FieldPlan& p, int64_t n_points);
int field_forward_generic(const sdfb200_field_t& f, const FieldPlan& p, const char* blob, const void* table, const sdfb200_field_in_t& in,
                          const sdfb200_field_out_t& out, float* ws, int gemm_planes, cudaStream_t st);

// field_tc.cu: the tensor-core section of the packed blob, and the fused kernel (p.fused).  rnd != NULL composites in the same
// launch and needs whole rays in every 128-point tile.
size_t field_tc_workspace_floats(const sdfb200_field_t& f);
int field_tc_pack(const sdfb200_field_t& f, const FieldPlan& p, char* blob, cudaStream_t st);
int field_tc_forward(const sdfb200_field_t& f, const FieldPlan& p, const char* blob, const void* table, const sdfb200_field_in_t& in,
                     const sdfb200_field_out_t& out, const sdfb200_field_render_t* rnd, float* ws, cudaStream_t st);

}  // namespace sdfb200
