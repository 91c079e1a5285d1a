// instantiation of the fused tensor-core field kernel: bf16x3 (two bf16 planes), torch-layout hash table
#include "field_tc_kernel.cuh"

namespace sdfb200 {
int launch_field_tc_p2_torch(const TcArgs& a, int grid, size_t smem, cudaStream_t st) { return launch_field_tc<2, SDFB200_GRID_TORCH>(a, grid, smem, st); }
}  // namespace sdfb200

#ifdef SDFB200_TC_TIMING
extern "C" int sdfb200_debug_tc_timing(long long* host_out_768) {
  SDFB_CUDA(cudaMemcpyFromSymbol(host_out_768, sdfb200::g_tc_timing, sizeof(sdfb200::g_tc_timing)));
  return 0;
}
#endif
