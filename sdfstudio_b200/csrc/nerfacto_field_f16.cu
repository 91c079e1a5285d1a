// fp16-table instantiation of the nerfacto background field kernel (tiny-cuda-nn's own storage precision)
#include "nerfacto_field.cuh"

namespace sdfb200 {
int launch_nerfacto_f16(const NerfactoArgs& a, int h, int hc, cudaStream_t st) { return launch_nerfacto_h<__half>(a, h, hc, st); }
}  // namespace sdfb200
