// fp16-table instantiations of k_hash_mlp_field (hash_mlp.cuh; tiny-cuda-nn's own storage precision)
#include "hash_mlp.cuh"

namespace sdfb200 {
int launch_hash_mlp_f16(const HashMlpArgs& a, int h, int hc, cudaStream_t st) { return launch_hash_mlp_t<__half>(a, h, hc, st); }
}  // namespace sdfb200
