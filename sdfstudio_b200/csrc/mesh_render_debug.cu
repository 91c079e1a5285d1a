// Debug hook of the mesh rasterizer (libsdfb200_dbg.so only): sdfb200_mesh_rasterize with the large-box threshold as an argument, so
// that tools/render_mesh_bench.py can time the per-thread and the block path on their own.
#include "common.cuh"
#include "../../include/sdfb200_debug.h"

namespace sdfb200 {
int mesh_rasterize(const float* vertices, const int64_t* faces, int64_t n_faces, const float* cams, int32_t n_frames, int32_t height, int32_t width,
                   float z_near, uint64_t* keys, int64_t large_pixels, void* stream);
}

extern "C" int sdfb200_debug_mesh_rasterize(const float* vertices, const int64_t* faces, int64_t n_faces, const float* cams, int32_t n_frames,
                                            int32_t height, int32_t width, float z_near, uint64_t* keys, int64_t large_pixels, void* stream) {
  return sdfb200::mesh_rasterize(vertices, faces, n_faces, cams, n_frames, height, width, z_near, keys, large_pixels, stream);
}
