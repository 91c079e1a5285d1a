// Shared declarations of the fused tensor-core field kernel: constants, launch arguments, launchers (one translation unit per
// (planes, table layout) instantiation: csrc/field_tc_p*_*.cu) and the host side (csrc/field_tc.cu).
#pragma once
#include "field_plan.h"

namespace sdfb200 {


constexpr int kEpiWarps = 8;                                 // two consumer warpgroups: MMAs + epilogues, 64 tile rows each
constexpr int kEpiThreads = kEpiWarps * 32;
constexpr int kTcThreads = kEpiThreads + 128;                // + one producer warpgroup (one thread streams the weights)
// register split after setmaxnreg.  The launch gets 168 per thread (65536 / 384, rounded down to a multiple of 8); the consumers can
// only take what the producer warpgroup gives back: 256 x (240 - 168) = 128 x (168 - 24)
constexpr int kConsumerRegs = 240;
constexpr int kProducerRegs = 24;
static_assert(2 * (kConsumerRegs - 168) <= 168 - kProducerRegs, "setmaxnreg.inc would wait for registers nobody frees");
constexpr int kStages = 5;        // weight ring depth (16 KB per stage at two planes, next to the 128 KB A operand)
constexpr int kKB = 16;           // K per streamed weight block of the 256-row layers (one 16 KB stage at two planes)
constexpr int kMaxGridDim = 32;
constexpr int kMaxPe = 60;        // PE columns (2 * 3 * degree), degree <= 10
constexpr int kPeRows = 64;       // rows reserved for the PE jacobian in the scratch
constexpr int kInK = 96;          // padded K of the two small-K operands (geo input, colour misc input)
constexpr float kHalfPiF = 1.5707963267948966f;
// kernel order of the geo input columns (K = 96): [grid features 0..31 | PE | x(3) | zero padding] -- every group of four hash
// levels is one aligned 16-byte operand chunk.  W0 (columns) and W0^T (rows) are permuted accordingly at pack time.
constexpr uint32_t kAPlane = 32 * 2048;   // one bf16 plane of the A operand: [K/8 = 32][128 rows][16 B]
// per-CTA scratch: softplus'(z1) unorm16 [64 KB] | h2 planes [P x 64 KB] | input jacobian (PE [64][128] f32 | grid [96][128] f32)
constexpr size_t kJRBytes = (size_t)(kPeRows + kMaxGridDim * 3) * 128 * 4;
__host__ __device__ constexpr size_t kScratchPerCta(int planes) { return 65536 + (size_t)planes * 65536 + kJRBytes; }

// layers in the order the kernel runs them (and the producer streams them)
enum { L_G0 = 0, L_G1, L_B1, L_B0, L_C0MISC, L_C0H, L_C1, L_COUNT };

// Weight tile of layer L: N rows (the MMA's N; B0's 96 input rows padded to 128), K (the geo input and the colour misc operand are
// kInK wide) and the K per streamed block.  Every block is exactly one ring stage (256 x kKB elements per plane): the pack plan, the
// producer and the MMAs all take the shapes from here.
__host__ __device__ constexpr int tc_layer_np(int L) { return L == L_B0 ? 128 : 256; }
__host__ __device__ constexpr int tc_layer_k(int L) { return L == L_G0 || L == L_C0MISC ? kInK : 256; }
__host__ __device__ constexpr int tc_layer_kblk(int L) { return kKB * 256 / tc_layer_np(L); }
constexpr bool tc_blocks_fill_stages() {
  for (int L = 0; L < L_COUNT; ++L)
    if (tc_layer_np(L) * tc_layer_kblk(L) != 256 * kKB || tc_layer_kblk(L) % 16 != 0 || tc_layer_k(L) % tc_layer_kblk(L) != 0) return false;
  return true;
}
static_assert(tc_blocks_fill_stages(), "every streamed weight block must be one full ring stage of whole K steps");

struct TcLayer {
  unsigned long long w_off;  // byte offset of the packed planes inside the blob
  int Np;                    // rows of the weight tile (MMA N, a multiple of 64)
  int nkb;                   // number of K blocks
  int kblk;                  // K per block (tc_layer_kblk)
};

struct TcArgs {
  sdfb200_grid_t grid;
  TcLayer layer[L_COUNT];
  int use_grid, pe_degree, use_pe, contraction, in_dim, pe_dim, grid_dim, app_dim, use_n_dot_v;
  int mode;  // 0: sdf only (G0, G1)   1: everything
  int n_samples, has_bins, n_tiles;
  long long n_points;
  float rgb_padding, cos_anneal;
  const float *origins, *directions, *bins, *appearance, *variance, *beta, *beta_min;
  const void* table;
  const char* blob;
  // fp32 section offsets (bytes)
  unsigned long long b_g0, b_g1, b_g2, w_g2, b_c0, b_c1, w_c2, b_c2;   // b_c0 = fused bias (bc0 + Wgf b2')
  char* scratch;
  unsigned long long scratch_per_cta;
  sdfb200_field_out_t out;
  TcRender rnd;
};

// one launcher per instantiation
int launch_field_tc_p2_torch(const TcArgs& a, int grid, size_t smem, cudaStream_t st);
int launch_field_tc_p2_tcnn(const TcArgs& a, int grid, size_t smem, cudaStream_t st);
int launch_field_tc_p1_torch(const TcArgs& a, int grid, size_t smem, cudaStream_t st);
int launch_field_tc_p1_tcnn(const TcArgs& a, int grid, size_t smem, cudaStream_t st);

}  // namespace sdfb200
