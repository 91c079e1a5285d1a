// Shared declarations of the fused tensor-core field kernel: constants, launch arguments, launchers (one translation unit per
// (planes, table layout) instantiation: csrc/field_tc_p*_*.cu) and the host side (csrc/field_tc.cu).
#pragma once
#include "field_plan.h"

namespace sdfb200 {


constexpr int kEpiWarps = 8;                                 // two consumer warpgroups: MMAs + epilogues, 64 tile rows each
constexpr int kEpiThreads = kEpiWarps * 32;
constexpr int kTcThreads = kEpiThreads + 128;                // + one producer warpgroup: warp 8 streams the weights, warps 9..11 encode
constexpr int kEncThreads = 96;                              // encoder warps: the geo input, Jacobians and colour-static columns of tile n + 1
// register split after setmaxnreg.  The launch gets 168 per thread (65536 / 384, rounded down to a multiple of 8); the consumers can
// only take what the producer warpgroup gives back: 256 x (216 - 168) = 128 x (168 - 72)
constexpr int kConsumerRegs = 216;
constexpr int kProducerRegs = 72;
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
constexpr uint32_t kImgPlane = (kInK / 8) * 128 * 16;      // one bf16 plane of a staged 96-column operand image (24 KB)
__host__ __device__ constexpr uint32_t tc_stage_bytes(int planes) { return (uint32_t)planes * 256 * kKB * 2; }   // one weight K-block

// rows of the epilogue parameters `prm` ([kPrmRows][256] f32): biases and the fp32 weight rows of the dot-product layers
enum { PRM_B_G0 = 0, PRM_B_G1, PRM_W_G2 /* row 0 */, PRM_B_C0, PRM_B_C1, PRM_W_C2 /* rows 0..2 */, kPrmRows = PRM_W_C2 + 3 };
// rows of the head inputs `hs` of one tile ([kHsRows][128] f32, one column per tile row)
enum { HS_SDF = 0, HS_GRAD /* x, y, z */, HS_RGB = HS_GRAD + 3 /* raw r, g, b */, kHsRows = HS_RGB + 3 };

// Dynamic shared memory of k_field_tc: byte offsets from its 1024-aligned base
struct TcSmem { size_t a, ring, prm, hs, coldesc, bytes; };
__host__ __device__ constexpr TcSmem tc_smem(int planes) {
  TcSmem s{};                                                  // a: A operand of every layer [P][32 chunks][128 rows][16 B]
  s.ring = s.a + (size_t)planes * kAPlane;                     // weight ring: kStages x one K-block
  s.prm = s.ring + (size_t)kStages * tc_stage_bytes(planes);   // epilogue parameters [kPrmRows][256] f32
  s.hs = s.prm + kPrmRows * 256 * 4;                           // head inputs by tile parity [2][kHsRows][128] f32
  s.coldesc = s.hs + 2 * kHsRows * 128 * 4;                    // EB0's view of the geo input columns 32..127 [96] float4 (ColDesc)
  s.bytes = s.coldesc + 96 * 16;
  return s;
}
constexpr size_t kSmemPerBlock = 232448;  // H100: 227 KB of shared memory per block (dynamic + static)
constexpr size_t kStaticSmem = 1024;      // the kernel's static shared memory (barriers): one 1024-byte slot, the dynamic part is 1024-aligned
static_assert(tc_smem(2).bytes + kStaticSmem <= kSmemPerBlock, "shared memory of k_field_tc at two planes");

// Per-CTA scratch of k_field_tc (caller workspace): byte offsets from the CTA's base.  sig and h2 are planes of [64 units][256 threads]
// x 4 B (kFragWords) in the accumulator-fragment order of the thread that writes and later reads them.
constexpr size_t kFragWords = 64 * 256;
struct TcScratch { size_t sig, h2, slots, slot_bytes, geo, cs, jpe, jg, bytes; };
__host__ __device__ constexpr TcScratch tc_scratch(int planes) {
  TcScratch s{};                                               // sig: softplus'(z1) as 2 x unorm16
  s.h2 = s.sig + kFragWords * 4;                               // h2 as bf16x2 planes [P]
  s.slots = s.h2 + (size_t)planes * kFragWords * 4;            // two staging slots (tile parity), slot_bytes apart, each with:
  s.cs = s.geo + (size_t)planes * kImgPlane;                   //   geo input image [P][12 chunks][128 rows][16 B] at geo = 0 and the
  s.jpe = s.cs + (size_t)planes * kImgPlane;                   //   colour-static image (same layout, chunk 0 unused); PE jacobian
  s.jg = s.jpe + (size_t)kPeRows * 128 * 4;                    //   [kPeRows][128] f32, grid jacobian [kMaxGridDim * 3][128] f32
  s.slot_bytes = s.jg + (size_t)kMaxGridDim * 3 * 128 * 4;
  s.bytes = s.slots + 2 * s.slot_bytes;                        // per CTA
  return s;
}
__host__ __device__ constexpr size_t kScratchPerCta(int planes) { return tc_scratch(planes).bytes; }

// layers in the order the kernel runs them (and the producer streams them)
enum { L_G0 = 0, L_G1, L_B1, L_B0, L_C0MISC, L_C0H, L_C1, L_COUNT };

// Weight tile of layer L: N rows (the MMA's N; B0's 96 input rows padded to 128), K (the geo input and the colour misc operand are
// kInK wide) and the K per streamed block.  Every block is exactly one ring stage (256 x kKB elements per plane): the pack plan, the
// producer and the MMAs all take the shapes from here.
__host__ __device__ constexpr int tc_layer_np(int L) { return L == L_B0 ? 128 : 256; }
__host__ __device__ constexpr int tc_layer_k(int L) { return L == L_G0 || L == L_C0MISC ? kInK : 256; }
__host__ __device__ constexpr int tc_layer_kblk(int L) { return kKB * 256 / tc_layer_np(L); }
__host__ __device__ constexpr int tc_layer_nkb(int L) { return tc_layer_k(L) / tc_layer_kblk(L); }
constexpr bool tc_blocks_fill_stages() {
  for (int L = 0; L < L_COUNT; ++L)
    if (tc_layer_np(L) * tc_layer_kblk(L) != 256 * kKB || tc_layer_kblk(L) % 16 != 0 || tc_layer_k(L) % tc_layer_kblk(L) != 0) return false;
  return true;
}
static_assert(tc_blocks_fill_stages(), "every streamed weight block must be one full ring stage of whole K steps");

struct TcLayer {
  unsigned long long w_off;  // byte offset of the packed planes inside the blob
};

struct TcArgs {
  sdfb200_grid_t grid;
  TcLayer layer[L_COUNT];
  int use_grid, pe_degree, use_pe, contraction, pe_dim, grid_dim, app_dim, use_n_dot_v;
  int mode;  // 0: sdf only (G0, G1)   1: everything
  int n_samples, has_bins, n_tiles;
  long long n_points;
  float rgb_padding, cos_anneal;
  const float *origins, *directions, *bins, *appearance, *variance, *beta, *beta_min;
  const void* table;
  const char* blob;
  // fp32 section offsets (bytes)
  unsigned long long b_g0, b_g1, b_g2, w_g2, b_c0, b_c1, w_c2, b_c2;   // b_c0 = fused bias (bc0 + Wgf b2')
  char* scratch;               // tc_scratch(P).bytes per CTA
  sdfb200_field_out_t out;
  int render;                  // per-ray compositing in the same kernel (requires 128 % n_samples == 0: every tile holds whole rays)
  sdfb200_field_render_t rnd;  // (clip_depth is applied after the kernel)
};

// one launcher per instantiation
int launch_field_tc_p2_torch(const TcArgs& a, int grid, size_t smem, cudaStream_t st);
int launch_field_tc_p2_tcnn(const TcArgs& a, int grid, size_t smem, cudaStream_t st);
int launch_field_tc_p1_torch(const TcArgs& a, int grid, size_t smem, cudaStream_t st);
int launch_field_tc_p1_tcnn(const TcArgs& a, int grid, size_t smem, cudaStream_t st);

}  // namespace sdfb200
