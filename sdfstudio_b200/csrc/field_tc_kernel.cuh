// Fused tensor-core evaluation of the SDF field (SDFB200_PRECISION_BF16X3 / _BF16) for the neus-facto family of shapes:
// geo MLP in-256-256-(1+256), colour MLP cin-256-256-3, analytic d sdf/dx, 2-feature hash grid (fp32 or fp16 table),
// optionally followed IN THE SAME KERNEL by the per-ray compositing (alpha / density -> transmittance -> weights -> rgb, depth,
// normal, accumulation: cameras/rays.py:131-230, model_components/renderers.py:53-118,171-261,284-295).
//
// Persistent CTAs, one 128-point tile at a time.  Two consumer warpgroups own 64 rows of the tile each and run every layer as wgmma
// m64n256k16 (m64n128k16 for B0; accumulator in registers, A operand in shared memory, weights streamed through a shared-memory
// ring filled by 1-D bulk copies from a pre-packed image).  A warpgroup only reads and writes its own rows of the A operand, so the
// two warpgroups meet only at the weight ring and at the per-point heads / compositing.  A third warpgroup gives its registers to
// the consumers (setmaxnreg) and keeps one thread filling the ring, so no consumer warpgroup stalls while a slot is being freed.
// Per tile (everything stays on chip except three L2-resident spills):
//   encode   one thread per point for position, contraction, hash gathers (+ jacobian), one for PE
//            -> bf16 split planes of the geo input (A operand columns 0..95)
//   G0 G1    h = softplus_100(W a + b), epilogue in registers, written over the A operand as the next layer's input
//   sdf      fp32 dot of h2 with row 0 of W2 on CUDA cores (exact fp32: the SDF drives NeuS alpha / Laplace density)
//   (no G2)  the geo feature is linear in h2, so colour layer 0 is pre-multiplied at pack time: Wc = Wgf W2', and h2 itself
//            (bf16 planes) takes an L2-resident round trip across the reverse sweep
//   B1 B0    reverse sweep: g2 = W2[0,:]*sp'(z2), g1 = (W1^T g2)*sp'(z1), gin = W0^T g1;  sp'(z1) spilled at G0
//   grad     d sdf/dx = gin_x + PE jacobian + grid jacobian / 4      (what autograd computes at sdf_field.py:647-654)
//   C0 C1    relu MLP on [x, dir-enc, grad, geo feature, appearance] (misc columns first, h2 accumulated onto them);
//            last 256->3 layer as fp32 dots; sigmoid + padding
//   heads    Laplace density, NeuS alpha, occupancy, normals; optional per-sample outputs
//   render   (fused mode) segmented prefix product over the rays of the tile in double, weights, per-ray sums
// MMA = wgmma bf16 x bf16 -> fp32.  bf16x3: a0*w0 + a1*w0 + a0*w1 with a = a0+a1, w = w0+w1 (error ~2^-16 relative, fp32 accumulate).
#pragma once
#include "field_tc.h"
#include "grid.cuh"
#include "tc_common.cuh"

namespace sdfb200 {
using namespace tc;

__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// sample position of point p (ray r, sample s): o + d * t_start, then SceneContraction (cameras/rays.py:61-73,
// spatial_distortions.py:66-73).  Also returns the ray direction, the bin start and the bin width.
struct PointGeom { float px, py, pz, dx, dy, dz, delta, t0, t1; long long ray; };
__device__ __forceinline__ PointGeom point_geom(const TcArgs& a, long long p) {
  PointGeom g;
  g.dx = g.dy = g.dz = 0.f; g.delta = 0.f; g.t0 = g.t1 = 0.f;
  g.ray = a.has_bins ? p / a.n_samples : p;
  if (a.has_bins) {
    const int smp = (int)(p - g.ray * a.n_samples);
    const float t0 = __ldg(a.bins + g.ray * (a.n_samples + 1) + smp);
    g.t0 = t0;
    g.t1 = __ldg(a.bins + g.ray * (a.n_samples + 1) + smp + 1);
    g.delta = __fsub_rn(g.t1, t0);
    g.dx = __ldg(a.directions + g.ray * 3); g.dy = __ldg(a.directions + g.ray * 3 + 1); g.dz = __ldg(a.directions + g.ray * 3 + 2);
    g.px = __fadd_rn(__ldg(a.origins + g.ray * 3 + 0), __fmul_rn(g.dx, t0));
    g.py = __fadd_rn(__ldg(a.origins + g.ray * 3 + 1), __fmul_rn(g.dy, t0));
    g.pz = __fadd_rn(__ldg(a.origins + g.ray * 3 + 2), __fmul_rn(g.dz, t0));
  } else {
    g.px = __ldg(a.origins + p * 3); g.py = __ldg(a.origins + p * 3 + 1); g.pz = __ldg(a.origins + p * 3 + 2);
    if (a.directions) { g.dx = __ldg(a.directions + p * 3); g.dy = __ldg(a.directions + p * 3 + 1); g.dz = __ldg(a.directions + p * 3 + 2); }
  }
  if (a.contraction != SDFB200_CONTRACT_NONE) {
    const float mag = a.contraction == SDFB200_CONTRACT_LINF
                          ? fmaxf(fabsf(g.px), fmaxf(fabsf(g.py), fabsf(g.pz)))
                          : sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(g.px, g.px), __fmul_rn(g.py, g.py)), __fmul_rn(g.pz, g.pz)));
    if (mag >= 1.f) {
      const float k = __fsub_rn(2.f, __fdiv_rn(1.f, mag));
      g.px = __fmul_rn(k, __fdiv_rn(g.px, mag)); g.py = __fmul_rn(k, __fdiv_rn(g.py, mag)); g.pz = __fmul_rn(k, __fdiv_rn(g.pz, mag));
    }
  }
  return g;
}

// accurate sin / sincos as real calls: one copy of the (long) range-reduction code instead of one per call site -- the roles of this
// kernel share the SM's instruction cache, and `no instruction` stalls were 20 % of all samples with everything inlined
static __device__ __noinline__ void sincos_call(float x, float* s, float* c) { sincosf(x, s, c); }
static __device__ __noinline__ float sin_call(float x) { return sinf(x); }

// Hash-grid part of the geo input of one tile (gather warps, one thread per point).  Outputs: operand chunks 0..3 (bf16 planes,
// kernel column order: four levels = one aligned 16-byte chunk) and, in the per-CTA global scratch, the grid jacobian
// [(col*3 + d)][row] (with the 1/4 of (x+2)/4 folded in).  One level at a time (smallest code).
template <int P, int LAYOUT>
__device__ __forceinline__ void encode_tile_grid(const TcArgs& a, int tile, int row, uint8_t* inA, uint8_t* enc, uint64_t pol_table) {
  float* Jg = reinterpret_cast<float*>(enc) + kPeRows * 128;
  const long long p_raw = (long long)tile * 128 + row;
  const long long p = p_raw < a.n_points ? p_raw : a.n_points - 1;
  const PointGeom g = point_geom(a, p);
  const float x01 = (g.px + 2.0f) * 0.25f, y01 = (g.py + 2.0f) * 0.25f, z01 = (g.pz + 2.0f) * 0.25f;   // sdf_field.py:384
  // one level at a time, rolled (code size): 8 gathers in flight per thread, feature columns as 2-byte operand stores
#pragma unroll 1
  for (int l = 0; l < 16; ++l) {
    float o[2] = {0.f, 0.f};
    float dj[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    if (a.use_grid && l < a.grid.n_levels && l < a.grid.active_levels) {
      LevelCtx c;
      float tv[8][2];
      level_prepare<LAYOUT>(a.grid, l, x01, y01, z01, c);
      level_fetch_rt2(a.grid, a.table, c, tv, pol_table);
      level_finish<2, LAYOUT>(a.grid, c, tv, o, dj);
    }
    store_a<P>(inA, kAPlane, row, 2 * l, o[0]);
    store_a<P>(inA, kAPlane, row, 2 * l + 1, o[1]);
    if (a.mode != 0 && l < a.grid.n_levels) {
#pragma unroll
      for (int f = 0; f < 2; ++f) {
        const int cg = l * 2 + f;
        Jg[(cg * 3 + 0) * 128 + row] = 0.25f * dj[f][0];
        Jg[(cg * 3 + 1) * 128 + row] = 0.25f * dj[f][1];
        Jg[(cg * 3 + 2) * 128 + row] = 0.25f * dj[f][2];
      }
    }
  }
}

// PE | x | zero padding: chunks 4..11 of the geo input.  Kernel column 32 + i holds PE_i, 32 + pe_dim + j holds x_j
template <int P>
__device__ __forceinline__ void encode_tile_pe(const TcArgs& a, int tile, int row, uint8_t* inA, uint8_t* enc) {
  float* Jpe = reinterpret_cast<float*>(enc);
  const long long p_raw = (long long)tile * 128 + row;
  const long long p = p_raw < a.n_points ? p_raw : a.n_points - 1;
  const PointGeom g = point_geom(a, p);
  const int deg = a.pe_degree, half = 3 * deg;
  const float pc[3] = {g.px, g.py, g.pz};
  // zero the chunks first (padding columns), then the live columns as 2-byte stores (same thread: program order)
  const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
  for (int ch = 4; ch < kInK / 8; ++ch) store_a_chunk<P>(inA, kAPlane, row, ch, z4, z4);
#pragma unroll 1
  for (int i = 0; i < a.pe_dim; ++i) {                       // sin(x 2^k) | sin(x 2^k + pi/2)   (encodings.py:194-198)
    const int ia = i >= half ? i - half : i;
    const int b = ia / deg, k = ia - b * deg;
    const float fr = (float)(1 << k);
    const float xb = b == 0 ? pc[0] : (b == 1 ? pc[1] : pc[2]);
    const float arg = i >= half ? xb * fr + kHalfPiF : xb * fr;
    float sv, cv;
    sincos_call(arg, &sv, &cv);
    store_a<P>(inA, kAPlane, row, 32 + i, a.use_pe ? sv : 0.f);
    // autograd of sin on the forward's own fp32 arguments: d/dx_b = 2^k cos(arg)
    if (a.mode != 0) Jpe[i * 128 + row] = a.use_pe ? fr * cv : 0.f;
  }
  store_a<P>(inA, kAPlane, row, 32 + a.pe_dim + 0, pc[0]);
  store_a<P>(inA, kAPlane, row, 32 + a.pe_dim + 1, pc[1]);
  store_a<P>(inA, kAPlane, row, 32 + a.pe_dim + 2, pc[2]);
}

// static colour-operand columns of a tile (kernel columns 8..95 = chunks 1..11): x(3) | dir-enc(24) | dir(3) | appearance | 0,
// written IN PLACE over the tile's geo input once G0 has consumed it (chunk 0 = [grad, n.v] comes from the epilogue warps)
template <int P>
__device__ __forceinline__ void colour_static_tile(const TcArgs& a, int tile, int row, uint8_t* inA) {
  const long long p_raw = (long long)tile * 128 + row;
  const long long p = p_raw < a.n_points ? p_raw : a.n_points - 1;
  const PointGeom g = point_geom(a, p);
  const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
  for (int ch = 1; ch < kInK / 8; ++ch) store_a_chunk<P>(inA, kAPlane, row, ch, z4, z4);
  store_a<P>(inA, kAPlane, row, 8 + 0, g.px); store_a<P>(inA, kAPlane, row, 8 + 1, g.py); store_a<P>(inA, kAPlane, row, 8 + 2, g.pz);
  // direction encoding: sin(d 2^k) | sin(d 2^k + pi/2), k = 0..3, then d itself (NeRFEncoding(4, include_input), encodings.py:167-208)
#pragma unroll 1
  for (int i = 0; i < 12; ++i) {
    const int b = i >> 2;
    const float db = b == 0 ? g.dx : (b == 1 ? g.dy : g.dz);
    const float arg = db * (float)(1 << (i & 3));
    store_a<P>(inA, kAPlane, row, 8 + 3 + i, sin_call(arg));
    store_a<P>(inA, kAPlane, row, 8 + 15 + i, sin_call(arg + kHalfPiF));
  }
  store_a<P>(inA, kAPlane, row, 8 + 27, g.dx); store_a<P>(inA, kAPlane, row, 8 + 28, g.dy); store_a<P>(inA, kAPlane, row, 8 + 29, g.dz);
  if (a.appearance != nullptr) {
#pragma unroll 1
    for (int j = 0; j < a.app_dim; ++j) store_a<P>(inA, kAPlane, row, 8 + 30 + j, __ldg(a.appearance + g.ray * a.app_dim + j));
  }
}

#ifdef SDFB200_TC_TIMING
// CTA 0, first 16 tiles, row = tile: clock64() of consumer thread 0 at [0] tile start, [1..7] end of the MMAs of layer 0..6 (ring
// order), [8] end of the encode, [15] tile end; cycle sums over the tile of [9] consumer thread 0 waiting for weights (full) and
// [10] the producer waiting for a free ring slot (empty)
__device__ long long g_tc_timing[16 * 32];   // only the timing build of ONE instantiation defines SDFB200_TC_TIMING
#define TC_PUT(tno, k, v)                                                                                            \
  do {                                                                                                               \
    if (blockIdx.x == 0 && (tno) >= 0 && (tno) < 16) g_tc_timing[(tno) * 32 + (k)] = (v);                            \
  } while (0)
#else
#define TC_PUT(tno, k, v) do { } while (0)
#endif
#define TC_STAMP(k) do { if (tid == 0) TC_PUT(tile_no, k, TC_CLOCK()); } while (0)

// Weight ring producer (one thread of the producer warpgroup): walks every K-block of every layer of every tile of this CTA in
// consumption order and issues the bulk copy of block j once its slot has been released (all 8 consumer warps are through block
// j - kStages).  Every block of every layer is one full stage (tc_blocks_fill_stages).
template <int P>
__device__ __forceinline__ void produce_all(const TcArgs& a, int nlayers, uint8_t* ring, uint64_t* full, uint64_t* empty) {
  constexpr uint32_t kStageBytes = (uint32_t)P * 256 * kKB * 2;
  uint32_t j = 0;
  int tile_no = 0;
  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x, ++tile_no) {
    long long waited = 0;
    for (int L = 0; L < nlayers; ++L) {
      const TcLayer& ly = a.layer[L];
      for (int kb = 0; kb < ly.nkb; ++kb, ++j)
        ring_fill<kStages>(ring, full, empty, j, reinterpret_cast<const uint8_t*>(a.blob) + ly.w_off, kb, kStageBytes, &waited);
    }
    TC_PUT(tile_no, 10, waited);
  }
}

// All MMAs of layer L for the 64 rows of a warpgroup: acc (+)= A[rows, K] W^T with one m64nN wgmma per product and K step (N = 256, or
// 128 for B0: acc[0..1]), the weight K-blocks taken from the ring in order.  Every consumer warp releases a slot once its MMAs on it are
// complete (empty barrier count = 8 warps).  Each block is drained before the next is issued: with the producer in its own warpgroup and
// 5 stages, keeping one block in flight (wait_group 1) measured no faster.
template <int P, int L>
__device__ __forceinline__ void layer_mma(float (&acc)[4][32], const TcLayer& ly, bool zero, uint32_t a_base, const uint8_t* ring, uint64_t* full,
                                          uint64_t* empty, uint32_t& it, int lane, long long& waited) {
  constexpr int N = tc_layer_np(L);
  constexpr int KSTEPS = tc_layer_kblk(L) / 16;              // K steps per ring stage
  constexpr uint32_t kStageBytes = (uint32_t)P * 256 * kKB * 2;
  constexpr uint32_t lbo_b = N * 16, plane_b = N * KSTEPS * 16 * 2;
  float (&d)[N / 2] = *reinterpret_cast<float (*)[N / 2]>(&acc[0][0]);
  if (zero) {
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  }
  for (int kb = 0; kb < ly.nkb; ++kb, ++it) {
    const int s = ring_wait<kStages>(full, it, &waited);
    const uint32_t wbase = smem_u32(ring + (size_t)s * kStageBytes);
    wg_fence_acc(d);
    wg_arrive();
#pragma unroll
    for (int j = 0; j < KSTEPS; ++j) {
      const int kstep = kb * KSTEPS + j;
      wgmma_kstep_wide_ss<P, N>(d, a_desc(a_base, kstep), a_desc(a_base + kAPlane, kstep), wbase + j * 2 * lbo_b, plane_b, lbo_b);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(d);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }
}

// What a consumer thread carries through the phases of a tile
struct TileCtx {
  const TcArgs& a;
  int tid, t, wg, wrow0;     // thread (0..255), thread in its warpgroup, warpgroup, first tile row of the warpgroup
  int r0, cq;                // accumulator rows r0, r0 + 8 of the tile and the column offset in every 8-column block
  uint8_t* abuf;             // A operand of every layer: [P][32 chunks][128 rows][16 B]
  const float* prm;          // [9][256] biases / fp32 weight rows used by the epilogues (smem: broadcast loads, not one LDG each)
  float* hs;                 // [7][128] per-row inputs of the heads: sdf, gradient (3), raw rgb (3)
  float* racc;               // [8][4] per-ray accumulators of the fused compositing (rays spanning several warps)
  float* lastrgb;            // [4][3]
  double* wtot;              // [4] per-warp scan totals of the fused compositing
  float sdf_bias;
  uint32_t* sig_s;           // per-CTA scratch: softplus'(z1) as 2 x unorm16, [64 units][256 threads]
  uint32_t* gf_s;            //                  h2 as bf16x2 planes, [P][64 units][256 threads]
  uint8_t* enc_s;            //                  input jacobian: PE [64][128] f32 | grid [96][128] f32
  uint64_t pol_table, pol_keep;   // L2 policies of the hash-table gathers and of the jacobian reads
};

// encode: thread t < 64 hash gathers of row wrow0 + t, thread t >= 64 PE / x of row wrow0 + t - 64
template <int P, int LAYOUT>
__device__ __forceinline__ void encode_tile(const TileCtx& x, int tile) {
  const TcArgs& a = x.a;
  const int row = x.wrow0 + (x.t & 63);
  if (x.t < 64) {
    encode_tile_grid<P, LAYOUT>(a, tile, row, x.abuf, x.enc_s, x.pol_table);
    const long long p = (long long)tile * 128 + row;
    if (p < a.n_points) {
      const PointGeom g = point_geom(a, p);
      if (a.out.points_norm) a.out.points_norm[p] = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(g.px, g.px), __fmul_rn(g.py, g.py)), __fmul_rn(g.pz, g.pz)));
      if (a.out.points) { a.out.points[p * 3] = g.px; a.out.points[p * 3 + 1] = g.py; a.out.points[p * 3 + 2] = g.pz; }
    }
  } else {
    encode_tile_pe<P>(a, tile, row, x.abuf, x.enc_s);
  }
}

// E0 (after G0): h1 = softplus(z1) -> A ; softplus'(z1) -> scratch
template <int P>
__device__ __forceinline__ void epi_e0(const TileCtx& x, const float (&acc)[4][32]) {
  const float* p_bg0 = x.prm;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const float2 b2 = *reinterpret_cast<const float2*>(p_bg0 + col);
      float h0, h1, s0, s1;
      softplus100_fast(acc[c][i] + b2.x, h0, s0);
      softplus100_fast(acc[c][i + 1] + b2.y, h1, s1);
      store_a_pair<P>(x.abuf, kAPlane, row, col, h0, h1);
      if (x.a.mode != 0) x.sig_s[(c * 16 + (i >> 1)) * 256 + x.tid] = __float2uint_rn(s0 * 65535.0f) | (__float2uint_rn(s1 * 65535.0f) << 16);
    }
  }
}

// E1 (after G1): sdf = W2[0,:] . h2 + b (fp32) -> output / heads ; h2 -> scratch planes ; g2 = W2[0,:] * softplus'(z2) -> A
template <int P>
__device__ __forceinline__ void epi_e1(const TileCtx& x, int tile, const float (&acc)[4][32]) {
  const TcArgs& a = x.a;
  const float* p_bg1 = x.prm + 256;
  const float* p_wg2 = x.prm + 768;       // row 0 of the last geo layer
  float sp[2] = {0.f, 0.f};
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), h = (i >> 1) & 1, row = frag_row(x.r0, i);
      const float2 b2 = *reinterpret_cast<const float2*>(p_bg1 + col);
      const float2 w2 = *reinterpret_cast<const float2*>(p_wg2 + col);
      float h0, h1, s0, s1;
      softplus100_fast(acc[c][i] + b2.x, h0, s0);
      softplus100_fast(acc[c][i + 1] + b2.y, h1, s1);
      sp[h] = fmaf(w2.x, h0, sp[h]);
      sp[h] = fmaf(w2.y, h1, sp[h]);
      if (a.mode != 0) {
        uint32_t hi, lo;
        split2(h0, h1, hi, lo);
        const int u = (c * 16 + (i >> 1)) * 256 + x.tid;
        x.gf_s[u] = hi;
        if (P > 1) x.gf_s[64 * 256 + u] = lo;
        store_a_pair<P>(x.abuf, kAPlane, row, col, w2.x * s0, w2.y * s1);
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    sp[h] += __shfl_xor_sync(0xffffffffu, sp[h], 1);
    sp[h] += __shfl_xor_sync(0xffffffffu, sp[h], 2);
  }
  if ((x.t & 3) < 2) {
    const int h = x.t & 1, row = x.r0 + 8 * h;
    const float sdf = sp[h] + x.sdf_bias;
    const long long p = (long long)tile * 128 + row;
    if (p < a.n_points && a.out.sdf) a.out.sdf[p] = sdf;
    x.hs[row] = sdf;
  }
}

// EB1 (after B1): g1 = (W1^T g2) * softplus'(z1) -> A
template <int P>
__device__ __forceinline__ void epi_eb1(const TileCtx& x, const float (&acc)[4][32]) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const uint32_t sw = x.sig_s[(c * 16 + (i >> 1)) * 256 + x.tid];
      const float s0 = (float)(sw & 0xFFFFu) * (1.0f / 65535.0f), s1 = (float)(sw >> 16) * (1.0f / 65535.0f);
      store_a_pair<P>(x.abuf, kAPlane, row, col, acc[c][i] * s0, acc[c][i + 1] * s1);
    }
  }
}

// EB0 (after B0): gin (96 cols, kernel order) . input jacobian -> d sdf / dx; then the colour misc operand over the (consumed) A columns
// 0..95: chunk 0 = [grad(3), n.v, 0 x4] (sdf_field.py:572-584; columns re-ordered at pack time) from the thread pair that owns the row,
// chunks 1..11 = [x, dir-enc, dir, appearance] one thread per row
template <int P>
__device__ __forceinline__ void epi_eb0(const TileCtx& x, int tile, const float (&acc)[4][32]) {
  const TcArgs& a = x.a;
  const float* Jpe = reinterpret_cast<const float*>(x.enc_s);
  const float* Jg = Jpe + kPeRows * 128;
  const int deg = a.pe_degree, half = 3 * deg;
  float gr[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
  for (int c = 0; c < 2; ++c) {
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = frag_col(x.cq, c, i), h = (i >> 1) & 1, row = frag_row(x.r0, i);
      const float g = acc[c][i];
      if (col < 32) {
        if (col < a.grid_dim) {
#pragma unroll
          for (int d3 = 0; d3 < 3; ++d3) gr[h][d3] = fmaf(g, ld_stream_f1(Jg + (col * 3 + d3) * 128 + row, x.pol_keep), gr[h][d3]);
        }
      } else {
        // PE column i -> axis (i mod 3 deg) / deg, factor 2^k cos(arg) ; x column -> its own axis, factor 1
        const int ip = col - 32;
        if (ip < a.pe_dim) {
          const int ia = ip >= half ? ip - half : ip;
          const int ax = ia < deg ? 0 : (ia < 2 * deg ? 1 : 2);
          const float tv = g * ld_stream_f1(Jpe + ip * 128 + row, x.pol_keep);
          gr[h][0] += ax == 0 ? tv : 0.f; gr[h][1] += ax == 1 ? tv : 0.f; gr[h][2] += ax == 2 ? tv : 0.f;
        } else if (ip - a.pe_dim < 3) {
          const int ax = ip - a.pe_dim;
          gr[h][0] += ax == 0 ? g : 0.f; gr[h][1] += ax == 1 ? g : 0.f; gr[h][2] += ax == 2 ? g : 0.f;
        }
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int d3 = 0; d3 < 3; ++d3) {
      gr[h][d3] += __shfl_xor_sync(0xffffffffu, gr[h][d3], 1);
      gr[h][d3] += __shfl_xor_sync(0xffffffffu, gr[h][d3], 2);
    }
  if ((x.t & 3) < 2) {
    const int h = x.t & 1, row = x.r0 + 8 * h;
    const long long p_raw = (long long)tile * 128 + row;
    const PointGeom pg = point_geom(a, p_raw < a.n_points ? p_raw : a.n_points - 1);
    const float grx = gr[h][0], gry = gr[h][1], grz = gr[h][2];
    const float gn = fmaxf(sqrtf(grx * grx + gry * gry + grz * grz), 1e-12f);      // F.normalize eps
    const float c0v[8] = {grx, gry, grz, a.use_n_dot_v ? (grx / gn) * pg.dx + (gry / gn) * pg.dy + (grz / gn) * pg.dz : 0.f, 0.f, 0.f, 0.f, 0.f};
    store_a_chunk<P>(x.abuf, kAPlane, row, 0, c0v);
    x.hs[128 + row] = grx; x.hs[256 + row] = gry; x.hs[384 + row] = grz;
  }
  if (x.t < 64) colour_static_tile<P>(a, tile, x.wrow0 + x.t, x.abuf);
}

// C0 h2 operand: h2 (bf16 planes, saved by E1) back from the scratch over the misc columns that C0's first part has consumed
template <int P>
__device__ __forceinline__ void reload_h2(const TileCtx& x) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const int u = (c * 16 + (i >> 1)) * 256 + x.tid;
      store_a_pair<P>(x.abuf, kAPlane, row, col, x.gf_s[u], x.gf_s[64 * 256 + u]);
    }
  }
}

// EC0 (after C0): relu -> A
template <int P>
__device__ __forceinline__ void epi_ec0(const TileCtx& x, const float (&acc)[4][32]) {
  const float* p_bc0 = x.prm + 1024;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const float2 b2 = *reinterpret_cast<const float2*>(p_bc0 + col);
      store_a_pair<P>(x.abuf, kAPlane, row, col, fmaxf(acc[c][i] + b2.x, 0.f), fmaxf(acc[c][i + 1] + b2.y, 0.f));
    }
  }
}

// EC1 (after C1): relu, last colour layer (256 -> 3) as fp32 dots -> heads
__device__ __forceinline__ void epi_ec1(const TileCtx& x, const float (&acc)[4][32]) {
  const float* p_bc1 = x.prm + 1280;
  const float* p_wc2 = x.prm + 1536;      // [3][256]
  float rr[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = frag_col(x.cq, c, i), h = (i >> 1) & 1;
      const float v = fmaxf(acc[c][i] + p_bc1[col], 0.f);
      rr[h][0] = fmaf(p_wc2[col], v, rr[h][0]);
      rr[h][1] = fmaf(p_wc2[256 + col], v, rr[h][1]);
      rr[h][2] = fmaf(p_wc2[512 + col], v, rr[h][2]);
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      rr[h][k] += __shfl_xor_sync(0xffffffffu, rr[h][k], 1);
      rr[h][k] += __shfl_xor_sync(0xffffffffu, rr[h][k], 2);
    }
  if ((x.t & 3) < 2) {
    const int h = x.t & 1, row = x.r0 + 8 * h;
    x.hs[512 + row] = rr[h][0]; x.hs[640 + row] = rr[h][1]; x.hs[768 + row] = rr[h][2];
  }
}

// per-point heads (warpgroup 0, thread = tile row) and, in fused mode, the per-ray compositing
__device__ __forceinline__ void heads_and_composite(const TileCtx& x, int tile) {
  const TcArgs& a = x.a;
  const float* hs = x.hs;
  float* racc = x.racc;
  float* lastrgb = x.lastrgb;
  double* wtot = x.wtot;
  const int row = x.t, wq = x.tid >> 5, lane = x.tid & 31;
  const float* b_c2 = reinterpret_cast<const float*>(a.blob + a.b_c2);
  const long long p_raw = (long long)tile * 128 + row;
  const bool valid = p_raw < a.n_points;
  const long long p = valid ? p_raw : a.n_points - 1;
  const PointGeom pg = point_geom(a, p);
  const float dirx = pg.dx, diry = pg.dy, dirz = pg.dz, delta = pg.delta;
  const float sdf = hs[row], grx = hs[128 + row], gry = hs[256 + row], grz = hs[384 + row];
  const float gn = fmaxf(sqrtf(grx * grx + gry * gry + grz * grz), 1e-12f);      // F.normalize eps
  const float nx = grx / gn, ny = gry / gn, nz = grz / gn;
  float rgbv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float raw = hs[512 + c * 128 + row] + __ldg(b_c2 + c);
    rgbv[c] = sigmoidf_(raw) * (1.f + 2.f * a.rgb_padding) - a.rgb_padding;
  }
  float density = 0.f, alpha = 0.f;
  if (a.out.density || (a.rnd.enabled && a.rnd.from_density)) {
    const float beta = fabsf(__ldg(a.beta)) + __ldg(a.beta_min);
    const float sg = sdf > 0.f ? 1.f : (sdf < 0.f ? -1.f : 0.f);
    density = (1.0f / beta) * (0.5f + 0.5f * sg * expm1f(-fabsf(sdf) / beta));
  }
  if (a.out.alpha || (a.rnd.enabled && !a.rnd.from_density)) {
    const float inv_s = fminf(fmaxf(expf(__ldg(a.variance) * 10.0f), 1e-6f), 1e6f);
    const float true_cos = dirx * grx + diry * gry + dirz * grz;
    const float iter_cos = -(fmaxf(-true_cos * 0.5f + 0.5f, 0.f) * (1.0f - a.cos_anneal) + fmaxf(-true_cos, 0.f) * a.cos_anneal);
    const float prev_cdf = sigmoidf_((sdf - iter_cos * delta * 0.5f) * inv_s), next_cdf = sigmoidf_((sdf + iter_cos * delta * 0.5f) * inv_s);
    alpha = fminf(fmaxf((prev_cdf - next_cdf + 1e-5f) / (prev_cdf + 1e-5f), 0.f), 1.f);
  }
  if (valid) {
    if (a.out.rgb) { a.out.rgb[p * 3] = rgbv[0]; a.out.rgb[p * 3 + 1] = rgbv[1]; a.out.rgb[p * 3 + 2] = rgbv[2]; }
    if (a.out.gradients) { a.out.gradients[p * 3] = grx; a.out.gradients[p * 3 + 1] = gry; a.out.gradients[p * 3 + 2] = grz; }
    if (a.out.normals) { a.out.normals[p * 3] = nx; a.out.normals[p * 3 + 1] = ny; a.out.normals[p * 3 + 2] = nz; }
    if (a.out.density) a.out.density[p] = density;
    if (a.out.occupancy) a.out.occupancy[p] = sigmoidf_(-10.0f * sdf);
    if (a.out.alpha) a.out.alpha[p] = alpha;
  }
  if (a.rnd.enabled) {
    // ---------------- fused compositing: the tile holds 128 / S whole rays; row -> (ray, sample) = (row / S, row % S) ----------------
    const int S = a.n_samples;
    const int s_idx = row % S;
    const int rl = row / S;                                   // ray within the tile
    const bool dens = a.rnd.from_density != 0;
    // factor by which the transmittance drops across this sample: 1 - alpha + 1e-7 (rays.py:204-206), or as an exponent
    // delta * sigma for the density form (rays.py:160-170)
    const float dd = valid ? __fmul_rn(delta, density) : 0.f;
    double f = dens ? (double)dd : (valid ? (double)__fadd_rn(__fsub_rn(1.0f, alpha), 1e-7f) : 1.0);
    double incl = f;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const double o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d && s_idx >= d) incl = dens ? incl + o : incl * o;
    }
    double excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0 || s_idx == 0) excl = dens ? 0.0 : 1.0;
    if (lane == 31) wtot[wq] = incl;
    named_sync(4, 128);
    if (S > 32) {
      const int first = (wq * 32 / S) * (S / 32);
      for (int w2 = first; w2 < wq; ++w2) excl = dens ? excl + wtot[w2] : excl * wtot[w2];
    }
    const float T = dens ? expf(-(float)excl) : (float)excl;
    const float al = dens ? __fsub_rn(1.0f, expf(-dd)) : alpha;
    const float w = valid ? __fmul_rn(al, T) : 0.f;
    const float mid = __fdiv_rn(__fadd_rn(pg.t0, pg.t1), 2.0f);            // (starts + ends) / 2, renderers.py:247
    if (valid && a.rnd.weights) a.rnd.weights[p] = w;
    float vs[8] = {w, w * rgbv[0], w * rgbv[1], w * rgbv[2], w * nx, w * ny, w * nz, w * mid};
    float smin = valid ? mid : INFINITY, smax = valid ? mid : -INFINITY;
    const int span = S < 32 ? S : 32;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      if (d < span) {
#pragma unroll
        for (int k = 0; k < 8; ++k) vs[k] += __shfl_down_sync(0xffffffffu, vs[k], d);
      }
      smin = fminf(smin, __shfl_xor_sync(0xffffffffu, smin, d));
      smax = fmaxf(smax, __shfl_xor_sync(0xffffffffu, smax, d));
    }
    if (a.rnd.steps_minmax && lane == 0 && smin <= smax) { atomic_min_float(a.rnd.steps_minmax, smin); atomic_max_float(a.rnd.steps_minmax + 1, smax); }
    if (S > 32) {
      if (lane == 0) {
#pragma unroll
        for (int k = 0; k < 8; ++k) atomicAdd(&racc[k * 4 + rl], vs[k]);
      }
      if (s_idx == S - 1) { lastrgb[rl * 3] = rgbv[0]; lastrgb[rl * 3 + 1] = rgbv[1]; lastrgb[rl * 3 + 2] = rgbv[2]; }
      named_sync(4, 128);
      if (s_idx == 0) {
#pragma unroll
        for (int k = 0; k < 8; ++k) { vs[k] = racc[k * 4 + rl]; racc[k * 4 + rl] = 0.f; }
      }
    }
    // transmittance after the last sample (alphas: transmittance[:, -1] = bg_transmittance, neus.py:101) / before it (densities: volsdf.py:67-68)
    double tot;
    float lr, lg, lb;
    if (S > 32) {
      const int first = (wq * 32 / S) * (S / 32);
      tot = dens ? 0.0 : 1.0;
      const int nw = dens ? S / 32 - 1 : S / 32;
      for (int w2 = first; w2 < first + nw; ++w2) tot = dens ? tot + wtot[w2] : tot * wtot[w2];
      lr = lastrgb[rl * 3]; lg = lastrgb[rl * 3 + 1]; lb = lastrgb[rl * 3 + 2];
    } else {
      const int last = (lane - s_idx) + S - 1;
      tot = __shfl_sync(0xffffffffu, dens ? excl : incl, last);
      lr = __shfl_sync(0xffffffffu, rgbv[0], last); lg = __shfl_sync(0xffffffffu, rgbv[1], last); lb = __shfl_sync(0xffffffffu, rgbv[2], last);
    }
    if (S > 32 && dens) {
      // exclusive sum at the last sample of the ray = transmittance exponent before the last sample; it lives in the last warp of the ray
      if (s_idx == S - 1) wtot[wq] = excl;       // (wtot of the ray's last warp is no longer needed by anyone else)
      named_sync(4, 128);
      tot = wtot[(wq * 32 / S) * (S / 32) + S / 32 - 1];
    }
    const long long ray = (long long)tile * (128 / S) + rl;
    if (s_idx == 0 && ray * S < a.n_points) {
      const float acc = vs[0];
      if (a.rnd.rgb) {
        float bgc[3] = {0.f, 0.f, 0.f};
        if (a.rnd.bg_mode == SDFB200_BG_COLOR) { bgc[0] = a.rnd.bg[0]; bgc[1] = a.rnd.bg[1]; bgc[2] = a.rnd.bg[2]; }
        else if (a.rnd.bg_mode == SDFB200_BG_PER_RAY) { bgc[0] = a.rnd.bg[ray * 3]; bgc[1] = a.rnd.bg[ray * 3 + 1]; bgc[2] = a.rnd.bg[ray * 3 + 2]; }
        else { bgc[0] = lr; bgc[1] = lg; bgc[2] = lb; }
        const float rem = 1.0f - acc;
        const float o[3] = {vs[1] + bgc[0] * rem, vs[2] + bgc[1] * rem, vs[3] + bgc[2] * rem};
#pragma unroll
        for (int c = 0; c < 3; ++c) a.rnd.rgb[ray * 3 + c] = a.rnd.clamp01 ? fminf(fmaxf(o[c], 0.f), 1.f) : o[c];
      }
      if (a.rnd.accumulation) a.rnd.accumulation[ray] = acc;
      if (a.rnd.normal) { a.rnd.normal[ray * 3] = vs[4]; a.rnd.normal[ray * 3 + 1] = vs[5]; a.rnd.normal[ray * 3 + 2] = vs[6]; }
      if (a.rnd.depth) a.rnd.depth[ray] = vs[7] / (acc + 1e-10f);
      if (a.rnd.bg_transmittance) a.rnd.bg_transmittance[ray] = dens ? expf(-(float)tot) : (float)tot;
    }
  }
}

template <int P, int LAYOUT>
__global__ void __launch_bounds__(kTcThreads, 1) k_field_tc(const __grid_constant__ TcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr uint32_t kStageBytes = (uint32_t)P * 256 * kKB * 2;        // one weight K-block, all planes (the 128-row layer: K blocks of 32)
  uint8_t* abuf = smem;                                                // A operand of every layer: [P][32 chunks][128 rows][16 B]
  uint8_t* ring = smem + P * kAPlane;
  float* fbuf = reinterpret_cast<float*>(ring + kStages * kStageBytes);
  float* prm = fbuf;                  // [9][256] biases / fp32 weight rows used by the epilogues
  float* hs = prm + 9 * 256;          // [7][128] per-row inputs of the heads: sdf, gradient (3), raw rgb (3)
  float* racc = hs + 7 * 128;         // [8][4] per-ray accumulators of the fused compositing (rays spanning several warps)
  float* lastrgb = racc + 32;         // [4][3]
  __shared__ uint64_t full[kStages], empty[kStages];
  __shared__ double wtot[4];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nlayers = a.mode == 0 ? 2 : L_COUNT;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kEpiWarps); }
    fence_barrier_init();
  }
  {
    const char* blob = a.blob;
    const float* src[9] = {reinterpret_cast<const float*>(blob + a.b_g0), reinterpret_cast<const float*>(blob + a.b_g1),
                           reinterpret_cast<const float*>(blob + a.b_g1), reinterpret_cast<const float*>(blob + a.w_g2),
                           reinterpret_cast<const float*>(blob + a.b_c0), reinterpret_cast<const float*>(blob + a.b_c1),
                           reinterpret_cast<const float*>(blob + a.w_c2), reinterpret_cast<const float*>(blob + a.w_c2) + 256,
                           reinterpret_cast<const float*>(blob + a.w_c2) + 512};
    for (int i = tid; i < 9 * 256; i += kTcThreads) prm[i] = src[i >> 8][i & 255];
    if (tid < 44) racc[tid] = 0.f;
  }
  __syncthreads();

  // ============================== producer warpgroup: one thread streams the weights ==============================
  if (tid >= kEpiThreads) {
    setmaxnreg_dec<kProducerRegs>();
    if (tid == kEpiThreads) produce_all<P>(a, nlayers, ring, full, empty);
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();

  // ============================== two warpgroups, 64 rows of the tile each ==============================
  const int wg = warp >> 2, t = tid & 127;
  const int wrow0 = wg * 64;
  const int wg_bar = 1 + wg;                                 // named barrier of this warpgroup
  const uint32_t a_base = smem_u32(abuf) + wrow0 * 16;
  const float sdf_bias = __ldg(reinterpret_cast<const float*>(a.blob + a.b_g2));
  char* scr = a.scratch + (size_t)blockIdx.x * a.scratch_per_cta;
  const TileCtx x{a, tid, t, wg, wrow0, frag_row0(wrow0, t), frag_cq(t), abuf, prm, hs, racc, lastrgb, wtot, sdf_bias,
                  reinterpret_cast<uint32_t*>(scr), reinterpret_cast<uint32_t*>(scr + 65536), reinterpret_cast<uint8_t*>(scr + 65536 + (size_t)P * 65536),
                  l2_policy_evict_last(), l2_policy_evict_normal()};
  uint32_t it = 0;
  long long waited = 0;
  float acc[4][32];
#define SYNC_A()                \
  do {                          \
    fence_async_smem();         \
    named_sync(wg_bar, 128);    \
  } while (0)
#define LAYER(L, zero)                                                                                 \
  do {                                                                                                 \
    layer_mma<P, L>(acc, a.layer[L], zero, a_base, ring, full, empty, it, lane, waited);               \
    named_sync(wg_bar, 128); /* every warp of the warpgroup is done reading this layer's A operand */  \
    TC_STAMP(1 + (L));                                                                                 \
  } while (0)

  int tile_no = -1;
  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    ++tile_no;
    TC_STAMP(0);
    waited = 0;
    encode_tile<P, LAYOUT>(x, tile);
    SYNC_A();
    TC_STAMP(8);
    LAYER(L_G0, true);
    epi_e0<P>(x, acc);
    SYNC_A();
    LAYER(L_G1, true);
    epi_e1<P>(x, tile, acc);
    if (a.mode == 0) continue;                 // sdf only
    SYNC_A();
    LAYER(L_B1, true);
    epi_eb1<P>(x, acc);
    SYNC_A();
    LAYER(L_B0, true);
    epi_eb0<P>(x, tile, acc);
    SYNC_A();
    LAYER(L_C0MISC, true);
    reload_h2<P>(x);
    SYNC_A();
    LAYER(L_C0H, false);                       // accumulates onto the misc columns' result
    epi_ec0<P>(x, acc);
    SYNC_A();
    LAYER(L_C1, true);
    epi_ec1(x, acc);
    named_sync(3, kEpiThreads);                // both warpgroups' head inputs are in `hs`
    if (wg == 0) heads_and_composite(x, tile);
    named_sync(3, kEpiThreads);                // `hs` / `racc` are rewritten by the next tile
    TC_STAMP(15);
    if (tid == 0) TC_PUT(tile_no, 9, waited);
  }
#undef SYNC_A
#undef LAYER
}

template <int P, int LAYOUT>
static int launch_field_tc(const TcArgs& a, int grid, size_t smem, cudaStream_t st) {
  SDFB_CUDA(cudaFuncSetAttribute(k_field_tc<P, LAYOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_field_tc<P, LAYOUT><<<grid, kTcThreads, smem, st>>>(a);
  SDFB_LAUNCHED("k_field_tc");
  return 0;
}

}  // namespace sdfb200
