// Fused tensor-core evaluation of the SDF field (SDFB200_PRECISION_BF16X3 / _BF16) for the neus-facto family of shapes:
// geo MLP in-256-256-(1+256), colour MLP cin-256-256-3, analytic d sdf/dx, 2-feature hash grid (fp32 or fp16 table),
// optionally followed IN THE SAME KERNEL by the per-ray compositing (alpha / density -> transmittance -> weights -> rgb, depth,
// normal, accumulation: cameras/rays.py:131-230, model_components/renderers.py:53-118,171-261,284-295).
//
// Persistent CTAs, one 128-point tile at a time.  Two consumer warpgroups own 64 rows of the tile each and run every layer as wgmma
// m64n256k16 (m64n128k16 for B0; accumulator in registers, A operand in shared memory, weights streamed through a shared-memory
// ring filled by 1-D bulk copies from a pre-packed image).  A warpgroup only reads and writes its own rows of the A operand, so the
// two warpgroups meet only at the weight ring.  A third warpgroup gives its registers to the consumers (setmaxnreg), keeps one thread
// filling the ring, so no consumer warpgroup stalls while a slot is being freed, and three encoder warps that stage the next tile and
// run the heads of the previous one.
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
//   heads    (the three encoder warps, a tile behind, 32-row chunks) Laplace density, NeuS alpha, occupancy, normals; optional
//            per-sample outputs
//   render   (fused mode, same warps) segmented prefix product over the rays of the tile in double, weights, per-ray sums
// MMA = wgmma bf16 x bf16 -> fp32.  bf16x3: a0*w0 + a1*w0 + a0*w1 with a = a0+a1, w = w0+w1 (error ~2^-16 relative, fp32 accumulate).
#pragma once
#include "field_tc.h"
#include "grid.cuh"
#include "tc_common.cuh"

namespace sdfb200 {
using namespace tc;

__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
constexpr int kEncBar = 3;   // named barrier of the encoder warps (0 is __syncthreads, 1 and 2 belong to the consumer warpgroups)

// Point p = tile * 128 + row of a call with bins (the last point for a row past the end): its ray p / n_samples and sample
// p mod n_samples, from those of the tile's first point (one 64-bit division) and a 32-bit division of the row's offset.  Returns the
// point's first bin edge (bins + ray * (n_samples + 1) + sample).
__device__ __forceinline__ const float* point_bin(const TcArgs& a, int tile, int row, long long& ray) {
  const long long p0 = (long long)tile * 128;
  const long long ray0 = p0 / a.n_samples;
  const int s = (int)(p0 - ray0 * a.n_samples) + (int)(min(p0 + row, a.n_points - 1) - p0);
  ray = ray0 + s / a.n_samples;
  return a.bins + ray * (a.n_samples + 1) + s % a.n_samples;
}

// sample position of point p = tile * 128 + row (the last point for a row past the end; ray r, sample s): o + d * t_start, then
// SceneContraction (cameras/rays.py:61-73, spatial_distortions.py:66-73).  Also returns the ray direction, the bin start and the bin
// width.
struct PointGeom { float px, py, pz, dx, dy, dz, delta, t0, t1; long long ray; };
__device__ __forceinline__ PointGeom point_geom(const TcArgs& a, int tile, int row) {
  const long long p = min((long long)tile * 128 + row, a.n_points - 1);
  PointGeom g;
  g.dx = g.dy = g.dz = 0.f; g.delta = 0.f; g.t0 = g.t1 = 0.f;
  g.ray = p;
  if (a.has_bins) {
    const float* bin = point_bin(a, tile, row, g.ray);
    const float t0 = __ldg(bin);
    g.t0 = t0;
    g.t1 = __ldg(bin + 1);
    g.delta = __fsub_rn(g.t1, t0);
    g.dx = __ldg(a.directions + g.ray * 3); g.dy = __ldg(a.directions + g.ray * 3 + 1); g.dz = __ldg(a.directions + g.ray * 3 + 2);
    g.px = __fadd_rn(__ldg(a.origins + g.ray * 3 + 0), __fmul_rn(g.dx, t0));
    g.py = __fadd_rn(__ldg(a.origins + g.ray * 3 + 1), __fmul_rn(g.dy, t0));
    g.pz = __fadd_rn(__ldg(a.origins + g.ray * 3 + 2), __fmul_rn(g.dz, t0));
  } else {
    g.px = __ldg(a.origins + p * 3); g.py = __ldg(a.origins + p * 3 + 1); g.pz = __ldg(a.origins + p * 3 + 2);
    if (a.directions) { g.dx = __ldg(a.directions + p * 3); g.dy = __ldg(a.directions + p * 3 + 1); g.dz = __ldg(a.directions + p * 3 + 2); }
  }
  // scene_contract's operations, written out: calling it moves the hoisted argument loads of the tcnn-layout instantiations and costs
  // them 16 more bytes of stack and 4 of spill (CUDA 12.9)
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

// accurate sin / sincos of the encoder warps.  Inlined: after setmaxnreg.dec a real call makes ptxas (CUDA 12.9) crash; both call
// sites are in the encoder loop, so this is two copies of the range reduction, not one per consumer epilogue
static __device__ __forceinline__ void sincos_call(float x, float* s, float* c) { sincosf(x, s, c); }
static __device__ __forceinline__ float sin_call(float x) { return sinf(x); }

// Staging slot s of the per-CTA scratch (tc_scratch)
template <int P>
struct Slot {
  uint8_t* base;
  __device__ __forceinline__ Slot(char* slots, uint32_t s) : base(reinterpret_cast<uint8_t*>(slots) + s * tc_scratch(P).slot_bytes) {}
  __device__ __forceinline__ uint8_t* geo() const { return base + tc_scratch(P).geo; }
  __device__ __forceinline__ uint8_t* cs() const { return base + tc_scratch(P).cs; }
  __device__ __forceinline__ float* jpe() const { return reinterpret_cast<float*>(base + tc_scratch(P).jpe); }
  __device__ __forceinline__ float* jg() const { return reinterpret_cast<float*>(base + tc_scratch(P).jg); }
  __device__ __forceinline__ float (*geom() const)[128] { return reinterpret_cast<float (*)[128]>(base + tc_scratch(P).geom); }
  __device__ __forceinline__ long long* ray() const { return reinterpret_cast<long long*>(base + tc_scratch(P).ray); }
};

// The point geometry of every row of a tile into its slot, rows et, et + 96 of encoder thread et: the staging items and EB0 read
// it from there instead of recomputing it (8 loads, and the contraction's divisions, per point and reader)
template <int P>
__device__ __forceinline__ void stage_geom(const TcArgs& a, int tile, int et, const Slot<P>& s) {
  float (*gm)[128] = s.geom();
#pragma unroll 1
  for (int row = et; row < 128; row += kEncThreads) {
    const PointGeom g = point_geom(a, tile, row);
    gm[GEOM_PX][row] = g.px; gm[GEOM_PY][row] = g.py; gm[GEOM_PZ][row] = g.pz;
    gm[GEOM_DX][row] = g.dx; gm[GEOM_DY][row] = g.dy; gm[GEOM_DZ][row] = g.dz;
    s.ray()[row] = g.ray;
  }
}

// Hash-grid part of the geo input of one tile, levels 4 grp .. 4 grp + 3 of one point (= operand chunk grp).  Outputs: bf16 planes
// of the staged geo input image (`img`, planes `plane` bytes apart, kernel column order: four levels = one aligned 16-byte chunk,
// written once per plane) and the grid jacobian Jg [(col*3 + d)][row] (with the 1/4 of (x+2)/4 folded in).  The item's 32 corner
// rows are first requested into L2 (no registers held), so that the level loop, one level at a time (smallest code, 8 gathers in
// flight), waits for L2 rather than for HBM on its four dependent gather round trips.
template <int P, int LAYOUT>
__device__ __forceinline__ void encode_tile_grid(const TcArgs& a, int row, int grp, const Slot<P>& s, uint64_t pol_table) {
  const float (*gm)[128] = s.geom();
  float* Jg = s.jg();
  const float x01 = (gm[GEOM_PX][row] + 2.0f) * 0.25f, y01 = (gm[GEOM_PY][row] + 2.0f) * 0.25f, z01 = (gm[GEOM_PZ][row] + 2.0f) * 0.25f;   // sdf_field.py:384
  const int l_end = min(4 * grp + 4, min(a.grid.n_levels, a.grid.active_levels));
  if (a.use_grid && a.mode != 0) {   // sdf-only calls (the samplers' passes) measured slower with it
#pragma unroll 1
    for (int l = 4 * grp; l < l_end; ++l) {
      LevelCtx c;
      level_prepare<LAYOUT>(a.grid, l, x01, y01, z01, c);
      if (a.grid.table_dtype == SDFB200_DT_F16) level_prefetch_l2<__half, 2>(a.table, c);
      else level_prefetch_l2<float, 2>(a.table, c);
    }
  }
  // the chunk's four (level) words per plane, shifted in level by level
  uint32_t h0 = 0u, h1 = 0u, h2 = 0u, h3 = 0u, l0 = 0u, l1 = 0u, l2 = 0u, l3 = 0u;
#pragma unroll 1
  for (int l = 4 * grp; l < 4 * grp + 4; ++l) {
    float o[2] = {0.f, 0.f};
    float dj[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    if (a.use_grid && l < l_end) {
      LevelCtx c;
      float tv[8][2];
      level_prepare<LAYOUT>(a.grid, l, x01, y01, z01, c);
      if (a.grid.table_dtype == SDFB200_DT_F16) level_fetch<__half, 2, true>(a.table, c, tv, pol_table);
      else level_fetch<float, 2, true>(a.table, c, tv, pol_table);
      level_finish<2, LAYOUT>(a.grid, c, tv, o, dj);
    }
    uint32_t hi, lo;
    split2(o[0], o[1], hi, lo);
    h0 = h1; h1 = h2; h2 = h3; h3 = hi;
    l0 = l1; l1 = l2; l2 = l3; l3 = lo;
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
  store_a_chunk<P>(s.geo(), kImgPlane, row, grp, make_uint4(h0, h1, h2, h3), make_uint4(l0, l1, l2, l3));
}

// PE | x | zero padding: chunks 4..11 of the geo input.  Kernel column 32 + i holds PE_i, 32 + pe_dim + j holds x_j.  Also the
// point outputs (contracted position and its norm) of a valid row, and the PE jacobian Jpe [i][row].
template <int P>
__device__ __forceinline__ void encode_tile_pe(const TcArgs& a, int tile, int row, const Slot<P>& s) {
  const long long p = (long long)tile * 128 + row;
  const float (*gm)[128] = s.geom();
  const float px = gm[GEOM_PX][row], py = gm[GEOM_PY][row], pz = gm[GEOM_PZ][row];
  if (p < a.n_points) {
    if (a.out.points_norm) a.out.points_norm[p] = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)), __fmul_rn(pz, pz)));
    if (a.out.points) { a.out.points[p * 3] = px; a.out.points[p * 3 + 1] = py; a.out.points[p * 3 + 2] = pz; }
  }
  const int deg = a.pe_degree, half = 3 * deg;
  uint8_t* img = s.geo();
  float* Jpe = s.jpe();
  // zero the chunks first (padding columns), then the live columns as 2-byte stores (same thread: program order).  Building whole
  // chunks in registers instead measured slower: every padding column then costs a pass of the column loop.
  const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
  for (int ch = 4; ch < kInK / 8; ++ch) store_a_chunk<P>(img, kImgPlane, row, ch, z4, z4);
#pragma unroll 1
  for (int i = 0; i < a.pe_dim; ++i) {                       // sin(x 2^k) | sin(x 2^k + pi/2)   (encodings.py:194-198)
    const int ia = i >= half ? i - half : i;
    const int b = ia / deg, k = ia - b * deg;
    const float fr = (float)(1 << k);
    const float xb = b == 0 ? px : (b == 1 ? py : pz);
    const float arg = i >= half ? xb * fr + kHalfPiF : xb * fr;
    float sv, cv;
    sincos_call(arg, &sv, &cv);
    store_a<P>(img, kImgPlane, row, 32 + i, a.use_pe ? sv : 0.f);
    // autograd of sin on the forward's own fp32 arguments: d/dx_b = 2^k cos(arg)
    if (a.mode != 0) Jpe[i * 128 + row] = a.use_pe ? fr * cv : 0.f;
  }
  store_a<P>(img, kImgPlane, row, 32 + a.pe_dim + 0, px);
  store_a<P>(img, kImgPlane, row, 32 + a.pe_dim + 1, py);
  store_a<P>(img, kImgPlane, row, 32 + a.pe_dim + 2, pz);
}

// direction-encoding value k (0..23) of direction (dx, dy, dz): sin(d_b 2^j) for k < 12, sin(d_b 2^j + pi/2) for k >= 12,
// b = (k mod 12) / 4, j = k mod 4 (NeRFEncoding(4), encodings.py:167-208).  d_b 2^j is exact, so a contracted d_b 2^j + pi/2 rounds
// the same.
__device__ __forceinline__ float dir_enc(float dx, float dy, float dz, int k) {
  const int i = k < 12 ? k : k - 12, b = i >> 2;
  const float db = b == 0 ? dx : (b == 1 ? dy : dz);
  const float arg = db * (float)(1 << (i & 3));
  return sin_call(k < 12 ? arg : arg + kHalfPiF);
}

// static colour-operand columns of a tile (kernel columns 8..95 = chunks 1..11): x(3) | dir-enc(24) | dir(3) | appearance | 0, staged in
// the same [plane][chunk][row][16 B] layout as the A operand; colour_copy bulk-copies them over the A columns that B0 has consumed
// (chunk 0 = [grad, n.v] comes from the epilogue).  Called by a whole warp for 32 consecutive rows (lane = row mod 32): when they are
// all samples of one ray, lane k < 24 evaluates direction-encoding value k once for the warp (the same sinf of the same argument).
template <int P>
__device__ __forceinline__ void colour_static_tile(const TcArgs& a, int row, const Slot<P>& s) {
  const float (*gm)[128] = s.geom();
  const float px = gm[GEOM_PX][row], py = gm[GEOM_PY][row], pz = gm[GEOM_PZ][row];
  const float dx = gm[GEOM_DX][row], dy = gm[GEOM_DY][row], dz = gm[GEOM_DZ][row];
  const long long ray = s.ray()[row];
  const bool one_ray = __match_any_sync(0xffffffffu, ray) == 0xffffffffu;
  const int lane = row & 31;
  const float own = one_ray && lane < 24 ? dir_enc(dx, dy, dz, lane) : 0.f;
  uint8_t* img = s.cs();
  const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
  for (int ch = 1; ch < kInK / 8; ++ch) store_a_chunk<P>(img, kImgPlane, row, ch, z4, z4);
  store_a<P>(img, kImgPlane, row, 8 + 0, px); store_a<P>(img, kImgPlane, row, 8 + 1, py); store_a<P>(img, kImgPlane, row, 8 + 2, pz);
  // direction encoding, then d itself (include_input)
#pragma unroll 1
  for (int k = 0; k < 24; ++k) {
    const float shared = __shfl_sync(0xffffffffu, own, k);
    store_a<P>(img, kImgPlane, row, 8 + 3 + k, one_ray ? shared : dir_enc(dx, dy, dz, k));
  }
  store_a<P>(img, kImgPlane, row, 8 + 27, dx); store_a<P>(img, kImgPlane, row, 8 + 28, dy); store_a<P>(img, kImgPlane, row, 8 + 29, dz);
  if (a.appearance != nullptr) {
#pragma unroll 1
    for (int j = 0; j < a.app_dim; ++j) store_a<P>(img, kImgPlane, row, 8 + 30 + j, __ldg(a.appearance + ray * a.app_dim + j));
  }
}

#ifdef SDFB200_TC_TIMING
// CTA 0, first 16 tiles, row = tile: clock64() of consumer thread 0 at [0] tile start, [1..7] end of the MMAs of layer 0..6 (ring
// order), [8] the tile's geo input has landed (a full; [8] - [0] is the consumers' wait for the encoder), [15] tile end = end of EC1
// (head inputs handed over), [18..23] end of the epilogues E0, E1, EB1, EB0, the late h2 copy issued, EC0 (before the SYNC_A that hands their A
// operand to the next layer's MMAs); cycle sums over the tile of [9] consumer thread 0 waiting for weights (ring full), [10] the producer
// waiting for a free ring slot (ring empty), [12] encoder thread 0 busy staging the tile, [13] encoder thread 0 waiting for its staging
// slot (enc empty), [14] encoder thread 0 running the tile's heads / compositing, [16] consumer thread 0 waiting for the tile's
// head-input buffer (hs empty), [17] encoder thread 0 waiting for the tile's head inputs (hs full), [24] [25] lane 0 of encoder
// warps 1, 2 busy staging the tile (warp 0: [12]), [26] [27] the same running the heads of the tile (warp 0: [14]), [28..30] encoder
// thread 0's heads split: per-row heads (geometry, sdf -> alpha / sigma, per-sample outputs), transmittance scan and weights, sums and
// the ray finish; [31] encoder thread 0 waiting at the encoder warps' barrier (kEncBar); [32 + 3 w + k] lane 0 of encoder warp w
// staging items of kind k (0 grid, 1 PE, 2 colour-static); [41 + w] lane 0 of encoder warp w staging the tile's point geometry,
// barrier included
__device__ long long g_tc_timing[16 * 48];   // only the timing build of ONE instantiation defines SDFB200_TC_TIMING
#define TC_PUT(tno, k, v)                                                                                            \
  do {                                                                                                               \
    if (blockIdx.x == 0 && (tno) >= 0 && (tno) < 16) g_tc_timing[(tno) * 48 + (k)] = (v);                            \
  } while (0)
#else
#define TC_PUT(tno, k, v) do { (void)(v); } while (0)
#endif
#define TC_STAMP(k) do { if (tid == 0) TC_PUT(tile_no, k, TC_CLOCK()); } while (0)

// Hand-offs between the roles (tc_common.cuh), used once per tile (n = the CTA's tile count) except the ring.  Arrival counts:
struct TcBars {
  Handoff<kStages> ring;  // weight ring, per K-block: full 1 + bytes, empty kEpiWarps
  Handoff<2> enc;         // staging slots: full kEncThreads (images written), empty kEpiThreads (after EB0; sdf-only: after a full)
  Handoff<1> a;           // A operand: full 1 + bytes (geo input landed), empty 2, one per consumer warpgroup (last layer has read A)
  Handoff<2> hs;          // head inputs: full kEpiThreads (after EC1), empty kEncThreads (the encoder warps are through the tile's heads);
                          // unused in sdf-only mode
  uint64_t cop[2][2];     // per consumer warpgroup, count 1 + bytes: [0] colour-static columns and h2 chunks 0..19 copied into A after
                          // B0, [1] h2 chunks 20..31 copied after C0-misc (colour_copy); unused in sdf-only mode
};

// Producer (one thread of the producer warpgroup).  Per tile: once the consumers have freed the A operand and the encoder has staged
// the tile, bulk-copies the staged geo input image into A columns 0..95; then walks every K-block of every layer in consumption order
// and issues the bulk copy of block j once its ring slot has been released (all 8 consumer warps are through block j - kStages).
// Every block of every layer is one full stage (tc_blocks_fill_stages).
template <int P>
__device__ __forceinline__ void produce_all(const TcArgs& a, int nlayers, uint8_t* abuf, uint8_t* ring, char* slots, TcBars& b) {
  uint32_t j = 0;
  int tile_no = 0;
  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x, ++tile_no) {
    long long waited = 0;
    b.a.wait_empty(tile_no);
    b.enc.wait_full(tile_no);
    const uint8_t* geo = Slot<P>(slots, b.enc.slot(tile_no)).geo();
    mbar_arrive_expect_tx(b.a.full_bar(tile_no), (uint32_t)P * kImgPlane);
#pragma unroll
    for (int pl = 0; pl < P; ++pl) bulk_g2s(abuf + pl * kAPlane, geo + pl * kImgPlane, kImgPlane, b.a.full_bar(tile_no));
    for (int L = 0; L < nlayers; ++L) {
      for (int kb = 0; kb < tc_layer_nkb(L); ++kb, ++j)
        ring_fill(b.ring, ring, j, reinterpret_cast<const uint8_t*>(a.blob) + a.layer[L].w_off, kb, tc_stage_bytes(P), &waited);
    }
    TC_PUT(tile_no, 10, waited);
  }
}

// All MMAs of layer L for the 64 rows of a warpgroup: acc (+)= A[rows, K] W^T with one m64nN wgmma per product and K step (N = 256, or
// 128 for B0: acc[0..1]), the weight K-blocks taken from the ring in order.  Every consumer warp releases a slot once its MMAs on it are
// complete (empty barrier count = 8 warps).  Each block is drained before the next is issued: with the producer in its own warpgroup and
// 5 stages, keeping one block in flight (wait_group 1) measured no faster.
// C0-h2 reads h2 where colour_copy put it: K step j (h2 chunks 2j, 2j + 1) from A chunks (2j + kInK / 8) mod 32, and waits for the late
// copy (`h2_late`, phase h2_parity) before the first K step it fills.  K order, weights and accumulation are those of any other layer.
constexpr int kH2Early = 32 - kInK / 8;   // h2 chunks 0 .. kH2Early - 1 land in A chunks kInK / 8 .. 31, the others in A chunks 0 .. kInK / 8 - 1
template <int P, int L>
__device__ __forceinline__ void layer_mma(float (&acc)[4][32], bool zero, uint32_t a_base, const uint8_t* ring, Handoff<kStages>& rb, uint32_t& it,
                                          int lane, long long& waited, uint64_t* h2_late, uint32_t h2_parity) {
  constexpr int N = tc_layer_np(L);
  constexpr int KSTEPS = tc_layer_kblk(L) / 16;              // K steps per ring stage
  constexpr uint32_t lbo_b = N * 16, plane_b = N * KSTEPS * 16 * 2;
  float (&d)[N / 2] = *reinterpret_cast<float (*)[N / 2]>(&acc[0][0]);
  if (zero) {
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  }
#pragma unroll 1
  for (int kb = 0; kb < tc_layer_nkb(L); ++kb, ++it) {
    if (L == L_C0H && kb * KSTEPS == kH2Early / 2) mbar_wait(h2_late, h2_parity);
    rb.wait_full(it, &waited);
    const uint32_t wbase = smem_u32(ring + (size_t)rb.slot(it) * tc_stage_bytes(P));
    wg_fence_acc(d);
    wg_arrive();
#pragma unroll
    for (int j = 0; j < KSTEPS; ++j) {
      const int kstep = kb * KSTEPS + j;
      const int ka = L == L_C0H ? (kstep + kInK / 16) % 16 : kstep;
      wgmma_kstep_wide_ss<P, N>(d, a_desc(a_base, ka), a_desc(a_base + kAPlane, ka), wbase + j * 2 * lbo_b, plane_b, lbo_b);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(d);
    __syncwarp();
    if (lane == 0) rb.arrive_empty(it);
  }
}

// What a consumer thread carries through the phases of a tile
struct TileCtx {
  const TcArgs& a;
  int tid, t, wg, wrow0;     // thread (0..255), thread in its warpgroup, warpgroup, first tile row of the warpgroup
  int r0, cq;                // accumulator rows r0, r0 + 8 of the tile and the column offset in every 8-column block
  uint8_t* abuf;             // shared memory (tc_smem): A operand
  const float (*prm)[256];   //   epilogue parameters (broadcast loads, not one LDG each)
  float (*hs)[128];          //   head inputs of the current tile
  const float4* coldesc;     //   EB0's column table
  float sdf_bias;
  uint32_t* sig_s;           // per-CTA scratch (tc_scratch): softplus'(z1)
  uint8_t* h2img;            //   h2 planes in the A operand's layout
  char* slots;               //   staging slots
  // this thread's 4-byte unit for the accumulator pair (c, i) in a [64 units][256 threads] scratch plane (sig_s)
  __device__ __forceinline__ int unit(int c, int i) const { return (c * 16 + (i >> 1)) * kEpiThreads + tid; }
};

// softplus'(z1) in [0, 1] as unorm16 without F2I / I2F: s * 65535 (rounded, then kept apart from the add so that it is not contracted
// into an FFMA) + 1.5 * 2^23 leaves round_to_nearest_even(s * 65535) in the low 16 bits, exactly what __float2uint_rn gives; the
// decode puts u back into the mantissa of 2^23 and subtracts 2^23 (exact)
__device__ __forceinline__ uint32_t unorm16x2_encode(float s0, float s1) {
  const float f0 = __fadd_rn(__fmul_rn(s0, 65535.0f), 12582912.0f), f1 = __fadd_rn(__fmul_rn(s1, 65535.0f), 12582912.0f);
  return __byte_perm(__float_as_uint(f0), __float_as_uint(f1), 0x5410);
}
__device__ __forceinline__ float unorm16_lo(uint32_t w) { return __fsub_rn(__uint_as_float(__byte_perm(w, 0x4B00u, 0x5410)), 8388608.0f) * (1.0f / 65535.0f); }
__device__ __forceinline__ float unorm16_hi(uint32_t w) { return __fsub_rn(__uint_as_float(__byte_perm(w, 0x4B00u, 0x5432)), 8388608.0f) * (1.0f / 65535.0f); }

// The epilogue parameters of the thread's columns in n64 block c, one float2 (columns cq, cq + 1) per 8-column block: element pairs
// i, i + 2 of the accumulator use v[i >> 2].  The epilogues load a block's parameters into registers before they store any of its
// results: `prm` and the A operand are both shared memory, so a parameter load placed after an A store cannot be moved above it, and
// loading per pair would make every pair wait for the one before (load -> softplus -> split -> store -> next load).
// The epilogues walk the four n64 blocks of the accumulator in a rolled loop: every pass works on acc[0], then moves blocks 1..3 down
// by one (96 register moves).  Unrolled, the seven epilogues were ~9 k instructions of straight-line code per tile that every consumer
// warp fetched once, next to the encoder warps' code; rolled, each is one block's worth, run four times.  The accumulator is consumed:
// the layer after an epilogue starts from zero.
__device__ __forceinline__ void acc_shift(float (&acc)[4][32]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[c][i] = acc[c + 1][i];
  }
}

template <int N>
__device__ __forceinline__ void load_prm_block(const float* prow, int cq, int c, int j0, float2 (&v)[N]) {
#pragma unroll
  for (int j = 0; j < N; ++j) v[j] = *reinterpret_cast<const float2*>(prow + frag_col(cq, c, 4 * (j0 + j)));
}

// E0 (after G0): h1 = softplus(z1) -> A ; softplus'(z1) -> scratch
template <int P>
__device__ __forceinline__ void epi_e0(const TileCtx& x, float (&acc)[4][32]) {
  const float* p_bg0 = x.prm[PRM_B_G0];
#pragma unroll 1
  for (int c = 0; c < 4; ++c, acc_shift(acc)) {
    float2 bias[8];
    load_prm_block(p_bg0, x.cq, c, 0, bias);
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const float2 b2 = bias[i >> 2];
      float h0, h1, s0, s1;
      softplus100_fast(acc[0][i] + b2.x, h0, s0);
      softplus100_fast(acc[0][i + 1] + b2.y, h1, s1);
      store_a_pair<P>(x.abuf, kAPlane, row, col, h0, h1);
      if (x.a.mode != 0) x.sig_s[x.unit(c, i)] = unorm16x2_encode(s0, s1);
    }
  }
}

// E1 (after G1): sdf = W2[0,:] . h2 + b (fp32) -> output / heads ; h2 -> scratch image (A layout, read back by colour_copy's bulk
// copies) ; g2 = W2[0,:] * softplus'(z2) -> A
template <int P>
__device__ __forceinline__ void epi_e1(const TileCtx& x, int tile, float (&acc)[4][32]) {
  const TcArgs& a = x.a;
  const float* p_bg1 = x.prm[PRM_B_G1];
  const float* p_wg2 = x.prm[PRM_W_G2];
  // one partial dot per accumulator row (r0, r0 + 8) as named scalars: an array indexed by the thread-dependent row below would live
  // in local memory, written back after every FMA because the generic stores in between may alias it
  float sp0 = 0.f, sp1 = 0.f;
#pragma unroll 1
  for (int c = 0; c < 4; ++c, acc_shift(acc)) {
    float2 bias[2], wrow[2];   // parameters of two 8-column blocks (4 pairs) at a time: whole n64 blocks spill at P = 1
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      if (i % 8 == 0) { load_prm_block(p_bg1, x.cq, c, i >> 2, bias); load_prm_block(p_wg2, x.cq, c, i >> 2, wrow); }
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const float2 b2 = bias[(i >> 2) & 1];
      const float2 w2 = wrow[(i >> 2) & 1];
      float h0, h1, s0, s1;
      softplus100_fast(acc[0][i] + b2.x, h0, s0);
      softplus100_fast(acc[0][i + 1] + b2.y, h1, s1);
      float& sp = frag_half(i) ? sp1 : sp0;
      sp = fmaf(w2.x, h0, sp);
      sp = fmaf(w2.y, h1, sp);
      if (a.mode != 0) {
        store_a_pair<P>(x.h2img, kAPlane, row, col, h0, h1);
        store_a_pair<P>(x.abuf, kAPlane, row, col, w2.x * s0, w2.y * s1);
      }
    }
  }
  // hand-off: h2 (generic stores, global) -> colour_copy's bulk copies (async proxy), behind the warpgroup barriers up to B0
  if (a.mode != 0) fence_async_global();
  sp0 = quad_sum(sp0);
  sp1 = quad_sum(sp1);
  if ((x.t & 3) < 2) {
    const int h = x.t & 1, row = x.r0 + 8 * h;
    const float sdf = (h ? sp1 : sp0) + x.sdf_bias;
    const long long p = (long long)tile * 128 + row;
    if (p < a.n_points && a.out.sdf) a.out.sdf[p] = sdf;
    if (a.mode != 0) x.hs[HS_SDF][row] = sdf;
  }
}

// EB1 (after B1): g1 = (W1^T g2) * softplus'(z1) -> A.  The 16 softplus' words of n64 block c + 1 are loaded (from L2) while block c is
// multiplied and stored, so their latency is paid once per tile rather than once per word.
template <int P>
__device__ __forceinline__ void epi_eb1(const TileCtx& x, float (&acc)[4][32]) {
  uint32_t sw[16], sw_next[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) sw[k] = x.sig_s[x.unit(0, 2 * k)];
#pragma unroll 1
  for (int c = 0; c < 4; ++c, acc_shift(acc)) {
    if (c < 3) {
#pragma unroll
      for (int k = 0; k < 16; ++k) sw_next[k] = x.sig_s[x.unit(c + 1, 2 * k)];
    }
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const uint32_t w = sw[i >> 1];
      store_a_pair<P>(x.abuf, kAPlane, row, col, acc[0][i] * unorm16_lo(w), acc[0][i + 1] * unorm16_hi(w));
    }
    if (c < 3) {
#pragma unroll
      for (int k = 0; k < 16; ++k) sw[k] = sw_next[k];
    }
  }
}

// EB0's view of geo input column 32 + ip (ColDesc): float4 {row of the PE jacobian (int bits; -1: none, factor 1), then the weights of
// the column on the x, y, z gradient}: PE column ip -> axis (ip mod 3 deg) / deg with factor 2^k cos(arg) from the jacobian, x column
// -> its own axis with factor 1, padding -> all weights 0
__device__ __forceinline__ float4 col_desc(const TcArgs& a, int ip) {
  const int deg = a.pe_degree, half = 3 * deg;
  int jrow = -1, ax = -1;
  if (ip < a.pe_dim) {
    const int ia = ip >= half ? ip - half : ip;
    ax = ia < deg ? 0 : (ia < 2 * deg ? 1 : 2);
    jrow = ip * 128;
  } else if (ip - a.pe_dim < 3) {
    ax = ip - a.pe_dim;
  }
  return make_float4(__int_as_float(jrow), ax == 0 ? 1.f : 0.f, ax == 1 ? 1.f : 0.f, ax == 2 ? 1.f : 0.f);
}

// Bulk copies of the colour MLP's A operand, issued by warp 0 of the warpgroup (lane 0 arms the barrier, every lane issues some of the
// 1 KB copies: one plane of one chunk of the warpgroup's 64 rows).  Early (after B0, `cop[wg][0]`): the colour-static columns
// (chunks 1..11 of the staging slot) into A chunks 1..11, h2 chunks 0..kH2Early - 1 into A chunks kInK / 8 .. 31.  Late (after C0-misc,
// `cop[wg][1]`): the other h2 chunks into A chunks 0..kInK / 8 - 1.  A chunks are free once the layer before has read them (its MMAs are
// complete and the warpgroup barrier is passed); earlier generic stores to them were fenced (SYNC_A).
template <int P>
__device__ __forceinline__ void copy_chunks(uint8_t* abuf, int a_chunk, const uint8_t* src, uint32_t src_plane, int src_chunk, int n, int wrow0,
                                            uint64_t* bar, int lane) {
  for (int k0 = 0; k0 < P * n; k0 += 32) {   // a warp-uniform trip count: the warp is converged again after the loop
    const int k = k0 + lane;
    if (k < P * n) {
      const int pl = k / n, c = k - pl * n;
      bulk_g2s(abuf + pl * kAPlane + (a_chunk + c) * kAChunk + wrow0 * 16, src + pl * src_plane + (src_chunk + c) * kAChunk + wrow0 * 16, 64 * 16, bar);
    }
  }
}
template <int P>
__device__ __forceinline__ void colour_copy(const TileCtx& x, bool early, const uint8_t* cs, uint64_t* bar) {
  constexpr int kMisc = kInK / 8;
  const int lane = x.t & 31;
  if (lane == 0) mbar_arrive_expect_tx(bar, (uint32_t)P * (early ? (kMisc - 1) + kH2Early : 32 - kH2Early) * 64 * 16);
  __syncwarp();
  if (early) {
    copy_chunks<P>(x.abuf, 1, cs, kImgPlane, 1, kMisc - 1, x.wrow0, bar, lane);
    copy_chunks<P>(x.abuf, kMisc, x.h2img, kAPlane, 0, kH2Early, x.wrow0, bar, lane);
  } else {
    copy_chunks<P>(x.abuf, 0, x.h2img, kAPlane, kH2Early, 32 - kH2Early, x.wrow0, bar, lane);
  }
}

// EB0 (after B0): gin (96 cols, kernel order) . input jacobian -> d sdf / dx -> chunk 0 of the colour misc operand over the (consumed)
// A columns: [grad(3), n.v, 0 x4] (sdf_field.py:572-584; columns re-ordered at pack time) from the thread pair that owns the row.  The
// other chunks ([x, dir-enc, dir, appearance], h2) arrive by colour_copy.
template <int P>
__device__ __forceinline__ void epi_eb0(const TileCtx& x, const Slot<P>& s, const float (&acc)[4][32]) {
  const TcArgs& a = x.a;
  const float* Jpe = s.jpe();
  const float* Jg = s.jg();
  // d sdf / dx of rows r0 (g*0) and r0 + 8 (g*1), named scalars (see epi_e1).  Every column is accumulated the same way whatever its
  // kind, the kind coming from the column table (ColDesc): a zero factor adds +-0, which leaves the sum as it is, so the result is
  // the one of accumulating the live columns alone
  float g0x = 0.f, g0y = 0.f, g0z = 0.f, g1x = 0.f, g1y = 0.f, g1z = 0.f;
#pragma unroll
  for (int c = 0; c < 2; ++c) {
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const bool h = frag_half(i);
      float& gx = h ? g1x : g0x;
      float& gy = h ? g1y : g0y;
      float& gz = h ? g1z : g0z;
      const float g = acc[c][i];
      if (c == 0 && i < 16) {                  // grid columns 0..31 (c, i are compile-time): g * grid jacobian row, or 0 past grid_dim
        const bool live = col < a.grid_dim;
        const float* j = Jg + col * 3 * 128 + row;
        const float jx = live ? j[0] : 0.f, jy = live ? j[128] : 0.f, jz = live ? j[256] : 0.f;
        gx = fmaf(g, jx, gx); gy = fmaf(g, jy, gy); gz = fmaf(g, jz, gz);
      } else {                                 // PE | x | padding: (g * factor) onto the column's axis
        const float4 d = x.coldesc[col - 32];
        const int jrow = __float_as_int(d.x);
        const float tv = __fmul_rn(g, jrow >= 0 ? Jpe[jrow + row] : 1.f);
        gx = fmaf(tv, d.y, gx); gy = fmaf(tv, d.z, gy); gz = fmaf(tv, d.w, gz);
      }
    }
  }
  g0x = quad_sum(g0x); g0y = quad_sum(g0y); g0z = quad_sum(g0z);
  g1x = quad_sum(g1x); g1y = quad_sum(g1y); g1z = quad_sum(g1z);
  if ((x.t & 3) < 2) {
    const int h = x.t & 1, row = x.r0 + 8 * h;
    const float (*gm)[128] = s.geom();
    const float grx = h ? g1x : g0x, gry = h ? g1y : g0y, grz = h ? g1z : g0z;
    const float3 n = normalize_eps(grx, gry, grz);
    const float c0v[8] = {grx, gry, grz, a.use_n_dot_v ? n.x * gm[GEOM_DX][row] + n.y * gm[GEOM_DY][row] + n.z * gm[GEOM_DZ][row] : 0.f,
                          0.f, 0.f, 0.f, 0.f};
    store_a_chunk<P>(x.abuf, kAPlane, row, 0, c0v);
    x.hs[HS_GRAD][row] = grx; x.hs[HS_GRAD + 1][row] = gry; x.hs[HS_GRAD + 2][row] = grz;
  }
}

// EC0 (after C0): relu -> A
template <int P>
__device__ __forceinline__ void epi_ec0(const TileCtx& x, float (&acc)[4][32]) {
  const float* p_bc0 = x.prm[PRM_B_C0];
#pragma unroll 1
  for (int c = 0; c < 4; ++c, acc_shift(acc)) {
    float2 bias[8];
    load_prm_block(p_bc0, x.cq, c, 0, bias);
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const float2 b2 = bias[i >> 2];
      store_a_pair<P>(x.abuf, kAPlane, row, col, fmaxf(acc[0][i] + b2.x, 0.f), fmaxf(acc[0][i + 1] + b2.y, 0.f));
    }
  }
}

// EC1 (after C1): relu, last colour layer (256 -> 3) as fp32 dots -> heads
__device__ __forceinline__ void epi_ec1(const TileCtx& x, float (&acc)[4][32]) {
  const float* p_bc1 = x.prm[PRM_B_C1];
  const float (*p_wc2)[256] = x.prm + PRM_W_C2;
  float r0r = 0.f, r0g = 0.f, r0b = 0.f, r1r = 0.f, r1g = 0.f, r1b = 0.f;   // rows r0, r0 + 8 (named scalars, see epi_e1)
#pragma unroll 1
  for (int c = 0; c < 4; ++c, acc_shift(acc)) {
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = frag_col(x.cq, c, i);
      const bool h = frag_half(i);
      float& rr = h ? r1r : r0r;
      float& rg = h ? r1g : r0g;
      float& rb = h ? r1b : r0b;
      const float v = fmaxf(acc[0][i] + p_bc1[col], 0.f);
      rr = fmaf(p_wc2[0][col], v, rr);
      rg = fmaf(p_wc2[1][col], v, rg);
      rb = fmaf(p_wc2[2][col], v, rb);
    }
  }
  r0r = quad_sum(r0r); r0g = quad_sum(r0g); r0b = quad_sum(r0b);
  r1r = quad_sum(r1r); r1g = quad_sum(r1g); r1b = quad_sum(r1b);
  if ((x.t & 3) < 2) {
    const int h = x.t & 1, row = x.r0 + 8 * h;
    x.hs[HS_RGB][row] = h ? r1r : r0r; x.hs[HS_RGB + 1][row] = h ? r1g : r0g; x.hs[HS_RGB + 2][row] = h ? r1b : r0b;
  }
}

// Per-point heads and, in fused mode, the per-ray compositing of a tile, spread over the three encoder warps.  They read the head
// inputs `hs` that the consumers left (sdf, gradient, raw rgb; the geometry is recomputed).  Encoder warp ew takes the 32-row chunks
// q = ew, ew + 3 of the tile (warp 0 two of the four), lane = row in the chunk.  A ray of S <= 32 samples lies in one chunk and is
// finished there (heads_rows).  A longer one spans S / 32 chunks, in general of different warps, and takes three phases with a barrier
// of the 96 encoder threads (kEncBar) between them:
//   1 (heads_rows)       per-row heads, the chunk's segmented factor scan and its total wtot[q]; the row's exclusive scan goes to `hx`,
//                        its alpha, normal and colour over its (already read) head inputs (HeadsRow)
//   2 (composite_chunk)  excl x= wtot[first .. q - 1] in chunk order, T, w, the weights, and the chunk's eight sums to csum[q]
//   3 (finish_rays)      the warp with the ray's last chunk adds the ray's chunk sums in chunk order, from 0, and finishes the ray
// Every value sees the operations of one warp walking the chunks in order, so nothing depends on which warp runs which chunk.
// wtot and csum are by tile parity: a warp may start phase 1 of the next tile while another still reads this tile's in phase 3.
struct HeadsXfer { double wtot[2][4]; float csum[2][4][8]; };
static_assert(sizeof(TcBars) + sizeof(HeadsXfer) <= kStaticSmem, "static shared memory of k_field_tc (kStaticSmem)");
// the rows of `hs` that phase 1 leaves for phase 2 of a ray longer than 32 samples, over the head inputs of the same row
enum { HR_ALPHA = HS_SDF /* alpha, or 1 - exp(-delta sigma) */, HR_NORMAL = HS_GRAD /* x, y, z */, HR_RGB = HS_RGB /* padded rgb */ };
// the end of a ray that a warp's phase 2 found in its chunks (at most one per warp: a ray spans >= 2 of the 4 chunks)
struct RayEnd { int q; double tot; float last[3]; };
// encoder thread 0's cycles in the three kinds of heads work (timing build)
struct HeadsClock { long long rows, scan, sums; };

// (starts + ends) / 2 of point tile * 128 + row (renderers.py:247), with the bin edges of point_geom
__device__ __forceinline__ float sample_mid(const TcArgs& a, int tile, int row) {
  if (!a.has_bins) return 0.f;
  long long ray;
  const float* b = point_bin(a, tile, row, ray);
  return __fdiv_rn(__fadd_rn(__ldg(b), __ldg(b + 1)), 2.0f);
}

// Phase 1 of chunk q (all of it for rays of S <= 32 samples and in unfused mode).  dmin / dmax: the thread's running depth range.
__device__ __forceinline__ void heads_rows(const TcArgs& a, float (*hs)[128], double* hx, double* wtot, int tile, int q, int lane,
                                           float& dmin, float& dmax, HeadsClock& clk) {
  long long tc0 = TC_CLOCK();
  const float* b_c2 = reinterpret_cast<const float*>(a.blob + a.b_c2);
  const int row = q * 32 + lane;
  const long long p_raw = (long long)tile * 128 + row;
  const bool valid = p_raw < a.n_points;
  const long long p = valid ? p_raw : a.n_points - 1;
  const PointGeom pg = point_geom(a, tile, row);
  const float dirx = pg.dx, diry = pg.dy, dirz = pg.dz, delta = pg.delta;
  const float sdf = hs[HS_SDF][row], grx = hs[HS_GRAD][row], gry = hs[HS_GRAD + 1][row], grz = hs[HS_GRAD + 2][row];
  const float3 nv = normalize_eps(grx, gry, grz);
  const float nx = nv.x, ny = nv.y, nz = nv.z;
  float rgbv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) rgbv[c] = padded_rgb(sigmoidf_(hs[HS_RGB + c][row] + __ldg(b_c2 + c)), a.rgb_padding);
  float density = 0.f, alpha = 0.f;
  if (a.out.density || (a.render && a.rnd.from_density)) density = sdf_density(sdf, __ldg(a.beta), __ldg(a.beta_min));
  if (a.out.alpha || (a.render && !a.rnd.from_density))
    alpha = neus_alpha(sdf, dirx * grx + diry * gry + dirz * grz, delta, __ldg(a.variance), a.cos_anneal);
  if (valid) {
    if (a.out.rgb) { a.out.rgb[p * 3] = rgbv[0]; a.out.rgb[p * 3 + 1] = rgbv[1]; a.out.rgb[p * 3 + 2] = rgbv[2]; }
    if (a.out.gradients) { a.out.gradients[p * 3] = grx; a.out.gradients[p * 3 + 1] = gry; a.out.gradients[p * 3 + 2] = grz; }
    if (a.out.normals) { a.out.normals[p * 3] = nx; a.out.normals[p * 3 + 1] = ny; a.out.normals[p * 3 + 2] = nz; }
    if (a.out.density) a.out.density[p] = density;
    if (a.out.occupancy) a.out.occupancy[p] = occupancy(sdf);
    if (a.out.alpha) a.out.alpha[p] = alpha;
  }
  { const long long c = TC_CLOCK(); clk.rows += c - tc0; tc0 = c; }
  if (!a.render) return;
  // ---------------- fused compositing: the tile holds 128 / S whole rays; row -> (ray, sample) = (row / S, row % S) ----------------
  const int S = a.n_samples;
  const int s_idx = row % S;
  const bool dens = a.rnd.from_density != 0;
  // factor by which the transmittance drops across this sample: 1 - alpha + 1e-7 (rays.py:204-206), or as an exponent
  // delta * sigma for the density form (rays.py:160-170)
  const float dd = valid ? __fmul_rn(delta, density) : 0.f;
  double f = dens ? (double)dd : (valid ? (double)neus_trans_factor(alpha) : 1.0);
  double incl = f;
  // segmented by ray (s_idx >= d), so not the plain warp_scan_incl of common.cuh
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const double o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d && s_idx >= d) incl = dens ? incl + o : incl * o;
  }
  double excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0 || s_idx == 0) excl = dens ? 0.0 : 1.0;
  const float al = dens ? __fsub_rn(1.0f, expf(-dd)) : alpha;
  const float mid = __fdiv_rn(__fadd_rn(pg.t0, pg.t1), 2.0f);            // (starts + ends) / 2, renderers.py:247
  if (valid) { dmin = fminf(dmin, mid); dmax = fmaxf(dmax, mid); }      // the batch's steps.min() / max() (renderers.py:257)
  if (S > 32) {                                                         // the ray spans chunks: phases 2 and 3 take it from here
    if (lane == 31) wtot[q] = incl;
    hx[row] = excl;
    hs[HR_ALPHA][row] = al;
    hs[HR_NORMAL][row] = nx; hs[HR_NORMAL + 1][row] = ny; hs[HR_NORMAL + 2][row] = nz;
    hs[HR_RGB][row] = rgbv[0]; hs[HR_RGB + 1][row] = rgbv[1]; hs[HR_RGB + 2][row] = rgbv[2];
    clk.scan += TC_CLOCK() - tc0;
    return;
  }
  const float T = dens ? expf(-(float)excl) : (float)excl;
  const float w = valid ? __fmul_rn(al, T) : 0.f;
  if (valid && a.rnd.weights) a.rnd.weights[p] = w;
  { const long long c = TC_CLOCK(); clk.scan += c - tc0; tc0 = c; }
  float vs[8] = {w, w * rgbv[0], w * rgbv[1], w * rgbv[2], w * nx, w * ny, w * nz, w * mid};
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    if (d < S) {
#pragma unroll
      for (int k = 0; k < 8; ++k) vs[k] += __shfl_down_sync(0xffffffffu, vs[k], d);
    }
  }
  // transmittance after the last sample (alphas: transmittance[:, -1] = bg_transmittance, neus.py:101) / before it (densities:
  // volsdf.py:67-68), and the colour of the last sample
  const int last = (lane - s_idx) + S - 1;
  const double tot = __shfl_sync(0xffffffffu, dens ? excl : incl, last);
  const float lc[3] = {__shfl_sync(0xffffffffu, rgbv[0], last), __shfl_sync(0xffffffffu, rgbv[1], last), __shfl_sync(0xffffffffu, rgbv[2], last)};
  const long long ray = (long long)tile * (128 / S) + row / S;
  if (s_idx == 0 && ray * S < a.n_points) {
    finish_ray(ray, vs[0], {vs[1], vs[2], vs[3]}, {vs[4], vs[5], vs[6]}, vs[7], a.rnd.bg_mode, a.rnd.bg, lc, a.rnd.clamp01, a.rnd.out.rgb,
               a.rnd.out.accumulation, a.rnd.out.normal, a.rnd.out.depth);
    if (a.rnd.bg_transmittance) a.rnd.bg_transmittance[ray] = dens ? expf(-(float)tot) : (float)tot;
  }
  clk.sums += TC_CLOCK() - tc0;
}

// Phase 2 of chunk q of a ray longer than 32 samples: the scan totals of the ray's earlier chunks, the weights and the chunk's sums
__device__ __forceinline__ void composite_chunk(const TcArgs& a, const float (*hs)[128], const double* hx, const double* wtot, float (*csum)[8],
                                                int tile, int q, int lane, RayEnd& end, HeadsClock& clk) {
  long long tc0 = TC_CLOCK();
  const int row = q * 32 + lane;
  const long long p_raw = (long long)tile * 128 + row;
  const bool valid = p_raw < a.n_points;
  const long long p = valid ? p_raw : a.n_points - 1;
  const int S = a.n_samples;
  const bool dens = a.rnd.from_density != 0;
  const int first = (q * 32 / S) * (S / 32);                            // first chunk of the ray
  double excl = hx[row];
  for (int w2 = first; w2 < q; ++w2) excl = dens ? excl + wtot[w2] : excl * wtot[w2];
  const float T = dens ? expf(-(float)excl) : (float)excl;
  const float w = valid ? __fmul_rn(hs[HR_ALPHA][row], T) : 0.f;
  if (valid && a.rnd.weights) a.rnd.weights[p] = w;
  { const long long c = TC_CLOCK(); clk.scan += c - tc0; tc0 = c; }
  const float rgbv[3] = {hs[HR_RGB][row], hs[HR_RGB + 1][row], hs[HR_RGB + 2][row]};
  float vs[8] = {w, w * rgbv[0], w * rgbv[1], w * rgbv[2], w * hs[HR_NORMAL][row], w * hs[HR_NORMAL + 1][row], w * hs[HR_NORMAL + 2][row],
                 w * sample_mid(a, tile, row)};
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
#pragma unroll
    for (int k = 0; k < 8; ++k) vs[k] += __shfl_down_sync(0xffffffffu, vs[k], d);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 8; ++k) csum[q][k] = vs[k];
  }
  if (q == first + S / 32 - 1) {                                        // the chunk ends the ray
    end.q = q;
    if (dens) {
      end.tot = __shfl_sync(0xffffffffu, excl, 31);
    } else {
      end.tot = 1.0;
      for (int w2 = first; w2 <= q; ++w2) end.tot *= wtot[w2];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) end.last[c] = __shfl_sync(0xffffffffu, rgbv[c], 31);
  }
  clk.sums += TC_CLOCK() - tc0;
}

// Phase 3: the ray that ends in this warp's chunks, from its chunk sums added in chunk order
__device__ __forceinline__ void finish_rays(const TcArgs& a, const float (*csum)[8], int tile, int lane, const RayEnd& end, HeadsClock& clk) {
  const long long tc0 = TC_CLOCK();
  const int S = a.n_samples;
  const long long ray = (long long)tile * (128 / S) + end.q * 32 / S;
  if (end.q >= 0 && lane == 0 && ray * S < a.n_points) {
    float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int w2 = end.q + 1 - S / 32; w2 <= end.q; ++w2) {
#pragma unroll
      for (int k = 0; k < 8; ++k) s[k] += csum[w2][k];
    }
    finish_ray(ray, s[0], {s[1], s[2], s[3]}, {s[4], s[5], s[6]}, s[7], a.rnd.bg_mode, a.rnd.bg, end.last, a.rnd.clamp01, a.rnd.out.rgb,
               a.rnd.out.accumulation, a.rnd.out.normal, a.rnd.out.depth);
    const bool dens = a.rnd.from_density != 0;
    if (a.rnd.bg_transmittance) a.rnd.bg_transmittance[ray] = dens ? expf(-(float)end.tot) : (float)end.tot;
  }
  clk.sums += TC_CLOCK() - tc0;
}

// An encoder warp's part of the heads of a tile: wait for the head inputs, run the warp's chunks, hand the buffer back
__device__ __forceinline__ void heads_of(const TcArgs& a, int tile, int tile_no, int ew, int lane, TcBars& b, float (*hs)[128], double* hx,
                                         HeadsXfer& xf, float& dmin, float& dmax) {
  long long waited = 0, bar_waited = 0;
  b.hs.wait_full(tile_no, &waited);
  const long long t0 = TC_CLOCK();
  float (*h)[128] = hs + b.hs.slot(tile_no) * kHsRows;
  double* wtot = xf.wtot[tile_no & 1];
  float (*csum)[8] = xf.csum[tile_no & 1];
  HeadsClock clk{0, 0, 0};
#pragma unroll 1
  for (int q = ew; q < 4; q += kEncThreads / 32) heads_rows(a, h, hx, wtot, tile, q, lane, dmin, dmax, clk);
  if (a.render && a.n_samples > 32) {
    long long c = TC_CLOCK();
    named_sync(kEncBar, kEncThreads);                 // every chunk's wtot is written
    bar_waited += TC_CLOCK() - c;
    RayEnd end{-1, 0.0, {0.f, 0.f, 0.f}};
#pragma unroll 1
    for (int q = ew; q < 4; q += kEncThreads / 32) composite_chunk(a, h, hx, wtot, csum, tile, q, lane, end, clk);
    c = TC_CLOCK();
    named_sync(kEncBar, kEncThreads);                 // every chunk's sums are written
    bar_waited += TC_CLOCK() - c;
    finish_rays(a, csum, tile, lane, end, clk);
  }
  b.hs.arrive_empty(tile_no);
  if (lane == 0) TC_PUT(tile_no, ew == 0 ? 14 : 25 + ew, TC_CLOCK() - t0);
  if (ew == 0 && lane == 0) { TC_PUT(tile_no, 17, waited); TC_PUT(tile_no, 28, clk.rows); TC_PUT(tile_no, 29, clk.scan); TC_PUT(tile_no, 30, clk.sums); TC_PUT(tile_no, 31, bar_waited); }
}

// Encoder warps (ew = 0..2, et = 32 ew + lane): walk the same tiles as the consumers and stage each one in its slot while the consumers
// run the tile before it.  A tile's staging starts with its point geometry (stage_geom, then the encoder warps' barrier), then 768
// items: 512 (point, group of four hash levels), then 128 x (PE | x, point outputs) and, with the colour MLP, 128 x colour-static
// columns.  Encoder warp ew takes items enc_item_begin(ew) .. enc_item_begin(ew + 1) - 1, lane = item mod 32: warp 0, which runs two
// of the four chunks of the heads, takes fewer (field_tc.h).  In sdf-only mode (640 items, no heads) item i goes to thread i % 96.
// Either way a warp walks whole 32-item batches, 32-aligned, so the kind of item is the same across the warp and ptxas, given the
// warp index as warp-uniform (k_field_tc), sees the shuffles of the colour-static items and of the heads as converged.  Except in sdf-only mode, the encoder warps then run the heads of the tile before (the one the consumers are
// finishing), and those of the last tile after the loop.  Staging tile n + 1 and the heads of tile n - 1 both fit in the consumers'
// tile n: slot n + 1 was freed at EB0 of tile n - 1, and the head inputs of tile n - 1 are ready when tile n starts.
template <int P, int LAYOUT>
__device__ __forceinline__ void encode_all(const TcArgs& a, int ew, int lane, char* slots, TcBars& b, uint64_t pol_table, float (*hs)[128],
                                           double* hx, HeadsXfer& xf) {
  const bool heads = a.mode != 0;
  const int et = ew * 32 + lane;
  const int i_begin = heads ? enc_item_begin(ew) : ew * 32, i_end = heads ? enc_item_begin(ew + 1) : 640, i_step = heads ? 32 : kEncThreads;
  float dmin = INFINITY, dmax = -INFINITY;       // the midpoints of this thread's rows, over every tile of the CTA
  int tile_no = 0;
  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x, ++tile_no) {
    long long waited = 0;
    b.enc.wait_empty(tile_no, &waited);
    const long long t0 = TC_CLOCK();
    const Slot<P> s(slots, b.enc.slot(tile_no));
    long long kind_grid = 0, kind_pe = 0, kind_cs = 0, geom = 0;   // staging cycles by item kind (timing build)
    stage_geom<P>(a, tile, et, s);
    named_sync(kEncBar, kEncThreads);        // every row's geometry is in the slot
    geom = TC_CLOCK() - t0;
#pragma unroll 1
    for (int ib = i_begin; ib < i_end; ib += i_step) {   // the warp's batch of items ib .. ib + 31
      const int row = (ib & 127) + lane;
      const long long c0 = TC_CLOCK();
      if (ib < 512) { encode_tile_grid<P, LAYOUT>(a, row, ib >> 7, s, pol_table); kind_grid += TC_CLOCK() - c0; }
      else if (ib < 640) { encode_tile_pe<P>(a, tile, row, s); kind_pe += TC_CLOCK() - c0; }
      else { colour_static_tile<P>(a, row, s); kind_cs += TC_CLOCK() - c0; }
    }
    fence_async_global();                    // the geo image is read by the producer's bulk copy (async proxy)
    b.enc.arrive_full(tile_no);
    if (et == 0) { TC_PUT(tile_no, 12, TC_CLOCK() - t0); TC_PUT(tile_no, 13, waited); }
    else if (lane == 0) TC_PUT(tile_no, 23 + ew, TC_CLOCK() - t0);
    if (lane == 0) {
      TC_PUT(tile_no, 32 + 3 * ew, kind_grid); TC_PUT(tile_no, 33 + 3 * ew, kind_pe); TC_PUT(tile_no, 34 + 3 * ew, kind_cs);
      TC_PUT(tile_no, 41 + ew, geom);
    }
    if (heads && tile_no > 0) heads_of(a, tile - (int)gridDim.x, tile_no - 1, ew, lane, b, hs, hx, xf, dmin, dmax);
  }
  if (heads && tile_no > 0) heads_of(a, blockIdx.x + (tile_no - 1) * (int)gridDim.x, tile_no - 1, ew, lane, b, hs, hx, xf, dmin, dmax);   // the last tile
  // one depth-range update per warp and CTA: min and max are exact, so the result is that of any order of updates
  if (heads && a.render && a.rnd.out.steps_minmax) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      dmin = fminf(dmin, __shfl_xor_sync(0xffffffffu, dmin, d));
      dmax = fmaxf(dmax, __shfl_xor_sync(0xffffffffu, dmax, d));
    }
    if (lane == 0 && dmin <= dmax) { atomic_min_float(a.rnd.out.steps_minmax, dmin); atomic_max_float(a.rnd.out.steps_minmax + 1, dmax); }
  }
}

template <int P, int LAYOUT>
__global__ void __launch_bounds__(kTcThreads, 1) k_field_tc(const __grid_constant__ TcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr TcSmem sm = tc_smem(P);
  constexpr TcScratch scr = tc_scratch(P);
  uint8_t* abuf = smem + sm.a;
  uint8_t* ring = smem + sm.ring;
  float (*prm)[256] = reinterpret_cast<float (*)[256]>(smem + sm.prm);
  float (*hs)[128] = reinterpret_cast<float (*)[128]>(smem + sm.hs);
  float4* coldesc = reinterpret_cast<float4*>(smem + sm.coldesc);
  double* hx = reinterpret_cast<double*>(smem + sm.hx);
  __shared__ TcBars bars;
  __shared__ HeadsXfer hxf;

  // the warp index as the canonical warp-uniform value (a shuffle from lane 0): the role dispatch below branches on it, so that ptxas
  // sees every role's shuffles as converged rather than wrapping each in a WARPSYNC.COLLECTIVE loop
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int nlayers = a.mode == 0 ? 2 : L_COUNT;
  char* cta_scr = a.scratch + (size_t)blockIdx.x * scr.bytes;
  char* slots = cta_scr + scr.slots;
  if (tid == 0) {
    bars.ring.init(1, kEpiWarps);
    bars.enc.init(kEncThreads, kEpiThreads);
    bars.hs.init(kEpiThreads, kEncThreads);
    bars.a.init(1, 2);
    for (int w = 0; w < 2; ++w) { mbar_init(&bars.cop[w][0], 1); mbar_init(&bars.cop[w][1], 1); }
    fence_barrier_init();
  }
  {
    const char* blob = a.blob;
    const float* src[kPrmRows] = {reinterpret_cast<const float*>(blob + a.b_g0), reinterpret_cast<const float*>(blob + a.b_g1),
                                  reinterpret_cast<const float*>(blob + a.w_g2), reinterpret_cast<const float*>(blob + a.b_c0),
                                  reinterpret_cast<const float*>(blob + a.b_c1), reinterpret_cast<const float*>(blob + a.w_c2),
                                  reinterpret_cast<const float*>(blob + a.w_c2) + 256, reinterpret_cast<const float*>(blob + a.w_c2) + 512};
    for (int i = tid; i < kPrmRows * 256; i += kTcThreads) prm[i >> 8][i & 255] = src[i >> 8][i & 255];
    if (tid < 96) coldesc[tid] = col_desc(a, tid);
  }
  __syncthreads();

  // ============ producer warpgroup: one thread streams the weights and the geo input, warps 9..11 encode the tile ahead ============
  constexpr int kEncWarp0 = (kTcThreads - kEncThreads) / 32;
  if (warp >= kEpiWarps) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kEpiWarps) {
      if (lane == 0) produce_all<P>(a, nlayers, abuf, ring, slots, bars);
    } else if (warp >= kEncWarp0) {
      encode_all<P, LAYOUT>(a, warp - kEncWarp0, lane, slots, bars, l2_policy_evict_last(), hs, hx, hxf);
    }
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();

  // ============================== two warpgroups, 64 rows of the tile each ==============================
  const int wg = warp >> 2, t = tid & 127;
  const int wrow0 = wg * 64;
  const int wg_bar = 1 + wg;                                 // named barrier of this warpgroup
  const uint32_t a_base = smem_u32(abuf) + wrow0 * 16;
  const float sdf_bias = __ldg(reinterpret_cast<const float*>(a.blob + a.b_g2));
  TileCtx x{a, tid, t, wg, wrow0, frag_row0(wrow0, t), frag_cq(t), abuf, prm, hs, coldesc, sdf_bias,
            reinterpret_cast<uint32_t*>(cta_scr + scr.sig), reinterpret_cast<uint8_t*>(cta_scr + scr.h2), slots};
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
    layer_mma<P, L>(acc, zero, a_base, ring, bars.ring, it, lane, waited, &bars.cop[wg][1], tile_no & 1); \
    named_sync(wg_bar, 128); /* every warp of the warpgroup is done reading this layer's A operand */  \
    TC_STAMP(1 + (L));                                                                                 \
  } while (0)

  int tile_no = -1;
  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    ++tile_no;
    TC_STAMP(0);
    waited = 0;
    const Slot<P> s(slots, bars.enc.slot(tile_no));
    x.hs = hs + bars.hs.slot(tile_no) * kHsRows;
    bars.a.wait_full(tile_no);                 // the geo input staged by the encoder warps has landed in A columns 0..95
    if (a.mode == 0) bars.enc.arrive_empty(tile_no);
    TC_STAMP(8);
    LAYER(L_G0, true);
    epi_e0<P>(x, acc);
    TC_STAMP(18);
    SYNC_A();
    LAYER(L_G1, true);
    if (a.mode == 0) {                         // sdf only: A is free for the next tile's geo input
      if (t == 0) bars.a.arrive_empty(tile_no);
      epi_e1<P>(x, tile, acc);
      continue;
    }
    {
      long long hs_waited = 0;
      bars.hs.wait_empty(tile_no, &hs_waited); // the encoder warps are done with the tile two before
      if (tid == 0) TC_PUT(tile_no, 16, hs_waited);
    }
    epi_e1<P>(x, tile, acc);
    TC_STAMP(19);
    SYNC_A();
    LAYER(L_B1, true);
    epi_eb1<P>(x, acc);
    TC_STAMP(20);
    SYNC_A();
    LAYER(L_B0, true);
    bars.enc.wait_full(tile_no);               // (long complete: the encoder's jacobian / colour-static stores are visible, and fenced
                                               // for the async proxy)
    if ((warp & 3) == 0) colour_copy<P>(x, true, s.cs(), &bars.cop[wg][0]);
    epi_eb0<P>(x, s, acc);
    mbar_wait(&bars.cop[wg][0], tile_no & 1);  // the colour-static columns and early h2 chunks have landed
    bars.enc.arrive_empty(tile_no);            // the slot's last reader (the early copy) is complete
    TC_STAMP(21);
    SYNC_A();
    LAYER(L_C0MISC, true);
    if ((warp & 3) == 0) colour_copy<P>(x, false, nullptr, &bars.cop[wg][1]);
    TC_STAMP(22);
    LAYER(L_C0H, false);                       // accumulates onto the misc columns' result; waits for the late h2 copy inside
    epi_ec0<P>(x, acc);
    TC_STAMP(23);
    SYNC_A();
    LAYER(L_C1, true);
    if (t == 0) bars.a.arrive_empty(tile_no);  // the last layer has read A: the next tile's geo input may land
    epi_ec1(x, acc);
    bars.hs.arrive_full(tile_no);              // the encoder warps take the tile from here
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
