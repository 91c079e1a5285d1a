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
//   heads    (one encoder warp, a tile behind) Laplace density, NeuS alpha, occupancy, normals; optional per-sample outputs
//   render   (fused mode, same warp) segmented prefix product over the rays of the tile in double, weights, per-ray sums
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

// accurate sin / sincos of the encoder warps.  Inlined: after setmaxnreg.dec a real call makes ptxas (CUDA 12.9) crash; both call
// sites are in the encoder loop, so this is two copies of the range reduction, not one per consumer epilogue
static __device__ __forceinline__ void sincos_call(float x, float* s, float* c) { sincosf(x, s, c); }
static __device__ __forceinline__ float sin_call(float x) { return sinf(x); }

// Hash-grid part of the geo input of one tile, levels 4 grp .. 4 grp + 3 of one point (= operand chunk grp).  Outputs: bf16 planes
// of the staged geo input image (`img`, planes `plane` bytes apart, kernel column order: four levels = one aligned 16-byte chunk)
// and the grid jacobian Jg [(col*3 + d)][row] (with the 1/4 of (x+2)/4 folded in).  One level at a time (smallest code).
template <int P, int LAYOUT>
__device__ __forceinline__ void encode_tile_grid(const TcArgs& a, int tile, int row, int grp, uint8_t* img, uint32_t plane, float* Jg,
                                                 uint64_t pol_table) {
  const long long p_raw = (long long)tile * 128 + row;
  const long long p = p_raw < a.n_points ? p_raw : a.n_points - 1;
  const PointGeom g = point_geom(a, p);
  const float x01 = (g.px + 2.0f) * 0.25f, y01 = (g.py + 2.0f) * 0.25f, z01 = (g.pz + 2.0f) * 0.25f;   // sdf_field.py:384
  // one level at a time, rolled (code size): 8 gathers in flight per thread, feature columns as 2-byte operand stores
#pragma unroll 1
  for (int l = 4 * grp; l < 4 * grp + 4; ++l) {
    float o[2] = {0.f, 0.f};
    float dj[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    if (a.use_grid && l < a.grid.n_levels && l < a.grid.active_levels) {
      LevelCtx c;
      float tv[8][2];
      level_prepare<LAYOUT>(a.grid, l, x01, y01, z01, c);
      level_fetch_rt2(a.grid, a.table, c, tv, pol_table);
      level_finish<2, LAYOUT>(a.grid, c, tv, o, dj);
    }
    store_a<P>(img, plane, row, 2 * l, o[0]);
    store_a<P>(img, plane, row, 2 * l + 1, o[1]);
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

// PE | x | zero padding: chunks 4..11 of the geo input.  Kernel column 32 + i holds PE_i, 32 + pe_dim + j holds x_j.  Also the
// point outputs (contracted position and its norm) of a valid row, and the PE jacobian Jpe [i][row].
template <int P>
__device__ __forceinline__ void encode_tile_pe(const TcArgs& a, int tile, int row, uint8_t* img, uint32_t plane, float* Jpe) {
  const long long p_raw = (long long)tile * 128 + row;
  const long long p = p_raw < a.n_points ? p_raw : a.n_points - 1;
  const PointGeom g = point_geom(a, p);
  if (p_raw < a.n_points) {
    if (a.out.points_norm) a.out.points_norm[p] = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(g.px, g.px), __fmul_rn(g.py, g.py)), __fmul_rn(g.pz, g.pz)));
    if (a.out.points) { a.out.points[p * 3] = g.px; a.out.points[p * 3 + 1] = g.py; a.out.points[p * 3 + 2] = g.pz; }
  }
  const int deg = a.pe_degree, half = 3 * deg;
  const float pc[3] = {g.px, g.py, g.pz};
  // zero the chunks first (padding columns), then the live columns as 2-byte stores (same thread: program order)
  const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
  for (int ch = 4; ch < kInK / 8; ++ch) store_a_chunk<P>(img, plane, row, ch, z4, z4);
#pragma unroll 1
  for (int i = 0; i < a.pe_dim; ++i) {                       // sin(x 2^k) | sin(x 2^k + pi/2)   (encodings.py:194-198)
    const int ia = i >= half ? i - half : i;
    const int b = ia / deg, k = ia - b * deg;
    const float fr = (float)(1 << k);
    const float xb = b == 0 ? pc[0] : (b == 1 ? pc[1] : pc[2]);
    const float arg = i >= half ? xb * fr + kHalfPiF : xb * fr;
    float sv, cv;
    sincos_call(arg, &sv, &cv);
    store_a<P>(img, plane, row, 32 + i, a.use_pe ? sv : 0.f);
    // autograd of sin on the forward's own fp32 arguments: d/dx_b = 2^k cos(arg)
    if (a.mode != 0) Jpe[i * 128 + row] = a.use_pe ? fr * cv : 0.f;
  }
  store_a<P>(img, plane, row, 32 + a.pe_dim + 0, pc[0]);
  store_a<P>(img, plane, row, 32 + a.pe_dim + 1, pc[1]);
  store_a<P>(img, plane, row, 32 + a.pe_dim + 2, pc[2]);
}

// static colour-operand columns of a tile (kernel columns 8..95 = chunks 1..11): x(3) | dir-enc(24) | dir(3) | appearance | 0, staged in
// the same [plane][chunk][row][16 B] layout as the A operand; EB0 copies them over the A columns that B0 has consumed (chunk 0 =
// [grad, n.v] comes from the epilogue)
template <int P>
__device__ __forceinline__ void colour_static_tile(const TcArgs& a, int tile, int row, uint8_t* img, uint32_t plane) {
  const long long p_raw = (long long)tile * 128 + row;
  const long long p = p_raw < a.n_points ? p_raw : a.n_points - 1;
  const PointGeom g = point_geom(a, p);
  const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
  for (int ch = 1; ch < kInK / 8; ++ch) store_a_chunk<P>(img, plane, row, ch, z4, z4);
  store_a<P>(img, plane, row, 8 + 0, g.px); store_a<P>(img, plane, row, 8 + 1, g.py); store_a<P>(img, plane, row, 8 + 2, g.pz);
  // direction encoding: sin(d 2^k) | sin(d 2^k + pi/2), k = 0..3, then d itself (NeRFEncoding(4, include_input), encodings.py:167-208)
#pragma unroll 1
  for (int i = 0; i < 12; ++i) {
    const int b = i >> 2;
    const float db = b == 0 ? g.dx : (b == 1 ? g.dy : g.dz);
    const float arg = db * (float)(1 << (i & 3));
    store_a<P>(img, plane, row, 8 + 3 + i, sin_call(arg));
    store_a<P>(img, plane, row, 8 + 15 + i, sin_call(arg + kHalfPiF));
  }
  store_a<P>(img, plane, row, 8 + 27, g.dx); store_a<P>(img, plane, row, 8 + 28, g.dy); store_a<P>(img, plane, row, 8 + 29, g.dz);
  if (a.appearance != nullptr) {
#pragma unroll 1
    for (int j = 0; j < a.app_dim; ++j) store_a<P>(img, plane, row, 8 + 30 + j, __ldg(a.appearance + g.ray * a.app_dim + j));
  }
}

// Staging slot s of the per-CTA scratch (tc_scratch)
template <int P>
struct Slot {
  uint8_t* base;
  __device__ __forceinline__ Slot(char* slots, uint32_t s) : base(reinterpret_cast<uint8_t*>(slots) + s * tc_scratch(P).slot_bytes) {}
  __device__ __forceinline__ uint8_t* geo() const { return base + tc_scratch(P).geo; }
  __device__ __forceinline__ uint8_t* cs() const { return base + tc_scratch(P).cs; }
  __device__ __forceinline__ float* jpe() const { return reinterpret_cast<float*>(base + tc_scratch(P).jpe); }
  __device__ __forceinline__ float* jg() const { return reinterpret_cast<float*>(base + tc_scratch(P).jg); }
};

#ifdef SDFB200_TC_TIMING
// CTA 0, first 16 tiles, row = tile: clock64() of consumer thread 0 at [0] tile start, [1..7] end of the MMAs of layer 0..6 (ring
// order), [8] the tile's geo input has landed (a full; [8] - [0] is the consumers' wait for the encoder), [15] tile end = end of EC1
// (head inputs handed over); cycle sums over the tile of [9] consumer thread 0 waiting for weights (ring full), [10] the producer
// waiting for a free ring slot (ring empty), [12] encoder thread 0 busy staging the tile, [13] encoder thread 0 waiting for its staging
// slot (enc empty), [14] encoder thread 0 (heads warp) running the tile's heads / compositing, [16] consumer thread 0 waiting for the
// tile's head-input buffer (hs empty), [17] the heads warp waiting for the tile's head inputs (hs full)
__device__ long long g_tc_timing[16 * 32];   // only the timing build of ONE instantiation defines SDFB200_TC_TIMING
#define TC_PUT(tno, k, v)                                                                                            \
  do {                                                                                                               \
    if (blockIdx.x == 0 && (tno) >= 0 && (tno) < 16) g_tc_timing[(tno) * 32 + (k)] = (v);                            \
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
  Handoff<2> hs;          // head inputs: full kEpiThreads (after EC1), empty 32 (the heads warp has read them); unused in sdf-only mode
};
static_assert(sizeof(TcBars) + 4 * sizeof(double) <= kStaticSmem, "static shared memory of k_field_tc (kStaticSmem)");

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
template <int P, int L>
__device__ __forceinline__ void layer_mma(float (&acc)[4][32], bool zero, uint32_t a_base, const uint8_t* ring, Handoff<kStages>& rb, uint32_t& it,
                                          int lane, long long& waited) {
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
    rb.wait_full(it, &waited);
    const uint32_t wbase = smem_u32(ring + (size_t)rb.slot(it) * tc_stage_bytes(P));
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
  uint32_t* gf_s;            //   h2 planes
  char* slots;               //   staging slots
  // this thread's 4-byte unit for the accumulator pair (c, i) in a [64 units][256 threads] scratch plane (sig_s, gf_s)
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

// E0 (after G0): h1 = softplus(z1) -> A ; softplus'(z1) -> scratch
template <int P>
__device__ __forceinline__ void epi_e0(const TileCtx& x, const float (&acc)[4][32]) {
  const float* p_bg0 = x.prm[PRM_B_G0];
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
      if (x.a.mode != 0) x.sig_s[x.unit(c, i)] = unorm16x2_encode(s0, s1);
    }
  }
}

// E1 (after G1): sdf = W2[0,:] . h2 + b (fp32) -> output / heads ; h2 -> scratch planes ; g2 = W2[0,:] * softplus'(z2) -> A
template <int P>
__device__ __forceinline__ void epi_e1(const TileCtx& x, int tile, const float (&acc)[4][32]) {
  const TcArgs& a = x.a;
  const float* p_bg1 = x.prm[PRM_B_G1];
  const float* p_wg2 = x.prm[PRM_W_G2];
  // one partial dot per accumulator row (r0, r0 + 8) as named scalars: an array indexed by the thread-dependent row below would live
  // in local memory, written back after every FMA because the generic stores in between may alias it
  float sp0 = 0.f, sp1 = 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const float2 b2 = *reinterpret_cast<const float2*>(p_bg1 + col);
      const float2 w2 = *reinterpret_cast<const float2*>(p_wg2 + col);
      float h0, h1, s0, s1;
      softplus100_fast(acc[c][i] + b2.x, h0, s0);
      softplus100_fast(acc[c][i + 1] + b2.y, h1, s1);
      float& sp = frag_half(i) ? sp1 : sp0;
      sp = fmaf(w2.x, h0, sp);
      sp = fmaf(w2.y, h1, sp);
      if (a.mode != 0) {
        uint32_t hi, lo;
        split2(h0, h1, hi, lo);
        const int u = x.unit(c, i);
        x.gf_s[u] = hi;
        if (P > 1) x.gf_s[kFragWords + u] = lo;
        store_a_pair<P>(x.abuf, kAPlane, row, col, w2.x * s0, w2.y * s1);
      }
    }
  }
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

// EB1 (after B1): g1 = (W1^T g2) * softplus'(z1) -> A
template <int P>
__device__ __forceinline__ void epi_eb1(const TileCtx& x, const float (&acc)[4][32]) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const uint32_t sw = x.sig_s[x.unit(c, i)];
      store_a_pair<P>(x.abuf, kAPlane, row, col, acc[c][i] * unorm16_lo(sw), acc[c][i + 1] * unorm16_hi(sw));
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

// EB0 (after B0): gin (96 cols, kernel order) . input jacobian -> d sdf / dx; then the colour misc operand over the (consumed) A columns
// 0..95: chunk 0 = [grad(3), n.v, 0 x4] (sdf_field.py:572-584; columns re-ordered at pack time) from the thread pair that owns the row,
// chunks 1..11 = [x, dir-enc, dir, appearance] copied from the tile's staging slot (16-byte units, the warpgroup's 64 rows)
template <int P>
__device__ __forceinline__ void epi_eb0(const TileCtx& x, int tile, const Slot<P>& s, const float (&acc)[4][32]) {
  const TcArgs& a = x.a;
  const float* Jpe = s.jpe();
  const float* Jg = s.jg();
  // colour-static units (below) loaded first, so that they are in flight together with the jacobian loads
  // unit k: plane k / (11 * 64), chunk 1 + (k / 64) % 11, row wrow0 + k % 64
  constexpr int kUnits = 11 * 64 * P, kPer = (kUnits + 127) / 128;
  uint4 v[kPer];
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    const int k = x.t + 128 * j, pl = k / (11 * 64), ch = 1 + (k - pl * 11 * 64) / 64, row = x.wrow0 + (k & 63);
    if (k < kUnits) v[j] = *reinterpret_cast<const uint4*>(s.cs() + pl * kImgPlane + ch * kAChunk + row * 16);
  }
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
    const long long p_raw = (long long)tile * 128 + row;
    const PointGeom pg = point_geom(a, p_raw < a.n_points ? p_raw : a.n_points - 1);
    const float grx = h ? g1x : g0x, gry = h ? g1y : g0y, grz = h ? g1z : g0z;
    const float gn = fmaxf(sqrtf(grx * grx + gry * gry + grz * grz), 1e-12f);      // F.normalize eps
    const float c0v[8] = {grx, gry, grz, a.use_n_dot_v ? (grx / gn) * pg.dx + (gry / gn) * pg.dy + (grz / gn) * pg.dz : 0.f, 0.f, 0.f, 0.f, 0.f};
    store_a_chunk<P>(x.abuf, kAPlane, row, 0, c0v);
    x.hs[HS_GRAD][row] = grx; x.hs[HS_GRAD + 1][row] = gry; x.hs[HS_GRAD + 2][row] = grz;
  }
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    const int k = x.t + 128 * j, pl = k / (11 * 64), ch = 1 + (k - pl * 11 * 64) / 64, row = x.wrow0 + (k & 63);
    if (k < kUnits) *reinterpret_cast<uint4*>(x.abuf + pl * kAPlane + ch * kAChunk + row * 16) = v[j];
  }
}

// C0 h2 operand: h2 (bf16 planes, saved by E1) back from the scratch over the misc columns that C0's first part has consumed
template <int P>
__device__ __forceinline__ void reload_h2(const TileCtx& x) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(x.cq, c, i), row = frag_row(x.r0, i);
      const int u = x.unit(c, i);
      store_a_pair<P>(x.abuf, kAPlane, row, col, x.gf_s[u], x.gf_s[kFragWords + u]);
    }
  }
}

// EC0 (after C0): relu -> A
template <int P>
__device__ __forceinline__ void epi_ec0(const TileCtx& x, const float (&acc)[4][32]) {
  const float* p_bc0 = x.prm[PRM_B_C0];
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
  const float* p_bc1 = x.prm[PRM_B_C1];
  const float (*p_wc2)[256] = x.prm + PRM_W_C2;
  float r0r = 0.f, r0g = 0.f, r0b = 0.f, r1r = 0.f, r1g = 0.f, r1b = 0.f;   // rows r0, r0 + 8 (named scalars, see epi_e1)
#pragma unroll
  for (int c = 0; c < 4; ++c) {
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = frag_col(x.cq, c, i);
      const bool h = frag_half(i);
      float& rr = h ? r1r : r0r;
      float& rg = h ? r1g : r0g;
      float& rb = h ? r1b : r0b;
      const float v = fmaxf(acc[c][i] + p_bc1[col], 0.f);
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

// Per-point heads and, in fused mode, the per-ray compositing of one tile, run by one encoder warp on the head inputs `hs` that the
// consumers left (sdf, gradient, raw rgb; the geometry is recomputed).  The warp walks the four 32-row chunks of the tile in order,
// lane = row in the chunk.  A ray of S <= 32 samples lies in one chunk; a longer one spans S / 32 chunks: the chunk totals of its
// transmittance scan go through `wtot` (chunk q -> wtot[q]) and its sums are carried from chunk to chunk in registers and written at
// its last chunk, always in the same order.
__device__ __forceinline__ void heads_and_composite(const TcArgs& a, const float (*hs)[128], int tile, int lane, double* wtot) {
  const float* b_c2 = reinterpret_cast<const float*>(a.blob + a.b_c2);
  float csum[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};     // sums of the chunks so far of a ray longer than 32 samples
#pragma unroll 1
  for (int q = 0; q < 4; ++q) {
  const int row = q * 32 + lane;
  const long long p_raw = (long long)tile * 128 + row;
  const bool valid = p_raw < a.n_points;
  const long long p = valid ? p_raw : a.n_points - 1;
  const PointGeom pg = point_geom(a, p);
  const float dirx = pg.dx, diry = pg.dy, dirz = pg.dz, delta = pg.delta;
  const float sdf = hs[HS_SDF][row], grx = hs[HS_GRAD][row], gry = hs[HS_GRAD + 1][row], grz = hs[HS_GRAD + 2][row];
  const float gn = fmaxf(sqrtf(grx * grx + gry * gry + grz * grz), 1e-12f);      // F.normalize eps
  const float nx = grx / gn, ny = gry / gn, nz = grz / gn;
  float rgbv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float raw = hs[HS_RGB + c][row] + __ldg(b_c2 + c);
    rgbv[c] = sigmoidf_(raw) * (1.f + 2.f * a.rgb_padding) - a.rgb_padding;
  }
  float density = 0.f, alpha = 0.f;
  if (a.out.density || (a.render && a.rnd.from_density)) {
    const float beta = fabsf(__ldg(a.beta)) + __ldg(a.beta_min);
    const float sg = sdf > 0.f ? 1.f : (sdf < 0.f ? -1.f : 0.f);
    density = (1.0f / beta) * (0.5f + 0.5f * sg * expm1f(-fabsf(sdf) / beta));
  }
  if (a.out.alpha || (a.render && !a.rnd.from_density)) {
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
  if (a.render) {
    // ---------------- fused compositing: the tile holds 128 / S whole rays; row -> (ray, sample) = (row / S, row % S) ----------------
    const int S = a.n_samples;
    const int s_idx = row % S;
    const bool dens = a.rnd.from_density != 0;
    const bool multi = S > 32;                                // the ray spans chunks (warp-uniform)
    const int first = multi ? (q * 32 / S) * (S / 32) : q;    // first chunk of the ray
    const bool ray_end = !multi || q == first + S / 32 - 1;   // this chunk ends the ray (warp-uniform)
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
    if (multi) {
      __syncwarp();                                           // every lane is through its reads of wtot from the chunk before
      if (lane == 31) wtot[q] = incl;
      __syncwarp();
      for (int w2 = first; w2 < q; ++w2) excl = dens ? excl + wtot[w2] : excl * wtot[w2];
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
    if (a.rnd.out.steps_minmax && lane == 0 && smin <= smax) { atomic_min_float(a.rnd.out.steps_minmax, smin); atomic_max_float(a.rnd.out.steps_minmax + 1, smax); }
    // transmittance after the last sample (alphas: transmittance[:, -1] = bg_transmittance, neus.py:101) / before it (densities:
    // volsdf.py:67-68), and the colour of the last sample
    double tot;
    float lr, lg, lb;
    if (multi) {
#pragma unroll
      for (int k = 0; k < 8; ++k) { csum[k] += vs[k]; vs[k] = csum[k]; }   // lane 0: the chunk's sums, then the ray's so far
      if (dens) {
        tot = __shfl_sync(0xffffffffu, excl, 31);
      } else {
        tot = 1.0;
        for (int w2 = first; w2 <= q; ++w2) tot *= wtot[w2];
      }
      lr = __shfl_sync(0xffffffffu, rgbv[0], 31); lg = __shfl_sync(0xffffffffu, rgbv[1], 31); lb = __shfl_sync(0xffffffffu, rgbv[2], 31);
    } else {
      const int last = (lane - s_idx) + S - 1;
      tot = __shfl_sync(0xffffffffu, dens ? excl : incl, last);
      lr = __shfl_sync(0xffffffffu, rgbv[0], last); lg = __shfl_sync(0xffffffffu, rgbv[1], last); lb = __shfl_sync(0xffffffffu, rgbv[2], last);
    }
    const long long ray = (long long)tile * (128 / S) + row / S;
    if (ray_end && s_idx == (multi ? S - 32 : 0) && ray * S < a.n_points) {
      const float acc = vs[0];
      if (a.rnd.out.rgb) {
        float bgc[3] = {0.f, 0.f, 0.f};
        if (a.rnd.bg_mode == SDFB200_BG_COLOR) { bgc[0] = a.rnd.bg[0]; bgc[1] = a.rnd.bg[1]; bgc[2] = a.rnd.bg[2]; }
        else if (a.rnd.bg_mode == SDFB200_BG_PER_RAY) { bgc[0] = a.rnd.bg[ray * 3]; bgc[1] = a.rnd.bg[ray * 3 + 1]; bgc[2] = a.rnd.bg[ray * 3 + 2]; }
        else { bgc[0] = lr; bgc[1] = lg; bgc[2] = lb; }
        const float rem = 1.0f - acc;
        const float o[3] = {vs[1] + bgc[0] * rem, vs[2] + bgc[1] * rem, vs[3] + bgc[2] * rem};
#pragma unroll
        for (int c = 0; c < 3; ++c) a.rnd.out.rgb[ray * 3 + c] = a.rnd.clamp01 ? fminf(fmaxf(o[c], 0.f), 1.f) : o[c];
      }
      if (a.rnd.out.accumulation) a.rnd.out.accumulation[ray] = acc;
      if (a.rnd.out.normal) { a.rnd.out.normal[ray * 3] = vs[4]; a.rnd.out.normal[ray * 3 + 1] = vs[5]; a.rnd.out.normal[ray * 3 + 2] = vs[6]; }
      if (a.rnd.out.depth) a.rnd.out.depth[ray] = vs[7] / (acc + 1e-10f);
      if (a.rnd.bg_transmittance) a.rnd.bg_transmittance[ray] = dens ? expf(-(float)tot) : (float)tot;
    }
    if (multi && ray_end) {
#pragma unroll
      for (int k = 0; k < 8; ++k) csum[k] = 0.f;
    }
  }
  }
}

// The heads warp's part of a tile: wait for its head inputs, run the heads, hand the buffer back
__device__ __forceinline__ void heads_of(const TcArgs& a, int tile, int tile_no, int lane, TcBars& b, float (*hs)[128], double* wtot) {
  long long waited = 0;
  b.hs.wait_full(tile_no, &waited);
  const long long t0 = TC_CLOCK();
  heads_and_composite(a, hs + b.hs.slot(tile_no) * kHsRows, tile, lane, wtot);
  b.hs.arrive_empty(tile_no);
  if (lane == 0) { TC_PUT(tile_no, 14, TC_CLOCK() - t0); TC_PUT(tile_no, 17, waited); }
}

// Encoder warps (et = 0..95): walk the same tiles as the consumers and stage each one in its slot while the consumers run the tile
// before it.  A tile is 768 items, 8 per thread: 512 (point, group of four hash levels), then 128 x (PE | x, point outputs) and, with
// the colour MLP, 128 x colour-static columns.  Item i goes to thread i % 96, so each warp runs 32 consecutive items of one kind.
// Except in sdf-only mode, the first encoder warp then runs the heads of the tile before (the one the consumers are finishing), and
// those of the last tile after the loop.  Staging tile n + 1 and the heads of tile n - 1 both fit in the consumers' tile n: slot
// n + 1 was freed at EB0 of tile n - 1, and the head inputs of tile n - 1 are ready when tile n starts.
template <int P, int LAYOUT>
__device__ __forceinline__ void encode_all(const TcArgs& a, int et, char* slots, TcBars& b, uint64_t pol_table, float (*hs)[128], double* wtot) {
  const int n_items = a.mode != 0 ? 768 : 640;
  const bool heads = a.mode != 0 && et < 32;     // the first encoder warp also runs the heads of the tile before
  int tile_no = 0;
  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x, ++tile_no) {
    long long waited = 0;
    b.enc.wait_empty(tile_no, &waited);
    const long long t0 = TC_CLOCK();
    const Slot<P> s(slots, b.enc.slot(tile_no));
#pragma unroll 1
    for (int i = et; i < n_items; i += kEncThreads) {
      const int row = i & 127;
      if (i < 512) encode_tile_grid<P, LAYOUT>(a, tile, row, i >> 7, s.geo(), kImgPlane, s.jg(), pol_table);
      else if (i < 640) encode_tile_pe<P>(a, tile, row, s.geo(), kImgPlane, s.jpe());
      else colour_static_tile<P>(a, tile, row, s.cs(), kImgPlane);
    }
    fence_async_global();                    // the geo image is read by the producer's bulk copy (async proxy)
    b.enc.arrive_full(tile_no);
    if (et == 0) { TC_PUT(tile_no, 12, TC_CLOCK() - t0); TC_PUT(tile_no, 13, waited); }
    if (heads && tile_no > 0) heads_of(a, tile - (int)gridDim.x, tile_no - 1, et, b, hs, wtot);
  }
  if (heads && tile_no > 0) heads_of(a, blockIdx.x + (tile_no - 1) * (int)gridDim.x, tile_no - 1, et, b, hs, wtot);   // the last tile
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
  __shared__ TcBars bars;
  __shared__ double wtot[4];          // chunk totals of the compositing scan (heads warp)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nlayers = a.mode == 0 ? 2 : L_COUNT;
  char* cta_scr = a.scratch + (size_t)blockIdx.x * scr.bytes;
  char* slots = cta_scr + scr.slots;
  if (tid == 0) {
    bars.ring.init(1, kEpiWarps);
    bars.enc.init(kEncThreads, kEpiThreads);
    bars.hs.init(kEpiThreads, 32);
    bars.a.init(1, 2);
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
  if (tid >= kEpiThreads) {
    setmaxnreg_dec<kProducerRegs>();
    if (tid == kEpiThreads) produce_all<P>(a, nlayers, abuf, ring, slots, bars);
    else if (tid >= kTcThreads - kEncThreads) encode_all<P, LAYOUT>(a, tid - (kTcThreads - kEncThreads), slots, bars, l2_policy_evict_last(), hs, wtot);
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
            reinterpret_cast<uint32_t*>(cta_scr + scr.sig), reinterpret_cast<uint32_t*>(cta_scr + scr.h2), slots};
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
    layer_mma<P, L>(acc, zero, a_base, ring, bars.ring, it, lane, waited);                             \
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
    SYNC_A();
    LAYER(L_G1, true);
    if (a.mode == 0) {                         // sdf only: A is free for the next tile's geo input
      if (t == 0) bars.a.arrive_empty(tile_no);
      epi_e1<P>(x, tile, acc);
      continue;
    }
    {
      long long hs_waited = 0;
      bars.hs.wait_empty(tile_no, &hs_waited); // the heads warp is done with the tile two before
      if (tid == 0) TC_PUT(tile_no, 16, hs_waited);
    }
    epi_e1<P>(x, tile, acc);
    SYNC_A();
    LAYER(L_B1, true);
    epi_eb1<P>(x, acc);
    SYNC_A();
    LAYER(L_B0, true);
    bars.enc.wait_full(tile_no);               // (long complete: makes the encoder's jacobian / colour-static stores visible)
    epi_eb0<P>(x, tile, s, acc);
    bars.enc.arrive_empty(tile_no);
    SYNC_A();
    LAYER(L_C0MISC, true);
    reload_h2<P>(x);
    SYNC_A();
    LAYER(L_C0H, false);                       // accumulates onto the misc columns' result
    epi_ec0<P>(x, acc);
    SYNC_A();
    LAYER(L_C1, true);
    if (t == 0) bars.a.arrive_empty(tile_no);  // the last layer has read A: the next tile's geo input may land
    epi_ec1(x, acc);
    bars.hs.arrive_full(tile_no);              // the heads warp takes the tile from here
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
