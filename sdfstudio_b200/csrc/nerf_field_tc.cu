// Vanilla NeRF background field (background_model="mlp", models/base_surface_model.py:188-201): the eval forward of NeRFField
// (nerfstudio/fields/vanilla_nerf_field.py:91-114 through fields/base_field.py:104-123) as one fused tensor-core kernel, and its C-ABI.
//
//   PE      sin(cat[x f_k, x f_k + pi/2]) | x           (encodings.py:167-208, 63 columns at SurfaceModel's shape)
//   L0..L7  Linear + ReLU, 256 wide, L4 takes cat([PE, h])   (field_components/mlp.py:80-99, out_activation ReLU)
//   density softplus(w_d . h8 + b_d)                         (field_heads.py:99-108, nn.Softplus: beta 1, threshold 20)
//   H0, H1  Linear + ReLU, 128 wide, H0 takes cat([dir-enc, h8])
//   rgb     sigmoid(W_rgb h + b_rgb)                         (field_heads.py:111-120)
//
// Persistent CTAs, one 128-sample tile at a time.  Two consumer warpgroups own 64 rows of the tile each: they encode their rows, run
// every layer as wgmma m64n256k16 (m64n128k16 for the head) with the accumulator in registers and the A operand in shared memory, and
// write each layer's ReLU output over the same A buffer as the next layer's input.  The positional encoding lives in a separate 64-column
// buffer until L4 has read it; the direction encoding then takes its place until H0.  One thread of a third warpgroup streams the
// weights, pre-packed in consumption order (tc_pack), through a ring of equal-sized stages.  The density and rgb heads are fp32 dots in
// the epilogues.  MMA = bf16 x bf16 -> fp32; bf16x3 (P = 2): a0 w0 + a1 w0 + a0 w1 with a = a0 + a1, w = w0 + w1.
#include "tc_common.cuh"
#include "tc_linear.h"

#include <algorithm>

namespace sdfb200 {
using namespace tc;

namespace nerf {

constexpr int kThreads = 384;              // two consumer warpgroups + the producer warpgroup
constexpr int kConsumerThreads = 256;
constexpr int kConsumerWarps = kConsumerThreads / 32;
// the launch gets 168 registers per thread; the producer warpgroup gives back what the consumers take: 256 x (232 - 168) = 128 x (168 - 40)
constexpr int kConsumerRegs = 232;
constexpr int kProducerRegs = 40;
static_assert(2 * (kConsumerRegs - 168) <= 168 - kProducerRegs, "setmaxnreg.inc would wait for registers nobody frees");

constexpr int kBase = 8, kSkip = 4, kWidth = 256, kHeadWidth = 128;
constexpr int kEncCols = 64;               // padded width of either encoding (at most 6 * 10 + 3 = 63 columns)
constexpr int kKB = 16;                    // K per streamed block of a 256-row layer; a 128-row layer streams 32 (the same bytes)
constexpr float kHalfPi = 1.5707963267948966f;
__host__ __device__ constexpr uint32_t stage_bytes(int planes) { return (uint32_t)planes * kWidth * kKB * 2; }
template <int P>
struct Stages { static constexpr int value = P == 2 ? 3 : 6; };

// weight blocks in the order the consumers take them (one ring stage each): L0 4 (PE), L1..L3 16, L4 4 (PE) + 16, L5..L7 16,
// H0 2 (direction encoding) + 8, H1 4
__host__ __device__ constexpr int layer_nkb(int L) { return L == 0 ? 4 : (L == kSkip ? 20 : (L < kBase ? 16 : (L == kBase ? 10 : 4))); }
__host__ __device__ constexpr int layer_enc_kb(int L) { return L == 0 || L == kSkip ? 4 : (L == kBase ? 2 : 0); }
__host__ __device__ constexpr int layer_first_block(int L) {
  int b = 0;
  for (int i = 0; i < L; ++i) b += layer_nkb(i);
  return b;
}
constexpr int kLayers = kBase + 2;
constexpr int kBlocks = layer_first_block(kLayers);
static_assert(kBlocks == 134, "weight blocks per tile");

// fp32 section at the start of the packed blob, copied to shared memory once per CTA: biases and the rows of the dot-product heads
enum : int {
  PRM_B_BASE = 0,                              // [8][256]
  PRM_B_HEAD = PRM_B_BASE + kBase * kWidth,    // [2][128]
  PRM_W_D = PRM_B_HEAD + 2 * kHeadWidth,       // [256]
  PRM_W_RGB = PRM_W_D + kWidth,                // [3][128]
  PRM_B_D = PRM_W_RGB + 3 * kHeadWidth,        // [1]
  PRM_B_RGB = PRM_B_D + 1,                     // [3]
  kPrmFloats = PRM_B_RGB + 3
};
constexpr size_t kBlobWOff = (kPrmFloats * 4 + 1023) / 1024 * 1024;   // the weight blocks start here (bulk copies need 16-byte alignment)
__host__ __device__ constexpr size_t packed_bytes(int planes) { return kBlobWOff + (size_t)kBlocks * stage_bytes(planes); }

// A operand / encoding buffer: [plane][k/8][128 rows][16 B] (tc_common.cuh), planes kAPlane / kEPlane bytes apart
constexpr uint32_t kAPlane = (kWidth / 8) * kAChunk;
constexpr uint32_t kEPlane = (kEncCols / 8) * kAChunk;

// Dynamic shared memory: byte offsets from its 1024-aligned base
struct NfSmem { size_t a, enc, ring, prm, bytes; };
__host__ __device__ constexpr NfSmem nf_smem(int planes, int stages) {
  NfSmem s{};                                                   // a: hidden activations, [P][32 chunks][128 rows][16 B]
  s.enc = s.a + (size_t)planes * kAPlane;                       // PE until L4, then the direction encoding until H0
  s.ring = s.enc + (size_t)planes * kEPlane;                    // weight ring: `stages` x one block
  s.prm = s.ring + (size_t)stages * stage_bytes(planes);        // fp32 section of the blob
  s.bytes = s.prm + kPrmFloats * 4;
  return s;
}
constexpr size_t kSmemPerBlock = 232448;   // H100: 227 KB of shared memory per block (dynamic + static)
constexpr size_t kStaticSmem = 1024;       // the ring barriers, in one 1024-byte slot (the dynamic part is 1024-aligned)
static_assert(nf_smem(2, Stages<2>::value).bytes + kStaticSmem <= kSmemPerBlock, "shared memory of k_nerf_field_tc at two planes");
static_assert(nf_smem(1, Stages<1>::value).bytes + kStaticSmem <= kSmemPerBlock, "shared memory of k_nerf_field_tc at one plane");

struct NfArgs {
  const char* blob;
  const float *origins, *directions, *bins;
  float *density, *rgb;
  long long n;
  int S, contraction, n_tiles;
  int pe_f, pe_inc, dir_f, dir_inc;
  float pe_freq[SDFB200_NERF_MAX_FREQS], dir_freq[SDFB200_NERF_MAX_FREQS];
};

__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// position (contracted) and direction of sample p (ray mode: the midpoint of its bin)
__device__ __forceinline__ void sample_geom(const NfArgs& a, long long p, float (&x)[3], float (&d)[3]) {
  if (a.S) {
    const long long r = p / a.S;
    ray_midpoint(a.origins, a.directions, a.bins, r, a.S, p - r * a.S, x);
#pragma unroll
    for (int c = 0; c < 3; ++c) d[c] = __ldg(a.directions + r * 3 + c);
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) { x[c] = __ldg(a.origins + p * 3 + c); d[c] = __ldg(a.directions + p * 3 + c); }
  }
  scene_contract(a.contraction, x[0], x[1], x[2]);
}

// column c of NeRFEncoding(v): sin(v_b f_k) at b F + k, sin(v_b f_k + pi/2) at 3F + b F + k (fp32 product, fp32 sum, accurate sinf), then
// v itself when included, then zero padding
__device__ __forceinline__ float enc_value(int c, const float (&v)[3], int F, const float* freqs, int inc) {
  const int h = 3 * F;
  if (c < 2 * h) {
    const int ia = c < h ? c : c - h;
    const int b = ia / F, k = ia - b * F;
    float arg = __fmul_rn(b == 0 ? v[0] : (b == 1 ? v[1] : v[2]), freqs[k]);
    if (c >= h) arg = __fadd_rn(arg, kHalfPi);
    return sinf(arg);
  }
  const int b = c - 2 * h;
  return inc && b < 3 ? (b == 0 ? v[0] : (b == 1 ? v[1] : v[2])) : 0.f;
}

// the position (dir = false) or direction encoding of the warpgroup's 64 rows into the encoding buffer: two threads per row, 32 columns each
template <int P>
__device__ __forceinline__ void encode_rows(const NfArgs& a, int tile, int t, int wrow0, uint8_t* ebuf, bool dir) {
  const int row = wrow0 + (t & 63), c0 = (t >> 6) * 32;
  const long long p_raw = (long long)tile * 128 + row;
  float x[3], d[3];
  sample_geom(a, p_raw < a.n ? p_raw : a.n - 1, x, d);
  const int F = dir ? a.dir_f : a.pe_f, inc = dir ? a.dir_inc : a.pe_inc;
  const float* freqs = dir ? a.dir_freq : a.pe_freq;
#pragma unroll 1
  for (int c = c0; c < c0 + 32; c += 2) {
    const float v0 = dir ? enc_value(c, d, F, freqs, inc) : enc_value(c, x, F, freqs, inc);
    const float v1 = dir ? enc_value(c + 1, d, F, freqs, inc) : enc_value(c + 1, x, F, freqs, inc);
    store_a_pair<P>(ebuf, kEPlane, row, c, v0, v1);
  }
}

// All MMAs of one layer for the 64 rows of a warpgroup: acc = A W^T, blocks taken from the ring in order; the first n_enc blocks read
// the encoding buffer, the rest the A buffer.  Every consumer warp releases a slot once its MMAs on it are complete.
template <int P, int N, int S>
__device__ __forceinline__ void layer_mma(float (&acc)[128], int nkb, int n_enc, uint32_t a_base, uint32_t e_base, const uint8_t* ring, Handoff<S>& rb,
                                          uint32_t& it, int lane) {
  constexpr int KBLK = kKB * kWidth / N, KS = KBLK / 16;
  constexpr uint32_t lbo_b = N * 16, plane_b = N * KBLK * 2;
  float (&d)[N / 2] = *reinterpret_cast<float (*)[N / 2]>(&acc[0]);
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
#pragma unroll 1
  for (int kb = 0; kb < nkb; ++kb, ++it) {
    rb.wait_full(it);
    const uint32_t wbase = smem_u32(ring + (size_t)rb.slot(it) * stage_bytes(P));
    const bool enc = kb < n_enc;
    const uint32_t base = enc ? e_base : a_base, plane = enc ? kEPlane : kAPlane;
    const int kb0 = enc ? kb : kb - n_enc;
    wg_fence_acc(d);
    wg_arrive();
#pragma unroll
    for (int j = 0; j < KS; ++j) {
      const int ks = kb0 * KS + j;
      wgmma_kstep_wide_ss<P, N>(d, a_desc(base, ks), a_desc(base + plane, ks), wbase + j * 2 * lbo_b, plane_b, lbo_b);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(d);
    __syncwarp();
    if (lane == 0) rb.arrive_empty(it);
  }
}

// ReLU(acc + b) of an N-wide layer over columns 0..N-1 of the A buffer.  With wd != nullptr (L7) also the density of the thread's rows:
// softplus(w_d . h + b_d) as an fp32 dot, one partial per accumulator row (named scalars: an array indexed by the row would live in
// local memory), summed over the quad in a fixed order
template <int P, int N>
__device__ __forceinline__ void epi_relu(const float (&acc)[128], const float* bias, uint8_t* abuf, int r0, int cq, const float* wd, float bd, int t,
                                         long long tile, const NfArgs& a) {
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int c = 0; c < N / 64; ++c) {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int col = frag_col(cq, c, i), row = frag_row(r0, i);
      const float2 b2 = *reinterpret_cast<const float2*>(bias + col);
      const float h0 = fmaxf(acc[c * 32 + i] + b2.x, 0.f), h1 = fmaxf(acc[c * 32 + i + 1] + b2.y, 0.f);
      store_a_pair<P>(abuf, kAPlane, row, col, h0, h1);
      if (wd) {
        const float2 w2 = *reinterpret_cast<const float2*>(wd + col);
        float& s = frag_half(i) ? s1 : s0;
        s = fmaf(w2.x, h0, s);
        s = fmaf(w2.y, h1, s);
      }
    }
  }
  if (wd) {
    s0 = quad_sum(s0);
    s1 = quad_sum(s1);
    if ((t & 3) < 2) {
      const int h = t & 1;
      const long long p = tile * 128 + r0 + 8 * h;
      const float z = (h ? s1 : s0) + bd;
      if (p < a.n) a.density[p] = z > 20.f ? z : log1pf(expf(z));
    }
  }
}

// H1: ReLU(acc + b), then rgb = sigmoid(W_rgb h + b_rgb) as three fp32 dots
__device__ __forceinline__ void epi_rgb(const float (&acc)[128], const float* prm, int r0, int cq, int t, long long tile, const NfArgs& a) {
  const float* bias = prm + PRM_B_HEAD + kHeadWidth;
  const float* w = prm + PRM_W_RGB;
  float r0r = 0.f, r0g = 0.f, r0b = 0.f, r1r = 0.f, r1g = 0.f, r1b = 0.f;
#pragma unroll
  for (int c = 0; c < kHeadWidth / 64; ++c) {
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = frag_col(cq, c, i);
      const bool h = frag_half(i);
      float& rr = h ? r1r : r0r;
      float& rg = h ? r1g : r0g;
      float& rb = h ? r1b : r0b;
      const float v = fmaxf(acc[c * 32 + i] + bias[col], 0.f);
      rr = fmaf(w[col], v, rr);
      rg = fmaf(w[kHeadWidth + col], v, rg);
      rb = fmaf(w[2 * kHeadWidth + col], v, rb);
    }
  }
  r0r = quad_sum(r0r); r0g = quad_sum(r0g); r0b = quad_sum(r0b);
  r1r = quad_sum(r1r); r1g = quad_sum(r1g); r1b = quad_sum(r1b);
  if ((t & 3) < 2) {
    const int h = t & 1;
    const long long p = tile * 128 + r0 + 8 * h;
    if (p < a.n) {
      a.rgb[p * 3 + 0] = sigmoidf_((h ? r1r : r0r) + prm[PRM_B_RGB + 0]);
      a.rgb[p * 3 + 1] = sigmoidf_((h ? r1g : r0g) + prm[PRM_B_RGB + 1]);
      a.rgb[p * 3 + 2] = sigmoidf_((h ? r1b : r0b) + prm[PRM_B_RGB + 2]);
    }
  }
}

template <int P>
__global__ void __launch_bounds__(kThreads, 1) k_nerf_field_tc(const __grid_constant__ NfArgs a) {
  constexpr int S = Stages<P>::value;
  constexpr NfSmem sm = nf_smem(P, S);
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* abuf = smem + sm.a;
  uint8_t* ebuf = smem + sm.enc;
  uint8_t* ring = smem + sm.ring;
  float* prm = reinterpret_cast<float*>(smem + sm.prm);
  __shared__ Handoff<S> rb;   // weight ring: full 1 + bytes, empty one arrival per consumer warp

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    rb.init(1, kConsumerWarps);
    fence_barrier_init();
  }
  for (int i = tid; i < kPrmFloats; i += kThreads) prm[i] = __ldg(reinterpret_cast<const float*>(a.blob) + i);
  __syncthreads();

  // ============ producer warpgroup: one thread streams every weight block of every tile ============
  if (tid >= kConsumerThreads) {
    setmaxnreg_dec<kProducerRegs>();
    if (tid == kConsumerThreads) {
      const uint8_t* blocks = reinterpret_cast<const uint8_t*>(a.blob) + kBlobWOff;
      uint32_t j = 0;
      for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x)
        for (int kb = 0; kb < kBlocks; ++kb, ++j) ring_fill(rb, ring, j, blocks, kb, stage_bytes(P));
    }
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();

  // ============ two consumer warpgroups, 64 rows of the tile each ============
  const int wg = warp >> 2, t = tid & 127, wrow0 = wg * 64, wg_bar = 1 + wg;
  const uint32_t a_base = smem_u32(abuf) + wrow0 * 16, e_base = smem_u32(ebuf) + wrow0 * 16;
  const int r0 = frag_row0(wrow0, t), cq = frag_cq(t);
  const float bd = prm[PRM_B_D];
  uint32_t it = 0;
  float acc[128];
  auto sync_a = [&]() {       // this warpgroup's operand writes are visible to its next MMAs
    fence_async_smem();
    named_sync(wg_bar, 128);
  };
  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    encode_rows<P>(a, tile, t, wrow0, ebuf, false);
    sync_a();
#pragma unroll 1
    for (int L = 0; L < kBase; ++L) {
      layer_mma<P, kWidth>(acc, layer_nkb(L), layer_enc_kb(L), a_base, e_base, ring, rb, it, lane);
      named_sync(wg_bar, 128);   // every warp of the warpgroup is done reading this layer's operands
      epi_relu<P, kWidth>(acc, prm + PRM_B_BASE + L * kWidth, abuf, r0, cq, L == kBase - 1 ? prm + PRM_W_D : nullptr, bd, t, tile, a);
      if (L == kSkip) encode_rows<P>(a, tile, t, wrow0, ebuf, true);   // L4 was the last reader of the PE
      sync_a();
    }
    layer_mma<P, kHeadWidth>(acc, layer_nkb(kBase), layer_enc_kb(kBase), a_base, e_base, ring, rb, it, lane);
    named_sync(wg_bar, 128);
    epi_relu<P, kHeadWidth>(acc, prm + PRM_B_HEAD, abuf, r0, cq, nullptr, 0.f, t, tile, a);
    sync_a();
    layer_mma<P, kHeadWidth>(acc, layer_nkb(kBase + 1), layer_enc_kb(kBase + 1), a_base, e_base, ring, rb, it, lane);
    named_sync(wg_bar, 128);   // the next tile's encoding and L0 epilogue may overwrite the operands
    epi_rgb(acc, prm, r0, cq, t, tile, a);
  }
}

int in_family(const sdfb200_nerf_field_t* f) {
  auto enc_ok = [](int F, int inc) { return F >= 0 && F <= SDFB200_NERF_MAX_FREQS && (inc == 0 || inc == 1) && 6 * F + 3 * inc >= 1; };
  return f != nullptr && f->base_layers == kBase && f->base_width == kWidth && f->skip_layer == kSkip && f->head_layers == 2 &&
         f->head_width == kHeadWidth && enc_ok(f->pe_frequencies, f->pe_include_input) && enc_ok(f->dir_frequencies, f->dir_include_input) &&
         f->contraction >= SDFB200_CONTRACT_NONE && f->contraction <= SDFB200_CONTRACT_L2 &&
         (f->precision == SDFB200_PRECISION_BF16X3 || f->precision == SDFB200_PRECISION_BF16);
}

int planes_of(const sdfb200_nerf_field_t* f) { return f->precision == SDFB200_PRECISION_BF16 ? 1 : 2; }

template <int P>
int launch(const NfArgs& a, cudaStream_t st) {
  const size_t smem = nf_smem(P, Stages<P>::value).bytes;
  SDFB_CUDA(cudaFuncSetAttribute(k_nerf_field_tc<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = (int)std::min<long long>(a.n_tiles, persistent_ctas());
  k_nerf_field_tc<P><<<grid, kThreads, smem, st>>>(a);
  SDFB_LAUNCHED("k_nerf_field_tc");
  return 0;
}

}  // namespace nerf
}  // namespace sdfb200

using namespace sdfb200;

extern "C" int sdfb200_nerf_field_in_family(const sdfb200_nerf_field_t* f) { return nerf::in_family(f); }

extern "C" size_t sdfb200_nerf_field_packed_bytes(const sdfb200_nerf_field_t* f) {
  return nerf::in_family(f) ? nerf::packed_bytes(nerf::planes_of(f)) : 0;
}

extern "C" int sdfb200_nerf_field_pack(const sdfb200_nerf_field_t* f, const float* const* weights, const float* const* biases, void* packed, void* stream) {
  using namespace nerf;
  SDFB_REQUIRE(f != nullptr, "NULL descriptor");
  if (!in_family(f)) return fail(SDFB200_EUNSUPPORTED, "nerf field: descriptor outside the fused kernel's family%s", "", 0);
  SDFB_REQUIRE(weights && biases && packed, "NULL pointer");
  for (int i = 0; i < kLayers + 2; ++i) SDFB_REQUIRE(weights[i] && biases[i], "NULL weight or bias");
  SDFB_REQUIRE(((uintptr_t)packed & 15) == 0, "packed must be 16-byte aligned");
  const int P = planes_of(f);
  const int pe = 6 * f->pe_frequencies + 3 * f->pe_include_input, dir = 6 * f->dir_frequencies + 3 * f->dir_include_input;
  cudaStream_t st = (cudaStream_t)stream;
  char* blob = (char*)packed;
  float* prm = (float*)blob;
  SDFB_CUDA(cudaMemsetAsync(blob, 0, kBlobWOff, st));
  auto copy = [&](int dst, const float* src, int n) { return cudaMemcpyAsync(prm + dst, src, (size_t)n * 4, cudaMemcpyDeviceToDevice, st); };
  for (int L = 0; L < kBase; ++L) SDFB_CUDA(copy(PRM_B_BASE + L * kWidth, biases[L], kWidth));
  for (int H = 0; H < 2; ++H) SDFB_CUDA(copy(PRM_B_HEAD + H * kHeadWidth, biases[kBase + H], kHeadWidth));
  SDFB_CUDA(copy(PRM_W_D, weights[kLayers], kWidth));
  SDFB_CUDA(copy(PRM_B_D, biases[kLayers], 1));
  SDFB_CUDA(copy(PRM_W_RGB, weights[kLayers + 1], 3 * kHeadWidth));
  SDFB_CUDA(copy(PRM_B_RGB, biases[kLayers + 1], 3));
  // block b of the stream at blob + kBlobWOff + b * stage; a layer whose input is cat([encoding, h]) is packed in two parts, the encoding's
  // columns zero padded to 64
  auto pack = [&](int L, int first, const float* W, int ldw, int N, int K, int nblocks) {
    const int np = L < kBase ? kWidth : kHeadWidth;
    return tc_pack(W, ldw, 0, N, K, np, kKB * kWidth / np, nblocks, P, nullptr, nullptr,
                   blob + kBlobWOff + (size_t)(layer_first_block(L) + first) * stage_bytes(P), st);
  };
  int r;
  for (int L = 0; L < kBase; ++L) {
    if (L == 0) r = pack(0, 0, weights[0], pe, kWidth, pe, 4);
    else if (L == kSkip) {
      r = pack(L, 0, weights[L], pe + kWidth, kWidth, pe, 4);
      if (!r) r = pack(L, 4, weights[L] + pe, pe + kWidth, kWidth, kWidth, 16);
    } else r = pack(L, 0, weights[L], kWidth, kWidth, kWidth, 16);
    if (r) return r;
  }
  r = pack(kBase, 0, weights[kBase], dir + kWidth, kHeadWidth, dir, 2);
  if (!r) r = pack(kBase, 2, weights[kBase] + dir, dir + kWidth, kHeadWidth, kWidth, 8);
  if (!r) r = pack(kBase + 1, 0, weights[kBase + 1], kHeadWidth, kHeadWidth, kHeadWidth, 4);
  return r;
}

extern "C" int sdfb200_nerf_field_forward(const sdfb200_nerf_field_t* f, const void* packed, const float* origins, const float* directions, const float* bins,
                                          int64_t n_rows, float* density, float* rgb, void* stream) {
  using namespace nerf;
  SDFB_REQUIRE(f != nullptr, "NULL descriptor");
  if (!in_family(f)) return fail(SDFB200_EUNSUPPORTED, "nerf field: descriptor outside the fused kernel's family%s", "", 0);
  SDFB_REQUIRE(f->n_samples >= 0 && n_rows >= 0, "bad sizes");
  const int64_t n = f->n_samples ? n_rows * f->n_samples : n_rows;
  if (n == 0) return 0;
  SDFB_REQUIRE(packed && origins && directions && density && rgb, "NULL pointer");
  SDFB_REQUIRE(f->n_samples == 0 || bins != nullptr, "ray mode needs bins");
  SDFB_REQUIRE(((uintptr_t)packed & 15) == 0, "packed must be 16-byte aligned");
  NfArgs a;
  a.blob = (const char*)packed;
  a.origins = origins; a.directions = directions; a.bins = f->n_samples ? bins : nullptr;
  a.density = density; a.rgb = rgb;
  a.n = n; a.S = f->n_samples; a.contraction = f->contraction; a.n_tiles = (int)ceil_div(n, 128);
  a.pe_f = f->pe_frequencies; a.pe_inc = f->pe_include_input; a.dir_f = f->dir_frequencies; a.dir_inc = f->dir_include_input;
  for (int k = 0; k < SDFB200_NERF_MAX_FREQS; ++k) { a.pe_freq[k] = f->pe_freqs[k]; a.dir_freq[k] = f->dir_freqs[k]; }
  cudaStream_t st = (cudaStream_t)stream;
  return planes_of(f) == 1 ? launch<1>(a, st) : launch<2>(a, st);
}
