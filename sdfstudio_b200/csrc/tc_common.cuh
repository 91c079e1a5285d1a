// sm_90a primitives of the tensor-core kernels: mbarrier, 1-D bulk async copy (TMA engine), wgmma (warpgroup MMA with the
// accumulator in registers, A from shared memory or registers, B from shared memory) and its shared-memory descriptors.
//
// Operand layout convention (A in smem and B): the canonical K-major NO-SWIZZLE layout
//     element (row r, k)  ->  byte  (k/8) * LBO + (r/8) * SBO + (r%8) * 16 + (k%8) * 2        (bf16)
// with SBO = 128 (8 rows x 16 B, i.e. rows are consecutive 16-byte units) and LBO = rows * 16.
// So a tile is stored as [k-chunk of 8][row][8 bf16]; advancing one MMA K step (16) moves the start by 2*LBO, advancing 64 rows
// (one m64 / n64 block) moves it by 1024 bytes.  Weights are pre-packed in global memory in exactly this order, so a stage is
// filled by one 1-D bulk copy.
#pragma once
#include "common.cuh"

namespace sdfb200 {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// adds the cycles it spent waiting to *waited in the timing build of the fused kernel (tools/tc_timing.py)
#ifdef SDFB200_TC_TIMING
#define TC_CLOCK() clock64()
#else
#define TC_CLOCK() 0ll
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, long long* waited = nullptr) {
  const long long w0 = TC_CLOCK();
  while (!mbar_try_wait(bar, parity)) {
  }
  if (waited) *waited += TC_CLOCK() - w0;
}

// ---- 1-D bulk async copy global -> shared (completes on an mbarrier with complete_tx) -----------------------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// make generic-proxy writes to shared memory visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// the same for generic-proxy writes to global memory that a later bulk copy reads
__device__ __forceinline__ void fence_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// ---- wgmma (warpgroup MMA, sm_90a) -------------------------------------------------------------------------------
// All 128 threads of a warpgroup issue these together.  The accumulator lives in registers; for m64nN thread t of the warpgroup
// holds rows 16 (t/32) + (t%32)/4 (+8) and, per 8-column block j, columns 8 j + 2 (t%4) (+1):
//     d[4 j + 2 h + e]  =  D(row 16 (t/32) + (t%32)/4 + 8 h, column 8 j + 2 (t%4) + e)
__device__ __forceinline__ void wg_arrive() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs (cute::warpgroup_fence_operand)
template <int R>
__device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 64] += A[smem desc, 64 x 16] * B[smem desc, 64 x 16]^T   (bf16 x bf16 -> fp32, both K-major)
__device__ __forceinline__ void wgmma64_ss(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc), "r"(1)
      : "memory");
}
// D[64 x 64] += A[registers, 64 x 16] * B[smem desc, 64 x 16]^T.  a: the m16n8k16-style fragment of the thread's rows
// (a[0] = (r, 2c..2c+1), a[1] = (r+8, 2c..), a[2] = (r, 2c+8..), a[3] = (r+8, 2c+8..), r = 16 (t/32) + (t%32)/4, c = t%4)
__device__ __forceinline__ void wgmma64_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1)
      : "memory");
}

// D[64 x N] += A[smem desc, 64 x 16] * B[smem desc, N x 16]^T for N = 128 / 256: one instruction reads A once for all N columns
__device__ __forceinline__ void wgmma128_ss(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(1)
      : "memory");
}
__device__ __forceinline__ void wgmma256_ss(float (&d)[128], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\twgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a_desc), "l"(b_desc), "r"(1)
      : "memory");
}

// ---- descriptors -------------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor, K-major, no swizzle (layout type 0): LBO = byte distance between the two 8 x 16-byte core
// matrices of one K step (K direction), SBO = byte distance between 8-row groups (M / N direction)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;                // base_offset = 0, layout_type = SWIZZLE_NONE (0)
}

// one K step (16) of a 64-row warpgroup tile against NCH 64-row blocks of B, bf16 (P = 1) or bf16x3 (P = 2: a0 w0 + a1 w0 + a0 w1):
// a0 / a1 = descriptors of the A planes, b_addr = shared address of plane 0 of B at this K step, b_plane = byte distance of plane 1,
// lbo_b = B's K-direction core-matrix stride.  Only the first nch (<= NCH, warp-uniform) blocks are issued.
template <int P, int NCH>
__device__ __forceinline__ void wgmma_kstep_ss(float (&acc)[NCH][32], uint64_t a0, uint64_t a1, uint32_t b_addr, uint32_t b_plane, uint32_t lbo_b, int nch) {
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    if (c < nch) {
      const uint64_t b0 = make_smem_desc(b_addr + c * 1024, lbo_b, 128);
      wgmma64_ss(acc[c], a0, b0);
      if (P > 1) {
        wgmma64_ss(acc[c], a1, b0);
        wgmma64_ss(acc[c], a0, make_smem_desc(b_addr + b_plane + c * 1024, lbo_b, 128));
      }
    }
  }
}

// the same K step against all N = 128 / 256 rows of B at once: acc is the m64nN fragment, i.e. wgmma_kstep_ss's acc[N / 64][32]
// flattened, and every element sees the same products in the same order
template <int P, int N>
__device__ __forceinline__ void wgmma_kstep_wide_ss(float (&acc)[N / 2], uint64_t a0, uint64_t a1, uint32_t b_addr, uint32_t b_plane, uint32_t lbo_b) {
  static_assert(N == 128 || N == 256, "wide wgmma: N = 128 or 256");
  const uint64_t b0 = make_smem_desc(b_addr, lbo_b, 128);
  if constexpr (N == 256) {
    wgmma256_ss(acc, a0, b0);
    if (P > 1) { wgmma256_ss(acc, a1, b0); wgmma256_ss(acc, a0, make_smem_desc(b_addr + b_plane, lbo_b, 128)); }
  } else {
    wgmma128_ss(acc, a0, b0);
    if (P > 1) { wgmma128_ss(acc, a1, b0); wgmma128_ss(acc, a0, make_smem_desc(b_addr + b_plane, lbo_b, 128)); }
  }
}

// per-warpgroup register budget of a warp-specialised kernel (all warps of the warpgroup execute it)
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// ---- bf16 split helpers ------------------------------------------------------------------------------------------
// x = hi + lo (+ O(2^-17 |x|)) with hi, lo bf16.  pack2 packs two bf16 (first element in the low half).
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = pack_bf16x2(a, b);
  const float ah = __uint_as_float(hi << 16), bh = __uint_as_float(hi & 0xFFFF0000u);
  lo = pack_bf16x2(a - ah, b - bh);
}

// ---- A operand in shared memory: [plane][k/8][128 rows][8 bf16], `plane` bytes apart ------------------------------------
constexpr uint32_t kAChunk = 128 * 16;   // one 8-column chunk of a 128-row plane (the descriptor's LBO)
// byte offset of element (row, col) inside one plane
__device__ __forceinline__ uint32_t a_off(int row, int col) { return (uint32_t)(col >> 3) * kAChunk + (uint32_t)row * 16u + (uint32_t)(col & 7) * 2u; }
// one element, split into P bf16 planes
template <int P>
__device__ __forceinline__ void store_a(uint8_t* a, uint32_t plane, int row, int col, float v) {
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  const uint32_t off = a_off(row, col);
  *reinterpret_cast<__nv_bfloat16*>(a + off) = hi;
  if (P > 1) *reinterpret_cast<__nv_bfloat16*>(a + plane + off) = __float2bfloat16_rn(v - __bfloat162float(hi));
}
// two adjacent columns (an accumulator element pair): one 4-byte unit per plane, already split
template <int P>
__device__ __forceinline__ void store_a_pair(uint8_t* a, uint32_t plane, int row, int col, uint32_t hi, uint32_t lo) {
  const uint32_t off = a_off(row, col);
  *reinterpret_cast<uint32_t*>(a + off) = hi;
  if (P > 1) *reinterpret_cast<uint32_t*>(a + plane + off) = lo;
}
template <int P>
__device__ __forceinline__ void store_a_pair(uint8_t* a, uint32_t plane, int row, int col, float v0, float v1) {
  uint32_t hi, lo;
  split2(v0, v1, hi, lo);
  store_a_pair<P>(a, plane, row, col, hi, lo);
}
// one 16-byte chunk (8 consecutive columns of one row), already split
template <int P>
__device__ __forceinline__ void store_a_chunk(uint8_t* a, uint32_t plane, int row, int chunk, uint4 hi, uint4 lo) {
  *reinterpret_cast<uint4*>(a + (size_t)chunk * kAChunk + row * 16) = hi;
  if (P > 1) *reinterpret_cast<uint4*>(a + plane + (size_t)chunk * kAChunk + row * 16) = lo;
}
template <int P>
__device__ __forceinline__ void store_a_chunk(uint8_t* a, uint32_t plane, int row, int chunk, const float (&v)[8]) {
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) split2(v[2 * e], v[2 * e + 1], hi[e], lo[e]);
  store_a_chunk<P>(a, plane, row, chunk, make_uint4(hi[0], hi[1], hi[2], hi[3]), make_uint4(lo[0], lo[1], lo[2], lo[3]));
}
// descriptor of one plane of a warpgroup's 64 rows (shared address `base`) at MMA K step `kstep`
__device__ __forceinline__ uint64_t a_desc(uint32_t base, int kstep) { return make_smem_desc(base + kstep * 2 * kAChunk, kAChunk, 128); }

// ---- accumulator fragment ---------------------------------------------------------------------------------------
// Thread t of the warpgroup whose 64 rows start at row0 holds rows r0 = frag_row0(row0, t) and r0 + 8 and, in every 8-column block,
// columns cq = frag_cq(t) and cq + 1.  Element i of n64 block c (the layout next to wgmma64_ss) sits at (frag_row(r0, i), frag_col(cq, c, i)).
__device__ __forceinline__ int frag_row0(int row0, int t) { return row0 + (t >> 5) * 16 + ((t & 31) >> 2); }
__device__ __forceinline__ int frag_cq(int t) { return (t & 3) * 2; }
__device__ __forceinline__ int frag_half(int i) { return (i >> 1) & 1; }   // element i is in row r0 (0) or r0 + 8 (1)
template <typename T>   // int, or long long for a global row index
__device__ __forceinline__ T frag_row(T r0, int i) { return r0 + 8 * frag_half(i); }
__device__ __forceinline__ int frag_col(int cq, int c, int i) { return c * 64 + (i >> 2) * 8 + cq + (i & 1); }

// sum over the four threads of a quad (the threads that share accumulator rows), in a fixed order: + lane ^ 1, then + lane ^ 2
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// ---- hand-off between roles -------------------------------------------------------------------------------------
// S slots with a full / empty mbarrier pair each (arrival counts set by the kernel); use n of the stream takes slot n % S.  The producing
// role waits for empty, fills the slot and arrives on full (or hands full to bulk copies); the consuming role waits for full and arrives
// on empty.  Both wait for phase (n / S) & 1, the producer with the other parity, so its first wait passes (a fresh barrier counts as
// having completed the phase before its first).
template <int S>
struct Handoff {
  uint64_t full[S], empty[S];
  __device__ __forceinline__ void init(uint32_t full_count, uint32_t empty_count) {
    for (int s = 0; s < S; ++s) { mbar_init(&full[s], full_count); mbar_init(&empty[s], empty_count); }
  }
  __device__ __forceinline__ static uint32_t slot(uint32_t n) { return n % S; }
  __device__ __forceinline__ static uint32_t phase(uint32_t n) { return (n / S) & 1; }
  __device__ __forceinline__ uint64_t* full_bar(uint32_t n) { return &full[slot(n)]; }
  __device__ __forceinline__ void wait_empty(uint32_t n, long long* waited = nullptr) { mbar_wait(&empty[slot(n)], phase(n) ^ 1, waited); }
  __device__ __forceinline__ void wait_full(uint32_t n, long long* waited = nullptr) { mbar_wait(&full[slot(n)], phase(n), waited); }
  __device__ __forceinline__ void arrive_full(uint32_t n) { mbar_arrive(&full[slot(n)]); }
  __device__ __forceinline__ void arrive_empty(uint32_t n) { mbar_arrive(&empty[slot(n)]); }
};

// ---- weight ring ------------------------------------------------------------------------------------------------
// S stages of `bytes` each at `ring`, handed off by h (full count 1); consumers take block j with wait_full(j), release it with arrive_empty(j).
// producer (one thread): once the slot of stream block j has been released, copy block kb of the packed image `blocks` into it
template <int S>
__device__ __forceinline__ void ring_fill(Handoff<S>& h, uint8_t* ring, uint32_t j, const uint8_t* blocks, int kb, uint32_t bytes,
                                          long long* waited = nullptr) {
  h.wait_empty(j, waited);
  mbar_arrive_expect_tx(h.full_bar(j), bytes);
  bulk_g2s(ring + (size_t)h.slot(j) * bytes, blocks + (size_t)kb * bytes, bytes, h.full_bar(j));
}

// ---- fast softplus_100 ------------------------------------------------------------------------------------------
// softplus_100 and its derivative through MUFU ex2 / lg2 / rcp: ~10 instructions instead of the ~100 of log1pf(expf(.)).  t = 100 z.
// Absolute error ~1e-7 on h (the quantity that feeds the next layer), i.e. at the level of fp32 rounding of the reference's own
// log1p(exp(.)).
__device__ __forceinline__ float fast_ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float fast_lg2(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float fast_rcp(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ void softplus100_fast(float z, float& h, float& dsig) {
  // exp(100 z) = 2^(z * 100 log2 e); log1p(e)/100 = lg2(1+e) * ln2/100.  For small e, 1+e rounds e to ~6e-8 absolute, i.e. an
  // absolute error of ~4e-10 on h: irrelevant next to the bf16x3 operand rounding (2^-17 relative).
  const float e = fast_ex2(fminf(z, 0.3f) * 144.26950408889634f);
  const float u = 1.0f + e;
  const bool lin = z > 0.2f;                                            // PyTorch's softplus threshold: beta*x > 20
  h = lin ? z : fast_lg2(u) * 0.006931471805599453f;
  dsig = lin ? 1.0f : e * fast_rcp(u);
}
__device__ __forceinline__ float softplus100_fast(float z) {
  float h, dsig;
  softplus100_fast(z, h, dsig);
  return h;
}
// softplus_100'(z) from h = softplus_100(z):  sigma(100 z) = 1 - exp(-100 h)
__device__ __forceinline__ float dsoftplus100_fast_from_h(float h) { return 1.0f - fast_ex2(h * -144.26950408889634f); }

}  // namespace tc
}  // namespace sdfb200
