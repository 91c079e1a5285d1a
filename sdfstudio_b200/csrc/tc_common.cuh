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
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// many-thread wait: back off between polls so the spinning warps do not eat the issue slots of the MMA / producer warps
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) __nanosleep(40);
}

// ---- 1-D bulk async copy global -> shared (completes on an mbarrier with complete_tx) -----------------------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// make generic-proxy writes to shared memory visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

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

// ---- streaming (evict_first) global accesses for the per-CTA scratch ------------------------------------------------
__device__ __forceinline__ void st_stream(void* p, uint4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_stream(void* p, float4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_stream(float* p, float v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ uint4 ld_stream_u4(const void* p, uint64_t pol) {
  uint4 v;
  asm volatile("ld.global.L2::cache_hint.v4.b32 {%0, %1, %2, %3}, [%4], %5;" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol) : "memory");
  return v;
}
__device__ __forceinline__ float ld_stream_f1(const float* p, uint64_t pol) {
  float v;
  asm volatile("ld.global.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol) : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_stream_f4(const void* p, uint64_t pol) {
  float4 v;
  asm volatile("ld.global.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol) : "memory");
  return v;
}

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
__device__ __forceinline__ float bf16lo_to_f32(uint32_t packed) { return __uint_as_float(packed << 16); }
__device__ __forceinline__ float bf16hi_to_f32(uint32_t packed) { return __uint_as_float(packed & 0xFFFF0000u); }

}  // namespace tc
}  // namespace sdfb200
