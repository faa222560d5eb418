// Thin inline-PTX wrappers for sm_90a: mbarrier, cp.async, TMA, clusters, wgmma, proxy fences.
// Hand-written for this repo; encodings follow the PTX ISA for sm_90a (see DESIGN.md section 2).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace cis {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------- cp.async (LDGSTS)
// 16-byte global->shared copy; src_bytes = 0 zero-fills the destination (used for SAME padding / ragged tails).
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// Asynchronous arrival: the mbarrier receives one arrive (not counted as pending) when ALL prior cp.async of this thread
// have landed -- no wait_group, the producer keeps running ahead.
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- TMA (bulk tensor) for the weight operand
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// 4-D tiled TMA load (tensor map in param/global space); coordinates may be negative / out of range => zero fill (= SAME padding).
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// 1-D bulk copy global -> shared through the TMA engine; completion = complete_tx(bytes) on the mbarrier.
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes),
               "r"(bar)
               : "memory");
}
// ---------------------------------------------------------------- thread-block clusters (split-K reduction through distributed shared memory)
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {   // every thread of every CTA of the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cta address of this CTA -> the same offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t dsmem_addr(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
__device__ __forceinline__ float4 dsmem_ld4(uint32_t caddr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(caddr) : "memory");
  return v;
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

// Programmatic dependent launch: let the next kernel of the stream start its prologue while this grid drains, and wait for the
// previous grid's memory before touching anything it produced.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------- per-warpgroup register budgets
// Every thread of the warpgroup executes the same setmaxnreg at a converged point.  .dec returns registers to the CTA's pool; .inc waits
// until the pool has them, so the counts of all warpgroups of a CTA must add up to no more than what it was launched with (a CTA of T
// threads compiled to R registers owns T * R).  R: a multiple of 8 in [24, 256].  Between two setmaxnreg the warps of the warpgroup
// must synchronise explicitly (named_bar_sync over the warpgroup).
template <int ID, int N>
__device__ __forceinline__ void named_bar_sync() {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory");
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}

// ---------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// A warpgroup = 4 consecutive warps starting at a warp index that is a multiple of 4; all 128 threads issue every wgmma.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D(64 x N, fp32 registers) (+)= A[smem desc] * B[smem desc], bf16 inputs; TA / TB = 1 selects an MN-major operand.
template <int N, int TA, int TB> struct Wgmma;
template <int TA, int TB> struct Wgmma<16, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
  }
};
template <int TA, int TB> struct Wgmma<32, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
  }
};
template <int TA, int TB> struct Wgmma<64, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
  }
};
template <int TA, int TB> struct Wgmma<128, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
  }
};

// ---------------------------------------------------------------- shared-memory matrix descriptors
// 64-bit descriptor: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | base_offset [49,52) = 0 | layout [62,64) (1 = SWIZZLE_128B).
// The 128B swizzle is a function of the absolute shared-memory address bits, so starts at any 16-byte (K steps) or 128-byte (rows,
// halo taps) offset from a 1024-aligned, swizzle-written tile keep base_offset = 0.
// Split form for hot issue loops: hi word is loop-invariant, lo word = start>>4 | LBO>>4<<16 advances by (bytes>>4) per K step.
__device__ __forceinline__ uint32_t desc_hi(uint32_t sbo_bytes) { return ((sbo_bytes >> 4) & 0x3FFF) | (1u << 30); }
// no-swizzle K-major layout (layout = 0): core matrices of 8 rows x 16 contiguous bytes; LBO = next core matrix along K, SBO = next 8 rows
__device__ __forceinline__ uint32_t desc_hi_ns(uint32_t sbo_bytes) { return (sbo_bytes >> 4) & 0x3FFF; }
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr, uint32_t lbo_bytes) {
  return ((saddr & 0x3FFFF) >> 4) | (((lbo_bytes >> 4) & 0x3FFF) << 16);
}

// One 128 x N x 16 MMA of the warpgroup: two m64 wgmma (rows 0-63 -> acc[0, N/2), rows 64-127 -> acc[N/2, N)).  a_half = descriptor
// start-field step from row 0 to row 64 of A (K-major: 8 core-matrix groups = 8 * SBO; MN-major: one 64-element atom = LBO).
template <int N, int TA, int TB>
__device__ __forceinline__ void mma128(float (&acc)[N], uint32_t alo, uint32_t ahi, uint32_t blo, uint32_t bhi, uint32_t a_half,
                                       uint32_t scale_d) {
  const uint64_t db = ((uint64_t)bhi << 32) | blo;
  Wgmma<N, TA, TB>::mma(*reinterpret_cast<float(*)[N / 2]>(&acc[0]), ((uint64_t)ahi << 32) | alo, db, scale_d);
  Wgmma<N, TA, TB>::mma(*reinterpret_cast<float(*)[N / 2]>(&acc[N / 2]), ((uint64_t)ahi << 32) | (alo + a_half), db, scale_d);
}

// ---------------------------------------------------------------- accumulator tiles in shared memory
// The warpgroup hands its finished 128-row fp32 accumulator to the epilogue warps through shared memory, stored as float4 COLUMNS:
// element (row, col) at ((col / 4) * 128 + row) * 16 + (col % 4) * 4 bytes, i.e. column c (a multiple of 4) starts c * 512 bytes
// after column 0.  A thread that owns one row then reads 16 columns as 4 x LDS.128 and a warp (32 consecutive rows) reads 512
// contiguous bytes per instruction.  This is also the layout the cluster split-K reduction reads through DSMEM.
static constexpr uint32_t kAccColBytes = 512;
// this thread's fragment of a 128 x N accumulator (wgmma layout) -> the tile at `base`
template <int N>
__device__ __forceinline__ void acc_store(const float (&acc)[N], uint32_t base, int wtid) {
  const int w = wtid >> 5, lane = wtid & 31;
  const int c2 = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = 64 * h + 16 * w + (lane >> 2);
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
      const int col = 8 * i + c2;
      const uint32_t a = base + (uint32_t)((col >> 2) * 2048 + row * 16 + (col & 3) * 4);
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(acc[h * (N / 2) + 4 * i]), "f"(acc[h * (N / 2) + 4 * i + 1]) : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a + 8 * 16), "f"(acc[h * (N / 2) + 4 * i + 2]), "f"(acc[h * (N / 2) + 4 * i + 3])
                   : "memory");
    }
  }
}
// 16 consecutive columns of one row; addr = tile + row * 16 + c0 * kAccColBytes (c0 a multiple of 4)
__device__ __forceinline__ void acc_ld16(uint32_t addr, float* v) {
#pragma unroll
  for (int h = 0; h < 4; ++h)
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v[4 * h]), "=f"(v[4 * h + 1]), "=f"(v[4 * h + 2]), "=f"(v[4 * h + 3])
                 : "r"(addr + (uint32_t)h * 2048)
                 : "memory");
}

// ---------------------------------------------------------------- small helpers
__device__ __forceinline__ float bf16lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16hi(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

}  // namespace cis
