// wgmma implicit-GEMM convolution engine for sm_90a (forward / data-gradient / transposed conv / weight-gradient).
//
// Replaces the TF1 op classes K1/K3/K5/K6 of SURVEY.md section 2.2 (tf.layers.conv2d, tf.nn.conv2d,
// tf.layers.conv2d_transpose and their tf.gradients twins; reference call sites
// models/utils/convolution_utils.py:46,81 and models/PWCNet/model_pwcnet.py:161-165,286,484-504,562-574).
//
// Design (see DESIGN.md): one CTA = one 128-row tile of the GEMM (rows = output pixels).  Four producer warps gather the
// im2col A tile (128 rows x 64 bf16 of K) and the packed-weight B tile straight into the canonical SWIZZLE_128B K-major
// shared-memory layout with 16-byte cp.async (zero-fill = SAME padding); an MMA warpgroup issues wgmma (two m64nBNk16 per
// 128-row K=16 step) with the fp32 accumulator in its registers and releases each smem stage through an mbarrier once its
// wgmma group has completed.  After the last K block it stores the accumulator to shared memory (acc_store) and the producer
// warps become the epilogue: read the accumulator rows, apply bias / residuals / activation and store bf16 and/or fp32 NHWC.
#include "ptx.cuh"
#include "../../include/cis_b200.h"
#include "common.cuh"
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

// cp.async (LDGSTS) writes shared memory through the generic proxy while wgmma reads it through the async proxy.  Every
// cp.async producer therefore publishes a stage itself: commit_group, wait_group<lag> (its own copies of the stage landed),
// fence.proxy.async, then a plain mbarrier.arrive -- the MMA warp needs no fence.  The lag keeps (stages - 1) groups in flight.

namespace cis {

// Developer-only pipeline trace (make trace -> libcis_b200_trace.so, tools/trace_conv.py): CTA (0,0,0) records SM-clock stamps of its
// MMA-issue loop so per-step wait / issue time can be read back.  Compiled out of the product library.
#ifdef CIS_TRACE
__device__ unsigned long long* g_trace = nullptr;
__device__ int g_trace_cap = 0;
#define CIS_TRACE_AT(slot)                                                                                         \
  do {                                                                                                             \
    if (g_trace && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && (slot) < g_trace_cap) g_trace[(slot)] = clock64(); \
  } while (0)
#else
#define CIS_TRACE_AT(slot) ((void)0)
#endif

static constexpr int kBM = 128;       // GEMM rows per CTA
static constexpr int kBK = 64;        // bf16 K elements per stage (128-byte swizzled rows)
static constexpr int kAStage = kBM * 128;
static constexpr int kThreads = 256;  // halo / wgrad kernels: 4 producer/epilogue warps + 1 MMA warpgroup
// conv_halo_kernel<BN, NWG>: warps 0-3 producers + epilogue, then NWG MMA warpgroups (warps 4-7, 4-11).
//   NWG = 1: 256 threads, two CTAs per SM (128 registers per thread), so one CTA's prologue and epilogue overlap the other's main
//   loop.  The producer warpgroup hands registers to the MMA warpgroup for the main loop (setmaxnreg: kProdRegs / kMmaRegs; 128
//   accumulator columns need ~168) and both return to kLaunchRegs for the epilogue.  BN >= 64: the MMA warps join the epilogue once
//   their accumulators are in shared memory (the wide epilogue is instruction-bound on its warps).
//   NWG = 2 (BN >= 64): two MMA warpgroups (warps 4-11) consume every weight stage, so each weight byte fetched from L2 feeds twice
//   the output rows; 384 threads, one CTA per SM (the 168-register budget of one warpgroup's 128 accumulator columns), the MMA warps
//   join the epilogue.
template <int BN, int NWG> struct HaloCfg {
  static_assert(NWG == 1 || (NWG == 2 && BN >= 64), "two MMA warpgroups only for BN >= 64");
  static constexpr int kMmaWarp = 4;                                   // first warp of the first MMA warpgroup
  static constexpr int kThreads = (kMmaWarp + 4 * NWG) * 32;
  static constexpr int kEpiWarps = (NWG == 1 && BN < 64) ? kMmaWarp : kThreads / 32;   // warps 0 .. kEpiWarps-1 run the epilogue
  static constexpr int kEpiParts = NWG == 1 ? (BN >= 64 ? 2 : 1) : BN / 32;   // column parts of a 32-row epilogue unit
  // accumulator registers per MMA thread: MT * BN <= kMaxAccCols (the host never stacks more tiles than that)
  static constexpr int kMaxMT = (128 / BN) < 4 ? (128 / BN) : 4;
  static constexpr int kCtasPerSm = NWG == 1 ? 2 : 1;
  static constexpr int kLaunchRegs = (65536 / (kCtasPerSm * kThreads)) & ~7;   // registers per thread under the launch bounds
  // main-loop budgets of the producer and MMA warpgroups (0: no setmaxnreg; BN = 16 holds its 64 accumulator columns in kLaunchRegs)
  static constexpr int kProdRegs = (NWG == 1 && BN >= 32) ? 88 : 0;
  static constexpr int kMmaRegs = (NWG == 1 && BN >= 32) ? 168 : 0;
  static_assert(kProdRegs == 0 || 128 * (kProdRegs + NWG * kMmaRegs) <= kThreads * kLaunchRegs,
                "setmaxnreg.inc would wait for registers the CTA does not own");
};
static constexpr int kMaxAccCols = 128;   // fp32 accumulator columns one MMA warpgroup holds in registers (128 per thread)
static constexpr int kGProducers = 256;   // gather kernel: 8 producer/epilogue warps (its cp.async address arithmetic is the bottleneck)
static constexpr int kGThreads = 384;     // + 1 MMA warpgroup

struct SrcS {
  const __nv_bfloat16* ptr;
  int pitch, c_off, chunks, n_mod;
};


// One 16-column chunk of the fused epilogue: bias -> (+bf16 accumulate | +fp32 residual) -> activation -> (+skip) -> stores.
__device__ __forceinline__ void epi_chunk(const CisConv& p, float (&v)[16], const int cg, const size_t dpix) {
  if (p.bias) {
#pragma unroll
    for (int e = 0; e < 16; ++e) v[e] += __ldg(p.bias + cg + e);
  }
  if (p.add_pre && cg < p.out_ch) {
    const uint4* a = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.add_pre) + dpix * p.add_pre_pitch +
                                                    p.add_pre_coff + cg);
    const int nv = (p.out_ch - cg >= 16) ? 2 : 1;
    for (int h2 = 0; h2 < nv; ++h2) {
      const uint4 u = __ldg(a + h2);
      const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        v[h2 * 8 + 2 * e] += bf16lo(w4[e]);
        v[h2 * 8 + 2 * e + 1] += bf16hi(w4[e]);
      }
    }
  }
  if (p.addf_pre) {
    for (int e = 0; e < 16 && cg + e < p.outf_ch; ++e) v[e] += __ldg(p.addf_pre + dpix * p.addf_pitch + p.addf_coff + cg + e);
  }
  if (p.act == CIS_ACT_ELU) {
#pragma unroll
    for (int e = 0; e < 16; ++e) v[e] = v[e] > 0.f ? v[e] : expm1f(v[e]);
  } else if (p.act == CIS_ACT_LEAKY) {
#pragma unroll
    for (int e = 0; e < 16; ++e) v[e] = v[e] > 0.f ? v[e] : v[e] * p.alpha;
  }
  if (p.add_post && cg < p.out_ch) {
    const uint4* a = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.add_post) + dpix * p.add_post_pitch +
                                                    p.add_post_coff + cg);
    const int nv = (p.out_ch - cg >= 16) ? 2 : 1;
    for (int h2 = 0; h2 < nv; ++h2) {
      const uint4 u = __ldg(a + h2);
      const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        v[h2 * 8 + 2 * e] += bf16lo(w4[e]);
        v[h2 * 8 + 2 * e + 1] += bf16hi(w4[e]);
      }
    }
  }
  if (p.mode == 1) {
    if (cg == 0) p.outf[dpix] = 1.f / (1.f + __expf(-(v[0] - v[1]) * 0.1f));
    return;
  }
  if (p.out && cg < p.out_ch) {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + dpix * p.out_pitch + p.out_coff + cg;
    if (((p.out_ch | p.out_coff | p.out_pitch) & 7) == 0) {
      uint4 u0 = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
      *reinterpret_cast<uint4*>(o) = u0;
      if (p.out_ch - cg >= 16) {
        uint4 u1 = make_uint4(pack_bf16(v[8], v[9]), pack_bf16(v[10], v[11]), pack_bf16(v[12], v[13]), pack_bf16(v[14], v[15]));
        *reinterpret_cast<uint4*>(o + 8) = u1;
      }
    } else {
      for (int e = 0; e < 16 && cg + e < p.out_ch; ++e) o[e] = __float2bfloat16(v[e]);
    }
  }
  if (p.outf && cg < p.outf_ch) {
    float* o = p.outf + dpix * p.outf_pitch + p.outf_coff + cg;
    for (int e = 0; e < 16 && cg + e < p.outf_ch; ++e) o[e] = v[e];
  }
}



// Latency-batched epilogue for NC x 16 accumulator columns of one row: residual loads are issued first, then the accumulator reads,
// then the arithmetic and the stores.  taddr = accumulator tile + row * 16 + first column * kAccColBytes.
template <int NC>
__device__ __forceinline__ void epi_group(const CisConv& p, const uint32_t taddr, const int cg0, const size_t dpix, const bool valid,
                                          const float* __restrict__ sbias) {
  // one residual operand per launch: add_pre (gradient accumulation, before the activation) or add_post (skip, after it)
  uint4 rres[NC][2];
  const bool is_pre = p.add_pre != nullptr;
  const __nv_bfloat16* rp = reinterpret_cast<const __nv_bfloat16*>(is_pre ? p.add_pre : p.add_post);
  const bool has_res = valid && rp != nullptr;
  const size_t roff = has_res ? (dpix * (is_pre ? p.add_pre_pitch : p.add_post_pitch) + (is_pre ? p.add_pre_coff : p.add_post_coff)) : 0;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const int cg = cg0 + 16 * c;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      rres[c][h] = make_uint4(0, 0, 0, 0);
      if (has_res && cg + 8 * h < p.out_ch) rres[c][h] = __ldg(reinterpret_cast<const uint4*>(rp + roff + cg) + h);
    }
  }
  if (!valid) return;
  float raw[NC][16];
#pragma unroll
  for (int c = 0; c < NC; ++c) acc_ld16(taddr + (uint32_t)(16 * c) * kAccColBytes, raw[c]);
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const int cg = cg0 + 16 * c;
    float v[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) v[e] = raw[c][e];
    if (p.bias) {
      const float4* sb = reinterpret_cast<const float4*>(sbias + (cg - cg0));   // sbias = this group's first column; 16-float aligned: 4 x LDS.128
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 b4 = sb[q];
        v[4 * q] += b4.x; v[4 * q + 1] += b4.y; v[4 * q + 2] += b4.z; v[4 * q + 3] += b4.w;
      }
    }
    if (is_pre) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t w4[4] = {rres[c][h].x, rres[c][h].y, rres[c][h].z, rres[c][h].w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          v[h * 8 + 2 * e] += bf16lo(w4[e]);
          v[h * 8 + 2 * e + 1] += bf16hi(w4[e]);
        }
      }
    }
    if (p.addf_pre) {
      for (int e = 0; e < 16 && cg + e < p.outf_ch; ++e) v[e] += __ldg(p.addf_pre + dpix * p.addf_pitch + p.addf_coff + cg + e);
    }
    if (p.act == CIS_ACT_ELU) {
      // exp through MUFU.EX2 (4 instructions per element instead of the ~40 of expm1f): |error| <= ~1e-7 absolute, far below the
      // bf16 rounding of the stored activation; the epilogue runs on one warp per scheduler, so instruction count IS its time
#pragma unroll
      for (int e = 0; e < 16; ++e) v[e] = v[e] > 0.f ? v[e] : __expf(v[e]) - 1.f;
    } else if (p.act == CIS_ACT_LEAKY) {
#pragma unroll
      for (int e = 0; e < 16; ++e) v[e] = v[e] > 0.f ? v[e] : v[e] * p.alpha;
    }
    if (!is_pre) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t w4[4] = {rres[c][h].x, rres[c][h].y, rres[c][h].z, rres[c][h].w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          v[h * 8 + 2 * e] += bf16lo(w4[e]);
          v[h * 8 + 2 * e + 1] += bf16hi(w4[e]);
        }
      }
    }
    if (p.mode == 1) {
      if (cg == 0) p.outf[dpix] = 1.f / (1.f + __expf(-(v[0] - v[1]) * 0.1f));
      continue;
    }
    if (p.out && cg < p.out_ch) {
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + dpix * p.out_pitch + p.out_coff + cg;
      if (((p.out_ch | p.out_coff | p.out_pitch) & 7) == 0) {
        *reinterpret_cast<uint4*>(o) = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
        if (p.out_ch - cg >= 16)
          *reinterpret_cast<uint4*>(o + 8) =
              make_uint4(pack_bf16(v[8], v[9]), pack_bf16(v[10], v[11]), pack_bf16(v[12], v[13]), pack_bf16(v[14], v[15]));
      } else {
        for (int e = 0; e < 16 && cg + e < p.out_ch; ++e) o[e] = __float2bfloat16(v[e]);
      }
    }
    if (p.outf && cg < p.outf_ch) {
      float* o = p.outf + dpix * p.outf_pitch + p.outf_coff + cg;
      for (int e = 0; e < 16 && cg + e < p.outf_ch; ++e) o[e] = v[e];
    }
  }
}
// columns [c_lo, c_hi) of one row (multiples of 16), in groups of 32 columns (register budget); sbias: the BN columns of THIS n-tile
template <int BN>
__device__ __forceinline__ void epi_cols(const CisConv& p, const uint32_t t_row, const int cbase, const size_t dpix, const bool valid,
                                         const float* __restrict__ sbias, const int c_lo, const int c_hi) {
  int c0 = c_lo;
#pragma unroll 1
  for (; c0 + 32 <= c_hi; c0 += 32) epi_group<2>(p, t_row + (uint32_t)c0 * kAccColBytes, cbase + c0, dpix, valid, sbias + c0);
  if (c0 < c_hi) epi_group<1>(p, t_row + (uint32_t)c0 * kAccColBytes, cbase + c0, dpix, valid, sbias + c0);
}
// all BN columns of one row
template <int BN>
__device__ __forceinline__ void epi_row(const CisConv& p, const uint32_t t_row, const int cbase, const size_t dpix, const bool valid,
                                        const float* __restrict__ sbias) {
  epi_cols<BN>(p, t_row, cbase, dpix, valid, sbias, 0, BN);
}

// ---- split-K (two launches): every CTA of a tile stores its partial accumulator to a private fp32 slice; splitk_finish_kernel sums the
// slices in a fixed order and runs the fused epilogue.
template <int BN>
__device__ __forceinline__ void splitk_store_partial(float* slice, uint32_t t_row, int row, int c_lo = 0, int c_hi = BN) {
  // slice = this split's private fp32 tile, stored as float4 COLUMNS: element (row, c) at ((c / 4) * 128 + row) * 4 + c % 4.  A warp
  // (32 consecutive accumulator rows, same columns) then writes 512 contiguous bytes per store instruction; a row-major layout would
  // make every st.v4 touch 32 different 128-byte lines and the LSU, not HBM, would bound the epilogue.  No atomics, fixed summation
  // order later.
#pragma unroll 1
  for (int c0 = c_lo; c0 < c_hi; c0 += 16) {
    float v[16];
    acc_ld16(t_row + (uint32_t)c0 * kAccColBytes, v);
    float4* o = reinterpret_cast<float4*>(slice) + (size_t)(c0 / 4) * kBM + row;
    o[0] = make_float4(v[0], v[1], v[2], v[3]);
    o[kBM] = make_float4(v[4], v[5], v[6], v[7]);
    o[2 * kBM] = make_float4(v[8], v[9], v[10], v[11]);
    o[3 * kBM] = make_float4(v[12], v[13], v[14], v[15]);
  }
}
// sum of the nsplit private slices of one tile for (row, c0..c0+15); loads are plain L2 loads (__ldcg) issued in batches of
// 4 slices x 4 float4 so their latencies overlap (volatile-asm loads would serialise the round trips)
template <int BN>
__device__ __forceinline__ void splitk_reduce16(const float* tile0, int nsplit, int row, int c0, float* v) {
#pragma unroll
  for (int e = 0; e < 16; ++e) v[e] = 0.f;
  const float4* q0 = reinterpret_cast<const float4*>(tile0) + (size_t)(c0 / 4) * kBM + row;    // float4-column layout of splitk_store_partial
  const size_t zstride = (size_t)kBM * BN / 4;
  int z = 0;
  for (; z + 4 <= nsplit; z += 4) {
    float4 t[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int h = 0; h < 4; ++h) t[u][h] = __ldcg(q0 + (size_t)(z + u) * zstride + h * kBM);
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        v[4 * h] += t[u][h].x; v[4 * h + 1] += t[u][h].y; v[4 * h + 2] += t[u][h].z; v[4 * h + 3] += t[u][h].w;
      }
  }
  for (; z < nsplit; ++z) {
    float4 t[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) t[h] = __ldcg(q0 + (size_t)z * zstride + h * kBM);
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      v[4 * h] += t[h].x; v[4 * h + 1] += t[h].y; v[4 * h + 2] += t[h].z; v[4 * h + 3] += t[h].w;
    }
  }
}
// Cluster split-K: every CTA of the cluster has written its partial tile to its own shared memory as float4 columns
// stage[(c4 * 128 + row)] (conflict-free: lanes = consecutive rows).  CTA `rank` of `S` then owns accumulator rows
// [rank * rpc, (rank + 1) * rpc): it sums the S partials in rank order (deterministic) through DSMEM and runs the fused epilogue.
template <int BN, typename DPIX>
__device__ __forceinline__ void cluster_reduce_rows(const CisConv& p, const uint32_t stage, const int S, const int rank, const int tid,
                                                    const int nthreads, const int cbase, DPIX dpix_of) {
  const int rpc = (kBM + S - 1) / S;
  const int r0 = rank * rpc, r1 = min(kBM, r0 + rpc);
  constexpr int G16 = BN / 16;
  for (int it = tid; it < (r1 - r0) * G16; it += nthreads) {
    const int row = r0 + it / G16, c0 = (it % G16) * 16;
    float v[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) v[e] = 0.f;
    for (int q = 0; q < S; ++q) {
      const uint32_t base = dsmem_addr(stage, (uint32_t)q);
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const float4 t = dsmem_ld4(base + (uint32_t)(((c0 / 4 + h) * kBM + row) * 16));
        v[4 * h] += t.x; v[4 * h + 1] += t.y; v[4 * h + 2] += t.z; v[4 * h + 3] += t.w;
      }
    }
    bool valid;
    const size_t dpix = dpix_of(row, valid);
    if (valid) epi_chunk(p, v, cbase + c0, dpix);
  }
}

// CPS: co-resident CTAs per SM the registers allow.  CPS = 2 (80 registers per thread) up to BN = 64, where the producer warpgroups
// lend 8 registers per thread to the MMA warpgroup for the main loop (setmaxnreg; 0 = none).  BN = 128 (128 accumulator columns next
// to 8 gathering warps) and the one-per-SM BN = 64 instance (grids of at most one CTA per SM) are compiled for CPS = 1.
template <int BN, int CPS>
struct FwdCfg {
  // kLag + 1 K blocks of gathers are in flight per producer thread (the im2col loads are L2 round trips).  A deeper ring costs
  // co-resident CTAs on the thin layers.
  static constexpr int kStages = (BN == 128) ? 3 : 4;
  static constexpr int kLag = kStages - 2;
  static constexpr int kBStage = BN * 128;
  static constexpr int kSmem = kStages * (kAStage + kBStage) + 1024;
  static_assert(kStages * (kAStage + kBStage) >= kBM * BN * 4, "the accumulator tile reuses the operand ring");
  static_assert(CPS == 1 || BN <= 64, "128 accumulator columns do not fit two CTAs per SM");
  static constexpr int kLaunchRegs = (65536 / (CPS * kGThreads)) & ~7;
  static constexpr int kProdRegs = (BN == 64 && CPS == 2) ? 72 : 0;
  static constexpr int kMmaRegs = (BN == 64 && CPS == 2) ? 96 : 0;
  static_assert(kProdRegs == 0 || 128 * (kProdRegs * kGProducers / 128 + kMmaRegs) <= kGThreads * kLaunchRegs,
                "setmaxnreg.inc would wait for registers the CTA does not own");
};

// CPS = 1: no minimum CTA count in the launch bounds (ptxas then keeps its own register choice, 90 for BN = 64 instead of 118)
template <int BN, int CPS>
__global__ void __launch_bounds__(kGThreads, CPS == 1 ? 0 : CPS) conv_igemm_kernel(const __grid_constant__ CisConv p) {
  using Cfg = FwdCfg<BN, CPS>;
  constexpr int S = Cfg::kStages;
  constexpr int kMmaWarp = kGProducers / 32;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t bars[2 * S + 1];
  __shared__ int s_dh[CIS_MAX_TAPS], s_dw[CIS_MAX_TAPS];
  __shared__ SrcS s_src[CIS_MAX_SRC];

  const uint32_t tile_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = tile_base;
  const uint32_t b_base = tile_base + S * kAStage;
  const uint32_t bar_full = smem_u32(&bars[0]);
  const uint32_t bar_empty = smem_u32(&bars[S]);
  const uint32_t bar_accum = smem_u32(&bars[2 * S]);

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int M = p.N * p.OH * p.OW;
  const int m_chunks = [&] {
    int s = 0;
    for (int i = 0; i < p.nsrc; ++i) s += p.src[i].chunks;
    return s;
  }();
  const int nkb_all = p.K_pad / kBK;
  const int nsplit = p.splits > 1 ? p.splits : 1;
  const int kper = (nkb_all + nsplit - 1) / nsplit;
  const int kb_lo = blockIdx.z * kper;
  const int nkb = min(kper, nkb_all - kb_lo);     // host guarantees nkb >= 1 for every split
  const int ny = blockIdx.y;
  __shared__ __align__(16) float s_bias[BN];
  pdl_launch_dependents();

  if (tid < p.ntaps) {
    s_dh[tid] = p.dh[tid];
    s_dw[tid] = p.dw[tid];
  }
  if (tid < p.nsrc) {
    s_src[tid].ptr = reinterpret_cast<const __nv_bfloat16*>(p.src[tid].ptr);
    s_src[tid].pitch = p.src[tid].pitch;
    s_src[tid].c_off = p.src[tid].c_off;
    s_src[tid].chunks = p.src[tid].chunks;
    s_src[tid].n_mod = p.src[tid].n_mod;
  }
  if (tid == kMmaWarp * 32) {
    for (int s = 0; s < S; ++s) {
      mbar_init(bar_full + 8 * s, kGProducers);
      mbar_init(bar_empty + 8 * s, 1);
    }
    mbar_init(bar_accum, 128);    // every thread of the MMA warpgroup, after storing its accumulator fragment
    fence_mbar_init();
  }
  pdl_wait();   // everything above touched only kernel parameters / shared memory
  if (tid < BN) s_bias[tid] = p.bias ? p.bias[ny * BN + tid] : 0.f;
  __syncthreads();
  if (tid == 0) CIS_TRACE_AT(0);

  if (warp < kMmaWarp) {
    // ------------------------------------------------------------------ producers: thread = (16-byte K chunk j, rows rl + 32 i)
    const int j = tid & 7;          // 16-byte chunk within the 128-byte K row
    const int rl = tid >> 3;        // 0..31
    const uint32_t sw_off = (uint32_t)((j ^ (rl & 7)) << 4);
    // Per-row constants (this thread's 4 rows): top-left input pixel, and the linear pixel index of it in the plain and in the
    // batch-broadcast (n % n_mod) view of the sources.  The K loop below is division-free: with integer divisions / 64-bit address
    // arithmetic per (K block, row) the producer warps are issue-bound, not bound by the loads.
    if constexpr (Cfg::kProdRegs > 0) setmaxnreg_dec<Cfg::kProdRegs>();
    int hb[4], wb[4], pre[4], prem[4];
    int nm0 = 0;                          // the batch-broadcast modulus (sources with n_mod > 0 share one; others: slow path)
    for (int i = 0; i < p.nsrc; ++i)
      if (p.src[i].n_mod > 0 && nm0 == 0) nm0 = p.src[i].n_mod;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int g = blockIdx.x * kBM + rl + 32 * i;
      if (g < M) {
        const int ow = g % p.OW;
        const int t = g / p.OW;
        const int oh = t % p.OH;
        const int n = t / p.OH;
        hb[i] = oh * p.sh;
        wb[i] = ow * p.sw;
        pre[i] = (n * p.H + hb[i]) * p.W + wb[i];
        prem[i] = ((nm0 ? n % nm0 : n) * p.H + hb[i]) * p.W + wb[i];
      } else {
        hb[i] = -(1 << 20);
        wb[i] = 0;
        pre[i] = prem[i] = 0;
      }
    }
    const __nv_bfloat16* wrow = reinterpret_cast<const __nv_bfloat16*>(p.wpack) + (size_t)(ny * BN + rl) * p.K_pad + j * 8;
    // (tap, channel chunk) of this thread's K chunk, advanced by 8 chunks per K block without dividing
    const int adv_t = 8 / m_chunks, adv_c = 8 - adv_t * m_chunks;
    int t = (kb_lo * 8 + j) / m_chunks, c = (kb_lo * 8 + j) - t * m_chunks;

    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % S;
      const uint32_t ph = (uint32_t)((kb / S) & 1);
      mbar_wait(bar_empty + 8 * s, ph ^ 1u);
      // ---- A: this thread's K chunk -> (tap t, source si, channel chunk cs)
      const bool kvalid = t < p.ntaps;
      const int tt = kvalid ? t : 0;
      int si = 0, cs = c;
      while (si < p.nsrc - 1 && cs >= s_src[si].chunks) {
        cs -= s_src[si].chunks;
        ++si;
      }
      const __nv_bfloat16* sp = s_src[si].ptr;
      const int pitch = s_src[si].pitch;
      const int nmod = s_src[si].n_mod;
      const int dh = s_dh[tt], dw = s_dw[tt];
      const int toff = dh * p.W + dw;
      const __nv_bfloat16* spc = sp + s_src[si].c_off + cs * 8;
      const bool slow_mod = nmod != 0 && nmod != nm0;
      const uint32_t a_dst = a_base + s * kAStage + rl * 128 + sw_off;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int h = hb[i] + dh, w = wb[i] + dw;
        const bool ok = kvalid && (unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W;
        int pix = (nmod ? prem[i] : pre[i]) + toff;
        if (slow_mod) {                    // a second, different modulus: recompute (never the case in this model)
          const int n = (pre[i] / (p.H * p.W)) % nmod;
          pix = (n * p.H + h) * p.W + w;
        }
        cp_async16(a_dst + i * 32 * 128, ok ? (const void*)(spc + (size_t)pix * pitch) : (const void*)sp, ok ? 16u : 0u);
      }
      t += adv_t;
      c += adv_c;
      if (c >= m_chunks) {
        c -= m_chunks;
        ++t;
      }
      // ---- B: packed weights, rows rl + 32 i
      const uint32_t b_dst = b_base + s * Cfg::kBStage + rl * 128 + sw_off;
      if constexpr (BN >= 32) {
#pragma unroll
        for (int i = 0; i < BN / 32; ++i) cp_async16(b_dst + i * 32 * 128, wrow + (size_t)i * 32 * p.K_pad + (kb_lo + kb) * kBK, 16u);
      } else {
        if (rl < BN) cp_async16(b_dst, wrow + (kb_lo + kb) * kBK, 16u);
      }
      cp_async_commit();
      if (kb >= Cfg::kLag) {         // publish block kb-kLag (its copies have landed) while the kLag younger blocks are in flight
        cp_async_wait<Cfg::kLag>();
        fence_proxy_async();
        mbar_arrive(bar_full + 8 * ((kb - Cfg::kLag) % S));
      }
    }
#pragma unroll
    for (int i = Cfg::kLag - 1; i >= 0; --i) {   // drain: block nkb-1-i has i younger groups behind it
      if (nkb - 1 - i < 0) continue;
      if (i == 3) cp_async_wait<3>();
      else if (i == 2) cp_async_wait<2>();
      else if (i == 1) cp_async_wait<1>();
      else cp_async_wait<0>();
      fence_proxy_async();
      mbar_arrive(bar_full + 8 * ((nkb - 1 - i) % S));
    }
    if constexpr (Cfg::kProdRegs > 0) {   // the MMA warpgroup returns its share after its last MMA
      named_bar_sync<2, kGProducers>();
      setmaxnreg_inc<Cfg::kLaunchRegs>();
    }

    // ------------------------------------------------------------------ epilogue: warps w and w + 4 share 32 accumulator rows and split the columns
    mbar_wait(bar_accum, 0);
    if (tid == 0) CIS_TRACE_AT(2);
    const int qtr = warp & 3, half = warp >> 2;
    const int row = qtr * 32 + lane;
    const int g = blockIdx.x * kBM + row;
    const bool valid = g < M;
    size_t dpix = 0;
    if (valid) {
      const int ow = g % p.OW;
      const int t = g / p.OW;
      const int oh = t % p.OH;
      const int n = t / p.OH;
      dpix = (size_t)(n * p.DH + oh * p.osh + p.oa) * p.DW + ow * p.osw + p.ob;
    }
    const uint32_t t_row = tile_base + (uint32_t)row * 16;          // the accumulator tile overlays the (dead) operand ring
    const int cbase = ny * BN;
    constexpr int kHalf = BN >= 32 ? BN / 2 : BN;                 // BN = 16: the first warp group does it all
    const int c_lo = half * kHalf, c_hi = (BN >= 32 || half == 0) ? c_lo + kHalf : c_lo;
    if (nsplit > 1 && p.sk_cluster) {
      // cluster split-K: the partial tile already sits in this CTA's shared memory in the layout the reduction below reads
    } else if (nsplit > 1) {
      // two-launch split-K: this split's private fp32 slice; splitk_finish_kernel reduces the slices and runs the fused epilogue
      const int tile_id = blockIdx.x * gridDim.y + ny;
      float* tile0 = p.sk_scratch + (size_t)tile_id * nsplit * kBM * BN;
      splitk_store_partial<BN>(tile0 + (size_t)blockIdx.z * kBM * BN, t_row, row, c_lo, c_hi);
    } else {
      epi_cols<BN>(p, t_row, cbase, dpix, valid, s_bias, c_lo, c_hi);
    }
  } else {
    // ------------------------------------------------------------------ MMA warpgroup
    if constexpr (Cfg::kMmaRegs > 0) setmaxnreg_inc<Cfg::kMmaRegs>();
    const int wtid = tid - kMmaWarp * 32;
    float acc[BN];
    const uint32_t dhi = desc_hi(1024);
    constexpr uint32_t a_half = (8 * 1024) >> 4;     // rows 64..127: 8 core-matrix groups of SBO = 1024 B further
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % S;
      mbar_wait(bar_full + 8 * s, (uint32_t)((kb / S) & 1));
      if (wtid == 0) CIS_TRACE_AT(8 + 2 * kb);
      const uint32_t alo = desc_lo(a_base + s * kAStage, 16), blo = desc_lo(b_base + s * Cfg::kBStage, 16);
      wg_fence();
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k) mma128<BN, 0, 0>(acc, alo + 2 * k, dhi, blo + 2 * k, dhi, a_half, (uint32_t)((kb | k) != 0));
      wg_commit();
      wg_wait<1>();                 // block kb-1 has been consumed: release its stage while block kb runs
      if (wtid == 0 && kb > 0) mbar_arrive(bar_empty + 8 * ((kb - 1) % S));
      if (wtid == 0) CIS_TRACE_AT(9 + 2 * kb);
    }
    wg_wait<0>();
    acc_store<BN>(acc, tile_base, wtid);   // every operand stage has been consumed: the ring is dead
    if constexpr (Cfg::kMmaRegs > 0) {
      named_bar_sync<3, 128>();
      setmaxnreg_dec<Cfg::kLaunchRegs>();
    }
    mbar_arrive(bar_accum);
  }
  if (nsplit > 1 && p.sk_cluster) {
    cluster_sync_all();                       // every CTA's partial tile is in its shared memory
    if (warp < kMmaWarp) {
      const int cbase = ny * BN;
      cluster_reduce_rows<BN>(p, tile_base, nsplit, (int)cluster_ctarank(), tid, kGProducers, cbase, [&](int row, bool& valid) -> size_t {
        const int g = blockIdx.x * kBM + row;
        valid = g < M;
        if (!valid) return 0;
        const int ow = g % p.OW;
        const int t = g / p.OW;
        const int oh = t % p.OH;
        const int n = t / p.OH;
        return (size_t)(n * p.DH + oh * p.osh + p.oa) * p.DW + ow * p.osw + p.ob;
      });
    }
    cluster_sync_all();                       // peers may still be reading this CTA's shared memory
  }
  if (tid == 0) CIS_TRACE_AT(3);
}


// ======================================================================================================= halo-resident conv
// Stride-1 gathers (forward convs incl. dilated ones, stride-1 data gradients, parity launches of stride-2 data gradients and
// of the 4x4 s2 transposed convs).  The CTA owns MT stacked tiles of 16x8 output pixels of one dilation phase; per 64-channel
// chunk the (16*MT+ey) x (8+ex) input halo is copied ONCE into shared memory (SWIZZLE_128B rows of 128 B = one pixel x 64 ch)
// and every tap (dy,dx) reads it in place: A descriptor start = halo + ((16*m+dy)*Wh + dx)*128, SBO = Wh*128.  The hardware
// applies the 128B swizzle on absolute shared-memory address bits, so 128-byte-granular starts and a
// non-1024 SBO are legal with base_offset = 0.  im2col traffic drops from k*k x to ~1.3 x and the packed weights of a
// (tap, chunk) are reused by the MT tiles.
static constexpr int kHaloMaxBStages = 8;
struct HaloMaps {
  // one 4-D (C, W, H, N) SWIZZLE_128B map per (concat source, stride-2 phase): index si * nph + phase; box = (64, Wh, Hh, 1)
  // (compact format: SWIZZLE_NONE, box (8, Wh, Hh, 1))
  CUtensorMap m[CIS_MAX_SRC * 4];
  // wrow = 1 (compact format only): the weights are read in place from a gather launch's row pack [n_tiles * BN][K_pad] through the 2-D
  // no-swizzle map w, box (8, BN): kgroup j of K=16 step s is the 8 K columns from wk[2 s + j], landed as BN rows of 16 B at
  // s * BN * 32 + j * BN * 16 (B descriptor: SBO 128, LBO BN * 16).  wrow = 0: pre-tiled weights at wpack.
  CUtensorMap w;
  int wrow;
  int16_t wk[2 * CIS_MAX_TAPS];
};
// weights of the K=16 steps [s0, s0 + ns) of output channels [n0, n0 + BN) from the row pack (HaloMaps::wrow) to dst
__device__ __forceinline__ void wrow_load(const HaloMaps& maps, const uint32_t dst, const uint32_t bar, const int s0, const int ns, const int n0,
                                          const int BN) {
  for (int s = 0; s < ns; ++s)
    for (int j = 0; j < 2; ++j) tma_load_2d(dst + (uint32_t)(s * BN * 32 + j * BN * 16), &maps.w, bar, maps.wk[2 * (s0 + s) + j], n0);
}

// wgmma of one weight stage (gt taps of one 64-channel chunk, MT stacked tiles, NK K=16 steps each), issued by the MMA warpgroup into
// the register accumulators acc[m] of the MT tiles.  The tap offsets come from a shared-memory table (a broadcast read); the offset
// two taps ahead is fetched before the current tap's wgmma are issued.  Every tap is its own straight-line fence .. commit group:
// with a branch or a loop between wgmma.fence and wgmma.commit_group ptxas serialises every wgmma of the kernel (C7520).
template <int NK, int MT, int BN, int MTM>
__device__ __forceinline__ void halo_issue_stage(float (&acc)[MTM][BN], const uint32_t hlo, uint32_t blo, const uint32_t* s_aoff, const int gt,
                                                 const uint32_t ahi, const uint32_t bhi, const uint32_t a_mstep, const uint32_t a_half,
                                                 const uint32_t bstep, const bool first) {
  uint32_t off0 = s_aoff[0], off1 = gt > 1 ? s_aoff[1] : 0u;
  int tt = 0;
#pragma unroll 1
  do {
    const uint32_t off2 = tt + 2 < gt ? s_aoff[tt + 2] : 0u;    // two taps ahead
    const uint32_t alo = hlo + off0;
    const uint32_t acc0 = (uint32_t)(!(first && tt == 0));
    wg_fence();
#pragma unroll
    for (int m = 0; m < MT; ++m) {
#pragma unroll
      for (int k = 0; k < NK; ++k) mma128<BN, 0, 0>(acc[m], alo + m * a_mstep + 2 * k, ahi, blo + 2 * k, bhi, a_half, k ? 1u : acc0);
    }
    wg_commit();
    off0 = off1;
    off1 = off2;
    blo += bstep;
  } while (++tt < gt);
}
// one weight stage with the K depth of the chunk (nk16 = 1..4 K=16 steps: the last chunk of a layer may be partial)
template <int MT, int BN, int MTM>
__device__ __forceinline__ void halo_issue_nk(const int nk16, float (&acc)[MTM][BN], const uint32_t hlo, const uint32_t blo, const uint32_t* s_aoff,
                                              const int gt, const uint32_t ahi, const uint32_t bhi, const uint32_t a_mstep, const uint32_t a_half,
                                              const uint32_t bstep, const bool first) {
  if (nk16 == 4) halo_issue_stage<4, MT>(acc, hlo, blo, s_aoff, gt, ahi, bhi, a_mstep, a_half, bstep, first);
  else if (nk16 == 1) halo_issue_stage<1, MT>(acc, hlo, blo, s_aoff, gt, ahi, bhi, a_mstep, a_half, bstep, first);
  else if (nk16 == 2) halo_issue_stage<2, MT>(acc, hlo, blo, s_aoff, gt, ahi, bhi, a_mstep, a_half, bstep, first);
  else halo_issue_stage<3, MT>(acc, hlo, blo, s_aoff, gt, ahi, bhi, a_mstep, a_half, bstep, first);
}
template <int BN, int MTM>
__device__ __forceinline__ void halo_issue_any(const int nk16, float (&acc)[MTM][BN], const uint32_t hlo, const uint32_t blo, const uint32_t* s_aoff,
                                               const int gt, const int MT, const uint32_t ahi, const uint32_t bhi, const uint32_t a_mstep,
                                               const uint32_t a_half, const uint32_t bstep, const bool first) {
  static_assert(MTM >= 1 && MTM <= 4, "1..4 stacked tiles");
  if (MT == 1) halo_issue_nk<1>(nk16, acc, hlo, blo, s_aoff, gt, ahi, bhi, a_mstep, a_half, bstep, first);
  else if constexpr (MTM >= 2) {
    if (MT == 2) halo_issue_nk<2>(nk16, acc, hlo, blo, s_aoff, gt, ahi, bhi, a_mstep, a_half, bstep, first);
    else if constexpr (MTM >= 3) {
      if (MT == 3) halo_issue_nk<3>(nk16, acc, hlo, blo, s_aoff, gt, ahi, bhi, a_mstep, a_half, bstep, first);
      else if constexpr (MTM >= 4) halo_issue_nk<4>(nk16, acc, hlo, blo, s_aoff, gt, ahi, bhi, a_mstep, a_half, bstep, first);
    }
  }
  wg_wait<0>();
}

// Compact thin-input halo (CisConv.thin = 8 / 16): one plane per 8 channels, 16 bytes per pixel, planes 128-byte aligned.
__host__ __device__ __forceinline__ int thin_plane_bytes(int HP) { return (HP * 16 + 127) & ~127; }
// K=16 steps of a tap list: one per tap, or one per tap pair in the compact 8-channel format
__host__ __device__ __forceinline__ int halo_nsteps(int thin, int ntaps) { return thin == 8 ? (ntaps + 1) / 2 : ntaps; }
// s_aoff entry of K=16 step s over the taps dh/dw[t0 .. t0 + nt): start of the step's A operand inside the halo in descriptor start-field
// units (16 B).  Compact format: OR-ed with its LBO (bits 16+), the distance to the second core matrix along K -- the next tap's origin
// (thin 8; the host lists the taps in increasing order of origin; an odd last tap pairs with itself against zero weights) or plane 1
// (thin 16).  Stride-2 phases (nph = 4): the planes of phase q follow those of phases 0 .. q-1, so the taps, listed phase by phase,
// still lie at increasing offsets and a pair may span two phases.
__device__ __forceinline__ uint32_t halo_tap_off(const CisConv& p, const int t, const int Wh, const uint32_t plane16) {
  int ph = 0;
  if (p.nph > 1)
    while (ph < p.nph - 1 && t >= p.ph_tap[ph + 1]) ++ph;
  return (uint32_t)(ph * (p.thin / 8)) * plane16 + (uint32_t)(p.dh[t] * Wh + p.dw[t]);
}
__device__ __forceinline__ uint32_t halo_step_off(const CisConv& p, const int t0, const int nt, const int s, const int Wh, const uint32_t plane16) {
  if (!p.thin) return (uint32_t)((p.dh[t0 + s] * Wh + p.dw[t0 + s]) * 8);   // * 128 B / 16
  const int ta = p.thin == 8 ? 2 * s : s;
  const uint32_t o0 = halo_tap_off(p, t0 + ta, Wh, plane16);
  if (p.thin == 16) return o0 | (plane16 << 16);
  const uint32_t o1 = ta + 1 < nt ? halo_tap_off(p, t0 + ta + 1, Wh, plane16) : o0;
  return o0 | ((o1 - o0) << 16);
}
// compact halo of a TMA producer: per stride-2 phase with steps (one phase when nph <= 1), one no-swizzle plane of 8 channels per 8-channel
// slice of the sources, phase-major.  expect_tx covers every plane.  src: CisSrc array (kernel parameters or their shared-memory copy).
template <typename Src>
__device__ __forceinline__ void thin_halo_load(const CisConv& p, const Src* src, const HaloMaps& maps, const uint32_t dst, const uint32_t bar,
                                               const int HP, const int x0, const int y0, const int n) {
  const int nph = p.nph > 1 ? p.nph : 1, npl = p.thin / 8, pb16 = thin_plane_bytes(HP);
  int nld = 0;
  for (int ph = 0; ph < nph; ++ph) nld += nph == 1 || p.ph_tap[ph + 1] > p.ph_tap[ph];
  mbar_expect_tx(bar, (uint32_t)(nld * npl * HP * 16));
  for (int ph = 0; ph < nph; ++ph) {
    if (nph > 1 && p.ph_tap[ph + 1] == p.ph_tap[ph]) continue;      // phase without taps (kernel size 1)
    for (int q = 0; q < npl; ++q) {
      int cq = q, sq = 0;
      while (sq < p.nsrc - 1 && cq >= src[sq].chunks) {
        cq -= src[sq].chunks;
        ++sq;
      }
      const int nm = src[sq].n_mod;
      tma_load_4d(dst + (ph * npl + q) * pb16, &maps.m[sq * nph + ph], bar, cq * 8, x0, y0, nm ? (n % nm) : n);
    }
  }
}

template <int BN, int NWG>
__global__ void __launch_bounds__(HaloCfg<BN, NWG>::kThreads, HaloCfg<BN, NWG>::kCtasPerSm) conv_halo_kernel(const __grid_constant__ CisConv p, const int halo_stage_bytes, const int BS, const int NHS,
                                                        const __grid_constant__ HaloMaps maps, const int use_tma, const int G) {
  // One weight pipeline stage = the tiles of G consecutive taps of one 64-channel chunk (contiguous in the pre-tiled operand, ONE
  // bulk copy): the MMA warpgroup pays the per-stage cost (mbarrier wait, wgmma fence / commit / wait, release) once per 4*MT*G
  // MMAs instead of once per 4*MT.  With NWG = 2 MMA warpgroups the CTA is MTC = 2 * MT tiles tall: warpgroup w owns tiles
  // w * MT .. w * MT + MT - 1 of the one shared halo and both consume every weight stage.
  using Cfg = HaloCfg<BN, NWG>;
  constexpr int kBStage = BN * 128;
  constexpr int kHMmaWarp_ = Cfg::kMmaWarp, kHThreads_ = Cfg::kThreads;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t bars[2 * 2 + 2 * kHaloMaxBStages + 1];
  __shared__ uint32_t s_aoff[CIS_MAX_TAPS];   // tap origin inside the halo, in descriptor start-field units (16 B)
  __shared__ SrcS s_src[CIS_MAX_SRC];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int MT = p.MT, MTC = NWG * MT, d = p.dil;   // MT tiles per MMA warpgroup, MTC per CTA
  const int nph = p.nph > 1 ? p.nph : 1;       // stride-2 forward conv: 4 space-to-depth phases, each with its own halo planes and tap range
  const int Wh = 8 + p.ex, Hh = 16 * MTC + p.ey, HP = Wh * Hh;
  const int thin = p.thin;
  const int nhph = thin ? 1 : nph;             // halo stages per chunk: the compact format stages every phase's planes in one
  const uint32_t wstep = thin ? BN * 32 : kBStage;                  // weight bytes of one K=16 step (compact) or one tap (64-channel chunk)
  const uint32_t stage_bytes = (uint32_t)G * wstep;
  const uint32_t tile_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t h_base = tile_base;                                // NHS halo stages
  const uint32_t b_base = tile_base + NHS * halo_stage_bytes;       // BS weight stages of G tap tiles each
  int* pixtab = reinterpret_cast<int*>(smem_raw + (b_base + BS * stage_bytes - smem_u32(smem_raw)));
  const uint32_t bar_hfull = smem_u32(&bars[0]), bar_hempty = smem_u32(&bars[2]);
  const uint32_t bar_bfull = smem_u32(&bars[4]), bar_bempty = smem_u32(&bars[4 + kHaloMaxBStages]);
  const uint32_t bar_accum = smem_u32(&bars[4 + 2 * kHaloMaxBStages]);

  // ---- grouped launch: blockIdx.z selects one of nsub sub-problems (own taps, halo origin, weights, output extent / offset)
  const bool grouped = p.nsub > 1;
  const int tap0 = grouped ? p.sub[blockIdx.z].tap0 : 0, ntaps = grouped ? p.sub[blockIdx.z].ntaps : p.ntaps;
  const int nst = halo_nsteps(thin, ntaps);    // K=16 steps (compact) or taps (64-channel chunks) per chunk
  const int hoy = grouped ? p.sub[blockIdx.z].hoy : p.hoy, hox = grouped ? p.sub[blockIdx.z].hox : p.hox;
  const int OHs = grouped ? p.sub[blockIdx.z].OH : p.OH, OWs = grouped ? p.sub[blockIdx.z].OW : p.OW;
  const int oa = grouped ? p.sub[blockIdx.z].oa : p.oa, ob = grouped ? p.sub[blockIdx.z].ob : p.ob;
  const void* const wpack = grouped ? p.sub[blockIdx.z].wpack : p.wpack;
  // ---- tile decode: blockIdx.x -> (tx, ty, phase, n)
  const int Hp0 = (OHs + d - 1) / d, Wp0 = (OWs + d - 1) / d;
  const int tiles_x = (Wp0 + 7) / 8, tiles_y = (Hp0 + 16 * MTC - 1) / (16 * MTC);
  if (grouped && (int)blockIdx.x >= tiles_x * tiles_y * p.N) return;   // the grid is sized for the largest sub-problem (uniform per CTA)
  int bid = blockIdx.x;
  const int tx = bid % tiles_x; bid /= tiles_x;
  const int ty = bid % tiles_y; bid /= tiles_y;
  const int ph = bid % (d * d);
  const int n = bid / (d * d);
  const int pa = ph / d, pb = ph % d;
  const int ny = blockIdx.y;
  int m_chunks = 0;
  for (int i = 0; i < p.nsrc; ++i) m_chunks += p.src[i].chunks;
  const int nchunks_all = (m_chunks + 7) / 8;  // 64-channel chunks
  const int nsplit = (!grouped && p.splits > 1) ? p.splits : 1;
  const int cper = (nchunks_all + nsplit - 1) / nsplit;
  const int cc_lo = grouped ? 0 : blockIdx.z * cper;
  const int nchunks = min(cper, nchunks_all - cc_lo);   // chunks handled by this CTA (host guarantees >= 1)
  __shared__ __align__(16) float s_bias[BN];
  pdl_launch_dependents();

  if (tid < nst) s_aoff[tid] = halo_step_off(p, tap0, ntaps, tid, Wh, (uint32_t)thin_plane_bytes(HP) >> 4);
  if (tid < p.nsrc) {
    s_src[tid].ptr = reinterpret_cast<const __nv_bfloat16*>(p.src[tid].ptr);
    s_src[tid].pitch = p.src[tid].pitch;
    s_src[tid].c_off = p.src[tid].c_off;
    s_src[tid].chunks = p.src[tid].chunks;
    s_src[tid].n_mod = p.src[tid].n_mod;
  }
  for (int q = tid; q < (use_tma ? 0 : HP); q += kHThreads_) {
    const int hy = q / Wh, hx = q - hy * Wh;
    const int gy = ty * 16 * MTC + hy + hoy, gx = tx * 8 + hx + hox;
    const int y = pa + d * gy, x = pb + d * gx;
    pixtab[q] = (gy >= 0 && gx >= 0 && y < p.H && x < p.W) ? (y * p.W + x) : -1;
  }
  if (tid == kHMmaWarp_ * 32) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(bar_hfull + 8 * s, use_tma ? 1 : 96);
      mbar_init(bar_hempty + 8 * s, NWG);
    }
    for (int s = 0; s < BS; ++s) {
      mbar_init(bar_bfull + 8 * s, 1);     // one expect_tx arrival; the bulk copy completes the transaction bytes
      mbar_init(bar_bempty + 8 * s, NWG);  // one release per MMA warpgroup
    }
    mbar_init(bar_accum, 128 * NWG);       // every thread of the MMA warpgroups, after storing its accumulator fragments
    fence_mbar_init();
  }
  if (use_tma && tid < p.nsrc) tma_prefetch_desc(&maps.m[tid]);   // descriptors live in the kernel parameters: fetch them before the grid dependency resolves
  pdl_wait();
  if (tid < BN) s_bias[tid] = p.bias ? p.bias[ny * BN + tid] : 0.f;
  __syncthreads();
  if (tid == 0) CIS_TRACE_AT(0);

  if (warp < kHMmaWarp_) {
    // ------------------------------------------------------------------ producers
    // Two independent roles so neither stream throttles the other: warps 0-1 stream the per-chunk halos (2 stages), warps 2-3
    // stream the per-(tap, chunk) weight tiles (BS stages).
    if constexpr (Cfg::kProdRegs > 0) setmaxnreg_dec<Cfg::kProdRegs>();
    if (use_tma) {
      if (tid == 0) {
        // halo through the TMA engine: one 4-D tiled load per 64-channel chunk (x phase), out-of-image pixels / channels are zero-filled
        int hcount = 0;
        for (int vc = 0; vc < nchunks * nhph; ++vc) {
          const int cc = vc / nhph, ph = vc - cc * nhph;
          if (nhph > 1 && p.ph_tap[ph + 1] == p.ph_tap[ph]) continue;      // phase without taps (kernel size 1)
          const int hs = hcount % NHS;
          mbar_wait(bar_hempty + 8 * hs, (uint32_t)(((hcount / NHS) & 1) ^ 1));
          ++hcount;
          int c = (cc_lo + cc) * 8, si = 0;
          while (si < p.nsrc - 1 && c >= s_src[si].chunks) {
            c -= s_src[si].chunks;
            ++si;
          }
          const int nmod = s_src[si].n_mod;
          if (thin) {
            // compact halo (single chunk, undilated): the planes of every phase in one stage
            thin_halo_load(p, s_src, maps, h_base + hs * halo_stage_bytes, bar_hfull + 8 * hs, HP, tx * 8 + hox, ty * 16 * MTC + hoy, n);
            continue;
          }
          mbar_expect_tx(bar_hfull + 8 * hs, (uint32_t)(HP * 128));
          // dilated layer: the map strides by d pixels from any start, the start carries this CTA's phase (pa, pb)
          tma_load_4d(h_base + hs * halo_stage_bytes, &maps.m[si * nph + ph], bar_hfull + 8 * hs, c * 8, pb + d * (tx * 8 + hox),
                      pa + d * (ty * 16 * MTC + hoy), nmod ? (n % nmod) : n);
        }
      }
      __syncwarp();
    } else if (warp != 2) {
      const int hid = warp == 3 ? tid - 32 : tid;   // 96 halo loader threads (warps 0, 1, 3)
      const int j = hid & 7, pl = hid >> 3;         // pl = 0..11
      for (int cc = 0; cc < nchunks; ++cc) {
        const int hs = cc % NHS;
        mbar_wait(bar_hempty + 8 * hs, (uint32_t)(((cc / NHS) & 1) ^ 1));
        const int rem = m_chunks - (cc_lo + cc) * 8;       // valid 16-byte chunks in this 64-channel chunk
        const int nk16 = rem >= 8 ? 4 : (rem + 1) / 2;     // K=16 MMA groups actually issued
        const bool need = j < 2 * nk16;
        const bool cvalid = j < rem;
        int c = (cc_lo + cc) * 8 + j, si = 0;
        if (cvalid) {
          while (si < p.nsrc - 1 && c >= s_src[si].chunks) {
            c -= s_src[si].chunks;
            ++si;
          }
        } else {
          c = 0;
        }
        const int nmod = s_src[si].n_mod, pitch = s_src[si].pitch;
        const int ne = nmod ? (n % nmod) : n;
        const __nv_bfloat16* sp = s_src[si].ptr;
        const __nv_bfloat16* sb = sp + (size_t)ne * p.H * p.W * pitch + s_src[si].c_off + c * 8;
        if (need) {
          const uint32_t hdst = h_base + hs * halo_stage_bytes + (uint32_t)(j << 4);
          for (int q = pl; q < HP; q += 12) {
            const int off = pixtab[q];
            const bool ok = cvalid && off >= 0;
            cp_async16((hdst + q * 128) ^ (uint32_t)((q & 7) << 4), ok ? (const void*)(sb + (size_t)off * pitch) : (const void*)sp,
                       ok ? 16u : 0u);
          }
        }
        cp_async_commit();
        if (NHS == 1) {
          cp_async_wait<0>();
          fence_proxy_async();
          mbar_arrive(bar_hfull);
        } else if (cc >= 1) {        // two stages: publish chunk cc-1 while chunk cc is in flight
          cp_async_wait<1>();
          fence_proxy_async();
          mbar_arrive(bar_hfull + 8 * ((cc - 1) % NHS));
        }
      }
      if (NHS > 1) {
        cp_async_wait<0>();
        fence_proxy_async();
        mbar_arrive(bar_hfull + 8 * ((nchunks - 1) % NHS));
      }
    }
    if (tid == 64) {
      // weights: pre-swizzled [n-tile][chunk][tap] tiles of BN x 128 B (cis_pack_weights_tiled); the tiles of the G taps of a stage
      // are adjacent in that layout -> ONE bulk copy per pipeline stage
      const uint8_t* wt = reinterpret_cast<const uint8_t*>(wpack) + ((size_t)ny * nchunks_all + cc_lo) * nst * wstep;
      int bs = 0;
      uint32_t bph = 1;           // parity to wait for on the empty barrier: the first pass over the ring finds every stage free
      for (int vc = 0; vc < nchunks * nhph; ++vc) {
        const int cc = vc / nhph, ph = vc - cc * nhph;
        const int tlo = nhph > 1 ? p.ph_tap[ph] : 0, thi = nhph > 1 ? p.ph_tap[ph + 1] : nst;
        for (int t0 = tlo; t0 < thi; t0 += G) {
          const uint32_t bytes = (uint32_t)min(G, thi - t0) * wstep;
          mbar_wait(bar_bempty + 8 * bs, bph);
          mbar_expect_tx(bar_bfull + 8 * bs, bytes);
          if (maps.wrow) wrow_load(maps, b_base + bs * stage_bytes, bar_bfull + 8 * bs, t0, min(G, thi - t0), ny * BN, BN);
          else bulk_g2s(b_base + bs * stage_bytes, wt + (size_t)(cc * nst + t0) * wstep, bytes, bar_bfull + 8 * bs);
          if (++bs == BS) {
            bs = 0;
            bph ^= 1u;
          }
        }
      }
    }
    __syncwarp();
    // back to the even split for the epilogue; the MMA warpgroup returns its share once its accumulators are in shared memory
    if constexpr (Cfg::kProdRegs > 0) {
      named_bar_sync<2, 128>();
      setmaxnreg_inc<Cfg::kLaunchRegs>();
    }
  } else {
    // ------------------------------------------------------------------ MMA warpgroup(s)
    if constexpr (Cfg::kMmaRegs > 0) setmaxnreg_inc<Cfg::kMmaRegs>();
    const int wg = NWG > 1 ? (warp - kHMmaWarp_) >> 2 : 0;
    const int wtid = tid - (kHMmaWarp_ + 4 * wg) * 32;
    constexpr int MTM = Cfg::kMaxMT;
    float acc[MTM][BN];
    // pixel pitch of the halo: 128 B (64-channel SWIZZLE_128B chunk) or 16 B (compact no-swizzle plane); B: 8-row groups 1024 / 256 B apart
    // (row-pack weights: 128 B, the two kgroups BN * 16 B apart)
    const uint32_t pix = thin ? 16u : 128u;
    const uint32_t ahi = thin ? desc_hi_ns((uint32_t)Wh * pix) : desc_hi((uint32_t)Wh * pix);
    const uint32_t bhi = thin ? desc_hi_ns(maps.wrow ? 128u : 256u) : desc_hi(1024), b_lbo = maps.wrow ? BN * 16u : thin ? 128u : 16u;
    const uint32_t a_mstep = (16u * Wh * pix) >> 4;   // descriptor start-field step between stacked M tiles
    const uint32_t a_half = (8u * Wh * pix) >> 4;     // rows 64..127 of a tile: 8 halo rows further
    const uint32_t a_wg = (uint32_t)(wg * MT) * a_mstep;        // this warpgroup's first tile inside the halo
    int bs = 0, hs = 0, it = 0;
    uint32_t bph = 0, hph = 0;
    bool any = false;
    for (int vc = 0; vc < nchunks * nhph; ++vc) {
      const int cc = vc / nhph, ph = vc - cc * nhph;
      const int tlo = nhph > 1 ? p.ph_tap[ph] : 0, thi = nhph > 1 ? p.ph_tap[ph + 1] : nst;
      if (thi == tlo) continue;
      const int rem = m_chunks - (cc_lo + cc) * 8;
      const int nk16 = rem >= 8 ? 4 : (rem + 1) / 2;
      mbar_wait(bar_hfull + 8 * hs, hph);
      if (vc == 0 && wtid == 0 && wg == 0) CIS_TRACE_AT(1);
      // compact format: the LBO of every step comes with its s_aoff entry
      const uint32_t hlo = desc_lo(h_base + hs * halo_stage_bytes, thin ? 0 : 16) + a_wg;
      for (int t0 = tlo; t0 < thi; t0 += G, ++it) {
        const int gt = min(G, thi - t0);
        mbar_wait(bar_bfull + 8 * bs, bph);
        if (wtid == 0 && wg == 0) CIS_TRACE_AT(8 + 2 * it);
        const uint32_t blo = desc_lo(b_base + bs * stage_bytes, b_lbo);
        halo_issue_any<BN, MTM>(nk16, acc, hlo, blo, s_aoff + t0, gt, MT, ahi, bhi, a_mstep, a_half, wstep >> 4, !any);
        if (wtid == 0) {   // one release per warpgroup
          mbar_arrive(bar_bempty + 8 * bs);
          if (t0 + G >= thi) mbar_arrive(bar_hempty + 8 * hs);
          if (wg == 0) CIS_TRACE_AT(9 + 2 * it);
        }
        any = true;
        if (++bs == BS) {
          bs = 0;
          bph ^= 1u;
        }
      }
      if (++hs == NHS) {
        hs = 0;
        hph ^= 1u;
      }
    }
    // every operand stage has been consumed: the accumulator tiles overlay the operand buffers.  Two warpgroups: the other one may
    // still be reading the last stages, so both finish their wgmma before either overwrites them.
    if constexpr (NWG > 1) asm volatile("bar.sync 1, %0;" ::"n"(128 * NWG) : "memory");
#pragma unroll
    for (int m = 0; m < MTM; ++m)
      if (m < MT) acc_store<BN>(acc[m], tile_base + (uint32_t)((wg * MT + m) * BN) * kAccColBytes, wtid);
    if constexpr (Cfg::kMmaRegs > 0) {
      named_bar_sync<3, 128>();
      setmaxnreg_dec<Cfg::kLaunchRegs>();
    }
    mbar_arrive(bar_accum);
  }

  if (warp < Cfg::kEpiWarps) {
    // ------------------------------------------------------------------ epilogue: unit u = (tile m, 32-row quarter, column part); warp w
    // takes units w, w + kEpiWarps, ...  (NWG = 1, BN >= 64: warps w and w + 4 share accumulator rows 32 (w % 4) .. 32 (w % 4) + 31 and
    // split the columns -- the epilogue is instruction-bound on its warps)
    mbar_wait(bar_accum, 0);
    if (tid == 0) CIS_TRACE_AT(2);
    constexpr int kParts = Cfg::kEpiParts, kCols = BN / kParts, kUnits = 4 * kParts;
    const int cbase = ny * BN;
    const int tile_id = blockIdx.x * gridDim.y + ny;
    // cluster split-K: the MTC partial tiles already sit in this CTA's shared memory in the layout the reduction below reads
    if (!(nsplit > 1 && p.sk_cluster)) {
#pragma unroll 1
      for (int u = warp; u < MTC * kUnits; u += Cfg::kEpiWarps) {
        const int m = u / kUnits, r = (u & 3) * 32 + lane, c_lo = ((u >> 2) % kParts) * kCols, c_hi = c_lo + kCols;
        const uint32_t t_row = tile_base + (uint32_t)(m * BN) * kAccColBytes + (uint32_t)r * 16;   // the operand buffers are dead
        if (nsplit > 1) {
          // two-launch split-K: this split's private fp32 slices; splitk_finish_kernel reduces them and runs the fused epilogue
          splitk_store_partial<BN>(p.sk_scratch + (((size_t)tile_id * MTC + m) * nsplit + blockIdx.z) * kBM * BN, t_row, r, c_lo, c_hi);
        } else {
          const int gy = ty * 16 * MTC + 16 * m + (r >> 3), gx = tx * 8 + (r & 7);
          const int oy = pa + d * gy, ox = pb + d * gx;
          const bool valid = oy < OHs && ox < OWs;
          const size_t dpix = valid ? ((size_t)(n * p.DH + oy * p.osh + oa) * p.DW + ox * p.osw + ob) : 0;
          epi_cols<BN>(p, t_row, cbase, dpix, valid, s_bias, c_lo, c_hi);
        }
      }
    }
  }
  if (nsplit > 1 && p.sk_cluster) {
    cluster_sync_all();                       // every CTA's partial tiles are in its shared memory
    if (warp < 4) {
      const int cbase = ny * BN;
      for (int m = 0; m < MTC; ++m)
        cluster_reduce_rows<BN>(p, tile_base + (uint32_t)m * (kBM * BN * 4), nsplit, (int)cluster_ctarank(), tid, 128, cbase,
                                [&](int row, bool& valid) -> size_t {
                                  const int gy = ty * 16 * MTC + 16 * m + (row >> 3), gx = tx * 8 + (row & 7);
                                  const int oy = pa + d * gy, ox = pb + d * gx;
                                  valid = oy < OHs && ox < OWs;
                                  return valid ? ((size_t)(n * p.DH + oy * p.osh + oa) * p.DW + ox * p.osw + ob) : 0;
                                });
    }
    cluster_sync_all();                       // peers may still be reading this CTA's shared memory
  }
  if (tid == 0) CIS_TRACE_AT(3);
}

// ======================================================================================================= split-K finish
// Second launch of split-K (letting the last-arriving CTA of a tile read all nsplit x 64 KB slices by itself would pull up to 1 MB
// through one SM).  Here the reduction + fused
// epilogue of a tile is spread over 128 * BN/16 threads of several CTAs: thread = (accumulator row, 16-column group), row fastest so
// the reads of the float4-column slices coalesce (the bf16 output is 1 / (2 * nsplit) of the bytes: its 32-byte pieces matter less).
template <int BN>
__global__ void __launch_bounds__(256) splitk_finish_kernel(const __grid_constant__ CisConv p) {
  constexpr int G = BN / 16;                               // 16-column groups per row
  constexpr int kBlock = (128 * G < 256) ? 128 * G : 256;
  constexpr int kSub = 128 * G / kBlock;                   // CTAs per (tile, m)
  pdl_launch_dependents();
  pdl_wait();
  const int tid = threadIdx.x;
  if (tid >= kBlock) return;
  const int m = blockIdx.z / kSub;
  const int item = (blockIdx.z % kSub) * kBlock + tid;
  const int r = item % 128, c0 = (item / 128) * 16;        // row fastest: a warp reads 512 contiguous bytes of every slice
  const int ny = blockIdx.y;
  const int nsplit = p.splits;
  const int tile_id = blockIdx.x * gridDim.y + ny;
  bool valid;
  size_t dpix = 0;
  const float* tile0;
  if (p.halo) {
    const int MT = p.MT * (p.nwg > 1 ? p.nwg : 1), d = p.dil;   // tiles per CTA
    const int Hp0 = (p.OH + d - 1) / d, Wp0 = (p.OW + d - 1) / d;
    const int tiles_x = (Wp0 + 7) / 8, tiles_y = (Hp0 + 16 * MT - 1) / (16 * MT);
    int bid = blockIdx.x;
    const int tx = bid % tiles_x; bid /= tiles_x;
    const int ty = bid % tiles_y; bid /= tiles_y;
    const int ph = bid % (d * d);
    const int n = bid / (d * d);
    const int pa = ph / d, pb = ph % d;
    const int gy = ty * 16 * MT + 16 * m + (r >> 3), gx = tx * 8 + (r & 7);
    const int oy = pa + d * gy, ox = pb + d * gx;
    valid = oy < p.OH && ox < p.OW;
    if (valid) dpix = (size_t)(n * p.DH + oy * p.osh + p.oa) * p.DW + ox * p.osw + p.ob;
    tile0 = p.sk_scratch + ((size_t)tile_id * MT + m) * nsplit * kBM * BN;
  } else {
    const int M = p.N * p.OH * p.OW;
    const int g = blockIdx.x * kBM + r;
    valid = g < M;
    if (valid) {
      const int ow = g % p.OW;
      const int t = g / p.OW;
      const int oh = t % p.OH;
      const int n = t / p.OH;
      dpix = (size_t)(n * p.DH + oh * p.osh + p.oa) * p.DW + ow * p.osw + p.ob;
    }
    tile0 = p.sk_scratch + (size_t)tile_id * nsplit * kBM * BN;
  }
  if (!valid) return;
  float v[16];
  splitk_reduce16<BN>(tile0, nsplit, r, c0, v);
  epi_chunk(p, v, ny * BN + c0, dpix);
}
// ======================================================================================================= persistent halo conv
// Same math as conv_halo_kernel (TMA halo path only) for layers with MANY output tiles per SM (high-resolution thin layers), where the
// per-CTA prologue (barrier init, first TMA round trip) and epilogue (accumulator read-back + stores) of the one-tile-per-CTA kernel
// cost more than its MMA loop.  Here a CTA is persistent and fully warp-specialised so those phases of neighbouring tiles overlap:
//   warps 0-3: MMA warpgroup | warps 4-7 / 8-11: two epilogue groups (accumulator rows 32 (warp % 4) ..) | warp 12: halo TMA
//   producer (NHS stages) | warp 13: weight producer.  Tile i is handed over in shared-memory accumulator stage i % AS to group i % AS.
// Weights: resident (ws = 1: the whole set of nchunks*ntaps tiles is fetched once per CTA and stays in shared memory while the CTA
// walks its tiles) when it fits, else re-streamed per tile in stages of G taps through a ring of BS stages.
// Every role walks the same static work list  w = blockIdx.x, blockIdx.x + gridDim.x, ...  of output tiles.
static constexpr int kPThreads = 448;
static constexpr int kPMaxAccCols = 64;    // MT * BN limit of the persistent kernel (register accumulators next to 13 other warps)

template <int BN>
__global__ void __launch_bounds__(kPThreads, 1) conv_halo_persist_kernel(const __grid_constant__ CisConv p, const int halo_stage_bytes,
                                                                       const int BS, const int NHS, const int AS, const int G,
                                                                       const __grid_constant__ HaloMaps maps, const int ws) {
  constexpr int kBStage = BN * 128;
  constexpr int kMaxHS = 4;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t bars[2 * kMaxHS + 2 * kHaloMaxBStages + 4];
  __shared__ uint32_t s_aoff[CIS_MAX_TAPS];
  __shared__ __align__(16) float s_bias[BN];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int MT = p.MT;
  const int Wh = 8 + p.ex, Hh = 16 * MT + p.ey, HP = Wh * Hh;
  const int thin = p.thin;
  const bool grouped = p.nsub > 1;             // grouped launch: the sub-problems' tiles one after the other in the work list
  const int nsb = grouped ? p.nsub : 1;
  const uint32_t wstep = thin ? BN * 32 : kBStage;                  // weight bytes of one K=16 step (compact) or one tap (64-channel chunk)
  const uint32_t stage_bytes = (uint32_t)G * wstep;
  const uint32_t tile_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t acc_bytes = (uint32_t)(MT * BN) * kAccColBytes;     // one accumulator stage (a multiple of 8 KB)
  const uint32_t acc_base = tile_base, h_base = tile_base + AS * acc_bytes, b_base = h_base + NHS * halo_stage_bytes;
  const uint32_t bar_hfull = smem_u32(&bars[0]), bar_hempty = smem_u32(&bars[kMaxHS]);
  const uint32_t bar_bfull = smem_u32(&bars[2 * kMaxHS]), bar_bempty = smem_u32(&bars[2 * kMaxHS + kHaloMaxBStages]);
  const uint32_t bar_tfull = smem_u32(&bars[2 * kMaxHS + 2 * kHaloMaxBStages]), bar_tempty = smem_u32(&bars[2 * kMaxHS + 2 * kHaloMaxBStages + 2]);

  __shared__ int s_tcum[5], s_sbase[5];      // per sub-problem: first work item, first K=16 step (tap) in s_aoff and the resident weights
  int m_chunks = 0;
  for (int i = 0; i < p.nsrc; ++i) m_chunks += p.src[i].chunks;
  const int nchunks = (m_chunks + 7) / 8;

  pdl_launch_dependents();
  {
    int tc = 0, sb = 0;
    for (int z = 0; z < nsb; ++z) {
      const int nt = grouped ? p.sub[z].ntaps : p.ntaps, t0 = grouped ? p.sub[z].tap0 : 0, ns = halo_nsteps(thin, nt);
      const int oh = grouped ? p.sub[z].OH : p.OH, ow = grouped ? p.sub[z].OW : p.OW;
      if (tid >= sb && tid < sb + ns) s_aoff[tid] = halo_step_off(p, t0, nt, tid - sb, Wh, (uint32_t)thin_plane_bytes(HP) >> 4);
      if (tid == 0) {
        s_tcum[z] = tc;
        s_sbase[z] = sb;
      }
      tc += ((ow + 7) / 8) * ((oh + 16 * MT - 1) / (16 * MT)) * p.N;
      sb += ns;
    }
    if (tid == 0) {
      s_tcum[nsb] = tc;
      s_sbase[nsb] = sb;
    }
  }
  if (tid == 0) {
    for (int s = 0; s < NHS; ++s) {
      mbar_init(bar_hfull + 8 * s, 1);
      mbar_init(bar_hempty + 8 * s, 1);
    }
    for (int s = 0; s < BS; ++s) {
      mbar_init(bar_bfull + 8 * s, 1);
      mbar_init(bar_bempty + 8 * s, 1);
    }
    for (int s = 0; s < AS; ++s) {
      mbar_init(bar_tfull + 8 * s, 128);  // every thread of the MMA warpgroup, after storing its fragments
      mbar_init(bar_tempty + 8 * s, 4);   // one arrival per warp of the epilogue group that drained the stage
    }
    fence_mbar_init();
  }
  if (tid < p.nsrc) tma_prefetch_desc(&maps.m[tid]);
  pdl_wait();
  if (tid < BN) s_bias[tid] = p.bias ? p.bias[tid] : 0.f;
  __syncthreads();
  const int total = s_tcum[nsb];
  // work item w -> (sub-problem z, tile column tx, tile row ty, image n)
  auto decode = [&](const int w, int& z, int& tx, int& ty, int& n) {
    z = 0;
    while (z + 1 < nsb && w >= s_tcum[z + 1]) ++z;
    const int tiles_x = ((grouped ? p.sub[z].OW : p.OW) + 7) / 8, tiles_y = ((grouped ? p.sub[z].OH : p.OH) + 16 * MT - 1) / (16 * MT);
    const int l = w - s_tcum[z];
    tx = l % tiles_x;
    ty = (l / tiles_x) % tiles_y;
    n = l / (tiles_x * tiles_y);
  };
  if (tid == 0) {
    CIS_TRACE_AT(0);
    CIS_TRACE_AT(4);      // slot 4 marks a persistent-kernel trace (tools/trace_persist.py)
  }

  if (warp == 12) {
    // ------------------------------------------------------------------ halo producer
    if (lane == 0) {
      int hs = 0;
      uint32_t hph = 1;
      for (int w = blockIdx.x; w < total; w += gridDim.x) {
        int z, tx, ty, n;
        decode(w, z, tx, ty, n);
        const int hox = grouped ? p.sub[z].hox : p.hox, hoy = grouped ? p.sub[z].hoy : p.hoy;
        for (int cc = 0; cc < nchunks; ++cc) {
          mbar_wait(bar_hempty + 8 * hs, hph);
          int c = cc * 8, si = 0;
          while (si < p.nsrc - 1 && c >= p.src[si].chunks) {
            c -= p.src[si].chunks;
            ++si;
          }
          int nmod = p.src[0].n_mod;
          if (si == 1) nmod = p.src[1].n_mod;
          if (si == 2) nmod = p.src[2].n_mod;
          if (si == 3) nmod = p.src[3].n_mod;
          if (thin) {
            // compact halo, every stride-2 phase's planes in one stage (see conv_halo_kernel)
            thin_halo_load(p, p.src, maps, h_base + hs * halo_stage_bytes, bar_hfull + 8 * hs, HP, tx * 8 + hox, ty * 16 * MT + hoy, n);
          } else {
            mbar_expect_tx(bar_hfull + 8 * hs, (uint32_t)(HP * 128));
            tma_load_4d(h_base + hs * halo_stage_bytes, &maps.m[si], bar_hfull + 8 * hs, c * 8, tx * 8 + hox, ty * 16 * MT + hoy,
                        nmod ? (n % nmod) : n);
          }
          if (++hs == NHS) {
            hs = 0;
            hph ^= 1u;
          }
        }
      }
    }
  } else if (warp == 13) {
    // ------------------------------------------------------------------ weight producer
    if (lane == 0) {
      const uint8_t* wt = reinterpret_cast<const uint8_t*>(p.wpack);
      const int nst = s_sbase[1];          // ungrouped: weight tiles per chunk
      if (ws) {
        // the resident set: every sub-problem's tiles at its first step (grouped launches have one chunk; the host checks)
        if ((int)blockIdx.x < total) {
          mbar_expect_tx(bar_bfull, (uint32_t)(nchunks * s_sbase[nsb] * wstep));
          if (maps.wrow) wrow_load(maps, b_base, bar_bfull, 0, nst, 0, BN);      // one chunk, one n-tile, not grouped (the host checks)
          for (int z = 0; z < nsb && !maps.wrow; ++z) {
            const uint8_t* wz = grouped ? reinterpret_cast<const uint8_t*>(p.sub[z].wpack) : wt;
            const int per = nchunks * (s_sbase[z + 1] - s_sbase[z]);
            for (int it = 0; it < per; it += 8) {      // bulk copies of up to 8 tiles (<= 128 KB each)
              const int nt = min(8, per - it);
              bulk_g2s(b_base + (s_sbase[z] + it) * wstep, wz + (size_t)it * wstep, (uint32_t)(nt * wstep), bar_bfull);
            }
          }
        }
      } else {
        int bs = 0;
        uint32_t bph = 1;
        for (int w = blockIdx.x; w < total; w += gridDim.x) {
          for (int cc = 0; cc < nchunks; ++cc) {
            for (int t0 = 0; t0 < nst; t0 += G) {
              const uint32_t bytes = (uint32_t)min(G, nst - t0) * wstep;
              mbar_wait(bar_bempty + 8 * bs, bph);
              mbar_expect_tx(bar_bfull + 8 * bs, bytes);
              if (maps.wrow) wrow_load(maps, b_base + bs * stage_bytes, bar_bfull + 8 * bs, t0, min(G, nst - t0), 0, BN);
              else bulk_g2s(b_base + bs * stage_bytes, wt + (size_t)(cc * nst + t0) * wstep, bytes, bar_bfull + 8 * bs);
              if (++bs == BS) {
                bs = 0;
                bph ^= 1u;
              }
            }
          }
        }
      }
    }
  } else if (warp < 4) {
    // ------------------------------------------------------------------ MMA warpgroup
    const int wtid = tid;
    constexpr int MTM = (kPMaxAccCols / BN) < 4 ? kPMaxAccCols / BN : 4;
    float acc[MTM][BN];
    const uint32_t pix = thin ? 16u : 128u;       // halo pixel pitch (see conv_halo_kernel)
    const uint32_t ahi = thin ? desc_hi_ns((uint32_t)Wh * pix) : desc_hi((uint32_t)Wh * pix);
    const uint32_t bhi = thin ? desc_hi_ns(maps.wrow ? 128u : 256u) : desc_hi(1024), b_lbo = maps.wrow ? BN * 16u : thin ? 128u : 16u;
    const uint32_t a_mstep = (16u * Wh * pix) >> 4;
    const uint32_t a_half = (8u * Wh * pix) >> 4;
    int hs = 0, bs = 0, as = 0;
    uint32_t hph = 0, bph = 0, tph = 1;
    if (ws && (int)blockIdx.x < total) mbar_wait(bar_bfull, 0u);      // the resident weight set; never released
    int wi = 0;
    for (int w = blockIdx.x; w < total; w += gridDim.x, ++wi) {
      if (wtid == 0) CIS_TRACE_AT(8 + 5 * wi);
      int z, tx, ty, n;
      decode(w, z, tx, ty, n);
      const int nst = s_sbase[z + 1] - s_sbase[z];
      const uint32_t* so = s_aoff + s_sbase[z];
      for (int cc = 0; cc < nchunks; ++cc) {
        const int rem = m_chunks - cc * 8;
        const int nk16 = rem >= 8 ? 4 : (rem + 1) / 2;
        mbar_wait(bar_hfull + 8 * hs, hph);
        if (cc == 0 && wtid == 0) CIS_TRACE_AT(10 + 5 * wi);
        const uint32_t hlo = desc_lo(h_base + hs * halo_stage_bytes, thin ? 0 : 16);
        const int gstep = ws ? nst : G;
        for (int t0 = 0; t0 < nst; t0 += gstep) {
          const int gt = min(gstep, nst - t0);
          if (!ws) mbar_wait(bar_bfull + 8 * bs, bph);
          const uint32_t blo = desc_lo(ws ? b_base + (uint32_t)(s_sbase[z] + cc * nst) * wstep : b_base + bs * stage_bytes, b_lbo);
          halo_issue_any<BN, MTM>(nk16, acc, hlo, blo, so + t0, gt, MT, ahi, bhi, a_mstep, a_half, wstep >> 4, (cc | t0) == 0);
          if (wtid == 0) {
            if (!ws) mbar_arrive(bar_bempty + 8 * bs);
            if (t0 + gstep >= nst) mbar_arrive(bar_hempty + 8 * hs);
          }
          if (!ws && ++bs == BS) {
            bs = 0;
            bph ^= 1u;
          }
        }
        if (++hs == NHS) {
          hs = 0;
          hph ^= 1u;
        }
      }
      // hand the tile to epilogue group `as` once that group has drained the stage's previous tile
      mbar_wait(bar_tempty + 8 * as, tph);
      if (wtid == 0) CIS_TRACE_AT(9 + 5 * wi);
#pragma unroll
      for (int m = 0; m < MTM; ++m)
        if (m < MT) acc_store<BN>(acc[m], acc_base + as * acc_bytes + (uint32_t)(m * BN) * kAccColBytes, wtid);
      mbar_arrive(bar_tfull + 8 * as);
      if (wtid == 0) CIS_TRACE_AT(11 + 5 * wi);
      if (++as == AS) {
        as = 0;
        tph ^= 1u;
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ epilogue: group g = (warp - 4) / 4 drains accumulator stage g
    const int grp = (warp - 4) >> 2, q = warp & 3;
    const int r = q * 32 + lane;
    if (grp < AS) {
      uint32_t tph = 0;
      int wi = 0;
      for (int w = blockIdx.x; w < total; w += gridDim.x, ++wi) {
        if (wi % AS != grp) continue;
        int z, tx, ty, n;
        decode(w, z, tx, ty, n);
        const int OHs = grouped ? p.sub[z].OH : p.OH, OWs = grouped ? p.sub[z].OW : p.OW;
        const int oa = grouped ? p.sub[z].oa : p.oa, ob = grouped ? p.sub[z].ob : p.ob;
        mbar_wait(bar_tfull + 8 * grp, tph);
        tph ^= 1u;
        for (int m = 0; m < MT; ++m) {
          const int oy = ty * 16 * MT + 16 * m + (r >> 3), ox = tx * 8 + (r & 7);
          const bool valid = oy < OHs && ox < OWs;
          const size_t dpix = valid ? ((size_t)(n * p.DH + oy * p.osh + oa) * p.DW + ox * p.osw + ob) : 0;
          epi_row<BN>(p, acc_base + grp * acc_bytes + (uint32_t)r * 16 + (uint32_t)(m * BN) * kAccColBytes, 0, dpix, valid, s_bias);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_tempty + 8 * grp);
        if (q == 0 && lane == 0) CIS_TRACE_AT(12 + 5 * wi);
      }
    }
  }
}

// ======================================================================================================= wgrad
// D[co][kcol] = sum_pix g[pix][co] * A[pix][kcol]; both operands are "MN-major" (the reduction dim = pixels is the slow
// dimension of NHWC), staged as two [64 pixels][64 channels] SWIZZLE_128B sub-tiles each.
static constexpr int kWStages = 3;
static constexpr int kWTile = 64 * 128;            // one [64 pix][64 ch] bf16 sub-tile
static constexpr int kWStage = 4 * kWTile;         // A (2 sub-tiles) + B (2 sub-tiles)
static constexpr int kWSmem = kWStages * kWStage + 1024;

struct WgradMaps {
  CUtensorMap g;                 // (C8, OW, OH, N) gradient slice, box (64, 8, 8, 1)
  CUtensorMap x[CIS_MAX_SRC];    // (C8, W, H, N) activation slices, box (64, 8, 8, 1)
};

__global__ void __launch_bounds__(kGThreads) conv_wgrad_kernel(const __grid_constant__ CisWgrad p, const __grid_constant__ WgradMaps maps) {
  constexpr int S = kWStages;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t bars[2 * S + 1];
  __shared__ int s_dh[CIS_MAX_TAPS], s_dw[CIS_MAX_TAPS];
  const uint32_t tile_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_full = smem_u32(&bars[0]);
  const uint32_t bar_empty = smem_u32(&bars[S]);
  const uint32_t bar_accum = smem_u32(&bars[2 * S]);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // blockDim = producer/epilogue warps + 1 MMA warpgroup: 4 + 4 on the TMA operand path (one thread issues the loads), 8 + 4 on the
  // cp.async gather path, whose address arithmetic is the bottleneck (thin or strided layers)
  const int nprod = (int)blockDim.x - 128, mma_warp = nprod >> 5;
  pdl_launch_dependents();
  if (tid < p.ntaps) {
    s_dh[tid] = p.dh[tid];
    s_dw[tid] = p.dw[tid];
  }
  const int M = p.N * p.OH * p.OW;  // reduction length (pixels)
  int m_chunks = 0;
  for (int i = 0; i < p.nsrc; ++i) m_chunks += p.src[i].chunks;
  const int k_chunks = p.ntaps * m_chunks;
  const int tiles_x = (p.OW + 7) / 8, tiles_y = (p.OH + 7) / 8;
  const int nkb_total = p.tma ? p.N * tiles_x * tiles_y : (M + 63) / 64;   // TMA path: one K block = one 8x8 pixel tile
  const int per = (nkb_total + p.splits - 1) / p.splits;
  const int kb0 = blockIdx.y * per;
  const int kb1 = min(kb0 + per, nkb_total);
  const int nkb = kb1 - kb0;
  if (nkb <= 0) return;  // never taken: cis_conv_wgrad rejects split counts that leave a split without work (its slice would be garbage)

  if (tid == mma_warp * 32) {
    for (int s = 0; s < S; ++s) {
      mbar_init(bar_full + 8 * s, p.tma ? 1 : nprod);
      mbar_init(bar_empty + 8 * s, 1);
    }
    mbar_init(bar_accum, 128);
    fence_mbar_init();
  }
  pdl_wait();
  __syncthreads();

  if (warp < mma_warp) {
    if (p.tma) {
      if (tid == 0) {
        // two 64-column groups of this CTA: group = tap * nchunks64 + chunk64 -> (tap offset, source map, channel offset)
        const int nch64 = (m_chunks + 7) / 8;
        int gsrc[2], gc0[2], gdh[2], gdw[2], gnm[2];
        bool gok[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int grp = blockIdx.x * 2 + u;
          gok[u] = grp < p.ntaps * nch64;
          const int t = gok[u] ? grp / nch64 : 0;
          int c = gok[u] ? (grp - t * nch64) * 8 : 0, si = 0;
          while (si < p.nsrc - 1 && c >= p.src[si].chunks) {
            c -= p.src[si].chunks;
            ++si;
          }
          gsrc[u] = si;
          gc0[u] = c * 8;
          gdh[u] = s_dh[t];
          gdw[u] = s_dw[t];
          int nm = p.src[0].n_mod;
          if (si == 1) nm = p.src[1].n_mod;
          if (si == 2) nm = p.src[2].n_mod;
          if (si == 3) nm = p.src[3].n_mod;
          gnm[u] = nm;
        }
        const int tpi = tiles_x * tiles_y;
        for (int it = 0; it < nkb; ++it) {
          const int s = it % S;
          mbar_wait(bar_empty + 8 * s, (uint32_t)(((it / S) & 1) ^ 1));
          const int kb = kb0 + it;
          const int n = kb / tpi, r = kb - n * tpi;
          const int ty = r / tiles_x, tx = r - ty * tiles_x;
          const uint32_t st = tile_base + s * kWStage, bar = bar_full + 8 * s;
          mbar_expect_tx(bar, 4 * kWTile);
          tma_load_4d(st, &maps.g, bar, 0, tx * 8, ty * 8, n);
          tma_load_4d(st + kWTile, &maps.g, bar, 64, tx * 8, ty * 8, n);          // channels >= extent: zero fill
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int ne = gnm[u] ? (n % gnm[u]) : n;
            // an invalid group (beyond the last tap) reads channel 1<<20 -> fully out of range -> zeros
            tma_load_4d(st + (2 + u) * kWTile, &maps.x[gsrc[u]], bar, gok[u] ? gc0[u] : (1 << 20), tx * 8 + gdw[u], ty * 8 + gdh[u], ne);
          }
        }
      }
      __syncwarp();
    } else {
    const int j = tid & 7, rl = tid >> 3;
    const uint32_t sw_off = (uint32_t)((j ^ (rl & 7)) << 4);
    // fixed per-thread decode of the two B (activation) chunks and two A (gradient) chunks
    const __nv_bfloat16* bptr[2];
    int bpitch[2], bcoff[2], bnmod[2], bdh[2], bdw[2];
    bool bvalid[2], avalid[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int q = blockIdx.x * 16 + u * 8 + j;
      bvalid[u] = q < k_chunks;
      int t = 0, c = 0;
      if (bvalid[u]) {
        t = q / m_chunks;
        c = q - t * m_chunks;
      }
      int si = 0;
      while (si < p.nsrc - 1 && c >= p.src[si].chunks) {
        c -= p.src[si].chunks;
        ++si;
      }
      // static unrolled select keeps p.src[] accesses at constant indices
      CisSrc sd = p.src[0];
      if (si == 1) sd = p.src[1];
      if (si == 2) sd = p.src[2];
      if (si == 3) sd = p.src[3];
      bptr[u] = reinterpret_cast<const __nv_bfloat16*>(sd.ptr);
      bpitch[u] = sd.pitch;
      bcoff[u] = sd.c_off + c * 8;
      bnmod[u] = sd.n_mod;
      bdh[u] = s_dh[t];
      bdw[u] = s_dw[t];
      avalid[u] = (u * 8 + j) < p.g_chunks;
    }
    const __nv_bfloat16* gp = reinterpret_cast<const __nv_bfloat16*>(p.g);

    for (int it = 0; it < nkb; ++it) {
      const int s = it % S;
      const uint32_t ph = (uint32_t)((it / S) & 1);
      mbar_wait(bar_empty + 8 * s, ph ^ 1u);
      const uint32_t st = tile_base + s * kWStage;
#pragma unroll
      for (int r = rl; r < 64; r += nprod >> 3) {
        const int g = (kb0 + it) * 64 + r;
        const bool rv = g < M;
        int n = 0, h0 = 0, w0 = 0;
        if (rv) {
          const int ow = g % p.OW;
          const int t = g / p.OW;
          h0 = (t % p.OH) * p.sh;
          n = t / p.OH;
          w0 = ow * p.sw;
        }
        const uint32_t dst = st + r * 128 + sw_off;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const bool ok = rv && avalid[u];
          const size_t off = ok ? ((size_t)g * p.g_pitch + p.g_coff + (u * 8 + j) * 8) : 0;
          cp_async16(dst + u * kWTile, gp + off, ok ? 16u : 0u);
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int h = h0 + bdh[u], w = w0 + bdw[u];
          const bool ok = rv && bvalid[u] && (unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W;
          const int ne = bnmod[u] ? (n % bnmod[u]) : n;
          const size_t off = ok ? ((size_t)((ne * p.H + h) * p.W + w) * bpitch[u] + bcoff[u]) : 0;
          cp_async16(dst + (2 + u) * kWTile, bptr[u] + off, ok ? 16u : 0u);
        }
      }
      cp_async_commit();
      if (it >= S - 1) {
        cp_async_wait<S - 1>();
        fence_proxy_async();
        mbar_arrive(bar_full + 8 * ((it - (S - 1)) % S));
      }
    }
    cp_async_wait<0>();
    fence_proxy_async();
    for (int it = nkb > S - 1 ? nkb - (S - 1) : 0; it < nkb; ++it) mbar_arrive(bar_full + 8 * (it % S));

    }
    // epilogue: row = output channel co, columns = packed K columns of this n-tile
    mbar_wait(bar_accum, 0);
    const int co = (warp & 3) * 32 + lane;          // warps w and w + 4 share 32 accumulator rows and split the 128 columns
    const uint32_t t_row = tile_base + (uint32_t)co * 16;
    const int c_lo = mma_warp == 8 ? (warp >> 2) * 64 : 0, c_hi = mma_warp == 8 ? c_lo + 64 : 128;
    const int kcol0 = blockIdx.x * 128;
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 16) {
      float v[16];
      acc_ld16(t_row + (uint32_t)c0 * kAccColBytes, v);
      if (co < p.Cout && kcol0 + c0 < p.K_pad) {     // K_pad % 64 == 0: a 16-column group is inside or outside as a whole
        // this split's private slice, float4-COLUMN layout [K_pad / 4][Cout][4]: the warp's 32 consecutive output channels write 512
        // contiguous bytes per store (row-major [Cout][K_pad] made every store touch 32 lines, the LSU-bound pattern of the split-K slices)
        float4* o = reinterpret_cast<float4*>(p.dwp) + (size_t)blockIdx.y * p.Cout * (p.K_pad / 4) + (size_t)((kcol0 + c0) / 4) * p.Cout + co;
        o[0] = make_float4(v[0], v[1], v[2], v[3]);
        o[p.Cout] = make_float4(v[4], v[5], v[6], v[7]);
        o[2 * p.Cout] = make_float4(v[8], v[9], v[10], v[11]);
        o[3 * p.Cout] = make_float4(v[12], v[13], v[14], v[15]);
      }
    }
  } else {
    // ------------------------------------------------------------------ MMA warpgroup (both operands MN-major)
    const int wtid = tid - mma_warp * 32;
    float acc[128];
    for (int it = 0; it < nkb; ++it) {
      const int s = it % S;
      mbar_wait(bar_full + 8 * s, (uint32_t)((it / S) & 1));
      const uint32_t st = tile_base + s * kWStage;
      // 16 pixels (K) per MMA = 16 rows x 128 B; MN atoms (64 channels) are kWTile apart (LBO), 8-row K groups 1024 B (SBO)
      const uint32_t alo = desc_lo(st, kWTile), blo = desc_lo(st + 2 * kWTile, kWTile), dhi = desc_hi(1024);
      wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) mma128<128, 1, 1>(acc, alo + 128 * k, dhi, blo + 128 * k, dhi, (uint32_t)kWTile >> 4, (uint32_t)((it | k) != 0));
      wg_commit();
      wg_wait<0>();
      if (wtid == 0) mbar_arrive(bar_empty + 8 * s);
    }
    acc_store<128>(acc, tile_base, wtid);     // every operand stage has been consumed: the accumulator overlays the ring
    mbar_arrive(bar_accum);
  }
}


// ======================================================================================================= halo-resident wgrad
// CisWgrad.tma == 2.  Swapped roles: D[kcol][co] = sum_pix x[pix + tap][c] * g[pix][co].  Per 8x8 pixel tile the CTA fetches ONE activation halo
// ((8+ex) x (8+ey) pixels x 64 channels, TMA, SWIZZLE_128B) and the gradient tile(s) (8x8 pixels x NH channels) and reads every tap
// in place: A = MN-major operand whose two 64-channel atoms are the taps 2q and 2q+1 (descriptor start = origin of tap 2q shifted
// by two tile rows per K step, LBO = distance between the two tap origins, SBO = Wh*128 between the 8-pixel rows), B = the gradient
// tile (N = NH output channels), one 128 x NH register accumulator per tap pair.  Relies on the tensor core applying the swizzle
// on absolute address bits for MN-major operands too.
// NH = min(64, Cout rounded to 16) is the MMA N: the gradient tile is exactly one MN-major swizzle atom wide (NH * 2 bytes: 128B / 64B /
// 32B swizzle), so no zero channels are fetched or multiplied beyond the 16-channel granule.  Each MMA warpgroup holds P = 128 / NH tap
// pairs (128 accumulator registers).  NWG = 2 adds a second MMA warpgroup on the same stages: Cout > 64 -> warpgroup w takes Cout half w
// over the same P pairs (the stage holds both 64-channel gradient halves); Cout <= 64 -> the CTA owns 2P pairs, split between the two.
// grid = (64-channel chunks of the input, pixel-tile splits, pair groups [x 64-channel halves of Cout when one warpgroup]);
// dwp layout = [split][co][K_pad].
static constexpr int kWHMaxStages = 6;
struct WgradHaloMaps {
  CUtensorMap g;                 // (C8, OW, OH, N) gradient slice, box (NH, 8, 8, 1)
  CUtensorMap x[CIS_MAX_SRC];    // (C8, W, H, N) activation slices, box (64, Wh, Hh, 1)
};
template <int NH> struct WgradHaloCfg {
  static_assert(NH == 16 || NH == 32 || NH == 64, "NH is 16, 32 or 64 output channels");
  static constexpr int kPairs = kMaxAccCols / NH;                    // tap pairs per MMA warpgroup
  static constexpr uint32_t kGRow = 2 * NH;                          // bytes per pixel of the gradient tile = its swizzle span
  static constexpr uint32_t kGTile = 64 * kGRow;                     // 8x8 pixels
  static constexpr uint32_t kLayout = NH == 64 ? 1u : NH == 32 ? 2u : 3u;   // descriptor layout type: SWIZZLE_128B / 64B / 32B
};

// tap pairs [qa, qa + np) and Cout half hf of MMA warpgroup w
template <int NH, int NWG>
__device__ __forceinline__ void wgrad_halo_wg_pairs(int w, int npairs, int cout, int& qa, int& np, int& hf) {
  constexpr int P = WgradHaloCfg<NH>::kPairs;
  const int nhalf = cout > 64 ? 2 : 1;
  if (NWG == 2 && nhalf == 2) {
    qa = blockIdx.z * P;
    np = min(P, npairs - qa);
    hf = w;
    return;
  }
  const int q0 = (blockIdx.z / nhalf) * (NWG * P);
  const int cnt = min(NWG * P, npairs - q0);
  const int h = NWG == 2 ? (cnt + 1) / 2 : cnt;                       // two warpgroups: balanced halves of the CTA's pairs
  qa = q0 + (w ? h : 0);
  np = w ? cnt - h : h;
  hf = blockIdx.z % nhalf;
}

template <int NH, int NWG>
__global__ void __launch_bounds__(128 * (1 + NWG)) conv_wgrad_halo_kernel(const __grid_constant__ CisWgrad p, const __grid_constant__ WgradHaloMaps maps,
                                                                          const int Wh, const int Hh, const int hoy, const int hox,
                                                                          const int stage_bytes, const int S) {
  using Cfg = WgradHaloCfg<NH>;
  constexpr int P = Cfg::kPairs;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t bars[2 * kWHMaxStages + 1];
  __shared__ int s_off[CIS_MAX_TAPS + 1];   // tap origin inside the halo, in pixel rows of 128 B
  const uint32_t tile_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_full = smem_u32(&bars[0]);
  const uint32_t bar_empty = smem_u32(&bars[kWHMaxStages]);
  const uint32_t bar_accum = smem_u32(&bars[2 * kWHMaxStages]);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_launch_dependents();
  if (tid < p.ntaps) s_off[tid] = (p.dh[tid] - hoy) * Wh + (p.dw[tid] - hox);
  if (tid == p.ntaps) s_off[tid] = 0;       // partner of an unpaired last tap (its accumulator rows are never stored)
  const bool wg_halves = NWG == 2 && p.Cout > 64;              // warpgroup w multiplies by gradient half w
  const int ng = wg_halves ? 2 : 1;                            // gradient tiles per stage
  const int halo_bytes = stage_bytes - ng * (int)Cfg::kGTile;  // [halo (1024-rounded)] [gradient tile(s)]
  const int tiles_x = (p.OW + 7) / 8, tiles_y = (p.OH + 7) / 8;
  const int nkb_total = p.N * tiles_x * tiles_y;
  const int per = (nkb_total + (int)gridDim.y - 1) / (int)gridDim.y;
  const int kb0 = blockIdx.y * per;
  const int nkb = min(per, nkb_total - kb0);
  if (nkb <= 0) return;   // uniform per CTA: before any barrier
  int m_chunks = 0;
  for (int i = 0; i < p.nsrc; ++i) m_chunks += p.src[i].chunks;
  const int nch64 = (m_chunks + 7) / 8;
  const int npairs = (p.ntaps + 1) / 2;
  const int c64 = blockIdx.x;

  if (tid == 128) {
    for (int s = 0; s < S; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, NWG);      // one release per MMA warpgroup
    }
    mbar_init(bar_accum, 128 * NWG);
    fence_mbar_init();
  }
  pdl_wait();
  __syncthreads();

  if (warp < 4) {
    if (tid == 0) {
      // which concat source holds this 64-channel chunk (sources except the last are 64-channel aligned)
      int c = c64 * 8, si = 0;
      while (si < p.nsrc - 1 && c >= p.src[si].chunks) {
        c -= p.src[si].chunks;
        ++si;
      }
      int nm = p.src[0].n_mod;
      if (si == 1) nm = p.src[1].n_mod;
      if (si == 2) nm = p.src[2].n_mod;
      if (si == 3) nm = p.src[3].n_mod;
      int qa, np, hf0;
      wgrad_halo_wg_pairs<NH, NWG>(0, npairs, p.Cout, qa, np, hf0);
      const int tpi = tiles_x * tiles_y;
      for (int it = 0; it < nkb; ++it) {
        const int s = it % S;
        mbar_wait(bar_empty + 8 * s, (uint32_t)(((it / S) & 1) ^ 1));
        const int kb = kb0 + it;
        const int n = kb / tpi, r = kb - n * tpi;
        const int ty = r / tiles_x, tx = r - ty * tiles_x;
        const uint32_t st = tile_base + s * stage_bytes, bar = bar_full + 8 * s;
        mbar_expect_tx(bar, (uint32_t)(Wh * Hh * 128 + ng * (int)Cfg::kGTile));
        tma_load_4d(st, &maps.x[si], bar, c * 8, tx * 8 + hox, ty * 8 + hoy, nm ? (n % nm) : n);     // out-of-image pixels / channels: zeros
        for (int h = 0; h < ng; ++h)
          tma_load_4d(st + halo_bytes + h * Cfg::kGTile, &maps.g, bar, (hf0 + h) * 64, tx * 8, ty * 8, n);
      }
    }
    __syncwarp();
    // ---- epilogue: accumulator row r = (tap parity r / 64, input channel r % 64) of every tap pair; columns = output channels
    mbar_wait(bar_accum, 0);
    const int r = warp * 32 + lane;
    const int cch = r & 63;
    const uint32_t t_row = tile_base + (uint32_t)r * 16;
    for (int w = 0; w < NWG; ++w) {
      int qa, np, hf;
      wgrad_halo_wg_pairs<NH, NWG>(w, npairs, p.Cout, qa, np, hf);
      for (int q = 0; q < np; ++q) {
        const int t = 2 * (qa + q) + (r >> 6);
        if (t >= p.ntaps) continue;
        const size_t kcol = ((size_t)t * nch64 + c64) * 64 + cch;
#pragma unroll 1
        for (int c0 = 0; c0 < NH && hf * 64 + c0 < p.Cout; c0 += 16) {
          float v[16];
          acc_ld16(t_row + (uint32_t)((w * P + q) * NH + c0) * kAccColBytes, v);
          for (int e = 0; e < 16; ++e) {
            const int co = hf * 64 + c0 + e;
            if (co < p.Cout) p.dwp[((size_t)blockIdx.y * p.Cout + co) * p.K_pad + kcol] = v[e];   // private slice; lanes = consecutive kcol: coalesced
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ MMA warpgroup(s) (warps 4-7, 8-11)
    const int wg = NWG > 1 ? (warp - 4) >> 2 : 0;
    const int wtid = tid - 128 * (1 + wg);
    int qa, np, hf;
    wgrad_halo_wg_pairs<NH, NWG>(wg, npairs, p.Cout, qa, np, hf);
    // the pair count depends on the warpgroup: read it through a shuffle so that ptxas knows it is warp-uniform (a wgmma guard it
    // takes for divergent makes it serialise the wgmma, C7520)
    np = __shfl_sync(0xffffffffu, np, 0);
    float acc[P][NH];
    const uint32_t ahi = desc_hi((uint32_t)(Wh * 128));
    const uint32_t bhi = (((8 * Cfg::kGRow) >> 4) & 0x3FFF) | (Cfg::kLayout << 30);   // SBO = 8 gradient pixels
    const uint32_t kstep = (uint32_t)(2 * Wh * 128) >> 4;                    // 16 pixels = two tile rows of the halo
    const uint32_t g_off = (uint32_t)halo_bytes + (wg_halves ? (uint32_t)wg * Cfg::kGTile : 0u);
    for (int it = 0; it < nkb; ++it) {
      const int s = it % S;
      mbar_wait(bar_full + 8 * s, (uint32_t)((it / S) & 1));
      const uint32_t st = tile_base + s * stage_bytes;
      const uint32_t blo0 = desc_lo(st + g_off, Cfg::kGTile);       // LBO unused: the tile is one swizzle atom wide
      wg_fence();
#pragma unroll
      for (int q = 0; q < P; ++q) {
        if (q < np) {
          const int o0 = s_off[2 * (qa + q)], o1 = s_off[2 * (qa + q) + 1];
          const uint32_t lbo = (uint32_t)((o1 > o0 ? o1 - o0 : 1) * 128);      // distance between the two tap origins
          const uint32_t alo0 = desc_lo(st + (uint32_t)(o0 * 128), lbo);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            mma128<NH, 1, 1>(acc[q], alo0 + k * kstep, ahi, blo0 + Cfg::kGRow * k, bhi, lbo >> 4, (uint32_t)((it | k) != 0));
        }
      }
      wg_commit();
      // release the stage once its wgmma are done (keeping one commit group in flight and releasing the stage behind the next one
      // measured slower on the H100)
      wg_wait<0>();
      if (wtid == 0) mbar_arrive(bar_empty + 8 * s);
    }
    // every operand stage has been consumed: the accumulators overlay the ring.  Two warpgroups: the other one may still be reading
    // the last stage, so both finish their wgmma before either overwrites it.
    if constexpr (NWG > 1) asm volatile("bar.sync 1, %0;" ::"n"(128 * NWG) : "memory");
#pragma unroll
    for (int q = 0; q < P; ++q)
      if (q < np) acc_store<NH>(acc[q], tile_base + (uint32_t)((wg * P + q) * NH) * kAccColBytes, wtid);
    mbar_arrive(bar_accum);
  }
}

}  // namespace cis

using namespace cis;

// Launch with programmatic stream serialization so the kernel's prologue can overlap the previous kernel's tail (the kernels call
// griddepcontrol.wait before touching dependent memory).  CIS_PDL=0 disables it.
static bool pdl_enabled() {
  static const bool on = !(getenv("CIS_PDL") && atoi(getenv("CIS_PDL")) == 0);
  return on;
}
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// launch_pdl + a thread-block cluster along grid.z (the split-K CTAs of one tile)
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl_zcluster(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cz, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = cz;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

template <int BN>
static cudaError_t launch_splitk_finish(const CisConv* d, dim3 main_grid, cudaStream_t st) {
  constexpr int G = BN / 16;
  constexpr int kBlock = (128 * G < 256) ? 128 * G : 256;
  constexpr int kSub = 128 * G / kBlock;
  const int mt = d->halo ? d->MT * (d->nwg > 1 ? d->nwg : 1) : 1;
  return launch_pdl(splitk_finish_kernel<BN>, dim3(main_grid.x, main_grid.y, mt * kSub), dim3(kBlock), 0, st, *d);
}

template <int BN, int CPS>
static int launch_fwd_cps(const CisConv* d, cudaStream_t st) {
  using Cfg = FwdCfg<BN, CPS>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_igemm_kernel<BN, CPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem);
    if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaFuncSetAttribute(conv_igemm)");
    attr_set = true;
  }
  const int M = d->N * d->OH * d->OW;
  int splits = d->splits > 1 ? d->splits : 1;
  if (splits > 1) {
    const int nkb = d->K_pad / kBK, per = (nkb + splits - 1) / splits;
    if ((!d->sk_scratch && !d->sk_cluster) || d->sk_counters || (splits - 1) * per >= nkb || (d->sk_cluster && splits > 8))
      return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm: bad split-K setup");
  }
  dim3 grid((M + kBM - 1) / kBM, d->n_tiles, splits);
  cudaError_t le = (splits > 1 && d->sk_cluster)
                       ? launch_pdl_zcluster(conv_igemm_kernel<BN, CPS>, grid, dim3(kGThreads), Cfg::kSmem, st, splits, *d)
                       : launch_pdl(conv_igemm_kernel<BN, CPS>, grid, dim3(kGThreads), Cfg::kSmem, st, *d);
  if (le != cudaSuccess) return cis_set_cuda_error(le, "launch(conv_igemm)");
  if (splits > 1 && !d->sk_cluster) {
    le = launch_splitk_finish<BN>(d, grid, st);
    if (le != cudaSuccess) return cis_set_cuda_error(le, "launch(splitk_finish)");
  }
  return cis_check_launch("conv_igemm");
}
// BN = 64 grids of at most one CTA per SM run the CPS = 1 instance: nothing overlaps there, and the producers' main-loop register
// budget of the CPS = 2 instance costs time (H100 SXM at 700 W, 4x48x80, 96 input channels, 120 CTAs: 14.0 us at CPS = 1, 17.3 at 2)
template <int BN>
static int launch_fwd(const CisConv* d, cudaStream_t st) {
  const long ncta = (long)((d->N * d->OH * d->OW + kBM - 1) / kBM) * d->n_tiles * (d->splits > 1 ? d->splits : 1);
  if constexpr (BN == 64) {
    if (ncta <= cis_num_sms()) return launch_fwd_cps<BN, 1>(d, st);
  }
  return launch_fwd_cps<BN, BN == 128 ? 1 : 2>(d, st);
}


typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}
// (C, W, H, N) bf16 map of one concat source slice; box (64, bw, bh, 1), 128B swizzle, zero OOB fill.  step = 2 selects the
// space-to-depth phase (py, px) of the image: pixel (y, x) of the map is input pixel (2y + py, 2x + px).
// step/py/px: a stride-2 phase view (coarser grid through the global strides, phase offset in the base address).
// estride: dilated layers -- ONE map per source, every estride-th pixel of a box that starts at any (phase-carrying) coordinate.
// bc / swz: box width in channels and its swizzle (the halo wgrad kernel's narrow gradient tiles: 16 channels = 32 B, 32 = 64 B).
static bool encode_src_map(CUtensorMap* m, const CisSrc& s, int N, int H, int W, int bw, int bh, int step = 1, int py = 0, int px = 0,
                           int estride = 1, int bc = 64, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn enc = get_encode_tiled();
  if (!enc) return false;
  const int nb = s.n_mod > 0 ? s.n_mod : N;
  const int Hq = (H - py + step - 1) / step, Wq = (W - px + step - 1) / step;
  if (Hq < 1 || Wq < 1) return false;
  cuuint64_t dims[4] = {(cuuint64_t)s.chunks * 8, (cuuint64_t)Wq, (cuuint64_t)Hq, (cuuint64_t)nb};
  cuuint64_t strides[3] = {(cuuint64_t)step * s.pitch * 2, (cuuint64_t)step * W * s.pitch * 2, (cuuint64_t)H * W * s.pitch * 2};
  cuuint32_t box[4] = {(cuuint32_t)bc, (cuuint32_t)(bw * estride), (cuuint32_t)(bh * estride), 1};   // extent in the un-strided pixel space
  cuuint32_t es[4] = {1, (cuuint32_t)estride, (cuuint32_t)estride, 1};
  void* base = (void*)((const char*)s.ptr + ((size_t)(py * W + px) * s.pitch + (size_t)s.c_off) * 2);
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

#ifdef CIS_TRACE
extern "C" int cis_trace_set(unsigned long long* buf, int cap) {
  cudaError_t e = cudaMemcpyToSymbol(cis::g_trace, &buf, sizeof(buf));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(cis::g_trace_cap, &cap, sizeof(cap));
  return e == cudaSuccess ? CIS_OK : cis_set_cuda_error(e, "cis_trace_set");
}
#endif

static int g_persist_mode = -1;   // -1: environment / default (1 = thin layers)
extern "C" int cis_set_persist_mode(int mode) {
  g_persist_mode = mode;
  return CIS_OK;
}

// Largest dynamic shared memory (a multiple of 1 KB) with which two CTAs of `kernel` fit on one SM: half the SM's shared memory, less
// the per-CTA reservation and the kernel's static shared memory (H100: 228 KB per SM, 1 KB reserved -> 112 KB).
template <typename K>
static int pair_smem_limit(K kernel) {
  int dev = 0, per_sm = 0, reserved = 0;
  cudaFuncAttributes fa;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev) != cudaSuccess ||
      cudaFuncGetAttributes(&fa, kernel) != cudaSuccess)
    return 112 * 1024;
  return (per_sm / 2 - reserved - (int)fa.sharedSizeBytes) & ~1023;
}

// wk: NULL = the weights are cis_pack_weights_tiled tiles at d->wpack; else (compact format) d->wpack is a gather launch's row pack
// [n_tiles * BN][K_pad] and wk[2 s + j] the K column of kgroup j of step s (HaloMaps::wrow)
template <int BN, int NWG>
static int launch_halo(const CisConv* d, cudaStream_t st, const int16_t* wk = nullptr) {
  const int MTC = d->MT * NWG;                                 // stacked 16x8 tiles per CTA
  const int Wh = 8 + d->ex, Hh = 16 * MTC + d->ey, HP = Wh * Hh;
  const int thin = d->thin;
  const int nph = d->nph > 1 ? d->nph : 1;
  // compact format: the planes of every stride-2 phase share one stage
  const int halo_stage = ((thin ? nph * (thin / 8) * thin_plane_bytes(HP) : HP * 128) + 1023) & ~1023;
  int chunks = 0;
  for (int i = 0; i < d->nsrc; ++i) chunks += d->src[i].chunks;
  if (thin && ((thin != 8 && thin != 16) || chunks * 8 != thin || d->dil != 1))
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm(halo): the compact format needs 8 or 16 undilated input channels");
  const int nchunks = (chunks + 7) / 8;
  const int nsub = d->nsub > 1 ? d->nsub : 1;                  // grouped launch: grid.z = sub-problem, no split-K
  const int nsp = (nsub == 1 && d->splits > 1) ? d->splits : 1;
  const int cper = (nchunks + nsp - 1) / nsp;                  // 64-channel chunks per CTA
  const int nhs = cper > 1 ? 2 : 1;                            // halo stages: double-buffer only when there is a next chunk to prefetch
  const int dd = d->dil;
  int tiles = 0, ntaps_max = d->ntaps;
  if (nsub > 1) {
    if (nsub > 4 || dd != 1 || d->splits > 1 || d->nph > 1) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm(halo): bad grouped launch");
    ntaps_max = 0;
    int tsum = 0;
    for (int i = 0; i < nsub; ++i) {
      const int t = ((d->sub[i].OW + 7) / 8) * ((d->sub[i].OH + 16 * MTC - 1) / (16 * MTC));
      if (t > tiles) tiles = t;
      if (d->sub[i].ntaps > ntaps_max) ntaps_max = d->sub[i].ntaps;
      if (d->sub[i].ntaps < 1 || d->sub[i].tap0 != tsum || !d->sub[i].wpack) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm(halo): bad sub-problem");
      tsum += d->sub[i].ntaps;
    }
    if (tsum != d->ntaps) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm(halo): sub-problem taps must add up to ntaps");
  } else {
    const int Hp0 = (d->OH + dd - 1) / dd, Wp0 = (d->OW + dd - 1) / dd;
    tiles = ((Wp0 + 7) / 8) * ((Hp0 + 16 * MTC - 1) / (16 * MTC));
  }
  if (thin == 8) {
    // a K=16 step reads its second tap at a positive LBO from the first: every sub-problem (stride-2 phases: every phase, whose planes
    // follow the previous phase's) lists its taps in increasing halo offset
    for (int i = 0; i < nsub; ++i) {
      const int t0 = nsub > 1 ? d->sub[i].tap0 : 0, nt = nsub > 1 ? d->sub[i].ntaps : d->ntaps;
      for (int t = t0 + 1; t < t0 + nt; ++t)
        if (!(nph > 1 && (t == d->ph_tap[1] || t == d->ph_tap[2] || t == d->ph_tap[3])) &&
            d->dh[t] * (8 + d->ex) + d->dw[t] < d->dh[t - 1] * (8 + d->ex) + d->dw[t - 1])
          return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm(halo): compact 8-channel taps must be listed in increasing halo offset");
    }
  }
  const int nst_max = halo_nsteps(thin, ntaps_max);            // weight tiles (K=16 steps or taps) per chunk
  const long ncta_all = (long)tiles * dd * dd * d->N * d->n_tiles * nsp * nsub;
  // ---- weight pipeline: G taps per stage (one bulk copy, one wait / commit of the MMA thread), BS stages
  static const int g_env = getenv("CIS_HALO_G") ? atoi(getenv("CIS_HALO_G")) : 0;            // experiments: force the group size
  static const int stage_kb = getenv("CIS_HALO_STAGE_KB") ? atoi(getenv("CIS_HALO_STAGE_KB")) : 48;
  const int kB = thin ? BN * 32 : BN * 128;
  int G = g_env > 0 ? g_env : (stage_kb * 1024) / kB;
  if (G < 1) G = 1;
  if (G > nst_max) G = nst_max;
  const int fixed = nhs * halo_stage + HP * 4 + 1024;
  // two co-resident CTAs per SM (NWG = 1: HaloCfg's register budget) overlap one CTA's prologue and epilogue with the other's main
  // loop -- when the grid has that many CTAs and each takes at most half the SM's shared memory.  NWG = 2 CTAs hold the register file
  // alone; their launches keep the weight ring they were tuned with.
  static const int lim_pair = HaloCfg<BN, NWG>::kCtasPerSm == 2 ? pair_smem_limit(conv_halo_kernel<BN, NWG>) : 113 * 1024;
  static const int lim_small_kb = getenv("CIS_HALO_SMALL_KB") ? atoi(getenv("CIS_HALO_SMALL_KB")) : 226;   // grids of <= one CTA per SM
  static const int lim_kb_wide = getenv("CIS_HALO_LIMIT_KB") ? atoi(getenv("CIS_HALO_LIMIT_KB")) : 0;
  static const int lim_kb_thin = getenv("CIS_HALO_LIMIT_THIN_KB") ? atoi(getenv("CIS_HALO_LIMIT_THIN_KB")) : 0;   // BN <= 32
  const int lim_kb = BN <= 32 ? lim_kb_thin : lim_kb_wide;
  const int lim = lim_kb > 0 ? lim_kb * 1024 : lim_pair;
  const int nsm = cis_num_sms();
  int limit = (ncta_all > nsm && fixed + 2 * kB <= lim) ? lim : 226 * 1024;
  if (ncta_all <= nsm && fixed + 2 * kB <= lim_small_kb * 1024) limit = lim_small_kb * 1024;
  while (G > 1 && fixed + 2 * G * kB > limit) --G;
  const int groups = cper * ((nsub > 1 ? 1 : (nst_max + G - 1) / G));   // pipeline stages one CTA walks (grouped: at least one per chunk)
  int BS = (limit - fixed) / (G * kB);
  if (BS > (ncta_all > nsm ? 4 : kHaloMaxBStages)) BS = ncta_all > nsm ? 4 : kHaloMaxBStages;
  if (BS > groups) BS = groups;
  if (BS < 1) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_conv_igemm(halo): tile does not fit shared memory");
  int smem = fixed + BS * G * kB;
  if (smem < MTC * kBM * BN * 4 + 1024) smem = MTC * kBM * BN * 4 + 1024;   // the fp32 accumulator tiles overlay the operand buffers
  if (smem > 226 * 1024) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_conv_igemm(halo): accumulator tiles do not fit shared memory");
  static int attr_smem = 0;
  if (smem > attr_smem) {
    cudaError_t e = cudaFuncSetAttribute(conv_halo_kernel<BN, NWG>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaFuncSetAttribute(conv_halo)");
    attr_smem = smem;
  }

  int splits = d->splits > 1 ? d->splits : 1;
  if (splits > 1) {
    const int per = (nchunks + splits - 1) / splits;
    if ((!d->sk_scratch && !d->sk_cluster) || d->sk_counters || (splits - 1) * per >= nchunks || (d->sk_cluster && splits > 8))
      return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm(halo): bad split-K setup");
  }
  dim3 grid(tiles * dd * dd * d->N, d->n_tiles, nsub > 1 ? nsub : splits);
  // TMA halo path: undilated, every concat source except the last a multiple of 64 channels (a chunk never straddles sources)
  HaloMaps maps;
  static const int dil_tma = getenv("CIS_DIL_TMA") ? atoi(getenv("CIS_DIL_TMA")) : 1;
  int use_tma = ((d->dil == 1 || dil_tma) && Wh * d->dil <= 256 && Hh * d->dil <= 256) ? 1 : 0;
  for (int i = 0; use_tma && !thin && i < d->nsrc - 1; ++i)
    if (d->src[i].chunks % 8) use_tma = 0;
  for (int i = 0; use_tma && i < d->nsrc; ++i) {
    if (((uintptr_t)d->src[i].ptr + (size_t)d->src[i].c_off * 2) % 16) use_tma = 0;
    for (int ph = 0; use_tma && ph < nph; ++ph)
      if (!(thin ? encode_src_map(&maps.m[i * nph + ph], d->src[i], d->N, d->H, d->W, Wh, Hh, nph > 1 ? 2 : 1, ph >> 1, ph & 1, 1, 8,
                                  CU_TENSOR_MAP_SWIZZLE_NONE)
                 : encode_src_map(&maps.m[i * nph + ph], d->src[i], d->N, d->H, d->W, Wh, Hh, nph > 1 ? 2 : 1, ph >> 1, ph & 1, d->dil)))
        use_tma = 0;
  }
  if (!use_tma) memset(&maps, 0, sizeof(maps));
  if (thin && !use_tma) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_conv_igemm(halo): the compact format needs the TMA halo path");
  if (nph > 1 && !use_tma) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_conv_igemm(halo): stride-2 phases need the TMA halo path");
  maps.wrow = 0;
  if (wk) {
    EncodeTiledFn enc = get_encode_tiled();
    const cuuint64_t dims[2] = {(cuuint64_t)d->K_pad, (cuuint64_t)d->n_tiles * BN}, strides[1] = {(cuuint64_t)d->K_pad * 2};
    const cuuint32_t box[2] = {8, (cuuint32_t)BN}, es[2] = {1, 1};
    if (!thin || nsub > 1 || !enc ||
        enc(&maps.w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(d->wpack), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_conv_igemm(halo): row-pack weight map");
    maps.wrow = 1;
    memcpy(maps.wk, wk, sizeof(maps.wk));
  }
  // persistent variant (conv_halo_persist_kernel): layers with many tiles per SM.  CIS_PERSIST_MODE / cis_set_persist_mode:
  //   0 off | 1 (default) layers whose whole weight set stays resident in shared memory and that have >= 2 tiles per SM |
  //   2 every eligible layer (tests) | 3 every layer whose weight set fits, whatever the tile count (tests)
  const int persist_mode = g_persist_mode >= 0 ? g_persist_mode : (getenv("CIS_PERSIST_MODE") ? atoi(getenv("CIS_PERSIST_MODE")) : 1);
  static const int p_min_tiles = getenv("CIS_PERSIST_MIN_TILES") ? atoi(getenv("CIS_PERSIST_MIN_TILES")) : 296;
  static const int p_ws_kb = getenv("CIS_PERSIST_WS_KB") ? atoi(getenv("CIS_PERSIST_WS_KB")) : 112;
  if constexpr (BN <= kPMaxAccCols && NWG == 1) {
   // grouped launches (one chunk, whole weight set resident): the sub-problems' tiles form one work list.  Stride-2 phases: compact
   // format only (one halo stage holds every phase)
   if (persist_mode > 0 && use_tma && d->n_tiles == 1 && splits == 1 && (nph == 1 || thin) && (nsub == 1 || nchunks == 1) && dd == 1 &&
       d->MT * BN <= kPMaxAccCols) {
    int total = tiles * d->N, per_tile = nchunks * nst_max;
    if (nsub > 1) {
      total = per_tile = 0;
      for (int i = 0; i < nsub; ++i) {
        total += ((d->sub[i].OW + 7) / 8) * ((d->sub[i].OH + 16 * d->MT - 1) / (16 * d->MT)) * d->N;
        per_tile += halo_nsteps(thin, d->sub[i].ntaps);
      }
    }
    const int acc_stage = d->MT * BN * (int)kAccColBytes;           // one shared-memory accumulator stage
    const int AS = 2;
    const int fixed_p = AS * acc_stage + 1024;
    const int ws_bytes = per_tile * kB;
    int p_nhs = nchunks >= 3 ? 4 : 3;
    while (p_nhs > 2 && p_nhs * halo_stage + fixed_p + (ws_bytes <= p_ws_kb * 1024 ? ws_bytes : 2 * G * kB) > 226 * 1024) --p_nhs;
    const bool ws_fits = ws_bytes <= p_ws_kb * 1024 && p_nhs * halo_stage + fixed_p + ws_bytes <= 226 * 1024;
    const bool take = persist_mode == 2 || (persist_mode == 3 && ws_fits) || (persist_mode == 1 && ws_fits && total >= p_min_tiles);
    int p_bs = 0, p_smem = 0;
    if (ws_fits) {
      p_bs = 1;
      p_smem = p_nhs * halo_stage + fixed_p + ws_bytes;
    } else {
      p_bs = (226 * 1024 - p_nhs * halo_stage - fixed_p) / (G * kB);
      if (p_bs > 4) p_bs = 4;
      p_smem = p_nhs * halo_stage + fixed_p + p_bs * G * kB;
    }
    if (take && (ws_fits || nsub == 1) && p_bs >= (ws_fits ? 1 : 2)) {
      static int attr_p = 0;   // largest dynamic-smem limit set so far on conv_halo_persist_kernel<BN>
      if (p_smem > attr_p) {
        cudaError_t e = cudaFuncSetAttribute(conv_halo_persist_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, p_smem);
        if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaFuncSetAttribute(conv_halo_persist)");
        attr_p = p_smem;
      }
      int cps = 0;                 // co-resident persistent CTAs per SM (shared memory, registers, threads)
      cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cps, conv_halo_persist_kernel<BN>, kPThreads, p_smem);
      if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor(conv_halo_persist)");
      if (cps < 1) cps = 1;
      int g = total < nsm * cps ? total : nsm * cps;
      cudaError_t le = launch_pdl(conv_halo_persist_kernel<BN>, dim3(g), dim3(kPThreads), p_smem, st, *d, halo_stage, p_bs, p_nhs, AS, G, maps,
                                  ws_fits ? 1 : 0);
      if (le != cudaSuccess) return cis_set_cuda_error(le, "launch(conv_halo_persist)");
      return cis_check_launch("conv_halo_persist");
    }
   }
  }
  cudaError_t le = (splits > 1 && d->sk_cluster)
                       ? launch_pdl_zcluster(conv_halo_kernel<BN, NWG>, grid, dim3(HaloCfg<BN, NWG>::kThreads), smem, st, splits, *d, halo_stage, BS, nhs, maps,
                                             use_tma, G)
                       : launch_pdl(conv_halo_kernel<BN, NWG>, grid, dim3(HaloCfg<BN, NWG>::kThreads), smem, st, *d, halo_stage, BS, nhs, maps, use_tma, G);
  if (le != cudaSuccess) return cis_set_cuda_error(le, "launch(conv_halo)");
  if (splits > 1 && !d->sk_cluster) {
    le = launch_splitk_finish<BN>(d, grid, st);
    if (le != cudaSuccess) return cis_set_cuda_error(le, "launch(splitk_finish)");
  }
  return cis_check_launch("conv_halo");
}

// A stride-2 gather launch whose sources total 8 or 16 channels, as a compact phase-halo launch (CisConv.nph = 4): input pixel
// (2 oh + u, 2 ow + v) of tap (u, v) is pixel (oh + u / 2, ow + v / 2) of the space-to-depth phase (u & 1, v & 1) (floor division).
// The taps are listed phase by phase, each phase in the gather order (increasing (dy, dx), as the compact 8-channel pairs need), and
// wk gives the row-pack K column of every step's two kgroups: the row pack's K index is tap * cin8 + channel; the second kgroup of an odd
// last 8-channel step starts at K_pad, outside the map, which the TMA engine fills with zeros.  The tile stack MT follows the planner's wave model (engine.setup_halo_s2).  Returns false
// (the gather kernel runs the launch) where the halo path does not apply.
static bool s2_phase_plan(const CisConv* g, CisConv* h, int16_t* wk) {
  int chunks = 0;
  for (int i = 0; i < g->nsrc; ++i) {
    chunks += g->src[i].chunks;
    if (((uintptr_t)g->src[i].ptr + (size_t)g->src[i].c_off * 2) % 16) return false;
  }
  const int thin = chunks * 8, BN = g->BN;
  if (g->sh != 2 || g->sw != 2 || (thin != 8 && thin != 16) || g->splits > 1 || g->nsub > 1 || g->nph > 1 || g->dil > 1 || g->H < 2 ||
      g->W < 2 || BN > 128 || g->K_pad > 32767)
    return false;
  const int nt = g->ntaps;
  int order[CIS_MAX_TAPS], bounds[5] = {0, 0, 0, 0, 0}, k = 0;
  for (int q = 0; q < 4; ++q) {
    for (int t = 0; t < nt; ++t)
      if (((g->dh[t] & 1) << 1 | (g->dw[t] & 1)) == q) order[k++] = t;
    bounds[q + 1] = k;
  }
  int hoy = 1 << 20, hox = 1 << 20, ey = 0, ex = 0;
  for (int t = 0; t < nt; ++t) {
    hoy = min(hoy, g->dh[t] >> 1);
    hox = min(hox, g->dw[t] >> 1);
  }
  *h = *g;
  for (int i = 0; i < nt; ++i) {
    h->dh[i] = (int16_t)((g->dh[order[i]] >> 1) - hoy);
    h->dw[i] = (int16_t)((g->dw[order[i]] >> 1) - hox);
    ey = max(ey, (int)h->dh[i]);
    ex = max(ex, (int)h->dw[i]);
  }
  // MT: the planner's wave model for the compact format (weights through the TMA engine and halo bytes ~40 B/clk/SM, K=16 steps)
  const int nst = halo_nsteps(thin, nt), kb = BN * 32, tiles_x = (g->OW + 7) / 8, nsm = cis_num_sms();
  int best_mt = 0;
  double best = 0.0;
  for (int MT = 1; MT <= 4; ++MT) {
    if (MT * BN > kMaxAccCols || 8 + ex > 256 || 16 * MT + ey > 256) continue;
    const int HP = (8 + ex) * (16 * MT + ey);
    const int halo = (4 * (thin / 8) * thin_plane_bytes(HP) + 1023) & ~1023, smem = halo + HP * 4 + 2048 + 2 * kb;
    if (smem > 227 * 1024) continue;
    const int tiles_y = (g->OH + 16 * MT - 1) / (16 * MT);
    if ((double)g->OH * g->OW < 0.2 * tiles_y * 16 * MT * tiles_x * 8) continue;
    const long ncta = (long)g->N * tiles_x * tiles_y * g->n_tiles;
    const int cps = max(1, min(225 * 1024 / smem, 4));
    const double t_mma = MT * 2.0 * BN * nst * 0.25, t_mem = (double)kb * nst / 40.0 + halo / 40.0;
    const double t_cta = fmax(t_mma, t_mem) + (4000.0 + 1500.0 * MT) / cps;
    const double cost = (double)((ncta + (long)nsm * cps - 1) / ((long)nsm * cps)) * cps * t_cta / fmin((double)cps, fmax(1.0, (double)ncta / nsm));
    if (!best_mt || cost < best - 1e-9) {
      best = cost;
      best_mt = MT;
    }
  }
  // grids under the persistent kernel's 296 tiles run one short CTA per tile that fetches its own weights: there the gather kernel is
  // faster (64x112x4, 5x5 on 16 channels, H100 SXM at 700 W: 10.2 us against 17.9 us)
  if (!best_mt || (long)g->N * tiles_x * ((g->OH + 16 * best_mt - 1) / (16 * best_mt)) * g->n_tiles < 296) return false;
  h->halo = 1;
  h->sh = h->sw = 1;                   // the phases absorb the stride; H x W stay the input size (tensor maps)
  h->dil = 1;
  h->MT = best_mt;
  h->nwg = 1;
  h->hoy = hoy;
  h->hox = hox;
  h->ey = ey;
  h->ex = ex;
  h->nph = 4;
  for (int q = 0; q < 5; ++q) h->ph_tap[q] = bounds[q];
  h->thin = thin;
  h->splits = 0;
  h->sk_cluster = 0;
  for (int s = 0; s < nst; ++s)
    for (int j = 0; j < 2; ++j) {
      const int i = thin == 8 ? 2 * s + j : s;
      wk[2 * s + j] = (int16_t)(thin == 8 ? (i < nt ? order[i] * 8 : g->K_pad) : order[i] * 16 + 8 * j);
    }
  return true;
}
extern "C" int cis_conv_s2_phase_plan(const CisConv* d, CisConv* h, int16_t* wk) {
  return d && h && wk && !d->halo && s2_phase_plan(d, h, wk) ? 1 : 0;
}

extern "C" int cis_conv_igemm(const CisConv* d, cis_stream_t stream) {
  if (!d || d->ntaps < 1 || d->ntaps > CIS_MAX_TAPS || d->nsrc < 1 || d->nsrc > CIS_MAX_SRC || d->K_pad % 64 != 0 || d->K_pad <= 0 ||
      d->n_tiles < 1 || !d->wpack)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm: bad descriptor");
  int chunks = 0;
  for (int i = 0; i < d->nsrc; ++i) {
    if ((d->src[i].pitch | d->src[i].c_off) & 7) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm: source pitch/c_off must be multiples of 8");
    chunks += d->src[i].chunks;
  }
  if (d->ntaps * chunks * 8 > d->K_pad) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm: K_pad smaller than taps*channels");
  if (d->mode == 1 && !d->outf) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm: mode 1 needs outf");
  if ((d->add_pre || d->add_post) && (((d->add_pre_pitch | d->add_pre_coff | d->add_post_pitch | d->add_post_coff | d->out_ch) & 7) != 0))
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm: residual slices must be 8-channel aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (d->halo) {
    if (d->MT < 1 || d->MT > 4 || d->MT * d->BN > kMaxAccCols || d->nwg < 0 || d->nwg > 2 || (d->nwg == 2 && d->BN < 64) || d->dil < 1 ||
        d->sh != 1 || d->sw != 1 || d->ey < 0 || d->ex < 0 ||
        (d->dil > 1 && (d->OH != d->H || d->OW != d->W)) || (d->nph > 1 && (d->nph != 4 || d->dil != 1 || d->ph_tap[0] != 0 || d->ph_tap[4] != d->ntaps)))
      return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_igemm(halo): bad tile parameters");
    switch (d->BN) {
      case 16: return launch_halo<16, 1>(d, st);
      case 32: return launch_halo<32, 1>(d, st);
      case 64: return d->nwg == 2 ? launch_halo<64, 2>(d, st) : launch_halo<64, 1>(d, st);
      case 128: return d->nwg == 2 ? launch_halo<128, 2>(d, st) : launch_halo<128, 1>(d, st);
      default: return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_conv_igemm: BN must be 16/32/64/128");
    }
  }
  CisConv h;
  int16_t wk[2 * CIS_MAX_TAPS];
  if (s2_phase_plan(d, &h, wk)) {     // thin stride-2 launch: halo bytes ~1x the input tile instead of the gather's ~k*k/4x
    switch (h.BN) {
      case 16: return launch_halo<16, 1>(&h, st, wk);
      case 32: return launch_halo<32, 1>(&h, st, wk);
      case 64: return launch_halo<64, 1>(&h, st, wk);
      case 128: return launch_halo<128, 1>(&h, st, wk);
    }
  }
  switch (d->BN) {
    case 16: return launch_fwd<16>(d, st);
    case 32: return launch_fwd<32>(d, st);
    case 64: return launch_fwd<64>(d, st);
    case 128: return launch_fwd<128>(d, st);
    default: return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_conv_igemm: BN must be 16/32/64/128");
  }
}

template <int NH, int NWG>
static int launch_wgrad_halo_t(const CisWgrad* d, cudaStream_t st, int nch64, int Wh, int Hh, int hoy, int hox, int halo_bytes) {
  using Cfg = WgradHaloCfg<NH>;
  const bool wg_halves = NWG == 2 && d->Cout > 64;
  const int stage = halo_bytes + (wg_halves ? 2 : 1) * (int)Cfg::kGTile;
  const int npairs = (d->ntaps + 1) / 2, nhalf = d->Cout > 64 ? 2 : 1;
  const int gz = wg_halves ? (npairs + Cfg::kPairs - 1) / Cfg::kPairs : nhalf * ((npairs + NWG * Cfg::kPairs - 1) / (NWG * Cfg::kPairs));
  int S = (200 * 1024) / stage;
  if (S > kWHMaxStages) S = kWHMaxStages;
  if (S < 2) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_conv_wgrad(halo): halo does not fit shared memory");
  int smem = S * stage + 1024;
  const int acc_smem = NWG * kMaxAccCols * (int)kAccColBytes + 1024;    // the accumulators overlay the stages
  if (smem < acc_smem) smem = acc_smem;
  static int attr_smem = 0;    // per instantiation
  if (smem > attr_smem) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgrad_halo_kernel<NH, NWG>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaFuncSetAttribute(conv_wgrad_halo)");
    attr_smem = smem;
  }
  WgradHaloMaps maps;
  memset(&maps, 0, sizeof(maps));
  CisSrc gs;
  gs.ptr = d->g; gs.pitch = d->g_pitch; gs.c_off = d->g_coff; gs.chunks = d->g_chunks; gs.n_mod = 0;
  const CUtensorMapSwizzle gswz = NH == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : NH == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
  bool ok = encode_src_map(&maps.g, gs, d->N, d->OH, d->OW, 8, 8, 1, 0, 0, 1, NH, gswz);
  for (int i = 0; ok && i < d->nsrc; ++i) ok = encode_src_map(&maps.x[i], d->src[i], d->N, d->H, d->W, Wh, Hh);
  if (!ok) return cis_set_error(CIS_ERR_CUDA, "cis_conv_wgrad(halo): cuTensorMapEncodeTiled failed / unavailable");
  dim3 grid(nch64, d->splits, gz);
  cudaError_t le = launch_pdl(conv_wgrad_halo_kernel<NH, NWG>, grid, dim3(128 * (1 + NWG)), (size_t)smem, st, *d, maps, Wh, Hh, hoy, hox, stage, S);
  if (le != cudaSuccess) return cis_set_cuda_error(le, "launch(conv_wgrad_halo)");
  return cis_check_launch("conv_wgrad_halo");
}

// Halo-resident swapped wgrad (CisWgrad.tma == 2).  Eligibility is re-checked here; the engine falls back to tma = 1.
static int launch_wgrad_halo(const CisWgrad* d, cudaStream_t st) {
  if (d->sh != 1 || d->sw != 1) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_wgrad(halo): needs a stride-1 layer");
  int chunks = 0;
  for (int i = 0; i < d->nsrc; ++i) chunks += d->src[i].chunks;
  for (int i = 0; i < d->nsrc - 1; ++i)
    if (d->src[i].chunks % 8) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_wgrad(halo): needs 64-channel aligned concat sources");
  const int nch64 = (chunks + 7) / 8;
  int hoy = d->dh[0], hox = d->dw[0], my = d->dh[0], mx = d->dw[0];
  for (int t = 1; t < d->ntaps; ++t) {
    if (d->dh[t] < hoy) hoy = d->dh[t];
    if (d->dw[t] < hox) hox = d->dw[t];
    if (d->dh[t] > my) my = d->dh[t];
    if (d->dw[t] > mx) mx = d->dw[t];
  }
  for (int t = 1; t < d->ntaps; ++t)    // pairs (2q, 2q+1) need increasing origins: taps are listed row-major
    if ((d->dh[t] - hoy) * 1024 + (d->dw[t] - hox) <= (d->dh[t - 1] - hoy) * 1024 + (d->dw[t - 1] - hox))
      return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_wgrad(halo): taps must be listed in increasing row-major order");
  const int Wh = 8 + (mx - hox), Hh = 8 + (my - hoy);
  if (Wh > 256 || Hh > 256) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_conv_wgrad(halo): tap extent too large");
  if (d->K_pad < d->ntaps * nch64 * 64) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_wgrad(halo): K_pad smaller than taps * 64-channel groups");
  const int nh = d->nh ? d->nh : 64, nwg = d->nwg ? d->nwg : 1;
  if ((nh != 16 && nh != 32 && nh != 64) || nh < (d->Cout > 64 ? 64 : (d->Cout + 15) / 16 * 16) || nwg < 1 || nwg > 2)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_wgrad(halo): nh must be 16/32/64 and cover Cout (64 above 64), nwg 1 or 2");
  const int halo_bytes = (Wh * Hh * 128 + 1023) & ~1023;
  switch (nh * 4 + nwg) {
    case 16 * 4 + 1: return launch_wgrad_halo_t<16, 1>(d, st, nch64, Wh, Hh, hoy, hox, halo_bytes);
    case 16 * 4 + 2: return launch_wgrad_halo_t<16, 2>(d, st, nch64, Wh, Hh, hoy, hox, halo_bytes);
    case 32 * 4 + 1: return launch_wgrad_halo_t<32, 1>(d, st, nch64, Wh, Hh, hoy, hox, halo_bytes);
    case 32 * 4 + 2: return launch_wgrad_halo_t<32, 2>(d, st, nch64, Wh, Hh, hoy, hox, halo_bytes);
    case 64 * 4 + 1: return launch_wgrad_halo_t<64, 1>(d, st, nch64, Wh, Hh, hoy, hox, halo_bytes);
    default: return launch_wgrad_halo_t<64, 2>(d, st, nch64, Wh, Hh, hoy, hox, halo_bytes);
  }
}

extern "C" int cis_conv_wgrad(const CisWgrad* d, cis_stream_t stream) {
  if (!d || d->ntaps < 1 || d->ntaps > CIS_MAX_TAPS || d->nsrc < 1 || d->nsrc > CIS_MAX_SRC || d->K_pad % 64 != 0 || d->Cout < 1 ||
      d->Cout > 128 || d->splits < 1 || !d->g || !d->dwp)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_wgrad: bad descriptor");
  {
    // every split must own at least one reduction block: its private slice of dwp is only defined if the CTA runs
    const long M = (long)d->N * d->OH * d->OW;
    const long nkb_total = d->tma ? (long)d->N * ((d->OW + 7) / 8) * ((d->OH + 7) / 8) : (M + 63) / 64;
    const long per = (nkb_total + d->splits - 1) / d->splits;
    if ((long)(d->splits - 1) * per >= nkb_total) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_wgrad: a split would own no reduction block");
  }
  if (d->tma == 2) return launch_wgrad_halo(d, (cudaStream_t)stream);
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWSmem);
    if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaFuncSetAttribute(conv_wgrad)");
    attr_set = true;
  }
  WgradMaps maps;
  memset(&maps, 0, sizeof(maps));
  if (d->tma) {
    if (d->sh != 1 || d->sw != 1) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_wgrad: TMA path needs a stride-1 layer");
    for (int i = 0; i < d->nsrc - 1; ++i)
      if (d->src[i].chunks % 8) return cis_set_error(CIS_ERR_BAD_ARG, "cis_conv_wgrad: TMA path needs 64-channel aligned concat sources");
    CisSrc gs;
    gs.ptr = d->g; gs.pitch = d->g_pitch; gs.c_off = d->g_coff; gs.chunks = d->g_chunks; gs.n_mod = 0;
    bool ok = encode_src_map(&maps.g, gs, d->N, d->OH, d->OW, 8, 8);
    for (int i = 0; ok && i < d->nsrc; ++i) ok = encode_src_map(&maps.x[i], d->src[i], d->N, d->H, d->W, 8, 8);
    if (!ok) return cis_set_error(CIS_ERR_CUDA, "cis_conv_wgrad: cuTensorMapEncodeTiled failed / unavailable");
  }
  dim3 grid((d->K_pad + 127) / 128, d->splits);
  cudaError_t le = launch_pdl(conv_wgrad_kernel, grid, dim3(d->tma ? kThreads : kGThreads), kWSmem, (cudaStream_t)stream, *d, maps);
  if (le != cudaSuccess) return cis_set_cuda_error(le, "launch(conv_wgrad)");
  return cis_check_launch("conv_wgrad");
}
