// HBM-bound kernels of the hot path: parameter packing, activation-gradient helpers, TF-1.13 resampling ops, the fused
// PWC-Net warp + cost volume, the fused mask (x) flow + Charbonnier loss, and clip + TF-Adam.
// Reference call sites are cited per kernel; semantics follow SURVEY.md Appendix A.
#include "ptx.cuh"
#include "../../include/cis_b200.h"
#include "common.cuh"
#include <math.h>

namespace cis {

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  f[0] = bf16lo(u.x); f[1] = bf16hi(u.x); f[2] = bf16lo(u.y); f[3] = bf16hi(u.y);
  f[4] = bf16lo(u.z); f[5] = bf16hi(u.z); f[6] = bf16lo(u.w); f[7] = bf16hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------ weights
// The five parameter-space ops (BN fold, two weight packs, gradient un-pack, BN chain rule) exist as single launches AND as one
// multi-job launch (cis_param_multi): blockIdx.y selects a job from a device-side table, so the ~75 per-layer launches that follow
// every optimiser step and the ~35 that end every backward pass become a handful.
__device__ __forceinline__ void pack_weights_body(size_t i, const float* __restrict__ w, const int* __restrict__ kmap, int K_pad, int rows, int cout,
                                                  int sn, const int* __restrict__ nmap, bf16* __restrict__ wp) {
  if (i >= (size_t)rows * K_pad) return;
  const int n = (int)(i / K_pad), k = (int)(i % K_pad);
  const int km = kmap[k];
  const int ne = nmap ? nmap[n] : (n < cout ? n : -1);
  const float v = (km >= 0 && ne >= 0) ? w[(size_t)km + (size_t)ne * sn] : 0.f;
  wp[i] = __float2bfloat16(v);
}
// Pre-swizzled weight tiles for the halo kernel: block (ny, cc, t) = BN rows x 128 B, row n holds K = 64 channels of chunk cc for
// tap t with the SWIZZLE_128B pattern already applied (16-byte chunk index ^= n & 7), so a plain bulk copy lands the wgmma operand layout.
__device__ __forceinline__ void pack_weights_tiled_body(size_t i, const float* __restrict__ w, const int* __restrict__ kmap, int cin8, int ntaps,
                                                        int n_tiles, int BN, int cout, int sn, const int* __restrict__ nmap,
                                                        bf16* __restrict__ out) {
  const int nchunks = (cin8 + 63) / 64;
  const size_t total = (size_t)n_tiles * nchunks * ntaps * BN * 64;
  if (i >= total) return;
  const int pos = (int)(i % 64);            // physical element position inside the 128-byte row
  size_t r = i / 64;
  const int n = (int)(r % BN); r /= BN;
  const int t = (int)(r % ntaps); r /= ntaps;
  const int cc = (int)(r % nchunks);
  const int ny = (int)(r / nchunks);
  const int kk = (((pos >> 3) ^ (n & 7)) << 3) | (pos & 7);   // logical channel within the chunk
  const int c = cc * 64 + kk;
  float v = 0.f;
  if (c < cin8) {
    const int km = kmap[t * cin8 + c];
    const int ng = ny * BN + n;
    const int ne = nmap ? nmap[ng] : (ng < cout ? ng : -1);
    if (km >= 0 && ne >= 0) v = w[(size_t)km + (size_t)ne * sn];
  }
  out[i] = __float2bfloat16(v);
}
// Forward orientation (sn == 1: the fp32 master weights are HWIO, output channel fastest): one block per (ny, cc, t) tile of BN x 64
// elements, read along n (contiguous in HWIO), transposed through shared memory, written along k (contiguous in the tile).  The flat
// form above reads a column of the [tap*cin][cout] matrix per warp: 4 useful bytes per 32-byte sector.  tile: >= 64 * (BN + 1) floats.
__device__ __forceinline__ void pack_weights_tiled_tile(int blk, const float* __restrict__ w, const int* __restrict__ kmap, int cin8, int ntaps,
                                                        int n_tiles, int BN, int cout, const int* __restrict__ nmap, bf16* __restrict__ out,
                                                        float* tile) {
  const int nchunks = (cin8 + 63) / 64;
  const int t = blk % ntaps;
  const int r = blk / ntaps;
  const int cc = r % nchunks, ny = r / nchunks;
  const int ld = BN + 1;
  for (int idx = threadIdx.x; idx < BN * 64; idx += blockDim.x) {
    const int n = idx % BN, kk = idx / BN;
    const int c = cc * 64 + kk;
    float v = 0.f;
    if (c < cin8) {
      const int km = kmap[t * cin8 + c];
      const int ng = ny * BN + n;
      const int ne = nmap ? nmap[ng] : (ng < cout ? ng : -1);
      if (km >= 0 && ne >= 0) v = w[(size_t)km + ne];
    }
    tile[kk * ld + n] = v;
  }
  __syncthreads();
  bf16* o = out + (size_t)blk * BN * 64;
  for (int idx = threadIdx.x; idx < BN * 64; idx += blockDim.x) {
    const int pos = idx & 63, n = idx >> 6;
    const int kk = (((pos >> 3) ^ (n & 7)) << 3) | (pos & 7);
    o[idx] = __float2bfloat16(tile[kk * ld + n]);
  }
}
// Compact (thin = 8 / 16 input channels) tiles of the halo kernel: block (ny, step s) = BN x 32 B, the no-swizzle K-major operand of
// one K=16 step.  Element (n, kgroup j, e) at ((n / 8) * 2 + j) * 64 + (n % 8) * 8 + e; kgroup j is tap 2s + j, channel e (thin 8) or
// tap s, channel 8j + e (thin 16).  i >= the tile set's size returns (the job's block count is that of the 64-channel layout).
__device__ __forceinline__ void pack_weights_thin_body(size_t i, const float* __restrict__ w, const int* __restrict__ kmap, int cin8, int ntaps,
                                                       int n_tiles, int BN, int cout, int sn, const int* __restrict__ nmap, int thin,
                                                       bf16* __restrict__ out) {
  const int nst = thin == 8 ? (ntaps + 1) / 2 : ntaps;
  if (i >= (size_t)n_tiles * nst * BN * 16) return;
  const int e = (int)(i % 8);
  const int n8 = (int)((i / 8) % 8);
  const int j = (int)((i / 64) % 2);
  size_t r = i / 128;
  const int ng8 = (int)(r % (BN / 8));
  r /= BN / 8;
  const int s = (int)(r % nst), ny = (int)(r / nst);
  const int t = thin == 8 ? 2 * s + j : s, c = thin == 8 ? e : 8 * j + e;
  float v = 0.f;
  if (t < ntaps && c < cin8) {
    const int km = kmap[t * cin8 + c];
    const int ng = ny * BN + ng8 * 8 + n8;
    const int ne = nmap ? nmap[ng] : (ng < cout ? ng : -1);
    if (km >= 0 && ne >= 0) v = w[(size_t)km + (size_t)ne * sn];
  }
  out[i] = __float2bfloat16(v);
}
__device__ __forceinline__ void unpack_wgrad_body(size_t i, const float* __restrict__ dwp, const int* __restrict__ kmap, int K_pad, int cout,
                                                  int nsplit, float* __restrict__ dw, const float* __restrict__ colpart, int nblocks, int nch,
                                                  float* __restrict__ db, int layout) {
  const size_t nw = (size_t)cout * K_pad;
  if (i < nw) {
    // slice element i -> (output channel n, packed column k): layout 0 = [cout][K_pad] (halo-resident wgrad), layout 1 = float4 columns
    // [K_pad / 4][cout][4] (gather / TMA-tile wgrad kernels).  Bits 8+ of layout: stride of n in dw (0 = 1, the HWIO slot; Cin for the
    // [kh,kw,Cout,Cin] slot of a transposed conv)
    const size_t sn = (layout >> 8) ? (size_t)(layout >> 8) : 1;
    int n, k;
    if ((layout & 0xff) == 0) {
      n = (int)(i / K_pad);
      k = (int)(i % K_pad);
    } else {
      const size_t g4 = i / ((size_t)cout * 4);
      const int rem = (int)(i - g4 * cout * 4);
      n = rem >> 2;
      k = (int)g4 * 4 + (rem & 3);
    }
    const int km = kmap[k];
    if (km < 0) return;
    // fixed-order sum of the private split-K slices; 8 independent loads in flight per thread
    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const float* q = dwp + i;
    int s = 0;
    for (; s + 8 <= nsplit; s += 8) {
      float t[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) t[u] = __ldcg(q + (size_t)(s + u) * nw);
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] += t[u];
    }
    for (; s < nsplit; ++s) a[0] += __ldcg(q + (size_t)s * nw);
    dw[(size_t)km + n * sn] = ((a[0] + a[1]) + (a[2] + a[3])) + ((a[4] + a[5]) + (a[6] + a[7]));
  } else if (colpart != nullptr && i - nw < (size_t)nch) {
    const int c = (int)(i - nw);
    float a = 0.f;
    for (int b = 0; b < nblocks; ++b) a += __ldcg(colpart + (size_t)b * nch + c);
    db[c] = a;
  }
}
#define BN_RSQRT 0.99950037468777323f /* 1/sqrt(1 + 1e-3): tf.layers.batch_normalization defaults, convolution_utils.py:50 */
__device__ __forceinline__ void bn_fold_body(size_t i, const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ gamma,
                                             const float* __restrict__ beta, size_t nw, int cout, float* __restrict__ w_eff,
                                             float* __restrict__ b_eff) {
  if (i < nw) w_eff[i] = w[i] * gamma[i % cout] * BN_RSQRT;
  if (i < (size_t)cout) b_eff[i] = bias[i] * gamma[i] * BN_RSQRT + beta[i];
}
// one 256-thread block per 8 output channels: thread = (channel co0 + tid % 8, row lane tid / 8), so a row of 8 channels is one 32-byte
// sector and every byte fetched is used (one block per channel walking a column of the [rows][cout] matrix would use 4 bytes of every
// 32-byte sector).  Fixed summation order.
static constexpr int kBnChainCo = 8;
__device__ __forceinline__ void bn_chain_body(int blk, const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ gamma,
                                              float* __restrict__ dwe, const float* __restrict__ dbe, size_t nw, int cout,
                                              float* __restrict__ dbias, float* __restrict__ dgamma, float* __restrict__ dbeta, float* red) {
  const int rows = (int)(nw / cout);
  const int cl = threadIdx.x & 7, rl = threadIdx.x >> 3;          // 8 channels x 32 row lanes
  const int co = blk * kBnChainCo + cl;
  const bool ok = co < cout;
  float acc = 0.f;
  if (ok)
    for (int r = rl; r < rows; r += 32) acc += dwe[(size_t)r * cout + co] * w[(size_t)r * cout + co];
  red[rl * 8 + cl] = acc;
  __syncthreads();
  float g = 0.f;
  if (ok) {
    g = gamma[co] * BN_RSQRT;
    if (rl == 0) {
      float v = 0.f;
      for (int q = 0; q < 32; ++q) v += red[q * 8 + cl];
      dgamma[co] = BN_RSQRT * (v + dbe[co] * bias[co]);
      dbias[co] = dbe[co] * g;
      dbeta[co] = dbe[co];
    }
    for (int r = rl; r < rows; r += 32) dwe[(size_t)r * cout + co] *= g;
  }
}
__global__ void pack_weights_kernel(const float* __restrict__ w, const int* __restrict__ kmap, int K_pad, int rows, int cout, int sn,
                                    const int* __restrict__ nmap, bf16* __restrict__ wp) {
  pdl_launch_dependents();
  pdl_wait();
  pack_weights_body((size_t)blockIdx.x * blockDim.x + threadIdx.x, w, kmap, K_pad, rows, cout, sn, nmap, wp);
}
__global__ void pack_weights_tiled_kernel(const float* __restrict__ w, const int* __restrict__ kmap, int cin8, int ntaps, int n_tiles, int BN,
                                          int cout, int sn, const int* __restrict__ nmap, bf16* __restrict__ out, int thin) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float tile[64 * 129];
  if (thin) pack_weights_thin_body((size_t)blockIdx.x * blockDim.x + threadIdx.x, w, kmap, cin8, ntaps, n_tiles, BN, cout, sn, nmap, thin, out);
  else if (sn == 1) pack_weights_tiled_tile(blockIdx.x, w, kmap, cin8, ntaps, n_tiles, BN, cout, nmap, out, tile);
  else pack_weights_tiled_body((size_t)blockIdx.x * blockDim.x + threadIdx.x, w, kmap, cin8, ntaps, n_tiles, BN, cout, sn, nmap, out);
}
__global__ void unpack_wgrad_kernel(const float* __restrict__ dwp, const int* __restrict__ kmap, int K_pad, int cout, int nsplit,
                                    float* __restrict__ dw, const float* __restrict__ colpart, int nblocks, int nch, float* __restrict__ db,
                                    int layout) {
  pdl_launch_dependents();
  pdl_wait();
  unpack_wgrad_body((size_t)blockIdx.x * blockDim.x + threadIdx.x, dwp, kmap, K_pad, cout, nsplit, dw, colpart, nblocks, nch, db, layout);
}
__global__ void bn_fold_kernel(const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ gamma,
                               const float* __restrict__ beta, size_t nw, int cout, float* __restrict__ w_eff, float* __restrict__ b_eff) {
  pdl_launch_dependents();
  pdl_wait();
  bn_fold_body((size_t)blockIdx.x * blockDim.x + threadIdx.x, w, bias, gamma, beta, nw, cout, w_eff, b_eff);
}
__global__ void bn_chain_kernel(const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ gamma,
                                float* __restrict__ dwe, const float* __restrict__ dbe, size_t nw, int cout, float* __restrict__ dbias,
                                float* __restrict__ dgamma, float* __restrict__ dbeta) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[256];
  bn_chain_body(blockIdx.x, w, bias, gamma, dwe, dbe, nw, cout, dbias, dgamma, dbeta, red);
}
// multi-job form: a flat 1-D grid; job j owns blocks [jobs[j].i[7], jobs[j+1].i[7]) (binary search), fields in the argument order of the
// single-launch entry points
__global__ void param_multi_kernel(const CisParamJob* __restrict__ jobs, int njobs) {
  pdl_launch_dependents();
  pdl_wait();
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {                       // last job whose first block is <= blockIdx.x
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].i[7] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const CisParamJob j = jobs[lo];
  const int blk = (int)blockIdx.x - j.i[7];
  const size_t i = (size_t)blk * blockDim.x + threadIdx.x;
  __shared__ float red[256];
  __shared__ float tile[64 * 129];
  switch (j.kind) {
    case CIS_JOB_PACK:
      pack_weights_body(i, (const float*)j.p[0], (const int*)j.p[1], j.i[0], j.i[1], j.i[2], j.i[3], (const int*)j.p[2], (bf16*)j.p[3]);
      break;
    case CIS_JOB_PACK_TILED:
      if (j.i[6]) {          // compact thin-input tiles (a fraction of the 64-channel layout the job's blocks are counted for)
        const size_t per = j.i[5] == 1 ? (size_t)j.i[3] * 64 : blockDim.x;
        for (size_t q = threadIdx.x; q < per; q += blockDim.x)
          pack_weights_thin_body((size_t)blk * per + q, (const float*)j.p[0], (const int*)j.p[1], j.i[0], j.i[1], j.i[2], j.i[3], j.i[4], j.i[5],
                                 (const int*)j.p[2], j.i[6], (bf16*)j.p[3]);
      } else if (j.i[5] == 1)       // forward orientation: one block per tile, transposed through shared memory
        pack_weights_tiled_tile(blk, (const float*)j.p[0], (const int*)j.p[1], j.i[0], j.i[1], j.i[2], j.i[3], j.i[4], (const int*)j.p[2],
                                (bf16*)j.p[3], tile);
      else
        pack_weights_tiled_body(i, (const float*)j.p[0], (const int*)j.p[1], j.i[0], j.i[1], j.i[2], j.i[3], j.i[4], j.i[5], (const int*)j.p[2],
                                (bf16*)j.p[3]);
      break;
    case CIS_JOB_UNPACK:
      unpack_wgrad_body(i, (const float*)j.p[0], (const int*)j.p[1], j.i[0], j.i[1], j.i[2], (float*)j.p[2], (const float*)j.p[3], j.i[3], j.i[4],
                        (float*)j.p[4], j.i[5]);
      break;
    case CIS_JOB_BN_FOLD:
      bn_fold_body(i, (const float*)j.p[0], (const float*)j.p[1], (const float*)j.p[2], (const float*)j.p[3], (size_t)j.n, j.i[0], (float*)j.p[4],
                   (float*)j.p[5]);
      break;
    case CIS_JOB_BN_CHAIN:      // one block per 8 output channels; the host gives the job exactly ceil(cout / 8) blocks
      bn_chain_body(blk, (const float*)j.p[0], (const float*)j.p[1], (const float*)j.p[2], (float*)j.p[3], (const float*)j.p[4], (size_t)j.n,
                    j.i[0], (float*)j.p[5], (float*)j.p[6], (float*)j.p[7], red);
      break;
  }
}

// ------------------------------------------------------------------------------------------------ gradient helpers
__global__ void dact_mul_kernel(bf16* g, int gp, int gc, const bf16* __restrict__ y, int yp, int yc, const bf16* __restrict__ res, int rp,
                                int rc, size_t npix, int chunks, int act, float alpha) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * chunks) return;
  const size_t pix = i / chunks;
  const int c = (int)(i % chunks) * 8;
  uint4* gpp = reinterpret_cast<uint4*>(g + pix * gp + gc + c);
  float gv[8], yv[8], rv[8];
  unpack8(*gpp, gv);
  unpack8(*reinterpret_cast<const uint4*>(y + pix * yp + yc + c), yv);
  if (res) {
    unpack8(*reinterpret_cast<const uint4*>(res + pix * rp + rc + c), rv);
#pragma unroll
    for (int e = 0; e < 8; ++e) yv[e] -= rv[e];
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float u = yv[e];
    const float d = (act == CIS_ACT_ELU) ? (u > 0.f ? 1.f : u + 1.f) : (u > 0.f ? 1.f : alpha);
    gv[e] *= d;
  }
  *gpp = pack8(gv);
}
__global__ void add_slice_kernel(bf16* dst, int dp, int dc, const bf16* __restrict__ src, int sp, int sc, size_t npix, int chunks, int reps,
                                 int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * chunks) return;
  const size_t pix = i / chunks;
  const int c = (int)(i % chunks) * 8;
  float a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, t[8];
  uint4* d = reinterpret_cast<uint4*>(dst + pix * dp + dc + c);
  if (accumulate) unpack8(*d, a);
  for (int j = 0; j < reps; ++j) {
    unpack8(*reinterpret_cast<const uint4*>(src + (pix + (size_t)j * npix) * sp + sc + c), t);
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] += t[e];
  }
  *d = pack8(a);
}
// part[blockIdx.x][c] = sum over this block's pixels of g[pix][c].  blockDim = 256 = P pixel lanes x chunks (chunks <= 32).
__global__ void colsum_kernel(const bf16* __restrict__ g, int gp, int gc, size_t npix, int nch, int chunks, float* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float sm[];  // [P][chunks*8]
  const int P = blockDim.x / chunks;
  const int ck = threadIdx.x % chunks, pl = threadIdx.x / chunks;
  float a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, t[8];
  if (pl < P) {
    for (size_t p = (size_t)blockIdx.x * P + pl; p < npix; p += (size_t)gridDim.x * P) {
      unpack8(*reinterpret_cast<const uint4*>(g + p * gp + gc + ck * 8), t);
#pragma unroll
      for (int e = 0; e < 8; ++e) a[e] += t[e];
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) sm[pl * chunks * 8 + ck * 8 + e] = a[e];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < nch; c += blockDim.x) {
    float s = 0.f;
    for (int q = 0; q < P; ++q) s += sm[q * chunks * 8 + c];
    part[(size_t)blockIdx.x * nch + c] = s;
  }
}

// dact_mul + colsum in one pass (layers that have an activation AND accumulate a bias gradient in this backward pass): g *= act'(y - res)
// in place, part[blockIdx.x][c] = this block's column sums of the ROUNDED product (what a separate colsum launch would read back).
__global__ void dact_colsum_kernel(bf16* g, int gp, int gc, const bf16* __restrict__ y, int yp, int yc, const bf16* __restrict__ res, int rp,
                                   int rc, size_t npix, int nch, int chunks, int act, float alpha, float* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float sm[];  // [P][chunks*8]
  const int P = blockDim.x / chunks;
  const int ck = threadIdx.x % chunks, pl = threadIdx.x / chunks;
  float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (pl < P) {
    for (size_t p = (size_t)blockIdx.x * P + pl; p < npix; p += (size_t)gridDim.x * P) {
      uint4* gpp = reinterpret_cast<uint4*>(g + p * gp + gc + ck * 8);
      float gv[8], yv[8], rv[8];
      unpack8(*gpp, gv);
      unpack8(*reinterpret_cast<const uint4*>(y + p * yp + yc + ck * 8), yv);
      if (res) {
        unpack8(*reinterpret_cast<const uint4*>(res + p * rp + rc + ck * 8), rv);
#pragma unroll
        for (int e = 0; e < 8; ++e) yv[e] -= rv[e];
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float u = yv[e];
        gv[e] *= (act == CIS_ACT_ELU) ? (u > 0.f ? 1.f : u + 1.f) : (u > 0.f ? 1.f : alpha);
      }
      const uint4 pk = pack8(gv);
      *gpp = pk;
      unpack8(pk, gv);
#pragma unroll
      for (int e = 0; e < 8; ++e) a[e] += gv[e];
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) sm[pl * chunks * 8 + ck * 8 + e] = a[e];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < nch; c += blockDim.x) {
    float s = 0.f;
    for (int q = 0; q < P; ++q) s += sm[q * chunks * 8 + c];
    part[(size_t)blockIdx.x * nch + c] = s;
  }
}

// ------------------------------------------------------------------------------------------------ resampling
// TF<=1.13 legacy bilinear (align_corners=False, no half-pixel centres): App. A.6.
struct Lerp {
  int lo, hi;
  float f;
};
__device__ __forceinline__ Lerp legacy_lerp(int d, int n_in, float scale) {
  const float s = d * scale;
  Lerp r;
  r.lo = (int)floorf(s);
  r.hi = min(r.lo + 1, n_in - 1);
  r.f = s - (float)r.lo;
  return r;
}
__global__ void resize_bilinear_bf16_kernel(const bf16* __restrict__ src, int sp, int sc, int N, int H, int W, bf16* __restrict__ dst, int dp,
                                            int dc, int OH, int OW, int chunks) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)N * OH * OW * chunks;
  if (i >= total) return;
  const int c = (int)(i % chunks) * 8;
  size_t pix = i / chunks;
  const int ox = (int)(pix % OW);
  const int oy = (int)((pix / OW) % OH);
  const int n = (int)(pix / ((size_t)OW * OH));
  const Lerp ly = legacy_lerp(oy, H, (float)H / (float)OH), lx = legacy_lerp(ox, W, (float)W / (float)OW);
  float tl[8], tr[8], bl[8], br[8], o[8];
  const bf16* b = src + (size_t)n * H * W * sp + sc + c;
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)ly.lo * W + lx.lo) * sp), tl);
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)ly.lo * W + lx.hi) * sp), tr);
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)ly.hi * W + lx.lo) * sp), bl);
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)ly.hi * W + lx.hi) * sp), br);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float t = tl[e] + (tr[e] - tl[e]) * lx.f;
    const float bo = bl[e] + (br[e] - bl[e]) * lx.f;
    o[e] = t + (bo - t) * ly.f;
  }
  *reinterpret_cast<uint4*>(dst + pix * dp + dc + c) = pack8(o);
}
// weight of source index i in destination index d (transpose of legacy_lerp)
__device__ __forceinline__ float legacy_w(int d, int i, int n_in, float scale) {
  const Lerp l = legacy_lerp(d, n_in, scale);
  return (l.lo == i ? 1.f - l.f : 0.f) + (l.hi == i ? l.f : 0.f);
}
__device__ __forceinline__ void legacy_range(int i, int n_out, float scale, int& d0, int& d1) {
  d0 = max(0, (int)floorf((i - 1) / scale) - 1);
  d1 = min(n_out - 1, (int)ceilf((i + 1) / scale) + 1);
}
__global__ void resize_bilinear_bf16_bwd_kernel(const bf16* __restrict__ dd, int dp, int dc, int N, int OH, int OW, bf16* ds, int sp, int sc,
                                                int H, int W, int chunks, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)N * H * W * chunks;
  if (i >= total) return;
  const int c = (int)(i % chunks) * 8;
  size_t pix = i / chunks;
  const int x = (int)(pix % W);
  const int y = (int)((pix / W) % H);
  const int n = (int)(pix / ((size_t)W * H));
  const float sy = (float)H / (float)OH, sx = (float)W / (float)OW;
  int y0, y1, x0, x1;
  legacy_range(y, OH, sy, y0, y1);
  legacy_range(x, OW, sx, x0, x1);
  float a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, t[8];
  uint4* o = reinterpret_cast<uint4*>(ds + pix * sp + sc + c);
  if (accumulate) unpack8(*o, a);
  for (int dy = y0; dy <= y1; ++dy) {
    const float wy = legacy_w(dy, y, H, sy);
    if (wy == 0.f) continue;
    for (int dx = x0; dx <= x1; ++dx) {
      const float wt = wy * legacy_w(dx, x, W, sx);
      if (wt == 0.f) continue;
      unpack8(*reinterpret_cast<const uint4*>(dd + ((size_t)(n * OH + dy) * OW + dx) * dp + dc + c), t);
#pragma unroll
      for (int e = 0; e < 8; ++e) a[e] += wt * t[e];
    }
  }
  *o = pack8(a);
}
// ---- fused resize + concat (recover decoder, convolution_utils.py:87-90 + nets.py:80-105): up to 4 sources of one resolution, each
// a channel slice of its own tensor (batch-broadcast when n_mod > 0), are legacy-bilinear resized to OH x OW and written side by side
// into ONE destination slice -- one launch instead of a resize per source plus a copy per source (and per broadcast replica).
struct RcArgs {
  CisSrc s[CIS_MAX_SRC];
  int nsrc;
};
__global__ void resize_concat_bf16_kernel(const RcArgs a, int N, int H, int W, bf16* __restrict__ dst, int dp, int dc, int OH, int OW,
                                          int total_chunks) {
  // grid.y = destination row (n, oy), grid.x * 256 threads = (ox, 8-channel chunk) of that row: no 64-bit divisions per thread
  pdl_launch_dependents();
  pdl_wait();
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (unsigned)(OW * total_chunks)) return;
  const int ox = (int)(t / (unsigned)total_chunks);
  int ck = (int)(t - (unsigned)ox * (unsigned)total_chunks);
  const int n = (int)(blockIdx.y / (unsigned)OH), oy = (int)(blockIdx.y - (unsigned)n * (unsigned)OH);
  const int off = ck * 8;
  int si = 0;
  while (si < a.nsrc - 1 && ck >= a.s[si].chunks) {
    ck -= a.s[si].chunks;
    ++si;
  }
  CisSrc sd = a.s[0];
  if (si == 1) sd = a.s[1];
  if (si == 2) sd = a.s[2];
  if (si == 3) sd = a.s[3];
  const int ns = sd.n_mod ? n % sd.n_mod : n;
  const bf16* b = reinterpret_cast<const bf16*>(sd.ptr) + (size_t)ns * H * W * sd.pitch + sd.c_off + ck * 8;
  uint4* o = reinterpret_cast<uint4*>(dst + ((size_t)blockIdx.y * OW + ox) * dp + dc + off);
  if (H == OH && W == OW) {          // same resolution: a plain gather of the channel slices
    *o = *reinterpret_cast<const uint4*>(b + ((size_t)oy * W + ox) * sd.pitch);
    return;
  }
  const Lerp ly = legacy_lerp(oy, H, (float)H / (float)OH), lx = legacy_lerp(ox, W, (float)W / (float)OW);
  float tl[8], tr[8], bl[8], br[8], r[8];
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)ly.lo * W + lx.lo) * sd.pitch), tl);
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)ly.lo * W + lx.hi) * sd.pitch), tr);
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)ly.hi * W + lx.lo) * sd.pitch), bl);
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)ly.hi * W + lx.hi) * sd.pitch), br);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float tp = tl[e] + (tr[e] - tl[e]) * lx.f;
    const float bo = bl[e] + (br[e] - bl[e]) * lx.f;
    r[e] = tp + (bo - tp) * ly.f;
  }
  *o = pack8(r);
}
// exact x2 case (OH = 2H, OW = 2W: every `deconv` of the recover decoder at power-of-two sizes): one thread per SOURCE pixel chunk loads the
// 2x2 source neighbourhood once and writes the four destination pixels it determines -- same lerp expressions (fractions 0 / 0.5, clamped
// last row / column), so the result is bit-identical to the generic kernel with a quarter of the loads and index arithmetic.
__global__ void resize_concat_x2_bf16_kernel(const RcArgs a, int N, int H, int W, bf16* __restrict__ dst, int dp, int dc, int total_chunks) {
  pdl_launch_dependents();
  pdl_wait();
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (unsigned)(W * total_chunks)) return;
  const int x = (int)(t / (unsigned)total_chunks);
  int ck = (int)(t - (unsigned)x * (unsigned)total_chunks);
  const int n = (int)(blockIdx.y / (unsigned)H), y = (int)(blockIdx.y - (unsigned)n * (unsigned)H);
  const int off = ck * 8;
  int si = 0;
  while (si < a.nsrc - 1 && ck >= a.s[si].chunks) {
    ck -= a.s[si].chunks;
    ++si;
  }
  CisSrc sd = a.s[0];
  if (si == 1) sd = a.s[1];
  if (si == 2) sd = a.s[2];
  if (si == 3) sd = a.s[3];
  const int ns = sd.n_mod ? n % sd.n_mod : n;
  const bf16* b = reinterpret_cast<const bf16*>(sd.ptr) + (size_t)ns * H * W * sd.pitch + sd.c_off + ck * 8;
  const int x1 = min(x + 1, W - 1), y1 = min(y + 1, H - 1);
  float s00[8], s01[8], s10[8], s11[8], r[8];
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)y * W + x) * sd.pitch), s00);
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)y * W + x1) * sd.pitch), s01);
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)y1 * W + x) * sd.pitch), s10);
  unpack8(*reinterpret_cast<const uint4*>(b + ((size_t)y1 * W + x1) * sd.pitch), s11);
  const int OW = 2 * W;
  bf16* o = dst + (((size_t)(n * 2 * H + 2 * y)) * OW + 2 * x) * dp + dc + off;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float fy = (q >> 1) ? 0.5f : 0.f, fx = (q & 1) ? 0.5f : 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float tp = s00[e] + (s01[e] - s00[e]) * fx;
      const float bo = s10[e] + (s11[e] - s10[e]) * fx;
      r[e] = tp + (bo - tp) * fy;
    }
    *reinterpret_cast<uint4*>(o + ((size_t)(q >> 1) * OW + (q & 1)) * dp) = pack8(r);
  }
}
// its transpose: for every source with want != 0, dsrc (=|+=) sum over broadcast replicas of R^T ddst[.., slice of that source]
struct RcGrad {
  void* ptr;
  int pitch, c_off, chunks, n_mod, want, accumulate;
};
struct RcGradArgs {
  RcGrad s[CIS_MAX_SRC];
  int nsrc;
};
__global__ void resize_concat_bf16_bwd_kernel(const bf16* __restrict__ dd, int dp, int dc, int N, int OH, int OW, const RcGradArgs a, int H,
                                              int W, int total_chunks) {
  // grid.y = source row (n, y), grid.x * 256 threads = (x, 8-channel chunk).  The x weights of the (<= 8 wide) candidate window are
  // evaluated once per thread, not once per (dy, dx) pair.
  pdl_launch_dependents();
  pdl_wait();
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (unsigned)(W * total_chunks)) return;
  const int x = (int)(t / (unsigned)total_chunks);
  int ck = (int)(t - (unsigned)x * (unsigned)total_chunks);
  const int n = (int)(blockIdx.y / (unsigned)H), y = (int)(blockIdx.y - (unsigned)n * (unsigned)H);
  const int off = ck * 8;
  int si = 0;
  while (si < a.nsrc - 1 && ck >= a.s[si].chunks) {
    ck -= a.s[si].chunks;
    ++si;
  }
  RcGrad sd = a.s[0];
  if (si == 1) sd = a.s[1];
  if (si == 2) sd = a.s[2];
  if (si == 3) sd = a.s[3];
  if (!sd.want || (sd.n_mod && n >= sd.n_mod)) return;
  const int reps = sd.n_mod ? N / sd.n_mod : 1;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, tv[8];
  uint4* o = reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(sd.ptr) + ((size_t)(n * H + y) * W + x) * sd.pitch + sd.c_off + ck * 8);
  if (sd.accumulate) unpack8(*o, acc);
  if (H == OH && W == OW) {          // same resolution: fold the broadcast replicas of this pixel
    for (int r = 0; r < reps; ++r) {
      unpack8(*reinterpret_cast<const uint4*>(dd + ((size_t)((n + r * sd.n_mod) * OH + y) * OW + x) * dp + dc + off), tv);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += tv[e];
    }
    *o = pack8(acc);
    return;
  }
  const float sy = (float)H / (float)OH, sx = (float)W / (float)OW;
  const bool x2 = OH == 2 * H && OW == 2 * W;     // exact x2: the transpose weights are 0.5 / 1 / 0.5 (1 on the clamped last row / column),
  int y0, y1, x0, x1;                             // the same values legacy_w returns, without evaluating it 14 times per thread
  if (x2) {
    y0 = max(2 * y - 1, 0);
    y1 = 2 * y + 1;
    x0 = max(2 * x - 1, 0);
    x1 = 2 * x + 1;
  } else {
    legacy_range(y, OH, sy, y0, y1);
    legacy_range(x, OW, sx, x0, x1);
  }
  const int nx = x1 - x0 + 1;
  const bool pre = nx <= 8;
  float wxv[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int dx = x0 + k;
    wxv[k] = !(pre && k < nx) ? 0.f : x2 ? ((dx == 2 * x || (dx == 2 * x + 1 && x == W - 1)) ? 1.f : 0.5f) : legacy_w(dx, x, W, sx);
  }
  for (int dy = y0; dy <= y1; ++dy) {
    const float wy = x2 ? ((dy == 2 * y || (dy == 2 * y + 1 && y == H - 1)) ? 1.f : 0.5f) : legacy_w(dy, y, H, sy);
    if (wy == 0.f) continue;
    if (pre) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float wt = wy * wxv[k];
        if (wt == 0.f) continue;
        for (int r = 0; r < reps; ++r) {
          unpack8(*reinterpret_cast<const uint4*>(dd + ((size_t)((n + r * sd.n_mod) * OH + dy) * OW + x0 + k) * dp + dc + off), tv);
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e] += wt * tv[e];
        }
      }
    } else {
      for (int dx = x0; dx <= x1; ++dx) {
        const float wt = wy * legacy_w(dx, x, W, sx);
        if (wt == 0.f) continue;
        for (int r = 0; r < reps; ++r) {
          unpack8(*reinterpret_cast<const uint4*>(dd + ((size_t)((n + r * sd.n_mod) * OH + dy) * OW + dx) * dp + dc + off), tv);
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e] += wt * tv[e];
        }
      }
    }
  }
  *o = pack8(acc);
}
// source step of tf.image.resize_* in TF 1.13 (no half-pixel centres): (in-1)/(out-1) with align_corners and out > 1, else in/out
template <bool AC>
__device__ __forceinline__ float resize_step(int n_in, int n_out) {
  return (AC && n_out > 1) ? (float)(n_in - 1) / (float)(n_out - 1) : (float)n_in / (float)n_out;
}
// AC = align_corners; AC = false is the legacy resize of the step graph (cis_resize_bilinear_f32)
template <bool AC>
__global__ void resize_bilinear_f32_kernel(const float* __restrict__ src, int N, int H, int W, int C, float* __restrict__ dst, int OH, int OW,
                                           float scale) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (size_t)N * OH * OW) return;
  const int ox = (int)(pix % OW);
  const int oy = (int)((pix / OW) % OH);
  const int n = (int)(pix / ((size_t)OW * OH));
  const Lerp ly = legacy_lerp(oy, H, resize_step<AC>(H, OH)), lx = legacy_lerp(ox, W, resize_step<AC>(W, OW));
  const float* b = src + (size_t)n * H * W * C;
  for (int c = 0; c < C; ++c) {
    const float tl = b[((size_t)ly.lo * W + lx.lo) * C + c], tr = b[((size_t)ly.lo * W + lx.hi) * C + c];
    const float bl = b[((size_t)ly.hi * W + lx.lo) * C + c], br = b[((size_t)ly.hi * W + lx.hi) * C + c];
    const float t = tl + (tr - tl) * lx.f, bo = bl + (br - bl) * lx.f;
    dst[pix * C + c] = (t + (bo - t) * ly.f) * scale;
  }
}
// central crop + legacy-bilinear resize back to OH x OW of ONE fp32 NHWC image (the multi-crop ensemble inputs,
// davis2016_data_utils.py:328-354 / 130-134): crop box (y0, x0, ch, cw) of the Hs x Ws source, same interpolation rule as above.
// FLOW = true: a 2-channel flow field whose vectors follow the resize, channel 0 times s0 and channel 1 times s1 (cis_crop_resize_flow_f32);
// FLOW = false reads neither scale and is the plain image crop.
template <bool FLOW>
__global__ void crop_resize_f32_kernel(const float* __restrict__ src, int Ws, int C, int y0, int x0, int ch, int cw, float* __restrict__ dst,
                                       int OH, int OW, float s0, float s1) {
  pdl_launch_dependents();
  pdl_wait();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= OH * OW) return;
  const int ox = pix % OW, oy = pix / OW;
  const Lerp ly = legacy_lerp(oy, ch, (float)ch / (float)OH), lx = legacy_lerp(ox, cw, (float)cw / (float)OW);
  const float* r0 = src + (size_t)(y0 + ly.lo) * Ws * C;
  const float* r1 = src + (size_t)(y0 + ly.hi) * Ws * C;
  for (int c = 0; c < C; ++c) {
    const float tl = r0[(x0 + lx.lo) * C + c], tr = r0[(x0 + lx.hi) * C + c];
    const float bl = r1[(x0 + lx.lo) * C + c], br = r1[(x0 + lx.hi) * C + c];
    const float t = tl + (tr - tl) * lx.f, bo = bl + (br - bl) * lx.f;
    const float v = t + (bo - t) * ly.f;
    dst[(size_t)pix * C + c] = FLOW ? v * (c == 0 ? s0 : s1) : v;
  }
}
// transpose of the fp32 legacy resize (times `scale`, the factor of cis_resize_bilinear_f32), result stored as a bf16 8-channel chunk
// (C <= 8 real channels)
__global__ void resize_f32_bwd_to_bf16_kernel(const float* __restrict__ dd, int N, int OH, int OW, int C, int H, int W, bf16* __restrict__ ds,
                                              int sp, float scale) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (size_t)N * H * W) return;
  const int x = (int)(pix % W);
  const int y = (int)((pix / W) % H);
  const int n = (int)(pix / ((size_t)W * H));
  const float sy = (float)H / (float)OH, sx = (float)W / (float)OW;
  int y0, y1, x0, x1;
  legacy_range(y, OH, sy, y0, y1);
  legacy_range(x, OW, sx, x0, x1);
  float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int dy = y0; dy <= y1; ++dy) {
    const float wy = legacy_w(dy, y, H, sy);
    if (wy == 0.f) continue;
    for (int dx = x0; dx <= x1; ++dx) {
      const float wt = wy * legacy_w(dx, x, W, sx);
      if (wt == 0.f) continue;
      const float* q = dd + ((size_t)(n * OH + dy) * OW + dx) * C;
      for (int c = 0; c < C; ++c) a[c] += wt * q[c];
    }
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) a[c] *= scale;
  *reinterpret_cast<uint4*>(ds + pix * sp) = pack8(a);
}
// tf.image.resize_nearest_neighbor(align_corners=True), out = 2*in: src = min(roundf(d*(in-1)/(out-1)), in-1)   App. A.5
__device__ __forceinline__ int nn_src(int d, int n_in) {
  const float scale = (float)(n_in - 1) / (float)(2 * n_in - 1);
  return min((int)roundf(d * scale), n_in - 1);
}
__global__ void upsample_nn2x_kernel(const bf16* __restrict__ src, int N, int H, int W, int pitch, bf16* __restrict__ dst) {
  // grid.y = destination row (n, oy); threads = (ox, 8-channel chunk): 32-bit index math, one source row per block row
  pdl_launch_dependents();
  pdl_wait();
  const int chunks = pitch / 8;
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (unsigned)(2 * W * chunks)) return;
  const int ox = (int)(t / (unsigned)chunks), c = (int)(t - (unsigned)ox * (unsigned)chunks) * 8;
  const int n = (int)(blockIdx.y / (unsigned)(2 * H)), oy = (int)(blockIdx.y - (unsigned)n * (unsigned)(2 * H));
  const int sy = nn_src(oy, H), sx = nn_src(ox, W);
  *reinterpret_cast<uint4*>(dst + ((size_t)blockIdx.y * 2 * W + ox) * pitch + c) =
      *reinterpret_cast<const uint4*>(src + ((size_t)(n * H + sy) * W + sx) * pitch + c);
}
__global__ void upsample_nn2x_bwd_kernel(const bf16* __restrict__ dd, int N, int H, int W, int pitch, bf16* ds, int accumulate) {
  // grid.y = source row (n, y); the (<= 6) candidate destination rows / columns are tested once per thread, not once per pair
  pdl_launch_dependents();
  pdl_wait();
  const int chunks = pitch / 8;
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (unsigned)(W * chunks)) return;
  const int x = (int)(t / (unsigned)chunks), c = (int)(t - (unsigned)x * (unsigned)chunks) * 8;
  const int n = (int)(blockIdx.y / (unsigned)H), y = (int)(blockIdx.y - (unsigned)n * (unsigned)H);
  float a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, tv[8];
  uint4* o = reinterpret_cast<uint4*>(ds + ((size_t)blockIdx.y * W + x) * pitch + c);
  if (accumulate) unpack8(*o, a);
  const int dx0 = max(0, 2 * x - 2), dx1 = min(2 * W - 1, 2 * x + 3);
  unsigned xm = 0;                                   // bit k: destination column dx0 + k maps to this source column
  for (int dx = dx0; dx <= dx1; ++dx)
    if (nn_src(dx, W) == x) xm |= 1u << (dx - dx0);
  for (int dy = max(0, 2 * y - 2); dy <= min(2 * H - 1, 2 * y + 3); ++dy) {
    if (nn_src(dy, H) != y) continue;
    const bf16* row = dd + ((size_t)(n * 2 * H + dy) * 2 * W) * pitch + c;
    for (int dx = dx0; dx <= dx1; ++dx) {
      if (!((xm >> (dx - dx0)) & 1u)) continue;
      unpack8(*reinterpret_cast<const uint4*>(row + (size_t)dx * pitch), tv);
#pragma unroll
      for (int e = 0; e < 8; ++e) a[e] += tv[e];
    }
  }
  *o = pack8(a);
}
// nearest source index: roundf with align_corners (App. A.5), floor without, clamped to in-1
template <bool AC>
__device__ __forceinline__ int nn_index(int d, int n_in, float step) {
  return min((int)(AC ? roundf(d * step) : floorf(d * step)), n_in - 1);
}
template <bool AC>
__global__ void resize_nn_f32_kernel(const float* __restrict__ src, int N, int H, int W, int C, float* __restrict__ dst, int OH, int OW) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (size_t)N * OH * OW) return;
  const int ox = (int)(pix % OW);
  const int oy = (int)((pix / OW) % OH);
  const int n = (int)(pix / ((size_t)OW * OH));
  const int sy = nn_index<AC>(oy, H, resize_step<AC>(H, OH)), sx = nn_index<AC>(ox, W, resize_step<AC>(W, OW));
  for (int c = 0; c < C; ++c) dst[pix * C + c] = src[((size_t)(n * H + sy) * W + sx) * C + c];
}
// Transpose of the four fp32 resizes as a gather: thread = one element (n, y, x, c) of dsrc.  Along each axis the source map d -> lo(d)
// (bilinear) or d -> index(d) (nearest) is monotone, so the outputs that read input index i form one contiguous range, found by binary
// search; each element sums its own rectangle of ddst in a fixed order -- no atomics, bit-identical run to run, for any scale.
template <bool NEAREST, bool AC>
__device__ __forceinline__ int resize_src_key(int d, int n_in, float step) {
  return NEAREST ? nn_index<AC>(d, n_in, step) : (int)floorf(d * step);
}
// first d in [0, n_out) whose key is >= v (n_out when none)
template <bool NEAREST, bool AC>
__device__ __forceinline__ int resize_lower_bound(int v, int n_in, int n_out, float step) {
  int lo = 0, hi = n_out;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (resize_src_key<NEAREST, AC>(mid, n_in, step) < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}
// weight of input index i in output index d
template <bool NEAREST, bool AC>
__device__ __forceinline__ float resize_w(int d, int i, int n_in, float step) {
  if (NEAREST) return nn_index<AC>(d, n_in, step) == i ? 1.f : 0.f;
  return legacy_w(d, i, n_in, step);
}
template <bool NEAREST, bool AC>
__global__ void resize_f32_bwd_kernel(const float* __restrict__ dd, int N, int OH, int OW, int C, int H, int W, float* __restrict__ ds) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)N * H * W * C) return;
  const int c = (int)(i % C);
  const size_t pix = i / C;
  const int x = (int)(pix % W);
  const int y = (int)((pix / W) % H);
  const int n = (int)(pix / ((size_t)W * H));
  const float sy = resize_step<AC>(H, OH), sx = resize_step<AC>(W, OW);
  // bilinear: outputs with lo in {i-1, i} read i (as hi or lo); nearest: outputs with index == i
  const int kd = NEAREST ? 0 : 1;
  const int y0 = resize_lower_bound<NEAREST, AC>(y - kd, H, OH, sy), y1 = resize_lower_bound<NEAREST, AC>(y + 1, H, OH, sy);
  const int x0 = resize_lower_bound<NEAREST, AC>(x - kd, W, OW, sx), x1 = resize_lower_bound<NEAREST, AC>(x + 1, W, OW, sx);
  float a = 0.f;
  for (int dy = y0; dy < y1; ++dy) {
    const float wy = resize_w<NEAREST, AC>(dy, y, H, sy);
    if (wy == 0.f) continue;
    const float* row = dd + ((size_t)(n * OH + dy) * OW) * C + c;
    for (int dx = x0; dx < x1; ++dx) {
      const float wt = wy * resize_w<NEAREST, AC>(dx, x, W, sx);
      if (wt != 0.f) a += wt * row[(size_t)dx * C];
    }
  }
  ds[i] = a;
}

// ------------------------------------------------------------------------------------------------ warp + cost volume
// dense_image_warp (core_warp.py:153-202): query = grid - flow, floor clamped to [0,size-2], alpha clamped to [0,1].
__device__ __forceinline__ void warp_coords(float q, int size, int& lo, float& a) {
  float fl = fminf(fmaxf(floorf(q), 0.f), (float)(size - 2));
  lo = (int)fl;
  a = fminf(fmaxf(q - fl, 0.f), 1.f);
}
__device__ __forceinline__ void warp_chunk(const bf16* __restrict__ img, int pitch, int h, int w, int b, float qy, float qx, float* o) {
  int y0, x0;
  float ay, ax;
  warp_coords(qy, h, y0, ay);
  warp_coords(qx, w, x0, ax);
  const bf16* base = img + ((size_t)(b * h + y0) * w + x0) * pitch;
  float tl[8], tr[8], bl[8], br[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(base)), tl);
  unpack8(__ldg(reinterpret_cast<const uint4*>(base + pitch)), tr);
  unpack8(__ldg(reinterpret_cast<const uint4*>(base + (size_t)w * pitch)), bl);
  unpack8(__ldg(reinterpret_cast<const uint4*>(base + (size_t)w * pitch + pitch)), br);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float t = ax * (tr[e] - tl[e]) + tl[e];
    const float bo = ax * (br[e] - bl[e]) + bl[e];
    o[e] = ay * (bo - t) + t;
  }
}
__global__ void dense_image_warp_kernel(const bf16* __restrict__ img, int pitch, int coff, const float* __restrict__ flow, float fs, int B,
                                        int h, int w, int chunks, bf16* __restrict__ out, int op) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * h * w * chunks) return;
  const int c = (int)(i % chunks) * 8;
  const size_t pix = i / chunks;
  const int x = (int)(pix % w), y = (int)((pix / w) % h), b = (int)(pix / ((size_t)w * h));
  float o[8];
  warp_chunk(img + coff + c, pitch, h, w, b, (float)y - flow[pix * 2] * fs, (float)x - flow[pix * 2 + 1] * fs, o);
  *reinterpret_cast<uint4*>(out + pix * op + c) = pack8(o);
}

// Search range R (core_costvol.py:20-40, model_pwcnet.py options 'search_range'), 1 <= R <= 4: (2R+1)^2 displacements over an 8x16 pixel
// tile and its (8+2R)x(16+2R) halo.  R = 4 is the upper bound: the backward's staging takes cv_bwd_smem(4) = 193,536 B, R = 5 would need
// 258,688 B, more than a block's 227 KB.
static constexpr int kCvTH = 8, kCvTW = 16, kCvRMax = 4;
static constexpr int kCvPitch = 36;                                        // floats per smem pixel row (32 ch + pad)
__host__ __device__ constexpr int cv_span(int R) { return 2 * R + 1; }
__host__ __device__ constexpr int cv_ndisp(int R) { return cv_span(R) * cv_span(R); }
__host__ __device__ constexpr int cv_hh(int R) { return kCvTH + 2 * R; }   // halo rows
__host__ __device__ constexpr int cv_hw(int R) { return kCvTW + 2 * R; }   // halo columns
constexpr int cv_smem(int R) { return (kCvTH * kCvTW + cv_hh(R) * cv_hw(R)) * kCvPitch * 4; }
static_assert(cv_smem(kCvRMax) == (128 + 16 * 24) * 36 * 4, "R = 4 keeps the 16 x 24 halo");
// R < 4: without a minimum-blocks hint ptxas caps the smaller instances at 48-64 registers and spills; two CTAs per SM (128 registers)
// removes the spills.  R = 4 keeps the plain __launch_bounds__(256) code (0 = no minimum).
constexpr int cv_min_blocks(int R) { return R == kCvRMax ? 0 : 2; }

template <int R>
__global__ void __launch_bounds__(256, cv_min_blocks(R)) warp_costvol_kernel(const bf16* __restrict__ c1, int c1p, int c1o, const bf16* __restrict__ c2, int c2p,
                                                           int c2o, const float* __restrict__ flow, float fs, int B, int h, int w, int C,
                                                           bf16* __restrict__ out, int op, int oo) {
  constexpr int S = cv_span(R), ND = cv_ndisp(R), HH = cv_hh(R), HW = cv_hw(R);
  static_assert(kCvTH * kCvTW * ND * 2 <= HH * HW * kCvPitch * 4, "the bf16 result staging fits the halo buffer");
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float cvs[];
  float* s1 = cvs;                                 // [128][36]
  float* s2 = cvs + kCvTH * kCvTW * kCvPitch;      // [HH * HW][36]
  const int tid = threadIdx.x;
  const int b = blockIdx.z, y0 = blockIdx.y * kCvTH, x0 = blockIdx.x * kCvTW;
  const int pix = tid & 127, py = pix >> 4, px = pix & 15;
  const int dyb = tid >> 7;  // this thread handles dy = dyb + 2k
  float acc[R + 1][S];
#pragma unroll
  for (int k = 0; k < R + 1; ++k)
#pragma unroll
    for (int d = 0; d < S; ++d) acc[k][d] = 0.f;
  const int Cp = (C + 7) & ~7;
  for (int cc = 0; cc < Cp; cc += 32) {
    const int nck = min(4, (Cp - cc) / 8);  // 8-channel chunks in this pass
    // c1 tile
    for (int it = tid; it < 128 * 4; it += 256) {
      const int p = it >> 2, ck = it & 3;
      const int y = y0 + (p >> 4), x = x0 + (p & 15);
      float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (ck < nck && y < h && x < w) unpack8(__ldg(reinterpret_cast<const uint4*>(c1 + ((size_t)(b * h + y) * w + x) * c1p + c1o + cc + ck * 8)), v);
      float4* d = reinterpret_cast<float4*>(s1 + p * kCvPitch + ck * 8);
      d[0] = make_float4(v[0], v[1], v[2], v[3]);
      d[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    // warped c2 halo (zero outside the image: tf.pad of the warped map, core_costvol.py:27)
    for (int it = tid; it < HH * HW * 4; it += 256) {
      const int p = it >> 2, ck = it & 3;
      const int y = y0 - R + p / HW, x = x0 - R + p % HW;
      float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (ck < nck && y >= 0 && y < h && x >= 0 && x < w) {
        if (flow) {
          const size_t fp = ((size_t)(b * h + y) * w + x) * 2;
          warp_chunk(c2 + c2o + cc + ck * 8, c2p, h, w, b, (float)y - __ldg(flow + fp) * fs, (float)x - __ldg(flow + fp + 1) * fs, v);
        } else {
          unpack8(__ldg(reinterpret_cast<const uint4*>(c2 + ((size_t)(b * h + y) * w + x) * c2p + c2o + cc + ck * 8)), v);
        }
      }
      float4* d = reinterpret_cast<float4*>(s2 + p * kCvPitch + ck * 8);
      d[0] = make_float4(v[0], v[1], v[2], v[3]);
      d[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < R + 1; ++k) {
      const int dy = dyb + 2 * k;
      if (dy < S) {
        const float* r2 = s2 + ((py + dy) * HW + px) * kCvPitch;
        const float* r1 = s1 + pix * kCvPitch;
        for (int c4 = 0; c4 < nck * 2; ++c4) {
          const float4 a = *reinterpret_cast<const float4*>(r1 + c4 * 4);
#pragma unroll
          for (int dx = 0; dx < S; ++dx) {
            const float4 q = *reinterpret_cast<const float4*>(r2 + dx * kCvPitch + c4 * 4);
            acc[k][dx] += a.x * q.x + a.y * q.y + a.z * q.z + a.w * q.w;
          }
        }
      }
    }
    __syncthreads();
  }
  // mean over the REAL channel count, leaky 0.1, stage [128][ND] bf16 in smem, coalesced store
  bf16* so = reinterpret_cast<bf16*>(s2);
  const float inv = 1.f / (float)C;
#pragma unroll
  for (int k = 0; k < R + 1; ++k) {
    const int dy = dyb + 2 * k;
    if (dy < S) {
#pragma unroll
      for (int dx = 0; dx < S; ++dx) {
        float v = acc[k][dx] * inv;
        v = v > 0.f ? v : 0.1f * v;
        so[pix * ND + dy * S + dx] = __float2bfloat16(v);
      }
    }
  }
  __syncthreads();
  for (int it = tid; it < 128 * ND; it += 256) {
    const int p = it / ND, ch = it % ND;
    const int y = y0 + (p >> 4), x = x0 + (p & 15);
    if (y < h && x < w) out[((size_t)(b * h + y) * w + x) * op + oo + ch] = so[it];
  }
}

// ------------------------------------------------------------------------------------------------ input packing
__global__ void pack_f32_to_bf16_kernel(const float* __restrict__ src, size_t npix, int C, float offset, bf16* __restrict__ dst, int dp, int dc) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int c = 0; c < C; ++c) v[c] = src[pix * C + c] + offset;
  *reinterpret_cast<uint4*>(dst + pix * dp + dc) = pack8(v);
}
__global__ void flow_stats_kernel(const float* __restrict__ flow, size_t hw, double* __restrict__ stats) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  double s0 = 0, s1 = 0, q0 = 0, q1 = 0;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (size_t)gridDim.x * blockDim.x) {
    const float2 f = *reinterpret_cast<const float2*>(flow + ((size_t)b * hw + p) * 2);
    s0 += f.x; s1 += f.y; q0 += (double)f.x * f.x; q1 += (double)f.y * f.y;
  }
  s0 = warp_sum_d(s0); s1 = warp_sum_d(s1); q0 = warp_sum_d(q0); q1 = warp_sum_d(q1);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(stats + b * 4 + 0, s0); atomicAdd(stats + b * 4 + 1, s1);
    atomicAdd(stats + b * 4 + 2, q0); atomicAdd(stats + b * 4 + 3, q1);
  }
}
__global__ void pack_generator_input_kernel(const float* __restrict__ image, const float* __restrict__ flow, const double* __restrict__ stats,
                                            size_t hw, bf16* __restrict__ dst) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= hw) return;
  const double n = (double)hw;
  const double m0 = stats[b * 4] / n, m1 = stats[b * 4 + 1] / n;
  const float r0 = (float)(1.0 / sqrt(stats[b * 4 + 2] / n - m0 * m0)), r1 = (float)(1.0 / sqrt(stats[b * 4 + 3] / n - m1 * m1));
  const size_t pix = (size_t)b * hw + p;
  float v[8] = {image[pix * 3], image[pix * 3 + 1], image[pix * 3 + 2], (flow[pix * 2] - (float)m0) * r0, (flow[pix * 2 + 1] - (float)m1) * r1,
                0, 0, 0};
  *reinterpret_cast<uint4*>(dst + pix * 8) = pack8(v);
}
// ---- stand-alone preprocess_flow_batch (flow_utils.py:5-12) and its gradient, fp32 [B,hw,2]
// mean and 1/sqrt(population variance) of channel k of sample b, from cis_flow_stats' sums; the same arithmetic as
// pack_generator_input_kernel, so the stand-alone call and the generator's fused input agree bit for bit
__device__ __forceinline__ void flow_moments(const double* __restrict__ stats, int b, double n, float* m, float* r) {
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const double mk = stats[b * 4 + k] / n;
    m[k] = (float)mk;
    r[k] = (float)(1.0 / sqrt(stats[b * 4 + 2 + k] / n - mk * mk));
  }
}
__global__ void flow_standardize_kernel(const float* __restrict__ flow, const double* __restrict__ stats, size_t hw, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= hw) return;
  float m[2], r[2];
  flow_moments(stats, b, (double)hw, m, r);
  const size_t i = ((size_t)b * hw + p) * 2;
  const float2 f = *reinterpret_cast<const float2*>(flow + i);
  *reinterpret_cast<float2*>(out + i) = make_float2((f.x - m[0]) * r[0], (f.y - m[1]) * r[1]);
}
// backward, pass 1: block x of sample b sums {g0, g1, g0*y0, g1*y1} over a fixed pixel subset (grid-stride), in double, reduced in a
// fixed order (warp butterfly, then the 8 warps in index order) into part[(b * kFlowStdBlocks + x) * 4 + k]
constexpr int kFlowStdBlocks = 64;
__global__ void flow_standardize_bwd_sums_kernel(const float* __restrict__ y, const float* __restrict__ g, size_t hw, double* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double sm[8][4];
  const int b = blockIdx.y;
  double s[4] = {0, 0, 0, 0};
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (size_t)gridDim.x * blockDim.x) {
    const size_t i = ((size_t)b * hw + p) * 2;
    const float2 gv = *reinterpret_cast<const float2*>(g + i), yv = *reinterpret_cast<const float2*>(y + i);
    s[0] += gv.x; s[1] += gv.y; s[2] += (double)gv.x * yv.x; s[3] += (double)gv.y * yv.y;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) s[k] = warp_sum_d(s[k]);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) sm[threadIdx.x >> 5][k] = s[k];
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    double t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sm[w][threadIdx.x];
    part[((size_t)b * gridDim.x + blockIdx.x) * 4 + threadIdx.x] = t;
  }
}
// pass 2: dx = (g - mean(g) - y * mean(g * y)) / sigma per (sample, channel); every block re-adds the kFlowStdBlocks partials in order
__global__ void flow_standardize_bwd_kernel(const float* __restrict__ y, const float* __restrict__ g, const double* __restrict__ stats,
                                            const double* __restrict__ part, size_t hw, float* __restrict__ dx) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float mean[4];
  const int b = blockIdx.y;
  if (threadIdx.x < 4) {
    double t = 0;
    for (int q = 0; q < kFlowStdBlocks; ++q) t += part[((size_t)b * kFlowStdBlocks + q) * 4 + threadIdx.x];
    mean[threadIdx.x] = (float)(t / (double)hw);
  }
  __syncthreads();
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= hw) return;
  float m[2], r[2];
  flow_moments(stats, b, (double)hw, m, r);
  const size_t i = ((size_t)b * hw + p) * 2;
  const float2 gv = *reinterpret_cast<const float2*>(g + i), yv = *reinterpret_cast<const float2*>(y + i);
  *reinterpret_cast<float2*>(dx + i) = make_float2((gv.x - mean[0] - yv.x * mean[2]) * r[0], (gv.y - mean[1] - yv.y * mean[3]) * r[1]);
}
// ---- masked end-point error of the recover net's held-out pass, same fixed-order rule as the standardisation gradient above.
// pass 1: block x of sample b sums {m*e, (1-m)*e, m, 1-m}, e = |pred - gt|_2, all in double, over a fixed pixel subset (grid-stride),
// reduced warp butterfly -> the 8 warps in index order into part[(b * kFlowStdBlocks + x) * 4 + k]
__global__ void masked_epe_sums_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const float* __restrict__ mask, size_t hw,
                                       double* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double sm[8][4];
  const int b = blockIdx.y;
  double s[4] = {0, 0, 0, 0};
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (size_t)gridDim.x * blockDim.x) {
    const size_t pix = (size_t)b * hw + p;
    const float2 pv = *reinterpret_cast<const float2*>(pred + pix * 2), gv = *reinterpret_cast<const float2*>(gt + pix * 2);
    const double dx = (double)pv.x - gv.x, dy = (double)pv.y - gv.y, e = sqrt(dx * dx + dy * dy), m = mask[pix];
    s[0] += m * e; s[1] += (1.0 - m) * e; s[2] += m; s[3] += 1.0 - m;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) s[k] = warp_sum_d(s[k]);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) sm[threadIdx.x >> 5][k] = s[k];
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    double t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sm[w][threadIdx.x];
    part[((size_t)b * gridDim.x + blockIdx.x) * 4 + threadIdx.x] = t;
  }
}
// pass 2: one block per sample, thread k adds the kFlowStdBlocks partials of sum k in block order
__global__ void masked_epe_reduce_kernel(const double* __restrict__ part, double* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, k = threadIdx.x;
  double t = 0;
  for (int q = 0; q < kFlowStdBlocks; ++q) t += part[((size_t)b * kFlowStdBlocks + q) * 4 + k];
  out[b * 4 + k] = t;
}

// ------------------------------------------------------------------------------------------------ mask (x) flow + loss
__global__ void mask_apply_kernel(const float* __restrict__ flow, const float* __restrict__ mask, size_t npix, bf16* __restrict__ dst) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const float m = mask[p], f0 = flow[p * 2], f1 = flow[p * 2 + 1];
  const float a[8] = {f0 * (1.f - m), f1 * (1.f - m), 1.f, 1.f - m, 0, 0, 0, 0};  // adversarial_learner.py:109 + nets.py:50-52
  const float c[8] = {f0 * m, f1 * m, 1.f, m, 0, 0, 0, 0};                          // :110 with mask = 1-m
  const float z[8] = {0, 0, 1.f, 0, 0, 0, 0, 0};                                    // :127-131
  *reinterpret_cast<uint4*>(dst + p * 8) = pack8(a);
  *reinterpret_cast<uint4*>(dst + (npix + p) * 8) = pack8(c);
  *reinterpret_cast<uint4*>(dst + (2 * npix + p) * 8) = pack8(z);
}
__device__ __forceinline__ float2 pred_at(const float* __restrict__ f1, int n, int h1, int w1, const Lerp& ly, const Lerp& lx) {
  const float2* b = reinterpret_cast<const float2*>(f1) + (size_t)n * h1 * w1;
  const float2 tl = b[(size_t)ly.lo * w1 + lx.lo], tr = b[(size_t)ly.lo * w1 + lx.hi];
  const float2 bl = b[(size_t)ly.hi * w1 + lx.lo], br = b[(size_t)ly.hi * w1 + lx.hi];
  float2 r;
  {
    const float t = tl.x + (tr.x - tl.x) * lx.f, bo = bl.x + (br.x - bl.x) * lx.f;
    r.x = t + (bo - t) * ly.f;
  }
  {
    const float t = tl.y + (tr.y - tl.y) * lx.f, bo = bl.y + (br.y - bl.y) * lx.f;
    r.y = t + (bo - t) * ly.f;
  }
  return r;
}
// charbonnier term (loss_utils.py:47-49) and its derivative w.r.t. pred
__device__ __forceinline__ float charb(float d, float cbn) {
  const float s = d * d + 1e-6f;
  return cbn == 0.5f ? sqrtf(s) : powf(s, cbn);
}
__device__ __forceinline__ float dcharb_dpred(float d, float cbn) {  // d = gt - pred
  const float s = d * d + 1e-6f;
  return cbn == 0.5f ? -d * rsqrtf(s) : -2.f * cbn * d * powf(s, cbn - 1.f);
}
// Stand-alone charbonnier_loss (loss_utils.py:34-51) for the functional API: sums[b] = sum_{p,c} ((gt-pred)^2 + 1e-6)^cbn * mask.
// mask_c = 1: one mask value per pixel (broadcast over the C channels), mask_c = C: one per element.  sums (double) must be zeroed.
__global__ void charbonnier_sum_kernel(const float* __restrict__ gt, const float* __restrict__ pred, const float* __restrict__ mask, size_t hw,
                                       int C, int mask_c, float cbn, double* __restrict__ sums) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  double acc = 0;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (size_t)gridDim.x * blockDim.x) {
    const size_t base = ((size_t)b * hw + p);
    for (int c = 0; c < C; ++c) {
      const float m = mask[mask_c == 1 ? base : base * C + c];
      acc += (double)(charb(gt[base * C + c] - pred[base * C + c], cbn) * m);
    }
  }
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) atomicAdd(sums + b, acc);
}
__global__ void cis_loss_fwd_kernel(const float* __restrict__ flow, const float* __restrict__ mask, const float* __restrict__ flow1, int B, int H,
                                    int W, int h1, int w1, float cbn, double* __restrict__ sums, float* __restrict__ pred_out) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const size_t hw = (size_t)H * W;
  float a[5] = {0, 0, 0, 0, 0};
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (size_t)gridDim.x * blockDim.x) {
    const int y = (int)(p / W), x = (int)(p % W);
    const Lerp ly = legacy_lerp(y, h1, (float)h1 / (float)H), lx = legacy_lerp(x, w1, (float)w1 / (float)W);
    const size_t pix = (size_t)b * hw + p;
    const float m = mask[pix];
    const float2 f = *reinterpret_cast<const float2*>(flow + pix * 2);
    float e[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const float2 pr = pred_at(flow1, j * B + b, h1, w1, ly, lx);
      e[j] = charb(f.x - pr.x, cbn) + charb(f.y - pr.y, cbn);
      if (pred_out) *reinterpret_cast<float2*>(pred_out + ((size_t)(j * B + b) * hw + p) * 2) = pr;
    }
    a[0] += m * e[0];           // rec           adversarial_learner.py:144
    a[1] += (1.f - m) * e[1];   // rec_compl     :149
    a[2] += e[2];               // image prior   :161
    a[3] += m * e[2];           // den_red       :179
    a[4] += (1.f - m) * e[2];   // den_red_compl :186
  }
  // block-level reduction first: one fp64 atomic per (block, sum) instead of one per warp -- tens of thousands of atomics on 20
  // addresses would serialise in L2 between the forward and the backward pass of every step
  __shared__ float red[8][5];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const float s = warp_sum(a[k]);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = s;
  }
  __syncthreads();
  if (threadIdx.x < 5) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += (double)red[w][threadIdx.x];
    atomicAdd(sums + b * 5 + threadIdx.x, t);
  }
}
__global__ void cis_loss_reduce_kernel(const double* __restrict__ sums, int B, int GB, double hw, float eps, float* __restrict__ scalars,
                                       float* __restrict__ coef) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double rec_total = 0, rr = 0, rrc = 0;
  for (int b = 0; b < B; ++b) {
    const double rec = sums[b * 5], recc = sums[b * 5 + 1], prior = sums[b * 5 + 2];
    const double D = sums[b * 5 + 3] + eps, Dc = sums[b * 5 + 4] + eps;
    rec_total += rec + recc + prior;
    rr += 1.0 - rec / D;
    rrc += 1.0 - recc / Dc;
    coef[b * 4 + 0] = (float)(-1.0 / (GB * D));
    coef[b * 4 + 1] = (float)(rec / (GB * D * D));
    coef[b * 4 + 2] = (float)(-1.0 / (GB * Dc));
    coef[b * 4 + 3] = (float)(recc / (GB * Dc * Dc));
  }
  scalars[2] = (float)(rr / GB);
  scalars[3] = (float)(rrc / GB);
  scalars[0] = scalars[2] + scalars[3];                  // generator loss  :194
  scalars[1] = (float)(rec_total / (hw * (double)GB));   // recover loss    :171-172
  scalars[4] = (float)(1.0 / (hw * (double)GB));
}
__global__ void cis_loss_bwd_kernel(const float* __restrict__ flow, const float* __restrict__ mask, const float* __restrict__ flow1,
                                    const float* __restrict__ coef, const float* __restrict__ scalars, int B, int H, int W, int h1, int w1,
                                    float cbn, int which, float* __restrict__ dpred, float* __restrict__ dmask) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const size_t hw = (size_t)H * W;
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= hw) return;
  const int y = (int)(p / W), x = (int)(p % W);
  const Lerp ly = legacy_lerp(y, h1, (float)h1 / (float)H), lx = legacy_lerp(x, w1, (float)w1 / (float)W);
  const size_t pix = (size_t)b * hw + p;
  const float m = mask[pix];
  const float2 f = *reinterpret_cast<const float2*>(flow + pix * 2);
  float2 pr[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) pr[j] = pred_at(flow1, j * B + b, h1, w1, ly, lx);
  float w0, w1c, w2;
  if (which == 0) {
    const float k = scalars[4];
    w0 = k * m; w1c = k * (1.f - m); w2 = k;
  } else {
    const float a = coef[b * 4], c = coef[b * 4 + 1], ac = coef[b * 4 + 2], ccq = coef[b * 4 + 3];
    w0 = a * m; w1c = ac * (1.f - m); w2 = c * m + ccq * (1.f - m);
    const float e0 = charb(f.x - pr[0].x, cbn) + charb(f.y - pr[0].y, cbn);
    const float e1 = charb(f.x - pr[1].x, cbn) + charb(f.y - pr[1].y, cbn);
    const float e2 = charb(f.x - pr[2].x, cbn) + charb(f.y - pr[2].y, cbn);
    dmask[pix] = a * e0 - ac * e1 + (c - ccq) * e2;
  }
  const float wj[3] = {w0, w1c, w2};
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    float2 g;
    g.x = wj[j] * dcharb_dpred(f.x - pr[j].x, cbn);
    g.y = wj[j] * dcharb_dpred(f.y - pr[j].y, cbn);
    *reinterpret_cast<float2*>(dpred + ((size_t)(j * B + b) * hw + p) * 2) = g;
  }
}
__global__ void mask_bwd_kernel(const float* __restrict__ flow, const float* __restrict__ mask, const float* __restrict__ dmd,
                                const bf16* __restrict__ din, size_t npix, bf16* __restrict__ dlogits) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const float m = mask[p];
  float dm = dmd[p];
  if (din) {      // NULL: the stand-alone mask head of the function-level generator_net (dmask -> dlogits only)
    const float f0 = flow[p * 2], f1 = flow[p * 2 + 1];
    float d0[8], d1[8];
    unpack8(*reinterpret_cast<const uint4*>(din + p * 8), d0);            // call 0 inputs [f(1-m), 1, 1-m]
    unpack8(*reinterpret_cast<const uint4*>(din + (npix + p) * 8), d1);   // call 1 inputs [f m, 1, m]
    dm += -(f0 * d0[0] + f1 * d0[1]) - d0[3];
    dm += (f0 * d1[0] + f1 * d1[1]) + d1[3];
  }
  const float dl = dm * m * (1.f - m) * 0.1f;  // m = sigmoid((l0-l1)/10)   nets.py:38-41
  const float v[8] = {dl, -dl, 0, 0, 0, 0, 0, 0};
  *reinterpret_cast<uint4*>(dlogits + p * 8) = pack8(v);
}

// ------------------------------------------------------------------------------------------------ optimiser
__global__ void grad_avg_abs_kernel(const float* __restrict__ g, const long long* __restrict__ seg, int nseg, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  // grid = (variables, kAvgAbsChunks): a variable of 2.4 M elements walked by ONE block is slow -- and on the critical path between
  // the backward pass and the optimiser of every generator step
  const int s = blockIdx.x;
  const long long a = seg[2 * s], e = seg[2 * s + 1];
  const long long per = (e - a + gridDim.y - 1) / gridDim.y;
  const long long lo = a + per * blockIdx.y, hi = lo + per < e ? lo + per : e;
  float acc = 0.f;
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) acc += fabsf(g[i]);
  __shared__ float red[32];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) atomicAdd(out, v / (float)(e - a) / (float)nseg);  // mean over variables of mean|g|  loss_utils.py:19-20
  }
}
__device__ __forceinline__ uint32_t hash32(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
  return (uint32_t)x;
}
__global__ void clip_adam_kernel(float* __restrict__ param, float* __restrict__ m, float* __restrict__ v, const float* __restrict__ grad, size_t n,
                                 float gscale, float clip, float lr, float b1, float b2, float eps, const long long* __restrict__ step,
                                 const float* __restrict__ avg_abs, int can_change, unsigned long long seed) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long t = step[0] + 1;
  float g = grad[i] * gscale;
  if (can_change && avg_abs[0] < 1e-5f) {
    const uint32_t r = hash32(seed ^ ((uint64_t)t << 40) ^ (uint64_t)i);
    g = fabsf((((float)r + 0.5f) * (1.f / 4294967296.f)) * 2.f * clip - clip);  // |U(-clip, clip)|   loss_utils.py:7-10,23
  } else {
    g = fminf(fmaxf(g, -clip), clip);                                            // loss_utils.py:4-5
  }
  const float lr_t = lr * sqrtf(1.f - powf(b2, (float)t)) / (1.f - powf(b1, (float)t));  // TF Adam (App. A.14)
  const float mi = b1 * m[i] + (1.f - b1) * g;
  const float vi = b2 * v[i] + (1.f - b2) * g * g;
  m[i] = mi;
  v[i] = vi;
  param[i] -= lr_t * mi / (sqrtf(vi) + eps);
}
__global__ void step_inc_kernel(long long* step) {
  pdl_launch_dependents();
  pdl_wait(); step[0] += 1; }
// Box occlusions of the recover-net pretraining.  Draw k of sample g at step t = hash32(seed ^ kBoxDomain ^ t<<40 ^ g<<2 ^ k): its own
// domain constant keeps it apart from the noise branch above, and integer arithmetic only keeps it restatable bit for bit on the host.
constexpr uint64_t kBoxDomain = 0x426f784d61736b73ULL;   // "BoxMasks"
__device__ __forceinline__ uint32_t box_draw(unsigned long long seed, long long t, long long g, int k) {
  return hash32((uint64_t)seed ^ kBoxDomain ^ ((uint64_t)t << 40) ^ ((uint64_t)g << 2) ^ (uint64_t)k);
}
__global__ void box_masks_kernel(float* __restrict__ mask, int H, int W, int lo_h, int hi_h, int lo_w, int hi_w, long long sample_offset,
                                 const long long* __restrict__ step, unsigned long long seed) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t hw = (size_t)H * W;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hw) return;
  const long long t = step[0], g = sample_offset + blockIdx.y;
  const uint32_t bh = (uint32_t)lo_h + box_draw(seed, t, g, 0) % (uint32_t)(hi_h - lo_h + 1);
  const uint32_t bw = (uint32_t)lo_w + box_draw(seed, t, g, 1) % (uint32_t)(hi_w - lo_w + 1);
  const uint32_t y0 = box_draw(seed, t, g, 2) % ((uint32_t)H - bh + 1);
  const uint32_t x0 = box_draw(seed, t, g, 3) % ((uint32_t)W - bw + 1);
  const uint32_t y = (uint32_t)(i / W), x = (uint32_t)(i - (size_t)y * W);
  mask[blockIdx.y * hw + i] = (y - y0 < bh && x - x0 < bw) ? 1.f : 0.f;   // unsigned: y < y0 wraps around and fails the test
}
__global__ void abs_sum_kernel(const float* __restrict__ g, size_t n, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  float acc = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) acc += fabsf(g[i]);
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}
__global__ void cast_f32_bf16_kernel(const float* __restrict__ s, size_t n, bf16* __restrict__ d) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = __float2bfloat16(s[i]);
}
__global__ void cast_bf16_f32_kernel(const bf16* __restrict__ s, size_t npix, int pitch, int coff, int C, float* __restrict__ d) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * C) return;
  const size_t p = i / C;
  const int c = (int)(i % C);
  d[i] = __bfloat162float(s[p * pitch + coff + c]);
}
__global__ void cast_bf16_f32_scaled_kernel(const bf16* __restrict__ s, size_t npix, int pitch, int coff, int C, float scale,
                                            float* __restrict__ d) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * C) return;
  const size_t p = i / C;
  const int c = (int)(i % C);
  d[i] = __bfloat162float(s[p * pitch + coff + c]) * scale;
}

// ------------------------------------------------------------------------------------------------ function-level backward
// Gradients of the stand-alone ops of models/functional.py.  The step graph never launches these.

// charbonnier_loss (loss_utils.py:34-51) backward, one thread per pixel: with g = dsum[b],
// dpred = g * m * d/dpred ((gt-pred)^2 + 1e-6)^cbn, dgt = -dpred, dmask = g * ((gt-pred)^2 + 1e-6)^cbn (mask_c = 1: summed over the
// C channels of the pixel in the thread).
__global__ void charbonnier_bwd_kernel(const float* __restrict__ gt, const float* __restrict__ pred, const float* __restrict__ mask, size_t hw,
                                       size_t npix, int C, int mask_c, float cbn, const float* __restrict__ dsum, float* __restrict__ dpred,
                                       float* __restrict__ dgt, float* __restrict__ dmask) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const float g = dsum[p / hw];
  float dm = 0.f;
  for (int c = 0; c < C; ++c) {
    const size_t e = p * C + c;
    const float d = gt[e] - pred[e];
    const float m = mask[mask_c == 1 ? p : e];
    const float dp = g * m * dcharb_dpred(d, cbn);
    if (dpred) dpred[e] = dp;
    if (dgt) dgt[e] = -dp;
    const float v = g * charb(d, cbn);
    if (mask_c == 1) dm += v;
    else if (dmask) dmask[e] = v;
  }
  if (mask_c == 1 && dmask) dmask[p] = dm;
}

// Gradient destinations of the backward kernels below, element (pixel, channel) at p[pix * pitch + off + c]: plain fp32 stores (the
// stand-alone ops) or bf16 slices of the engine's gradient buffers, overwritten or accumulated into (acc != 0; PWC-Net backward).
struct F32Out {
  float* p;
  int pitch, off;
  __device__ __forceinline__ void put(size_t pix, int c, float v) const { p[pix * pitch + off + c] = v; }
};
struct Bf16Out {
  bf16* p;
  int pitch, off, acc;
  __device__ __forceinline__ void put(size_t pix, int c, float v) const {
    bf16* q = p + pix * pitch + off + c;
    *q = __float2bfloat16(acc ? __bfloat162float(*q) + v : v);
  }
};
__device__ __forceinline__ float ldf(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ldf(const bf16* p) { return __bfloat162float(*p); }

// dense_image_warp (core_warp.py:42-202) backward, one thread per pixel.  dflow is local: the floor carries no gradient, alpha =
// clip(q - floor, 0, 1) passes it where 0 <= q - floor <= 1 (inclusive, as the gradient of tf.clip_by_value), and q = grid - fs * flow.
// dimage is a scatter (the flow is unbounded): fp64 atomics into dimg, rounded once by round_f64_kernel.  dflow.p == NULL: no dflow.
template <class OF>
__global__ void dense_image_warp_bwd_kernel(const bf16* __restrict__ img, int pitch, int coff, const float* __restrict__ flow, float fs, int B,
                                            int h, int w, int C, const float* __restrict__ dout, double* __restrict__ dimg, const OF dflow) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (size_t)B * h * w) return;
  const int x = (int)(pix % w), y = (int)((pix / w) % h), b = (int)(pix / ((size_t)w * h));
  const float qy = (float)y - flow[pix * 2] * fs, qx = (float)x - flow[pix * 2 + 1] * fs;
  int y0, x0;
  float ay, ax;
  warp_coords(qy, h, y0, ay);
  warp_coords(qx, w, x0, ax);
  const float ry = qy - (float)y0, rx = qx - (float)x0;
  const bool pass_y = ry >= 0.f && ry <= 1.f, pass_x = rx >= 0.f && rx <= 1.f;
  const size_t q00 = (size_t)(b * h + y0) * w + x0;
  const bf16* base = img + coff + q00 * pitch;
  const float* go = dout + pix * C;
  const double w00 = (1.0 - ax) * (1.0 - ay), w01 = (double)ax * (1.0 - ay), w10 = (1.0 - ax) * (double)ay, w11 = (double)ax * ay;
  float sy = 0.f, sx = 0.f;
  for (int c0 = 0; c0 < C; c0 += 8) {
    float tl[8], tr[8], bl[8], br[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(base + c0)), tl);
    unpack8(__ldg(reinterpret_cast<const uint4*>(base + pitch + c0)), tr);
    unpack8(__ldg(reinterpret_cast<const uint4*>(base + (size_t)w * pitch + c0)), bl);
    unpack8(__ldg(reinterpret_cast<const uint4*>(base + (size_t)w * pitch + pitch + c0)), br);
    const int n = min(8, C - c0);
    for (int e = 0; e < n; ++e) {
      const float g = go[c0 + e];
      const float t = ax * (tr[e] - tl[e]) + tl[e];
      const float bo = ax * (br[e] - bl[e]) + bl[e];
      sy += g * (bo - t);
      sx += g * (ay * (br[e] - bl[e]) + (1.f - ay) * (tr[e] - tl[e]));
      if (dimg) {
        const double gd = (double)g;
        atomicAdd(dimg + q00 * C + c0 + e, gd * w00);
        atomicAdd(dimg + (q00 + 1) * C + c0 + e, gd * w01);
        atomicAdd(dimg + (q00 + w) * C + c0 + e, gd * w10);
        atomicAdd(dimg + (q00 + w + 1) * C + c0 + e, gd * w11);
      }
    }
  }
  if (dflow.p) {
    dflow.put(pix, 0, pass_y ? -fs * sy : 0.f);
    dflow.put(pix, 1, pass_x ? -fs * sx : 0.f);
  }
}
// The four output-parity planes of a 2H x 2W gradient slice (C <= 8 channels from channel sc, any alignment): plane a*2+b, pixel (n,y,x) =
// src(n, 2y + a, 2x + b) as one zero-padded 8-channel chunk -- the gradient operands of a k4 s2 transposed conv's weight gradient.
__global__ void parity_split_bf16_kernel(const bf16* __restrict__ src, int sp, int sc, int N, int H, int W, int C, bf16* __restrict__ dst, int dp) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t npix = (size_t)N * H * W;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 4 * npix) return;
  const int q = (int)(i / npix);
  const size_t pix = i - (size_t)q * npix;
  const int x = (int)(pix % W), y = (int)((pix / W) % H), n = (int)(pix / ((size_t)W * H));
  const bf16* s = src + ((size_t)(n * 2 * H + 2 * y + (q >> 1)) * 2 * W + 2 * x + (q & 1)) * sp + sc;
  float v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = c < C ? __bfloat162float(s[c]) : 0.f;
  *reinterpret_cast<uint4*>(dst + i * dp) = pack8(v);
}
// the fp64 scatter sums [npix][C], rounded once into their destination
template <class O>
__global__ void round_f64_kernel(const double* __restrict__ s, size_t npix, int C, const O d) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < npix * C) d.put(i / C, (int)(i % C), (float)s[i]);
}

// cost_volume (core_costvol.py:20-40) backward, and with flow != NULL the backward of cis_warp_costvol's fused warp, search range R.
// Pass 1: gs[p][d] = dout[p][d] * leaky0.1'(pre[p][d]) / C, the pre-activation recomputed from the bf16 c1 / c2 slices through the
// forward's 8x16 tile + (8+2R)x(16+2R) zero-padded halo staging (c2 warped by fs * flow in the halo, as the forward does).  dout: fp32 or
// a bf16 slice, element d of pixel p at dout[p * dp + doff + d]; gs is [npix][(2R+1)^2].
template <int R, typename TD>
__global__ void __launch_bounds__(256, cv_min_blocks(R)) costvol_bwd_gate_kernel(const bf16* __restrict__ c1, int c1p, int c1o, const bf16* __restrict__ c2, int c2p,
                                                               int c2o, const float* __restrict__ flow, float fs, const TD* __restrict__ dout,
                                                               int dp, int doff, int B, int h, int w, int C, float* __restrict__ gs) {
  constexpr int S = cv_span(R), ND = cv_ndisp(R), HH = cv_hh(R), HW = cv_hw(R);
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float cvs[];
  float* s1 = cvs;                                 // [128][36]
  float* s2 = cvs + kCvTH * kCvTW * kCvPitch;      // [HH * HW][36]
  const int tid = threadIdx.x;
  const int b = blockIdx.z, y0 = blockIdx.y * kCvTH, x0 = blockIdx.x * kCvTW;
  const int pix = tid & 127, py = pix >> 4, px = pix & 15;
  const int dyb = tid >> 7;  // this thread handles dy = dyb + 2k
  float acc[R + 1][S];
#pragma unroll
  for (int k = 0; k < R + 1; ++k)
#pragma unroll
    for (int d = 0; d < S; ++d) acc[k][d] = 0.f;
  const int Cp = (C + 7) & ~7;
  for (int cc = 0; cc < Cp; cc += 32) {
    const int nck = min(4, (Cp - cc) / 8);
    for (int it = tid; it < 128 * 4; it += 256) {
      const int p = it >> 2, ck = it & 3;
      const int y = y0 + (p >> 4), x = x0 + (p & 15);
      float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (ck < nck && y < h && x < w) unpack8(__ldg(reinterpret_cast<const uint4*>(c1 + ((size_t)(b * h + y) * w + x) * c1p + c1o + cc + ck * 8)), v);
      float4* d = reinterpret_cast<float4*>(s1 + p * kCvPitch + ck * 8);
      d[0] = make_float4(v[0], v[1], v[2], v[3]);
      d[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    for (int it = tid; it < HH * HW * 4; it += 256) {
      const int p = it >> 2, ck = it & 3;
      const int y = y0 - R + p / HW, x = x0 - R + p % HW;
      float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (ck < nck && y >= 0 && y < h && x >= 0 && x < w) {
        if (flow) {
          const size_t fp = ((size_t)(b * h + y) * w + x) * 2;
          warp_chunk(c2 + c2o + cc + ck * 8, c2p, h, w, b, (float)y - __ldg(flow + fp) * fs, (float)x - __ldg(flow + fp + 1) * fs, v);
        } else {
          unpack8(__ldg(reinterpret_cast<const uint4*>(c2 + ((size_t)(b * h + y) * w + x) * c2p + c2o + cc + ck * 8)), v);
        }
      }
      float4* d = reinterpret_cast<float4*>(s2 + p * kCvPitch + ck * 8);
      d[0] = make_float4(v[0], v[1], v[2], v[3]);
      d[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < R + 1; ++k) {
      const int dy = dyb + 2 * k;
      if (dy < S) {
        const float* r2 = s2 + ((py + dy) * HW + px) * kCvPitch;
        const float* r1 = s1 + pix * kCvPitch;
        for (int c4 = 0; c4 < nck * 2; ++c4) {
          const float4 a = *reinterpret_cast<const float4*>(r1 + c4 * 4);
#pragma unroll
          for (int dx = 0; dx < S; ++dx) {
            const float4 q = *reinterpret_cast<const float4*>(r2 + dx * kCvPitch + c4 * 4);
            acc[k][dx] += a.x * q.x + a.y * q.y + a.z * q.z + a.w * q.w;
          }
        }
      }
    }
    __syncthreads();
  }
  const int y = y0 + py, x = x0 + px;
  if (y >= h || x >= w) return;
  const size_t q = (size_t)(b * h + y) * w + x, o = q * ND;
  const TD* dq = dout + q * dp + doff;
  const float inv = 1.f / (float)C;
#pragma unroll
  for (int k = 0; k < R + 1; ++k) {
    const int dy = dyb + 2 * k;
    if (dy < S) {
#pragma unroll
      for (int dx = 0; dx < S; ++dx) gs[o + dy * S + dx] = ldf(dq + dy * S + dx) * (acc[k][dx] * inv > 0.f ? inv : 0.1f * inv);
    }
  }
}
// Pass 2, both sums as gathers over the (2R+1)^2 displacements (fixed order, no atomics):
//   dc1[p]   = sum_d gs[p][d]     * warp[p + d]
//   dwarp[q] = sum_d gs[q - d][d] * c1[q - d]
// A CTA owns an 8x16 pixel tile.  It stages gs of its own pixels ([128][ND]) and the shifted planes gs[q - d][d] ([ND][128], zero where
// q - d leaves the map: those displacements read the zero padding in the forward) once, then c1 and warp (8+2R)x(16+2R) halos per
// 32-channel pass (flow != NULL: the warp halo recomputed from c2 and fs * flow, never stored in HBM).
constexpr int cv_bwd_smem(int R) { return (2 * kCvTH * kCvTW * cv_ndisp(R) + 2 * cv_hh(R) * cv_hw(R) * kCvPitch) * 4; }
static_assert(cv_bwd_smem(kCvRMax) == 193536 && cv_bwd_smem(kCvRMax + 1) > 227 * 1024, "R = 4 is the largest range that fits a block");
template <int R, class O1, class O2>
__global__ void __launch_bounds__(256, cv_min_blocks(R)) costvol_bwd_kernel(const bf16* __restrict__ c1, int c1p, int c1o, const bf16* __restrict__ c2, int c2p,
                                                          int c2o, const float* __restrict__ flow, float fs, const float* __restrict__ gs, int B,
                                                          int h, int w, int C, const O1 dc1, const O2 dwarp) {
  constexpr int S = cv_span(R), ND = cv_ndisp(R), HH = cv_hh(R), HW = cv_hw(R);
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float cvs[];
  float* gself = cvs;                              // [128][ND]
  float* gsh = gself + kCvTH * kCvTW * ND;         // [ND][128]
  float* h1 = gsh + kCvTH * kCvTW * ND;            // c1 halo   [HH * HW][36]
  float* h2 = h1 + HH * HW * kCvPitch;             // warp halo [HH * HW][36]
  const int tid = threadIdx.x;
  const int b = blockIdx.z, y0 = blockIdx.y * kCvTH, x0 = blockIdx.x * kCvTW;
  for (int it = tid; it < kCvTH * kCvTW * ND; it += 256) {
    const int p = it / ND, d = it % ND;
    const int y = y0 + (p >> 4), x = x0 + (p & 15);
    gself[it] = (y < h && x < w) ? __ldg(gs + ((size_t)(b * h + y) * w + x) * ND + d) : 0.f;
  }
  for (int it = tid; it < kCvTH * kCvTW * ND; it += 256) {
    const int d = it >> 7, q = it & 127;
    const int y = y0 + (q >> 4) - (d / S - R), x = x0 + (q & 15) - (d % S - R);
    gsh[it] = (y >= 0 && y < h && x >= 0 && x < w) ? __ldg(gs + ((size_t)(b * h + y) * w + x) * ND + d) : 0.f;
  }
  const int pix = tid & 127, py = pix >> 4, px = pix & 15;
  const int ck0 = (tid >> 7) * 2;   // this thread's two 8-channel chunks of the pass
  const int oy = y0 + py, ox = x0 + px;
  const bool own = oy < h && ox < w;
  const size_t op = (size_t)(b * h + oy) * w + ox;
  const int Cp = (C + 7) & ~7;
  for (int cc = 0; cc < Cp; cc += 32) {
    const int nck = min(4, (Cp - cc) / 8);
    for (int it = tid; it < HH * HW * 4; it += 256) {
      const int p = it >> 2, ck = it & 3;
      const int y = y0 - R + p / HW, x = x0 - R + p % HW;
      float v1[8] = {0, 0, 0, 0, 0, 0, 0, 0}, v2[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (ck < nck && y >= 0 && y < h && x >= 0 && x < w) {
        const size_t q = (size_t)(b * h + y) * w + x;
        unpack8(__ldg(reinterpret_cast<const uint4*>(c1 + q * c1p + c1o + cc + ck * 8)), v1);
        if (flow)
          warp_chunk(c2 + c2o + cc + ck * 8, c2p, h, w, b, (float)y - __ldg(flow + 2 * q) * fs, (float)x - __ldg(flow + 2 * q + 1) * fs, v2);
        else
          unpack8(__ldg(reinterpret_cast<const uint4*>(c2 + q * c2p + c2o + cc + ck * 8)), v2);
      }
      float4* d1 = reinterpret_cast<float4*>(h1 + p * kCvPitch + ck * 8);
      float4* d2 = reinterpret_cast<float4*>(h2 + p * kCvPitch + ck * 8);
      d1[0] = make_float4(v1[0], v1[1], v1[2], v1[3]);
      d1[1] = make_float4(v1[4], v1[5], v1[6], v1[7]);
      d2[0] = make_float4(v2[0], v2[1], v2[2], v2[3]);
      d2[1] = make_float4(v2[4], v2[5], v2[6], v2[7]);
    }
    __syncthreads();
    if (ck0 < nck) {
      float a1[16], a2[16];
#pragma unroll
      for (int e = 0; e < 16; ++e) a1[e] = a2[e] = 0.f;
      for (int dy = 0; dy < S; ++dy) {
        for (int dx = 0; dx < S; ++dx) {
          const int d = dy * S + dx;
          const float g1 = gself[pix * ND + d], g2 = gsh[d * 128 + pix];
          const float* r2 = h2 + ((py + dy) * HW + px + dx) * kCvPitch + ck0 * 8;                    // warp[p + d]
          const float* r1 = h1 + ((py + 2 * R - dy) * HW + px + 2 * R - dx) * kCvPitch + ck0 * 8;    // c1[q - d]
#pragma unroll
          for (int e4 = 0; e4 < 4; ++e4) {
            const float4 u = *reinterpret_cast<const float4*>(r2 + e4 * 4);
            const float4 v = *reinterpret_cast<const float4*>(r1 + e4 * 4);
            a1[e4 * 4 + 0] += g1 * u.x; a1[e4 * 4 + 1] += g1 * u.y; a1[e4 * 4 + 2] += g1 * u.z; a1[e4 * 4 + 3] += g1 * u.w;
            a2[e4 * 4 + 0] += g2 * v.x; a2[e4 * 4 + 1] += g2 * v.y; a2[e4 * 4 + 2] += g2 * v.z; a2[e4 * 4 + 3] += g2 * v.w;
          }
        }
      }
      if (own) {
        const int cbase = cc + ck0 * 8;
        const int n = min(16, C - cbase);
        for (int e = 0; e < n; ++e) {
          dc1.put(op, cbase + e, a1[e]);
          dwarp.put(op, cbase + e, a2[e]);
        }
      }
    }
    __syncthreads();
  }
}

}  // namespace cis

using namespace cis;
#include <stdlib.h>
#include <string.h>

// every kernel here starts with griddepcontrol.launch_dependents + griddepcontrol.wait, so it may be launched with programmatic
// stream serialization: its CTAs are scheduled while the previous kernel drains (CIS_PDL=0 turns the attribute off).
static bool misc_pdl_enabled() {
  static const bool on = !(getenv("CIS_PDL") && atoi(getenv("CIS_PDL")) == 0);
  return on;
}
template <typename... KArgs, typename... Args>
static void cis_launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
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
  cfg.numAttrs = misc_pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
#define CIS_LAUNCH(kern, grid, block, smem, st, ...) cis_launch(kern, dim3(grid), dim3(block), (size_t)(smem), st, __VA_ARGS__)
#define ST ((cudaStream_t)stream)
static inline unsigned nblk(size_t n, int t = 256) { return (unsigned)((n + t - 1) / t); }
typedef const __nv_bfloat16* cbf;
typedef __nv_bfloat16* mbf;

// ---- warp + cost volume, forward and backward, for search range R (the three entry points without a range argument are R = 4)
template <int R>
static int warp_costvol_fwd(const void* c1, int32_t c1p, int32_t c1o, const void* c2, int32_t c2p, int32_t c2o, const float* flow, float fs,
                            int32_t B, int32_t h, int32_t w, int32_t C, void* out, int32_t op, int32_t oo, cis_stream_t stream) {
  if (h < 2 || w < 2) return cis_set_error(CIS_ERR_BAD_ARG, "cis_warp_costvol: needs h,w >= 2 (core_warp.py:188)");
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(warp_costvol_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, cv_smem(R));
    if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaFuncSetAttribute(warp_costvol)");
    attr = true;
  }
  dim3 grid((w + kCvTW - 1) / kCvTW, (h + kCvTH - 1) / kCvTH, B);
  CIS_LAUNCH(warp_costvol_kernel<R>, grid, 256, cv_smem(R), ST, (cbf)c1, c1p, c1o, (cbf)c2, c2p, c2o, flow, fs, B, h, w, C, (mbf)out, op, oo);
  return cis_check_launch("warp_costvol");
}
template <int R>
static int cost_volume_bwd(const void* c1, int32_t c1p, int32_t c1o, const void* warp, int32_t wp, int32_t wo, const float* dout, int32_t B,
                           int32_t h, int32_t w, int32_t C, float* gscratch, float* dc1, float* dwarp, cis_stream_t stream) {
  if (h < 2 || w < 2) return cis_set_error(CIS_ERR_BAD_ARG, "cis_cost_volume_bwd: needs h,w >= 2 (core_warp.py:188)");
  if (!gscratch || !dc1 || !dwarp) return cis_set_error(CIS_ERR_BAD_ARG, "cis_cost_volume_bwd: NULL output or scratch");
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(costvol_bwd_gate_kernel<R, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, cv_smem(R));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(costvol_bwd_kernel<R, F32Out, F32Out>, cudaFuncAttributeMaxDynamicSharedMemorySize, cv_bwd_smem(R));
    if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaFuncSetAttribute(costvol_bwd)");
    attr = true;
  }
  dim3 grid((w + kCvTW - 1) / kCvTW, (h + kCvTH - 1) / kCvTH, B);
  CIS_LAUNCH((costvol_bwd_gate_kernel<R, float>), grid, 256, cv_smem(R), ST, (cbf)c1, c1p, c1o, (cbf)warp, wp, wo, (const float*)nullptr, 1.f, dout,
             cv_ndisp(R), 0, B, h, w, C, gscratch);
  CIS_LAUNCH((costvol_bwd_kernel<R, F32Out, F32Out>), grid, 256, cv_bwd_smem(R), ST, (cbf)c1, c1p, c1o, (cbf)warp, wp, wo, (const float*)nullptr,
             1.f, (const float*)gscratch, B, h, w, C, F32Out{dc1, C, 0}, F32Out{dwarp, C, 0});
  return cis_check_launch("cost_volume_bwd");
}
template <int R>
static int warp_costvol_bwd(const void* c1, int32_t c1p, int32_t c1o, const void* c2, int32_t c2p, int32_t c2o, const float* flow, float fs,
                            int32_t B, int32_t h, int32_t w, int32_t C, const void* dcorr, int32_t dcp, int32_t dco, void* dc1, int32_t dc1p,
                            int32_t dc1o, void* dc2, int32_t dc2p, int32_t dc2o, void* dflow, int32_t dfp, int32_t dfo, int32_t accumulate,
                            float* gscratch, float* wscratch, double* dscratch, cis_stream_t stream) {
  if (h < 2 || w < 2) return cis_set_error(CIS_ERR_BAD_ARG, "cis_warp_costvol_bwd: needs h,w >= 2 (core_warp.py:188)");
  if (!dcorr || !dc1 || !dc2 || !gscratch) return cis_set_error(CIS_ERR_BAD_ARG, "cis_warp_costvol_bwd: NULL gradient or scratch");
  if (flow && (!dflow || !wscratch || !dscratch)) return cis_set_error(CIS_ERR_BAD_ARG, "cis_warp_costvol_bwd: the warp needs dflow and scratch");
  if ((c1p | c1o | c2p | c2o) & 7) return cis_set_error(CIS_ERR_BAD_ARG, "cis_warp_costvol_bwd: feature slices must be 8-channel aligned");
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(costvol_bwd_gate_kernel<R, bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, cv_smem(R));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(costvol_bwd_kernel<R, Bf16Out, F32Out>, cudaFuncAttributeMaxDynamicSharedMemorySize, cv_bwd_smem(R));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(costvol_bwd_kernel<R, Bf16Out, Bf16Out>, cudaFuncAttributeMaxDynamicSharedMemorySize, cv_bwd_smem(R));
    if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaFuncSetAttribute(warp_costvol_bwd)");
    attr = true;
  }
  const Bf16Out o1{(mbf)dc1, dc1p, dc1o, accumulate & 1}, o2{(mbf)dc2, dc2p, dc2o, (accumulate >> 1) & 1};
  dim3 grid((w + kCvTW - 1) / kCvTW, (h + kCvTH - 1) / kCvTH, B);
  CIS_LAUNCH((costvol_bwd_gate_kernel<R, bf16>), grid, 256, cv_smem(R), ST, (cbf)c1, c1p, c1o, (cbf)c2, c2p, c2o, flow, fs, (cbf)dcorr, dcp, dco, B,
             h, w, C, gscratch);
  if (!flow) {       // level 6: no warp, dwarp is dc2
    CIS_LAUNCH((costvol_bwd_kernel<R, Bf16Out, Bf16Out>), grid, 256, cv_bwd_smem(R), ST, (cbf)c1, c1p, c1o, (cbf)c2, c2p, c2o, flow, fs,
               (const float*)gscratch, B, h, w, C, o1, o2);
    return cis_check_launch("warp_costvol_bwd");
  }
  CIS_LAUNCH((costvol_bwd_kernel<R, Bf16Out, F32Out>), grid, 256, cv_bwd_smem(R), ST, (cbf)c1, c1p, c1o, (cbf)c2, c2p, c2o, flow, fs,
             (const float*)gscratch, B, h, w, C, o1, F32Out{wscratch, C, 0});
  const size_t npix = (size_t)B * h * w;
  cudaError_t e = cudaMemsetAsync(dscratch, 0, npix * C * sizeof(double), ST);
  if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaMemsetAsync");
  CIS_LAUNCH(dense_image_warp_bwd_kernel<Bf16Out>, nblk(npix), 256, 0, ST, (cbf)c2, c2p, c2o, flow, fs, B, h, w, C, (const float*)wscratch, dscratch,
             Bf16Out{(mbf)dflow, dfp, dfo, (accumulate >> 2) & 1});
  CIS_LAUNCH(round_f64_kernel<Bf16Out>, nblk(npix * C), 256, 0, ST, (const double*)dscratch, npix, C, o2);
  return cis_check_launch("warp_costvol_bwd");
}
#define CIS_CV_DISPATCH(fn, what, ...)                                                                                  \
  switch (search_range) {                                                                                              \
    case 1: return fn<1>(__VA_ARGS__);                                                                                 \
    case 2: return fn<2>(__VA_ARGS__);                                                                                 \
    case 3: return fn<3>(__VA_ARGS__);                                                                                 \
    case 4: return fn<4>(__VA_ARGS__);                                                                                 \
    default: return cis_set_error(CIS_ERR_BAD_ARG, what ": search_range must be 1, 2, 3 or 4");                       \
  }

// ------------------------------------------------------------------------------------------------ PWC-Net training
// Multi-scale flow loss (cis_flow_multiscale_loss).  Level i = 0..4 is pyramid level l = 6 - i at (H >> l) x (W >> l).  The target is
// sampled from the ground truth on the fly with the legacy bilinear rule of resize_bilinear_f32_kernel<false>, vectors times f = s_c / 2^l.
struct FlowLossArgs {
  CisFlowPyr pyr;
  const float* gt;
  int B, H, W, GH, GW;
  float s0, s1;
  int robust;
  float eps, q;
};
__device__ __forceinline__ float2 flow_level_diff(const FlowLossArgs& a, int i, int b, int y, int x) {
  const int l = 6 - i, h = a.H >> l, w = a.W >> l;
  const Lerp ly = legacy_lerp(y, a.GH, (float)a.GH / (float)h), lx = legacy_lerp(x, a.GW, (float)a.GW / (float)w);
  const float* g = a.gt + (size_t)b * a.GH * a.GW * 2;
  const float2 tl = *reinterpret_cast<const float2*>(g + ((size_t)ly.lo * a.GW + lx.lo) * 2);
  const float2 tr = *reinterpret_cast<const float2*>(g + ((size_t)ly.lo * a.GW + lx.hi) * 2);
  const float2 bl = *reinterpret_cast<const float2*>(g + ((size_t)ly.hi * a.GW + lx.lo) * 2);
  const float2 br = *reinterpret_cast<const float2*>(g + ((size_t)ly.hi * a.GW + lx.hi) * 2);
  const float t0 = tl.x + (tr.x - tl.x) * lx.f, b0 = bl.x + (br.x - bl.x) * lx.f;
  const float t1 = tl.y + (tr.y - tl.y) * lx.f, b1 = bl.y + (br.y - bl.y) * lx.f;
  const float inv = 1.f / (float)(1 << l);   // exact
  const float2 f = *reinterpret_cast<const float2*>(a.pyr.flow[i] + (((size_t)b * h + y) * w + x) * 2);
  return make_float2(f.x - (t0 + (b0 - t0) * ly.f) * (a.s0 * inv), f.y - (t1 + (b1 - t1) * ly.f) * (a.s1 * inv));
}
// pass 1: block x of (sample b, level i) sums rho over a fixed pixel subset (grid-stride) in double, reduced warp butterfly -> the 8 warps
// in index order into part[(i * B + b) * kFlowStdBlocks + x]
__global__ void flow_loss_sums_kernel(FlowLossArgs a, double* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double sm[8];
  const int b = blockIdx.y, i = blockIdx.z, l = 6 - i, w = a.W >> l;
  const size_t hw = (size_t)(a.H >> l) * w;
  double s = 0;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < hw; p += (size_t)gridDim.x * blockDim.x) {
    const float2 d = flow_level_diff(a, i, b, (int)(p / w), (int)(p % w));
    if (a.robust) s += pow(fabs((double)d.x) + fabs((double)d.y) + (double)a.eps, (double)a.q);
    else s += sqrt((double)d.x * d.x + (double)d.y * d.y);
  }
  s = warp_sum_d(s);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += sm[k];
    part[((size_t)i * a.B + b) * gridDim.x + blockIdx.x] = t;
  }
}
// pass 2: one block per sample, thread i adds level i's kFlowStdBlocks partials in block order
__global__ void flow_loss_reduce_kernel(const double* __restrict__ part, int B, double* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, i = threadIdx.x;
  double t = 0;
  for (int q = 0; q < kFlowStdBlocks; ++q) t += part[((size_t)i * B + b) * kFlowStdBlocks + q];
  out[b * 5 + i] = t;
}
// backward: one thread per pixel of the five levels, levels laid end to end (i = 0 first)
__global__ void flow_loss_bwd_kernel(FlowLossArgs a, size_t total) {
  pdl_launch_dependents();
  pdl_wait();
  size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  int i = 0;
  for (; i < 4; ++i) {
    const size_t n = (size_t)a.B * (a.H >> (6 - i)) * (a.W >> (6 - i));
    if (p < n) break;
    p -= n;
  }
  const int l = 6 - i, h = a.H >> l, w = a.W >> l;
  const int x = (int)(p % w), y = (int)((p / w) % h), b = (int)(p / ((size_t)w * h));
  const float2 d = flow_level_diff(a, i, b, y, x);
  float g0, g1;
  if (a.robust) {
    const float k = a.q * powf(fabsf(d.x) + fabsf(d.y) + a.eps, a.q - 1.f);
    g0 = d.x > 0.f ? k : (d.x < 0.f ? -k : 0.f);
    g1 = d.y > 0.f ? k : (d.y < 0.f ? -k : 0.f);
  } else {
    const float n = sqrtf(d.x * d.x + d.y * d.y);
    g0 = n > 0.f ? d.x / n : 0.f;
    g1 = n > 0.f ? d.y / n : 0.f;
  }
  const float wt = a.pyr.weight[i];
  const Bf16Out o{(bf16*)a.pyr.grad[i], a.pyr.pitch[i], a.pyr.c_off[i], a.pyr.accumulate[i]};
  o.put(p, 0, wt * g0);
  o.put(p, 1, wt * g1);
}
// TF-Adam on grad + decay * param inside the kernel segments (binary search over the sorted segment starts), no clip
__global__ void adam_l2_kernel(float* __restrict__ param, float* __restrict__ m, float* __restrict__ v, const float* __restrict__ grad, size_t n,
                               const long long* __restrict__ seg, int nseg, float decay, const float* __restrict__ lr, float b1, float b2, float eps,
                               const long long* __restrict__ step) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lo = 0, hi = nseg;                      // first segment whose start is > i
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (seg[2 * mid] <= (long long)i) lo = mid + 1;
    else hi = mid;
  }
  const float w = param[i];
  float g = grad[i];
  if (lo > 0 && (long long)i < seg[2 * (lo - 1) + 1]) g += decay * w;
  const long long t = step[0] + 1;
  const float lr_t = lr[0] * sqrtf(1.f - powf(b2, (float)t)) / (1.f - powf(b1, (float)t));
  const float mi = b1 * m[i] + (1.f - b1) * g;
  const float vi = b2 * v[i] + (1.f - b2) * g * g;
  m[i] = mi;
  v[i] = vi;
  param[i] = w - lr_t * mi / (sqrtf(vi) + eps);
}
static int flow_loss_args(const char* what, const CisFlowPyr* pyr, const float* gt, int32_t B, int32_t H, int32_t W, int32_t GH, int32_t GW,
                          float s0, float s1, int32_t robust, float eps, float q, FlowLossArgs& a) {
  if (!pyr || !gt || B < 1 || B > 65535 || H < 64 || W < 64 || H % 64 || W % 64 || GH < 1 || GW < 1 || (robust != 0 && robust != 1))
    return cis_set_error(CIS_ERR_BAD_ARG, what);
  // gt and the level flows are read as float2: 8-byte aligned pairs
  if ((uintptr_t)gt & 7) return cis_set_error(CIS_ERR_BAD_ARG, what);
  for (int i = 0; i < 5; ++i)
    if (!pyr->flow[i] || ((uintptr_t)pyr->flow[i] & 7)) return cis_set_error(CIS_ERR_BAD_ARG, what);
  a = FlowLossArgs{*pyr, gt, B, H, W, GH, GW, s0, s1, robust, eps, q};
  return CIS_OK;
}

// ------------------------------------------------------------------------------------------------ unsupervised flow loss
// Occlusion-masked census + edge-aware second-order smoothness (cis_unsup_flow_loss, formulas in cis_b200.h).  Direction n < B runs
// pair (img1, img2) of sample n, direction n >= B the swapped pair of sample n - B; S / T = first / second frame of the direction.
// Launches: (1) unsup_warp_mask_kernel, one thread per pixel: T~ and M;  (2) unsup_census_kernel, 64 blocks per direction walking
// 16x32 tiles whose 22x38 halo (3-pixel apron) of g(S) and T~ sits in shared memory: c, psi, k = M psi'(c), and the smoothness term
// read from global memory, summed in double, block partials in a fixed order;  (3) unsup_reduce_kernel: the 64 partials per direction
// in block order.  The backward is one launch of unsup_bwd_kernel over the same tiles (g(S), T~ and k halos).
constexpr int kUnsupTY = 16, kUnsupTX = 32, kUnsupR = 3, kUnsupHY = kUnsupTY + 2 * kUnsupR, kUnsupHX = kUnsupTX + 2 * kUnsupR;
constexpr int kUnsupBlocks = 64;
struct UnsupArgs {
  const float* flow;
  const float* img1;
  const float* img2;
  int B, H, W;
};
__device__ __forceinline__ const float* unsup_frame(const UnsupArgs& a, int n, bool second) {
  const bool fwd = n < a.B;
  const float* f = (fwd != second) ? a.img1 : a.img2;
  return f + (size_t)(fwd ? n : n - a.B) * a.H * a.W * 3;
}
// g(I) = 255 (0.2989 R + 0.5870 G + 0.1140 B) of I + 0.5, I = one frame's fp32 RGB.  In double, rounded once: the census divides
// gray-level differences by sqrt(0.81 + v^2), so their fp32 rounding (not the frames') sets the precision of the loss.
__device__ __forceinline__ float unsup_gray(const float* f, size_t pix) {
  const float* p = f + pix * 3;
  return (float)(255.0 * (0.2989 * ((double)p[0] + 0.5) + 0.5870 * ((double)p[1] + 0.5) + 0.1140 * ((double)p[2] + 0.5)));
}
// dense_image_warp's sample of g(T) at q: the four corners, the clamped floor, alpha and r = q - floor (the gradient passes where
// 0 <= r <= 1).  q = p - F in double: in fp32 its rounding (2^-17 at x = 640) moves the sample by more than the census resolves.
struct UnsupSample {
  int y0, x0;
  float ay, ax, tl, tr, bl, br;
  bool pass_y, pass_x;
};
__device__ __forceinline__ void unsup_coords(double q, int size, int& lo, float& a, bool& pass) {
  const double fl = fmin(fmax(floor(q), 0.0), (double)(size - 2)), r = q - fl;
  lo = (int)fl;
  a = (float)fmin(fmax(r, 0.0), 1.0);
  pass = r >= 0.0 && r <= 1.0;
}
__device__ __forceinline__ UnsupSample unsup_sample(const float* T, int H, int W, double qy, double qx) {
  UnsupSample s;
  unsup_coords(qy, H, s.y0, s.ay, s.pass_y);
  unsup_coords(qx, W, s.x0, s.ax, s.pass_x);
  const size_t q00 = (size_t)s.y0 * W + s.x0;
  s.tl = unsup_gray(T, q00);
  s.tr = unsup_gray(T, q00 + 1);
  s.bl = unsup_gray(T, q00 + W);
  s.br = unsup_gray(T, q00 + W + 1);
  return s;
}
// the census transform's soft sign of a difference, t = v / sqrt(0.81 + v^2)
__device__ __forceinline__ float unsup_t(float v) { return v * rsqrtf(0.81f + v * v); }
// second-order smoothness of axis (dy, dx) at (y, x), the centre inside [1, size-2] along the axis: weight w and the second differences
// l_c = F_c(p+e) - 2F_c(p) + F_c(p-e), in double and set to 0 when |l_c| <= 2^-18 (|F_c(p+e)| + 2|F_c(p)| + |F_c(p-e)|): fp32 flows
// cannot hold an exactly linear run (the final x4 bilinear upsampling makes three pixels in four one), so its second difference is
// rounding noise, whose sign -- the gradient of |.| -- would be noise too
__device__ __forceinline__ void unsup_smooth_terms(const UnsupArgs& a, int n, int y, int x, int dy, int dx, float& w, double l[2]) {
  const float* S = unsup_frame(a, n, false);
  const size_t pp = (size_t)(y + dy) * a.W + (x + dx), pm = (size_t)(y - dy) * a.W + (x - dx), p0 = (size_t)y * a.W + x;
  const float e = fabsf(S[pp * 3] - S[pm * 3]) + fabsf(S[pp * 3 + 1] - S[pm * 3 + 1]) + fabsf(S[pp * 3 + 2] - S[pm * 3 + 2]);
  w = expf(-10.f * (e * (1.f / 3.f)) * 0.5f);
  const float2* F = reinterpret_cast<const float2*>(a.flow) + (size_t)n * a.H * a.W;
  const float2 fp = F[pp], f0 = F[p0], fm = F[pm];
  l[0] = (double)fp.x - 2.0 * (double)f0.x + (double)fm.x;
  l[1] = (double)fp.y - 2.0 * (double)f0.y + (double)fm.y;
  if (fabs(l[0]) <= 0x1p-18 * (fabs((double)fp.x) + 2.0 * fabs((double)f0.x) + fabs((double)fm.x))) l[0] = 0.0;
  if (fabs(l[1]) <= 0x1p-18 * (fabs((double)fp.y) + 2.0 * fabs((double)f0.y) + fabs((double)fm.y))) l[1] = 0.0;
}
// (1) per pixel of direction n: T~(p) = g(T) at q = p - F(p), and M(p) = V(p) (1 - O(p)) with the partner direction's flow sampled at q
__global__ void unsup_warp_mask_kernel(UnsupArgs a, float* __restrict__ warped, float* __restrict__ mask) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t hw = (size_t)a.H * a.W, i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * (size_t)a.B * hw) return;
  const int n = (int)(i / hw), p = (int)(i % hw), y = p / a.W, x = p % a.W;
  const float2 f = reinterpret_cast<const float2*>(a.flow)[i];
  const double qy = (double)y - f.x, qx = (double)x - f.y;
  const UnsupSample s = unsup_sample(unsup_frame(a, n, true), a.H, a.W, qy, qx);
  const float top = s.ax * (s.tr - s.tl) + s.tl, bot = s.ax * (s.br - s.bl) + s.bl;
  warped[i] = s.ay * (bot - top) + top;
  const int m = n < a.B ? n + a.B : n - a.B;
  const float2* G = reinterpret_cast<const float2*>(a.flow) + (size_t)m * hw + (size_t)s.y0 * a.W + s.x0;
  const float2 g00 = G[0], g01 = G[1], g10 = G[a.W], g11 = G[a.W + 1];
  const float t0 = s.ax * (g01.x - g00.x) + g00.x, b0 = s.ax * (g11.x - g10.x) + g10.x;
  const float t1 = s.ax * (g01.y - g00.y) + g00.y, b1 = s.ax * (g11.y - g10.y) + g10.y;
  const float h0 = s.ay * (b0 - t0) + t0, h1 = s.ay * (b1 - t1) + t1;
  const float s0 = f.x + h0, s1 = f.y + h1;
  const bool vis = qy >= 0.0 && qy <= (double)(a.H - 1) && qx >= 0.0 && qx <= (double)(a.W - 1);
  const bool occ = s0 * s0 + s1 * s1 > 0.01f * (f.x * f.x + f.y * f.y + h0 * h0 + h1 * h1) + 0.5f;
  mask[i] = (vis && !occ) ? 1.f : 0.f;
}
// the halo of tile (ty0, tx0) of direction n: g(S), T~ and, for the backward, k; zero outside the frame (never read there)
__device__ __forceinline__ void unsup_load_halo(const UnsupArgs& a, int n, int ty0, int tx0, const float* __restrict__ warped,
                                                const float* __restrict__ coef, float (*gs)[kUnsupHX], float (*tw)[kUnsupHX],
                                                float (*kk)[kUnsupHX]) {
  const float* S = unsup_frame(a, n, false);
  const size_t base = (size_t)n * a.H * a.W;
  for (int e = threadIdx.x; e < kUnsupHY * kUnsupHX; e += blockDim.x) {
    const int hy = e / kUnsupHX, hx = e % kUnsupHX, y = ty0 + hy - kUnsupR, x = tx0 + hx - kUnsupR;
    const bool in = y >= 0 && y < a.H && x >= 0 && x < a.W;
    const size_t p = in ? (size_t)y * a.W + x : 0;
    gs[hy][hx] = in ? unsup_gray(S, p) : 0.f;
    tw[hy][hx] = in ? warped[base + p] : 0.f;
    if (kk) kk[hy][hx] = in ? coef[base + p] : 0.f;
  }
}
// (2) census + smoothness.  Block x of direction n walks tiles x, x + 64, ...; each thread owns two pixels of a tile.  Partials:
// part[(n * 64 + x) * 2 + {0, 1}] = {sum M psi, sum w s} of the block's pixels (warp butterfly, then the 8 warps in index order).
__global__ void __launch_bounds__(256) unsup_census_kernel(UnsupArgs a, const float* __restrict__ warped, const float* __restrict__ mask,
                                                           float* __restrict__ coef, double* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float gs[kUnsupHY][kUnsupHX], tw[kUnsupHY][kUnsupHX];
  __shared__ double red[8][2];
  const int n = blockIdx.x / kUnsupBlocks, blk = blockIdx.x % kUnsupBlocks;
  const int tiles_x = (a.W + kUnsupTX - 1) / kUnsupTX, tiles = tiles_x * ((a.H + kUnsupTY - 1) / kUnsupTY);
  const size_t base = (size_t)n * a.H * a.W;
  double photo = 0, smooth = 0;
  for (int t = blk; t < tiles; t += kUnsupBlocks) {
    const int ty0 = (t / tiles_x) * kUnsupTY, tx0 = (t % tiles_x) * kUnsupTX;
    __syncthreads();                                  // the previous tile's reads are done
    unsup_load_halo(a, n, ty0, tx0, warped, nullptr, gs, tw, nullptr);
    __syncthreads();
    for (int e = threadIdx.x; e < kUnsupTY * kUnsupTX; e += blockDim.x) {
      const int ly = e / kUnsupTX, lx = e % kUnsupTX, y = ty0 + ly, x = tx0 + lx;
      if (y >= a.H || x >= a.W) continue;
      const int cy = ly + kUnsupR, cx = lx + kUnsupR;
      const float s0 = gs[cy][cx], w0 = tw[cy][cx];
      float c = 0.f;
      for (int dy = -kUnsupR; dy <= kUnsupR; ++dy) {
        if (y + dy < 0 || y + dy >= a.H) continue;
#pragma unroll
        for (int dx = -kUnsupR; dx <= kUnsupR; ++dx) {
          if ((dy == 0 && dx == 0) || x + dx < 0 || x + dx >= a.W) continue;
          const float d = unsup_t(gs[cy + dy][cx + dx] - s0) - unsup_t(tw[cy + dy][cx + dx] - w0);
          c += d * d / (0.1f + d * d);
        }
      }
      const size_t p = base + (size_t)y * a.W + x;
      const float m = mask[p];
      photo += (double)(m * powf(c + 0.01f, 0.4f));
      coef[p] = m * 0.4f * powf(c + 0.01f, -0.6f);
      for (int ax = 0; ax < 2; ++ax) {
        const int dy = ax == 0, dx = ax == 1;
        if ((ax == 0 && (y < 1 || y > a.H - 2)) || (ax == 1 && (x < 1 || x > a.W - 2))) continue;
        float w;
        double l[2];
        unsup_smooth_terms(a, n, y, x, dy, dx, w, l);
        smooth += (double)w * (fabs(l[0]) + fabs(l[1]));
      }
    }
  }
  photo = warp_sum_d(photo);
  smooth = warp_sum_d(smooth);
  if ((threadIdx.x & 31) == 0) {
    red[threadIdx.x >> 5][0] = photo;
    red[threadIdx.x >> 5][1] = smooth;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    double s = 0;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += red[k][threadIdx.x];
    part[((size_t)n * kUnsupBlocks + blk) * 2 + threadIdx.x] = s;
  }
}
// (3) one block per direction, thread i adds component i of the 64 partials in block order
__global__ void unsup_reduce_kernel(const double* __restrict__ part, double* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.x, i = threadIdx.x;
  double s = 0;
  for (int k = 0; k < kUnsupBlocks; ++k) s += part[((size_t)n * kUnsupBlocks + k) * 2 + i];
  out[n * 2 + i] = s;
}
// backward, one thread per pixel r of a 16x32 tile (grid: tiles x 2B).  Census: dT~(r) = -sum_delta (k(r+delta) + k(r)) h(r, r+delta),
// h = d/du of (dt^2 / (0.1 + dt^2)), dt = t_S - t(u), u = T~(r+delta) - T~(r) (each window's term is odd in the pair's order, so the
// gather over the windows holding r folds into one sweep of r's own window), chained through dense_image_warp's dflow rule.
// Smoothness: the 5-point gather of w_a sign(second difference) from the centres r - e_a, r, r + e_a.
__global__ void __launch_bounds__(256) unsup_bwd_kernel(UnsupArgs a, const float* __restrict__ warped, const float* __restrict__ coef,
                                                        float w_photo, float w_smooth, float* __restrict__ dflow) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float gs[kUnsupHY][kUnsupHX], tw[kUnsupHY][kUnsupHX], kk[kUnsupHY][kUnsupHX];
  const int tiles_x = (a.W + kUnsupTX - 1) / kUnsupTX, tiles = tiles_x * ((a.H + kUnsupTY - 1) / kUnsupTY);
  const int n = blockIdx.x / tiles, t = blockIdx.x % tiles;
  const int ty0 = (t / tiles_x) * kUnsupTY, tx0 = (t % tiles_x) * kUnsupTX;
  unsup_load_halo(a, n, ty0, tx0, warped, coef, gs, tw, kk);
  __syncthreads();
  const size_t base = (size_t)n * a.H * a.W;
  for (int e = threadIdx.x; e < kUnsupTY * kUnsupTX; e += blockDim.x) {
    const int ly = e / kUnsupTX, lx = e % kUnsupTX, y = ty0 + ly, x = tx0 + lx;
    if (y >= a.H || x >= a.W) continue;
    const int cy = ly + kUnsupR, cx = lx + kUnsupR;
    const float s0 = gs[cy][cx], w0 = tw[cy][cx], k0 = kk[cy][cx];
    float g = 0.f;
    for (int dy = -kUnsupR; dy <= kUnsupR; ++dy) {
      if (y + dy < 0 || y + dy >= a.H) continue;
#pragma unroll
      for (int dx = -kUnsupR; dx <= kUnsupR; ++dx) {
        if ((dy == 0 && dx == 0) || x + dx < 0 || x + dx >= a.W) continue;
        const float u = tw[cy + dy][cx + dx] - w0, iu = rsqrtf(0.81f + u * u);
        const float d = unsup_t(gs[cy + dy][cx + dx] - s0) - u * iu, den = 0.1f + d * d;
        g += (kk[cy + dy][cx + dx] + k0) * (-0.2f * d / (den * den)) * (0.81f * iu * iu * iu);
      }
    }
    const float dtw = -g * w_photo;
    const size_t pix = base + (size_t)y * a.W + x;
    const float2 f = reinterpret_cast<const float2*>(a.flow)[pix];
    const UnsupSample s = unsup_sample(unsup_frame(a, n, true), a.H, a.W, (double)y - f.x, (double)x - f.y);
    const float top = s.ax * (s.tr - s.tl) + s.tl, bot = s.ax * (s.br - s.bl) + s.bl;
    float d0 = s.pass_y ? -dtw * (bot - top) : 0.f;
    float d1 = s.pass_x ? -dtw * (s.ay * (s.br - s.bl) + (1.f - s.ay) * (s.tr - s.tl)) : 0.f;
    float sm0 = 0.f, sm1 = 0.f;
    for (int ax = 0; ax < 2; ++ax) {
      const int dy = ax == 0, dx = ax == 1, pos = ax == 0 ? y : x, size = ax == 0 ? a.H : a.W;
      for (int o = -1; o <= 1; ++o) {                // centre r + o e_a: coefficient -2 at o = 0, 1 at o = +-1
        const int c = pos + o;
        if (c < 1 || c > size - 2) continue;
        float w;
        double l[2];
        unsup_smooth_terms(a, n, y + o * dy, x + o * dx, dy, dx, w, l);
        const float cw = (o == 0 ? -2.f : 1.f) * w;
        sm0 += cw * (float)((l[0] > 0) - (l[0] < 0));
        sm1 += cw * (float)((l[1] > 0) - (l[1] < 0));
      }
    }
    d0 += w_smooth * sm0;
    d1 += w_smooth * sm1;
    reinterpret_cast<float2*>(dflow)[pix] = make_float2(d0, d1);
  }
}
static int unsup_args(const char* what, const float* flow, const float* img1, const float* img2, int32_t B, int32_t H, int32_t W,
                      UnsupArgs& a) {
  // the flow is read as float2: 8-byte aligned pairs
  if (!flow || !img1 || !img2 || B < 1 || B > 65535 || H < 3 || W < 3 || ((uintptr_t)flow & 7)) return cis_set_error(CIS_ERR_BAD_ARG, what);
  a = UnsupArgs{flow, img1, img2, B, H, W};
  return CIS_OK;
}

extern "C" {

int cis_pack_weights(const float* w, const int32_t* kmap, int32_t K_pad, int32_t rows, int32_t cout, int32_t sn, const int32_t* nmap, void* wp,
                     cis_stream_t stream) {
  CIS_LAUNCH(pack_weights_kernel, nblk((size_t)rows * K_pad), 256, 0, ST, w, kmap, K_pad, rows, cout, sn, nmap, (mbf)wp);
  return cis_check_launch("pack_weights");
}
int cis_pack_weights_tiled(const float* w, const int32_t* kmap, int32_t cin8, int32_t ntaps, int32_t n_tiles, int32_t BN, int32_t cout, int32_t sn,
                           const int32_t* nmap, void* out, int32_t thin, cis_stream_t stream) {
  const size_t total = thin ? (size_t)n_tiles * (thin == 8 ? (ntaps + 1) / 2 : ntaps) * BN * 16
                            : (size_t)n_tiles * ((cin8 + 63) / 64) * ntaps * BN * 64;
  const unsigned blocks = (sn == 1 && !thin) ? (unsigned)(n_tiles * ((cin8 + 63) / 64) * ntaps) : nblk(total);
  if (BN > 128) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_pack_weights_tiled: BN > 128");
  if (thin && (cin8 != thin || (thin != 8 && thin != 16))) return cis_set_error(CIS_ERR_BAD_ARG, "cis_pack_weights_tiled: thin must be 8 or 16 = cin8");
  CIS_LAUNCH(pack_weights_tiled_kernel, blocks, 256, 0, ST, w, kmap, cin8, ntaps, n_tiles, BN, cout, sn, nmap, (mbf)out, thin);
  return cis_check_launch("pack_weights_tiled");
}
int cis_unpack_wgrad(const float* dwp, const int32_t* kmap, int32_t K_pad, int32_t cout, int32_t nsplit, float* dw, const float* colpart,
                     int32_t nblocks, int32_t nch, float* db, int32_t layout, cis_stream_t stream) {
  if (nsplit < 1 || (colpart && (nblocks < 1 || !db)) || ((layout & 0xff) != 0 && (layout & 0xff) != 1) || layout < 0 || K_pad % 4)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_unpack_wgrad: bad split / column-sum / layout arguments");
  CIS_LAUNCH(unpack_wgrad_kernel, nblk((size_t)cout * K_pad + (colpart ? nch : 0)), 256, 0, ST, dwp, kmap, K_pad, cout, nsplit, dw, colpart, nblocks,
             nch, db, layout);
  return cis_check_launch("unpack_wgrad");
}
int cis_param_multi(const CisParamJob* jobs_dev, int32_t njobs, int32_t total_blocks, cis_stream_t stream) {
  if (!jobs_dev || njobs < 1 || total_blocks < 1) return cis_set_error(CIS_ERR_BAD_ARG, "cis_param_multi: bad job table");
  CIS_LAUNCH(param_multi_kernel, (unsigned)total_blocks, 256, 0, ST, jobs_dev, njobs);
  return cis_check_launch("param_multi");
}
int cis_bn_fold(const float* w, const float* bias, const float* gamma, const float* beta, int64_t nw, int32_t cout, float* w_eff, float* b_eff,
                cis_stream_t stream) {
  CIS_LAUNCH(bn_fold_kernel, nblk((size_t)nw), 256, 0, ST, w, bias, gamma, beta, (size_t)nw, cout, w_eff, b_eff);
  return cis_check_launch("bn_fold");
}
int cis_bn_chain(const float* w, const float* bias, const float* gamma, float* dwe, const float* dbe, int64_t nw, int32_t cout, float* dbias,
                 float* dgamma, float* dbeta, cis_stream_t stream) {
  CIS_LAUNCH(bn_chain_kernel, (unsigned)((cout + kBnChainCo - 1) / kBnChainCo), 256, 0, ST, w, bias, gamma, dwe, dbe, (size_t)nw, cout, dbias, dgamma, dbeta);
  return cis_check_launch("bn_chain");
}
int cis_dact_mul(void* g, int32_t gp, int32_t gc, const void* y, int32_t yp, int32_t yc, const void* res, int32_t rp, int32_t rc, int64_t npix,
                 int32_t chunks, int32_t act, float alpha, cis_stream_t stream) {
  if (act == CIS_ACT_NONE) return CIS_OK;
  CIS_LAUNCH(dact_mul_kernel, nblk((size_t)npix * chunks), 256, 0, ST, (mbf)g, gp, gc, (cbf)y, yp, yc, (cbf)res, rp, rc, (size_t)npix, chunks, act, alpha);
  return cis_check_launch("dact_mul");
}
int cis_add_slice(void* dst, int32_t dp, int32_t dc, const void* src, int32_t sp, int32_t sc, int64_t npix, int32_t chunks, int32_t reps,
                  int32_t accumulate, cis_stream_t stream) {
  CIS_LAUNCH(add_slice_kernel, nblk((size_t)npix * chunks), 256, 0, ST, (mbf)dst, dp, dc, (cbf)src, sp, sc, (size_t)npix, chunks, reps, accumulate);
  return cis_check_launch("add_slice");
}
int cis_colsum(const void* g, int32_t gp, int32_t gc, int64_t npix, int32_t nch, float* part, int32_t nblocks, cis_stream_t stream) {
  const int chunks = (nch + 7) / 8;
  if (chunks > 32) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_colsum: more than 256 channels");
  if (nblocks < 1 || nblocks > 592) return cis_set_error(CIS_ERR_BAD_ARG, "cis_colsum: nblocks must be in [1, 592]");
  const int P = 256 / chunks;
  CIS_LAUNCH(colsum_kernel, (unsigned)nblocks, 256, P * chunks * 8 * sizeof(float), ST, (cbf)g, gp, gc, (size_t)npix, nch, chunks, part);
  return cis_check_launch("colsum");
}
int cis_zero(void* ptr, int64_t nbytes, cis_stream_t stream) {
  if (!ptr || nbytes < 0) return cis_set_error(CIS_ERR_BAD_ARG, "cis_zero: bad buffer");
  cudaError_t e = cudaMemsetAsync(ptr, 0, (size_t)nbytes, ST);     // a memset node under graph capture: no kernel, no library launch
  if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaMemsetAsync");
  return CIS_OK;
}
int cis_dact_colsum(void* g, int32_t gp, int32_t gc, const void* y, int32_t yp, int32_t yc, const void* res, int32_t rp, int32_t rc, int64_t npix,
                    int32_t nch, int32_t act, float alpha, float* part, int32_t nblocks, cis_stream_t stream) {
  const int chunks = (nch + 7) / 8;
  if (act == CIS_ACT_NONE) return cis_colsum(g, gp, gc, npix, nch, part, nblocks, stream);
  if (chunks > 32) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_dact_colsum: more than 256 channels");
  if (nblocks < 1 || nblocks > 592) return cis_set_error(CIS_ERR_BAD_ARG, "cis_dact_colsum: nblocks must be in [1, 592]");
  const int P = 256 / chunks;
  CIS_LAUNCH(dact_colsum_kernel, (unsigned)nblocks, 256, P * chunks * 8 * sizeof(float), ST, (mbf)g, gp, gc, (cbf)y, yp, yc, (cbf)res, rp, rc,
             (size_t)npix, nch, chunks, act, alpha, part);
  return cis_check_launch("dact_colsum");
}
int cis_resize_bilinear_bf16(const void* src, int32_t sp, int32_t sc, int32_t N, int32_t H, int32_t W, void* dst, int32_t dp, int32_t dc, int32_t OH,
                             int32_t OW, int32_t chunks, cis_stream_t stream) {
  CIS_LAUNCH(resize_bilinear_bf16_kernel, nblk((size_t)N * OH * OW * chunks), 256, 0, ST, (cbf)src, sp, sc, N, H, W, (mbf)dst, dp, dc, OH, OW, chunks);
  return cis_check_launch("resize_bilinear_bf16");
}
int cis_resize_bilinear_bf16_bwd(const void* dd, int32_t dp, int32_t dc, int32_t N, int32_t OH, int32_t OW, void* ds, int32_t sp, int32_t sc, int32_t H,
                                 int32_t W, int32_t chunks, int32_t accumulate, cis_stream_t stream) {
  CIS_LAUNCH(resize_bilinear_bf16_bwd_kernel, nblk((size_t)N * H * W * chunks), 256, 0, ST, (cbf)dd, dp, dc, N, OH, OW, (mbf)ds, sp, sc, H, W, chunks,
                                                                                     accumulate);
  return cis_check_launch("resize_bilinear_bf16_bwd");
}
int cis_resize_concat_bf16(const CisSrc* srcs, int32_t nsrc, int32_t N, int32_t H, int32_t W, void* dst, int32_t dp, int32_t dc, int32_t OH, int32_t OW,
                           cis_stream_t stream) {
  if (!srcs || nsrc < 1 || nsrc > CIS_MAX_SRC) return cis_set_error(CIS_ERR_BAD_ARG, "cis_resize_concat_bf16: 1..4 sources");
  RcArgs a;
  a.nsrc = nsrc;
  int total = 0;
  for (int i = 0; i < nsrc; ++i) {
    a.s[i] = srcs[i];
    if ((srcs[i].pitch | srcs[i].c_off) & 7) return cis_set_error(CIS_ERR_BAD_ARG, "cis_resize_concat_bf16: slices must be 8-channel aligned");
    total += srcs[i].chunks;
  }
  if ((dp | dc) & 7) return cis_set_error(CIS_ERR_BAD_ARG, "cis_resize_concat_bf16: destination must be 8-channel aligned");
  if ((size_t)N * OH > 65535 || (size_t)OW * total > 0x7fffffff) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_resize_concat_bf16: too many rows");
  if (OH == 2 * H && OW == 2 * W) {
    CIS_LAUNCH(resize_concat_x2_bf16_kernel, dim3((unsigned)((W * total + 255) / 256), (unsigned)(N * H)), 256, 0, ST, a, N, H, W, (mbf)dst, dp, dc, total);
    return cis_check_launch("resize_concat_x2_bf16");
  }
  CIS_LAUNCH(resize_concat_bf16_kernel, dim3((unsigned)((OW * total + 255) / 256), (unsigned)(N * OH)), 256, 0, ST, a, N, H, W, (mbf)dst, dp, dc, OH, OW,
             total);
  return cis_check_launch("resize_concat_bf16");
}
int cis_resize_concat_bf16_bwd(const void* ddst, int32_t dp, int32_t dc, int32_t N, int32_t OH, int32_t OW, const CisSrc* grads, const int32_t* want,
                               const int32_t* accumulate, int32_t nsrc, int32_t H, int32_t W, cis_stream_t stream) {
  if (!grads || nsrc < 1 || nsrc > CIS_MAX_SRC) return cis_set_error(CIS_ERR_BAD_ARG, "cis_resize_concat_bf16_bwd: 1..4 sources");
  RcGradArgs a;
  a.nsrc = nsrc;
  int total = 0;
  for (int i = 0; i < nsrc; ++i) {
    a.s[i].ptr = const_cast<void*>(grads[i].ptr);
    a.s[i].pitch = grads[i].pitch;
    a.s[i].c_off = grads[i].c_off;
    a.s[i].chunks = grads[i].chunks;
    a.s[i].n_mod = grads[i].n_mod;
    a.s[i].want = want[i];
    a.s[i].accumulate = accumulate[i];
    if (want[i] && (!grads[i].ptr || ((grads[i].pitch | grads[i].c_off) & 7))) return cis_set_error(CIS_ERR_BAD_ARG, "cis_resize_concat_bf16_bwd: bad gradient slice");
    if (grads[i].n_mod && N % grads[i].n_mod) return cis_set_error(CIS_ERR_BAD_ARG, "cis_resize_concat_bf16_bwd: N must be a multiple of n_mod");
    total += grads[i].chunks;
  }
  if ((size_t)N * H > 65535 || (size_t)W * total > 0x7fffffff) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_resize_concat_bf16_bwd: too many rows");
  CIS_LAUNCH(resize_concat_bf16_bwd_kernel, dim3((unsigned)((W * total + 255) / 256), (unsigned)(N * H)), 256, 0, ST, (cbf)ddst, dp, dc, N, OH, OW, a, H,
             W, total);
  return cis_check_launch("resize_concat_bf16_bwd");
}
int cis_resize_bilinear_f32(const float* src, int32_t N, int32_t H, int32_t W, int32_t C, float* dst, int32_t OH, int32_t OW, float scale,
                            cis_stream_t stream) {
  CIS_LAUNCH(resize_bilinear_f32_kernel<false>, nblk((size_t)N * OH * OW), 256, 0, ST, src, N, H, W, C, dst, OH, OW, scale);
  return cis_check_launch("resize_bilinear_f32");
}
int cis_crop_resize_bilinear_f32(const float* src, int32_t Hs, int32_t Ws, int32_t C, int32_t y0, int32_t x0, int32_t ch, int32_t cw, float* dst,
                                 int32_t OH, int32_t OW, cis_stream_t stream) {
  if (!src || !dst || y0 < 0 || x0 < 0 || ch < 1 || cw < 1 || y0 + ch > Hs || x0 + cw > Ws || OH < 1 || OW < 1)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_crop_resize_bilinear_f32: crop box outside the image");
  CIS_LAUNCH(crop_resize_f32_kernel<false>, nblk((size_t)OH * OW), 256, 0, ST, src, Ws, C, y0, x0, ch, cw, dst, OH, OW, 1.f, 1.f);
  return cis_check_launch("crop_resize_f32");
}
int cis_crop_resize_flow_f32(const float* src, int32_t Hs, int32_t Ws, int32_t y0, int32_t x0, int32_t ch, int32_t cw, float* dst, int32_t OH,
                             int32_t OW, float s0, float s1, cis_stream_t stream) {
  if (!src || !dst || y0 < 0 || x0 < 0 || ch < 1 || cw < 1 || y0 + ch > Hs || x0 + cw > Ws || OH < 1 || OW < 1)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_crop_resize_flow_f32: crop box outside the image");
  CIS_LAUNCH(crop_resize_f32_kernel<true>, nblk((size_t)OH * OW), 256, 0, ST, src, Ws, 2, y0, x0, ch, cw, dst, OH, OW, s0, s1);
  return cis_check_launch("crop_resize_flow_f32");
}
int cis_upsample_nn2x(const void* src, int32_t N, int32_t H, int32_t W, int32_t pitch, void* dst, cis_stream_t stream) {
  if ((size_t)N * 2 * H > 65535) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_upsample_nn2x: too many rows");
  CIS_LAUNCH(upsample_nn2x_kernel, dim3((unsigned)((2 * W * (pitch / 8) + 255) / 256), (unsigned)(N * 2 * H)), 256, 0, ST, (cbf)src, N, H, W, pitch,
             (mbf)dst);
  return cis_check_launch("upsample_nn2x");
}
int cis_upsample_nn2x_bwd(const void* dd, int32_t N, int32_t H, int32_t W, int32_t pitch, void* ds, int32_t accumulate, cis_stream_t stream) {
  if ((size_t)N * H > 65535) return cis_set_error(CIS_ERR_UNSUPPORTED, "cis_upsample_nn2x_bwd: too many rows");
  CIS_LAUNCH(upsample_nn2x_bwd_kernel, dim3((unsigned)((W * (pitch / 8) + 255) / 256), (unsigned)(N * H)), 256, 0, ST, (cbf)dd, N, H, W, pitch, (mbf)ds,
             accumulate);
  return cis_check_launch("upsample_nn2x_bwd");
}
int cis_resize_nn_f32(const float* src, int32_t N, int32_t H, int32_t W, int32_t C, float* dst, int32_t OH, int32_t OW, cis_stream_t stream) {
  CIS_LAUNCH(resize_nn_f32_kernel<false>, nblk((size_t)N * OH * OW), 256, 0, ST, src, N, H, W, C, dst, OH, OW);
  return cis_check_launch("resize_nn_f32");
}
static int resize_f32_args(const char* what, const void* src, const void* dst, int32_t N, int32_t H, int32_t W, int32_t C, int32_t OH,
                           int32_t OW, int32_t method, int32_t align_corners) {
  if (method != CIS_RESIZE_BILINEAR && method != CIS_RESIZE_NEAREST) return cis_set_error(CIS_ERR_BAD_ARG, what);
  if (align_corners != 0 && align_corners != 1) return cis_set_error(CIS_ERR_BAD_ARG, what);
  if (!src || !dst || N < 1 || H < 1 || W < 1 || C < 1 || OH < 1 || OW < 1) return cis_set_error(CIS_ERR_BAD_ARG, what);
  return CIS_OK;
}
int cis_resize_f32(const float* src, int32_t N, int32_t H, int32_t W, int32_t C, float* dst, int32_t OH, int32_t OW, int32_t method,
                   int32_t align_corners, cis_stream_t stream) {
  const int rc = resize_f32_args("cis_resize_f32: bad method, align_corners, pointer or size", src, dst, N, H, W, C, OH, OW, method,
                                 align_corners);
  if (rc) return rc;
  const unsigned g = nblk((size_t)N * OH * OW);
  if (method == CIS_RESIZE_BILINEAR) {
    if (align_corners) CIS_LAUNCH(resize_bilinear_f32_kernel<true>, g, 256, 0, ST, src, N, H, W, C, dst, OH, OW, 1.f);
    else CIS_LAUNCH(resize_bilinear_f32_kernel<false>, g, 256, 0, ST, src, N, H, W, C, dst, OH, OW, 1.f);
  } else {
    if (align_corners) CIS_LAUNCH(resize_nn_f32_kernel<true>, g, 256, 0, ST, src, N, H, W, C, dst, OH, OW);
    else CIS_LAUNCH(resize_nn_f32_kernel<false>, g, 256, 0, ST, src, N, H, W, C, dst, OH, OW);
  }
  return cis_check_launch("resize_f32");
}
int cis_resize_f32_bwd(const float* ddst, int32_t N, int32_t OH, int32_t OW, int32_t C, int32_t H, int32_t W, float* dsrc, int32_t method,
                       int32_t align_corners, cis_stream_t stream) {
  const int rc = resize_f32_args("cis_resize_f32_bwd: bad method, align_corners, pointer or size", ddst, dsrc, N, H, W, C, OH, OW, method,
                                 align_corners);
  if (rc) return rc;
  const unsigned g = nblk((size_t)N * H * W * C);
  if (method == CIS_RESIZE_BILINEAR) {
    if (align_corners) CIS_LAUNCH((resize_f32_bwd_kernel<false, true>), g, 256, 0, ST, ddst, N, OH, OW, C, H, W, dsrc);
    else CIS_LAUNCH((resize_f32_bwd_kernel<false, false>), g, 256, 0, ST, ddst, N, OH, OW, C, H, W, dsrc);
  } else {
    if (align_corners) CIS_LAUNCH((resize_f32_bwd_kernel<true, true>), g, 256, 0, ST, ddst, N, OH, OW, C, H, W, dsrc);
    else CIS_LAUNCH((resize_f32_bwd_kernel<true, false>), g, 256, 0, ST, ddst, N, OH, OW, C, H, W, dsrc);
  }
  return cis_check_launch("resize_f32_bwd");
}
int cis_warp_costvol(const void* c1, int32_t c1p, int32_t c1o, const void* c2, int32_t c2p, int32_t c2o, const float* flow, float fs, int32_t B,
                     int32_t h, int32_t w, int32_t C, void* out, int32_t op, int32_t oo, cis_stream_t stream) {
  return warp_costvol_fwd<4>(c1, c1p, c1o, c2, c2p, c2o, flow, fs, B, h, w, C, out, op, oo, stream);
}
int cis_warp_costvol_r(const void* c1, int32_t c1p, int32_t c1o, const void* c2, int32_t c2p, int32_t c2o, const float* flow, float fs, int32_t B,
                       int32_t h, int32_t w, int32_t C, void* out, int32_t op, int32_t oo, int32_t search_range, cis_stream_t stream) {
  CIS_CV_DISPATCH(warp_costvol_fwd, "cis_warp_costvol_r", c1, c1p, c1o, c2, c2p, c2o, flow, fs, B, h, w, C, out, op, oo, stream)
}
int cis_dense_image_warp(const void* img, int32_t pitch, int32_t coff, const float* flow, float fs, int32_t B, int32_t h, int32_t w, int32_t C,
                         void* out, int32_t op, cis_stream_t stream) {
  const int chunks = (C + 7) / 8;
  CIS_LAUNCH(dense_image_warp_kernel, nblk((size_t)B * h * w * chunks), 256, 0, ST, (cbf)img, pitch, coff, flow, fs, B, h, w, chunks, (mbf)out, op);
  return cis_check_launch("dense_image_warp");
}
int cis_pack_f32_to_bf16(const float* src, int64_t npix, int32_t C, float offset, void* dst, int32_t dp, int32_t dc, cis_stream_t stream) {
  if (C > 8) return cis_set_error(CIS_ERR_BAD_ARG, "cis_pack_f32_to_bf16: C > 8");
  CIS_LAUNCH(pack_f32_to_bf16_kernel, nblk((size_t)npix), 256, 0, ST, src, (size_t)npix, C, offset, (mbf)dst, dp, dc);
  return cis_check_launch("pack_f32_to_bf16");
}
int cis_flow_stats(const float* flow, int32_t B, int64_t hw, double* stats, cis_stream_t stream) {
  dim3 grid(64, B);
  CIS_LAUNCH(flow_stats_kernel, grid, 256, 0, ST, flow, (size_t)hw, stats);
  return cis_check_launch("flow_stats");
}
int cis_pack_generator_input(const float* image, const float* flow, const double* stats, int32_t B, int64_t hw, void* dst, cis_stream_t stream) {
  dim3 grid(nblk((size_t)hw), B);
  CIS_LAUNCH(pack_generator_input_kernel, grid, 256, 0, ST, image, flow, stats, (size_t)hw, (mbf)dst);
  return cis_check_launch("pack_generator_input");
}
int cis_flow_standardize(const float* flow, const double* stats, int32_t B, int64_t hw, float* out, cis_stream_t stream) {
  if (!flow || !stats || !out || B < 1 || hw < 1) return cis_set_error(CIS_ERR_BAD_ARG, "cis_flow_standardize: bad pointer or size");
  CIS_LAUNCH(flow_standardize_kernel, dim3(nblk((size_t)hw), B), 256, 0, ST, flow, stats, (size_t)hw, out);
  return cis_check_launch("flow_standardize");
}
int cis_flow_standardize_bwd(const float* y, const float* dy, const double* stats, int32_t B, int64_t hw, double* scratch, float* dx,
                             cis_stream_t stream) {
  if (!y || !dy || !stats || !scratch || !dx || B < 1 || hw < 1)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_flow_standardize_bwd: bad pointer or size");
  CIS_LAUNCH(flow_standardize_bwd_sums_kernel, dim3(kFlowStdBlocks, B), 256, 0, ST, y, dy, (size_t)hw, scratch);
  CIS_LAUNCH(flow_standardize_bwd_kernel, dim3(nblk((size_t)hw), B), 256, 0, ST, y, dy, stats, (const double*)scratch, (size_t)hw, dx);
  return cis_check_launch("flow_standardize_bwd");
}
int cis_masked_epe(const float* pred, const float* gt, const float* mask, int32_t B, int64_t hw, double* scratch, double* out,
                   cis_stream_t stream) {
  if (!pred || !gt || !mask || !scratch || !out || B < 1 || B > 65535 || hw < 1)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_masked_epe: bad pointer or size");
  CIS_LAUNCH(masked_epe_sums_kernel, dim3(kFlowStdBlocks, B), 256, 0, ST, pred, gt, mask, (size_t)hw, scratch);
  CIS_LAUNCH(masked_epe_reduce_kernel, B, 4, 0, ST, (const double*)scratch, out);
  return cis_check_launch("masked_epe");
}
int cis_mask_apply(const float* flow, const float* mask, int32_t B, int64_t hw, void* dst, cis_stream_t stream) {
  CIS_LAUNCH(mask_apply_kernel, nblk((size_t)B * hw), 256, 0, ST, flow, mask, (size_t)B * hw, (mbf)dst);
  return cis_check_launch("mask_apply");
}
int cis_box_masks(float* mask, int32_t B, int32_t H, int32_t W, int32_t lo_h, int32_t hi_h, int32_t lo_w, int32_t hi_w, int64_t sample_offset,
                  const long long* step, uint64_t seed, cis_stream_t stream) {
  if (!mask || !step || B < 1 || B > 65535 || sample_offset < 0) return cis_set_error(CIS_ERR_BAD_ARG, "cis_box_masks: bad buffer, batch or sample offset");
  if (lo_h < 1 || lo_w < 1 || hi_h < lo_h || hi_w < lo_w || hi_h > H || hi_w > W)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_box_masks: box sides need 1 <= lo <= hi <= image side");
  CIS_LAUNCH(box_masks_kernel, dim3(nblk((size_t)H * W), B), 256, 0, ST, mask, H, W, lo_h, hi_h, lo_w, hi_w, (long long)sample_offset, step,
             (unsigned long long)seed);
  return cis_check_launch("box_masks");
}
int cis_charbonnier_sum(const float* gt, const float* pred, const float* mask, int32_t B, int64_t hw, int32_t C, int32_t mask_c, float cbn,
                        double* sums, cis_stream_t stream) {
  if (C < 1 || (mask_c != 1 && mask_c != C)) return cis_set_error(CIS_ERR_BAD_ARG, "cis_charbonnier_sum: mask must have 1 or C channels");
  dim3 grid(64, B);
  CIS_LAUNCH(charbonnier_sum_kernel, grid, 256, 0, ST, gt, pred, mask, (size_t)hw, C, mask_c, cbn, sums);
  return cis_check_launch("charbonnier_sum");
}
int cis_cis_loss_fwd(const float* flow, const float* mask, const float* flow1, int32_t B, int32_t H, int32_t W, int32_t h1, int32_t w1, float cbn,
                     double* sums, float* pred_out, cis_stream_t stream) {
  dim3 grid(cis_num_sms(), B);
  CIS_LAUNCH(cis_loss_fwd_kernel, grid, 256, 0, ST, flow, mask, flow1, B, H, W, h1, w1, cbn, sums, pred_out);
  return cis_check_launch("cis_loss_fwd");
}
int cis_cis_loss_reduce(const double* sums, int32_t B, int32_t global_batch, int64_t hw, float epsilon, float* scalars, float* coef,
                        cis_stream_t stream) {
  CIS_LAUNCH(cis_loss_reduce_kernel, 1, 32, 0, ST, sums, B, global_batch, (double)hw, epsilon, scalars, coef);
  return cis_check_launch("cis_loss_reduce");
}
int cis_cis_loss_bwd(const float* flow, const float* mask, const float* flow1, const float* coef, const float* scalars, int32_t B, int32_t H,
                     int32_t W, int32_t h1, int32_t w1, float cbn, int32_t which, float* dpred, float* dmask, cis_stream_t stream) {
  dim3 grid(nblk((size_t)H * W), B);
  CIS_LAUNCH(cis_loss_bwd_kernel, grid, 256, 0, ST, flow, mask, flow1, coef, scalars, B, H, W, h1, w1, cbn, which, dpred, dmask);
  return cis_check_launch("cis_loss_bwd");
}
int cis_resize_f32_bwd_to_bf16(const float* dd, int32_t N, int32_t OH, int32_t OW, int32_t C, int32_t H, int32_t W, void* ds, int32_t sp,
                               cis_stream_t stream) {
  if (C > 8) return cis_set_error(CIS_ERR_BAD_ARG, "cis_resize_f32_bwd_to_bf16: C > 8");
  CIS_LAUNCH(resize_f32_bwd_to_bf16_kernel, nblk((size_t)N * H * W), 256, 0, ST, dd, N, OH, OW, C, H, W, (mbf)ds, sp, 1.f);
  return cis_check_launch("resize_f32_bwd_to_bf16");
}
int cis_resize_f32_bwd_to_bf16_scaled(const float* dd, int32_t N, int32_t OH, int32_t OW, int32_t C, int32_t H, int32_t W, void* ds, int32_t sp,
                                      float scale, cis_stream_t stream) {
  if (C > 8) return cis_set_error(CIS_ERR_BAD_ARG, "cis_resize_f32_bwd_to_bf16_scaled: C > 8");
  CIS_LAUNCH(resize_f32_bwd_to_bf16_kernel, nblk((size_t)N * H * W), 256, 0, ST, dd, N, OH, OW, C, H, W, (mbf)ds, sp, scale);
  return cis_check_launch("resize_f32_bwd_to_bf16_scaled");
}
int cis_mask_bwd(const float* flow, const float* mask, const float* dmd, const void* din, int32_t B, int64_t hw, void* dlogits, cis_stream_t stream) {
  if (din && !flow) return cis_set_error(CIS_ERR_BAD_ARG, "cis_mask_bwd: the recover-input chain (d_in) needs the flow");
  CIS_LAUNCH(mask_bwd_kernel, nblk((size_t)B * hw), 256, 0, ST, flow, mask, dmd, (cbf)din, (size_t)B * hw, (mbf)dlogits);
  return cis_check_launch("mask_bwd");
}
int cis_abs_sum(const float* g, int64_t n, float* stat, cis_stream_t stream) {
  CIS_LAUNCH(abs_sum_kernel, 296, 256, 0, ST, g, (size_t)n, stat);
  return cis_check_launch("abs_sum");
}
int cis_grad_avg_abs(const float* g, const int64_t* seg_off, int32_t nseg, float* out_avg, cis_stream_t stream) {
  CIS_LAUNCH(grad_avg_abs_kernel, dim3((unsigned)nseg, 16), 256, 0, ST, g, (const long long*)seg_off, nseg, out_avg);
  return cis_check_launch("grad_avg_abs");
}
int cis_clip_adam(float* param, float* m, float* v, const float* grad, int64_t n, float grad_scale, float clip, float lr, float beta1, float beta2,
                  float eps, int64_t* step_state, const float* avg_abs, int32_t can_change, uint64_t seed, cis_stream_t stream) {
  if (can_change && !avg_abs) return cis_set_error(CIS_ERR_BAD_ARG, "cis_clip_adam: can_change needs avg_abs");
  CIS_LAUNCH(clip_adam_kernel, nblk((size_t)n), 256, 0, ST, param, m, v, grad, (size_t)n, grad_scale, clip, lr, beta1, beta2, eps,
                                                    (const long long*)step_state, avg_abs, can_change, (unsigned long long)seed);
  CIS_LAUNCH(step_inc_kernel, 1, 1, 0, ST, (long long*)step_state);
  return cis_check_launch("clip_adam");
}
int cis_cast_f32_to_bf16(const float* src, int64_t n, void* dst, cis_stream_t stream) {
  CIS_LAUNCH(cast_f32_bf16_kernel, nblk((size_t)n), 256, 0, ST, src, (size_t)n, (mbf)dst);
  return cis_check_launch("cast_f32_to_bf16");
}
int cis_cast_bf16_to_f32(const void* src, int64_t npix, int32_t pitch, int32_t coff, int32_t C, float* dst, cis_stream_t stream) {
  CIS_LAUNCH(cast_bf16_f32_kernel, nblk((size_t)npix * C), 256, 0, ST, (cbf)src, (size_t)npix, pitch, coff, C, dst);
  return cis_check_launch("cast_bf16_to_f32");
}
int cis_cast_bf16_to_f32_scaled(const void* src, int64_t npix, int32_t pitch, int32_t coff, int32_t C, float scale, float* dst,
                                cis_stream_t stream) {
  CIS_LAUNCH(cast_bf16_f32_scaled_kernel, nblk((size_t)npix * C), 256, 0, ST, (cbf)src, (size_t)npix, pitch, coff, C, scale, dst);
  return cis_check_launch("cast_bf16_to_f32_scaled");
}
int cis_charbonnier_bwd(const float* gt, const float* pred, const float* mask, int32_t B, int64_t hw, int32_t C, int32_t mask_c, float cbn,
                        const float* dsum, float* dpred, float* dgt, float* dmask, cis_stream_t stream) {
  if (C < 1 || (mask_c != 1 && mask_c != C)) return cis_set_error(CIS_ERR_BAD_ARG, "cis_charbonnier_bwd: mask must have 1 or C channels");
  if (!dsum) return cis_set_error(CIS_ERR_BAD_ARG, "cis_charbonnier_bwd: no upstream gradient");
  CIS_LAUNCH(charbonnier_bwd_kernel, nblk((size_t)B * hw), 256, 0, ST, gt, pred, mask, (size_t)hw, (size_t)B * hw, C, mask_c, cbn, dsum, dpred, dgt,
             dmask);
  return cis_check_launch("charbonnier_bwd");
}
int cis_dense_image_warp_bwd(const void* img, int32_t pitch, int32_t coff, const float* flow, float fs, int32_t B, int32_t h, int32_t w,
                             int32_t C, const float* dout, float* dimage, double* scratch, float* dflow, cis_stream_t stream) {
  if (h < 2 || w < 2) return cis_set_error(CIS_ERR_BAD_ARG, "cis_dense_image_warp_bwd: needs h,w >= 2 (core_warp.py:188)");
  if ((pitch | coff) & 7 || coff + ((C + 7) & ~7) > pitch) return cis_set_error(CIS_ERR_BAD_ARG, "cis_dense_image_warp_bwd: bad image slice");
  if (dimage && !scratch) return cis_set_error(CIS_ERR_BAD_ARG, "cis_dense_image_warp_bwd: dimage needs the fp64 scratch");
  const size_t npix = (size_t)B * h * w;
  if (dimage) {
    cudaError_t e = cudaMemsetAsync(scratch, 0, npix * C * sizeof(double), ST);
    if (e != cudaSuccess) return cis_set_cuda_error(e, "cudaMemsetAsync");
  }
  CIS_LAUNCH(dense_image_warp_bwd_kernel<F32Out>, nblk(npix), 256, 0, ST, (cbf)img, pitch, coff, flow, fs, B, h, w, C, dout,
             dimage ? scratch : nullptr, F32Out{dflow, 2, 0});
  if (dimage) CIS_LAUNCH(round_f64_kernel<F32Out>, nblk(npix * C), 256, 0, ST, (const double*)scratch, npix, C, F32Out{dimage, C, 0});
  return cis_check_launch("dense_image_warp_bwd");
}
int cis_cost_volume_bwd(const void* c1, int32_t c1p, int32_t c1o, const void* warp, int32_t wp, int32_t wo, const float* dout, int32_t B, int32_t h,
                        int32_t w, int32_t C, float* gscratch, float* dc1, float* dwarp, cis_stream_t stream) {
  return cost_volume_bwd<4>(c1, c1p, c1o, warp, wp, wo, dout, B, h, w, C, gscratch, dc1, dwarp, stream);
}
int cis_cost_volume_bwd_r(const void* c1, int32_t c1p, int32_t c1o, const void* warp, int32_t wp, int32_t wo, const float* dout, int32_t B,
                          int32_t h, int32_t w, int32_t C, float* gscratch, float* dc1, float* dwarp, int32_t search_range, cis_stream_t stream) {
  CIS_CV_DISPATCH(cost_volume_bwd, "cis_cost_volume_bwd_r", c1, c1p, c1o, warp, wp, wo, dout, B, h, w, C, gscratch, dc1, dwarp, stream)
}
int cis_warp_costvol_bwd(const void* c1, int32_t c1p, int32_t c1o, const void* c2, int32_t c2p, int32_t c2o, const float* flow, float fs,
                         int32_t B, int32_t h, int32_t w, int32_t C, const void* dcorr, int32_t dcp, int32_t dco, void* dc1, int32_t dc1p,
                         int32_t dc1o, void* dc2, int32_t dc2p, int32_t dc2o, void* dflow, int32_t dfp, int32_t dfo, int32_t accumulate,
                         float* gscratch, float* wscratch, double* dscratch, cis_stream_t stream) {
  return warp_costvol_bwd<4>(c1, c1p, c1o, c2, c2p, c2o, flow, fs, B, h, w, C, dcorr, dcp, dco, dc1, dc1p, dc1o, dc2, dc2p, dc2o, dflow, dfp, dfo,
                             accumulate, gscratch, wscratch, dscratch, stream);
}
int cis_warp_costvol_bwd_r(const void* c1, int32_t c1p, int32_t c1o, const void* c2, int32_t c2p, int32_t c2o, const float* flow, float fs,
                           int32_t B, int32_t h, int32_t w, int32_t C, const void* dcorr, int32_t dcp, int32_t dco, void* dc1, int32_t dc1p,
                           int32_t dc1o, void* dc2, int32_t dc2p, int32_t dc2o, void* dflow, int32_t dfp, int32_t dfo, int32_t accumulate,
                           float* gscratch, float* wscratch, double* dscratch, int32_t search_range, cis_stream_t stream) {
  CIS_CV_DISPATCH(warp_costvol_bwd, "cis_warp_costvol_bwd_r", c1, c1p, c1o, c2, c2p, c2o, flow, fs, B, h, w, C, dcorr, dcp, dco, dc1, dc1p, dc1o,
                  dc2, dc2p, dc2o, dflow, dfp, dfo, accumulate, gscratch, wscratch, dscratch, stream)
}
int cis_parity_split_bf16(const void* src, int32_t sp, int32_t sc, int32_t N, int32_t H, int32_t W, int32_t C, void* dst, int32_t dp,
                          cis_stream_t stream) {
  if (C < 1 || C > 8 || dp < 8 || (dp & 7)) return cis_set_error(CIS_ERR_BAD_ARG, "cis_parity_split_bf16: 1..8 channels into 8-aligned planes");
  CIS_LAUNCH(parity_split_bf16_kernel, nblk((size_t)4 * N * H * W), 256, 0, ST, (cbf)src, sp, sc, N, H, W, C, (mbf)dst, dp);
  return cis_check_launch("parity_split_bf16");
}
int cis_flow_multiscale_loss(const CisFlowPyr* pyr, const float* gt, int32_t B, int32_t H, int32_t W, int32_t GH, int32_t GW, float s0,
                             float s1, int32_t robust, float eps, float q, double* scratch, double* out, cis_stream_t stream) {
  FlowLossArgs a;
  const int rc = flow_loss_args("cis_flow_multiscale_loss: bad pyramid, size, rho or alignment", pyr, gt, B, H, W, GH, GW, s0, s1, robust, eps, q, a);
  if (rc) return rc;
  if (!scratch || !out) return cis_set_error(CIS_ERR_BAD_ARG, "cis_flow_multiscale_loss: no scratch or output");
  CIS_LAUNCH(flow_loss_sums_kernel, dim3(kFlowStdBlocks, B, 5), 256, 0, ST, a, scratch);
  CIS_LAUNCH(flow_loss_reduce_kernel, B, 5, 0, ST, (const double*)scratch, B, out);
  return cis_check_launch("flow_multiscale_loss");
}
int cis_flow_multiscale_loss_bwd(const CisFlowPyr* pyr, const float* gt, int32_t B, int32_t H, int32_t W, int32_t GH, int32_t GW, float s0,
                                 float s1, int32_t robust, float eps, float q, cis_stream_t stream) {
  FlowLossArgs a;
  const int rc = flow_loss_args("cis_flow_multiscale_loss_bwd: bad pyramid, size, rho or alignment", pyr, gt, B, H, W, GH, GW, s0, s1, robust, eps, q, a);
  if (rc) return rc;
  size_t total = 0;
  for (int i = 0; i < 5; ++i) {
    if (!pyr->grad[i] || pyr->pitch[i] < 2 || pyr->c_off[i] < 0 || pyr->c_off[i] + 2 > pyr->pitch[i])
      return cis_set_error(CIS_ERR_BAD_ARG, "cis_flow_multiscale_loss_bwd: bad gradient slice");
    total += (size_t)B * (H >> (6 - i)) * (W >> (6 - i));
  }
  CIS_LAUNCH(flow_loss_bwd_kernel, nblk(total), 256, 0, ST, a, total);
  return cis_check_launch("flow_multiscale_loss_bwd");
}
int cis_adam_l2(float* param, float* m, float* v, const float* grad, int64_t n, const int64_t* seg, int32_t nseg, float decay, const float* lr,
                float beta1, float beta2, float eps, int64_t* step_state, cis_stream_t stream) {
  if (!param || !m || !v || !grad || n < 1 || nseg < 0 || (nseg > 0 && !seg) || !lr || !step_state)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_adam_l2: bad buffer, size or segment list");
  CIS_LAUNCH(adam_l2_kernel, nblk((size_t)n), 256, 0, ST, param, m, v, grad, (size_t)n, (const long long*)seg, nseg, decay, lr, beta1, beta2, eps,
             (const long long*)step_state);
  CIS_LAUNCH(step_inc_kernel, 1, 1, 0, ST, (long long*)step_state);
  return cis_check_launch("adam_l2");
}
int cis_unsup_flow_loss(const float* flow, const float* img1, const float* img2, int32_t B, int32_t H, int32_t W, float* warped, float* mask,
                        float* coef, double* scratch, double* out, cis_stream_t stream) {
  UnsupArgs a;
  const int rc = unsup_args("cis_unsup_flow_loss: bad frames, flow alignment or size (B 1..65535, H, W >= 3)", flow, img1, img2, B, H, W, a);
  if (rc) return rc;
  if (!warped || !mask || !coef || !scratch || !out) return cis_set_error(CIS_ERR_BAD_ARG, "cis_unsup_flow_loss: no buffer, scratch or output");
  CIS_LAUNCH(unsup_warp_mask_kernel, nblk((size_t)2 * B * H * W), 256, 0, ST, a, warped, mask);
  CIS_LAUNCH(unsup_census_kernel, 2 * B * kUnsupBlocks, 256, 0, ST, a, (const float*)warped, (const float*)mask, coef, scratch);
  CIS_LAUNCH(unsup_reduce_kernel, 2 * B, 2, 0, ST, (const double*)scratch, out);
  return cis_check_launch("unsup_flow_loss");
}
int cis_unsup_flow_loss_bwd(const float* flow, const float* img1, const float* img2, int32_t B, int32_t H, int32_t W, const float* warped,
                            const float* coef, float w_photo, float w_smooth, float* dflow, cis_stream_t stream) {
  UnsupArgs a;
  const int rc = unsup_args("cis_unsup_flow_loss_bwd: bad frames, flow alignment or size (B 1..65535, H, W >= 3)", flow, img1, img2, B, H, W, a);
  if (rc) return rc;
  const size_t blocks = (size_t)((H + kUnsupTY - 1) / kUnsupTY) * ((W + kUnsupTX - 1) / kUnsupTX) * 2 * B;
  if (!warped || !coef || !dflow || ((uintptr_t)dflow & 7) || blocks > 0x7fffffff)
    return cis_set_error(CIS_ERR_BAD_ARG, "cis_unsup_flow_loss_bwd: bad buffer, dflow alignment or grid size");
  CIS_LAUNCH(unsup_bwd_kernel, (unsigned)blocks, 256, 0, ST, a, warped, coef, w_photo, w_smooth, dflow);
  return cis_check_launch("unsup_flow_loss_bwd");
}

}  // extern "C"
