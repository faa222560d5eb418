// Error plumbing + version of libcis_b200.so (C ABI declared in include/cis_b200.h).
#include "../../include/cis_b200.h"
#include "common.cuh"
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <math.h>

static thread_local char g_err[512] = "";

int cis_set_error(int code, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return code;
}
int cis_set_cuda_error(cudaError_t e, const char* where) {
  snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
  return CIS_ERR_CUDA;
}
int cis_check_launch(const char* where) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cis_set_cuda_error(e, where);
  return CIS_OK;
}
int cis_num_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) return 132;
  return n;
}
extern "C" const char* cis_last_error(void) { return g_err; }
extern "C" int cis_version(void) { return 100; }

// ---- host CRC-32C, slicing-by-8 (tables built once) ----------------------------------------------------------------------
static uint32_t g_crc_tab[8][256];
static bool g_crc_init = false;
static void crc_init() {
  for (uint32_t i = 0; i < 256; i++) {
    uint32_t c = i;
    for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : (c >> 1);
    g_crc_tab[0][i] = c;
  }
  for (uint32_t i = 0; i < 256; i++)
    for (int t = 1; t < 8; t++) g_crc_tab[t][i] = (g_crc_tab[t - 1][i] >> 8) ^ g_crc_tab[0][g_crc_tab[t - 1][i] & 0xff];
  g_crc_init = true;
}
extern "C" uint32_t cis_crc32c(uint32_t crc, const void* data, size_t n) {
  if (!g_crc_init) crc_init();
  const unsigned char* p = (const unsigned char*)data;
  uint32_t c = ~crc;
  while (n && ((uintptr_t)p & 7)) { c = g_crc_tab[0][(c ^ *p++) & 0xff] ^ (c >> 8); n--; }
  while (n >= 8) {
    uint64_t v;
    memcpy(&v, p, 8);
    v ^= c;
    c = g_crc_tab[7][v & 0xff] ^ g_crc_tab[6][(v >> 8) & 0xff] ^ g_crc_tab[5][(v >> 16) & 0xff] ^ g_crc_tab[4][(v >> 24) & 0xff] ^
        g_crc_tab[3][(v >> 32) & 0xff] ^ g_crc_tab[2][(v >> 40) & 0xff] ^ g_crc_tab[1][(v >> 48) & 0xff] ^ g_crc_tab[0][v >> 56];
    p += 8; n -= 8;
  }
  while (n--) c = g_crc_tab[0][(c ^ *p++) & 0xff] ^ (c >> 8);
  return ~c;
}

// ---- host-side frame preprocessing for the dataset readers (SURVEY 8f-2) -------------------------------------------------------
// tf.image.resize_images (legacy bilinear: src = dst * in/out, no half-pixel shift, neighbours clamped) on an HWC float image; the
// arithmetic order matches the numpy restatement in data/davis2016_data_utils.py (t = tl + (tr - tl) * fx, ...) so both agree bit
// for bit.  Replaces the tf.data map functions of the reference (data/davis2016_data_utils.py:84-134) on the CPU; ~1.5 ms per
// 384x640x3 frame instead of ~35 ms in numpy, which is what keeps a 6-thread reader near the GPU step rate.
// per-axis sample table: lower index, upper index (clamped), fraction -- computed once per call
static void host_axis(int n_in, int n_out, int* lo, int* hi, float* fr) {
  const float s = (float)((double)n_in / (double)n_out);
  for (int o = 0; o < n_out; ++o) {
    const float f = (float)o * s;
    const int a = (int)floorf(f);
    lo[o] = a;
    hi[o] = a + 1 < n_in ? a + 1 : n_in - 1;
    fr[o] = f - (float)a;
  }
}
extern "C" int cis_host_resize_bilinear_legacy(const float* src, int32_t H, int32_t W, int32_t C, float* dst, int32_t OH, int32_t OW) {
  if (!src || !dst || H < 1 || W < 1 || C < 1 || OH < 1 || OW < 1) return cis_set_error(CIS_ERR_BAD_ARG, "cis_host_resize_bilinear_legacy: bad arguments");
  int* xl = (int*)malloc(sizeof(int) * 2 * (size_t)(OW + OH));
  float* xf = (float*)malloc(sizeof(float) * (size_t)(OW + OH));
  if (!xl || !xf) { free(xl); free(xf); return cis_set_error(CIS_ERR_BAD_ARG, "cis_host_resize_bilinear_legacy: out of memory"); }
  int *xh = xl + OW, *yl = xh + OW, *yh = yl + OH;
  float* yf = xf + OW;
  host_axis(W, OW, xl, xh, xf);
  host_axis(H, OH, yl, yh, yf);
  for (int oy = 0; oy < OH; ++oy) {
    const float fy = yf[oy];
    const float* r0 = src + (size_t)yl[oy] * W * C;
    const float* r1 = src + (size_t)yh[oy] * W * C;
    float* o = dst + (size_t)oy * OW * C;
    for (int ox = 0; ox < OW; ++ox) {
      const float fx = xf[ox];
      const float *tl = r0 + (size_t)xl[ox] * C, *tr = r0 + (size_t)xh[ox] * C, *bl = r1 + (size_t)xl[ox] * C, *br = r1 + (size_t)xh[ox] * C;
      for (int c = 0; c < C; ++c) {
        const float t = tl[c] + (tr[c] - tl[c]) * fx;
        const float b = bl[c] + (br[c] - bl[c]) * fx;
        o[(size_t)ox * C + c] = t + (b - t) * fy;
      }
    }
  }
  free(xl);
  free(xf);
  return CIS_OK;
}
// decoded BGR uint8 frame -> RGB float (v / 255 - 0.5, preprocess_image :84-90) resized to OH x OW with the same legacy rule, in one pass
extern "C" int cis_host_bgr8_to_rgb_resized(const unsigned char* bgr, int32_t H, int32_t W, float* dst, int32_t OH, int32_t OW) {
  if (!bgr || !dst || H < 1 || W < 1 || OH < 1 || OW < 1) return cis_set_error(CIS_ERR_BAD_ARG, "cis_host_bgr8_to_rgb_resized: bad arguments");
  float lut[256];
  for (int v = 0; v < 256; ++v) lut[v] = (float)v / 255.0f - 0.5f;
  int* xl = (int*)malloc(sizeof(int) * 2 * (size_t)(OW + OH));
  float* xf = (float*)malloc(sizeof(float) * (size_t)(OW + OH));
  if (!xl || !xf) { free(xl); free(xf); return cis_set_error(CIS_ERR_BAD_ARG, "cis_host_bgr8_to_rgb_resized: out of memory"); }
  int *xh = xl + OW, *yl = xh + OW, *yh = yl + OH;
  float* yf = xf + OW;
  host_axis(W, OW, xl, xh, xf);
  host_axis(H, OH, yl, yh, yf);
  for (int oy = 0; oy < OH; ++oy) {
    const float fy = yf[oy];
    const unsigned char* r0 = bgr + (size_t)yl[oy] * W * 3;
    const unsigned char* r1 = bgr + (size_t)yh[oy] * W * 3;
    float* o = dst + (size_t)oy * OW * 3;
    for (int ox = 0; ox < OW; ++ox) {
      const float fx = xf[ox];
      const int a = xl[ox] * 3, b2 = xh[ox] * 3;
      for (int c = 0; c < 3; ++c) {
        const int s = 2 - c;   // BGR -> RGB
        const float tl = lut[r0[a + s]], tr = lut[r0[b2 + s]], bl = lut[r1[a + s]], br = lut[r1[b2 + s]];
        const float t = tl + (tr - tl) * fx;
        const float b = bl + (br - bl) * fx;
        o[ox * 3 + c] = t + (b - t) * fy;
      }
    }
  }
  free(xl);
  free(xf);
  return CIS_OK;
}
