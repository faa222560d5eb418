/* cis_b200.h - C ABI of libcis_b200.so: the sm_90a kernels behind the adversarial motion-segmentation hot path.
 *
 * The reference (antonilo/unsupervised_detection @ 46cae6e) has no FFI layer: its "operators" are TensorFlow 1.13 graph
 * ops called from Python (SURVEY.md section 8b).  Each entry point below replaces the TF op class used at the cited
 * reference call site.  All pointers are DEVICE pointers owned by the caller (torch-allocated), every call only enqueues
 * work on `stream` and returns immediately; return value 0 = OK, non-zero = CIS_ERR_* (see cis_last_error()).
 * No torch types appear in any signature.  Layout everywhere: NHWC, activations bf16 with the channel pitch a multiple
 * of 8 (16-byte pixels chunks), flows/masks/losses fp32.
 */
#ifndef CIS_B200_H_
#define CIS_B200_H_
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* cis_stream_t; /* cudaStream_t */

enum { CIS_OK = 0, CIS_ERR_BAD_ARG = 1, CIS_ERR_UNSUPPORTED = 2, CIS_ERR_CUDA = 3 };
enum { CIS_ACT_NONE = 0, CIS_ACT_ELU = 1, CIS_ACT_LEAKY = 2 };
enum { CIS_MAX_TAPS = 49, CIS_MAX_SRC = 4 };

/* One channel slice of a bf16 NHWC tensor: a member of a virtual concat (tf.concat, nets.py:78-105,
 * model_pwcnet.py:482-502) that is never materialised. */
typedef struct {
  const void* ptr; /* bf16 base of the underlying buffer [N,H,W,pitch] */
  int32_t pitch;   /* channels per pixel of the underlying buffer (multiple of 8) */
  int32_t c_off;   /* first channel of the slice (multiple of 8) */
  int32_t chunks;  /* slice width in 8-channel chunks */
  int32_t n_mod;   /* >0: batch index taken modulo n_mod (features shared by the 3 recover_net calls) */
} CisSrc;

/* Implicit-GEMM convolution on the tensor cores (wgmma): D[rows=(n,oh,ow)][BN] = sum_k A[row][k] * Wp[n][k],
 * A[row][(t,c)] = src[n, oh*sh + dh[t], ow*sw + dw[t], c] (zero outside the image = TF 'SAME' padding).
 * With suitable tap tables this one kernel is: tf.layers.conv2d / tf.nn.conv2d forward (convolution_utils.py:46,81;
 * model_pwcnet.py:161-165,484-504,562-574), its data gradient (stride 1: flipped taps; stride 2: four parity launches),
 * and tf.layers.conv2d_transpose k4 s2 (model_pwcnet.py:286; four parity launches). */
typedef struct {
  int32_t N, H, W;   /* source batch / height / width */
  int32_t OH, OW;    /* GEMM row grid; rows = N*OH*OW */
  int32_t sh, sw;    /* source coordinate = row coordinate * s + tap offset */
  int32_t ntaps;
  int16_t dh[CIS_MAX_TAPS];
  int16_t dw[CIS_MAX_TAPS];
  int32_t nsrc;
  CisSrc src[CIS_MAX_SRC];
  const void* wpack; /* halo=0: bf16 [n_tiles*BN][K_pad], K order (tap, concat channel), K_pad multiple of 64;
                        halo=1: pre-swizzled tiles from cis_pack_weights_tiled */
  int32_t K_pad;
  int32_t BN;        /* N tile: 16, 32, 64 or 128 */
  int32_t n_tiles;   /* grid.y; padded output channels = n_tiles*BN */
  const float* bias; /* fp32 [n_tiles*BN] or NULL */
  int32_t act;       /* CIS_ACT_* */
  float alpha;       /* leaky slope */
  int32_t DH, DW;    /* destination height / width */
  int32_t osh, osw, oa, ob; /* destination pixel = (oh*osh + oa, ow*osw + ob) */
  void* out;         /* bf16 destination or NULL */
  int32_t out_pitch, out_coff, out_ch;
  float* outf;       /* fp32 destination or NULL */
  int32_t outf_pitch, outf_coff, outf_ch;
  const void* add_pre; /* bf16, added before the activation (gradient accumulation) */
  int32_t add_pre_pitch, add_pre_coff;
  const float* addf_pre; /* fp32, added before the activation (PWC flow + context residual, model_pwcnet.py:576) */
  int32_t addf_pitch, addf_coff;
  const void* add_post; /* bf16, added after the activation (generator skips, nets.py:29,32,33) */
  int32_t add_post_pitch, add_post_coff;
  int32_t mode;      /* 0 normal; 1: outf[pix] = sigmoid((l0 - l1)/10)  (nets.py:38-41) */
  /* halo-resident variant (stride-1 gathers only): the CTA tile is MT stacked 16x8-pixel blocks of dilation phase (a,b);
   * the (16*MT+ey) x (8+ex) input halo of a 64-channel chunk is staged ONCE in shared memory and all taps read it through
   * shifted wgmma descriptors.  dh/dw then hold tap offsets >= 0 relative to the halo origin, in units of `dil` pixels. */
  int32_t halo;      /* 0: generic per-tap gather kernel, 1: halo-resident kernel */
  int32_t dil;       /* dilation = phase period (1 for undilated) */
  int32_t MT;        /* 1..4 stacked M tiles per MMA warpgroup (MT*BN <= 128 register accumulator columns); see nwg */
  int32_t hoy, hox;  /* halo origin relative to the tile origin (phase units, <= 0) */
  int32_t ey, ex;    /* halo extent beyond the tile (max tap offset) */
  /* Split-K for launches that cover only a few SMs (low-resolution layers): grid.z = splits CTAs share one output tile, each reduces a
   * range of the K loop (64-wide K blocks for the gather kernel, 64-channel chunks for the halo kernel) and stores its partial fp32
   * tile to a private slice of sk_scratch; a second kernel launched by the same call sums the slices in a fixed order
   * (deterministic) and runs the fused epilogue spread over many CTAs. */
  int32_t splits;        /* 0/1 = off */
  float* sk_scratch;     /* >= tiles * splits * 128 * BN floats (tiles = grid.x * grid.y * MT * max(nwg, 1)); need not be initialised */
  int32_t* sk_counters;  /* must be NULL (the single-launch ticket mode of round 1 was removed; the field keeps the struct layout) */
  /* Stride-2 forward convolution on the halo kernel (halo = 1, sh = sw = 1 in this descriptor, H x W = the INPUT size): the input is
   * read as nph = 4 space-to-depth phases in(2y + py, 2x + px), phase index py*2 + px; taps are listed phase by phase in PHASE
   * coordinates (dh/dw relative to the halo origin of the phase images) and taps [ph_tap[i], ph_tap[i+1]) belong to phase i.  With
   * `thin` set, ph_tap still counts taps, not K=16 steps: one halo stage holds the planes of the four phases, phase-major, so an
   * 8-channel step pairs taps 2s and 2s+1 even where they belong to two phases (the second one's origin lies in a later plane).
   * nph = 0/1: ordinary stride-1 gather. */
  int32_t nph;
  int32_t ph_tap[5];
  /* 1: the `splits` CTAs of a tile form a thread-block cluster (2..8 CTAs) and reduce their partial accumulators through distributed
   * shared memory inside the conv kernel (fixed summation order, fused epilogue spread over the cluster): no sk_scratch, no second launch. */
  int32_t sk_cluster;
  /* Grouped launch (halo kernel, splits <= 1): nsub = 2..4 sub-problems that share sources, epilogue, BN / n_tiles / MT and the halo box
   * (ey, ex) but have their own tap set, halo origin, packed weights, output extent and output offset -- the four output-parity
   * launches of a stride-2 data gradient or of conv2d_transpose(k4, s2) as ONE launch (blockIdx.z = sub-problem).  The taps of all
   * sub-problems are listed back to back in dh / dw (ntaps = their total); nsub = 0/1: ordinary launch. */
  int32_t nsub;
  struct {
    int32_t tap0, ntaps;      /* this sub-problem's taps: dh/dw[tap0 .. tap0 + ntaps) */
    int32_t hoy, hox;         /* halo origin relative to the output tile */
    int32_t OH, OW, oa, ob;   /* output extent and offset inside the (DH, DW) destination grid (stride osh / osw) */
    const void* wpack;        /* pre-tiled weights of this sub-problem */
  } sub[4];
  /* halo kernel, BN >= 64: 2 = two MMA warpgroups share every weight stage, each owning MT stacked tiles, so the CTA covers 2*MT tiles
   * (16*2*MT output rows per column of tiles; split-K scratch and the grid count CTAs of that height).  0/1: one warpgroup. */
  int32_t nwg;
  /* halo kernel, undilated (stride 1 or nph = 4), sources totalling 8 or 16 channels: the compact K-dense operand format.  0: 64-channel
   * SWIZZLE_128B chunks, one K=16 step per tap.  8 / 16: the halo is staged without swizzle at 16 bytes per pixel, one plane per 8
   * channels, so 8 consecutive halo pixels are one wgmma core matrix; a K=16 step covers two taps (8: taps 2s, 2s+1, LBO = the distance of
   * their origins, which the host lists in increasing order) or one tap (16: LBO = the plane distance).  wpack / sub[].wpack then hold
   * cis_pack_weights_tiled(thin) tiles. */
  int32_t thin;
} CisConv;

/* Weight gradient of the same convolution: dWp[co][(t,c)] = sum_rows g[row][co] * A[row][(t,c)]  (fp32).  The reduction over rows
 * is split over `splits` CTAs per column tile; every split writes its own private slice of Cout x K_pad floats with plain stores
 * (element order: [co][K_pad] for tma == 2, float4 columns [K_pad/4][co][4] for tma 0 / 1 -- see cis_unpack_wgrad's `layout`)
 * (no atomics, nothing to zero) and cis_unpack_wgrad sums the slices in a fixed order -- the weight gradient is bit-reproducible.
 * Replaces the conv2d backprop-filter ops TF1 emits for tf.gradients (loss_utils.py:17). */
typedef struct {
  int32_t N, H, W, OH, OW, sh, sw, ntaps;
  int16_t dh[CIS_MAX_TAPS];
  int16_t dw[CIS_MAX_TAPS];
  int32_t nsrc;
  CisSrc src[CIS_MAX_SRC];
  const void* g;     /* bf16 gradient w.r.t. the pre-activation output on the (n,oh,ow) row grid */
  int32_t g_pitch, g_coff, g_chunks;
  float* dwp;        /* fp32 [splits][Cout][K_pad] private slices; every split must own >= 1 reduction block (ceil-division on the host) */
  int32_t Cout;      /* <= 128 */
  int32_t K_pad;
  int32_t splits;    /* split-K factor (grid.y) */
  int32_t tma;       /* 2: experimental halo-resident variant of 1 (same dwp layout; one activation halo per pixel tile, taps read in place);
                        1: stride-1 layer, operands fetched as 8x8-pixel TMA tiles; dwp columns are then laid out per tap in
                        64-channel groups: col = (tap*ceil(Cin8/64) + chunk64)*64 + c, K_pad = that extent rounded to 128 */
  /* tma == 2 tiling.  nh = MMA N (16 / 32 / 64; 0 = 64): at least Cout rounded up to 16, and 64 when Cout > 64; one MMA warpgroup
   * holds 128 / nh tap pairs.  nwg = MMA warpgroups per CTA (0/1 = one, 2 = two on the same stages: the two 64-channel halves of
   * Cout when Cout > 64, else twice the tap pairs). */
  int32_t nh;
  int32_t nwg;
} CisWgrad;

const char* cis_last_error(void);
int cis_version(void);
/* Host-side CRC-32C (Castagnoli, reflected 0x82F63B78), extend form: returns crc32c(concat(A, data)) given crc = crc32c(A)
 * (pass 0 to start).  Used by the TF tensor-bundle checkpoint reader/writer (SURVEY 8f-1); it replaces
 * tensorflow/core/lib/hash/crc32c.h (TensorFlow 1.13, third-party, not vendored in the reference) behind
 * tf.train.Saver (models/adversarial_learner.py:326-331).  Not a stream operation; no GPU needed. */
uint32_t cis_crc32c(uint32_t crc, const void* data, size_t n);
/* Host-side frame preprocessing for the dataset readers (no GPU, not stream operations; thread-safe, callers run them from a thread pool).
 * tf.image.resize_images legacy bilinear on an HWC float image, and the fused decode-side step of preprocess_image
 * (data/davis2016_data_utils.py:84-90 of the reference): BGR uint8 -> RGB float v/255-0.5 -> legacy bilinear to OH x OW. */
int cis_host_resize_bilinear_legacy(const float* src, int32_t H, int32_t W, int32_t C, float* dst, int32_t OH, int32_t OW);
int cis_host_bgr8_to_rgb_resized(const unsigned char* bgr, int32_t H, int32_t W, float* dst, int32_t OH, int32_t OW);

/* A gather launch (halo = 0) with stride 2 whose sources total 8 or 16 channels and whose grid has at least 296 16x8 tiles runs on the
 * halo kernels as a compact phase-halo launch (nph = 4, thin set) that reads its weights in place from the row pack wpack.  cis_conv_s2_phase_plan (host only, no stream) returns 1
 * and that launch's descriptor in *h, with the row-pack K column of kgroup j of K=16 step s in wk[2 s + j] (2 * CIS_MAX_TAPS entries),
 * or 0 when cis_conv_igemm runs d on the gather kernel. */
int cis_conv_igemm(const CisConv* d, cis_stream_t stream);
int cis_conv_s2_phase_plan(const CisConv* d, CisConv* h, int16_t* wk);
/* which launches use the persistent warp-specialised halo kernel: 0 none, 1 thin single-chunk layers (default), 2 all eligible,
 * 3 = 1 + the weight-stationary variant for thin layers whose whole weight set fits in shared memory (experimental),
 * -1 back to the default / CIS_PERSIST_MODE environment variable.  Host-side switch, not a stream operation. */
int cis_set_persist_mode(int mode);
int cis_conv_wgrad(const CisWgrad* d, cis_stream_t stream);

/* ---- parameter-space helpers (fp32 master weights <-> packed bf16 operands) ---- */
/* wp[n][k] = (kmap[k] >= 0 && ne >= 0) ? w[kmap[k] + ne*sn] : 0 for n < rows, ne = nmap ? nmap[n] : (n < cout ? n : -1). */
int cis_pack_weights(const float* w, const int32_t* kmap, int32_t K_pad, int32_t rows, int32_t cout, int32_t sn, const int32_t* nmap,
                     void* wp, cis_stream_t stream);
/* halo-kernel operand: out[(ny, chunk, tap)][n][64] bf16 blocks of BN x 128 B with the SWIZZLE_128B pattern pre-applied; kmap is the
 * same tap-major map (k = tap*cin8 + channel).  thin = 8 / 16 (CisConv.thin, cin8 == thin): out[(ny, step)] = BN x 32 B no-swizzle
 * K=16 tiles instead, core matrix (n / 8, kgroup) at (n / 8) * 256 + kgroup * 128 bytes; kgroup j of step s is tap 2s + j (thin 8, zero
 * past the last tap) or channels 8j .. 8j + 7 of tap s (thin 16). */
int cis_pack_weights_tiled(const float* w, const int32_t* kmap, int32_t cin8, int32_t ntaps, int32_t n_tiles, int32_t BN, int32_t cout,
                           int32_t sn, const int32_t* nmap, void* out, int32_t thin, cis_stream_t stream);
/* dw[kmap[k] + n*sn] = sum_{s < nsplit} dwp[s](n, k) for kmap[k] >= 0, n < cout (fixed summation order);
 * and, when colpart != NULL, the bias gradient db[c] = sum_{b < nblocks} colpart[b][c], c < nch (the partials of cis_colsum).
 * layout bits 0-7 = how cis_conv_wgrad stored a slice: 0 = [cout][K_pad] (CisWgrad.tma == 2), 1 = float4 columns [K_pad/4][cout][4]
 * (tma 0 / 1); bits 8+ = sn, the stride of n in dw (0 means 1: the HWIO slot of a conv; Cin: the [kh,kw,Cout,Cin] slot of a transposed
 * conv, model_pwcnet.py:286). */
int cis_unpack_wgrad(const float* dwp, const int32_t* kmap, int32_t K_pad, int32_t cout, int32_t nsplit, float* dw, const float* colpart,
                     int32_t nblocks, int32_t nch, float* db, int32_t layout, cis_stream_t stream);
/* tf.layers.batch_normalization in inference mode folded into the conv (convolution_utils.py:46-51):
 * w_eff = w * gamma/sqrt(1+1e-3); b_eff = bias*gamma/sqrt(1+1e-3) + beta. */
int cis_bn_fold(const float* w, const float* bias, const float* gamma, const float* beta, int64_t nw, int32_t cout, float* w_eff,
                float* b_eff, cis_stream_t stream);
/* chain rule back to (w, bias, gamma, beta) from (dw_eff, db_eff); dw_eff is overwritten in place by dw. */
int cis_bn_chain(const float* w, const float* bias, const float* gamma, float* dw_eff_to_dw, const float* db_eff, int64_t nw,
                 int32_t cout, float* dbias, float* dgamma, float* dbeta, cis_stream_t stream);

/* Multi-job form of the five parameter-space ops above: ONE launch over a flat grid of 256-thread blocks.  A job holds the arguments of
 * the single-launch entry point of its kind in order: pointers in p[], the size_t argument (nw) in n, the int arguments in i[0..6]
 * (bn_chain: p[0..7] = w, bias, gamma, dw_eff, db_eff, dbias, dgamma, dbeta), and in i[7] the index of its first block; job j owns blocks
 * [i[7] of j, i[7] of j+1) and needs ceil(elements / 256) of them (bn_chain: cout).  The table lives in device memory, sorted by i[7];
 * total_blocks = the sum.  Jobs of one launch must not depend on each other. */
enum { CIS_JOB_PACK = 0, CIS_JOB_PACK_TILED = 1, CIS_JOB_UNPACK = 2, CIS_JOB_BN_FOLD = 3, CIS_JOB_BN_CHAIN = 4 };
typedef struct {
  int32_t kind;
  int32_t i[8];
  int64_t n;
  const void* p[8];
} CisParamJob;
int cis_param_multi(const CisParamJob* jobs_dev, int32_t njobs, int32_t total_blocks, cis_stream_t stream);

/* ---- elementwise / reduction helpers on bf16 NHWC slices ---- */
/* g *= act'(y - res)   (ELU: u>0 ? 1 : u+1; leaky: u>0 ? 1 : alpha) */
int cis_dact_mul(void* g, int32_t g_pitch, int32_t g_coff, const void* y, int32_t y_pitch, int32_t y_coff, const void* res,
                 int32_t res_pitch, int32_t res_coff, int64_t npix, int32_t chunks, int32_t act, float alpha, cis_stream_t stream);
/* dst (=|+=) sum_{j<reps} src[(pix + j*npix_dst)]  : gradient accumulation and the 3-call fold of shared features */
int cis_add_slice(void* dst, int32_t dst_pitch, int32_t dst_coff, const void* src, int32_t src_pitch, int32_t src_coff,
                  int64_t npix_dst, int32_t chunks, int32_t reps, int32_t accumulate, cis_stream_t stream);
/* part[b][c] = sum over the pixels of block b of g[pix][c], c < nch, b < nblocks (<= 592): per-block partial column sums, no atomics;
 * cis_unpack_wgrad adds them up in block order (deterministic bias gradient). */
int cis_colsum(const void* g, int32_t g_pitch, int32_t g_coff, int64_t npix, int32_t nch, float* part, int32_t nblocks, cis_stream_t stream);

/* zero-fill of the small accumulators a step starts from (flow statistics, loss sums, gradient magnitude): stream-ordered memset */
int cis_zero(void* ptr, int64_t nbytes, cis_stream_t stream);

/* cis_dact_mul and cis_colsum of the same gradient slice in one pass: g *= act'(y - res) in place, part[b][c] = block b's column sums of
 * the rounded product (bit-identical to the two separate calls with the same nblocks). */
int cis_dact_colsum(void* g, int32_t g_pitch, int32_t g_coff, const void* y, int32_t y_pitch, int32_t y_coff, const void* res,
                    int32_t res_pitch, int32_t res_coff, int64_t npix, int32_t nch, int32_t act, float alpha, float* part, int32_t nblocks,
                    cis_stream_t stream);

/* ---- resampling (App. A.5/A.6 semantics) ---- */
/* tf.image.resize_images / resize_bilinear legacy (convolution_utils.py:88, nets.py:108) on a bf16 slice */
int cis_resize_bilinear_bf16(const void* src, int32_t s_pitch, int32_t s_coff, int32_t N, int32_t H, int32_t W, void* dst,
                             int32_t d_pitch, int32_t d_coff, int32_t OH, int32_t OW, int32_t chunks, cis_stream_t stream);
/* fused resize + concat of the recover decoder (convolution_utils.py:87-90 feeding nets.py:80-105): up to 4 sources of one resolution
 * (channel slices, batch-broadcast when n_mod > 0) -> legacy-bilinear to OH x OW -> side by side into one destination slice.
 * H x W == OH x OW makes it a plain concat copy. */
int cis_resize_concat_bf16(const CisSrc* srcs, int32_t nsrc, int32_t N, int32_t H, int32_t W, void* dst, int32_t d_pitch, int32_t d_coff,
                           int32_t OH, int32_t OW, cis_stream_t stream);
/* its transpose: for every source i with want[i]: grads[i] (=|+= when accumulate[i]) sum over broadcast replicas of R^T ddst[slice i];
 * grads[i].chunks must equal the forward source's (it positions the slice inside ddst), N = batch rows of ddst processed. */
int cis_resize_concat_bf16_bwd(const void* ddst, int32_t d_pitch, int32_t d_coff, int32_t N, int32_t OH, int32_t OW, const CisSrc* grads,
                               const int32_t* want, const int32_t* accumulate, int32_t nsrc, int32_t H, int32_t W, cis_stream_t stream);
/* its transpose: dsrc (=|+=) R^T ddst */
int cis_resize_bilinear_bf16_bwd(const void* ddst, int32_t d_pitch, int32_t d_coff, int32_t N, int32_t OH, int32_t OW, void* dsrc,
                                 int32_t s_pitch, int32_t s_coff, int32_t H, int32_t W, int32_t chunks, int32_t accumulate,
                                 cis_stream_t stream);
/* fp32, C channels: dst = scale * resize(src)  (adversarial_learner.py:87-97, model_pwcnet.py:646) */
int cis_resize_bilinear_f32(const float* src, int32_t N, int32_t H, int32_t W, int32_t C, float* dst, int32_t OH, int32_t OW,
                            float scale, cis_stream_t stream);
/* tf.image.resize_nearest_neighbor(align_corners=True) x2 (convolution_utils.py:71) and its transpose */
int cis_upsample_nn2x(const void* src, int32_t N, int32_t H, int32_t W, int32_t pitch, void* dst, cis_stream_t stream);
int cis_upsample_nn2x_bwd(const void* ddst, int32_t N, int32_t H, int32_t W, int32_t pitch, void* dsrc, int32_t accumulate,
                          cis_stream_t stream);
/* central crop (box y0, x0, ch, cw of ONE Hs x Ws x C fp32 NHWC image) resized back to OH x OW with the legacy bilinear rule: the
 * multi-crop test-time augmentation of test_generator_ensemble (data/davis2016_data_utils.py:130-134, 328-354) on the device */
int cis_crop_resize_bilinear_f32(const float* src, int32_t Hs, int32_t Ws, int32_t C, int32_t y0, int32_t x0, int32_t ch, int32_t cw, float* dst,
                                 int32_t OH, int32_t OW, cis_stream_t stream);
/* the same crop and resize of ONE Hs x Ws x 2 flow field, whose vectors follow the resize: channel 0 times s0, channel 1 times s1
 * (PWC-Net's channel order: s0 = OH / ch for rows, s1 = OW / cw for columns) -- the supplied flow of the multi-crop ensemble */
int cis_crop_resize_flow_f32(const float* src, int32_t Hs, int32_t Ws, int32_t y0, int32_t x0, int32_t ch, int32_t cw, float* dst, int32_t OH,
                             int32_t OW, float s0, float s1, cis_stream_t stream);
/* tf.image.resize_images(NEAREST_NEIGHBOR) for GT masks (adversarial_learner.py:92-94) */
int cis_resize_nn_f32(const float* src, int32_t N, int32_t H, int32_t W, int32_t C, float* dst, int32_t OH, int32_t OW,
                      cis_stream_t stream);
/* tf.image.resize_bilinear / resize_nearest_neighbor with TF 1.13 semantics (no half-pixel centres) on fp32 NHWC [N,H,W,C] -> [N,OH,OW,C],
 * any sizes up or down (the `func` of convolution_utils.py:4-24).  Step = (in-1)/(out-1) when align_corners and out > 1, else in/out (fp32);
 * bilinear: lo = floor(d*step), hi = min(lo+1, in-1); nearest: roundf(d*step) with align_corners, floor without, clamped to in-1.
 * method = CIS_RESIZE_*, align_corners = 0 / 1 (CIS_ERR_BAD_ARG otherwise, and for sizes < 1).  method = BILINEAR, align_corners = 0
 * computes cis_resize_bilinear_f32 with scale 1; NEAREST, 0 computes cis_resize_nn_f32. */
enum { CIS_RESIZE_BILINEAR = 0, CIS_RESIZE_NEAREST = 1 };
int cis_resize_f32(const float* src, int32_t N, int32_t H, int32_t W, int32_t C, float* dst, int32_t OH, int32_t OW, int32_t method,
                   int32_t align_corners, cis_stream_t stream);
/* its transpose: dsrc [N,H,W,C] = R^T ddst [N,OH,OW,C] (overwritten).  A gather with no atomics: every dsrc element sums its own
 * contiguous rectangle of ddst in a fixed order, so the result is bit-identical run to run, for downsampling as well. */
int cis_resize_f32_bwd(const float* ddst, int32_t N, int32_t OH, int32_t OW, int32_t C, int32_t H, int32_t W, float* dsrc, int32_t method,
                       int32_t align_corners, cis_stream_t stream);

/* ---- PWC-Net warp + cost volume (core_warp.py:153-202 fused into core_costvol.py:20-40) ----
 * out[b,y,x,9*dy+dx] = leaky0.1( mean_c c1[b,y,x,c] * warp(c2, flow)[b,y+dy-4,x+dx-4,c] ), zero outside; flow may be
 * NULL (level 6: no warp).  flow is fp32 [B,h,w,2] and is multiplied by flow_scale (model_pwcnet.py:616-617). */
int cis_warp_costvol(const void* c1, int32_t c1_pitch, int32_t c1_coff, const void* c2, int32_t c2_pitch, int32_t c2_coff,
                     const float* flow, float flow_scale, int32_t B, int32_t h, int32_t w, int32_t C, void* out, int32_t out_pitch,
                     int32_t out_coff, cis_stream_t stream);
/* the same for search range 1 <= search_range <= 4 (model_pwcnet.py option 'search_range'; cis_warp_costvol is search_range = 4):
 * (2r+1)^2 channels out[b,y,x,(2r+1)*dy+dx], displacement (dy-r, dx-r).  CIS_ERR_BAD_ARG outside 1..4. */
int cis_warp_costvol_r(const void* c1, int32_t c1_pitch, int32_t c1_coff, const void* c2, int32_t c2_pitch, int32_t c2_coff,
                       const float* flow, float flow_scale, int32_t B, int32_t h, int32_t w, int32_t C, void* out, int32_t out_pitch,
                       int32_t out_coff, int32_t search_range, cis_stream_t stream);
/* standalone dense_image_warp (core_warp.py:153) on a bf16 slice -> bf16, for parity tests of the gather */
int cis_dense_image_warp(const void* img, int32_t pitch, int32_t coff, const float* flow, float flow_scale, int32_t B, int32_t h,
                         int32_t w, int32_t C, void* out, int32_t out_pitch, cis_stream_t stream);

/* ---- input packing ---- */
/* bf16 [N,H,W,8] = (src fp32 [N,H,W,C] + offset), zero padded (model_pwcnet.py:39-56 adapt_x) */
int cis_pack_f32_to_bf16(const float* src, int64_t npix, int32_t C, float offset, void* dst, int32_t d_pitch, int32_t d_coff,
                         cis_stream_t stream);
/* per-sample sums for tf.nn.moments (flow_utils.py:10): stats[b] = {sum f0, sum f1, sum f0^2, sum f1^2} (double, zeroed) */
int cis_flow_stats(const float* flow, int32_t B, int64_t hw, double* stats, cis_stream_t stream);
/* generator input = concat(image, (flow-mean)/sqrt(var)) -> bf16 [B,H,W,8]  (nets.py:14, flow_utils.py:5-12) */
int cis_pack_generator_input(const float* image, const float* flow, const double* stats, int32_t B, int64_t hw, void* dst,
                             cis_stream_t stream);
/* stand-alone preprocess_flow_batch (flow_utils.py:5-12): out fp32 [B,hw,2] = (flow - mean) / sqrt(population variance) per sample and
 * channel, no epsilon, with the statistics of cis_flow_stats (the normalisation cis_pack_generator_input applies, in fp32) */
int cis_flow_standardize(const float* flow, const double* stats, int32_t B, int64_t hw, float* out, cis_stream_t stream);
/* its gradient: dx = (dy - mean(dy) - y * mean(dy * y)) / sigma per sample and channel, y = the forward output.  The two means are
 * fixed-order reductions through `scratch` (double [B * 256], need not be initialised): bit-identical run to run. */
int cis_flow_standardize_bwd(const float* y, const float* dy, const double* stats, int32_t B, int64_t hw, double* scratch, float* dx,
                             cis_stream_t stream);
/* held-out end-point error of the recover net: for each sample b of pred, gt (fp32 [B,hw,2]) and mask (fp32 [B,hw]), with
 * e = ||pred - gt||_2 per pixel, out[b*4 + 0..3] = {sum m*e, sum (1-m)*e, sum m, sum (1-m)} in double.  Fixed-order reductions
 * through `scratch` (double [B * 256], need not be initialised), no atomics: bit-identical run to run.  out need not be zeroed. */
int cis_masked_epe(const float* pred, const float* gt, const float* mask, int32_t B, int64_t hw, double* scratch, double* out,
                   cis_stream_t stream);

/* ---- mask (x) flow + Charbonnier contextual-information loss (adversarial_learner.py:107-110,141-204) ---- */
/* recover inputs, batch 3B: [flow*(1-m),1,1-m | flow*m,1,m | 0,0,1,0] -> bf16 [3B,H,W,8] (nets.py:50-53) */
int cis_mask_apply(const float* flow, const float* mask, int32_t B, int64_t hw, void* dst, cis_stream_t stream);
/* box occlusions of the recover-net pretraining: mask fp32 [B,H,W,1] = 1 inside one box per sample, 0 elsewhere.  Sample b's box is four
 * counter-hash draws r_k = hash32(seed ^ D ^ t<<40 ^ g<<2 ^ k), k = 0..3, D = 0x426f784d61736b73, t = step[0] (device int64, read when the
 * kernel runs: the Adam step counter, so graph replays draw new boxes), g = sample_offset + b (the global sample index under data
 * parallelism), hash32 = the 64-bit MurmurHash3 finaliser truncated to 32 bits; all modulo operations unsigned 32-bit:
 * bh = lo_h + r0 % (hi_h-lo_h+1), bw = lo_w + r1 % (hi_w-lo_w+1), y0 = r2 % (H-bh+1), x0 = r3 % (W-bw+1); rows [y0, y0+bh), columns
 * [x0, x0+bw).  CIS_ERR_BAD_ARG unless 1 <= lo <= hi <= the image side (both axes), 1 <= B <= 65535, sample_offset >= 0. */
int cis_box_masks(float* mask, int32_t B, int32_t H, int32_t W, int32_t lo_h, int32_t hi_h, int32_t lo_w, int32_t hi_w, int64_t sample_offset,
                  const long long* step, uint64_t seed, cis_stream_t stream);
/* stand-alone charbonnier_loss (loss_utils.py:34-51): sums[b] += sum over pixels and C channels of ((gt-pred)^2 + 1e-6)^cbn * mask;
 * mask_c = 1 (one value per pixel) or C (one per element); sums = double [B], zeroed by the caller */
int cis_charbonnier_sum(const float* gt, const float* pred, const float* mask, int32_t B, int64_t hw, int32_t C, int32_t mask_c, float cbn,
                        double* sums, cis_stream_t stream);
/* sums[b] = {rec, rec_c, prior, den, den_c} (fp32 via double atomics; zeroed).  flow1 = fp32 [3B,H/2,W/2,2] recover
 * outputs before the final bilinear x2 (nets.py:108), which is fused here. */
int cis_cis_loss_fwd(const float* flow, const float* mask, const float* flow1, int32_t B, int32_t H, int32_t W, int32_t h1,
                     int32_t w1, float cbn, double* sums, float* pred_out /* optional [3B,H,W,2] */, cis_stream_t stream);
/* scalars[0]=generator loss, [1]=recover loss, [2]=red_rate, [3]=red_rate_compl, [4]=1/(H*W*global_batch);
 * coef[b*4..] = per-sample partial derivatives of the generator loss w.r.t. {rec, den, rec_c, den_c}.
 * global_batch = config.batch_size of the whole (data-parallel) job; losses are this rank's partial sums / global_batch. */
int cis_cis_loss_reduce(const double* sums, int32_t B, int32_t global_batch, int64_t hw, float epsilon, float* scalars, float* coef,
                        cis_stream_t stream);
/* which = 0: d recover_loss, 1: d generator_loss.  Writes dpred [3B,H,W,2] fp32 and (generator) the direct dL/dmask term. */
int cis_cis_loss_bwd(const float* flow, const float* mask, const float* flow1, const float* coef, const float* scalars, int32_t B,
                     int32_t H, int32_t W, int32_t h1, int32_t w1, float cbn, int32_t which, float* dpred, float* dmask,
                     cis_stream_t stream);
/* transpose of the final x2 resize: dflow1 [3B,h1,w1,2] -> bf16 [3B,h1,w1,8] gradient for the flow1 conv */
int cis_resize_f32_bwd_to_bf16(const float* ddst, int32_t N, int32_t OH, int32_t OW, int32_t C, int32_t H, int32_t W, void* dsrc,
                               int32_t s_pitch, cis_stream_t stream);
/* the same times `scale` (the final x4 of PWC-Net's flow, model_pwcnet.py:646) */
int cis_resize_f32_bwd_to_bf16_scaled(const float* ddst, int32_t N, int32_t OH, int32_t OW, int32_t C, int32_t H, int32_t W, void* dsrc,
                                      int32_t s_pitch, float scale, cis_stream_t stream);
/* mask backward: dmask += chain through the recover inputs (d_in bf16 [>=2B,H,W,8], gradient of cis_mask_apply's output);
 * then through softmax(x/10)[0] -> bf16 gradient of the 2 logits [B,H,W,8].  d_in = NULL skips the recover-input chain (flow may then
 * be NULL too): dlogits from dmask_direct alone, the stand-alone mask head of the function-level generator_net. */
int cis_mask_bwd(const float* flow, const float* mask, const float* dmask_direct, const void* d_in, int32_t B, int64_t hw,
                 void* dlogits, cis_stream_t stream);

/* ---- optimiser: clip / noise + TF-Adam (loss_utils.py:12-32, adversarial_learner.py:216-217) ---- */
/* stat[0] += sum|g| over [0,n)  (zeroed by caller); used for the can_change test */
int cis_abs_sum(const float* g, int64_t n, float* stat, cis_stream_t stream);
/* out_avg += mean over variables of mean|g_v| (loss_utils.py:19-20); seg = int64 [nseg][2] = {start,end} of each variable */
int cis_grad_avg_abs(const float* g, const int64_t* seg_off, int32_t nseg, float* out_avg, cis_stream_t stream);
/* step_state: device int64 {t}; advanced by this call.  can_change != 0 enables the noise branch on *avg_abs < 1e-5. */
int cis_clip_adam(float* param, float* m, float* v, const float* grad, int64_t n, float grad_scale, float clip, float lr, float beta1,
                  float beta2, float eps, int64_t* step_state, const float* avg_abs, int32_t can_change, uint64_t seed,
                  cis_stream_t stream);
int cis_cast_f32_to_bf16(const float* src, int64_t n, void* dst, cis_stream_t stream);
int cis_cast_bf16_to_f32(const void* src, int64_t npix, int32_t pitch, int32_t coff, int32_t C, float* dst, cis_stream_t stream);
/* dst[p][c] = scale * src[p][coff + c] (the sign of an input gradient read out of a bf16 gradient slice) */
int cis_cast_bf16_to_f32_scaled(const void* src, int64_t npix, int32_t pitch, int32_t coff, int32_t C, float scale, float* dst,
                                cis_stream_t stream);

/* ---- gradients of the stand-alone ops of the function-level API (models/functional.py; not used by the step graph) ---- */
/* charbonnier_loss backward (loss_utils.py:34-51): dsum = fp32 [B] upstream gradient of cis_charbonnier_sum's per-sample sums;
 * dpred = dsum * mask * d/dpred ((gt-pred)^2 + 1e-6)^cbn, dgt = -dpred, dmask = dsum * ((gt-pred)^2 + 1e-6)^cbn, summed over the
 * C channels of a pixel when mask_c = 1.  Any of dpred / dgt / dmask may be NULL.  No atomics. */
int cis_charbonnier_bwd(const float* gt, const float* pred, const float* mask, int32_t B, int64_t hw, int32_t C, int32_t mask_c, float cbn,
                        const float* dsum, float* dpred, float* dgt, float* dmask, cis_stream_t stream);
/* dense_image_warp backward (core_warp.py:42-202, clamping of SURVEY App. A.8) for the forward of cis_dense_image_warp; dout fp32
 * [B,h,w,C].  dflow (fp32 [B,h,w,2], or NULL) is per pixel: the floor carries no gradient, alpha = clip(q - floor, 0, 1) passes it
 * where 0 <= q - floor <= 1, q = grid - flow_scale * flow.  dimage (fp32 [B,h,w,C], or NULL) is a scatter: accumulated with fp64
 * atomics into `scratch` (double [B,h,w,C], zeroed by this call) and rounded to fp32 once -- order-dependent below 1e-15 relative. */
int cis_dense_image_warp_bwd(const void* img, int32_t pitch, int32_t coff, const float* flow, float flow_scale, int32_t B, int32_t h,
                             int32_t w, int32_t C, const float* dout, float* dimage, double* scratch, float* dflow, cis_stream_t stream);
/* cost_volume backward (core_costvol.py:20-40 as cis_warp_costvol evaluates it with flow = NULL): dout fp32 [B,h,w,81];
 * g'[p,d] = dout[p,d] * leaky0.1'(recomputed pre-activation) goes to gscratch (fp32 [B,h,w,81]), then
 * dc1[p] = sum_d g'[p,d] warp[p+d] / C and dwarp[q] = sum_d g'[q-d,d] c1[q-d] / C (fp32 [B,h,w,C]), displacements that leave the map
 * contributing nothing.  Both are gathers over shared-memory halo tiles: no atomics, bit-reproducible. */
int cis_cost_volume_bwd(const void* c1, int32_t c1_pitch, int32_t c1_coff, const void* warp, int32_t warp_pitch, int32_t warp_coff,
                        const float* dout, int32_t B, int32_t h, int32_t w, int32_t C, float* gscratch, float* dc1, float* dwarp,
                        cis_stream_t stream);
/* the same for search range 1..4: dout and gscratch are fp32 [B,h,w,(2r+1)^2] (CIS_ERR_BAD_ARG outside 1..4) */
int cis_cost_volume_bwd_r(const void* c1, int32_t c1_pitch, int32_t c1_coff, const void* warp, int32_t warp_pitch, int32_t warp_coff,
                          const float* dout, int32_t B, int32_t h, int32_t w, int32_t C, float* gscratch, float* dc1, float* dwarp,
                          int32_t search_range, cis_stream_t stream);

/* ---- PWC-Net backward (function-level predict_from_img_pairs; the step graph keeps PWC-Net frozen) ---- */
/* Transpose of cis_warp_costvol, same feature operands (c1, c2, flow, flow_scale; flow = NULL at level 6).  dcorr = bf16 gradient of the 81
 * correlation channels (dcorr[p * dc_pitch + dc_coff + d]).  Results, bf16 slices, each overwritten or accumulated into (accumulate bit 0:
 * dc1, bit 1: dc2, bit 2: dflow): dc1 and dwarp are the gathers of cis_cost_volume_bwd, with the warped c2 recomputed in the shared-memory
 * halo tiles as the forward does; with a flow, dc2 is the scatter of cis_dense_image_warp_bwd (fp64 atomics into dscratch, rounded
 * once) and dflow = d(flow) (the flow_scale factor included, inclusive clip rule of core_warp.py) goes to channels 0-1 of its slice.
 * Scratch: gscratch fp32 [B,h,w,81]; with a flow, wscratch fp32 [B,h,w,C] (dwarp) and dscratch double [B,h,w,C] (zeroed here). */
int cis_warp_costvol_bwd(const void* c1, int32_t c1_pitch, int32_t c1_coff, const void* c2, int32_t c2_pitch, int32_t c2_coff, const float* flow,
                         float flow_scale, int32_t B, int32_t h, int32_t w, int32_t C, const void* dcorr, int32_t dc_pitch, int32_t dc_coff,
                         void* dc1, int32_t dc1_pitch, int32_t dc1_coff, void* dc2, int32_t dc2_pitch, int32_t dc2_coff, void* dflow,
                         int32_t dflow_pitch, int32_t dflow_coff, int32_t accumulate, float* gscratch, float* wscratch, double* dscratch,
                         cis_stream_t stream);
/* the same for search range 1..4: dcorr holds (2r+1)^2 channels and gscratch is fp32 [B,h,w,(2r+1)^2] (CIS_ERR_BAD_ARG outside 1..4) */
int cis_warp_costvol_bwd_r(const void* c1, int32_t c1_pitch, int32_t c1_coff, const void* c2, int32_t c2_pitch, int32_t c2_coff,
                           const float* flow, float flow_scale, int32_t B, int32_t h, int32_t w, int32_t C, const void* dcorr,
                           int32_t dc_pitch, int32_t dc_coff, void* dc1, int32_t dc1_pitch, int32_t dc1_coff, void* dc2, int32_t dc2_pitch,
                           int32_t dc2_coff, void* dflow, int32_t dflow_pitch, int32_t dflow_coff, int32_t accumulate, float* gscratch,
                           float* wscratch, double* dscratch, int32_t search_range, cis_stream_t stream);
/* dst plane a*2+b [N,H,W,d_pitch] (one zero-padded 8-channel chunk per pixel) = src(n, 2y+a, 2x+b, s_coff .. s_coff+C), C <= 8, s_coff any:
 * the output-parity gradient operands of the weight gradient of conv2d_transpose(k4, s2) */
int cis_parity_split_bf16(const void* src, int32_t s_pitch, int32_t s_coff, int32_t N, int32_t H, int32_t W, int32_t C, void* dst,
                          int32_t d_pitch, cis_stream_t stream);

/* ---- PWC-Net training (tfoptflow's multi-scale objective, as defined in DESIGN.md: not checked against TensorFlow) ----
 * Level i = 0..4 is pyramid level l = 6 - i: flow[i] = the refined fp32 flow [B, H >> l, W >> l, 2] of the network at input size H x W;
 * grad[i] = the bf16 gradient of that level's flow Act (element (pixel, c) at grad[i][pixel * pitch[i] + c_off[i] + c], c = 0, 1),
 * overwritten or, with accumulate[i], added to; weight[i] = the backward's factor alpha_l / global batch. */
typedef struct {
  const float* flow[5];
  void* grad[5];
  int32_t pitch[5];
  int32_t c_off[5];
  int32_t accumulate[5];
  float weight[5];
} CisFlowPyr;
/* gt = fp32 [B, GH, GW, 2], the ground-truth flow in PWC-Net's channel order.  Target of level l: g_l = R_l(gt) * (s_c / 2^l) for channel
 * c, R_l = the legacy bilinear resize to the level's size (cis_resize_bilinear_f32's rule), sampled on the fly; s0, s1 = the vectors' scale
 * from the gt grid to the input grid (1 when GH x GW = H x W).  rho(d), d = flow_l - g_l: robust = 0: ||d||_2; robust = 1:
 * (|d0| + |d1| + eps)^q.  out = double [B, 5]: out[b * 5 + i] = sum over level i's pixels of sample b of rho.  The sums are double,
 * reduced in a fixed order through scratch (double [5 * B * 64], need not be initialised), no atomics: bit-identical run to run.
 * gt and flow[0..4] are read as pairs of floats and must be 8-byte aligned (a tensor's base address is).
 * CIS_ERR_BAD_ARG unless H and W are multiples of 64, 1 <= B <= 65535, GH, GW >= 1, and the alignment holds. */
int cis_flow_multiscale_loss(const CisFlowPyr* pyr, const float* gt, int32_t B, int32_t H, int32_t W, int32_t GH, int32_t GW, float s0,
                             float s1, int32_t robust, float eps, float q, double* scratch, double* out, cis_stream_t stream);
/* its backward, all five levels in one launch: grad[i] (=|+=) weight[i] * d rho / d flow_l per pixel.  The gradient of ||d||_2 is
 * d / ||d||_2, and 0 at d = 0; that of |d_c| is sign(d_c), 0 at d_c = 0. */
int cis_flow_multiscale_loss_bwd(const CisFlowPyr* pyr, const float* gt, int32_t B, int32_t H, int32_t W, int32_t GH, int32_t GW, float s0,
                                 float s1, int32_t robust, float eps, float q, cis_stream_t stream);
/* TF-Adam with L2 weight decay, no clip: g' = grad + decay * param inside the segments seg = int64 [nseg][2] {start, end} (device,
 * sorted and disjoint: the kernel variables), g' = grad elsewhere; then cis_clip_adam's update (lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t),
 * t = step_state[0] + 1) over [0, n).  lr = device float [1], read when the kernel runs (a rate schedule needs no re-capture).
 * step_state is advanced by this call. */
int cis_adam_l2(float* param, float* m, float* v, const float* grad, int64_t n, const int64_t* seg, int32_t nseg, float decay, const float* lr,
                float beta1, float beta2, float eps, int64_t* step_state, cis_stream_t stream);

/* ---- exponential moving average of the weights (tf.train.ExponentialMovingAverage(decay, num_updates=t)) ----
 * t = step_state[0], read when the kernel runs: the step counter the optimiser launch just before this one (cis_clip_adam /
 * cis_adam_l2) advanced, so CUDA-graph replays need no host.  d = min(decay, (1 + t) / (10 + t)) in fp64, rounded once to fp32; then
 * over [0, n): shadow = shadow - (shadow - param) * (1 - d), each fp32 operation rounded on its own (no FMA), bit-identical to the
 * same three numpy fp32 operations.  Padding entries included: zeros in both stay zero.  CIS_ERR_BAD_ARG for a NULL buffer, n < 1 or a
 * decay outside (0, 1). */
int cis_ema_update(float* shadow, const float* param, int64_t n, float decay, const int64_t* step_state, cis_stream_t stream);

/* ---- Unsupervised fine-tuning of PWC-Net (occlusion-masked census + second-order smoothness, restated from UnFlow's published
 * recipe as defined in DESIGN.md: not checked against any other implementation) ----
 * img1, img2 = fp32 RGB [B, H, W, 3] in [-0.5, 0.5]; flow = fp32 [2B, H, W, 2] in PWC-Net's order and sign, pixels of H x W: direction
 * n < B is the pair (img1[n], img2[n]), n >= B the swapped pair (img2[n-B], img1[n-B]); S / T = its first / second frame, n' = n -+ B its
 * partner direction.  Per pixel p = (y, x) of direction n, with F = flow[n]:
 *   g(I) = 255 (0.2989 R + 0.5870 G + 0.1140 B) of I + 0.5;  q = (y - F0, x - F1);  T~(p) = g(T) sampled at q by dense_image_warp's rule
 *   (floor clamped to [0, size-2], alpha = clip(q - floor, 0, 1));  V = [0 <= q_y <= H-1 and 0 <= q_x <= W-1];  F^ = flow[n'] sampled at q
 *   by the same rule;  O = [|F + F^|^2 > 0.01 (|F|^2 + |F^|^2) + 0.5];  M = V (1 - O), which carries no gradient.
 *   Census over the offsets d != 0 of the 7x7 window with p + d inside the frame: t_X = v / sqrt(0.81 + v^2), v = X(p+d) - X(p), for X =
 *   g(S) and X = T~;  c = sum_d e^2 / (0.1 + e^2), e = t_S - t_T~;  psi = (c + 0.01)^0.4.
 *   Smoothness, for each axis a with p +- e_a inside the frame: s_a = sum_c |l_c|, l_c = F_c(p+e_a) - 2 F_c(p) + F_c(p-e_a) (gradient of
 *   |.|: sign, 0 at 0), where l_c counts as 0 when |l_c| <= 2^-18 (|F_c(p+e_a)| + 2 |F_c(p)| + |F_c(p-e_a)|), the rounding level of fp32
 *   flows; w_a = exp(-10 * mean over RGB of |S(p+e_a) - S(p-e_a)| / 2).
 * out = double [2B, 2]: out[n] = {sum_p M psi, sum_p sum_a w_a s_a}; the sums are double, reduced in a fixed order through scratch
 * (double [2 * 2B * 64], need not be initialised), no atomics: bit-identical run to run.  Per-pixel buffers for the backward, fp32
 * [2B, H, W]: warped = T~, mask = M, coef = M psi'(c).  Three launches: warp + mask, census + smoothness with block partials, reduction.
 * flow is read as pairs of floats and must be 8-byte aligned.  CIS_ERR_BAD_ARG unless 1 <= B <= 65535, H, W >= 3 and the alignment holds. */
int cis_unsup_flow_loss(const float* flow, const float* img1, const float* img2, int32_t B, int32_t H, int32_t W, float* warped, float* mask,
                        float* coef, double* scratch, double* out, cis_stream_t stream);
/* its backward, one launch: dflow = fp32 [2B, H, W, 2] (overwritten, 8-byte aligned) = w_photo * d(sum_p M psi) / dF + w_smooth *
 * d(sum_p sum_a w_a s_a) / dF, each direction's own flow only (M and F^ carry no gradient).  The census term is a gather: T~(r) collects
 * coef * dc / dT~(r) from the <= 49 windows holding r, then dense_image_warp's dflow rule (alpha passes it where 0 <= q - floor <= 1);
 * the smoothness term is a 5-point gather.  No atomics.  warped / coef: the forward's buffers.  Same argument checks as the forward. */
int cis_unsup_flow_loss_bwd(const float* flow, const float* img1, const float* img2, int32_t B, int32_t H, int32_t W, const float* warped,
                            const float* coef, float w_photo, float w_smooth, float* dflow, cis_stream_t stream);

/* ---- Geometric + photometric augmentation of supervised PWC-Net training pairs (restated from the FlowNet / PWC-Net papers'
 * description, as defined in DESIGN.md; the ranges are chosen here and not checked against any other implementation) ----
 * Pixel centres are at integer (x, y) of the H x W grid, c = ((W-1)/2, (H-1)/2), R(th) = [[cos th, -sin th], [sin th, cos th]] on (x, y).
 * Frame 1 and the ground truth sample their source at T1(p) = c + t + R(th)(p - c)/s; frame 2 at T2 = T1 o Tr, Tr(p) = c + t_r +
 * R(th_r)(p - c)/s_r.  Every range below is [lo, hi], drawn uniformly; angles in degrees; translations as fractions of (W, H). */
typedef struct {
  float scale[2];          /* s                      default [0.9, 2.0] */
  float rotate[2];         /* th                     default [-17, 17] */
  float translate[2];      /* t = (u W, u' H)        default [-0.2, 0.2] */
  float rel_scale[2];      /* s_r                    default [0.95, 1.05] */
  float rel_rotate[2];     /* th_r                   default [-3, 3] */
  float rel_translate[2];  /* t_r = (u W, u' H)      default [-0.03, 0.03] */
  float color[2];          /* m_c, log-uniform       default [0.5, 2] */
  float contrast[2];       /* kappa                  default [-0.8, 0.4] */
  float brightness;        /* std of beta ~ N(0, .)  default 0.2 */
  float gamma[2];          /* gamma                  default [0.7, 1.5] */
  float noise[2];          /* sigma                  default [0, 0.04] */
} CisFlowAug;
#define CIS_FLOW_AUG_ROW 32
/* Per-sample parameters: params = fp32 [B, CIS_FLOW_AUG_ROW], row b for the global sample g = sample_offset + b at step t = step[0]
 * (device int64, read when the kernel runs: the Adam step counter, so CUDA-graph replays draw new parameters; data-parallel ranks with
 * sample_offset = rank * local batch draw what one GPU running the global batch draws).  Draw k is r_k = hash32(seed ^ D ^ t<<40 ^ g<<10 ^
 * k), D = 0x466c6f774175676d, hash32 = the 64-bit MurmurHash3 finaliser truncated to 32 bits (cis_box_masks'), U_k = (r_k + 0.5) / 2^32.
 * Geometry attempt a = 0..63 draws k = 8a + j: j = 0 s, 1 th, 2 t_x, 3 t_y, 4 s_r, 5 th_r, 6 t_r.x, 7 t_r.y (lo + (hi - lo) U_k, in
 * double).  It is accepted when the four corners (0,0), (W-1,0), (0,H-1), (W-1,H-1) map under T1 and under T2 into [0, W-1] x [0, H-1]
 * (tested in double); the first accepted attempt is used, and after 64 rejections the identity.  Photometric draws k = 512 + j: j = 0..2
 * m_c = exp(ln lo + (ln hi - ln lo) U_k), 3 kappa, 4 and 5 beta = brightness sqrt(-2 ln U_516) cos(2 pi U_517), 6 gamma, 7 sigma, 8 the
 * noise key r_520.  Row layout (each affine map as (r0, r1, r2, r3, r4, r5): q = (r0 x + r1 y + r2, r3 x + r4 y + r5), formed in double
 * and rounded): [0, 6) T1, [6, 12) T2, [12, 18) T2^-1, [18, 21) m_c, 21 1 + kappa, 22 beta, 23 gamma, 24 sigma, 25 the noise key (uint32
 * bits), 26 the accepted attempt (64 = identity), [27, 32) 0.  One thread per sample, no atomics.  CIS_ERR_BAD_ARG unless 1 <= B <= 65535,
 * H, W >= 2, sample_offset >= 0, the buffers are non-null and every range has lo <= hi with scale, rel_scale and color lo > 0. */
int cis_flow_aug_params(const CisFlowAug* ranges, int32_t B, int32_t H, int32_t W, int64_t sample_offset, const long long* step,
                        uint64_t seed, float* params, cis_stream_t stream);
/* The augmented pair and flow, one pass, one thread per output pixel p of each sample: img1, img2 = fp32 RGB [B, H, W, 3] in [-0.5, 0.5],
 * gt = fp32 [B, H, W, 2] in PWC-Net's order (ch0 = -v, ch1 = -u).  Samples use dense_image_warp's bilinear rule (floor clamped to
 * [0, size-2], fraction clamped to [0, 1]).  img1_out(p) = phot(img1 at T1(p)), img2_out(p) = phot(img2 at T2(p)); flow: q = T1(p), (u, v)
 * = gt at q (converted from PWC-Net's order), p2 = T2^-1(q + (u, v)), gt_out(p) = p2 - p in PWC-Net's order.  phot, on v = sample + 0.5
 * per channel c: v *= m_c; v = 0.5 + (1 + kappa)(v - 0.5); v += beta; v = clamp(v, 0, 1)^gamma; v = clamp(v + sigma n, 0, 1); out = v -
 * 0.5, n = sqrt(-2 ln U1) cos(2 pi U2), U1 = (hash32(N ^ key<<32 ^ 2i) + 0.5) / 2^32, U2 the same with 2i + 1, N = 0x4175674e6f697365,
 * i = ((f H + y) W + x) 3 + c, f = 0 for frame 1 and 1 for frame 2 (sigma = 0 skips n).  gt and gt_out are read / written as float pairs and must be 8-byte
 * aligned; the outputs must not alias the inputs.  CIS_ERR_BAD_ARG unless 1 <= B <= 65535, H, W >= 2, 6 H W < 2^31, the buffers are
 * non-null and the alignment holds. */
int cis_flow_augment(const float* img1, const float* img2, const float* gt, const float* params, int32_t B, int32_t H, int32_t W,
                     float* img1_out, float* img2_out, float* gt_out, cis_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* CIS_B200_H_ */
