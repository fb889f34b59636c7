/* daala_b200.h -- C ABI of libdaala_b200.so: an H100 (sm_90a) implementation of
 * the per-block encode hot path of xiph/daala.
 *
 * Two families of entry points:
 *
 * (1) DROP-IN SYMBOLS (section A): the reference's own od_* names and
 *     prototypes, taking HOST pointers, synchronous, individually bit-exact.
 *     They are what daalaenc/daaladec (or the od_state_opt_vtbl /
 *     od_enc_opt_vtbl slots, reference src/state.h:112-131, src/encint.h:77-98)
 *     bind to; INTEGRATION.md shows the vtable initialiser a maintainer adds.
 *     Each call stages its operands through pinned memory and launches a
 *     kernel, so they are functional, not fast.
 *
 * (2) BATCH ENTRY POINTS (section B, daala_b200_*): DEVICE pointers + a CUDA
 *     stream; whole frames per launch.  This is the throughput path that the
 *     host driver (daala_b200/ Python mirror, or a batching shim inside
 *     libdaalaenc) uses.  All return 0 on success or a cudaError_t value.
 *
 * There is no CPU fallback: if no CUDA device is usable the drop-in symbols
 * abort() with a message (the reference's hot-path functions return void and
 * cannot report errors; cf. od_fatal_impl, src/internal.c:394) and the batch
 * entry points return the CUDA error.
 */
#ifndef DAALA_B200_H
#define DAALA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int32_t od_coeff; /* reference: src/filter.h:29 */

/* ======================================================================== */
/* A. Drop-in symbols (host pointers)                                        */
/* ======================================================================== */

/* 1-D reversible integer DCT-II / inverse.  reference: src/dct.h:70-183,
   definitions src/dct.c:87,127,166,286,366,659,4219,4321,4422,4622. */
void od_bin_fdct4(od_coeff y[4], const od_coeff *x, int xstride);
void od_bin_idct4(od_coeff *x, int xstride, const od_coeff y[4]);
void od_bin_fdct8(od_coeff y[8], const od_coeff *x, int xstride);
void od_bin_idct8(od_coeff *x, int xstride, const od_coeff y[8]);
void od_bin_fdct16(od_coeff y[16], const od_coeff *x, int xstride);
void od_bin_idct16(od_coeff *x, int xstride, const od_coeff y[16]);
void od_bin_fdct32(od_coeff y[32], const od_coeff *x, int xstride);
void od_bin_idct32(od_coeff *x, int xstride, const od_coeff y[32]);
void od_bin_fdct64(od_coeff y[64], const od_coeff *x, int xstride);
void od_bin_idct64(od_coeff *x, int xstride, const od_coeff y[64]);

/* 2-D separable transforms = the od_dct_func_2d slots fdct_2d[]/idct_2d[] of
   od_state_opt_vtbl.  reference: src/dct.c:151,158,351,358,792,800,4890-4920;
   typedef src/dct.h:62-63. */
void od_bin_fdct4x4(od_coeff *y, int ystride, const od_coeff *x, int xstride);
void od_bin_idct4x4(od_coeff *x, int xstride, const od_coeff *y, int ystride);
void od_bin_fdct8x8(od_coeff *y, int ystride, const od_coeff *x, int xstride);
void od_bin_idct8x8(od_coeff *x, int xstride, const od_coeff *y, int ystride);
void od_bin_fdct16x16(od_coeff *y, int ystride, const od_coeff *x, int xstride);
void od_bin_idct16x16(od_coeff *x, int xstride, const od_coeff *y, int ystride);
void od_bin_fdct32x32(od_coeff *y, int ystride, const od_coeff *x, int xstride);
void od_bin_idct32x32(od_coeff *x, int xstride, const od_coeff *y, int ystride);
void od_bin_fdct64x64(od_coeff *y, int ystride, const od_coeff *x, int xstride);
void od_bin_idct64x64(od_coeff *x, int xstride, const od_coeff *y, int ystride);
/* src/dct.c:4822 / :4861 (prototypes src/dct.h): the multi-level Haar wavelet of the lossless path, n = 1 << ln */
/* TF resolution switching, reference src/tf.h:47-67 / src/tf.c:38-277 (csrc/tf_kernels.cu).  Blocks up to
   64x64; dst may alias src where the reference allows it. */
void od_tf_up_h_lp(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int dx, int n);
void od_tf_up_v_lp(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int dy, int n);
void od_tf_up_hv_lp(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int dx, int dy, int n);
void od_tf_up_hv(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int n);
void od_tf_down_hv(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int n);
void od_convert_block_down(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int curr_size,
                           int dest_size, int filter);
void od_tf_filter_2d(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int n);
void od_tf_filter_inv_2d(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int n);

void od_haar(od_coeff *y, int ystride, const od_coeff *x, int xstride, int ln);
void od_haar_inv(od_coeff *x, int xstride, const od_coeff *y, int ystride, int ln);

typedef void (*od_dct_func_2d)(od_coeff *out, int out_stride, const od_coeff *in, int in_stride);
/* reference: OD_FDCT_2D_C / OD_IDCT_2D_C, src/dct.c:54-68 (last entry NULL). */
extern const od_dct_func_2d OD_FDCT_2D_CUDA[6];
extern const od_dct_func_2d OD_IDCT_2D_CUDA[6];

/* The same tables under the reference's own names (src/dct.c:54-84; src/dct.h:62-75), for builds that
   link this library in place of the reference's dct.o. */
typedef void (*od_fdct_func_1d)(od_coeff *out, const od_coeff *in, int in_stride);
typedef void (*od_idct_func_1d)(od_coeff *out, int out_stride, const od_coeff *in);
extern const od_dct_func_2d OD_FDCT_2D_C[6];
extern const od_dct_func_2d OD_IDCT_2D_C[6];
extern const od_fdct_func_1d OD_FDCT_1D[6];
extern const od_idct_func_1d OD_IDCT_1D[6];

/* 4-point lapped pre/post filter and its appliers.
   reference: src/filter.h:44-87, definitions src/filter.c:147,195,1459,1485,
   1529,1561. */
void od_pre_filter4(od_coeff _y[4], const od_coeff _x[4]);
void od_post_filter4(od_coeff _x[4], const od_coeff _y[4]);
/* The larger lapping filters (dead in the codec, OD_FILT_SIZE() == 0, but exported by the
   reference and used by its dcttest / tools): src/filter.c:279,366,519,678,852,1146. */
void od_pre_filter8(od_coeff _y[8], const od_coeff _x[8]);
void od_post_filter8(od_coeff _x[8], const od_coeff _y[8]);
void od_pre_filter16(od_coeff _y[16], const od_coeff _x[16]);
void od_post_filter16(od_coeff _x[16], const od_coeff _y[16]);
void od_pre_filter32(od_coeff _y[32], const od_coeff _x[32]);
void od_post_filter32(od_coeff _x[32], const od_coeff _y[32]);
typedef void (*od_filter_func)(od_coeff _out[], const od_coeff _in[]);
extern const od_filter_func OD_PRE_FILTER_CUDA[4];   /* OD_PRE_FILTER, src/filter.c:115 */
extern const od_filter_func OD_POST_FILTER_CUDA[4];  /* OD_POST_FILTER, src/filter.c:122 */
extern const od_filter_func OD_PRE_FILTER[5];        /* the reference's names, src/filter.h:45-46 */
extern const od_filter_func OD_POST_FILTER[5];
extern const int OD_FILTER_PARAMS4[4];               /* src/filter.c:142 */
void od_prefilter_split(od_coeff *c0, int stride, int bs, int f, int hfilter, int vfilter);
void od_postfilter_split(od_coeff *c0, int stride, int bs, int f, int q, unsigned char *skip,
                         int skip_stride, int hfilter, int vfilter);
void od_apply_prefilter_frame_sbs(od_coeff *c, int stride, int nhsb, int nvsb, int xdec, int ydec);
void od_apply_postfilter_frame_sbs(od_coeff *c, int stride, int nhsb, int nvsb, int xdec, int ydec,
                                   int q, unsigned char *skip, int skip_stride);

/* PVQ helpers shared by encoder and decoder (src/pvq.h:148-175; definitions src/pvq.c:428-1115)
   and the scalar RDO quantiser (src/pvq_encoder.c:730).  Each call is one single-thread launch of
   the same device functions the batch kernels use: exact, and only meant for ABI completeness. */
int16_t od_pvq_sin(int32_t x);
int16_t od_pvq_cos(int32_t x);
int od_vector_log_mag(const od_coeff *x, int n);
int od_compute_householder(int16_t *r, int n, int32_t gr, int *sign, int shift);
void od_apply_householder(int16_t *out, const int16_t *x, const int16_t *r, int n);
void od_pvq_synthesis_partial(od_coeff *xcoeff, const od_coeff *ypulse, const int16_t *r, int n, int noref,
                              int32_t g, int32_t theta, int m, int s, const int16_t *qm_inv);
int32_t od_gain_expand(int32_t cg, int q0, int16_t beta);
int32_t od_pvq_compute_gain(const int16_t *x, int n, int q0, int32_t *g, int16_t beta, int bshift);
int od_pvq_compute_max_theta(int32_t qcg, int16_t beta);
int32_t od_pvq_compute_theta(int t, int max_theta);
int od_pvq_compute_k(int32_t qcg, int itheta, int32_t theta, int noref, int n, int16_t beta, int nodesync);
int od_rdo_quant(od_coeff x, int q, double delta0, double pvq_norm_lambda);

/* Motion-compensation and block-matching slots of od_state_opt_vtbl
   (src/state.h:113-121) and od_enc_opt_vtbl (src/encint.h:77-98).  The names
   carry a _cuda suffix because the reference's C kernels keep their _c names in
   the same link; the vtable initialiser of INTEGRATION.md installs them.
   `state` is unused (the reference only reads its od_copy_nxn table). */
void od_mc_predict1fmv8_cuda(void *state, unsigned char *dst, const unsigned char *src, int systride,
                             int32_t mvx, int32_t mvy, int log_xblk_sz, int log_yblk_sz);
void od_mc_blend_full8_cuda(unsigned char *dst, int dystride, const unsigned char *src[4],
                            int log_xblk_sz, int log_yblk_sz);
void od_mc_blend_full_split8_cuda(unsigned char *dst, int dystride, const unsigned char *src[4], int c,
                                  int s, int log_xblk_sz, int log_yblk_sz);
int32_t od_mc_compute_sad8_4x4_cuda(const unsigned char *src, int systride, const unsigned char *ref, int dystride);
int32_t od_mc_compute_sad8_8x8_cuda(const unsigned char *src, int systride, const unsigned char *ref, int dystride);
int32_t od_mc_compute_sad8_16x16_cuda(const unsigned char *src, int systride, const unsigned char *ref, int dystride);
int32_t od_mc_compute_sad8_32x32_cuda(const unsigned char *src, int systride, const unsigned char *ref, int dystride);
int32_t od_mc_compute_sad8_64x64_cuda(const unsigned char *src, int systride, const unsigned char *ref, int dystride);
int32_t od_mc_compute_satd8_4x4_cuda(const unsigned char *src, int systride, const unsigned char *ref, int dystride);
int32_t od_mc_compute_satd8_8x8_cuda(const unsigned char *src, int systride, const unsigned char *ref, int dystride);
int32_t od_mc_compute_satd8_16x16_cuda(const unsigned char *src, int systride, const unsigned char *ref, int dystride);
int32_t od_mc_compute_satd8_32x32_cuda(const unsigned char *src, int systride, const unsigned char *ref, int dystride);
int32_t od_mc_compute_satd8_64x64_cuda(const unsigned char *src, int systride, const unsigned char *ref, int dystride);

/* ======================================================================== */
/* B. Batch entry points (device pointers, asynchronous on `stream`)         */
/* ======================================================================== */

/* One plane of a frame resident in HBM; plane size is implied by the frame
   geometry ((nhsb*64) >> xdec) x ((nvsb*64) >> xdec). */
typedef struct daala_b200_plane {
  const uint8_t *pixels;   /* forward input (u8) */
  int32_t *coeffs;         /* forward output / inverse input: the `d` plane, blocks in place */
  int32_t *lapped;         /* inverse intermediate: `c` plane before the superblock postfilter */
  uint8_t *pixels_out;     /* inverse output (u8) */
  int pixel_stride;
  int coeff_stride;
  int lapped_stride;
  int pixel_out_stride;
  int xdec;                /* xdec == ydec: 0 or 1 */
  int pad_;
  /* Elements between consecutive frames of a batch in each buffer (0 when nframes == 1). */
  long long pixel_frame_pitch;
  long long coeff_frame_pitch;
  long long lapped_frame_pitch;
  long long pixel_out_frame_pitch;
} daala_b200_plane;

typedef struct daala_b200_frame {
  daala_b200_plane plane[3];
  const uint8_t *bsize;    /* device copy of state->bsize: one byte (0..4) per 8x8 luma unit */
  int bstride;
  int nhsb, nvsb;
  int pic_w, pic_h;        /* luma picture size (info.pic_width/pic_height) */
  int haar_dc;             /* 1 on keyframes: DC Haar pyramid of od_compute_dcts */
  int nframes;             /* frames in the batch (>= 1); same geometry, independent content */
  int sb_row0, sb_rows;    /* superblock rows [sb_row0, sb_row0 + sb_rows) are processed: the
                              multi-GPU shard of this rank; whole frame = 0, nvsb */
  int pad_;
  long long bsize_frame_pitch;
  /* Optional: when post16[p] is set, daala_b200_sb_postfilter_store_frame writes plane p after the superblock
     postfilter as int16 (the reference's etmp, input of od_dering) with the geometry of pixels_out, INSTEAD of
     the clamped 8-bit pixels. */
  int16_t *post16[3];
} daala_b200_frame;

/* u8 planes -> coefficient planes: od_ref_plane_to_coeff (src/state.c:1259) +
   od_apply_prefilter_frame_sbs (src/filter.c:1529) + od_compute_dcts
   (src/encode.c:1455) for every superblock of every plane, one launch. */
int daala_b200_forward_frame(const daala_b200_frame *f, int nplanes, void *stream);
/* Same result with the input window fetched by plain loads instead of TMA
   (automatically used when a plane is not 16-byte aligned; exported as a test hook). */
int daala_b200_forward_frame_no_tma(const daala_b200_frame *f, int nplanes, void *stream);

/* coefficient planes -> u8 planes: per-leaf idct_2d (src/encode.c:1397) +
   od_postfilter_split (src/filter.c:1485) bottom-up, then
   od_apply_postfilter_frame_sbs (src/filter.c:1561) + od_coeff_to_ref_plane
   (src/state.c:1323).  Two launches. */
int daala_b200_inverse_frame(const daala_b200_frame *f, int nplanes, void *stream);
/* First half only (writes plane[].lapped). */
int daala_b200_inverse_frame_lapped(const daala_b200_frame *f, int nplanes, void *stream);

/* Second half only (reads plane[].lapped incl. 2 rows of halo around the
   processed superblock rows, writes plane[].pixels_out).  A multi-GPU rank calls
   _lapped, exchanges the border rows with its neighbours, then this. */
int daala_b200_sb_postfilter_store_frame(const daala_b200_frame *f, int nplanes, void *stream);

/* In-place superblock-edge filters of one int32 plane on the device. */
int daala_b200_plane_sb_filter(int32_t *c, int stride, int nhsb, int nvsb, int xdec, int ydec,
                               int post, void *stream);

/* `count` contiguous groups of n (4, 8, 16 or 32) ints through the n-point pre (post = 0) or
   post filter, in place. */
int daala_b200_lapfilter(int32_t *v, long count, int n, int post, void *stream);
/* `count` packed (1<<ln)^2 blocks (ln = 1..6) through od_haar (inverse = 0) or od_haar_inv (1), in place. */
int daala_b200_haar_blocks(int32_t *blocks, int count, int ln, int inverse, void *stream);
/* `count` packed (1<<ln)^2 blocks, contiguous, transformed in place.
   mode 0/1: 2-D forward/inverse; mode 2/3: every row as a 1-D forward/inverse. */
int daala_b200_block_transform(int32_t *blocks, int count, int ln, int mode, void *stream);

/* ---- PVQ (perceptual vector quantisation) --------------------------------- */

/* One transform block of the PVQ batch. */
typedef struct daala_b200_pvq_block {
  int32_t coef_off;        /* offset of this block's coding-order vector in in/ref/out/y;
                              the vector holds n^2 (n <= 16) or 512 (n >= 32) coefficients */
  uint16_t x0, y0;         /* top-left sample of the block inside its plane */
  uint8_t bs;              /* log2(n) - 2: 0..4 */
  uint8_t pli;             /* plane index */
  uint8_t xdec;            /* plane decimation (selects the 4:2:0 half of the QM tables) */
  uint8_t frame;           /* frame of the batch this block belongs to */
} daala_b200_pvq_block;

/* All pointers are device pointers.  Result arrays are indexed [block*9 + band]
   (PVQ_MAX_PARTITIONS = 9, reference src/pvq.h:38) or [block]. */
typedef struct daala_b200_pvq_params {
  const daala_b200_pvq_block *blocks;
  int32_t *in;             /* dblock: coefficients in coding order (od_raster_to_coding_order) */
  int32_t *ref;            /* predt: prediction in coding order; negated in place by the CfL flip */
  int32_t *out;            /* scalar_out: de-quantised coefficients in coding order */
  int32_t *y;              /* PVQ pulse vectors (what the entropy coder codes) */
  int32_t *res_gain;       /* coded gain index per band: pvq_theta's return value */
  int32_t *res_theta;      /* itheta per band (-1: no reference) */
  int32_t *res_max_theta;
  int32_t *res_k;          /* pulses per band */
  double *res_skip_term;   /* per band: skip_dist - best_dist */
  double *res_skip_diff;   /* per block: ordered sum of the terms above */
  int32_t *res_flip;       /* per block: CfL flip flag */
  int32_t *res_dc;         /* per block: scalar-quantised DC index (inter frames) */
  int16_t *y16;            /* optional (may be NULL): the pulse vectors again, packed to 16 bits by the
                              scatter kernels -- the form copied back to the host entropy coder */
  const int16_t *qm;       /* state->qm: od_init_qm, src/pvq.c:322 (2*qm_stride entries) */
  const int16_t *qm_inv;
  int32_t *coef_plane[3];  /* `d` planes (raster): gather source / scatter destination */
  const int32_t *pred_plane[3]; /* `md` planes or NULL (prediction = 0) */
  long long plane_frame_pitch[3];
  int plane_stride[3];
  int qm_stride;           /* OD_QM_STRIDE = 5456 */
  int q0;                  /* max(1, state->quantizer) */
  int is_keyframe;
  int use_masking;         /* activity masking: beta = 1.5 on luma blocks > 4x4 */
  int pad_;
  double pvq_norm_lambda;  /* enc->pvq_norm_lambda */
  uint8_t pvq_qm_q4[3][32];/* state->pvq_qm_q4[pli][OD_QM_SIZE = 30] */
} daala_b200_pvq_params;

/* Per-band search + synthesis (pvq_theta, src/pvq_encoder.c:333, speed > 0 rate
   model) for `count` bands listed as (block << 4 | band); nmax = 16, 32 or 128
   bounds the band size of this list (bands are launched per size class). */
int daala_b200_pvq_encode_bands(const daala_b200_pvq_params *prm, const uint32_t *band_list, int count,
                                int nmax, void *stream);
/* Same with an explicit kernel choice: mode 0 = the measured-best mix (scalar
   thread-per-band kernels for n <= 32, one warp = 32 lanes x 4 registers per
   band for n = 128), 1 = group-cooperative kernels with the literal sequential
   arg-max scan forced (test hook for the rare inexact-product regime), 2 = scalar
   kernels everywhere (what _encode_bands launches), 3 = group-cooperative
   kernels everywhere.  All four give identical results.  Any other mode returns
   cudaErrorInvalidValue before anything is launched, also when count <= 0. */
int daala_b200_pvq_encode_bands_mode(const daala_b200_pvq_params *prm, const uint32_t *band_list, int count,
                                     int nmax, int mode, void *stream);
/* Work ordering of a band list (3 kernel launches): `ordered` receives the entries of `band_list`
   bucketed by (wave, expected search work), heaviest first inside each wave.  The lanes of a warp of
   the band kernels then run similar trip counts (1.3-2x on real data); results do not depend on the
   order.  entry_wave[i] (NULL = all 0) is the wave of entry i, entries of a wave stay inside that
   wave's range, so a caller's per-wave (first, count) slices remain valid.  Reads prm->in (run
   _coding_order_gather first).  Scratch: keys[count], bins[daala_b200_pvq_order_bins()]. */
int daala_b200_pvq_order_by_work(const daala_b200_pvq_params *prm, const uint32_t *band_list,
                                 const uint16_t *entry_wave, int count, int nwaves, int nmax, uint32_t *ordered,
                                 uint16_t *keys, int32_t *bins, void *stream);
int daala_b200_pvq_order_bins(void);

/* Keyframe luma with the reference's H/V intra prediction, as a band-granular wavefront
   (od_encode_compute_pred, src/encode.c:858): od_hv_intra_pred (src/intra.c:37) couples band b of a block
   only to band b of the same-size top / left neighbour (row-0 bands 1/4/7: top, column-0 bands 2/5/8:
   left, bands 3/6: none, band 0: both).  For the entries of `band_list` ((block << 4) | band, all of
   one dependency depth >= 2) this writes the bands' slices of `ref` from the neighbours' `out`; the
   caller then runs daala_b200_pvq_encode_bands[_mode] on the same slice.  dep_top / dep_left: index of
   the neighbour block in prm->blocks or -1. */
int daala_b200_pvq_intra_band_ref(const daala_b200_pvq_params *prm, const int32_t *dep_top, const int32_t *dep_left,
                                  const uint32_t *band_list, int count, void *stream);
/* Chroma-from-luma prediction planes for keyframe chroma blocks (od_resample_luma_coeffs,
   src/intra.c:72, 4:2:0) from the quantised luma plane coef_plane[0]; bit 7 of a block's `xdec`
   field marks "the luma area is coded as 4x4 blocks" (TF merge + OD_CFL_SCALING4). */
int daala_b200_pvq_cfl_pred(const daala_b200_pvq_params *prm, int32_t *pred_plane, long long pred_frame_pitch,
                            int pred_stride, int nblocks, void *stream);
/* Per block: ordered skip_diff sum, DC handling (keyframe: out[0] = in[0];
   inter: scalar quantiser of src/encode.c:1337-1344, 1377-1378). */
int daala_b200_pvq_block_finish(const daala_b200_pvq_params *prm, int nblocks, void *stream);
/* Keyframe chroma CfL sign flip of the reference vectors (src/pvq_encoder.c:847-871). */
int daala_b200_pvq_cfl_flip(const daala_b200_pvq_params *prm, int nblocks, void *stream);
/* od_raster_to_coding_order (src/partition.c:123) for a block list:
   which = 0: in <- coef_plane, which = 1: ref <- pred_plane (zeros when NULL). */
int daala_b200_coding_order_gather(const daala_b200_pvq_params *prm, int nblocks, int which, void *stream);
/* od_init_skipped_coeffs (src/state.c:1347) + od_coding_order_to_raster
   (src/partition.c:157): out -> coef_plane. */
int daala_b200_coding_order_scatter(const daala_b200_pvq_params *prm, int nblocks, void *stream);

/* ---- Deringing (SURVEY.md 8(f) rank 1) ------------------------------------ */

/* One plane through od_dering (reference src/dering.c:252, DAALA_ODINTRIN form) for every superblock:
   y <- dering(x), both int16 planes of (nhsb*64 >> xdec) x (nvsb*64 >> xdec) samples (device
   pointers; x is state->etmp[pli], y the filtered copy).  dir: one int32 per 8x8 luma block,
   [nvsb*8][dir_stride]; written when pli == 0, read for the chroma planes (run luma first).
   bskip: this plane's skip flags, one byte per 4x4 block (state->bskip[pli]).  threshold: the
   level's threshold (OD_DERING_GAIN_TABLE[level] * base, times 0.6 for chroma, call site
   src/encode.c:2822); sb_threshold (nullable) overrides it per superblock, [nvsb*nhsb].
   overlap: OD_DERING_CHECK_OVERLAP; coeff_shift: OD_COEFF_SHIFT. */
typedef struct daala_b200_dering_params {
  int16_t *y;
  const int16_t *x;
  int32_t *dir;
  const uint8_t *bskip;
  const int32_t *sb_threshold;
  int ystride, xstride, dir_stride, skip_stride;
  int nhsb, nvsb, xdec, pli;
  int threshold, overlap, coeff_shift;
  int dir_format;   /* 0: dir holds plain directions 0..7.  1: the luma pass stores direction | variance << 3;
                       2: the luma pass READS that instead of searching again (same input plane, another
                       threshold); chroma passes mask the direction out when dir_format != 0 */
} daala_b200_dering_params;
int daala_b200_dering_plane(const daala_b200_dering_params *prm, void *stream);

/* Perceptual distortion od_compute_dist (static, reference src/encode.c:1180) of `count` packed
   n x n block pairs (n = 8, 16, 32 or 64; device pointers), one double per pair.  qm_is_flat:
   enc->qm == OD_FLAT_QM (plain squared error).  Agrees with the reference to 1e-12 relative (the CUDA
   library's pow is not glibc's; everything else is exact), tests/test_gpu_dist.py. */
int daala_b200_compute_dist(const int32_t *x, const int32_t *y, int count, int n, int qm_is_flat,
                            int use_activity_masking, int coded_quantizer, double *out, void *stream);

/* The deringing level search of one frame (reference src/encode.c:2680-2811; csrc/dering_search.cu).
   etmp: the luma reconstruction after the postfilter as int16 (state->etmp[0], what
   daala_b200_frame.post16[0] receives), src: the 8-bit source luma (enc->curr_img), both DEVICE pointers
   of nhsb*64 x nvsb*64 samples.  bskip: luma skip flags, one byte per 4x4 block (device; NULL: nothing
   skipped, the keyframe case).  quantizer / coded_quantizer: state->quantizer, state->coded_quantizer;
   dering_lambda: enc->dering_lambda (src/rate.c:1086).
   cdf (HOST, [11][6], state->adapt.dering_cdf) is read and adapted exactly as the encoder's; levels (HOST,
   [nvsb*nhsb]) receives state->dering_level; dist_out (HOST, nullable, [6][nvsb*nhsb]) the distortions the
   decision was made on.  Synchronises the stream.  The decision alone (shared with the decoder's context
   modelling, src/decode.c:1040) is daala_b200_dering_decide: `coded` (nullable) flags the superblocks with
   at least one coded 4x4 block. */
typedef struct daala_b200_dering_search_params {
  const int16_t *etmp;
  const uint8_t *src;
  const uint8_t *bskip;
  int etmp_stride, src_stride, skip_stride;
  int nhsb, nvsb;
  int quantizer, coded_quantizer;
  int qm_is_flat, use_activity_masking, is_keyframe;
  double dering_lambda;
} daala_b200_dering_search_params;
void daala_b200_dering_cdf_init(uint16_t *cdf, int *increment);
int daala_b200_dering_decide(const double *dist, int nhdr, int nvdr, int is_keyframe, double dering_lambda,
                             const uint8_t *coded, uint16_t *cdf, int increment, uint8_t *levels);
int daala_b200_dering_search(const daala_b200_dering_search_params *prm, uint16_t *cdf, int increment,
                             uint8_t *levels, double *dist_out, void *stream);

/* ---- Host-side work-list construction (no GPU involved) -------------------- */

/* Everything the keyframe PVQ stage consumes besides pixels, derived from the block-size maps of a
   batch (state->bsize of every frame: one byte per 8x8 luma unit = log2(block size) - 2; 4:2:0):
   luma blocks sorted by (dependency depth, frame, y0, x0) with coef_off assigned, the same-size top /
   left neighbour of each (od_hv_intra_pred, src/intra.c:46-47) as indices into that array, and per
   size class c (0: n <= 16, 1: n = 32, 2: n = 128) the band-granular wave lists -- chain[c] sorted by
   (wave, band, block) with wave w occupying [wave_first[c][w], + wave_count[c][w]), chain_wave[c][i]
   the wave of entry i, bulk[c] the dependency-free bands 3 / 6 -- ready for
   daala_b200_pvq_intra_band_ref / _pvq_encode_bands / _pvq_order_by_work; chroma blocks of both
   planes sorted by (size, frame, plane, y0, x0), bit 7 of xdec set where the co-located luma is coded
   as 4x4 blocks (od_resample_luma_coeffs, src/intra.c:78), with their per-class band lists.
   Linear passes and counting sorts, frames in parallel on up to `nthreads` host threads.  All
   arrays are malloc'd and owned by the returned object; free with _host_keyframe_lists_free.
   NULL on bad arguments / out of memory.  nframes <= 255. */
typedef struct daala_b200_keyframe_lists {
  int n_luma, n_chroma;
  daala_b200_pvq_block *luma, *chroma;
  int32_t *dep_top, *dep_left, *depth;             /* [n_luma] */
  long long luma_total, chroma_total;              /* coefficients in the coding-order buffers */
  uint32_t *chain[3];
  uint16_t *chain_wave[3];
  int32_t *wave_first[3], *wave_count[3];
  uint32_t *bulk[3];
  uint32_t *chroma_list[3];
  int n_chain[3], n_waves[3], n_bulk[3], n_chroma_list[3];
} daala_b200_keyframe_lists;

daala_b200_keyframe_lists *daala_b200_host_keyframe_lists(const uint8_t *bsize, int nframes,
                                                          long long bsize_frame_pitch, int bstride, int nhsb,
                                                          int nvsb, int nthreads);
void daala_b200_host_keyframe_lists_free(daala_b200_keyframe_lists *lists);

/* ---- Keyframe engine: the whole hot path of a batch of keyframes, host buffers in / out --------- */

/* The batched, GPU-resident equivalent of od_encode_coefficients (reference src/encode.c:2539) for
   keyframes, minus the serial entropy coder: per frame u8 planes + the block-size map state->bsize in,
   reconstruction + PVQ symbols out.  Inside (csrc/kf_engine.cu): work lists built on the device from
   the block-size maps EVERY step (leaf descriptors by prefix scan, od_hv_intra_pred neighbours,
   dependency-ordered band items), fused lapped prefilter + fDCT, luma PVQ with H/V intra prediction as
   one persistent kernel with per-band acquire / release flags, chroma CfL + PVQ as three phase kernels
   (setup / search / finish), iDCT + postfilters;
   one CUDA graph per engine.  Two engines give a double-buffered pipeline (submit one, wait for the
   other). */
typedef struct daala_b200_kf daala_b200_kf;

typedef struct daala_b200_kf_config {
  int pic_w, pic_h;            /* luma picture size; frames are padded to whole 64x64 superblocks */
  int nframes;                 /* frames per batch (1..255), independent keyframes of one geometry */
  int q0;                      /* state->quantizer; lossy engines (lossless = 0) refuse it outside [1,
                                  DAALA_B200_KF_MAX_Q0], the range of a daala_b200_kf_frame_quant record's */
  int use_masking;             /* activity masking (OD_PVQ_BETA, src/pvq.c:205) */
  int qm_stride;               /* OD_QM_STRIDE = 5456 */
  double pvq_norm_lambda;      /* enc->pvq_norm_lambda */
  uint8_t pvq_qm_q4[3][32];    /* state->pvq_qm_q4 */
  const int16_t *qm, *qm_inv;  /* HOST: state->qm / qm_inv, 2*qm_stride entries each (copied) */
  int sb_row0, sb_rows;        /* superblock rows of this rank's shard (sb_rows <= 0: whole frames) */
  int max_blocks_div;          /* 0/1: capacity for all-4x4 maps; d > 1: 1/d of that (saves HBM) */
  int persist_ctas_per_sm;     /* 0 = default */
  int dering;                  /* 1: the reconstruction goes through od_dering with the per-superblock levels of
                                  daala_b200_kf_io.dering_level (the final application of src/encode.c:2812-2842).
                                  2: the engine also SEARCHES the levels (src/encode.c:2708-2811: five filtered
                                  candidates + the unfiltered one scored by od_compute_dist + lambda * adaptive-CDF
                                  rate, decision per frame on the device) and returns them in
                                  daala_b200_kf_io.dering_level_out; needs coded_quantizer / qm_is_flat /
                                  dering_lambda below */
  void *stream;                /* cudaStream_t to run on, or NULL: the engine creates its own */
  int coded_quantizer;         /* state->coded_quantizer (scale of od_compute_dist, src/encode.c:1221); dering == 2 or
                                  inter_finish == 2 */
  int qm_is_flat;              /* enc->qm == OD_FLAT_QM: od_compute_dist is the plain squared error; dering == 2 or
                                  inter_finish == 2 */
  double dering_lambda;        /* enc->dering_lambda (src/rate.c:1086); dering == 2 or inter_finish == 2 */
  int symbol_stream;           /* 1: every step also packs the PVQ symbols of each frame in bitstream order
                                  (daala_b200_kf_sym_block below) for daala_b200_kf_io.sym_*; 0 (default): the step
                                  is exactly the one without the stream.
                                  2: the P-frame stream (requires inter = 1): the stream of 1 with flip = 0 and one
                                  daala_b200_kf_sym_dc record per block (daala_b200_kf_io.sym_dc); with inter_finish
                                  the finishing pass also takes its decisions in stream order
                                  (daala_b200_kf_finish_io.stream_skip / stream_dc).
                                  3: the mixed stream of a frame_types = 1 engine: each frame's block records in the
                                  kind of its frame, a keyframe's as 1 with haar_dc_quant writes them (CfL flip,
                                  daala_b200_kf_sym_hdc records; its daala_b200_kf_sym_dc records are {0, 0}), a P / B
                                  frame's as 2 does (flip 0, daala_b200_kf_sym_dc records; its daala_b200_kf_sym_hdc
                                  records are all zero, which no keyframe record is); with inter_finish the finishing
                                  pass takes its decisions in stream order as with 2.
                                  1 is refused with inter (a keyframe block has no scalar DC), 2 without it, 3 without
                                  frame_types and 1 and 2 with it; other values are refused */
  int inter;                   /* 0 (default): keyframes, exactly the engine described above.
                                  1: P-frame residual mode.  Every frame is coded as od_encode_coefficients codes a
                                  non-key frame, entropy coding and the coder-state skip decision left to the host:
                                  the motion-compensated prediction is an INPUT (daala_b200_kf_io.pred_pixels), it
                                  goes through the same prefilters + fDCT as the source (no DC Haar pyramid on either)
                                  and is the reference vector of every band of every plane (pvq_theta with
                                  is_keyframe = 0: no H/V intra prediction, no CfL, no flip).  No band depends on
                                  another block, so luma and chroma both run as the three phase kernels (setup /
                                  search / finish) of keyframe chroma and the persistent chain kernel is not launched.  DC is the scalar
                                  quantisation of in[0] - ref[0] with the band-0 quantiser (index in
                                  daala_b200_kf_io.luma_dc / chroma_dc); the uncoded tail of 32x32 / 64x64 blocks is
                                  the transformed prediction (od_init_skipped_coeffs for inter frames).
                                  Not defined, and refused by daala_b200_kf_create, together with dering,
                                  symbol_stream = 1 (2 is its stream) or a row shard (sb_rows > 0) */
  int inter_mc;                /* 0 (default): with inter, the prediction planes are the host input pred_pixels.
                                  1: the engine makes the prediction itself, as od_state_mc_predict does
                                  (reference src/state.c:932), from each frame's MV grid
                                  (daala_b200_kf_io.mv_grid) and its GOLD and PREV pictures in a pool of reference
                                  pictures (daala_b200_kf_io.ref_pixels / ref_slot).  Two steps inside the graph: the
                                  leaves of od_state_pred_block's split recursion per 64x64 MV block (work-list
                                  phase) and the OBMC prediction of every leaf in all three planes (forward phase,
                                  before the transforms).  Reference pixels outside the picture are read at the
                                  nearest edge pixel, which is the reference's edge extension inside its 64 / 32
                                  pixels of padding.  Requires inter = 1; refused by daala_b200_kf_create
                                  otherwise */
  int mc_refs;                 /* inter_mc: capacity of the reference-picture pool in pictures; 0 = 2 * nframes */
  int inter_finish;            /* 0 (default): nothing below exists; the engine is exactly the one without this field.
                                  1: the engine also has the finishing pass daala_b200_kf_finish (the host coder's skip
                                  and DC decisions, the skip map bskip, deringing over it, final reconstruction), and
                                  each step writes daala_b200_kf_io.luma_dc_resid / chroma_dc_resid (as does an engine
                                  with symbol_stream = 2).
                                  2: the same pass, which also SEARCHES the deringing levels of every frame instead of
                                  taking them (src/encode.c:2708-2811 for a P frame, see daala_b200_kf_finish_io);
                                  needs coded_quantizer / qm_is_flat / dering_lambda above.
                                  1 and 2 require inter = 1; refused by daala_b200_kf_create otherwise */
  int late_skip;               /* 0 (default): nothing below exists; the engine is exactly the one without this field.
                                  1: each step also computes the late-skip distortions of every block
                                  (daala_b200_kf_late_skip below, returned through daala_b200_kf_io.luma_late_skip /
                                  chroma_late_skip / sym_late_skip), with coded_quantizer, qm_is_flat and use_masking
                                  (enc->use_activity_masking) above.  Requires inter = 1; other values, and 1 without
                                  inter, are refused by daala_b200_kf_create */
  int mc_next;                 /* 0 (default): nothing below exists; the engine is exactly the one without this field.
                                  1: B frames (OD_SET_B_FRAMES).  A vertex with ref 2 (OD_FRAME_NEXT) is predicted from
                                  the frame's NEXT picture (daala_b200_kf_io.ref_slot_next) with its second vector mv1
                                  (daala_b200_kf_io.mv1_grid), as od_state_pred_block_from_setup does (reference
                                  src/state.c:647-660); refs 0 and 1 work as before and their mv1 is not read (the
                                  encoder leaves stale vectors there).  Nothing after the prediction differs from a P
                                  frame.  mc_refs = 0 then means 3 * nframes.  Requires inter_mc = 1; other values, and
                                  1 without inter_mc, are refused by daala_b200_kf_create */
  int frame_quant;             /* 0 (default): every frame is coded at this config's quantizer: the engine makes one
                                  daala_b200_kf_frame_quant record per frame from q0, coded_quantizer, dering_lambda
                                  and pvq_qm_q4 at create, and its kernels read those records.
                                  1: every frame of a step has its own quantizer: daala_b200_kf_io.frame_quant gives one
                                  daala_b200_kf_frame_quant per frame, and the step and the finishing pass read no
                                  per-frame field of this config (q0, coded_quantizer, dering_lambda, pvq_qm_q4).  The
                                  stream settings use_masking, qm / qm_inv, qm_is_flat and pvq_norm_lambda stay
                                  engine-wide: the frames of one batch must share them.  Requires inter = 1; other
                                  values, and 1 without inter, are refused by daala_b200_kf_create */
  int lossless;                /* 0 (default): nothing below exists; the engine is exactly the one without this field.
                                  1: every frame is coded at quantizer 0 (OD_SET_QUANT 0), the reference's lossless
                                  Haar-wavelet path (OD_LOSSLESS, src/internal.h:131): every superblock is one 64x64 block
                                  (32x32 in 4:2:0 chroma), c = pixel - 128, d = od_haar(c), no lapping, no deringing,
                                  a quantizer of 1 everywhere.  The step returns each block's residual
                                  (daala_b200_kf_io.ll_coeffs), the three root sums the host's tree coder starts from
                                  (daala_b200_kf_ll_block) and the reconstruction the decoder makes, which equals the
                                  (padded) input.  Keyframes (inter = 0): the residual is d, its DC the difference to the
                                  superblock DC predictor of od_quantize_haar_dc_sb (src/encode.c:1537-1590).  P and B
                                  frames (inter = 1, prediction planes from the host or made by inter_mc [+ mc_next]):
                                  outside the picture the input is replaced by the prediction (src/encode.c:2589-2602),
                                  the residual is d - od_haar(prediction), DC included.  q0, pvq_qm_q4, the other
                                  quantizer fields and io.bsize are not read.  Refused by daala_b200_kf_create with a
                                  value other than 0 or 1, and 1 together with dering, symbol_stream, late_skip,
                                  inter_finish, frame_quant or a row shard (sb_rows > 0) */
  int haar_dc_quant;           /* 0 (default): keyframes are reconstructed with their unquantised DCs (the inverse
                                  undoes the forward transform's Haar DC pyramid); nothing below exists.
                                  1: the step quantises the keyframe DCs as the reference encoder does: per plane,
                                  od_quantize_haar_dc_sb and od_quantize_haar_dc_level (src/encode.c:1537-1657, with the
                                  RDO increment rated on the adapting DC model) in od_encode_recursive's order, one warp
                                  per (frame, plane) beside the luma chain kernel.  The coefficient planes, out[0] of
                                  every block, the 4x4-chroma CfL reference and the reconstruction then carry the
                                  quantised DCs; daala_b200_kf_io.dc_index returns the coded indices.  q0, pvq_qm_q4 and
                                  pvq_norm_lambda are the chain's quantizer and lambda.  Refused by daala_b200_kf_create
                                  with a value other than 0 or 1, and 1 together with inter (unless frame_types = 1),
                                  lossless or a row shard (sb_rows > 0: the superblock predictor reads the row above) */
  int keyframe_quant;          /* 0 (default): every keyframe is coded at this config's quantizer, through records
                                  made from it as with frame_quant = 0.
                                  1: the keyframe counterpart of frame_quant: every keyframe of a step has its own
                                  quantizer, one daala_b200_kf_frame_quant per frame in daala_b200_kf_io.frame_quant.
                                  The luma chain kernel, the phase kernels, the DC chain (haar_dc_quant) and the
                                  deringing stage (its thresholds and, with dering = 2, the level search's distortion
                                  scale and lambda) read the block's or superblock's frame's record, and the step reads
                                  no per-frame field of this config (q0, coded_quantizer, dering_lambda, pvq_qm_q4).
                                  use_masking, qm / qm_inv, qm_is_flat and pvq_norm_lambda stay engine-wide: they are
                                  stream settings, and the frames of one batch must share them.  A host encoder fills
                                  a keyframe's record with q0 = max(1, state->quantizer), state->coded_quantizer,
                                  enc->dering_lambda and the pvq_qm_q4 od_interp_qm set for that keyframe (reference
                                  src/encode.c:3050-3075).  Refused by daala_b200_kf_create with a value other than 0
                                  or 1, and 1 together with inter (P and B frames have frame_quant), lossless or a
                                  row shard (sb_rows > 0) */
  int frame_types;             /* 0 (default): nothing below exists; the engine is exactly the one without this field.
                                  1: keyframes and P / B frames in one batch.  Every step takes one type per frame
                                  (daala_b200_kf_io.frame_type: 1 = keyframe, 0 = P or B frame).  A keyframe is coded
                                  exactly as an engine with keyframe_quant = 1 and haar_dc_quant = 1 codes it (DC Haar
                                  pyramid and DC chain, luma through the chain kernel, CfL chroma), a P or B frame exactly
                                  as the frame_quant = 1 inter engine codes it; each frame reads its own
                                  daala_b200_kf_frame_quant record.  One captured graph serves every mix of types: the
                                  type table goes to the device with the records.  The finishing pass leaves a keyframe's
                                  coefficients as the step coded them (its skip and DC entries are not read, its bskip is
                                  all zero) and deringes it at its given level (inter_finish = 1) or at the level the
                                  keyframe rule searches (inter_finish = 2: every superblock, up / left CDF context);
                                  ref_slot_out stores keyframes like any other frame.  Requires inter = 1, frame_quant = 1,
                                  haar_dc_quant = 1 and inter_finish 1 or 2 (inter_mc and mc_next are allowed); refused by
                                  daala_b200_kf_create with a value other than 0 or 1, and 1 together with symbol_stream
                                  1 or 2 (3 is the mixed stream), late_skip, lossless, dering (a keyframe is deringed in
                                  the finishing pass) or a row shard (sb_rows > 0) */
} daala_b200_kf_config;

/* config.lossless: the root sums of one block (od_compute_max_tree, src/encode.c:899-919, over the residual of
   daala_b200_kf_io.ll_coeffs): what od_wavelet_quantize codes first (src/encode.c:1029-1049).  tree[0] is the tree of
   the horizontal root (x, y) = (1, 0) (tree_sum[0][1]: every sub-band at column offset 1 << level, row offset 0),
   tree[1] that of (0, 1) (tree_sum[1][0]), tree[2] that of (1, 1) (tree_sum[1][1]); each is the sum of |residual| over
   its sub-bands.  The DC is in no tree. */
typedef struct daala_b200_kf_ll_block {   /* 16 bytes */
  int32_t tree[3];
  int32_t reserved;        /* 0 */
} daala_b200_kf_ll_block;

/* The quantizer of one frame of a batch (config.frame_quant = 1 or config.keyframe_quant = 1; other lossy engines make
   theirs from the config), what od_enc_rc_select_quantizers_and_lambdas
   (reference src/rate.c:727-835, :1086) left in state / enc for that frame, and the pvq_qm_q4 table in force
   (src/encode.c:3050-3075).  Submit refuses a record with q0 outside [1, 8191] (8191 = od_codedquantizer_to_quantizer(63);
   lossless frames, quantizer 0, are coded by an engine with config.lossless), coded_quantizer outside [1, 63], a dering_lambda that is negative or
   not finite, or a pvq_qm_q4 entry of 0. */
typedef struct daala_b200_kf_frame_quant {   /* 112 bytes, 8-byte aligned */
  int32_t q0;                 /* max(1, state->quantizer) of this frame */
  int32_t coded_quantizer;    /* state->coded_quantizer: od_compute_dist's scale */
  double dering_lambda;       /* enc->dering_lambda of this frame */
  uint8_t pvq_qm_q4[3][32];   /* state->pvq_qm_q4 in force for this frame */
} daala_b200_kf_frame_quant;
#define DAALA_B200_KF_MAX_Q0 8191

/* One vertex of a P frame's MV grid, as od_mv_grid_pt (reference src/mc.h:73-84) holds it after od_mv_est. */
typedef struct daala_b200_mv_pt {  /* 12 bytes */
  int32_t mv[2];           /* x, y in 1/8 luma pixel */
  uint8_t valid;           /* the vertex is coded: the MV block with this vertex at its centre is split */
  uint8_t ref;             /* picture the vector points into: 0 = OD_FRAME_GOLD, 1 = OD_FRAME_PREV, and on
                              config.mc_next engines 2 = OD_FRAME_NEXT (predicted with mv1, daala_b200_kf_io.mv1_grid) */
  uint8_t pad_[2];
} daala_b200_mv_pt;

typedef struct daala_b200_kf_totals {
  long long n_luma, luma_coefs, n_chroma, chroma_coefs;
} daala_b200_kf_totals;

/* Symbol stream (config.symbol_stream): what the serial entropy coder reads, per frame in bitstream order.
   Coding order: superblocks in raster order (of the engine's shard, sb_row0 / sb_rows), in each planes 0, 1, 2,
   in each plane the quadtree leaves depth-first with the children top-left, top-right, bottom-left,
   bottom-right (od_encode_recursive, reference src/encode.c:1780-1787 and :2605-2656; with 4:2:0 one 4x4 chroma
   block per 8x8 unit whose luma is coded as 4x4 blocks).  For a batch, three arrays hold the frames one after
   the other, and a per-frame index (daala_b200_kf_sym_frame) says where each frame's part is:
     blocks  one daala_b200_kf_sym_block per leaf block;
     bands   per block nbands(bs) = 1, 4, 7, 9, 9 records {coded gain index, itheta, max_theta, K} as int16[4]
             (the values of daala_b200_kf_io.*_res), in band order;
     pulses  per band with K > 0 the n - (itheta != -1) values pvq_encode_partition hands to od_encode_pvq_codeword
             (src/pvq_encoder.c:719-720; n = the band's size), each an int8 when K <= 127 and a little-endian
             int16 otherwise (|y| <= K, so K gives the width).  Bands with K = 0 have no bytes. */
typedef struct daala_b200_kf_sym_block {   /* 24 bytes, 8-byte aligned */
  double skip_diff;        /* the block's skip_diff (as daala_b200_kf_io.*_skip_diff) */
  uint32_t pulse_off;      /* byte offset of the block's first pulse inside its frame's pulse bytes */
  uint32_t band_off;       /* index of the block's first band record inside its frame's band records */
  uint16_t x0, y0;         /* top-left sample of the block inside its plane */
  uint8_t bs;              /* log2(n) - 2 */
  uint8_t pli;             /* plane 0, 1, 2 */
  uint8_t flip;            /* keyframe CfL sign flip (chroma); 0 for luma */
  uint8_t reserved;        /* 0 */
} daala_b200_kf_sym_block;

/* symbol_stream = 2 (P frames) and 3 (mixed batches; {0, 0} on a keyframe's block records): one record per block
   record, at the same index as the daala_b200_kf_sym_block it belongs to (a frame's part is first_block / n_blocks of
   the index, as for the block records). */
typedef struct daala_b200_kf_sym_dc {      /* 8 bytes */
  int32_t qdc;             /* the step's scalar DC index (as daala_b200_kf_io.luma_dc / chroma_dc) */
  int32_t dc_resid;        /* the unquantised DC residual in[0] - ref[0] (as daala_b200_kf_io.*_dc_resid), what the
                              host's od_rdo_quant quantises (src/pvq_encoder.c:886 / :956) */
} daala_b200_kf_sym_dc;

/* config.late_skip = 1: the four distortions od_block_encode's late skip (reference src/encode.c:1412-1450) can ask
   for, one record per block.  All are od_compute_dist(c_orig, c, n) of src/encode.c:1180 (coded_quantizer, qm_is_flat,
   use_masking of the config), n = 4 << bs with the plane-local bs.  c_orig is the block's samples after the SB-edge
   and split prefilters (`c` at src/encode.c:1283), mc_orig the same for the prediction; every other c is the leaf
   iDCT (no postfilter, the c_noskip of :1420-1423) of a candidate coefficient block:
     dist_skip          d = md, the late skip (:1444-1448); its reconstruction is mc_orig itself;
     noskip_coded_dc0   AC as the step coded it (its `d`, with md as the uncoded tail of 32x32 / 64x64 blocks),
                        d[0] = md[0];
     noskip_coded_dcq   the same AC, d[0] = md[0] + q1 * dc_quant;
     noskip_pred_dcq    AC = md (the PVQ skip, src/pvq_encoder.c:975), d[0] = md[0] + q1 * dc_quant;
   dc_quant = max(1, q0 * pvq_qm_q4[pli][bs * (bs + 1)] >> 4) is the step's band-0 quantiser and
   q1 = OD_DIV_R0(dc_resid, dc_quant), dc_resid = in[0] - ref[0] (daala_b200_kf_sym_dc.dc_resid).
   Why these four: od_rdo_quant (src/pvq_encoder.c:730-741) returns 0 or q1 whatever the coder's DC rate, and the AC
   is either coded or md.  Of the four (AC, DC) pairs, (md, 0) is od_pvq_encode's own skip (no late-skip test; its
   distortion is dist_skip); the other three are the dist_noskip candidates.  The host coder picks the record field
   of its (pvq_skip, dc) pair -- (0, 0) noskip_coded_dc0, (0, q1) noskip_coded_dcq, (1, q1) noskip_pred_dcq -- and runs
   the reference's test (:1431) with its own rates and enc->bs_rdo_lambda:
     late skip  <=>  dist_skip + lambda * rate_skip < dist_noskip + lambda * rate_noskip
   then, when it wins, hands skip = 1, dc = 0 for the block to daala_b200_kf_finish.  Blocks with bs = 0 (4x4 luma
   and 4x4 chroma) have no late skip (has_late_skip_rdo, :1280) and an all-zero record. */
typedef struct daala_b200_kf_late_skip {   /* 32 bytes */
  double dist_skip;         /* od_compute_dist(c_orig, mc_orig, n) */
  double noskip_coded_dc0;  /* od_compute_dist(c_orig, idct(coded AC, d[0] = md[0]), n) */
  double noskip_coded_dcq;  /* ... coded AC, d[0] = md[0] + q1 * dc_quant */
  double noskip_pred_dcq;   /* ... AC = md (PVQ skip), d[0] = md[0] + q1 * dc_quant */
} daala_b200_kf_late_skip;

/* Engines with symbol_stream = 1 and haar_dc_quant = 1, and keyframes in the mixed stream (symbol_stream = 3, where a
   P / B frame's records are all zero: no keyframe record is, since the superblock DC has bsi = 4 and every other record
   child >= 1, so an all-zero record marks a P / B frame): the keyframe's DC symbols in the order od_encode_coefficients
   codes them (reference src/encode.c:2605-2656, :1765-1787), one record per block record, so a frame's part is
   first_block / n_blocks of the index as for the block records.  A quadtree with L leaves has (L - 1) / 3 split nodes,
   and the reference codes one superblock DC per (superblock, plane) and three indices per split node: L symbols.  Per
   (superblock, plane) the records fill the index range of its block records: the superblock DC first, then each split
   node's three (child 1, 2, 3) in pre-order with the children top-left, top-right, bottom-left, bottom-right.  A host
   coder emits record j just before block record `block` (after, on luma with child == 1, the node's split symbol,
   src/encode.c:1765-1769): generic_encode of |value| on the plane's DC model with ex_sb_dc[pli] (child 0) or
   ex_dc[pli][bsi][child - 1], then the sign bit when value != 0 (od_ec_enc_bits(ec, value < 0, 1)). */
typedef struct daala_b200_kf_sym_hdc {     /* 12 bytes */
  int32_t value;           /* the signed coded index (what daala_b200_kf_io.dc_index holds at the node's position) */
  uint32_t block;          /* frame-relative index of the block record the coder emits this symbol before: the first
                              leaf, in coding order, of the superblock (child 0) or of the split node (1..3) */
  uint8_t pli;
  uint8_t bsi;             /* child 0: 4 (the superblock).  1..3: the bsi od_quantize_haar_dc_level is called with
                              (od_encode_recursive's bsi - 1, the luma size index also for chroma): ex_dc[pli][bsi] */
  uint8_t child;           /* 0: the superblock DC; 1..3: x[child] of the split node */
  uint8_t reserved;        /* 0 */
} daala_b200_kf_sym_hdc;

typedef struct daala_b200_kf_sym_frame {   /* one frame's part of the batch-wide arrays (indices, not bytes, */
  int64_t first_block, n_blocks;           /* except for the pulses) */
  int64_t first_band, n_bands;
  int64_t first_byte, n_bytes;
} daala_b200_kf_sym_frame;

typedef struct daala_b200_kf_sym_bounds {  /* worst-case lengths, in the units of the daala_b200_kf_io.sym_* capacities */
  long long index, blocks, bands, pulse_bytes;
} daala_b200_kf_sym_bounds;

/* Host buffers of one batch.  Inputs: padded planes [nframes][plane_h][plane_w] u8 and block-size
   maps [nframes][nvsb*8][nhsb*8] (one byte per 8x8 luma unit = log2(size) - 2).  Outputs (each may be
   NULL = not copied back): reconstruction planes; block descriptors in scan order of the 8x8 units
   (frame, row, column; the four 4x4 blocks of a unit in raster order; chroma: plane 1 then plane 2 per
   unit); per block 9 band records {coded gain index (pvq_theta's return value), itheta, max_theta, K}
   as int16[4]; the pulse vectors in coding order (16 bit) at each block's coef_off; per block
   skip_diff; per chroma block the CfL flip flag.  Sized by daala_b200_kf_count_blocks.  Pinned memory
   (daala_b200_host_alloc) makes the copies asynchronous. */
typedef struct daala_b200_kf_io {
  const uint8_t *pixels[3];
  const uint8_t *bsize;
  const uint8_t *dering_level;          /* [nframes][nvsb][nhsb] levels 0..5 (state->dering_level); config.dering only */
  const daala_b200_kf_totals *totals;   /* optional: result of _count_blocks for `bsize` */
  uint8_t *pixels_out[3];
  daala_b200_pvq_block *luma_blocks, *chroma_blocks;
  int16_t *luma_res, *chroma_res;       /* [n_blocks][9][4] */
  int16_t *luma_y16, *chroma_y16;       /* [coefs] */
  double *luma_skip_diff, *chroma_skip_diff;
  int32_t *chroma_flip;
  int32_t *counts;                      /* 32 ints of device-side counters (diagnostics) */
  uint8_t *dering_level_out;            /* [nframes][nvsb][nhsb]: the levels applied (config.dering == 2: the searched ones) */
  /* Symbol stream (config.symbol_stream): pinned host buffers (daala_b200_host_alloc / cudaHostAlloc) with their
     capacities in frames, block records, band records and bytes, at least daala_b200_kf_symbol_bounds; NULL = not
     copied.  Only the used part of each array is copied, by a kernel that reads the lengths on the device. */
  daala_b200_kf_sym_frame *sym_index;
  long long sym_index_cap;
  daala_b200_kf_sym_block *sym_blocks;
  long long sym_blocks_cap;
  int16_t *sym_bands;                   /* [n][4] */
  long long sym_bands_cap;
  uint8_t *sym_pulses;
  long long sym_pulses_cap;
  /* config.inter only (required there, ignored otherwise; luma_dc / chroma_dc are optional with symbol_stream = 2 or 3,
     whose sym_dc carries the same indices). */
  const uint8_t *pred_pixels[3];        /* motion-compensated prediction planes, shapes and padding of `pixels` */
  int32_t *luma_dc, *chroma_dc;         /* [n_blocks]: the scalar-quantised DC index qdc of each block (keyframes code
                                           DC in the Haar pyramid instead), block order of luma_res / chroma_res */
  /* config.inter_mc only (required there except pred_pixels_out; pred_pixels must then be NULL). */
  const uint8_t *ref_pixels[3];         /* pool of nrefs reference pictures [nrefs][plane_h][plane_w] u8: each the
                                           frame-sized area of one of state->ref_imgs, without the edge extension */
  int nrefs;                            /* pictures in the pool, 1..mc_refs */
  const int32_t *ref_slot;              /* [nframes][2]: pool slots of each frame's GOLD and PREV pictures (equal
                                           when the frame predicts from one picture) */
  const daala_b200_mv_pt *mv_grid;      /* [nframes][nvsb*8 + 1][nhsb*8 + 1]: each frame's state->mv_grid */
  uint8_t *pred_pixels_out[3];          /* optional: the prediction planes the engine made, layout of pixels */
  /* config.inter_finish or symbol_stream = 2 / 3 only (optional, NULL = not copied). */
  int32_t *luma_dc_resid, *chroma_dc_resid; /* [n_blocks]: each block's unquantised DC residual in[0] - ref[0] (what the
                                           host's od_rdo_quant quantises, src/pvq_encoder.c:886 / :956), block order
                                           of luma_dc / chroma_dc */
  /* config.inter_mc only.  0 (default): the step uploads ref_pixels into slots [0, nrefs) of the engine's pool, as
     described above.  1: the step reads the pool as it stands and uploads no picture; ref_pixels[0..2] must then be
     NULL and nrefs 0, and every ref_slot entry must lie in [0, mc_refs) and name a slot that holds a picture.  A slot
     holds one once daala_b200_kf_pool_load, a submit with ref_resident = 0 (slots [0, nrefs)) or a finish with
     daala_b200_kf_finish_io.ref_slot_out has written it.  Everything is ordered by call order on the engine's
     stream: a step submitted before the finish that rewrites its PREV slot reads the old picture. */
  int ref_resident;
  /* config.symbol_stream = 2 or 3 only: the DC records of the stream (daala_b200_kf_sym_dc), a pinned host buffer with
     its capacity in records, at least daala_b200_kf_symbol_bounds(...).blocks; NULL = not copied.  Only the used part
     is copied, as for the other stream arrays. */
  daala_b200_kf_sym_dc *sym_dc;
  long long sym_dc_cap;
  /* config.late_skip = 1 only (optional, NULL = not copied): the late-skip records (daala_b200_kf_late_skip) in the
     block order of luma_res / chroma_res ([n_blocks] each) ... */
  daala_b200_kf_late_skip *luma_late_skip, *chroma_late_skip;
  /* ... and, with symbol_stream = 2, in stream order: one record per block record at the same index as sym_blocks, a
     pinned host buffer with its capacity in records, at least daala_b200_kf_symbol_bounds(...).blocks.  Only the used
     part is copied, as for sym_dc. */
  daala_b200_kf_late_skip *sym_late_skip;
  long long sym_late_skip_cap;
  /* config.mc_next only (required there, refused otherwise).  The same submit checks as ref_slot apply to
     ref_slot_next: within [0, nrefs) for an upload step, within [0, mc_refs) and holding a picture with ref_resident. */
  const int32_t *ref_slot_next;         /* [nframes]: pool slot of each frame's NEXT picture */
  const int32_t *mv1_grid;              /* [nframes][nvsb*8 + 1][nhsb*8 + 1][2]: each vertex's mv1 (od_mv_grid_pt.mv1,
                                           src/mc.h:73-84) in 1/8 luma pixel, read only where ref == 2 */
  /* config.frame_quant = 1 or config.keyframe_quant = 1 only (required there, refused otherwise): [nframes] records,
     frame f coded at frame_quant[f].  They go to the device with the step's other inputs; the finishing pass after the
     step uses the same records. */
  const daala_b200_kf_frame_quant *frame_quant;
  /* config.lossless only (refused otherwise; each optional, NULL = not copied).  ll_coeffs[p]: [nframes][plane_h][plane_w]
     int16, each block's residual in raster order at the block's own place (the layout of the `d` planes); the DC slot
     holds the coded DC: d[0] minus the superblock DC predictor on keyframes, d[0] - md[0] on P and B frames.  Every
     value fits int16 (the bound is derived in DESIGN.md).  ll_blocks: [nframes][nvsb][nhsb][3] records, one per
     superblock and plane.  The reconstruction goes to pixels_out. */
  int16_t *ll_coeffs[3];
  daala_b200_kf_ll_block *ll_blocks;
  /* config.lossless with inter_mc only (refused otherwise; optional): [nframes] the pool slot that receives frame f's
     reconstruction, -1 = not stored, as daala_b200_kf_finish_io.ref_slot_out does for a lossy step; entries must lie
     in [-1, mc_refs) and name distinct slots.  The stored slots then hold a picture (ref_resident).  The step's own
     prediction is made before the store, so a frame may name its own PREV slot. */
  const int32_t *ll_ref_slot_out;
  /* config.haar_dc_quant only (refused otherwise; each optional, NULL = not copied): [nframes][plane_h / 4][plane_w / 4]
     int32, plane p's signed keyframe DC indices at 4x4 granularity: a superblock's DC index at the superblock's origin,
     the three indices of a split node (its children's Haar coefficients x[1], x[2], x[3]) at the origins of its
     children 1, 2, 3 (top right, bottom left, bottom right), 0 everywhere else.  INTEGRATION.md describes the order
     the coder reads them in. */
  int32_t *dc_index[3];
  /* config.symbol_stream = 1 with haar_dc_quant = 1, or symbol_stream = 3, only (refused otherwise): the keyframe DC
     records of the stream (daala_b200_kf_sym_hdc; all zero on a P / B frame's block records of the mixed stream), a
     pinned host buffer with its capacity in records, at least daala_b200_kf_symbol_bounds(...).blocks; NULL = not
     copied.  Only the used part is copied, as for sym_dc.  With them the index grids dc_index are optional. */
  daala_b200_kf_sym_hdc *sym_hdc;
  long long sym_hdc_cap;
  /* config.frame_types = 1 only (required there, refused otherwise): [nframes] 1 = keyframe, 0 = P or B frame; any other
     value is refused.  Outputs of one kind are 0 for the blocks and frames of the other: chroma_flip and dc_index[0..2]
     for P / B frames; luma_dc / chroma_dc, luma_dc_resid / chroma_dc_resid and pred_pixels_out (inter_mc) for keyframes.
     With inter_mc a keyframe has no prediction: its ref_slot / ref_slot_next entries and its MV grid are not read or
     checked, and it adds nothing to counts[19] / counts[20]. */
  const uint8_t *frame_type;
} daala_b200_kf_io;

/* The finishing pass of a P-frame batch (config.inter_finish), daala_b200_kf_finish: the host coder's per-block
   decisions in, the reconstruction the decoder will make out.  Decision arrays are in the block order of
   luma_res / chroma_res of the last submitted step.
     skip = 0: the block's coefficients are those the step coded, with d[0] = md[0] + dc * dc_quant;
     skip = 1: d = md over the whole block (the PVQ skip of src/pvq_encoder.c:951-977, AC = prediction; the late
               skip of src/encode.c:1412-1450 is skip = 1 with dc = 0), then d[0] = md[0] + dc * dc_quant.
   dc_quant = max(1, q0 * pvq_qm_q4[pli][bs * (bs + 1)] >> 4), the step's band-0 quantiser (config.frame_quant: the
   block's frame's record).  A block counts as
   skipped in bskip when skip && dc == 0 (od_pvq_encode's return value with has_dc_skip, src/encode.c:1364-1371,
   :1690-1691).  Then the inverse, the split and superblock-edge postfilters (they ignore the skip flags without
   OD_DEBLOCKING, src/filter.c:1505-1509, :1596-1598) and the deringing of src/encode.c:2695-2842 with the given
   levels: a superblock none of whose 4x4 luma units is coded is forced to level 0 (:2724-2738), chroma thresholds
   are x0.6, od_dering reads the real skip map (src/dering.c:297-325).  |dc| must not exceed
   DAALA_B200_KF_FINISH_DC_LIMIT / DQ, DQ the largest dc_quant of the engine over planes and block sizes (with
   config.frame_quant: of the last step, over its records, planes and block sizes), so that
   dc * dc_quant stays within 2^30 and md[0] + dc * dc_quant within od_coeff.  The pass equals the reference bit for
   bit while every sample of the reconstruction before deringing (state->ctmp, after the superblock-edge postfilter)
   fits int16, as it always does for 8-bit content with decisions near the step's own DC indices: the pass keeps that
   plane only as the int16 deringing input (state->etmp, src/encode.c:2703-2705), so beyond it a superblock at level 0,
   and the level search's unfiltered candidate, see the int16 truncation where the reference keeps od_coeff.
   config.inter_finish = 2: the pass searches the levels itself, between the superblock-edge postfilter and the
   deringing, as the keyframe search of config.dering = 2 with the three rules of a P frame: every filtered candidate
   reads the frame's own luma skip map; a superblock with no coded 4x4 luma unit is not searched, gets level 0 and does
   not adapt the CDF; the CDF context is always 0 (no up / left neighbours).  The score of a level is od_compute_dist of
   the candidate against the step's source luma plus dering_lambda times its cost under the frame's adaptive CDF, which
   starts from the initial CDFs for every frame.  dering_level must then be NULL; dering_level_out returns the searched
   levels, which are the levels applied (the host coder codes them and adapts its own dering CDF with them). */
#define DAALA_B200_KF_FINISH_DC_LIMIT (1 << 30)
typedef struct daala_b200_kf_finish_io {
  const uint8_t *luma_skip, *chroma_skip;  /* [n_blocks]: 0 or 1 (required) */
  const int32_t *luma_dc, *chroma_dc;      /* [n_blocks]: the final DC index of each block (required) */
  const uint8_t *dering_level;             /* [nframes][nvsb][nhsb] levels 0..5; NULL = all 0.  config.inter_finish = 2:
                                              must be NULL (the pass searches them) */
  uint8_t *pixels_out[3];                  /* optional: the reconstruction, layout of daala_b200_kf_io.pixels */
  uint8_t *bskip_out[3];                   /* optional: state->bskip[pli] of every frame, [nframes][plane_h / 4][nhsb * 16]
                                              (one byte per 4x4 block of the plane, row stride state->skip_stride for
                                              every plane; the columns past plane_w / 4 of a chroma row are 0) */
  uint8_t *dering_level_out;               /* optional: [nframes][nvsb][nhsb] the levels applied (config.inter_finish
                                              = 2: the searched ones) */
  const int32_t *ref_slot_out;             /* optional, engines with config.inter_mc and inter_finish: [nframes] the slot
                                              of the engine's reference-picture pool that receives frame f's
                                              reconstruction after the final deringing, -1 = not stored; NULL = nothing
                                              stored.  The picture is stored as the pass made it, which is a valid
                                              reference as it is (the prediction's clamped reads are the edge
                                              extension).  Entries must lie in [-1, mc_refs) and name distinct slots.
                                              Rewriting a slot the last step read (a frame's own PREV slot) is legal:
                                              the step's prediction and md are already made, and a repeated finish
                                              reads md, never the pool; the last finish wins. */
  /* The decisions in stream order (engines with config.symbol_stream = 2 or 3): one entry per block of the last
     submitted step, in the order of that step's sym_blocks, frames one after the other (n_luma + n_chroma entries).  A
     call gives either these two or the four classic arrays above, never both; the same checks apply to either form.
     With symbol_stream = 3 a keyframe's entries are checked like the others and otherwise not read, as in the classic
     form. */
  const uint8_t *stream_skip;              /* 0 or 1 */
  const int32_t *stream_dc;                /* the final DC index */
} daala_b200_kf_finish_io;

typedef struct daala_b200_kf_buffers {  /* device pointers of an engine (tests, device-resident callers) */
  uint8_t *pixels[3];
  int32_t *coeffs[3];
  int32_t *lapped[3];
  uint8_t *pixels_out[3];
  int plane_w[3], plane_h[3];
  uint8_t *bsize;
  int32_t *counts;
  daala_b200_pvq_block *luma_blocks, *chroma_blocks;
  int32_t *dep_top, *dep_left;          /* same-size neighbour above / left of each luma block, or -1 */
  int32_t *succ_bottom, *succ_right;    /* the inverse: the block that waits for this one, or -1 */
  uint32_t *luma_items[3];              /* dependency-free luma items (bands 3 / 6) per class */
  uint32_t *luma_heads;                 /* row / column chain items ready from the start; counts[15] of them, in
                                           descending order of chain weight (the order the chain kernel takes them) */
  uint32_t *luma_heads0;                /* band-0 items ready from the start; counts[16] of them */
  uint32_t *chroma_items[3];
  int16_t *luma_res, *chroma_res, *luma_y16, *chroma_y16;
  double *luma_skip_diff, *chroma_skip_diff;
  int32_t *chroma_flip;
  int max_luma_blocks, max_chroma_blocks;
  void *stream;
  long long bytes_allocated;
  uint8_t *pred_pixels[3];              /* config.inter: the prediction pixels and their transform md (the */
  int32_t *pred_coeffs[3];              /* layout of pixels / coeffs); NULL otherwise */
  uint32_t *luma_heads_raw;             /* luma_heads in the order the dependency builder found them, and the */
  int32_t *luma_head_bin;               /* weight bin of each: 12287 - min(chain length x class cost, 12287) */
  uint8_t *ref_pixels[3];               /* config.inter_mc: the reference-picture pool ([mc_refs][plane_h][plane_w]), */
  int32_t *ref_slot;                    /* the slot map ([nframes][2]) and the MV grids ([nframes][nvsb*8 + 1] */
  daala_b200_mv_pt *mv_grid;            /* [nhsb*8 + 1]) the prediction step reads; NULL otherwise */
  int mc_refs;                          /* pictures the pool holds (0 without inter_mc) */
  int32_t *ref_slot_next;               /* config.mc_next: the NEXT slots ([nframes]) and the mv1 grids */
  int32_t *mv1_grid;                    /* ([nframes][nvsb*8 + 1][nhsb*8 + 1][2]); NULL otherwise */
  daala_b200_kf_frame_quant *frame_quant;   /* config.frame_quant or keyframe_quant: the step's records ([nframes]);
                                               NULL otherwise.  Replace them with daala_b200_kf_load_frame_quant,
                                               which also loads the tables derived from them */
  int32_t *haar_dc[3];                  /* config.haar_dc_quant: the DC chain's reconstructed DCs per plane, one entry per
                                           4x4 unit (leaf DCs at leaf origins), the three planes of a frame together
                                           (frame f of plane p at haar_dc[p] + f * (g0 + 2 g1), g = plane grid size) */
  int32_t *dc_index[3];                 /* and the index grids ([nframes][plane_h / 4][plane_w / 4]); else NULL */
  daala_b200_kf_sym_hdc *sym_hdc;       /* config.symbol_stream = 1 with haar_dc_quant, or 3: the step's keyframe DC
                                           records, the frames one after the other from index 0 (what io.sym_hdc
                                           receives, max_luma_blocks + max_chroma_blocks entries); else NULL */
} daala_b200_kf_buffers;

#define DAALA_B200_KF_LISTS 1
#define DAALA_B200_KF_FORWARD 2
#define DAALA_B200_KF_PVQ_LUMA 4
#define DAALA_B200_KF_INVERSE 8
#define DAALA_B200_KF_PVQ_CHROMA 16
#define DAALA_B200_KF_PVQ (DAALA_B200_KF_PVQ_LUMA | DAALA_B200_KF_PVQ_CHROMA)
#define DAALA_B200_KF_ALL 31
#define DAALA_B200_KF_SEARCH_ONLY 64   /* with _PVQ_*: only the persistent search kernels (measurement) */

daala_b200_kf *daala_b200_kf_create(const daala_b200_kf_config *cfg);   /* NULL on failure */
void daala_b200_kf_destroy(daala_b200_kf *kf);
/* The engine's last error message; with kf == NULL why this thread's last daala_b200_kf_create returned NULL. */
const char *daala_b200_kf_error(const daala_b200_kf *kf);
int daala_b200_kf_device_buffers(daala_b200_kf *kf, daala_b200_kf_buffers *out);
int daala_b200_kf_launches_per_step(const daala_b200_kf *kf);   /* kernel launches of one whole step */
/* Runs the selected phases on the engine's stream with inputs already in HBM (asynchronous);
   use_graph: replay the captured CUDA graph (DAALA_B200_KF_ALL only). */
int daala_b200_kf_run_device(daala_b200_kf *kf, int phases, int use_graph);
/* `reps` repetitions of the phases timed with CUDA events on the engine's stream; *ms = total. */
int daala_b200_kf_time_device(daala_b200_kf *kf, int phases, int use_graph, int reps, float *ms);
/* Host-side totals implied by block-size maps (sizes of the result arrays). */
int daala_b200_kf_count_blocks(const uint8_t *bsize, int nframes, long long frame_pitch, int bstride, int nhsb,
                               int nvsb, int sb_row0, int sb_rows, daala_b200_kf_totals *out);
/* Worst-case lengths of the symbol stream arrays of a batch with these totals: every block, every band, two bytes
   per coefficient. */
int daala_b200_kf_symbol_bounds(const daala_b200_kf_totals *t, int nframes, daala_b200_kf_sym_bounds *out);
/* With config.inter, DAALA_B200_KF_PVQ_LUMA selects the luma phase kernels.
   H2D of the inputs, the whole step, D2H of the requested outputs: enqueued, not waited for.  Every refusal returns
   cudaErrorInvalidValue with a message in daala_b200_kf_error, before anything is copied or launched: the device
   buffers, the reference-picture pool and what run_device replays are those of the last accepted step.  Submit
   refuses a NULL pixels plane, a NULL bsize (lossy engines), a NULL dering_level on a dering = 1 engine, a batch with
   more luma or chroma blocks than the engine's capacity (see max_blocks_div), a request for symbol stream outputs
   from an engine created without symbol_stream (sym_dc: without symbol_stream 2 or 3), a stream capacity below
   daala_b200_kf_symbol_bounds, a stream buffer that is not pinned host memory, or (config.inter) a NULL pred_pixels
   plane, luma_dc or chroma_dc (the last two are optional with symbol_stream 2 or 3), a late-skip output on an engine
   without late_skip, sym_late_skip without symbol_stream = 2, and sym_hdc on an engine without both
   symbol_stream = 1 and haar_dc_quant = 1 or symbol_stream = 3.  With config.inter_mc it refuses, the same
   way, a NULL mv_grid, ref_pixels plane or ref_slot, pred_pixels given, nrefs outside [1, mc_refs] and a slot outside
   [0, nrefs); with ref_resident = 1 it refuses instead ref_pixels given, nrefs other than 0, a slot outside
   [0, mc_refs) and a slot that holds no picture.  With config.mc_next the same checks cover ref_slot_next, and a NULL
   ref_slot_next or mv1_grid is refused; either given to an engine without mc_next is refused.  The step counts in
   `counts` the leaf corners whose vertex has a ref other than 0 or 1 (counts[19]; with mc_next other than 0, 1 or 2)
   and the corner windows (with the 6-tap filter's apron of -2..+3 pixels) that reach more than 64 luma / 32 chroma
   pixels outside the plane (counts[20]; with mc_next the window of the vector the corner reads, mv1 on NEXT
   vertices), where the reference encoder's result is undefined.  With config.frame_quant or keyframe_quant it
   refuses a NULL frame_quant and a record out of range (see daala_b200_kf_frame_quant); frame_quant given to an engine
   with neither is refused.  ll_coeffs, ll_blocks and ll_ref_slot_out are refused on an engine without
   config.lossless, and ll_ref_slot_out also without inter_mc, with an entry outside [-1, mc_refs) or with two frames
   naming one slot.  A lossless engine reads neither bsize nor totals, and returns none of the PVQ outputs. */
int daala_b200_kf_submit(daala_b200_kf *kf, const daala_b200_kf_io *io);
/* What submit derives on the host from the n records of a config.frame_quant step (no GPU involved, no validation):
   tbl[f][0][g] / tbl[f][1][g] (nullable) the luma / chroma deringing threshold of level g for frame f,
   (int)(OD_DERING_GAIN_TABLE[g] * q0^0.84182) and the same times 0.6 (reference src/encode.c:2694, :2822) with that
   frame's q0; the return value is the finishing pass's DC limit for the step, DAALA_B200_KF_FINISH_DC_LIMIT / the
   largest dc_quant over the records, planes and block sizes. */
int daala_b200_kf_frame_quant_derive(const daala_b200_kf_frame_quant *rec, int n, int32_t (*tbl)[2][6]);
/* config.frame_quant or keyframe_quant, for run_device without a submit: checks the [nframes] records as submit does
   and copies them into the engine's device buffers with what submit derives from them (each frame's deringing
   thresholds and its band quantisers max(1, q0 * pvq_qm_q4[pli][i] >> 4), which the PVQ kernels, the DC quantisers
   and the finishing pass read), on the engine's stream, and waits for the copies.  The finishing pass's DC limit is
   not changed (a submit sets it). */
int daala_b200_kf_load_frame_quant(daala_b200_kf *kf, const daala_b200_kf_frame_quant *rec);
/* The finishing pass (config.inter_finish, see daala_b200_kf_finish_io) on the last submitted step: H2D of the
   decisions and levels, the pass's kernels as one CUDA graph (captured at the first call; with config.inter_finish
   = 2 it includes the level search), D2H of the requested outputs; enqueued on the engine's stream like submit,
   waited for with daala_b200_kf_wait.  The step's outputs and its d / md planes are not modified (the decisions are
   applied to a plane of their own), so the pass may run any number of times after one step.  Refused with
   cudaErrorInvalidValue and a message in daala_b200_kf_error, before anything is copied or launched: an engine
   without inter_finish, no step submitted yet, a NULL decision array (neither form complete), both forms given, the
   stream form on an engine without symbol_stream 2 or 3, a skip value other than 0 or 1, a level above
   5, a |dc| above DAALA_B200_KF_FINISH_DC_LIMIT / DQ, (config.inter_finish = 2) a non-NULL dering_level, and a
   ref_slot_out on an engine without inter_mc, with an entry outside [-1, mc_refs) or with two frames naming one slot.
   With ref_slot_out the pass's last kernel copies each stored frame's reconstruction into its pool slot.  With the
   stream form the decisions are copied into staging buffers and the pass's first kernel scatters them into block
   order through the step's slot -> block map. */
int daala_b200_kf_finish(daala_b200_kf *kf, const daala_b200_kf_finish_io *io);
/* Enqueues on the engine's stream the copies of one frame-sized picture (planes[p]: [plane_h][plane_w] u8, the layout
   of one frame of daala_b200_kf_io.pixels) into slot `slot` of the reference-picture pool (config.inter_mc), with
   cudaMemcpyDefault: the source may be host memory or device memory of the engine's device, for example a keyframe
   engine's daala_b200_kf_buffers.pixels_out[p] + f * plane_h[p] * plane_w[p], which brings a GOP's keyframe into the
   pool without a host round trip (wait for that engine first: the copy runs on this engine's stream).  Host buffers must stay valid until daala_b200_kf_wait, as submit's.  Ordered by
   call order with submit and finish: a step submitted before the load reads the slot's previous picture.  Refused
   with cudaErrorInvalidValue and a message in daala_b200_kf_error, before anything is copied: an engine without
   inter_mc, a slot outside [0, mc_refs) and a NULL plane. */
int daala_b200_kf_pool_load(daala_b200_kf *kf, int slot, const uint8_t *const planes[3]);
int daala_b200_kf_wait(daala_b200_kf *kf);
int daala_b200_kf_encode(daala_b200_kf *kf, const daala_b200_kf_io *io);   /* submit + wait */
int daala_b200_device_copy(void *dst, const void *src, size_t bytes, int kind);  /* 0 H2D, 1 D2H, 2 D2D; synchronous */
void *daala_b200_host_alloc(size_t bytes);   /* pinned host memory */
void daala_b200_host_free(void *p);

/* ---- Motion compensation / block matching (8-bit references) ------------- */

/* One OBMC block: four corner motion vectors in 1/8 pel (rotational order:
   top-left, top-right, bottom-right, bottom-left; already scaled for the
   plane), outside corner `oc` and split state `s` as in od_mc_predict
   (reference src/mc.c:2006, src/state.c:627-671). */
typedef struct daala_b200_mc_block {
  int32_t mvx[4];
  int32_t mvy[4];
  uint16_t x0, y0;         /* block origin in the plane */
  uint8_t log_xblk, log_yblk;
  uint8_t oc, s;
} daala_b200_mc_block;

/* One block-matching candidate: square block of edge 1 << log_blk at (x0, y0),
   displaced by (mvx, mvy) 1/8 pel in the reference plane. */
typedef struct daala_b200_match_job {
  int32_t mvx, mvy;
  uint16_t x0, y0;
  uint8_t log_blk;
  uint8_t pad_[3];
} daala_b200_match_job;

/* OBMC prediction of `count` blocks into dst (od_state_pred_block's inner
   operation, src/state.c:627; od_mc_predict1fmv8_c + od_mc_blend_full(_split)8_c).
   `ref` points at pixel (0,0) of a reference plane with enough padding for the
   displaced (n+5)^2 windows (the reference keeps OD_BUFFER_PADDING = 96 px). */
int daala_b200_mc_predict_blocks(const uint8_t *ref, int ref_stride, uint8_t *dst, int dst_stride,
                                 const daala_b200_mc_block *blocks, int count, void *stream);
/* SAD (use_satd = 0) or SATD (1) of every job's interpolated reference block
   against the current frame: od_mv_est_bma_sad's inner operation
   (src/mcenc.c:2224) = mc_predict1fmv + od_mc_compute_sad8_c (:1333) or
   od_mc_compute_satd8_NxN_c (:1560-1612). */
int daala_b200_mc_match_candidates(const uint8_t *cur, int cur_stride, const uint8_t *ref, int ref_stride,
                                   const daala_b200_match_job *jobs, int count, int use_satd, int32_t *result,
                                   void *stream);
/* od_mv_est_bma_sad (static, src/mcenc.c:2224): the complete cost of a half-pel BMA candidate -- per plane
   the displaced block's single-MV prediction and its SAD against the current picture through od_enc_sad's
   clipping to the picture (src/mcenc.c:1615), chroma >> OD_MC_CHROMA_SCALE, summed.  (bx, by): luma position
   of the block (may be negative: BMA blocks are centred on grid points); (mvx, mvy): half-pel units;
   block edge = 8 << log_mvb_sz luma pixels (log_mvb_sz 0..3).  cur[p]: pixel (0,0) of the current picture's planes; ref[p]:
   pixel (0,0) of reference planes padded like state->ref_imgs (od_img_edge_ext).  nplanes = 3 with
   OD_MC_USE_CHROMA, else 1. */
typedef struct daala_b200_bma_job {
  int32_t bx, by, mvx, mvy, log_mvb_sz;
} daala_b200_bma_job;
int daala_b200_mv_bma_sad(const uint8_t *const cur[3], const int cur_stride[3], const uint8_t *const ref[3],
                          const int ref_stride[3], int pic_w, int pic_h, int nplanes,
                          const daala_b200_bma_job *jobs, int count, int32_t *result, void *stream);
/* od_mv_est_sad (static, src/mcenc.c:2267): the OBMC-based cost of `count` MV-grid blocks.  blocks[3 * q + p] is
   candidate q's block record in plane p (od_state_pred_block_from_setup, src/state.c:627: four corner MVs scaled
   for the plane, oc, s); prediction of every plane (od_mc_predict) + od_enc_sad against the current picture,
   chroma >> OD_MC_CHROMA_SCALE.  Planes as for daala_b200_mv_bma_sad. */
int daala_b200_mv_est_sad(const uint8_t *const cur[3], const int cur_stride[3], const uint8_t *const ref[3],
                          const int ref_stride[3], int pic_w, int pic_h, int nplanes,
                          const daala_b200_mc_block *blocks, int count, int32_t *result, void *stream);
/* Batched mc_predict1fmv: job q's block goes to dst + q*dst_pitch (row stride
   = block width).  log_yblk < 0: square blocks. */
int daala_b200_mc_predict1fmv_batch(const uint8_t *ref, int ref_stride, uint8_t *dst, int dst_pitch,
                                    const daala_b200_match_job *jobs, int count, int log_yblk, void *stream);
/* Blend of four packed predictions (mc_blend_full when s == 3, else
   mc_blend_full_split). */
int daala_b200_mc_blend_packed(const uint8_t *preds, int pitch, uint8_t *dst, int dst_stride, int oc, int s,
                               int log_xblk, int log_yblk, void *stream);

/* Library/device information.  Returns the number of usable CUDA devices. */
int daala_b200_device_count(void);
const char *daala_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* DAALA_B200_H */
