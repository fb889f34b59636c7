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
   kernels everywhere, 10 + c = alternative lanes-per-band geometries, 20/21/30/31 =
   register-cap (occupancy) variants (tuning). */
int daala_b200_pvq_encode_bands_mode(const daala_b200_pvq_params *prm, const uint32_t *band_list, int count,
                                     int nmax, int mode, void *stream);
/* Keyframe luma WITH the reference's H/V intra prediction (od_hv_intra_pred,
   src/intra.c:37; od_encode_compute_pred, src/encode.c:858): one warp per block runs gather,
   prediction from the quantised neighbours, every band, and the scatter back into
   coef_plane[0]; blocks wait for their top / left same-size neighbours through `done`
   (done[i] == epoch once block i is reconstructed).  `blocks` must list luma blocks only, in
   raster order of their origin per frame; dep_top / dep_left give the neighbour's block index or
   -1 (daala_b200/pvq.py: intra_dependencies).  Fills the same result arrays as the band kernels. */
int daala_b200_pvq_luma_intra(const daala_b200_pvq_params *prm, const int32_t *dep_top, const int32_t *dep_left,
                              int32_t *done, int epoch, int nblocks, void *stream);
/* Wave-synchronous form of the same computation: luma blocks sorted by dependency depth; for
   each wave (blocks [first, first+count) of one depth) the caller runs _intra_gather, the band
   kernels on the wave's slices of the band lists, _block_finish_range and
   _coding_order_scatter_range.  dep_top / dep_left only need their sign here. */
int daala_b200_pvq_intra_gather(const daala_b200_pvq_params *prm, const int32_t *dep_top, const int32_t *dep_left,
                                int first, int count, void *stream);
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

/* Band-granular wavefront (the default): od_hv_intra_pred (src/intra.c:37) couples band b of a block
   only to band b of the same-size top / left neighbour (row-0 bands 1/4/7: top, column-0 bands 2/5/8:
   left, bands 3/6: none, band 0: both).  For the entries of `band_list` ((block << 4) | band, all of
   one dependency depth >= 2) this writes the bands' slices of `ref` from the neighbours' `out`; the
   caller then runs daala_b200_pvq_encode_bands[_mode] on the same slice.  dep_top / dep_left: index of
   the neighbour block in prm->blocks or -1. */
int daala_b200_pvq_intra_band_ref(const daala_b200_pvq_params *prm, const int32_t *dep_top, const int32_t *dep_left,
                                  const uint32_t *band_list, int count, void *stream);
int daala_b200_pvq_block_finish_range(const daala_b200_pvq_params *prm, int first, int count, void *stream);
int daala_b200_coding_order_scatter_range(const daala_b200_pvq_params *prm, int first, int count, void *stream);
/* The same split by block size (chains only connect blocks of equal size): `ids` lists the
   blocks of one size in raster order.  _ids: one warp per block (used for 4x4 blocks);
   _class (bs = 1..4): one CTA per block, one warp per band.  The launches of different sizes are
   independent and may run on different streams. */
int daala_b200_pvq_luma_intra_ids(const daala_b200_pvq_params *prm, const int32_t *ids, int count,
                                  const int32_t *dep_top, const int32_t *dep_left, int32_t *done, int epoch,
                                  void *stream);
int daala_b200_pvq_luma_intra_class(const daala_b200_pvq_params *prm, const int32_t *ids, int count, int bs,
                                    const int32_t *dep_top, const int32_t *dep_left, int32_t *done, int epoch,
                                    void *stream);
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
   one persistent kernel with per-band acquire / release flags, chroma CfL + PVQ, iDCT + postfilters;
   one CUDA graph per engine.  Two engines give a double-buffered pipeline (submit one, wait for the
   other). */
typedef struct daala_b200_kf daala_b200_kf;

typedef struct daala_b200_kf_config {
  int pic_w, pic_h;            /* luma picture size; frames are padded to whole 64x64 superblocks */
  int nframes;                 /* frames per batch (1..255), independent keyframes of one geometry */
  int q0;                      /* state->quantizer */
  int use_masking;             /* activity masking (OD_PVQ_BETA, src/pvq.c:205) */
  int qm_stride;               /* OD_QM_STRIDE = 5456 */
  double pvq_norm_lambda;      /* enc->pvq_norm_lambda */
  uint8_t pvq_qm_q4[3][32];    /* state->pvq_qm_q4 */
  const int16_t *qm, *qm_inv;  /* HOST: state->qm / qm_inv, 2*qm_stride entries each (copied) */
  int sb_row0, sb_rows;        /* superblock rows of this rank's shard (sb_rows <= 0: whole frames) */
  int max_blocks_div;          /* 0/1: capacity for all-4x4 maps; d > 1: 1/d of that (saves HBM) */
  int persist_ctas_per_sm;     /* 0 = default */
  int split_free;              /* dependency-free bands as three phase kernels (setup / search / finish) with
                                  the band context in HBM records instead of the persistent kernel:
                                  0 = no, 1 = chroma, 2 = chroma and luma bands 3 / 6 */
  int dering;                  /* 1: the reconstruction goes through od_dering with the per-superblock levels of
                                  daala_b200_kf_io.dering_level (the final application of src/encode.c:2812-2842).
                                  2: the engine also SEARCHES the levels (src/encode.c:2708-2811: five filtered
                                  candidates + the unfiltered one scored by od_compute_dist + lambda * adaptive-CDF
                                  rate, decision per frame on the device) and returns them in
                                  daala_b200_kf_io.dering_level_out; needs coded_quantizer / qm_is_flat /
                                  dering_lambda below */
  int noref_prepass;           /* 1: the no-reference searches of every luma chain band run ahead of the chains in a
                                  fully parallel kernel (they do not depend on the prediction) */
  int level_chains;            /* luma intra chains: 0 = persistent kernel with a dependency queue, 1 = one
                                  level-synchronous kernel (phases separated by grid barriers); implies
                                  split_free = 2 */
  void *stream;                /* cudaStream_t to run on, or NULL: the engine creates its own */
  int coded_quantizer;         /* state->coded_quantizer (scale of od_compute_dist, src/encode.c:1221); dering == 2 */
  int qm_is_flat;              /* enc->qm == OD_FLAT_QM: od_compute_dist is the plain squared error; dering == 2 */
  double dering_lambda;        /* enc->dering_lambda (src/rate.c:1086); dering == 2 */
} daala_b200_kf_config;

typedef struct daala_b200_kf_totals {
  long long n_luma, luma_coefs, n_chroma, chroma_coefs;
} daala_b200_kf_totals;

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
} daala_b200_kf_io;

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
  uint32_t *luma_heads;                 /* row / column chain items ready from the start; counts[15] of them */
  uint32_t *luma_heads0;                /* band-0 items ready from the start; counts[16] of them */
  uint32_t *chroma_items[3];
  int16_t *luma_res, *chroma_res, *luma_y16, *chroma_y16;
  double *luma_skip_diff, *chroma_skip_diff;
  int32_t *chroma_flip;
  int max_luma_blocks, max_chroma_blocks;
  void *stream;
  long long bytes_allocated;
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
/* H2D of the inputs, the whole step, D2H of the requested outputs: enqueued, not waited for. */
int daala_b200_kf_submit(daala_b200_kf *kf, const daala_b200_kf_io *io);
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
