/* oracle/port.h -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C restatement ("port") of the xiph/daala per-block hot path, used by
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg as the
 * CHECKER.  Nothing in daala_b200/ may include, link or call this.
 * Pinned against the real reference (oracle/_ref/libdaala_ref.so, built from
 * the reference sources by oracle/Makefile) in tests/test_oracle_port.py.
 */
#ifndef DAALA_ORACLE_PORT_H
#define DAALA_ORACLE_PORT_H
#include <stdint.h>

typedef int32_t od_coeff;

/* port_dct.c -- src/dct.c */
void port_bin_fdct(int ln, od_coeff *y, const od_coeff *x, int xstride);
void port_bin_idct(int ln, od_coeff *x, int xstride, const od_coeff *y);
void port_bin_fdct2d(int ln, od_coeff *y, int ystride, const od_coeff *x, int xstride);
void port_haar(od_coeff *y, int ystride, const od_coeff *x, int xstride, int ln);
/* perceptual block distortion of the RDO loops (reference src/encode.c:1180) */
double port_compute_dist(const od_coeff *x, const od_coeff *y, int n, int qm_is_flat, int use_activity_masking,
 int coded_quantizer);
/* deringing of one superblock (oracle for the next hot-path row; reference src/dering.c) */
int port_dering_find_direction(const int16_t *img, int stride, int32_t *var, int coeff_shift);
void port_dering(int16_t *y, int ystride, const int16_t *x, int xstride, int nhb, int nvb, int sbx, int sby,
 int nhsb, int nvsb, int xdec, int dir[8][8], int pli, const unsigned char *bskip, int skip_stride, int threshold,
 int overlap, int coeff_shift);
void port_haar_inv(od_coeff *x, int xstride, const od_coeff *y, int ystride, int ln);
void port_bin_idct2d(int ln, od_coeff *x, int xstride, const od_coeff *y, int ystride);

/* port_filter.c -- src/filter.c */
void port_pre_filter4(od_coeff y[4], const od_coeff x[4]);
void port_post_filter4(od_coeff x[4], const od_coeff y[4]);
void port_pre_filter_n(int n, od_coeff *y, const od_coeff *x);
void port_post_filter_n(int n, od_coeff *x, const od_coeff *y);
void port_prefilter_split(od_coeff *c0, int stride, int bs, int hfilter, int vfilter);
void port_postfilter_split(od_coeff *c0, int stride, int bs, int hfilter, int vfilter);
void port_apply_prefilter_frame_sbs(od_coeff *c0, int stride, int nhsb, int nvsb, int xdec, int ydec);
void port_apply_postfilter_frame_sbs(od_coeff *c0, int stride, int nhsb, int nvsb, int xdec, int ydec);

/* port_partition.c -- src/partition.c */
void port_raster_to_coding_order(od_coeff *dst, int n, const od_coeff *src, int stride);
void port_coding_order_to_raster(od_coeff *dst, int stride, const od_coeff *src, int n);

/* port_mc.c -- src/mc.c, src/mcenc.c */
void port_mc_predict1fmv8(unsigned char *dst, const unsigned char *src, int systride, int32_t mvx,
 int32_t mvy, int log_xblk_sz, int log_yblk_sz);
void port_mc_blend_full8(unsigned char *dst, int dystride, const unsigned char *src[4],
 int log_xblk_sz, int log_yblk_sz);
void port_mc_blend_full_split8(unsigned char *dst, int dystride, const unsigned char *src[4], int oc,
 int s, int log_xblk_sz, int log_yblk_sz);
void port_mc_predict(unsigned char *dst, int dystride, const unsigned char *src, int systride,
 const int32_t mvx[4], const int32_t mvy[4], int oc, int s, int log_xblk_sz, int log_yblk_sz);
int32_t port_mc_compute_sad8(const unsigned char *src, int systride, const unsigned char *ref,
 int dystride, int w, int h);
int32_t port_mc_compute_satd8(int ln, const unsigned char *src, int systride, const unsigned char *ref,
 int rystride);

/* port_tf.c -- src/tf.c, src/intra.c */
void port_tf_up_h_lp(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int dx, int n);
void port_tf_up_v_lp(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int dy, int n);
void port_tf_up_hv_lp(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int dx, int dy, int n);
void port_tf_up_hv(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int n);
void port_tf_down_hv(od_coeff *dst, int dstride, const od_coeff *src, int sstride, int n);
void port_hv_intra_pred(od_coeff *pred, const od_coeff *d, int w, int bx, int by,
 const unsigned char *bsize, int bstride, int bs);
void port_resample_luma_coeffs_420(od_coeff *chroma_pred, int cpstride, const od_coeff *decoded_luma,
 int dlstride, int bs, int luma_is_4x4);

#endif
