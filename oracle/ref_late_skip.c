/* oracle/ref_late_skip.c -- TEST INFRASTRUCTURE ONLY.
 * late_skip_driver.inc bound to the REAL reference functions, with the bindings of ref_pipeline.c and the reference's
 * od_compute_dist (oracle_ref_compute_dist, ref_hooks_encode.c).  The frame driver is included again under a prefix of
 * its own (oracle_ref_ls_), so that the late-skip driver can use its forward_plane; the exported name is
 * oracle_ref_ls_late_skip_plane.  Linked by late_skip.mk with the objects of _ref/libdaala_ref.so into
 * _ref/libdaala_ref_late_skip.so. */
#include "filter.h"
#include "dct.h"
#define PIPE(name) oracle_ref_ls_##name
#define X_FDCT2D(ln, y, ys, x, xs) (*OD_FDCT_2D_C[(ln) - 2])(y, ys, x, xs)
#define X_IDCT2D(ln, x, xs, y, ys) (*OD_IDCT_2D_C[(ln) - 2])(x, xs, y, ys)
#define X_PRE_SPLIT(c, stride, bs, h, v) od_prefilter_split(c, stride, bs, 0, h, v)
#define X_POST_SPLIT(c, stride, bs, h, v) od_postfilter_split(c, stride, bs, 0, 0, NULL, 0, h, v)
#define X_PRE_SBS(c, stride, nhsb, nvsb, xdec) od_apply_prefilter_frame_sbs(c, stride, nhsb, nvsb, xdec, xdec)
#define X_POST_SBS(c, stride, nhsb, nvsb, xdec) \
  od_apply_postfilter_frame_sbs(c, stride, nhsb, nvsb, xdec, xdec, 0, NULL, 0)
#include "partition.h"
int oracle_ref_pvq_theta(od_coeff *out, const od_coeff *x0, const od_coeff *r0,
 int n, int q0, od_coeff *y, int *itheta, int *max_theta, int *vk,
 int beta, double *skip_diff, int nodesync, int is_keyframe, int pli,
 const void *adapt, const int16_t *qm, const int16_t *qm_inv,
 double pvq_norm_lambda, int speed);
#define X_TO_CODING(dst, n, src, stride) od_raster_to_coding_order(dst, n, src, stride)
#define X_FROM_CODING(dst, stride, src, n) od_coding_order_to_raster(dst, stride, src, n)
#define X_PVQ_THETA(out, x0, r0, n, q, y, it, mt, k, beta, sd, kf, pli, qm, qmi, lam) \
  oracle_ref_pvq_theta(out, x0, r0, n, q, y, it, mt, k, beta, sd, 1, kf, pli, NULL, qm, qmi, lam, 1)
#include "intra.h"
#define X_HV_PRED(pred, d, w, bx, by, bsize, bstride, bs) \
  od_hv_intra_pred(pred, d, w, bx, by, (unsigned char *)(bsize), bstride, bs)
#define X_CFL_PRED(pred, n, luma, lw, bs, obs) od_resample_luma_coeffs(pred, n, luma, lw, 1, 1, bs, obs)
#include "ref_dering_vtbl.h"
#include <stdlib.h>
#define X_DERING_SEARCH(src, ss, ctmp, nhsb, nvsb, q, cq, qm, masking, lambda, cdf, levels) abort()
#define X_DERING(y, ys, x, xs, sbx, sby, nhsb, nvsb, xdec, dir, pli, bskip, ss, thr) \
  od_dering(oracle_dering_vtbl(), y, ys, x, xs, 8, 8, sbx, sby, nhsb, nvsb, xdec, dir, pli, bskip, ss, thr, \
   OD_DERING_CHECK_OVERLAP, OD_COEFF_SHIFT)
#include "pipeline_driver.inc"
double oracle_ref_compute_dist(od_coeff *x, od_coeff *y, int n, int qm, int use_activity_masking,
 int coded_quantizer);
/* enc->qm: OD_FLAT_QM (0) or OD_HVS_QM (1) */
#define X_DIST(x, y, n, flat, masking, cq) oracle_ref_compute_dist(x, y, n, (flat) ? 0 : 1, masking, cq)
#include "late_skip_driver.inc"
