/* oracle/port_late_skip.c -- TEST INFRASTRUCTURE ONLY.
 * late_skip_driver.inc bound to the plain-C port, with the port's bindings of port_pipeline.c and port_compute_dist.
 * The frame driver is included again under a prefix of its own (oracle_port_ls_), so that the late-skip driver can
 * use its forward_plane; the exported name is oracle_port_ls_late_skip_plane. */
#include "port.h"
#define PIPE(name) oracle_port_ls_##name
#define X_FDCT2D(ln, y, ys, x, xs) port_bin_fdct2d(ln, y, ys, x, xs)
#define X_IDCT2D(ln, x, xs, y, ys) port_bin_idct2d(ln, x, xs, y, ys)
#define X_PRE_SPLIT(c, stride, bs, h, v) port_prefilter_split(c, stride, bs, h, v)
#define X_POST_SPLIT(c, stride, bs, h, v) port_postfilter_split(c, stride, bs, h, v)
#define X_PRE_SBS(c, stride, nhsb, nvsb, xdec) port_apply_prefilter_frame_sbs(c, stride, nhsb, nvsb, xdec, xdec)
#define X_POST_SBS(c, stride, nhsb, nvsb, xdec) port_apply_postfilter_frame_sbs(c, stride, nhsb, nvsb, xdec, xdec)
#include "port_pvq.h"
#define X_TO_CODING(dst, n, src, stride) port_raster_to_coding_order(dst, n, src, stride)
#define X_FROM_CODING(dst, stride, src, n) port_coding_order_to_raster(dst, stride, src, n)
#define X_PVQ_THETA(out, x0, r0, n, q, y, it, mt, k, beta, sd, kf, pli, qm, qmi, lam) \
  port_pvq_theta(out, x0, r0, n, q, y, it, mt, k, beta, sd, kf, pli, qm, qmi, lam)
#define X_HV_PRED(pred, d, w, bx, by, bsize, bstride, bs) port_hv_intra_pred(pred, d, w, bx, by, bsize, bstride, bs)
#define X_CFL_PRED(pred, n, luma, lw, bs, obs) port_resample_luma_coeffs_420(pred, n, luma, lw, bs, (obs) == 0)
#include <stdlib.h>
#define X_DERING_SEARCH(src, ss, ctmp, nhsb, nvsb, q, cq, qm, masking, lambda, cdf, levels) abort()
#define X_DERING(y, ys, x, xs, sbx, sby, nhsb, nvsb, xdec, dir, pli, bskip, ss, thr) \
  port_dering(y, ys, x, xs, 8, 8, sbx, sby, nhsb, nvsb, xdec, dir, pli, bskip, ss, thr, 1, 4)
#include "pipeline_driver.inc"
#define X_DIST(x, y, n, flat, masking, cq) port_compute_dist(x, y, n, flat, masking, cq)
#include "late_skip_driver.inc"
