/* tests/oracle_visits.c -- TEST INFRASTRUCTURE ONLY.
 * oracle/pipeline_driver.inc bound to the plain-C port exactly as oracle/port_pipeline.c binds it, except that
 * the first raster -> coding order conversion of every block (pvq_block's read of the coefficient plane at the
 * block's origin) is recorded.  oracle_visit_pvq_plane_rec then lists the leaf blocks of a plane in the order
 * the driver's pvq_recurse visits them -- the reference's od_encode_recursive order -- without touching the
 * oracle sources.  Built by tests/test_symbol_stream.py against oracle/libdaala_port.so. */
#include <stddef.h>
#include "port.h"
#include "port_pvq.h"

static const od_coeff *visit_plane;
static long visit_plane_len;
static int visit_stride;
static int32_t *visit_out;
static long visit_cap;
static long visit_n;

static void visit_to_coding(od_coeff *dst, int n, const od_coeff *src, int stride) {
  if (visit_plane && src >= visit_plane && src < visit_plane + visit_plane_len) {
    long off = (long)(src - visit_plane);
    if (visit_n < visit_cap) {
      visit_out[3 * visit_n + 0] = (int32_t)(off % visit_stride);
      visit_out[3 * visit_n + 1] = (int32_t)(off / visit_stride);
      visit_out[3 * visit_n + 2] = n;
    }
    visit_n++;
  }
  port_raster_to_coding_order(dst, n, src, stride);
}

#define PIPE(name) oracle_visit_##name
#define X_FDCT2D(ln, y, ys, x, xs) port_bin_fdct2d(ln, y, ys, x, xs)
#define X_IDCT2D(ln, x, xs, y, ys) port_bin_idct2d(ln, x, xs, y, ys)
#define X_PRE_SPLIT(c, stride, bs, h, v) port_prefilter_split(c, stride, bs, h, v)
#define X_POST_SPLIT(c, stride, bs, h, v) port_postfilter_split(c, stride, bs, h, v)
#define X_PRE_SBS(c, stride, nhsb, nvsb, xdec) port_apply_prefilter_frame_sbs(c, stride, nhsb, nvsb, xdec, xdec)
#define X_POST_SBS(c, stride, nhsb, nvsb, xdec) port_apply_postfilter_frame_sbs(c, stride, nhsb, nvsb, xdec, xdec)
#define X_TO_CODING(dst, n, src, stride) visit_to_coding(dst, n, src, stride)
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

/* Leaf blocks of plane `pli` in visit order: out[3*i + {0, 1, 2}] = x0, y0 (plane samples) and the block's
   edge n.  d is the plane's coefficients (quantised in place), h its height in samples.  Returns the number of
   blocks (only the first `cap` are written). */
long oracle_visits(od_coeff *d, int h, int nhsb, int nvsb, int xdec, int pli, const uint8_t *bsize, int bstride,
                   int q0, const int16_t *qm, const int16_t *qm_inv, const uint8_t *pvq_qm_q4, const od_coeff *luma_d,
                   int32_t *out, long cap) {
  visit_plane = d;
  visit_stride = (nhsb * 64) >> xdec;
  visit_plane_len = (long)visit_stride * h;
  visit_out = out;
  visit_cap = cap;
  visit_n = 0;
  oracle_visit_pvq_plane_rec(d, NULL, nhsb, nvsb, xdec, pli, bsize, bstride, q0, 1, 1, 0.147, qm, qm_inv, pvq_qm_q4,
                             NULL, pli == 0, luma_d, NULL, NULL);
  visit_plane = NULL;
  return visit_n;
}
