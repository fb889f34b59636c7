/* oracle/ref_hooks_haar_dc.c -- TEST INFRASTRUCTURE ONLY.
 * The keyframe DC driver of the engine's haar_dc_quant tests (tests/haar_dc_oracle.py).  Compiles the reference's
 * src/encode.c in place to reach its statics, so haar_dc.mk links it into a library of its own with the reference
 * build's objects other than the TUs that include encode.c too (ref_hooks_encode.c) or call into them
 * (ref_pipeline.c). */
#include "encode.c"

/* The superblock DC predictor of od_quantize_haar_dc_sb (src/encode.c:1563-1582) from sb_dc_mem, restated only to
   recover the coded index of a superblock DC (the reference's own call below does the quantisation). */
static od_coeff drv_sb_dc_pred(const od_coeff *m, int nhsb, int bx, int by, int has_ur) {
  if (by > 0 && bx > 0) {
    if (has_ur) {
      return (22*m[by*nhsb + bx - 1] - 9*m[(by - 1)*nhsb + bx - 1] + 15*m[(by - 1)*nhsb + bx]
       + 4*m[(by - 1)*nhsb + bx + 1] + 16) >> 5;
    }
    return (23*m[by*nhsb + bx - 1] - 10*m[(by - 1)*nhsb + bx - 1] + 19*m[(by - 1)*nhsb + bx] + 16) >> 5;
  }
  if (by > 0) return m[(by - 1)*nhsb + bx];
  if (bx > 0) return m[by*nhsb + bx - 1];
  return 0;
}

static int drv_dc_quant(daala_enc_ctx *enc, int pli) {
  return OD_MAXI(1, enc->state.quantizer*enc->state.pvq_qm_q4[pli][od_qm_get_index(OD_NBSIZES - 1, 0)] >> 4);
}

/* The split-node part of od_encode_recursive (src/encode.c:1660-1787) for a keyframe: od_quantize_haar_dc_level on
   every split node depth-first, the gradients passed by value.  The node's three indices are recovered from what the
   reference left in d: OD_HAAR_KERNEL with the middle terms swapped undoes the call's own kernel (src/tf.h:27-33),
   giving x[1..3] = quant * ac_quant (+ the gradient terms). */
static void drv_recursive(daala_enc_ctx *enc, od_mb_enc_ctx *ctx, int pli, int bx, int by, int bsi, int xdec,
 od_coeff hgrad, od_coeff vgrad, int32_t *idx, int istride) {
  int obs;
  int bs;
  int w;
  int ln;
  int dc_quant;
  int acq0;
  int acq1;
  od_coeff h0;
  od_coeff v0;
  od_coeff x0;
  od_coeff x1;
  od_coeff x2;
  od_coeff x3;
  od_coeff *d;
  obs = OD_BLOCK_SIZE4x4(enc->state.bsize, enc->state.bstride, bx << bsi, by << bsi);
  bs = OD_MAXI(obs, xdec);
  if (bs == bsi) return;
  h0 = hgrad;
  v0 = vgrad;
  od_quantize_haar_dc_level(enc, ctx, pli, 2*bx, 2*by, bsi - 1, xdec, &hgrad, &vgrad);
  w = enc->state.frame_width >> xdec;
  ln = bsi - 1 - xdec + 2;
  d = ctx->d[pli];
  x0 = d[((2*by) << ln)*w + ((2*bx) << ln)];
  x1 = d[((2*by) << ln)*w + ((2*bx + 1) << ln)];
  x2 = d[((2*by + 1) << ln)*w + ((2*bx) << ln)];
  x3 = d[((2*by + 1) << ln)*w + ((2*bx + 1) << ln)];
  OD_HAAR_KERNEL(x0, x2, x1, x3);
  dc_quant = drv_dc_quant(enc, pli);
  acq0 = (dc_quant*OD_DC_QM[bsi - 1 - xdec][0] + 8) >> 4;
  acq1 = (dc_quant*OD_DC_QM[bsi - 1 - xdec][1] + 8) >> 4;
  idx[(((2*by) << ln) >> 2)*istride + (((2*bx + 1) << ln) >> 2)] = (x1 - h0/5)/acq0;
  idx[(((2*by + 1) << ln) >> 2)*istride + (((2*bx) << ln) >> 2)] = (x2 - v0/5)/acq0;
  idx[(((2*by + 1) << ln) >> 2)*istride + (((2*bx + 1) << ln) >> 2)] = x3/acq1;
  drv_recursive(enc, ctx, pli, 2*bx + 0, 2*by + 0, bsi - 1, xdec, hgrad, vgrad, idx, istride);
  drv_recursive(enc, ctx, pli, 2*bx + 1, 2*by + 0, bsi - 1, xdec, hgrad, vgrad, idx, istride);
  drv_recursive(enc, ctx, pli, 2*bx + 0, 2*by + 1, bsi - 1, xdec, hgrad, vgrad, idx, istride);
  drv_recursive(enc, ctx, pli, 2*bx + 1, 2*by + 1, bsi - 1, xdec, hgrad, vgrad, idx, istride);
}

/* The keyframe DC chain of od_encode_coefficients (src/encode.c:2604-2656, the final pass) on a real encoder of
   pic_w x pic_h (4:2:0): od_adapt_ctx_reset, then per superblock in raster order, planes 0..2 inside, the reference's
   od_compute_dcts (lossy), od_quantize_haar_dc_sb (has_ur = sby > 0 && sbx < nhsb - 1, gradients from 0) and
   od_quantize_haar_dc_level on every split node in od_encode_recursive's order.  The PVQ coding between the DC calls
   reads no DC symbol model and writes no DC of its plane, so it is left out.
   src: frame-sized planes Y, U, V one after the other (u8); ctmp = (src - 128) << OD_COEFF_SHIFT and
   od_apply_prefilter_frame_sbs, as od_encode_coefficients prepares it.  bsize: [nvsb * 8][nhsb * 8] (one byte per
   8x8 luma unit).  quantizer, pvq_qm_q4 [3][OD_QM_SIZE] and pvq_norm_lambda: the frame's settings.
   Outputs (frame-sized planes Y U V, int32): d_pre the `d` planes after od_compute_dcts (the unquantised Haar DC
   pyramid), d_post the same after the DC chain (every leaf DC final); idx ([plane_h / 4][plane_w / 4] per plane) the
   signed coded indices: a superblock's at its origin, a split node's three at the origins of its children 1..3,
   0 elsewhere.  Returns 0, or < 0 when the encoder cannot be created. */
int oracle_ref_haar_dc_frame(int pic_w, int pic_h, const unsigned char *src, const unsigned char *bsize, int quantizer,
 const unsigned char *pvq_qm_q4, double pvq_norm_lambda, int32_t *d_pre, int32_t *d_post, int32_t *idx) {
  daala_info info;
  daala_enc_ctx *enc;
  od_state *state;
  od_mb_enc_ctx mbctx;
  size_t off[3];
  size_t ioff[3];
  int fw;
  int fh;
  int nhsb;
  int nvsb;
  int pli;
  int sbx;
  int sby;
  int x;
  int y;
  daala_info_init(&info);
  info.pic_width = pic_w;
  info.pic_height = pic_h;
  info.timebase_numerator = 30;
  info.timebase_denominator = 1;
  info.frame_duration = 1;
  info.pixel_aspect_numerator = 1;
  info.pixel_aspect_denominator = 1;
  info.nplanes = 3;
  info.plane_info[0].xdec = info.plane_info[0].ydec = 0;
  info.plane_info[1].xdec = info.plane_info[1].ydec = 1;
  info.plane_info[2].xdec = info.plane_info[2].ydec = 1;
  info.keyframe_rate = 256;
  enc = daala_encode_create(&info);
  if (enc == NULL) return -1;
  state = &enc->state;
  state->quantizer = quantizer;
  enc->pvq_norm_lambda = pvq_norm_lambda;
  memcpy(state->pvq_qm_q4, pvq_qm_q4, 3*OD_QM_SIZE);
  fw = state->frame_width;
  fh = state->frame_height;
  nhsb = state->nhsb;
  nvsb = state->nvsb;
  for (y = 0; y < nvsb*8; y++) {
    for (x = 0; x < nhsb*8; x++) state->bsize[y*state->bstride + x] = bsize[(size_t)y*nhsb*8 + x];
  }
  od_adapt_ctx_reset(&state->adapt, 1);
  od_ec_enc_reset(&enc->ec);
  off[0] = 0;
  off[1] = (size_t)fw*fh;
  off[2] = off[1] + (size_t)(fw >> 1)*(fh >> 1);
  ioff[0] = 0;
  ioff[1] = off[1] >> 4;
  ioff[2] = off[2] >> 4;
  OD_CLEAR(&mbctx, 1);
  mbctx.is_keyframe = 1;
  mbctx.use_haar_wavelet = 0;
  mbctx.d = state->dtmp;
  for (pli = 0; pli < 3; pli++) {
    int xdec = state->info.plane_info[pli].xdec;
    int ydec = state->info.plane_info[pli].ydec;
    int w = fw >> xdec;
    int h = fh >> ydec;
    for (y = 0; y < h; y++) {
      for (x = 0; x < w; x++) {
        state->ctmp[pli][y*w + x] = (src[off[pli] + (size_t)y*w + x] - 128) << OD_COEFF_SHIFT;
      }
    }
    od_apply_prefilter_frame_sbs(state->ctmp[pli], w, nhsb, nvsb, xdec, ydec);
    memset(idx + ioff[pli], 0, sizeof(*idx)*(size_t)(w >> 2)*(h >> 2));
  }
  for (sby = 0; sby < nvsb; sby++) {
    for (sbx = 0; sbx < nhsb; sbx++) {
      for (pli = 0; pli < 3; pli++) {
        int xdec = state->info.plane_info[pli].xdec;
        int ydec = state->info.plane_info[pli].ydec;
        int w = fw >> xdec;
        int ln = OD_LOG_BSIZE_MAX - xdec;
        int n = 1 << ln;
        int bo = (sby << ln)*w + (sbx << ln);
        int has_ur = sby > 0 && sbx < nhsb - 1;
        od_coeff *d = state->dtmp[pli];
        od_coeff hgrad;
        od_coeff vgrad;
        od_coeff pred;
        int i;
        int j;
        hgrad = vgrad = 0;
        mbctx.c = state->ctmp[pli];
        mbctx.mc = state->mctmp[pli];
        mbctx.md = state->mdtmp[pli];
        mbctx.l = state->lbuf[pli];
        od_compute_dcts(enc, &mbctx, pli, sbx, sby, OD_NBSIZES - 1, xdec, ydec, 0);
        for (i = 0; i < n; i++) {
          for (j = 0; j < n; j++) d_pre[off[pli] + bo + (size_t)i*w + j] = d[bo + i*w + j];
        }
        pred = drv_sb_dc_pred(state->sb_dc_mem[pli], nhsb, sbx, sby, has_ur);
        od_quantize_haar_dc_sb(enc, &mbctx, pli, sbx, sby, xdec, ydec, has_ur, &hgrad, &vgrad);
        idx[ioff[pli] + (size_t)((sby << ln) >> 2)*(w >> 2) + ((sbx << ln) >> 2)] =
         (d[bo] - pred)/drv_dc_quant(enc, pli);
        drv_recursive(enc, &mbctx, pli, sbx, sby, OD_NBSIZES - 1, xdec, hgrad, vgrad, idx + ioff[pli], w >> 2);
        for (i = 0; i < n; i++) {
          for (j = 0; j < n; j++) d_post[off[pli] + bo + (size_t)i*w + j] = d[bo + i*w + j];
        }
      }
    }
  }
  daala_encode_free(enc);
  return 0;
}

/* The WHOLE reference encoder on one 4:2:0 8-bit picture (frame-sized planes Y, U, V one after the other, pic_w x
   pic_h of them read with the frame's strides) coded as a keyframe through the public API at OD_SET_QUANT quant and
   OD_SET_COMPLEXITY complexity.  Exports what the final pass used: the block-size map (bsize_out, [nvsb * 8][nhsb * 8]),
   the `d` planes it left in state.dtmp (d_out, frame-sized planes Y U V), and its quantizer (quantizer_out,
   state.quantizer), pvq_qm_q4 (q4_out, [3][OD_QM_SIZE]) and pvq_norm_lambda (lambda_out).  The leaf DCs of d_out are the
   final-pass DC chain's: od_pvq_encode codes no keyframe DC and od_block_encode stores scalar_out[0] = dblock[0]
   whatever the skip decision (src/encode.c:1376-1377).  Returns 0, or < 0 on an encoder error. */
int oracle_ref_haar_dc_encode_keyframe(int pic_w, int pic_h, const unsigned char *src, int quant, int complexity,
 unsigned char *bsize_out, int32_t *d_out, int *quantizer_out, unsigned char *q4_out, double *lambda_out) {
  daala_info info;
  daala_enc_ctx *enc;
  daala_image img;
  daala_packet op;
  size_t off[3];
  int fw;
  int fh;
  int pli;
  int i;
  int j;
  int ret;
  daala_info_init(&info);
  info.pic_width = pic_w;
  info.pic_height = pic_h;
  info.timebase_numerator = 30;
  info.timebase_denominator = 1;
  info.frame_duration = 1;
  info.pixel_aspect_numerator = 1;
  info.pixel_aspect_denominator = 1;
  info.nplanes = 3;
  info.plane_info[0].xdec = info.plane_info[0].ydec = 0;
  info.plane_info[1].xdec = info.plane_info[1].ydec = 1;
  info.plane_info[2].xdec = info.plane_info[2].ydec = 1;
  info.keyframe_rate = 1;
  enc = daala_encode_create(&info);
  if (enc == NULL) return -1;
  daala_encode_ctl(enc, OD_SET_QUANT, &quant, sizeof(quant));
  daala_encode_ctl(enc, OD_SET_COMPLEXITY, &complexity, sizeof(complexity));
  fw = enc->state.frame_width;
  fh = enc->state.frame_height;
  off[0] = 0;
  off[1] = (size_t)fw*fh;
  off[2] = off[1] + (size_t)(fw >> 1)*(fh >> 1);
  img.nplanes = 3;
  img.width = pic_w;
  img.height = pic_h;
  for (pli = 0; pli < 3; pli++) {
    img.planes[pli].data = (unsigned char *)src + off[pli];
    img.planes[pli].xdec = img.planes[pli].ydec = pli > 0;
    img.planes[pli].xstride = 1;
    img.planes[pli].ystride = fw >> (pli > 0);
    img.planes[pli].bitdepth = 8;
  }
  ret = daala_encode_img_in(enc, &img, 1);
  if (ret < 0 || daala_encode_packet_out(enc, 1, &op) <= 0) {
    daala_encode_free(enc);
    return ret < 0 ? ret : -2;
  }
  for (i = 0; i < enc->state.nvsb*8; i++) {
    for (j = 0; j < enc->state.nhsb*8; j++) {
      bsize_out[(size_t)i*enc->state.nhsb*8 + j] = enc->state.bsize[i*enc->state.bstride + j];
    }
  }
  for (pli = 0; pli < 3; pli++) {
    size_t n = (size_t)(fw >> (pli > 0))*(fh >> (pli > 0));
    for (i = 0; i < (int)n; i++) d_out[off[pli] + i] = enc->state.dtmp[pli][i];
  }
  *quantizer_out = enc->state.quantizer;
  memcpy(q4_out, enc->state.pvq_qm_q4, 3*OD_QM_SIZE);
  *lambda_out = enc->pvq_norm_lambda;
  daala_encode_free(enc);
  return 0;
}
