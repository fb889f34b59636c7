/* oracle/ref_hooks_encode.c -- TEST INFRASTRUCTURE ONLY.
 * Compiles the reference's src/encode.c in place (see ref_hooks_pvq.c). */
#include "encode.c"
#include "ref_dering_vtbl.h"

/* od_compute_dist (static, src/encode.c:1180) on a minimal encoder context: only enc->qm,
   enc->use_activity_masking and enc->state.coded_quantizer are read. */
double oracle_ref_compute_dist(od_coeff *x, od_coeff *y, int n, int qm, int use_activity_masking,
 int coded_quantizer) {
  daala_enc_ctx *enc;
  double d;
  enc = (daala_enc_ctx *)calloc(1, sizeof(*enc));
  enc->qm = qm;
  enc->use_activity_masking = use_activity_masking;
  enc->state.coded_quantizer = coded_quantizer;
  d = od_compute_dist(enc, x, y, n);
  free(enc);
  return d;
}

/* The WHOLE reference encoder on one 4:2:0 8-bit picture coded as a keyframe, through the public API
   (include/daala/daalaenc.h), exporting what its RDO decided: the block-size map (one byte per 8x8
   luma unit, [nvsb*8][nhsb*8]), the deringing level per superblock ([nvsb][nhsb]) and the size and a
   checksum of the coded packet.  Gives tests real block-size decisions instead of synthetic quadtrees. */
int oracle_ref_encode_keyframe(int w, int h, unsigned char *y, unsigned char *u, unsigned char *v,
 int quant, int complexity, unsigned char *bsize_out, unsigned char *dering_out, long *packet_bytes,
 unsigned *packet_sum) {
  daala_info info;
  daala_enc_ctx *enc;
  daala_image img;
  daala_packet op;
  int pli;
  int i;
  int j;
  int ret;
  daala_info_init(&info);
  info.pic_width = w;
  info.pic_height = h;
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
  img.nplanes = 3;
  img.width = w;
  img.height = h;
  for (pli = 0; pli < 3; pli++) {
    img.planes[pli].data = pli == 0 ? y : pli == 1 ? u : v;
    img.planes[pli].xdec = img.planes[pli].ydec = pli > 0;
    img.planes[pli].xstride = 1;
    img.planes[pli].ystride = pli == 0 ? w : (w + 1) >> 1;
    img.planes[pli].bitdepth = 8;
  }
  ret = daala_encode_img_in(enc, &img, 1);
  if (ret < 0) {
    daala_encode_free(enc);
    return ret;
  }
  ret = daala_encode_packet_out(enc, 1, &op);
  if (ret <= 0) {
    daala_encode_free(enc);
    return -2;
  }
  *packet_bytes = op.bytes;
  *packet_sum = 0;
  for (i = 0; i < op.bytes; i++) *packet_sum = *packet_sum*31 + op.packet[i];
  for (i = 0; i < enc->state.nvsb*8; i++) {
    for (j = 0; j < enc->state.nhsb*8; j++) {
      bsize_out[i*enc->state.nhsb*8 + j] = enc->state.bsize[i*enc->state.bstride + j];
    }
  }
  for (i = 0; i < enc->state.nvsb*enc->state.nhsb; i++) {
    dering_out[i] = enc->state.dering_level ? enc->state.dering_level[i] : 0;
  }
  daala_encode_free(enc);
  return 0;
}

/* Multi-frame variant (keyframe + P frames) returning every packet's size and checksum: the
   reference side of the drop-in link test (dropin_main.c). */
#include "daala/daaladec.h"
#define ENCODE_FRAMES_NAME oracle_ref_encode_frames
#include "encode_frames.inc"

/* The deringing level search of od_encode_coefficients (src/encode.c:2680-2811) as a driver over the
   reference's own od_compute_dist, od_dering (with the function table of this build, ref_dering_vtbl.h),
   od_encode_cdf_cost and od_encode_cdf_adapt: luma
   reconstruction `ctmp` (od_coeff, stride nhsb*64) against the 8-bit source.  bskip may be NULL (nothing
   skipped).  cdf is state->adapt.dering_cdf ([11][6], in/out); dist_out (nullable) receives the six
   distortions of every superblock, [6][nvsb*nhsb]; levels the decisions. */
int oracle_ref_dering_search(unsigned char *src, int src_stride, const od_coeff *ctmp, int nhsb, int nvsb,
 int quantizer, int coded_quantizer, int qm, int use_activity_masking, int is_keyframe, double dering_lambda,
 const unsigned char *bskip, int skip_stride, uint16_t *cdf, int increment, unsigned char *levels,
 double *dist_out) {
  daala_enc_ctx *enc;
  od_state *state;
  int16_t *etmp;
  unsigned char *noskip;
  int w;
  int nsb;
  int sb;
  int k;
  double base;
  enc = (daala_enc_ctx *)calloc(1, sizeof(*enc));
  state = &enc->state;
  enc->qm = qm;
  enc->use_activity_masking = use_activity_masking;
  state->coded_quantizer = coded_quantizer;
  od_ec_enc_init(&enc->ec, 1 << 16);
  w = nhsb*OD_BSIZE_MAX;
  nsb = nhsb*nvsb;
  etmp = (int16_t *)malloc(sizeof(*etmp)*w*nvsb*OD_BSIZE_MAX);
  for (k = 0; k < w*nvsb*OD_BSIZE_MAX; k++) etmp[k] = (int16_t)ctmp[k];
  noskip = NULL;
  if (bskip == NULL) {
    skip_stride = nhsb*16;
    noskip = (unsigned char *)calloc((size_t)skip_stride*nvsb*16, 1);
    bskip = noskip;
  }
  base = pow(quantizer, 0.84182);
  for (sb = 0; sb < nsb; sb++) {
    od_coeff orig[OD_BSIZE_MAX*OD_BSIZE_MAX];
    od_coeff cand[OD_BSIZE_MAX*OD_BSIZE_MAX];
    int16_t filt[OD_BSIZE_MAX*OD_BSIZE_MAX];
    int dir[OD_DERING_NBLOCKS][OD_DERING_NBLOCKS];
    double score[OD_DERING_LEVELS];
    const unsigned char *sk;
    int sbx;
    int sby;
    int gi;
    int any;
    int c;
    int best;
    sbx = sb%nhsb;
    sby = sb/nhsb;
    sk = bskip + sby*16*skip_stride + sbx*16;
    any = 0;
    for (k = 0; k < 256; k++) any |= !sk[(k >> 4)*skip_stride + (k & 15)];
    levels[sb] = 0;
    if (dist_out) for (gi = 0; gi < OD_DERING_LEVELS; gi++) dist_out[gi*nsb + sb] = 0;
    if (!any) continue;
    od_ref_buf_to_coeff(state, orig, OD_BSIZE_MAX, 0, src + sby*OD_BSIZE_MAX*src_stride + sbx*OD_BSIZE_MAX,
     1, src_stride, OD_BSIZE_MAX, OD_BSIZE_MAX);
    c = 0;
    if (is_keyframe) {
      int up;
      int left;
      up = left = sby > 0 ? levels[sb - nhsb] : 0;
      if (sbx > 0) {
        left = levels[sb - 1];
        if (sby == 0) up = left;
      }
      c = up + left;
    }
    for (gi = 0; gi < OD_DERING_LEVELS; gi++) {
      double d;
      if (gi == 0) {
        for (k = 0; k < OD_BSIZE_MAX*OD_BSIZE_MAX; k++) {
          cand[k] = ctmp[(sby*OD_BSIZE_MAX + (k >> 6))*w + sbx*OD_BSIZE_MAX + (k & 63)];
        }
      }
      else {
        od_dering(oracle_dering_vtbl(), filt, OD_BSIZE_MAX, etmp + sby*OD_BSIZE_MAX*w + sbx*OD_BSIZE_MAX, w,
         OD_DERING_NBLOCKS, OD_DERING_NBLOCKS, sbx, sby, nhsb, nvsb, 0, dir, 0, (unsigned char *)sk, skip_stride,
         (int)(OD_DERING_GAIN_TABLE[gi]*base), OD_DERING_CHECK_OVERLAP, OD_COEFF_SHIFT);
        for (k = 0; k < OD_BSIZE_MAX*OD_BSIZE_MAX; k++) cand[k] = filt[k];
      }
      d = od_compute_dist(enc, orig, cand, OD_BSIZE_MAX);
      if (dist_out) dist_out[gi*nsb + sb] = d;
      score[gi] = d + dering_lambda*od_encode_cdf_cost(gi, cdf + c*OD_DERING_LEVELS, OD_DERING_LEVELS);
    }
    best = 0;
    for (gi = 1; gi < OD_DERING_LEVELS; gi++) if (score[gi] < score[best]) best = gi;
    levels[sb] = best;
    od_encode_cdf_adapt(&enc->ec, best, cdf + c*OD_DERING_LEVELS, OD_DERING_LEVELS, increment);
  }
  od_ec_enc_clear(&enc->ec);
  free(noskip);
  free(etmp);
  free(enc);
  return 0;
}

/* The quantizer settings the reference encoder itself uses for a keyframe followed by one P frame, through the
   public API: OD_SET_QUANT = quant, OD_SET_ACTIVITY_MASKING = masking, OD_SET_QM = qm (OD_FLAT_QM / OD_HVS_QM), on a
   mid-grey w x h picture (rate control is off, so nothing here depends on the content).  After each frame is
   coded, f = 0 (keyframe) / 1 (P frame), it reads back from the encoder context: quantizer[f] and
   coded_quantizer[f] (state.quantizer / coded_quantizer), pvq_qm_q4[f][3][OD_QM_SIZE], qm_out[f] / qm_inv_out[f]
   ([OD_QM_BUFFER_SIZE] each), pvq_norm_lambda[f] and dering_lambda[f]. */
int oracle_ref_encoder_settings(int w, int h, int quant, int masking, int qm, int *quantizer, int *coded_quantizer,
 unsigned char *pvq_qm_q4, int16_t *qm_out, int16_t *qm_inv_out, double *pvq_norm_lambda, double *dering_lambda) {
  daala_info info;
  daala_enc_ctx *enc;
  daala_image img;
  daala_packet op;
  unsigned char *planes[3];
  int pli;
  int f;
  int ret;
  daala_info_init(&info);
  info.pic_width = w;
  info.pic_height = h;
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
  if (daala_encode_ctl(enc, OD_SET_QUANT, &quant, sizeof(quant)) != OD_SUCCESS
   || daala_encode_ctl(enc, OD_SET_ACTIVITY_MASKING, &masking, sizeof(masking)) != OD_SUCCESS
   || daala_encode_ctl(enc, OD_SET_QM, &qm, sizeof(qm)) != OD_SUCCESS) {
    daala_encode_free(enc);
    return -2;
  }
  img.nplanes = 3;
  img.width = w;
  img.height = h;
  ret = 0;
  for (pli = 0; pli < 3; pli++) {
    planes[pli] = (unsigned char *)malloc((size_t)w*h);
    memset(planes[pli], 128, (size_t)w*h);
    img.planes[pli].data = planes[pli];
    img.planes[pli].xdec = img.planes[pli].ydec = pli > 0;
    img.planes[pli].xstride = 1;
    img.planes[pli].ystride = pli == 0 ? w : (w + 1) >> 1;
    img.planes[pli].bitdepth = 8;
  }
  for (f = 0; f < 2 && ret == 0; f++) {
    if (daala_encode_img_in(enc, &img, 1) < 0) ret = -3;
    else if (daala_encode_packet_out(enc, f == 1, &op) <= 0) ret = -4;
    else if ((f == 0) != (enc->state.frame_type == OD_I_FRAME)) ret = -5;
    else {
      quantizer[f] = enc->state.quantizer;
      coded_quantizer[f] = enc->state.coded_quantizer;
      memcpy(pvq_qm_q4 + f*3*OD_QM_SIZE, enc->state.pvq_qm_q4, 3*OD_QM_SIZE);
      memcpy(qm_out + f*OD_QM_BUFFER_SIZE, enc->state.qm, sizeof(*qm_out)*OD_QM_BUFFER_SIZE);
      memcpy(qm_inv_out + f*OD_QM_BUFFER_SIZE, enc->state.qm_inv, sizeof(*qm_inv_out)*OD_QM_BUFFER_SIZE);
      pvq_norm_lambda[f] = enc->pvq_norm_lambda;
      dering_lambda[f] = enc->dering_lambda;
    }
  }
  for (pli = 0; pli < 3; pli++) free(planes[pli]);
  daala_encode_free(enc);
  return ret;
}
