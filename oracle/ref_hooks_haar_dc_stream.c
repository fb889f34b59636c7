/* oracle/ref_hooks_haar_dc_stream.c -- TEST INFRASTRUCTURE ONLY.
 * The coded bytes of a keyframe's DC symbols, two ways, for the engine's keyframe DC records (symbol_stream = 1 with
 * haar_dc_quant = 1; tests/haar_dc_stream_oracle.py):
 *   oracle_ref_haar_dc_frame_bytes  the range-coder output of the reference's own DC chain, as the keyframe DC driver of
 *                                   ref_hooks_haar_dc.c runs it (od_compute_dcts, od_quantize_haar_dc_sb and
 *                                   od_quantize_haar_dc_level in od_encode_recursive's order, nothing else coded);
 *   oracle_ref_haar_dc_replay       a list of daala_b200_kf_sym_hdc records replayed through the reference's
 *                                   generic_encode and od_ec_enc_bits on a fresh encoder.
 * Equal bytes mean equal values, order and model contexts.  Includes ref_hooks_haar_dc.c (and through it the
 * reference's src/encode.c) for its statics, so haar_dc_stream.mk links it into a library of its own, as haar_dc.mk does
 * for the driver. */
#include "ref_hooks_haar_dc.c"

/* daala_b200_kf_sym_hdc (include/daala_b200.h), 12 bytes. */
typedef struct {
  int32_t value;
  uint32_t block;
  uint8_t pli;
  uint8_t bsi;
  uint8_t child;
  uint8_t reserved;
} strm_hdc_rec;

static daala_enc_ctx *strm_create(int pic_w, int pic_h) {
  daala_info info;
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
  return daala_encode_create(&info);
}

/* od_ec_enc_done of the encoder into out (cap bytes); returns the byte count, or -3 when it does not fit. */
static int strm_done(daala_enc_ctx *enc, unsigned char *out, int cap) {
  uint32_t nbytes;
  unsigned char *buf;
  buf = od_ec_enc_done(&enc->ec, &nbytes);
  if ((int)nbytes > cap) return -3;
  memcpy(out, buf, nbytes);
  return (int)nbytes;
}

/* The split-node part of od_encode_recursive for a keyframe (src/encode.c:1660-1787): od_quantize_haar_dc_level on
   every split node depth-first, the gradients passed by value. */
static void strm_recursive(daala_enc_ctx *enc, od_mb_enc_ctx *ctx, int pli, int bx, int by, int bsi, int xdec,
 od_coeff hgrad, od_coeff vgrad) {
  int obs;
  obs = OD_BLOCK_SIZE4x4(enc->state.bsize, enc->state.bstride, bx << bsi, by << bsi);
  if (OD_MAXI(obs, xdec) == bsi) return;
  od_quantize_haar_dc_level(enc, ctx, pli, 2*bx, 2*by, bsi - 1, xdec, &hgrad, &vgrad);
  strm_recursive(enc, ctx, pli, 2*bx + 0, 2*by + 0, bsi - 1, xdec, hgrad, vgrad);
  strm_recursive(enc, ctx, pli, 2*bx + 1, 2*by + 0, bsi - 1, xdec, hgrad, vgrad);
  strm_recursive(enc, ctx, pli, 2*bx + 0, 2*by + 1, bsi - 1, xdec, hgrad, vgrad);
  strm_recursive(enc, ctx, pli, 2*bx + 1, 2*by + 1, bsi - 1, xdec, hgrad, vgrad);
}

/* The keyframe DC chain of oracle_ref_haar_dc_frame (same arguments and the same steps on a real encoder) and the
   bytes it coded: od_ec_enc_done after the last superblock, into out (cap bytes).  Returns the byte count, or < 0. */
int oracle_ref_haar_dc_frame_bytes(int pic_w, int pic_h, const unsigned char *src, const unsigned char *bsize,
 int quantizer, const unsigned char *pvq_qm_q4, double pvq_norm_lambda, unsigned char *out, int cap) {
  daala_enc_ctx *enc;
  od_state *state;
  od_mb_enc_ctx mbctx;
  size_t off[3];
  int fw;
  int fh;
  int nhsb;
  int nvsb;
  int pli;
  int sbx;
  int sby;
  int x;
  int y;
  int ret;
  enc = strm_create(pic_w, pic_h);
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
  }
  for (sby = 0; sby < nvsb; sby++) {
    for (sbx = 0; sbx < nhsb; sbx++) {
      for (pli = 0; pli < 3; pli++) {
        int xdec = state->info.plane_info[pli].xdec;
        int ydec = state->info.plane_info[pli].ydec;
        od_coeff hgrad;
        od_coeff vgrad;
        hgrad = vgrad = 0;
        mbctx.c = state->ctmp[pli];
        mbctx.mc = state->mctmp[pli];
        mbctx.md = state->mdtmp[pli];
        mbctx.l = state->lbuf[pli];
        od_compute_dcts(enc, &mbctx, pli, sbx, sby, OD_NBSIZES - 1, xdec, ydec, 0);
        od_quantize_haar_dc_sb(enc, &mbctx, pli, sbx, sby, xdec, ydec, sby > 0 && sbx < nhsb - 1, &hgrad, &vgrad);
        strm_recursive(enc, &mbctx, pli, sbx, sby, OD_NBSIZES - 1, xdec, hgrad, vgrad);
      }
    }
  }
  ret = strm_done(enc, out, cap);
  daala_encode_free(enc);
  return ret;
}

/* The records recs[0..n) of one frame coded on a fresh encoder of pic_w x pic_h after od_adapt_ctx_reset, as
   od_quantize_haar_dc_sb / od_quantize_haar_dc_level code a value (src/encode.c:1583-1585, :1630-1632):
   generic_encode of |value| with max -1 and integration 2 on model_dc[pli] and ex_sb_dc[pli] (child 0) or
   ex_dc[pli][bsi][child - 1], then the sign bit when value != 0.  The bytes go to out (cap bytes).  Returns the byte
   count, -1 when the encoder cannot be created, -2 on a record outside the models. */
int oracle_ref_haar_dc_replay(int pic_w, int pic_h, const void *recs, int n, unsigned char *out, int cap) {
  const strm_hdc_rec *r;
  daala_enc_ctx *enc;
  od_adapt_ctx *adapt;
  int i;
  int ret;
  enc = strm_create(pic_w, pic_h);
  if (enc == NULL) return -1;
  adapt = &enc->state.adapt;
  od_adapt_ctx_reset(adapt, 1);
  od_ec_enc_reset(&enc->ec);
  r = (const strm_hdc_rec *)recs;
  for (i = 0; i < n; i++) {
    int v = r[i].value;
    int *ex;
    if (r[i].pli >= 3 || r[i].child > 3 || (r[i].child > 0 && r[i].bsi >= OD_NBSIZES)) {
      daala_encode_free(enc);
      return -2;
    }
    ex = r[i].child == 0 ? &adapt->ex_sb_dc[r[i].pli] : &adapt->ex_dc[r[i].pli][r[i].bsi][r[i].child - 1];
    generic_encode(&enc->ec, &adapt->model_dc[r[i].pli], abs(v), -1, ex, 2);
    if (v) od_ec_enc_bits(&enc->ec, v < 0, 1);
  }
  ret = strm_done(enc, out, cap);
  daala_encode_free(enc);
  return ret;
}
