/* oracle/ref_hooks_lossless.c -- TEST INFRASTRUCTURE ONLY.
 * The lossless (quantizer 0) frame driver of the engine's lossless tests (tests/lossless_oracle.py).  Compiles the
 * reference's src/encode.c in place to reach its statics, so lossless.mk links it into a library of its own with the
 * reference build's objects other than the TUs that include encode.c too (ref_hooks_encode.c) or call into them
 * (ref_pipeline.c). */
#include "encode.c"

/* One frame as od_encode_coefficients codes it at quantizer 0 (OD_LOSSLESS, src/internal.h:131), on a real encoder of
   pic_w x pic_h whose state.quantizer is 0 and whose superblocks are all OD_BLOCK_64X64 (src/encode.c:3087-3089).
   src (and, for a P or B frame, pred) hold the frame-sized planes Y, U, V one after the other, u8.  Per plane:
     ctmp = src - 128 (od_ref_plane_to_coeff, lossless); P / B frames: mctmp = pred - 128 and the samples of ctmp
     outside the picture replaced by mctmp's (the loops of src/encode.c:2589-2602, restated);
   then per superblock in raster order, planes 0..2 inside:
     keyframes: od_compute_dcts(use_haar = 1) and od_quantize_haar_dc_sb with has_ur = sby > 0 && sbx < nhsb - 1;
     P / B frames: od_compute_dcts(use_haar = 1) of ctmp into d and of mctmp into md (what od_block_encode's
     od_haar calls compute for one 64x64 block, src/encode.c:1292-1299);
     od_encode_compute_pred for the block's prediction (0 on keyframes, md otherwise), the residual of
     od_wavelet_quantize's first loop with q = 1 (src/encode.c:1012-1027), the DC of src/encode.c:1337-1343 with
     dc_quant = 1 (P / B) or dc0 = d[0] - the superblock DC predictor (keyframes), and od_compute_max_tree's three roots.
   Outputs (frame-sized planes, Y U V): d_out the `d` planes (od_coeff; the keyframe DCs as od_quantize_haar_dc_sb
   leaves them), resid_out the residual with the coded DC in each block's DC slot; roots_out [nvsb][nhsb][3][3]:
   tree_sum[0][1], [1][0], [1][1] per plane.  Returns 0, or < 0 when the encoder cannot be created. */
int oracle_ref_lossless_frame(int pic_w, int pic_h, int keyframe, const unsigned char *src,
 const unsigned char *pred, int32_t *d_out, int32_t *resid_out, int32_t *roots_out) {
  daala_info info;
  daala_enc_ctx *enc;
  od_state *state;
  od_mb_enc_ctx mbctx;
  od_coeff *md_planes[OD_NPLANES_MAX];
  od_coeff pred_blk[OD_BSIZE_MAX*OD_BSIZE_MAX];
  od_coeff out[OD_BSIZE_MAX*OD_BSIZE_MAX];
  od_coeff tree_sum[OD_BSIZE_MAX][OD_BSIZE_MAX];
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
  state->quantizer = 0;
  od_state_init_superblock_split(state, OD_BLOCK_64X64);
  od_adapt_ctx_reset(&state->adapt, keyframe);
  od_ec_enc_reset(&enc->ec);
  fw = state->frame_width;
  fh = state->frame_height;
  nhsb = state->nhsb;
  nvsb = state->nvsb;
  off[0] = 0;
  off[1] = (size_t)fw*fh;
  off[2] = off[1] + (size_t)(fw >> 1)*(fh >> 1);
  OD_CLEAR(&mbctx, 1);
  mbctx.is_keyframe = keyframe;
  mbctx.use_haar_wavelet = 1;
  mbctx.d = state->dtmp;
  for (pli = 0; pli < 3; pli++) {
    int xdec = state->info.plane_info[pli].xdec;
    int ydec = state->info.plane_info[pli].ydec;
    int w = fw >> xdec;
    int h = fh >> ydec;
    for (y = 0; y < h; y++) {
      for (x = 0; x < w; x++) {
        state->ctmp[pli][y*w + x] = src[off[pli] + (size_t)y*w + x] - 128;
        if (!keyframe) state->mctmp[pli][y*w + x] = pred[off[pli] + (size_t)y*w + x] - 128;
      }
    }
    if (!keyframe) {
      int pic_width = state->info.pic_width >> xdec;
      int pic_height = state->info.pic_height >> ydec;
      for (x = pic_width; x < w; x++) {
        for (y = 0; y < h; y++) state->ctmp[pli][y*w + x] = state->mctmp[pli][y*w + x];
      }
      for (y = pic_height; y < h; y++) {
        for (x = 0; x < w; x++) state->ctmp[pli][y*w + x] = state->mctmp[pli][y*w + x];
      }
    }
    md_planes[pli] = state->mdtmp[pli];
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
        od_coeff *d = state->dtmp[pli];
        od_coeff dc;
        int32_t *roots;
        int i;
        int j;
        mbctx.c = state->ctmp[pli];
        mbctx.mc = state->mctmp[pli];
        mbctx.md = state->mdtmp[pli];
        mbctx.l = state->lbuf[pli];
        od_compute_dcts(enc, &mbctx, pli, sbx, sby, OD_NBSIZES - 1, xdec, ydec, 1);
        if (keyframe) {
          od_coeff hgrad;
          od_coeff vgrad;
          od_coeff d0;
          int quantizer;
          int q4;
          int qi;
          d0 = d[bo];
          /* The predictor: the same call with a DC quantiser coarser than any |dc0| codes quant = 0, so it leaves the
             predictor itself in d[bo] (sb_dc_curr = 0*dc_quant + sb_dc_pred); the coded call below then sets d[bo]
             and sb_dc_mem back to d0 (lossless: quant = dc0). */
          quantizer = state->quantizer;
          qi = od_qm_get_index(OD_NBSIZES - 1, 0);
          q4 = state->pvq_qm_q4[pli][qi];
          state->quantizer = 1 << 20;
          state->pvq_qm_q4[pli][qi] = 16;
          od_quantize_haar_dc_sb(enc, &mbctx, pli, sbx, sby, xdec, ydec, sby > 0 && sbx < nhsb - 1, &hgrad, &vgrad);
          dc = d0 - d[bo];
          state->quantizer = quantizer;
          state->pvq_qm_q4[pli][qi] = q4;
          d[bo] = d0;
          od_quantize_haar_dc_sb(enc, &mbctx, pli, sbx, sby, xdec, ydec, sby > 0 && sbx < nhsb - 1, &hgrad, &vgrad);
        }
        else {
          mbctx.c = state->mctmp[pli];
          mbctx.d = md_planes;
          od_compute_dcts(enc, &mbctx, pli, sbx, sby, OD_NBSIZES - 1, xdec, ydec, 1);
          mbctx.c = state->ctmp[pli];
          mbctx.d = state->dtmp;
        }
        od_encode_compute_pred(enc, &mbctx, pred_blk, d, ln - 2, pli, sbx << (ln - 2), sby << (ln - 2));
        for (i = 0; i < n; i++) {
          for (j = 0; j < n; j++) out[i*n + j] = OD_DIV_R0(d[bo + i*w + j] - pred_blk[i*n + j], 1);
        }
        if (!keyframe) {
          /* src/encode.c:1337-1343 with dc_quant = max(1, quantizer) = 1 */
          if (abs(d[bo] - pred_blk[0]) < 1*141/256) dc = 0;
          else dc = OD_DIV_R0(d[bo] - pred_blk[0], 1);
        }
        out[0] = dc;
        od_compute_max_tree(tree_sum, 1, 0, out, ln);
        od_compute_max_tree(tree_sum, 0, 1, out, ln);
        od_compute_max_tree(tree_sum, 1, 1, out, ln);
        roots = roots_out + ((size_t)(sby*nhsb + sbx)*3 + pli)*3;
        roots[0] = tree_sum[0][1];
        roots[1] = tree_sum[1][0];
        roots[2] = tree_sum[1][1];
        for (i = 0; i < n; i++) {
          for (j = 0; j < n; j++) {
            d_out[off[pli] + bo + (size_t)i*w + j] = d[bo + i*w + j];
            resid_out[off[pli] + bo + (size_t)i*w + j] = out[i*n + j];
          }
        }
      }
    }
  }
  daala_encode_free(enc);
  return 0;
}
