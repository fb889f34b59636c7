/* oracle/ref_hooks_inter_mc.c -- TEST INFRASTRUCTURE ONLY.
 * Hooks for the engine's P-frame prediction from MV grids, linked with the reference build's objects into
 * _ref/libdaala_ref_inter_mc.so by inter_mc.mk: od_state_mc_predict with two reference pictures, and real P frames
 * captured from the whole reference encoder.  Only non-static reference functions and the public encoder API are
 * used, so this TU includes headers only. */
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include "state.h"
#include "mc.h"
#include "util.h"
#include "encint.h"
#include "daala/codec.h"
#include "daala/daalaenc.h"

void od_mc_predict1fmv8_c(od_state *state, unsigned char *dst,
 const unsigned char *src, int systride, int32_t mvx, int32_t mvy,
 int log_xblk_sz, int log_yblk_sz);
void od_mc_blend_full8_c(unsigned char *dst, int dystride,
 const unsigned char *src[4], int log_xblk_sz, int log_yblk_sz);
void od_mc_blend_full_split8_c(unsigned char *dst, int dystride,
 const unsigned char *src[4], int oc, int s, int log_xblk_sz, int log_yblk_sz);

/* The two-picture form of oracle_ref_state_mc_predict: od_state_mc_predict on a real od_state whose
   ref_imgs[0] holds the OD_FRAME_GOLD picture and ref_imgs[1] the OD_FRAME_PREV picture (both loaded with
   od_img_edge_ext), or, with same != 0, one picture for both (ref_imgi[GOLD] = ref_imgi[PREV]: the num_refs = 1
   case of src/encode.c:3014-3017; prev_* are then not read).  Every vertex takes valid, mv and ref (0 = GOLD,
   1 = PREV) from the caller: (nvmvbs+1) x (nhmvbs+1) entries row-major.  Planes are frame-sized.  seconds (may be
   NULL) receives the wall time of the od_state_mc_predict call alone. */
int oracle_ref_state_mc_predict2(int pic_w, int pic_h, const unsigned char *gold_y, const unsigned char *gold_u,
 const unsigned char *gold_v, const unsigned char *prev_y, const unsigned char *prev_u,
 const unsigned char *prev_v, int same, const unsigned char *valid, const int32_t *mv,
 const unsigned char *ref, unsigned char *out_y, unsigned char *out_u, unsigned char *out_v, double *seconds) {
  struct timespec t0;
  struct timespec t1;
  od_state st;
  daala_info info;
  const unsigned char *refp[2][3];
  unsigned char *outp[3];
  int pli;
  int r;
  int vx;
  int vy;
  int y;
  daala_info_init(&info);
  info.pic_width = pic_w;
  info.pic_height = pic_h;
  info.nplanes = 3;
  info.plane_info[0].xdec = info.plane_info[0].ydec = 0;
  info.plane_info[1].xdec = info.plane_info[1].ydec = 1;
  info.plane_info[2].xdec = info.plane_info[2].ydec = 1;
  info.bitdepth_mode = OD_BITDEPTH_MODE_8;
  info.full_precision_references = 0;
  info.timebase_numerator = 30; info.timebase_denominator = 1; info.frame_duration = 1;
  info.pixel_aspect_numerator = 1; info.pixel_aspect_denominator = 1;
  info.keyframe_rate = 256;
  if (od_state_init(&st, &info) < 0) return -1;
  st.opt_vtbl.mc_predict1fmv = od_mc_predict1fmv8_c;
  st.opt_vtbl.mc_blend_full = od_mc_blend_full8_c;
  st.opt_vtbl.mc_blend_full_split = od_mc_blend_full_split8_c;
  st.ref_imgi[OD_FRAME_GOLD] = 0;
  st.ref_imgi[OD_FRAME_PREV] = same ? 0 : 1;
  st.ref_imgi[OD_FRAME_SELF] = 2;
  refp[0][0] = gold_y; refp[0][1] = gold_u; refp[0][2] = gold_v;
  refp[1][0] = prev_y; refp[1][1] = prev_u; refp[1][2] = prev_v;
  outp[0] = out_y; outp[1] = out_u; outp[2] = out_v;
  for (r = 0; r < (same ? 1 : 2); r++) {
    for (pli = 0; pli < 3; pli++) {
      daala_image_plane *ip = st.ref_imgs[r].planes + pli;
      int w = st.frame_width >> ip->xdec;
      int h = st.frame_height >> ip->ydec;
      for (y = 0; y < h; y++) memcpy(ip->data + y*ip->ystride, refp[r][pli] + y*w, w);
    }
    od_img_edge_ext(st.ref_imgs + r);
  }
  for (vy = 0; vy <= st.nvmvbs; vy++) {
    for (vx = 0; vx <= st.nhmvbs; vx++) {
      od_mv_grid_pt *g = st.mv_grid[vy] + vx;
      int i = vy*(st.nhmvbs + 1) + vx;
      g->valid = valid[i];
      g->mv[0] = mv[2*i];
      g->mv[1] = mv[2*i + 1];
      g->ref = ref[i];
    }
  }
  clock_gettime(CLOCK_MONOTONIC, &t0);
  od_state_mc_predict(&st, st.ref_imgs + 2);
  clock_gettime(CLOCK_MONOTONIC, &t1);
  if (seconds) *seconds = (t1.tv_sec - t0.tv_sec) + 1e-9*(t1.tv_nsec - t0.tv_nsec);
  for (pli = 0; pli < 3; pli++) {
    daala_image_plane *ip = st.ref_imgs[2].planes + pli;
    int w = st.frame_width >> ip->xdec;
    int h = st.frame_height >> ip->ydec;
    for (y = 0; y < h; y++) memcpy(outp[pli] + y*w, ip->data + y*ip->ystride, w);
  }
  od_state_clear(&st);
  return 0;
}

/* Real P frames: the whole reference encoder through its public API on encode_frames.inc's synthetic content,
   frame 0 a keyframe and frames 1 .. nframes-1 P frames (keyframe_rate = 256) at `complexity`.  For each P frame
   f (output index f - 1), frame-sized planes (Y then U then V, fw*fh*3/2 bytes per picture):
     src    the encoder's padded input picture (enc->curr_img after daala_encode_img_in);
     gold, prev  the OD_FRAME_GOLD / OD_FRAME_PREV pictures it predicted from, snapshot before daala_encode_img_in
            (the reference buffers rotate at the end of the frame); same[f - 1] = 1 when they were one picture;
     pred   od_state_mc_predict re-run on the encoder's own state after the frame, with ref_imgi[GOLD] / [PREV]
            set back to the two pictures of the frame (the buffers they were are not reused before the next frame);
   and bsize ([nvsb*8][nhsb*8], state->bsize), valid / ref / mv (state->mv_grid, (nvmvbs+1) x (nhmvbs+1),
   mv as int32 pairs). */
int oracle_ref_capture_p_frames(int w, int h, int nframes, int quant, int complexity, unsigned char *src,
 unsigned char *gold, unsigned char *prev, int *same, unsigned char *pred, unsigned char *bsize,
 unsigned char *valid, unsigned char *ref, int32_t *mv) {
  daala_info info;
  daala_enc_ctx *enc;
  daala_image img;
  daala_packet op;
  unsigned char *planes[3];
  unsigned s = 12345;
  int f;
  int pli;
  int ret = 0;
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
  daala_encode_ctl(enc, OD_SET_QUANT, &quant, sizeof(quant));
  daala_encode_ctl(enc, OD_SET_COMPLEXITY, &complexity, sizeof(complexity));
  for (pli = 0; pli < 3; pli++) planes[pli] = (unsigned char *)malloc((size_t)w*h);
  for (f = 0; f < nframes && ret == 0; f++) {
    od_state *st = &enc->state;
    int fw = st->frame_width;
    int fh = st->frame_height;
    size_t pic = (size_t)fw*fh + 2*(size_t)(fw >> 1)*(fh >> 1);
    int gi = st->ref_imgi[OD_FRAME_GOLD];
    int pi = st->ref_imgi[OD_FRAME_PREV];
    int x;
    int y;
    for (pli = 0; pli < 3; pli++) {
      int pw = pli ? w >> 1 : w;
      int ph = pli ? h >> 1 : h;
      for (y = 0; y < ph; y++) {
        for (x = 0; x < pw; x++) {
          int v;
          s = s*1103515245u + 12345u;
          v = 128 + 60*((x + 3*f)%97)/97 + 40*((y + 2*f)%61)/61 - 50 + (int)(((s >> 16) & 0x7fff)%9) - 4;
          planes[pli][y*pw + x] = v < 0 ? 0 : v > 255 ? 255 : v;
        }
      }
    }
    if (f > 0) {
      /* copy out the frame-sized area of image `im` (ref_imgs or the input) into dst */
#define CAPTURE_PICTURE(dst, im) do { \
        unsigned char *d_ = (dst); \
        for (pli = 0; pli < 3; pli++) { \
          const daala_image_plane *ip_ = (im)->planes + pli; \
          int pw_ = fw >> ip_->xdec; \
          int ph_ = fh >> ip_->ydec; \
          for (y = 0; y < ph_; y++) memcpy(d_ + (size_t)y*pw_, ip_->data + (ptrdiff_t)y*ip_->ystride, pw_); \
          d_ += (size_t)pw_*ph_; \
        } \
      } while (0)
      CAPTURE_PICTURE(gold + (f - 1)*pic, st->ref_imgs + gi);
      CAPTURE_PICTURE(prev + (f - 1)*pic, st->ref_imgs + pi);
      same[f - 1] = gi == pi;
    }
    img.nplanes = 3;
    img.width = w;
    img.height = h;
    for (pli = 0; pli < 3; pli++) {
      img.planes[pli].data = planes[pli];
      img.planes[pli].xdec = img.planes[pli].ydec = pli > 0;
      img.planes[pli].xstride = 1;
      img.planes[pli].ystride = pli == 0 ? w : w >> 1;
      img.planes[pli].bitdepth = 8;
    }
    if (daala_encode_img_in(enc, &img, 1) < 0) { ret = -2; break; }
    if (daala_encode_packet_out(enc, f + 1 == nframes, &op) <= 0) { ret = -3; break; }
    if (f > 0) {
      daala_image out;
      unsigned char *buf = (unsigned char *)malloc(pic);
      int si = st->ref_imgi[OD_FRAME_GOLD];
      int sp = st->ref_imgi[OD_FRAME_PREV];
      int vx;
      int vy;
      int i;
      int j;
      CAPTURE_PICTURE(src + (f - 1)*pic, enc->curr_img);
      out = st->ref_imgs[0];
      out.planes[0].data = buf;
      out.planes[0].ystride = fw;
      out.planes[1].data = buf + (size_t)fw*fh;
      out.planes[1].ystride = fw >> 1;
      out.planes[2].data = buf + (size_t)fw*fh + (size_t)(fw >> 1)*(fh >> 1);
      out.planes[2].ystride = fw >> 1;
      for (pli = 0; pli < 3; pli++) out.planes[pli].xstride = 1;
      st->ref_imgi[OD_FRAME_GOLD] = gi;
      st->ref_imgi[OD_FRAME_PREV] = pi;
      od_state_mc_predict(st, &out);
      st->ref_imgi[OD_FRAME_GOLD] = si;
      st->ref_imgi[OD_FRAME_PREV] = sp;
      memcpy(pred + (f - 1)*pic, buf, pic);
      free(buf);
      for (i = 0; i < st->nvsb*8; i++) {
        for (j = 0; j < st->nhsb*8; j++) {
          bsize[(size_t)(f - 1)*st->nvsb*8*st->nhsb*8 + i*st->nhsb*8 + j] = st->bsize[i*st->bstride + j];
        }
      }
      for (vy = 0; vy <= st->nvmvbs; vy++) {
        for (vx = 0; vx <= st->nhmvbs; vx++) {
          const od_mv_grid_pt *g = st->mv_grid[vy] + vx;
          size_t k = (size_t)(f - 1)*(st->nvmvbs + 1)*(st->nhmvbs + 1) + (size_t)vy*(st->nhmvbs + 1) + vx;
          valid[k] = g->valid;
          ref[k] = g->ref;
          mv[2*k] = g->mv[0];
          mv[2*k + 1] = g->mv[1];
        }
      }
    }
#undef CAPTURE_PICTURE
  }
  for (pli = 0; pli < 3; pli++) free(planes[pli]);
  daala_encode_free(enc);
  return ret;
}
