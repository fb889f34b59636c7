/* oracle/ref_hooks_bframes.c -- TEST INFRASTRUCTURE ONLY.
 * Hooks for the engine's B-frame prediction (config.mc_next), linked with the reference build's objects into
 * _ref/libdaala_ref_bframes.so by bframes.mk: od_state_mc_predict with GOLD, PREV and NEXT pictures, and whole
 * B-frame sequences captured from the reference encoder.  Only non-static reference functions and the public encoder
 * API are used, so this TU includes headers only. */
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
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

/* The three-picture form for B frames: od_state_mc_predict on a real od_state whose ref_imgi[GOLD / PREV / NEXT] name
   the pictures gold / prev / next.  Pictures passed by the same Y pointer share one buffer (any two, or all three, may
   be one picture), the others each load into a buffer of their own with od_img_edge_ext.  Every vertex takes valid,
   mv, mv1 and ref (0 = GOLD, 1 = PREV, 2 = NEXT) from the caller, (nvmvbs+1) x (nhmvbs+1) entries row-major, mv and
   mv1 as int32 pairs; the reference reads mv1 where ref == OD_FRAME_NEXT (src/state.c:654-660). */
int oracle_ref_state_mc_predict3(int pic_w, int pic_h, const unsigned char *const gold[3],
 const unsigned char *const prev[3], const unsigned char *const next[3], const unsigned char *valid,
 const int32_t *mv, const int32_t *mv1, const unsigned char *ref, unsigned char *out_y, unsigned char *out_u,
 unsigned char *out_v) {
  od_state st;
  daala_info info;
  const unsigned char *const *pics[3];
  unsigned char *outp[3];
  int nbuf;
  int k;
  int pli;
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
  pics[0] = gold; pics[1] = prev; pics[2] = next;
  nbuf = 0;
  for (k = 0; k < 3; k++) {
    int j;
    for (j = 0; j < k && pics[j][0] != pics[k][0]; j++);
    if (j < k) {
      st.ref_imgi[k] = st.ref_imgi[j];
      continue;
    }
    st.ref_imgi[k] = nbuf;
    for (pli = 0; pli < 3; pli++) {
      daala_image_plane *ip = st.ref_imgs[nbuf].planes + pli;
      int w = st.frame_width >> ip->xdec;
      int h = st.frame_height >> ip->ydec;
      for (y = 0; y < h; y++) memcpy(ip->data + y*ip->ystride, pics[k][pli] + y*w, w);
    }
    od_img_edge_ext(st.ref_imgs + nbuf);
    nbuf++;
  }
  st.ref_imgi[OD_FRAME_SELF] = 3;
  outp[0] = out_y; outp[1] = out_u; outp[2] = out_v;
  for (vy = 0; vy <= st.nvmvbs; vy++) {
    for (vx = 0; vx <= st.nhmvbs; vx++) {
      od_mv_grid_pt *g = st.mv_grid[vy] + vx;
      int i = vy*(st.nhmvbs + 1) + vx;
      g->valid = valid[i];
      g->mv[0] = mv[2*i];
      g->mv[1] = mv[2*i + 1];
      g->mv1[0] = mv1[2*i];
      g->mv1[1] = mv1[2*i + 1];
      g->ref = ref[i];
    }
  }
  od_state_mc_predict(&st, st.ref_imgs + 3);
  for (pli = 0; pli < 3; pli++) {
    daala_image_plane *ip = st.ref_imgs[3].planes + pli;
    int w = st.frame_width >> ip->xdec;
    int h = st.frame_height >> ip->ydec;
    for (y = 0; y < h; y++) memcpy(outp[pli] + y*w, ip->data + y*ip->ystride, w);
  }
  od_state_clear(&st);
  return 0;
}

/* A whole B-frame sequence through the reference encoder's public API with OD_SET_B_FRAMES = b_frames, on the
   synthetic content of oracle_ref_capture_p_frames (ref_hooks_inter_mc.c; display frame f is its frame f), the caller draining
   daala_encode_packet_out after every daala_encode_img_in (the last image with last = 1).  Every coded frame k, in
   coding order (one per packet, src/encode.c:3274-3292), records:
     number[k], type[k] (OD_I/P/B_FRAME), golden[k], quantizer[k] (state->quantizer) and
     refi[4k .. 4k+3]  the ref_imgi[GOLD, PREV, NEXT, SELF] the frame used: GOLD, PREV and NEXT are snapshot before
                       the packet call, with the one rule od_encode_frame applies when it starts (src/encode.c:2986-2989:
                       a P frame of a B-frame sequence moves NEXT into PREV); SELF is read after the call (the end of
                       the frame rotates GOLD / PREV / NEXT, never SELF);
     src, gold, prev, next, pred  frame-sized pictures (Y then U then V, fw*fh*3/2 bytes each): the padded input, the
                       three reference pictures of the frame (zeros where refi is -1; read after the call, as SELF is a
                       buffer none of them uses), and od_state_mc_predict re-run with the frame's own ref_imgi (zeros for
                       keyframes);
     bsize, valid, ref, mv, mv1  state->bsize and state->mv_grid after the frame, as oracle_ref_capture_p_frames.
   Returns the number of coded frames (nframes), or < 0 on failure. */
int oracle_ref_capture_b_frames(int w, int h, int nframes, int b_frames, int keyframe_rate, int quant, int complexity,
 int *number, int *type, int *golden, int *refi, int *quantizer, unsigned char *src, unsigned char *gold,
 unsigned char *prev, unsigned char *next, unsigned char *pred, unsigned char *bsize, unsigned char *valid,
 unsigned char *ref, int32_t *mv, int32_t *mv1) {
  daala_info info;
  daala_enc_ctx *enc;
  daala_image img;
  daala_packet op;
  unsigned char *planes[3];
  unsigned s = 12345;
  int f;
  int k;
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
  info.keyframe_rate = keyframe_rate;
  enc = daala_encode_create(&info);
  if (enc == NULL) return -1;
  daala_encode_ctl(enc, OD_SET_QUANT, &quant, sizeof(quant));
  daala_encode_ctl(enc, OD_SET_COMPLEXITY, &complexity, sizeof(complexity));
  if (daala_encode_ctl(enc, OD_SET_B_FRAMES, &b_frames, sizeof(b_frames)) != OD_SUCCESS) {
    daala_encode_free(enc);
    return -4;
  }
  for (pli = 0; pli < 3; pli++) planes[pli] = (unsigned char *)malloc((size_t)w*h);
  k = 0;
  for (f = 0; f < nframes && ret == 0; f++) {
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
    for (;;) {
      od_state *st = &enc->state;
      int fw = st->frame_width;
      int fh = st->frame_height;
      size_t pic = (size_t)fw*fh + 2*(size_t)(fw >> 1)*(fh >> 1);
      int used[4];
      int saved[4];
      int r;
      int vx;
      int vy;
      int i;
      int j;
      for (r = 0; r < 4; r++) used[r] = st->ref_imgi[r];
      if (daala_encode_packet_out(enc, f + 1 == nframes, &op) <= 0) break;
      if (k >= nframes) { ret = -3; break; }
      type[k] = st->frame_type;
      if (b_frames != 0 && type[k] == OD_P_FRAME) used[OD_FRAME_PREV] = used[OD_FRAME_NEXT];
      used[OD_FRAME_SELF] = st->ref_imgi[OD_FRAME_SELF];
      number[k] = (int)enc->curr_display_order;
      golden[k] = type[k] == OD_I_FRAME || (st->ref_imgi[OD_FRAME_GOLD] == used[OD_FRAME_SELF]);
      quantizer[k] = st->quantizer;
      for (r = 0; r < 4; r++) refi[4*k + r] = used[r];
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
      CAPTURE_PICTURE(src + k*pic, enc->curr_img);
      if (used[OD_FRAME_GOLD] >= 0) CAPTURE_PICTURE(gold + k*pic, st->ref_imgs + used[OD_FRAME_GOLD]);
      if (used[OD_FRAME_PREV] >= 0) CAPTURE_PICTURE(prev + k*pic, st->ref_imgs + used[OD_FRAME_PREV]);
      if (used[OD_FRAME_NEXT] >= 0) CAPTURE_PICTURE(next + k*pic, st->ref_imgs + used[OD_FRAME_NEXT]);
#undef CAPTURE_PICTURE
      if (type[k] != OD_I_FRAME) {
        daala_image out;
        unsigned char *buf = (unsigned char *)malloc(pic);
        out = st->ref_imgs[0];
        out.planes[0].data = buf;
        out.planes[0].ystride = fw;
        out.planes[1].data = buf + (size_t)fw*fh;
        out.planes[1].ystride = fw >> 1;
        out.planes[2].data = buf + (size_t)fw*fh + (size_t)(fw >> 1)*(fh >> 1);
        out.planes[2].ystride = fw >> 1;
        for (pli = 0; pli < 3; pli++) out.planes[pli].xstride = 1;
        for (r = 0; r < 4; r++) {
          saved[r] = st->ref_imgi[r];
          st->ref_imgi[r] = used[r];
        }
        od_state_mc_predict(st, &out);
        for (r = 0; r < 4; r++) st->ref_imgi[r] = saved[r];
        memcpy(pred + k*pic, buf, pic);
        free(buf);
      }
      for (i = 0; i < st->nvsb*8; i++) {
        for (j = 0; j < st->nhsb*8; j++) {
          bsize[(size_t)k*st->nvsb*8*st->nhsb*8 + i*st->nhsb*8 + j] = st->bsize[i*st->bstride + j];
        }
      }
      for (vy = 0; vy <= st->nvmvbs; vy++) {
        for (vx = 0; vx <= st->nhmvbs; vx++) {
          const od_mv_grid_pt *g = st->mv_grid[vy] + vx;
          size_t q = (size_t)k*(st->nvmvbs + 1)*(st->nhmvbs + 1) + (size_t)vy*(st->nhmvbs + 1) + vx;
          valid[q] = g->valid;
          ref[q] = g->ref;
          mv[2*q] = g->mv[0];
          mv[2*q + 1] = g->mv[1];
          mv1[2*q] = g->mv1[0];
          mv1[2*q + 1] = g->mv1[1];
        }
      }
      k++;
    }
  }
  for (pli = 0; pli < 3; pli++) free(planes[pli]);
  daala_encode_free(enc);
  return ret == 0 ? k : ret;
}
