// Internal: the deringing level search of a batch of frames as a sequence of launches on one stream, without
// allocations or synchronisation (CUDA-graph capturable) -- csrc/dering_search.cu, used by the keyframe engine's
// deringing stage (config.dering = 2) and by the P-frame finishing pass (config.inter_finish = 2).
#pragma once
#include <stdint.h>

#include "daala_b200.h"

struct daala_b200_dering_search_batch {
  const int16_t* etmp;      // [F] luma planes after the SB-edge postfilter (state->etmp[0]), row stride = width
  const uint8_t* src;       // [F] source luma planes
  long long etmp_pitch, src_pitch;   // elements between consecutive frames
  int etmp_stride, src_stride;
  int nframes, nhsb, nvsb;
  int threshold[6];         // (int)(OD_DERING_GAIN_TABLE[gi] * quantizer^0.84182)
  int coded_quantizer, qm_is_flat, use_activity_masking;
  double dering_lambda;
  // skip flags of every filtered candidate (state->bskip[0]): [nvsb * 16][skip_stride] per frame, skip_pitch bytes
  // apart; keyframes pass one all-zero map with skip_pitch 0
  const uint8_t* bskip;
  int skip_stride;
  long long skip_pitch;
  // [F][nvsb * nhsb] (nullable): the superblock has a coded 4x4 luma unit; the others get level 0, are not scored and
  // do not adapt the CDF (src/encode.c:2724-2738)
  const uint8_t* coded;
  int is_keyframe;          // context up + left (keyframes), else 0 (src/encode.c:2753-2769)
  const uint8_t* frame_type; // nullable [F]: frame f's is_keyframe (the engine's frame_types), replacing the field above
  // scratch / outputs (device)
  int16_t* filt;            // [F] filtered planes (same geometry as etmp, pitch = width * height)
  int32_t *orig, *cand;     // [F * nsb][64 * 64]
  int32_t* dir;             // [F][nvsb * 8][nhsb * 8], left in the packed direction | variance << 3 format
  double* dist;             // [6][F * nsb]
  uint8_t* levels;          // out: [F][nvsb * nhsb]
  // the engine's (NULL in daala_b200_dering_search): per frame records (coded_quantizer and dering_lambda replace the
  // fields above) and threshold tables ([F][2][6], replacing `threshold`), and the scratch of the filtered candidates'
  // per-superblock thresholds, [5][F * nsb]
  const daala_b200_kf_frame_quant* fq;
  const int32_t* frame_tbl;
  int32_t* cand_thr;
};
extern "C" int daala_b200_dering_search_enqueue(const daala_b200_dering_search_batch* b, void* stream);

// daala_b200_compute_dist with each pair i scaled by the coded_quantizer of fq[i / per_frame] (fq NULL: coded_quantizer)
int daala_b200_compute_dist_frames(const int32_t* x, const int32_t* y, int count, int n, int qm_is_flat,
                                   int use_activity_masking, int coded_quantizer, const daala_b200_kf_frame_quant* fq,
                                   int per_frame, double* out, void* stream);

// The deringing threshold of every level at `quantizer` (src/encode.c:2697, :2822): tbl[0][g] luma,
// (int)(OD_DERING_GAIN_TABLE[g] * quantizer^0.84182); tbl[1][g] chroma, the same product * 0.6.
void daala_b200_dering_threshold_table(int quantizer, int tbl[2][6]);

// od_dering of `nframes` planes of one geometry in one launch (csrc/dering_kernels.cu): element pitches between the
// frames' planes, direction maps and threshold maps, skip_pitch bytes between their skip maps (0: one map for every
// frame); y8 (nullable) receives the u8 reconstruction instead of the int16 plane.
int daala_b200_dering_plane_frames(const daala_b200_dering_params* prm, int nframes, long long y_pitch,
                                   long long x_pitch, long long dir_pitch, long long thr_pitch, long long skip_pitch,
                                   uint8_t* y8, void* stream);
