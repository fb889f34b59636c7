// Internal: the deringing level search of a batch of frames as a sequence of launches on one stream, without
// allocations or synchronisation (CUDA-graph capturable) -- csrc/dering_search.cu, used by the keyframe engine's
// deringing stage (config.dering = 2) and by the P-frame finishing pass (config.inter_finish = 2).
#pragma once
#include <stdint.h>

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
  // scratch / outputs (device)
  int16_t* filt;            // [F] filtered planes (same geometry as etmp, pitch = width * height)
  int32_t *orig, *cand;     // [F * nsb][64 * 64]
  int32_t* dir;             // [F][nvsb * 8][nhsb * 8], left in the packed direction | variance << 3 format
  double* dist;             // [6][F * nsb]
  uint8_t* levels;          // out: [F][nvsb * nhsb]
};
extern "C" int daala_b200_dering_search_enqueue(const daala_b200_dering_search_batch* b, void* stream);
