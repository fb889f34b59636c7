// Internal: the keyframe DC chain of the keyframe engine (config.haar_dc_quant) as one launch on one stream, without
// allocations or synchronisation (CUDA-graph capturable) -- csrc/haar_dc.cu, launched by csrc/kf_engine.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// Every pointer is a device pointer.  Planes are frame-sized ([F][plane_h][plane_w], the engine's padded geometry,
// 4:2:0); the grids have one entry per 4x4 unit of their plane ([plane_h / 4][plane_w / 4] per frame): the index grids
// of a plane one frame after the other, the DC grids grid_frame_pitch entries apart.
struct daala_b200_haar_dc_batch {
  const int32_t* coeffs[3];   // the `d` planes: the unquantised Haar DC pyramid the forward transform leaves
  int32_t* dc[3];             // out: the reconstructed DC of every coded position; at a leaf block's origin its final DC
  int32_t* index[3];          // out: the signed coded indices (SB DC at the SB origin, a split node's three at the
                              // origins of its children 1..3), 0 elsewhere
  const uint8_t* bsize;       // [F][nvsb * 8][nhsb * 8] block-size maps
  int F, nhsb, nvsb;
  int plane_w[3], plane_h[3];
  long long grid_frame_pitch;  // entries between the DC grids of consecutive frames
  double pvq_norm_lambda;
  // each frame's band quantisers ([F][3][32], max(1, q0 * pvq_qm_q4[pli][i] >> 4) of its record); frame f's dc_quant of
  // plane p is entry [f][p][20] (od_qm_get_index(OD_NBSIZES - 1, 0))
  const int32_t* fq_bq;
  // nullable [F]: with the engine's frame_types, 1 on keyframes; the other frames' index grids are cleared and nothing
  // else of them is read or written
  const uint8_t* frame_type;
};

// One warp per (frame, plane): grid F * 3.
extern "C" int daala_b200_launch_haar_dc(const daala_b200_haar_dc_batch* b, cudaStream_t stream);
