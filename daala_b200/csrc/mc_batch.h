// Internal: the keyframe engine's prediction step for P frames from MV grids (config.inter_mc), implemented in
// mc_kernels.cu beside the interpolator and blend it reuses, launched by kf_engine.cu inside its graph.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "daala_b200.h"

// Every pointer is a device pointer.  Planes are frame-sized ([plane_h][plane_w], the engine's padded geometry);
// the MV grid of a frame has (nvsb*8 + 1) rows of (nhsb*8 + 1) vertices.
struct daala_b200_mc_batch {
  const daala_b200_mv_pt* grid;    // [F][nvsb*8 + 1][nhsb*8 + 1]
  const int32_t* ref_slot;         // [F][2]: pool slots of OD_FRAME_GOLD, OD_FRAME_PREV
  const uint8_t* ref[3];           // pool: [nslots][plane_h][plane_w]
  uint8_t* pred[3];                // [F][plane_h][plane_w]
  uint32_t* leaves;                // [F][nvsb*nhsb][64] leaf records (see mc_kernels.cu), a count per segment in
  int32_t* nleaves;                // [F][nvsb*nhsb]
  int32_t* bad_ref;                // counter: leaf corners whose vertex has a ref other than 0 / 1 (0 / 1 / 2 with mv1)
  int32_t* beyond;                 // counter: corner windows reaching past the reference's edge extension
  int F, nhsb, nvsb, nslots;
  int plane_w[3], plane_h[3];
  // config.mc_next (B frames), NULL otherwise: a vertex with ref 2 (OD_FRAME_NEXT) is predicted from the frame's NEXT
  // picture with its second vector mv1 (od_state_pred_block_from_setup, reference src/state.c:647-660)
  const int32_t* ref_slot_next;    // [F]: pool slot of OD_FRAME_NEXT
  const int32_t* mv1;              // [F][nvsb*8 + 1][nhsb*8 + 1][2]: each vertex's mv1 in 1/8 luma pixel
  // nullable [F]: the engine's frame_types, 1 on keyframes, which have no leaves and a prediction of 0
  const uint8_t* frame_type;
};

// od_state_pred_block's split recursion for every (frame, 64x64 MV block): its leaves and both counters.
extern "C" int daala_b200_launch_mc_leaves(const daala_b200_mc_batch* b, int grid, cudaStream_t stream);
// OBMC of every leaf in every plane into `pred` (reads the leaves of the launch above).
extern "C" int daala_b200_launch_mc_obmc(const daala_b200_mc_batch* b, int grid, cudaStream_t stream);
