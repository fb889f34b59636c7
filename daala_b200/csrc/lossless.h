// Internal: the lossless step of the keyframe engine (config.lossless; quantizer 0, the reference's Haar-wavelet path)
// as launches on one stream, without allocations or synchronisation (CUDA-graph capturable) -- csrc/lossless.cu,
// launched by csrc/kf_engine.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// Every pointer is a device pointer.  Planes are frame-sized ([F][plane_h][plane_w], the engine's padded geometry);
// every superblock of every plane is one block of n = 64 >> xdec.
struct daala_b200_lossless_batch {
  const uint8_t* src[3];      // the input pictures
  const uint8_t* pred[3];     // P / B frames: the prediction planes; NULL on keyframes
  int16_t* coeffs[3];         // daala_b200_kf_io.ll_coeffs: each block's residual at the block's place
  int32_t* blocks;            // [F][nvsb][nhsb][3][4]: the three root tree sums and a reserved 0
  int32_t* dc;                // keyframes: [F][nvsb][nhsb][3] each block's DC d[0], the superblock DC predictor's input
  uint8_t* out[3];            // the reconstruction
  uint8_t* pool[3];           // inter_mc: the reference-picture pool ([slots][plane_h][plane_w]), else NULL
  const int32_t* slot_out;    // inter_mc: [F] the pool slot of each frame's reconstruction, -1 = not stored
  int F, nhsb, nvsb, pic_w, pic_h;
  int plane_w[3], plane_h[3];
};

// Keyframes (pred == NULL): two launches, the forward transform and the DC prediction + reconstruction.  P / B frames:
// one launch.
extern "C" int daala_b200_launch_lossless(const daala_b200_lossless_batch* b, cudaStream_t stream);
