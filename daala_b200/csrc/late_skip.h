// Internal: the late-skip distortions of a P-frame step (config.late_skip) as launches on one stream, without
// allocations or synchronisation (CUDA-graph capturable) -- csrc/late_skip.cu, used by the keyframe engine
// (csrc/kf_engine.cu) after the finishing scatter of both stages.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "daala_b200.h"

struct daala_b200_late_skip_batch {
  const daala_b200_pvq_block* blocks[2];   // luma, chroma block lists
  const int32_t* count[2];                 // device counters: blocks in each list
  int max_blocks[2];
  const int32_t* d_orig[3];                // per plane: the unquantised coefficients (the step's forward output)
  const int32_t* d[3];                     // the coded coefficients (after k_finish_scatter<true>)
  const int32_t* md[3];                    // the transformed prediction
  long long plane_pitch[3];                // elements between frames
  int plane_stride[3];
  int qm_is_flat, use_activity_masking;    // od_compute_dist's parameters, with each frame's coded_quantizer
  const daala_b200_kf_frame_quant* fq;     // [F] each frame's record (its coded_quantizer)
  const int32_t* fq_bq;                    // [F][3][32] each frame's band quantisers (the DC's: [bs * (bs + 1)])
  daala_b200_kf_late_skip* out[2];         // per block of each list
  // scratch: the blocks of each size class 8x8 .. 64x64 (list << 31 | block), cls_cap[c] entries from cls_off[c] of
  // cls_items, and their counts cls_n[4] (cleared by the enqueue)
  uint32_t* cls_items;
  long long cls_off[4], cls_cap[4];
  int32_t* cls_n;
};

// Entries of cls_items a batch of `px` samples (all planes and frames) needs: every block of class c covers
// (8 << c)^2 samples.
long long daala_b200_late_skip_class_caps(long long px, long long off[4], long long cap[4]);

// Launches of daala_b200_late_skip_enqueue: the size-class split (which also zeroes the records of 4x4 blocks) and one
// launch per size class.
constexpr int kLateSkipLaunches = 5;

// [memset of cls_n], the split, then per size class `ctas` CTAs of 64 threads over batches of 4096 samples.
int daala_b200_late_skip_enqueue(const daala_b200_late_skip_batch* b, int ctas, cudaStream_t stream);
