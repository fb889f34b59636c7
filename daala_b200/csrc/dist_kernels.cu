// Perceptual block distortion of the RDO loops (reference src/encode.c: od_compute_var_4x4 :1081,
// od_compute_dist_8x8 :1111, od_compute_dist :1180) for a batch of packed n x n block pairs --
// SURVEY.md 8(f) rank 2: the metric the deringing level search and the block-size decision evaluate.
//
// Parity: tests/test_gpu_dist.py against oracle/port_dist.c (bit-identical to od_compute_dist); consumers:
// the deringing level search, csrc/dering_search.cu, and (through dist_device.cuh) the late-skip kernel.
//
// Mapping: one 64-thread CTA per block pair running block_dist (dist_device.cuh, which gives the operation order).
// sqrt is IEEE (-prec-sqrt=true); pow comes from the CUDA math library (<= 2 ulp), so the HVS result is compared
// with a 1e-12 relative tolerance rather than bit for bit.
#include <cuda_runtime.h>
#include <stdint.h>

#include "daala_b200.h"
#include "dist_device.cuh"

namespace daala_b200 {
namespace dist {

__global__ void __launch_bounds__(kDistThreads)
k_compute_dist(const int32_t* __restrict__ xs, const int32_t* __restrict__ ys, int n, int qm_is_flat,
               int use_activity_masking, double scale, double* __restrict__ out,
               const daala_b200_kf_frame_quant* __restrict__ fq, int per_frame) {
  extern __shared__ __align__(16) int32_t smem[];
  const size_t nn = (size_t)n * n;
  const double d = block_dist(xs + blockIdx.x * nn, n, 0, ys + blockIdx.x * nn, n, 0, __ffs(n) - 1, 1, qm_is_flat,
                              use_activity_masking, scale, smem);
  // fq: scale is 1.0 and the pair's frame's scale is applied here (block_dist's last multiplication; x * 1.0 is exact)
  if (threadIdx.x == 0)
    out[blockIdx.x] = fq && !qm_is_flat ? d * dist_scale(fq[blockIdx.x / per_frame].coded_quantizer) : d;
}

}  // namespace dist
}  // namespace daala_b200

// daala_b200_compute_dist, or (fq non-NULL) each pair i scaled by the coded_quantizer of record fq[i / per_frame]
int daala_b200_compute_dist_frames(const int32_t* x, const int32_t* y, int count, int n, int qm_is_flat,
                                   int use_activity_masking, int coded_quantizer, const daala_b200_kf_frame_quant* fq,
                                   int per_frame, double* out, void* stream) {
  if (count <= 0) return 0;
  if (n != 8 && n != 16 && n != 32 && n != 64) return (int)cudaErrorInvalidValue;
  const size_t smem = daala_b200::dist::dist_scratch_bytes(n);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(daala_b200::dist::k_compute_dist, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  daala_b200::dist::k_compute_dist<<<count, daala_b200::dist::kDistThreads, smem, (cudaStream_t)stream>>>(
      x, y, n, qm_is_flat, use_activity_masking, fq ? 1.0 : daala_b200::dist::dist_scale(coded_quantizer), out, fq,
      per_frame);
  return (int)cudaGetLastError();
}

extern "C" int daala_b200_compute_dist(const int32_t* x, const int32_t* y, int count, int n, int qm_is_flat,
                                       int use_activity_masking, int coded_quantizer, double* out, void* stream) {
  return daala_b200_compute_dist_frames(x, y, count, n, qm_is_flat, use_activity_masking, coded_quantizer, nullptr, 1,
                                        out, stream);
}
