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
               int use_activity_masking, double scale, double* __restrict__ out) {
  extern __shared__ __align__(16) int32_t smem[];
  const size_t nn = (size_t)n * n;
  const double d = block_dist(xs + blockIdx.x * nn, n, 0, ys + blockIdx.x * nn, n, 0, __ffs(n) - 1, 1, qm_is_flat,
                              use_activity_masking, scale, smem);
  if (threadIdx.x == 0) out[blockIdx.x] = d;
}

}  // namespace dist
}  // namespace daala_b200

extern "C" int daala_b200_compute_dist(const int32_t* x, const int32_t* y, int count, int n, int qm_is_flat,
                                       int use_activity_masking, int coded_quantizer, double* out, void* stream) {
  if (count <= 0) return 0;
  if (n != 8 && n != 16 && n != 32 && n != 64) return (int)cudaErrorInvalidValue;
  const size_t smem = daala_b200::dist::dist_scratch_bytes(n);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(daala_b200::dist::k_compute_dist, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  daala_b200::dist::k_compute_dist<<<count, daala_b200::dist::kDistThreads, smem, (cudaStream_t)stream>>>(
      x, y, n, qm_is_flat, use_activity_masking, daala_b200::dist::dist_scale(coded_quantizer), out);
  return (int)cudaGetLastError();
}
