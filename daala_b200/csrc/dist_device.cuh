// od_compute_dist (reference src/encode.c:1180, with od_compute_var_4x4 :1081 and od_compute_dist_8x8 :1111) of a few
// n x n block pairs of one size as a __device__ function of a 64-thread CTA: the body of k_compute_dist
// (dist_kernels.cu, one pair per CTA) and of the keyframe engine's late-skip kernel (late_skip.cu, 4096 samples per
// CTA).
//
// HVS path: the error x - y is low-passed by the separable [1 5 1] kernel in shared memory (integer, exact); one
// thread per 8x8 sub-block evaluates the nine overlapping 4x4 window variances and the activity factor in double
// precision in the reference's operation order, and one thread per pair adds its sub-block results in raster order
// and applies the coded-quantizer scale (double addition is not associative).  Flat path (enc->qm == OD_FLAT_QM): the plain
// squared error.  Every term is an integer and so is every partial sum; while the total stays below 2^53 (any two
// blocks of lapped-domain samples, |x - y| < 2^20) each partial sum is exact, so the parallel sum equals the
// reference's index-order sum bit for bit.
#pragma once
#include <limits.h>
#include <math.h>
#include <stdint.h>

namespace daala_b200 {
namespace dist {

constexpr int kDistThreads = 64;

__device__ __forceinline__ int window_var(const int32_t* p, int stride) {
  int s = 0, s2 = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int t = p[i * stride + j] >> 2;
      s += t;
      s2 += t * t;
    }
  }
  return s2 - (s * s >> 4);
}

// The coded-quantizer scale of the HVS path (src/encode.c:1221-1223): 1.7 below 36, 1.2 from 47, linear in between.
__host__ __device__ inline double dist_scale(int coded_quantizer) {
  return coded_quantizer >= 47 ? 1.2 : coded_quantizer <= 36 ? 1.7
         : 1.7 + (1.2 - 1.7) * (coded_quantizer - 36) / (47 - 36);
}

// Shared memory block_dist needs for g blocks of n x n: err and rows (g * n * n int32 each), then 64 doubles (the
// sub-block results, or the flat path's partial sums).
__host__ __device__ constexpr int dist_scratch_bytes(int n, int g = 1) {
  return (int)(sizeof(int32_t) * 2 * g * n * n + sizeof(double) * kDistThreads);
}

// od_compute_dist of g block pairs of n x n (n = 1 << ln, 8..64; g * n * n <= 4096, so g divides 64): pair k is
// x + k * xb / y + k * yb, rows xs / ys apart (global or shared memory).  scratch: dist_scratch_bytes(n, g) of
// 8-byte aligned shared memory.  Called by all kDistThreads threads of the CTA; thread k < g returns the distortion of
// pair k (the others return 0).  Ends with a barrier, so the caller may rewrite x, y and the scratch afterwards.
__device__ __forceinline__ double block_dist(const int32_t* x, int xs, int xb, const int32_t* y, int ys, int yb, int ln,
                                             int g, int qm_is_flat, int use_activity_masking, double scale,
                                             int32_t* scratch) {
  const int n = 1 << ln, nn = n * n, tot = g * nn;
  const int t = threadIdx.x;
  int32_t* err = scratch;          // g * n * n
  int32_t* rows = scratch + tot;   // g * n * n, then reused for the low-passed error
  double* part = (double*)(scratch + 2 * tot);
  double total = 0;
  if (qm_is_flat) {
    const int per = kDistThreads / g;   // threads per pair
    const int k = t / per, u = t - k * per;
    double s = 0;
    for (int idx = u; idx < nn; idx += per) {
      const int i = idx >> ln, j = idx & (n - 1);
      const double d = x[k * xb + i * xs + j] - y[k * yb + i * ys + j];
      s += d * d;
    }
    part[t] = s;
    __syncthreads();
    if (t < g)
      for (int v = 0; v < per; v++) total += part[t * per + v];
    __syncthreads();
    return total;
  }
  for (int idx = t; idx < tot; idx += kDistThreads) {
    const int k = idx >> (2 * ln), i = (idx >> ln) & (n - 1), j = idx & (n - 1);
    err[idx] = x[k * xb + i * xs + j] - y[k * yb + i * ys + j];
  }
  __syncthreads();
  for (int idx = t; idx < tot; idx += kDistThreads) {
    const int j = idx & (n - 1);
    const int32_t* e = err + (idx - j);
    int32_t v;
    if (j == 0) v = 5 * e[0] + 2 * e[1];
    else if (j == n - 1) v = 5 * e[n - 1] + 2 * e[n - 2];
    else v = 5 * e[j] + e[j - 1] + e[j + 1];
    rows[idx] = v;
  }
  __syncthreads();
  // vertical pass into err (the raw error is no longer needed)
  for (int idx = t; idx < tot; idx += kDistThreads) {
    const int i = (idx >> ln) & (n - 1);
    int32_t v;
    if (i == 0) v = 5 * rows[idx] + 2 * rows[idx + n];
    else if (i == n - 1) v = 5 * rows[idx] + 2 * rows[idx - n];
    else v = 5 * rows[idx] + rows[idx - n] + rows[idx + n];
    err[idx] = v;
  }
  __syncthreads();
  const int nb = n >> 3, nsub = nb * nb;
  if (t < g * nsub) {
    const int k = t / nsub, r = t - k * nsub;
    const int bi = r / nb, bj = r - bi * nb;
    const int32_t* px = x + k * xb + bi * 8 * xs + bj * 8;
    const int32_t* py = y + k * yb + bi * 8 * ys + bj * 8;
    const int32_t* lp = err + k * nn + bi * 8 * n + bj * 8;
    double inv_sum = 0, texture = 0, energy = 0;
    int lowest = INT_MAX;
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) {
        const int vx = window_var(px + 2 * i * xs + 2 * j, xs);
        const int vy = window_var(py + 2 * i * ys + 2 * j, ys);
        if (vx < lowest) lowest = vx;
        inv_sum += 1. / (1 + vx);
        texture += vx - 2 * sqrt(vx * (double)vy) + vy;
      }
    }
    const double stat = use_activity_masking ? 9. / inv_sum : (double)lowest;
    const double activity = (use_activity_masking ? 1.95 : 1.62) * pow(.25 + stat / (1 << 2 * 4), -1. / 6);
    for (int i = 0; i < 8; i++)
      for (int j = 0; j < 8; j++) energy += lp[i * n + j] * (double)lp[i * n + j];
    energy *= 0.92 / (7 * 7 * 7 * 7);
    part[t] = activity * activity * (energy + texture);
  }
  __syncthreads();
  if (t < g) {
    for (int v = 0; v < nsub; v++) total += part[t * nsub + v];   // the sub-blocks in raster order
    total *= scale;
  }
  __syncthreads();
  return total;
}

}  // namespace dist
}  // namespace daala_b200
