// The level loops of od_haar / od_haar_inv (reference src/dct.c:4822 / :4861), the multi-level 2-D Haar wavelet of the
// lossless path, for one n x n block (n = 1 << ln <= 64) worked on by one CTA of kThreads threads.  Shared by
// k_haar_blocks (frame_transform.cu) and the lossless step's kernels (lossless.cu).
//
// Every level is "read all 2x2 groups, then write": the reference's serial loop order only makes its in-place update
// equal to that (forward: LL(i,j) is consumed by group (i/2, j/2), visited earlier; inverse: groups are visited in
// descending order).  Sub-band placement as the reference: lh -> (i, j + np), hl -> (i + np, j), hh -> (i + np, j + np),
// with OD_HAAR_KERNEL(a, b, c, d) (src/tf.h:34) taking b = the sample BELOW a and c = the one to its RIGHT.
#pragma once

namespace daala_b200 {

// t: the block (row stride n) on entry, the LL scratch of every level after it.  y (row stride ystride) receives the
// detail sub-bands and, last, y[0] = the DC.  t and y must not overlap.  Ends without a barrier after the write of
// y[0] (thread 0).
template <int kThreads, class T>
__device__ __forceinline__ void haar_forward_levels(int* t, T* y, int ystride, int ln) {
  const int n = 1 << ln;
  for (int level = 0; level < ln; level++) {
    const int np = n >> level >> 1;
    int keep[4096 / 4 / kThreads];   // np * np <= 1024 groups
    int q = 0;
    for (int idx = threadIdx.x; idx < np * np; idx += kThreads, q++) {
      const int i = idx / np, j = idx - i * np;
      int ll = t[2 * i * n + 2 * j], lh = t[(2 * i + 1) * n + 2 * j];
      int hl = t[2 * i * n + 2 * j + 1], hh = t[(2 * i + 1) * n + 2 * j + 1];
      ll += hl;
      hh -= lh;
      const int m = (ll - hh) >> 1;
      lh = m - lh;
      hl = m - hl;
      ll -= lh;
      hh += hl;
      keep[q] = ll;
      y[i * ystride + j + np] = (T)lh;
      y[(i + np) * ystride + j] = (T)hl;
      y[(i + np) * ystride + j + np] = (T)hh;
    }
    __syncthreads();
    q = 0;
    for (int idx = threadIdx.x; idx < np * np; idx += kThreads, q++) {
      const int i = idx / np, j = idx - i * np;
      t[i * n + j] = keep[q];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) y[0] = (T)t[0];
}

// The inverse: y (row stride ystride) holds the sub-bands, t (row stride n) receives the block.  Starts with a barrier
// after t[0] = y[0] and ends with one.
template <int kThreads, class T>
__device__ __forceinline__ void haar_inverse_levels(int* t, const T* y, int ystride, int ln) {
  const int n = 1 << ln;
  if (threadIdx.x == 0) t[0] = y[0];
  __syncthreads();
  for (int level = ln - 1; level >= 0; level--) {
    const int np = 1 << (ln - 1 - level);
    constexpr int kMax = 4096 / 4 / kThreads;
    int a4[kMax], b4[kMax], c4[kMax], d4[kMax];
    int q = 0;
    for (int idx = threadIdx.x; idx < np * np; idx += kThreads, q++) {
      const int i = idx / np, j = idx - i * np;
      int ll = t[i * n + j], lh = y[i * ystride + j + np], hl = y[(i + np) * ystride + j];
      int hh = y[(i + np) * ystride + j + np];
      ll += hl;
      hh -= lh;
      const int m = (ll - hh) >> 1;
      lh = m - lh;
      hl = m - hl;
      ll -= lh;
      hh += hl;
      a4[q] = ll; b4[q] = lh; c4[q] = hl; d4[q] = hh;
    }
    __syncthreads();
    q = 0;
    for (int idx = threadIdx.x; idx < np * np; idx += kThreads, q++) {
      const int i = idx / np, j = idx - i * np;
      t[2 * i * n + 2 * j] = a4[q];
      t[(2 * i + 1) * n + 2 * j] = b4[q];
      t[2 * i * n + 2 * j + 1] = c4[q];
      t[(2 * i + 1) * n + 2 * j + 1] = d4[q];
    }
    __syncthreads();
  }
}

}  // namespace daala_b200
