// Motion compensation and block-matching kernels for sm_90a (H100, 8-bit path).
//
// k_obmc_blocks:    for each block of a list, up to four 1/8-pel predictions
//                   (6-tap separable windowed-sinc interpolation) and the
//                   bilinear overlapped-block blend, written straight into the
//                   destination plane.  Restates od_mc_predict1fmv8_c
//                   (reference src/mc.c:94), od_mc_blend_full8_c (:352),
//                   od_mc_blend_full_split8_c (:1104) as driven by
//                   od_mc_predict_singleref (:1965) / od_state_pred_block
//                   (src/state.c:627-709).
// k_match_candidates: for each (block, candidate MV): interpolate the
//                   displaced reference block and return its SAD or SATD
//                   against the current frame -- the inner operation of
//                   od_mv_est_bma_sad (src/mcenc.c:2224) with
//                   od_mc_compute_sad8_c (:1333) / od_mc_compute_satd8 (:1467,
//                   sum-of-8x8 rule :1517).  SAD uses __vabsdiffu4 on packed
//                   pixels and warp-shuffle reductions.
// One CTA per job; the (n+5)-row horizontal stage lives in shared memory.
#include <cuda_runtime.h>
#include <stdint.h>

#include "daala_b200.h"

namespace daala_b200 {
namespace mc {

constexpr int kThreads = 128;
constexpr int kMaxN = 64;     // OD_MVBSIZE_MAX
constexpr int kApron = 5;     // OD_SUBPEL_BUFF_APRON_SZ: 2 rows above, 3 below

// 6-tap bank for the eight 1/8-pel phases, 7-bit coefficients
// (OD_SUBPEL_FILTER_SET, reference src/mc.c:66-77).
__constant__ short kSubpel[8][6] = {
    {0, 0, 128, 0, 0, 0},   {1, -9, 122, 18, -5, 1},  {3, -15, 112, 37, -11, 2}, {3, -18, 97, 58, -15, 3},
    {4, -20, 80, 80, -20, 4}, {3, -15, 58, 97, -18, 3}, {2, -11, 37, 112, -15, 3}, {1, -5, 18, 122, -9, 1}};

__device__ __forceinline__ unsigned char clamp255(int v) { return (unsigned char)(v < 0 ? 0 : v > 255 ? 255 : v); }

// CTA-cooperative single-MV prediction of an nx x ny block into `out` (row
// stride nx).  `src` points at the block's own position in the reference
// plane; mv in 1/8 pel.  `buf` holds (ny + 5) * nx int16.
__device__ void predict_block(unsigned char* out, short* buf, const unsigned char* src, int stride,
                              int mvx, int mvy, int lx, int ly) {
  const int nx = 1 << lx, ny = 1 << ly;
  const int fxi = mvx & 7, fyi = mvy & 7;
  const unsigned char* p = src + (mvx >> 3) + (mvy >> 3) * stride;
  if (!fxi && !fyi) {
    for (int i = threadIdx.x; i < nx * ny; i += blockDim.x) out[i] = p[(i >> lx) * stride + (i & (nx - 1))];
    __syncthreads();
    return;
  }
  // Horizontal stage, rows -2 .. ny+2, biased by -(128 << 7) to fit int16.
  for (int i = threadIdx.x; i < nx * (ny + kApron); i += blockDim.x) {
    int r = (i >> lx) - 2, c = i & (nx - 1);
    const unsigned char* row = p + r * stride + c;
    int v;
    if (fxi) {
      v = 0;
#pragma unroll
      for (int k = 0; k < 6; k++) v += row[k - 2] * kSubpel[fxi][k];
      v -= 128 << 7;
    } else {
      v = (row[0] << 7) - (128 << 7);
    }
    buf[i] = (short)v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nx * ny; i += blockDim.x) {
    const short* b = buf + i + 2 * nx;
    int v;
    if (fyi) {
      int sum = 0;
#pragma unroll
      for (int k = 0; k < 6; k++) sum += b[(k - 2) * nx] * kSubpel[fyi][k];
      v = (sum + (1 << 13) + (128 << 14)) >> 14;   // OD_SUBPEL_RND_OFFSET3, src/mc.h:84
    } else {
      v = (b[0] + (1 << 6) + (128 << 7)) >> 7;     // OD_SUBPEL_RND_OFFSET4, src/mc.h:86
    }
    out[i] = clamp255(v);
  }
  __syncthreads();
}

// Blend weights of od_mc_setup_s_split (src/mc.c:1056) in closed form:
// w_k(i, j) = s0_k + j*dsdj_k + i*(dsdi_k + j*dd_k).
struct SplitWeights {
  int s0[4], dsdi[4], dsdj[4], dd[4];
};

__device__ __forceinline__ SplitWeights split_weights(int oc, int s, int lx, int ly) {
  SplitWeights w;
  w.s0[0] = 2 << (lx + ly); w.s0[1] = w.s0[2] = w.s0[3] = 0;
  w.dsdi[0] = -(2 << lx); w.dsdi[1] = 2 << lx; w.dsdi[2] = w.dsdi[3] = 0;
  w.dsdj[0] = -(2 << ly); w.dsdj[1] = w.dsdj[2] = 0; w.dsdj[3] = 2 << ly;
  w.dd[0] = w.dd[2] = 2; w.dd[1] = w.dd[3] = -2;
#pragma unroll
  for (int e = 0; e < 2; e++) {
    if (!(s & (1 << e))) {
      int k = (oc + (e ? 3 : 1)) & 3;
#pragma unroll
      for (int q = 0; q < 4; q++) {
        // (k and oc are runtime indices; unrolled selects keep the arrays in registers)
        if (q == k) { w.s0[q] >>= 1; w.dsdi[q] >>= 1; w.dsdj[q] >>= 1; w.dd[q] >>= 1; }
      }
      int hs = 0, hi = 0, hj = 0, hd = 0;
#pragma unroll
      for (int q = 0; q < 4; q++) if (q == k) { hs = w.s0[q]; hi = w.dsdi[q]; hj = w.dsdj[q]; hd = w.dd[q]; }
#pragma unroll
      for (int q = 0; q < 4; q++) if (q == oc) { w.s0[q] += hs; w.dsdi[q] += hi; w.dsdj[q] += hj; w.dd[q] += hd; }
    }
  }
  return w;
}

// OBMC prediction of one block (od_mc_predict_singleref, src/mc.c:1965) by the CTA into out[j * out_stride + i]:
// up to four single-MV predictions (re-used when two corners share a MV) + od_mc_blend_full(_split)8_c.
__device__ void obmc_block(unsigned char* out, int out_stride, unsigned char (&pred)[4][kMaxN * kMaxN], short* buf,
                           const unsigned char* ref, int ref_stride, const daala_b200_mc_block& b) {
  const int lx = b.log_xblk, ly = b.log_yblk;
  const int nx = 1 << lx, ny = 1 << ly;
  const unsigned char* src = ref + (size_t)b.y0 * ref_stride + b.x0;
  int which[4];
  for (int k = 0; k < 4; k++) {
    which[k] = k;
    for (int q = 0; q < k; q++) {
      if (b.mvx[q] == b.mvx[k] && b.mvy[q] == b.mvy[k]) { which[k] = which[q]; break; }
    }
    if (which[k] == k) predict_block(pred[k], buf, src, ref_stride, b.mvx[k], b.mvy[k], lx, ly);
  }
  const unsigned char* p0 = pred[which[0]];
  const unsigned char* p1 = pred[which[1]];
  const unsigned char* p2 = pred[which[2]];
  const unsigned char* p3 = pred[which[3]];
  if (b.s == 3) {
    const int l2 = lx + ly;
    for (int idx = threadIdx.x; idx < nx * ny; idx += blockDim.x) {
      int i = idx & (nx - 1), j = idx >> lx;
      int a = p0[idx], c = p3[idx];
      a = (a << lx) + (p1[idx] - a) * i;
      c = (c << lx) + (p2[idx] - c) * i;
      out[(size_t)j * out_stride + i] = (unsigned char)(((a << ly) + (c - a) * j + (1 << (l2 - 1))) >> l2);
    }
  } else {
    const SplitWeights w = split_weights(b.oc, b.s, lx, ly);
    const int l2p1 = lx + ly + 1;
    for (int idx = threadIdx.x; idx < nx * ny; idx += blockDim.x) {
      int i = idx & (nx - 1), j = idx >> lx;
      int a = p0[idx];
      int acc = (a << l2p1) + (p1[idx] - a) * (w.s0[1] + j * w.dsdj[1] + i * (w.dsdi[1] + j * w.dd[1]))
                + (p2[idx] - a) * (w.s0[2] + j * w.dsdj[2] + i * (w.dsdi[2] + j * w.dd[2]))
                + (p3[idx] - a) * (w.s0[3] + j * w.dsdj[3] + i * (w.dsdi[3] + j * w.dd[3]));
      out[(size_t)j * out_stride + i] = (unsigned char)((acc + (1 << (l2p1 - 1))) >> l2p1);
    }
  }
}

__global__ void __launch_bounds__(kThreads)
k_obmc_blocks(const unsigned char* __restrict__ ref, int ref_stride, unsigned char* __restrict__ dst,
              int dst_stride, const daala_b200_mc_block* __restrict__ blocks) {
  __shared__ unsigned char pred[4][kMaxN * kMaxN];
  __shared__ short buf[(kMaxN + kApron) * kMaxN];
  const daala_b200_mc_block b = blocks[blockIdx.x];
  obmc_block(dst + (size_t)b.y0 * dst_stride + b.x0, dst_stride, pred, buf, ref, ref_stride, b);
}

// 8-point Walsh-Hadamard on registers (ordering is irrelevant for a sum of magnitudes).
__device__ __forceinline__ void wht8(int (&v)[8]) {
#pragma unroll
  for (int len = 1; len < 8; len <<= 1) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      if (!(i & len)) {
        int a = v[i], b = v[i + len];
        v[i] = a + b;
        v[i + len] = a - b;
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads)
k_match_candidates(const unsigned char* __restrict__ cur, int cur_stride, const unsigned char* __restrict__ ref,
                   int ref_stride, const daala_b200_match_job* __restrict__ jobs, int use_satd,
                   int32_t* __restrict__ result) {
  __shared__ __align__(16) unsigned char pred[kMaxN * kMaxN];
  // interpolation scratch (8.8 KB of int16) first, SATD workspace (n*n + 64 ints) afterwards
  __shared__ int work[kMaxN * kMaxN + 64];
  __shared__ int partial[kThreads / 32];
  short* buf = reinterpret_cast<short*>(work);
  const daala_b200_match_job job = jobs[blockIdx.x];
  const int ln = job.log_blk, n = 1 << ln;
  predict_block(pred, buf, ref + (size_t)job.y0 * ref_stride + job.x0, ref_stride, job.mvx, job.mvy, ln, ln);
  const unsigned char* c0 = cur + (size_t)job.y0 * cur_stride + job.x0;
  int acc = 0;
  if (!use_satd) {
    // four pixels per step: |a - b| per byte, then a byte-wise sum (dot with 1s)
    const bool aligned = ((((size_t)c0) | (size_t)cur_stride) & 3) == 0;
    for (int q = threadIdx.x; q < (n * n) >> 2; q += blockDim.x) {
      int idx = q << 2, r = idx >> ln, c = idx & (n - 1);
      unsigned pv = *reinterpret_cast<const unsigned*>(pred + idx);
      unsigned cv;
      const unsigned char* cp = c0 + (size_t)r * cur_stride + c;
      if (aligned) cv = *reinterpret_cast<const unsigned*>(cp);
      else cv = cp[0] | (cp[1] << 8) | (cp[2] << 16) | ((unsigned)cp[3] << 24);
      acc = (int)__dp4a(__vabsdiffu4(pv, cv), 0x01010101u, (unsigned)acc);
    }
  } else if (ln == 2) {
    // one 4x4 transform: thread t < 4 owns row t, then columns through shared memory
    int* w = work;
    if (threadIdx.x < 4) {
      int r = threadIdx.x, v[4];
      for (int k = 0; k < 4; k++) v[k] = c0[(size_t)r * cur_stride + k] - pred[r * 4 + k];
      int a = v[0] + v[1], b = v[0] - v[1], c = v[2] + v[3], d = v[2] - v[3];
      w[r * 4 + 0] = a + c; w[r * 4 + 1] = b + d; w[r * 4 + 2] = a - c; w[r * 4 + 3] = b - d;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
      int k = threadIdx.x;
      int a = w[k] + w[4 + k], b = w[k] - w[4 + k], c = w[8 + k] + w[12 + k], d = w[8 + k] - w[12 + k];
      acc = abs(a + c) + abs(b + d) + abs(a - c) + abs(b - d);
    }
  } else {
    // sum of 8x8 SATDs, each (sum |H| + 4) >> 3.  Row pass into shared memory,
    // column pass + magnitude sum per 8x8 block, rounded per block.
    int* w = work;
    for (int item = threadIdx.x; item < (n * n) >> 3; item += blockDim.x) {
      int r = item / (n >> 3), c8 = (item % (n >> 3)) << 3;
      int v[8];
#pragma unroll
      for (int k = 0; k < 8; k++) v[k] = c0[(size_t)r * cur_stride + c8 + k] - pred[r * n + c8 + k];
      wht8(v);
#pragma unroll
      for (int k = 0; k < 8; k++) w[r * n + c8 + k] = v[k];
    }
    __syncthreads();
    // one thread per (8x8 block, column); block sums need the per-block rounding,
    // so accumulate per block in shared memory
    int* bsum = w + n * n;  // (n/8)^2 <= 64 ints
    for (int i = threadIdx.x; i < (n >> 3) * (n >> 3); i += blockDim.x) bsum[i] = 0;
    __syncthreads();
    for (int item = threadIdx.x; item < (n * n) >> 3; item += blockDim.x) {
      int col = item % n, br = item / n;  // br: 8-row band
      int v[8];
#pragma unroll
      for (int k = 0; k < 8; k++) v[k] = w[(br * 8 + k) * n + col];
      wht8(v);
      int s = 0;
#pragma unroll
      for (int k = 0; k < 8; k++) s += abs(v[k]);
      atomicAdd(&bsum[br * (n >> 3) + (col >> 3)], s);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (n >> 3) * (n >> 3); i += blockDim.x) acc += (bsum[i] + 4) >> 3;
  }
  // CTA reduction: shuffles inside a warp, then across warps
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) partial[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int i = 0; i < kThreads / 32; i++) total += partial[i];
    if (use_satd && ln == 2) total = (total + 2) >> 2;
    result[blockIdx.x] = total;
  }
}

// Stand-alone single-MV prediction of a list of blocks into packed buffers
// (the mc_predict1fmv vtable slot, batched).  dst block q occupies n_x*n_y
// bytes at dst + q*dst_pitch.
__global__ void __launch_bounds__(kThreads)
k_predict1fmv(const unsigned char* __restrict__ ref, int ref_stride, unsigned char* __restrict__ dst,
              int dst_pitch, const daala_b200_match_job* __restrict__ jobs, int log_yblk_override) {
  __shared__ unsigned char pred[kMaxN * kMaxN];
  __shared__ short buf[(kMaxN + kApron) * kMaxN];
  const daala_b200_match_job job = jobs[blockIdx.x];
  const int lx = job.log_blk, ly = log_yblk_override >= 0 ? log_yblk_override : lx;
  predict_block(pred, buf, ref + (size_t)job.y0 * ref_stride + job.x0, ref_stride, job.mvx, job.mvy, lx, ly);
  unsigned char* out = dst + (size_t)blockIdx.x * dst_pitch;
  for (int i = threadIdx.x; i < (1 << (lx + ly)); i += blockDim.x) out[i] = pred[i];
}

// Blend of four packed predictions (row stride nx each, `pitch` bytes apart):
// the stand-alone mc_blend_full / mc_blend_full_split vtable slots.
__global__ void __launch_bounds__(kThreads)
k_blend_packed(const unsigned char* __restrict__ preds, int pitch, unsigned char* __restrict__ dst,
               int dst_stride, int oc, int s, int lx, int ly) {
  const int nx = 1 << lx, ny = 1 << ly;
  const unsigned char* p0 = preds;
  const unsigned char* p1 = preds + pitch;
  const unsigned char* p2 = preds + 2 * pitch;
  const unsigned char* p3 = preds + 3 * pitch;
  const SplitWeights w = split_weights(oc, s == 3 ? 3 : s, lx, ly);
  for (int idx = threadIdx.x + blockIdx.x * blockDim.x; idx < nx * ny; idx += blockDim.x * gridDim.x) {
    int i = idx & (nx - 1), j = idx >> lx;
    if (s == 3) {
      const int l2 = lx + ly;
      int a = p0[idx], c = p3[idx];
      a = (a << lx) + (p1[idx] - a) * i;
      c = (c << lx) + (p2[idx] - c) * i;
      dst[(size_t)j * dst_stride + i] = (unsigned char)(((a << ly) + (c - a) * j + (1 << (l2 - 1))) >> l2);
    } else {
      const int l2p1 = lx + ly + 1;
      int a = p0[idx];
      int acc = (a << l2p1) + (p1[idx] - a) * (w.s0[1] + j * w.dsdj[1] + i * (w.dsdi[1] + j * w.dd[1]))
                + (p2[idx] - a) * (w.s0[2] + j * w.dsdj[2] + i * (w.dsdi[2] + j * w.dd[2]))
                + (p3[idx] - a) * (w.s0[3] + j * w.dsdj[3] + i * (w.dsdi[3] + j * w.dd[3]));
      dst[(size_t)j * dst_stride + i] = (unsigned char)((acc + (1 << (l2p1 - 1))) >> l2p1);
    }
  }
}


// od_mv_est_bma_sad (src/mcenc.c:2224) for one candidate per CTA: per plane the single-MV prediction of the
// displaced block (half-pel BMA vector scaled to the plane, mc_predict1fmv) and its SAD against the current
// picture through od_enc_sad's clipping to the active picture region (src/mcenc.c:1615-1680: blocks hang over
// the picture edge, and over its top / left for the centred BMA blocks); chroma SADs enter >> OD_MC_CHROMA_SCALE.
struct BmaPlanes {
  const unsigned char* cur[3];
  const unsigned char* ref[3];
  int cur_stride[3], ref_stride[3];
  int pic_w, pic_h, nplanes;
};

__global__ void __launch_bounds__(kThreads)
k_bma_sad(const __grid_constant__ BmaPlanes P, const daala_b200_bma_job* __restrict__ jobs, int32_t* __restrict__ result) {
  __shared__ __align__(16) unsigned char pred[kMaxN * kMaxN];
  __shared__ short buf[(kMaxN + kApron) * kMaxN];
  __shared__ int partial[kThreads / 32];
  const daala_b200_bma_job job = jobs[blockIdx.x];
  int total = 0;
  for (int pli = 0; pli < P.nplanes; pli++) {
    const int dec = pli > 0;
    const int ln = job.log_mvb_sz + 3 - dec, n = 1 << ln;   // OD_LOG_MVBSIZE_MIN = 3
    int x = job.bx >> dec, y = job.by >> dec;
    predict_block(pred, buf, P.ref[pli] + (ptrdiff_t)y * P.ref_stride[pli] + x, P.ref_stride[pli],
                  job.mvx * (1 << (2 - dec)), job.mvy * (1 << (2 - dec)), ln, ln);
    int w = n, h = n, px = 0, py = 0;
    if (x < 0) { w += x; px = -x; x = 0; }
    if (y < 0) { h += y; py = -y; y = 0; }
    const int plane_w = (P.pic_w + dec) >> dec, plane_h = (P.pic_h + dec) >> dec;   // OD_PLANE_SZ
    w = min(w, plane_w - x);
    h = min(h, plane_h - y);
    int acc = 0;
    if (w > 0 && h > 0) {
      const unsigned char* c0 = P.cur[pli] + (size_t)y * P.cur_stride[pli] + x;
      for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
        const int r = i / w, c = i - r * w;
        acc += abs((int)c0[(size_t)r * P.cur_stride[pli] + c] - (int)pred[(r + py) * n + c + px]);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) partial[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      int sad = 0;
      for (int k = 0; k < kThreads / 32; k++) sad += partial[k];
      total += sad >> (dec ? 2 : 0);
    }
    __syncthreads();   // pred / buf / partial are reused by the next plane
  }
  if (threadIdx.x == 0) result[blockIdx.x] = total;
}

// od_mv_est_sad (src/mcenc.c:2267): the OBMC prediction of a MV-grid block in every plane and its SAD against the
// current picture (od_enc_sad: clipped to the picture), chroma >> OD_MC_CHROMA_SCALE.  One CTA per candidate,
// blocks[3 * job + plane] = the plane's block record (od_state_pred_block_from_setup's MVs).
__global__ void __launch_bounds__(kThreads)
k_est_sad(const __grid_constant__ BmaPlanes P, const daala_b200_mc_block* __restrict__ blocks, int32_t* __restrict__ result) {
  __shared__ unsigned char pred[4][kMaxN * kMaxN];
  __shared__ short buf[(kMaxN + kApron) * kMaxN];
  __shared__ unsigned char blend[kMaxN * kMaxN];
  __shared__ int partial[kThreads / 32];
  int total = 0;
  for (int pli = 0; pli < P.nplanes; pli++) {
    const daala_b200_mc_block b = blocks[3 * blockIdx.x + pli];
    const int dec = pli > 0;
    const int nx = 1 << b.log_xblk, ny = 1 << b.log_yblk;
    obmc_block(blend, nx, pred, buf, P.ref[pli], P.ref_stride[pli], b);
    __syncthreads();
    const int plane_w = (P.pic_w + dec) >> dec, plane_h = (P.pic_h + dec) >> dec;   // OD_PLANE_SZ
    const int w = min(nx, plane_w - (int)b.x0), h = min(ny, plane_h - (int)b.y0);
    int acc = 0;
    if (w > 0 && h > 0) {
      const unsigned char* c0 = P.cur[pli] + (size_t)b.y0 * P.cur_stride[pli] + b.x0;
      for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
        const int r = i / w, c = i - r * w;
        acc += abs((int)c0[(size_t)r * P.cur_stride[pli] + c] - (int)blend[r * nx + c]);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) partial[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      int sad = 0;
      for (int k = 0; k < kThreads / 32; k++) sad += partial[k];
      total += sad >> (dec ? 2 : 0);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) result[blockIdx.x] = total;
}

}  // namespace mc
}  // namespace daala_b200

using namespace daala_b200::mc;

extern "C" {

int daala_b200_mv_est_sad(const uint8_t* const cur[3], const int cur_stride[3], const uint8_t* const ref[3],
                          const int ref_stride[3], int pic_w, int pic_h, int nplanes,
                          const daala_b200_mc_block* blocks, int count, int32_t* result, void* stream) {
  if (!cur || !ref || !blocks || !result || nplanes < 1 || nplanes > 3 || count < 0) return (int)cudaErrorInvalidValue;
  if (count == 0) return 0;
  daala_b200::mc::BmaPlanes P;
  for (int i = 0; i < 3; i++) {
    P.cur[i] = i < nplanes ? cur[i] : nullptr;
    P.ref[i] = i < nplanes ? ref[i] : nullptr;
    P.cur_stride[i] = i < nplanes ? cur_stride[i] : 0;
    P.ref_stride[i] = i < nplanes ? ref_stride[i] : 0;
  }
  P.pic_w = pic_w;
  P.pic_h = pic_h;
  P.nplanes = nplanes;
  daala_b200::mc::k_est_sad<<<count, daala_b200::mc::kThreads, 0, (cudaStream_t)stream>>>(P, blocks, result);
  return (int)cudaGetLastError();
}

int daala_b200_mv_bma_sad(const uint8_t* const cur[3], const int cur_stride[3], const uint8_t* const ref[3],
                                     const int ref_stride[3], int pic_w, int pic_h, int nplanes,
                                     const daala_b200_bma_job* jobs, int count, int32_t* result, void* stream) {
  if (!cur || !ref || !jobs || !result || nplanes < 1 || nplanes > 3 || count < 0) return (int)cudaErrorInvalidValue;
  if (count == 0) return 0;
  daala_b200::mc::BmaPlanes P;
  for (int i = 0; i < 3; i++) {
    P.cur[i] = i < nplanes ? cur[i] : nullptr;
    P.ref[i] = i < nplanes ? ref[i] : nullptr;
    P.cur_stride[i] = i < nplanes ? cur_stride[i] : 0;
    P.ref_stride[i] = i < nplanes ? ref_stride[i] : 0;
  }
  P.pic_w = pic_w;
  P.pic_h = pic_h;
  P.nplanes = nplanes;
  daala_b200::mc::k_bma_sad<<<count, daala_b200::mc::kThreads, 0, (cudaStream_t)stream>>>(P, jobs, result);
  return (int)cudaGetLastError();
}


int daala_b200_mc_predict_blocks(const uint8_t* ref, int ref_stride, uint8_t* dst, int dst_stride,
                                 const daala_b200_mc_block* blocks, int count, void* stream) {
  if (count <= 0) return 0;
  k_obmc_blocks<<<count, kThreads, 0, (cudaStream_t)stream>>>(ref, ref_stride, dst, dst_stride, blocks);
  return (int)cudaGetLastError();
}

int daala_b200_mc_match_candidates(const uint8_t* cur, int cur_stride, const uint8_t* ref, int ref_stride,
                                   const daala_b200_match_job* jobs, int count, int use_satd, int32_t* result,
                                   void* stream) {
  if (count <= 0) return 0;
  k_match_candidates<<<count, kThreads, 0, (cudaStream_t)stream>>>(cur, cur_stride, ref, ref_stride, jobs,
                                                                  use_satd, result);
  return (int)cudaGetLastError();
}

int daala_b200_mc_predict1fmv_batch(const uint8_t* ref, int ref_stride, uint8_t* dst, int dst_pitch,
                                    const daala_b200_match_job* jobs, int count, int log_yblk, void* stream) {
  if (count <= 0) return 0;
  k_predict1fmv<<<count, kThreads, 0, (cudaStream_t)stream>>>(ref, ref_stride, dst, dst_pitch, jobs, log_yblk);
  return (int)cudaGetLastError();
}

int daala_b200_mc_blend_packed(const uint8_t* preds, int pitch, uint8_t* dst, int dst_stride, int oc, int s,
                               int log_xblk, int log_yblk, void* stream) {
  k_blend_packed<<<1, kThreads, 0, (cudaStream_t)stream>>>(preds, pitch, dst, dst_stride, oc, s, log_xblk,
                                                            log_yblk);
  return (int)cudaGetLastError();
}

}  // extern "C"
