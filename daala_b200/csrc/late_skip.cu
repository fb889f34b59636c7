// The late-skip distortions of every block of a P-frame step (config.late_skip; include/daala_b200.h,
// daala_b200_kf_late_skip): od_block_encode's late-skip test (reference src/encode.c:1412-1450) compares
// od_compute_dist(c_orig, c_noskip) with od_compute_dist(c_orig, mc_orig), where c_orig / mc_orig are the prefiltered
// source / prediction of the block and c_noskip the leaf iDCT of what was coded.  The coded block depends on the DC
// and PVQ-skip decisions the host coder takes just before, but those have three outcomes besides od_pvq_encode's own
// skip, so the step computes all four distortions and the host picks one.
//
// c_orig and mc_orig are not stored anywhere: the lifting DCT is reversible, so they are the leaf iDCTs of the
// unquantised coefficients d_orig and of md.  Per block: five leaf iDCTs (c_orig, then the candidates mc_orig and the
// three noskip blocks, one at a time in a second tile) with the lifting networks of gen/dct_lifting.cuh (rows, then
// columns: od_bin_idctNxN), and four od_compute_dist with block_dist of dist_device.cuh.
//
// Mapping: k_late_skip_split sorts the blocks with bs > 0 into one list per size class and zeroes the records of 4x4
// blocks; then one launch per class, in which a 64-thread CTA takes 4096 samples at a time (64 8x8, 16 16x16, 4
// 32x32 or one 64x64 block), so every iDCT pass and the distortion's sub-block phase keep all 64 threads busy.
// Tiles have an odd row pitch (n + 1), which makes both iDCT passes bank-conflict free.
#include <cuda_runtime.h>
#include <stdint.h>

#include "daala_b200.h"
#include "dist_device.cuh"
#include "gen/dct_lifting.cuh"
#include "late_skip.h"

namespace daala_b200 {
namespace lateskip {

using dist::kDistThreads;

constexpr int kSamples = 4096;   // per CTA batch

// block i of the two lists together (luma first), or false past their end
__device__ __forceinline__ bool ls_block(const daala_b200_late_skip_batch& P, int i, int* list, int* blk) {
  const int nl = min(*P.count[0], P.max_blocks[0]), nc = min(*P.count[1], P.max_blocks[1]);
  if (i >= nl + nc) return false;
  *list = i >= nl;
  *blk = i >= nl ? i - nl : i;
  return true;
}

__global__ void __launch_bounds__(256) k_late_skip_split(const __grid_constant__ daala_b200_late_skip_batch P) {
  const int nth = gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  int list, blk;
  for (int base = blockIdx.x * blockDim.x; ; base += nth) {   // whole warps: the append is warp-aggregated
    const bool in = ls_block(P, base + (int)threadIdx.x, &list, &blk);
    if (!__any_sync(0xffffffffu, in)) break;
    int c = -1;
    if (in) {
      const int bs = P.blocks[list][blk].bs;
      if (bs == 0) P.out[list][blk] = daala_b200_kf_late_skip{0, 0, 0, 0};
      else c = bs - 1;
    }
    const unsigned same = __match_any_sync(0xffffffffu, c);
    const int leader = __ffs(same) - 1;
    int at = 0;
    if (c >= 0 && lane == leader) at = atomicAdd(&P.cls_n[c], __popc(same));
    at = __shfl_sync(0xffffffffu, at, leader) + __popc(same & ((1u << lane) - 1u));
    if (c >= 0 && at < P.cls_cap[c]) P.cls_items[P.cls_off[c] + at] = (uint32_t)blk | (list ? 0x80000000u : 0u);
  }
}

// od_bin_idctNxN of the g blocks of a tile (block k at tile + k * n * pitch): rows, then columns.
template <int LN>
__device__ __forceinline__ void idct_tile(int32_t* tile, int g) {
  constexpr int N = 1 << LN, P = N + 1;
#pragma unroll 1
  for (int pass = 0; pass < 2; pass++) {
    const bool cols = pass == 1;
    for (int m = threadIdx.x; m < g * N; m += kDistThreads) {
      const int k = m >> LN, r = m & (N - 1);
      int32_t* p = tile + k * N * P + (cols ? r : r * P);
      const int s = cols ? P : 1;
      int v[N];
#pragma unroll
      for (int q = 0; q < N; q++) v[q] = p[q * s];
      Lifting<N>::inv(v);
#pragma unroll
      for (int q = 0; q < N; q++) p[q * s] = v[q];
    }
    __syncthreads();
  }
}

template <int LN>
__global__ void __launch_bounds__(kDistThreads) k_late_skip(const __grid_constant__ daala_b200_late_skip_batch P) {
  constexpr int N = 1 << LN, NP = N * (N + 1), G = kSamples >> (2 * LN);
  extern __shared__ __align__(16) int32_t smem[];
  int32_t* scratch = smem;                                              // block_dist's
  int32_t* A = smem + dist::dist_scratch_bytes(N, G) / 4;              // c_orig of each slot
  int32_t* B = A + G * NP;                                             // the candidate being scored
  __shared__ const int32_t* s_dor[G];
  __shared__ const int32_t* s_d[G];
  __shared__ const int32_t* s_md[G];
  __shared__ int s_stride[G];
  __shared__ int32_t s_dc[G][2];                                       // md[0], md[0] + q1 * dc_quant
  __shared__ double s_scale[G];                                        // the slot's frame's dist_scale
  const int c = LN - 3;
  const int n = min(P.cls_n[c], (int)P.cls_cap[c]);
  const uint32_t* items = P.cls_items + P.cls_off[c];
  const int t = threadIdx.x;
  for (int b0 = blockIdx.x * G; b0 < n; b0 += gridDim.x * G) {
    if (t < G) {
      s_dor[t] = nullptr;
      if (b0 + t < n) {
        const uint32_t id = items[b0 + t];
        const daala_b200_pvq_block b = P.blocks[id >> 31][id & 0x7fffffffu];
        const int stride = P.plane_stride[b.pli];
        const size_t o = b.frame * P.plane_pitch[b.pli] + (size_t)b.y0 * stride + b.x0;
        s_dor[t] = P.d_orig[b.pli] + o;
        s_d[t] = P.d[b.pli] + o;
        s_md[t] = P.md[b.pli] + o;
        s_stride[t] = stride;
        const int dc_quant = P.fq_bq[(b.frame * 3 + b.pli) * 32 + b.bs * (b.bs + 1)];
        const int32_t md0 = s_md[t][0], resid = s_dor[t][0] - md0;
        const int half = ((dc_quant + 1) >> 1) - 1;
        const int32_t q1 = (resid + (resid < 0 ? -half : half)) / dc_quant;   // OD_DIV_R0 (src/odintrin.h:123)
        s_dc[t][0] = md0;
        s_dc[t][1] = md0 + q1 * dc_quant;
        s_scale[t] = dist::dist_scale(P.fq[b.frame].coded_quantizer);
      }
    }
    __syncthreads();
    // candidate -1: c_orig into A; 0: mc_orig; 1: coded AC, DC md[0]; 2: coded AC, DC q1; 3: md, DC q1
    daala_b200_kf_late_skip rec;
#pragma unroll 1
    for (int cand = -1; cand < 4; cand++) {
      int32_t* dst = cand < 0 ? A : B;
      for (int idx = t; idx < G * N * N; idx += kDistThreads) {
        const int k = idx >> (2 * LN), i = (idx >> LN) & (N - 1), j = idx & (N - 1);
        int32_t v = 0;
        if (s_dor[k]) {
          const int32_t* src = cand < 0 ? s_dor[k] : cand == 1 || cand == 2 ? s_d[k] : s_md[k];
          v = idx & (N * N - 1) ? src[(size_t)i * s_stride[k] + j] : cand <= 0 ? src[0] : s_dc[k][cand != 1];
        }
        dst[k * NP + i * (N + 1) + j] = v;
      }
      __syncthreads();
      idct_tile<LN>(dst, G);
      if (cand >= 0) {
        // the HVS totals are scaled per slot at the end (the scale is block_dist's last multiplication; x * 1.0 is
        // exact)
        const double d = dist::block_dist(A, N + 1, NP, B, N + 1, NP, LN, G, P.qm_is_flat, P.use_activity_masking, 1.0,
                                          scratch);
        if (cand == 0) rec.dist_skip = d;
        else if (cand == 1) rec.noskip_coded_dc0 = d;
        else if (cand == 2) rec.noskip_coded_dcq = d;
        else rec.noskip_pred_dcq = d;
      }
    }
    if (t < G && b0 + t < n) {
      if (!P.qm_is_flat) {
        const double sc = s_scale[t];
        rec.dist_skip *= sc;
        rec.noskip_coded_dc0 *= sc;
        rec.noskip_coded_dcq *= sc;
        rec.noskip_pred_dcq *= sc;
      }
      const uint32_t id = items[b0 + t];
      P.out[id >> 31][id & 0x7fffffffu] = rec;
    }
    __syncthreads();
  }
}

template <int LN>
static int launch(const daala_b200_late_skip_batch* b, int ctas, cudaStream_t s) {
  constexpr int N = 1 << LN, G = kSamples >> (2 * LN);
  const int smem = dist::dist_scratch_bytes(N, G) + 2 * G * N * (N + 1) * (int)sizeof(int32_t);
  cudaError_t e = cudaFuncSetAttribute(k_late_skip<LN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  k_late_skip<LN><<<ctas, kDistThreads, smem, s>>>(*b);
  return (int)cudaGetLastError();
}

}  // namespace lateskip
}  // namespace daala_b200

using namespace daala_b200::lateskip;

long long daala_b200_late_skip_class_caps(long long px, long long off[4], long long cap[4]) {
  long long total = 0;
  for (int c = 0; c < 4; c++) {
    const long long n = 8ll << c;
    off[c] = total;
    cap[c] = px / (n * n) + 64;
    total += cap[c];
  }
  return total;
}

int daala_b200_late_skip_enqueue(const daala_b200_late_skip_batch* b, int ctas, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(b->cls_n, 0, 4 * sizeof(int32_t), s);
  if (e != cudaSuccess) return (int)e;
  k_late_skip_split<<<ctas, 256, 0, s>>>(*b);
  int rc = launch<3>(b, ctas, s);
  if (!rc) rc = launch<4>(b, ctas, s);
  if (!rc) rc = launch<5>(b, ctas, s);
  if (!rc) rc = launch<6>(b, ctas, s);
  return rc ? rc : (int)cudaGetLastError();
}
