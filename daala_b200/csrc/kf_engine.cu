// Keyframe engine: the whole per-block encode hot path of a batch of keyframes as ONE device-resident,
// CUDA-graph-captured step behind a C ABI that takes HOST buffers (include/daala_b200.h, "Keyframe
// engine").  It is the batched equivalent of od_encode_coefficients (reference src/encode.c:2539) for
// keyframes minus the serial entropy coder:
//
//   u8 planes + state->bsize maps
//     -> work lists built ON THE DEVICE from the block-size maps (every step; a live encoder changes
//        block sizes every frame): leaf-block descriptors by a prefix scan over the 8x8 units, same-size
//        top / left neighbours of od_hv_intra_pred (src/intra.c:46-47), per size class the (block, band)
//        items counting-sorted by their position along the intra-prediction dependency chains
//     -> fused lapped prefilter + fDCT (frame_transform.cu)
//     -> luma PVQ with the H/V intra predictor: ONE persistent kernel, warps pull items by ticket in
//        dependency order and wait on per-(block, band) flags of the neighbours they read
//        (acquire / release) -- no per-wave launches
//     -> chroma-from-luma prediction + CfL flip + chroma PVQ (same persistent kernel, no dependencies)
//     -> iDCT + lapped postfilters -> u8 reconstruction, packed symbols for the host entropy coder
//     -> (config.symbol_stream) the same symbols per frame in bitstream order with 8/16-bit pulses.
//
// config.inter: the residual of a batch of P frames the same way.  The motion-compensated prediction planes are
// a second input (config.inter_mc: made in the graph from MV grids and a pool of reference pictures, before the
// forward transform; config.mc_next adds B frames: a NEXT picture per frame and each vertex's second vector mv1);
// they take the same forward transform (no DC Haar pyramid on either side) and their
// coefficients `md` are the reference vector of every band (pvq_theta with is_keyframe = 0).  Without an intra
// predictor every (block, band) of every plane is dependency-free: luma and chroma both go through the three
// phase kernels (k_pvq_split) and the persistent chain kernel is not launched.  config.late_skip adds the four
// late-skip distortions of every block (late_skip.cu) after the finishing scatter of both stages.
//
// Nothing returns to the host between the H2D of the inputs and the D2H of the results; list sizes
// live in device memory (`cnt`), every kernel is launched with a fixed grid and loops / pulls tickets
// up to the device-side counts, so the step is captured once into a CUDA graph.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <new>
#include <vector>

#include "daala_b200.h"
#include "dering_search.h"
#include "late_skip.h"
#include "lossless.h"
#include "haar_dc.h"
#include "mc_batch.h"
#include "gen/coding_order.inc"
#include "pvq_math.cuh"
#include "pvq_warp.cuh"
#include "pvq_common.cuh"

namespace daala_b200 {
namespace kf {

using namespace daala_b200::pvq;

// ---- device-side counters ----------------------------------------------------------------------
enum Cnt {
  kNLuma = 0, kNChroma, kLumaCoefs, kChromaCoefs,
  kNItemsL = 4,      // [3] luma dependency-free items per class (bands 3 / 6: classes 1 / 2; inter: every band)
  kNItemsC = 7,      // [3] chroma items per class (n <= 16, 32, 128)
  kTotalHi = 14,     // luma chain items in total
  kNHeads = 15,      // row / column chain items ready from the start (no same-size neighbour to wait for)
  kNHeads0 = 16,     // band-0 items ready from the start
  kError = 17,
  kDepsDone = 18,    // CTAs of k_luma_deps that have finished (the last one scans the chain heads' weight bins)
  kMcBadRef = 19,    // config.inter_mc: leaf corners whose vertex has a ref other than GOLD / PREV (/ NEXT: mc_next)
  kMcBeyond = 20,    //                  corner windows reaching past the reference's edge extension
  // the words the persistent kernels hammer with atomics each sit in a 128-byte line of their own
  kHeadLoL = 32,     // ticket of the luma dependency-free lists
  kHeadLoC = 64,     // ticket of the chroma lists
  kHeadHi = 96,      // luma chain queue: next slot to claim
  kTailHi = 128,     //                   next slot to fill
  kDoneHi = 160,     // band-0 items finished (flushed by warps when they go idle)
  kHeadCh = 192,     // ticket of the row / column chain heads
  kWaiters = 224,    // warps parked on a future band-0 slot
  kTraceN = 240,     // DAALA_B200_CHAIN_TRACE: records written by k_pvq_persist
  kCntWords = 256
};

constexpr int kTile = 1024;        // units per scan tile
// weight bins of the chain heads (weight_bin); the count sets how finely k_chroma_items orders the heads
constexpr int kHeadBins = 12288;

struct Lists {
  const uint8_t* bsize;            // [F][UH][bstride]
  int bstride;
  long long bsize_pitch;
  int F, UW, UH;                   // 8x8-luma units per frame
  int u_row0, u_rows;              // unit rows of this rank's shard
  int ntiles;
  int4* tile_sum;                  // [ntiles] then exclusive prefixes in place
  int32_t* unit_lbase;             // [F*UH*UW] index of the first luma block whose origin is in the unit
  // keyframes: [F*UH*UW] coding offset of the first luma block of a unit with block origins (the CfL source of its
  // chroma blocks); kept from the last step that listed them, zero before; NULL on inter engines
  int32_t* unit_loff;
  daala_b200_pvq_block* luma;
  daala_b200_pvq_block* chroma;
  int32_t* dep_top;                // same-size neighbour above / to the left (od_hv_intra_pred), or -1
  int32_t* dep_left;
  int32_t* succ_bottom;            // inverse: the block whose dep_top / dep_left is this one, or -1
  int32_t* succ_right;
  uint32_t* items_l[3];            // dependency-free luma items per class
  uint32_t* items_c[3];
  uint32_t* heads;                 // row / column chain items that are ready from the start, heaviest chain first
  uint32_t* heads0;                // band-0 items that are ready from the start
  // chain heads as k_luma_deps finds them, each with its bin in descending order of chain weight; k_luma_deps
  // counts the bins and its last CTA scans them, k_chroma_items scatters the heads into `heads`
  uint32_t* heads_raw;
  int32_t* head_bin;
  int32_t* head_hist;              // [kHeadBins] counts, then exclusive offsets
  int32_t* head_cursor;            // [kHeadBins]
  int32_t* cnt;                    // [kCntWords]
  int max_luma, max_chroma;        // capacities (blocks)
};

__device__ __forceinline__ int4 add4(int4 a, int4 b) { return make_int4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

// (luma blocks, luma coefficients, chroma blocks per plane, chroma coefficients per plane) whose
// origin lies in unit (ux, uy): leaf rule of od_compute_dcts / od_encode_recursive
// (src/encode.c:1466-1470: the size is read at the block's top-left unit; bs = max(obs, xdec)).
__device__ __forceinline__ int4 unit_counts(int b, int ux, int uy) {
  if (b == 0) return make_int4(4, 64, 1, 16);
  const int span = 1 << (b - 1);
  if ((ux & (span - 1)) | (uy & (span - 1))) return make_int4(0, 0, 0, 0);
  const int lc = b == 1 ? 64 : b == 2 ? 256 : 512;
  const int cc = b == 1 ? 16 : b == 2 ? 64 : b == 3 ? 256 : 512;
  return make_int4(1, lc, 1, cc);
}

__device__ __forceinline__ bool unit_of(const Lists& L, long long i, int* f, int* uy, int* ux, int* b) {
  const long long per = (long long)L.u_rows * L.UW;
  if (i >= per * L.F) return false;
  *f = (int)(i / per);
  const int r = (int)(i - (long long)*f * per);
  *uy = L.u_row0 + r / L.UW;
  *ux = r % L.UW;
  *b = L.bsize[*f * L.bsize_pitch + (long long)*uy * L.bstride + *ux];
  return true;
}

__global__ void __launch_bounds__(kTile) k_unit_tile_sums(const __grid_constant__ Lists L) {
  __shared__ int4 part[32];
  const long long i = (long long)blockIdx.x * kTile + threadIdx.x;
  int f, uy, ux, b;
  int4 v = make_int4(0, 0, 0, 0);
  if (unit_of(L, i, &f, &uy, &ux, &b)) v = unit_counts(b, ux, uy);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
    v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    v.z += __shfl_xor_sync(0xffffffffu, v.z, o);
    v.w += __shfl_xor_sync(0xffffffffu, v.w, o);
  }
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    int4 s = make_int4(0, 0, 0, 0);
    for (int w = 0; w < kTile / 32; w++) s = add4(s, part[w]);
    L.tile_sum[blockIdx.x] = s;
  }
}

// One CTA: exclusive scan of the tile sums, totals, reset of the per-step counters, new epoch.
__global__ void __launch_bounds__(1024) k_tile_scan(const __grid_constant__ Lists L) {
  __shared__ int4 part[1024];
  __shared__ int4 carry;
  const int t = threadIdx.x;
  if (t == 0) carry = make_int4(0, 0, 0, 0);
  __syncthreads();
  for (int base = 0; base < L.ntiles; base += 1024) {
    const int i = base + t;
    const int4 v = i < L.ntiles ? L.tile_sum[i] : make_int4(0, 0, 0, 0);
    part[t] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const int4 a = t >= o ? part[t - o] : make_int4(0, 0, 0, 0);
      __syncthreads();
      part[t] = add4(part[t], a);
      __syncthreads();
    }
    const int4 incl = part[t], c = carry;
    if (i < L.ntiles) L.tile_sum[i] = make_int4(c.x + incl.x - v.x, c.y + incl.y - v.y, c.z + incl.z - v.z, c.w + incl.w - v.w);
    __syncthreads();
    if (t == 1023) carry = add4(c, incl);
    __syncthreads();
  }
  if (t == 0) {
    const int4 tot = carry;
    L.cnt[kNLuma] = tot.x;
    L.cnt[kLumaCoefs] = tot.y;
    L.cnt[kNChroma] = 2 * tot.z;
    L.cnt[kChromaCoefs] = 2 * tot.w;
    for (int c = 0; c < 3; c++) {
      L.cnt[kNItemsL + c] = 0;
      L.cnt[kNItemsC + c] = 0;
    }
    L.cnt[kTotalHi] = 0;
    L.cnt[kNHeads] = 0;
    L.cnt[kNHeads0] = 0;
    L.cnt[kDepsDone] = 0;
    // set on every step, so that an over-capacity batch does not flag the batches after it
    L.cnt[kError] = tot.x > L.max_luma || 2 * tot.z > L.max_chroma ? 1 : 0;
  }
}

__device__ __forceinline__ void put_block(daala_b200_pvq_block* dst, int coef_off, int x0, int y0, int bs, int pli,
                                          int xdec, int frame) {
  // one 12-byte record = three 32-bit stores
  int32_t* w = reinterpret_cast<int32_t*>(dst);
  w[0] = coef_off;
  w[1] = (x0 & 0xffff) | (y0 << 16);
  w[2] = bs | (pli << 8) | (xdec << 16) | (frame << 24);
}

__global__ void __launch_bounds__(kTile) k_unit_emit(const __grid_constant__ Lists L) {
  __shared__ int4 wsum[32];
  const long long i = (long long)blockIdx.x * kTile + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int f = 0, uy = 0, ux = 0, b = 0;
  const bool valid = unit_of(L, i, &f, &uy, &ux, &b);
  const int4 v = valid ? unit_counts(b, ux, uy) : make_int4(0, 0, 0, 0);
  int4 s = v;  // inclusive warp scan
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int4 a;
    a.x = __shfl_up_sync(0xffffffffu, s.x, o);
    a.y = __shfl_up_sync(0xffffffffu, s.y, o);
    a.z = __shfl_up_sync(0xffffffffu, s.z, o);
    a.w = __shfl_up_sync(0xffffffffu, s.w, o);
    if (lane >= o) s = add4(s, a);
  }
  if (lane == 31) wsum[warp] = s;
  __syncthreads();
  int4 pre = L.tile_sum[blockIdx.x];
  for (int w = 0; w < warp; w++) pre = add4(pre, wsum[w]);
  pre = make_int4(pre.x + s.x - v.x, pre.y + s.y - v.y, pre.z + s.z - v.z, pre.w + s.w - v.w);
  if (!valid) return;
  L.unit_lbase[((long long)f * L.UH + uy) * L.UW + ux] = pre.x;
  if (v.x == 0) return;
  if (pre.x + v.x > L.max_luma || 2 * (pre.z + v.z) > L.max_chroma) return;   // flagged by k_tile_scan
  if (L.unit_loff) L.unit_loff[((long long)f * L.UH + uy) * L.UW + ux] = pre.y;
  if (b == 0) {
    for (int q = 0; q < 4; q++)
      put_block(L.luma + pre.x + q, pre.y + 16 * q, ux * 8 + (q & 1) * 4, uy * 8 + (q >> 1) * 4, 0, 0, 0, f);
  } else {
    put_block(L.luma + pre.x, pre.y, ux * 8, uy * 8, b, 0, 0, f);
  }
  // 4:2:0 chroma: bs = max(obs, 1) - 1; bit 7 of xdec: the co-located luma is coded as 4x4 blocks
  // (od_resample_luma_coeffs' chroma_bs == 0 case, src/intra.c:78)
  const int cbs = (b > 1 ? b : 1) - 1;
  const int xd = 1 | (b == 0 ? 0x80 : 0);
  put_block(L.chroma + 2 * pre.z, 2 * pre.w, ux * 4, uy * 4, cbs, 1, xd, f);
  put_block(L.chroma + 2 * pre.z + 1, 2 * pre.w + v.w, ux * 4, uy * 4, cbs, 2, xd, f);
}

__device__ __forceinline__ int band_class(int band) { return band < 3 ? 0 : band < 6 ? 1 : 2; }

// warp-aggregated append of `v` to list[*counter] by the lanes with `pred`; the index written, or -1
__device__ __forceinline__ int append(uint32_t* list, int32_t* counter, bool pred, uint32_t v) {
  const unsigned m = __ballot_sync(__activemask(), pred);
  if (!pred) return -1;
  const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(counter, __popc(m));
  base = __shfl_sync(m, base, leader);
  const int pos = base + __popc(m & ((1u << lane) - 1u));
  list[pos] = v;
  return pos;
}

// warp-aggregated atomicAdd(&ctr[key], 1) by the calling lanes; the old value of the lane's own slot
__device__ __forceinline__ int count_key(int32_t* ctr, int key) {
  const unsigned same = __match_any_sync(__activemask(), key);
  const int lane = threadIdx.x & 31, leader = __ffs(same) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(&ctr[key], __popc(same));
  return __shfl_sync(same, base, leader) + __popc(same & ((1u << lane) - 1u));
}

// Cost of one chain item per band class (n <= 16, 32, 128 coefficients) in units of 10 us: the mean duration of an
// item of the class in k_pvq_persist while every warp is busy, 73 / 89 / 178 us on bench.py's workload (one
// H100 80GB HBM3 at 700 W, tools/chain_timeline.py, DESIGN.md section 5).  A chain's weight is its length in blocks
// times this; the bin of the weight orders the chain heads.
constexpr int kChainCost0 = 7, kChainCost1 = 9, kChainCost2 = 18;
__device__ __forceinline__ int weight_bin(int len, int band) {
  const int c = band_class(band);
  const int w = len * (c == 0 ? kChainCost0 : c == 1 ? kChainCost1 : kChainCost2);
  return kHeadBins - 1 - min(w, kHeadBins - 1);   // heaviest first
}

// Length in blocks of the column (down) or row chain that starts at the block (x0, y0, bs) of `map`: its
// same-size successors, by the test k_luma_deps uses for dep_top / dep_left, inside the coded unit rows.
__device__ int chain_length(const Lists& L, const uint8_t* map, int x0, int y0, int bs, bool down) {
  const int nn = 4 << bs, y_end = (L.u_row0 + L.u_rows) * 8, x_end = L.UW * 8;
  int len = 1;
  for (int x = x0 + (down ? 0 : nn), y = y0 + (down ? nn : 0); x < x_end && y < y_end;
       x += down ? 0 : nn, y += down ? nn : 0, len++) {
    if (map[(long long)(y >> 3) * L.bstride + (x >> 3)] != bs) break;
    const int py = down ? y - 1 : y, px = down ? x : x - 1;
    if (map[(long long)(py >> 3) * L.bstride + (px >> 3)] != bs) break;
  }
  return len;
}

// One CTA of kThreads: exclusive scan of kHeadBins counts in place (+ a copy as scatter cursors).  The counts are
// read past L1: the last CTA of k_luma_deps scans what the other CTAs of that launch counted.
template <int kThreads>
__device__ __forceinline__ void scan_bins(int32_t* hist, int32_t* cursor) {
  __shared__ int part[kThreads];
  constexpr int kPer = kHeadBins / kThreads;
  const int t = threadIdx.x;
  int v[kPer], sum = 0;
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    v[i] = __ldcg(hist + t * kPer + i);
    sum += v[i];
  }
  part[t] = sum;
  __syncthreads();
  for (int o = 1; o < kThreads; o <<= 1) {
    const int add = t >= o ? part[t - o] : 0;
    __syncthreads();
    part[t] += add;
    __syncthreads();
  }
  int run = part[t] - sum;
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    hist[t * kPer + i] = run;
    cursor[t * kPer + i] = run;
    run += v[i];
  }
}

// Luma dependency structure.  od_hv_intra_pred (src/intra.c:37) predicts band b of a block from band b of
// the same-size TOP neighbour (row-0 bands 1/4/7), the LEFT one (column-0 bands 2/5/8), both (band 0) or
// nothing (bands 3/6).  Per block: the two neighbours and, inverted, the blocks that wait for this one;
// per (block, band): a dependency-free item, a chain head (ready now) or a chain link (made ready by the
// persistent kernel when its neighbours are done).  Row / column chain heads also get the weight bin of their chain.
__global__ void __launch_bounds__(256) k_luma_deps(const __grid_constant__ Lists L) {
  const int n = min(L.cnt[kNLuma], L.max_luma);
  const int nth = gridDim.x * blockDim.x;
  for (int base = blockIdx.x * blockDim.x; base < n; base += nth) {
    const int blk = base + threadIdx.x;
    const bool in = blk < n;
    int bs = 0, top = -1, left = -1;
    if (in) {
      const daala_b200_pvq_block b = L.luma[blk];
      const int x0 = b.x0, y0 = b.y0, f = b.frame;
      bs = b.bs;
      const int nn = 4 << bs;
      const uint8_t* map = L.bsize + f * L.bsize_pitch;
      if (y0 - nn >= L.u_row0 * 8 && map[(long long)((y0 - 1) >> 3) * L.bstride + (x0 >> 3)] == bs) {
        const int ty = y0 - nn;
        top = L.unit_lbase[((long long)f * L.UH + (ty >> 3)) * L.UW + (x0 >> 3)] +
              (bs == 0 ? ((ty >> 2) & 1) * 2 + ((x0 >> 2) & 1) : 0);
      }
      if (x0 > 0 && map[(long long)(y0 >> 3) * L.bstride + ((x0 - 1) >> 3)] == bs) {
        const int lx = x0 - nn;
        left = L.unit_lbase[((long long)f * L.UH + (y0 >> 3)) * L.UW + (lx >> 3)] +
               (bs == 0 ? ((y0 >> 2) & 1) * 2 + ((lx >> 2) & 1) : 0);
      }
      L.dep_top[blk] = top;
      L.dep_left[blk] = left;
      if (top >= 0) L.succ_bottom[top] = blk;      // succ_* were preset to -1
      if (left >= 0) L.succ_right[left] = blk;
    }
    const int nb = in ? num_bands(bs) : 0;
    // lengths of the column / row chains this block starts (the same for every band of a size class)
    int len_down = 0, len_across = 0;
    if (nb > 1) {
      const daala_b200_pvq_block b = L.luma[blk];
      const uint8_t* map = L.bsize + b.frame * L.bsize_pitch;
      if (top < 0) len_down = chain_length(L, map, b.x0, b.y0, bs, true);
      if (left < 0) len_across = chain_length(L, map, b.x0, b.y0, bs, false);
    }
    int chain = 0;
    for (int band = 0; band < 9; band++) {
      const bool has = band < nb;
      const bool is_free = band == 3 || band == 6;
      const int r = band % 3;
      const bool waits = band == 0 ? (top >= 0 || left >= 0) : r == 1 ? top >= 0 : left >= 0;
      const uint32_t item = ((uint32_t)blk << 4) | band;
      if (band == 3 || band == 6) {
        append(L.items_l[band_class(band)], &L.cnt[kNItemsL + band_class(band)], has, item);
      } else if (band == 0) {
        append(L.heads0, &L.cnt[kNHeads0], has && !waits, item);
      } else {
        const int pos = append(L.heads_raw, &L.cnt[kNHeads], has && !waits, item);
        if (pos >= 0) {
          const int bin = weight_bin(r == 1 ? len_down : len_across, band);
          L.head_bin[pos] = bin;
          count_key(L.head_hist, bin);
        }
      }
      chain += has && !is_free;
    }
    // total number of chain items
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) chain += __shfl_xor_sync(0xffffffffu, chain, o);
    if ((threadIdx.x & 31) == 0 && chain) atomicAdd(&L.cnt[kTotalHi], chain);
  }
  // the last CTA to finish scans the weight bins of the chain heads; k_chroma_items sorts them
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&L.cnt[kDepsDone], 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (last) {
    __threadfence();
    scan_bins<256>(L.head_hist, L.head_cursor);
  }
}

// Chroma items: no dependencies between blocks; compaction per class (order is free).  Keyframes: first the luma
// chain heads into `heads` by the weight bins k_luma_deps scanned, heaviest first (the order inside a bin is free).
__global__ void __launch_bounds__(256) k_chroma_items(const __grid_constant__ Lists L) {
  const int nh = L.cnt[kNHeads];   // 0 in inter mode
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nh; i += gridDim.x * blockDim.x)
    L.heads[count_key(L.head_cursor, L.head_bin[i])] = L.heads_raw[i];
  const int n = min(L.cnt[kNChroma], L.max_chroma);
  for (int blk = blockIdx.x * blockDim.x + threadIdx.x; blk < n; blk += gridDim.x * blockDim.x) {
    const int bs = L.chroma[blk].bs;
    const int nb = num_bands(bs);
    for (int band = 0; band < nb; band++) {
      const int c = band_class(band);
      // warp-aggregated append
      const unsigned m = __activemask();
      const unsigned same = __match_any_sync(m, c);
      const int leader = __ffs(same) - 1, lane = threadIdx.x & 31;
      int base = 0;
      if (lane == leader) base = atomicAdd(&L.cnt[kNItemsC + c], __popc(same));
      base = __shfl_sync(same, base, leader);
      L.items_c[c][base + __popc(same & ((1u << lane) - 1u))] = ((uint32_t)blk << 4) | band;
    }
  }
}

// Inter frames: no intra predictor, so every luma (block, band) is a dependency-free item as well; item
// encoding and classes of k_chroma_items, in place of k_luma_deps.
__global__ void __launch_bounds__(256) k_luma_items(const __grid_constant__ Lists L) {
  const int n = min(L.cnt[kNLuma], L.max_luma);
  const int nth = gridDim.x * blockDim.x;
  for (int base = blockIdx.x * blockDim.x; base < n; base += nth) {   // whole warps: append() is warp-aggregated
    const int blk = base + threadIdx.x;
    const int nb = blk < n ? num_bands(L.luma[blk].bs) : 0;
    for (int band = 0; band < 9; band++) {
      const int c = band_class(band);
      append(L.items_l[c], &L.cnt[kNItemsL + c], band < nb, ((uint32_t)blk << 4) | band);
    }
  }
}

// ---- PVQ stage -----------------------------------------------------------------------------------
struct Stage {
  daala_b200_pvq_params prm;
  const uint32_t* items[3];        // dependency-free items per class (taken largest class first)
  // luma only: row / column chain heads, heaviest chain first (static list; a chain is then walked by one
  // warp), and the band-0 queue = [heads0 (static) | ring filled at run time]
  const uint32_t* heads;
  const uint32_t* heads0;
  uint32_t* ring;
  const int32_t* dep_top;
  const int32_t* dep_left;
  const int32_t* succ_bottom;
  const int32_t* succ_right;
  int32_t* join0;                  // [nblocks] band 0: neighbours finished so far (it may wait for two)
  int32_t* cnt;
  int n_items_at, head_lo_at, n_blocks_at;
  int max_blocks;
  // split path (phases as separate kernels over the dependency-free item lists): context records of one
  // chunk of items per class
  int16_t* sp_vec[3];              // [slots][3][vstride]
  int32_t* sp_lanes[3];            // [slots][kCtxLaneWords][16]
  int32_t* sp_uni[3];              // [slots][kCtxUniWords]
  int16_t* sp_snap[3];             // [slots][kMaxEvents][vstride]
  int sp_slots[3];                 // slots per chunk
  int sp_chunks[3];                // chunks that cover the list capacity of the class
  int max_waiters;                 // warps that may park on future band-0 slots; the others exit when idle
  const double* rsqrt_tbl;         // [kTableDoubles] the reference's 1/sqrt(i) and theta-rate terms (pvq_fill_rsqrt_table)
  int16_t* res_pack;               // [nblocks*9][4]: gain, itheta, max_theta, k (what the coder reads)
  // keyframe chroma: the CfL source, the luma stage's coding-order input (its DC) and output (the quantised
  // coefficients), and Lists::unit_loff; NULL otherwise.  config.haar_dc_quant: cfl_in is, in both keyframe stages,
  // the DC chain's grids of reconstructed DCs (hdc_grid), which the kHdc instantiations read in place of in[0]
  const int32_t* cfl_in;
  const int32_t* cfl_out;
  const int32_t* cfl_loff;
  int32_t* dc_resid;               // config.inter_finish or symbol_stream = 2: per block in[0] - ref[0], else NULL
  // [F][3][32] each frame's band quantisers max(1, q0 * pvq_qm_q4[pli][i] >> 4), filled on the host from the records
  // (one load per item)
  const int32_t* fq_bq;
#ifdef DAALA_B200_CHAIN_TRACE
  struct ChainTraceRec* trace;     // luma: one record per item k_pvq_persist runs, up to trace_cap
  int trace_cap;
#endif
};

#ifdef DAALA_B200_CHAIN_TRACE
// Timeline of the luma chain kernel, compiled only into the library tools/chain_timeline.py builds (the production
// kernel does not contain it).  32 bytes per item.
struct ChainTraceRec {
  unsigned long long t0, t1;       // %globaltimer (ns) when the warp started / finished the item
  uint32_t item;                   // (block << 4) | band
  uint32_t cta;                    // one warp per CTA
  uint16_t sm;
  uint8_t bs;
  uint8_t kind;                    // 0 band-0 queue slot, 1 row / column chain head, 2 free item, 3 chain successor
  uint32_t pad;
};

__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __noinline__ void trace_item(const Stage& S, uint32_t item, int kind, unsigned long long t0, int lane) {
  __syncwarp();
  if (lane != 0) return;
  const unsigned long long t1 = globaltimer();
  const int i = atomicAdd(&S.cnt[kTraceN], 1);
  if (i >= S.trace_cap) return;
  uint32_t sm;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
  ChainTraceRec r;
  r.t0 = t0;
  r.t1 = t1;
  r.item = item;
  r.cta = blockIdx.x;
  r.sm = (uint16_t)sm;
  r.bs = (uint8_t)S.prm.blocks[item >> 4].bs;
  r.kind = (uint8_t)kind;
  r.pad = 0;
  S.trace[i] = r;
}
#endif

// config.haar_dc_quant: the DC chain's grid of plane `pli` of frame `frame` (one entry per 4x4 unit, the leaf DCs at the
// leaf origins).  The grids of a frame lie together, planes 0, 1, 2: daala_b200_haar_dc_batch.grid_frame_pitch.
__device__ __forceinline__ const int32_t* hdc_grid(const Stage& S, int frame, int pli) {
  const long long g0 = S.prm.plane_frame_pitch[0] >> 4, g1 = S.prm.plane_frame_pitch[1] >> 4;
  return S.cfl_in + frame * (g0 + 2 * g1) + (pli ? g0 + (pli - 1) * g1 : 0);
}

// OD_CFL_SCALING4 (src/intra.c), indexed [column][row]
__constant__ int kCflScaling4[4][4] = {{128, 128, 100, 36}, {128, 80, 71, 35}, {100, 71, 35, 31}, {36, 35, 31, 18}};

// Chroma-from-luma reference of coefficient i (coding order) of keyframe chroma block b (od_resample_luma_coeffs,
// src/intra.c:72), read from the luma stage's coding-order buffers; `lo` is the coding offset of the co-located luma.
// Every block size codes the same nested layout (scan_rc does not depend on it) and a chroma block codes no more
// coefficients than its luma block (512 at most), so chroma index i is luma index i.  Position 0 is the luma DC of
// the plane k_finish_scatter writes on keyframes, the unquantised Haar DC in[0]; kHdc (config.haar_dc_quant): the
// quantised DC of the luma block at that place, from the DC chain's luma grid.
template <bool kHdc = false>
__device__ __forceinline__ int32_t cfl_ref(const Stage& S, const daala_b200_pvq_block& b, int lo, int i) {
  // luma 4x4 unit (u, v) of the block's co-located luma, in the luma grid of the block's frame
  auto ldc = [&](int u, int v) {
    return hdc_grid(S, b.frame, 0)[(long long)((b.y0 >> 1) + v) * (S.prm.plane_stride[0] >> 2) + (b.x0 >> 1) + u];
  };
  if (!(b.xdec & 0x80)) return i == 0 ? (kHdc ? ldc(0, 0) : S.cfl_in[lo]) : S.cfl_out[lo + i];
  // four 4x4 luma blocks (k_unit_emit: block q = 2 row + column, coefficients at lo + 16 q) -> one 4x4 chroma
  // prediction: od_tf_up_hv_lp (src/tf.c:82) + OD_CFL_SCALING4.  Output (r, c) comes from sample (r >> 1, c >> 1)
  // of each luma block; kScan4 lists rasters 4, 1, 5 first, so sample (y, x) of a 4x4 block is coefficient y + 2 x.
  int r = 0, c = 0;
  if (i) scan_rc(i, &r, &c);
  const int y = r >> 1, x = c >> 1, at = y + 2 * x;
  int ll = at ? S.cfl_out[lo + at] : kHdc ? ldc(0, 0) : S.cfl_in[lo];
  int lh = at ? S.cfl_out[lo + 16 + at] : kHdc ? ldc(1, 0) : S.cfl_in[lo + 16];
  int hl = at ? S.cfl_out[lo + 32 + at] : kHdc ? ldc(0, 1) : S.cfl_in[lo + 32];
  int hh = at ? S.cfl_out[lo + 48 + at] : kHdc ? ldc(1, 1) : S.cfl_in[lo + 48];
  ll += lh; hh -= hl;
  const int t = (ll - hh) >> 1;
  hl = t - hl; lh = t - lh;
  ll -= hl; hh += lh;
  // (2y + vs, 2x + hs) <- ll, (2y + vs, 2x + 1 - hs) <- lh, (2y + 1 - vs, 2x + hs) <- hl, the rest <- hh, with
  // vs = y, hs = x: the first kind of row is r = 3y, of column c = 3x
  const int v = r == 3 * y ? (c == 3 * x ? ll : lh) : (c == 3 * x ? hl : hh);
  return (kCflScaling4[c][r] * v + 64) >> 7;
}

// raster -> coding order of every block (od_raster_to_coding_order, src/partition.c:123); keyframe chroma:
// also the CfL prediction and its sign flip (src/pvq_encoder.c:847-871); inter frames, all planes alike: the
// reference vector is the transformed prediction md (prm.pred_plane), never flipped.  One warp per block.
enum { kGatherLuma = 0, kGatherChroma = 1, kGatherInter = 2 };
template <int kKind, bool kHdc = false>
__global__ void __launch_bounds__(256) k_gather(const __grid_constant__ Stage S) {
  const daala_b200_pvq_params& prm = S.prm;
  const int n = min(S.cnt[S.n_blocks_at], S.max_blocks);
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int blk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; blk < n; blk += nwarps) {
    const daala_b200_pvq_block b = prm.blocks[blk];
    const int ln = b.bs + 2;
    const int len = ln >= 5 ? 512 : 1 << (2 * ln);
    const int stride = prm.plane_stride[b.pli];
    const int32_t* src = prm.coef_plane[b.pli] + b.frame * prm.plane_frame_pitch[b.pli] + (size_t)b.y0 * stride + b.x0;
    int32_t* vin = prm.in + b.coef_off;
    if (kKind == kGatherLuma) {
      for (int i = lane; i < len; i += 32) vin[i] = i == 0 ? src[0] : src[scan_to_raster(i, ln, stride)];
    } else if (kKind == kGatherInter) {
      const int32_t* psrc = prm.pred_plane[b.pli] + b.frame * prm.plane_frame_pitch[b.pli] + (size_t)b.y0 * stride + b.x0;
      int32_t* vref = prm.ref + b.coef_off;
      for (int i = lane; i < len; i += 32) {
        const int at = i == 0 ? 0 : scan_to_raster(i, ln, stride);
        vin[i] = src[at];
        vref[i] = psrc[at];
      }
    } else {
      // the co-located luma at (2 x0, 2 y0): the unit of the block's origin (4x4 chroma samples) has its offset
      const int lo = S.cfl_loff[b.frame * (prm.plane_frame_pitch[b.pli] >> 4) + (long long)(b.y0 >> 2) * (stride >> 2) +
                                (b.x0 >> 2)];
      int32_t* vref = prm.ref + b.coef_off;
      const int qoff = prm.qm_stride + ((((1 << (2 * b.bs)) - 1) << 4) / 3);
      int32_t xy = 0;
      for (int i = lane; i < len; i += 32) {
        const int32_t vi = i == 0 ? src[0] : src[scan_to_raster(i, ln, stride)];
        const int32_t vr = cfl_ref<kHdc>(S, b, lo, i);
        vin[i] = vi;
        vref[i] = vr;
        if (i >= 1 && i < 16) {
          const int32_t rq = vr * prm.qm[qoff + i], inq = vi * prm.qm[qoff + i];
          xy += (int32_t)((rq * (int64_t)inq) >> ((kQmShift + 4) << 1));
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) xy += __shfl_xor_sync(0xffffffffu, xy, o);
      const int flip = xy < 0;
      __syncwarp();
      if (flip) {
        const int end = band_start(num_bands(b.bs));
        for (int i = 1 + lane; i < end; i += 32) vref[i] = -vref[i];
      }
      if (lane == 0) prm.res_flip[blk] = flip;
    }
  }
}

// One warp per CTA of the persistent kernel: a warp that runs out of work frees its registers and shared
// memory at once (a CTA only retires when all of its warps have), so the next kernel -- another engine's
// batch -- fills the SM while the last dependency chains of this one are still being walked.
constexpr int kPersistThreads = 32;
// resident CTAs per SM the persistent PVQ kernel is compiled for (register cap = 65536 / 32 / this = 64)
constexpr int kPersistCtas = 32;
// all of them resident: per CTA the warp's scratch (quantise_band_warp) plus the 1 KB the SM reserves, within
// the 228 KB of shared memory an sm_90 SM has (kf_alloc checks the same at run time)
static_assert(kPersistCtas * (kPersistThreads / 32 * kSnapEntries * (int)sizeof(int16_t) + 1024) <= 228 * 1024,
              "k_pvq_persist's shared scratch does not fit kPersistCtas CTAs per SM");
constexpr uint32_t kNoItem = 0xffffffffu;
constexpr uint32_t kExit = 0xfffffffeu;

__device__ __forceinline__ int ld_relaxed(const int32_t* p) {
  int v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void push_chain(const Stage& S, int blk, int band) {
  const int pos = atomicAdd(&S.cnt[kTailHi], 1) - S.cnt[kNHeads0];
  st_release((int*)&S.ring[pos], (int)(((uint32_t)blk << 4) | band));
}

// Next item for an idle warp of the luma stage (uniform), or kNoItem when the stage has nothing left for it.
// In this order: (1) a filled slot of the band-0 queue -- band 0 is a 2-D wavefront over each
//  same-size region, the deepest dependency structure of a frame, so it goes first; (2) the head of a row
//  or column chain; (3) a dependency-free item; (4) a ticket for a FUTURE band-0 slot, waited for on the
//  slot itself (distinct addresses: no hot spot).  `done` = band-0 items this warp finished since it was
//  last here; the warp whose flush completes the count releases every waiter with kExit.
__device__ __forceinline__ uint32_t next_item(const Stage& S, int lane, int* done, bool* waiter) {
  int slot = -1, head = -1, lo = -1, nheads0 = 0, fin = -1;
  if (lane == 0) {
    const int n2 = S.cnt[S.n_items_at + 2], n1 = S.cnt[S.n_items_at + 1], n0 = S.cnt[S.n_items_at];
    const int nlo = n0 + n1 + n2;
    nheads0 = S.cnt[kNHeads0];
    if (*done) {
      const int d = atomicAdd(&S.cnt[kDoneHi], *done) + *done;
      if (d == S.cnt[kNLuma]) {   // every luma block has a band 0
        __threadfence();
        fin = ld_relaxed(&S.cnt[kTailHi]) - nheads0;   // final: every push happened before its item finished
      }
    }
    if (ld_relaxed(&S.cnt[kHeadHi]) < ld_relaxed(&S.cnt[kTailHi])) slot = atomicAdd(&S.cnt[kHeadHi], 1);
    if (slot < 0 && ld_relaxed(&S.cnt[kHeadCh]) < S.cnt[kNHeads]) {
      const int h = atomicAdd(&S.cnt[kHeadCh], 1);
      if (h < S.cnt[kNHeads]) head = h;
    }
    if (slot < 0 && head < 0 && ld_relaxed(&S.cnt[S.head_lo_at]) < nlo) {
      const int l = atomicAdd(&S.cnt[S.head_lo_at], 1);
      if (l < nlo) lo = l;
    }
    if (slot < 0 && head < 0 && lo < 0) {
      // nothing to do right now: park on the next band-0 slot -- unless enough warps already do; the rest
      // leave and free their SM resources for whatever kernel comes next (another engine's batch)
      if (!*waiter && atomicAdd(&S.cnt[kWaiters], 1) < S.max_waiters) *waiter = true;
      if (*waiter) slot = atomicAdd(&S.cnt[kHeadHi], 1);
    }
  }
  *done = 0;
  fin = __shfl_sync(0xffffffffu, fin, 0);
  if (fin >= 0) {
    // every warp holds at most one ticket: slots [fin, fin + #warps] cover all of them, now and later
    const int nw = (gridDim.x * blockDim.x) >> 5;
#pragma unroll 1
    for (int i = lane; i <= nw; i += 32) st_release((int*)&S.ring[fin + i], (int)kExit);
  }
  head = __shfl_sync(0xffffffffu, head, 0);
  if (head >= 0) return S.heads[head];
  slot = __shfl_sync(0xffffffffu, slot, 0);
  lo = __shfl_sync(0xffffffffu, lo, 0);
  if (slot >= 0) {
    nheads0 = __shfl_sync(0xffffffffu, nheads0, 0);
    if (slot < nheads0) return S.heads0[slot];
    // every lane acquires: what the producer wrote before its release is visible to all of them
    uint32_t v;
    while ((v = (uint32_t)ld_acquire((const int*)&S.ring[slot - nheads0])) == kNoItem) __nanosleep(500);
    return v == kExit ? kNoItem : v;
  }
  if (lo >= 0) {
    const int n2 = S.cnt[S.n_items_at + 2], n1 = S.cnt[S.n_items_at + 1];
    return lo < n2 ? S.items[2][lo] : lo < n2 + n1 ? S.items[1][lo - n2] : S.items[0][lo - n2 - n1];
  }
  return kNoItem;
}

// The band's H/V intra prediction (od_hv_intra_pred, src/intra.c:37-62) from the quantised neighbours into
// prm.ref.  Element j of the band is owned by lane j % 32: the lane that writes ref[j] is the one that
// reads it.  The neighbours' `out` is read past L1 (ld.global.cg): bands 0, 1, 2 of a block share a 128-byte
// line, so this SM may hold a copy of the line from before the band that is read now was written, and the
// plain fences that order the producers' stores do not invalidate L1.
__device__ __forceinline__ void intra_band_ref(const Stage& S, int blk, int band, int coef_off, int lane) {
  const daala_b200_pvq_params& prm = S.prm;
  const int start = band_start(band);
  const int bn = band_start(band + 1) - start;
  const int r = band % 3;
  int top = -1, left = -1;
  if (band == 0 || r == 1) top = S.dep_top[blk];
  if (band == 0 || r == 2) left = S.dep_left[blk];
  if (band == 3 || band == 6) top = left = -1;
  const int32_t* ot = top >= 0 ? prm.out + prm.blocks[top].coef_off : nullptr;
  const int32_t* ol = left >= 0 ? prm.out + prm.blocks[left].coef_off : nullptr;
  bool low_from_top = false;
  if (band == 0) {
    // coding-order indices of (0,1) (0,2) (0,3) and (1,0) (2,0) (3,0) in the 4x4 stage; double
    // sums of exact integers as in od_hv_intra_pred (src/intra.c:51-52)
    double g1 = 0, g2 = 0;
    if (ot) { double a = __ldcg(ot + 2), bb = __ldcg(ot + 5), c = __ldcg(ot + 9); g1 += a * a; g1 += bb * bb; g1 += c * c; }
    if (ol) { double a = __ldcg(ol + 1), bb = __ldcg(ol + 4), c = __ldcg(ol + 7); g2 += a * a; g2 += bb * bb; g2 += c * c; }
    low_from_top = g1 > g2;
  }
  int32_t* vref = prm.ref + coef_off;
  for (int i = start + lane; i < start + bn; i += 32) {
    int r2, c2;
    scan_rc(i, &r2, &c2);
    int32_t p = 0;
    if (r2 == 0 && c2 > 0 && ot && (c2 >= 4 || low_from_top)) p = __ldcg(ot + i);
    if (c2 == 0 && r2 > 0 && ol && (r2 >= 4 || !low_from_top)) p = __ldcg(ol + i);
    vref[i] = p;
  }
}

// One luma (block, band) item by one warp: the band's prediction is built from the quantised neighbours first
// (od_hv_intra_pred, src/intra.c:37-62).  The band quantiser is the block's frame's entry of S.fq_bq.
__device__ __forceinline__ void run_item(const Stage& S, uint32_t item, int lane, int16_t* snap) {
  const daala_b200_pvq_params& prm = S.prm;
  const int blk = (int)(item >> 4), band = (int)(item & 15);
  const daala_b200_pvq_block b = prm.blocks[blk];
  const int bs = b.bs, pli = b.pli;
  const int start = band_start(band);
  const int bn = band_start(band + 1) - start;
  const size_t off = (size_t)b.coef_off + start;
  intra_band_ref(S, blk, band, b.coef_off, lane);
  const int qidx = bs * (bs + 1) + (band + 1) - (band + 1) / 3;
  const int q = S.fq_bq[(b.frame * 3 + pli) * 32 + qidx];
  const int beta = (prm.use_masking && pli == 0 && bs > 0) ? kBeta15 : kBeta1;
  const int qoff = (b.xdec & 1 ? prm.qm_stride : 0) + ((((1 << (2 * bs)) - 1) << 4) / 3) + start;
  int itheta, max_theta, k;
  double skip_term;
  const int gain = quantise_band_warp<0>(lane, snap, S.rsqrt_tbl, prm.out + off, prm.in + off, prm.ref + off, bn, q,
                                         prm.y + off, &itheta, &max_theta, &k, beta, &skip_term, prm.is_keyframe, pli,
                                         prm.qm + qoff, prm.qm_inv + qoff, prm.pvq_norm_lambda);
  if (lane == 0) {
    const size_t r = (size_t)blk * 9 + band;
    prm.res_skip_term[r] = skip_term;
    short4 pk;
    pk.x = (short)gain; pk.y = (short)itheta; pk.z = (short)max_theta; pk.w = (short)k;
    reinterpret_cast<short4*>(S.res_pack)[r] = pk;
  }
}

// ---- split path ------------------------------------------------------------------------------------------
// The three phases of a band (pvq_warp.cuh: band_setup / band_search / band_finish) as three kernels over a
// chunk of a dependency-free item list, the context of every band parked in an HBM record in between.
// Why: the fused per-band code is ~50 KB of straight-line SASS plus the search loops, far beyond the
// instruction cache; the persistent kernel spends most of its issue slots waiting for instruction fetch
// (no_instruction is the first stall reason).  One phase at a
// time on the whole GPU keeps the resident code small.  Only items without dependencies can go this way
// (keyframe chroma, every band of an inter frame); keyframe luma stays in the persistent kernel.
struct ItemGeom {
  int blk, band, bn, q, beta, pli, qoff;
  size_t off;
};
__device__ __forceinline__ ItemGeom item_geom(const Stage& S, uint32_t item) {
  const daala_b200_pvq_params& prm = S.prm;
  ItemGeom g;
  g.blk = (int)(item >> 4);
  g.band = (int)(item & 15);
  const daala_b200_pvq_block b = prm.blocks[g.blk];
  const int bs = b.bs;
  g.pli = b.pli;
  const int start = band_start(g.band);
  g.bn = band_start(g.band + 1) - start;
  g.off = (size_t)b.coef_off + start;
  const int qidx = bs * (bs + 1) + (g.band + 1) - (g.band + 1) / 3;
  g.q = S.fq_bq[(b.frame * 3 + g.pli) * 32 + qidx];
  g.beta = (prm.use_masking && g.pli == 0 && bs > 0) ? kBeta15 : kBeta1;
  g.qoff = (b.xdec & 1 ? prm.qm_stride : 0) + ((((1 << (2 * bs)) - 1) << 4) / 3) + start;
  return g;
}

// kPhase 0 / 1 / 2 = setup / search / finish of the items [chunk * slots, ...) of class `cls`.
template <int kPhase, int kMode>
__global__ void __launch_bounds__(128) k_pvq_split(const __grid_constant__ Stage S, int cls, int chunk) {
  const daala_b200_pvq_params& prm = S.prm;
  const int lane = threadIdx.x & 31;
  const int slots = S.sp_slots[cls];
  const int first = chunk * slots;
  const int count = min(S.cnt[S.n_items_at + cls] - first, slots);
  const int vs = cls == 2 ? 128 : 32;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < count; i += nwarps) {
    const ItemGeom g = item_geom(S, S.items[cls][first + i]);
    int16_t* vec = S.sp_vec[cls] + (size_t)i * 3 * vs;
    int32_t* lanes = S.sp_lanes[cls] + (size_t)i * kCtxLaneWords * 16;
    int32_t* uni = S.sp_uni[cls] + (size_t)i * kCtxUniWords;
    int16_t* snap = S.sp_snap[cls] + (size_t)i * kMaxEvents * vs;
    const int32_t* r0 = prm.ref + g.off;
    BandCtx B;
    if (kPhase == 0) {
      band_setup<kMode>(lane, B, prm.in + g.off, r0, g.bn, g.q, g.beta, prm.is_keyframe, g.pli, prm.qm + g.qoff,
                 prm.pvq_norm_lambda, S.rsqrt_tbl);
      band_ctx_store_setup(lane, B, g.bn, vec, vs, lanes, uni);
    } else if (kPhase == 1) {
      band_ctx_load_search(lane, B, g.bn, vec, vs, lanes);
      band_search<kMode>(lane, B, g.bn, snap, vs, S.rsqrt_tbl);
      band_ctx_store_search(lane, B, lanes);
    } else {
      band_ctx_load_finish(lane, B, g.bn, vec, vs, lanes, uni);
      int itheta, max_theta, k;
      double skip_term;
      const int gain = band_finish<kMode>(lane, B, snap, vs, prm.out + g.off, r0, g.bn, g.q, prm.y + g.off, &itheta, &max_theta, &k,
                                   g.beta, &skip_term, prm.is_keyframe, g.pli, prm.qm_inv + g.qoff, prm.pvq_norm_lambda);
      if (lane == 0) {
        const size_t r = (size_t)g.blk * 9 + g.band;
        prm.res_skip_term[r] = skip_term;
        short4 pk;
        pk.x = (short)gain; pk.y = (short)itheta; pk.z = (short)max_theta; pk.w = (short)k;
        reinterpret_cast<short4*>(S.res_pack)[r] = pk;
      }
    }
  }
}

// Persistent PVQ kernel of the keyframe luma stage: one warp = one band at a time.  The chain items of the H/V
// intra predictor form a dependency graph (per size class: band 0 a 2-D wavefront, bands 1/4/7 columns,
// bands 2/5/8 rows).  A warp that finishes a chain item CONTINUES with a successor it made ready -- a
// column or row is walked by one warp without touching the queue -- and pushes a second ready
// successor (band 0 forks) into the chain queue.
__global__ void __launch_bounds__(kPersistThreads, kPersistCtas) k_pvq_persist(const __grid_constant__ Stage S) {
  // per warp: the pulses of every search event of a band and the band's parked context (quantise_band_warp)
  __shared__ __align__(16) int16_t snap_all[kPersistThreads / 32][kSnapEntries];
  const int lane = threadIdx.x & 31;
  int16_t* snap = snap_all[threadIdx.x >> 5];
  int done = 0;
  bool waiter = false;
  for (;;) {
    uint32_t item = next_item(S, lane, &done, &waiter);
    if (item == kNoItem) return;
#ifdef DAALA_B200_CHAIN_TRACE
    int kind = (item & 15) == 0 ? 0 : (item & 15) == 3 || (item & 15) == 6 ? 2 : 1;
#endif
    for (;;) {
      const int band = (int)(item & 15);
#ifdef DAALA_B200_CHAIN_TRACE
      const unsigned long long t0 = globaltimer();
#endif
      run_item(S, item, lane, snap);
#ifdef DAALA_B200_CHAIN_TRACE
      trace_item(S, item, kind, t0, lane);
      kind = 3;
#endif
      if (band == 3 || band == 6) break;
      done += band == 0;
      // results of this item -> visible to whoever runs a successor (this warp included: other lanes)
      __threadfence();
      __syncwarp();
      uint32_t next = kNoItem;
      if (lane == 0) {
        const int blk = (int)(item >> 4);
        if (band == 0) {
          const int nb[2] = {S.succ_bottom[blk], S.succ_right[blk]};
          for (int i = 0; i < 2; i++) {
            if (nb[i] < 0) continue;
            const int need = (S.dep_top[nb[i]] >= 0) + (S.dep_left[nb[i]] >= 0);
            if (need == 2 && atomicAdd(&S.join0[nb[i]], 1) != 1) continue;   // the other neighbour is not done yet
            if (next == kNoItem) {
              next = (uint32_t)nb[i] << 4;
            } else {
              __threadfence();   // (join) the other neighbour's results are ordered before the push
              push_chain(S, nb[i], 0);
            }
          }
        } else {
          const int nb = band % 3 == 1 ? S.succ_bottom[blk] : S.succ_right[blk];
          if (nb >= 0) next = ((uint32_t)nb << 4) | band;
        }
      }
      next = __shfl_sync(0xffffffffu, next, 0);
      if (next == kNoItem) break;
      // (join) what the other neighbour's warp released before its atomic is visible to every lane
      __threadfence();
      item = next;
    }
  }
}

__global__ void k_fill_rsqrt(double* tbl) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kTableDoubles) pvq_fill_rsqrt_table(tbl, i);
}

// Start of the PVQ stages in `stages` (kBeginLuma | kBeginChroma): the tickets; the chain queue starts with the
// heads.  Neither stage touches the other's tickets, so the whole step starts both at once.
enum { kBeginLuma = 1, kBeginChroma = 2 };
__global__ void k_begin_pvq(int32_t* cnt, int stages) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (stages & kBeginLuma) {
      cnt[kHeadLoL] = 0;
      cnt[kHeadHi] = 0;
      cnt[kTailHi] = cnt[kNHeads0];
      cnt[kDoneHi] = 0;
      cnt[kHeadCh] = 0;
      cnt[kWaiters] = 0;
#ifdef DAALA_B200_CHAIN_TRACE
      cnt[kTraceN] = 0;
#endif
    }
    if (stages & kBeginChroma) cnt[kHeadLoC] = 0;
  }
}

// Per block, after all its bands: ordered skip_diff sum (src/pvq_encoder.c:875-880), keyframe DC
// (scalar_out[0] = dblock[0], src/encode.c:1381), od_init_skipped_coeffs (src/state.c:1347) +
// od_coding_order_to_raster (src/partition.c:157) back into the coefficient plane, pulses packed to
// 16 bits for the host entropy coder.  One warp per block.
// kInter: DC is the scalar quantisation of in[0] - ref[0] with the band-0 quantiser (od_block_encode's
// non-keyframe branch; the index goes to prm.res_dc), and the uncoded tail of 32x32 / 64x64 blocks is the
// transformed prediction (od_init_skipped_coeffs for inter frames).
// kHdc (keyframes with config.haar_dc_quant): the DC is the quantised one the DC chain left in its grid, into out[0]
// and the coefficient plane.
template <bool kInter, bool kHdc = false>
__global__ void __launch_bounds__(256) k_finish_scatter(const __grid_constant__ Stage S) {
  const daala_b200_pvq_params& prm = S.prm;
  const int n = min(S.cnt[S.n_blocks_at], S.max_blocks);
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int blk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; blk < n; blk += nwarps) {
    const daala_b200_pvq_block b = prm.blocks[blk];
    const int ln = b.bs + 2, nn = 1 << ln;
    const int len = ln >= 5 ? 512 : 1 << (2 * ln);
    const int stride = prm.plane_stride[b.pli];
    int32_t* dst = prm.coef_plane[b.pli] + b.frame * prm.plane_frame_pitch[b.pli] + (size_t)b.y0 * stride + b.x0;
    const int32_t* src = prm.out + b.coef_off;
    if (lane == 0) {
      const int nb = num_bands(b.bs);
      double sd = 0;
      for (int i = 0; i < nb; i++) sd += prm.res_skip_term[(size_t)blk * 9 + i];
      prm.res_skip_diff[blk] = sd;
      if (kHdc) {
        prm.out[b.coef_off] = dst[0] = hdc_grid(S, b.frame, b.pli)[(long long)(b.y0 >> 2) * (stride >> 2) + (b.x0 >> 2)];
      } else if (!kInter) {
        prm.out[b.coef_off] = prm.in[b.coef_off];
      } else {
        const int dc_quant = S.fq_bq[(b.frame * 3 + b.pli) * 32 + b.bs * (b.bs + 1)];
        const int32_t r = prm.ref[b.coef_off], diff = prm.in[b.coef_off] - r;
        int qdc = 0;
        if (abs(diff) >= dc_quant * 141 / 256) {
          const int half = ((dc_quant + 1) >> 1) - 1;
          qdc = (diff + (diff < 0 ? -half : half)) / dc_quant;
        }
        prm.out[b.coef_off] = dst[0] = qdc * dc_quant + r;
        prm.res_dc[blk] = qdc;
        if (S.dc_resid) S.dc_resid[blk] = diff;
      }
    }
    if (ln >= 5) {
      const int32_t* mdp = kInter ? prm.pred_plane[b.pli] + b.frame * prm.plane_frame_pitch[b.pli] + (size_t)b.y0 * stride + b.x0
                                  : nullptr;
      for (int i = lane; i < nn * nn; i += 32) {
        const size_t at = (size_t)(i >> ln) * stride + (i & (nn - 1));
        if (i) dst[at] = kInter ? mdp[at] : 0;
      }
      __syncwarp();
    }
    for (int i = lane + 1; i < len; i += 32) dst[scan_to_raster(i, ln, stride)] = src[i];
    const int32_t* y = prm.y + b.coef_off;
    for (int i = lane; i < len; i += 32) prm.y16[b.coef_off + i] = i ? (int16_t)y[i] : (int16_t)0;
  }
}

// ---- deringing stage (optional) ---------------------------------------------------------------------------
// od_encode_coefficients' final deringing application (src/encode.c:2812-2842) with the per-superblock levels
// given by the caller (the level SEARCH is serial: CDF adaptation + neighbour context; like the block sizes its
// result is an input of the hot path): etmp = ctmp after the SB-edge postfilter, od_dering of every superblock
// with threshold = OD_DERING_GAIN_TABLE[level] * quantizer^0.84182 (* 0.6 on chroma), od_coeff_to_ref_plane
// (the deringing kernel stores the u8 reconstruction itself).
// thr[pl][f][sb] = table[pl][level[f][sb]].  P-frame finishing pass: `coded` (else NULL) flags the superblocks with a
// coded 4x4 luma unit; the others are forced to level 0 (src/encode.c:2724-2738), and the level applied goes to
// `applied`.  `frame_tbl` ([F][2][6]) holds each frame's table, the frame of superblock i being i / nsb.
__global__ void k_dering_thresholds(const uint8_t* __restrict__ level, int32_t* __restrict__ thr_luma,
                                    int32_t* __restrict__ thr_chroma, int n, const uint8_t* __restrict__ coded,
                                    uint8_t* __restrict__ applied, const int32_t* __restrict__ frame_tbl, int nsb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int g = level[i] < 6 ? level[i] : 5;
  if (coded) {
    if (!coded[i]) g = 0;
    applied[i] = (uint8_t)g;
  }
  const int32_t* t = frame_tbl + (size_t)(i / nsb) * 12;
  thr_luma[i] = t[g];
  thr_chroma[i] = t[6 + g];
}

// ---- P-frame finishing pass (config.inter_finish) ----------------------------------------------------------------
// The host coder's per-block decisions applied to the coefficients of the last step, in a plane of their own (the
// step's d / md stay as they are), and the skip map they imply.  Both kernels walk the luma list, then the chroma list.
struct Fin {
  const daala_b200_pvq_block* blocks[2];   // luma, chroma
  const uint8_t* skip[2];                  // per block: 0 or 1
  const int32_t* dc[2];                    // per block: the final DC index
  const int32_t* cnt;
  int max_blocks[2];
  const int32_t* d[3];                     // the step's `d` and `md` planes
  const int32_t* md[3];
  int32_t* out[3];                         // patched planes
  long long plane_pitch[3];
  int plane_stride[3];
  uint8_t* bskip[3];                       // [F][plane_h / 4][skip_stride]
  long long skip_pitch[3];
  int skip_stride;                         // state->skip_stride = nhsb * 16
  uint8_t* coded;                          // [F][nvsb][nhsb]: a luma 4x4 unit of the superblock is coded (preset 0)
  int nhsb, nvsb;
  const int32_t* fq_bq;                    // [F][3][32] each frame's band quantisers (Stage::fq_bq)
};

// block i of the two lists together (luma first), or false past their end
__device__ __forceinline__ bool fin_block(const Fin& P, int i, int* list, int* blk) {
  const int nl = min(P.cnt[kNLuma], P.max_blocks[0]), nc = min(P.cnt[kNChroma], P.max_blocks[1]);
  if (i >= nl + nc) return false;
  *list = i >= nl;
  *blk = i >= nl ? i - nl : i;
  return true;
}

// One warp per block.  skip = 0: the step's coefficients; skip = 1: md over the whole block (AC = prediction,
// src/pvq_encoder.c:975; the late skip's d = md, src/encode.c:1444-1448); either way DC = md[0] + dc * dc_quant
// (src/encode.c:1373-1374 with the band-0 quantiser of :1333-1334).
__global__ void __launch_bounds__(256) k_fin_patch(const __grid_constant__ Fin P) {
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  int list, blk;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; fin_block(P, i, &list, &blk); i += nwarps) {
    const daala_b200_pvq_block b = P.blocks[list][blk];
    const int ln = b.bs + 2, nn = 1 << ln;
    const int stride = P.plane_stride[b.pli];
    const size_t o = b.frame * P.plane_pitch[b.pli] + (size_t)b.y0 * stride + b.x0;
    const int32_t* src = (P.skip[list][blk] ? P.md[b.pli] : P.d[b.pli]) + o;
    const int32_t* mdp = P.md[b.pli] + o;
    int32_t* dst = P.out[b.pli] + o;
    const int dc_quant = P.fq_bq[(b.frame * 3 + b.pli) * 32 + b.bs * (b.bs + 1)];
    const int32_t dc0 = mdp[0] + P.dc[list][blk] * dc_quant;
    for (int k = lane; k < nn * nn; k += 32) {
      const size_t at = (size_t)(k >> ln) * stride + (k & (nn - 1));
      dst[at] = k ? src[at] : dc0;
    }
  }
}

// One warp per block: bskip = skip && dc == 0 over the block's 4x4 units (src/encode.c:1690-1691, :1821-1825), and
// the coded flag of the superblock of a luma block that is not skipped.
__global__ void __launch_bounds__(256) k_fin_skip_map(const __grid_constant__ Fin P) {
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  int list, blk;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; fin_block(P, i, &list, &blk); i += nwarps) {
    const daala_b200_pvq_block b = P.blocks[list][blk];
    const uint8_t s = P.skip[list][blk] && P.dc[list][blk] == 0;
    const int nu = 1 << b.bs;   // 4x4 units per side
    uint8_t* m = P.bskip[b.pli] + b.frame * P.skip_pitch[b.pli] + (size_t)(b.y0 >> 2) * P.skip_stride + (b.x0 >> 2);
    for (int k = lane; k < nu * nu; k += 32) m[(size_t)(k >> b.bs) * P.skip_stride + (k & (nu - 1))] = s;
    if (lane == 0 && b.pli == 0 && !s) P.coded[((size_t)b.frame * P.nvsb + (b.y0 >> 6)) * P.nhsb + (b.x0 >> 6)] = 1;
  }
}

// cfg.inter_mc with cfg.inter_finish: the pass's reconstruction of frame f into slot slot[f] of the reference-picture
// pool (-1: not stored), the last node of the finishing graph.  The table lives on the device so that the one
// captured graph serves every call.  A frame's planes have the pool's layout, and the pool's clamped reads are the
// reference's edge extension (DESIGN §3.5), so the picture is stored as it is.
struct PoolStore {
  const uint8_t* src[3];           // fin_pixels: [F][plane_h][plane_w]
  uint8_t* pool[3];                // ref_pixels: [mc_refs][plane_h][plane_w]
  long long plane_bytes[3];        // plane_h * plane_w, a multiple of 16 * 32 (plane widths are multiples of 32)
  const int32_t* slot;             // [F]
};

// One launch for every frame and plane: blockIdx.y = frame * 3 + plane, the CTAs of a plane stride over its rows as
// 16-byte words (a plane is a whole number of words, and every row starts on one).
__global__ void __launch_bounds__(256) k_fin_pool_store(const __grid_constant__ PoolStore S) {
  const int f = blockIdx.y / 3, p = blockIdx.y - 3 * f;
  const int slot = S.slot[f];
  if (slot < 0) return;
  const long long n = S.plane_bytes[p] >> 4;
  const uint4* __restrict__ src = reinterpret_cast<const uint4*>(S.src[p] + f * S.plane_bytes[p]);
  uint4* __restrict__ dst = reinterpret_cast<uint4*>(S.pool[p] + slot * S.plane_bytes[p]);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = src[i];
}

// ---- symbol stream (optional, config.symbol_stream) -------------------------------------------------------
// The PVQ symbols of every frame in bitstream order (include/daala_b200.h, daala_b200_kf_sym_block): per
// superblock in raster order planes 0, 1, 2, inside a plane the quadtree leaves depth-first with children
// top-left, top-right, bottom-left, bottom-right (od_encode_recursive, src/encode.c:1780-1787, called per
// superblock and plane at src/encode.c:2605-2656).  That depth-first order is the Z order of the leaves'
// origins, so a block's position is its superblock's base plus the number of leaves of its plane whose origin
// comes first in Z order: a warp scan over the 64 units of a superblock in Z order.  Then per block the band
// count and pulse bytes (they depend on K), a prefix scan over the blocks in stream order, and the pack.
struct Sym {
  const uint8_t* bsize;
  int bstride;
  long long bsize_pitch;
  int F, nhsb, sb_rows, u_row0;
  int nsb;                         // superblocks per frame in this shard (nhsb * sb_rows)
  uint32_t* unit_rank;             // [F][sb_rows*8][nhsb*8]: luma | chroma << 16 leaves earlier in the superblock
  uint32_t* sb_cnt;                // [F*nsb]: luma | chroma-per-plane << 16 leaves of the superblock
  int32_t* sb_base;                // [F*nsb]: first slot of the superblock (exclusive prefix over the batch)
  uint32_t* order;                 // [cap_blocks]: slot -> block (bit 31: chroma list)
  longlong2* off;                  // [cap_blocks]: (bands, pulse bytes) of the slot, then exclusive prefixes
  longlong2* tile;                 // [ntiles]: tile sums, then exclusive prefixes
  long long* tot;                  // [4]: slots, bands, pulse bytes of the batch
  int ntiles, cap_blocks;
  long long cap_bands, cap_bytes;
  daala_b200_kf_sym_frame* index;  // [F]
  daala_b200_kf_sym_block* blocks; // [cap_blocks]
  short4* bands;                   // [cap_bands]
  uint8_t* pulses;                 // [cap_bytes]
  const daala_b200_pvq_block* list[2];   // luma / chroma block lists and their PVQ results
  const short4* res[2];
  const int32_t* y[2];
  const double* skip_diff[2];
  const int32_t* flip;
  const int32_t* cnt;
  int max_luma, max_chroma;
  // symbol_stream = 2 (P frames): the DC record of each slot, from the step's DC index and unquantised residual
  daala_b200_kf_sym_dc* dc;        // [cap_blocks]
  const int32_t* qdc[2];
  const int32_t* dc_resid[2];
  // with config.late_skip: the late-skip record of each slot, from the block-order records (else NULL)
  daala_b200_kf_late_skip* late_skip;   // [cap_blocks]
  const daala_b200_kf_late_skip* ls_block[2];
  // symbol_stream = 1 with haar_dc_quant: the keyframe DC record of each slot, from the DC chain's index grids (else NULL)
  daala_b200_kf_sym_hdc* hdc;      // [cap_blocks]
  const int32_t* hdc_index[3];     // [F][gh][gw] per plane
  int gw[3], gh[3];                // index grid width / height (4x4 units of the plane)
};

// Bytes the band's pulses take in the stream: the n - (itheta != -1) values pvq_encode_partition hands to
// od_encode_pvq_codeword (src/pvq_encoder.c:719-720), one byte each for K <= 127, two above.
__device__ __forceinline__ int sym_band_bytes(int band, short4 r) {
  if (r.w <= 0) return 0;
  const int n = band_start(band + 1) - band_start(band) - (r.y != -1);
  return r.w > 127 ? 2 * n : n;
}

// One warp per superblock: lane l holds the units 2l and 2l + 1 in Z order.
__global__ void __launch_bounds__(256) k_sym_rank(const __grid_constant__ Sym S) {
  const int lane = threadIdx.x & 31;
  const int sb = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (sb >= S.F * S.nsb) return;   // whole warps
  const int f = sb / S.nsb, r = sb % S.nsb;
  const int sby = r / S.nhsb, sbx = r % S.nhsb;
  const int uw = S.nhsb * 8;
  uint32_t v[2];
  long long at[2];
  for (int h = 0; h < 2; h++) {
    const int m = 2 * lane + h;    // Z order: x in the even bits, y in the odd bits
    const int dx = (m & 1) | ((m >> 1) & 2) | ((m >> 2) & 4);
    const int dy = ((m >> 1) & 1) | ((m >> 2) & 2) | ((m >> 3) & 4);
    const int ux = sbx * 8 + dx, uy = S.u_row0 + sby * 8 + dy;
    const int b = S.bsize[f * S.bsize_pitch + (long long)uy * S.bstride + ux];
    const int4 c = unit_counts(b, ux, uy);
    v[h] = (uint32_t)c.x | ((uint32_t)c.z << 16);
    at[h] = ((long long)f * S.sb_rows * 8 + (uy - S.u_row0)) * uw + ux;
  }
  const uint32_t s = v[0] + v[1];
  uint32_t inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t a = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += a;
  }
  S.unit_rank[at[0]] = inc - s;
  S.unit_rank[at[1]] = inc - s + v[0];
  if (lane == 31) S.sb_cnt[sb] = inc;
}

// One CTA: exclusive scan of the superblocks' block counts (luma + 2 chroma planes) -> first slots.
__global__ void __launch_bounds__(1024) k_sym_sb_scan(const __grid_constant__ Sym S) {
  __shared__ int part[1024];
  __shared__ int carry;
  const int t = threadIdx.x;
  const int n = S.F * S.nsb;
  if (t == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + t;
    const uint32_t c = i < n ? S.sb_cnt[i] : 0u;
    const int v = (int)(c & 0xffff) + 2 * (int)(c >> 16);
    part[t] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const int a = t >= o ? part[t - o] : 0;
      __syncthreads();
      part[t] += a;
      __syncthreads();
    }
    const int incl = part[t], c0 = carry;
    if (i < n) S.sb_base[i] = c0 + incl - v;
    __syncthreads();
    if (t == 1023) carry = c0 + incl;
    __syncthreads();
  }
  if (t == 0) S.tot[0] = min(carry, S.cap_blocks);
}

// symbol_stream = 1 with haar_dc_quant: the keyframe DC records (daala_b200_kf_sym_hdc), one warp per (frame, superblock,
// plane).  od_encode_recursive (src/encode.c:1660-1787) codes the superblock DC, then at every split node, before its
// children, the node's three indices: a quadtree with L leaves gives 1 + 3 (L - 1) / 3 = L records, which fill the slots
// of the (superblock, plane)'s L block records.  Pre-order is the Z order of the nodes' origins, coarser nodes first at
// a shared origin, so a node's place among the split nodes is a warp scan over the superblock's 64 units in Z order
// (lane l: units 2l and 2l + 1, as k_sym_rank) of the split nodes whose origin each unit is.  A node is split when it and
// every ancestor read a size below their own at their origin (max(obs, xdec) < bsi, the map at the node's 8x8 unit);
// its first leaf is the leaf at its origin unit, whose slot k_sym_rank / k_sym_sb_scan already give.
__global__ void __launch_bounds__(256) k_sym_hdc(const __grid_constant__ Sym S) {
  const int lane = threadIdx.x & 31;
  const int item = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (item >= S.F * S.nsb * 3) return;   // whole warps
  const int sb = item / 3, pli = item - 3 * sb;
  const int f = sb / S.nsb, r = sb % S.nsb;
  const int sby = r / S.nhsb, sbx = r % S.nhsb;
  const int uw = S.nhsb * 8, xdec = pli ? 1 : 0;
  int b[2], ux[2], uy[2];
  for (int h = 0; h < 2; h++) {
    const int m = 2 * lane + h;
    ux[h] = sbx * 8 + ((m & 1) | ((m >> 1) & 2) | ((m >> 2) & 4));
    uy[h] = S.u_row0 + sby * 8 + (((m >> 1) & 1) | ((m >> 2) & 2) | ((m >> 3) & 4));
    b[h] = max((int)S.bsize[f * S.bsize_pitch + (long long)uy[h] * S.bstride + ux[h]], xdec);
  }
  // the sizes at the origins of the unit's 16x16, 32x32 and 64x64 luma ancestors (Z codes multiple of 4, 16, 64: even)
  const int b2 = __shfl_sync(0xffffffffu, b[0], lane & ~1);
  const int b3 = __shfl_sync(0xffffffffu, b[0], lane & ~7);
  const int b4 = __shfl_sync(0xffffffffu, b[0], 0);
  const bool s4 = b4 < 4, s3 = s4 && b3 < 3, s2 = s3 && b2 < 2;
  // the split nodes whose origin is each of the lane's units: bit 4 - bsi of the mask, so the coarsest is the lowest bit
  int mask[2];
  for (int h = 0; h < 2; h++) {
    const int m = 2 * lane + h;
    mask[h] = (m == 0 && s4 ? 1 : 0) | ((m & 15) == 0 && s3 ? 2 : 0) | ((m & 3) == 0 && s2 ? 4 : 0) |
              (s2 && b[h] < 1 ? 8 : 0);
  }
  const int n = __popc(mask[0]) + __popc(mask[1]);
  int inc = n;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += a;
  }
  const uint32_t sc = S.sb_cnt[sb];
  const int plane_off = pli ? (int)(sc & 0xffff) + (pli - 1) * (int)(sc >> 16) : 0;
  const long long base = (long long)S.sb_base[sb] + plane_off;            // the (superblock, plane)'s first slot
  const long long first = S.sb_base[f * S.nsb];                           // the frame's first slot
  const int32_t* grid = S.hdc_index[pli] + (long long)f * S.gw[pli] * S.gh[pli];
  const int gsh = pli ? 0 : 1;   // 4x4 units of the plane per 8x8 luma unit: log2 2 (luma) or 1 (4:2:0 chroma)
  if (lane == 0 && base < S.cap_blocks) {
    daala_b200_kf_sym_hdc d;
    d.value = grid[(long long)(uy[0] << gsh) * S.gw[pli] + (ux[0] << gsh)];
    d.block = (uint32_t)(base - first);
    d.pli = (uint8_t)pli;
    d.bsi = 4;
    d.child = 0;
    d.reserved = 0;
    S.hdc[base] = d;
  }
  int k = inc - n;   // split nodes before the lane's first unit, in pre-order
  for (int h = 0; h < 2; h++) {
    if (!mask[h]) continue;
    const uint32_t rk = S.unit_rank[((long long)f * S.sb_rows * 8 + (uy[h] - S.u_row0)) * uw + ux[h]];
    const uint32_t block = (uint32_t)(base - first) + (pli ? rk >> 16 : rk & 0xffff);
    const int gx = ux[h] << gsh, gy = uy[h] << gsh;
    for (int bsi = 4; bsi >= 1; bsi--) {
      if (!(mask[h] & (1 << (4 - bsi)))) continue;
      const int half = 1 << (bsi - 1 - xdec);   // child offset in 4x4 units of the plane
      for (int c = 1; c <= 3; c++) {
        const long long slot = base + 1 + 3 * k + (c - 1);
        if (slot >= S.cap_blocks) break;
        daala_b200_kf_sym_hdc d;
        d.value = grid[(long long)(gy + (c >> 1) * half) * S.gw[pli] + gx + (c & 1) * half];
        d.block = block;
        d.pli = (uint8_t)pli;
        d.bsi = (uint8_t)(bsi - 1);
        d.child = (uint8_t)c;
        d.reserved = 0;
        S.hdc[slot] = d;
      }
      k++;
    }
  }
}

// Per block (luma list, then chroma list): its slot, and the slot's band count and pulse bytes.
__global__ void __launch_bounds__(256) k_sym_place(const __grid_constant__ Sym S) {
  const int nl = min(S.cnt[kNLuma], S.max_luma), nc = min(S.cnt[kNChroma], S.max_chroma);
  const int uw = S.nhsb * 8;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nl + nc; i += gridDim.x * blockDim.x) {
    const int ch = i >= nl;
    const int blk = ch ? i - nl : i;
    const daala_b200_pvq_block b = S.list[ch][blk];
    const int sh = ch ? 2 : 3;   // plane samples per 8x8 luma unit: 4 (4:2:0 chroma) or 8
    const int ux = b.x0 >> sh, uy = b.y0 >> sh;
    const int sb = b.frame * S.nsb + ((uy - S.u_row0) >> 3) * S.nhsb + (ux >> 3);
    const uint32_t rk = S.unit_rank[((long long)b.frame * S.sb_rows * 8 + (uy - S.u_row0)) * uw + ux];
    const uint32_t sc = S.sb_cnt[sb];
    int pos = S.sb_base[sb];
    if (!ch) pos += (int)(rk & 0xffff) + (b.bs == 0 ? ((b.y0 >> 2) & 1) * 2 + ((b.x0 >> 2) & 1) : 0);
    else pos += (int)(sc & 0xffff) + (b.pli - 1) * (int)(sc >> 16) + (int)(rk >> 16);
    if (pos >= S.cap_blocks) continue;
    S.order[pos] = (uint32_t)blk | (ch ? 0x80000000u : 0u);
    const short4* r = S.res[ch] + (size_t)blk * 9;
    const int nb = num_bands(b.bs);
    long long bytes = 0;
    for (int j = 0; j < nb; j++) bytes += sym_band_bytes(j, r[j]);
    S.off[pos] = make_longlong2(nb, bytes);
  }
}

__device__ __forceinline__ longlong2 add2(longlong2 a, longlong2 b) { return make_longlong2(a.x + b.x, a.y + b.y); }

__global__ void __launch_bounds__(kTile) k_sym_tile_sums(const __grid_constant__ Sym S) {
  __shared__ longlong2 part[32];
  const long long i = (long long)blockIdx.x * kTile + threadIdx.x;
  longlong2 v = i < S.tot[0] ? S.off[i] : make_longlong2(0, 0);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
    v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
  }
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    longlong2 s = make_longlong2(0, 0);
    for (int w = 0; w < kTile / 32; w++) s = add2(s, part[w]);
    S.tile[blockIdx.x] = s;
  }
}

// One CTA: exclusive scan of the tile sums in place; the batch's band and byte totals.
__global__ void __launch_bounds__(1024) k_sym_tile_scan(const __grid_constant__ Sym S) {
  __shared__ longlong2 part[1024];
  __shared__ longlong2 carry;
  const int t = threadIdx.x;
  if (t == 0) carry = make_longlong2(0, 0);
  __syncthreads();
  for (int base = 0; base < S.ntiles; base += 1024) {
    const int i = base + t;
    const longlong2 v = i < S.ntiles ? S.tile[i] : make_longlong2(0, 0);
    part[t] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const longlong2 a = t >= o ? part[t - o] : make_longlong2(0, 0);
      __syncthreads();
      part[t] = add2(part[t], a);
      __syncthreads();
    }
    const longlong2 incl = part[t], c = carry;
    if (i < S.ntiles) S.tile[i] = make_longlong2(c.x + incl.x - v.x, c.y + incl.y - v.y);
    __syncthreads();
    if (t == 1023) carry = add2(c, incl);
    __syncthreads();
  }
  if (t == 0) {
    S.tot[1] = carry.x;
    S.tot[2] = carry.y;
  }
}

// Per slot: (bands, bytes) -> exclusive prefixes over the batch, in place.
__global__ void __launch_bounds__(kTile) k_sym_offsets(const __grid_constant__ Sym S) {
  __shared__ longlong2 wsum[32];
  const long long i = (long long)blockIdx.x * kTile + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool valid = i < S.tot[0];
  const longlong2 v = valid ? S.off[i] : make_longlong2(0, 0);
  longlong2 s = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long ax = __shfl_up_sync(0xffffffffu, s.x, o), ay = __shfl_up_sync(0xffffffffu, s.y, o);
    if (lane >= o) s = make_longlong2(s.x + ax, s.y + ay);
  }
  if (lane == 31) wsum[warp] = s;
  __syncthreads();
  longlong2 pre = S.tile[blockIdx.x];
  for (int w = 0; w < warp; w++) pre = add2(pre, wsum[w]);
  if (valid) S.off[i] = make_longlong2(pre.x + s.x - v.x, pre.y + s.y - v.y);
}

// One warp per slot: the block record, its band records and the pulses of its bands with K > 0.  kInter (symbol_stream
// = 2): flip is 0 (P frames have no CfL; res_flip is never written) and the slot's DC record is written too, and with
// config.late_skip its late-skip record.
template <bool kInter>
__global__ void __launch_bounds__(256) k_sym_pack(const __grid_constant__ Sym S) {
  const int lane = threadIdx.x & 31;
  const long long n = S.tot[0];
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (long long slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; slot < n; slot += nwarps) {
    const uint32_t id = S.order[slot];
    const int ch = id >> 31, blk = (int)(id & 0x7fffffffu);
    const daala_b200_pvq_block b = S.list[ch][blk];
    const long long first = S.sb_base[b.frame * S.nsb];   // the frame's first slot
    const longlong2 o = S.off[slot], o0 = first < n ? S.off[first] : o;
    const short4* r = S.res[ch] + (size_t)blk * 9;
    const int nb = num_bands(b.bs);
    int bytes = 0;
    for (int j = 0; j < nb; j++) bytes += sym_band_bytes(j, r[j]);
    // only an over-capacity step (flagged in counts[kError]; submit refuses such a batch) can leave stale slots
    if (o.x + nb > S.cap_bands || o.y + bytes > S.cap_bytes) continue;
    if (lane == 0) {
      daala_b200_kf_sym_block rec;
      rec.skip_diff = S.skip_diff[ch][blk];
      rec.pulse_off = (uint32_t)(o.y - o0.y);
      rec.band_off = (uint32_t)(o.x - o0.x);
      rec.x0 = b.x0;
      rec.y0 = b.y0;
      rec.bs = b.bs;
      rec.pli = b.pli;
      rec.flip = !kInter && ch ? (uint8_t)S.flip[blk] : 0;
      rec.reserved = 0;
      S.blocks[slot] = rec;
      if (kInter) {
        daala_b200_kf_sym_dc d;
        d.qdc = S.qdc[ch][blk];
        d.dc_resid = S.dc_resid[ch][blk];
        S.dc[slot] = d;
        if (S.late_skip) S.late_skip[slot] = S.ls_block[ch][blk];
      }
    }
    if (lane < nb) S.bands[o.x + lane] = r[lane];
    const int32_t* y = S.y[ch] + b.coef_off;
    uint8_t* dst = S.pulses + o.y;
    for (int j = 0; j < nb; j++) {
      const short4 q = r[j];
      const int len = sym_band_bytes(j, q);
      if (!len) continue;
      const int st = band_start(j);
      if (q.w > 127) {
        for (int t = lane; t < len / 2; t += 32) {
          const int v = y[st + t];
          dst[2 * t] = (uint8_t)(v & 0xff);
          dst[2 * t + 1] = (uint8_t)((v >> 8) & 0xff);
        }
      } else {
        for (int t = lane; t < len; t += 32) dst[t] = (uint8_t)(y[st + t] & 0xff);
      }
      dst += len;
    }
  }
}

// Per frame: where its blocks, bands and pulse bytes are in the batch-wide arrays.
__global__ void k_sym_index(const __grid_constant__ Sym S) {
  for (int f = threadIdx.x; f < S.F; f += blockDim.x) {
    const long long n = S.tot[0];
    const long long s0 = S.sb_base[f * S.nsb];
    const long long s1 = f + 1 < S.F ? S.sb_base[(f + 1) * S.nsb] : n;
    const longlong2 a = s0 < n ? S.off[s0] : make_longlong2(S.tot[1], S.tot[2]);
    const longlong2 e = s1 < n ? S.off[s1] : make_longlong2(S.tot[1], S.tot[2]);
    daala_b200_kf_sym_frame x;
    x.first_block = s0;
    x.n_blocks = s1 - s0;
    x.first_band = a.x;
    x.n_bands = e.x - a.x;
    x.first_byte = a.y;
    x.n_bytes = e.y - a.y;
    S.index[f] = x;
  }
}

// Copy of the used part of each stream array into the caller's pinned host buffers (device-addressable):
// the lengths are only known on the device.  Segment 0 index, 1 block records, 2 band records, 3 pulses, 4 DC records,
// 5 late-skip records and 6 keyframe DC records (one per block record each).
constexpr int kSymSegs = 7;
struct SymCopy {
  const uint8_t* src[kSymSegs];
  uint8_t* dst[kSymSegs];
  long long unit[kSymSegs];        // bytes per element; segment 0 has a fixed length
  long long cap[kSymSegs];         // bytes: the smaller of the host buffer and the device array
  long long index_bytes;
  const long long* tot;
};

__global__ void __launch_bounds__(256) k_sym_copy(const __grid_constant__ SymCopy C) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nth = (long long)gridDim.x * blockDim.x;
  for (int seg = 0; seg < kSymSegs; seg++) {
    if (!C.dst[seg]) continue;
    const long long want = seg == 0 ? C.index_bytes : C.tot[seg >= 4 ? 0 : seg - 1] * C.unit[seg];
    const long long len = want < C.cap[seg] ? want : C.cap[seg];
    const uint8_t* s = C.src[seg];
    uint8_t* d = C.dst[seg];
    long long done = 0;
    if ((((uintptr_t)s | (uintptr_t)d) & 15) == 0) {
      const long long n16 = len >> 4;
      for (long long i = tid; i < n16; i += nth)
        reinterpret_cast<uint4*>(d)[i] = reinterpret_cast<const uint4*>(s)[i];
      done = n16 << 4;
    }
    for (long long i = done + tid; i < len; i += nth) d[i] = s[i];
  }
}

// symbol_stream = 2 with inter_finish: the finishing pass's decisions given in stream order (finish_io.stream_skip /
// stream_dc, staged in skip / dc) scattered into the block order the pass reads, through the step's slot -> block map.
// The first node of the finishing graph; `form` (set by each finish call) is 0 for the classic form, which the call
// copied into fin_skip / fin_dc itself.
struct Unstream {
  const uint32_t* order;           // Sym.order
  const long long* tot;            // Sym.tot: tot[0] slots
  const uint8_t* skip;             // [cap_blocks] in stream order
  const int32_t* dc;
  uint8_t* fin_skip[2];            // luma / chroma, block order
  int32_t* fin_dc[2];
  const int32_t* form;             // 1: stream form
};

__global__ void __launch_bounds__(256) k_fin_unstream(const __grid_constant__ Unstream U) {
  if (!*U.form) return;
  const long long n = U.tot[0];
  for (long long slot = (long long)blockIdx.x * blockDim.x + threadIdx.x; slot < n;
       slot += (long long)gridDim.x * blockDim.x) {
    const uint32_t id = U.order[slot];
    const int ch = id >> 31, blk = (int)(id & 0x7fffffffu);
    U.fin_skip[ch][blk] = U.skip[slot];
    U.fin_dc[ch][blk] = U.dc[slot];
  }
}

}  // namespace kf
}  // namespace daala_b200

// =====================================================================================================
// Host side of the engine
// =====================================================================================================
using namespace daala_b200::kf;

extern "C" int daala_b200_launch_forward(const daala_b200_frame* prm, int nplanes, cudaStream_t stream);
extern "C" int daala_b200_launch_inverse(const daala_b200_frame* prm, int nplanes, cudaStream_t stream);
extern "C" int daala_b200_launch_inverse_lapped_only(const daala_b200_frame* prm, int plane0, int nplanes,
                                                     cudaStream_t stream);
extern "C" int daala_b200_launch_sb_postfilter_store(const daala_b200_frame* prm, int plane0, int nplanes,
                                                     cudaStream_t stream);

// One deringing pass over the batch (od_encode_coefficients' final application, src/encode.c:2812-2842): the step's on
// keyframes (config.dering) or the finishing pass's on P frames (config.inter_finish).  The two differ only in the data
// below, so enqueue_dering runs either.
struct Dering {
  daala_b200_frame frame;          // the planes it inverts; post16 = etmp, pixels_out = the u8 reconstruction
  const uint8_t* skip[3];          // per plane: [F][plane_h / 4][skip_stride], skip_pitch[p] apart (0: one map)
  long long skip_pitch[3];
  int skip_stride;
  uint8_t* level;                  // [F][nvsb][nhsb]: what the thresholds read and the search writes
  const uint8_t* coded;            // nullable: superblocks with a coded luma 4x4 unit; the others get level 0 ...
  uint8_t* applied;                // ... and the level applied lands here
  const int32_t* frame_tbl;        // [F][2][6] luma / chroma threshold per level of each frame
  int32_t* thr[2];                 // luma / chroma threshold per superblock
  int32_t* dir;                    // [F][nvsb*8][nhsb*8]
  bool search;                     // the level search runs first, described by `sb`
  daala_b200_dering_search_batch sb;
};

// The events of kf_enqueue_step_forked, one per fork or join.
enum { kEvLists, kEvForward, kEvLumaBands, kEvLumaScatter, kEvChroma, kEvHaarDc, kNumEvents };

struct daala_b200_kf {
  daala_b200_kf_config cfg;
  int nhsb, nvsb, F;
  int plane_w[3], plane_h[3];
  cudaStream_t stream;
  bool own_stream;
  cudaStream_t side;               // keyframe engines: the second branch of the forked step (engine-owned, highest priority)
  cudaEvent_t ev[kNumEvents];
  cudaGraph_t graph;
  cudaGraphExec_t exec;
  bool captured;
  // device buffers
  uint8_t* pixels[3];
  int32_t* coeffs[3];
  int32_t* lapped[3];
  uint8_t* pixels_out[3];
  uint8_t* pred_pixels[3];         // cfg.inter: the prediction planes and their transform md
  int32_t* pred_coeffs[3];
  uint8_t* bsize;
  int16_t *qm, *qm_inv;
  double* rsqrt_tbl;
  int16_t* sp_vec[3];
  int32_t* sp_lanes[3];
  int32_t* sp_uni[3];
  int16_t* sp_snap[3];
  int sp_slots[3];
  Dering dering;                   // cfg.dering or cfg.inter_finish
  Lists lists;
  Stage luma, chroma;
  Sym sym;                         // symbol stream (cfg.symbol_stream); zero otherwise
  daala_b200_frame frame;
  daala_b200_frame frame_fwd;      // keyframes: `frame` for the forward transform, which always builds the DC pyramid
  daala_b200_frame frame_pred;     // cfg.inter: `frame` with the prediction planes as the forward transform's input / output
  // cfg.inter_mc: the reference-picture pool, slot map, MV grids and per-MV-block leaf segments
  uint8_t* ref_pixels[3];
  int32_t* ref_slot;
  daala_b200_mv_pt* mv_grid;
  int32_t* ref_slot_next;          // cfg.mc_next: each frame's NEXT slot and the mv1 grids; NULL otherwise
  int32_t* mv1_grid;
  uint32_t* mc_leaves;
  int32_t* mc_nleaves;
  daala_b200_mc_batch mc;
  // cfg.inter_finish: the finishing pass's inputs (decisions per block), its planes (patched coefficients, inverted in
  // place; the reconstruction), the skip maps, the superblock flags, the levels applied, and its own CUDA graph
  uint8_t* fin_skip[2];
  int32_t* fin_dc[2];
  int32_t* dc_resid[2];
  int32_t* fin_coeffs[3];
  uint8_t* fin_pixels[3];
  uint8_t* fin_bskip[3];
  uint8_t *fin_level, *fin_coded;
  Fin fin;
  cudaGraph_t fin_graph;
  cudaGraphExec_t fin_exec;
  bool fin_captured;
  int fin_dc_limit;                // largest |dc| finish accepts: DAALA_B200_KF_FINISH_DC_LIMIT / the largest dc_quant
                                   // of the last step's records
  // Lossy engines: each frame's record, its deringing threshold table ([F][2][6], daala_b200_dering_threshold_table of
  // its q0) and its band quantisers ([F][3][32], Stage::fq_bq).  The tables are computed on the host by fq_derive_host:
  // once at create from the config, or per step with frame_quant / keyframe_quant.
  daala_b200_kf_frame_quant* fq;
  int32_t* fq_tbl;
  std::vector<int32_t> fq_tbl_host;
  int32_t* fq_bq;
  std::vector<int32_t> fq_bq_host;
  // cfg.inter_mc with cfg.inter_finish: the pool slot of each frame's reconstruction (finish_io.ref_slot_out, -1 = not
  // stored) and the store that reads it
  int32_t* fin_slot_out;
  PoolStore store;
  // cfg.symbol_stream = 2 with cfg.inter_finish: the decisions of a stream-order finish (staged), the form flag
  // k_fin_unstream reads, and its parameters
  uint8_t* fin_stream_skip;
  int32_t* fin_stream_dc;
  int32_t* fin_form;
  Unstream unstream;
  // cfg.late_skip: the unquantised coefficients (a copy of `coeffs` taken before the finishing scatter), the records
  // per block of each list, and the parameters of the late-skip launches
  int32_t* d_orig[3];
  daala_b200_kf_late_skip* late_skip[2];
  daala_b200_late_skip_batch lsb;
  // cfg.lossless: the residual planes, the root-sum records, the keyframe DCs, the slot table of ll_ref_slot_out and the
  // parameters of the step (csrc/lossless.cu)
  int16_t* ll_coeffs[3];
  int32_t* ll_blocks;
  int32_t* ll_dc;
  int32_t* ll_slot_out;
  daala_b200_lossless_batch ll;
  // cfg.haar_dc_quant: the DC chain's grids (reconstructed DCs of all planes, frame by frame; signed indices per plane)
  // and its launch parameters
  int32_t* hdc;
  int32_t* hdc_index[3];
  daala_b200_haar_dc_batch hdcb;
  std::vector<uint8_t> slot_filled;  // cfg.inter_mc, per pool slot: something has written a picture there
  bool have_step;                  // a step has been submitted; last_tot are its totals
  daala_b200_kf_totals last_tot;
  std::vector<void*> allocs;       // every device buffer dalloc made; daala_b200_kf_destroy frees these
  size_t bytes_allocated;
  size_t chain_cap;                // entries of the chain queue (heads / ring)
  int sms;
  char err[256];
};

#define KF_CHECK(x)                                                                       \
  do {                                                                                    \
    cudaError_t e_ = (x);                                                                 \
    if (e_ != cudaSuccess) {                                                              \
      snprintf(kf->err, sizeof(kf->err), "%s: %s", #x, cudaGetErrorString(e_));           \
      return (int)e_;                                                                     \
    }                                                                                     \
  } while (0)

template <class T>
static cudaError_t dalloc(daala_b200_kf* kf, T** p, size_t n) {
  const size_t bytes = (n ? n : 1) * sizeof(T);
  cudaError_t e = cudaMalloc((void**)p, bytes);
  if (e == cudaSuccess) {
    kf->allocs.push_back(*p);
    kf->bytes_allocated += bytes;
    e = cudaMemset(*p, 0, bytes);
  }
  return e;
}

// cfg.inter_mc: the reference-picture pool, the slot map, the MV grids and the leaf segments of the prediction step
// (kf->pred_pixels must exist: the prediction's destination).
static int mc_alloc(daala_b200_kf* kf) {
  const int F = kf->F;
  daala_b200_mc_batch& B = kf->mc;
  const size_t nsb = (size_t)kf->nhsb * kf->nvsb;
  for (int p = 0; p < 3; p++) {
    KF_CHECK(dalloc(kf, &kf->ref_pixels[p], (size_t)kf->plane_w[p] * kf->plane_h[p] * kf->cfg.mc_refs));
    B.ref[p] = kf->ref_pixels[p];
    B.pred[p] = kf->pred_pixels[p];
    B.plane_w[p] = kf->plane_w[p];
    B.plane_h[p] = kf->plane_h[p];
  }
  KF_CHECK(dalloc(kf, &kf->ref_slot, (size_t)2 * F));
  KF_CHECK(dalloc(kf, &kf->mv_grid, (size_t)F * (kf->nvsb * 8 + 1) * (kf->nhsb * 8 + 1)));
  KF_CHECK(dalloc(kf, &kf->mc_leaves, (size_t)F * nsb * 64));
  KF_CHECK(dalloc(kf, &kf->mc_nleaves, (size_t)F * nsb));
  B.grid = kf->mv_grid;
  B.ref_slot = kf->ref_slot;
  B.leaves = kf->mc_leaves;
  B.nleaves = kf->mc_nleaves;
  B.F = F;
  B.nhsb = kf->nhsb;
  B.nvsb = kf->nvsb;
  B.nslots = kf->cfg.mc_refs;
  if (kf->cfg.mc_next) {
    KF_CHECK(dalloc(kf, &kf->ref_slot_next, (size_t)F));
    KF_CHECK(dalloc(kf, &kf->mv1_grid, (size_t)F * (kf->nvsb * 8 + 1) * (kf->nhsb * 8 + 1) * 2));
    B.ref_slot_next = kf->ref_slot_next;
    B.mv1 = kf->mv1_grid;
  }
  return 0;
}

// cfg.lossless: the input, prediction and reconstruction planes, [inter_mc: the pool], the counters and the lossless
// step's own buffers; nothing of the PVQ step.
static int ll_alloc(daala_b200_kf* kf) {
  const int F = kf->F;
  daala_b200_lossless_batch& B = kf->ll;
  memset(&B, 0, sizeof(B));
  for (int p = 0; p < 3; p++) {
    const size_t n = (size_t)kf->plane_w[p] * kf->plane_h[p] * F;
    KF_CHECK(dalloc(kf, &kf->pixels[p], n));
    KF_CHECK(dalloc(kf, &kf->pixels_out[p], n));
    KF_CHECK(dalloc(kf, &kf->ll_coeffs[p], n));
    if (kf->cfg.inter) KF_CHECK(dalloc(kf, &kf->pred_pixels[p], n));
    B.src[p] = kf->pixels[p];
    B.pred[p] = kf->pred_pixels[p];
    B.coeffs[p] = kf->ll_coeffs[p];
    B.out[p] = kf->pixels_out[p];
    B.plane_w[p] = kf->plane_w[p];
    B.plane_h[p] = kf->plane_h[p];
  }
  const size_t nrec = (size_t)F * kf->nhsb * kf->nvsb * 3;
  KF_CHECK(dalloc(kf, &kf->ll_blocks, nrec * 4));
  KF_CHECK(dalloc(kf, &kf->ll_dc, nrec));
  KF_CHECK(dalloc(kf, &kf->lists.cnt, (size_t)kCntWords));
  kf->mc.bad_ref = kf->lists.cnt + kMcBadRef;
  kf->mc.beyond = kf->lists.cnt + kMcBeyond;
  if (kf->cfg.inter_mc) {
    int rc = mc_alloc(kf);
    if (rc) return rc;
    KF_CHECK(dalloc(kf, &kf->ll_slot_out, (size_t)F));
    for (int p = 0; p < 3; p++) B.pool[p] = kf->ref_pixels[p];
    B.slot_out = kf->ll_slot_out;
  }
  B.blocks = kf->ll_blocks;
  B.dc = kf->ll_dc;
  B.F = F;
  B.nhsb = kf->nhsb;
  B.nvsb = kf->nvsb;
  B.pic_w = kf->cfg.pic_w;
  B.pic_h = kf->cfg.pic_h;
  // dalloc's clears run on the legacy default stream (see the end of kf_alloc)
  KF_CHECK(cudaDeviceSynchronize());
  return 0;
}

// The records of a step ([F]): why they are refused, or nullptr when every one is in range; then the host tables hold
// each frame's deringing thresholds (daala_b200_kf_frame_quant_derive) and band quantisers, and *dc_limit is the
// finishing pass's DC limit.  check = false: records made from the config, whose fields a mode that does not read them
// may leave out of range (coded_quantizer = 0 without dering = 2); create has checked q0.
static const char* fq_derive_host(daala_b200_kf* kf, const daala_b200_kf_frame_quant* rec, bool check, int* dc_limit) {
  if (!rec) return "frame_quant: the records ([nframes]) are required";
  const int F = kf->F;
  for (int f = 0; check && f < F; f++) {
    const daala_b200_kf_frame_quant& r = rec[f];
    if (r.q0 < 1 || r.q0 > DAALA_B200_KF_MAX_Q0) return "a record's q0 is outside [1, 8191]";
    if (r.coded_quantizer < 1 || r.coded_quantizer > 63) return "a record's coded_quantizer is outside [1, 63]";
    if (!std::isfinite(r.dering_lambda) || r.dering_lambda < 0) return "a record's dering_lambda is negative or not finite";
    for (int p = 0; p < 3; p++)
      for (int i = 0; i < 30; i++)   // OD_QM_SIZE entries are read
        if (r.pvq_qm_q4[p][i] < 1) return "a record's pvq_qm_q4 entry is 0";
  }
  *dc_limit = daala_b200_kf_frame_quant_derive(rec, F, reinterpret_cast<int32_t(*)[2][6]>(kf->fq_tbl_host.data()));
  for (int f = 0; f < F; f++)
    for (int p = 0; p < 3; p++)
      for (int i = 0; i < 30; i++)
        kf->fq_bq_host[(size_t)(f * 3 + p) * 32 + i] = std::max(1, (rec[f].q0 * rec[f].pvq_qm_q4[p][i]) >> 4);
  return nullptr;
}

// The H2D of the records fq_derive_host accepted and of its tables, on `s`.
static cudaError_t fq_copy(daala_b200_kf* kf, const daala_b200_kf_frame_quant* rec, cudaStream_t s) {
  const int F = kf->F;
  cudaError_t e = cudaMemcpyAsync(kf->fq, rec, sizeof(daala_b200_kf_frame_quant) * F, cudaMemcpyHostToDevice, s);
  if (!e) e = cudaMemcpyAsync(kf->fq_tbl, kf->fq_tbl_host.data(), sizeof(int32_t) * 12 * F, cudaMemcpyHostToDevice, s);
  if (!e) e = cudaMemcpyAsync(kf->fq_bq, kf->fq_bq_host.data(), sizeof(int32_t) * 96 * F, cudaMemcpyHostToDevice, s);
  return e;
}

static int kf_alloc(daala_b200_kf* kf) {
  if (kf->cfg.lossless) return ll_alloc(kf);
  const int F = kf->F;
  const bool inter = kf->cfg.inter != 0;
  const long long luma_px = (long long)kf->plane_w[0] * kf->plane_h[0];
  for (int p = 0; p < 3; p++) {
    const size_t n = (size_t)kf->plane_w[p] * kf->plane_h[p] * F;
    KF_CHECK(dalloc(kf, &kf->pixels[p], n));
    KF_CHECK(dalloc(kf, &kf->coeffs[p], n));
    KF_CHECK(dalloc(kf, &kf->lapped[p], n));
    KF_CHECK(dalloc(kf, &kf->pixels_out[p], n));
    if (inter) {
      KF_CHECK(dalloc(kf, &kf->pred_pixels[p], n));
      KF_CHECK(dalloc(kf, &kf->pred_coeffs[p], n));
    }
  }
  const int UW = kf->nhsb * 8, UH = kf->nvsb * 8;
  KF_CHECK(dalloc(kf, &kf->bsize, (size_t)F * UW * UH));
  if (kf->cfg.inter_mc) {
    const int rc = mc_alloc(kf);
    if (rc) return rc;
  }
  KF_CHECK(dalloc(kf, &kf->fq, (size_t)F));
  KF_CHECK(dalloc(kf, &kf->fq_tbl, (size_t)F * 12));
  KF_CHECK(dalloc(kf, &kf->fq_bq, (size_t)F * 96));
  kf->fq_tbl_host.assign((size_t)F * 12, 0);
  kf->fq_bq_host.assign((size_t)F * 96, 1);
  KF_CHECK(dalloc(kf, &kf->qm, (size_t)2 * kf->cfg.qm_stride));
  KF_CHECK(dalloc(kf, &kf->qm_inv, (size_t)2 * kf->cfg.qm_stride));
  KF_CHECK(dalloc(kf, &kf->rsqrt_tbl, (size_t)kTableDoubles));
  KF_CHECK(cudaMemcpy(kf->qm, kf->cfg.qm, sizeof(int16_t) * 2 * kf->cfg.qm_stride, cudaMemcpyHostToDevice));
  KF_CHECK(cudaMemcpy(kf->qm_inv, kf->cfg.qm_inv, sizeof(int16_t) * 2 * kf->cfg.qm_stride, cudaMemcpyHostToDevice));

  Lists& L = kf->lists;
  memset(&L, 0, sizeof(L));
  L.bsize = kf->bsize;
  L.bstride = UW;
  L.bsize_pitch = (long long)UW * UH;
  L.F = F;
  L.UW = UW;
  L.UH = UH;
  L.u_row0 = kf->cfg.sb_row0 * 8;
  L.u_rows = kf->cfg.sb_rows * 8;
  const long long nunits = (long long)F * L.u_rows * UW;
  L.ntiles = (int)((nunits + kTile - 1) / kTile);
  // capacities: every unit coded as four 4x4 luma blocks / one 4x4 chroma block per plane, unless the
  // caller bounds the smallest block size it will ever submit
  const int div = kf->cfg.max_blocks_div > 0 ? kf->cfg.max_blocks_div : 1;
  L.max_luma = (int)(nunits * 4 / div) + 64;
  L.max_chroma = (int)(nunits * 2 / div) + 64;
  KF_CHECK(dalloc(kf, &L.tile_sum, (size_t)L.ntiles));
  KF_CHECK(dalloc(kf, &L.unit_lbase, (size_t)F * UW * UH));
  if (!inter) KF_CHECK(dalloc(kf, &L.unit_loff, (size_t)F * UW * UH));
  KF_CHECK(dalloc(kf, &L.luma, (size_t)L.max_luma));
  KF_CHECK(dalloc(kf, &L.chroma, (size_t)L.max_chroma));
  // the intra dependency structure (neighbours, chain heads, ring) is a keyframe matter
  const size_t ndep = inter ? 0 : (size_t)L.max_luma;
  KF_CHECK(dalloc(kf, &L.dep_top, ndep));
  KF_CHECK(dalloc(kf, &L.dep_left, ndep));
  KF_CHECK(dalloc(kf, &L.succ_bottom, ndep));
  KF_CHECK(dalloc(kf, &L.succ_right, ndep));
  // item capacities follow from the pixel count alone: one band per 4x4 block is the densest case
  const size_t luma_shard_px = (size_t)F * L.u_rows * UW * 64;
  kf->chain_cap = luma_shard_px / 16 + 64 + (size_t)kf->sms * 64;   // + one exit slot per persistent warp
  // keyframes: bands 3 / 6 only.  inter: every band; class 0 (bands 0..2) is densest on an all-4x4 map (one item
  // per block) or an all-8x8 one (three per block), classes 1 / 2 on all-8x8 / all-16x16 maps, one item per block
  const size_t cap_l0 = (size_t)L.max_luma * 3 < luma_shard_px / 16 ? (size_t)L.max_luma * 3 : luma_shard_px / 16;
  const size_t cap_l[3] = {inter ? cap_l0 + 64 : 64, luma_shard_px / 64 + 64, luma_shard_px / 256 + 64};
  const size_t cap_c[3] = {(size_t)L.max_chroma * 3 / 2 + 64, luma_shard_px / 4 * 2 * 3 / 64 + 64,
                           luma_shard_px / 4 * 2 * 3 / 256 + 64};
  for (int c = 0; c < 3; c++) {
    KF_CHECK(dalloc(kf, &L.items_l[c], cap_l[c]));
    KF_CHECK(dalloc(kf, &L.items_c[c], cap_c[c]));
  }
  {
    // context records of one chunk of items per class (pvq_warp.cuh: band_ctx_*)
    const int slots[3] = {1 << 19, 1 << 19, 3 << 15};
    for (int c = 0; c < 3; c++) {
      const int vs = c == 2 ? 128 : 32;
      kf->sp_slots[c] = slots[c];
      KF_CHECK(dalloc(kf, &kf->sp_vec[c], (size_t)slots[c] * 3 * vs));
      KF_CHECK(dalloc(kf, &kf->sp_lanes[c], (size_t)slots[c] * kCtxLaneWords * 16));
      KF_CHECK(dalloc(kf, &kf->sp_uni[c], (size_t)slots[c] * kCtxUniWords));
      KF_CHECK(dalloc(kf, &kf->sp_snap[c], (size_t)slots[c] * kMaxEvents * vs));
    }
  }
  {
    // the persistent grid is sized to be resident at once: 32 one-warp CTAs with kSnapEntries of shared
    // scratch each (plus the 1 KB the SM reserves per CTA) need 223 of the SM's 228 KB
    const int want = kf->cfg.persist_ctas_per_sm > 0 ? kf->cfg.persist_ctas_per_sm : kPersistCtas;
    int per_sm = 0;
    KF_CHECK(cudaFuncSetAttribute(k_pvq_persist, cudaFuncAttributePreferredSharedMemoryCarveout,
                                  cudaSharedmemCarveoutMaxShared));
    KF_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pvq_persist, kPersistThreads, 0));
    if (per_sm < want) {
      snprintf(kf->err, sizeof(kf->err), "k_pvq_persist: %d CTAs per SM resident, %d wanted", per_sm, want);
      return (int)cudaErrorLaunchOutOfResources;
    }
  }
  KF_CHECK(dalloc(kf, &L.heads, inter ? 0 : kf->chain_cap));
  KF_CHECK(dalloc(kf, &L.heads_raw, inter ? 0 : kf->chain_cap));
  KF_CHECK(dalloc(kf, &L.head_bin, inter ? 0 : kf->chain_cap));
  KF_CHECK(dalloc(kf, &L.head_hist, inter ? 0 : (size_t)kHeadBins));
  KF_CHECK(dalloc(kf, &L.head_cursor, inter ? 0 : (size_t)kHeadBins));
  KF_CHECK(dalloc(kf, &L.heads0, ndep));
  KF_CHECK(dalloc(kf, &L.cnt, (size_t)kCntWords));
  kf->mc.bad_ref = L.cnt + kMcBadRef;
  kf->mc.beyond = L.cnt + kMcBeyond;

  auto setup_stage = [&](Stage& S, bool chroma) -> int {
    memset(&S, 0, sizeof(S));
    daala_b200_pvq_params& p = S.prm;
    const size_t ncoef = chroma ? luma_shard_px / 2 + 1024 : luma_shard_px + 1024;
    const size_t nblk = chroma ? L.max_chroma : L.max_luma;
    p.blocks = chroma ? L.chroma : L.luma;
    KF_CHECK(dalloc(kf, &p.in, ncoef));
    KF_CHECK(dalloc(kf, &p.ref, ncoef));
    KF_CHECK(dalloc(kf, &p.out, ncoef));
    KF_CHECK(dalloc(kf, &p.y, ncoef));
    KF_CHECK(dalloc(kf, &p.y16, ncoef));
    KF_CHECK(dalloc(kf, &p.res_skip_term, nblk * 9));
    KF_CHECK(dalloc(kf, &p.res_skip_diff, nblk));
    KF_CHECK(dalloc(kf, &p.res_flip, nblk));
    KF_CHECK(dalloc(kf, &S.res_pack, nblk * 9 * 4));
    p.res_gain = p.res_theta = p.res_max_theta = p.res_k = nullptr;   // packed into res_pack here
    p.res_dc = nullptr;
    if (inter) KF_CHECK(dalloc(kf, &p.res_dc, nblk));
    p.qm = kf->qm;
    p.qm_inv = kf->qm_inv;
    for (int i = 0; i < 3; i++) {
      p.coef_plane[i] = kf->coeffs[i];
      p.pred_plane[i] = kf->pred_coeffs[i];
      p.plane_frame_pitch[i] = (long long)kf->plane_w[i] * kf->plane_h[i];
      p.plane_stride[i] = kf->plane_w[i];
    }
    p.qm_stride = kf->cfg.qm_stride;
    p.is_keyframe = inter ? 0 : 1;
    p.use_masking = kf->cfg.use_masking;
    p.pvq_norm_lambda = kf->cfg.pvq_norm_lambda;
    S.fq_bq = kf->fq_bq;
    for (int c = 0; c < 3; c++) S.items[c] = chroma ? L.items_c[c] : L.items_l[c];
    S.cnt = L.cnt;
    S.rsqrt_tbl = kf->rsqrt_tbl;
    for (int c = 0; c < 3; c++) {
      S.sp_vec[c] = kf->sp_vec[c];
      S.sp_lanes[c] = kf->sp_lanes[c];
      S.sp_uni[c] = kf->sp_uni[c];
      S.sp_snap[c] = kf->sp_snap[c];
      S.sp_slots[c] = kf->sp_slots[c];
      const size_t cap = chroma ? cap_c[c] : cap_l[c];
      S.sp_chunks[c] = kf->sp_slots[c] > 0 ? (int)((cap + kf->sp_slots[c] - 1) / kf->sp_slots[c]) : 0;
    }
    S.max_waiters = kf->sms * 8;
    S.n_items_at = chroma ? kNItemsC : kNItemsL;
    S.head_lo_at = chroma ? kHeadLoC : kHeadLoL;
    S.n_blocks_at = chroma ? kNChroma : kNLuma;
    S.max_blocks = (int)nblk;
#ifdef DAALA_B200_CHAIN_TRACE
    if (!chroma && !inter) {
      S.trace_cap = (int)(luma_shard_px / 16);   // one band per 16 pixels at most
      KF_CHECK(dalloc(kf, &S.trace, (size_t)S.trace_cap));
    }
#endif
    if (!chroma) {
      S.dep_top = L.dep_top;
      S.dep_left = L.dep_left;
      S.succ_bottom = L.succ_bottom;
      S.succ_right = L.succ_right;
      S.heads = L.heads;
      S.heads0 = L.heads0;
      KF_CHECK(dalloc(kf, &S.ring, inter ? 0 : kf->chain_cap));
      KF_CHECK(dalloc(kf, &S.join0, ndep));
    }
    return 0;
  };
  int rc = setup_stage(kf->luma, false);
  if (rc) return rc;
  rc = setup_stage(kf->chroma, true);
  if (rc) return rc;
  if (!inter) {
    Stage& C = kf->chroma;
    C.cfl_in = kf->luma.prm.in;
    C.cfl_out = kf->luma.prm.out;
    C.cfl_loff = L.unit_loff;
  }
  if (kf->cfg.haar_dc_quant) {
    daala_b200_haar_dc_batch& H = kf->hdcb;
    memset(&H, 0, sizeof(H));
    const size_t g0 = (size_t)(kf->plane_w[0] >> 2) * (kf->plane_h[0] >> 2), g1 = (size_t)(kf->plane_w[1] >> 2) * (kf->plane_h[1] >> 2);
    KF_CHECK(dalloc(kf, &kf->hdc, (g0 + 2 * g1) * F));
    H.grid_frame_pitch = (long long)(g0 + 2 * g1);
    kf->luma.cfl_in = kf->chroma.cfl_in = kf->hdc;
    for (int p = 0; p < 3; p++) {
      KF_CHECK(dalloc(kf, &kf->hdc_index[p], (p ? g1 : g0) * F));
      H.coeffs[p] = kf->coeffs[p];
      H.dc[p] = kf->hdc + (p ? g0 + (p - 1) * g1 : 0);
      H.index[p] = kf->hdc_index[p];
      H.plane_w[p] = kf->plane_w[p];
      H.plane_h[p] = kf->plane_h[p];
    }
    H.bsize = kf->bsize;
    H.F = F;
    H.nhsb = kf->nhsb;
    H.nvsb = kf->nvsb;
    H.pvq_norm_lambda = kf->cfg.pvq_norm_lambda;
    H.fq_bq = kf->fq_bq;
  }
  (void)luma_px;
  // the unquantised DC residual per block: what the host's od_rdo_quant needs, returned classically (inter_finish) or
  // in the stream's DC records (symbol_stream = 2)
  if (kf->cfg.inter_finish || kf->cfg.symbol_stream == 2)
    for (int c = 0; c < 2; c++) {
      Stage& S = c ? kf->chroma : kf->luma;
      KF_CHECK(dalloc(kf, &kf->dc_resid[c], (size_t)S.max_blocks));
      S.dc_resid = kf->dc_resid[c];
    }
  if (kf->cfg.symbol_stream) {
    Sym& Y = kf->sym;
    memset(&Y, 0, sizeof(Y));
    Y.bsize = kf->bsize;
    Y.bstride = UW;
    Y.bsize_pitch = (long long)UW * UH;
    Y.F = F;
    Y.nhsb = kf->nhsb;
    Y.sb_rows = kf->cfg.sb_rows;
    Y.u_row0 = L.u_row0;
    Y.nsb = kf->nhsb * kf->cfg.sb_rows;
    Y.cap_blocks = L.max_luma + L.max_chroma;
    Y.ntiles = (Y.cap_blocks + kTile - 1) / kTile;
    // every band has at least 8 coefficients and 4x4 / 8x8 blocks have one band per 16: bands <= coefficients / 16
    const size_t ncoef = (luma_shard_px + 1024) + (luma_shard_px / 2 + 1024);
    KF_CHECK(dalloc(kf, &Y.unit_rank, (size_t)F * L.u_rows * UW));
    KF_CHECK(dalloc(kf, &Y.sb_cnt, (size_t)F * Y.nsb));
    KF_CHECK(dalloc(kf, &Y.sb_base, (size_t)F * Y.nsb));
    KF_CHECK(dalloc(kf, &Y.order, (size_t)Y.cap_blocks));
    KF_CHECK(dalloc(kf, &Y.off, (size_t)Y.cap_blocks));
    KF_CHECK(dalloc(kf, &Y.tile, (size_t)Y.ntiles));
    KF_CHECK(dalloc(kf, &Y.tot, (size_t)4));
    KF_CHECK(dalloc(kf, &Y.index, (size_t)F));
    KF_CHECK(dalloc(kf, &Y.blocks, (size_t)Y.cap_blocks));
    Y.cap_bands = (long long)(ncoef / 16);
    Y.cap_bytes = (long long)(2 * ncoef);
    KF_CHECK(dalloc(kf, &Y.bands, ncoef / 16));
    KF_CHECK(dalloc(kf, &Y.pulses, 2 * ncoef));
    for (int c = 0; c < 2; c++) {
      const Stage& S = c ? kf->chroma : kf->luma;
      Y.list[c] = S.prm.blocks;
      Y.res[c] = reinterpret_cast<const short4*>(S.res_pack);
      Y.y[c] = S.prm.y;
      Y.skip_diff[c] = S.prm.res_skip_diff;
    }
    Y.flip = kf->chroma.prm.res_flip;
    Y.cnt = L.cnt;
    Y.max_luma = L.max_luma;
    Y.max_chroma = L.max_chroma;
    if (kf->cfg.symbol_stream == 2) {
      KF_CHECK(dalloc(kf, &Y.dc, (size_t)Y.cap_blocks));
      for (int c = 0; c < 2; c++) {
        Y.qdc[c] = (c ? kf->chroma : kf->luma).prm.res_dc;
        Y.dc_resid[c] = kf->dc_resid[c];
      }
    }
    if (kf->cfg.haar_dc_quant) {
      KF_CHECK(dalloc(kf, &Y.hdc, (size_t)Y.cap_blocks));
      for (int p = 0; p < 3; p++) {
        Y.hdc_index[p] = kf->hdc_index[p];
        Y.gw[p] = kf->plane_w[p] >> 2;
        Y.gh[p] = kf->plane_h[p] >> 2;
      }
    }
  }
  if (kf->cfg.late_skip) {
    daala_b200_late_skip_batch& B = kf->lsb;
    memset(&B, 0, sizeof(B));
    long long px = 0;
    for (int p = 0; p < 3; p++) {
      const size_t n = (size_t)kf->plane_w[p] * kf->plane_h[p] * F;
      KF_CHECK(dalloc(kf, &kf->d_orig[p], n));
      px += (long long)n;
      B.d_orig[p] = kf->d_orig[p];
      B.d[p] = kf->coeffs[p];
      B.md[p] = kf->pred_coeffs[p];
      B.plane_pitch[p] = (long long)kf->plane_w[p] * kf->plane_h[p];
      B.plane_stride[p] = kf->plane_w[p];
    }
    for (int c = 0; c < 2; c++) {
      const Stage& S = c ? kf->chroma : kf->luma;
      KF_CHECK(dalloc(kf, &kf->late_skip[c], (size_t)S.max_blocks));
      B.blocks[c] = S.prm.blocks;
      B.count[c] = L.cnt + S.n_blocks_at;
      B.max_blocks[c] = S.max_blocks;
      B.out[c] = kf->late_skip[c];
    }
    KF_CHECK(dalloc(kf, &B.cls_items, (size_t)daala_b200_late_skip_class_caps(px, B.cls_off, B.cls_cap)));
    KF_CHECK(dalloc(kf, &B.cls_n, (size_t)4));
    B.qm_is_flat = kf->cfg.qm_is_flat;
    B.use_activity_masking = kf->cfg.use_masking;
    B.fq = kf->fq;
    B.fq_bq = kf->fq_bq;
    if (kf->cfg.symbol_stream == 2) {
      Sym& Y = kf->sym;
      KF_CHECK(dalloc(kf, &Y.late_skip, (size_t)Y.cap_blocks));
      Y.ls_block[0] = kf->late_skip[0];
      Y.ls_block[1] = kf->late_skip[1];
    }
  }

  daala_b200_frame& f = kf->frame;
  memset(&f, 0, sizeof(f));
  for (int p = 0; p < 3; p++) {
    daala_b200_plane& pl = f.plane[p];
    pl.pixels = kf->pixels[p];
    pl.coeffs = kf->coeffs[p];
    pl.lapped = kf->lapped[p];
    pl.pixels_out = kf->pixels_out[p];
    pl.pixel_stride = pl.coeff_stride = pl.lapped_stride = pl.pixel_out_stride = kf->plane_w[p];
    pl.xdec = p ? 1 : 0;
    pl.pixel_frame_pitch = pl.coeff_frame_pitch = pl.lapped_frame_pitch = pl.pixel_out_frame_pitch =
        (long long)kf->plane_w[p] * kf->plane_h[p];
  }
  f.bsize = kf->bsize;
  f.bstride = UW;
  f.bsize_frame_pitch = (long long)UW * UH;
  f.nhsb = kf->nhsb;
  f.nvsb = kf->nvsb;
  f.pic_w = kf->cfg.pic_w;
  f.pic_h = kf->cfg.pic_h;
  // haar_dc_quant: the leaf DCs the finishing scatter stores are final, as on P frames, so the inverse skips the
  // pyramid; the forward (frame_fwd) still builds it for the DC chain
  f.haar_dc = inter || kf->cfg.haar_dc_quant ? 0 : 1;
  f.nframes = F;
  f.sb_row0 = kf->cfg.sb_row0;
  f.sb_rows = kf->cfg.sb_rows;
  kf->frame_pred = f;
  kf->frame_fwd = f;
  kf->frame_fwd.haar_dc = inter ? 0 : 1;
  for (int p = 0; p < 3; p++) {
    kf->frame_pred.plane[p].pixels = kf->pred_pixels[p];
    kf->frame_pred.plane[p].coeffs = kf->pred_coeffs[p];
  }
  if (kf->cfg.inter_finish) {
    const size_t nsb = (size_t)F * kf->nhsb * kf->nvsb;
    Fin& P = kf->fin;
    memset(&P, 0, sizeof(P));
    for (int c = 0; c < 2; c++) {
      const Stage& S = c ? kf->chroma : kf->luma;
      KF_CHECK(dalloc(kf, &kf->fin_skip[c], (size_t)S.max_blocks));
      KF_CHECK(dalloc(kf, &kf->fin_dc[c], (size_t)S.max_blocks));
      P.blocks[c] = S.prm.blocks;
      P.skip[c] = kf->fin_skip[c];
      P.dc[c] = kf->fin_dc[c];
      P.max_blocks[c] = S.max_blocks;
    }
    P.cnt = L.cnt;
    P.skip_stride = kf->nhsb * 16;
    for (int p = 0; p < 3; p++) {
      const size_t n = (size_t)kf->plane_w[p] * kf->plane_h[p] * F;
      KF_CHECK(dalloc(kf, &kf->fin_coeffs[p], n));
      KF_CHECK(dalloc(kf, &kf->fin_pixels[p], n));
      P.skip_pitch[p] = (long long)(kf->plane_h[p] / 4) * P.skip_stride;
      KF_CHECK(dalloc(kf, &kf->fin_bskip[p], (size_t)P.skip_pitch[p] * F));
      P.d[p] = kf->coeffs[p];
      P.md[p] = kf->pred_coeffs[p];
      P.out[p] = kf->fin_coeffs[p];
      P.plane_pitch[p] = (long long)kf->plane_w[p] * kf->plane_h[p];
      P.plane_stride[p] = kf->plane_w[p];
      P.bskip[p] = kf->fin_bskip[p];
    }
    KF_CHECK(dalloc(kf, &kf->fin_level, nsb));
    KF_CHECK(dalloc(kf, &kf->fin_coded, nsb));
    P.coded = kf->fin_coded;
    P.nhsb = kf->nhsb;
    P.nvsb = kf->nvsb;
    P.fq_bq = kf->fq_bq;
    if (kf->cfg.inter_mc) {
      KF_CHECK(dalloc(kf, &kf->fin_slot_out, (size_t)F));
      PoolStore& W = kf->store;
      for (int p = 0; p < 3; p++) {
        W.src[p] = kf->fin_pixels[p];
        W.pool[p] = kf->ref_pixels[p];
        W.plane_bytes[p] = (long long)kf->plane_w[p] * kf->plane_h[p];
      }
      W.slot = kf->fin_slot_out;
    }
    if (kf->cfg.symbol_stream == 2) {
      Unstream& U = kf->unstream;
      KF_CHECK(dalloc(kf, &kf->fin_stream_skip, (size_t)kf->sym.cap_blocks));
      KF_CHECK(dalloc(kf, &kf->fin_stream_dc, (size_t)kf->sym.cap_blocks));
      KF_CHECK(dalloc(kf, &kf->fin_form, (size_t)1));
      U.order = kf->sym.order;
      U.tot = kf->sym.tot;
      U.skip = kf->fin_stream_skip;
      U.dc = kf->fin_stream_dc;
      for (int c = 0; c < 2; c++) {
        U.fin_skip[c] = kf->fin_skip[c];
        U.fin_dc[c] = kf->fin_dc[c];
      }
      U.form = kf->fin_form;
    }
  }
  // the deringing pass: the step's on keyframes (cfg.dering) or the finishing pass's (cfg.inter_finish); inter refuses
  // dering, so an engine has at most one.  Level 2 of either searches the levels first.
  const int dering = kf->cfg.dering ? kf->cfg.dering : kf->cfg.inter_finish;
  if (dering) {
    const size_t nsb = (size_t)F * kf->nhsb * kf->nvsb;
    Dering& D = kf->dering;
    D.frame = kf->frame;
    D.skip_stride = kf->nhsb * 16;
    uint8_t* zero_skip = nullptr;   // keyframes never mark a block skipped (src/encode.c:1690): one map for all frames
    if (!kf->cfg.inter_finish) KF_CHECK(dalloc(kf, &zero_skip, nsb * 256 + 64));
    for (int p = 0; p < 3; p++) {
      KF_CHECK(dalloc(kf, &D.frame.post16[p], (size_t)kf->plane_w[p] * kf->plane_h[p] * F));
      if (kf->cfg.inter_finish) {
        // the patched coefficients, inverted in place (k_inverse_sb only touches its own superblock)
        D.frame.plane[p].coeffs = D.frame.plane[p].lapped = kf->fin_coeffs[p];
        D.frame.plane[p].pixels_out = kf->fin_pixels[p];
        D.skip[p] = kf->fin_bskip[p];
        D.skip_pitch[p] = kf->fin.skip_pitch[p];
      } else {
        D.skip[p] = zero_skip;
      }
    }
    KF_CHECK(dalloc(kf, &D.level, nsb));
    KF_CHECK(dalloc(kf, &D.thr[0], nsb));
    KF_CHECK(dalloc(kf, &D.thr[1], nsb));
    KF_CHECK(dalloc(kf, &D.dir, nsb * 64));
    D.coded = kf->fin_coded;
    D.applied = kf->fin_level;
    D.frame_tbl = kf->fq_tbl;
    D.search = dering == 2;
    if (D.search) {
      // src/encode.c:2708-2811 for every frame of the batch.  P frames (src/encode.c:2720-2811): the frame's own skip
      // map under every candidate, superblocks without a coded luma 4x4 unit neither scored nor adapted, context 0
      daala_b200_dering_search_batch& b = D.sb;
      b.etmp = D.frame.post16[0];
      b.src = kf->pixels[0];
      b.etmp_pitch = b.src_pitch = (long long)kf->plane_w[0] * kf->plane_h[0];
      b.etmp_stride = b.src_stride = kf->plane_w[0];
      b.nframes = F;
      b.nhsb = kf->nhsb;
      b.nvsb = kf->nvsb;
      b.qm_is_flat = kf->cfg.qm_is_flat;
      b.use_activity_masking = kf->cfg.use_masking;
      b.bskip = D.skip[0];
      b.skip_stride = D.skip_stride;
      b.skip_pitch = D.skip_pitch[0];
      b.coded = D.coded;
      b.is_keyframe = inter ? 0 : 1;
      KF_CHECK(dalloc(kf, &b.filt, (size_t)kf->plane_w[0] * kf->plane_h[0] * F));
      KF_CHECK(dalloc(kf, &b.orig, nsb * 4096));
      KF_CHECK(dalloc(kf, &b.cand, nsb * 4096));
      KF_CHECK(dalloc(kf, &b.dist, nsb * 6));
      b.dir = D.dir;
      b.levels = D.level;   // what the thresholds read; on P frames its level 0 agrees with the forced one
      b.fq = kf->fq;
      b.frame_tbl = kf->fq_tbl;
      KF_CHECK(dalloc(kf, &b.cand_thr, nsb * 5));
    }
  }
  // dalloc's cudaMemset runs on the legacy default stream, asynchronously, and the engine's stream does not
  // synchronise with it (cudaStreamNonBlocking): wait for every clear before anything is launched -- the table
  // fill below used to race with the clear of its own buffer (intermittently all-zero 1/sqrt table)
  KF_CHECK(cudaDeviceSynchronize());
  k_fill_rsqrt<<<(kTableDoubles + 255) / 256, 256, 0, kf->stream>>>(kf->rsqrt_tbl);
  KF_CHECK(cudaGetLastError());
  // every frame at the config's quantizer; frame_quant / keyframe_quant replace the records with each step's
  std::vector<daala_b200_kf_frame_quant> rec((size_t)F);
  for (daala_b200_kf_frame_quant& r : rec) {
    r.q0 = kf->cfg.q0;
    r.coded_quantizer = kf->cfg.coded_quantizer;
    r.dering_lambda = kf->cfg.dering_lambda;
    memcpy(r.pvq_qm_q4, kf->cfg.pvq_qm_q4, sizeof(r.pvq_qm_q4));
  }
  fq_derive_host(kf, rec.data(), false, &kf->fin_dc_limit);
  KF_CHECK(fq_copy(kf, rec.data(), kf->stream));
  KF_CHECK(cudaStreamSynchronize(kf->stream));
  return 0;
}

// Inverse of planes [p0, p0 + n): iDCT + split postfilters -> lapped planes; SB-edge postfilter -> the u8 planes, or
// etmp (int16) when frame.post16 is set (the deringing stage's input).
static int enqueue_recon(const daala_b200_frame& frame, int p0, int n, cudaStream_t s) {
  const int rc = daala_b200_launch_inverse_lapped_only(&frame, p0, n, s);
  return rc ? rc : daala_b200_launch_sb_postfilter_store(&frame, p0, n, s);
}

// od_dering of all frames of plane p in one launch, storing the u8 reconstruction.
static int enqueue_dering_plane(daala_b200_kf* kf, const Dering& D, int p, cudaStream_t s) {
  const int nsb = kf->nhsb * kf->nvsb;
  const long long per = (long long)kf->plane_w[p] * kf->plane_h[p];
  daala_b200_dering_params dp;
  memset(&dp, 0, sizeof(dp));
  dp.y = nullptr;   // u8 output only
  dp.x = D.frame.post16[p];
  dp.dir = D.dir;
  dp.bskip = D.skip[p];
  dp.sb_threshold = D.thr[p ? 1 : 0];
  dp.ystride = dp.xstride = kf->plane_w[p];
  dp.dir_stride = kf->nhsb * 8;
  dp.skip_stride = D.skip_stride;
  dp.nhsb = kf->nhsb;
  dp.nvsb = kf->nvsb;
  dp.xdec = p ? 1 : 0;
  dp.pli = p;
  dp.overlap = 1;      // OD_DERING_CHECK_OVERLAP
  dp.coeff_shift = 4;  // OD_COEFF_SHIFT
  // after a search the direction map is already there, packed with the variance; neither depends on the skip map
  // (src/dering.c:280-287)
  dp.dir_format = D.search ? 2 : 0;
  return daala_b200_dering_plane_frames(&dp, kf->F, per, per, (long long)nsb * 64, nsb, D.skip_pitch[p],
                                        D.frame.plane[p].pixels_out, s);
}

// The deringing pass D after the inverse: [the level search -> D.level]; thresholds per superblock (both plane
// kinds); od_dering of plane 0, which writes the direction map the chroma planes read.
static int enqueue_dering_luma(daala_b200_kf* kf, const Dering& D, cudaStream_t s) {
  if (D.search) {
    const int rc = daala_b200_dering_search_enqueue(&D.sb, s);
    if (rc) return rc;
  }
  const int nsb = kf->nhsb * kf->nvsb;
  k_dering_thresholds<<<(kf->F * nsb + 255) / 256, 256, 0, s>>>(D.level, D.thr[0], D.thr[1], kf->F * nsb, D.coded,
                                                                   D.applied, D.frame_tbl, nsb);
  return enqueue_dering_plane(kf, D, 0, s);
}

// The deringing pass D over the whole batch on one stream: inverse of all planes, then enqueue_dering_luma, then
// od_dering of the chroma planes.
static int enqueue_dering(daala_b200_kf* kf, const Dering& D, cudaStream_t s) {
  int rc = enqueue_recon(D.frame, 0, 3, s);
  if (!rc) rc = enqueue_dering_luma(kf, D, s);
  for (int p = 1; !rc && p < 3; p++) rc = enqueue_dering_plane(kf, D, p, s);
  return rc;
}

// Kernel launches of enqueue_dering with the inverse in `parts` plane ranges: inverse, SB postfilter -> int16 per
// range, [level search: the candidates' thresholds, 5 filtered candidates, 6 packs, 6 distortion passes, decision],
// thresholds, dering + u8 store per plane.
static int dering_launches(const Dering& D, int parts) {
  return 2 * parts + (D.search ? 1 + 5 + 6 + 6 + 1 : 0) + 1 + 3;
}

// Everything between "inputs are in HBM" and "results are in HBM", on kf->stream.
// the three phase kernels over every chunk of every class of a stage's dependency-free lists
static void enqueue_split(daala_b200_kf* kf, const Stage& S, cudaStream_t s) {
  const int grid = kf->sms * 16;
  for (int cls = 2; cls >= 0; cls--) {
    for (int chunk = 0; chunk < S.sp_chunks[cls]; chunk++) {
      if (cls == 2) {
        k_pvq_split<0, 2><<<grid, 128, 0, s>>>(S, cls, chunk);
        k_pvq_split<1, 2><<<grid, 128, 0, s>>>(S, cls, chunk);
        k_pvq_split<2, 2><<<grid, 128, 0, s>>>(S, cls, chunk);
      } else {
        k_pvq_split<0, 1><<<grid, 128, 0, s>>>(S, cls, chunk);
        k_pvq_split<1, 1><<<grid, 128, 0, s>>>(S, cls, chunk);
        k_pvq_split<2, 1><<<grid, 128, 0, s>>>(S, cls, chunk);
      }
    }
  }
}

// The symbol stream of the step (cfg.symbol_stream), after both stages' k_finish_scatter: rank, superblock scan,
// [haar_dc_quant: the keyframe DC records, after the DC chain], place, the three scan kernels, pack (kInter: with the DC
// records), index.
template <bool kInter>
static void enqueue_sym(const Sym& Y, int wide, cudaStream_t s) {
  k_sym_rank<<<(Y.F * Y.nsb + 7) / 8, 256, 0, s>>>(Y);
  k_sym_sb_scan<<<1, 1024, 0, s>>>(Y);
  if (!kInter && Y.hdc) k_sym_hdc<<<(Y.F * Y.nsb * 3 + 7) / 8, 256, 0, s>>>(Y);
  k_sym_place<<<wide, 256, 0, s>>>(Y);
  k_sym_tile_sums<<<Y.ntiles, kTile, 0, s>>>(Y);
  k_sym_tile_scan<<<1, 1024, 0, s>>>(Y);
  k_sym_offsets<<<Y.ntiles, kTile, 0, s>>>(Y);
  k_sym_pack<kInter><<<wide, 256, 0, s>>>(Y);
  k_sym_index<<<1, 256, 0, s>>>(Y);
}

// config.inter: the same step for P-frame residuals.  Both plane sets through the forward transform (two
// launches: the kernel's tensor maps describe one pixel allocation each), every band of both stages through
// the phase kernels with the transformed prediction as reference.
static int kf_enqueue_step_inter(daala_b200_kf* kf, int phases) {
  cudaStream_t s = kf->stream;
  const Lists& L = kf->lists;
  const int wide = kf->sms * 8;
  if (phases & DAALA_B200_KF_LISTS) {
    k_unit_tile_sums<<<L.ntiles, kTile, 0, s>>>(L);
    k_tile_scan<<<1, 1024, 0, s>>>(L);
    k_unit_emit<<<L.ntiles, kTile, 0, s>>>(L);
    k_luma_items<<<wide, 256, 0, s>>>(L);
    k_chroma_items<<<wide, 256, 0, s>>>(L);
    if (kf->cfg.inter_mc) {
      if (cudaMemsetAsync(L.cnt + kMcBadRef, 0, 2 * sizeof(int32_t), s) != cudaSuccess) return (int)cudaGetLastError();
      int rc = daala_b200_launch_mc_leaves(&kf->mc, wide, s);
      if (rc) return rc;
    }
  }
  if (phases & DAALA_B200_KF_FORWARD) {
    int rc = kf->cfg.inter_mc ? daala_b200_launch_mc_obmc(&kf->mc, wide, s) : 0;
    if (!rc) rc = daala_b200_launch_forward(&kf->frame, 3, s);
    if (rc) return rc;
    // late_skip: the unquantised coefficients, before k_finish_scatter<true> overwrites them with the coded ones
    for (int p = 0; kf->cfg.late_skip && p < 3; p++)
      if (cudaMemcpyAsync(kf->d_orig[p], kf->coeffs[p], sizeof(int32_t) * kf->plane_w[p] * kf->plane_h[p] * kf->F,
                          cudaMemcpyDeviceToDevice, s) != cudaSuccess)
        return (int)cudaGetLastError();
    rc = daala_b200_launch_forward(&kf->frame_pred, 3, s);
    if (rc) return rc;
  }
  const bool core = (phases & DAALA_B200_KF_SEARCH_ONLY) != 0;
  for (const Stage* S : {&kf->luma, &kf->chroma}) {
    if (!(phases & (S == &kf->luma ? DAALA_B200_KF_PVQ_LUMA : DAALA_B200_KF_PVQ_CHROMA))) continue;
    if (!core) k_gather<kGatherInter><<<wide, 256, 0, s>>>(*S);
    enqueue_split(kf, *S, s);
    if (!core) k_finish_scatter<true><<<wide, 256, 0, s>>>(*S);
  }
  if (!core && (phases & DAALA_B200_KF_PVQ_CHROMA) && kf->cfg.late_skip) {
    const int rc = daala_b200_late_skip_enqueue(&kf->lsb, kf->sms * 3, s);
    if (rc) return rc;
  }
  if (!core && (phases & DAALA_B200_KF_PVQ_CHROMA) && kf->cfg.symbol_stream) enqueue_sym<true>(kf->sym, wide, s);
  if (phases & DAALA_B200_KF_INVERSE) {
    int rc = daala_b200_launch_inverse(&kf->frame, 3, s);
    if (rc) return rc;
  }
  return (int)cudaGetLastError();
}

// Keyframe work lists from the block-size maps.
static int enqueue_lists(daala_b200_kf* kf, cudaStream_t s) {
  const Lists& L = kf->lists;
  const int wide = kf->sms * 8;
  k_unit_tile_sums<<<L.ntiles, kTile, 0, s>>>(L);
  k_tile_scan<<<1, 1024, 0, s>>>(L);
  k_unit_emit<<<L.ntiles, kTile, 0, s>>>(L);
  const size_t nl = (size_t)L.max_luma * sizeof(int32_t);
  if (cudaMemsetAsync(L.succ_bottom, 0xff, nl, s) != cudaSuccess || cudaMemsetAsync(L.succ_right, 0xff, nl, s) != cudaSuccess)
    return (int)cudaGetLastError();
  if (cudaMemsetAsync(L.head_hist, 0, sizeof(int32_t) * kHeadBins, s) != cudaSuccess) return (int)cudaGetLastError();
  k_luma_deps<<<wide, 256, 0, s>>>(L);
  k_chroma_items<<<wide, 256, 0, s>>>(L);
  return 0;
}

// The luma PVQ stage up to its last band: the tickets of the stages in `begin`, gather, the chain kernel.  `core`
// (_SEARCH_ONLY, measurement): just the search kernels, on the coding-order buffers a previous full pass left behind
// (same inputs, same results).
static int enqueue_luma_bands(daala_b200_kf* kf, bool core, int begin, cudaStream_t s) {
  const int wide = kf->sms * 8;
  const int persist = kf->sms * (kf->cfg.persist_ctas_per_sm > 0 ? kf->cfg.persist_ctas_per_sm : kPersistCtas);
  if (cudaMemsetAsync(kf->luma.ring, 0xff, kf->chain_cap * sizeof(uint32_t), s) != cudaSuccess ||
      cudaMemsetAsync(kf->luma.join0, 0, (size_t)kf->luma.max_blocks * sizeof(int32_t), s) != cudaSuccess)
    return (int)cudaGetLastError();
  k_begin_pvq<<<1, 32, 0, s>>>(kf->lists.cnt, begin);
  if (!core) k_gather<kGatherLuma><<<wide, 256, 0, s>>>(kf->luma);
  k_pvq_persist<<<persist, kPersistThreads, 0, s>>>(kf->luma);
  return 0;
}

// The chroma PVQ stage: [its tickets], gather with the CfL reference (it reads the luma stage's coding-order buffers, so it needs
// the luma bands, not the luma scatter), the bands, the scatter into the coefficient planes.
static void enqueue_chroma(daala_b200_kf* kf, bool core, bool begin, cudaStream_t s) {
  const int wide = kf->sms * 8;
  const bool hdc = kf->cfg.haar_dc_quant != 0;
  if (begin) k_begin_pvq<<<1, 32, 0, s>>>(kf->lists.cnt, kBeginChroma);
  if (!core && hdc) k_gather<kGatherChroma, true><<<wide, 256, 0, s>>>(kf->chroma);
  else if (!core) k_gather<kGatherChroma><<<wide, 256, 0, s>>>(kf->chroma);
  enqueue_split(kf, kf->chroma, s);
  if (!core && hdc) k_finish_scatter<false, true><<<wide, 256, 0, s>>>(kf->chroma);
  else if (!core) k_finish_scatter<false><<<wide, 256, 0, s>>>(kf->chroma);
}

// The whole keyframe step (DAALA_B200_KF_ALL) as two branches, kf->stream and kf->side, forked and joined with
// events (captured into the step graph as parallel branches; live launches order the same way):
//   lists on kf->stream beside the forward transform on kf->side; join;
//   both stages' tickets, luma bands (the chain kernel) on kf->stream; fork;
//   kf->side: chroma stage, [symbol stream, after the luma scatter], inverse + SB postfilter of planes 1-2;
//   kf->stream: luma scatter, inverse + SB postfilter of plane 0, [level search, thresholds, od_dering of plane 0];
//   join; [od_dering of planes 1-2: they read the direction map plane 0 writes].
// haar_dc_quant: the DC chain runs on kf->side right after the forward transform, after kEvForward is recorded, so the
// luma bands do not wait for it; the chroma stage follows it by stream order and the luma scatter waits for kEvHaarDc.
// The branches write disjoint buffers; only the order of independent work differs from the phase-by-phase path.
static int kf_enqueue_step_forked(daala_b200_kf* kf) {
  cudaStream_t s = kf->stream, c = kf->side;
  const daala_b200_frame& fr = kf->cfg.dering ? kf->dering.frame : kf->frame;
  auto fork = [](cudaEvent_t e, cudaStream_t from, cudaStream_t to) {
    return cudaEventRecord(e, from) == cudaSuccess && cudaStreamWaitEvent(to, e, 0) == cudaSuccess;
  };
  if (!fork(kf->ev[kEvLists], s, c)) return (int)cudaGetLastError();
  int rc = daala_b200_launch_forward(&kf->frame_fwd, 3, c);
  if (!rc) rc = enqueue_lists(kf, s);
  if (rc) return rc;
  if (!fork(kf->ev[kEvForward], c, s)) return (int)cudaGetLastError();
  const bool hdc = kf->cfg.haar_dc_quant != 0;
  if (hdc) {
    rc = daala_b200_launch_haar_dc(&kf->hdcb, c);
    if (rc) return rc;
    if (cudaEventRecord(kf->ev[kEvHaarDc], c) != cudaSuccess) return (int)cudaGetLastError();
  }
  rc = enqueue_luma_bands(kf, false, kBeginLuma | kBeginChroma, s);
  if (rc) return rc;
  if (!fork(kf->ev[kEvLumaBands], s, c)) return (int)cudaGetLastError();
  enqueue_chroma(kf, false, false, c);
  // 16 waves of short CTAs instead of one resident wave: priority only orders CTAs that are still waiting, so a grid
  // that fits the GPU at once would hold every SM until it is done and stall the chroma gather behind it
  if (hdc) {
    if (cudaStreamWaitEvent(s, kf->ev[kEvHaarDc], 0) != cudaSuccess) return (int)cudaGetLastError();
    k_finish_scatter<false, true><<<kf->sms * 128, 256, 0, s>>>(kf->luma);
  } else {
    k_finish_scatter<false><<<kf->sms * 128, 256, 0, s>>>(kf->luma);
  }
  if (kf->cfg.symbol_stream) {
    if (!fork(kf->ev[kEvLumaScatter], s, c)) return (int)cudaGetLastError();
    enqueue_sym<false>(kf->sym, kf->sms * 8, c);
  }
  rc = enqueue_recon(fr, 1, 2, c);
  if (!rc) rc = enqueue_recon(fr, 0, 1, s);
  if (!rc && kf->cfg.dering) rc = enqueue_dering_luma(kf, kf->dering, s);
  if (rc) return rc;
  if (!fork(kf->ev[kEvChroma], c, s)) return (int)cudaGetLastError();
  for (int p = 1; kf->cfg.dering && p < 3; p++) {
    rc = enqueue_dering_plane(kf, kf->dering, p, s);
    if (rc) return rc;
  }
  return (int)cudaGetLastError();
}

// config.lossless: the whole step, one phase.  [inter_mc: leaf enumeration and OBMC, unchanged], the lossless kernels.
static int kf_enqueue_step_lossless(daala_b200_kf* kf, int phases) {
  if (phases != DAALA_B200_KF_ALL) {
    snprintf(kf->err, sizeof(kf->err), "a lossless step runs whole (DAALA_B200_KF_ALL)");
    return (int)cudaErrorInvalidValue;
  }
  cudaStream_t s = kf->stream;
  const int wide = kf->sms * 8;
  if (kf->cfg.inter_mc) {
    if (cudaMemsetAsync(kf->lists.cnt + kMcBadRef, 0, 2 * sizeof(int32_t), s) != cudaSuccess) return (int)cudaGetLastError();
    int rc = daala_b200_launch_mc_leaves(&kf->mc, wide, s);
    if (!rc) rc = daala_b200_launch_mc_obmc(&kf->mc, wide, s);
    if (rc) return rc;
  }
  return daala_b200_launch_lossless(&kf->ll, s);
}

// One step on kf->stream phase by phase (a partial phase mask: per-phase timings), or the whole step forked.
static int kf_enqueue_step(daala_b200_kf* kf, int phases) {
  if (kf->cfg.lossless) return kf_enqueue_step_lossless(kf, phases);
  if (kf->cfg.inter) return kf_enqueue_step_inter(kf, phases);
  if (phases == DAALA_B200_KF_ALL) return kf_enqueue_step_forked(kf);
  cudaStream_t s = kf->stream;
  if (phases & DAALA_B200_KF_LISTS) {
    const int rc = enqueue_lists(kf, s);
    if (rc) return rc;
  }
  if (phases & DAALA_B200_KF_FORWARD) {
    int rc = daala_b200_launch_forward(&kf->frame_fwd, 3, s);
    if (!rc && kf->cfg.haar_dc_quant) rc = daala_b200_launch_haar_dc(&kf->hdcb, s);
    if (rc) return rc;
  }
  const bool core = (phases & DAALA_B200_KF_SEARCH_ONLY) != 0;
  if (phases & DAALA_B200_KF_PVQ_LUMA) {
    const int rc = enqueue_luma_bands(kf, core, kBeginLuma, s);
    if (rc) return rc;
    if (!core && kf->cfg.haar_dc_quant) k_finish_scatter<false, true><<<kf->sms * 8, 256, 0, s>>>(kf->luma);
    else if (!core) k_finish_scatter<false><<<kf->sms * 8, 256, 0, s>>>(kf->luma);
  }
  if (phases & DAALA_B200_KF_PVQ_CHROMA) {
    enqueue_chroma(kf, core, true, s);
    if (!core && kf->cfg.symbol_stream) enqueue_sym<false>(kf->sym, kf->sms * 8, s);
  }
  if (phases & DAALA_B200_KF_INVERSE) {
    int rc = kf->cfg.dering ? enqueue_dering(kf, kf->dering, s) : daala_b200_launch_inverse(&kf->frame, 3, s);
    if (rc) return rc;
  }
  return (int)cudaGetLastError();
}

// config.inter_finish: the kernels of the finishing pass, between the H2D of the decisions / levels and the D2H of
// the results.  [symbol_stream = 2: the stream-order decisions into block order], patch and skip map, then the
// deringing pass with the real skip maps (enqueue_dering: the inverse in place on the patched plane, [inter_finish = 2:
// the level search], thresholds with the forced level 0, od_dering), [inter_mc: the store of the reconstruction into
// the pool slots of fin_slot_out].
static int kf_enqueue_finish(daala_b200_kf* kf) {
  cudaStream_t s = kf->stream;
  const int wide = kf->sms * 8;
  if (kf->fin_form) k_fin_unstream<<<wide, 256, 0, s>>>(kf->unstream);
  if (cudaMemsetAsync(kf->fin_coded, 0, (size_t)kf->F * kf->nhsb * kf->nvsb, s) != cudaSuccess)
    return (int)cudaGetLastError();
  k_fin_patch<<<wide, 256, 0, s>>>(kf->fin);
  k_fin_skip_map<<<wide, 256, 0, s>>>(kf->fin);
  const int rc = enqueue_dering(kf, kf->dering, s);
  if (rc) return rc;
  if (kf->fin_slot_out) k_fin_pool_store<<<dim3(wide > kf->F ? wide / kf->F : 1, 3 * kf->F), 256, 0, s>>>(kf->store);
  return (int)cudaGetLastError();
}

extern "C" {

// why the last daala_b200_kf_create of this thread returned NULL (daala_b200_kf_error(NULL))
static thread_local char g_create_err[256] = "null engine";

daala_b200_kf* daala_b200_kf_create(const daala_b200_kf_config* cfg) {
  snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: invalid configuration");
  if (cfg && cfg->inter_mc && (cfg->inter_mc != 1 || cfg->inter != 1)) {
    snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: inter_mc is 0 or 1, and 1 requires inter = 1");
    return nullptr;
  }
  if (cfg && cfg->mc_next && (cfg->mc_next != 1 || cfg->inter_mc != 1)) {
    snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: mc_next is 0 or 1, and 1 requires inter_mc = 1");
    return nullptr;
  }
  if (cfg && cfg->inter_finish && (cfg->inter_finish < 0 || cfg->inter_finish > 2 || cfg->inter != 1)) {
    snprintf(g_create_err, sizeof(g_create_err),
             "daala_b200_kf_create: inter_finish is 0, 1 or 2, and 1 and 2 require inter = 1");
    return nullptr;
  }
  if (cfg && (cfg->symbol_stream < 0 || cfg->symbol_stream > 2 || (cfg->symbol_stream == 2 && cfg->inter != 1))) {
    snprintf(g_create_err, sizeof(g_create_err),
             "daala_b200_kf_create: symbol_stream is 0, 1 or 2, and 2 requires inter = 1 (a keyframe's DC goes through "
             "the Haar pyramid and has no scalar index)");
    return nullptr;
  }
  if (cfg && cfg->late_skip && (cfg->late_skip != 1 || cfg->inter != 1)) {
    snprintf(g_create_err, sizeof(g_create_err),
             "daala_b200_kf_create: late_skip is 0 or 1, and 1 requires inter = 1 (keyframes have no late skip)");
    return nullptr;
  }
  if (cfg && cfg->frame_quant && (cfg->frame_quant != 1 || cfg->inter != 1)) {
    snprintf(g_create_err, sizeof(g_create_err),
             "daala_b200_kf_create: frame_quant is 0 or 1, and 1 requires inter = 1 (keyframes: keyframe_quant = 1)");
    return nullptr;
  }
  if (cfg && cfg->keyframe_quant) {
    // the kernels that read the quantizer in these modes have no per-frame form
    const char* with = cfg->keyframe_quant != 1 ? "a value other than 0 or 1"
                       : cfg->inter ? "inter (P and B frames take their records with frame_quant = 1)"
                       : cfg->lossless ? "lossless (every frame is at quantizer 0)"
                       : cfg->sb_rows > 0 ? "a row shard (sb_rows > 0)" : nullptr;
    if (with) {
      snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: keyframe_quant is not defined with %s", with);
      return nullptr;
    }
  }
  if (cfg && cfg->lossless) {
    // the lossless path has no PVQ, no deringing and no coder-side state: none of these stages exists for it
    const char* with = cfg->lossless != 1 ? "a value other than 0 or 1"
                       : cfg->dering ? "dering (lossless frames skip deringing)"
                       : cfg->symbol_stream ? "symbol_stream (the stream is the PVQ symbols)"
                       : cfg->late_skip ? "late_skip"
                       : cfg->inter_finish ? "inter_finish"
                       : cfg->frame_quant ? "frame_quant (every frame is at quantizer 0)"
                       : cfg->sb_rows > 0 ? "a row shard (sb_rows > 0)" : nullptr;
    if (with) {
      snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: lossless is not defined with %s", with);
      return nullptr;
    }
  }
  if (cfg && cfg->haar_dc_quant) {
    // the chain quantises the Haar DC pyramid of lossy keyframes; the superblock predictor reads the superblocks above,
    // across any row shard
    const char* with = cfg->haar_dc_quant != 1 ? "a value other than 0 or 1"
                       : cfg->inter ? "inter (P and B frames code a scalar DC per block)"
                       : cfg->lossless ? "lossless (its keyframe DCs are coded exactly)"
                       : cfg->sb_rows > 0 ? "a row shard (sb_rows > 0)" : nullptr;
    if (with) {
      snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: haar_dc_quant is not defined with %s", with);
      return nullptr;
    }
  }
  if (cfg && !cfg->lossless && (cfg->q0 < 1 || cfg->q0 > DAALA_B200_KF_MAX_Q0)) {
    // the records made from the config follow the records' rule (quantizer 0 is the lossless engine's)
    snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: q0 is outside [1, %d] (lossless = 1 codes quantizer 0)",
             DAALA_B200_KF_MAX_Q0);
    return nullptr;
  }
  if (cfg && cfg->mc_refs < 0) {
    snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: mc_refs < 0");
    return nullptr;
  }
  if (cfg && cfg->inter) {
    // P-frame residual mode is defined for whole frames through the phase kernels, without the stages whose
    // inter form this engine does not have
    const char* with = cfg->inter != 1 ? "a value other than 0 or 1"
                       : cfg->dering ? "dering (the all-zero skip map of the deringing stage is a keyframe property)"
                       : cfg->symbol_stream == 1 ? "symbol_stream = 1 (its block record has no DC field; "
                                                   "symbol_stream = 2 is the P-frame stream)"
                       : cfg->sb_rows > 0 ? "a row shard (sb_rows > 0)" : nullptr;
    if (with) {
      snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: inter is not defined with %s", with);
      return nullptr;
    }
  }
  if (!cfg || cfg->pic_w <= 0 || cfg->pic_h <= 0 || cfg->nframes <= 0 || cfg->nframes > 255 || !cfg->qm ||
      !cfg->qm_inv || cfg->qm_stride <= 0)
    return nullptr;
  daala_b200_kf* kf = new (std::nothrow) daala_b200_kf();   // value-initialised: every field zero
  if (!kf) return nullptr;
  kf->cfg = *cfg;
  kf->nhsb = (cfg->pic_w + 63) / 64;
  kf->nvsb = (cfg->pic_h + 63) / 64;
  kf->F = cfg->nframes;
  if (kf->cfg.inter_mc && kf->cfg.mc_refs == 0) kf->cfg.mc_refs = (kf->cfg.mc_next ? 3 : 2) * kf->F;
  if (!kf->cfg.inter_mc) kf->cfg.mc_refs = 0;
  kf->slot_filled.assign((size_t)kf->cfg.mc_refs, 0);
  if (kf->cfg.sb_rows <= 0) {
    kf->cfg.sb_row0 = 0;
    kf->cfg.sb_rows = kf->nvsb;
  }
  for (int p = 0; p < 3; p++) {
    kf->plane_w[p] = (kf->nhsb * 64) >> (p ? 1 : 0);
    kf->plane_h[p] = (kf->nvsb * 64) >> (p ? 1 : 0);
  }
  // coefficient offsets are 32-bit (ADVICE r1): the whole batch must stay below 2^31 coded coefficients
  if ((long long)kf->plane_w[0] * kf->plane_h[0] * kf->F >= (1ll << 31)) {
    delete kf;
    return nullptr;
  }
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    delete kf;
    return nullptr;
  }
  kf->sms = prop.multiProcessorCount;
  if (cfg->stream) {
    kf->stream = (cudaStream_t)cfg->stream;
  } else {
    if (cudaStreamCreateWithFlags(&kf->stream, cudaStreamNonBlocking) != cudaSuccess) {
      delete kf;
      return nullptr;
    }
    kf->own_stream = true;
  }
  if (!cfg->inter && !cfg->lossless) {
    // the side branch carries the longer chain (the chroma stage) at the highest priority: the luma branch's CTAs
    // then take the SMs the chroma kernels leave idle instead of delaying them
    int least = 0, greatest = 0;
    bool ok = cudaDeviceGetStreamPriorityRange(&least, &greatest) == cudaSuccess &&
              cudaStreamCreateWithPriority(&kf->side, cudaStreamNonBlocking, greatest) == cudaSuccess;
    for (int i = 0; ok && i < kNumEvents; i++) ok = cudaEventCreateWithFlags(&kf->ev[i], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) {
      snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: cannot create the second stream and its events");
      daala_b200_kf_destroy(kf);
      return nullptr;
    }
  }
  if (kf_alloc(kf) != 0) {
    fprintf(stderr, "daala_b200_kf_create: %s\n", kf->err);
    snprintf(g_create_err, sizeof(g_create_err), "daala_b200_kf_create: %s", kf->err);
    // leak-free teardown is the destroy function's job
    daala_b200_kf_destroy(kf);
    return nullptr;
  }
  return kf;
}

void daala_b200_kf_destroy(daala_b200_kf* kf) {
  if (!kf) return;
  cudaStreamSynchronize(kf->stream);
  if (kf->exec) cudaGraphExecDestroy(kf->exec);
  if (kf->graph) cudaGraphDestroy(kf->graph);
  if (kf->fin_exec) cudaGraphExecDestroy(kf->fin_exec);
  if (kf->fin_graph) cudaGraphDestroy(kf->fin_graph);
  for (void* p : kf->allocs) cudaFree(p);
  for (cudaEvent_t e : kf->ev)
    if (e) cudaEventDestroy(e);
  if (kf->side) cudaStreamDestroy(kf->side);
  if (kf->own_stream) cudaStreamDestroy(kf->stream);
  delete kf;
}

const char* daala_b200_kf_error(const daala_b200_kf* kf) { return kf ? kf->err : g_create_err; }

#ifdef DAALA_B200_CHAIN_TRACE
// tools/chain_timeline.py: the luma chain kernel's trace records (device) and their capacity; the count written by
// the last luma stage is counts[kTraceN]
int daala_b200_kf_chain_trace(daala_b200_kf* kf, void** recs, int* cap) {
  if (!kf || !recs || !cap) return (int)cudaErrorInvalidValue;
  *recs = kf->luma.trace;
  *cap = kf->luma.trace_cap;
  return 0;
}
#endif

// Kernel launches of one whole step (kf_enqueue_step with DAALA_B200_KF_ALL), memset nodes not counted.
int daala_b200_kf_launches_per_step(const daala_b200_kf* kf) {
  if (!kf) return 0;
  // lossless: [leaves + OBMC], the forward kernel, [keyframes: the DC + reconstruction kernel]
  if (kf->cfg.lossless) return (kf->cfg.inter_mc ? 2 : 0) + (kf->cfg.inter ? 1 : 2);
  auto split = [](const Stage& S) { return 3 * (S.sp_chunks[0] + S.sp_chunks[1] + S.sp_chunks[2]); };
  // inter: work lists, two forward launches, per stage gather + phase kernels + finish, inverse + SB postfilter;
  // inter_mc: leaf enumeration and OBMC
  // [symbol_stream = 2: the 8 stream kernels]; [late_skip: the size-class split and one launch per class]
  if (kf->cfg.inter)
    return 5 + 2 + (2 + split(kf->luma)) + (2 + split(kf->chroma)) + 2 + (kf->cfg.inter_mc ? 2 : 0) +
           (kf->cfg.symbol_stream ? 8 : 0) + (kf->cfg.late_skip ? kLateSkipLaunches : 0);
  int n = 5;                                                                      // work lists
  n += 1 + (kf->cfg.haar_dc_quant ? 1 : 0);                                       // forward, [DC chain]
  n += 3 + 1;                                                                     // luma: begin (both stages), gather, chains, finish
  n += 2 + split(kf->chroma);                                                     // chroma: gather, phase kernels, finish
  // inverse + SB postfilter of plane 0 and of planes 1-2, [the rest of the deringing pass]
  n += kf->cfg.dering ? dering_launches(kf->dering, 2) : 4;
  // symbol stream: rank, superblock scan, [haar_dc_quant: DC records], place, 3 scan kernels, pack, index
  if (kf->cfg.symbol_stream) n += 8 + (kf->cfg.haar_dc_quant ? 1 : 0);
  return n;
}

int daala_b200_kf_device_buffers(daala_b200_kf* kf, daala_b200_kf_buffers* out) {
  if (!kf || !out) return (int)cudaErrorInvalidValue;
  memset(out, 0, sizeof(*out));
  for (int p = 0; p < 3; p++) {
    out->pixels[p] = kf->pixels[p];
    out->coeffs[p] = kf->coeffs[p];
    out->lapped[p] = kf->lapped[p];
    out->pixels_out[p] = kf->pixels_out[p];
    out->plane_w[p] = kf->plane_w[p];
    out->plane_h[p] = kf->plane_h[p];
  }
  out->bsize = kf->bsize;
  out->counts = kf->lists.cnt;
  out->luma_blocks = kf->lists.luma;
  out->chroma_blocks = kf->lists.chroma;
  out->dep_top = kf->lists.dep_top;
  out->dep_left = kf->lists.dep_left;
  for (int c = 0; c < 3; c++) {
    out->luma_items[c] = kf->lists.items_l[c];
    out->chroma_items[c] = kf->lists.items_c[c];
  }
  out->luma_heads = kf->lists.heads;
  out->luma_heads0 = kf->lists.heads0;
  out->luma_heads_raw = kf->lists.heads_raw;
  out->luma_head_bin = kf->lists.head_bin;
  out->succ_bottom = kf->lists.succ_bottom;
  out->succ_right = kf->lists.succ_right;
  out->luma_res = kf->luma.res_pack;
  out->chroma_res = kf->chroma.res_pack;
  out->luma_y16 = kf->luma.prm.y16;
  out->chroma_y16 = kf->chroma.prm.y16;
  out->luma_skip_diff = kf->luma.prm.res_skip_diff;
  out->chroma_skip_diff = kf->chroma.prm.res_skip_diff;
  out->chroma_flip = kf->chroma.prm.res_flip;
  out->max_luma_blocks = kf->lists.max_luma;
  out->max_chroma_blocks = kf->lists.max_chroma;
  out->stream = kf->stream;
  out->bytes_allocated = (long long)kf->bytes_allocated;
  for (int p = 0; p < 3; p++) {
    out->pred_pixels[p] = kf->pred_pixels[p];
    out->pred_coeffs[p] = kf->pred_coeffs[p];
    out->ref_pixels[p] = kf->ref_pixels[p];
  }
  out->ref_slot = kf->ref_slot;
  out->mv_grid = kf->mv_grid;
  out->mc_refs = kf->cfg.mc_refs;
  out->ref_slot_next = kf->ref_slot_next;
  out->mv1_grid = kf->mv1_grid;
  out->frame_quant = kf->cfg.frame_quant || kf->cfg.keyframe_quant ? kf->fq : nullptr;
  for (int p = 0; p < 3; p++) {
    out->haar_dc[p] = kf->hdcb.dc[p];
    out->dc_index[p] = kf->hdc_index[p];
  }
  out->sym_hdc = kf->sym.hdc;
  return 0;
}

int daala_b200_kf_run_device(daala_b200_kf* kf, int phases, int use_graph) {
  if (!kf) return (int)cudaErrorInvalidValue;
  if (!use_graph || phases != DAALA_B200_KF_ALL) return kf_enqueue_step(kf, phases);
  if (!kf->captured) {
    // warm-up outside the capture: module loading and the TMA descriptor encode are not capturable
    int rc = kf_enqueue_step(kf, phases);
    if (rc) return rc;
    KF_CHECK(cudaStreamSynchronize(kf->stream));
    KF_CHECK(cudaStreamBeginCapture(kf->stream, cudaStreamCaptureModeThreadLocal));
    rc = kf_enqueue_step(kf, phases);
    cudaError_t e = cudaStreamEndCapture(kf->stream, &kf->graph);
    if (rc) return rc;
    KF_CHECK(e);
    // the captured nodes keep their stream's priority (kf->side's branch first)
    KF_CHECK(cudaGraphInstantiate(&kf->exec, kf->graph, cudaGraphInstantiateFlagUseNodePriority));
    kf->captured = true;
  }
  KF_CHECK(cudaGraphLaunch(kf->exec, kf->stream));
  return 0;
}

// `reps` repetitions of the selected phases timed with CUDA events on the engine's stream (inputs
// resident in HBM); returns the total in milliseconds.
int daala_b200_kf_time_device(daala_b200_kf* kf, int phases, int use_graph, int reps, float* ms) {
  if (!kf || !ms || reps <= 0) return (int)cudaErrorInvalidValue;
  cudaEvent_t e0, e1;
  KF_CHECK(cudaEventCreate(&e0));
  KF_CHECK(cudaEventCreate(&e1));
  if (use_graph && phases == DAALA_B200_KF_ALL && !kf->captured) {
    int rc = daala_b200_kf_run_device(kf, phases, 1);
    if (rc) return rc;
  }
  KF_CHECK(cudaStreamSynchronize(kf->stream));
  KF_CHECK(cudaEventRecord(e0, kf->stream));
  for (int i = 0; i < reps; i++) {
    int rc = daala_b200_kf_run_device(kf, phases, use_graph);
    if (rc) return rc;
  }
  KF_CHECK(cudaEventRecord(e1, kf->stream));
  KF_CHECK(cudaEventSynchronize(e1));
  KF_CHECK(cudaEventElapsedTime(ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 0;
}

// Totals that follow from the block-size maps (what the host needs to size its result buffers):
// the same leaf rule as unit_counts above, on the host.
int daala_b200_kf_count_blocks(const uint8_t* bsize, int nframes, long long frame_pitch, int bstride, int nhsb,
                               int nvsb, int sb_row0, int sb_rows, daala_b200_kf_totals* out) {
  if (!bsize || !out) return (int)cudaErrorInvalidValue;
  long long nl = 0, cl = 0, nc = 0, cc = 0;
  if (sb_rows <= 0) { sb_row0 = 0; sb_rows = nvsb; }
  for (int f = 0; f < nframes; f++) {
    for (int uy = sb_row0 * 8; uy < (sb_row0 + sb_rows) * 8; uy++) {
      const uint8_t* row = bsize + f * frame_pitch + (long long)uy * bstride;
      for (int ux = 0; ux < nhsb * 8; ux++) {
        const int b = row[ux];
        if (b == 0) { nl += 4; cl += 64; nc += 1; cc += 16; continue; }
        const int span = 1 << (b - 1);
        if ((ux & (span - 1)) | (uy & (span - 1))) continue;
        nl += 1;
        cl += b == 1 ? 64 : b == 2 ? 256 : 512;
        nc += 1;
        cc += b == 1 ? 16 : b == 2 ? 64 : b == 3 ? 256 : 512;
      }
    }
  }
  out->n_luma = nl;
  out->luma_coefs = cl;
  out->n_chroma = 2 * nc;
  out->chroma_coefs = 2 * cc;
  return 0;
}

// Worst-case lengths of the symbol stream arrays for a batch with the given totals: every block, every band
// (9 per block, and never more than one per 16 coefficients: 4x4 and 8x8 blocks have exactly that many, larger
// ones fewer), two bytes per coded coefficient.
int daala_b200_kf_symbol_bounds(const daala_b200_kf_totals* t, int nframes, daala_b200_kf_sym_bounds* out) {
  if (!t || !out || nframes <= 0) return (int)cudaErrorInvalidValue;
  const long long blocks = t->n_luma + t->n_chroma, coefs = t->luma_coefs + t->chroma_coefs;
  out->index = nframes;
  out->blocks = blocks;
  out->bands = 9 * blocks < coefs / 16 ? 9 * blocks : coefs / 16;
  out->pulse_bytes = 2 * coefs;
  return 0;
}

// A requested stream buffer: large enough, and pinned host memory the device can write (its device address).
static int sym_target(const void* p, long long cap, long long need, uint8_t** dev) {
  *dev = nullptr;
  if (!p) return 0;
  if (cap < need) return (int)cudaErrorInvalidValue;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return (int)cudaErrorInvalidValue;
  }
  if (a.type != cudaMemoryTypeHost || !a.devicePointer) return (int)cudaErrorInvalidValue;
  *dev = (uint8_t*)a.devicePointer;
  return 0;
}

int daala_b200_kf_load_frame_quant(daala_b200_kf* kf, const daala_b200_kf_frame_quant* rec) {
  if (!kf) return (int)cudaErrorInvalidValue;
  int dc_limit = 0;
  const char* why = !kf->cfg.frame_quant && !kf->cfg.keyframe_quant
                        ? "needs an engine with frame_quant = 1 or keyframe_quant = 1"
                        : fq_derive_host(kf, rec, true, &dc_limit);
  if (why) {
    snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_load_frame_quant: %s", why);
    return (int)cudaErrorInvalidValue;
  }
  KF_CHECK(fq_copy(kf, rec, kf->stream));
  KF_CHECK(cudaStreamSynchronize(kf->stream));   // the host tables are reused by the next call
  return 0;
}

int daala_b200_kf_submit(daala_b200_kf* kf, const daala_b200_kf_io* io) {
  if (!kf || !io) return (int)cudaErrorInvalidValue;
  cudaStream_t s = kf->stream;
  const int F = kf->F;
  const bool lossless = kf->cfg.lossless != 0;
  if (!io->bsize && !lossless) return (int)cudaErrorInvalidValue;
  // refuse a batch with more blocks than the work lists hold before anything is copied or launched: the
  // step would otherwise run on truncated lists (a lossless step has no block lists)
  daala_b200_kf_totals tot;
  memset(&tot, 0, sizeof(tot));
  if (lossless) {
  } else if (io->totals) {
    tot = *io->totals;
  } else {
    daala_b200_kf_count_blocks(io->bsize, F, (long long)kf->nhsb * 8 * kf->nvsb * 8, kf->nhsb * 8, kf->nhsb, kf->nvsb,
                               kf->cfg.sb_row0, kf->cfg.sb_rows, &tot);
  }
  if (tot.n_luma > kf->lists.max_luma || tot.n_chroma > kf->lists.max_chroma) return (int)cudaErrorInvalidValue;
  const bool have_pred = io->pred_pixels[0] || io->pred_pixels[1] || io->pred_pixels[2];
  // symbol_stream = 2: the stream's DC records carry the DC indices, so the classic arrays are optional; a lossless
  // step has no scalar DC index
  const bool need_dc = !lossless && kf->cfg.symbol_stream != 2 && (!io->luma_dc || !io->chroma_dc);
  // the lossless outputs: only a lossless engine has them, and only one with the pool stores into it
  const bool want_ll = io->ll_coeffs[0] || io->ll_coeffs[1] || io->ll_coeffs[2] || io->ll_blocks;
  const char* ll_why = (want_ll || io->ll_ref_slot_out) && !lossless
                           ? "ll_coeffs / ll_blocks / ll_ref_slot_out need an engine with lossless = 1"
                       : io->ll_ref_slot_out && !kf->cfg.inter_mc
                           ? "ll_ref_slot_out needs an engine with inter_mc (the reference-picture pool)"
                           : nullptr;
  for (int f = 0; !ll_why && io->ll_ref_slot_out && f < F; f++) {
    const int32_t r = io->ll_ref_slot_out[f];
    if (r < -1 || r >= kf->cfg.mc_refs) ll_why = "an ll_ref_slot_out entry is outside [-1, mc_refs)";
    for (int g = 0; !ll_why && r >= 0 && g < f; g++)
      if (io->ll_ref_slot_out[g] == r) ll_why = "two frames name the same ll_ref_slot_out slot";
  }
  if (ll_why) {
    snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_submit: %s", ll_why);
    return (int)cudaErrorInvalidValue;
  }
  if ((io->dc_index[0] || io->dc_index[1] || io->dc_index[2]) && !kf->cfg.haar_dc_quant) {
    snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_submit: dc_index needs an engine with haar_dc_quant = 1");
    return (int)cudaErrorInvalidValue;
  }
  if (kf->cfg.inter && !kf->cfg.inter_mc &&
      (!io->pred_pixels[0] || !io->pred_pixels[1] || !io->pred_pixels[2] || need_dc)) {
    snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_submit: an inter engine needs pred_pixels[0..2], luma_dc and chroma_dc");
    return (int)cudaErrorInvalidValue;
  }
  if ((io->ref_slot_next || io->mv1_grid) && !kf->cfg.mc_next) {
    snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_submit: ref_slot_next and mv1_grid need an engine with mc_next");
    return (int)cudaErrorInvalidValue;
  }
  if (io->ref_resident && !kf->cfg.inter_mc) {
    snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_submit: ref_resident needs an engine with inter_mc");
    return (int)cudaErrorInvalidValue;
  }
  if (kf->cfg.inter_mc) {
    const bool resident = io->ref_resident != 0;
    const bool any_ref = io->ref_pixels[0] || io->ref_pixels[1] || io->ref_pixels[2];
    const char* why = need_dc ? "luma_dc and chroma_dc are required"
                      : !io->mv_grid ? "mv_grid is required"
                      : io->ref_resident != 0 && io->ref_resident != 1 ? "ref_resident is 0 or 1"
                      : resident && any_ref ? "ref_resident: ref_pixels must be NULL (the step reads the pool as it stands)"
                      : resident && io->nrefs != 0 ? "ref_resident: nrefs must be 0"
                      : !resident && (!io->ref_pixels[0] || !io->ref_pixels[1] || !io->ref_pixels[2])
                          ? "ref_pixels[0..2] are required"
                      : !io->ref_slot ? "ref_slot is required"
                      : kf->cfg.mc_next && !io->ref_slot_next ? "mc_next: ref_slot_next is required"
                      : kf->cfg.mc_next && !io->mv1_grid ? "mc_next: mv1_grid is required"
                      : have_pred ? "pred_pixels is refused: the engine makes the prediction"
                      : !resident && (io->nrefs < 1 || io->nrefs > kf->cfg.mc_refs) ? "nrefs is outside [1, mc_refs]"
                                                                                    : nullptr;
    // the GOLD / PREV slots, then (mc_next) the NEXT slots
    const int nslot = (kf->cfg.mc_next ? 3 : 2) * F;
    bool in_next = false;
    for (int i = 0; !why && i < nslot; i++) {
      const int32_t r = i < 2 * F ? io->ref_slot[i] : io->ref_slot_next[i - 2 * F];
      in_next = i >= 2 * F;
      if (!resident && (r < 0 || r >= io->nrefs)) why = "a ref_slot entry is outside [0, nrefs)";
      else if (resident && (r < 0 || r >= kf->cfg.mc_refs)) why = "ref_resident: a ref_slot entry is outside [0, mc_refs)";
      else if (resident && !kf->slot_filled[r])
        why = "ref_resident: a ref_slot entry names a pool slot that holds no picture (pool_load, a host-upload "
              "submit or a finish with ref_slot_out writes one)";
    }
    if (why) {
      snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_submit: inter_mc: %s%s", why, in_next ? " (ref_slot_next)" : "");
      return (int)cudaErrorInvalidValue;
    }
  }
  // late-skip records: only an engine with late_skip has them, and only a symbol_stream = 2 engine in stream order
  const char* ls_why = (io->luma_late_skip || io->chroma_late_skip || io->sym_late_skip) && !kf->cfg.late_skip
                           ? "luma_late_skip / chroma_late_skip / sym_late_skip need an engine with late_skip = 1"
                       : io->sym_late_skip && kf->cfg.symbol_stream != 2
                           ? "sym_late_skip needs an engine with symbol_stream = 2"
                           : nullptr;
  if (ls_why) {
    snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_submit: %s", ls_why);
    return (int)cudaErrorInvalidValue;
  }
  // per-frame quantizers: every record in range; then each frame's deringing thresholds and band quantisers and the
  // finishing pass's DC limit of this step
  int fq_dc_limit = 0;
  const bool fq_mode = kf->cfg.frame_quant || kf->cfg.keyframe_quant;
  if (io->frame_quant || fq_mode) {
    const char* why = !fq_mode ? "frame_quant needs an engine with frame_quant = 1 or keyframe_quant = 1"
                               : fq_derive_host(kf, io->frame_quant, true, &fq_dc_limit);
    if (why) {
      snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_submit: %s", why);
      return (int)cudaErrorInvalidValue;
    }
  }
  // symbol stream: the engine must produce it, and every requested buffer must hold the worst case and be pinned
  SymCopy sc;
  memset(&sc, 0, sizeof(sc));
  const bool want_sym = io->sym_index || io->sym_blocks || io->sym_bands || io->sym_pulses || io->sym_dc ||
                        io->sym_late_skip || io->sym_hdc;
  if (want_sym) {
    if (io->sym_hdc && !(kf->cfg.symbol_stream == 1 && kf->cfg.haar_dc_quant)) {
      snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_submit: sym_hdc needs an engine with symbol_stream = 1 and haar_dc_quant = 1");
      return (int)cudaErrorInvalidValue;
    }
    if (!kf->cfg.symbol_stream) return (int)cudaErrorInvalidValue;
    if (io->sym_dc && kf->cfg.symbol_stream != 2) {
      snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_submit: sym_dc needs an engine with symbol_stream = 2");
      return (int)cudaErrorInvalidValue;
    }
    daala_b200_kf_sym_bounds bd;
    daala_b200_kf_symbol_bounds(&tot, F, &bd);
    int e = sym_target(io->sym_index, io->sym_index_cap, bd.index, &sc.dst[0]);
    if (!e) e = sym_target(io->sym_blocks, io->sym_blocks_cap, bd.blocks, &sc.dst[1]);
    if (!e) e = sym_target(io->sym_bands, io->sym_bands_cap, bd.bands, &sc.dst[2]);
    if (!e) e = sym_target(io->sym_pulses, io->sym_pulses_cap, bd.pulse_bytes, &sc.dst[3]);
    if (!e) e = sym_target(io->sym_dc, io->sym_dc_cap, bd.blocks, &sc.dst[4]);
    if (e) return e;
    if (sym_target(io->sym_late_skip, io->sym_late_skip_cap, bd.blocks, &sc.dst[5])) {
      snprintf(kf->err, sizeof(kf->err),
               "daala_b200_kf_submit: sym_late_skip must be pinned host memory of at least "
               "daala_b200_kf_symbol_bounds(...).blocks records");
      return (int)cudaErrorInvalidValue;
    }
    if (sym_target(io->sym_hdc, io->sym_hdc_cap, bd.blocks, &sc.dst[6])) {
      snprintf(kf->err, sizeof(kf->err),
               "daala_b200_kf_submit: sym_hdc must be pinned host memory of at least "
               "daala_b200_kf_symbol_bounds(...).blocks records");
      return (int)cudaErrorInvalidValue;
    }
    const Sym& Y = kf->sym;
    sc.src[0] = (const uint8_t*)Y.index;
    sc.src[1] = (const uint8_t*)Y.blocks;
    sc.src[2] = (const uint8_t*)Y.bands;
    sc.src[3] = Y.pulses;
    sc.src[4] = (const uint8_t*)Y.dc;
    sc.src[5] = (const uint8_t*)Y.late_skip;
    sc.src[6] = (const uint8_t*)Y.hdc;
    sc.unit[1] = sizeof(daala_b200_kf_sym_block);
    sc.unit[2] = 4 * sizeof(int16_t);
    sc.unit[3] = 1;
    sc.unit[4] = sizeof(daala_b200_kf_sym_dc);
    sc.unit[5] = sizeof(daala_b200_kf_late_skip);
    sc.unit[6] = sizeof(daala_b200_kf_sym_hdc);
    sc.index_bytes = (long long)F * sizeof(daala_b200_kf_sym_frame);
    sc.tot = Y.tot;
    const long long host[kSymSegs] = {io->sym_index_cap * (long long)sizeof(daala_b200_kf_sym_frame),
                                      io->sym_blocks_cap * (long long)sizeof(daala_b200_kf_sym_block),
                                      io->sym_bands_cap * 8, io->sym_pulses_cap,
                                      io->sym_dc_cap * (long long)sizeof(daala_b200_kf_sym_dc),
                                      io->sym_late_skip_cap * (long long)sizeof(daala_b200_kf_late_skip),
                                      io->sym_hdc_cap * (long long)sizeof(daala_b200_kf_sym_hdc)};
    const long long dev[kSymSegs] = {sc.index_bytes, (long long)Y.cap_blocks * (long long)sizeof(daala_b200_kf_sym_block),
                                     Y.cap_bands * 8, Y.cap_bytes,
                                     Y.dc ? (long long)Y.cap_blocks * (long long)sizeof(daala_b200_kf_sym_dc) : 0,
                                     Y.late_skip ? (long long)Y.cap_blocks * (long long)sizeof(daala_b200_kf_late_skip) : 0,
                                     Y.hdc ? (long long)Y.cap_blocks * (long long)sizeof(daala_b200_kf_sym_hdc) : 0};
    for (int i = 0; i < kSymSegs; i++) sc.cap[i] = host[i] < dev[i] ? host[i] : dev[i];
  }
  for (int p = 0; p < 3; p++) {
    if (!io->pixels[p]) return (int)cudaErrorInvalidValue;
    KF_CHECK(cudaMemcpyAsync(kf->pixels[p], io->pixels[p], (size_t)kf->plane_w[p] * kf->plane_h[p] * F,
                             cudaMemcpyHostToDevice, s));
    if (kf->cfg.inter_mc) {
      if (!io->ref_resident)
        KF_CHECK(cudaMemcpyAsync(kf->ref_pixels[p], io->ref_pixels[p],
                                 (size_t)kf->plane_w[p] * kf->plane_h[p] * io->nrefs, cudaMemcpyHostToDevice, s));
    } else if (kf->cfg.inter)
      KF_CHECK(cudaMemcpyAsync(kf->pred_pixels[p], io->pred_pixels[p], (size_t)kf->plane_w[p] * kf->plane_h[p] * F,
                               cudaMemcpyHostToDevice, s));
  }
  if (kf->cfg.inter_mc) {
    if (!io->ref_resident) std::fill(kf->slot_filled.begin(), kf->slot_filled.begin() + io->nrefs, 1);
    KF_CHECK(cudaMemcpyAsync(kf->ref_slot, io->ref_slot, sizeof(int32_t) * 2 * F, cudaMemcpyHostToDevice, s));
    KF_CHECK(cudaMemcpyAsync(kf->mv_grid, io->mv_grid,
                             sizeof(daala_b200_mv_pt) * F * (kf->nvsb * 8 + 1) * (kf->nhsb * 8 + 1),
                             cudaMemcpyHostToDevice, s));
    if (kf->cfg.mc_next) {
      KF_CHECK(cudaMemcpyAsync(kf->ref_slot_next, io->ref_slot_next, sizeof(int32_t) * F, cudaMemcpyHostToDevice, s));
      KF_CHECK(cudaMemcpyAsync(kf->mv1_grid, io->mv1_grid,
                               sizeof(int32_t) * 2 * F * (kf->nvsb * 8 + 1) * (kf->nhsb * 8 + 1),
                               cudaMemcpyHostToDevice, s));
    }
  }
  if (fq_mode) KF_CHECK(fq_copy(kf, io->frame_quant, s));
  const size_t map_bytes = (size_t)kf->nhsb * 8 * kf->nvsb * 8 * F;
  if (!lossless) KF_CHECK(cudaMemcpyAsync(kf->bsize, io->bsize, map_bytes, cudaMemcpyHostToDevice, s));
  // the graph's lossless kernels read the slot table: NULL stores nothing (every entry -1)
  if (io->ll_ref_slot_out) KF_CHECK(cudaMemcpyAsync(kf->ll_slot_out, io->ll_ref_slot_out, 4 * (size_t)F, cudaMemcpyHostToDevice, s));
  else if (kf->ll_slot_out) KF_CHECK(cudaMemsetAsync(kf->ll_slot_out, 0xFF, 4 * (size_t)F, s));
  if (kf->cfg.dering == 1) {
    if (!io->dering_level) return (int)cudaErrorInvalidValue;
    KF_CHECK(cudaMemcpyAsync(kf->dering.level, io->dering_level, (size_t)kf->nhsb * kf->nvsb * F, cudaMemcpyHostToDevice, s));
  }
  const int rc = daala_b200_kf_run_device(kf, DAALA_B200_KF_ALL, 1);
  if (rc) return rc;
  kf->have_step = true;
  kf->last_tot = tot;
  if (fq_mode) kf->fin_dc_limit = fq_dc_limit;
  for (int p = 0; p < 3; p++)
    if (io->pixels_out[p])
      KF_CHECK(cudaMemcpyAsync(io->pixels_out[p], kf->pixels_out[p], (size_t)kf->plane_w[p] * kf->plane_h[p] * F,
                               cudaMemcpyDeviceToHost, s));
  if (lossless) {
    for (int f = 0; io->ll_ref_slot_out && f < F; f++)
      if (io->ll_ref_slot_out[f] >= 0) kf->slot_filled[io->ll_ref_slot_out[f]] = 1;
    for (int p = 0; p < 3; p++) {
      const size_t n = (size_t)kf->plane_w[p] * kf->plane_h[p] * F;
      if (io->ll_coeffs[p]) KF_CHECK(cudaMemcpyAsync(io->ll_coeffs[p], kf->ll_coeffs[p], 2 * n, cudaMemcpyDeviceToHost, s));
      if (kf->cfg.inter_mc && io->pred_pixels_out[p])
        KF_CHECK(cudaMemcpyAsync(io->pred_pixels_out[p], kf->pred_pixels[p], n, cudaMemcpyDeviceToHost, s));
    }
    if (io->ll_blocks)
      KF_CHECK(cudaMemcpyAsync(io->ll_blocks, kf->ll_blocks, sizeof(daala_b200_kf_ll_block) * F * kf->nhsb * kf->nvsb * 3,
                               cudaMemcpyDeviceToHost, s));
    if (io->counts) KF_CHECK(cudaMemcpyAsync(io->counts, kf->lists.cnt, sizeof(int32_t) * 32, cudaMemcpyDeviceToHost, s));
    return 0;
  }
  if (io->luma_blocks) KF_CHECK(cudaMemcpyAsync(io->luma_blocks, kf->lists.luma, sizeof(daala_b200_pvq_block) * tot.n_luma, cudaMemcpyDeviceToHost, s));
  if (io->chroma_blocks) KF_CHECK(cudaMemcpyAsync(io->chroma_blocks, kf->lists.chroma, sizeof(daala_b200_pvq_block) * tot.n_chroma, cudaMemcpyDeviceToHost, s));
  if (io->luma_res) KF_CHECK(cudaMemcpyAsync(io->luma_res, kf->luma.res_pack, 8 * 9 * (size_t)tot.n_luma, cudaMemcpyDeviceToHost, s));
  if (io->chroma_res) KF_CHECK(cudaMemcpyAsync(io->chroma_res, kf->chroma.res_pack, 8 * 9 * (size_t)tot.n_chroma, cudaMemcpyDeviceToHost, s));
  if (io->luma_y16) KF_CHECK(cudaMemcpyAsync(io->luma_y16, kf->luma.prm.y16, 2 * (size_t)tot.luma_coefs, cudaMemcpyDeviceToHost, s));
  if (io->chroma_y16) KF_CHECK(cudaMemcpyAsync(io->chroma_y16, kf->chroma.prm.y16, 2 * (size_t)tot.chroma_coefs, cudaMemcpyDeviceToHost, s));
  if (io->luma_skip_diff) KF_CHECK(cudaMemcpyAsync(io->luma_skip_diff, kf->luma.prm.res_skip_diff, 8 * (size_t)tot.n_luma, cudaMemcpyDeviceToHost, s));
  if (io->chroma_skip_diff) KF_CHECK(cudaMemcpyAsync(io->chroma_skip_diff, kf->chroma.prm.res_skip_diff, 8 * (size_t)tot.n_chroma, cudaMemcpyDeviceToHost, s));
  if (io->chroma_flip) KF_CHECK(cudaMemcpyAsync(io->chroma_flip, kf->chroma.prm.res_flip, 4 * (size_t)tot.n_chroma, cudaMemcpyDeviceToHost, s));
  for (int p = 0; p < 3; p++)
    if (kf->cfg.inter_mc && io->pred_pixels_out[p])
      KF_CHECK(cudaMemcpyAsync(io->pred_pixels_out[p], kf->pred_pixels[p], (size_t)kf->plane_w[p] * kf->plane_h[p] * F,
                               cudaMemcpyDeviceToHost, s));
  if (kf->cfg.inter && io->luma_dc)
    KF_CHECK(cudaMemcpyAsync(io->luma_dc, kf->luma.prm.res_dc, 4 * (size_t)tot.n_luma, cudaMemcpyDeviceToHost, s));
  if (kf->cfg.inter && io->chroma_dc)
    KF_CHECK(cudaMemcpyAsync(io->chroma_dc, kf->chroma.prm.res_dc, 4 * (size_t)tot.n_chroma, cudaMemcpyDeviceToHost, s));
  if (kf->dc_resid[0] && io->luma_dc_resid)
    KF_CHECK(cudaMemcpyAsync(io->luma_dc_resid, kf->dc_resid[0], 4 * (size_t)tot.n_luma, cudaMemcpyDeviceToHost, s));
  if (kf->dc_resid[1] && io->chroma_dc_resid)
    KF_CHECK(cudaMemcpyAsync(io->chroma_dc_resid, kf->dc_resid[1], 4 * (size_t)tot.n_chroma, cudaMemcpyDeviceToHost, s));
  if (io->luma_late_skip)
    KF_CHECK(cudaMemcpyAsync(io->luma_late_skip, kf->late_skip[0], sizeof(daala_b200_kf_late_skip) * tot.n_luma,
                             cudaMemcpyDeviceToHost, s));
  if (io->chroma_late_skip)
    KF_CHECK(cudaMemcpyAsync(io->chroma_late_skip, kf->late_skip[1], sizeof(daala_b200_kf_late_skip) * tot.n_chroma,
                             cudaMemcpyDeviceToHost, s));
  if (io->counts) KF_CHECK(cudaMemcpyAsync(io->counts, kf->lists.cnt, sizeof(int32_t) * 32, cudaMemcpyDeviceToHost, s));
  for (int p = 0; p < 3; p++)
    if (io->dc_index[p])
      KF_CHECK(cudaMemcpyAsync(io->dc_index[p], kf->hdc_index[p],
                               sizeof(int32_t) * (kf->plane_w[p] >> 2) * (kf->plane_h[p] >> 2) * F, cudaMemcpyDeviceToHost, s));
  if (io->dering_level_out && kf->cfg.dering)
    KF_CHECK(cudaMemcpyAsync(io->dering_level_out, kf->dering.level, (size_t)kf->nhsb * kf->nvsb * F, cudaMemcpyDeviceToHost, s));
  if (want_sym) {
    k_sym_copy<<<kf->sms * 4, 256, 0, s>>>(sc);
    KF_CHECK(cudaGetLastError());
  }
  return 0;
}

int daala_b200_kf_frame_quant_derive(const daala_b200_kf_frame_quant* rec, int n, int32_t (*tbl)[2][6]) {
  int dq_max = 1;
  for (int f = 0; f < n; f++) {
    for (int p = 0; p < 3; p++)
      for (int bs = 0; bs < 5; bs++) {
        const int dq = (rec[f].q0 * rec[f].pvq_qm_q4[p][bs * (bs + 1)]) >> 4;
        if (dq > dq_max) dq_max = dq;
      }
    if (tbl) daala_b200_dering_threshold_table(rec[f].q0, tbl[f]);
  }
  return DAALA_B200_KF_FINISH_DC_LIMIT / dq_max;
}

int daala_b200_kf_finish(daala_b200_kf* kf, const daala_b200_kf_finish_io* io) {
  if (!kf || !io) return (int)cudaErrorInvalidValue;
  const int F = kf->F;
  const size_t nsb = (size_t)F * kf->nhsb * kf->nvsb;
  const long long nb[2] = {kf->last_tot.n_luma, kf->last_tot.n_chroma};
  // the decisions in block order (the classic form: luma, chroma) or in stream order (one array of nb[0] + nb[1])
  const bool stream = io->stream_skip || io->stream_dc;
  const bool classic = io->luma_skip || io->chroma_skip || io->luma_dc || io->chroma_dc;
  const int nforms = stream ? 1 : 2;
  const long long ns[2] = {stream ? nb[0] + nb[1] : nb[0], stream ? 0 : nb[1]};
  const uint8_t* skip[2] = {stream ? io->stream_skip : io->luma_skip, io->chroma_skip};
  const int32_t* dc[2] = {stream ? io->stream_dc : io->luma_dc, io->chroma_dc};
  // every refusal before anything is copied or launched
  const char* why = !kf->cfg.inter_finish ? "the engine was created without inter_finish"
                    : !kf->have_step ? "no step has been submitted"
                    : stream && classic
                        ? "both forms of the decisions are given (luma_skip / chroma_skip / luma_dc / chroma_dc and "
                          "stream_skip / stream_dc): give one"
                    : stream && !kf->fin_form ? "stream_skip / stream_dc need an engine with symbol_stream = 2"
                    : stream && (!io->stream_skip || !io->stream_dc) ? "stream_skip and stream_dc are required together"
                    : !stream && (!skip[0] || !skip[1] || !dc[0] || !dc[1])
                        ? "luma_skip, chroma_skip, luma_dc and chroma_dc are required"
                    : kf->cfg.inter_finish == 2 && io->dering_level
                        ? "dering_level must be NULL on an inter_finish = 2 engine (the pass searches the levels)"
                    : io->ref_slot_out && !kf->fin_slot_out
                        ? "ref_slot_out needs an engine with inter_mc (the reference-picture pool)"
                        : nullptr;
  for (int f = 0; !why && io->ref_slot_out && f < F; f++) {
    const int32_t r = io->ref_slot_out[f];
    if (r < -1 || r >= kf->cfg.mc_refs) why = "a ref_slot_out entry is outside [-1, mc_refs)";
    for (int g = 0; !why && r >= 0 && g < f; g++)
      if (io->ref_slot_out[g] == r) why = "two frames name the same ref_slot_out slot";
  }
  for (int c = 0; !why && c < nforms; c++)
    for (long long i = 0; i < ns[c]; i++) {
      if (skip[c][i] > 1) {
        why = "a skip value is neither 0 nor 1";
        break;
      }
      if (dc[c][i] > kf->fin_dc_limit || dc[c][i] < -kf->fin_dc_limit) {
        why = "a |dc| exceeds DAALA_B200_KF_FINISH_DC_LIMIT / the largest dc_quant";
        break;
      }
    }
  for (size_t i = 0; !why && io->dering_level && i < nsb; i++)
    if (io->dering_level[i] > 5) why = "a dering level is above 5";
  if (why) {
    snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_finish: %s", why);
    return (int)cudaErrorInvalidValue;
  }
  cudaStream_t s = kf->stream;
  if (stream) {
    KF_CHECK(cudaMemcpyAsync(kf->fin_stream_skip, skip[0], (size_t)ns[0], cudaMemcpyHostToDevice, s));
    KF_CHECK(cudaMemcpyAsync(kf->fin_stream_dc, dc[0], 4 * (size_t)ns[0], cudaMemcpyHostToDevice, s));
  } else {
    for (int c = 0; c < 2; c++) {
      KF_CHECK(cudaMemcpyAsync(kf->fin_skip[c], skip[c], (size_t)nb[c], cudaMemcpyHostToDevice, s));
      KF_CHECK(cudaMemcpyAsync(kf->fin_dc[c], dc[c], 4 * (size_t)nb[c], cudaMemcpyHostToDevice, s));
    }
  }
  // the graph's k_fin_unstream reads the form: the one captured graph serves both
  if (kf->fin_form) KF_CHECK(cudaMemsetAsync(kf->fin_form, stream ? 1 : 0, sizeof(int32_t), s));
  // inter_finish = 2: the graph's search writes the levels
  if (io->dering_level) KF_CHECK(cudaMemcpyAsync(kf->dering.level, io->dering_level, nsb, cudaMemcpyHostToDevice, s));
  else if (kf->cfg.inter_finish == 1) KF_CHECK(cudaMemsetAsync(kf->dering.level, 0, nsb, s));
  // the graph's pool store reads the slot table: NULL stores nothing (every entry -1)
  if (io->ref_slot_out) KF_CHECK(cudaMemcpyAsync(kf->fin_slot_out, io->ref_slot_out, 4 * (size_t)F, cudaMemcpyHostToDevice, s));
  else if (kf->fin_slot_out) KF_CHECK(cudaMemsetAsync(kf->fin_slot_out, 0xFF, 4 * (size_t)F, s));
  if (!kf->fin_captured) {
    // as the step's graph: a first run outside the capture loads the kernels
    int rc = kf_enqueue_finish(kf);
    if (rc) return rc;
    KF_CHECK(cudaStreamSynchronize(s));
    KF_CHECK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    rc = kf_enqueue_finish(kf);
    cudaError_t e = cudaStreamEndCapture(s, &kf->fin_graph);
    if (rc) return rc;
    KF_CHECK(e);
    KF_CHECK(cudaGraphInstantiate(&kf->fin_exec, kf->fin_graph, 0));
    kf->fin_captured = true;
  }
  KF_CHECK(cudaGraphLaunch(kf->fin_exec, s));
  for (int f = 0; io->ref_slot_out && f < F; f++)
    if (io->ref_slot_out[f] >= 0) kf->slot_filled[io->ref_slot_out[f]] = 1;
  for (int p = 0; p < 3; p++) {
    const size_t n = (size_t)kf->plane_w[p] * kf->plane_h[p] * F;
    if (io->pixels_out[p]) KF_CHECK(cudaMemcpyAsync(io->pixels_out[p], kf->fin_pixels[p], n, cudaMemcpyDeviceToHost, s));
    if (io->bskip_out[p])
      KF_CHECK(cudaMemcpyAsync(io->bskip_out[p], kf->fin_bskip[p], (size_t)kf->fin.skip_pitch[p] * F, cudaMemcpyDeviceToHost, s));
  }
  if (io->dering_level_out) KF_CHECK(cudaMemcpyAsync(io->dering_level_out, kf->fin_level, nsb, cudaMemcpyDeviceToHost, s));
  return 0;
}

int daala_b200_kf_pool_load(daala_b200_kf* kf, int slot, const uint8_t* const planes[3]) {
  if (!kf) return (int)cudaErrorInvalidValue;
  const char* why = !kf->cfg.inter_mc ? "the engine was created without inter_mc (it has no reference-picture pool)"
                    : slot < 0 || slot >= kf->cfg.mc_refs ? "slot is outside [0, mc_refs)"
                    : !planes || !planes[0] || !planes[1] || !planes[2] ? "planes[0..2] are required"
                                                                        : nullptr;
  if (why) {
    snprintf(kf->err, sizeof(kf->err), "daala_b200_kf_pool_load: %s", why);
    return (int)cudaErrorInvalidValue;
  }
  for (int p = 0; p < 3; p++) {
    const size_t n = (size_t)kf->plane_w[p] * kf->plane_h[p];
    KF_CHECK(cudaMemcpyAsync(kf->ref_pixels[p] + slot * n, planes[p], n, cudaMemcpyDefault, kf->stream));
  }
  kf->slot_filled[slot] = 1;
  return 0;
}

int daala_b200_kf_wait(daala_b200_kf* kf) {
  if (!kf) return (int)cudaErrorInvalidValue;
  KF_CHECK(cudaStreamSynchronize(kf->stream));
  return 0;
}

int daala_b200_kf_encode(daala_b200_kf* kf, const daala_b200_kf_io* io) {
  int rc = daala_b200_kf_submit(kf, io);
  if (rc) return rc;
  return daala_b200_kf_wait(kf);
}

// Synchronous copy helper for tests / device-resident callers without a CUDA binding of their own:
// kind 0 = host -> device, 1 = device -> host, 2 = device -> device.
int daala_b200_device_copy(void* dst, const void* src, size_t bytes, int kind) {
  const cudaMemcpyKind k = kind == 0 ? cudaMemcpyHostToDevice : kind == 1 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  cudaError_t e = cudaMemcpy(dst, src, bytes, k);
  return (int)e;
}

void* daala_b200_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
  return p;
}
void daala_b200_host_free(void* p) { if (p) cudaFreeHost(p); }

}  // extern "C"
