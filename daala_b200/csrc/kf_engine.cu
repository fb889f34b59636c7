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
//     -> iDCT + lapped postfilters -> u8 reconstruction, packed symbols for the host entropy coder.
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

#include <mutex>

#include "daala_b200.h"
#include "dering_search.h"
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
  kNItemsL = 4,      // [3] luma dependency-free items per class (bands 3 / 6: classes 1 / 2)
  kNItemsC = 7,      // [3] chroma items per class (n <= 16, 32, 128)
  kTotalHi = 14,     // luma chain items in total
  kNHeads = 15,      // row / column chain items ready from the start (no same-size neighbour to wait for)
  kNHeads0 = 16,     // band-0 items ready from the start
  kError = 17,
  // the words the persistent kernels hammer with atomics each sit in a 128-byte line of their own
  kHeadLoL = 32,     // ticket of the luma dependency-free lists
  kHeadLoC = 64,     // ticket of the chroma lists
  kHeadHi = 96,      // luma chain queue: next slot to claim
  kTailHi = 128,     //                   next slot to fill
  kDoneHi = 160,     // band-0 items finished (flushed by warps when they go idle)
  kHeadCh = 192,     // ticket of the row / column chain heads
  kWaiters = 224,    // warps parked on a future band-0 slot
  kCntWords = 256
};

constexpr int kTile = 1024;        // units per scan tile
constexpr int kMaxLevels = 4096;   // (plane width + height) / 4 of an 8K frame is 3008
constexpr int kLevelBins = kMaxLevels * 3;

struct Lists {
  const uint8_t* bsize;            // [F][UH][bstride]
  int bstride;
  long long bsize_pitch;
  int F, UW, UH;                   // 8x8-luma units per frame
  int u_row0, u_rows;              // unit rows of this rank's shard
  int ntiles;
  int4* tile_sum;                  // [ntiles] then exclusive prefixes in place
  int32_t* unit_lbase;             // [F*UH*UW] index of the first luma block whose origin is in the unit
  daala_b200_pvq_block* luma;
  daala_b200_pvq_block* chroma;
  int32_t* dep_top;                // same-size neighbour above / to the left (od_hv_intra_pred), or -1
  int32_t* dep_left;
  int32_t* succ_bottom;            // inverse: the block whose dep_top / dep_left is this one, or -1
  int32_t* succ_right;
  uint32_t* items_l[3];            // dependency-free luma items per class
  uint32_t* items_c[3];
  uint32_t* heads;                 // row / column chain items that are ready from the start
  uint32_t* heads0;                // band-0 items that are ready from the start
  int32_t* cnt;                    // [kCntWords]
  // level path: chain items counting-sorted by dependency level (position along the chain in units of the
  // block size; larger bands first inside a level)
  int32_t* lvl_hist;               // [kLevelBins] counts, then exclusive offsets
  int32_t* lvl_cursor;             // [kLevelBins]
  uint32_t* lvl_items;             // sorted chain items
  int nlevels;
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
    if (tot.x > L.max_luma || 2 * tot.z > L.max_chroma) L.cnt[kError] = 1;
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

// Dependency level of a chain item: its position along the chain in units of its own block size (band 0:
// the anti-diagonal).  Items only depend on same-size neighbours, whose level is smaller by one; bin =
// level * 3 + (2 - class) so that the 128-coefficient bands of a level come first.
__device__ __forceinline__ int level_bin(int band, int bs, int x0, int y0, int y_first) {
  const int sh = bs + 2, bx = x0 >> sh, by = (y0 - y_first) >> sh;
  const int r = band % 3;
  const int lvl = band == 0 ? bx + by : r == 1 ? by : bx;
  return lvl * 3 + (2 - band_class(band));
}

// warp-aggregated append of `v` to list[*counter] by the lanes with `pred`
__device__ __forceinline__ void append(uint32_t* list, int32_t* counter, bool pred, uint32_t v) {
  const unsigned m = __ballot_sync(__activemask(), pred);
  if (!pred) return;
  const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(counter, __popc(m));
  base = __shfl_sync(m, base, leader);
  list[base + __popc(m & ((1u << lane) - 1u))] = v;
}

// Luma dependency structure.  od_hv_intra_pred (src/intra.c:37) predicts band b of a block from band b of
// the same-size TOP neighbour (row-0 bands 1/4/7), the LEFT one (column-0 bands 2/5/8), both (band 0) or
// nothing (bands 3/6).  Per block: the two neighbours and, inverted, the blocks that wait for this one;
// per (block, band): a dependency-free item, a chain head (ready now) or a chain link (made ready by the
// persistent kernel when its neighbours are done).
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
    int chain = 0;
    for (int band = 0; band < 9; band++) {
      const bool has = band < nb;
      const bool is_free = band == 3 || band == 6;
      const int r = band % 3;
      const bool waits = band == 0 ? (top >= 0 || left >= 0) : r == 1 ? top >= 0 : left >= 0;
      const uint32_t item = ((uint32_t)blk << 4) | band;
      if (band == 3 || band == 6) append(L.items_l[band_class(band)], &L.cnt[kNItemsL + band_class(band)], has, item);
      else if (band == 0) append(L.heads0, &L.cnt[kNHeads0], has && !waits, item);
      else append(L.heads, &L.cnt[kNHeads], has && !waits, item);
      chain += has && !is_free;
      if (has && !is_free && L.lvl_hist) {
        const daala_b200_pvq_block b = L.luma[blk];
        atomicAdd(&L.lvl_hist[level_bin(band, bs, b.x0, b.y0, L.u_row0 * 8)], 1);
      }
    }
    // total number of chain items
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) chain += __shfl_xor_sync(0xffffffffu, chain, o);
    if ((threadIdx.x & 31) == 0 && chain) atomicAdd(&L.cnt[kTotalHi], chain);
  }
}

// One CTA: exclusive scan of the level bins in place (+ a copy as scatter cursors).
__global__ void __launch_bounds__(1024) k_level_scan(const __grid_constant__ Lists L) {
  __shared__ int part[1024];
  constexpr int kPer = kLevelBins / 1024;
  const int t = threadIdx.x;
  int v[kPer], sum = 0;
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    v[i] = L.lvl_hist[t * kPer + i];
    sum += v[i];
  }
  part[t] = sum;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int add = t >= o ? part[t - o] : 0;
    __syncthreads();
    part[t] += add;
    __syncthreads();
  }
  int run = part[t] - sum;
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    L.lvl_hist[t * kPer + i] = run;
    L.lvl_cursor[t * kPer + i] = run;
    run += v[i];
  }
}

__global__ void __launch_bounds__(256) k_level_scatter(const __grid_constant__ Lists L) {
  const int n = min(L.cnt[kNLuma], L.max_luma);
  for (int blk = blockIdx.x * blockDim.x + threadIdx.x; blk < n; blk += gridDim.x * blockDim.x) {
    const daala_b200_pvq_block b = L.luma[blk];
    const int nb = num_bands(b.bs);
    for (int band = 0; band < nb; band++) {
      if (band == 3 || band == 6) continue;
      const int pos = atomicAdd(&L.lvl_cursor[level_bin(band, b.bs, b.x0, b.y0, L.u_row0 * 8)], 1);
      L.lvl_items[pos] = ((uint32_t)blk << 4) | band;
    }
  }
}

// Chroma items: no dependencies between blocks; compaction per class (order is free).
__global__ void __launch_bounds__(256) k_chroma_items(const __grid_constant__ Lists L) {
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

// ---- PVQ stage -----------------------------------------------------------------------------------
struct Stage {
  daala_b200_pvq_params prm;
  const uint32_t* items[3];        // dependency-free items per class (taken largest class first)
  // luma only: row / column chain heads (static list; a chain is then walked by one warp), and the
  // band-0 queue = [heads0 (static) | ring filled at run time]
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
  // level path: chain items sorted by level; one record of context per position inside a level
  const int32_t* lvl_off;          // [kLevelBins] exclusive offsets of the bins
  const uint32_t* lvl_items;
  int nlevels, lvl_slots;
  int16_t* lv_vec; int32_t* lv_lanes; int32_t* lv_uni; int16_t* lv_snap;
  int32_t* lv_bar;                 // grid barrier counter
  // luma: the no-reference events of every chain band, searched ahead of the chains (k_pvq_prepass)
  int32_t* pre_ev;                 // [coefs / 8][kPreEvWords], record of a band at (coef_off + band start) >> 3
  int16_t* pre_snap;               // [2 * coefs]: the events' pulses at 2 * (coef_off + band start)
  int max_waiters;                 // warps that may park on future band-0 slots; the others exit when idle
  int skip_lo;                     // the persistent kernel leaves the dependency-free lists to the split path
  const double* rsqrt_tbl;         // [kTableDoubles] the reference's 1/sqrt(i) and theta-rate terms (pvq_fill_rsqrt_table)
  int16_t* res_pack;               // [nblocks*9][4]: gain, itheta, max_theta, k (what the coder reads)
  const int32_t* cfl_plane;        // chroma: prediction plane (chroma geometry), else NULL
  long long cfl_pitch;
  int cfl_stride;
};

// raster -> coding order of every block (od_raster_to_coding_order, src/partition.c:123); chroma:
// also the CfL prediction and its sign flip (src/pvq_encoder.c:847-871).  One warp per block.
template <bool kChroma>
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
    if (!kChroma) {
      for (int i = lane; i < len; i += 32) vin[i] = i == 0 ? src[0] : src[scan_to_raster(i, ln, stride)];
    } else {
      const int32_t* psrc = S.cfl_plane + b.frame * S.cfl_pitch + (size_t)b.y0 * S.cfl_stride + b.x0;
      int32_t* vref = prm.ref + b.coef_off;
      const int qoff = prm.qm_stride + ((((1 << (2 * b.bs)) - 1) << 4) / 3);
      int32_t xy = 0;
      for (int i = lane; i < len; i += 32) {
        const int32_t vi = i == 0 ? src[0] : src[scan_to_raster(i, ln, stride)];
        const int32_t vr = i == 0 ? psrc[0] : psrc[scan_to_raster(i, ln, S.cfl_stride)];
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

// Chroma-from-luma prediction planes (od_resample_luma_coeffs, src/intra.c:72): see k_cfl_pred of
// pvq_kernels.cu; here with the block count on the device.  One warp per chroma block of plane 1
// (plane 2 shares the prediction).
__global__ void __launch_bounds__(256) k_cfl_plane(const __grid_constant__ Stage S, int32_t* pred_plane) {
  const daala_b200_pvq_params& prm = S.prm;
  const int n = min(S.cnt[S.n_blocks_at], S.max_blocks);
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int blk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; blk < n; blk += nwarps) {
    const daala_b200_pvq_block b = prm.blocks[blk];
    if (b.pli != 1) continue;
    const int nn = 4 << b.bs;
    const int lstride = prm.plane_stride[0];
    const int32_t* luma = prm.coef_plane[0] + b.frame * prm.plane_frame_pitch[0] + (size_t)(2 * b.y0) * lstride + 2 * b.x0;
    int32_t* dst = pred_plane + b.frame * S.cfl_pitch + (size_t)b.y0 * S.cfl_stride + b.x0;
    if (b.xdec & 0x80) {
      // four 4x4 luma blocks -> one 4x4 chroma prediction: od_tf_up_hv_lp (src/tf.c:82) + OD_CFL_SCALING4
      const int scaling4[4][4] = {{128, 128, 100, 36}, {128, 80, 71, 35}, {100, 71, 35, 31}, {36, 35, 31, 18}};
      if (lane < 4) {
        const int x = lane & 1, y = lane >> 1;
        int ll = luma[(size_t)y * lstride + x], lh = luma[(size_t)y * lstride + x + 4];
        int hl = luma[(size_t)(y + 4) * lstride + x], hh = luma[(size_t)(y + 4) * lstride + x + 4];
        ll += lh; hh -= hl;
        const int t = (ll - hh) >> 1;
        hl = t - hl; lh = t - lh;
        ll -= hl; hh += lh;
        const int hs = x & 1, vs = y & 1;
        int r, c;
        r = 2 * y + vs; c = 2 * x + hs;         dst[(size_t)r * S.cfl_stride + c] = (scaling4[c][r] * ll + 64) >> 7;
        r = 2 * y + vs; c = 2 * x + 1 - hs;     dst[(size_t)r * S.cfl_stride + c] = (scaling4[c][r] * lh + 64) >> 7;
        r = 2 * y + 1 - vs; c = 2 * x + hs;     dst[(size_t)r * S.cfl_stride + c] = (scaling4[c][r] * hl + 64) >> 7;
        r = 2 * y + 1 - vs; c = 2 * x + 1 - hs; dst[(size_t)r * S.cfl_stride + c] = (scaling4[c][r] * hh + 64) >> 7;
      }
    } else {
      // only the coded prefix is ever read; copying the whole low-frequency quarter keeps this simple
      const int lim = nn > 32 ? 32 : nn;
      for (int i = lane; i < lim * lim; i += 32) {
        const int r = i / lim, c = i % lim;
        dst[(size_t)r * S.cfl_stride + c] = luma[(size_t)r * lstride + c];
      }
    }
  }
}

// resident CTAs per SM the persistent PVQ kernel is compiled for (register cap = 65536 / 128 / this)
#ifndef DAALA_PERSIST_SPECIALISE
#define DAALA_PERSIST_SPECIALISE 0
#endif
#ifndef DAALA_PERSIST_MIN_CTAS
#define DAALA_PERSIST_MIN_CTAS 8
#endif
// warps per CTA of the persistent kernel.  1: a warp that runs out of work frees its registers and shared
// memory at once (a CTA only retires when all of its warps have), so the next kernel -- another engine's
// batch -- fills the SM while the last dependency chains of this one are still being walked.
#ifndef DAALA_PERSIST_WARPS
#define DAALA_PERSIST_WARPS 1
#endif
constexpr int kPersistThreads = 32 * DAALA_PERSIST_WARPS;
constexpr int kPersistCtas = DAALA_PERSIST_MIN_CTAS * 4 / DAALA_PERSIST_WARPS;   // per SM, same number of warps
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

// Next item for an idle warp (uniform), or kNoItem when the stage has nothing left for it.
//  chroma (kIntra = false): a ticket into the item lists, largest bands first.
//  luma, in this order: (1) a filled slot of the band-0 queue -- band 0 is a 2-D wavefront over each
//  same-size region, the deepest dependency structure of a frame, so it goes first; (2) the head of a row
//  or column chain; (3) a dependency-free item; (4) a ticket for a FUTURE band-0 slot, waited for on the
//  slot itself (distinct addresses: no hot spot).  `done` = band-0 items this warp finished since it was
//  last here; the warp whose flush completes the count releases every waiter with kExit.
template <bool kIntra>
__device__ __forceinline__ uint32_t next_item(const Stage& S, int lane, int* done, bool* waiter) {
  int slot = -1, head = -1, lo = -1, nheads0 = 0, fin = -1;
  if (lane == 0) {
    const int n2 = S.cnt[S.n_items_at + 2], n1 = S.cnt[S.n_items_at + 1], n0 = S.cnt[S.n_items_at];
    const int nlo = S.skip_lo ? 0 : n0 + n1 + n2;
    if (kIntra) {
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
    }
    if (slot < 0 && head < 0 && ld_relaxed(&S.cnt[S.head_lo_at]) < nlo) {
      const int l = atomicAdd(&S.cnt[S.head_lo_at], 1);
      if (l < nlo) lo = l;
    }
    if (kIntra && slot < 0 && head < 0 && lo < 0) {
      // nothing to do right now: park on the next band-0 slot -- unless enough warps already do; the rest
      // leave and free their SM resources for whatever kernel comes next (another engine's batch)
      if (!*waiter && atomicAdd(&S.cnt[kWaiters], 1) < S.max_waiters) *waiter = true;
      if (*waiter) slot = atomicAdd(&S.cnt[kHeadHi], 1);
    }
  }
  *done = 0;
  if (kIntra) {
    fin = __shfl_sync(0xffffffffu, fin, 0);
    if (fin >= 0) {
      // every warp holds at most one ticket: slots [fin, fin + #warps] cover all of them, now and later
      const int nw = (gridDim.x * blockDim.x) >> 5;
      for (int i = lane; i <= nw; i += 32) st_release((int*)&S.ring[fin + i], (int)kExit);
    }
    head = __shfl_sync(0xffffffffu, head, 0);
    if (head >= 0) return S.heads[head];
  }
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

// One (block, band) item by one warp.  kIntra: the band's prediction is built from the quantised
// neighbours first (od_hv_intra_pred, src/intra.c:37-62).
template <bool kIntra>
__device__ __forceinline__ void run_item(const Stage& S, uint32_t item, int lane, int16_t* snap) {
  const daala_b200_pvq_params& prm = S.prm;
  const int blk = (int)(item >> 4), band = (int)(item & 15);
  const daala_b200_pvq_block b = prm.blocks[blk];
  const int bs = b.bs, pli = b.pli;
  const int start = band_start(band);
  const int bn = band_start(band + 1) - start;
  const size_t off = (size_t)b.coef_off + start;
  if (kIntra) intra_band_ref(S, blk, band, b.coef_off, lane);
  int qidx = bs * (bs + 1) + (band + 1) - (band + 1) / 3;
  int q = (prm.q0 * prm.pvq_qm_q4[pli][qidx]) >> 4;
  if (q < 1) q = 1;
  const int beta = (prm.use_masking && pli == 0 && bs > 0) ? kBeta15 : kBeta1;
  const int qoff = (b.xdec & 1 ? prm.qm_stride : 0) + ((((1 << (2 * bs)) - 1) << 4) / 3) + start;
  int itheta, max_theta, k;
  double skip_term;
  const bool pre = kIntra && S.pre_ev && band != 3 && band != 6;
  // size-class specialised instantiations (DAALA_PERSIST_SPECIALISE): a band then executes less straight-line
  // code, at the price of a larger kernel
  const int32_t* pev = pre ? S.pre_ev + (off >> 3) * kPreEvWords : nullptr;
  const int16_t* psn = pre ? S.pre_snap + 2 * off : nullptr;
  int gain;
#if DAALA_PERSIST_SPECIALISE
  if (bn > 32)
    gain = quantise_band_warp<2>(lane, snap, S.rsqrt_tbl, prm.out + off, prm.in + off, prm.ref + off, bn, q, prm.y + off,
                                 &itheta, &max_theta, &k, beta, &skip_term, prm.is_keyframe, pli, prm.qm + qoff,
                                 prm.qm_inv + qoff, prm.pvq_norm_lambda, pev, psn);
  else
    gain = quantise_band_warp<1>(lane, snap, S.rsqrt_tbl, prm.out + off, prm.in + off, prm.ref + off, bn, q, prm.y + off,
                                 &itheta, &max_theta, &k, beta, &skip_term, prm.is_keyframe, pli, prm.qm + qoff,
                                 prm.qm_inv + qoff, prm.pvq_norm_lambda, pev, psn);
#else
  gain = quantise_band_warp<0>(lane, snap, S.rsqrt_tbl, prm.out + off, prm.in + off, prm.ref + off, bn, q, prm.y + off,
                               &itheta, &max_theta, &k, beta, &skip_term, prm.is_keyframe, pli, prm.qm + qoff,
                               prm.qm_inv + qoff, prm.pvq_norm_lambda, pev, psn);
#endif
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
// (chroma; luma bands 3 / 6); the intra chains stay in the persistent kernel.
struct ItemGeom {
  int blk, band, bn, q, beta, pli, qoff;
  size_t off;
};
__device__ __forceinline__ ItemGeom item_geom(const daala_b200_pvq_params& prm, uint32_t item) {
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
  int q = (prm.q0 * prm.pvq_qm_q4[g.pli][qidx]) >> 4;
  g.q = q < 1 ? 1 : q;
  g.beta = (prm.use_masking && g.pli == 0 && bs > 0) ? kBeta15 : kBeta1;
  g.qoff = (b.xdec & 1 ? prm.qm_stride : 0) + ((((1 << (2 * bs)) - 1) << 4) / 3) + start;
  return g;
}

// kPhase 0 / 1 / 2 = setup / search / finish of the items [chunk * slots, ...) of class `cls`.
// kZeroRef: the prediction is all zero (luma bands 3 / 6).
template <int kPhase, bool kZeroRef, int kMode>
__global__ void __launch_bounds__(128) k_pvq_split(const __grid_constant__ Stage S, int cls, int chunk) {
  const daala_b200_pvq_params& prm = S.prm;
  const int lane = threadIdx.x & 31;
  const int slots = S.sp_slots[cls];
  const int first = chunk * slots;
  const int count = min(S.cnt[S.n_items_at + cls] - first, slots);
  const int vs = cls == 2 ? 128 : 32;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < count; i += nwarps) {
    const ItemGeom g = item_geom(prm, S.items[cls][first + i]);
    int16_t* vec = S.sp_vec[cls] + (size_t)i * 3 * vs;
    int32_t* lanes = S.sp_lanes[cls] + (size_t)i * kCtxLaneWords * 16;
    int32_t* uni = S.sp_uni[cls] + (size_t)i * kCtxUniWords;
    int16_t* snap = S.sp_snap[cls] + (size_t)i * kMaxEvents * vs;
    const int32_t* r0 = kZeroRef ? nullptr : prm.ref + g.off;
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

// ---- prepass ---------------------------------------------------------------------------------------------
// Keyframe luma always evaluates the no-reference candidates of pvq_theta (src/pvq_encoder.c:573-606), and
// they depend on the input vector alone: their searches (two from scratch per band, the larger half of a
// chain band's work) run here for every chain band at once, fully parallel, and the chain walk imports the
// results (band_noref_export / band_search's pre_ev) -- that work leaves the dependency-bound kernel.
template <int kMode>
__global__ void __launch_bounds__(128) k_pvq_prepass(const __grid_constant__ Stage S) {
  const daala_b200_pvq_params& prm = S.prm;
  __shared__ int16_t snap_all[4][2 * kMaxN];
  const int lane = threadIdx.x & 31;
  int16_t* snap = snap_all[threadIdx.x >> 5];
  const int nblk = min(S.cnt[S.n_blocks_at], S.max_blocks);
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  // kMode 1: bands 0, 1, 2, 4, 5 (n <= 32); kMode 2: bands 7, 8 (n = 128)
  const int per = kMode == 2 ? 2 : 5;
  for (long long i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < (long long)nblk * per; i += nwarps) {
    const int blk = (int)(i / per), sel = (int)(i % per);
    const int band = kMode == 2 ? 7 + sel : (sel < 3 ? sel : sel + 1);
    if (band >= num_bands(prm.blocks[blk].bs)) continue;
    const ItemGeom g = item_geom(prm, ((uint32_t)blk << 4) | band);
    BandCtx B;
    band_setup<kMode>(lane, B, prm.in + g.off, nullptr, g.bn, g.q, g.beta, prm.is_keyframe, g.pli, prm.qm + g.qoff,
                      prm.pvq_norm_lambda, S.rsqrt_tbl);
    band_search<kMode>(lane, B, g.bn, snap, kMaxN, S.rsqrt_tbl);
    band_noref_export(lane, B, g.bn, snap, kMaxN, S.pre_ev + (g.off >> 3) * kPreEvWords, S.pre_snap + 2 * g.off);
  }
}

// ---- level path -----------------------------------------------------------------------------------------
// The luma intra chains, level-synchronously: all chain items of one dependency level are independent, so
// the whole GPU runs phase A (prediction from the neighbours + band_setup) for the level, then phase B
// (searches), then phase C (costs, fold, synthesis), with a grid-wide barrier in between -- at any time
// only one phase's code is being executed anywhere (see "split path" above for why that matters), and
// nobody ever waits on a flag.  One persistent launch, all CTAs resident (the host sizes the grid).
__device__ __forceinline__ void grid_barrier(int32_t* bar, int* target, int nctas) {
  __syncthreads();
  if (threadIdx.x == 0) {
    *target += nctas;
    __threadfence();
    atomicAdd(bar, 1);
    while (ld_acquire(bar) < *target) {}
  }
  __syncthreads();
}

__global__ void __launch_bounds__(128, 4) k_pvq_levels(const __grid_constant__ Stage S) {
  const daala_b200_pvq_params& prm = S.prm;
  __shared__ int bar_target;
  if (threadIdx.x == 0) bar_target = 0;
  const int lane = threadIdx.x & 31;
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int total = S.cnt[kTotalHi];
  constexpr int vs = 128;
  for (int lvl = 0; lvl < S.nlevels; lvl++) {
    const int base = S.lvl_off[lvl * 3];
    const int end = lvl + 1 < kMaxLevels ? S.lvl_off[(lvl + 1) * 3] : total;
    if (end - base > S.lvl_slots && threadIdx.x == 0 && blockIdx.x == 0) S.cnt[kError] = 2;
    const int n = min(end - base, S.lvl_slots);
    if (n <= 0) continue;   // uniform: every CTA reads the same offsets
    for (int phase = 0; phase < 3; phase++) {
      for (int i = w; i < n; i += nwarps) {
        const uint32_t item = S.lvl_items[base + i];
        const ItemGeom g = item_geom(prm, item);
        int16_t* vec = S.lv_vec + (size_t)i * 3 * vs;
        int32_t* lanes = S.lv_lanes + (size_t)i * kCtxLaneWords * 16;
        int32_t* uni = S.lv_uni + (size_t)i * kCtxUniWords;
        int16_t* snap = S.lv_snap + (size_t)i * kMaxEvents * vs;
        BandCtx B;
        if (phase == 0) {
          intra_band_ref(S, g.blk, g.band, (int)(g.off - band_start(g.band)), lane);
          band_setup<0>(lane, B, prm.in + g.off, prm.ref + g.off, g.bn, g.q, g.beta, prm.is_keyframe, g.pli,
                        prm.qm + g.qoff, prm.pvq_norm_lambda, S.rsqrt_tbl);
          band_ctx_store_setup(lane, B, g.bn, vec, vs, lanes, uni);
        } else if (phase == 1) {
          band_ctx_load_search(lane, B, g.bn, vec, vs, lanes);
          band_search<0>(lane, B, g.bn, snap, vs, S.rsqrt_tbl);
          band_ctx_store_search(lane, B, lanes);
        } else {
          band_ctx_load_finish(lane, B, g.bn, vec, vs, lanes, uni);
          int itheta, max_theta, k;
          double skip_term;
          const int gain = band_finish<0>(lane, B, snap, vs, prm.out + g.off, prm.ref + g.off, g.bn, g.q, prm.y + g.off,
                                          &itheta, &max_theta, &k, g.beta, &skip_term, prm.is_keyframe, g.pli,
                                          prm.qm_inv + g.qoff, prm.pvq_norm_lambda);
          if (lane == 0) {
            const size_t r = (size_t)g.blk * 9 + g.band;
            prm.res_skip_term[r] = skip_term;
            short4 pk;
            pk.x = (short)gain; pk.y = (short)itheta; pk.z = (short)max_theta; pk.w = (short)k;
            reinterpret_cast<short4*>(S.res_pack)[r] = pk;
          }
        }
      }
      grid_barrier(S.lv_bar, &bar_target, gridDim.x);
    }
  }
}

// Persistent PVQ kernel: one warp = one band at a time.  Luma (kIntra): the chain items of the H/V
// intra predictor form a dependency graph (per size class: band 0 a 2-D wavefront, bands 1/4/7 columns,
// bands 2/5/8 rows).  A warp that finishes a chain item CONTINUES with a successor it made ready -- a
// column or row is walked by one warp without touching the queue -- and pushes a second ready
// successor (band 0 forks) into the chain queue.
template <bool kIntra>
__global__ void __launch_bounds__(kPersistThreads, kPersistCtas) k_pvq_persist(const __grid_constant__ Stage S) {
  __shared__ int16_t snap_all[DAALA_PERSIST_WARPS][kSnapEntries];   // per warp: the pulses of every search event of a band
  const int lane = threadIdx.x & 31;
  int16_t* snap = snap_all[threadIdx.x >> 5];
  int done = 0;
  bool waiter = false;
  for (;;) {
    uint32_t item = next_item<kIntra>(S, lane, &done, &waiter);
    if (item == kNoItem) return;
    for (;;) {
      const int band = (int)(item & 15);
      run_item<kIntra>(S, item, lane, snap);
      if (!kIntra || band == 3 || band == 6) break;
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

// Start of a PVQ stage: the tickets; the chain queue starts with the heads.
__global__ void k_begin_pvq(int32_t* cnt, int luma) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (luma) {
      cnt[kHeadLoL] = 0;
      cnt[kHeadHi] = 0;
      cnt[kTailHi] = cnt[kNHeads0];
      cnt[kDoneHi] = 0;
      cnt[kHeadCh] = 0;
      cnt[kWaiters] = 0;
    } else {
      cnt[kHeadLoC] = 0;
    }
  }
}

// Per block, after all its bands: ordered skip_diff sum (src/pvq_encoder.c:875-880), keyframe DC
// (scalar_out[0] = dblock[0], src/encode.c:1381), od_init_skipped_coeffs (src/state.c:1347) +
// od_coding_order_to_raster (src/partition.c:157) back into the coefficient plane, pulses packed to
// 16 bits for the host entropy coder.  One warp per block.
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
      prm.out[b.coef_off] = prm.in[b.coef_off];
    }
    if (ln >= 5) {
      for (int i = lane; i < nn * nn; i += 32) if (i) dst[(size_t)(i >> ln) * stride + (i & (nn - 1))] = 0;
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
// with threshold = OD_DERING_GAIN_TABLE[level] * quantizer^0.84182 (* 0.6 on chroma), od_coeff_to_ref_plane.
// (c + 8 >> 4) + 128 clamped: od_coeff_to_ref_plane, src/state.c:1283
__global__ void k_i16_to_u8(const int16_t* __restrict__ src, uint8_t* __restrict__ dst, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int v = ((src[i] + 8) >> 4) + 128;
    dst[i] = (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
  }
}
// thr[pl][f][sb] = table[pl][level[f][sb]]
__global__ void k_dering_thresholds(const uint8_t* __restrict__ level, int32_t* __restrict__ thr_luma,
                                    int32_t* __restrict__ thr_chroma, int n, int4 tl_lo, int2 tl_hi, int4 tc_lo, int2 tc_hi) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int tl[6] = {tl_lo.x, tl_lo.y, tl_lo.z, tl_lo.w, tl_hi.x, tl_hi.y};
  const int tc[6] = {tc_lo.x, tc_lo.y, tc_lo.z, tc_lo.w, tc_hi.x, tc_hi.y};
  const int g = level[i] < 6 ? level[i] : 5;
  thr_luma[i] = tl[g];
  thr_chroma[i] = tc[g];
}

}  // namespace kf
}  // namespace daala_b200

// =====================================================================================================
// Host side of the engine
// =====================================================================================================
using namespace daala_b200::kf;

extern "C" int daala_b200_launch_forward(const daala_b200_frame* prm, int nplanes, cudaStream_t stream);
extern "C" int daala_b200_launch_inverse(const daala_b200_frame* prm, int nplanes, cudaStream_t stream);
extern "C" int daala_b200_launch_inverse_lapped_only(const daala_b200_frame* prm, int nplanes, cudaStream_t stream);
extern "C" int daala_b200_launch_sb_postfilter_store(const daala_b200_frame* prm, int nplanes, cudaStream_t stream);
extern "C" int daala_b200_dering_plane_batch(const daala_b200_dering_params* prm, int nframes, long long y_pitch,
                                             long long x_pitch, long long dir_pitch, long long thr_pitch, void* stream);

struct daala_b200_kf {
  daala_b200_kf_config cfg;
  int nhsb, nvsb, F;
  int plane_w[3], plane_h[3];
  cudaStream_t stream;
  bool own_stream;
  cudaGraph_t graph;
  cudaGraphExec_t exec;
  bool captured;
  // device buffers
  uint8_t* pixels[3];
  int32_t* coeffs[3];
  int32_t* lapped[3];
  uint8_t* pixels_out[3];
  uint8_t* bsize;
  int32_t* cfl_plane;
  int16_t *qm, *qm_inv;
  double* rsqrt_tbl;
  int16_t* sp_vec[3];
  int32_t* sp_lanes[3];
  int32_t* sp_uni[3];
  int16_t* sp_snap[3];
  int sp_slots[3];
  int16_t* lv_vec;
  int32_t* lv_lanes;
  int32_t* lv_uni;
  int16_t* lv_snap;
  int32_t* lv_bar;
  int lvl_slots, lvl_grid;
  // deringing stage
  uint8_t* dering_level;           // [F][nvsb][nhsb]
  int32_t *dering_thr[2];          // luma / chroma thresholds per superblock
  int16_t *dering_in[3], *dering_out[3];
  int32_t* dering_dir;             // [F][nvsb*8][nhsb*8]
  uint8_t* dering_skip;            // all zero: keyframes never mark a block skipped (src/encode.c:1690)
  int dering_tbl[2][6];
  // level search (cfg.dering == 2): packed superblock pairs and the 6 x F x nsb distortions
  int32_t *dering_orig, *dering_cand;
  double* dering_dist;
  Lists lists;
  Stage luma, chroma;
  daala_b200_frame frame;
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
    kf->bytes_allocated += bytes;
    e = cudaMemset(*p, 0, bytes);
  }
  return e;
}

static int kf_alloc(daala_b200_kf* kf) {
  const int F = kf->F;
  const long long luma_px = (long long)kf->plane_w[0] * kf->plane_h[0];
  for (int p = 0; p < 3; p++) {
    const size_t n = (size_t)kf->plane_w[p] * kf->plane_h[p] * F;
    KF_CHECK(dalloc(kf, &kf->pixels[p], n));
    KF_CHECK(dalloc(kf, &kf->coeffs[p], n));
    KF_CHECK(dalloc(kf, &kf->lapped[p], n));
    KF_CHECK(dalloc(kf, &kf->pixels_out[p], n));
  }
  const int UW = kf->nhsb * 8, UH = kf->nvsb * 8;
  KF_CHECK(dalloc(kf, &kf->bsize, (size_t)F * UW * UH));
  KF_CHECK(dalloc(kf, &kf->cfl_plane, (size_t)kf->plane_w[1] * kf->plane_h[1] * F));
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
  KF_CHECK(dalloc(kf, &L.luma, (size_t)L.max_luma));
  KF_CHECK(dalloc(kf, &L.chroma, (size_t)L.max_chroma));
  KF_CHECK(dalloc(kf, &L.dep_top, (size_t)L.max_luma));
  KF_CHECK(dalloc(kf, &L.dep_left, (size_t)L.max_luma));
  KF_CHECK(dalloc(kf, &L.succ_bottom, (size_t)L.max_luma));
  KF_CHECK(dalloc(kf, &L.succ_right, (size_t)L.max_luma));
  // item capacities follow from the pixel count alone: one band per 4x4 block is the densest case
  const size_t luma_shard_px = (size_t)F * L.u_rows * UW * 64;
  kf->chain_cap = luma_shard_px / 16 + 64 + (size_t)kf->sms * 64;   // + one exit slot per persistent warp
  const size_t cap_l[3] = {64, luma_shard_px / 64 + 64, luma_shard_px / 256 + 64};   // bands 3 / 6 only
  const size_t cap_c[3] = {(size_t)L.max_chroma * 3 / 2 + 64, luma_shard_px / 4 * 2 * 3 / 64 + 64,
                           luma_shard_px / 4 * 2 * 3 / 256 + 64};
  for (int c = 0; c < 3; c++) {
    KF_CHECK(dalloc(kf, &L.items_l[c], cap_l[c]));
    KF_CHECK(dalloc(kf, &L.items_c[c], cap_c[c]));
  }
  if (kf->cfg.split_free > 0) {
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
  if (kf->cfg.level_chains) {
    KF_CHECK(dalloc(kf, &L.lvl_hist, (size_t)kLevelBins));
    KF_CHECK(dalloc(kf, &L.lvl_cursor, (size_t)kLevelBins));
    KF_CHECK(dalloc(kf, &L.lvl_items, kf->chain_cap));
    L.nlevels = (kf->plane_w[0] + L.u_rows * 8) / 4 + 2;
    if (L.nlevels >= kMaxLevels) return (int)cudaErrorInvalidValue;
    kf->lvl_slots = 2048 * F;
    KF_CHECK(dalloc(kf, &kf->lv_vec, (size_t)kf->lvl_slots * 3 * 128));
    KF_CHECK(dalloc(kf, &kf->lv_lanes, (size_t)kf->lvl_slots * kCtxLaneWords * 16));
    KF_CHECK(dalloc(kf, &kf->lv_uni, (size_t)kf->lvl_slots * kCtxUniWords));
    KF_CHECK(dalloc(kf, &kf->lv_snap, (size_t)kf->lvl_slots * kMaxEvents * 128));
    KF_CHECK(dalloc(kf, &kf->lv_bar, (size_t)32));
    int per_sm = 0;
    KF_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pvq_levels, 128, 0));
    if (per_sm < 1) return (int)cudaErrorLaunchOutOfResources;
    kf->lvl_grid = per_sm * kf->sms;   // all CTAs resident: the kernel synchronises the whole grid
  }
  KF_CHECK(dalloc(kf, &L.heads, kf->chain_cap));
  KF_CHECK(dalloc(kf, &L.heads0, (size_t)L.max_luma));
  KF_CHECK(dalloc(kf, &L.cnt, (size_t)kCntWords));

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
    p.qm = kf->qm;
    p.qm_inv = kf->qm_inv;
    for (int i = 0; i < 3; i++) {
      p.coef_plane[i] = kf->coeffs[i];
      p.pred_plane[i] = nullptr;
      p.plane_frame_pitch[i] = (long long)kf->plane_w[i] * kf->plane_h[i];
      p.plane_stride[i] = kf->plane_w[i];
    }
    p.qm_stride = kf->cfg.qm_stride;
    p.q0 = kf->cfg.q0 > 1 ? kf->cfg.q0 : 1;
    p.is_keyframe = 1;
    p.use_masking = kf->cfg.use_masking;
    p.pvq_norm_lambda = kf->cfg.pvq_norm_lambda;
    memcpy(p.pvq_qm_q4, kf->cfg.pvq_qm_q4, sizeof(p.pvq_qm_q4));
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
    S.skip_lo = chroma ? 0 : kf->cfg.split_free > 1;
    S.max_waiters = getenv("DAALA_B200_MAX_WAITERS") ? atoi(getenv("DAALA_B200_MAX_WAITERS")) : kf->sms * 8;
    if (!chroma && kf->cfg.noref_prepass) {
      KF_CHECK(dalloc(kf, &S.pre_ev, (ncoef / 8 + 2) * kPreEvWords));
      KF_CHECK(dalloc(kf, &S.pre_snap, 2 * ncoef));
    }
    if (!chroma) {
      S.lvl_off = L.lvl_hist;
      S.lvl_items = L.lvl_items;
      S.nlevels = L.nlevels;
      S.lvl_slots = kf->lvl_slots;
      S.lv_vec = kf->lv_vec;
      S.lv_lanes = kf->lv_lanes;
      S.lv_uni = kf->lv_uni;
      S.lv_snap = kf->lv_snap;
      S.lv_bar = kf->lv_bar;
    }
    S.n_items_at = chroma ? kNItemsC : kNItemsL;
    S.head_lo_at = chroma ? kHeadLoC : kHeadLoL;
    S.n_blocks_at = chroma ? kNChroma : kNLuma;
    S.max_blocks = (int)nblk;
    if (!chroma) {
      S.dep_top = L.dep_top;
      S.dep_left = L.dep_left;
      S.succ_bottom = L.succ_bottom;
      S.succ_right = L.succ_right;
      S.heads = L.heads;
      S.heads0 = L.heads0;
      KF_CHECK(dalloc(kf, &S.ring, kf->chain_cap));
      KF_CHECK(dalloc(kf, &S.join0, nblk));
    } else {
      S.cfl_plane = kf->cfl_plane;
      S.cfl_pitch = (long long)kf->plane_w[1] * kf->plane_h[1];
      S.cfl_stride = kf->plane_w[1];
    }
    return 0;
  };
  int rc = setup_stage(kf->luma, false);
  if (rc) return rc;
  rc = setup_stage(kf->chroma, true);
  if (rc) return rc;
  (void)luma_px;

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
  f.haar_dc = 1;
  f.nframes = F;
  f.sb_row0 = kf->cfg.sb_row0;
  f.sb_rows = kf->cfg.sb_rows;
  if (kf->cfg.dering) {
    const size_t nsb = (size_t)F * kf->nhsb * kf->nvsb;
    KF_CHECK(dalloc(kf, &kf->dering_level, nsb));
    KF_CHECK(dalloc(kf, &kf->dering_thr[0], nsb));
    KF_CHECK(dalloc(kf, &kf->dering_thr[1], nsb));
    KF_CHECK(dalloc(kf, &kf->dering_dir, nsb * 64));
    KF_CHECK(dalloc(kf, &kf->dering_skip, nsb * 256 + 64));
    for (int p = 0; p < 3; p++) {
      const size_t n = (size_t)kf->plane_w[p] * kf->plane_h[p] * F;
      KF_CHECK(dalloc(kf, &kf->dering_in[p], n));
      KF_CHECK(dalloc(kf, &kf->dering_out[p], n));
    }
    if (kf->cfg.dering == 2) {
      KF_CHECK(dalloc(kf, &kf->dering_orig, nsb * 4096));
      KF_CHECK(dalloc(kf, &kf->dering_cand, nsb * 4096));
      KF_CHECK(dalloc(kf, &kf->dering_dist, nsb * 6));
    }
    // thresholds per level: (int)(OD_DERING_GAIN_TABLE[gi] * pow(quantizer, 0.84182) * (luma ? 1 : 0.6)), src/encode.c:2697,2822
    const double gain[6] = {0, 0.5, 0.707, 1, 1.41, 2};
    const double base = pow((double)kf->cfg.q0, 0.84182);
    for (int g = 0; g < 6; g++) {
      kf->dering_tbl[0][g] = (int)(gain[g] * base * 1);
      kf->dering_tbl[1][g] = (int)(gain[g] * base * 0.6);
    }
  }
  // dalloc's cudaMemset runs on the legacy default stream, asynchronously, and the engine's stream does not
  // synchronise with it (cudaStreamNonBlocking): wait for every clear before anything is launched -- the table
  // fill below used to race with the clear of its own buffer (intermittently all-zero 1/sqrt table)
  KF_CHECK(cudaDeviceSynchronize());
  k_fill_rsqrt<<<(kTableDoubles + 255) / 256, 256, 0, kf->stream>>>(kf->rsqrt_tbl);
  KF_CHECK(cudaGetLastError());
  KF_CHECK(cudaStreamSynchronize(kf->stream));
  return 0;
}

// Everything between "inputs are in HBM" and "results are in HBM", on kf->stream.
// the three phase kernels over every chunk of every class of a stage's dependency-free lists
template <bool kZeroRef>
static void enqueue_split(daala_b200_kf* kf, const Stage& S, cudaStream_t s) {
  const int grid = kf->sms * 16;
  for (int cls = 2; cls >= 0; cls--) {
    for (int chunk = 0; chunk < S.sp_chunks[cls]; chunk++) {
      if (cls == 2) {
        k_pvq_split<0, kZeroRef, 2><<<grid, 128, 0, s>>>(S, cls, chunk);
        k_pvq_split<1, kZeroRef, 2><<<grid, 128, 0, s>>>(S, cls, chunk);
        k_pvq_split<2, kZeroRef, 2><<<grid, 128, 0, s>>>(S, cls, chunk);
      } else {
        k_pvq_split<0, kZeroRef, 1><<<grid, 128, 0, s>>>(S, cls, chunk);
        k_pvq_split<1, kZeroRef, 1><<<grid, 128, 0, s>>>(S, cls, chunk);
        k_pvq_split<2, kZeroRef, 1><<<grid, 128, 0, s>>>(S, cls, chunk);
      }
    }
  }
}

static int kf_enqueue_step(daala_b200_kf* kf, int phases) {
  cudaStream_t s = kf->stream;
  const Lists& L = kf->lists;
  const int wide = kf->sms * 8;
  if (phases & DAALA_B200_KF_LISTS) {
    k_unit_tile_sums<<<L.ntiles, kTile, 0, s>>>(L);
    k_tile_scan<<<1, 1024, 0, s>>>(L);
    k_unit_emit<<<L.ntiles, kTile, 0, s>>>(L);
    const size_t nl = (size_t)L.max_luma * sizeof(int32_t);
    if (cudaMemsetAsync(L.succ_bottom, 0xff, nl, s) != cudaSuccess || cudaMemsetAsync(L.succ_right, 0xff, nl, s) != cudaSuccess)
      return (int)cudaGetLastError();
    if (L.lvl_hist && cudaMemsetAsync(L.lvl_hist, 0, sizeof(int32_t) * kLevelBins, s) != cudaSuccess) return (int)cudaGetLastError();
    k_luma_deps<<<wide, 256, 0, s>>>(L);
    if (L.lvl_hist) {
      k_level_scan<<<1, 1024, 0, s>>>(L);
      k_level_scatter<<<wide, 256, 0, s>>>(L);
    }
    k_chroma_items<<<wide, 256, 0, s>>>(L);
  }
  if (phases & DAALA_B200_KF_FORWARD) {
    int rc = daala_b200_launch_forward(&kf->frame, 3, s);
    if (rc) return rc;
  }
  const int persist = kf->sms * (kf->cfg.persist_ctas_per_sm > 0 ? kf->cfg.persist_ctas_per_sm : kPersistCtas);
  // _SEARCH_ONLY (measurement): just the persistent search kernels, on the coding-order buffers a
  // previous full pass left behind (same inputs, same results)
  const bool core = (phases & DAALA_B200_KF_SEARCH_ONLY) != 0;
  if (phases & DAALA_B200_KF_PVQ_LUMA) {
    if (cudaMemsetAsync(kf->luma.ring, 0xff, kf->chain_cap * sizeof(uint32_t), s) != cudaSuccess ||
        cudaMemsetAsync(kf->luma.join0, 0, (size_t)kf->luma.max_blocks * sizeof(int32_t), s) != cudaSuccess)
      return (int)cudaGetLastError();
    k_begin_pvq<<<1, 32, 0, s>>>(kf->lists.cnt, 1);
    if (!core) k_gather<false><<<wide, 256, 0, s>>>(kf->luma);
    if (kf->cfg.split_free > 1) enqueue_split<true>(kf, kf->luma, s);
    if (kf->luma.pre_ev) {
      k_pvq_prepass<2><<<kf->sms * 16, 128, 0, s>>>(kf->luma);
      k_pvq_prepass<1><<<kf->sms * 16, 128, 0, s>>>(kf->luma);
    }
    if (kf->cfg.level_chains) {
      if (cudaMemsetAsync(kf->lv_bar, 0, sizeof(int32_t) * 32, s) != cudaSuccess) return (int)cudaGetLastError();
      k_pvq_levels<<<kf->lvl_grid, 128, 0, s>>>(kf->luma);
    } else {
      k_pvq_persist<true><<<persist, kPersistThreads, 0, s>>>(kf->luma);
    }
    if (!core) k_finish_scatter<<<wide, 256, 0, s>>>(kf->luma);
  }
  if (phases & DAALA_B200_KF_PVQ_CHROMA) {
    k_begin_pvq<<<1, 32, 0, s>>>(kf->lists.cnt, 0);
    if (!core) k_cfl_plane<<<wide, 256, 0, s>>>(kf->chroma, kf->cfl_plane);
    if (!core) k_gather<true><<<wide, 256, 0, s>>>(kf->chroma);
    if (kf->cfg.split_free > 0) enqueue_split<false>(kf, kf->chroma, s);
    else k_pvq_persist<false><<<persist, kPersistThreads, 0, s>>>(kf->chroma);
    if (!core) k_finish_scatter<<<wide, 256, 0, s>>>(kf->chroma);
  }
  if ((phases & DAALA_B200_KF_INVERSE) && !kf->cfg.dering) {
    int rc = daala_b200_launch_inverse(&kf->frame, 3, s);
    if (rc) return rc;
  }
  if ((phases & DAALA_B200_KF_INVERSE) && kf->cfg.dering) {
    // iDCT + split postfilters -> lapped planes; SB-edge postfilter -> etmp (int16, the fused kernel's optional
    // output); od_dering of all frames per plane in one launch, luma first (it writes the direction map chroma
    // reads); -> u8
    int rc = daala_b200_launch_inverse_lapped_only(&kf->frame, 3, s);
    if (rc) return rc;
    daala_b200_frame f16 = kf->frame;
    for (int p = 0; p < 3; p++) f16.post16[p] = kf->dering_in[p];
    rc = daala_b200_launch_sb_postfilter_store(&f16, 3, s);
    if (rc) return rc;
    const int nsb = kf->nhsb * kf->nvsb;
    const bool search = kf->cfg.dering == 2;
    if (search) {
      // the level search of src/encode.c:2708-2811 for every frame of the batch: levels -> kf->dering_level
      daala_b200_dering_search_batch sb;
      memset(&sb, 0, sizeof(sb));
      sb.etmp = kf->dering_in[0];
      sb.src = kf->pixels[0];
      sb.etmp_pitch = sb.src_pitch = (long long)kf->plane_w[0] * kf->plane_h[0];
      sb.etmp_stride = sb.src_stride = kf->plane_w[0];
      sb.nframes = kf->F;
      sb.nhsb = kf->nhsb;
      sb.nvsb = kf->nvsb;
      for (int g = 0; g < 6; g++) sb.threshold[g] = kf->dering_tbl[0][g];
      sb.coded_quantizer = kf->cfg.coded_quantizer;
      sb.qm_is_flat = kf->cfg.qm_is_flat;
      sb.use_activity_masking = kf->cfg.use_masking;
      sb.dering_lambda = kf->cfg.dering_lambda;
      sb.filt = kf->dering_out[0];     // free until the final application below overwrites it
      sb.orig = kf->dering_orig;
      sb.cand = kf->dering_cand;
      sb.dir = kf->dering_dir;
      sb.zskip = kf->dering_skip;
      sb.dist = kf->dering_dist;
      sb.levels = kf->dering_level;
      rc = daala_b200_dering_search_enqueue(&sb, s);
      if (rc) return rc;
    }
    k_dering_thresholds<<<(kf->F * nsb + 255) / 256, 256, 0, s>>>(
        kf->dering_level, kf->dering_thr[0], kf->dering_thr[1], kf->F * nsb,
        make_int4(kf->dering_tbl[0][0], kf->dering_tbl[0][1], kf->dering_tbl[0][2], kf->dering_tbl[0][3]),
        make_int2(kf->dering_tbl[0][4], kf->dering_tbl[0][5]),
        make_int4(kf->dering_tbl[1][0], kf->dering_tbl[1][1], kf->dering_tbl[1][2], kf->dering_tbl[1][3]),
        make_int2(kf->dering_tbl[1][4], kf->dering_tbl[1][5]));
    for (int p = 0; p < 3; p++) {
      const long long per = (long long)kf->plane_w[p] * kf->plane_h[p];
      daala_b200_dering_params dp;
      memset(&dp, 0, sizeof(dp));
      dp.y = kf->dering_out[p];
      dp.x = kf->dering_in[p];
      dp.dir = kf->dering_dir;
      dp.bskip = kf->dering_skip;
      dp.sb_threshold = kf->dering_thr[p ? 1 : 0];
      dp.ystride = dp.xstride = kf->plane_w[p];
      dp.dir_stride = kf->nhsb * 8;
      dp.skip_stride = kf->nhsb * 16;
      dp.nhsb = kf->nhsb;
      dp.nvsb = kf->nvsb;
      dp.xdec = p ? 1 : 0;
      dp.pli = p;
      dp.threshold = 0;
      dp.overlap = 1;      // OD_DERING_CHECK_OVERLAP
      dp.coeff_shift = 4;  // OD_COEFF_SHIFT
      dp.dir_format = search ? 2 : 0;   // after a search the direction map is already there (packed with the variance)
      rc = daala_b200_dering_plane_batch(&dp, kf->F, per, per, (long long)nsb * 64, nsb, s);
      if (rc) return rc;
    }
    for (int p = 0; p < 3; p++)
      k_i16_to_u8<<<wide, 256, 0, s>>>(kf->dering_out[p], kf->pixels_out[p], (long)kf->plane_w[p] * kf->plane_h[p] * kf->F);
  }
  return (int)cudaGetLastError();
}

extern "C" {

daala_b200_kf* daala_b200_kf_create(const daala_b200_kf_config* cfg) {
  if (!cfg || cfg->pic_w <= 0 || cfg->pic_h <= 0 || cfg->nframes <= 0 || cfg->nframes > 255 || !cfg->qm ||
      !cfg->qm_inv || cfg->qm_stride <= 0)
    return nullptr;
  daala_b200_kf* kf = (daala_b200_kf*)calloc(1, sizeof(daala_b200_kf));
  if (!kf) return nullptr;
  kf->cfg = *cfg;
  if (kf->cfg.level_chains && kf->cfg.split_free < 2) kf->cfg.split_free = 2;   // the level kernel only walks the chains
  kf->nhsb = (cfg->pic_w + 63) / 64;
  kf->nvsb = (cfg->pic_h + 63) / 64;
  kf->F = cfg->nframes;
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
    free(kf);
    return nullptr;
  }
  int dev = 0;
  cudaDeviceProp prop;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    free(kf);
    return nullptr;
  }
  kf->sms = prop.multiProcessorCount;
  if (cfg->stream) {
    kf->stream = (cudaStream_t)cfg->stream;
  } else {
    if (cudaStreamCreateWithFlags(&kf->stream, cudaStreamNonBlocking) != cudaSuccess) {
      free(kf);
      return nullptr;
    }
    kf->own_stream = true;
  }
  if (kf_alloc(kf) != 0) {
    fprintf(stderr, "daala_b200_kf_create: %s\n", kf->err);
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
  for (int p = 0; p < 3; p++) {
    cudaFree(kf->pixels[p]);
    cudaFree(kf->coeffs[p]);
    cudaFree(kf->lapped[p]);
    cudaFree(kf->pixels_out[p]);
  }
  cudaFree(kf->bsize);
  cudaFree(kf->cfl_plane);
  cudaFree(kf->qm);
  cudaFree(kf->qm_inv);
  cudaFree(kf->rsqrt_tbl);
  for (int c = 0; c < 3; c++) {
    cudaFree(kf->sp_vec[c]);
    cudaFree(kf->sp_lanes[c]);
    cudaFree(kf->sp_uni[c]);
    cudaFree(kf->sp_snap[c]);
  }
  Lists& L = kf->lists;
  cudaFree(L.tile_sum);
  cudaFree(L.unit_lbase);
  cudaFree(L.luma);
  cudaFree(L.chroma);
  cudaFree(L.dep_top);
  cudaFree(L.dep_left);
  for (int c = 0; c < 3; c++) {
    cudaFree(L.items_l[c]);
    cudaFree(L.items_c[c]);
  }
  cudaFree(L.heads);
  cudaFree(L.heads0);
  cudaFree(L.lvl_hist);
  cudaFree(L.lvl_cursor);
  cudaFree(L.lvl_items);
  cudaFree(kf->lv_vec);
  cudaFree(kf->lv_lanes);
  cudaFree(kf->lv_uni);
  cudaFree(kf->lv_snap);
  cudaFree(kf->lv_bar);
  cudaFree(kf->dering_level);
  cudaFree(kf->dering_orig);
  cudaFree(kf->dering_cand);
  cudaFree(kf->dering_dist);
  cudaFree(kf->dering_thr[0]);
  cudaFree(kf->dering_thr[1]);
  cudaFree(kf->dering_dir);
  cudaFree(kf->dering_skip);
  for (int p = 0; p < 3; p++) {
    cudaFree(kf->dering_in[p]);
    cudaFree(kf->dering_out[p]);
  }
  cudaFree(L.succ_bottom);
  cudaFree(L.succ_right);
  cudaFree(L.cnt);
  for (Stage* S : {&kf->luma, &kf->chroma}) {
    cudaFree(S->prm.in);
    cudaFree(S->prm.ref);
    cudaFree(S->prm.out);
    cudaFree(S->prm.y);
    cudaFree(S->prm.y16);
    cudaFree(S->prm.res_skip_term);
    cudaFree(S->prm.res_skip_diff);
    cudaFree(S->prm.res_flip);
    cudaFree(S->res_pack);
    cudaFree(S->ring);
    cudaFree(S->join0);
    cudaFree(S->pre_ev);
    cudaFree(S->pre_snap);
  }
  if (kf->own_stream) cudaStreamDestroy(kf->stream);
  free(kf);
}

const char* daala_b200_kf_error(const daala_b200_kf* kf) { return kf ? kf->err : "null engine"; }

// Kernel launches of one whole step (kf_enqueue_step with DAALA_B200_KF_ALL), memset nodes not counted.
int daala_b200_kf_launches_per_step(const daala_b200_kf* kf) {
  if (!kf) return 0;
  auto split = [](const Stage& S) { return 3 * (S.sp_chunks[0] + S.sp_chunks[1] + S.sp_chunks[2]); };
  int n = 5 + (kf->cfg.level_chains ? 2 : 0);                                    // work lists
  n += 1;                                                                         // forward
  n += 3 + 1 + (kf->cfg.split_free > 1 ? split(kf->luma) : 0) + (kf->luma.pre_ev ? 2 : 0);   // luma: begin, gather, [prepass], chains, finish
  n += 4 + (kf->cfg.split_free > 0 ? split(kf->chroma) : 1);                      // chroma: begin, cfl, gather, bands, finish
  if (!kf->cfg.dering) n += 2;                                                    // inverse, SB postfilter + store
  else n += 1 + 1 + 1 + 3 + 3;   // inverse, SB postfilter -> int16, thresholds, dering per plane, store
  if (kf->cfg.dering == 2) n += 5 + 6 + 6 + 1;   // level search: 5 filtered candidates, 6 packs, 6 distortion passes, decision
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
    KF_CHECK(cudaGraphInstantiate(&kf->exec, kf->graph, 0));
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

// With level_chains the compute phases of different engines never overlap on the device: the level kernel
// synchronises its whole grid and needs every CTA resident, which two such kernels in flight could deny
// each other.  Copies of one
// engine still overlap the compute of another (that is what double buffering is for).
static std::mutex g_compute_mu;
static cudaEvent_t g_last_compute = nullptr;

int daala_b200_kf_submit(daala_b200_kf* kf, const daala_b200_kf_io* io) {
  if (!kf || !io) return (int)cudaErrorInvalidValue;
  cudaStream_t s = kf->stream;
  const int F = kf->F;
  for (int p = 0; p < 3; p++) {
    if (!io->pixels[p]) return (int)cudaErrorInvalidValue;
    KF_CHECK(cudaMemcpyAsync(kf->pixels[p], io->pixels[p], (size_t)kf->plane_w[p] * kf->plane_h[p] * F,
                             cudaMemcpyHostToDevice, s));
  }
  const size_t map_bytes = (size_t)kf->nhsb * 8 * kf->nvsb * 8 * F;
  KF_CHECK(cudaMemcpyAsync(kf->bsize, io->bsize, map_bytes, cudaMemcpyHostToDevice, s));
  if (kf->cfg.dering == 1) {
    if (!io->dering_level) return (int)cudaErrorInvalidValue;
    KF_CHECK(cudaMemcpyAsync(kf->dering_level, io->dering_level, (size_t)kf->nhsb * kf->nvsb * F, cudaMemcpyHostToDevice, s));
  }
  int rc;
  {
    std::lock_guard<std::mutex> lock(g_compute_mu);
    if (!g_last_compute) KF_CHECK(cudaEventCreateWithFlags(&g_last_compute, cudaEventDisableTiming));
    else if (kf->cfg.level_chains) KF_CHECK(cudaStreamWaitEvent(s, g_last_compute, 0));
    rc = daala_b200_kf_run_device(kf, DAALA_B200_KF_ALL, 1);
    if (rc) return rc;
    KF_CHECK(cudaEventRecord(g_last_compute, s));
  }
  daala_b200_kf_totals tot;
  if (io->totals) tot = *io->totals;
  else daala_b200_kf_count_blocks(io->bsize, F, (long long)kf->nhsb * 8 * kf->nvsb * 8, kf->nhsb * 8, kf->nhsb, kf->nvsb,
                                  kf->cfg.sb_row0, kf->cfg.sb_rows, &tot);
  if (tot.n_luma > kf->lists.max_luma || tot.n_chroma > kf->lists.max_chroma) return (int)cudaErrorInvalidValue;
  for (int p = 0; p < 3; p++)
    if (io->pixels_out[p])
      KF_CHECK(cudaMemcpyAsync(io->pixels_out[p], kf->pixels_out[p], (size_t)kf->plane_w[p] * kf->plane_h[p] * F,
                               cudaMemcpyDeviceToHost, s));
  if (io->luma_blocks) KF_CHECK(cudaMemcpyAsync(io->luma_blocks, kf->lists.luma, sizeof(daala_b200_pvq_block) * tot.n_luma, cudaMemcpyDeviceToHost, s));
  if (io->chroma_blocks) KF_CHECK(cudaMemcpyAsync(io->chroma_blocks, kf->lists.chroma, sizeof(daala_b200_pvq_block) * tot.n_chroma, cudaMemcpyDeviceToHost, s));
  if (io->luma_res) KF_CHECK(cudaMemcpyAsync(io->luma_res, kf->luma.res_pack, 8 * 9 * (size_t)tot.n_luma, cudaMemcpyDeviceToHost, s));
  if (io->chroma_res) KF_CHECK(cudaMemcpyAsync(io->chroma_res, kf->chroma.res_pack, 8 * 9 * (size_t)tot.n_chroma, cudaMemcpyDeviceToHost, s));
  if (io->luma_y16) KF_CHECK(cudaMemcpyAsync(io->luma_y16, kf->luma.prm.y16, 2 * (size_t)tot.luma_coefs, cudaMemcpyDeviceToHost, s));
  if (io->chroma_y16) KF_CHECK(cudaMemcpyAsync(io->chroma_y16, kf->chroma.prm.y16, 2 * (size_t)tot.chroma_coefs, cudaMemcpyDeviceToHost, s));
  if (io->luma_skip_diff) KF_CHECK(cudaMemcpyAsync(io->luma_skip_diff, kf->luma.prm.res_skip_diff, 8 * (size_t)tot.n_luma, cudaMemcpyDeviceToHost, s));
  if (io->chroma_skip_diff) KF_CHECK(cudaMemcpyAsync(io->chroma_skip_diff, kf->chroma.prm.res_skip_diff, 8 * (size_t)tot.n_chroma, cudaMemcpyDeviceToHost, s));
  if (io->chroma_flip) KF_CHECK(cudaMemcpyAsync(io->chroma_flip, kf->chroma.prm.res_flip, 4 * (size_t)tot.n_chroma, cudaMemcpyDeviceToHost, s));
  if (io->counts) KF_CHECK(cudaMemcpyAsync(io->counts, kf->lists.cnt, sizeof(int32_t) * 32, cudaMemcpyDeviceToHost, s));
  if (io->dering_level_out && kf->cfg.dering)
    KF_CHECK(cudaMemcpyAsync(io->dering_level_out, kf->dering_level, (size_t)kf->nhsb * kf->nvsb * F, cudaMemcpyDeviceToHost, s));
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
