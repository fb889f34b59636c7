// Directional deringing filter of whole planes (reference src/dering.c: od_dering :252 with
// od_dir_find8 :61, od_filter_dering_direction_c :132, od_filter_dering_orthogonal_c :172,
// od_compute_thresh :237) -- SURVEY.md 8(f) rank 1, the row after the transform / PVQ / MC path.
//
// Parity: bit-exact against oracle/port_dering.c (pinned against od_dering) in tests/test_gpu_dering.py and
// tests/test_gpu_dering_kernel.py.
// Consumers: the keyframe engine's deringing stage (csrc/kf_engine.cu, levels given, u8 output) and the level
// search (csrc/dering_search.cu, src/encode.c:2680-2811).
//
// Mapping: one 256-thread CTA per superblock, sized for 4 CTAs per SM (at most 64 registers, no local memory).
//  * The (B+6) x (B+8) int16 window (3-sample apron, 30000 where the frame ends; one spare column each side so
//    that every row is staged as aligned 4-sample groups) is loaded once into shared memory, row by row.
//  * Direction search (luma): every thread scores 2 of the 8 directions of one 8x8 block.  A warp's lanes take
//    32 blocks and the same pair of directions, so the switch that selects the pair's straight-line bodies is
//    warp-uniform and the 15 line sums of a direction stay in registers (compile-time indices).  The 8 costs of
//    a block meet in shared memory, where one thread per block picks the direction.
//  * One thread per block then derives the threshold, the skip decision and the block's tap offsets into the
//    window, so the filter passes read their per-block parameters from shared memory.
//  * The two filter passes run on pairs of adjacent pixels out of shared memory with 32-bit loads and stores
//    (pass 2 reads pass 1's output inside the superblock and the unfiltered apron outside it, as the
//    reference's `in` buffer does).
// HBM traffic is the minimum: every sample is read once (+apron) and written once, as int16 or, for the keyframe
// engine's final application, straight as the u8 reconstruction (od_coeff_to_ref_plane).
#include <cuda_runtime.h>
#include <stdint.h>

#include "daala_b200.h"
#include "dering_search.h"

namespace daala_b200 {
namespace dering {

constexpr int kBorder = 3;              // apron the filter reads on every side
constexpr int kPad = 4;                 // window columns left of the superblock: 4-sample groups stay 8-byte aligned
constexpr int kPitch = 64 + 2 * kPad + 4;   // 76 int16: 8-byte aligned rows, block rows 8 apart on different banks
constexpr int kRows = 64 + 2 * kBorder;
constexpr int kOutside = 30000;

// step k = 1..3 along direction d as (rows, columns); OD_DIRECTION_OFFSETS_TABLE, src/dering.c:39-48
__constant__ signed char kStep[8][3][2] = {
    {{-1, 1}, {-2, 2}, {-3, 3}}, {{0, 1}, {-1, 2}, {-1, 3}}, {{0, 1}, {0, 2}, {0, 3}}, {{0, 1}, {1, 2}, {1, 3}},
    {{1, 1}, {2, 2}, {3, 3}},    {{1, 0}, {2, 1}, {3, 1}},   {{1, 0}, {2, 0}, {3, 0}}, {{1, 0}, {2, -1}, {3, -1}},
};
// OD_THRESH_TABLE_Q8, src/dering.c:225
__constant__ short kThreshQ8[18] = {128, 134, 150, 168, 188, 210, 234, 262, 292, 327, 365, 408, 455, 509, 569, 635, 710, 768};

__host__ __device__ constexpr int line_of(int d, int i, int j) {
  return d == 0 ? i + j : d == 1 ? i + j / 2 : d == 2 ? i : d == 3 ? 3 + i - j / 2 : d == 4 ? 7 + i - j
       : d == 5 ? 3 - i / 2 + j : d == 6 ? j : i / 2 + j;
}

// number of pixels of an 8x8 block on line l of direction d
__host__ __device__ constexpr int line_len(int d, int l) {
  int n = 0;
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 8; j++) n += line_of(d, i, j) == l;
  return n;
}

// Cost of direction D for the 8x8 block at `img` (shared-memory window, pitch kPitch, 8-byte aligned rows): the
// sum over the lines of D of (line sum)^2 * (840 / line length), the integers of od_dir_find8.  Integer sums do
// not depend on the order of the additions.
template <int D>
__device__ __forceinline__ int32_t dir_cost(const int16_t* img, int coeff_shift) {
  int sum[15];
#pragma unroll
  for (int l = 0; l < 15; l++) sum[l] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const uint2 w = *reinterpret_cast<const uint2*>(img + i * kPitch + 4 * h);
      const int v[4] = {(int)(int16_t)(w.x & 0xffff), (int)w.x >> 16, (int)(int16_t)(w.y & 0xffff), (int)w.y >> 16};
#pragma unroll
      for (int k = 0; k < 4; k++) sum[line_of(D, i, 4 * h + k)] += v[k] >> coeff_shift;
    }
  }
  int32_t c = 0;
#pragma unroll
  for (int l = 0; l < 15; l++)
    if (line_len(D, l)) c += sum[l] * sum[l] * (840 / line_len(D, l));
  return c;
}

// one tap of pass 1: |a| < t adds w * a (int16 arithmetic, as the reference)
__device__ __forceinline__ int16_t tap(int16_t acc, int s, int c, int w, int t) {
  const int16_t a = (int16_t)(s - c);
  return abs((int)a) < t ? (int16_t)(acc + w * a) : acc;
}

// pass 1 of one pixel at `s` (window), taps o0..o2 along the direction
__device__ __forceinline__ int16_t pass1(const int16_t* s, int c, int4 tp) {
  int16_t acc = 0;
  acc = tap(acc, s[tp.x], c, 3, tp.w);
  acc = tap(acc, s[-tp.x], c, 3, tp.w);
  acc = tap(acc, s[tp.y], c, 2, tp.w);
  acc = tap(acc, s[-tp.y], c, 2, tp.w);
  acc = tap(acc, s[tp.z], c, 1, tp.w);
  acc = tap(acc, s[-tp.z], c, 1, tp.w);
  return (int16_t)(c + ((acc + 8) >> 4));
}

// pass 2 of one pixel at `s` (pass-1 plane): c its pass-1 value, c0 its input value, o the step across the
// direction, t / t3 the block's threshold and a third of it
__device__ __forceinline__ int16_t pass2(const int16_t* s, int c, int c0, int o, int t, int t3) {
  const int moved = abs(c - c0);
  const int16_t lim = (int16_t)(t3 + moved < t ? t3 + moved : t);
  int16_t acc = 0;
  int16_t q;
  q = (int16_t)(s[o] - c);
  if (abs((int)q) < lim) acc = (int16_t)(acc + q);
  q = (int16_t)(s[-o] - c);
  if (abs((int)q) < lim) acc = (int16_t)(acc + q);
  q = (int16_t)(s[2 * o] - c);
  if (abs((int)q) < lim) acc = (int16_t)(acc + q);
  q = (int16_t)(s[-2 * o] - c);
  if (abs((int)q) < lim) acc = (int16_t)(acc + q);
  return (int16_t)(c + ((3 * acc + 8) >> 4));
}

// (c + 8 >> 4) + 128 clamped: od_coeff_to_ref_plane, src/state.c:1283
__device__ __forceinline__ uint32_t to_u8(int v) {
  v = ((v + 8) >> 4) + 128;
  return (uint32_t)(v < 0 ? 0 : v > 255 ? 255 : v);
}

__device__ __forceinline__ int lo16(uint32_t w) { return (int)(int16_t)(w & 0xffff); }
__device__ __forceinline__ int hi16(uint32_t w) { return (int)w >> 16; }

// frames of a batch: blockIdx.z, element pitches between consecutive frames (all zero for a single plane);
// y8 (nullable): store the u8 reconstruction there (pitch y, stride ystride) instead of the int16 plane y;
// skip: pitch of the skip map (0: one map for every frame)
struct BatchPitch {
  long long y, x, dir, thr;
  uint8_t* y8;
  long long skip;
};

__global__ void __launch_bounds__(256, 4) k_dering_sb(const __grid_constant__ daala_b200_dering_params p,
                                                      const __grid_constant__ BatchPitch bp) {
  __shared__ __align__(16) int16_t win[kRows * kPitch];   // unfiltered input + apron
  __shared__ __align__(16) int16_t mid[kRows * kPitch];   // pass-1 output inside the superblock, input in the apron
  __shared__ int32_t s_cost[8][64];                       // direction search: cost[d][block]
  __shared__ int4 s_tap[64];                              // per block: pass-1 offsets o0..o2, threshold
  __shared__ int2 s_orth[64];                             // per block: pass-2 offset, threshold / 3
  const int sbx = blockIdx.x, sby = blockIdx.y, z = blockIdx.z;
  const int lb = 3 - p.xdec, lgB = 6 - p.xdec, B = 1 << lgB;
  const int16_t* x = p.x + z * bp.x + (size_t)sby * B * p.xstride + (size_t)sbx * B;
  int32_t* dir = p.dir + z * bp.dir;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // stage the window: row r holds input row r - 3, column c input column c - 4; one lane per 4-sample group.
  // Groups never straddle the superblock's edges, so a group is wholly inside or wholly outside the frame.
  {
    const bool top = sby != 0, bottom = sby != p.nvsb - 1, left = sbx != 0, right = sbx != p.nhsb - 1;
    const bool vec = ((uintptr_t)p.x & 7) == 0 && (p.xstride & 3) == 0 && (bp.x & 3) == 0;
    const int groups = (B >> 2) + 2;
    const int j = (lane << 2) - kPad;
    const bool col_in = j < 0 ? left : j >= B ? right : true;
    const bool col_apron = j < 0 || j >= B;
    for (int r = warp; r < B + 2 * kBorder && lane < groups; r += 8) {
      const int i = r - kBorder;
      const bool inside = col_in && (i < 0 ? top : i >= B ? bottom : true);
      uint2 v = make_uint2(((uint32_t)kOutside << 16) | kOutside, ((uint32_t)kOutside << 16) | kOutside);
      if (inside) {
        const int16_t* src = x + (ptrdiff_t)i * p.xstride + j;
        if (vec) {
          v = *reinterpret_cast<const uint2*>(src);
        } else {
          v.x = (uint16_t)src[0] | ((uint32_t)(uint16_t)src[1] << 16);
          v.y = (uint16_t)src[2] | ((uint32_t)(uint16_t)src[3] << 16);
        }
      }
      *reinterpret_cast<uint2*>(win + r * kPitch + (lane << 2)) = v;
      if (col_apron || i < 0 || i >= B) *reinterpret_cast<uint2*>(mid + r * kPitch + (lane << 2)) = v;
    }
  }
  __syncthreads();
  const int16_t* in = win + kBorder * kPitch + kPad;
  int16_t* in2 = mid + kBorder * kPitch + kPad;

  // direction search: warp w scores directions (w & 3) and (w & 3) + 4 of blocks 32 * (w >> 2) + lane
  const bool search = p.pli == 0 && p.dir_format != 2;
  if (search) {
    const int blk = ((warp >> 2) << 5) | lane, q = warp & 3;
    const int16_t* img = in + (blk >> 3) * 8 * kPitch + (blk & 7) * 8;
    int32_t lo, hi;
    switch (q) {
      case 0: lo = dir_cost<0>(img, p.coeff_shift); hi = dir_cost<4>(img, p.coeff_shift); break;
      case 1: lo = dir_cost<1>(img, p.coeff_shift); hi = dir_cost<5>(img, p.coeff_shift); break;
      case 2: lo = dir_cost<2>(img, p.coeff_shift); hi = dir_cost<6>(img, p.coeff_shift); break;
      default: lo = dir_cost<3>(img, p.coeff_shift); hi = dir_cost<7>(img, p.coeff_shift); break;
    }
    s_cost[q][blk] = lo;
    s_cost[q + 4][blk] = hi;
    __syncthreads();
  }

  // per block: direction, threshold, skip decision, tap offsets
  if (threadIdx.x < 64) {
    const int by = threadIdx.x >> 3, bx = threadIdx.x & 7;
    int32_t* dslot = dir + (size_t)(sby * 8 + by) * p.dir_stride + sbx * 8 + bx;
    const int base = p.sb_threshold ? p.sb_threshold[z * bp.thr + sby * p.nhsb + sbx] : p.threshold;
    int d, thr;
    if (p.pli == 0) {
      int32_t var;
      if (search) {
        // the first direction whose cost is strictly greater, from a best cost of 0 (od_dir_find8)
        int32_t best_cost = 0, opp = s_cost[4][threadIdx.x];
        d = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) {
          const int32_t c = s_cost[k][threadIdx.x];
          if (c > best_cost) {
            best_cost = c;
            d = k;
            opp = s_cost[(k + 4) & 7][threadIdx.x];
          }
        }
        var = (best_cost - opp) >> 10;
        *dslot = p.dir_format == 1 ? (d | (var << 3)) : d;
      } else {
        // direction and variance of an earlier pass over the same input (the level search filters one plane
        // five times, and the final application a sixth)
        const int packed = *dslot;
        d = packed & 7;
        var = packed >> 3;
      }
      int v = var >> 6;
      if (v > 32767) v = 32767;
      const int lg = v ? 32 - __clz(v) : 0;
      thr = (base * kThreshQ8[lg] + 128) >> 8;
    } else {
      d = p.dir_format ? (*dslot & 7) : *dslot;
      thr = base;
    }
    // skipped neighbourhood -> untouched (DAALA_ODINTRIN form, src/dering.c:298-318)
    int u0 = 0, v0 = 0, u1 = 2 >> p.xdec, v1 = 2 >> p.xdec;
    if (p.overlap) {
      u0 -= sbx != 0;
      v0 -= sby != 0;
      u1 += sbx != p.nhsb - 1;
      v1 += sby != p.nvsb - 1;
    }
    // per-plane skip flags, one per 4x4 block of THIS plane: 16 >> xdec flags per superblock side
    // (call site src/encode.c:2789-2791)
    const uint8_t* sk = p.bskip + z * bp.skip + (size_t)(sby * (16 >> p.xdec)) * p.skip_stride + sbx * (16 >> p.xdec);
    bool all = true;
    for (int i = v0; i < v1; i++)
      for (int j = u0; j < u1; j++) all = all && sk[(ptrdiff_t)(((by << 1) >> p.xdec) + i) * p.skip_stride + ((bx << 1) >> p.xdec) + j];
    if (all) thr = 0;
    s_tap[threadIdx.x] = make_int4(kStep[d][0][0] * kPitch + kStep[d][0][1], kStep[d][1][0] * kPitch + kStep[d][1][1],
                                   kStep[d][2][0] * kPitch + kStep[d][2][1], thr);
    s_orth[threadIdx.x] = make_int2((d > 0 && d < 4) ? kPitch : 1, thr / 3);
  }
  __syncthreads();

  // pass 1: along the direction, taps 3 2 1 on either side; pixel pairs (i, j), (i, j + 1)
  const int pair_shift = lgB - 1;
  for (int g = threadIdx.x; g < (B * B >> 1); g += 256) {
    const int i = g >> pair_shift, j = (g & ((B >> 1) - 1)) << 1;
    const int4 tp = s_tap[((i >> lb) << 3) | (j >> lb)];
    const int16_t* s = in + i * kPitch + j;
    const uint32_t cw = *reinterpret_cast<const uint32_t*>(s);
    const int16_t r0 = pass1(s, lo16(cw), tp), r1 = pass1(s + 1, hi16(cw), tp);
    *reinterpret_cast<uint32_t*>(in2 + i * kPitch + j) = (uint16_t)r0 | ((uint32_t)(uint16_t)r1 << 16);
  }
  __syncthreads();

  // pass 2: across it, four unit taps with the tighter, change-dependent threshold
  const size_t frame_y = (size_t)z * bp.y + (size_t)sby * B * p.ystride + (size_t)sbx * B;
  uint8_t* y8 = bp.y8 ? bp.y8 + frame_y : nullptr;
  int16_t* y16 = bp.y8 ? nullptr : p.y + frame_y;
  const bool even = (p.ystride & 1) == 0 && (bp.y & 1) == 0 &&
                    (bp.y8 ? ((uintptr_t)bp.y8 & 1) == 0 : ((uintptr_t)p.y & 3) == 0);
  for (int g = threadIdx.x; g < (B * B >> 1); g += 256) {
    const int i = g >> pair_shift, j = (g & ((B >> 1) - 1)) << 1;
    const int blk = ((i >> lb) << 3) | (j >> lb);
    const int t = s_tap[blk].w;
    const int2 oq = s_orth[blk];
    const int16_t* s = in2 + i * kPitch + j;
    const uint32_t cw = *reinterpret_cast<const uint32_t*>(s);
    const uint32_t c0w = *reinterpret_cast<const uint32_t*>(in + i * kPitch + j);
    const int16_t r0 = pass2(s, lo16(cw), lo16(c0w), oq.x, t, oq.y);
    const int16_t r1 = pass2(s + 1, hi16(cw), hi16(c0w), oq.x, t, oq.y);
    const size_t at = (size_t)i * p.ystride + j;
    if (y8) {
      const uint32_t u0 = to_u8(r0), u1 = to_u8(r1);
      if (even) {
        *reinterpret_cast<uint16_t*>(y8 + at) = (uint16_t)(u0 | (u1 << 8));
      } else {
        y8[at] = (uint8_t)u0;
        y8[at + 1] = (uint8_t)u1;
      }
    } else if (even) {
      *reinterpret_cast<uint32_t*>(y16 + at) = (uint16_t)r0 | ((uint32_t)(uint16_t)r1 << 16);
    } else {
      y16[at] = r0;
      y16[at + 1] = r1;
    }
  }
}

}  // namespace dering
}  // namespace daala_b200

// `nframes` planes of one geometry in one launch (internal: the keyframe engine's deringing stage, the P-frame
// finishing pass and the level search; the exported entry points below are its single-plane and one-skip-map forms).
// Element pitches between consecutive frames; skip_pitch: bytes between the frames' skip maps (0: one map for every
// frame, as on keyframes).  y8 (nullable): write the u8 reconstruction od_coeff_to_ref_plane makes of the filtered
// plane there, with the int16 plane's strides, instead of the int16 plane (prm->y may then be null).
int daala_b200_dering_plane_frames(const daala_b200_dering_params* prm, int nframes, long long y_pitch,
                                   long long x_pitch, long long dir_pitch, long long thr_pitch, long long skip_pitch,
                                   uint8_t* y8, void* stream) {
  if (!prm || nframes < 1 || prm->nhsb < 1 || prm->nvsb < 1 || prm->xdec < 0 || prm->xdec > 1) return (int)cudaErrorInvalidValue;
  // not in place: a superblock's apron would read its neighbours' filtered output
  if (!prm->x || (!prm->y && !y8) || (const void*)prm->x == (const void*)prm->y) return (int)cudaErrorInvalidValue;
  dim3 grid(prm->nhsb, prm->nvsb, nframes);
  daala_b200::dering::BatchPitch bp = {y_pitch, x_pitch, dir_pitch, thr_pitch, y8, skip_pitch};
  daala_b200::dering::k_dering_sb<<<grid, 256, 0, (cudaStream_t)stream>>>(*prm, bp);
  return (int)cudaGetLastError();
}

extern "C" int daala_b200_dering_plane(const daala_b200_dering_params* prm, void* stream) {
  if (prm && !prm->y) return (int)cudaErrorInvalidValue;
  return daala_b200_dering_plane_frames(prm, 1, 0, 0, 0, 0, 0, nullptr, stream);
}

// The batch with one skip map for every frame.
extern "C" int daala_b200_dering_plane_batch(const daala_b200_dering_params* prm, int nframes, long long y_pitch,
                                             long long x_pitch, long long dir_pitch, long long thr_pitch, uint8_t* y8,
                                             void* stream) {
  return daala_b200_dering_plane_frames(prm, nframes, y_pitch, x_pitch, dir_pitch, thr_pitch, 0, y8, stream);
}
