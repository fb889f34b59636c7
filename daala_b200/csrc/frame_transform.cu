// Fused lapped-transform frame kernels for sm_90a (H100).
//
// Forward  (encoder analysis), one CTA per superblock of one plane:
//   u8 pixels -> (p-128)<<4 -> superblock-edge prefilter -> per split node
//   interior-cross prefilter (top-down) -> leaf fDCT (4..64 points, 2-D)
//   -> keyframe DC Haar pyramid (bottom-up) -> int32 coefficient plane `d`.
//   Restates, for a whole frame in one launch, what the reference does with
//   od_ref_plane_to_coeff (src/state.c:1259) + od_apply_prefilter_frame_sbs
//   (src/filter.c:1529) + od_compute_dcts (src/encode.c:1455).
//
// Inverse (reconstruction), two launches:
//   k_inverse_sb:   d -> inverse DC Haar (top-down) -> leaf iDCT -> split
//                   postfilters (bottom-up) -> int32 plane `c`
//                   (od_block_encode's idct_2d, src/encode.c:1397, and
//                   od_postfilter_split, src/filter.c:1485, for a whole frame)
//   k_sb_postfilter_store: superblock-edge postfilter + clamp to u8
//                   (od_apply_postfilter_frame_sbs src/filter.c:1561 +
//                   od_coeff_to_ref_plane src/state.c:1323).
//
// Work mapping: a 1-D N-point transform is straight-line integer lifting code
// (gen/dct_lifting.cuh) run by ONE thread on N registers; the 2-D transform is
// a column pass and a row pass over a shared-memory tile whose pitch is odd
// (5 mod 32), so both passes are bank-conflict free without a transpose.
// Tensor cores are not used: these are rounding lifting networks, not GEMMs.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "gen/dct_lifting.cuh"
#include "lapped_filter.cuh"
#include "frame_transform.h"
#include "haar.cuh"

namespace daala_b200 {

#ifndef DAALA_XFORM_THREADS
#define DAALA_XFORM_THREADS 64
#endif
// Threads per superblock CTA.  Small CTAs win (measured 256 -> 64: forward 2.05 -> 1.05 ms per
// 16 4K frames): the phases of one superblock are latency chains separated by barriers, so the
// SM is kept busy by MANY independent superblocks (8 CTAs/SM at 128 registers, 26 KB smem each)
// rather than by many warps of one.
constexpr int kThreads = DAALA_XFORM_THREADS;
constexpr int kPostThreads = 128;               // superblock-edge postfilter kernel
constexpr int kCtasPerSm = 512 / kThreads;      // 128 registers per thread
constexpr int kGridCap = 132 * 8;               // grid-stride kernels: 8 CTAs on each of the H100's 132 SMs
constexpr int kMaxB = 64;            // superblock edge in luma pixels
constexpr int kHalo = 2;             // lapping reaches 2 samples across an edge
constexpr int kMaxT = kMaxB + 2 * kHalo;
constexpr int kMaxPitch = kMaxT + 1; // 69 = 5 mod 32; chroma 37 = 5 mod 32

// ---------------------------------------------------------------------------
// TMA staging of the 8-bit input window.  One 3-D tensor map per plane
// (x, y, frame); the (B+4)^2 window of a superblock is fetched by ONE
// cp.async.bulk.tensor issued by thread 0.  The innermost start coordinate of
// a tiled TMA copy must be 16-byte aligned (an unaligned x raises "illegal
// instruction"; measured with tools/probe/tma_probe.cu), so the box
// starts 16 samples left of the superblock and is 96 (luma) / 64 (chroma)
// bytes wide; the window proper begins at byte 14 of each row.  Out-of-frame
// samples are zero filled by the hardware, so frame borders need no branches.
// ---------------------------------------------------------------------------
struct TmaMaps {
  CUtensorMap plane[3];
};

template <int XDEC> struct RawTile {
  static constexpr int B = kMaxB >> XDEC;
  static constexpr int rows = B + 2 * kHalo;
  static constexpr int lead = 16;                                     // aligned start: x0 - 16
  static constexpr int width = ((lead + B + kHalo + 15) / 16) * 16;     // 96 / 64
  static constexpr int skip = lead - kHalo;                            // 14: first window byte
  static constexpr int bytes = rows * width;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(phase) : "memory");
  }
}

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int x, int y, int z, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar)) : "memory");
}

// ---------------------------------------------------------------------------
// Leaf-size lookup for one superblock.  `leaf[v*8+u]` = log2 of the transform
// size, in PLANE pixels, covering the 8x8-luma unit (u, v) of this superblock:
// max(obs, xdec) - xdec + 2 with obs the entry of the reference's
// state->bsize map (OD_BLOCK_SIZE4x4, src/block_size.h; recursion rule
// src/encode.c:1467-1470).
// ---------------------------------------------------------------------------
// B, P and the unit shift are compile-time (kernels are specialised per
// plane decimation) so that all index arithmetic is shifts and constant
// multiplies -- runtime integer division would saturate the XU pipe.
template <int B_, int P_>
struct SbCtxT {
  static constexpr int B = B_;                      // superblock edge in plane pixels (64 >> xdec)
  static constexpr int P = P_;                      // tile pitch in ints
  static constexpr int ushift = (B_ == 64) ? 3 : 2; // plane pixels -> 8x8-luma unit: 3 - xdec
  static constexpr int logB = (B_ == 64) ? 6 : 5;
  int x0, y0;   // plane coordinates of the superblock origin
};

// Per-superblock work lists, built once in shared memory from the block-size
// map so that every later phase iterates over exactly its active items (no
// per-item quadtree lookups, no idle iterations):
//   blk[c][..]  leaf blocks of transform size 4 << c (c = 0..4), position packed (y << 8 | x)
//   node[l][..] split nodes of edge 8 << l (l = 0..3), with their filter gates
// Leaf sizes follow od_compute_dcts (src/encode.c:1466-1470): bs = max(obs, xdec)
// read at the block's top-left corner of the reference's state->bsize map.
struct SbLists {
  unsigned short blk[256 + 64 + 16 + 4 + 1];
  unsigned short node[64 + 16 + 4 + 1];
  int nblk[5];
  int nnode[4];
  unsigned char wcnt[8][9];  // per-(virtual-)warp counts while the lists are being built
};
__device__ __forceinline__ constexpr int blk_base(int c) { return c == 0 ? 0 : c == 1 ? 256 : c == 2 ? 320 : c == 3 ? 336 : 340; }
// 0, 64, 80, 84: one byte per level (a select chain costs four instructions where l is a run-time value)
__device__ __forceinline__ constexpr int node_base(int l) { return (int)((0x54504000u >> (8 * l)) & 0xffu); }
constexpr unsigned short kGateH = 0x4000;  // hfilter allowed (node inside the picture horizontally)
constexpr unsigned short kGateV = 0x8000;  // vfilter allowed

// Must be called by all threads; ends with the lists visible to the CTA.
// One thread per 8x8-luma unit of the superblock (64 units, warps 0 and 1): the leaf / split-node flags of a
// unit follow from its own block-size entry and its alignment, so nine ballots give the rank inside the warp
// and one count of warp 0 the offset of warp 1.  A luma unit coded as 4x4 blocks emits its four leaves.
template <int XDEC>
__device__ __forceinline__ void build_lists(SbLists& L, const unsigned char* bsize, int bstride, int sbx,
                                            int sby, int x0, int y0, int pic_w, int pic_h) {
  static_assert(kThreads >= 64, "one thread per 8x8-luma unit");
  constexpr int B = kMaxB >> XDEC;
  constexpr int USZ = 8 >> XDEC;                 // unit edge in plane pixels
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int bx = t & 7, by = (t >> 3) & 7;
  unsigned flags = 0;
  unsigned rank[9];
  if (t < 64) {
    const int obs = bsize[(sby * 8 + by) * bstride + sbx * 8 + bx];
    const int c = (obs > XDEC ? obs : XDEC) - XDEC;   // log2(n) - 2 of the leaf covering this unit
    const unsigned lt = (1u << lane) - 1u;
    const int xy = bx | by;
    // category 0..4: leaf origin of class c; 5..8: split node of edge 8 << (cat - 5)
#pragma unroll
    for (int cat = 0; cat < 9; cat++) {
      bool f;
      if (cat < 5) {
        // leaf edge 4 << cat pixels = this many units (a 4x4 luma leaf is half a unit: every unit qualifies)
        const int a = XDEC ? (1 << cat) : (cat ? (1 << (cat - 1)) : 1);
        f = c == cat && !(xy & (a - 1));
      } else {
        // a node exists at positions aligned to its size and is split iff the leaf at its corner is
        // smaller (src/encode.c:1466: the block size is read at the corner)
        const int l = cat - 5, S = 8 << l;
        const int a = XDEC ? (2 << l) : (1 << l);
        f = S <= B && !(xy & (a - 1)) && c < 1 + l;
      }
      const unsigned b = __ballot_sync(0xffffffffu, f);
      flags |= (unsigned)f << cat;
      rank[cat] = __popc(b & lt);
      if (lane == 0) L.wcnt[w][cat] = (unsigned char)__popc(b);
    }
  }
  __syncthreads();
  if (t < 64) {
    const unsigned short pos = (unsigned short)(((by * USZ) << 8) | (bx * USZ));
#pragma unroll
    for (int cat = 0; cat < 9; cat++) {
      const int n0 = L.wcnt[0][cat], n1 = L.wcnt[1][cat];
      const int at = (w ? n0 : 0) + (int)rank[cat];
      constexpr bool kQuad = XDEC == 0;           // luma 4x4 leaves come four to a unit
      if (t == 0) {
        if (cat < 5) L.nblk[cat] = (cat == 0 && kQuad) ? 4 * (n0 + n1) : n0 + n1;
        else L.nnode[cat - 5] = n0 + n1;
      }
      if (flags & (1u << cat)) {
        if (cat == 0 && kQuad) {
          L.blk[4 * at + 0] = pos;
          L.blk[4 * at + 1] = (unsigned short)(pos + 4);
          L.blk[4 * at + 2] = (unsigned short)(pos + (4 << 8));
          L.blk[4 * at + 3] = (unsigned short)(pos + (4 << 8) + 4);
        } else if (cat < 5) {
          L.blk[blk_base(cat) + at] = pos;
        } else {
          const int S = 8 << (cat - 5);
          unsigned short v = pos;
          // gates compare PLANE coordinates with the LUMA picture size (src/encode.c:1487-1488)
          if (x0 + bx * USZ + S <= pic_w) v |= kGateH;
          if (y0 + by * USZ + S <= pic_h) v |= kGateV;
          L.node[node_base(cat - 5) + at] = v;
        }
      }
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// One pass of 1-D transforms over every leaf of size 2^(C+2) in the tile.
// kFwd:  pass 0 = columns, pass 1 = rows   (od_bin_fdctNxN, src/dct.c:151-156)
// !kFwd: pass 0 = rows,    pass 1 = columns (od_bin_idctNxN, src/dct.c:158-163)
// `tile` points at the superblock's (0,0) sample inside the shared tile.
// ---------------------------------------------------------------------------
template <int C, bool kFwd, int P>
__device__ __forceinline__ void transform_pass(int* tile, const SbLists& L, bool along_columns) {
  constexpr int LN = C + 2;
  constexpr int N = 1 << LN;
  const int items = L.nblk[C] << LN;
  for (int item = threadIdx.x; item < items; item += kThreads) {
    const int pos = L.blk[blk_base(C) + (item >> LN)];
    const int k = item & (N - 1);
    const int px = (pos & 255) + (along_columns ? k : 0);
    const int py = (pos >> 8) + (along_columns ? 0 : k);
    int* p = tile + py * P + px;
    int v[N];
    // compile-time strides (immediate offsets) for both directions around ONE copy of the network
    if (along_columns) {
#pragma unroll
      for (int q = 0; q < N; q++) v[q] = p[q * P];
    } else {
#pragma unroll
      for (int q = 0; q < N; q++) v[q] = p[q];
    }
    if (kFwd) Lifting<N>::fwd(v); else Lifting<N>::inv(v);
    if (along_columns) {
#pragma unroll
      for (int q = 0; q < N; q++) p[q * P] = v[q];
    } else {
#pragma unroll
      for (int q = 0; q < N; q++) p[q] = v[q];
    }
  }
}

// Not inlined on purpose: luma and chroma bodies call ONE copy of the five transform sizes
// (the 64-point network alone is ~2500 instructions; duplicating it thrashes the i-cache).
template <bool kFwd, int P>
__device__ __noinline__ void transform_all_leaves(int* tile, const SbLists& L) {
#pragma unroll 1
  for (int pass = 0; pass < 2; pass++) {
    const bool cols = kFwd ? (pass == 0) : (pass == 1);
    if (L.nblk[4]) transform_pass<4, kFwd, P>(tile, L, cols);
    if (L.nblk[3]) transform_pass<3, kFwd, P>(tile, L, cols);
    if (L.nblk[2]) transform_pass<2, kFwd, P>(tile, L, cols);
    if (L.nblk[1]) transform_pass<1, kFwd, P>(tile, L, cols);
    if (L.nblk[0]) transform_pass<0, kFwd, P>(tile, L, cols);
    __syncthreads();
  }
}

// Interior-cross lapping of every split node of edge 8 << l.
// Prefilter: horizontal edge (vertical taps) first, then the vertical edge
// (od_prefilter_split, src/filter.c:1467-1481); postfilter: the reverse
// (od_postfilter_split, src/filter.c:1510-1525).
template <bool kPost, int P>
__device__ __forceinline__ void split_filter_level(int* tile, const SbLists& L, int l, bool vertical_taps) {
  const int logS = 3 + l, S = 1 << logS;
  const int items = L.nnode[l] << logS;
  const unsigned short gate = vertical_taps ? kGateH : kGateV;
  for (int item = threadIdx.x; item < items; item += kThreads) {
    const int v = L.node[node_base(l) + (item >> logS)];
    if (!(v & gate)) continue;
    const int a = item & (S - 1);
    const int nx = v & 255, ny = (v >> 8) & 63;
    if (vertical_taps) lap4_inplace<kPost>(tile + (ny + S / 2 - 2) * P + nx + a, P);
    else lap4_inplace<kPost>(tile + (ny + a) * P + nx + S / 2 - 2, 1);
  }
}

// DC Haar pyramid over the children of every split node of edge 8 << l
// (src/encode.c:1497-1510 forward; the inverse applies the same kernel with
// the two middle terms swapped, cf. od_quantize_haar_dc_level :1651).
template <bool kInverse, int P>
__device__ __forceinline__ void haar_dc_level(int* tile, const SbLists& L, int l) {
  const int S = 8 << l;
  for (int item = threadIdx.x; item < L.nnode[l]; item += kThreads) {
    const int v = L.node[node_base(l) + item];
    int* p00 = tile + ((v >> 8) & 63) * P + (v & 255);
    int* p01 = p00 + S / 2;
    int* p10 = p00 + (S / 2) * P;
    int* p11 = p10 + S / 2;
    int ll = *p00, hl, lh, hh = *p11;
    // OD_HAAR_KERNEL(ll, lh, hl, hh), src/tf.h:35-46
    if (kInverse) { lh = *p01; hl = *p10; } else { lh = *p10; hl = *p01; }
    ll += hl;
    hh -= lh;
    int t = (ll - hh) >> 1;
    lh = t - lh;
    hl = t - hl;
    ll -= lh;
    hh += hl;
    *p00 = ll;
    *p11 = hh;
    if (kInverse) { *p01 = lh; *p10 = hl; } else { *p10 = lh; *p01 = hl; }
  }
}

// ---------------------------------------------------------------------------
// Superblock tile <-> int32 plane, four columns per thread.  Eight lanes cover 32 columns of one row and a
// warp four rows: the rows sit P = 5 (mod 32) words apart in shared memory, so the four scalar shared
// accesses of a warp touch 32 different banks, and every row segment is one 128-byte global transaction.
// Needs 16-byte aligned rows (checked by the caller, which keeps the scalar loop for odd layouts).
// ---------------------------------------------------------------------------
template <int B, int P, bool kToGlobal, int kNumThreads = kThreads>
__device__ __forceinline__ void tile_copy4(int* tile, int32_t* g, size_t gstride) {
  constexpr int kHalves = B / 32;
  constexpr int kWarps = kNumThreads / 32;
  static_assert(kWarps % kHalves == 0 && B % (4 * (kWarps / kHalves)) == 0, "row groups must tile the superblock");
  constexpr int kRowsPerIter = 4 * (kWarps / kHalves);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = (warp % kHalves) * 32 + (lane & 7) * 4;
  const int row0 = (warp / kHalves) * 4 + (lane >> 3);
  int* sp = tile + row0 * P + col;
  int32_t* gp = g + (size_t)row0 * gstride + col;
#pragma unroll 8
  for (int r = row0; r < B; r += kRowsPerIter) {
    if (kToGlobal) {
      *reinterpret_cast<int4*>(gp) = make_int4(sp[0], sp[1], sp[2], sp[3]);
    } else {
      const int4 v = *reinterpret_cast<const int4*>(gp);
      sp[0] = v.x;
      sp[1] = v.y;
      sp[2] = v.z;
      sp[3] = v.w;
    }
    sp += kRowsPerIter * P;
    gp += (size_t)kRowsPerIter * gstride;
  }
}
__device__ __forceinline__ bool rows_aligned16(const void* p, long long stride_elems) {
  return ((reinterpret_cast<uintptr_t>(p) | (uintptr_t)(stride_elems * 4)) & 15u) == 0;
}

// ---------------------------------------------------------------------------
// Per-frame forms of the forward transform's frame-wide settings (device tables of [nframes], each nullable): haar[f]
// replaces prm.haar_dc for frame f (the engine's batches of keyframes and P frames build the DC pyramid on keyframes
// only), and a frame with skip[f] set is not transformed at all (the prediction planes of those batches' keyframes).
struct FrameMasks {
  const uint8_t* haar;
  const uint8_t* skip;
};

// Forward kernel.  grid = (nhsb*sb_rows, nplanes, nframes).
// ---------------------------------------------------------------------------
template <int XDEC, bool kTma>
__device__ __forceinline__ void forward_sb_body(const FrameXformParams& prm, const PlaneXform& pl,
                                                int* tile_s, SbLists& lists, const CUtensorMap* map,
                                                unsigned char* raw, uint64_t* bar, const FrameMasks& fm) {
  constexpr int B = kMaxB >> XDEC;
  constexpr int T = B + 2 * kHalo;
  // one pitch (69 = 5 mod 32) for luma AND chroma tiles: the transform / filter code is then
  // instantiated once and shared by both plane types (half the instruction footprint)
  constexpr int P = kMaxPitch;
  using Sb = SbCtxT<B, P>;
  const int sbx = blockIdx.x % prm.nhsb, sby = prm.sb_row0 + blockIdx.x / prm.nhsb;
  const int fr = blockIdx.z;
  if (fm.skip && fm.skip[fr]) return;   // the whole CTA: nothing below is written for this frame
  const bool haar_dc = fm.haar ? fm.haar[fr] != 0 : prm.haar_dc != 0;
  Sb s;
  s.x0 = sbx * B;
  s.y0 = sby * B;
  const int pw = prm.nhsb * B, ph = prm.nvsb * B;
  // Stage the (B+4)^2 pixel window as (p-128) << OD_COEFF_SHIFT (src/state.c:1233).
  if (kTma) {
    constexpr int RW = RawTile<XDEC>::width;
    if (threadIdx.x == 0) {
      mbar_init(bar, 1);
      mbar_expect_tx(bar, RawTile<XDEC>::bytes);
      tma_load_3d(raw, map, s.x0 - RawTile<XDEC>::lead, s.y0 - kHalo, fr, bar);
    }
    // the work lists are built while the copy is in flight; the __syncthreads inside also
    // orders the barrier initialisation before anybody polls it
    build_lists<XDEC>(lists, prm.bsize + fr * prm.bsize_frame_pitch, prm.bstride, sbx, sby, s.x0, s.y0,
                      prm.pic_w, prm.pic_h);
    mbar_wait(bar, 0);
    // one aligned raw word (four window bytes) per item: window column c sits at raw byte skip + c, so the
    // words kW0 .. kW0 + kWords - 1 of a row hold the T columns, the first and the last one only partly
    constexpr int kSkip = RawTile<XDEC>::skip;
    constexpr int kW0 = kSkip / 4;
    constexpr int kWords = (kSkip + T + 3) / 4 - kW0;
    for (int i = threadIdx.x; i < T * kWords; i += kThreads) {
      const int r = i / kWords, m = i - r * kWords;
      const unsigned w = *reinterpret_cast<const unsigned*>(raw + r * RW + 4 * (kW0 + m));
      const int c0 = 4 * (kW0 + m) - kSkip;
      int* t = tile_s + r * P + c0;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int c = c0 + j;
        if (c >= 0 && c < T) t[j] = ((int)((w >> (8 * j)) & 255u) - 128) * 16;
      }
    }
  } else {
    build_lists<XDEC>(lists, prm.bsize + fr * prm.bsize_frame_pitch, prm.bstride, sbx, sby, s.x0, s.y0,
                      prm.pic_w, prm.pic_h);
    const uint8_t* src = pl.pixels + fr * pl.pixel_frame_pitch;
    for (int i = threadIdx.x; i < T * T; i += kThreads) {
      int r = i / T, c = i - r * T;
      int gx = s.x0 + c - kHalo, gy = s.y0 + r - kHalo;
      int v = 0;
      if (gx >= 0 && gx < pw && gy >= 0 && gy < ph) v = ((int)src[(size_t)gy * pl.pixel_stride + gx] - 128) * 16;
      tile_s[r * P + c] = v;
    }
  }
  __syncthreads();
  // Superblock-edge prefilter: all horizontal edges first (vertical taps),
  // then all vertical edges (src/filter.c:1541-1557).
  {
    const bool top = sby > 0, bottom = sby + 1 < prm.nvsb;
    for (int i = threadIdx.x; i < 2 * T; i += kThreads) {
      int e = i >= T, c = i - e * T;
      if (e == 0 ? top : bottom) lap4_inplace<false>(tile_s + (e ? B : 0) * P + c, P);
    }
    __syncthreads();
    const bool left = sbx > 0, right = sbx + 1 < prm.nhsb;
    for (int i = threadIdx.x; i < 2 * B; i += kThreads) {
      int r = i % B + kHalo, e = i / B;
      if (e == 0 ? left : right) lap4_inplace<false>(tile_s + r * P + (e ? B : 0), 1);
    }
    __syncthreads();
  }
  int* tile = tile_s + kHalo * P + kHalo;
  // Top-down split prefilters (levels without split nodes cost nothing).
#pragma unroll 1
  for (int l = Sb::logB - 3; l >= 0; l--) {
    if (lists.nnode[l] == 0) continue;
    split_filter_level<false, P>(tile, lists, l, true);
    __syncthreads();
    split_filter_level<false, P>(tile, lists, l, false);
    __syncthreads();
  }
#ifdef DAALA_DEBUG_LISTS
  if (threadIdx.x == 0 && XDEC == 1 && sbx == 1 && sby == 1 && blockIdx.y == 1) {
    printf("chroma lists: nblk %d %d %d %d %d nnode %d %d %d %d\n", lists.nblk[0], lists.nblk[1], lists.nblk[2],
           lists.nblk[3], lists.nblk[4], lists.nnode[0], lists.nnode[1], lists.nnode[2], lists.nnode[3]);
    for (int c = 0; c < 4; c++) for (int i = 0; i < lists.nblk[c]; i++) printf("blk c%d (%d,%d)\n", c, lists.blk[blk_base(c) + i] & 255, lists.blk[blk_base(c) + i] >> 8);
    for (int l = 0; l < 3; l++) for (int i = 0; i < lists.nnode[l]; i++) printf("node l%d (%d,%d) gates %x\n", l, lists.node[node_base(l) + i] & 255, (lists.node[node_base(l) + i] >> 8) & 63, lists.node[node_base(l) + i] >> 14);
  }
#endif
  transform_all_leaves<true, P>(tile, lists);
  if (haar_dc) {
#pragma unroll 1
    for (int l = 0; l <= Sb::logB - 3; l++) {
      if (lists.nnode[l] == 0) continue;
      haar_dc_level<false, P>(tile, lists, l);
      __syncthreads();
    }
  }
  int32_t* dst = pl.coeffs + fr * pl.coeff_frame_pitch + (size_t)s.y0 * pl.coeff_stride + s.x0;
  if (rows_aligned16(dst, pl.coeff_stride)) {
    tile_copy4<B, P, true>(tile, dst, pl.coeff_stride);
    return;
  }
  for (int i = threadIdx.x; i < B * B; i += kThreads) {
    int r = i / B, c = i % B;
    dst[(size_t)r * pl.coeff_stride + c] = tile[r * P + c];
  }
}

__global__ void __launch_bounds__(kThreads, kCtasPerSm)
k_forward_sb(const __grid_constant__ FrameXformParams prm, const __grid_constant__ FrameMasks fm) {
  __shared__ int tile_s[kMaxT * kMaxPitch];
  __shared__ SbLists lists;
  const PlaneXform& pl = prm.plane[blockIdx.y];
  if (pl.xdec == 0) forward_sb_body<0, false>(prm, pl, tile_s, lists, nullptr, nullptr, nullptr, fm);
  else forward_sb_body<1, false>(prm, pl, tile_s, lists, nullptr, nullptr, nullptr, fm);
}

// Same with the input window staged by TMA (the default when the planes meet
// the 16-byte alignment rules of tensor maps).
__global__ void __launch_bounds__(kThreads, kCtasPerSm)
k_forward_sb_tma(const __grid_constant__ FrameXformParams prm, const __grid_constant__ CUtensorMap map0,
                 const __grid_constant__ CUtensorMap map1, const __grid_constant__ CUtensorMap map2,
                 const __grid_constant__ FrameMasks fm) {
  __shared__ int tile_s[kMaxT * kMaxPitch];
  __shared__ __align__(128) unsigned char raw[RawTile<0>::bytes];
  __shared__ __align__(8) uint64_t bar;
  __shared__ SbLists lists;
  const PlaneXform& pl = prm.plane[blockIdx.y];
  // the descriptor must stay in parameter space: select between the three
  // kernel parameters, never index an array of them (that would copy to local)
  const CUtensorMap* map = blockIdx.y == 0 ? &map0 : (blockIdx.y == 1 ? &map1 : &map2);
  if (pl.xdec == 0) forward_sb_body<0, true>(prm, pl, tile_s, lists, map, raw, &bar, fm);
  else forward_sb_body<1, true>(prm, pl, tile_s, lists, map, raw, &bar, fm);
}

// ---------------------------------------------------------------------------
// Inverse kernel 1: coefficients -> lapped-domain samples (int32 plane).
// ---------------------------------------------------------------------------
template <int XDEC>
__device__ __forceinline__ void inverse_sb_body(const FrameXformParams& prm, const PlaneXform& pl,
                                                int* tile, SbLists& lists) {
  constexpr int B = kMaxB >> XDEC;
  constexpr int P = kMaxPitch;  // shared with the forward kernel's instantiations
  using Sb = SbCtxT<B, P>;
  const int sbx = blockIdx.x % prm.nhsb, sby = prm.sb_row0 + blockIdx.x / prm.nhsb;
  const int fr = blockIdx.z;
  Sb s;
  s.x0 = sbx * B;
  s.y0 = sby * B;
  const int32_t* srcp = pl.coeffs + fr * pl.coeff_frame_pitch + (size_t)s.y0 * pl.coeff_stride + s.x0;
  if (rows_aligned16(srcp, pl.coeff_stride)) {
    tile_copy4<B, P, false>(tile, const_cast<int32_t*>(srcp), pl.coeff_stride);
  } else {
    for (int i = threadIdx.x; i < B * B; i += kThreads) {
      int r = i / B, c = i % B;
      tile[r * P + c] = srcp[(size_t)r * pl.coeff_stride + c];
    }
  }
  build_lists<XDEC>(lists, prm.bsize + fr * prm.bsize_frame_pitch, prm.bstride, sbx, sby, s.x0, s.y0,
                    prm.pic_w, prm.pic_h);  // ends with a CTA barrier: tile and lists are visible
  if (prm.haar_dc) {
#pragma unroll 1
    for (int l = Sb::logB - 3; l >= 0; l--) {
      if (lists.nnode[l] == 0) continue;
      haar_dc_level<true, P>(tile, lists, l);
      __syncthreads();
    }
  }
  transform_all_leaves<false, P>(tile, lists);
  // Bottom-up split postfilters: vertical edge first, then horizontal.
#pragma unroll 1
  for (int l = 0; l <= Sb::logB - 3; l++) {
    if (lists.nnode[l] == 0) continue;
    split_filter_level<true, P>(tile, lists, l, false);
    __syncthreads();
    split_filter_level<true, P>(tile, lists, l, true);
    __syncthreads();
  }
  int32_t* dst = pl.lapped + fr * pl.lapped_frame_pitch + (size_t)s.y0 * pl.lapped_stride + s.x0;
  if (rows_aligned16(dst, pl.lapped_stride)) {
    tile_copy4<B, P, true>(tile, dst, pl.lapped_stride);
    return;
  }
  for (int i = threadIdx.x; i < B * B; i += kThreads) {
    int r = i / B, c = i % B;
    dst[(size_t)r * pl.lapped_stride + c] = tile[r * P + c];
  }
}

__global__ void __launch_bounds__(kThreads, kCtasPerSm)
k_inverse_sb(const __grid_constant__ FrameXformParams prm) {
  __shared__ int tile_s[kMaxB * kMaxPitch];
  __shared__ SbLists lists;
  const PlaneXform& pl = prm.plane[blockIdx.y];
  if (pl.xdec == 0) inverse_sb_body<0>(prm, pl, tile_s, lists);
  else inverse_sb_body<1>(prm, pl, tile_s, lists);
}

// ---------------------------------------------------------------------------
// Inverse kernel 2: superblock-edge postfilter + clamp to 8 bits.
// One CTA per superblock; reads a (B+4)^2 window of the lapped plane.
// Vertical edges first (horizontal taps), then horizontal edges
// (src/filter.c:1599-1617); store OD_CLAMP255(((v + 8) >> 4) + 128)
// (src/state.c:1300-1303).
// ---------------------------------------------------------------------------
template <int XDEC>
__device__ __forceinline__ void sb_postfilter_store_body(const FrameXformParams& prm,
                                                         const PlaneXform& pl, int* tile_s) {
  constexpr int B = kMaxB >> XDEC;
  constexpr int T = B + 2 * kHalo;
  constexpr int P = T + 1;
  const int sbx = blockIdx.x % prm.nhsb, sby = prm.sb_row0 + blockIdx.x / prm.nhsb;
  const int fr = blockIdx.z;
  const int32_t* lap = pl.lapped + fr * pl.lapped_frame_pitch;
  const int x0 = sbx * B, y0 = sby * B;
  const int pw = prm.nhsb * B, ph = prm.nvsb * B;
  const int32_t* core = lap + (size_t)y0 * pl.lapped_stride + x0;
  if (rows_aligned16(core, pl.lapped_stride)) {
    // the superblock itself with 128-bit loads, then the 2-sample frame around it (zero outside the plane)
    tile_copy4<B, P, false, kPostThreads>(tile_s + kHalo * P + kHalo, const_cast<int32_t*>(core), pl.lapped_stride);
    for (int i = threadIdx.x; i < 4 * T + 4 * B; i += kPostThreads) {
      int r, c;
      if (i < 4 * T) {
        const int k = i / T;                 // rows -2, -1, B, B+1 of the window, all T columns
        r = k < 2 ? k : B + k;
        c = i - k * T;
      } else {
        const int j = i - 4 * T, k = j / B;  // columns -2, -1, B, B+1, the B rows in between
        c = k < 2 ? k : B + k;
        r = j - k * B + kHalo;
      }
      const int gx = x0 + c - kHalo, gy = y0 + r - kHalo;
      int v = 0;
      if (gx >= 0 && gx < pw && gy >= 0 && gy < ph) v = lap[(size_t)gy * pl.lapped_stride + gx];
      tile_s[r * P + c] = v;
    }
  } else {
    for (int i = threadIdx.x; i < T * T; i += kPostThreads) {
      int r = i / T, c = i - r * T;
      int gx = x0 + c - kHalo, gy = y0 + r - kHalo;
      int v = 0;
      if (gx >= 0 && gx < pw && gy >= 0 && gy < ph) v = lap[(size_t)gy * pl.lapped_stride + gx];
      tile_s[r * P + c] = v;
    }
  }
  __syncthreads();
  const bool left = sbx > 0, right = sbx + 1 < prm.nhsb;
  for (int i = threadIdx.x; i < 2 * T; i += kPostThreads) {
    int e = i >= T, r = i - e * T;
    if (e == 0 ? left : right) lap4_inplace<true>(tile_s + r * P + (e ? B : 0), 1);
  }
  __syncthreads();
  const bool top = sby > 0, bottom = sby + 1 < prm.nvsb;
  for (int i = threadIdx.x; i < 2 * B; i += kPostThreads) {
    int c = i % B + kHalo, e = i / B;
    if (e == 0 ? top : bottom) lap4_inplace<true>(tile_s + (e ? B : 0) * P + c, P);
  }
  __syncthreads();
  if (prm.post16[blockIdx.y]) {
    // the deringing stage's input (state->etmp): the filtered samples as int16, two per 32-bit store
    int16_t* d16 = prm.post16[blockIdx.y] + fr * pl.pixel_out_frame_pitch + (size_t)y0 * pl.pixel_out_stride + x0;
    for (int i = threadIdx.x; i < B * B / 2; i += kPostThreads) {
      int r = i / (B / 2), c2 = (i % (B / 2)) * 2;
      const int* p = tile_s + (r + kHalo) * P + c2 + kHalo;
      const unsigned w = ((unsigned)p[0] & 0xffffu) | ((unsigned)p[1] << 16);
      *reinterpret_cast<unsigned*>(d16 + (size_t)r * pl.pixel_out_stride + c2) = w;
    }
    return;
  }
  uint8_t* dst = pl.pixels_out + fr * pl.pixel_out_frame_pitch + (size_t)y0 * pl.pixel_out_stride + x0;
  // Four pixels per thread, packed into one 32-bit store.
  for (int i = threadIdx.x; i < B * B / 4; i += kPostThreads) {
    int r = i / (B / 4), c4 = (i % (B / 4)) * 4;
    const int* p = tile_s + (r + kHalo) * P + c4 + kHalo;
    unsigned w = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      int v = ((p[k] + 8) >> 4) + 128;
      v = v < 0 ? 0 : (v > 255 ? 255 : v);
      w |= (unsigned)v << (8 * k);
    }
    *reinterpret_cast<unsigned*>(dst + (size_t)r * pl.pixel_out_stride + c4) = w;
  }
}

__global__ void __launch_bounds__(kPostThreads)
k_sb_postfilter_store(const __grid_constant__ FrameXformParams prm) {
  __shared__ int tile_s[kMaxT * kMaxPitch];
  const PlaneXform& pl = prm.plane[blockIdx.y];
  if (pl.xdec == 0) sb_postfilter_store_body<0>(prm, pl, tile_s);
  else sb_postfilter_store_body<1>(prm, pl, tile_s);
}

// ---------------------------------------------------------------------------
// Plane-wide superblock-edge filters on an int32 plane, in place (the
// stand-alone forms of od_apply_prefilter_frame_sbs / _postfilter_).
// One launch per direction; `vertical_taps` selects horizontal edges.
// ---------------------------------------------------------------------------
template <bool kPost>
__global__ void k_plane_sb_edges(int32_t* c, int stride, int nhsb, int nvsb, int sbw, int sbh,
                                 bool vertical_taps) {
  const int w = nhsb * sbw, h = nvsb * sbh;
  const int along = vertical_taps ? w : h;
  const int edges = (vertical_taps ? nvsb : nhsb) - 1;
  const long total = (long)along * edges;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total;
       i += (long)gridDim.x * blockDim.x) {
    int a = (int)(i % along), e = (int)(i / along) + 1;
    if (vertical_taps) lap4_inplace<kPost>(c + (size_t)(e * sbh - 2) * stride + a, stride);
    else lap4_inplace<kPost>(c + (size_t)a * stride + e * sbw - 2, 1);
  }
}

// ---------------------------------------------------------------------------
// Batched stand-alone block transforms: `count` packed n x n blocks
// (row-major, contiguous).  One CTA per block; used by the per-call od_bin_*
// entry points and by the dcttest-style parity tests.
// mode: 0 = 2-D forward, 1 = 2-D inverse, 2 = 1-D forward (rows), 3 = 1-D inverse (rows)
// ---------------------------------------------------------------------------
template <int L>
__global__ void __launch_bounds__(64)
k_block_transform(int32_t* blocks, int mode) {
  constexpr int N = 1 << L;
  constexpr int P = N + 5;
  __shared__ int t[N * P];
  int32_t* blk = blocks + (size_t)blockIdx.x * N * N;
  for (int i = threadIdx.x; i < N * N; i += blockDim.x) t[(i / N) * P + (i % N)] = blk[i];
  __syncthreads();
  const bool fwd = (mode & 1) == 0;
  const int passes = mode < 2 ? 2 : 1;
  for (int pass = 0; pass < passes; pass++) {
    bool cols = mode < 2 ? (fwd ? pass == 0 : pass == 1) : false;
    if (threadIdx.x < N) {
      int* p = cols ? t + threadIdx.x : t + threadIdx.x * P;
      int stride = cols ? P : 1;
      int v[N];
#pragma unroll
      for (int k = 0; k < N; k++) v[k] = p[k * stride];
      if (fwd) Lifting<N>::fwd(v); else Lifting<N>::inv(v);
#pragma unroll
      for (int k = 0; k < N; k++) p[k * stride] = v[k];
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < N * N; i += blockDim.x) blk[i] = t[(i / N) * P + (i % N)];
}

// Batched 4-point filters: `count` groups of four ints.
__global__ void k_filter4_batch(int32_t* v, long count, int post) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < count;
       i += (long)gridDim.x * blockDim.x) {
    if (post) lap4_inplace<true>(v + 4 * i, 1); else lap4_inplace<false>(v + 4 * i, 1);
  }
}

// Batched N-point lapped filters (N = 8, 16, 32): `count` groups of N ints.
template <int N>
__global__ void k_lapfilter_batch(int32_t* v, long count, int post) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < count; i += (long)gridDim.x * blockDim.x) {
    int t[N];
#pragma unroll
    for (int k = 0; k < N; k++) t[k] = v[i * N + k];
    if (post) LapFilter<N>::post(t); else LapFilter<N>::pre(t);
#pragma unroll
    for (int k = 0; k < N; k++) v[i * N + k] = t[k];
  }
}

// Interior-cross filter of `count` packed n x n nodes (od_prefilter_split /
// od_postfilter_split on stand-alone blocks).
__global__ void k_split_filter_batch(int32_t* blocks, int n, int post, int hfilter, int vfilter) {
  int32_t* b = blocks + (size_t)blockIdx.x * n * n;
  for (int phase = 0; phase < 2; phase++) {
    bool vertical_taps = post ? phase == 1 : phase == 0;
    if (vertical_taps ? hfilter : vfilter) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (vertical_taps) {
          if (post) lap4_inplace<true>(b + (n / 2 - 2) * n + i, n); else lap4_inplace<false>(b + (n / 2 - 2) * n + i, n);
        } else {
          if (post) lap4_inplace<true>(b + i * n + n / 2 - 2, 1); else lap4_inplace<false>(b + i * n + n / 2 - 2, 1);
        }
      }
    }
    __syncthreads();
  }
}

}  // namespace daala_b200

using namespace daala_b200;

// od_haar / od_haar_inv (src/dct.c:4822 / :4861): the multi-level 2-D Haar wavelet of the lossless
// path, one CTA per packed n x n block, in place (the level loops: haar.cuh).
template <bool kInverse>
__global__ void __launch_bounds__(256) k_haar_blocks(int32_t* __restrict__ blocks, int ln) {
  __shared__ int t[64 * 64];
  const int n = 1 << ln;
  int32_t* g = blocks + (size_t)blockIdx.x * n * n;
  if (!kInverse) {
    for (int i = threadIdx.x; i < n * n; i += 256) t[i] = g[i];
    __syncthreads();
    haar_forward_levels<256>(t, g, n, ln);
  } else {
    haar_inverse_levels<256>(t, g, n, ln);
    for (int i = threadIdx.x; i < n * n; i += 256) g[i] = t[i];
  }
}

extern "C" {

// Tensor maps are encoded with the driver entry point fetched through the
// runtime (no link-time dependency on libcuda).  Returns false when a plane
// cannot be described (alignment), in which case the plain-load kernel runs.
static bool encode_input_maps(const FrameXformParams* prm, int nplanes, TmaMaps* maps) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      encode = (PFN_cuTensorMapEncodeTiled_v12000)fn;
  }
  if (!encode) return false;
  memset(maps, 0, sizeof(*maps));
  for (int p = 0; p < nplanes; p++) {
    const PlaneXform& pl = prm->plane[p];
    const int B = kMaxB >> pl.xdec;
    const cuuint64_t w = (cuuint64_t)prm->nhsb * B, h = (cuuint64_t)prm->nvsb * B;
    const cuuint64_t fpitch = prm->nframes > 1 ? (cuuint64_t)pl.pixel_frame_pitch : w * h;
    if (((uintptr_t)pl.pixels & 15) || (pl.pixel_stride & 15) || (fpitch & 15) || pl.pixel_stride <= 0) return false;
    cuuint64_t dims[3] = {w, h, (cuuint64_t)prm->nframes};
    cuuint64_t strides[2] = {(cuuint64_t)pl.pixel_stride, fpitch};
    cuuint32_t box[3] = {(cuuint32_t)(pl.xdec ? RawTile<1>::width : RawTile<0>::width),
                         (cuuint32_t)(B + 2 * kHalo), 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = encode(&maps->plane[p], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void*)pl.pixels, dims, strides, box,
                        estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return false;
  }
  return true;
}

int daala_b200_launch_forward_masked(const FrameXformParams* prm, int nplanes, const uint8_t* haar_frames,
                                     const uint8_t* skip_frames, cudaStream_t stream) {
  dim3 grid(prm->nhsb * prm->sb_rows, nplanes, prm->nframes);
  const FrameMasks fm = {haar_frames, skip_frames};
  TmaMaps maps;
  if (encode_input_maps(prm, nplanes, &maps))
    k_forward_sb_tma<<<grid, kThreads, 0, stream>>>(*prm, maps.plane[0], maps.plane[1], maps.plane[2], fm);
  else k_forward_sb<<<grid, kThreads, 0, stream>>>(*prm, fm);
  return (int)cudaGetLastError();
}

int daala_b200_launch_forward(const FrameXformParams* prm, int nplanes, cudaStream_t stream) {
  return daala_b200_launch_forward_masked(prm, nplanes, nullptr, nullptr, stream);
}

// Test hook: force the plain-load variant.
int daala_b200_launch_forward_no_tma(const FrameXformParams* prm, int nplanes, cudaStream_t stream) {
  dim3 grid(prm->nhsb * prm->sb_rows, nplanes, prm->nframes);
  k_forward_sb<<<grid, kThreads, 0, stream>>>(*prm, FrameMasks{nullptr, nullptr});
  return (int)cudaGetLastError();
}

int daala_b200_launch_inverse(const FrameXformParams* prm, int nplanes, cudaStream_t stream) {
  dim3 grid(prm->nhsb * prm->sb_rows, nplanes, prm->nframes);
  k_inverse_sb<<<grid, kThreads, 0, stream>>>(*prm);
  k_sb_postfilter_store<<<grid, kPostThreads, 0, stream>>>(*prm);
  return (int)cudaGetLastError();
}

// The kernels take their plane from blockIdx.y: planes [plane0, plane0 + nplanes) of prm become planes
// [0, nplanes) of the launch's copy.
static FrameXformParams plane_range(const FrameXformParams* prm, int plane0) {
  FrameXformParams q = *prm;
  for (int p = 0; p + plane0 < 3; p++) {
    q.plane[p] = prm->plane[plane0 + p];
    q.post16[p] = prm->post16[plane0 + p];
  }
  return q;
}

int daala_b200_launch_inverse_lapped_only(const FrameXformParams* prm, int plane0, int nplanes, cudaStream_t stream) {
  if (plane0 < 0 || nplanes < 1 || plane0 + nplanes > 3) return (int)cudaErrorInvalidValue;
  dim3 grid(prm->nhsb * prm->sb_rows, nplanes, prm->nframes);
  k_inverse_sb<<<grid, kThreads, 0, stream>>>(plane_range(prm, plane0));
  return (int)cudaGetLastError();
}

int daala_b200_launch_sb_postfilter_store(const FrameXformParams* prm, int plane0, int nplanes, cudaStream_t stream) {
  if (plane0 < 0 || nplanes < 1 || plane0 + nplanes > 3) return (int)cudaErrorInvalidValue;
  dim3 grid(prm->nhsb * prm->sb_rows, nplanes, prm->nframes);
  k_sb_postfilter_store<<<grid, kPostThreads, 0, stream>>>(plane_range(prm, plane0));
  return (int)cudaGetLastError();
}

int daala_b200_launch_plane_sb_filter(int32_t* c, int stride, int nhsb, int nvsb, int xdec, int ydec,
                                      int post, cudaStream_t stream) {
  const int sbw = 64 >> xdec, sbh = 64 >> ydec;
  for (int phase = 0; phase < 2; phase++) {
    bool vertical_taps = post ? phase == 1 : phase == 0;
    long total = vertical_taps ? (long)nhsb * sbw * (nvsb - 1) : (long)nvsb * sbh * (nhsb - 1);
    if (total <= 0) continue;
    int blocks = (int)((total + 255) / 256);
    if (blocks > kGridCap) blocks = kGridCap;
    if (post) k_plane_sb_edges<true><<<blocks, 256, 0, stream>>>(c, stride, nhsb, nvsb, sbw, sbh, vertical_taps);
    else k_plane_sb_edges<false><<<blocks, 256, 0, stream>>>(c, stride, nhsb, nvsb, sbw, sbh, vertical_taps);
  }
  return (int)cudaGetLastError();
}

int daala_b200_launch_block_transform(int32_t* blocks, int count, int ln, int mode, cudaStream_t stream) {
  if (count <= 0) return 0;
  switch (ln) {
    case 2: k_block_transform<2><<<count, 64, 0, stream>>>(blocks, mode); break;
    case 3: k_block_transform<3><<<count, 64, 0, stream>>>(blocks, mode); break;
    case 4: k_block_transform<4><<<count, 64, 0, stream>>>(blocks, mode); break;
    case 5: k_block_transform<5><<<count, 64, 0, stream>>>(blocks, mode); break;
    case 6: k_block_transform<6><<<count, 64, 0, stream>>>(blocks, mode); break;
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)cudaGetLastError();
}

int daala_b200_launch_haar_blocks(int32_t* blocks, int count, int ln, int inverse, cudaStream_t stream) {
  if (count <= 0) return 0;
  if (ln < 1 || ln > 6) return (int)cudaErrorInvalidValue;
  if (inverse) k_haar_blocks<true><<<count, 256, 0, stream>>>(blocks, ln);
  else k_haar_blocks<false><<<count, 256, 0, stream>>>(blocks, ln);
  return (int)cudaGetLastError();
}

int daala_b200_launch_filter4(int32_t* v, long count, int post, cudaStream_t stream) {
  if (count <= 0) return 0;
  int blocks = (int)((count + 255) / 256);
  if (blocks > kGridCap) blocks = kGridCap;
  k_filter4_batch<<<blocks, 256, 0, stream>>>(v, count, post);
  return (int)cudaGetLastError();
}

int daala_b200_launch_lapfilter(int32_t* v, long count, int n, int post, cudaStream_t stream) {
  if (count <= 0) return 0;
  int blocks = (int)((count + 127) / 128);
  if (blocks > kGridCap) blocks = kGridCap;
  if (n == 4) k_filter4_batch<<<blocks, 128, 0, stream>>>(v, count, post);
  else if (n == 8) k_lapfilter_batch<8><<<blocks, 128, 0, stream>>>(v, count, post);
  else if (n == 16) k_lapfilter_batch<16><<<blocks, 128, 0, stream>>>(v, count, post);
  else if (n == 32) k_lapfilter_batch<32><<<blocks, 128, 0, stream>>>(v, count, post);
  else return (int)cudaErrorInvalidValue;
  return (int)cudaGetLastError();
}

int daala_b200_launch_split_filter(int32_t* blocks, int count, int n, int post, int hfilter, int vfilter,
                                   cudaStream_t stream) {
  if (count <= 0) return 0;
  k_split_filter_batch<<<count, 64, 0, stream>>>(blocks, n, post, hfilter, vfilter);
  return (int)cudaGetLastError();
}

}  // extern "C"
