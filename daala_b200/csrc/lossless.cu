// The keyframe engine's lossless step (config.lossless): frames coded at quantizer 0, the reference's Haar-wavelet path
// (OD_LOSSLESS, reference src/internal.h:131).  Every superblock is one 64x64 block (32x32 in 4:2:0 chroma), with no
// lapping, no deringing, and a quantizer of 1 everywhere (src/encode.c:3027, :3087-3089, :2570-2680).  Per block:
//   c   = pixel - 128 (od_ref_buf_to_coeff, shift 0); P / B frames replace every sample outside the picture with the
//         prediction's (src/encode.c:2589-2602), keyframes keep their input padding;
//   d   = od_haar(c), and on P / B frames md = od_haar(mc) of the prediction;
//   out = d - md over the AC sub-bands (od_wavelet_quantize, src/encode.c:1012-1027, q = 1; md = 0 on keyframes);
//   DC  = d[0] - md[0] on P / B frames (src/encode.c:1337-1343, dead zone 0); on keyframes d[0] minus the superblock
//         DC predictor of the neighbours' DCs (od_quantize_haar_dc_sb, src/encode.c:1537-1590, dc_quant = 1: the
//         neighbours' DCs are their unquantised d[0]);
//   the root sums tree_sum[0][1], [1][0], [1][1] of od_compute_max_tree (src/encode.c:899-919) over `out`;
//   the reconstruction the decoder makes: the emitted residual plus the prediction, od_haar_inv, + 128 and clamp.
// One CTA of 256 threads per (superblock, plane, frame); the block lives in shared memory from the u8 load to the u8
// store.  Keyframes need the DCs of the neighbouring superblocks, so their step is two kernels.
#include <cuda_runtime.h>
#include <stdint.h>

#include "haar.cuh"
#include "lossless.h"

namespace daala_b200 {
namespace lossless {

constexpr int kThreads = 256;

struct Block {
  int sbx, sby, p, f, ln, n, W;
  size_t org;     // offset of the block's first sample in the plane arrays
  size_t plane;   // samples per frame of this plane
};

__device__ __forceinline__ Block block_of(const daala_b200_lossless_batch& B) {
  Block k;
  k.sbx = blockIdx.x % B.nhsb;
  k.sby = blockIdx.x / B.nhsb;
  k.p = blockIdx.y;
  k.f = blockIdx.z;
  k.ln = k.p ? 5 : 6;
  k.n = 1 << k.ln;
  k.W = B.plane_w[k.p];
  k.plane = (size_t)k.W * B.plane_h[k.p];
  k.org = k.f * k.plane + (size_t)k.sby * k.n * k.W + (size_t)k.sbx * k.n;
  return k;
}

__device__ __forceinline__ size_t record(const daala_b200_lossless_batch& B, const Block& k) {
  return (((size_t)k.f * B.nvsb + k.sby) * B.nhsb + k.sbx) * 3 + k.p;
}

// The three root sums of od_compute_max_tree over `out` (row stride W): sample (r, c) != (0, 0) belongs to the tree of
// (1, 0) when r < 2^L, of (0, 1) when c < 2^L, else of (1, 1), with L = ilog(max(r, c)) - 1 its sub-band level.
__device__ __forceinline__ void tree_sums(const int acc_in[3], int32_t* rec) {
  __shared__ int red[3][kThreads / 32];
  int acc[3] = {acc_in[0], acc_in[1], acc_in[2]};
  for (int d = 0; d < 3; d++)
    for (int o = 16; o > 0; o >>= 1) acc[d] += __shfl_xor_sync(0xffffffffu, acc[d], o);
  if ((threadIdx.x & 31) == 0)
    for (int d = 0; d < 3; d++) red[d][threadIdx.x >> 5] = acc[d];
  __syncthreads();
  if (threadIdx.x < 4) {
    int s = 0;
    if (threadIdx.x < 3)
      for (int w = 0; w < kThreads / 32; w++) s += red[threadIdx.x][w];
    rec[threadIdx.x] = s;
  }
}

__device__ __forceinline__ int tree_of(int r, int c) {
  const int s = 1 << (31 - __clz(r > c ? r : c));
  return r < s ? 0 : c < s ? 1 : 2;
}

// od_coeff_to_ref_buf of the block in t (lossless: + 128, clamp) into the reconstruction and, on inter_mc engines, the
// frame's pool slot.
__device__ __forceinline__ void store_pixels(const daala_b200_lossless_batch& B, const Block& k, const int* t) {
  const int slot = B.slot_out ? B.slot_out[k.f] : -1;
  uint8_t* out = B.out[k.p] + k.org;
  uint8_t* pool = slot >= 0 ? B.pool[k.p] + (size_t)slot * k.plane + (k.org - k.f * k.plane) : nullptr;
  for (int i = threadIdx.x; i < k.n * k.n; i += kThreads) {
    const int v = t[i] + 128;
    const uint8_t u = (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
    const size_t o = (size_t)(i >> k.ln) * k.W + (i & (k.n - 1));
    out[o] = u;
    if (pool) pool[o] = u;
  }
}

// Forward transform, residual and root sums of every block.  kInter: also md, the padding rule, the DC residual and
// the reconstruction; keyframes leave the DC slot of `coeffs` and the reconstruction to k_ll_dc_recon and store d[0].
template <bool kInter>
__global__ void __launch_bounds__(kThreads) k_ll_forward(const __grid_constant__ daala_b200_lossless_batch B) {
  __shared__ int t[64 * 64];
  __shared__ int yd[64 * 64];
  __shared__ int16_t ym[kInter ? 64 * 64 : 1];   // |md| <= 8192 (DESIGN.md, lossless section)
  const Block k = block_of(B);
  const int nn = k.n * k.n;
  const uint8_t* src = B.src[k.p] + k.org;
  const uint8_t* pred = kInter ? B.pred[k.p] + k.org : nullptr;
  if (kInter) {
    for (int i = threadIdx.x; i < nn; i += kThreads) t[i] = pred[(size_t)(i >> k.ln) * k.W + (i & (k.n - 1))] - 128;
    __syncthreads();
    haar_forward_levels<kThreads>(t, ym, k.n, k.ln);
    __syncthreads();
  }
  // the picture area of this plane (4:2:0: pic_w >> 1, as the reference's padding loop)
  const int pw = B.pic_w >> (k.p ? 1 : 0), ph = B.pic_h >> (k.p ? 1 : 0);
  for (int i = threadIdx.x; i < nn; i += kThreads) {
    const int r = i >> k.ln, c = i & (k.n - 1);
    const size_t o = (size_t)r * k.W + c;
    const bool inside = k.sbx * k.n + c < pw && k.sby * k.n + r < ph;
    t[i] = (kInter && !inside ? pred[o] : src[o]) - 128;
  }
  __syncthreads();
  haar_forward_levels<kThreads>(t, yd, k.n, k.ln);
  __syncthreads();
  int16_t* out = B.coeffs[k.p] + k.org;
  int acc[3] = {0, 0, 0};
  for (int i = threadIdx.x; i < nn; i += kThreads) {
    const int r = i >> k.ln, c = i & (k.n - 1);
    if (!kInter && i == 0) continue;
    const int16_t v = (int16_t)(kInter ? yd[i] - ym[i] : yd[i]);
    out[(size_t)r * k.W + c] = v;
    if (i) acc[tree_of(r, c)] += v < 0 ? -v : v;
    if (kInter) yd[i] = v + ym[i];   // what the decoder adds back (src/encode.c:1377-1378, :1069-1077)
  }
  tree_sums(acc, B.blocks + 4 * record(B, k));
  if (!kInter) {
    if (threadIdx.x == 0) B.dc[record(B, k)] = yd[0];
    return;
  }
  haar_inverse_levels<kThreads>(t, yd, k.n, k.ln);
  store_pixels(B, k, t);
}

// Keyframes: the superblock DC predictor of od_quantize_haar_dc_sb from the left, up, up-left and up-right DCs (the
// stored d[0] of k_ll_forward), dc0 = d[0] - predictor into the DC slot, then the reconstruction from the stored
// residual with d[0] = dc0 + predictor.
__global__ void __launch_bounds__(kThreads) k_ll_dc_recon(const __grid_constant__ daala_b200_lossless_batch B) {
  __shared__ int t[64 * 64];
  __shared__ int yd[64 * 64];
  const Block k = block_of(B);
  const int32_t* dc = B.dc + ((size_t)k.f * B.nvsb * B.nhsb) * 3 + k.p;
  auto at = [&](int y, int x) { return dc[((size_t)y * B.nhsb + x) * 3]; };
  int pred;
  if (k.sby > 0 && k.sbx > 0) {
    if (k.sbx < B.nhsb - 1)   // has_ur = sby > 0 && sbx < nhsb - 1 (src/encode.c:2640)
      pred = (22 * at(k.sby, k.sbx - 1) - 9 * at(k.sby - 1, k.sbx - 1) + 15 * at(k.sby - 1, k.sbx) +
              4 * at(k.sby - 1, k.sbx + 1) + 16) >> 5;
    else
      pred = (23 * at(k.sby, k.sbx - 1) - 10 * at(k.sby - 1, k.sbx - 1) + 19 * at(k.sby - 1, k.sbx) + 16) >> 5;
  } else if (k.sby > 0) {
    pred = at(k.sby - 1, k.sbx);
  } else if (k.sbx > 0) {
    pred = at(k.sby, k.sbx - 1);
  } else {
    pred = 0;
  }
  const int16_t dc0 = (int16_t)(at(k.sby, k.sbx) - pred);   // |dc0| <= 21420 (DESIGN.md, lossless section)
  int16_t* out = B.coeffs[k.p] + k.org;
  const int nn = k.n * k.n;
  for (int i = threadIdx.x; i < nn; i += kThreads) {
    const size_t o = (size_t)(i >> k.ln) * k.W + (i & (k.n - 1));
    if (i == 0) {
      out[0] = dc0;
      yd[0] = dc0 + pred;
    } else {
      yd[i] = out[o];
    }
  }
  __syncthreads();
  haar_inverse_levels<kThreads>(t, yd, k.n, k.ln);
  store_pixels(B, k, t);
}

}  // namespace lossless
}  // namespace daala_b200

extern "C" int daala_b200_launch_lossless(const daala_b200_lossless_batch* b, cudaStream_t stream) {
  using namespace daala_b200::lossless;
  const dim3 grid(b->nhsb * b->nvsb, 3, b->F);
  if (b->pred[0]) {
    k_ll_forward<true><<<grid, kThreads, 0, stream>>>(*b);
  } else {
    k_ll_forward<false><<<grid, kThreads, 0, stream>>>(*b);
    k_ll_dc_recon<<<grid, kThreads, 0, stream>>>(*b);
  }
  return (int)cudaGetLastError();
}
