// The keyframe DC chain (config.haar_dc_quant): od_quantize_haar_dc_sb and od_quantize_haar_dc_level (reference
// src/encode.c:1537-1657) in od_encode_recursive's order (:1765-1787, :2605-2656), on the unquantised Haar DC pyramid
// the forward transform leaves in the `d` planes.  daala_b200/haardc.py restates it in numpy.
//
// Each plane's decisions depend only on that plane's DC symbols: the models (one generic model, ex_sb_dc, ex_dc[5][3])
// start from od_adapt_ctx_reset on every keyframe and nothing else in the step reads or adapts them.  So the chain is
// one serial walk per (frame, plane), one warp each; the warp clears the index grid, then lane 0 walks.  The rate
// estimate uses the CUDA library's log() (the reference: glibc's), in double, with the library's -fmad=false.
#include <math.h>

#include "haar_dc.h"

namespace daala_b200 {
namespace haar_dc {

constexpr int kTables = 12;                                        // GENERIC_TABLES
__constant__ int kDcQm[4][2] = {{21, 25}, {18, 20}, {17, 18}, {17, 17}};   // OD_DC_QM, src/state.c:48

__device__ __forceinline__ int ilog(int v) { return v ? 32 - __clz(v) : 0; }

// log_ex, src/generic_code.c:109
__device__ __forceinline__ int log_ex(int ex_q16) {
  const int lg = ilog(ex_q16);
  int odd;
  if (lg < 15) {
    odd = ex_q16 * ex_q16 > 2 << 2 * lg;
  } else {
    const int tmp = ex_q16 >> (lg - 8);
    odd = tmp * tmp > (1 << 15);
  }
  const int r = 2 * lg - 33 + odd;
  return r > 0 ? r : 0;
}

// generic_encode_cost with max = -1, src/generic_encoder.c:161
__device__ double gen_cost(const int* cdfs, int x, int ex_q16) {
  const int lg_q1 = log_ex(ex_q16);
  const int shift = max(0, (lg_q1 - 5) >> 1);
  const int* cdf = cdfs + 16 * min(kTables - 1, lg_q1);
  int xs = (x + (1 << shift >> 1)) >> shift;
  int extra = shift ? shift - (xs == 0) : 0;
  xs = min(15, xs);
  if (xs == 15) extra += 2;
  return extra - M_LOG2E * log((double)(cdf[xs] - (xs == 0 ? 0 : cdf[xs - 1])) / cdf[15]);
}

// The model side of generic_encode with max = -1 and integration 2 (src/generic_encoder.c:99, generic_model_update
// src/generic_code.c:136): the CDF increment (with its renormalisation) and the ex_q16 update.
__device__ void gen_adapt(int* cdfs, int x, int* ex_q16) {
  const int lg_q1 = log_ex(*ex_q16);
  const int shift = max(0, (lg_q1 - 5) >> 1);
  int* cdf = cdfs + 16 * min(kTables - 1, lg_q1);
  const int xs = (x + (1 << shift >> 1)) >> shift;
  if (cdf[15] + 64 > 32767)
    for (int i = 0; i < 16; i++) cdf[i] = (cdf[i] >> 1) + i + 1;
  for (int i = min(15, xs); i < 16; i++) cdf[i] += 64;
  x = min(x, 32767);
  *ex_q16 += ((x << 16) - *ex_q16) >> 2;
}

struct Node {
  int bx, by, bsi;
  int hgrad, vgrad;
};

// The quantiser is that of the warp's frame, B.fq_bq.
__global__ void __launch_bounds__(32) k_haar_dc(const __grid_constant__ daala_b200_haar_dc_batch B) {
  extern __shared__ int sb_mem[];                 // [2][nhsb]: quantised SB DCs of the row above and of this row
  __shared__ int cdfs[kTables * 16];
  const int f = blockIdx.x / 3, pli = blockIdx.x % 3;
  const int xdec = pli ? 1 : 0;
  const int pw = B.plane_w[pli], gw = pw >> 2;
  const size_t gn = (size_t)gw * (B.plane_h[pli] >> 2);
  const int32_t* d = B.coeffs[pli] + (size_t)f * pw * B.plane_h[pli];
  int32_t* dc = B.dc[pli] + f * B.grid_frame_pitch;
  int32_t* idx = B.index[pli] + f * gn;
  const uint8_t* bsize = B.bsize + (size_t)f * B.nhsb * 8 * B.nvsb * 8;
  const int bstride = B.nhsb * 8;
  for (size_t i = threadIdx.x; i < gn; i += 32) idx[i] = 0;
  for (int i = threadIdx.x; i < kTables * 16; i += 32) cdfs[i] = ((i & 15) + 1) * 64;   // generic_model_init
  __syncwarp();
  if (threadIdx.x != 0 || (B.frame_type && !B.frame_type[f])) return;
  const int ex0 = pli ? 8 : 32768;
  int ex_sb = ex0;
  int ex_dc[5][3];
  for (int i = 0; i < 5; i++)
    for (int j = 0; j < 3; j++) ex_dc[i][j] = ex0;
  const int dq = B.fq_bq[(f * 3 + pli) * 32 + 20];
  const double lam = B.pvq_norm_lambda;
  const int nhsb = B.nhsb;
  const int lsb = 6 - xdec;                       // log2 of the superblock edge in this plane
  Node stack[16];
  for (int sby = 0; sby < B.nvsb; sby++) {
    int* up = sb_mem + ((sby + 1) & 1) * nhsb;
    int* cur = sb_mem + (sby & 1) * nhsb;
    for (int sbx = 0; sbx < nhsb; sbx++) {
      // od_quantize_haar_dc_sb, src/encode.c:1537-1590
      const bool has_ur = sby > 0 && sbx < nhsb - 1;
      int pred;
      if (sby > 0 && sbx > 0) {
        pred = has_ur ? (22 * cur[sbx - 1] - 9 * up[sbx - 1] + 15 * up[sbx] + 4 * up[sbx + 1] + 16) >> 5
                      : (23 * cur[sbx - 1] - 10 * up[sbx - 1] + 19 * up[sbx] + 16) >> 5;
      } else if (sby > 0) {
        pred = up[sbx];
      } else if (sbx > 0) {
        pred = cur[sbx - 1];
      } else {
        pred = 0;
      }
      const int oy = sby << lsb, ox = sbx << lsb;
      const int dc0 = d[(size_t)oy * pw + ox] - pred;
      const int half = ((dq + 1) >> 1) - 1;
      const int quant = (dc0 + (dc0 < 0 ? -half : half)) / dq;    // OD_DIV_R0
      gen_adapt(cdfs, abs(quant), &ex_sb);
      const int v = quant * dq + pred;
      cur[sbx] = v;
      dc[(oy >> 2) * gw + (ox >> 2)] = v;
      idx[(oy >> 2) * gw + (ox >> 2)] = quant;
      int sp = 0;
      stack[sp++] = Node{sbx, sby, 4, sbx > 0 ? cur[sbx - 1] - v : 0, sby > 0 ? up[sbx] - v : 0};
      // od_encode_recursive's split nodes depth-first: popping TL first, each child with its parent's gradients
      while (sp > 0) {
        Node n = stack[--sp];
        const int obs = bsize[(size_t)((n.by << n.bsi) >> 1) * bstride + ((n.bx << n.bsi) >> 1)];
        if (max(obs, xdec) >= n.bsi) continue;   // a leaf (>: a map that is no quadtree; the walk stays bounded)
        // od_quantize_haar_dc_level(2 bx, 2 by, bsi - 1), src/encode.c:1592-1657
        const int bsi = n.bsi - 1, bx = 2 * n.bx, by = 2 * n.by;
        const int ln = bsi - xdec + 2;
        const int acq0 = (dq * kDcQm[bsi - xdec][0] + 8) >> 4, acq1 = (dq * kDcQm[bsi - xdec][1] + 8) >> 4;
        const int y0 = by << ln, y1 = (by + 1) << ln, x0 = bx << ln, x1 = (bx + 1) << ln;
        int x[4];
        x[0] = dc[(y0 >> 2) * gw + (x0 >> 2)];
        x[1] = d[(size_t)y0 * pw + x1] - n.hgrad / 5;
        x[2] = d[(size_t)y1 * pw + x0] - n.vgrad / 5;
        x[3] = d[(size_t)y1 * pw + x1];
        const int at[4] = {(y0 >> 2) * gw + (x0 >> 2), (y0 >> 2) * gw + (x1 >> 2), (y1 >> 2) * gw + (x0 >> 2),
                           (y1 >> 2) * gw + (x1 >> 2)};
#pragma unroll 1
        for (int i = 1; i < 4; i++) {
          const int q = i == 3 ? acq1 : acq0;
          const bool sign = x[i] < 0;
          const int a = abs(x[i]);
          int* ex = &ex_dc[bsi][i - 1];
          int qi = a / q;
          double cost = gen_cost(cdfs, qi + 1, *ex);
          cost -= gen_cost(cdfs, qi, *ex);
          if (qi == 0) cost += 1;
          if (q * q - 2 * q * (a - qi * q) + q * q * lam * cost < 0) qi++;
          gen_adapt(cdfs, qi, ex);
          idx[at[i]] = sign ? -qi : qi;
          x[i] = sign ? -qi * q : qi * q;
        }
        x[1] += n.hgrad / 5;
        x[2] += n.vgrad / 5;
        const int hg = x[1], vg = x[2];
        // OD_HAAR_KERNEL(x[0], x[1], x[2], x[3]), src/tf.h:34
        int ll = x[0], lh = x[1], hl = x[2], hh = x[3];
        ll += hl;
        hh -= lh;
        const int t = (ll - hh) >> 1;
        lh = t - lh;
        hl = t - hl;
        ll -= lh;
        hh += hl;
        dc[at[0]] = ll;
        dc[at[1]] = lh;
        dc[at[2]] = hl;
        dc[at[3]] = hh;
        stack[sp++] = Node{bx + 1, by + 1, bsi, hg, vg};
        stack[sp++] = Node{bx, by + 1, bsi, hg, vg};
        stack[sp++] = Node{bx + 1, by, bsi, hg, vg};
        stack[sp++] = Node{bx, by, bsi, hg, vg};
      }
    }
  }
}

}  // namespace haar_dc
}  // namespace daala_b200

extern "C" int daala_b200_launch_haar_dc(const daala_b200_haar_dc_batch* b, cudaStream_t stream) {
  using namespace daala_b200::haar_dc;
  k_haar_dc<<<b->F * 3, 32, sizeof(int) * 2 * b->nhsb, stream>>>(*b);
  return (int)cudaGetLastError();
}
