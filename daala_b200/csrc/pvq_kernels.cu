// PVQ band quantisation kernels for sm_90a (H100).
//
// k_pvq_bands<NMAX>: one THREAD quantises one band (partition) of one
//   transform block -- the full gain / theta / K candidate search of the
//   reference's pvq_theta (src/pvq_encoder.c:333) including the double
//   precision pulse search pvq_search_rdo_double (:93), the closed-form rate of
//   od_pvq_rate (:247, speed > 0 branch) and the decoder-identical synthesis
//   od_pvq_synthesis_partial (src/pvq.c:1037).  The host sorts bands into size
//   classes (n = 15/8, 32, 128) so the threads of a warp run the same loop
//   bounds; per-thread scratch lives in (interleaved, hence coalesced) local
//   memory.  Every double-precision expression keeps the reference's
//   operation order (library is built with -fmad=false) so that the chosen
//   indices (qg, theta, K, pulses) are bit-exact.
// k_coding_order_gather / _scatter: raster <-> coding order of whole block
//   lists (od_raster_to_coding_order, od_coding_order_to_raster,
//   src/partition.c:123/157, od_init_skipped_coeffs src/state.c:1347).
// k_cfl_flip: keyframe-chroma CfL sign decision (src/pvq_encoder.c:847-871).
// k_block_skip_diff: ordered per-block sum of the bands' skip_diff terms.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "daala_b200.h"
#include "gen/coding_order.inc"
#include "pvq_math.cuh"
#include "pvq_coop.cuh"
#include "pvq_common.cuh"

namespace daala_b200 {
namespace pvq {

constexpr int kSkipZero = 1;
constexpr int kSkipCopy = 2;

__device__ __forceinline__ double rsqrt_small(int i) { return rsqrt_small_tbl(i); }

// src/pvq_encoder.c:93.  x[] (|xcoeff| as double) is caller scratch of n entries.
__device__ __noinline__ double search_rdo(const int16_t* xcoeff, int n, int k, int32_t* ypulse, double g2,
                             double pvq_norm_lambda, int prev_k, double* x) {
  double xx = 0, xy = 0, yy = 0;
  for (int j = 0; j < n; j++) {
    x[j] = fabs((double)(float)xcoeff[j]);
    xx += x[j] * x[j];
  }
  double norm_1 = 1. / sqrt(1e-30 + xx);
  double lambda = pvq_norm_lambda / (1e-30 + g2);
  int i = 0;
  if (prev_k > 0 && prev_k <= k) {
    for (int j = 0; j < n; j++) {
      ypulse[j] = abs(ypulse[j]);
      xy += x[j] * ypulse[j];
      yy += ypulse[j] * ypulse[j];
      i += ypulse[j];
    }
  } else if (k > 2) {
    double l1_norm = 0;
    for (int j = 0; j < n; j++) l1_norm += x[j];
    double l1_inv = 1. / (l1_norm > 1e-100 ? l1_norm : 1e-100);
    for (int j = 0; j < n; j++) {
      double tmp = k * x[j] * l1_inv;
      int f = (int)floor(tmp);
      ypulse[j] = f > 0 ? f : 0;
      xy += x[j] * ypulse[j];
      yy += ypulse[j] * ypulse[j];
      i += ypulse[j];
    }
  } else {
    for (int j = 0; j < n; j++) ypulse[j] = 0;
  }
  int rdo_pulses = 1 + k / 4;
  double delta_rate = 3. / n;
  double accel_rate = 0.;
  if (k == 1) {
    if (n == 15) {
      accel_rate = -8. / n;
      delta_rate = 4.5 / n - accel_rate;
    } else if (n == 8) {
      accel_rate = 5.7 / n;
      delta_rate = 9.3 / n - accel_rate;
    }
  }
  for (; i < k - rdo_pulses; i++) {
    int pos = 0;
    double best_xy = -10, best_yy = 1;
    for (int j = 0; j < n; j++) {
      double tmp_xy = xy + x[j];
      double tmp_yy = yy + 2 * ypulse[j] + 1;
      tmp_xy *= tmp_xy;
      if (j == 0 || tmp_xy * best_yy > best_xy * tmp_yy) {
        best_xy = tmp_xy;
        best_yy = tmp_yy;
        pos = j;
      }
    }
    xy = xy + x[pos];
    yy = yy + 2 * ypulse[pos] + 1;
    ypulse[pos]++;
  }
  for (; i < k; i++) {
    double tbl[4];
    int pos = 0;
    double best_cost = -1e5;
    for (int j = 0; j < 4; j++) tbl[j] = rsqrt_small((int)(yy + 2 * j + 1));
    for (int j = 0; j < n; j++) {
      double tmp_xy = xy + x[j];
      int yj = ypulse[j];
      double tmp_yy = yj < 4 ? (yj == 0 ? tbl[0] : yj == 1 ? tbl[1] : yj == 2 ? tbl[2] : tbl[3])
                             : rsqrt_small((int)(yy + 2 * yj + 1));
      tmp_xy = 2 * tmp_xy * norm_1 * tmp_yy - lambda * j * (delta_rate + j * accel_rate);
      if (j == 0 || tmp_xy > best_cost) {
        best_cost = tmp_xy;
        pos = j;
      }
    }
    xy = xy + x[pos];
    yy = yy + 2 * ypulse[pos] + 1;
    ypulse[pos]++;
  }
  for (int j = 0; j < n; j++)
    if (xcoeff[j] < 0) ypulse[j] = -ypulse[j];
  return xy / (1e-100 + sqrt(xx * yy));
}

// src/pvq_encoder.c:247, closed-form branch.
__device__ __noinline__ double band_rate(int qg, int icgr, int theta, int ts, const int32_t* y0, int k, int n,
                            int is_keyframe, int pli) {
  double rate;
  if (k == 0) {
    rate = 0;
  } else {
    int sum = 0;
    for (int i = 0; i < n - (theta != -1); i++) sum += i * abs(y0[i]);
    double f = sum / (double)(k * n);
    double t = log(n * 2 * (1 * f + .025)) * k / n;
    rate = (1 + .4 * f) * n * (M_LOG2E * log(1 + (0 > t ? 0 : t))) + 3;
  }
  if (qg > 0 && theta >= 0) {
    rate += .9 * (M_LOG2E * log((double)ts));
    if (is_keyframe && pli == 0) rate += 6;
    if (qg == icgr) rate -= .5;
  }
  return rate;
}

__device__ __forceinline__ int neg_interleave(int x, int ref) {
  if (x < ref) return -2 * (x - ref) - 1;
  if (x < 2 * ref) return 2 * (x - ref);
  return x - 1;
}

__device__ __noinline__ int householder_setup(int16_t* r, int n, int32_t gr, int* sign, int shift) {
  int m = 0;
  int16_t maxr = 0;
  for (int i = 0; i < n; i++) {
    int a = abs((int)r[i]);
    if (a > maxr) {
      maxr = (int16_t)a;
      m = i;
    }
  }
  int s = r[m] > 0 ? 1 : -1;
  r[m] = (int16_t)(r[m] + shr_round(gr * s, shift));
  *sign = s;
  return m;
}

__device__ __noinline__ void householder_apply(int16_t* out, const int16_t* x, const int16_t* r, int n) {
  int32_t l2r = 0, proj = 0;
  for (int i = 0; i < n; i++) l2r += mul16(r[i], r[i]);
  for (int i = 0; i < n; i++) proj += mul16(r[i], x[i]);
  int l2r_shift = (ilog((uint32_t)l2r) - 1) - 14;
  int16_t l2r_norm = (int16_t)vshr_round(l2r, l2r_shift);
  int16_t rcp = rcp16(l2r_norm);
  int proj_shift = (ilog((uint32_t)abs(proj)) - 1) - 14;
  int16_t proj_norm = (int16_t)vshr_round(proj, proj_shift);
  int16_t proj_1 = (int16_t)mul16_q15(proj_norm, rcp);
  int outshift = 14 - proj_shift - 1 + l2r_shift;
  if (outshift > 30) outshift = 30;
  if (outshift >= 0) {
    for (int i = 0; i < n; i++) out[i] = (int16_t)(x[i] - shr_round(mul16(r[i], proj_1), outshift));
  } else {
    for (int i = 0; i < n; i++) out[i] = (int16_t)(x[i] - shl(mul16(r[i], proj_1), -outshift));
  }
}

__device__ __noinline__ void synthesis(int32_t* xcoeff, const int32_t* ypulse, const int16_t* r16, int n, int noref,
                          int32_t g, int32_t theta, int m, int s, const int16_t* qm_inv, int16_t* xs) {
  int nn = n - !noref;
  int yy = 0;
  for (int i = 0; i < nn; i++) yy += ypulse[i] * (int32_t)ypulse[i];
  int gshift = ilog((uint32_t)g) - 14;
  if (gshift < 0) gshift = 0;
  int32_t scale;
  if (yy == 0) {
    scale = 0;
  } else {
    int rshift;
    int16_t rs = rsqrt32(yy, &rshift);
    scale = vshr_round64(rs * (int64_t)g, rshift + gshift - 16);
  }
  int qshift = kQmInvShift - gshift;
  if (noref) {
    for (int i = 0; i < n; i++) {
      int32_t x = mul16_32_q16(ypulse[i], scale);
      xcoeff[i] = shr_round(x * qm_inv[i], qshift);
    }
  } else {
    scale = round32(scale * (1. / 32768) * pvq_sin(theta));
    for (int i = 0; i < m; i++) xs[i] = (int16_t)mul16_32_q16(ypulse[i], scale);
    xs[m] = (int16_t)floor(.5 + -s * (shr_round(g, gshift)) * (1. / 32768) * pvq_cos(theta));
    for (int i = m; i < nn; i++) xs[i + 1] = (int16_t)mul16_32_q16(ypulse[i], scale);
    householder_apply(xs, xs, r16, n);
    for (int i = 0; i < n; i++) xcoeff[i] = shr_round(xs[i] * qm_inv[i], qshift);
  }
}

struct Cand {
  int gain, k, theta, ts;
  int32_t qtheta, qcg;
};

// One band.  Returns the coded gain index; results through pointers.
template <int NMAX>
__device__ int quantise_band(int32_t* out, const int32_t* x0, const int32_t* r0, int n, int q0, int32_t* y,
                             int* itheta, int* max_theta, int* vk, int beta, double* skip_term,
                             int is_keyframe, int pli, const int16_t* qm, const int16_t* qm_inv,
                             double pvq_norm_lambda) {
  const double gain_weight = 1.4;
  const double cgain_1 = 1. / kCgainOne;
  const double cgain_2 = cgain_1 * cgain_1;
  const double theta_scale = (1 << kThetaShift) * 2. / M_PI;
  const double theta_scale_1 = 1. / theta_scale;
  const double trig_1 = 1. / 32768;
  int32_t y_tmp[NMAX];
  int16_t x16[NMAX];
  int16_t r16[NMAX];
  int16_t xr[NMAX];
  double xd[NMAX];
  int32_t g, gr;
  int32_t theta = 0, best_qtheta = 0;
  int qg = 0, best_k = 0, noref = 1, m = 0, s = 1, skip = 0;
  int r_is_null = 1;
  double corr = 0;
  // od_vector_log_mag, src/pvq.c:472
  int xshift, rshift;
  {
    int32_t sx = 0, sr = 0;
    for (int i = 0; i < n; i++) {
      int16_t tx = (int16_t)(x0[i] >> 8), tr = (int16_t)(r0[i] >> 8);
      sx += tx * (int32_t)tx;
      sr += tr * (int32_t)tr;
    }
    xshift = 9 + ilog((uint32_t)(n + sx)) / 2 - 15;
    rshift = 9 + ilog((uint32_t)(n + sr)) / 2 - 14;
    if (xshift < 0) xshift = 0;
    if (rshift < 0) rshift = 0;
  }
  int32_t accx = 0, accr = 0;
  for (int i = 0; i < n; i++) {
    x16[i] = (int16_t)shr_round(x0[i] * qm[i], kQmShift + xshift);
    r16[i] = (int16_t)shr_round(r0[i] * qm[i], kQmShift + rshift);
    corr += mul16(x16[i], r16[i]);
    accx += x16[i] * (int32_t)x16[i];
    accr += r16[i] * (int32_t)r16[i];
    if (r0[i]) r_is_null = 0;
  }
  const int cfl_enabled = is_keyframe && pli != 0;
  int32_t cg = compute_gain_from_energy(accx, q0, &g, beta, xshift);
  int32_t cgr = compute_gain_from_energy(accr, q0, &gr, beta, rshift);
  if (cfl_enabled) cgr = kCgainOne;
  int icgr = shr_round(cgr, kCgainShift);
  int32_t gain_offset = cgr - shl(icgr, kCgainShift);
  double dist = gain_weight * cg * cg * cgain_2;
  double best_dist = dist;
  double best_cost = dist + pvq_norm_lambda * band_rate(0, 0, -1, 0, nullptr, 0, n, is_keyframe, pli);
  *itheta = -1;
  *max_theta = 0;
  for (int i = 0; i < n; i++) y[i] = 0;
  corr = corr / (1e-100 + g * (double)gr / shl(1, xshift + rshift));
  corr = corr < 1. ? corr : 1.;
  corr = corr > -1. ? corr : -1.;
  double skip_dist;
  if (is_keyframe) {
    skip_dist = gain_weight * cg * cg * cgain_2;
  } else {
    skip_dist = gain_weight * (cg - cgr) * (cg - cgr) + cgr * (double)cg * (2 - 2 * corr);
    skip_dist *= cgain_2;
  }
  if (!is_keyframe) {
    int32_t scgr = gain_offset > 0 ? gain_offset : 0;
    if (icgr == 0) {
      best_dist = gain_weight * (cg - scgr) * (cg - scgr) + scgr * (double)cg * (2 - 2 * corr);
      best_dist *= cgain_2;
    }
    best_cost = best_dist + pvq_norm_lambda * band_rate(0, icgr, 0, 0, nullptr, 0, n, is_keyframe, pli);
    best_qtheta = 0;
    *itheta = 0;
    *max_theta = 0;
    noref = 0;
  }
  const double dist0 = best_dist;
  if (!r_is_null && corr > 0) {
    Cand items[20];
    int nitems = 0;
    int gain_bound = (cg - gain_offset) >> kCgainShift;
    int prev_k = 0;
    double cos_dist = 0;
    theta = round32(theta_scale * acos(corr));
    m = householder_setup(r16, n, gr, &s, rshift);
    householder_apply(xr, x16, r16, n);
    for (int i = m; i < n - 1; i++) xr[i] = xr[i + 1];
    for (int i = gain_bound - 1 > 1 ? gain_bound - 1 : 1; i <= gain_bound + 1; i++) {
      int32_t qcg = shl(i, kCgainShift) + gain_offset;
      int ts = compute_max_theta(qcg, beta);
      int lo = (int)floor(.5 + theta * theta_scale_1 * 2 / M_PI * ts) - 2;
      int hi = (int)ceil(theta * theta_scale_1 * 2 / M_PI * ts);
      if (lo < 0) lo = 0;
      if (hi > ts - 1) hi = ts - 1;
      for (int j = lo; j <= hi; j++) {
        Cand c;
        c.gain = i;
        c.theta = j;
        c.qtheta = compute_theta(j, ts);
        c.k = compute_k(qcg, j, 0, n, beta);
        c.qcg = qcg;
        c.ts = ts;
        // stable insertion by (k, gain): the order glibc's merge-sort qsort
        // produces at src/pvq_encoder.c:504
        int p = nitems++;
        while (p > 0 && (items[p - 1].k > c.k || (items[p - 1].k == c.k && items[p - 1].gain > c.gain))) {
          items[p] = items[p - 1];
          p--;
        }
        items[p] = c;
      }
    }
    for (int idx = 0; idx < nitems; idx++) {
      const Cand c = items[idx];
      const int32_t qcg = c.qcg, qtheta = c.qtheta;
      const int k = c.k;
      double dist_theta = 2 - 2. * pvq_cos(theta - qtheta) * trig_1;
      dist = gain_weight * (qcg - cg) * (qcg - cg) + qcg * (double)cg * dist_theta;
      dist *= cgain_2;
      if (dist > dist0 + 1.0 * pvq_norm_lambda && k != 0) continue;
      double sin_prod = pvq_sin(theta) * trig_1 * pvq_sin(qtheta) * trig_1;
      if (k == 0) {
        cos_dist = 0;
        for (int i = 0; i < n - 1; i++) y_tmp[i] = 0;
      } else if (k != prev_k) {
        cos_dist = search_rdo(xr, n - 1, k, y_tmp, qcg * (double)cg * sin_prod * cgain_2, pvq_norm_lambda,
                              prev_k, xd);
      }
      prev_k = k;
      dist_theta = 2 - 2. * pvq_cos(theta - qtheta) * trig_1 + sin_prod * (2 - 2 * cos_dist);
      dist = gain_weight * (qcg - cg) * (qcg - cg) + qcg * (double)cg * dist_theta;
      dist *= cgain_2;
      double cost = dist + pvq_norm_lambda * band_rate(c.gain, icgr, c.theta, c.ts, y_tmp, k, n, is_keyframe, pli);
      if (cost < best_cost) {
        best_cost = cost;
        best_dist = dist;
        qg = c.gain;
        best_k = k;
        best_qtheta = qtheta;
        *itheta = c.theta;
        *max_theta = c.ts;
        noref = 0;
        for (int i = 0; i < n - 1; i++) y[i] = y_tmp[i];
      }
    }
  }
  if ((is_keyframe && pli == 0) || corr < .5 || cg < (int32_t)shl(2, kCgainShift)) {
    int gain_bound = cg >> kCgainShift;
    int prev_k = 0;
    for (int i = gain_bound > 1 ? gain_bound : 1; i <= gain_bound + 1; i++) {
      int32_t qcg = shl(i, kCgainShift);
      int k = compute_k(qcg, -1, 1, n, beta);
      dist = gain_weight * (qcg - cg) * (qcg - cg);
      dist *= cgain_2;
      if (dist > dist0 && k != 0) continue;
      double cos_dist = search_rdo(x16, n, k, y_tmp, qcg * (double)cg * cgain_2, pvq_norm_lambda, prev_k, xd);
      prev_k = k;
      dist = gain_weight * (qcg - cg) * (qcg - cg) + qcg * (double)cg * (2 - 2 * cos_dist);
      dist *= cgain_2;
      double cost = dist + pvq_norm_lambda * band_rate(i, 0, -1, 0, y_tmp, k, n, is_keyframe, pli);
      if (cost <= best_cost) {
        best_cost = cost;
        best_dist = dist;
        qg = i;
        noref = 1;
        best_k = k;
        *itheta = -1;
        *max_theta = 0;
        for (int j = 0; j < n; j++) y[j] = y_tmp[j];
      }
    }
  }
  theta = best_qtheta;
  if (noref) {
    if (qg == 0) skip = kSkipZero;
  } else {
    if (!is_keyframe && qg == 0) skip = icgr ? kSkipZero : kSkipCopy;
    if (qg == icgr && *itheta == 0 && !cfl_enabled) skip = kSkipCopy;
  }
  if (skip) {
    if (skip == kSkipCopy) {
      for (int i = 0; i < n; i++) out[i] = r0[i];
    } else {
      for (int i = 0; i < n; i++) out[i] = 0;
    }
  } else {
    if (noref) gain_offset = 0;
    g = gain_expand(shl(qg, kCgainShift) + gain_offset, q0, beta);
    synthesis(out, y, r16, n, noref, g, theta, m, s, qm_inv, xr);
  }
  *vk = best_k;
  *skip_term = skip_dist - best_dist;
  if (is_keyframe) return noref ? qg : neg_interleave(qg, icgr);
  return noref ? qg - 1 : neg_interleave(qg + 1, icgr + 1);
}

// ---------------------------------------------------------------------------
// Kernels
// ---------------------------------------------------------------------------

// band_list entries: (block index << 4) | band index.
template <int NMAX, int kMinCtas = 4>
__global__ void __launch_bounds__(128, kMinCtas)
k_pvq_bands(const __grid_constant__ daala_b200_pvq_params prm, const uint32_t* __restrict__ band_list,
            int count) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  const uint32_t e = band_list[t];
  const int blk = (int)(e >> 4), band = (int)(e & 15);
  const daala_b200_pvq_block b = prm.blocks[blk];
  const int bs = b.bs, pli = b.pli;
  const int start = band_start(band);
  const int n = band_start(band + 1) - start;
  const size_t off = (size_t)b.coef_off + start;
  // quantiser of this band: od_pvq_encode, src/pvq_encoder.c:873-874
  int qidx = bs * (bs + 1) + (band + 1) - (band + 1) / 3;
  int q = (prm.q0 * prm.pvq_qm_q4[pli][qidx]) >> 4;
  if (q < 1) q = 1;
  // OD_PVQ_BETA, src/pvq.c:205-268: 1.5 only on luma with masking, sizes > 4x4
  const int beta = (prm.use_masking && pli == 0 && bs > 0) ? kBeta15 : kBeta1;
  // od_qm_offset(bs, xdec), src/pvq.c:306
  const int qoff = (b.xdec ? prm.qm_stride : 0) + ((((1 << (2 * bs)) - 1) << 4) / 3) + start;
  int itheta, max_theta, k;
  double skip_term;
  int32_t* y = prm.y + off;
  int gain = quantise_band<NMAX>(prm.out + off, prm.in + off, prm.ref + off, n, q, y, &itheta, &max_theta, &k,
                                 beta, &skip_term, prm.is_keyframe, pli, prm.qm + qoff, prm.qm_inv + qoff,
                                 prm.pvq_norm_lambda);
  const size_t r = (size_t)blk * 9 + band;
  prm.res_gain[r] = gain;
  prm.res_theta[r] = itheta;
  prm.res_max_theta[r] = max_theta;
  prm.res_k[r] = k;
  prm.res_skip_term[r] = skip_term;
}

// Group-cooperative variant (pvq_coop.cuh): G lanes per band, registers only.
template <int G, int E, bool kForceScan, int kMinCtas = 4>
__global__ void __launch_bounds__(128, kMinCtas)
k_pvq_bands_coop(const __grid_constant__ daala_b200_pvq_params prm, const uint32_t* __restrict__ band_list,
                 int count) {
  const Group<G, E> grp;
  constexpr int kBandsPerCta = 128 / G;
  const int t = blockIdx.x * kBandsPerCta + (threadIdx.x / G);
  // whole groups leave together; partial warps keep the shuffle masks valid
  if (t >= count) return;
  const uint32_t e = band_list[t];
  const int blk = (int)(e >> 4), band = (int)(e & 15);
  const daala_b200_pvq_block b = prm.blocks[blk];
  const int bs = b.bs, pli = b.pli;
  const int start = band_start(band);
  const int n = band_start(band + 1) - start;
  const size_t off = (size_t)b.coef_off + start;
  int qidx = bs * (bs + 1) + (band + 1) - (band + 1) / 3;
  int q = (prm.q0 * prm.pvq_qm_q4[pli][qidx]) >> 4;
  if (q < 1) q = 1;
  const int beta = (prm.use_masking && pli == 0 && bs > 0) ? kBeta15 : kBeta1;
  const int qoff = (b.xdec ? prm.qm_stride : 0) + ((((1 << (2 * bs)) - 1) << 4) / 3) + start;
  int itheta, max_theta, k;
  double skip_term;
  int gain = quantise_band_coop<G, E, kForceScan>(grp, prm.out + off, prm.in + off, prm.ref + off, n, q,
                                                  prm.y + off, &itheta, &max_theta, &k, beta, &skip_term,
                                                  prm.is_keyframe, pli, prm.qm + qoff, prm.qm_inv + qoff,
                                                  prm.pvq_norm_lambda);
  if (grp.lane == 0) {
    const size_t r = (size_t)blk * 9 + band;
    prm.res_gain[r] = gain;
    prm.res_theta[r] = itheta;
    prm.res_max_theta[r] = max_theta;
    prm.res_k[r] = k;
    prm.res_skip_term[r] = skip_term;
  }
}

// ---------------------------------------------------------------------------
// Work ordering.  The trip counts of the search (candidates x pulses) grow with the band's gain, and
// the lanes of a warp wait for the slowest one: a launch whose entries are grouped by expected work
// runs 1.3-2x faster than the same entries in raster order (measured on real data).  Results are
// stored per (block, band), so the order inside a launch is free.  Three small kernels bucket a band
// list by (wave, work bin), heaviest first: keys + histogram, exclusive scan, scatter.
// ---------------------------------------------------------------------------
constexpr int kMaxOrderBins = 8192;   // bins of one ordering call: waves x bins per wave
constexpr int kMaxWaveBins = 2048;

// G lanes per entry.  Work proxy: energy of the band relative to its quantiser, scaled by n^2
// (K grows with gain / q, the search costs K x n), binned on a log scale: bins_per_wave / 32 bins per
// octave.  The bins must be fine: K steps with the quantised gain, and a launch only runs at the
// speed of a fully sorted one when neighbouring entries share K (measured: 64 half-octave bins gave
// none of the gain of a full sort on the CfL chroma bands, whose energies cluster within an octave).
template <int G>
__global__ void __launch_bounds__(256)
k_band_work_keys(const __grid_constant__ daala_b200_pvq_params prm, const uint32_t* __restrict__ band_list,
                 const uint16_t* __restrict__ entry_wave, int count, int bins_per_wave,
                 uint16_t* __restrict__ keys, int* __restrict__ hist) {
  const int slot = (blockIdx.x * blockDim.x + threadIdx.x) / G, lane = threadIdx.x % G;
  const bool valid = slot < count;
  float acc = 0.f;
  int n = 1, q = 1;
  if (valid) {
    const uint32_t e = band_list[slot];
    const int blk = (int)(e >> 4), band = (int)(e & 15);
    const daala_b200_pvq_block b = prm.blocks[blk];
    const int start = band_start(band);
    n = band_start(band + 1) - start;
    const int qidx = b.bs * (b.bs + 1) + (band + 1) - (band + 1) / 3;
    q = (prm.q0 * prm.pvq_qm_q4[b.pli][qidx]) >> 4;
    if (q < 1) q = 1;
    const int32_t* x = prm.in + (size_t)b.coef_off + start;
    for (int i = lane; i < n; i += G) {
      const float v = (float)x[i];
      acc += v * v;
    }
  }
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o, G);
  if (valid && lane == 0) {
    const float w = acc * (float)(n * n) / ((float)q * (float)q);
    int bin = (int)(log2f(w + 1.f) * (float)bins_per_wave * (1.f / 32.f));
    bin = bin < 0 ? 0 : bin > bins_per_wave - 1 ? bins_per_wave - 1 : bin;
    const int wave = entry_wave ? entry_wave[slot] : 0;
    const int key = wave * bins_per_wave + (bins_per_wave - 1 - bin);
    keys[slot] = (uint16_t)key;
    atomicAdd(&hist[key], 1);
  }
}

// hist[0..nbins) -> exclusive prefix sums in place (nbins <= kMaxOrderBins, one CTA of 1024 threads)
__global__ void __launch_bounds__(1024) k_bin_scan(int* __restrict__ hist, int nbins) {
  __shared__ int part[1024];
  constexpr int kPer = kMaxOrderBins / 1024;
  const int t = threadIdx.x;
  int v[kPer], sum = 0;
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    const int j = t * kPer + i;
    v[i] = j < nbins ? hist[j] : 0;
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
    const int j = t * kPer + i;
    if (j < nbins) hist[j] = run;
    run += v[i];
  }
}

__global__ void __launch_bounds__(256)
k_bin_scatter(const uint32_t* __restrict__ band_list, const uint16_t* __restrict__ keys, int count,
              int* __restrict__ cursor, uint32_t* __restrict__ ordered) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= count) return;
  const int key = keys[slot];
  const unsigned active = __activemask();
  const unsigned same = __match_any_sync(active, key);
  const int leader = __ffs(same) - 1, lane = threadIdx.x & 31;
  int base = 0;
  if (lane == leader) base = atomicAdd(&cursor[key], __popc(same));
  base = __shfl_sync(same, base, leader);
  ordered[base + __popc(same & ((1u << lane) - 1u))] = band_list[slot];
}

// Per block: ordered sum of the bands' skip_diff terms (`*skip_diff += ...`
// runs over the bands in order at src/pvq_encoder.c:875-880; double addition
// is not associative, so the order is kept) and the DC coefficient:
// keyframes keep the Haar-coded DC (scalar_out[0] = dblock[0],
// src/encode.c:1381); inter frames use the plain scalar quantiser of
// src/encode.c:1337-1344 and reconstruct it as in :1377-1378.
__global__ void k_block_finish(const __grid_constant__ daala_b200_pvq_params prm, int first, int nblocks) {
  int blk = blockIdx.x * blockDim.x + threadIdx.x;
  if (blk >= nblocks) return;
  blk += first;
  const daala_b200_pvq_block b = prm.blocks[blk];
  int nb = num_bands(b.bs);
  double sd = 0;
  for (int i = 0; i < nb; i++) sd += prm.res_skip_term[(size_t)blk * 9 + i];
  prm.res_skip_diff[blk] = sd;
  const int32_t in0 = prm.in[b.coef_off], ref0 = prm.ref[b.coef_off];
  if (prm.is_keyframe) {
    prm.out[b.coef_off] = in0;
    prm.res_dc[blk] = 0;
  } else {
    int dc_quant = (prm.q0 * prm.pvq_qm_q4[b.pli][b.bs * (b.bs + 1)]) >> 4;
    if (dc_quant < 1) dc_quant = 1;
    int diff = in0 - ref0;
    int qdc;
    if (abs(diff) < dc_quant * 141 / 256) {
      qdc = 0;
    } else {
      // OD_DIV_R0(diff, dc_quant), src/odintrin.h:123
      int half = ((dc_quant + 1) >> 1) - 1;
      qdc = (diff + (diff < 0 ? -half : half)) / dc_quant;
    }
    prm.res_dc[blk] = qdc;
    prm.out[b.coef_off] = qdc * dc_quant + ref0;
  }
}

// Keyframe chroma: decide the CfL flip from the first band and negate the
// reference of the whole block when cos(theta) < 0 (src/pvq_encoder.c:847-871).
__global__ void k_cfl_flip(const __grid_constant__ daala_b200_pvq_params prm, int nblocks) {
  int blk = blockIdx.x * blockDim.x + threadIdx.x;
  if (blk >= nblocks) return;
  const daala_b200_pvq_block b = prm.blocks[blk];
  int flip = 0;
  if (b.pli != 0 && prm.is_keyframe) {
    const int bs = b.bs;
    const int qoff = (b.xdec ? prm.qm_stride : 0) + ((((1 << (2 * bs)) - 1) << 4) / 3);
    const int32_t* in = prm.in + b.coef_off;
    int32_t* ref = prm.ref + b.coef_off;
    int32_t xy = 0;
    for (int i = 1; i < 16; i++) {
      int32_t rq = ref[i] * prm.qm[qoff + i];
      int32_t inq = in[i] * prm.qm[qoff + i];
      // OD_SHR(rq*(int64_t)inq, OD_SHL(OD_QM_SHIFT + OD_CFL_FLIP_SHIFT, 1)), OD_CFL_FLIP_SHIFT = 4
      xy += (int32_t)((rq * (int64_t)inq) >> ((kQmShift + 4) << 1));
    }
    if (xy < 0) {
      flip = 1;
      const int end = band_start(num_bands(bs));
      for (int i = 1; i < end; i++) ref[i] = -ref[i];
    }
  }
  prm.res_flip[blk] = flip;
}

// Raster (block inside a coefficient plane) -> coding order, one warp per block.
// Only the coded prefix is produced: n^2 for n <= 16, 512 for 32 and 64
// (OD_LAYOUT32/64 in src/partition.c:40-55 cover nothing beyond it).
__global__ void k_coding_order_gather(const __grid_constant__ daala_b200_pvq_params prm, int nblocks,
                                      int which /*0: in <- coeffs, 1: ref <- pred*/) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= nblocks) return;
  const daala_b200_pvq_block b = prm.blocks[warp];
  const int ln = b.bs + 2;
  const int len = ln >= 5 ? 512 : 1 << (2 * ln);
  const int32_t* plane = which ? prm.pred_plane[b.pli] : prm.coef_plane[b.pli];
  if (plane) plane += b.frame * prm.plane_frame_pitch[b.pli];
  const int stride = prm.plane_stride[b.pli];
  int32_t* dst = (which ? prm.ref : prm.in) + b.coef_off;
  if (plane == nullptr) {
    for (int i = lane; i < len; i += 32) dst[i] = 0;
    return;
  }
  const int32_t* src = plane + (size_t)b.y0 * stride + b.x0;
  for (int i = lane; i < len; i += 32) dst[i] = i == 0 ? src[0] : src[scan_to_raster(i, ln, stride)];
}

// Coding order -> raster, with od_init_skipped_coeffs first (keyframe: zero
// everything but DC; otherwise copy the prediction), then the coded prefix.
// DC: the keyframe path keeps the block's (Haar-coded) DC, src/encode.c:1384.
__global__ void k_coding_order_scatter(const __grid_constant__ daala_b200_pvq_params prm, int first, int nblocks) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= nblocks) return;
  const daala_b200_pvq_block b = prm.blocks[first + warp];
  const int ln = b.bs + 2, n = 1 << ln;
  const int len = ln >= 5 ? 512 : 1 << (2 * ln);
  const int stride = prm.plane_stride[b.pli];
  const long long fp = b.frame * prm.plane_frame_pitch[b.pli];
  int32_t* dst = prm.coef_plane[b.pli] + fp + (size_t)b.y0 * stride + b.x0;
  const int32_t* pred = prm.pred_plane[b.pli] ? prm.pred_plane[b.pli] + fp + (size_t)b.y0 * stride + b.x0 : nullptr;
  const int32_t* src = prm.out + b.coef_off;
  if (ln >= 5) {
    for (int i = lane; i < n * n; i += 32) {
      int r = i >> ln, c = i & (n - 1);
      if (prm.is_keyframe) {
        if (i) dst[r * stride + c] = 0;
      } else {
        dst[r * stride + c] = pred ? pred[r * stride + c] : 0;
      }
    }
    __syncwarp();
  }
  for (int i = lane; i < len; i += 32) {
    if (i == 0) {
      if (!prm.is_keyframe) dst[0] = src[0];
    } else {
      dst[scan_to_raster(i, ln, stride)] = src[i];
    }
  }
  if (prm.y16) {
    const int32_t* y = prm.y + b.coef_off;
    for (int i = lane; i < len; i += 32) prm.y16[b.coef_off + i] = (int16_t)y[i];
  }
}

// Keyframe luma with the reference's H/V intra prediction (od_hv_intra_pred, src/intra.c:37): the
// prediction of a block is row 0 / column 0 of the QUANTISED coefficients of its top / left neighbour
// of the same size, so blocks form dependency chains (SURVEY.md 0.8).  It is built band by band:
// od_hv_intra_pred only fills row 0 and column 0 of the block (src/intra.c:53-60), and the neighbour
// it reads has the SAME size, so coefficient (0, c) / (r, 0) sits at the same coding-order index -- and
// in the same band -- in both blocks: band b of a block depends on band b of its top / left neighbour
// only.  Of the bands of OD_BAND_OFFSETS, 1/4/7
// hold row-0 coefficients (top chain only), 2/5/8 column-0 coefficients (left chain only), 3/6 neither
// (no dependency at all) and 0 the three low coefficients of each, whose source is chosen by the
// neighbours' energies (:51-52, :55-60) -- again band-0 values only.  One warp per band-list entry
// writes that band's slice of `ref` from the neighbours' `out` (coding order, already dequantised).
__global__ void k_intra_band_ref(const __grid_constant__ daala_b200_pvq_params prm,
                                 const int32_t* __restrict__ dep_top, const int32_t* __restrict__ dep_left,
                                 const uint32_t* __restrict__ band_list, int count) {
  const int slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (slot >= count) return;
  const uint32_t e = band_list[slot];
  const int blk = (int)(e >> 4), band = (int)(e & 15);
  const int t = dep_top[blk], l = dep_left[blk];
  const int32_t* ot = t >= 0 ? prm.out + prm.blocks[t].coef_off : nullptr;
  const int32_t* ol = l >= 0 ? prm.out + prm.blocks[l].coef_off : nullptr;
  bool low_from_top = false;
  if (band == 0) {
    // coding-order indices of (0,1) (0,2) (0,3) and (1,0) (2,0) (3,0) in OD_ZIGZAG4
    double g1 = 0, g2 = 0;
    if (ot) { double a = ot[2], b = ot[5], c = ot[9]; g1 += a * a; g1 += b * b; g1 += c * c; }
    if (ol) { double a = ol[1], b = ol[4], c = ol[7]; g2 += a * a; g2 += b * b; g2 += c * c; }
    low_from_top = g1 > g2;
  }
  const int start = band_start(band), n = band_start(band + 1) - start;
  int32_t* vref = prm.ref + prm.blocks[blk].coef_off;
  for (int i = start + lane; i < start + n; i += 32) {
    int v, sh;
    if (i < 16) { v = kScan4[i - 1]; sh = 2; }
    else if (i < 64) { v = kScan8[i - 16]; sh = 3; }
    else if (i < 256) { v = kScan16[i - 64]; sh = 4; }
    else { v = kScan32[i - 256]; sh = 5; }
    const int r = v >> sh, c = v & ((1 << sh) - 1);
    int32_t p = 0;
    if (r == 0 && c > 0 && ot && (c >= 4 || low_from_top)) p = ot[i];
    if (c == 0 && r > 0 && ol && (r >= 4 || !low_from_top)) p = ol[i];
    vref[i] = p;
  }
}

// Chroma-from-luma prediction of keyframe chroma blocks (od_resample_luma_coeffs,
// src/intra.c:72, 4:2:0): the low-frequency quarter of the quantised luma block,
// or -- when the luma area is coded as four 4x4 blocks -- their 2x2 TF merge
// (od_tf_up_hv_lp, src/tf.c:82) scaled by OD_CFL_SCALING4.  One thread per
// coefficient; writes an n x n block into the chroma-sized prediction plane.
__global__ void k_cfl_pred(const __grid_constant__ daala_b200_pvq_params prm, int32_t* pred_plane,
                           long long pred_frame_pitch, int pred_stride, int nblocks) {
  const int blk = blockIdx.x;
  if (blk >= nblocks) return;
  const daala_b200_pvq_block b = prm.blocks[blk];
  if (b.pli == 0) return;
  const int n = 4 << b.bs;
  const int lstride = prm.plane_stride[0];
  const int32_t* luma = prm.coef_plane[0] + b.frame * prm.plane_frame_pitch[0] + (size_t)(2 * b.y0) * lstride + 2 * b.x0;
  int32_t* dst = pred_plane + b.frame * pred_frame_pitch + (size_t)b.y0 * pred_stride + b.x0;
  if (b.xdec & 0x80) {
    // four 4x4 luma blocks -> one 4x4 chroma prediction
    const int scaling4[4][4] = {{128, 128, 100, 36}, {128, 80, 71, 35}, {100, 71, 35, 31}, {36, 35, 31, 18}};
    if (threadIdx.x < 4) {
      const int x = threadIdx.x & 1, y = threadIdx.x >> 1;
      int ll = luma[(size_t)y * lstride + x], lh = luma[(size_t)y * lstride + x + 4];
      int hl = luma[(size_t)(y + 4) * lstride + x], hh = luma[(size_t)(y + 4) * lstride + x + 4];
      // OD_HAAR_KERNEL(ll, hl, lh, hh): the reference swaps the middle terms here
      ll += lh; hh -= hl;
      int t = (ll - hh) >> 1;
      hl = t - hl; lh = t - lh;
      ll -= hl; hh += lh;
      const int hs = x & 1, vs = y & 1;
      int r, c;
      r = 2 * y + vs; c = 2 * x + hs;         dst[(size_t)r * pred_stride + c] = (scaling4[c][r] * ll + 64) >> 7;
      r = 2 * y + vs; c = 2 * x + 1 - hs;     dst[(size_t)r * pred_stride + c] = (scaling4[c][r] * lh + 64) >> 7;
      r = 2 * y + 1 - vs; c = 2 * x + hs;     dst[(size_t)r * pred_stride + c] = (scaling4[c][r] * hl + 64) >> 7;
      r = 2 * y + 1 - vs; c = 2 * x + 1 - hs; dst[(size_t)r * pred_stride + c] = (scaling4[c][r] * hh + 64) >> 7;
    }
  } else {
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
      int r = i / n, c = i % n;
      dst[(size_t)r * pred_stride + c] = luma[(size_t)r * lstride + c];
    }
  }
}

// ---------------------------------------------------------------------------
// Scalar helpers of src/pvq.h:148-175 for the host-pointer ABI: one thread runs
// the same device functions the batch kernels use.  Marshalling buffer layout
// (ints): args[16] | a16[2][128] (as int16) | a32[2][128] | qmi[128] (int16) | dargs[2] (double)
// ---------------------------------------------------------------------------
struct HelperBuf {
  int32_t args[16];
  int16_t a16[2][kMaxN];
  int32_t a32[2][kMaxN];
  int16_t qmi[kMaxN];
  double dargs[2];
};

__global__ void k_pvq_helper(HelperBuf* b, int op) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int32_t* a = b->args;
  switch (op) {
    case 0: a[15] = (int16_t)pvq_sin(a[0]); break;
    case 1: a[15] = (int16_t)pvq_cos(a[0]); break;
    case 2: {  // od_vector_log_mag(x, n)
      int32_t sum = 0;
      for (int i = 0; i < a[0]; i++) { int16_t t = (int16_t)(b->a32[0][i] >> 8); sum += t * (int32_t)t; }
      a[15] = 9 + ilog((uint32_t)(a[0] + sum)) / 2;
      break;
    }
    case 3: { int sign; a[15] = householder_setup(b->a16[0], a[0], a[1], &sign, a[2]); a[14] = sign; break; }
    case 4: householder_apply(b->a16[1], b->a16[1], b->a16[0], a[0]); break;
    case 5: {  // od_pvq_synthesis_partial(xcoeff, ypulse, r, n, noref, g, theta, m, s, qm_inv)
      int16_t scratch[kMaxN];
      synthesis(b->a32[1], b->a32[0], b->a16[0], a[0], a[1], a[2], a[3], a[4], a[5], b->qmi, scratch);
      break;
    }
    case 6: a[15] = gain_expand(a[0], a[1], a[2]); break;
    case 7: {  // od_pvq_compute_gain(x, n, q0, &g, beta, bshift)
      int32_t acc = 0, g;
      for (int i = 0; i < a[0]; i++) acc += b->a16[0][i] * (int32_t)b->a16[0][i];
      a[15] = compute_gain_from_energy(acc, a[1], &g, a[2], a[3]);
      a[14] = g;
      break;
    }
    case 8: a[15] = compute_max_theta(a[0], a[1]); break;
    case 9: a[15] = compute_theta(a[0], a[1]); break;
    case 10: a[15] = compute_k(a[0], a[1], a[2], a[3], a[4]); break;
    case 11: {  // od_rdo_quant(x, q, delta0, pvq_norm_lambda), src/pvq_encoder.c:730
      int t = (int)(256 * b->dargs[1] * b->dargs[0] / 2);
      t = t < 0 ? 0 : (t > 128 ? 128 : t);  // OD_CLAMPI(0, t, 128)
      const int threshold = 128 + t, x = a[0], q = a[1];
      if (abs(x) < q * threshold / 256) a[15] = 0;
      else { int half = ((q + 1) >> 1) - 1; a[15] = (x + (x < 0 ? -half : half)) / q; }
      break;
    }
    default: a[15] = 0;
  }
}

}  // namespace pvq
}  // namespace daala_b200

using namespace daala_b200::pvq;

template <int G, int E, bool kForceScan, int kMinCtas = 4>
static void launch_coop(const daala_b200_pvq_params* prm, const uint32_t* band_list, int count, cudaStream_t s) {
  const int per = 128 / G, blocks = (count + per - 1) / per;
  k_pvq_bands_coop<G, E, kForceScan, kMinCtas><<<blocks, 128, 0, s>>>(*prm, band_list, count);
}


extern "C" {

int daala_b200_pvq_encode_bands(const daala_b200_pvq_params* prm, const uint32_t* band_list, int count,
                                int nmax, void* stream) {
  if (count <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int threads = 128;
  const int blocks = (count + threads - 1) / threads;
  // 64 registers (8 CTAs per SM): the search is latency-bound at 16 warps per SM, the spills stay in L1
  if (nmax <= 16) k_pvq_bands<16, 8><<<blocks, threads, 0, s>>>(*prm, band_list, count);
  else if (nmax <= 32) k_pvq_bands<32, 8><<<blocks, threads, 0, s>>>(*prm, band_list, count);
  else k_pvq_bands<128, 4><<<blocks, threads, 0, s>>>(*prm, band_list, count);
  return (int)cudaGetLastError();
}

// mode 0: best measured mix (see below), 1: group-cooperative kernels with the literal sequential arg-max scan
// forced (test hook), 2: scalar thread-per-band kernels, 3: group-cooperative kernels everywhere.  Any other mode
// is refused before anything is launched.
int daala_b200_pvq_encode_bands_mode(const daala_b200_pvq_params* prm, const uint32_t* band_list, int count,
                                     int nmax, int mode, void* stream) {
  if (mode < 0 || mode > 3) return (int)cudaErrorInvalidValue;
  if (count <= 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  if (mode == 2) return daala_b200_pvq_encode_bands(prm, band_list, count, nmax, stream);
  const int cls = nmax <= 16 ? 0 : nmax <= 32 ? 1 : 2;
  if (mode == 0) {
    // chosen by timing on real with-reference data: scalar threads for the short bands, a whole warp
    // (32 lanes x 4 registers, capped at 80 registers = 6 CTAs per SM) for the 128-coefficient bands
    if (cls < 2) return daala_b200_pvq_encode_bands(prm, band_list, count, nmax, stream);
    launch_coop<32, 4, false, 6>(prm, band_list, count, s);
    return (int)cudaGetLastError();
  }
  if (mode == 1) {
    if (cls == 0) launch_coop<4, 4, true>(prm, band_list, count, s);
    else if (cls == 1) launch_coop<8, 4, true>(prm, band_list, count, s);
    else launch_coop<32, 4, true>(prm, band_list, count, s);
  } else {
    if (cls == 0) launch_coop<4, 4, false>(prm, band_list, count, s);
    else if (cls == 1) launch_coop<8, 4, false>(prm, band_list, count, s);
    else launch_coop<32, 4, false>(prm, band_list, count, s);
  }
  return (int)cudaGetLastError();
}

int daala_b200_pvq_order_by_work(const daala_b200_pvq_params* prm, const uint32_t* band_list,
                                 const uint16_t* entry_wave, int count, int nwaves, int nmax, uint32_t* ordered,
                                 uint16_t* keys, int32_t* bins, void* stream) {
  if (count <= 0) return 0;
  if (nwaves < 1 || nwaves > kMaxOrderBins) return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  int bpw = kMaxWaveBins;
  while (bpw > 1 && nwaves * bpw > kMaxOrderBins) bpw >>= 1;
  const int nbins = nwaves * bpw;
  cudaError_t err = cudaMemsetAsync(bins, 0, sizeof(int32_t) * nbins, s);
  if (err != cudaSuccess) return (int)err;
  if (nmax <= 16) {
    k_band_work_keys<4><<<(count * 4 + 255) / 256, 256, 0, s>>>(*prm, band_list, entry_wave, count, bpw, keys, bins);
  } else if (nmax <= 32) {
    k_band_work_keys<8><<<(count * 8 + 255) / 256, 256, 0, s>>>(*prm, band_list, entry_wave, count, bpw, keys, bins);
  } else {
    k_band_work_keys<32><<<(int)(((long long)count * 32 + 255) / 256), 256, 0, s>>>(*prm, band_list, entry_wave,
                                                                                    count, bpw, keys, bins);
  }
  k_bin_scan<<<1, 1024, 0, s>>>(bins, nbins);
  k_bin_scatter<<<(count + 255) / 256, 256, 0, s>>>(band_list, keys, count, bins, ordered);
  return (int)cudaGetLastError();
}

int daala_b200_pvq_order_bins(void) { return kMaxOrderBins; }

int daala_b200_pvq_intra_band_ref(const daala_b200_pvq_params* prm, const int32_t* dep_top, const int32_t* dep_left,
                                  const uint32_t* band_list, int count, void* stream) {
  if (count <= 0) return 0;
  k_intra_band_ref<<<(count * 32 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(*prm, dep_top, dep_left, band_list,
                                                                               count);
  return (int)cudaGetLastError();
}

int daala_b200_pvq_cfl_pred(const daala_b200_pvq_params* prm, int32_t* pred_plane, long long pred_frame_pitch,
                            int pred_stride, int nblocks, void* stream) {
  if (nblocks <= 0) return 0;
  k_cfl_pred<<<nblocks, 64, 0, (cudaStream_t)stream>>>(*prm, pred_plane, pred_frame_pitch, pred_stride, nblocks);
  return (int)cudaGetLastError();
}

int daala_b200_pvq_helper_launch(void* buf, int op, void* stream) {
  k_pvq_helper<<<1, 32, 0, (cudaStream_t)stream>>>((HelperBuf*)buf, op);
  return (int)cudaGetLastError();
}
int daala_b200_pvq_helper_bytes(void) { return (int)sizeof(HelperBuf); }

int daala_b200_pvq_block_finish(const daala_b200_pvq_params* prm, int nblocks, void* stream) {
  if (nblocks <= 0) return 0;
  k_block_finish<<<(nblocks + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*prm, 0, nblocks);
  return (int)cudaGetLastError();
}

int daala_b200_pvq_cfl_flip(const daala_b200_pvq_params* prm, int nblocks, void* stream) {
  if (nblocks <= 0) return 0;
  k_cfl_flip<<<(nblocks + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*prm, nblocks);
  return (int)cudaGetLastError();
}

int daala_b200_coding_order_gather(const daala_b200_pvq_params* prm, int nblocks, int which, void* stream) {
  if (nblocks <= 0) return 0;
  k_coding_order_gather<<<(nblocks * 32 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(*prm, nblocks, which);
  return (int)cudaGetLastError();
}

int daala_b200_coding_order_scatter(const daala_b200_pvq_params* prm, int nblocks, void* stream) {
  if (nblocks <= 0) return 0;
  k_coding_order_scatter<<<(nblocks * 32 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(*prm, 0, nblocks);
  return (int)cudaGetLastError();
}

}  // extern "C"
