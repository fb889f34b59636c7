// Group-cooperative PVQ band quantiser: G lanes of a warp own one band, each
// lane keeps E coefficients (element j lives in lane j % G, slot j / G) in
// REGISTERS -- no per-thread scratch arrays, no local memory.  n = 128 bands
// use a whole warp (G = 32, E = 4), n = 32 bands a quarter warp (G = 8), the
// 15/8-coefficient bands four lanes.  Same algorithm and bit-exact results as
// the scalar quantise_band<> of pvq_kernels.cu (reference pvq_theta,
// src/pvq_encoder.c:333):
//  * every sum the reference accumulates in double is a sum of exactly
//    representable integers far below 2^53, hence order independent; they are
//    reduced as integers with shuffles;
//  * the greedy pulse search takes an arg-max per pulse.  The reference scans
//    j = 0..n-1 and keeps the first maximum (strict ">").  For the RDO pulses
//    that is a maximum over independent doubles, so a tree reduction with
//    lowest-index tie-break is identical.  For the plain pulses the comparison
//    is the cross-multiplied ratio test tmp_xy*best_yy > best_xy*tmp_yy; it is
//    exact (and therefore a consistent order) whenever the products stay
//    below 2^53, which is checked per pulse; otherwise the group falls back to
//    the literal sequential scan.
#pragma once
#include <math.h>
#include <stdint.h>

#include "pvq_math.cuh"

namespace daala_b200 {
namespace pvq {

// shuffles move 32/64-bit values; 16-bit lanes travel as int
template <class T> struct ShuffleAs { using type = T; };
template <> struct ShuffleAs<int16_t> { using type = int; };

template <int G, int E>
struct Group {
  unsigned mask;
  int lane;  // lane inside the group
  __device__ __forceinline__ Group() {
    const int l = threadIdx.x & 31;
    lane = l & (G - 1);
    mask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (l & ~(G - 1)));
  }
  __device__ __forceinline__ int idx(int e) const { return e * G + lane; }
  template <class T>
  __device__ __forceinline__ T sum(T v) const {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o, G);
    return v;
  }
  __device__ __forceinline__ int any(int v) const {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v |= __shfl_xor_sync(mask, v, o, G);
    return v;
  }
  template <class T>
  __device__ __forceinline__ T from(T v, int src_lane) const { return __shfl_sync(mask, v, src_lane, G); }
  // value of element j of a distributed array
  template <class T>
  __device__ __forceinline__ T elem(const T (&a)[E], int j) const {
    using S = typename ShuffleAs<T>::type;
    const int e = j / G;
    S v = a[0];
#pragma unroll
    for (int q = 1; q < E; q++) if (q == e) v = a[q];
    return (T)from(v, j & (G - 1));
  }
  // b[e] = value of element idx(e) + 1 (0 past the end)
  template <class T>
  __device__ __forceinline__ void shift_down(T (&b)[E], const T (&a)[E]) const {
#pragma unroll
    for (int e = 0; e < E; e++) {
      using S = typename ShuffleAs<T>::type;
      S t1 = __shfl_sync(mask, (S)a[e], (lane + 1) & (G - 1), G);
      S t2 = e + 1 < E ? __shfl_sync(mask, (S)a[e + 1 < E ? e + 1 : e], 0, G) : (S)0;
      b[e] = (T)(lane == G - 1 ? t2 : t1);
    }
  }
  // b[e] = value of element idx(e) - 1 (0 before the start)
  template <class T>
  __device__ __forceinline__ void shift_up(T (&b)[E], const T (&a)[E]) const {
#pragma unroll
    for (int e = 0; e < E; e++) {
      using S = typename ShuffleAs<T>::type;
      S t1 = __shfl_sync(mask, (S)a[e], (lane + G - 1) & (G - 1), G);
      S t2 = e > 0 ? __shfl_sync(mask, (S)a[e > 0 ? e - 1 : 0], G - 1, G) : (S)0;
      b[e] = (T)(lane == 0 ? t2 : t1);
    }
  }
};

__device__ __forceinline__ double rsqrt_small_c(int i) { return rsqrt_small_tbl(i); }

// pvq_search_rdo_double (src/pvq_encoder.c:93) on a distributed vector.
template <int G, int E, bool kForceScan>
__device__ double search_rdo_coop(const Group<G, E>& grp, const int16_t (&xc)[E], int n, int k, int (&y)[E],
                                  double g2, double pvq_norm_lambda, int prev_k) {
  double x[E];
  long long sxx = 0;
  int xmax = 0;
#pragma unroll
  for (int e = 0; e < E; e++) {
    const bool valid = grp.idx(e) < n;
    int a = valid ? abs((int)xc[e]) : 0;
    x[e] = (double)a;  // == fabs((float)xcoeff[j]): |int16| is exact in float
    sxx += (long long)a * a;
    xmax = a > xmax ? a : xmax;
  }
  const double xx = (double)grp.sum(sxx);
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) {
    int t = __shfl_xor_sync(grp.mask, xmax, o, G);
    xmax = t > xmax ? t : xmax;
  }
  const double norm_1 = 1. / sqrt(1e-30 + xx);
  const double lambda = pvq_norm_lambda / (1e-30 + g2);
  double xy = 0, yy = 0;
  int i = 0;
  if (prev_k > 0 && prev_k <= k) {
    long long sxy = 0;
    int syy = 0, si = 0;
#pragma unroll
    for (int e = 0; e < E; e++) {
      y[e] = grp.idx(e) < n ? abs(y[e]) : 0;
      sxy += (long long)x[e] * y[e];
      syy += y[e] * y[e];
      si += y[e];
    }
    xy = (double)grp.sum(sxy);
    yy = (double)grp.sum(syy);
    i = grp.sum(si);
  } else if (k > 2) {
    long long sl1 = 0;
#pragma unroll
    for (int e = 0; e < E; e++) sl1 += (long long)x[e];
    const double l1_norm = (double)grp.sum(sl1);
    const double l1_inv = 1. / (l1_norm > 1e-100 ? l1_norm : 1e-100);
    long long sxy = 0;
    int syy = 0, si = 0;
#pragma unroll
    for (int e = 0; e < E; e++) {
      double tmp = k * x[e] * l1_inv;
      int f = (int)floor(tmp);
      y[e] = (grp.idx(e) < n && f > 0) ? f : 0;
      sxy += (long long)x[e] * y[e];
      syy += y[e] * y[e];
      si += y[e];
    }
    xy = (double)grp.sum(sxy);
    yy = (double)grp.sum(syy);
    i = grp.sum(si);
  } else {
#pragma unroll
    for (int e = 0; e < E; e++) y[e] = 0;
  }
  const int rdo_pulses = 1 + k / 4;
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
  // --- plain pulses: maximise (xy + x_j)^2 / (yy + 2 y_j + 1) -----------------
  for (; i < k - rdo_pulses; i++) {
    int pos;
    // all products exact below 2^53 <=> the ratio test is a consistent order
    const double bound = (xy + xmax) * (xy + xmax) * (yy + 2. * i + 1.);
    if (!kForceScan && bound < 4503599627370496.) {
      double ba = -1., bb = 1.;
      int bj = 0x7fffffff;
#pragma unroll
      for (int e = 0; e < E; e++) {
        if (grp.idx(e) < n) {
          double a = xy + x[e];
          double b = yy + 2 * y[e] + 1;
          a *= a;
          if (bj == 0x7fffffff || a * bb > ba * b) { ba = a; bb = b; bj = grp.idx(e); }
        }
      }
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) {
        double oa = __shfl_xor_sync(grp.mask, ba, o, G);
        double ob = __shfl_xor_sync(grp.mask, bb, o, G);
        int oj = __shfl_xor_sync(grp.mask, bj, o, G);
        double l = oa * bb, r = ba * ob;
        if (l > r || (l == r && oj < bj)) { ba = oa; bb = ob; bj = oj; }
      }
      pos = bj;
    } else {
      // literal sequential scan (src/pvq_encoder.c:163-174), candidates broadcast in order
      double ba = -10, bb = 1;
      pos = 0;
      for (int j = 0; j < n; j++) {
        double xj = grp.elem(x, j);
        int yj = grp.elem(y, j);
        double a = xy + xj;
        double b = yy + 2 * yj + 1;
        a *= a;
        if (j == 0 || a * bb > ba * b) { ba = a; bb = b; pos = j; }
      }
    }
    const double xp = grp.elem(x, pos);
    const int yp = grp.elem(y, pos);
    xy = xy + xp;
    yy = yy + 2 * yp + 1;
#pragma unroll
    for (int e = 0; e < E; e++) if (grp.idx(e) == pos) y[e]++;
  }
  // --- RDO pulses ---------------------------------------------------------------
  for (; i < k; i++) {
    double tbl[4];
#pragma unroll
    for (int j = 0; j < 4; j++) tbl[j] = rsqrt_small_c((int)(yy + 2 * j + 1));
    double bv = 0;
    int bj = 0x7fffffff;
#pragma unroll
    for (int e = 0; e < E; e++) {
      const int j = grp.idx(e);
      if (j < n) {
        double t = xy + x[e];
        const int yj = y[e];
        double ryy = yj < 4 ? (yj == 0 ? tbl[0] : yj == 1 ? tbl[1] : yj == 2 ? tbl[2] : tbl[3])
                            : rsqrt_small_c((int)(yy + 2 * yj + 1));
        t = 2 * t * norm_1 * ryy - lambda * j * (delta_rate + j * accel_rate);
        if (bj == 0x7fffffff || t > bv) { bv = t; bj = j; }
      }
    }
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) {
      double ov = __shfl_xor_sync(grp.mask, bv, o, G);
      int oj = __shfl_xor_sync(grp.mask, bj, o, G);
      if (oj != 0x7fffffff && (bj == 0x7fffffff || ov > bv || (ov == bv && oj < bj))) { bv = ov; bj = oj; }
    }
    const int pos = bj;
    const double xp = grp.elem(x, pos);
    const int yp = grp.elem(y, pos);
    xy = xy + xp;
    yy = yy + 2 * yp + 1;
#pragma unroll
    for (int e = 0; e < E; e++) if (grp.idx(e) == pos) y[e]++;
  }
#pragma unroll
  for (int e = 0; e < E; e++) if (xc[e] < 0) y[e] = -y[e];
  return xy / (1e-100 + sqrt(xx * yy));
}

// od_pvq_rate, closed-form branch (src/pvq_encoder.c:247).
template <int G, int E>
__device__ double band_rate_coop(const Group<G, E>& grp, int qg, int icgr, int theta, int ts, const int (&y0)[E],
                                 int k, int n, int is_keyframe, int pli) {
  double rate;
  if (k == 0) {
    rate = 0;
  } else {
    int s = 0;
    const int lim = n - (theta != -1);
#pragma unroll
    for (int e = 0; e < E; e++) if (grp.idx(e) < lim) s += grp.idx(e) * abs(y0[e]);
    const int sum = grp.sum(s);
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

// od_apply_householder (src/pvq.c:560) on distributed int16 vectors; in place allowed.
template <int G, int E>
__device__ void householder_apply_coop(const Group<G, E>& grp, int16_t (&out)[E], const int16_t (&x)[E],
                                       const int16_t (&r)[E], int n) {
  int32_t l2r = 0, proj = 0;
#pragma unroll
  for (int e = 0; e < E; e++) {
    if (grp.idx(e) < n) {
      l2r += mul16(r[e], r[e]);
      proj += mul16(r[e], x[e]);
    }
  }
  l2r = grp.sum(l2r);
  proj = grp.sum(proj);
  int l2r_shift = (ilog((uint32_t)l2r) - 1) - 14;
  int16_t l2r_norm = (int16_t)vshr_round(l2r, l2r_shift);
  int16_t rcp = rcp16(l2r_norm);
  int proj_shift = (ilog((uint32_t)abs(proj)) - 1) - 14;
  int16_t proj_norm = (int16_t)vshr_round(proj, proj_shift);
  int16_t proj_1 = (int16_t)mul16_q15(proj_norm, rcp);
  int outshift = 14 - proj_shift - 1 + l2r_shift;
  if (outshift > 30) outshift = 30;
#pragma unroll
  for (int e = 0; e < E; e++) {
    int32_t t = mul16(r[e], proj_1);
    t = outshift >= 0 ? shr_round(t, outshift) : shl(t, -outshift);
    out[e] = (int16_t)(x[e] - t);
  }
}

struct CandC {
  int gain, k, theta, ts;
  int32_t qtheta, qcg;
  int noref;
};

// One band by G lanes.  x0/r0/out/y/qm/qm_inv point at the band's first entry.
// Scalar results are identical in every lane of the group.
template <int G, int E, bool kForceScan>
__device__ int quantise_band_coop(const Group<G, E>& grp, int32_t* out, const int32_t* x0, const int32_t* r0,
                                  int n, int q0, int32_t* yout, int* itheta, int* max_theta, int* vk, int beta,
                                  double* skip_term, int is_keyframe, int pli, const int16_t* qm,
                                  const int16_t* qm_inv, double pvq_norm_lambda) {
  const double gain_weight = 1.4;
  const double cgain_1 = 1. / kCgainOne;
  const double cgain_2 = cgain_1 * cgain_1;
  const double theta_scale = (1 << kThetaShift) * 2. / M_PI;
  const double theta_scale_1 = 1. / theta_scale;
  const double trig_1 = 1. / 32768;
  int32_t xv[E], rv[E];
  int16_t qmv[E];
  int16_t x16[E], r16[E], xr[E];
  int y[E], y_tmp[E];
  int32_t sx = 0, sr = 0;
  int r_nonnull = 0;
#pragma unroll
  for (int e = 0; e < E; e++) {
    const int j = grp.idx(e);
    const bool valid = j < n;
    xv[e] = valid ? x0[j] : 0;
    rv[e] = valid ? r0[j] : 0;
    qmv[e] = valid ? qm[j] : (int16_t)0;
    int16_t tx = (int16_t)(xv[e] >> 8), tr = (int16_t)(rv[e] >> 8);
    sx += tx * (int32_t)tx;
    sr += tr * (int32_t)tr;
    r_nonnull |= rv[e] != 0;
    y[e] = 0;
    y_tmp[e] = 0;
  }
  sx = grp.sum(sx);
  sr = grp.sum(sr);
  r_nonnull = grp.any(r_nonnull);
  int xshift = 9 + ilog((uint32_t)(n + sx)) / 2 - 15;
  int rshift = 9 + ilog((uint32_t)(n + sr)) / 2 - 14;
  if (xshift < 0) xshift = 0;
  if (rshift < 0) rshift = 0;
  long long scorr = 0;
  int32_t accx = 0, accr = 0;
#pragma unroll
  for (int e = 0; e < E; e++) {
    x16[e] = (int16_t)shr_round(xv[e] * qmv[e], kQmShift + xshift);
    r16[e] = (int16_t)shr_round(rv[e] * qmv[e], kQmShift + rshift);
    scorr += mul16(x16[e], r16[e]);
    accx += x16[e] * (int32_t)x16[e];
    accr += r16[e] * (int32_t)r16[e];
  }
  double corr = (double)grp.sum(scorr);
  accx = grp.sum(accx);
  accr = grp.sum(accr);
  int32_t g, gr;
  const int cfl_enabled = is_keyframe && pli != 0;
  int32_t cg = compute_gain_from_energy(accx, q0, &g, beta, xshift);
  int32_t cgr = compute_gain_from_energy(accr, q0, &gr, beta, rshift);
  if (cfl_enabled) cgr = kCgainOne;
  int icgr = shr_round(cgr, kCgainShift);
  int32_t gain_offset = cgr - shl(icgr, kCgainShift);
  int32_t theta = 0, best_qtheta = 0;
  int qg = 0, best_k = 0, noref = 1, m = 0, s = 1, skip = 0;
  double dist = gain_weight * cg * cg * cgain_2;
  double best_dist = dist;
  double best_cost = dist + pvq_norm_lambda * 0.;  // od_pvq_rate(0, 0, -1, 0, ...) == 0
  *itheta = -1;
  *max_theta = 0;
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
    best_cost = best_dist + pvq_norm_lambda * 0.;  // od_pvq_rate(0, icgr, 0, 0, ...) == 0
    best_qtheta = 0;
    *itheta = 0;
    *max_theta = 0;
    noref = 0;
  }
  const double dist0 = best_dist;
  // One candidate list and ONE search / rate call site for both passes of pvq_theta (with-reference
  // candidates in (k, gain) order, src/pvq_encoder.c:504-560, then the no-reference gains, :573-606):
  // the search is most of this kernel's code, and its instruction footprint is what the warps stall on,
  // so it is instantiated once.
  CandC items[22];
  int nitems = 0;
  if (r_nonnull && corr > 0) {
    int gain_bound = (cg - gain_offset) >> kCgainShift;
    theta = round32(theta_scale * acos(corr));
    // od_compute_householder, src/pvq.c:498: first largest |r|
    {
      int bv = -1, bj = 0;
#pragma unroll
      for (int e = 0; e < E; e++) {
        int a = grp.idx(e) < n ? abs((int)r16[e]) : -1;
        if (a > bv) { bv = a; bj = grp.idx(e); }
      }
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) {
        int ov = __shfl_xor_sync(grp.mask, bv, o, G);
        int oj = __shfl_xor_sync(grp.mask, bj, o, G);
        if (ov > bv || (ov == bv && oj < bj)) { bv = ov; bj = oj; }
      }
      // the reference's scan starts from maxr = 0 with strict ">": an all-zero vector keeps m = 0
      m = bv > 0 ? bj : 0;
      const int rm = grp.elem(r16, m);
      s = rm > 0 ? 1 : -1;
#pragma unroll
      for (int e = 0; e < E; e++)
        if (grp.idx(e) == m) r16[e] = (int16_t)(r16[e] + shr_round(gr * s, rshift));
    }
    householder_apply_coop(grp, xr, x16, r16, n);
    {
      int16_t nxt[E];
      grp.shift_down(nxt, xr);
#pragma unroll
      for (int e = 0; e < E; e++) if (grp.idx(e) >= m) xr[e] = nxt[e];
    }
    for (int i = gain_bound - 1 > 1 ? gain_bound - 1 : 1; i <= gain_bound + 1; i++) {
      int32_t qcg = shl(i, kCgainShift) + gain_offset;
      int ts = compute_max_theta(qcg, beta);
      int lo = (int)floor(.5 + theta * theta_scale_1 * 2 / M_PI * ts) - 2;
      int hi = (int)ceil(theta * theta_scale_1 * 2 / M_PI * ts);
      if (lo < 0) lo = 0;
      if (hi > ts - 1) hi = ts - 1;
      for (int j = lo; j <= hi; j++) {
        CandC c;
        c.gain = i;
        c.theta = j;
        c.qtheta = compute_theta(j, ts);
        c.k = compute_k(qcg, j, 0, n, beta);
        c.qcg = qcg;
        c.ts = ts;
        c.noref = 0;
        int p = nitems++;
        while (p > 0 && (items[p - 1].k > c.k || (items[p - 1].k == c.k && items[p - 1].gain > c.gain))) {
          items[p] = items[p - 1];
          p--;
        }
        items[p] = c;
      }
    }
  }
  const int first_noref = nitems;
  if ((is_keyframe && pli == 0) || corr < .5 || cg < (int32_t)shl(2, kCgainShift)) {
    int gain_bound = cg >> kCgainShift;
    for (int i = gain_bound > 1 ? gain_bound : 1; i <= gain_bound + 1; i++) {
      CandC c;
      c.gain = i;
      c.theta = -1;
      c.qtheta = 0;
      c.qcg = shl(i, kCgainShift);
      c.k = compute_k(c.qcg, -1, 1, n, beta);
      c.ts = 0;
      c.noref = 1;
      items[nitems++] = c;
    }
  }
  {
    int prev_k = 0;
    double cos_dist = 0;
    const double sin_theta = pvq_sin(theta) * trig_1;
    for (int idx = 0; idx < nitems; idx++) {
      const CandC c = items[idx];
      const int32_t qcg = c.qcg, qtheta = c.qtheta;
      const int k = c.k;
      if (idx == first_noref) prev_k = 0;
      double sin_prod = 0;
      if (c.noref) {
        dist = gain_weight * (qcg - cg) * (qcg - cg);
        dist *= cgain_2;
        if (dist > dist0 && k != 0) continue;
      } else {
        double dist_theta = 2 - 2. * pvq_cos(theta - qtheta) * trig_1;
        dist = gain_weight * (qcg - cg) * (qcg - cg) + qcg * (double)cg * dist_theta;
        dist *= cgain_2;
        if (dist > dist0 + 1.0 * pvq_norm_lambda && k != 0) continue;
        sin_prod = sin_theta * pvq_sin(qtheta) * trig_1;
      }
      if (!c.noref && k == 0) {
        cos_dist = 0;
#pragma unroll
        for (int e = 0; e < E; e++) y_tmp[e] = 0;
      } else if (c.noref || k != prev_k) {
        int16_t xin[E];
#pragma unroll
        for (int e = 0; e < E; e++) xin[e] = c.noref ? x16[e] : xr[e];
        const double g2 = c.noref ? qcg * (double)cg * cgain_2 : qcg * (double)cg * sin_prod * cgain_2;
        cos_dist = search_rdo_coop<G, E, kForceScan>(grp, xin, c.noref ? n : n - 1, k, y_tmp, g2, pvq_norm_lambda,
                                                     prev_k);
      }
      prev_k = k;
      if (c.noref) {
        dist = gain_weight * (qcg - cg) * (qcg - cg) + qcg * (double)cg * (2 - 2 * cos_dist);
      } else {
        double dist_theta = 2 - 2. * pvq_cos(theta - qtheta) * trig_1 + sin_prod * (2 - 2 * cos_dist);
        dist = gain_weight * (qcg - cg) * (qcg - cg) + qcg * (double)cg * dist_theta;
      }
      dist *= cgain_2;
      const double cost = dist + pvq_norm_lambda * band_rate_coop(grp, c.gain, c.noref ? 0 : icgr, c.theta, c.ts,
                                                                  y_tmp, k, n, is_keyframe, pli);
      if (c.noref ? cost <= best_cost : cost < best_cost) {
        best_cost = cost;
        best_dist = dist;
        qg = c.gain;
        best_k = k;
        noref = c.noref;
        best_qtheta = c.noref ? best_qtheta : qtheta;
        *itheta = c.theta;
        *max_theta = c.ts;
#pragma unroll
        for (int e = 0; e < E; e++) y[e] = (c.noref || grp.idx(e) < n - 1) ? y_tmp[e] : 0;
      }
    }
  }
  theta = best_qtheta;
  if (noref) {
    if (qg == 0) skip = 1;
  } else {
    if (!is_keyframe && qg == 0) skip = icgr ? 1 : 2;
    if (qg == icgr && *itheta == 0 && !cfl_enabled) skip = 2;
  }
  int32_t res[E];
  if (skip) {
#pragma unroll
    for (int e = 0; e < E; e++) res[e] = skip == 2 ? rv[e] : 0;
  } else {
    if (noref) gain_offset = 0;
    g = gain_expand(shl(qg, kCgainShift) + gain_offset, q0, beta);
    // od_pvq_synthesis_partial, src/pvq.c:1037
    const int nn = n - !noref;
    int syy = 0;
#pragma unroll
    for (int e = 0; e < E; e++) if (grp.idx(e) < nn) syy += y[e] * y[e];
    const int yy = grp.sum(syy);
    int gshift = ilog((uint32_t)g) - 14;
    if (gshift < 0) gshift = 0;
    int32_t scale;
    if (yy == 0) {
      scale = 0;
    } else {
      int rsh;
      int16_t rs = rsqrt32(yy, &rsh);
      scale = vshr_round64(rs * (int64_t)g, rsh + gshift - 16);
    }
    const int qshift = kQmInvShift - gshift;
    if (noref) {
#pragma unroll
      for (int e = 0; e < E; e++) {
        int32_t v = mul16_32_q16(y[e], scale);
        res[e] = grp.idx(e) < n ? shr_round(v * qm_inv[grp.idx(e)], qshift) : 0;
      }
    } else {
      scale = round32(scale * (1. / 32768) * pvq_sin(theta));
      int16_t xs[E], f[E], fprev[E];
#pragma unroll
      for (int e = 0; e < E; e++) f[e] = grp.idx(e) < nn ? (int16_t)mul16_32_q16(y[e], scale) : (int16_t)0;
      grp.shift_up(fprev, f);
      const int16_t xm = (int16_t)floor(.5 + -s * (shr_round(g, gshift)) * (1. / 32768) * pvq_cos(theta));
#pragma unroll
      for (int e = 0; e < E; e++) {
        const int j = grp.idx(e);
        xs[e] = j < m ? f[e] : (j == m ? xm : fprev[e]);
        if (j >= n) xs[e] = 0;
      }
      householder_apply_coop(grp, xs, xs, r16, n);
#pragma unroll
      for (int e = 0; e < E; e++)
        res[e] = grp.idx(e) < n ? shr_round(xs[e] * qm_inv[grp.idx(e)], qshift) : 0;
    }
  }
#pragma unroll
  for (int e = 0; e < E; e++) {
    const int j = grp.idx(e);
    if (j < n) {
      out[j] = res[e];
      yout[j] = y[e];
    }
  }
  *vk = best_k;
  *skip_term = skip_dist - best_dist;
  if (is_keyframe) return noref ? qg : (qg < icgr ? -2 * (qg - icgr) - 1 : (qg < 2 * icgr ? 2 * (qg - icgr) : qg - 1));
  {
    const int a = qg + 1, b = icgr + 1;
    return noref ? qg - 1 : (a < b ? -2 * (a - b) - 1 : (a < 2 * b ? 2 * (a - b) : a - 1));
  }
}

}  // namespace pvq
}  // namespace daala_b200
