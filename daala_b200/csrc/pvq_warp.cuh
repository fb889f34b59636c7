// Warp-per-band PVQ band quantiser (reference pvq_theta, src/pvq_encoder.c:333, with the closed-form
// rate of od_pvq_rate, :247, and pvq_search_rdo_double, :93).
//
// ONE warp owns ONE band.  Design goals: (1) the latency of a single band is what the keyframe luma
// intra wavefront is bound by (od_hv_intra_pred couples a band to the same band of the top / left
// neighbour, src/intra.c:37), so everything the reference does serially per band but is independent per
// CANDIDATE runs one candidate per lane; (2) the greedy pulse search costs one redux.sync per pulse
// instead of a five-level shuffle tree; (3) a small instruction footprint: the kernel is bound by
// instruction fetch as soon as its straight-line code outgrows the 32 KB L1.5 instruction cache,
// so the long double-precision sequences (log, acos, sqrt, divide) and the
// fixed-point helpers exist once, out of line, and only the search loop is specialised by band size.
//
//  * Element j of the band lives in lane j % 32, slot j / 32, in registers (1 slot for n <= 32, 4 for
//    n = 128).
//  * Every sum the reference accumulates in double is a sum of exactly representable integers far below
//    2^53, hence order independent: reduced as integers with redux.sync (__reduce_add_sync).
//  * Candidates (gain i, theta j) of pvq_theta: lane c < 12 holds with-reference candidate
//    (gain index c / 4, theta index c % 4) in the reference's insertion order, lanes 12 / 13 the
//    no-reference gains.  Quantised angle, K, distortion pre-test, lambda, rate constants: computed once,
//    in parallel.  The reference's stable sort by K and its `prev_k` reuse of search results are
//    reproduced by processing "events" = runs of surviving candidates with equal K in ascending K order:
//    one (incremental) search per event.  The pulses of every event are parked in shared memory
//    (16 bit), its scalars (xy, yy, sum j|y_j|) in lane `event`; after the last search the square roots,
//    divisions and logarithms of ALL events run in parallel (one event per lane), then the costs (one
//    candidate per lane), then the reference's sequential `<` / `<=` fold, and the winner's pulses are
//    read back.
//  * Per-pulse arg-max.  Plain pulses maximise (xy + x_j)^2 / (yy + 2 y_j + 1): every lane builds an
//    f32 approximation of the ratio (relative error < 2^-20), redux.max picks the approximate maximum
//    and the elements within 64 ulps of it are the contenders.  The exact maximum is always a
//    contender; if there is exactly one it is the reference's choice.  Otherwise (ties, near ties, or
//    products that could exceed 2^53, where the reference's own comparisons round) the contenders are
//    compared with the reference's literal double-precision test in index order.  RDO pulses maximise
//    a double; its f32 rounding is monotone, so the contenders are the elements whose rounded value
//    equals the maximum.  Their 1/sqrt(yy + 2 y_j + 1) factors come from a table of the reference's
//    expression (built once on the device with the same code; a square root + division per element and
//    pulse was a tenth of all instructions).
//
// Pulses must fit 16 bits (K <= 32767), like the symbol stream the engine hands to the host coder.
//
// The function compiles for the host under DAALA_B200_EMU (tests/emu/simt_emu.h supplies the warp
// primitives on 32 fibres) so that CPU tests can pin it against the reference build.
#pragma once
#include <math.h>
#include <stdint.h>

#include "pvq_math.cuh"

namespace daala_b200 {
namespace pvq {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kMaxEvents = 14;                      // <= 12 with-reference K values + 2 no-reference gains
constexpr int kRsqrtEntries = 1 << 16;              // table of the reference's 1/sqrt(i), i < 65536
constexpr int kLogEntries = 1 << 12;                // table of .9 * (M_LOG2E * log(ts)) behind it
constexpr int kTableDoubles = kRsqrtEntries + kLogEntries;

// below this bound every product of the plain-pulse ratio test is exact in double (tests lower it to
// force the literal-scan path)
#ifndef DAALA_B200_PVQ_EXACT_BOUND
#define DAALA_B200_PVQ_EXACT_BOUND 4503599627370496.
#endif
// coverage counters of the host emulation build (tests/emu); nothing on the device
#ifdef DAALA_B200_EMU_STATS
#define PVQ_WARP_STAT(i) (daala_b200_pvq_warp_stats[i]++)
#else
#define PVQ_WARP_STAT(i) ((void)0)
#endif

__device__ __forceinline__ int wsum(int v) { return __reduce_add_sync(kFull, v); }
__device__ __forceinline__ int wmax(int v) { return __reduce_max_sync(kFull, v); }
__device__ __forceinline__ int wmin(int v) { return __reduce_min_sync(kFull, v); }
__device__ __forceinline__ unsigned wmaxu(unsigned v) { return __reduce_max_sync(kFull, v); }
// exact 64-bit sum of per-lane values |s| < 2^55
__device__ __forceinline__ long long wsum64(long long s) {
  const int lo = (int)(s & 0xffffff);
  const int hi = (int)(s >> 24);
  return ((long long)wsum(hi) << 24) + wsum(lo);
}
// v of lane `src` (per-lane source allowed)
__device__ __forceinline__ double wfetch(double v, int src) {
  int lo = __double2loint(v), hi = __double2hiint(v);
  lo = __shfl_sync(kFull, lo, src);
  hi = __shfl_sync(kFull, hi, src);
  return __hiloint2double(hi, lo);
}
// monotone map of a float onto signed integers
__device__ __forceinline__ int ordered_key(float f) {
  const int b = __float_as_int(f);
  return b ^ ((b >> 31) & 0x7fffffff);
}
// a[slot] of a register array without dynamic indexing
__device__ __forceinline__ int pick4(const int (&a)[4], int slot) {
  int v = a[0];
#pragma unroll
  for (int e = 1; e < 4; e++) if (slot == e) v = a[e];
  return v;
}

// ---- out-of-line helpers: one copy of each long instruction sequence ------------------------------------
static __device__ __noinline__ double nl_log(double x) { return log(x); }
static __device__ __noinline__ double nl_acos(double x) { return acos(x); }
static __device__ __noinline__ double nl_sqrt(double x) { return sqrt(x); }
static __device__ __noinline__ double nl_div(double a, double b) { return a / b; }
static __device__ __noinline__ int nl_cos(int32_t x) { return pvq_cos(x); }
// 1/sqrt(i) as pvq_search_rdo_double's od_rsqrt_table / 1./sqrt(i) (src/pvq_encoder.c:53,190)
static __device__ __noinline__ double nl_rsqrt_small(int i) {
  if (i <= 16) return kRsqrtSmall[i - 1];
  return 1. / sqrt((double)i);
}
// entry i of the tables (kTableDoubles of them): what pvq_search_rdo_double / od_pvq_rate compute for that argument
__device__ __forceinline__ void pvq_fill_rsqrt_table(double* rsq, int i) {
  if (i < kRsqrtEntries) rsq[i] = i > 0 ? nl_rsqrt_small(i) : 0.;
  else rsq[i] = .9 * (M_LOG2E * nl_log((double)(i > kRsqrtEntries ? i - kRsqrtEntries : 1)));   // od_pvq_rate's theta term
}
// (companded gain, gain) of a 16-bit vector with energy `acc`: od_pvq_compute_gain, src/pvq.c:824
static __device__ __noinline__ long long nl_gain(int32_t acc, int q0, int beta, int bshift) {
  int32_t g;
  const int32_t cg = compute_gain_from_energy(acc, q0, &g, beta, bshift);
  return ((long long)cg << 32) | (uint32_t)g;
}
// quantised angle and K of one candidate (od_pvq_compute_theta :874, od_pvq_compute_k :902)
static __device__ __noinline__ long long nl_theta_k(int32_t qcg, int j, int ts, int noref, int n, int beta) {
  const int32_t qtheta = noref ? 0 : compute_theta(j, ts);
  const int k = compute_k(qcg, j, noref, n, beta);
  return ((long long)qtheta << 32) | (uint32_t)k;
}

// od_apply_householder (src/pvq.c:560) on distributed int16 vectors; in place allowed.
__device__ __forceinline__ void householder_apply_warp(int lane, bool big, int (&out)[4], const int (&x)[4],
                                                       const int (&r)[4], int n) {
  int32_t l2r = 0, proj = 0;
#pragma unroll
  for (int e = 0; e < 4; e++) {
    if (e && !big) break;
    if (e * 32 + lane < n) {
      l2r += mul16(r[e], r[e]);
      proj += mul16(r[e], x[e]);
    }
  }
  l2r = wsum(l2r);
  proj = wsum(proj);
  int l2r_shift = (ilog((uint32_t)l2r) - 1) - 14;
  int16_t l2r_norm = (int16_t)vshr_round(l2r, l2r_shift);
  int16_t rcp = rcp16(l2r_norm);
  int proj_shift = (ilog((uint32_t)abs(proj)) - 1) - 14;
  int16_t proj_norm = (int16_t)vshr_round(proj, proj_shift);
  int16_t proj_1 = (int16_t)mul16_q15(proj_norm, rcp);
  int outshift = 14 - proj_shift - 1 + l2r_shift;
  if (outshift > 30) outshift = 30;
#pragma unroll
  for (int e = 0; e < 4; e++) {
    if (e && !big) break;
    int32_t t = mul16(r[e], proj_1);
    t = outshift >= 0 ? shr_round(t, outshift) : shl(t, -outshift);
    out[e] = (int16_t)(x[e] - t);
  }
}

// What one search phase (with-reference: the reflected vector without element m; no-reference: the
// vector itself) keeps for all its events.
// |x| <= 32768 converts exactly to float and double, so the reference's fabs((double)(float)xcoeff[j]) is
// (double)xa[j], converted where it is used rather than kept in registers.
struct SearchVec {
  int xa[4];      // |x|, 0 past the end
  double xx, norm_1, l1_norm;
  double delta_rate;   // 3. / nn
  int xmax, nn;
};

template <int E>
__device__ __forceinline__ void search_init(int lane, SearchVec& v, const int (&src)[4], int nn) {
  long long sxx = 0;
  int xmax = 0, sl1 = 0;
#pragma unroll
  for (int e = 0; e < E; e++) {
    const int a = e * 32 + lane < nn ? abs(src[e]) : 0;
    v.xa[e] = a;
    sxx += (long long)a * a;
    sl1 += a;
    xmax = a > xmax ? a : xmax;
  }
  v.xx = (double)wsum64(sxx);
  v.xmax = wmax(xmax);
  v.l1_norm = (double)wsum(sl1);
  v.norm_1 = nl_div(1., nl_sqrt(1e-30 + v.xx));
  v.delta_rate = nl_div(3., (double)nn);
  v.nn = nn;
}

// The start of pvq_search_rdo_double (src/pvq_encoder.c:93) on magnitudes: the pulses reused from the
// previous search (prev_k of them) or the projection onto the pyramid; *xy, *yy = the running sums, returns
// the number of pulses placed.  One copy for both size classes (`big`: 4 slots), outside the per-pulse loop.
__device__ __forceinline__ int search_start(int lane, const SearchVec& v, int (&ya)[4], int k, int prev_k, bool big,
                                            double* xy, double* yy) {
  const int nn = v.nn;
  long long sxy = 0, syy = 0;
  int si = 0;
  if (prev_k > 0 && prev_k <= k) {
#pragma unroll
    for (int e = 0; e < 4; e++) {
      if (e && !big) break;
      if (e * 32 + lane >= nn) ya[e] = 0;
      sxy += (long long)v.xa[e] * ya[e];
      syy += (long long)ya[e] * ya[e];
      si += ya[e];
    }
  } else if (k > 2) {
    const double l1_inv = nl_div(1., v.l1_norm > 1e-100 ? v.l1_norm : 1e-100);
#pragma unroll
    for (int e = 0; e < 4; e++) {
      if (e && !big) break;
      const double tmp = k * (double)v.xa[e] * l1_inv;
      const int f = (int)floor(tmp);
      ya[e] = (e * 32 + lane < nn && f > 0) ? f : 0;
      sxy += (long long)v.xa[e] * ya[e];
      syy += (long long)ya[e] * ya[e];
      si += ya[e];
    }
  } else {
#pragma unroll
    for (int e = 0; e < 4; e++) ya[e] = 0;
    *xy = 0;
    *yy = 0;
    return 0;
  }
  *xy = (double)wsum64(sxy);
  *yy = (double)wsum64(syy);
  return wsum(si);
}

// The per-pulse loop of pvq_search_rdo_double, specialised by the slots per lane: from i pulses (ya, xy, yy
// as search_start left them) to k; *xy_out, *yy_out = the reference's running sums at the end.
template <int E>
__device__ __forceinline__ void search_event(int lane, const SearchVec& v, int (&ya)[4], int k, int i, double xy,
                                             double yy, double lambda, const double* rsq, double* xy_out,
                                             double* yy_out) {
  const int nn = v.nn;
  const int rdo_pulses = 1 + k / 4;
  double delta_rate = v.delta_rate;
  double accel_rate = 0.;
  if (k == 1) {
    if (nn == 15) {
      accel_rate = -8. / 15;
      delta_rate = 4.5 / 15 - accel_rate;
    } else if (nn == 8) {
      accel_rate = 5.7 / 8;
      delta_rate = 9.3 / 8 - accel_rate;
    }
  }
  for (; i < k; i++) {
    const bool plain = i < k - rdo_pulses;
    bool cont[E];    // contenders per slot
    double tval[E];  // RDO: the element's objective
    int total;
    if (plain) {
      const double bound = (xy + v.xmax) * (xy + v.xmax) * (yy + 2. * i + 1.);
      if (bound < DAALA_B200_PVQ_EXACT_BOUND) {
        const float xyf = (float)xy, yyf1 = (float)(yy + 1.);
        unsigned key[E], kmax = 0;
#pragma unroll
        for (int e = 0; e < E; e++) {
          float a = xyf + (float)v.xa[e];
          a *= a;
          const float b = yyf1 + (float)(2 * ya[e]);
          key[e] = e * 32 + lane < nn ? __float_as_uint(__fdividef(a, b)) : 0u;
          kmax = key[e] > kmax ? key[e] : kmax;
        }
        const unsigned mx = wmaxu(kmax);
        const unsigned thr = mx > 64u ? mx - 64u : 0u;
        int cnt = 0;
#pragma unroll
        for (int e = 0; e < E; e++) {
          cont[e] = e * 32 + lane < nn && key[e] >= thr;
          cnt += cont[e];
        }
        total = wsum(cnt);
      } else {
        // products may round: the reference's literal scan over every element
#pragma unroll
        for (int e = 0; e < E; e++) cont[e] = e * 32 + lane < nn;
        total = 2;
        PVQ_WARP_STAT(3);
      }
#pragma unroll
      for (int e = 0; e < E; e++) tval[e] = 0;
    } else {
      // 1/sqrt(yy + 2 y_j + 1): the reference's expression, tabulated for arguments below kRsqrtEntries
      const int iyy = yy < 1e9 ? (int)yy : 1000000000;
      int key[E], kmax = (int)0x80000000;
#pragma unroll
      for (int e = 0; e < E; e++) {
        const int j = e * 32 + lane;
        const int arg = iyy + 2 * ya[e] + 1;
        const double ryy = arg < kRsqrtEntries ? rsq[arg] : nl_rsqrt_small((int)(yy + 2 * ya[e] + 1));
        double t = xy + (double)v.xa[e];
        t = 2 * t * v.norm_1 * ryy - lambda * j * (delta_rate + j * accel_rate);
        tval[e] = t;
        key[e] = j < nn ? ordered_key((float)t) : (int)0x80000000;
        kmax = key[e] > kmax ? key[e] : kmax;
      }
      const int mx = wmax(kmax);
      int cnt = 0;
#pragma unroll
      for (int e = 0; e < E; e++) {
        cont[e] = e * 32 + lane < nn && key[e] == mx;
        cnt += cont[e];
      }
      total = wsum(cnt);
    }
    PVQ_WARP_STAT(total == 1 ? 0 : plain ? 1 : 2);
    int pos;  // index of the chosen element
    if (total == 1) {
      int mine = -1;
#pragma unroll
      for (int e = 0; e < E; e++) if (cont[e]) mine = e * 32 + lane;
      const unsigned who = __ballot_sync(kFull, mine >= 0);
      pos = __shfl_sync(kFull, mine, __ffs(who) - 1);
    } else {
      // the reference's sequential scan restricted to the contenders, in index order: one loop body for
      // all slots
      pos = -1;
      double ba = 0, bb = 1;
      unsigned mk[E];
#pragma unroll
      for (int e = 0; e < E; e++) mk[e] = __ballot_sync(kFull, cont[e]);
      int e = 0;
      unsigned m = mk[0];
      for (;;) {
        while (!m && ++e < E) {
#pragma unroll
          for (int t = 1; t < E; t++) if (e == t) m = mk[t];
        }
        if (!m) break;
        const int l = __ffs(m) - 1;
        m &= m - 1;
        int sxa = v.xa[0], sya = ya[0];
        double stv = tval[0];
#pragma unroll
        for (int t = 1; t < E; t++) if (e == t) { sxa = v.xa[t]; sya = ya[t]; stv = tval[t]; }
        if (plain) {
          const int xj = __shfl_sync(kFull, sxa, l);
          const int yj = __shfl_sync(kFull, sya, l);
          double a = xy + (double)xj;
          const double b = yy + 2 * yj + 1;
          a *= a;
          if (pos < 0 || a * bb > ba * b) { ba = a; bb = b; pos = e * 32 + l; }
        } else {
          const double t = wfetch(stv, l);
          if (pos < 0 || t > ba) { ba = t; pos = e * 32 + l; }
        }
      }
    }
    const int src = pos & 31, slot = pos >> 5;
    int sx = v.xa[0], sy = ya[0];
#pragma unroll
    for (int e = 1; e < E; e++) if (slot == e) { sx = v.xa[e]; sy = ya[e]; }
    const int px = __shfl_sync(kFull, sx, src);
    const int py = __shfl_sync(kFull, sy, src);
    xy = xy + (double)px;
    yy = yy + 2 * py + 1;
#pragma unroll
    for (int e = 0; e < E; e++) if (e * 32 + lane == pos) ya[e]++;
  }
  *xy_out = xy;
  *yy_out = yy;
}

// What the three phases of one band share.  Between the phases it is parked in a record (band_ctx_*):
// in the warp's shared scratch when one warp runs them back to back (quantise_band_warp), in HBM when they
// run as separate kernels.
struct BandCtx {
  int x16[4], r16[4], xr[4];             // the vectors (int16 values), r16 after od_compute_householder
  int32_t cg, g, gain_offset;            // uniform
  int icgr, m, s;
  double best_dist, best_cost, skip_dist;
  int c_gain, c_theta, c_ts, c_k, c_cosd, c_alive, c_ev;   // lane c: candidate c
  int32_t c_qcg, c_qtheta;
  double c_sinprod, c_lambda, c_rate_ts;
  double e_xy, e_yy, e_xx;               // lane e: event e
  int e_sum, e_k, e_zero;
};

// ---- the context as a record -----------------------------------------------------------------------------
// vec: int16 [3][vstride] (x16, r16, xr); lanes: int32 [kCtxLaneWords][16] (only lanes 0..15 carry
// candidates / events); uni: int32 [kCtxUniWords].
constexpr int kCtxLaneWords = 24;
constexpr int kCtxUniWords = 16;
// The per-warp scratch quantise_band_warp takes, in int16 entries (4-byte aligned): the pulses of every
// search event (kMaxEvents rows of kMaxN), then the parked context (vec with vstride kMaxN, lanes, uni).
constexpr int kSnapEntries = kMaxEvents * kMaxN + 3 * kMaxN + 2 * (kCtxLaneWords * 16 + kCtxUniWords);

// Orders a warp's stores to a record before its lanes read each other's entries.  (The host emulation
// switches lanes only at collectives, in lane order, and every entry is read by its writer or a higher lane.)
#ifdef __CUDACC__
__device__ __forceinline__ void ctx_sync() { __syncwarp(); }
#else
inline void ctx_sync() {}
#endif

__device__ __forceinline__ void ctx_put_d(int32_t* lanes, int w, int lane, double v) {
  lanes[w * 16 + lane] = __double2loint(v);
  lanes[(w + 1) * 16 + lane] = __double2hiint(v);
}
__device__ __forceinline__ double ctx_get_d(const int32_t* lanes, int w, int lane) {
  return __hiloint2double(lanes[(w + 1) * 16 + lane], lanes[w * 16 + lane]);
}

// after band_setup
__device__ __forceinline__ void band_ctx_store_setup(int lane, const BandCtx& B, int n, int16_t* vec, int vstride,
                                                     int32_t* lanes, int32_t* uni) {
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const int j = e * 32 + lane;
    if (j < n) {
      vec[j] = (int16_t)B.x16[e];
      vec[vstride + j] = (int16_t)B.r16[e];
      vec[2 * vstride + j] = (int16_t)B.xr[e];
    }
  }
  if (lane < 16) {
    lanes[0 * 16 + lane] = B.c_gain;
    lanes[1 * 16 + lane] = B.c_theta;
    lanes[2 * 16 + lane] = B.c_ts;
    lanes[3 * 16 + lane] = B.c_k;
    lanes[4 * 16 + lane] = B.c_cosd;
    lanes[5 * 16 + lane] = B.c_alive;
    lanes[6 * 16 + lane] = B.c_qcg;
    lanes[7 * 16 + lane] = B.c_qtheta;
    ctx_put_d(lanes, 8, lane, B.c_sinprod);
    ctx_put_d(lanes, 10, lane, B.c_lambda);
    ctx_put_d(lanes, 12, lane, B.c_rate_ts);
  }
  if (lane == 0) {
    uni[0] = B.cg; uni[1] = B.g; uni[2] = B.gain_offset; uni[3] = B.icgr; uni[4] = B.m; uni[5] = B.s;
    uni[6] = __double2loint(B.best_dist); uni[7] = __double2hiint(B.best_dist);
    uni[8] = __double2loint(B.best_cost); uni[9] = __double2hiint(B.best_cost);
    uni[10] = __double2loint(B.skip_dist); uni[11] = __double2hiint(B.skip_dist);
  }
}
// what band_search needs
__device__ __forceinline__ void band_ctx_load_search(int lane, BandCtx& B, int n, const int16_t* vec, int vstride,
                                                     const int32_t* lanes) {
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const int j = e * 32 + lane;
    B.x16[e] = j < n ? vec[j] : 0;
    B.xr[e] = j < n ? vec[2 * vstride + j] : 0;
  }
  const int l = lane & 15;
  B.c_k = lanes[3 * 16 + l];
  B.c_alive = lane < 16 ? lanes[5 * 16 + l] : 0;
  B.c_lambda = ctx_get_d(lanes, 10, l);
}
// after band_search
__device__ __forceinline__ void band_ctx_store_search(int lane, const BandCtx& B, int32_t* lanes) {
  if (lane < 16) {
    lanes[14 * 16 + lane] = B.c_ev;
    ctx_put_d(lanes, 15, lane, B.e_xy);
    ctx_put_d(lanes, 17, lane, B.e_yy);
    ctx_put_d(lanes, 19, lane, B.e_xx);
    lanes[21 * 16 + lane] = B.e_sum;
    lanes[22 * 16 + lane] = B.e_k;
    lanes[23 * 16 + lane] = B.e_zero;
  }
}
// everything, for band_finish
__device__ __forceinline__ void band_ctx_load_finish(int lane, BandCtx& B, int n, const int16_t* vec, int vstride,
                                                     const int32_t* lanes, const int32_t* uni) {
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const int j = e * 32 + lane;
    B.x16[e] = j < n ? vec[j] : 0;
    B.r16[e] = j < n ? vec[vstride + j] : 0;
    B.xr[e] = j < n ? vec[2 * vstride + j] : 0;
  }
  const int l = lane & 15;
  const bool on = lane < 16;
  B.c_gain = lanes[0 * 16 + l];
  B.c_theta = lanes[1 * 16 + l];
  B.c_ts = lanes[2 * 16 + l];
  B.c_k = lanes[3 * 16 + l];
  B.c_cosd = lanes[4 * 16 + l];
  B.c_alive = on ? lanes[5 * 16 + l] : 0;
  B.c_qcg = lanes[6 * 16 + l];
  B.c_qtheta = lanes[7 * 16 + l];
  B.c_sinprod = ctx_get_d(lanes, 8, l);
  B.c_lambda = ctx_get_d(lanes, 10, l);
  B.c_rate_ts = ctx_get_d(lanes, 12, l);
  B.c_ev = on ? lanes[14 * 16 + l] : -1;
  B.e_xy = on ? ctx_get_d(lanes, 15, l) : 0.;
  B.e_yy = on ? ctx_get_d(lanes, 17, l) : 0.;
  B.e_xx = on ? ctx_get_d(lanes, 19, l) : 0.;
  B.e_sum = on ? lanes[21 * 16 + l] : 0;
  B.e_k = on ? lanes[22 * 16 + l] : 0;
  B.e_zero = on ? lanes[23 * 16 + l] : 0;
  B.cg = uni[0]; B.g = uni[1]; B.gain_offset = uni[2]; B.icgr = uni[3]; B.m = uni[4]; B.s = uni[5];
  B.best_dist = __hiloint2double(uni[7], uni[6]);
  B.best_cost = __hiloint2double(uni[9], uni[8]);
  B.skip_dist = __hiloint2double(uni[11], uni[10]);
}

// Phase A of a band: everything of pvq_theta (src/pvq_encoder.c:333) before the first search.
// x0 / r0 / qm point at the band's first entry (r0 == NULL: no prediction, all zero).  int16 quantities of the reference are kept sign-extended
// in ints; scalar results are identical in every lane.
// kMode (all phases): 0 = the band size decides at run time, 1 = n <= 32 only, 2 = n = 128 only (kernels that
// serve one size class drop the other one's code and registers).
template <int kMode>
__device__ __forceinline__ void band_setup(int lane, BandCtx& B, const int32_t* x0, const int32_t* r0, int n, int q0,
                                           int beta, int is_keyframe, int pli, const int16_t* qm,
                                           double pvq_norm_lambda, const double* rsq) {
  int (&x16)[4] = B.x16; int (&r16)[4] = B.r16; int (&xr)[4] = B.xr;
  int32_t &cg = B.cg, &g = B.g, &gain_offset = B.gain_offset;
  int &icgr = B.icgr, &m = B.m, &s = B.s;
  double &best_dist = B.best_dist, &best_cost = B.best_cost, &skip_dist = B.skip_dist;
  int &c_gain = B.c_gain, &c_theta = B.c_theta, &c_ts = B.c_ts, &c_k = B.c_k, &c_cosd = B.c_cosd, &c_alive = B.c_alive;
  int32_t &c_qcg = B.c_qcg, &c_qtheta = B.c_qtheta;
  double &c_sinprod = B.c_sinprod, &c_lambda = B.c_lambda, &c_rate_ts = B.c_rate_ts;

  const double gain_weight = 1.4;
  const double cgain_1 = 1. / kCgainOne;
  const double cgain_2 = cgain_1 * cgain_1;
  const double theta_scale = (1 << kThetaShift) * 2. / M_PI;
  const double theta_scale_1 = 1. / theta_scale;
  const double trig_1 = 1. / 32768;
  const bool big = kMode == 0 ? n > 32 : kMode == 2;
  int xshift, rshift, r_nonnull = 0;
  {
    int32_t xv[4], rv[4];
    int32_t sx = 0, sr = 0;
#pragma unroll
    for (int e = 0; e < 4; e++) {
      xv[e] = rv[e] = 0;
      if (e && !big) continue;
      const int j = e * 32 + lane;
      if (j < n) {
        xv[e] = x0[j];
        rv[e] = r0 ? r0[j] : 0;
      }
      const int16_t tx = (int16_t)(xv[e] >> 8), tr = (int16_t)(rv[e] >> 8);
      sx += tx * (int32_t)tx;
      sr += tr * (int32_t)tr;
      r_nonnull |= rv[e] != 0;
    }
    sx = wsum(sx);
    sr = wsum(sr);
    r_nonnull = __any_sync(kFull, r_nonnull);
    xshift = 9 + ilog((uint32_t)(n + sx)) / 2 - 15;
    rshift = 9 + ilog((uint32_t)(n + sr)) / 2 - 14;
    if (xshift < 0) xshift = 0;
    if (rshift < 0) rshift = 0;
#pragma unroll
    for (int e = 0; e < 4; e++) {
      x16[e] = r16[e] = xr[e] = 0;
      if (e && !big) continue;
      const int j = e * 32 + lane;
      const int qmv = j < n ? qm[j] : 0;
      x16[e] = (int16_t)shr_round(xv[e] * qmv, kQmShift + xshift);
      r16[e] = (int16_t)shr_round(rv[e] * qmv, kQmShift + rshift);
    }
  }
  long long scorr = 0;
  int32_t accx = 0, accr = 0;
#pragma unroll
  for (int e = 0; e < 4; e++) {
    if (e && !big) break;
    scorr += mul16(x16[e], r16[e]);
    accx += x16[e] * x16[e];
    accr += r16[e] * r16[e];
  }
  double corr = (double)wsum64(scorr);
  accx = wsum(accx);
  accr = wsum(accr);
  // the two gains in parallel: even lanes the input's, odd lanes the reference's
  int32_t gr, cgr;
  {
    const long long pk = nl_gain(lane & 1 ? accr : accx, q0, beta, lane & 1 ? rshift : xshift);
    const int gl = (int)(uint32_t)pk, cgl = (int)(pk >> 32);
    g = __shfl_sync(kFull, gl, 0);
    cg = __shfl_sync(kFull, cgl, 0);
    gr = __shfl_sync(kFull, gl, 1);
    cgr = __shfl_sync(kFull, cgl, 1);
  }
  const int cfl_enabled = is_keyframe && pli != 0;
  if (cfl_enabled) cgr = kCgainOne;
  icgr = shr_round(cgr, kCgainShift);
  gain_offset = cgr - shl(icgr, kCgainShift);
  best_dist = gain_weight * cg * cg * cgain_2;
  best_cost = best_dist + pvq_norm_lambda * 0.;  // od_pvq_rate(0, 0, -1, 0, ...) == 0
  corr = nl_div(corr, 1e-100 + nl_div(g * (double)gr, (double)shl(1, xshift + rshift)));
  corr = corr < 1. ? corr : 1.;
  corr = corr > -1. ? corr : -1.;
  if (is_keyframe) {
    skip_dist = gain_weight * cg * cg * cgain_2;
  } else {
    skip_dist = gain_weight * (cg - cgr) * (cg - cgr) + cgr * (double)cg * (2 - 2 * corr);
    skip_dist *= cgain_2;
    const int32_t scgr = gain_offset > 0 ? gain_offset : 0;
    if (icgr == 0) {
      best_dist = gain_weight * (cg - scgr) * (cg - scgr) + scgr * (double)cg * (2 - 2 * corr);
      best_dist *= cgain_2;
    }
    best_cost = best_dist + pvq_norm_lambda * 0.;  // od_pvq_rate(0, icgr, 0, 0, ...) == 0
  }
  const double dist0 = best_dist;

  // ---- with-reference setup: angle, Householder reflection (uniform) ------------------------------------
  const bool have_ref = r_nonnull && corr > 0;
  int32_t theta = 0;
  m = 0;
  s = 1;
  if (have_ref) {
    theta = round32(theta_scale * nl_acos(corr));
    // od_compute_householder, src/pvq.c:498: first largest |r| (strict ">" from maxr = 0)
    int key = -1;
#pragma unroll
    for (int e = 0; e < 4; e++) {
      if (e && !big) break;
      const int j = e * 32 + lane;
      const int kk = j < n ? (abs(r16[e]) << 7) | (127 - j) : -1;
      key = kk > key ? kk : key;
    }
    key = wmax(key);
    m = (key >> 7) > 0 ? 127 - (key & 127) : 0;
    const int rm = __shfl_sync(kFull, pick4(r16, m >> 5), m & 31);
    s = rm > 0 ? 1 : -1;
#pragma unroll
    for (int e = 0; e < 4; e++)
      if (e * 32 + lane == m) r16[e] = (int16_t)(r16[e] + shr_round(gr * s, rshift));
    householder_apply_warp(lane, big, xr, x16, r16, n);
    // drop element m: xr[j] <- xr[j + 1] for j >= m
#pragma unroll
    for (int e = 0; e < 4; e++) {
      if (e && !big) break;
      const int t1 = __shfl_sync(kFull, xr[e], (lane + 1) & 31);
      const int t2 = e + 1 < 4 ? __shfl_sync(kFull, xr[e + 1 < 4 ? e + 1 : e], 0) : 0;
      const int nxt = lane == 31 ? t2 : t1;
      if (e * 32 + lane >= m) xr[e] = nxt;
    }
  }

  // ---- candidates: one per lane (the same calls for both kinds, with per-lane arguments) ----------------
  c_gain = 0; c_theta = -1; c_ts = 0; c_k = 0; c_cosd = 0; c_qcg = 0; c_qtheta = 0;
  c_sinprod = 0; c_lambda = 0; c_rate_ts = 0;
  bool c_valid = false;
  {
    const bool wref = lane < 12;
    const bool nref = lane == 12 || lane == 13;
    int i = 0, j = -1;
    if (wref && have_ref) {
      const int gain_bound = (cg - gain_offset) >> kCgainShift;
      i = (gain_bound - 1 > 1 ? gain_bound - 1 : 1) + (lane >> 2);
      c_valid = i <= gain_bound + 1;
      c_qcg = shl(i, kCgainShift) + gain_offset;
    } else if (nref && ((is_keyframe && pli == 0) || corr < .5 || cg < (int32_t)shl(2, kCgainShift))) {
      const int gain_bound = cg >> kCgainShift;
      i = (gain_bound > 1 ? gain_bound : 1) + (lane - 12);
      c_valid = i <= gain_bound + 1;
      c_qcg = shl(i, kCgainShift);
    }
    if (!c_valid) c_qcg = kCgainOne;   // harmless arguments for the idle lanes
    if (wref) {
      c_ts = compute_max_theta(c_qcg, beta);
      int lo = (int)floor(.5 + nl_div(theta * theta_scale_1 * 2, M_PI) * c_ts) - 2;
      int hi = (int)ceil(nl_div(theta * theta_scale_1 * 2, M_PI) * c_ts);
      if (lo < 0) lo = 0;
      if (hi > c_ts - 1) hi = c_ts - 1;
      j = lo + (lane & 3);
      c_valid = c_valid && j <= hi;
    } else {
      c_ts = 0;
    }
    const long long tk = nl_theta_k(c_qcg, j, c_ts, !wref, n, beta);
    c_qtheta = (int32_t)(tk >> 32);
    c_k = (int)(uint32_t)tk;
    c_gain = i;
    c_theta = wref ? j : -1;
    // distortion pre-tests (src/pvq_encoder.c:529,582), lambda of the search, rate constants
    c_cosd = nl_cos(theta - c_qtheta);
    const int sin_q = nl_cos(32768 - c_qtheta), sin_t = nl_cos(32768 - theta);
    double dist = gain_weight * (c_qcg - cg) * (c_qcg - cg);
    double g2 = c_qcg * (double)cg;
    if (wref) {
      const double dist_theta = 2 - 2. * c_cosd * trig_1;
      dist = dist + c_qcg * (double)cg * dist_theta;
      const double sin_theta = sin_t * trig_1;
      c_sinprod = sin_theta * sin_q * trig_1;
      g2 = g2 * c_sinprod;
    }
    dist *= cgain_2;
    g2 = g2 * cgain_2;
    c_alive = c_valid && !(wref ? dist > dist0 + 1.0 * pvq_norm_lambda && c_k != 0 : dist > dist0 && c_k != 0);
    c_lambda = nl_div(pvq_norm_lambda, 1e-30 + g2);
    c_rate_ts = c_ts < kLogEntries ? rsq[kRsqrtEntries + (c_ts > 0 ? c_ts : 1)]
                                   : .9 * (M_LOG2E * nl_log((double)c_ts));
  }
}

// Phase B: the searches of all events.  `snap`: kMaxEvents rows of snap_stride int16, private to the band.
template <int kMode>
__device__ __forceinline__ void band_search(int lane, BandCtx& B, int n, int16_t* snap, int snap_stride,
                                            const double* rsq, const int32_t* pre_ev = nullptr,
                                            const int16_t* pre_snap = nullptr) {
  const bool big = kMode == 0 ? n > 32 : kMode == 2;
  const int (&x16)[4] = B.x16; const int (&xr)[4] = B.xr;
  const int &c_k = B.c_k, &c_alive = B.c_alive;
  const double &c_lambda = B.c_lambda;
  int &c_ev = B.c_ev;
  double &e_xy = B.e_xy, &e_yy = B.e_yy, &e_xx = B.e_xx;
  int &e_sum = B.e_sum, &e_k = B.e_k, &e_zero = B.e_zero;
  unsigned alive_w = __ballot_sync(kFull, c_alive && lane < 12);
  unsigned alive_n = __ballot_sync(kFull, c_alive && lane >= 12);
  if (pre_ev) alive_n = 0;   // the no-reference events were searched ahead of time (band_noref_export)

  // ---- events: the searches ---------------------------------------------------------------------------
  int ya[4];  // pulses of the running search, magnitudes (the reference's y_tmp without signs)
#pragma unroll
  for (int e = 0; e < 4; e++) ya[e] = 0;
  SearchVec sv;
  sv.nn = n;
  sv.xx = 0;
  int prev_k = 0, nev = 0;
  c_ev = -1;
  int phase = 0;  // 1: with-reference vector loaded, 2: no-reference vector
  e_xy = 0; e_yy = 0; e_xx = 0; e_sum = 0; e_k = 0; e_zero = 0;   // lane `event`: scalars of that event
  while (alive_w | alive_n) {
    unsigned grp;
    int kcur, leader;
    const bool noref_ev = alive_w == 0;
    if (!noref_ev) {
      const int key = (alive_w >> lane) & 1 ? (c_k << 4) | lane : 0x7fffffff;
      const int mn = wmin(key);
      kcur = mn >> 4;
      leader = mn & 15;
      grp = __ballot_sync(kFull, ((alive_w >> lane) & 1) && c_k == kcur);
      alive_w &= ~grp;
    } else {
      leader = __ffs(alive_n) - 1;
      grp = 1u << leader;
      alive_n &= ~grp;
      kcur = __shfl_sync(kFull, c_k, leader);
    }
    const int want = noref_ev ? 2 : 1;
    if (phase != want) {
      // (the first no-reference candidate of the list restarts the pulse reuse: prev_k = 0)
      phase = want;
      prev_k = 0;
      // element-wise: a reference to one of the two arrays, chosen at run time, would put both (and the
      // context around them) in local memory
      int src[4];
#pragma unroll
      for (int e = 0; e < 4; e++) src[e] = noref_ev ? x16[e] : xr[e];
      if (big) search_init<4>(lane, sv, src, noref_ev ? n : n - 1);
      else search_init<1>(lane, sv, src, noref_ev ? n : n - 1);
    }
    double xy = 0, yy = 0;
    const bool zero_ev = !noref_ev && kcur == 0;
    if (zero_ev) {
#pragma unroll
      for (int e = 0; e < 4; e++) ya[e] = 0;
    } else {
      const double lambda = wfetch(c_lambda, leader);
      const int i = search_start(lane, sv, ya, kcur, prev_k, big, &xy, &yy);
      if (big) search_event<4>(lane, sv, ya, kcur, i, xy, yy, lambda, rsq, &xy, &yy);
      else search_event<1>(lane, sv, ya, kcur, i, xy, yy, lambda, rsq, &xy, &yy);
    }
    prev_k = kcur;
    int sj = 0;
#pragma unroll
    for (int e = 0; e < 4; e++) {
      if (e && !big) break;
      const int j = e * 32 + lane;
      if (j < sv.nn) sj += j * ya[e];
      if (j < n) snap[nev * snap_stride + j] = (int16_t)(j < sv.nn ? ya[e] : 0);
    }
    sj = wsum(sj);
    if (lane == nev) {
      e_xy = xy;
      e_yy = yy;
      e_xx = sv.xx;
      e_sum = sj;
      e_k = kcur;
      e_zero = zero_ev;
    }
    if ((grp >> lane) & 1) c_ev = nev;
    nev++;
  }
  if (pre_ev) {
    // import the no-reference events: they follow the with-reference ones in the reference's candidate order
    const int cev = (lane == 12 || lane == 13) ? pre_ev[lane - 12] : -1;
    const int nimp = wmax(cev) + 1;
    if (cev >= 0) c_ev = nev + cev;
    if (lane >= nev && lane < nev + nimp) {
      const int32_t* r = pre_ev + 2 + (lane - nev) * 9;
      e_xy = __hiloint2double(r[1], r[0]);
      e_yy = __hiloint2double(r[3], r[2]);
      e_xx = __hiloint2double(r[5], r[4]);
      e_sum = r[6];
      e_k = r[7];
      e_zero = r[8];
    }
    for (int ev = 0; ev < nimp; ev++) {
#pragma unroll
      for (int e = 0; e < 4; e++) {
        if (e && !big) break;
        const int j = e * 32 + lane;
        if (j < n) snap[(nev + ev) * snap_stride + j] = pre_snap[ev * n + j];
      }
    }
  }

}

// Phase C: costs, the reference's fold, synthesis of the winner (od_pvq_synthesis_partial, src/pvq.c:1037).
// Returns the coded gain index.
template <int kMode>
__device__ __forceinline__ int band_finish(int lane, const BandCtx& B, const int16_t* snap, int snap_stride, int32_t* out,
                                           const int32_t* r0, int n, int q0, int32_t* yout, int* itheta,
                                           int* max_theta, int* vk, int beta, double* skip_term, int is_keyframe,
                                           int pli, const int16_t* qm_inv, double pvq_norm_lambda) {
  const double gain_weight = 1.4;
  const double cgain_1 = 1. / kCgainOne;
  const double cgain_2 = cgain_1 * cgain_1;
  const double trig_1 = 1. / 32768;
  const bool big = kMode == 0 ? n > 32 : kMode == 2;
  const int cfl_enabled = is_keyframe && pli != 0;
  const int (&x16)[4] = B.x16; const int (&r16)[4] = B.r16; const int (&xr)[4] = B.xr;
  const int32_t cg = B.cg;
  int32_t g = B.g, gain_offset = B.gain_offset;
  const int icgr = B.icgr, m = B.m, s = B.s;
  double best_dist = B.best_dist, best_cost = B.best_cost;
  const double skip_dist = B.skip_dist;
  const int c_gain = B.c_gain, c_theta = B.c_theta, c_ts = B.c_ts, c_k = B.c_k, c_cosd = B.c_cosd, c_ev = B.c_ev;
  const int32_t c_qcg = B.c_qcg, c_qtheta = B.c_qtheta;
  const double c_sinprod = B.c_sinprod, c_rate_ts = B.c_rate_ts;
  const double e_xy = B.e_xy, e_yy = B.e_yy, e_xx = B.e_xx;
  const int e_sum = B.e_sum, e_k = B.e_k, e_zero = B.e_zero;
  int32_t theta = 0;
  // ---- all events in parallel: cos distance and the shared part of od_pvq_rate (src/pvq_encoder.c:247) ---
  double e_cos = 0, e_rate = 0;
  {
    const int kk = e_k > 0 ? e_k : 1;
    const double cd = nl_div(e_xy, 1e-100 + nl_sqrt(e_xx * e_yy));
    const double f = nl_div((double)e_sum, (double)(kk * n));
    const double t = nl_div(nl_log(n * 2 * (1 * f + .025)) * kk, (double)n);
    const double rate = (1 + .4 * f) * n * (M_LOG2E * nl_log(1 + (0 > t ? 0 : t))) + 3;
    e_cos = e_zero ? 0. : cd;
    e_rate = e_k == 0 ? 0. : rate;
  }
  // ---- all candidates in parallel: cost ----------------------------------------------------------------
  double c_dist = 0, cost = 0;
  {
    const int src = c_ev >= 0 ? c_ev : 0;
    const double cos_dist = wfetch(e_cos, src);
    double rate = wfetch(e_rate, src);
    double dist;
    if (lane >= 12) {
      dist = gain_weight * (c_qcg - cg) * (c_qcg - cg) + c_qcg * (double)cg * (2 - 2 * cos_dist);
    } else {
      if (c_gain > 0 && c_theta >= 0) {
        rate += c_rate_ts;
        if (is_keyframe && pli == 0) rate += 6;
        if (c_gain == icgr) rate -= .5;
      }
      const double dist_theta = 2 - 2. * c_cosd * trig_1 + c_sinprod * (2 - 2 * cos_dist);
      dist = gain_weight * (c_qcg - cg) * (c_qcg - cg) + c_qcg * (double)cg * dist_theta;
    }
    dist *= cgain_2;
    c_dist = dist;
    cost = dist + pvq_norm_lambda * rate;
  }
  // ---- the reference's fold, in its order: events ascending, candidates of an event in insertion order ----
  int best_lane = -1;
  {
    unsigned rem = __ballot_sync(kFull, c_ev >= 0);
    while (rem) {
      const int key = (rem >> lane) & 1 ? (c_ev << 5) | lane : 0x7fffffff;
      const int l = wmin(key) & 31;
      rem &= ~(1u << l);
      const double cl = wfetch(cost, l);
      if (l >= 12 ? cl <= best_cost : cl < best_cost) {
        best_cost = cl;
        best_lane = l;
      }
    }
  }

  // ---- the winner --------------------------------------------------------------------------------------
  int qg = 0, best_k = 0;
  int noref = is_keyframe ? 1 : 0;
  *itheta = is_keyframe ? -1 : 0;
  *max_theta = 0;
  // theta: best_qtheta
  int ybest[4];
#pragma unroll
  for (int e = 0; e < 4; e++) ybest[e] = 0;
  if (best_lane >= 0) {
    qg = __shfl_sync(kFull, c_gain, best_lane);
    best_k = __shfl_sync(kFull, c_k, best_lane);
    *itheta = __shfl_sync(kFull, c_theta, best_lane);
    *max_theta = __shfl_sync(kFull, c_ts, best_lane);
    theta = __shfl_sync(kFull, c_qtheta, best_lane);
    best_dist = wfetch(c_dist, best_lane);
    noref = best_lane >= 12;
    const int ev = __shfl_sync(kFull, c_ev, best_lane);
#pragma unroll
    for (int e = 0; e < 4; e++) {
      if (e && !big) break;
      const int j = e * 32 + lane;
      const int v = noref ? x16[e] : xr[e];
      const int a = j < n ? snap[ev * snap_stride + j] : 0;
      ybest[e] = j < (noref ? n : n - 1) ? (v < 0 ? -a : a) : 0;
    }
  }
  int skip = 0;
  if (noref) {
    if (qg == 0) skip = 1;
  } else {
    if (!is_keyframe && qg == 0) skip = icgr ? 1 : 2;
    if (qg == icgr && *itheta == 0 && !cfl_enabled) skip = 2;
  }
  int32_t res[4];
  if (skip) {
#pragma unroll
    for (int e = 0; e < 4; e++) res[e] = (skip == 2 && r0 && e * 32 + lane < n) ? r0[e * 32 + lane] : 0;
  } else {
    if (noref) gain_offset = 0;
    g = gain_expand(shl(qg, kCgainShift) + gain_offset, q0, beta);
    // od_pvq_synthesis_partial, src/pvq.c:1037
    const int nn = n - !noref;
    int syy = 0;
#pragma unroll
    for (int e = 0; e < 4; e++) if (e * 32 + lane < nn) syy += ybest[e] * ybest[e];
    const int yy = wsum(syy);
    int gshift = ilog((uint32_t)g) - 14;
    if (gshift < 0) gshift = 0;
    int32_t scale;
    if (yy == 0) {
      scale = 0;
    } else {
      int rsh;
      const int16_t rs = rsqrt32(yy, &rsh);
      scale = vshr_round64(rs * (int64_t)g, rsh + gshift - 16);
    }
    const int qshift = kQmInvShift - gshift;
    int xs[4];
    if (noref) {
#pragma unroll
      for (int e = 0; e < 4; e++) xs[e] = mul16_32_q16(ybest[e], scale);
    } else {
      scale = round32(scale * (1. / 32768) * nl_cos(32768 - theta));
      int f[4];
#pragma unroll
      for (int e = 0; e < 4; e++) f[e] = e * 32 + lane < nn ? (int16_t)mul16_32_q16(ybest[e], scale) : 0;
      const int xm = (int16_t)floor(.5 + -s * (shr_round(g, gshift)) * (1. / 32768) * nl_cos(theta));
#pragma unroll
      for (int e = 0; e < 4; e++) {
        xs[e] = 0;
        if (e && !big) continue;
        // value of element idx - 1
        const int t1 = __shfl_sync(kFull, f[e], (lane + 31) & 31);
        const int t2 = e > 0 ? __shfl_sync(kFull, f[e > 0 ? e - 1 : 0], 31) : 0;
        const int fprev = lane == 0 ? t2 : t1;
        const int j = e * 32 + lane;
        xs[e] = j < m ? f[e] : (j == m ? xm : fprev);
        if (j >= n) xs[e] = 0;
      }
      householder_apply_warp(lane, big, xs, xs, r16, n);
    }
#pragma unroll
    for (int e = 0; e < 4; e++) {
      const int j = e * 32 + lane;
      res[e] = j < n ? shr_round(xs[e] * qm_inv[j], qshift) : 0;
    }
  }
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const int j = e * 32 + lane;
    if (j < n) {
      out[j] = res[e];
      yout[j] = ybest[e];
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

// No-reference events searched ahead of time (keyframe luma: they depend on the input vector alone, while
// the with-reference half of pvq_theta has to wait for the neighbours the prediction comes from).  After
// band_setup with r0 = NULL and band_search: pre_ev = {c_ev of lanes 12, 13; per event xy, yy, xx, sum, k,
// zero} (20 words), pre_snap = the events' pulses, n int16 each.
constexpr int kPreEvWords = 20;
__device__ __forceinline__ void band_noref_export(int lane, const BandCtx& B, int n, const int16_t* snap,
                                                  int snap_stride, int32_t* pre_ev, int16_t* pre_snap) {
  const int cev = (lane == 12 || lane == 13) ? B.c_ev : -1;
  const int nev = wmax(cev) + 1;
  if (lane == 12 || lane == 13) pre_ev[lane - 12] = B.c_ev;
  if (lane < nev) {
    int32_t* r = pre_ev + 2 + lane * 9;
    r[0] = __double2loint(B.e_xy); r[1] = __double2hiint(B.e_xy);
    r[2] = __double2loint(B.e_yy); r[3] = __double2hiint(B.e_yy);
    r[4] = __double2loint(B.e_xx); r[5] = __double2hiint(B.e_xx);
    r[6] = B.e_sum; r[7] = B.e_k; r[8] = B.e_zero;
  }
  for (int ev = 0; ev < nev; ev++)
    for (int j = lane; j < n; j += 32) pre_snap[ev * n + j] = snap[ev * snap_stride + j];
}

// One band by one warp, the three phases back to back.  `snap`: kSnapEntries int16 of scratch private to
// the warp (shared memory); `rsq`: kTableDoubles doubles filled by pvq_fill_rsqrt_table.
// The context is parked in the scratch between the phases, so that only what the search reads is live
// across it: held in registers throughout, the whole context does not fit the 64 registers a thread of the
// persistent kernel has and would spill to local memory.
template <int kMode = 0>
__device__ __forceinline__ int quantise_band_warp(int lane, int16_t* snap, const double* rsq, int32_t* out, const int32_t* x0,
                                                  const int32_t* r0, int n, int q0, int32_t* yout, int* itheta,
                                                  int* max_theta, int* vk, int beta, double* skip_term, int is_keyframe,
                                                  int pli, const int16_t* qm, const int16_t* qm_inv,
                                                  double pvq_norm_lambda, const int32_t* pre_ev = nullptr,
                                                  const int16_t* pre_snap = nullptr) {
  int16_t* vec = snap + kMaxEvents * kMaxN;
  int32_t* lanes = reinterpret_cast<int32_t*>(vec + 3 * kMaxN);
  int32_t* uni = lanes + kCtxLaneWords * 16;
  {
    BandCtx B;
    band_setup<kMode>(lane, B, x0, r0, n, q0, beta, is_keyframe, pli, qm, pvq_norm_lambda, rsq);
    ctx_sync();   // the previous band's reads of the record come first
    band_ctx_store_setup(lane, B, n, vec, kMaxN, lanes, uni);
  }
  ctx_sync();
  {
    BandCtx B;
    band_ctx_load_search(lane, B, n, vec, kMaxN, lanes);
    band_search<kMode>(lane, B, n, snap, kMaxN, rsq, pre_ev, pre_snap);
    band_ctx_store_search(lane, B, lanes);
  }
  ctx_sync();
  BandCtx B;
  band_ctx_load_finish(lane, B, n, vec, kMaxN, lanes, uni);
  return band_finish<kMode>(lane, B, snap, kMaxN, out, r0, n, q0, yout, itheta, max_theta, vk, beta, skip_term, is_keyframe, pli,
                     qm_inv, pvq_norm_lambda);
}

}  // namespace pvq
}  // namespace daala_b200
