// Fixed-point PVQ arithmetic of Daala (OD_FLOAT_PVQ off) as device functions.
//
// Bit-exact restatements of the reference's shared encoder/decoder math,
// src/pvq.c: od_pvq_cos/sin :428/461, od_vector_log_mag :472,
// od_compute_householder :498, od_rcp :526, od_apply_householder :560,
// od_exp2/od_log2/od_pow :638-695, od_gain_compand :706, od_sqrt :739,
// od_gain_expand :766, od_pvq_compute_gain :824, od_pvq_compute_max_theta :855,
// od_pvq_compute_theta :874, od_pvq_compute_k :902, od_rsqrt :998,
// od_pvq_synthesis_partial :1037.  Q formats: gains Q8 (OD_CGAIN_SHIFT),
// beta Q12, angles in units of (pi/2)/32768, QM Q11 / inverse QM Q12.
// The 16-bit truncations below are semantic (the reference computes in
// int16_t); do not "simplify" them.
#pragma once
#include <stdint.h>

namespace daala_b200 {
namespace pvq {

constexpr int kCgainShift = 8;
constexpr int kCgainOne = 1 << kCgainShift;
constexpr int kCompandShift = 12;
constexpr int kBetaShift = 12;
constexpr int kBeta1 = 4096;
constexpr int kBeta15 = 6144;
constexpr int kQmShift = 11;
constexpr int kQmInvShift = 12;
constexpr int kThetaShift = 15;
constexpr int kMaxN = 128;  // OD_MAX_PVQ_SIZE

// 1/sqrt(i), i = 1..16, with the reference's 6-digit constants (od_rsqrt_table,
// src/pvq_encoder.c:53); larger arguments use 1./sqrt(i).  Kept in constant memory:
// a function-local array would be re-materialised on the stack at every call.
static __constant__ double kRsqrtSmall[16] = {1.000000, 0.707107, 0.577350, 0.500000, 0.447214, 0.408248,
                                       0.377964, 0.353553, 0.333333, 0.316228, 0.301511, 0.288675,
                                       0.277350, 0.267261, 0.258199, 0.250000};
// the rare large argument: out of line, the double-precision sqrt + divide sequences are long and this
// is used inside the hottest loops (instruction-cache footprint)
static __device__ __noinline__ double rsqrt_large(int i) { return 1. / sqrt((double)i); }
__device__ __forceinline__ double rsqrt_small_tbl(int i) {
  if (i <= 16) return kRsqrtSmall[i - 1];
  return rsqrt_large(i);
}

__device__ __forceinline__ int ilog(uint32_t v) { return v ? 32 - __clz((int)v) : 0; }
__device__ __forceinline__ int32_t shl(int32_t a, int s) { return (int32_t)((uint32_t)a << s); }
__device__ __forceinline__ int32_t shr_round(int32_t x, int s) { return (x + ((1 << s) >> 1)) >> s; }
__device__ __forceinline__ int32_t shr_round64(int64_t x, int s) {
  return (int32_t)((x + ((1 << s) >> 1)) >> s);
}
__device__ __forceinline__ int32_t vshr(int32_t x, int s) { return s > 0 ? x >> s : shl(x, -s); }
__device__ __forceinline__ int32_t vshr_round(int32_t x, int s) {
  return s > 0 ? shr_round(x, s) : shl(x, -s);
}
__device__ __forceinline__ int32_t vshr_round64(int64_t x, int s) {
  return s > 0 ? shr_round64(x, s) : shl((int32_t)x, -s);
}
__device__ __forceinline__ int32_t mul16(int32_t a, int32_t b) {
  return (int32_t)(int16_t)a * (int32_t)(int16_t)b;
}
__device__ __forceinline__ int32_t mul16_q15(int32_t a, int32_t b) { return mul16(a, b) >> 15; }
__device__ __forceinline__ int32_t mul16_q16(int32_t a, int32_t b) { return mul16(a, b) >> 16; }
__device__ __forceinline__ int32_t mul16_qbeta(int32_t a, int32_t b) { return mul16(a, b) >> kBetaShift; }
__device__ __forceinline__ int32_t mul16_32_q16(int32_t a, int32_t b) {
  return (int32_t)(((int16_t)a * (int64_t)b) >> 16);
}
__device__ __forceinline__ int32_t round32(double x) { return (int32_t)floor(.5 + x); }

__device__ __forceinline__ int16_t cos_quarter(int16_t x) {
  int16_t x2 = (int16_t)mul16_q15(x, x);
  int32_t v = (1073758164 - x * x + x2 * (-7654 + mul16_q16(x2, 16573 + mul16_q16(-2529, x2)))) >> 15;
  return (int16_t)(v < 32767 ? v : 32767);
}

__device__ __forceinline__ int pvq_cos(int32_t x) {
  x &= 0x1ffff;
  if (x > (1 << 16)) x = (1 << 17) - x;
  if (x & 0x7fff) {
    if (x < (1 << 15)) return cos_quarter((int16_t)x);
    return (int16_t)-cos_quarter((int16_t)(65536 - x));
  }
  if (x & 0xffff) return 0;
  if (x & 0x1ffff) return -32767;
  return 32767;
}

__device__ __forceinline__ int pvq_sin(int32_t x) { return pvq_cos(32768 - x); }

__device__ __forceinline__ int16_t rcp16(int16_t x) {
  int i = ilog((uint32_t)(int32_t)x) - 1;
  int16_t n = (int16_t)(vshr_round(x, i - 15) - 32768);
  int16_t r = (int16_t)(30840 + mul16_q15(-15420, n));
  r = (int16_t)(r - mul16_q15(r, mul16_q15(r, n) + r - 32768));
  r = (int16_t)(r - (1 + mul16_q15(r, mul16_q15(r, n) + r - 32768)));
  return (int16_t)vshr_round(r, i - 14);
}

__device__ __forceinline__ int16_t beta_rcp(int16_t beta) {
  if (beta == kBeta1) return kBeta1;
  if (beta == kBeta15) return 2731;
  return (int16_t)shr_round(rcp16((int16_t)(beta << (15 - 1 - kBetaShift))), 14 + 1 - kBetaShift);
}

__device__ __forceinline__ int32_t exp2_q15(int32_t x) {
  int integer = x >> 15;
  if (integer > 14) return 0x7f000000;
  if (integer < -15) return 0;
  int32_t f = x - shl(integer, 15);
  int32_t frac = mul16_q15(f, 22709 + mul16_q15(f, 7913 + mul16_q15(f, 1704 + mul16_q15(f, 443))));
  return vshr_round(32768 + frac, -integer) + 1;
}

__device__ __forceinline__ int16_t log2_q15(int16_t x) {
  return (int16_t)(x + mul16_q15(x, 14482 + mul16_q15(x, -23234 + mul16_q15(x, 13643
      + mul16_q15(x, -6403 + mul16_q15(x, 1515))))));
}

__device__ __forceinline__ int32_t pow_q(int32_t x, int16_t beta) {
  if (x == 0) return 0;
  int log2_x = ilog((uint32_t)x) - 1;
  int16_t t = (int16_t)(vshr(x, log2_x - 15) - 32768);
  int32_t logr = log2_q15(t) + (log2_x - kCompandShift) * 32768;
  logr = (int32_t)(((int16_t)beta * (int64_t)logr) >> kBetaShift);
  return exp2_q15(logr);
}

__device__ __forceinline__ int16_t rsqrt_norm(int16_t t) {
  int16_t n = (int16_t)(t - 32768);
  int32_t r = 23565 + mul16_q15(n, -13481 + mul16_q15(n, 6711));
  int32_t r2 = r * r;
  int32_t y = (((r2 >> 15) * n + r2) >> 12) - 131077;
  int32_t ry = r * y;
  return (int16_t)(r + ((((ry >> 16) * (3 * y) >> 3) - ry) >> 18));
}

__device__ __forceinline__ int16_t rsqrt32(int32_t x, int* shift) {
  int k = (ilog((uint32_t)x) - 1) >> 1;
  int s = 2 * k - 14;
  int16_t t = (int16_t)vshr(x, s);
  *shift = 14 + ((s + 16) >> 1);
  return rsqrt_norm(t);
}

__device__ __forceinline__ int16_t sqrt32(int32_t x, int* shift) {
  if (x == 0) {
    *shift = 0;
    return 0;
  }
  int k = (ilog((uint32_t)x) - 1) >> 1;
  int s = 2 * k - 14;
  int32_t t = vshr(x, s);
  *shift = 15 - ((s + 16) >> 1);
  int32_t v = shr_round(t * rsqrt_norm((int16_t)t), 15);
  return (int16_t)(v < 32767 ? v : 32767);
}

__device__ __forceinline__ int32_t gain_compand(int32_t g, int q0, int16_t beta) {
  if (beta == kBeta1) return (kCgainOne * g + (q0 >> 1)) / q0;
  int32_t e = pow_q(g, beta_rcp(beta));
  e <<= kCgainShift + kCompandShift - 15;
  return (e + (q0 >> 1)) / q0;
}

__device__ __forceinline__ int32_t gain_expand(int32_t cg0, int q0, int beta) {
  if (beta == kBeta1) return shr_round(cg0 * q0, kCgainShift);
  if (beta == kBeta15) {
    int outshift;
    int32_t irt = sqrt32(cg0 * q0, &outshift);
    int64_t tmp = cg0 * q0 * (int64_t)irt;
    return vshr_round64(tmp, kCgainShift + outshift + ((kCgainShift + kCompandShift) >> 1));
  }
  return shr_round(pow_q(shr_round(cg0 * q0, kCgainShift), (int16_t)beta), 15 - kCompandShift);
}

// Gain of a 16-bit vector whose sum of squares is `acc`.
__device__ __forceinline__ int32_t compute_gain_from_energy(int32_t acc, int q0, int32_t* g, int beta,
                                                            int bshift) {
  int sqrt_shift;
  int32_t irt = sqrt32(acc, &sqrt_shift);
  *g = vshr_round(irt, sqrt_shift - bshift);
  return gain_compand(*g, q0, (int16_t)beta);
}

__device__ __forceinline__ int compute_max_theta(int32_t qcg, int beta) {
  int ts = shr_round(qcg * mul16_qbeta(402, beta_rcp((int16_t)beta)), kCgainShift * 2);
  if (qcg < 358) ts = 1;
  return ts;
}

__device__ __forceinline__ int32_t compute_theta(int t, int max_theta) {
  if (max_theta == 0) return 0;
  return ((1 << kThetaShift) * (t < max_theta - 1 ? t : max_theta - 1) + (max_theta >> 1)) / max_theta;
}

// sqrt((n+3)/2) / sqrt((n+2)/2) in Q10, indexed by ilog(n + 1) (od_sqrt_table, src/pvq.c:909).
__device__ __forceinline__ int sqrt_tbl(int which, int idx) {
  // idx in {4,5,6,8}: n = 8,15,32,128 (and n-1 variants)
  switch (idx) {
    case 4: return which ? 2401 : 2290;
    case 5: return which ? 3072 : 2985;
    case 6: return which ? 4284 : 4222;
    case 8: return which ? 8287 : 8256;
    case 10: return which ? 16432 : 16416;
    case 12: return 32767;
    default: return 0;
  }
}

// nodesync == 1 always (OD_ROBUST_STREAM, src/internal.h:118).
__device__ __forceinline__ int compute_k(int32_t qcg, int itheta, int noref, int n, int beta) {
  int k;
  if (noref) {
    if (qcg == 0) return 0;
    if (n == 15 && qcg == kCgainOne && beta > 5120) return 1;
    k = shr_round64((int64_t)((qcg - (int64_t)51)
        * mul16_qbeta(beta_rcp((int16_t)beta), sqrt_tbl(1, ilog((uint32_t)(n + 1))))), kCgainShift + 10);
    return k > 1 ? k : 1;
  }
  if (itheta == 0) return 0;
  k = vshr_round64((shl(itheta, 15) - 6554) * (int64_t)sqrt_tbl(0, ilog((uint32_t)(n + 1))), 10 + 15);
  return k > 1 ? k : 1;
}

}  // namespace pvq
}  // namespace daala_b200
