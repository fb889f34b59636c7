// Small device helpers shared by the PVQ translation units (pvq_kernels.cu, kf_engine.cu).
// Include after gen/coding_order.inc.
#pragma once
#include <stdint.h>

namespace daala_b200 {
namespace pvq {

// Band boundaries in coding order (OD_BAND_OFFSETS, src/partition.c:85-91).
// 1, then 16, 24, 32 times 4^g for g = 0, 1, 2: arithmetic rather than a table, which a run-time index
// would put in local memory.
__device__ __forceinline__ int band_start(int band) {
  const int g = (band - 1) / 3, r = (band - 1) - 3 * g;
  return band == 0 ? 1 : (16 + 8 * r) << (2 * g);
}

__device__ __forceinline__ int num_bands(int bs) { return bs == 0 ? 1 : bs == 1 ? 4 : bs == 2 ? 7 : 9; }

// Coding-order index i (1 <= i < coded length) -> (row, column) of the coefficient inside its block:
// stage m of od_raster_to_coding_order (src/partition.c:123) lists raster indices of an m x m layout.
__device__ __forceinline__ void scan_rc(int i, int* r, int* c) {
  int v, sh;
  if (i < 16) { v = kScan4[i - 1]; sh = 2; }
  else if (i < 64) { v = kScan8[i - 16]; sh = 3; }
  else if (i < 256) { v = kScan16[i - 64]; sh = 4; }
  else { v = kScan32[i - 256]; sh = 5; }
  *r = v >> sh;
  *c = v & ((1 << sh) - 1);
}

__device__ __forceinline__ int scan_to_raster(int i, int ln, int stride) {
  int r, c;
  (void)ln;
  scan_rc(i, &r, &c);
  return r * stride + c;
}

__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

}  // namespace pvq
}  // namespace daala_b200
