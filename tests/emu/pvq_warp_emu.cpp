// The warp-per-band PVQ quantiser (daala_b200/csrc/pvq_warp.cuh) compiled for the host on the SIMT
// emulation of simt_emu.h: lets the CPU test suite pin the device algorithm against the reference build.
// Test infrastructure; never loaded by the product path.
#include "simt_emu.h"

// [0] unique contender, [1] plain-pulse exact fallback, [2] RDO-pulse exact fallback, [3] literal scan (x32 lanes)
#define DAALA_B200_EMU_STATS
extern "C" { long long daala_b200_pvq_warp_stats[4]; }

#include "pvq_warp.cuh"

using namespace daala_b200::pvq;

extern "C" int emu_quantise_band(int32_t* out, const int32_t* x0, const int32_t* r0, int n, int q0, int32_t* y, int* itheta,
                                 int* max_theta, int* vk, int beta, double* skip_term, int is_keyframe, int pli,
                                 const int16_t* qm, const int16_t* qm_inv, double lambda) {
  int gain[32], it[32], mt[32], k[32];
  double sd[32];
  static int16_t snap[kSnapEntries];
  static double* rsq = nullptr;
  if (!rsq) {
    rsq = new double[kTableDoubles];
    for (int i = 0; i < kTableDoubles; i++) pvq_fill_rsqrt_table(rsq, i);
  }
  simt_emu::run_warp([&](int lane) {
    gain[lane] = quantise_band_warp(lane, snap, rsq, out, x0, r0, n, q0, y, &it[lane], &mt[lane], &k[lane], beta, &sd[lane],
                                    is_keyframe, pli, qm, qm_inv, lambda);
  });
  if (getenv("DAALA_B200_EMU_SPLIT")) {
    // the same band through the three phases with the context parked in a record in between
    static int16_t vec[3 * kMaxN];
    static int32_t lanes[kCtxLaneWords * 16], uni[kCtxUniWords];
    static int16_t gsnap[kSnapEntries];
    const int vs = n > 32 ? 128 : 32;
    simt_emu::run_warp([&](int lane) {
      BandCtx B;
      if (n > 32) band_setup<2>(lane, B, x0, r0, n, q0, beta, is_keyframe, pli, qm, lambda, rsq);
      else band_setup<1>(lane, B, x0, r0, n, q0, beta, is_keyframe, pli, qm, lambda, rsq);
      band_ctx_store_setup(lane, B, n, vec, vs, lanes, uni);
    });
    simt_emu::run_warp([&](int lane) {
      BandCtx B;
      band_ctx_load_search(lane, B, n, vec, vs, lanes);
      if (n > 32) band_search<2>(lane, B, n, gsnap, vs, rsq);
      else band_search<1>(lane, B, n, gsnap, vs, rsq);
      band_ctx_store_search(lane, B, lanes);
    });
    simt_emu::run_warp([&](int lane) {
      BandCtx B;
      band_ctx_load_finish(lane, B, n, vec, vs, lanes, uni);
      gain[lane] = n > 32 ? band_finish<2>(lane, B, gsnap, vs, out, r0, n, q0, y, &it[lane], &mt[lane], &k[lane], beta,
                                           &sd[lane], is_keyframe, pli, qm_inv, lambda)
                          : band_finish<1>(lane, B, gsnap, vs, out, r0, n, q0, y, &it[lane], &mt[lane], &k[lane], beta,
                                           &sd[lane], is_keyframe, pli, qm_inv, lambda);
    });
  }
  for (int l = 1; l < 32; l++) {
    if (gain[l] != gain[0] || it[l] != it[0] || mt[l] != mt[0] || k[l] != k[0] || sd[l] != sd[0]) {
      fprintf(stderr, "emu_quantise_band: lanes disagree on scalar results\n");
      abort();
    }
  }
  *itheta = it[0];
  *max_theta = mt[0];
  *vk = k[0];
  *skip_term = sd[0];
  return gain[0];
}
