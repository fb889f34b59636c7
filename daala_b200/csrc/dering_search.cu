// Deringing level search of one frame (reference src/encode.c:2680-2811) -- SURVEY.md 8(f) rank 1, the
// caller of od_dering and od_compute_dist: for every 64x64 luma superblock the five filtered candidates
// (thresholds OD_DERING_GAIN_TABLE[gi] * quantizer^0.84182) and the unfiltered reconstruction are scored with
// the perceptual distortion against the source, and the level with the smallest dist + lambda * rate wins,
// rate being the cost of the level under an adaptive CDF whose context is the two neighbours' levels.
//
// Split the way the dependencies run:
//  * every filtered candidate reads the UNFILTERED plane (state->etmp), so the 6 x nsb distortions are
//    independent: 5 launches of the plane filter (csrc/dering_kernels.cu), 6 launches of a pack kernel
//    (superblock -> od_coeff pairs in raster order, the source through od_ref_buf_to_coeff,
//    src/state.c:1216) and of the distortion kernel (csrc/dist_kernels.cu), one copy of 6 x nsb doubles back;
//  * the decision itself is a raster scan whose CDF adapts after every superblock and whose context is
//    the decided levels above and to the left: a few thousand scalar steps per 4K frame, run on the host
//    (daala_b200_dering_decide, also exported on its own: it is the part the reference's decoder shares,
//    src/decode.c:1040-1053).
// daala_b200_dering_search is host-driven (allocates its scratch per call, one frame).  daala_b200_dering_search_enqueue
// is the batched, graph-capturable form, decision on the device included, that the keyframe engine (dering = 2) and the
// P-frame finishing pass (inter_finish = 2, real skip maps, uncoded superblocks left out, one context) run.  Both score
// the candidates with enqueue_candidates.  Parity: tests/test_host_logic.py (decision vs the reference's CDF functions),
// tests/test_gpu_dering.py (whole search vs the reference's loop, oracle/ref_hooks_encode.c).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "daala_b200.h"
#include "dering_search.h"

namespace daala_b200 {
namespace dering_search {

constexpr int kLevels = 6;             // OD_DERING_LEVELS, src/dering.h:41
constexpr int kContexts = 2 * kLevels - 1;
// OD_DERING_GAIN_TABLE, src/dering.c:50
const double kGain[kLevels] = {0, 0.5, 0.707, 1, 1.41, 2};

// One CTA per superblock of each frame, grid (nsb, F): cand <- the superblock of `plane` as od_coeff, orig
// (optional) <- the source superblock as (p - 128) << 4.
__global__ void __launch_bounds__(256) k_pack_sb_batch(const int16_t* __restrict__ plane, long long ppitch, int pstride,
                                                       const uint8_t* __restrict__ src, long long spitch, int sstride,
                                                       int nhsb, int32_t* __restrict__ cand, int32_t* __restrict__ orig) {
  const int sb = blockIdx.x, sbx = sb % nhsb, sby = sb / nhsb, f = blockIdx.y;
  const size_t slot = ((size_t)f * gridDim.x + sb) * 4096;
  const int16_t* p = plane + f * ppitch + (size_t)sby * 64 * pstride + sbx * 64;
  for (int idx = threadIdx.x; idx < 4096; idx += 256) cand[slot + idx] = p[(size_t)(idx >> 6) * pstride + (idx & 63)];
  if (orig) {
    const uint8_t* s = src + f * spitch + (size_t)sby * 64 * sstride + sbx * 64;
    for (int idx = threadIdx.x; idx < 4096; idx += 256)
      orig[slot + idx] = ((int)s[(size_t)(idx >> 6) * sstride + (idx & 63)] - 128) * 16;
  }
}

// The decision of daala_b200_dering_decide on the device, one thread per frame: every frame starts from the initial
// CDFs (the adaptation state is reset per frame, src/encode.c:3080).  Same operations as the host function, `coded`
// (nullable, [F][nsb]) and `is_keyframe` included; log() is the CUDA library's, so a decision could differ from the
// host's only where two scores agree to the last bits.
// fq (nullable): frame f's lambda is fq[f].dering_lambda.
__global__ void k_dering_decide(const double* __restrict__ dist, int nframes, int nhdr, int nvdr, double lambda,
                                const uint8_t* __restrict__ coded, int is_keyframe, uint8_t* __restrict__ levels,
                                const daala_b200_kf_frame_quant* __restrict__ fq, const uint8_t* __restrict__ frame_type) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nframes) return;
  if (frame_type) is_keyframe = frame_type[f];
  if (fq) lambda = fq[f].dering_lambda;
  const int nsb = nhdr * nvdr;
  const size_t per_level = (size_t)nframes * nsb;
  const double* d = dist + (size_t)f * nsb;
  const uint8_t* cf = coded ? coded + (size_t)f * nsb : nullptr;
  uint8_t* lv = levels + (size_t)f * nsb;
  unsigned short cdf[kContexts][kLevels];
  for (int c = 0; c < kContexts; c++)
    for (int j = 0; j < kLevels; j++) cdf[c][j] = (unsigned short)(32 * j + 32);
  for (int sby = 0; sby < nvdr; sby++) {
    for (int sbx = 0; sbx < nhdr; sbx++) {
      const int sb = sby * nhdr + sbx;
      if (cf && !cf[sb]) {   // every 4x4 block skipped: not searched, not signalled (src/encode.c:2727-2738)
        lv[sb] = 0;
        continue;
      }
      int left = 0, up = 0;
      if (is_keyframe) {
        if (sby > 0) left = up = lv[sb - nhdr];
        if (sbx > 0) {
          left = lv[sb - 1];
          if (sby == 0) up = left;
        }
      }
      unsigned short* m = cdf[up + left];
      const int total = m[kLevels - 1];
      int best = 0;
      double best_dist = 0;
      for (int gi = 0; gi < kLevels; gi++) {
        const int prev = gi ? m[gi - 1] : 0;
        const double prob = (m[gi] - prev) / (double)total;
        const double score = d[gi * per_level + sb] + lambda * -(M_LOG2E * log(prob));
        if (gi == 0 || score < best_dist) {
          best_dist = score;
          best = gi;
        }
      }
      lv[sb] = (uint8_t)best;
      if (m[kLevels - 1] + 128 > 32767)
        for (int i = 0; i < kLevels; i++) m[i] = (unsigned short)((m[i] >> 1) + i + 1);
      for (int i = best; i < kLevels; i++) m[i] = (unsigned short)(m[i] + 128);
    }
  }
}

// Per-frame thresholds (the engine's search): thr[gi - 1][f * nsb + sb] = frame_tbl[f][0][gi] for the five filtered
// candidates, the per-superblock threshold maps their od_dering passes read.
__global__ void k_cand_thresholds(const int32_t* __restrict__ frame_tbl, int n, int nsb, int32_t* __restrict__ thr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t* t = frame_tbl + (size_t)(i / nsb) * 12;
  for (int gi = 1; gi < kLevels; gi++) thr[(size_t)(gi - 1) * n + i] = t[gi];
}

// od_encode_cdf_cost, src/generic_encoder.c:198
inline double cdf_cost(int val, const uint16_t* cdf) {
  const int total = cdf[kLevels - 1];
  const int prev = val ? cdf[val - 1] : 0;
  const double prob = (cdf[val] - prev) / (double)total;
  return -(M_LOG2E * log(prob));
}

// the model update of od_encode_cdf_adapt, src/generic_encoder.c:74-85
inline void cdf_adapt(int val, uint16_t* cdf, int increment) {
  if (cdf[kLevels - 1] + increment > 32767)
    for (int i = 0; i < kLevels; i++) cdf[i] = (uint16_t)((cdf[i] >> 1) + i + 1);
  for (int i = val; i < kLevels; i++) cdf[i] = (uint16_t)(cdf[i] + increment);
}

}  // namespace dering_search
}  // namespace daala_b200

using namespace daala_b200::dering_search;

extern "C" void daala_b200_dering_cdf_init(uint16_t* cdf, int* increment) {
  // src/state.c:573-574: increment 128, OD_CDFS_INIT(dering_cdf, increment >> 2)
  for (int c = 0; c < kContexts; c++)
    for (int j = 0; j < kLevels; j++) cdf[c * kLevels + j] = (uint16_t)(32 * j + 32);
  if (increment) *increment = 128;
}

extern "C" int daala_b200_dering_decide(const double* dist, int nhdr, int nvdr, int is_keyframe, double dering_lambda,
                                        const uint8_t* coded, uint16_t* cdf, int increment, uint8_t* levels) {
  if (!dist || !cdf || !levels || nhdr < 1 || nvdr < 1) return -1;
  const int nsb = nhdr * nvdr;
  for (int sby = 0; sby < nvdr; sby++) {
    for (int sbx = 0; sbx < nhdr; sbx++) {
      const int sb = sby * nhdr + sbx;
      levels[sb] = 0;
      if (coded && !coded[sb]) continue;     // every 4x4 block skipped: not signalled (src/encode.c:2727-2738)
      int c = 0;
      if (is_keyframe) {
        int left = 0, up = 0;
        if (sby > 0) left = up = levels[sb - nhdr];
        if (sbx > 0) {
          left = levels[sb - 1];
          if (sby == 0) up = left;
        }
        c = up + left;
      }
      uint16_t* m = cdf + c * kLevels;
      int best = 0;
      double best_dist = dist[sb] + dering_lambda * cdf_cost(0, m);
      for (int gi = 1; gi < kLevels; gi++) {
        const double d = dist[(size_t)gi * nsb + sb] + dering_lambda * cdf_cost(gi, m);
        if (d < best_dist) {
          best_dist = d;
          best = gi;
        }
      }
      levels[sb] = (uint8_t)best;
      cdf_adapt(best, m, increment);
    }
  }
  return 0;
}


void daala_b200_dering_threshold_table(int quantizer, int tbl[2][6]) {
  const double base = pow((double)quantizer, 0.84182);   // src/encode.c:2694
  for (int g = 0; g < kLevels; g++) {
    tbl[0][g] = (int)(kGain[g] * base);
    tbl[1][g] = (int)(kGain[g] * base * 0.6);
  }
}

// The distortion of every candidate of every superblock of the batch, b->dist[gi][f * nsb + sb]: the unfiltered plane
// (gi = 0) and the five filtered ones, each packed next to the source and measured.  The first filter pass finds the
// directions and stores them with the variance (dir_format 1); the later passes filter the same plane and re-use them.
static int enqueue_candidates(const daala_b200_dering_search_batch* b, cudaStream_t st) {
  const int nsb = b->nhsb * b->nvsb, F = b->nframes;
  const int w = b->nhsb * 64, h = b->nvsb * 64;
  const long long filt_pitch = (long long)w * h;
  if (b->frame_tbl) {
    k_cand_thresholds<<<(F * nsb + 255) / 256, 256, 0, st>>>(b->frame_tbl, F * nsb, nsb, b->cand_thr);
    cudaError_t e = cudaGetLastError();
    if (e) return (int)e;
  }
  for (int gi = 0; gi < kLevels; gi++) {
    const int16_t* plane = b->etmp;
    long long ppitch = b->etmp_pitch;
    int pstride = b->etmp_stride;
    if (gi) {
      daala_b200_dering_params dp;
      memset(&dp, 0, sizeof(dp));
      dp.y = b->filt;
      dp.x = b->etmp;
      dp.dir = b->dir;
      dp.bskip = b->bskip;
      dp.ystride = w;
      dp.xstride = b->etmp_stride;
      dp.dir_stride = b->nhsb * 8;
      dp.skip_stride = b->skip_stride;
      dp.nhsb = b->nhsb;
      dp.nvsb = b->nvsb;
      dp.threshold = b->threshold[gi];
      dp.sb_threshold = b->frame_tbl ? b->cand_thr + (size_t)(gi - 1) * F * nsb : nullptr;
      dp.overlap = 1;
      dp.coeff_shift = 4;
      dp.dir_format = gi == 1 ? 1 : 2;
      const int r = daala_b200_dering_plane_frames(&dp, F, filt_pitch, b->etmp_pitch, (long long)nsb * 64,
                                                   b->frame_tbl ? nsb : 0, b->skip_pitch, nullptr, st);
      if (r) return r;
      plane = b->filt;
      ppitch = filt_pitch;
      pstride = w;
    }
    k_pack_sb_batch<<<dim3(nsb, F), 256, 0, st>>>(plane, ppitch, pstride, b->src, b->src_pitch, b->src_stride, b->nhsb,
                                                  b->cand, gi == 0 ? b->orig : nullptr);
    cudaError_t e = cudaGetLastError();
    if (e) return (int)e;
    const int r = daala_b200_compute_dist_frames(b->orig, b->cand, F * nsb, 64, b->qm_is_flat, b->use_activity_masking,
                                                 b->coded_quantizer, b->fq, nsb, b->dist + (size_t)gi * F * nsb, st);
    if (r) return r;
  }
  return 0;
}

extern "C" int daala_b200_dering_search(const daala_b200_dering_search_params* p, uint16_t* cdf, int increment,
                                        uint8_t* levels, double* dist_out, void* stream_) {
  if (!p || !p->etmp || !p->src || !cdf || !levels || p->nhsb < 1 || p->nvsb < 1) return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream_;
  const int nhsb = p->nhsb, nvsb = p->nvsb, nsb = nhsb * nvsb;
  const int w = nhsb * 64, h = nvsb * 64;
  const int skip_stride = p->bskip ? p->skip_stride : nhsb * 16;
  daala_b200_dering_search_batch b;
  memset(&b, 0, sizeof(b));
  uint8_t* zskip = nullptr;
  cudaError_t e = cudaSuccess;
  auto done = [&](cudaError_t err) {
    cudaFree(b.filt); cudaFree(b.orig); cudaFree(b.cand); cudaFree(b.dir); cudaFree(zskip); cudaFree(b.dist);
    return (int)err;
  };
  if ((e = cudaMalloc(&b.filt, sizeof(int16_t) * (size_t)w * h))) return done(e);
  if ((e = cudaMalloc(&b.orig, sizeof(int32_t) * (size_t)nsb * 4096))) return done(e);
  if ((e = cudaMalloc(&b.cand, sizeof(int32_t) * (size_t)nsb * 4096))) return done(e);
  if ((e = cudaMalloc(&b.dir, sizeof(int32_t) * (size_t)nsb * 64))) return done(e);
  if ((e = cudaMalloc(&b.dist, sizeof(double) * (size_t)kLevels * nsb))) return done(e);
  if (!p->bskip) {
    if ((e = cudaMalloc(&zskip, (size_t)nsb * 256))) return done(e);
    if ((e = cudaMemsetAsync(zskip, 0, (size_t)nsb * 256, st))) return done(e);
  }
  b.etmp = p->etmp;
  b.src = p->src;
  b.etmp_stride = p->etmp_stride;
  b.src_stride = p->src_stride;
  b.nframes = 1;
  b.nhsb = nhsb;
  b.nvsb = nvsb;
  int tbl[2][6];
  daala_b200_dering_threshold_table(p->quantizer, tbl);
  memcpy(b.threshold, tbl[0], sizeof(b.threshold));
  b.coded_quantizer = p->coded_quantizer;
  b.qm_is_flat = p->qm_is_flat;
  b.use_activity_masking = p->use_activity_masking;
  b.bskip = p->bskip ? p->bskip : zskip;
  b.skip_stride = skip_stride;
  const int rc = enqueue_candidates(&b, st);
  if (rc) return done((cudaError_t)rc);
  std::vector<double> hdist((size_t)kLevels * nsb);
  if ((e = cudaMemcpyAsync(hdist.data(), b.dist, sizeof(double) * hdist.size(), cudaMemcpyDeviceToHost, st))) return done(e);
  // superblocks whose 4x4 blocks are all skipped are neither searched nor signalled
  std::vector<uint8_t> coded;
  if (p->bskip) {
    std::vector<uint8_t> hs((size_t)nvsb * 16 * skip_stride);
    if ((e = cudaMemcpyAsync(hs.data(), p->bskip, hs.size(), cudaMemcpyDeviceToHost, st))) return done(e);
    if ((e = cudaStreamSynchronize(st))) return done(e);
    coded.assign(nsb, 0);
    for (int sb = 0; sb < nsb; sb++)
      for (int j = 0; j < 16; j++)
        for (int i = 0; i < 16; i++)
          if (!hs[(size_t)((sb / nhsb) * 16 + j) * skip_stride + (sb % nhsb) * 16 + i]) coded[sb] = 1;
  }
  if ((e = cudaStreamSynchronize(st))) return done(e);
  if (dist_out) memcpy(dist_out, hdist.data(), sizeof(double) * hdist.size());
  const int r = daala_b200_dering_decide(hdist.data(), nhsb, nvsb, p->is_keyframe, p->dering_lambda,
                                         p->bskip ? coded.data() : nullptr, cdf, increment, levels);
  done(cudaSuccess);
  return r;
}

extern "C" int daala_b200_dering_search_enqueue(const daala_b200_dering_search_batch* b, void* stream_) {
  if (!b || !b->etmp || !b->src || !b->filt || !b->orig || !b->cand || !b->dir || !b->bskip || !b->dist || !b->levels ||
      b->nframes < 1 || b->nhsb < 1 || b->nvsb < 1 || b->skip_stride < b->nhsb * 16 || b->skip_pitch < 0)
    return (int)cudaErrorInvalidValue;
  cudaStream_t st = (cudaStream_t)stream_;
  const int r = enqueue_candidates(b, st);
  if (r) return r;
  k_dering_decide<<<(b->nframes + 31) / 32, 32, 0, st>>>(b->dist, b->nframes, b->nhsb, b->nvsb, b->dering_lambda,
                                                         b->coded, b->is_keyframe, b->levels, b->fq, b->frame_type);
  return (int)cudaGetLastError();
}
