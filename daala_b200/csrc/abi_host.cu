// C-ABI layer of libdaala_b200.so.
//
//  * Section A of include/daala_b200.h: the reference's od_* symbols with HOST
//    pointers.  Each call packs its operand into pinned staging memory, runs
//    the matching kernel on a private stream and unpacks the result --
//    synchronous and bit-exact, like the C functions they replace
//    (reference: src/dct.c, src/filter.c).
//  * Section B: thin wrappers that forward device pointers to the launchers
//    in frame_transform.cu.
//
// No CPU fallback: a missing/unusable GPU is fatal for section A (the
// reference prototypes return void) and an error code for section B.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <stddef.h>

#include <mutex>

#include "daala_b200.h"
#include "frame_transform.h"

extern "C" {
int daala_b200_launch_forward(const FrameXformParams* prm, int nplanes, cudaStream_t stream);
int daala_b200_launch_forward_no_tma(const FrameXformParams* prm, int nplanes, cudaStream_t stream);
int daala_b200_launch_inverse(const FrameXformParams* prm, int nplanes, cudaStream_t stream);
int daala_b200_launch_inverse_lapped_only(const FrameXformParams* prm, int nplanes, cudaStream_t stream);
int daala_b200_launch_sb_postfilter_store(const FrameXformParams* prm, int nplanes, cudaStream_t stream);
int daala_b200_launch_plane_sb_filter(int32_t* c, int stride, int nhsb, int nvsb, int xdec, int ydec,
                                      int post, cudaStream_t stream);
int daala_b200_launch_block_transform(int32_t* blocks, int count, int ln, int mode, cudaStream_t stream);
int daala_b200_launch_filter4(int32_t* v, long count, int post, cudaStream_t stream);
int daala_b200_launch_haar_blocks(int32_t* blocks, int count, int ln, int inverse, cudaStream_t stream);
int daala_b200_pvq_helper_launch(void* buf, int op, void* stream);
int daala_b200_pvq_helper_bytes(void);
int daala_b200_launch_lapfilter(int32_t* v, long count, int n, int post, cudaStream_t stream);
int daala_b200_launch_split_filter(int32_t* blocks, int count, int n, int post, int hfilter, int vfilter,
                                   cudaStream_t stream);
}

namespace {

[[noreturn]] void fatal(const char* what, cudaError_t err) {
  fprintf(stderr, "libdaala_b200: fatal: %s: %s (no CPU fallback exists)\n", what,
          cudaGetErrorString(err));
  abort();
}

#define CK(call)                                    \
  do {                                              \
    cudaError_t e_ = (call);                        \
    if (e_ != cudaSuccess) fatal(#call, e_);        \
  } while (0)

// Per-process staging context for the host-pointer entry points.
struct HostCtx {
  cudaStream_t stream = nullptr;
  void* pinned = nullptr;
  void* dev = nullptr;
  size_t cap = 0;
  std::mutex mu;

  void ensure(size_t bytes) {
    if (!stream) {
      int n = 0;
      cudaError_t e = cudaGetDeviceCount(&n);
      if (e != cudaSuccess || n == 0) fatal("cudaGetDeviceCount", e == cudaSuccess ? cudaErrorNoDevice : e);
      CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    }
    if (bytes > cap) {
      size_t ncap = cap ? cap : (size_t)1 << 20;
      while (ncap < bytes) ncap <<= 1;
      if (pinned) CK(cudaFreeHost(pinned));
      if (dev) CK(cudaFree(dev));
      CK(cudaMallocHost(&pinned, ncap));
      CK(cudaMalloc(&dev, ncap));
      cap = ncap;
    }
  }
  void h2d(size_t bytes) { CK(cudaMemcpyAsync(dev, pinned, bytes, cudaMemcpyHostToDevice, stream)); }
  void d2h(size_t bytes) {
    CK(cudaMemcpyAsync(pinned, dev, bytes, cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
  }
};

HostCtx& ctx() {
  static HostCtx c;
  return c;
}

void check_launch(int rc, const char* what) {
  if (rc != 0) fatal(what, (cudaError_t)rc);
}

void dct1d(int ln, bool inverse, od_coeff* out, int out_stride, const od_coeff* in, int in_stride) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g(c.mu);
  const int n = 1 << ln;
  c.ensure(sizeof(od_coeff) * n * n);
  od_coeff* p = (od_coeff*)c.pinned;
  // The 1-D kernel transforms rows of a packed n x n block; only row 0 is used.
  memset(p, 0, sizeof(od_coeff) * n * n);
  for (int i = 0; i < n; i++) p[i] = in[i * in_stride];
  c.h2d(sizeof(od_coeff) * n * n);
  check_launch(daala_b200_launch_block_transform((int32_t*)c.dev, 1, ln, inverse ? 3 : 2, c.stream),
               "block_transform(1d)");
  c.d2h(sizeof(od_coeff) * n);
  for (int i = 0; i < n; i++) out[i * out_stride] = p[i];
}

void haar2d(int ln, bool inverse, od_coeff* out, int out_stride, const od_coeff* in, int in_stride) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g(c.mu);
  const int n = 1 << ln;
  c.ensure(sizeof(od_coeff) * n * n);
  od_coeff* p = (od_coeff*)c.pinned;
  for (int i = 0; i < n; i++) memcpy(p + i * n, in + (size_t)i * in_stride, sizeof(od_coeff) * n);
  c.h2d(sizeof(od_coeff) * n * n);
  check_launch(daala_b200_launch_haar_blocks((int32_t*)c.dev, 1, ln, inverse ? 1 : 0, c.stream), "haar_blocks");
  c.d2h(sizeof(od_coeff) * n * n);
  for (int i = 0; i < n; i++) memcpy(out + (size_t)i * out_stride, p + i * n, sizeof(od_coeff) * n);
}

void dct2d(int ln, bool inverse, od_coeff* out, int out_stride, const od_coeff* in, int in_stride) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g(c.mu);
  const int n = 1 << ln;
  c.ensure(sizeof(od_coeff) * n * n);
  od_coeff* p = (od_coeff*)c.pinned;
  for (int i = 0; i < n; i++) memcpy(p + i * n, in + (size_t)i * in_stride, sizeof(od_coeff) * n);
  c.h2d(sizeof(od_coeff) * n * n);
  check_launch(daala_b200_launch_block_transform((int32_t*)c.dev, 1, ln, inverse ? 1 : 0, c.stream),
               "block_transform(2d)");
  c.d2h(sizeof(od_coeff) * n * n);
  for (int i = 0; i < n; i++) memcpy(out + (size_t)i * out_stride, p + i * n, sizeof(od_coeff) * n);
}

void filter4(bool post, od_coeff* out, const od_coeff* in) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g(c.mu);
  c.ensure(sizeof(od_coeff) * 4);
  memcpy(c.pinned, in, sizeof(od_coeff) * 4);
  c.h2d(sizeof(od_coeff) * 4);
  check_launch(daala_b200_launch_filter4((int32_t*)c.dev, 1, post, c.stream), "filter4");
  c.d2h(sizeof(od_coeff) * 4);
  memcpy(out, c.pinned, sizeof(od_coeff) * 4);
}

void lapfilter_n(int n, bool post, od_coeff* out, const od_coeff* in) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g(c.mu);
  c.ensure(sizeof(od_coeff) * n);
  memcpy(c.pinned, in, sizeof(od_coeff) * n);
  c.h2d(sizeof(od_coeff) * n);
  check_launch(daala_b200_launch_lapfilter((int32_t*)c.dev, 1, n, post, c.stream), "lapfilter");
  c.d2h(sizeof(od_coeff) * n);
  memcpy(out, c.pinned, sizeof(od_coeff) * n);
}

void split_filter(bool post, od_coeff* c0, int stride, int bs, int hfilter, int vfilter) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g(c.mu);
  const int n = 4 << bs;
  c.ensure(sizeof(od_coeff) * n * n);
  od_coeff* p = (od_coeff*)c.pinned;
  for (int i = 0; i < n; i++) memcpy(p + i * n, c0 + (size_t)i * stride, sizeof(od_coeff) * n);
  c.h2d(sizeof(od_coeff) * n * n);
  check_launch(daala_b200_launch_split_filter((int32_t*)c.dev, 1, n, post, hfilter, vfilter, c.stream),
               "split_filter");
  c.d2h(sizeof(od_coeff) * n * n);
  for (int i = 0; i < n; i++) memcpy(c0 + (size_t)i * stride, p + i * n, sizeof(od_coeff) * n);
}

void plane_sb_filter(bool post, od_coeff* c0, int stride, int nhsb, int nvsb, int xdec, int ydec) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g(c.mu);
  const int w = (nhsb * 64) >> xdec, h = (nvsb * 64) >> ydec;
  const size_t bytes = sizeof(od_coeff) * (size_t)w * h;
  c.ensure(bytes);
  od_coeff* p = (od_coeff*)c.pinned;
  for (int i = 0; i < h; i++) memcpy(p + (size_t)i * w, c0 + (size_t)i * stride, sizeof(od_coeff) * w);
  c.h2d(bytes);
  check_launch(daala_b200_launch_plane_sb_filter((int32_t*)c.dev, w, nhsb, nvsb, xdec, ydec, post, c.stream),
               "plane_sb_filter");
  c.d2h(bytes);
  for (int i = 0; i < h; i++) memcpy(c0 + (size_t)i * stride, p + (size_t)i * w, sizeof(od_coeff) * w);
}

}  // namespace

extern "C" {

// ---- Section A ------------------------------------------------------------
#define DAALA_B200_DCT(N, LN)                                                                     \
  void od_bin_fdct##N(od_coeff* y, const od_coeff* x, int xstride) { dct1d(LN, false, y, 1, x, xstride); } \
  void od_bin_idct##N(od_coeff* x, int xstride, const od_coeff* y) { dct1d(LN, true, x, xstride, y, 1); }  \
  void od_bin_fdct##N##x##N(od_coeff* y, int ystride, const od_coeff* x, int xstride) {          \
    dct2d(LN, false, y, ystride, x, xstride);                                                    \
  }                                                                                              \
  void od_bin_idct##N##x##N(od_coeff* x, int xstride, const od_coeff* y, int ystride) {          \
    dct2d(LN, true, x, xstride, y, ystride);                                                     \
  }
DAALA_B200_DCT(4, 2)
DAALA_B200_DCT(8, 3)
DAALA_B200_DCT(16, 4)
DAALA_B200_DCT(32, 5)
DAALA_B200_DCT(64, 6)

/* src/dct.c:4822 / :4861 */
void od_haar(od_coeff* y, int ystride, const od_coeff* x, int xstride, int ln) { haar2d(ln, false, y, ystride, x, xstride); }
void od_haar_inv(od_coeff* x, int xstride, const od_coeff* y, int ystride, int ln) { haar2d(ln, true, x, xstride, y, ystride); }

const od_dct_func_2d OD_FDCT_2D_CUDA[6] = {od_bin_fdct4x4,   od_bin_fdct8x8,   od_bin_fdct16x16,
                                           od_bin_fdct32x32, od_bin_fdct64x64, nullptr};
const od_dct_func_2d OD_IDCT_2D_CUDA[6] = {od_bin_idct4x4,   od_bin_idct8x8,   od_bin_idct16x16,
                                           od_bin_idct32x32, od_bin_idct64x64, nullptr};

void od_pre_filter4(od_coeff _y[4], const od_coeff _x[4]) { filter4(false, _y, _x); }
void od_post_filter4(od_coeff _x[4], const od_coeff _y[4]) { filter4(true, _x, _y); }

void od_pre_filter8(od_coeff _y[8], const od_coeff _x[8]) { lapfilter_n(8, false, _y, _x); }
void od_post_filter8(od_coeff _x[8], const od_coeff _y[8]) { lapfilter_n(8, true, _x, _y); }
void od_pre_filter16(od_coeff _y[16], const od_coeff _x[16]) { lapfilter_n(16, false, _y, _x); }
void od_post_filter16(od_coeff _x[16], const od_coeff _y[16]) { lapfilter_n(16, true, _x, _y); }
void od_pre_filter32(od_coeff _y[32], const od_coeff _x[32]) { lapfilter_n(32, false, _y, _x); }
void od_post_filter32(od_coeff _x[32], const od_coeff _y[32]) { lapfilter_n(32, true, _x, _y); }

// The reference's own table names (src/dct.c:54-84), so that linking this library INSTEAD of the
// reference's dct.o / filter.o resolves OD_COPY(state->opt_vtbl.fdct_2d, OD_FDCT_2D_C, ...) of
// od_state_opt_vtbl_init_c (src/state.c:341-342) and the dcttest / tools users of the 1-D tables.
const od_dct_func_2d OD_FDCT_2D_C[6] = {od_bin_fdct4x4,   od_bin_fdct8x8,   od_bin_fdct16x16,
                                        od_bin_fdct32x32, od_bin_fdct64x64, nullptr};
const od_dct_func_2d OD_IDCT_2D_C[6] = {od_bin_idct4x4,   od_bin_idct8x8,   od_bin_idct16x16,
                                        od_bin_idct32x32, od_bin_idct64x64, nullptr};
const od_fdct_func_1d OD_FDCT_1D[6] = {od_bin_fdct4, od_bin_fdct8, od_bin_fdct16, od_bin_fdct32, od_bin_fdct64, nullptr};
const od_idct_func_1d OD_IDCT_1D[6] = {od_bin_idct4, od_bin_idct8, od_bin_idct16, od_bin_idct32, od_bin_idct64, nullptr};

// reference: OD_PRE_FILTER / OD_POST_FILTER, src/filter.c:115-127
const od_filter_func OD_PRE_FILTER_CUDA[4] = {od_pre_filter4, od_pre_filter8, od_pre_filter16, od_pre_filter32};
const od_filter_func OD_POST_FILTER_CUDA[4] = {od_post_filter4, od_post_filter8, od_post_filter16, od_post_filter32};

// the reference's names (OD_NBSIZES = 5 entries, the last one NULL) and the 4-point filter's parameters
const od_filter_func OD_PRE_FILTER[5] = {od_pre_filter4, od_pre_filter8, od_pre_filter16, od_pre_filter32, nullptr};
const od_filter_func OD_POST_FILTER[5] = {od_post_filter4, od_post_filter8, od_post_filter16, od_post_filter32, nullptr};
const int OD_FILTER_PARAMS4[4] = {85, 75, -15, 33};   // src/filter.c:137-146

int daala_b200_lapfilter(int32_t* v, long count, int n, int post, void* stream) {
  return daala_b200_launch_lapfilter(v, count, n, post, (cudaStream_t)stream);
}

void od_prefilter_split(od_coeff* c0, int stride, int bs, int f, int hfilter, int vfilter) {
  (void)f;  // OD_FILT_SIZE() == 0: always the 4-point filter (src/filter.h:77)
  split_filter(false, c0, stride, bs, hfilter, vfilter);
}

void od_postfilter_split(od_coeff* c0, int stride, int bs, int f, int q, unsigned char* skip,
                         int skip_stride, int hfilter, int vfilter) {
  (void)f; (void)q; (void)skip; (void)skip_stride;  // deblocking branch is compiled out upstream
  split_filter(true, c0, stride, bs, hfilter, vfilter);
}

void od_apply_prefilter_frame_sbs(od_coeff* c, int stride, int nhsb, int nvsb, int xdec, int ydec) {
  plane_sb_filter(false, c, stride, nhsb, nvsb, xdec, ydec);
}

void od_apply_postfilter_frame_sbs(od_coeff* c, int stride, int nhsb, int nvsb, int xdec, int ydec,
                                   int q, unsigned char* skip, int skip_stride) {
  (void)q; (void)skip; (void)skip_stride;
  plane_sb_filter(true, c, stride, nhsb, nvsb, xdec, ydec);
}

// Motion compensation / block matching with host pointers.
void od_mc_predict1fmv8_cuda(void* state, unsigned char* dst, const unsigned char* src, int systride,
                             int32_t mvx, int32_t mvy, int log_xblk_sz, int log_yblk_sz) {
  (void)state;
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g(c.mu);
  const int nx = 1 << log_xblk_sz, ny = 1 << log_yblk_sz;
  const int W = nx + 5, H = ny + 5;  // 2 px left/top, 3 px right/bottom (OD_SUBPEL_*_APRON_SZ)
  const size_t win = (size_t)W * H, job_off = (win + 15) & ~(size_t)15, out_off = job_off + 16;
  c.ensure(out_off + (size_t)nx * ny);
  unsigned char* p = (unsigned char*)c.pinned;
  // stage only what od_mc_predict1fmv8_c reads (src/mc.c:94): the 2 + 3 sample apron exists in a direction only
  // when the vector has a fractional part there -- an integer vector touches the block alone, and the caller's
  // buffer may end right after it
  const unsigned char* s0 = src + ((mvx >> 3) - 2) + (ptrdiff_t)((mvy >> 3) - 2) * systride;
  const int c_lo = (mvx & 7) ? 0 : 2, c_hi = (mvx & 7) ? W : 2 + nx;
  const int r_lo = (mvy & 7) ? 0 : 2, r_hi = (mvy & 7) ? H : 2 + ny;
  memset(p, 0, win);
  for (int r = r_lo; r < r_hi; r++) memcpy(p + (size_t)r * W + c_lo, s0 + (ptrdiff_t)r * systride + c_lo, c_hi - c_lo);
  daala_b200_match_job job;
  memset(&job, 0, sizeof(job));
  job.mvx = mvx & 7; job.mvy = mvy & 7; job.x0 = 2; job.y0 = 2; job.log_blk = (uint8_t)log_xblk_sz;
  memcpy(p + job_off, &job, sizeof(job));
  c.h2d(out_off);
  unsigned char* d = (unsigned char*)c.dev;
  check_launch(daala_b200_mc_predict1fmv_batch(d, W, d + out_off, nx * ny, (const daala_b200_match_job*)(d + job_off),
                                               1, log_yblk_sz, c.stream), "mc_predict1fmv");
  CK(cudaMemcpyAsync(p + out_off, d + out_off, (size_t)nx * ny, cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  memcpy(dst, p + out_off, (size_t)nx * ny);
}

static void blend_host(unsigned char* dst, int dystride, const unsigned char* src[4], int oc, int s, int lx, int ly) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g(c.mu);
  const int nx = 1 << lx, ny = 1 << ly, n2 = nx * ny;
  c.ensure((size_t)5 * n2);
  unsigned char* p = (unsigned char*)c.pinned;
  for (int k = 0; k < 4; k++) memcpy(p + (size_t)k * n2, src[k], n2);
  c.h2d((size_t)4 * n2);
  unsigned char* d = (unsigned char*)c.dev;
  check_launch(daala_b200_mc_blend_packed(d, n2, d + (size_t)4 * n2, nx, oc, s, lx, ly, c.stream), "mc_blend");
  CK(cudaMemcpyAsync(p + (size_t)4 * n2, d + (size_t)4 * n2, n2, cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  for (int j = 0; j < ny; j++) memcpy(dst + (size_t)j * dystride, p + (size_t)4 * n2 + (size_t)j * nx, nx);
}

void od_mc_blend_full8_cuda(unsigned char* dst, int dystride, const unsigned char* src[4], int log_xblk_sz,
                            int log_yblk_sz) {
  blend_host(dst, dystride, src, 0, 3, log_xblk_sz, log_yblk_sz);
}

void od_mc_blend_full_split8_cuda(unsigned char* dst, int dystride, const unsigned char* src[4], int c, int s,
                                  int log_xblk_sz, int log_yblk_sz) {
  blend_host(dst, dystride, src, c, s, log_xblk_sz, log_yblk_sz);
}

static int32_t match_host(int ln, int use_satd, const unsigned char* src, int systride, const unsigned char* ref,
                          int dystride) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g(c.mu);
  const int n = 1 << ln, n2 = n * n;
  const size_t job_off = (size_t)2 * n2, res_off = job_off + 16;
  c.ensure(res_off + 16);
  unsigned char* p = (unsigned char*)c.pinned;
  for (int j = 0; j < n; j++) {
    memcpy(p + (size_t)j * n, src + (ptrdiff_t)j * systride, n);
    memcpy(p + n2 + (size_t)j * n, ref + (ptrdiff_t)j * dystride, n);
  }
  daala_b200_match_job job;
  memset(&job, 0, sizeof(job));
  job.log_blk = (uint8_t)ln;
  memcpy(p + job_off, &job, sizeof(job));
  c.h2d(res_off);
  unsigned char* d = (unsigned char*)c.dev;
  check_launch(daala_b200_mc_match_candidates(d, n, d + n2, n, (const daala_b200_match_job*)(d + job_off), 1,
                                              use_satd, (int32_t*)(d + res_off), c.stream), "mc_match");
  CK(cudaMemcpyAsync(p + res_off, d + res_off, 4, cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  int32_t r;
  memcpy(&r, p + res_off, 4);
  return r;
}

#define DAALA_B200_MATCH(N, LN)                                                                            \
  int32_t od_mc_compute_sad8_##N##x##N##_cuda(const unsigned char* src, int systride, const unsigned char* ref, \
                                              int dystride) {                                             \
    return match_host(LN, 0, src, systride, ref, dystride);                                               \
  }                                                                                                       \
  int32_t od_mc_compute_satd8_##N##x##N##_cuda(const unsigned char* src, int systride, const unsigned char* ref, \
                                               int dystride) {                                            \
    return match_host(LN, 1, src, systride, ref, dystride);                                               \
  }
DAALA_B200_MATCH(4, 2)
DAALA_B200_MATCH(8, 3)
DAALA_B200_MATCH(16, 4)
DAALA_B200_MATCH(32, 5)
DAALA_B200_MATCH(64, 6)

// Scalar PVQ helpers with host pointers (src/pvq.h:148-175, src/pvq_encoder.h:46).
struct PvqHelperBuf {
  int32_t args[16];
  int16_t a16[2][128];
  int32_t a32[2][128];
  int16_t qmi[128];
  double dargs[2];
};

static PvqHelperBuf* helper_begin(HostCtx& c) {
  if ((size_t)daala_b200_pvq_helper_bytes() != sizeof(PvqHelperBuf)) fatal("pvq helper layout", cudaErrorInvalidValue);
  c.ensure(sizeof(PvqHelperBuf));
  PvqHelperBuf* b = (PvqHelperBuf*)c.pinned;
  memset(b, 0, sizeof(*b));
  return b;
}

static void helper_run(HostCtx& c, int op) {
  c.h2d(sizeof(PvqHelperBuf));
  check_launch(daala_b200_pvq_helper_launch(c.dev, op, c.stream), "pvq_helper");
  c.d2h(sizeof(PvqHelperBuf));
}

#define HELPER_SCALAR(OP, ...)                      \
  HostCtx& c = ctx();                               \
  std::lock_guard<std::mutex> g_(c.mu);             \
  PvqHelperBuf* b = helper_begin(c);                \
  { int32_t v_[] = {__VA_ARGS__}; memcpy(b->args, v_, sizeof(v_)); } \
  helper_run(c, OP);

int16_t od_pvq_sin(int32_t x) { HELPER_SCALAR(0, x) return (int16_t)b->args[15]; }
int16_t od_pvq_cos(int32_t x) { HELPER_SCALAR(1, x) return (int16_t)b->args[15]; }
int32_t od_gain_expand(int32_t cg, int q0, int16_t beta) { HELPER_SCALAR(6, cg, q0, beta) return b->args[15]; }
int od_pvq_compute_max_theta(int32_t qcg, int16_t beta) { HELPER_SCALAR(8, qcg, beta) return b->args[15]; }
int32_t od_pvq_compute_theta(int t, int max_theta) { HELPER_SCALAR(9, t, max_theta) return b->args[15]; }
int od_pvq_compute_k(int32_t qcg, int itheta, int32_t theta, int noref, int n, int16_t beta, int nodesync) {
  (void)theta; (void)nodesync;  // robust-stream rule only (OD_ROBUST_STREAM, src/internal.h:118)
  HELPER_SCALAR(10, qcg, itheta, noref, n, beta)
  return b->args[15];
}

int od_vector_log_mag(const od_coeff* x, int n) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g_(c.mu);
  PvqHelperBuf* b = helper_begin(c);
  b->args[0] = n;
  memcpy(b->a32[0], x, sizeof(od_coeff) * n);
  helper_run(c, 2);
  return b->args[15];
}

int od_compute_householder(int16_t* r, int n, int32_t gr, int* sign, int shift) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g_(c.mu);
  PvqHelperBuf* b = helper_begin(c);
  b->args[0] = n; b->args[1] = gr; b->args[2] = shift;
  memcpy(b->a16[0], r, sizeof(int16_t) * n);
  helper_run(c, 3);
  memcpy(r, b->a16[0], sizeof(int16_t) * n);
  *sign = b->args[14];
  return b->args[15];
}

void od_apply_householder(int16_t* out, const int16_t* x, const int16_t* r, int n) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g_(c.mu);
  PvqHelperBuf* b = helper_begin(c);
  b->args[0] = n;
  memcpy(b->a16[0], r, sizeof(int16_t) * n);
  memcpy(b->a16[1], x, sizeof(int16_t) * n);
  helper_run(c, 4);
  memcpy(out, b->a16[1], sizeof(int16_t) * n);
}

void od_pvq_synthesis_partial(od_coeff* xcoeff, const od_coeff* ypulse, const int16_t* r, int n, int noref,
                              int32_t g, int32_t theta, int m, int s, const int16_t* qm_inv) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g_(c.mu);
  PvqHelperBuf* b = helper_begin(c);
  b->args[0] = n; b->args[1] = noref; b->args[2] = g; b->args[3] = theta; b->args[4] = m; b->args[5] = s;
  memcpy(b->a32[0], ypulse, sizeof(od_coeff) * (n - !noref));
  if (r) memcpy(b->a16[0], r, sizeof(int16_t) * n);
  memcpy(b->qmi, qm_inv, sizeof(int16_t) * n);
  helper_run(c, 5);
  memcpy(xcoeff, b->a32[1], sizeof(od_coeff) * n);
}

int32_t od_pvq_compute_gain(const int16_t* x, int n, int q0, int32_t* g, int16_t beta, int bshift) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g_(c.mu);
  PvqHelperBuf* b = helper_begin(c);
  b->args[0] = n; b->args[1] = q0; b->args[2] = beta; b->args[3] = bshift;
  memcpy(b->a16[0], x, sizeof(int16_t) * n);
  helper_run(c, 7);
  *g = b->args[14];
  return b->args[15];
}

int od_rdo_quant(od_coeff x, int q, double delta0, double pvq_norm_lambda) {
  HostCtx& c = ctx();
  std::lock_guard<std::mutex> g_(c.mu);
  PvqHelperBuf* b = helper_begin(c);
  b->args[0] = x; b->args[1] = q; b->dargs[0] = delta0; b->dargs[1] = pvq_norm_lambda;
  helper_run(c, 11);
  return b->args[15];
}

// ---- Section B ------------------------------------------------------------
int daala_b200_forward_frame(const daala_b200_frame* f, int nplanes, void* stream) {
  return daala_b200_launch_forward(f, nplanes, (cudaStream_t)stream);
}
int daala_b200_forward_frame_no_tma(const daala_b200_frame* f, int nplanes, void* stream) {
  return daala_b200_launch_forward_no_tma(f, nplanes, (cudaStream_t)stream);
}
int daala_b200_inverse_frame(const daala_b200_frame* f, int nplanes, void* stream) {
  return daala_b200_launch_inverse(f, nplanes, (cudaStream_t)stream);
}
int daala_b200_inverse_frame_lapped(const daala_b200_frame* f, int nplanes, void* stream) {
  return daala_b200_launch_inverse_lapped_only(f, nplanes, (cudaStream_t)stream);
}
int daala_b200_sb_postfilter_store_frame(const daala_b200_frame* f, int nplanes, void* stream) {
  return daala_b200_launch_sb_postfilter_store(f, nplanes, (cudaStream_t)stream);
}
int daala_b200_plane_sb_filter(int32_t* c, int stride, int nhsb, int nvsb, int xdec, int ydec, int post,
                               void* stream) {
  return daala_b200_launch_plane_sb_filter(c, stride, nhsb, nvsb, xdec, ydec, post, (cudaStream_t)stream);
}
int daala_b200_haar_blocks(int32_t* blocks, int count, int ln, int inverse, void* stream) {
  return daala_b200_launch_haar_blocks(blocks, count, ln, inverse, (cudaStream_t)stream);
}

int daala_b200_block_transform(int32_t* blocks, int count, int ln, int mode, void* stream) {
  return daala_b200_launch_block_transform(blocks, count, ln, mode, (cudaStream_t)stream);
}

int daala_b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

const char* daala_b200_version(void) { return "daala_b200 0.1 (sm_90a)"; }

}  // extern "C"
