// orbs.cu -- batched stream pipeline (north_star's "batched many-frame mode"): per frame t of a batch the device
// does what Tracking::GrabImageRGBD -> Frame::Frame(RGB-D) -> TrackWithMotionModel's SearchByProjection do on the
// CPU (src/Tracking.cc:331-375,1324-1352; src/Frame.cc:176-240), with no host round trip between the stages.
#include <memory>
#include <new>

#include "dynm.cuh"
#include "dynm_plane.cuh"
#include "flow.cuh"
#include "orbm_host.h"
#include "orbx_host.h"

using namespace b200;

namespace b200 {

struct GlueOut {     // SoA per frame, stride cap
  float *x, *y, *ang, *uright, *depth, *xw;
  int* oct;
  uint8_t* valid;
};

// Frame::ComputeStereoFromRGBD (src/Frame.cc:850-871) + Frame::UnprojectStereo (:879-899) for every keypoint,
// and the AoS -> SoA split the matcher kernel reads.
__global__ void __launch_bounds__(256) k_frame_glue(const OrbxKeyPoint* __restrict__ kps, const int* __restrict__ nkp,
                                                    int cap, const float* __restrict__ depth,
                                                    const uint16_t* __restrict__ kpd16, float depth_factor, int rows,
                                                    int cols, const float* __restrict__ Tcw, float fx, float fy,
                                                    float cx, float cy, float bf, GlueOut o) {
  const int f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nkp[f]) return;
  const size_t g = (size_t)f * cap + i;
  const OrbxKeyPoint kp = kps[g];
  const float* T = Tcw + (size_t)f * 16;
  const float u = kp.x, v = kp.y;
  // imDepth.at<float>(v,u) (src/Frame.cc:863).  kpd16: the CV_16U sensor pixel, already fetched per keypoint by
  // k_depth_prefetch, converted like convertTo(CV_32F, mDepthMapFactor) does (src/Tracking.cc:366-367).
  const float d = kpd16 ? __fmul_rn((float)kpd16[g], depth_factor)
                        : depth[(size_t)f * rows * cols + (size_t)(int)v * cols + (int)u];
  o.x[g] = u; o.y[g] = v; o.ang[g] = kp.angle; o.oct[g] = kp.octave;
  float ur = -1.f, dd = -1.f;
  uint8_t ok = 0;
  if (d > 0) {
    dd = d;
    ur = __fsub_rn(u, __fdiv_rn(bf, d));
    const float invfx = __fdiv_rn(1.0f, fx), invfy = __fdiv_rn(1.0f, fy);   // src/Frame.cc:215-216
    const float x = __fmul_rn(__fmul_rn(__fsub_rn(u, cx), d), invfx);
    const float y = __fmul_rn(__fmul_rn(__fsub_rn(v, cy), d), invfy);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float Rwc[3] = {T[0 * 4 + r], T[1 * 4 + r], T[2 * 4 + r]};   // mRwc = mRcw.t()
      // mOw = -mRwc*mtcw (src/Frame.cc:373 -- this fork multiplies the EVALUATED transpose, so the product takes the
      // small-matrix gemm path: float accumulation left to right, alpha = -1)
      const float ow = -__fadd_rn(__fadd_rn(__fmul_rn(Rwc[0], T[3]), __fmul_rn(Rwc[1], T[7])), __fmul_rn(Rwc[2], T[11]));
      o.xw[g * 3 + r] = gemm3(Rwc, x, y, d, ow);
    }
    ok = 1;
  }
  o.uright[g] = ur; o.depth[g] = dd; o.valid[g] = ok;
}

// Depth under the selected keypoints, fetched as soon as the selection exists (the final KeyPoint coordinates are the
// level coordinates times the level's scale factor, src/ORBextractor.cc:1104-1110, exactly as k_orient_desc forms them)
// -- on a side stream, so the PCIe round trips of the in-place host reads overlap blur and descriptors.
// The reads are latency-bound on the host link (microseconds each, a bounded number in flight), not on the SMs, and
// every read that is queued behind that bound sits in the SM -> L2 request path in front of the HBM traffic of the
// kernels running beside it: one thread per item queues hundreds of thousands of reads and stalls the blur beside it,
// one CTA leaves the link idle.  So: DEPTH_PF_CTAS small CTAs walk the (frame, keypoint) items with DEPTH_PF_UNROLL
// reads in flight per thread.
constexpr int DEPTH_PF_THREADS = 256, DEPTH_PF_UNROLL = 4, DEPTH_PF_CTAS = 8;
__global__ void __launch_bounds__(DEPTH_PF_THREADS) k_depth_prefetch(LevelTab lt, const unsigned* __restrict__ sel,
                                                        const int* __restrict__ selcnt, int sel_per_frame, int cap,
                                                        const uint16_t* __restrict__ depth16, int rows, int cols, int f0,
                                                        int nframes, uint16_t* __restrict__ kpd16) {
  const long long total = (long long)nframes * cap, stride = (long long)gridDim.x * DEPTH_PF_THREADS;
  for (long long base = (long long)blockIdx.x * DEPTH_PF_THREADS + threadIdx.x; base < total; base += stride * DEPTH_PF_UNROLL) {
    const uint16_t* src[DEPTH_PF_UNROLL];
    long long dst[DEPTH_PF_UNROLL];
#pragma unroll
    for (int k = 0; k < DEPTH_PF_UNROLL; ++k) {
      src[k] = nullptr;
      const long long it = base + k * stride;
      if (it >= total) continue;
      const int f = f0 + (int)(it / cap), j = (int)(it % cap);
      const int* sc = selcnt + (size_t)f * lt.nlevels;
      int l = -1, idx = 0, acc = 0;
      for (int q = 0; q < lt.nlevels; ++q) {
        const int c = sc[q];
        if (l < 0 && j < acc + c) { l = q; idx = j - acc; }
        acc += c;
      }
      if (l < 0) continue;
      const unsigned pk = sel[(size_t)f * sel_per_frame + lt.sel_off[l] + idx];
      const float s = lt.sf[l];
      const float u = (l != 0) ? __fmul_rn((float)kp_x(pk), s) : (float)kp_x(pk);
      const float v = (l != 0) ? __fmul_rn((float)kp_y(pk), s) : (float)kp_y(pk);
      src[k] = depth16 + (size_t)f * rows * cols + (size_t)(int)v * cols + (int)u;
      dst[k] = (long long)f * cap + j;
    }
    uint16_t val[DEPTH_PF_UNROLL];
#pragma unroll
    for (int k = 0; k < DEPTH_PF_UNROLL; ++k) val[k] = src[k] ? *src[k] : (uint16_t)0;
#pragma unroll
    for (int k = 0; k < DEPTH_PF_UNROLL; ++k)
      if (src[k]) kpd16[dst[k]] = val[k];
  }
}

__global__ void k_fill_i32(int* p, int v, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// ---- TrackHomo (perfect/src/Tracking.cc:1331-1399) of homography batches --------------------------------------------
// Per frame, what TrackHomo did: HC_WORDS ints, and out[10] doubles (H, found) beside them.
enum { HC_BRANCH, HC_NMATCH, HC_NPAIRS, HC_NFIT, HC_WARP, HC_WORDS };
constexpr int HC_MIN_MATCHES = 20;   // `nmatches<20` (perfect/src/Tracking.cc:1366,1374)
constexpr int HC_MIN_PAIRS = 50;     // `points_current.size() > 50` (:1381)
constexpr int HC_PAIR_THREADS = 1024;

// `if(nmatches<20)` (perfect/src/Tracking.cc:1366): the search at 2 th takes the last frame's keypoints as its queries;
// otherwise it takes none, and its kernels return at once.
__global__ void k_hc_retry(const int* __restrict__ nmatch, const int* __restrict__ nlast, int* __restrict__ retry,
                           int* __restrict__ nlast2) {
  *retry = *nmatch < HC_MIN_MATCHES;
  *nlast2 = *retry ? *nlast : 0;
}

// After the searches: the pairs of the final search (the second when *retry) in the order the overload pushes them (query i, the last frame's
// keypoint i, ascending; perfect/src/ORBmatcher.cc:1835-1836) as findHomography(points_current, points_last) takes them
// (src = the current keypoint, dst = the last one), then the branch: fewer than 20 matches, at most 50 pairs, or the fit
// with n = the pair count.  out (H, found) starts at zero: the empty H of every branch without a model.
__global__ void __launch_bounds__(HC_PAIR_THREADS) k_hc_pairs(const int* __restrict__ retry, const int* __restrict__ acc1,
                                                              const int* __restrict__ nm1, const int* __restrict__ acc2,
                                                              const int* __restrict__ nm2,
                                                              const int* __restrict__ nlast, const float* __restrict__ lx,
                                                              const float* __restrict__ ly, const float* __restrict__ cx,
                                                              const float* __restrict__ cy, float2* __restrict__ src,
                                                              float2* __restrict__ dst, int* __restrict__ st,
                                                              double* __restrict__ out) {
  __shared__ int ws[HC_PAIR_THREADS / 32];
  __shared__ int base;
  const int t = threadIdx.x, nl = *nlast;
  const int* acc = *retry ? acc2 : acc1;
  const int* nmatch = *retry ? nm2 : nm1;
  if (t == 0) base = 0;
  if (t < 10) out[t] = 0.0;
  __syncthreads();
  for (int b0 = 0; b0 < nl; b0 += HC_PAIR_THREADS) {
    const int i = b0 + t, a = i < nl ? acc[i] : -1;
    const unsigned bal = __ballot_sync(0xffffffffu, a >= 0);
    if ((t & 31) == 0) ws[t >> 5] = __popc(bal);
    __syncthreads();
    if (t == 0) {
      int s = base;
      for (int w = 0; w < HC_PAIR_THREADS / 32; ++w) { const int c = ws[w]; ws[w] = s; s += c; }
      base = s;
    }
    __syncthreads();
    if (a >= 0) {
      const int o = ws[t >> 5] + __popc(bal & ((1u << (t & 31)) - 1u));
      src[o] = make_float2(cx[a], cy[a]);
      dst[o] = make_float2(lx[i], ly[i]);
    }
    __syncthreads();
  }
  if (t == 0) {
    const int m = *nmatch, np = base;
    const bool fit = m >= HC_MIN_MATCHES && np > HC_MIN_PAIRS;
    st[HC_BRANCH] = m < HC_MIN_MATCHES ? ORBS_HOMO_FEW_MATCHES : fit ? ORBS_HOMO_NO_MODEL : ORBS_HOMO_FEW_PAIRS;
    st[HC_NMATCH] = m;
    st[HC_NPAIRS] = np;
    st[HC_NFIT] = fit ? np : 0;
    st[HC_WARP] = 0;
  }
}

// `if(flag && !homo.empty())` (perfect/src/Tracking.cc:713): a found model warps the frame
__global__ void k_hc_found(const double* __restrict__ out, int* __restrict__ st) {
  if (st[HC_NFIT] && out[9] != 0.0) {
    st[HC_BRANCH] = ORBS_HOMO_WARPED;
    st[HC_WARP] = 1;
  }
}

// ---- orbs_continue: the last frame of a batch, kept as the next batch's frame -1 --------------------------------------
struct CarryOut {
  float *x, *y, *ang, *xw;
  int* oct;
  uint8_t *valid, *desc;
  int* n;
  float* T;
  uint8_t* img;   // NULL: no image is carried
};
struct CarrySrc {   // one frame of a batch: its glue SoA, descriptors, count and pose
  const float *x, *y, *ang, *xw;
  const int* oct;
  const uint8_t *valid, *desc;
  const int* n;
  const float* T;
};

// Row y = 0: the frame's keypoint count, pose, glue SoA (what LastView and k_hc_pairs read) and descriptors.  Row y = 1:
// the px-byte image its ComputeMask received -- `warped` when *warp is set (HC_WARP of a homography batch), else `gray`.
// CARRY_CTAS CTAs per row walk either (a few thousand keypoints, a fraction of a megabyte of image).
constexpr int CARRY_CTAS = 64;
__global__ void __launch_bounds__(256) k_carry_gather(CarrySrc s, const uint8_t* __restrict__ gray,
                                                      const uint8_t* __restrict__ warped, const int* __restrict__ warp,
                                                      size_t px, CarryOut o) {
  const int stride = gridDim.x * blockDim.x, i0 = blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.y == 0) {
    const int n = *s.n;
    if (i0 == 0) *o.n = n;
    if (i0 < 16) o.T[i0] = s.T[i0];
    for (int i = i0; i < n; i += stride) {
      o.x[i] = s.x[i]; o.y[i] = s.y[i]; o.ang[i] = s.ang[i]; o.oct[i] = s.oct[i]; o.valid[i] = s.valid[i];
#pragma unroll
      for (int r = 0; r < 3; ++r) o.xw[3 * i + r] = s.xw[3 * i + r];
      const uint4* d = reinterpret_cast<const uint4*>(s.desc) + 2 * i;
      uint4* e = reinterpret_cast<uint4*>(o.desc) + 2 * i;
      e[0] = d[0]; e[1] = d[1];
    }
    return;
  }
  const uint8_t* src = (warp && *warp) ? warped : gray;
  for (size_t i = i0; i < px; i += stride) o.img[i] = src[i];
}

}  // namespace b200

// An executable graph, re-targeted in place to each newly captured graph of the same shape (else instantiated anew).
struct GraphExec {
  cudaGraphExec_t g = nullptr;
  GraphExec() = default;
  GraphExec(const GraphExec&) = delete;
  GraphExec& operator=(const GraphExec&) = delete;
  ~GraphExec() { if (g) cudaGraphExecDestroy(g); }
  int update(cudaGraph_t graph) {
    if (g) {
      cudaGraphExecUpdateResultInfo info;
      if (cudaGraphExecUpdate(g, graph, &info) == cudaSuccess) return B200ORB_OK;
      cudaGetLastError();
      cudaGraphExecDestroy(g);
      g = nullptr;
    }
    B200_CUDA(cudaGraphInstantiate(&g, graph, 0));
    return B200ORB_OK;
  }
};

// Host batches are uploaded in at most MAX_CHUNKS chunks (orbs_set_chunk_frames sets their size).
static constexpr int MAX_CHUNKS = 7;

// The variants a continued batch must share with the batch it continues (the depth kind and host / device may differ).
enum BatchVariant { BV_PLAIN, BV_FLOW, BV_DEVICE_FLOW, BV_HOMOGRAPHY };
static int batch_variant(const OrbsBatch* b) {
  return b->homography ? BV_HOMOGRAPHY : b->device_flow ? BV_DEVICE_FLOW : b->flow ? BV_FLOW : BV_PLAIN;
}
// OrbsParams of two handles whose batches may form one sequence: everything but the batch capacity
static bool same_params(OrbsParams a, OrbsParams b) {
  a.max_frames = b.max_frames = 0;
  return memcmp(&a, &b, sizeof(a)) == 0;
}

// One enqueued batch, as the readers and orbs_continue see it.  F = 0: no batch.
struct BatchRecord {
  int F = 0, rows = 0, cols = 0, cap = 0;
  int variant = BV_PLAIN;     // flow, device_flow and homography batches are masked; only homography batches ran TrackHomo
  int seq_end = 0;            // the sequence position after it, saturated at 2 (TrackHomo asks: first, second or later)
  const float* dT = nullptr;  // a device batch's poses, the caller's buffer; NULL: a host batch, whose poses are in d_T
  OrbsParams prm{};
};

struct orbs {
  OrbsParams prm{};
  int device = 0;
  std::unique_ptr<orbx> ex;
  long long launches = 0;
  int rows = 0, cols = 0, maxF = 0, cap = 0;
  // Geometry block, carved for (rows, cols, maxF, cap): the glue's SoA, the match results and the scratch of the
  // non-fused LAST search.
  DeviceBlock geom;
  float *d_x = nullptr, *d_y = nullptr, *d_ang = nullptr, *d_ur = nullptr, *d_dep = nullptr, *d_xw = nullptr;
  int* d_oct = nullptr;
  uint8_t* d_valid = nullptr;
  int *d_c2l = nullptr, *d_nm = nullptr, *d_acc = nullptr;
  void* d_match_scratch = nullptr;
  // Host-input block, carved by the first host batch: the uploaded inputs and the depth under the keypoints.
  DeviceBlock in;
  int in_depth_bytes = -1;  // depth staging per pixel it holds: 4 for f32 input, 2 for pageable CV_16U, 0 for page-locked,
                            // -1 while it holds no inputs of the current geometry
  uint8_t* d_gray = nullptr;
  float* d_T = nullptr;
  uint16_t* d_kpd16 = nullptr;    // [maxF][cap] CV_16U depth under the keypoints
  void* d_depth = nullptr;        // [maxF][rows][cols] uploaded depth, f32 or CV_16U
  const uint16_t* gather_src = nullptr;   // the CV_16U batch k_depth_prefetch reads during a call
  int chunk_frames = 128;   // frames per upload chunk of host batches
  Stream copy_stream;
  Stream gather_stream;     // k_depth_prefetch, beside the extractor's stream
  Event chunk_ev[MAX_CHUNKS];
  Event inputs_free_ev;     // the previous call's kernels are done with the host-input block
  Event sel_ev, gather_ev;
  Event compute_done_ev;    // recorded after the last kernel of a host batch (before its downloads)
  orbs* chain_prev = nullptr;              // orbs_chain_after: the next host batch's kernels wait for that handle's kernels
  // Dynamic-mask block, reserved by the first masked batch: the final bit plane and mask sum per frame, and the flow of
  // host batches (uploaded or computed on the device).
  DeviceBlock dyn;
  uint32_t* d_plane = nullptr;   // [maxF][rows][ceil(cols / 32)]
  unsigned* d_msum = nullptr;    // [maxF]
  float* d_flow = nullptr;       // [maxF][rows / 2][cols / 2][2]
  uint8_t* d_prev_gray = nullptr;   // prev_gray of batches with device_flow
  FbGeom fbg;                       // and their Farneback geometry and scratch (chunks of min(maxF, FB_CHUNK) frames)
  FbScratch fbs{};
  // Homography block, reserved by the first homography batch: TrackHomo's per-frame record, its searches' outputs, the
  // pairs, findHomography's scratch and the warped frame.  The iteration table has a block of its own, filled once per
  // keypoint capacity.
  DeviceBlock homo, homo_tab;
  int* d_hstate = nullptr;       // [maxF][HC_WORDS]
  double* d_hout = nullptr;      // [maxF][10]
  int *d_hacc = nullptr, *d_hc2l = nullptr, *d_hnm = nullptr;   // [2][cap], [2][cap], [2]: the searches at th and 2 th
  int *d_hretry = nullptr, *d_hnl2 = nullptr;
  float2 *d_hsrc = nullptr, *d_hdst = nullptr;
  uint8_t *d_hmask = nullptr, *d_dest = nullptr;
  HfScratch hfs{};
  double* d_tab = nullptr;
  int tab_cap = 0;
  GraphExec chain_exec;          // the last homography batch's launches, replayed with one graph launch
  // The last batch: cleared before orbs_submit changes any state, written once a batch is wholly enqueued.
  BatchRecord last;
  // Carry block, reserved by orbs_continue: the frame before a continued batch (frame P, the last frame of the last batch
  // of the handle continued) -- its keypoint count, pose, glue SoA and descriptors, and for device_flow and homography
  // batches the full-resolution image its ComputeMask received.  Written on P's handle's stream; carry_ev follows the
  // copy, carry_free_ev the last kernel of this handle that reads it.
  DeviceBlock carry;
  CarryOut cy{};
  Event carry_ev, carry_free_ev;
  struct {
    bool pending = false;        // the next batch continues; consumed by that batch
    BatchRecord from;            // the batch whose last frame the carry holds
  } cont;
  int create_streams() {
    B200_CHECK(copy_stream.create());
    B200_CHECK(gather_stream.create());
    for (Event& e : chunk_ev) B200_CHECK(e.create());
    for (Event* e : {&inputs_free_ev, &sel_ev, &gather_ev, &compute_done_ev, &carry_ev, &carry_free_ev}) B200_CHECK(e->create());
    return B200ORB_OK;
  }
  // The carry for frames of r x c pixels and keypoint capacity kc; img: with the image.  Grow-only; a replaced block is
  // freed by cudaFree, which waits for the device.
  int ensure_carry(int r, int c, int kc, bool img) {
    return carry.reserve(ex->stream, [&](Carver& t) {
      const size_t n = kc;
      cy.x = t.take<float>(n); cy.y = t.take<float>(n); cy.ang = t.take<float>(n); cy.xw = t.take<float>(3 * n);
      cy.oct = t.take<int>(n); cy.valid = t.take<uint8_t>(n); cy.desc = t.take<uint8_t>(32 * n); cy.n = t.take<int>(1);
      cy.T = t.take<float>(16);
      cy.img = img ? t.take<uint8_t>((size_t)r * c) : nullptr;
    });
  }
  // A continued batch of keypoint capacity kcap, before it touches any state: the frame it continues has its geometry,
  // parameters, keypoint capacity and variant, and no prev_gray competes with it.
  int check_continue(const OrbsBatch* b, int kcap) const {
    const BatchRecord& p = cont.from;
    const char* why = b->rows != p.rows || b->cols != p.cols ? "its image size"
                      : !same_params(prm, p.prm)            ? "its OrbsParams"
                      : kcap != p.cap                       ? "its keypoint capacity"
                      : batch_variant(b) != p.variant       ? "its variant"
                      : b->prev_gray                        ? "prev_gray"
                                                            : nullptr;
    if (why) {
      set_error("a continued batch differs from the frame it continues in %s", why);
      return B200ORB_EINVAL;
    }
    return B200ORB_OK;
  }
  // depth_bytes: depth staging per pixel a host batch needs; -1 for a device batch, which needs no host-input
  // block.  Either block is replaced only after the stream is synchronised: every copy-stream and gather-stream
  // operation of earlier calls is joined into it by an event.
  int ensure(int r, int c, int F, int depth_bytes) {
    B200_CHECK(ex->ensure_geometry(r, c, F));
    if (!(r == rows && c == cols && F <= maxF && ex->cap == cap)) {
      rows = 0;   // no geometry until its block exists
      in_depth_bytes = -1;   // the host-input block is sized for the old geometry
      const int nF = std::max(F, ex->maxF), ncap = ex->cap;
      const size_t n = (size_t)nF * ncap;
      B200_CHECK(geom.carve(ex->stream, [&](Carver& t) {
        d_x = t.take<float>(n); d_y = t.take<float>(n); d_ang = t.take<float>(n); d_ur = t.take<float>(n);
        d_dep = t.take<float>(n); d_xw = t.take<float>(3 * n); d_oct = t.take<int>(n); d_valid = t.take<uint8_t>(n);
        d_c2l = t.take<int>(n); d_nm = t.take<int>(nF); d_acc = t.take<int>(n);
        d_match_scratch = t.take<char>(match_last_scratch_bytes(nF, ncap, ncap));
      }));
      rows = r; cols = c; maxF = nF; cap = ncap;
    }
    if (depth_bytes > in_depth_bytes) {
      in_depth_bytes = -1;
      const size_t px = (size_t)maxF * rows * cols;
      B200_CHECK(in.carve(ex->stream, [&](Carver& t) {
        d_gray = t.take<uint8_t>(px); d_T = t.take<float>((size_t)maxF * 16);
        d_kpd16 = t.take<uint16_t>((size_t)maxF * cap); d_depth = t.take<uint8_t>(px * depth_bytes);
      }));
      in_depth_bytes = depth_bytes;
    }
    return B200ORB_OK;
  }
  // Masked batches, before they touch any state: the flow field is at least 2 x 2 and both bit planes of a frame fit one
  // CTA's shared memory (on an H100, 232448 bytes: rows * ceil(cols / 32) <= 29039, e.g. 1280 x 725).
  int check_masked(int r, int c) const {
    B200_CHECK(dynm_check_geometry(r / 2, c / 2, r, c));
    int optin = 0;
    B200_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    if (dynp_smem_bytes(r, c) > (size_t)optin) {
      set_error("masked tracking of %dx%d images needs %zu bytes of shared memory per CTA (two bit planes of the mask); the "
                "device allows %d: rows * ceil(cols / 32) must be at most %d", c, r, dynp_smem_bytes(r, c), optin,
                (optin / 4 - 33) / 2);
      return B200ORB_EINVAL;
    }
    return B200ORB_OK;
  }
  // host_flow: d_flow receives the caller's flow; dev_flow (the Farneback geometry of the batch, or NULL): the device
  // computes it there and needs the Farneback scratch
  int ensure_dyn(bool host_flow, const FbGeom* dev_flow) {
    const size_t planes = (size_t)maxF * rows * dynp_words(cols);
    const size_t flow = host_flow || dev_flow ? (size_t)maxF * (rows / 2) * (cols / 2) * 2 : 0;
    if (dev_flow) fbg = *dev_flow;
    return dyn.reserve(ex->stream, [&](Carver& t) {
      d_plane = t.take<uint32_t>(planes); d_msum = t.take<unsigned>(maxF); d_flow = t.take<float>(flow);
      d_prev_gray = nullptr;
      if (dev_flow) {
        d_prev_gray = t.take<uint8_t>((size_t)rows * cols);
        fb_take(t, fbs, fbg, fb_chunk());
      }
    });
  }
  int fb_chunk() const { return std::min(maxF, FB_CHUNK); }
  // Homography batches: TrackHomo's record and scratch, and the iteration table of findHomography for every pair count
  // the fit can take (51 .. cap), computed once on the host.
  int ensure_homo() {
    const size_t px = (size_t)rows * cols;
    B200_CHECK(homo.reserve(ex->stream, [&](Carver& t) {
      d_hstate = t.take<int>((size_t)maxF * HC_WORDS); d_hout = t.take<double>((size_t)maxF * 10);
      d_hacc = t.take<int>(2 * (size_t)cap); d_hc2l = t.take<int>(2 * (size_t)cap); d_hnm = t.take<int>(2);
      d_hretry = t.take<int>(1); d_hnl2 = t.take<int>(1);
      d_hsrc = t.take<float2>(cap); d_hdst = t.take<float2>(cap); d_hmask = t.take<uint8_t>(cap);
      d_dest = t.take<uint8_t>(px);
      hf_take(t, hfs, cap);
    }));
    if (tab_cap == cap) return B200ORB_OK;
    tab_cap = 0;
    std::vector<double> tab;
    if (cap > HC_MIN_PAIRS) hf_tab(HC_MIN_PAIRS + 1, cap, tab);
    B200_CHECK(homo_tab.carve(ex->stream, [&](Carver& t) { d_tab = t.take<double>(tab.size()); }));
    // From pageable memory the copy is staged before the call returns (so `tab` may go), and it may wait for the work
    // already on the stream: once per handle and keypoint capacity, on its first homography batch.
    B200_CUDA(cudaMemcpyAsync(d_tab, tab.data(), tab.size() * sizeof(double), cudaMemcpyHostToDevice, ex->stream));
    tab_cap = cap;
    return B200ORB_OK;
  }
  // Flow::ComputeMask + the masked Frame constructor's keypoint filter (perfect/src/Flow.cc:24-47, perfect/src/Frame.cc:
  // 356-377) on frames [f0, f0 + F) the extractor has just run, in place; kpd16 (the CV_16U depth under the keypoints)
  // moves with them.  dflow: [F][rows / 2][cols / 2][2] f32 of those frames.
  int mask_filter(const float* dflow, float thr, uint16_t* kpd16, int f0, int F) {
    if (thr < 40.0f) thr = 40.0f;   // perfect/src/Flow.cc:24
    const size_t o = (size_t)f0 * cap;
    return launch_dynm_plane_filter(F, dflow, rows / 2, cols / 2, thr, rows, cols, d_plane + (size_t)f0 * rows * dynp_words(cols),
                                    d_msum + f0, ex->d_kps + o, ex->d_desc + o * 32, kpd16 ? kpd16 + o : nullptr, ex->d_n + f0,
                                    cap, ex->stream, &launches);
  }
  // Frame glue of frames [f0, f0 + F) as their keypoints stand.  Depth is the gathered CV_16U value under each keypoint
  // times `factor` when kpd16 is given, else the f32 image batch dd.
  void glue(int f0, int F, const float* dd, const uint16_t* kpd16, float factor, const float* dT) {
    const size_t o = (size_t)f0 * cap;
    GlueOut go{d_x + o, d_y + o, d_ang + o, d_ur + o, d_dep + o, d_xw + 3 * o, d_oct + o, d_valid + o};
    k_frame_glue<<<dim3((cap + 255) / 256, F), 256, 0, ex->stream>>>(ex->d_kps + o, ex->d_n + f0, cap,
                                                                    dd ? dd + (size_t)f0 * rows * cols : nullptr,
                                                                    kpd16 ? kpd16 + o : nullptr, factor, rows, cols,
                                                                    dT + 16 * (size_t)f0, prm.fx, prm.fy, prm.cx, prm.cy,
                                                                    prm.bf, go);
    ++launches;
  }
  // The glued frame f of the batch as the last frame of a search (instance p: frame f + p).  nlast: its query counts
  // (NULL: its keypoint counts).
  LastView frame_last(int f, const int* nlast, const float* dT) const {
    const size_t o = (size_t)f * cap;
    return LastView{d_xw + 3 * o, d_valid + o, d_oct + o, d_ang + o, ex->d_desc + o * 32, nullptr,
                    nlast ? nlast : ex->d_n + f, dT + 16 * (size_t)f, (size_t)cap};
  }
  // The carried frame P (orbs_continue) as the last frame of frame 0's search
  LastView carry_last(const int* nlast) const {
    return LastView{cy.xw, cy.valid, cy.oct, cy.ang, cy.desc, nullptr, nlast ? nlast : cy.n, cy.T, (size_t)cap};
  }
  // SearchByProjection(frame f0 + p, instance p of lv, th, mono = 0) for p = 0 .. npairs - 1 on the glued frames:
  // acc[p][last keypoint] (the query's accepted current keypoint before the rotation prune), c2l[p][cur keypoint], nm[p].
  int search(int f0, int npairs, const LastView& lv, float th, float nnratio, int check_ori, const float* dT, int* acc,
             int* c2l, int* nm) {
    MatchCam cam;
    memset(&cam, 0, sizeof(cam));
    cam.fx = prm.fx; cam.fy = prm.fy; cam.cx = prm.cx; cam.cy = prm.cy; cam.bf = prm.bf;
    cam.b = prm.bf / prm.fx;                       // mb = mbf/fx, src/Frame.cc:218
    cam.min_x = 0.f; cam.max_x = (float)cols;      // no distortion: ComputeImageBounds, src/Frame.cc:617-623
    cam.min_y = 0.f; cam.max_y = (float)rows;
    for (int l = 0; l < prm.orb.nlevels; ++l) cam.sf[l] = ex->sf[l];
    cam.th = th; cam.nnratio = nnratio; cam.mono = 0; cam.check_ori = check_ori;
    cam.nlevels = prm.orb.nlevels;
    cam.last_obs_default = 1;                      // last-frame points behave like mapped points (Observations()>0)
    const size_t c = cap, n = (size_t)f0 * c;
    CurView cv;
    memset(&cv, 0, sizeof(cv));
    cv.x = d_x + n; cv.y = d_y + n; cv.ang = d_ang + n; cv.uright = d_ur + n; cv.oct = d_oct + n;
    cv.desc = ex->d_desc + n * 32; cv.obs = nullptr; cv.n = ex->d_n + f0; cv.Tcw = dT + 16 * (size_t)f0; cv.stride = c;
    return launch_match_last(cv, lv, cam, npairs, d_match_scratch, acc, c2l, nm, ex->stream, &launches);
  }
  // The perfect variant's live path frame after frame (perfect/src/Tracking.cc:703-719): TrackHomo against the filtered
  // frame t-1, ComputeMask of the frame warped by its H (perfect/src/Flow.cc:73-80) or of the frame itself, and the masked
  // constructor's filter, before frame t+1's TrackHomo reads frame t's filtered keypoints.  Each frame has the same
  // launches; the branch is decided on the device (HC_* record) and the kernels of a branch not taken return at once.
  // The launches (about 60 per frame, more than the device's queue of pending launches holds) are captured into a graph
  // and go to the stream as one graph launch, so that orbs_submit never waits for the device to drain that queue.
  // s: the frames of the sequence before this batch (saturated at 2); with s > 0 the carried frame P is frame -1.
  int homography_chain(const uint16_t* kpd16, float factor, const float* dT, float thr, int F, int s) {
    cudaStream_t st = ex->stream;
    B200_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const int rc = chain_launches(kpd16, factor, dT, thr, F, s);
    cudaGraph_t g = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(st, &g);
    if (rc != B200ORB_OK || ce != cudaSuccess) {
      if (g) cudaGraphDestroy(g);
      if (rc != B200ORB_OK) return rc;
      B200_CUDA(ce);
    }
    const int ur = chain_exec.update(g);
    cudaGraphDestroy(g);
    B200_CHECK(ur);
    B200_CUDA(cudaGraphLaunch(chain_exec.g, st));
    return B200ORB_OK;
  }
  int chain_launches(const uint16_t* kpd16, float factor, const float* dT, float thr, int F, int s) {
    cudaStream_t st = ex->stream;
    const size_t px = (size_t)rows * cols, hpx = (size_t)fbg.H * fbg.W, fpx = hpx * 2, c = cap;
    // sequence frame 0: ORBS_HOMO_NO_LAST
    B200_CUDA(cudaMemsetAsync(d_hstate, 0, (size_t)F * HC_WORDS * sizeof(int), st));
    B200_CUDA(cudaMemsetAsync(d_hout, 0, (size_t)F * 10 * sizeof(double), st));
    if (s <= 1 && 1 - s < F) {   // sequence frame 1: mVelocity is first set by frame 1's Track
      k_fill_i32<<<1, 32, 0, st>>>(d_hstate + (1 - s) * HC_WORDS + HC_BRANCH, ORBS_HOMO_NO_VELOCITY, 1);
      ++launches;
    }
    int t0 = 0;
    if (s == 0) {
      // sequence frame 0: no mImGrayLast, the zero field (mask = ones); mImGrayLast = pyrDown(gray_0)
      fb_pyrdown(st, fbg, d_gray, nullptr, 1, rows, cols, fbs.half, &launches);
      B200_CUDA(cudaMemsetAsync(d_flow, 0, fpx * sizeof(float), st));
      B200_CHECK(mask_filter(d_flow, thr, const_cast<uint16_t*>(kpd16), 0, 1));
      t0 = 1;
    } else {
      // mImGrayLast = pyrDown of what P's ComputeMask received
      fb_pyrdown(st, fbg, cy.img, nullptr, 1, rows, cols, fbs.half, &launches);
    }
    for (int t = t0; t < F; ++t) {
      const uint8_t* dest = d_gray + (size_t)t * px;
      if (s + t >= 2) {
        int* S = d_hstate + (size_t)t * HC_WORDS;
        double* O = d_hout + (size_t)t * 10;
        // the last frame: the filtered frame t-1, or P before frame 0 (glued by its own batch)
        const int* nl = t ? ex->d_n + t - 1 : cy.n;
        const float *lx = t ? d_x + (t - 1) * c : cy.x, *ly = t ? d_y + (t - 1) * c : cy.y;
        glue(t ? t - 1 : 0, t ? 2 : 1, nullptr, kpd16, factor, dT);   // the filtered frame t-1 and the unfiltered frame t
        // ORBmatcher matcher(0.9, true) (perfect/src/Tracking.cc:1345): nnratio 0.9 and checkOri on
        B200_CHECK(search(t, 1, t ? frame_last(t - 1, nullptr, dT) : carry_last(nullptr), prm.th, 0.9f, 1, dT, d_hacc,
                          d_hc2l, d_hnm));
        k_hc_retry<<<1, 1, 0, st>>>(d_hnm, nl, d_hretry, d_hnl2);
        ++launches;
        B200_CHECK(search(t, 1, t ? frame_last(t - 1, d_hnl2, dT) : carry_last(d_hnl2), 2 * prm.th, 0.9f, 1, dT,
                          d_hacc + c, d_hc2l + c, d_hnm + 1));
        k_hc_pairs<<<1, HC_PAIR_THREADS, 0, st>>>(d_hretry, d_hacc, d_hnm, d_hacc + c, d_hnm + 1, nl, lx, ly, d_x + t * c,
                                                  d_y + t * c, d_hsrc, d_hdst, S, O);
        ++launches;
        B200_CHECK(launch_hf_fit(st, d_hsrc, d_hdst, S + HC_NFIT, true, d_tab, HC_MIN_PAIRS + 1, hfs, O, d_hmask, &launches));
        k_hc_found<<<1, 1, 0, st>>>(O, S);
        ++launches;
        B200_CHECK(launch_warp(st, dest, 1, rows, cols, O, S + HC_WARP, d_dest, &launches));
        dest = d_dest;
      }
      // Farneback(mImGrayLast, pyrDown(dest)), then mImGrayLast = pyrDown(dest) (the swap of perfect/src/Flow.cc:50):
      // the previous frame's WARPED half image whenever that frame took the homography branch
      fb_pyrdown(st, fbg, dest, nullptr, 1, rows, cols, fbs.half + hpx, &launches);
      B200_CHECK(fb_pairs(st, fbg, fbs, 2, d_flow + (size_t)t * fpx, &launches));
      B200_CUDA(cudaMemcpyAsync(fbs.half, fbs.half + hpx, hpx, cudaMemcpyDeviceToDevice, st));
      B200_CHECK(mask_filter(d_flow + (size_t)t * fpx, thr, const_cast<uint16_t*>(kpd16), t, 1));
    }
    return B200ORB_OK;
  }
  // Frame glue and SearchByProjection(t, t-1) of the F frames the extractor has just run.  cont: frame 0 is searched
  // against the carried frame P.
  int run(const float* dd, const uint16_t* kpd16, float factor, const float* dT, int F, bool cont) {
    cudaStream_t st = ex->stream;
    glue(0, F, dd, kpd16, factor, dT);
    B200_CHECK(ex->prof_mark(ST_GLUE + 1));
    if (cont) {
      B200_CHECK(search(0, 1, carry_last(nullptr), prm.th, prm.nnratio, prm.check_ori, dT, d_acc, d_c2l, d_nm));
    } else {   // frame 0 of the batch has no predecessor: all -1, 0 matches
      k_fill_i32<<<(cap + 255) / 256, 256, 0, st>>>(d_c2l, -1, (size_t)cap);
      ++launches;
      B200_CUDA(cudaMemsetAsync(d_nm, 0, 4, st));
    }
    if (F > 1)
      B200_CHECK(search(1, F - 1, frame_last(0, nullptr, dT), prm.th, prm.nnratio, prm.check_ori, dT, d_acc, d_c2l + cap,
                        d_nm + 1));
    return ex->prof_mark(ST_MATCH + 1);
  }
};

// The one check of every reader of the last batch and of orbs_continue: h holds a batch, `frame` is one of its frames and
// the batch is of the kind the reader needs.
enum LastNeed { ANY_BATCH, MASKED_BATCH, HOMO_BATCH };
static int check_last(const orbs* h, int frame, LastNeed need) {
  const char* why = !h                                                       ? "bad argument"
                    : !h->last.F                                             ? "no results"
                    : need == MASKED_BATCH && h->last.variant == BV_PLAIN    ? "the last batch was not masked"
                    : need == HOMO_BATCH && h->last.variant != BV_HOMOGRAPHY ? "the last batch was not a homography batch"
                    : frame < 0 || frame >= h->last.F                        ? "frame outside the last batch"
                                                                             : nullptr;
  if (why) set_error("%s", why);
  return why ? B200ORB_EINVAL : B200ORB_OK;
}

extern "C" {

int orbs_create(const OrbsParams* p, int device, orbs_t** out) {
  if (!p || !out) { set_error("null argument"); return B200ORB_EINVAL; }
  *out = nullptr;
  orbx_t* ex = nullptr;
  B200_CHECK(orbx_create(&p->orb, device, &ex));
  DeviceGuard g(device);
  std::unique_ptr<orbs> h(new (std::nothrow) orbs());
  if (!h) { delete ex; set_error("out of host memory"); return B200ORB_EINVAL; }
  h->prm = *p;
  h->device = device;
  h->ex.reset(ex);
  B200_CHECK(h->create_streams());
  *out = h.release();
  return B200ORB_OK;
}
void orbs_destroy(orbs_t* h) { destroy_handle(h); }

int orbs_device_results(orbs_t* h, const OrbxKeyPoint** d_kps, const uint8_t** d_desc, const int32_t** d_nkp,
                        const int32_t** d_cur2last, const int32_t** d_nmatch, int* cap) {
  B200_CHECK(check_last(h, 0, ANY_BATCH));
  if (d_kps) *d_kps = h->ex->d_kps;
  if (d_desc) *d_desc = h->ex->d_desc;
  if (d_nkp) *d_nkp = h->ex->d_n;
  if (d_cur2last) *d_cur2last = h->d_c2l;
  if (d_nmatch) *d_nmatch = h->d_nm;
  if (cap) *cap = h->last.cap;
  return B200ORB_OK;
}

// Frame-glue outputs of frame `frame` of the last batch (Frame::ComputeStereoFromRGBD + UnprojectStereo per keypoint):
// mvuRight, mvDepth, the world point of the keypoint under the frame's pose, and whether it has depth.
int orbs_read_frame_glue(orbs_t* h, int frame, float* uright, float* depth, float* xw, uint8_t* valid, int cap) {
  B200_CHECK(check_last(h, frame, ANY_BATCH));
  if (cap < h->last.cap) { set_error("cap %d < the last batch's keypoint capacity %d", cap, h->last.cap); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  const size_t o = (size_t)frame * h->last.cap, n = (size_t)h->last.cap;
  cudaStream_t st = h->ex->stream;
  if (uright) B200_CUDA(cudaMemcpyAsync(uright, h->d_ur + o, 4 * n, cudaMemcpyDeviceToHost, st));
  if (depth) B200_CUDA(cudaMemcpyAsync(depth, h->d_dep + o, 4 * n, cudaMemcpyDeviceToHost, st));
  if (xw) B200_CUDA(cudaMemcpyAsync(xw, h->d_xw + o * 3, 12 * n, cudaMemcpyDeviceToHost, st));
  if (valid) B200_CUDA(cudaMemcpyAsync(valid, h->d_valid + o, n, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  return B200ORB_OK;
}

// orbx::after_select hook of CV_16U batches: the keypoints of frames [f0, f0 + F) are selected -> fetch the depth
// under them on the side stream (the stream of the extractor goes on with blur and descriptors meanwhile)
static int orbs_after_select(void* ctx, int f0, int F) {
  orbs* h = static_cast<orbs*>(ctx);
  orbx* ex = h->ex.get();
  B200_CUDA(cudaEventRecord(h->sel_ev, ex->stream));
  B200_CUDA(cudaStreamWaitEvent(h->gather_stream, h->sel_ev, 0));
  const long long items = (long long)F * h->cap;
  const int pf_grid = (int)std::min<long long>(DEPTH_PF_CTAS, (items + DEPTH_PF_THREADS - 1) / DEPTH_PF_THREADS);
  k_depth_prefetch<<<pf_grid, DEPTH_PF_THREADS, 0, h->gather_stream>>>(ex->ltab, ex->d_sel, ex->d_selcnt, ex->sel_per_frame, h->cap,
                                                                       h->gather_src, h->rows, h->cols, f0, F, h->d_kpd16);
  ++h->launches;
  B200_CUDA(cudaEventRecord(h->gather_ev, h->gather_stream));
  return B200ORB_OK;
}

// The eight batch forms include/b200orb.h lists under OrbsBatch; every other combination is refused.
static bool batch_form_ok(const OrbsBatch* b, const OrbsResults* out) {
  if (!b->gray || !b->Tcw || b->nframes <= 0 || b->rows <= 0 || b->cols <= 0) return false;
  if (!b->depth == !b->depth_u16 || (b->flow && b->device_flow) || (b->prev_gray && !b->device_flow)) return false;
  if (b->homography != 0 && (b->homography != 1 || b->device || !b->depth_u16 || !b->device_flow || b->prev_gray)) return false;
  if (b->device) return !out && b->depth && !b->device_flow;
  return out && out->kps && out->desc && out->nkp && out->cur2last && out->nmatch &&
         (b->depth_u16 || !(b->flow || b->device_flow));
}

// Host batch: the inputs go up in chunks on a copy stream while the extractor already works on the chunks that have
// arrived (PCIe and SMs overlap); everything after extraction runs on the whole batch.  d16_alias: the device alias of
// page-locked CV_16U depth, read in place; depth_bytes: the depth uploaded per pixel.
static int upload_and_extract(orbs_t* h, const OrbsBatch* b, const uint16_t* d16_alias, int depth_bytes) {
  cudaStream_t st = h->ex->stream;
  const int cols = b->cols;
  const size_t px = (size_t)b->rows * cols, F = b->nframes, fpx = (size_t)(b->rows / 2) * (cols / 2) * 2;
  const char* depth_up = b->depth ? (const char*)b->depth : (const char*)b->depth_u16;
  const int nchunk = (int)std::min<size_t>(MAX_CHUNKS, (F + h->chunk_frames - 1) / h->chunk_frames);   // >= 64-frame chunks keep each launch wide enough
  h->gather_src = d16_alias ? d16_alias : static_cast<const uint16_t*>(h->d_depth);
  h->ex->after_select = b->depth_u16 ? &orbs_after_select : nullptr;
  h->ex->after_select_ctx = h;
  B200_CUDA(cudaEventRecord(h->inputs_free_ev, st));
  B200_CUDA(cudaStreamWaitEvent(h->copy_stream, h->inputs_free_ev, 0));
  // orbs_chain_after: this batch's kernels start when the other handle's kernels are done -- the uploads enqueued
  // below (copy stream) and that handle's downloads run meanwhile, and kernels of two batches never share the SMs.
  // The uploads start only once that handle's in-place depth reads (k_depth_prefetch) are done: both cross the host
  // link toward the device, the reads are latency-bound and its matcher waits for them, while these uploads are
  // needed only when this batch's kernels start.
  if (h->chain_prev) {
    B200_CUDA(cudaStreamWaitEvent(st, h->chain_prev->compute_done_ev, 0));
    B200_CUDA(cudaStreamWaitEvent(h->copy_stream, h->chain_prev->gather_ev, 0));
  }
  h->chain_prev = nullptr;
  if (b->prev_gray)
    B200_CUDA(cudaMemcpyAsync(h->d_prev_gray, b->prev_gray, px, cudaMemcpyHostToDevice, h->copy_stream));
  for (int c = 0; c < nchunk; ++c) {
    const size_t f0 = F * c / nchunk, f1 = F * (c + 1) / nchunk;
    B200_CUDA(cudaMemcpyAsync(h->d_gray + px * f0, b->gray + px * f0, px * (f1 - f0), cudaMemcpyHostToDevice, h->copy_stream));
    const size_t o = px * f0 * depth_bytes;
    if (depth_bytes)
      B200_CUDA(cudaMemcpyAsync((char*)h->d_depth + o, depth_up + o, px * (f1 - f0) * depth_bytes, cudaMemcpyHostToDevice,
                                h->copy_stream));
    if (b->flow)
      B200_CUDA(cudaMemcpyAsync(h->d_flow + fpx * f0, b->flow + fpx * f0, fpx * (f1 - f0) * 4, cudaMemcpyHostToDevice,
                                h->copy_stream));
    B200_CUDA(cudaEventRecord(h->chunk_ev[c], h->copy_stream));
    B200_CUDA(cudaStreamWaitEvent(st, h->chunk_ev[c], 0));
    B200_CHECK(h->ex->run(h->d_gray + px * f0, cols, px, (int)(f1 - f0), (int)f0));
  }
  h->ex->after_select = nullptr;
  if (b->depth_u16) B200_CUDA(cudaStreamWaitEvent(st, h->gather_ev, 0));   // the last chunk's prefetch (the side stream is in order)
  return B200ORB_OK;
}

// Host batch: the results of the F frames go down into `out` behind the batch's kernels.
static int download(orbs_t* h, const OrbsResults* out, size_t F) {
  cudaStream_t st = h->ex->stream;
  const size_t hc = h->cap, cap = out->cap;
  if (cap == hc) {
    B200_CUDA(cudaMemcpyAsync(out->kps, h->ex->d_kps, sizeof(OrbxKeyPoint) * hc * F, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(out->desc, h->ex->d_desc, 32 * hc * F, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(out->cur2last, h->d_c2l, 4 * hc * F, cudaMemcpyDeviceToHost, st));
  } else {
    B200_CUDA(cudaMemcpy2DAsync(out->kps, sizeof(OrbxKeyPoint) * cap, h->ex->d_kps, sizeof(OrbxKeyPoint) * hc,
                                sizeof(OrbxKeyPoint) * hc, F, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpy2DAsync(out->desc, 32 * cap, h->ex->d_desc, 32 * hc, 32 * hc, F, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpy2DAsync(out->cur2last, 4 * cap, h->d_c2l, 4 * hc, 4 * hc, F, cudaMemcpyDeviceToHost, st));
  }
  B200_CUDA(cudaMemcpyAsync(out->nkp, h->ex->d_n, 4 * F, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaMemcpyAsync(out->nmatch, h->d_nm, 4 * F, cudaMemcpyDeviceToHost, st));
  return B200ORB_OK;
}

int orbs_submit(orbs_t* h, const OrbsBatch* b, const OrbsResults* out) {
  if (!h || !b || !batch_form_ok(b, out)) { set_error("bad argument"); return B200ORB_EINVAL; }
  // Every refusal comes before the first state change.
  const int F = b->nframes, rows = b->rows, cols = b->cols;
  const bool masked = b->flow || b->device_flow;
  if (masked) B200_CHECK(h->check_masked(rows, cols));
  FbGeom fg;
  if (b->device_flow) B200_CHECK(fb_geometry(rows / 2, cols / 2, &fg));
  int kcap = 0;   // the keypoint capacity ensure() gives the handle for this image size
  B200_CHECK(orbx_max_keypoints_for(h->ex.get(), rows, cols, &kcap));
  if (b->homography && kcap > HF_MAX_PAIRS) {   // TrackHomo's pairs go to findHomography, which takes at most HF_MAX_PAIRS
    set_error("homography batches take at most %d keypoints per frame (findHomography's pairs), not %d", HF_MAX_PAIRS, kcap);
    return B200ORB_EINVAL;
  }
  const bool cont = h->cont.pending;
  if (cont) B200_CHECK(h->check_continue(b, kcap));
  if (out && out->cap < kcap) { set_error("cap %d < required %d (orbx_max_keypoints)", out->cap, kcap); return B200ORB_ECAP; }
  DeviceGuard g(h->device);
  // The only CV_16U depth pixels the tracking path ever reads are the ones under the keypoints
  // (Frame::ComputeStereoFromRGBD); k_depth_prefetch fetches them as soon as a chunk's keypoints are selected.
  // Page-locked depth (cudaHostAlloc / cudaHostRegister, e.g. torch.pin_memory) is read in place over PCIe, so its
  // 0.6 MB/frame images are never uploaded; pageable depth is uploaded next to the gray images and read from HBM.
  const uint16_t* d16_alias = nullptr;
  if (b->depth_u16) {
    cudaPointerAttributes at;
    void* dev_alias = nullptr;
    if (cudaPointerGetAttributes(&at, b->depth_u16) == cudaSuccess && at.type == cudaMemoryTypeHost &&
        cudaHostGetDevicePointer(&dev_alias, const_cast<uint16_t*>(b->depth_u16), 0) == cudaSuccess && dev_alias)
      d16_alias = reinterpret_cast<const uint16_t*>(dev_alias);
    else
      cudaGetLastError();
  }
  const int depth_bytes = b->device ? -1 : b->depth ? 4 : (d16_alias ? 0 : 2);   // per pixel uploaded
  // From here on a failure leaves the handle with no batch: its buffers may have been replaced or partly written.
  h->last = BatchRecord{};
  B200_CHECK(h->ensure(rows, cols, F, depth_bytes));
  if (masked) B200_CHECK(h->ensure_dyn(b->flow && !b->device, b->device_flow ? &fg : nullptr));
  if (b->homography) B200_CHECK(h->ensure_homo());
  // The continuation is consumed by this batch; its frames take sequence positions s .. s + F - 1.
  const int s = cont ? h->cont.from.seq_end : 0;
  h->cont.pending = false;
  // Device batch: every input is read in place from HBM.  Host batch: from the uploaded copies.
  const float *dd = b->depth, *dflow = b->flow, *dT = b->Tcw;
  if (b->device) {
    B200_CHECK(h->ex->run(b->gray, cols, (size_t)rows * cols, F));
  } else {
    B200_CHECK(upload_and_extract(h, b, d16_alias, depth_bytes));
    dd = b->depth ? static_cast<const float*>(h->d_depth) : nullptr;
    dflow = h->d_flow;
    dT = h->d_T;
  }
  cudaStream_t st = h->ex->stream;
  if (cont) B200_CUDA(cudaStreamWaitEvent(st, h->carry_ev, 0));   // the carry copy, on the other handle's stream
  if (!b->device) B200_CUDA(cudaMemcpyAsync(h->d_T, b->Tcw, (size_t)F * 64, cudaMemcpyHostToDevice, st));
  uint16_t* kpd16 = b->depth_u16 ? h->d_kpd16 : nullptr;
  if (b->homography) {
    B200_CHECK(h->homography_chain(kpd16, b->depth_factor, dT, b->binary_threshold, F, s));
  } else {
    // frame 0's flow: from prev_gray, from P's image when continued, else the zero field
    if (b->device_flow)
      B200_CHECK(fb_batch(st, h->fbg, h->fbs, h->fb_chunk(), h->d_gray,
                          b->prev_gray ? h->d_prev_gray : cont ? h->cy.img : nullptr, F, rows, cols, h->d_flow,
                          &h->launches));
    if (masked) B200_CHECK(h->mask_filter(dflow, b->binary_threshold, kpd16, 0, F));
  }
  B200_CHECK(h->run(dd, kpd16, b->depth_factor, dT, F, cont));
  if (cont) B200_CUDA(cudaEventRecord(h->carry_free_ev, st));   // the last read of the carry
  if (!b->device) {
    B200_CUDA(cudaEventRecord(h->compute_done_ev, st));
    B200_CHECK(download(h, out, F));
  }
  h->last = BatchRecord{F, rows, cols, kcap, batch_variant(b), std::min(2, s + F), b->device ? b->Tcw : nullptr, h->prm};
  return B200ORB_OK;
}

// The dynamic mask of frame `frame` of the last batch, if that batch was masked: FrameDrawer's mDynMask
// (perfect/src/FrameDrawer.cc:262), unpacked to one byte per pixel, and whether the 65 % rule filtered the frame.
int orbs_read_dynamic_mask(orbs_t* h, int frame, uint8_t* mask, int* filtered) {
  B200_CHECK(check_last(h, frame, MASKED_BATCH));
  DeviceGuard g(h->device);
  const int rows = h->last.rows, cols = h->last.cols, nw = dynp_words(cols);
  std::vector<uint32_t> words((size_t)rows * nw);
  unsigned sum = 0;
  cudaStream_t st = h->ex->stream;
  B200_CUDA(cudaMemcpyAsync(words.data(), h->d_plane + (size_t)frame * rows * nw, words.size() * 4, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaMemcpyAsync(&sum, h->d_msum + frame, 4, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  if (mask)
    for (int y = 0; y < rows; ++y)
      for (int x = 0; x < cols; ++x) mask[(size_t)y * cols + x] = (words[(size_t)y * nw + (x >> 5)] >> (x & 31)) & 1u;
  if (filtered) *filtered = (double)sum > (double)(rows * cols) * 0.65;
  return B200ORB_OK;
}

// What TrackHomo did for frame `frame` of the last batch, if that batch was a homography batch.
int orbs_read_homography(orbs_t* h, int frame, double H[9], int* branch, int* nmatches, int* npairs) {
  B200_CHECK(check_last(h, frame, HOMO_BATCH));
  DeviceGuard g(h->device);
  int st[HC_WORDS];
  double out[10];
  cudaStream_t s = h->ex->stream;
  B200_CUDA(cudaMemcpyAsync(st, h->d_hstate + (size_t)frame * HC_WORDS, sizeof(st), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaMemcpyAsync(out, h->d_hout + (size_t)frame * 10, sizeof(out), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  if (H)
    for (int i = 0; i < 9; ++i) H[i] = out[i];
  if (branch) *branch = st[HC_BRANCH];
  if (nmatches) *nmatches = st[HC_NMATCH];
  if (npairs) *npairs = st[HC_NPAIRS];
  return B200ORB_OK;
}

// frames per upload chunk of host batches (default 128; at most MAX_CHUNKS per call): smaller chunks start the
// extraction earlier, larger ones keep the launches wider
int orbs_set_chunk_frames(orbs_t* h, int frames) {
  if (!h || frames <= 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  h->chunk_frames = frames;
  return B200ORB_OK;
}

// The next host batch submitted to `h` starts its kernels only when the kernels of `prev`'s last submitted batch
// are done, and its uploads only when `prev`'s in-place depth reads are done.  Two handles submitted alternately with this form a 3-stage pipeline:
// upload of batch k+1 | kernels of batch k | download of batch k-1.
int orbs_chain_after(orbs_t* h, orbs_t* prev) {
  if (!h || !prev || h == prev || h->device != prev->device) { set_error("bad argument"); return B200ORB_EINVAL; }
  h->chain_prev = prev;
  return B200ORB_OK;
}

// h's next batch continues the sequence of prev's last batch: its last frame P is copied into h's carry on prev's
// stream, behind that batch and before anything submitted to prev later.  The copy waits for h's last batch that read the
// carry and for a continuation still pending on h; h's next batch waits for the copy.
int orbs_continue(orbs_t* h, orbs_t* prev) {
  if (!h || !prev || h->device != prev->device) { set_error("bad argument"); return B200ORB_EINVAL; }
  B200_CHECK(check_last(prev, 0, ANY_BATCH));
  DeviceGuard g(h->device);
  const BatchRecord& p = prev->last;
  const bool img = p.variant == BV_DEVICE_FLOW || p.variant == BV_HOMOGRAPHY;
  B200_CHECK(h->ensure_carry(p.rows, p.cols, p.cap, img));
  cudaStream_t ps = prev->ex->stream;
  B200_CUDA(cudaStreamWaitEvent(ps, h->carry_free_ev, 0));
  if (h->cont.pending) B200_CUDA(cudaStreamWaitEvent(ps, h->carry_ev, 0));
  const int f = p.F - 1;
  const size_t o = (size_t)f * p.cap, px = (size_t)p.rows * p.cols;
  const CarrySrc src{prev->d_x + o, prev->d_y + o, prev->d_ang + o, prev->d_xw + 3 * o, prev->d_oct + o, prev->d_valid + o,
                     prev->ex->d_desc + 32 * o, prev->ex->d_n + f, (p.dT ? p.dT : prev->d_T) + 16 * (size_t)f};
  const bool homo = p.variant == BV_HOMOGRAPHY;
  k_carry_gather<<<dim3(CARRY_CTAS, img ? 2 : 1), 256, 0, ps>>>(
      src, img ? prev->d_gray + f * px : nullptr, homo ? prev->d_dest : nullptr,
      homo ? prev->d_hstate + f * HC_WORDS + HC_WARP : nullptr, px, h->cy);
  ++h->launches;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaEventRecord(h->carry_ev, ps));
  h->cont.pending = true;
  h->cont.from = p;
  return B200ORB_OK;
}

int orbs_sync(orbs_t* h) {
  if (!h) return B200ORB_EINVAL;
  DeviceGuard g(h->device);
  B200_CUDA(cudaStreamSynchronize(h->ex->stream));
  return B200ORB_OK;
}
void* orbs_stream(orbs_t* h) { return h ? (void*)(cudaStream_t)h->ex->stream : nullptr; }
long long orbs_launch_count(const orbs_t* h) { return h ? h->launches + h->ex->launches : 0; }
orbx_t* orbs_extractor(orbs_t* h) { return h ? h->ex.get() : nullptr; }

}  // extern "C"
