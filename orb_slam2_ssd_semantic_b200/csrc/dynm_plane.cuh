// dynm_plane.cuh -- Flow::ComputeMask + the masked RGB-D Frame constructor's keypoint loop (perfect/src/Flow.cc:24-47,
// perfect/src/Frame.cc:356-377) on bit planes: the stages as device functions of one mask word or one chunk of keypoints,
// whoever drives them.  Two drivers, both in dynm.cu: k_dynm_plane_filter (the batch tracker, orbs.cu, launches it through
// launch_dynm_plane_filter below between extraction and the frame glue: one CTA per frame, both planes in shared memory)
// and the per-stage dynm_* entries (grid-wide launches over planes in global memory).
#pragma once
#include "common.cuh"

namespace b200 {

// One row-pass value of cv::pyrUp (pyrUp_<FltCast<float,6>>) at output column X of a source row; `row` points at the
// channel's first element, consecutive pixels are `cn` floats apart.  w >= 2.
__device__ __forceinline__ float pyrup_row(const float* __restrict__ row, int X, int w, int cn) {
  const int x = X >> 1;
  const float x0 = row[(size_t)x * cn];
  if ((X & 1) == 0) {
    if (x == 0) return __fadd_rn(__fmul_rn(x0, 6.f), __fmul_rn(row[cn], 2.f));
    if (x == w - 1) return __fadd_rn(row[(size_t)(x - 1) * cn], __fmul_rn(x0, 7.f));
    return __fadd_rn(__fadd_rn(__fmul_rn(x0, 6.f), row[(size_t)(x - 1) * cn]), row[(size_t)(x + 1) * cn]);
  }
  if (x == w - 1) return __fmul_rn(x0, 8.f);
  return __fmul_rn(__fadd_rn(x0, row[(size_t)(x + 1) * cn]), 4.f);
}

__device__ __forceinline__ float pyrup_at(const float* __restrict__ src, int X, int Y, int w, int h, int cn, int c) {
  const int y = Y >> 1;
  const size_t rs = (size_t)w * cn;
  const int yn = (y + 1 < h) ? y + 1 : h - 1;   // borderInterpolate(2 (y+1), 2 h, REFLECT_101) / 2
  const float r1 = pyrup_row(src + (size_t)y * rs + c, X, w, cn);
  const float r2 = pyrup_row(src + (size_t)yn * rs + c, X, w, cn);
  if ((Y & 1) == 0) {
    const int yp = (y > 0) ? y - 1 : 1;
    const float r0 = pyrup_row(src + (size_t)yp * rs + c, X, w, cn);
    return __fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(r1, 6.f), r0), r2), 0.015625f);
  }
  return __fmul_rn(__fmul_rn(__fadd_rn(r1, r2), 4.f), 0.015625f);
}

// EINVAL (with a message) unless the flow field is at least 2 x 2 and the mask_rows x mask_cols mask belongs to it.
int dynm_check_geometry(int rows, int cols, int mask_rows, int mask_cols);

// ---- bit planes ------------------------------------------------------------------------------------------------------
// A mask of H x W pixels is H rows of NW = ceil(W / 32) words; bit j of word k of a row is pixel 32 k + j.  `last` masks
// the bits of a row's last word that lie inside the image.  The tracker's CTA of a frame holds two planes (ping-pong) plus
// the scan scratch, all dynamic shared memory:
constexpr int DYNP_THREADS = 512;
__host__ __device__ constexpr int dynp_words(int W) { return (W + 31) >> 5; }
__host__ __device__ constexpr uint32_t dynp_last(int W) { return (W & 31) ? ((1u << (W & 31)) - 1u) : 0xffffffffu; }
__host__ __device__ constexpr size_t dynp_smem_bytes(int H, int W) { return ((size_t)2 * H * dynp_words(W) + 33) * 4; }

// The 21 x 21 MORPH_ELLIPSE of perfect/src/Flow.cc:39-41, cv::getStructuringElement's row dy spanning dx = -hw .. hw with
// hw = cvRound(r sqrt((r^2 - dy^2) / r^2)), r = 10: the half width of the rows |dy| = 0..10 (pinned to cv2 by
// test_element_matches_cv2 through dynm_element).
constexpr int DYNM_R = 10;
constexpr int DYNM_K = 2 * DYNM_R + 1;
constexpr int DYNM_HALF_WIDTH[DYNM_R + 1] = {10, 10, 10, 10, 9, 9, 8, 7, 6, 4, 0};

// Band b of the decomposition takes the rows |dy| <= dynp_band(b), whose half widths are all >= dynp_width(b).  Erosion =
// AND over b of H_width(b)(AND of the band's rows), H_w = the horizontal erosion by w: exact, because H_w distributes over
// AND and a row's own (wider) erosion is contained in H_w of it, provided every row's half width is that of the widest
// band containing it.  Dilation likewise with OR.
__host__ __device__ constexpr int dynp_band(int b) { return b == 0 ? 3 : 4 + b; }
__host__ __device__ constexpr int dynp_width(int b) { return b == 0 ? 10 : b == 1 ? 9 : b == 6 ? 0 : b == 5 ? 4 : 10 - b; }
constexpr bool dynp_bands_are_the_ellipse() {
  if (dynp_band(6) != DYNM_R) return false;
  for (int b = 1; b < 7; ++b)
    if (dynp_band(b) <= dynp_band(b - 1) || dynp_width(b) >= dynp_width(b - 1)) return false;
  for (int d = 0, b = 0; d <= DYNM_R; ++d) {
    while (dynp_band(b) < d) ++b;   // the first band holding row d is its widest
    if (DYNM_HALF_WIDTH[d] != dynp_width(b)) return false;
  }
  return true;
}
static_assert(dynp_bands_are_the_ellipse(), "the 7 bands must decompose the 21 x 21 ellipse exactly");

// Threshold loop of Flow::ComputeMask (:24-41) at pixel (X, Y) of an H x W mask row, W the row's width: pyrUp of the
// half-resolution flow fl (h x w x 2 f32), 1 where x*x + y*y < thr (NaN: 0).  Pixels beyond the 2h x 2w the up-sampled
// flow covers keep the initial 1 (:25), and so do bits beyond W: the padding of the first erosion.  The caller packs a
// warp's 32 pixels into a word with __ballot_sync.
__device__ __forceinline__ bool dynp_threshold(const float* __restrict__ fl, int h, int w, float thr, int X, int Y, int W) {
  if (X >= W || X >= 2 * w || Y >= 2 * h) return true;
  const float fx = pyrup_at(fl, X, Y, w, h, 2, 0), fy = pyrup_at(fl, X, Y, w, h, 2, 1);
  return __fadd_rn(__fmul_rn(fx, fx), __fmul_rn(fy, fy)) < thr;
}

// Word wx of row y of one erode (ERODE) or dilate pass over the H x nw plane src (shared or global memory).  Outside pixels
// never win (cv's default border): rows outside the image are skipped, the words left and right of a row read as PAD, and
// the bits beyond W in a row's last word hold PAD of the pass that reads them -- OUT_ONES sets them for a following
// erosion, else they are cleared.
template <bool ERODE, bool OUT_ONES>
__device__ __forceinline__ uint32_t dynp_morph_word(const uint32_t* __restrict__ src, int y, int wx, int H, int nw,
                                                    uint32_t last) {
  constexpr uint32_t PAD = ERODE ? 0xffffffffu : 0u;   // also the identity of the combine
  uint32_t l = PAD, c = PAD, r = PAD, acc = PAD;
#pragma unroll
  for (int b = 0; b < 7; ++b) {
#pragma unroll
    for (int d = (b == 0 ? 0 : dynp_band(b - 1) + 1); d <= dynp_band(b); ++d) {
#pragma unroll
      for (int sgn = 0; sgn < (d ? 2 : 1); ++sgn) {
        const int yy = sgn ? y - d : y + d;
        if (yy < 0 || yy >= H) continue;
        const uint32_t* s = src + yy * nw + wx;
        const uint32_t vl = wx > 0 ? s[-1] : PAD, vc = s[0], vr = wx + 1 < nw ? s[1] : PAD;
        if (ERODE) { l &= vl; c &= vc; r &= vr; } else { l |= vl; c |= vc; r |= vr; }
      }
    }
    uint32_t hm = c;
#pragma unroll
    for (int k = 1; k <= dynp_width(b); ++k) {   // pixel x + k and pixel x - k at bit x
      const uint32_t t = ERODE ? (__funnelshift_r(c, r, k) & __funnelshift_l(l, c, k))
                               : (__funnelshift_r(c, r, k) | __funnelshift_l(l, c, k));
      hm = ERODE ? (hm & t) : (hm | t);
    }
    acc = ERODE ? (acc & hm) : (acc | hm);
  }
  if (wx == nw - 1) acc = OUT_ONES ? (acc | ~last) : (acc & last);
  return acc;
}

// The keypoint loop of the masked constructor (perfect/src/Frame.cc:358-375) on frame f in the extractor's [F][cap]
// layout: the first n keypoints (n = min(counts[f], cap), read by the caller before any barrier) for which
// keep(y, x) holds, (y, x) = imMask.at<uchar>(pt.y, pt.x)'s pixel (float -> int truncation, clamped into the rows x cols
// mask), are compacted in place, order kept, with their descriptors and, when kpd16 is given, the CV_16U depth gathered
// under them; counts[f] becomes their number.  Called by all DYNP_THREADS threads of the CTA; ws = 33 ints of shared
// scratch.  In place is safe: each chunk of DYNP_THREADS keypoints is read before the scan's barriers and written after
// them, to positions at or below its own, so no later chunk's input is overwritten.
template <class Keep>
__device__ __forceinline__ void dynp_compact(int f, int n, int cap, int rows, int cols, OrbxKeyPoint* __restrict__ kps,
                                             uint8_t* __restrict__ desc, uint16_t* __restrict__ kpd16,
                                             int* __restrict__ counts, int* ws, Keep keep) {
  OrbxKeyPoint* k = kps + (size_t)f * cap;
  uint4* d = reinterpret_cast<uint4*>(desc + (size_t)f * cap * 32);
  uint16_t* z = kpd16 ? kpd16 + (size_t)f * cap : nullptr;
  int base = 0;
  for (int i0 = 0; i0 < n; i0 += DYNP_THREADS) {
    const int i = i0 + threadIdx.x;
    bool kept = false;
    OrbxKeyPoint kp;
    uint4 d0, d1;
    uint16_t dz = 0;
    if (i < n) {
      kp = k[i];
      d0 = d[2 * (size_t)i];
      d1 = d[2 * (size_t)i + 1];
      if (z) dz = z[i];
      kept = keep(min(max((int)kp.y, 0), rows - 1), min(max((int)kp.x, 0), cols - 1));
    }
    int tot;
    const int pos = base + block_excl_scan(kept ? 1 : 0, ws, &tot);
    if (kept) {
      k[pos] = kp;
      d[2 * (size_t)pos] = d0;
      d[2 * (size_t)pos + 1] = d1;
      if (z) z[pos] = dz;
    }
    base += tot;
  }
  if (threadIdx.x == 0) counts[f] = base;
}

// One erode or dilate pass over the tracker CTA's plane: dst = the pass of src, also copied to gdst when given.  Returns
// this thread's popcount of what it wrote.
template <bool ERODE, bool OUT_ONES>
__device__ __forceinline__ unsigned plane_morph(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, int H, int nw,
                                                uint32_t last, uint32_t* __restrict__ gdst) {
  unsigned pop = 0;
  for (int it = threadIdx.x; it < H * nw; it += blockDim.x) {
    const int y = it / nw;
    const uint32_t acc = dynp_morph_word<ERODE, OUT_ONES>(src, y, it - y * nw, H, nw, last);
    dst[it] = acc;
    if (gdst) gdst[it] = acc;
    pop += __popc(acc);
  }
  return pop;
}

// One CTA per frame f of F frames of a batch, after extraction (k_dynm_plane_filter, dynm.cu): threshold, erode, erode,
// dilate of the half-resolution flow [F][h][w][2] into two bit planes in shared memory; the final plane goes to planes[f]
// (H x dynp_words(W) words) and its popcount, cv::sum(mask), to sums[f]; then the masked constructor's filter, in place on
// the extractor's [F][cap] outputs (kps, desc, counts and, when given, kpd16).  Sets the kernel's dynamic shared memory
// to dynp_smem_bytes(H, W), which the caller has checked against the device.
int launch_dynm_plane_filter(int F, const float* flow, int h, int w, float thr, int H, int W, uint32_t* planes, unsigned* sums,
                             OrbxKeyPoint* kps, uint8_t* desc, uint16_t* kpd16, int* counts, int cap, cudaStream_t stream,
                             long long* launches);

}  // namespace b200
