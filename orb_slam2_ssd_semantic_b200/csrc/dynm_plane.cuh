// dynm_plane.cuh -- Flow::ComputeMask + the masked RGB-D Frame constructor's keypoint loop (perfect/src/Flow.cc:24-47,
// perfect/src/Frame.cc:356-377) for whole batches, one CTA per frame on bit planes in shared memory; the batch tracker
// (orbs.cu) runs it between extraction and the frame glue.  pyrup_row / pyrup_at and dynm_check_geometry are shared with
// the per-stage dynm_* entries (dynm.cu).
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

static int dynm_check_geometry(int rows, int cols, int mask_rows, int mask_cols) {
  if (rows < 2 || cols < 2) { set_error("flow field smaller than 2x2"); return B200ORB_EINVAL; }
  if (mask_rows < 2 * rows || mask_rows > 2 * rows + 1 || mask_cols < 2 * cols || mask_cols > 2 * cols + 1) {
    set_error("mask %dx%d does not belong to a %dx%d flow field (the gray image is 2 rows (+1) x 2 cols (+1))", mask_cols,
              mask_rows, cols, rows);
    return B200ORB_EINVAL;
  }
  return B200ORB_OK;
}

// ---- bit planes ------------------------------------------------------------------------------------------------------
// A mask of H x W pixels is H rows of NW = ceil(W / 32) words; bit j of word k of a row is pixel 32 k + j.  The CTA of a
// frame holds two planes (ping-pong) plus the scan scratch, all dynamic shared memory:
constexpr int DYNP_THREADS = 512;
__host__ __device__ constexpr int dynp_words(int W) { return (W + 31) >> 5; }
__host__ __device__ constexpr size_t dynp_smem_bytes(int H, int W) { return ((size_t)2 * H * dynp_words(W) + 33) * 4; }

// The 21 x 21 MORPH_ELLIPSE (dynm_create's table, perfect/src/Flow.cc:39-41) has half widths 10,10,10,10,9,9,8,7,6,4,0 for
// |dy| = 0..10: band b of the decomposition takes the rows |dy| <= dynp_band(b), whose half widths are all
// >= dynp_width(b).  Erosion = AND over b of H_width(b)(AND of the band's rows), H_w = the horizontal erosion by w: exact,
// because H_w distributes over AND and a row's own (wider) erosion is contained in H_w of it.  Dilation likewise with OR.
__host__ __device__ constexpr int dynp_band(int b) { return b == 0 ? 3 : 4 + b; }
__host__ __device__ constexpr int dynp_width(int b) { return b == 0 ? 10 : b == 1 ? 9 : b == 6 ? 0 : b == 5 ? 4 : 10 - b; }

// One erode (ERODE) or dilate pass src -> dst over the whole plane.  Outside pixels never win (cv's default border): rows
// outside the image are skipped, the words left and right of a row read as PAD, and the bits beyond W in a row's last
// word hold PAD of the pass that reads them -- OUT_ONES sets them in dst for a following erosion, else they are cleared.
// Returns this thread's popcount of what it wrote.
template <bool ERODE, bool OUT_ONES>
__device__ __forceinline__ unsigned plane_morph(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, int H, int nw,
                                                uint32_t last, uint32_t* __restrict__ gdst) {
  constexpr uint32_t PAD = ERODE ? 0xffffffffu : 0u;   // also the identity of the combine
  unsigned pop = 0;
  for (int it = threadIdx.x; it < H * nw; it += blockDim.x) {
    const int y = it / nw, wx = it - y * nw;
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
    dst[it] = acc;
    if (gdst) gdst[it] = acc;
    pop += __popc(acc);
  }
  return pop;
}

// One CTA per frame f of a batch, after extraction:
//   threshold  pyrUp of the half-resolution flow (h x w x 2 f32), bit = x*x + y*y < thr (NaN: 0); pixels beyond the 2h x 2w
//              the up-sampled flow covers keep 1 (:25); __ballot_sync packs a warp's 32 pixels into one word
//   morphology erode, erode, dilate on the planes; the final plane goes to planes[f] (H x NW words), its popcount to sums[f]
//   filter     cv::sum(mask) > rows*cols*0.65 -> keep the keypoints whose pixel is 1, order kept, compacted in place in
//              the extractor's [F][cap] layout (keypoints, descriptors, counts and, when given, the CV_16U depth gathered
//              under each keypoint).  Each chunk of DYNP_THREADS keypoints is read before the scan's barriers and written
//              after them, to positions at or below its own, so no later chunk's input is overwritten.
__global__ void __launch_bounds__(DYNP_THREADS, 2) k_dynm_plane_filter(const float* __restrict__ flow, int h, int w, float thr,
                                                                     int H, int W, uint32_t* __restrict__ planes,
                                                                     unsigned* __restrict__ sums, OrbxKeyPoint* __restrict__ kps,
                                                                     uint8_t* __restrict__ desc, uint16_t* __restrict__ kpd16,
                                                                     int* __restrict__ counts, int cap) {
  extern __shared__ uint32_t dynp_sm[];
  const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const int nw = dynp_words(W), nwords = H * nw;
  uint32_t* A = dynp_sm;
  uint32_t* B = dynp_sm + nwords;
  int* ws = reinterpret_cast<int*>(dynp_sm + 2 * nwords);
  const uint32_t last = (W & 31) ? ((1u << (W & 31)) - 1u) : 0xffffffffu;
  const int n = min(counts[f], cap);
  const float* fl = flow + (size_t)f * h * w * 2;
  for (int it = tid >> 5; it < nwords; it += DYNP_THREADS / 32) {
    const int Y = it / nw, X = (it - Y * nw) * 32 + lane;
    bool m = true;   // beyond W: the erosion's padding
    if (X < W && X < 2 * w && Y < 2 * h) {
      const float fx = pyrup_at(fl, X, Y, w, h, 2, 0), fy = pyrup_at(fl, X, Y, w, h, 2, 1);
      m = __fadd_rn(__fmul_rn(fx, fx), __fmul_rn(fy, fy)) < thr;
    }
    const uint32_t bits = __ballot_sync(0xffffffffu, m);
    if (lane == 0) A[it] = bits;
  }
  __syncthreads();
  plane_morph<true, true>(A, B, H, nw, last, nullptr);
  __syncthreads();
  plane_morph<true, false>(B, A, H, nw, last, nullptr);
  __syncthreads();
  const unsigned pop = plane_morph<false, false>(A, B, H, nw, last, planes + (size_t)f * nwords);
  int total;
  block_excl_scan((int)pop, ws, &total);   // its barriers also publish B
  if (tid == 0) sums[f] = (unsigned)total;
  const bool filter = (double)total > (double)(H * W) * 0.65;   // perfect/src/Frame.cc:358, as k_dynm_filter decides
  OrbxKeyPoint* k = kps + (size_t)f * cap;
  uint4* d = reinterpret_cast<uint4*>(desc + (size_t)f * cap * 32);
  uint16_t* z = kpd16 ? kpd16 + (size_t)f * cap : nullptr;
  int base = 0;
  for (int i0 = 0; i0 < n; i0 += DYNP_THREADS) {
    const int i = i0 + tid;
    bool keep = false;
    OrbxKeyPoint kp;
    uint4 d0, d1;
    uint16_t dz = 0;
    if (i < n) {
      kp = k[i];
      d0 = d[2 * (size_t)i];
      d1 = d[2 * (size_t)i + 1];
      if (z) dz = z[i];
      // imMask.at<uchar>(pt.y, pt.x) with k_dynm_filter's clamped truncation
      const int yy = min(max((int)kp.y, 0), H - 1), xx = min(max((int)kp.x, 0), W - 1);
      keep = !filter || ((B[yy * nw + (xx >> 5)] >> (xx & 31)) & 1u);
    }
    int tot;
    const int pos = base + block_excl_scan(keep ? 1 : 0, ws, &tot);
    if (keep) {
      k[pos] = kp;
      d[2 * (size_t)pos] = d0;
      d[2 * (size_t)pos + 1] = d1;
      if (z) z[pos] = dz;
    }
    base += tot;
  }
  if (tid == 0) counts[f] = base;
}

}  // namespace b200
