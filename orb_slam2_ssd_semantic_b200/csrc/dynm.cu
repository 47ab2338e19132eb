// dynm.cu -- the dynamic-mask stages of the `perfect` variant (SURVEY §8(f4), the parts that are plain image arithmetic):
//   * FlowSLAM::Flow::ComputeMask after calcOpticalFlowFarneback (perfect/src/Flow.cc:29-49): pyrUp of the half-resolution
//     flow field, mask = 0 where |flow|^2 >= max(threshold, 40), then erode, erode, dilate with the 21x21 MORPH_ELLIPSE
//     element;
//   * the masked RGB-D Frame constructor (perfect/src/Frame.cc:356-377): when more than 65 % of the mask is 1, keypoints
//     whose pixel is not 1 are dropped (with their descriptors), order kept.
// The dense optical flow itself (pyrDown + OpenCV's Farneback) is flow.cu's, behind dynm_farneback and
// dynm_flow_batch_device below.  Everything here is bit-exact with cv2 too: cv::pyrUp's float sequence
// (row pass: x*6 + left + right / (x + right)*4, reflect-101 on the left / top, replicate on the right / bottom; column
// pass the same, times 1/64) and cv::erode / cv::dilate with the default border (outside pixels are ignored) were pinned
// against cv2 4.13 (tools/make_dynmask_golden.py -> tests/golden/dynmask_*.npz).
#include <stdlib.h>

#include <memory>
#include <new>

#include "dynm.cuh"
#include "dynm_plane.cuh"
#include "flow.cuh"

namespace b200 {

// The per-stage entries drive dynm_plane.cuh's functions with grid-wide launches over two global-memory bit planes per
// frame, so they take any geometry; the tracker's one-CTA-per-frame kernel is bound by shared memory.  blockIdx.y = frame.

// threshold -> plane, one warp per word
__global__ void __launch_bounds__(256) k_dynm_threshold(const float* __restrict__ flow, int h, int w, float thr, int H, int W,
                                                        uint32_t* __restrict__ planes) {
  const int nw = dynp_words(W), it = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (it >= H * nw) return;   // whole warps
  const int Y = it / nw, X = (it - Y * nw) * 32 + lane;
  const uint32_t bits = __ballot_sync(0xffffffffu, dynp_threshold(flow + (size_t)blockIdx.y * h * w * 2, h, w, thr, X, Y, W));
  if (lane == 0) planes[(size_t)blockIdx.y * H * nw + it] = bits;
}

// erode plane src -> plane dst, one thread per word
template <bool OUT_ONES>
__global__ void __launch_bounds__(256) k_dynm_erode(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, int H, int W) {
  const int nw = dynp_words(W), it = blockIdx.x * 256 + threadIdx.x;
  if (it >= H * nw) return;
  const size_t o = (size_t)blockIdx.y * H * nw;
  const int y = it / nw;
  dst[o + it] = dynp_morph_word<true, OUT_ONES>(src + o, y, it - y * nw, H, nw, dynp_last(W));
}

// dilate plane src -> the caller's H x W byte mask, one thread per word; lane j then stores bit j of each of its warp's 32
// words in turn, so a store covers 32 consecutive pixels
__global__ void __launch_bounds__(256) k_dynm_dilate_unpack(const uint32_t* __restrict__ src, uint8_t* __restrict__ mask, int H,
                                                            int W) {
  const int nw = dynp_words(W), nwords = H * nw, it = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31;
  src += (size_t)blockIdx.y * nwords;
  mask += (size_t)blockIdx.y * H * W;
  uint32_t word = 0;
  if (it < nwords) {
    const int y = it / nw;
    word = dynp_morph_word<false, false>(src, y, it - y * nw, H, nw, dynp_last(W));
  }
  for (int k = 0, ik = it - lane; k < 32 && ik < nwords; ++k, ++ik) {   // ik is warp-uniform
    const uint32_t wk = __shfl_sync(0xffffffffu, word, k);
    const int y = ik / nw, X = (ik - y * nw) * 32 + lane;
    if (X < W) mask[(size_t)y * W + X] = (wk >> lane) & 1u;
  }
}

// The masked constructor (perfect/src/Frame.cc:357-375) on frame f = blockIdx.x: cv::sum(imMask) of the caller's bytes, in
// 64 bits (every byte counts by its value), then the keypoints whose pixel is exactly 1 are kept, in place.
__global__ void __launch_bounds__(DYNP_THREADS) k_dynm_filter(const uint8_t* __restrict__ mask, int rows, int cols,
                                                              OrbxKeyPoint* __restrict__ kps, uint8_t* __restrict__ desc,
                                                              int* __restrict__ counts, int cap) {
  __shared__ int ws[33];
  __shared__ unsigned long long part[DYNP_THREADS / 32];
  const int f = blockIdx.x, tid = threadIdx.x;
  const int n = min(counts[f], cap);
  const size_t npx = (size_t)rows * cols;
  const uint8_t* m = mask + (size_t)f * npx;
  const size_t head = min(npx, (size_t)(-(uintptr_t)m & 15)), nv = (npx - head) / 16;   // bytes before the first uint4
  const uint4* v = reinterpret_cast<const uint4*>(m + head);
  unsigned long long s = tid < head ? m[tid] : 0;
  for (size_t i = tid; i < nv; i += DYNP_THREADS) {
    const uint4 q = v[i];
    const unsigned one = 0x01010101u;
    s += __dp4a(q.x, one, __dp4a(q.y, one, __dp4a(q.z, one, __dp4a(q.w, one, 0u))));
  }
  for (size_t i = head + nv * 16 + tid; i < npx; i += DYNP_THREADS) s += m[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) part[tid >> 5] = s;
  __syncthreads();
  s = 0;
#pragma unroll
  for (int i = 0; i < DYNP_THREADS / 32; ++i) s += part[i];
  const bool filter = (double)s > (double)(rows * cols) * 0.65;   // :358
  dynp_compact(f, n, cap, rows, cols, kps, desc, nullptr, counts, ws,
               [&](int y, int x) { return !filter || m[(size_t)y * cols + x] == 1; });
}

// One CTA per frame f of a batch, after extraction: threshold into plane A, erode, erode, dilate between A and B; the final
// plane also goes to planes[f] (H x NW words) and its popcount, cv::sum(mask), to sums[f]; then the masked constructor's
// filter, in place on the extractor's outputs.
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
  const uint32_t last = dynp_last(W);
  const int n = min(counts[f], cap);
  const float* fl = flow + (size_t)f * h * w * 2;
  for (int it = tid >> 5; it < nwords; it += DYNP_THREADS / 32) {
    const int Y = it / nw, X = (it - Y * nw) * 32 + lane;
    const uint32_t bits = __ballot_sync(0xffffffffu, dynp_threshold(fl, h, w, thr, X, Y, W));
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
  const bool filter = (double)total > (double)(H * W) * 0.65;   // perfect/src/Frame.cc:358
  dynp_compact(f, n, cap, H, W, kps, desc, kpd16, counts, ws,
               [&](int y, int x) { return !filter || ((B[y * nw + (x >> 5)] >> (x & 31)) & 1u); });
}

int launch_dynm_plane_filter(int F, const float* flow, int h, int w, float thr, int H, int W, uint32_t* planes, unsigned* sums,
                             OrbxKeyPoint* kps, uint8_t* desc, uint16_t* kpd16, int* counts, int cap, cudaStream_t stream,
                             long long* launches) {
  const size_t smem = dynp_smem_bytes(H, W);
  B200_CUDA(cudaFuncSetAttribute(k_dynm_plane_filter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_dynm_plane_filter<<<F, DYNP_THREADS, smem, stream>>>(flow, h, w, thr, H, W, planes, sums, kps, desc, kpd16, counts, cap);
  ++*launches;
  B200_CUDA(cudaGetLastError());
  return B200ORB_OK;
}

int dynm_check_geometry(int rows, int cols, int mask_rows, int mask_cols) {
  if (rows < 2 || cols < 2) { set_error("flow field smaller than 2x2"); return B200ORB_EINVAL; }
  if (mask_rows < 2 * rows || mask_rows > 2 * rows + 1 || mask_cols < 2 * cols || mask_cols > 2 * cols + 1) {
    set_error("mask %dx%d does not belong to a %dx%d flow field (the gray image is 2 rows (+1) x 2 cols (+1))", mask_cols,
              mask_rows, cols, rows);
    return B200ORB_EINVAL;
  }
  return B200ORB_OK;
}

}  // namespace b200

using namespace b200;

// device core of ComputeMask: d_flow [F][rows][cols][2] -> d_mask [F][H][W]; d_planes = 2 F H ceil(W / 32) words
static int dynm_mask_core(dynm* h, const float* d_flow, int F, int rows, int cols, float thr, uint8_t* d_mask,
                          uint32_t* d_planes, int H, int W) {
  const int nwords = H * dynp_words(W);
  uint32_t *A = d_planes, *B = d_planes + (size_t)F * nwords;
  const dim3 words((nwords + 255) / 256, F);
  if (thr < 40.0f) thr = 40.0f;   // :24
  k_dynm_threshold<<<dim3((nwords + 7) / 8, F), 256, 0, h->stream>>>(d_flow, rows, cols, thr, H, W, A);
  k_dynm_erode<true><<<words, 256, 0, h->stream>>>(A, B, H, W);
  k_dynm_erode<false><<<words, 256, 0, h->stream>>>(B, A, H, W);
  k_dynm_dilate_unpack<<<words, 256, 0, h->stream>>>(A, d_mask, H, W);
  h->launches += 4;
  B200_CUDA(cudaGetLastError());
  return B200ORB_OK;
}

static int dynm_filter_core(dynm* h, const uint8_t* d_mask, int F, int rows, int cols, OrbxKeyPoint* d_kps, uint8_t* d_desc,
                            int32_t* d_counts, int cap) {
  k_dynm_filter<<<F, DYNP_THREADS, 0, h->stream>>>(d_mask, rows, cols, d_kps, d_desc, d_counts, cap);
  h->launches += 1;
  B200_CUDA(cudaGetLastError());
  return B200ORB_OK;
}

extern "C" {

int dynm_create(int device, dynm_t** out) {
  if (!out) { set_error("bad argument"); return B200ORB_EINVAL; }
  *out = nullptr;
  B200_CHECK(check_device(device));
  DeviceGuard g(device);
  std::unique_ptr<dynm> h(new (std::nothrow) dynm());
  if (!h) { set_error("out of host memory"); return B200ORB_EINVAL; }
  h->device = device;
  B200_CHECK(h->stream.create());
  *out = h.release();
  return B200ORB_OK;
}
void dynm_destroy(dynm_t* h) { destroy_handle(h); }
long long dynm_launch_count(const dynm_t* h) { return h ? h->launches : 0; }
void* dynm_stream(dynm_t* h) { return h ? (void*)(cudaStream_t)h->stream : nullptr; }
int dynm_sync(dynm_t* h) {
  if (!h) { set_error("bad argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}
int dynm_element(const dynm_t* h, uint8_t* element /* 21 x 21 */) {
  if (!h || !element) { set_error("bad argument"); return B200ORB_EINVAL; }
  for (int i = 0; i < DYNM_K; ++i)
    for (int j = 0; j < DYNM_K; ++j) element[i * DYNM_K + j] = abs(j - DYNM_R) <= DYNM_HALF_WIDTH[abs(i - DYNM_R)] ? 1 : 0;
  return B200ORB_OK;
}

int dynm_mask_from_flow_batch_device(dynm_t* h, const float* d_flow, int nframes, int rows, int cols, float binary_threshold,
                                     uint8_t* d_mask, int mask_rows, int mask_cols) {
  if (!h || nframes < 0 || (nframes > 0 && (!d_flow || !d_mask))) { set_error("bad argument"); return B200ORB_EINVAL; }
  if (nframes == 0) return B200ORB_OK;
  B200_CHECK(dynm_check_geometry(rows, cols, mask_rows, mask_cols));
  DeviceGuard g(h->device);
  uint32_t* d_planes;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) {
    d_planes = t.take<uint32_t>((size_t)2 * nframes * mask_rows * dynp_words(mask_cols));
  }));
  return dynm_mask_core(h, d_flow, nframes, rows, cols, binary_threshold, d_mask, d_planes, mask_rows, mask_cols);
}

int dynm_mask_from_flow(dynm_t* h, const float* flow, int rows, int cols, float binary_threshold, uint8_t* mask, int mask_rows,
                        int mask_cols) {
  if (!h || !flow || !mask) { set_error("bad argument"); return B200ORB_EINVAL; }
  B200_CHECK(dynm_check_geometry(rows, cols, mask_rows, mask_cols));
  DeviceGuard g(h->device);
  float* d_flow;
  uint8_t* d_mask;
  uint32_t* d_planes;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) {
    d_flow = t.take<float>((size_t)rows * cols * 2); d_mask = t.take<uint8_t>((size_t)mask_rows * mask_cols);
    d_planes = t.take<uint32_t>((size_t)2 * mask_rows * dynp_words(mask_cols));
  }));
  B200_CUDA(cudaMemcpyAsync(d_flow, flow, (size_t)rows * cols * 8, cudaMemcpyHostToDevice, h->stream));
  B200_CHECK(dynm_mask_core(h, d_flow, 1, rows, cols, binary_threshold, d_mask, d_planes, mask_rows, mask_cols));
  B200_CUDA(cudaMemcpyAsync(mask, d_mask, (size_t)mask_rows * mask_cols, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int dynm_filter_keypoints_batch_device(dynm_t* h, const uint8_t* d_mask, int nframes, int rows, int cols, OrbxKeyPoint* d_kps,
                                       uint8_t* d_desc, int32_t* d_counts, int cap) {
  if (!h || nframes < 0 || cap < 0 || (nframes > 0 && (!d_mask || !d_kps || !d_desc || !d_counts))) {
    set_error("bad argument");
    return B200ORB_EINVAL;
  }
  if (nframes == 0 || cap == 0) return B200ORB_OK;
  if (rows < 1 || cols < 1) { set_error("empty mask"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  return dynm_filter_core(h, d_mask, nframes, rows, cols, d_kps, d_desc, d_counts, cap);
}

int dynm_filter_keypoints(dynm_t* h, const uint8_t* mask, int rows, int cols, size_t stride, OrbxKeyPoint* kps, uint8_t* desc,
                          int n, int* n_out) {
  if (!h || !n_out || n < 0 || (n > 0 && (!mask || !kps || !desc))) { set_error("bad argument"); return B200ORB_EINVAL; }
  *n_out = 0;
  if (n == 0) return B200ORB_OK;   // :379 the constructor returns on an empty frame either way
  if (rows < 1 || cols < 1 || stride < (size_t)cols) { set_error("bad mask geometry"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  uint8_t *d_mask, *d_desc;
  OrbxKeyPoint* d_kps;
  int32_t* d_cnt;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) {
    d_mask = t.take<uint8_t>((size_t)rows * cols); d_kps = t.take<OrbxKeyPoint>(n); d_desc = t.take<uint8_t>((size_t)n * 32);
    d_cnt = t.take<int32_t>(1);
  }));
  B200_CUDA(cudaMemcpy2DAsync(d_mask, cols, mask, stride, cols, rows, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_kps, kps, (size_t)n * sizeof(OrbxKeyPoint), cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_desc, desc, (size_t)n * 32, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_cnt, &n, 4, cudaMemcpyHostToDevice, h->stream));
  B200_CHECK(dynm_filter_core(h, d_mask, 1, rows, cols, d_kps, d_desc, d_cnt, n));
  int m = 0;
  B200_CUDA(cudaMemcpyAsync(&m, d_cnt, 4, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  if (m < 0 || m > n) { set_error("internal: filtered count %d of %d", m, n); return B200ORB_ECUDA; }
  B200_CUDA(cudaMemcpyAsync(kps, d_kps, (size_t)m * sizeof(OrbxKeyPoint), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(desc, d_desc, (size_t)m * 32, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  *n_out = m;
  return B200ORB_OK;
}

int dynm_farneback(dynm_t* h, const uint8_t* prev, const uint8_t* cur, int rows, int cols, float* flow) {
  if (!h || !prev || !cur || !flow) { set_error("bad argument"); return B200ORB_EINVAL; }
  FbGeom g;
  B200_CHECK(fb_geometry(rows, cols, &g));
  DeviceGuard dg(h->device);
  const size_t px = (size_t)rows * cols;
  FbScratch s;
  float* d_out;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) { fb_take(t, s, g, 1); d_out = t.take<float>(px * 2); }));
  B200_CUDA(cudaMemcpyAsync(s.half, prev, px, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(s.half + px, cur, px, cudaMemcpyHostToDevice, h->stream));
  B200_CHECK(fb_pairs(h->stream, g, s, 2, d_out, &h->launches));
  B200_CUDA(cudaMemcpyAsync(flow, d_out, px * 2 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int dynm_flow_batch_device(dynm_t* h, const uint8_t* d_gray, const uint8_t* d_prev, int nframes, int rows, int cols,
                           float* d_flow) {
  if (!h || nframes < 0 || (nframes > 0 && (!d_gray || !d_flow))) { set_error("bad argument"); return B200ORB_EINVAL; }
  FbGeom g;
  B200_CHECK(fb_geometry(rows / 2, cols / 2, &g));
  if (nframes == 0) return B200ORB_OK;
  DeviceGuard dg(h->device);
  const int C = std::min(nframes, FB_CHUNK);
  FbScratch s;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) { fb_take(t, s, g, C); }));
  return fb_batch(h->stream, g, s, C, d_gray, d_prev, nframes, rows, cols, d_flow, &h->launches);
}

}  // extern "C"
