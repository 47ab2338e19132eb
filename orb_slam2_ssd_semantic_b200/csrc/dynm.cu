// dynm.cu -- the dynamic-mask stages of the `perfect` variant (SURVEY §8(f4), the parts that are plain image arithmetic):
//   * FlowSLAM::Flow::ComputeMask after calcOpticalFlowFarneback (perfect/src/Flow.cc:29-49): pyrUp of the half-resolution
//     flow field, mask = 0 where |flow|^2 >= max(threshold, 40), then erode, erode, dilate with the 21x21 MORPH_ELLIPSE
//     element;
//   * the masked RGB-D Frame constructor (perfect/src/Frame.cc:356-377): when more than 65 % of the mask is 1, keypoints
//     whose pixel is not 1 are dropped (with their descriptors), order kept.
// The dense optical flow itself (OpenCV's Farneback) stays on the host side of the boundary: its float accumulation
// order is OpenCV's SIMD code and cannot be restated bit for bit.  Everything here can: cv::pyrUp's float sequence
// (row pass: x*6 + left + right / (x + right)*4, reflect-101 on the left / top, replicate on the right / bottom; column
// pass the same, times 1/64) and cv::erode / cv::dilate with the default border (outside pixels are ignored) were pinned
// against cv2 4.13 (tools/make_dynmask_golden.py -> tests/golden/dynmask_*.npz).
#include <math.h>

#include <memory>
#include <new>

#include "dynm_plane.cuh"   // pyrup_at, dynm_check_geometry

namespace b200 {

constexpr int DYNM_R = 10;                 // dilation_size, perfect/src/Flow.cc:39
constexpr int DYNM_K = 2 * DYNM_R + 1;     // 21 x 21 element

struct EllipseTab { int hw[DYNM_K]; };     // half width of the element's row dy + DYNM_R

// pyrUp(flow) + the threshold loop of Flow::ComputeMask (:31-41): mask = 1, 0 where x*x + y*y >= thr (NaN -> 0)
// The mask has the gray image's size H x W (2h <= H <= 2h + 1, same for W): pixels beyond flow2 keep the initial 1 (:25).
__global__ void __launch_bounds__(256) k_dynm_flow_mask(const float* __restrict__ flow, int h, int w, float thr,
                                                        uint8_t* __restrict__ mask, int H, int W) {
  const int X = blockIdx.x * 32 + (threadIdx.x & 31), Y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (X >= W || Y >= H) return;
  uint8_t m = 1;
  if (X < 2 * w && Y < 2 * h) {
    const float* f = flow + (size_t)blockIdx.z * h * w * 2;
    const float fx = pyrup_at(f, X, Y, w, h, 2, 0), fy = pyrup_at(f, X, Y, w, h, 2, 1);
    const float t2 = __fadd_rn(__fmul_rn(fx, fx), __fmul_rn(fy, fy));
    m = (t2 < thr) ? 1 : 0;
  }
  mask[(size_t)blockIdx.z * H * W + (size_t)Y * W + X] = m;
}

// cv::erode / cv::dilate with the 21x21 ellipse, anchor at the centre, default border value (pixels outside the image
// never win: +inf for erode, -inf for dilate)
template <bool ERODE>
__global__ void __launch_bounds__(256) k_dynm_morph(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int H,
                                                    int W, EllipseTab tab) {
  const int X = blockIdx.x * 32 + (threadIdx.x & 31), Y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (X >= W || Y >= H) return;
  const uint8_t* s = src + (size_t)blockIdx.z * H * W;
  int acc = ERODE ? 255 : 0;
#pragma unroll 1
  for (int dy = -DYNM_R; dy <= DYNM_R; ++dy) {
    const int yy = Y + dy;
    if (yy < 0 || yy >= H) continue;
    const int hw = tab.hw[dy + DYNM_R];
    const int x0 = max(X - hw, 0), x1 = min(X + hw, W - 1);
    const uint8_t* r = s + (size_t)yy * W;
    for (int xx = x0; xx <= x1; ++xx) {
      const int v = r[xx];
      acc = ERODE ? min(acc, v) : max(acc, v);
    }
  }
  dst[(size_t)blockIdx.z * H * W + (size_t)Y * W + X] = (uint8_t)acc;
}

// cv::sum(imMask) per frame (perfect/src/Frame.cc:357)
__global__ void __launch_bounds__(256) k_dynm_mask_sum(const uint8_t* __restrict__ mask, size_t npx,
                                                       unsigned long long* __restrict__ sums) {
  const uint8_t* m = mask + (size_t)blockIdx.y * npx;
  unsigned s = 0;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < npx; i += (size_t)gridDim.x * 256) s += m[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(&sums[blockIdx.y], (unsigned long long)s);
}

// The keypoint loop of the masked constructor (:358-375), one CTA per frame, order-preserving compaction into the
// scratch arrays.  `keep all` when the mask's sum is not above 65 % of the pixels (:358).
__global__ void __launch_bounds__(256) k_dynm_filter(const uint8_t* __restrict__ mask, int rows, int cols,
                                                     const unsigned long long* __restrict__ sums,
                                                     const OrbxKeyPoint* __restrict__ kps, const uint8_t* __restrict__ desc,
                                                     const int* __restrict__ counts, int cap,
                                                     OrbxKeyPoint* __restrict__ okps, uint8_t* __restrict__ odesc,
                                                     int* __restrict__ ocounts) {
  __shared__ int ws[33];
  const int f = blockIdx.x, tid = threadIdx.x;
  const int n = min(counts[f], cap);
  const bool filter = (double)sums[f] > (double)(rows * cols) * 0.65;
  const uint8_t* m = mask + (size_t)f * rows * cols;
  const OrbxKeyPoint* k = kps + (size_t)f * cap;
  const uint4* d = reinterpret_cast<const uint4*>(desc + (size_t)f * cap * 32);
  OrbxKeyPoint* ok = okps + (size_t)f * cap;
  uint4* od = reinterpret_cast<uint4*>(odesc + (size_t)f * cap * 32);
  int base = 0;
  for (int i0 = 0; i0 < n; i0 += 256) {
    const int i = i0 + tid;
    bool keep = false;
    OrbxKeyPoint kp;
    if (i < n) {
      kp = k[i];
      // imMask.at<uchar>(pt.y, pt.x): float -> int truncates; keypoints lie inside the image (19 <= x <= w - 20)
      const int yy = min(max((int)kp.y, 0), rows - 1), xx = min(max((int)kp.x, 0), cols - 1);
      keep = !filter || m[(size_t)yy * cols + xx] == 1;
    }
    int tot;
    const int pos = block_excl_scan(keep ? 1 : 0, ws, &tot);
    if (keep) {
      ok[base + pos] = kp;
      od[2 * (size_t)(base + pos)] = d[2 * (size_t)i];
      od[2 * (size_t)(base + pos) + 1] = d[2 * (size_t)i + 1];
    }
    base += tot;
    __syncthreads();
  }
  if (tid == 0) ocounts[f] = base;
}

}  // namespace b200

using namespace b200;

struct dynm {
  int device = 0;
  Stream stream;
  long long launches = 0;
  EllipseTab tab;
  DeviceBlock buf;   // each entry carves its buffer list out of it
};

struct FilterScratch {   // dynm_filter_core's outputs before they are copied back over the inputs
  unsigned long long* sums;
  OrbxKeyPoint* kps;
  uint8_t* desc;
  int* cnt;
  void take(Carver& c, int F, int cap) {
    sums = c.take<unsigned long long>(F); kps = c.take<OrbxKeyPoint>((size_t)F * cap);
    desc = c.take<uint8_t>((size_t)F * cap * 32); cnt = c.take<int>(F);
  }
};

// device core of ComputeMask: d_flow [F][rows][cols][2] -> d_mask [F][H][W]; d_tmp = one more set of mask planes
static int dynm_mask_core(dynm* h, const float* d_flow, int F, int rows, int cols, float thr, uint8_t* d_mask, uint8_t* d_tmp,
                          int H, int W) {
  const dim3 grd((W + 31) / 32, (H + 7) / 8, F);
  if (thr < 40.0f) thr = 40.0f;   // :24
  k_dynm_flow_mask<<<grd, 256, 0, h->stream>>>(d_flow, rows, cols, thr, d_mask, H, W);
  k_dynm_morph<true><<<grd, 256, 0, h->stream>>>(d_mask, d_tmp, H, W, h->tab);
  k_dynm_morph<true><<<grd, 256, 0, h->stream>>>(d_tmp, d_mask, H, W, h->tab);
  k_dynm_morph<false><<<grd, 256, 0, h->stream>>>(d_mask, d_tmp, H, W, h->tab);
  h->launches += 4;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(d_mask, d_tmp, (size_t)F * H * W, cudaMemcpyDeviceToDevice, h->stream));
  return B200ORB_OK;
}

static int dynm_filter_core(dynm* h, const uint8_t* d_mask, int F, int rows, int cols, OrbxKeyPoint* d_kps, uint8_t* d_desc,
                            int32_t* d_counts, int cap, const FilterScratch& t) {
  B200_CUDA(cudaMemsetAsync(t.sums, 0, (size_t)F * 8, h->stream));
  k_dynm_mask_sum<<<dim3(64, F), 256, 0, h->stream>>>(d_mask, (size_t)rows * cols, t.sums);
  k_dynm_filter<<<F, 256, 0, h->stream>>>(d_mask, rows, cols, t.sums, d_kps, d_desc, d_counts, cap, t.kps, t.desc, t.cnt);
  h->launches += 2;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(d_kps, t.kps, (size_t)F * cap * sizeof(OrbxKeyPoint), cudaMemcpyDeviceToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_desc, t.desc, (size_t)F * cap * 32, cudaMemcpyDeviceToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_counts, t.cnt, (size_t)F * 4, cudaMemcpyDeviceToDevice, h->stream));
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
  // cv::getStructuringElement(MORPH_ELLIPSE, Size(21, 21)): row i spans c - dx .. c + dx, dx = cvRound(c sqrt((r^2 - dy^2) / r^2))
  const int r = DYNM_R, c = DYNM_R;
  const double inv_r2 = 1.0 / ((double)r * r);
  for (int i = 0; i < DYNM_K; ++i) {
    const int dy = i - r;
    h->tab.hw[i] = (int)lrint(c * sqrt((double)(r * r - dy * dy) * inv_r2));
  }
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
    for (int j = 0; j < DYNM_K; ++j) element[i * DYNM_K + j] = (j >= DYNM_R - h->tab.hw[i] && j <= DYNM_R + h->tab.hw[i]) ? 1 : 0;
  return B200ORB_OK;
}

int dynm_mask_from_flow_batch_device(dynm_t* h, const float* d_flow, int nframes, int rows, int cols, float binary_threshold,
                                     uint8_t* d_mask, int mask_rows, int mask_cols) {
  if (!h || nframes < 0 || (nframes > 0 && (!d_flow || !d_mask))) { set_error("bad argument"); return B200ORB_EINVAL; }
  if (nframes == 0) return B200ORB_OK;
  B200_CHECK(dynm_check_geometry(rows, cols, mask_rows, mask_cols));
  DeviceGuard g(h->device);
  uint8_t* d_tmp;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) { d_tmp = t.take<uint8_t>((size_t)nframes * mask_rows * mask_cols); }));
  return dynm_mask_core(h, d_flow, nframes, rows, cols, binary_threshold, d_mask, d_tmp, mask_rows, mask_cols);
}

int dynm_mask_from_flow(dynm_t* h, const float* flow, int rows, int cols, float binary_threshold, uint8_t* mask, int mask_rows,
                        int mask_cols) {
  if (!h || !flow || !mask) { set_error("bad argument"); return B200ORB_EINVAL; }
  B200_CHECK(dynm_check_geometry(rows, cols, mask_rows, mask_cols));
  DeviceGuard g(h->device);
  float* d_flow;
  uint8_t *d_mask, *d_tmp;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) {
    d_flow = t.take<float>((size_t)rows * cols * 2);
    d_mask = t.take<uint8_t>((size_t)mask_rows * mask_cols); d_tmp = t.take<uint8_t>((size_t)mask_rows * mask_cols);
  }));
  B200_CUDA(cudaMemcpyAsync(d_flow, flow, (size_t)rows * cols * 8, cudaMemcpyHostToDevice, h->stream));
  B200_CHECK(dynm_mask_core(h, d_flow, 1, rows, cols, binary_threshold, d_mask, d_tmp, mask_rows, mask_cols));
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
  FilterScratch fs;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) { fs.take(t, nframes, cap); }));
  return dynm_filter_core(h, d_mask, nframes, rows, cols, d_kps, d_desc, d_counts, cap, fs);
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
  FilterScratch fs;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) {
    d_mask = t.take<uint8_t>((size_t)rows * cols); d_kps = t.take<OrbxKeyPoint>(n); d_desc = t.take<uint8_t>((size_t)n * 32);
    d_cnt = t.take<int32_t>(1);
    fs.take(t, 1, n);
  }));
  B200_CUDA(cudaMemcpy2DAsync(d_mask, cols, mask, stride, cols, rows, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_kps, kps, (size_t)n * sizeof(OrbxKeyPoint), cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_desc, desc, (size_t)n * 32, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_cnt, &n, 4, cudaMemcpyHostToDevice, h->stream));
  B200_CHECK(dynm_filter_core(h, d_mask, 1, rows, cols, d_kps, d_desc, d_cnt, n, fs));
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

}  // extern "C"
