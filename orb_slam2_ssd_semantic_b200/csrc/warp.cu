// warp.cu -- the homography branch of the perfect variant's ComputeMask (perfect/src/Flow.cc:73-80):
// cv::warpPerspective(GrayImg, dest, Homo, GrayImg.size()) on the device -- u8, one channel, INTER_LINEAR,
// BORDER_CONSTANT 0, no WARP_INVERSE_MAP -- bit for bit as OpenCV 4.13 computes it (its integer path gives the same bytes
// at every dispatch level).  oracle/homography_py.py restates each step and tests/test_homography_cpu.py pins it to cv2:
//   * cv::invert's closed-form 3x3 inverse of Homo in double (zeros when det == 0);
//   * WarpPerspectiveInvoker's column blocks of bw0 = min(1024 / min(16, rows), cols) pixels: X0, Y0, W0 are taken at the
//     block's first column and warpPerspectiveBlockline adds M0 x1, M3 x1, M6 x1 for the block-relative column x1, so the
//     block origin is part of the result;
//   * W = W ? 32 / W : 0, clamp to [INT_MIN, INT_MAX], round half to even, source pixel = saturate_cast<short>(X >> 5),
//     sub-pixel index X & 31;
//   * remapBilinear with initInterTab2D's 15-bit fixed-point weights; taps outside the image read 0.
// Every double expression is written in OpenCV's order of operations; the library builds with --fmad=false, so none of
// them is contracted into an FMA (OpenCV's x86-64 baseline build has none either).
#include "dynm.cuh"

namespace b200 {

constexpr int WARP_THREADS = 128;
constexpr int WARP_MAX_SIDE = 32766;   // cv::remap asserts every side < SHRT_MAX

// cv::invert(S, D, DECOMP_LU) for a 3x3 CV_64F matrix: det3, then the cofactors times 1 / det; a singular S gives zeros
__device__ void warp_invert3(const double* __restrict__ S, double* __restrict__ D) {
  const double d = S[0] * (S[4] * S[8] - S[5] * S[7]) - S[1] * (S[3] * S[8] - S[5] * S[6]) + S[2] * (S[3] * S[7] - S[4] * S[6]);
  if (d == 0.0) {
    for (int i = 0; i < 9; ++i) D[i] = 0.0;
    return;
  }
  const double r = 1.0 / d;
  D[0] = (S[4] * S[8] - S[5] * S[7]) * r;
  D[1] = (S[2] * S[7] - S[1] * S[8]) * r;
  D[2] = (S[1] * S[5] - S[2] * S[4]) * r;
  D[3] = (S[5] * S[6] - S[3] * S[8]) * r;
  D[4] = (S[0] * S[8] - S[2] * S[6]) * r;
  D[5] = (S[2] * S[3] - S[0] * S[5]) * r;
  D[6] = (S[3] * S[7] - S[4] * S[6]) * r;
  D[7] = (S[1] * S[6] - S[0] * S[7]) * r;
  D[8] = (S[0] * S[4] - S[1] * S[3]) * r;
}

// std::max(INT_MIN, std::min(INT_MAX, v)) then saturate_cast<int> (cvRound: half to even)
__device__ __forceinline__ int warp_fixed(double v) {
  v = v < 2147483647.0 ? v : 2147483647.0;
  v = -2147483648.0 < v ? v : -2147483648.0;
  return __double2int_rn(v);
}

__device__ __forceinline__ int warp_tap(const uint8_t* __restrict__ src, int rows, int cols, int y, int x) {
  return ((unsigned)x < (unsigned)cols && (unsigned)y < (unsigned)rows) ? src[(size_t)y * cols + x] : 0;
}

// One thread per destination pixel: blockIdx.y = row, blockIdx.z = frame.  H[f] is the forward map (row-major double[9]);
// each CTA inverts it once into shared memory.  take (nullable): a frame whose take[f] is 0 is copied, not warped (the
// batched TrackHomo chain's frames without a model: dest = GrayImg).
__global__ void __launch_bounds__(WARP_THREADS) k_warp_perspective(const uint8_t* __restrict__ src, int rows, int cols, int bw0,
                                                                    const double* __restrict__ H, const int* __restrict__ take,
                                                                    uint8_t* __restrict__ dst) {
  __shared__ double M[9];
  const size_t plane = (size_t)rows * cols;
  src += blockIdx.z * plane;
  dst += blockIdx.z * plane;
  const int x = blockIdx.x * WARP_THREADS + threadIdx.x, y = blockIdx.y;
  if (take && !take[blockIdx.z]) {
    if (x < cols) dst[(size_t)y * cols + x] = src[(size_t)y * cols + x];
    return;
  }
  if (threadIdx.x == 0) warp_invert3(H + 9 * blockIdx.z, M);
  __syncthreads();
  if (x >= cols) return;
  const int x1 = x % bw0, xb = x - x1;
  const double dx1 = x1, dxb = xb, dy = y;
  const double X0 = M[0] * dxb + M[1] * dy + M[2];
  const double Y0 = M[3] * dxb + M[4] * dy + M[5];
  const double W0 = M[6] * dxb + M[7] * dy + M[8];
  double W = W0 + M[6] * dx1;
  W = W != 0.0 ? 32.0 / W : 0.0;
  const int X = warp_fixed((X0 + M[0] * dx1) * W);
  const int Y = warp_fixed((Y0 + M[3] * dx1) * W);
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);
  const int tx = X & 31, ty = Y & 31;
  // initInterTab2D(INTER_LINEAR, fixed point): the (0, 0) weight of 32768 saturates to 32767
  const int w00 = min((32 - ty) * (32 - tx) * 32, 32767), w01 = (32 - ty) * tx * 32, w10 = ty * (32 - tx) * 32,
            w11 = ty * tx * 32;
  const int v = warp_tap(src, rows, cols, sy, sx) * w00 + warp_tap(src, rows, cols, sy, sx + 1) * w01 +
                warp_tap(src, rows, cols, sy + 1, sx) * w10 + warp_tap(src, rows, cols, sy + 1, sx + 1) * w11;
  dst[(size_t)y * cols + x] = (uint8_t)min((v + (1 << 14)) >> 15, 255);
}

// d_H: nframes forward maps; d_src / d_dst: nframes rows x cols u8 images back to back
int launch_warp(cudaStream_t stream, const uint8_t* d_src, int nframes, int rows, int cols, const double* d_H, const int* take,
                uint8_t* d_dst, long long* launches) {
  const int bh0 = std::min(16, rows), bw0 = std::min(1024 / bh0, cols);
  k_warp_perspective<<<dim3((cols + WARP_THREADS - 1) / WARP_THREADS, rows, nframes), WARP_THREADS, 0, stream>>>(
      d_src, rows, cols, bw0, d_H, take, d_dst);
  ++*launches;
  B200_CUDA(cudaGetLastError());
  return B200ORB_OK;
}

static int warp_check(int nframes, int rows, int cols) {
  if (rows < 1 || cols < 1 || rows > WARP_MAX_SIDE || cols > WARP_MAX_SIDE) {
    set_error("warpPerspective takes images of 1 .. %d pixels a side, not %dx%d", WARP_MAX_SIDE, cols, rows);
    return B200ORB_EINVAL;
  }
  if (nframes > 65535) { set_error("at most 65535 frames per call"); return B200ORB_EINVAL; }
  return B200ORB_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int dynm_warp_perspective(dynm_t* h, const uint8_t* gray, int rows, int cols, const double* H, uint8_t* dst) {
  if (!h || !gray || !H || !dst) { set_error("bad argument"); return B200ORB_EINVAL; }
  B200_CHECK(warp_check(1, rows, cols));
  DeviceGuard g(h->device);
  const size_t px = (size_t)rows * cols;
  uint8_t *d_src, *d_dst;
  double* d_H;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) {
    d_src = t.take<uint8_t>(px); d_dst = t.take<uint8_t>(px); d_H = t.take<double>(9);
  }));
  B200_CUDA(cudaMemcpyAsync(d_src, gray, px, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_H, H, 9 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  B200_CHECK(launch_warp(h->stream, d_src, 1, rows, cols, d_H, nullptr, d_dst, &h->launches));
  B200_CUDA(cudaMemcpyAsync(dst, d_dst, px, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int dynm_warp_perspective_batch_device(dynm_t* h, const uint8_t* d_gray, int nframes, int rows, int cols, const double* d_H,
                                       uint8_t* d_dst) {
  if (!h || nframes < 0 || (nframes > 0 && (!d_gray || !d_H || !d_dst))) { set_error("bad argument"); return B200ORB_EINVAL; }
  B200_CHECK(warp_check(nframes, rows, cols));
  if (nframes == 0) return B200ORB_OK;
  DeviceGuard g(h->device);
  return launch_warp(h->stream, d_gray, nframes, rows, cols, d_H, nullptr, d_dst, &h->launches);
}

}  // extern "C"
