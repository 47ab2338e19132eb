// flow.cu -- the dense optical flow of FlowSLAM::Flow::ComputeMask (perfect/src/Flow.cc:26,29) on the device:
//   pyrDown(GrayImg, Size(cols / 2, rows / 2)) of the u8 gray image, then
//   calcOpticalFlowFarneback(prev, cur, flow, 0.5, 3, 15, 3, 5, 1.2, 0) of consecutive half-resolution images,
// bit for bit as OpenCV 4.13 computes it at its baseline dispatch level (SSE2/SSE3 code, no FMA, no IPP): the same float
// and double operations in the same order per output element (oracle/farneback_py.py restates that order and is pinned
// against cv2).  The library is built with --fmad=false, so no product-plus-sum is contracted here either.
//
// Per pyramid level k (coarse to fine) and per image: GaussianBlur of the whole half-resolution image (reflect-101) ->
// resize(INTER_LINEAR) to the level size -> FarnebackPolyExp; per pair: the previous level's flow resized and doubled,
// FarnebackUpdateMatrices, then 3 x FarnebackUpdateFlow_Blur (box filter 15 x 15: running column sums in double,
// sequential in y, then running row sums sequential in x with the 2 x 2 solve) with the matrices updated between the
// iterations.  OpenCV updates them in stripes while it sweeps; each stripe holds rows the sweep no longer reads, so a full
// sweep followed by a full update is the same computation.
#include <cmath>

#include "flow.cuh"

namespace b200 {

constexpr int FB_N = 5;                 // poly_n
constexpr int FB_M = 7;                 // winsize 15 / 2
constexpr int FB_MIN_LEVEL = 32;        // optflowgf.cpp's min_size: a level is added while both sides stay >= 32
constexpr int FB_MIN_SIDE = 16;         // half-resolution sides the kernels accept (>= 2 x the 5-pixel border band)
constexpr int FB_MAX_SIDE = 2048;

// Level blur kernels: cv::getGaussianKernel(ksize, sigma, CV_32F) at sigma = (1/scale - 1)/2, ksize = max(cvRound(5 sigma)
// | 1, 3) for scales 1, 1/2, 1/4, 1/8.  OpenCV evaluates them with its soft-float exp; these are its float results.
__constant__ uint32_t c_fb_gauss[4][19] = {
    {0x3e800000, 0x3f000000, 0x3e800000},
    {0x3dda2055, 0x3f4977eb, 0x3dda2055},
    {0x3bf98261, 0x3d13c359, 0x3de06eab, 0x3e5a9135, 0x3e887a8d, 0x3e5a9135, 0x3de06eab, 0x3d13c359, 0x3bf98261},
    {0x3b89ceeb, 0x3c09e8b2, 0x3c7e61e5, 0x3cd838ba, 0x3d2960e9, 0x3d7490c3, 0x3da2b91f, 0x3dc79039, 0x3de18f0c, 0x3deaf4ab,
     0x3de18f0c, 0x3dc79039, 0x3da2b91f, 0x3d7490c3, 0x3d2960e9, 0x3cd838ba, 0x3c7e61e5, 0x3c09e8b2, 0x3b89ceeb}};
__host__ __device__ constexpr int FB_GAUSS_KSIZE[4] = {3, 3, 9, 19};

struct FbTables {
  float g[2 * FB_N + 1], xg[2 * FB_N + 1], xxg[2 * FB_N + 1];   // index x + FB_N
  double ig11, ig03, ig33, ig55;
};
__device__ __forceinline__ float fb_gauss(int level, int i) { return __uint_as_float(c_fb_gauss[level][i]); }

// FarnebackPrepareGaussian(5, 1.2): float tables from libm exp, the 6 x 6 moment matrix in double and its inverse as
// invert(G, DECOMP_CHOLESKY) computes it (Cholesky with reciprocal diagonal, then forward and back substitution of I).
static FbTables fb_tables() {
  FbTables T;
  const int n = FB_N;
  const double sigma = 1.2;
  double s = 0.;
  for (int x = -n; x <= n; ++x) {
    T.g[x + n] = (float)std::exp(-x * x / (2 * sigma * sigma));
    s += T.g[x + n];
  }
  s = 1. / s;
  for (int x = -n; x <= n; ++x) {
    T.g[x + n] = (float)(T.g[x + n] * s);
    T.xg[x + n] = (float)(x * T.g[x + n]);
    T.xxg[x + n] = (float)(x * x * T.g[x + n]);
  }
  double G[6][6] = {};
  for (int y = -n; y <= n; ++y)
    for (int x = -n; x <= n; ++x) {
      const float gy = T.g[y + n], gx = T.g[x + n];
      G[0][0] += gy * gx;
      G[1][1] += gy * gx * x * x;
      G[3][3] += gy * gx * x * x * x * x;
      G[5][5] += gy * gx * x * x * y * y;
    }
  G[2][2] = G[0][3] = G[0][4] = G[3][0] = G[4][0] = G[1][1];
  G[4][4] = G[3][3];
  G[3][4] = G[4][3] = G[5][5];
  double L[6][6], B[6][6];
  memcpy(L, G, sizeof(L));
  for (int i = 0; i < 6; ++i) {
    for (int j = 0; j < i; ++j) {
      double t = L[i][j];
      for (int k = 0; k < j; ++k) t -= L[i][k] * L[j][k];
      L[i][j] = t * L[j][j];
    }
    double t = L[i][i];
    for (int k = 0; k < i; ++k) t -= L[i][k] * L[i][k];
    L[i][i] = 1. / std::sqrt(t);
  }
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) B[i][j] = i == j ? 1. : 0.;
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      double t = B[i][j];
      for (int k = 0; k < i; ++k) t -= L[i][k] * B[k][j];
      B[i][j] = t * L[i][i];
    }
  for (int i = 5; i >= 0; --i)
    for (int j = 0; j < 6; ++j) {
      double t = B[i][j];
      for (int k = 5; k > i; --k) t -= L[k][i] * B[k][j];
      B[i][j] = t * L[i][i];
    }
  T.ig11 = B[1][1];
  T.ig03 = B[0][3];
  T.ig33 = B[3][3];
  T.ig55 = B[5][5];
  return T;
}

int fb_geometry(int H, int W, FbGeom* g) {
  if (H < FB_MIN_SIDE || W < FB_MIN_SIDE || H > FB_MAX_SIDE || W > FB_MAX_SIDE) {
    set_error("dense flow of %dx%d half-resolution images: both sides must lie in [%d, %d]", W, H, FB_MIN_SIDE, FB_MAX_SIDE);
    return B200ORB_EINVAL;
  }
  g->H = H;
  g->W = W;
  double scale = 1.;
  int k = 0;
  for (; k < FB_LEVELS; ++k) {
    scale *= 0.5;
    if (W * scale < FB_MIN_LEVEL || H * scale < FB_MIN_LEVEL) break;
  }
  g->top = k;
  for (k = 0, scale = 1.; k <= g->top; ++k, scale *= 0.5) {
    g->h[k] = (int)std::nearbyint(H * scale);
    g->w[k] = (int)std::nearbyint(W * scale);
  }
  return B200ORB_OK;
}

void fb_take(Carver& t, FbScratch& s, const FbGeom& g, int C) {
  const size_t px = (size_t)g.H * g.W, px1 = g.top ? (size_t)g.h[1] * g.w[1] : 1, I = (size_t)C + 1;
  s.half = t.take<uint8_t>(I * px);
  s.tmp = t.take<float>(I * px);
  s.blur = t.take<float>(I * px);
  s.img = t.take<float>(I * px1);
  s.R = t.take<float>(I * px * 5);
  s.M = t.take<float>((size_t)C * px * 5);
  s.V = t.take<double>((size_t)C * px * 5);
  s.fl[0] = t.take<float>((size_t)C * px1 * 2);
  s.fl[1] = t.take<float>((size_t)C * px1 * 2);
}

__device__ __forceinline__ int fb_reflect101(int p, int n) {   // cv::borderInterpolate(p, n, BORDER_REFLECT_101)
  if (n == 1) return 0;
  while ((unsigned)p >= (unsigned)n) p = p < 0 ? -p : 2 * (n - 1) - p;
  return p;
}

// pyrDown of u8 images (5 x 5 [1 4 6 4 1]^2 / 256, reflect-101, round half up); image i = blockIdx.y reads `first` for
// i == 0 and rest + (i - 1) * SH * SW otherwise.
__global__ void __launch_bounds__(256) k_fb_pyrdown(const uint8_t* __restrict__ first, const uint8_t* __restrict__ rest, int SH,
                                                    int SW, uint8_t* __restrict__ dst, int H, int W) {
  const int i = blockIdx.y, p = blockIdx.x * 256 + threadIdx.x;
  if (p >= H * W) return;
  const uint8_t* src = i == 0 ? first : rest + (size_t)(i - 1) * SH * SW;
  const int y = p / W, x = p - y * W;
  const int w5[5] = {1, 4, 6, 4, 1};
  int xs[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) xs[j] = fb_reflect101(2 * x + j - 2, SW);
  int s = 0;
#pragma unroll
  for (int r = 0; r < 5; ++r) {
    const uint8_t* row = src + (size_t)fb_reflect101(2 * y + r - 2, SH) * SW;
    int t = 0;
#pragma unroll
    for (int j = 0; j < 5; ++j) t += w5[j] * row[xs[j]];
    s += w5[r] * t;
  }
  dst[(size_t)i * H * W + p] = (uint8_t)((s + 128) >> 8);
}

// GaussianBlur row pass of the u8 image (converted to float), reflect-101: ksize 3 (l + r)*k0 + c*k1 (SymmRowSmallFilter),
// larger sizes c0*k0 + c1*k1 + ... left to right (RowFilter).
__global__ void __launch_bounds__(256) k_fb_blur_row(const uint8_t* __restrict__ src, float* __restrict__ dst, int H, int W,
                                                     int level) {
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= H * W) return;
  const size_t o = (size_t)blockIdx.y * H * W;
  const int n = FB_GAUSS_KSIZE[level], y = p / W, x = p - y * W, r = n / 2;
  const uint8_t* row = src + o + (size_t)y * W;
  float s;
  if (n == 3) {
    s = ((float)row[fb_reflect101(x - 1, W)] + (float)row[fb_reflect101(x + 1, W)]) * fb_gauss(level, 2) +
        (float)row[x] * fb_gauss(level, 1);
  } else {
    s = (float)row[fb_reflect101(x - r, W)] * fb_gauss(level, 0);
    for (int i = 1; i < n; ++i) s = s + (float)row[fb_reflect101(x - r + i, W)] * fb_gauss(level, i);
  }
  dst[o + p] = s;
}

// column pass: ksize 3 (u + d)*k0 + c*k1 (SymmColumnSmallFilter), larger c*k[r] then += (d_i + u_i)*k[r + i]
// (SymmColumnFilter)
__global__ void __launch_bounds__(256) k_fb_blur_col(const float* __restrict__ src, float* __restrict__ dst, int H, int W,
                                                     int level) {
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= H * W) return;
  const size_t o = (size_t)blockIdx.y * H * W;
  const int n = FB_GAUSS_KSIZE[level], y = p / W, x = p - y * W, r = n / 2;
  const float* s0 = src + o + x;
  float s;
  if (n == 3) {
    s = (s0[(size_t)fb_reflect101(y - 1, H) * W] + s0[(size_t)fb_reflect101(y + 1, H) * W]) * fb_gauss(level, 2) +
        s0[(size_t)y * W] * fb_gauss(level, 1);
  } else {
    s = s0[(size_t)y * W] * fb_gauss(level, r);
    for (int i = 1; i <= r; ++i)
      s = s + (s0[(size_t)fb_reflect101(y + i, H) * W] + s0[(size_t)fb_reflect101(y - i, H) * W]) * fb_gauss(level, r + i);
  }
  dst[o + p] = s;
}

// resize(INTER_LINEAR) of float images with cn channels, image = blockIdx.y.  `area`: both sides exactly halved, which
// OpenCV runs as INTER_AREA's fast path (single channel: (a00 + a01) + (a10 + a11) for the outputs its 4-wide SIMD loop
// covers, ((a00 + a01) + a10) + a11 for the rest of a row, times 0.25).  Otherwise bilinear with float taps
// f = (float)((d + 0.5)*scale - 0.5): x taps clamped to the first / last pixel, y taps on clamped rows, h = s0*a0 + s1*a1,
// out = h0*b0 + h1*b1.  `twice`: flow *= 1/pyr_scale, which OpenCV evaluates as x*2 + 0.
__global__ void __launch_bounds__(256) k_fb_resize(const float* __restrict__ src, int SH, int SW, float* __restrict__ dst, int h,
                                                   int w, int cn, int area, double scale_x, double scale_y, int twice) {
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= h * w * cn) return;
  const int y = p / (w * cn), xc = p - y * w * cn, x = xc / cn, c = xc - x * cn;
  const float* S = src + (size_t)blockIdx.y * SH * SW * cn;
  float v;
  if (area) {
    const float* r0 = S + (size_t)(2 * y) * SW + 2 * x;
    const float* r1 = r0 + SW;
    v = x < (w & ~3) ? ((r0[0] + r0[1]) + (r1[0] + r1[1])) * 0.25f : (((r0[0] + r0[1]) + r1[0]) + r1[1]) * 0.25f;
  } else {
    float fx = (float)((x + 0.5) * scale_x - 0.5);
    int sx = (int)floorf(fx);
    fx -= (float)sx;
    const bool right = sx + 1 >= SW;   // this and every later column: the last pixel itself
    if (sx < 0) { fx = 0.f; sx = 0; }
    float fy = (float)((y + 0.5) * scale_y - 0.5);
    const int sy = (int)floorf(fy);
    fy -= (float)sy;
    const float* r0 = S + (size_t)min(max(sy, 0), SH - 1) * SW * cn;
    const float* r1 = S + (size_t)min(max(sy + 1, 0), SH - 1) * SW * cn;
    float h0, h1;
    if (right) {
      h0 = r0[(SW - 1) * cn + c];
      h1 = r1[(SW - 1) * cn + c];
    } else {
      const float a0 = 1.f - fx, a1 = fx;
      h0 = r0[sx * cn + c] * a0 + r0[(sx + 1) * cn + c] * a1;
      h1 = r1[sx * cn + c] * a0 + r1[(sx + 1) * cn + c] * a1;
    }
    v = h0 * (1.f - fy) + h1 * fy;
  }
  if (twice) v = v * 2.f + 0.f;
  dst[(size_t)blockIdx.y * h * w * cn + p] = v;
}

// FarnebackPolyExp of row y = blockIdx.x of image blockIdx.y: the vertical taps of the whole row into shared memory (float,
// replicated rows), then per pixel the horizontal taps in double (replicated columns); out = (r3, r2, r5, r4, r6) scaled.
__global__ void __launch_bounds__(256) k_fb_polyexp(const float* __restrict__ src, float* __restrict__ R, int h, int w,
                                                    FbTables T) {
  extern __shared__ float row[];   // [w][3]
  const int y = blockIdx.x;
  const float* I = src + (size_t)blockIdx.y * h * w;
  for (int x = threadIdx.x; x < w; x += blockDim.x) {
    float r0 = I[(size_t)y * w + x] * T.g[FB_N], r1 = 0.f, r2 = 0.f;
#pragma unroll
    for (int k = 1; k <= FB_N; ++k) {
      const float s0 = I[(size_t)max(y - k, 0) * w + x], s1 = I[(size_t)min(y + k, h - 1) * w + x];
      const float p = s0 + s1;
      r0 = r0 + T.g[FB_N + k] * p;
      r1 = r1 + T.xg[FB_N + k] * (s1 - s0);
      r2 = r2 + T.xxg[FB_N + k] * p;
    }
    row[x * 3] = r0;
    row[x * 3 + 1] = r1;
    row[x * 3 + 2] = r2;
  }
  __syncthreads();
  float* out = R + ((size_t)blockIdx.y * h + y) * w * 5;
  for (int x = threadIdx.x; x < w; x += blockDim.x) {
    const float g0 = T.g[FB_N];
    double b1 = row[x * 3] * g0, b2 = 0, b3 = row[x * 3 + 1] * g0, b4 = 0, b5 = row[x * 3 + 2] * g0, b6 = 0;
#pragma unroll
    for (int k = 1; k <= FB_N; ++k) {
      const float* P = row + min(x + k, w - 1) * 3;
      const float* Q = row + max(x - k, 0) * 3;
      const float gk = T.g[FB_N + k], xgk = T.xg[FB_N + k];
      const double tg = P[0] + Q[0];
      b1 = b1 + tg * (double)gk;
      b4 = b4 + tg * (double)T.xxg[FB_N + k];
      b2 = b2 + (double)((P[0] - Q[0]) * xgk);
      b3 = b3 + (double)((P[1] + Q[1]) * gk);
      b6 = b6 + (double)((P[1] - Q[1]) * xgk);
      b5 = b5 + (double)((P[2] + Q[2]) * gk);
    }
    out[x * 5 + 0] = (float)(b3 * T.ig11);
    out[x * 5 + 1] = (float)(b2 * T.ig11);
    out[x * 5 + 2] = (float)(b1 * T.ig03 + b5 * T.ig33);
    out[x * 5 + 3] = (float)(b1 * T.ig03 + b4 * T.ig33);
    out[x * 5 + 4] = (float)(b6 * T.ig55);
  }
}

// FarnebackUpdateMatrices of pair blockIdx.y (R0 = image i, R1 = image i + 1): R1 fetched bilinearly at the displaced
// position (inside the image only), the 5-pixel border band weighted by 0.14, 0.14, 0.4472, 0.4472, 0.4472.
__global__ void __launch_bounds__(256) k_fb_update(const float* __restrict__ R, const float* __restrict__ flow, float* __restrict__ M,
                                                   int h, int w) {
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= h * w) return;
  const size_t img = (size_t)h * w * 5, i = blockIdx.y;
  const float* R0 = R + i * img + (size_t)p * 5;
  const float* R1 = R + (i + 1) * img;
  const float* fl = flow + (i * h * w + p) * 2;
  const int y = p / w, x = p - y * w;
  const float dx = fl[0], dy = fl[1];
  float fx = (float)x + dx, fy = (float)y + dy;
  const int x1 = (int)floorf(fx), y1 = (int)floorf(fy);
  fx -= (float)x1;
  fy -= (float)y1;
  float r2, r3, r4, r5, r6;
  if ((unsigned)x1 < (unsigned)(w - 1) && (unsigned)y1 < (unsigned)(h - 1)) {
    const float a00 = (1.f - fx) * (1.f - fy), a01 = fx * (1.f - fy), a10 = (1.f - fx) * fy, a11 = fx * fy;
    const float* q = R1 + ((size_t)y1 * w + x1) * 5;
    const size_t s = (size_t)w * 5;
    float r[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) r[c] = a00 * q[c] + a01 * q[5 + c] + a10 * q[s + c] + a11 * q[s + 5 + c];
    r2 = r[0];
    r3 = r[1];
    r4 = (R0[2] + r[2]) * 0.5f;
    r5 = (R0[3] + r[3]) * 0.5f;
    r6 = (R0[4] + r[4]) * 0.25f;
  } else {
    r2 = r3 = 0.f;
    r4 = R0[2];
    r5 = R0[3];
    r6 = R0[4] * 0.5f;
  }
  r2 = (R0[0] - r2) * 0.5f;
  r3 = (R0[1] - r3) * 0.5f;
  r2 += r4 * dy + r6 * dx;
  r3 += r6 * dy + r5 * dx;
  if (x < 5 || x >= w - 5 || y < 5 || y >= h - 5) {
    const float bw[5] = {0.14f, 0.14f, 0.4472f, 0.4472f, 0.4472f};
    const float scale = (x < 5 ? bw[x] : 1.f) * (x >= w - 5 ? bw[w - x - 1] : 1.f) * (y < 5 ? bw[y] : 1.f) *
                        (y >= h - 5 ? bw[h - y - 1] : 1.f);
    r2 *= scale;
    r3 *= scale;
    r4 *= scale;
    r5 *= scale;
    r6 *= scale;
  }
  float* m = M + (i * h * w + p) * 5;
  m[0] = r4 * r4 + r6 * r6;
  m[1] = (r4 + r5) * r6;
  m[2] = r5 * r5 + r6 * r6;
  m[3] = r4 * r2 + r6 * r3;
  m[4] = r6 * r2 + r5 * r3;
}

// FarnebackUpdateFlow_Blur, vertical part: one thread per (pair, matrix element j of a row), sequential down the column;
// the sum is initialised to row 0 x (m + 2) (a float product) plus rows 1 .. m-1, then each row adds the float difference
// of the entering and leaving rows (replicated at the borders).  V holds the sum as it stands at each row.
__global__ void __launch_bounds__(256) k_fb_vsum(const float* __restrict__ M, double* __restrict__ V, int h, int w) {
  const int w5 = w * 5, j = blockIdx.x * 256 + threadIdx.x;
  if (j >= w5) return;
  const size_t o = (size_t)blockIdx.y * h * w5;
  const float* m = M + o + j;
  double* v = V + o + j;
  double s = m[0] * (float)(FB_M + 2);
  for (int y = 1; y < FB_M; ++y) s += m[(size_t)min(y, h - 1) * w5];
  for (int y = 0; y < h; ++y) {
    s += m[(size_t)min(y + FB_M, h - 1) * w5] - m[(size_t)max(y - FB_M - 1, 0) * w5];
    v[(size_t)y * w5] = s;
  }
}

// horizontal part + solve: one thread per (pair, row), sequential along the row over the column sums (replicated columns),
// idet = 1/(g11 g22 - g12^2 + 1e-3), flow = ((g11 h2 - g12 h1) idet, (g22 h1 - g12 h2) idet) in double, stored as float.
__global__ void __launch_bounds__(128) k_fb_hsolve(const double* __restrict__ V, float* __restrict__ flow, int h, int w) {
  const int y = blockIdx.x * 128 + threadIdx.x;
  if (y >= h) return;
  const size_t i = blockIdx.y;
  const double* v = V + (i * h + y) * w * 5;
  float* fl = flow + (i * h + y) * w * 2;
  double a[5];
#pragma unroll
  for (int c = 0; c < 5; ++c) a[c] = v[c] * (FB_M + 2);
  for (int x = 1; x < FB_M; ++x) {
    const double* q = v + min(x, w - 1) * 5;
#pragma unroll
    for (int c = 0; c < 5; ++c) a[c] += q[c];
  }
  const double scale = 1. / ((2 * FB_M + 1) * (2 * FB_M + 1));
  for (int x = 0; x < w; ++x) {
    const double* in = v + min(x + FB_M, w - 1) * 5;
    const double* out = v + max(x - FB_M - 1, 0) * 5;
#pragma unroll
    for (int c = 0; c < 5; ++c) a[c] += in[c] - out[c];
    const double g11 = a[0] * scale, g12 = a[1] * scale, g22 = a[2] * scale, h1 = a[3] * scale, h2 = a[4] * scale;
    const double idet = 1. / (g11 * g22 - g12 * g12 + 1e-3);
    fl[x * 2] = (float)((g11 * h2 - g12 * h1) * idet);
    fl[x * 2 + 1] = (float)((g22 * h1 - g12 * h2) * idet);
  }
}

static inline unsigned fb_blocks(size_t n, int t) { return (unsigned)((n + t - 1) / t); }

int fb_pairs(cudaStream_t st, const FbGeom& g, const FbScratch& s, int nimg, float* out, long long* launches) {
  static const FbTables T = fb_tables();
  const int P = nimg - 1, H = g.H, W = g.W;
  const size_t px = (size_t)H * W;
  float* prev_flow = nullptr;
  for (int k = g.top; k >= 0; --k) {
    const int h = g.h[k], w = g.w[k];
    k_fb_blur_row<<<dim3(fb_blocks(px, 256), nimg), 256, 0, st>>>(s.half, s.tmp, H, W, k);
    k_fb_blur_col<<<dim3(fb_blocks(px, 256), nimg), 256, 0, st>>>(s.tmp, s.blur, H, W, k);
    *launches += 2;
    const float* I = s.blur;
    if (h != H || w != W) {
      const double sx = 1. / ((double)w / W), sy = 1. / ((double)h / H);
      k_fb_resize<<<dim3(fb_blocks((size_t)h * w, 256), nimg), 256, 0, st>>>(s.blur, H, W, s.img, h, w, 1,
                                                                              sx == 2. && sy == 2., sx, sy, 0);
      ++*launches;
      I = s.img;
    }
    k_fb_polyexp<<<dim3(h, nimg), 256, (size_t)w * 3 * sizeof(float), st>>>(I, s.R, h, w, T);
    ++*launches;
    float* flow = k == 0 ? out : s.fl[k & 1];
    if (!prev_flow) {
      B200_CUDA(cudaMemsetAsync(flow, 0, (size_t)P * h * w * 2 * sizeof(float), st));
    } else {
      const int ph = g.h[k + 1], pw = g.w[k + 1];
      k_fb_resize<<<dim3(fb_blocks((size_t)h * w * 2, 256), P), 256, 0, st>>>(prev_flow, ph, pw, flow, h, w, 2, 0,
                                                                               1. / ((double)w / pw), 1. / ((double)h / ph), 1);
      ++*launches;
    }
    const dim3 pix(fb_blocks((size_t)h * w, 256), P);
    k_fb_update<<<pix, 256, 0, st>>>(s.R, flow, s.M, h, w);
    ++*launches;
    for (int it = 0; it < 3; ++it) {
      k_fb_vsum<<<dim3(fb_blocks((size_t)w * 5, 256), P), 256, 0, st>>>(s.M, s.V, h, w);
      k_fb_hsolve<<<dim3(fb_blocks(h, 128), P), 128, 0, st>>>(s.V, flow, h, w);
      *launches += 2;
      if (it < 2) {
        k_fb_update<<<pix, 256, 0, st>>>(s.R, flow, s.M, h, w);
        ++*launches;
      }
    }
    prev_flow = flow;
  }
  B200_CUDA(cudaGetLastError());
  return B200ORB_OK;
}

void fb_pyrdown(cudaStream_t st, const FbGeom& g, const uint8_t* first, const uint8_t* rest, int nimg, int SH, int SW,
                uint8_t* dst, long long* launches) {
  k_fb_pyrdown<<<dim3(fb_blocks((size_t)g.H * g.W, 256), nimg), 256, 0, st>>>(first, rest, SH, SW, dst, g.H, g.W);
  ++*launches;
}

int fb_batch(cudaStream_t st, const FbGeom& g, const FbScratch& s, int C, const uint8_t* d_gray, const uint8_t* d_prev,
             int n, int SH, int SW, float* out, long long* launches) {
  const size_t spx = (size_t)SH * SW, fpx = (size_t)g.H * g.W * 2;
  if (!d_prev) B200_CUDA(cudaMemsetAsync(out, 0, fpx * sizeof(float), st));
  for (int f0 = 0; f0 < n; f0 += C) {
    const int f1 = std::min(n, f0 + C), t0 = (f0 == 0 && !d_prev) ? 1 : f0;
    if (t0 >= f1) continue;
    const int nimg = f1 - t0 + 1;
    const uint8_t* first = t0 == 0 ? d_prev : d_gray + (size_t)(t0 - 1) * spx;
    fb_pyrdown(st, g, first, d_gray + (size_t)t0 * spx, nimg, SH, SW, s.half, launches);
    B200_CHECK(fb_pairs(st, g, s, nimg, out + (size_t)t0 * fpx, launches));
  }
  return B200ORB_OK;
}

}  // namespace b200
