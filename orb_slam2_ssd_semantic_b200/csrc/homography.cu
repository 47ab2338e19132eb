// homography.cu -- the homography branch's model: cv::findHomography(points_current, points_last, RANSAC, 3) as TrackHomo
// calls it (perfect/src/Tracking.cc:1386; maxIters 2000, confidence 0.995), the Levenberg-Marquardt refinement included,
// on the device.  It follows OpenCV 4.13's baseline code (cv::setUseOptimized(false)) in the order of operations that
// tests/homography_lm.py restates on top of oracle/homography_py.py, so it equals that restatement bit for bit (and cv2
// bit for bit below 50 inliers; from 100 residual rows a cv2 built with LAPACK sums J^T r in its BLAS's order):
//   k_hf_draw        one warp: lane 0 draws 32 candidate 4-index subsets from cv::RNG((uint64)-1) (the stream and the
//                    duplicate redraws depend on no pair), the lanes run checkSubset on one candidate each, a ballot keeps
//                    the accepted ones in draw order; it stops at 2000 accepted subsets, or at 10000 consecutive
//                    rejections (getSubset's failure, which ends RANSAC there);
//   k_hf_hypotheses  one CTA per accepted subset: runKernel of its 4 pairs, then the float computeError of every pair
//                    and the count of errors <= 9;
//   k_hf_refine      one CTA: one thread scans the hypotheses in iteration order (good > max(max_good, 3), the adaptive
//                    niters from the host's libm table), then the ordered inlier compaction, runKernel on the inliers,
//                    LMSolver's at most 10 iterations over 9 parameters, H times 1 / H22 and the mask of the refined H.
// Every sum whose order the restatement fixes is one thread's sequential loop; everything else is one thread per pair
// or per matrix entry, and the Jacobi sweeps are one warp (lane 0 picks the pivot, lanes 0..8 rotate).  The library builds with --fmad=false, so no expression is contracted into an FMA (OpenCV's
// x86-64 baseline has none either); log and pow run on the host (glibc) and reach the device as a table.
#include <cfloat>
#include <cmath>
#include <vector>

#include "dynm.cuh"

namespace b200 {

constexpr int HF_MAX_ITERS = 2000;
constexpr int HF_MAX_ATTEMPTS = 10000;
constexpr int HF_LM_ITERS = 10;
constexpr int HF_HYP_THREADS = 128;
constexpr int HF_REFINE_THREADS = 512;
constexpr double HF_DBL_EPS = 2.220446049250313e-16;
constexpr double HF_FLT_EPS = 1.1920928955078125e-07;
constexpr float HF_THRESH2 = 9.0f;   // ransacReprojThreshold 3, squared

// ---- runKernel ---------------------------------------------------------------------------------------------------------

// lapack.cpp's own hypot
__device__ double hf_hypot(double a, double b) {
  a = fabs(a); b = fabs(b);
  if (a > b) { b /= a; return a * sqrt(1 + b * b); }
  if (b > 0) { a /= b; return b * sqrt(1 + a * a); }
  return 0.0;
}

struct HfJacobi {
  double A[81], V[81], W[9];
  int indR[9], indC[9];
};

__device__ void hf_index(HfJacobi& J, int k) {
  const int n = 9;
  if (k < n - 1) {
    int m = k + 1;
    double mv = fabs(J.A[k * 9 + k + 1]);
    for (int i = k + 2; i < n; ++i)
      if (mv < fabs(J.A[k * 9 + i])) { mv = fabs(J.A[k * 9 + i]); m = i; }
    J.indR[k] = m;
  }
  if (k > 0) {
    int m = 0;
    double mv = fabs(J.A[k]);
    for (int i = 1; i < k; ++i)
      if (mv < fabs(J.A[i * 9 + k])) { mv = fabs(J.A[i * 9 + k]); m = i; }
    J.indC[k] = m;
  }
}

// cv::eigen of the symmetric 9x9 J.A (JacobiImpl_): eigenvalues descending in W, eigenvectors in the rows of V.  Called
// by all 32 lanes of one warp: lane 0 picks each pivot and its rotation in JacobiImpl_'s order, lanes 0..8 apply the
// rotation to column / row i (each element is touched by one lane and once, so the result is the serial sweep's), and
// lanes 0 and 1 refresh the two pivot indices.
__device__ __forceinline__ void hf_eigen(HfJacobi& J) {
  const int n = 9, lane = threadIdx.x & 31;
  if (lane < n) {
    for (int j = 0; j < n; ++j) J.V[lane * 9 + j] = lane == j ? 1.0 : 0.0;
    J.W[lane] = J.A[lane * 9 + lane];
  }
  __syncwarp();
  if (lane < n) hf_index(J, lane);   // reads A only, writes indR / indC of its own row
  __syncwarp();
  for (int iter = 0; iter < n * n * 30; ++iter) {
    int k = 0, l = 0;
    double c = 0.0, s = 0.0;
    bool stop = false;
    if (lane == 0) {
      double mv = fabs(J.A[J.indR[0]]);
      for (int i = 1; i < n - 1; ++i)
        if (mv < fabs(J.A[i * 9 + J.indR[i]])) { mv = fabs(J.A[i * 9 + J.indR[i]]); k = i; }
      l = J.indR[k];
      for (int i = 1; i < n; ++i)
        if (mv < fabs(J.A[J.indC[i] * 9 + i])) { mv = fabs(J.A[J.indC[i] * 9 + i]); k = J.indC[i]; l = i; }
      const double p = J.A[k * 9 + l];
      stop = fabs(p) <= HF_DBL_EPS;
      if (!stop) {
        const double y = (J.W[l] - J.W[k]) * 0.5;
        double t = fabs(y) + hf_hypot(p, y);
        s = hf_hypot(p, t);
        c = t / s;
        s = p / s;
        t = (p / t) * p;
        if (y < 0) { s = -s; t = -t; }
        J.A[k * 9 + l] = 0.0;
        J.W[k] -= t;
        J.W[l] += t;
      }
    }
    if (__shfl_sync(0xffffffffu, stop, 0)) break;
    k = __shfl_sync(0xffffffffu, k, 0);
    l = __shfl_sync(0xffffffffu, l, 0);
    c = __shfl_sync(0xffffffffu, c, 0);
    s = __shfl_sync(0xffffffffu, s, 0);
    if (lane < n) {
      const int i = lane;
      double *a = nullptr, *b = nullptr;
      if (i < k) { a = &J.A[i * 9 + k]; b = &J.A[i * 9 + l]; }
      else if (k < i && i < l) { a = &J.A[k * 9 + i]; b = &J.A[i * 9 + l]; }
      else if (i > l) { a = &J.A[k * 9 + i]; b = &J.A[l * 9 + i]; }
      if (a) {
        const double a0 = *a, b0 = *b;
        *a = a0 * c - b0 * s;
        *b = a0 * s + b0 * c;
      }
      const double v0 = J.V[k * 9 + i], v1 = J.V[l * 9 + i];
      J.V[k * 9 + i] = v0 * c - v1 * s;
      J.V[l * 9 + i] = v0 * s + v1 * c;
    }
    __syncwarp();
    if (lane < 2) hf_index(J, lane == 0 ? k : l);
    __syncwarp();
  }
  for (int k = 0; k < n - 1; ++k) {
    int m = k;
    if (lane == 0)
      for (int i = k + 1; i < n; ++i)
        if (J.W[m] < J.W[i]) m = i;
    m = __shfl_sync(0xffffffffu, m, 0);
    if (k != m) {
      if (lane == 0) { const double t = J.W[m]; J.W[m] = J.W[k]; J.W[k] = t; }
      if (lane < n) { const double t = J.V[m * 9 + lane]; J.V[m * 9 + lane] = J.V[k * 9 + lane]; J.V[k * 9 + lane] = t; }
    }
    __syncwarp();
  }
}

// entry j of runKernel's row Lx = (X, Y, 1, 0, 0, 0, -x X, -x Y, -x) (row 0) or Ly = (0, 0, 0, X, Y, 1, -y X, -y Y, -y)
__device__ __forceinline__ double hf_lrow(int j, double X, double Y, double u, int row) {
  if (j < 6) {
    if (j / 3 != row) return 0.0;
    const int c = j % 3;
    return c == 0 ? X : c == 1 ? Y : 1.0;
  }
  return j == 6 ? -u * X : j == 7 ? -u * Y : -u;
}

struct HfKernel {
  HfJacobi jac;
  double c[4], s[4];   // cmx, cmy, cMx, cMy; smx, smy, sMx, sMy
  int ok;
};

// HomographyEstimatorCallback::runKernel of M (src) -> m (dst), n pairs, by the whole CTA.  H (row-major, shared or
// global) is written only when the set is not degenerate; K.ok says which.
__device__ __forceinline__ void hf_run_kernel(const float2* __restrict__ M, const float2* __restrict__ m, int n, HfKernel& K, double* H) {
  const int t = threadIdx.x;
  if (t < 4) {   // centroids, each a sequential sum
    double s = 0.0;
    for (int i = 0; i < n; ++i) {
      const float2 p = t < 2 ? m[i] : M[i];
      s += (double)((t & 1) ? p.y : p.x);
    }
    K.c[t] = s / n;
  }
  __syncthreads();
  if (t < 4) {   // mean absolute deviations
    double s = 0.0;
    const double c = K.c[t];
    for (int i = 0; i < n; ++i) {
      const float2 p = t < 2 ? m[i] : M[i];
      s += fabs((double)((t & 1) ? p.y : p.x) - c);
    }
    K.s[t] = s;
  }
  __syncthreads();
  const bool degenerate = fabs(K.s[0]) < HF_DBL_EPS || fabs(K.s[1]) < HF_DBL_EPS || fabs(K.s[2]) < HF_DBL_EPS ||
                          fabs(K.s[3]) < HF_DBL_EPS;
  if (degenerate) {
    if (t == 0) K.ok = 0;
    __syncthreads();
    return;
  }
  const double smx = n / K.s[0], smy = n / K.s[1], sMx = n / K.s[2], sMy = n / K.s[3];
  const double cmx = K.c[0], cmy = K.c[1], cMx = K.c[2], cMy = K.c[3];
  for (int e = t; e < 81; e += blockDim.x) {   // LtL: entry (j, k >= j) a sequential sum over the pairs
    const int j = e / 9, k = e % 9;
    if (k < j) continue;
    double s = 0.0;
    for (int i = 0; i < n; ++i) {
      const double x = ((double)m[i].x - cmx) * smx, y = ((double)m[i].y - cmy) * smy;
      const double X = ((double)M[i].x - cMx) * sMx, Y = ((double)M[i].y - cMy) * sMy;
      s += hf_lrow(j, X, Y, x, 0) * hf_lrow(k, X, Y, x, 0) + hf_lrow(j, X, Y, y, 1) * hf_lrow(k, X, Y, y, 1);
    }
    K.jac.A[j * 9 + k] = s;
    K.jac.A[k * 9 + j] = s;
  }
  __syncthreads();
  if (t < 32) {   // the eigenvector of the smallest eigenvalue, de-normalised: inv_hnorm V8 hnorm2, times 1 / H22
    hf_eigen(K.jac);
    double* T = K.jac.A;   // A is spent: T in A[0..8], the product in A[9..17]
    if (t < 9) {   // the scales again from shared memory (the same IEEE quotients) rather than kept live across the sweep
      const double smx = n / K.s[0], smy = n / K.s[1], cmx = K.c[0], cmy = K.c[1];
      const int i = t / 3, j = t % 3;
      const double* V8 = K.jac.V + 72;
      const double a0 = i == 0 ? 1. / smx : 0, a1 = i == 1 ? 1. / smy : 0, a2 = i == 0 ? cmx : i == 1 ? cmy : 1;
      T[t] = (a0 * V8[j] + a1 * V8[3 + j]) + a2 * V8[6 + j];
    }
    __syncwarp();
    if (t < 9) {
      const double sMx = n / K.s[2], sMy = n / K.s[3], cMx = K.c[2], cMy = K.c[3];
      const int i = t / 3, j = t % 3;
      const double b0 = j == 0 ? sMx : j == 2 ? -cMx * sMx : 0, b1 = j == 1 ? sMy : j == 2 ? -cMy * sMy : 0,
                   b2 = j == 2 ? 1 : 0;
      T[9 + t] = (T[i * 3] * b0 + T[i * 3 + 1] * b1) + T[i * 3 + 2] * b2;
    }
    __syncwarp();
    if (t < 9) H[t] = T[9 + t] * (1.0 / T[17]);
    if (t == 0) K.ok = 1;
  }
  __syncthreads();
}

// HomographyEstimatorCallback::computeError: float, from the float-cast model
__device__ __forceinline__ float hf_error(const float* Hf, float2 M, float2 m) {
  const float ww = 1.f / (Hf[6] * M.x + Hf[7] * M.y + 1.f);
  const float dx = (Hf[0] * M.x + Hf[1] * M.y + Hf[2]) * ww - m.x;
  const float dy = (Hf[3] * M.x + Hf[4] * M.y + Hf[5]) * ww - m.y;
  return dx * dx + dy * dy;
}

// ---- RANSAC ------------------------------------------------------------------------------------------------------------

// haveCollinearPoints of the last point: each difference is a float subtraction (Point2f - Point2f) widened to double,
// the products, sums and the comparison are double
__device__ bool hf_collinear(const float2* P) {
  const int i = 3;
  for (int j = 0; j < i; ++j) {
    const double dx1 = (double)(P[j].x - P[i].x), dy1 = (double)(P[j].y - P[i].y);
    for (int k = 0; k < j; ++k) {
      const double dx2 = (double)(P[k].x - P[i].x), dy2 = (double)(P[k].y - P[i].y);
      if (fabs(dx2 * dy1 - dy2 * dx1) <= HF_FLT_EPS * (fabs(dx1) + fabs(dy1) + fabs(dx2) + fabs(dy2))) return true;
    }
  }
  return false;
}

__device__ double hf_det3(const float2* P, int a, int b, int c) {
  const double a00 = P[a].x, a01 = P[a].y, a10 = P[b].x, a11 = P[b].y, a20 = P[c].x, a21 = P[c].y;
  return a00 * (a11 * 1.0 - a21 * 1.0) - a01 * (a10 * 1.0 - a20 * 1.0) + 1.0 * (a10 * a21 - a20 * a11);
}

// checkSubset of 4 pairs
__device__ bool hf_check_subset(const float2* __restrict__ src, const float2* __restrict__ dst, const int* idx) {
  float2 s[4], d[4];
  for (int q = 0; q < 4; ++q) { s[q] = src[idx[q]]; d[q] = dst[idx[q]]; }
  if (hf_collinear(s) || hf_collinear(d)) return false;
  const int tri[4][3] = {{0, 1, 2}, {1, 2, 3}, {0, 2, 3}, {0, 1, 3}};
  int neg = 0;
  for (int q = 0; q < 4; ++q)
    neg += hf_det3(s, tri[q][0], tri[q][1], tri[q][2]) * hf_det3(d, tri[q][0], tri[q][1], tri[q][2]) < 0;
  return neg == 0 || neg == 4;
}

// The fit kernels read the pair count n from device memory; n == 0 (a frame of the batched chain that takes no fit) makes
// every one of them return at once.
__global__ void __launch_bounds__(32) k_hf_draw(const float2* __restrict__ src, const float2* __restrict__ dst,
                                                const int* __restrict__ np, int* __restrict__ subsets,
                                                int* __restrict__ nsub) {
  __shared__ int cand[32][4];
  const int lane = threadIdx.x, n = *np;
  if (n == 0) return;
  unsigned long long state = ~0ull;
  int accepted = 0, rejected = 0;
  bool done = false;
  while (!done) {
    if (lane == 0) {
      for (int c = 0; c < 32; ++c)
        for (int q = 0; q < 4; ++q) {
          int v;
          for (;;) {
            state = (unsigned long long)(unsigned)state * 4164903690ull + (state >> 32);
            v = (int)((unsigned)state % (unsigned)n);
            bool dup = false;
            for (int r = 0; r < q; ++r) dup |= cand[c][r] == v;
            if (!dup) break;
          }
          cand[c][q] = v;
        }
    }
    __syncwarp();
    const unsigned ok = __ballot_sync(0xffffffffu, hf_check_subset(src, dst, cand[lane]));
    if (lane == 0) {
      for (int c = 0; c < 32 && !done; ++c) {
        if (ok >> c & 1u) {
          for (int q = 0; q < 4; ++q) subsets[accepted * 4 + q] = cand[c][q];
          rejected = 0;
          done = ++accepted == HF_MAX_ITERS;
        } else {
          done = ++rejected == HF_MAX_ATTEMPTS;
        }
      }
    }
    done = __shfl_sync(0xffffffffu, done, 0);
    __syncwarp();
  }
  if (lane == 0) *nsub = accepted;
}

__global__ void __launch_bounds__(HF_HYP_THREADS) k_hf_hypotheses(const float2* __restrict__ src, const float2* __restrict__ dst,
                                                                  const int* __restrict__ np, const int* __restrict__ subsets,
                                                                  const int* __restrict__ nsub, double* __restrict__ hyp,
                                                                  int* __restrict__ good) {
  __shared__ HfKernel K;
  __shared__ float2 S[4], D[4];
  __shared__ double H[9];
  __shared__ float Hf[9];
  const int it = blockIdx.x, n = *np;
  if (n == 0 || it >= *nsub) return;
  if (threadIdx.x < 4) {
    const int i = subsets[it * 4 + threadIdx.x];
    S[threadIdx.x] = src[i];
    D[threadIdx.x] = dst[i];
  }
  __syncthreads();
  hf_run_kernel(S, D, 4, K, H);
  if (!K.ok) {
    if (threadIdx.x == 0) good[it] = -1;
    return;
  }
  if (threadIdx.x < 9) {
    hyp[it * 9 + threadIdx.x] = H[threadIdx.x];
    Hf[threadIdx.x] = (float)H[threadIdx.x];
  }
  __syncthreads();
  int cnt = 0;
  for (int base = 0; base < n; base += HF_HYP_THREADS) {
    const int i = base + threadIdx.x;
    cnt += __syncthreads_count(i < n && hf_error(Hf, src[i], dst[i]) <= HF_THRESH2);
  }
  if (threadIdx.x == 0) good[it] = cnt;
}

// ---- refinement --------------------------------------------------------------------------------------------------------

struct HfRefine {
  HfKernel K;
  double x[9], xd[9], d[9], v[9], D[9], A[81], Hk[9], acc[8];
  double S, Sd, lambda, lc, rinf;
  float Hf[9];
  double nu;
  int best, ninl, need_inv, warp_base[HF_REFINE_THREADS / 32];
};

// residuals (and, with J, the Jacobian) of parameters h for the ni pairs: HomographyRefineCallback::compute
__device__ void hf_residuals(const float2* __restrict__ M, const float2* __restrict__ m, int ni, const double* h,
                             double* __restrict__ r, double* __restrict__ J) {
  for (int i = threadIdx.x; i < ni; i += blockDim.x) {
    const double Mx = M[i].x, My = M[i].y;
    double ww = (h[6] * Mx + h[7] * My) + h[8];
    ww = fabs(ww) > HF_DBL_EPS ? 1. / ww : 0;
    const double xi = ((h[0] * Mx + h[1] * My) + h[2]) * ww;
    const double yi = ((h[3] * Mx + h[4] * My) + h[5]) * ww;
    r[2 * i] = xi - (double)m[i].x;
    r[2 * i + 1] = yi - (double)m[i].y;
    if (J) {
      double* Jx = J + (size_t)18 * i;
      Jx[0] = Mx * ww; Jx[1] = My * ww; Jx[2] = ww;
      Jx[3] = Jx[4] = Jx[5] = 0.;
      Jx[6] = -Mx * ww * xi; Jx[7] = -My * ww * xi; Jx[8] = -ww * xi;
      Jx[9] = Jx[10] = Jx[11] = 0.;
      Jx[12] = Mx * ww; Jx[13] = My * ww; Jx[14] = ww;
      Jx[15] = -Mx * ww * yi; Jx[16] = -My * ww * yi; Jx[17] = -ww * yi;
    }
  }
}

// norm(r, NORM_L2SQR) of len doubles: eight sequential lane accumulators (4 v_float64x2 registers over blocks of 8),
// combined by thread 0 with the tail; the caller syncs before and reads R.acc[0] after.
__device__ void hf_norm_l2sqr(const double* __restrict__ r, int len, HfRefine& R) {
  const int n8 = len / 8 * 8, t = threadIdx.x;
  if (t < 8) {
    double s = 0.0;
    for (int i = t; i < n8; i += 8) s += r[i] * r[i];
    R.acc[t] = s;
  }
  __syncthreads();
  if (t == 0) {
    double lane[2] = {0.0, 0.0};
    for (int q = 0; q < 4; ++q)
      for (int l = 0; l < 2; ++l) lane[l] = lane[l] + R.acc[2 * q + l];
    double s = 0.0 + (lane[0] + lane[1]);
    for (int i = n8; i < len; ++i) s += r[i] * r[i];
    R.acc[0] = s;
  }
  __syncthreads();
}

// mulTransposed(J, A, true) and gemm(J, r, 1, noArray(), 0, v, GEMM_1_T) for rows = 2 ni
__device__ void hf_normal_equations(const double* __restrict__ J, const double* __restrict__ r, int rows, HfRefine& R) {
  const int t = threadIdx.x;
  if (t < 81) {
    const int i = t / 9, j = t % 9;
    if (j >= i) {
      double s = 0.0;
      for (int k = 0; k < rows; ++k) s += J[(size_t)k * 9 + i] * J[(size_t)k * 9 + j];
      R.A[i * 9 + j] = s;
      R.A[j * 9 + i] = s;
    }
  } else if (t >= 96 && t < 105) {
    const int c = t - 96, n4 = rows / 4 * 4;
    double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    for (int k = 0; k < n4; k += 4) {
      s0 += J[(size_t)k * 9 + c] * r[k];
      s1 += J[(size_t)(k + 1) * 9 + c] * r[k + 1];
      s2 += J[(size_t)(k + 2) * 9 + c] * r[k + 2];
      s3 += J[(size_t)(k + 3) * 9 + c] * r[k + 3];
    }
    for (int k = n4; k < rows; ++k) s0 += J[(size_t)k * 9 + c] * r[k];
    R.v[c] = (((s0 + s1) + s2) + s3) * 1.0;
  }
}

// Mat::dot of two 9-vectors (dotProd_64f at baseline: dotProd_'s loop unrolled by 4, then the tail in order)
__device__ double hf_dot9(const double* a, const double* b) {
  double r = 0.0;
  for (int i = 0; i < 8; i += 4) r += ((a[i] * b[i] + a[i + 1] * b[i + 1]) + a[i + 2] * b[i + 2]) + a[i + 3] * b[i + 3];
  r += a[8] * b[8];
  return r;
}

// SVBkSb's basis of the symmetric R.K.jac.A: Jacobi, then the threshold 2 DBL_EPSILON times the sequential sum of W
__device__ double hf_eig_basis(HfJacobi& J) {
  hf_eigen(J);
  double s = 0.0;
  for (int k = 0; k < 9; ++k) s += J.W[k];
  return s * (2 * HF_DBL_EPS);
}

// One warp: solve(Ap, v, d, DECOMP_EIG) with Ap in J.A; lane j accumulates x[j] over the kept eigenpairs in order
__device__ void hf_solve_eig(HfJacobi& J, const double* b, double* x) {
  const double thr = hf_eig_basis(J);
  const int lane = threadIdx.x & 31;
  double xj = 0.0;
  for (int k = 0; k < 9; ++k) {
    const double wk = J.W[k];
    if (fabs(wk) <= thr) continue;
    double s = 0.0;
    for (int j = 0; j < 9; ++j) s += J.V[k * 9 + j] * b[j];
    s = s * (1.0 / wk);
    if (lane < 9) xj = xj + s * J.V[k * 9 + lane];
  }
  if (lane < 9) x[lane] = xj;
  __syncwarp();
}

// One warp: the largest |diag(invert(A, DECOMP_EIG))|, at least DBL_EPSILON, with A in J.A (every lane gets it)
__device__ double hf_inverse_diag_max(HfJacobi& J) {
  const double thr = hf_eig_basis(J);
  const int lane = threadIdx.x & 31;
  double X = 0.0;
  if (lane < 9)
    for (int k = 0; k < 9; ++k) {
      const double wk = J.W[k];
      if (fabs(wk) <= thr) continue;
      const double wi = 1.0 / wk;
      X = X + J.V[k * 9 + lane] * (J.V[k * 9 + lane] * wi);
    }
  double maxval = lane < 9 ? fabs(X) : 0.0;
  for (int o = 16; o; o >>= 1) maxval = fmax(maxval, __shfl_xor_sync(0xffffffffu, maxval, o));
  return fmax(HF_DBL_EPS, maxval);
}

// the largest |r_i| over len doubles, by the whole CTA into R.rinf
__device__ void hf_norm_inf(const double* __restrict__ r, int len, HfRefine& R) {
  double m = 0.0;
  for (int i = threadIdx.x; i < len; i += blockDim.x) m = fmax(m, fabs(r[i]));
  for (int o = 16; o; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (threadIdx.x == 0) R.rinf = 0.0;
  __syncthreads();
  if ((threadIdx.x & 31) == 0)
    atomicMax((unsigned long long*)&R.rinf, (unsigned long long)__double_as_longlong(m));   // m >= 0: bits order as values
  __syncthreads();
}

// out[0..8] H, out[9] found (as a double), mask n bytes.  tab: hf_tab's rows n0 = tab_n0 and up; row n holds tab[g] =
// log(1 - (1 - ep)^4) for g good pairs (NaN where 1 - (1 - ep)^4 < DBL_MIN), then log(max(1 - confidence, DBL_MIN)).
__global__ void __launch_bounds__(HF_REFINE_THREADS) k_hf_refine(const float2* __restrict__ src, const float2* __restrict__ dst,
                                                                 const int* __restrict__ np, const int* __restrict__ nsub,
                                                                 const double* __restrict__ hyp, const int* __restrict__ good,
                                                                 const double* __restrict__ tab, int tab_n0,
                                                                 float2* __restrict__ isrc, float2* __restrict__ idst,
                                                                 double* __restrict__ J, double* __restrict__ r,
                                                                 double* __restrict__ rd, double* __restrict__ out,
                                                                 uint8_t* __restrict__ mask) {
  __shared__ HfRefine R;
  const int t = threadIdx.x, n = *np;
  if (n == 0) return;
  tab += hf_tab_row(n, tab_n0);
  if (n == 4) {   // runKernel of all four pairs, unrefined, mask all ones
    hf_run_kernel(src, dst, 4, R.K, R.x);
    if (t < 9) out[t] = R.K.ok ? R.x[t] : 0.0;
    if (t == 9) out[9] = R.K.ok;
    if (t < 4) mask[t] = R.K.ok;
    return;
  }
  if (t == 0) {   // RANSACPointSetRegistrator::run's loop over the hypotheses in iteration order
    const int K = *nsub;
    int niters = HF_MAX_ITERS, max_good = 0, best = -1;
    const double num = tab[n + 1];
    for (int it = 0; it < niters && it < K; ++it) {
      const int g = good[it];
      if (g > max(max_good, 3)) {
        best = it;
        max_good = g;
        const double denom = tab[g];   // RANSACUpdateNumIters(0.995, (n - g) / n, 4, niters)
        if (isnan(denom)) niters = 0;
        else if (!(denom >= 0 || -num >= niters * (-denom))) niters = __double2int_rn(num / denom);
      }
    }
    R.best = max_good > 0 ? best : -1;
  }
  __syncthreads();
  if (R.best < 0) {
    if (t < 10) out[t] = 0.0;
    for (int i = t; i < n; i += blockDim.x) mask[i] = 0;
    return;
  }
  if (t < 9) {
    R.x[t] = hyp[R.best * 9 + t];
    R.Hf[t] = (float)R.x[t];
  }
  if (t == 0) R.ninl = 0;
  __syncthreads();
  // ordered compaction of the best hypothesis' inliers
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + t;
    const bool in = i < n && hf_error(R.Hf, src[i], dst[i]) <= HF_THRESH2;
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if ((t & 31) == 0) R.warp_base[t >> 5] = __popc(b);
    __syncthreads();
    if (t == 0) {
      int s = R.ninl;
      for (int w = 0; w < HF_REFINE_THREADS / 32; ++w) { const int c = R.warp_base[w]; R.warp_base[w] = s; s += c; }
      R.ninl = s;
    }
    __syncthreads();
    if (in) {
      const int o = R.warp_base[t >> 5] + __popc(b & ((1u << (t & 31)) - 1u));
      isrc[o] = src[i];
      idst[o] = dst[i];
    }
    __syncthreads();
  }
  const int ni = R.ninl, rows = 2 * ni;
  hf_run_kernel(isrc, idst, ni, R.K, R.Hk);
  if (R.K.ok && t < 9) R.x[t] = R.Hk[t];
  __syncthreads();
  // LMSolverImpl::run
  hf_residuals(isrc, idst, ni, R.x, r, J);
  __syncthreads();
  hf_norm_l2sqr(r, rows, R);
  if (t == 0) R.S = R.acc[0];
  hf_normal_equations(J, r, rows, R);
  __syncthreads();
  if (t < 9) R.D[t] = R.A[t * 9 + t];
  if (t == 0) { R.lambda = 1.0; R.lc = 0.75; R.need_inv = 0; }
  __syncthreads();
  for (int iter = 0;;) {
    if (t < 32) {   // d = solve(A + lambda diag(D), v, DECOMP_EIG), xd = x - d
      if (t < 9) {
        for (int j = 0; j < 9; ++j) R.K.jac.A[t * 9 + j] = R.A[t * 9 + j];
        R.K.jac.A[t * 9 + t] += R.lambda * R.D[t];
      }
      __syncwarp();
      hf_solve_eig(R.K.jac, R.v, R.d);
      if (t < 9) R.xd[t] = R.x[t] - R.d[t];
    }
    __syncthreads();
    hf_residuals(isrc, idst, ni, R.xd, rd, nullptr);
    __syncthreads();
    hf_norm_l2sqr(rd, rows, R);
    if (t == 0) {
      const double S = R.S, Sd = R.acc[0];
      R.need_inv = 0;
      R.Sd = Sd;
      double temp_d[9];
      for (int i = 0; i < 9; ++i) {   // gemm(A, d, -1, v, 2)
        double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
        for (int k = 0; k < 8; k += 4) {
          s0 += R.A[i * 9 + k] * R.d[k]; s1 += R.A[i * 9 + k + 1] * R.d[k + 1];
          s2 += R.A[i * 9 + k + 2] * R.d[k + 2]; s3 += R.A[i * 9 + k + 3] * R.d[k + 3];
        }
        s0 += R.A[i * 9 + 8] * R.d[8];
        temp_d[i] = (((s0 + s1) + s2) + s3) * -1.0 + R.v[i] * 2.0;
      }
      const double dS = hf_dot9(R.d, temp_d);
      const double Rg = (S - Sd) / (fabs(dS) > HF_DBL_EPS ? dS : 1);
      if (Rg > 0.75) {
        R.lambda *= 0.5;
        if (R.lambda < R.lc) R.lambda = 0;
      } else if (Rg < 0.25) {
        const double tv = hf_dot9(R.d, R.v);
        double nu = (Sd - S) / (fabs(tv) > HF_DBL_EPS ? tv : 1) + 2;
        nu = fmin(fmax(nu, 2.), 10.);
        R.nu = nu;
        R.need_inv = R.lambda == 0;
        if (!R.need_inv) R.lambda *= nu;
      }
    }
    __syncthreads();
    if (R.need_inv) {   // lambda = lc = 1 / max |diag(invert(A, DECOMP_EIG))|, nu halved, then lambda *= nu
      if (t < 32) {
        if (t < 9)
          for (int j = 0; j < 9; ++j) R.K.jac.A[t * 9 + j] = R.A[t * 9 + j];
        __syncwarp();
        const double maxval = hf_inverse_diag_max(R.K.jac);
        if (t == 0) {
          R.lambda = R.lc = 1. / maxval;
          R.lambda *= R.nu * 0.5;
        }
      }
      __syncthreads();
    }
    const bool accept = R.Sd < R.S;
    __syncthreads();
    if (accept) {   // accept the step: x = xd, new residuals, Jacobian and normal equations
      if (t < 9) R.x[t] = R.xd[t];
      if (t == 0) R.S = R.Sd;
      __syncthreads();
      hf_residuals(isrc, idst, ni, R.x, r, J);
      __syncthreads();
      hf_normal_equations(J, r, rows, R);
      __syncthreads();
    }
    ++iter;
    hf_norm_inf(r, rows, R);
    const double rinf = R.rinf;
    double dinf = 0.0;
    for (int i = 0; i < 9; ++i) dinf = fmax(dinf, fabs(R.d[i]));
    __syncthreads();
    if (!(iter < HF_LM_ITERS && dinf >= HF_FLT_EPS && rinf >= HF_FLT_EPS)) break;
  }
  // H.convertTo(H, CV_64F, scaleFor(H22)), then the mask of the refined H over every pair
  if (t == 0) {
    const double h22 = R.x[8];
    const double s = fabs(h22) > HF_FLT_EPS ? 1. / h22 : 1.;
    for (int i = 0; i < 9; ++i) {
      R.x[i] = R.x[i] * s + 0.0;
      R.Hf[i] = (float)R.x[i];
    }
  }
  __syncthreads();
  if (t < 9) out[t] = R.x[t];
  if (t == 9) out[9] = 1.0;
  for (int i = t; i < n; i += blockDim.x) mask[i] = hf_error(R.Hf, src[i], dst[i]) <= HF_THRESH2;
}

void hf_tab(int n0, int n1, std::vector<double>& tab) {
  tab.resize(hf_tab_row(n1 + 1, n0));
  const double num = std::log(std::max(1. - 0.995, DBL_MIN));
  for (int n = n0; n <= n1; ++n) {   // RANSACUpdateNumIters(0.995, (n - g) / n, 4, niters)'s log and pow
    double* row = tab.data() + hf_tab_row(n, n0);
    for (int g = 0; g <= n; ++g) {
      double ep = (double)(n - g) / n;
      ep = std::min(std::max(ep, 0.), 1.);
      const double denom = 1. - std::pow(1. - ep, 4);
      row[g] = denom < DBL_MIN ? std::nan("") : std::log(denom);
    }
    row[n + 1] = num;
  }
}

void hf_take(Carver& t, HfScratch& s, int cap) {
  s.isrc = t.take<float2>(cap); s.idst = t.take<float2>(cap);
  s.sub = t.take<int>(4 * HF_MAX_ITERS); s.nsub = t.take<int>(1); s.good = t.take<int>(HF_MAX_ITERS);
  s.hyp = t.take<double>(9 * HF_MAX_ITERS); s.J = t.take<double>((size_t)18 * cap);
  s.r = t.take<double>(2 * (size_t)cap); s.rd = t.take<double>(2 * (size_t)cap);
}

int launch_hf_fit(cudaStream_t st, const float2* src, const float2* dst, const int* d_n, bool ransac, const double* tab,
                  int tab_n0, const HfScratch& s, double* out, uint8_t* mask, long long* launches) {
  if (ransac) {
    k_hf_draw<<<1, 32, 0, st>>>(src, dst, d_n, s.sub, s.nsub);
    k_hf_hypotheses<<<HF_MAX_ITERS, HF_HYP_THREADS, 0, st>>>(src, dst, d_n, s.sub, s.nsub, s.hyp, s.good);
    *launches += 2;
  }
  k_hf_refine<<<1, HF_REFINE_THREADS, 0, st>>>(src, dst, d_n, s.nsub, s.hyp, s.good, tab, tab_n0, s.isrc, s.idst, s.J, s.r,
                                               s.rd, out, mask);
  ++*launches;
  B200_CUDA(cudaGetLastError());
  return B200ORB_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int dynm_find_homography(dynm_t* h, const float* src, const float* dst, int n, double H[9], uint8_t* mask, int* found) {
  if (!h || !src || !dst || !H || !mask || !found) { set_error("bad argument"); return B200ORB_EINVAL; }
  if (n < 4 || n > HF_MAX_PAIRS) {
    set_error("findHomography takes 4 .. %d pairs, not %d", HF_MAX_PAIRS, n);
    return B200ORB_EINVAL;
  }
  std::vector<double> tab;
  hf_tab(n, n, tab);
  DeviceGuard g(h->device);
  float2 *d_src, *d_dst;
  int* d_n;
  double *d_tab, *d_out;
  uint8_t* d_mask;
  HfScratch s;
  B200_CHECK(h->buf.reserve(h->stream, [&](Carver& t) {
    d_src = t.take<float2>(n); d_dst = t.take<float2>(n); d_n = t.take<int>(1); d_tab = t.take<double>(tab.size());
    d_out = t.take<double>(10); d_mask = t.take<uint8_t>(n);
    hf_take(t, s, n);
  }));
  B200_CUDA(cudaMemcpyAsync(d_src, src, n * sizeof(float2), cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_dst, dst, n * sizeof(float2), cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_n, &n, sizeof(int), cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_tab, tab.data(), tab.size() * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  B200_CHECK(launch_hf_fit(h->stream, d_src, d_dst, d_n, n > 4, d_tab, n, s, d_out, d_mask, &h->launches));
  double out[10];
  B200_CUDA(cudaMemcpyAsync(out, d_out, sizeof(out), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(mask, d_mask, n, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  for (int i = 0; i < 9; ++i) H[i] = out[i];
  *found = out[9] != 0.0;
  return B200ORB_OK;
}

}  // extern "C"
