// orbm_extra.cuh -- the matcher entry points that need no ordered claim resolve, and the one that is a plain
// sequential loop:
//   BEST   per-query best keypoint in a keyframe (window walk + level range + optional chi-square gate + Hamming):
//          the device part of Fuse(KeyFrame*, vector<MapPoint*>, th)        src/ORBmatcher.cc:1031-1182
//                             Fuse(KeyFrame*, Scw, vpPoints, th, vpReplace)  src/ORBmatcher.cc:1198-1318
//                             SearchBySim3 (both directions)                 src/ORBmatcher.cc:1334-1558
//          none of which lets a query see what earlier queries did to the keyframe's keypoints.
//   TRI    SearchForTriangulation (src/ORBmatcher.cc:827-1019): BoW-node-wise Hamming search with the epipole and
//          epipolar-line gates; the reference never sets vbMatched2 (:909 reads it, nothing writes it), so the queries
//          are independent; "dist > bestDist -> continue" makes the LAST minimum among the gate-passers win.
//   INIT   SearchForInitialization (src/ORBmatcher.cc:523-651): level-0 window search where a closer match STEALS an
//          already matched keypoint (vMatchedDistance) -- loop-carried through every query, run once per session
//          (monocular initialisation), so ONE warp walks the queries in order and does each window walk itself.
#pragma once
#include "orbm_match.cuh"

namespace b200 {

// ---------------------------------------------------------------------------------------------------------------------
// BEST
// ---------------------------------------------------------------------------------------------------------------------
struct BestGate {
  int mode;                 // 0: none; 1: Fuse reprojection gate (:1118-1146)
  const float* inv_sigma2;  // pKF->mvInvLevelSigma2 (device)
  const float* kp_uright;   // pKF->mvuRight (device)
};

__global__ void __launch_bounds__(CAND_WARPS * 32) k_best_generic(CurView cv, QueriesView qv, MatchCam cam, BestGate gate,
                                                                  int* __restrict__ best_idx, int* __restrict__ best_dist) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * CAND_WARPS + (threadIdx.x >> 5);
  if (i >= qv.n[0]) return;
  int bi = -1, bd = 0x7fffffff;
  QueryGeom q;
  if (setup_generic_query(qv, i, q)) {
    const uint8_t* d = qv.desc + (size_t)i * 32;
    const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(d)), d1 = __ldg(reinterpret_cast<const uint4*>(d) + 1);
    WalkCtx g = make_ctx(cv, cam, 0);
    g.obs = nullptr;        // no claim state of any kind
    g.uright = nullptr;     // the window walk has no stereo gate in these searches
    const float qu = q.u, qvv = q.v, qur = q.ur;
    unsigned long long bk = ~0ull;
    warp_walk(g, q, d0, d1, [&](int ord, int idx, int dist) {
      if (gate.mode == 1) {
        const float kpx = g.x[idx], kpy = g.y[idx], kpr = gate.kp_uright[idx];
        const float ex = __fsub_rn(qu, kpx), ey = __fsub_rn(qvv, kpy);
        const float is2 = gate.inv_sigma2[g.oct[idx]];
        if (kpr >= 0) {
          const float er = __fsub_rn(qur, kpr);
          const float e2 = __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(er, er));
          if ((double)__fmul_rn(e2, is2) > 7.8) return;
        } else {
          const float e2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
          if ((double)__fmul_rn(e2, is2) > 5.99) return;
        }
      }
      const unsigned long long kk = key64(dist, ord, idx);
      bk = (kk < bk) ? kk : bk;
    });
    bk = warp_min64(bk);
    if (bk != ~0ull) { bi = (int)(bk & 0x3fffffull); bd = (int)(bk >> 44); }
  }
  if (lane == 0) { best_idx[i] = bi; best_dist[i] = bd; }
}

// ---------------------------------------------------------------------------------------------------------------------
// TRI
// ---------------------------------------------------------------------------------------------------------------------
struct TriView {
  const int* q_idx1;       // keypoint of pKF1 per query (host merge-join; MapPoint-free, stereo filter applied)
  const int* f_beg;        // range of the matching pKF2 node inside f_idx
  const int* f_end;
  const unsigned* f_idx;
  const uint8_t *desc1, *desc2;
  const float *x1, *y1, *ang1, *ur1;
  const float *x2, *y2, *ang2, *ur2;
  const int* oct2;
  const uint8_t* blocked2;   // pKF2 keypoint already holds a MapPoint
  float F12[9];
  float ex, ey;
  float sf2[MAX_LEVELS], sigma2_2[MAX_LEVELS];
  int only_stereo, nq, n1;
};

__global__ void __launch_bounds__(CAND_WARPS * 32) k_tri_best(TriView t, int* __restrict__ matches12) {
  const int lane = threadIdx.x & 31;
  const int q = blockIdx.x * CAND_WARPS + (threadIdx.x >> 5);
  if (q >= t.nq) return;
  const int idx1 = t.q_idx1[q];
  const uint8_t* d = t.desc1 + (size_t)idx1 * 32;
  const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(d)), d1 = __ldg(reinterpret_cast<const uint4*>(d) + 1);
  const float x1 = t.x1[idx1], y1 = t.y1[idx1];
  const bool stereo1 = t.ur1[idx1] >= 0;
  // epipolar line of kp1 in image 2 (CheckDistEpipolarLine :175-194)
  const float a = __fadd_rn(__fadd_rn(__fmul_rn(x1, t.F12[0]), __fmul_rn(y1, t.F12[3])), t.F12[6]);
  const float b = __fadd_rn(__fadd_rn(__fmul_rn(x1, t.F12[1]), __fmul_rn(y1, t.F12[4])), t.F12[7]);
  const float c = __fadd_rn(__fadd_rn(__fmul_rn(x1, t.F12[2]), __fmul_rn(y1, t.F12[5])), t.F12[8]);
  const float den = __fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b));
  const int beg = t.f_beg[q], n = t.f_end[q] - beg;
  // key: dist in the high bits, REVERSED position below it -> the minimum is the smallest distance, last occurrence
  unsigned long long bk = ~0ull;
  for (int e = lane; e < n; e += 32) {
    const int idx2 = (int)t.f_idx[beg + e];
    if (t.blocked2[idx2]) continue;
    const bool stereo2 = t.ur2[idx2] >= 0;
    if (t.only_stereo && !stereo2) continue;
    const int dist = hamming256(d0, d1, t.desc2 + (size_t)idx2 * 32);
    if (dist > ORBM_TH_LOW) continue;
    const float x2 = t.x2[idx2], y2 = t.y2[idx2];
    const int o2 = t.oct2[idx2];
    if (!stereo1 && !stereo2) {
      const float dx = __fsub_rn(t.ex, x2), dy = __fsub_rn(t.ey, y2);
      if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < __fmul_rn(100.f, t.sf2[o2])) continue;
    }
    if (den == 0.f) continue;
    const float num = __fadd_rn(__fadd_rn(__fmul_rn(a, x2), __fmul_rn(b, y2)), c);
    const float dsqr = __fdiv_rn(__fmul_rn(num, num), den);
    if (!((double)dsqr < 3.84 * (double)t.sigma2_2[o2])) continue;
    const unsigned long long kk = ((unsigned long long)dist << 44) | ((unsigned long long)(0x3fffff - e) << 22) |
                                  (unsigned long long)idx2;
    bk = (kk < bk) ? kk : bk;
  }
  bk = warp_min64(bk);
  if (lane == 0) matches12[idx1] = (bk != ~0ull) ? (int)(bk & 0x3fffffull) : -1;
}

// rotation histogram of the matched pKF1 keypoints + prune (:986-1005) + count; one warp
__global__ void __launch_bounds__(32) k_tri_prune(TriView t, int check_ori, int* __restrict__ matches12, int* __restrict__ nmatch) {
  __shared__ int s_hist[ORBM_HISTO_LENGTH];
  __shared__ int s_keep[3];
  const int lane = threadIdx.x;
  for (int b = lane; b < ORBM_HISTO_LENGTH; b += 32) s_hist[b] = 0;
  __syncwarp();
  int cnt = 0;
  for (int i = lane; i < t.n1; i += 32) {
    const int m = matches12[i];
    if (m >= 0) { ++cnt; if (check_ori) atomicAdd(&s_hist[rot_bin(t.ang1[i], t.ang2[m])], 1); }
  }
  __syncwarp();
  if (check_ori) {
    if (lane == 0) three_maxima(s_hist, s_keep);
    __syncwarp();
    for (int i = lane; i < t.n1; i += 32) {
      const int m = matches12[i];
      if (m >= 0) {
        const int bin = rot_bin(t.ang1[i], t.ang2[m]);
        if (bin != s_keep[0] && bin != s_keep[1] && bin != s_keep[2]) { matches12[i] = -1; --cnt; }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) *nmatch = cnt;
}

// ---------------------------------------------------------------------------------------------------------------------
// INIT
// ---------------------------------------------------------------------------------------------------------------------
struct InitView {
  const int* oct1;
  const float* ang1;
  const uint8_t* desc1;
  float* prev_xy;        // vbPrevMatched, n1 x 2 (in / out)
  int n1;
  int* matched_dist;     // n2 (scratch)
  int* match21;          // n2 (scratch)
  int* bin1;             // n1 (scratch): histogram bin the query was pushed into, or -1
};

__global__ void __launch_bounds__(32) k_init_search(CurView f2, InitView v, MatchCam cam, int window, float nnratio,
                                                    int check_ori, int* __restrict__ matches12, int* __restrict__ nmatch) {
  __shared__ int s_hist[ORBM_HISTO_LENGTH];
  __shared__ int s_keep[3];
  const int lane = threadIdx.x;
  const int n2 = f2.n[0];
  for (int j = lane; j < n2; j += 32) { v.matched_dist[j] = 0x7fffffff; v.match21[j] = -1; }
  for (int i = lane; i < v.n1; i += 32) { matches12[i] = -1; v.bin1[i] = -1; }
  for (int b = lane; b < ORBM_HISTO_LENGTH; b += 32) s_hist[b] = 0;
  __syncwarp();
  WalkCtx g = make_ctx(f2, cam, 0);
  g.obs = nullptr;
  g.uright = nullptr;
  for (int i1 = 0; i1 < v.n1; ++i1) {
    if (v.oct1[i1] > 0) continue;                          // :540-542 (warp-uniform)
    QueryGeom q;
    q.u = v.prev_xy[2 * i1]; q.v = v.prev_xy[2 * i1 + 1]; q.r = (float)window; q.rr = q.r; q.ur = 0.f;
    q.min_level = 0; q.max_level = 0;                      // GetFeaturesInArea(x, y, windowSize, level1, level1)
    if (isnan(q.u) || isnan(q.v)) continue;
    const uint8_t* d = v.desc1 + (size_t)i1 * 32;
    const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(d)), d1 = __ldg(reinterpret_cast<const uint4*>(d) + 1);
    // per lane: smallest and second smallest key (dist, ord) among the candidates a closer earlier match does not block
    unsigned long long k1 = ~0ull, k2 = ~0ull;
    warp_walk(g, q, d0, d1, [&](int ord, int idx, int dist) {
      if (v.matched_dist[idx] <= dist) return;            // :565-566
      const unsigned long long kk = key64(dist, ord, idx);
      if (kk < k1) { k2 = k1; k1 = kk; }
      else if (kk < k2) k2 = kk;
    });
    const unsigned long long K1 = warp_min64(k1);
    if (K1 == ~0ull) continue;
    const unsigned long long K2 = warp_min64(k1 == K1 ? k2 : k1);
    const int bestDist = (int)(K1 >> 44), bestIdx2 = (int)(K1 & 0x3fffffull);
    const int bestDist2 = (K2 == ~0ull) ? 0x7fffffff : (int)(K2 >> 44);
    if (bestDist <= ORBM_TH_LOW && (float)bestDist < __fmul_rn((float)bestDist2, nnratio)) {   // :579-581
      if (lane == 0) {
        const int prev = v.match21[bestIdx2];
        if (prev >= 0) matches12[prev] = -1;               // a stolen match: the earlier query loses it (:583-587)
        matches12[i1] = bestIdx2;
        v.match21[bestIdx2] = i1;
        v.matched_dist[bestIdx2] = bestDist;
        if (check_ori) {
          const int bin = rot_bin(v.ang1[i1], f2.ang[bestIdx2]);
          v.bin1[i1] = bin;
          s_hist[bin] += 1;
        }
      }
    }
    __syncwarp();
  }
  // nmatches as the reference counts it: +1 per accepted query, -1 per steal, -1 per pruned entry that is still matched;
  // equivalently the number of queries that still hold a match after the prune
  __syncwarp();
  if (check_ori) {
    if (lane == 0) three_maxima(s_hist, s_keep);
    __syncwarp();
    for (int i = lane; i < v.n1; i += 32) {
      const int bin = v.bin1[i];
      if (bin >= 0 && bin != s_keep[0] && bin != s_keep[1] && bin != s_keep[2] && matches12[i] >= 0) matches12[i] = -1;
    }
  }
  __syncwarp();
  int cnt = 0;
  for (int i = lane; i < v.n1; i += 32) {
    const int m = matches12[i];
    if (m >= 0) {
      ++cnt;
      v.prev_xy[2 * i] = f2.x[m];            // :640-642
      v.prev_xy[2 * i + 1] = f2.y[m];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) *nmatch = cnt;
}

// ---------------------------------------------------------------------------------------------------------------------
// Frame glue: Frame::isInFrustum (src/Frame.cc:387-451) and Frame::UndistortKeyPoints (src/Frame.cc:559-590)
// ---------------------------------------------------------------------------------------------------------------------
struct FrustumView {
  const float *xw, *normal, *min_dist, *max_dist;   // GetWorldPos(), GetNormal(), mfMinDistance, mfMaxDistance
  int n;
  float Tcw[16];
  float fx, fy, cx, cy, bf, min_x, max_x, min_y, max_y;
  float cos_limit;
  float level_thr[MAX_LEVELS];   // PredictScale as thresholds on ratio = mfMaxDistance / dist (built on the host with libm)
  int nlevels;
};

__global__ void k_is_in_frustum(FrustumView f, uint8_t* __restrict__ in_view, float* __restrict__ px, float* __restrict__ py,
                                float* __restrict__ pxr, int* __restrict__ level, float* __restrict__ vcos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= f.n) return;
  in_view[i] = 0;
  const float* T = f.Tcw;
  const float P[3] = {f.xw[3 * i], f.xw[3 * i + 1], f.xw[3 * i + 2]};
  const float PcX = gemm3(T + 0, P[0], P[1], P[2], T[3]);      // mRcw*P+mtcw
  const float PcY = gemm3(T + 4, P[0], P[1], P[2], T[7]);
  const float PcZ = gemm3(T + 8, P[0], P[1], P[2], T[11]);
  if (PcZ < 0.0f) return;
  const float invz = __fdiv_rn(1.0f, PcZ);
  const float u = __fadd_rn(__fmul_rn(__fmul_rn(f.fx, PcX), invz), f.cx);
  const float v = __fadd_rn(__fmul_rn(__fmul_rn(f.fy, PcY), invz), f.cy);
  if (u < f.min_x || u > f.max_x) return;
  if (v < f.min_y || v > f.max_y) return;
  const float maxDistance = __fmul_rn(1.2f, f.max_dist[i]);     // GetMaxDistanceInvariance (src/MapPoint.cc:436-437)
  const float minDistance = __fmul_rn(0.8f, f.min_dist[i]);
  float Ow[3];
#pragma unroll
  for (int a = 0; a < 3; ++a)   // mOw = -mRwc*mtcw (src/Frame.cc:373): small-matrix gemm, float accumulation
    Ow[a] = -__fadd_rn(__fadd_rn(__fmul_rn(T[0 * 4 + a], T[3]), __fmul_rn(T[1 * 4 + a], T[7])), __fmul_rn(T[2 * 4 + a], T[11]));
  const float PO[3] = {__fsub_rn(P[0], Ow[0]), __fsub_rn(P[1], Ow[1]), __fsub_rn(P[2], Ow[2])};
  double n2 = 0, dot = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    n2 = __dadd_rn(n2, __dmul_rn((double)PO[a], (double)PO[a]));
    dot = __dadd_rn(dot, __dmul_rn((double)PO[a], (double)f.normal[3 * i + a]));
  }
  const float dist = (float)sqrt(n2);
  if (dist < minDistance || dist > maxDistance) return;
  const float viewCos = (float)__ddiv_rn(dot, (double)dist);
  if (viewCos < f.cos_limit) return;
  const float ratio = __fdiv_rn(f.max_dist[i], dist);           // MapPoint::PredictScale (src/MapPoint.cc:463-478)
  int lvl = 0;
  for (int k = 0; k < f.nlevels - 1; ++k) lvl += (ratio > f.level_thr[k]) ? 1 : 0;
  in_view[i] = 1;
  px[i] = u; py[i] = v;
  pxr[i] = __fsub_rn(u, __fmul_rn(f.bf, invz));
  level[i] = lvl;
  vcos[i] = viewCos;
}

// cv::undistortPoints(src, dst, K, distCoeffs, R = I, P = K): 5 fixed-point iterations in double (OpenCV's default
// termination criteria), result stored as float.  k = k1 k2 p1 p2 k3.
struct UndistortParams { double fx, fy, cx, cy, k[5]; };
__global__ void k_undistort_points(UndistortParams p, const float* __restrict__ in, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double ifx = __ddiv_rn(1.0, p.fx), ify = __ddiv_rn(1.0, p.fy);
  const double u = in[2 * i], v = in[2 * i + 1];
  double x = __dmul_rn(__dsub_rn(u, p.cx), ifx), y = __dmul_rn(__dsub_rn(v, p.cy), ify);
  const double x0 = x, y0 = y;
  for (int j = 0; j < 5; ++j) {
    const double r2 = __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y));
    const double poly = __dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.k[4], r2), p.k[1]), r2), p.k[0]), r2);
    const double icdist = __ddiv_rn(1.0, __dadd_rn(1.0, poly));
    if (icdist < 0) { x = x0; y = y0; break; }
    const double dx = __dadd_rn(__dmul_rn(__dmul_rn(__dmul_rn(2.0, p.k[2]), x), y),
                                __dmul_rn(p.k[3], __dadd_rn(r2, __dmul_rn(__dmul_rn(2.0, x), x))));
    const double dy = __dadd_rn(__dmul_rn(p.k[2], __dadd_rn(r2, __dmul_rn(__dmul_rn(2.0, y), y))),
                                __dmul_rn(__dmul_rn(__dmul_rn(2.0, p.k[3]), x), y));
    x = __dmul_rn(__dsub_rn(x0, dx), icdist);
    y = __dmul_rn(__dsub_rn(y0, dy), icdist);
  }
  out[2 * i] = (float)__dadd_rn(__dmul_rn(x, p.fx), p.cx);
  out[2 * i + 1] = (float)__dadd_rn(__dmul_rn(y, p.fy), p.cy);
}

}  // namespace b200
