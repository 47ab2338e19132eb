// oracle/homo_harness.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
//
// C entry points around the `perfect` tree's OWN translation units for the point-pair overload of
// ORBmatcher::SearchByProjection(CurrentFrame, LastFrame, th, bMono, points_last, points_current)
// (perfect/src/ORBmatcher.cc:1727-1880) that TrackHomo calls (perfect/src/Tracking.cc:1331-1399).  homo_pairs fills
// perfect-tree Frames and MapPoints from the flat views of include/b200orb.h (the way oracle/refsrc_harness.cpp does for
// the T tree) and calls the overload; homo_sequence replays the matcher calls of one RGB-D frame of the perfect tree's
// Tracking on its images (TrackHomo, the masked constructor, TrackWithMotionModel).  Nothing here restates reference logic.
//
// oracle/homo.mk compiles this file twice: with the perfect tree's own ORBextractor.cc / ORBmatcher.cc / Frame.cc /
// KeyFrame.cc / MapPoint.cc / Map.cc into _ref/libhomoref.so (exports refperfect_homo_*), and with -DREFSRC_SHIM against
// the shims, with the perfect tree's Frame.cc / KeyFrame.cc / MapPoint.cc / Map.cc on top of libb200orb.so, into
// _ref/libshimperfect.so (exports shimperfect_homo_*).  tests/test_homo_pairs_gpu.py asserts shimperfect_* ==
// refperfect_*, tests/test_homo_pairs_cpu.py the restatement == refperfect_homo_pairs.
//
// The quad-tree's list nodes come from a bump arena (as in oracle/refperfect_harness.cpp: DistributeOctTree orders
// equal-size nodes by heap address, perfect/src/ORBextractor.cc, so two extractions of one image only agree in ORDER when
// "higher address" means "created later" in both).
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <list>
#include <map>
#include <mutex>
#include <new>
#include <vector>

#include "../include/b200orb.h"

#define private public
#define protected public
#include "ORBextractor.h"
#include "ORBmatcher.h"
#include "Frame.h"
#include "KeyFrame.h"
#include "MapPoint.h"
#include "Map.h"
#include "KeyFrameDatabase.h"
#undef private
#undef protected

namespace ORB_SLAM2 {
// out-of-path symbols the translation units leave undefined: the key-frame database (KeyFrame::SetBadFlag; the shim build
// has shim/KeyFrameDatabase.h) and the two quaternion helpers of the perfect tree's map save / load (perfect/src/Map.cc:
// 163,354; Eigen is absent).  Never reached.
#ifndef REFSRC_SHIM
void KeyFrameDatabase::erase(KeyFrame*) {}
#endif
std::vector<float> Converter::toQuaternion(const cv::Mat&) { abort(); }
void Converter::RmatOfQuat(cv::Mat&, const cv::Mat&) { abort(); }
}  // namespace ORB_SLAM2

using namespace ORB_SLAM2;

#ifdef REFSRC_SHIM
#define P(name) shimperfect_##name
#else
#define P(name) refperfect_##name
#endif

namespace {
#ifdef REFSRC_SHIM
const size_t kNodeBytes = 0;   // no quad-tree on the host in the shim build
#else
const size_t kNodeBytes = sizeof(std::_List_node<ExtractorNode>);
#endif
const size_t kArenaBytes = 16u << 20;
char* g_arena = nullptr;
size_t g_used = 0;
bool g_on = false;
std::mutex g_mu;   // Frame keeps intrinsics / bounds in statics, the arena is global: one call at a time
void arena_reset() {
  if (!g_arena) g_arena = (char*)malloc(kArenaBytes);
  g_used = 0;
  g_on = g_arena != nullptr;
}
}  // namespace
void* operator new(size_t n) {
  if (g_on && kNodeBytes && n == kNodeBytes && g_used + ((n + 15) & ~size_t(15)) <= kArenaBytes) {
    void* p = g_arena + g_used;
    g_used += (n + 15) & ~size_t(15);
    return p;
  }
  void* p = malloc(n ? n : 1);
  if (!p) throw std::bad_alloc();
  return p;
}
void operator delete(void* p) noexcept {
  if (g_arena && (char*)p >= g_arena && (char*)p < g_arena + kArenaBytes) return;
  free(p);
}
void operator delete(void* p, size_t) noexcept { operator delete(p); }

namespace {
Map g_map;

cv::Mat mat44(const float* T) {
  cv::Mat m(4, 4, CV_32F);
  memcpy(m.data, T, 16 * sizeof(float));
  return m;
}
void copy_tables(Frame* F, const float* sf, int nlevels) {
  F->mnScaleLevels = nlevels;
  F->mfScaleFactor = nlevels > 1 ? sf[1] : 1.2f;
  F->mfLogScaleFactor = log(F->mfScaleFactor);
  F->mvScaleFactors.assign(sf, sf + nlevels);
  F->mvInvScaleFactors.resize(nlevels); F->mvLevelSigma2.resize(nlevels); F->mvInvLevelSigma2.resize(nlevels);
  for (int l = 0; l < nlevels; ++l) {
    F->mvInvScaleFactors[l] = 1.0f / F->mvScaleFactors[l];
    F->mvLevelSigma2[l] = F->mvScaleFactors[l] * F->mvScaleFactors[l];
    F->mvInvLevelSigma2[l] = 1.0f / F->mvLevelSigma2[l];
  }
}
// mvKeys[i].pt = kxy[i] (the distorted keypoint; NULL: the undistorted one), mvKeysUn[i] from the flat view
void fill_keys(Frame* F, int n, const float* x, const float* y, const int32_t* oct, const float* ang, const float* kxy) {
  F->N = n;
  F->mvKeys.resize(n); F->mvKeysUn.resize(n);
  for (int i = 0; i < n; ++i) {
    F->mvKeysUn[i] = cv::KeyPoint(x[i], y[i], 31.f, ang[i], 0.f, oct[i]);
    F->mvKeys[i] = kxy ? cv::KeyPoint(kxy[2 * i], kxy[2 * i + 1], 31.f, ang[i], 0.f, oct[i]) : F->mvKeysUn[i];
  }
  F->mvpMapPoints.assign(n, static_cast<MapPoint*>(NULL));
  F->mvbOutlier.assign(n, false);
}
// the current Frame as the RGB-D constructor leaves it (perfect/src/Frame.cc:255-322) minus the extraction; sets the statics
Frame* current_frame(const OrbmFrame* f, const float* kxy) {
  Frame* F = new Frame();
  F->mpORBvocabulary = nullptr; F->mpORBextractorLeft = nullptr; F->mpORBextractorRight = nullptr;
  F->mnId = Frame::nNextId++;
  F->mbf = f->bf; F->mb = f->b; F->mThDepth = 40.0f * f->b;
  fill_keys(F, f->n, f->x, f->y, f->octave, f->angle, kxy);
  F->mvuRight.assign(f->uright, f->uright + f->n);
  F->mvDepth.assign(f->n, -1.f);
  F->mDescriptors.create(f->n, 32, CV_8U);
  if (f->n) memcpy(F->mDescriptors.data, f->desc, (size_t)f->n * 32);
  copy_tables(F, f->scale_factors, f->nlevels);
  Frame::fx = f->fx; Frame::fy = f->fy; Frame::cx = f->cx; Frame::cy = f->cy;
  Frame::invfx = 1.0f / f->fx; Frame::invfy = 1.0f / f->fy;
  Frame::mnMinX = f->min_x; Frame::mnMaxX = f->max_x; Frame::mnMinY = f->min_y; Frame::mnMaxY = f->max_y;
  Frame::mfGridElementWidthInv = static_cast<float>(FRAME_GRID_COLS) / static_cast<float>(Frame::mnMaxX - Frame::mnMinX);
  Frame::mfGridElementHeightInv = static_cast<float>(FRAME_GRID_ROWS) / static_cast<float>(Frame::mnMaxY - Frame::mnMinY);
  Frame::mbInitialComputations = false;
  F->mK = cv::Mat::eye(3, 3, CV_32F);
  F->mK.at<float>(0, 0) = f->fx; F->mK.at<float>(1, 1) = f->fy; F->mK.at<float>(0, 2) = f->cx; F->mK.at<float>(1, 2) = f->cy;
  F->mDistCoef = cv::Mat::zeros(4, 1, CV_32F);
  F->AssignFeaturesToGrid();
  F->SetPose(mat44(f->Tcw));
  return F;
}
// the last Frame: what the search reads of it (N, mvpMapPoints, mvbOutlier, mvKeys[i].octave / .pt, mvKeysUn[i].angle, mTcw)
// plus one MapPoint per valid or outlier entry, made by the MapPoint(Pos, Map*, Frame*, idx) constructor with this frame
// (its descriptor row is the MapPoint's); the statics are left alone.  id[mp] = i.
Frame* last_frame(const OrbmLast* l, const float* kxy, const uint8_t* outlier, const float* sf, int nlevels,
                  std::map<MapPoint*, int>& id) {
  Frame* F = new Frame();
  F->mpORBvocabulary = nullptr; F->mpORBextractorLeft = nullptr; F->mpORBextractorRight = nullptr;
  F->mnId = Frame::nNextId++;
  std::vector<float> zf(l->n, 0.f);
  fill_keys(F, l->n, zf.data(), zf.data(), l->octave, l->angle, kxy);
  F->mvuRight.assign(l->n, -1.f);
  F->mvDepth.assign(l->n, -1.f);
  F->mDescriptors.create(l->n, 32, CV_8U);
  if (l->n) memcpy(F->mDescriptors.data, l->mp_desc, (size_t)l->n * 32);
  copy_tables(F, sf, nlevels);
  F->SetPose(mat44(l->Tcw));
  for (int i = 0; i < l->n; ++i) {
    const bool out = outlier && outlier[i];
    if (!l->valid[i] && !out) continue;
    cv::Mat pos(3, 1, CV_32F);
    memcpy(pos.data, l->xw + 3 * (size_t)i, 12);
    MapPoint* mp = new MapPoint(pos, &g_map, F, i);
    mp->nObs = l->mp_obs ? l->mp_obs[i] : 0;
    F->mvpMapPoints[i] = mp;
    F->mvbOutlier[i] = out;
    id[mp] = i;
  }
  return F;
}
void flatten(const std::vector<MapPoint*>& v, const std::map<MapPoint*, int>& id, int32_t* out) {
  for (size_t j = 0; j < v.size(); ++j) out[j] = v[j] ? id.at(v[j]) : -1;
}
void put_points(const std::vector<cv::Point2f>& v, float* out) {
  for (size_t k = 0; k < v.size(); ++k) { out[2 * k] = v[k].x; out[2 * k + 1] = v[k].y; }
}
void release(Frame* L, std::map<MapPoint*, int>& id) {
  for (auto& kv : id) delete kv.first;
  delete L;
}
}  // namespace

extern "C" {

// gray u8, depth f32 metres, mask u8, all rows x cols.  kps_* : cap x 28 bytes (cv::KeyPoint), desc_* : cap x 32.
// -> 0, or -2 when cap is too small.
// ORBmatcher::SearchByProjection(CurrentFrame, LastFrame, th, bMono, points_last, points_current) of the perfect tree
// (perfect/src/ORBmatcher.cc:1727-1880) on flat views.  cur_kxy / last_kxy: n x 2 distorted keypoints (mvKeys[i].pt; NULL:
// the undistorted ones), last_outlier: mvbOutlier (NULL: none; an outlier entry still gets its MapPoint).  cur->mp_obs is
// not read: the current frame starts with no MapPoints, as TrackHomo leaves it (perfect/src/Tracking.cc:1352).
// pts_last / pts_cur: cap x 2 floats holding *n_last / *n_cur points on entry; the call appends to them.
// -> 0, or -2 when cap is too small (nothing is written then).
int P(homo_pairs)(const OrbmFrame* cur, const float* cur_kxy, const OrbmLast* last, const float* last_kxy,
                  const uint8_t* last_outlier, float th, int mono, float nnratio, int check_ori, int32_t* cur2last,
                  float* pts_last, int* n_last, float* pts_cur, int* n_cur, int cap, int* nmatches_out) {
  std::lock_guard<std::mutex> lk(g_mu);
  std::map<MapPoint*, int> id;
  Frame* L = last_frame(last, last_kxy, last_outlier, cur->scale_factors, cur->nlevels, id);
  Frame* C = current_frame(cur, cur_kxy);
  std::vector<cv::Point2f> pl(*n_last), pc(*n_cur);
  for (int k = 0; k < *n_last; ++k) pl[k] = cv::Point2f(pts_last[2 * k], pts_last[2 * k + 1]);
  for (int k = 0; k < *n_cur; ++k) pc[k] = cv::Point2f(pts_cur[2 * k], pts_cur[2 * k + 1]);
  ORBmatcher m(nnratio, check_ori != 0);
  *nmatches_out = m.SearchByProjection(*C, *L, th, mono != 0, pl, pc);
  flatten(C->mvpMapPoints, id, cur2last);
  int rc = -2;
  if ((int)pl.size() <= cap && (int)pc.size() <= cap) {
    put_points(pl, pts_last); put_points(pc, pts_cur);
    *n_last = (int)pl.size(); *n_cur = (int)pc.size();
    rc = 0;
  }
  delete C;
  release(L, id);
  return rc;
}

// The matcher calls of one RGB-D frame of the perfect tree's Tracking, on the images: the plain constructor
// (perfect/src/Tracking.cc:685); TrackHomo's search at th, cleared and repeated at 2*th below 20 matches (:1349-1373); the
// masked constructor (:716); TrackWithMotionModel's search, likewise (:1922-1940).  Both frames take the pose Tcw (what
// mVelocity * mLastFrame.mTcw gives); the last frame comes from the flat view as in homo_pairs.  Returns, for the homo
// step: both point vectors, nmatches, the plain frame's N and pointer state; for the motion step: nmatches, the masked
// frame's N and pointer state.  -> 0, or -2 when cap is too small.
int P(homo_sequence)(const uint8_t* gray, const float* depth, const uint8_t* mask, int rows, int cols, int nfeatures,
                     float scaleFactor, int nlevels, int iniTh, int minTh, float fx, float fy, float cx, float cy, float bf,
                     const float* Tcw, const OrbmLast* last, const float* last_kxy, const uint8_t* last_outlier, int th,
                     int mono, float* pts_last, float* pts_cur, int* n_pts, int32_t* homo_c2l, int* homo_n, int* homo_nm,
                     int32_t* track_c2l, int* track_n, int* track_nm, int cap) {
  std::lock_guard<std::mutex> lk(g_mu);
  ORBextractor ex(nfeatures, scaleFactor, nlevels, iniTh, minTh);
  cv::Mat K = cv::Mat::eye(3, 3, CV_32F);
  K.at<float>(0, 0) = fx; K.at<float>(1, 1) = fy; K.at<float>(0, 2) = cx; K.at<float>(1, 2) = cy;
  cv::Mat D = cv::Mat::zeros(4, 1, CV_32F);
  cv::Mat g(rows, cols, CV_8UC1, (void*)gray), d(rows, cols, CV_32F, (void*)depth), m(rows, cols, CV_8UC1, (void*)mask);
  const float thDepth = bf * 40.0f / fx;
  Frame::mbInitialComputations = true;
  arena_reset();
  Frame A(g, d, 0.0, &ex, nullptr, K, D, bf, thDepth);
  g_on = false;
  std::map<MapPoint*, int> id;
  Frame* L = last_frame(last, last_kxy, last_outlier, A.mvScaleFactors.data(), A.mnScaleLevels, id);
  ORBmatcher matcher(0.9, true);
  A.SetPose(mat44(Tcw));
  std::fill(A.mvpMapPoints.begin(), A.mvpMapPoints.end(), static_cast<MapPoint*>(NULL));
  std::vector<cv::Point2f> pl, pc;
  int nm = matcher.SearchByProjection(A, *L, th, mono != 0, pl, pc);
  if (nm < 20) {
    pl.clear(); pc.clear();
    std::fill(A.mvpMapPoints.begin(), A.mvpMapPoints.end(), static_cast<MapPoint*>(NULL));
    nm = matcher.SearchByProjection(A, *L, 2 * th, mono != 0, pl, pc);
  }
  *homo_nm = nm; *homo_n = A.N; *n_pts = (int)pl.size();
  int rc = -2;
  if (A.N <= cap && (int)pl.size() <= cap && pl.size() == pc.size()) {
    flatten(A.mvpMapPoints, id, homo_c2l);
    put_points(pl, pts_last); put_points(pc, pts_cur);
    rc = 0;
  }
  arena_reset();
  Frame B(g, d, m, 0.0, &ex, nullptr, K, D, bf, thDepth);
  g_on = false;
  B.SetPose(mat44(Tcw));
  std::fill(B.mvpMapPoints.begin(), B.mvpMapPoints.end(), static_cast<MapPoint*>(NULL));
  nm = matcher.SearchByProjection(B, *L, th, mono != 0);
  if (nm < 20) {
    std::fill(B.mvpMapPoints.begin(), B.mvpMapPoints.end(), static_cast<MapPoint*>(NULL));
    nm = matcher.SearchByProjection(B, *L, 2 * th, mono != 0);
  }
  *track_nm = nm; *track_n = B.N;
  if (B.N <= cap) flatten(B.mvpMapPoints, id, track_c2l);
  else rc = -2;
  release(L, id);
  return rc;
}

}  // extern "C"
