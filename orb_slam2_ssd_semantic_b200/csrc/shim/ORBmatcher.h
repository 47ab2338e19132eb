// shim/ORBmatcher.h -- drop-in for the reference's include/ORBmatcher.h: same include guard, namespace, class name and
// the complete public surface (include/ORBmatcher.h:37-118), implemented on top of the C-ABI of libb200orb.so.
// Put this directory BEFORE the reference's include/ on the include path: Tracking.cc, LocalMapping.cc, LoopClosing.cc,
// Frame.cc, KeyFrame.cc, MapPoint.cc, Sim3Solver.cc then compile unchanged (the GPU test suite does exactly that with the
// reference's own Frame.cc / KeyFrame.cc / MapPoint.cc: oracle/Makefile, target `shim`).
// The same header stands in for perfect/include/ORBmatcher.h, which declares one member more: the 2-D point-pair overload
// of SearchByProjection(Frame&, const Frame&, ...) that the perfect tree's TrackHomo calls (perfect/include/ORBmatcher.h:
// 64-68).  The T tree never calls it, so there the extra member does nothing (oracle/homo.mk builds the perfect
// tree's Frame.cc / KeyFrame.cc / MapPoint.cc / Map.cc against this directory).
//
// The reference's searches walk and MUTATE the Frame / KeyFrame / MapPoint object graph.  Each member below
//   1. flattens what the search reads into the array views of include/b200orb.h; the few scalar lines per MapPoint that
//      set up a query (projection, distance / viewing-angle gates, PredictScale, radius) run here with the reference's own
//      cv::Mat expressions and the reference's own MapPoint / KeyFrame methods, so their arithmetic is the reference's;
//   2. calls the GPU for everything that is data-parallel: window walks, Hamming distances, the ordered "already matched"
//      rule, rotation histograms;
//   3. applies the pointer mutations on the host in the reference's order.
#ifndef ORBMATCHER_H
#define ORBMATCHER_H

#include <climits>
#include <cmath>
#include <cstring>
#include <set>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include <opencv2/core/core.hpp>
#include <opencv2/features2d/features2d.hpp>

#include "MapPoint.h"
#include "KeyFrame.h"
#include "Frame.h"

#include "b200orb.h"

namespace ORB_SLAM2 {

class ORBmatcher {
 public:
  ORBmatcher(float nnratio = 0.6, bool checkOri = true) : mfNNratio(nnratio), mbCheckOrientation(checkOri) { open(); }
  ORBmatcher(const ORBmatcher& o) : mfNNratio(o.mfNNratio), mbCheckOrientation(o.mbCheckOrientation) { open(); }
  ORBmatcher& operator=(const ORBmatcher& o) { mfNNratio = o.mfNNratio; mbCheckOrientation = o.mbCheckOrientation; return *this; }
  ~ORBmatcher() { orbm_destroy(h_); }

  // src/ORBmatcher.cc:1968-1984
  static int DescriptorDistance(const cv::Mat& a, const cv::Mat& b) { return orbm_hamming(a.ptr(0), b.ptr(0)); }

  // ---- src/ORBmatcher.cc:63-156 --------------------------------------------------------------------------------------
  int SearchByProjection(Frame& F, const std::vector<MapPoint*>& vpMapPoints, const float th = 3) {
    FlatFrame cur;
    flatten(F, cur, true);
    const int np = (int)vpMapPoints.size();
    std::vector<uint8_t> inview(np, 0), desc((size_t)(np > 0 ? np : 1) * 32, 0);
    std::vector<float> px(np), py(np), pxr(np), vc(np);
    std::vector<int32_t> lvl(np, 0), obs(np, 0);
    for (int i = 0; i < np; ++i) {
      MapPoint* pMP = vpMapPoints[i];
      if (!pMP->mbTrackInView || pMP->isBad()) continue;
      inview[i] = 1;
      px[i] = pMP->mTrackProjX; py[i] = pMP->mTrackProjY; pxr[i] = pMP->mTrackProjXR;
      lvl[i] = pMP->mnTrackScaleLevel; vc[i] = pMP->mTrackViewCos; obs[i] = pMP->Observations();
      cv::Mat d = pMP->GetDescriptor();
      std::memcpy(&desc[(size_t)i * 32], d.ptr(0), 32);
    }
    OrbmTrackPoints P;
    P.n = np; P.track_in_view = inview.data(); P.proj_x = px.data(); P.proj_y = py.data(); P.proj_xr = pxr.data();
    P.scale_level = lvl.data(); P.view_cos = vc.data(); P.mp_desc = desc.data(); P.mp_obs = obs.data();
    std::vector<int32_t> f2p(cur.n > 0 ? cur.n : 1, -1);
    int nmatches = 0;
    check(orbm_search_by_projection_points(h_, &cur.view, &P, th, mfNNratio, f2p.data(), &nmatches));
    for (int j = 0; j < cur.n; ++j)
      if (f2p[j] >= 0) F.mvpMapPoints[j] = vpMapPoints[f2p[j]];
    return nmatches;
  }

  // ---- src/ORBmatcher.cc:1578-1724 -----------------------------------------------------------------------------------
  int SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono) {
    return search_last(CurrentFrame, LastFrame, th, bMono, NULL);
  }

  // ---- perfect/src/ORBmatcher.cc:1727-1880 (TrackHomo, perfect/src/Tracking.cc:1362,1371) ----------------------------
  // The search above plus one point pair per accepted query, pushed before the rotation prune (:1835-1836): the prune
  // leaves the pairs it unmatches in place.  Appends, never clears; the points are the distorted mvKeys.
  int SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono,
                         std::vector<cv::Point2f>& points_last, std::vector<cv::Point2f>& points_current) {
    std::vector<int32_t> acc;
    const int nmatches = search_last(CurrentFrame, LastFrame, th, bMono, &acc);
    for (int i = 0; i < LastFrame.N; ++i)
      if (acc[i] >= 0) {
        points_last.push_back(LastFrame.mvKeys[i].pt);
        points_current.push_back(CurrentFrame.mvKeys[acc[i]].pt);
      }
    return nmatches;
  }

  // ---- src/ORBmatcher.cc:1757-1899 (relocalisation) -------------------------------------------------------------------
  int SearchByProjection(Frame& CurrentFrame, KeyFrame* pKF, const std::set<MapPoint*>& sAlreadyFound, const float th,
                         const int ORBdist) {
    const cv::Mat Rcw = CurrentFrame.mTcw.rowRange(0, 3).colRange(0, 3);
    const cv::Mat tcw = CurrentFrame.mTcw.rowRange(0, 3).col(3);
    const cv::Mat Ow = -Rcw.t() * tcw;
    const std::vector<MapPoint*> vpMPs = pKF->GetMapPointMatches();
    Queries Q((int)vpMPs.size(), false, true);
    for (size_t i = 0, iend = vpMPs.size(); i < iend; i++) {
      MapPoint* pMP = vpMPs[i];
      if (!pMP || pMP->isBad() || sAlreadyFound.count(pMP)) continue;
      cv::Mat x3Dw = pMP->GetWorldPos();
      cv::Mat x3Dc = Rcw * x3Dw + tcw;
      const float xc = x3Dc.at<float>(0);
      const float yc = x3Dc.at<float>(1);
      const float invzc = 1.0 / x3Dc.at<float>(2);
      const float u = CurrentFrame.fx * xc * invzc + CurrentFrame.cx;
      const float v = CurrentFrame.fy * yc * invzc + CurrentFrame.cy;
      if (u < CurrentFrame.mnMinX || u > CurrentFrame.mnMaxX) continue;
      if (v < CurrentFrame.mnMinY || v > CurrentFrame.mnMaxY) continue;
      cv::Mat PO = x3Dw - Ow;
      float dist3D = cv::norm(PO);
      const float maxDistance = pMP->GetMaxDistanceInvariance();
      const float minDistance = pMP->GetMinDistanceInvariance();
      if (dist3D < minDistance || dist3D > maxDistance) continue;
      int nPredictedLevel = pMP->PredictScale(dist3D, &CurrentFrame);
      const float radius = th * CurrentFrame.mvScaleFactors[nPredictedLevel];
      Q.set((int)i, u, v, radius, nPredictedLevel - 1, nPredictedLevel + 1, pMP, pKF->mvKeysUn[i].angle, 0.f);
    }
    FlatFrame cur;
    flatten(CurrentFrame, cur, true);
    std::vector<int32_t> c2q(cur.n > 0 ? cur.n : 1, -1);
    int nmatches = 0;
    OrbmQueries q = Q.view();
    check(orbm_search_projected(h_, &cur.view, &q, ORBdist, /*claim_rule=*/1, mbCheckOrientation ? 1 : 0, c2q.data(), &nmatches));
    for (int j = 0; j < cur.n; ++j) {
      if (c2q[j] >= 0) CurrentFrame.mvpMapPoints[j] = vpMPs[c2q[j]];
      else if (c2q[j] == -1) CurrentFrame.mvpMapPoints[j] = static_cast<MapPoint*>(NULL);
    }
    return nmatches;
  }

  // ---- src/ORBmatcher.cc:378-498 (loop closing) ------------------------------------------------------------------------
  int SearchByProjection(KeyFrame* pKF, cv::Mat Scw, const std::vector<MapPoint*>& vpPoints, std::vector<MapPoint*>& vpMatched,
                         int th) {
    const float& fx = pKF->fx;
    const float& fy = pKF->fy;
    const float& cx = pKF->cx;
    const float& cy = pKF->cy;
    cv::Mat sRcw = Scw.rowRange(0, 3).colRange(0, 3);
    const float scw = sqrt(sRcw.row(0).dot(sRcw.row(0)));
    cv::Mat Rcw = sRcw / scw;
    cv::Mat tcw = Scw.rowRange(0, 3).col(3) / scw;
    cv::Mat Ow = -Rcw.t() * tcw;
    std::set<MapPoint*> spAlreadyFound(vpMatched.begin(), vpMatched.end());
    spAlreadyFound.erase(static_cast<MapPoint*>(NULL));
    Queries Q((int)vpPoints.size(), false, false);
    for (int iMP = 0, iendMP = (int)vpPoints.size(); iMP < iendMP; iMP++) {
      MapPoint* pMP = vpPoints[iMP];
      if (pMP->isBad() || spAlreadyFound.count(pMP)) continue;
      cv::Mat p3Dw = pMP->GetWorldPos();
      cv::Mat p3Dc = Rcw * p3Dw + tcw;
      if (p3Dc.at<float>(2) < 0.0) continue;
      const float invz = 1 / p3Dc.at<float>(2);
      const float x = p3Dc.at<float>(0) * invz;
      const float y = p3Dc.at<float>(1) * invz;
      const float u = fx * x + cx;
      const float v = fy * y + cy;
      if (!pKF->IsInImage(u, v)) continue;
      const float maxDistance = pMP->GetMaxDistanceInvariance();
      const float minDistance = pMP->GetMinDistanceInvariance();
      cv::Mat PO = p3Dw - Ow;
      const float dist = cv::norm(PO);
      if (dist < minDistance || dist > maxDistance) continue;
      cv::Mat Pn = pMP->GetNormal();
      if (PO.dot(Pn) < 0.5 * dist) continue;
      int nPredictedLevel = pMP->PredictScale(dist, pKF);
      const float radius = th * pKF->mvScaleFactors[nPredictedLevel];
      Q.set(iMP, u, v, radius, nPredictedLevel - 1, nPredictedLevel, pMP, 0.f, 0.f);
    }
    FlatFrame kf;
    flatten_kf(pKF, kf);
    for (int j = 0; j < kf.n; ++j) kf.obs[j] = vpMatched[j] ? 1 : -1;   // `if(vpMatched[idx]) continue;` (:468-469)
    std::vector<int32_t> k2q(kf.n > 0 ? kf.n : 1, -1);
    int nmatches = 0;
    OrbmQueries q = Q.view();
    check(orbm_search_projected(h_, &kf.view, &q, TH_LOW, /*claim_rule=*/1, /*check_ori=*/0, k2q.data(), &nmatches));
    for (int j = 0; j < kf.n; ++j)
      if (k2q[j] >= 0) vpMatched[j] = vpPoints[k2q[j]];
    return nmatches;
  }

  // ---- src/ORBmatcher.cc:217-363 -------------------------------------------------------------------------------------
  int SearchByBoW(KeyFrame* pKF, Frame& F, std::vector<MapPoint*>& vpMapPointMatches) {
    const std::vector<MapPoint*> vpMapPointsKF = pKF->GetMapPointMatches();
    FlatBow kf, fr;
    flatten_bow(pKF->mDescriptors, pKF->mvKeysUn, pKF->mFeatVec, &vpMapPointsKF, kf);
    flatten_bow(F.mDescriptors, F.mvKeys, F.mFeatVec, (const std::vector<MapPoint*>*)NULL, fr);   // mvKeys: :308
    std::vector<int32_t> f2kf(fr.view.n > 0 ? fr.view.n : 1, -1);
    int nmatches = 0;
    check(orbm_search_by_bow(h_, &kf.view, &fr.view, mfNNratio, mbCheckOrientation ? 1 : 0, f2kf.data(), &nmatches));
    vpMapPointMatches = std::vector<MapPoint*>(F.N, static_cast<MapPoint*>(NULL));
    for (int i = 0; i < F.N; ++i)
      if (f2kf[i] >= 0) vpMapPointMatches[i] = vpMapPointsKF[f2kf[i]];
    return nmatches;
  }

  // ---- src/ORBmatcher.cc:665-812 -------------------------------------------------------------------------------------
  int SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, std::vector<MapPoint*>& vpMatches12) {
    const std::vector<MapPoint*> vpMapPoints1 = pKF1->GetMapPointMatches(), vpMapPoints2 = pKF2->GetMapPointMatches();
    FlatBow k1, k2;
    flatten_bow(pKF1->mDescriptors, pKF1->mvKeysUn, pKF1->mFeatVec, &vpMapPoints1, k1);
    flatten_bow(pKF2->mDescriptors, pKF2->mvKeysUn, pKF2->mFeatVec, &vpMapPoints2, k2);
    std::vector<int32_t> m12(k1.view.n > 0 ? k1.view.n : 1, -1);
    int nmatches = 0;
    check(orbm_search_by_bow_kf(h_, &k1.view, &k2.view, mfNNratio, mbCheckOrientation ? 1 : 0, m12.data(), &nmatches));
    vpMatches12 = std::vector<MapPoint*>(vpMapPoints1.size(), static_cast<MapPoint*>(NULL));
    for (size_t i = 0; i < vpMapPoints1.size(); ++i)
      if (m12[i] >= 0) vpMatches12[i] = vpMapPoints2[m12[i]];
    return nmatches;
  }

  // ---- src/ORBmatcher.cc:523-651 -------------------------------------------------------------------------------------
  int SearchForInitialization(Frame& F1, Frame& F2, std::vector<cv::Point2f>& vbPrevMatched, std::vector<int>& vnMatches12,
                              int windowSize = 10) {
    FlatFrame f1, f2;
    flatten(F1, f1, false);
    flatten(F2, f2, false);
    const int n1 = (int)F1.mvKeysUn.size();
    std::vector<float> prev((size_t)(n1 > 0 ? n1 : 1) * 2);
    for (int i = 0; i < n1; ++i) { prev[2 * i] = vbPrevMatched[i].x; prev[2 * i + 1] = vbPrevMatched[i].y; }
    std::vector<int32_t> m12(n1 > 0 ? n1 : 1, -1);
    int nmatches = 0;
    check(orbm_search_for_initialization(h_, &f1.view, &f2.view, prev.data(), windowSize, mfNNratio, mbCheckOrientation ? 1 : 0,
                                         m12.data(), &nmatches));
    vnMatches12 = std::vector<int>(n1, -1);
    for (int i = 0; i < n1; ++i) {
      vnMatches12[i] = m12[i];
      if (m12[i] >= 0) vbPrevMatched[i] = F2.mvKeysUn[m12[i]].pt;   // :640-642
    }
    return nmatches;
  }

  // ---- src/ORBmatcher.cc:827-1019 ------------------------------------------------------------------------------------
  int SearchForTriangulation(KeyFrame* pKF1, KeyFrame* pKF2, cv::Mat F12, std::vector<std::pair<size_t, size_t> >& vMatchedPairs,
                             const bool bOnlyStereo) {
    // epipole of camera 1 in image 2 (:835-839)
    cv::Mat Cw = pKF1->GetCameraCenter();
    cv::Mat R2w = pKF2->GetRotation();
    cv::Mat t2w = pKF2->GetTranslation();
    cv::Mat C2 = R2w * Cw + t2w;
    const float invz = 1.0f / C2.at<float>(2);
    const float ex = pKF2->fx * C2.at<float>(0) * invz + pKF2->cx;
    const float ey = pKF2->fy * C2.at<float>(1) * invz + pKF2->cy;
    FlatTri k1, k2;
    flatten_tri(pKF1, k1);
    flatten_tri(pKF2, k2);
    float F[9];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) F[r * 3 + c] = F12.at<float>(r, c);
    std::vector<int32_t> m12(pKF1->N > 0 ? pKF1->N : 1, -1);
    int nmatches = 0;
    check(orbm_search_for_triangulation(h_, &k1.view, &k2.view, F, ex, ey, pKF2->mvScaleFactors.data(), pKF2->mvLevelSigma2.data(),
                                        (int)pKF2->mvScaleFactors.size(), bOnlyStereo ? 1 : 0, mbCheckOrientation ? 1 : 0, m12.data(),
                                        &nmatches));
    vMatchedPairs.clear();
    vMatchedPairs.reserve(nmatches);
    for (int i = 0; i < pKF1->N; ++i)
      if (m12[i] >= 0) vMatchedPairs.push_back(std::make_pair((size_t)i, (size_t)m12[i]));
    return nmatches;
  }

  // ---- src/ORBmatcher.cc:1334-1558 -----------------------------------------------------------------------------------
  int SearchBySim3(KeyFrame* pKF1, KeyFrame* pKF2, std::vector<MapPoint*>& vpMatches12, const float& s12, const cv::Mat& R12,
                   const cv::Mat& t12, const float th) {
    const float& fx = pKF1->fx;
    const float& fy = pKF1->fy;
    const float& cx = pKF1->cx;
    const float& cy = pKF1->cy;
    cv::Mat R1w = pKF1->GetRotation();
    cv::Mat t1w = pKF1->GetTranslation();
    cv::Mat R2w = pKF2->GetRotation();
    cv::Mat t2w = pKF2->GetTranslation();
    cv::Mat sR12 = s12 * R12;
    cv::Mat sR21 = (1.0 / s12) * R12.t();
    cv::Mat t21 = -sR21 * t12;
    const std::vector<MapPoint*> vpMapPoints1 = pKF1->GetMapPointMatches();
    const int N1 = (int)vpMapPoints1.size();
    const std::vector<MapPoint*> vpMapPoints2 = pKF2->GetMapPointMatches();
    const int N2 = (int)vpMapPoints2.size();
    std::vector<bool> vbAlreadyMatched1(N1, false);
    std::vector<bool> vbAlreadyMatched2(N2, false);
    for (int i = 0; i < N1; i++) {
      MapPoint* pMP = vpMatches12[i];
      if (pMP) {
        vbAlreadyMatched1[i] = true;
        int idx2 = pMP->GetIndexInKeyFrame(pKF2);
        if (idx2 >= 0 && idx2 < N2) vbAlreadyMatched2[idx2] = true;
      }
    }
    Queries Q1(N1, false, false), Q2(N2, false, false);
    for (int i1 = 0; i1 < N1; i1++) {     // points of pKF1 projected into pKF2 (:1387-1448)
      MapPoint* pMP = vpMapPoints1[i1];
      if (!pMP || vbAlreadyMatched1[i1]) continue;
      if (pMP->isBad()) continue;
      cv::Mat p3Dw = pMP->GetWorldPos();
      cv::Mat p3Dc1 = R1w * p3Dw + t1w;
      cv::Mat p3Dc2 = sR21 * p3Dc1 + t21;
      if (p3Dc2.at<float>(2) < 0.0) continue;
      const float invz = 1.0 / p3Dc2.at<float>(2);
      const float x = p3Dc2.at<float>(0) * invz;
      const float y = p3Dc2.at<float>(1) * invz;
      const float u = fx * x + cx;
      const float v = fy * y + cy;
      if (!pKF2->IsInImage(u, v)) continue;
      const float maxDistance = pMP->GetMaxDistanceInvariance();
      const float minDistance = pMP->GetMinDistanceInvariance();
      const float dist3D = cv::norm(p3Dc2);
      if (dist3D < minDistance || dist3D > maxDistance) continue;
      const int nPredictedLevel = pMP->PredictScale(dist3D, pKF2);
      const float radius = th * pKF2->mvScaleFactors[nPredictedLevel];
      Q1.set(i1, u, v, radius, nPredictedLevel - 1, nPredictedLevel, pMP, 0.f, 0.f);
    }
    for (int i2 = 0; i2 < N2; i2++) {     // points of pKF2 projected into pKF1 (:1460-1521)
      MapPoint* pMP = vpMapPoints2[i2];
      if (!pMP || vbAlreadyMatched2[i2]) continue;
      if (pMP->isBad()) continue;
      cv::Mat p3Dw = pMP->GetWorldPos();
      cv::Mat p3Dc2 = R2w * p3Dw + t2w;
      cv::Mat p3Dc1 = sR12 * p3Dc2 + t12;
      if (p3Dc1.at<float>(2) < 0.0) continue;
      const float invz = 1.0 / p3Dc1.at<float>(2);
      const float x = p3Dc1.at<float>(0) * invz;
      const float y = p3Dc1.at<float>(1) * invz;
      const float u = fx * x + cx;
      const float v = fy * y + cy;
      if (!pKF1->IsInImage(u, v)) continue;
      const float maxDistance = pMP->GetMaxDistanceInvariance();
      const float minDistance = pMP->GetMinDistanceInvariance();
      const float dist3D = cv::norm(p3Dc1);
      if (dist3D < minDistance || dist3D > maxDistance) continue;
      const int nPredictedLevel = pMP->PredictScale(dist3D, pKF1);
      const float radius = th * pKF1->mvScaleFactors[nPredictedLevel];
      Q2.set(i2, u, v, radius, nPredictedLevel - 1, nPredictedLevel, pMP, 0.f, 0.f);
    }
    FlatFrame k1, k2;
    flatten_kf(pKF1, k1);
    flatten_kf(pKF2, k2);
    std::vector<int32_t> b1(N1 > 0 ? N1 : 1, -1), d1(N1 > 0 ? N1 : 1, INT_MAX), b2(N2 > 0 ? N2 : 1, -1), d2(N2 > 0 ? N2 : 1, INT_MAX);
    OrbmQueries q1 = Q1.view(), q2 = Q2.view();
    check(orbm_search_best(h_, &k2.view, &q1, 0, NULL, b1.data(), d1.data()));
    check(orbm_search_best(h_, &k1.view, &q2, 0, NULL, b2.data(), d2.data()));
    std::vector<int> vnMatch1(N1, -1), vnMatch2(N2, -1);
    for (int i1 = 0; i1 < N1; ++i1) if (b1[i1] >= 0 && d1[i1] <= TH_HIGH) vnMatch1[i1] = b1[i1];
    for (int i2 = 0; i2 < N2; ++i2) if (b2[i2] >= 0 && d2[i2] <= TH_HIGH) vnMatch2[i2] = b2[i2];
    int nFound = 0;                       // cross check (:1524-1539)
    for (int i1 = 0; i1 < N1; i1++) {
      int idx2 = vnMatch1[i1];
      if (idx2 >= 0) {
        int idx1 = vnMatch2[idx2];
        if (idx1 == i1) { vpMatches12[i1] = vpMapPoints2[idx2]; nFound++; }
      }
    }
    return nFound;
  }

  // ---- src/ORBmatcher.cc:1031-1182 -----------------------------------------------------------------------------------
  int Fuse(KeyFrame* pKF, const std::vector<MapPoint*>& vpMapPoints, const float th = 3.0) {
    cv::Mat Rcw = pKF->GetRotation();
    cv::Mat tcw = pKF->GetTranslation();
    const float& fx = pKF->fx;
    const float& fy = pKF->fy;
    const float& cx = pKF->cx;
    const float& cy = pKF->cy;
    const float& bf = pKF->mbf;
    cv::Mat Ow = pKF->GetCameraCenter();
    const int nMPs = (int)vpMapPoints.size();
    Queries Q(nMPs, true, false);
    for (int i = 0; i < nMPs; i++) {      // query geometry of every candidate; the state tests run in the replay below
      MapPoint* pMP = vpMapPoints[i];
      if (!pMP) continue;
      cv::Mat p3Dw = pMP->GetWorldPos();
      cv::Mat p3Dc = Rcw * p3Dw + tcw;
      if (p3Dc.at<float>(2) < 0.0f) continue;
      const float invz = 1 / p3Dc.at<float>(2);
      const float x = p3Dc.at<float>(0) * invz;
      const float y = p3Dc.at<float>(1) * invz;
      const float u = fx * x + cx;
      const float v = fy * y + cy;
      if (!pKF->IsInImage(u, v)) continue;
      const float maxDistance = pMP->GetMaxDistanceInvariance();
      const float minDistance = pMP->GetMinDistanceInvariance();
      cv::Mat PO = p3Dw - Ow;
      const float dist3D = cv::norm(PO);
      if (dist3D < minDistance || dist3D > maxDistance) continue;
      cv::Mat Pn = pMP->GetNormal();
      if (PO.dot(Pn) < 0.5 * dist3D) continue;
      int nPredictedLevel = pMP->PredictScale(dist3D, pKF);
      const float radius = th * pKF->mvScaleFactors[nPredictedLevel];
      const float ur = u - bf * invz;
      Q.set(i, u, v, radius, nPredictedLevel - 1, nPredictedLevel, pMP, 0.f, ur);
    }
    FlatFrame kf;
    flatten_kf(pKF, kf);
    std::vector<int32_t> best(nMPs > 0 ? nMPs : 1, -1), bdist(nMPs > 0 ? nMPs : 1, INT_MAX);
    OrbmQueries q = Q.view();
    check(orbm_search_best(h_, &kf.view, &q, /*gate=*/1, pKF->mvInvLevelSigma2.data(), best.data(), bdist.data()));
    int nFused = 0;
    for (int i = 0; i < nMPs; i++) {      // :1044-1048, :1156-1178 in the reference's order, on the live graph
      MapPoint* pMP = vpMapPoints[i];
      if (!pMP) continue;
      if (pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;
      if (!Q.valid[i] || best[i] < 0) continue;
      if (bdist[i] <= TH_LOW) {
        const int bestIdx = best[i];
        MapPoint* pMPinKF = pKF->GetMapPoint(bestIdx);
        if (pMPinKF) {
          if (!pMPinKF->isBad()) {
            if (pMPinKF->Observations() > pMP->Observations()) pMP->Replace(pMPinKF);
            else pMPinKF->Replace(pMP);
          }
        } else {
          pMP->AddObservation(pKF, bestIdx);
          pKF->AddMapPoint(pMP, bestIdx);
        }
        nFused++;
      }
    }
    return nFused;
  }

  // ---- src/ORBmatcher.cc:1198-1318 -----------------------------------------------------------------------------------
  int Fuse(KeyFrame* pKF, cv::Mat Scw, const std::vector<MapPoint*>& vpPoints, float th, std::vector<MapPoint*>& vpReplacePoint) {
    const float& fx = pKF->fx;
    const float& fy = pKF->fy;
    const float& cx = pKF->cx;
    const float& cy = pKF->cy;
    cv::Mat sRcw = Scw.rowRange(0, 3).colRange(0, 3);
    const float scw = sqrt(sRcw.row(0).dot(sRcw.row(0)));
    cv::Mat Rcw = sRcw / scw;
    cv::Mat tcw = Scw.rowRange(0, 3).col(3) / scw;
    cv::Mat Ow = -Rcw.t() * tcw;
    const std::set<MapPoint*> spAlreadyFound = pKF->GetMapPoints();
    const int nPoints = (int)vpPoints.size();
    Queries Q(nPoints, false, false);
    for (int iMP = 0; iMP < nPoints; iMP++) {
      MapPoint* pMP = vpPoints[iMP];
      if (!pMP) continue;
      if (pMP->isBad() || spAlreadyFound.count(pMP)) continue;
      cv::Mat p3Dw = pMP->GetWorldPos();
      cv::Mat p3Dc = Rcw * p3Dw + tcw;
      if (p3Dc.at<float>(2) < 0.0f) continue;
      const float invz = 1.0 / p3Dc.at<float>(2);
      const float x = p3Dc.at<float>(0) * invz;
      const float y = p3Dc.at<float>(1) * invz;
      const float u = fx * x + cx;
      const float v = fy * y + cy;
      if (!pKF->IsInImage(u, v)) continue;
      const float maxDistance = pMP->GetMaxDistanceInvariance();
      const float minDistance = pMP->GetMinDistanceInvariance();
      cv::Mat PO = p3Dw - Ow;
      const float dist3D = cv::norm(PO);
      if (dist3D < minDistance || dist3D > maxDistance) continue;
      cv::Mat Pn = pMP->GetNormal();
      if (PO.dot(Pn) < 0.5 * dist3D) continue;
      int nPredictedLevel = pMP->PredictScale(dist3D, pKF);
      const float radius = th * pKF->mvScaleFactors[nPredictedLevel];
      Q.set(iMP, u, v, radius, nPredictedLevel - 1, nPredictedLevel, pMP, 0.f, 0.f);
    }
    FlatFrame kf;
    flatten_kf(pKF, kf);
    std::vector<int32_t> best(nPoints > 0 ? nPoints : 1, -1), bdist(nPoints > 0 ? nPoints : 1, INT_MAX);
    OrbmQueries q = Q.view();
    check(orbm_search_best(h_, &kf.view, &q, /*gate=*/0, NULL, best.data(), bdist.data()));
    int nFused = 0;
    for (int iMP = 0; iMP < nPoints; iMP++) {   // :1288-1312; the skip tests above do not depend on earlier iterations
      if (!Q.valid[iMP] || best[iMP] < 0) continue;
      MapPoint* pMP = vpPoints[iMP];
      if (bdist[iMP] <= TH_LOW) {
        const int bestIdx = best[iMP];
        MapPoint* pMPinKF = pKF->GetMapPoint(bestIdx);
        if (pMPinKF) {
          if (!pMPinKF->isBad()) vpReplacePoint[iMP] = pMPinKF;
        } else {
          pMP->AddObservation(pKF, bestIdx);
          pKF->AddMapPoint(pMP, bestIdx);
        }
        nFused++;
      }
    }
    return nFused;
  }

 public:
  static const int TH_LOW;
  static const int TH_HIGH;
  static const int HISTO_LENGTH;

 protected:
  // both (Frame&, const Frame&) overloads; acc != NULL: the per-query accepted current keypoint, or -1
  int search_last(Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono, std::vector<int32_t>* acc) {
    FlatFrame cur;
    flatten(CurrentFrame, cur, true);
    const int nl = LastFrame.N;
    std::vector<float> xw((size_t)(nl > 0 ? nl : 1) * 3, 0.f), lang(nl);
    std::vector<uint8_t> valid(nl, 0), ldesc((size_t)(nl > 0 ? nl : 1) * 32, 0);
    std::vector<int32_t> loct(nl), lobs(nl, 0);
    for (int i = 0; i < nl; ++i) {
      MapPoint* pMP = LastFrame.mvpMapPoints[i];
      loct[i] = LastFrame.mvKeys[i].octave;
      lang[i] = LastFrame.mvKeysUn[i].angle;
      if (pMP && !LastFrame.mvbOutlier[i]) {
        valid[i] = 1;
        cv::Mat p = pMP->GetWorldPos();
        for (int k = 0; k < 3; ++k) xw[(size_t)i * 3 + k] = p.at<float>(k);
        cv::Mat d = pMP->GetDescriptor();
        std::memcpy(&ldesc[(size_t)i * 32], d.ptr(0), 32);
        lobs[i] = pMP->Observations();
      }
    }
    OrbmLast L;
    L.n = nl; L.xw = xw.data(); L.valid = valid.data(); L.octave = loct.data(); L.angle = lang.data();
    L.mp_desc = ldesc.data(); L.mp_obs = lobs.data();
    copy_pose(LastFrame.mTcw, L.Tcw);
    std::vector<int32_t> c2l(cur.n > 0 ? cur.n : 1, -1);
    int nmatches = 0;
    if (acc) {
      acc->assign(nl > 0 ? nl : 1, -1);
      check(orbm_search_by_projection_last_pairs(h_, &cur.view, &L, th, bMono ? 1 : 0, mfNNratio, mbCheckOrientation ? 1 : 0,
                                                 c2l.data(), acc->data(), &nmatches));
    } else {
      check(orbm_search_by_projection_last(h_, &cur.view, &L, th, bMono ? 1 : 0, mfNNratio, mbCheckOrientation ? 1 : 0,
                                           c2l.data(), &nmatches));
    }
    for (int j = 0; j < cur.n; ++j) {      // the pointer state the reference leaves behind (:1680,:1716)
      if (c2l[j] >= 0) CurrentFrame.mvpMapPoints[j] = LastFrame.mvpMapPoints[c2l[j]];
      else if (c2l[j] == -1) CurrentFrame.mvpMapPoints[j] = static_cast<MapPoint*>(NULL);
    }
    return nmatches;
  }

  void open() {
    int dev = 0;
    if (const char* e = std::getenv("B200ORB_DEVICE")) dev = std::atoi(e);
    if (orbm_create(dev, &h_) != B200ORB_OK)   // the reference's constructor cannot fail; a missing GPU must be loud
      throw std::runtime_error(std::string("ORBmatcher(B200): ") + b200orb_last_error());
  }
  static void check(int rc) {
    if (rc != B200ORB_OK) throw std::runtime_error(std::string("ORBmatcher(B200): ") + b200orb_last_error());
  }
  struct FlatFrame {
    int n = 0;
    std::vector<float> x, y, ang, ur, sf;
    std::vector<int32_t> oct, obs;
    std::vector<uint8_t> desc;
    OrbmFrame view;
  };
  struct Queries {   // OrbmQueries under construction; slot i = MapPoint i of the caller's list
    std::vector<uint8_t> valid, desc;
    std::vector<float> u, v, r, ur, ang;
    std::vector<int32_t> mn, mx, obs;
    bool with_ur, with_ang;
    Queries(int n, bool with_ur_, bool with_ang_)
        : valid(n > 0 ? n : 1, 0), desc((size_t)(n > 0 ? n : 1) * 32, 0), u(n > 0 ? n : 1), v(n > 0 ? n : 1), r(n > 0 ? n : 1),
          ur(n > 0 ? n : 1), ang(n > 0 ? n : 1, 0.f), mn(n > 0 ? n : 1, 0), mx(n > 0 ? n : 1, 0), obs(n > 0 ? n : 1, 1),
          with_ur(with_ur_), with_ang(with_ang_), n_(n) {}
    void set(int i, float u_, float v_, float r_, int mn_, int mx_, MapPoint* pMP, float ang_, float ur_) {
      valid[i] = 1; u[i] = u_; v[i] = v_; r[i] = r_; mn[i] = mn_; mx[i] = mx_; ang[i] = ang_; ur[i] = ur_;
      cv::Mat d = pMP->GetDescriptor();
      std::memcpy(&desc[(size_t)i * 32], d.ptr(0), 32);
    }
    OrbmQueries view() const {
      OrbmQueries q;
      q.n = n_; q.valid = valid.data(); q.u = u.data(); q.v = v.data(); q.radius = r.data(); q.min_level = mn.data();
      q.max_level = mx.data(); q.uright = with_ur ? ur.data() : NULL; q.desc = desc.data(); q.angle = ang.data(); q.obs = NULL;
      return q;
    }
    int n_;
  };
  static void copy_pose(const cv::Mat& T, float out[16]) {
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) out[r * 4 + c] = T.at<float>(r, c);
  }
  template <class Keys>
  static void fill_keys(FlatFrame& o, const Keys& keysUn, const std::vector<float>& uRight, const cv::Mat& descriptors,
                        const std::vector<float>& sf) {
    const int n = (int)keysUn.size();
    o.n = n;
    const int m = n > 0 ? n : 1;
    o.x.resize(m); o.y.resize(m); o.ang.resize(m); o.ur.resize(m); o.oct.resize(m); o.obs.assign(m, -1);
    o.desc.resize((size_t)m * 32);
    for (int i = 0; i < n; ++i) {
      o.x[i] = keysUn[i].pt.x; o.y[i] = keysUn[i].pt.y; o.ang[i] = keysUn[i].angle; o.oct[i] = keysUn[i].octave;
      o.ur[i] = uRight[i];
      std::memcpy(&o.desc[(size_t)i * 32], descriptors.ptr(i), 32);
    }
    o.sf.assign(sf.begin(), sf.end());
    OrbmFrame& v = o.view;
    v.n = n; v.x = o.x.data(); v.y = o.y.data(); v.octave = o.oct.data(); v.angle = o.ang.data(); v.uright = o.ur.data();
    v.desc = o.desc.data(); v.mp_obs = o.obs.data();
    v.scale_factors = o.sf.data(); v.nlevels = (int)o.sf.size();
  }
  static void flatten(Frame& F, FlatFrame& o, bool with_mp_state) {
    fill_keys(o, F.mvKeysUn, F.mvuRight, F.mDescriptors, F.mvScaleFactors);
    if (with_mp_state)
      for (int i = 0; i < o.n; ++i)
        if (F.mvpMapPoints[i]) o.obs[i] = F.mvpMapPoints[i]->Observations();
    OrbmFrame& v = o.view;
    if (!F.mTcw.empty()) copy_pose(F.mTcw, v.Tcw);
    else { const float I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}; std::memcpy(v.Tcw, I, sizeof(I)); }
    v.fx = F.fx; v.fy = F.fy; v.cx = F.cx; v.cy = F.cy; v.bf = F.mbf; v.b = F.mb;
    v.min_x = Frame::mnMinX; v.max_x = Frame::mnMaxX; v.min_y = Frame::mnMinY; v.max_y = Frame::mnMaxY;
  }
  // a KeyFrame as the "searched" side: its grid is the Frame's grid it was built from (src/KeyFrame.cc:57-66)
  static void flatten_kf(KeyFrame* pKF, FlatFrame& o) {
    fill_keys(o, pKF->mvKeysUn, pKF->mvuRight, pKF->mDescriptors, pKF->mvScaleFactors);
    OrbmFrame& v = o.view;
    copy_pose(pKF->GetPose(), v.Tcw);
    v.fx = pKF->fx; v.fy = pKF->fy; v.cx = pKF->cx; v.cy = pKF->cy; v.bf = pKF->mbf; v.b = pKF->mb;
    v.min_x = pKF->mnMinX; v.max_x = pKF->mnMaxX; v.min_y = pKF->mnMinY; v.max_y = pKF->mnMaxY;
  }
  struct FlatBow {
    std::vector<uint8_t> desc, valid;
    std::vector<float> ang;
    std::vector<uint32_t> node_ids, idx;
    std::vector<int32_t> node_off;
    OrbmBow view;
  };
  template <class FeatVec>
  static void flatten_featvec(const FeatVec& fv, std::vector<uint32_t>& node_ids, std::vector<int32_t>& node_off,
                              std::vector<uint32_t>& idx) {
    node_off.assign(1, 0);
    for (typename FeatVec::const_iterator it = fv.begin(); it != fv.end(); ++it) {
      node_ids.push_back((uint32_t)it->first);
      for (size_t k = 0; k < it->second.size(); ++k) idx.push_back((uint32_t)it->second[k]);
      node_off.push_back((int32_t)idx.size());
    }
    if (idx.empty()) idx.push_back(0);
    if (node_ids.empty()) node_ids.push_back(0);
  }
  // descriptors + angles + the FeatureVector (ordered map: ascending node ids) flattened; mps == NULL: no validity mask
  template <class Keys, class FeatVec>
  static void flatten_bow(const cv::Mat& descriptors, const Keys& keys, const FeatVec& fv, const std::vector<MapPoint*>* mps,
                          FlatBow& o) {
    const int n = (int)keys.size();
    o.desc.resize((size_t)(n > 0 ? n : 1) * 32);
    o.ang.resize(n > 0 ? n : 1);
    for (int i = 0; i < n; ++i) {
      std::memcpy(&o.desc[(size_t)i * 32], descriptors.ptr(i), 32);
      o.ang[i] = keys[i].angle;
    }
    if (mps) {
      o.valid.assign(n > 0 ? n : 1, 0);
      for (int i = 0; i < n; ++i) {
        MapPoint* p = (*mps)[i];
        o.valid[i] = (p && !p->isBad()) ? 1 : 0;
      }
    }
    flatten_featvec(fv, o.node_ids, o.node_off, o.idx);
    OrbmBow& v = o.view;
    v.n = n; v.desc = o.desc.data(); v.angle = o.ang.data(); v.valid = mps ? o.valid.data() : NULL;
    v.n_nodes = (int)o.node_off.size() - 1; v.node_ids = o.node_ids.data(); v.node_off = o.node_off.data(); v.idx = o.idx.data();
  }
  struct FlatTri {
    std::vector<uint8_t> desc, has_mp;
    std::vector<float> x, y, ang, ur;
    std::vector<int32_t> oct, node_off;
    std::vector<uint32_t> node_ids, idx;
    OrbmTriKF view;
  };
  static void flatten_tri(KeyFrame* pKF, FlatTri& o) {
    const int n = pKF->N, m = n > 0 ? n : 1;
    o.desc.resize((size_t)m * 32); o.has_mp.assign(m, 0); o.x.resize(m); o.y.resize(m); o.ang.resize(m); o.ur.resize(m); o.oct.resize(m);
    const std::vector<MapPoint*> mps = pKF->GetMapPointMatches();
    for (int i = 0; i < n; ++i) {
      std::memcpy(&o.desc[(size_t)i * 32], pKF->mDescriptors.ptr(i), 32);
      const cv::KeyPoint& kp = pKF->mvKeysUn[i];
      o.x[i] = kp.pt.x; o.y[i] = kp.pt.y; o.ang[i] = kp.angle; o.oct[i] = kp.octave; o.ur[i] = pKF->mvuRight[i];
      o.has_mp[i] = mps[i] ? 1 : 0;
    }
    flatten_featvec(pKF->mFeatVec, o.node_ids, o.node_off, o.idx);
    OrbmTriKF& v = o.view;
    v.n = n; v.desc = o.desc.data(); v.x = o.x.data(); v.y = o.y.data(); v.angle = o.ang.data(); v.uright = o.ur.data();
    v.octave = o.oct.data(); v.has_mp = o.has_mp.data();
    v.n_nodes = (int)o.node_off.size() - 1; v.node_ids = o.node_ids.data(); v.node_off = o.node_off.data(); v.idx = o.idx.data();
  }

  float mfNNratio;
  bool mbCheckOrientation;
  orbm_t* h_ = nullptr;
};

// src/ORBmatcher.cc:39-41; weak so that the header can be included from every caller's translation unit
__attribute__((weak)) const int ORBmatcher::TH_HIGH = ORBM_TH_HIGH;
__attribute__((weak)) const int ORBmatcher::TH_LOW = ORBM_TH_LOW;
__attribute__((weak)) const int ORBmatcher::HISTO_LENGTH = ORBM_HISTO_LENGTH;

}  // namespace ORB_SLAM2
#endif  // ORBMATCHER_H
