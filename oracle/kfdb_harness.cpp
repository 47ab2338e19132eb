// oracle/kfdb_harness.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
//
// C entry point around the reference's own src/KeyFrameDatabase.cc (and src/KeyFrame.cc for the covisibility graph),
// compiled unmodified from the reference tree into oracle/_ref/ by oracle/kfdb.mk:
//   _ref/libkfdbsrc.so   the reference's KeyFrameDatabase.cc with the objects of target `ref` (exports refsrc_kfdb_run)
//   _ref/libkfdbshim.so  the reference's Frame.cc / KeyFrame.cc / MapPoint.cc / Map.cc compiled against the shims with
//                        shim/KeyFrameDatabase.h force-included, linked against libb200orb.so (exports shimsrc_kfdb_run)
// tests/test_kfdb_cpu.py pins oracle/kfdb_py.py to the first; tests/test_kfdb_gpu.py asserts the second == the first.
// Nothing here restates reference logic; `#define private public` only opens the classes so that a Frame and KeyFrames
// can be filled from arrays.
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <list>
#include <map>
#include <mutex>
#include <new>
#include <set>
#include <vector>

#include "../include/b200orb.h"

#define private public
#define protected public
#include "KeyFrameDatabase.h"   // first: in the shim build this is shim/KeyFrameDatabase.h (see oracle/kfdb.mk)
#include "Frame.h"
#include "KeyFrame.h"
#include "Map.h"
#include "ORBVocabulary.h"
#undef private
#undef protected

using namespace ORB_SLAM2;

#ifdef REFSRC_SHIM
#define X(name) shimsrc_##name
#else
#define X(name) refsrc_##name
#endif

namespace {

std::mutex g_mu;
Map g_map;

// A one-keypoint Frame as the RGB-D constructor leaves it minus the extraction (identity pose, 640x480 bounds, 8 levels):
// every KeyFrame and every relocalisation query Frame is a copy of it.  The database reads none of its geometry.
Frame* proto_frame() {
  static Frame* F = nullptr;
  if (F) return F;
  static const float sf[8] = {1, 1.2f, 1.44f, 1.728f, 2.0736f, 2.48832f, 2.985984f, 3.5831808f};
  F = new Frame();
  F->mpORBvocabulary = nullptr; F->mpORBextractorLeft = nullptr; F->mpORBextractorRight = nullptr;
  F->mnId = Frame::nNextId++;
  F->mTimeStamp = 0;
  F->mbf = 40; F->mb = 0.08f; F->mThDepth = 40.0f * F->mb;
  F->N = 1;
  cv::KeyPoint kp(1.f, 1.f, 31.f, 0.f, 0.f, 0);
  F->mvKeys.assign(1, kp); F->mvKeysUn.assign(1, kp);
  F->mvuRight.assign(1, 0.f); F->mvDepth.assign(1, -1.f);
  F->mDescriptors = cv::Mat::zeros(1, 32, CV_8U);
  F->mvpMapPoints.assign(1, static_cast<MapPoint*>(NULL));
  F->mvbOutlier.assign(1, false);
  F->mnScaleLevels = 8; F->mfScaleFactor = sf[1]; F->mfLogScaleFactor = log(F->mfScaleFactor);
  F->mvScaleFactors.assign(sf, sf + 8);
  F->mvInvScaleFactors.resize(8); F->mvLevelSigma2.resize(8); F->mvInvLevelSigma2.resize(8);
  for (int l = 0; l < 8; ++l) {
    F->mvInvScaleFactors[l] = 1.0f / sf[l];
    F->mvLevelSigma2[l] = sf[l] * sf[l];
    F->mvInvLevelSigma2[l] = 1.0f / F->mvLevelSigma2[l];
  }
  Frame::fx = Frame::fy = 500; Frame::cx = 320; Frame::cy = 240; Frame::invfx = Frame::invfy = 1.0f / 500;
  Frame::mnMinX = 0; Frame::mnMaxX = 640; Frame::mnMinY = 0; Frame::mnMaxY = 480;
  Frame::mfGridElementWidthInv = static_cast<float>(FRAME_GRID_COLS) / 640.f;
  Frame::mfGridElementHeightInv = static_cast<float>(FRAME_GRID_ROWS) / 480.f;
  Frame::mbInitialComputations = false;
  F->mK = cv::Mat::eye(3, 3, CV_32F);
  F->mK.at<float>(0, 0) = 500; F->mK.at<float>(1, 1) = 500; F->mK.at<float>(0, 2) = 320; F->mK.at<float>(1, 2) = 240;
  F->mDistCoef = cv::Mat::zeros(4, 1, CV_32F);
  F->AssignFeaturesToGrid();
  F->SetPose(cv::Mat::eye(4, 4, CV_32F));
  return F;
}

}  // namespace

extern "C" {

// ---------------------------------------------------------------------------------------------------------------------
// KeyFrameDatabase (src/KeyFrameDatabase.cc) on real KeyFrames: a script of add / erase / clear / query operations.
// Keyframe i has BowVector words / weights [word_off[i], word_off[i+1]), mnId kf_id[i] and the six database members
// init[i]; edges (a, b, weight) are AddConnection'ed both ways.  The KeyFrames lie in ONE allocation in index order, so
// that UpdateBestCovisibles' (weight, KeyFrame*) sort orders equal weights by index (higher index first).
// op_code: 0 add(op_arg), 1 erase(op_arg), 2 clear, 3 DetectRelocalizationCandidates of a Frame with mnId op_id and
// BowVector q[q_off[op_arg], q_off[op_arg+1]), 4 DetectLoopCandidates(keyframe op_arg, op_min).
// Outputs: the candidates of query op o as keyframe indices in cand[cand_off[o], cand_off[o+1]); the six members of every
// keyframe after every query (members_every_query) or once at the end; GetBestCovisibilityKeyFrames(10) per keyframe in
// neigh[11 * i] (count, then indices); op_sec[o] the steady_clock seconds of each Detect call.  -2: cand_cap too small.
int X(kfdb_run)(int n_words, int n_kf, const uint32_t* words, const double* weights, const int64_t* word_off,
                const uint64_t* kf_id, const OrbvDbMembers* init, int n_edges, const int32_t* edges, int n_ops,
                const int32_t* op_code, const int32_t* op_arg, const uint64_t* op_id, const float* op_min,
                const uint32_t* qwords, const double* qweights, const int64_t* q_off, int32_t* cand, int64_t cand_cap,
                int64_t* cand_off, int members_every_query, OrbvDbMembers* members, int32_t* neigh, double* op_sec) {
  std::lock_guard<std::mutex> lk(g_mu);
  Frame* g_proto = proto_frame();
  ORBVocabulary voc;   // KeyFrameDatabase reads size() only: a root with n_words leaves
  {
    std::vector<DBoW2::NodeId> par(n_words + 1, 0);
    std::vector<cv::Mat> nd(n_words + 1);
    std::vector<DBoW2::WordValue> w(n_words + 1, 0.0);
    voc.build(n_words, 1, par, nd, w);
  }
  KeyFrame* kfs = static_cast<KeyFrame*>(::operator new(sizeof(KeyFrame) * (size_t)std::max(n_kf, 1)));
  for (int i = 0; i < n_kf; ++i) {
    KeyFrame* K = new (kfs + i) KeyFrame(*g_proto, &g_map, nullptr);
    K->mGrid.clear();   // 3072 empty cells per keyframe; nothing here reads them
    K->mGrid.shrink_to_fit();
    K->mnId = kf_id[i];
    for (int64_t j = word_off[i]; j < word_off[i + 1]; ++j) K->mBowVec[words[j]] = weights[j];
    K->mnLoopQuery = init[i].loop_query; K->mnLoopWords = init[i].loop_words; K->mLoopScore = init[i].loop_score;
    K->mnRelocQuery = init[i].reloc_query; K->mnRelocWords = init[i].reloc_words; K->mRelocScore = init[i].reloc_score;
  }
  for (int e = 0; e < n_edges; ++e) {
    kfs[edges[3 * e]].AddConnection(kfs + edges[3 * e + 1], edges[3 * e + 2]);
    kfs[edges[3 * e + 1]].AddConnection(kfs + edges[3 * e], edges[3 * e + 2]);
  }
  for (int i = 0; i < n_kf; ++i) {
    const std::vector<KeyFrame*> v = kfs[i].GetBestCovisibilityKeyFrames(10);
    neigh[11 * i] = (int32_t)v.size();
    for (size_t j = 0; j < v.size(); ++j) neigh[11 * i + 1 + j] = (int32_t)(v[j] - kfs);
  }
  auto snapshot = [&](OrbvDbMembers* m) {
    for (int i = 0; i < n_kf; ++i) {
      const KeyFrame& K = kfs[i];
      m[i].loop_query = K.mnLoopQuery; m[i].loop_words = K.mnLoopWords; m[i].loop_score = K.mLoopScore;
      m[i].reloc_query = K.mnRelocQuery; m[i].reloc_words = K.mnRelocWords; m[i].reloc_score = K.mRelocScore;
    }
  };
  int rc = 0;
  {
    KeyFrameDatabase db(voc);
    int64_t nc = 0;
    int nq = 0;
    cand_off[0] = 0;
    for (int o = 0; o < n_ops; ++o) {
      std::vector<KeyFrame*> v;
      op_sec[o] = 0;
      if (op_code[o] == 0) db.add(kfs + op_arg[o]);
      else if (op_code[o] == 1) db.erase(kfs + op_arg[o]);
      else if (op_code[o] == 2) db.clear();
      else {
        Frame F(*g_proto);
        if (op_code[o] == 3) {
          F.mnId = op_id[o];
          for (int64_t j = q_off[op_arg[o]]; j < q_off[op_arg[o] + 1]; ++j) F.mBowVec[qwords[j]] = qweights[j];
        }
        const auto t0 = std::chrono::steady_clock::now();
        v = op_code[o] == 3 ? db.DetectRelocalizationCandidates(&F) : db.DetectLoopCandidates(kfs + op_arg[o], op_min[o]);
        op_sec[o] = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (members_every_query) snapshot(members + (size_t)n_kf * nq++);
      }
      if (nc + (int64_t)v.size() > cand_cap) { rc = -2; break; }
      for (KeyFrame* p : v) cand[nc++] = (int32_t)(p - kfs);
      cand_off[o + 1] = nc;
    }
  }
  if (!members_every_query) snapshot(members);
  for (int i = 0; i < n_kf; ++i) kfs[i].~KeyFrame();
  ::operator delete(kfs);
  return rc;
}

}  // extern "C"
