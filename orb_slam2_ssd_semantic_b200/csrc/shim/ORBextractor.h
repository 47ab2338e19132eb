// shim/ORBextractor.h -- drop-in for the reference's include/ORBextractor.h: same namespace, class name, constructor,
// operator() signature, getters and the public mvImagePyramid member (include/ORBextractor.h:41-118), implemented
// on top of the C-ABI of libb200orb.so.  Frame.cc / Tracking.cc compile against it unchanged:
//   Tracking.cc:210-218   new ORBextractor(nFeatures, fScaleFactor, nLevels, fIniThFAST, fMinThFAST)
//   Frame.cc:340,342      (*mpORBextractorLeft)(im, cv::Mat(), mvKeys, mDescriptors)
//   Frame.cc:111-117      GetLevels() / GetScaleFactors() / ...
// Build with the OpenCV headers the reference already uses.  (This repo has no OpenCV C++; its tests compile the shims
// against the stand-in headers of oracle/standin/, together with the reference's own Frame.cc / KeyFrame.cc / MapPoint.cc.)
// mvImagePyramid is read back by the stereo matcher only (src/Frame.cc:649,761-778); it is filled lazily by
// SyncImagePyramid(), or after every operator() when ORBextractor::EagerPyramid() = true (or B200ORB_EAGER_PYRAMID=1) is
// set once at start-up -- stereo callers do that and stay otherwise unchanged.
#ifndef ORBEXTRACTOR_H
#define ORBEXTRACTOR_H

#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include <cstdlib>
#include <cstring>

#include <opencv2/opencv.hpp>

#include "b200orb.h"

namespace ORB_SLAM2 {

class ORBextractor {
 public:
  enum { HARRIS_SCORE = 0, FAST_SCORE = 1 };

  ORBextractor(int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST)
      : nfeatures(nfeatures), scaleFactor(scaleFactor), nlevels(nlevels), iniThFAST(iniThFAST), minThFAST(minThFAST) {
    OrbxParams p{nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST};
    int dev = 0;
    if (const char* e = std::getenv("B200ORB_DEVICE")) dev = std::atoi(e);
    if (orbx_create(&p, dev, &h_) != B200ORB_OK)   // the reference's ctor cannot fail; a missing GPU must be loud
      throw std::runtime_error(std::string("ORBextractor(B200): ") + b200orb_last_error());
    mvScaleFactor.resize(nlevels); mvInvScaleFactor.resize(nlevels);
    mvLevelSigma2.resize(nlevels); mvInvLevelSigma2.resize(nlevels);
    orbx_scale_tables(h_, mvScaleFactor.data(), mvInvScaleFactor.data(), mvLevelSigma2.data(), mvInvLevelSigma2.data(),
                      nullptr);
    mvImagePyramid.resize(nlevels);
  }
  ~ORBextractor() { orbx_destroy(h_); }
  ORBextractor(const ORBextractor&) = delete;
  ORBextractor& operator=(const ORBextractor&) = delete;
  // takes over the handle: perfect/src/Map.cc:239 copy-initialises an extractor from a temporary, which before C++17
  // needs a copy or move constructor
  ORBextractor(ORBextractor&& o)
      : mvImagePyramid(std::move(o.mvImagePyramid)), nfeatures(o.nfeatures), scaleFactor(o.scaleFactor), nlevels(o.nlevels),
        iniThFAST(o.iniThFAST), minThFAST(o.minThFAST), mvScaleFactor(std::move(o.mvScaleFactor)),
        mvInvScaleFactor(std::move(o.mvInvScaleFactor)), mvLevelSigma2(std::move(o.mvLevelSigma2)),
        mvInvLevelSigma2(std::move(o.mvInvLevelSigma2)), h_(o.h_), kps_(std::move(o.kps_)), desc_(std::move(o.desc_)),
        pyramid_valid_(o.pyramid_valid_) {
    o.h_ = nullptr;
  }

  // src/ORBextractor.cc:1052-1114.  `mask` is ignored exactly like the reference ignores it.
  void operator()(cv::InputArray _image, cv::InputArray /*mask*/, std::vector<cv::KeyPoint>& _keypoints,
                  cv::OutputArray _descriptors) {
    if (_image.empty()) return;                       // :1055
    cv::Mat image = _image.getMat();
    if (image.type() != CV_8UC1) throw std::invalid_argument("ORBextractor: image must be CV_8UC1");   // assert :1059
    int cap = 0, n = 0;
    if (orbx_max_keypoints_for(h_, image.rows, image.cols, &cap) != B200ORB_OK)
      throw std::runtime_error(std::string("ORBextractor(B200): ") + b200orb_last_error());
    kps_.resize(cap);
    desc_.resize((size_t)cap * 32);
    if (orbx_extract(h_, image.data, image.rows, image.cols, image.step, kps_.data(), desc_.data(), cap, &n) != B200ORB_OK)
      throw std::runtime_error(std::string("ORBextractor(B200): ") + b200orb_last_error());
    if (n == 0) {
      _descriptors.release();                         // :1073-1074
    } else {
      _descriptors.create(n, 32, CV_8U);              // :1077
      cv::Mat d = _descriptors.getMat();
      for (int i = 0; i < n; ++i) std::memcpy(d.ptr(i), &desc_[(size_t)i * 32], 32);
    }
    _keypoints.clear();
    _keypoints.reserve(n);
    for (int i = 0; i < n; ++i) {
      const OrbxKeyPoint& k = kps_[i];
      _keypoints.push_back(cv::KeyPoint(k.x, k.y, k.size, k.angle, k.response, k.octave, k.class_id));
    }
    pyramid_valid_ = false;
    if (EagerPyramid()) SyncImagePyramid();
  }

  // process-wide switch: fill the public mvImagePyramid member after every extraction (stereo callers)
  static bool& EagerPyramid() {
    static bool on = [] { const char* e = std::getenv("B200ORB_EAGER_PYRAMID"); return e && e[0] == '1'; }();
    return on;
  }

  int inline GetLevels() { return nlevels; }
  float inline GetScaleFactor() { return scaleFactor; }
  std::vector<float> inline GetScaleFactors() { return mvScaleFactor; }
  std::vector<float> inline GetInverseScaleFactors() { return mvInvScaleFactor; }
  std::vector<float> inline GetScaleSigmaSquares() { return mvLevelSigma2; }
  std::vector<float> inline GetInverseScaleSigmaSquares() { return mvInvLevelSigma2; }

  // include/ORBextractor.h:80 (see EagerPyramid above)
  std::vector<cv::Mat> mvImagePyramid;
  void SyncImagePyramid() {
    if (pyramid_valid_) return;
    for (int l = 0; l < nlevels; ++l) {
      int r = 0, c = 0;
      if (orbx_level_dims(h_, l, &r, &c) != B200ORB_OK) return;
      cv::Mat whole(r + 38, c + 38, CV_8UC1);
      orbx_get_level(h_, 0, l, 1, whole.data, whole.step);
      mvImagePyramid[l] = whole(cv::Rect(19, 19, c, r));   // ROI inside the bordered parent, like :1128
    }
    pyramid_valid_ = true;
  }

  orbx_t* handle() { return h_; }

 protected:
  int nfeatures;
  double scaleFactor;
  int nlevels, iniThFAST, minThFAST;
  std::vector<float> mvScaleFactor, mvInvScaleFactor, mvLevelSigma2, mvInvLevelSigma2;
  orbx_t* h_ = nullptr;
  std::vector<OrbxKeyPoint> kps_;
  std::vector<uint8_t> desc_;
  bool pyramid_valid_ = false;
};

}  // namespace ORB_SLAM2
#endif
