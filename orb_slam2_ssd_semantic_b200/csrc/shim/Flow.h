// shim/Flow.h -- drop-in for the reference's perfect/include/Flow.h (same guard, same class): FlowSLAM::Flow keeps its
// interface (ComputeMask x2), its two members and its host-side OpenCV calls (pyrDown of the gray image,
// calcOpticalFlowFarneback, warpPerspective -- perfect/src/Flow.cc:26,29,78); everything after
// the optical flow -- pyrUp of the flow field, the threshold loop, erode, erode, dilate with the 21x21 ellipse
// (perfect/src/Flow.cc:30-47) -- runs on the GPU through dynm_mask_from_flow (include/b200orb.h).  The library has
// device twins of the host calls too (dynm_farneback, dynm_warp_perspective), but the shim keeps OpenCV's: the host
// build's Farneback (AVX2 / FMA dispatch) differs in the last bits from the baseline dispatch the device twin follows,
// and warping alone on the device would only add an upload and a download between two host calls.  There is no CPU
// fallback: the constructor throws when the library has no device.
#ifndef FLOW_H
#define FLOW_H

#include <opencv2/opencv.hpp>

#include <stdexcept>
#include <string>

#include "b200orb.h"

namespace FlowSLAM {

class Flow {
 private:
  cv::Mat mImGrayLast;
  cv::Mat mImGrayCurrent;
  dynm_t* h_ = nullptr;

 public:
  explicit Flow(int device = 0) {
    if (dynm_create(device, &h_) != B200ORB_OK) throw std::runtime_error(std::string("FlowSLAM::Flow: ") + b200orb_last_error());
  }
  ~Flow() { dynm_destroy(h_); }
  Flow(const Flow&) = delete;
  Flow& operator=(const Flow&) = delete;

  // perfect/src/Flow.cc:17-52
  void ComputeMask(const cv::Mat& GrayImg, cv::Mat& mask, float BInaryThreshold) {
    if (GrayImg.empty()) return;
    mask = cv::Mat::ones(GrayImg.rows, GrayImg.cols, CV_8U);
    cv::pyrDown(GrayImg, mImGrayCurrent, cv::Size(GrayImg.cols / 2, GrayImg.rows / 2));
    if (mImGrayLast.data) {
      cv::Mat flow;
      cv::calcOpticalFlowFarneback(mImGrayLast, mImGrayCurrent, flow, 0.5, 3, 15, 3, 5, 1.2, 0);   // host: OpenCV's own code
      if (!flow.isContinuous()) flow = flow.clone();
      if (!mask.isContinuous()) mask = mask.clone();
      if (dynm_mask_from_flow(h_, flow.ptr<float>(0), flow.rows, flow.cols, BInaryThreshold, mask.ptr<uchar>(0), mask.rows,
                              mask.cols) != B200ORB_OK)
        throw std::runtime_error(std::string("FlowSLAM::Flow::ComputeMask: ") + b200orb_last_error());
    }
    std::swap(mImGrayLast, mImGrayCurrent);
  }

  // perfect/src/Flow.cc:73-80
  void ComputeMask(const cv::Mat& GrayImg, const cv::Mat& Homo, cv::Mat& mask, float BInaryThreshold) {
    cv::Mat dest;
    cv::warpPerspective(GrayImg, dest, Homo, GrayImg.size());
    ComputeMask(dest, mask, BInaryThreshold);
  }
};

}  // namespace FlowSLAM

#endif  // FLOW_H
