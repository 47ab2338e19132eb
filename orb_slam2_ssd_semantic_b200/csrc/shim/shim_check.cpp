// Compiles the extractor and mapping shim headers (against whatever <opencv2/opencv.hpp> the include path offers: the
// tests use the stand-in of oracle/standin/) and exercises them when a GPU is present.  The matcher shim needs the
// reference's Frame / KeyFrame / MapPoint classes and is tested through oracle/_ref/libshimsrc.so instead.
#include <cstdio>
#include <cstdlib>
#include <map>
#include <string>

#include "ORBextractor.h"
#include "pointcloudmapping.h"

struct MockKeyFrame {   // what PointCloudMapping reads from a KeyFrame (P variant: images stored on the keyframe)
  cv::Mat pose = cv::Mat::eye(4, 4, CV_32F), mImDep, mImRGB;
  float fx = 535.4f, fy = 539.2f, cx = 320.1f, cy = 247.6f;
  cv::Mat GetPose() { return pose.clone(); }
};

// `shim_check extract nfeatures nlevels rows cols image.u8 out.bin`: one frame through a FRESH ORBextractor(nfeatures, 1.2,
// nlevels, 20, 7); writes the keypoint count, the keypoints as OrbxKeyPoint records and the descriptor rows.
static int extract_to_file(char** a) {
  const int nf = std::atoi(a[0]), nl = std::atoi(a[1]), rows = std::atoi(a[2]), cols = std::atoi(a[3]);
  cv::Mat img(rows, cols, CV_8UC1);
  FILE* f = std::fopen(a[4], "rb");
  if (!f || std::fread(img.data, 1, (size_t)rows * cols, f) != (size_t)rows * cols) return 5;
  std::fclose(f);
  ORB_SLAM2::ORBextractor ex(nf, 1.2f, nl, 20, 7);
  std::vector<cv::KeyPoint> kps;
  cv::Mat desc, mask;
  ex(img, mask, kps, desc);
  FILE* o = std::fopen(a[5], "wb");
  if (!o) return 5;
  const int n = (int)kps.size();
  std::fwrite(&n, sizeof(int), 1, o);
  for (const cv::KeyPoint& k : kps) {
    OrbxKeyPoint r{k.pt.x, k.pt.y, k.size, k.angle, k.response, k.octave, k.class_id};
    std::fwrite(&r, sizeof(r), 1, o);
  }
  for (int i = 0; i < n; ++i) std::fwrite(desc.ptr(i), 1, 32, o);
  std::fclose(o);
  std::printf("keypoints %d\n", n);
  return 0;
}

int main(int argc, char** argv) {
  if (argc == 8 && std::string(argv[1]) == "extract") return extract_to_file(argv + 2);
  if (b200orb_device_count() == 0) {
    try {
      ORB_SLAM2::ORBextractor e(1000, 1.2f, 8, 20, 7);
      std::printf("UNEXPECTED: constructed without a GPU\n");
      return 2;
    } catch (const std::exception& ex) {
      std::printf("no GPU -> loud failure: %s\n", ex.what());
      return 0;
    }
  }
  ORB_SLAM2::ORBextractor ex(1000, 1.2f, 8, 20, 7);
  cv::Mat img(480, 640, CV_8UC1);
  unsigned s = 12345u;
  for (int i = 0; i < 480 * 640; ++i) { s = s * 1664525u + 1013904223u; img.data[i] = (uint8_t)((s >> 24) & 0xff); }
  std::vector<cv::KeyPoint> kps;
  cv::Mat desc, mask;
  ex(img, mask, kps, desc);
  std::printf("keypoints %zu desc %dx%d levels %d sf1 %.4f\n", kps.size(), desc.rows, desc.cols, ex.GetLevels(),
              ex.GetScaleFactors()[1]);
  ex.SyncImagePyramid();
  std::printf("pyramid L7 %dx%d\n", ex.mvImagePyramid[7].cols, ex.mvImagePyramid[7].rows);
  PointCloudMapping pcm(0.05);
  cv::Mat depth(480, 640, CV_32F), rgb(480, 640 * 3, CV_8UC1);
  for (int r = 0; r < 480; ++r) for (int c = 0; c < 640; ++c) depth.at<float>(r, c) = 1.5f + 0.001f * c;
  float Tcw[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  pcm.insertKeyFrame(Tcw, 535.4f, 539.2f, 320.1f, 247.6f, img, depth, rgb);
  pcm.shutdown();
  std::printf("leaves %lld\n", (long long)pcm.numLeaves());
  {   // UpdateOctomap: the newest keyframe of the list is never inserted (perfect/src/MapDrawer.cc:615)
    PointCloudMapping lag(0.05);
    MockKeyFrame a, b, c;
    for (MockKeyFrame* k : {&a, &b, &c}) { k->mImDep = depth; k->mImRGB = rgb; }
    b.pose.at<float>(0, 3) = -2.5f; c.pose.at<float>(0, 3) = -5.0f;
    std::vector<MockKeyFrame*> v = {&a};
    lag.UpdateOctomap(v);
    lag.shutdown();
    const long long n0 = lag.numLeaves();
    v.push_back(&b); lag.UpdateOctomap(v); lag.shutdown();
    const long long n1 = lag.numLeaves();
    v.push_back(&c); lag.UpdateOctomap(v); lag.shutdown();
    const long long n2 = lag.numLeaves();
    std::printf("UpdateOctomap lag: %lld %lld %lld\n", n0, n1, n2);
    if (!(n0 == 0 && n1 > 0 && n2 > n1)) return 4;
  }
  PointCloudMappingT pcmT(0.04);                       // T variant: accumulated cloud + whole-map VoxelGrid refilter
  pcmT.insertKeyFrame(Tcw, 535.4f, 539.2f, 320.1f, 247.6f, img, depth, rgb);
  const long long raw = pcmT.globalMapSize();
  pcmT.update();
  pcmT.shutdown();
  std::printf("global map %lld -> %lld points\n", raw, pcmT.globalMapSize());
  return (kps.size() >= 1000 && desc.rows == (int)kps.size() && pcm.numLeaves() > 0 && raw == 480 * 640 &&
          pcmT.globalMapSize() > 0 && pcmT.globalMapSize() < raw) ? 0 : 1;
}
