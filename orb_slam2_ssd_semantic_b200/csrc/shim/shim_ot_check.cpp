// A C++ caller that knows shim/pointcloudmapping.h only: build a map, write it as an `.ot` file, read the file into a
// second map, keep inserting into both, and write both again.  argv[1], argv[2], argv[3]: the file of the first save and
// the two files after the resume (the test compares them and parses them).
#include <cstdio>
#include <vector>

#include "pointcloudmapping.h"

struct MockKeyFrame {   // what PointCloudMapping reads from a KeyFrame (P variant: images stored on the keyframe)
  cv::Mat pose = cv::Mat::eye(4, 4, CV_32F), mImDep, mImRGB;
  float fx = 535.4f, fy = 539.2f, cx = 320.1f, cy = 247.6f;
  cv::Mat GetPose() { return pose.clone(); }
};

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  cv::Mat depth(480, 640, CV_32F), rgb(480, 640 * 3, CV_8UC1);
  unsigned s = 777u;
  for (int r = 0; r < 480; ++r)
    for (int c = 0; c < 640; ++c) {
      depth.at<float>(r, c) = 1.25f + 0.002f * c + 0.001f * r;
      s = s * 1664525u + 1013904223u;
      for (int k = 0; k < 3; ++k) rgb.data[(r * 640 + c) * 3 + k] = (uint8_t)(s >> (8 * k + 8));
    }
  MockKeyFrame kf[4];
  for (int i = 0; i < 4; ++i) {
    kf[i].mImDep = depth;
    kf[i].mImRGB = rgb;
    kf[i].pose.at<float>(0, 3) = -0.4f * i;
  }
  try {
    PointCloudMapping a(0.05), b(0.05);
    std::vector<MockKeyFrame*> v = {&kf[0], &kf[1], &kf[2]};   // UpdateOctomap inserts all but the newest
    a.UpdateOctomap(v);
    a.SaveOctoMap(argv[1]);
    b.LoadOctoMap(std::string(argv[1]));
    const long long na = a.numLeaves(), nb = b.numLeaves();
    cv::Mat gray;
    a.insertKeyFrame(&kf[3], gray, depth, rgb);
    b.insertKeyFrame(&kf[3], gray, depth, rgb);
    a.SaveOctoMap(argv[2]);
    b.SaveOctoMap(argv[3]);
    std::printf("saved %lld cells, loaded %lld, resumed to %lld and %lld\n", na, nb, a.numLeaves(), b.numLeaves());
    if (!(na > 0 && na == nb && a.numLeaves() > na && a.numLeaves() == b.numLeaves())) return 1;
    bool refused = false;
    try {
      PointCloudMapping other(0.1);
      other.LoadOctoMap(std::string(argv[1]));
    } catch (const std::exception& ex) {
      std::printf("other resolution refused: %s\n", ex.what());
      refused = true;
    }
    return refused ? 0 : 3;
  } catch (const std::exception& ex) {
    std::printf("FAILED: %s\n", ex.what());
    return 4;
  }
}
