// shim_sem_check.cpp -- drives PointCloudMappingT's semantic overload (shim/pointcloudmapping.h) over a keyframe sequence
// read from a file and prints the cluster database and the size of globalMap after the refilter, every float as its
// bit pattern so that the caller can compare bit for bit.
//
// Input (little-endian): int32 rows, cols, n_keyframes; float32 fx, fy, cx, cy, resolution; then per keyframe:
// float32 Tcw[16], float32 depth[rows*cols], uint8 bgr[rows*cols*3], int32 n_objects, and per object float32 x, y, width,
// height, int32 class_id, float32 prob, char object_name[16] (NUL-padded).
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "pointcloudmapping.h"

struct Object {   // src/ncnn_dect.h:12-18
  cv::Rect_<float> rect;
  std::string object_name;
  int class_id;
  float prob;
};

static unsigned bits(float v) {
  unsigned u;
  memcpy(&u, &v, 4);
  return u;
}

template <class T>
static bool get(FILE* f, T* p, size_t n = 1) { return fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
  if (argc != 2) { fprintf(stderr, "usage: shim_sem_check <sequence file>\n"); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  int32_t rows, cols, nkf;
  float fx, fy, cx, cy, res;
  if (!get(f, &rows) || !get(f, &cols) || !get(f, &nkf) || !get(f, &fx) || !get(f, &fy) || !get(f, &cx) || !get(f, &cy) ||
      !get(f, &res)) { fprintf(stderr, "short header\n"); return 2; }
  try {
    PointCloudMappingT map(res);
    std::vector<float> depth((size_t)rows * cols);
    std::vector<unsigned char> bgr((size_t)rows * cols * 3);
    for (int i = 0; i < nkf; ++i) {
      float Tcw[16];
      int32_t n;
      if (!get(f, Tcw, 16) || !get(f, depth.data(), depth.size()) || !get(f, bgr.data(), bgr.size()) || !get(f, &n)) {
        fprintf(stderr, "short keyframe %d\n", i);
        return 2;
      }
      std::vector<Object> objects(n);
      for (Object& o : objects) {
        float r[4];
        char name[16];
        if (!get(f, r, 4) || !get(f, &o.class_id) || !get(f, &o.prob) || !get(f, name, 16)) { fprintf(stderr, "short object\n"); return 2; }
        o.rect = cv::Rect_<float>(r[0], r[1], r[2], r[3]);
        o.object_name = std::string(name, strnlen(name, 16));
      }
      cv::Mat gray, dm(rows, cols, CV_32F, depth.data()), cm(rows, cols, CV_8UC3, bgr.data());
      map.insertKeyFrame(Tcw, fx, fy, cx, cy, gray, dm, cm, objects);
    }
    map.update();
    for (const Cluster& c : map.clusters())
      printf("cluster %s %d %08x %08x %08x %08x %08x %08x %08x %08x %08x %08x\n", c.object_name.c_str(), c.class_id, bits(c.prob),
             bits(c.centroid[0]), bits(c.centroid[1]), bits(c.centroid[2]), bits(c.minPt[0]), bits(c.minPt[1]), bits(c.minPt[2]),
             bits(c.maxPt[0]), bits(c.maxPt[1]), bits(c.maxPt[2]));
    printf("globalMap %lld\n", map.globalMapSize());
  } catch (const std::exception& e) {
    printf("error: %s\n", e.what());
    return 1;
  }
  fclose(f);
  return 0;
}
