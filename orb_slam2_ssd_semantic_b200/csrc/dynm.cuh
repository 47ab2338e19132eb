// dynm.cuh -- the dynm_* handle (include/b200orb.h), shared by the modules that implement its entries: dynm.cu (mask,
// keypoint filter, flow) and warp.cu (the homography branch's warpPerspective).
#pragma once
#include "common.cuh"

struct dynm {
  int device = 0;
  b200::Stream stream;
  long long launches = 0;
  b200::DeviceBlock buf;   // each entry carves its buffer list out of it
};
