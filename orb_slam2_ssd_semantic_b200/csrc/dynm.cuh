// dynm.cuh -- the dynm_* handle (include/b200orb.h), shared by the modules that implement its entries: dynm.cu (mask,
// keypoint filter, flow), warp.cu (the homography branch's warpPerspective) and homography.cu (findHomography); and the
// device launchers of those two that the batched TrackHomo chain (orbs.cu) shares with the entries.
#pragma once
#include <vector>

#include "common.cuh"

namespace b200 {

constexpr int HF_MAX_PAIRS = 8192;   // findHomography's pair capacity

// findHomography's device scratch for up to `cap` pairs
struct HfScratch {
  float2 *isrc, *idst;
  int *sub, *nsub, *good;
  double *hyp, *J, *r, *rd;
};
void hf_take(Carver& t, HfScratch& s, int cap);
// The table of RANSACUpdateNumIters' log and pow for every n in [n0, n1] pairs, from the host's libm: row n (n + 2 doubles:
// g = 0 .. n good pairs, then log(1 - confidence)) starts at hf_tab_row(n, n0).
__host__ __device__ inline size_t hf_tab_row(int n, int n0) { return (size_t)(n - n0) * (size_t)(n0 + n + 3) / 2; }
void hf_tab(int n0, int n1, std::vector<double>& tab);
// cv::findHomography(src, dst, RANSAC, 3) of the *d_n pairs (n0 <= *d_n, the rows of `tab`) -> out[0..8] H, out[9] found,
// mask[*d_n].  *d_n == 0: nothing is written.  ransac = false only for exactly 4 pairs (runKernel of all four).
int launch_hf_fit(cudaStream_t st, const float2* src, const float2* dst, const int* d_n, bool ransac, const double* tab,
                  int tab_n0, const HfScratch& s, double* out, uint8_t* mask, long long* launches);
// warpPerspective of nframes u8 images d_src[n] by d_H[n][9] into d_dst[n]; take (NULL: every frame): frame n with
// take[n] == 0 copies its source instead.
int launch_warp(cudaStream_t st, const uint8_t* d_src, int nframes, int rows, int cols, const double* d_H, const int* take,
                uint8_t* d_dst, long long* launches);

}  // namespace b200

struct dynm {
  int device = 0;
  b200::Stream stream;
  long long launches = 0;
  b200::DeviceBlock buf;   // each entry carves its buffer list out of it
};
