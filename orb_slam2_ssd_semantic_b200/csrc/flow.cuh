// flow.cuh -- the dense optical flow of flow.cu (pyrDown + OpenCV's Farneback, bit for bit) as the dynamic-mask entries
// (dynm.cu) and the masked batch tracker (orbs.cu) drive it: its geometry, its scratch and its host drivers.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int FB_LEVELS = 3;
constexpr int FB_CHUNK = 64;            // frames per pass through the scratch buffers

// Pyramid geometry of a half-resolution rows x cols pair: top = the coarsest level index, h[k] x w[k] = cvRound(side *
// 0.5^k) (half to even).
struct FbGeom {
  int H = 0, W = 0, top = 0;
  int h[FB_LEVELS + 1] = {}, w[FB_LEVELS + 1] = {};
};

// Scratch of one chunk of up to C pairs (C + 1 images) of H x W half-resolution images.
struct FbScratch {
  uint8_t* half;   // [C + 1][H][W] u8
  float* tmp;      // [C + 1][H][W] row pass of the blur
  float* blur;     // [C + 1][H][W]
  float* img;      // [C + 1][h1][w1] the blurred image at level k >= 1
  float* R;        // [C + 1][H][W][5] polynomial expansions
  float* M;        // [C][H][W][5] the matrices of FarnebackUpdateMatrices
  double* V;       // [C][H][W][5] the running column sums of each row
  float* fl[2];    // [C][h1][w1][2] flow of levels >= 1, ping-pong
};

// The geometry of H x W half-resolution images; EINVAL (with a message) for sides outside the range the kernels accept.
int fb_geometry(int H, int W, FbGeom* g);
// Carves the scratch of chunks of C pairs.
void fb_take(Carver& t, FbScratch& s, const FbGeom& g, int C);
// Farneback of the nimg - 1 consecutive pairs of the half-resolution images in s.half -> out [nimg - 1][H][W][2].
int fb_pairs(cudaStream_t st, const FbGeom& g, const FbScratch& s, int nimg, float* out, long long* launches);
// pyrDown(Size(SW / 2, SH / 2)) of nimg SH x SW u8 images into dst [nimg][H][W]: image 0 is `first`, image i > 0 is
// rest + (i - 1) SH SW.
void fb_pyrdown(cudaStream_t st, const FbGeom& g, const uint8_t* first, const uint8_t* rest, int nimg, int SH, int SW,
                uint8_t* dst, long long* launches);
// Flow::ComputeMask's pyrDown + Farneback for n full-resolution frames in HBM (SH x SW each): out[t] is the flow from
// frame t-1 to frame t, where frame -1 is `d_prev`; without it out[0] is the zero field.  Chunks of at most C frames.
int fb_batch(cudaStream_t st, const FbGeom& g, const FbScratch& s, int C, const uint8_t* d_gray, const uint8_t* d_prev,
             int n, int SH, int SW, float* out, long long* launches);

}  // namespace b200
