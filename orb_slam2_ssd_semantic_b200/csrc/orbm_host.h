// orbm_host.h -- matcher handle (a stream + a grow-only device arena for the host-buffer entry points) and the views of
// the LAST search that the stream pipeline (orbs.cu) shares with it.  The kernels are orbm_kernels.cuh's.
#pragma once
#include "common.cuh"

namespace b200 {

struct MatchCam {            // per-call constants (Frame statics + ORBmatcher ctor args)
  float fx, fy, cx, cy, bf, b;
  float min_x, max_x, min_y, max_y;
  float sf[MAX_LEVELS];
  float th, nnratio;
  int mono, check_ori, nlevels;
  int last_obs_default;      // Observations() of query MapPoints when no array is given
};

struct CurView {             // SoA view of the "current" frames; instance p reads at p*stride
  const float *x, *y, *ang, *uright;
  const int* oct;
  const uint8_t* desc;
  const int* obs;            // nullable: pre-existing mvpMapPoints state (-1 NULL, else Observations())
  const int* n;
  const float* Tcw;          // p*16
  const int* goff;           // p*(GRID_CELLS+1)
  const int* gidx;           // p*stride
  size_t stride;
};

struct LastView {            // LastFrame side; instance p reads at p*stride
  const float* xw;
  const uint8_t* valid;
  const int* oct;
  const float* ang;
  const uint8_t* desc;
  const int* obs;            // nullable
  const int* n;
  const float* Tcw;
  size_t stride;
};

// cv::Mat small-matrix gemm row: float accumulation, "+C" added in double (see oracle/match_ref.cpp header)
__device__ __forceinline__ float gemm3(const float* a, float b0, float b1, float b2, float c) {
  const float t = __fadd_rn(__fadd_rn(__fmul_rn(a[0], b0), __fmul_rn(a[1], b1)), __fmul_rn(a[2], b2));
  return __double2float_rn(__dadd_rn((double)t, (double)c));
}

}  // namespace b200

struct orbm {
  int device = 0;
  b200::Stream stream;
  long long launches = 0;
  b200::DeviceBlock arena;   // each entry carves its complete buffer list out of it
};

// Shared with the stream pipeline (orbs.cu): the LAST search of `npairs` (cur, last) pairs.  Frame pairs that fit in
// shared memory run the fused kernel; larger ones run separate query / grid / candidate / resolve kernels on device
// scratch of match_last_scratch_bytes(npairs, cv.stride, lv.stride) bytes (0, and d_scratch may be null, when fused).
size_t match_last_scratch_bytes(int npairs, size_t cstride, size_t lstride);
int launch_match_last(const b200::CurView& cv, const b200::LastView& lv, const b200::MatchCam& cam, int npairs,
                      void* d_scratch, int* d_accepted, int* d_cur2last, int* d_nmatch, cudaStream_t stream,
                      long long* launches);
