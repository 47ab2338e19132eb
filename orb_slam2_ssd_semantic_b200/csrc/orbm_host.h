// orbm_host.h -- matcher handle: a stream + a grow-only device arena for the host-buffer entry points.
#pragma once
#include "orbm_match.cuh"

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
