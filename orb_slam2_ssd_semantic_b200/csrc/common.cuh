// common.cuh -- shared helpers of libb200orb.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <stdio.h>
#include <string.h>

#include "../../include/b200orb.h"

namespace b200 {

void set_error(const char* fmt, ...);

#define B200_CUDA(expr)                                                                      \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      b200::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));  \
      return B200ORB_ECUDA;                                                                  \
    }                                                                                        \
  } while (0)

#define B200_CHECK(rc_expr)        \
  do {                             \
    int _rc = (rc_expr);           \
    if (_rc != B200ORB_OK) return _rc; \
  } while (0)

static inline int align_up(int v, int a) { return (v + a - 1) / a * a; }
static inline size_t align_up_sz(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Sequential sub-allocation out of one device block, 256-byte aligned.  Against a null base it only measures: `off` is
// then the size the same sequence of take() calls needs.  A take() past `cap` returns null and marks the carver overrun.
struct Carver {
  char* base;
  size_t cap, off = 0;
  bool overrun = false;
  explicit Carver(void* b = nullptr, size_t c = SIZE_MAX) : base((char*)b), cap(c) {}
  template <class T>
  T* take(size_t n) {
    const size_t at = off;
    off = align_up_sz(off + std::max<size_t>(n, 1) * sizeof(T), 256);
    if (off > cap) overrun = true;
    return (base && !overrun) ? (T*)(base + at) : nullptr;
  }
};

// One device allocation for a buffer list: `take_all` carves the list, once against a null base to measure it, then
// out of the new block.  *bytes = the block's size.
template <class F>
static int alloc_carved(void** block, F&& take_all, size_t* bytes = nullptr) {
  Carver probe;
  take_all(probe);
  B200_CUDA(cudaMalloc(block, probe.off));
  Carver c(*block, probe.off);
  take_all(c);
  if (bytes) *bytes = probe.off;
  return B200ORB_OK;
}

// RAII device guard: every ABI call runs on its handle's device and restores the caller's.
struct DeviceGuard {
  int prev = -1;
  bool ok = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; }
    ok = (cudaSetDevice(dev) == cudaSuccess);
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

int check_device(int device);   // B200ORB_OK or ENOGPU/EINVAL with message

// SM count of `device`: the fixed grids of the grid-stride sweeps are a small multiple of it (132 on an H100 SXM).
static inline int sm_count(int device) {
  int n = 0;
  return (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && n > 0) ? n : 1;
}

constexpr int MAX_LEVELS = 16;
constexpr int EDGE_THRESHOLD = 19;     // src/ORBextractor.cc:54
constexpr int PATCH_SIZE = 31;         // :52
constexpr int HALF_PATCH_SIZE = 15;    // :53
constexpr int FAST_BORDER = 16;        // EDGE_THRESHOLD-3, :780

// ---- device helpers -------------------------------------------------------------------------
__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// Exclusive scan of one int per thread across the block. `ws` = shared scratch of >= 33 ints.
// Returns the exclusive prefix; *total = block sum. Contains __syncthreads (all threads must call).
__device__ __forceinline__ int block_excl_scan(int v, int* ws, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  int inc = warp_incl_scan(v, lane);
  __syncthreads();   // protect ws reuse
  if (lane == 31) ws[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int w = (lane < nw) ? ws[lane] : 0;
    int winc = warp_incl_scan(w, lane);
    ws[lane] = winc - w;
    if (lane == 31) ws[32] = winc;
  }
  __syncthreads();
  *total = ws[32];
  return ws[wid] + inc - v;
}

}  // namespace b200
