// common.cuh -- shared helpers of libb200orb.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <stdio.h>
#include <string.h>
#include <utility>

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

// One allocation holding a buffer list, device (cudaMalloc) or page-locked host (cudaHostAlloc) memory.  `take_all`
// carves the list: once against a null base to measure it, which also nulls every buffer pointer, then out of the
// block.  A block is replaced only after `stream`, the last stream that used it, is synchronised, and `bytes` is set
// only once its allocation exists: after a failed allocation the block is empty and the next call allocates again.
// The destructor frees without a stream: cudaFree and cudaFreeHost synchronise with the device.
template <bool PINNED>
struct Block {
  void* p = nullptr;
  size_t bytes = 0;
  Block() = default;
  Block(Block&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  Block& operator=(Block&& o) noexcept {   // swaps: `o` frees the old block
    std::swap(p, o.p);
    std::swap(bytes, o.bytes);
    return *this;
  }
  ~Block() { release(); }
  // exactly the size of the list
  template <class F>
  int carve(cudaStream_t stream, F&& take_all) {
    Carver probe;
    take_all(probe);
    return alloc(stream, probe.off, take_all);
  }
  // grow-only: re-carved in place when the list fits, else grown to 1.5x the list, rounded up to 1 MiB
  template <class F>
  int reserve(cudaStream_t stream, F&& take_all) {
    Carver probe;
    take_all(probe);
    if (probe.off > bytes) return alloc(stream, align_up_sz(probe.off + probe.off / 2, 1 << 20), take_all);
    return cut(take_all);
  }

 private:
  void release() {
    if (p) PINNED ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr;
    bytes = 0;
  }
  template <class F>
  int alloc(cudaStream_t stream, size_t n, F& take_all) {
    if (p) {
      B200_CUDA(cudaStreamSynchronize(stream));
      release();
    }
    void* q = nullptr;
    const cudaError_t e = PINNED ? cudaHostAlloc(&q, n, cudaHostAllocDefault) : cudaMalloc(&q, n);
    if (e != cudaSuccess) cudaGetLastError();   // consume the refusal, so that the next launch check does not report it
    B200_CUDA(e);
    p = q;
    bytes = n;
    return cut(take_all);
  }
  template <class F>
  int cut(F& take_all) {
    Carver c(p, bytes);
    take_all(c);
    if (c.overrun) { set_error("buffer list larger than its block"); return B200ORB_EINVAL; }
    return B200ORB_OK;
  }
};
using DeviceBlock = Block<false>;
using HostBlock = Block<true>;

// A stream or event, created once and destroyed with its owner.  create(): a stream is non-blocking, `arg` is its
// priority; an event records timing only when `arg` is nonzero.
static inline cudaError_t cuda_create(cudaStream_t* s, int priority) {
  return cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, priority);
}
static inline cudaError_t cuda_create(cudaEvent_t* e, int timing) {
  return cudaEventCreateWithFlags(e, timing ? cudaEventDefault : cudaEventDisableTiming);
}
static inline void cuda_destroy(cudaStream_t s) { cudaStreamDestroy(s); }
static inline void cuda_destroy(cudaEvent_t e) { cudaEventDestroy(e); }
template <class T>
struct Owned {
  T h = nullptr;
  Owned() = default;
  Owned(Owned&& o) noexcept : h(o.h) { o.h = nullptr; }
  Owned(const Owned&) = delete;
  Owned& operator=(const Owned&) = delete;
  ~Owned() {
    if (h) cuda_destroy(h);
  }
  int create(int arg = 0) {
    B200_CUDA(cuda_create(&h, arg));
    return B200ORB_OK;
  }
  operator T() const { return h; }
};
using Stream = Owned<cudaStream_t>;
using Event = Owned<cudaEvent_t>;

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

// Every *_destroy: the handle's members free themselves, on its device.
template <class H>
static void destroy_handle(H* h) {
  if (!h) return;
  DeviceGuard g(h->device);
  delete h;
}

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
