// gcm.cu -- the T-variant dense map: an accumulated world-frame colour cloud, re-filtered as a whole by a VoxelGrid
// after every batch of keyframes (PointCloudMapping::viewer, src/pointcloudmapping.cc:395-500: generatePointCloud :131-194,
// removeNaNFromPointCloud + "*globalMap += *out_pt" :482-485, "voxel.setInputCloud(globalMap); voxel.filter(*tmp);
// globalMap->swap(*tmp)" :490-493).  PCL semantics follow oracle/occ_ref.cpp (occ_ref_global_refilter), which states them.
//
// The refilter of N points is order-exact and fully parallel:
//   bounding box (ordered-int atomics) -> linear cell index per point -> stable radix sort of (index, position)
//   -> cell heads -> one thread per cell sums its points in sorted (= input) order in float -> centroids in index order.
// Non-finite points stay in the list with the no-cell key (gcm.cuh) and fall off the end of the sort
// (removeNaNFromPointCloud).
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <memory>
#include <new>

#include "gcm.cuh"

namespace b200 {

__device__ __forceinline__ unsigned f2ord(float f) {   // order-preserving float -> unsigned
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned o) {
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// generatePointCloud (:160-186): every pixel, no gate; transformPointCloud with Tcw^-1 in double
__global__ void k_gcm_backproject(const float* __restrict__ depth, const uint8_t* __restrict__ bgr, int rows, int cols,
                                  float fx, float fy, float cx, float cy, const double* __restrict__ RtTi /*[12]*/,
                                  float* __restrict__ xyz, uint8_t* __restrict__ rgb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols, c = i - r * cols;
  const float d = depth[i];
  const float xf = ((float)c - cx) * d / fx, yf = ((float)r - cy) * d / fy;   // float, true division (--fmad=false)
  const double px = xf, py = yf, pz = d;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    // transformPointCloud copies non-finite points unchanged when the cloud is not dense; they are dropped later anyway
    xyz[(size_t)i * 3 + k] = (float)(RtTi[k * 3 + 0] * px + RtTi[k * 3 + 1] * py + RtTi[k * 3 + 2] * pz + RtTi[9 + k]);
  }
  rgb[(size_t)i * 3 + 0] = bgr[(size_t)i * 3 + 2];   // r,g,b from the BGR image (:178-180)
  rgb[(size_t)i * 3 + 1] = bgr[(size_t)i * 3 + 1];
  rgb[(size_t)i * 3 + 2] = bgr[(size_t)i * 3 + 0];
}

__global__ void k_gcm_minmax(const float* __restrict__ xyz, long long n, unsigned* __restrict__ mm /*[6] min xyz, max xyz*/) {
  unsigned lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float x = xyz[i * 3], y = xyz[i * 3 + 1], z = xyz[i * 3 + 2];
    if (!(isfinite(x) && isfinite(y) && isfinite(z))) continue;
    const unsigned o[3] = {f2ord(x), f2ord(y), f2ord(z)};
#pragma unroll
    for (int k = 0; k < 3; ++k) { lo[k] = min(lo[k], o[k]); hi[k] = max(hi[k], o[k]); }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    lo[k] = __reduce_min_sync(0xffffffffu, lo[k]);
    hi[k] = __reduce_max_sync(0xffffffffu, hi[k]);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { atomicMin(&mm[k], lo[k]); atomicMax(&mm[3 + k], hi[k]); }
  }
}

// PCL VoxelGrid::applyFilter: the overflow test, then min_b = floor(min * inv), div_b, linear index.  Where the index
// space overflows int (flag[0]), PCL builds no grid and neither does this: every point keeps the no-cell key, and no
// div_b product is formed (it could overflow int).
__global__ void k_gcm_index(const float* __restrict__ xyz, long long n, float inv, const unsigned* __restrict__ mm,
                            unsigned* __restrict__ idx, int* __restrict__ pos, int* __restrict__ flag) {
  const float mn[3] = {ord2f(mm[0]), ord2f(mm[1]), ord2f(mm[2])}, mx[3] = {ord2f(mm[3]), ord2f(mm[4]), ord2f(mm[5])};
  const long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1,
                  dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  const bool grid = dx * dy * dz <= 2147483647LL;
  if (!grid && blockIdx.x == 0 && threadIdx.x == 0) flag[0] = 1;
  int min_b[3] = {0, 0, 0}, m1 = 0, m2 = 0;
  if (grid) {
    int div_b[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      min_b[k] = (int)floorf(mn[k] * inv);
      div_b[k] = (int)floorf(mx[k] * inv) - min_b[k] + 1;
    }
    m1 = div_b[0];
    m2 = div_b[0] * div_b[1];
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float x = xyz[i * 3], y = xyz[i * 3 + 1], z = xyz[i * 3 + 2];
    unsigned v = gcm_no_cell<unsigned>();
    if (grid && isfinite(x) && isfinite(y) && isfinite(z)) {
      const int i0 = (int)(floorf(x * inv) - (float)min_b[0]);
      const int i1 = (int)(floorf(y * inv) - (float)min_b[1]);
      const int i2 = (int)(floorf(z * inv) - (float)min_b[2]);
      v = (unsigned)(i0 + i1 * m1 + i2 * m2);
    }
    idx[i] = v;
    pos[i] = (int)i;
  }
}

// gcm_refilter's overflow path: the positions of the finite points (read from the points: there are no cell keys),
// and their gather
struct GcmFinite {
  const float* xyz;
  __device__ bool operator()(int i) const {
    const size_t p = (size_t)i * 3;
    return isfinite(xyz[p]) && isfinite(xyz[p + 1]) && isfinite(xyz[p + 2]);
  }
};

__global__ void k_gcm_gather(const int* __restrict__ sel, const int* __restrict__ m, const float* __restrict__ xyz,
                             const uint8_t* __restrict__ rgb, float* __restrict__ oxyz, uint8_t* __restrict__ orgb) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= *m) return;
  const size_t p = (size_t)sel[u];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    oxyz[(size_t)u * 3 + k] = xyz[p * 3 + k];
    orgb[(size_t)u * 3 + k] = rgb[p * 3 + k];
  }
}

int gcm_backproject(gcm* h, const float* d_depth, const uint8_t* d_bgr, int rows, int cols, float fx, float fy, float cx,
                    float cy) {
  const long long npix = (long long)rows * cols;
  k_gcm_backproject<<<(unsigned)((npix + 255) / 256), 256, 0, h->stream>>>(d_depth, d_bgr, rows, cols, fx, fy, cx, cy, h->d_T,
                                                                          h->d_xyz + h->n * 3, h->d_rgb + h->n * 3);
  ++h->launches;
  B200_CUDA(cudaGetLastError());
  h->n += npix;
  return B200ORB_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int gcm_create(float leaf, int device, gcm_t** out) {
  if (!out || !(leaf > 0)) { set_error("bad argument"); return B200ORB_EINVAL; }
  *out = nullptr;
  B200_CHECK(check_device(device));
  DeviceGuard g(device);
  std::unique_ptr<gcm> h(new (std::nothrow) gcm());
  if (!h) { set_error("out of host memory"); return B200ORB_EINVAL; }
  h->device = device;
  h->sms = sm_count(device);
  h->leaf = leaf;
  B200_CHECK(h->stream.create());
  B200_CHECK(h->words.carve(h->stream, [&](Carver& t) {
    h->d_mm = t.take<unsigned>(6); h->d_flag = t.take<int>(2); h->d_T = t.take<double>(12);
  }));
  *out = h.release();
  return B200ORB_OK;
}
void gcm_destroy(gcm_t* h) { destroy_handle(h); }

int gcm_add_keyframe_device(gcm_t* h, const float* d_depth, const uint8_t* d_bgr, int rows, int cols, const float Tcw[16],
                            float fx, float fy, float cx, float cy) {
  if (!h || !d_depth || !d_bgr || !Tcw || rows <= 0 || cols <= 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  const long long npix = (long long)rows * cols;
  B200_CHECK(h->reserve(h->n + npix));
  double RtTi[12], R[9], t[3];
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) R[i * 3 + j] = (double)Tcw[i * 4 + j]; t[i] = (double)Tcw[i * 4 + 3]; }
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) RtTi[i * 3 + j] = R[j * 3 + i];
    RtTi[9 + i] = -(R[0 * 3 + i] * t[0] + R[1 * 3 + i] * t[1] + R[2 * 3 + i] * t[2]);
  }
  B200_CUDA(cudaMemcpyAsync(h->d_T, RtTi, sizeof(RtTi), cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));   // RtTi is a local; the call is not on a hot path
  return gcm_backproject(h, d_depth, d_bgr, rows, cols, fx, fy, cx, cy);
}

int gcm_add_keyframe(gcm_t* h, const float* depth, const uint8_t* bgr, int rows, int cols, const float Tcw[16], float fx,
                     float fy, float cx, float cy) {
  if (!h || !depth || !bgr || !Tcw || rows <= 0 || cols <= 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  const size_t npix = (size_t)rows * cols;
  float* d_depth;
  uint8_t* d_bgr;
  B200_CHECK(h->stage.reserve(h->stream, [&](Carver& t) { d_depth = t.take<float>(npix); d_bgr = t.take<uint8_t>(3 * npix); }));
  B200_CUDA(cudaMemcpyAsync(d_depth, depth, npix * 4, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_bgr, bgr, npix * 3, cudaMemcpyHostToDevice, h->stream));
  B200_CHECK(gcm_add_keyframe_device(h, d_depth, d_bgr, rows, cols, Tcw, fx, fy, cx, cy));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

// voxel.setInputCloud(globalMap); voxel.filter(*tmp); globalMap->swap(*tmp)  (src/pointcloudmapping.cc:490-493)
int gcm_refilter(gcm_t* h) {
  if (!h) { set_error("null argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  if (h->n == 0) return B200ORB_OK;
  if (h->n > 2147483647LL) { set_error("global map larger than 2^31 points"); return B200ORB_ECAP; }
  cudaStream_t st = h->stream;
  const long long n = h->n;
  const float inv = 1.0f / h->leaf;
  // CUB scratch for the largest of the three primitives at n points
  size_t s1 = 0, s2 = 0, s3 = 0;
  unsigned *d_idx, *d_idx2;
  int *d_pos, *d_pos2, *d_starts;
  uint8_t* d_head;
  void* d_tmp;
  cub::DeviceRadixSort::SortPairs(nullptr, s1, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, (int)n, 0, 32,
                                  st);
  cub::DeviceSelect::Flagged(nullptr, s2, thrust::counting_iterator<int>(0), (uint8_t*)nullptr, (int*)nullptr, (int*)nullptr,
                             (int)n, st);
  cub::DeviceSelect::If(nullptr, s3, thrust::counting_iterator<int>(0), (int*)nullptr, (int*)nullptr, (int)n, GcmFinite{nullptr},
                        st);
  const size_t tmp_bytes = std::max(std::max(s1, s2), s3);
  B200_CHECK(h->sort.reserve(st, [&](Carver& t) {
    d_idx = t.take<unsigned>(n); d_idx2 = t.take<unsigned>(n); d_pos = t.take<int>(n); d_pos2 = t.take<int>(n);
    d_starts = t.take<int>(n); d_head = t.take<uint8_t>(n); d_tmp = t.take<char>(tmp_bytes);
  }));
  static const unsigned mm0[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
  B200_CUDA(cudaMemcpyAsync(h->d_mm, mm0, 24, cudaMemcpyHostToDevice, st));
  B200_CUDA(cudaMemsetAsync(h->d_flag, 0, 8, st));
  k_gcm_minmax<<<2 * h->sms, 256, 0, st>>>(h->d_xyz, n, h->d_mm);
  k_gcm_index<<<4 * h->sms, 256, 0, st>>>(h->d_xyz, n, inv, h->d_mm, d_idx, d_pos, h->d_flag);
  size_t tb = tmp_bytes;
  B200_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, d_idx, d_idx2, d_pos, d_pos2, (int)n, 0, 32, st));
  k_gcm_heads<unsigned><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_idx2, n, d_head);
  tb = tmp_bytes;
  B200_CUDA(cub::DeviceSelect::Flagged(d_tmp, tb, thrust::counting_iterator<int>(0), d_head, d_starts, h->d_flag + 1, (int)n,
                                       st));
  int flag[2] = {0, 0};
  B200_CUDA(cudaMemcpyAsync(flag, h->d_flag, 8, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  h->launches += 5;
  if (flag[0]) {   // PCL: "Leaf size is too small for the input dataset. Integer indices would overflow." -> output = input
    // The reference's globalMap never holds a non-finite point (removeNaNFromPointCloud runs before "*globalMap += ...",
    // :484-485), so the map keeps its finite points, in insertion order.
    tb = tmp_bytes;
    B200_CUDA(cub::DeviceSelect::If(d_tmp, tb, thrust::counting_iterator<int>(0), d_starts, h->d_flag + 1, (int)n,
                                    GcmFinite{h->d_xyz}, st));
    k_gcm_gather<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_starts, h->d_flag + 1, h->d_xyz, h->d_rgb, h->d_xyz2, h->d_rgb2);
    h->launches += 2;
    B200_CUDA(cudaGetLastError());
    int kept = 0;
    B200_CUDA(cudaMemcpyAsync(&kept, h->d_flag + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    std::swap(h->d_xyz, h->d_xyz2);
    std::swap(h->d_rgb, h->d_rgb2);
    h->n = kept;
    set_error("VoxelGrid index space overflows int for this leaf size (PCL returns the cloud unfiltered)");
    return B200ORB_EGEOM;
  }
  const int cells = flag[1];
  if (cells > 0) {
    k_gcm_centroids<unsigned, true><<<(unsigned)((cells + 127) / 128), 128, 0, st>>>(d_idx2, d_pos2, d_starts, h->d_flag + 1, n,
                                                                                     h->d_xyz, h->d_rgb, h->d_xyz2, h->d_rgb2);
    ++h->launches;
  }
  B200_CUDA(cudaGetLastError());
  std::swap(h->d_xyz, h->d_xyz2);
  std::swap(h->d_rgb, h->d_rgb2);
  h->n = cells;
  return B200ORB_OK;
}

long long gcm_size(const gcm_t* h) { return h ? h->n : -1; }

int gcm_export(gcm_t* h, float* xyz, uint8_t* rgb, long long cap, long long* n) {
  if (!h || !n) { set_error("null argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  *n = h->n;
  if (!xyz) return B200ORB_OK;
  if (h->n > cap) { set_error("cap %lld < %lld points", cap, h->n); return B200ORB_ECAP; }
  B200_CUDA(cudaMemcpyAsync(xyz, h->d_xyz, (size_t)12 * h->n, cudaMemcpyDeviceToHost, h->stream));
  if (rgb) B200_CUDA(cudaMemcpyAsync(rgb, h->d_rgb, (size_t)3 * h->n, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int gcm_sync(gcm_t* h) {
  if (!h) return B200ORB_EINVAL;
  DeviceGuard g(h->device);
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}
long long gcm_launch_count(const gcm_t* h) { return h ? h->launches : 0; }

}  // extern "C"
