// gcm.cuh -- the T-variant dense map's handle and what its semantic clusters (gcm_sem.cu) share with the map's VoxelGrid
// (gcm.cu): the cell heads and centroids of a sorted key list, and the back-projection of a keyframe into the map.
#pragma once
#include "common.cuh"

namespace b200 {

// Key = unsigned (the map's cell index) or unsigned long long (gcm_sem.cu: box << 32 | cell index).  Cell indices
// exist only in a grid that passes PCL's overflow test (where it fails, k_gcm_index gives every point the no-cell key
// and k_sem_cellkey numbers the points instead).  Such an index lies in [0, INT_MAX] -- INT_MAX itself included: div_b
// may exceed PCL's dx, dy, dz by one, so the last cell can have index INT_MAX -- and a box is below 2^31, so the
// all-ones key is never a cell: it marks a point without one and sorts last.
template <class Key>
__host__ __device__ constexpr Key gcm_no_cell() {
  static_assert(Key(0) < Key(-1), "cell keys are unsigned");
  return ~Key(0);
}

template <class Key>
__global__ void k_gcm_heads(const Key* __restrict__ idx_sorted, long long n, uint8_t* __restrict__ head) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Key v = idx_sorted[i];
  head[i] = (v != gcm_no_cell<Key>()) && (i == 0 || idx_sorted[i - 1] != v);
}

// one thread per cell: sequential float sums in sorted (= input) order, centroid = sum / count (colour only if kRgb)
template <class Key, bool kRgb>
__global__ void k_gcm_centroids(const Key* __restrict__ idx_sorted, const int* __restrict__ pos_sorted,
                                const int* __restrict__ starts, const int* __restrict__ ncells, long long n,
                                const float* __restrict__ xyz, const uint8_t* __restrict__ rgb,
                                float* __restrict__ oxyz, uint8_t* __restrict__ orgb) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= *ncells) return;
  const int b = starts[u];
  const Key key = idx_sorted[b];
  float sx = 0.f, sy = 0.f, sz = 0.f, sr = 0.f, sg = 0.f, sb = 0.f;
  int e = b;
  for (; e < n && idx_sorted[e] == key; ++e) {
    const size_t p = (size_t)pos_sorted[e];
    sx += xyz[p * 3]; sy += xyz[p * 3 + 1]; sz += xyz[p * 3 + 2];
    if (kRgb) { sr += (float)rgb[p * 3]; sg += (float)rgb[p * 3 + 1]; sb += (float)rgb[p * 3 + 2]; }
  }
  const float fn = (float)(e - b);
  oxyz[(size_t)u * 3] = sx / fn; oxyz[(size_t)u * 3 + 1] = sy / fn; oxyz[(size_t)u * 3 + 2] = sz / fn;
  if (!kRgb) return;
  orgb[(size_t)u * 3] = (uint8_t)(sr / fn); orgb[(size_t)u * 3 + 1] = (uint8_t)(sg / fn); orgb[(size_t)u * 3 + 2] = (uint8_t)(sb / fn);
}

}  // namespace b200

struct gcm {
  int device = 0;
  int sms = 1;
  float leaf = 0.f;
  b200::Stream stream;
  long long launches = 0;
  long long n = 0, cap = 0;   // points in the global map / capacity of the point block
  b200::DeviceBlock words;
  unsigned* d_mm = nullptr;
  int* d_flag = nullptr;      // [0] overflow, [1] number of cells
  double* d_T = nullptr;      // Rt (9) + ti (3)
  b200::DeviceBlock points;   // two sets of `cap` points: the map, and gcm_refilter's output
  float *d_xyz = nullptr, *d_xyz2 = nullptr;
  uint8_t *d_rgb = nullptr, *d_rgb2 = nullptr;
  b200::DeviceBlock sort;     // gcm_refilter's sort of the map and its CUB scratch
  b200::DeviceBlock stage;    // gcm_add_keyframe's uploads
  b200::DeviceBlock sem_pos, sem_pts;   // gcm_add_keyframe_objects: per-position scratch, per-band-point scratch (gcm_sem.cu)
  int reserve(long long need) {
    if (need <= cap) return B200ORB_OK;
    const long long nc = std::max<long long>(need, cap * 2);
    b200::DeviceBlock grown;
    float *xyz, *xyz2;
    uint8_t *rgb, *rgb2;
    B200_CHECK(grown.carve(stream, [&](b200::Carver& t) {
      xyz = t.take<float>(3 * nc); rgb = t.take<uint8_t>(3 * nc); xyz2 = t.take<float>(3 * nc); rgb2 = t.take<uint8_t>(3 * nc);
    }));
    if (n > 0) {
      B200_CUDA(cudaMemcpyAsync(xyz, d_xyz, 12 * n, cudaMemcpyDeviceToDevice, stream));
      B200_CUDA(cudaMemcpyAsync(rgb, d_rgb, 3 * n, cudaMemcpyDeviceToDevice, stream));
    }
    B200_CUDA(cudaStreamSynchronize(stream));
    points = std::move(grown);
    d_xyz = xyz; d_rgb = rgb; d_xyz2 = xyz2; d_rgb2 = rgb2;
    cap = nc;
    return B200ORB_OK;
  }
};

namespace b200 {
// generatePointCloud (src/pointcloudmapping.cc:160-186) of one keyframe, k_gcm_backproject in gcm.cu: its rows x cols
// points, transformed by the pose in h->d_T, are appended to the map, which has room for them.
int gcm_backproject(gcm* h, const float* d_depth, const uint8_t* d_bgr, int rows, int cols, float fx, float fy, float cx,
                    float cy);
}  // namespace b200
