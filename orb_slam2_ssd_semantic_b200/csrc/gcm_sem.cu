// gcm_sem.cu -- the semantic object clusters of PointCloudMapping::viewer (src/pointcloudmapping.cc:399-488) for one
// keyframe and any number of detector boxes: draw_rect_with_depth_threshold (:197-244) paints each box's depth band and
// lists its flat indices, generatePointCloud runs on the painted image (gcm_backproject, gcm.cu), and every box's
// band points go through ExtractIndices, StatisticalOutlierRemoval(50, 1.0), VoxelGrid(resolution), compute3DCentroid
// and getMinMax3D (:443-476).  PCL semantics follow oracle/sem_ref.cpp, which states them.
//
//   per box (one thread, sequential float sum)   mean depth over the 30-70 % window
//   per pixel                                    band test against every box, the last box that holds the pixel paints
//   per band position (CUB select)               the band list in the reference's (k, j) order, wraps and repeats included
//   per band point                               its world point, gathered from the cloud just appended to the map
//   per query, candidates tiled in shared memory the 51 smallest squared distances -> mean of the 50 square roots
//   per box (one thread, sequential double sums) SOR mean / stddev -> threshold
//   CUB select                                   ordered keep-compaction
//   per box bounding box, then one stable radix sort of (box << 32 | cell) with gcm.cuh's cell heads and float sums
//   per box (one thread)                         centroid (float sums in cell order) and min / max
// The host syncs twice, to size the per-point buffers and the sort; the call is synchronous like gcm_add_keyframe.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <cfloat>
#include <cmath>
#include <vector>

#include "gcm.cuh"

namespace b200 {

constexpr int SEM_CLASSES = 21;       // colors_ / obj_size_ have 21 entries (:50-70)
constexpr int SEM_MEAN_K = 50;        // stat.setMeanK(50) (:75)
constexpr int SEM_K = SEM_MEAN_K + 1; // nearestKSearch(mean_k_ + 1): the point itself and its 50 neighbours
constexpr int SEM_NN_THREADS = 128;
constexpr float SEM_MAX_RECT = 16777216.f;   // 2^24 px: keeps every (int) conversion and index product in range

// colors_ (:50-60), B,G,R: i*10 + 40 grey, except bottle 5, chair 9, person 15, tvmonitor 20
__constant__ uint8_t c_sem_colors[SEM_CLASSES][3] = {
    {40, 40, 40},    {50, 50, 50},    {60, 60, 60},    {70, 70, 70},    {80, 80, 80},    {255, 0, 255},
    {100, 100, 100}, {110, 110, 110}, {120, 120, 120}, {255, 0, 0},     {140, 140, 140}, {150, 150, 150},
    {160, 160, 160}, {170, 170, 170}, {180, 180, 180}, {0, 0, 255},     {200, 200, 200}, {210, 210, 210},
    {220, 220, 220}, {230, 230, 230}, {0, 255, 0}};

struct SemBox {
  long long beg;   // (int)rect.x + ((int)rect.y - 1) * cols - 1 (:206)
  int pos0;        // first band position of this box in the keyframe's position space
  int wi;          // (int)rect.width
  int k0, k1;      // mean-depth rows [k0, k1): k from (int)((int)h*0.3) while k < (int)h*0.7 (:211)
  int hk, wj;      // band rows [0, hk) = (int)h - 1, band columns [0, wj) = (int)w - 2 of each row (:228-232)
  int cls;
};

struct SemNnBlock { int begin, end, q0; };    // a box's band points [begin, end) and this block's first query

struct SemVoxel { int min_b[3], mul[3]; int overflow; };

__device__ __forceinline__ long long sem_floor_div(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// abs(depth[j] - depth_threshold) < 0.4 (:234): float abs, double compare; NaN never passes
__device__ __forceinline__ bool sem_in_band(float d, float thr) { return (double)fabsf(d - thr) < 0.4; }

// the box holding band position p: the last box whose first position is <= p (boxes without positions share the next
// box's pos0 and lose to it)
__device__ __forceinline__ int sem_box_of(const SemBox* __restrict__ box, int B, int p) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (box[mid].pos0 <= p) lo = mid; else hi = mid - 1;
  }
  return lo;
}
__device__ __forceinline__ long long sem_flat(const SemBox& x, int p, int cols) {
  const int q = p - x.pos0, k = q / x.wj, jj = q - k * x.wj;
  return x.beg + (long long)k * cols + jj;   // start = beg + k*cols, j = start + jj: wraps into the next row
}

// :208-225, one thread per box: the float sum is sequential in row-major order
__global__ void k_sem_mean(const float* __restrict__ depth, long long npix, int cols, const SemBox* __restrict__ box, int B,
                           float* __restrict__ thr) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const SemBox x = box[b];
  float sum = 0.f;
  int count = 0;
  for (int k = x.k0; k < x.k1; ++k) {
    const long long start = x.beg + (long long)k * cols;
    const long long j0 = (long long)((double)start + x.wi * 0.3), j1 = (long long)((double)start + x.wi * 0.7);
    for (long long j = j0; j < j1; ++j) {
      if (j < 0 || j >= npix) continue;   // deviation: the reference reads out of bounds here
      const float d = depth[j];
      if (d < 0.5 || d > 6) continue;     // NaN passes this test and poisons the sum, as in the reference
      sum += d;
      ++count;
    }
  }
  thr[b] = count > 0 ? sum / (float)count : 0.f;
}

// :237-239 + :439: the colour image generatePointCloud reads -- each pixel takes the colour of the LAST box whose band
// holds it.  Pixel i lies in box b's (k, jj) grid iff some k in [0, hk) has jj = i - beg - k*cols in [0, wj).
__global__ void k_sem_paint(const float* __restrict__ depth, const uint8_t* __restrict__ bgr, long long npix, int cols,
                            const SemBox* __restrict__ box, const float* __restrict__ thr, int B, uint8_t* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  uint8_t c0 = bgr[i * 3], c1 = bgr[i * 3 + 1], c2 = bgr[i * 3 + 2];
  const float d = depth[i];
  for (int b = B - 1; b >= 0; --b) {
    const SemBox x = box[b];
    if (x.hk == 0 || x.wj == 0 || !sem_in_band(d, thr[b])) continue;
    const long long off = i - x.beg;
    const long long kmax = min((long long)x.hk - 1, sem_floor_div(off, cols));
    const long long kmin = max(0LL, -sem_floor_div(-(off - x.wj + 1), cols));
    if (kmin > kmax) continue;
    c0 = c_sem_colors[x.cls][0]; c1 = c_sem_colors[x.cls][1]; c2 = c_sem_colors[x.cls][2];
    break;
  }
  out[i * 3] = c0; out[i * 3 + 1] = c1; out[i * 3 + 2] = c2;
}

// indices.indices.push_back(j) (:236): position p is listed iff its flat index is in the image and in the band
struct SemBandPred {
  const float* depth;
  const SemBox* box;
  const float* thr;
  int B, cols;
  long long npix;
  __device__ bool operator()(int p) const {
    const int b = sem_box_of(box, B, p);
    const long long j = sem_flat(box[b], p, cols);
    return j >= 0 && j < npix && sem_in_band(depth[j], thr[b]);
  }
};

// out[b] = first index of arr[0, *n) with arr >= v[b], out[B] = *n (arr ascending)
__global__ void k_sem_starts(const int* __restrict__ arr, const int* __restrict__ n, const int* __restrict__ v, int B,
                             int* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > B) return;
  const int N = *n;
  if (b == B) { out[B] = N; return; }
  int lo = 0, hi = N;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (arr[mid] < v[b]) lo = mid + 1; else hi = mid;
  }
  out[b] = lo;
}

// extract_indices.filter (:449-452): band point i's world point is cloud point j of the keyframe just appended
__global__ void k_sem_gather(const int* __restrict__ sel, int N, const SemBox* __restrict__ box, int B, int cols,
                             const float* __restrict__ cloud, float* __restrict__ bxyz, int* __restrict__ ibox) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int p = sel[i], b = sem_box_of(box, B, p);
  const long long j = sem_flat(box[b], p, cols);
  bxyz[(size_t)i * 3] = cloud[j * 3]; bxyz[(size_t)i * 3 + 1] = cloud[j * 3 + 1]; bxyz[(size_t)i * 3 + 2] = cloud[j * 3 + 2];
  ibox[i] = b;
}

// StatisticalOutlierRemoval's first pass: nearestKSearch(i, 51) over the box's points (FLANN L2_Simple<float>:
// ((0 + dx*dx) + dy*dy) + dz*dz, no FMA), then distance = (float)(sum_{k=1..50} sqrt(d_k) in double, ascending / 50).
// Only the multiset of the 51 smallest values matters (ties are equal values); each query keeps it sorted in a
// column of shared memory.
__global__ void __launch_bounds__(SEM_NN_THREADS) k_sem_knn(const float* __restrict__ bxyz,
                                                            const SemNnBlock* __restrict__ blocks, float* __restrict__ dist) {
  __shared__ float top[SEM_K * SEM_NN_THREADS];
  __shared__ float tx[SEM_NN_THREADS], ty[SEM_NN_THREADS], tz[SEM_NN_THREADS];
  const SemNnBlock blk = blocks[blockIdx.x];
  const int t = threadIdx.x, q = blk.q0 + t;
  const bool act = q < blk.end;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (act) { qx = bxyz[(size_t)q * 3]; qy = bxyz[(size_t)q * 3 + 1]; qz = bxyz[(size_t)q * 3 + 2]; }
#pragma unroll 1
  for (int k = 0; k < SEM_K; ++k) top[k * SEM_NN_THREADS + t] = INFINITY;
  float kth = INFINITY;
  // tiles from the block's own one onwards, wrapping: band order is raster order, so the nearest candidates come first
  // and few later ones reach the list (the multiset does not depend on the order)
  const int ntiles = (blk.end - blk.begin + SEM_NN_THREADS - 1) / SEM_NN_THREADS, t0 = (blk.q0 - blk.begin) / SEM_NN_THREADS;
  for (int s = 0; s < ntiles; ++s) {
    const int c0 = blk.begin + ((t0 + s) % ntiles) * SEM_NN_THREADS;
    __syncthreads();
    if (c0 + t < blk.end) {
      const size_t c = (size_t)(c0 + t) * 3;
      tx[t] = bxyz[c]; ty[t] = bxyz[c + 1]; tz[t] = bxyz[c + 2];
    }
    __syncthreads();
    if (!act) continue;
    const int m = min(SEM_NN_THREADS, blk.end - c0);
    for (int u = 0; u < m; ++u) {
      const float dx = __fsub_rn(qx, tx[u]), dy = __fsub_rn(qy, ty[u]), dz = __fsub_rn(qz, tz[u]);
      const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      if (d < kth) {
        int p = SEM_K - 1;
        for (; p > 0; --p) {
          const float v = top[(p - 1) * SEM_NN_THREADS + t];
          if (!(v > d)) break;
          top[p * SEM_NN_THREADS + t] = v;
        }
        top[p * SEM_NN_THREADS + t] = d;
        kth = top[(SEM_K - 1) * SEM_NN_THREADS + t];
      }
    }
  }
  if (!act) return;
  double s = 0.0;
  for (int k = 1; k < SEM_K; ++k) s += sqrt((double)top[k * SEM_NN_THREADS + t]);
  dist[q] = (float)(s / SEM_MEAN_K);
}

// the second half of the first pass: sum += distance, sq_sum += distance*distance (float product), mean, variance,
// threshold = mean + 1.0 * stddev -- sequential double sums in band order, one thread per box
__global__ void k_sem_sor(const float* __restrict__ dist, const int* __restrict__ bstart, int B, double* __restrict__ sthr) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int s = bstart[b], e = bstart[b + 1];
  if (e - s < SEM_K) return;
  double sum = 0.0, sq_sum = 0.0;
  for (int i = s; i < e; ++i) {
    const float d = dist[i];
    sum += d;
    sq_sum += __fmul_rn(d, d);
  }
  const double n = (double)(e - s);
  const double mean = sum / n;
  const double variance = (sq_sum - sum * sum / n) / (n - 1);
  sthr[b] = mean + 1.0 * sqrt(variance);
}

// the second pass: a point is kept iff !(distance > threshold)
__global__ void k_sem_keep(const float* __restrict__ dist, const int* __restrict__ ibox, const int* __restrict__ bstart,
                           const double* __restrict__ sthr, int N, uint8_t* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int b = ibox[i];
  keep[i] = (bstart[b + 1] - bstart[b] >= SEM_K) && !((double)dist[i] > sthr[b]);
}

// VoxelGrid::applyFilter per box: bounding box of the box's inliers, min_b / div_b, and PCL's int-overflow test
// (as k_gcm_minmax + k_gcm_index do for the whole map).  One block per box.
__global__ void k_sem_bbox(const float* __restrict__ bxyz, const int* __restrict__ kept, const int* __restrict__ kstart,
                           float inv, SemVoxel* __restrict__ vg) {
  const int b = blockIdx.x, s = kstart[b], e = kstart[b + 1];
  if (s == e) return;
  __shared__ float red[6][32];
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = s + threadIdx.x; i < e; i += blockDim.x) {
    const size_t t = (size_t)kept[i] * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) { lo[k] = fminf(lo[k], bxyz[t + k]); hi[k] = fmaxf(hi[k], bxyz[t + k]); }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k)
    for (int o = 16; o > 0; o >>= 1) {
      lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
      hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
    }
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { red[k][w] = lo[k]; red[3 + k][w] = hi[k]; }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  float mn[3], mx[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    mn[k] = red[k][0]; mx[k] = red[3 + k][0];
    for (int u = 1; u < nw; ++u) { mn[k] = fminf(mn[k], red[k][u]); mx[k] = fmaxf(mx[k], red[3 + k][u]); }
  }
  SemVoxel v;
  const long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1,
                  dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  v.overflow = dx * dy * dz > 2147483647LL;
  int div_b[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    v.min_b[k] = (int)floorf(mn[k] * inv);
    div_b[k] = (int)floorf(mx[k] * inv) - v.min_b[k] + 1;
  }
  v.mul[0] = 1; v.mul[1] = div_b[0]; v.mul[2] = div_b[0] * div_b[1];
  vg[b] = v;
}

// sort key of inlier i: box << 32 | linear cell index; where the box's index space overflows, PCL returns the input
// unchanged, so every point becomes its own cell in input order (a centroid of one point is the point)
__global__ void k_sem_cellkey(const float* __restrict__ bxyz, const int* __restrict__ kept, int nk, const int* __restrict__ ibox,
                              const int* __restrict__ kstart, const SemVoxel* __restrict__ vg, float inv,
                              float* __restrict__ kxyz, unsigned long long* __restrict__ key, int* __restrict__ pos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nk) return;
  const int t = kept[i], b = ibox[t];
  const float x = bxyz[(size_t)t * 3], y = bxyz[(size_t)t * 3 + 1], z = bxyz[(size_t)t * 3 + 2];
  kxyz[(size_t)i * 3] = x; kxyz[(size_t)i * 3 + 1] = y; kxyz[(size_t)i * 3 + 2] = z;
  const SemVoxel v = vg[b];
  int cell;
  if (v.overflow) {
    cell = i - kstart[b];
  } else {
    const int i0 = (int)(floorf(x * inv) - (float)v.min_b[0]);
    const int i1 = (int)(floorf(y * inv) - (float)v.min_b[1]);
    const int i2 = (int)(floorf(z * inv) - (float)v.min_b[2]);
    cell = i0 * v.mul[0] + i1 * v.mul[1] + i2 * v.mul[2];
  }
  key[i] = ((unsigned long long)b << 32) | (unsigned)cell;
  pos[i] = i;
}

// compute3DCentroid (float sums in output order, / count as float) and getMinMax3D over the box's voxel centroids, or
// over its inliers themselves where its VoxelGrid overflowed (a one-point centroid 0.f + x would turn -0.0 into +0.0)
__global__ void k_sem_finish(const unsigned long long* __restrict__ key, const int* __restrict__ cstart,
                             const int* __restrict__ ncells, const float* __restrict__ cxyz, const float* __restrict__ kxyz,
                             const SemVoxel* __restrict__ vg, const int* __restrict__ bstart, const int* __restrict__ kstart,
                             int B, GcmCluster* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  GcmCluster c = {};
  c.n_band = bstart[b + 1] - bstart[b];
  c.status = c.n_band >= SEM_K ? GCM_CLUSTER : GCM_FEW_POINTS;
  if (c.status == GCM_CLUSTER) {
    const int nc = *ncells;
    int lo = 0, hi = nc;   // first cell of box b
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if ((int)(key[cstart[mid]] >> 32) < b) lo = mid + 1; else hi = mid;
    }
    const int c0 = lo;
    hi = nc;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if ((int)(key[cstart[mid]] >> 32) <= b) lo = mid + 1; else hi = mid;
    }
    c.n_inliers = kstart[b + 1] - kstart[b];
    c.n_voxels = lo - c0;
    const float* vox = c.n_voxels > 0 && vg[b].overflow ? kxyz + (size_t)kstart[b] * 3 : cxyz + (size_t)c0 * 3;
    float s[3] = {0.f, 0.f, 0.f}, mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int u = 0; u < c.n_voxels; ++u)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float v = vox[(size_t)u * 3 + k];
        s[k] += v;
        mn[k] = v < mn[k] ? v : mn[k];
        mx[k] = v > mx[k] ? v : mx[k];
      }
#pragma unroll
    for (int k = 0; k < 3; ++k) { c.centroid[k] = s[k] / (float)c.n_voxels; c.min_pt[k] = mn[k]; c.max_pt[k] = mx[k]; }
  }
  out[b] = c;
}

}  // namespace b200

namespace b200 {
// the boxes first: their checks need no device
static int sem_check_args(const gcm_t* h, const void* depth, const void* bgr, int rows, int cols, const float* Tcw,
                          long long keyframe_index, const GcmObject* objs, int n_objs, const GcmCluster* clusters_out) {
  if (n_objs < 0 || (n_objs > 0 && (!objs || !clusters_out))) { set_error("bad argument"); return B200ORB_EINVAL; }
  for (int t = 0; t < n_objs; ++t) {
    const GcmObject& o = objs[t];
    if (o.class_id < 0 || o.class_id >= SEM_CLASSES) {
      set_error("object %d: class_id %d outside [0, %d) (colors_ / obj_size_ have 21 entries)", t, o.class_id, SEM_CLASSES);
      return B200ORB_EINVAL;
    }
    const float r[4] = {o.x, o.y, o.width, o.height};
    for (float v : r)
      if (!(std::fabs(v) <= SEM_MAX_RECT)) { set_error("object %d: rectangle not finite or beyond 2^24 px", t); return B200ORB_EINVAL; }
  }
  if (!h || !depth || !bgr || !Tcw || rows <= 0 || cols <= 0 || keyframe_index < 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  return B200ORB_OK;
}
}  // namespace b200

using namespace b200;

extern "C" {

int gcm_add_keyframe_objects_device(gcm_t* h, const float* d_depth, const uint8_t* d_bgr, int rows, int cols,
                                    const float Tcw[16], float fx, float fy, float cx, float cy, long long keyframe_index,
                                    const GcmObject* objs, int n_objs, GcmCluster* clusters_out) {
  B200_CHECK(sem_check_args(h, d_depth, d_bgr, rows, cols, Tcw, keyframe_index, objs, n_objs, clusters_out));
  if (keyframe_index % 2 == 0 && n_objs == 0) return B200ORB_OK;   // :434, the keyframe adds nothing
  DeviceGuard g(h->device);
  cudaStream_t st = h->stream;
  const long long npix = (long long)rows * cols;
  // the boxes that pass the gate (:418), in detector order
  std::vector<SemBox> box;
  std::vector<int> slot, pos0;
  long long ptot = 0;
  for (int t = 0; t < n_objs; ++t) {
    const GcmObject& o = objs[t];
    clusters_out[t] = GcmCluster{};
    clusters_out[t].status = GCM_BELOW_PROB;
    if (!((double)o.prob > 0.54)) continue;
    SemBox x;
    const int hi = (int)o.height;
    x.wi = (int)o.width;
    x.beg = (long long)(int)o.x + ((long long)(int)o.y - 1) * cols - 1;
    x.k0 = (int)(hi * 0.3);
    x.k1 = std::max(x.k0, (int)std::ceil(hi * 0.7));   // the first k with !(k < (int)h*0.7)
    x.hk = std::max(hi - 1, 0);
    x.wj = std::max(x.wi - 2, 0);
    x.cls = o.class_id;
    x.pos0 = (int)std::min<long long>(ptot, 2147483647LL);
    ptot += (long long)x.hk * x.wj;
    box.push_back(x);
    slot.push_back(t);
    pos0.push_back(x.pos0);
  }
  if (ptot > 2147483647LL) { set_error("the boxes span %lld band positions (> 2^31 - 1)", ptot); return B200ORB_ECAP; }
  const int B = (int)box.size(), P = (int)ptot;
  B200_CHECK(h->reserve(h->n + npix));
  double RtTi[12], R[9], tt[3];
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) R[i * 3 + j] = (double)Tcw[i * 4 + j]; tt[i] = (double)Tcw[i * 4 + 3]; }
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) RtTi[i * 3 + j] = R[j * 3 + i];
    RtTi[9 + i] = -(R[0 * 3 + i] * tt[0] + R[1 * 3 + i] * tt[1] + R[2 * 3 + i] * tt[2]);
  }
  // phase 1: mean depths, painting, the cloud, the band lists
  SemBox* d_box = nullptr;
  float* d_thr = nullptr;
  int *d_pos0 = nullptr, *d_bstart = nullptr, *d_sel = nullptr, *d_nsel = nullptr;
  uint8_t* d_paint = nullptr;
  void* d_tmp = nullptr;
  size_t sel_bytes = 0;
  const SemBandPred pred{d_depth, nullptr, nullptr, B, cols, npix};
  if (P > 0) cub::DeviceSelect::If(nullptr, sel_bytes, thrust::counting_iterator<int>(0), (int*)nullptr, (int*)nullptr, P, pred, st);
  B200_CHECK(h->sem_pos.reserve(st, [&](Carver& t) {
    d_box = t.take<SemBox>(B); d_thr = t.take<float>(B); d_pos0 = t.take<int>(B); d_bstart = t.take<int>(B + 1);
    d_sel = t.take<int>(P); d_nsel = t.take<int>(1); d_paint = t.take<uint8_t>(B > 0 ? 3 * npix : 1);
    d_tmp = t.take<char>(sel_bytes);
  }));
  B200_CUDA(cudaMemcpyAsync(h->d_T, RtTi, sizeof(RtTi), cudaMemcpyHostToDevice, st));
  if (B > 0) {
    B200_CUDA(cudaMemcpyAsync(d_box, box.data(), sizeof(SemBox) * B, cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemcpyAsync(d_pos0, pos0.data(), sizeof(int) * B, cudaMemcpyHostToDevice, st));
    k_sem_mean<<<(B + 63) / 64, 64, 0, st>>>(d_depth, npix, cols, d_box, B, d_thr);
    k_sem_paint<<<(unsigned)((npix + 255) / 256), 256, 0, st>>>(d_depth, d_bgr, npix, cols, d_box, d_thr, B, d_paint);
    h->launches += 2;
  }
  const long long n0 = h->n;
  B200_CHECK(gcm_backproject(h, d_depth, B > 0 ? d_paint : d_bgr, rows, cols, fx, fy, cx, cy));
  if (B == 0) { B200_CUDA(cudaStreamSynchronize(st)); return B200ORB_OK; }
  std::vector<int> bstart(B + 1, 0);
  if (P > 0) {
    const SemBandPred p{d_depth, d_box, d_thr, B, cols, npix};
    size_t tb = sel_bytes;
    B200_CUDA(cub::DeviceSelect::If(d_tmp, tb, thrust::counting_iterator<int>(0), d_sel, d_nsel, P, p, st));
    k_sem_starts<<<(B + 64) / 64, 64, 0, st>>>(d_sel, d_nsel, d_pos0, B, d_bstart);
    h->launches += 2;
    B200_CUDA(cudaMemcpyAsync(bstart.data(), d_bstart, sizeof(int) * (B + 1), cudaMemcpyDeviceToHost, st));
  }
  B200_CUDA(cudaStreamSynchronize(st));
  const int N = bstart[B];
  std::vector<SemNnBlock> nnb;
  for (int b = 0; b < B; ++b)
    if (bstart[b + 1] - bstart[b] >= SEM_K)
      for (int q = bstart[b]; q < bstart[b + 1]; q += SEM_NN_THREADS) nnb.push_back(SemNnBlock{bstart[b], bstart[b + 1], q});
  std::vector<GcmCluster> res(B);
  if (nnb.empty()) {   // no box reaches 51 band points
    for (int b = 0; b < B; ++b) {
      res[b] = GcmCluster{};
      res[b].status = GCM_FEW_POINTS;
      res[b].n_band = bstart[b + 1] - bstart[b];
    }
  } else {
    // phase 2: SOR, VoxelGrid, centroid and extent of every box
    float *d_bxyz, *d_dist, *d_kxyz, *d_cxyz;
    int *d_ibox, *d_kept, *d_nk, *d_kstart, *d_pos, *d_pos2, *d_cstart, *d_ncells, *d_bst;
    unsigned long long *d_key, *d_key2;
    uint8_t *d_keep, *d_head;
    double* d_sthr;
    SemVoxel* d_vg;
    SemNnBlock* d_nnb;
    GcmCluster* d_out;
    void* d_tmp2;
    int end_bit = 32;   // box bits above the 32 cell bits
    while ((1LL << (end_bit - 32)) < B) ++end_bit;
    size_t s1 = 0, s2 = 0;
    cub::DeviceSelect::Flagged(nullptr, s1, thrust::counting_iterator<int>(0), (uint8_t*)nullptr, (int*)nullptr, (int*)nullptr,
                               N, st);
    cub::DeviceRadixSort::SortPairs(nullptr, s2, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr,
                                    (int*)nullptr, N, 0, end_bit, st);
    const size_t tmp_bytes = std::max(s1, s2);
    B200_CHECK(h->sem_pts.reserve(st, [&](Carver& t) {
      d_bxyz = t.take<float>(3 * (size_t)N); d_kxyz = t.take<float>(3 * (size_t)N); d_cxyz = t.take<float>(3 * (size_t)N);
      d_dist = t.take<float>(N); d_ibox = t.take<int>(N); d_kept = t.take<int>(N); d_pos = t.take<int>(N);
      d_pos2 = t.take<int>(N); d_cstart = t.take<int>(N); d_key = t.take<unsigned long long>(N);
      d_key2 = t.take<unsigned long long>(N); d_keep = t.take<uint8_t>(N); d_head = t.take<uint8_t>(N);
      d_nk = t.take<int>(1); d_ncells = t.take<int>(1); d_kstart = t.take<int>(B + 1); d_bst = t.take<int>(B + 1);
      d_sthr = t.take<double>(B); d_vg = t.take<SemVoxel>(B); d_out = t.take<GcmCluster>(B);
      d_nnb = t.take<SemNnBlock>(nnb.size()); d_tmp2 = t.take<char>(tmp_bytes);
    }));
    B200_CUDA(cudaMemcpyAsync(d_bst, bstart.data(), sizeof(int) * (B + 1), cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaMemcpyAsync(d_nnb, nnb.data(), sizeof(SemNnBlock) * nnb.size(), cudaMemcpyHostToDevice, st));
    const unsigned gN = (unsigned)((N + 255) / 256), gB = (unsigned)((B + 63) / 64);
    const float inv = 1.0f / h->leaf;
    k_sem_gather<<<gN, 256, 0, st>>>(d_sel, N, d_box, B, cols, h->d_xyz + n0 * 3, d_bxyz, d_ibox);
    k_sem_knn<<<(unsigned)nnb.size(), SEM_NN_THREADS, 0, st>>>(d_bxyz, d_nnb, d_dist);
    k_sem_sor<<<gB, 64, 0, st>>>(d_dist, d_bst, B, d_sthr);
    k_sem_keep<<<gN, 256, 0, st>>>(d_dist, d_ibox, d_bst, d_sthr, N, d_keep);
    size_t tb = tmp_bytes;
    B200_CUDA(cub::DeviceSelect::Flagged(d_tmp2, tb, thrust::counting_iterator<int>(0), d_keep, d_kept, d_nk, N, st));
    k_sem_starts<<<(B + 64) / 64, 64, 0, st>>>(d_kept, d_nk, d_bst, B, d_kstart);
    k_sem_bbox<<<B, 256, 0, st>>>(d_bxyz, d_kept, d_kstart, inv, d_vg);
    int nk = 0;
    B200_CUDA(cudaMemcpyAsync(&nk, d_nk, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    h->launches += 7;
    if (nk == 0) {   // every box lost every point (a zero-variance box whose mean rounds below its distances)
      B200_CUDA(cudaMemsetAsync(d_ncells, 0, sizeof(int), st));
    } else {
      k_sem_cellkey<<<(unsigned)((nk + 255) / 256), 256, 0, st>>>(d_bxyz, d_kept, nk, d_ibox, d_kstart, d_vg, inv, d_kxyz, d_key,
                                                                  d_pos);
      tb = tmp_bytes;
      B200_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp2, tb, d_key, d_key2, d_pos, d_pos2, nk, 0, end_bit, st));
      k_gcm_heads<unsigned long long><<<(unsigned)((nk + 255) / 256), 256, 0, st>>>(d_key2, nk, d_head);
      tb = tmp_bytes;
      B200_CUDA(cub::DeviceSelect::Flagged(d_tmp2, tb, thrust::counting_iterator<int>(0), d_head, d_cstart, d_ncells, nk, st));
      k_gcm_centroids<unsigned long long, false><<<(unsigned)((nk + 127) / 128), 128, 0, st>>>(
          d_key2, d_pos2, d_cstart, d_ncells, nk, d_kxyz, nullptr, d_cxyz, nullptr);
      h->launches += 4;
    }
    k_sem_finish<<<gB, 64, 0, st>>>(d_key2, d_cstart, d_ncells, d_cxyz, d_kxyz, d_vg, d_bst, d_kstart, B, d_out);
    ++h->launches;
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpyAsync(res.data(), d_out, sizeof(GcmCluster) * B, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
  }
  for (int b = 0; b < B; ++b) clusters_out[slot[b]] = res[b];
  return B200ORB_OK;
}

int gcm_add_keyframe_objects(gcm_t* h, const float* depth, const uint8_t* bgr, int rows, int cols, const float Tcw[16],
                             float fx, float fy, float cx, float cy, long long keyframe_index, const GcmObject* objs,
                             int n_objs, GcmCluster* clusters_out) {
  B200_CHECK(sem_check_args(h, depth, bgr, rows, cols, Tcw, keyframe_index, objs, n_objs, clusters_out));
  if (keyframe_index % 2 == 0 && n_objs == 0) return B200ORB_OK;   // :434: nothing to upload
  DeviceGuard g(h->device);
  const size_t npix = (size_t)rows * cols;
  float* d_depth;
  uint8_t* d_bgr;
  B200_CHECK(h->stage.reserve(h->stream, [&](Carver& t) { d_depth = t.take<float>(npix); d_bgr = t.take<uint8_t>(3 * npix); }));
  B200_CUDA(cudaMemcpyAsync(d_depth, depth, npix * 4, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(d_bgr, bgr, npix * 3, cudaMemcpyHostToDevice, h->stream));
  B200_CHECK(gcm_add_keyframe_objects_device(h, d_depth, d_bgr, rows, cols, Tcw, fx, fy, cx, cy, keyframe_index, objs, n_objs,
                                             clusters_out));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

}  // extern "C"
