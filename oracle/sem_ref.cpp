// oracle/sem_ref.cpp -- CPU restatement of the semantic object clusters of the T variant's mapping thread
// (src/pointcloudmapping.cc:399-488).  TEST INFRASTRUCTURE ONLY; built into oracle/libsem_oracle.so by oracle/sem.mk
// with the oracle's flags (-O3 -ffp-contract=off).
//
// UNPINNED to a reference binary: src/pointcloudmapping.cc needs PCL, VTK, boost and Eigen, none of which are here.  The
// reference's own expressions (draw_rect_with_depth_threshold :197-244, the gate :418, the skip :434, the colour table
// :47-60) are restated line by line; the three PCL 1.7 filters are restated from their definitions:
//   ExtractIndices           the points at the band indices, in band order, repeats included
//   StatisticalOutlierRemoval(mean_k 50, stddev_mul 1.0): for every point the 51 nearest neighbours (itself included) by
//                            FLANN's L2_Simple<float> ((0 + dx*dx) + dy*dy) + dz*dz, sorted ascending; distance =
//                            static_cast<float>(dist_sum / mean_k) with dist_sum = sum_{k=1..50} sqrt(nn_dists[k]) in
//                            double; sum += distance, sq_sum += distance * distance; mean = sum / n,
//                            variance = (sq_sum - sum * sum / n) / (n - 1), threshold = mean + 1.0 * sqrt(variance);
//                            a point stays iff !(distance > threshold)
//   VoxelGrid(resolution)    as occ_ref_global_refilter (occ_ref.cpp), xyz only; where the index space overflows int PCL
//                            hands the input back unfiltered
// The two lines below marked UNPINNED are the only readings of PCL internals that cannot be checked here; SEM_ALT_SQRT and
// SEM_ALT_SQSUM select the other reading of each (tests/test_semantic_cpu.py counts the keep decisions that flip).
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "../include/b200orb.h"

namespace {

enum { SEM_ALT_SQRT = 1, SEM_ALT_SQSUM = 2 };
constexpr int MEAN_K = 50;

// PointCloudMapping::PointCloudMapping (:50-60): colors_ as cv::Scalar(B, G, R) doubles
void make_colors(double c[21][3]) {
  for (int i = 0; i < 21; i++) c[i][0] = c[i][1] = c[i][2] = i * 10 + 40;
  const double special[4][4] = {{5, 255, 0, 255}, {9, 255, 0, 0}, {15, 0, 0, 255}, {20, 0, 255, 0}};
  for (const auto& s : special) for (int k = 0; k < 3; k++) c[(int)s[0]][k] = s[1 + k];
}

// draw_rect_with_depth_threshold (:197-244) with the reference's int / double conversions.  Deviation: flat indices
// outside [0, rows*cols) are skipped where the reference reads (and writes) out of bounds.
float band(const float* depth, unsigned char* color, int rows, int cols, const GcmObject& o, const double scalar[3],
           std::vector<int>& indices) {
  const long long npix = (long long)rows * cols;
  int beg = (int)o.x + ((int)o.y - 1) * cols - 1;                           // :206
  int count = 0;
  float sum = 0;
  for (int k = (int)o.height * 0.3; k < (int)o.height * 0.7; k++) {         // :211
    int start = beg + k * cols;
    int end = start + (int)o.width * 0.7;
    for (int j = start + (int)o.width * 0.3; j < end; j++) {                // :215
      if (j < 0 || j >= npix) continue;
      float d = depth[j];
      if (d < 0.5 || d > 6) continue;                                       // :218
      sum += d;
      count++;
    }
  }
  float depth_threshold = 0.0;
  if (count > 0) depth_threshold = sum / count;                             // :225
  for (int k = 0; k < (int)o.height - 1; k++) {                             // :228
    int start = beg + k * cols;
    int end = start + (int)o.width - 1;
    for (int j = start; j < end - 1; j++) {                                 // :232
      if (j < 0 || j >= npix) continue;
      if (std::abs(depth[j] - depth_threshold) < 0.4) {                     // :234, float abs, double compare
        indices.push_back(j);
        if (color) {
          color[j * 3 + 0] = scalar[0];
          color[j * 3 + 1] = scalar[1];
          color[j * 3 + 2] = scalar[2];
        }
      }
    }
  }
  return depth_threshold;
}

// generatePointCloud (:160-189): every pixel, Tcw^-1 applied in double (as occ_ref_backproject_all)
void cloud(const float* depth, const unsigned char* col, int rows, int cols, const float* Tcw, float fx, float fy, float cx,
           float cy, float* xyz, unsigned char* rgb) {
  double R[9], t[3], Rt[9], ti[3];
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) R[i * 3 + j] = (double)Tcw[i * 4 + j]; t[i] = (double)Tcw[i * 4 + 3]; }
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Rt[i * 3 + j] = R[j * 3 + i];
    ti[i] = -(R[0 * 3 + i] * t[0] + R[1 * 3 + i] * t[1] + R[2 * 3 + i] * t[2]);
  }
  for (int r = 0; r < rows; r++)
    for (int c = 0; c < cols; c++) {
      const size_t i = (size_t)r * cols + c;
      const float d = depth[i];
      const float xf = (c - cx) * d / fx, yf = (r - cy) * d / fy;
      const double px = xf, py = yf, pz = d;
      for (int k = 0; k < 3; ++k) xyz[3 * i + k] = (float)(Rt[k * 3 + 0] * px + Rt[k * 3 + 1] * py + Rt[k * 3 + 2] * pz + ti[k]);
      if (rgb) { rgb[3 * i] = col[i * 3 + 2]; rgb[3 * i + 1] = col[i * 3 + 1]; rgb[3 * i + 2] = col[i * 3 + 0]; }
    }
}

// brute force: for every point the k smallest squared distances to the n points (itself included), ascending
void knn(const float* p, int n, int k, float* out) {
  const int nt = std::max(1, std::min<int>(32, (int)std::thread::hardware_concurrency()));
  auto work = [&](int q0, int q1) {
    std::vector<float> d(n);
    for (int q = q0; q < q1; ++q) {
      for (int c = 0; c < n; ++c) {
        const float dx = p[3 * q] - p[3 * c], dy = p[3 * q + 1] - p[3 * c + 1], dz = p[3 * q + 2] - p[3 * c + 2];
        float r = 0;                                        // flann::L2_Simple<float>: result += diff * diff
        r += dx * dx;
        r += dy * dy;
        r += dz * dz;
        d[c] = r;
      }
      std::nth_element(d.begin(), d.begin() + (k - 1), d.end());
      std::sort(d.begin(), d.begin() + k);
      std::copy(d.begin(), d.begin() + k, out + (size_t)q * k);
    }
  };
  std::vector<std::thread> th;
  const int step = (n + nt - 1) / nt;
  for (int q0 = 0; q0 < n; q0 += step) th.emplace_back(work, q0, std::min(n, q0 + step));
  for (auto& t : th) t.join();
}

// StatisticalOutlierRemoval::applyFilterIndices, n >= mean_k + 1 finite points -> number kept
int sor(const float* p, int n, int reading, float* distances, unsigned char* keep) {
  std::vector<float> nn((size_t)n * (MEAN_K + 1));
  knn(p, n, MEAN_K + 1, nn.data());
  for (int i = 0; i < n; ++i) {
    const float* nn_dists = nn.data() + (size_t)i * (MEAN_K + 1);
    double dist_sum = 0.0;
    for (int k = 1; k < MEAN_K + 1; ++k)   // UNPINNED: sqrt of the float distance taken in double
      dist_sum += (reading & SEM_ALT_SQRT) ? (double)std::sqrt(nn_dists[k]) : std::sqrt((double)nn_dists[k]);
    distances[i] = static_cast<float>(dist_sum / MEAN_K);
  }
  double sum = 0, sq_sum = 0;
  for (int i = 0; i < n; ++i) {
    sum += distances[i];                   // UNPINNED: distances[i] * distances[i] multiplied in float
    sq_sum += (reading & SEM_ALT_SQSUM) ? (double)distances[i] * (double)distances[i] : (double)(distances[i] * distances[i]);
  }
  const double mean = sum / static_cast<double>(n);
  const double variance = (sq_sum - sum * sum / static_cast<double>(n)) / (static_cast<double>(n) - 1);
  const double stddev = std::sqrt(variance);
  const double distance_threshold = mean + 1.0 * stddev;
  int kept = 0;
  for (int i = 0; i < n; ++i) {
    keep[i] = !(distances[i] > distance_threshold);
    kept += keep[i];
  }
  return kept;
}

// VoxelGrid on an all-finite cloud (occ_ref_global_refilter, xyz only); the input itself where the index space overflows
std::vector<float> voxel(const std::vector<float>& p, float leaf) {
  const long long n = (long long)p.size() / 3;
  if (n == 0) return {};
  const float inv = 1.0f / leaf;
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (long long i = 0; i < n; ++i)
    for (int k = 0; k < 3; ++k) { mn[k] = std::min(mn[k], p[3 * i + k]); mx[k] = std::max(mx[k], p[3 * i + k]); }
  const long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1,
                  dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  if (dx * dy * dz > 2147483647LL) return p;
  int min_b[3], div_b[3];
  for (int k = 0; k < 3; ++k) {
    min_b[k] = (int)std::floor(mn[k] * inv);
    div_b[k] = (int)std::floor(mx[k] * inv) - min_b[k] + 1;
  }
  const int mul[3] = {1, div_b[0], div_b[0] * div_b[1]};
  std::vector<std::pair<int, long long>> iv;
  for (long long i = 0; i < n; ++i) {
    int idx = 0;
    for (int k = 0; k < 3; ++k) idx += (int)(std::floor(p[3 * i + k] * inv) - (float)min_b[k]) * mul[k];
    iv.emplace_back(idx, i);
  }
  std::stable_sort(iv.begin(), iv.end(), [](const std::pair<int, long long>& a, const std::pair<int, long long>& b) { return a.first < b.first; });
  std::vector<float> out;
  for (size_t b = 0; b < iv.size();) {
    size_t e = b;
    float s[3] = {0, 0, 0};
    for (; e < iv.size() && iv[e].first == iv[b].first; ++e)
      for (int k = 0; k < 3; ++k) s[k] += p[3 * iv[e].second + k];
    const float fn = (float)(e - b);
    for (int k = 0; k < 3; ++k) out.push_back(s[k] / fn);
    b = e;
  }
  return out;
}

// :451-476 for one box's band points: SOR -> VoxelGrid -> compute3DCentroid -> getMinMax3D
GcmCluster cluster(const float* band_xyz, int n, float leaf, int reading) {
  GcmCluster c = {};
  c.n_band = n;
  if (n < MEAN_K + 1) { c.status = GCM_FEW_POINTS; return c; }   // deviation: PCL reads past its neighbour list here
  c.status = GCM_CLUSTER;
  std::vector<float> dist(n);
  std::vector<unsigned char> keep(n);
  sor(band_xyz, n, reading, dist.data(), keep.data());
  std::vector<float> in;
  for (int i = 0; i < n; ++i)
    if (keep[i]) in.insert(in.end(), band_xyz + 3 * i, band_xyz + 3 * i + 3);
  c.n_inliers = (int)(in.size() / 3);
  const std::vector<float> v = voxel(in, leaf);
  c.n_voxels = (int)(v.size() / 3);
  float s[3] = {0, 0, 0}, mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int i = 0; i < c.n_voxels; ++i)
    for (int k = 0; k < 3; ++k) {
      s[k] += v[3 * i + k];
      mn[k] = std::min(mn[k], v[3 * i + k]);
      mx[k] = std::max(mx[k], v[3 * i + k]);
    }
  for (int k = 0; k < 3; ++k) {
    c.centroid[k] = s[k] / (float)c.n_voxels;
    c.min_pt[k] = mn[k];
    c.max_pt[k] = mx[k];
  }
  return c;
}

}  // namespace

extern "C" {

// one box's band (draw_rect_with_depth_threshold): paints `bgr` when given; -> number of indices (all written when
// <= cap), *thr = the mean depth
long long sem_ref_band(const float* depth, unsigned char* bgr, int rows, int cols, const GcmObject* obj, float* thr, int* idx,
                       long long cap) {
  double colors[21][3];
  make_colors(colors);
  std::vector<int> ind;
  *thr = band(depth, bgr, rows, cols, *obj, colors[obj->class_id], ind);
  std::copy(ind.begin(), ind.begin() + std::min<long long>(cap, (long long)ind.size()), idx);
  return (long long)ind.size();
}

void sem_ref_knn(const float* xyz, int n, int k, float* out) { knn(xyz, n, k, out); }

int sem_ref_sor(const float* xyz, int n, int reading, float* distances, unsigned char* keep) {
  return sor(xyz, n, reading, distances, keep);
}

void sem_ref_cluster(const float* xyz, int n, float leaf, int reading, GcmCluster* out) { *out = cluster(xyz, n, leaf, reading); }

// One keyframe of the loop body (:413-485).  `bgr` is painted in place; when the keyframe is not skipped the world cloud
// of the painted image is written to xyz / rgb (rows*cols points, pixel order, before removeNaNFromPointCloud).
// -> 1 when the keyframe adds its cloud, 0 when it is skipped (:434).
int sem_ref_keyframe(const float* depth, unsigned char* bgr, int rows, int cols, const float* Tcw, float fx, float fy, float cx,
                     float cy, long long i, const GcmObject* objects, int n_objs, float leaf, int reading, GcmCluster* out,
                     float* xyz, unsigned char* rgb) {
  double colors[21][3];
  make_colors(colors);
  std::vector<std::vector<int>> vec_indices;
  std::vector<int> slot;
  for (int t = 0; t < n_objs; t++) {
    const GcmObject& obj = objects[t];
    out[t] = GcmCluster{};
    out[t].status = GCM_BELOW_PROB;
    if (obj.prob > 0.54) {                                                  // :418
      std::vector<int> indices;
      band(depth, bgr, rows, cols, obj, colors[obj.class_id], indices);
      vec_indices.push_back(indices);
      slot.push_back(t);
    }
  }
  if ((i % 2 == 0) && (n_objs == 0)) return 0;                              // :434
  const size_t npix = (size_t)rows * cols;
  std::vector<float> p(3 * npix);
  cloud(depth, bgr, rows, cols, Tcw, fx, fy, cx, cy, p.data(), rgb);
  if (xyz) std::copy(p.begin(), p.end(), xyz);
  for (size_t n = 0; n < vec_indices.size(); n++) {
    const std::vector<int>& ind = vec_indices[n];
    std::vector<float> before;                                              // extract_indices.filter (:449-452)
    for (int j : ind) before.insert(before.end(), p.begin() + 3 * (size_t)j, p.begin() + 3 * (size_t)j + 3);
    out[slot[n]] = cluster(before.data(), (int)ind.size(), leaf, reading);
  }
  return 1;
}

}  // extern "C"
