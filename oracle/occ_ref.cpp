// oracle/occ_ref.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
//
// CPU restatement of the keyframe -> point cloud -> OctoMap occupancy path:
//   MapDrawer::GeneratePointCloud   perfect/src/MapDrawer.cc:641-675 (back-projection, gates, VoxelGrid 1 cm, transform)
//   MapDrawer::InsertScan           perfect/src/MapDrawer.cc:946-1025
//   MapDrawer ctor octree params    perfect/src/MapDrawer.cc:51-56
//   PointCloudMapping::generatePointCloud (T variant, all pixels, no gate)  src/pointcloudmapping.cc:131-194
// Third-party semantics restated from their published behaviour (NOT vendored; parity unpinned, SURVEY §8(c)):
//   PCL 1.7 VoxelGrid (SURVEY App. A.7), pcl::transformPointCloud<PointT,double>, octomap 1.9 OcTreeKey /
//   coordToKeyChecked / computeRayKeys / updateNode log-odds (SURVEY App. A.6).  The shipped artefact octomap.ot pins
//   the log-odds constants and clamps (tests/test_golden_cpu.py).
// Where PCL leaves an order unspecified (std::sort of equal voxel indices) the oracle sums a voxel's points in
// pixel row-major order; the RANSAC ground split is replaced by a supplied per-pixel label (voxel label = label of
// its first pixel).
#include <algorithm>
#include <atomic>
#include <thread>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <tuple>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../include/b200orb.h"

namespace {

struct OccMap {
  OcmParams p;
  double res, res_factor;
  float hit_log, miss_log, cmin, cmax;
  std::unordered_map<uint64_t, float> leaves;
  std::unordered_map<uint64_t, uint32_t> colors;
  // last scan
  std::vector<float> pts;
  std::vector<uint8_t> pts_rgb, pts_label;

  explicit OccMap(const OcmParams& q) : p(q) {
    res = q.resolution;
    res_factor = 1.0 / res;
    auto logodds = [](double pr) { return (float)std::log(pr / (1 - pr)); };   // octomap::logodds
    hit_log = logodds(q.prob_hit);
    miss_log = logodds(q.prob_miss);
    cmin = logodds(q.clamp_min);
    cmax = logodds(q.clamp_max);
  }
  static uint64_t pack(const uint16_t k[3]) { return (uint64_t)k[0] | ((uint64_t)k[1] << 16) | ((uint64_t)k[2] << 32); }
  // coordToKeyChecked, tree_max_val = 32768.  A non-finite coordinate never makes a key: octomap gets there on x86 only
  // through the undefined int conversion of NaN (INT_MIN); here the rule is explicit, and the range test is made before
  // the conversion.
  bool coord_to_key(double c, uint16_t& k) const {
    if (!std::isfinite(c)) return false;
    const double f = std::floor(res_factor * c);
    if (!(f >= -32768.0 && f < 32768.0)) return false;
    k = (uint16_t)((int)f + 32768);
    return true;
  }
  bool point_to_key(const float* pt, uint16_t k[3]) const {
    return coord_to_key((double)pt[0], k[0]) && coord_to_key((double)pt[1], k[1]) && coord_to_key((double)pt[2], k[2]);
  }
  double key_to_coord(uint16_t k) const { return (double((int)k - 32768) + 0.5) * res; }

  // OcTreeBaseImpl::computeRayKeys (end cell excluded)
  bool ray_keys(const float* o, const float* e, std::vector<uint64_t>& ray) const {
    ray.clear();
    uint16_t ko[3], ke[3];
    if (!point_to_key(o, ko) || !point_to_key(e, ke)) return false;
    if (ko[0] == ke[0] && ko[1] == ke[1] && ko[2] == ke[2]) return true;
    ray.push_back(pack(ko));
    float dir[3] = {e[0] - o[0], e[1] - o[1], e[2] - o[2]};
    // octomath::Vector3::norm() of octomap 1.9.x: sqrt(norm_sq()) with norm_sq() = x*x + y*y + z*z evaluated in FLOAT
    // (the components are floats), widened to double only for the sqrt; 1.6-1.8 summed the float products in a double
    const float n2 = dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2];
    const float length = (float)std::sqrt((double)n2);
    for (int i = 0; i < 3; ++i) dir[i] /= length;
    int step[3];
    double tMax[3], tDelta[3];
    uint16_t cur[3] = {ko[0], ko[1], ko[2]};
    for (int i = 0; i < 3; ++i) {
      if (dir[i] > 0.0) step[i] = 1;
      else if (dir[i] < 0.0) step[i] = -1;
      else step[i] = 0;
      if (step[i] != 0) {
        double voxelBorder = key_to_coord(cur[i]);
        voxelBorder += (float)(step[i] * res * 0.5);
        tMax[i] = (voxelBorder - o[i]) / dir[i];
        tDelta[i] = res / std::fabs(dir[i]);
      } else {
        tMax[i] = 1.7976931348623157e308;
        tDelta[i] = 1.7976931348623157e308;
      }
    }
    for (;;) {
      unsigned dim;
      if (tMax[0] < tMax[1]) dim = (tMax[0] < tMax[2]) ? 0 : 2;
      else dim = (tMax[1] < tMax[2]) ? 1 : 2;
      cur[dim] = (uint16_t)(cur[dim] + step[dim]);
      tMax[dim] += tDelta[dim];
      if (cur[0] == ke[0] && cur[1] == ke[1] && cur[2] == ke[2]) break;
      const double dist = std::min(std::min(tMax[0], tMax[1]), tMax[2]);
      if (dist > length) break;
      ray.push_back(pack(cur));
    }
    return true;
  }

  void update(uint64_t key, bool occupied) {   // OccupancyOcTreeBase::updateNode -> updateNodeLogOdds
    const float d = occupied ? hit_log : miss_log;
    auto it = leaves.find(key);
    if (it == leaves.end()) it = leaves.emplace(key, 0.0f).first;
    float v = it->second + d;
    if (v < cmin) v = cmin;
    if (v > cmax) v = cmax;
    it->second = v;
  }

  // MapDrawer::GeneratePointCloud: gates + VoxelGrid + transform; fills pts/pts_rgb/pts_label
  void generate(const float* depth, const uint8_t* rgb, int rows, int cols, const float* Tcw, float fx, float fy,
                float cx, float cy, const uint8_t* label) {
    struct Acc { float sx = 0, sy = 0, sz = 0, sr = 0, sg = 0, sb = 0; int n = 0; uint8_t label = 0; };
    std::map<std::tuple<int, int, int>, Acc> vox;   // ordered by (iz, iy, ix): PCL's ascending linear index
    // NaN depth passes both gates (:655); those pixels form one cell of their own (emitted last) rather than one whose
    // index comes from an undefined int conversion.  Its centroid is NaN, so it never makes an octree key.
    Acc nonfinite;
    std::vector<float> raw;
    std::vector<uint8_t> raw_rgb, raw_label;
    const bool filter = p.leaf > 0;
    const float inv_leaf = filter ? 1.0f / p.leaf : 0.f;
    for (int m = 0; m < rows; ++m)
      for (int n = 0; n < cols; ++n) {
        const float d = depth[(size_t)m * cols + n];
        if (d < p.depth_min || d > p.depth_max) continue;            // :655
        const float z = d;
        const float x = (n - cx) * z / fx;                          // :658-659
        const float y = (m - cy) * z / fy;
        if (y < -p.y_max || y > p.y_max) continue;                  // :660
        const uint8_t* c = rgb + ((size_t)m * cols + n) * 3;        // b,g,r
        const uint8_t lab = label ? label[(size_t)m * cols + n] : 0;
        if (!filter) {
          raw.push_back(x); raw.push_back(y); raw.push_back(z);
          raw_rgb.push_back(c[2]); raw_rgb.push_back(c[1]); raw_rgb.push_back(c[0]);
          raw_label.push_back(lab);
          continue;
        }
        const bool finite = std::isfinite(x) && std::isfinite(y) && std::isfinite(z);
        const int ix = finite ? (int)std::floor(x * inv_leaf) : 0, iy = finite ? (int)std::floor(y * inv_leaf) : 0,
                  iz = finite ? (int)std::floor(z * inv_leaf) : 0;
        Acc& a = finite ? vox[std::make_tuple(iz, iy, ix)] : nonfinite;
        if (a.n == 0) a.label = lab;
        a.sx += x; a.sy += y; a.sz += z;
        a.sr += (float)c[2]; a.sg += (float)c[1]; a.sb += (float)c[0];
        a.n++;
      }
    if (filter) {
      if (nonfinite.n) vox.emplace(std::make_tuple(INT_MAX, INT_MAX, INT_MAX), nonfinite);   // sorts last
      for (auto& kv : vox) {
        const Acc& a = kv.second;
        const float fn = (float)a.n;
        raw.push_back(a.sx / fn); raw.push_back(a.sy / fn); raw.push_back(a.sz / fn);
        raw_rgb.push_back((uint8_t)(a.sr / fn)); raw_rgb.push_back((uint8_t)(a.sg / fn)); raw_rgb.push_back((uint8_t)(a.sb / fn));
        raw_label.push_back(a.label);
      }
    }
    // pcl::transformPointCloud(cloud, temp, T.inverse().matrix()) with T = toSE3Quat(Tcw) (double)
    double R[9], t[3], Rt[9], ti[3];
    for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) R[i * 3 + j] = (double)Tcw[i * 4 + j]; t[i] = (double)Tcw[i * 4 + 3]; }
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) Rt[i * 3 + j] = R[j * 3 + i];
      ti[i] = -(R[0 * 3 + i] * t[0] + R[1 * 3 + i] * t[1] + R[2 * 3 + i] * t[2]);
    }
    const size_t np = raw.size() / 3;
    pts.resize(np * 3);
    for (size_t k = 0; k < np; ++k) {
      const double px = raw[3 * k], py = raw[3 * k + 1], pz = raw[3 * k + 2];
      for (int i = 0; i < 3; ++i)
        pts[3 * k + i] = (float)(Rt[i * 3 + 0] * px + Rt[i * 3 + 1] * py + Rt[i * 3 + 2] * pz + ti[i]);
    }
    pts_rgb = raw_rgb;
    pts_label = raw_label;
    // perfect/src/MapDrawer.cc:676-680: "if(temp.size()<50) ground = temp" -- a cloud of fewer than 50 points skips the
    // plane extraction and is ALL ground (free rays only, no occupied endpoints), whatever a label would say
    if (np < 50) std::fill(pts_label.begin(), pts_label.end(), (uint8_t)1);
  }

  // MapDrawer::InsertScan :946-1025 (+ UpdateOctomap's sensorOrigin quirk :619,631-632: translation of Tcw)
  void insert_scan(const float* Tcw) {
    const float origin[3] = {Tcw[3], Tcw[7], Tcw[11]};
    std::unordered_set<uint64_t> free_cells, occupied;
    std::vector<uint64_t> ray;
    const size_t np = pts.size() / 3;
    for (size_t k = 0; k < np; ++k) {
      const float* pt = &pts[3 * k];
      if (pts_label[k]) {            // ground: only clears space along the ray
        if (ray_keys(origin, pt, ray)) free_cells.insert(ray.begin(), ray.end());
      } else {                       // non-ground: endpoint occupied (its ray is computed but unused, :988-991)
        uint16_t key[3];
        if (point_to_key(pt, key)) {
          occupied.insert(pack(key));
          colors[pack(key)] = (uint32_t)pts_rgb[3 * k] | ((uint32_t)pts_rgb[3 * k + 1] << 8) | ((uint32_t)pts_rgb[3 * k + 2] << 16);
        }
      }
    }
    for (uint64_t k : free_cells)
      if (occupied.find(k) == occupied.end()) update(k, false);
    for (uint64_t k : occupied) update(k, true);
  }
};

}  // namespace

extern "C" {

void occ_ref_default_params(OcmParams* p) {
  p->resolution = 0.05; p->prob_hit = 0.7; p->prob_miss = 0.4; p->clamp_min = 0.12; p->clamp_max = 0.97;
  p->depth_min = 0.5f; p->depth_max = 3.0f; p->y_max = 3.0f; p->leaf = 0.01f; p->map_capacity = 0;
}
void* occ_ref_create(const OcmParams* p) { return new OccMap(*p); }
void occ_ref_destroy(void* h) { delete (OccMap*)h; }
void occ_ref_constants(void* h, float* out4) {
  OccMap* m = (OccMap*)h;
  out4[0] = m->hit_log; out4[1] = m->miss_log; out4[2] = m->cmin; out4[3] = m->cmax;
}
int occ_ref_insert_keyframe(void* h, const float* depth, const uint8_t* rgb, int rows, int cols, const float* Tcw,
                            float fx, float fy, float cx, float cy, const uint8_t* label) {
  OccMap* m = (OccMap*)h;
  m->generate(depth, rgb, rows, cols, Tcw, fx, fy, cx, cy, label);
  m->insert_scan(Tcw);
  return (int)(m->pts.size() / 3);
}
// Baseline driver for a batch of keyframes: GeneratePointCloud (back-projection + VoxelGrid + transform) of the keyframes
// runs on `nthreads` host threads -- keyframes are independent up to that point, and the reference parallelises its own
// back-projection loop with OpenMP (src/pointcloudmapping.cc:169) -- while InsertScan into the one shared tree stays
// sequential in keyframe order, as it has to.  label may be NULL; label_stride = pixels between label images.
int occ_ref_insert_keyframes_mt(void* h, const float* depth, const uint8_t* rgb, const uint8_t* label, int rows, int cols,
                                const int* idx, int n, const float* Tcw, float fx, float fy, float cx, float cy, int nthreads) {
  OccMap* m = (OccMap*)h;
  const size_t px = (size_t)rows * cols;
  std::vector<OccMap*> parts(n, nullptr);
  std::atomic<int> next(0);
  std::vector<std::thread> th;
  for (int t = 0; t < std::max(1, std::min(nthreads, n)); ++t)
    th.emplace_back([&]() {
      for (int i = next++; i < n; i = next++) {
        OccMap* q = new OccMap(m->p);
        q->generate(depth + px * idx[i], rgb + px * 3 * idx[i], rows, cols, Tcw + 16 * i, fx, fy, cx, cy,
                    label ? label + px * idx[i] : nullptr);
        parts[i] = q;
      }
    });
  for (auto& t : th) t.join();
  for (int i = 0; i < n; ++i) {
    m->pts.swap(parts[i]->pts); m->pts_rgb.swap(parts[i]->pts_rgb); m->pts_label.swap(parts[i]->pts_label);
    m->insert_scan(Tcw + 16 * i);
    delete parts[i];
  }
  return n;
}
int occ_ref_last_points(void* h, float* xyz, uint8_t* rgb, uint8_t* label, int cap) {
  OccMap* m = (OccMap*)h;
  const int n = (int)(m->pts.size() / 3);
  if (n > cap) return -n;
  memcpy(xyz, m->pts.data(), sizeof(float) * 3 * n);
  if (rgb) memcpy(rgb, m->pts_rgb.data(), 3 * (size_t)n);
  if (label) memcpy(label, m->pts_label.data(), (size_t)n);
  return n;
}
long long occ_ref_num_leaves(void* h) { return (long long)((OccMap*)h)->leaves.size(); }
long long occ_ref_export_leaves(void* h, uint16_t* keys, float* logodds, long long cap) {
  OccMap* m = (OccMap*)h;
  long long n = 0;
  for (auto& kv : m->leaves) {
    if (n >= cap) break;
    keys[3 * n] = (uint16_t)(kv.first & 0xffff);
    keys[3 * n + 1] = (uint16_t)((kv.first >> 16) & 0xffff);
    keys[3 * n + 2] = (uint16_t)((kv.first >> 32) & 0xffff);
    logodds[n] = kv.second;
    ++n;
  }
  return n;
}
// ray keys of a single (origin, end) pair for direct DDA tests; returns count or -1 (out of range)
int occ_ref_ray(void* h, const float* origin, const float* end, uint16_t* keys, int cap) {
  OccMap* m = (OccMap*)h;
  std::vector<uint64_t> ray;
  if (!m->ray_keys(origin, end, ray)) return -1;
  int n = 0;
  for (uint64_t k : ray) {
    if (n < cap) { keys[3 * n] = (uint16_t)(k & 0xffff); keys[3 * n + 1] = (uint16_t)((k >> 16) & 0xffff); keys[3 * n + 2] = (uint16_t)((k >> 32) & 0xffff); }
    ++n;
  }
  return n;
}
// T variant (src/pointcloudmapping.cc:131-194): every pixel, no gate, d=0 -> camera centre.  out: rows*cols*3 floats
void occ_ref_backproject_all(const float* depth, int rows, int cols, const float* Tcw, float fx, float fy, float cx,
                             float cy, float* out) {
  double R[9], t[3], Rt[9], ti[3];
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) R[i * 3 + j] = (double)Tcw[i * 4 + j]; t[i] = (double)Tcw[i * 4 + 3]; }
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Rt[i * 3 + j] = R[j * 3 + i];
    ti[i] = -(R[0 * 3 + i] * t[0] + R[1 * 3 + i] * t[1] + R[2 * 3 + i] * t[2]);
  }
  for (int r = 0; r < rows; ++r)
    for (int c = 0; c < cols; ++c) {
      const size_t i = (size_t)r * cols + c;
      const float d = depth[i];
      const float xf = (c - cx) * d / fx, yf = (r - cy) * d / fy;   // float, like the reference (:174-176)
      const double px = xf, py = yf, pz = d;
      for (int k = 0; k < 3; ++k) out[3 * i + k] = (float)(Rt[k * 3 + 0] * px + Rt[k * 3 + 1] * py + Rt[k * 3 + 2] * pz + ti[k]);
    }
}

// T variant, global map refilter (src/pointcloudmapping.cc:485-493): globalMap += cloud (NaN points removed, order kept),
// then pcl::VoxelGrid(leaf = resolution) over the whole accumulated cloud, globalMap.swap(filtered).
// PCL VoxelGrid<PointXYZRGBA>::applyFilter restated (SURVEY App. A.7): bounding box of the finite points, min_b/div_b from
// floor(min*inv_leaf), linear cell index per point, sort by index, per cell the centroid of x,y,z (float sums in sorted
// order, divided by the count as float) and of r,g,b (float sums, truncated), cells emitted in ascending index order.
// std::sort leaves the order of equal indices open: the oracle keeps the input order (stable), like the P variant.
// in: n points (non-finite ones are skipped like removeNaNFromPointCloud / the !is_dense branch do); returns the number of
// output points, -1 if the index space overflows int (PCL warns and returns the input unfiltered), -2 if cap is too small.
long long occ_ref_global_refilter(const float* xyz, const uint8_t* rgb, long long n, float leaf, float* out_xyz,
                                  uint8_t* out_rgb, long long cap) {
  const float inv = 1.0f / leaf;
  float mn[3] = {3.4028235e38f, 3.4028235e38f, 3.4028235e38f}, mx[3] = {-3.4028235e38f, -3.4028235e38f, -3.4028235e38f};
  long long nf = 0;
  for (long long i = 0; i < n; ++i) {
    const float* p = xyz + 3 * i;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    for (int k = 0; k < 3; ++k) { mn[k] = std::min(mn[k], p[k]); mx[k] = std::max(mx[k], p[k]); }
    ++nf;
  }
  if (nf == 0) return 0;
  const long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1,
                  dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  if (dx * dy * dz > 2147483647LL) return -1;
  int min_b[3], max_b[3], div_b[3];
  for (int k = 0; k < 3; ++k) {
    min_b[k] = (int)std::floor(mn[k] * inv);
    max_b[k] = (int)std::floor(mx[k] * inv);
    div_b[k] = max_b[k] - min_b[k] + 1;
  }
  const int mul[3] = {1, div_b[0], div_b[0] * div_b[1]};
  std::vector<std::pair<int, long long>> iv;
  iv.reserve((size_t)nf);
  for (long long i = 0; i < n; ++i) {
    const float* p = xyz + 3 * i;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    const int i0 = (int)(std::floor(p[0] * inv) - (float)min_b[0]);
    const int i1 = (int)(std::floor(p[1] * inv) - (float)min_b[1]);
    const int i2 = (int)(std::floor(p[2] * inv) - (float)min_b[2]);
    iv.emplace_back(i0 * mul[0] + i1 * mul[1] + i2 * mul[2], i);
  }
  std::stable_sort(iv.begin(), iv.end(), [](const std::pair<int, long long>& a, const std::pair<int, long long>& b) { return a.first < b.first; });
  long long m = 0;
  for (size_t b = 0; b < iv.size();) {
    size_t e = b;
    float sx = 0, sy = 0, sz = 0, sr = 0, sg = 0, sb = 0;
    while (e < iv.size() && iv[e].first == iv[b].first) {
      const long long i = iv[e].second;
      sx += xyz[3 * i]; sy += xyz[3 * i + 1]; sz += xyz[3 * i + 2];
      sr += (float)rgb[3 * i]; sg += (float)rgb[3 * i + 1]; sb += (float)rgb[3 * i + 2];
      ++e;
    }
    if (m >= cap) return -2;
    const float fn = (float)(e - b);
    out_xyz[3 * m] = sx / fn; out_xyz[3 * m + 1] = sy / fn; out_xyz[3 * m + 2] = sz / fn;
    out_rgb[3 * m] = (uint8_t)(sr / fn); out_rgb[3 * m + 1] = (uint8_t)(sg / fn); out_rgb[3 * m + 2] = (uint8_t)(sb / fn);
    ++m;
    b = e;
  }
  return m;
}

}  // extern "C"
