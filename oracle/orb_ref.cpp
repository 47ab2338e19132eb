// oracle/orb_ref.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
//
// CPU restatement of the reference's ORB extractor (src/ORBextractor.cc) with the un-vendored
// OpenCV primitives replaced by the integer models of SURVEY.md Appendix A.  Only tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this.
//
// Parity status: the reference cannot be compiled here (no OpenCV C++/Eigen/PCL/octomap, SURVEY F6)
// and ships no golden vectors for this path (SURVEY §4).  The primitives below are pinned bit-exactly
// against cv2 4.13.0 (tests/test_oracle_cv2.py + oracle/orb_cv2.py) -- the whole extractor against a
// cv2-based line-by-line Python restatement; the reference's own output depends on the OpenCV version
// it is linked to (SURVEY F5), so relative to "the reference binary" parity is unpinned.
//
// Build: g++ -O3 -march=native -ffp-contract=off -std=c++17 -shared -fPIC   (see oracle/Makefile)
// -ffp-contract=off: the reference T build compiles C++ for baseline x86-64 (src/CMakeLists.txt:19),
// so float a*b+c is never fused (SURVEY H2).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <list>
#include <vector>

#include "../include/glibc_sincosf.h"

namespace {

static const signed char kPattern[1024] = {
#include "../include/orb_pattern_31.inc"
};

const int PATCH_SIZE = 31;        // src/ORBextractor.cc:52
const int HALF_PATCH_SIZE = 15;   // :53
const int EDGE_THRESHOLD = 19;    // :54


struct KeyPoint {  // cv::KeyPoint layout, 28 bytes
  float x, y, size, angle, response;
  int octave, class_id;
};

struct Plane {
  int w = 0, h = 0, stride = 0;
  std::vector<uint8_t> d;
  void alloc(int w_, int h_) { w = w_; h = h_; stride = w_; d.assign((size_t)w_ * h_, 0); }
  uint8_t* row(int y) { return d.data() + (size_t)y * stride; }
  const uint8_t* row(int y) const { return d.data() + (size_t)y * stride; }
};

}  // namespace
#include "standin/cv_prims.hpp"
namespace {
using namespace cvprim;

// ---------------------------------------------------------------------------------------------
// Extractor (src/ORBextractor.cc:399-466 ctor, :1052-1145 operator()/ComputePyramid)
// ---------------------------------------------------------------------------------------------
struct Node {  // ExtractorNode, include/ORBextractor.h (UL/UR/BL/BR + vKeys + bNoMore)
  int ULx, ULy, URx, URy, BLx, BLy, BRx, BRy;
  std::vector<KeyPoint> keys;
  bool noMore = false;
  long seq = 0;  // creation sequence number: surrogate for the heap address used by sort() at :686
  std::list<Node>::iterator lit;
};

struct Extractor {
  int nfeatures;
  double scaleFactor;  // include/ORBextractor.h: member is double, ctor arg float
  int nlevels, iniTh, minTh;
  std::vector<float> sf, sigma2, invsf, invsigma2;
  std::vector<int> nfeat;
  int umax[HALF_PATCH_SIZE + 1];
  std::vector<Plane> pyr;      // bordered level buffers (w+38)x(h+38); level image is the ROI at (19,19)
  std::vector<int> lw, lh;
  std::vector<std::vector<KeyPoint>> cand;   // per level: vToDistributeKeys of the last extract (:788-843)
  long seq_counter = 0;

  Extractor(int nf, float sfac, int nl, int ini, int mn)
      : nfeatures(nf), scaleFactor(sfac), nlevels(nl), iniTh(ini), minTh(mn) {
    sf.resize(nl); sigma2.resize(nl); invsf.resize(nl); invsigma2.resize(nl); nfeat.resize(nl);
    sf[0] = 1.0f; sigma2[0] = 1.0f;
    for (int i = 1; i < nl; ++i) {
      sf[i] = (float)(sf[i - 1] * scaleFactor);   // :411 float*double -> float
      sigma2[i] = sf[i] * sf[i];
    }
    for (int i = 0; i < nl; ++i) { invsf[i] = 1.0f / sf[i]; invsigma2[i] = 1.0f / sigma2[i]; }
    float factor = (float)(1.0f / scaleFactor);    // :426
    float nDesired = nfeatures * (1 - factor) / (1 - (float)std::pow((double)factor, (double)nlevels));
    int sum = 0;
    for (int l = 0; l < nl - 1; ++l) {
      nfeat[l] = cvRoundf(nDesired);
      sum += nfeat[l];
      nDesired *= factor;
    }
    nfeat[nl - 1] = std::max(nfeatures - sum, 0);
    // umax (:449-465)
    int v, v0, vmax = (int)std::floor(HALF_PATCH_SIZE * std::sqrt(2.f) / 2 + 1);
    int vmin = (int)std::ceil(HALF_PATCH_SIZE * std::sqrt(2.f) / 2);
    const double hp2 = HALF_PATCH_SIZE * HALF_PATCH_SIZE;
    for (v = 0; v <= vmax; ++v) umax[v] = cvRoundd(std::sqrt(hp2 - v * v));
    for (v = HALF_PATCH_SIZE, v0 = 0; v >= vmin; --v) {
      while (umax[v0] == umax[v0 + 1]) ++v0;
      umax[v] = v0;
      ++v0;
    }
    pyr.resize(nl); lw.resize(nl); lh.resize(nl); cand.resize(nl);
  }

  uint8_t* lvl(int l, int y) { return pyr[l].row(y + EDGE_THRESHOLD) + EDGE_THRESHOLD; }

  void make_border(int l) {  // copyMakeBorder(BORDER_REFLECT_101), :1136-1142
    Plane& P = pyr[l];
    int w = lw[l], h = lh[l], B = EDGE_THRESHOLD;
    for (int y = 0; y < h + 2 * B; ++y) {
      int sy = reflect101(y - B, h);
      uint8_t* drow = P.row(y);
      const uint8_t* srow = P.row(sy + B) + B;
      if (y < B || y >= h + B) memcpy(drow + B, srow, w);
      for (int x = 0; x < B; ++x) drow[x] = srow[reflect101(x - B, w)];
      for (int x = w + B; x < w + 2 * B; ++x) drow[x] = srow[reflect101(x - B, w)];
    }
  }

  void compute_pyramid(const uint8_t* img, int rows, int cols, int stride) {  // :1117-1145
    for (int l = 0; l < nlevels; ++l) {
      float scale = invsf[l];
      lw[l] = cvRoundf((float)cols * scale);
      lh[l] = cvRoundf((float)rows * scale);
      pyr[l].alloc(lw[l] + 2 * EDGE_THRESHOLD, lh[l] + 2 * EDGE_THRESHOLD);
      if (l == 0) {
        for (int y = 0; y < rows; ++y) memcpy(lvl(0, y), img + (size_t)y * stride, cols);
      } else {
        resize_linear_u8(lvl(l - 1, 0), lw[l - 1], lh[l - 1], pyr[l - 1].stride, lvl(l, 0), lw[l], lh[l],
                         pyr[l].stride);
      }
      make_border(l);
    }
  }

  // ExtractorNode::DivideNode :478-534
  static void divide(const Node& p, Node& n1, Node& n2, Node& n3, Node& n4) {
    const int halfX = (int)std::ceil(static_cast<float>(p.URx - p.ULx) / 2);
    const int halfY = (int)std::ceil(static_cast<float>(p.BRy - p.ULy) / 2);
    n1.ULx = p.ULx; n1.ULy = p.ULy;
    n1.URx = p.ULx + halfX; n1.URy = p.ULy;
    n1.BLx = p.ULx; n1.BLy = p.ULy + halfY;
    n1.BRx = p.ULx + halfX; n1.BRy = p.ULy + halfY;
    n2.ULx = n1.URx; n2.ULy = n1.URy;
    n2.URx = p.URx; n2.URy = p.URy;
    n2.BLx = n1.BRx; n2.BLy = n1.BRy;
    n2.BRx = p.URx; n2.BRy = p.ULy + halfY;
    n3.ULx = n1.BLx; n3.ULy = n1.BLy;
    n3.URx = n1.BRx; n3.URy = n1.BRy;
    n3.BLx = p.BLx; n3.BLy = p.BLy;
    n3.BRx = n1.BRx; n3.BRy = p.BLy;
    n4.ULx = n3.URx; n4.ULy = n3.URy;
    n4.URx = n2.BRx; n4.URy = n2.BRy;
    n4.BLx = n3.BRx; n4.BLy = n3.BRy;
    n4.BRx = p.BRx; n4.BRy = p.BRy;
    for (const KeyPoint& kp : p.keys) {
      if (kp.x < n1.URx) {
        if (kp.y < n1.BRy) n1.keys.push_back(kp);
        else n3.keys.push_back(kp);
      } else if (kp.y < n1.BRy) n2.keys.push_back(kp);
      else n4.keys.push_back(kp);
    }
    if (n1.keys.size() == 1) n1.noMore = true;
    if (n2.keys.size() == 1) n2.noMore = true;
    if (n3.keys.size() == 1) n3.noMore = true;
    if (n4.keys.size() == 1) n4.noMore = true;
  }

  struct SizeSeq {
    int size; long seq; Node* node;
    bool operator<(const SizeSeq& o) const { return size != o.size ? size < o.size : seq < o.seq; }
  };

  // DistributeOctTree :540-765.  Returns -1 if the reference would divide by zero (nIni == 0).  With `trace`, appends
  // one record of TRACE_INTS ints per round (see orb_ref_distribute); the result does not depend on it.
  static const int TRACE_INTS = 5;
  int distribute(const std::vector<KeyPoint>& in, int minX, int maxX, int minY, int maxY, int N,
                 std::vector<KeyPoint>& out, std::vector<int>* trace = nullptr) {
    out.clear();
    const int nIni = (int)std::round(static_cast<float>(maxX - minX) / (maxY - minY));
    if (nIni <= 0) return -1;
    const float hX = static_cast<float>(maxX - minX) / nIni;
    std::list<Node> nodes;
    std::vector<Node*> ini(nIni);
    for (int i = 0; i < nIni; ++i) {
      Node ni;
      ni.ULx = (int)(hX * static_cast<float>(i)); ni.ULy = 0;
      ni.URx = (int)(hX * static_cast<float>(i + 1)); ni.URy = 0;
      ni.BLx = ni.ULx; ni.BLy = maxY - minY;
      ni.BRx = ni.URx; ni.BRy = maxY - minY;
      ni.seq = seq_counter++;
      nodes.push_back(ni);
      ini[i] = &nodes.back();
    }
    for (const KeyPoint& kp : in) {
      int idx = (int)(kp.x / hX);
      if (idx >= nIni) idx = nIni - 1;  // (reference would index out of bounds; cannot happen for x < maxX-minX)
      ini[idx]->keys.push_back(kp);
    }
    for (auto lit = nodes.begin(); lit != nodes.end();) {
      if (lit->keys.size() == 1) { lit->noMore = true; ++lit; }
      else if (lit->keys.empty()) lit = nodes.erase(lit);
      else ++lit;
    }
    bool finish = false;
    std::vector<SizeSeq> vss;
    auto record = [&](int kind, int before, int count, int splits) {
      if (trace) trace->insert(trace->end(), {kind, before, (int)nodes.size(), count, splits});
    };
    auto push_child = [&](Node& n, std::vector<SizeSeq>& v, int* nToExpand) {
      if (n.keys.size() > 0) {
        n.seq = seq_counter++;
        nodes.push_front(n);
        if (n.keys.size() > 1) {
          if (nToExpand) ++*nToExpand;
          v.push_back({(int)n.keys.size(), nodes.front().seq, &nodes.front()});
          nodes.front().lit = nodes.begin();
        }
      }
    };
    while (!finish) {
      int prevSize = (int)nodes.size();
      auto lit = nodes.begin();
      int nToExpand = 0, splits = 0;
      vss.clear();
      while (lit != nodes.end()) {
        if (lit->noMore) { ++lit; continue; }
        Node n1, n2, n3, n4;
        divide(*lit, n1, n2, n3, n4);
        push_child(n1, vss, &nToExpand);
        push_child(n2, vss, &nToExpand);
        push_child(n3, vss, &nToExpand);
        push_child(n4, vss, &nToExpand);
        lit = nodes.erase(lit);
        ++splits;
      }
      record(0, prevSize, nToExpand, splits);
      if ((int)nodes.size() >= N || (int)nodes.size() == prevSize) {
        finish = true;
      } else if (((int)nodes.size() + nToExpand * 3) > N) {
        while (!finish) {
          prevSize = (int)nodes.size();
          std::vector<SizeSeq> prev = vss;
          vss.clear();
          std::sort(prev.begin(), prev.end());   // :686 (size, address) -> (size, creation seq)
          int divided = 0;
          for (int j = (int)prev.size() - 1; j >= 0; --j) {
            Node n1, n2, n3, n4;
            divide(*prev[j].node, n1, n2, n3, n4);
            push_child(n1, vss, nullptr);
            push_child(n2, vss, nullptr);
            push_child(n3, vss, nullptr);
            push_child(n4, vss, nullptr);
            nodes.erase(prev[j].node->lit);
            ++divided;
            if ((int)nodes.size() >= N) break;
          }
          record(1, prevSize, (int)prev.size(), divided);
          if ((int)nodes.size() >= N || (int)nodes.size() == prevSize) finish = true;
        }
      }
    }
    for (auto& n : nodes) {   // :746-762 first key with maximal response
      const KeyPoint* best = &n.keys[0];
      float maxR = best->response;
      for (size_t k = 1; k < n.keys.size(); ++k)
        if (n.keys[k].response > maxR) { best = &n.keys[k]; maxR = n.keys[k].response; }
      out.push_back(*best);
    }
    return 0;
  }

  // IC_Angle :59-88 on the un-blurred bordered level
  float ic_angle(int l, float ptx, float pty) {
    int m01 = 0, m10 = 0;
    const int step = pyr[l].stride;
    const uint8_t* center = lvl(l, cvRoundf(pty)) + cvRoundf(ptx);
    for (int u = -HALF_PATCH_SIZE; u <= HALF_PATCH_SIZE; ++u) m10 += u * center[u];
    for (int v = 1; v <= HALF_PATCH_SIZE; ++v) {
      int vsum = 0, d = umax[v];
      for (int u = -d; u <= d; ++u) {
        int vp = center[u + v * step], vm = center[u - v * step];
        vsum += (vp - vm);
        m10 += u * (vp + vm);
      }
      m01 += v * vsum;
    }
    return fast_atan2_deg((float)m01, (float)m10);
  }

  // computeOrbDescriptor :92-131 on the blurred (unbordered) level
  static void descriptor(const KeyPoint& kp, const uint8_t* img, int step, uint8_t* desc) {
    const float factorPI = (float)(3.14159265358979323846 / 180.f);
    float angle = kp.angle * factorPI;
    float a = cosf(angle), b = sinf(angle);
    const uint8_t* center = img + (size_t)cvRoundf(kp.y) * step + cvRoundf(kp.x);
    const signed char* pat = kPattern;
    auto get = [&](int idx) -> int {
      float px = (float)pat[2 * idx], py = (float)pat[2 * idx + 1];
      int yy = cvRoundf(px * b + py * a);
      int xx = cvRoundf(px * a - py * b);
      return center[yy * step + xx];
    };
    for (int i = 0; i < 32; ++i, pat += 32) {
      int val = 0;
      for (int k = 0; k < 8; ++k) {
        int t0 = get(2 * k), t1 = get(2 * k + 1);
        val |= (t0 < t1) << k;
      }
      desc[i] = (uint8_t)val;
    }
  }

  // ComputeKeyPointsOctTree :771-862 (per level), returns per-level FAST candidate count via cand[]
  int keypoints_level(int level, std::vector<KeyPoint>& keypoints, int* ncand) {
    const float W = 30;
    const int minBorderX = EDGE_THRESHOLD - 3, minBorderY = minBorderX;
    const int maxBorderX = lw[level] - EDGE_THRESHOLD + 3;
    const int maxBorderY = lh[level] - EDGE_THRESHOLD + 3;
    const float width = (float)(maxBorderX - minBorderX), height = (float)(maxBorderY - minBorderY);
    std::vector<KeyPoint>& toDist = cand[level];
    toDist.clear();
    keypoints.clear();
    if (ncand) *ncand = 0;
    if (width <= 0 || height <= 0) return 0;
    const int nCols = (int)(width / W), nRows = (int)(height / W);
    if (nCols <= 0 || nRows <= 0) return 0;   // reference divides by zero here (image too small)
    const int wCell = (int)std::ceil(width / nCols), hCell = (int)std::ceil(height / nRows);
    std::vector<FastKp> cell;
    std::vector<int> scratch;
    for (int i = 0; i < nRows; ++i) {
      const float iniY = (float)(minBorderY + i * hCell);
      float maxY = iniY + hCell + 6;
      if (iniY >= maxBorderY - 3) continue;
      if (maxY > maxBorderY) maxY = (float)maxBorderY;
      for (int j = 0; j < nCols; ++j) {
        const float iniX = (float)(minBorderX + j * wCell);
        float maxX = iniX + wCell + 6;
        if (iniX >= maxBorderX - 6) continue;
        if (maxX > maxBorderX) maxX = (float)maxBorderX;
        const int x0 = (int)iniX, y0 = (int)iniY, rw = (int)maxX - x0, rh = (int)maxY - y0;
        const uint8_t* roi = lvl(level, y0) + x0;
        fast9_roi(roi, rw, rh, pyr[level].stride, iniTh, cell, scratch);
        if (cell.empty()) fast9_roi(roi, rw, rh, pyr[level].stride, minTh, cell, scratch);
        for (const FastKp& f : cell) {
          KeyPoint kp;
          kp.x = (float)f.x + j * wCell;   // :831-832
          kp.y = (float)f.y + i * hCell;
          kp.size = 7.f; kp.angle = -1.f; kp.response = (float)f.score; kp.octave = 0; kp.class_id = -1;
          toDist.push_back(kp);
        }
      }
    }
    if (ncand) *ncand = (int)toDist.size();
    if (toDist.empty()) return 0;  // reference: DistributeOctTree on empty input yields empty output
    int rc = distribute(toDist, minBorderX, maxBorderX, minBorderY, maxBorderY, nfeat[level], keypoints);
    if (rc) return rc;
    const int scaledPatchSize = (int)(PATCH_SIZE * sf[level]);
    for (KeyPoint& kp : keypoints) {
      kp.x += minBorderX; kp.y += minBorderY; kp.octave = level; kp.size = (float)scaledPatchSize;
    }
    return 0;
  }

  int extract(const uint8_t* img, int rows, int cols, int stride, KeyPoint* okp, uint8_t* odesc, int cap,
              int* cand /*nlevels or null*/) {
    if (!img || rows <= 0 || cols <= 0) return 0;  // :1055 empty image -> return
    compute_pyramid(img, rows, cols, stride);
    std::vector<std::vector<KeyPoint>> all(nlevels);
    for (int l = 0; l < nlevels; ++l) {
      int rc = keypoints_level(l, all[l], cand ? cand + l : nullptr);
      if (rc) return rc;
    }
    for (int l = 0; l < nlevels; ++l)
      for (KeyPoint& kp : all[l]) kp.angle = ic_angle(l, kp.x, kp.y);
    int n = 0;
    Plane work, blur;
    for (int l = 0; l < nlevels; ++l) {
      if (all[l].empty()) continue;
      blur.alloc(lw[l], lh[l]);
      gaussian7_u8(lvl(l, 0), lw[l], lh[l], pyr[l].stride, blur.d.data(), blur.stride);
      for (KeyPoint& kp : all[l]) {
        if (n >= cap) return -2;
        descriptor(kp, blur.d.data(), blur.stride, odesc + (size_t)n * 32);
        KeyPoint o = kp;
        if (l != 0) { o.x *= sf[l]; o.y *= sf[l]; }   // :1104-1110
        okp[n++] = o;
      }
    }
    return n;
  }
};

}  // namespace

extern "C" {

void* orb_ref_create(int nfeatures, float scaleFactor, int nlevels, int iniTh, int minTh) {
  return new Extractor(nfeatures, scaleFactor, nlevels, iniTh, minTh);
}
void orb_ref_destroy(void* h) { delete (Extractor*)h; }

// returns n >= 0, or <0 on error (-1: degenerate aspect ratio, -2: output capacity too small)
int orb_ref_extract(void* h, const uint8_t* img, int rows, int cols, int stride, void* kps, uint8_t* desc,
                    int cap, int* cand_per_level) {
  return ((Extractor*)h)->extract(img, rows, cols, stride, (KeyPoint*)kps, desc, cap, cand_per_level);
}
void orb_ref_tables(void* h, float* sf, float* invsf, float* sigma2, float* invsigma2, int* nfeat, int* umax) {
  Extractor* e = (Extractor*)h;
  for (int i = 0; i < e->nlevels; ++i) {
    sf[i] = e->sf[i]; invsf[i] = e->invsf[i]; sigma2[i] = e->sigma2[i]; invsigma2[i] = e->invsigma2[i];
    nfeat[i] = e->nfeat[i];
  }
  for (int i = 0; i <= HALF_PATCH_SIZE; ++i) umax[i] = e->umax[i];
}
int orb_ref_level_dims(void* h, int level, int* w, int* hgt) {
  Extractor* e = (Extractor*)h;
  if (level < 0 || level >= e->nlevels) return -1;
  *w = e->lw[level]; *hgt = e->lh[level];
  return 0;
}
// bordered=0: w x h level image; bordered=1: (w+38) x (h+38) buffer with the REFLECT_101 frame
void orb_ref_get_level(void* h, int level, int bordered, uint8_t* dst) {
  Extractor* e = (Extractor*)h;
  int w = e->lw[level], hh = e->lh[level];
  if (bordered) {
    memcpy(dst, e->pyr[level].d.data(), e->pyr[level].d.size());
  } else {
    for (int y = 0; y < hh; ++y) memcpy(dst + (size_t)y * w, e->lvl(level, y), w);
  }
}

// FAST candidates of `level` of the last extract, in vToDistributeKeys order: triples (x, y, score) in level pixels
// (shifted by minBorderX / minBorderY).  Returns the count; writes only when it fits in cap.
int orb_ref_candidates(void* h, int level, int* out, int cap) {
  Extractor* e = (Extractor*)h;
  if (level < 0 || level >= e->nlevels) return -1;
  const std::vector<KeyPoint>& v = e->cand[level];
  const int n = (int)v.size(), minBorder = EDGE_THRESHOLD - 3;
  if (n > cap) return n;
  for (int i = 0; i < n; ++i) {
    out[3 * i] = (int)v[i].x + minBorder;
    out[3 * i + 1] = (int)v[i].y + minBorder;
    out[3 * i + 2] = (int)v[i].response;
  }
  return n;
}

// ---- primitives exposed for direct pinning against cv2 ----
void orb_ref_resize(const uint8_t* src, int sw, int sh, uint8_t* dst, int dw, int dh) {
  resize_linear_u8(src, sw, sh, sw, dst, dw, dh, dw);
}
void orb_ref_blur(const uint8_t* src, int w, int h, uint8_t* dst) { gaussian7_u8(src, w, h, w, dst, w); }
// out: triples (x, y, score); returns count (<= cap written)
int orb_ref_fast(const uint8_t* roi, int rw, int rh, int stride, int t, int* out, int cap) {
  std::vector<FastKp> v;
  std::vector<int> scratch;
  fast9_roi(roi, rw, rh, stride, t, v, scratch);
  int n = 0;
  for (const FastKp& f : v) {
    if (n < cap) { out[3 * n] = f.x; out[3 * n + 1] = f.y; out[3 * n + 2] = f.score; }
    ++n;
  }
  return n;
}
float orb_ref_fast_atan2(float y, float x) { return fast_atan2_deg(y, x); }
// count of floats in [lo_bits, hi_bits] (stepping by `step`) where the restated glibc sinf/cosf (include/glibc_sincosf.h,
// the algorithm the CUDA kernel runs) differs from the host libm the oracle calls
long orb_ref_sincosf_mismatches(uint32_t lo_bits, uint32_t hi_bits, uint32_t step) {
  long bad = 0;
  for (uint64_t u = lo_bits; u <= hi_bits; u += step) {
    float x;
    uint32_t uu = (uint32_t)u;
    memcpy(&x, &uu, 4);
    if (b200_cosf(x) != cosf(x)) ++bad;
    if (b200_sinf(x) != sinf(x)) ++bad;
  }
  return bad;
}
void orb_ref_descriptor(const uint8_t* img, int step, float x, float y, float angle, uint8_t* desc) {
  KeyPoint kp{x, y, 31.f, angle, 0.f, 0, -1};
  Extractor::descriptor(kp, img, step, desc);
}
// DistributeOctTree alone: in/out are KeyPoint arrays; returns n_out or <0.  trace (may be null): one record of 5 ints
// per round -- kind (0: a sweep, :608-667; 1: an iteration of the largest-first loop, :678-739), the list size before
// and after it, nToExpand (sweep: children holding more than one keypoint) or m (largest-first: the nodes it sorts), and
// how many nodes it split (a largest-first iteration stops splitting once the list reaches N).  *nrounds = the number
// of rounds; the first trace_cap / 5 are written.
int orb_ref_distribute(const void* in, int n_in, int minX, int maxX, int minY, int maxY, int N, void* out,
                       int cap, int* trace, int trace_cap, int* nrounds) {
  Extractor e(1000, 1.2f, 1, 20, 7);
  std::vector<KeyPoint> vi((const KeyPoint*)in, (const KeyPoint*)in + n_in), vo;
  std::vector<int> tr;
  if (nrounds) *nrounds = 0;
  if (n_in == 0) return 0;
  int rc = e.distribute(vi, minX, maxX, minY, maxY, N, vo, &tr);
  if (rc) return rc;
  if (nrounds) *nrounds = (int)tr.size() / Extractor::TRACE_INTS;
  if (trace) memcpy(trace, tr.data(), sizeof(int) * std::min((size_t)std::max(trace_cap, 0), tr.size()));
  if ((int)vo.size() > cap) return -2;
  memcpy(out, vo.data(), vo.size() * sizeof(KeyPoint));
  return (int)vo.size();
}

// Frame::UndistortKeyPoints (src/Frame.cc:559-590) on xy pairs: cv::undistortPoints(K, dist, R = I, P = K)
void orb_ref_undistort(const float* xy_in, int n, const float* K, const float* dist, int ndist, float* xy_out) {
  if (ndist == 0 || dist[0] == 0.0f) { memcpy(xy_out, xy_in, sizeof(float) * 2 * (size_t)n); return; }
  double k[5] = {0, 0, 0, 0, 0};
  for (int i = 0; i < ndist && i < 5; ++i) k[i] = dist[i];
  for (int i = 0; i < n; ++i) {
    double x, y;
    undistort_point(xy_in[2 * i], xy_in[2 * i + 1], K[0], K[4], K[2], K[5], k, &x, &y);
    xy_out[2 * i] = (float)x; xy_out[2 * i + 1] = (float)y;
  }
}

}  // extern "C"
