// orbx.cu -- host side + C-ABI of the ORB extractor (reference: src/ORBextractor.cc,
// include/ORBextractor.h).  Kernels live in orbx_kernels.cuh.
#include <cmath>
#include <cstdlib>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <utility>
#include <vector>

#include "orbx_kernels.cuh"
#include "orbx_host.h"

namespace b200 {

static const signed char kPatternHost[1024] = {
#include "../../include/orb_pattern_31.inc"
};

// One formulation per stage, each chosen on an H100 SXM (80 GB HBM3, 400 W power limit) with 96-frame batches of 2000
// features, all giving identical bytes: k_orient_desc's formulation takes the orientation stage from 0.228 to 0.209 ms
// per batch against one warp per keypoint; staging up to four FAST tile rows per warp step and clearing the score map
// with 128-bit stores takes FAST from 0.441 to 0.438 ms against two rows and 32-bit stores; FAST CTAs of 1, 2 or 4
// cells instead of FAST_WARPS = 8 move that stage by under 1 %.  The quad-tree's register budget is explained at
// k_quadtree.  What the host still selects follows from the input: the FAST tile pitch from the cell size, and k_resize
// instead of k_resize_g for scale factors above 2.

static inline int cv_round_f(float v) { return (int)lrintf(v); }
static inline int cv_round_d(double v) { return (int)lrint(v); }

// A kernel's dynamic shared-memory limit belongs to the kernel on the current device, not to a handle: raise it to the
// largest size any handle has needed and never lower it, so that handles of different geometries or quotas, on any
// thread, can launch after one another.
static int raise_smem_limit(const void* kernel, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> limit;
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(mu);
  size_t& cur = limit[{kernel, dev}];
  if (bytes <= cur) return B200ORB_OK;
  B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  cur = bytes;
  return B200ORB_OK;
}

}  // namespace b200

using namespace b200;

// =====================================================================================================
// handle
// =====================================================================================================
int orbx::init(const OrbxParams& p, int dev) {
  prm = p;
  device = dev;
  const int nl = p.nlevels;
  // ---- ctor arithmetic, src/ORBextractor.cc:404-465 (scaleFactor member is double, ctor arg float) ----
  const double scaleFactor = (double)p.scale_factor;
  sf[0] = 1.0f; sigma2[0] = 1.0f;
  for (int i = 1; i < nl; ++i) {
    sf[i] = (float)(sf[i - 1] * scaleFactor);
    sigma2[i] = sf[i] * sf[i];
  }
  for (int i = 0; i < nl; ++i) { invsf[i] = 1.0f / sf[i]; invsigma2[i] = 1.0f / sigma2[i]; }
  const float factor = (float)(1.0f / scaleFactor);
  float nDesired = p.nfeatures * (1 - factor) / (1 - (float)std::pow((double)factor, (double)nl));
  int sum = 0;
  for (int l = 0; l < nl - 1; ++l) {
    nfeat[l] = cv_round_f(nDesired);
    sum += nfeat[l];
    nDesired *= factor;
  }
  nfeat[nl - 1] = std::max(p.nfeatures - sum, 0);
  int v, v0;
  const int vmax = (int)std::floor(HALF_PATCH_SIZE * std::sqrt(2.f) / 2 + 1);
  const int vmin = (int)std::ceil(HALF_PATCH_SIZE * std::sqrt(2.f) / 2);
  const double hp2 = HALF_PATCH_SIZE * HALF_PATCH_SIZE;
  for (v = 0; v <= vmax; ++v) otab.umax[v] = cv_round_d(std::sqrt(hp2 - v * v));
  for (v = HALF_PATCH_SIZE, v0 = 0; v >= vmin; --v) {
    while (otab.umax[v0] == otab.umax[v0 + 1]) ++v0;
    otab.umax[v] = v0;
    ++v0;
  }
  B200_CHECK(stream.create());
  for (v = 1; v <= HALF_PATCH_SIZE; ++v)   // k_orient_desc tests the circular mask as v <= vmax(|u|)
    if (otab.umax[v] > otab.umax[v - 1]) { set_error("umax table is not non-increasing"); return B200ORB_EINVAL; }
  // k_orient_desc reads the descriptor's tests from a tile of reach OD_BR.  A point (px, py) lands at
  // round(px*cos - py*sin), round(px*sin + py*cos): both terms are at most |(px, py)| in magnitude, up to the relative
  // error of glibc's cosf / sinf and of three rounded float ops (< 1e-6; 2^-16 leaves room), so the rounded offset is
  // at most floor(|(px, py)| * (1 + 2^-16) + 0.5) at every angle.  ORB's pattern: 18, from (-13, -13) at 45 degrees.
  int reach = 0;
  for (int i = 0; i < 512; ++i) {
    const double r = std::hypot((double)kPatternHost[2 * i], (double)kPatternHost[2 * i + 1]);
    reach = std::max(reach, (int)std::floor(r * (1.0 + 1.0 / 65536) + 0.5));
  }
  if (reach > OD_BR) { set_error("descriptor pattern reaches %d px, beyond the %d-px patch tile", reach, OD_BR); return B200ORB_EINVAL; }
  float pat[1024];
  for (int i = 0; i < 1024; ++i) pat[i] = (float)kPatternHost[i];
  B200_CHECK(patf.carve(stream, [&](Carver& t) { d_patf = t.take<float4>(256); }));
  B200_CUDA(cudaMemcpyAsync(d_patf, pat, sizeof(pat), cudaMemcpyHostToDevice, stream));
  B200_CUDA(cudaStreamSynchronize(stream));
  return B200ORB_OK;
}

// Level sizes, FAST cells and the quad-tree's per-level constants of a rows x cols image, with every refusal of
// extraction; host arithmetic only.  The selection capacity of level l is max(N_l + 3, 4*nIni_l): DistributeOctTree's
// first sweep may return four nodes per initial node (nIni grows with the aspect ratio: 58 at 4000 x 100), and a later
// round stops as soon as the list reaches N_l, at most 3 nodes past it.
int orbx::plan_geometry(int r, int c, GeomPlan& g) const {
  if (r > 4095 || c > 4095) { set_error("image %dx%d exceeds the 4095-px packing limit", c, r); return B200ORB_EINVAL; }
  const int nl = prm.nlevels;
  int* lw = g.lw;
  int* lh = g.lh;
  // level sizes (:1121-1122)
  for (int l = 0; l < nl; ++l) {
    lw[l] = cv_round_f((float)c * invsf[l]);
    lh[l] = cv_round_f((float)r * invsf[l]);
    if (lw[l] <= 2 * EDGE_THRESHOLD - 6 + 0 || lh[l] <= 2 * EDGE_THRESHOLD - 6 + 0) {
      set_error("level %d is %dx%d: too small for the 16-px FAST border (reference would crash)", l, lw[l], lh[l]);
      return B200ORB_EGEOM;
    }
  }
  // FAST cells (:775-815) and quad-tree constants (:545-547)
  std::vector<CellDesc>& cells = g.cells;
  cells.clear();
  LevelTab& ltab = g.ltab;
  int slots = 0, selcap = 0, qcap = 8;
  memset(&ltab, 0, sizeof(ltab));
  ltab.nlevels = nl;
  for (int l = 0; l < nl; ++l) {
    ltab.cell_begin[l] = (int)cells.size();
    ltab.slot_begin[l] = slots;
    const int minBX = FAST_BORDER, minBY = FAST_BORDER;
    const int maxBX = lw[l] - EDGE_THRESHOLD + 3, maxBY = lh[l] - EDGE_THRESHOLD + 3;
    const float width = (float)(maxBX - minBX), height = (float)(maxBY - minBY);
    const float W = 30;
    const int nCols = (int)(width / W), nRows = (int)(height / W);
    if (nCols <= 0 || nRows <= 0) {
      set_error("level %d (%dx%d) has no 30-px FAST cell: the reference divides by zero here", l, lw[l], lh[l]);
      return B200ORB_EGEOM;
    }
    const int wCell = (int)std::ceil(width / nCols), hCell = (int)std::ceil(height / nRows);
    for (int i = 0; i < nRows; ++i) {
      const float iniY = (float)(minBY + i * hCell);
      float maxY = iniY + hCell + 6;
      if (iniY >= maxBY - 3) continue;
      if (maxY > maxBY) maxY = (float)maxBY;
      for (int j = 0; j < nCols; ++j) {
        const float iniX = (float)(minBX + j * wCell);
        float maxX = iniX + wCell + 6;
        if (iniX >= maxBX - 6) continue;
        if (maxX > maxBX) maxX = (float)maxBX;
        CellDesc cd;
        cd.level = (short)l;
        cd.x0 = (short)iniX; cd.y0 = (short)iniY;
        cd.rw = (short)((int)maxX - (int)iniX); cd.rh = (short)((int)maxY - (int)iniY);
        cd.pad = 0;
        cd.slot_off = slots;
        if (cd.rw > FAST_MAX_ROI - 2 || cd.rh > FAST_MAX_ROI) { set_error("FAST cell larger than %d px", FAST_MAX_ROI); return B200ORB_EGEOM; }
        // k_orient_desc's patch tiles reach EDGE_THRESHOLD px around a keypoint: the detection range [x0+3, x0+rw-3)
        // x [y0+3, y0+rh-3) must keep that far from every side of the level
        if (cd.x0 + 3 < EDGE_THRESHOLD || cd.y0 + 3 < EDGE_THRESHOLD || cd.x0 + cd.rw - 4 + EDGE_THRESHOLD > lw[l] - 1 ||
            cd.y0 + cd.rh - 4 + EDGE_THRESHOLD > lh[l] - 1) {
          set_error("FAST cell of level %d reaches within %d px of its side", l, EDGE_THRESHOLD);
          return B200ORB_EGEOM;
        }
        const int iw = cd.rw - 6, ih = cd.rh - 6;
        if (iw > 0 && ih > 0) slots += ((iw + 1) / 2) * ((ih + 1) / 2);
        cells.push_back(cd);
      }
    }
    const int nIni = (int)std::round(static_cast<float>(maxBX - minBX) / (maxBY - minBY));
    if (nIni <= 0) { set_error("aspect ratio of level %d makes nIni = 0 (reference divides by zero)", l); return B200ORB_EGEOM; }
    ltab.n_ini[l] = nIni;
    ltab.hx[l] = static_cast<float>(maxBX - minBX) / nIni;
    ltab.box_h[l] = maxBY - minBY;
    ltab.nfeat[l] = nfeat[l];
    ltab.sf[l] = sf[l];
    ltab.kp_size[l] = (float)(int)(PATCH_SIZE * sf[l]);
    const int capl = std::max(nfeat[l] + 3, 4 * nIni);
    ltab.sel_off[l] = selcap;
    selcap += capl;
    qcap = std::max(qcap, capl + 1);
  }
  ltab.cell_begin[nl] = (int)cells.size();
  ltab.slot_begin[nl] = slots;
  ltab.sel_off[nl] = selcap;
  g.slots = slots;
  g.qt_cap = align_up(qcap, 8);
  if (qt_smem_bytes(g.qt_cap) > 100 * 1024) { set_error("nfeatures too large for the quad-tree kernel's shared memory"); return B200ORB_EINVAL; }
  return B200ORB_OK;
}

// (re)build every geometry-dependent table and buffer for F frames of rows x cols
int orbx::ensure_geometry(int r, int c, int F) {
  if (r == rows && c == cols && F <= maxF) return B200ORB_OK;
  GeomPlan g;
  B200_CHECK(plan_geometry(r, c, g));
  const int keepF = (r == rows && c == cols) ? std::max(F, maxF) : F;
  rows = cols = maxF = 0;   // no geometry until its block exists
  have_results = false;
  const int nl = prm.nlevels;
  size_t off = 0;
  for (int l = 0; l < nl; ++l) {
    lw[l] = g.lw[l];
    lh[l] = g.lh[l];
    lpitch[l] = align_up(lw[l], 16);
    loff[l] = off;
    off += (size_t)lpitch[l] * lh[l];
  }
  frame_bytes = align_up_sz(off, 256);
  // resize tables (SURVEY App. A.2)
  std::vector<int2> xt, yt;
  std::vector<int4> xg;
  resize_group_ok = true;
  for (int l = 1; l < nl; ++l) {
    xt_off[l] = (int)xt.size();
    yt_off[l] = (int)yt.size();
    auto fill = [](int dn, int sn, std::vector<int2>& t) {
      const double scale = 1.0 / ((double)dn / sn);
      for (int d = 0; d < dn; ++d) {
        float f = (float)((d + 0.5) * scale - 0.5);
        int i = (int)std::floor(f);
        f -= (float)i;
        if (i < 0) { i = 0; f = 0.f; }
        if (i >= sn - 1) { i = sn - 1; f = 0.f; }
        const int a0 = (short)cv_round_f((1.f - f) * 2048.f), a1 = (short)cv_round_f(f * 2048.f);
        t.push_back(make_int2(i, (a0 & 0xffff) | (a1 << 16)));
      }
    };
    fill(lw[l], lw[l - 1], xt);
    fill(lh[l], lh[l - 1], yt);
    // group table of k_resize_g
    xg_off[l] = (int)xg.size();
    for (int dx0 = 0; dx0 < lw[l]; dx0 += 4) {
      const int2* t = xt.data() + xt_off[l];
      int sx[4], cf[4];
      for (int i = 0; i < 4; ++i) { const int2 e = t[std::min(dx0 + i, lw[l] - 1)]; sx[i] = e.x; cf[i] = e.y; }
      for (int i = 1; i < 4; ++i) if (sx[i] < sx[0]) sx[i] = sx[0];   // (replicated tail entries never precede sx[0])
      int sels = 0;
      for (int i = 0; i < 4; ++i) {
        const int dlt = sx[i] - sx[0];
        if (dlt + 1 > 7) resize_group_ok = false;   // scale > 2: the byte-window path does not apply
        sels |= (((dlt & 7) | (((dlt + 1) & 7) << 4)) & 0xff) << (8 * i);
      }
      xg.push_back(make_int4(sx[0] >> 2, 8 * (sx[0] & 3), sels, 0));
      xg.push_back(make_int4(cf[0], cf[1], cf[2], cf[3]));
    }
  }
  const std::vector<CellDesc>& cells = g.cells;
  ltab = g.ltab;
  ncells = (int)cells.size();
  {
    int rwm = 0, rhm = 0, det = 0;
    for (const CellDesc& cd : cells) {
      rwm = std::max(rwm, (int)cd.rw); rhm = std::max(rhm, (int)cd.rh);
      det = std::max(det, ((int)cd.rw - 6) * ((int)cd.rh - 6));
    }
    fast_clist_cap = align_up(std::max(det, 8), 8);   // every detection pixel of a cell may be a corner
    fast_tp = (rwm + 3 <= FAST_TP_SMALL) ? FAST_TP_SMALL : FAST_TP_BIG;
    fast_rows_max = rhm;
    fast_smem = (size_t)FAST_WARPS * (2 * rhm * fast_tp + 2 * FAST_QLEN + 2 * fast_clist_cap);
    if (fast_smem > 48 * 1024) {
      B200_CHECK(raise_smem_limit((const void*)k_fast_cells<FAST_TP_BIG>, fast_smem));
      B200_CHECK(raise_smem_limit((const void*)k_fast_cells<FAST_TP_SMALL>, fast_smem));
    }
  }
  slots_per_frame = align_up(g.slots, 4);
  sel_per_frame = ltab.sel_off[nl];
  cap = sel_per_frame;
  qt_cap = g.qt_cap;
  qt_smem = qt_smem_bytes(qt_cap);
  B200_CHECK(raise_smem_limit((const void*)k_quadtree, qt_smem));

  std::vector<BlurTile> bt;
  for (int l = 0; l < nl; ++l)
    for (int y = 0; y < lh[l]; y += BLS_ROWS)
      for (int x = 0; x < lw[l]; x += 128) bt.push_back(BlurTile{(short)l, (short)x, (short)y, 0});
  n_blur_tiles = (int)bt.size();
  std::vector<BlurEdge> be;
  for (int l = 0; l < nl; ++l)
    for (int x = 0; x < lw[l]; x += 4)
      if (x < 4 || x + 8 > lw[l])
        for (int y = 0; y < lh[l]; y += BLS_ROWS) be.push_back(BlurEdge{(short)l, (short)x, (short)y, 0});
  n_blur_edges = (int)be.size();

  const size_t Fz = (size_t)keepF;
  B200_CHECK(geom.carve(stream, [&](Carver& t) {
    d_raw = t.take<uint8_t>(frame_bytes * Fz); d_blur = t.take<uint8_t>(frame_bytes * Fz);
    d_cells = t.take<CellDesc>(ncells); d_cand = t.take<unsigned>(slots_per_frame * Fz);
    d_cellcnt = t.take<int>(ncells * Fz); d_qkp = t.take<unsigned>(slots_per_frame * Fz);
    d_qnode = t.take<int>(slots_per_frame * Fz); d_sel = t.take<unsigned>(sel_per_frame * Fz);
    d_selcnt = t.take<int>(nl * Fz); d_candcnt = t.take<int>(nl * Fz);
    d_kps = t.take<OrbxKeyPoint>(cap * Fz); d_desc = t.take<uint8_t>(32 * cap * Fz); d_n = t.take<int>(Fz);
    d_xt = t.take<int2>(xt.size()); d_yt = t.take<int2>(yt.size()); d_xg = t.take<int4>(xg.size());
    d_blur_tiles = t.take<BlurTile>(bt.size()); d_blur_edges = t.take<BlurEdge>(be.size());
  }));
  B200_CUDA(cudaMemcpyAsync(d_blur_edges, be.data(), sizeof(BlurEdge) * be.size(), cudaMemcpyHostToDevice, stream));
  B200_CUDA(cudaMemcpyAsync(d_blur_tiles, bt.data(), sizeof(BlurTile) * bt.size(), cudaMemcpyHostToDevice, stream));
  B200_CUDA(cudaMemcpyAsync(d_cells, cells.data(), sizeof(CellDesc) * ncells, cudaMemcpyHostToDevice, stream));
  if (!xt.empty()) B200_CUDA(cudaMemcpyAsync(d_xt, xt.data(), sizeof(int2) * xt.size(), cudaMemcpyHostToDevice, stream));
  if (!yt.empty()) B200_CUDA(cudaMemcpyAsync(d_yt, yt.data(), sizeof(int2) * yt.size(), cudaMemcpyHostToDevice, stream));
  if (!xg.empty()) B200_CUDA(cudaMemcpyAsync(d_xg, xg.data(), sizeof(int4) * xg.size(), cudaMemcpyHostToDevice, stream));
  B200_CUDA(cudaStreamSynchronize(stream));   // the tables are locals
  rows = r; cols = c; maxF = keepF;
  // blurred pyramid view never changes; raw view's level 0 may alias the caller's buffer per call
  for (int l = 0; l < nl; ++l) {
    blurv.p[l] = d_blur + loff[l]; blurv.fstride[l] = frame_bytes; blurv.pitch[l] = lpitch[l];
    blurv.w[l] = lw[l]; blurv.h[l] = lh[l];
    rawv.p[l] = d_raw + loff[l]; rawv.fstride[l] = frame_bytes; rawv.pitch[l] = lpitch[l];
    rawv.w[l] = lw[l]; rawv.h[l] = lh[l];
  }
  return B200ORB_OK;
}

// Enqueue the whole extractor for frames [f0, f0+F) of the batch; d_l0 = level 0 of frame f0.  Ranges of one batch may be
// enqueued one after another (the host path uploads and extracts in chunks so that PCIe and the SMs overlap).
int orbx::run(const uint8_t* d_l0, int pitch0, size_t fstride0, int F, int f0) {
  const int nl = prm.nlevels;
  B200_CHECK(prof_begin(F));
  // The kernels read level rows as aligned 32-bit words.  A level 0 that is not 4-byte aligned (pointer, pitch or frame
  // stride) is copied into the internal plane first.  The ranges of one batch all take the same branch: their pointers
  // differ by multiples of fstride0.
  if ((((uintptr_t)d_l0) | (uintptr_t)pitch0 | fstride0) & 3) {
    uint8_t* staged = d_raw + (size_t)f0 * frame_bytes;
    for (int f = 0; f < F; ++f)
      B200_CUDA(cudaMemcpy2DAsync(staged + (size_t)f * frame_bytes, lpitch[0], d_l0 + (size_t)f * fstride0, pitch0, lw[0],
                                  lh[0], cudaMemcpyDeviceToDevice, stream));
    d_l0 = staged;
    pitch0 = lpitch[0];
    fstride0 = frame_bytes;
  }
  // frame-range views: every per-frame array is addressed as base + frame * stride inside the kernels
  PyrView rawv = this->rawv, blurv = this->blurv;
  for (int l = 1; l < nl; ++l) rawv.p[l] += (size_t)f0 * rawv.fstride[l];
  for (int l = 0; l < nl; ++l) blurv.p[l] += (size_t)f0 * blurv.fstride[l];
  rawv.p[0] = const_cast<uint8_t*>(d_l0);
  rawv.pitch[0] = pitch0;
  rawv.fstride[0] = fstride0;
  if (f0 == 0) {   // what orbx_get_level reads back
    this->rawv.p[0] = const_cast<uint8_t*>(d_l0); this->rawv.pitch[0] = pitch0; this->rawv.fstride[0] = fstride0;
  }
  unsigned* d_cand = this->d_cand + (size_t)f0 * slots_per_frame;
  int* d_cellcnt = this->d_cellcnt + (size_t)f0 * ncells;
  unsigned* d_qkp = this->d_qkp + (size_t)f0 * slots_per_frame;
  int* d_qnode = this->d_qnode + (size_t)f0 * slots_per_frame;
  unsigned* d_sel = this->d_sel + (size_t)f0 * sel_per_frame;
  int* d_selcnt = this->d_selcnt + (size_t)f0 * nl;
  int* d_candcnt = this->d_candcnt + (size_t)f0 * nl;
  OrbxKeyPoint* d_kps = this->d_kps + (size_t)f0 * cap;
  uint8_t* d_desc = this->d_desc + (size_t)f0 * cap * 32;
  int* d_n = this->d_n + f0;
  // K1 pyramid
  for (int l = 1; l < nl; ++l) {
    dim3 blk(32, 8), grd((lw[l] + 127) / 128, (lh[l] + 7) / 8, F);
    // k_resize_g needs the 4 outputs of a thread within an 8-byte source window (scale factor <= 2)
    if (resize_group_ok)
      k_resize_g<<<grd, blk, 0, stream>>>(rawv.p[l - 1], rawv.pitch[l - 1], rawv.fstride[l - 1], lh[l - 1], rawv.p[l],
                                         rawv.pitch[l], rawv.fstride[l], lw[l], lh[l], d_xg + xg_off[l], d_yt + yt_off[l]);
    else
      k_resize<<<grd, blk, 0, stream>>>(rawv.p[l - 1], rawv.pitch[l - 1], rawv.fstride[l - 1], lw[l - 1], lh[l - 1],
                                       rawv.p[l], rawv.pitch[l], rawv.fstride[l], lw[l], lh[l], d_xt + xt_off[l],
                                       d_yt + yt_off[l]);
    ++launches;
  }
  B200_CHECK(prof_mark(ST_RESIZE + 1));
  // K2 FAST cells
  auto* fast_kernel = fast_tp == FAST_TP_SMALL ? k_fast_cells<FAST_TP_SMALL> : k_fast_cells<FAST_TP_BIG>;
  fast_kernel<<<dim3((ncells + FAST_WARPS - 1) / FAST_WARPS, F), FAST_THREADS, fast_smem, stream>>>(
      rawv, d_cells, ncells, slots_per_frame, prm.ini_th_fast, prm.min_th_fast, d_cand, d_cellcnt, fast_rows_max,
      fast_clist_cap);
  ++launches;
  B200_CHECK(prof_mark(ST_FAST + 1));
  // K3 quad-tree: one CTA per (level, frame)
  k_quadtree<<<dim3(nl, F), QT_THREADS, qt_smem, stream>>>(ltab, d_cells, d_cand, d_cellcnt, ncells, slots_per_frame,
                                                           QtScratchView{d_qkp, d_qnode}, qt_cap, d_sel, d_selcnt,
                                                           d_candcnt, sel_per_frame);
  ++launches;
  B200_CHECK(prof_mark(ST_QUADTREE + 1));
  if (after_select) B200_CHECK(after_select(after_select_ctx, f0, F));
  // K4 blur: one launch over every (level, 128x35 tile, frame), one over the border column groups
  k_blur7_strip<<<dim3(n_blur_tiles, F), 32, 0, stream>>>(rawv, blurv, d_blur_tiles);
  k_blur7_edges<<<dim3((n_blur_edges + 63) / 64, F), 64, 0, stream>>>(rawv, blurv, d_blur_edges, n_blur_edges);
  launches += 2;
  B200_CHECK(prof_mark(ST_BLUR + 1));
  // K5 orientation + descriptors
  k_orient_desc<<<dim3((cap + OD_WARPS * OD_KPW - 1) / (OD_WARPS * OD_KPW), F), OD_WARPS * 32, 0, stream>>>(
      ltab, otab, rawv, blurv, d_patf, d_sel, d_selcnt, sel_per_frame, d_kps, d_desc, d_n, cap);
  ++launches;
  B200_CHECK(prof_mark(ST_ORIENT_DESC + 1));
  B200_CUDA(cudaGetLastError());
  lastF = f0 + F;
  have_results = true;
  return B200ORB_OK;
}

int orbx::prof_begin(int frames) {
  if (!profile) return B200ORB_OK;
  prof_runs.emplace_back();
  prof_runs.back().frames = frames;
  return prof_mark(0);
}

int orbx::prof_mark(int boundary) {
  if (!profile || prof_runs.empty()) return B200ORB_OK;
  StageEvents& se = prof_runs.back();
  B200_CHECK(se.ev[boundary].create(/*timing=*/1));
  B200_CUDA(cudaEventRecord(se.ev[boundary], stream));
  return B200ORB_OK;
}

// =====================================================================================================
// C-ABI
// =====================================================================================================
extern "C" {

int b200orb_get_tuning(int* exp_mask, int* fast_wpc, int* qt_minblocks) {
  if (exp_mask) *exp_mask = 3;   // both bits: k_orient_desc's formulation (1) and the four-row FAST tile staging (2)
  if (fast_wpc) *fast_wpc = FAST_WARPS;
  if (qt_minblocks) *qt_minblocks = QT_MIN_CTAS;
  return B200ORB_OK;
}

int orbx_create(const OrbxParams* p, int device, orbx_t** out) {
  if (!p || !out) { set_error("null argument"); return B200ORB_EINVAL; }
  *out = nullptr;
  if (p->nlevels < 1 || p->nlevels > MAX_LEVELS || p->nfeatures < 0 || !(p->scale_factor > 1.0f) ||
      p->ini_th_fast < p->min_th_fast || p->min_th_fast < 0 || p->ini_th_fast > 254) {
    set_error("bad OrbxParams (nlevels 1..%d, scale_factor > 1, 0 <= minTh <= iniTh <= 254)", MAX_LEVELS);
    return B200ORB_EINVAL;
  }
  B200_CHECK(check_device(device));
  DeviceGuard g(device);
  std::unique_ptr<orbx> h(new (std::nothrow) orbx());
  if (!h) { set_error("out of host memory"); return B200ORB_EINVAL; }
  B200_CHECK(h->init(*p, device));
  *out = h.release();
  return B200ORB_OK;
}

void orbx_destroy(orbx_t* h) { destroy_handle(h); }

int orbx_max_keypoints(const orbx_t* h) {
  if (!h) return 0;
  // before the first extract: sum over levels of max(N_l + 3, 16), the bound of images with nIni <= 4 on every level;
  // wider images need orbx_max_keypoints_for.  After it: the capacity of the current geometry.
  int s = 0;
  for (int l = 0; l < h->prm.nlevels; ++l) s += std::max(h->nfeat[l] + 3, 16);
  return std::max(s, h->cap);
}

int orbx_max_keypoints_for(const orbx_t* h, int rows, int cols, int* n) {
  if (!h || !n) { set_error("null argument"); return B200ORB_EINVAL; }
  *n = 0;
  if (rows <= 0 || cols <= 0) return B200ORB_OK;   // an empty image returns no keypoints (:1055)
  GeomPlan g;
  B200_CHECK(h->plan_geometry(rows, cols, g));
  *n = g.ltab.sel_off[h->prm.nlevels];
  return B200ORB_OK;
}

static int extract_common(orbx* h, const uint8_t* gray, bool on_device, int nframes, int rows, int cols,
                          size_t stride, size_t frame_stride) {
  if (!gray) { set_error("null image"); return B200ORB_EINVAL; }
  if (stride < (size_t)cols || (nframes > 1 && frame_stride < stride * (size_t)(rows - 1) + cols)) {
    set_error("bad stride");
    return B200ORB_EINVAL;
  }
  B200_CHECK(h->ensure_geometry(rows, cols, nframes));
  if (on_device) {
    if (stride > 0x7fffffff) { set_error("stride too large"); return B200ORB_EINVAL; }
    return h->run(gray, (int)stride, frame_stride, nframes);
  }
  // host images: stage through the internal level-0 planes (pitch = cols rounded up to 16)
  for (int f = 0; f < nframes; ++f)
    B200_CUDA(cudaMemcpy2DAsync(h->d_raw + (size_t)f * h->frame_bytes, h->lpitch[0], gray + (size_t)f * frame_stride,
                                stride, cols, rows, cudaMemcpyHostToDevice, h->stream));
  return h->run(h->d_raw, h->lpitch[0], h->frame_bytes, nframes);
}

int orbx_extract_batch(orbx_t* h, const uint8_t* gray, int nframes, int rows, int cols, size_t stride,
                       size_t frame_stride, OrbxKeyPoint* kps, uint8_t* desc, int cap, int* n_out) {
  if (!h || !n_out) { set_error("null argument"); return B200ORB_EINVAL; }
  if (nframes <= 0) return B200ORB_OK;
  if (rows <= 0 || cols <= 0) {   // :1055 empty image -> outputs untouched
    for (int f = 0; f < nframes; ++f) n_out[f] = 0;
    return B200ORB_OK;
  }
  if (!kps || !desc || cap <= 0) { set_error("null/empty output buffers"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  B200_CHECK(extract_common(h, gray, false, nframes, rows, cols, stride, frame_stride));
  const size_t kn = (size_t)h->cap * nframes;
  OrbxKeyPoint* hk;
  uint8_t* hd;
  int* hn;
  B200_CHECK(h->stage.reserve(h->stream, [&](Carver& t) {
    hk = t.take<OrbxKeyPoint>(kn); hd = t.take<uint8_t>(32 * kn); hn = t.take<int>(nframes);
  }));
  B200_CUDA(cudaMemcpyAsync(hn, h->d_n, sizeof(int) * nframes, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(hk, h->d_kps, sizeof(OrbxKeyPoint) * kn, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(hd, h->d_desc, 32 * kn, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  int rc = B200ORB_OK;
  for (int f = 0; f < nframes; ++f) {
    const int n = hn[f];
    n_out[f] = n;
    if (n > cap) { set_error("frame %d produced %d keypoints > cap %d", f, n, cap); rc = B200ORB_ECAP; continue; }
    memcpy(kps + (size_t)f * cap, hk + (size_t)f * h->cap, sizeof(OrbxKeyPoint) * n);
    memcpy(desc + (size_t)f * cap * 32, hd + (size_t)f * h->cap * 32, (size_t)32 * n);
  }
  return rc;
}

int orbx_extract(orbx_t* h, const uint8_t* gray, int rows, int cols, size_t stride, OrbxKeyPoint* kps,
                 uint8_t* desc, int cap, int* n_out) {
  return orbx_extract_batch(h, gray, 1, rows, cols, stride, stride * (size_t)(rows > 0 ? rows : 0), kps, desc, cap,
                            n_out);
}

int orbx_extract_batch_device(orbx_t* h, const uint8_t* d_gray, int nframes, int rows, int cols, size_t stride,
                              size_t frame_stride) {
  if (!h) { set_error("null handle"); return B200ORB_EINVAL; }
  if (nframes <= 0 || rows <= 0 || cols <= 0) { set_error("empty batch"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  return extract_common(h, d_gray, true, nframes, rows, cols, stride, frame_stride);
}

int orbx_device_results(orbx_t* h, const OrbxKeyPoint** d_kps, const uint8_t** d_desc, const int32_t** d_counts,
                        int* cap) {
  if (!h || !h->have_results) { set_error("no results"); return B200ORB_EINVAL; }
  if (d_kps) *d_kps = h->d_kps;
  if (d_desc) *d_desc = h->d_desc;
  if (d_counts) *d_counts = h->d_n;
  if (cap) *cap = h->cap;
  return B200ORB_OK;
}

int orbx_sync(orbx_t* h) {
  if (!h) return B200ORB_EINVAL;
  DeviceGuard g(h->device);
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}
void* orbx_stream(orbx_t* h) { return h ? (void*)(cudaStream_t)h->stream : nullptr; }

int orbx_level_dims(const orbx_t* h, int level, int* rows, int* cols) {
  if (!h || level < 0 || level >= h->prm.nlevels || h->rows == 0) { set_error("bad level / no geometry yet"); return B200ORB_EINVAL; }
  if (rows) *rows = h->lh[level];
  if (cols) *cols = h->lw[level];
  return B200ORB_OK;
}

int orbx_get_level(orbx_t* h, int frame, int level, int kind, uint8_t* dst, size_t dst_stride) {
  if (!h || !dst || !h->have_results || level < 0 || level >= h->prm.nlevels || frame < 0 || frame >= h->lastF ||
      kind < 0 || kind > 2) {
    set_error("bad argument / no extract yet");
    return B200ORB_EINVAL;
  }
  DeviceGuard g(h->device);
  const int w = h->lw[level], hh = h->lh[level];
  const PyrView& v = (kind == 2) ? h->blurv : h->rawv;
  const uint8_t* src = v.p[level] + (size_t)frame * v.fstride[level];
  if (kind != 1) {
    if (dst_stride < (size_t)w) { set_error("dst_stride too small"); return B200ORB_EINVAL; }
    B200_CUDA(cudaMemcpy2DAsync(dst, dst_stride, src, v.pitch[level], w, hh, cudaMemcpyDeviceToHost, h->stream));
    B200_CUDA(cudaStreamSynchronize(h->stream));
    return B200ORB_OK;
  }
  const int B = EDGE_THRESHOLD, bw = w + 2 * B, bh = hh + 2 * B;
  if (dst_stride < (size_t)bw) { set_error("dst_stride too small"); return B200ORB_EINVAL; }
  uint8_t* d_tmp;
  B200_CHECK(h->tmp.reserve(h->stream, [&](Carver& t) { d_tmp = t.take<uint8_t>((size_t)bw * bh); }));
  dim3 blk(32, 8), grd((bw + 31) / 32, (bh + 7) / 8);
  k_border_copy<<<grd, blk, 0, h->stream>>>(src, h->rawv.pitch[level], w, hh, d_tmp, bw, B);
  ++h->launches;
  B200_CUDA(cudaMemcpy2DAsync(dst, dst_stride, d_tmp, bw, bw, bh, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int orbx_scale_tables(const orbx_t* h, float* sf, float* inv_sf, float* sigma2, float* inv_sigma2,
                      int* features_per_level) {
  if (!h) return B200ORB_EINVAL;
  for (int i = 0; i < h->prm.nlevels; ++i) {
    if (sf) sf[i] = h->sf[i];
    if (inv_sf) inv_sf[i] = h->invsf[i];
    if (sigma2) sigma2[i] = h->sigma2[i];
    if (inv_sigma2) inv_sigma2[i] = h->invsigma2[i];
    if (features_per_level) features_per_level[i] = h->nfeat[i];
  }
  return B200ORB_OK;
}

int orbx_candidates_per_level(orbx_t* h, int frame, int* counts) {
  if (!h || !counts || !h->have_results || frame < 0 || frame >= h->lastF) { set_error("bad argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  B200_CUDA(cudaMemcpyAsync(counts, h->d_candcnt + (size_t)frame * h->prm.nlevels, sizeof(int) * h->prm.nlevels,
                            cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int orbx_get_candidates(orbx_t* h, int frame, int level, int32_t* xys, int cap, int* n) {
  if (!h || !n || !h->have_results || level < 0 || level >= h->prm.nlevels || frame < 0 || frame >= h->lastF) {
    set_error("bad argument / no extract yet");
    return B200ORB_EINVAL;
  }
  DeviceGuard g(h->device);
  const int c0 = h->ltab.cell_begin[level], nc = h->ltab.cell_begin[level + 1] - c0;
  const int s0 = h->ltab.slot_begin[level], ns = h->ltab.slot_begin[level + 1] - s0;
  std::vector<CellDesc> cells(nc);
  std::vector<int> cnt(nc);
  std::vector<unsigned> slots(ns);
  B200_CUDA(cudaMemcpyAsync(cells.data(), h->d_cells + c0, sizeof(CellDesc) * nc, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(cnt.data(), h->d_cellcnt + (size_t)frame * h->ncells + c0, sizeof(int) * nc,
                            cudaMemcpyDeviceToHost, h->stream));
  if (ns > 0)
    B200_CUDA(cudaMemcpyAsync(slots.data(), h->d_cand + (size_t)frame * h->slots_per_frame + s0, sizeof(unsigned) * ns,
                              cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  int total = 0;
  for (int c = 0; c < nc; ++c) total += cnt[c];
  *n = total;
  if (cap < total) { set_error("level %d has %d FAST candidates > cap %d", level, total, cap); return B200ORB_ECAP; }
  if (total > 0 && !xys) { set_error("null output buffer"); return B200ORB_EINVAL; }
  // the cells' segments in cell order: the order k_quadtree gathers them in
  int k = 0;
  for (int c = 0; c < nc; ++c)
    for (int i = 0; i < cnt[c]; ++i, ++k) {
      const unsigned v = slots[cells[c].slot_off - s0 + i];
      xys[3 * k] = (int32_t)(v & 0xfff);
      xys[3 * k + 1] = (int32_t)((v >> 12) & 0xfff);
      xys[3 * k + 2] = (int32_t)(v >> 24);
    }
  return B200ORB_OK;
}

int orbx_distribute(orbx_t* h, int rows, int cols, int level, int N, const int32_t* xys, int n, int32_t* out, int cap,
                    int* n_out) {
  if (!h || !n_out || !out || (n > 0 && !xys)) { set_error("null argument"); return B200ORB_EINVAL; }
  if (rows <= 0 || cols <= 0 || level < 0 || level >= h->prm.nlevels || n < 0) {
    set_error("bad geometry, level or count");
    return B200ORB_EINVAL;
  }
  if (N < 0 || N > h->nfeat[level]) { set_error("N = %d outside 0..%d", N, h->nfeat[level]); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  B200_CHECK(h->ensure_geometry(rows, cols, 1));
  // the distribution region of the level (:783-786): x in [16, maxBorderX), y in [16, maxBorderY)
  const int maxBX = h->lw[level] - EDGE_THRESHOLD + 3, maxBY = h->lh[level] - EDGE_THRESHOLD + 3;
  for (int i = 0; i < n; ++i) {
    const int x = xys[3 * i], y = xys[3 * i + 1], r = xys[3 * i + 2];
    if (x < FAST_BORDER || x >= maxBX || y < FAST_BORDER || y >= maxBY || r < 0 || r > 255) {
      set_error("candidate %d (%d, %d, %d) outside [%d, %d) x [%d, %d) x [0, 255]", i, x, y, r, FAST_BORDER, maxBX,
                FAST_BORDER, maxBY);
      return B200ORB_EINVAL;
    }
  }
  const LevelTab& lt = h->ltab;
  const int c0 = lt.cell_begin[level], nc = lt.cell_begin[level + 1] - c0;
  const int s0 = lt.slot_begin[level], ns = lt.slot_begin[level + 1] - s0;
  if (n > ns) { set_error("%d candidates > the %d slots of level %d", n, ns, level); return B200ORB_ECAP; }
  // the list in order through the level's cell segments, each filled up to its slot count: k_quadtree's gather
  // concatenates exactly the caller's list
  std::vector<CellDesc> cells(nc);
  B200_CUDA(cudaMemcpyAsync(cells.data(), h->d_cells + c0, sizeof(CellDesc) * nc, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  std::vector<unsigned> slots(std::max(ns, 1));
  std::vector<int> cnt(h->ncells, 0);
  for (int i = 0; i < n; ++i) slots[i] = (unsigned)xys[3 * i] | ((unsigned)xys[3 * i + 1] << 12) | ((unsigned)xys[3 * i + 2] << 24);
  for (int c = 0, k = 0; c < nc && k < n; ++c) {
    const int end = (c + 1 < nc) ? cells[c + 1].slot_off - s0 : ns;
    cnt[c0 + c] = std::min(n, end) - k;
    k += cnt[c0 + c];
  }
  h->have_results = false;   // the candidates, selections and counts of frame 0 are overwritten
  if (n > 0)
    B200_CUDA(cudaMemcpyAsync(h->d_cand + s0, slots.data(), sizeof(unsigned) * n, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(h->d_cellcnt, cnt.data(), sizeof(int) * h->ncells, cudaMemcpyHostToDevice, h->stream));
  LevelTab ltab = lt;
  ltab.nfeat[level] = N;
  k_quadtree<<<dim3(h->prm.nlevels, 1), QT_THREADS, h->qt_smem, h->stream>>>(
      ltab, h->d_cells, h->d_cand, h->d_cellcnt, h->ncells, h->slots_per_frame, QtScratchView{h->d_qkp, h->d_qnode},
      h->qt_cap, h->d_sel, h->d_selcnt, h->d_candcnt, h->sel_per_frame);
  ++h->launches;
  B200_CUDA(cudaGetLastError());
  int m = 0;
  B200_CUDA(cudaMemcpyAsync(&m, h->d_selcnt + level, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  *n_out = m;
  if (cap < m) { set_error("%d keypoints selected > cap %d", m, cap); return B200ORB_ECAP; }
  std::vector<unsigned> sel(std::max(m, 1));
  if (m > 0) {
    B200_CUDA(cudaMemcpyAsync(sel.data(), h->d_sel + lt.sel_off[level], sizeof(unsigned) * m, cudaMemcpyDeviceToHost,
                              h->stream));
    B200_CUDA(cudaStreamSynchronize(h->stream));
  }
  for (int j = 0; j < m; ++j) {
    out[3 * j] = (int32_t)(sel[j] & 0xfff);
    out[3 * j + 1] = (int32_t)((sel[j] >> 12) & 0xfff);
    out[3 * j + 2] = (int32_t)(sel[j] >> 24);
  }
  return B200ORB_OK;
}

long long orbx_launch_count(const orbx_t* h) { return h ? h->launches : 0; }

int orbx_profile_enable(orbx_t* h, int on) {
  if (!h) return B200ORB_EINVAL;
  h->profile = on != 0;
  return B200ORB_OK;
}

// Sum of per-stage device time (ms) and frames over every run() since the last read; synchronises the stream.
int orbx_profile_read(orbx_t* h, float* ms /*B200ORB_NUM_STAGES*/, long long* frames, int* runs) {
  if (!h || !ms) return B200ORB_EINVAL;
  DeviceGuard g(h->device);
  B200_CUDA(cudaStreamSynchronize(h->stream));
  for (int s = 0; s < ST_COUNT; ++s) ms[s] = 0.f;
  long long fr = 0;
  for (StageEvents& se : h->prof_runs) {
    fr += se.frames;
    int prev = 0;
    for (int b = 1; b <= ST_COUNT; ++b) {
      if (!se.ev[b]) continue;
      float t = 0.f;
      if (se.ev[prev]) cudaEventElapsedTime(&t, se.ev[prev], se.ev[b]);
      ms[b - 1] += t;
      prev = b;
    }
  }
  if (frames) *frames = fr;
  if (runs) *runs = (int)h->prof_runs.size();
  h->prof_runs.clear();
  return B200ORB_OK;
}

}  // extern "C"
