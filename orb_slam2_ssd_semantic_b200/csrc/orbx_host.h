// orbx_host.h -- definition of the extractor handle and the types of its tables (shared by orbx.cu and the stream
// pipeline orbs.cu).  The kernels are orbx_kernels.cuh's.
#pragma once
#include <vector>

#include "common.cuh"

namespace b200 {

struct PyrView {                 // one image pyramid (raw or blurred) of a batch
  uint8_t* p[MAX_LEVELS];        // frame 0 of level l
  size_t fstride[MAX_LEVELS];    // bytes between consecutive frames of level l
  int pitch[MAX_LEVELS];
  int w[MAX_LEVELS], h[MAX_LEVELS];
};

struct CellDesc {                // one FAST cell (src/ORBextractor.cc:798-838)
  short level;
  short x0, y0;                  // ROI origin in level coordinates (= iniX, iniY)
  short rw, rh;                  // ROI size (maxX-iniX, maxY-iniY); detection range is the ROI minus 3 px
  short pad;
  int slot_off;                  // offset of this cell's segment inside a frame's cand[]
};

struct LevelTab {                // per-level constants of the extractor
  int cell_begin[MAX_LEVELS + 1];   // cells of level l: [cell_begin[l], cell_begin[l+1])
  int slot_begin[MAX_LEVELS + 1];   // cand slots of level l
  int nfeat[MAX_LEVELS];            // mnFeaturesPerLevel
  int sel_off[MAX_LEVELS + 1];      // offset of level l inside a frame's sel[] / capacity
  int n_ini[MAX_LEVELS];            // DistributeOctTree nIni (:545)
  int box_h[MAX_LEVELS];            // maxBorderY-minBorderY: height of the initial nodes (:558)
  float hx[MAX_LEVELS];             // DistributeOctTree hX (:547)
  float sf[MAX_LEVELS];             // mvScaleFactor
  float kp_size[MAX_LEVELS];        // (float)(int)(PATCH_SIZE*mvScaleFactor[l]) (:846)
  int nlevels;
};

__device__ __forceinline__ unsigned pack_kp(int x, int y, int resp) {
  return (unsigned)x | ((unsigned)y << 12) | ((unsigned)resp << 24);
}
__device__ __forceinline__ int kp_x(unsigned v) { return v & 0xfff; }
__device__ __forceinline__ int kp_y(unsigned v) { return (v >> 12) & 0xfff; }
__device__ __forceinline__ int kp_r(unsigned v) { return v >> 24; }

struct OrientTab {
  int umax[HALF_PATCH_SIZE + 1];
};

struct GeomPlan {                // what orbx::plan_geometry derives from rows x cols
  int lw[MAX_LEVELS], lh[MAX_LEVELS];
  std::vector<CellDesc> cells;
  LevelTab ltab;                 // ltab.sel_off[nlevels]: keypoints one frame can return
  int slots = 0, qt_cap = 0;     // FAST candidate slots per frame; quad-tree list capacity
};

struct BlurTile { short level, x0, y0, pad; };   // one warp-tile of k_blur7_strip: 128 columns x BLS_ROWS rows of one level
struct BlurEdge { short level, x0, y0, pad; };   // one border column group of k_blur7_edges

enum { ST_RESIZE = 0, ST_FAST, ST_QUADTREE, ST_BLUR, ST_ORIENT_DESC, ST_GLUE, ST_MATCH, ST_COUNT };
struct StageEvents {
  Event ev[ST_COUNT + 1];   // null: the boundary was not recorded
  int frames = 0;
};
}  // namespace b200

struct orbx {
  OrbxParams prm{};
  int device = 0;
  b200::Stream stream;
  long long launches = 0;
  // optional hook, called by run() right after the keypoint selection of frames [f0, f0 + F) has been enqueued
  // (the batch tracker uses it to start fetching the depth under the selected keypoints while blur / descriptors run)
  int (*after_select)(void* ctx, int f0, int F) = nullptr;
  void* after_select_ctx = nullptr;
  // tables of the constructor (src/ORBextractor.cc:404-465)
  float sf[b200::MAX_LEVELS], invsf[b200::MAX_LEVELS], sigma2[b200::MAX_LEVELS], invsigma2[b200::MAX_LEVELS];
  int nfeat[b200::MAX_LEVELS];
  b200::OrientTab otab{};
  b200::DeviceBlock patf;
  float4* d_patf = nullptr;   // the 256 tests as float4 (x0, y0, x1, y1), for k_orient_desc
  // geometry-dependent state
  int rows = 0, cols = 0, maxF = 0, lastF = 0;
  int lw[b200::MAX_LEVELS], lh[b200::MAX_LEVELS], lpitch[b200::MAX_LEVELS];
  size_t loff[b200::MAX_LEVELS];
  size_t frame_bytes = 0;
  int xt_off[b200::MAX_LEVELS], yt_off[b200::MAX_LEVELS], xg_off[b200::MAX_LEVELS];
  b200::LevelTab ltab{};
  b200::PyrView rawv{}, blurv{};
  b200::DeviceBlock geom;   // carved for (rows, cols, maxF): every d_ array below
  int ncells = 0, slots_per_frame = 0, sel_per_frame = 0, cap = 0, qt_cap = 0;
  size_t qt_smem = 0;
  int fast_tp = 0, fast_rows_max = 0, fast_clist_cap = 0;
  size_t fast_smem = 0;
  uint8_t *d_raw = nullptr, *d_blur = nullptr;
  b200::CellDesc* d_cells = nullptr;
  unsigned* d_cand = nullptr;
  int* d_cellcnt = nullptr;
  unsigned* d_qkp = nullptr;
  int* d_qnode = nullptr;
  unsigned* d_sel = nullptr;
  int *d_selcnt = nullptr, *d_candcnt = nullptr;
  OrbxKeyPoint* d_kps = nullptr;
  uint8_t* d_desc = nullptr;
  int* d_n = nullptr;
  int2 *d_xt = nullptr, *d_yt = nullptr;
  bool resize_group_ok = true;
  int4* d_xg = nullptr;   // per 4-output group: {first source word, 8*byte phase, PRMT selectors, -} + 4 coefficient pairs
  b200::BlurTile* d_blur_tiles = nullptr;
  b200::BlurEdge* d_blur_edges = nullptr;
  int n_blur_tiles = 0, n_blur_edges = 0;
  b200::DeviceBlock tmp;    // orbx_get_level's bordered copy
  b200::HostBlock stage;    // orbx_extract_batch's downloads
  bool have_results = false;
  // optional per-stage CUDA-event timing (bench.py's roofline leg): one event set per run(), read lazily
  bool profile = false;
  std::vector<b200::StageEvents> prof_runs;

  int init(const OrbxParams& p, int dev);
  int plan_geometry(int r, int c, b200::GeomPlan& g) const;
  int ensure_geometry(int r, int c, int F);
  int run(const uint8_t* d_l0, int pitch0, size_t fstride0, int F, int f0 = 0);
  int prof_mark(int boundary);   // record event `boundary` of the current run (no-op unless profiling)
  int prof_begin(int frames);
};
