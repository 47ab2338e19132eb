// ocm.cu -- keyframe RGB-D -> point cloud -> occupancy (OctoMap log-odds) on sm_90a.
// Reference: MapDrawer::GeneratePointCloud / InsertScan / ctor params (perfect/src/MapDrawer.cc:641-675, 946-1025,
// 51-56), UpdateOctomap's sensor-origin quirk (:619,631-632), PointCloudMapping::insertKeyFrame (class surface,
// include/pointcloudmapping.h:50-56).  Third-party semantics (PCL VoxelGrid, pcl::transformPointCloud, octomap
// keys / computeRayKeys / updateNode) follow oracle/occ_ref.cpp, which states them.
//
// HBM layout:
//   leaf table   open-addressing hash of the 1-cm VoxelGrid cells of ONE keyframe (key = 3 x 21-bit cell index), one
//                16-byte record per cell: key, pixel count, position in the keyframe's cell list.  Per-cell state after
//                binning (count, bucket offset) lives in dense arrays indexed by that position.  Pixels of a cell are
//                bucketed, sorted ascending and summed sequentially in float so the centroid equals the oracle's
//                pixel-order sum bit for bit.
//   points       world-frame centroids of the last keyframe (xyz f32, rgb, ground label), unordered
//   map          persistent open-addressing hash: key (3 x u16 OcTreeKey packed in u64) -> float log-odds, colour, the
//                clamp-add summary (a, lo, hi) used by the multi-GPU merge, and the batch masks: bit j of the hit / miss
//                word = keyframe j of the running batch observed the voxel occupied / free.  The scan of ALL keyframes
//                of a batch only ORs bits (order-free, one launch); one more launch replays each touched voxel's bits in
//                keyframe order, which reproduces the sequential clamped updates exactly.
//   tree         on demand (ocm_tree_build, ocm_tree.cuh): the map as octomap's pruned ColorOcTree, 8-byte nodes in
//                pre-order plus the pruned leaves -- what an `.ot` file holds; ocm_read_ot goes the other way.
#include <algorithm>
#include <memory>
#include <new>
#include <vector>

#include <dlfcn.h>
#include <nccl.h>

#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace b200 {

constexpr unsigned long long EMPTY_KEY = ~0ull;

__device__ __forceinline__ unsigned long long hash64(unsigned long long k) {   // splitmix64 finaliser
  k ^= k >> 30; k *= 0xbf58476d1ce4e5b9ull;
  k ^= k >> 27; k *= 0x94d049bb133111ebull;
  k ^= k >> 31;
  return k;
}
// Home slot of a key in a power-of-two table.  Tables below 2^32 slots (every one in practice) take a 32-bit mix of the
// two key halves (murmur3 block + finaliser): about half the instructions of the 64-bit multiplies, and the probe is on
// the inner loop of the free-space rays (k_ocm_scan_keys: the 64-bit hash was 19 % of its instructions).
__device__ __forceinline__ long long hash_slot(unsigned long long k, long long mask) {
  if ((unsigned long long)mask >> 32) return (long long)(hash64(k) & (unsigned long long)mask);
  unsigned h = (unsigned)k * 0xcc9e2d51u;
  h = __funnelshift_l(h, h, 15) * 0x1b873593u;
  h ^= (unsigned)(k >> 32) * 0x85ebca6bu;
  h ^= h >> 16; h *= 0x85ebca6bu;
  h ^= h >> 13; h *= 0xc2b2ae35u;
  h ^= h >> 16;
  return (long long)(h & (unsigned)mask);
}

// Linear probe of a power-of-two open-addressing table whose keys lie STRIDE 8-byte words apart (1: a key array;
// sizeof(LeafRec) / 8: the key field of the leaf records).  Returns whether the key has a slot, and *slot = that slot.
// INSERT: find-or-insert (false only when the table is full), *fresh = this call created the entry.  Otherwise find
// only.  (A found flag rather than "slot or -1": the compiler cannot prove a slot non-negative, so a sign test costs
// the map's callers a compare and a select -- 32 instructions in k_ocm_scan_keys.  k_ocm_bin wants that test.)
template <int STRIDE, bool INSERT = true>
__device__ __forceinline__ bool table_probe(unsigned long long* keys, long long mask, unsigned long long key,
                                            long long* slot, bool* fresh) {
  long long s = hash_slot(key, mask);
  bool found = false;
  *fresh = false;
  for (long long probe = 0; probe <= mask; ++probe) {
    unsigned long long* p = keys + s * STRIDE;
    const unsigned long long cur = *p;
    if (cur == key) { found = true; break; }
    if (cur == EMPTY_KEY) {
      if (!INSERT) break;
      const unsigned long long old = atomicCAS(p, EMPTY_KEY, key);
      if (old == EMPTY_KEY) { *fresh = true; found = true; break; }
      if (old == key) { found = true; break; }
    }
    s = (s + 1) & mask;
  }
  *slot = s;
  return found;
}

// Error codes the kernels leave in the handle's error word (check_err turns them into messages).
constexpr int ERR_LEAF_TABLE_FULL = 1;
constexpr int ERR_MAP_FULL = 2;

struct OcmConst {
  float fx, fy, cx, cy;
  float depth_min, depth_max, y_max, inv_leaf;
  double res, res_factor;
  double Rt[9], ti[3];     // Twc = inverse of Tcw, double (pcl::transformPointCloud<.., double>)
  float origin[3];         // translation of Tcw (UpdateOctomap quirk)
  int rows, cols;
};

// One 16-byte record per VoxelGrid cell.  k_ocm_bin inserts the key and adds the pixel counts; k_ocm_ranges moves the
// count to the dense arrays, stores the cell's list position for k_ocm_scatter and empties the record for the next
// keyframe in the same 16-byte store (the stale `cell` is never read before k_ocm_ranges writes it again).
struct __align__(16) LeafRec {
  unsigned long long key;
  int count;
  int cell;      // position in the keyframe's cell list (valid from k_ocm_ranges to k_ocm_scatter)
};
static_assert(sizeof(LeafRec) == 16, "one 16-byte record per leaf");
__host__ __device__ __forceinline__ LeafRec empty_leaf() {
  LeafRec r{};
  r.key = EMPTY_KEY;
  return r;
}
struct LeafTable {
  LeafRec* rec;
  long long mask;
};

struct MapView {
  unsigned long long* keys;
  float* val;
  float *a, *lo, *hi;   // clamp-add summary since the last merge: f(x) = min(max(x + a, lo), hi)
  unsigned* rgb;
  int* nleaves;
  long long mask;
  // batch accumulation: which keyframes of the running batch hit (high word) / missed (low word) the voxel, the colour
  // of its latest hit (keyframe << 24 | rgb); k_ocm_apply finds the touched voxels by sweeping the masks
  unsigned long long* bm;
  unsigned* bm_rgb;
  // merge epochs (ocm_merge_nccl): value of the voxel at the last merge, and the list of voxels whose summary left the
  // identity since then (what this rank has to send)
  float* base;
  int* elist;
  int* nelist;
  unsigned long long* nupd;   // cumulative number of (voxel, keyframe) log-odds updates (bench.py: U of B_map)
};

// find-or-insert of a voxel, counting the voxels the map holds; false when the map is full.
__device__ __forceinline__ bool map_slot(const MapView& m, unsigned long long key, long long* s) {
  bool fresh;
  const bool found = table_probe<1>(m.keys, m.mask, key, s, &fresh);
  if (fresh) atomicAdd(m.nleaves, 1);
  return found;
}

// Record "keyframe j of the batch observed voxel `key` as occupied / free".  Order-free (atomicOr), so every keyframe
// of a batch can be scanned in one launch; k_ocm_apply replays the bits of each voxel in keyframe order.
__device__ __forceinline__ bool map_touch(const MapView& m, unsigned long long key, int j, bool occupied, unsigned rgb) {
  long long s;
  if (!map_slot(m, key, &s)) return false;
  // Fire and forget: no atomic here returns a value.  (The free-space rays used to wait on the atomicOr's old value to
  // build a list of touched voxels: 35 % of k_ocm_scan_keys' stall samples.  Dirty-block flags instead of the list were
  // worse: the hash scatters a batch over every block, and millions of flag stores / flag reads land on 64 cache lines.
  // k_ocm_apply simply sweeps the 8-byte masks of the whole table: 67 MB per batch at the default capacity.)
  const unsigned long long bit = occupied ? (1ull << (32 + j)) : (1ull << j);
  atomicOr(&m.bm[s], bit);
  if (occupied) atomicMax(&m.bm_rgb[s], ((unsigned)j << 24) | (rgb & 0xffffffu));
  return true;
}

// Everything one keyframe needs between back-projection and the map update.  A batch of keyframes runs every stage
// as ONE launch (blockIdx.y = job = bit index of the keyframe in the batch masks of the map).
struct KfScratch {
  LeafTable leaf;
  int *pix_slot, *pix_rank, *bucket;   // pix_rank: position of the pixel inside its cell's bucket
  // the keyframe's cell list (cell = position in it = point index): leaf-table slot, pixel count, bucket offset
  int *cell_slot, *cell_count, *cell_off;
  int* counters;   // [0] pixels, [1] voxels (= points)
  float* pts;
  uint8_t *pts_rgb, *pts_label;
};
struct KfJob {
  OcmConst c;
  const float* depth;
  const uint8_t* rgb;
  const uint8_t* label;
  KfScratch s;
};

__device__ __forceinline__ bool backproject(const OcmConst& c, const float* __restrict__ depth, int pix, float& x,
                                            float& y, float& z) {
  const int m = pix / c.cols, n = pix - m * c.cols;
  const float d = depth[pix];
  if (d < c.depth_min || d > c.depth_max) return false;       // MapDrawer.cc:655 (NaN fails neither test: kept like the reference)
  z = d;
  x = ((float)n - c.cx) * z / c.fx;                           // :658-659 (float, true division; --fmad=false)
  y = ((float)m - c.cy) * z / c.fy;
  if (y < -c.y_max || y > c.y_max) return false;             // :660
  return true;
}

// VoxelGrid cell of a gated point: 21 bits per axis (ocm_insert_* refuse gates and intrinsics that would let
// |coord / leaf| reach 2^20, where cells would alias).  NaN depth passes both gates (MapDrawer.cc:655 keeps it); those
// pixels share one cell of their own, NONFINITE_CELL (bit 63: no real cell has it, and it is not a sentinel of k_ocm_bin),
// instead of the cell that cvt's NaN -> 0 would give them.  Their centroid is NaN, so they never reach the map.
constexpr unsigned long long NONFINITE_CELL = 1ull << 63;
__device__ __forceinline__ unsigned long long leaf_key(const OcmConst& c, float x, float y, float z) {
  if (!(isfinite(x) && isfinite(y) && isfinite(z))) return NONFINITE_CELL;
  const long long ix = (long long)floorf(x * c.inv_leaf) + (1 << 20);
  const long long iy = (long long)floorf(y * c.inv_leaf) + (1 << 20);
  const long long iz = (long long)floorf(z * c.inv_leaf) + (1 << 20);
  return (unsigned long long)(ix & 0x1fffff) | ((unsigned long long)(iy & 0x1fffff) << 21) |
         ((unsigned long long)(iz & 0x1fffff) << 42);
}

// K11a: gate + VoxelGrid cell of every pixel, binned per CTA tile of BIN_TW x BIN_TH pixels (one thread per pixel, one
// warp per tile row).  The tile's distinct cells are deduplicated in shared memory, and each (tile, cell) makes the only
// global accesses of the tile for that cell: one find-or-insert probe of the leaf table and one atomicAdd of its pixel
// count, whose return value is the tile's first position in the cell's bucket.  New cells are appended to the cell list
// with one atomicAdd per CTA.  Inside the tile, the positions follow ascending pixel index (rows of the tile in order,
// lanes in order), so a cell's bucket is a few ascending runs.  32 x 16 rather than 32 x 8: k_ocm_bin itself costs the
// same with either, but the cell list is appended tile by tile, so taller tiles hand k_ocm_scan_keys points that lie
// closer together and its free-cell cache hits more often (one bench step's insert 16.7 against 17.4 ms, H100 80 GB
// HBM3 at 700 W).
constexpr int BIN_TW = 32, BIN_TH = 16, BIN_THREADS = BIN_TW * BIN_TH;
// The shared table has twice as many entries as the tile has pixels: it cannot fill up, even when every pixel is its own
// cell.
constexpr int BIN_SLOTS = 2 * BIN_THREADS;
static_assert(BIN_TW == 32 && BIN_TH <= 16, "a tile row is one warp; the per-row counts of a cell are 16 bytes");

__device__ __forceinline__ int bytes_sum(unsigned w) { return (int)__dp4a(w, 0x01010101u, 0u); }

__global__ void __launch_bounds__(BIN_THREADS) k_ocm_bin(const KfJob* __restrict__ jobs, int* __restrict__ err) {
  __shared__ unsigned long long s_key[BIN_SLOTS];
  __shared__ uint4 s_rows[BIN_SLOTS];     // byte r: pixels of the cell in tile row r
  __shared__ int s_slot[BIN_SLOTS], s_base[BIN_SLOTS];
  __shared__ int s_fresh, s_fresh_base;
  const KfJob& J = jobs[blockIdx.y];
  const OcmConst& c = J.c;
  const LeafTable lt = J.s.leaf;
  for (int i = threadIdx.x; i < BIN_SLOTS; i += BIN_THREADS) {
    s_key[i] = EMPTY_KEY;
    s_rows[i] = make_uint4(0u, 0u, 0u, 0u);
  }
  if (threadIdx.x == 0) s_fresh = 0;
  const int lane = threadIdx.x & 31, row = threadIdx.x >> 5;
  const int tiles_x = (c.cols + BIN_TW - 1) / BIN_TW;
  const int ty = blockIdx.x / tiles_x, tx = blockIdx.x - ty * tiles_x;
  const int px = tx * BIN_TW + lane, py = ty * BIN_TH + row;
  const int pix = (px < c.cols && py < c.rows) ? py * c.cols + px : -1;
  float x, y, z;
  const bool ok = pix >= 0 && backproject(c, J.depth, pix, x, y, z);
  const unsigned long long key = ok ? leaf_key(c, x, y, z) : EMPTY_KEY;
  const unsigned grp = __match_any_sync(0xffffffffu, key);
  const int leader = __ffs(grp) - 1;       // lowest lane of the group = smallest pixel of the cell in this row
  const bool lead = ok && lane == leader;
  __syncthreads();
  int ls = 0;                              // the cell's entry in the shared table
  if (lead) {
    ls = (int)hash_slot(key, BIN_SLOTS - 1);
    for (;;) {
      const unsigned long long old = atomicCAS(&s_key[ls], EMPTY_KEY, key);
      if (old == EMPTY_KEY || old == key) break;
      ls = (ls + 1) & (BIN_SLOTS - 1);
    }
    reinterpret_cast<unsigned char*>(&s_rows[ls])[row] = (unsigned char)__popc(grp);
  }
  __syncthreads();
  int before = 0, slot = -1, pos = -1;     // before: pixels of the cell in the rows above
  if (lead) {
    const uint4 r = s_rows[ls];
    const unsigned w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = row - 4 * i;           // bytes of word i that belong to rows above this one
      before += bytes_sum(k <= 0 ? 0u : (k >= 4 ? w[i] : w[i] & ((1u << (8 * k)) - 1u)));
    }
    if (before == 0) {                     // first row of the cell in the tile: the tile's one global probe for it
      const int total = bytes_sum(r.x) + bytes_sum(r.y) + bytes_sum(r.z) + bytes_sum(r.w);
      bool fresh;
      long long s;
      if (!table_probe<sizeof(LeafRec) / 8>(&lt.rec->key, lt.mask, key, &s, &fresh)) {
        atomicExch(err, ERR_LEAF_TABLE_FULL);
        s_slot[ls] = -1;
        s_base[ls] = 0;
      } else {
        slot = (int)s;
        s_slot[ls] = slot;
        s_base[ls] = atomicAdd(&lt.rec[s].count, total);
        if (fresh) pos = atomicAdd(&s_fresh, 1);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_fresh) s_fresh_base = atomicAdd(&J.s.counters[1], s_fresh);
  __syncthreads();
  if (pos >= 0) J.s.cell_slot[s_fresh_base + pos] = slot;
  int rank = 0;
  if (lead) {
    slot = s_slot[ls];
    rank = s_base[ls] + before;
  }
  slot = __shfl_sync(0xffffffffu, slot, leader);
  rank = __shfl_sync(0xffffffffu, rank, leader) + __popc(grp & ((1u << lane) - 1u));
  if (pix >= 0) {
    J.s.pix_slot[pix] = ok ? slot : -1;
    J.s.pix_rank[pix] = rank;
  }
}

// K11b: bucket ranges of the cells in list order (the cloud is a set, so any order would do): a block scan of the
// counts and one atomicAdd per CTA and round.  Moves each cell's count into the dense arrays and empties its leaf record,
// leaving only the cell's list position there for k_ocm_scatter.
constexpr int RANGES_THREADS = 256;
__global__ void __launch_bounds__(RANGES_THREADS) k_ocm_ranges(const KfJob* __restrict__ jobs) {
  using Scan = cub::BlockScan<int, RANGES_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int s_base;
  const KfJob& J = jobs[blockIdx.y];
  LeafRec* __restrict__ rec = J.s.leaf.rec;
  const int n = J.s.counters[1];
  for (int v0 = blockIdx.x * RANGES_THREADS; v0 < n; v0 += gridDim.x * RANGES_THREADS) {
    const int v = v0 + threadIdx.x;
    int s = 0, cnt = 0;
    if (v < n) {
      s = J.s.cell_slot[v];
      cnt = rec[s].count;
    }
    int off, total;
    Scan(tmp).ExclusiveSum(cnt, off, total);
    if (threadIdx.x == 0) s_base = atomicAdd(&J.s.counters[0], total);
    __syncthreads();
    if (v < n) {
      J.s.cell_count[v] = cnt;
      J.s.cell_off[v] = s_base + off;
      LeafRec r = empty_leaf();
      r.cell = v;
      rec[s] = r;
    }
    __syncthreads();   // tmp and s_base are reused by the next round
  }
}

// K11c: scatter the pixel indices into their cell's bucket
__global__ void k_ocm_scatter(const KfJob* __restrict__ jobs) {
  const KfJob& J = jobs[blockIdx.y];
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= J.c.rows * J.c.cols) return;
  const int s = J.s.pix_slot[pix];
  if (s >= 0) J.s.bucket[J.s.cell_off[J.s.leaf.rec[s].cell] + J.s.pix_rank[pix]] = pix;   // ranks come from k_ocm_bin
}

// K11d: per cell: restore pixel order, sequential float centroid (PCL VoxelGrid), transform to the world frame in
// double (pcl::transformPointCloud), emit the point.  The label is that of the cell's smallest pixel.
__global__ void k_ocm_centroids(const KfJob* __restrict__ jobs) {
  const KfJob& J = jobs[blockIdx.y];
  const OcmConst& c = J.c;
  const float* __restrict__ depth = J.depth;
  const uint8_t* __restrict__ rgb = J.rgb;
  const uint8_t* __restrict__ label = J.label;
  const int* __restrict__ cell_count = J.s.cell_count;
  const int* __restrict__ cell_off = J.s.cell_off;
  int* __restrict__ bucket = J.s.bucket;
  float* __restrict__ pts = J.s.pts;
  uint8_t* __restrict__ pts_rgb = J.s.pts_rgb;
  uint8_t* __restrict__ pts_label = J.s.pts_label;
  const int ncells = J.s.counters[1];
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < ncells; v += gridDim.x * blockDim.x) {
    const int n = cell_count[v];
    int* b = bucket + cell_off[v];
    for (int i = 1; i < n; ++i) {   // insertion sort: ascending pixel index = row-major order
      const int val = b[i];
      int j = i - 1;
      while (j >= 0 && b[j] > val) { b[j + 1] = b[j]; --j; }
      b[j + 1] = val;
    }
    float sx = 0.f, sy = 0.f, sz = 0.f, sr = 0.f, sg = 0.f, sb = 0.f;
    for (int i = 0; i < n; ++i) {
      float x, y, z;
      backproject(c, depth, b[i], x, y, z);
      sx += x; sy += y; sz += z;
      const uint8_t* col = rgb + (size_t)b[i] * 3;   // b,g,r (cv::Mat BGR)
      sr += (float)col[2]; sg += (float)col[1]; sb += (float)col[0];
    }
    const float fn = (float)n;
    const double px = (double)(sx / fn), py = (double)(sy / fn), pz = (double)(sz / fn);
#pragma unroll
    for (int i = 0; i < 3; ++i)
      pts[(size_t)v * 3 + i] = (float)(c.Rt[i * 3 + 0] * px + c.Rt[i * 3 + 1] * py + c.Rt[i * 3 + 2] * pz + c.ti[i]);
    pts_rgb[(size_t)v * 3 + 0] = (uint8_t)(sr / fn);
    pts_rgb[(size_t)v * 3 + 1] = (uint8_t)(sg / fn);
    pts_rgb[(size_t)v * 3 + 2] = (uint8_t)(sb / fn);
    pts_label[v] = label ? label[b[0]] : 0;
  }
}

// leaf <= 0: no VoxelGrid; every gated pixel is a point (used for the T-variant style clouds)
__global__ void k_ocm_points_nofilter(const KfJob* __restrict__ jobs) {
  const KfJob& J = jobs[blockIdx.y];
  const OcmConst& c = J.c;
  const float* __restrict__ depth = J.depth;
  const uint8_t* __restrict__ rgb = J.rgb;
  const uint8_t* __restrict__ label = J.label;
  int* __restrict__ counters = J.s.counters;
  float* __restrict__ pts = J.s.pts;
  uint8_t* __restrict__ pts_rgb = J.s.pts_rgb;
  uint8_t* __restrict__ pts_label = J.s.pts_label;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= c.rows * c.cols) return;
  float x, y, z;
  if (!backproject(c, depth, pix, x, y, z)) return;
  const int v = atomicAdd(&counters[1], 1);
  const double px = x, py = y, pz = z;
#pragma unroll
  for (int i = 0; i < 3; ++i)
    pts[(size_t)v * 3 + i] = (float)(c.Rt[i * 3 + 0] * px + c.Rt[i * 3 + 1] * py + c.Rt[i * 3 + 2] * pz + c.ti[i]);
  const uint8_t* col = rgb + (size_t)pix * 3;
  pts_rgb[(size_t)v * 3 + 0] = col[2]; pts_rgb[(size_t)v * 3 + 1] = col[1]; pts_rgb[(size_t)v * 3 + 2] = col[0];
  pts_label[v] = label ? label[pix] : 0;
}

// coordToKeyChecked.  The range test is made on the double, before the conversion: a non-finite coordinate never makes a
// key (cvt turns NaN into 0, which would be the in-range key 32768, and +-inf into INT_MAX / INT_MIN).
__device__ __forceinline__ bool coord_to_key(const OcmConst& c, float coord, int& k) {
  const double f = floor(c.res_factor * (double)coord);
  k = (int)f + 32768;
  return f >= -32768.0 && f < 32768.0;
}
__device__ __forceinline__ unsigned long long pack_key(int kx, int ky, int kz) {
  return (unsigned long long)kx | ((unsigned long long)ky << 16) | ((unsigned long long)kz << 32);
}

// K12/K13: per point -> occupied endpoint key, or (ground) the free cells along the ray (computeRayKeys); the
// observations go straight into the map's batch masks (bit = keyframe).
// Free-space rays of neighbouring ground points run through the same cells for most of their length (they share the
// origin), and a miss is idempotent inside one keyframe (atomicOr of the same bit): every CTA keeps a small direct-mapped
// cache of the free cells it has already reported and skips the repeats -- the global hash probes + atomics were the whole
// kernel (long-scoreboard bound), most of them redundant.
constexpr int SCAN_CACHE = 2048;
__device__ __forceinline__ bool scan_touch_free(const MapView& m, unsigned long long* seen, unsigned long long key, int j) {
  const unsigned h = ((unsigned)key * 73856093u ^ (unsigned)(key >> 16) * 19349663u ^ (unsigned)(key >> 32) * 83492791u) &
                     (SCAN_CACHE - 1);
  if (seen[h] == key) return true;
  seen[h] = key;   // benign race: at worst a repeat reaches the map
  return map_touch(m, key, j, false, 0u);
}

__device__ __forceinline__ void scan_point(const KfJob& J, const MapView& m, unsigned long long* s_seen, int j, int v,
                                           bool all_ground, int* __restrict__ err) {
  const OcmConst& c = J.c;
  const float* __restrict__ pts = J.s.pts;
  const uint8_t* __restrict__ pts_label = J.s.pts_label;
  const uint8_t* __restrict__ pts_rgb = J.s.pts_rgb;
  const float e[3] = {pts[(size_t)v * 3], pts[(size_t)v * 3 + 1], pts[(size_t)v * 3 + 2]};
  int ke[3];
  const bool end_ok = coord_to_key(c, e[0], ke[0]) && coord_to_key(c, e[1], ke[1]) && coord_to_key(c, e[2], ke[2]);
  if (!pts_label[v] && !all_ground) {
    if (end_ok) {
      const unsigned rgb = (unsigned)pts_rgb[(size_t)v * 3] | ((unsigned)pts_rgb[(size_t)v * 3 + 1] << 8) |
                           ((unsigned)pts_rgb[(size_t)v * 3 + 2] << 16);
      if (!map_touch(m, pack_key(ke[0], ke[1], ke[2]), j, true, rgb)) atomicExch(err, ERR_MAP_FULL);
    }
    return;
  }
  int ko[3];
  if (!end_ok || !coord_to_key(c, c.origin[0], ko[0]) || !coord_to_key(c, c.origin[1], ko[1]) ||
      !coord_to_key(c, c.origin[2], ko[2]))
    return;
  if (ko[0] == ke[0] && ko[1] == ke[1] && ko[2] == ke[2]) return;
  if (!scan_touch_free(m, s_seen, pack_key(ko[0], ko[1], ko[2]), j)) atomicExch(err, ERR_MAP_FULL);
  float dir[3] = {e[0] - c.origin[0], e[1] - c.origin[1], e[2] - c.origin[2]};
  // octomath::Vector3::norm() of octomap 1.9.x: norm_sq() = x*x + y*y + z*z in float, widened for the sqrt only
  const float n2 = __fadd_rn(__fadd_rn(__fmul_rn(dir[0], dir[0]), __fmul_rn(dir[1], dir[1])), __fmul_rn(dir[2], dir[2]));
  const float length = (float)sqrt((double)n2);
#pragma unroll
  for (int i = 0; i < 3; ++i) dir[i] = dir[i] / length;
  int step[3], cur[3] = {ko[0], ko[1], ko[2]};
  double tMax[3], tDelta[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    step[i] = (dir[i] > 0.f) ? 1 : ((dir[i] < 0.f) ? -1 : 0);
    if (step[i] != 0) {
      double border = ((double)(cur[i] - 32768) + 0.5) * c.res;
      border += (double)(float)((double)step[i] * c.res * 0.5);
      tMax[i] = (border - (double)c.origin[i]) / (double)dir[i];
      tDelta[i] = c.res / fabs((double)dir[i]);
    } else {
      tMax[i] = 1.7976931348623157e308;
      tDelta[i] = 1.7976931348623157e308;
    }
  }
  // computeRayKeys' loop (octomap OcTreeBaseImpl.hxx:  step along the axis of the smallest tMax; stop at the end key;
  // stop when min(tMax) after the step exceeds the ray length; else the cell is free).  min(tMax) after a step IS the
  // tMax of the axis the next step takes, so the distance test of cell k rides on the axis selection of step k+1 and
  // the cell is reported one iteration late (`pending`): no separate three-way double minimum per cell.
  bool pending = false;
  unsigned long long pending_key = 0ull;
  const double dlen = (double)length;
  for (int guard = 0; guard < 3 * 65536; ++guard) {
    const bool a01 = tMax[0] < tMax[1];
    const double t01 = a01 ? tMax[0] : tMax[1];
    const bool a2 = t01 < tMax[2];            // (tMax[0] < tMax[2]) or (tMax[1] < tMax[2]), whichever axis leads
    const double tmin = a2 ? t01 : tMax[2];
    if (pending) {
      if (tmin > dlen) break;
      if (!scan_touch_free(m, s_seen, pending_key, j)) { atomicExch(err, ERR_MAP_FULL); break; }
    }
    const bool d0 = a2 && a01, d1 = a2 && !a01, d2 = !a2;
    // (no dynamic register indexing, no branches: predicated updates)
    cur[0] = d0 ? ((cur[0] + step[0]) & 0xffff) : cur[0];
    cur[1] = d1 ? ((cur[1] + step[1]) & 0xffff) : cur[1];
    cur[2] = d2 ? ((cur[2] + step[2]) & 0xffff) : cur[2];
    tMax[0] = d0 ? tMax[0] + tDelta[0] : tMax[0];
    tMax[1] = d1 ? tMax[1] + tDelta[1] : tMax[1];
    tMax[2] = d2 ? tMax[2] + tDelta[2] : tMax[2];
    if (cur[0] == ke[0] && cur[1] == ke[1] && cur[2] == ke[2]) break;
    pending = true;
    pending_key = pack_key(cur[0], cur[1], cur[2]);
  }
}

__global__ void __launch_bounds__(256) k_ocm_scan_keys(const KfJob* __restrict__ jobs, MapView m, int* __restrict__ err) {
  __shared__ unsigned long long s_seen[SCAN_CACHE];
  for (int i = threadIdx.x; i < SCAN_CACHE; i += blockDim.x) s_seen[i] = EMPTY_KEY;
  __syncthreads();
  const int j = blockIdx.y;
  const KfJob& J = jobs[j];
  const int n = J.s.counters[1];
  // perfect/src/MapDrawer.cc:676-680: a cloud of fewer than 50 points skips the plane extraction and is ALL ground
  const bool all_ground = n < 50;
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x)
    scan_point(J, m, s_seen, j, v, all_ground, err);
}

// K14: replay, voxel by voxel, the observations of the batch in keyframe order (MapDrawer.cc:1007-1022 per keyframe:
// free \ occupied get a miss, occupied get a hit; updateNodeLogOdds clamps after every add, so the order matters and
// is kept).  Grid-stride sweep over the batch masks of the whole table (16-byte loads); the masks of the voxels found
// are cleared for the next batch.
__device__ __forceinline__ int apply_slot(const MapView& m, long long s, unsigned long long w, float hit_log, float miss_log,
                                          float cmin, float cmax) {
  m.bm[s] = 0ull;
  const unsigned hit = (unsigned)(w >> 32), miss = (unsigned)w & ~hit;
  float v = m.val[s], a = m.a[s], lo = m.lo[s], hi = m.hi[s];
  if (a == 0.f && lo == -INFINITY) m.elist[atomicAdd(m.nelist, 1)] = (int)s;   // first update of this merge epoch
  unsigned all = hit | miss;
  const int nup = __popc(all);
  while (all) {
    const int j = __ffs(all) - 1;
    all &= all - 1u;
    const float d = ((hit >> j) & 1u) ? hit_log : miss_log;
    v = fminf(fmaxf(v + d, cmin), cmax);
    a = a + d;
    lo = fminf(fmaxf(lo + d, cmin), cmax);
    hi = fminf(fmaxf(hi + d, cmin), cmax);
  }
  m.val[s] = v; m.a[s] = a; m.lo[s] = lo; m.hi[s] = hi;
  if (hit) { m.rgb[s] = (m.bm_rgb[s] & 0xffffffu) | 0x01000000u; m.bm_rgb[s] = 0u; }   // top byte 1: coloured this epoch
  return nup;
}

__global__ void k_ocm_apply(float hit_log, float miss_log, float cmin, float cmax, MapView m) {
  const long long C = m.mask + 1;   // power of two >= 2
  const ulonglong2* __restrict__ bm2 = reinterpret_cast<const ulonglong2*>(m.bm);
  int nup = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < C / 2; i += (long long)gridDim.x * blockDim.x) {
    const ulonglong2 w = bm2[i];
    if (w.x) nup += apply_slot(m, 2 * i, w.x, hit_log, miss_log, cmin, cmax);
    if (w.y) nup += apply_slot(m, 2 * i + 1, w.y, hit_log, miss_log, cmin, cmax);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nup += __shfl_xor_sync(0xffffffffu, nup, o);
  if ((threadIdx.x & 31) == 0 && nup) atomicAdd(m.nupd, (unsigned long long)nup);
}

template <class T>
__global__ void k_ocm_fill(T* p, T v, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// export: compact the map's leaves into dense arrays
__global__ void k_ocm_export(MapView m, long long* __restrict__ counter, long long cap, unsigned short* __restrict__ keys3,
                             float* __restrict__ val, unsigned char* __restrict__ rgb) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > m.mask) return;
  const unsigned long long k = m.keys[i];
  if (k == EMPTY_KEY) return;
  const long long o = (long long)atomicAdd((unsigned long long*)counter, 1ull);
  if (o >= cap) return;
  keys3[o * 3] = (unsigned short)(k & 0xffff); keys3[o * 3 + 1] = (unsigned short)((k >> 16) & 0xffff); keys3[o * 3 + 2] = (unsigned short)((k >> 32) & 0xffff);
  val[o] = m.val[i];
  const unsigned c = m.rgb[i];
  rgb[o * 3] = c & 0xff; rgb[o * 3 + 1] = (c >> 8) & 0xff; rgb[o * 3 + 2] = (c >> 16) & 0xff;
}

// ---- epoch merge (ocm_merge_nccl) -------------------------------------------------------------------------------------
// One shard = SoA records {key u64, a, lo, hi f32, rgb u32} of the voxels a rank updated since the last merge (24 B each).
struct MergeShard {
  unsigned long long* keys;
  float *a, *lo, *hi;
  unsigned* rgb;
};
__host__ __device__ inline MergeShard merge_shard_at(void* region, long long n) {
  MergeShard r;
  char* p = (char*)region;
  r.keys = (unsigned long long*)p; p += 8 * n;
  r.a = (float*)p; p += 4 * n;
  r.lo = (float*)p; p += 4 * n;
  r.hi = (float*)p; p += 4 * n;
  r.rgb = (unsigned*)p;
  return r;
}
// pack this rank's epoch summaries and roll its own voxels back to the value of the last merge: afterwards EVERY rank
// replays ALL shards (its own included) in rank order on the same base values, so all ranks end with identical maps
__global__ void k_merge_pack(MapView m, int n, MergeShard o) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = m.elist[i];
  o.keys[i] = m.keys[s];
  o.a[i] = m.a[s]; o.lo[i] = m.lo[s]; o.hi[i] = m.hi[s];
  const unsigned c = m.rgb[s];
  const bool fresh = (c >> 24) == 1u;
  o.rgb[i] = fresh ? (c & 0xffffffu) : 0xffffffffu;
  if (fresh) m.rgb[s] = c & 0xffffffu;
  m.val[s] = m.base[s];
  m.a[s] = 0.f; m.lo[s] = -INFINITY; m.hi[s] = INFINITY;
}
// apply one shard: v <- min(max(v + a, lo), hi) per voxel (keys of a shard are distinct; shards run as consecutive launches)
__global__ void k_merge_apply(MapView m, long long n, MergeShard g, int* __restrict__ slots, int* __restrict__ err) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long s;
  if (!map_slot(m, g.keys[i], &s)) { atomicExch(err, ERR_MAP_FULL); slots[i] = -1; return; }
  m.val[s] = fminf(fmaxf(m.val[s] + g.a[i], g.lo[i]), g.hi[i]);
  const unsigned c = g.rgb[i];
  if (c != 0xffffffffu) m.rgb[s] = c;
  slots[i] = (int)s;
}
__global__ void k_merge_commit(MapView m, long long n, const int* __restrict__ slots) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = slots[i];
  if (s >= 0) m.base[s] = m.val[s];
}

__global__ void k_ocm_query(MapView m, unsigned long long key, float* out, int* found) {
  bool fresh;
  long long s;
  const bool f = table_probe<1, false>(m.keys, m.mask, key, &s, &fresh);
  *found = f;
  *out = f ? m.val[s] : 0.f;
}

// imDepth.convertTo(CV_32F, mDepthMapFactor) (src/Tracking.cc:366-367): float(u16) * factor, 4 pixels per thread
__global__ void k_depth_u16_to_f32(const ushort4* __restrict__ src, float4* __restrict__ dst, float factor, size_t n4) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const ushort4 v = src[i];
  dst[i] = make_float4(__fmul_rn((float)v.x, factor), __fmul_rn((float)v.y, factor), __fmul_rn((float)v.z, factor),
                       __fmul_rn((float)v.w, factor));
}

}  // namespace b200

#include "ocm_tree.cuh"

using namespace b200;

struct ocm {
  OcmParams prm{};
  int device = 0;
  int sms = 1;
  Stream stream;
  long long launches = 0;
  float hit_log, miss_log, cmin, cmax;
  // the map and the handle's device words: one allocation (take_block)
  DeviceBlock block;
  MapView map{};
  long long map_cap = 0;
  static constexpr int MAX_SLOTS = 32;
  int* d_counters = nullptr;          // 4 ints per slot
  int* d_err = nullptr;               // ERR_* of the last failing kernel, 0 = none
  long long* d_export_counter = nullptr;
  float* d_query_val = nullptr;       // k_ocm_query's result
  int* d_query_found = nullptr;
  // per-keyframe scratch: one slot per keyframe of a batch, one allocation each (grown on demand, self-cleaning
  // between uses)
  int rows = 0, cols = 0;
  struct Slot {
    DeviceBlock block;
    KfScratch k;
  };
  std::vector<Slot> slots;
  static constexpr int JOB_RING = 8;
  DeviceBlock jobs_d;                 // device copy of the running batch, JOB_RING batches deep
  HostBlock jobs_h;                   // page-locked staging of the same
  KfJob *d_jobs = nullptr, *h_jobs = nullptr;
  Event job_ev[JOB_RING];
  int job_head = 0;
  int last_slot = 0;
  // staging of the host-buffer inserts
  DeviceBlock stage;
  uint16_t* st_d16 = nullptr;         // ocm_insert_keyframes_u16_labeled only
  float* st_depth = nullptr;
  uint8_t *st_rgb = nullptr, *st_label = nullptr;
  DeviceBlock exp;                    // ocm_export_leaves' outputs
  // ocm_merge_nccl: the count of every rank (device and page-locked), then the send, receive and slot buffers
  DeviceBlock mg_counts;
  HostBlock mg_counts_h;
  DeviceBlock mg;
  Event mg_ev[2];                     // orders the merge after the caller's stream, and the caller's stream after it
  // ocm_tree_build: per-cell workspace, and the tree of the last build (tree_nodes < 0: none yet)
  DeviceBlock tree_ws, tree_res;
  TreeWork tw{};
  TreeOut tree{};
  long long tree_nodes = -1, tree_leaves = 0;
  DeviceBlock load;                   // ocm_read_ot's leaves

  // Every array 256-byte aligned by the Carver (k_ocm_apply reads bm in 16-byte words).
  void take_block(Carver& c) {
    const long long C = map_cap;
    map.keys = c.take<unsigned long long>(C); map.val = c.take<float>(C); map.a = c.take<float>(C);
    map.lo = c.take<float>(C); map.hi = c.take<float>(C); map.rgb = c.take<unsigned>(C); map.nleaves = c.take<int>(1);
    map.bm = c.take<unsigned long long>(C); map.bm_rgb = c.take<unsigned>(C); map.base = c.take<float>(C);
    map.elist = c.take<int>(C); map.nelist = c.take<int>(1); map.nupd = c.take<unsigned long long>(1);
    d_counters = c.take<int>(4 * MAX_SLOTS); d_err = c.take<int>(1); d_export_counter = c.take<long long>(1);
    d_query_val = c.take<float>(1); d_query_found = c.take<int>(1);
  }
  template <class T>
  void fill(T* p, T v, long long n) {
    k_ocm_fill<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p, v, n);
    ++launches;
  }
  int ensure_scratch(int r, int c, int nslots = 1);
  int ensure_staging(size_t npix);
  int insert_batch(int n, const float* const* dd, const uint8_t* const* drgb, const uint8_t* const* dlabel, int r, int c,
                   const float* Tcw, float fx, float fy, float cx, float cy);
  int insert(const float* dd, const uint8_t* drgb, const uint8_t* dlabel, int r, int c, const float* Tcw, float fx,
             float fy, float cx, float cy) {
    return insert_batch(1, &dd, &drgb, &dlabel, r, c, Tcw, fx, fy, cx, cy);
  }
  // CTAs per keyframe of the kernels that loop over a keyframe's cells (k_ocm_ranges, k_ocm_centroids,
  // k_ocm_scan_keys, 256 threads each): the cell count is only known on the device, so the grid is fixed --
  // CELL_CTAS_PER_SM per SM, shared by the B keyframes of the launch -- and each CTA loops over the cells.
  static constexpr int CELL_CTAS_PER_SM = 8;
  unsigned cell_ctas(int B) const { return (unsigned)std::max(1, (CELL_CTAS_PER_SM * sms + B - 1) / B); }
  int check_err();
  int clear_map();
  int scan(unsigned long long* data, int n);
  int build_tree();
  int read_ot(const uint8_t* bytes, int64_t n);
};

static long long pow2_at_least(long long v) {
  long long p = 1;
  while (p < v) p <<= 1;
  return p;
}

int ocm::ensure_scratch(int r, int c, int nslots) {
  if (r != rows || c != cols) {
    B200_CUDA(cudaStreamSynchronize(stream));
    slots.clear();
    rows = r; cols = c;
  }
  nslots = std::min(std::max(nslots, 1), (int)MAX_SLOTS);
  B200_CHECK(jobs_d.reserve(stream, [&](Carver& t) { d_jobs = t.take<KfJob>(MAX_SLOTS * JOB_RING); }));
  B200_CHECK(jobs_h.reserve(stream, [&](Carver& t) { h_jobs = t.take<KfJob>(MAX_SLOTS * JOB_RING); }));
  const long long npix = (long long)r * c;
  const long long leaf_cap = pow2_at_least(2 * npix);
  while ((int)slots.size() < nslots) {
    Slot s;
    KfScratch& k = s.k;
    B200_CHECK(s.block.carve(stream, [&](Carver& t) {
      k.leaf.rec = t.take<LeafRec>(leaf_cap);
      k.pix_slot = t.take<int>(npix); k.pix_rank = t.take<int>(npix); k.bucket = t.take<int>(npix);
      k.cell_slot = t.take<int>(npix); k.cell_count = t.take<int>(npix); k.cell_off = t.take<int>(npix);
      k.pts = t.take<float>(3 * npix); k.pts_rgb = t.take<uint8_t>(3 * npix); k.pts_label = t.take<uint8_t>(npix);
    }));
    k.leaf.mask = leaf_cap - 1;
    k.counters = d_counters + 4 * slots.size();
    fill(k.leaf.rec, empty_leaf(), leaf_cap);
    B200_CUDA(cudaGetLastError());
    slots.push_back(std::move(s));
  }
  return B200ORB_OK;
}

int ocm::ensure_staging(size_t npix) {
  return stage.reserve(stream, [&](Carver& t) {
    st_d16 = t.take<uint16_t>(npix); st_depth = t.take<float>(npix); st_rgb = t.take<uint8_t>(3 * npix);
    st_label = t.take<uint8_t>(npix);
  });
}

int ocm::check_err() {
  int e = 0;
  B200_CUDA(cudaMemcpyAsync(&e, d_err, 4, cudaMemcpyDeviceToHost, stream));
  B200_CUDA(cudaStreamSynchronize(stream));
  if (e) {
    B200_CUDA(cudaMemsetAsync(d_err, 0, 4, stream));
    set_error("occupancy insert: %s",
              e == ERR_LEAF_TABLE_FULL ? "VoxelGrid table full" : "map full (raise OcmParams.map_capacity)");
    return B200ORB_ECAP;
  }
  return B200ORB_OK;
}

// The empty map: no voxel, every clamp-add summary at the identity, no batch mask, the handle's device words zero.
int ocm::clear_map() {
  const long long C = map_cap;
  B200_CUDA(cudaMemsetAsync(block.p, 0, block.bytes, stream));
  fill(map.keys, EMPTY_KEY, C); fill(map.lo, -INFINITY, C); fill(map.hi, INFINITY, C);
  B200_CUDA(cudaMemsetAsync(map.rgb, 0xff, 4 * C, stream));
  return B200ORB_OK;
}

// The VoxelGrid cell key holds 21 bits per axis (leaf_key): distinct cells alias once |coord / leaf| reaches 2^20, so
// gates and intrinsics that allow it are refused.  Float rounding is monotonic, so the largest |coord * inv_leaf| a gated
// pixel can produce is the one of the outermost pixel column / row at the largest |depth|, computed here with the same
// float operations as backproject() and leaf_key().  (A NaN gate lets every depth through: refused as well.)
static int check_leaf_range(const OcmParams& p, int rows, int cols, float fx, float fy, float cx, float cy) {
  if (!(p.leaf > 0)) return B200ORB_OK;   // no VoxelGrid
  const float inv_leaf = 1.0f / p.leaf;
  const float z = std::isnan(p.depth_min) || std::isnan(p.depth_max) ? INFINITY
                                                                     : std::max(std::fabs(p.depth_min), std::fabs(p.depth_max));
  auto reach = [z](int last, float c, float f) {   // max over pixel index 0..last of |(n - c) * z / f|
    return std::max(std::fabs((0.f - c) * z / f), std::fabs(((float)last - c) * z / f));
  };
  const float b[3] = {reach(cols - 1, cx, fx) * inv_leaf, std::min(reach(rows - 1, cy, fy), std::fabs(p.y_max)) * inv_leaf,
                      z * inv_leaf};
  if (!(b[0] < 1048576.f && b[1] < 1048576.f && b[2] < 1048576.f)) {
    set_error("occupancy insert: |coord / leaf| can reach (%g, %g, %g); the VoxelGrid cell key needs it below 2^20 "
              "(lower depth_max / y_max or raise leaf)", b[0], b[1], b[2]);
    return B200ORB_EINVAL;
  }
  return B200ORB_OK;
}

// n keyframes (insertion order = array order), up to MAX_SLOTS per round of launches: every stage is one launch for
// the whole round, including the map update (per-voxel replay of the round's observations in keyframe order).
int ocm::insert_batch(int n, const float* const* dd, const uint8_t* const* drgb, const uint8_t* const* dlabel, int r, int c,
                      const float* Tcw_all, float fx, float fy, float cx, float cy) {
  B200_CHECK(check_leaf_range(prm, r, c, fx, fy, cx, cy));
  B200_CHECK(ensure_scratch(r, c, n));
  const int npix = r * c;
  for (int b0 = 0; b0 < n; b0 += (int)slots.size()) {
    const int B = std::min((int)slots.size(), n - b0);
    const int ring = job_head;
    job_head = (job_head + 1) % JOB_RING;
    B200_CUDA(cudaEventSynchronize(job_ev[ring]));   // the batch that used this staging entry has been uploaded
    KfJob* hj = h_jobs + (size_t)ring * MAX_SLOTS;
    KfJob* dj = d_jobs + (size_t)ring * MAX_SLOTS;
    for (int j = 0; j < B; ++j) {
      const float* Tcw = Tcw_all + 16 * (b0 + j);
      KfJob& J = hj[j];
      OcmConst& k = J.c;
      memset(&k, 0, sizeof(k));
      k.fx = fx; k.fy = fy; k.cx = cx; k.cy = cy;
      k.depth_min = prm.depth_min; k.depth_max = prm.depth_max; k.y_max = prm.y_max;
      k.inv_leaf = prm.leaf > 0 ? 1.0f / prm.leaf : 0.f;
      k.res = prm.resolution; k.res_factor = 1.0 / prm.resolution;
      double R[9], t[3];
      for (int i = 0; i < 3; ++i) { for (int q = 0; q < 3; ++q) R[i * 3 + q] = (double)Tcw[i * 4 + q]; t[i] = (double)Tcw[i * 4 + 3]; }
      for (int i = 0; i < 3; ++i) {
        for (int q = 0; q < 3; ++q) k.Rt[i * 3 + q] = R[q * 3 + i];
        k.ti[i] = -(R[0 * 3 + i] * t[0] + R[1 * 3 + i] * t[1] + R[2 * 3 + i] * t[2]);
      }
      k.origin[0] = Tcw[3]; k.origin[1] = Tcw[7]; k.origin[2] = Tcw[11];
      k.rows = r; k.cols = c;
      J.depth = dd[b0 + j]; J.rgb = drgb[b0 + j]; J.label = dlabel ? dlabel[b0 + j] : nullptr;
      J.s = slots[j].k;
    }
    B200_CUDA(cudaMemcpyAsync(dj, hj, sizeof(KfJob) * B, cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaEventRecord(job_ev[ring], stream));
    B200_CUDA(cudaMemsetAsync(d_counters, 0, 16 * B, stream));
    const dim3 g256((npix + 255) / 256, B), gcell(cell_ctas(B), B);
    if (prm.leaf > 0) {
      const dim3 gt(((c + BIN_TW - 1) / BIN_TW) * ((r + BIN_TH - 1) / BIN_TH), B);
      k_ocm_bin<<<gt, BIN_THREADS, 0, stream>>>(dj, d_err);
      k_ocm_ranges<<<gcell, RANGES_THREADS, 0, stream>>>(dj);
      k_ocm_scatter<<<g256, 256, 0, stream>>>(dj);
      k_ocm_centroids<<<gcell, 256, 0, stream>>>(dj);
      launches += 4;
    } else {
      k_ocm_points_nofilter<<<g256, 256, 0, stream>>>(dj);
      launches += 1;
    }
    k_ocm_scan_keys<<<gcell, 256, 0, stream>>>(dj, map, d_err);
    // grid-stride sweep on a fixed grid (8 CTAs per SM)
    k_ocm_apply<<<8 * sms, 256, 0, stream>>>(hit_log, miss_log, cmin, cmax, map);
    launches += 2;
    last_slot = B - 1;
    B200_CUDA(cudaGetLastError());
  }
  return B200ORB_OK;
}

// Exclusive scan of n 64-bit words in place; the total lands in tw.total.
int ocm::scan(unsigned long long* data, int n) {
  const int tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  k_ocm_tree_scan_tiles<<<tiles, SCAN_THREADS, 0, stream>>>(data, n, tw.sums);
  k_ocm_tree_scan_sums<<<1, SCAN_THREADS, 0, stream>>>(tw.sums, tiles, tw.total);
  k_ocm_tree_scan_apply<<<tiles, SCAN_THREADS, 0, stream>>>(data, n, tw.sums);
  launches += 3;
  B200_CUDA(cudaGetLastError());
  return B200ORB_OK;
}

// Hash -> pruned tree (ocm_tree.cuh), on the map's stream after everything enqueued there.  The host reads two counts,
// the cells and then the nodes and leaves, to size the buffers; no cell and no node passes through it.
int ocm::build_tree() {
  tree_nodes = -1;
  int n = 0;
  B200_CUDA(cudaMemcpyAsync(&n, map.nleaves, 4, cudaMemcpyDeviceToHost, stream));
  B200_CUDA(cudaStreamSynchronize(stream));
  B200_CHECK(check_err());   // a map that overflowed is not written
  if (n == 0) { tree_nodes = tree_leaves = 0; return B200ORB_OK; }
  size_t sort_bytes = 0;
  B200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const unsigned long long*)nullptr,
                                            (unsigned long long*)nullptr, (const unsigned*)nullptr, (unsigned*)nullptr, n, 0,
                                            48, (cudaStream_t)stream));
  B200_CHECK(tree_ws.reserve(stream, [&](Carver& t) {
    tw.code_in = t.take<unsigned long long>(n); tw.code = t.take<unsigned long long>(n);
    tw.slot_in = t.take<unsigned>(n); tw.slot = t.take<unsigned>(n);
    tw.val = t.take<float>(n); tw.rgb = t.take<unsigned>(n);
    tw.run = t.take<unsigned long long>(n); tw.off = t.take<unsigned long long>(n);
    tw.lcp = t.take<signed char>(n); tw.top = t.take<signed char>(n);
    tw.sums = t.take<unsigned long long>((n + SCAN_TILE - 1) / SCAN_TILE); tw.total = t.take<unsigned long long>(1);
    tw.count = t.take<int>(1); tw.sort_tmp = t.take<char>(sort_bytes);
  }));
  const unsigned cells = (unsigned)((n + 255) / 256);
  B200_CUDA(cudaMemsetAsync(tw.count, 0, 4, stream));
  k_ocm_tree_gather<<<(unsigned)((map_cap + 255) / 256), 256, 0, stream>>>(map, n, tw.code_in, tw.slot_in, tw.count);
  B200_CUDA(cub::DeviceRadixSort::SortPairs(tw.sort_tmp, sort_bytes, (const unsigned long long*)tw.code_in, tw.code,
                                            (const unsigned*)tw.slot_in, tw.slot, n, 0, 48, (cudaStream_t)stream));
  k_ocm_tree_cells<<<cells, 256, 0, stream>>>(map, n, tw.slot, tw.val, tw.rgb, tw.run);
  launches += 2;
  B200_CHECK(scan(tw.run, n));
  k_ocm_tree_classify<<<cells, 256, 0, stream>>>(n, tw.code, tw.run, tw.lcp, tw.top, tw.off);
  ++launches;
  B200_CHECK(scan(tw.off, n));
  unsigned long long total = 0;
  B200_CUDA(cudaMemcpyAsync(&total, tw.total, 8, cudaMemcpyDeviceToHost, stream));
  B200_CUDA(cudaStreamSynchronize(stream));
  const long long nn = (long long)(total & 0xffffffffull), nl = (long long)(total >> 32);
  B200_CHECK(tree_res.reserve(stream, [&](Carver& t) {
    tree.nodes = t.take<uint2>(nn); tree.keys = t.take<unsigned short>(3 * nl); tree.depth = t.take<unsigned char>(nl);
    tree.val = t.take<float>(nl); tree.rgb = t.take<unsigned char>(3 * nl);
  }));
  k_ocm_tree_leaves<<<cells, 256, 0, stream>>>(n, tw.code, tw.val, tw.rgb, tw.lcp, tw.top, tw.off, tree);
  for (int d = 15; d >= 0; --d)
    k_ocm_tree_inner<<<cells, 256, 0, stream>>>(n, d, tw.code, tw.val, tw.lcp, tw.top, tw.off, tree.nodes);
  launches += 17;
  B200_CUDA(cudaGetLastError());
  tree_nodes = nn; tree_leaves = nl;
  return B200ORB_OK;
}

// Replace the map by the leaves of an `.ot` file.  Everything that can be refused is refused before the table is touched.
int ocm::read_ot(const uint8_t* bytes, int64_t n) {
  double res = 0;
  std::vector<OtLeaf> leaves;
  B200_CHECK(parse_ot(bytes, n, &res, &leaves));
  char mine[32];
  snprintf(mine, sizeof(mine), "%g", prm.resolution);   // the resolution as a file carries it
  if (res != strtod(mine, nullptr)) {
    set_error(".ot: res %g, this map has %s", res, mine);
    return B200ORB_EINVAL;
  }
  const size_t nl = leaves.size();
  std::vector<long long> first(nl + 1, 0);
  for (size_t i = 0; i < nl; ++i) {
    first[i + 1] = first[i] + (1ll << (3 * (16 - leaves[i].depth)));
    if (first[i + 1] > map_cap) {
      set_error(".ot: more than %lld cells, the map holds %lld (raise OcmParams.map_capacity)", first[i], map_cap);
      return B200ORB_ECAP;
    }
  }
  unsigned long long* key = nullptr;
  float* val = nullptr;
  unsigned* rgb = nullptr;
  unsigned char* depth = nullptr;
  long long* d_first = nullptr;
  B200_CHECK(load.reserve(stream, [&](Carver& t) {
    key = t.take<unsigned long long>(nl); d_first = t.take<long long>(nl); val = t.take<float>(nl);
    rgb = t.take<unsigned>(nl); depth = t.take<unsigned char>(nl);
  }));
  B200_CHECK(clear_map());
  if (nl > 0) {
    std::vector<unsigned long long> hk(nl);
    std::vector<float> hv(nl);
    std::vector<unsigned> hc(nl);
    std::vector<unsigned char> hd(nl);
    for (size_t i = 0; i < nl; ++i) {
      const OtLeaf& l = leaves[i];
      hk[i] = (unsigned long long)l.key[0] | (unsigned long long)l.key[1] << 16 | (unsigned long long)l.key[2] << 32;
      hv[i] = l.val;
      hc[i] = (unsigned)l.rgb[0] | (unsigned)l.rgb[1] << 8 | (unsigned)l.rgb[2] << 16;
      hd[i] = l.depth;
    }
    B200_CUDA(cudaMemcpyAsync(key, hk.data(), 8 * nl, cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaMemcpyAsync(d_first, first.data(), 8 * nl, cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaMemcpyAsync(val, hv.data(), 4 * nl, cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaMemcpyAsync(rgb, hc.data(), 4 * nl, cudaMemcpyHostToDevice, stream));
    B200_CUDA(cudaMemcpyAsync(depth, hd.data(), nl, cudaMemcpyHostToDevice, stream));
    const long long cells = first[nl];
    k_ocm_tree_expand<<<(unsigned)((cells + 255) / 256), 256, 0, stream>>>(map, (int)nl, cells, key, depth, val, rgb, d_first,
                                                                          d_err);
    ++launches;
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaStreamSynchronize(stream));   // the staging vectors go out of scope
  }
  return check_err();
}

extern "C" {

void ocm_default_params(OcmParams* p) {
  if (!p) return;
  p->resolution = 0.05; p->prob_hit = 0.7; p->prob_miss = 0.4; p->clamp_min = 0.12; p->clamp_max = 0.97;
  p->depth_min = 0.5f; p->depth_max = 3.0f; p->y_max = 3.0f; p->leaf = 0.01f; p->map_capacity = 0;
}

int ocm_create(const OcmParams* p, int device, ocm_t** out) {
  if (!p || !out) { set_error("null argument"); return B200ORB_EINVAL; }
  *out = nullptr;
  if (!(p->resolution > 0) || !(p->prob_hit > 0 && p->prob_hit < 1) || !(p->prob_miss > 0 && p->prob_miss < 1) ||
      !(p->clamp_min > 0 && p->clamp_min < p->clamp_max && p->clamp_max < 1)) {
    set_error("bad OcmParams");
    return B200ORB_EINVAL;
  }
  B200_CHECK(check_device(device));
  DeviceGuard g(device);
  std::unique_ptr<ocm> h(new (std::nothrow) ocm());
  if (!h) { set_error("out of host memory"); return B200ORB_EINVAL; }
  h->prm = *p;
  h->device = device;
  h->sms = sm_count(device);
  auto logodds = [](double pr) { return (float)log(pr / (1 - pr)); };   // octomap::logodds (float)
  h->hit_log = logodds(p->prob_hit); h->miss_log = logodds(p->prob_miss);
  h->cmin = logodds(p->clamp_min); h->cmax = logodds(p->clamp_max);
  h->map_cap = pow2_at_least(p->map_capacity > 0 ? std::max<long long>(p->map_capacity, 2) : (1ll << 23));
  // highest stream priority: the mapper is a chain of small dependent kernels running BESIDE the tracking batch;
  // with default priority every link waits behind thousands of queued tracking CTAs, with high priority its CTAs
  // take the next free SM slots.
  int lo_p = 0, hi_p = 0;
  cudaDeviceGetStreamPriorityRange(&lo_p, &hi_p);
  B200_CHECK(h->stream.create(hi_p));
  for (Event& e : h->job_ev) B200_CHECK(e.create());
  for (Event& e : h->mg_ev) B200_CHECK(e.create());
  h->map.mask = h->map_cap - 1;
  B200_CHECK(h->block.carve(h->stream, [&](Carver& t) { h->take_block(t); }));
  B200_CHECK(h->clear_map());
  B200_CUDA(cudaStreamSynchronize(h->stream));
  *out = h.release();
  return B200ORB_OK;
}
void ocm_destroy(ocm_t* h) { destroy_handle(h); }

int ocm_insert_keyframe_device(ocm_t* h, const float* d_depth, const uint8_t* d_rgb, int rows, int cols,
                               const float Tcw[16], float fx, float fy, float cx, float cy, const uint8_t* d_label) {
  if (!h || !d_depth || !d_rgb || !Tcw || rows <= 0 || cols <= 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  return h->insert(d_depth, d_rgb, d_label, rows, cols, Tcw, fx, fy, cx, cy);
}

int ocm_insert_keyframes_labeled_device(ocm_t* h, const float* d_depth, const uint8_t* d_rgb, const uint8_t* d_label,
                                        int rows, int cols, const int32_t* depth_idx, const int32_t* rgb_idx,
                                        const int32_t* label_idx, int n, const float* Tcw, float fx, float fy, float cx,
                                        float cy) {
  if (!h || !d_depth || !d_rgb || !depth_idx || !Tcw || rows <= 0 || cols <= 0 || n < 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  const size_t npix = (size_t)rows * cols;
  std::vector<const float*> dd(n);
  std::vector<const uint8_t*> dc(n), dl(n);
  for (int i = 0; i < n; ++i) {
    const int di = depth_idx[i], ri = rgb_idx ? rgb_idx[i] : depth_idx[i], li = label_idx ? label_idx[i] : depth_idx[i];
    if (di < 0 || ri < 0 || li < 0) { set_error("negative frame index"); return B200ORB_EINVAL; }
    dd[i] = d_depth + npix * di;
    dc[i] = d_rgb + npix * 3 * ri;
    dl[i] = d_label ? d_label + npix * li : nullptr;
  }
  if (n == 0) return B200ORB_OK;
  return h->insert_batch(n, dd.data(), dc.data(), d_label ? dl.data() : nullptr, rows, cols, Tcw, fx, fy, cx, cy);
}

int ocm_insert_keyframes_u16_labeled(ocm_t* h, const uint16_t* depth_u16, const uint8_t* rgb, const uint8_t* label, int rows,
                                     int cols, int n, float depth_factor, const float* Tcw, float fx, float fy, float cx,
                                     float cy) {
  if (!h || !depth_u16 || !rgb || !Tcw || rows <= 0 || cols <= 0 || n < 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  if (n == 0) return B200ORB_OK;
  DeviceGuard g(h->device);
  const size_t npix = (size_t)rows * cols, tot = npix * n;
  if ((npix % 4) != 0) { set_error("rows*cols must be a multiple of 4"); return B200ORB_EINVAL; }
  B200_CHECK(h->ensure_scratch(rows, cols));
  B200_CHECK(h->ensure_staging(tot));
  if (label) B200_CUDA(cudaMemcpyAsync(h->st_label, label, tot, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(h->st_d16, depth_u16, tot * 2, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(h->st_rgb, rgb, tot * 3, cudaMemcpyHostToDevice, h->stream));
  k_depth_u16_to_f32<<<(unsigned)((tot / 4 + 255) / 256), 256, 0, h->stream>>>(
      reinterpret_cast<const ushort4*>(h->st_d16), reinterpret_cast<float4*>(h->st_depth), depth_factor, tot / 4);
  ++h->launches;
  std::vector<const float*> dd(n);
  std::vector<const uint8_t*> dc(n), dl(n);
  for (int i = 0; i < n; ++i) { dd[i] = h->st_depth + npix * i; dc[i] = h->st_rgb + npix * 3 * i; dl[i] = h->st_label + npix * i; }
  return h->insert_batch(n, dd.data(), dc.data(), label ? dl.data() : nullptr, rows, cols, Tcw, fx, fy, cx, cy);
}

int ocm_insert_keyframe(ocm_t* h, const float* depth, const uint8_t* rgb, int rows, int cols, const float Tcw[16],
                        float fx, float fy, float cx, float cy, const uint8_t* ground_label) {
  if (!h || !depth || !rgb || !Tcw || rows <= 0 || cols <= 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  B200_CHECK(h->ensure_scratch(rows, cols));
  const size_t npix = (size_t)rows * cols;
  B200_CHECK(h->ensure_staging(npix));
  B200_CUDA(cudaMemcpyAsync(h->st_depth, depth, npix * 4, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemcpyAsync(h->st_rgb, rgb, npix * 3, cudaMemcpyHostToDevice, h->stream));
  if (ground_label) B200_CUDA(cudaMemcpyAsync(h->st_label, ground_label, npix, cudaMemcpyHostToDevice, h->stream));
  B200_CHECK(h->insert(h->st_depth, h->st_rgb, ground_label ? h->st_label : nullptr, rows, cols, Tcw, fx, fy, cx, cy));
  return h->check_err();
}

int ocm_last_points(ocm_t* h, float* xyz, uint8_t* rgb, int cap, int* n) {
  if (!h || !n) { set_error("null argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  int cnt[2] = {0, 0};
  if (h->slots.empty()) { *n = 0; return B200ORB_OK; }
  const KfScratch& ls = h->slots[h->last_slot].k;
  B200_CUDA(cudaMemcpyAsync(cnt, ls.counters, 8, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  *n = cnt[1];
  if (!xyz) return B200ORB_OK;
  if (cnt[1] > cap) { set_error("cap %d < %d points", cap, cnt[1]); return B200ORB_ECAP; }
  B200_CUDA(cudaMemcpyAsync(xyz, ls.pts, (size_t)12 * cnt[1], cudaMemcpyDeviceToHost, h->stream));
  if (rgb) B200_CUDA(cudaMemcpyAsync(rgb, ls.pts_rgb, (size_t)3 * cnt[1], cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int64_t ocm_num_leaves(ocm_t* h) {
  if (!h) return -1;
  DeviceGuard g(h->device);
  int n = 0;
  if (cudaMemcpyAsync(&n, h->map.nleaves, 4, cudaMemcpyDeviceToHost, h->stream) != cudaSuccess) return -1;
  cudaStreamSynchronize(h->stream);
  return n;
}

int ocm_export_leaves(ocm_t* h, uint16_t* keys, float* logodds, uint8_t* rgb, int64_t cap, int64_t* n) {
  if (!h || !keys || !logodds || cap < 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  unsigned short* dk;
  float* dv;
  unsigned char* dc;
  B200_CHECK(h->exp.reserve(h->stream, [&](Carver& t) {
    dk = t.take<unsigned short>(3 * cap); dv = t.take<float>(cap); dc = t.take<unsigned char>(3 * cap);
  }));
  long long cnt = 0;
  B200_CUDA(cudaMemsetAsync(h->d_export_counter, 0, 8, h->stream));
  k_ocm_export<<<(unsigned)((h->map_cap + 255) / 256), 256, 0, h->stream>>>(h->map, h->d_export_counter, cap, dk, dv, dc);
  ++h->launches;
  B200_CUDA(cudaMemcpyAsync(&cnt, h->d_export_counter, 8, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  if (n) *n = cnt;
  if (cnt > cap) { set_error("export cap %lld < %lld entries", (long long)cap, cnt); return B200ORB_ECAP; }
  B200_CUDA(cudaMemcpyAsync(keys, dk, 6 * cnt, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(logodds, dv, 4 * cnt, cudaMemcpyDeviceToHost, h->stream));
  if (rgb) B200_CUDA(cudaMemcpyAsync(rgb, dc, 3 * cnt, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int ocm_query(ocm_t* h, const float xyz[3], float* logodds, int* found) {
  if (!h || !xyz || !logodds || !found) { set_error("null argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  int k[3];
  const double rf = 1.0 / h->prm.resolution;
  for (int i = 0; i < 3; ++i) {   // coord_to_key's rule: a non-finite coordinate has no key
    const double f = floor(rf * (double)xyz[i]);
    if (!(f >= -32768.0 && f < 32768.0)) { *found = 0; *logodds = 0; return B200ORB_OK; }
    k[i] = (int)f + 32768;
  }
  const unsigned long long key = (unsigned long long)k[0] | ((unsigned long long)k[1] << 16) | ((unsigned long long)k[2] << 32);
  k_ocm_query<<<1, 1, 0, h->stream>>>(h->map, key, h->d_query_val, h->d_query_found);
  ++h->launches;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(logodds, h->d_query_val, 4, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(found, h->d_query_found, 4, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

// ---- multi-GPU map merge over NCCL (SURVEY §8(b) ocm_merge_nccl, §8(e)) ---------------------------------------------
// NCCL is bound at run time (dlopen of libnccl.so.2 -- the copy torch already loaded when there is one), so the library
// has no link-time dependency on it and single-GPU users never touch it.
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*CommCount)(const ncclComm_t, int*) = nullptr;
  ncclResult_t (*CommUserRank)(const ncclComm_t, int*) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi* nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* L = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!L) L = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (L) {
      api.lib = L;
      *(void**)&api.GetUniqueId = dlsym(L, "ncclGetUniqueId");
      *(void**)&api.CommInitRank = dlsym(L, "ncclCommInitRank");
      *(void**)&api.CommDestroy = dlsym(L, "ncclCommDestroy");
      *(void**)&api.CommCount = dlsym(L, "ncclCommCount");
      *(void**)&api.CommUserRank = dlsym(L, "ncclCommUserRank");
      *(void**)&api.AllGather = dlsym(L, "ncclAllGather");
      *(void**)&api.Broadcast = dlsym(L, "ncclBroadcast");
      *(void**)&api.GroupStart = dlsym(L, "ncclGroupStart");
      *(void**)&api.GroupEnd = dlsym(L, "ncclGroupEnd");
      *(void**)&api.GetErrorString = dlsym(L, "ncclGetErrorString");
      if (!api.GetUniqueId || !api.CommInitRank || !api.AllGather || !api.Broadcast || !api.GroupStart || !api.GroupEnd ||
          !api.CommCount || !api.CommUserRank || !api.CommDestroy || !api.GetErrorString)
        api.lib = nullptr;
    }
  }
  if (!api.lib) { set_error("NCCL not available (dlopen libnccl.so.2 failed)"); return nullptr; }
  return &api;
}
#define B200_NCCL(api, expr)                                                                       \
  do {                                                                                             \
    ncclResult_t _r = (expr);                                                                      \
    if (_r != ncclSuccess) { set_error("%s -> %s", #expr, (api)->GetErrorString(_r)); return B200ORB_ECUDA; } \
  } while (0)

int ocm_nccl_unique_id(uint8_t id[128]) {
  NcclApi* N = nccl_api();
  if (!N || !id) return B200ORB_EINVAL;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId");
  ncclUniqueId u;
  B200_NCCL(N, N->GetUniqueId(&u));
  memcpy(id, &u, 128);
  return B200ORB_OK;
}
int ocm_nccl_comm_create(const uint8_t id[128], int rank, int world, int device, void** comm) {
  NcclApi* N = nccl_api();
  if (!N || !id || !comm || world < 1 || rank < 0 || rank >= world) { if (N) set_error("bad argument"); return B200ORB_EINVAL; }
  B200_CHECK(check_device(device));
  DeviceGuard g(device);
  ncclUniqueId u;
  memcpy(&u, id, 128);
  ncclComm_t c = nullptr;
  B200_NCCL(N, N->CommInitRank(&c, world, u, rank));
  *comm = (void*)c;
  return B200ORB_OK;
}
int ocm_nccl_comm_destroy(void* comm) {
  NcclApi* N = nccl_api();
  if (!N) return B200ORB_EINVAL;
  if (comm) N->CommDestroy((ncclComm_t)comm);
  return B200ORB_OK;
}

int ocm_merge_nccl(ocm_t* h, void* comm_, void* stream_, OcmMergeStats* st) {
  if (!h) { set_error("null argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  cudaStream_t S = h->stream;
  if (stream_ && (cudaStream_t)stream_ != S) {   // order after the caller's stream
    B200_CUDA(cudaEventRecord(h->mg_ev[0], (cudaStream_t)stream_));
    B200_CUDA(cudaStreamWaitEvent(S, h->mg_ev[0], 0));
  }
  NcclApi* N = nullptr;
  ncclComm_t comm = (ncclComm_t)comm_;
  int world = 1, rank = 0;
  if (comm) {
    N = nccl_api();
    if (!N) return B200ORB_EINVAL;
    B200_NCCL(N, N->CommCount(comm, &world));
    B200_NCCL(N, N->CommUserRank(comm, &rank));
  }
  int *counts, *counts_h;
  B200_CHECK(h->mg_counts.reserve(S, [&](Carver& t) { counts = t.take<int>(world); }));
  B200_CHECK(h->mg_counts_h.reserve(S, [&](Carver& t) { counts_h = t.take<int>(world); }));
  // 1. counts: one int per rank (the only host synchronisation of the merge)
  if (comm) B200_NCCL(N, N->AllGather(h->map.nelist, counts, 1, ncclInt32, comm, S));
  else B200_CUDA(cudaMemcpyAsync(counts, h->map.nelist, 4, cudaMemcpyDeviceToDevice, S));
  B200_CUDA(cudaMemcpyAsync(counts_h, counts, 4 * world, cudaMemcpyDeviceToHost, S));
  B200_CUDA(cudaStreamSynchronize(S));
  std::vector<long long> off(world + 1, 0);   // byte offsets of the shards in the receive buffer (16-byte aligned)
  long long total = 0;
  for (int r = 0; r < world; ++r) {
    off[r + 1] = (long long)align_up_sz((size_t)(off[r] + 24ll * counts_h[r]), 16);
    total += counts_h[r];
  }
  const long long n_own = counts_h[rank];
  char *send, *recv;
  int* slots;
  B200_CHECK(h->mg.reserve(S, [&](Carver& t) {
    send = t.take<char>(24 * n_own); recv = t.take<char>(off[world]); slots = t.take<int>(total);
  }));
  // 2. pack own summaries, roll own voxels back to the last merge
  if (n_own > 0) {
    k_merge_pack<<<(unsigned)((n_own + 255) / 256), 256, 0, S>>>(h->map, (int)n_own, merge_shard_at(send, n_own));
    ++h->launches;
  }
  B200_CUDA(cudaMemsetAsync(h->map.nelist, 0, 4, S));
  // 3. exchange: every rank broadcasts its shard (exact sizes, one grouped NCCL call over NVLink)
  if (comm && world > 1) {
    B200_NCCL(N, N->GroupStart());
    for (int r = 0; r < world; ++r) {
      const size_t bytes = 24 * (size_t)counts_h[r];
      if (bytes == 0) continue;
      B200_NCCL(N, N->Broadcast(r == rank ? send : nullptr, recv + off[r], bytes, ncclUint8, r, comm, S));
    }
    B200_NCCL(N, N->GroupEnd());
  } else if (n_own > 0) {
    B200_CUDA(cudaMemcpyAsync(recv, send, 24 * n_own, cudaMemcpyDeviceToDevice, S));
  }
  // 4. replay all shards in rank (= keyframe) order, then make the result the base of the next epoch
  long long done = 0;
  for (int r = 0; r < world; ++r) {
    const long long n = counts_h[r];
    if (n == 0) continue;
    k_merge_apply<<<(unsigned)((n + 255) / 256), 256, 0, S>>>(h->map, n, merge_shard_at(recv + off[r], n),
                                                             slots + done, h->d_err);
    ++h->launches;
    done += n;
  }
  if (total > 0) {
    k_merge_commit<<<(unsigned)((total + 255) / 256), 256, 0, S>>>(h->map, total, slots);
    ++h->launches;
  }
  B200_CUDA(cudaGetLastError());
  if (stream_ && (cudaStream_t)stream_ != S) {
    B200_CUDA(cudaEventRecord(h->mg_ev[1], S));
    B200_CUDA(cudaStreamWaitEvent((cudaStream_t)stream_, h->mg_ev[1], 0));
  }
  if (st) { st->world = world; st->rank = rank; st->records_sent = n_own; st->records_total = total; st->bytes_sent = 24 * n_own; st->bytes_received = 24 * (total - n_own); }
  return B200ORB_OK;
}

int ocm_last_batch_stats(ocm_t* h, int64_t* points, int64_t* voxels_touched) {
  if (!h) { set_error("null argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  std::vector<int> c(4 * ocm::MAX_SLOTS, 0);
  unsigned long long nt = 0;
  B200_CUDA(cudaMemcpyAsync(c.data(), h->d_counters, 16 * ocm::MAX_SLOTS, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(&nt, h->map.nupd, 8, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  long long p = 0;
  for (int j = 0; j <= h->last_slot && j < ocm::MAX_SLOTS; ++j) p += c[4 * j + 1];
  if (points) *points = p;
  if (voxels_touched) *voxels_touched = (int64_t)nt;
  return B200ORB_OK;
}

int ocm_tree_build(ocm_t* h, int64_t* n_nodes, int64_t* n_leaves) {
  if (!h) { set_error("null argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  B200_CHECK(h->build_tree());
  if (n_nodes) *n_nodes = h->tree_nodes;
  if (n_leaves) *n_leaves = h->tree_leaves;
  return B200ORB_OK;
}

int ocm_write_ot(ocm_t* h, uint8_t* buf, int64_t cap, int64_t* n) {
  if (!h || (buf && cap < 0)) { set_error("bad argument"); return B200ORB_EINVAL; }
  if (h->tree_nodes < 0) { set_error("no tree: call ocm_tree_build first"); return B200ORB_EINVAL; }
  const std::string hdr = ot_header(h->tree_nodes, h->prm.resolution);
  const int64_t need = (int64_t)hdr.size() + 8 * h->tree_nodes;
  if (n) *n = need;
  if (!buf) return B200ORB_OK;
  if (cap < need) { set_error(".ot buffer of %lld bytes < %lld", (long long)cap, (long long)need); return B200ORB_ECAP; }
  DeviceGuard g(h->device);
  memcpy(buf, hdr.data(), hdr.size());
  if (h->tree_nodes > 0) {
    B200_CUDA(cudaMemcpyAsync(buf + hdr.size(), h->tree.nodes, 8 * h->tree_nodes, cudaMemcpyDeviceToHost, h->stream));
    B200_CUDA(cudaStreamSynchronize(h->stream));
  }
  return B200ORB_OK;
}

int ocm_tree_leaves(ocm_t* h, uint16_t* keys, uint8_t* depth, float* logodds, uint8_t* rgb, int64_t cap, int64_t* n) {
  if (!h || cap < 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  if (h->tree_nodes < 0) { set_error("no tree: call ocm_tree_build first"); return B200ORB_EINVAL; }
  const long long nl = h->tree_leaves;
  if (n) *n = nl;
  if (!keys && !depth && !logodds && !rgb) return B200ORB_OK;
  if (cap < nl) { set_error("cap %lld < %lld pruned leaves", (long long)cap, nl); return B200ORB_ECAP; }
  if (nl == 0) return B200ORB_OK;
  DeviceGuard g(h->device);
  if (keys) B200_CUDA(cudaMemcpyAsync(keys, h->tree.keys, 6 * nl, cudaMemcpyDeviceToHost, h->stream));
  if (depth) B200_CUDA(cudaMemcpyAsync(depth, h->tree.depth, nl, cudaMemcpyDeviceToHost, h->stream));
  if (logodds) B200_CUDA(cudaMemcpyAsync(logodds, h->tree.val, 4 * nl, cudaMemcpyDeviceToHost, h->stream));
  if (rgb) B200_CUDA(cudaMemcpyAsync(rgb, h->tree.rgb, 3 * nl, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int ocm_save_ot(ocm_t* h, const char* path, int64_t* n_nodes) {
  if (!h || !path) { set_error("null argument"); return B200ORB_EINVAL; }
  B200_CHECK(ocm_tree_build(h, n_nodes, nullptr));
  int64_t bytes = 0;
  B200_CHECK(ocm_write_ot(h, nullptr, 0, &bytes));
  std::vector<uint8_t> buf((size_t)bytes);
  B200_CHECK(ocm_write_ot(h, buf.data(), bytes, nullptr));
  FILE* f = fopen(path, "wb");
  const bool ok = f && fwrite(buf.data(), 1, buf.size(), f) == buf.size();
  if ((f && fclose(f) != 0) || !ok) { set_error("cannot write %s", path); return B200ORB_EINVAL; }
  return B200ORB_OK;
}

int ocm_read_ot(ocm_t* h, const uint8_t* bytes, int64_t n) {
  if (!h || n < 0 || (!bytes && n > 0)) { set_error("bad argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  return h->read_ot(bytes, n);
}

// a whole file; false (with the error set) when it cannot be read
static bool read_file(const char* path, std::vector<uint8_t>* out) {
  FILE* f = fopen(path, "rb");
  if (!f) { set_error("cannot open %s", path); return false; }
  uint8_t chunk[1 << 16];
  size_t got;
  while ((got = fread(chunk, 1, sizeof(chunk), f)) > 0) out->insert(out->end(), chunk, chunk + got);
  const bool ok = !ferror(f);
  fclose(f);
  if (!ok) set_error("cannot read %s", path);
  return ok;
}

int ocm_load_ot(ocm_t* h, const char* path) {
  if (!h || !path) { set_error("null argument"); return B200ORB_EINVAL; }
  std::vector<uint8_t> bytes;
  if (!read_file(path, &bytes)) return B200ORB_EINVAL;
  return ocm_read_ot(h, bytes.data(), (int64_t)bytes.size());
}

int ocm_ot_leaves(const uint8_t* bytes, int64_t n, double* res, uint16_t* keys, uint8_t* depth, float* logodds, uint8_t* rgb,
                  int64_t cap, int64_t* n_out) {
  if (n < 0 || (!bytes && n > 0) || cap < 0) { set_error("bad argument"); return B200ORB_EINVAL; }
  double r = 0;
  std::vector<OtLeaf> leaves;
  B200_CHECK(parse_ot(bytes, n, &r, &leaves));
  const int64_t nl = (int64_t)leaves.size();
  if ((keys || depth || logodds || rgb) && cap < nl) {
    if (n_out) *n_out = nl;
    set_error("cap %lld < %lld leaves", (long long)cap, (long long)nl);
    return B200ORB_ECAP;
  }
  if (n_out) *n_out = nl;
  if (res) *res = r;
  for (int64_t i = 0; i < nl; ++i) {
    const OtLeaf& l = leaves[i];
    if (keys) memcpy(keys + 3 * i, l.key, 6);
    if (depth) depth[i] = l.depth;
    if (logodds) logodds[i] = l.val;
    if (rgb) memcpy(rgb + 3 * i, l.rgb, 3);
  }
  return B200ORB_OK;
}

int ocm_sync(ocm_t* h) {
  if (!h) return B200ORB_EINVAL;
  DeviceGuard g(h->device);
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return h->check_err();
}
void* ocm_stream(ocm_t* h) { return h ? (void*)(cudaStream_t)h->stream : nullptr; }
long long ocm_launch_count(const ocm_t* h) { return h ? h->launches : 0; }

}  // extern "C"
