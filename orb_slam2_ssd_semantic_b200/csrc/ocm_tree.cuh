// ocm_tree.cuh -- the occupancy map as octomap's pruned ColorOcTree, and back (included from ocm.cu).
// Reference: InsertScan's m_octree->prune() (perfect/src/MapDrawer.cc:1024) and the tree walks of MapDrawer::SaveOctoMap /
// LoadOctoMap (:1103-1117: AbstractOcTree::write / read).  Semantics are those of octree_io.build_ot, the numpy oracle:
// child index at depth d of a 16-bit key = bit (15 - d) of x | y << 1 | z << 2, pre-order = children 0..7, inner value =
// max over the children, inner colour white, and a node whose 8 children are childless leaves of equal value (float ==)
// and colour becomes that leaf, cascading upwards.
//
// Build.  The N cells of the hash are sorted by their 48-bit Morton code (x least significant of each triple), so a node
// (depth d, prefix p) is a contiguous segment of the sorted cells.  A segment is a PRUNED LEAF candidate iff it is FULL
// (8^(16-d) cells: with distinct sorted codes, iff its first and last code are the segment's first and last possible
// code) and UNIFORM (no boundary between two runs of equal (value, colour) inside it).  Full and uniform holds for every
// descendant of a full and uniform node, so the bottom-up cascade of pruneNode collapses into that one test, and a node
// is emitted iff its parent fails it.  The nodes whose segment starts at sorted cell i are the depths lcp(i-1, i) + 1 ..
// 16 (lcp in whole levels; -1 for i = 0), emitted down to top(i), the shallowest full-uniform depth on cell i's path;
// pre-order is (segment start, depth), so an exclusive scan of the per-cell emitted counts gives every node its place.
// Inner nodes take their value and child mask from their (at most 8) children, one launch per depth, deepest first.
//
// Load.  The header and the pre-order walk (sequential, a few hundred thousand nodes) run on the host; the device expands
// every leaf of depth d into its (2^(16-d))^3 depth-16 cells and inserts them with the map's find-or-insert probe.
#pragma once
#include <string>

#include <cub/device/device_radix_sort.cuh>

namespace b200 {

// bit i of a 16-bit key -> bit 3 i, and back
__host__ __device__ __forceinline__ unsigned long long spread3(unsigned long long x) {
  x &= 0xffffull;
  x = (x | x << 32) & 0x1f00000000ffffull;
  x = (x | x << 16) & 0x1f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}
__host__ __device__ __forceinline__ unsigned compact3(unsigned long long x) {
  x &= 0x1249249249249249ull;
  x = (x ^ (x >> 2)) & 0x10c30c30c30c30c3ull;
  x = (x ^ (x >> 4)) & 0x100f00f00f00f00full;
  x = (x ^ (x >> 8)) & 0x1f0000ff0000ffull;
  x = (x ^ (x >> 16)) & 0x1f00000000ffffull;
  x = (x ^ (x >> 32)) & 0xffffull;
  return (unsigned)x;
}

// Per-cell workspace of one build (N cells) and the words of the two scans.
struct TreeWork {
  unsigned long long *code_in, *code;   // Morton codes in hash order / sorted
  unsigned *slot_in, *slot;             // the cell's slot of the hash, same orders
  float* val;                           // sorted cells: log-odds, colour
  unsigned* rgb;
  unsigned long long* run;              // number of run boundaries before cell i: equal for two cells of one run
  unsigned long long* off;              // low word: index of cell i's first node; high word: index of its pruned leaf
  signed char *lcp, *top;
  unsigned long long* sums;             // per-tile sums of a scan
  unsigned long long* total;            // of the last scan: low word = nodes, high word = pruned leaves
  int* count;                           // cells gathered
  void* sort_tmp;
};
// The result: octomap's 8-byte nodes in pre-order ({log-odds bits, r | g << 8 | b << 16 | child mask << 24}) and the
// pruned leaves in the same order.
struct TreeOut {
  uint2* nodes;
  unsigned short* keys;   // min corner, 3 per leaf
  unsigned char* depth;
  float* val;
  unsigned char* rgb;     // 3 per leaf
};

__global__ void k_ocm_tree_gather(MapView m, int n, unsigned long long* __restrict__ code, unsigned* __restrict__ slot,
                                  int* __restrict__ count) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s > m.mask) return;
  const unsigned long long k = m.keys[s];
  if (k == EMPTY_KEY) return;
  const int o = atomicAdd(count, 1);
  if (o >= n) return;
  code[o] = spread3(k) | spread3(k >> 16) << 1 | spread3(k >> 32) << 2;
  slot[o] = (unsigned)s;
}

// value and colour of the sorted cells; run[i] = 1 where cell i + 1 starts another run of equal (value, colour)
__global__ void k_ocm_tree_cells(MapView m, int n, const unsigned* __restrict__ slot, float* __restrict__ val,
                                 unsigned* __restrict__ rgb, unsigned long long* __restrict__ run) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned s = slot[i];
  const float v = m.val[s];
  const unsigned c = m.rgb[s] & 0xffffffu;
  val[i] = v;
  rgb[i] = c;
  bool boundary = true;
  if (i + 1 < n) {
    const unsigned t = slot[i + 1];
    boundary = !(m.val[t] == v && (m.rgb[t] & 0xffffffu) == c);
  }
  run[i] = boundary ? 1ull : 0ull;
}

// ---- exclusive scan of 64-bit words, in place: tile sums, one CTA over the sums, tiles again ---------------------------
constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 4, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ unsigned long long block_excl_scan64(unsigned long long v, unsigned long long* ws,
                                                                unsigned long long* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned long long inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();   // ws may still be read from the previous call
  if (lane == 31) ws[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    const unsigned long long w = lane < SCAN_THREADS / 32 ? ws[lane] : 0ull;
    unsigned long long winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    ws[lane] = winc - w;
    if (lane == 31) ws[32] = winc;
  }
  __syncthreads();
  *total = ws[32];
  return ws[wid] + inc - v;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_ocm_tree_scan_tiles(const unsigned long long* __restrict__ data, int n,
                                                                      unsigned long long* __restrict__ sums) {
  __shared__ unsigned long long ws[33];
  const int base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  unsigned long long v = 0ull;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k) v += base + k < n ? data[base + k] : 0ull;
  unsigned long long total;
  block_excl_scan64(v, ws, &total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(SCAN_THREADS) k_ocm_tree_scan_sums(unsigned long long* __restrict__ sums, int nb,
                                                                     unsigned long long* __restrict__ total) {
  __shared__ unsigned long long ws[33];
  unsigned long long carry = 0ull;
  for (int b0 = 0; b0 < nb; b0 += SCAN_THREADS) {
    const int b = b0 + threadIdx.x;
    const unsigned long long v = b < nb ? sums[b] : 0ull;
    unsigned long long chunk;
    const unsigned long long e = block_excl_scan64(v, ws, &chunk);
    if (b < nb) sums[b] = carry + e;
    carry += chunk;
  }
  if (threadIdx.x == 0) *total = carry;
}
__global__ void __launch_bounds__(SCAN_THREADS) k_ocm_tree_scan_apply(unsigned long long* __restrict__ data, int n,
                                                                      const unsigned long long* __restrict__ sums) {
  __shared__ unsigned long long ws[33];
  const int base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  unsigned long long x[SCAN_ITEMS], v = 0ull;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k) {
    x[k] = base + k < n ? data[base + k] : 0ull;
    v += x[k];
  }
  unsigned long long total;
  unsigned long long e = block_excl_scan64(v, ws, &total) + sums[blockIdx.x];
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; ++k) {
    if (base + k < n) data[base + k] = e;
    e += x[k];
  }
}

// Is the depth-d node on the path of sorted cell i (code c) full and uniform?
__device__ __forceinline__ bool tree_full_uniform(const unsigned long long* __restrict__ code,
                                                  const unsigned long long* __restrict__ run, int n, int i,
                                                  unsigned long long c, int d) {
  const unsigned long long size = 1ull << (3 * (16 - d));
  if (size > (unsigned long long)n) return false;
  const unsigned long long first = c & ~(size - 1ull), ahead = c - first;   // a full segment holds every code from `first`
  if (ahead > (unsigned long long)i) return false;
  const long long j = (long long)i - (long long)ahead, e = j + (long long)size - 1;
  if (e >= n) return false;
  return code[j] == first && code[e] == first + size - 1ull && run[j] == run[e];
}

// per cell: levels shared with the previous cell, the depth of its pruned leaf, how many nodes start at it
__global__ void k_ocm_tree_classify(int n, const unsigned long long* __restrict__ code,
                                    const unsigned long long* __restrict__ run, signed char* __restrict__ lcp,
                                    signed char* __restrict__ top, unsigned long long* __restrict__ off) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long c = code[i];
  int l = -1;
  if (i > 0) l = 15 - (63 - __clzll((long long)(c ^ code[i - 1]))) / 3;
  int d = 16;
  while (d > 0 && tree_full_uniform(code, run, n, i, c, d - 1)) --d;
  lcp[i] = (signed char)l;
  top[i] = (signed char)d;
  off[i] = d > l ? (unsigned long long)(d - l) | (1ull << 32) : 0ull;   // nodes of depths l + 1 .. d, one of them a leaf
}

__device__ __forceinline__ int tree_node_index(unsigned long long off, int lcp, int depth) {
  return (int)(unsigned)off + depth - lcp - 1;
}

__global__ void k_ocm_tree_leaves(int n, const unsigned long long* __restrict__ code, const float* __restrict__ val,
                                  const unsigned* __restrict__ rgb, const signed char* __restrict__ lcp,
                                  const signed char* __restrict__ top, const unsigned long long* __restrict__ off,
                                  TreeOut o) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int l = lcp[i], d = top[i];
  if (d <= l) return;   // inside a pruned leaf that starts at an earlier cell
  const unsigned long long c = code[i];   // the leaf's segment starts here: its min corner
  const unsigned col = rgb[i];
  o.nodes[tree_node_index(off[i], l, d)] = make_uint2(__float_as_uint(val[i]), col);
  const size_t q = (size_t)(off[i] >> 32);
  o.keys[q * 3] = (unsigned short)compact3(c); o.keys[q * 3 + 1] = (unsigned short)compact3(c >> 1);
  o.keys[q * 3 + 2] = (unsigned short)compact3(c >> 2);
  o.depth[q] = (unsigned char)d;
  o.val[q] = val[i];
  o.rgb[q * 3] = col & 0xff; o.rgb[q * 3 + 1] = (col >> 8) & 0xff; o.rgb[q * 3 + 2] = (col >> 16) & 0xff;
}

// The inner nodes of depth d (launched for d = 15 .. 0: the children's values are in place).
__global__ void k_ocm_tree_inner(int n, int d, const unsigned long long* __restrict__ code, const float* __restrict__ val,
                                 const signed char* __restrict__ lcp, const signed char* __restrict__ top,
                                 const unsigned long long* __restrict__ off, uint2* __restrict__ nodes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int l = lcp[i];
  if (!(l < d && d < top[i])) return;
  const int shift = 3 * (15 - d);                    // of a child's prefix
  const unsigned long long prefix = code[i] >> (shift + 3);
  const long long child_cells = 1ll << shift;
  unsigned mask = 0u;
  float mx = 0.f;
  int j = i;
  while (j < n && (code[j] >> (shift + 3)) == prefix) {
    const unsigned long long child = code[j] >> shift;
    const float v = top[j] == d + 1 ? val[j] : __uint_as_float(nodes[tree_node_index(off[j], j == i ? l : lcp[j], d + 1)].x);
    mx = mask ? fmaxf(mx, v) : v;
    mask |= 1u << (unsigned)(child & 7ull);
    // first cell past this child: its codes are distinct, so it holds at most child_cells cells
    long long lo = (long long)j + 1, hi = min((long long)n, (long long)j + child_cells);
    const unsigned long long next = (child + 1ull) << shift;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (code[mid] < next) lo = mid + 1; else hi = mid;
    }
    j = (int)lo;
  }
  nodes[tree_node_index(off[i], l, d)] = make_uint2(__float_as_uint(mx), 0xffffffu | mask << 24);
}

// ---- load ---------------------------------------------------------------------------------------------------------------
// A leaf of a parsed file: min-corner key, depth, log-odds, colour.
struct OtLeaf {
  uint16_t key[3];
  uint8_t depth;
  float val;
  uint8_t rgb[3];
};

// One thread per depth-16 cell: cell t belongs to the leaf whose range of first[] holds t.
__global__ void k_ocm_tree_expand(MapView m, int n_leaves, long long n_cells, const unsigned long long* __restrict__ key,
                                  const unsigned char* __restrict__ depth, const float* __restrict__ val,
                                  const unsigned* __restrict__ rgb, const long long* __restrict__ first,
                                  int* __restrict__ err) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_cells) return;
  int lo = 0, hi = n_leaves - 1;   // last leaf with first[leaf] <= t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= t) lo = mid; else hi = mid - 1;
  }
  const int bits = 16 - depth[lo];
  const unsigned long long r = (unsigned long long)(t - first[lo]), side = (1ull << bits) - 1ull;
  const unsigned long long k = key[lo] + ((r & side) | ((r >> bits) & side) << 16 | (r >> (2 * bits)) << 32);
  long long s;
  if (!map_slot(m, k, &s)) { atomicExch(err, ERR_MAP_FULL); return; }
  m.val[s] = val[lo];
  m.base[s] = val[lo];
  m.rgb[s] = rgb[lo];
}

// octomap's file header, as AbstractOcTree::write prints it (`res` through an ostream: %g)
static std::string ot_header(long long n_nodes, double res) {
  char b[256];
  snprintf(b, sizeof(b),
           "# Octomap OcTree file\n# (feel free to add / change comments, but leave the first line as it is!)\n#\n"
           "id ColorOcTree\nsize %lld\nres %g\ndata\n", n_nodes, res);
  return b;
}

// `.ot` bytes -> resolution and leaves in file order.  Every refusal happens here, on the host.
static int parse_ot(const uint8_t* b, int64_t n, double* res_out, std::vector<OtLeaf>* leaves) {
  static const char first_line[] = "# Octomap OcTree file";
  if (n < (int64_t)sizeof(first_line) - 1 || memcmp(b, first_line, sizeof(first_line) - 1) != 0) {
    set_error(".ot: the first line is not \"%s\"", first_line);
    return B200ORB_EINVAL;
  }
  // AbstractOcTree::readHeader: whitespace-separated tokens; `#` starts a comment line; `data` ends the header line
  int64_t p = 0;
  auto skip_line = [&] { while (p < n && b[p++] != '\n') {} };
  auto token = [&] {
    while (p < n && (b[p] == ' ' || b[p] == '\t' || b[p] == '\r' || b[p] == '\n')) ++p;
    const int64_t s = p;
    while (p < n && !(b[p] == ' ' || b[p] == '\t' || b[p] == '\r' || b[p] == '\n')) ++p;
    return std::string((const char*)b + s, (size_t)std::min<int64_t>(p - s, 64));
  };
  std::string id, size_txt, res_txt;
  bool data = false;
  while (p < n) {
    const std::string t = token();
    if (t.empty()) break;
    if (t == "data") { skip_line(); data = true; break; }
    if (t[0] == '#') skip_line();
    else if (t == "id") id = token();
    else if (t == "size") size_txt = token();
    else if (t == "res") res_txt = token();
    else skip_line();
  }
  if (!data) { set_error(".ot: no `data` line"); return B200ORB_EINVAL; }
  if (id != "ColorOcTree") { set_error(".ot: id `%s`, this map reads ColorOcTree", id.c_str()); return B200ORB_EINVAL; }
  char* end = nullptr;
  const long long size = strtoll(size_txt.c_str(), &end, 10);
  if (size_txt.empty() || *end || size < 0) { set_error(".ot: bad size `%s`", size_txt.c_str()); return B200ORB_EINVAL; }
  const double res = strtod(res_txt.c_str(), &end);
  if (res_txt.empty() || *end || !(res > 0)) { set_error(".ot: bad res `%s`", res_txt.c_str()); return B200ORB_EINVAL; }
  const int64_t body = n - p;
  if (size > body / 8 || size * 8 != body) {
    set_error(".ot: size %lld needs %lld bytes of nodes, %lld are present", size, size * 8, (long long)body);
    return B200ORB_EINVAL;
  }
  // pre-order walk: the child masks give every node its key and depth
  struct Pending { uint16_t key[3]; uint8_t depth; };
  std::vector<Pending> stack;
  std::vector<OtLeaf> out;
  if (size > 0) stack.push_back(Pending{{0, 0, 0}, 0});
  long long at = 0;
  while (!stack.empty()) {
    const Pending me = stack.back();
    stack.pop_back();
    if (at >= size) { set_error(".ot: the child masks run past the last of the %lld nodes", size); return B200ORB_EINVAL; }
    const uint8_t* node = b + p + 8 * at++;
    const unsigned mask = node[7];
    if (!mask) {
      OtLeaf lf;
      memcpy(lf.key, me.key, sizeof(lf.key));
      lf.depth = me.depth;
      memcpy(&lf.val, node, 4);
      memcpy(lf.rgb, node + 4, 3);
      out.push_back(lf);
      continue;
    }
    if (me.depth >= 16) { set_error(".ot: the tree is deeper than 16 levels"); return B200ORB_EINVAL; }
    const uint16_t bit = (uint16_t)(1u << (15 - me.depth));
    for (int c = 7; c >= 0; --c) {
      if (!(mask >> c & 1u)) continue;
      Pending ch = me;
      ++ch.depth;
      if (c & 1) ch.key[0] |= bit;
      if (c & 2) ch.key[1] |= bit;
      if (c & 4) ch.key[2] |= bit;
      stack.push_back(ch);
    }
  }
  if (at != size) { set_error(".ot: %lld nodes after the end of the tree", size - at); return B200ORB_EINVAL; }
  *res_out = res;
  leaves->swap(out);
  return B200ORB_OK;
}

}  // namespace b200
