// orbm_kernels.cuh -- sm_90a kernels of the ORB matcher (reference: src/ORBmatcher.cc + the Frame grid helpers of
// src/Frame.cc).  Integer / bitwise work: xor + popcount + warp reductions, no tensor cores.
//
// Every search of the reference has the same shape: an ordered list of QUERIES (map points / keyframe features),
// each with an ordered CANDIDATE list (GetFeaturesInArea window walk, or the features of one BoW node), a Hamming
// distance per candidate, and a loop-carried "already claimed" state that makes query i depend on queries < i
// (src/ORBmatcher.cc:113-115, 273-274, 1656-1658).  The GPU splits that into
//   K7  k_grid_build     AssignFeaturesToGrid (src/Frame.cc:319-334): 64x48 CSR per frame, cell lists in ascending
//                        keypoint index (= push_back order); block_grid_build, which k_match_last_fused also runs
//   K8  k_cand_generic   one WARP per query, all queries of all instances in parallel: everything that does not depend
//                        on the claimed state -- window walk in the reference's (ix, iy, insertion) order, static
//                        filters, Hamming distances -> candidate list  list[q][ord] = dist << 20 | idx.  The window
//                        geometry comes from query arrays (LAST: k_last_queries projects the last frame's points);
//                        k_cand_bow lists the features of one BoW node instead
//   K9  k_resolve_generic one warp per instance walks the queries IN ORDER; per query a warp-wide redux.min over
//                        (dist << 6 | ord) of the unclaimed entries reproduces "first minimum wins" exactly; then
//                        the rotation histogram / ComputeThreeMaxima prune (K10).  k_resolve_points (best-two ratio
//                        test) and k_resolve_bow are the variants of the other claim rules.
// A query with more than LCAP candidates is flagged and re-walked inside the resolve (exact, just slower).
// k_match_last_fused does K7-K10 of one LAST frame pair in one CTA when the pair fits in shared memory.
#pragma once
#include "orbm_host.h"

namespace b200 {

constexpr int GRID_COLS = ORBM_GRID_COLS, GRID_ROWS = ORBM_GRID_ROWS, GRID_CELLS = GRID_COLS * GRID_ROWS;
constexpr int LCAP = 64;                 // candidate-list capacity per query
constexpr unsigned KEY_INF = 0xffffffffu;

__device__ __forceinline__ int hamming256(const uint4 a0, const uint4 a1, const uint8_t* b) {
  // generic loads: the candidate descriptors live in shared memory in the fused kernel, in global memory otherwise
  const uint4 b0 = *reinterpret_cast<const uint4*>(b), b1 = *(reinterpret_cast<const uint4*>(b) + 1);
  return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
         __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

__device__ __forceinline__ int grid_cell(float x, float y, float min_x, float min_y, float inv_w, float inv_h) {
  // PosInGrid (src/Frame.cc:522-531): round(), not floor(); keypoints outside the 64x48 grid are dropped
  const int px = (int)roundf(__fmul_rn(__fsub_rn(x, min_x), inv_w));
  const int py = (int)roundf(__fmul_rn(__fsub_rn(y, min_y), inv_h));
  if (px < 0 || px >= GRID_COLS || py < 0 || py >= GRID_ROWS) return -1;
  return px * GRID_ROWS + py;
}

// The 64x48 CSR grid of one frame's n keypoints, built by the whole block: off[GRID_CELLS + 1] and idx[n] receive it,
// cur[GRID_CELLS] is scratch that the caller has zeroed (and published with a block barrier), ws[33] is scan scratch.
// No barrier after the last step.
__device__ __forceinline__ void block_grid_build(const float* x, const float* y, int n, float min_x, float min_y,
                                                 float inv_w, float inv_h, int* off, int* cur, int* idx, int* ws) {
  const int tid = threadIdx.x, nthr = blockDim.x;
  for (int i = tid; i < n; i += nthr) {
    const int c = grid_cell(x[i], y[i], min_x, min_y, inv_w, inv_h);
    if (c >= 0) atomicAdd(&cur[c], 1);
  }
  __syncthreads();
  {
    const int per = (GRID_CELLS + nthr - 1) / nthr;
    const int beg = min(GRID_CELLS, tid * per), end = min(GRID_CELLS, beg + per);
    int s = 0;
    for (int c = beg; c < end; ++c) s += cur[c];
    int total;
    int run = block_excl_scan(s, ws, &total);
    for (int c = beg; c < end; ++c) {
      off[c] = run;
      run += cur[c];
      cur[c] = 0;
    }
    if (tid == 0) off[GRID_CELLS] = total;
    __syncthreads();
  }
  for (int i = tid; i < n; i += nthr) {   // unordered fill ...
    const int c = grid_cell(x[i], y[i], min_x, min_y, inv_w, inv_h);
    if (c >= 0) idx[off[c] + atomicAdd(&cur[c], 1)] = i;
  }
  __syncthreads();
  for (int c = tid; c < GRID_CELLS; c += nthr) {   // ... then restore the push_back order (ascending index)
    const int b = off[c], e = off[c + 1];
    for (int i = b + 1; i < e; ++i) {
      const int v = idx[i];
      int j = i - 1;
      while (j >= b && idx[j] > v) { idx[j + 1] = idx[j]; --j; }
      idx[j + 1] = v;
    }
  }
}

// K7: one CTA per frame.  goff[f][GRID_CELLS+1], gidx[f][stride].
__global__ void __launch_bounds__(256) k_grid_build(const float* __restrict__ x, const float* __restrict__ y,
                                                    const int* __restrict__ nkp, size_t stride, float min_x,
                                                    float max_x, float min_y, float max_y, int* __restrict__ goff,
                                                    int* __restrict__ gidx) {
  __shared__ int off[GRID_CELLS + 1];
  __shared__ int cur[GRID_CELLS];
  __shared__ int ws[33];
  const int f = blockIdx.x, tid = threadIdx.x, nthr = blockDim.x;
  const float inv_w = __fdiv_rn((float)GRID_COLS, __fsub_rn(max_x, min_x));   // src/Frame.cc:221-222
  const float inv_h = __fdiv_rn((float)GRID_ROWS, __fsub_rn(max_y, min_y));
  for (int c = tid; c < GRID_CELLS; c += nthr) cur[c] = 0;
  __syncthreads();
  block_grid_build(x + (size_t)f * stride, y + (size_t)f * stride, nkp[f], min_x, min_y, inv_w, inv_h, off, cur,
                   gidx + (size_t)f * stride, ws);
  int* go = goff + (size_t)f * (GRID_CELLS + 1);
  for (int c = tid; c <= GRID_CELLS; c += nthr) go[c] = off[c];
}

struct QueryGeom {   // what the window walk of one query needs
  float u, v, r, ur, rr;   // centre, window radius, predicted right coordinate, right-coordinate tolerance
  int min_level, max_level;
};

struct WalkCtx {     // per-instance pointers of the current frame
  const int* off;
  const int* idx;
  const float *x, *y, *uright;
  const int *oct, *obs;
  const uint8_t* desc;
  float min_x, min_y, inv_w, inv_h;
  int obs_block_min;   // a pre-existing MapPoint blocks its keypoint iff obs >= this (1: claim rule 0, 0: claim rule 1)
};

// GetFeaturesInArea (src/Frame.cc:465-518) fused with the static part of the candidate loops of the projection
// searches, executed by a whole warp: lanes own consecutive cells of the (ix outer, iy inner) walk, a warp scan turns
// per-cell pass counts into the candidate's position `ord` in the reference's visiting order.  emit(ord, idx, dist)
// is called by the lane that owns the candidate.  Returns the number of candidates (warp-uniform).
template <class Emit>
__device__ __forceinline__ int warp_walk(const WalkCtx& g, const QueryGeom& q, const uint4 d0, const uint4 d1,
                                         Emit emit) {
  const int lane = threadIdx.x & 31;
  const int x0 = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(q.u, g.min_x), q.r), g.inv_w)));
  if (x0 >= GRID_COLS) return 0;
  const int x1 = min(GRID_COLS - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(q.u, g.min_x), q.r), g.inv_w)));
  if (x1 < 0) return 0;
  const int y0 = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(q.v, g.min_y), q.r), g.inv_h)));
  if (y0 >= GRID_ROWS) return 0;
  const int y1 = min(GRID_ROWS - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(q.v, g.min_y), q.r), g.inv_h)));
  if (y1 < 0) return 0;
  if (x1 < x0 || y1 < y0) return 0;
  const bool bCheckLevels = (q.min_level > 0) || (q.max_level >= 0);
  const int ny = y1 - y0 + 1, ncell = (x1 - x0 + 1) * ny;
  auto pass = [&](int idx) -> bool {
    if (bCheckLevels) {
      const int o = g.oct[idx];
      if (o < q.min_level) return false;
      if (q.max_level >= 0 && o > q.max_level) return false;
    }
    const float dx = __fsub_rn(g.x[idx], q.u), dy = __fsub_rn(g.y[idx], q.v);
    if (!(fabsf(dx) < q.r && fabsf(dy) < q.r)) return false;
    if (g.obs && g.obs[idx] >= g.obs_block_min) return false;   // pre-existing MapPoint that blocks: never a candidate
    if (g.uright) {   // stereo / RGB-D gate (null for the overloads without it)
      const float ur = g.uright[idx];
      if (ur > 0) {
        const float er = fabsf(__fsub_rn(q.ur, ur));
        if (er > q.rr) return false;
      }
    }
    return true;
  };
  const int nx = x1 - x0 + 1;
  if (nx <= 32) {
    // Cells are stored column-major (cell = ix*GRID_ROWS + iy), so one grid column of the window is ONE contiguous
    // CSR range [off[ix*48+y0], off[ix*48+y1+1]) already in the reference's visiting order.  Lane j owns column j's
    // range; a warp scan flattens the (few dozen) entries of all columns, and the lanes then test / score 32 entries
    // per step instead of walking cells.
    int rs = 0, len = 0;
    if (lane < nx) {
      const int cbase = (x0 + lane) * GRID_ROWS;
      rs = g.off[cbase + y0];
      len = g.off[cbase + y1 + 1] - rs;
    }
    const int cum = warp_incl_scan(len, lane);
    const int T = __shfl_sync(0xffffffffu, cum, 31);
    int total = 0;
    for (int base = 0; base < T; base += 32) {
      const int t = base + lane;
      int j = 0;
      for (int k = 0; k < nx; ++k) j += (__shfl_sync(0xffffffffu, cum, k) <= t) ? 1 : 0;   // column holding entry t
      const int jj = min(j, nx - 1);
      const int cj = __shfl_sync(0xffffffffu, cum, jj), lj = __shfl_sync(0xffffffffu, len, jj),
                rj = __shfl_sync(0xffffffffu, rs, jj);
      bool ok = false;
      int idx = 0;
      if (t < T) {
        idx = g.idx[rj + (t - (cj - lj))];
        ok = pass(idx);
      }
      const unsigned bal = __ballot_sync(0xffffffffu, ok);
      if (ok) emit(total + __popc(bal & ((1u << lane) - 1u)), idx, hamming256(d0, d1, g.desc + (size_t)idx * 32));
      total += __popc(bal);
    }
    return total;
  }
  int total = 0;
  for (int base = 0; base < ncell; base += 32) {
    const int c = base + lane;
    int e0 = 0, e1 = 0, cnt = 0;
    if (c < ncell) {
      const int cx = c / ny;
      const int cell = (x0 + cx) * GRID_ROWS + (y0 + (c - cx * ny));
      e0 = g.off[cell]; e1 = g.off[cell + 1];
      for (int e = e0; e < e1; ++e) cnt += pass(g.idx[e]) ? 1 : 0;
    }
    const int inc = warp_incl_scan(cnt, lane);
    int r = total + inc - cnt;
    if (cnt) {
      for (int e = e0; e < e1; ++e) {
        const int idx = g.idx[e];
        if (pass(idx)) {
          emit(r, idx, hamming256(d0, d1, g.desc + (size_t)idx * 32));
          ++r;
        }
      }
    }
    total += __shfl_sync(0xffffffffu, inc, 31);
  }
  return total;
}

// ComputeThreeMaxima (src/ORBmatcher.cc:1912-1957) over 30 bin counts; returns the kept bins in keep[3]
__device__ __forceinline__ void three_maxima(const int* hist, int* keep) {
  int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
  for (int i = 0; i < ORBM_HISTO_LENGTH; ++i) {
    const int s = hist[i];
    if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
    else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
    else if (s > max3) { max3 = s; ind3 = i; }
  }
  if ((float)max2 < __fmul_rn(0.1f, (float)max1)) { ind2 = -1; ind3 = -1; }
  else if ((float)max3 < __fmul_rn(0.1f, (float)max1)) { ind3 = -1; }
  keep[0] = ind1; keep[1] = ind2; keep[2] = ind3;
}

__device__ __forceinline__ int rot_bin(float a1, float a2) {   // :1685-1690, factor = 1/HISTO_LENGTH (sic)
  float rot = __fsub_rn(a1, a2);
  if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
  int bin = (int)roundf(__fmul_rn(rot, 1.0f / ORBM_HISTO_LENGTH));
  if (bin == ORBM_HISTO_LENGTH) bin = 0;
  return bin;
}

}  // namespace b200
