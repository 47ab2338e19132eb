// orbm_match.cuh -- candidate (K8) and order-exact resolve (K9/K10) kernels of the three searches:
//   LAST    SearchByProjection(Frame&, const Frame&, th, bMono)          src/ORBmatcher.cc:1578-1724
//   POINTS  SearchByProjection(Frame&, const vector<MapPoint*>&, th)      src/ORBmatcher.cc:63-156
//   BOW     SearchByBoW(KeyFrame*, Frame&, vector<MapPoint*>&)            src/ORBmatcher.cc:217-363
#pragma once
#include "orbm_kernels.cuh"

namespace b200 {

constexpr int CAND_WARPS = 8;

struct ListView {            // per query: LCAP entries + count (negative = overflowed, true count = -n)
  unsigned* list;
  int* count;
};

__device__ __forceinline__ WalkCtx make_ctx(const CurView& cv, const MatchCam& cam, int p) {
  WalkCtx g;
  const size_t co = (size_t)p * cv.stride;
  g.off = cv.goff + (size_t)p * (GRID_CELLS + 1);
  g.idx = cv.gidx + co;
  g.x = cv.x + co; g.y = cv.y + co; g.uright = cv.uright + co; g.oct = cv.oct + co;
  g.obs = cv.obs ? cv.obs + co : nullptr;
  g.desc = cv.desc + co * 32;
  g.min_x = cam.min_x; g.min_y = cam.min_y;
  g.inv_w = __fdiv_rn((float)GRID_COLS, __fsub_rn(cam.max_x, cam.min_x));
  g.inv_h = __fdiv_rn((float)GRID_ROWS, __fsub_rn(cam.max_y, cam.min_y));
  g.obs_block_min = 1;
  return g;
}

// forward / backward decision of the LAST search (:1590-1602); warp-uniform
__device__ __forceinline__ void motion_flags(const MatchCam& cam, const float* Tc, const float* Tl, bool& fwd, bool& bwd) {
  float twc[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {   // -Rcw.t()*tcw through the generic (double-accumulating) gemm
    double s = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) s = __dadd_rn(s, __dmul_rn((double)Tc[k * 4 + i], (double)Tc[k * 4 + 3]));
    twc[i] = __double2float_rn(-s);
  }
  const float Rl2[3] = {Tl[8], Tl[9], Tl[10]};
  const float tlc2 = gemm3(Rl2, twc[0], twc[1], twc[2], Tl[11]);
  fwd = (tlc2 > cam.b) && !cam.mono;
  bwd = (-tlc2 > cam.b) && !cam.mono;
}

// Projection + window set-up of one last-frame MapPoint (:1616-1644).
__device__ __forceinline__ bool setup_last_query(const MatchCam& cam, const float* Rt, bool bForward, bool bBackward,
                                                 const float* __restrict__ xw, int octave, QueryGeom& q) {
  const float R0[3] = {Rt[0], Rt[1], Rt[2]}, R1[3] = {Rt[4], Rt[5], Rt[6]}, R2[3] = {Rt[8], Rt[9], Rt[10]};
  const float xc = gemm3(R0, xw[0], xw[1], xw[2], Rt[3]);
  const float yc = gemm3(R1, xw[0], xw[1], xw[2], Rt[7]);
  const float zc = gemm3(R2, xw[0], xw[1], xw[2], Rt[11]);
  const float invzc = __double2float_rn(__ddiv_rn(1.0, (double)zc));   // const float invzc = 1.0/x3Dc.at<float>(2)
  if (invzc < 0) return false;
  const float u = __fadd_rn(__fmul_rn(__fmul_rn(cam.fx, xc), invzc), cam.cx);
  const float v = __fadd_rn(__fmul_rn(__fmul_rn(cam.fy, yc), invzc), cam.cy);
  if (isnan(u) || isnan(v)) return false;   // reference: UB; documented deviation (oracle does the same)
  if (u < cam.min_x || u > cam.max_x) return false;
  if (v < cam.min_y || v > cam.max_y) return false;
  q.u = u; q.v = v;
  q.r = __fmul_rn(cam.th, cam.sf[octave]);
  q.rr = q.r;
  q.ur = __fsub_rn(u, __fmul_rn(cam.bf, invzc));
  if (bForward) { q.min_level = octave; q.max_level = -1; }
  else if (bBackward) { q.min_level = 0; q.max_level = octave; }
  else { q.min_level = octave - 1; q.max_level = octave + 1; }
  return true;
}

// K8 (BOW): queries are (KF keypoint, F node range) pairs prepared by the host merge-join of the two FeatureVectors
struct BowQueries {
  const int* kf_idx;       // realIdxKF of query q
  const int* f_beg;        // range of the matching F node inside f_idx
  const int* f_end;
  const unsigned* f_idx;   // concatenated F node lists (realIdxF)
  const uint8_t* kf_desc;
  const uint8_t* f_desc;
  const float *kf_ang, *f_ang;
  const uint8_t* f_valid;  // nullable: side-2 entries that may be matched at all (KF-KF overload: MapPoint non-NULL && !isBad())
  int nq, nf, nkf;
};

__global__ void __launch_bounds__(CAND_WARPS * 32) k_cand_bow(BowQueries bq, ListView out) {
  const int lane = threadIdx.x & 31;
  const int q = blockIdx.x * CAND_WARPS + (threadIdx.x >> 5);
  if (q >= bq.nq) return;
  const uint8_t* d = bq.kf_desc + (size_t)bq.kf_idx[q] * 32;
  const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(d)), d1 = __ldg(reinterpret_cast<const uint4*>(d) + 1);
  const int b = bq.f_beg[q], n = bq.f_end[q] - b;
  unsigned* list = out.list + (size_t)q * LCAP;
  for (int e = lane; e < n && e < LCAP; e += 32) {
    const unsigned idx = bq.f_idx[b + e];
    list[e] = (bq.f_valid && !bq.f_valid[idx]) ? KEY_INF
                                                : (((unsigned)hamming256(d0, d1, bq.f_desc + (size_t)idx * 32) << 20) | idx);
  }
  if (lane == 0) out.count[q] = (n > LCAP) ? -n : n;
}

// ---------------------------------------------------------------------------------------------------------------------
// K9 helpers: warp-wide "first minimum among unclaimed entries" over one candidate list
// ---------------------------------------------------------------------------------------------------------------------
struct Pick { int idx, dist, ord; };

// entries e = lane and lane+32 held in registers (v0, v1); `skip` = ord to ignore (second-best pass) or -1
__device__ __forceinline__ Pick pick_min(unsigned v0, unsigned v1, int n, const uint8_t* taken, int skip, int lane) {
  unsigned k0 = KEY_INF, k1 = KEY_INF;
  if (lane < n && lane != skip && v0 != KEY_INF && !taken[v0 & 0xfffffu]) k0 = ((v0 >> 20) << 6) | (unsigned)lane;
  if (lane + 32 < n && lane + 32 != skip && v1 != KEY_INF && !taken[v1 & 0xfffffu]) k1 = ((v1 >> 20) << 6) | (unsigned)(lane + 32);
  const unsigned m = __reduce_min_sync(0xffffffffu, min(k0, k1));
  Pick pk{-1, 256, -1};
  if (m != KEY_INF) {
    pk.ord = (int)(m & 63u);
    pk.dist = (int)(m >> 6);
    const unsigned src = (pk.ord < 32) ? v0 : v1;
    pk.idx = (int)(__shfl_sync(0xffffffffu, src, pk.ord & 31) & 0xfffffu);
  }
  return pk;
}

// 64-bit (dist, ord, idx) warp min used by the overflow re-walks
__device__ __forceinline__ unsigned long long warp_min64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o);
    v = (t < v) ? t : v;
  }
  return v;
}
__device__ __forceinline__ unsigned long long key64(int dist, int ord, int idx) {
  return ((unsigned long long)dist << 44) | ((unsigned long long)ord << 22) | (unsigned long long)idx;
}

// Resolve of a query whose candidate list overflowed LCAP: the window walk again, first minimum (dist, ord) among the
// keypoints not claimed so far.  best_idx / best_dist are left alone when there is none.
__device__ __forceinline__ void first_unclaimed_min(const WalkCtx& g, const QueryGeom& q, const uint8_t* desc,
                                                    const uint8_t* taken, int& best_idx, int& best_dist) {
  const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(desc)), d1 = __ldg(reinterpret_cast<const uint4*>(desc) + 1);
  unsigned long long bk = ~0ull;
  warp_walk(g, q, d0, d1, [&](int ord, int idx, int dist) {
    if (!taken[idx]) { const unsigned long long k = key64(dist, ord, idx); bk = (k < bk) ? k : bk; }
  });
  bk = warp_min64(bk);
  if (bk != ~0ull) { best_idx = (int)(bk & 0x3fffffull); best_dist = (int)(bk >> 44); }
}

// rotation histogram + prune shared by LAST and BOW (:1700-1721 / :338-360).  accepted[q] = claimed cur index or -1;
// state[] is the pointer state of the current frame; returns the number of pruned entries (warp-uniform).
__device__ __forceinline__ int prune_rotation(int nq, const int* accepted, const float* qang, const int* qmap,
                                              const float* cang, int* state, int* s_hist, int* s_keep, int lane,
                                              bool state_by_query = false) {
  for (int b = lane; b < ORBM_HISTO_LENGTH; b += 32) s_hist[b] = 0;
  __syncwarp();
  for (int i = lane; i < nq; i += 32) {
    const int idx = accepted[i];
    if (idx >= 0) atomicAdd(&s_hist[rot_bin(qang[qmap ? qmap[i] : i], cang[idx])], 1);
  }
  __syncwarp();
  if (lane == 0) three_maxima(s_hist, s_keep);
  __syncwarp();
  int pr = 0;
  for (int i = lane; i < nq; i += 32) {
    const int idx = accepted[i];
    if (idx >= 0) {
      const int bin = rot_bin(qang[qmap ? qmap[i] : i], cang[idx]);
      if (bin != s_keep[0] && bin != s_keep[1] && bin != s_keep[2]) {
        state[state_by_query ? qmap[i] : idx] = -1;   // every writer stores NULL: order-free
        ++pr;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) pr += __shfl_xor_sync(0xffffffffu, pr, o);
  return pr;
}

// ---------------------------------------------------------------------------------------------------------------------
// Fused LAST search: one CTA per frame pair does K7 + K8 + K9 + K10 with the current frame's keypoints, descriptors
// and 64x48 grid staged in shared memory (every dependent load of the window walk becomes a shared-memory load), and
// the ordered resolve fed through a shared-memory ring of candidate lists that the other warps refill while warp 0
// resolves.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int MF_THREADS = 512;
constexpr int MF_RING = 64;   // candidate lists in flight between the producer warps and the resolving warp
constexpr int MF_LSTR = LCAP + 1;   // slot stride in words: odd, so 32 lanes walking 32 lists hit 32 banks

// grid-build scratch (one counter per cell), reused as the candidate ring: MF_RING lists + lengths, claim flags, ready flags
__host__ __device__ inline size_t mf_ring_bytes() {
  const size_t ring = (size_t)MF_RING * MF_LSTR * 4 + (size_t)3 * MF_RING * 4, grid = (size_t)GRID_CELLS * 4;
  return ((ring > grid ? ring : grid) + 15) & ~(size_t)15;
}
__host__ __device__ inline size_t mf_smem_bytes(int cmax, int lmax) {
  return (size_t)(GRID_CELLS + 1) * 4 + mf_ring_bytes() + (size_t)cmax * (4 + 4 + 4 + 4 + 4 + 32 + 4 + 1) +
         (size_t)lmax * 20 + 64;
}

__global__ void __launch_bounds__(MF_THREADS) k_match_last_fused(CurView cv, LastView lv, MatchCam cam, int* accepted,
                                                                 int* cur2last, int* nmatch, int cmax, int lmax) {
  extern __shared__ __align__(16) unsigned char fsm[];
  __shared__ int ws[33];
  __shared__ int s_hist[ORBM_HISTO_LENGTH];
  __shared__ int s_keep[3];
  __shared__ int s_nacc, s_pruned, s_next, s_consumed;
  const int p = blockIdx.x, tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31, warp = tid >> 5;
  const int nc = cv.n[p], nl = lv.n[p];
  const size_t co = (size_t)p * cv.stride, lo = (size_t)p * lv.stride;
  // carve shared memory
  unsigned char* q = fsm;
  uint4* s_desc = reinterpret_cast<uint4*>(q); q += (size_t)cmax * 32;
  int* s_off = reinterpret_cast<int*>(q); q += (size_t)(GRID_CELLS + 1) * 4;
  int* s_cur = reinterpret_cast<int*>(q); q += mf_ring_bytes();           // grid-build scratch, later the list ring
  int* s_idx = reinterpret_cast<int*>(q); q += (size_t)cmax * 4;
  float* s_x = reinterpret_cast<float*>(q); q += (size_t)cmax * 4;
  float* s_y = reinterpret_cast<float*>(q); q += (size_t)cmax * 4;
  float* s_ur = reinterpret_cast<float*>(q); q += (size_t)cmax * 4;
  int* s_oct = reinterpret_cast<int*>(q); q += (size_t)cmax * 4;
  int* state = reinterpret_cast<int*>(q); q += (size_t)cmax * 4;
  float* q_u = reinterpret_cast<float*>(q); q += (size_t)lmax * 4;      // per-query window geometry (phase B1)
  float* q_v = reinterpret_cast<float*>(q); q += (size_t)lmax * 4;
  float* q_r = reinterpret_cast<float*>(q); q += (size_t)lmax * 4;
  float* q_ur = reinterpret_cast<float*>(q); q += (size_t)lmax * 4;
  int* q_lv = reinterpret_cast<int*>(q); q += (size_t)lmax * 4;         // (min_level + 1) | (max_level + 1) << 8 | ok << 16
  uint8_t* taken = q;
  const int* cobs = cv.obs ? cv.obs + co : nullptr;

  // ---- stage the current frame -------------------------------------------------------------------------------------
  for (int j = tid; j < nc; j += nthr) {
    s_x[j] = cv.x[co + j]; s_y[j] = cv.y[co + j]; s_ur[j] = cv.uright[co + j]; s_oct[j] = cv.oct[co + j];
    state[j] = (cobs && cobs[j] >= 0) ? -2 : -1;
    taken[j] = 0;
  }
  {
    const uint4* gd = reinterpret_cast<const uint4*>(cv.desc + co * 32);
    for (int j = tid; j < nc * 2; j += nthr) s_desc[j] = __ldg(gd + j);
  }
  for (int c = tid; c < GRID_CELLS; c += nthr) s_cur[c] = 0;
  if (tid < ORBM_HISTO_LENGTH) s_hist[tid] = 0;
  if (tid == 0) { s_nacc = 0; s_pruned = 0; }
  __syncthreads();
  // ---- K7 grid in shared memory ---------------------------------------------------------------------------------------
  const float inv_w = __fdiv_rn((float)GRID_COLS, __fsub_rn(cam.max_x, cam.min_x));
  const float inv_h = __fdiv_rn((float)GRID_ROWS, __fsub_rn(cam.max_y, cam.min_y));
  block_grid_build(s_x, s_y, nc, cam.min_x, cam.min_y, inv_w, inv_h, s_off, s_cur, s_idx, ws);
  __syncthreads();
  WalkCtx g;
  g.off = s_off; g.idx = s_idx; g.x = s_x; g.y = s_y; g.uright = s_ur; g.oct = s_oct; g.obs = cobs;
  g.desc = reinterpret_cast<const uint8_t*>(s_desc);
  g.min_x = cam.min_x; g.min_y = cam.min_y; g.inv_w = inv_w; g.inv_h = inv_h; g.obs_block_min = 1;
  bool fwd, bwd;
  motion_flags(cam, cv.Tcw + (size_t)p * 16, lv.Tcw + (size_t)p * 16, fwd, bwd);
  const float* Tc = cv.Tcw + (size_t)p * 16;
  // ---- K8a: projection + window of every query, one THREAD per query (scalar double-precision chain off the
  //      warp-serial path) -----------------------------------------------------------------------------------------
  for (int i = tid; i < nl; i += nthr) {
    int packed = 0;
    if (lv.valid[lo + i]) {
      QueryGeom qg;
      if (setup_last_query(cam, Tc, fwd, bwd, lv.xw + (lo + i) * 3, lv.oct[lo + i], qg)) {
        q_u[i] = qg.u; q_v[i] = qg.v; q_r[i] = qg.r; q_ur[i] = qg.ur;
        packed = ((qg.min_level + 1) & 0xff) | (((qg.max_level + 1) & 0xff) << 8) | (1 << 16);
      }
    }
    q_lv[i] = packed;
  }
  __syncthreads();
  // ---- K8b + K9, decoupled through a shared-memory ring of MF_RING candidate lists ------------------------------------
  // Producer warps (1..15) take queries in order from a counter, build the candidate list of query i in slot i % MF_RING
  // and publish it (ready[slot] = i + 1); warp 0 resolves the queries in order -- the only loop-carried state (claimed
  // current keypoints) lives in that one warp -- and frees the slots (s_consumed).  No block barrier inside: an
  // expensive window only delays its own warp.
  unsigned* ring = reinterpret_cast<unsigned*>(s_cur);   // MF_RING x MF_LSTR words (grid scratch region)
  int* rcnt = reinterpret_cast<int*>(ring + MF_RING * MF_LSTR);   // list lengths (negative: overflowed)
  int* robs = rcnt + MF_RING;                                   // "query claims its match" flags
  volatile int* ready = robs + MF_RING;                         // i + 1 once slot i % MF_RING holds query i
  const int* lobs = lv.obs ? lv.obs + lo : nullptr;
  int* acc = accepted + lo;
  int n_acc = 0;
  for (int j = tid; j < MF_RING; j += nthr) ready[j] = 0;
  if (tid == 0) { s_next = 0; s_consumed = 0; }
  __syncthreads();
  if (warp > 0) {
    const uint4* dbase = reinterpret_cast<const uint4*>(lv.desc + lo * 32);
    for (;;) {
      int i = 0;
      if (lane == 0) i = atomicAdd(&s_next, 1);
      i = __shfl_sync(0xffffffffu, i, 0);
      if (i >= nl) break;
      const int slot = i % MF_RING;
      int cnt = 0;
      const int packed = q_lv[i];
      uint4 d0 = make_uint4(0, 0, 0, 0), d1 = d0;
      if (packed >> 16) { d0 = __ldg(dbase + 2 * (size_t)i); d1 = __ldg(dbase + 2 * (size_t)i + 1); }
      int qobs = cam.last_obs_default;   // requested now, needed when the list is published
      if (lobs && lane == 0) qobs = __ldg(lobs + i);
      // slot still holds query i - MF_RING?  Every lane polls (one broadcast load per iteration, warp-uniform exit): a
      // lane-0-only spin leaves the warp split in two for the whole walk below.
      while (i - *(volatile int*)&s_consumed >= MF_RING) __nanosleep(32);
      __syncwarp();
      if (packed >> 16) {
        QueryGeom qg;
        qg.u = q_u[i]; qg.v = q_v[i]; qg.r = q_r[i]; qg.rr = qg.r; qg.ur = q_ur[i];
        qg.min_level = (packed & 0xff) - 1; qg.max_level = ((packed >> 8) & 0xff) - 1;
        unsigned* list = ring + slot * MF_LSTR;
        cnt = warp_walk(g, qg, d0, d1, [&](int ord, int idx, int dist) {
          if (ord < LCAP) list[ord] = ((unsigned)dist << 20) | (unsigned)idx;
        });
      }
      __syncwarp();
      if (lane == 0) {
        rcnt[slot] = (cnt > LCAP) ? -cnt : cnt;
        robs[slot] = qobs > 0;
        __threadfence_block();
        ready[slot] = i + 1;
      }
    }
  } else {
    // Resolving warp: 32 consecutive queries per step, lane = query.  Every lane picks the first minimum of its own
    // list among the keypoints not claimed so far (speculatively ignoring the other lanes of the step).  A pick is
    // final when no earlier lane of the step claims the same keypoint; all lanes before the first conflicting one are
    // therefore final, the rest pick again in the next round (at least the first open lane finishes per round, and a
    // conflict needs two map points choosing the same keypoint, so one or two rounds are the rule).  The sequential
    // semantics of the reference loop (src/ORBmatcher.cc:1612-1698) are preserved exactly: a claimed keypoint is
    // invisible to later queries, an unclaimed assignment is overwritten by the later query (atomicMax on the query
    // index).  Nothing on this path touches global memory.
    for (int base = 0; base < nl; base += 32) {
      const int i = base + lane;
      const bool active = i < nl;
      const int slot = i % MF_RING;
      while (!__all_sync(0xffffffffu, !active || ready[slot] == i + 1)) __nanosleep(20);
      __syncwarp();
      const int cn = active ? rcnt[slot] : 0;
      const int claims = active ? robs[slot] : 0;
      const unsigned* list = ring + slot * MF_LSTR;
      int a = -1;
      if (__any_sync(0xffffffffu, cn < 0)) {
        // a list of this step overflowed LCAP (rare): resolve the 32 queries one after the other, exact re-walk for
        // the overflowed ones
        for (int t = 0; t < 32 && base + t < nl; ++t) {
          const int it = base + t, st_ = it % MF_RING;
          const int cnt_t = __shfl_sync(0xffffffffu, cn, t);
          int best_idx = -1, best_dist = 256;
          if (cnt_t > 0) {
            const unsigned v0 = ring[st_ * MF_LSTR + lane], v1 = ring[st_ * MF_LSTR + lane + 32];
            unsigned k0 = KEY_INF, k1 = KEY_INF;
            if (lane < cnt_t && !taken[v0 & 0xfffu]) k0 = ((v0 >> 20) << 18) | ((unsigned)lane << 12) | (v0 & 0xfffu);
            if (lane + 32 < cnt_t && !taken[v1 & 0xfffu]) k1 = ((v1 >> 20) << 18) | ((unsigned)(lane + 32) << 12) | (v1 & 0xfffu);
            const unsigned m = __reduce_min_sync(0xffffffffu, min(k0, k1));
            if (m != KEY_INF) { best_idx = (int)(m & 0xfffu); best_dist = (int)(m >> 18); }
          } else if (cnt_t < 0) {
            QueryGeom qg;
            if (setup_last_query(cam, Tc, fwd, bwd, lv.xw + (lo + it) * 3, lv.oct[lo + it], qg))
              first_unclaimed_min(g, qg, lv.desc + (lo + it) * 32, taken, best_idx, best_dist);
          }
          const bool acc_t = best_idx >= 0 && best_dist <= ORBM_TH_HIGH;
          if (acc_t) {
            ++n_acc;
            if (lane == t) {
              a = best_idx;
              state[best_idx] = it;
              if (claims) taken[best_idx] = 1;
            }
          }
          __syncwarp();
        }
      } else {
        unsigned open = __ballot_sync(0xffffffffu, active && cn > 0);
        while (open) {
          int pick = -1;
          if ((open >> lane) & 1u) {
            unsigned best = KEY_INF;   // dist << 18 | position << 12 | index: the first minimum in list order
            for (int e = 0; e < cn; ++e) {
              const unsigned v = list[e];
              if (!taken[v & 0xfffu]) best = min(best, ((v >> 20) << 18) | ((unsigned)e << 12) | (v & 0xfffu));
            }
            if (best != KEY_INF && (int)(best >> 18) <= ORBM_TH_HIGH) pick = (int)(best & 0xfffu);
          }
          // equal picks among the open lanes; a lane conflicts when an EARLIER open lane that claims picked the same
          const unsigned same = __match_any_sync(0xffffffffu, (pick >= 0) ? pick : -1 - lane);
          const unsigned claimers = __ballot_sync(0xffffffffu, pick >= 0 && claims);
          const bool conflict = pick >= 0 && (same & claimers & ((1u << lane) - 1u)) != 0u;
          const unsigned cm = __ballot_sync(0xffffffffu, conflict);
          const unsigned fin = open & (cm ? ((1u << (__ffs(cm) - 1)) - 1u) : 0xffffffffu);
          if ((fin >> lane) & 1u) {
            a = pick;
            if (pick >= 0) {
              atomicMax(&state[pick], i);   // the later query of a step overwrites an unclaimed assignment
              if (claims) taken[pick] = 1;
            }
          }
          n_acc += __popc(__ballot_sync(0xffffffffu, ((fin >> lane) & 1u) && pick >= 0));
          open &= ~fin;
          __syncwarp();
        }
      }
      if (active) q_lv[i] = a;   // accepted index, staged in shared memory (q_lv[i] was consumed by query i's producer)
      __syncwarp();
      if (lane == 0) *(volatile int*)&s_consumed = min(base + 32, nl);
    }
  }
  __syncthreads();
  for (int i = tid; i < nl; i += nthr) acc[i] = q_lv[i];
  if (tid == 0) s_nacc = n_acc;
  __syncthreads();
  // ---- K10 rotation consistency -------------------------------------------------------------------------------------
  const float* lang = lv.ang + lo;
  const float* cang = cv.ang + co;
  if (cam.check_ori) {
    for (int i = tid; i < nl; i += nthr) {
      const int idx = acc[i];
      if (idx >= 0) atomicAdd(&s_hist[rot_bin(lang[i], cang[idx])], 1);
    }
    __syncthreads();
    if (tid == 0) three_maxima(s_hist, s_keep);
    __syncthreads();
    int pr = 0;
    for (int i = tid; i < nl; i += nthr) {
      const int idx = acc[i];
      if (idx >= 0) {
        const int bin = rot_bin(lang[i], cang[idx]);
        if (bin != s_keep[0] && bin != s_keep[1] && bin != s_keep[2]) { state[idx] = -1; ++pr; }
      }
    }
    if (pr) atomicAdd(&s_pruned, pr);
    __syncthreads();
  }
  int* out = cur2last + co;
  for (int j = tid; j < nc; j += nthr) out[j] = state[j];
  if (tid == 0) nmatch[p] = s_nacc - s_pruned;
}

// ---------------------------------------------------------------------------------------------------------------------
// Windowed searches on query geometry held in arrays: every projection search except the fused LAST kernel.  Instance
// p matches queries [p*stride, p*stride + n[p]) against current frame p.
// ---------------------------------------------------------------------------------------------------------------------
struct QueriesView {
  const uint8_t* valid;
  const float *u, *v, *radius, *uright, *ang;   // uright nullable: no stereo gate
  const int *min_level, *max_level, *obs;       // obs nullable: every query has MatchCam::last_obs_default
  const uint8_t* desc;
  const int* n;                                 // per instance
  size_t stride;
};

__device__ __forceinline__ bool setup_generic_query(const QueriesView& qv, size_t i, QueryGeom& q) {
  if (!qv.valid[i]) return false;
  q.u = qv.u[i]; q.v = qv.v[i]; q.r = qv.radius[i]; q.rr = q.r;
  q.ur = qv.uright ? qv.uright[i] : 0.f;
  q.min_level = qv.min_level[i]; q.max_level = qv.max_level[i];
  return !(isnan(q.u) || isnan(q.v));
}

// window walk context of instance p; claim rule 1 lets any pre-existing MapPoint block its keypoint
__device__ __forceinline__ WalkCtx query_ctx(const CurView& cv, const QueriesView& qv, const MatchCam& cam, int p,
                                             int claim_rule) {
  WalkCtx g = make_ctx(cv, cam, p);
  g.obs_block_min = claim_rule ? 0 : 1;
  if (!qv.uright) g.uright = nullptr;
  return g;
}

// K8a of the LAST search when the frames do not fit the fused kernel: projection + window of every last-frame point
// into query arrays laid out like the last frame.  grid = (ceil(lstride / 256), npairs), one thread per query.
__global__ void __launch_bounds__(256) k_last_queries(CurView cv, LastView lv, MatchCam cam, uint8_t* valid, float* u,
                                                      float* v, float* radius, float* uright, int* min_level,
                                                      int* max_level) {
  const int p = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= lv.n[p]) return;
  const size_t k = (size_t)p * lv.stride + i;
  const float* Tc = cv.Tcw + (size_t)p * 16;
  bool fwd, bwd;
  motion_flags(cam, Tc, lv.Tcw + (size_t)p * 16, fwd, bwd);
  QueryGeom q;
  const bool ok = lv.valid[k] && setup_last_query(cam, Tc, fwd, bwd, lv.xw + k * 3, lv.oct[k], q);
  if (ok) { u[k] = q.u; v[k] = q.v; radius[k] = q.r; uright[k] = q.ur; min_level[k] = q.min_level; max_level[k] = q.max_level; }
  valid[k] = ok;
}

// K8: grid = (ceil(stride / CAND_WARPS), instances); one warp per query
__global__ void __launch_bounds__(CAND_WARPS * 32) k_cand_generic(CurView cv, QueriesView qv, MatchCam cam, int claim_rule,
                                                                  ListView out) {
  const int p = blockIdx.y, lane = threadIdx.x & 31;
  const int i = blockIdx.x * CAND_WARPS + (threadIdx.x >> 5);
  if (i >= qv.n[p]) return;
  const size_t k = (size_t)p * qv.stride + i;
  unsigned* list = out.list + k * LCAP;
  int cnt = 0;
  QueryGeom q;
  if (setup_generic_query(qv, k, q)) {
    const uint8_t* d = qv.desc + k * 32;
    const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(d)), d1 = __ldg(reinterpret_cast<const uint4*>(d) + 1);
    const WalkCtx g = query_ctx(cv, qv, cam, p, claim_rule);
    cnt = warp_walk(g, q, d0, d1, [&](int ord, int idx, int dist) {
      if (ord < LCAP) list[ord] = ((unsigned)dist << 20) | (unsigned)idx;
    });
  }
  if (lane == 0) out.count[k] = (cnt > LCAP) ? -cnt : cnt;
}

// K9/K10: one warp per instance.  The queries in order take the first minimum among the unclaimed candidates up to
// max_dist; a query claims its keypoint under claim rule 1, or under rule 0 when its MapPoint has observations.  Then
// the rotation prune.  dynamic smem: state[cmax] ints + taken[cmax] bytes
__global__ void __launch_bounds__(32) k_resolve_generic(CurView cv, QueriesView qv, MatchCam cam, int max_dist,
                                                        int claim_rule, ListView in, int* accepted, int* cur2q,
                                                        int* nmatch, int cmax) {
  extern __shared__ __align__(16) unsigned char rsm[];
  __shared__ int s_hist[ORBM_HISTO_LENGTH];
  __shared__ int s_keep[3];
  int* state = reinterpret_cast<int*>(rsm);
  uint8_t* taken = rsm + (size_t)cmax * 4;
  const int p = blockIdx.x, lane = threadIdx.x;
  const int nc = cv.n[p], nq = qv.n[p];
  const size_t co = (size_t)p * cv.stride, qo = (size_t)p * qv.stride;
  const int* cobs = cv.obs ? cv.obs + co : nullptr;
  const int* qobs = qv.obs ? qv.obs + qo : nullptr;
  int* acc = accepted + qo;
  for (int j = lane; j < nc; j += 32) {
    state[j] = (cobs && cobs[j] >= 0) ? -2 : -1;
    taken[j] = 0;
  }
  __syncwarp();
  const WalkCtx g = query_ctx(cv, qv, cam, p, claim_rule);
  int n_acc = 0;
  // software pipeline: entries of query i+1 are loaded while query i is resolved
  const unsigned* L = in.list + qo * LCAP;
  const int* C = in.count + qo;
  unsigned v0 = 0, v1 = 0;
  int cn = 0;
  if (nq > 0) { cn = C[0]; v0 = L[lane]; v1 = L[lane + 32]; }
  for (int i = 0; i < nq; ++i) {
    unsigned nv0 = 0, nv1 = 0;
    int ncn = 0;
    if (i + 1 < nq) { ncn = C[i + 1]; nv0 = L[(size_t)(i + 1) * LCAP + lane]; nv1 = L[(size_t)(i + 1) * LCAP + lane + 32]; }
    int best_idx = -1, best_dist = 256;
    if (cn > 0) {
      const Pick pk = pick_min(v0, v1, cn, taken, -1, lane);
      best_idx = pk.idx; best_dist = pk.dist;
    } else if (cn < 0) {   // overflowed list: exact re-walk with the claimed filter
      QueryGeom q;
      if (setup_generic_query(qv, qo + i, q)) first_unclaimed_min(g, q, qv.desc + (qo + i) * 32, taken, best_idx, best_dist);
    }
    int a = -1;
    if (best_idx >= 0 && best_dist <= max_dist) {
      a = best_idx;
      ++n_acc;
      if (lane == 0) {
        state[best_idx] = i;
        if (claim_rule || (qobs ? qobs[i] : cam.last_obs_default) > 0) taken[best_idx] = 1;
      }
    }
    if (lane == 0) acc[i] = a;
    __syncwarp();
    v0 = nv0; v1 = nv1; cn = ncn;
  }
  int pruned = 0;
  if (cam.check_ori) pruned = prune_rotation(nq, acc, qv.ang + qo, nullptr, cv.ang + co, state, s_hist, s_keep, lane);
  __syncwarp();
  int* out = cur2q + co;
  for (int j = lane; j < nc; j += 32) out[j] = state[j];
  if (lane == 0) nmatch[p] = n_acc - pruned;
}

// K9 (POINTS): best and second best among unclaimed candidates, level-aware ratio test (:98-152).  The reference's
// `dist < bestDist` / `dist < bestDist2` chain starts both at 256, so a candidate at distance 256 is never recorded:
// it must not become the runner-up, whose level decides whether the ratio test applies at all.
__global__ void __launch_bounds__(32) k_resolve_points(CurView cv, QueriesView qv, MatchCam cam, ListView in, int* f2pt,
                                                       int* nmatch, int cmax) {
  extern __shared__ __align__(16) unsigned char rsm[];
  int* state = reinterpret_cast<int*>(rsm);
  uint8_t* taken = rsm + (size_t)cmax * 4;
  const int lane = threadIdx.x;
  const int nc = cv.n[0];
  for (int j = lane; j < nc; j += 32) {
    state[j] = (cv.obs && cv.obs[j] >= 0) ? -2 : -1;
    taken[j] = 0;
  }
  __syncwarp();
  const WalkCtx g = make_ctx(cv, cam, 0);
  int n_acc = 0;
  const int nq = qv.n[0];
  for (int i = 0; i < nq; ++i) {
    const int cn = in.count[i];
    if (cn == 0) continue;
    int bestIdx = -1, bestDist = 256, bestDist2 = 256, bestLevel = -1, bestLevel2 = -1;
    if (cn > 0) {
      unsigned v0 = in.list[(size_t)i * LCAP + lane], v1 = in.list[(size_t)i * LCAP + lane + 32];
      if ((v0 >> 20) >= 256u) v0 = KEY_INF;
      if ((v1 >> 20) >= 256u) v1 = KEY_INF;
      const Pick p1 = pick_min(v0, v1, cn, taken, -1, lane);
      if (p1.idx >= 0) {
        bestIdx = p1.idx; bestDist = p1.dist; bestLevel = cv.oct[p1.idx];
        const Pick p2 = pick_min(v0, v1, cn, taken, p1.ord, lane);
        if (p2.idx >= 0) { bestDist2 = p2.dist; bestLevel2 = cv.oct[p2.idx]; }
      }
    } else {
      QueryGeom q;
      if (setup_generic_query(qv, i, q)) {
        const uint8_t* d = qv.desc + (size_t)i * 32;
        const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(d)), d1 = __ldg(reinterpret_cast<const uint4*>(d) + 1);
        unsigned long long b1 = ~0ull, b2 = ~0ull;   // two smallest keys per lane
        warp_walk(g, q, d0, d1, [&](int ord, int idx, int dist) {
          if (!taken[idx] && dist < 256) {
            const unsigned long long k = key64(dist, ord, idx);
            if (k < b1) { b2 = b1; b1 = k; } else if (k < b2) b2 = k;
          }
        });
        const unsigned long long m1 = warp_min64(b1);
        if (m1 != ~0ull) {
          bestIdx = (int)(m1 & 0x3fffffull); bestDist = (int)(m1 >> 44); bestLevel = cv.oct[bestIdx];
          const unsigned long long m2 = warp_min64((b1 == m1) ? b2 : b1);
          if (m2 != ~0ull) { bestDist2 = (int)(m2 >> 44); bestLevel2 = cv.oct[(int)(m2 & 0x3fffffull)]; }
        }
      }
    }
    if (bestIdx >= 0 && bestDist <= ORBM_TH_HIGH) {
      if (bestLevel == bestLevel2 && (float)bestDist > __fmul_rn(cam.nnratio, (float)bestDist2)) continue;
      ++n_acc;
      if (lane == 0) {
        state[bestIdx] = i;
        if ((qv.obs ? qv.obs[i] : cam.last_obs_default) > 0) taken[bestIdx] = 1;
      }
      __syncwarp();
    }
  }
  __syncwarp();
  for (int j = lane; j < nc; j += 32) f2pt[j] = state[j];
  if (lane == 0) *nmatch = n_acc;
}

// K9/K10 (BOW): claimed = any assignment (:273-274); TH_LOW and ratio on the two best (:292-299)
// kfkf = 1: SearchByBoW(KeyFrame*, KeyFrame*, vpMatches12) (:665-812): output indexed by the FIRST keyframe's keypoints,
// strict bestDist1 < TH_LOW, side-2 validity filter; kfkf = 0: the (KeyFrame*, Frame&) overload (:217-363).
__global__ void __launch_bounds__(32) k_resolve_bow(BowQueries bq, float nnratio, int check_ori, int kfkf, ListView in,
                                                    int* accepted, int* f2kf, int* nmatch, int cmax) {
  extern __shared__ __align__(16) unsigned char rsm[];
  __shared__ int s_hist[ORBM_HISTO_LENGTH];
  __shared__ int s_keep[3];
  int* state = reinterpret_cast<int*>(rsm);
  uint8_t* taken = rsm + (size_t)cmax * 4;
  const int lane = threadIdx.x;
  const int nstate = kfkf ? bq.nkf : bq.nf;
  for (int j = lane; j < nstate; j += 32) state[j] = -1;
  for (int j = lane; j < bq.nf; j += 32) taken[j] = 0;
  __syncwarp();
  int n_acc = 0;
  for (int q = 0; q < bq.nq; ++q) {
    const int cn = in.count[q];
    int a = -1;
    int best1 = 256, best2 = 256, bestIdx = -1;
    if (cn > 0) {
      const unsigned v0 = in.list[(size_t)q * LCAP + lane], v1 = in.list[(size_t)q * LCAP + lane + 32];
      const Pick p1 = pick_min(v0, v1, cn, taken, -1, lane);
      if (p1.idx >= 0) {
        bestIdx = p1.idx; best1 = p1.dist;
        const Pick p2 = pick_min(v0, v1, cn, taken, p1.ord, lane);
        if (p2.idx >= 0) best2 = p2.dist;
      }
    } else if (cn < 0) {   // long node list: recompute over the whole range
      const uint8_t* d = bq.kf_desc + (size_t)bq.kf_idx[q] * 32;
      const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(d)), d1 = __ldg(reinterpret_cast<const uint4*>(d) + 1);
      unsigned long long b1 = ~0ull, b2 = ~0ull;
      const int b = bq.f_beg[q], n = -cn;
      for (int e = lane; e < n; e += 32) {
        const int idx = (int)bq.f_idx[b + e];
        if (!taken[idx] && !(bq.f_valid && !bq.f_valid[idx])) {
          const unsigned long long k = key64(hamming256(d0, d1, bq.f_desc + (size_t)idx * 32), e, idx);
          if (k < b1) { b2 = b1; b1 = k; } else if (k < b2) b2 = k;
        }
      }
      const unsigned long long m1 = warp_min64(b1);
      if (m1 != ~0ull) {
        bestIdx = (int)(m1 & 0x3fffffull); best1 = (int)(m1 >> 44);
        const unsigned long long m2 = warp_min64((b1 == m1) ? b2 : b1);
        if (m2 != ~0ull) best2 = (int)(m2 >> 44);
      }
    }
    const bool under = kfkf ? (best1 < ORBM_TH_LOW) : (best1 <= ORBM_TH_LOW);   // :751 '<' vs :292 '<='
    if (bestIdx >= 0 && under && (float)best1 < __fmul_rn(nnratio, (float)best2)) {
      a = bestIdx;
      ++n_acc;
      if (lane == 0) {
        if (kfkf) state[bq.kf_idx[q]] = bestIdx; else state[bestIdx] = bq.kf_idx[q];
        taken[bestIdx] = 1;
      }
    }
    if (lane == 0) accepted[q] = a;
    __syncwarp();
  }
  int pruned = 0;
  if (check_ori) pruned = prune_rotation(bq.nq, accepted, bq.kf_ang, bq.kf_idx, bq.f_ang, state, s_hist, s_keep, lane, kfkf != 0);
  __syncwarp();
  for (int j = lane; j < nstate; j += 32) f2kf[j] = state[j];
  if (lane == 0) *nmatch = n_acc - pruned;
}

}  // namespace b200
