// orbx_kernels.cuh -- sm_90a kernels of the ORB extractor (reference: src/ORBextractor.cc).
//
// Data layout in HBM (one batch of F frames, identical geometry):
//   pyramid   level l : F planes of h_l rows x pitch_l bytes (pitch_l = w_l rounded up to 16), no border --
//             the 19-px REFLECT_101 frame of ComputePyramid (:1125-1142) is never read by anything that
//             feeds operator()'s outputs (SURVEY App. B.12); orbx_get_level synthesises it on read-back.
//             Level 0 aliases the caller's device buffer when the batch is already resident and its rows are
//             4-byte aligned; otherwise it is staged into the internal plane, so every plane's rows are aligned.
//   blurred   same layout, GaussianBlur 7x7 sigma 2 of every level (:1094-1095)
//   cand      per frame: one fixed segment per FAST cell (worst-case capacity ceil(iw/2)*ceil(ih/2): strict
//             3x3 NMS forbids 8-adjacent survivors), packed u32 x:12 | y:12 | response:8, row-major in cell
//   cellcnt   per frame, per cell survivor count
//   sel       per (frame, level): quad-tree survivors in the reference's list order, same packing
//   kps/desc  per frame: cap x OrbxKeyPoint (28 B) / cap x 32 B, level-major like operator() concatenates
#pragma once
#include "orbx_host.h"
#define B200_HD __host__ __device__ __forceinline__
#include "../../include/glibc_sincosf.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------------
// K1  pyramid level l from level l-1: cv::resize INTER_LINEAR 8UC1 (SURVEY App. A.2; call site :1134).
//     xt/yt: per destination index {source offset, a0 | a1<<16} with the 11-bit coefficients.
//     One thread -> 4 horizontally adjacent destination pixels -> one 32-bit store.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_resize(const uint8_t* __restrict__ src, int spitch, size_t sfs, int sw,
                                                int sh, uint8_t* __restrict__ dst, int dpitch, size_t dfs,
                                                int dw, int dh, const int2* __restrict__ xt,
                                                const int2* __restrict__ yt) {
  const int dx0 = (blockIdx.x * 32 + threadIdx.x) * 4;
  const int dy = blockIdx.y * 8 + threadIdx.y;
  if (dx0 >= dw || dy >= dh) return;
  const uint8_t* s = src + (size_t)blockIdx.z * sfs;
  uint8_t* d = dst + (size_t)blockIdx.z * dfs;
  const int2 ty = __ldg(&yt[dy]);
  const int sy0 = ty.x, sy1 = min(sy0 + 1, sh - 1);
  const int b0 = (short)(ty.y & 0xffff), b1 = (short)(ty.y >> 16);
  const uint8_t* r0 = s + (size_t)sy0 * spitch;
  const uint8_t* r1 = s + (size_t)sy1 * spitch;
  unsigned out = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int dx = dx0 + i;
    if (dx < dw) {
      const int2 tx = __ldg(&xt[dx]);
      const int x0 = tx.x, x1 = min(x0 + 1, sw - 1);
      const int a0 = (short)(tx.y & 0xffff), a1 = (short)(tx.y >> 16);
      const int h0 = r0[x0] * a0 + r0[x1] * a1;
      const int h1 = r1[x0] * a0 + r1[x1] * a1;
      const int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
      out |= (unsigned)(v & 0xff) << (8 * i);
    }
  }
  *reinterpret_cast<unsigned*>(d + (size_t)dy * dpitch + dx0) = out;   // pitch is a multiple of 16
}

// K1 (group-table path): a thread's 4 adjacent outputs start at a fixed destination column (a multiple of 4), so
// everything that depends only on the columns is tabulated per GROUP: first source word, byte phase, the four PRMT
// selectors (relative to the group's first source byte) and the four coefficient pairs -- two 128-bit loads.  The two
// source rows are funnel-shifted into 8-byte windows that start at the group's first source byte; each output then
// costs one PRMT + one IDP.2A per row plus the vertical pass.  Same integer arithmetic as k_resize (needs scale <= 2:
// the 4 outputs read at most 8 consecutive source bytes).
__global__ void __launch_bounds__(256) k_resize_g(const uint8_t* __restrict__ src, int spitch, size_t sfs, int sh,
                                                  uint8_t* __restrict__ dst, int dpitch, size_t dfs, int dw, int dh,
                                                  const int4* __restrict__ xg /* 2 per group */,
                                                  const int2* __restrict__ yt) {
  const int g = blockIdx.x * 32 + threadIdx.x;
  const int dx0 = g * 4;
  const int dy = blockIdx.y * 8 + threadIdx.y;
  if (dx0 >= dw || dy >= dh) return;
  const uint8_t* s = src + (size_t)blockIdx.z * sfs;
  uint8_t* d = dst + (size_t)blockIdx.z * dfs;
  const int2 ty = __ldg(&yt[dy]);
  const int sy0 = ty.x, sy1 = min(sy0 + 1, sh - 1);
  const int b0 = (short)(ty.y & 0xffff), b1 = (short)(ty.y >> 16);
  const int4 ga = __ldg(&xg[2 * g]), gc = __ldg(&xg[2 * g + 1]);   // {word, 8*phase, selectors, -} / coefficients
  const int wlast = (spitch >> 2) - 1;                              // never read past the row's last word
  const int w0 = ga.x, w1 = min(ga.x + 1, wlast), w2 = min(ga.x + 2, wlast);
  const unsigned* r0 = reinterpret_cast<const unsigned*>(s + (size_t)sy0 * spitch);
  const unsigned* r1 = reinterpret_cast<const unsigned*>(s + (size_t)sy1 * spitch);
  const unsigned a0 = __ldg(r0 + w0), a1 = __ldg(r0 + w1), a2 = __ldg(r0 + w2);
  const unsigned c0 = __ldg(r1 + w0), c1 = __ldg(r1 + w1), c2 = __ldg(r1 + w2);
  const unsigned ph = (unsigned)ga.y;
  const unsigned A_lo = __funnelshift_r(a0, a1, ph), A_hi = __funnelshift_r(a1, a2, ph);   // bytes sx0 .. sx0+7
  const unsigned C_lo = __funnelshift_r(c0, c1, ph), C_hi = __funnelshift_r(c1, c2, ph);
  const unsigned sels = (unsigned)ga.z;
  const int co[4] = {gc.x, gc.y, gc.z, gc.w};
  unsigned out = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const unsigned sel = sels >> (8 * i);   // low two nibbles: bytes d_i, d_i+1 of the window
    const unsigned p0 = __byte_perm(A_lo, A_hi, sel), p1 = __byte_perm(C_lo, C_hi, sel);
    const int h0 = (int)__dp2a_lo((unsigned)co[i], p0, 0u);   // a0*s[x] + a1*s[x+1]
    const int h1 = (int)__dp2a_lo((unsigned)co[i], p1, 0u);
    const int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
    out |= (unsigned)(v & 0xff) << (8 * i);
  }
  *reinterpret_cast<unsigned*>(d + (size_t)dy * dpitch + dx0) = out;   // pitch is a multiple of 16
}

// ---------------------------------------------------------------------------------------------------
// K2  per-cell FAST-9/16 + strict 3x3 NMS with the ini/min threshold fallback
//     (cv::FAST TYPE_9_16 nonmax=true, SURVEY App. A.4; call sites :818,:823; cell loop :798-838).
//     One CTA per (cell, frame).  m(p) = max over 16 arcs of max(min d, min -d) is threshold-independent,
//     so it is evaluated once per pixel; "corner at t" is m > t and the score is m-1.  Survivors are
//     written row-major into the cell's fixed segment, so concatenating the segments cell-major reproduces
//     vToDistributeKeys' order.
// ---------------------------------------------------------------------------------------------------
constexpr int FAST_WARPS = 8;
constexpr int FAST_THREADS = FAST_WARPS * 32;
constexpr int FAST_MAX_ROI = 72;   // ROI side bound enforced at create (cell <= 60 px + 6, padded)
constexpr int FAST_TP_SMALL = 48;  // compile-time tile pitches (>= 3 + ROI width, multiple of 4): ring offsets are
constexpr int FAST_TP_BIG = 80;
constexpr int FAST_QLEN = 256;     // per-warp ring of pixels that passed the compass test (<= 31 pending + 128 new)    // immediates; SMALL serves ROIs up to 45 px (640x480: 43), BIG the general case

// m(p) of one pixel.  Packing: one IMAD per ring pixel gives lo16 = 256 + (c - r), hi16 = 256 + (r - c) (biased,
// both in [1, 511], so no borrow crosses the halves); min3/max3 on s16x2 then evaluate the bright and the dark
// arcs at once: a3[i] = min(v[i..i+2]), a9[i] = min(a3[i], a3[i+3], a3[i+6]) = min over the 9-arc starting at i.
// P = row pitch of the tile in bytes.
template <int P>
__device__ __forceinline__ int fast_m_exact(const uint8_t* c) {
  const int bias = 256 * 65537 - (int)c[0] * 65535;
  unsigned v[16];
  v[0] = (unsigned)((int)c[3 * P] * 65535 + bias);       v[1] = (unsigned)((int)c[3 * P + 1] * 65535 + bias);
  v[2] = (unsigned)((int)c[2 * P + 2] * 65535 + bias);   v[3] = (unsigned)((int)c[P + 3] * 65535 + bias);
  v[4] = (unsigned)((int)c[3] * 65535 + bias);           v[5] = (unsigned)((int)c[-P + 3] * 65535 + bias);
  v[6] = (unsigned)((int)c[-2 * P + 2] * 65535 + bias);  v[7] = (unsigned)((int)c[-3 * P + 1] * 65535 + bias);
  v[8] = (unsigned)((int)c[-3 * P] * 65535 + bias);      v[9] = (unsigned)((int)c[-3 * P - 1] * 65535 + bias);
  v[10] = (unsigned)((int)c[-2 * P - 2] * 65535 + bias); v[11] = (unsigned)((int)c[-P - 3] * 65535 + bias);
  v[12] = (unsigned)((int)c[-3] * 65535 + bias);         v[13] = (unsigned)((int)c[P - 3] * 65535 + bias);
  v[14] = (unsigned)((int)c[2 * P - 2] * 65535 + bias);  v[15] = (unsigned)((int)c[3 * P - 1] * 65535 + bias);
  unsigned a3[16], a9[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) a3[i] = __vimin3_s16x2(v[i], v[(i + 1) & 15], v[(i + 2) & 15]);
#pragma unroll
  for (int i = 0; i < 16; ++i) a9[i] = __vimin3_s16x2(a3[i], a3[(i + 3) & 15], a3[(i + 6) & 15]);
  unsigned m0 = __vimax3_s16x2(a9[0], a9[1], a9[2]);
  unsigned m1 = __vimax3_s16x2(a9[3], a9[4], a9[5]);
  unsigned m2 = __vimax3_s16x2(a9[6], a9[7], a9[8]);
  unsigned m3 = __vimax3_s16x2(a9[9], a9[10], a9[11]);
  unsigned m4 = __vimax3_s16x2(a9[12], a9[13], a9[14]);
  m0 = __vimax3_s16x2(m0, m1, m2);
  m3 = __vimax3_s16x2(m3, m4, a9[15]);
  m0 = __vmaxs2(m0, m3);
  // halves hold 256 + min(d) over the best bright arc / 256 + min(-d) over the best dark arc
  return max(0, max((int)(m0 & 0xffffu), (int)(m0 >> 16)) - 256);
}

// One WARP per (cell, frame), FAST_WARPS cells per CTA, no block-level synchronisation.  Per-warp shared memory: the ROI
// and its score map interleaved row by row (pixel row y at y*2*TP, its score row at y*2*TP + TP, so one base register
// and compile-time offsets address both), a ring of pixels that passed the compass test, and the list of corners.
//   sweep   a thread owns one aligned tile word (4 pixels) of one row, several rows per warp step: compass test;
//           passing pixels are queued;
//   dense   whenever 32 pixels are queued, a full warp evaluates their exact m(p); corners (m > t) go to the corner
//           list -- the queue is FIFO over a row-major sweep, so the list is row-major as well;
//   NMS     32 corners at a time: strict 3x3 maximum, order-preserving compaction into the cell's output segment.
// Level rows are 4-byte aligned (the host stages an unaligned level 0), so the ROI is fetched as aligned 32-bit words
// and kept at the same byte phase (pixel x of the ROI sits at column (x0 & 3) + x).
template <int TP>
__global__ void __launch_bounds__(FAST_THREADS, 4) k_fast_cells(PyrView pyr, const CellDesc* __restrict__ cells,
                                                                int ncells, int slots_per_frame, int ini_th,
                                                                int min_th, unsigned* __restrict__ cand,
                                                                int* __restrict__ cellcnt, int rows_max,
                                                                int clist_cap) {
  extern __shared__ __align__(16) uint8_t fsm[];
  constexpr int P = 2 * TP;   // row pitch of the interleaved tile
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int cell = blockIdx.x * FAST_WARPS + w, f = blockIdx.y;
  if (cell >= ncells) return;
  uint8_t* tile = fsm + (size_t)w * (rows_max * P + 2 * FAST_QLEN + 2 * clist_cap);
  unsigned short* queue = reinterpret_cast<unsigned short*>(tile + (size_t)rows_max * P);
  unsigned short* clist = queue + FAST_QLEN;   // corners at t, row-major
  const CellDesc cd = cells[cell];
  const int l = cd.level, rw = cd.rw, rh = cd.rh;
  const int pitch = pyr.pitch[l];
  const int sh = cd.x0 & 3;   // byte phase of the ROI inside its first word
  {
    const uint8_t* img = pyr.p[l] + (size_t)f * pyr.fstride[l] + (size_t)cd.y0 * pitch + (cd.x0 - sh);
    const int nw = (sh + rw + 3) >> 2;   // words per ROI row (<= (3 + FAST_MAX_ROI + 3) / 4 = 19)
    // up to four rows per warp step: lane = r * nw + k (640x480: nw = 10 -> 3 rows, 30 lanes); no integer division
    const int rpl = (nw <= 8) ? 4 : (nw <= 10) ? 3 : (nw <= 16) ? 2 : 1;
    const int r0 = (lane >= nw) + (lane >= 2 * nw) + (lane >= 3 * nw), k = lane - r0 * nw;
    if (r0 < rpl && k < nw) {
      const unsigned* src = reinterpret_cast<const unsigned*>(img + (size_t)r0 * pitch) + k;
      unsigned* dst = reinterpret_cast<unsigned*>(tile + r0 * P) + k;
      const size_t sstep = (size_t)rpl * (pitch >> 2);
      for (int y = r0; y < rh; y += rpl, src += sstep, dst += rpl * (P / 4)) *dst = __ldg(src);
    }
    // the sweep only writes the scores of corners: clear every score row once (rows 2 .. rh-3 are read by the NMS);
    // tile, P and TP are multiples of 16 bytes: 128-bit stores
    constexpr int QPR = TP / 16;
    for (int i = lane; i < (rh - 4) * QPR; i += 32) {
      const int y = 2 + i / QPR, q = i - (y - 2) * QPR;
      reinterpret_cast<uint4*>(tile + y * P + TP)[q] = make_uint4(0u, 0u, 0u, 0u);
    }
  }
  __syncwarp();
  unsigned* out = cand + (size_t)f * slots_per_frame + cd.slot_off;
  const unsigned lt_mask = (1u << lane) - 1u;
  int total = 0;
  // pass 0: everything at ini_th (pixels with m <= ini_th can neither be corners nor outscore one at that threshold);
  // pass 1 (:821, only when the cell is EMPTY AFTER non-max suppression): the same at min_th.
  for (int pass = 0; pass < 2 && total == 0; ++pass) {
    const int t = pass ? min_th : ini_th;
    if (pass == 1 && ini_th == min_th) break;
    int qh = 0, qn = 0;   // candidate ring (warp-uniform head / fill)
    int cn = 0;           // corners at t found so far (warp-uniform)
    // exact m of the queued pixel `o` (tile offset) of the lanes with `on`, score map + corner list update
    auto dense = [&](int o, bool on) {
      bool cr = false;
      if (on) {
        const int m = fast_m_exact<P>(tile + o);
        cr = m > t;
        tile[o + TP] = (uint8_t)(cr ? m : 0);
      }
      const unsigned cb = __ballot_sync(0xffffffffu, cr);
      if (cr) clist[cn + __popc(cb & lt_mask)] = (unsigned short)o;
      cn += __popc(cb);
    };
    // Word sweep: a thread owns the 4 pixels of one aligned tile word (columns 4g .. 4g+3) of one row; several rows per
    // warp step.  The compass test is necessary for a corner at t: a 9-arc always holds one pixel of each opposite
    // compass pair, and all its pixels lie on the same side of the centre.  It runs on pixel PAIRS in s16x2 lanes,
    // bright and dark polarity in separate registers:
    //   bright: 256 + r - c,  dark: 256 + c - r   (one IADD3 each per ring pixel and pixel pair, operands spread from the
    //   byte lanes by one PRMT), q = min(max(v0, v8), max(v4, v12)) per polarity, hit <=> q > 256 + t in either.
    // Queue positions are the pixels' ranks in ROW-MAJOR order (lanes are ordered (row, word); inside a word by column),
    // so the corner list the dense phase builds stays row-major.
    const unsigned kq = (unsigned)(0x7fff - 256 - t) * 0x10001u;
    const int gA = (sh + 3) >> 2, gB = (sh + rw - 4) >> 2, NW = gB - gA + 1;
    const int RPI = 32 / NW;                       // rows per warp step (NW <= 19 < 32)
    const int rs = lane / NW, g = gA + (lane - rs * NW);
    const int cmin = sh + 3, cmax = sh + rw - 3;   // detection columns [cmin, cmax) in tile coordinates
    const unsigned* trow = reinterpret_cast<const unsigned*>(tile);
    for (int y0 = 3; y0 < rh - 3; y0 += RPI) {
      const int y = y0 + rs;
      unsigned hits = 0;                           // bit k: pixel 4g+k of row y passed
      if (rs < RPI && y < rh - 3) {
        const unsigned* wr = trow + (y * P) / 4;
        const unsigned wc = wr[g], wl = wr[max(g - 1, 0)], wn = wr[g + 1];
        const unsigned w0 = wr[g + (3 * P) / 4], w8 = wr[g - (3 * P) / 4];
        const unsigned w12 = __funnelshift_r(wl, wc, 8);     // bytes x-3 of the four pixels
        const unsigned w4 = __funnelshift_r(wc, wn, 24);     // bytes x+3
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {                     // pixel pairs (0,2) and (1,3)
          const unsigned sel = h2 ? 0x4341u : 0x4240u;
          const unsigned C = __byte_perm(wc, 0u, sel), R0 = __byte_perm(w0, 0u, sel), R8 = __byte_perm(w8, 0u, sel);
          const unsigned R4 = __byte_perm(w4, 0u, sel), R12 = __byte_perm(w12, 0u, sel);
          const unsigned cb = 0x01000100u - C, cd = 0x01000100u + C;   // halves stay in [1, 511]: no borrow / carry across
          const unsigned qb = __vmins2(__vmaxs2(R0 + cb, R8 + cb), __vmaxs2(R4 + cb, R12 + cb));
          const unsigned qd = __vmins2(__vmaxs2(cd - R0, cd - R8), __vmaxs2(cd - R4, cd - R12));
          const unsigned hb = ((qb + kq) | (qd + kq)) & 0x80008000u;
          if (hb & 0x8000u) hits |= 1u << h2;
          if (hb & 0x80000000u) hits |= 4u << h2;
        }
        const int c0 = 4 * g;                                // drop the pixels outside the detection columns
        unsigned cm = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) cm |= ((c0 + k >= cmin) && (c0 + k < cmax)) ? (1u << k) : 0u;
        hits &= cm;
      }
      const unsigned b0 = __ballot_sync(0xffffffffu, hits & 1u), b1 = __ballot_sync(0xffffffffu, hits & 2u);
      const unsigned b2 = __ballot_sync(0xffffffffu, hits & 4u), b3 = __ballot_sync(0xffffffffu, hits & 8u);
      if (hits) {
        int pos = qh + qn + __popc(b0 & lt_mask) + __popc(b1 & lt_mask) + __popc(b2 & lt_mask) + __popc(b3 & lt_mask);
        const int o = y * P + 4 * g;
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (hits & (1u << k)) { queue[pos & (FAST_QLEN - 1)] = (unsigned short)(o + k); ++pos; }
      }
      qn += __popc(b0) + __popc(b1) + __popc(b2) + __popc(b3);
      while (qn >= 32) {
        __syncwarp();
        dense(queue[(qh + lane) & (FAST_QLEN - 1)], true);
        qh += 32;
        qn -= 32;
      }
    }
    __syncwarp();
    dense((lane < qn) ? queue[(qh + lane) & (FAST_QLEN - 1)] : 0, lane < qn);
    __syncwarp();
    // NMS (strict 3x3 maximum of the scores; a neighbour that is no corner at t scores 0) over the corner list, 32
    // corners at a time, + order-preserving compaction (one ballot per batch, running offset).
    for (int base = 0; base < cn; base += 32) {
      bool keep = false;
      int m = 0, o = 0;
      if (base + lane < cn) {
        o = clist[base + lane];
        const uint8_t* qq = tile + o + TP;
        m = qq[0];
        const int n0 = max(max((int)qq[-P - 1], (int)qq[-P]), (int)qq[-P + 1]);
        const int n1 = max(max((int)qq[-1], (int)qq[1]), (int)qq[P - 1]);
        const int n2 = max((int)qq[P], (int)qq[P + 1]);
        keep = m > max(max(max(n0, n1), n2), 1);   // score m-1 vs neighbour scores (m_q-1 if m_q > t, else 0)
      }
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const int y = o / P, x = o - y * P - sh;
        out[total + __popc(bal & lt_mask)] = pack_kp(cd.x0 + x, cd.y0 + y, m - 1);
      }
      total += __popc(bal);
    }
    __syncwarp();
  }
  if (lane == 0) cellcnt[(size_t)f * ncells + cell] = total;
}

// ---------------------------------------------------------------------------------------------------
// K3  DistributeOctTree (src/ORBextractor.cc:540-765) + DivideNode (:478-534), one CTA per (level, frame).
//     The std::list is held as an array in list order (front = index 0); one "round" splits a set of nodes
//     in a given processing order and rebuilds the list exactly as the push_front/erase sequence would:
//       [children of the LAST processed node (n4,n3,n2,n1) ... children of the FIRST processed node]
//       ++ [untouched nodes in their old relative order].
//     Sweep rounds (:608-667) process every node holding >1 keypoints in list order.  Largest-first rounds
//     (:678-739) process them by (size desc, creation desc); nodes created in one round sit in the list in
//     reverse creation order, so "later created first" == "smaller list index first" -- no addresses needed
//     (the reference's heap-address tie-break is replaced by this documented surrogate, SURVEY H3).
//     Keypoints keep their original (cell-major, row-major) index, so "first key with maximal response"
//     (:752-759) is an atomicMax over (response << 24 | ~index).
// ---------------------------------------------------------------------------------------------------
constexpr int QT_THREADS = 512;
constexpr int QT_WARPS = QT_THREADS / 32;
constexpr int QT_UNTOUCHED = 0x40000000;   // flag in QtSmem::cpos: the node keeps its box this round

struct QtScratchView {
  unsigned* qkp;    // [F][slots_per_frame] gathered candidates (contiguous per level at slot_begin[l])
  int* qnode;       // [F][slots_per_frame] list index of each candidate's node
};

// Dynamic shared memory, cap entries per array.  Every array sits at an offset from the one base that depends on cap
// only: a table of array pointers picked at run time would live in local memory.  The list read in a round has parity
// `cur`, the list built from it `cur ^ 1`; box, cnt and the child populations cc are double-buffered by that parity.
struct QtSmem {
  unsigned char* base;
  int cap;
  __device__ short4* box(int par) const { return (short4*)base + par * cap; }
  // [cap][4] keypoints per quadrant of every node: the child populations, counted while the keypoints are re-homed
  __device__ int* cc(int par) const { return (int*)(base + 16 * cap) + par * 4 * cap; }
  __device__ int* cpos() const { return (int*)(base + 48 * cap); }   // [cap][4] new list index of each child
  // the largest-first rank's sort keys, two per entry, over cpos (written only after the sort)
  __device__ unsigned long long* key() const { return (unsigned long long*)(base + 48 * cap); }
  __device__ int* cnt(int par) const { return (int*)(base + 64 * cap) + par * cap; }
  __device__ int* rk() const { return (int*)(base + 72 * cap); }       // processing rank or -1 (largest-first)
  __device__ int* npos() const { return (int*)(base + 76 * cap); }     // new list index of untouched nodes
  __device__ int* byrank() const { return (int*)(base + 80 * cap); }   // node index by processing rank
  __device__ int* pre() const { return (int*)(base + 84 * cap); }      // inclusive prefix of child counts by rank
};

__host__ __device__ inline size_t qt_smem_bytes(int cap) { return (size_t)cap * (2 * 8 + 2 * 4 + 16 + 16 + 16 + 4 * 4); }

// orbx.cu refuses qt_smem_bytes(qt_cap) > 100 KiB, so a list never holds more nodes than this.  A sweep round's scan
// sums (candidate flag | non-empty children << 16) over the list: both fields must stay below their 16 bits.
constexpr int QT_CAP_MAX = 100 * 1024 / 88;
static_assert(QT_CAP_MAX < (1 << 16) && 4 * QT_CAP_MAX < (1 << 15), "quad-tree scan fields overflow");

__device__ __forceinline__ int qt_quadrant(short4 b, unsigned kp) {
  // DivideNode's assignment (:509-523); node boxes are relative to (minBorderX, minBorderY) = (16,16)
  const int x = kp_x(kp) - FAST_BORDER, y = kp_y(kp) - FAST_BORDER;
  const int mx = b.x + ((b.z - b.x + 1) >> 1);   // UL.x + ceil((UR.x-UL.x)/2)
  const int my = b.y + ((b.w - b.y + 1) >> 1);
  return (x < mx) ? ((y < my) ? 0 : 2) : ((y < my) ? 1 : 3);
}

// Shared-memory counter increment with warp aggregation: the early rounds of the quad-tree funnel tens of thousands of
// keypoints into a handful of counters (1 initial node, 4, 16, ... quadrant counters), where plain atomicAdd serialises
// 32-way inside every warp.  Lanes that hit the same counter elect a leader that adds the group's population.
// All 32 lanes must call; `active` masks the tail.
__device__ __forceinline__ void qt_count(int* ctr, int idx, bool active) {
  const unsigned act = __ballot_sync(0xffffffffu, active);
  if (active) {
    const unsigned grp = __match_any_sync(act, idx);
    if ((int)(threadIdx.x & 31) == __ffs(grp) - 1) atomicAdd(&ctr[idx], __popc(grp));
  }
}

// Exclusive scan of one int per thread across the CTA with a single barrier: every warp scans the QT_WARPS warp totals
// itself.  Returns the exclusive prefix; *total = CTA sum.  All threads must call, and a barrier must separate this
// call from the last read of `ws` (>= QT_WARPS ints) by the scan before it.
__device__ __forceinline__ int qt_block_scan(int v, int* ws, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int inc = warp_incl_scan(v, lane);
  if (lane == 31) ws[wid] = inc;
  __syncthreads();
  const int w = (lane < QT_WARPS) ? ws[lane] : 0;
  const int winc = warp_incl_scan(w, lane);
  *total = __shfl_sync(0xffffffffu, winc, 31);
  return __shfl_sync(0xffffffffu, winc - w, wid) + inc - v;
}

// in-place exclusive scan of a[0..n) (shared memory); returns the total. All threads must call; ends with a barrier.
__device__ int qt_scan_array(int* a, int n, int* ws) {
  const int per = (n + QT_THREADS - 1) / QT_THREADS;   // launch contract: blockDim.x == QT_THREADS (a shift, not a division)
  const int beg = min(n, (int)threadIdx.x * per), end = min(n, beg + per);
  int s = 0;
  for (int i = beg; i < end; ++i) s += a[i];
  int total;
  int run = qt_block_scan(s, ws, &total);
  for (int i = beg; i < end; ++i) {
    const int v = a[i];
    a[i] = run;
    run += v;
  }
  __syncthreads();
  return total;
}

__device__ __forceinline__ int qt_nonempty(const int* c) { return (c[0] > 0) + (c[1] > 0) + (c[2] > 0) + (c[3] > 0); }

// A node holding cnt keypoints with child populations c[0..3], as one scan value: candidate flag | non-empty children << 16
__device__ __forceinline__ int qt_split(int cnt, const int* c) { return cnt > 1 ? 1 | (qt_nonempty(c) << 16) : 0; }

// DivideNode (:478-534) of node i of the list of parity cur: its non-empty children n4, n3, n2, n1 take positions
// p, p+1, ... of the list being built.  Returns how many of them hold more than one keypoint.
__device__ __forceinline__ int qt_divide(const QtSmem& S, int cur, int i, int p) {
  const short4 b = S.box(cur)[i];
  const int* c = S.cc(cur) + i * 4;
  const int mx = b.x + ((b.z - b.x + 1) >> 1), my = b.y + ((b.w - b.y + 1) >> 1);
  int exp = 0;
#pragma unroll
  for (int q = 3; q >= 0; --q) {
    const int cq = c[q];
    if (cq > 0) {
      S.cpos()[i * 4 + q] = p;
      short4 nb;
      nb.x = (q & 1) ? mx : b.x;
      nb.z = (q & 1) ? b.z : mx;
      nb.y = (q & 2) ? my : b.y;
      nb.w = (q & 2) ? b.w : my;
      S.box(cur ^ 1)[p] = nb;
      S.cnt(cur ^ 1)[p] = cq;
      exp += (cq > 1);
      ++p;
    }
  }
  return exp;
}

// Bitonic sort of key[0..P) into descending order, P a power of two.  All threads must call; ends with a barrier.
__device__ void qt_sort_desc(unsigned long long* key, int P) {
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll 1
      for (int q = threadIdx.x; q < (P >> 1); q += QT_THREADS) {
        const int i = ((q & ~(j - 1)) << 1) | (q & (j - 1)), l = i | j;   // the pair (i, i + j) of this stage
        const unsigned long long a = key[i], b = key[l];
        if (((i & k) == 0) == (a < b)) {   // descending where bit k of i is clear, ascending where it is set
          key[i] = b;
          key[l] = a;
        }
      }
      __syncthreads();
    }
}

// Register budget: 4 CTAs per SM, 32 registers on sm_90a and no stack frame (at a budget of 2 CTAs per SM the compiler
// takes 46 registers, at 3 it takes 39).  A sweep round costs three barriers (its one scan, and one on each side of the
// re-homing pass), and the budget hardly moves the stage any more.  Measured in bench.py on an H100 SXM (80 GB HBM3,
// 700 W power limit), back to back: the stage takes 7.77 / 7.24 / 7.32-7.41 ms per 4240-frame step at 2 / 3 / 4 CTAs per
// SM (one run each for 2 and 3, three for 4), `value` 52.9 k / 53.9 k / 53.7-54.0 k and `e2e` 37.3 k / 35.6 k /
// 34.5-36.4 k frames/s, all before chained batches ordered their uploads after the other batch's depth reads (orbs.cu):
// the slower stage at 2 CTAs per SM had started those reads later.  With that ordering, 4 CTAs per SM keeps `e2e` at the
// previous kernel's level (34.6-35.4 k against 34.2-35.0 k, alternated), so the budget stays where it was.
constexpr int QT_MIN_CTAS = 4;
__global__ void __launch_bounds__(QT_THREADS, QT_MIN_CTAS) k_quadtree(LevelTab lt, const CellDesc* __restrict__ cells,
                                                            const unsigned* __restrict__ cand,
                                                            const int* __restrict__ cellcnt, int ncells,
                                                            int slots_per_frame, QtScratchView sc, int qt_cap,
                                                            unsigned* __restrict__ sel, int* __restrict__ selcnt,
                                                            int* __restrict__ candcnt, int sel_per_frame) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int ws[33];
  __shared__ int s_coff[QT_THREADS];
  __shared__ int s_expand, s_rstar;
  const int l = blockIdx.x, f = blockIdx.y, tid = threadIdx.x, nthr = blockDim.x;
  const int nlev = lt.nlevels;
  const int N = lt.nfeat[l];
  const QtSmem S{smem_raw, qt_cap};
  const unsigned* fcand = cand + (size_t)f * slots_per_frame;
  const int* fcnt = cellcnt + (size_t)f * ncells;
  // Per-candidate arrays (packed keypoint + node id) stay in the L2-resident global scratch: staging them in shared
  // memory costs CTA-level concurrency.
  unsigned* __restrict__ qkp = sc.qkp + (size_t)f * slots_per_frame + lt.slot_begin[l];
  int* __restrict__ qnode = sc.qnode + (size_t)f * slots_per_frame + lt.slot_begin[l];
  // ---- gather this level's per-cell segments into one contiguous, order-preserving list -----------
  const int cb = lt.cell_begin[l], nc = lt.cell_begin[l + 1] - cb;
  int K = 0;
  for (int base = 0; base < nc; base += nthr) {
    const int c = base + tid;
    const int cn = (c < nc) ? fcnt[cb + c] : 0;
    int tot;
    const int off = block_excl_scan(cn, ws, &tot);
    s_coff[tid] = K + off;
    __syncthreads();
    const int nw = nthr >> 5, w = tid >> 5, lane = tid & 31;
    const int m = min(nthr, nc - base);
    for (int ci = w; ci < m; ci += nw) {
      const int n_c = fcnt[cb + base + ci];
      const unsigned* srcp = fcand + cells[cb + base + ci].slot_off;
      unsigned* dstp = qkp + s_coff[ci];
      for (int i = lane; i < n_c; i += 32) dstp[i] = srcp[i];
    }
    K += tot;
    __syncthreads();
  }
  if (tid == 0) candcnt[(size_t)f * nlev + l] = K;
  if (K == 0) {   // DistributeOctTree on an empty input returns an empty list
    if (tid == 0) selcnt[(size_t)f * nlev + l] = 0;
    return;
  }

  // ---- initial nodes (:553-587) ---------------------------------------------------------------------
  const int nIni = lt.n_ini[l];
  const float hX = lt.hx[l];
  const int boxH = lt.box_h[l];
  int cur = 0;
  int* icnt = S.cc(1);   // nIni counters
  for (int i = tid; i < nIni; i += nthr) icnt[i] = 0;
  __syncthreads();
  for (int k = tid; k < K; k += nthr) {
    const float xr = (float)(kp_x(qkp[k]) - FAST_BORDER);
    int ii = (int)__fdiv_rn(xr, hX);
    ii = min(ii, nIni - 1);
    qnode[k] = ii;
    atomicAdd(&icnt[ii], 1);
  }
  __syncthreads();
  for (int i = tid; i < nIni; i += nthr) S.npos()[i] = (icnt[i] > 0) ? 1 : 0;
  __syncthreads();
  int n = qt_scan_array(S.npos(), nIni, ws);
  for (int i = tid; i < nIni; i += nthr) {
    if (icnt[i] > 0) {
      const int p = S.npos()[i];
      S.box(0)[p] = make_short4((short)(int)__fmul_rn(hX, (float)i), 0, (short)(int)__fmul_rn(hX, (float)(i + 1)),
                                (short)boxH);
      S.cnt(0)[p] = icnt[i];
    }
  }
  for (int i = tid; i < nIni * 4; i += nthr) S.cc(0)[i] = 0;
  __syncthreads();
  // compact the node ids and count, per node, the keypoints of each quadrant (the child populations of round 0)
  for (int k = tid; k < K; k += nthr) {
    const int p = S.npos()[qnode[k]];
    qnode[k] = p;
    atomicAdd(&S.cc(0)[p * 4 + qt_quadrant(S.box(0)[p], qkp[k])], 1);
  }
  __syncthreads();

  // ---- rounds -------------------------------------------------------------------------------------------
  // A thread owns the contiguous list range [beg, end) in the round's scan and in the sweep's writes.  The loops over
  // that range and the sort's pair loop stay rolled: unrolled, they push the per-round state out of the 32 registers.
  for (bool largest = false;;) {
    const short4* box = S.box(cur);
    const int* cnt = S.cnt(cur);
    const int* cc = S.cc(cur);
    if (tid == 0) s_expand = 0;   // last read before the previous round's final barrier
    // (1) one scan of (candidate flag | non-empty children << 16) over the list.  The child populations cc were counted
    //     while the keypoints were re-homed last round.
    const int per = (n + QT_THREADS - 1) / QT_THREADS;
    const int beg = min(n, tid * per), end = min(n, beg + per);
    int run = 0;
    for (int i = beg; i < end; ++i) run += qt_split(cnt[i], cc + i * 4);
    int tot;
    run = qt_block_scan(run, ws, &tot);
    const int m = tot & 0xffff;   // candidates: nodes holding more than one keypoint
    int TC, nUn, myexp = 0;       // children created this round, nodes left untouched
    if (!largest) {
      // (2) sweep round (:608-667): every candidate splits, in list order, so node i's exclusive sums place it.  Its
      //     rank is the number of candidates before it; children of rank r fill [TC - pre[r], TC - pre[r-1]) with pre the
      //     inclusive prefix of non-empty children; an untouched node keeps its order behind all TC children.
      TC = tot >> 16;
      nUn = n - m;
#pragma unroll 1
      for (int i = beg; i < end; ++i) {
        const int v = qt_split(cnt[i], cc + i * 4);
        if (v) {
          myexp += qt_divide(S, cur, i, TC - (run >> 16) - (v >> 16));
        } else {
          const int p = TC + i - (run & 0xffff);
          S.box(cur ^ 1)[p] = box[i];
          S.cnt(cur ^ 1)[p] = cnt[i];
          int* cp = S.cpos() + i * 4;
          cp[0] = cp[1] = cp[2] = cp[3] = p | QT_UNTOUCHED;
        }
        run += v;
      }
    } else {
      // (2) largest-first round (:678-739): candidates in (size desc, list index asc) order, i.e. the 64-bit keys
      //     size << 32 | ~index sorted descending; the scan's flag prefix is each candidate's slot in the key array.
      unsigned long long* key = S.key();
      for (int i = beg; i < end; ++i) {
        const int v = qt_split(cnt[i], cc + i * 4);
        if (v) key[run & 0xffff] = ((unsigned long long)cnt[i] << 32) | (unsigned)~i;
        else S.rk()[i] = -1;
        run += v;
      }
      const int P = (m > 1) ? 1 << (32 - __clz(m - 1)) : m;   // m rounded up to a power of two, <= 2 * cap keys
      for (int r = m + tid; r < P; r += nthr) key[r] = 0;      // below every candidate's key
      __syncthreads();
      qt_sort_desc(key, P);
      for (int r = tid; r < m; r += nthr) {
        const int i = ~(unsigned)key[r];
        S.rk()[i] = r;
        S.byrank()[r] = i;
        S.pre()[r] = qt_nonempty(cc + i * 4);
      }
      if (tid == 0) s_rstar = m - 1;
      __syncthreads();
      // inclusive prefix over processing order of the number of non-empty children
      qt_scan_array(S.pre(), m, ws);   // exclusive in place ...
      for (int r = tid; r < m; r += nthr) S.pre()[r] += qt_nonempty(cc + S.byrank()[r] * 4);   // ... inclusive
      __syncthreads();
      // :732 stop right after the split that reaches N
      for (int r = tid; r < m; r += nthr) {
        const bool now = (n + S.pre()[r] - (r + 1)) >= N;
        const bool before = (r > 0) && ((n + S.pre()[r - 1] - r) >= N);
        if (now && !before) s_rstar = r;
      }
      __syncthreads();
      const int rstar = s_rstar;
      TC = (m > 0) ? S.pre()[rstar] : 0;
      // new list index of untouched nodes
      for (int i = tid; i < n; i += nthr) {
        const int r = S.rk()[i];
        S.npos()[i] = (r < 0 || r > rstar) ? 1 : 0;
      }
      __syncthreads();
      nUn = qt_scan_array(S.npos(), n, ws);
      for (int i = tid; i < n; i += nthr) {
        const int r = S.rk()[i];
        if (r < 0 || r > rstar) {
          const int p = TC + S.npos()[i];
          S.box(cur ^ 1)[p] = box[i];
          S.cnt(cur ^ 1)[p] = cnt[i];
          int* cp = S.cpos() + i * 4;
          cp[0] = cp[1] = cp[2] = cp[3] = p | QT_UNTOUCHED;
        }
      }
      // children: block of rank r starts at TC - pre[r]
      for (int r = tid; r <= rstar && r < m; r += nthr) myexp += qt_divide(S, cur, S.byrank()[r], TC - S.pre()[r]);
    }
    if (myexp) atomicAdd(&s_expand, myexp);
    int* ncc = S.cc(cur ^ 1);
    for (int i = tid; i < (TC + nUn) * 4; i += nthr) ncc[i] = 0;
    __syncthreads();
    const int nToExpand = s_expand;
    // (3) re-home the keypoints; the same pass counts the quadrant populations inside the NEW nodes, i.e. the child
    //     populations the next round needs (one pass over the keypoints per round instead of two)
    // cpos[p][q] holds the new list index for quadrant q of node p -- for untouched nodes the node's own new index in
    // all four entries, flagged -- so the loop needs no branch on the node state and one box load: the child's box, and
    // with it the quadrant the keypoint will fall into NEXT round, follows from the parent's box and q.
    const int* cpos = S.cpos();
    for (int k = tid; k < K; k += nthr) {
      const int p = qnode[k];
      const unsigned kp = qkp[k];
      const short4 b = box[p];
      const int x = kp_x(kp) - FAST_BORDER, y = kp_y(kp) - FAST_BORDER;
      const int mx = b.x + ((b.z - b.x + 1) >> 1), my = b.y + ((b.w - b.y + 1) >> 1);
      const int qx = (x < mx) ? 0 : 1, qy = (y < my) ? 0 : 1;
      const int q = qx | (qy << 1);
      const int v = cpos[p * 4 + q];
      const int np = v & 0x3fffffff;
      int q2 = q;
      if (!(v & QT_UNTOUCHED)) {   // the node was split: quadrant inside child q (DivideNode :478-534 of the child)
        const int cx0 = qx ? mx : b.x, cx1 = qx ? b.z : mx, cy0 = qy ? my : b.y, cy1 = qy ? b.w : my;
        const int cmx = cx0 + ((cx1 - cx0 + 1) >> 1), cmy = cy0 + ((cy1 - cy0 + 1) >> 1);
        q2 = ((x < cmx) ? 0 : 1) | ((y < cmy) ? 0 : 2);
      }
      qnode[k] = np;
      atomicAdd(&ncc[np * 4 + q2], 1);
    }
    const bool grew = (TC + nUn != n);
    n = TC + nUn;
    cur ^= 1;
    __syncthreads();
    // (4) termination logic (:671-675, :736-737)
    if (n >= N || !grew) break;
    if ((n + nToExpand * 3) > N) largest = true;
  }

  // ---- best keypoint of every node (:746-762), output in list order --------------------------------------
  unsigned* best = (unsigned*)S.cc(cur);
  for (int i = tid; i < n; i += nthr) best[i] = 0;
  __syncthreads();
  for (int k = tid; k < K; k += nthr)
    atomicMax(&best[qnode[k]], ((unsigned)kp_r(qkp[k]) << 24) | (0xffffffu - (unsigned)k));
  __syncthreads();
  unsigned* out = sel + (size_t)f * sel_per_frame + lt.sel_off[l];
  for (int i = tid; i < n; i += nthr) out[i] = qkp[0xffffffu - (best[i] & 0xffffffu)];
  if (tid == 0) selcnt[(size_t)f * nlev + l] = n;
}

// ---------------------------------------------------------------------------------------------------
// K5  orientation (IC_Angle :59-88 on the raw level) + steered BRIEF (computeOrbDescriptor :92-131 on the
//     blurred level) + final KeyPoint assembly (:846-856, :1104-1110).  One warp per keypoint at a time.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {   // cv::fastAtan2, SURVEY App. A.5 (no FMA)
  const float scale = (float)(180.0 / 3.14159265358979323846);
  const float P1 = __fmul_rn(0.9997878412794807f, scale), P3 = __fmul_rn(-0.3258083974640975f, scale),
              P5 = __fmul_rn(0.1555786518463281f, scale), P7 = __fmul_rn(-0.04432655554792128f, scale);
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  if (ax >= ay) {
    c = __fdiv_rn(ay, __fadd_rn(ax, 2.2204460492503131e-16f));
    c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(P7, c2), P5), c2), P3), c2), P1), c);
  } else {
    c = __fdiv_rn(ax, __fadd_rn(ay, 2.2204460492503131e-16f));
    c2 = __fmul_rn(c, c);
    a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(P7, c2), P5), c2), P3), c2), P1), c));
  }
  if (x < 0) a = __fsub_rn(180.f, a);
  if (y < 0) a = __fsub_rn(360.f, a);
  return a;
}

constexpr int OD_WARPS = 8;

// The formulation keeps the instruction count down: the straightforward one (a warp per keypoint, the pattern as int8
// pairs, the level found by a scan) is issue-bound, with many of its instructions on the XU pipe (I2F / F2I
// conversions).
//   * a warp handles KPW keypoints, so the per-CTA set-up (pattern into shared memory, level offsets) is paid once per
//     8 * KPW keypoints instead of once per 8;
//   * the pattern sits in shared memory as float4 (x0, y0, x1, y1) per test: one LDS.128 instead of LDS.32 + 4 I2F.S8;
//   * the level of keypoint j comes from one ballot over the per-level inclusive counts (lane q holds level q) instead
//     of an 8-iteration scan per warp;
//   * IC_Angle walks two row pointers (+pitch / -pitch) instead of rebuilding a 64-bit address from u + v * pitch per
//     load, tests the circular mask as v <= vmax(|u|) (umax is non-increasing in v -- checked at create -- so
//     {v : |u| <= umax[v]} is the prefix 1..vmax), and accumulates sum(vp + vm) with one 3-input add per row, the
//     multiplication by u once at the end (exact: integers).
// The descriptor reads its blurred patch from the warp's own shared-memory tile, staged per keypoint with aligned 32-bit
// loads, a lane per (row, word), three rows per warp step.  Gathered straight from the level, each of its 16 byte gathers
// touched 20-30 distinct 128-byte lines (the 32 tests of a step scatter over a 37x37 window).
//   * The tile starts at the word holding x-R, R = OD_BR = 18, and has R/2+1 = 10 words per row: with p = (x-R) & 3 it
//     holds the bytes x-R-p .. x+R+3-p, so it covers x-R .. x+R for every phase, and its last word is the one holding
//     x+R.  Pixel (x+c, y+r) sits at byte (R + r) * 4 * OD_BP + p + R + c.  The host bounds the descriptor's reach over
//     every angle at create (max over the 512 pattern points of round(|(x, y)|), with room for the rounding of the
//     kernel's float ops: 18) and refuses a pattern that reaches further.
//   * Bounds: every FAST cell's detection range lies at least EDGE_THRESHOLD = 19 px inside its level (checked per cell
//     at create; the levels carry no border here), so rows y-18 .. y+18 and columns x-18 .. x+18 exist.  The first word
//     starts at (x-R) & ~3 >= 0; the last one is the word holding x+R <= w-1, and the blurred planes' pitch is a multiple
//     of 16 that is at least w, so no word crosses the row's pitch.
//   * The row pitch in words is odd (11): the 32 scattered byte reads of a descriptor step spread over the banks instead
//     of repeating every 32 / gcd(pitch, 32) rows; the staging stores of three rows (30 words) are conflict-free.
//   * 8 warps x 1628 B of tiles + the 4 KB pattern keep 8 CTAs per SM within a 164 KB shared-memory carve-out, which
//     leaves 92 KB of L1 to the raw rows IC_Angle reads (31 loads of 31 adjacent bytes).  Measured on an H100 SXM (80 GB HBM3, 700 W power limit), serial stage time per 16 x 265 frames
//     of 2000 features: 7.88 ms against 8.08-8.10 for the gathers from global memory; staging the raw patch as well
//     (31 x 9 words more per warp, the shared-memory carve-out at 228 KB and 28 KB of L1 left) took 9.68-9.73 ms, and
//     9.58 with cp.async staging, and 8.31-8.41 / 8.80-8.85 ms at 6 / 4 CTAs per SM.
constexpr int OD_KPW = 4;             // keypoints per warp
constexpr int OD_BR = 18;             // tile reach
constexpr int OD_BW = OD_BR / 2 + 1;  // words per tile row
constexpr int OD_BP = 11;             // tile pitch in words (odd)
constexpr int OD_BROWS = 2 * OD_BR + 1;
static_assert(OD_BR % 2 == 0 && OD_BR <= EDGE_THRESHOLD, "the tile's reach must be even and stay inside the level");
static_assert(OD_BP >= OD_BW && (OD_BP & 1) && 3 * OD_BW <= 32, "tile pitch: wide enough and odd; three rows per step");

__global__ void __launch_bounds__(OD_WARPS * 32, 8) k_orient_desc(LevelTab lt, OrientTab ot, PyrView raw, PyrView blr,
                                                               const float4* __restrict__ patf /* 256 tests */,
                                                               const unsigned* __restrict__ sel,
                                                               const int* __restrict__ selcnt, int sel_per_frame,
                                                               OrbxKeyPoint* __restrict__ kps,
                                                               uint8_t* __restrict__ desc, int* __restrict__ nout,
                                                               int cap) {
  __shared__ float4 spat[256];   // test pr: points 2 pr and 2 pr + 1 of the pattern, as floats
  __shared__ unsigned stile[OD_WARPS][OD_BROWS * OD_BP];   // per warp: the blurred patch of its current keypoint
  for (int i = threadIdx.x; i < 256; i += OD_WARPS * 32) spat[i] = __ldg(patf + i);
  const int f = blockIdx.y, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  // inclusive keypoint counts per level: lane q holds levels 0..q (lanes >= nlevels hold the total)
  const int cq = (lane < lt.nlevels) ? selcnt[(size_t)f * lt.nlevels + lane] : 0;
  const int incl = warp_incl_scan(cq, lane);
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  if (blockIdx.x == 0 && threadIdx.x == 0) nout[f] = min(total, cap);
  const int u = lane - HALF_PATCH_SIZE, au = abs(u);
  int vmaxu = 0;   // rows v = 1 .. vmaxu of column u lie inside the circular patch
#pragma unroll
  for (int v = 1; v <= HALF_PATCH_SIZE; ++v) vmaxu += (au <= ot.umax[v]) ? 1 : 0;
  __syncthreads();
  const int jmax = min(total, cap);
#pragma unroll 1
  for (int i = 0; i < OD_KPW; ++i) {
    const int j = (blockIdx.x * OD_KPW + i) * OD_WARPS + w;
    if (j >= jmax) break;   // warp-uniform
    // level of keypoint j: the first level whose inclusive count exceeds j
    const int l = __popc(__ballot_sync(0xffffffffu, lane < lt.nlevels && incl <= j));
    const int before = __shfl_sync(0xffffffffu, incl, max(l - 1, 0));
    const int idx = j - ((l > 0) ? before : 0);
    const unsigned pk = sel[(size_t)f * sel_per_frame + lt.sel_off[l] + idx];
    const int x = kp_x(pk), y = kp_y(pk);
    const ptrdiff_t rp = raw.pitch[l];
    {
      const int bp4 = blr.pitch[l] >> 2;   // pitches are multiples of 16
      const unsigned* src = reinterpret_cast<const unsigned*>(blr.p[l] + (size_t)f * blr.fstride[l] +
                                                              (size_t)(y - OD_BR) * blr.pitch[l] + ((x - OD_BR) & ~3));
      const int r = lane / OD_BW, k = lane - r * OD_BW;
      __syncwarp();   // the previous keypoint's reads of the tile are done
      if (r < 3) {
#pragma unroll
        for (int yy = 0; yy < OD_BROWS; yy += 3)
          if (yy + r < OD_BROWS) stile[w][(yy + r) * OD_BP + k] = __ldg(src + (size_t)(yy + r) * bp4 + k);
      }
      __syncwarp();
    }
    // ---- IC_Angle: lane <-> column u = lane-15 (31 columns), rows +-v through two walking pointers ----
    int s = 0, m01 = 0;
    if (lane < 31) {
      const uint8_t* pp = raw.p[l] + (size_t)f * raw.fstride[l] + (size_t)y * rp + (x + u);
      const uint8_t* pm = pp;
      s = *pp;
#pragma unroll
      for (int v = 1; v <= HALF_PATCH_SIZE; ++v) {
        pp += rp; pm -= rp;
        if (v <= vmaxu) {
          const int vp = *pp, vm = *pm;
          s += vp + vm;
          m01 += v * (vp - vm);
        }
      }
    }
    int m10 = u * s;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      m10 += __shfl_xor_sync(0xffffffffu, m10, o);
      m01 += __shfl_xor_sync(0xffffffffu, m01, o);
    }
    const float angle = fast_atan2_deg((float)m01, (float)m10);
    // ---- steered BRIEF ----
    const float factorPI = (float)(3.14159265358979323846 / 180.f);
    const float ang = __fmul_rn(angle, factorPI);
    const float a = b200_cosf(ang), b = b200_sinf(ang);   // glibc's cosf / sinf (not correctly rounded): same algorithm
    const uint8_t* bc = reinterpret_cast<const uint8_t*>(stile[w]) + OD_BR * 4 * OD_BP + ((x - OD_BR) & 3) + OD_BR;
    unsigned word = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float4 t = spat[k * 32 + lane];   // test k*32+lane -> bit (k*32+lane) of the descriptor
      const int r0 = __float2int_rn(__fadd_rn(__fmul_rn(t.x, b), __fmul_rn(t.y, a)));
      const int c0 = __float2int_rn(__fsub_rn(__fmul_rn(t.x, a), __fmul_rn(t.y, b)));
      const int r1 = __float2int_rn(__fadd_rn(__fmul_rn(t.z, b), __fmul_rn(t.w, a)));
      const int c1 = __float2int_rn(__fsub_rn(__fmul_rn(t.z, a), __fmul_rn(t.w, b)));
      const int t0 = bc[r0 * (4 * OD_BP) + c0], t1 = bc[r1 * (4 * OD_BP) + c1];
      const unsigned bits = __ballot_sync(0xffffffffu, t0 < t1);
      if (lane == k) word = bits;
    }
    if (lane < 8) reinterpret_cast<unsigned*>(desc + ((size_t)f * cap + j) * 32)[lane] = word;
    if (lane == 0) {
      OrbxKeyPoint kp;
      const float sc = lt.sf[l];
      kp.x = (l != 0) ? __fmul_rn((float)x, sc) : (float)x;
      kp.y = (l != 0) ? __fmul_rn((float)y, sc) : (float)y;
      kp.size = lt.kp_size[l];
      kp.angle = angle;
      kp.response = (float)kp_r(pk);
      kp.octave = l;
      kp.class_id = -1;
      kps[(size_t)f * cap + j] = kp;
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// K4  GaussianBlur 7x7 sigma 2, BORDER_REFLECT_101 (SURVEY App. A.3; call site :1094-1095).
//     Integer kernel [18,34,48,56,48,34,18]/256 in both passes, (v + 32768) >> 16.
//     Register sliding window: one thread owns 4 adjacent columns and walks down BLS_ROWS rows of a strip.  Per row it
//     reads the 10 source bytes as three aligned 32-bit words, builds the byte pairs P_k = b[k] | b[k+2] << 16 with one
//     funnel shift + mask each, and evaluates the horizontal pass on two pixels per register (every partial sum stays
//     below 2^16, so the halves never carry into each other).  The last 7 rows of horizontal sums live in a statically
//     rotated register ring for the vertical pass -- no shared memory, no intermediate plane.  Requires 4-byte aligned
//     rows, which every plane has.
// ---------------------------------------------------------------------------------------------------
constexpr int BLS_ROWS = 35;   // multiple of 7: the ring rotation is unrolled by 7

__device__ __forceinline__ int reflect101(int p, int n) {
  if (n == 1) return 0;
  while (p < 0 || p >= n) p = (p < 0) ? -p : 2 * (n - 1) - p;
  return p;
}

struct HRow { unsigned h02, h13; };   // horizontal sums of pixels (0,2) and (1,3) of the thread's 4 columns

__device__ __forceinline__ HRow blur_hrow_words(unsigned w0, unsigned w1, unsigned w2) {
  // w0..w2 = bytes x0-4 .. x0+7.  P[k] = byte(k+1) | byte(k+3) << 16, i.e. source pixels x0-3+k and x0-1+k
  unsigned P[8];
  P[0] = __funnelshift_r(w0, w1, 8) & 0x00ff00ffu;    // bytes 1,3
  P[1] = __funnelshift_r(w0, w1, 16) & 0x00ff00ffu;   // bytes 2,4
  P[2] = __funnelshift_r(w0, w1, 24) & 0x00ff00ffu;   // bytes 3,5
  P[3] = w1 & 0x00ff00ffu;                            // bytes 4,6
  P[4] = __funnelshift_r(w1, w2, 8) & 0x00ff00ffu;    // bytes 5,7
  P[5] = __funnelshift_r(w1, w2, 16) & 0x00ff00ffu;   // bytes 6,8
  P[6] = __funnelshift_r(w1, w2, 24) & 0x00ff00ffu;   // bytes 7,9
  P[7] = w2 & 0x00ff00ffu;                            // bytes 8,10
  HRow r;   // output pixel i uses source bytes i+1 .. i+7; pair (0,2) = P[0..6], pair (1,3) = P[1..7]
  r.h02 = 18u * (P[0] + P[6]) + 34u * (P[1] + P[5]) + 48u * (P[2] + P[4]) + 56u * P[3];
  r.h13 = 18u * (P[1] + P[7]) + 34u * (P[2] + P[6]) + 48u * (P[3] + P[5]) + 56u * P[4];
  return r;
}

// The same horizontal sums with byte dot products: output pixel i needs the 7 bytes i+1 .. i+7 of the 12-byte window;
// bytes i+1..i+4 and i+5..i+8 are two funnel shifts of the three words (none for i = 3), and two IDP.4A against the
// coefficient words (18,34,48,56) / (48,34,18,0) give the exact integer sum.  h[0..3] are at most 255*256 = 65280.
__device__ __forceinline__ void blur_hrow_dp(unsigned w0, unsigned w1, unsigned w2, unsigned h[4]) {
  constexpr unsigned cA = 18u | (34u << 8) | (48u << 16) | (56u << 24), cB = 48u | (34u << 8) | (18u << 16);
  h[0] = __dp4a(__funnelshift_r(w0, w1, 8), cA, __dp4a(__funnelshift_r(w1, w2, 8), cB, 0u));
  h[1] = __dp4a(__funnelshift_r(w0, w1, 16), cA, __dp4a(__funnelshift_r(w1, w2, 16), cB, 0u));
  h[2] = __dp4a(__funnelshift_r(w0, w1, 24), cA, __dp4a(__funnelshift_r(w1, w2, 24), cB, 0u));
  h[3] = __dp4a(w1, cA, __dp4a(w2, cB, 0u));
}

// interior column groups only (x0 >= 4 and x0 + 8 <= w): three aligned word loads, no border logic
__device__ __forceinline__ HRow blur_hrow(const uint8_t* __restrict__ row, int x0) {
  const unsigned* p = reinterpret_cast<const unsigned*>(row + x0 - 4);
  return blur_hrow_words(__ldg(p), __ldg(p + 1), __ldg(p + 2));
}

// border column groups: the same three words assembled through BORDER_REFLECT_101
__device__ __forceinline__ HRow blur_hrow_border(const uint8_t* __restrict__ row, int x0, int w) {
  unsigned b[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) b[i] = __ldg(row + reflect101(x0 - 4 + i, w));
  return blur_hrow_words(b[0] | (b[1] << 8) | (b[2] << 16) | (b[3] << 24), b[4] | (b[5] << 8) | (b[6] << 16) | (b[7] << 24),
                         b[8] | (b[9] << 8) | (b[10] << 16) | (b[11] << 24));
}

// All levels in ONE launch (a thread walks 35+6 rows sequentially, so a per-level launch is bounded below by that
// latency chain; one launch lets the small levels hide inside the big ones).  One warp per tile, blockIdx.y = frame.
__global__ void __launch_bounds__(32) k_blur7_strip(PyrView src, PyrView dstv, const BlurTile* __restrict__ tiles) {
  const BlurTile t = tiles[blockIdx.x];
  const int l = t.level, w = src.w[l], h = src.h[l];
  const int x0 = t.x0 + threadIdx.x * 4;
  if (x0 < 4 || x0 + 8 > w) return;   // border column groups (<= 3 per row) are done by k_blur7_edges
  const int spitch = src.pitch[l], dpitch = dstv.pitch[l];
  const uint8_t* s = src.p[l] + (size_t)blockIdx.y * src.fstride[l];
  uint8_t* d = dstv.p[l] + (size_t)blockIdx.y * dstv.fstride[l];
  const int y0 = t.y0, y1 = min(h, y0 + BLS_ROWS);
  unsigned ring[7][4];   // unpacked horizontal sums (pixels 0..3) of 7 consecutive rows, slot = row phase
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const HRow r = blur_hrow(s + (size_t)reflect101(y0 - 3 + j, h) * spitch, x0);
    ring[j][0] = r.h02 & 0xffffu; ring[j][2] = r.h02 >> 16; ring[j][1] = r.h13 & 0xffffu; ring[j][3] = r.h13 >> 16;
  }
  for (int yb = y0; yb < y1; yb += 7) {
    if (yb + 7 <= y1) {
      // full block: all 21 source words of the 7 new rows are requested before the first one is used, so a warp keeps
      // 7 rows (2.7 KB) in flight instead of one -- the walk is latency-bound otherwise
      unsigned W[7][3];
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        const unsigned* p = reinterpret_cast<const unsigned*>(s + (size_t)reflect101(yb + k + 3, h) * spitch + x0 - 4);
        W[k][0] = __ldg(p); W[k][1] = __ldg(p + 1); W[k][2] = __ldg(p + 2);
      }
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        blur_hrow_dp(W[k][0], W[k][1], W[k][2], ring[(k + 6) % 7]);
        unsigned out = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const unsigned v = 18u * (ring[k % 7][i] + ring[(k + 6) % 7][i]) + 34u * (ring[(k + 1) % 7][i] + ring[(k + 5) % 7][i]) +
                             48u * (ring[(k + 2) % 7][i] + ring[(k + 4) % 7][i]) + 56u * ring[(k + 3) % 7][i];
          out |= ((v + 32768u) >> 16) << (8 * i);
        }
        *reinterpret_cast<unsigned*>(d + (size_t)(yb + k) * dpitch + x0) = out;   // dst pitch is a multiple of 16
      }
      continue;
    }
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const int y = yb + k;
      if (y < y1) {
        // rows y-3 .. y+2 sit in slots (k+0)%7 .. (k+5)%7; the new row y+3 goes to slot (k+6)%7
        const HRow r = blur_hrow(s + (size_t)reflect101(y + 3, h) * spitch, x0);
        ring[(k + 6) % 7][0] = r.h02 & 0xffffu; ring[(k + 6) % 7][2] = r.h02 >> 16;
        ring[(k + 6) % 7][1] = r.h13 & 0xffffu; ring[(k + 6) % 7][3] = r.h13 >> 16;
        unsigned out = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const unsigned v = 18u * (ring[k % 7][i] + ring[(k + 6) % 7][i]) + 34u * (ring[(k + 1) % 7][i] + ring[(k + 5) % 7][i]) +
                             48u * (ring[(k + 2) % 7][i] + ring[(k + 4) % 7][i]) + 56u * ring[(k + 3) % 7][i];
          out |= ((v + 32768u) >> 16) << (8 * i);
        }
        *reinterpret_cast<unsigned*>(d + (size_t)y * dpitch + x0) = out;   // dst pitch is a multiple of 16
      }
    }
  }
}

// Border column groups of every level (the group at x0 = 0 and the last one or two groups): same register-ring walk
// as k_blur7_strip with the horizontal pass fetched through BORDER_REFLECT_101; one thread per (group, 35-row strip).
// ~3 % of the pixels.
__global__ void __launch_bounds__(64) k_blur7_edges(PyrView src, PyrView dstv, const BlurEdge* __restrict__ edges, int nedges) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nedges) return;
  const BlurEdge e = edges[i];
  const int l = e.level, x0 = e.x0, w = src.w[l], h = src.h[l], spitch = src.pitch[l], dpitch = dstv.pitch[l];
  const uint8_t* s = src.p[l] + (size_t)blockIdx.y * src.fstride[l];
  uint8_t* d = dstv.p[l] + (size_t)blockIdx.y * dstv.fstride[l];
  const int y0 = e.y0, y1 = min(h, y0 + BLS_ROWS);
  unsigned ring[7][4];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const HRow r = blur_hrow_border(s + (size_t)reflect101(y0 - 3 + j, h) * spitch, x0, w);
    ring[j][0] = r.h02 & 0xffffu; ring[j][2] = r.h02 >> 16; ring[j][1] = r.h13 & 0xffffu; ring[j][3] = r.h13 >> 16;
  }
  for (int yb = y0; yb < y1; yb += 7) {
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const int y = yb + k;
      if (y < y1) {
        const HRow r = blur_hrow_border(s + (size_t)reflect101(y + 3, h) * spitch, x0, w);
        ring[(k + 6) % 7][0] = r.h02 & 0xffffu; ring[(k + 6) % 7][2] = r.h02 >> 16;
        ring[(k + 6) % 7][1] = r.h13 & 0xffffu; ring[(k + 6) % 7][3] = r.h13 >> 16;
        unsigned out = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const unsigned v = 18u * (ring[k % 7][q] + ring[(k + 6) % 7][q]) + 34u * (ring[(k + 1) % 7][q] + ring[(k + 5) % 7][q]) +
                             48u * (ring[(k + 2) % 7][q] + ring[(k + 4) % 7][q]) + 56u * ring[(k + 3) % 7][q];
          out |= ((v + 32768u) >> 16) << (8 * q);
        }
        *reinterpret_cast<unsigned*>(d + (size_t)y * dpitch + x0) = out;
      }
    }
  }
}

// bordered level read-back for orbx_get_level (copyMakeBorder BORDER_REFLECT_101, :1136-1142)
__global__ void k_border_copy(const uint8_t* __restrict__ src, int spitch, int w, int h, uint8_t* __restrict__ dst,
                              int dpitch, int B) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w + 2 * B || y >= h + 2 * B) return;
  dst[(size_t)y * dpitch + x] = src[(size_t)reflect101(y - B, h) * spitch + reflect101(x - B, w)];
}

}  // namespace b200
