// orbm.cu -- host side + C-ABI of the ORB matcher (reference: src/ORBmatcher.cc, include/ORBmatcher.h).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <memory>
#include <new>
#include <vector>

#include "orbm_host.h"
#include "orbm_extra.cuh"

using namespace b200;

namespace {
int resolve_smem(int cmax, size_t* smem, const void* func) {
  *smem = (size_t)cmax * 5 + 16;
  if (*smem > 200 * 1024) { set_error("too many keypoints per frame for the matcher's shared memory"); return B200ORB_EINVAL; }
  if (*smem > 48 * 1024) B200_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem));
  return B200ORB_OK;
}

// The fused LAST kernel stages a frame pair in shared memory, and its resolve key holds a keypoint index in 12 bits.
bool match_last_fused(int cmax, int lmax) { return mf_smem_bytes(cmax, align_up(lmax, 16)) <= 200 * 1024 && cmax <= 4096; }

struct LastScratch {   // the non-fused LAST path: query arrays, grids and candidate lists of every pair
  int *goff, *gidx, *count, *min_level, *max_level;
  unsigned* list;
  uint8_t* valid;
  float *u, *v, *radius, *uright;
};

LastScratch take_last_scratch(Carver& c, int npairs, size_t cstride, size_t lstride) {
  const size_t nc = (size_t)npairs * cstride, nq = (size_t)npairs * lstride;
  LastScratch s;
  s.goff = c.take<int>((size_t)npairs * (GRID_CELLS + 1)); s.gidx = c.take<int>(nc);
  s.list = c.take<unsigned>(nq * LCAP); s.count = c.take<int>(nq);
  s.valid = c.take<uint8_t>(nq); s.u = c.take<float>(nq); s.v = c.take<float>(nq); s.radius = c.take<float>(nq);
  s.uright = c.take<float>(nq); s.min_level = c.take<int>(nq); s.max_level = c.take<int>(nq);
  return s;
}
}  // namespace

size_t match_last_scratch_bytes(int npairs, size_t cstride, size_t lstride) {
  if (match_last_fused(align_up((int)cstride, 16), (int)lstride)) return 0;
  Carver probe;
  take_last_scratch(probe, npairs, cstride, lstride);
  return probe.off;
}

int launch_match_last(const CurView& cv_in, const LastView& lv, const MatchCam& cam, int npairs, void* d_scratch,
                      int* d_accepted, int* d_cur2last, int* d_nmatch, cudaStream_t stream, long long* launches) {
  const int cmax = align_up((int)cv_in.stride, 16), lmax = (int)lv.stride;
  if (match_last_fused(cmax, lmax)) {
    const int lmax16 = align_up(lmax, 16);
    const size_t smem = mf_smem_bytes(cmax, lmax16);
    B200_CUDA(cudaFuncSetAttribute(k_match_last_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_match_last_fused<<<npairs, MF_THREADS, smem, stream>>>(cv_in, lv, cam, d_accepted, d_cur2last, d_nmatch, cmax, lmax16);
    if (launches) *launches += 1;
    B200_CUDA(cudaGetLastError());
    return B200ORB_OK;
  }
  if (!d_scratch) { set_error("no scratch for the non-fused LAST search"); return B200ORB_EINVAL; }
  Carver c(d_scratch);
  const LastScratch s = take_last_scratch(c, npairs, cv_in.stride, lv.stride);
  CurView cv = cv_in;
  cv.goff = s.goff; cv.gidx = s.gidx;
  k_last_queries<<<dim3((lmax + 255) / 256, npairs), 256, 0, stream>>>(cv, lv, cam, s.valid, s.u, s.v, s.radius, s.uright,
                                                                      s.min_level, s.max_level);
  k_grid_build<<<npairs, 256, 0, stream>>>(cv.x, cv.y, cv.n, cv.stride, cam.min_x, cam.max_x, cam.min_y, cam.max_y, s.goff,
                                          s.gidx);
  const QueriesView qv{s.valid, s.u, s.v, s.radius, s.uright, lv.ang, s.min_level, s.max_level, lv.obs, lv.desc, lv.n,
                       lv.stride};
  const ListView lsv{s.list, s.count};
  k_cand_generic<<<dim3((lmax + CAND_WARPS - 1) / CAND_WARPS, npairs), CAND_WARPS * 32, 0, stream>>>(cv, qv, cam, 0, lsv);
  size_t smem;
  B200_CHECK(resolve_smem(cmax, &smem, (const void*)k_resolve_generic));
  k_resolve_generic<<<npairs, 32, smem, stream>>>(cv, qv, cam, ORBM_TH_HIGH, 0, lsv, d_accepted, d_cur2last, d_nmatch, cmax);
  if (launches) *launches += 4;
  B200_CUDA(cudaGetLastError());
  return B200ORB_OK;
}

extern "C" {

int orbm_hamming(const uint8_t a[32], const uint8_t b[32]) {   // DescriptorDistance, src/ORBmatcher.cc:1968-1984
  int d = 0;
  for (int i = 0; i < 32; i += 4) {
    uint32_t x, y;
    memcpy(&x, a + i, 4);
    memcpy(&y, b + i, 4);
    d += __builtin_popcount(x ^ y);
  }
  return d;
}

int orbm_create(int device, orbm_t** out) {
  if (!out) { set_error("null argument"); return B200ORB_EINVAL; }
  *out = nullptr;
  B200_CHECK(check_device(device));
  DeviceGuard g(device);
  std::unique_ptr<orbm> h(new (std::nothrow) orbm());
  if (!h) { set_error("out of host memory"); return B200ORB_EINVAL; }
  h->device = device;
  B200_CHECK(h->stream.create());
  *out = h.release();
  return B200ORB_OK;
}
void orbm_destroy(orbm_t* h) { destroy_handle(h); }
long long orbm_launch_count(const orbm_t* h) { return h ? h->launches : 0; }

static int fill_cam(const OrbmFrame* f, float th, int mono, float nnratio, int check_ori, MatchCam* cam) {
  if (f->nlevels < 1 || f->nlevels > MAX_LEVELS || !f->scale_factors) { set_error("bad scale factor table"); return B200ORB_EINVAL; }
  if (!(f->max_x > f->min_x) || !(f->max_y > f->min_y)) { set_error("bad image bounds"); return B200ORB_EINVAL; }
  memset(cam, 0, sizeof(*cam));
  cam->fx = f->fx; cam->fy = f->fy; cam->cx = f->cx; cam->cy = f->cy; cam->bf = f->bf; cam->b = f->b;
  cam->min_x = f->min_x; cam->max_x = f->max_x; cam->min_y = f->min_y; cam->max_y = f->max_y;
  for (int i = 0; i < f->nlevels; ++i) cam->sf[i] = f->scale_factors[i];
  cam->th = th; cam->nnratio = nnratio; cam->mono = mono; cam->check_ori = check_ori; cam->nlevels = f->nlevels;
  return B200ORB_OK;
}

#define UP(dst, src, count, T)                                                                              \
  B200_CUDA(cudaMemcpyAsync((void*)(dst), (src), sizeof(T) * (size_t)(count), cudaMemcpyHostToDevice, h->stream))

// the current-frame arrays and grid of a single instance
static void take_cur(Carver& c, const OrbmFrame* cur, CurView* cv) {
  const size_t nc = cur->n;
  memset(cv, 0, sizeof(*cv));
  cv->x = c.take<float>(nc); cv->y = c.take<float>(nc); cv->ang = c.take<float>(nc); cv->uright = c.take<float>(nc);
  cv->oct = c.take<int>(nc); cv->desc = c.take<uint8_t>(nc * 32); cv->obs = cur->mp_obs ? c.take<int>(nc) : nullptr;
  cv->n = c.take<int>(1); cv->Tcw = c.take<float>(16);
  cv->goff = c.take<int>(GRID_CELLS + 1); cv->gidx = c.take<int>(nc);
  cv->stride = nc;
}

static int upload_cur(orbm* h, const OrbmFrame* cur, const CurView& cv) {
  const size_t nc = cur->n;
  UP(cv.x, cur->x, nc, float); UP(cv.y, cur->y, nc, float); UP(cv.ang, cur->angle, nc, float);
  UP(cv.uright, cur->uright, nc, float); UP(cv.oct, cur->octave, nc, int); UP(cv.desc, cur->desc, nc * 32, uint8_t);
  if (cv.obs) UP(cv.obs, cur->mp_obs, nc, int);
  UP(cv.n, &cur->n, 1, int); UP(cv.Tcw, cur->Tcw, 16, float);
  return B200ORB_OK;
}

static void grid_build(orbm* h, const CurView& cv, const MatchCam& cam) {
  k_grid_build<<<1, 256, 0, h->stream>>>(cv.x, cv.y, cv.n, cv.stride, cam.min_x, cam.max_x, cam.min_y, cam.max_y,
                                         (int*)cv.goff, (int*)cv.gidx);
}

static int check_cur(const OrbmFrame* cur) {
  if (cur->n < 0 || cur->n >= (1 << 20)) { set_error("bad keypoint count"); return B200ORB_EINVAL; }
  if (cur->n > 0 && (!cur->x || !cur->y || !cur->octave || !cur->angle || !cur->uright || !cur->desc)) {
    set_error("null keypoint array");
    return B200ORB_EINVAL;
  }
  return B200ORB_OK;
}

// both (cur, last) entries: last2cur_accepted == NULL is orbm_search_by_projection_last
static int search_last(orbm_t* h, const OrbmFrame* cur, const OrbmLast* last, float th, int mono, float nnratio,
                       int check_ori, int32_t* cur2last, int32_t* last2cur_accepted, int* nmatches) {
  if (!h || !cur || !last || !cur2last || !nmatches) { set_error("null argument"); return B200ORB_EINVAL; }
  B200_CHECK(check_cur(cur));
  if (last->n < 0) { set_error("bad keypoint count"); return B200ORB_EINVAL; }
  *nmatches = 0;
  if (last2cur_accepted)
    for (int i = 0; i < last->n; ++i) last2cur_accepted[i] = -1;
  if (cur->n == 0) return B200ORB_OK;
  if (last->n == 0) {
    for (int j = 0; j < cur->n; ++j) cur2last[j] = (cur->mp_obs && cur->mp_obs[j] >= 0) ? -2 : -1;
    return B200ORB_OK;
  }
  for (int i = 0; i < last->n; ++i)
    if (last->valid[i] && (last->octave[i] < 0 || last->octave[i] >= cur->nlevels)) { set_error("octave out of range"); return B200ORB_EINVAL; }
  MatchCam cam;
  B200_CHECK(fill_cam(cur, th, mono, nnratio, check_ori, &cam));
  cam.last_obs_default = 0;
  DeviceGuard g(h->device);
  const size_t nc = cur->n, nl = last->n;
  CurView cv;
  LastView lv{};
  int *d_out, *d_nm, *d_acc;
  uint8_t* d_scratch;
  B200_CHECK(h->arena.reserve(h->stream, [&](Carver& c) {
    take_cur(c, cur, &cv);
    lv.xw = c.take<float>(nl * 3); lv.valid = c.take<uint8_t>(nl); lv.oct = c.take<int>(nl); lv.ang = c.take<float>(nl);
    lv.desc = c.take<uint8_t>(nl * 32); lv.obs = last->mp_obs ? c.take<int>(nl) : nullptr;
    lv.n = c.take<int>(1); lv.Tcw = c.take<float>(16); lv.stride = nl;
    d_out = c.take<int>(nc); d_nm = c.take<int>(1); d_acc = c.take<int>(nl);
    d_scratch = c.take<uint8_t>(match_last_scratch_bytes(1, nc, nl));
  }));
  B200_CHECK(upload_cur(h, cur, cv));
  UP(lv.xw, last->xw, nl * 3, float); UP(lv.valid, last->valid, nl, uint8_t); UP(lv.oct, last->octave, nl, int);
  UP(lv.ang, last->angle, nl, float); UP(lv.desc, last->mp_desc, nl * 32, uint8_t);
  if (lv.obs) UP(lv.obs, last->mp_obs, nl, int);
  UP(lv.n, &last->n, 1, int); UP(lv.Tcw, last->Tcw, 16, float);
  B200_CHECK(launch_match_last(cv, lv, cam, 1, d_scratch, d_acc, d_out, d_nm, h->stream, &h->launches));
  B200_CUDA(cudaMemcpyAsync(cur2last, d_out, sizeof(int) * nc, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(nmatches, d_nm, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (last2cur_accepted)
    B200_CUDA(cudaMemcpyAsync(last2cur_accepted, d_acc, sizeof(int) * nl, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int orbm_search_by_projection_last(orbm_t* h, const OrbmFrame* cur, const OrbmLast* last, float th, int mono,
                                   float nnratio, int check_ori, int32_t* cur2last, int* nmatches) {
  return search_last(h, cur, last, th, mono, nnratio, check_ori, cur2last, nullptr, nmatches);
}

int orbm_search_by_projection_last_pairs(orbm_t* h, const OrbmFrame* cur, const OrbmLast* last, float th, int mono,
                                         float nnratio, int check_ori, int32_t* cur2last, int32_t* last2cur_accepted,
                                         int* nmatches) {
  if (!last2cur_accepted) { set_error("null argument"); return B200ORB_EINVAL; }
  return search_last(h, cur, last, th, mono, nnratio, check_ori, cur2last, last2cur_accepted, nmatches);
}

int orbm_search_by_projection_points(orbm_t* h, const OrbmFrame* f, const OrbmTrackPoints* pts, float th, float nnratio,
                                     int32_t* f2pt, int* nmatches) {
  if (!h || !f || !pts || !f2pt || !nmatches) { set_error("null argument"); return B200ORB_EINVAL; }
  B200_CHECK(check_cur(f));
  if (pts->n < 0) { set_error("bad point count"); return B200ORB_EINVAL; }
  *nmatches = 0;
  if (f->n == 0) return B200ORB_OK;
  if (pts->n == 0) {
    for (int j = 0; j < f->n; ++j) f2pt[j] = (f->mp_obs && f->mp_obs[j] >= 0) ? -2 : -1;
    return B200ORB_OK;
  }
  MatchCam cam;
  B200_CHECK(fill_cam(f, th, 0, nnratio, 0, &cam));
  cam.last_obs_default = 1;
  // the window of every point in view (:79-91): radius RadiusByViewingCos (:159-165) * th * mvScaleFactors[level],
  // levels [level - 1, level]
  const size_t nc = f->n, np = pts->n;
  std::vector<float> radius(np, 0.f);
  std::vector<int> min_level(np, 0), max_level(np, 0);
  for (size_t i = 0; i < np; ++i) {
    if (!pts->track_in_view[i]) continue;
    const int lvl = pts->scale_level[i];
    if (lvl < 0 || lvl >= f->nlevels) { set_error("scale level out of range"); return B200ORB_EINVAL; }
    float r = ((double)pts->view_cos[i] > 0.998) ? 2.5f : 4.0f;
    if (th != 1.0f) r *= th;
    radius[i] = r * f->scale_factors[lvl];
    min_level[i] = lvl - 1; max_level[i] = lvl;
  }
  DeviceGuard g(h->device);
  CurView cv;
  QueriesView qv{};
  ListView lsv;
  int *d_out, *d_nm;
  B200_CHECK(h->arena.reserve(h->stream, [&](Carver& c) {
    take_cur(c, f, &cv);
    qv.valid = c.take<uint8_t>(np); qv.u = c.take<float>(np); qv.v = c.take<float>(np); qv.radius = c.take<float>(np);
    qv.uright = c.take<float>(np); qv.min_level = c.take<int>(np); qv.max_level = c.take<int>(np);
    qv.obs = pts->mp_obs ? c.take<int>(np) : nullptr; qv.desc = c.take<uint8_t>(np * 32); qv.n = c.take<int>(1);
    qv.stride = np;
    lsv.list = c.take<unsigned>(np * LCAP); lsv.count = c.take<int>(np);
    d_out = c.take<int>(nc); d_nm = c.take<int>(1);
  }));
  B200_CHECK(upload_cur(h, f, cv));
  UP(qv.valid, pts->track_in_view, np, uint8_t); UP(qv.u, pts->proj_x, np, float); UP(qv.v, pts->proj_y, np, float);
  UP(qv.radius, radius.data(), np, float); UP(qv.uright, pts->proj_xr, np, float);
  UP(qv.min_level, min_level.data(), np, int); UP(qv.max_level, max_level.data(), np, int);
  UP(qv.desc, pts->mp_desc, np * 32, uint8_t);
  if (qv.obs) UP(qv.obs, pts->mp_obs, np, int);
  UP(qv.n, &pts->n, 1, int);
  grid_build(h, cv, cam);
  k_cand_generic<<<((int)np + CAND_WARPS - 1) / CAND_WARPS, CAND_WARPS * 32, 0, h->stream>>>(cv, qv, cam, 0, lsv);
  size_t smem;
  const int cmax = align_up((int)nc, 16);
  B200_CHECK(resolve_smem(cmax, &smem, (const void*)k_resolve_points));
  k_resolve_points<<<1, 32, smem, h->stream>>>(cv, qv, cam, lsv, d_out, d_nm, cmax);
  h->launches += 3;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(f2pt, d_out, sizeof(int) * nc, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(nmatches, d_nm, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int orbm_search_projected(orbm_t* h, const OrbmFrame* cur, const OrbmQueries* q, int max_dist, int claim_rule,
                          int check_ori, int32_t* cur2q, int* nmatches) {
  if (!h || !cur || !q || !cur2q || !nmatches) { set_error("null argument"); return B200ORB_EINVAL; }
  B200_CHECK(check_cur(cur));
  if (q->n < 0) { set_error("bad query count"); return B200ORB_EINVAL; }
  *nmatches = 0;
  if (cur->n == 0) return B200ORB_OK;
  if (q->n == 0) {
    for (int j = 0; j < cur->n; ++j) cur2q[j] = (cur->mp_obs && cur->mp_obs[j] >= 0) ? -2 : -1;
    return B200ORB_OK;
  }
  if (!q->valid || !q->u || !q->v || !q->radius || !q->min_level || !q->max_level || !q->desc || (check_ori && !q->angle)) {
    set_error("null query array");
    return B200ORB_EINVAL;
  }
  MatchCam cam;
  B200_CHECK(fill_cam(cur, 0.f, 0, 0.f, check_ori, &cam));
  cam.last_obs_default = 1;   // OrbmQueries::obs NULL: every query claims its match
  DeviceGuard g(h->device);
  const size_t nc = cur->n, nq = q->n;
  CurView cv;
  QueriesView qv{};
  ListView lsv;
  int *d_acc, *d_out, *d_nm;
  B200_CHECK(h->arena.reserve(h->stream, [&](Carver& c) {
    take_cur(c, cur, &cv);
    qv.valid = c.take<uint8_t>(nq); qv.u = c.take<float>(nq); qv.v = c.take<float>(nq); qv.radius = c.take<float>(nq);
    qv.min_level = c.take<int>(nq); qv.max_level = c.take<int>(nq); qv.uright = q->uright ? c.take<float>(nq) : nullptr;
    qv.ang = c.take<float>(nq); qv.obs = q->obs ? c.take<int>(nq) : nullptr; qv.desc = c.take<uint8_t>(nq * 32);
    qv.n = c.take<int>(1); qv.stride = nq;
    lsv.list = c.take<unsigned>(nq * LCAP); lsv.count = c.take<int>(nq);
    d_acc = c.take<int>(nq); d_out = c.take<int>(nc); d_nm = c.take<int>(1);
  }));
  B200_CHECK(upload_cur(h, cur, cv));
  UP(qv.valid, q->valid, nq, uint8_t); UP(qv.u, q->u, nq, float); UP(qv.v, q->v, nq, float);
  UP(qv.radius, q->radius, nq, float); UP(qv.min_level, q->min_level, nq, int); UP(qv.max_level, q->max_level, nq, int);
  UP(qv.desc, q->desc, nq * 32, uint8_t);
  if (qv.uright) UP(qv.uright, q->uright, nq, float);
  if (q->angle) UP(qv.ang, q->angle, nq, float);
  if (qv.obs) UP(qv.obs, q->obs, nq, int);
  UP(qv.n, &q->n, 1, int);
  grid_build(h, cv, cam);
  k_cand_generic<<<((int)nq + CAND_WARPS - 1) / CAND_WARPS, CAND_WARPS * 32, 0, h->stream>>>(cv, qv, cam, claim_rule, lsv);
  size_t smem;
  const int cmax = align_up((int)nc, 16);
  B200_CHECK(resolve_smem(cmax, &smem, (const void*)k_resolve_generic));
  k_resolve_generic<<<1, 32, smem, h->stream>>>(cv, qv, cam, max_dist, claim_rule, lsv, d_acc, d_out, d_nm, cmax);
  h->launches += 3;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(cur2q, d_out, sizeof(int) * nc, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(nmatches, d_nm, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int orbm_search_best(orbm_t* h, const OrbmFrame* kf, const OrbmQueries* q, int gate, const float* inv_level_sigma2,
                     int32_t* best_idx, int32_t* best_dist) {
  if (!h || !kf || !q || !best_idx || !best_dist) { set_error("null argument"); return B200ORB_EINVAL; }
  B200_CHECK(check_cur(kf));
  if (q->n < 0) { set_error("bad query count"); return B200ORB_EINVAL; }
  for (int i = 0; i < q->n; ++i) { best_idx[i] = -1; best_dist[i] = 0x7fffffff; }
  if (kf->n == 0 || q->n == 0) return B200ORB_OK;
  if (!q->valid || !q->u || !q->v || !q->radius || !q->min_level || !q->max_level || !q->desc) { set_error("null query array"); return B200ORB_EINVAL; }
  if (gate == 1 && (!inv_level_sigma2 || !q->uright)) { set_error("the Fuse gate needs inv_level_sigma2 and the predicted right coordinates"); return B200ORB_EINVAL; }
  if (gate != 0 && gate != 1) { set_error("bad gate"); return B200ORB_EINVAL; }
  MatchCam cam;
  B200_CHECK(fill_cam(kf, 0.f, 0, 0.f, 0, &cam));
  DeviceGuard g(h->device);
  const size_t nq = q->n;
  OrbmFrame kf2 = *kf;
  kf2.mp_obs = nullptr;
  CurView cv;
  QueriesView qv{};
  float* d_is2;
  int *d_bi, *d_bd;
  B200_CHECK(h->arena.reserve(h->stream, [&](Carver& c) {
    take_cur(c, &kf2, &cv);
    qv.valid = c.take<uint8_t>(nq); qv.u = c.take<float>(nq); qv.v = c.take<float>(nq); qv.radius = c.take<float>(nq);
    qv.min_level = c.take<int>(nq); qv.max_level = c.take<int>(nq); qv.uright = q->uright ? c.take<float>(nq) : nullptr;
    qv.desc = c.take<uint8_t>(nq * 32); qv.n = c.take<int>(1); qv.stride = nq;
    d_is2 = c.take<float>(MAX_LEVELS); d_bi = c.take<int>(nq); d_bd = c.take<int>(nq);
  }));
  B200_CHECK(upload_cur(h, &kf2, cv));
  UP(qv.valid, q->valid, nq, uint8_t); UP(qv.u, q->u, nq, float); UP(qv.v, q->v, nq, float);
  UP(qv.radius, q->radius, nq, float); UP(qv.min_level, q->min_level, nq, int); UP(qv.max_level, q->max_level, nq, int);
  UP(qv.desc, q->desc, nq * 32, uint8_t);
  if (qv.uright) UP(qv.uright, q->uright, nq, float);
  UP(qv.n, &q->n, 1, int);
  if (gate == 1) UP(d_is2, inv_level_sigma2, kf->nlevels, float);
  BestGate bg{gate, d_is2, cv.uright};
  grid_build(h, cv, cam);
  k_best_generic<<<((int)nq + CAND_WARPS - 1) / CAND_WARPS, CAND_WARPS * 32, 0, h->stream>>>(cv, qv, cam, bg, d_bi, d_bd);
  h->launches += 2;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(best_idx, d_bi, sizeof(int) * nq, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(best_dist, d_bd, sizeof(int) * nq, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int orbm_search_for_initialization(orbm_t* h, const OrbmFrame* f1, const OrbmFrame* f2, float* prev_xy, int window,
                                   float nnratio, int check_ori, int32_t* matches12, int* nmatches) {
  if (!h || !f1 || !f2 || !prev_xy || !matches12 || !nmatches) { set_error("null argument"); return B200ORB_EINVAL; }
  B200_CHECK(check_cur(f1));
  B200_CHECK(check_cur(f2));
  *nmatches = 0;
  for (int i = 0; i < f1->n; ++i) matches12[i] = -1;
  if (f1->n == 0 || f2->n == 0) return B200ORB_OK;
  MatchCam cam;
  B200_CHECK(fill_cam(f2, 0.f, 0, nnratio, check_ori, &cam));
  DeviceGuard g(h->device);
  const size_t n1 = f1->n, n2 = f2->n;
  OrbmFrame f2c = *f2;
  f2c.mp_obs = nullptr;
  CurView cv;
  InitView iv{};
  int *d_out, *d_nm;
  B200_CHECK(h->arena.reserve(h->stream, [&](Carver& c) {
    take_cur(c, &f2c, &cv);
    iv.oct1 = c.take<int>(n1); iv.ang1 = c.take<float>(n1); iv.desc1 = c.take<uint8_t>(n1 * 32);
    iv.prev_xy = c.take<float>(n1 * 2); iv.matched_dist = c.take<int>(n2); iv.match21 = c.take<int>(n2);
    iv.bin1 = c.take<int>(n1); iv.n1 = (int)n1;
    d_out = c.take<int>(n1); d_nm = c.take<int>(1);
  }));
  B200_CHECK(upload_cur(h, &f2c, cv));
  UP(iv.oct1, f1->octave, n1, int); UP(iv.ang1, f1->angle, n1, float); UP(iv.desc1, f1->desc, n1 * 32, uint8_t);
  UP(iv.prev_xy, prev_xy, n1 * 2, float);
  grid_build(h, cv, cam);
  k_init_search<<<1, 32, 0, h->stream>>>(cv, iv, cam, window, nnratio, check_ori, d_out, d_nm);
  h->launches += 2;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(matches12, d_out, sizeof(int) * n1, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(prev_xy, iv.prev_xy, sizeof(float) * 2 * n1, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(nmatches, d_nm, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int orbm_search_for_triangulation(orbm_t* h, const OrbmTriKF* k1, const OrbmTriKF* k2, const float F12[9], float ex, float ey,
                                  const float* scale_factors2, const float* level_sigma2_2, int nlevels, int only_stereo,
                                  int check_ori, int32_t* matches12, int* nmatches) {
  if (!h || !k1 || !k2 || !F12 || !scale_factors2 || !level_sigma2_2 || !matches12 || !nmatches) { set_error("null argument"); return B200ORB_EINVAL; }
  if (k1->n < 0 || k2->n < 0 || k1->n_nodes < 0 || k2->n_nodes < 0 || k2->n >= (1 << 22) || nlevels < 1 || nlevels > MAX_LEVELS) { set_error("bad counts"); return B200ORB_EINVAL; }
  *nmatches = 0;
  for (int i = 0; i < k1->n; ++i) matches12[i] = -1;
  if (k1->n == 0 || k2->n == 0 || k1->n_nodes == 0 || k2->n_nodes == 0) return B200ORB_OK;
  for (int i = 0; i < k2->n; ++i)
    if (k2->octave[i] < 0 || k2->octave[i] >= nlevels) { set_error("octave out of range"); return B200ORB_EINVAL; }
  // merge-join of the FeatureVectors (:861-983); per pKF1 keypoint without MapPoint (and stereo when bOnlyStereo) one query
  std::vector<int> q1, qb, qe;
  {
    int a = 0, b = 0;
    while (a < k1->n_nodes && b < k2->n_nodes) {
      const uint32_t ka = k1->node_ids[a], kb = k2->node_ids[b];
      if (ka == kb) {
        for (int i = k1->node_off[a]; i < k1->node_off[a + 1]; ++i) {
          const uint32_t r = k1->idx[i];
          if (r >= (uint32_t)k1->n) { set_error("KF1 index out of range"); return B200ORB_EINVAL; }
          if (k1->has_mp && k1->has_mp[r]) continue;
          if (only_stereo && !(k1->uright[r] >= 0)) continue;
          q1.push_back((int)r); qb.push_back(k2->node_off[b]); qe.push_back(k2->node_off[b + 1]);
        }
        ++a; ++b;
      } else if (ka < kb) {
        a = (int)(std::lower_bound(k1->node_ids, k1->node_ids + k1->n_nodes, kb) - k1->node_ids);
      } else {
        b = (int)(std::lower_bound(k2->node_ids, k2->node_ids + k2->n_nodes, ka) - k2->node_ids);
      }
    }
  }
  const size_t nq = q1.size(), nfi = (size_t)k2->node_off[k2->n_nodes];
  if (nq == 0) return B200ORB_OK;
  for (size_t i = 0; i < nfi; ++i)
    if (k2->idx[i] >= (uint32_t)k2->n) { set_error("KF2 index out of range"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  const size_t n1 = k1->n, n2 = k2->n;
  TriView t;
  memset(&t, 0, sizeof(t));
  int *d_out, *d_nm;
  B200_CHECK(h->arena.reserve(h->stream, [&](Carver& c) {
    t.q_idx1 = c.take<int>(nq); t.f_beg = c.take<int>(nq); t.f_end = c.take<int>(nq); t.f_idx = c.take<unsigned>(nfi);
    t.desc1 = c.take<uint8_t>(n1 * 32); t.desc2 = c.take<uint8_t>(n2 * 32);
    t.x1 = c.take<float>(n1); t.y1 = c.take<float>(n1); t.ang1 = c.take<float>(n1); t.ur1 = c.take<float>(n1);
    t.x2 = c.take<float>(n2); t.y2 = c.take<float>(n2); t.ang2 = c.take<float>(n2); t.ur2 = c.take<float>(n2);
    t.oct2 = c.take<int>(n2); t.blocked2 = c.take<uint8_t>(n2);
    d_out = c.take<int>(n1); d_nm = c.take<int>(1);
  }));
  std::vector<uint8_t> blocked(n2, 0);
  if (k2->has_mp) memcpy(blocked.data(), k2->has_mp, n2);
  UP(t.q_idx1, q1.data(), nq, int); UP(t.f_beg, qb.data(), nq, int); UP(t.f_end, qe.data(), nq, int);
  UP(t.f_idx, k2->idx, nfi, unsigned); UP(t.desc1, k1->desc, n1 * 32, uint8_t); UP(t.desc2, k2->desc, n2 * 32, uint8_t);
  UP(t.x1, k1->x, n1, float); UP(t.y1, k1->y, n1, float); UP(t.ang1, k1->angle, n1, float); UP(t.ur1, k1->uright, n1, float);
  UP(t.x2, k2->x, n2, float); UP(t.y2, k2->y, n2, float); UP(t.ang2, k2->angle, n2, float); UP(t.ur2, k2->uright, n2, float);
  UP(t.oct2, k2->octave, n2, int); UP(t.blocked2, blocked.data(), n2, uint8_t);
  B200_CUDA(cudaMemsetAsync(d_out, 0xff, sizeof(int) * n1, h->stream));
  for (int i = 0; i < 9; ++i) t.F12[i] = F12[i];
  t.ex = ex; t.ey = ey;
  for (int i = 0; i < nlevels; ++i) { t.sf2[i] = scale_factors2[i]; t.sigma2_2[i] = level_sigma2_2[i]; }
  t.only_stereo = only_stereo; t.nq = (int)nq; t.n1 = (int)n1;
  B200_CUDA(cudaStreamSynchronize(h->stream));   // `blocked` (host vector) has been read by the upload
  k_tri_best<<<((int)nq + CAND_WARPS - 1) / CAND_WARPS, CAND_WARPS * 32, 0, h->stream>>>(t, d_out);
  k_tri_prune<<<1, 32, 0, h->stream>>>(t, check_ori, d_out, d_nm);
  h->launches += 2;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(matches12, d_out, sizeof(int) * n1, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(nmatches, d_nm, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

// smallest-to-largest thresholds t_k on ratio with  ceil(logf(ratio) / L) <= k  <=>  ratio <= t_k : MapPoint::PredictScale
// (src/MapPoint.cc:463-478) evaluates ceil(log(ratio)/mfLogScaleFactor) with the HOST's libm; bisecting the float line with
// that very function gives the device an exact, transcendental-free form of it
static void predict_scale_thresholds(float log_scale_factor, int nlevels, float* thr) {
  auto level = [&](float r) { return (int)std::ceil(std::log(r) / log_scale_factor); };
  for (int k = 0; k < nlevels - 1; ++k) {
    uint32_t lo = 0x00000001u, hi = 0x7f7fffffu;   // positive finite floats, ordered like their bit patterns
    float flo, fhi;
    memcpy(&fhi, &hi, 4);
    if (level(fhi) <= k) { thr[k] = fhi; continue; }
    memcpy(&flo, &lo, 4);
    if (level(flo) > k) { thr[k] = 0.f; continue; }
    while (hi - lo > 1) {   // invariant: level(lo) <= k < level(hi)
      const uint32_t mid = lo + (hi - lo) / 2;
      float fm;
      memcpy(&fm, &mid, 4);
      if (level(fm) <= k) lo = mid; else hi = mid;
    }
    memcpy(&thr[k], &lo, 4);
  }
}

int orbm_is_in_frustum(orbm_t* h, const OrbmFrame* f, const OrbmFrustumPoints* p, float viewing_cos_limit,
                       float log_scale_factor, uint8_t* in_view, float* proj_x, float* proj_y, float* proj_xr,
                       int32_t* scale_level, float* view_cos) {
  if (!h || !f || !p || !in_view || !proj_x || !proj_y || !proj_xr || !scale_level || !view_cos) { set_error("null argument"); return B200ORB_EINVAL; }
  if (p->n < 0 || f->nlevels < 1 || f->nlevels > MAX_LEVELS || !(log_scale_factor > 0)) { set_error("bad argument"); return B200ORB_EINVAL; }
  if (p->n == 0) return B200ORB_OK;
  if (!p->xw || !p->normal || !p->min_dist || !p->max_dist) { set_error("null point array"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  const size_t n = p->n;
  float *d_xw, *d_nrm, *d_mn, *d_mx, *d_px, *d_py, *d_pxr, *d_vc;
  uint8_t* d_in;
  int* d_lvl;
  B200_CHECK(h->arena.reserve(h->stream, [&](Carver& c) {
    d_xw = c.take<float>(n * 3); d_nrm = c.take<float>(n * 3); d_mn = c.take<float>(n); d_mx = c.take<float>(n);
    d_in = c.take<uint8_t>(n); d_px = c.take<float>(n); d_py = c.take<float>(n); d_pxr = c.take<float>(n);
    d_lvl = c.take<int>(n); d_vc = c.take<float>(n);
  }));
  UP(d_xw, p->xw, n * 3, float); UP(d_nrm, p->normal, n * 3, float); UP(d_mn, p->min_dist, n, float); UP(d_mx, p->max_dist, n, float);
  B200_CUDA(cudaMemsetAsync(d_px, 0, 4 * n, h->stream)); B200_CUDA(cudaMemsetAsync(d_py, 0, 4 * n, h->stream));
  B200_CUDA(cudaMemsetAsync(d_pxr, 0, 4 * n, h->stream)); B200_CUDA(cudaMemsetAsync(d_lvl, 0, 4 * n, h->stream));
  B200_CUDA(cudaMemsetAsync(d_vc, 0, 4 * n, h->stream));
  FrustumView v;
  memset(&v, 0, sizeof(v));
  v.xw = d_xw; v.normal = d_nrm; v.min_dist = d_mn; v.max_dist = d_mx; v.n = (int)n;
  memcpy(v.Tcw, f->Tcw, 64);
  v.fx = f->fx; v.fy = f->fy; v.cx = f->cx; v.cy = f->cy; v.bf = f->bf;
  v.min_x = f->min_x; v.max_x = f->max_x; v.min_y = f->min_y; v.max_y = f->max_y;
  v.cos_limit = viewing_cos_limit; v.nlevels = f->nlevels;
  predict_scale_thresholds(log_scale_factor, f->nlevels, v.level_thr);
  k_is_in_frustum<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(v, d_in, d_px, d_py, d_pxr, d_lvl, d_vc);
  ++h->launches;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(in_view, d_in, n, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(proj_x, d_px, 4 * n, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(proj_y, d_py, 4 * n, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(proj_xr, d_pxr, 4 * n, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(scale_level, d_lvl, 4 * n, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(view_cos, d_vc, 4 * n, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int orbm_undistort_keypoints(orbm_t* h, const float* xy_in, int n, const float K[9], const float* dist, int ndist,
                             float* xy_out) {
  if (!h || !K || (n > 0 && (!xy_in || !xy_out)) || n < 0 || ndist < 0 || ndist > 5 || (ndist > 0 && !dist)) { set_error("bad argument"); return B200ORB_EINVAL; }
  if (n == 0) return B200ORB_OK;
  if (ndist == 0 || dist[0] == 0.0f) {   // src/Frame.cc:561-565: mvKeysUn = mvKeys
    memcpy(xy_out, xy_in, sizeof(float) * 2 * (size_t)n);
    return B200ORB_OK;
  }
  DeviceGuard g(h->device);
  float *d_in, *d_out;
  B200_CHECK(h->arena.reserve(h->stream, [&](Carver& c) {
    d_in = c.take<float>((size_t)n * 2); d_out = c.take<float>((size_t)n * 2);
  }));
  UP(d_in, xy_in, (size_t)n * 2, float);
  UndistortParams p;
  p.fx = K[0]; p.fy = K[4]; p.cx = K[2]; p.cy = K[5];
  for (int i = 0; i < 5; ++i) p.k[i] = i < ndist ? (double)dist[i] : 0.0;
  k_undistort_points<<<(n + 255) / 256, 256, 0, h->stream>>>(p, d_in, d_out, n);
  ++h->launches;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(xy_out, d_out, sizeof(float) * 2 * (size_t)n, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

static int bow_impl(orbm_t* h, const OrbmBow* kf, const OrbmBow* f, float nnratio, int check_ori, int kfkf, int32_t* f2kf,
                    int* nmatches) {
  if (!h || !kf || !f || !f2kf || !nmatches) { set_error("null argument"); return B200ORB_EINVAL; }
  if (kf->n < 0 || f->n < 0 || kf->n_nodes < 0 || f->n_nodes < 0 || f->n >= (1 << 20)) { set_error("bad counts"); return B200ORB_EINVAL; }
  *nmatches = 0;
  const int nout = kfkf ? kf->n : f->n;
  for (int j = 0; j < nout; ++j) f2kf[j] = -1;
  if (kf->n == 0 || f->n == 0 || kf->n_nodes == 0 || f->n_nodes == 0) return B200ORB_OK;
  // merge-join of the two FeatureVectors (:242-335): equal node ids pair up; queries in the reference's visiting order
  std::vector<int> q_kf, q_beg, q_end;
  {
    int a = 0, b = 0;
    while (a < kf->n_nodes && b < f->n_nodes) {
      const uint32_t ka = kf->node_ids[a], kb = f->node_ids[b];
      if (ka == kb) {
        for (int i = kf->node_off[a]; i < kf->node_off[a + 1]; ++i) {
          const uint32_t r = kf->idx[i];
          if (r >= (uint32_t)kf->n) { set_error("KF index out of range"); return B200ORB_EINVAL; }
          if (kf->valid && !kf->valid[r]) continue;
          q_kf.push_back((int)r); q_beg.push_back(f->node_off[b]); q_end.push_back(f->node_off[b + 1]);
        }
        ++a; ++b;
      } else if (ka < kb) {
        a = (int)(std::lower_bound(kf->node_ids, kf->node_ids + kf->n_nodes, kb) - kf->node_ids);
      } else {
        b = (int)(std::lower_bound(f->node_ids, f->node_ids + f->n_nodes, ka) - f->node_ids);
      }
    }
  }
  const size_t nq = q_kf.size(), nfi = (size_t)f->node_off[f->n_nodes];
  if (nq == 0) return B200ORB_OK;
  for (size_t i = 0; i < nfi; ++i)
    if (f->idx[i] >= (uint32_t)f->n) { set_error("F index out of range"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  int *d_qkf, *d_qb, *d_qe, *d_count, *d_acc, *d_out, *d_nm;
  unsigned *d_fidx, *d_list;
  uint8_t *d_kd, *d_fd, *d_fvalid;
  float *d_ka, *d_fa;
  B200_CHECK(h->arena.reserve(h->stream, [&](Carver& c) {
    d_qkf = c.take<int>(nq); d_qb = c.take<int>(nq); d_qe = c.take<int>(nq); d_fidx = c.take<unsigned>(nfi);
    d_kd = c.take<uint8_t>((size_t)kf->n * 32); d_fd = c.take<uint8_t>((size_t)f->n * 32);
    d_ka = c.take<float>(kf->n); d_fa = c.take<float>(f->n);
    d_list = c.take<unsigned>(nq * LCAP); d_count = c.take<int>(nq); d_acc = c.take<int>(nq);
    d_out = c.take<int>(nout); d_nm = c.take<int>(1);
    d_fvalid = (kfkf && f->valid) ? c.take<uint8_t>(f->n) : nullptr;
  }));
  if (d_fvalid) UP(d_fvalid, f->valid, f->n, uint8_t);
  UP(d_qkf, q_kf.data(), nq, int); UP(d_qb, q_beg.data(), nq, int); UP(d_qe, q_end.data(), nq, int);
  UP(d_fidx, f->idx, nfi, unsigned); UP(d_kd, kf->desc, (size_t)kf->n * 32, uint8_t); UP(d_fd, f->desc, (size_t)f->n * 32, uint8_t);
  UP(d_ka, kf->angle, kf->n, float); UP(d_fa, f->angle, f->n, float);
  BowQueries bq{d_qkf, d_qb, d_qe, d_fidx, d_kd, d_fd, d_ka, d_fa, d_fvalid, (int)nq, f->n, kf->n};
  ListView lsv{d_list, d_count};
  k_cand_bow<<<((int)nq + CAND_WARPS - 1) / CAND_WARPS, CAND_WARPS * 32, 0, h->stream>>>(bq, lsv);
  size_t smem;
  const int cmax = align_up(std::max(f->n, kf->n), 16);
  B200_CHECK(resolve_smem(cmax, &smem, (const void*)k_resolve_bow));
  k_resolve_bow<<<1, 32, smem, h->stream>>>(bq, nnratio, check_ori, kfkf, lsv, d_acc, d_out, d_nm, cmax);
  h->launches += 2;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(f2kf, d_out, sizeof(int) * (size_t)nout, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(nmatches, d_nm, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

int orbm_search_by_bow(orbm_t* h, const OrbmBow* kf, const OrbmBow* f, float nnratio, int check_ori, int32_t* f2kf,
                       int* nmatches) {
  return bow_impl(h, kf, f, nnratio, check_ori, 0, f2kf, nmatches);
}

int orbm_search_by_bow_kf(orbm_t* h, const OrbmBow* kf1, const OrbmBow* kf2, float nnratio, int check_ori,
                          int32_t* matches12, int* nmatches) {
  return bow_impl(h, kf1, kf2, nnratio, check_ori, 1, matches12, nmatches);
}

}  // extern "C"
