// orbv_db.cu -- the key-frame database: KeyFrameDatabase (src/KeyFrameDatabase.cc) add / erase / clear and the walk,
// common-word counts and L1 scores of DetectLoopCandidates / DetectRelocalizationCandidates.
//
// Representation.  The reference keeps an inverted file: per word a std::list<KeyFrame*> in add order.  A keyframe's
// BowVector is computed once (KeyFrame::ComputeBoW guards it with empty()), so every add of one keyframe puts it into the
// same lists, and erase removes its first occurrence from each of them.  A forward index therefore reproduces the lists:
// per slot its sorted BowVector, how many times it is in the database (`mult`) and the add sequence number of its earliest
// live add (`seq`).  A slot added twice is counted twice and keeps its first position; erase drops the earliest add; erase
// then add moves the slot to the end of every list.  A slot's first encounter in the reference's walk (query words
// ascending, each list in add order) is in the list of its smallest common word, at its earliest live add: the walk order
// is the order of the key (smallest common word, seq).
//
// One query, all on the handle's stream, one host sync:
//   k_db_walk      one warp per slot: intersect the slot's words with the query's (staged in shared memory when they
//                  fit; binary search per lane), count (ballot + popc) times mult, first common word; apply the walk's
//                  member updates (:86-104, :207-222) to the slot's mirror; max of the appended words; the sort key
//   radix sort     (key, slot) pairs: appended slots in walk order, then the other met slots by slot, then the rest
//   k_db_score     one warp per appended slot above minCommonWords = (int)(max * 0.8f): TemplatedVocabulary::score's
//                  terms per lane, summed in ascending word order by a shuffle chain (the sum's order is the result)
//   k_db_finalize  the met slots' records, written straight into the pinned result block
#include <cub/device/device_radix_sort.cuh>

#include <deque>
#include <memory>
#include <new>
#include <vector>

#include "common.cuh"

namespace b200 {

struct DbSlot {
  unsigned off;    // first word in the pool
  int n;           // BowVector size
  int mult;        // live adds
  unsigned seq;    // add sequence number of the earliest live add
  OrbvDbMembers m;
};
static_assert(sizeof(DbSlot) == 48, "slot record layout");

constexpr int DB_MAX_SLOTS = 1 << 24;
constexpr int DB_QSMEM = 4096;   // query words staged in shared memory up to this many (16 KiB)
constexpr int DB_THREADS = 512;

struct DbQuery {
  const unsigned* qw;   // query words, ascending
  const double* qv;     // query weights
  int nq;
  const int* conn;      // connected slots, ascending (loop queries)
  int nconn;
  int kind;
  unsigned long long id;
  int seq_bits;         // key = word << seq_bits | seq (appended), n_words << seq_bits | slot (met), else `unmet`
  unsigned n_words;
  unsigned long long unmet;
};

__device__ __forceinline__ int db_lower_bound(const unsigned* a, int n, unsigned x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ const unsigned* db_stage_query(const DbQuery& q, unsigned* sq) {
  if (q.nq > DB_QSMEM) return q.qw;
  for (int i = threadIdx.x; i < q.nq; i += blockDim.x) sq[i] = q.qw[i];
  __syncthreads();
  return sq;
}

__global__ void __launch_bounds__(DB_THREADS) k_db_walk(DbQuery q, DbSlot* __restrict__ slots, int S,
                                                        const unsigned* __restrict__ pool_w,
                                                        unsigned long long* __restrict__ key, int* __restrict__ val,
                                                        int* __restrict__ cnt) {
  extern __shared__ unsigned sq[];
  const unsigned* qw = db_stage_query(q, sq);
  const int lane = threadIdx.x & 31;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  for (int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < S; s += nwarps) {
    const unsigned off = slots[s].off;
    const int n = slots[s].n, mult = slots[s].mult;
    int c = 0;
    unsigned fw = 0xffffffffu;
    if (mult > 0)
      for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        unsigned w = 0;
        bool hit = false;
        if (i < n) {
          w = pool_w[off + i];
          const int p = db_lower_bound(qw, q.nq, w);
          hit = p < q.nq && qw[p] == w;
        }
        const unsigned b = __ballot_sync(0xffffffffu, hit);
        if (b && c == 0) fw = __shfl_sync(0xffffffffu, w, __ffs(b) - 1);
        c += __popc(b);
      }
    if (lane != 0) continue;
    val[s] = s;
    if (c == 0) { key[s] = q.unmet; continue; }
    OrbvDbMembers& m = slots[s].m;
    uint64_t& query = q.kind == ORBV_DB_LOOP ? m.loop_query : m.reloc_query;
    int& words = q.kind == ORBV_DB_LOOP ? m.loop_words : m.reloc_words;
    const int times = c * mult;   // one increment per list occurrence
    bool appended = false;
    if (query != q.id) {
      // loop: a connected keyframe is reset at every meeting and never marked, so it ends at 1 (:93-102)
      const int p = q.kind == ORBV_DB_LOOP ? db_lower_bound((const unsigned*)q.conn, q.nconn, (unsigned)s) : q.nconn;
      if (p < q.nconn && q.conn[p] == s) {
        words = 1;
      } else {
        words = times;
        query = q.id;
        appended = true;
      }
    } else {
      words += times;
    }
    atomicAdd(&cnt[2], 1);
    if (appended) {
      atomicAdd(&cnt[1], 1);
      atomicMax(&cnt[0], words);
      key[s] = ((unsigned long long)fw << q.seq_bits) | slots[s].seq;
    } else {
      key[s] = ((unsigned long long)q.n_words << q.seq_bits) | (unsigned)s;
    }
  }
}

__device__ __forceinline__ bool db_appended(const DbQuery& q, unsigned long long k) {
  return (k >> q.seq_bits) < q.n_words;
}
__device__ __forceinline__ int db_min_common(const int* cnt) { return (int)(cnt[0] * 0.8f); }

__global__ void __launch_bounds__(DB_THREADS) k_db_score(DbQuery q, DbSlot* __restrict__ slots, int S,
                                                         const unsigned* __restrict__ pool_w,
                                                         const double* __restrict__ pool_v,
                                                         const unsigned long long* __restrict__ key,
                                                         const int* __restrict__ cnt) {
  extern __shared__ unsigned sq[];
  const unsigned* qw = db_stage_query(q, sq);
  const int lane = threadIdx.x & 31;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  const int min_common = db_min_common(cnt);
  for (int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < S; s += nwarps) {
    if (!db_appended(q, key[s])) continue;
    OrbvDbMembers& m = slots[s].m;
    if ((q.kind == ORBV_DB_LOOP ? m.loop_words : m.reloc_words) <= min_common) continue;
    const unsigned off = slots[s].off;
    const int n = slots[s].n;
    double score = 0;   // TemplatedVocabulary::score, L1: v1 = the query, v2 = the keyframe
    for (int i0 = 0; i0 < n; i0 += 32) {
      const int i = i0 + lane;
      double term = 0;
      bool hit = false;
      if (i < n) {
        const unsigned w = pool_w[off + i];
        const int p = db_lower_bound(qw, q.nq, w);
        if (p < q.nq && qw[p] == w) {
          const double a = q.qv[p], b = pool_v[off + i];
          term = fabs(a - b) - fabs(a) - fabs(b);
          hit = true;
        }
      }
      for (unsigned b = __ballot_sync(0xffffffffu, hit); b; b &= b - 1)
        score += __shfl_sync(0xffffffffu, term, __ffs(b) - 1);
    }
    if (lane == 0) {
      const float si = (float)(-score / 2.0);
      if (q.kind == ORBV_DB_LOOP) m.loop_score = si;
      else m.reloc_score = si;
    }
  }
}

__global__ void __launch_bounds__(256) k_db_finalize(DbQuery q, const DbSlot* __restrict__ slots,
                                                     const unsigned long long* __restrict__ key,
                                                     const int* __restrict__ order, const int* __restrict__ cnt,
                                                     OrbvDbHit* __restrict__ out, int* __restrict__ hdr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n_app = cnt[1], n_met = cnt[2];
  if (i == 0) { hdr[0] = n_app; hdr[1] = n_met; }
  if (i >= n_met) return;
  const int s = order[i];
  const OrbvDbMembers& m = slots[s].m;
  const bool loop = q.kind == ORBV_DB_LOOP;
  OrbvDbHit r;
  r.slot = s;
  r.words = loop ? m.loop_words : m.reloc_words;
  r.query = loop ? m.loop_query : m.reloc_query;
  r.score = loop ? m.loop_score : m.reloc_score;
  r.flags = i < n_app ? ORBV_DB_APPENDED | (r.words > db_min_common(cnt) ? ORBV_DB_SCORED : 0) : 0;
  out[i] = r;
}

static int db_bits(unsigned long long x) {   // bits to hold every value < x
  int b = 0;
  while (b < 64 && (1ull << b) < x) ++b;
  return b;
}

// Grows `b` to at least `need` bytes (1.5x, rounded up to 1 MiB), keeping its first `keep` bytes and zeroing the rest.
static int db_grow(DeviceBlock& b, cudaStream_t s, size_t keep, size_t need) {
  if (need <= b.bytes) return B200ORB_OK;
  DeviceBlock nb;
  const size_t n = align_up_sz(need + need / 2, 1 << 20);
  B200_CHECK(nb.carve(s, [&](Carver& t) { t.take<char>(n); }));
  if (keep) B200_CUDA(cudaMemcpyAsync(nb.p, b.p, keep, cudaMemcpyDeviceToDevice, s));
  B200_CUDA(cudaMemsetAsync((char*)nb.p + keep, 0, nb.bytes - keep, s));
  B200_CUDA(cudaStreamSynchronize(s));
  b = std::move(nb);   // nb now holds the old block and frees it
  return B200ORB_OK;
}

static int db_check_words(const uint32_t* words, const double* weights, int n, int n_words) {
  if (n < 0 || (n > 0 && (!words || !weights))) { set_error("bad argument"); return B200ORB_EINVAL; }
  for (int i = 0; i < n; ++i) {
    if (words[i] >= (uint32_t)n_words) { set_error("word id %u >= n_words %d", words[i], n_words); return B200ORB_EINVAL; }
    if (i > 0 && words[i] <= words[i - 1]) { set_error("word ids not strictly ascending at %d", i); return B200ORB_EINVAL; }
  }
  return B200ORB_OK;
}

}  // namespace b200

using namespace b200;

struct orbv_db {
  struct HostSlot {
    bool known = false;
    unsigned off = 0;
    int n = 0;
    std::deque<unsigned> seqs;   // sequence numbers of the live adds, oldest first
  };
  int device = 0;
  int n_words = 0;
  Stream stream;
  long long launches = 0;
  std::vector<HostSlot> hs;
  int n_live = 0;             // slots with mult > 0
  size_t pool_used = 0;       // words in the pool
  unsigned seq_next = 0;
  DeviceBlock pool_w, pool_v, slots;
  DeviceBlock work;
  HostBlock io;               // query staging (copied to the front of `work` in one go) and the result records

  DbSlot* d_slots() { return (DbSlot*)slots.p; }
  int upload(int s, const OrbvDbMembers* m) {
    const HostSlot& h = hs[s];
    DbSlot r;
    r.off = h.off; r.n = h.n; r.mult = (int)h.seqs.size(); r.seq = h.seqs.empty() ? 0u : h.seqs.front();
    if (m) r.m = *m;
    B200_CUDA(cudaMemcpyAsync(d_slots() + s, &r, m ? sizeof(DbSlot) : offsetof(DbSlot, m), cudaMemcpyHostToDevice, stream));
    return B200ORB_OK;
  }
};

extern "C" {

int orbv_db_create(int device, int n_words, orbv_db_t** out) {
  if (!out || n_words < 1) { set_error("bad argument"); return B200ORB_EINVAL; }
  *out = nullptr;
  B200_CHECK(check_device(device));
  DeviceGuard g(device);
  std::unique_ptr<orbv_db> h(new (std::nothrow) orbv_db());
  if (!h) { set_error("out of host memory"); return B200ORB_EINVAL; }
  h->device = device;
  h->n_words = n_words;
  B200_CHECK(h->stream.create());
  *out = h.release();
  return B200ORB_OK;
}
void orbv_db_destroy(orbv_db_t* h) { destroy_handle(h); }
long long orbv_db_launch_count(const orbv_db_t* h) { return h ? h->launches : 0; }

int orbv_db_add(orbv_db_t* h, int slot, const uint32_t* words, const double* weights, int n, const OrbvDbMembers* members) {
  if (!h || slot < 0 || slot >= DB_MAX_SLOTS) { set_error("bad argument (slot %d)", slot); return B200ORB_EINVAL; }
  B200_CHECK(db_check_words(words, weights, n, h->n_words));
  if (h->seq_next == 0xffffffffu) { set_error("add sequence exhausted: clear the database"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  if (slot >= (int)h->hs.size()) {
    B200_CHECK(db_grow(h->slots, h->stream, h->hs.size() * sizeof(DbSlot), (size_t)(slot + 1) * sizeof(DbSlot)));
    h->hs.resize(slot + 1);
  }
  orbv_db::HostSlot& s = h->hs[slot];
  if (s.seqs.empty()) {   // not in the database: its BowVector goes to the end of the pool
    const size_t need = h->pool_used + (size_t)n;
    if (need > 0xffffffffull) { set_error("word pool full: clear the database"); return B200ORB_EINVAL; }
    B200_CHECK(db_grow(h->pool_w, h->stream, h->pool_used * 4, need * 4));
    B200_CHECK(db_grow(h->pool_v, h->stream, h->pool_used * 8, need * 8));
    if (n) {
      B200_CUDA(cudaMemcpyAsync((unsigned*)h->pool_w.p + h->pool_used, words, (size_t)n * 4, cudaMemcpyHostToDevice, h->stream));
      B200_CUDA(cudaMemcpyAsync((double*)h->pool_v.p + h->pool_used, weights, (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
    }
    s.off = (unsigned)h->pool_used;
    s.n = n;
    h->pool_used = need;
    ++h->n_live;
  }
  s.seqs.push_back(h->seq_next++);
  OrbvDbMembers zero{};
  const OrbvDbMembers* m = members ? members : (s.known ? nullptr : &zero);
  s.known = true;
  return h->upload(slot, m);
}

int orbv_db_erase(orbv_db_t* h, int slot) {
  if (!h || slot < 0 || slot >= (int)h->hs.size() || !h->hs[slot].known) {
    set_error("unknown slot %d", slot);
    return B200ORB_EINVAL;
  }
  orbv_db::HostSlot& s = h->hs[slot];
  if (s.seqs.empty()) return B200ORB_OK;
  DeviceGuard g(h->device);
  s.seqs.pop_front();
  if (s.seqs.empty()) --h->n_live;
  return h->upload(slot, nullptr);
}

int orbv_db_clear(orbv_db_t* h) {
  if (!h) { set_error("bad argument"); return B200ORB_EINVAL; }
  DeviceGuard g(h->device);
  for (size_t i = 0; i < h->hs.size(); ++i)
    if (!h->hs[i].seqs.empty()) {
      h->hs[i].seqs.clear();
      B200_CHECK(h->upload((int)i, nullptr));
    }
  h->n_live = 0;
  h->pool_used = 0;
  h->seq_next = 0;
  return B200ORB_OK;
}

int orbv_db_state(orbv_db_t* h, int slot, OrbvDbMembers* members, int* count, int* n_live) {
  if (!h || slot < -1) { set_error("bad argument"); return B200ORB_EINVAL; }
  if (n_live) *n_live = h->n_live;
  if (slot == -1) return B200ORB_OK;
  if (slot >= (int)h->hs.size() || !h->hs[slot].known) { set_error("unknown slot %d", slot); return B200ORB_EINVAL; }
  if (count) *count = (int)h->hs[slot].seqs.size();
  if (members) {
    DeviceGuard g(h->device);
    B200_CUDA(cudaMemcpyAsync(members, &h->d_slots()[slot].m, sizeof(OrbvDbMembers), cudaMemcpyDeviceToHost, h->stream));
    B200_CUDA(cudaStreamSynchronize(h->stream));
  }
  return B200ORB_OK;
}

int orbv_db_query(orbv_db_t* h, int kind, uint64_t query_id, const uint32_t* words, const double* weights, int n,
                  const int32_t* connected, int n_connected, OrbvDbHit* out, int cap, int* n_appended, int* n_met) {
  if (!h || (kind != ORBV_DB_RELOC && kind != ORBV_DB_LOOP) || !n_appended || !n_met || n_connected < 0 ||
      (n_connected > 0 && !connected) || cap < 0 || (cap > 0 && !out)) {
    set_error("bad argument");
    return B200ORB_EINVAL;
  }
  B200_CHECK(db_check_words(words, weights, n, h->n_words));
  std::vector<int> conn;
  if (kind == ORBV_DB_LOOP) {
    conn.assign(connected, connected + n_connected);
    for (int c : conn)
      if (c < 0 || c >= DB_MAX_SLOTS) { set_error("connected slot %d out of range", c); return B200ORB_EINVAL; }
    std::sort(conn.begin(), conn.end());
    conn.erase(std::unique(conn.begin(), conn.end()), conn.end());
  }
  if (cap < h->n_live) { set_error("cap %d < %d slots in the database", cap, h->n_live); return B200ORB_ECAP; }
  *n_appended = *n_met = 0;
  if (n == 0 || h->n_live == 0) return B200ORB_OK;   // the walk meets nobody
  DeviceGuard g(h->device);
  const int S = (int)h->hs.size(), nc = (int)conn.size();
  DbQuery q;
  q.nq = n; q.nconn = nc; q.kind = kind; q.id = query_id; q.n_words = (unsigned)h->n_words;
  q.seq_bits = db_bits(std::max<unsigned long long>(h->seq_next, (unsigned long long)S));
  const int end_bit = q.seq_bits + db_bits((unsigned long long)h->n_words + 2);
  q.unmet = (unsigned long long)(h->n_words + 1ull) << q.seq_bits;
  size_t sort_bytes = 0;
  B200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const unsigned long long*)nullptr,
                                            (unsigned long long*)nullptr, (const int*)nullptr, (int*)nullptr, S, 0,
                                            end_bit, (cudaStream_t)h->stream));
  // the inputs lead both blocks in the same carving, so that one copy moves them
  double *hv, *dv;
  unsigned *hw, *dw;
  int *hc, *dc, *hdr, *cnt, *val, *order;
  OrbvDbHit* hits;
  unsigned long long *key, *key_sorted;
  char* tmp;
  size_t in_bytes = 0;
  B200_CHECK(h->io.reserve(h->stream, [&](Carver& t) {
    hv = t.take<double>(n); hw = t.take<unsigned>(n); hc = t.take<int>(nc);
    in_bytes = t.off;
    hits = t.take<OrbvDbHit>(S); hdr = t.take<int>(2);
  }));
  B200_CHECK(h->work.reserve(h->stream, [&](Carver& t) {
    dv = t.take<double>(n); dw = t.take<unsigned>(n); dc = t.take<int>(nc);
    key = t.take<unsigned long long>(S); key_sorted = t.take<unsigned long long>(S);
    val = t.take<int>(S); order = t.take<int>(S); cnt = t.take<int>(4); tmp = t.take<char>(sort_bytes);
  }));
  memcpy(hv, weights, (size_t)n * 8);
  memcpy(hw, words, (size_t)n * 4);
  if (nc) memcpy(hc, conn.data(), (size_t)nc * 4);
  B200_CUDA(cudaMemcpyAsync(h->work.p, h->io.p, in_bytes, cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaMemsetAsync(cnt, 0, 4 * sizeof(int), h->stream));
  q.qw = dw; q.qv = dv; q.conn = dc;
  const int blocks = std::min((S + DB_THREADS / 32 - 1) / (DB_THREADS / 32), 4 * sm_count(h->device));
  const size_t smem = n <= DB_QSMEM ? (size_t)n * 4 : 0;
  k_db_walk<<<blocks, DB_THREADS, smem, h->stream>>>(q, h->d_slots(), S, (const unsigned*)h->pool_w.p, key, val, cnt);
  B200_CUDA(cub::DeviceRadixSort::SortPairs(tmp, sort_bytes, (const unsigned long long*)key, key_sorted, (const int*)val,
                                            order, S, 0, end_bit, (cudaStream_t)h->stream));
  k_db_score<<<blocks, DB_THREADS, smem, h->stream>>>(q, h->d_slots(), S, (const unsigned*)h->pool_w.p,
                                                      (const double*)h->pool_v.p, key, cnt);
  k_db_finalize<<<(S + 255) / 256, 256, 0, h->stream>>>(q, h->d_slots(), key, order, cnt, hits, hdr);
  h->launches += 3;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaStreamSynchronize(h->stream));
  *n_appended = hdr[0];
  *n_met = hdr[1];
  if (hdr[1]) memcpy(out, hits, (size_t)hdr[1] * sizeof(OrbvDbHit));
  return B200ORB_OK;
}

}  // extern "C"
