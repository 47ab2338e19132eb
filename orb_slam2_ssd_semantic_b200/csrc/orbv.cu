// orbv.cu -- the BoW transform: Frame::ComputeBoW / KeyFrame::ComputeBoW -> DBoW2 TemplatedVocabulary::transform
// (src/Frame.cc:546-555, src/KeyFrame.cc:75-84; vocabulary tree of Thirdparty/DBoW2, k = 10, L = 6 for ORBvoc).
// The vocabulary lives in HBM as a breadth-first re-numbered k-ary tree (children of a node contiguous, in their DBoW2
// order); every descriptor descends it level by level, at each level picking the FIRST child at minimal Hamming distance
// (strict <, like DBoW2's loop).  One warp per descriptor: lane c scores child c (two 16-byte loads + 8 popc), a warp
// min over (distance << 8 | child) picks the branch; ORBvoc's 35 MB of node descriptors fit in the H100's 50 MB L2 after
// the first frames.  Outputs per descriptor: word id, word weight, id of the ancestor `levelsup` levels above the leaves --
// the BowVector / FeatureVector maps are assembled from them in feature order by the caller (their double accumulation
// order is part of the result).
#include <memory>
#include <new>
#include <vector>

#include "common.cuh"

namespace b200 {

struct VocView {
  const uint4* desc;        // 2 x uint4 per node (new numbering)
  const int* first_child;   // new index of the first child, -1 for a leaf
  const int* n_children;
  const int* orig_id;       // DBoW2 node id
  const int* word_id;       // leaves: word id
  const double* weight;
  int L;
};

__global__ void __launch_bounds__(256) k_bow_transform(VocView v, const uint8_t* __restrict__ desc, int n, int levelsup,
                                                       unsigned* __restrict__ word, double* __restrict__ weight,
                                                       unsigned* __restrict__ node) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(desc + (size_t)i * 32));
  const uint4 d1 = __ldg(reinterpret_cast<const uint4*>(desc + (size_t)i * 32) + 1);
  const int nid_level = v.L - levelsup;
  int cur = 0, level = 0, nid = 0;   // nid_level <= 0: the root (DBoW2: *nid = 0)
  while (v.first_child[cur] >= 0) {
    ++level;
    const int fc = v.first_child[cur], nc = v.n_children[cur];
    unsigned best = 0xffffffffu;
    for (int c0 = 0; c0 < nc; c0 += 32) {   // k <= 32 in practice (ORBvoc: 10): one round
      const int c = c0 + lane;
      unsigned key = 0xffffffffu;
      if (c < nc) {
        const uint4 a = __ldg(v.desc + 2 * (size_t)(fc + c)), b = __ldg(v.desc + 2 * (size_t)(fc + c) + 1);
        const int dist = __popc(a.x ^ d0.x) + __popc(a.y ^ d0.y) + __popc(a.z ^ d0.z) + __popc(a.w ^ d0.w) +
                         __popc(b.x ^ d1.x) + __popc(b.y ^ d1.y) + __popc(b.z ^ d1.z) + __popc(b.w ^ d1.w);
        key = ((unsigned)dist << 16) | (unsigned)c;
      }
      best = min(best, __reduce_min_sync(0xffffffffu, key));
    }
    cur = fc + (int)(best & 0xffffu);
    if (level == nid_level) nid = v.orig_id[cur];
  }
  if (lane == 0) { word[i] = (unsigned)v.word_id[cur]; weight[i] = v.weight[cur]; node[i] = (unsigned)nid; }
}

}  // namespace b200

using namespace b200;

struct orbv {
  int device = 0;
  Stream stream;
  long long launches = 0;
  int k = 0, L = 0, n_nodes = 0, n_words = 0;
  DeviceBlock tree;   // the renumbered vocabulary tree, uploaded once by orbv_create
  VocView v{};
  DeviceBlock io;     // orbv_transform's inputs and outputs
};

// The tree's arrays in the layout of the device block; orbv_create fills a host copy of the same layout.
struct TreeArrays {
  uint8_t* desc;
  int *first, *nch, *orig, *word;
  double* weight;
  void take(Carver& t, int n) {
    desc = t.take<uint8_t>((size_t)n * 32); first = t.take<int>(n); nch = t.take<int>(n); orig = t.take<int>(n);
    word = t.take<int>(n); weight = t.take<double>(n);
  }
};

extern "C" {

int orbv_create(int device, int k, int L, int n_nodes, const int32_t* parent, const uint8_t* desc, const double* weight,
                const int32_t* word_id, orbv_t** out) {
  if (!out || !parent || !desc || !weight || n_nodes < 2 || k < 2 || L < 1) { set_error("bad argument"); return B200ORB_EINVAL; }
  *out = nullptr;
  for (int i = 1; i < n_nodes; ++i)
    if (parent[i] < 0 || parent[i] >= i) { set_error("parent[i] must be < i (node 0 = root)"); return B200ORB_EINVAL; }
  B200_CHECK(check_device(device));
  DeviceGuard g(device);
  // children in ascending DBoW2 id, breadth-first renumbering so that siblings are contiguous
  std::vector<std::vector<int>> ch(n_nodes);
  for (int i = 1; i < n_nodes; ++i) ch[parent[i]].push_back(i);
  std::vector<int> order;   // new index -> DBoW2 id
  order.reserve(n_nodes);
  order.push_back(0);
  TreeArrays ht, dt;
  Carver probe;
  ht.take(probe, n_nodes);
  std::vector<char> staging(probe.off);
  Carver hc(staging.data(), staging.size());
  ht.take(hc, n_nodes);
  for (size_t q = 0; q < order.size(); ++q) {
    const int id = order[q];
    ht.first[q] = ch[id].empty() ? -1 : (int)order.size();
    ht.nch[q] = (int)ch[id].size();
    for (int c : ch[id]) order.push_back(c);
  }
  if ((int)order.size() != n_nodes) { set_error("the parent array is not a tree rooted at node 0"); return B200ORB_EINVAL; }
  // word ids: as given (a vocabulary file states them per leaf), else leaves in ascending node id (createWords)
  std::vector<int> word_of(n_nodes, -1);
  int nw = 0;
  for (int id = 1; id < n_nodes; ++id)
    if (ch[id].empty()) { word_of[id] = word_id ? word_id[id] : nw; ++nw; }
  for (int q = 0; q < n_nodes; ++q) {
    const int id = order[q];
    memcpy(ht.desc + (size_t)q * 32, desc + (size_t)id * 32, 32);
    ht.orig[q] = id; ht.word[q] = word_of[id] < 0 ? 0 : word_of[id]; ht.weight[q] = weight[id];
  }
  std::unique_ptr<orbv> h(new (std::nothrow) orbv());
  if (!h) { set_error("out of host memory"); return B200ORB_EINVAL; }
  h->device = device; h->k = k; h->L = L; h->n_nodes = n_nodes; h->n_words = nw;
  B200_CHECK(h->stream.create());
  B200_CHECK(h->tree.carve(h->stream, [&](Carver& t) { dt.take(t, n_nodes); }));
  B200_CUDA(cudaMemcpyAsync(h->tree.p, staging.data(), staging.size(), cudaMemcpyHostToDevice, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  h->v = VocView{(const uint4*)dt.desc, dt.first, dt.nch, dt.orig, dt.word, dt.weight, L};
  *out = h.release();
  return B200ORB_OK;
}
void orbv_destroy(orbv_t* h) { destroy_handle(h); }
int orbv_num_words(const orbv_t* h) { return h ? h->n_words : 0; }
long long orbv_launch_count(const orbv_t* h) { return h ? h->launches : 0; }

int orbv_transform(orbv_t* h, const uint8_t* desc, int n, int levelsup, uint32_t* word_id, double* word_weight,
                   uint32_t* node_id) {
  if (!h || n < 0 || (n > 0 && (!desc || !word_id || !word_weight || !node_id))) { set_error("bad argument"); return B200ORB_EINVAL; }
  if (n == 0) return B200ORB_OK;
  DeviceGuard g(h->device);
  double* d_w;
  uint8_t* d_d;
  unsigned *d_word, *d_node;
  B200_CHECK(h->io.reserve(h->stream, [&](Carver& t) {
    d_w = t.take<double>(n); d_d = t.take<uint8_t>((size_t)n * 32); d_word = t.take<unsigned>(n); d_node = t.take<unsigned>(n);
  }));
  B200_CUDA(cudaMemcpyAsync(d_d, desc, (size_t)n * 32, cudaMemcpyHostToDevice, h->stream));
  k_bow_transform<<<(n + 7) / 8, 256, 0, h->stream>>>(h->v, d_d, n, levelsup, d_word, d_w, d_node);
  ++h->launches;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(word_id, d_word, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(word_weight, d_w, (size_t)n * 8, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaMemcpyAsync(node_id, d_node, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
  B200_CUDA(cudaStreamSynchronize(h->stream));
  return B200ORB_OK;
}

}  // extern "C"
