// shim/ORBVocabulary.h -- drop-in for the reference's include/ORBVocabulary.h (same guard, same name): ORBVocabulary stays
// a DBoW2 TemplatedVocabulary (loading, scoring, everything else is DBoW2's), but the transform Frame::ComputeBoW and
// KeyFrame::ComputeBoW call (src/Frame.cc:546-555, src/KeyFrame.cc:75-84) descends the tree on the GPU (orbv_transform);
// the BowVector / FeatureVector maps are then assembled in feature order exactly as TemplatedVocabulary::transform does.
// The tree is uploaded on first use from DBoW2's own node array (a vocabulary loaded afterwards: call InvalidateDevice()).
#ifndef ORBVOCABULARY_H
#define ORBVOCABULARY_H

#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "Thirdparty/DBoW2/DBoW2/FORB.h"
#include "Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h"

#include "b200orb.h"

namespace ORB_SLAM2 {

class ORBVocabulary : public DBoW2::TemplatedVocabulary<DBoW2::FORB::TDescriptor, DBoW2::FORB> {
  typedef DBoW2::TemplatedVocabulary<DBoW2::FORB::TDescriptor, DBoW2::FORB> Base;

 public:
  ORBVocabulary(int k = 10, int L = 5, DBoW2::WeightingType weighting = DBoW2::TF_IDF, DBoW2::ScoringType scoring = DBoW2::L1_NORM)
      : Base(k, L, weighting, scoring) {}
  ~ORBVocabulary() { orbv_destroy(h_); }
  void InvalidateDevice() { orbv_destroy(h_); h_ = nullptr; }
  DBoW2::ScoringType getScoringType() const { return m_scoring; }   // DBoW2's accessor (shim/KeyFrameDatabase.h reads it)

  using Base::transform;   // the single-feature overloads stay DBoW2's
  void transform(const std::vector<DBoW2::FORB::TDescriptor>& features, DBoW2::BowVector& v, DBoW2::FeatureVector& fv,
                 int levelsup) const {
    v.clear();
    fv.clear();
    if (this->empty()) return;
    upload();
    const int n = (int)features.size();
    std::vector<uint8_t> desc((size_t)(n > 0 ? n : 1) * 32);
    for (int i = 0; i < n; ++i) std::memcpy(&desc[(size_t)i * 32], features[i].ptr(0), 32);
    std::vector<uint32_t> word(n > 0 ? n : 1), node(n > 0 ? n : 1);
    std::vector<double> w(n > 0 ? n : 1);
    if (orbv_transform(h_, desc.data(), n, levelsup, word.data(), w.data(), node.data()) != B200ORB_OK)
      throw std::runtime_error(std::string("ORBVocabulary(B200): ") + b200orb_last_error());
    const bool tf = (m_weighting == DBoW2::TF_IDF || m_weighting == DBoW2::TF);
    const bool must = (m_scoring == DBoW2::L1_NORM || m_scoring == DBoW2::L2_NORM);
    for (int i = 0; i < n; ++i) {
      if (!(w[i] > 0)) continue;   // stopped word
      if (tf) v.addWeight(word[i], w[i]);
      else v.addIfNotExist(word[i], w[i]);
      fv.addFeature(node[i], (unsigned int)i);
    }
    if (tf && !v.empty() && !must) {
      const double nd = (double)v.size();
      for (DBoW2::BowVector::iterator vit = v.begin(); vit != v.end(); ++vit) vit->second /= nd;
    }
    if (must) v.normalize(m_scoring == DBoW2::L2_NORM ? DBoW2::L2 : DBoW2::L1);
  }

 protected:
  void upload() const {
    if (h_) return;
    const int nn = (int)m_nodes.size();
    std::vector<int32_t> parent(nn, 0), wid(nn, 0);
    std::vector<uint8_t> desc((size_t)nn * 32, 0);
    std::vector<double> weight(nn, 0.0);
    for (int i = 0; i < nn; ++i) {
      parent[i] = (int32_t)m_nodes[i].parent;
      weight[i] = m_nodes[i].weight;
      wid[i] = (int32_t)m_nodes[i].word_id;
      if (i > 0 && !m_nodes[i].descriptor.empty()) std::memcpy(&desc[(size_t)i * 32], m_nodes[i].descriptor.ptr(0), 32);
    }
    int dev = 0;
    if (const char* e = std::getenv("B200ORB_DEVICE")) dev = std::atoi(e);
    if (orbv_create(dev, m_k, m_L, nn, parent.data(), desc.data(), weight.data(), wid.data(), &h_) != B200ORB_OK)
      throw std::runtime_error(std::string("ORBVocabulary(B200): ") + b200orb_last_error());
  }
  mutable orbv_t* h_ = nullptr;
};

}  // namespace ORB_SLAM2
#endif  // ORBVOCABULARY_H
