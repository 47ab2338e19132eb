// shim/KeyFrameDatabase.h -- drop-in for the reference's include/KeyFrameDatabase.h: same include guard, namespace, class
// name and public surface, on top of the key-frame database of libb200orb.so (orbv_db_*, include/b200orb.h).
// Put this directory BEFORE the reference's include/ on the include path (include/KeyFrame.h includes it too).
//
// The inverted-file walk, the common-word counts and the L1 scores of DetectRelocalizationCandidates /
// DetectLoopCandidates run on the GPU; the call returns the keyframes the walk met with their new mnLoop* / mnReloc*
// values, which are written back here, so that the objects hold exactly what the reference leaves on them.  The rest --
// the covisibility accumulation and the 0.75f * bestAccScore filter (src/KeyFrameDatabase.cc:141-196, :255-308) -- is
// the reference's own code below, on the real objects: it reads GetBestCovisibilityKeyFrames(10), and in relocalisation
// the mRelocScore a neighbour kept from an earlier query, as the reference does.
//
// include/KeyFrame.h includes this header before KeyFrame is complete, so every member that touches a KeyFrame or a Frame
// is a template on that type: its body is checked where it is instantiated, at the end of the including translation unit.
// The device scores with DBoW2's L1 score only (ORBvoc is L1_NORM); another scoring type throws, as does a missing GPU.
#ifndef KEYFRAMEDATABASE_H
#define KEYFRAMEDATABASE_H

#include <vector>
#include <list>
#include <set>
#include <map>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <utility>

#include "KeyFrame.h"
#include "Frame.h"
#include "ORBVocabulary.h"

#include <mutex>

#include "b200orb.h"

namespace ORB_SLAM2
{

class KeyFrame;
class Frame;

class KeyFrameDatabase
{
public:

    KeyFrameDatabase(const ORBVocabulary &voc) : mpVoc(&voc)
    {
        if (voc.getScoringType() != DBoW2::L1_NORM)
            throw std::runtime_error("KeyFrameDatabase(B200): the device scores with DBoW2's L1 score only");
        int dev = 0;
        if (const char* e = std::getenv("B200ORB_DEVICE")) dev = std::atoi(e);
        check(orbv_db_create(dev, (int)voc.size(), &h_));
    }
    ~KeyFrameDatabase() { orbv_db_destroy(h_); }
    KeyFrameDatabase(const KeyFrameDatabase&) = delete;
    KeyFrameDatabase& operator=(const KeyFrameDatabase&) = delete;

   void add(KeyFrame* pKF) { addT(pKF); }

   void erase(KeyFrame* pKF) { eraseT(pKF); }

   void clear()
   {
       std::unique_lock<std::mutex> lock(mMutex);
       check(orbv_db_clear(h_));
   }

   // Loop Detection
   std::vector<KeyFrame *> DetectLoopCandidates(KeyFrame* pKF, float minScore) { return loopT(pKF, minScore); }

   // Relocalization
   std::vector<KeyFrame*> DetectRelocalizationCandidates(Frame* F) { return relocT<KeyFrame>(F); }

protected:

  // Associated vocabulary
  const ORBVocabulary* mpVoc;

  // Mutex
  std::mutex mMutex;

private:
  orbv_db_t* h_ = nullptr;
  std::map<KeyFrame*, int> mSlot;      // keyframe -> device slot
  std::vector<KeyFrame*> mvpSlotKF;    // device slot -> keyframe

  static void check(int rc)
  {
      if (rc != B200ORB_OK) throw std::runtime_error(std::string("KeyFrameDatabase(B200): ") + b200orb_last_error());
  }

  template <class BowVector>
  static void flat(const BowVector& bow, std::vector<uint32_t>& w, std::vector<double>& v)
  {
      w.clear(); v.clear();
      for (typename BowVector::const_iterator it = bow.begin(); it != bow.end(); ++it) { w.push_back(it->first); v.push_back(it->second); }
  }

  template <class KF>
  void addT(KF* pKF)
  {
      std::unique_lock<std::mutex> lock(mMutex);
      typename std::map<KeyFrame*, int>::iterator it = mSlot.find(pKF);
      const int s = it != mSlot.end() ? it->second : (int)mvpSlotKF.size();
      std::vector<uint32_t> w;
      std::vector<double> v;
      flat(pKF->mBowVec, w, v);
      OrbvDbMembers m;
      m.loop_query = pKF->mnLoopQuery; m.loop_words = pKF->mnLoopWords; m.loop_score = pKF->mLoopScore;
      m.reloc_query = pKF->mnRelocQuery; m.reloc_words = pKF->mnRelocWords; m.reloc_score = pKF->mRelocScore;
      check(orbv_db_add(h_, s, w.data(), v.data(), (int)w.size(), &m));
      if (it == mSlot.end()) { mSlot[pKF] = s; mvpSlotKF.push_back(pKF); }
  }

  template <class KF>
  void eraseT(KF* pKF)
  {
      std::unique_lock<std::mutex> lock(mMutex);
      typename std::map<KeyFrame*, int>::iterator it = mSlot.find(pKF);
      if (it != mSlot.end()) check(orbv_db_erase(h_, it->second));
  }

  // The walk and the scores on the device; the met keyframes' members written back.  Returns lKFsSharingWords in order.
  template <class KF, class BowVector>
  std::list<KF*> walk(int kind, uint64_t id, const BowVector& bow, const std::vector<int32_t>& connected)
  {
      std::vector<uint32_t> w;
      std::vector<double> v;
      flat(bow, w, v);
      int nlive = 0, napp = 0, nmet = 0;
      check(orbv_db_state(h_, -1, NULL, NULL, &nlive));
      std::vector<OrbvDbHit> hits(nlive > 0 ? nlive : 1);
      check(orbv_db_query(h_, kind, id, w.data(), v.data(), (int)w.size(), connected.data(), (int)connected.size(),
                          hits.data(), nlive, &napp, &nmet));
      std::list<KF*> lKFsSharingWords;
      for (int i = 0; i < nmet; ++i) {
          KF* pKFi = static_cast<KF*>(mvpSlotKF[hits[i].slot]);
          if (kind == ORBV_DB_LOOP) {
              pKFi->mnLoopQuery = hits[i].query; pKFi->mnLoopWords = hits[i].words; pKFi->mLoopScore = hits[i].score;
          } else {
              pKFi->mnRelocQuery = hits[i].query; pKFi->mnRelocWords = hits[i].words; pKFi->mRelocScore = hits[i].score;
          }
          if (i < napp) lKFsSharingWords.push_back(pKFi);
      }
      return lKFsSharingWords;
  }

  // src/KeyFrameDatabase.cc:76-197
  template <class KF>
  std::vector<KF*> loopT(KF* pKF, float minScore)
  {
      std::set<KF*> spConnectedKeyFrames = pKF->GetConnectedKeyFrames();
      std::list<KF*> lKFsSharingWords;
      {
          std::unique_lock<std::mutex> lock(mMutex);
          std::vector<int32_t> connected;
          for (typename std::set<KF*>::iterator sit = spConnectedKeyFrames.begin(); sit != spConnectedKeyFrames.end(); sit++) {
              typename std::map<KeyFrame*, int>::iterator it = mSlot.find(*sit);
              if (it != mSlot.end()) connected.push_back(it->second);
          }
          lKFsSharingWords = walk<KF>(ORBV_DB_LOOP, pKF->mnId, pKF->mBowVec, connected);
      }

      if(lKFsSharingWords.empty())
          return std::vector<KF*>();

      std::list<std::pair<float,KF*> > lScoreAndMatch;

      int maxCommonWords=0;
      for(typename std::list<KF*>::iterator lit=lKFsSharingWords.begin(), lend= lKFsSharingWords.end(); lit!=lend; lit++)
      {
          if((*lit)->mnLoopWords>maxCommonWords)
              maxCommonWords=(*lit)->mnLoopWords;
      }

      int minCommonWords = maxCommonWords*0.8f;

      // the scores are the device's (mLoopScore of the keyframes above minCommonWords)
      for(typename std::list<KF*>::iterator lit=lKFsSharingWords.begin(), lend= lKFsSharingWords.end(); lit!=lend; lit++)
      {
          KF* pKFi = *lit;

          if(pKFi->mnLoopWords>minCommonWords)
          {
              float si = pKFi->mLoopScore;
              if(si>=minScore)
                  lScoreAndMatch.push_back(std::make_pair(si,pKFi));
          }
      }

      if(lScoreAndMatch.empty())
          return std::vector<KF*>();

      std::list<std::pair<float,KF*> > lAccScoreAndMatch;
      float bestAccScore = minScore;

      for(typename std::list<std::pair<float,KF*> >::iterator it=lScoreAndMatch.begin(), itend=lScoreAndMatch.end(); it!=itend; it++)
      {
          KF* pKFi = it->second;
          std::vector<KF*> vpNeighs = pKFi->GetBestCovisibilityKeyFrames(10);

          float bestScore = it->first;
          float accScore = it->first;
          KF* pBestKF = pKFi;
          for(typename std::vector<KF*>::iterator vit=vpNeighs.begin(), vend=vpNeighs.end(); vit!=vend; vit++)
          {
              KF* pKF2 = *vit;
              if(pKF2->mnLoopQuery==pKF->mnId && pKF2->mnLoopWords>minCommonWords)
              {
                  accScore+=pKF2->mLoopScore;
                  if(pKF2->mLoopScore>bestScore)
                  {
                      pBestKF=pKF2;
                      bestScore = pKF2->mLoopScore;
                  }
              }
          }

          lAccScoreAndMatch.push_back(std::make_pair(accScore,pBestKF));
          if(accScore>bestAccScore)
              bestAccScore=accScore;
      }

      float minScoreToRetain = 0.75f*bestAccScore;

      std::set<KF*> spAlreadyAddedKF;
      std::vector<KF*> vpLoopCandidates;
      vpLoopCandidates.reserve(lAccScoreAndMatch.size());

      for(typename std::list<std::pair<float,KF*> >::iterator it=lAccScoreAndMatch.begin(), itend=lAccScoreAndMatch.end(); it!=itend; it++)
      {
          if(it->first>minScoreToRetain)
          {
              KF* pKFi = it->second;
              if(!spAlreadyAddedKF.count(pKFi))
              {
                  vpLoopCandidates.push_back(pKFi);
                  spAlreadyAddedKF.insert(pKFi);
              }
          }
      }

      return vpLoopCandidates;
  }

  // src/KeyFrameDatabase.cc:199-309
  template <class KF, class FR>
  std::vector<KF*> relocT(FR* F)
  {
      std::list<KF*> lKFsSharingWords;
      {
          std::unique_lock<std::mutex> lock(mMutex);
          lKFsSharingWords = walk<KF>(ORBV_DB_RELOC, F->mnId, F->mBowVec, std::vector<int32_t>());
      }
      if(lKFsSharingWords.empty())
          return std::vector<KF*>();

      int maxCommonWords=0;
      for(typename std::list<KF*>::iterator lit=lKFsSharingWords.begin(), lend= lKFsSharingWords.end(); lit!=lend; lit++)
      {
          if((*lit)->mnRelocWords>maxCommonWords)
              maxCommonWords=(*lit)->mnRelocWords;
      }

      int minCommonWords = maxCommonWords*0.8f;

      std::list<std::pair<float,KF*> > lScoreAndMatch;

      // the scores are the device's (mRelocScore of the keyframes above minCommonWords)
      for(typename std::list<KF*>::iterator lit=lKFsSharingWords.begin(), lend= lKFsSharingWords.end(); lit!=lend; lit++)
      {
          KF* pKFi = *lit;

          if(pKFi->mnRelocWords>minCommonWords)
          {
              float si = pKFi->mRelocScore;
              lScoreAndMatch.push_back(std::make_pair(si,pKFi));
          }
      }

      if(lScoreAndMatch.empty())
          return std::vector<KF*>();

      std::list<std::pair<float,KF*> > lAccScoreAndMatch;
      float bestAccScore = 0;

      for(typename std::list<std::pair<float,KF*> >::iterator it=lScoreAndMatch.begin(), itend=lScoreAndMatch.end(); it!=itend; it++)
      {
          KF* pKFi = it->second;
          std::vector<KF*> vpNeighs = pKFi->GetBestCovisibilityKeyFrames(10);

          float bestScore = it->first;
          float accScore = bestScore;
          KF* pBestKF = pKFi;
          for(typename std::vector<KF*>::iterator vit=vpNeighs.begin(), vend=vpNeighs.end(); vit!=vend; vit++)
          {
              KF* pKF2 = *vit;
              if(pKF2->mnRelocQuery!=F->mnId)
                  continue;

              accScore+=pKF2->mRelocScore;
              if(pKF2->mRelocScore>bestScore)
              {
                  pBestKF=pKF2;
                  bestScore = pKF2->mRelocScore;
              }

          }
          lAccScoreAndMatch.push_back(std::make_pair(accScore,pBestKF));
          if(accScore>bestAccScore)
              bestAccScore=accScore;
      }

      float minScoreToRetain = 0.75f*bestAccScore;
      std::set<KF*> spAlreadyAddedKF;
      std::vector<KF*> vpRelocCandidates;
      vpRelocCandidates.reserve(lAccScoreAndMatch.size());
      for(typename std::list<std::pair<float,KF*> >::iterator it=lAccScoreAndMatch.begin(), itend=lAccScoreAndMatch.end(); it!=itend; it++)
      {
          const float &si = it->first;
          if(si>minScoreToRetain)
          {
              KF* pKFi = it->second;
              if(!spAlreadyAddedKF.count(pKFi))
              {
                  vpRelocCandidates.push_back(pKFi);
                  spAlreadyAddedKF.insert(pKFi);
              }
          }
      }

      return vpRelocCandidates;
  }
};

} //namespace ORB_SLAM

#endif
