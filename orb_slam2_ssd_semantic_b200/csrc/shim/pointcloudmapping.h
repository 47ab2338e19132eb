// shim/pointcloudmapping.h -- PointCloudMapping with the reference's public surface (include/pointcloudmapping.h:50-56,
// perfect/include/pointcloudmapping.h:23-28) in its occupancy mode: insertKeyFrame() forwards the keyframe's pose,
// intrinsics, depth and colour image to ocm_insert_keyframe (MapDrawer::GeneratePointCloud + InsertScan semantics,
// perfect/src/MapDrawer.cc:641-675,946-1025).  The reference's insertKeyFrame only clones + notifies and a worker
// thread does the work (src/pointcloudmapping.cc:116-128,362-525); here the GPU stream plays the worker: the call
// enqueues and returns, shutdown() drains it.
#ifndef POINTCLOUDMAPPING_H
#define POINTCLOUDMAPPING_H

#include <stdexcept>
#include <string>
#include <vector>

#include <cstdlib>
#include <Eigen/Core>
#include <opencv2/opencv.hpp>

#include "b200orb.h"

class PointCloudMapping {
 public:
  explicit PointCloudMapping(double resolution_) : resolution(resolution_) {
    OcmParams p;
    ocm_default_params(&p);
    p.resolution = resolution_;
    int dev = 0;
    if (const char* e = std::getenv("B200ORB_DEVICE")) dev = std::atoi(e);
    if (ocm_create(&p, dev, &h_) != B200ORB_OK)
      throw std::runtime_error(std::string("PointCloudMapping(B200): ") + b200orb_last_error());
  }
  ~PointCloudMapping() { ocm_destroy(h_); }
  PointCloudMapping(const PointCloudMapping&) = delete;
  PointCloudMapping& operator=(const PointCloudMapping&) = delete;

  // Reference: insertKeyFrame(KeyFrame* kf, cv::Mat& color, cv::Mat& depth, cv::Mat& imgRGB) -- the KeyFrame supplies
  // GetPose() (Tcw, CV_32F 4x4) and fx/fy/cx/cy.  Template keeps this header free of KeyFrame.h.
  template <class KeyFrameT>
  void insertKeyFrame(KeyFrameT* kf, cv::Mat& color, cv::Mat& depth, cv::Mat& imgRGB) {
    cv::Mat T = kf->GetPose();
    float Tcw[16];
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) Tcw[r * 4 + c] = T.template at<float>(r, c);
    insertKeyFrame(Tcw, kf->fx, kf->fy, kf->cx, kf->cy, color, depth, imgRGB);
  }
  void insertKeyFrame(const float Tcw[16], float fx, float fy, float cx, float cy, cv::Mat& /*gray*/, cv::Mat& depth,
                      cv::Mat& imgRGB) {
    if (ocm_insert_keyframe(h_, reinterpret_cast<const float*>(depth.data), imgRGB.data, depth.rows, depth.cols, Tcw, fx,
                            fy, cx, cy, nullptr) != B200ORB_OK)
      throw std::runtime_error(std::string("PointCloudMapping(B200): ") + b200orb_last_error());
  }
  // MapDrawer::UpdateOctomap (perfect/src/MapDrawer.cc:610-638): given the list of all keyframes so far, insert
  // [lastKeyframeSize, N-1) -- the reference never inserts the NEWEST keyframe (`i < N-1`, :615) -- and remember N-1.
  // KeyFrameT supplies GetPose(), fx/fy/cx/cy and the images the P variant stores on the keyframe (mImDep, mImRGB).
  template <class KeyFrameT>
  void UpdateOctomap(const std::vector<KeyFrameT*>& vKFs) {
    const int N = (int)vKFs.size();
    if (N > 1) {
      for (size_t i = lastKeyframeSize; i < (unsigned int)N - 1; i++) {
        cv::Mat gray;
        insertKeyFrame(vKFs[i], gray, vKFs[i]->mImDep, vKFs[i]->mImRGB);
      }
      lastKeyframeSize = N - 1;
    }
  }
  // MapDrawer::SaveOctoMap / LoadOctoMap (perfect/src/MapDrawer.cc:1103-1117): the map as a pruned ColorOcTree `.ot`
  // file.  Loading replaces the map, as the reference replaces m_octree; keyframes inserted afterwards continue from it.
  void SaveOctoMap(const char* filename) {
    if (ocm_save_ot(h_, filename, nullptr) != B200ORB_OK)
      throw std::runtime_error(std::string("PointCloudMapping(B200): ") + b200orb_last_error());
  }
  void LoadOctoMap() { LoadOctoMap("octomap.ot"); }   // the reference's fixed name (:1115)
  void LoadOctoMap(const std::string& filename) {
    if (ocm_load_ot(h_, filename.c_str()) != B200ORB_OK)
      throw std::runtime_error(std::string("PointCloudMapping(B200): ") + b200orb_last_error());
  }
  void shutdown() { ocm_sync(h_); }     // src/pointcloudmapping.cc:104-113 joins the viewer thread
  void update() {}                      // T variant's map refresh hook: nothing to do, the map lives in HBM
  long long numLeaves() { return (long long)ocm_num_leaves(h_); }
  ocm_t* handle() { return h_; }

 protected:
  double resolution;
  ocm_t* h_ = nullptr;
  size_t lastKeyframeSize = 0;
};

// The T variant of the same class (src/pointcloudmapping.cc): no occupancy tree, the map is the accumulated colour cloud
// `globalMap`, re-filtered by VoxelGrid(resolution) after every batch of new keyframes (:395-500).  insertKeyFrame()
// appends the keyframe's full cloud (generatePointCloud :131-194), update() runs the refilter the viewer thread runs when
// it wakes up, globalMapSize()/copyGlobalMap() expose what the viewer / global_color.pcd receive (:496-521).
// The overload that takes the detector's objects runs the semantic part of the same loop (:413-485, the ncnn detector
// itself stays with the caller): it paints each box's depth band into the keyframe's cloud, skips even keyframes without
// objects, and merges each box's cluster into clusters() on the host (sem_merge, :246-322).  The overload without
// objects neither paints nor skips.

// The reference's cluster record (include/pointcloudmapping.h:33-42)
typedef struct Cluster {
  std::string object_name;
  int class_id;
  float prob;
  Eigen::Vector3f minPt;
  Eigen::Vector3f maxPt;
  Eigen::Vector3f centroid;
  bool operator==(const std::string& x) { return this->object_name == x; }
} Cluster;

class PointCloudMappingT {
 public:
  explicit PointCloudMappingT(double resolution_) : resolution(resolution_) {
    obj_size_.assign(21, 0.6f);   // :62-70
    obj_size_[5] = 0.06f;
    obj_size_[9] = 0.5f;
    obj_size_[15] = 0.35f;
    obj_size_[20] = 0.25f;
    int dev = 0;
    if (const char* e = std::getenv("B200ORB_DEVICE")) dev = std::atoi(e);
    if (gcm_create((float)resolution_, dev, &h_) != B200ORB_OK)
      throw std::runtime_error(std::string("PointCloudMapping(B200, T): ") + b200orb_last_error());
  }
  ~PointCloudMappingT() { gcm_destroy(h_); }
  PointCloudMappingT(const PointCloudMappingT&) = delete;
  PointCloudMappingT& operator=(const PointCloudMappingT&) = delete;

  template <class KeyFrameT>
  void insertKeyFrame(KeyFrameT* kf, cv::Mat& color, cv::Mat& depth, cv::Mat& imgRGB) {
    cv::Mat T = kf->GetPose();
    float Tcw[16];
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) Tcw[r * 4 + c] = T.template at<float>(r, c);
    insertKeyFrame(Tcw, kf->fx, kf->fy, kf->cx, kf->cy, color, depth, imgRGB);
  }
  void insertKeyFrame(const float Tcw[16], float fx, float fy, float cx, float cy, cv::Mat& /*gray*/, cv::Mat& depth,
                      cv::Mat& imgRGB) {
    if (gcm_add_keyframe(h_, reinterpret_cast<const float*>(depth.data), imgRGB.data, depth.rows, depth.cols, Tcw, fx, fy,
                         cx, cy) != B200ORB_OK)
      throw std::runtime_error(std::string("PointCloudMapping(B200, T): ") + b200orb_last_error());
    ++keyframes_;
  }
  // The keyframe with the detector's objects (ObjectT: src/ncnn_dect.h:12-18 -- rect, object_name, class_id, prob), as
  // viewer() handles keyframe i = the number of keyframes inserted before it through either overload (:399-485).
  template <class KeyFrameT, class ObjectT>
  void insertKeyFrame(KeyFrameT* kf, cv::Mat& color, cv::Mat& depth, cv::Mat& imgRGB, const std::vector<ObjectT>& objects) {
    cv::Mat T = kf->GetPose();
    float Tcw[16];
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) Tcw[r * 4 + c] = T.template at<float>(r, c);
    insertKeyFrame(Tcw, kf->fx, kf->fy, kf->cx, kf->cy, color, depth, imgRGB, objects);
  }
  template <class ObjectT>
  void insertKeyFrame(const float Tcw[16], float fx, float fy, float cx, float cy, cv::Mat& /*gray*/, cv::Mat& depth,
                      cv::Mat& imgRGB, const std::vector<ObjectT>& objects) {
    std::vector<GcmObject> objs(objects.size());
    for (size_t t = 0; t < objects.size(); ++t) {
      const ObjectT& o = objects[t];
      objs[t] = GcmObject{o.rect.x, o.rect.y, o.rect.width, o.rect.height, (int32_t)o.class_id, o.prob};
    }
    std::vector<GcmCluster> rec(objects.size());
    if (gcm_add_keyframe_objects(h_, reinterpret_cast<const float*>(depth.data), imgRGB.data, depth.rows, depth.cols, Tcw, fx,
                                 fy, cx, cy, keyframes_, objs.data(), (int)objs.size(), rec.data()) != B200ORB_OK)
      throw std::runtime_error(std::string("PointCloudMapping(B200, T): ") + b200orb_last_error());
    ++keyframes_;
    for (size_t t = 0; t < objects.size(); ++t) {   // :443-478; boxes below 51 band points make no cluster
      if (rec[t].status != GCM_CLUSTER) continue;
      Cluster cluster;
      cluster.object_name = objects[t].object_name;
      cluster.class_id = objects[t].class_id;
      cluster.prob = objects[t].prob;
      cluster.minPt = Eigen::Vector3f(rec[t].min_pt[0], rec[t].min_pt[1], rec[t].min_pt[2]);
      cluster.maxPt = Eigen::Vector3f(rec[t].max_pt[0], rec[t].max_pt[1], rec[t].max_pt[2]);
      cluster.centroid = Eigen::Vector3f(rec[t].centroid[0], rec[t].centroid[1], rec[t].centroid[2]);
      sem_merge(cluster);
    }
  }
  const std::vector<Cluster>& clusters() const { return clusters_; }
  void update() {   // the viewer thread's wake-up after new keyframes: voxel.filter(globalMap) + swap
    if (gcm_refilter(h_) != B200ORB_OK) throw std::runtime_error(std::string("PointCloudMapping(B200, T): ") + b200orb_last_error());
  }
  void shutdown() { gcm_sync(h_); }
  long long globalMapSize() { return gcm_size(h_); }
  long long copyGlobalMap(float* xyz, unsigned char* rgb, long long cap) {
    long long n = 0;
    if (gcm_export(h_, xyz, rgb, cap, &n) != B200ORB_OK) throw std::runtime_error(std::string("PointCloudMapping(B200, T): ") + b200orb_last_error());
    return n;
  }
  gcm_t* handle() { return h_; }

 protected:
  // sem_merge (:246-322): the same-named cluster with the nearest centroid absorbs the new one when it is closer than
  // obj_size_[class_id]; prob and centroid become the means, minPt the element-wise min -- and maxPt the element-wise
  // MIN of the two maxima, as the reference writes it (:308-310)
  void sem_merge(const Cluster& cluster) {
    Cluster* best_close = nullptr;
    float center_distance = 100;
    for (Cluster& c : clusters_) {
      if (!(c == cluster.object_name)) continue;
      Eigen::Vector3f dis_vec = cluster.centroid - c.centroid;
      float dist = dis_vec.norm();
      if (dist < center_distance) {
        center_distance = dist;
        best_close = &c;
      }
    }
    if (best_close && center_distance < obj_size_[cluster.class_id]) {
      best_close->prob = (best_close->prob + cluster.prob) / 2.0;
      best_close->centroid = (best_close->centroid + cluster.centroid) / 2.0;
      Eigen::Vector3f mn, mx;
      for (int k = 0; k < 3; ++k) {
        mn[k] = best_close->minPt[k] > cluster.minPt[k] ? cluster.minPt[k] : best_close->minPt[k];
        mx[k] = best_close->maxPt[k] > cluster.maxPt[k] ? cluster.maxPt[k] : best_close->maxPt[k];
      }
      best_close->minPt = mn;
      best_close->maxPt = mx;
    } else {
      clusters_.push_back(cluster);
    }
  }

  double resolution;
  gcm_t* h_ = nullptr;
  long long keyframes_ = 0;        // the `i` of viewer()'s loop over both overloads
  std::vector<float> obj_size_;
  std::vector<Cluster> clusters_;
};
#endif
