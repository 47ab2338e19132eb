/* b200orb.h -- C-ABI of libb200orb.so: the H100 (sm_90a) implementation of the ORB-SLAM2 hot path.
 *
 * The reference (Ewenwan/ORB_SLAM2_SSD_Semantic) has no FFI layer; its boundary is the public surface of
 * three C++ classes (SURVEY.md §8(b)).  Every entry point below names the reference member it replaces
 * (file:line relative to the reference root).  INTEGRATION.md shows the header-only C++ shim classes
 * (orb_slam2_ssd_semantic_b200/csrc/shim/) that keep those class surfaces source-compatible on top of this ABI.
 *
 * Conventions: plain C, caller-owned buffers, int status (0 = OK, <0 = B200ORB_E*), never aborts/exits,
 * no exceptions cross the boundary.  Opaque handles own device memory and one CUDA stream each; calls on
 * DISTINCT handles are re-entrant (the reference runs L/R extractors on two threads, src/Frame.cc:121-124,
 * and matchers on three).  Pointers named d_* are CUDA device pointers, everything else is host memory.
 */
#ifndef B200ORB_H_
#define B200ORB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200ORB_OK 0
#define B200ORB_EINVAL (-1)     /* bad argument */
#define B200ORB_ECAP (-2)       /* caller buffer too small */
#define B200ORB_ECUDA (-3)      /* CUDA runtime error (see b200orb_last_error) */
#define B200ORB_ENOGPU (-4)     /* no usable CUDA device: there is NO CPU fallback */
#define B200ORB_EGEOM (-5)      /* image geometry the reference itself cannot process */

const char* b200orb_last_error(void);   /* thread-local message of the last failing call */
int b200orb_device_count(void);         /* number of CUDA devices visible (0 if none / no driver) */
const char* b200orb_version(void);
/* Read-only report of the extractor kernels this build runs (fixed at compile time; NULL pointers are skipped):
 * exp_mask = 3 (the orientation + descriptor formulation, bit 0, and the four-row FAST tile staging, bit 1),
 * fast_wpc = FAST cells per CTA (8), qt_minblocks = the quad-tree's register budget in CTAs per SM (4). */
int b200orb_get_tuning(int* exp_mask, int* fast_wpc, int* qt_minblocks);

/* ------------------------------------------------------------------------------------------------
 * ORB extractor  --  ORB_SLAM2::ORBextractor (include/ORBextractor.h:41-118, src/ORBextractor.cc)
 * ------------------------------------------------------------------------------------------------ */
typedef struct orbx orbx_t;

typedef struct {            /* ctor arguments, src/ORBextractor.cc:399-400 */
  int nfeatures;
  float scale_factor;
  int nlevels;
  int ini_th_fast;
  int min_th_fast;
} OrbxParams;

typedef struct {            /* cv::KeyPoint, 28 bytes, what operator() appends to _keypoints */
  float x, y, size, angle, response;
  int32_t octave, class_id;
} OrbxKeyPoint;

/* ORBextractor::ORBextractor (src/ORBextractor.cc:399-466).  device = CUDA ordinal. */
int orbx_create(const OrbxParams* p, int device, orbx_t** out);
void orbx_destroy(orbx_t* h);

/* Keypoints one frame can return, summed over the levels: max(N_l + 3, 4*nIni_l), where nIni_l, DistributeOctTree's
 * number of initial nodes (src/ORBextractor.cc:545), follows from the level's aspect ratio.  orbx_max_keypoints_for gives
 * the bound of a rows x cols image without allocating anything; it refuses what extraction refuses (rows or cols <= 0:
 * *n = 0, OK).  orbx_max_keypoints gives that of the handle's current geometry, or, before the first extract, the bound
 * of images with nIni <= 4 on every level -- wide images (100 x 4000: nIni = 58) need more. */
int orbx_max_keypoints(const orbx_t* h);
int orbx_max_keypoints_for(const orbx_t* h, int rows, int cols, int* n);

/* ORBextractor::operator() (src/ORBextractor.cc:1052-1114) on one HOST image (CV_8UC1, row stride in bytes).
 * kps[cap], desc[cap*32] are host buffers; *n_out keypoints are written level-major exactly as the
 * reference orders them.  rows==0||cols==0 -> *n_out = 0, OK (reference: silent return, :1055). */
int orbx_extract(orbx_t* h, const uint8_t* gray, int rows, int cols, size_t stride,
                 OrbxKeyPoint* kps, uint8_t* desc, int cap, int* n_out);

/* Batched many-frame mode (north_star): nframes images of identical geometry, frame f at
 * gray + f*frame_stride.  Outputs: kps[f*cap ..], desc[(f*cap)*32 ..], n_out[f].  Host buffers. */
int orbx_extract_batch(orbx_t* h, const uint8_t* gray, int nframes, int rows, int cols, size_t stride,
                       size_t frame_stride, OrbxKeyPoint* kps, uint8_t* desc, int cap, int* n_out);

/* Same, with the images already resident in HBM (d_gray) and results LEFT in HBM: after the call
 * orbx_device_results() returns device pointers valid until the next extract on this handle.
 * Asynchronous on the handle's stream; orbx_sync() waits. */
int orbx_extract_batch_device(orbx_t* h, const uint8_t* d_gray, int nframes, int rows, int cols,
                              size_t stride, size_t frame_stride);
int orbx_device_results(orbx_t* h, const OrbxKeyPoint** d_kps, const uint8_t** d_desc,
                        const int32_t** d_counts, int* cap);
int orbx_sync(orbx_t* h);
void* orbx_stream(orbx_t* h);   /* cudaStream_t the handle launches on */

/* Backs the public member mvImagePyramid (include/ORBextractor.h:80): level image of frame `frame` of the
 * last extract.  kind=0: rows x cols level (the ROI the reference stores); kind=1: the
 * (rows+38)x(cols+38) parent buffer with the BORDER_REFLECT_101 frame (src/ORBextractor.cc:1125-1142);
 * kind=2: rows x cols GaussianBlur 7x7 of the level, the image the descriptors read (:1094-1095). */
int orbx_level_dims(const orbx_t* h, int level, int* rows, int* cols);
int orbx_get_level(orbx_t* h, int frame, int level, int kind, uint8_t* dst, size_t dst_stride);

/* GetScaleFactors / GetInverseScaleFactors / GetScaleSigmaSquares / GetInverseScaleSigmaSquares
 * (include/ORBextractor.h:63-77) + mnFeaturesPerLevel; each array has nlevels entries (NULL = skip). */
int orbx_scale_tables(const orbx_t* h, float* sf, float* inv_sf, float* sigma2, float* inv_sigma2,
                      int* features_per_level);

/* Diagnostics for parity tests: FAST candidates per level of frame `frame` of the last extract. */
int orbx_candidates_per_level(orbx_t* h, int frame, int* counts /*nlevels*/);
/* The FAST candidates of one level of frame `frame` of the last extract, in the order the quad-tree reads them
 * (vToDistributeKeys, src/ORBextractor.cc:788-843): cell by cell, row-major inside a cell.  xys[3*i..3*i+2] = x, y (level
 * pixels) and score.  *n = the count; cap < *n: B200ORB_ECAP and nothing written. */
int orbx_get_candidates(orbx_t* h, int frame, int level, int32_t* xys, int cap, int* n);
/* DistributeOctTree (src/ORBextractor.cc:540-765) alone, run by the extractor's quad-tree kernel on a caller's candidate
 * list for level `level` of a rows x cols geometry.  xys[3*i..3*i+2] = x, y (level pixels) and score, in
 * vToDistributeKeys order, n of them; N = the level's target, 0 <= N <= mnFeaturesPerLevel[level].  out[3*j..] = the
 * selected keypoints in list order, *n_out = their count (cap < *n_out: B200ORB_ECAP, nothing written).  Refused with
 * nothing launched: a level or N out of range, a coordinate outside the level's distribution region [16, maxBorderX) x
 * [16, maxBorderY), a score outside 0..255, null pointers, and (B200ORB_ECAP) n above the level's FAST slot capacity.
 * Synchronous.  Replaces the handle's last results: the read-backs above refuse until the next extract. */
int orbx_distribute(orbx_t* h, int rows, int cols, int level, int N, const int32_t* xys, int n, int32_t* out, int cap,
                    int* n_out);
/* Number of CUDA kernels launched by this handle since creation (bench.py's gpu_launches). */
long long orbx_launch_count(const orbx_t* h);
/* Per-stage device time via CUDA events on the handle's stream (bench.py's roofline leg).  Stages:
 * 0 pyramid resize, 1 FAST cells, 2 quad-tree, 3 blur, 4 orientation+descriptor, 5 frame glue, 6 match
 * (5,6 only when driven through orbs_*).  read() sums ms per stage over all runs since the last read. */
#define B200ORB_NUM_STAGES 7
int orbx_profile_enable(orbx_t* h, int on);
int orbx_profile_read(orbx_t* h, float* ms, long long* frames, int* runs);

/* ------------------------------------------------------------------------------------------------
 * ORB matcher  --  ORB_SLAM2::ORBmatcher (include/ORBmatcher.h:37-118, src/ORBmatcher.cc)
 * ------------------------------------------------------------------------------------------------ */
#define ORBM_TH_HIGH 100      /* src/ORBmatcher.cc:39 */
#define ORBM_TH_LOW 50        /* :40 */
#define ORBM_HISTO_LENGTH 30  /* :41 */
#define ORBM_GRID_COLS 64     /* include/Frame.h:26 */
#define ORBM_GRID_ROWS 48     /* include/Frame.h:25 */

/* ORBmatcher::DescriptorDistance (src/ORBmatcher.cc:1968-1984): Hamming distance of two 256-bit rows. */
int orbm_hamming(const uint8_t a[32], const uint8_t b[32]);

typedef struct orbm orbm_t;   /* workspace + stream; the matcher itself is stateless like the reference's */
int orbm_create(int device, orbm_t** out);
void orbm_destroy(orbm_t* h);
long long orbm_launch_count(const orbm_t* h);

/* Flat view of the "current" Frame the searches read (src/Frame.cc / include/Frame.h). */
typedef struct {
  int n;                      /* Frame::N */
  const float* x;             /* mvKeysUn[i].pt.x */
  const float* y;             /* mvKeysUn[i].pt.y */
  const int32_t* octave;      /* mvKeysUn[i].octave */
  const float* angle;         /* mvKeysUn[i].angle */
  const float* uright;        /* mvuRight[i] (<=0: none) */
  const uint8_t* desc;        /* mDescriptors, n x 32 */
  const int32_t* mp_obs;      /* per keypoint: -1 if mvpMapPoints[i]==NULL else that MapPoint's Observations();
                                 NULL = all -1 (what Tracking does before the call, src/Tracking.cc:1337) */
  float Tcw[16];              /* mTcw row-major 4x4 */
  float fx, fy, cx, cy, bf, b;        /* mbf, mb */
  float min_x, max_x, min_y, max_y;   /* mnMinX.. (static image bounds) */
  const float* scale_factors; /* mvScaleFactors, nlevels entries */
  int nlevels;
} OrbmFrame;

/* "Last frame" side of SearchByProjection(Frame&, const Frame&, th, bMono). */
typedef struct {
  int n;                      /* LastFrame.N */
  const float* xw;            /* n x 3: pMP->GetWorldPos() of LastFrame.mvpMapPoints[i] (ignored where !valid) */
  const uint8_t* valid;       /* 1 iff mvpMapPoints[i] != NULL && !mvbOutlier[i] */
  const int32_t* octave;      /* LastFrame.mvKeys[i].octave */
  const float* angle;         /* LastFrame.mvKeysUn[i].angle */
  const uint8_t* mp_desc;     /* n x 32: pMP->GetDescriptor() */
  const int32_t* mp_obs;      /* pMP->Observations() (decides whether a claimed keypoint blocks later queries,
                                 src/ORBmatcher.cc:1656-1658); NULL = all 0 */
  float Tcw[16];              /* LastFrame.mTcw */
} OrbmLast;

/* ORBmatcher::SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, th, bMono)
 * (src/ORBmatcher.cc:1578-1724).  cur2last[cur.n]: index i of the LastFrame keypoint whose MapPoint ends up
 * in CurrentFrame.mvpMapPoints[j], or -1 (NULL) -- i.e. exactly the pointer state the reference leaves
 * (pre-existing entries given through cur->mp_obs are reported as -2 when they survive untouched).
 * *nmatches = the function's return value (may double-count, SURVEY App. B.8).  Host buffers. */
int orbm_search_by_projection_last(orbm_t* h, const OrbmFrame* cur, const OrbmLast* last, float th, int mono,
                                   float nnratio, int check_ori, int32_t* cur2last, int* nmatches);

/* The perfect tree's overload SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, th, bMono,
 * vector<cv::Point2f>& points_last, vector<cv::Point2f>& points_current) (perfect/src/ORBmatcher.cc:1727-1880):
 * the same search, plus the claim list it pushes the 2-D point pairs from (:1835-1836, inside `bestDist<=TH_HIGH`,
 * BEFORE the rotation prune).  last2cur_accepted[last.n]: the current keypoint bestIdx2 that query i accepted, or -1;
 * a pair the prune later drops stays listed, and a current keypoint whose MapPoint has no observations can appear
 * twice.  The caller builds the pairs (mvKeys[i].pt, mvKeys[j].pt) in ascending i.  cur2last and *nmatches are those of
 * orbm_search_by_projection_last; same kernels, same results.  Host buffers. */
int orbm_search_by_projection_last_pairs(orbm_t* h, const OrbmFrame* cur, const OrbmLast* last, float th, int mono,
                                         float nnratio, int check_ori, int32_t* cur2last, int32_t* last2cur_accepted,
                                         int* nmatches);

/* Local-map search: ORBmatcher::SearchByProjection(Frame &F, const vector<MapPoint*>&, th)
 * (src/ORBmatcher.cc:63-156); the per-MapPoint fields are those Frame::isInFrustum fills (src/Frame.cc:387-451). */
typedef struct {
  int n;
  const uint8_t* track_in_view;   /* mbTrackInView && !isBad() */
  const float* proj_x;            /* mTrackProjX */
  const float* proj_y;            /* mTrackProjY */
  const float* proj_xr;           /* mTrackProjXR */
  const int32_t* scale_level;     /* mnTrackScaleLevel */
  const float* view_cos;          /* mTrackViewCos */
  const uint8_t* mp_desc;         /* n x 32 */
  const int32_t* mp_obs;          /* Observations(); NULL = all 1 */
} OrbmTrackPoints;
int orbm_search_by_projection_points(orbm_t* h, const OrbmFrame* f, const OrbmTrackPoints* pts, float th,
                                     float nnratio, int32_t* f2pt, int* nmatches);

/* Generic guided search for the remaining projection overloads: the caller (shim) has already projected its MapPoints
 * and chosen window + octave range per query -- SearchByProjection(Frame&, KeyFrame*, set, th, ORBdist)
 * (src/ORBmatcher.cc:1757-1899, relocalisation) and the Sim3 / loop-closing variants do that part in a dozen
 * scalar lines each (PredictScale, distance gates) -- and the GPU does what they share: GetFeaturesInArea, the Hamming
 * loop, the ordered "already matched" rule, the rotation histogram.
 *   claim_rule 0: a keypoint blocks later queries iff the MapPoint holding it has Observations()>0 (:1656-1658)
 *   claim_rule 1: any MapPoint already on the keypoint blocks it (:1830-1831 `if(CurrentFrame.mvpMapPoints[i2]) continue`)
 * cur2q[j] = query index now on keypoint j (-1 NULL, -2 untouched pre-existing). */
typedef struct {
  int n;
  const uint8_t* valid;        /* query takes part (MapPoint non-NULL, !isBad(), in image, distance gates passed) */
  const float* u;              /* projected pixel */
  const float* v;
  const float* radius;         /* th * mvScaleFactors[nPredictedLevel] */
  const int32_t* min_level;    /* GetFeaturesInArea(minLevel, maxLevel) semantics (src/Frame.cc:486-506) */
  const int32_t* max_level;
  const float* uright;         /* predicted right coordinate for the stereo gate; NULL = no gate */
  const uint8_t* desc;         /* n x 32: pMP->GetDescriptor() */
  const float* angle;          /* angle used for the rotation histogram (e.g. pKF->mvKeysUn[i].angle) */
  const int32_t* obs;          /* Observations() per query (claim_rule 0); NULL = all 1 */
} OrbmQueries;
int orbm_search_projected(orbm_t* h, const OrbmFrame* cur, const OrbmQueries* q, int max_dist, int claim_rule,
                          int check_ori, int32_t* cur2q, int* nmatches);

/* ORBmatcher::SearchByBoW(KeyFrame*, Frame&, vector<MapPoint*>&) (src/ORBmatcher.cc:217-363).
 * The two DBoW2::FeatureVector maps are given flattened and sorted by node id:
 * node_ids[k] (strictly ascending), indices of node k = idx[node_off[k] .. node_off[k+1]). */
typedef struct {
  int n;                       /* keypoints */
  const uint8_t* desc;         /* n x 32 */
  const float* angle;          /* KF: mvKeysUn[i].angle ; F: mvKeys[i].angle (src/ORBmatcher.cc:301,308) */
  const uint8_t* valid;        /* KF side: MapPoint non-NULL && !isBad(); F side: NULL */
  int n_nodes;
  const uint32_t* node_ids;
  const int32_t* node_off;     /* n_nodes+1 */
  const uint32_t* idx;
} OrbmBow;
int orbm_search_by_bow(orbm_t* h, const OrbmBow* kf, const OrbmBow* f, float nnratio, int check_ori,
                       int32_t* f2kf /* f->n, -1 = none */, int* nmatches);
/* ORBmatcher::SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, vector<MapPoint*>& vpMatches12) (src/ORBmatcher.cc:665-812,
 * loop closing): both sides carry `valid` (MapPoint non-NULL && !isBad()); matches12[kf1->n] = index of the pKF2
 * keypoint whose MapPoint lands in vpMatches12[i], or -1. */
int orbm_search_by_bow_kf(orbm_t* h, const OrbmBow* kf1, const OrbmBow* kf2, float nnratio, int check_ori,
                          int32_t* matches12, int* nmatches);

/* Per-query best keypoint of a keyframe, with NO claim state: the device part of
 *   Fuse(KeyFrame*, const vector<MapPoint*>&, th)            src/ORBmatcher.cc:1031-1182   gate 1 (reprojection chi-square,
 *                                                            :1118-1146: needs q->uright = u - bf*invz and inv_level_sigma2)
 *   Fuse(KeyFrame*, Scw, vpPoints, th, vpReplacePoint)       src/ORBmatcher.cc:1198-1318   gate 0
 *   SearchBySim3 (each direction)                            src/ORBmatcher.cc:1334-1558   gate 0
 * The caller (shim) projects its MapPoints and passes the distance / viewing-angle gates, PredictScale and the radius
 * exactly as those loop heads do (queries: u, v, radius, min_level = nPredictedLevel-1, max_level = nPredictedLevel,
 * descriptor); the device walks KeyFrame::GetFeaturesInArea (src/KeyFrame.cc:659-698), applies the level range and the
 * gate and returns the FIRST minimum of the Hamming distance: best_idx[i] (-1: no candidate), best_dist[i].  What happens
 * with a match (Replace / AddObservation / mutual-consistency test) stays with the caller, in the reference's order --
 * none of it feeds back into later queries' candidate sets. */
int orbm_search_best(orbm_t* h, const OrbmFrame* kf, const OrbmQueries* q, int gate, const float* inv_level_sigma2,
                     int32_t* best_idx, int32_t* best_dist);

/* ORBmatcher::SearchForInitialization(Frame& F1, Frame& F2, vector<Point2f>& vbPrevMatched, vector<int>& vnMatches12,
 * int windowSize) (src/ORBmatcher.cc:523-651).  F1 supplies octave / angle / descriptors, F2 additionally its grid;
 * prev_xy[n1][2] = vbPrevMatched (in / out); matches12[n1] = vnMatches12. */
int orbm_search_for_initialization(orbm_t* h, const OrbmFrame* f1, const OrbmFrame* f2, float* prev_xy, int window,
                                   float nnratio, int check_ori, int32_t* matches12, int* nmatches);

/* ORBmatcher::SearchForTriangulation(KeyFrame* pKF1, KeyFrame* pKF2, cv::Mat F12, vector<pair<size_t,size_t>>&,
 * bOnlyStereo) (src/ORBmatcher.cc:827-1019).  Both keyframes flattened with their FeatureVector (as OrbmBow), undistorted
 * keypoints, right coordinates and MapPoint occupancy; F12 row-major 3x3; (ex, ey) = the epipole the caller computes from
 * the two poses (:835-839); scale_factors2 / level_sigma2_2 = pKF2->mvScaleFactors / mvLevelSigma2.  matches12[k1->n] =
 * pKF2 keypoint matched to pKF1 keypoint i or -1 (the caller turns it into vMatchedPairs in index order). */
typedef struct {
  int n;
  const uint8_t* desc;         /* n x 32 */
  const float* x;              /* mvKeysUn[i].pt */
  const float* y;
  const float* angle;
  const float* uright;         /* mvuRight (>= 0: stereo) */
  const int32_t* octave;
  const uint8_t* has_mp;       /* GetMapPoint(i) != NULL */
  int n_nodes;
  const uint32_t* node_ids;
  const int32_t* node_off;
  const uint32_t* idx;
} OrbmTriKF;
int orbm_search_for_triangulation(orbm_t* h, const OrbmTriKF* kf1, const OrbmTriKF* kf2, const float F12[9], float ex,
                                  float ey, const float* scale_factors2, const float* level_sigma2_2, int nlevels,
                                  int only_stereo, int check_ori, int32_t* matches12, int* nmatches);

/* Frame::isInFrustum (src/Frame.cc:387-451) for n MapPoints at once -- what Tracking::SearchLocalPoints runs per local
 * MapPoint before SearchByProjection(Frame&, vector<MapPoint*>&, th) (src/Tracking.cc:1931-1946): projection, image and
 * distance-invariance gates, viewing-angle gate, MapPoint::PredictScale.  The outputs are exactly the per-MapPoint fields
 * OrbmTrackPoints wants (mbTrackInView, mTrackProjX/Y/XR, mnTrackScaleLevel, mTrackViewCos); entries not in view are 0.
 * log_scale_factor = Frame::mfLogScaleFactor; min_dist / max_dist = mfMinDistance / mfMaxDistance (raw members). */
typedef struct {
  int n;
  const float* xw;        /* n x 3 GetWorldPos() */
  const float* normal;    /* n x 3 GetNormal() */
  const float* min_dist;  /* mfMinDistance */
  const float* max_dist;  /* mfMaxDistance */
} OrbmFrustumPoints;
int orbm_is_in_frustum(orbm_t* h, const OrbmFrame* f, const OrbmFrustumPoints* p, float viewing_cos_limit,
                       float log_scale_factor, uint8_t* in_view, float* proj_x, float* proj_y, float* proj_xr,
                       int32_t* scale_level, float* view_cos);

/* Frame::UndistortKeyPoints (src/Frame.cc:559-590): cv::undistortPoints(pts, pts, mK, mDistCoef, Mat(), mK) on n keypoint
 * positions (xy interleaved); K row-major 3x3, dist = k1 k2 p1 p2 [k3].  dist[0] == 0 copies the input (:561-565). */
int orbm_undistort_keypoints(orbm_t* h, const float* xy_in, int n, const float K[9], const float* dist, int ndist,
                             float* xy_out);

/* ------------------------------------------------------------------------------------------------
 * BoW transform -- Frame::ComputeBoW / KeyFrame::ComputeBoW (src/Frame.cc:546-555, src/KeyFrame.cc:75-84):
 * mpORBvocabulary->transform(vCurrentDesc, mBowVec, mFeatVec, 4) of DBoW2's TemplatedVocabulary (k-ary tree; ORBvoc: k = 10,
 * L = 6).  orbv_create uploads the tree: node 0 = root, parent[i] < i, children visited in ascending node id, leaves are
 * the words numbered in ascending node id, desc n_nodes x 32, weight = node weights (TF-IDF: the idf of the word).
 * orbv_transform descends every descriptor (first child at minimal Hamming distance per level) and returns per feature
 * the word id, the word's weight and the id of the ancestor `levelsup` levels above the leaves (0 = root when L - levelsup
 * <= 0).  The caller builds the maps in feature order exactly like TemplatedVocabulary::transform does:
 *   if (weight > 0) { BowVector.addWeight(word, weight); FeatureVector.addFeature(node, i); }  then  BowVector.normalize(L1).
 * ------------------------------------------------------------------------------------------------ */
typedef struct orbv orbv_t;
int orbv_create(int device, int k, int L, int n_nodes, const int32_t* parent, const uint8_t* desc, const double* weight,
                const int32_t* word_id /* per node, read at leaves; NULL = leaves numbered in ascending node id */, orbv_t** out);
void orbv_destroy(orbv_t* h);
int orbv_num_words(const orbv_t* h);
long long orbv_launch_count(const orbv_t* h);
int orbv_transform(orbv_t* h, const uint8_t* desc, int n, int levelsup, uint32_t* word_id, double* word_weight,
                   uint32_t* node_id);

/* ------------------------------------------------------------------------------------------------
 * Key-frame database -- KeyFrameDatabase (src/KeyFrameDatabase.cc): the inverted file of add / erase / clear (:39-73) and
 * the walk, the common-word counts and the L1 scores of DetectLoopCandidates (:76-139) and
 * DetectRelocalizationCandidates (:199-253).  The covisibility accumulation and the 0.75f * bestAccScore filter that follow
 * (:141-196, :255-308) read GetBestCovisibilityKeyFrames(10) of the caller's objects and stay with the caller
 * (shim/KeyFrameDatabase.h).
 *
 * A slot is the caller's handle of one keyframe (0 <= slot < 2^24).  The database keeps per slot its BowVector (ascending
 * word ids < n_words, L1-scoring weights) and a mirror of the six KeyFrame members the database writes (OrbvDbMembers).
 *   orbv_db_add    KeyFrameDatabase::add (:39-45).  A slot added k times without an erase is in each of its lists k times
 *                  and counted k times.  `members`: the keyframe's current values (NULL keeps the mirror; a slot never
 *                  added before starts at zero).  A slot already in the database keeps the BowVector it was added with.
 *   orbv_db_erase  KeyFrameDatabase::erase (:47-67) with the BowVector the slot was added with: removes the slot's earliest
 *                  add from every list; a slot not in the database is left as it is (the reference's loops find nothing).
 *   orbv_db_clear  KeyFrameDatabase::clear (:69-73): every list empty; the mirrors stay (they are the objects' members).
 *   orbv_db_query  the walk and the scores of one query: kind ORBV_DB_RELOC (query_id = Frame::mnId) or ORBV_DB_LOOP
 *                  (query_id = KeyFrame::mnId, connected = GetConnectedKeyFrames() as slots; unknown keyframes may be left
 *                  out).  words / weights: the query's BowVector.  out[0 .. *n_appended) are lKFsSharingWords in list
 *                  order (flag ORBV_DB_SCORED when words > minCommonWords: score = (float)TemplatedVocabulary::score);
 *                  out[*n_appended .. *n_met) are the other slots the walk met.  Every record carries the slot's new
 *                  query / words / score of `kind`; slots the walk did not meet are unchanged.  The loop filter si >=
 *                  minScore is the caller's.  cap >= orbv_db_state's *n_live (else B200ORB_ECAP, nothing changes).
 *   orbv_db_state  one slot's mirror and how many times it is in the database (NULL outputs are skipped; slot -1: only
 *                  *n_live, the number of slots in the database).
 * B200ORB_EINVAL: a word id >= n_words, word ids not strictly ascending, a slot out of range, an unknown slot for
 * orbv_db_erase / orbv_db_state.  One host sync per query (the result copy).
 * ------------------------------------------------------------------------------------------------ */
typedef struct orbv_db orbv_db_t;
typedef struct {
  uint64_t loop_query;   /* mnLoopQuery */
  int32_t loop_words;    /* mnLoopWords */
  float loop_score;      /* mLoopScore */
  uint64_t reloc_query;  /* mnRelocQuery */
  int32_t reloc_words;   /* mnRelocWords */
  float reloc_score;     /* mRelocScore */
} OrbvDbMembers;
typedef struct {
  int32_t slot;
  int32_t words;         /* mnRelocWords / mnLoopWords after the walk */
  uint64_t query;        /* mnRelocQuery / mnLoopQuery after the walk */
  float score;           /* mRelocScore / mLoopScore after the query */
  int32_t flags;         /* ORBV_DB_APPENDED | ORBV_DB_SCORED */
} OrbvDbHit;
#define ORBV_DB_RELOC 0
#define ORBV_DB_LOOP 1
#define ORBV_DB_APPENDED 1
#define ORBV_DB_SCORED 2
int orbv_db_create(int device, int n_words, orbv_db_t** out);
void orbv_db_destroy(orbv_db_t* h);
int orbv_db_add(orbv_db_t* h, int slot, const uint32_t* words, const double* weights, int n, const OrbvDbMembers* members);
int orbv_db_erase(orbv_db_t* h, int slot);
int orbv_db_clear(orbv_db_t* h);
int orbv_db_query(orbv_db_t* h, int kind, uint64_t query_id, const uint32_t* words, const double* weights, int n,
                  const int32_t* connected, int n_connected, OrbvDbHit* out, int cap, int* n_appended, int* n_met);
int orbv_db_state(orbv_db_t* h, int slot, OrbvDbMembers* members, int* count, int* n_live);
long long orbv_db_launch_count(const orbv_db_t* h);

/* ------------------------------------------------------------------------------------------------
 * Dynamic-mask stages of the `perfect` variant (SURVEY 8(f4), the image-arithmetic parts):
 *   FlowSLAM::Flow::ComputeMask (perfect/include/Flow.h:24-27, perfect/src/Flow.cc:17-52) after the call of
 *   cv::calcOpticalFlowFarneback -- which stays on the host side: OpenCV's own float code -- i.e. pyrUp of the half-
 *   resolution flow field (:30), mask = 1 except 0 where x*x + y*y >= max(BInaryThreshold, 40) (:24,31-41), then
 *   erode, erode, dilate with getStructuringElement(MORPH_ELLIPSE, 21x21) (:42-47);
 *   and the keypoint loop of the masked RGB-D Frame constructor (perfect/src/Frame.cc:356-377): if cv::sum(mask) >
 *   rows*cols*0.65, keypoints whose pixel mask.at<uchar>(pt.y, pt.x) is not 1 are dropped together with their
 *   descriptor rows, order kept; otherwise nothing is dropped.
 * flow: rows x cols x 2 float (CV_32FC2, continuous) at half resolution; mask: mask_rows x mask_cols bytes (0 / 1),
 * continuous, the size of the gray image (2 rows <= mask_rows <= 2 rows + 1, likewise the columns: pyrDown halves with
 * truncation); pixels beyond the 2 rows x 2 cols the up-sampled flow covers keep their initial 1 (:25).
 * ------------------------------------------------------------------------------------------------ */
typedef struct dynm dynm_t;
int dynm_create(int device, dynm_t** out);
void dynm_destroy(dynm_t* h);
long long dynm_launch_count(const dynm_t* h);
void* dynm_stream(dynm_t* h);
int dynm_sync(dynm_t* h);
int dynm_element(const dynm_t* h, uint8_t* element /* 21 x 21: the structuring element in use */);
int dynm_mask_from_flow(dynm_t* h, const float* flow, int rows, int cols, float binary_threshold, uint8_t* mask, int mask_rows,
                        int mask_cols);
/* nframes flow fields / masks back to back in HBM, asynchronous on the handle's stream */
int dynm_mask_from_flow_batch_device(dynm_t* h, const float* d_flow, int nframes, int rows, int cols, float binary_threshold,
                                     uint8_t* d_mask, int mask_rows, int mask_cols);
/* host buffers, filtered in place; *n_out keypoints remain */
int dynm_filter_keypoints(dynm_t* h, const uint8_t* mask, int rows, int cols, size_t stride, OrbxKeyPoint* kps, uint8_t* desc,
                          int n, int* n_out);
/* the layout of orbx_device_results / orbs_device_results: kps [nframes][cap], desc [nframes][cap][32], counts [nframes],
 * masks [nframes][rows][cols]; filtered in place, asynchronous on the handle's stream */
int dynm_filter_keypoints_batch_device(dynm_t* h, const uint8_t* d_mask, int nframes, int rows, int cols, OrbxKeyPoint* d_kps,
                                       uint8_t* d_desc, int32_t* d_counts, int cap);
/* The dense optical flow of ComputeMask on the device (perfect/src/Flow.cc:26,29): pyrDown of the u8 gray image to
 * Size(cols / 2, rows / 2), then calcOpticalFlowFarneback(prev, cur, flow, 0.5, 3, 15, 3, 5, 1.2, 0) of the previous and
 * current half-resolution images, bit for bit as OpenCV 4.13 computes it at its baseline dispatch level
 * (cv::setUseOptimized(false): SSE2/SSE3 code, no FMA, no IPP; with AVX2/FMA dispatch OpenCV's own result differs in
 * the last bits).  Both half-resolution sides must lie in [16, 2048]; other sizes return B200ORB_EINVAL.
 *
 * dynm_farneback: exactly the call at Flow.cc:29 with its fixed arguments.  prev, cur: rows x cols u8 (continuous,
 * half resolution); flow: rows x cols x 2 f32 (CV_32FC2).  Host buffers, synchronous. */
int dynm_farneback(dynm_t* h, const uint8_t* prev, const uint8_t* cur, int rows, int cols, float* flow);
/* Flow.cc:26-29 for nframes consecutive full-resolution gray images d_gray[n][rows][cols] u8 in HBM: pyrDown of each, then
 * the flow from frame t-1 to frame t into d_flow[t][rows / 2][cols / 2][2] f32 -- the layout
 * OrbsBatch.flow takes.  d_prev is the frame before d_gray[0] (rows x cols u8 in HBM); NULL: the sequence
 * starts at d_gray[0], whose flow is the zero field (the reference's first-frame `mask = ones`).  Asynchronous on the
 * handle's stream; the scratch grows with min(nframes, 64) frames of the geometry (about 7 MB per frame at 640 x 480). */
int dynm_flow_batch_device(dynm_t* h, const uint8_t* d_gray, const uint8_t* d_prev, int nframes, int rows, int cols,
                           float* d_flow);
/* The homography branch of ComputeMask (perfect/src/Flow.cc:73-80): cv::warpPerspective(GrayImg, dest, Homo,
 * GrayImg.size()) on the device -- u8, one channel, INTER_LINEAR, BORDER_CONSTANT 0, Homo inverted first (no
 * WARP_INVERSE_MAP) -- bit for bit as OpenCV 4.13 computes it, at every dispatch level.  H: the forward map as
 * findHomography returns it, row-major double[9]; a singular H inverts to zeros and, as in OpenCV, every pixel then takes
 * the value of pixel (0, 0).  Both sides must lie in [1, 32766] (cv::remap asserts < SHRT_MAX); other sizes return
 * B200ORB_EINVAL before anything is enqueued.
 *
 * dynm_warp_perspective: gray, dst: rows x cols u8 (continuous).  Host buffers, synchronous. */
int dynm_warp_perspective(dynm_t* h, const uint8_t* gray, int rows, int cols, const double* H, uint8_t* dst);
/* nframes images d_gray[n][rows][cols] u8, each warped by its own d_H[n][9] into d_dst[n][rows][cols] (all in HBM; d_dst
 * must not overlap d_gray).  At most 65535 frames per call.  Asynchronous on the handle's stream. */
int dynm_warp_perspective_batch_device(dynm_t* h, const uint8_t* d_gray, int nframes, int rows, int cols, const double* d_H,
                                       uint8_t* d_dst);
/* The homography TrackHomo feeds that warp (perfect/src/Tracking.cc:1386): cv::findHomography(points_current,
 * points_last, RANSAC, 3) with maxIters 2000 and confidence 0.995 -- RANSAC, runKernel on the inliers, the
 * Levenberg-Marquardt refinement (at most 10 iterations over 9 parameters), H scaled by 1 / H22 and the mask of the
 * refined H (float reprojection error <= 9) -- in the order of operations of OpenCV 4.13's baseline dispatch
 * (cv::setUseOptimized(false)), as tests/homography_lm.py restates it: equal to that restatement bit for bit, and to
 * cv2 bit for bit below 50 inliers (from 100 residual rows a cv2 built with LAPACK sums J^T r in its BLAS's order).  src = points_current, dst = points_last:
 * float[n][2] host buffers; synchronous.  Exactly 4 pairs: runKernel of all four, unrefined, mask all ones.  No model
 * (every subset degenerate, or getSubset rejecting 10000 draws in a row before the first hypothesis): *found = 0, H
 * zeros and mask all zeros, as cv2 returns an empty H and a zero mask.  Otherwise *found = 1 and H is row-major double[9].
 * n outside [4, 8192] or a NULL pointer returns B200ORB_EINVAL before anything is enqueued. */
int dynm_find_homography(dynm_t* h, const float* src, const float* dst, int n, double H[9], uint8_t* mask, int* found);

/* ------------------------------------------------------------------------------------------------
 * Stream pipeline (batched many-frame mode of north_star): per frame t of a batch, what
 * Tracking::GrabImageRGBD -> Frame::Frame(RGB-D) -> TrackWithMotionModel's SearchByProjection do
 * (src/Tracking.cc:331-375,1324-1352; src/Frame.cc:176-240): extract, ComputeStereoFromRGBD
 * (src/Frame.cc:850-871), AssignFeaturesToGrid (:319-334), UnprojectStereo (:879-899) of frame t-1's
 * keypoints into "map points", then SearchByProjection(frame t, frame t-1, th, mono=0).
 * ------------------------------------------------------------------------------------------------ */
typedef struct orbs orbs_t;
typedef struct {
  OrbxParams orb;
  float fx, fy, cx, cy, bf;     /* Camera.* of the YAML (perfect/Examples/RGB-D/TUM3.yaml:8-25) */
  float th;                     /* search window, 15 in src/Tracking.cc:1346 */
  float nnratio;                /* 0.9 (src/Tracking.cc:1327) */
  int check_ori;                /* 1 */
  int max_frames;               /* batch capacity */
} OrbsParams;
int orbs_create(const OrbsParams* p, int device, orbs_t** out);
void orbs_destroy(orbs_t* h);
/* One batch of orbs_submit: gray[n][rows][cols] u8, Tcw[n][16] f32 row-major, one depth image per frame.  Exactly eight
 * forms are accepted:
 *   host batches (device = 0):    f32 depth | CV_16U depth | CV_16U depth + flow | CV_16U depth + device_flow |
 *                                 CV_16U depth + device_flow + homography (prev_gray NULL)
 *   device batches (device = 1):  f32 depth | f32 depth + flow
 * Every other combination -- and a NULL input, a non-positive size, both depths or neither, prev_gray without
 * device_flow, homography other than 0 or 1 -- returns B200ORB_EINVAL before anything is enqueued and before any handle
 * state changes. */
typedef struct {
  int nframes, rows, cols;
  int device;                   /* 1: every input below is an HBM pointer and the results stay in HBM
                                   (orbs_device_results); 0: host buffers, uploaded in chunks (orbs_set_chunk_frames) */
  const uint8_t* gray;          /* [n][rows][cols] u8 */
  const float* depth;           /* [n][rows][cols] f32 metres, or NULL when depth_u16 is given */
  /* The depth image as the sensor delivers it (CV_16U, e.g. TUM PNGs; host batches only).  The tracking path reads depth
   * only under the keypoints (Frame::ComputeStereoFromRGBD, src/Frame.cc:850-871): the device gathers those pixels and
   * converts them as imDepth.convertTo(CV_32F, mDepthMapFactor) of Tracking::GrabImageRGBD does (src/Tracking.cc:366-367;
   * float multiply by depth_factor = 1.0f / DepthMapFactor).  When depth_u16 is page-locked host memory (cudaHostAlloc /
   * cudaHostRegister) the pixels are read in place over PCIe and the depth images are not uploaded at all; pageable
   * depth is uploaded as CV_16U, half the host->device traffic of f32 depth. */
  const uint16_t* depth_u16;
  float depth_factor;
  const float* Tcw;             /* [n][16] */
  /* Masked batches: the `perfect` variant's live path per frame (perfect/src/Tracking.cc:703-719).  Between extraction
   * and the frame glue, one kernel per batch does Flow::ComputeMask after calcOpticalFlowFarneback (perfect/src/Flow.cc:
   * 14-53: pyrUp of the flow, mask = 0 where x*x + y*y >= max(binary_threshold, 40), erode, erode, dilate with the 21 x 21
   * ellipse) and the keypoint loop of the masked RGB-D Frame constructor (perfect/src/Frame.cc:328-427, :356-377: when the
   * mask's sum is above 65 % of the pixels, keypoints whose pixel is not 1 are dropped with their descriptors, order
   * kept).  Frame t is then tracked against the filtered frame t-1 with SearchByProjection(cur, last)
   * (perfect/src/Tracking.cc:1933), and orbs_read_dynamic_mask returns the mask FrameDrawer receives
   * (perfect/src/FrameDrawer.cc:262).
   * flow[n][rows/2][cols/2][2] f32 is what calcOpticalFlowFarneback returns for the pyrDown'ed previous and current gray
   * images (CV_32FC2, continuous); mask pixels beyond the 2 (rows/2) x 2 (cols/2) it covers stay 1.  A frame without a
   * previous image (the sequence's first) takes a zero flow field: its mask is all ones and it keeps every keypoint, the
   * reference's `mask = ones` case.  A host batch uploads it chunk by chunk next to the gray images.  The results keep the
   * layout of unmasked batches and describe the FILTERED frames (nkp, kps, desc, cur2last against frame t-1's filtered
   * keypoints), as do orbs_device_results and orbs_read_frame_glue.  A masked batch launches one kernel more than the
   * same unmasked batch; orbx_profile_read counts its time in stage 5.
   * Geometry (flow and device_flow): a frame's mask is held as two bit planes in one CTA's shared memory,
   * 8 * rows * ceil(cols / 32) + 132 bytes; on an H100 (232448 bytes per CTA) rows * ceil(cols / 32) <= 29039: 1280 x 720
   * and 1241 x 376 fit, 1280 x 725 is the largest 1280-wide image.  Larger images and flow fields under 2 x 2 return
   * B200ORB_EINVAL before anything is enqueued. */
  const float* flow;
  /* Masked host batches whose flow the device computes (perfect/src/Flow.cc:26-29, as dynm_flow_batch_device) from the
   * gray images the batch uploads anyway, in place of flow; nothing but prev_gray is uploaded beyond what the unmasked
   * batch uploads.  Sizes dynm_flow_batch_device rejects return B200ORB_EINVAL before anything is enqueued. */
  int device_flow;
  /* With device_flow: the rows x cols u8 frame before gray[0]; NULL: the sequence starts at gray[0], which takes the zero
   * field.  The predecessor is an argument rather than handle state, so two handles chained with orbs_chain_after can
   * carry one sequence: each batch passes the last gray frame of the batch before.  This repairs frame 0's flow only;
   * orbs_continue carries the whole last frame (its keypoints for frame 0's search as well as its image), and a
   * continued batch must leave prev_gray NULL. */
  const uint8_t* prev_gray;
  float binary_threshold;       /* masked batches: Flow::ComputeMask's threshold (raised to 40) */
  /* 1: the masked batch follows the reference's live path in full (perfect/src/Tracking.cc:703-719): before each frame's
   * ComputeMask, TrackHomo (:1331-1399) searches the UNFILTERED keypoints of frame t against the FILTERED keypoints of
   * frame t-1 (SearchByProjection(cur, last, th, mono = 0, points_last, points_current) of ORBmatcher(0.9, true), whatever
   * OrbsParams' nnratio and check_ori), retries at 2 th
   * below 20 matches, and with at least 20 matches and more than 50 pairs fits H = findHomography(points_current,
   * points_last, RANSAC, 3) as dynm_find_homography does; a found H makes the frame's mask ComputeMask(GrayImg, H)
   * (perfect/src/Flow.cc:73-80: the frame warped by H as dynm_warp_perspective does, then Farneback against the previous
   * half image), every other frame takes ComputeMask(GrayImg).  The previous half image is pyrDown of what the previous
   * frame's ComputeMask received: its warped image when it took the homography branch.  The sequence's frame 0 has no
   * last frame (zero field) and its frame 1 no velocity yet (mVelocity is first set by frame 1's Track): frames 0 and 1
   * of a batch that starts a sequence, and the frames of a continued batch (orbs_continue) at those sequence positions.
   * Poses: as the batch's motion-model search, TrackHomo projects frame t-1's points, unprojected from its filtered
   * keypoints under Tcw[t-1], with Tcw[t].  Everything runs on the device with no host round trip inside the batch;
   * orbs_read_homography reports each frame's branch.  Only the homography form above; a handle whose keypoint capacity
   * (orbx_max_keypoints_for) exceeds 8192, findHomography's pair limit, returns B200ORB_EINVAL.  The chain's
   * launches go to the stream as one CUDA graph, so orbs_submit does not wait here either.  0: none of this. */
  int homography;
} OrbsBatch;
/* Host results: kps[n][cap], desc[n][cap][32], nkp[n], cur2last[n][cap] (frame 0: all -1 unless the batch continues a
 * sequence, orbs_continue), nmatch[n]; cap below the keypoint capacity of the batch's image size
 * (orbx_max_keypoints_for) returns B200ORB_ECAP. */
typedef struct { OrbxKeyPoint* kps; uint8_t* desc; int32_t* nkp; int32_t* cur2last; int32_t* nmatch; int cap; } OrbsResults;
/* Tracks one batch; out is non-NULL exactly when !b->device.  Never waits: uploads, kernels and result downloads are
 * enqueued on the handle's streams (orbs_stream for the kernels) and the results are valid after orbs_sync(h); the
 * host buffers must stay untouched until then.  With page-locked host buffers the copies are plain DMA, and two
 * handles used alternately keep two batches in flight, so the upload of batch k+1 and the download of batch k-1 overlap
 * the kernels of batch k (what the reference's grab thread / tracking thread split does for one frame,
 * Examples/RGB-D/rgbd_tum.cc:88-109, done here for whole batches).
 * Only host batches take part in orbs_chain_after: a host batch consumes the dependency set on h and records the end
 * of its kernels for a handle chained after h.  A device batch neither waits for the dependency (it stays set for h's
 * next host batch) nor records.
 * Every refusal -- B200ORB_EINVAL for the forms, sizes and continuations described here and B200ORB_ECAP -- returns
 * before anything is enqueued and before any handle state changes; the last batch stays readable.  A submit that fails
 * after that point (an allocation, a launch) leaves h with no batch: orbs_device_results, the orbs_read_* entries and
 * orbs_continue(., h) return B200ORB_EINVAL until a batch succeeds. */
int orbs_submit(orbs_t* h, const OrbsBatch* b, const OrbsResults* out);
/* Pipelining aid for two handles used alternately: the next host batch submitted to h starts its kernels only when the
 * kernels of prev's last host batch are done; h's uploads and prev's downloads proceed meanwhile, so the stages
 * upload(k+1) | kernels(k) | download(k-1) overlap without two batches' kernels sharing the SMs.  The dependency is
 * consumed by h's next host batch; prev must stay alive until then. */
int orbs_chain_after(orbs_t* h, orbs_t* prev);
/* The next batch submitted to h continues the sequence whose last frame is the last frame of the last batch submitted
 * to prev (prev may be h).  That frame P, exactly as its batch left it (for masked and homography batches: the filtered
 * keypoints and descriptors, glued under P's own Tcw), becomes frame -1 of h's next batch:
 *   plain and caller-flow batches: frame 0 runs SearchByProjection(frame 0, P, th, mono = 0) with OrbsParams' nnratio
 *     and check_ori; cur2last[0] indexes P's keypoints and nmatch[0] is its match count;
 *   device_flow batches: frame 0's flow is Farneback(pyrDown(P's gray image), pyrDown(gray[0])), then the search above;
 *   homography batches: a frame at sequence position g (the frames before the batch plus its index in the batch) is
 *     ORBS_HOMO_NO_LAST only for g = 0 and ORBS_HOMO_NO_VELOCITY only for g = 1; every other frame, frame 0 included,
 *     takes the full TrackHomo step with P as frame 0's last frame, whose previous half image is pyrDown of what P's
 *     ComputeMask received (its warped image when P took the homography branch).
 * The orbs_read_* entries and orbs_device_results describe frame 0 of a continued batch like any other frame.
 * P's keypoint count, pose, glue, descriptors and (device_flow and homography batches) image are copied into h on prev's
 * stream, behind prev's last batch and before anything submitted to prev later; the copy first waits for h's batches that
 * still read an earlier copy, and h's next batch waits for it.  prev may be destroyed once this returns.  A device
 * batch's Tcw buffer must still hold its poses when its handle is continued.  Exactly one batch consumes the
 * continuation; the batch after it starts a new sequence unless orbs_continue is called again.
 * B200ORB_EINVAL, with nothing enqueued and both handles as they were: a NULL handle, a prev that holds no batch, or a
 * prev on another device.  orbs_submit then refuses with B200ORB_EINVAL, before anything is enqueued and with the
 * continuation still pending, a batch whose rows / cols, OrbsParams (all but max_frames) or keypoint capacity differ from
 * P's, a batch of another variant than P's (plain, caller flow, device_flow, homography; the depth kind and host / device
 * may differ within the forms OrbsBatch lists) and a batch with prev_gray.  Launches one kernel. */
int orbs_continue(orbs_t* h, orbs_t* prev);
/* Frames per upload chunk of host batches (default 128, at most 7 chunks per call): the extraction of a chunk
 * starts as soon as it has arrived while the next one is still crossing PCIe.  Gray images and any depth that is
 * uploaded go up chunk by chunk. */
int orbs_set_chunk_frames(orbs_t* h, int frames);
int orbs_device_results(orbs_t* h, const OrbxKeyPoint** d_kps, const uint8_t** d_desc, const int32_t** d_nkp,
                        const int32_t** d_cur2last, const int32_t** d_nmatch, int* cap);
/* Frame glue of frame `frame`, in [0, nframes) of the last batch: mvuRight / mvDepth (Frame::ComputeStereoFromRGBD,
 * src/Frame.cc:850-871), the world point Frame::UnprojectStereo gives per keypoint under that frame's pose (:879-899) and
 * whether the keypoint has depth; host arrays of at least the handle's keypoint capacity (NULL = skip). */
int orbs_read_frame_glue(orbs_t* h, int frame, float* uright, float* depth, float* xw, uint8_t* valid, int cap);
/* Frame `frame` of the last batch, which must have been masked: mask[rows][cols] 0 / 1 (the Flow::ComputeMask result,
 * FrameDrawer's mDynMask), *filtered = whether the 65 % rule dropped keypoints of this frame (NULL = skip either). */
int orbs_read_dynamic_mask(orbs_t* h, int frame, uint8_t* mask, int* filtered);
/* What TrackHomo did for frame `frame` of the last batch, which must have been a homography batch (synchronises): *branch
 * one of ORBS_HOMO_*, *nmatches the count of its final search (0 for frames 0 and 1), *npairs points_current.size() after
 * it, and H the model findHomography returned, row-major (zeros when there is none).  NULL = skip. */
#define ORBS_HOMO_NO_LAST 0         /* frame 0 of the batch: no last frame */
#define ORBS_HOMO_NO_VELOCITY 1     /* frame 1: no velocity yet */
#define ORBS_HOMO_FEW_MATCHES 2     /* fewer than 20 matches after the retry at 2 th */
#define ORBS_HOMO_FEW_PAIRS 3       /* at least 20 matches, at most 50 pairs */
#define ORBS_HOMO_NO_MODEL 4        /* findHomography found no model (empty H) */
#define ORBS_HOMO_WARPED 5          /* H found: the mask is that of the warped frame */
int orbs_read_homography(orbs_t* h, int frame, double H[9], int* branch, int* nmatches, int* npairs);
int orbs_sync(orbs_t* h);
void* orbs_stream(orbs_t* h);
long long orbs_launch_count(const orbs_t* h);
orbx_t* orbs_extractor(orbs_t* h);

/* ------------------------------------------------------------------------------------------------
 * Dense mapping -- PointCloudMapping (include/pointcloudmapping.h:50-56) with the OctoMap occupancy
 * semantics of perfect/src/MapDrawer.cc:51-56,610-675,946-1025 (SURVEY F3).
 * ------------------------------------------------------------------------------------------------ */
typedef struct ocm ocm_t;
typedef struct {
  double resolution;            /* octoMap.res, 0.05 (perfect/Examples/RGB-D/my_rgbd_ty_api_adj.yaml:82) */
  double prob_hit, prob_miss;   /* 0.7 / 0.4   (perfect/src/MapDrawer.cc:55-56) */
  double clamp_min, clamp_max;  /* 0.12 / 0.97 (perfect/src/MapDrawer.cc:53-54) */
  float depth_min, depth_max;   /* 0.5 / 3.0   (perfect/src/MapDrawer.cc:655) */
  float y_max;                  /* 3.0: keep |y| <= y_max (:660) */
  float leaf;                   /* 0.01 VoxelGrid leaf (:669); <=0 disables the pre-filter */
  int64_t map_capacity;         /* voxel hash capacity (slots); 0 = default */
} OcmParams;
void ocm_default_params(OcmParams* p);
int ocm_create(const OcmParams* p, int device, ocm_t** out);
void ocm_destroy(ocm_t* h);
/* One keyframe: MapDrawer::GeneratePointCloud (:641-675) + InsertScan (:946-1025) with a supplied
 * ground label per pixel (NULL = all non-ground, the reference's fallback when RANSAC finds no plane).
 * depth f32 metres, rgb u8 BGR-interleaved as cv::Mat (kf->mImRGB), Tcw row-major (KeyFrame::GetPose()). */
int ocm_insert_keyframe(ocm_t* h, const float* depth, const uint8_t* rgb, int rows, int cols,
                        const float Tcw[16], float fx, float fy, float cx, float cy,
                        const uint8_t* ground_label);
int ocm_insert_keyframe_device(ocm_t* h, const float* d_depth, const uint8_t* d_rgb, int rows, int cols,
                               const float Tcw[16], float fx, float fy, float cx, float cy,
                               const uint8_t* d_ground_label);
/* World-frame points of the LAST inserted keyframe after gating + leaf filter + transform (xyz f32 x n,
 * unordered: compare as sets). */
int ocm_last_points(ocm_t* h, float* xyz, uint8_t* rgb, int cap, int* n);
/* Leaf export: keys (3 x u16 per leaf, octomap OcTreeKey), log-odds f32; unordered. */
int64_t ocm_num_leaves(ocm_t* h);
int ocm_export_leaves(ocm_t* h, uint16_t* keys, float* logodds, uint8_t* rgb, int64_t cap, int64_t* n);
int ocm_query(ocm_t* h, const float xyz[3], float* logodds, int* found);
/* Batched variant for a resident RGB-D stream: inserts keyframes frame_idx[0..n) (in that order) of a batch laid out
 * as depth[F][rows][cols] f32, rgb[F][rows][cols][3] u8 in HBM, Tcw[n][16] on the host (one pose per inserted
 * keyframe); keyframe i reads depth image depth_idx[i] and colour image rgb_idx[i] (NULL = depth_idx) of the two
 * batches.  One call enqueues everything on the handle's stream (what UpdateOctomap's loop does,
 * perfect/src/MapDrawer.cc:610-638).  d_label[F][rows][cols] is a per-pixel ground label batch (NULL = all
 * non-ground); keyframe i reads label image label_idx[i] (NULL = depth_idx).  Labels stand in for the reference's
 * RANSAC floor split (perfect/src/MapDrawer.cc:686-774): ground points only clear space along their rays (:961-969). */
int ocm_insert_keyframes_labeled_device(ocm_t* h, const float* d_depth, const uint8_t* d_rgb, const uint8_t* d_label,
                                        int rows, int cols, const int32_t* depth_idx, const int32_t* rgb_idx,
                                        const int32_t* label_idx, int n, const float* Tcw, float fx, float fy, float cx,
                                        float cy);
/* Host-buffer form for a batch of keyframes as the reference's callers hold them: the sensor's CV_16U depth images
 * (imDepth before convertTo, src/Tracking.cc:353-367; depth_factor = 1.0f / DepthMapFactor) and the colour images
 * handed to insertKeyFrame (src/Tracking.cc:1889), depth_u16[n][rows][cols], rgb[n][rows][cols][3], Tcw[n][16], and
 * the ground labels label[n][rows][cols] (NULL = all non-ground).  Uploads, the conversion and the n inserts are
 * enqueued on the map's stream and the call returns; the host buffers (page-locked for a truly asynchronous upload)
 * must stay untouched until ocm_sync(h). */
int ocm_insert_keyframes_u16_labeled(ocm_t* h, const uint16_t* depth_u16, const uint8_t* rgb, const uint8_t* label, int rows,
                                     int cols, int n, float depth_factor, const float* Tcw, float fx, float fy, float cx,
                                     float cy);
/* ocm_merge_nccl (SURVEY §8(b),(e)): the one exchange step of the frame-sharded mode.  Every rank has inserted its own
 * keyframes (a contiguous range, rank order = keyframe order) since the last merge; the call all-gathers the per-voxel
 * clamp-add summaries of that epoch (24-byte records: key u64, a, lo, hi f32, colour u32) over NCCL / NVLink and replays
 * the shards of ALL ranks in rank order on the values of the last merge, so every rank ends with the map a single process
 * inserting all keyframes in order would hold (log-odds equal up to float re-association, << 1e-5).  One host
 * synchronisation (the counts); everything else is enqueued on the map's stream.  comm = ncclComm_t (NULL: single rank,
 * the call just closes the epoch); stream = a cudaStream_t the merge is ordered after / before (NULL: the map's own). */
typedef struct {
  int world, rank;
  int64_t records_sent, records_total;     /* voxels this rank sent / all ranks together */
  int64_t bytes_sent, bytes_received;      /* 24 B per record */
} OcmMergeStats;
int ocm_merge_nccl(ocm_t* h, void* nccl_comm, void* stream, OcmMergeStats* stats);
/* Helpers to obtain an ncclComm_t without linking NCCL: rank 0 calls ocm_nccl_unique_id and hands the 128 bytes to the
 * other ranks through whatever plumbing the host has (torch.distributed.broadcast in the Python mirror). */
int ocm_nccl_unique_id(uint8_t id[128]);
int ocm_nccl_comm_create(const uint8_t id[128], int rank, int world, int device, void** nccl_comm);
int ocm_nccl_comm_destroy(void* nccl_comm);
/* Counters for bench.py's B_map: points = P of the LAST round of keyframes (at most 32) a batch insert ran (points that
 * survived gates + leaf filter, summed over the round's keyframes); voxel_updates = CUMULATIVE number of (voxel, keyframe)
 * log-odds updates since the map was created (U summed over every keyframe so far). */
int ocm_last_batch_stats(ocm_t* h, int64_t* points, int64_t* voxel_updates);
/* The map as octomap's pruned ColorOcTree, and back (`.ot` files: what octovis reads, what MapDrawer saves and loads).
 *   ocm_tree_build   InsertScan's m_octree->prune() (perfect/src/MapDrawer.cc:1024) and the walk of the tree's write():
 *                    builds, in device memory of the handle, the pruned tree of the map as it stands after everything
 *                    enqueued so far -- the 8-byte nodes octomap writes, in pre-order (inner value = max child, inner
 *                    colour white, 8 equal childless children collapse into their parent, cascading) -- and its leaves.
 *                    The tree is a snapshot: the three readers below return the last build until the next one.
 *   ocm_write_ot     the file's bytes, header (`id ColorOcTree`, `size` = nodes, `res` as an ostream prints a double) and
 *                    nodes; buf == NULL: *n = size only.  An empty map writes the header with `size 0`.
 *   ocm_tree_leaves  the pruned leaves in file order: key of the min corner (3 x u16), depth (16 = one cell; a leaf of
 *                    depth d covers (2^(16-d))^3 cells), log-odds, colour -- the cells MapDrawer::DrawOctoMap walks
 *                    (:406-416).  Any output may be NULL; all NULL: *n only.
 *   ocm_save_ot      MapDrawer::SaveOctoMap (:1103-1111): ocm_tree_build + ocm_write_ot into `path`; *n_nodes (NULL = skip).
 *   ocm_read_ot      MapDrawer::LoadOctoMap (:1113-1117), from memory: REPLACES the map's contents by the file's leaves,
 *                    pruned leaves expanded to their depth-16 cells, inner nodes ignored.  Afterwards the handle is a map
 *                    that was just merged: inserts, ocm_merge_nccl, ocm_query and ocm_export_leaves continue from it.
 *                    Refused with the map untouched: an id other than ColorOcTree, a `res` other than the handle's,
 *                    a `size` that disagrees with the bytes or the child masks, a tree deeper than 16 (B200ORB_EINVAL);
 *                    more cells than the map's capacity (B200ORB_ECAP).
 *   ocm_load_ot      the same from a file.
 *   ocm_ot_leaves    the parser alone, on the host (no handle, no GPU): the leaves of `.ot` bytes in file order, as
 *                    ocm_tree_leaves returns them.  cap too small: B200ORB_ECAP, *n_out = leaves; nothing else written. */
int ocm_tree_build(ocm_t* h, int64_t* n_nodes, int64_t* n_leaves);
int ocm_write_ot(ocm_t* h, uint8_t* buf, int64_t cap, int64_t* n);
int ocm_tree_leaves(ocm_t* h, uint16_t* keys, uint8_t* depth, float* logodds, uint8_t* rgb, int64_t cap, int64_t* n);
int ocm_save_ot(ocm_t* h, const char* path, int64_t* n_nodes);
int ocm_read_ot(ocm_t* h, const uint8_t* bytes, int64_t n);
int ocm_load_ot(ocm_t* h, const char* path);
int ocm_ot_leaves(const uint8_t* bytes, int64_t n, double* res, uint16_t* keys, uint8_t* depth, float* logodds,
                  uint8_t* rgb, int64_t cap, int64_t* n_out);
int ocm_sync(ocm_t* h);
void* ocm_stream(ocm_t* h);
long long ocm_launch_count(const ocm_t* h);

/* ---------------------------------------------------------------------------------------------------------------------
 * T-variant dense map: the accumulated colour cloud of PointCloudMapping::viewer (src/pointcloudmapping.cc:395-500).
 *   gcm_add_keyframe[_device]  generatePointCloud (:131-194: every pixel, no depth gate, world frame through Tcw^-1 in
 *                              double) + removeNaNFromPointCloud + "*globalMap += *out_pt" (:482-485); depth f32 metres,
 *                              colour image BGR u8 [rows][cols][3]
 *   gcm_refilter               "voxel.setInputCloud(globalMap); voxel.filter(*tmp); globalMap->swap(*tmp)" (:490-493),
 *                              VoxelGrid leaf = the constructor's resolution (:40)
 *   gcm_export                 the points of globalMap (what viewer / global_color.pcd receive, :496-521), cell order
 * B200ORB_EGEOM from gcm_refilter: the cell index space overflows int for this leaf (PCL leaves the cloud unfiltered);
 * the map then keeps its finite points in insertion order, as the reference's globalMap, which never holds a NaN. */
typedef struct gcm gcm_t;
int gcm_create(float leaf, int device, gcm_t** out);
void gcm_destroy(gcm_t* h);
int gcm_add_keyframe(gcm_t* h, const float* depth, const uint8_t* bgr, int rows, int cols, const float Tcw[16], float fx,
                     float fy, float cx, float cy);
int gcm_add_keyframe_device(gcm_t* h, const float* d_depth, const uint8_t* d_bgr, int rows, int cols, const float Tcw[16],
                            float fx, float fy, float cx, float cy);
int gcm_refilter(gcm_t* h);
long long gcm_size(const gcm_t* h);
int gcm_export(gcm_t* h, float* xyz, uint8_t* rgb, long long cap, long long* n);
int gcm_sync(gcm_t* h);
long long gcm_launch_count(const gcm_t* h);

/* Semantic object clusters of the same loop (src/pointcloudmapping.cc:399-488).  The ncnn SSD detector stays outside:
 * the caller passes its boxes (src/ncnn_dect.h:12-18, detector order).  For keyframe number `keyframe_index` (the `i`
 * of :399, counted from 0 over every keyframe the map has been given):
 *   - a box is used iff (double)prob > 0.54 (:418), else its record is GCM_BELOW_PROB;
 *   - draw_rect_with_depth_threshold (:197-244, :426): the box's mean depth over its 30-70 % window, and its band
 *     (|depth - mean| < 0.4) inside the rectangle shifted one row up and one column left; band pixels are painted in
 *     colors_[class_id] (:47-60, B,G,R), a later box over an earlier one.  Flat indices wrap into the next row and
 *     repeat, as the reference's do.  Deviation: indices outside [0, rows*cols) are skipped (the reference reads and
 *     writes out of bounds there: boxes at x < 1 or y < 1 or past the bottom edge);
 *   - "if((i%2==0)&&(objects.size()==0)) continue;" (:434): an even keyframe with n_objs == 0 adds nothing;
 *   - otherwise generatePointCloud on the PAINTED image is appended to globalMap exactly as gcm_add_keyframe does
 *     (:439, :482-485), and every used box gets ExtractIndices on its band, StatisticalOutlierRemoval (mean_k 50,
 *     stddev_mul 1.0, :75-76), VoxelGrid(resolution), compute3DCentroid and getMinMax3D (:443-476) -> GCM_CLUSTER.
 *     Deviation: a box with fewer than 51 band points gets GCM_FEW_POINTS and no cluster (PCL's filter reads past the
 *     neighbour list it gets back there, and an empty box leaves the centroid uninitialised).
 * clusters_out has n_objs records, one per box in order.  sem_merge (:246-322) stays with the caller, over the records
 * and the detector's object names.  B200ORB_EINVAL for a class_id outside [0, 21) (the 21-entry colors_ / obj_size_
 * tables, :50-70) or a non-finite rectangle or one beyond 2^24 px; B200ORB_ECAP when the boxes span more than 2^31 - 1
 * band positions.  Synchronous like gcm_add_keyframe; the _device twin reads depth / colour from device memory, while
 * objs and clusters_out stay on the host. */
typedef struct GcmObject {
  float x, y, width, height; /* cv::Rect_<float> */
  int32_t class_id;
  float prob;
} GcmObject;
#define GCM_CLUSTER 0    /* a cluster: every field below is set */
#define GCM_BELOW_PROB 1 /* prob <= 0.54: the box is not used (n_* are 0) */
#define GCM_FEW_POINTS 2 /* fewer than 51 band points: n_band is set, no cluster */
typedef struct GcmCluster {
  int32_t status;
  int32_t n_band;    /* band indices (with repeats) = points ExtractIndices hands on */
  int32_t n_inliers; /* after StatisticalOutlierRemoval */
  int32_t n_voxels;  /* after VoxelGrid (= n_inliers where its index space overflows int: PCL returns the input) */
  float centroid[3], min_pt[3], max_pt[3];
} GcmCluster;
int gcm_add_keyframe_objects(gcm_t* h, const float* depth, const uint8_t* bgr, int rows, int cols, const float Tcw[16],
                             float fx, float fy, float cx, float cy, long long keyframe_index, const GcmObject* objs,
                             int n_objs, GcmCluster* clusters_out);
int gcm_add_keyframe_objects_device(gcm_t* h, const float* d_depth, const uint8_t* d_bgr, int rows, int cols,
                                    const float Tcw[16], float fx, float fy, float cx, float cy, long long keyframe_index,
                                    const GcmObject* objs, int n_objs, GcmCluster* clusters_out);

#ifdef __cplusplus
}
#endif
#endif /* B200ORB_H_ */
