"""Restatement of a homography batch (OrbsBatch.homography = 1): the perfect variant's live path frame after frame
(perfect/src/Tracking.cc:703-719) on the batch's model of poses and depth.  TEST INFRASTRUCTURE ONLY.

It composes the pinned restatements of each stage:
  extraction, frame glue, SearchByProjection(cur, last)   oracle/ref.py (RefExtractor, stereo_unproject through
                                                          tests/helpers.frame_views, search_by_projection_last)
  TrackHomo's point-pair search                            oracle/homo_ref.py
  findHomography(points_current, points_last, RANSAC, 3)   tests/homography_lm.find_homography
  warpPerspective                                          oracle/homography_py.warp_perspective
  pyrDown + calcOpticalFlowFarneback                       oracle/farneback_py
  ComputeMask after the flow, the masked constructor       oracle/dynmask_py
with the control flow of Tracking::TrackHomo and Flow::ComputeMask, cited line by line below.  The 20 / 50 thresholds
and the warped previous half image come from perfect/src/Tracking.cc, which the oracle cannot build: restated, not
pinned."""
from __future__ import annotations

import numpy as np

from oracle import dynmask_py, farneback_py, homo_ref, homography_py, ref
from tests import homography_lm
from tests.helpers import frame_views

NO_LAST, NO_VELOCITY, FEW_MATCHES, FEW_PAIRS, NO_MODEL, WARPED = range(6)
NNRATIO = 0.9   # ORBmatcher matcher(0.9, true), perfect/src/Tracking.cc:1345


def track_homo(cur, last, cur_kxy, last_kxy, th):
    """TrackHomo's searches (perfect/src/Tracking.cc:1355-1372) -> (nmatches, cur2last, points_last, points_current,
    retried).  The vectors start empty; below 20 matches they are cleared and the search runs again at 2 th."""
    nm, c2l, acc = homo_ref.search_by_projection_last_pairs(cur, last, th, False, NNRATIO, True)   # :1355-1356
    retried = nm < 20                                                                                # :1359
    if retried:                                                                                      # :1361-1365
        nm, c2l, acc = homo_ref.search_by_projection_last_pairs(cur, last, 2 * th, False, NNRATIO, True)
    i = np.flatnonzero(acc >= 0)   # one pair per accepted query, in query order (perfect/src/ORBmatcher.cc:1835-1836)
    return nm, c2l, last_kxy[i].astype(np.float32), cur_kxy[acc[i]].astype(np.float32), retried


def _xy(K):
    return np.stack([K["x"], K["y"]], 1).astype(np.float32)


def run(gray, depth, T, nfeatures, th=15.0, binary_threshold=40.0):
    """gray [F][rows][cols] u8, depth [F][rows][cols] f32 metres (the CV_16U image times its factor), T [F][4][4] ->
    per frame dict: branch, nmatches, npairs, retried, H (9 doubles, zeros without a model), mask, filtered, kps, desc,
    nm, c2l (what the batch's motion-model search gives the filtered frame)."""
    F, rows, cols = gray.shape
    R = ref.RefExtractor(nfeatures, 1.2, 8, 20, 7)
    h2, w2 = rows // 2, cols // 2
    out, filt = [], []
    last_half = None
    for t in range(F):
        K, D = R(gray[t])
        rec = dict(branch=NO_LAST if t == 0 else NO_VELOCITY, nmatches=0, npairs=0, retried=False, H=np.zeros(9))
        dest = gray[t]
        if t >= 2:   # TrackHomo needs mState == OK and a velocity: set by frame 1's Track (perfect/src/Tracking.cc:1346)
            Kl, Dl = filt[t - 1]
            cur, last = frame_views(ref, K, D, depth[t], T[t], Kl, Dl, depth[t - 1], T[t - 1], R.mvScaleFactor,
                                    rows=rows, cols=cols)
            nm, _, pl, pc, retried = track_homo(cur, last, _xy(K), _xy(Kl), th)
            rec.update(nmatches=nm, npairs=len(pc), retried=retried)
            if nm < 20:                                        # :1374-1380
                rec["branch"] = FEW_MATCHES
            elif len(pc) <= 50:                                # :1381, then :1393-1398
                rec["branch"] = FEW_PAIRS
            else:
                H, _ = homography_lm.find_homography(pc, pl)   # :1386, points_last = H * points_current
                if H is None:                                  # `flag && !homo.empty()` (:713)
                    rec["branch"] = NO_MODEL
                else:
                    rec.update(branch=WARPED, H=np.asarray(H, np.float64).reshape(9))
                    dest = homography_py.warp_perspective(gray[t], H)   # perfect/src/Flow.cc:78
        # ComputeMask(dest) (perfect/src/Flow.cc:25-50): pyrDown, Farneback against mImGrayLast, then the swap that keeps
        # this frame's (possibly warped) half image for the next frame
        cur_half = farneback_py.pyr_down(dest, h2, w2)
        if last_half is None:
            flow = np.zeros((h2, w2, 2), np.float32)           # mask = ones
        else:
            flow = farneback_py.farneback(last_half, cur_half)
        last_half = cur_half
        mask = dynmask_py.mask_from_flow(flow, binary_threshold, (rows, cols))
        Kf, Df = dynmask_py.filter_keypoints(mask, K, D)
        filt.append((Kf, Df))
        rec.update(mask=mask, filtered=float(mask.sum()) > rows * cols * 0.65, kps=Kf, desc=Df)
        if t == 0:
            rec.update(nm=0, c2l=np.full(len(Kf), -1, np.int32))
        else:   # TrackWithMotionModel's search of the filtered frames, as the batch's run() does
            cur, last = frame_views(ref, Kf, Df, depth[t], T[t], filt[t - 1][0], filt[t - 1][1], depth[t - 1], T[t - 1],
                                    R.mvScaleFactor, rows=rows, cols=cols)
            nm, c2l = ref.search_by_projection_last(cur, last, th, False, NNRATIO, True)
            rec.update(nm=int(nm), c2l=np.asarray(c2l, np.int32))
        out.append(rec)
    return out
