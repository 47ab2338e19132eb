"""Host-side mirror of ORB_SLAM2::ORBmatcher (reference include/ORBmatcher.h:37-118) over the C-ABI.

The reference's methods walk Frame/KeyFrame/MapPoint objects and mutate them; here the same searches take the
flat views the C++ shim builds (FrameView / LastView of _abi.py) and return the index vectors the shim turns
back into pointer assignments.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._abi import BowView, FrameView, LastView, QueriesView, TrackPointsView, TriKFView, ptr  # noqa: F401


class ORBmatcher:
    TH_LOW = 50       # src/ORBmatcher.cc:40
    TH_HIGH = 100     # :39
    HISTO_LENGTH = 30  # :41

    def __init__(self, nnratio: float = 0.6, checkOri: bool = True, device: int = 0):
        self.mfNNratio = float(nnratio)
        self.mbCheckOrientation = bool(checkOri)
        self._L = _lib.lib()
        self._h = C.c_void_p()
        _lib.check(self._L.orbm_create(int(device), C.byref(self._h)))

    def __del__(self):
        try:
            if self._h:
                self._L.orbm_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    @staticmethod
    def DescriptorDistance(a: np.ndarray, b: np.ndarray) -> int:
        a = np.ascontiguousarray(a, np.uint8)
        b = np.ascontiguousarray(b, np.uint8)
        assert a.size == 32 and b.size == 32
        return int(_lib.lib().orbm_hamming(ptr(a), ptr(b)))

    def SearchByProjection(self, F: FrameView, other, th: float, bMono: bool = False):
        """Overloads of the reference:
          (Frame&, const Frame& LastFrame, th, bMono)      src/ORBmatcher.cc:1578-1724  -> other is a LastView
          (Frame&, const vector<MapPoint*>&, th)            src/ORBmatcher.cc:63-156     -> other is a TrackPointsView
        Returns (nmatches, index vector): entry j = index of the LastFrame keypoint / MapPoint now held by
        F.mvpMapPoints[j] (-1 NULL, -2 untouched pre-existing entry)."""
        out = np.full(F.n, -1, np.int32)
        nm = C.c_int(0)
        fs, os_ = F.struct(), other.struct()
        if isinstance(other, LastView):
            _lib.check(self._L.orbm_search_by_projection_last(self._h, C.byref(fs), C.byref(os_), float(th), int(bMono),
                                                              self.mfNNratio, int(self.mbCheckOrientation), ptr(out),
                                                              C.byref(nm)))
        elif isinstance(other, TrackPointsView):
            _lib.check(self._L.orbm_search_by_projection_points(self._h, C.byref(fs), C.byref(os_), float(th),
                                                                self.mfNNratio, ptr(out), C.byref(nm)))
        else:
            raise TypeError("SearchByProjection: second argument must be a LastView or a TrackPointsView")
        return nm.value, out

    def SearchByProjectionPairs(self, F: FrameView, last: LastView, th: float, bMono: bool = False):
        """The perfect tree's (Frame&, const Frame& LastFrame, th, bMono, points_last, points_current)
        (perfect/src/ORBmatcher.cc:1727-1880) -> (nmatches, cur2last, pairs).  nmatches and cur2last are those of
        SearchByProjection(F, last, th, bMono); pairs is a k x 2 int32 array of (i, j): last keypoint i accepted current
        keypoint j, in ascending i, taken before the rotation prune.  The reference pushes
        (LastFrame.mvKeys[i].pt, CurrentFrame.mvKeys[j].pt) for each row: the distorted keypoints."""
        out = np.full(F.n, -1, np.int32)
        acc = np.full(max(last.n, 1), -1, np.int32)
        nm = C.c_int(0)
        fs, ls = F.struct(), last.struct()
        _lib.check(self._L.orbm_search_by_projection_last_pairs(self._h, C.byref(fs), C.byref(ls), float(th), int(bMono),
                                                                self.mfNNratio, int(self.mbCheckOrientation), ptr(out),
                                                                ptr(acc), C.byref(nm)))
        i = np.flatnonzero(acc[:last.n] >= 0).astype(np.int32)
        return nm.value, out, np.stack([i, acc[i]], axis=1).reshape(-1, 2)

    def SearchProjected(self, F: FrameView, queries: QueriesView, max_dist: int, claim_rule: int = 1):
        """Shared tail of the projection overloads whose geometry the caller computes (relocalisation
        src/ORBmatcher.cc:1757-1899 -> claim_rule 1, max_dist = ORBdist; see include/b200orb.h)."""
        out = np.full(F.n, -1, np.int32)
        nm = C.c_int(0)
        fs, qs = F.struct(), queries.struct()
        _lib.check(self._L.orbm_search_projected(self._h, C.byref(fs), C.byref(qs), int(max_dist), int(claim_rule),
                                                 int(self.mbCheckOrientation), ptr(out), C.byref(nm)))
        return nm.value, out

    def SearchByBoW(self, pKF: BowView, F: BowView):
        """SearchByBoW(KeyFrame*, Frame&, vector<MapPoint*>&) (src/ORBmatcher.cc:217-363) -> (nmatches, f2kf) with
        f2kf[j] = keyframe keypoint whose MapPoint lands in vpMapPointMatches[j], or -1."""
        out = np.full(F.n, -1, np.int32)
        nm = C.c_int(0)
        ks, fs = pKF.struct(), F.struct()
        _lib.check(self._L.orbm_search_by_bow(self._h, C.byref(ks), C.byref(fs), self.mfNNratio,
                                              int(self.mbCheckOrientation), ptr(out), C.byref(nm)))
        return nm.value, out

    def SearchByBoWKF(self, pKF1: BowView, pKF2: BowView):
        """SearchByBoW(KeyFrame*, KeyFrame*, vpMatches12) (src/ORBmatcher.cc:665-812) -> (nmatches, matches12) with
        matches12[i] = pKF2 keypoint matched to pKF1 keypoint i, or -1."""
        out = np.full(pKF1.n, -1, np.int32)
        nm = C.c_int(0)
        a, b = pKF1.struct(), pKF2.struct()
        _lib.check(self._L.orbm_search_by_bow_kf(self._h, C.byref(a), C.byref(b), self.mfNNratio,
                                                 int(self.mbCheckOrientation), ptr(out), C.byref(nm)))
        return nm.value, out

    def SearchBest(self, KF: FrameView, queries: QueriesView, gate: int = 0, inv_level_sigma2=None):
        """Per-query best keypoint of a keyframe, no claim state: the device part of both Fuse overloads (gate 1 / 0,
        src/ORBmatcher.cc:1031-1182, 1198-1318) and of SearchBySim3 (:1334-1558) -> (best_idx, best_dist)."""
        bi = np.full(max(queries.n, 1), -1, np.int32)
        bd = np.full(max(queries.n, 1), 2 ** 31 - 1, np.int32)
        ks, qs = KF.struct(), queries.struct()
        is2 = None if inv_level_sigma2 is None else np.ascontiguousarray(inv_level_sigma2, np.float32)
        _lib.check(self._L.orbm_search_best(self._h, C.byref(ks), C.byref(qs), int(gate), ptr(is2), ptr(bi), ptr(bd)))
        return bi[:queries.n], bd[:queries.n]

    def SearchForInitialization(self, F1: FrameView, F2: FrameView, vbPrevMatched, windowSize: int = 10):
        """src/ORBmatcher.cc:523-651 -> (nmatches, vnMatches12, updated vbPrevMatched)."""
        prev = np.ascontiguousarray(vbPrevMatched, np.float32).reshape(-1, 2).copy()
        out = np.full(max(F1.n, 1), -1, np.int32)
        nm = C.c_int(0)
        a, b = F1.struct(), F2.struct()
        _lib.check(self._L.orbm_search_for_initialization(self._h, C.byref(a), C.byref(b), ptr(prev), int(windowSize),
                                                          self.mfNNratio, int(self.mbCheckOrientation), ptr(out), C.byref(nm)))
        return nm.value, out[:F1.n], prev

    def SearchForTriangulation(self, pKF1: TriKFView, pKF2: TriKFView, F12, epipole, scale_factors2, level_sigma2_2,
                               bOnlyStereo: bool = False):
        """src/ORBmatcher.cc:827-1019 -> (nmatches, matches12); epipole = (ex, ey) of :835-839."""
        F = np.ascontiguousarray(F12, np.float32).reshape(9)
        sf = np.ascontiguousarray(scale_factors2, np.float32)
        s2 = np.ascontiguousarray(level_sigma2_2, np.float32)
        out = np.full(max(pKF1.n, 1), -1, np.int32)
        nm = C.c_int(0)
        a, b = pKF1.struct(), pKF2.struct()
        _lib.check(self._L.orbm_search_for_triangulation(self._h, C.byref(a), C.byref(b), ptr(F), float(epipole[0]),
                                                         float(epipole[1]), ptr(sf), ptr(s2), len(sf), int(bOnlyStereo),
                                                         int(self.mbCheckOrientation), ptr(out), C.byref(nm)))
        return nm.value, out[:pKF1.n]

    def IsInFrustum(self, F: FrameView, xw, normal, min_dist, max_dist, viewingCosLimit: float, log_scale_factor: float):
        """Frame::isInFrustum (src/Frame.cc:387-451) for n MapPoints -> a TrackPointsView-ready tuple
        (in_view, proj_x, proj_y, proj_xr, scale_level, view_cos)."""
        from ._abi import OrbmFrustumPoints
        xw = np.ascontiguousarray(xw, np.float32).reshape(-1, 3)
        nr = np.ascontiguousarray(normal, np.float32).reshape(-1, 3)
        mn, mx = np.ascontiguousarray(min_dist, np.float32), np.ascontiguousarray(max_dist, np.float32)
        n = len(xw)
        p = OrbmFrustumPoints(n, ptr(xw), ptr(nr), ptr(mn), ptr(mx))
        iv = np.zeros(max(n, 1), np.uint8)
        px, py, pxr, vc = [np.zeros(max(n, 1), np.float32) for _ in range(4)]
        lvl = np.zeros(max(n, 1), np.int32)
        fs = F.struct()
        _lib.check(self._L.orbm_is_in_frustum(self._h, C.byref(fs), C.byref(p), float(viewingCosLimit), float(log_scale_factor),
                                              ptr(iv), ptr(px), ptr(py), ptr(pxr), ptr(lvl), ptr(vc)))
        return iv[:n], px[:n], py[:n], pxr[:n], lvl[:n], vc[:n]

    def UndistortKeyPoints(self, xy, K, dist):
        """Frame::UndistortKeyPoints (src/Frame.cc:559-590) on n x 2 keypoint positions."""
        xy = np.ascontiguousarray(xy, np.float32).reshape(-1, 2)
        K = np.ascontiguousarray(K, np.float32).reshape(9)
        d = np.ascontiguousarray(dist, np.float32)
        out = np.zeros_like(xy)
        _lib.check(self._L.orbm_undistort_keypoints(self._h, ptr(xy), len(xy), ptr(K), ptr(d), len(d), ptr(out)))
        return out

    def launch_count(self) -> int:
        return int(self._L.orbm_launch_count(self._h))
