"""ctypes mirrors of the structs declared in include/b200orb.h (no library loading here)."""
from __future__ import annotations

import ctypes as C

import numpy as np

vp = C.c_void_p


class OrbxParams(C.Structure):
    _fields_ = [("nfeatures", C.c_int), ("scale_factor", C.c_float), ("nlevels", C.c_int),
                ("ini_th_fast", C.c_int), ("min_th_fast", C.c_int)]


class OrbmFrame(C.Structure):
    _fields_ = [("n", C.c_int), ("x", vp), ("y", vp), ("octave", vp), ("angle", vp), ("uright", vp), ("desc", vp),
                ("mp_obs", vp), ("Tcw", C.c_float * 16),
                ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("bf", C.c_float),
                ("b", C.c_float),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("scale_factors", vp), ("nlevels", C.c_int)]


class OrbmLast(C.Structure):
    _fields_ = [("n", C.c_int), ("xw", vp), ("valid", vp), ("octave", vp), ("angle", vp), ("mp_desc", vp),
                ("mp_obs", vp), ("Tcw", C.c_float * 16)]


class OrbmTrackPoints(C.Structure):
    _fields_ = [("n", C.c_int), ("track_in_view", vp), ("proj_x", vp), ("proj_y", vp), ("proj_xr", vp),
                ("scale_level", vp), ("view_cos", vp), ("mp_desc", vp), ("mp_obs", vp)]


class OrbmQueries(C.Structure):
    _fields_ = [("n", C.c_int), ("valid", vp), ("u", vp), ("v", vp), ("radius", vp), ("min_level", vp), ("max_level", vp),
                ("uright", vp), ("desc", vp), ("angle", vp), ("obs", vp)]


class OrbmBow(C.Structure):
    _fields_ = [("n", C.c_int), ("desc", vp), ("angle", vp), ("valid", vp), ("n_nodes", C.c_int), ("node_ids", vp),
                ("node_off", vp), ("idx", vp)]


class OrbsParams(C.Structure):
    _fields_ = [("orb", OrbxParams), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
                ("bf", C.c_float), ("th", C.c_float), ("nnratio", C.c_float), ("check_ori", C.c_int),
                ("max_frames", C.c_int)]


class OrbsBatch(C.Structure):
    _fields_ = [("nframes", C.c_int), ("rows", C.c_int), ("cols", C.c_int), ("device", C.c_int), ("gray", vp),
                ("depth", vp), ("depth_u16", vp), ("depth_factor", C.c_float), ("Tcw", vp), ("flow", vp),
                ("device_flow", C.c_int), ("prev_gray", vp), ("binary_threshold", C.c_float), ("homography", C.c_int)]


class OrbsResults(C.Structure):
    _fields_ = [("kps", vp), ("desc", vp), ("nkp", vp), ("cur2last", vp), ("nmatch", vp), ("cap", C.c_int)]


class OcmParams(C.Structure):
    _fields_ = [("resolution", C.c_double), ("prob_hit", C.c_double), ("prob_miss", C.c_double),
                ("clamp_min", C.c_double), ("clamp_max", C.c_double), ("depth_min", C.c_float),
                ("depth_max", C.c_float), ("y_max", C.c_float), ("leaf", C.c_float), ("map_capacity", C.c_int64)]


def ptr(a):
    """numpy array (or None) -> void*; keeps no reference: callers hold the arrays alive."""
    if a is None:
        return None
    return a.ctypes.data_as(vp)


class FrameView:
    """Flat view of a Frame for the matcher (what the C++ shim extracts from ORB_SLAM2::Frame)."""

    def __init__(self, x, y, octave, angle, uright, desc, Tcw, fx, fy, cx, cy, bf, min_x, max_x, min_y, max_y,
                 scale_factors, mp_obs=None):
        f32, i32 = np.float32, np.int32
        self.x = np.ascontiguousarray(x, f32)
        self.y = np.ascontiguousarray(y, f32)
        self.octave = np.ascontiguousarray(octave, i32)
        self.angle = np.ascontiguousarray(angle, f32)
        self.uright = np.ascontiguousarray(uright, f32)
        self.desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        self.mp_obs = None if mp_obs is None else np.ascontiguousarray(mp_obs, i32)
        self.Tcw = np.ascontiguousarray(Tcw, f32).reshape(16)
        self.scale_factors = np.ascontiguousarray(scale_factors, f32)
        self.cam = (float(fx), float(fy), float(cx), float(cy), float(bf))
        self.bounds = (float(min_x), float(max_x), float(min_y), float(max_y))
        self.n = len(self.x)

    def struct(self) -> OrbmFrame:
        s = OrbmFrame()
        s.n = self.n
        s.x, s.y, s.octave, s.angle = ptr(self.x), ptr(self.y), ptr(self.octave), ptr(self.angle)
        s.uright, s.desc, s.mp_obs = ptr(self.uright), ptr(self.desc), ptr(self.mp_obs)
        s.Tcw = (C.c_float * 16)(*self.Tcw.tolist())
        s.fx, s.fy, s.cx, s.cy, s.bf = self.cam
        s.b = np.float32(np.float32(self.cam[4]) / np.float32(self.cam[0]))   # mb = mbf/fx (src/Frame.cc:218)
        s.min_x, s.max_x, s.min_y, s.max_y = self.bounds
        s.scale_factors = ptr(self.scale_factors)
        s.nlevels = len(self.scale_factors)
        return s


class LastView:
    """LastFrame side of SearchByProjection(CurrentFrame, LastFrame)."""

    def __init__(self, xw, valid, octave, angle, mp_desc, Tcw, mp_obs=None):
        self.xw = np.ascontiguousarray(xw, np.float32).reshape(-1, 3)
        self.valid = np.ascontiguousarray(valid, np.uint8)
        self.octave = np.ascontiguousarray(octave, np.int32)
        self.angle = np.ascontiguousarray(angle, np.float32)
        self.mp_desc = np.ascontiguousarray(mp_desc, np.uint8).reshape(-1, 32)
        self.mp_obs = None if mp_obs is None else np.ascontiguousarray(mp_obs, np.int32)
        self.Tcw = np.ascontiguousarray(Tcw, np.float32).reshape(16)
        self.n = len(self.valid)

    def struct(self) -> OrbmLast:
        s = OrbmLast()
        s.n = self.n
        s.xw, s.valid, s.octave, s.angle = ptr(self.xw), ptr(self.valid), ptr(self.octave), ptr(self.angle)
        s.mp_desc, s.mp_obs = ptr(self.mp_desc), ptr(self.mp_obs)
        s.Tcw = (C.c_float * 16)(*self.Tcw.tolist())
        return s


class TrackPointsView:
    """Local-map MapPoints as Frame::isInFrustum leaves them (src/Frame.cc:387-451)."""

    def __init__(self, track_in_view, proj_x, proj_y, proj_xr, scale_level, view_cos, mp_desc, mp_obs=None):
        self.track_in_view = np.ascontiguousarray(track_in_view, np.uint8)
        self.proj_x = np.ascontiguousarray(proj_x, np.float32)
        self.proj_y = np.ascontiguousarray(proj_y, np.float32)
        self.proj_xr = np.ascontiguousarray(proj_xr, np.float32)
        self.scale_level = np.ascontiguousarray(scale_level, np.int32)
        self.view_cos = np.ascontiguousarray(view_cos, np.float32)
        self.mp_desc = np.ascontiguousarray(mp_desc, np.uint8).reshape(-1, 32)
        self.mp_obs = None if mp_obs is None else np.ascontiguousarray(mp_obs, np.int32)
        self.n = len(self.track_in_view)

    def struct(self) -> OrbmTrackPoints:
        s = OrbmTrackPoints()
        s.n = self.n
        s.track_in_view, s.proj_x, s.proj_y, s.proj_xr = ptr(self.track_in_view), ptr(self.proj_x), ptr(self.proj_y), ptr(self.proj_xr)
        s.scale_level, s.view_cos, s.mp_desc, s.mp_obs = ptr(self.scale_level), ptr(self.view_cos), ptr(self.mp_desc), ptr(self.mp_obs)
        return s


class BowView:
    """One side of SearchByBoW: descriptors + angles + the DBoW2::FeatureVector flattened (node ids ascending)."""

    def __init__(self, desc, angle, feat_vec: dict, valid=None):
        self.desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        self.angle = np.ascontiguousarray(angle, np.float32)
        self.valid = None if valid is None else np.ascontiguousarray(valid, np.uint8)
        ids = sorted(feat_vec.keys())
        self.node_ids = np.array(ids, np.uint32)
        off = [0]
        idx = []
        for k in ids:
            idx.extend(int(v) for v in feat_vec[k])
            off.append(len(idx))
        self.node_off = np.array(off, np.int32)
        self.idx = np.array(idx if idx else [0], np.uint32)
        self.n = len(self.desc)

    def struct(self) -> OrbmBow:
        s = OrbmBow()
        s.n = self.n
        s.desc, s.angle, s.valid = ptr(self.desc), ptr(self.angle), ptr(self.valid)
        s.n_nodes = len(self.node_ids)
        s.node_ids, s.node_off, s.idx = ptr(self.node_ids), ptr(self.node_off), ptr(self.idx)
        return s


class QueriesView:
    """Pre-projected MapPoints for the generic guided search (orbm_search_projected)."""

    def __init__(self, valid, u, v, radius, min_level, max_level, desc, angle, uright=None, obs=None):
        self.valid = np.ascontiguousarray(valid, np.uint8)
        self.u = np.ascontiguousarray(u, np.float32)
        self.v = np.ascontiguousarray(v, np.float32)
        self.radius = np.ascontiguousarray(radius, np.float32)
        self.min_level = np.ascontiguousarray(min_level, np.int32)
        self.max_level = np.ascontiguousarray(max_level, np.int32)
        self.desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        self.angle = np.ascontiguousarray(angle, np.float32)
        self.uright = None if uright is None else np.ascontiguousarray(uright, np.float32)
        self.obs = None if obs is None else np.ascontiguousarray(obs, np.int32)
        self.n = len(self.valid)

    def struct(self) -> OrbmQueries:
        s = OrbmQueries()
        s.n = self.n
        s.valid, s.u, s.v, s.radius = ptr(self.valid), ptr(self.u), ptr(self.v), ptr(self.radius)
        s.min_level, s.max_level, s.uright = ptr(self.min_level), ptr(self.max_level), ptr(self.uright)
        s.desc, s.angle, s.obs = ptr(self.desc), ptr(self.angle), ptr(self.obs)
        return s


class OcmMergeStats(C.Structure):
    _fields_ = [("world", C.c_int), ("rank", C.c_int), ("records_sent", C.c_int64), ("records_total", C.c_int64),
                ("bytes_sent", C.c_int64), ("bytes_received", C.c_int64)]


class OrbmTriKF(C.Structure):
    _fields_ = [("n", C.c_int), ("desc", vp), ("x", vp), ("y", vp), ("angle", vp), ("uright", vp), ("octave", vp), ("has_mp", vp),
                ("n_nodes", C.c_int), ("node_ids", vp), ("node_off", vp), ("idx", vp)]


class TriKFView:
    """A keyframe as SearchForTriangulation reads it: undistorted keypoints, right coordinates, MapPoint occupancy and
    the DBoW2::FeatureVector flattened (node ids ascending)."""

    def __init__(self, x, y, octave, angle, uright, desc, has_mp, feat_vec: dict):
        self.x = np.ascontiguousarray(x, np.float32)
        self.y = np.ascontiguousarray(y, np.float32)
        self.octave = np.ascontiguousarray(octave, np.int32)
        self.angle = np.ascontiguousarray(angle, np.float32)
        self.uright = np.ascontiguousarray(uright, np.float32)
        self.desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        self.has_mp = np.ascontiguousarray(has_mp, np.uint8)
        ids = sorted(feat_vec.keys())
        self.node_ids = np.array(ids if ids else [0], np.uint32)
        off, idx = [0], []
        for k in ids:
            idx.extend(int(v) for v in feat_vec[k])
            off.append(len(idx))
        self.node_off = np.array(off, np.int32)
        self.idx = np.array(idx if idx else [0], np.uint32)
        self.n_nodes = len(ids)
        self.n = len(self.x)

    def struct(self) -> OrbmTriKF:
        s = OrbmTriKF()
        s.n = self.n
        s.desc, s.x, s.y, s.angle, s.uright = ptr(self.desc), ptr(self.x), ptr(self.y), ptr(self.angle), ptr(self.uright)
        s.octave, s.has_mp = ptr(self.octave), ptr(self.has_mp)
        s.n_nodes = self.n_nodes
        s.node_ids, s.node_off, s.idx = ptr(self.node_ids), ptr(self.node_off), ptr(self.idx)
        return s


class OrbmFrustumPoints(C.Structure):
    _fields_ = [("n", C.c_int), ("xw", vp), ("normal", vp), ("min_dist", vp), ("max_dist", vp)]


# T-variant semantic clusters (gcm_add_keyframe_objects)
GCM_CLUSTER, GCM_BELOW_PROB, GCM_FEW_POINTS = 0, 1, 2
GCM_OBJECT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("width", "<f4"), ("height", "<f4"), ("class_id", "<i4"),
                             ("prob", "<f4")])


class GcmCluster(C.Structure):
    _fields_ = [("status", C.c_int32), ("n_band", C.c_int32), ("n_inliers", C.c_int32), ("n_voxels", C.c_int32),
                ("centroid", C.c_float * 3), ("min_pt", C.c_float * 3), ("max_pt", C.c_float * 3)]


def gcm_objects(objects) -> np.ndarray:
    """Detector boxes -> GcmObject array: a GCM_OBJECT_DTYPE array, or (x, y, width, height, class_id, prob) tuples."""
    if isinstance(objects, np.ndarray) and objects.dtype == GCM_OBJECT_DTYPE:
        return np.ascontiguousarray(objects)
    return np.array([tuple(o) for o in objects], GCM_OBJECT_DTYPE)
