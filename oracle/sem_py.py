"""ctypes front-end of oracle/libsem_oracle.so (oracle/sem_ref.cpp, built by oracle/sem.mk): the semantic object clusters
of the T variant's mapping thread restated on the CPU.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from orb_slam2_ssd_semantic_b200._abi import GcmCluster, gcm_objects

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libsem_oracle.so")
ALT_SQRT, ALT_SQSUM = 1, 2      # the other reading of each unpinned PCL line (sem_ref.cpp)
_lib = None


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-C", _HERE, "-f", "sem.mk", "-s"])
        L = C.CDLL(_SO)
        vp, i, f = C.c_void_p, C.c_int, C.c_float
        L.sem_ref_band.restype = C.c_longlong
        L.sem_ref_band.argtypes = [vp, vp, i, i, vp, C.POINTER(f), vp, C.c_longlong]
        L.sem_ref_knn.restype = None
        L.sem_ref_knn.argtypes = [vp, i, i, vp]
        L.sem_ref_sor.argtypes = [vp, i, i, vp, vp]
        L.sem_ref_cluster.restype = None
        L.sem_ref_cluster.argtypes = [vp, i, f, i, C.POINTER(GcmCluster)]
        L.sem_ref_keyframe.argtypes = [vp, vp, i, i, vp, f, f, f, f, C.c_longlong, vp, i, f, i, vp, vp, vp]
        _lib = L
    return _lib


def band(depth, obj, bgr=None):
    """draw_rect_with_depth_threshold for one box -> (flat indices in (k, j) order, mean depth); paints bgr in place."""
    depth = np.ascontiguousarray(depth, np.float32)
    rows, cols = depth.shape
    o = gcm_objects([obj])
    thr = C.c_float(0)
    n = lib().sem_ref_band(_p(depth), _p(bgr), rows, cols, _p(o), C.byref(thr), None, 0)
    idx = np.zeros(max(n, 1), np.int32)
    lib().sem_ref_band(_p(depth), None, rows, cols, _p(o), C.byref(thr), _p(idx), n)
    return idx[:n], np.float32(thr.value)


def knn(xyz, k=51):
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    out = np.zeros((len(xyz), k), np.float32)
    lib().sem_ref_knn(_p(xyz), len(xyz), k, _p(out))
    return out


def sor(xyz, reading=0):
    """-> (mean neighbour distance per point, keep mask)."""
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    d = np.zeros(len(xyz), np.float32)
    keep = np.zeros(len(xyz), np.uint8)
    lib().sem_ref_sor(_p(xyz), len(xyz), reading, _p(d), _p(keep))
    return d, keep.astype(bool)


def cluster(xyz, leaf, reading=0) -> GcmCluster:
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    c = GcmCluster()
    lib().sem_ref_cluster(_p(xyz), len(xyz), float(np.float32(leaf)), reading, C.byref(c))
    return c


def keyframe(depth, bgr, Tcw, fx, fy, cx, cy, i, objects, leaf, reading=0):
    """One keyframe of the loop (:413-485) -> (records, painted bgr, (xyz, rgb) of the cloud or None when skipped)."""
    depth = np.ascontiguousarray(depth, np.float32)
    bgr = np.array(bgr, np.uint8, copy=True, order="C")
    rows, cols = depth.shape
    o = gcm_objects(objects)
    T = np.ascontiguousarray(Tcw, np.float32).reshape(16)
    out = (GcmCluster * max(len(o), 1))()
    xyz = np.zeros((rows * cols, 3), np.float32)
    rgb = np.zeros((rows * cols, 3), np.uint8)
    added = lib().sem_ref_keyframe(_p(depth), _p(bgr), rows, cols, _p(T), float(fx), float(fy), float(cx), float(cy), int(i),
                                   _p(o) if len(o) else None, len(o), float(np.float32(leaf)), reading, out, _p(xyz), _p(rgb))
    return list(out)[:len(o)], bgr, ((xyz, rgb) if added else None)
