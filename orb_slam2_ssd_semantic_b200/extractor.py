"""Host-side mirror of ORB_SLAM2::ORBextractor (reference include/ORBextractor.h:41-118) over the C-ABI.

Same constructor arguments, same getters, `__call__` plays operator() (src/ORBextractor.cc:1052-1114):
keypoints come back as a structured array with cv::KeyPoint's fields, descriptors as an N x 32 uint8 matrix.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])
assert KP_DTYPE.itemsize == 28


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class ORBextractor:
    HARRIS_SCORE = 0
    FAST_SCORE = 1

    def __init__(self, nfeatures: int = 1000, scaleFactor: float = 1.2, nlevels: int = 8, iniThFAST: int = 20,
                 minThFAST: int = 7, device: int = 0):
        self._L = _lib.lib()
        self._h = C.c_void_p()
        p = _lib.OrbxParams(int(nfeatures), float(scaleFactor), int(nlevels), int(iniThFAST), int(minThFAST))
        _lib.check(self._L.orbx_create(C.byref(p), int(device), C.byref(self._h)))
        self.nlevels = int(nlevels)
        self.nfeatures = int(nfeatures)
        self.scaleFactor = float(np.float32(scaleFactor))
        self.device = int(device)
        sf, inv, s2, is2 = (np.zeros(nlevels, np.float32) for _ in range(4))
        nf = np.zeros(nlevels, np.int32)
        _lib.check(self._L.orbx_scale_tables(self._h, _p(sf), _p(inv), _p(s2), _p(is2), _p(nf)))
        self._sf, self._inv, self._s2, self._is2, self.mnFeaturesPerLevel = sf, inv, s2, is2, nf
        self._nframes_last = 0

    def __del__(self):
        try:
            if self._h:
                self._L.orbx_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    # -- getters, include/ORBextractor.h:57-77 ---------------------------------------------------------
    def GetLevels(self) -> int:
        return self.nlevels

    def GetScaleFactor(self) -> float:
        return self.scaleFactor

    def GetScaleFactors(self) -> np.ndarray:
        return self._sf.copy()

    def GetInverseScaleFactors(self) -> np.ndarray:
        return self._inv.copy()

    def GetScaleSigmaSquares(self) -> np.ndarray:
        return self._s2.copy()

    def GetInverseScaleSigmaSquares(self) -> np.ndarray:
        return self._is2.copy()

    @property
    def handle(self):
        return self._h

    def max_keypoints(self, rows: int | None = None, cols: int | None = None) -> int:
        """Keypoints one frame can return: for a rows x cols image (refused like extraction refuses it), or without a
        geometry orbx_max_keypoints' value for the handle's current one."""
        if rows is None:
            return int(self._L.orbx_max_keypoints(self._h))
        n = C.c_int(0)
        _lib.check(self._L.orbx_max_keypoints_for(self._h, int(rows), int(cols), C.byref(n)))
        return n.value

    # -- operator() ---------------------------------------------------------------------------------------
    def __call__(self, image: np.ndarray, mask=None):
        """operator()(image, mask, keypoints, descriptors); mask is ignored like the reference (:1052)."""
        if image is None or image.size == 0:
            return np.zeros(0, KP_DTYPE), np.zeros((0, 32), np.uint8)
        if image.dtype != np.uint8 or image.ndim != 2:
            raise ValueError("image must be CV_8UC1 (reference asserts, src/ORBextractor.cc:1059)")
        if image.strides[1] != 1:
            image = np.ascontiguousarray(image)
        cap = self.max_keypoints(*image.shape)
        kps = np.zeros(cap, KP_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = C.c_int(0)
        _lib.check(self._L.orbx_extract(self._h, _p(image), image.shape[0], image.shape[1], image.strides[0], _p(kps),
                                        _p(desc), cap, C.byref(n)))
        self._nframes_last = 1
        return kps[:n.value].copy(), desc[:n.value].copy()

    def extract_batch(self, images: np.ndarray):
        """Batched many-frame mode: images [F, rows, cols] u8 -> list of (keypoints, descriptors)."""
        if images.dtype != np.uint8 or images.ndim != 3:
            raise ValueError("images must be [F, rows, cols] uint8")
        images = np.ascontiguousarray(images)
        F, rows, cols = images.shape
        cap = self.max_keypoints(rows, cols)
        kps = np.zeros((F, cap), KP_DTYPE)
        desc = np.zeros((F, cap, 32), np.uint8)
        n = np.zeros(F, np.int32)
        _lib.check(self._L.orbx_extract_batch(self._h, _p(images), F, rows, cols, images.strides[1], images.strides[0],
                                              _p(kps), _p(desc), cap, _p(n)))
        self._nframes_last = F
        return [(kps[f, :n[f]].copy(), desc[f, :n[f]].copy()) for f in range(F)]

    # -- mvImagePyramid (include/ORBextractor.h:80) -----------------------------------------------------------
    def image_pyramid_level(self, level: int, frame: int = 0, bordered: bool = False, blurred: bool = False) -> np.ndarray:
        """Level `level` of frame `frame` of the last extract; `bordered` adds the REFLECT_101 frame, `blurred` returns the
        7x7 Gaussian blur of the level that the descriptors read instead."""
        if bordered and blurred:
            raise ValueError("the blurred level has no bordered form")
        r, c = C.c_int(), C.c_int()
        _lib.check(self._L.orbx_level_dims(self._h, level, C.byref(r), C.byref(c)))
        shp = (r.value + 38, c.value + 38) if bordered else (r.value, c.value)
        out = np.zeros(shp, np.uint8)
        kind = 2 if blurred else int(bordered)
        _lib.check(self._L.orbx_get_level(self._h, frame, level, kind, _p(out), out.strides[0]))
        return out

    @property
    def mvImagePyramid(self):
        return [self.image_pyramid_level(l) for l in range(self.nlevels)]

    def candidates_per_level(self, frame: int = 0) -> np.ndarray:
        out = np.zeros(self.nlevels, np.int32)
        _lib.check(self._L.orbx_candidates_per_level(self._h, frame, _p(out)))
        return out

    def fast_candidates(self, level: int, frame: int = 0) -> np.ndarray:
        """FAST survivors of one level, [n, 3] int32 (x, y, score) in level pixels, in the quad-tree's input order."""
        n = C.c_int(0)
        rc = self._L.orbx_get_candidates(self._h, frame, level, None, 0, C.byref(n))
        if rc != -2:   # B200ORB_ECAP: *n is the count, nothing written
            _lib.check(rc)
        out = np.zeros((max(n.value, 1), 3), np.int32)
        _lib.check(self._L.orbx_get_candidates(self._h, frame, level, _p(out), n.value, C.byref(n)))
        return out[:n.value]

    def distribute(self, rows: int, cols: int, level: int, N: int, xys: np.ndarray) -> np.ndarray:
        """DistributeOctTree alone on the device: the extractor's quad-tree kernel on the candidate list xys ([n, 3] int32
        x, y, score in level pixels, vToDistributeKeys order) of level `level` of a rows x cols image, with target N.
        Returns the selected keypoints, [m, 3] int32 in list order.  The pyramid and candidate read-backs refuse until
        the next extract."""
        xys = np.ascontiguousarray(xys, np.int32).reshape(-1, 3)
        n = len(xys)
        out = np.zeros((max(n, 1), 3), np.int32)   # every selected node holds at least one of the n candidates
        m = C.c_int(0)
        _lib.check(self._L.orbx_distribute(self._h, int(rows), int(cols), int(level), int(N), _p(xys), n, _p(out), len(out),
                                           C.byref(m)))
        return out[:m.value].copy()

    def launch_count(self) -> int:
        return int(self._L.orbx_launch_count(self._h))
