"""Host-side mirror of the `perfect` variant's dynamic-mask stages over the C-ABI (include/b200orb.h, dynm_*).

`Flow` follows FlowSLAM::Flow (perfect/include/Flow.h:18-37): ComputeMask(GrayImg, BInaryThreshold) keeps the previous
half-resolution gray image and returns the static / dynamic mask.  The dense optical flow between the two half-resolution
images is OpenCV's calcOpticalFlowFarneback in the reference (perfect/src/Flow.cc:29) and is a host callable here
(`flow_fn(prev, cur) -> rows x cols x 2 float32`, default: cv2's, when cv2 is importable); `DynamicMask.farneback` is the
same call on the GPU, bit-exact with OpenCV 4.13 at its baseline dispatch level (`Flow(flow_fn=dm.farneback)`).
Everything after it -- pyrUp of the flow, the threshold loop, erode, erode, dilate -- runs on the GPU
(dynm_mask_from_flow).  The homography overload (perfect/src/Flow.cc:73-80, `ComputeMask(GrayImg, Homo=H)` here) first
warps the gray image by cv::warpPerspective on the GPU (`DynamicMask.warp_perspective`, bit-exact with OpenCV 4.13).

`filter_keypoints` is the keypoint loop of the masked RGB-D Frame constructor (perfect/src/Frame.cc:356-377).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .extractor import KP_DTYPE


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class DynamicMask:
    """Handle of the dynm_* entry points (one CUDA stream + scratch)."""

    def __init__(self, device: int = 0):
        self._L = _lib.lib()
        self._h = C.c_void_p()
        _lib.check(self._L.dynm_create(int(device), C.byref(self._h)))

    def __del__(self):
        try:
            if self._h:
                self._L.dynm_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    def element(self) -> np.ndarray:
        el = np.zeros((21, 21), np.uint8)
        _lib.check(self._L.dynm_element(self._h, _p(el)))
        return el

    def mask_from_flow(self, flow: np.ndarray, binary_threshold: float = 40.0, shape=None) -> np.ndarray:
        """flow rows x cols x 2 float32 (half resolution) -> mask uint8 (1 static, 0 dynamic) of the gray image's `shape`
        (default 2 rows x 2 cols; an odd-sized gray image has one more row / column, which stays 1 before the erosion)."""
        flow = np.ascontiguousarray(flow, np.float32)
        if flow.ndim != 3 or flow.shape[2] != 2:
            raise ValueError("flow must be rows x cols x 2 float32")
        rows, cols = flow.shape[:2]
        mr, mc = (2 * rows, 2 * cols) if shape is None else (int(shape[0]), int(shape[1]))
        mask = np.zeros((mr, mc), np.uint8)
        _lib.check(self._L.dynm_mask_from_flow(self._h, _p(flow), rows, cols, float(binary_threshold), _p(mask), mr, mc))
        return mask

    def filter_keypoints(self, mask: np.ndarray, kps: np.ndarray, desc: np.ndarray):
        """-> (kps, desc) kept by the masked Frame constructor's loop."""
        if mask.dtype != np.uint8 or mask.ndim != 2:
            raise ValueError("mask must be rows x cols uint8")
        if mask.strides[1] != 1:
            mask = np.ascontiguousarray(mask)
        kps = np.ascontiguousarray(kps, KP_DTYPE).copy()
        desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32).copy()
        n = C.c_int(0)
        _lib.check(self._L.dynm_filter_keypoints(self._h, _p(mask), mask.shape[0], mask.shape[1], mask.strides[0], _p(kps),
                                                 _p(desc), len(kps), C.byref(n)))
        return kps[:n.value].copy(), desc[:n.value].copy()

    def farneback(self, prev: np.ndarray, cur: np.ndarray) -> np.ndarray:
        """calcOpticalFlowFarneback(prev, cur, None, 0.5, 3, 15, 3, 5, 1.2, 0) of two half-resolution u8 images on the GPU
        (perfect/src/Flow.cc:29), bit-exact with OpenCV 4.13 at its baseline dispatch level -> rows x cols x 2 float32."""
        prev = np.ascontiguousarray(prev, np.uint8)
        cur = np.ascontiguousarray(cur, np.uint8)
        if prev.ndim != 2 or prev.shape != cur.shape:
            raise ValueError("prev and cur must be two rows x cols uint8 images of one size")
        rows, cols = prev.shape
        flow = np.zeros((rows, cols, 2), np.float32)
        _lib.check(self._L.dynm_farneback(self._h, _p(prev), _p(cur), rows, cols, _p(flow)))
        return flow

    def flow_batch_device(self, d_gray: int, d_prev, nframes: int, rows: int, cols: int, d_flow: int):
        """pyrDown + Farneback (Flow.cc:26-29) of nframes full-resolution u8 frames in HBM (device pointers) into
        d_flow[nframes][rows/2][cols/2][2] f32; d_prev = the frame before d_gray[0] or None / 0 (frame 0 then takes the
        zero field).  Asynchronous on this handle's stream (stream())."""
        _lib.check(self._L.dynm_flow_batch_device(self._h, C.c_void_p(d_gray), C.c_void_p(d_prev or None), int(nframes),
                                                  int(rows), int(cols), C.c_void_p(d_flow)))

    def warp_perspective(self, gray: np.ndarray, H) -> np.ndarray:
        """cv::warpPerspective(gray, dest, H, gray.size()) on the GPU (perfect/src/Flow.cc:78: INTER_LINEAR,
        BORDER_CONSTANT 0, H inverted first), bit-exact with OpenCV 4.13.  H: the 3x3 forward map -> rows x cols uint8."""
        gray = np.ascontiguousarray(gray, np.uint8)
        H = np.ascontiguousarray(H, np.float64)
        if gray.ndim != 2:
            raise ValueError("gray must be rows x cols uint8")
        if H.size != 9:
            raise ValueError("H must be a 3x3 matrix")
        dst = np.zeros_like(gray)
        _lib.check(self._L.dynm_warp_perspective(self._h, _p(gray), gray.shape[0], gray.shape[1], _p(H), _p(dst)))
        return dst

    def warp_perspective_batch_device(self, d_gray: int, nframes: int, rows: int, cols: int, d_H: int, d_dst: int):
        """warp_perspective of nframes u8 images in HBM (device pointers), frame n by its own H d_H[n][9] float64, into
        d_dst[nframes][rows][cols].  Asynchronous on this handle's stream (stream())."""
        _lib.check(self._L.dynm_warp_perspective_batch_device(self._h, C.c_void_p(d_gray), int(nframes), int(rows),
                                                              int(cols), C.c_void_p(d_H), C.c_void_p(d_dst)))

    def find_homography(self, points_current, points_last):
        """cv::findHomography(points_current, points_last, RANSAC, 3) on the GPU (perfect/src/Tracking.cc:1386), the
        LM refinement included, in OpenCV 4.13's baseline order of operations -> (H 3x3 float64 or None when no model
        is found, mask uint8[n]).  4 <= n <= 8192 pairs, float32 [n][2] each."""
        src = np.ascontiguousarray(points_current, np.float32).reshape(-1, 2)
        dst = np.ascontiguousarray(points_last, np.float32).reshape(-1, 2)
        if len(src) != len(dst):
            raise ValueError("points_current and points_last must have the same length")
        n = len(src)
        H = np.zeros(9, np.float64)
        mask = np.zeros(max(n, 1), np.uint8)
        found = C.c_int(0)
        _lib.check(self._L.dynm_find_homography(self._h, _p(src), _p(dst), n, _p(H), _p(mask), C.byref(found)))
        return (H.reshape(3, 3) if found.value else None), mask[:n]

    def stream(self) -> int:
        return int(self._L.dynm_stream(self._h) or 0)

    def sync(self):
        _lib.check(self._L.dynm_sync(self._h))

    def launch_count(self) -> int:
        return int(self._L.dynm_launch_count(self._h))


def _farneback_cv2(prev: np.ndarray, cur: np.ndarray) -> np.ndarray:
    import cv2   # the reference's own dependency for this call (perfect/src/Flow.cc:29)
    return cv2.calcOpticalFlowFarneback(prev, cur, None, 0.5, 3, 15, 3, 5, 1.2, 0)


def _pyr_down_cv2(gray: np.ndarray) -> np.ndarray:
    import cv2
    return cv2.pyrDown(gray, dstsize=(gray.shape[1] // 2, gray.shape[0] // 2))


class Flow:
    """FlowSLAM::Flow (perfect/include/Flow.h:18-37)."""

    def __init__(self, device: int = 0, flow_fn=None, pyr_down_fn=None):
        self._dm = DynamicMask(device)
        self._flow_fn = flow_fn or _farneback_cv2
        self._pyr_down = pyr_down_fn or _pyr_down_cv2
        self.mImGrayLast = None
        self.mImGrayCurrent = None

    def ComputeMask(self, GrayImg: np.ndarray, BInaryThreshold: float = 40.0, Homo=None):
        """-> mask (rows x cols uint8, 1 = static) or None for an empty image (the reference leaves `mask` untouched).
        Homo (3x3, the forward map findHomography returns): the overload of Flow.cc:73-80, which computes the mask of
        warpPerspective(GrayImg, Homo) -- warped on the GPU -- instead of GrayImg's.  An empty GrayImg returns None with
        Homo too, where the reference's warpPerspective of the empty Mat throws."""
        if Homo is not None and GrayImg is not None and GrayImg.size:
            GrayImg = self._dm.warp_perspective(GrayImg, Homo)          # :78
        if GrayImg is None or GrayImg.size == 0:
            return None
        mask = np.ones(GrayImg.shape[:2], np.uint8)                      # :25
        self.mImGrayCurrent = self._pyr_down(GrayImg)                    # :26
        if self.mImGrayLast is not None:                                 # :28
            flow = self._flow_fn(self.mImGrayLast, self.mImGrayCurrent)  # :29 (host: OpenCV's Farneback)
            mask = self._dm.mask_from_flow(flow, BInaryThreshold, GrayImg.shape[:2])   # :30-47 on the GPU
        self.mImGrayLast, self.mImGrayCurrent = self.mImGrayCurrent, self.mImGrayLast   # :50
        return mask
