"""Seeded inputs for the homography branch's warp (`cv::warpPerspective(GrayImg, dest, Homo, GrayImg.size())`,
perfect/src/Flow.cc:78): tests/test_homography_*.py and tools/make_homography_golden.py.

H is the forward map as findHomography returns it (row-major 3x3 double); warpPerspective inverts it.

  identity       H = I
  shift_int      integer translation (7, -3)
  shift_sub      sub-pixel translation (2.37, -1.61): every tap weight in use
  rotation       12 degrees about the image centre, slight zoom
  room           a small camera-motion homography of the kind TrackHomo estimates between consecutive frames
  perspective    strong perspective whose w = M6 x + M7 y + M8 of the inverse crosses zero inside the image
  w_zero         w of the inverse exactly 0 on the whole column x = 64 (the W ? 32 / W : 0 branch)
  outside        maps every pixel far outside the source (all border)
  huge           coordinates beyond the int and short ranges (the clamps and saturate_casts)
  singular       det H == 0: invert yields zeros, every pixel samples (0, 0)
"""
from __future__ import annotations

import numpy as np

from orb_slam2_ssd_semantic_b200 import synth

SIZES = ((480, 640), (720, 1280), (195, 323))
CASES = ("identity", "shift_int", "shift_sub", "rotation", "room", "perspective", "w_zero", "outside", "huge", "singular")


def image(rows: int, cols: int, seed: int = 11) -> np.ndarray:
    """A textured rows x cols u8 frame with noise (every intensity level and sharp edges)."""
    t = synth.texture(seed, rows, cols, nrect=80, nline=40)
    t = t + np.random.Generator(np.random.PCG64(seed)).normal(0, 6.0, t.shape)
    return np.clip(np.rint(t), 0, 255).astype(np.uint8)


def homography(case: str, rows: int, cols: int) -> np.ndarray:
    """-> the forward 3x3 double H of the case for a rows x cols image."""
    cx, cy = (cols - 1) / 2.0, (rows - 1) / 2.0
    if case == "identity":
        return np.eye(3)
    if case == "shift_int":
        return np.array([[1, 0, 7], [0, 1, -3], [0, 0, 1]], np.float64)
    if case == "shift_sub":
        return np.array([[1, 0, 2.37], [0, 1, -1.61], [0, 0, 1]], np.float64)
    if case == "rotation":
        a, s = np.deg2rad(12.0), 1.03
        c, n = s * np.cos(a), s * np.sin(a)
        return np.array([[c, -n, cx - c * cx + n * cy], [n, c, cy - n * cx - c * cy], [0, 0, 1]], np.float64)
    if case == "room":
        return np.array([[1.0041, 0.0127, -3.82], [-0.0093, 0.9987, 1.27], [2.1e-5, -1.4e-5, 1.0]], np.float64)
    if case == "perspective":
        # inverse with w = 1 - x / (0.6 cols) + 0.1 y / rows: zero on a slanted line inside the image
        Minv = np.array([[1.0, 0.2, 5.0], [0.1, 1.0, -4.0], [-1.0 / (0.6 * cols), 0.1 / rows, 1.0]], np.float64)
        return np.linalg.inv(Minv)
    if case == "w_zero":
        # inverse with w = (x - 64) (1 / 64): exactly zero at x = 64 (a block start, so W0 is exactly 0 there)
        Minv = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [1.0 / 64, 0.0, -1.0]], np.float64)
        return np.linalg.inv(Minv)
    if case == "outside":
        return np.array([[1, 0, -5.0 * cols], [0, 1, 3.0 * rows], [0, 0, 1]], np.float64)
    if case == "huge":
        Minv = np.array([[3e6, 1e5, -1e9], [-2e5, 4e6, 7e8], [1e-3, 2e-3, 1e-3]], np.float64)
        return np.linalg.inv(Minv)
    if case == "singular":
        return np.array([[1, 2, 3], [2, 4, 6], [0.5, 0.1, 1]], np.float64)
    raise ValueError(case)
