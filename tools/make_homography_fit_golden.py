"""Writes tests/golden/homography_fit.npz: for every set of tests/homography_fit_cases.py, the pairs and what
cv2.findHomography(points_current, points_last, RANSAC, 3) returns at cv2.setUseOptimized(False) -- H (NaN when no
model) and the mask -- so that the GPU tests need neither cv2 nor the reference.  `exact` marks the sets whose
refinement runs on fewer than 100 residual rows (fewer than 50 inliers): there cv2 computes J^T r itself, and the
restatement (tests/homography_lm.py) equals it bit for bit; from 100 rows a cv2 built with LAPACK hands J^T r to its
BLAS, whose order of operations depends on the BLAS kernel the host CPU selects.

    python tools/make_homography_fit_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cv2  # noqa: E402

from oracle import homography_py as HP  # noqa: E402
from tests import homography_fit_cases as HC  # noqa: E402


def main():
    cv2.setUseOptimized(False)
    z = {}
    names = []
    for name, src, dst in HC.cases():
        H, mask = cv2.findHomography(src, dst, cv2.RANSAC, 3)
        names.append(name)
        z[name + "/src"] = src
        z[name + "/dst"] = dst
        z[name + "/H"] = np.full((3, 3), np.nan) if H is None else H
        z[name + "/mask"] = np.zeros(len(src), np.uint8) if mask is None else mask.ravel().astype(np.uint8)
        inl = HP.ransac(src, dst)[1] if len(src) > 4 else None
        z[name + "/exact"] = np.array(inl is None or int(inl.sum()) < 50)
    z["names"] = np.array(names)
    path = os.path.join(ROOT, "tests", "golden", "homography_fit.npz")
    np.savez_compressed(path, **z)
    print("wrote", path, len(names), "sets")


if __name__ == "__main__":
    main()
