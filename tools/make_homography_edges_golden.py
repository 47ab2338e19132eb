"""Writes tests/golden/homography_edges.npz: for every crafted set of tests/homography_edge_cases.py, the pairs and what
cv2.findHomography(points_current, points_last, RANSAC, 3) returns at cv2.setUseOptimized(False) -- H (NaN when no
model) and the mask -- so that the GPU tests need no cv2.  `exact` marks the sets whose refinement runs on fewer than
100 residual rows (fewer than 50 inliers), where the restatement equals cv2 bit for bit; from 100 rows a cv2 built with
LAPACK hands J^T r to its BLAS (see tools/make_homography_fit_golden.py).

    python tools/make_homography_edges_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cv2  # noqa: E402

from oracle import homography_py as HP  # noqa: E402
from tests import homography_edge_cases as EC  # noqa: E402


def main():
    cv2.setUseOptimized(False)
    z = {}
    names = []
    for name, src, dst in EC.cases():
        H, mask = cv2.findHomography(src, dst, cv2.RANSAC, 3)
        names.append(name)
        z[name + "/src"] = src
        z[name + "/dst"] = dst
        z[name + "/H"] = np.full((3, 3), np.nan) if H is None else H
        z[name + "/mask"] = np.zeros(len(src), np.uint8) if mask is None else mask.ravel().astype(np.uint8)
        inl = HP.ransac(src, dst)[1] if len(src) > 4 else None
        z[name + "/exact"] = np.array(inl is None or int(inl.sum()) < 50)
    z["names"] = np.array(names)
    path = os.path.join(ROOT, "tests", "golden", "homography_edges.npz")
    np.savez_compressed(path, **z)
    print("wrote", path, len(names), "sets")


if __name__ == "__main__":
    main()
