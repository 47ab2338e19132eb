"""Writes tests/golden/undistort_cv2.npz: cv2.undistortPoints(xy, K, dist, None, K) -- what Frame::UndistortKeyPoints
calls (src/Frame.cc:559-590) -- on the crafted points and coefficient sets of tests/frame_cases.py, so that the
undistortion oracle is pinned to OpenCV on machines without cv2.  Sets whose k1 is zero are not stored: Frame.cc copies
the keypoints there and never calls OpenCV.

    python tools/make_undistort_golden.py"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import frame_cases as FC  # noqa: E402


def main():
    xy = FC.undistort_points()
    K = FC.UNDIST_K.reshape(3, 3)
    out = {"xy": xy, "K": FC.UNDIST_K, "cv2_version": np.array(cv2.__version__)}
    for name, d in FC.undistort_cases():
        if len(d) == 0 or d[0] == 0:
            continue
        key = name.split("/", 1)[1]
        out["dist/" + key] = d
        out["out/" + key] = cv2.undistortPoints(xy.reshape(-1, 1, 2), K, d, None, K).reshape(-1, 2).astype(np.float32)
    path = os.path.join(ROOT, "tests", "golden", "undistort_cv2.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "with OpenCV", cv2.__version__)


if __name__ == "__main__":
    main()
