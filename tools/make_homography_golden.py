"""Writes tests/golden/homography_warp.npz: cv2 4.13's warpPerspective with the arguments of perfect/src/Flow.cc:78
(INTER_LINEAR, BORDER_CONSTANT 0, destination size = source size) on every case of tests/warp_cases.py, for one
120 x 160 image.  The warp's integer path gives the same bytes at every dispatch level; the tool checks that before it
writes.  Fields: src (rows x cols u8), cases (names), H (n x 3 x 3 float64, forward maps), dst (n x rows x cols u8).

    python tools/make_homography_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import warp_cases as WC  # noqa: E402

ROWS, COLS = 120, 160


def main():
    import cv2
    was = cv2.useOptimized()
    src = WC.image(ROWS, COLS)
    Hs = np.stack([WC.homography(c, ROWS, COLS) for c in WC.CASES])
    try:
        out = []
        for opt in (False, True):
            cv2.setUseOptimized(opt)
            out.append(np.stack([cv2.warpPerspective(src, H, (COLS, ROWS)) for H in Hs]))
    finally:
        cv2.setUseOptimized(was)
    assert (out[0] == out[1]).all(), "cv2's warp differs between dispatch levels"
    path = os.path.join(ROOT, "tests", "golden", "homography_warp.npz")
    np.savez_compressed(path, src=src, cases=np.array(WC.CASES), H=Hs, dst=out[0], cv2_version=cv2.__version__)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
