"""Writes tests/golden/farneback_*.npz: cv2 4.13's calcOpticalFlowFarneback at its baseline dispatch level
(cv2.setUseOptimized(False)) with the arguments of perfect/src/Flow.cc:29, on pyrDown'ed pairs of tests/flow_scenes.py.
Each file holds gray (the two full-resolution frames), prev / cur (cv2.pyrDown of them, Size(cols/2, rows/2)) and flow.

    python tools/make_flow_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import flow_scenes as S  # noqa: E402

CASES = (("room", 120, 160), ("blobs", 97, 161), ("border", 64, 80), ("identical", 63, 80), ("flat", 16, 16))


def main():
    import cv2
    was = cv2.useOptimized()
    cv2.setUseOptimized(False)
    try:
        for scene, rows, cols in CASES:
            g = S.frames(scene, 2 * rows, 2 * cols, 2)
            prev, cur = (cv2.pyrDown(x, dstsize=(cols, rows)) for x in g)
            flow = cv2.calcOpticalFlowFarneback(prev, cur, None, 0.5, 3, 15, 3, 5, 1.2, 0)
            path = os.path.join(ROOT, "tests", "golden", "farneback_%s.npz" % scene)
            np.savez_compressed(path, gray=g, prev=prev, cur=cur, flow=flow, cv2_version=cv2.__version__)
            print(path, os.path.getsize(path))
    finally:
        cv2.setUseOptimized(was)


if __name__ == "__main__":
    main()
