"""Writes tests/golden/flow_edges.npz: for every crafted pair of tests/flow_edge_cases.py, the SHA-256 digest
(tests/refpins.digest) of its inputs and of what cv2.calcOpticalFlowFarneback(prev, cur, None, 0.5, 3, 15, 3, 5, 1.2, 0)
returns at cv2.setUseOptimized(False), so that the GPU tests need no cv2.  Pairs of at most 4,096 pixels also store
prev, cur and the flow themselves; the flows of textured pairs barely compress (about 6.6 bytes per pixel), so larger
pairs keep only their digests and the file stays near 45 kB.

    python tools/make_farneback_edges_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cv2  # noqa: E402

from tests import flow_edge_cases as EC  # noqa: E402
from tests.refpins import digest  # noqa: E402

MAX_STORED_PIXELS = 4096


def main():
    cv2.setUseOptimized(False)
    z = {}
    names = []
    for c in EC.cases():
        flow = cv2.calcOpticalFlowFarneback(c.prev, c.cur, None, 0.5, 3, 15, 3, 5, 1.2, 0)
        names.append(c.name)
        z[c.name + "/inputs_sha256"] = np.array(digest((c.prev, c.cur)))
        z[c.name + "/flow_sha256"] = np.array(digest(flow))
        if c.prev.size <= MAX_STORED_PIXELS:
            z[c.name + "/prev"] = c.prev
            z[c.name + "/cur"] = c.cur
            z[c.name + "/flow"] = flow
    z["names"] = np.array(names)
    path = os.path.join(ROOT, "tests", "golden", "flow_edges.npz")
    np.savez_compressed(path, **z)
    print("wrote", path, len(names), "pairs,", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
