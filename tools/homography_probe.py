"""Times findHomography(points_current, points_last, RANSAC, 3) on TrackHomo pair lists of about 51, 200, 1000 and
2000 pairs (the point-pair SearchByProjection restatement on tests/homo_cases.py's random frame pairs of 1000 and 2000
keypoints, and prefixes of them):

  host_ms     dynm_find_homography, host clock around the synchronous call (uploads, kernels, downloads, sync)
  device_ms   CUDA events recorded on the handle's stream before and after the call's enqueued work
  cv2_ms      cv2.findHomography on the host at its default dispatch, and at cv2.setUseOptimized(False)

Each is the median (p10-p90) of --calls calls after --warmup calls.  The first line names the card and its power limit.

    python tools/homography_probe.py [--calls 100] [--warmup 10]"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask  # noqa: E402
from tests import homography_fit_cases as HC  # noqa: E402


def _stats(v):
    v = np.asarray(v)
    return "%.3f (%.3f-%.3f)" % (np.median(v), np.percentile(v, 10), np.percentile(v, 90))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    print("card, power limit:", _card())
    rt = C.CDLL("libcudart.so.12") if sys.platform.startswith("linux") else None
    dm = DynamicMask()
    stream = C.c_void_p(dm.stream())
    e0, e1 = C.c_void_p(), C.c_void_p()
    rt.cudaEventCreate(C.byref(e0))
    rt.cudaEventCreate(C.byref(e1))
    try:
        import cv2
    except ImportError:
        cv2 = None
    sets = {name: (s, d) for name, s, d in HC.track_homo_pairs()}
    order = ["track_homo_1000_first_51", "track_homo_1000_first_200", "track_homo_1000", "track_homo_2000"]
    for name in order:
        src, dst = sets[name]
        host, dev = [], []
        for k in range(a.warmup + a.calls):
            rt.cudaEventRecord(e0, stream)
            t = time.perf_counter()
            dm.find_homography(src, dst)
            t = (time.perf_counter() - t) * 1e3
            rt.cudaEventRecord(e1, stream)
            rt.cudaEventSynchronize(e1)
            ms = C.c_float()
            rt.cudaEventElapsedTime(C.byref(ms), e0, e1)
            if k >= a.warmup:
                host.append(t)
                dev.append(ms.value)
        line = "%-28s n=%5d  host_ms %s  device_ms %s" % (name, len(src), _stats(host), _stats(dev))
        if cv2 is not None:
            was = cv2.useOptimized()
            for opt in (True, False):
                cv2.setUseOptimized(opt)
                v = []
                for k in range(a.warmup + a.calls):
                    t = time.perf_counter()
                    cv2.findHomography(src, dst, cv2.RANSAC, 3)
                    if k >= a.warmup:
                        v.append((time.perf_counter() - t) * 1e3)
                line += "  cv2_%s_ms %s" % ("default" if opt else "baseline", _stats(v))
            cv2.setUseOptimized(was)
        print(line, flush=True)
    rt.cudaEventDestroy(e0)
    rt.cudaEventDestroy(e1)


if __name__ == "__main__":
    main()
