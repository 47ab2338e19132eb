"""What the device warpPerspective of the homography branch (perfect/src/Flow.cc:78) costs on the bench's room workload,
one JSON line:

  batch_ms     dynm_warp_perspective_batch_device over --frames 640 x 480 room frames in HBM, each by its own H, CUDA
               events on the handle's stream; us_per_frame = batch_ms / frames
  single_ms    dynm_warp_perspective of one frame (host buffers: upload, warp, download, sync), host clock
  cv2_ms       cv2.warpPerspective of one frame on this machine's CPU (its default dispatch and thread count); absent
               without cv2
Each: median and p10 - p90 over --reps runs after a warm-up.  The card's name and power limit are read in the same run.
Development aid, not a bench value; writes nothing.

usage: warp_probe.py [--frames 265] [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from orb_slam2_ssd_semantic_b200 import synth  # noqa: E402
from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(ms):
    ms = np.asarray(ms, np.float64)
    return {"median": round(float(np.median(ms)), 3), "p10": round(float(np.percentile(ms, 10)), 3),
            "p90": round(float(np.percentile(ms, 90)), 3), "n": int(len(ms))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=265)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    F, rows, cols = a.frames, 480, 640
    if not torch.cuda.is_available():
        sys.exit("warp_probe: no GPU")
    rs = synth.RoomStream(seed=1234, n=F)
    gray_h = np.stack([rs.frame(t)[0] for t in range(F)])
    rng = np.random.Generator(np.random.PCG64(1))
    Hs = np.repeat(np.eye(3)[None], F, axis=0) + rng.normal(0, 1e-3, (F, 3, 3)) * [[1, 1, 3000], [1, 1, 3000], [1e-2, 1e-2, 0]]
    dm = DynamicMask(0)
    gray = torch.from_numpy(gray_h).cuda()
    H = torch.from_numpy(Hs).cuda()
    out = torch.empty_like(gray)
    s = torch.cuda.ExternalStream(dm.stream())
    torch.cuda.synchronize()

    def run():
        dm.warp_perspective_batch_device(gray.data_ptr(), F, rows, cols, H.data_ptr(), out.data_ptr())

    run()
    dm.sync()
    n0 = dm.launch_count()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.reps)]
    for e0, e1 in ev:
        e0.record(s)
        run()
        e1.record(s)
    dm.sync()
    batch = [e0.elapsed_time(e1) for e0, e1 in ev]
    launches = (dm.launch_count() - n0) / a.reps
    one = []
    dm.warp_perspective(gray_h[0], Hs[0])
    for _ in range(a.reps):
        t0 = time.perf_counter()
        dm.warp_perspective(gray_h[0], Hs[0])
        one.append((time.perf_counter() - t0) * 1e3)
    b = stats(batch)
    res = {"card": card(), "frames": F, "size": [cols, rows], "batch_ms": b,
           "us_per_frame": round(b["median"] * 1e3 / F, 2), "launches_per_batch": launches, "single_ms": stats(one)}
    try:
        import cv2
        c = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            cv2.warpPerspective(gray_h[0], Hs[0], (cols, rows))
            c.append((time.perf_counter() - t0) * 1e3)
        res["cv2_ms"] = stats(c)
    except ImportError:
        pass
    print(json.dumps(res))


if __name__ == "__main__":
    main()
