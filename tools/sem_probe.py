"""Per-keyframe cost of the semantic object clusters (gcm_add_keyframe_objects_device) on the room scene: 1, 4 and 16
boxes of about 100x100, 200x300 and 400x400 px (width x height).  Each configuration: 3 warm-up calls, then the median of
20 calls, each timed with CUDA events around the (synchronous) call.  The records of the first call are checked against
the CPU oracle (oracle/sem_ref.cpp) where its brute-force 51-NN finishes in reasonable time (every box at most
--check-limit band points).  Prints the card and its power limit beside the numbers.

    python tools/sem_probe.py [--reps 20] [--check-limit 40000] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from orb_slam2_ssd_semantic_b200 import GlobalCloudMapping, synth  # noqa: E402

LEAF = 0.04
K = (synth.FX, synth.FY, synth.CX, synth.CY)


def boxes(n, w, h):
    """n boxes of w x h px laid out over the 640 x 480 image (overlapping where they do not fit), cycling classes."""
    out = []
    for b in range(n):
        gx, gy = b % 4, b // 4
        x = 10.0 + (640.0 - w - 20.0) * (gx / 3.0 if n > 1 else 0.5)
        y = 10.0 + (480.0 - h - 20.0) * (gy / 3.0 if n > 4 else 0.5)
        out.append((float(np.float32(max(x, 1.0))), float(np.float32(max(y, 1.0))), float(w), float(h), (5, 9, 15, 20)[b % 4], 0.9))
    return out


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check-limit", type=int, default=40000)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    _, depth, rgb, T = synth.RoomStream(seed=1234, n=827).frame(0)
    rows, cols = depth.shape
    d_depth, d_bgr = torch.from_numpy(depth).cuda(), torch.from_numpy(np.ascontiguousarray(rgb)).cuda()
    torch.cuda.synchronize()
    card = torch.cuda.get_device_name(0)
    print("card: %s, power limit: %s" % (card, power_limit()))
    res = []
    for w, h in ((100, 100), (200, 300), (400, 400)):
        for n in (1, 4, 16):
            objs = boxes(n, w, h)
            gm = GlobalCloudMapping(LEAF)
            ts = []
            recs = None
            for r in range(a.warmup + a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = gm.insert_keyframe_objects_device(d_depth.data_ptr(), d_bgr.data_ptr(), rows, cols, T, *K, 1, objs)
                e1.record()
                torch.cuda.synchronize()
                if recs is None:
                    recs = out
                if r >= a.warmup:
                    ts.append(e0.elapsed_time(e1))
                if gm.size() > 30 * rows * cols:
                    gm = GlobalCloudMapping(LEAF)
            nb = [r.n_band for r in recs]
            check = "not run (a box above %d band points)" % a.check_limit
            if max(nb) <= a.check_limit:
                from oracle import sem_py
                ref, _, _ = sem_py.keyframe(depth, rgb, T, *K, 1, objs, LEAF)
                same = all((g.status, g.n_band, g.n_inliers, g.n_voxels, list(g.centroid), list(g.min_pt), list(g.max_pt)) ==
                           (q.status, q.n_band, q.n_inliers, q.n_voxels, list(q.centroid), list(q.min_pt), list(q.max_pt))
                           for g, q in zip(recs, ref))
                check = "bit-exact" if same else "MISMATCH"
            row = dict(boxes=n, w=w, h=h, band_points=int(sum(nb)), max_band=int(max(nb)), median_ms=float(np.median(ts)),
                       min_ms=float(np.min(ts)), oracle=check)
            res.append(row)
            print("%2d boxes %3dx%3d  band points %7d (largest %6d)  median %8.3f ms  min %8.3f ms  oracle: %s" % (
                n, w, h, row["band_points"], row["max_band"], row["median_ms"], row["min_ms"], check))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(card=card, power_limit=power_limit(), results=res), f, indent=1)
    return 0 if all(r["oracle"] != "MISMATCH" for r in res) else 1


if __name__ == "__main__":
    sys.exit(main())
