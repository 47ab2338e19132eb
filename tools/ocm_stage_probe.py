"""Where one bench step's occupancy insert spends its time: the 368 keyframes of a step (16 batches of 23, 640 x 480,
0.05 m map, floor label as ground) inserted on the map's own stream with nothing else running, as bench.py's "mapping
alone" does.  Prints one JSON line: the card, its power limit, the event time of a whole step's insert (median of
--reps steps), and, from a separate run under torch.profiler, the device time per step of each insert kernel.
Development aid, not a bench value; writes nothing.

usage: ocm_stage_probe.py [--warmup 3] [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from orb_slam2_ssd_semantic_b200 import PointCloudMapping, synth  # noqa: E402

KERNELS = ("k_ocm_bin", "k_ocm_ranges", "k_ocm_scatter", "k_ocm_centroids", "k_ocm_scan_keys", "k_ocm_apply")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    _, depth, rgb, label, T = bench.make_batch(0, bench.BATCH)
    kf = np.array([t for t in range(bench.BATCH) if t % bench.KF_EVERY == 0], np.int32)
    poses = [bench.shifted_poses(T[kf], r) for r in range(bench.ROOMS)]
    d_depth, d_rgb, d_label = (torch.from_numpy(x).to(dev) for x in (depth, rgb, label))
    pcm = PointCloudMapping(0.05, device=0)
    ext = torch.cuda.ExternalStream(pcm.stream(), device=dev)
    step_no = [0]

    def step():   # one bench step's inserts: SUB batches, each on the next orientation of the room
        k = step_no[0]
        step_no[0] += 1
        for b in range(bench.SUB):
            pcm.insert_keyframes_device(d_depth.data_ptr(), d_rgb.data_ptr(), bench.ROWS, bench.COLS, kf,
                                        poses[(k * bench.SUB + b) % bench.ROOMS], synth.FX, synth.FY, synth.CX, synth.CY,
                                        d_label=d_label.data_ptr())

    for _ in range(a.warmup):
        step()
    pcm.sync()
    ms = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(ext)
        step()
        e1.record(ext)
        pcm.sync()
        ms.append(e0.elapsed_time(e1))
    points, _ = pcm.last_batch_stats()

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            step()
        pcm.sync()
    per_kernel = {}
    for e in prof.key_averages():
        name = next((k for k in KERNELS if k in e.key), None)
        if name:
            us = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
            per_kernel[name] = per_kernel.get(name, 0.0) + us / a.reps / 1e3
    vg = sum(per_kernel.get(k, 0.0) for k in KERNELS[:4])
    print(json.dumps({"card": card(), "keyframes_per_step": int(len(kf) * bench.SUB),
                      "insert_ms_per_step_median": round(float(np.median(ms)), 3),
                      "insert_ms_per_step_min_max": [round(min(ms), 3), round(max(ms), 3)],
                      "kernel_ms_per_step": {k: round(per_kernel.get(k, 0.0), 3) for k in KERNELS},
                      "voxelgrid_ms_per_step": round(vg, 3),
                      "points_last_round": int(points)}), flush=True)


if __name__ == "__main__":
    main()
