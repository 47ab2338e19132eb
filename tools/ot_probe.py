"""Timing of the `.ot` writer: the device tree (ocm_tree_build + ocm_write_ot, CUDA events on the map's stream) beside the
numpy one (export_leaves + octree_io.build_ot, host clock), both arms in one call, alternating, on two maps: the
reference's own tree (~391 k cells) and the map bench.py's room scene reaches after one step (16 batches of 23 keyframes,
16 world orientations).  Prints one JSON line per map with the card's name and power limit beside the numbers.

    python tools/ot_probe.py [--reps 20] [--warmup 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or "unknown"


def reference_map():
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    from orb_slam2_ssd_semantic_b200 import octree_io as O
    z = np.load(os.path.join(ROOT, "tests", "golden", "octomap_nodes.npz"))
    nodes = np.zeros(len(z["v"]), O.NODE_DT)
    nodes["v"], nodes["rgb"], nodes["child"] = z["v"], z["rgb"], z["child"]
    pcm = PointCloudMapping(0.05)
    pcm.read_ot(str(z["header"]).encode() + nodes.tobytes())
    return pcm


def bench_step_map():
    import torch
    import bench
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping, synth
    rs = synth.RoomStream(seed=1234, n=bench.BATCH)
    kfs = list(range(0, bench.BATCH, bench.KF_EVERY))
    fr = [rs.frame(t, with_label=True) for t in kfs]
    depth = torch.from_numpy(np.stack([f[1] for f in fr])).cuda()
    rgb = torch.from_numpy(np.stack([f[2] for f in fr])).cuda()
    label = torch.from_numpy(np.stack([f[4] for f in fr])).cuda()
    T = np.stack([f[3] for f in fr]).astype(np.float32)
    pcm = PointCloudMapping(0.05)
    for b in range(bench.SUB):
        pcm.insert_keyframes_device(depth.data_ptr(), rgb.data_ptr(), bench.ROWS, bench.COLS, list(range(len(kfs))),
                                    bench.shifted_poses(T, b % bench.ROOMS), synth.FX, synth.FY, synth.CX, synth.CY,
                                    d_label=label.data_ptr())
    pcm.sync()
    return pcm


def measure(name, pcm, reps, warmup):
    import torch
    from orb_slam2_ssd_semantic_b200 import octree_io as O
    ext = torch.cuda.ExternalStream(pcm.stream())
    dev_ms, dev_wall_ms, host_ms = [], [], []
    same = True
    nn = nl = 0
    for r in range(warmup + reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(ext)
        nn, nl = pcm.tree_build()
        got = pcm.write_ot()
        e1.record(ext)
        e1.synchronize()
        t1 = time.perf_counter()
        k, v, c = pcm.export_leaves()
        want = O.build_ot(k, v, c, 0.05, "0.05")
        t2 = time.perf_counter()
        same = same and got == want
        if r >= warmup:
            dev_ms.append(e0.elapsed_time(e1)); dev_wall_ms.append((t1 - t0) * 1e3); host_ms.append((t2 - t1) * 1e3)
    med = lambda a: float(np.median(a))   # noqa: E731
    print(json.dumps({"map": name, "cells": pcm.num_leaves(), "nodes": nn, "pruned_leaves": nl, "bytes_identical": same,
                      "device_tree_build_plus_write_ms": {"events_median": med(dev_ms), "events_min": min(dev_ms),
                                                          "events_max": max(dev_ms), "host_clock_median": med(dev_wall_ms)},
                      "numpy_export_plus_build_ot_ms": {"host_clock_median": med(host_ms), "min": min(host_ms),
                                                        "max": max(host_ms)},
                      "reps": reps, "warmup": warmup, "card": card()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ot_probe: no CUDA device; a timing needs the GPU")
    measure("reference octomap.ot", reference_map(), a.reps, a.warmup)
    measure("bench room scene after one step", bench_step_map(), a.reps, a.warmup)


if __name__ == "__main__":
    main()
