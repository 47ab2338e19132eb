"""What the device dense flow costs on the bench's room workload (640 x 480 gray frames, 265-frame batches), one JSON line:

  flow_batch_ms     dynm_flow_batch_device alone (pyrDown + Farneback of 265 consecutive pairs, inputs in HBM), CUDA events
  track_flow_ms     track_batch_u16_flow (host buffers; orbs_submit with the flow computed on the device)
  track_masked_ms   track_batch_u16_masked fed the same flow precomputed (orbs_submit uploads it with the batch)
  cv2_ms            cv2.calcOpticalFlowFarneback of the same 265 half-resolution pairs on this machine's CPU (its default
                    dispatch), with cv2's default thread count and with one thread; absent without cv2
Each: median and p10 - p90 over --reps runs after a warm-up; the two tracker forms are alternated.  The card's name and
power limit are read in the same run.  --profile: a separate run under torch.profiler giving each flow kernel's device
time per batch instead.  Development aid, not a bench value; writes nothing unless --trace DIR is given.

usage: flow_probe.py [--frames 265] [--reps 20] [--nfeatures 2000] [--profile] [--trace DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from orb_slam2_ssd_semantic_b200 import StreamTracker, synth  # noqa: E402
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
    ap.add_argument("--nfeatures", type=int, default=2000)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--trace", default=None)
    a = ap.parse_args()
    F, rows, cols = a.frames, 480, 640
    if not torch.cuda.is_available():
        sys.exit("flow_probe: no GPU")
    rs = synth.RoomStream(seed=1234, n=F)
    fr = [rs.frame(t) for t in range(F)]
    gray_h = np.stack([f[0] for f in fr])
    d16_h = np.rint(np.stack([f[1] for f in fr]).astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    T_h = np.stack([f[3] for f in fr]).astype(np.float32)
    factor = np.float32(1.0 / synth.DEPTH_FACTOR)
    dm = DynamicMask(0)
    gray = torch.from_numpy(gray_h).cuda()
    flow = torch.empty((F, rows // 2, cols // 2, 2), dtype=torch.float32, device="cuda")
    s = torch.cuda.ExternalStream(dm.stream())
    torch.cuda.synchronize()

    def run_flow():
        dm.flow_batch_device(gray.data_ptr(), None, F, rows, cols, flow.data_ptr())

    run_flow()
    dm.sync()
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                run_flow()
            dm.sync()
        per = {}
        for e in prof.key_averages():
            if e.key.startswith("_ZN4b2004k_fb") or "k_fb_" in e.key:
                name = e.key.split("k_fb_")[1].split("E")[0] if "k_fb_" in e.key else e.key
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                per["k_fb_" + name.rstrip("0123456789")] = round(t / 3 / 1000.0, 3)
        if a.trace:
            os.makedirs(a.trace, exist_ok=True)
            prof.export_chrome_trace(os.path.join(a.trace, "flow_probe.pt.trace.json"))
        print(json.dumps({"card": card(), "frames": F, "size": [cols, rows], "kernel_ms_per_batch": per}))
        return
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.reps)]
    for e0, e1 in ev:
        e0.record(s)
        run_flow()
        e1.record(s)
    dm.sync()
    flow_ms = [e0.elapsed_time(e1) for e0, e1 in ev]
    flow_h = flow.cpu().numpy()

    mk = lambda: StreamTracker(a.nfeatures, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, 15.0, 0.9, True, F)
    st_f, st_m = mk(), mk()
    out_f, out_m = st_f.alloc_outputs(F), st_m.alloc_outputs(F)
    st_f.track_batch_u16_flow(gray_h, d16_h, factor, T_h, None, 40.0, out_f)
    st_m.track_batch_u16_masked(gray_h, d16_h, factor, T_h, flow_h, 40.0, out_m)
    assert (out_f[2] == out_m[2]).all() and (out_f[4] == out_m[4]).all(), "device flow and precomputed flow disagree"
    tf, tm = [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        st_f.track_batch_u16_flow(gray_h, d16_h, factor, T_h, None, 40.0, out_f)
        tf.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        st_m.track_batch_u16_masked(gray_h, d16_h, factor, T_h, flow_h, 40.0, out_m)
        tm.append((time.perf_counter() - t0) * 1e3)
    res = {"card": card(), "frames": F, "size": [cols, rows], "flow_batch_ms": stats(flow_ms), "track_flow_ms": stats(tf),
           "track_masked_ms": stats(tm)}
    try:
        import cv2
        half = [cv2.pyrDown(g, dstsize=(cols // 2, rows // 2)) for g in gray_h]
        cpu = {}
        n0 = cv2.getNumThreads()
        for label, nt in (("default_threads", n0), ("one_thread", 1)):
            cv2.setNumThreads(nt)
            t0 = time.perf_counter()
            for t in range(1, F):
                cv2.calcOpticalFlowFarneback(half[t - 1], half[t], None, 0.5, 3, 15, 3, 5, 1.2, 0)
            cpu[label] = round((time.perf_counter() - t0) * 1e3, 1)
        cv2.setNumThreads(n0)
        cpu["threads_default"] = n0
        cpu["cpu_count"] = os.cpu_count()
        res["cv2_ms"] = cpu
    except ImportError:
        pass
    print(json.dumps(res))


if __name__ == "__main__":
    main()
