"""What homography batches (OrbsBatch.homography = 1, TrackHomo chained frame by frame on the device) cost on the bench's
room workload with a moving object (640 x 480, ORBextractor(2000, ...), 265-frame batches, page-locked CV_16U inputs):
batch time and time per frame for 1, 4 and 16 handles, each on its own stream, submitted together and timed with CUDA
events recorded on each handle's stream before and after its submit (first start to last end; median and p10-p90 of
--reps batches after --warmup), beside the host time the submits take to return; the same frames as device_flow batches
(the no-homography branch on every frame) for comparison; and, when cv2 is importable, the reference's host path on the
first 64 frames (findHomography of the frame's own TrackHomo pairs + warpPerspective + pyrDown +
calcOpticalFlowFarneback), the pairs found by the pinned point-pair search on the batch's keypoints.
Development aid, not a bench value; writes nothing.

usage: homo_chain_probe.py [--frames 265] [--nfeatures 2000] [--reps 10] [--warmup 2] [--profile]
  --profile: one separate run under torch.profiler instead, printing the device time per kernel of one homography batch."""
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

FACTOR = np.float32(1.0 / synth.DEPTH_FACTOR)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def frames(F, seed=1234):
    """RoomStream frames with a textured disc moving 7 px per frame (what the dynamic mask removes)."""
    rs = synth.RoomStream(seed=seed, n=F)
    fr = [rs.frame(t) for t in range(F)]
    gray = np.stack([f[0] for f in fr])
    d16 = np.rint(np.stack([f[1] for f in fr]).astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    T = np.stack([f[3] for f in fr]).astype(np.float32).reshape(F, 16)
    tex = np.clip(np.rint(synth.texture(seed + 1, 480, 640, nrect=300, nline=120)), 0, 255).astype(np.uint8)
    yy, xx = np.mgrid[0:480, 0:640]
    for t in range(F):
        m = (yy - 240) ** 2 + (xx - (40 + (7 * t) % 560)) ** 2 < 60 ** 2
        gray[t][m] = np.roll(tex, 7 * t, axis=1)[m]
    return gray, d16, T


def pinned(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    return t, t.numpy()


def tracker(F, nfeatures):
    return StreamTracker(nfeatures, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, 15.0, 0.9,
                         max_frames=F)


def timed(handles, submit, reps, warmup):
    streams = [torch.cuda.ExternalStream(st.stream()) for st, _ in handles]
    ts, hs = [], []
    for r in range(warmup + reps):
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in handles]
        t0 = time.perf_counter()
        for (st, out), s, (a, b) in zip(handles, streams, ev):
            a.record(s)
            submit(st, out)
            b.record(s)
        host = time.perf_counter() - t0
        for st, _ in handles:
            st.sync()
        if r >= warmup:
            first = ev[0][0]
            ts.append(max(first.elapsed_time(b) for _, b in ev) - min(first.elapsed_time(a) for a, _ in ev))
            hs.append(host * 1e3)
    ts = np.array(ts)
    return dict(median_ms=float(np.median(ts)), p10_ms=float(np.percentile(ts, 10)), p90_ms=float(np.percentile(ts, 90)),
                submit_host_ms=float(np.median(hs)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=265)
    ap.add_argument("--nfeatures", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("homo_chain_probe: no CUDA device")
    F = a.frames
    gray, d16, T = frames(F)
    keep = [pinned(x) for x in (gray, d16, T)]
    g, d, tt = (k[1] for k in keep)
    res = dict(card=card(), frames=F, nfeatures=a.nfeatures)

    def homo(st, out):
        st.submit_batch_u16_homography(g, d, FACTOR, tt, 40.0, out)

    def flow(st, out):
        st.submit_batch_u16_flow(g, d, FACTOR, tt, None, 40.0, out)

    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        st = tracker(F, a.nfeatures)
        out = st.alloc_outputs(F, pinned=True)
        homo(st, out)
        st.sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            homo(st, out)
            st.sync()
        per = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                k = e.name if len(e.name) < 60 else e.name[:60]
                n, us = per.get(k, (0, 0.0))
                per[k] = (n + 1, us + e.device_time)
        tot = sum(v[1] for v in per.values())
        res["profile"] = {k: dict(calls=n, ms=round(us / 1e3, 3), ms_per_frame=round(us / 1e3 / F, 4),
                                  share=round(us / tot, 4)) for k, (n, us) in sorted(per.items(), key=lambda kv: -kv[1][1])}
        res["profile_total_ms"] = round(tot / 1e3, 3)
        print(json.dumps(res, indent=1))
        return
    for n in (1, 4, 16):
        hs = []
        for _ in range(n):
            st = tracker(F, a.nfeatures)
            hs.append((st, st.alloc_outputs(F, pinned=True)))
        r = timed(hs, homo, a.reps, a.warmup)
        branches = [hs[0][0].homography(t)[0] for t in range(F)]
        r.update(ms_per_frame=r["median_ms"] / (n * F), frames_per_s=n * F / r["median_ms"] * 1e3,
                 branches={b: branches.count(b) for b in sorted(set(branches))})
        res["homography_%d" % n] = r
        if n == 1:
            cap = hs[0][0].device_results()[1]
            res["keypoint_capacity"] = cap
            res["iteration_table_MB"] = (cap - 50) * (cap + 55) / 2 * 8 / 2 ** 20   # hf_tab rows 51 .. cap, n + 2 doubles
        rf = timed(hs, flow, a.reps, a.warmup)
        rf.update(ms_per_frame=rf["median_ms"] / (n * F), frames_per_s=n * F / rf["median_ms"] * 1e3)
        res["device_flow_%d" % n] = rf
        del hs
        torch.cuda.empty_cache()
    try:
        import cv2
    except ImportError:
        res["cv2_host_path"] = "not measured: cv2 is not importable here"
    else:
        from oracle import ref
        from orb_slam2_ssd_semantic_b200.matcher import ORBmatcher
        from tests.helpers import frame_views
        n = min(F, 64)
        T44 = T.reshape(F, 4, 4)
        depth = d16.astype(np.float32) * FACTOR
        plain, homo_st = tracker(n, a.nfeatures), tracker(n, a.nfeatures)
        kp, de, nk, _, _ = plain.track_batch_u16(gray[:n], d16[:n], FACTOR, T44[:n])
        fk, fd, fn, _, _ = homo_st.track_batch_u16_homography(gray[:n], d16[:n], FACTOR, T44[:n])
        sf = ref.RefExtractor(a.nfeatures, 1.2, 8, 20, 7).mvScaleFactor
        mt = ORBmatcher(0.9, True)
        ts = []
        for t in range(2, n):
            K, D, Kl, Dl = kp[t, :nk[t]], de[t, :nk[t]], fk[t - 1, :fn[t - 1]], fd[t - 1, :fn[t - 1]]
            cur, last = frame_views(ref, K, D, depth[t], T44[t], Kl, Dl, depth[t - 1], T44[t - 1], sf)
            nm, _, pairs = mt.SearchByProjectionPairs(cur, last, 15.0, False)
            if nm < 20:
                nm, _, pairs = mt.SearchByProjectionPairs(cur, last, 30.0, False)
            if nm < 20 or len(pairs) <= 50:
                continue
            pc = np.stack([K["x"][pairs[:, 1]], K["y"][pairs[:, 1]]], 1).astype(np.float32)
            pl = np.stack([Kl["x"][pairs[:, 0]], Kl["y"][pairs[:, 0]]], 1).astype(np.float32)
            half_a = cv2.pyrDown(gray[t - 1])
            t0 = time.perf_counter()
            H, _ = cv2.findHomography(pc, pl, cv2.RANSAC, 3)
            w = cv2.warpPerspective(gray[t], H, (640, 480)) if H is not None else gray[t]
            cv2.calcOpticalFlowFarneback(half_a, cv2.pyrDown(w), None, 0.5, 3, 15, 3, 5, 1.2, 0)
            ts.append(time.perf_counter() - t0)
        res["cv2_host_path"] = dict(ms_per_frame_median=float(np.median(ts) * 1e3), frames=len(ts),
                                    threads=cv2.getNumThreads())
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
