"""What continuing a sequence across batches (orbs_continue) costs on the bench's room workload (640 x 480,
ORBextractor(2000, ...), 4 batches of 265 RoomStream frames, page-locked CV_16U inputs and outputs): the same four batches
on one handle, once as independent batches and once with each batch after the first continuing the one before
(continue_after(self) before its submit), for plain CV_16U host batches and for homography batches.  Each batch is timed
with CUDA events recorded on the handle's stream before the continue / submit and after the submit; median and p10-p90 of
batches 1-3 over --reps sequences of each kind, alternated, after --warmup.  Reports the extra device time and the extra launches per continued
batch, with the card's name and power limit read in the same run.  Development aid, not a bench value; writes nothing.

usage: continue_probe.py [--frames 265] [--batches 4] [--nfeatures 2000] [--reps 5] [--warmup 1]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from orb_slam2_ssd_semantic_b200 import StreamTracker, synth  # noqa: E402

FACTOR = np.float32(1.0 / synth.DEPTH_FACTOR)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def frames(n, seed=1234):
    """n RoomStream frames, rendered by a process pool (about 0.08 s per 640 x 480 frame on one core)."""
    from multiprocessing import Pool
    rs = synth.RoomStream(seed=seed, n=n)
    with Pool(min(16, os.cpu_count() or 1)) as pool:
        fr = pool.map(rs.frame, range(n), chunksize=8)
    gray = np.stack([f[0] for f in fr])
    d16 = np.rint(np.stack([f[1] for f in fr]).astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    T = np.stack([f[3] for f in fr]).astype(np.float32).reshape(n, 16)
    return gray, d16, T


def sequence(st, submit, batches, F, cont):
    """One pass over the batches -> per batch (device ms, launches)."""
    s = torch.cuda.ExternalStream(st.stream())
    out = []
    for k in range(batches):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = st.launch_count()
        a.record(s)
        if cont and k:
            st.continue_after(st)
        submit(st, k)
        b.record(s)
        st.sync()
        out.append((a.elapsed_time(b), st.launch_count() - n0))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=265)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--nfeatures", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("continue_probe: no CUDA device")
    F, nb = a.frames, a.batches
    gray, d16, T = frames(F * nb)
    keep = [torch.from_numpy(np.ascontiguousarray(x)).pin_memory() for x in (gray, d16, T)]
    g, d, tt = (k.numpy() for k in keep)
    res = dict(card=card(), frames_per_batch=F, batches=nb, nfeatures=a.nfeatures)
    st = StreamTracker(a.nfeatures, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, 15.0, 0.9,
                       max_frames=F)
    out = st.alloc_outputs(F, pinned=True)
    sl = lambda k: slice(k * F, (k + 1) * F)  # noqa: E731
    forms = dict(
        plain_u16=lambda st, k: st.submit_batch_u16(g[sl(k)], d[sl(k)], FACTOR, tt[sl(k)], out),
        homography=lambda st, k: st.submit_batch_u16_homography(g[sl(k)], d[sl(k)], FACTOR, tt[sl(k)], 40.0, out))
    for name, submit in forms.items():
        r, got = {}, {False: ([], []), True: ([], [])}
        for rep in range(a.warmup + a.reps):   # the two ways alternate, so that both see the same machine
            for cont in (False, True):
                seq = sequence(st, submit, nb, F, cont)
                if rep >= a.warmup:
                    got[cont][0].extend(m for m, _ in seq[1:])
                    got[cont][1].extend(n for _, n in seq[1:])
        for cont, (ms, launches) in got.items():
            ms = np.array(ms)
            r["continued" if cont else "independent"] = dict(
                median_ms=float(np.median(ms)), p10_ms=float(np.percentile(ms, 10)), p90_ms=float(np.percentile(ms, 90)),
                launches=sorted(set(launches)))
        ind, con = r["independent"], r["continued"]
        r["extra_ms_per_batch"] = con["median_ms"] - ind["median_ms"]
        r["extra_launches_per_batch"] = [c - i for c, i in zip(con["launches"], ind["launches"])]
        res[name] = r
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
