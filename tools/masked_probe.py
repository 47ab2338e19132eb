"""What masked tracking costs on the bench's room workload (640 x 480, ORBextractor(2000, ...), 265-frame batches): unmasked
vs masked batches of the same frames, alternated and repeated, CUDA events around > 1 s of back-to-back batches with the
inputs resident in HBM; then the host-buffer form (two handles submitted alternately, page-locked inputs) timed with a host
clock around work that ends in a synchronise.  The flow has moving blobs, and every 5th frame a band that leaves at most
65 % of the mask at 1, so some frames are filtered and some are not.  Development aid, not a bench value; writes nothing.

usage: masked_probe.py [--frames 265] [--nfeatures 2000] [--reps 5] [--profile]
  --profile: one separate run under torch.profiler instead, printing the device time of the mask + filter kernel
  (k_dynm_plane_filter) per batch and per frame."""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def flows(F, seed=700):
    out = np.empty((F, 240, 320, 2), np.float32)
    for t in range(F):
        if t == 0:
            out[t] = 0.0                                   # no previous image: mask = ones
        else:
            out[t] = synth.flow_field(seed + t, 240, 320, blobs=6)
            if t % 5 == 0:
                out[t, :120, :, 0] += 50.0                 # half the image moving: the 65 % rule keeps every keypoint
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=265)
    ap.add_argument("--nfeatures", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    F, dev = a.frames, torch.device("cuda", 0)
    rs = synth.RoomStream(seed=1234, n=F)
    fr = [rs.frame(t) for t in range(F)]
    gray_h, depth_h = np.stack([f[0] for f in fr]), np.stack([f[1] for f in fr])
    T_h = np.stack([f[3] for f in fr]).astype(np.float32)
    flow_h = flows(F)
    d16_h = np.rint(depth_h.astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    factor = np.float32(1.0 / synth.DEPTH_FACTOR)
    gray, depth, T, flow = (torch.from_numpy(x).to(dev) for x in (gray_h, depth_h, T_h, flow_h))
    mk = lambda: StreamTracker(a.nfeatures, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, 15.0, 0.9, True, F)
    st = mk()
    ext = torch.cuda.ExternalStream(st.stream(), device=dev)

    def unmasked():
        st.track_batch_device(gray.data_ptr(), depth.data_ptr(), T.data_ptr(), F, 480, 640)

    def masked():
        st.track_batch_masked_device(gray.data_ptr(), depth.data_ptr(), T.data_ptr(), flow.data_ptr(), 40.0, F, 480, 640)

    torch.cuda.synchronize()
    for fn in (unmasked, masked, unmasked, masked):
        fn()
    st.sync()
    filtered = [st.dynamic_mask(t)[1] for t in range(F)]
    info = {"card": card(), "frames": F, "nfeatures": a.nfeatures, "filtered_frames": int(sum(filtered))}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        n = 10
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                masked()
            st.sync()
        ev = [e for e in prof.key_averages() if "k_dynm_plane_filter" in e.key]
        us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in ev) / n
        print(json.dumps(dict(info, mode="profile", mask_kernel_us_per_batch=round(us, 2),
                              mask_kernel_us_per_frame=round(us / F, 4), launches=sum(e.count for e in ev))))
        return

    def window(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ext)
        for _ in range(n):
            fn()
        e1.record(ext)
        st.sync()
        return e0.elapsed_time(e1)

    n = max(4, int(1.2e3 / (window(unmasked, 4) / 4)) + 1)    # > 1.2 s per timed window
    res = {"unmasked": [], "masked": []}
    for _ in range(a.reps):
        for name, fn in (("unmasked", unmasked), ("masked", masked)):
            res[name].append(F * n / (window(fn, n) / 1e3))
    out = dict(info, mode="device", batches_per_window=n)
    for k, v in res.items():
        out[k + "_fps_median"] = round(float(np.median(v)), 1)
        out[k + "_fps_min_max"] = [round(min(v), 1), round(max(v), 1)]
    out["masked_over_unmasked"] = round(out["masked_fps_median"] / out["unmasked_fps_median"], 4)
    print(json.dumps(out), flush=True)

    # host buffers, page-locked: two handles submitted alternately (upload | kernels | download overlap)
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x)).pin_memory()
    p_gray, p_d16, p_T, p_flow = pin(gray_h), pin(d16_h), pin(T_h), pin(flow_h)
    trk = [mk(), mk()]
    outs = [t.alloc_outputs(F, pinned=True) for t in trk]

    def run_host(masked_, nb):
        t0 = time.perf_counter()
        for k in range(nb):
            h = trk[k & 1]
            if k >= 2:
                h.sync()
            h.chain_after(trk[(k + 1) & 1])
            if masked_:
                h.submit_batch_u16_masked(p_gray.numpy(), p_d16.numpy(), factor, p_T.numpy(), p_flow.numpy(), 40.0, outs[k & 1])
            else:
                h.submit_batch_u16(p_gray.numpy(), p_d16.numpy(), factor, p_T.numpy(), outs[k & 1])
        trk[0].sync()
        trk[1].sync()
        return time.perf_counter() - t0

    run_host(False, 4)
    run_host(True, 4)
    nb = max(4, int(1.2 / (run_host(False, 4) / 4)) + 1)
    res = {"unmasked": [], "masked": []}
    for _ in range(a.reps):
        for name, m in (("unmasked", False), ("masked", True)):
            res[name].append(F * nb / run_host(m, nb))
    out = dict(info, mode="host_pinned_submit", batches_per_window=nb,
               flow_h2d_bytes_per_frame=int(flow_h[0].nbytes), gray_h2d_bytes_per_frame=int(gray_h[0].nbytes))
    for k, v in res.items():
        out[k + "_fps_median"] = round(float(np.median(v)), 1)
        out[k + "_fps_min_max"] = [round(min(v), 1), round(max(v), 1)]
    out["masked_over_unmasked"] = round(out["masked_fps_median"] / out["unmasked_fps_median"], 4)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
