"""Where the host-buffer (e2e) path spends its time: one 256-frame batch through each entry alone, host clock around a
call that waits.  Development aid (not a bench value).  usage: e2e_probe.py [frames] [nfeatures]"""
import sys, time
import numpy as np
sys.path.insert(0, ".")
import torch
from orb_slam2_ssd_semantic_b200 import PointCloudMapping, StreamTracker, synth

F = int(sys.argv[1]) if len(sys.argv) > 1 else 256
nfeat = int(sys.argv[2]) if len(sys.argv) > 2 else 2000
rs = synth.RoomStream(seed=1234, n=F)
fr = [rs.frame(t, with_label=True) for t in range(F)]
pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
gray_h, depth_f = np.stack([f[0] for f in fr]), np.stack([f[1] for f in fr])
d16_h = np.rint(depth_f.astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
rgb_h, lab_h = np.stack([f[2] for f in fr]), np.stack([f[4] for f in fr])
Th = np.stack([f[3] for f in fr]).astype(np.float32)
p_gray, p_d16, p_T = pin(gray_h), pin(d16_h), pin(Th)
kfs = list(range(0, F, 12))
p_kd, p_kc, p_kl = pin(d16_h[kfs]), pin(rgb_h[kfs]), pin(lab_h[kfs])
gray, depth = p_gray.cuda(), torch.from_numpy(depth_f).cuda()
rgb, lab, T = torch.from_numpy(rgb_h).cuda(), torch.from_numpy(lab_h).cuda(), p_T.cuda()
factor = np.float32(1.0 / synth.DEPTH_FACTOR)
st = StreamTracker(nfeat, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, max_frames=F)
st.set_chunk_frames(F)
out = st.alloc_outputs(F, pinned=True)
pcm = PointCloudMapping(0.05)


def timeit(name, fn, n=6):
    fn(); torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    print("%-44s %7.3f ms" % (name, (time.perf_counter() - t0) / n * 1e3), flush=True)


def dev():
    st.track_batch_device(gray.data_ptr(), depth.data_ptr(), T.data_ptr(), F, 480, 640); st.sync()
def host():
    st.track_batch_u16(p_gray.numpy(), p_d16.numpy(), factor, p_T.numpy(), out)
def host_pageable_depth():
    st.track_batch_u16(p_gray.numpy(), d16_h, factor, p_T.numpy(), out)
def kdev():
    pcm.insert_keyframes_device(depth.data_ptr(), rgb.data_ptr(), 480, 640, kfs, Th[kfs], synth.FX, synth.FY, synth.CX, synth.CY,
                                d_label=lab.data_ptr()); pcm.sync()
def khost():
    pcm.insert_keyframes_u16(p_kd.numpy(), p_kc.numpy(), factor, Th[kfs], synth.FX, synth.FY, synth.CX, synth.CY, label=p_kl.numpy()); pcm.sync()
def h2d():
    gray.copy_(p_gray, non_blocking=True); torch.cuda.synchronize()
dback = [torch.empty(a.shape, dtype=torch.uint8).pin_memory() if False else None for a in ()]

timeit("tracker, inputs resident", dev)
timeit("tracker, host buffers (page-locked depth)", host)
timeit("tracker, host buffers (pageable depth)", host_pageable_depth)
timeit("gray H2D alone (%.1f MB)" % (gray_h.nbytes / 1e6), h2d)
timeit("mapper, inputs resident (%d kf)" % len(kfs), kdev)
timeit("mapper, host buffers", khost)
st.profile_enable(True)
for _ in range(3):
    host()
ms, frames, runs = st.profile_read()
print({k: round(v / runs, 3) for k, v in ms.items()}, "ms per batch, host path")
for _ in range(3):
    dev()
ms, frames, runs = st.profile_read()
print({k: round(v / runs, 3) for k, v in ms.items()}, "ms per batch, device path")
print("outputs D2H bytes:", sum(a.nbytes for a in out))
