"""The dense flow on the device (dynm_farneback, dynm_flow_batch_device, orbs_*_u16_flow) against the restatement
oracle/farneback_py.py (pinned to cv2 4.13 at baseline dispatch by tests/test_farneback_cpu.py), bit for bit, and the
masked tracker fed by it against the masked tracker fed the restatement's flow."""
import glob
import os

import numpy as np
import pytest

from oracle import farneback_py as FB
from tests import flow_scenes as S

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _same(a, b):
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape
    assert (a.view(np.uint32) == b.view(np.uint32)).all(), "max |diff| %g" % np.abs(a.astype(np.float64) - b).max()


@pytest.fixture(scope="module")
def dm():
    from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask
    return DynamicMask(0)


def _oracle_flows(gray, prev=None):
    """-> [n][rows/2][cols/2][2]: zero field for frame 0 without prev, else the restatement of each consecutive pair."""
    n, rows, cols = gray.shape
    h, w = rows // 2, cols // 2
    half = [FB.pyr_down(g, h, w) for g in gray]
    out = [FB.farneback(FB.pyr_down(prev, h, w), half[0]) if prev is not None else np.zeros((h, w, 2), np.float32)]
    out += [FB.farneback(half[t - 1], half[t]) for t in range(1, n)]
    return np.stack(out)


@pytest.mark.parametrize("rows,cols", S.HALF_SIZES)
@pytest.mark.parametrize("scene", S.SCENES)
def test_farneback_equals_restatement(dm, scene, rows, cols):
    g = S.frames(scene, 2 * rows, 2 * cols, 2)
    prev, cur = FB.pyr_down(g[0], rows, cols), FB.pyr_down(g[1], rows, cols)
    _same(dm.farneback(prev, cur), FB.farneback(prev, cur))


def test_farneback_equals_goldens(dm):
    files = sorted(glob.glob(os.path.join(GOLDEN, "farneback_*.npz")))
    assert files
    for f in files:
        z = np.load(f)
        _same(dm.farneback(z["prev"], z["cur"]), z["flow"])


def _flow_batch(dm, gray, prev=None):
    import torch
    n, rows, cols = gray.shape
    g = torch.from_numpy(np.ascontiguousarray(gray)).cuda()
    p = torch.from_numpy(np.ascontiguousarray(prev)).cuda() if prev is not None else None
    out = torch.full((n, rows // 2, cols // 2, 2), float("nan"), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    dm.flow_batch_device(g.data_ptr(), p.data_ptr() if p is not None else None, n, rows, cols, out.data_ptr())
    dm.sync()
    return out.cpu().numpy()


@pytest.mark.parametrize("scene,rows,cols", [("room", 480, 640), ("blobs", 195, 323), ("border", 128, 160)])
def test_flow_batch_device_equals_restatement(dm, scene, rows, cols):
    seq = S.frames(scene, rows, cols, 4)
    _same(_flow_batch(dm, seq[1:]), _oracle_flows(seq[1:]))
    _same(_flow_batch(dm, seq[1:], seq[0]), _oracle_flows(seq[1:], seq[0]))
    assert not _flow_batch(dm, seq[1:])[0].any()


def test_flow_batch_device_across_frame_chunks(dm):
    """More frames than one pass through the scratch holds (64): pairs that straddle a chunk boundary."""
    seq = S.frames("blobs", 64, 80, 131)
    _same(_flow_batch(dm, seq[1:], seq[0]), _oracle_flows(seq[1:], seq[0]))
    _same(_flow_batch(dm, seq[:65]), _oracle_flows(seq[:65]))


def test_flow_batch_then_masked_device_equals_masked_with_oracle_flow(dm):
    """dynm_flow_batch_device composed with track_batch_masked_device == the masked path fed the restatement's flow."""
    import torch
    from tests.test_masked_tracking_gpu import _batch, _device_out, _same as same_out, _tracker
    F = 4
    gray, d16, depth, factor, T = _batch(1234, F)
    st = _tracker(2000, F)
    want = [x.copy() for x in st.track_batch_u16_masked(gray, d16, factor, T, _oracle_flows(gray), 40.0)]
    masks = [st.dynamic_mask(t) for t in range(F)]
    g, d, t = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (gray, depth, T.astype(np.float32)))
    fl = torch.empty((F, 240, 320, 2), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    dm.flow_batch_device(g.data_ptr(), None, F, 480, 640, fl.data_ptr())
    dm.sync()
    dev = _tracker(2000, F)
    dev.track_batch_masked_device(g.data_ptr(), d.data_ptr(), t.data_ptr(), fl.data_ptr(), 40.0, F, 480, 640)
    dev.sync()
    same_out(want, _device_out(dev, F))
    for k in range(F):
        m, f = dev.dynamic_mask(k)
        assert (m == masks[k][0]).all() and f == masks[k][1]


def _masked_flow_scene(F, seed=1234):
    """The scene of test_masked_tracking_gpu.py with a textured disc moving 16 px per frame over the wall (8 px at half
    resolution, above the sqrt(40) px threshold), so some masks are not all ones."""
    from tests.test_masked_tracking_gpu import _batch
    gray, d16, depth, factor, T = _batch(seed, F)
    tex = S.frames("identical", 480, 640, 1, seed=seed)[0]
    yy, xx = np.mgrid[0:480, 0:640]
    for t in range(F):
        m = (yy - 240) ** 2 + (xx - 160 - 16 * t) ** 2 < 90 ** 2
        gray[t][m] = np.roll(tex, 16 * t, axis=1)[m]
    return gray, d16, depth, factor, T


def test_track_flow_equals_masked_with_oracle_flow():
    """track_batch_u16_flow == track_batch_u16_masked fed the restatement's flow, 2000 features: every output and
    every frame's dynamic mask; then two batches chained by prev_gray == one batch of twice the frames."""
    from tests.test_masked_tracking_gpu import _same as same_out, _tracker
    F = 6
    gray, d16, _, factor, T = _masked_flow_scene(F)
    flow = _oracle_flows(gray)
    a, b = _tracker(2000, F), _tracker(2000, F)
    want = [x.copy() for x in a.track_batch_u16_masked(gray, d16, factor, T, flow, 40.0)]
    got = [x.copy() for x in b.track_batch_u16_flow(gray, d16, factor, T, None, 40.0)]
    same_out(want, got)
    masks = []
    for t in range(F):
        ma, fa = a.dynamic_mask(t)
        mb, fb = b.dynamic_mask(t)
        assert (ma == mb).all() and fa == fb, t
        masks.append(ma)
    assert min(m.mean() for m in masks) < 0.97
    h = F // 2
    first = [x.copy() for x in b.track_batch_u16_flow(gray[:h], d16[:h], factor, T[:h], None, 40.0)]
    m1 = [b.dynamic_mask(t)[0] for t in range(h)]
    second = [x.copy() for x in b.track_batch_u16_flow(gray[h:], d16[h:], factor, T[h:], gray[h - 1], 40.0)]
    m2 = [b.dynamic_mask(t)[0] for t in range(F - h)]
    for t in range(F):
        m = (m1 + m2)[t]
        assert (m == masks[t]).all(), t
    n = got[2]
    assert (first[2] == n[:h]).all() and (second[2] == n[h:]).all()
    for k, part in ((0, first), (h, second)):
        for t in range(len(part[2])):
            c = part[2][t]
            assert part[0][t, :c].tobytes() == got[0][k + t, :c].tobytes() and (part[1][t, :c] == got[1][k + t, :c]).all()
            if t > 0:
                assert (part[3][t, :c] == got[3][k + t, :c]).all() and part[4][t] == got[4][k + t]


def test_submit_flow_on_chained_handles_equals_track_form():
    """submit_batch_u16_flow on two alternating handles chained with orbs_chain_after, each batch carrying the last
    gray frame of the batch before as prev_gray == track_batch_u16_flow, batch by batch."""
    import torch
    from tests.test_masked_tracking_gpu import _same as same_out, _tracker
    F, B = 3, 3
    gray, d16, _, factor, T = _masked_flow_scene(F * B, seed=77)
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    batches = [(pin(gray[k * F:(k + 1) * F]), pin(d16[k * F:(k + 1) * F]), pin(T[k * F:(k + 1) * F].astype(np.float32)),
                pin(gray[k * F - 1]) if k else None) for k in range(B)]
    ref = _tracker(1000, F)
    want = [[x.copy() for x in ref.track_batch_u16_flow(g.numpy(), d.numpy(), factor, t.numpy(),
                                                        None if p is None else p.numpy(), 40.0)] for g, d, t, p in batches]
    trk = [_tracker(1000, F), _tracker(1000, F)]
    outs = [t.alloc_outputs(F, pinned=True) for t in trk]
    got = []
    for k, (g, d, t, p) in enumerate(batches):
        if k >= 2:
            trk[k & 1].sync()
            got.append([x.copy() for x in outs[k & 1]])
        trk[k & 1].chain_after(trk[(k + 1) & 1])
        trk[k & 1].submit_batch_u16_flow(g.numpy(), d.numpy(), factor, t.numpy(), None if p is None else p.numpy(), 40.0,
                                         outs[k & 1])
    for k in range(B - 2, B):
        trk[k & 1].sync()
        got.append([x.copy() for x in outs[k & 1]])
    for w, g in zip(want, got):
        same_out(w, g)


def test_rejected_sizes_and_nulls(dm):
    """B200ORB_EINVAL before anything is enqueued: no launch is counted."""
    import ctypes as C
    from orb_slam2_ssd_semantic_b200 import _lib
    from tests.test_masked_tracking_gpu import _tracker
    L = _lib.lib()
    EINVAL = -1
    n0 = dm.launch_count()
    img = np.zeros((15, 40), np.uint8)
    f = np.zeros((15, 40, 2), np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert L.dynm_farneback(dm._h, p(img), p(img), 15, 40, p(f)) == EINVAL
    big = np.zeros((16, 2049), np.uint8)
    assert L.dynm_farneback(dm._h, p(big), p(big), 16, 2049, p(np.zeros((16, 2049, 2), np.float32))) == EINVAL
    ok = np.zeros((16, 16), np.uint8)
    assert L.dynm_farneback(dm._h, None, p(ok), 16, 16, p(f)) == EINVAL
    assert L.dynm_farneback(dm._h, p(ok), p(ok), 16, 16, None) == EINVAL
    assert L.dynm_farneback(None, p(ok), p(ok), 16, 16, p(f)) == EINVAL
    d = C.c_void_p(1 << 40)   # never dereferenced: the geometry is rejected first
    assert L.dynm_flow_batch_device(dm._h, d, None, 2, 31, 64, d) == EINVAL
    assert L.dynm_flow_batch_device(dm._h, d, None, 2, 64, 4098, d) == EINVAL
    assert L.dynm_flow_batch_device(dm._h, None, None, 2, 64, 64, d) == EINVAL
    assert L.dynm_flow_batch_device(dm._h, d, None, 2, 64, 64, None) == EINVAL
    assert L.dynm_flow_batch_device(dm._h, d, None, -1, 64, 64, d) == EINVAL
    assert dm.launch_count() == n0
    st = _tracker(1000, 2)
    n1 = st.launch_count()
    gray = np.zeros((2, 30, 64), np.uint8)
    with pytest.raises(Exception):
        st.track_batch_u16_flow(gray, np.zeros(gray.shape, np.uint16), 1.0, np.tile(np.eye(4, dtype=np.float32), (2, 1, 1)))
    with pytest.raises(ValueError):
        st.track_batch_u16_flow(np.zeros((2, 64, 64), np.uint8), np.zeros((2, 64, 64), np.uint16), 1.0,
                                np.tile(np.eye(4, dtype=np.float32), (2, 1, 1)), np.zeros((64, 63), np.uint8))
    assert st.launch_count() == n1


def test_flow_mirror_with_device_flow_equals_restatement(dm):
    """Flow(flow_fn=dm.farneback).ComputeMask == the mirror fed the restatement's flow."""
    from orb_slam2_ssd_semantic_b200.dynmask import Flow
    seq = S.frames("blobs", 240, 320, 3)
    half = lambda g: FB.pyr_down(g, g.shape[0] // 2, g.shape[1] // 2)
    a = Flow(flow_fn=dm.farneback, pyr_down_fn=half)
    b = Flow(flow_fn=FB.farneback, pyr_down_fn=half)
    for g in seq:
        assert (a.ComputeMask(g) == b.ComputeMask(g)).all()
