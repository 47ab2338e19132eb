"""orbs_submit refuses every batch outside its eight forms with B200ORB_EINVAL, and a results buffer below the batch's
keypoint capacity with B200ORB_ECAP, before it enqueues anything or changes the handle: no launch, the last batch's
results and dynamic masks still readable, the handle still continuing that batch exactly like the unsplit sequence, and
the next valid batch byte-identical to the same batch on a fresh handle.  The readers take only frames of the last
batch, and a submit that fails after its refusals leaves the handle with no batch and usable."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth

pytestmark = pytest.mark.gpu

F, ROWS, COLS = 4, 480, 640
EINVAL, ECAP, ECUDA = -1, -2, -3
FACTOR = np.float32(1.0 / synth.DEPTH_FACTOR)


def _tracker(max_frames=F):
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    return StreamTracker(1000, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, th=15.0, nnratio=0.9,
                         max_frames=max_frames)


@pytest.fixture(scope="module")
def data():
    """2 F frames: the valid batch is the first F, the batch that continues it the next F."""
    import torch
    ws = synth.WallStream(seed=77, n=2 * F, h=ROWS, w=COLS)
    frames = [ws.frame(t) for t in range(2 * F)]
    gray = np.stack([f[0] for f in frames])
    depth = np.stack([f[1] for f in frames]).astype(np.float32)
    d16 = np.rint(depth.astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    T = np.ascontiguousarray(np.stack([f[3] for f in frames]), np.float32)
    flow = np.stack([np.zeros((ROWS // 2, COLS // 2, 2), np.float32)] +
                    [synth.flow_field(300 + t, ROWS // 2, COLS // 2, blobs=6) for t in range(1, 2 * F)])
    flow = flow.astype(np.float32)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in
           dict(gray=gray, depth=depth, d16=d16.view(np.int16), T=T, flow=flow).items()}
    return dict(gray=gray, depth=depth, d16=d16, T=T, flow=flow, prev=np.ascontiguousarray(gray[0]), dev=dev)


def _masked(st, d, a, b):
    """Frames [a, b) as one batch with CV_16U depth and the caller's flow (uploads, the depth gather, the dynamic-mask
    block and the mask kernel), waited for."""
    return st.track_batch_u16_masked(d["gray"][a:b], d["d16"][a:b], FACTOR, d["T"][a:b], d["flow"][a:b], 40.0)


def _valid(st, d):
    """The batch every handle runs after the refusals: the first F frames."""
    outs = _masked(st, d, 0, F)
    glue = [st.frame_glue(t, int(outs[2][t])) for t in range(F)]
    masks = [st.dynamic_mask(t) for t in range(F)]
    return outs, glue, masks


def _records(st, outs, masked=True):
    """Per frame of the last batch: its first nkp keypoints, descriptors and cur2last, nmatch, glue and mask."""
    kps, desc, nkp, c2l, nm = outs
    recs = []
    for t, n in enumerate(int(x) for x in nkp):
        rec = (kps[t, :n].tobytes(), desc[t, :n].tobytes(), c2l[t, :n].tobytes(), int(nm[t]),
               tuple(x.tobytes() for x in st.frame_glue(t, n)))
        if masked:
            m, f = st.dynamic_mask(t)
            rec += (m.tobytes(), f)
        recs.append(rec)
    return recs


def _same(a, b):
    (oa, ga, ma), (ob, gb, mb) = a, b
    for x, y in zip(oa, ob):
        assert x.tobytes() == y.tobytes()
    for x, y in zip(ga, gb):
        assert all(u.tobytes() == v.tobytes() for u, v in zip(x, y))
    for (m1, f1), (m2, f2) in zip(ma, mb):
        assert m1.tobytes() == m2.tobytes() and f1 == f2


def _host(d, **kw):
    from orb_slam2_ssd_semantic_b200._abi import ptr
    b = dict(nframes=F, rows=ROWS, cols=COLS, device=0, gray=ptr(d["gray"]), depth=None, depth_u16=ptr(d["d16"]),
             depth_factor=1.0 / synth.DEPTH_FACTOR, Tcw=ptr(d["T"]), flow=None, device_flow=0, prev_gray=None,
             binary_threshold=40.0)
    b.update(kw)
    return b


def _device(d, **kw):
    g = d["dev"]
    b = dict(nframes=F, rows=ROWS, cols=COLS, device=1, gray=g["gray"].data_ptr(), depth=g["depth"].data_ptr(),
             depth_u16=None, depth_factor=0.0, Tcw=g["T"].data_ptr(), flow=None, device_flow=0, prev_gray=None,
             binary_threshold=40.0)
    b.update(kw)
    return b


def _ptr(d, k):
    from orb_slam2_ssd_semantic_b200._abi import ptr
    return ptr(d[k])


# (id, batch fields, host results (None: none; else their cap is the handle's plus this), return code) -- each one a
# combination outside the eight forms, or a results buffer one keypoint short
REFUSED = [
    ("host_f32_flow", lambda d: _host(d, depth=_ptr(d, "depth"), depth_u16=None, flow=_ptr(d, "flow")), 0, EINVAL),
    ("host_f32_device_flow", lambda d: _host(d, depth=_ptr(d, "depth"), depth_u16=None, device_flow=1), 0, EINVAL),
    ("host_flow_and_device_flow", lambda d: _host(d, flow=_ptr(d, "flow"), device_flow=1), 0, EINVAL),
    ("host_both_depths", lambda d: _host(d, depth=_ptr(d, "depth")), 0, EINVAL),
    ("host_no_depth", lambda d: _host(d, depth_u16=None), 0, EINVAL),
    ("host_prev_gray_without_device_flow", lambda d: _host(d, prev_gray=_ptr(d, "prev")), 0, EINVAL),
    ("host_prev_gray_with_flow", lambda d: _host(d, flow=_ptr(d, "flow"), prev_gray=_ptr(d, "prev")), 0, EINVAL),
    ("host_no_gray", lambda d: _host(d, gray=None), 0, EINVAL),
    ("host_no_Tcw", lambda d: _host(d, Tcw=None), 0, EINVAL),
    ("host_zero_frames", lambda d: _host(d, nframes=0), 0, EINVAL),
    ("host_negative_rows", lambda d: _host(d, rows=-ROWS), 0, EINVAL),
    ("host_zero_cols", lambda d: _host(d, cols=0), 0, EINVAL),
    ("host_without_results", lambda d: _host(d), None, EINVAL),
    ("device_u16", lambda d: _device(d, depth=None, depth_u16=d["dev"]["d16"].data_ptr()), None, EINVAL),
    ("device_u16_flow", lambda d: _device(d, depth=None, depth_u16=d["dev"]["d16"].data_ptr(),
                                          flow=d["dev"]["flow"].data_ptr()), None, EINVAL),
    ("device_device_flow", lambda d: _device(d, device_flow=1), None, EINVAL),
    ("device_flow_and_device_flow", lambda d: _device(d, flow=d["dev"]["flow"].data_ptr(), device_flow=1), None,
     EINVAL),
    ("device_both_depths", lambda d: _device(d, depth_u16=d["dev"]["d16"].data_ptr()), None, EINVAL),
    ("device_no_depth", lambda d: _device(d, depth=None), None, EINVAL),
    ("device_no_gray", lambda d: _device(d, gray=None), None, EINVAL),
    ("device_zero_frames", lambda d: _device(d, nframes=0), None, EINVAL),
    ("device_with_results", lambda d: _device(d), 0, EINVAL),
    # more frames than the handle has held: refused before the blocks of the larger batch are carved
    ("host_cap_short_more_frames", lambda d: _host(d, nframes=2 * F, flow=_ptr(d, "flow")), -1, ECAP),
]


@pytest.fixture(scope="module")
def fresh(data):
    return _valid(_tracker(), data)


@pytest.fixture(scope="module")
def unsplit(data):
    """Frames F .. 2 F - 1 of the 2 F frames tracked as one batch: what a batch continuing the valid batch gives."""
    st = _tracker(2 * F)
    return _records(st, _masked(st, data, 0, 2 * F))[F:]


@pytest.mark.parametrize("case", [c[0] for c in REFUSED])
def test_refused_batch_changes_nothing(data, fresh, unsplit, case):
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200._abi import OrbsBatch, OrbsResults, ptr
    make, out_cap, want_rc = next((m, o, r) for c, m, o, r in REFUSED if c == case)

    def refuse(st):
        outs = st.alloc_outputs(2 * F)
        res = OrbsResults(*[ptr(a) for a in outs], st.cap + (out_cap or 0))
        n0 = st.launch_count()
        rc = st._L.orbs_submit(st._h, C.byref(OrbsBatch(**make(data))), None if out_cap is None else C.byref(res))
        assert rc == want_rc, _lib.lib().b200orb_last_error()
        st.sync()
        assert st.launch_count() == n0
        assert all(a.tobytes() == np.zeros_like(a).tobytes() for a in outs)

    first = _tracker()         # refused before its first batch
    refuse(first)
    _same(_valid(first, data), fresh)
    # and after one, on a handle that has held only its F frames: the last batch's results and masks stay readable and
    # unchanged, the next batch equals a fresh handle's, and the handle continues its last batch as if the refused one had
    # never come
    st = _tracker()
    _same(_valid(st, data), fresh)
    refuse(st)
    _same((fresh[0], [st.frame_glue(t, int(fresh[0][2][t])) for t in range(F)], [st.dynamic_mask(t) for t in range(F)]),
          fresh)
    _same(_valid(st, data), fresh)
    refuse(st)
    st.continue_after(st)
    assert _records(st, _masked(st, data, F, 2 * F)) == unsplit


@pytest.mark.parametrize("form", ["u16", "masked", "homography"])
def test_readers_take_frames_of_the_last_batch_only(data, form):
    """A 2 F-frame batch, then an F-frame batch on a handle of frame capacity 2 F: frame F belongs to the earlier batch
    only, so every reader of the last batch refuses it (and reads frame F - 1)."""
    from orb_slam2_ssd_semantic_b200 import B200OrbError
    d, st = data, _tracker(2 * F)
    for a, b in ((0, 2 * F), (F, 2 * F)):
        if form == "u16":
            st.track_batch_u16(d["gray"][a:b], d["d16"][a:b], FACTOR, d["T"][a:b])
        elif form == "masked":
            _masked(st, d, a, b)
        else:
            st.track_batch_u16_homography(d["gray"][a:b], d["d16"][a:b], FACTOR, d["T"][a:b], 40.0)
    readers = [lambda t: st.frame_glue(t, 1)]
    readers += [st.dynamic_mask] * (form != "u16") + [st.homography] * (form == "homography")
    for read in readers:
        read(F - 1)
        with pytest.raises(B200OrbError):
            read(F)


def _device_batch(st, d):
    g = d["dev"]
    st.track_batch_device(g["gray"].data_ptr(), g["depth"].data_ptr(), g["T"].data_ptr(), F, ROWS, COLS)
    st.sync()
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    from tests.test_extractor_gpu import _device_to_host
    (p_kps, p_desc, p_nkp, p_c2l, p_nm), cap = st.device_results()
    outs = (_device_to_host(p_kps, KP_DTYPE.itemsize * cap * F).view(KP_DTYPE).reshape(F, cap),
            _device_to_host(p_desc, 32 * cap * F).reshape(F, cap, 32), _device_to_host(p_nkp, 4 * F).view(np.int32),
            _device_to_host(p_c2l, 4 * cap * F).view(np.int32).reshape(F, cap),
            _device_to_host(p_nm, 4 * F).view(np.int32))
    return _records(st, outs, masked=False)


def test_failed_submit_leaves_no_batch(data):
    """A device batch of so many frames that the extractor's pyramid block exceeds the card: the handle's blocks are
    released, the allocation is refused (an ordinary error return, before any input is read) and the batch fails with
    B200ORB_ECUDA.  The handle then holds no batch -- no device results, no frame glue, nothing to continue -- and its
    next batch equals the same batch on a fresh handle."""
    import torch
    from orb_slam2_ssd_semantic_b200 import B200OrbError, _lib
    from orb_slam2_ssd_semantic_b200._abi import OrbsBatch
    L = _lib.lib()
    st, other = _tracker(), _tracker()
    _device_batch(st, data)
    want = _device_batch(other, data)
    huge = torch.cuda.mem_get_info()[1] // (2 * ROWS * COLS) + 1   # the raw and blurred level 0 alone exceed the card
    tiny = torch.zeros(64, dtype=torch.float32, device="cuda")
    b = _device(data, nframes=huge, gray=tiny.data_ptr(), depth=tiny.data_ptr(), Tcw=tiny.data_ptr())
    assert L.orbs_submit(st._h, C.byref(OrbsBatch(**b)), None) == ECUDA, L.b200orb_last_error()
    assert L.orbs_device_results(st._h, None, None, None, None, None, None) == EINVAL
    with pytest.raises(B200OrbError):
        st.frame_glue(0, 1)
    n0 = other.launch_count()
    assert L.orbs_continue(other._h, st._h) == EINVAL
    assert other.launch_count() == n0
    assert _device_batch(st, data) == want


def test_null_handle_and_batch_refused(data):
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200._abi import OrbsBatch
    st = _tracker()
    L, n0 = _lib.lib(), st.launch_count()
    assert L.orbs_submit(None, C.byref(OrbsBatch(**_device(data))), None) == EINVAL
    assert L.orbs_submit(st._h, None, None) == EINVAL
    assert st.launch_count() == n0
