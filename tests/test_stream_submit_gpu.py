"""orbs_submit refuses every batch outside its seven forms with B200ORB_EINVAL before it enqueues anything or changes the
handle: no launch, the last batch's results and dynamic masks still readable, and the next valid batch byte-identical to
the same batch on a fresh handle."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth

pytestmark = pytest.mark.gpu

F, ROWS, COLS = 3, 480, 640
EINVAL = -1


def _tracker():
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    return StreamTracker(1000, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, th=15.0, nnratio=0.9,
                         max_frames=F)


@pytest.fixture(scope="module")
def data():
    import torch
    ws = synth.WallStream(seed=77, n=F, h=ROWS, w=COLS)
    frames = [ws.frame(t) for t in range(F)]
    gray = np.stack([f[0] for f in frames])
    depth = np.stack([f[1] for f in frames]).astype(np.float32)
    d16 = np.rint(depth.astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    T = np.ascontiguousarray(np.stack([f[3] for f in frames]), np.float32)
    flow = np.stack([np.zeros((ROWS // 2, COLS // 2, 2), np.float32)] +
                    [synth.flow_field(300 + t, ROWS // 2, COLS // 2, blobs=6) for t in range(1, F)]).astype(np.float32)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in
           dict(gray=gray, depth=depth, d16=d16.view(np.int16), T=T, flow=flow).items()}
    return dict(gray=gray, depth=depth, d16=d16, T=T, flow=flow, prev=np.ascontiguousarray(gray[0]), dev=dev)


def _valid(st, d):
    """The batch every handle runs after the refusals: CV_16U depth and the caller's flow (uploads, the depth gather,
    the dynamic-mask block and the mask kernel)."""
    outs = st.track_batch_u16_masked(d["gray"], d["d16"], np.float32(1.0 / synth.DEPTH_FACTOR), d["T"], d["flow"], 40.0)
    glue = [st.frame_glue(t, int(outs[2][t])) for t in range(F)]
    masks = [st.dynamic_mask(t) for t in range(F)]
    return outs, glue, masks


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


# (id, batch fields, host results given) -- each one a combination outside the seven forms
REFUSED = [
    ("host_f32_flow", lambda d: _host(d, depth=_ptr(d, "depth"), depth_u16=None, flow=_ptr(d, "flow")), True),
    ("host_f32_device_flow", lambda d: _host(d, depth=_ptr(d, "depth"), depth_u16=None, device_flow=1), True),
    ("host_flow_and_device_flow", lambda d: _host(d, flow=_ptr(d, "flow"), device_flow=1), True),
    ("host_both_depths", lambda d: _host(d, depth=_ptr(d, "depth")), True),
    ("host_no_depth", lambda d: _host(d, depth_u16=None), True),
    ("host_prev_gray_without_device_flow", lambda d: _host(d, prev_gray=_ptr(d, "prev")), True),
    ("host_prev_gray_with_flow", lambda d: _host(d, flow=_ptr(d, "flow"), prev_gray=_ptr(d, "prev")), True),
    ("host_no_gray", lambda d: _host(d, gray=None), True),
    ("host_no_Tcw", lambda d: _host(d, Tcw=None), True),
    ("host_zero_frames", lambda d: _host(d, nframes=0), True),
    ("host_negative_rows", lambda d: _host(d, rows=-ROWS), True),
    ("host_zero_cols", lambda d: _host(d, cols=0), True),
    ("host_without_results", lambda d: _host(d), False),
    ("device_u16", lambda d: _device(d, depth=None, depth_u16=d["dev"]["d16"].data_ptr()), False),
    ("device_u16_flow", lambda d: _device(d, depth=None, depth_u16=d["dev"]["d16"].data_ptr(),
                                          flow=d["dev"]["flow"].data_ptr()), False),
    ("device_device_flow", lambda d: _device(d, device_flow=1), False),
    ("device_flow_and_device_flow", lambda d: _device(d, flow=d["dev"]["flow"].data_ptr(), device_flow=1), False),
    ("device_both_depths", lambda d: _device(d, depth_u16=d["dev"]["d16"].data_ptr()), False),
    ("device_no_depth", lambda d: _device(d, depth=None), False),
    ("device_no_gray", lambda d: _device(d, gray=None), False),
    ("device_zero_frames", lambda d: _device(d, nframes=0), False),
    ("device_with_results", lambda d: _device(d), True),
]


@pytest.fixture(scope="module")
def fresh(data):
    return _valid(_tracker(), data)


@pytest.mark.parametrize("case", [c[0] for c in REFUSED])
def test_refused_batch_changes_nothing(data, fresh, case):
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200._abi import OrbsBatch, OrbsResults, ptr
    make, with_out = next((m, o) for c, m, o in REFUSED if c == case)

    def refuse(st):
        outs = st.alloc_outputs(F)
        res = OrbsResults(*[ptr(a) for a in outs], st.cap)
        n0 = st.launch_count()
        rc = st._L.orbs_submit(st._h, C.byref(OrbsBatch(**make(data))), C.byref(res) if with_out else None)
        assert rc == EINVAL, _lib.lib().b200orb_last_error()
        st.sync()
        assert st.launch_count() == n0
        assert all(a.tobytes() == np.zeros_like(a).tobytes() for a in outs)

    st = _tracker()            # refused before its first batch
    refuse(st)
    _same(_valid(st, data), fresh)
    refuse(st)                 # and after one: the last batch's results and masks stay readable and unchanged
    _same((fresh[0], [st.frame_glue(t, int(fresh[0][2][t])) for t in range(F)], [st.dynamic_mask(t) for t in range(F)]),
          fresh)
    _same(_valid(st, data), fresh)


def test_null_handle_and_batch_refused(data):
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200._abi import OrbsBatch
    st = _tracker()
    L, n0 = _lib.lib(), st.launch_count()
    assert L.orbs_submit(None, C.byref(OrbsBatch(**_device(data))), None) == EINVAL
    assert L.orbs_submit(st._h, None, None) == EINVAL
    assert st.launch_count() == n0
