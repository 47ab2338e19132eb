"""orbs_continue: one sequence tracked across batches.  The single batch is the oracle (pinned to the reference's sources
for plain and masked batches, and to tests/homography_chain_ref.py for homography batches), so a sequence split into
continued batches must give, frame for frame and bit for bit, what the unsplit batch gives:

  * test_plain_split / test_masked_split: 24 RoomStream frames in every host and device form, split (1, 23), (2, 22),
    (11, 13) and (8, 8, 8) on one handle continuing itself; keypoints, descriptors, counts, cur2last, nmatch, the frame
    glue and the dynamic masks; frame 0 of each continued batch finds matches;
  * test_device_flow_equals_prev_gray: a continued device_flow batch equals the same batch given prev_gray;
  * test_homography_split: the homography chain split (1, ..), (2, ..), (3, ..), at a frame whose predecessor warped and
    (1, 1, 1, ..), against homography_chain_ref.run over the whole sequence;
  * test_alternating_handles / test_prev_destroyed / test_chunk_size: two handles alternating with orbs_chain_after +
    orbs_continue, a prev destroyed right after orbs_continue, small upload chunks;
  * test_continuation_is_consumed: the batch after a continued one starts a new sequence;
  * test_refusals: every refused orbs_continue and continued orbs_submit returns EINVAL with no launch, no output and the
    pending continuation still usable."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth

pytestmark = pytest.mark.gpu

CAM = (synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
ROWS, COLS, N = 480, 640, 24
TH, THR = 15.0, 40.0
EINVAL = -1
FACTOR = np.float32(1.0 / synth.DEPTH_FACTOR)
SPLITS = [(1, 23), (2, 22), (11, 13), (8, 8, 8)]


def _tracker(max_frames=N, nfeatures=1000, th=TH):
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    return StreamTracker(nfeatures, 1.2, 8, 20, 7, *CAM, th=th, nnratio=0.9, max_frames=max_frames)


@pytest.fixture(scope="module")
def room():
    import torch
    rs = synth.RoomStream(seed=11, n=N)
    fr = [rs.frame(t) for t in range(N)]
    gray = np.ascontiguousarray(np.stack([f[0] for f in fr]))
    d16 = np.rint(np.stack([f[1] for f in fr]).astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    depth = d16.astype(np.float32) * FACTOR
    T = np.ascontiguousarray(np.stack([f[3] for f in fr]), np.float32)
    h, w = ROWS // 2, COLS // 2
    flow = np.stack([np.zeros((h, w, 2), np.float32)] + [synth.flow_field(500 + t, h, w, blobs=6) for t in range(1, N)])
    flow = np.ascontiguousarray(flow, np.float32)
    d = dict(gray=gray, d16=d16, depth=depth, T=T, flow=flow)
    d["dev"] = {k: torch.from_numpy(d[k]).cuda() for k in ("gray", "depth", "T", "flow")}
    d["pin"] = {k: torch.from_numpy(d[k]).pin_memory() for k in ("gray", "d16", "T")}
    return d


def _pinned_outputs(st, F):
    import torch
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    keep, outs = [], []
    for s, dt in [((F, st.cap), KP_DTYPE), ((F, st.cap, 32), np.uint8), ((F,), np.int32), ((F, st.cap), np.int32),
                  ((F,), np.int32)]:
        t = torch.zeros(int(np.prod(s)) * np.dtype(dt).itemsize, dtype=torch.uint8).pin_memory()
        keep.append(t)
        outs.append(t.numpy().view(dt).reshape(s))
    return keep, tuple(outs)


def _device_outputs(st, F):
    from tests.test_extractor_gpu import _device_to_host
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    (p_kps, p_desc, p_nkp, p_c2l, p_nm), cap = st.device_results()
    return (_device_to_host(p_kps, KP_DTYPE.itemsize * cap * F).view(KP_DTYPE).reshape(F, cap),
            _device_to_host(p_desc, 32 * cap * F).reshape(F, cap, 32), _device_to_host(p_nkp, 4 * F).view(np.int32),
            _device_to_host(p_c2l, 4 * cap * F).view(np.int32).reshape(F, cap), _device_to_host(p_nm, 4 * F).view(np.int32))


def _submit(form, st, d, a, b):
    """Frames [a, b) of the sequence as one batch of `form` on st, waited for.  -> the five outputs."""
    g, d16, T, fl = d["gray"][a:b], d["d16"][a:b], d["T"][a:b], d["flow"][a:b]
    if form == "f32":
        return st.track_batch(g, d["depth"][a:b], T)
    if form == "u16":
        return st.track_batch_u16(g, d16, FACTOR, T)
    if form == "u16_pinned":
        p = d["pin"]
        keep, out = _pinned_outputs(st, b - a)
        st.submit_batch_u16(p["gray"].numpy()[a:b], p["d16"].numpy()[a:b], FACTOR, p["T"].numpy()[a:b], out)
        st.sync()
        return tuple(np.array(o) for o in out)
    if form == "flow":
        return st.track_batch_u16_masked(g, d16, FACTOR, T, fl, THR)
    if form == "device_flow":
        return st.track_batch_u16_flow(g, d16, FACTOR, T, None, THR)
    dv = d["dev"]
    px = ROWS * COLS
    args = (dv["gray"].data_ptr() + a * px, dv["depth"].data_ptr() + 4 * a * px, dv["T"].data_ptr() + 64 * a)
    if form == "device":
        st.track_batch_device(*args, b - a, ROWS, COLS)
    else:
        assert form == "device_masked"
        st.track_batch_masked_device(*args, dv["flow"].data_ptr() + 4 * a * (px // 2), THR, b - a, ROWS, COLS)
    st.sync()
    return _device_outputs(st, b - a)


def _frames(st, res, masked):
    """Per frame: what the batch left for it (the first nkp entries of every row, the glue, the mask)."""
    kps, desc, nkp, c2l, nm = res
    out = []
    for t in range(len(nkp)):
        n = int(nkp[t])
        rec = dict(n=n, kps=kps[t, :n].tobytes(), desc=desc[t, :n].tobytes(), c2l=c2l[t, :n].tobytes(), nm=int(nm[t]),
                   glue=tuple(x.tobytes() for x in st.frame_glue(t, n)))
        if masked:
            m, f = st.dynamic_mask(t)
            rec.update(mask=m.tobytes(), filtered=f)
        out.append(rec)
    return out


def _run(form, sizes, d, masked=False, st=None):
    """The sequence's first sum(sizes) frames as batches of the given sizes on one handle continuing itself.  -> per frame
    records, and the nmatch of frame 0 of every continued batch."""
    st = st or _tracker()
    recs, first, a = [], [], 0
    for i, s in enumerate(sizes):
        if i:
            st.continue_after(st)
        res = _submit(form, st, d, a, a + s)
        if i:
            first.append(int(res[4][0]))
        recs += _frames(st, res, masked)
        a += s
    return recs, first


def _same_frames(got, want, skip_frame0_match=()):
    assert len(got) == len(want)
    for t, (x, y) in enumerate(zip(got, want)):
        if t in skip_frame0_match:
            x, y = dict(x, c2l=None, nm=None), dict(y, c2l=None, nm=None)
        assert x == y, t


@pytest.fixture(scope="module")
def whole(room):
    cache = {}

    def get(form, masked=False):
        if form not in cache:
            cache[form] = _run(form, (N,), room, masked)[0]
        return cache[form]
    return get


@pytest.mark.parametrize("form", ["f32", "u16", "u16_pinned", "device"])
@pytest.mark.parametrize("sizes", SPLITS, ids=lambda s: "-".join(map(str, s)))
def test_plain_split(room, whole, form, sizes):
    got, first = _run(form, sizes, room)
    _same_frames(got, whole(form))
    assert min(first) > 0, first


@pytest.mark.parametrize("form", ["flow", "device_masked", "device_flow"])
@pytest.mark.parametrize("sizes", SPLITS, ids=lambda s: "-".join(map(str, s)))
def test_masked_split(room, whole, form, sizes):
    got, first = _run(form, sizes, room, masked=True)
    _same_frames(got, whole(form, True))
    assert min(first) > 0, first


def test_plain_split_non_fused(room):
    """3000 features: frame 0's single-pair search and the batch's pairs take the non-fused LAST kernels."""
    st = _tracker(nfeatures=3000)
    want = _run("u16", (8,), room, st=_tracker(nfeatures=3000))[0]
    got, first = _run("u16", (3, 5), room, st=st)
    assert st.cap > 2000 and max(r["n"] for r in got) > 2000
    _same_frames(got, want)
    assert min(first) > 0


def test_device_flow_equals_prev_gray(room):
    """A continued device_flow batch and the same batch with prev_gray = the last gray frame before it: the same flow,
    masks and filtered keypoints; only frame 0's search differs (the prev_gray batch has no last frame)."""
    a = _tracker()
    _submit("device_flow", a, room, 0, 11)
    a.continue_after(a)
    got = _frames(a, _submit("device_flow", a, room, 11, N), True)
    b = _tracker()
    res = b.track_batch_u16_flow(room["gray"][11:], room["d16"][11:], FACTOR, room["T"][11:], room["gray"][10], THR)
    want = _frames(b, res, True)
    _same_frames(got, want, skip_frame0_match=(0,))
    assert want[0]["nm"] == 0 and got[0]["nm"] > 0


# ---- homography batches ----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def homo_seq():
    from tests import homography_chain_ref as HR
    from tests.test_homography_chain_gpu import chain_scene
    gray, d16, T = chain_scene(F=12, jump=6, windows=((8, 90),), flat=10)
    want = HR.run(gray, d16.astype(np.float32) * FACTOR, T, 1000, TH, THR)
    return gray, d16, T, want


def _homo_splits():
    return [(1, 11), (2, 10), (3, 9), "after_warp", (1, 1, 1, 9)]


@pytest.mark.parametrize("sizes", _homo_splits(), ids=lambda s: s if isinstance(s, str) else "-".join(map(str, s)))
def test_homography_split(homo_seq, sizes):
    from tests import homography_chain_ref as HR
    from tests.test_homography_chain_gpu import _check_against
    gray, d16, T, want = homo_seq
    F = len(gray)
    if sizes == "after_warp":   # a boundary right after a warped frame: frame 0's previous half image is P's warped image
        w = [t for t in range(2, F) if want[t - 1]["branch"] == HR.WARPED]
        assert w, [r["branch"] for r in want]
        sizes = (w[0], F - w[0])
    st = _tracker(F)
    a = 0
    for i, s in enumerate(sizes):
        if i:
            st.continue_after(st)
        res = st.track_batch_u16_homography(gray[a:a + s], d16[a:a + s], FACTOR, T[a:a + s], THR)
        _check_against(st, res, want[a:a + s])
        a += s


# ---- handles ---------------------------------------------------------------------------------------------------------

def test_alternating_handles(room, whole):
    """Two handles (of different batch capacities) alternating A, B, A, B with orbs_chain_after + orbs_continue, every
    batch submitted before any is waited for."""
    import torch
    A, B = _tracker(), _tracker(max_frames=8)
    p = room["pin"]
    hs, sizes, a, prev = [A, B, A, B], (5, 7, 6, 6), 0, None
    outs, keep = [], []
    for h, s in zip(hs, sizes):
        if prev is not None:
            h.chain_after(prev)
            h.continue_after(prev)
        k, out = _pinned_outputs(h, s)
        keep.append(k)
        h.submit_batch_u16(p["gray"].numpy()[a:a + s], p["d16"].numpy()[a:a + s], FACTOR, p["T"].numpy()[a:a + s], out)
        outs.append(out)
        a, prev = a + s, h
    A.sync()
    B.sync()
    torch.cuda.synchronize()
    want = whole("u16_pinned")
    t = 0
    for k, out in enumerate(outs):
        kps, desc, nkp, c2l, nm = out
        for i in range(len(nkp)):
            n, w = int(nkp[i]), want[t]
            assert (n, kps[i, :n].tobytes(), desc[i, :n].tobytes(), c2l[i, :n].tobytes(), int(nm[i])) == \
                (w["n"], w["kps"], w["desc"], w["c2l"], w["nm"]), t
            t += 1
        assert k == 0 or nm[0] > 0


def test_prev_destroyed(room, whole):
    A, B = _tracker(), _tracker()
    _submit("u16", A, room, 0, 10)
    B.continue_after(A)
    A._L.orbs_destroy(A._h)
    A._h = C.c_void_p()
    got = _frames(B, _submit("u16", B, room, 10, N), False)
    _same_frames(got, whole("u16")[10:])


def test_prev_destroyed_homography(homo_seq):
    from tests.test_homography_chain_gpu import _check_against
    gray, d16, T, want = homo_seq
    A, B = _tracker(12), _tracker(12)
    A.track_batch_u16_homography(gray[:7], d16[:7], FACTOR, T[:7], THR)
    B.continue_after(A)
    A._L.orbs_destroy(A._h)
    A._h = C.c_void_p()
    res = B.track_batch_u16_homography(gray[7:], d16[7:], FACTOR, T[7:], THR)
    _check_against(B, res, want[7:])


@pytest.mark.parametrize("form", ["u16_pinned", "device_flow"])
def test_chunk_size(room, whole, form):
    st = _tracker()
    st.set_chunk_frames(3)
    got, _ = _run(form, (8, 8, 8), room, masked=form == "device_flow", st=st)
    _same_frames(got, whole(form, form == "device_flow"))


def test_continuation_is_consumed(room):
    """The batch after a continued one, without a new orbs_continue, equals the same batch on a fresh handle, with the
    same launches."""
    st = _tracker()
    _submit("u16", st, room, 0, 8)
    st.continue_after(st)
    _submit("u16", st, room, 8, 16)
    n0 = st.launch_count()
    got = _frames(st, _submit("u16", st, room, 16, N), False)
    launches = st.launch_count() - n0
    fresh = _tracker()
    m0 = fresh.launch_count()
    want = _frames(fresh, _submit("u16", fresh, room, 16, N), False)
    assert got == want and launches == fresh.launch_count() - m0
    assert got[0]["nm"] == 0


# ---- refusals --------------------------------------------------------------------------------------------------------

def _batch(d, a, b, **kw):
    from orb_slam2_ssd_semantic_b200._abi import ptr
    f = dict(nframes=b - a, rows=ROWS, cols=COLS, device=0, gray=ptr(d["gray"][a:b]), depth=None,
             depth_u16=ptr(d["d16"][a:b]), depth_factor=float(FACTOR), Tcw=ptr(d["T"][a:b]), flow=None, device_flow=0,
             prev_gray=None, binary_threshold=THR, homography=0)
    f.update(kw)
    return f


def _refuse(st, fields):
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200._abi import OrbsBatch, OrbsResults, ptr
    F = fields["nframes"]
    outs = st.alloc_outputs(F)
    n0 = st.launch_count()
    rc = st._L.orbs_submit(st._h, C.byref(OrbsBatch(**fields)), C.byref(OrbsResults(*[ptr(a) for a in outs], st.cap)))
    assert rc == EINVAL, _lib.lib().b200orb_last_error()
    st.sync()
    assert st.launch_count() == n0
    assert all(a.tobytes() == np.zeros_like(a).tobytes() for a in outs)


def test_refusals(room, whole):
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200._abi import ptr
    L = _lib.lib()
    d = room
    small = {k: np.ascontiguousarray(d[k][8:16, :240, :320]) for k in ("gray", "d16")}
    small_T = np.ascontiguousarray(d["T"][8:16])

    A, B, empty = _tracker(), _tracker(), _tracker()
    _submit("u16", A, d, 0, 8)
    nA, nB = A.launch_count(), B.launch_count()
    # orbs_continue: NULL handles, a prev without a batch
    assert L.orbs_continue(None, A._h) == EINVAL
    assert L.orbs_continue(B._h, None) == EINVAL
    assert L.orbs_continue(B._h, empty._h) == EINVAL
    assert (A.launch_count(), B.launch_count()) == (nA, nB)

    B.continue_after(A)
    assert L.orbs_continue(B._h, empty._h) == EINVAL   # leaves the pending continuation as it was
    cases = [
        dict(nframes=8, rows=240, cols=320, gray=ptr(small["gray"]), depth_u16=ptr(small["d16"]), Tcw=ptr(small_T)),
        dict(flow=ptr(d["flow"][8:16])),                       # another variant: caller flow
        dict(device_flow=1),                                   # device_flow
        dict(device_flow=1, homography=1),                     # homography
    ]
    for kw in cases:
        _refuse(B, _batch(d, 8, 16, **kw))
    # other OrbsParams: a handle with another search window continues A
    C3 = _tracker(th=20.0)
    C3.continue_after(A)
    _refuse(C3, _batch(d, 8, 16))
    # the continuation is still pending and usable
    got = _frames(B, _submit("u16", B, d, 8, 16), False)
    _same_frames(got, whole("u16")[8:16])
    assert got[0]["nm"] > 0

    # prev_gray together with a continuation (of a device_flow batch)
    D, E = _tracker(), _tracker()
    _submit("device_flow", D, d, 0, 8)
    E.continue_after(D)
    _refuse(E, _batch(d, 8, 16, device_flow=1, prev_gray=ptr(np.ascontiguousarray(d["gray"][7]))))
    _refuse(E, _batch(d, 8, 16))                               # and a plain batch after a device_flow one
    got = _frames(E, _submit("device_flow", E, d, 8, 16), True)
    _same_frames(got, whole("device_flow", True)[8:16])
