"""GPU parity of the batched tracker's masked frames (the `perfect` variant's live path, perfect/src/Tracking.cc:703-719):
per frame the dynamic mask from the half-resolution flow, the masked constructor's keypoint filter and SearchByProjection
against the previous filtered frame, against the oracle run stage by stage on the CPU (RefExtractor ->
dynmask_py.mask_from_flow -> dynmask_py.filter_keypoints -> frame_views -> search_by_projection_last)."""
import os

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth
from tests.helpers import frame_views

pytestmark = pytest.mark.gpu

CAM = (synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)


def _batch(seed, F, rows=480, cols=640):
    ws = synth.WallStream(seed=seed, n=F, h=rows, w=cols)
    frames = [ws.frame(t) for t in range(F)]
    gray = np.stack([f[0] for f in frames])
    T = np.stack([f[3] for f in frames])
    d16 = np.rint(np.stack([f[1] for f in frames]).astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    factor = np.float32(1.0 / synth.DEPTH_FACTOR)
    return gray, d16, d16.astype(np.float32) * factor, factor, T


def _blob(h, w, cy, cx, ry, rx, v):
    """Zero flow with one fast elliptic blob (half-resolution coordinates)."""
    f = np.zeros((h, w, 2), np.float32)
    yy, xx = np.mgrid[0:h, 0:w]
    f[((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1.0] = v
    return f


def _band(k, h=240, w=320):
    """Zero flow except a full-width band of rows [0, k) moving at 50 px: the final mask keeps whole rows, so its sum moves
    in steps of two image rows."""
    f = np.zeros((h, w, 2), np.float32)
    f[:k, :, 0] = 50.0
    return f


def _flows(F, rows, cols, seed):
    """Frame 0 without a predecessor (zero flow), then synthetic Farneback-like fields with moving blobs."""
    h, w = rows // 2, cols // 2
    return np.stack([np.zeros((h, w, 2), np.float32)] + [synth.flow_field(seed + t, h, w, blobs=6) for t in range(1, F)])


def _tracker(nfeatures=1000, max_frames=8):
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    return StreamTracker(nfeatures, 1.2, 8, 20, 7, *CAM, th=15.0, nnratio=0.9, max_frames=max_frames)


def _masked_parity(oracle, gray, d16, depth, factor, T, flow, thr=40.0, nfeatures=1000):
    """track_batch_u16_masked (pageable CV_16U depth: the gathered depth moves with the filtered keypoints) against the
    oracle, frame by frame, bit for bit.  -> per frame (filtered, keypoints extracted, keypoints kept)."""
    from oracle import dynmask_py as O
    F, rows, cols = gray.shape
    st = _tracker(nfeatures, F)
    kps, desc, nkp, c2l, nm = st.track_batch_u16_masked(gray, d16, factor, T, flow, thr)
    R = oracle.RefExtractor(nfeatures, 1.2, 8, 20, 7)
    prev, out = None, []
    for t in range(F):
        K, D = R(gray[t])
        mask = O.mask_from_flow(flow[t], thr, (rows, cols))
        Kf, Df = O.filter_keypoints(mask, K, D)
        filt = float(mask.sum()) > rows * cols * 0.65
        m, f = st.dynamic_mask(t)
        assert (m == mask).all() and f == filt, t
        assert nkp[t] == len(Kf), t
        assert kps[t, :nkp[t]].tobytes() == Kf.tobytes() and (desc[t, :nkp[t]] == Df).all(), t
        if prev is None:
            assert nm[t] == 0 and (c2l[t, :nkp[t]] == -1).all()
        else:
            cur, last = frame_views(oracle, Kf, Df, depth[t], T[t], prev[0], prev[1], depth[t - 1], T[t - 1], R.mvScaleFactor,
                                    obs=1, rows=rows, cols=cols)
            n_ref, ref = oracle.search_by_projection_last(cur, last, 15.0, False, 0.9, True)
            assert nm[t] == n_ref and (c2l[t, :nkp[t]] == ref).all(), t
        prev = (Kf, Df)
        out.append((filt, len(K), len(Kf)))
    return out, nm


def test_masked_batch_matches_oracle(oracle):
    """640 x 480, 6 frames: zero flow (frame 0), a typical field, a mask at most 65 % ones (keeps everything), NaN / +-inf /
    1e20 flow values, a fast blob that removes keypoints, another typical field."""
    gray, d16, depth, factor, T = _batch(1234, 6)
    flow = _flows(6, 480, 640, 300)
    flow[2] = _band(120)
    flow[3, 17, 23] = (np.nan, 1.0)
    flow[3, 100, 200] = (np.inf, 0.0)
    flow[3, 50, 60] = (-np.inf, 2.0)
    flow[3, 0, 0] = (1e20, 1e20)
    flow[3, 239, 319] = (0.0, np.nan)
    flow[4] = _blob(240, 320, 120, 160, 50, 70, (30.0, -12.0))
    fr, nm = _masked_parity(oracle, gray, d16, depth, factor, T, flow)
    assert fr[0][0] and fr[0][1] == fr[0][2]                  # all-ones mask: filter on, nothing dropped
    assert not fr[2][0] and fr[2][1] == fr[2][2]              # <= 65 %: nothing dropped
    assert fr[4][0] and fr[4][2] < fr[4][1] - 50              # the blob's keypoints are gone
    assert fr[3][2] < fr[3][1]
    assert nm[1:].min() > 100


def test_masked_batch_kitti_width(oracle):
    """376 x 1241: the half-resolution flow is 188 x 620, so mask column 1240 lies beyond the 1240 columns it covers."""
    gray, d16, depth, factor, T = _batch(77, 3, 376, 1241)
    flow = _flows(3, 376, 1241, 310)
    flow[2] = _blob(188, 620, 90, 560, 40, 80, (20.0, 5.0))   # a blob reaching the covered columns' edge
    fr, nm = _masked_parity(oracle, gray, d16, depth, factor, T, flow)
    assert fr[2][2] < fr[2][1] and nm[1:].min() > 50


def test_masked_batch_odd_image(oracle):
    """481 x 641 gray images: the mask's last row and column are not covered by the 240 x 320 flow and stay 1."""
    gray, d16, depth, factor, T = _batch(79, 3, 481, 641)
    flow = _flows(3, 481, 641, 320)
    fr, nm = _masked_parity(oracle, gray, d16, depth, factor, T, flow, thr=55.5)
    assert nm[1:].min() > 50


def test_masked_batch_non_fused(oracle):
    """3000 features: the frame pairs go through the non-fused LAST kernels."""
    gray, d16, depth, factor, T = _batch(1234, 3)
    flow = _flows(3, 480, 640, 330)
    fr, nm = _masked_parity(oracle, gray, d16, depth, factor, T, flow, nfeatures=3000)
    assert max(f[1] for f in fr) > 2000 and nm[1:].min() > 100


def test_65_percent_rule_both_sides(oracle):
    """Full-width bands whose final masks sum to exactly 0.65 * rows * cols (not above: nothing is dropped) and to two image
    rows more, the next sum a band of the half-resolution flow can give (above: the band's keypoints are dropped)."""
    from oracle import dynmask_py as O
    at, above = O.mask_from_flow(_band(79), 40.0), O.mask_from_flow(_band(78), 40.0)
    assert at.sum() == 199680 and float(at.sum()) == 480 * 640 * 0.65 and above.sum() == 199680 + 2 * 640
    gray, d16, depth, factor, T = _batch(1234, 4)
    flow = np.stack([np.zeros((240, 320, 2), np.float32), _band(79), _band(78), _band(79)])
    fr, _ = _masked_parity(oracle, gray, d16, depth, factor, T, flow)
    assert [f[0] for f in fr] == [True, False, True, False]
    assert fr[1][1] == fr[1][2] and fr[2][2] < fr[2][1] and fr[3][1] == fr[3][2]


def _device_out(st, F):
    from tests.test_extractor_gpu import _device_to_host
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    (p_kps, p_desc, p_nkp, p_c2l, p_nm), cap = st.device_results()
    return (_device_to_host(p_kps, KP_DTYPE.itemsize * cap * F).view(KP_DTYPE).reshape(F, cap),
            _device_to_host(p_desc, 32 * cap * F).reshape(F, cap, 32), _device_to_host(p_nkp, 4 * F).view(np.int32),
            _device_to_host(p_c2l, 4 * cap * F).view(np.int32).reshape(F, cap), _device_to_host(p_nm, 4 * F).view(np.int32))


def _same(a, b):
    """Equal outputs of two batches: counts, and every keypoint / descriptor / match of the kept keypoints."""
    n = a[2]
    assert (b[2] == n).all() and (b[4] == a[4]).all()
    for f in range(len(n)):
        assert a[0][f, :n[f]].tobytes() == b[0][f, :n[f]].tobytes()
        assert (a[1][f, :n[f]] == b[1][f, :n[f]]).all() and (a[3][f, :n[f]] == b[3][f, :n[f]]).all()


def test_host_and_device_paths_equal():
    """track_batch_u16_masked with pageable and with page-locked CV_16U depth == track_batch_masked_device on the matching
    f32 depth in HBM, and the masks they leave are equal."""
    import torch
    F = 4
    gray, d16, depth, factor, T = _batch(78, F)
    flow = _flows(F, 480, 640, 340)
    st = _tracker(1000, F)
    pageable = [x.copy() for x in st.track_batch_u16_masked(gray, d16, factor, T, flow, 40.0)]
    masks = [st.dynamic_mask(t) for t in range(F)]
    pinned = torch.from_numpy(d16).pin_memory()
    locked = [x.copy() for x in st.track_batch_u16_masked(gray, pinned.numpy(), factor, T, flow, 40.0)]
    dev = _tracker(1000, F)
    g, d, t, fl = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (gray, depth, T.astype(np.float32), flow))
    torch.cuda.synchronize()
    dev.track_batch_masked_device(g.data_ptr(), d.data_ptr(), t.data_ptr(), fl.data_ptr(), 40.0, F, 480, 640)
    dev.sync()
    for o in (locked, _device_out(dev, F)):
        _same(pageable, o)
    for t in range(F):
        m, f = dev.dynamic_mask(t)
        assert (m == masks[t][0]).all() and f == masks[t][1]
    assert any(f < 0.99 for f in (m.mean() for m, _ in masks))


def test_two_masked_batches_in_flight_equal_synchronous_calls():
    """submit_batch_u16_masked on two alternating handles chained with orbs_chain_after == synchronous
    track_batch_u16_masked, batch by batch."""
    import torch
    F = 5
    batches = []
    for b in range(3):
        gray, d16, _, factor, T = _batch(9 + b, F)
        flow = _flows(F, 480, 640, 400 + 10 * b)
        pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
        batches.append((pin(gray), pin(d16), pin(T.astype(np.float32)), pin(flow)))
    ref = _tracker(1000, F)
    want = [[x.copy() for x in ref.track_batch_u16_masked(g.numpy(), d.numpy(), factor, T.numpy(), fl.numpy(), 40.0)]
            for g, d, T, fl in batches]
    trk = [_tracker(1000, F), _tracker(1000, F)]
    outs = [t.alloc_outputs(F, pinned=True) for t in trk]
    got = []
    for k, (g, d, T, fl) in enumerate(batches):
        if k >= 2:
            trk[k & 1].sync()
            got.append([x.copy() for x in outs[k & 1]])
        trk[k & 1].chain_after(trk[(k + 1) & 1])
        trk[k & 1].submit_batch_u16_masked(g.numpy(), d.numpy(), factor, T.numpy(), fl.numpy(), 40.0, outs[k & 1])
    for k in range(len(batches) - 2, len(batches)):
        trk[k & 1].sync()
        got.append([x.copy() for x in outs[k & 1]])
    for w, g in zip(want, got):
        _same(w, g)
    with pytest.raises(ValueError):
        trk[0].submit_batch_u16_masked(batches[0][0].numpy(), batches[0][1].numpy(), factor, batches[0][2].numpy(),
                                       batches[0][3].numpy()[:, ::2], 40.0, outs[0])


def test_zero_flow_equals_unmasked_batch():
    """Zero flow everywhere: every mask is all ones, so every output is byte-identical to track_batch_u16; the masked batch
    launches exactly one kernel more (the mask + filter kernel)."""
    F = 4
    gray, d16, _, factor, T = _batch(81, F)
    flow = np.zeros((F, 240, 320, 2), np.float32)
    st = _tracker(1000, F)
    n0 = st.launch_count()
    a = [x.copy() for x in st.track_batch_u16(gray, d16, factor, T)]
    n1 = st.launch_count()
    b = [x.copy() for x in st.track_batch_u16_masked(gray, d16, factor, T, flow, 40.0)]
    n2 = st.launch_count()
    c = [x.copy() for x in st.track_batch_u16(gray, d16, factor, T)]
    n3 = st.launch_count()
    for x, y, z in zip(a, b, c):
        assert x.tobytes() == y.tobytes() == z.tobytes()
    assert n2 - n1 == (n1 - n0) + 1 and n3 - n2 == n1 - n0
    from orb_slam2_ssd_semantic_b200 import B200OrbError
    with pytest.raises(B200OrbError):            # the last batch was not masked
        st.dynamic_mask(0)


def test_geometry_limit():
    """The largest 1280-wide image whose two bit planes fit one CTA's shared memory runs (and its mask is right); one row
    more is refused with B200OrbError before anything is enqueued, and the handle then still tracks a 640 x 480 batch
    exactly like a fresh handle."""
    import torch
    from oracle import dynmask_py as O
    from orb_slam2_ssd_semantic_b200 import B200OrbError
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    rmax = (optin // 4 - 33) // 2 // 40                       # rows * ceil(1280 / 32) words per plane
    assert rmax >= 720
    st = _tracker(1000, 2)
    gray, d16, _, factor, T = _batch(82, 2, rmax, 1280)
    flow = _flows(2, rmax, 1280, 500)
    kps, desc, nkp, c2l, nm = st.track_batch_u16_masked(gray, d16, factor, T, flow, 40.0)
    m, _ = st.dynamic_mask(1)
    assert (m == O.mask_from_flow(flow[1], 40.0, (rmax, 1280))).all() and nm[1] > 50
    gray2, d162, _, _, T2 = _batch(82, 2, rmax + 1, 1280)
    with pytest.raises(B200OrbError):
        st.track_batch_u16_masked(gray2, d162, factor, T2, _flows(2, rmax + 1, 1280, 500), 40.0)
    gray, d16, _, factor, T = _batch(83, 3)
    flow = _flows(3, 480, 640, 510)
    fresh = _tracker(1000, 2)
    _same(fresh.track_batch_u16_masked(gray, d16, factor, T, flow, 40.0), st.track_batch_u16_masked(gray, d16, factor, T, flow, 40.0))


def test_masked_frames_equal_the_reference_masked_constructor(oracle):
    """At full size (640 x 480, 2000 features) the keypoints and descriptors of every masked frame equal what the perfect
    tree's own masked RGB-D Frame constructor keeps (perfect/src/Frame.cc:328-427, compiled unmodified into
    oracle/_ref/librefperfect.so) for the same mask.  The matches need no pin of their own: the perfect tree's
    SearchByProjection(cur, last) (perfect/src/ORBmatcher.cc:1578-1725) is the T tree's, which the oracle is pinned to."""
    from oracle import ref
    if not os.path.exists(ref._PERFSO):
        pytest.skip("oracle/_ref/librefperfect.so was not built (the reference sources are absent)")
    from oracle import dynmask_py as O
    F = 4
    gray, d16, depth, factor, T = _batch(1234, F)
    flow = _flows(F, 480, 640, 600)
    flow[2] = _band(120)
    flow[3] = _blob(240, 320, 100, 200, 60, 60, (25.0, 25.0))
    st = _tracker(2000, F)
    kps, desc, nkp, c2l, nm = st.track_batch_u16_masked(gray, d16, factor, T, flow, 40.0)
    dropped = 0
    for t in range(F):
        mask = O.mask_from_flow(flow[t], 40.0)
        (kp, _), (km, dm) = ref.perfect_frames(gray[t], depth[t], mask, nfeatures=2000, fx=synth.FX, fy=synth.FY, cx=synth.CX,
                                               cy=synth.CY, bf=synth.BF)
        assert nkp[t] == len(km) and kps[t, :nkp[t]].tobytes() == km.tobytes() and (desc[t, :nkp[t]] == dm).all(), t
        dropped += len(kp) - len(km)
    assert dropped > 100
