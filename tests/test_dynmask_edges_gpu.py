"""GPU parity of the dynamic mask on the crafted cases of tests/dynmask_cases.py, bit for bit: the per-stage entries
(dynm_mask_from_flow, dynm_mask_from_flow_batch_device, dynm_filter_keypoints, dynm_filter_keypoints_batch_device,
dynm_farneback, dynm_flow_batch_device) against the cv2-pinned oracles, the batch tracker's one-CTA-per-frame mask kernel
at widths around the 32-pixel words, and the host-buffer batches split into uneven upload chunks against one chunk."""
import ctypes as C

import numpy as np
import pytest

from oracle import dynmask_py as O
from oracle import farneback_py as FB
from orb_slam2_ssd_semantic_b200 import synth
from tests import dynmask_cases as D
from tests.helpers import frame_views

pytestmark = pytest.mark.gpu

MASKS = D.mask_cases()
FAMILIES = sorted({c.name.split("/")[0] for c in MASKS})
LOOKUPS = D.lookup_cases()
FLOWS = D.flow_cases()


@pytest.fixture(scope="module")
def dm():
    from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask
    return DynamicMask(0)


@pytest.fixture(scope="module")
def fb_ref():
    """The restatement's flow of each Farneback case, computed once per module (2048 x 2048 takes about 30 s)."""
    cache = {}

    def get(case):
        if case.name not in cache:
            cache[case.name] = FB.farneback(*case.pair())
        return cache[case.name]
    return get


def _bits_equal(a, b):
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and (a.view(np.uint32) == b.view(np.uint32)).all()


# ---- masks ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("family", FAMILIES)
def test_mask_from_flow_equals_oracle(dm, family):
    bad = [c.name for c in MASKS if c.name.split("/")[0] == family
           and not (dm.mask_from_flow(c.flow, c.thr, c.shape) == O.mask_from_flow(c.flow, c.thr, c.shape)).all()]
    assert not bad


@pytest.mark.parametrize("family", FAMILIES)
def test_mask_batch_device_equals_oracle(dm, family):
    """Cases of one geometry and threshold go through dynm_mask_from_flow_batch_device as one batch."""
    import torch
    from orb_slam2_ssd_semantic_b200 import _lib
    groups = {}
    for c in MASKS:
        if c.name.split("/")[0] == family:
            groups.setdefault((c.flow.shape, c.shape, c.thr), []).append(c)
    bad = []
    for (fshape, shape, thr), cases in groups.items():
        F = len(cases)
        d_flow = torch.from_numpy(np.stack([c.flow for c in cases])).cuda()
        d_mask = torch.full((F,) + shape, 7, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        _lib.check(_lib.lib().dynm_mask_from_flow_batch_device(dm._h, C.c_void_p(d_flow.data_ptr()), F, fshape[0], fshape[1], thr,
                                                               C.c_void_p(d_mask.data_ptr()), shape[0], shape[1]))
        dm.sync()
        out = d_mask.cpu().numpy()
        bad += [c.name for c, m in zip(cases, out) if not (m == O.mask_from_flow(c.flow, c.thr, c.shape)).all()]
    assert not bad


@pytest.mark.parametrize("rows,cols", D.TRACKER_SHAPES)
def test_tracker_mask_kernel_at_word_widths(oracle, dm, rows, cols):
    """k_dynm_plane_filter (orbs_read_dynamic_mask) == the oracle == the per-stage entry on crafted band flows whose edges sit
    at word boundaries, with static bands of 20 and 25 px against the right side; the kept keypoints, descriptors and
    matches as in test_masked_tracking_gpu._masked_parity."""
    from tests.test_masked_tracking_gpu import _batch, _masked_parity
    gray, d16, depth, factor, T = _batch(600 + cols, 3, rows, cols)
    flow = D.tracker_flows(rows, cols)
    for t in range(3):
        want = O.mask_from_flow(flow[t], D.THR, (rows, cols))
        assert (dm.mask_from_flow(flow[t], D.THR, (rows, cols)) == want).all(), t
    fr, nm = _masked_parity(oracle, gray, d16, depth, factor, T, flow, thr=D.THR)
    assert fr[1][2] < fr[1][1] and nm[1:].min() > 20


# ---- keypoint filter -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", LOOKUPS, ids=[c.name for c in LOOKUPS])
def test_filter_keypoints_equals_oracle(dm, case):
    kr, dr = case.expected()
    k2, d2 = dm.filter_keypoints(case.mask, case.kps, case.desc)
    assert len(k2) == len(kr) and k2.tobytes() == kr.tobytes() and (d2 == dr).all()
    assert 0 < len(kr) < len(case.kps)


def test_filter_batch_device_equals_oracle(dm):
    """dynm_filter_keypoints_batch_device on the extractor's [F][cap] layout: the lookup cases of one mask shape as one batch
    with cap = the largest count, the others one frame each."""
    import torch
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    groups = {}
    for c in LOOKUPS:
        groups.setdefault(c.mask.shape, []).append(c)
    for shape, cases in groups.items():
        F, cap = len(cases), max(len(c.kps) for c in cases)
        kps = np.zeros((F, cap), KP_DTYPE)
        desc = np.zeros((F, cap, 32), np.uint8)
        cnt = np.array([len(c.kps) for c in cases], np.int32)
        for f, c in enumerate(cases):
            kps[f, :cnt[f]], desc[f, :cnt[f]] = c.kps, c.desc
        masks = np.stack([c.mask for c in cases])
        d_k = torch.from_numpy(kps.view(np.uint8).reshape(F, cap * KP_DTYPE.itemsize)).cuda()
        d_d, d_n, d_m = torch.from_numpy(desc).cuda(), torch.from_numpy(cnt).cuda(), torch.from_numpy(masks).cuda()
        torch.cuda.synchronize()
        _lib.check(_lib.lib().dynm_filter_keypoints_batch_device(dm._h, C.c_void_p(d_m.data_ptr()), F, shape[0], shape[1],
                                                                 C.c_void_p(d_k.data_ptr()), C.c_void_p(d_d.data_ptr()),
                                                                 C.c_void_p(d_n.data_ptr()), cap))
        dm.sync()
        n = d_n.cpu().numpy()
        kp = d_k.cpu().numpy().reshape(-1).view(KP_DTYPE).reshape(F, cap)
        ds = d_d.cpu().numpy()
        for f, c in enumerate(cases):
            kr, dr = c.expected()
            assert n[f] == len(kr) and kp[f, :n[f]].tobytes() == kr.tobytes() and (ds[f, :n[f]] == dr).all(), c.name


# ---- Farneback -----------------------------------------------------------------------------------------------------

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


@pytest.mark.parametrize("case", FLOWS, ids=[c.name for c in FLOWS])
def test_farneback_equals_restatement(dm, fb_ref, case):
    from orb_slam2_ssd_semantic_b200 import B200OrbError
    prev, cur = case.pair()
    if case.refused:
        with pytest.raises(B200OrbError):
            dm.farneback(prev, cur)
        with pytest.raises(B200OrbError):
            _flow_batch(dm, case.gray)
        return
    want = fb_ref(case)
    assert _bits_equal(dm.farneback(prev, cur), want)
    both = _flow_batch(dm, case.gray)
    assert not both[0].any() and _bits_equal(both[1], want)
    assert _bits_equal(_flow_batch(dm, case.gray[1:], case.gray[0])[0], want)


# ---- upload chunks -------------------------------------------------------------------------------------------------

F_CHUNK = 9
CHUNKINGS = (1, 2, 3, 8, 9, 128)    # 7, 5, 3, 2, 1, 1 chunks of 9 frames


def _chunk_inputs():
    from tests.test_masked_tracking_gpu import _band, _batch, _blob, _flows
    gray, d16, depth, factor, T = _batch(4321, F_CHUNK + 1)
    flow = _flows(F_CHUNK, 480, 640, 900)
    flow[3] = _band(60)
    flow[6] = _blob(240, 320, 120, 100, 60, 50, (20.0, 9.0))
    flow[8] = D.tracker_flows(480, 640)[1]
    return gray, d16, depth, factor, T, flow


def _run(st, entry, gray, d16, factor, T, flow, prev):
    if entry == "u16":
        out = st.track_batch_u16(gray, d16, factor, T)
    elif entry == "masked":
        out = st.track_batch_u16_masked(gray, d16, factor, T, flow, 40.0)
    else:
        out = st.track_batch_u16_flow(gray, d16, factor, T, prev, 40.0)
    out = [x.copy() for x in out]
    n = out[2]
    glue = [[a.copy() for a in st.frame_glue(t, int(n[t]))] for t in range(len(n))]
    masks = [st.dynamic_mask(t) for t in range(len(n))] if entry != "u16" else None
    return out, glue, masks


def _glue_bytes(g):
    """(uright, depth, xw, valid) as bytes; xw only where valid (the glue writes no world point without depth)."""
    ur, dp, xw, va = (np.asarray(x) for x in g)
    v = va.astype(bool)
    return (ur.astype(np.float32).tobytes(), dp.astype(np.float32).tobytes(), xw.astype(np.float32)[v].tobytes(),
            va.astype(np.uint8).tobytes())


def _same_run(a, b):
    (oa, ga, ma), (ob, gb, mb) = a, b
    n = oa[2]
    assert (ob[2] == n).all() and (ob[4] == oa[4]).all()
    for f in range(len(n)):
        assert oa[0][f, :n[f]].tobytes() == ob[0][f, :n[f]].tobytes(), f
        assert (oa[1][f, :n[f]] == ob[1][f, :n[f]]).all() and (oa[3][f, :n[f]] == ob[3][f, :n[f]]).all(), f
        assert _glue_bytes(ga[f]) == _glue_bytes(gb[f]), f
        if ma is not None:
            assert (ma[f][0] == mb[f][0]).all() and ma[f][1] == mb[f][1], f


def _oracle_check(oracle, run, gray, depth, T, flow):
    """One chunked run against the oracle frame by frame: extraction, the mask and its filter (flow given), the frame glue
    and SearchByProjection(t, t-1)."""
    (kps, desc, nkp, c2l, nm), glue, masks = run
    F, rows, cols = gray.shape
    R = oracle.RefExtractor(1000, 1.2, 8, 20, 7)
    prev = None
    for t in range(F):
        K, Dd = R(gray[t])
        if flow is not None:
            mask = O.mask_from_flow(flow[t], 40.0, (rows, cols))
            assert (masks[t][0] == mask).all(), t
            K, Dd = O.filter_keypoints(mask, K, Dd)
        assert nkp[t] == len(K) and kps[t, :nkp[t]].tobytes() == K.tobytes() and (desc[t, :nkp[t]] == Dd).all(), t
        ref = oracle.stereo_unproject(K, depth[t], T[t], synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
        assert _glue_bytes(glue[t]) == _glue_bytes(ref), t
        if prev is None:
            assert nm[t] == 0
        else:
            cur, last = frame_views(oracle, K, Dd, depth[t], T[t], prev[0], prev[1], depth[t - 1], T[t - 1], R.mvScaleFactor,
                                    obs=1, rows=rows, cols=cols)
            n_ref, m_ref = oracle.search_by_projection_last(cur, last, 15.0, False, 0.9, True)
            assert nm[t] == n_ref and (c2l[t, :nkp[t]] == m_ref).all(), t
        prev = (K, Dd)


@pytest.mark.parametrize("entry", ["u16", "masked", "flow"])
def test_upload_chunks_equal_one_chunk(oracle, entry):
    """F = 9 frames through set_chunk_frames(1, 2, 3, 8, 9, 128): 7 uneven chunks, then 5, 3, 2, 1, 1.  Every output of
    every chunking equals the single-chunk run byte for byte -- keypoints, descriptors, counts, cur2last, match counts,
    the frame glue and each frame's dynamic mask -- with pageable and page-locked CV_16U depth (u16, masked) and with and
    without prev_gray (flow).  The 5-chunk run also equals the oracle (flow: the masked entry fed the restatement's flow,
    itself checked against the oracle)."""
    import torch
    from orb_slam2_ssd_semantic_b200 import B200OrbError
    from tests.test_masked_tracking_gpu import _tracker
    gray_all, d16_all, depth_all, factor, T_all, flow = _chunk_inputs()
    gray, d16, depth, T = gray_all[1:], d16_all[1:], depth_all[1:], T_all[1:]
    st = _tracker(1000, F_CHUNK)
    with pytest.raises(B200OrbError):
        st.set_chunk_frames(0)
    if entry == "flow":
        variants = [("noprev", d16, None), ("prev", d16, gray_all[0])]
    else:
        variants = [("pageable", d16, None), ("pinned", torch.from_numpy(d16).pin_memory().numpy(), None)]
    for vname, dd, prev in variants:
        runs = {}
        for k in CHUNKINGS:
            st.set_chunk_frames(k)
            runs[k] = _run(st, entry, gray, dd, factor, T, flow, prev)
        for k in CHUNKINGS[:-1]:
            _same_run(runs[128], runs[k])
        if vname in ("pageable", "noprev"):
            if entry == "flow":
                want = np.stack([np.zeros((240, 320, 2), np.float32)]
                                + [FB.farneback(FB.pyr_down(gray[t - 1], 240, 320), FB.pyr_down(gray[t], 240, 320))
                                   for t in range(1, F_CHUNK)])
                st.set_chunk_frames(2)
                masked = _run(st, "masked", gray, dd, factor, T, want, None)
                _oracle_check(oracle, masked, gray, depth, T, want)
                _same_run(masked, runs[2])
            else:
                _oracle_check(oracle, runs[2], gray, depth, T, flow if entry == "masked" else None)
    if entry == "masked":
        assert any(not m[0].all() for m in runs[128][2])
