"""GPU parity of homography batches (OrbsBatch.homography = 1): TrackHomo (perfect/src/Tracking.cc:1331-1399) chained frame
after frame on the device, in front of the flow mask and keypoint filter (perfect/src/Tracking.cc:703-719).

  * test_chain_equals_restatement: the batch against tests/homography_chain_ref.py (the oracles of every stage composed
    with TrackHomo's control flow) on a 12-frame sequence whose frames take the branches no last frame, no velocity,
    warped, warped after a successful retry at 2 th, few pairs and few matches; bit for bit on every frame's branch,
    counts, H, mask, filtered keypoints and descriptors, cur2last and nmatch;
  * test_chain_equals_pinned_entries: the same control flow driven from the host through the separately pinned entries
    (orbm_search_by_projection_last_pairs, dynm_find_homography, dynm_warp_perspective, dynm_farneback,
    dynm_mask_from_flow, dynm_filter_keypoints) on a 24-frame sequence crafted so that frames take every branch but "no
    model" (which needs degenerate pair sets); every frame's branch, counts, H, mask, filtered keypoints, cur2last and
    nmatch are equal bit for bit;
  * test_no_warp_equals_device_flow: on a sequence where no frame warps, the batch equals the device_flow batch;
  * test_submit_does_not_wait: orbs_submit of a homography batch returns while the stream is still busy;
  * test_rejected_forms_change_nothing: every refused homography form returns EINVAL with no state change."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth
from tests.helpers import frame_views

pytestmark = pytest.mark.gpu

CAM = (synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
ROWS, COLS = 480, 640
TH, THR = 15.0, 40.0
EINVAL = -1
FACTOR = np.float32(1.0 / synth.DEPTH_FACTOR)


def _tracker(F, nfeatures=1000):
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    return StreamTracker(nfeatures, 1.2, 8, 20, 7, *CAM, th=TH, nnratio=0.9, max_frames=F)


def _disc(h, w, cy, cx, r):
    yy, xx = np.mgrid[0:h, 0:w]
    return (yy - cy) ** 2 + (xx - cx) ** 2 < r * r


def chain_scene(F=24, seed=31, jump=8, windows=((13, 90), (16, 130)), flat=20):
    """RoomStream frames (the camera moves, so consecutive frames are related by a homography on the walls) with
      * a textured disc moving 9 px per frame across the image: dynamic, the mask removes it;
      * frame `jump` shifted 24 px to the right with its depth (the projections of frame jump-1's points miss the th
        window and need 2 th; frame jump+1 sees the same shift back);
      * frames showing the scene only through a square window of the given side, grey elsewhere (few pairs);
      * frame `flat` one grey level (no keypoints: fewer than 20 matches here and in the frame after it).
    -> gray [F][480][640] u8, depth_u16 [F][480][640], Tcw [F][4][4] f32."""
    rs = synth.RoomStream(seed=seed, n=F)
    fr = [rs.frame(t) for t in range(F)]
    gray = np.stack([f[0] for f in fr]).copy()
    d16 = np.rint(np.stack([f[1] for f in fr]).astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    T = np.stack([f[3] for f in fr]).astype(np.float32)
    tex = np.clip(np.rint(synth.texture(seed + 1, ROWS, COLS, nrect=300, nline=120)), 0, 255).astype(np.uint8)
    for t in range(F):
        m = _disc(ROWS, COLS, 240, 120 + 9 * t, 70)
        gray[t][m] = np.roll(tex, 9 * t, axis=1)[m]
    if jump is not None:
        gray[jump] = np.roll(gray[jump], 24, axis=1)
        d16[jump] = np.roll(d16[jump], 24, axis=1)
    for t, side in windows:
        keep = np.zeros((ROWS, COLS), bool)
        keep[240 - side // 2:240 + side // 2, 420 - side // 2:420 + side // 2] = True
        gray[t][~keep] = 128
    if flat is not None:
        gray[flat] = 128
    return np.ascontiguousarray(gray), np.ascontiguousarray(d16), np.ascontiguousarray(T)


def no_warp_scene(F=8):
    """chain_scene's frames seen through an 80 px window each: every frame finds fewer than 20 matches or at most 50
    pairs, so none warps."""
    return chain_scene(F, jump=None, windows=tuple((t, 80) for t in range(F)), flat=None)


def _kept(K, Kf):
    """Indices of the filtered keypoints Kf in K (the filter keeps order)."""
    idx, j = [], 0
    for i in range(len(K)):
        if j < len(Kf) and K[i].tobytes() == Kf[j].tobytes():
            idx.append(i)
            j += 1
    assert j == len(Kf)
    return np.array(idx, np.int64)


def host_chain(gray, d16, T, nfeatures=1000):
    """The chain through the pinned host entries: TrackHomo's two searches, findHomography, warpPerspective, pyrDown +
    Farneback, the mask and the filter, frame after frame; then SearchByProjection of the filtered frames.  The unfiltered
    keypoints come from an unmasked batch of the same frames.  -> per frame dict."""
    from oracle import farneback_py as FB
    from oracle import ref
    from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask
    from orb_slam2_ssd_semantic_b200.matcher import ORBmatcher
    F = len(gray)
    st = _tracker(F, nfeatures)
    kps, desc, nkp, _, _ = st.track_batch_u16(gray, d16, FACTOR, T)
    sf = ref.RefExtractor(nfeatures, 1.2, 8, 20, 7).mvScaleFactor
    depth = d16.astype(np.float32) * FACTOR
    dm, mt = DynamicMask(), ORBmatcher(0.9, True)
    H2, W2 = ROWS // 2, COLS // 2
    out, filt = [], []
    last_half = FB.pyr_down(gray[0], H2, W2)
    for t in range(F):
        K, D = kps[t, :nkp[t]], desc[t, :nkp[t]]
        rec = dict(branch=1 if t == 1 else 0, nmatches=0, npairs=0, H=np.zeros(9))
        dest = gray[t]
        if t == 0:
            flow = np.zeros((H2, W2, 2), np.float32)
        else:
            if t >= 2:
                Kl, Dl = filt[t - 1]
                cur, last = frame_views(ref, K, D, depth[t], T[t], Kl, Dl, depth[t - 1], T[t - 1], sf)
                nm, _, pairs = mt.SearchByProjectionPairs(cur, last, TH, False)
                if nm < 20:
                    nm, _, pairs = mt.SearchByProjectionPairs(cur, last, 2 * TH, False)
                src = np.stack([K["x"][pairs[:, 1]], K["y"][pairs[:, 1]]], 1).astype(np.float32)
                dst = np.stack([Kl["x"][pairs[:, 0]], Kl["y"][pairs[:, 0]]], 1).astype(np.float32)
                rec.update(nmatches=nm, npairs=len(pairs))
                if nm < 20:
                    rec["branch"] = 2
                elif len(pairs) <= 50:
                    rec["branch"] = 3
                else:
                    H, _ = dm.find_homography(src, dst)
                    rec["branch"] = 4 if H is None else 5
                    if H is not None:
                        rec["H"] = H.reshape(9)
                        dest = dm.warp_perspective(gray[t], H)
            cur_half = FB.pyr_down(dest, H2, W2)
            flow = dm.farneback(last_half, cur_half)
            last_half = cur_half
        mask = dm.mask_from_flow(flow, THR, (ROWS, COLS))
        Kf, Df = dm.filter_keypoints(mask, K, D)
        _kept(K, Kf)
        filt.append((Kf, Df))
        rec.update(mask=mask, filtered=float(mask.sum()) > ROWS * COLS * 0.65, kps=Kf, desc=Df)
        if t == 0:
            rec.update(nm=0, c2l=np.full(len(Kf), -1, np.int32))
        else:
            cur, last = frame_views(ref, Kf, Df, depth[t], T[t], filt[t - 1][0], filt[t - 1][1], depth[t - 1], T[t - 1], sf)
            nm, c2l = ORBmatcher(0.9, True).SearchByProjection(cur, last, TH, False)
            rec.update(nm=nm, c2l=c2l)
        out.append(rec)
    return out


BRANCH = ("no_last", "no_velocity", "few_matches", "few_pairs", "no_model", "warped")


def _check_against(st, res, ref_frames):
    kps, desc, nkp, c2l, nm = res
    for t, r in enumerate(ref_frames):
        name, nmatches, npairs, H = st.homography(t)
        assert (name, nmatches, npairs) == (BRANCH[r["branch"]], r["nmatches"], r["npairs"]), t
        Hb = np.zeros(9) if H is None else H.reshape(9)
        assert Hb.tobytes() == np.asarray(r["H"], np.float64).tobytes(), t
        m, f = st.dynamic_mask(t)
        assert (m == r["mask"]).all() and f == r["filtered"], t
        n = int(nkp[t])
        assert n == len(r["kps"]) and kps[t, :n].tobytes() == r["kps"].tobytes(), t
        assert (desc[t, :n] == r["desc"]).all(), t
        assert nm[t] == r["nm"] and (c2l[t, :n] == r["c2l"]).all(), t


def test_chain_equals_restatement():
    from tests import homography_chain_ref as HR
    gray, d16, T = chain_scene(F=12, jump=6, windows=((8, 90),), flat=10)
    F = len(gray)
    st = _tracker(F)
    res = st.track_batch_u16_homography(gray, d16, FACTOR, T, THR)
    want = HR.run(gray, d16.astype(np.float32) * FACTOR, T, 1000, TH, THR)
    _check_against(st, res, want)
    seen = {BRANCH[r["branch"]] for r in want}
    assert {"no_last", "no_velocity", "few_matches", "few_pairs", "warped"} <= seen, seen
    assert any(r["retried"] and r["nmatches"] >= 20 for r in want)   # the 2 th search decided a frame


def test_chain_equals_pinned_entries():
    gray, d16, T = chain_scene()
    F = len(gray)
    st = _tracker(F)
    res = st.track_batch_u16_homography(gray, d16, FACTOR, T, THR)
    ref_frames = host_chain(gray, d16, T)
    seen = [st.homography(t)[0] for t in range(F)]
    print("branches:", seen, "pairs:", [st.homography(t)[2] for t in range(F)])
    _check_against(st, res, ref_frames)
    assert {"no_last", "no_velocity", "few_matches", "few_pairs", "warped"} <= set(seen), seen


def test_no_warp_equals_device_flow():
    gray, d16, T = no_warp_scene()
    F = len(gray)
    a = _tracker(F)
    ra = a.track_batch_u16_homography(gray, d16, FACTOR, T, THR)
    b = _tracker(F)
    rb = b.track_batch_u16_flow(gray, d16, FACTOR, T, None, THR)
    assert all(a.homography(t)[0] != "warped" for t in range(F))
    for x, y in zip(ra, rb):
        assert x.tobytes() == y.tobytes()
    for t in range(F):
        ma, fa = a.dynamic_mask(t)
        mb, fb = b.dynamic_mask(t)
        assert (ma == mb).all() and fa == fb, t


def _pinned(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    return t, t.numpy()


def test_submit_does_not_wait():
    """A 265-frame homography batch (about 16,000 kernels) behind a long spin on the handle's stream: orbs_submit returns
    before the spin ends, so it neither waited for the device nor for room in the launch queue; the results then equal
    those of a synchronous run."""
    import time

    import torch
    base = chain_scene()
    F = 265
    gray, d16, T = (np.ascontiguousarray(np.resize(a, (F,) + a.shape[1:])) for a in base)
    st = _tracker(F)
    want = st.track_batch_u16_homography(gray, d16, FACTOR, T, THR)
    want_h = [st.homography(t) for t in range(F)]
    keep = [_pinned(a) for a in (gray, d16, T.reshape(F, 16))]
    g, d, tt = (k[1] for k in keep)
    out = st.alloc_outputs(F, pinned=True)
    stream = torch.cuda.ExternalStream(st.stream())
    spun = torch.cuda.Event()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(6_000_000_000)   # a few seconds of spinning on the handle's stream
        spun.record(stream)
    t0 = time.perf_counter()
    st.submit_batch_u16_homography(g, d, FACTOR, tt, THR, out)
    took = time.perf_counter() - t0
    still_spinning = not spun.query()
    st.sync()
    assert still_spinning, "orbs_submit waited for the device (%.3f s)" % took
    for x, y in zip(out, want):
        assert x.tobytes() == y.tobytes()
    for t in range(F):
        a, b = st.homography(t), want_h[t]
        assert a[:3] == b[:3] and (a[3] is None) == (b[3] is None)
        assert a[3] is None or a[3].tobytes() == b[3].tobytes()


def test_rejected_forms_change_nothing():
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200._abi import OrbsBatch, OrbsResults, ptr
    gray, d16, T = chain_scene(F=4, jump=2, windows=(), flat=3)
    F = len(gray)
    T16 = T.reshape(F, 16)
    depth = d16.astype(np.float32) * FACTOR
    flow = np.zeros((F, ROWS // 2, COLS // 2, 2), np.float32)
    prev = gray[0].copy()
    st = _tracker(F)
    want = st.track_batch_u16_homography(gray, d16, FACTOR, T, THR)
    want_h = [st.homography(t)[:3] for t in range(F)]
    want_m = [st.dynamic_mask(t)[0] for t in range(F)]

    def host(**kw):
        b = dict(nframes=F, rows=ROWS, cols=COLS, device=0, gray=ptr(gray), depth=None, depth_u16=ptr(d16),
                 depth_factor=float(FACTOR), Tcw=ptr(T16), flow=None, device_flow=1, prev_gray=None,
                 binary_threshold=THR, homography=1)
        b.update(kw)
        return b

    cases = [host(homography=2), host(homography=-1), host(device_flow=0), host(device_flow=0, flow=ptr(flow)),
             host(prev_gray=ptr(prev)), host(depth=ptr(depth), depth_u16=None)]

    def refuse(h, b, with_out=True):
        outs = h.alloc_outputs(F)
        res = OrbsResults(*[ptr(a) for a in outs], h.cap)
        n0 = h.launch_count()
        rc = h._L.orbs_submit(h._h, C.byref(OrbsBatch(**b)), C.byref(res) if with_out else None)
        assert rc == EINVAL, _lib.lib().b200orb_last_error()
        h.sync()
        assert h.launch_count() == n0
        assert all(a.tobytes() == np.zeros_like(a).tobytes() for a in outs)

    for b in cases:
        refuse(st, b)
    # a handle whose keypoint capacity exceeds findHomography's 8192 pairs, if the extractor takes one at all
    for nf in (8200, 8400, 8600, 8800):
        try:
            big = _tracker(F, nfeatures=nf)
        except Exception:
            continue
        n = C.c_int(0)
        if big._L.orbx_max_keypoints_for(big._L.orbs_extractor(big._h), ROWS, COLS, C.byref(n)) == 0 and n.value > 8192:
            refuse(big, host())
            break
    # a device batch with the homography flag (inputs in HBM)
    import torch
    dg, dd, dT = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (gray, depth, T16))
    refuse(st, dict(nframes=F, rows=ROWS, cols=COLS, device=1, gray=dg.data_ptr(), depth=dd.data_ptr(), depth_u16=None,
                    depth_factor=0.0, Tcw=dT.data_ptr(), flow=None, device_flow=0, prev_gray=None,
                    binary_threshold=THR, homography=1), with_out=False)
    # the last batch's results stay readable and unchanged
    assert [st.homography(t)[:3] for t in range(F)] == want_h
    assert all((st.dynamic_mask(t)[0] == want_m[t]).all() for t in range(F))
    again = st.track_batch_u16_homography(gray, d16, FACTOR, T, THR)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(again, want))
    # a batch of another form leaves nothing to read
    st.track_batch_u16(gray, d16, FACTOR, T)
    H = np.zeros(9)
    br, nm, npairs = C.c_int(), C.c_int(), C.c_int()
    assert st._L.orbs_read_homography(st._h, 0, ptr(H), C.byref(br), C.byref(nm), C.byref(npairs)) == EINVAL
