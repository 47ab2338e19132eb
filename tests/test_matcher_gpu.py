"""GPU parity of ORBmatcher::SearchByProjection(Cur, Last) through the C-ABI vs the CPU oracle (bit-exact)."""
import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth
from tests.helpers import frame_views

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def stream_feats(oracle):
    ws = synth.WallStream(seed=1234, n=8)
    R = oracle.RefExtractor(1000, 1.2, 8, 20, 7)
    out = []
    for t in (0, 1, 2, 5):
        gray, depth, rgb, T = ws.frame(t)
        K, D = R(gray)
        out.append((K, D, depth, T))
    return out, R.mvScaleFactor.copy()


@pytest.mark.parametrize("obs", [0, 1])
@pytest.mark.parametrize("th", [15.0, 7.0, 30.0])
def test_projection_last_stream(oracle, stream_feats, obs, th):
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    feats, sf = stream_feats
    m = ORBmatcher(0.9, True)
    for a in range(1, len(feats)):
        Kc, Dc, dc, Tc = feats[a]
        Kl, Dl, dl, Tl = feats[a - 1]
        cur, last = frame_views(oracle, Kc, Dc, dc, Tc, Kl, Dl, dl, Tl, sf, obs=obs)
        n_ref, ref = oracle.search_by_projection_last(cur, last, th, False, 0.9, True)
        n_gpu, gpu = m.SearchByProjection(cur, last, th, False)
        assert n_ref > 50, "test is vacuous: %d matches" % n_ref
        assert n_gpu == n_ref
        assert (gpu == ref).all(), np.nonzero(gpu != ref)[0][:10]


def test_projection_last_noisy_pose_and_flags(oracle, stream_feats):
    """Pose noise, forward/backward motion branches, no orientation check, mono, pre-existing MapPoints."""
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    feats, sf = stream_feats
    rng = np.random.default_rng(7)
    Kc, Dc, dc, Tc = feats[1]
    Kl, Dl, dl, Tl = feats[0]
    for case in range(8):
        T = Tc.copy()
        T[:3, 3] += rng.normal(0, 0.01, 3).astype(np.float32)
        if case == 1:
            T[2, 3] += 0.5     # |tlc.z| > mb: one of the forward/backward octave windows
        if case == 2:
            T[2, 3] -= 0.5
        cur, last = frame_views(oracle, Kc, Dc, dc, T, Kl, Dl, dl, Tl, sf, obs=1)
        if case == 3:
            cur.mp_obs = rng.integers(-1, 3, size=cur.n).astype(np.int32)
        if case == 4:
            last.valid[::3] = 0
        check_ori = case != 5
        mono = case == 6
        m = ORBmatcher(0.9, check_ori)
        n_ref, ref = oracle.search_by_projection_last(cur, last, 15.0, mono, 0.9, check_ori)
        n_gpu, gpu = m.SearchByProjection(cur, last, 15.0, mono)
        assert n_gpu == n_ref and (gpu == ref).all(), "case %d" % case


def test_projection_last_crowded(oracle):
    """Many more than K candidates per window and heavy claiming: exercises the re-walk path."""
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    from orb_slam2_ssd_semantic_b200._abi import FrameView, LastView
    rng = np.random.default_rng(3)
    n = 600
    x = rng.uniform(300, 340, n).astype(np.float32)
    y = rng.uniform(220, 260, n).astype(np.float32)
    base = rng.integers(0, 256, size=(1, 32), dtype=np.uint8)
    desc = np.repeat(base, n, 0)
    flip = rng.integers(0, 256, size=(n, 2), dtype=np.uint8)
    desc[:, :2] ^= flip            # all descriptors within a few bits of each other
    sf = (1.2 ** np.arange(8)).astype(np.float32)
    T = np.eye(4, dtype=np.float32)
    cur = FrameView(x, y, np.zeros(n, np.int32), rng.uniform(0, 360, n).astype(np.float32), np.full(n, -1, np.float32),
                    desc, T, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, 0, 640, 0, 480, sf)
    z = 2.0
    xw = np.stack([(x - synth.CX) * z / synth.FX, (y - synth.CY) * z / synth.FY, np.full(n, z)], 1).astype(np.float32)
    last = LastView(xw, np.ones(n, np.uint8), np.zeros(n, np.int32), rng.uniform(0, 360, n).astype(np.float32), desc,
                    T, mp_obs=np.ones(n, np.int32))
    m = ORBmatcher(0.9, True)
    n_ref, ref = oracle.search_by_projection_last(cur, last, 15.0, False, 0.9, True)
    n_gpu, gpu = m.SearchByProjection(cur, last, 15.0, False)
    assert n_gpu == n_ref and (gpu == ref).all()


def test_hamming_matches_oracle(oracle):
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    rng = np.random.default_rng(0)
    for _ in range(50):
        a, b = rng.integers(0, 256, size=(2, 32), dtype=np.uint8)
        assert ORBmatcher.DescriptorDistance(a, b) == oracle.hamming(a, b) == int(np.unpackbits(a ^ b).sum())


def _points_view(oracle, K, D, depth, T_pts, T_cur, sf, rng, noise=0.0):
    """MapPoints = unprojected keypoints of another frame; the isInFrustum fields are computed here in float like
    src/Frame.cc:387-451 does (the C-ABI takes them as inputs)."""
    from orb_slam2_ssd_semantic_b200._abi import TrackPointsView
    _, _, xw, valid = oracle.stereo_unproject(K, depth, T_pts, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
    R, t = T_cur[:3, :3].astype(np.float32), T_cur[:3, 3].astype(np.float32)
    Pc = (xw @ R.T + t).astype(np.float32)
    invz = (np.float32(1.0) / Pc[:, 2]).astype(np.float32)
    u = (np.float32(synth.FX) * Pc[:, 0] * invz + np.float32(synth.CX)).astype(np.float32) + rng.normal(0, noise, len(K)).astype(np.float32)
    v = (np.float32(synth.FY) * Pc[:, 1] * invz + np.float32(synth.CY)).astype(np.float32) + rng.normal(0, noise, len(K)).astype(np.float32)
    inview = (valid > 0) & (Pc[:, 2] > 0) & (u >= 0) & (u <= 640) & (v >= 0) & (v <= 480)
    xr = (u - np.float32(synth.BF) * invz).astype(np.float32)
    level = np.clip(K["octave"] + rng.integers(-1, 2, len(K)), 0, 7).astype(np.int32)
    vcos = np.where(rng.random(len(K)) < 0.5, 0.9995, 0.9).astype(np.float32)
    return TrackPointsView(inview.astype(np.uint8), u, v, xr, level, vcos, D, mp_obs=rng.integers(0, 3, len(K)).astype(np.int32))


@pytest.mark.parametrize("th", [1.0, 3.0, 5.0])
def test_projection_points_local_map(oracle, stream_feats, th):
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    from orb_slam2_ssd_semantic_b200._abi import FrameView
    feats, sf = stream_feats
    rng = np.random.default_rng(11)
    Kc, Dc, dc, Tc = feats[2]
    ur, _, _, _ = oracle.stereo_unproject(Kc, dc, Tc, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
    for src in (0, 1, 3):
        Kl, Dl, dl, Tl = feats[src]
        F = FrameView(Kc["x"], Kc["y"], Kc["octave"], Kc["angle"], ur, Dc, Tc, synth.FX, synth.FY, synth.CX, synth.CY,
                      synth.BF, 0.0, 640.0, 0.0, 480.0, sf)
        if src == 3:
            F.mp_obs = rng.integers(-1, 2, F.n).astype(np.int32)
        pts = _points_view(oracle, Kl, Dl, dl, Tl, Tc, sf, rng, noise=0.5)
        for ratio in (0.8, 0.6):
            n_ref, ref = oracle.search_by_projection_points(F, pts, th, ratio)
            n_gpu, gpu = ORBmatcher(ratio, True).SearchByProjection(F, pts, th)
            assert n_ref > 20
            assert n_gpu == n_ref and (gpu == ref).all(), (src, th, ratio)


def _bow_view(D, ang, rng, nwords, valid=None):
    """Synthetic FeatureVector: node = a few descriptor bits (stands in for the absent DBoW2 vocabulary)."""
    from orb_slam2_ssd_semantic_b200._abi import BowView
    node = (D[:, 0].astype(np.int64) * 7 + D[:, 5].astype(np.int64)) % nwords
    fv = {}
    for i, w in enumerate(node):
        fv.setdefault(int(w), []).append(i)
    return BowView(D, ang, fv, valid)


@pytest.mark.parametrize("nwords", [3, 40, 400])
def test_search_by_bow(oracle, stream_feats, nwords):
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    feats, sf = stream_feats
    rng = np.random.default_rng(13)
    Kk, Dk, _, _ = feats[0]
    Kf, Df, _, _ = feats[1]
    valid = (rng.random(len(Kk)) < 0.8).astype(np.uint8)
    kf = _bow_view(Dk, Kk["angle"], rng, nwords, valid)
    f = _bow_view(Df, Kf["angle"], rng, nwords)
    for ratio, ori in ((0.7, True), (0.9, True), (0.75, False)):
        n_ref, ref = oracle.search_by_bow(kf, f, ratio, ori)
        n_gpu, gpu = ORBmatcher(ratio, ori).SearchByBoW(kf, f)
        assert n_gpu == n_ref and (gpu == ref).all(), (nwords, ratio, ori)
    assert n_ref > 5


def test_projection_last_huge_frame_uses_unfused_path(oracle):
    """More keypoints than fit the fused kernel's shared memory (and more than its 12-bit keypoint index) -> the separate
    query / grid / candidate / resolve kernels, on a single frame pair."""
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    from orb_slam2_ssd_semantic_b200._abi import FrameView, LastView
    rng = np.random.default_rng(21)
    n = 5000
    x = rng.uniform(5, 635, n).astype(np.float32)
    y = rng.uniform(5, 475, n).astype(np.float32)
    desc = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    sf = (1.2 ** np.arange(8)).astype(np.float32)
    T = np.eye(4, dtype=np.float32)
    cur = FrameView(x, y, rng.integers(0, 8, n), rng.uniform(0, 360, n).astype(np.float32), np.full(n, -1, np.float32), desc,
                    T, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, 0, 640, 0, 480, sf)
    z = 2.0
    m = 3000
    sel = rng.integers(0, n, m)
    xw = np.stack([(x[sel] + rng.normal(0, 2, m) - synth.CX) * z / synth.FX, (y[sel] + rng.normal(0, 2, m) - synth.CY) * z / synth.FY,
                   np.full(m, z)], 1).astype(np.float32)
    d2 = desc[sel].copy()
    d2[:, :3] ^= rng.integers(0, 256, size=(m, 3), dtype=np.uint8)
    last = LastView(xw, np.ones(m, np.uint8), cur.octave[sel], rng.uniform(0, 360, m).astype(np.float32), d2, T,
                    mp_obs=rng.integers(0, 2, m).astype(np.int32))
    n_ref, ref = oracle.search_by_projection_last(cur, last, 15.0, False, 0.9, True)
    n_gpu, gpu = ORBmatcher(0.9, True).SearchByProjection(cur, last, 15.0, False)
    assert n_ref > 500 and n_gpu == n_ref and (gpu == ref).all()


def test_search_projected_relocalisation_variant(oracle, stream_feats):
    """SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist) (src/ORBmatcher.cc:1757-1899) through the
    generic API: the shim side (projection, distance gates, MapPoint::PredictScale src/MapPoint.cc:448-480) is done
    here in float like the reference; the candidate loop / claim rule / rotation prune run on the GPU."""
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    from orb_slam2_ssd_semantic_b200._abi import FrameView, QueriesView
    feats, sf = stream_feats
    rng = np.random.default_rng(17)
    Kc, Dc, dc, Tc = feats[3]
    Kk, Dk, dk, Tk = feats[0]
    ur, _, _, _ = oracle.stereo_unproject(Kc, dc, Tc, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
    _, _, xw, valid = oracle.stereo_unproject(Kk, dk, Tk, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
    R, t = Tc[:3, :3].astype(np.float32), Tc[:3, 3].astype(np.float32)
    Pc = (xw @ R.T + t).astype(np.float32)
    invz = (np.float32(1.0) / Pc[:, 2]).astype(np.float32)
    u = (np.float32(synth.FX) * Pc[:, 0] * invz + np.float32(synth.CX)).astype(np.float32)
    v = (np.float32(synth.FY) * Pc[:, 1] * invz + np.float32(synth.CY)).astype(np.float32)
    Ow = (-R.T @ t).astype(np.float32)
    dist3d = np.linalg.norm(xw - Ow, axis=1).astype(np.float32)
    maxd = dist3d * sf[Kk["octave"]] * np.float32(1.2)          # mfMaxDistance ~ dist * levelScaleFactor (MapPoint.cc:404-417)
    ratio = maxd / dist3d
    lvl = np.clip(np.ceil(np.log(ratio) / np.log(np.float32(1.2))).astype(np.int32), 0, 7)   # PredictScale
    ok = (valid > 0) & (u >= 0) & (u <= 640) & (v >= 0) & (v <= 480) & (rng.random(len(Kk)) < 0.9)
    # last tuple: SearchByProjection(KeyFrame*, Scw, vpPoints, vpMatched, th) (src/ORBmatcher.cc:378-498, loop closing):
    # levels [pred-1, pred], best <= TH_LOW = 50, no orientation check, any matched keypoint is skipped
    for th, orbdist, ori, top in ((10.0, 100, True, 1), (3.0, 64, True, 1), (10.0, 100, False, 1), (10.0, 50, False, 0)):
        q = QueriesView(ok.astype(np.uint8), u, v, (np.float32(th) * sf[lvl]).astype(np.float32), lvl - 1, lvl + top, Dk,
                        Kk["angle"])
        F = FrameView(Kc["x"], Kc["y"], Kc["octave"], Kc["angle"], ur, Dc, Tc, synth.FX, synth.FY, synth.CX, synth.CY,
                      synth.BF, 0.0, 640.0, 0.0, 480.0, sf, mp_obs=np.where(rng.random(len(Kc)) < 0.1, 0, -1).astype(np.int32))
        n_ref, ref = oracle.search_projected(F, q, orbdist, 1, ori)
        n_gpu, gpu = ORBmatcher(0.9, ori).SearchProjected(F, q, orbdist, 1)
        assert n_ref > 30 and n_gpu == n_ref and (gpu == ref).all(), (th, orbdist, ori, top)
    # claim rule 0 with a stereo gate == the LAST semantics on supplied geometry
    q = QueriesView(ok.astype(np.uint8), u, v, (np.float32(15.0) * sf[Kk["octave"]]).astype(np.float32), Kk["octave"] - 1,
                    Kk["octave"] + 1, Dk, Kk["angle"], uright=(u - np.float32(synth.BF) * invz).astype(np.float32),
                    obs=rng.integers(0, 2, len(Kk)).astype(np.int32))
    F.mp_obs = None
    n_ref, ref = oracle.search_projected(F, q, 100, 0, True)
    n_gpu, gpu = ORBmatcher(0.9, True).SearchProjected(F, q, 100, 0)
    assert n_ref > 100 and n_gpu == n_ref and (gpu == ref).all()


@pytest.mark.parametrize("nwords", [5, 60])
def test_search_by_bow_keyframe_keyframe(oracle, stream_feats, nwords):
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    feats, sf = stream_feats
    rng = np.random.default_rng(23)
    K1, D1, _, _ = feats[0]
    K2, D2, _, _ = feats[2]
    k1 = _bow_view(D1, K1["angle"], rng, nwords, (rng.random(len(K1)) < 0.85).astype(np.uint8))
    k2 = _bow_view(D2, K2["angle"], rng, nwords, (rng.random(len(K2)) < 0.85).astype(np.uint8))
    for ratio, ori in ((0.75, True), (0.95, True), (0.8, False)):
        n_ref, ref = oracle.search_by_bow_kf(k1, k2, ratio, ori)
        n_gpu, gpu = ORBmatcher(ratio, ori).SearchByBoWKF(k1, k2)
        assert n_gpu == n_ref and (gpu == ref).all(), (nwords, ratio, ori)
    assert n_ref > 5


@pytest.mark.parametrize("path", sorted(__import__("glob").glob(__import__("os").path.join(__import__("os").path.dirname(__import__("os").path.abspath(__file__)), "golden", "match_mapbin_*.npz"))))
def test_projection_last_on_reference_mapbin_keyframes(oracle, path):
    """GPU SearchByProjection(cur, last) on REAL keyframes of the reference's map.bin (tests/golden/match_mapbin_*.npz:
    real ORB keypoints, descriptors, map points) == the committed golden == the oracle, at three window sizes."""
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    from orb_slam2_ssd_semantic_b200._abi import FrameView, LastView
    z = np.load(path)
    fx, fy, cx, cy, bf = [float(v) for v in z["cam"]]
    cur = FrameView(z["cur_x"], z["cur_y"], z["cur_oct"], z["cur_angle"], z["cur_uright"], z["cur_desc"], z["cur_Tcw"], fx, fy, cx,
                    cy, bf, 0.0, 640.0, 0.0, 480.0, z["sf"])
    last = LastView(z["last_xw"], z["last_valid"], z["last_oct"], z["last_angle"], z["last_desc"], z["last_Tcw"],
                    mp_obs=np.ones(len(z["last_valid"]), np.int32))
    m = ORBmatcher(0.9, True)
    n, c2l = m.SearchByProjection(cur, last, float(z["th"]))
    assert n == int(z["nmatches"]) and (c2l == z["cur2last"]).all() and n > 100
    for th in (7.0, 30.0):
        for mono in (False, True):
            a = m.SearchByProjection(cur, last, th, mono)
            b = oracle.search_by_projection_last(cur, last, th, mono, 0.9, True)
            assert a[0] == b[0] and (a[1] == b[1]).all(), (th, mono)
