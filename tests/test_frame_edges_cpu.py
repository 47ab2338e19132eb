"""The crafted Frame-member cases of tests/frame_cases.py on the CPU: every case really contains the edge it names
(recomputed here in numpy, with libm's logf through ctypes), and the flat oracles equal the reference's own sources on
them -- Frame::isInFrustum + MapPoint::PredictScale and Frame::UndistortKeyPoints / ComputeStereoFromRGBD /
UnprojectStereo (src/Frame.cc, src/MapPoint.cc through oracle/_ref/librefsrc.so), cv2.undistortPoints, and
Frame::ComputeBoW on the DBoW2 stand-in.  The reference's results are pinned as digests in
tests/golden/frame_edges_pins.json (tests/refpins.py's format): where oracle/_ref is built they are also compared live;
REFSRC_RECORD=1 rewrites them."""
import json
import math
import os

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth
from tests import frame_cases as FC
from tests.refpins import RECORD, Pins, digest

CASES = FC.all_cases()
FRUSTUM = [c for c in CASES if c.kind == "frustum"]
BOW = [c for c in CASES if c.kind == "bow"]
PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frame_edges_pins.json")
GOLDEN_CV2 = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "undistort_cv2.npz")
f32 = np.float32


class FramePins(Pins):
    """Pinned digests; the reference is also run live where oracle/_ref is built."""

    def __init__(self, live):
        self.live = live
        self.d = {}
        if os.path.exists(PINS):
            with open(PINS) as f:
                self.d = json.load(f)

    def check(self, key, ours, reference):
        if self.live and not RECORD:
            assert digest(reference()) == digest(ours), key
        super().check(key, ours, reference)

    def save(self):
        if RECORD:
            with open(PINS, "w") as f:
                json.dump(self.d, f, indent=0, sort_keys=True)
                f.write("\n")


@pytest.fixture(scope="module")
def pins(oracle):
    live = os.path.exists(oracle._REFSO) or RECORD
    if live:
        oracle.reflib()
    p = FramePins(live)
    yield p
    p.save()


def _unclamped_level(r, lsf):
    return math.ceil(float(f32(FC.logf(r) / f32(lsf))))


@pytest.mark.parametrize("case", FRUSTUM, ids=[c.name for c in FRUSTUM])
def test_frustum_case_contains_its_edge(case):
    assert case.edges
    m = FC.frustum_mirror(case)
    F = case.kw["F"]
    for e in case.edges:
        if e[0] == "eq":
            _, q, i, want = e
            assert FC.bits(m[q][i]) == FC.bits(want), (e, m[q][i])
        elif e[0] == "nan":
            assert np.isnan(m[e[1]][e[2]]), e
        elif e[0] == "bounds":
            lo_x, hi_x, lo_y, hi_y = (f32(b) for b in F.bounds)
            u, v = m["u"], m["v"]
            on = [u[1] == lo_x, u[0] == hi_x, v[3] == lo_y, v[2] == hi_y]
            one_ulp_in = [FC.down(u[1]) == lo_x, FC.up(u[0]) == hi_x, FC.down(v[3]) == lo_y, FC.up(v[2]) == hi_y]
            one_ulp_out = [FC.up(u[1]) == lo_x, FC.down(u[0]) == hi_x, FC.up(v[3]) == lo_y, FC.down(v[2]) == hi_y]
            assert all({"on": on, "inside": one_ulp_in, "outside": one_ulp_out}[e[1]]), e
        elif e[0] == "threshold":
            _, k, t = e
            lsf = case.kw["lsf"]
            assert _unclamped_level(t, lsf) <= k < _unclamped_level(FC.up(t), lsf), e
            assert any(FC.bits(r) == FC.bits(t) for r in m["ratio"])
        elif e[0] == "level":
            _, i, lvl = e
            assert FC.predict_level(m["ratio"][i], case.kw["lsf"], case.kw["nlevels"]) == lvl, e
        else:
            raise AssertionError(e)


def test_every_frustum_gate_is_crossed():
    """Over all cases: both signed zeros and both subnormal signs of PcZ, and for each scale factor 1.2 / 1.5 / 2.0 and
    nlevels 1 / 8 / MAX_LEVELS a ratio on every threshold, both its neighbours, one below 1 and one past the top."""
    names = {c.name for c in FRUSTUM}
    for sf in ("1.2", "1.5", "2.0"):
        for nl in (1, 8, FC.MAX_LEVELS):
            assert "predict/sf%s/nl%d" % (sf, nl) in names
    for c in FRUSTUM:
        if c.name.startswith("predict/"):
            m = FC.frustum_mirror(c)
            nl = c.kw["nlevels"]
            assert (m["ratio"] < 1).any() and max(FC.predict_level(r, c.kw["lsf"], nl) for r in m["ratio"]) == nl - 1
            assert sum(e[0] == "threshold" for e in c.edges) == nl - 1


def frustum_oracle(oracle, case, which="oracle"):
    """The six outputs of isInFrustum; the level of a point whose ratio the reference feeds to (int)ceil(inf / NaN)
    (undefined behaviour) is left out."""
    kw = case.kw
    r = oracle.is_in_frustum(kw["F"], kw["xw"], kw["normal"], kw["mind"], kw["maxd"], kw["cos_limit"], kw["lsf"], which)
    return list(r[:4]) + [r[4][~kw["undefined"]], r[5]]


def test_frustum_oracle_equals_reference_sources(oracle, pins):
    """match_ref_is_in_frustum == the reference's Frame::isInFrustum + MapPoint::PredictScale on every crafted case."""
    for case in FRUSTUM:
        pins.check("frame_edges/%s" % case.name, frustum_oracle(oracle, case),
                   lambda: frustum_oracle(oracle, case, "refsrc"))


@pytest.mark.parametrize("case", BOW, ids=[c.name for c in BOW])
def test_bow_case_contains_its_edge(case):
    kw = case.kw
    t, nd, desc = kw["tree"], kw["node_desc"], kw["desc"]
    parent = kw["parent"]
    depth = np.zeros(len(parent), int)
    for i in range(1, len(parent)):
        depth[i] = depth[parent[i]] + 1
    is_leaf = FC.leaf_word_ids(parent) >= 0
    for e in case.edges:
        if e[0] == "nchildren":
            assert len(t.children(e[1])) == e[2] > 32, e
        elif e[0] == "fewer":
            counts = [len(t.children(i)) for i in range(len(parent)) if not is_leaf[i] and i]
            assert min(counts) < t.k, counts
        elif e[0] == "picks":   # feature f is closest to child `want` of its level-`lvl` choice, with want >= 32
            _, f, lvl, want = e
            sib = t.children(parent[want])
            d = [FC.hamming(desc[f], nd[c]) for c in sib]
            assert sib.index(want) >= 32 and d[sib.index(want)] == 0 and d.count(0) == 1
        elif e[0] == "tie":   # feature f is at one minimal distance from two siblings
            _, f, lvl, (a, b) = e
            sib = t.children(parent[a])
            d = [FC.hamming(desc[f], nd[c]) for c in sib]
            assert b in sib and d[sib.index(a)] == d[sib.index(b)] == min(d) and sib.index(a) < sib.index(b)
        elif e[0] == "stopped":
            w = kw["weight"]
            hits = {FC.descend(parent, nd, w, np.arange(len(parent)), d, kw["L"], 4)[0] for d in desc}
            assert any(w[h] == 0 for h in hits) and any(w[h] > 0 for h in hits)
        elif e[0] == "n_mod8":
            assert len(desc) % 8 != 0
        elif e[0] == "depths":
            ld = depth[is_leaf]
            assert ld.min() == e[1] and ld.max() == e[2]
        elif e[0] == "shallow_hit":   # some feature ends on a leaf above the FeatureVector's node level
            lv = kw["L"] - e[1]
            ends = [FC.descend(parent, nd, kw["weight"], np.arange(len(parent)), d, kw["L"], 4)[0] for d in desc]
            assert any(depth[x] < lv and kw["weight"][x] > 0 for x in ends)
        elif e[0] == "same_word":   # one live word hit by many features
            ends = [FC.descend(parent, nd, kw["weight"], np.arange(len(parent)), d, kw["L"], 4)[0] for d in desc]
            assert max(ends.count(x) for x in set(ends) if kw["weight"][x] > 0) >= e[1]
        elif e[0] == "live":        # feature f ends on a word that is not stopped
            end = FC.descend(parent, nd, kw["weight"], np.arange(len(parent)), desc[e[1]], kw["L"], 4)[0]
            assert kw["weight"][end] > 0
        elif e[0] == "d256":        # the walk of feature f leaves `node` with every child at distance 256
            _, f, node = e
            trace = []
            FC.descend(parent, nd, kw["weight"], np.arange(len(parent)), desc[f], kw["L"], 4, trace)
            at = [dists for cur, dists in trace if cur == node]
            assert len(at) == 1 and len(at[0]) == t.k and set(at[0]) == {256}, trace
        elif e[0] == "permuted":
            wid = kw["word_id"][is_leaf]
            assert len(set(wid.tolist())) == len(wid) and (np.diff(wid) < 0).any()
        else:
            raise AssertionError(e)


def test_bow_restatements_agree_on_crafted_trees(oracle, pins):
    """oracle.bow_transform_py == Frame::ComputeBoW of the reference on the DBoW2 stand-in (levelsup 4, word ids in leaf
    order: what the reference can take); and, at every levelsup a case names, the per-feature descent of
    tests/frame_cases.py assembled like TemplatedVocabulary::transform == bow_transform_py.  On the shallow-leaf case
    the walk never reaches the FeatureVector's level for some features: the stand-in starts from node 0 there, where
    DBoW2 reads an uninitialised NodeId -- the node id of those features is the stand-in's, not a DBoW2 guarantee."""
    for case in BOW:
        kw = case.kw
        args = (kw["k"], kw["L"], kw["parent"], kw["node_desc"], kw["weight"], kw["desc"])
        ours = oracle.bow_transform_py(*args, levelsup=4)
        pins.check("frame_edges/%s" % case.name, ours, lambda: oracle.src_bow_transform(*args, "refsrc"))
        for ls in kw["levelsups"]:
            asc = FC.Case(case.name, "bow", dict(kw, word_id=None), [])
            assert digest(FC.assemble(*FC.bow_expected_raw(asc, ls))) == digest(oracle.bow_transform_py(*args, levelsup=ls)), \
                (case.name, ls)


def test_undistort_oracle_equals_cv2():
    """orb_ref_undistort == cv2.undistortPoints (OpenCV 4.13, stored in tests/golden/undistort_cv2.npz by
    tools/make_undistort_golden.py; also live where cv2 imports) on every crafted set whose k1 is non-zero, the
    icdist < 0 exits included; where k1 is zero or -0.0, Frame::UndistortKeyPoints copies the keypoints."""
    from oracle import ref
    z = np.load(GOLDEN_CV2)
    xy, K = z["xy"], z["K"]
    assert xy.tobytes() == FC.undistort_points().tobytes() and K.tobytes() == FC.UNDIST_K.tobytes()
    try:
        import cv2
    except ImportError:
        cv2 = None
    n_icdist = 0
    for name, d in FC.undistort_cases():
        got = ref.undistort(xy, K, d)
        key = name.split("/", 1)[1]
        if len(d) == 0 or d[0] == 0:
            assert got.tobytes() == xy.tobytes(), name
            assert "out/" + key not in z.files
            continue
        assert z["dist/" + key].tobytes() == d.tobytes(), name
        assert got.tobytes() == z["out/" + key].tobytes(), name
        if cv2 is not None:
            live = cv2.undistortPoints(xy.reshape(-1, 1, 2), K.reshape(3, 3), d, None, K.reshape(3, 3)).reshape(-1, 2)
            assert got.tobytes() == np.asarray(live, np.float32).tobytes(), name
        n_icdist += int(FC.undistort_icdist(xy, K, d).sum())
    assert n_icdist > 100


def test_undistort_cases_contain_their_edges():
    names = dict(FC.undistort_cases())
    xy = FC.undistort_points()
    assert FC.bits(names["undistort/k1_negative_zero_copies_ndist5"][0]) == 0x80000000
    assert FC.bits(names["undistort/k1_negative_zero_copies_ndist4"][0]) == 0x80000000
    assert (names["undistort/k1_zero_copies_despite_k2_p1_p2"][1:] != 0).all()
    for n in ("undistort/icdist_negative", "undistort/icdist_negative_k3", "undistort/ndist5_k3_icdist_negative"):
        hit = FC.undistort_icdist(xy, FC.UNDIST_K, names[n])
        assert hit.any() and not hit.all(), n
    assert FC.UNDIST_K[0] != FC.UNDIST_K[4]
    assert ((xy == [FC.UNDIST_K[2], FC.UNDIST_K[5]]).all(1)).any()
    assert (np.abs(xy) > 5000).any()
    assert {len(d) for d in names.values()} == {0, 4, 5}


def test_undistort_oracle_equals_reference_frame(oracle, pins):
    """UndistortKeyPoints through the reference's RGB-D Frame constructor (four coefficients, the harness's form) on the
    crafted coefficient sets: the copy short-cut at k1 = 0 and k1 = -0.0, ndist 4, and a strong negative k1."""
    assert sum(len(d) == 4 and d[0] == 0 and np.signbit(d[0]) for _, d in FC.undistort_cases()) == 1
    gray = synth.synth_frame(77, 0)
    depth = np.ones(gray.shape, np.float32)
    K = FC.UNDIST_K
    kps, _ = oracle.RefExtractor(600, 1.2, 8, 20, 7)(gray)
    xy = np.stack([kps["x"], kps["y"]], 1)
    for name, d in FC.undistort_cases():
        if len(d) != 4:
            continue
        un = oracle.undistort(xy, K, d)

        def reference():
            Kun = oracle.src_frame_rgbd(gray, depth, np.eye(4, dtype=np.float32), K[0], K[4], K[2], K[5], FC.BF,
                                        nfeatures=600, dist=d)[0]
            return Kun["x"], Kun["y"]
        pins.check("frame_edges/frame_%s" % name, (un[:, 0], un[:, 1]), reference)


def glue_inputs(oracle, u16):
    """(gray, float depth the reference sees, CV_16U depth or None, keypoints) of the crafted glue frame."""
    gray = synth.synth_frame(4321, 1)
    kps, _ = oracle.RefExtractor(1000, 1.2, 8, 20, 7)(gray)
    if u16:
        d16 = FC.glue_depth_u16(*gray.shape, kps)
        return gray, d16.astype(f32) * FC.DEPTH_FACTOR, d16, kps
    return gray, FC.glue_depth(*gray.shape, kps), None, kps


def glue_oracle(oracle, kps, depth):
    ur, dp, xw, va = oracle.stereo_unproject(kps, depth, FC.GLUE_T, FC.FX, FC.FY, FC.CX, FC.CY, FC.BF)
    return ur, dp, va, xw[va > 0]


@pytest.mark.parametrize("u16", [False, True], ids=["float", "u16"])
def test_glue_case_contains_its_edges(oracle, u16):
    gray, depth, d16, kps = glue_inputs(oracle, u16)
    px = depth[kps["y"].astype(int), kps["x"].astype(int)]
    if u16:
        raw = d16[kps["y"].astype(int), kps["x"].astype(int)]
        assert (raw == 0).any() and (raw == 65535).any()
    else:
        for e in FC.GLUE_EDGE:
            assert (FC.bits(px) == FC.bits(e)).any() or (np.isnan(e) and np.isnan(px).any()), e
        with np.errstate(all="ignore"):
            assert np.isinf(f32(FC.BF) / px[px > 0]).any()
    # level > 0 coordinates just below an integer: truncation and rounding read different pixels with different depths
    frac_y = kps["y"] - np.floor(kps["y"])
    near = (kps["octave"] > 0) & (frac_y > 0.99)
    assert near.any()
    yi, xi = kps["y"].astype(int), kps["x"].astype(int)
    assert (FC.bits(depth[yi[near], xi[near]]) != FC.bits(depth[np.minimum(yi[near] + 1, gray.shape[0] - 1), xi[near]])).all()


@pytest.mark.parametrize("u16", [False, True], ids=["float", "u16"])
def test_glue_oracle_equals_reference_sources(oracle, pins, u16):
    """frame_ref_stereo_unproject == the reference's ComputeStereoFromRGBD + UnprojectStereo (its RGB-D Frame
    constructor) on the crafted depth images: the d > 0 gate on 0, -0.0, negative, NaN, +inf, subnormal and tiny depth,
    and the (int) truncation of level > 0 coordinates."""
    gray, depth, _, kps = glue_inputs(oracle, u16)
    ours = glue_oracle(oracle, kps, depth)

    def reference():
        K2, _, ur, dp, xw, va = oracle.src_frame_rgbd(gray, depth, FC.GLUE_T, FC.FX, FC.FY, FC.CX, FC.CY, FC.BF)
        assert K2.tobytes() == kps.tobytes()
        return ur, dp, va, xw[va > 0]
    pins.check("frame_edges/glue_%s" % ("u16" if u16 else "float"), ours, reference)
    assert 0 < ours[2].sum() < len(kps)
