"""findHomography(RANSAC, 3) on crafted sets (tests/homography_edge_cases.py): the restatement (tests/homography_lm.py)
against cv2 4.13 live at cv2.setUseOptimized(False), bit for bit on H, mask and found where the refinement runs on fewer
than 100 residual rows, within the BLAS hand-off's bound above; and, for every case, a check that it reaches the edge
it is named after, so that a case which drifts off its edge fails instead of passing silently."""
import os

import numpy as np
import pytest

from oracle import homography_py as HP
from tests import homography_edge_cases as EC
from tests import homography_lm as HL

CASES = {name: (src, dst) for name, src, dst in EC.cases()}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "homography_edges.npz")
NINE = np.float32(9.0)


@pytest.fixture
def cv2():
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    cv2.setUseOptimized(False)
    yield cv2
    cv2.setUseOptimized(was)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _same(a, b):
    (Ha, ma), (Hb, mb) = a, b
    return (Ha is None) == (Hb is None) and (Ha is None or (_bits(Ha) == _bits(Hb)).all()) and (ma == mb).all()


def exact(src, dst) -> bool:
    """cv2 sums J^T r itself (and equals the restatement bit for bit) below 100 residual rows, i.e. 50 inliers."""
    if len(src) == 4:
        return True
    inl = HP.ransac(src, dst)[1]
    return inl is None or int(inl.sum()) < 50


# ---- readings that OpenCV does not use: each case that targets them must tell them apart -------------------------------


def _collinear_double(P) -> bool:
    """haveCollinearPoints with exact double differences (OpenCV subtracts in float)."""
    i = len(P) - 1
    for j in range(i):
        dx1, dy1 = float(P[j][0]) - float(P[i][0]), float(P[j][1]) - float(P[i][1])
        for k in range(j):
            dx2, dy2 = float(P[k][0]) - float(P[i][0]), float(P[k][1]) - float(P[i][1])
            if abs(dx2 * dy1 - dy2 * dx1) <= HP.FLT_EPS * (abs(dx1) + abs(dy1) + abs(dx2) + abs(dy2)):
                return True
    return False


def _dot_two_lanes(a, b) -> float:
    """Mat::dot as one v_float64x2 accumulator over blocks of 4 (not OpenCV's baseline order)."""
    p = np.asarray(a, np.float64).ravel() * np.asarray(b, np.float64).ravel()
    n4 = len(p) // 4 * 4
    return (0.0 + (HL._seq(p[0:n4:2]) + HL._seq(p[1:n4:2]))) + HL._seq(p[n4:])


def _with(monkeypatch, obj, attr, fn, src, dst):
    with monkeypatch.context() as m:
        m.setattr(obj, attr, fn)
        return HL.find_homography(src, dst)


def trace(src, dst):
    """RANSACPointSetRegistrator::run's loop, recorded: -> dict(hyps=[(subset, H, good)], best, max_good, it,
    exhausted) where exhausted says getSubset gave up (10000 rejections in a row)."""
    n = len(src)
    rng = HP.CvRNG()
    niters, max_good, best, it, hyps = HL.MAX_ITERS, 0, -1, 0, []
    while it < niters:
        idx = HP.get_subset(src, dst, rng)
        if idx is None:
            return dict(hyps=hyps, best=best, max_good=max_good, it=it, exhausted=True)
        H = HP.run_kernel(src[idx], dst[idx])
        good = -1
        if H is not None:
            good = int((HP.reprojection_errors(H, src, dst) <= NINE).sum())
            if good > max(max_good, 3):
                best, max_good = it, good
                niters = HP.update_num_iters(HL.CONFIDENCE, (n - good) / n, 4, niters)
        hyps.append((idx, H, good))
        it += 1
    return dict(hyps=hyps, best=best, max_good=max_good, it=it, exhausted=False)


def _first(name):
    src, dst = CASES[name]
    sub = EC.subset_stream(len(src), 1)[0]
    return src[sub], dst[sub]


def _neg(s, d) -> int:
    neg = 0
    for t in ((0, 1, 2), (1, 2, 3), (0, 2, 3), (0, 1, 3)):
        a = HP._det3([[float(s[q][0]), float(s[q][1]), 1.0] for q in t])
        b = HP._det3([[float(d[q][0]), float(d[q][1]), 1.0] for q in t])
        neg += a * b < 0
    return neg


# ---- edge checks, one per case ----------------------------------------------------------------------------------------


def _edge_collinear_split(name, float_says):
    def check(src, dst, monkeypatch):
        s, d = _first(name)
        assert HP._collinear(s) == float_says and _collinear_double(s) == (not float_says)
        with monkeypatch.context() as m:
            m.setattr(HP, "_collinear", _collinear_double)
            double_verdict = HP.check_subset(s, d)
        assert HP.check_subset(s, d) != double_verdict
    return check


def _edge_result_depends_on_collinear_reading(src, dst, monkeypatch):
    assert not _same(HL.find_homography(src, dst), _with(monkeypatch, HP, "_collinear", _collinear_double, src, dst))


def _edge_16126(src, dst, monkeypatch):
    _edge_result_depends_on_collinear_reading(src, dst, monkeypatch)
    assert not _same(HL.find_homography(src, dst), _with(monkeypatch, HL, "dot", _dot_two_lanes, src, dst))


def _edge_first_subset_collinear(name, coincident=False, near=False):
    def check(src, dst, monkeypatch):
        s, d = _first(name)
        assert HP._collinear(s) and _collinear_double(s) and not HP.check_subset(s, d)
        if coincident:
            assert (s[3] == s[1]).all()
        if near:
            assert (s[3] != s[0]).any() and np.abs(s[3] - s[0]).max() == np.spacing(np.float32(0.0625))
    return check


def _edge_integer_agree(src, dst, monkeypatch):
    assert (src == np.rint(src)).all() and (dst == np.rint(dst)).all()
    for sub in EC.subset_stream(len(src), 200):
        for P in (src[sub], dst[sub]):
            assert HP._collinear(P) == _collinear_double(P)


def _edge_orient(k):
    def check(src, dst, monkeypatch):
        s, d = _first("orient_%d_flipped" % k)
        assert not HP._collinear(s) and not HP._collinear(d)
        assert _neg(s, d) == k
        assert HP.check_subset(s, d) == (k in (0, 4))
    return check


def _edge_zero_det(mirrored):
    def check(src, dst, monkeypatch):
        s, d = _first("orient_zero_det_" + ("mirrored" if mirrored else "kept"))
        tri = [[float(s[q][0]), float(s[q][1]), 1.0] for q in (0, 1, 2)]
        trd = [[float(d[q][0]), float(d[q][1]), 1.0] for q in (0, 1, 2)]
        assert HP._det3(tri) == 0.0 and HP._det3(trd) != 0.0
        assert _neg(s, d) == (3 if mirrored else 0)
        assert HP.check_subset(s, d) == (not mirrored)
    return check


def _edge_exhausted_no_model(src, dst, monkeypatch):
    t = trace(src, dst)
    assert t["exhausted"] and t["it"] == 0 and HL.find_homography(src, dst)[0] is None


def _edge_exhausted_after_first(src, dst, monkeypatch):
    t = trace(src, dst)
    assert t["exhausted"] and t["it"] == 1 and t["best"] == 0 and t["max_good"] >= 4
    assert HL.find_homography(src, dst)[0] is not None


def _edge_threshold(src, dst, monkeypatch):
    t = trace(src, dst)
    H = HL.find_homography(src, dst)[0]
    above = np.nextafter(NINE, np.float32(np.inf))
    for model in (t["hyps"][t["best"]][1], H):
        e = HP.reprojection_errors(model, src, dst)
        assert e[EC.THRESH_PAIR] == NINE and e[EC.THRESH_PAIR + 1] == NINE and e[EC.ABOVE_PAIR] == above
    m = HL.find_homography(src, dst)[1]
    assert m[EC.THRESH_PAIR] == 1 and m[EC.THRESH_PAIR + 1] == 1 and m[EC.ABOVE_PAIR] == 0


def _edge_scan_3(src, dst, monkeypatch):
    t = trace(src, dst)
    assert t["hyps"][0][2] == 3 and t["best"] > 0 and t["max_good"] > 3


def _edge_scan_equal(src, dst, monkeypatch):
    t = trace(src, dst)
    b = t["best"]
    later = [h for h in t["hyps"][b + 1:] if h[2] == t["max_good"]]
    assert later and any(not (_bits(h[1]) == _bits(t["hyps"][b][1])).all() for h in later)
    Hb = t["hyps"][b][1]
    assert any(np.abs(h[1] - Hb).max() > 1e-3 * np.abs(Hb).max() for h in later)   # another model, not a rounding


def _edge_scan_all_inliers(src, dst, monkeypatch):
    t = trace(src, dst)
    assert t["it"] == 1 and t["max_good"] == len(src)
    assert 1.0 - (1.0 - 0.0) ** 4 < HP.DBL_MIN and HP.update_num_iters(HL.CONFIDENCE, 0.0, 4, HL.MAX_ITERS) == 0


def _edge_scan_clamp(src, dst, monkeypatch):
    t = trace(src, dst)
    n, g = len(src), t["max_good"]
    num, denom = np.log(1 - HL.CONFIDENCE), np.log(1.0 - (1.0 - (n - g) / n) ** 4)
    assert -num >= HL.MAX_ITERS * -denom      # the clamp, not the rounded quotient
    assert HP.update_num_iters(HL.CONFIDENCE, (n - g) / n, 4, HL.MAX_ITERS) == HL.MAX_ITERS and t["it"] == HL.MAX_ITERS


def _deviation(P, axis):
    P = np.asarray(P, np.float32)
    c = 0.0
    for v in P[:, axis]:
        c += float(v)
    c /= len(P)
    return sum(abs(float(v) - c) for v in P[:, axis])


def _edge_degenerate(side, axis, below, zero=False):
    def check(src, dst, monkeypatch):
        s = _deviation(src if side == "src" else dst, axis)
        assert (s == 0.0) if zero else ((0.0 < s < HP.DBL_EPS) if below else (HP.DBL_EPS < s < 4 * HP.DBL_EPS))
        assert (HP.run_kernel(src, dst) is None) == below
        assert (HL.find_homography(src, dst)[0] is None) == below
    return check


def _edge_zero_residuals(src, dst, monkeypatch):
    """the identity: half the residuals are exactly 0, all of them below FLT_EPSILON, and the LM stops on its residual
    criterion after one iteration"""
    x, it = HL.lm_refine(HP.run_kernel(src, dst), src, dst)
    r, _ = HL.refine_residuals(x, src, dst)
    assert it == 1 and HL.norm_inf(r) < HL.FLT_EPS and (r == 0.0).sum() >= len(r) // 2


def _edge_large_coords(src, dst, monkeypatch):
    assert src.min() >= 1e4 and dst.min() >= 5e3 and max(src.max(), dst.max()) >= 9e4


def _edge_negative_coords(src, dst, monkeypatch):
    assert (src < 0).all() and (dst < 0).mean() > 0.5


def _edge_mask_differs(src, dst, monkeypatch):
    inl = HP.ransac(src, dst)[1]
    assert (inl.astype(np.uint8) != HL.find_homography(src, dst)[1]).any()


def _edge_count(n, side):
    def check(src, dst, monkeypatch):
        assert len(src) == n
        if n > 4:
            g = int(HP.ransac(src, dst)[1].sum())
            assert (g < 50) == (side == "below"), g
    return check


def _edge_level0(src, dst, monkeypatch):
    assert (src == np.rint(src)).all() and (dst == np.rint(dst)).all()


def _edge_scaled(src, dst, monkeypatch):
    for P in (src, dst):
        ok = np.zeros(len(P), bool)
        for s in EC.LEVEL_SCALES:
            q = np.rint(P.astype(np.float64) / float(s)).astype(np.float32)
            ok |= ((q * s).astype(np.float32) == P).all(1)
        assert ok.all()
    assert (src != np.rint(src)).any()


EDGES = {
    "collinear_float_only": _edge_collinear_split("collinear_float_only", True),
    "collinear_double_only": _edge_collinear_split("collinear_double_only", False),
    "collinear_cv2_13541": _edge_result_depends_on_collinear_reading,
    "collinear_cv2_16126_lm_dot": _edge_16126,
    "collinear_exact": _edge_first_subset_collinear("collinear_exact"),
    "collinear_coincident": _edge_first_subset_collinear("collinear_coincident", coincident=True),
    "collinear_near_coincident": _edge_first_subset_collinear("collinear_near_coincident", near=True),
    "collinear_horizontal": _edge_first_subset_collinear("collinear_horizontal"),
    "collinear_vertical": _edge_first_subset_collinear("collinear_vertical"),
    "collinear_integer_agree": _edge_integer_agree,
    **{"orient_%d_flipped" % k: _edge_orient(k) for k in range(5)},
    "orient_zero_det_mirrored": _edge_zero_det(True),
    "orient_zero_det_kept": _edge_zero_det(False),
    "draws_exhausted_no_model": _edge_exhausted_no_model,
    "draws_exhausted_after_first_hypothesis": _edge_exhausted_after_first,
    "threshold_exactly_9": _edge_threshold,
    "scan_first_hypothesis_3_inliers": _edge_scan_3,
    "scan_equal_counts_keep_first": _edge_scan_equal,
    "scan_all_inliers_one_iteration": _edge_scan_all_inliers,
    "scan_max_iters_clamp": _edge_scan_clamp,
    "degenerate_n4_src_x_constant": _edge_degenerate("src", 0, True, zero=True),
    "degenerate_n4_src_y_below_dbl_eps": _edge_degenerate("src", 1, True),
    "degenerate_n4_dst_x_above_dbl_eps": _edge_degenerate("dst", 0, False),
    "refine_zero_residuals": _edge_zero_residuals,
    "refine_coords_1e4_1e5": _edge_large_coords,
    "refine_negative_coords": _edge_negative_coords,
    "refine_mask_differs_from_ransac": _edge_mask_differs,
    "count_n4": _edge_count(4, "below"),
    "count_n5": _edge_count(5, "below"),
    "count_n50_out1": _edge_count(50, "below"),
    "count_n50_out0": _edge_count(50, "below"),
    "count_n51_out2": _edge_count(51, "below"),
    "count_n51_out1": _edge_count(51, "above"),
    "count_n99_out50": _edge_count(99, "below"),
    "count_n99_out20": _edge_count(99, "above"),
    "count_n100_out51": _edge_count(100, "below"),
    "count_n100_out30": _edge_count(100, "above"),
    "trackhomo_level0_integers": _edge_level0,
    "trackhomo_scaled_levels": _edge_scaled,
}


def test_every_case_has_an_edge_check():
    assert sorted(EDGES) == sorted(CASES)


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_reaches_its_edge(name, monkeypatch):
    EDGES[name](*CASES[name], monkeypatch)


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_equals_cv2(cv2, name):
    src, dst = CASES[name]
    H, mask = cv2.findHomography(src, dst, cv2.RANSAC, 3)
    mask = np.zeros(len(src), np.uint8) if mask is None else mask.ravel()
    mine, mmask = HL.find_homography(src, dst)
    assert (H is None) == (mine is None)
    if exact(src, dst):
        assert _same((mine, mmask), (H, mask))
    else:
        assert np.abs(mine - H).max() <= 1e-6 * np.abs(H).max()
        assert (mmask != mask).sum() <= max(2, len(src) // 500)


def test_golden_equals_restatement():
    """tests/golden/homography_edges.npz (cv2's results, written by tools/make_homography_edges_golden.py) holds these
    very sets, and the restatement reproduces it."""
    z = np.load(GOLDEN)
    assert sorted(str(n) for n in z["names"]) == sorted(CASES)
    for name, (src, dst) in CASES.items():
        assert (z[name + "/src"] == src).all() and (z[name + "/dst"] == dst).all(), name
        Hc = z[name + "/H"]
        Hc = None if np.isnan(Hc).any() else Hc
        mine = HL.find_homography(src, dst)
        assert bool(z[name + "/exact"]) == exact(src, dst), name
        if exact(src, dst):
            assert _same(mine, (Hc, z[name + "/mask"])), name
        else:
            assert np.abs(mine[0] - Hc).max() <= 1e-6 * np.abs(Hc).max(), name


def test_both_sides_of_the_hand_off_are_covered():
    sides = [exact(*CASES[n]) for n in CASES if n.startswith("count_n")]
    assert any(sides) and not all(sides)


def test_dot_is_unrolled_by_four():
    """Mat::dot's order on a vector where the two orders round differently: ((p0 + p1) + p2) + p3 per block of four."""
    a = np.array([1.0, 1e16, -1e16, 1.0, 1.0, 2.0 ** -60, 3.0, -3.0, 0.5])
    b = np.ones(9)
    assert HL.dot(a, b) == ((((1.0 + 1e16) + -1e16) + 1.0) + (((1.0 + 2.0 ** -60) + 3.0) + -3.0)) + 0.5
    assert HL.dot(a, b) != _dot_two_lanes(a, b)
