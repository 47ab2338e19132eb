"""The crafted dynamic-mask cases of tests/dynmask_cases.py on the CPU: every case reaches the edge it is named after
(checked on the oracle's intermediate masks, the float32 sums and the Farneback restatement's pyramid), the mask oracle
equals cv2 live on every mask case, and the Farneback restatement equals cv2 at its baseline dispatch on every flow case
(both skipped without cv2)."""
import numpy as np
import pytest

from oracle import dynmask_py as O
from oracle import farneback_py as FB
from tests import dynmask_cases as D

MASKS = D.mask_cases()
LOOKUPS = D.lookup_cases()
FLOWS = D.flow_cases()


def _line(m, axis):
    """The 0/1 profile of a mask that is constant along the other axis (asserted)."""
    ref = m[0] if axis == 1 else m[:, 0]
    assert ((m == ref[None, :]) if axis == 1 else (m == ref[:, None])).all()
    return ref


def _check_mask_edge(case, st, kind, p):
    m0, e1, e2, fin = st
    H, W = case.shape
    if kind == "band":
        axis, s, e = p
        want = np.zeros(W if axis == 1 else H, np.uint8)
        want[s:e] = 1
        assert (_line(m0, axis) == want).all()
    elif kind == "survive":
        axis, cols = p
        got = np.nonzero(_line(e2, axis))[0].tolist()
        assert got == list(cols)
        assert fin.any() == bool(cols)
    elif kind == "phase":
        (pp,) = p
        surv = [e for e in case.edges if e[0] == "survive"][0][2]
        assert len(surv) == 1 and surv[0] % 32 == pp
    elif kind == "word":
        word, nw = p
        surv = [e for e in case.edges if e[0] == "survive"][0][2]
        assert surv[0] // 32 == word and (W + 31) // 32 == nw
    elif kind == "side":
        (side,) = p
        axis, s, e = [x for x in case.edges if x[0] == "band"][0][1:]
        n = W if axis == 1 else H
        width = e - s
        assert (s == 0) == (side in ("left", "top")) and (e == n) == (side in ("right", "bottom"))
        # outside pixels never erode: each erosion takes 10 px off the inner edge only
        for m, k in ((e1, 10), (e2, 20)):
            want = np.zeros(n, np.uint8)
            if width > k:
                if s == 0:
                    want[:width - k] = 1
                else:
                    want[s + k:] = 1
            assert (_line(m, axis) == want).all()
    elif kind == "wmod":
        assert W % 32 == p[0]
    elif kind == "zeros":
        (zs,) = p
        assert sorted(map(tuple, np.argwhere(m0 == 0).tolist())) == [tuple(z) for z in zs]
    elif kind == "bits":
        zs = [e for e in case.edges if e[0] == "zeros"][0][1]
        assert sorted({x & 31 for _, x in zs}) == p[0]
    elif kind == "corner":
        zs = [e for e in case.edges if e[0] == "zeros"][0][1]
        h2, w2 = 2 * case.flow.shape[0] - 1, 2 * case.flow.shape[1] - 1
        assert any(y in (0, h2) and x in (0, w2) for y, x in zs)
    elif kind == "words":
        nw, mod = p
        assert (W + 31) // 32 == nw and W % 32 == mod
    elif kind == "short":
        assert H == p[0] < 21
    elif kind == "beyond":
        hb, wb = p
        h, w = case.flow.shape[:2]
        assert (H - 2 * h, W - 2 * w) == (hb, wb)
        assert m0[2 * h:].all() and m0[:, 2 * w:].all()
    elif kind == "mixed":
        assert 0 < m0.mean() < 1
    elif kind == "gap":
        (c,) = p
        assert (_line(m0[:2 * case.flow.shape[0]], 1) == (np.arange(W) != c)).all()
    elif kind == "tie":
        c, which = p
        f2 = O.pyr_up(case.flow)
        t2 = D.sum32(f2[c][0], f2[c][1])
        thr = np.float32(case.thr)
        if which == "at":
            assert t2 == thr and m0[c] == 0
        else:
            assert t2 == D.down(thr) and m0[c] == 1
    elif kind == "fma":
        c, which = p
        f2 = O.pyr_up(case.flow)
        fx, fy = f2[c][0], f2[c][1]
        t2 = D.sum32(fx, fy)
        fused = D.fma32(fx, fx, np.float32(fy * fy)) if which.startswith("xx") else D.fma32(fy, fy, np.float32(fx * fx))
        assert (fused < t2) if which.endswith("below") else (fused > t2)
    elif kind == "floor":
        cs, thr = p
        f2 = O.pyr_up(case.flow)
        t2 = [D.sum32(f2[c][0], f2[c][1]) for c in cs]
        assert t2[:3] == [D.down(40), np.float32(40), D.up(40)] and t2[3] < 40
        eff = max(np.float32(thr), np.float32(40))
        assert [int(m0[c]) for c in cs] == [int(t < eff) for t in t2]
        if thr < 40:       # without the floor some pixel would flip
            assert any((t < np.float32(thr)) != (t < eff) for t in t2)
    elif kind == "nan":
        f2 = O.pyr_up(case.flow)
        for y, x, ch in p[0]:
            assert np.isnan(f2[y, x, ch]) and m0[y, x] == 0
        assert m0.mean() > 0.9
    else:
        raise AssertionError(kind)


@pytest.mark.parametrize("case", MASKS, ids=[c.name for c in MASKS])
def test_mask_case_reaches_its_edge(case):
    assert case.edges
    st = D.stages(case.flow, case.thr, case.shape)
    assert (st[3] == O.mask_from_flow(case.flow, case.thr, case.shape)).all()
    for kind, *p in case.edges:
        _check_mask_edge(case, st, kind, p)


def test_every_family_is_present():
    edges = [(c.name.split("/")[0], e) for c in MASKS for e in c.edges]
    kinds = {e[0] for _, e in edges}
    assert kinds >= {"band", "survive", "phase", "word", "side", "wmod", "zeros", "bits", "corner", "words", "short", "beyond",
                     "mixed", "gap", "tie", "fma", "floor", "nan"}
    assert {e[1] for _, e in edges if e[0] == "phase"} == set(range(32))
    assert {e[1] for _, e in edges if e[0] == "word"} == {0, 1, 3}
    assert {e[1] for _, e in edges if e[0] == "side"} == {"left", "right", "top", "bottom"}
    assert {e[1] for _, e in edges if e[0] == "wmod"} == {0, 1, 23, 31}
    assert {b for _, e in edges if e[0] == "bits" for b in e[1]} >= {0, 31}
    assert {e[1] for _, e in edges if e[0] == "words"} >= {1, 2}
    assert {e[2] for _, e in edges if e[0] == "words"} >= {0, 1, 31}
    assert min(e[1] for _, e in edges if e[0] == "short") < 11 and max(e[1] for _, e in edges if e[0] == "short") >= 11
    assert {(e[1], e[2]) for _, e in edges if e[0] == "beyond"} >= {(0, 1), (1, 0), (1, 1)}
    assert {e[2] for _, e in edges if e[0] == "tie"} == {"at", "ulp"}
    assert {e[2] for _, e in edges if e[0] == "fma"} == {"xx_below", "xx_above", "yy_below", "yy_above"}
    floors = {e[2] for _, e in edges if e[0] == "floor"}
    assert {float(D.down(40)), 40.0, float(D.up(40))} <= floors and min(floors) < 0
    # the 40 / 41 / 42 px bands: nothing, one column, two columns left after two erosions
    surv = {c.name.split("/")[1]: len([e for e in c.edges if e[0] == "survive"][0][2]) for c in MASKS
            if c.name.startswith("phase/")}
    assert surv == {"w40": 0, "w41": 1, "w42": 2}


@pytest.mark.parametrize("family", sorted({c.name.split("/")[0] for c in MASKS}))
def test_mask_oracle_equals_cv2_live(family):
    cv2 = pytest.importorskip("cv2")
    k = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (21, 21), (10, 10))
    n = 0
    for case in MASKS:
        if case.name.split("/")[0] != family:
            continue
        h, w = case.flow.shape[:2]
        up = cv2.pyrUp(case.flow, dstsize=(2 * w, 2 * h))
        f2 = O.pyr_up(case.flow)
        assert (np.isnan(up) == np.isnan(f2)).all() and (up[~np.isnan(up)] == f2[~np.isnan(f2)]).all(), case.name
        m0 = np.ones(case.shape, np.uint8)
        with np.errstate(invalid="ignore"):
            t2 = up[..., 0] * up[..., 0] + up[..., 1] * up[..., 1]
            m0[:2 * h, :2 * w] = (t2 < max(np.float32(case.thr), np.float32(40.0))).astype(np.uint8)
        ref = cv2.dilate(cv2.erode(cv2.erode(m0, k), k), k)
        assert (O.mask_from_flow(case.flow, case.thr, case.shape) == ref).all(), case.name
        n += 1
    assert n > 0


# ---- keypoint lookups ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", LOOKUPS, ids=[c.name for c in LOOKUPS])
def test_lookup_case_reaches_its_edge(case):
    m = case.mask
    assert m.sum() > 0.65 * m.size                  # the filter is on
    lk = case.lookup_kps()
    keep = m[lk["y"].astype(int), lk["x"].astype(int)] == 1
    kept, _ = case.expected()
    assert len(kept) == keep.sum() and kept.tobytes() == case.kps[keep].tobytes()
    x, y = case.kps["x"], case.kps["y"]
    for kind, *p in case.edges:
        if kind == "phase":
            (pp,) = p
            row = 2 + 3 * pp
            sel = lk["y"].astype(int) == row
            xs = lk["x"][sel].astype(int)
            assert {32 + pp - 1, 32 + pp, 32 + pp + 2, 32 + pp + 3} <= set(xs.tolist())
            assert keep[sel].any() and not keep[sel].all()
        elif kind == "trunc":
            rnd = m[np.clip(np.rint(y), 0, m.shape[0] - 1).astype(int), np.clip(np.rint(x), 0, m.shape[1] - 1).astype(int)] == 1
            assert (rnd != keep).any()               # rounding instead of truncating would change the result
            frac = x - np.floor(x)
            assert (frac > 0.99).any() and (frac == 0.5).any() and (frac == 0).any()
        elif kind == "last":
            assert (lk["x"] == m.shape[1] - 1).any() and (lk["y"] == m.shape[0] - 1).any()
            assert (x > m.shape[1] - 1).any() and (y > m.shape[0] - 1).any()
        elif kind == "outside":
            assert case.clamped
            out = (x < 0) | (y < 0) | (x >= m.shape[1]) | (y >= m.shape[0])
            assert out.any() and keep[out].any() and not keep[out].all()
        elif kind == "count":
            n, pat, nkeep = p
            assert len(case.kps) == n and keep.sum() == nkeep
            i = np.nonzero(keep)[0]
            if pat == "all-but-first":
                assert i.tolist() == list(range(1, n))
            elif pat == "alternate":
                assert i.tolist() == list(range(1, n, 2))
            else:
                assert all(k % 512 == 511 or k == n - 1 for k in i)
        else:
            raise AssertionError(kind)


def test_every_lookup_family_is_present():
    edges = [e for c in LOOKUPS for e in c.edges]
    assert {e[1] for e in edges if e[0] == "phase"} == set(range(32))
    assert {e[0] for e in edges} == {"phase", "trunc", "last", "outside", "count"}
    assert {e[1] for e in edges if e[0] == "count"} == {511, 512, 513, 1024, 1025}
    assert {e[2] for e in edges if e[0] == "count"} == {"all-but-first", "alternate", "last-of-chunk"}


# ---- Farneback ---------------------------------------------------------------------------------------------------------

def _crossings(flow):
    """Image sides across which the displaced fetch of FarnebackUpdateMatrices leaves the image for some pixel."""
    h, w = flow.shape[:2]
    yy, xx = np.mgrid[0:h, 0:w]
    x1 = np.floor(xx.astype(np.float32) + flow[..., 0])
    y1 = np.floor(yy.astype(np.float32) + flow[..., 1])
    return {s for s, hit in (("left", x1 < 0), ("right", x1 >= w - 1), ("top", y1 < 0), ("bottom", y1 >= h - 1)) if hit.any()}


@pytest.mark.parametrize("case", [c for c in FLOWS if not c.name.startswith("fb/size2048x2048")],
                         ids=[c.name for c in FLOWS if not c.name.startswith("fb/size2048x2048")])
def test_flow_case_reaches_its_edge(case):
    h, w = case.half
    assert case.gray.shape == (2, 2 * h, 2 * w)
    for kind, *p in case.edges:
        if kind == "size":
            assert (h, w) == tuple(p) and min(h, w) == 16 and max(h, w) == 2048
        elif kind == "refused":
            assert max(h, w) == 2049
        elif kind == "tie":
            top = FB.level_count(h, w)
            ties = []
            for k in range(2, top + 1):
                for side in (h, w):
                    v = side * 0.5 ** k
                    if v - np.floor(v) == 0.5:
                        ties.append((k, side, int(np.rint(v)), int(np.floor(v + 0.5))))
            assert ties and all(r % 2 == 0 for _, _, r, _ in ties)
            assert [FB.level_size(h, w, k) for k in range(top + 1)] == [(int(np.rint(h * 0.5 ** k)), int(np.rint(w * 0.5 ** k)))
                                                                          for k in range(top + 1)]
        elif kind == "shift":
            dy, dx = p
            prev, cur = case.pair()
            tr = {}
            FB.farneback(prev, cur, trace=tr)
            want = {s for s, on in (("right", dx > 0), ("left", dx < 0), ("bottom", dy > 0), ("top", dy < 0)) if on}
            assert want <= _crossings(tr["flow_in"][-1]), tr["flow_in"][-1].mean((0, 1))
        elif kind == "checker":
            g = case.gray
            assert set(np.unique(g[0]).tolist()) == {0, 255} and (g[1] == 255 - g[0]).all()
        else:
            raise AssertionError(kind)


def test_every_flow_family_is_present():
    edges = [e for c in FLOWS for e in c.edges]
    assert {tuple(e[1:]) for e in edges if e[0] == "size"} == {(16, 2048), (2048, 16), (2048, 2048)}
    ties = [tuple(e[1:]) for e in edges if e[0] == "tie"]
    lv = lambda n, k: n * 0.5 ** k
    # level-2 and level-3 ties, each rounding down (round half up would differ) and up
    for k in (2, 3):
        sides = {n for t in ties for n in t if lv(n, k) % 1 == 0.5 and FB.level_count(*t) >= k}
        assert any(int(np.rint(lv(n, k))) < lv(n, k) for n in sides) and any(int(np.rint(lv(n, k))) > lv(n, k) for n in sides)
    sides = set()
    for e in edges:
        if e[0] == "shift":
            dy, dx = e[1:]
            sides |= {s for s, on in (("right", dx > 0), ("left", dx < 0), ("bottom", dy > 0), ("top", dy < 0)) if on}
            assert 8 <= max(abs(dy), abs(dx)) <= 40
    assert sides == {"left", "right", "top", "bottom"}
    assert any(e[0] == "checker" for e in edges) and any(e[0] == "refused" for e in edges)


@pytest.fixture
def cv2_baseline():
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    cv2.setUseOptimized(False)
    yield cv2
    cv2.setUseOptimized(was)


@pytest.mark.parametrize("case", [c for c in FLOWS if not c.refused], ids=[c.name for c in FLOWS if not c.refused])
def test_flow_restatement_equals_cv2(cv2_baseline, case):
    h, w = case.half
    prev, cur = case.pair()
    for g, half in zip(case.gray, (prev, cur)):
        assert (cv2_baseline.pyrDown(g, dstsize=(w, h)) == half).all()
    want = cv2_baseline.calcOpticalFlowFarneback(prev, cur, None, 0.5, 3, 15, 3, 5, 1.2, 0)
    got = FB.farneback(prev, cur)
    assert (got.view(np.uint32) == want.view(np.uint32)).all()
