"""The crafted pairs of tests/flow_edge_cases.py on the CPU: every case reaches each edge it declares (evidence from the
restatement's trace, each level's UpdateMatrices / box filter / solve replayed from its polynomial expansions and
incoming flow), the restatement (oracle/farneback_py.py) equals cv2 4.13 at baseline dispatch bit for bit on every case,
and tests/golden/flow_edges.npz (tools/make_farneback_edges_golden.py) holds the same inputs and flows."""
import functools
import os

import numpy as np
import pytest

from oracle import farneback_py as FB
from tests import flow_edge_cases as EC
from tests import flow_scenes as S
from tests.refpins import digest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flow_edges.npz")
CASES = {c.name: c for c in EC.cases()}
NAMES = list(CASES)
AXIS = {"rows": 0, "cols": 1}
REPLAY = {"sample", "det_small", "det_zero", "m_max", "beyond_reach"}


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    assert a.shape == b.shape
    assert (_bits(a) == _bits(b)).all(), "max |diff| %g" % np.abs(a.astype(np.float64) - b).max()


def resize_path(H, W, h, w):
    if (h, w) == (H, W):
        return "copy"
    return "area" if 1.0 / (w / W) == 2.0 and 1.0 / (h / H) == 2.0 else "linear"


def _samples(flow, where):
    """The UpdateMatrices sample positions x1 = floor(x + dx), y1 = floor(y + dy) of this flow, by edge."""
    h, w = flow.shape[:2]
    yy, xx = np.mgrid[0:h, 0:w]
    x1 = np.floor(xx.astype(np.float32) + flow[..., 0]).astype(np.int64)
    y1 = np.floor(yy.astype(np.float32) + flow[..., 1]).astype(np.int64)
    for key, hit in (("x=-1", x1 == -1), ("y=-1", y1 == -1), ("x=w-2", x1 == w - 2), ("y=h-2", y1 == h - 2),
                     ("x=w-1", x1 == w - 1), ("y=h-1", y1 == h - 1),
                     ("far", (x1 < -1) | (x1 >= w) | (y1 < -1) | (y1 >= h))):
        where[key] = where.get(key, 0) + int(hit.sum())


def evidence(prev, cur, replay=True):
    """-> dict: level sizes, resize paths, the flow upsample's clamps into each level below the top and the flow; with
    `replay`, also the sample positions of every UpdateMatrices, max |M| and the solve counts (the flow is then the
    replay's, checked equal to farneback's)."""
    H, W = prev.shape
    top = FB.level_count(H, W)
    sizes = [FB.level_size(H, W, k) for k in range(top + 1)]
    clamps = []
    for k in range(top):
        (h, w), (ph, pw) = sizes[k], sizes[k + 1]
        sx, _ = FB._linear_tab(pw, w)
        clamps.append((bool((sx < 0).any()), bool((sx + 1 >= pw).any())))
    ev = {"sizes": sizes, "paths": [resize_path(H, W, h, w) for h, w in sizes], "clamps": clamps}
    if not replay:
        ev["flow"] = FB.farneback(prev, cur)
        return ev
    tr, where, counts, m_max = {}, {}, {}, 0.0
    want = FB.farneback(prev, cur, trace=tr)
    for li in range(top + 1):
        R0, R1 = tr["R"][2 * li], tr["R"][2 * li + 1]
        flow = tr["flow_in"][li]
        for _ in range(FB.ITERATIONS):
            _samples(flow, where)
            M = FB.update_matrices(R0, R1, flow)
            m_max = max(m_max, float(np.abs(M).max()))
            flow = FB.horizontal_solve(FB.vertical_sums(M), counts=counts)
    _same(flow, want)
    ev.update(where=where, counts=counts, m_max=m_max, flow=flow)
    return ev


@functools.lru_cache(maxsize=None)
def _evidence(name):
    c = CASES[name]
    return evidence(c.prev, c.cur, replay=any(e[0] in REPLAY for e in c.edges))


@functools.lru_cache(maxsize=None)
def _scenes_m_max():
    out = {}
    for scene in S.SCENES:
        g = S.frames(scene, 480, 640, 2)
        out[scene] = evidence(FB.pyr_down(g[0], 240, 320), FB.pyr_down(g[1], 240, 320))["m_max"]
    return out


def check_edge(c, ev, e):
    """Assert that case c (evidence ev) reaches edge e."""
    H, W = c.prev.shape
    kind = e[0]
    if kind == "levels":
        assert tuple(ev["sizes"]) == e[1]
    elif kind == "resize":
        assert tuple(ev["paths"]) == e[1]
    elif kind == "area_tail":
        assert len(ev["paths"]) > 1 and ev["paths"][1] == "area" and ev["sizes"][1][1] % 8 == e[1]
    elif kind == "halves":
        (h1, w1), ax = ev["sizes"][1], AXIS[e[1]]
        halved = (H == 2 * h1, W == 2 * w1)
        assert halved[ax] and not halved[1 - ax]
    elif kind == "round":
        _, k, axis, way = e
        v = (H, W)[AXIS[axis]] * 0.5 ** k
        assert k < len(ev["sizes"]) and v - np.floor(v) == 0.5
        assert ev["sizes"][k][AXIS[axis]] == (np.ceil(v) if way == "up" else np.floor(v))
    elif kind in ("cut_below", "cut_at"):
        _, axis, k = e
        side, other = (H, W)[AXIS[axis]] * 0.5 ** k, (H, W)[1 - AXIS[axis]] * 0.5 ** k
        assert other >= FB.MIN_SIZE
        if kind == "cut_below":
            assert len(ev["sizes"]) == k and FB.MIN_SIZE - 0.5 ** k <= side < FB.MIN_SIZE
        else:
            assert len(ev["sizes"]) > k and side == FB.MIN_SIZE
    elif kind == "side":
        assert (H, W)[AXIS[e[1]]] == e[2]
    elif kind == "upsample_clamps":
        assert ev["clamps"] and all(left and right for left, right in ev["clamps"])
    elif kind == "sample":
        assert ev["where"][e[1]] > 0
    elif kind in ("det_small", "det_zero"):
        assert ev["counts"][kind] > 0
    elif kind == "saturated":
        assert np.isin(c.prev, (0, 255)).all() and np.isin(c.cur, (0, 255)).all()
    elif kind == "same":
        assert (c.prev == c.cur).all()
    elif kind == "m_max":
        assert ev["m_max"] > max(_scenes_m_max().values())
    elif kind == "one_dim":
        assert (c.prev == c.prev[:, :1]).all() and (c.cur == c.cur[:, :1]).all() and (c.prev != c.cur).any()
    elif kind == "impulse":
        assert np.count_nonzero(c.prev) == 1 and np.count_nonzero(c.cur) == 1 and (c.prev != c.cur).any()
    elif kind == "inverted":
        assert (c.cur == 255 - c.prev).all()
    elif kind == "brightness":
        p = c.prev.astype(np.int64)
        ok = p + e[1] <= 255
        assert ok.mean() > 0.9 and (c.cur[ok] == p[ok] + e[1]).all()
    elif kind == "beyond_reach":
        _, dx, dy = e
        h, w = ev["flow"].shape[:2]
        mid = ev["flow"][h // 4:3 * h // 4, w // 4:3 * w // 4].reshape(-1, 2)
        got = np.median(mid, axis=0)
        assert np.hypot(got[0], got[1]) < 0.5 * np.hypot(dx, dy)
        p, q = c.prev.astype(np.int64), c.cur.astype(np.int64)
        ys, xs = slice(max(dy, 0) + 4, h + min(dy, 0) - 4), slice(max(dx, 0) + 4, w + min(dx, 0) - 4)
        ys0, xs0 = slice(ys.start - dy, ys.stop - dy), slice(xs.start - dx, xs.stop - dx)
        assert np.abs(q[ys, xs] - p[ys0, xs0]).mean() < 3      # cur(x) == prev(x - d) up to the per-frame noise
    else:
        raise AssertionError("unknown edge %r" % (e,))


@pytest.mark.parametrize("name", NAMES)
def test_case_reaches_its_edges(name):
    c = CASES[name]
    assert c.edges
    ev = _evidence(name)
    for e in c.edges:
        check_edge(c, ev, e)
    assert np.isfinite(ev["flow"]).all()


def test_cases_cover_every_edge():
    """Every resize path, tail residue, rounding, cut, range end and sample position is some case's declared edge."""
    edges = {e for c in CASES.values() for e in c.edges}
    kinds = {e[0] for e in edges}
    assert {e[1] for e in edges if e[0] == "area_tail"} == set(range(8))
    assert {(k, axis, way) for kind, *rest in edges if kind == "round" for k, axis, way in [rest]} == \
        {(k, axis, way) for k in (1, 2, 3) for axis in AXIS for way in ("up", "down")}
    for kind in ("cut_below", "cut_at"):
        assert {(axis, k) for kd, *rest in edges if kd == kind for axis, k in [rest]} >= \
            {(axis, k) for axis in AXIS for k in (1, 2, 3)}
    assert {(a, n) for kd, *rest in edges if kd == "side" for a, n in [rest]} == \
        {(a, n) for a in AXIS for n in (16, 2048)}
    assert {e[1] for e in edges if e[0] == "sample"} == {"x=-1", "y=-1", "x=w-2", "y=h-2", "x=w-1", "y=h-1", "far"}
    assert {"det_small", "det_zero", "saturated", "same", "m_max", "one_dim", "impulse", "inverted", "brightness",
            "beyond_reach", "upsample_clamps"} <= kinds
    assert {e[1] for e in edges if e[0] == "halves"} == set(AXIS)
    paths = {p for kd, *rest in edges if kd == "resize" for p in rest[0]}
    assert paths == {"copy", "area", "linear"}


@pytest.fixture(scope="module")
def cv2_baseline():
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    cv2.setUseOptimized(False)
    yield cv2
    cv2.setUseOptimized(was)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_equals_cv2(cv2_baseline, name):
    c = CASES[name]
    want = cv2_baseline.calcOpticalFlowFarneback(c.prev, c.cur, None, 0.5, 3, 15, 3, 5, 1.2, 0)
    _same(_evidence(name)["flow"], want)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_golden_lists_every_case(golden):
    assert [str(n) for n in golden["names"]] == NAMES


@pytest.mark.parametrize("name", NAMES)
def test_golden_equals_restatement(golden, name):
    """The stored input digest first, so that a change in the case generator reads as such, not as a flow mismatch."""
    c = CASES[name]
    assert str(golden[name + "/inputs_sha256"]) == digest((c.prev, c.cur)), "tests/flow_edge_cases.py drifted"
    flow = _evidence(name)["flow"]
    assert str(golden[name + "/flow_sha256"]) == digest(flow)
    if name + "/flow" in golden:
        assert (golden[name + "/prev"] == c.prev).all() and (golden[name + "/cur"] == c.cur).all()
        _same(flow, golden[name + "/flow"])
