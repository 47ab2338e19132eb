"""The crafted matcher cases of tests/match_cases.py on the CPU: every case really contains the edge it claims
(recomputed here in numpy from the case's inputs), and the oracle (oracle/match_ref.cpp) equals the reference's own
ORBmatcher.cc on it.  The reference's results are pinned in tests/golden/refsrc_pins.json (tests/refpins.py);
REFSRC_RECORD=1 runs the reference live where oracle/_ref is built and records them."""
import math

import numpy as np
import pytest

from tests import match_cases as M
from tests.refpins import RECORD, Pins

CASES = M.all_cases()
PINNED = ("last", "points", "bow", "bow_kf", "init")
F32 = np.float32


@pytest.fixture(scope="module")
def src(oracle):
    if RECORD:
        oracle.reflib()
    return oracle


@pytest.fixture(scope="module")
def pins():
    p = Pins()
    yield p
    p.save()


def _c_round(v):
    return int(math.floor(v + 0.5)) if v >= 0 else -int(math.floor(-v + 0.5))


def _window(case, i):
    """(distance, keypoint) of every candidate of query i of a LAST case: inside its window and level range, pre-existing
    points with observations excluded (numpy, from the case's inputs)."""
    S, th = case.kw["scene"], case.kw["th"]
    q = S.q[i]
    if not q["valid"] or q["z"] < 0:
        return []
    r = F32(F32(th) * M.SF[q["oct"]])
    out = []
    for j, (x, y, o, d, _, _, obs) in enumerate(S.k):
        if obs >= 1 or not (q["oct"] - 1 <= o <= q["oct"] + 1):
            continue
        if abs(F32(F32(x) - F32(q["u"]))) < r and abs(F32(F32(y) - F32(q["v"]))) < r:
            out.append((M.hamming(q["desc"], d), j))
    return out


def _picks(case, honour_claims):
    """Per query, the minimum-distance candidate (within TH_HIGH) among the keypoints not claimed by an earlier query
    (honour_claims) or among all of them; the lower index on equal distances (the check only asks whether two queries of
    one step land on the same keypoint)."""
    S = case.kw["scene"]
    taken, out = set(), []
    for i in range(len(S.q)):
        c = [(d, j) for d, j in _window(case, i) if not (honour_claims and j in taken)]
        p = min(c)[1] if c and min(c)[0] <= M.TH_HIGH else None
        if p is not None and S.q[i]["obs"] > 0:
            taken.add(p)
        out.append(p)
    return out


def _three_maxima(counts):
    """ComputeThreeMaxima over bin counts (strict '>': on equal counts the earlier bin wins)."""
    h = [0] * 30
    for b, c in counts:
        h[b] = c
    m, ind = [0, 0, 0], [-1, -1, -1]
    for i, c in enumerate(h):
        if c > m[0]:
            m, ind = [c, m[0], m[1]], [i, ind[0], ind[1]]
        elif c > m[1]:
            m, ind = [m[0], c, m[1]], [ind[0], i, ind[1]]
        elif c > m[2]:
            m[2], ind[2] = c, i
    return m, ind


def _check_edge(case, kind, p):
    if kind == "dist":
        qd, cd, d = p
        assert M.hamming(qd, cd) == d
    elif kind == "tie":
        d = {M.hamming(qd, cd) for qd, cd in p}
        assert len(p) >= 2 and len(d) == 1, d
    elif kind == "order":
        assert p == (True, True), "the later keypoint index must sit in an earlier grid column"
    elif kind == "ratio":
        best, second, nn = p
        assert np.float32(best) == np.float32(np.float32(nn) * np.float32(second))
    elif kind == "cell":
        x, lo, hi, cells, want = p
        got = M.grid_coord(x, lo, hi, cells)
        assert got == want and got - math.floor(got) == 0.5
        assert _c_round(got) != int(np.rint(got)) or want == 63.5
    elif kind == "eq":
        assert p[0] == p[1]
    elif kind == "motion":
        tz = p
        fwd, bwd = -tz > M.BF / M.FX, tz > M.BF / M.FX
        assert (fwd, bwd) == {0.0: (False, False), -1.0: (True, False), 1.0: (False, True)}[tz]
    elif kind == "clip":
        for u, r, lo, hi in p:
            inv = np.float32(M.GRID_COLS / (hi - lo))
            x0 = math.floor(np.float32(np.float32(u - lo) - np.float32(r)) * inv)
            x1 = math.ceil(np.float32(np.float32(u - lo) + np.float32(r)) * inv)
            assert x0 < 0 or x1 > M.GRID_COLS - 1
    elif kind == "cols":
        u, r, lo, hi, wide = p
        n = M.window_columns(u, r, lo, hi)
        assert (n > 32) == wide, n
    elif kind == "half":
        assert p == 0.5
    elif kind == "bins":
        counts, claim = p
        m, ind = _three_maxima(counts)
        tenth = F32(F32(0.1) * F32(m[0]))
        if claim == "equal":   # four bins of one count: the first three in bin order are the maxima, the fourth loses
            same = sorted(b for b, c in counts if c == m[0])
            assert len(same) >= 4 and ind == same[:3] and m[1] == m[2] == m[0]
        elif claim == "kept":
            assert F32(m[1]) == tenth and F32(m[2]) == tenth
        else:
            assert claim == "dropped" and F32(m[1]) >= tenth and F32(m[2]) < tenth < F32(m[2] + 1)
    elif kind == "conflict":
        nl = len(case.kw["scene"].q)

        def shared(best):
            return [(i, j) for s in range(0, nl, 32) for i in range(s, min(s + 32, nl))
                    for j in range(i + 1, min(s + 32, nl)) if best[i] is not None and best[i] == best[j]]
        assert shared(_picks(case, True)), "no step with two queries whose first unclaimed minimum is one keypoint"
        if nl > 31:   # lanes 0 and 31 of the first step go for the same keypoint
            assert (0, 31) in shared(_picks(case, False))
    elif kind == "crowd":
        lcap, r = p
        S = case.kw["scene"]
        counts = [sum(1 for k in S.k if abs(F32(k[0] - q["u"])) < r and abs(F32(k[1] - q["v"])) < r) for q in S.q[:32]]
        assert max(counts) > lcap
    elif kind == "epipolar":   # every keyframe-2 keypoint is on its query's epipolar line or clearly off it
        k1, k2 = p
        F = M.tri_fundamental().astype(np.float64)
        on = off = 0
        for a in range(len(k1.node_ids)):
            i1 = int(k1.idx[k1.node_off[a]])
            b = int(np.nonzero(k2.node_ids == k1.node_ids[a])[0][0])
            l = np.array([k1.x[i1], k1.y[i1], 1.0]) @ F
            for i2 in k2.idx[k2.node_off[b]:k2.node_off[b + 1]]:
                d2 = (l[0] * k2.x[i2] + l[1] * k2.y[i2] + l[2]) ** 2 / (l[0] ** 2 + l[1] ** 2)
                assert d2 < 0.01 or d2 > 3.84 * 10, d2
                on, off = on + (d2 < 0.01), off + (d2 > 0.01)
        assert on > 0 and off > 0
    else:
        raise AssertionError(kind)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_case_contains_its_edge(case):
    assert case.edges
    for kind, p in case.edges:
        _check_edge(case, kind, p)


def test_every_family_is_present():
    kinds = {c.kind for c in CASES}
    assert kinds == {"last", "points", "projected", "best", "bow", "bow_kf", "init", "tri"}
    last = [c for c in CASES if c.kind == "last"]
    assert {len(c.kw["scene"].q) for c in last if c.name.startswith("last/claims")} >= {31, 32, 33, 64, 65, 200}
    cols = [M.window_columns(*e[1][:4]) for c in last for e in c.edges if e[0] == "cols"]
    assert min(cols) <= 32 < max(cols)


def test_oracle_equals_reference_sources_on_crafted_cases(src, pins):
    """oracle == the reference's ORBmatcher.cc on every crafted case of the flat searches, LAST also with the current
    frame padded past the fused kernel's limit."""
    n = 0
    for case in CASES:
        if case.kind not in PINNED:
            continue
        pads = (0, 4200) if case.kind == "last" else (0,)
        for pad in pads:
            ours = M.run(case, "oracle", src, pad)
            pins.check("match_edges/%s/%d" % (case.name, pad), ours, lambda: M.run(case, "refsrc", src, pad))
            n += int(ours[0])
    assert n > 300


def test_best_and_triangulation_equal_reference_sources(src, pins):
    """The per-query best search (KeyFrame::GetFeaturesInArea + DescriptorDistance) and SearchForTriangulation have no
    flat entry in the reference: they run on real KeyFrames through SrcMembers (kf_best, triangulation)."""
    members = src.SrcMembers("refsrc") if RECORD else None
    for case in CASES:
        if case.kind == "best":
            S, kw = case.kw["scene"], case.kw
            F, q = S.frame(), S.queries(kw["radius"], kw["levels"])
            ours = src.search_best(F, q, 0)
            assert (ours[0] >= 0).all()
            pins.check("match_edges/%s" % case.name, ours, lambda: members.kf_best(F, q))
        elif case.kind == "tri":
            kw = case.kw
            reference = lambda: members.triangulation(kw["k1"], kw["k2"], M.TRI_T1, M.TRI_T2, kw["cam"],
                                                      M.tri_fundamental(), False, 0.6, True)
            # the reference's own epipole feeds the oracle (keyframe 1 is stereo, so it gates nothing here)
            ep = pins.array("match_edges/%s/epipole" % case.name, lambda: reference()[2], np.float32)
            ours = M.run(case, "oracle", src, epipole=ep)
            assert ours[0] >= 4
            pins.check("match_edges/%s" % case.name, ours, lambda: reference()[:2])


def test_projected_oracle_equals_restatement(oracle):
    """SearchProjected has no flat entry in the reference: oracle/match_ref.cpp against the independent Python
    restatement (oracle/match_py.py) on the crafted projected cases."""
    from oracle import match_py
    for case in CASES:
        if case.kind != "projected":
            continue
        S, kw = case.kw["scene"], case.kw
        F, q = S.frame(with_obs=True), S.queries(kw["radius"], kw["levels"], uright=True)
        a = oracle.search_projected(F, q, kw["max_dist"], kw["rule"], True)
        b = match_py.search_projected(F, q, kw["max_dist"], kw["rule"], True)
        assert a[0] == b[0] and (a[1] == b[1]).all(), case.name
        assert a[0] > 0
