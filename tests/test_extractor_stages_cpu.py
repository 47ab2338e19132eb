"""CPU checks of tests/extractor_cases.py: every case reaches the edge it names, recomputed in numpy on the oracle's
results, and the oracle's FAST candidates, blur and resize equal cv2 on every crafted level."""
import numpy as np
import pytest

from oracle import ref
from tests import extractor_cases as E

CASES = E.all_cases()
FAMILIES = sorted({c.name.split("/")[0] for c in CASES})


def _run(case):
    R = ref.RefExtractor(*case.params)
    R(case.img)
    return R


def _cand_sets(R, nlevels):
    return [set(map(tuple, R.candidates(l).tolist())) for l in range(nlevels)]


def test_every_family_present():
    assert FAMILIES == ["blur", "cells", "fallback", "fast", "nms", "resize"]


def test_oracle_candidates_match_counts_and_cells():
    """R.candidates(l) is the level's vToDistributeKeys: as many as candidates_per_level, each inside its cell's detection
    range, cells in order and row-major inside a cell."""
    for case in CASES:
        R = _run(case)
        sizes = E.level_sizes(*case.img.shape, case.params[1], case.params[2])
        for l, (lh, lw) in enumerate(sizes):
            c = R.candidates(l)
            assert len(c) == R.candidates_per_level[l], case.name
            cs = E.cells(lh, lw)
            rank = [cs.index(E.cell_of(cs, x, y)) for x, y, _ in c]
            key = [(r, y, x) for r, (x, y, _) in zip(rank, c)]
            assert key == sorted(key), case.name
            assert (c[:, 2] >= 1).all() and (c[:, 2] <= 254).all(), case.name


@pytest.mark.parametrize("name", [c.name for c in CASES if c.want or c.absent or c.cell_counts])
def test_fast_case_reaches_its_edge(name):
    case = next(c for c in CASES if c.name == name)
    R = _run(case)
    s = _cand_sets(R, case.params[2])
    img0 = case.img
    for l, x, y, score in case.want:
        assert (x, y, score) in s[l], (name, x, y, score)
        if l == 0:
            assert E.fast_m(img0, x, y) == score + 1
    for l, x, y in case.absent:
        assert not any(c[0] == x and c[1] == y for c in s[l]), (name, x, y)
    for (l, x0, y0), n in case.cell_counts.items():
        cell = next(c for c in E.cells(*R.level(l).shape) if c[:2] == (x0, y0))
        inside = [c for c in s[l] if E.cell_of([cell], c[0], c[1])]
        assert len(inside) == n, (name, cell, inside)


def test_threshold_arcs_sit_exactly_at_the_threshold():
    """Every arc feature's m is t or t + 1 exactly, with the compass pixel of a half-covered opposite pair at exactly t + 1
    (so a compass test built from t + 1 misses it), for every start 0..15, both polarities, at iniTh and minTh; the
    features of m == t behind a compass pair at t + 1 reach the exact test (where m >= t would take them)."""
    for case in CASES:
        if not case.name.startswith("fast/arcs"):
            continue
        _, _, _, ini, mn = case.params
        seen = set()
        for (_, x, y, score) in case.want:
            m = score + 1
            c = int(case.img[y, x])
            d = [int(case.img[y + dy, x + dx]) - c for dx, dy in E.RING]
            start = next(s for s in range(16) if all(abs(d[(s + i) % 16]) == m for i in range(9)))
            sign = 1 if d[start] > 0 else -1
            halves = [p for p in ((0, 8), (4, 12)) if sum((k - start) % 16 < 9 for k in p) == 1]
            assert halves and all(abs(d[k]) == m for p in halves for k in p if (k - start) % 16 < 9)
            seen.add((start, sign, m))
        assert seen == {(s, g, m) for s in range(16) for g in (1, -1) for m in (ini + 1, mn + 1)}, case.name
        behind = 0
        for (_, x, y) in case.absent:
            m = E.fast_m(case.img, x, y)
            assert m in (ini, mn)
            c = int(case.img[y, x])
            d = [int(case.img[y + dy, x + dx]) - c for dx, dy in E.RING]
            q = max(min(max(d[0], d[8]), max(d[4], d[12])), min(max(-d[0], -d[8]), max(-d[4], -d[12])))
            behind += q > m
        assert behind == 64, case.name   # 16 starts x 2 polarities x 2 thresholds pass the compass test with m == t


def test_fallback_cell_empty_after_nms_at_ini_not_before():
    """Cell 0 of the fallback image: at iniTh 20 the pair is two corners (m = 255) that NMS removes, so the cell is empty
    after NMS with corners before it; at minTh 7 the dot of 15 survives alone."""
    case = next(c for c in CASES if c.name == "fallback/ini20_min7")
    roi = case.img[16:16 + 38, 16:16 + 37]
    assert E.fast_m(case.img, 25, 25) == E.fast_m(case.img, 26, 25) == 255
    assert len(ref.fast(roi, 20)) == 0 and ref.fast(roi, 7).tolist() == [[24, 24, 14]]
    assert E.fast_m(case.img, 40, 40) == 15


def test_cells_cover_every_byte_phase_and_both_pitches():
    phases = set()
    for case in CASES:
        if not case.name.startswith("cells/"):
            continue
        R = _run(case)
        cs = E.cells(*case.img.shape)
        for x, y, _ in R.candidates(0):
            phases.add(E.cell_of(cs, x, y)[0] & 3)
    assert phases == {0, 1, 2, 3}
    from tests.test_boundaries_gpu import geometry
    (_, small), (_, big) = E.pitch_widths()
    assert geometry(480, small, 1000, 1.2, 8)["rw_max"] + 3 == 48 and geometry(480, big, 1000, 1.2, 8)["rw_max"] + 3 == 49


def test_straddling_pairs_survive_in_both_cells():
    """In the edge-dot cases each cell's last-column dot and the next cell's first-column dot are one pixel apart, and both
    are candidates (each cell scores only its own detection range)."""
    case = next(c for c in CASES if c.name == "cells/edges_480x640")
    R = _run(case)
    s = {(x, y) for x, y, _ in R.candidates(0)}
    pairs = [(x, y) for x, y in s if (x + 1, y) in s]
    assert len(pairs) >= 19 * 14 - 14


def test_blur_cases_cover_sizes_and_ties_on_every_path():
    """w % 4 and the last strip tile's interior groups, h % 35, and exact rounding ties written by the strip kernel's
    full-block and tail paths and by the edge kernel, in the first and last three rows and columns too."""
    sizes = [c.img.shape for c in CASES if c.name.startswith("blur/") and c.params[2] == 1]
    assert {w % 4 for _, w in sizes} == {0, 1, 2, 3}
    assert {h % 35 for h, _ in sizes} >= {0, 1, 6, 7, 8, 34}
    last_tile = set()
    for h, w in sizes:
        x0 = (w - 1) // 128 * 128
        last_tile.add(sum(1 for g in range(x0, min(w, x0 + 128), 4) if g >= 4 and g + 8 <= w))
    assert last_tile >= {0, 1, 2}
    paths, border = set(), set()
    for case in CASES:
        if not case.name.startswith("blur/impulses"):
            continue
        h, w = case.img.shape
        for y, x in zip(*np.nonzero(E.blur_sum(case.img) % 65536 == 32768)):
            paths.add(E.blur_path(h, w, y, x))
            if min(y, h - 1 - y) < 3:
                border.add("row")
            if min(x, w - 1 - x) < 3:
                border.add("col")
    assert paths == {("strip", "full"), ("strip", "tail"), ("edge", "full"), ("edge", "tail")}
    assert border == {"row", "col"}


def _cv2_candidates(cv2, img, cs, ini, mn):
    out = []
    for x0, y0, rw, rh in cs:
        roi = np.ascontiguousarray(img[y0:y0 + rh, x0:x0 + rw])
        k = cv2.FastFeatureDetector_create(threshold=ini, nonmaxSuppression=True).detect(roi)
        if not k:
            k = cv2.FastFeatureDetector_create(threshold=mn, nonmaxSuppression=True).detect(roi)
        out += [(x0 + int(p.pt[0]), y0 + int(p.pt[1]), int(p.response)) for p in k]
    return np.array(out, np.int32).reshape(-1, 3)


@pytest.mark.parametrize("family", FAMILIES)
def test_oracle_stages_equal_cv2(family):
    """On every crafted level: the oracle's candidates equal cv2's FAST (nonmax) on each cell's ROI with the fallback,
    its resize equals cv2.resize of the level above, and its blur equals cv2.GaussianBlur and the numpy integer sum."""
    cv2 = pytest.importorskip("cv2")
    for case in CASES:
        if case.name.split("/")[0] != family:
            continue
        R = _run(case)
        _, scale, nl, ini, mn = case.params
        for l in range(nl):
            lv = R.level(l)
            if l == 0:
                assert (lv == case.img).all()
            else:
                prev = R.level(l - 1)
                assert (cv2.resize(prev, (lv.shape[1], lv.shape[0]), interpolation=cv2.INTER_LINEAR) == lv).all(), (case.name, l)
                assert (ref.resize(prev, lv.shape[1], lv.shape[0]) == lv).all()
            assert np.array_equal(R.candidates(l), _cv2_candidates(cv2, lv, E.cells(*lv.shape), ini, mn)), (case.name, l)
            b = ref.blur(lv)
            assert (b == cv2.GaussianBlur(lv, (7, 7), 2, sigmaY=2, borderType=cv2.BORDER_REFLECT_101)).all(), (case.name, l)
            assert (b == E.blur_exact(lv)).all(), (case.name, l)


def test_resize_cases_reach_both_kernels():
    """The resize family's scale factors take the pyramid through k_resize_g (scale <= 2) and k_resize."""
    from tests.test_boundaries_gpu import resize_grouped
    sides = {resize_grouped(E.level_sizes(480, 640, c.params[1], c.params[2])) for c in CASES if c.name.startswith("resize/")}
    assert sides == {True, False}
    assert all(c.params[2] >= 3 for c in CASES if c.name.startswith("resize/"))
