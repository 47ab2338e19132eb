"""The crafted quad-tree cases of tests/quadtree_cases.py on the CPU: every case reaches the edge it is named for (from the
oracle's round trace or the level geometry), and the oracle's DistributeOctTree equals the reference's own on it, pinned in
tests/golden/refsrc_pins.json under quadtree/<case>.  Also the whole extractor on images wide enough that a level has
more than four initial nodes, where a frame returns up to 4*nIni keypoints per level instead of N_l + 3."""
import numpy as np
import pytest

from tests import quadtree_cases as Q
from tests.refpins import Pins

CASES = Q.all_cases()

# (rows, cols, nfeatures, nlevels): the reference returns 4*nIni keypoints on level 0, far above nfeatures
WIDE = [(100, 4000, 10, 1), (120, 2000, 20, 2), (200, 3000, 30, 4)]


def wide_image(rows, cols, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (rows, cols), dtype=np.uint8)


@pytest.fixture(scope="module")
def pins(oracle):
    p = Pins()
    yield p
    p.save()


def test_every_case_reaches_its_edge(oracle):
    missed = []
    for c in CASES:
        g = Q.geometry(c.params, c.rows, c.cols, c.level)
        assert 0 <= c.N <= g.nfeat and 0 < len(c.xys) <= g.slots, c.name
        x, y, s = c.xys[:, 0] - Q.B, c.xys[:, 1] - Q.B, c.xys[:, 2]
        assert (x >= 0).all() and (x < g.W).all() and (y >= 0).all() and (y < g.H).all() and (s >= 0).all() and \
            (s <= 255).all(), c.name
        out, tr = Q.oracle_distribute(c, oracle, trace=True)
        if not c.reached(c, tr, g):
            missed.append((c.name, c.edge, tr.tolist()))
        # what one list can return: its distinct pixels, and max(N + 3, 4*nIni) (orbx_max_keypoints_for's bound)
        assert len(out) <= max(c.N + 3, 4 * g.n_ini), c.name
    assert not missed, missed
    families = {c.name.split("/")[0] for c in CASES}
    assert families == {"ini", "halving", "dup", "term", "rank", "best", "size"}, families


def test_rank_sizes_cover_the_sort_padding(oracle):
    """m around the powers of two the bitonic sort pads to, one pair per thread and several, and the level-0 quota's
    largest m (one below N = 1156)."""
    ms = set()
    for c in CASES:
        if c.name.startswith("rank/m"):
            _, tr = Q.oracle_distribute(c, oracle, trace=True)
            ms |= {int(r["count"]) for r in tr if r["kind"] == Q.LARGEST}
    assert {1, 2, 3, 4, 5, 511, 512, 513, 1024, 1025, 1155} <= ms, sorted(ms)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_case_equals_reference_sources(oracle, pins, case):
    k, g = Q.oracle_input(case, oracle)
    a = oracle.distribute(k, 0, g.W, 0, g.H, case.N)
    pins.check("quadtree/%s" % case.name, a, lambda: oracle.src_distribute(k, 0, g.W, 0, g.H, case.N))


@pytest.mark.parametrize("rows,cols,nfeatures,nlevels", WIDE)
def test_wide_image_equals_reference_sources(oracle, pins, rows, cols, nfeatures, nlevels):
    img = wide_image(rows, cols)
    prm = (nfeatures, 1.2, nlevels, 20, 7)
    R = oracle.RefExtractor(*prm)
    K, D = R(img)
    w, h = oracle.level_region(rows, cols, 1.0)
    assert oracle.n_ini(w, h) > 4 and len(K) > nfeatures + 3 * nlevels   # beyond the old nfeatures-based sizing
    assert len(K) <= oracle.max_keypoints(R.mnFeaturesPerLevel, R.mvInvScaleFactor, rows, cols)
    pins.check("extract_wide/%dx%d/%s" % (rows, cols, prm), (K, D), lambda: oracle.SrcExtractor(*prm)(img))
