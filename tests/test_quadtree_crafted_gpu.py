"""GPU: k_quadtree on the crafted candidate lists of tests/quadtree_cases.py, through orbx_distribute, bit for bit against
the oracle's DistributeOctTree (the count and (x, y, score) of every selected keypoint in list order); the entry's
refusals; and output sizing on images whose levels have more than four initial nodes, on a fresh handle."""
import ctypes as C

import numpy as np
import pytest

from tests import quadtree_cases as Q
from tests.test_quadtree_cases_cpu import WIDE, wide_image

pytestmark = pytest.mark.gpu

CASES = Q.all_cases()
EINVAL, ECAP = -1, -2


@pytest.fixture(scope="module")
def extractors():
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    cache = {}

    def get(params):
        if params not in cache:
            cache[params] = ORBextractor(*params)
        return cache[params]
    return get


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_case_equals_oracle(oracle, extractors, case):
    got = extractors(case.params).distribute(case.rows, case.cols, case.level, case.N, case.xys)
    want = Q.oracle_distribute(case, oracle)
    assert got.dtype == np.int32 and got.shape == want.shape, (case.edge, got.shape, want.shape)
    bad = np.flatnonzero((got != want).any(1))
    assert not len(bad), (case.edge, bad[:8].tolist(), got[bad[:8]].tolist(), want[bad[:8]].tolist())


def _call(ex, rows, cols, level, N, xys, n=None, out="buf", n_out="int"):
    from orb_slam2_ssd_semantic_b200 import _lib
    xys = None if xys is None else np.ascontiguousarray(xys, np.int32)
    buf = np.zeros((max(len(xys) if xys is not None else 1, 1), 3), np.int32)
    m = C.c_int(-7)
    return _lib.lib().orbx_distribute(ex.handle, rows, cols, level, N,
                                      None if xys is None else xys.ctypes.data_as(C.c_void_p),
                                      len(xys) if n is None else n,
                                      buf.ctypes.data_as(C.c_void_p) if out == "buf" else None, len(buf),
                                      C.byref(m) if n_out == "int" else None), m.value


def test_refusals_launch_nothing(extractors):
    params = (1000, 1.2, 8, 20, 7)
    ex = extractors(params)
    g0, g7 = Q.geometry(params, 480, 640, 0), Q.geometry(params, 480, 640, 7)
    ok = Q._xys([(0, 0), (g0.W - 1, g0.H - 1)], scores=[0, 255])
    assert _call(ex, 480, 640, 0, 10, ok) == (0, 2)
    assert _call(ex, 480, 640, 7, g7.nfeat, Q._xys([(g7.W - 1, g7.H - 1)], scores=[9])) == (0, 1)
    before = ex.launch_count()
    refused = [
        ("level -1", (480, 640, -1, 10, ok), EINVAL), ("level 8", (480, 640, 8, 10, ok), EINVAL),
        ("N -1", (480, 640, 0, -1, ok), EINVAL), ("N > N_0", (480, 640, 0, g0.nfeat + 1, ok), EINVAL),
        ("N > N_7", (480, 640, 7, g7.nfeat + 1, Q._xys([(0, 0)], scores=[1])), EINVAL),
        ("x = 15", (480, 640, 0, 10, [[15, 20, 1]]), EINVAL), ("y = 15", (480, 640, 0, 10, [[20, 15, 1]]), EINVAL),
        ("x = 16 + W", (480, 640, 0, 10, [[16 + g0.W, 20, 1]]), EINVAL),
        ("y = 16 + H", (480, 640, 0, 10, [[20, 16 + g0.H, 1]]), EINVAL),
        ("x = 16 + W on level 7", (480, 640, 7, 10, [[16 + g7.W, 20, 1]]), EINVAL),
        ("score -1", (480, 640, 0, 10, [[20, 20, -1]]), EINVAL), ("score 256", (480, 640, 0, 10, [[20, 20, 256]]), EINVAL),
        ("n above the slots", (480, 640, 7, 10, np.tile([[20, 20, 1]], (g7.slots + 1, 1))), ECAP),
    ]
    for what, args, rc in refused:
        assert _call(ex, *args)[0] == rc, what
    assert _call(ex, 480, 640, 0, 10, None, n=2)[0] == EINVAL                 # null list
    assert _call(ex, 480, 640, 0, 10, ok, out=None)[0] == EINVAL              # null output
    assert _call(ex, 480, 640, 0, 10, ok, n_out=None)[0] == EINVAL            # null count
    assert ex.launch_count() == before
    # exactly at the slot capacity it runs
    full = np.tile([[20, 20, 1]], (g7.slots, 1))
    assert _call(ex, 480, 640, 7, 10, full) == (0, 1)
    # the count comes back with ECAP and nothing is written when cap is too small
    from orb_slam2_ssd_semantic_b200 import _lib
    four = Q._xys(Q._quad_tree_list((0, 0, g0.W, g0.H), 1, 4), seed=3)
    buf = np.full((3, 3), -5, np.int32)
    m = C.c_int(0)
    assert _lib.lib().orbx_distribute(ex.handle, 480, 640, 0, 4, four.ctypes.data_as(C.c_void_p), 4,
                                      buf.ctypes.data_as(C.c_void_p), 3, C.byref(m)) == ECAP
    assert m.value == 4 and (buf == -5).all()


def test_readbacks_refuse_after_distribute_until_next_extract(extractors):
    from orb_slam2_ssd_semantic_b200 import _lib
    L = _lib.lib()
    params = (1000, 1.2, 8, 20, 7)
    ex = extractors(params)
    img = wide_image(480, 640, seed=4)
    ex(img)
    n = C.c_int(0)
    cand = np.zeros((70000, 3), np.int32)
    lvl = np.zeros((480, 640), np.uint8)
    counts = np.zeros(8, np.int32)

    def readbacks():
        return (L.orbx_get_candidates(ex.handle, 0, 0, cand.ctypes.data_as(C.c_void_p), len(cand), C.byref(n)),
                L.orbx_get_level(ex.handle, 0, 0, 0, lvl.ctypes.data_as(C.c_void_p), 640),
                L.orbx_candidates_per_level(ex.handle, 0, counts.ctypes.data_as(C.c_void_p)),
                L.orbx_device_results(ex.handle, None, None, None, None))
    assert readbacks() == (0, 0, 0, 0)
    ex.distribute(480, 640, 0, 10, Q._xys([(5, 5), (300, 200)], seed=1))
    assert readbacks() == (EINVAL,) * 4
    ex(img)
    assert readbacks() == (0, 0, 0, 0)


@pytest.mark.parametrize("rows,cols,nfeatures,nlevels", WIDE)
def test_fresh_extractor_on_wide_images(oracle, rows, cols, nfeatures, nlevels):
    """A fresh handle's first frame and first batch: levels with nIni > 4 return up to 4*nIni keypoints."""
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    prm = (nfeatures, 1.2, nlevels, 20, 7)
    img, img2 = wide_image(rows, cols), wide_image(rows, cols, seed=1)
    R = oracle.RefExtractor(*prm)
    want = [R(img), R(img2)]
    assert len(want[0][0]) > nfeatures + 3 * nlevels + 64
    K, D = ORBextractor(*prm)(img)
    assert K.tobytes() == want[0][0].tobytes() and np.array_equal(D, want[0][1])
    out = ORBextractor(*prm).extract_batch(np.stack([img, img2]))
    for (K, D), (K2, D2) in zip(out, want):
        assert K.tobytes() == K2.tobytes() and np.array_equal(D, D2)


def test_handles_with_different_quadtree_memory_alternate(oracle):
    """The quad-tree's dynamic shared memory follows the level quota (here 1003 and 220 list entries): a handle that sized
    its geometry first still launches after another handle sized a smaller one, in both orders."""
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    img = wide_image(480, 640, seed=2)
    big, small = ORBextractor(1000, 1.2, 1, 20, 7), ORBextractor(1000, 1.2, 8, 20, 7)
    want = {id(big): oracle.RefExtractor(1000, 1.2, 1, 20, 7)(img)[0], id(small): oracle.RefExtractor(1000, 1.2, 8, 20, 7)(img)[0]}
    for ex in (big, small, big, small):
        assert ex(img)[0].tobytes() == want[id(ex)].tobytes()


def test_max_keypoints_for_is_reached(oracle):
    """orbx_max_keypoints_for == what the kernel returns on the list whose first sweep gives 4*nIni > N + 3, without
    allocating (a fresh handle still reports the geometry-free bound afterwards)."""
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    case = next(c for c in CASES if c.name == "ini/nini58/all_quadrants")
    ex = ORBextractor(*case.params)
    bound = ex.max_keypoints(case.rows, case.cols)
    fresh = ex.max_keypoints()
    assert bound == oracle.max_keypoints(ex.mnFeaturesPerLevel, ex.GetInverseScaleFactors(), case.rows, case.cols)
    assert fresh == max(case.N + 3, 16) < bound
    assert ex.max_keypoints() == fresh   # the query allocated no geometry
    got = ex.distribute(case.rows, case.cols, case.level, case.N, case.xys)
    assert len(got) == bound == 4 * 58
    assert ex.max_keypoints() == bound   # the handle now has that geometry
    from orb_slam2_ssd_semantic_b200 import _lib
    n = C.c_int(-1)
    assert _lib.lib().orbx_max_keypoints_for(ex.handle, 0, 640, C.byref(n)) == 0 and n.value == 0
    assert _lib.lib().orbx_max_keypoints_for(ex.handle, 480, 4096, C.byref(n)) == EINVAL
    assert _lib.lib().orbx_max_keypoints_for(ex.handle, 20, 640, C.byref(n)) == -5   # B200ORB_EGEOM: level 0 is 20 px tall
