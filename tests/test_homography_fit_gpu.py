"""dynm_find_homography -- findHomography(points_current, points_last, RANSAC, 3) with its LM refinement on the device --
against the restatement (tests/homography_lm.py) and cv2's results stored in tests/golden/homography_fit.npz: H, mask
and found bit for bit, on every stored set, on TrackHomo's pair lists, at 8192 pairs, and on the argument checks (which
enqueue nothing); and the homography branch chained on the device: the point-pair search, the fit, the warp."""
import os

import numpy as np
import pytest

from tests import homography_fit_cases as HC
from tests import homography_lm as HL

pytestmark = pytest.mark.gpu
EINVAL = -1   # B200ORB_EINVAL
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "homography_fit.npz")


@pytest.fixture(scope="module")
def dm():
    from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask
    return DynamicMask()


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _same(got, want):
    (Hg, mg), (Hw, mw) = got, want
    assert (Hg is None) == (Hw is None)
    assert Hg is None or (_bits(Hg) == _bits(Hw)).all()
    assert (np.asarray(mg, np.uint8) == np.asarray(mw, np.uint8)).all()


def test_golden_sets_equal_restatement_and_cv2(dm):
    z = np.load(GOLDEN)
    exact = 0
    for name in z["names"]:
        src, dst = z[name + "/src"], z[name + "/dst"]
        got = dm.find_homography(src, dst)
        _same(got, HL.find_homography(src, dst))
        if bool(z[name + "/exact"]):
            Hc = z[name + "/H"]
            _same(got, (None if np.isnan(Hc).any() else Hc, z[name + "/mask"]))
            exact += 1
    assert exact >= 10


def test_largest_set(dm):
    src, dst = HC.related(8192, 8192, 0.3)
    got = dm.find_homography(src, dst)
    assert got[0] is not None
    _same(got, HL.find_homography(src, dst))


def test_no_model_and_exhausted_draws(dm):
    same = np.full((6, 2), 7.0, np.float32)
    H, mask = dm.find_homography(same, same)
    assert H is None and (mask == 0).all() and len(mask) == 6
    t = np.arange(12, dtype=np.float32)
    line = np.stack([t * 3 + 1, t * 2 + 5], 1)
    H, mask = dm.find_homography(line, line[::-1])
    assert H is None and (mask == 0).all()


def test_track_homo_pairs(dm):
    for name, src, dst in HC.track_homo_pairs():
        got = dm.find_homography(src, dst)
        assert got[0] is not None, name
        _same(got, HL.find_homography(src, dst))


def test_bad_arguments_enqueue_nothing(dm):
    from orb_slam2_ssd_semantic_b200 import _lib
    L = _lib.lib()
    four = np.array([[0, 0], [9, 1], [2, 8], [7, 7]], np.float32)
    big = np.zeros((8193, 2), np.float32)
    H = np.zeros(9)
    m = np.zeros(8193, np.uint8)
    f = np.zeros(1, np.int32)
    p = (lambda a: a.ctypes.data)
    before = dm.launch_count()
    bad = [(dm._h, p(four), p(four), 3, p(H), p(m), p(f)),
           (dm._h, p(big), p(big), 8193, p(H), p(m), p(f)),
           (dm._h, p(four), p(four), -1, p(H), p(m), p(f)),
           (dm._h, None, p(four), 4, p(H), p(m), p(f)),
           (dm._h, p(four), None, 4, p(H), p(m), p(f)),
           (dm._h, p(four), p(four), 4, None, p(m), p(f)),
           (dm._h, p(four), p(four), 4, p(H), None, p(f)),
           (dm._h, p(four), p(four), 4, p(H), p(m), None)]
    for args in bad:
        assert L.dynm_find_homography(*args) == EINVAL
    assert L.dynm_find_homography(None, p(four), p(four), 4, p(H), p(m), p(f)) != 0
    assert dm.launch_count() == before
    for n in (3, 8193):
        with pytest.raises(Exception):
            dm.find_homography(np.zeros((n, 2), np.float32), np.zeros((n, 2), np.float32))
    assert dm.launch_count() == before
    got = dm.find_homography(four, four)   # 4 pairs are accepted: runKernel of all four, mask all ones
    _same(got, HL.find_homography(four, four))
    assert dm.launch_count() > before


def test_chained_search_fit_warp(dm):
    """TrackHomo then ComputeMask's warp, all on the device: orbm_search_by_projection_last_pairs, dynm_find_homography
    on its pairs, dynm_warp_perspective of the frame by that H -- equal to the restatement of the same pairs."""
    import ctypes as C

    from oracle import homo_ref
    from oracle import homography_py as HP
    from orb_slam2_ssd_semantic_b200 import ORBmatcher, _lib, synth
    from orb_slam2_ssd_semantic_b200._abi import ptr
    from tests import homo_cases

    case = homo_cases.random_case(1000, 1)
    m = ORBmatcher(0.9, True)

    def device_search(cur, last, th, mono):
        out = np.full(max(cur.n, 1), -5, np.int32)
        acc = np.full(max(last.n, 1), -5, np.int32)
        nm = C.c_int(-5)
        cs, ls = cur.struct(), last.struct()
        _lib.check(_lib.lib().orbm_search_by_projection_last_pairs(m._h, C.byref(cs), C.byref(ls), float(th), int(mono),
                                                                   0.9, 1, ptr(out), ptr(acc), C.byref(nm)))
        return nm.value, out[:cur.n], acc[:last.n]

    _, _, pl, pc = homo_cases.run_restatement(case, device_search)[-1]
    _, _, rpl, rpc = homo_cases.run_restatement(
        case, lambda cur, last, th, mono: homo_ref.search_by_projection_last_pairs(cur, last, th, mono, 0.9, True))[-1]
    assert pl.tobytes() == rpl.tobytes() and pc.tobytes() == rpc.tobytes()
    H, mask = dm.find_homography(pc, pl)
    _same((H, mask), HL.find_homography(rpc, rpl))
    gray = synth.synth_frame(1234, 1)
    assert (dm.warp_perspective(gray, H) == HP.warp_perspective(gray, H)).all()
