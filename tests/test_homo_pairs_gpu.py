"""The perfect tree's point-pair overload of SearchByProjection(cur, last) (perfect/src/ORBmatcher.cc:1727-1880) on the
GPU, bit for bit:
  * the C-ABI (orbm_search_by_projection_last_pairs) == the restatement (pinned to the perfect tree's own code by
    tests/test_homo_pairs_cpu.py): nmatches, cur2last and the accepted list, on every crafted and random case;
  * its cur2last and nmatches == those of orbm_search_by_projection_last on the same inputs;
  * the Python mirror (ORBmatcher.SearchByProjectionPairs) == the C-ABI;
  * where oracle/_ref is built: the shim (shim/ORBmatcher.h) under the perfect tree's own Frame.cc / MapPoint.cc
    (libshimperfect.so) leaves what the perfect tree's own ORBmatcher.cc leaves (libhomoref.so) -- on every case, and
    on TrackHomo's two-step call sequence followed by the masked Frame constructor and TrackWithMotionModel's search."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import homo_ref
from tests import homo_cases
from tests.refpins import digest

pytestmark = pytest.mark.gpu
CASES = sorted(homo_cases.crafted()) + sorted(homo_cases.random_cases())


def _case(name):
    crafted = homo_cases.crafted()
    if name in crafted:
        return crafted[name]
    return homo_cases.random_case(*homo_cases.random_cases()[name])


def _abi_pairs(m, cur, last, th, mono):
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200._abi import ptr
    out = np.full(max(cur.n, 1), -5, np.int32)
    acc = np.full(max(last.n, 1), -5, np.int32)
    nm = C.c_int(-5)
    cs, ls = cur.struct(), last.struct()
    _lib.check(_lib.lib().orbm_search_by_projection_last_pairs(m._h, C.byref(cs), C.byref(ls), float(th), int(mono), 0.9, 1,
                                                              ptr(out), ptr(acc), C.byref(nm)))
    return nm.value, out[:cur.n], acc[:last.n]


@pytest.mark.parametrize("name", CASES)
def test_device_equals_restatement(name):
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    case = _case(name)
    m = ORBmatcher(0.9, True)
    for th in case.ths:
        got = _abi_pairs(m, case.cur, case.last, th, case.mono)
        want = homo_ref.search_by_projection_last_pairs(case.cur, case.last, th, case.mono, 0.9, True)
        assert got[0] == want[0] and got[1].tobytes() == want[1].tobytes() and got[2].tobytes() == want[2].tobytes(), th
        n4, c4 = m.SearchByProjection(case.cur, case.last, th, case.mono)   # the 4-argument entry: same results
        assert n4 == got[0] and c4.tobytes() == got[1].tobytes()
        nm, c2l, pairs = m.SearchByProjectionPairs(case.cur, case.last, th, case.mono)   # the Python mirror
        i = np.flatnonzero(got[2] >= 0)
        assert nm == got[0] and c2l.tobytes() == got[1].tobytes()
        assert pairs.dtype == np.int32 and pairs.shape == (len(i), 2)
        assert pairs[:, 0].tolist() == i.tolist() and pairs[:, 1].tolist() == got[2][i].tolist()
    res = homo_cases.run_restatement(case, lambda cur, last, th, mono: _abi_pairs(m, cur, last, th, mono))
    if name in homo_cases.crafted():
        homo_cases.edge(case, res)


def test_fused_and_generic_paths_both_run():
    """The random pairs sit on both sides of the fused kernel's limit: one launch below it, four above."""
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    m = ORBmatcher(0.9, True)
    for n, launches in ((homo_cases.SYM_FUSED, 1), (homo_cases.SYM_FUSED + 1, 4)):
        case = homo_cases.random_case(n, 3)
        before = m.launch_count()
        m.SearchByProjectionPairs(case.cur, case.last, 15.0, False)
        assert m.launch_count() - before == launches, n


def test_null_accepted_buffer_is_refused():
    from orb_slam2_ssd_semantic_b200 import ORBmatcher, lib
    case = homo_cases.crafted()["prune_kept"]
    m = ORBmatcher(0.9, True)
    out = np.zeros(case.cur.n, np.int32)
    nm = C.c_int(0)
    cs, ls = case.cur.struct(), case.last.struct()
    assert lib().orbm_search_by_projection_last_pairs(m._h, C.byref(cs), C.byref(ls), 15.0, 0, 0.9, 1,
                                                      out.ctypes.data, None, C.byref(nm)) == -1


def _built():
    return os.path.exists(homo_cases.REF_SO) and os.path.exists(homo_cases.SHIM_SO)


@pytest.mark.parametrize("name", CASES)
def test_shim_on_perfect_tree_objects_equals_perfect_tree(name):
    if not _built():
        pytest.skip("oracle/_ref is not built")
    case = _case(name)
    R = homo_cases.harness(homo_cases.REF_SO, "refperfect_")
    S = homo_cases.harness(homo_cases.SHIM_SO, "shimperfect_")
    want = homo_cases.run_harness(case, R, "refperfect_")
    assert digest(homo_cases.run_harness(case, S, "shimperfect_")) == digest(want)


@pytest.mark.parametrize("shift", [0.0, 0.2])
def test_track_homo_masked_frame_motion_model_sequence(shift):
    """TrackHomo (th, then cleared and 2*th below 20 matches), the masked constructor, TrackWithMotionModel's search: on
    the shim everything equals the perfect tree's own code -- both point vectors, both nmatches, both pointer states."""
    if not _built():
        pytest.skip("oracle/_ref is not built")
    inp = homo_cases.sequence_inputs(shift=shift)
    R = homo_cases.harness(homo_cases.REF_SO, "refperfect_")
    S = homo_cases.harness(homo_cases.SHIM_SO, "shimperfect_")
    want = homo_cases.run_sequence(inp, R, "refperfect_")
    got = homo_cases.run_sequence(inp, S, "shimperfect_")
    assert want[0] > 0 and len(want[2]) >= want[0] and len(want[5]) < len(want[1])   # pairs found, the mask dropped keypoints
    for a, b, what in zip(got, want, ("homo nmatches", "homo state", "points_last", "points_current", "track nmatches",
                                      "track state")):
        assert digest(a) == digest(b), what
