"""The perfect tree's point-pair overload of SearchByProjection(cur, last) (perfect/src/ORBmatcher.cc:1727-1880), CPU
side: the restatement (oracle/homo_ref.py, on top of oracle/match_ref.cpp) equals the perfect tree's own overload on
real Frames and MapPoints (oracle/homo_harness.cpp, refperfect_homo_pairs in oracle/_ref/libhomoref.so), bit for bit --
nmatches, the pointer state and both point vectors of every call -- live where libhomoref.so is built and through
digests pinned in tests/golden/homo_pins.json otherwise (tests/refpins.py's format;
REFSRC_RECORD=1 rewrites them).  Where the reference tree is present, the perfect tree's sources also compile against the
shims (oracle/homo.mk) and link; without a GPU the shim refuses to construct."""
import ctypes as C
import json
import os
import subprocess

import pytest

from oracle import homo_ref
from tests import homo_cases
from tests.refpins import RECORD, Pins, digest

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "homo_pins.json")
CRAFTED = homo_cases.crafted()
REF_TREE = "/root/reference/perfect/src/Frame.cc"


class HomoPins(Pins):
    def __init__(self):
        with open(PINS) as f:
            self.d = json.load(f)

    def save(self):
        if RECORD:
            with open(PINS, "w") as f:
                json.dump(self.d, f, indent=0, sort_keys=True)
                f.write("\n")


@pytest.fixture(scope="module")
def pins():
    p = HomoPins()
    yield p
    p.save()


def _restatement(case):
    return homo_cases.run_restatement(
        case, lambda cur, last, th, mono: homo_ref.search_by_projection_last_pairs(cur, last, th, mono, 0.9, True))


def _check(pins, case):
    ours = _restatement(case)
    reference = lambda: homo_cases.run_harness(case, homo_cases.harness(homo_cases.REF_SO, "refperfect_"), "refperfect_")
    if os.path.exists(homo_cases.REF_SO):
        assert digest(reference()) == digest(ours), case.name
    pins.check("homo/" + case.name, ours, reference)
    return ours


@pytest.mark.parametrize("name", sorted(CRAFTED))
def test_restatement_equals_perfect_tree_crafted(pins, name):
    case = CRAFTED[name]
    homo_cases.edge(case, _check(pins, case))


@pytest.mark.parametrize("name", sorted(homo_cases.random_cases()))
def test_restatement_equals_perfect_tree_random(pins, name):
    n, seed = homo_cases.random_cases()[name]
    case = homo_cases.random_case(n, seed)
    res = _check(pins, case)
    nm, c2l, pl, _ = res[0]
    assert len(pl) > n // 4 and len(pl) > nm   # many pairs, some of them pruned


def test_perfect_tree_compiles_against_the_shims():
    """perfect/src/Frame.cc, KeyFrame.cc, MapPoint.cc, Map.cc, unmodified, against the shims: the library links against
    libb200orb.so and exports the harness entries; without a GPU the shim's constructor fails loudly."""
    if not os.path.exists(REF_TREE):
        pytest.skip("the reference is not on this box")
    import torch
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["make", "-C", os.path.join(root, "oracle"), "-f", "homo.mk", "-s"])
    L = homo_cases.harness(homo_cases.SHIM_SO, "shimperfect_")
    for name in ("homo_pairs", "homo_sequence"):
        assert hasattr(L, "shimperfect_" + name), name
    if torch.cuda.is_available():
        pytest.skip("GPU present: exercised by tests/test_homo_pairs_gpu.py")
    out = subprocess.run(["python", "-c", _LOUD % (root, homo_cases.SHIM_SO)], capture_output=True, text=True, timeout=300)
    assert out.returncode != 0 and "no CPU fallback" in out.stderr, out.stderr[-2000:]


# the shim's ORBmatcher throws from the harness (a C++ exception through a C frame ends the process): run it apart
_LOUD = """
import sys
sys.path.insert(0, %r)
from tests import homo_cases
case = homo_cases.crafted()["prune_kept"]
homo_cases.run_harness(case, homo_cases.harness(%r, "shimperfect_"), "shimperfect_")
"""


def test_pairs_entry_is_declared_and_bound():
    import orb_slam2_ssd_semantic_b200 as pkg
    from orb_slam2_ssd_semantic_b200._lib import EXPORTS
    assert "orbm_search_by_projection_last_pairs" in EXPORTS
    L = pkg.lib()
    assert len(L.orbm_search_by_projection_last_pairs.argtypes) == 10
    nm = C.c_int(0)
    assert L.orbm_search_by_projection_last_pairs(None, None, None, 15.0, 0, 0.9, 1, None, None, C.byref(nm)) == -1
