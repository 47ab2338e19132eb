"""dynm_find_homography on the crafted sets of tests/homography_edge_cases.py: H, mask and found equal to the restatement
(tests/homography_lm.py) bit for bit on every set, and to cv2's results stored in tests/golden/homography_edges.npz bit
for bit where the refinement runs on fewer than 100 residual rows (within the BLAS hand-off's bound above).

The homography batches (orbs_submit with homography = 1) run the same fit (launch_hf_fit) on pairs of keypoints the
extractor found in the frames, so they cannot be handed these crafted coordinates; tests/test_homography_chain_gpu.py
pins the fit inside the batch on its own frames."""
import os

import numpy as np
import pytest

from tests import homography_lm as HL

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "homography_edges.npz")
Z = np.load(GOLDEN)
NAMES = [str(n) for n in Z["names"]]


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


@pytest.mark.parametrize("name", NAMES)
def test_case_equals_restatement_and_cv2(dm, name):
    src, dst = Z[name + "/src"], Z[name + "/dst"]
    got = dm.find_homography(src, dst)
    _same(got, HL.find_homography(src, dst))
    Hc, mc = Z[name + "/H"], Z[name + "/mask"]
    Hc = None if np.isnan(Hc).any() else Hc
    if bool(Z[name + "/exact"]):
        _same(got, (Hc, mc))
    else:
        assert np.abs(got[0] - Hc).max() <= 1e-6 * np.abs(Hc).max()
        assert (got[1] != mc).sum() <= max(2, len(src) // 500)
