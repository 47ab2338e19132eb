"""The homography branch's warp (perfect/src/Flow.cc:78): the restatement oracle/homography_py.py against cv2 4.13 live,
bit for bit, at cv2.setUseOptimized(False) and (True) -- the 3x3 inverse (as uint64), the warped bytes on every case and
size of tests/warp_cases.py -- and against the goldens tools/make_homography_golden.py wrote.  Also the C-ABI surface of
the new entries (declared, exported, bound) and the shim header, which keeps the host call."""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import homography_py as HP
from tests import warp_cases as WC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "homography_warp.npz")
ENTRIES = ("dynm_warp_perspective", "dynm_warp_perspective_batch_device")


@pytest.fixture(params=[False, True], ids=["baseline", "optimized"])
def cv2_at(request):
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    cv2.setUseOptimized(request.param)
    yield cv2
    cv2.setUseOptimized(was)


def _random_h(rng):
    H = np.eye(3) + rng.normal(0, 0.05, (3, 3))
    H[2, :2] *= 0.01
    H[:2, 2] += rng.normal(0, 10, 2)
    return H


def test_invert_equals_cv2(cv2_at):
    rng = np.random.Generator(np.random.PCG64(3))
    Hs = [_random_h(rng) for _ in range(50)] + [WC.homography(c, 480, 640) for c in WC.CASES]
    for H in Hs:
        ok, want = cv2_at.invert(H)
        got = HP.invert3(H)
        assert (got.view(np.uint64) == want.view(np.uint64)).all()
    assert not HP.invert3(WC.homography("singular", 480, 640)).any()


@pytest.mark.parametrize("rows,cols", WC.SIZES + ((16, 2000), (7, 5), (1, 1)))
@pytest.mark.parametrize("case", WC.CASES)
def test_warp_equals_cv2(cv2_at, case, rows, cols):
    src = WC.image(rows, cols)
    H = WC.homography(case, rows, cols)
    want = cv2_at.warpPerspective(src, H, (cols, rows))
    got = HP.warp_perspective(src, H)
    assert got.shape == want.shape and (got == want).all(), "%d of %d bytes differ" % ((got != want).sum(), got.size)


def test_warp_equals_cv2_random_maps(cv2_at):
    rng = np.random.Generator(np.random.PCG64(5))
    src = WC.image(195, 323, seed=4)
    for _ in range(20):
        H = _random_h(rng)
        assert (HP.warp_perspective(src, H) == cv2_at.warpPerspective(src, H, (323, 195))).all()


def test_cases_reach_every_branch():
    """The suite's inputs cover what the integer path distinguishes: W == 0, short-saturated source coordinates, every
    sub-pixel index."""
    rows, cols = 480, 640
    seen = {"w0": False, "short": False}
    tx_all = set()
    for case in WC.CASES:
        M = HP.invert3(WC.homography(case, rows, cols))
        sx, sy, tx, ty = HP.warp_map(M, rows, cols)
        bw0 = HP.block_width(rows, cols)
        xs = np.arange(cols)
        W = (M[2, 0] * ((xs // bw0) * bw0) + M[2, 1] * np.arange(rows)[:, None]) + M[2, 2] + M[2, 0] * (xs % bw0)
        seen["w0"] |= bool((W == 0).any())
        seen["short"] |= bool(((sx == 32767) | (sx == -32768) | (sy == 32767) | (sy == -32768)).any())
        tx_all |= set(np.unique(tx).tolist())
    assert all(seen.values()), seen
    assert tx_all == set(range(32))


def test_warp_equals_goldens():
    z = np.load(GOLDEN)
    assert [str(c) for c in z["cases"]] == list(WC.CASES)
    assert (z["src"] == WC.image(*z["src"].shape)).all()
    for c, H, dst in zip(z["cases"], z["H"], z["dst"]):
        assert (HP.warp_perspective(z["src"], H) == dst).all(), c


def test_warp_rejects_what_cv2_rejects():
    with pytest.raises(ValueError):
        HP.warp_perspective(np.zeros((2, 32767), np.uint8), np.eye(3))
    with pytest.raises(ValueError):
        HP.warp_perspective(np.zeros((4, 4), np.float32), np.eye(3))


def _declared():
    txt = open(os.path.join(ROOT, "include", "b200orb.h")).read()
    return set(re.findall(r"\b(dynm_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", "", txt, flags=re.S)))


def test_entries_declared_exported_and_bound():
    from orb_slam2_ssd_semantic_b200 import _lib
    L = _lib.lib()
    for name in ENTRIES:
        assert name in _declared() and name in _lib.EXPORTS
        assert hasattr(L, name) and getattr(L, name).argtypes


def test_entries_refuse_without_a_handle():
    from orb_slam2_ssd_semantic_b200 import _lib
    L = _lib.lib()
    g = np.zeros((4, 4), np.uint8)
    H = np.eye(3)
    assert L.dynm_warp_perspective(None, g.ctypes.data, 4, 4, H.ctypes.data, g.ctypes.data) != 0
    assert L.dynm_warp_perspective_batch_device(None, None, 1, 4, 4, None, None) != 0


def test_flow_shim_still_syntax_checks():
    shim = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200", "csrc", "shim")
    subprocess.check_call(["g++", "-std=c++14", "-fsyntax-only", "-Wall", "-x", "c++", "-include",
                           os.path.join(ROOT, "oracle", "standin", "flow_decls.hpp"), os.path.join(shim, "Flow.h"),
                           "-I" + os.path.join(ROOT, "oracle", "standin"), "-I" + os.path.join(ROOT, "include")])
