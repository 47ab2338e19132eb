"""The dense-flow restatement (oracle/farneback_py.py) against cv2 4.13 at its baseline dispatch level
(cv2.setUseOptimized(False)), bit for bit (uint32 view): the pyrDown of Flow.cc:26, each stage cv2 exposes (GaussianBlur,
resize, the Cholesky inverse, the Gaussian kernels), the flow after one level / one iteration, and the full call of
Flow.cc:29 on every scene and size of tests/flow_scenes.py; and against the goldens tools/make_flow_golden.py wrote."""
import glob
import os

import numpy as np
import pytest

from oracle import farneback_py as FB
from tests import flow_scenes as S

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture
def cv2_baseline():
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    cv2.setUseOptimized(False)
    yield cv2
    cv2.setUseOptimized(was)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    assert a.shape == b.shape
    assert (_bits(a) == _bits(b)).all(), "max |diff| %g" % np.abs(a.astype(np.float64) - b).max()


def _half_pair(scene, rows, cols, t0=0):
    g = S.frames(scene, 2 * rows, 2 * cols, 2, t0=t0)
    return FB.pyr_down(g[0], rows, cols), FB.pyr_down(g[1], rows, cols)


@pytest.mark.parametrize("rows,cols", [(480, 640), (194, 322), (195, 323), (32, 32), (33, 35)])
def test_pyr_down_equals_cv2(cv2_baseline, rows, cols):
    g = S.frames("room" if rows == 480 else "blobs", rows, cols, 1)[0]
    want = cv2_baseline.pyrDown(g, dstsize=(cols // 2, rows // 2))
    assert (FB.pyr_down(g, rows // 2, cols // 2) == want).all()


def test_gaussian_kernels_and_inverse_equal_cv2(cv2_baseline):
    for k, (ksize, sigma, _) in FB.GAUSS_KERNELS.items():
        assert ksize == max(int(np.rint(sigma * 5)) | 1, 3)
        assert (_bits(FB.level_kernel(k)) == _bits(cv2_baseline.getGaussianKernel(ksize, sigma, cv2_baseline.CV_32F).ravel())).all()
    g, xg, xxg, G, ig11, ig03, ig33, ig55 = FB.prepare_gaussian()
    _, inv = cv2_baseline.invert(G, flags=cv2_baseline.DECOMP_CHOLESKY)
    assert (FB.cholesky_inverse(G).view(np.uint64) == inv.view(np.uint64)).all()
    assert (ig11, ig03, ig33, ig55) == (inv[1, 1], inv[0, 3], inv[3, 3], inv[5, 5])
    assert abs(float(g.sum()) - 1.0) < 1e-6 and (g == g[::-1]).all() and (xg == -xg[::-1]).all()


@pytest.mark.parametrize("rows,cols", [(240, 320), (97, 161), (98, 162), (16, 16)])
def test_blur_and_resize_stages_equal_cv2(cv2_baseline, rows, cols):
    img = _half_pair("blobs", rows, cols)[0].astype(np.float32)
    for k, (ksize, sigma, _) in FB.GAUSS_KERNELS.items():
        b = FB.gaussian_blur(img, FB.level_kernel(k))
        _same(b, cv2_baseline.GaussianBlur(img, (ksize, ksize), sigma, sigmaY=sigma))
        for lk in range(1, 4):
            h, w = FB.level_size(rows, cols, lk)
            _same(FB.resize_linear(b, h, w), cv2_baseline.resize(b, (w, h), interpolation=cv2_baseline.INTER_LINEAR))
    fl = np.random.Generator(np.random.PCG64(5)).normal(0, 4, (rows // 2, cols // 2, 2)).astype(np.float32)
    _same(FB.resize_linear(fl, rows, cols), cv2_baseline.resize(fl, (cols, rows), interpolation=cv2_baseline.INTER_LINEAR))


@pytest.mark.parametrize("levels,iterations", [(0, 1), (0, 3), (1, 1)])
def test_partial_calls_equal_cv2(cv2_baseline, levels, iterations):
    """One level and one iteration (PolyExp, UpdateMatrices at zero flow, one box-filter solve), then the matrices
    updated between iterations, then the level change (flow resize and doubling)."""
    prev, cur = _half_pair("room", 240, 320)
    want = cv2_baseline.calcOpticalFlowFarneback(prev, cur, None, 0.5, levels, 15, iterations, 5, 1.2, 0)
    _same(FB.farneback(prev, cur, levels, iterations), want)


@pytest.mark.parametrize("rows,cols", S.HALF_SIZES)
@pytest.mark.parametrize("scene", S.SCENES)
def test_flow_equals_cv2(cv2_baseline, scene, rows, cols):
    prev, cur = _half_pair(scene, rows, cols)
    want = cv2_baseline.calcOpticalFlowFarneback(prev, cur, None, 0.5, 3, 15, 3, 5, 1.2, 0)
    _same(FB.farneback(prev, cur), want)


def test_level_cut_offs():
    """optflowgf.cpp stops adding levels once a side would drop under 32: the sizes of HALF_SIZES straddle each cut."""
    assert [FB.level_count(r, c) for r, c in S.HALF_SIZES] == [2, 1, 1, 0, 1, 2, 3, 0]


def test_baseline_dispatch_is_the_reproducible_target(cv2_baseline):
    """cv2's own flow at its optimized dispatch is not part of the contract; where the machine's dispatch differs, it is
    not this restatement's.  The baseline result does not depend on the thread count."""
    prev, cur = _half_pair("blobs", 240, 320)
    n = cv2_baseline.getNumThreads()
    try:
        cv2_baseline.setNumThreads(1)
        one = cv2_baseline.calcOpticalFlowFarneback(prev, cur, None, 0.5, 3, 15, 3, 5, 1.2, 0)
    finally:
        cv2_baseline.setNumThreads(n)
    _same(FB.farneback(prev, cur), one)


def test_goldens():
    files = sorted(glob.glob(os.path.join(GOLDEN, "farneback_*.npz")))
    assert len(files) >= 4
    for f in files:
        z = np.load(f)
        _same(FB.farneback(z["prev"], z["cur"]), z["flow"])
        g = z["gray"]
        assert (FB.pyr_down(g[0], *z["prev"].shape) == z["prev"]).all() and (FB.pyr_down(g[1], *z["cur"].shape) == z["cur"]).all()
