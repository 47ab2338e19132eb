"""findHomography(src, dst, RANSAC, 3) up to its refinement (perfect/src/Tracking.cc:1386): the restatement in
oracle/homography_py.py against cv2 4.13 live, at cv2.setUseOptimized(False) and (True), at every stage cv2 exposes:

  * eigen_sym == cv2.eigen (values and vectors as uint64) -- the Jacobi sweep runKernel calls;
  * run_kernel == cv2.findHomography of exactly 4 pairs (RANSAC and method 0 both return runKernel unrefined);
  * the RANSAC inlier set: cv2.findHomography(inliers, method 0) -- runKernel + LM refinement of exactly those pairs --
    equals cv2.findHomography(all, RANSAC) bit for bit, so the subset draws, checkSubset, the hypotheses, the float
    errors and the adaptive stop select the very inliers cv2 refines; and cv2's returned mask is the inlier set of its
    refined H under the restated error (<= 9 in float).
The LM refinement itself is not restated: the restatement's unrefined H differs from cv2's refined H."""
import numpy as np
import pytest

from oracle import homography_py as HP


@pytest.fixture(params=[False, True], ids=["baseline", "optimized"])
def cv2_at(request):
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    cv2.setUseOptimized(request.param)
    yield cv2
    cv2.setUseOptimized(was)


def _pairs(cv2, rng, n, noise=0.7, outliers=0.4):
    src = rng.uniform(0, 640, (n, 2)).astype(np.float32)
    Ht = np.eye(3) + rng.normal(0, 0.05, (3, 3))
    Ht[2, :2] *= 0.001
    d = cv2.perspectiveTransform(src[None].astype(np.float64), Ht)[0] + rng.normal(0, noise, (n, 2))
    out = rng.random(n) < outliers
    d[out] = rng.uniform(0, 640, (int(out.sum()), 2))
    return src, d.astype(np.float32)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def test_eigen_equals_cv2(cv2_at):
    rng = np.random.Generator(np.random.PCG64(1))
    for _ in range(60):
        B = rng.normal(size=(12, 9))
        ok, w, v = cv2_at.eigen(B.T @ B)
        W, V = HP.eigen_sym(B.T @ B)
        assert (_bits(W) == _bits(w.ravel())).all() and (_bits(V) == _bits(v)).all()


def test_run_kernel_equals_cv2_on_four_pairs(cv2_at):
    rng = np.random.Generator(np.random.PCG64(2))
    for _ in range(100):
        src, dst = _pairs(cv2_at, rng, 4, outliers=0.0)
        for method in (0, cv2_at.RANSAC):
            H, mask = cv2_at.findHomography(src, dst, method, 3)
            mine = HP.run_kernel(src, dst)
            assert (H is None) == (mine is None)
            if H is not None:
                assert (_bits(mine) == _bits(H)).all()


def test_degenerate_pairs_give_no_model(cv2_at):
    src = np.full((6, 2), 7.0, np.float32)
    H, _ = cv2_at.findHomography(src, src, cv2_at.RANSAC, 3)
    assert H is None and HP.ransac(src, src)[0] is None
    with pytest.raises(ValueError):
        HP.ransac(src[:3], src[:3])


@pytest.mark.parametrize("n", [5, 8, 20, 51, 200, 2000])
def test_ransac_inliers_are_the_ones_cv2_refines(cv2_at, n):
    rng = np.random.Generator(np.random.PCG64(100 + n))
    checked = 0
    for trial in range(12 if n < 2000 else 3):
        src, dst = _pairs(cv2_at, rng, n, outliers=rng.uniform(0.0, 0.6))
        H, mask = cv2_at.findHomography(src, dst, cv2_at.RANSAC, 3)
        Hr, inl, iters = HP.ransac(src, dst)
        assert (H is None) == (Hr is None)
        if H is None or inl.sum() <= 4:   # 4 inliers: cv2 refines them, its method 0 on 4 pairs does not
            continue
        H0, _ = cv2_at.findHomography(src[inl], dst[inl], 0)
        assert (_bits(H0) == _bits(H)).all(), "trial %d: the restated inlier set is not the one cv2 refined" % trial
        assert ((HP.reprojection_errors(H, src, dst) <= np.float32(9)) == mask.ravel().astype(bool)).all()
        checked += 1
    assert checked >= 2


def test_ransac_adaptive_stop_and_full_run(cv2_at):
    """50 % outliers end early; pairs with one inlier model of 5 among 40 random pairs run all 2000 iterations."""
    rng = np.random.Generator(np.random.PCG64(7))
    src, dst = _pairs(cv2_at, rng, 200, noise=0.3, outliers=0.5)
    _, _, iters = HP.ransac(src, dst)
    assert 0 < iters < 2000
    src = rng.uniform(0, 640, (40, 2)).astype(np.float32)
    dst = rng.uniform(0, 640, (40, 2)).astype(np.float32)
    H, mask = cv2_at.findHomography(src, dst, cv2_at.RANSAC, 3)
    Hr, inl, iters = HP.ransac(src, dst)
    assert iters == 2000 and (H is None) == (Hr is None)
