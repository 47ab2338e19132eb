"""findHomography's refinement and the whole RANSAC, 3 call (perfect/src/Tracking.cc:1386): the restatement in
tests/homography_lm.py against cv2 4.13 live at cv2.setUseOptimized(False), bit for bit:

  * each matrix primitive the LM solver calls: mulTransposed, gemm (J^T r and A d -1 + v 2), norm L2SQR and INF,
    solve and invert with DECOMP_EIG (the dot product is pinned through the whole call);
  * lm_refine(run_kernel(all pairs)) against findHomography(method 0), which is runKernel plus the LM on every pair,
    for 5 to 49 pairs;
  * find_homography's H and mask against findHomography(RANSAC, 3) on sets refined over fewer than 50 inliers, and
    on the sets stored in tests/golden/homography_fit.npz.

From 100 residual rows (50 inliers) a cv2 built with LAPACK computes J^T r with its BLAS's dgemm instead of its own
loop; the order of that sum belongs to the BLAS kernel the host CPU selects, so there the test pins the hand-off itself
and bounds the distance between the two refined H."""
import os

import numpy as np
import pytest

from oracle import homography_py as HP
from tests import homography_fit_cases as HC
from tests import homography_lm as HL

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "homography_fit.npz")


@pytest.fixture
def cv2():
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    cv2.setUseOptimized(False)
    yield cv2
    cv2.setUseOptimized(was)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _eq(a, b):
    return a.shape == b.shape and (_bits(a) == _bits(b)).all()


def test_primitives_equal_cv2(cv2):
    rng = np.random.Generator(np.random.PCG64(11))
    for _ in range(100):
        m = int(rng.integers(1, 100))
        J = rng.normal(size=(m, 9)) * 10.0 ** rng.uniform(-3, 3, size=(1, 9))
        r = rng.normal(size=(m, 1))
        assert _eq(HL.mul_transposed(J), cv2.mulTransposed(J, True))
        assert _eq(HL.gemm_t(J, r), cv2.gemm(J, r, 1, None, 0, flags=cv2.GEMM_1_T).ravel())
        assert HL.norm_l2sqr(r) == cv2.norm(r, cv2.NORM_L2SQR)
        assert HL.norm_inf(r) == cv2.norm(r, cv2.NORM_INF)
        A = J.T @ J
        d = rng.normal(size=(9, 1))
        v = rng.normal(size=(9, 1))
        assert _eq(HL.gemm(A, d, -1.0, v, 2.0), cv2.gemm(A, d, -1, v, 2).ravel())
        assert _eq(HL.solve_eig(A, v), cv2.solve(A, v, flags=cv2.DECOMP_EIG)[1].ravel())
        assert _eq(HL.invert_eig(A), cv2.invert(A, flags=cv2.DECOMP_EIG)[1])
    # a rank-deficient matrix: SVBkSb drops the eigenvalues below its threshold
    B = rng.normal(size=(5, 9))
    A = B.T @ B
    assert _eq(HL.invert_eig(A), cv2.invert(A, flags=cv2.DECOMP_EIG)[1])


def test_mul_transposed_is_sequential_at_every_height(cv2):
    rng = np.random.Generator(np.random.PCG64(12))
    for m in (100, 1000, 16384):
        J = rng.normal(size=(m, 9))
        assert _eq(HL.mul_transposed(J), cv2.mulTransposed(J, True))
        assert HL.norm_l2sqr(J[:, 0]) == cv2.norm(J[:, 0], cv2.NORM_L2SQR)


def test_large_gemm_goes_to_blas(cv2):
    """From 100 rows, J^T r is no longer OpenCV's loop: the restatement keeps that loop's order (OpenCV without a BLAS),
    cv2 may differ from it in the last bits and no further."""
    rng = np.random.Generator(np.random.PCG64(13))
    J = rng.normal(size=(400, 9))
    r = rng.normal(size=(400, 1))
    got, want = HL.gemm_t(J, r), cv2.gemm(J, r, 1, None, 0, flags=cv2.GEMM_1_T).ravel()
    assert np.abs(got - want).max() <= 1e-12 * np.abs(J).sum(0).max()


@pytest.mark.parametrize("n", [5, 8, 13, 20, 33, 49])
def test_lm_refine_equals_cv2_method_0(cv2, n):
    for seed in range(8):
        src, dst = HC.related(500 * n + seed, n, 0.0)
        H, _ = cv2.findHomography(src, dst, 0)
        H0 = HP.run_kernel(src, dst)
        mine, _ = HL.lm_refine(H0, src, dst)
        assert _eq(HL.scale_for(mine), H), "n %d seed %d" % (n, seed)


def test_lm_refine_close_to_cv2_beyond_the_blas_hand_off(cv2):
    for n in (60, 500, 2000):
        src, dst = HC.related(77 + n, n, 0.0)
        H, _ = cv2.findHomography(src, dst, 0)
        mine = HL.scale_for(HL.lm_refine(HP.run_kernel(src, dst), src, dst)[0])
        assert np.abs(mine - H).max() <= 1e-6 * np.abs(H).max()


@pytest.mark.parametrize("n", [4, 5, 8, 20, 51])
def test_find_homography_equals_cv2(cv2, n):
    checked = 0
    for seed in range(12):
        src, dst = HC.related(3000 * n + seed, n, (0.0, 0.3, 0.6)[seed % 3])
        inl = HP.ransac(src, dst)[1]
        if inl is not None and inl.sum() >= 50:
            continue
        H, mask = cv2.findHomography(src, dst, cv2.RANSAC, 3)
        mine, mmask = HL.find_homography(src, dst)
        assert (H is None) == (mine is None)
        assert H is None or _eq(mine, H)
        assert (mmask == mask.ravel()).all()
        checked += 1
    assert checked >= 6


def test_find_homography_masks_match_cv2_on_large_sets(cv2):
    for n in (200, 2000, 8192):
        src, dst = HC.related(n, n, 0.3)
        H, mask = cv2.findHomography(src, dst, cv2.RANSAC, 3)
        mine, mmask = HL.find_homography(src, dst)
        assert np.abs(mine - H).max() <= 1e-6 * np.abs(H).max()
        assert (mmask != mask.ravel()).sum() <= max(2, n // 500)


def test_no_model_and_argument_errors(cv2):
    same = np.full((6, 2), 7.0, np.float32)
    H, mask = cv2.findHomography(same, same, cv2.RANSAC, 3)
    mine, mmask = HL.find_homography(same, same)
    assert H is None and mine is None and (mmask == mask.ravel()).all() and len(mmask) == 6
    with pytest.raises(ValueError):
        HL.find_homography(same[:3], same[:3])


def test_golden_sets():
    z = np.load(GOLDEN)
    exact = 0
    for name in z["names"]:
        src, dst = z[name + "/src"], z[name + "/dst"]
        H, mask = HL.find_homography(src, dst)
        Hc = z[name + "/H"]
        assert (H is None) == bool(np.isnan(Hc).any()), name
        if bool(z[name + "/exact"]):
            assert H is None or _eq(H, Hc), name
            assert (mask == z[name + "/mask"]).all(), name
            exact += 1
        else:
            assert np.abs(H - Hc).max() <= 1e-6 * np.abs(Hc).max(), name
    assert exact >= 10


def test_track_homo_pairs(cv2):
    """TrackHomo's own pair lists: H and mask equal cv2 bit for bit below 50 inliers, within the BLAS hand-off above."""
    for name, src, dst in HC.track_homo_pairs():
        H, mask = cv2.findHomography(src, dst, cv2.RANSAC, 3)
        mine, mmask = HL.find_homography(src, dst)
        assert (H is None) == (mine is None), name
        if H is None:
            continue
        if HP.ransac(src, dst)[1].sum() < 50:
            assert _eq(mine, H) and (mmask == mask.ravel()).all(), name
        else:
            assert np.abs(mine - H).max() <= 1e-6 * np.abs(H).max(), name
            assert (mmask != mask.ravel()).sum() <= max(2, len(src) // 500), name


def test_thread_count_changes_no_bit(cv2):
    """cv2's result does not depend on its thread count, so the single-threaded restatement pins the call as such."""
    was = cv2.getNumThreads()
    try:
        for name, src, dst in HC.cases()[:12] + HC.track_homo_pairs()[:1]:
            got = []
            for k in (1, 4):
                cv2.setNumThreads(k)
                got.append(cv2.findHomography(src, dst, cv2.RANSAC, 3))
            (H1, m1), (H4, m4) = got
            assert (H1 is None) == (H4 is None), name
            assert H1 is None or _eq(H1, H4), name
            assert (m1 == m4).all(), name
    finally:
        cv2.setNumThreads(was)


def test_noise_set_runs_every_iteration():
    name, src, dst = [c for c in HC.cases() if c[0] == "noise_40_full_run"][0]
    H, inl, iters = HP.ransac(src, dst)
    assert iters == 2000 and H is not None
    assert HL.find_homography(src, dst)[0] is not None
