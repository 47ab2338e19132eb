"""Restatement of the whole `findHomography(points_current, points_last, RANSAC, 3)` call of TrackHomo
(perfect/src/Tracking.cc:1386), Levenberg-Marquardt refinement included, at OpenCV 4.13's baseline dispatch
(cv2.setUseOptimized(False)).  It extends the RANSAC restatement of oracle/homography_py.py (the subset draws,
runKernel, the float errors and the adaptive iteration count, pinned there) with what comes after it:

  * the ordered compaction of the inliers and runKernel on them;
  * LMSolverImpl::run (the classic solver of levmarq.cpp) with HomographyRefineCallback over 9 parameters, at most 10
    iterations, eps = FLT_EPSILON: gain ratio R against Rlo = 0.25 / Rhi = 0.75, lambda = 1 and lc = 0.75 at the start,
    the damping D = diag(A) taken once from the first Jacobian, the nu update and invert(A, DECOMP_EIG) when lambda
    reaches 0;
  * H scaled by scaleFor(H22) (convertTo with alpha = 1 / H22);
  * the returned mask recomputed from the refined H: float error <= 9 over every pair.

Each matrix primitive the solver calls is a function of its own with the order of operations of OpenCV's baseline
code, which still runs SSE2 universal intrinsics (tests/test_homography_lm_cpu.py pins each against cv2):

  mul_transposed(J)     MulTransposedR: every entry of J^T J one sequential sum over the rows
  gemm_t(J, r)          GEMMSingleMul with a one-column result (taken as A * B^T): four interleaved accumulators over
  gemm(A, d, al, c, be)   k = 4j + q, the tail added into the first, then ((s0 + s1) + s2) + s3; times alpha plus beta c
  norm_l2sqr(r)         NormL2_SIMD<double>: four v_float64x2 accumulators over blocks of 8, each reduced across the
                        accumulators then the lanes, the tail added in order
  norm_inf(r)           the largest magnitude (no rounding)
  dot(a, b)             dotProd_64f: a running sum, each block of 4 products summed left to right and added to it,
                        then the remaining products in order
  solve_eig(A, b)       solve(A, b, x, DECOMP_EIG) and invert(A, X, DECOMP_EIG): the Jacobi eigen-decomposition of
  invert_eig(A)           oracle/homography_py.eigen_sym, then SVBkSb: eigenvalues at most 2 DBL_EPSILON times their
                        (signed, sequential) sum are dropped, every kept eigenpair adds into x (or X) in order

A sequential sum is `np.cumsum` started from +0.0 (C's `s = 0; s += ...`), so its order and its signed zeros are C's.
"""
from __future__ import annotations

import numpy as np

from oracle import homography_py as HP

FLT_EPS = HP.FLT_EPS
DBL_EPS = HP.DBL_EPS
THRESHOLD = 3.0            # Tracking.cc:1386: RANSAC, ransacReprojThreshold 3
CONFIDENCE = 0.995         # findHomography's defaults: confidence 0.995, maxIters 2000
MAX_ITERS = 2000
LM_ITERS = 10              # LMSolver::create(HomographyRefineCallback, 10)


def _seq(x) -> float:
    """C's `double s = 0; for (...) s += x[k];` over an array of double terms."""
    x = np.asarray(x, np.float64)
    return float(np.cumsum(np.concatenate(([0.0], x)))[-1]) if len(x) else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# Primitives


def mul_transposed(J) -> np.ndarray:
    """mulTransposed(J, A, true): A[i][j] = sum_k J[k][i] J[k][j], sequential in k, computed for j >= i and mirrored."""
    J = np.asarray(J, np.float64)
    c = J.shape[1]
    A = np.zeros((c, c))
    for i in range(c):
        for j in range(i, c):
            A[i, j] = A[j, i] = _seq(J[:, i] * J[:, j])
    return A


def _dot4(a, b) -> float:
    """GEMMSingleMul's A * B^T inner product: s_q over k = 4j + q, the tail into s0, then ((s0 + s1) + s2) + s3."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    n4 = len(a) // 4 * 4
    p = a * b
    s = [_seq(p[q:n4:4]) for q in range(4)]
    s[0] = float(np.cumsum(np.concatenate(([s[0]], p[n4:])))[-1])
    return ((s[0] + s[1]) + s[2]) + s[3]


def gemm_t(J, r) -> np.ndarray:
    """gemm(J, r, 1, noArray(), 0, v, GEMM_1_T) with a column r -> J^T r."""
    J = np.asarray(J, np.float64)
    r = np.asarray(r, np.float64).ravel()
    return np.array([_dot4(J[:, i], r) * 1.0 for i in range(J.shape[1])])


def gemm(A, d, alpha: float, c, beta: float) -> np.ndarray:
    """gemm(A, d, alpha, c, beta) with a column d: (A d) alpha + c beta, one row at a time."""
    A = np.asarray(A, np.float64)
    d = np.asarray(d, np.float64).ravel()
    c = np.asarray(c, np.float64).ravel()
    return np.array([_dot4(A[i], d) * alpha + c[i] * beta for i in range(A.shape[0])])


def norm_l2sqr(r) -> float:
    """norm(r, NORM_L2SQR) of doubles: accumulators acc[q][l] over r[8j + 2q + l], reduced ((a0 + a1) + a2) + a3 per
    lane, then lane 0 + lane 1, then the tail r[8j..] in order."""
    r = np.asarray(r, np.float64).ravel()
    n8 = len(r) // 8 * 8
    sq = r * r
    lane = [0.0, 0.0]
    for q in range(4):
        for l in range(2):
            lane[l] = lane[l] + _seq(sq[2 * q + l:n8:8])
    return float(np.cumsum(np.concatenate(([0.0 + (lane[0] + lane[1])], sq[n8:])))[-1])


def norm_inf(r) -> float:
    """norm(r, NORM_INF): the largest |r_i| (0 for an empty vector)."""
    r = np.asarray(r, np.float64).ravel()
    return float(np.abs(r).max()) if len(r) else 0.0


def dot(a, b) -> float:
    """Mat::dot of two double vectors (dotProd_64f at baseline dispatch, dotProd_ unrolled by 4): r = 0, then
    r += ((p0 + p1) + p2) + p3 per block of four products, then the remaining products added to r in order."""
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    n4 = len(a) // 4 * 4
    p = a * b
    r = 0.0
    for i in range(0, n4, 4):
        r += ((p[i] + p[i + 1]) + p[i + 2]) + p[i + 3]
    for i in range(n4, len(p)):
        r += p[i]
    return float(r)


def _svbksb_basis(A):
    W, V = HP.eigen_sym(A)
    return W, V, _seq(W) * (2 * DBL_EPS)


def solve_eig(A, b) -> np.ndarray:
    """solve(A, b, x, DECOMP_EIG) for a symmetric A and a column b: x += (sum_j v_k[j] b[j] / w_k) v_k per kept k."""
    W, V, thr = _svbksb_basis(A)
    b = np.asarray(b, np.float64).ravel()
    x = np.zeros(len(W))
    for k in range(len(W)):
        wi = float(W[k])
        if abs(wi) <= thr:
            continue
        s = _seq(V[k] * b) * (1.0 / wi)
        x = x + s * V[k]
    return x


def invert_eig(A) -> np.ndarray:
    """invert(A, X, DECOMP_EIG) for a symmetric A: X[i][j] += v_k[i] (v_k[j] / w_k) per kept k."""
    W, V, thr = _svbksb_basis(A)
    n = len(W)
    X = np.zeros((n, n))
    for k in range(n):
        wi = float(W[k])
        if abs(wi) <= thr:
            continue
        X = X + V[k][:, None] * (V[k] * (1.0 / wi))[None, :]
    return X


# ---------------------------------------------------------------------------------------------------------------------
# HomographyRefineCallback and the solver


def refine_residuals(h, M, m, jacobian: bool = True):
    """HomographyRefineCallback::compute of the 9 parameters h: the 2n residuals (x then y of each pair) and the 2n x 9
    Jacobian, in double from the float pairs."""
    h = np.asarray(h, np.float64).ravel()
    Mx = np.asarray(M, np.float32)[:, 0].astype(np.float64)
    My = np.asarray(M, np.float32)[:, 1].astype(np.float64)
    mx = np.asarray(m, np.float32)[:, 0].astype(np.float64)
    my = np.asarray(m, np.float32)[:, 1].astype(np.float64)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        ww = (h[6] * Mx + h[7] * My) + h[8]
        ww = np.where(np.abs(ww) > DBL_EPS, 1.0 / np.where(ww != 0, ww, 1.0), 0.0)
        xi = ((h[0] * Mx + h[1] * My) + h[2]) * ww
        yi = ((h[3] * Mx + h[4] * My) + h[5]) * ww
        n = len(Mx)
        err = np.empty(2 * n)
        err[0::2] = xi - mx
        err[1::2] = yi - my
        if not jacobian:
            return err, None
        J = np.zeros((2 * n, 9))
        J[0::2, 0] = Mx * ww; J[0::2, 1] = My * ww; J[0::2, 2] = ww
        J[0::2, 6] = (-Mx * ww) * xi; J[0::2, 7] = (-My * ww) * xi; J[0::2, 8] = -ww * xi
        J[1::2, 3] = Mx * ww; J[1::2, 4] = My * ww; J[1::2, 5] = ww
        J[1::2, 6] = (-Mx * ww) * yi; J[1::2, 7] = (-My * ww) * yi; J[1::2, 8] = -ww * yi
    return err, J


def lm_refine(H, M, m, max_iters: int = LM_ITERS):
    """LMSolverImpl::run(H8) with HomographyRefineCallback(M, m) -> (refined 3x3 double, iterations run)."""
    x = np.asarray(H, np.float64).reshape(9).copy()
    r, J = refine_residuals(x, M, m)
    S = norm_l2sqr(r)
    A = mul_transposed(J)
    v = gemm_t(J, r)
    D = np.diag(A).copy()
    Rlo, Rhi = 0.25, 0.75
    lam, lc, it = 1.0, 0.75, 0
    while True:
        Ap = A.copy()
        for i in range(9):
            Ap[i, i] += lam * D[i]
        d = solve_eig(Ap, v)
        xd = x - d
        rd, _ = refine_residuals(xd, M, m, jacobian=False)
        Sd = norm_l2sqr(rd)
        temp_d = gemm(A, d, -1.0, v, 2.0)
        dS = dot(d, temp_d)
        R = (S - Sd) / (dS if abs(dS) > DBL_EPS else 1.0)
        if R > Rhi:
            lam *= 0.5
            if lam < lc:
                lam = 0.0
        elif R < Rlo:
            t = dot(d, v)
            nu = (Sd - S) / (t if abs(t) > DBL_EPS else 1.0) + 2
            nu = min(max(nu, 2.0), 10.0)
            if lam == 0:
                Ai = invert_eig(A)
                maxval = DBL_EPS
                for i in range(9):
                    maxval = max(maxval, abs(float(Ai[i, i])))
                lam = lc = 1.0 / maxval
                nu *= 0.5
            lam *= nu
        if Sd < S:
            S = Sd
            x = xd
            r, J = refine_residuals(x, M, m)
            A = mul_transposed(J)
            v = gemm_t(J, r)
        it += 1
        if not (it < max_iters and norm_inf(d) >= FLT_EPS and norm_inf(r) >= FLT_EPS):
            break
    return x.reshape(3, 3), it


def scale_for(H) -> np.ndarray:
    """H.convertTo(H, CV_64F, scaleFor(H22)): every element times 1 / H22 when |H22| > FLT_EPSILON."""
    H = np.asarray(H, np.float64)
    h22 = float(H[2, 2])
    s = 1.0 / h22 if abs(h22) > FLT_EPS else 1.0
    return H * s + 0.0


def find_homography(src, dst):
    """cv::findHomography(src, dst, RANSAC, 3) with maxIters 2000 and confidence 0.995 -> (H 3x3 double or None,
    mask uint8[n]) as cv2 returns them.  Exactly 4 pairs: runKernel unrefined, mask all ones.  No model: (None, zeros).
    Fewer than 4 pairs raises ValueError (cv2 throws)."""
    src = np.asarray(src, np.float32).reshape(-1, 2)
    dst = np.asarray(dst, np.float32).reshape(-1, 2)
    n = len(src)
    if n < 4 or len(dst) != n:
        raise ValueError("findHomography needs at least 4 pairs")
    H, inl, _ = HP.ransac(src, dst, THRESHOLD, CONFIDENCE, MAX_ITERS)
    if H is None:
        return None, np.zeros(n, np.uint8)
    if n == 4:
        return H, np.ones(4, np.uint8)
    s, d = src[inl], dst[inl]
    if len(s) > 0:
        H0 = HP.run_kernel(s, d)
        if H0 is not None:
            H = H0
        H, _ = lm_refine(H, s, d)
        H = scale_for(H)
    mask = HP.reprojection_errors(H, src, dst) <= np.float32(THRESHOLD * THRESHOLD)
    return H, mask.astype(np.uint8)
