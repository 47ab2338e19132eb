"""Restatement of the homography branch's warp, `cv::warpPerspective(GrayImg, dest, Homo, GrayImg.size())`
(perfect/src/Flow.cc:78): u8, one channel, INTER_LINEAR, BORDER_CONSTANT 0, destination size = source size.  It follows
OpenCV 4.13's integer path operation by operation, so it equals cv2 bit for bit at any dispatch level
(tests/test_homography_cpu.py):

  * `invert(M, M)` (DECOMP_LU; no WARP_INVERSE_MAP at Flow.cc:78): the closed-form 3x3 inverse of cv::invert, det3 and the
    nine cofactor products times 1 / det, in double; a singular matrix (det == 0) inverts to zeros.
  * WarpPerspectiveInvoker: the image is walked in blocks of bh0 x bw0 pixels (bh0 = min(16, rows),
    bw0 = min(1024 / bh0, cols)); per row y of a block that starts at column xb, X0 = M0 xb + M1 y + M2 (Y0, W0 alike),
    and per column x1 of the block (warpPerspectiveBlockline): W = W0 + M6 x1, W = W ? 32 / W : 0,
    fX = max(INT_MIN, min(INT_MAX, (X0 + M0 x1) W)), X = saturate_cast<int>(fX) (round half to even), source pixel
    saturate_cast<short>(X >> 5) and 5-bit sub-pixel index X & 31 (Y alike).
  * remapBilinear with the fixed-point table of initInterTab2D (INTER_REMAP_COEF_BITS = 15): weights
    (32 - ty)(32 - tx) 32, (32 - ty) tx 32, ty (32 - tx) 32, ty tx 32 (the first saturates to 32767 at tx = ty = 0, which
    leaves every u8 value unchanged), taps outside the image read the border value 0, result (sum + 2^14) >> 15.

Every operation is a single IEEE double operation, an integer one, or a comparison, so numpy reproduces it exactly.
"""
from __future__ import annotations

import math

import numpy as np

INTER_BITS = 5
INTER_TAB_SIZE = 1 << INTER_BITS
COEF_BITS = 15
INT_MIN, INT_MAX = float(-2 ** 31), float(2 ** 31 - 1)


def invert3(H) -> np.ndarray:
    """cv::invert(H, Hinv, DECOMP_LU) of a 3x3 double matrix (its closed form for n == 3); zeros when det == 0."""
    S = np.asarray(H, np.float64).reshape(3, 3)
    d = (S[0, 0] * (S[1, 1] * S[2, 2] - S[1, 2] * S[2, 1])
         - S[0, 1] * (S[1, 0] * S[2, 2] - S[1, 2] * S[2, 0])
         + S[0, 2] * (S[1, 0] * S[2, 1] - S[1, 1] * S[2, 0]))
    t = np.zeros(9, np.float64)
    if d != 0.0:
        d = 1.0 / d
        t[0] = (S[1, 1] * S[2, 2] - S[1, 2] * S[2, 1]) * d
        t[1] = (S[0, 2] * S[2, 1] - S[0, 1] * S[2, 2]) * d
        t[2] = (S[0, 1] * S[1, 2] - S[0, 2] * S[1, 1]) * d
        t[3] = (S[1, 2] * S[2, 0] - S[1, 0] * S[2, 2]) * d
        t[4] = (S[0, 0] * S[2, 2] - S[0, 2] * S[2, 0]) * d
        t[5] = (S[0, 2] * S[1, 0] - S[0, 0] * S[1, 2]) * d
        t[6] = (S[1, 0] * S[2, 1] - S[1, 1] * S[2, 0]) * d
        t[7] = (S[0, 1] * S[2, 0] - S[0, 0] * S[2, 1]) * d
        t[8] = (S[0, 0] * S[1, 1] - S[0, 1] * S[1, 0]) * d
    return t.reshape(3, 3)


def block_width(rows: int, cols: int) -> int:
    """bw0 of WarpPerspectiveInvoker: the column blocks whose first column anchors X0, Y0, W0."""
    bh0 = min(32 // 2, rows)
    return min(32 * 32 // bh0, cols)


def warp_map(M, rows: int, cols: int):
    """-> (sx, sy, tx, ty) int64 rows x cols: the source pixel and 5-bit sub-pixel index of every destination pixel for
    the inverse map M (3x3 double), as warpPerspectiveBlockline computes them."""
    M = np.asarray(M, np.float64).reshape(9)
    bw0 = block_width(rows, cols)
    xs = np.arange(cols)
    xb = ((xs // bw0) * bw0).astype(np.float64)[None, :]
    x1 = (xs % bw0).astype(np.float64)[None, :]
    y = np.arange(rows, dtype=np.float64)[:, None]
    X0 = (M[0] * xb + M[1] * y) + M[2]
    Y0 = (M[3] * xb + M[4] * y) + M[5]
    W0 = (M[6] * xb + M[7] * y) + M[8]
    W = W0 + M[6] * x1
    nz = W != 0
    W = np.where(nz, INTER_TAB_SIZE / np.where(nz, W, 1.0), 0.0)

    def fixed(v):   # std::max(INT_MIN, std::min(INT_MAX, v)), then saturate_cast<int> (cvRound: half to even)
        v = np.where(v < INT_MAX, v, INT_MAX)
        v = np.where(INT_MIN < v, v, INT_MIN)
        return np.rint(v).astype(np.int64)

    X = fixed((X0 + M[0] * x1) * W)
    Y = fixed((Y0 + M[3] * x1) * W)
    sx = np.clip(X >> INTER_BITS, -32768, 32767)
    sy = np.clip(Y >> INTER_BITS, -32768, 32767)
    return sx, sy, X & (INTER_TAB_SIZE - 1), Y & (INTER_TAB_SIZE - 1)


def warp_perspective(src: np.ndarray, H) -> np.ndarray:
    """cv::warpPerspective(src, dst, H, src.size()) with the defaults of Flow.cc:78 -> rows x cols uint8."""
    src = np.asarray(src)
    if src.dtype != np.uint8 or src.ndim != 2:
        raise ValueError("src must be rows x cols uint8")
    rows, cols = src.shape
    if not (0 < rows < 32767 and 0 < cols < 32767):
        raise ValueError("remap takes sides below SHRT_MAX")
    sx, sy, tx, ty = warp_map(invert3(H), rows, cols)
    w = (np.minimum((INTER_TAB_SIZE - ty) * (INTER_TAB_SIZE - tx) * INTER_TAB_SIZE, 32767),
         (INTER_TAB_SIZE - ty) * tx * INTER_TAB_SIZE, ty * (INTER_TAB_SIZE - tx) * INTER_TAB_SIZE,
         ty * tx * INTER_TAB_SIZE)
    s = src.astype(np.int64)
    acc = np.zeros((rows, cols), np.int64)
    for k, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        yy, xx = sy + dy, sx + dx
        inside = (xx >= 0) & (xx < cols) & (yy >= 0) & (yy < rows)
        acc += np.where(inside, s[np.clip(yy, 0, rows - 1), np.clip(xx, 0, cols - 1)], 0) * w[k]
    return np.clip((acc + (1 << (COEF_BITS - 1))) >> COEF_BITS, 0, 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# findHomography(src, dst, RANSAC, 3) (perfect/src/Tracking.cc:1386 calls it with the TrackHomo pairs), up to the
# Levenberg-Marquardt refinement: OpenCV 4.13's classic RANSACPointSetRegistrator with HomographyEstimatorCallback,
# maxIters 2000, confidence 0.995.  tests/test_homography_ransac_cpu.py pins each stage cv2 exposes: the Jacobi
# eigen-decomposition (cv2.eigen), runKernel (findHomography of exactly 4 points, which returns it unrefined) and the
# RANSAC inlier set (cv2's own refit of these inliers equals cv2's RANSAC result bit for bit).  The refinement
# (LMSolver on the inliers, then the mask of the refined H) is NOT restated: ransac() returns the unrefined model.

DBL_EPS = float(np.finfo(np.float64).eps)
FLT_EPS = float(np.finfo(np.float32).eps)
DBL_MIN = float(np.finfo(np.float64).tiny)
U64 = (1 << 64) - 1


def _hypot(a: float, b: float) -> float:
    """lapack.cpp's own hypot (not libm's): the larger magnitude times sqrt(1 + ratio^2)."""
    a, b = abs(a), abs(b)
    if a > b:
        b /= a
        return a * math.sqrt(1 + b * b)
    if b > 0:
        a /= b
        return b * math.sqrt(1 + a * a)
    return 0.0


def eigen_sym(A0):
    """cv::eigen of a symmetric double matrix (JacobiImpl_): the largest off-diagonal pivot from the per-row / per-column
    maximum indices, one rotation per sweep step, eigenvalues sorted descending -> (w[n], V[n][n], rows = vectors)."""
    A = [[float(v) for v in r] for r in np.asarray(A0, np.float64)]
    n = len(A)
    V = [[1.0 if i == j else 0.0 for j in range(n)] for i in range(n)]
    W = [A[k][k] for k in range(n)]
    indR, indC = [0] * n, [0] * n

    def index(k):
        if k < n - 1:
            m, mv = k + 1, abs(A[k][k + 1])
            for i in range(k + 2, n):
                if mv < abs(A[k][i]):
                    mv, m = abs(A[k][i]), i
            indR[k] = m
        if k > 0:
            m, mv = 0, abs(A[0][k])
            for i in range(1, k):
                if mv < abs(A[i][k]):
                    mv, m = abs(A[i][k]), i
            indC[k] = m

    for k in range(n):
        index(k)
    for _ in range(n * n * 30 if n > 1 else 0):
        k, mv = 0, abs(A[0][indR[0]])
        for i in range(1, n - 1):
            if mv < abs(A[i][indR[i]]):
                mv, k = abs(A[i][indR[i]]), i
        l = indR[k]
        for i in range(1, n):
            if mv < abs(A[indC[i]][i]):
                mv, k, l = abs(A[indC[i]][i]), indC[i], i
        p = A[k][l]
        if abs(p) <= DBL_EPS:
            break
        y = (W[l] - W[k]) * 0.5
        t = abs(y) + _hypot(p, y)
        s = _hypot(p, t)
        c = t / s
        s = p / s
        t = (p / t) * p
        if y < 0:
            s, t = -s, -t
        A[k][l] = 0.0
        W[k] -= t
        W[l] += t

        def rot(a0, b0):
            return a0 * c - b0 * s, a0 * s + b0 * c
        for i in range(k):
            A[i][k], A[i][l] = rot(A[i][k], A[i][l])
        for i in range(k + 1, l):
            A[k][i], A[i][l] = rot(A[k][i], A[i][l])
        for i in range(l + 1, n):
            A[k][i], A[l][i] = rot(A[k][i], A[l][i])
        for i in range(n):
            V[k][i], V[l][i] = rot(V[k][i], V[l][i])
        index(k)
        index(l)
    for k in range(n - 1):
        m = k
        for i in range(k + 1, n):
            if W[m] < W[i]:
                m = i
        if k != m:
            W[m], W[k] = W[k], W[m]
            V[m], V[k] = V[k], V[m]
    return np.array(W), np.array(V)


def _mul3(A, B):
    C = np.zeros((3, 3))
    for i in range(3):
        for j in range(3):
            C[i, j] = (A[i, 0] * B[0, j] + A[i, 1] * B[1, j]) + A[i, 2] * B[2, j]
    return C


def run_kernel(M, m):
    """HomographyEstimatorCallback::runKernel of float32 pairs M (src) -> m (dst): centroid / mean-deviation
    normalisation in double, the 9x9 LtL (upper triangle, point by point), eigen_sym, the eigenvector of the smallest
    eigenvalue de-normalised and scaled by 1 / H22 -> 3x3 double, or None for a degenerate set."""
    M = np.asarray(M, np.float32)
    m = np.asarray(m, np.float32)
    n = len(M)
    cmx = cmy = cMx = cMy = 0.0
    for i in range(n):
        cmx += float(m[i, 0]); cmy += float(m[i, 1]); cMx += float(M[i, 0]); cMy += float(M[i, 1])
    cmx, cmy, cMx, cMy = cmx / n, cmy / n, cMx / n, cMy / n
    smx = smy = sMx = sMy = 0.0
    for i in range(n):
        smx += abs(float(m[i, 0]) - cmx); smy += abs(float(m[i, 1]) - cmy)
        sMx += abs(float(M[i, 0]) - cMx); sMy += abs(float(M[i, 1]) - cMy)
    if abs(smx) < DBL_EPS or abs(smy) < DBL_EPS or abs(sMx) < DBL_EPS or abs(sMy) < DBL_EPS:
        return None
    smx, smy, sMx, sMy = n / smx, n / smy, n / sMx, n / sMy
    inv_hnorm = np.array([[1. / smx, 0, cmx], [0, 1. / smy, cmy], [0, 0, 1]])
    hnorm2 = np.array([[sMx, 0, -cMx * sMx], [0, sMy, -cMy * sMy], [0, 0, 1]])
    L = [[0.0] * 9 for _ in range(9)]
    for i in range(n):
        x, y = (float(m[i, 0]) - cmx) * smx, (float(m[i, 1]) - cmy) * smy
        X, Y = (float(M[i, 0]) - cMx) * sMx, (float(M[i, 1]) - cMy) * sMy
        Lx = (X, Y, 1.0, 0.0, 0.0, 0.0, -x * X, -x * Y, -x)
        Ly = (0.0, 0.0, 0.0, X, Y, 1.0, -y * X, -y * Y, -y)
        for j in range(9):
            for k in range(j, 9):
                L[j][k] += Lx[j] * Lx[k] + Ly[j] * Ly[k]
    for j in range(9):
        for k in range(j):
            L[j][k] = L[k][j]
    _, V = eigen_sym(L)
    H = _mul3(_mul3(inv_hnorm, V[8].reshape(3, 3)), hnorm2)
    return H * (1.0 / H[2, 2])


class CvRNG:
    """cv::RNG (multiply-with-carry, a = 4164903690), seeded as RANSACPointSetRegistrator::run seeds it: (uint64)-1."""

    def __init__(self, state: int = U64):
        self.state = state

    def next(self) -> int:
        self.state = ((self.state & 0xffffffff) * 4164903690 + (self.state >> 32)) & U64
        return self.state & 0xffffffff

    def uniform(self, a: int, b: int) -> int:
        return a + self.next() % (b - a) if a < b else a


def _collinear(P) -> bool:
    """haveCollinearPoints: the last point against every pair of the earlier ones (and near-coincident points).  Each
    difference is taken in float, as OpenCV's Point2f subtraction does, and widened to double; the products, the sums
    and the comparison are double."""
    P = np.asarray(P, np.float32)
    i = len(P) - 1
    for j in range(i):
        dx1, dy1 = float(P[j][0] - P[i][0]), float(P[j][1] - P[i][1])
        for k in range(j):
            dx2, dy2 = float(P[k][0] - P[i][0]), float(P[k][1] - P[i][1])
            if abs(dx2 * dy1 - dy2 * dx1) <= FLT_EPS * (abs(dx1) + abs(dy1) + abs(dx2) + abs(dy2)):
                return True
    return False


def _det3(a) -> float:
    return (a[0][0] * (a[1][1] * a[2][2] - a[2][1] * a[1][2]) - a[0][1] * (a[1][0] * a[2][2] - a[2][0] * a[1][2])
            + a[0][2] * (a[1][0] * a[2][1] - a[2][0] * a[1][1]))


def check_subset(s, d) -> bool:
    """HomographyEstimatorCallback::checkSubset of 4 pairs: no collinear last point on either side, and the four
    triangle orientations agree between the two sides (all or none flipped)."""
    if _collinear(s) or _collinear(d):
        return False
    neg = 0
    for t in ((0, 1, 2), (1, 2, 3), (0, 2, 3), (0, 1, 3)):
        A = [[float(s[q][0]), float(s[q][1]), 1.0] for q in t]
        B = [[float(d[q][0]), float(d[q][1]), 1.0] for q in t]
        neg += _det3(A) * _det3(B) < 0
    return neg == 0 or neg == 4


def get_subset(src, dst, rng: CvRNG, max_attempts: int = 10000):
    """RANSACPointSetRegistrator::getSubset: 4 distinct indices drawn in turn, the whole subset redrawn while
    checkSubset rejects it -> index list, or None after max_attempts."""
    n = len(src)
    for _ in range(max_attempts):
        idx = []
        for _ in range(4):
            while True:
                v = rng.uniform(0, n)
                if v not in idx:
                    break
            idx.append(v)
        if check_subset(src[idx], dst[idx]):
            return idx
    return None


def reprojection_errors(H, M, m) -> np.ndarray:
    """HomographyEstimatorCallback::computeError: in float from the float-cast model (H22 taken as 1)."""
    Hf = np.asarray(H, np.float64).ravel().astype(np.float32)
    M = np.asarray(M, np.float32)
    m = np.asarray(m, np.float32)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        ww = np.float32(1) / (Hf[6] * M[:, 0] + Hf[7] * M[:, 1] + np.float32(1))
        dx = (Hf[0] * M[:, 0] + Hf[1] * M[:, 1] + Hf[2]) * ww - m[:, 0]
        dy = (Hf[3] * M[:, 0] + Hf[4] * M[:, 1] + Hf[5]) * ww - m[:, 1]
        return dx * dx + dy * dy


def update_num_iters(p: float, ep: float, model_points: int, max_iters: int) -> int:
    """RANSACUpdateNumIters (libm's log and pow, cvRound)."""
    p, ep = min(max(p, 0.), 1.), min(max(ep, 0.), 1.)
    num = max(1. - p, DBL_MIN)
    denom = 1. - math.pow(1. - ep, model_points)
    if denom < DBL_MIN:
        return 0
    num, denom = math.log(num), math.log(denom)
    return max_iters if (denom >= 0 or -num >= max_iters * (-denom)) else int(round(num / denom))


def ransac(src, dst, threshold: float = 3.0, confidence: float = 0.995, max_iters: int = 2000):
    """RANSACPointSetRegistrator::run with HomographyEstimatorCallback: -> (H, inliers bool[n], iterations run) of the
    best model before findHomography's refinement, or (None, None, iterations) when no model is found.  Exactly 4
    pairs: runKernel of all of them.  Fewer than 4 raises ValueError (cv2 throws)."""
    src = np.asarray(src, np.float32).reshape(-1, 2)
    dst = np.asarray(dst, np.float32).reshape(-1, 2)
    n = len(src)
    if n < 4 or len(dst) != n:
        raise ValueError("findHomography needs at least 4 pairs")
    if n == 4:
        H = run_kernel(src, dst)
        return (None, None, 0) if H is None else (H, np.ones(4, bool), 0)
    rng = CvRNG()
    t = np.float32(threshold * threshold)
    niters, best, best_mask, max_good, it = max_iters, None, None, 0, 0
    while it < niters:
        idx = get_subset(src, dst, rng)
        if idx is None:
            if it == 0:
                return None, None, 0
            break
        H = run_kernel(src[idx], dst[idx])
        if H is not None:
            mask = reprojection_errors(H, src, dst) <= t
            good = int(mask.sum())
            if good > max(max_good, 3):
                best, best_mask, max_good = H, mask, good
                niters = update_num_iters(confidence, (n - good) / n, 4, niters)
        it += 1
    return (best, best_mask, it) if max_good > 0 else (None, None, it)
