"""CPU restatement (numpy) of cv::calcOpticalFlowFarneback -- TEST INFRASTRUCTURE ONLY (tests/, tools/): never imported by
the product.  It restates OpenCV 4.13's CPU code at its baseline dispatch level (cv2.setUseOptimized(False): SSE2/SSE3,
no FMA, no IPP) for the arguments of perfect/src/Flow.cc's one call,

    calcOpticalFlowFarneback(prev, cur, flow, 0.5, 3, 15, 3, 5, 1.2, 0)

(pyr_scale 0.5, levels 3, winsize 15, iterations 3, poly_n 5, poly_sigma 1.2, no flags), plus the u8 pyrDown that makes the
half-resolution images (Flow.cc:26).  Every float and double operation follows OpenCV's order per output element; the
running sums of the box filter stay sequential.  tests/test_farneback_cpu.py pins each stage against cv2 live and through
tests/golden/farneback_*.npz.  At OpenCV's optimized dispatch (AVX2/FMA, IPP) cv2's own flow differs from this one: the
blur, resize and convert stages round differently there.

The device kernels (csrc/flow.cu) follow this file operation for operation.
"""
from __future__ import annotations

import math

import numpy as np

F32 = np.float32
F64 = np.float64

PYR_SCALE, LEVELS, WINSIZE, ITERATIONS, POLY_N, POLY_SIGMA = 0.5, 3, 15, 3, 5, 1.2
MIN_SIZE = 32          # a pyramid level is added only while both sides stay >= 32

# cv::getGaussianKernel(ksize, sigma, CV_32F) for the level blurs (sigma = (1/scale - 1)/2 at scales 1, 1/2, 1/4, 1/8).
# OpenCV computes them with its own soft-float exp; these are its float32 results, as uint32 (pinned against cv2 live).
GAUSS_KERNELS = {
    0: (3, 0.0, (0x3e800000, 0x3f000000, 0x3e800000)),
    1: (3, 0.5, (0x3dda2055, 0x3f4977eb, 0x3dda2055)),
    2: (9, 1.5, (0x3bf98261, 0x3d13c359, 0x3de06eab, 0x3e5a9135, 0x3e887a8d, 0x3e5a9135, 0x3de06eab, 0x3d13c359,
                 0x3bf98261)),
    3: (19, 3.5, (0x3b89ceeb, 0x3c09e8b2, 0x3c7e61e5, 0x3cd838ba, 0x3d2960e9, 0x3d7490c3, 0x3da2b91f, 0x3dc79039,
                  0x3de18f0c, 0x3deaf4ab, 0x3de18f0c, 0x3dc79039, 0x3da2b91f, 0x3d7490c3, 0x3d2960e9, 0x3cd838ba,
                  0x3c7e61e5, 0x3c09e8b2, 0x3b89ceeb)),
}


def level_kernel(k: int) -> np.ndarray:
    ksize, sigma, bits = GAUSS_KERNELS[k]
    return np.array(bits, np.uint32).view(np.float32)


def level_count(rows: int, cols: int) -> int:
    """The coarsest level index: levels stop below MIN_SIZE (so 320x240 has levels 2, 1, 0)."""
    scale, k = 1.0, 0
    while k < LEVELS:
        scale *= PYR_SCALE
        if cols * scale < MIN_SIZE or rows * scale < MIN_SIZE:
            break
        k += 1
    return k


def level_size(rows: int, cols: int, k: int):
    scale = 1.0
    for _ in range(k):
        scale *= PYR_SCALE
    return int(np.rint(rows * scale)), int(np.rint(cols * scale))   # cvRound: half to even


def border_reflect101(p: np.ndarray, n: int) -> np.ndarray:
    """cv::borderInterpolate(p, n, BORDER_REFLECT_101), any distance outside."""
    p = np.array(p, np.int64)
    if n == 1:
        return np.zeros_like(p)
    out = p.copy()
    bad = (out < 0) | (out >= n)
    while bad.any():
        q = out[bad]
        q = np.where(q < 0, -q, 2 * (n - 1) - q)
        out[bad] = q
        bad = (out < 0) | (out >= n)
    return out


# ---- u8 pyrDown (Flow.cc:26), 5x5 [1 4 6 4 1]^2 / 256, reflect-101 ----------------------------------------------------

def pyr_down(src: np.ndarray, rows: int, cols: int) -> np.ndarray:
    src = np.asarray(src, np.uint8)
    H, W = src.shape
    w = np.array([1, 4, 6, 4, 1], np.int64)
    xs = border_reflect101(2 * np.arange(cols)[:, None] + np.arange(5)[None, :] - 2, W)
    ys = border_reflect101(2 * np.arange(rows)[:, None] + np.arange(5)[None, :] - 2, H)
    s = src.astype(np.int64)
    rowp = (s[:, xs] * w[None, None, :]).sum(-1)              # H x cols
    colp = (rowp[ys] * w[None, :, None]).sum(1)                # rows x cols
    return ((colp + 128) >> 8).astype(np.uint8)


# ---- GaussianBlur of a float image: separable, reflect-101 --------------------------------------------------------------

def gaussian_blur(img: np.ndarray, kern: np.ndarray) -> np.ndarray:
    """sepFilter2D's float path.  ksize 3: row (l + r)*k1 + c*k0, column (u + d)*k1 + c*k0 (SymmRow/ColumnSmallFilter);
    larger: row c0*k0 + c1*k1 + ... left to right (RowFilter), column c*k[r] then += (u_i + d_i)*k[r+i] (SymmColumnFilter)."""
    img = np.asarray(img, F32)
    H, W = img.shape
    n = len(kern)
    r = n // 2
    xs = border_reflect101(np.arange(W)[None, :] + np.arange(-r, r + 1)[:, None], W)    # n x W
    ys = border_reflect101(np.arange(H)[None, :] + np.arange(-r, r + 1)[:, None], H)
    if n == 3:
        row = (img[:, xs[0]] + img[:, xs[2]]) * kern[2] + img[:, xs[1]] * kern[1]
    else:
        row = img[:, xs[0]] * kern[0]
        for i in range(1, n):
            row = row + img[:, xs[i]] * kern[i]
    if n == 3:
        return (row[ys[0]] + row[ys[2]]) * kern[2] + row[ys[1]] * kern[1]
    out = row[ys[r]] * kern[r]
    for i in range(1, r + 1):
        out = out + (row[ys[r + i]] + row[ys[r - i]]) * kern[r + i]
    return out


# ---- resize(INTER_LINEAR) of a float image ------------------------------------------------------------------------------

def _linear_tab(ssize: int, dsize: int):
    scale = 1.0 / (dsize / ssize)
    d = np.arange(dsize, dtype=F64)
    f = ((d + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(F32)).astype(F32)
    return s, f


def resize_linear(src: np.ndarray, rows: int, cols: int) -> np.ndarray:
    """cv::resize(src, Size(cols, rows), INTER_LINEAR) of a float (rows x cols [x cn]) image.  Same size: a copy.  An exact
    halving of both sides is INTER_AREA's fast path: (a00 + a01) + (a10 + a11) in groups of 4 outputs, the tail of a row
    ((a00 + a01) + a10) + a11, times 0.25.  Otherwise bilinear: float taps from (d + 0.5)*scale - 0.5, x clamped to the
    edge pixel, y taps on replicated rows; h = s0*a0 + s1*a1, out = h0*b0 + h1*b1."""
    src = np.asarray(src, F32)
    H, W = src.shape[:2]
    if (H, W) == (rows, cols):
        return src.copy()
    sx_, sy_ = 1.0 / (cols / W), 1.0 / (rows / H)
    if sx_ == 2.0 and sy_ == 2.0:
        a00 = src[0:2 * rows:2, 0:2 * cols:2]
        a01 = src[0:2 * rows:2, 1:2 * cols:2]
        a10 = src[1:2 * rows:2, 0:2 * cols:2]
        a11 = src[1:2 * rows:2, 1:2 * cols:2]
        out = ((a00 + a01) + (a10 + a11)) * F32(0.25)
        cn = 1 if src.ndim == 2 else src.shape[2]
        vec = 4 if cn == 1 else 0                         # SIMD groups of 4 outputs (single channel only)
        tail = (cols // vec) * vec if vec else 0
        out[:, tail:] = (((a00 + a01) + a10) + a11)[:, tail:] * F32(0.25)
        return out
    sx, fx = _linear_tab(W, cols)
    xmask = sx < 0
    fx[xmask] = 0
    sx[xmask] = 0
    edge = sx + 1 >= W
    fx[edge & (sx >= W - 1)] = 0
    sx[edge & (sx >= W - 1)] = W - 1
    xmax = int(np.argmax(edge)) if edge.any() else cols
    a0 = (F32(1) - fx).astype(F32)
    a1 = fx
    sy, fy = _linear_tab(H, rows)
    b0 = (F32(1) - fy).astype(F32)
    b1 = fy
    y0 = np.clip(sy, 0, H - 1)
    y1 = np.clip(sy + 1, 0, H - 1)
    ext = (slice(None),) + (None,) * (src.ndim - 2)

    def hpass(r):
        x1 = np.minimum(sx + 1, W - 1)
        h = r[:, sx] * a0[None, :][(slice(None), slice(None)) + ext[1:]] + \
            r[:, x1] * a1[None, :][(slice(None), slice(None)) + ext[1:]]
        h[:, xmax:] = r[:, sx[xmax:]]
        return h
    h0, h1 = hpass(src[y0]), hpass(src[y1])
    bb0 = b0[(slice(None), None) + ext[1:]]
    bb1 = b1[(slice(None), None) + ext[1:]]
    return h0 * bb0 + h1 * bb1


# ---- FarnebackPrepareGaussian ------------------------------------------------------------------------------------------

def cholesky_inverse(G: np.ndarray) -> np.ndarray:
    """invert(G, DECOMP_CHOLESKY): hal::Cholesky64 (L stored with reciprocal diagonal) solving L L^T X = I."""
    m = G.shape[0]
    L = np.array(G, F64)
    for i in range(m):
        for j in range(i):
            s = L[i, j]
            for k in range(j):
                s -= L[i, k] * L[j, k]
            L[i, j] = s * L[j, j]
        s = L[i, i]
        for k in range(i):
            t = L[i, k]
            s -= t * t
        L[i, i] = 1.0 / math.sqrt(s)
    b = np.eye(m, dtype=F64)
    for i in range(m):
        for j in range(m):
            s = b[i, j]
            for k in range(i):
                s -= L[i, k] * b[k, j]
            b[i, j] = s * L[i, i]
    for i in range(m - 1, -1, -1):
        for j in range(m):
            s = b[i, j]
            for k in range(m - 1, i, -1):
                s -= L[k, i] * b[k, j]
            b[i, j] = s * L[i, i]
    return b


def prepare_gaussian(n: int = POLY_N, sigma: float = POLY_SIGMA):
    """-> g, xg, xxg (float32, index x + n for x in -n..n), the 6x6 double matrix G and ig11, ig03, ig33, ig55."""
    g = np.zeros(2 * n + 1, F32)
    s = 0.0
    for x in range(-n, n + 1):
        g[x + n] = F32(math.exp(-x * x / (2 * sigma * sigma)))
        s += float(g[x + n])
    s = 1.0 / s
    xg = np.zeros_like(g)
    xxg = np.zeros_like(g)
    for x in range(-n, n + 1):
        g[x + n] = F32(float(g[x + n]) * s)
        xg[x + n] = F32(x) * g[x + n]
        xxg[x + n] = F32(x * x) * g[x + n]
    G = np.zeros((6, 6), F64)
    for y in range(-n, n + 1):
        for x in range(-n, n + 1):
            gg = g[y + n] * g[x + n]
            fx = F32(x)
            fy = F32(y)
            G[0, 0] += float(gg)
            G[1, 1] += float(gg * fx * fx)
            G[3, 3] += float(gg * fx * fx * fx * fx)
            G[5, 5] += float(gg * fx * fx * fy * fy)
    G[2, 2] = G[0, 3] = G[0, 4] = G[3, 0] = G[4, 0] = G[1, 1]
    G[4, 4] = G[3, 3]
    G[3, 4] = G[4, 3] = G[5, 5]
    iG = cholesky_inverse(G)
    return g, xg, xxg, G, iG[1, 1], iG[0, 3], iG[3, 3], iG[5, 5]


# ---- FarnebackPolyExp --------------------------------------------------------------------------------------------------

def poly_exp(src: np.ndarray, n: int = POLY_N, sigma: float = POLY_SIGMA) -> np.ndarray:
    """-> rows x cols x 5 float32: (r3, r2, r5, r4, r6) scaled by the inverse moments, replicate borders."""
    g, xg, xxg, _, ig11, ig03, ig33, ig55 = prepare_gaussian(n, sigma)
    src = np.asarray(src, F32)
    H, W = src.shape
    ys = np.arange(H)
    r0 = src * g[n]
    r1 = np.zeros_like(src)
    r2 = np.zeros_like(src)
    for k in range(1, n + 1):
        s0 = src[np.maximum(ys - k, 0)]
        s1 = src[np.minimum(ys + k, H - 1)]
        p = s0 + s1
        r0 = r0 + g[n + k] * p
        r1 = r1 + xg[n + k] * (s1 - s0)
        r2 = r2 + xxg[n + k] * p
    xs = np.arange(W)
    b1 = (r0 * g[n]).astype(F64)
    b2 = np.zeros((H, W), F64)
    b3 = (r1 * g[n]).astype(F64)
    b4 = np.zeros((H, W), F64)
    b5 = (r2 * g[n]).astype(F64)
    b6 = np.zeros((H, W), F64)
    for k in range(1, n + 1):
        xp = np.minimum(xs + k, W - 1)
        xm = np.maximum(xs - k, 0)
        tg = (r0[:, xp] + r0[:, xm]).astype(F64)
        b1 = b1 + tg * F64(g[n + k])
        b4 = b4 + tg * F64(xxg[n + k])
        b2 = b2 + ((r0[:, xp] - r0[:, xm]) * xg[n + k]).astype(F64)
        b3 = b3 + ((r1[:, xp] + r1[:, xm]) * g[n + k]).astype(F64)
        b6 = b6 + ((r1[:, xp] - r1[:, xm]) * xg[n + k]).astype(F64)
        b5 = b5 + ((r2[:, xp] + r2[:, xm]) * g[n + k]).astype(F64)
    out = np.empty((H, W, 5), F32)
    out[..., 0] = (b3 * ig11).astype(F32)
    out[..., 1] = (b2 * ig11).astype(F32)
    out[..., 2] = (b1 * ig03 + b5 * ig33).astype(F32)
    out[..., 3] = (b1 * ig03 + b4 * ig33).astype(F32)
    out[..., 4] = (b6 * ig55).astype(F32)
    return out


# ---- FarnebackUpdateMatrices -------------------------------------------------------------------------------------------

BORDER_W = np.array([0.14, 0.14, 0.4472, 0.4472, 0.4472], F32)


def update_matrices(R0: np.ndarray, R1: np.ndarray, flow: np.ndarray) -> np.ndarray:
    H, W = flow.shape[:2]
    yy, xx = np.mgrid[0:H, 0:W]
    dx = flow[..., 0]
    dy = flow[..., 1]
    fx = xx.astype(F32) + dx
    fy = yy.astype(F32) + dy
    x1 = np.floor(fx).astype(np.int64)
    y1 = np.floor(fy).astype(np.int64)
    fx = fx - x1.astype(F32)
    fy = fy - y1.astype(F32)
    inside = (x1 >= 0) & (x1 < W - 1) & (y1 >= 0) & (y1 < H - 1)
    xi = np.clip(x1, 0, W - 2)
    yi = np.clip(y1, 0, H - 2)
    one = F32(1)
    a00 = (one - fx) * (one - fy)
    a01 = fx * (one - fy)
    a10 = (one - fx) * fy
    a11 = fx * fy
    p00, p01, p10, p11 = R1[yi, xi], R1[yi, xi + 1], R1[yi + 1, xi], R1[yi + 1, xi + 1]
    r = [((a00 * p00[..., c] + a01 * p01[..., c]) + a10 * p10[..., c]) + a11 * p11[..., c] for c in range(5)]
    r2, r3, r4, r5, r6 = r
    r4 = np.where(inside, (R0[..., 2] + r4) * F32(0.5), R0[..., 2])
    r5 = np.where(inside, (R0[..., 3] + r5) * F32(0.5), R0[..., 3])
    r6 = np.where(inside, (R0[..., 4] + r6) * F32(0.25), R0[..., 4] * F32(0.5))
    r2 = np.where(inside, r2, F32(0))
    r3 = np.where(inside, r3, F32(0))
    r2 = (R0[..., 0] - r2) * F32(0.5)
    r3 = (R0[..., 1] - r3) * F32(0.5)
    r2 = r2 + (r4 * dy + r6 * dx)                  # r2 += r4*dy + r6*dx
    r3 = r3 + (r6 * dy + r5 * dx)
    B = 5                                          # sizes >= 2*B: every pixel has at most one left/right, top/bottom factor
    bx = np.ones(W, F32)
    by = np.ones(H, F32)
    lo, hi = BORDER_W, BORDER_W[::-1]
    sl, sr, st, sb = bx.copy(), bx.copy(), by.copy(), by.copy()
    sl[:B], sr[W - B:], st[:B], sb[H - B:] = lo, hi, lo, hi
    scale = ((sl[None, :] * sr[None, :]) * st[:, None]) * sb[:, None]
    edge = (xx < B) | (xx >= W - B) | (yy < B) | (yy >= H - B)
    r2, r3, r4, r5, r6 = (np.where(edge, v * scale, v) for v in (r2, r3, r4, r5, r6))
    M = np.empty((H, W, 5), F32)
    M[..., 0] = r4 * r4 + r6 * r6
    M[..., 1] = (r4 + r5) * r6
    M[..., 2] = r5 * r5 + r6 * r6
    M[..., 3] = r4 * r2 + r6 * r3
    M[..., 4] = r6 * r2 + r5 * r3
    return M


# ---- FarnebackUpdateFlow_Blur ------------------------------------------------------------------------------------------

def vertical_sums(M: np.ndarray, winsize: int = WINSIZE) -> np.ndarray:
    """-> H x W x 5 double: the box filter's running column sums as they stand at each row (sequential in y)."""
    H, W = M.shape[:2]
    m = winsize // 2
    Mf = M.reshape(H, W * 5)
    vs = (Mf[0] * F32(m + 2)).astype(F64)
    for y in range(1, m):
        vs = vs + Mf[min(y, H - 1)].astype(F64)
    out = np.empty((H, W * 5), F64)
    for y in range(H):
        vs = vs + (Mf[min(y + m, H - 1)] - Mf[max(y - m - 1, 0)]).astype(F64)
        out[y] = vs
    return out.reshape(H, W, 5)


def horizontal_solve(V: np.ndarray, winsize: int = WINSIZE, counts: dict | None = None) -> np.ndarray:
    """Running row sums over the column sums (replicated borders, sequential in x) and the 2x2 solve per pixel.
    `counts` (a dict) accumulates how many solves had det = g11*g22 - g12^2 below 1e-3 with h != 0 ("det_small") and
    exactly 0 ("det_zero")."""
    H, W = V.shape[:2]
    m = winsize // 2
    scale = 1.0 / (winsize * winsize)
    xs = np.clip(np.arange(-m - 1, W + m + 1), 0, W - 1)
    Vp = V[:, xs]                                  # index x + m + 1
    acc = Vp[:, m + 1] * F64(m + 2)
    for x in range(1, m):
        acc = acc + Vp[:, x + m + 1]
    flow = np.empty((H, W, 2), F32)
    for x in range(W):
        acc = acc + (Vp[:, x + 2 * m + 1] - Vp[:, x])
        g11, g12, g22, h1, h2 = (acc[:, c] * scale for c in range(5))
        if counts is not None:
            det = g11 * g22 - g12 * g12
            counts["det_small"] = counts.get("det_small", 0) + int(((det < 1e-3) & ((h1 != 0) | (h2 != 0))).sum())
            counts["det_zero"] = counts.get("det_zero", 0) + int((det == 0).sum())
        idet = 1.0 / (g11 * g22 - g12 * g12 + 1e-3)
        flow[:, x, 0] = ((g11 * h2 - g12 * h1) * idet).astype(F32)
        flow[:, x, 1] = ((g22 * h1 - g12 * h2) * idet).astype(F32)
    return flow


# ---- the whole call ----------------------------------------------------------------------------------------------------

def farneback(prev: np.ndarray, cur: np.ndarray, levels: int = LEVELS, iterations: int = ITERATIONS,
              trace: dict | None = None) -> np.ndarray:
    """calcOpticalFlowFarneback(prev, cur, None, 0.5, levels, 15, iterations, 5, 1.2, 0) of two u8 images -> rows x cols x 2
    float32.  `levels` / `iterations` other than 3 exist for stage-by-stage comparison with cv2; `trace` (a dict) receives
    each level's blurred/resized images, polynomial expansions and flows."""
    prev = np.asarray(prev, np.uint8)
    cur = np.asarray(cur, np.uint8)
    H, W = prev.shape
    scale, k = 1.0, 0
    while k < levels:
        scale *= PYR_SCALE
        if W * scale < MIN_SIZE or H * scale < MIN_SIZE:
            break
        k += 1
    top = k
    prev_flow = None
    flow = None
    for k in range(top, -1, -1):
        h, w = level_size(H, W, k)
        if prev_flow is None:
            flow = np.zeros((h, w, 2), F32)
        else:
            flow = resize_linear(prev_flow, h, w) * F32(1.0 / PYR_SCALE) + F32(0)
        kern = level_kernel(k)
        R = []
        for img in (prev, cur):
            I = resize_linear(gaussian_blur(img.astype(F32), kern), h, w)
            R.append(poly_exp(I))
            if trace is not None:
                trace.setdefault("I", []).append(I)
        if trace is not None:
            trace.setdefault("R", []).extend(R)
            trace.setdefault("flow_in", []).append(flow.copy())
        M = update_matrices(R[0], R[1], flow)
        for i in range(iterations):
            flow = horizontal_solve(vertical_sums(M))
            if i < iterations - 1:
                M = update_matrices(R[0], R[1], flow)
        prev_flow = flow
    return flow
