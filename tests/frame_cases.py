"""Deterministic crafted cases for the per-point / per-keypoint Frame members that run on the device: isInFrustum +
PredictScale (orbm_is_in_frustum), UndistortKeyPoints (orbm_undistort_keypoints), ComputeStereoFromRGBD +
UnprojectStereo (k_frame_glue, behind track_batch / track_batch_u16) and ComputeBoW (orbv_transform + the map
assembly of vocabulary.py).  Each case is named after the one edge it makes observable.

isInFrustum: identity or axis-permuted Tcw with integer translation, so PcX / PcY / PcZ are exact and the camera centre
is exact.  A point at Pc = (0, 0, z) has dist == z and, with normal (nx, 0, c), viewCos == c exactly, so the distance and
angle gates are hit by placing z or c on the gate float and its two neighbours.  PredictScale: ratio = mfMaxDistance /
dist with dist == 1 is mfMaxDistance itself, placed on each threshold float of predict_scale_thresholds (found here by
bisection with libm's logf, the function the reference and the host calls) and on its two neighbours.

Every case carries `edges`: claims about its own inputs that tests/test_frame_edges_cpu.py recomputes in numpy (with
libm's logf through ctypes), so a case that stops containing its edge fails instead of silently testing nothing."""
import ctypes as C
import ctypes.util
import math

import numpy as np

from orb_slam2_ssd_semantic_b200._abi import FrameView

f32 = np.float32
FX = FY = 512.0
CX, CY = 320.0, 240.0
BF = 40.0
MAX_LEVELS = 16            # common.cuh
INF = float("inf")

_libm = C.CDLL(ctypes.util.find_library("m"))
_libm.logf.restype = C.c_float
_libm.logf.argtypes = [C.c_float]


def logf(x):
    """libm's logf: what std::log(float) is in MapPoint::PredictScale and in predict_scale_thresholds (numpy's float32
    log has its own SIMD implementation and may differ in the last bit)."""
    return f32(_libm.logf(float(x)))


def up(x):
    return f32(np.nextafter(f32(x), f32(INF)))


def down(x):
    return f32(np.nextafter(f32(x), f32(-INF)))


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


class Case:
    def __init__(self, name, kind, kw, edges):
        self.name, self.kind, self.kw, self.edges = name, kind, kw, edges

    def __repr__(self):
        return "Case(%s)" % self.name


# ---------------------------------------------------------------------------------------------------------------------
# isInFrustum + PredictScale
# ---------------------------------------------------------------------------------------------------------------------
def predict_level(ratio, lsf, nlevels):
    """MapPoint::PredictScale (src/MapPoint.cc:463-478) with libm's logf: ceil(logf(ratio) / lsf), float division,
    clamped to [0, nlevels - 1]."""
    q = f32(logf(ratio) / f32(lsf))
    n = math.ceil(float(q))
    return 0 if n < 0 else min(n, nlevels - 1)


def thresholds(lsf, nlevels):
    """t_k = the largest positive float whose unclamped level is <= k, k = 0 .. nlevels - 2 (bisection over the bit
    patterns of the positive finite floats)."""
    def level(b):
        return math.ceil(float(f32(logf(np.uint32(b).view(np.float32)) / f32(lsf))))
    out = []
    for k in range(nlevels - 1):
        lo, hi = 1, 0x7f7fffff
        assert level(lo) <= k < level(hi)
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if level(mid) <= k:
                lo = mid
            else:
                hi = mid
        out.append(np.uint32(lo).view(np.float32))
    return out


def frustum_mirror(case):
    """The device's / oracle's float arithmetic of Frame::isInFrustum, per point (numpy float32 / float64 scalars)."""
    kw = case.kw
    F, P, N = kw["F"], kw["xw"].astype(f32), kw["normal"].astype(f32)
    T = F.Tcw.astype(f32)
    fx, fy, cx, cy, bf = (f32(v) for v in F.cam)
    out = {k: [] for k in ("PcX", "PcY", "PcZ", "u", "v", "minD", "maxD", "dist", "viewCos", "ratio")}

    def gemm3(a, b, c):
        t = f32(f32(f32(a[0] * b[0]) + f32(a[1] * b[1])) + f32(a[2] * b[2]))
        return f32(np.float64(t) + np.float64(c))
    Ow = [-f32(f32(f32(T[a] * T[3]) + f32(T[4 + a] * T[7])) + f32(T[8 + a] * T[11])) for a in range(3)]
    with np.errstate(all="ignore"):
        for i in range(len(P)):
            p = P[i]
            pc = [gemm3(T[4 * r:4 * r + 3], p, T[4 * r + 3]) for r in range(3)]
            invz = f32(f32(1.0) / pc[2])
            u = f32(f32(f32(fx * pc[0]) * invz) + cx)
            v = f32(f32(f32(fy * pc[1]) * invz) + cy)
            po = [f32(p[a] - Ow[a]) for a in range(3)]
            n2 = dot = np.float64(0)
            for a in range(3):
                n2 = n2 + np.float64(po[a]) * np.float64(po[a])
                dot = dot + np.float64(po[a]) * np.float64(N[i, a])
            dist = f32(np.sqrt(n2))
            for k, val in zip(out, (pc[0], pc[1], pc[2], u, v, f32(f32(0.8) * f32(kw["mind"][i])),
                                    f32(f32(1.2) * f32(kw["maxd"][i])), dist, f32(dot / np.float64(dist)),
                                    f32(f32(kw["maxd"][i]) / dist))):
                out[k].append(val)
    return {k: np.array(v, f32) for k, v in out.items()}


def _frame(T, bounds, nlevels=8, sf=1.2):
    z = np.zeros(1, f32)
    scale = np.cumprod(np.concatenate([[f32(1.0)], np.full(nlevels - 1, f32(sf), f32)])).astype(f32)
    return FrameView(z, z, np.zeros(1, np.int32), z, z, np.zeros((1, 32), np.uint8), T, FX, FY, CX, CY, BF, *bounds,
                     scale)


def _pose(perm=(0, 1, 2), t=(1.0, -2.0, 3.0)):
    """Tcw with an axis permutation for rotation (row r picks world axis perm[r]) and an integer translation."""
    T = np.zeros((4, 4), f32)
    for r, c in enumerate(perm):
        T[r, c] = 1.0
    T[:3, 3] = np.array(t, f32)
    T[3, 3] = 1.0
    return T


def _world(T, pc):
    """World points for camera points pc under an axis-permuted T (exact: Pw = R^T (pc - t))."""
    R, t = T[:3, :3].astype(np.float64), T[:3, 3].astype(np.float64)
    return ((np.asarray(pc, np.float64) - t) @ R).astype(f32)


def _fcase(name, T, bounds, pc=None, xw=None, normal=None, mind=None, maxd=None, cos_limit=0.5, sf=1.2, nlevels=8,
           undefined=None, edges=()):
    xw = _world(T, pc) if xw is None else np.asarray(xw, f32)
    n = len(xw)
    if normal is None:   # unit vectors along PO: viewCos ~ 1
        po = xw.astype(np.float64) + T[:3, 3].astype(np.float64) @ T[:3, :3].astype(np.float64)
        nrm = np.linalg.norm(po, axis=1)
        normal = np.where(nrm[:, None] > 0, po / np.maximum(nrm, 1e-30)[:, None], [0.0, 0.0, 1.0])
    kw = dict(F=_frame(T, bounds, nlevels, sf), xw=xw, normal=np.asarray(normal, f32).reshape(n, 3),
              mind=np.asarray(mind if mind is not None else np.full(n, 1.0), f32),
              maxd=np.asarray(maxd if maxd is not None else np.full(n, 4.0), f32),
              cos_limit=f32(cos_limit), lsf=float(logf(sf)), nlevels=nlevels,
              undefined=np.zeros(n, bool) if undefined is None else np.asarray(undefined, bool))
    return Case(name, "frustum", kw, list(edges))


def frustum_cases():
    cases = []
    everywhere = (-INF, INF, -INF, INF)
    # PcZ on the `PcZ < 0` gate: +0.0 and -0.0 pass (u = +-inf with unbounded limits), the subnormals on either side,
    # and Pc = (0, 0, +0.0), whose u, v, viewCos are NaN and pass every gate as NaN.  That last point's dist is 0, so its
    # ratio is inf: the reference takes (int)ceil(inf) there, which is undefined, so its level is not compared.
    T = _pose(t=(0.0, 0.0, -0.0))
    xw = np.array([[1, 1, 0.0], [-1, -1, -0.0], [1, 1, 1e-45], [1, 1, -1e-45], [0, 0, 0.0], [1, 1, 2]], f32)
    cases.append(_fcase("frustum/pcz_signed_zero_and_subnormal", T, everywhere, xw=xw,
                        normal=np.tile([0.0, 0.0, 1.0], (6, 1)), mind=[1, 1, 1, 1, 0, 1], maxd=[4, 4, 4, 4, 4, 4],
                        cos_limit=-1.0, undefined=[0, 0, 0, 0, 1, 0],
                        edges=[("eq", "PcZ", 0, f32(0.0)), ("eq", "PcZ", 1, f32(-0.0)), ("eq", "PcZ", 2, f32(1e-45)),
                               ("eq", "PcZ", 3, f32(-1e-45)), ("eq", "PcZ", 4, f32(0.0)), ("nan", "u", 4),
                               ("nan", "v", 4), ("nan", "viewCos", 4), ("eq", "dist", 4, f32(0.0)),
                               ("eq", "u", 0, f32(INF)), ("eq", "u", 1, f32(INF))]))
    # u / v on the inclusive image bounds: u in {64, 576}, v in {112, 368}, under an axis-permuted rotation
    T = _pose(perm=(1, 2, 0))
    pc = [[1, 0, 2], [-1, 0, 2], [0, 0.5, 2], [0, -0.5, 2]]
    for tag, lo, hi in (("on", lambda x: f32(x), lambda x: f32(x)), ("inside", down, up), ("outside", up, down)):
        bounds = (lo(64), hi(576), lo(112), hi(368))
        cases.append(_fcase("frustum/uv_bounds_" + tag, T, bounds, pc=pc,
                            edges=[("eq", "u", 0, f32(576)), ("eq", "u", 1, f32(64)), ("eq", "v", 2, f32(368)),
                                   ("eq", "v", 3, f32(112)), ("bounds", tag)]))
    # the 0.8f / 1.2f distance gates at equality: Pc = (0, 0, z) has dist == z exactly
    T = _pose()
    g_lo = f32(f32(0.8) * f32(2.5))
    g_hi = f32(f32(1.2) * f32(5.0))
    zs = [down(g_lo), g_lo, up(g_lo), down(g_hi), g_hi, up(g_hi)]
    cases.append(_fcase("frustum/distance_gates_at_equality", T, (0, 640, 0, 480), pc=[[0, 0, z] for z in zs],
                        normal=np.tile([0.0, 0.0, 1.0], (6, 1)), mind=np.full(6, 2.5), maxd=np.full(6, 5.0),
                        edges=[("eq", "dist", i, zs[i]) for i in range(6)] +
                              [("eq", "minD", 0, up(zs[0])), ("eq", "minD", 1, zs[1]), ("eq", "minD", 2, down(zs[2])),
                               ("eq", "maxD", 3, up(zs[3])), ("eq", "maxD", 4, zs[4]), ("eq", "maxD", 5, down(zs[5]))]))
    # viewCos < cos_limit at exactly 0.5 and one float either side
    cs = [down(0.5), f32(0.5), up(0.5)]
    nrm = [[math.sqrt(1 - float(c) ** 2), 0.0, float(c)] for c in cs]
    cases.append(_fcase("frustum/view_cos_at_limit", T, (0, 640, 0, 480), pc=[[0, 0, 2]] * 3,
                        normal=np.array(nrm, f32) * np.array([1, 1, 0], f32) + np.array([[0, 0, c] for c in cs], f32),
                        edges=[("eq", "viewCos", i, cs[i]) for i in range(3)]))
    cases.extend(predict_cases())
    return cases


def predict_cases():
    """ratio on every threshold float of predict_scale_thresholds and its two neighbours, a ratio below 1 and one past
    the top level, for scale factors 1.2 / 1.5 / 2.0 at nlevels 1, 8 and MAX_LEVELS."""
    T = _pose()
    out = []
    for sf in (1.2, 1.5, 2.0):
        for nl in (1, 8, MAX_LEVELS):
            lsf = logf(sf)
            thr = thresholds(lsf, nl)
            top = thr[-1] if thr else f32(1.0)
            ratios = [f32(0.9), f32(1.0)] if not thr else [f32(0.9)]
            for t in thr:
                ratios += [down(t), t, up(t)]
            ratios += [up(top), f32(top * 8)]
            n = len(ratios)
            edges = [("eq", "ratio", i, r) for i, r in enumerate(ratios)]
            edges += [("threshold", k, t) for k, t in enumerate(thr)]
            edges += [("level", i, predict_level(r, lsf, nl)) for i, r in enumerate(ratios)]
            out.append(_fcase("predict/sf%.1f/nl%d" % (sf, nl), T, (0, 640, 0, 480), pc=[[0, 0, 1]] * n,
                              normal=np.tile([0.0, 0.0, 1.0], (n, 1)), mind=np.full(n, 1.0), maxd=ratios, sf=sf,
                              nlevels=nl, edges=edges))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# UndistortKeyPoints
# ---------------------------------------------------------------------------------------------------------------------
UNDIST_K = np.array([500.0, 0, 320.0, 0, 520.0, 240.0, 0, 0, 1], f32)   # fx != fy


def undistort_points():
    """The principal point, the image corners and centre lines, and points far outside the image."""
    pts = [[320, 240], [0, 0], [639, 479], [0, 479], [639, 0], [320, 0], [0, 240], [319.5, 240.25], [320, 240.5],
           [-2000, 240], [2400, -1800], [5000, 6000], [-40000, 30000], [321, 241]]
    g = np.stack(np.meshgrid(np.linspace(-300, 940, 9), np.linspace(-200, 680, 7)), -1).reshape(-1, 2)
    return np.concatenate([np.array(pts, f32), g.astype(f32)])


def undistort_cases():
    """(name, dist coefficients) -- ndist is len(dist)."""
    return [
        ("undistort/k1_zero_copies_despite_k2_p1_p2", np.array([0.0, 0.3, 0.01, -0.02], f32)),
        ("undistort/k1_negative_zero_copies_ndist5", np.array([-0.0, 0.2, 0.001, 0.002, 0.5], f32)),
        ("undistort/ndist0_copies", np.zeros(0, f32)),
        ("undistort/k1_negative_zero_copies_ndist4", np.array([-0.0, -0.3, 0.002, -0.001], f32)),
        ("undistort/ndist4", np.array([-0.28, 0.07, 0.0002, 0.0001], f32)),
        ("undistort/ndist5", np.array([0.26, -0.95, -0.005, 0.003, 1.16], f32)),
        ("undistort/ndist5_k3_icdist_negative", np.array([0.05, 0.0, 0.0, 0.0, -0.4], f32)),
        ("undistort/icdist_negative", np.array([-0.9, 0.0, 0.001, 0.001], f32)),
        ("undistort/icdist_negative_k3", np.array([0.1, 0.0, 0.0, 0.0, -0.5], f32)),
    ]


def undistort_icdist(xy, K, dist):
    """Per point: whether some iteration of the fixed-point loop meets icdist < 0 (the early exit)."""
    k = np.zeros(5)
    k[:len(dist)] = dist
    fx, fy, cx, cy = (float(K[i]) for i in (0, 4, 2, 5))
    out = []
    for u, v in np.asarray(xy, np.float64):
        x0, y0 = (u - cx) * (1 / fx), (v - cy) * (1 / fy)
        x, y, hit = x0, y0, False
        for _ in range(5):
            r2 = x * x + y * y
            ic = 1 / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
            if ic < 0:
                hit = True
                break
            dx = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x)
            dy = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y
            x, y = (x0 - dx) * ic, (y0 - dy) * ic
        out.append(hit)
    return np.array(out)


# ---------------------------------------------------------------------------------------------------------------------
# ComputeStereoFromRGBD + UnprojectStereo (k_frame_glue)
# ---------------------------------------------------------------------------------------------------------------------
GLUE_T = _pose(perm=(0, 2, 1), t=(1.0, 2.0, -1.0))
# depths the `d > 0` gate must sort: 0, -0, negative, NaN, +inf, subnormal (bf / d overflows uright), tiny normal
GLUE_EDGE = np.array([0.0, -0.0, -1.5, np.nan, np.inf, 1e-45, 1e-39, 1e-38, 2e-38, 3.0], f32)


def glue_depth(rows, cols, kps):
    """A float depth image with a distinct value at every pixel (so a keypoint read from the neighbouring pixel is seen)
    and the edge depths of GLUE_EDGE at every third keypoint's pixel (imDepth.at<float>(v, u): truncation)."""
    d = (f32(0.5) + np.arange(rows * cols, dtype=np.float64).reshape(rows, cols) * 2.0 ** -16).astype(f32)
    for j, i in enumerate(range(0, len(kps), 3)):
        d[int(kps["y"][i]), int(kps["x"][i])] = GLUE_EDGE[j % len(GLUE_EDGE)]
    return d


def glue_depth_u16(rows, cols, kps):
    """A CV_16U sensor image with distinct values (mod 65536) and 0 / 65535 at every fourth keypoint's pixel."""
    d = ((np.arange(rows * cols, dtype=np.int64).reshape(rows, cols) * 7 + 1) % 65536).astype(np.uint16)
    for j, i in enumerate(range(0, len(kps), 4)):
        d[int(kps["y"][i]), int(kps["x"][i])] = (0, 65535)[j % 2]
    return d


DEPTH_FACTOR = f32(1.0 / 5000.0)


# ---------------------------------------------------------------------------------------------------------------------
# ComputeBoW: hand-built vocabulary trees
# ---------------------------------------------------------------------------------------------------------------------
def flip(d, k, salt):
    """d with exactly k of its 256 bits flipped."""
    out = np.array(d, np.uint8).copy()
    for b in np.random.default_rng(salt).permutation(256)[:k]:
        out[b >> 3] ^= np.uint8(1 << (b & 7))
    return out


def hamming(a, b):
    return int(np.unpackbits(np.bitwise_xor(np.asarray(a, np.uint8), np.asarray(b, np.uint8))).sum())


class Tree:
    """A vocabulary in DBoW2's node-id order (node 0 = root, parent[i] < i, siblings in ascending id)."""

    def __init__(self, k, L):
        self.k, self.L = k, L
        self.parent, self.desc, self.weight = [0], [np.zeros(32, np.uint8)], [0.0]

    def add(self, p, d, w=0.0):
        self.parent.append(p)
        self.desc.append(np.asarray(d, np.uint8))
        self.weight.append(float(w))
        return len(self.parent) - 1

    def arrays(self):
        return np.array(self.parent, np.int32), np.stack(self.desc).astype(np.uint8), np.array(self.weight, np.float64)

    def children(self, i):
        return [j for j in range(1, len(self.parent)) if self.parent[j] == i]


def descend(parent, node_desc, weight, word_id, desc, L, levelsup, trace=None):
    """DBoW2 TemplatedVocabulary::transform for one descriptor (the first child at minimal distance, strict <) ->
    (word id, weight, node id levelsup levels above the leaves; 0 where the walk never reaches that level).
    trace, if a list, receives (node, distances to each of its children) for every node the walk leaves."""
    ch = [[] for _ in range(len(parent))]
    for i in range(1, len(parent)):
        ch[parent[i]].append(i)
    cur, lvl, nid = 0, 0, 0
    while ch[cur]:
        lvl += 1
        dists = [hamming(desc, node_desc[c]) for c in ch[cur]]
        best, bd = ch[cur][0], dists[0]
        for c, d in zip(ch[cur][1:], dists[1:]):
            if d < bd:
                best, bd = c, d
        if trace is not None:
            trace.append((cur, dists))
        cur = best
        if lvl == L - levelsup:
            nid = cur
    return int(word_id[cur]), float(weight[cur]), nid


def leaf_word_ids(parent):
    """createWords' numbering: leaves in ascending node id."""
    n = len(parent)
    has = np.zeros(n, bool)
    has[np.asarray(parent[1:])] = True
    wid = np.full(n, -1, np.int64)
    leaves = [i for i in range(1, n) if not has[i]]
    wid[leaves] = np.arange(len(leaves))
    return wid


def _rand(rng):
    return rng.integers(0, 256, 32, dtype=np.uint8)


def _wide(k, seed):
    """Root with k children (k = 33 / 40 take a second 32-lane round), each with k or fewer leaf children; duplicate
    sibling descriptors in both lane rounds; stopped leaves.  -> (tree, indices of the two identical root children)."""
    rng = np.random.default_rng(seed)
    t = Tree(k, 2)
    mids = [t.add(0, _rand(rng)) for _ in range(k)]
    dup = (5, 37 if k > 37 else k - 1)                   # identical siblings across the two lane rounds
    t.desc[mids[dup[1]]] = t.desc[mids[dup[0]]].copy()
    for j, m in enumerate(mids):
        nc = k if j % 3 == 0 else 1 + (j * 7) % k        # fewer children on most nodes
        for c in range(nc):
            w = 0.0 if (c % 11 == 4) else 0.25 + 0.125 * ((c * 5 + j) % 13)
            t.add(m, flip(t.desc[m], 30 + (c % 20), seed * 1000 + j * 64 + c), w)
    return t, dup


def _uneven(k, seed, L=6):
    """Leaves at every depth 1 .. L (a chain of k-ary nodes where one child per level continues)."""
    rng = np.random.default_rng(seed)
    t = Tree(k, L)
    frontier = [0]
    for lvl in range(1, L + 1):
        nxt = []
        for p in frontier:
            for c in range(k):
                w = 0.0 if (lvl + c) % 7 == 3 else 0.5 + 0.25 * ((lvl * 3 + c) % 9)
                i = t.add(p, flip(t.desc[p], 40 // lvl + 6, seed * 977 + len(t.parent)) if p else _rand(rng), w)
                if lvl < L and (c == 0 or (lvl == 2 and c == 1 and k > 2)):
                    t.weight[i] = 0.0
                    nxt.append(i)
        frontier = nxt
    return t


def _ties(seed):
    """k = 10, L = 3: every node's children include a pair of identical descriptors, except those of root child 1, which
    all carry the complement of root child 1's descriptor (a query equal to root child 1 goes there and then meets
    distance 256 at every child; those children are live leaves with distinct weights, so which one the tie picks shows
    in the word).  Root children 4 .. 9 are leaves with weight 0 (stopped words)."""
    rng = np.random.default_rng(seed)
    t = Tree(10, 3)
    frontier = [0]
    for lvl in range(1, 4):
        nxt = []
        for pi, p in enumerate(frontier[:4]):
            base = [_rand(rng) if p == 0 else flip(t.desc[p], 20, seed * 31 + len(t.parent) + c) for c in range(10)]
            base[7] = base[2].copy()
            if lvl == 2 and pi == 1:
                base = [~t.desc[p] for _ in range(10)]
            for c in range(10):
                w = 0.0 if lvl < 3 else (0.0 if c == 4 else 1.0 + 0.5 * c)
                if lvl == 2 and pi == 1:   # leaves (only the first four level-2 nodes get children), all live
                    w = 1.0 + 0.25 * c
                i = t.add(p, base[c], w)
                if lvl < 3:
                    nxt.append(i)
        frontier = nxt
    return t


def _descs_for(t, seed, n):
    """Descriptors at chosen Hamming distances from chosen nodes: copies of leaves and of inner nodes, a few bits off,
    complements, many copies of one live leaf (one word hit by many features), random ones.  Copies are taken only of
    the live leaves that a copy's walk actually reaches."""
    rng = np.random.default_rng(seed)
    parent, nd, w = t.arrays()
    leaves = np.nonzero(leaf_word_ids(parent) >= 0)[0]
    ids = np.arange(len(parent))
    live = [x for x in leaves if w[x] > 0 and descend(parent, nd, w, ids, nd[x], t.L, 4)[0] == x]   # reached by a copy
    out = []
    for j in range(n):
        r = j % 6
        if r == 0:
            out.append(nd[live[(j * 7) % len(live)]].copy())
        elif r == 1:
            out.append(flip(nd[leaves[(j * 13) % len(leaves)]], 1 + j % 9, seed + j))
        elif r == 2:
            out.append(nd[1 + (j * 5) % (len(parent) - 1)].copy())
        elif r == 3:
            out.append(~nd[1 + (j * 3) % (len(parent) - 1)])
        elif r == 4:
            out.append(nd[live[0]].copy())
        else:
            out.append(_rand(rng))
    return np.stack(out).astype(np.uint8)


def bow_cases():
    """Case(kw: parent, node_desc, weight, word_id (None = ascending), desc, levelsup list)."""
    out = []

    def case(name, t, desc, levelsups, word_id=None, edges=()):
        p, nd, w = t.arrays()
        out.append(Case(name, "bow", dict(k=t.k, L=t.L, parent=p, node_desc=nd, weight=w, word_id=word_id, desc=desc,
                                          levelsups=levelsups, tree=t), list(edges)))

    for k in (33, 40):
        t, dup = _wide(k, k)
        nd = t.arrays()[1]
        mids = t.children(0)
        d = _descs_for(t, k, 8 * 37 + 5)
        # a query equal to a second-round child (c >= 32) and one equal to the duplicated pair
        d[0] = nd[mids[k - 1]]
        d[1] = nd[mids[dup[0]]]
        picks = [("picks", 0, 1, mids[k - 1])] if k - 1 != dup[1] else []   # k = 33: its one second-round child is tied
        case("bow/k%d_second_lane_round_and_cross_round_tie" % k, t, d, [0, 1, 2, 4],
             edges=picks + [("nchildren", 0, k), ("fewer", True),
                    ("tie", 1, 1, (mids[dup[0]], mids[dup[1]])), ("stopped", True), ("n_mod8", True)])
    t = _uneven(2, 7)
    case("bow/k2_uneven_depth_levelsup_0_to_L", t, _descs_for(t, 7, 301), [0, 1, 3, 4, 5, 6, 9],
         edges=[("depths", 1, 6), ("stopped", True), ("n_mod8", True)])
    t = _uneven(3, 8, L=6)
    case("bow/k3_uneven_depth_shallow_leaf_above_nid_level", t, _descs_for(t, 8, 203), [1, 4],
         edges=[("depths", 1, 6), ("shallow_hit", 4)])
    t = _ties(9)
    nd = t.arrays()[1]
    d = _descs_for(t, 9, 8 * 40 + 3)
    l1 = t.children(0)
    d[2] = nd[l1[2]]
    case("bow/k10_sibling_ties_first_child_wins", t, d, [4, 1, 0],
         edges=[("tie", 2, 1, (l1[2], l1[7])), ("stopped", True), ("same_word", 40)])
    # root child 1's children all carry its complement: a query equal to root child 1 walks there, then meets 256 ten times
    d2 = d.copy()
    d2[3] = nd[l1[1]]
    case("bow/k10_distance_256_to_every_child", t, d2, [4], edges=[("d256", 3, l1[1]), ("live", 3)])
    # caller-given word ids, not ascending
    t = _wide(33, 5)[0]
    p = t.arrays()[0]
    leaves = np.nonzero(leaf_word_ids(p) >= 0)[0]
    perm = np.random.default_rng(5).permutation(len(leaves))
    wid = np.full(len(p), -1, np.int32)
    wid[leaves] = perm * 3 + 7
    case("bow/k33_permuted_word_ids", t, _descs_for(t, 5, 129), [4, 1], word_id=wid,
         edges=[("permuted", True)])
    # n = 1 and n = 7: a partial last warp group of 8
    t = _ties(10)
    dd = _descs_for(t, 10, 8)
    case("bow/k10_one_feature", t, dd[:1], [4], edges=[("live", 0)])
    case("bow/k10_seven_features", t, dd[:7], [4], edges=[("live", 0)])
    return out


def bow_expected_raw(case, levelsup):
    """(word, weight, node) per feature through `descend`."""
    kw = case.kw
    wid = kw["word_id"] if kw["word_id"] is not None else leaf_word_ids(kw["parent"])
    r = [descend(kw["parent"], kw["node_desc"], kw["weight"], wid, d, kw["L"], levelsup) for d in kw["desc"]]
    return (np.array([a for a, _, _ in r], np.uint32), np.array([b for _, b, _ in r], np.float64),
            np.array([c for _, _, c in r], np.uint32))


def assemble(word, weight, node):
    """TemplatedVocabulary::transform's maps from the per-feature results: BowVector::addWeight in feature order,
    FeatureVector::addFeature, stopped words (weight 0) left out of both, L1 normalisation in word order."""
    bow, fv = {}, {}
    for i in range(len(word)):
        if not weight[i] > 0:
            continue
        bow[int(word[i])] = bow.get(int(word[i]), 0.0) + float(weight[i])
        fv.setdefault(int(node[i]), []).append(i)
    norm = 0.0
    for k in sorted(bow):
        norm += abs(bow[k])
    if norm > 0:
        for k in bow:
            bow[k] /= norm
    return bow, fv


def all_cases():
    return frustum_cases() + bow_cases()
