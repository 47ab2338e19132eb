"""Crafted candidate lists for DistributeOctTree (src/ORBextractor.cc:540-765), the extractor's quad-tree stage.

Each case is a level of an extractor geometry (params, rows x cols, level), a target N and a candidate list xys ([n, 3]
int32: x, y in level pixels and the FAST score, in vToDistributeKeys order).  The lists do not come from FAST, so they can
hold what FAST never produces (adjacent or repeated pixels, points on the region's last column and row) and aim at the
conditions that decide the output: initial-node boundaries, halving lines, sweep / largest-first termination, the
largest-first rank and its ties, and the best-key choice.  `edge` names the condition and `reached(case, trace, geo)`
says whether the oracle's round trace (oracle/ref.py: distribute(..., trace=True)) and the level geometry show it.

tests/test_quadtree_cases_cpu.py asserts that every case reaches its edge and that the oracle equals the reference's
own DistributeOctTree on it; tests/test_quadtree_crafted_gpu.py runs every case through the device kernel."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable

import numpy as np

from tests.test_boundaries_gpu import QT_LIMIT_8, fast_cells, level_features, level_sizes

B = 16                    # minBorderX = minBorderY = EDGE_THRESHOLD - 3 (:780)
SWEEP, LARGEST = 0, 1     # oracle/ref.py SWEEP, LARGEST_FIRST


@dataclass
class Geo:
    """Level geometry of a case: distribution region W x H (maxBorder - minBorder), nIni, hX, slot capacity, N_l."""
    W: int
    H: int
    n_ini: int
    hx: np.float32
    slots: int
    nfeat: int

    def ini_ul(self, i):   # initial node i's UL.x (:557): (int)(hX * i) in float
        return int(np.float32(self.hx) * np.float32(i))

    def ini_index(self, x_rel):   # the initial node of a keypoint (:566): (int)(kp.pt.x / hX)
        return min(int(np.float32(x_rel) / np.float32(self.hx)), self.n_ini - 1)


def geometry(params, rows, cols, level) -> Geo:
    nfeatures, scale, nlevels = params[0], params[1], params[2]
    lh, lw = level_sizes(rows, cols, scale, nlevels)[level]
    W, H = lw - 32, lh - 32
    nini = int(math.floor(float(np.float32(W) / np.float32(H)) + 0.5))
    slots = 0
    for rw, rh in fast_cells(lh, lw):
        if rw - 6 > 0 and rh - 6 > 0:
            slots += ((rw - 5) // 2) * ((rh - 5) // 2)
    return Geo(W, H, nini, np.float32(np.float32(W) / np.float32(nini)), slots,
               level_features(nfeatures, scale, nlevels)[level])


@dataclass
class Case:
    name: str
    params: tuple
    rows: int
    cols: int
    level: int
    N: int
    xys: np.ndarray
    edge: str
    reached: Callable = field(repr=False)


P1 = (1000, 1.2, 1, 20, 7)          # one level: N up to 1000
P8 = (1000, 1.2, 8, 20, 7)
PQ = (QT_LIMIT_8, 1.2, 8, 20, 7)    # level-0 quota 1156: the largest the quad-tree's shared memory takes


def _xys(pts, scores=None, seed=0):
    pts = np.asarray(pts, np.int64).reshape(-1, 2)
    if scores is None:
        scores = np.random.default_rng(seed).integers(0, 256, len(pts))
    out = np.zeros((len(pts), 3), np.int32)
    out[:, 0] = pts[:, 0] + B
    out[:, 1] = pts[:, 1] + B
    out[:, 2] = np.asarray(scores, np.int64) if np.ndim(scores) else scores
    return out


# ---- box arithmetic of DivideNode (:478-534), boxes relative to (minBorderX, minBorderY) --------------------------
def halves(box):
    x0, y0, x1, y1 = box
    mx, my = x0 + math.ceil((x1 - x0) / 2), y0 + math.ceil((y1 - y0) / 2)
    return mx, my


def child(box, q):
    """Quadrant q (0 UL, 1 UR, 2 BL, 3 BR) of a box, as DivideNode builds n1..n4."""
    x0, y0, x1, y1 = box
    mx, my = halves(box)
    return (mx if q & 1 else x0, my if q & 2 else y0, x1 if q & 1 else mx, y1 if q & 2 else my)


def cell(box, path):
    for q in path:
        box = child(box, q)
    return box


def inside(box):
    """A pixel strictly inside a box (its UL corner), for boxes of side >= 1."""
    return box[0], box[1]


def pair_in(box):
    """Two pixels of a box that the next split separates (UL and BR quadrants)."""
    return [inside(child(box, 0)), inside(child(box, 3))]


def leaves(root, depth, count, seed, per_parent=4):
    """`count` distinct cells of depth `depth` under root, grouped by parent: as few depth-1 parents as `per_parent`
    children each allows, parents spread over the tree in a random order."""
    rng = np.random.default_rng(seed)
    nparents = -(-count // per_parent)
    parents = rng.choice(4 ** (depth - 1), nparents, replace=False)
    paths = []
    for k, p in enumerate(parents):
        path = [(int(p) >> (2 * (depth - 2 - d))) & 3 for d in range(depth - 1)]
        for q in range(min(per_parent, count - k * per_parent)):
            paths.append(path + [q])
    return [cell(root, p) for p in paths]


def rounds(tr, kind=None):
    return [r for r in tr if kind is None or r["kind"] == kind]


# ---- edge predicates -------------------------------------------------------------------------------------------
def first_sweep_after(n):
    return lambda c, tr, g: tr[0]["kind"] == SWEEP and tr[0]["after"] == n


def largest_first_m(m):
    return lambda c, tr, g: any(r["kind"] == LARGEST and r["count"] == m for r in tr)


def stall(kind):
    return lambda c, tr, g: tr[-1]["kind"] == kind and tr[-1]["after"] == tr[-1]["before"] and tr[-1]["after"] < c.N


def sweeps_at_least(k):
    return lambda c, tr, g: len(rounds(tr, SWEEP)) >= k


def _stop(where):
    def f(c, tr, g):
        lf = rounds(tr, LARGEST)
        if not lf:
            return False
        r = lf[0]
        if where == "rank0":
            return r["splits"] == 1 and r["after"] >= c.N and r["count"] > 1
        if where == "last":
            return r["splits"] == r["count"] > 1 and r["after"] >= c.N
        return r["splits"] == r["count"] and r["after"] < c.N and len(lf) >= 2 and lf[1]["splits"] > 0
    return f


def _continue_sweep(c, tr, g):   # :675 n + 3*nToExpand == N: the loop sweeps again
    return len(tr) >= 2 and tr[0]["after"] + 3 * tr[0]["count"] == c.N and tr[1]["kind"] == SWEEP


def _start_largest(c, tr, g):    # n + 3*nToExpand == N + 1: the largest-first loop starts
    return len(tr) >= 2 and tr[0]["after"] + 3 * tr[0]["count"] == c.N + 1 and tr[1]["kind"] == LARGEST


def always(c, tr, g):
    return True


# ---- families --------------------------------------------------------------------------------------------------
def _ini_geometries():
    """(tag, params, rows, cols, level): nIni = 1, 2, 3, 4, 5, 8 and 58 at level 0, and 3 and 9 at level 2 of a 3-level
    handle.  Regions of non-integer hX, so floor(i*hX) and ceil(i*hX) differ."""
    P3 = (1000, 1.2, 3, 20, 7)
    return [("nini1", P1, 132, 139, 0), ("nini2", P1, 132, 239, 0), ("nini3", P1, 132, 339, 0),
            ("nini4", P1, 132, 439, 0), ("nini5", P1, 132, 539, 0), ("nini8", P1, 112, 675, 0),
            ("nini58", (10, 1.2, 1, 20, 7), 100, 4000, 0), ("l2_nini3", P3, 200, 500, 2), ("l2_nini9", P3, 150, 1000, 2)]


def ini_cases():
    out = []
    for tag, params, rows, cols, level in _ini_geometries():
        g = geometry(params, rows, cols, level)
        want = int(tag.split("nini")[1])
        pts = []
        for i in range(1, g.n_ini):
            t = float(np.float32(g.hx) * np.float32(i))
            for x in (math.floor(t) - 1, math.floor(t), math.ceil(t), math.ceil(t) + 1):
                pts += [(x, g.H // 3), (x, 2 * g.H // 3)]
        pts += [(0, 0), (g.W - 1, g.H - 1), (g.W - 1, 0), (0, g.H - 1)]
        N = min(g.nfeat, max(1, len(pts) // 3))

        def at_boundaries(c, tr, g, want=want):
            # floor(i*hX) of a non-integer i*hX lies in node i-1, on that node's UR.x column
            ok = g.n_ini == want
            for i in range(1, g.n_ini):
                t = float(np.float32(g.hx) * np.float32(i))
                if t != math.floor(t):
                    ok &= g.ini_index(math.floor(t)) == i - 1 and g.ini_ul(i) == math.floor(t)
            return ok
        out.append(Case("ini/%s/boundaries" % tag, params, rows, cols, level, N, _xys(pts, seed=len(out)),
                        "nIni = %d; keypoints at floor / ceil(i*hX) and +-1" % want, at_boundaries))
        # every initial node with four populated quadrants: the first sweep returns 4*nIni > N + 3
        quad = []
        for i in range(g.n_ini):
            box = (g.ini_ul(i), 0, g.ini_ul(i + 1), g.H)
            for q in range(4):
                b = child(box, q)
                quad += [(b[0] + 1, b[1] + 1), (b[0] + 2, b[1] + 2)]   # UL.x of node i may belong to node i-1
        Nq = min(g.nfeat, 4 * g.n_ini - 4) if g.n_ini > 1 else 0
        out.append(Case("ini/%s/all_quadrants" % tag, params, rows, cols, level, Nq, _xys(quad, seed=len(out)),
                        "first sweep returns 4*nIni > N + 3",
                        lambda c, tr, g: tr[0]["after"] == 4 * g.n_ini > c.N + 3))
        # each initial node's halving lines and the pixels before them: the node's box, (int)(i*hX) to (int)((i+1)*hX),
        # decides where they fall
        mid = []
        for i in range(g.n_ini):
            mx, my = halves((g.ini_ul(i), 0, g.ini_ul(i + 1), g.H))
            mid += [(mx - 1, my - 1), (mx, my - 1), (mx - 1, my), (mx, my)]
        out.append(Case("ini/%s/node_midlines" % tag, params, rows, cols, level, min(g.nfeat, 4 * g.n_ini), _xys(mid, seed=len(out)),
                        "keypoints on every initial node's halving lines", lambda c, tr, g: tr[0]["after"] == 4 * g.n_ini))
        if g.n_ini >= 4:   # empty initial nodes between populated ones, single-key initial nodes
            sparse = []
            for i in range(g.n_ini):
                x0, x1 = g.ini_ul(i), g.ini_ul(i + 1)
                if i % 3 == 1:
                    continue                                   # empty
                if i % 3 == 2:
                    sparse.append((x0 + 1, g.H // 2))          # one key: bNoMore from the start
                else:
                    sparse += [(x0 + 1 + k * (x1 - x0) // 5, k * g.H // 5) for k in range(5)]
            out.append(Case("ini/%s/empty_and_single" % tag, params, rows, cols, level, min(g.nfeat, 2 * g.n_ini),
                            _xys(sparse, seed=len(out)), "empty and single-key initial nodes",
                            lambda c, tr, g: tr[0]["before"] < g.n_ini))
    return out


def halving_cases():
    out = []
    for tag, rows, cols in (("even", 480, 640), ("odd", 479, 639), ("small_odd", 63, 81)):
        g = geometry(P1, rows, cols, 0)
        root = (0, 0, g.W, g.H)
        pts, box = [], root
        for d in range(9):   # the midline column / row and the one before it, following one quadrant down
            mx, my = halves(box)
            if box[2] - box[0] < 2 or box[3] - box[1] < 2:
                break
            pts += [(mx, my), (mx - 1, my - 1), (mx, my - 1), (mx - 1, my), (mx, box[1]), (box[0], my)]
            box = child(box, (d * 3) % 4)
        out.append(Case("halving/%s/midlines" % tag, P1, rows, cols, 0, min(g.nfeat, 400), _xys(pts, seed=d),
                        "keypoints on the halving lines and one before them, depth >= 6", sweeps_at_least(6)))
    for tag, rows, cols in (("even", 112, 144), ("odd", 111, 143), ("small_odd", 63, 81)):
        # a full row and a full column of adjacent pixels: every round splits some node, until boxes of side 1 hold
        # the column's vertical pairs and their splits make boxes of side 0
        g = geometry(P1, rows, cols, 0)
        pix = [(x, g.H // 2) for x in range(g.W)] + [(g.W // 3, y) for y in range(g.H)]
        out.append(Case("halving/%s/pixel_row_and_column" % tag, P1, rows, cols, 0, min(g.nfeat, 400),
                        _xys(pix, seed=5), "boxes of side 1 and 0",
                        lambda c, tr, g: tr[-1]["after"] == len({(x, y) for x, y, _ in c.xys.tolist()})))
    g = geometry(P1, 480, 640, 0)
    row = [(x, 200) for x in range(0, g.W, 2)]
    col = [(300, y) for y in range(g.H)]
    out.append(Case("halving/one_row", P1, 480, 640, 0, 150, _xys(row, seed=1), "every keypoint on one row",
                    sweeps_at_least(5)))
    out.append(Case("halving/one_column", P1, 480, 640, 0, 100, _xys(col, seed=2), "every keypoint on one column",
                    sweeps_at_least(5)))
    out.append(Case("halving/last_column_and_row", P1, 480, 640, 0, 12,
                    _xys([(g.W - 1, y) for y in range(0, g.H, 7)] + [(x, g.H - 1) for x in range(0, g.W, 9)], seed=3),
                    "keypoints on the region's last column and row", always))
    return out


def duplicate_cases():
    out = []
    g = geometry(P1, 480, 640, 0)
    for reps in (2, 3, 33, 600):
        pile = [(123, 77)] * reps
        out.append(Case("dup/alone_%d" % reps, P1, 480, 640, 0, 50, _xys(pile, seed=reps),
                        "one pixel %d times: the sweep stops growing" % reps, stall(SWEEP)))
        beside = pile + [(124, 77), (400, 300), (401, 301), (5, 400)] + [(123, 78)] * 2
        out.append(Case("dup/beside_%d" % reps, P1, 480, 640, 0, 60, _xys(beside, seed=reps + 1),
                        "one pixel %d times beside other points" % reps, always))
    one = [(200, 150)] * 40
    out.append(Case("dup/whole_level_one_pixel", P8, 480, 640, 5, 20, _xys(one, seed=9),
                    "every candidate of the level on one pixel", stall(SWEEP)))
    # four piles in the four quadrants: the largest-first iteration splits all four and the list does not grow
    piles = []
    for q in range(4):
        b = child((0, 0, g.W, g.H), q)
        piles += [inside(b)] * (3 + q)
    out.append(Case("dup/stall_in_largest_first", P1, 480, 640, 0, 5, _xys(piles, seed=11),
                    "a largest-first iteration that does not grow the list", stall(LARGEST)))
    # duplicates differing only in score (best key: the first maximal one in list order)
    sc = [(50, 60)] * 6 + [(300, 200)] * 5
    out.append(Case("best/dup_scores", P1, 480, 640, 0, 2, _xys(sc, scores=[3, 9, 9, 1, 9, 0, 7, 7, 2, 7, 6]),
                    "duplicates that differ only in score", always))
    return out


def _quad_tree_list(root, depth, fan):
    """Points in `fan` quadrants of every node, `depth` levels down: fan**depth leaves, one point each."""
    boxes = [root]
    for _ in range(depth):
        boxes = [child(b, q) for b in boxes for q in range(fan)]
    return [inside(b) for b in boxes]


def termination_cases():
    out = []
    g = geometry(P1, 480, 640, 0)
    root = (0, 0, g.W, g.H)
    four = _quad_tree_list(root, 1, 4)
    out.append(Case("term/first_sweep_eq_N", P1, 480, 640, 0, 4, _xys([p for p in four for _ in (0,)], seed=1),
                    "the first sweep ends at n == N", lambda c, tr, g: len(tr) == 1 and tr[0]["after"] == c.N))
    sixteen = _quad_tree_list(root, 2, 4)
    three = [p for p in sixteen if cell_of(root, p)[0] != 3]
    out.append(Case("term/first_sweep_N_minus_1", P1, 480, 640, 0, 4, _xys(three, seed=2),
                    "the first sweep ends at n == N - 1", lambda c, tr, g: tr[0]["after"] == c.N - 1))
    # after the first sweep n = 4, nToExpand = 4: N = 16 sweeps on, N = 15 starts the largest-first loop
    sixty4 = _quad_tree_list(root, 3, 4)
    out.append(Case("term/n_plus_3e_eq_N", P1, 480, 640, 0, 16, _xys(sixty4, seed=3),
                    "n + 3*nToExpand == N: the sweep continues", _continue_sweep))
    out.append(Case("term/n_plus_3e_eq_N_plus_1", P1, 480, 640, 0, 15, _xys(sixty4, seed=4),
                    "n + 3*nToExpand == N + 1: largest-first starts", _start_largest))
    # largest-first over 4 nodes of 16, 12, 8 and 4 points, each splitting into 4 children: +3 per split
    sized = []
    for q, k in zip(range(4), (4, 3, 2, 1)):
        sub = [child(child(root, q), s) for s in range(4)]
        for b in sub:
            sized += [inside(child(b, t)) for t in range(k)]
    # sweep 1: n = 4, e = 4 -> 16 > N: the first largest-first iteration splits the 16-point node first (+3), ...
    out.append(Case("term/lf_stop_rank0", P1, 480, 640, 0, 6, _xys(sized, seed=5), "largest-first stops at rank 0",
                    _stop("rank0")))
    out.append(Case("term/lf_stop_last_rank", P1, 480, 640, 0, 14, _xys(sized, seed=6), "largest-first stops at the last rank",
                    _stop("last")))
    # four diagonal runs of 8 points: every split makes 2 children, +1 per split, so 4 splits do not reach N = 15 and the
    # next iteration runs over the 8 new children
    diag = []
    for q in range(4):
        x0, y0, x1, y1 = child(root, q)
        diag += [(x0 + t * (x1 - x0) // 8, y0 + t * (y1 - y0) // 8) for t in range(8)]
    out.append(Case("term/lf_not_reached", P1, 480, 640, 0, 15, _xys(diag, seed=7),
                    "largest-first not reached: a further iteration over the new children", _stop("none")))
    rng = np.random.default_rng(8)
    blob = [(int(x), int(y)) for x, y in zip(rng.integers(0, g.W, 700), rng.integers(0, g.H, 700))]
    out.append(Case("term/N0", P1, 480, 640, 0, 0, _xys(blob, seed=8), "N = 0: one sweep", lambda c, tr, g: len(tr) == 1))
    out.append(Case("term/N1", P1, 480, 640, 0, 1, _xys(blob, seed=9), "N = 1: one sweep", lambda c, tr, g: len(tr) == 1))
    return out


def cell_of(root, p):
    """Quadrant path of depth 1 of point p."""
    mx, my = halves(root)
    return [(1 if p[0] >= mx else 0) | (2 if p[1] >= my else 0)]


def rank_cases():
    """Largest-first over m nodes of two points each, all created by one sweep: every key ties on size."""
    out = []
    g = geometry(PQ, 480, 640, 0)
    root = (0, 0, g.W, g.H)
    for m, N, depth in ((1, 3, 1), (2, 5, 1), (3, 7, 1), (4, 9, 1), (5, 19, 2), (511, 1156, 5), (512, 1156, 5),
                        (513, 1156, 5), (1024, 1156, 6), (1025, 1156, 6), (1155, 1156, 6)):
        per = 4 if m > 4 else m
        cells = leaves(root, depth, m, seed=m, per_parent=per) if depth > 1 else [child(root, q) for q in range(m)]
        pts = [p for b in cells for p in pair_in(b)]
        if m == 1:
            pts.append(inside(child(root, 3)))   # a single-key node beside it, so that the first sweep grows the list
        out.append(Case("rank/m%d" % m, PQ, 480, 640, 0, N, _xys(pts, seed=m), "largest-first over m = %d" % m,
                        largest_first_m(m)))
    # equal sizes from different parents and rounds over >= 3 largest-first iterations: the 16 depth-2 nodes hold
    # diagonal runs (split 4 -> 2 -> 1, one more node per split) or pairs at distances that separate them only after 1, 2
    # or 3 more halvings (until then a split leaves one child of the same size 2)
    runs = []
    for k in range(16):
        x0, y0, x1, y1 = cell(root, [k // 4, k % 4])
        if k % 2 == 0:
            runs += [(x0 + t * (x1 - x0) // 4, y0 + t * (y1 - y0) // 4) for t in range(4)]
        else:
            d = (x1 - x0) >> (1 + (k // 2) % 4)
            runs += [(x0 + 1, y0 + 1), (x0 + 1 + d, y0 + 1 + d)]
    out.append(Case("rank/ties_three_iterations", PQ, 480, 640, 0, 60, _xys(runs, seed=100),
                    "equal sizes over >= 3 largest-first iterations", lambda c, tr, g: len(rounds(tr, LARGEST)) >= 3))
    return out


def best_key_cases():
    out = []
    g = geometry(P1, 480, 640, 0)
    root = (0, 0, g.W, g.H)
    nodes = [child(root, q) for q in range(4)]
    pts = [inside(b) for b in nodes for _ in range(1)] + [(b[0] + 5, b[1] + 5) for b in nodes]
    out.append(Case("best/all_equal", P1, 480, 640, 0, 4, _xys(pts, scores=77), "all scores equal: the first wins",
                    always))
    last = []
    sc = []
    for b in nodes:
        last += [(b[0] + k, b[1] + 2 * k) for k in range(6)]
        sc += [10, 20, 30, 40, 50, 200]
    out.append(Case("best/max_at_last_index", P1, 480, 640, 0, 4, _xys(last, scores=sc), "the maximum at a node's last index",
                    always))
    ext = []
    se = []
    for k, b in enumerate(nodes):
        ext += [(b[0] + 2, b[1] + 3), (b[0] + 9, b[1] + 1), (b[0] + 4, b[1] + 8)]
        se += [[0, 0, 0], [255, 0, 255], [0, 255, 0], [255, 255, 255]][k]
    out.append(Case("best/scores_0_255", P1, 480, 640, 0, 4, _xys(ext, scores=se), "scores 0 and 255", always))
    return out


def size_cases():
    out = []
    g = geometry(P1, 480, 640, 0)
    out.append(Case("size/K1", P1, 480, 640, 0, 10, _xys([(g.W - 1, g.H - 1)], seed=1), "K = 1", always))
    out.append(Case("size/K2", P1, 480, 640, 0, 10, _xys([(0, 0), (0, 0)], scores=[4, 4]), "K = 2", always))
    gs = geometry(P1, 100, 120, 0)   # a small level: K at the level's slot capacity
    rng = np.random.default_rng(5)
    full = list(zip(rng.integers(0, gs.W, gs.slots).tolist(), rng.integers(0, gs.H, gs.slots).tolist()))
    out.append(Case("size/K_at_slot_capacity", P1, 100, 120, 0, min(gs.nfeat, 150), _xys(full, seed=5),
                    "K = the level's slot capacity", lambda c, tr, g: len(c.xys) == g.slots))
    # the same list on every level of an 8-level handle: the per-level slot and selection offsets
    g7 = geometry(P8, 480, 640, 7)
    rng = np.random.default_rng(6)
    same = list(zip(rng.integers(0, g7.W, 300).tolist(), rng.integers(0, g7.H, 300).tolist()))
    frac = np.random.default_rng(7).random((300, 2))
    for l in range(8):
        gl = geometry(P8, 480, 640, l)
        out.append(Case("size/every_level/L%d" % l, P8, 480, 640, l, min(gl.nfeat, 60), _xys(same, seed=6),
                        "the same list on level %d of 8" % l, always))
        scaled = (frac * [gl.W, gl.H]).astype(np.int64)   # the same list stretched over the level's region
        out.append(Case("size/every_level_scaled/L%d" % l, P8, 480, 640, l, min(gl.nfeat, 60), _xys(scaled, seed=8),
                        "one list stretched over level %d of 8" % l, lambda c, tr, g: len(tr) >= 3))
    return out


def all_cases():
    cases = ini_cases() + halving_cases() + duplicate_cases() + termination_cases() + rank_cases() + best_key_cases() + \
        size_cases()
    names = [c.name for c in cases]
    assert len(names) == len(set(names)), "duplicate case names"
    return cases


def oracle_input(case, oracle):
    """The case as the oracle's DistributeOctTree input: KeyPoints relative to (minBorderX, minBorderY), and the region."""
    g = geometry(case.params, case.rows, case.cols, case.level)
    k = np.zeros(len(case.xys), oracle.KP_DTYPE)
    k["x"] = case.xys[:, 0] - B
    k["y"] = case.xys[:, 1] - B
    k["response"] = case.xys[:, 2]
    k["size"] = 7
    k["angle"] = -1
    k["class_id"] = -1
    return k, g


def oracle_distribute(case, oracle, trace=False):
    """-> selected keypoints [m, 3] int32 (x, y, score in level pixels, list order)[, the round trace]."""
    k, g = oracle_input(case, oracle)
    r = oracle.distribute(k, 0, g.W, 0, g.H, case.N, trace=trace)
    a, tr = r if trace else (r, None)
    out = np.stack([a["x"].astype(np.int32) + B, a["y"].astype(np.int32) + B, a["response"].astype(np.int32)], 1)
    return (out.reshape(-1, 3), tr) if trace else out.reshape(-1, 3)
