"""Deterministic crafted cases for the ORB matcher: inputs placed exactly on the value edges where a restatement of
ORBmatcher.cc goes wrong -- distances at the thresholds and ratio bounds, exact distance ties decided by the visiting
order, keypoints at half a grid cell, windows whose edge passes through a keypoint, rotations at half a histogram bin,
and queries of one 32-query resolve step claiming the same keypoint.

Camera: fx = fy = 512, integer cx / cy, identity rotation, camera depth z in {1, 2}: the LAST projection
fx * xc * invzc + cx is then exact in float, so a keypoint can sit at an exact offset from the projected u, v.  A
candidate at Hamming distance d is the query's descriptor with exactly d bits flipped (the complement for 256).

Every case carries `edges`: (kind, payload) claims about its own inputs that tests/test_matcher_edges_cpu.py checks in
numpy, so a case that stops containing its edge fails instead of silently testing nothing."""
import math

import numpy as np

from orb_slam2_ssd_semantic_b200._abi import BowView, FrameView, LastView, QueriesView, TrackPointsView

f32 = np.float32
FX = FY = 512.0
CX, CY = 320.0, 240.0
BF = 40.0                 # b = bf / fx = 0.078125; the predicted right coordinate is u - 20 at z = 2
SF = np.cumprod(np.concatenate([[f32(1.0)], np.full(7, f32(1.2), f32)])).astype(f32)
TH_HIGH, TH_LOW = 100, 50
GRID_COLS, GRID_ROWS = 64, 48
LAST_NNRATIO = 0.9
LCAP = 64                 # orbm_kernels.cuh: candidate-list capacity per query
BOUNDS = (0.0, 640.0, 0.0, 480.0)
# width 512 and height 384: inv_w = inv_h = 1/8 exactly, so a keypoint can sit at exactly half a cell
HALF_BOUNDS = (3.25, 515.25, 2.75, 386.75)


def flip(d, k, salt):
    """d with exactly k of its 256 bits flipped."""
    out = np.array(d, np.uint8).copy()
    for b in np.random.default_rng(salt).permutation(256)[:k]:
        out[b >> 3] ^= np.uint8(1 << (b & 7))
    return out


def hamming(a, b):
    return int(np.unpackbits(np.bitwise_xor(np.asarray(a, np.uint8), np.asarray(b, np.uint8))).sum())


def window_columns(u, r, min_x, max_x):
    """Grid columns of GetFeaturesInArea's window (src/Frame.cc:471-477), in float like the reference."""
    inv_w = f32(f32(GRID_COLS) / f32(f32(max_x) - f32(min_x)))
    x0 = max(0, int(math.floor(f32(f32(f32(u) - f32(min_x)) - f32(r)) * inv_w)))
    x1 = min(GRID_COLS - 1, int(math.ceil(f32(f32(f32(u) - f32(min_x)) + f32(r)) * inv_w)))
    return x1 - x0 + 1


def grid_coord(x, lo, hi, cells):
    """(x - min) * inv, the value PosInGrid rounds (src/Frame.cc:522-531)."""
    inv = f32(f32(cells) / f32(f32(hi) - f32(lo)))
    return float(f32(f32(f32(x) - f32(lo)) * inv))


def rot_value(a_query, a_cur):
    """rot * factor of the orientation histogram (:1685-1690 and the other searches)."""
    r = f32(f32(a_query) - f32(a_cur))
    if r < 0:
        r = f32(r + f32(360.0))
    return float(f32(r * f32(f32(1.0) / f32(30))))


class Case:
    def __init__(self, name, kind, edges, **kw):
        self.name, self.kind, self.edges, self.kw = name, kind, list(edges), kw

    def __repr__(self):
        return self.name


class Scene:
    """Keypoints of one current frame and the queries into it, added site by site."""

    def __init__(self, seed):
        self.k = []
        self.q = []
        self.rng = np.random.default_rng(seed)
        self.salt = seed * 1000

    def base(self):
        return self.rng.integers(0, 256, 32, dtype=np.uint8)

    def cand(self, qd, d):
        self.salt += 1
        return flip(qd, d, self.salt)

    def kp(self, x, y, desc, oct=0, angle=100.0, uright=-1.0, obs=-1):
        self.k.append((x, y, oct, desc, angle, uright, obs))
        return len(self.k) - 1

    def query(self, u, v, desc, oct=0, angle=100.0, valid=1, obs=1, z=2.0, view_cos=1.0, xr=None):
        self.q.append(dict(u=u, v=v, desc=desc, oct=oct, angle=angle, valid=valid, obs=obs, z=z, view_cos=view_cos, xr=xr))
        return len(self.q) - 1

    def frame(self, bounds=BOUNDS, tz=0.0, pad=0, with_obs=None):
        k = self.k
        n = len(k)
        col = lambda j, t: np.array([p[j] for p in k], t) if n else np.zeros(0, t)
        x, y, octv, ang, ur, obs = col(0, f32), col(1, f32), col(2, np.int32), col(4, f32), col(5, f32), col(6, np.int32)
        desc = np.stack([p[3] for p in k]) if n else np.zeros((0, 32), np.uint8)
        if pad:   # keypoints that PosInGrid drops: every crafted index moves up by `pad`
            x = np.concatenate([np.full(pad, -1000.0, f32), x])
            y = np.concatenate([np.full(pad, -1000.0, f32), y])
            octv = np.concatenate([np.zeros(pad, np.int32), octv])
            ang = np.concatenate([np.zeros(pad, f32), ang])
            ur = np.concatenate([np.full(pad, -1.0, f32), ur])
            obs = np.concatenate([np.full(pad, -1, np.int32), obs])
            desc = np.concatenate([np.zeros((pad, 32), np.uint8), desc])
        T = np.eye(4, dtype=f32)
        T[2, 3] = tz
        use_obs = (obs >= 0).any() if with_obs is None else with_obs
        return FrameView(x, y, octv, ang, ur, desc, T, FX, FY, CX, CY, BF, *bounds, SF, mp_obs=obs if use_obs else None)

    def last(self, tz=0.0):
        q = self.q
        z = np.array([p["z"] for p in q], np.float64)
        u = np.array([p["u"] for p in q], np.float64)
        v = np.array([p["v"] for p in q], np.float64)
        xw = np.stack([(u - CX) * z / FX, (v - CY) * z / FY, z - tz], 1).astype(f32)
        assert ((u - CX) * z / FX == xw[:, 0]).all() and ((v - CY) * z / FY == xw[:, 1]).all()
        return LastView(xw, np.array([p["valid"] for p in q], np.uint8), np.array([p["oct"] for p in q], np.int32),
                        np.array([p["angle"] for p in q], f32), np.stack([p["desc"] for p in q]), np.eye(4, dtype=f32),
                        mp_obs=np.array([p["obs"] for p in q], np.int32))

    def points(self):
        q = self.q
        px = np.array([p["u"] for p in q], f32)
        xr = np.array([p["xr"] if p["xr"] is not None else p["u"] - 20.0 for p in q], f32)
        return TrackPointsView(np.array([p["valid"] for p in q], np.uint8), px, np.array([p["v"] for p in q], f32), xr,
                               np.array([p["oct"] for p in q], np.int32), np.array([p["view_cos"] for p in q], f32),
                               np.stack([p["desc"] for p in q]), mp_obs=np.array([p["obs"] for p in q], np.int32))

    def queries(self, radius, levels, uright=False):
        q = self.q
        lv = np.array(levels, np.int32).reshape(-1, 2) if np.ndim(levels) == 2 else np.tile(np.array(levels, np.int32), (len(q), 1))
        return QueriesView(np.array([p["valid"] for p in q], np.uint8), np.array([p["u"] for p in q], f32),
                           np.array([p["v"] for p in q], f32), np.full(len(q), radius, f32), lv[:, 0], lv[:, 1],
                           np.stack([p["desc"] for p in q]), np.array([p["angle"] for p in q], f32),
                           uright=np.array([p["u"] - 20.0 for p in q], f32) if uright else None,
                           obs=np.array([p["obs"] for p in q], np.int32))


def _dist_edges(S, pairs):
    """("dist", (query desc, keypoint desc, d)) for every (query, keypoint, d)."""
    return [("dist", (S.q[qi]["desc"], S.k[ki][3], d)) for qi, ki, d in pairs]


# ---------------------------------------------------------------------------------------------------------------------
# SearchByProjection(Frame&, const Frame&, th, bMono)
# ---------------------------------------------------------------------------------------------------------------------
def _last(name, S, th, edges, bounds=BOUNDS, tz=0.0, ori=True, mono=False):
    return Case(name, "last", edges, scene=S, th=th, bounds=bounds, tz=tz, ori=ori, mono=mono)


def last_views(case, pad=0):
    S, kw = case.kw["scene"], case.kw
    return S.frame(kw["bounds"], kw["tz"], pad), S.last(kw["tz"])


def _last_threshold():
    S = Scene(1)
    pairs = []
    for j, d in enumerate((100, 101, 99)):
        qd = S.base()
        S.query(100.0 + 150 * j, 100.0, qd, oct=1)
        pairs.append((j, S.kp(101.0 + 150 * j, 100.0, S.cand(qd, d), oct=1), d))
    return _last("last/th_high_100_101", S, 10.0, _dist_edges(S, pairs))


def _last_ties():
    """Three candidates at one distance: the later index 1 sits in an earlier grid column than index 0, index 2 shares
    index 1's cell.  The first in the (ix, iy, insertion) order wins."""
    S = Scene(2)
    qd = S.base()
    S.query(204.0, 100.0, qd)
    a = S.kp(211.0, 100.0, S.cand(qd, 30))     # column round(21.1) = 21
    b = S.kp(197.0, 100.0, S.cand(qd, 30))     # column 20
    c = S.kp(199.0, 101.0, S.cand(qd, 30))     # column 20, same cell as b
    S.kp(204.0, 108.0, S.cand(qd, 31))
    edges = [("tie", [(qd, S.k[i][3]) for i in (a, b, c)]), ("order", (S.k[b][0] < S.k[a][0], b > a))]
    return _last("last/ties_visit_order", S, 10.0, edges)


def _last_grid_half():
    """PosInGrid at -0.5, 62.5 and 63.5 cells (round half away from zero: dropped, cell 63, dropped) on bounds with
    non-integer minima, and queries at u == min_x and u == max_x."""
    S = Scene(3)
    mnx, mxx, mny, mxy = HALF_BOUNDS
    # -0.5: dropped -> the worse keypoint inside the grid wins
    qd = S.base()
    S.query(mnx + 1.0, 100.75, qd)
    S.kp(mnx - 4.0, 100.75, S.cand(qd, 10))
    S.kp(mnx + 6.0, 100.75, S.cand(qd, 20))
    # 62.5 -> column 63, after the tie partner in column 62
    qd = S.base()
    S.query(mnx + 499.0, 200.75, qd)
    S.kp(mnx + 500.0, 200.75, S.cand(qd, 15))
    S.kp(mnx + 497.0, 200.75, S.cand(qd, 15))
    # 63.5 -> dropped
    qd = S.base()
    S.query(mnx + 511.0, 300.75, qd)
    S.kp(mnx + 508.0, 300.75, S.cand(qd, 10))
    S.kp(mnx + 506.0, 300.75, S.cand(qd, 30))
    # u == min_x, u == max_x
    qd = S.base()
    S.query(mnx, 150.75, qd)
    S.kp(mnx + 2.0, 150.75, S.cand(qd, 5))
    qd = S.base()
    S.query(mxx, 50.75, qd)
    S.kp(mxx - 5.0, 50.75, S.cand(qd, 7))
    edges = [("cell", (mnx - 4.0, mnx, mxx, GRID_COLS, -0.5)), ("cell", (mnx + 500.0, mnx, mxx, GRID_COLS, 62.5)),
             ("cell", (mnx + 508.0, mnx, mxx, GRID_COLS, 63.5))]
    return _last("last/grid_half_cells", S, 6.0, edges, bounds=HALF_BOUNDS)


def _last_window_edge():
    S = Scene(4)
    qd = S.base()
    S.query(200.0, 200.0, qd)
    S.kp(210.0, 200.0, S.cand(qd, 5))                            # |dx| == r: outside
    S.kp(float(np.nextafter(f32(210.0), f32(0))), 200.0, S.cand(qd, 20))   # just inside
    S.kp(200.0, 190.0, S.cand(qd, 3))                            # |dy| == r: outside
    # stereo gate: predicted right coordinate 400 - 20 = 380, radius 10
    qd = S.base()
    S.query(400.0, 200.0, qd)
    S.kp(401.0, 200.0, S.cand(qd, 30), uright=390.0)             # er == r: passes
    S.kp(402.0, 201.0, S.cand(qd, 10), uright=float(np.nextafter(f32(390.0), f32(1000))))   # er > r
    qd = S.base()
    S.query(500.0, 300.0, qd)
    S.kp(501.0, 300.0, S.cand(qd, 40), uright=0.0)               # uright == 0: no gate
    edges = [("eq", (float(f32(f32(210.0) - f32(200.0))), 10.0)), ("eq", (float(f32(f32(380.0) - f32(390.0))), -10.0))]
    return _last("last/window_edge_and_stereo_gate", S, 10.0, edges)


def _last_levels(tz, name):
    """Level windows at octave 0 and 7 (no motion), forward motion (octave 0: no level check), backward motion."""
    S = Scene(5)
    for j, (qo, good, bad) in enumerate([(0, 1, 2), (7, 6, 5), (3, 4, 1), (0, 7, 3), (3, 0, 4)]):
        qd = S.base()
        S.query(80.0 + 110 * j, 240.0, qd, oct=qo, z=1.0 if j % 2 else 2.0)
        S.kp(81.0 + 110 * j, 240.0, S.cand(qd, 40), oct=good)
        S.kp(79.0 + 110 * j, 241.0, S.cand(qd, 20), oct=bad)
    return _last(name, S, 2.0, [("motion", tz)], tz=tz)


def _last_clipped():
    S = Scene(6)
    for j, (u, v) in enumerate([(2.0, 3.0), (638.0, 478.0), (1.0, 477.0), (639.0, 1.0)]):
        qd = S.base()
        S.query(u, v, qd)
        S.kp(min(max(u + 12.0, 0.0), 639.0) if u < 320 else u - 12.0, v + (9.0 if v < 240 else -9.0), S.cand(qd, 25))
    return _last("last/windows_clipped", S, 30.0, [("clip", [(2.0, 30.0, 0.0, 640.0), (638.0, 30.0, 0.0, 640.0)])])


def _last_branch(w, h):
    """One query at octave 7, th 30 (r = 107.5 px) in the middle of a w x h frame, with equal-distance keypoints where
    the one in the earlier column sits in the later row and has the larger index: the ix-outer order picks it."""
    S = Scene(7)
    u, v = w / 2.0, h / 2.0
    qd = S.base()
    S.query(u, v, qd, oct=7)
    for j in range(40):
        dx, dy = float((j * 37) % 190 - 95), float((j * 53) % 170 - 85)
        S.kp(u + dx, v + dy, S.cand(qd, 60 + j % 3), oct=6 + j % 2)
    b = S.kp(u + 40.0, v - 50.0, S.cand(qd, 12), oct=7)
    a = S.kp(u - 40.0, v + 50.0, S.cand(qd, 12), oct=7)
    r = float(f32(f32(30.0) * SF[7]))
    edges = [("cols", (u, r, 0.0, float(w), w == 320)), ("tie", [(qd, S.k[a][3]), (qd, S.k[b][3])])]
    return _last("last/warp_walk_%dx%d" % (w, h), S, 30.0, edges, bounds=(0.0, float(w), 0.0, float(h)))


def _claim_scene(nl, seed, crowd=False):
    """nl queries at sites 32 px apart, two consecutive queries per site (plus query 31 on query 0's site), claim flags
    cycling through claim->claim, claim->no claim, no claim->claim, no claim->no claim.  Every site has keypoints at
    distances 20, 30, 40 from the site's descriptor.  Some queries are invalid, behind the camera or see an empty window;
    some keypoints hold pre-existing MapPoints with Observations() -1, 0 and 1.  crowd: site 3 also holds 70 keypoints
    (an overflowed candidate list) inside a step with conflicts."""
    S = Scene(seed)
    site_of = [i // 2 for i in range(nl)]
    if nl > 31:
        site_of[31] = site_of[0]
    pattern = [(1, 1), (1, 0), (0, 1), (0, 0)]
    sites = {}
    for s in sorted(set(site_of)):
        x, y = 24.0 + 32.0 * (s % 19), 24.0 + 32.0 * (s // 19)
        qd = S.base()
        sites[s] = (x, y, qd)
        if s % 11 == 7:
            continue                                             # empty window
        S.kp(x + 2.0, y + 1.0, S.cand(qd, 20), oct=1, obs=0 if s % 13 == 5 else -1)
        S.kp(x - 3.0, y + 2.0, S.cand(qd, 30), oct=1, obs=1 if s % 13 == 6 else -1)
        S.kp(x + 1.0, y - 3.0, S.cand(qd, 40), oct=1)
        if crowd and s == 3:
            for j in range(70):
                S.kp(x - 4.0 + j % 9, y - 4.0 + (j // 9) % 9, S.cand(qd, 45 + j % 7), oct=1)
    for i in range(nl):
        x, y, qd = sites[site_of[i]]
        S.query(x, y, qd, oct=1, obs=pattern[(i // 2) % 4][i % 2], valid=0 if i % 17 == 9 else 1,
                z=-2.0 if i % 23 == 11 else 2.0, angle=100.0 + (i % 3))
    return S, site_of


def _last_claims(nl, crowd=False):
    S, site_of = _claim_scene(nl, 100 + nl, crowd)
    return _last("last/claims_nl%d%s" % (nl, "_overflow" if crowd else ""), S, 5.0,
                 [("conflict", None)] + ([("crowd", (LCAP, float(f32(f32(5.0) * SF[1]))))] if crowd else []))


def _last_rotation():
    """rot at exactly 15 (half a bin: bin 1, where rintf gives 0) and its float neighbours, a tiny negative rot
    (360 - eps); bin 1 holds 13 matches, so bin 0 is kept with two entries and dropped with one; an overwritten
    assignment whose bin is pruned."""
    S = Scene(8)
    angles = [130.0] * 11 + [115.0, float(np.nextafter(f32(115.0), f32(0))), float(np.nextafter(f32(115.0), f32(200))),
                             float(np.nextafter(f32(100.0), f32(0))), 145.0, 175.0, 205.0]
    for j, a in enumerate(angles):
        qd = S.base()
        x, y = 40.0 + 60.0 * (j % 10), 60.0 + 80.0 * (j // 10)
        S.query(x, y, qd, angle=a, obs=1)
        S.kp(x + 1.0, y, S.cand(qd, 10), angle=100.0)
    # overwrite: query A (no claim) takes K with a pruned rotation, query B (no claim) then takes K with rot 30
    qd = S.base()
    S.query(400.0, 400.0, qd, angle=100.0 + 200.0, obs=0)
    S.query(400.0, 400.0, qd, angle=130.0, obs=0)
    S.kp(401.0, 400.0, S.cand(qd, 10), angle=100.0)
    edges = [("half", rot_value(115.0, 100.0))]
    return _last("last/rotation_bins", S, 5.0, edges)


def _last_maxima(counts, name, claim):
    """ComputeThreeMaxima on crafted bin counts: counts[b] matches with rot = 30 * b.  claim: "equal" (equal counts,
    the earlier bin wins), "kept" (max2 and max3 exactly max1 / 10 in float), "dropped" (max3 just below it)."""
    S = Scene(9)
    j = 0
    for b, c in counts:
        for _ in range(c):
            qd = S.base()
            x, y = 30.0 + 40.0 * (j % 15), 30.0 + 40.0 * (j // 15)
            S.query(x, y, qd, angle=100.0 + 30.0 * b)
            S.kp(x + 1.0, y, S.cand(qd, 10), angle=100.0)
            j += 1
    return _last(name, S, 5.0, [("bins", (counts, claim))])


def last_cases():
    return ([_last_threshold(), _last_ties(), _last_grid_half(), _last_window_edge(),
             _last_levels(0.0, "last/levels_no_motion"), _last_levels(-1.0, "last/levels_forward"),
             _last_levels(1.0, "last/levels_backward"), _last_clipped(), _last_branch(320, 240), _last_branch(640, 480),
             _last_rotation(),
             _last_maxima([(0, 10), (3, 10), (5, 10), (7, 10)], "last/maxima_equal_counts", "equal"),
             _last_maxima([(2, 10), (4, 1), (6, 1)], "last/maxima_tenth_kept", "kept"),
             _last_maxima([(2, 11), (4, 11), (6, 1), (8, 1)], "last/maxima_tenth_dropped", "dropped")] +
            [_last_claims(nl) for nl in (31, 32, 33, 64, 65, 200)] + [_last_claims(64, True), _last_claims(200, True)])


# ---------------------------------------------------------------------------------------------------------------------
# SearchByProjection(Frame&, const vector<MapPoint*>&, th): window 2.5 * sf[level] px (th 1, viewing cos > 0.998)
# ---------------------------------------------------------------------------------------------------------------------
def _points(name, S, nnratio, edges):
    return Case(name, "points", edges, scene=S, th=1.0, nnratio=nnratio)


def _points_sites(S, specs):
    """specs: per query (level, [(d, level), ...]) -> the candidates sit 1 px apart around the query."""
    pairs = []
    for j, (lvl, cands) in enumerate(specs):
        qd = S.base()
        x, y = 40.0 + 60.0 * (j % 10), 40.0 + 60.0 * (j // 10)
        qi = S.query(x, y, qd, oct=lvl)
        for e, (d, kl) in enumerate(cands):
            pairs.append((qi, S.kp(x + (e % 2) - 0.5 * (e // 2), y + 0.5 * (e // 2), S.cand(qd, d), oct=kl), d))
    return pairs


def points_cases():
    out = []
    S = Scene(20)
    pairs = _points_sites(S, [(1, [(100, 1)]), (1, [(101, 1)]), (2, [(100, 2), (256, 2)])])
    out.append(_points("points/th_high_100_101", S, 0.8, _dist_edges(S, pairs)))
    # ratio at equality: 60 vs 80 * 0.75 (accepted: '>' rejects), one past (61), different levels (no ratio test)
    S = Scene(21)
    specs = [(2, [(60, 2), (80, 2)]), (2, [(80, 2), (60, 2)]), (2, [(61, 2), (80, 2)]), (2, [(61, 2), (80, 1)]),
             (2, [(90, 1), (80, 2)])]
    pairs = _points_sites(S, specs)
    out.append(_points("points/ratio_equality", S, 0.75, _dist_edges(S, pairs) + [("ratio", (60, 80, 0.75))]))
    # the runner-up at distance 256, both orders: never recorded by the reference
    for nn in (0.3, 0.8):
        S = Scene(22)
        pairs = _points_sites(S, [(2, [(90, 2), (256, 2)]), (2, [(256, 2), (90, 2)]), (3, [(256, 3), (40, 3), (256, 3)])])
        out.append(_points("points/runner_up_256_nn%g" % nn, S, nn, _dist_edges(S, pairs)))
    # exact ties, first in visiting order; a claimed tie partner
    S = Scene(23)
    qd = S.base()
    S.query(295.0, 200.0, qd, oct=1, obs=0)
    a = S.kp(297.0, 200.0, S.cand(qd, 33), oct=1)    # column 30
    b = S.kp(293.0, 200.0, S.cand(qd, 33), oct=0)    # column 29: visited first
    S.query(295.0, 200.0, qd, oct=1, obs=1)
    S.query(295.0, 200.0, qd, oct=1, obs=1)
    out.append(_points("points/ties", S, 0.8, [("tie", [(qd, S.k[a][3]), (qd, S.k[b][3])]),
                                               ("order", (S.k[b][0] < S.k[a][0], b > a))]))
    # the runner-up at distance 256 in a window of more than LCAP candidates (the overflow re-walk), both orders
    S = Scene(24)
    r = float(f32(f32(2.5) * SF[7]))
    for j in range(2):
        qd = S.base()
        x, y = 100.0 + 200.0 * j, 200.0
        S.query(x, y, qd, oct=7)
        offs = [(dx, dy) for dx in range(-8, 9) for dy in range(-8, 9)][:70]
        best = 0 if j == 0 else len(offs) - 1
        for e, (dx, dy) in enumerate(offs):
            S.kp(x + dx, y + dy, S.cand(qd, 90 if e == best else 256), oct=7)
    out.append(_points("points/runner_up_256_overflow_nn0.3", S, 0.3, [("crowd", (LCAP, r))]))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# SearchProjected (claim rules 0 and 1) and the per-query best search
# ---------------------------------------------------------------------------------------------------------------------
def projected_cases():
    out = []
    for rule in (0, 1):
        for md in (64, 100):
            S = Scene(30)
            pairs = []
            for j, d in enumerate((md, md + 1)):
                qd = S.base()
                S.query(50.0 + 100 * j, 60.0, qd)
                pairs.append((j, S.kp(51.0 + 100 * j, 60.0, S.cand(qd, d), oct=1), d))
            # ties + claims: three queries on one site, keypoints with pre-existing points of 0 and 1 observations
            qd = S.base()
            for obs in (0, 1, 0):
                S.query(300.0, 300.0, qd, obs=obs)
            a = S.kp(303.0, 300.0, S.cand(qd, 20), oct=1)
            b = S.kp(297.0, 301.0, S.cand(qd, 20), oct=1)
            S.kp(300.0, 302.0, S.cand(qd, 10), oct=1, obs=0)
            S.kp(300.0, 298.0, S.cand(qd, 5), oct=1, obs=1)
            edges = _dist_edges(S, pairs) + [("tie", [(qd, S.k[a][3]), (qd, S.k[b][3])])]
            out.append(Case("projected/rule%d_max%d" % (rule, md), "projected", edges, scene=S, max_dist=md, rule=rule,
                            radius=6.0, levels=(0, 2)))
    return out


def best_cases():
    S = Scene(40)
    qd = S.base()
    S.query(204.0, 100.0, qd)
    a = S.kp(211.0, 100.0, S.cand(qd, 30))
    b = S.kp(197.0, 100.0, S.cand(qd, 30))
    S.kp(199.0, 101.0, S.cand(qd, 30))
    qd2 = S.base()
    S.query(400.0, 300.0, qd2)
    S.kp(400.0, 300.0, S.cand(qd2, 256))
    return [Case("best/ties_and_256", "best", [("tie", [(qd, S.k[a][3]), (qd, S.k[b][3])])], scene=S, radius=10.0,
                 levels=(0, 7))]


# ---------------------------------------------------------------------------------------------------------------------
# SearchByBoW (KF, F) and (KF, KF), SearchForInitialization
# ---------------------------------------------------------------------------------------------------------------------
def _bow_case(name, kind, nnratio, specs, seed):
    """specs: per node, the keyframe-side query distances list: [(d, ...)] -> one query per node with candidates at
    those distances on the other side, in that order."""
    rng = np.random.default_rng(seed)
    d1, d2, fv1, fv2 = [], [], {}, {}
    edges = []
    salt = seed * 1000
    for node, cands in enumerate(specs):
        qd = rng.integers(0, 256, 32, dtype=np.uint8)
        fv1[node * 2] = [len(d1)]
        d1.append(qd)
        fv2[node * 2] = []
        for d in cands:
            salt += 1
            c = flip(qd, d, salt)
            fv2[node * 2].append(len(d2))
            d2.append(c)
            edges.append(("dist", (qd, c, d)))
    a1 = np.full(len(d1), 100.0, f32)
    a2 = np.full(len(d2), 100.0, f32)
    kf = BowView(np.stack(d1), a1, fv1, valid=np.ones(len(d1), np.uint8))
    fr = BowView(np.stack(d2), a2, fv2, valid=np.ones(len(d2), np.uint8) if kind == "bow_kf" else None)
    return Case(name, kind, edges, kf=kf, fr=fr, nnratio=nnratio)


def bow_cases():
    out = []
    out.append(_bow_case("bow/th_low_50_51", "bow", 0.7, [[50], [51], [50, 256]], 50))
    out.append(_bow_case("bow_kf/th_low_49_50", "bow_kf", 0.7, [[49], [50], [49, 256]], 51))
    for kind in ("bow", "bow_kf"):
        c = _bow_case("%s/ratio_equality" % kind, kind, 0.75, [[45, 60], [60, 45], [44, 60], [45, 61], [30, 30, 40]], 52)
        c.edges.append(("ratio", (45, 60, 0.75)))
        out.append(c)
        out.append(_bow_case("%s/runner_up_256" % kind, kind, 0.3, [[40, 256], [256, 40]], 53))
    return out


def init_cases():
    """Level-0 keypoints of frame 1 search frame 2 around their previous position: TH_LOW at 50 / 51, the ratio at
    equality (strict '<'), an exact tie (rejected by the ratio), and a later query stealing an already matched keypoint
    with a strictly lower distance (its entry stays in the orientation histogram)."""
    S = Scene(60)
    pairs = []
    for j, cands in enumerate([[50], [51], [45, 60], [44, 60], [30, 30], [25]]):
        qd = S.base()
        x = 60.0 + 90.0 * j
        S.query(x, 100.0, qd, angle=100.0 + 40.0 * (j == 5))
        for e, d in enumerate(cands):
            pairs.append((j, S.kp(x + 2.0 * e - 1.0, 100.0, S.cand(qd, d)), d))
    stolen = pairs[-1][1]
    S.query(S.q[5]["u"] + 3.0, 100.0, flip(S.k[stolen][3], 20, 99))
    pairs.append((6, stolen, 20))
    q = S.q
    n1 = len(q)
    F1 = FrameView([p["u"] for p in q], [p["v"] for p in q], np.zeros(n1, np.int32), [p["angle"] for p in q],
                   np.full(n1, -1.0, f32), np.stack([p["desc"] for p in q]), np.eye(4, dtype=f32), FX, FY, CX, CY, BF,
                   *BOUNDS, SF)
    prev = np.stack([F1.x, F1.y], 1)
    edges = _dist_edges(S, pairs) + [("ratio", (45, 60, 0.75))]
    return [Case("init/thresholds_ratio_ties_steal", "init", edges, F1=F1, F2=S.frame(), prev=prev, window=10,
                 nnratio=0.75)]


# ---------------------------------------------------------------------------------------------------------------------
# SearchForTriangulation: bestDist starts at TH_LOW and a candidate at `dist <= bestDist` replaces the best (:896, :923),
# so ties go to the LAST minimum.  Keyframe 1 is stereo (no epipole gate); keyframe 2's keypoints sit on the epipolar
# line of their query unless stated otherwise.
# ---------------------------------------------------------------------------------------------------------------------
TRI_T1 = np.eye(4, dtype=f32)
TRI_T2 = np.eye(4, dtype=f32)
TRI_T2[:3, 3] = (0.3, 0.02, 0.05)


def tri_fundamental():
    """F12 with x1^T F12 x2 = 0 for TRI_T1, TRI_T2 (LocalMapping::ComputeF12: K^-T [t12]x R12 K^-1)."""
    from tests.members_gen import fundamental
    return fundamental(TRI_T1, TRI_T2)


def tri_cases():
    from orb_slam2_ssd_semantic_b200._abi import TriKFView
    F12 = tri_fundamental().astype(np.float64)
    rng = np.random.default_rng(70)
    salt = 70000
    x1, y1, d1, fv1 = [], [], [], {}
    x2, y2, d2, mp2, fv2 = [], [], [], [], {}
    # per node: the candidates' (distance, off the epipolar line, already holds a MapPoint), in node order
    specs = [[(50, 0, 0)], [(51, 0, 0)], [(30, 0, 0), (30, 0, 0), (31, 0, 0)], [(20, 0, 0), (25, 0, 0), (20, 0, 0)],
             [(40, 0, 0), (10, 1, 0)], [(35, 0, 0), (5, 0, 1), (35, 0, 0)], [(49, 0, 0), (50, 0, 0), (50, 0, 0)]]
    edges = []
    for node, cands in enumerate(specs):
        qd = rng.integers(0, 256, 32, dtype=np.uint8)
        px, py = 60.0 + 80.0 * node, 100.0 + 40.0 * (node % 3)
        fv1[node * 3] = [len(x1)]
        x1.append(px); y1.append(py); d1.append(qd)
        la, lb, lc = px * F12[0, 0] + py * F12[1, 0] + F12[2, 0], px * F12[0, 1] + py * F12[1, 1] + F12[2, 1], \
            px * F12[0, 2] + py * F12[1, 2] + F12[2, 2]
        fv2[node * 3] = []
        tie = []
        for e, (d, off, has) in enumerate(cands):
            salt += 1
            c = flip(qd, d, salt)
            xx = px - 30.0 + 7.0 * e
            fv2[node * 3].append(len(x2))
            x2.append(xx); y2.append(-(la * xx + lc) / lb + (25.0 if off else 0.0)); d2.append(c); mp2.append(has)
            edges.append(("dist", (qd, c, d)))
            if not off and not has and d == min(dd for dd, o, h in cands if not o and not h):
                tie.append((qd, c))
        if len(tie) > 1:
            edges.append(("tie", tie))
    n1, n2 = len(x1), len(x2)
    k1 = TriKFView(x1, y1, np.zeros(n1, np.int32), np.full(n1, 100.0, f32), np.array(x1, f32) - 20.0, np.stack(d1),
                   np.zeros(n1, np.uint8), fv1)
    k2 = TriKFView(x2, y2, np.zeros(n2, np.int32), np.full(n2, 100.0, f32), np.full(n2, -1.0, f32), np.stack(d2),
                   np.array(mp2, np.uint8), fv2)
    edges.append(("epipolar", (k1, k2)))
    cam = FrameView([0.0], [0.0], [0], [0.0], [-1.0], np.zeros((1, 32), np.uint8), TRI_T1, FX, FY, CX, CY, BF, *BOUNDS, SF)
    return [Case("tri/th_low_and_last_minimum_ties", "tri", edges, k1=k1, k2=k2, cam=cam)]


def tri_epipole():
    """(ex, ey) of keyframe 1's centre in keyframe 2 (:835-839), in float."""
    C2 = TRI_T2[:3, :3] @ (-TRI_T1[:3, :3].T @ TRI_T1[:3, 3]) + TRI_T2[:3, 3]
    invz = f32(f32(1.0) / f32(C2[2]))
    return (float(f32(f32(f32(FX) * f32(C2[0])) * invz) + f32(CX)), float(f32(f32(f32(FY) * f32(C2[1])) * invz) + f32(CY)))


def all_cases():
    return (last_cases() + points_cases() + projected_cases() + best_cases() + bow_cases() + init_cases() +
            tri_cases())


# ---------------------------------------------------------------------------------------------------------------------
# one entry point per implementation: "oracle" (oracle/ref.py, the flat CPU restatement), "refsrc" (the reference's own
# ORBmatcher.cc), "gpu" (ORBmatcher over the C-ABI)
# ---------------------------------------------------------------------------------------------------------------------
def run(case, impl, o=None, pad=0, epipole=None):
    kw = case.kw
    k = case.kind
    if impl == "gpu":
        from orb_slam2_ssd_semantic_b200 import ORBmatcher
    if k == "last":
        cur, last = last_views(case, pad)
        if impl == "gpu":
            return ORBmatcher(LAST_NNRATIO, kw["ori"]).SearchByProjection(cur, last, kw["th"], kw["mono"])
        f = o.search_by_projection_last if impl == "oracle" else o.src_search_by_projection_last
        return f(cur, last, kw["th"], kw["mono"], LAST_NNRATIO, kw["ori"])
    if k == "points":
        F, pts = kw["scene"].frame(), kw["scene"].points()
        if impl == "gpu":
            return ORBmatcher(kw["nnratio"], True).SearchByProjection(F, pts, kw["th"])
        f = o.search_by_projection_points if impl == "oracle" else o.src_search_by_projection_points
        return f(F, pts, kw["th"], kw["nnratio"])
    if k == "projected":
        S = kw["scene"]
        F, q = S.frame(with_obs=True), S.queries(kw["radius"], kw["levels"], uright=True)
        if impl == "gpu":
            return ORBmatcher(0.9, True).SearchProjected(F, q, kw["max_dist"], kw["rule"])
        return o.search_projected(F, q, kw["max_dist"], kw["rule"], True)
    if k == "best":
        S = kw["scene"]
        F, q = S.frame(), S.queries(kw["radius"], kw["levels"])
        if impl == "gpu":
            return ORBmatcher(0.9, True).SearchBest(F, q, 0)
        return o.search_best(F, q, 0)
    if k in ("bow", "bow_kf"):
        if impl == "gpu":
            m = ORBmatcher(kw["nnratio"], True)
            return (m.SearchByBoW if k == "bow" else m.SearchByBoWKF)(kw["kf"], kw["fr"])
        name = "search_by_bow" if k == "bow" else "search_by_bow_kf"
        return getattr(o, name if impl == "oracle" else "src_" + name)(kw["kf"], kw["fr"], kw["nnratio"], True)
    if k == "tri":
        k1, k2, F12 = kw["k1"], kw["k2"], tri_fundamental()
        epipole = tri_epipole() if epipole is None else epipole
        if impl == "gpu":
            return ORBmatcher(0.6, True).SearchForTriangulation(k1, k2, F12, epipole, SF, SF * SF, False)
        return o.search_for_triangulation(k1, k2, F12, epipole, SF, SF * SF, False, True)
    if k == "init":
        if impl == "gpu":
            return ORBmatcher(kw["nnratio"], True).SearchForInitialization(kw["F1"], kw["F2"], kw["prev"], kw["window"])
        f = o.search_for_initialization if impl == "oracle" else o.src_search_for_initialization
        return f(kw["F1"], kw["F2"], kw["prev"], kw["window"], kw["nnratio"], True)
    raise ValueError(k)
