"""Deterministic crafted cases for the T variant's two VoxelGrid passes (PCL VoxelGrid::applyFilter as restated by
oracle/occ_ref.cpp and oracle/sem_ref.cpp): the refilter of the whole accumulated map (gcm_refilter, csrc/gcm.cu) and
the per-box grids of the semantic clusters (gcm_add_keyframe_objects, csrc/gcm_sem.cu).  Each case is named after the
edge it makes observable; tests/test_voxelgrid_edges_cpu.py recomputes in float32 numpy that it really contains it.

Arbitrary map points come from 1x1 keyframes: depth d, cx = cy = 0, R = I and translation t give the point
(-t0, -t1, d - t2).  A refilter case is a list of rounds, each a list of keyframes (depth, bgr, Tcw, fx, fy, cx, cy) that
are added before one refilter; the expected input is always taken from oracle.backproject_all, never from the formula."""
import numpy as np

from tests import sem_scenes

f32 = np.float32
INT_MAX = 2 ** 31 - 1
INF = f32(np.inf)


def up(x, n=1):
    for _ in range(n):
        x = np.nextafter(f32(x), INF)
    return f32(x)


def down(x, n=1):
    for _ in range(n):
        x = np.nextafter(f32(x), -INF)
    return f32(x)


def inv_of(leaf):
    """1.0f / leaf, as gcm_refilter and the oracles compute it."""
    return f32(1.0) / f32(leaf)


class Case:
    def __init__(self, name, leaf, rounds):
        self.name, self.leaf, self.rounds = name, f32(leaf), rounds


def point_kf(x, y, z, rgb=(0, 0, 0), fx=1.0, fy=1.0, cx=0.0, cy=0.0):
    """A 1x1 keyframe whose one pixel back-projects to (x, y, z) (for finite x, y, z)."""
    T = np.eye(4, dtype=np.float32)
    T[0, 3], T[1, 3] = -f32(x), -f32(y)
    bgr = np.array([[[rgb[2], rgb[1], rgb[0]]]], np.uint8)
    return (np.array([[z]], np.float32), bgr, T, fx, fy, cx, cy)


def _colours(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, 3)).astype(np.uint8)


def points_round(pts, seed=0):
    pts = np.asarray(pts, np.float32).reshape(-1, 3)
    return [point_kf(*p, rgb=c) for p, c in zip(pts, _colours(len(pts), seed))]


# --------------------------------------------------------------------------------------------------------------------
# cell boundaries

def boundary_x(k, inv):
    """A float x with x * inv exactly the integer k in float32 (None if no float near k / inv has it)."""
    x0 = f32(f32(k) / inv)
    for x in [x0] + [up(x0, i) for i in range(1, 64)] + [down(x0, i) for i in range(1, 64)]:
        if f32(x * inv) == f32(k):
            return x
    return None


def boundary_values(leaf, sign):
    """Boundary floats x (x * inv integral) and their float neighbours on both sides."""
    inv = inv_of(leaf)
    out = []
    for k in (1, 2, 3, 7, 10, 25, 26, 99, 100, 1001, 12345):
        x = boundary_x(sign * k, inv)
        if x is not None:
            out += [down(x), x, up(x)]
    return np.array(out, np.float32)


def boundary_case(leaf, sign):
    v = boundary_values(leaf, sign)
    inv = inv_of(leaf)
    c = f32(sign * f32(0.5) / inv)            # a cell centre on the other axes
    pts = [(x, c, c) for x in v] + [(c, x, c) for x in v] + [(c, c, x) for x in v]
    name = "cell_boundaries_leaf%s_%s" % (("%g" % leaf).replace(".", "p"), "neg" if sign < 0 else "pos")
    return Case(name, leaf, [points_round(pts, seed=len(v))])


# --------------------------------------------------------------------------------------------------------------------
# negative coordinates, floor against truncation, signed zeros

def negative_cases():
    rng = np.random.default_rng(5)
    leaf = f32(0.05)
    inv = inv_of(leaf)
    neg = rng.uniform(-3.3, -0.01, (160, 3)).astype(np.float32)
    edges = np.array([boundary_x(-k, inv) for k in (1, 2, 20, 33)], np.float32)
    neg = np.concatenate([neg, np.stack([edges, edges, edges], 1), np.stack([down(edges), up(edges), edges], 1)])
    assert (neg < 0).all()
    a = f32(0.04)
    ia = inv_of(a)
    # |x * inv| < 1 on both sides of zero: floor gives cells -1 and 0, truncation gives 0 for both
    frac = [f32(s * f / ia) for s in (-1, 1) for f in (0.1, 0.3, 0.7, 0.97)]
    mixed = [(x, y, z) for x in frac for y in frac[::3] for z in frac[::2]]
    mixed += [(boundary_x(-1, ia), f32(0.01), f32(0.01)), (boundary_x(1, ia), f32(-0.01), f32(0.01))]
    zeros = [
        (np.array([[f32(-0.0)]], np.float32), np.array([[[9, 8, 7]]], np.uint8), np.eye(4, dtype=np.float32), 1.0, 1.0, 0.0, 0.0),
        (np.array([[f32(0.0)]], np.float32), np.array([[[1, 2, 3]]], np.uint8), np.eye(4, dtype=np.float32), 1.0, 1.0, 0.0, 0.0),
    ]   # depth -0.0 with t = 0 back-projects to (-0, -0, -0), depth +0.0 to (+0, +0, +0)
    return [Case("negative_map_floor_not_truncation", leaf, [points_round(neg, seed=1)]),
            Case("mixed_sign_min_b_negative", a, [points_round(mixed, seed=2)]),
            Case("signed_zeros_one_cell", a, [zeros + points_round([(f32(-0.3) / ia, f32(0.2) / ia, f32(-0.9) / ia)], seed=3)])]


# --------------------------------------------------------------------------------------------------------------------
# floor(x * inv) - (float)min_b rounds beyond 2^24: a tie to even merges two cells that int arithmetic keeps apart

def float_sub_cases():
    out = []
    # min_b = 1 and floors of 2^24 + 2j: floor - 1.0 is odd, halfway between two floats of spacing 2
    xs = [f32(1.5)] + [f32(2 ** 24 + 2 * j) for j in range(1, 8)]
    pts = [(x, f32(0.5), f32(0.5)) for x in xs] + [(f32(2 ** 24 + 4), f32(1.5), f32(2.5))]
    out.append(Case("float_sub_ties_min_b_small", 1.0, [points_round(pts, seed=4)]))
    # min_b = 2^24 + 2 and floors of 2^25 + 2^24 + 4j: the differences are 2 mod 4, halfway between floats of spacing 4
    m = f32(2 ** 24 + 2)
    xs = [m] + [f32(2 ** 25 + 2 ** 24 + 4 * j) for j in range(1, 9)]
    pts = [(x, f32(1.25), f32(0.75)) for x in xs] + [(xs[3], f32(0.25), f32(1.75))]
    out.append(Case("float_sub_ties_min_b_beyond_2p24", 1.0, [points_round(pts, seed=5)]))
    # the same at leaf 0.5 (inv 2), on the y axis
    xs = [f32(0.75)] + [f32((2 ** 24 + 2 * j) / 2) for j in range(1, 8)]
    pts = [(f32(0.25), y, f32(0.25)) for y in xs]
    out.append(Case("float_sub_ties_y_leaf0p5", 0.5, [points_round(pts, seed=6)]))
    return out


# --------------------------------------------------------------------------------------------------------------------
# PCL's overflow test: dx*dy*dz = (long long)((max - min) * inv) + 1 per axis, against INT_MAX

def overflow_cases():
    out = []
    # the largest reachable product <= INT_MAX: INT_MAX is prime, one axis of INT_MAX needs a float in [2^31-2, 2^31-1)
    # (there is none), so 2^31 - 2 = 32767 * 32769 * 2
    lo = [(0.0, 0.0, 0.0), (32766.5, 32768.5, 1.5), (16000.25, 3.0, 0.5), (0.0, 32768.5, 1.5), (32766.5, 0.0, 0.0),
          (32766.0, 32768.0, 1.0), (32765.99, 32767.99, 0.99)]
    out.append(Case("overflow_test_product_int_max_minus_1", 1.0, [points_round(lo, seed=7)]))
    # the smallest product above INT_MAX: 2^31 = 2048 * 2048 * 512; NaN points among them leave the map, the rest stays
    # in insertion order; a second and a third round keep overflowing
    hi = points_round([(0.0, 0.0, 0.0), (1.0, 2.0, 3.0), (2047.5, 2047.5, 511.5), (2047.5, 0.0, 0.0)], seed=8)
    nan = point_kf(0.0, 0.0, np.nan)
    hi = [hi[0], nan, hi[1], hi[2], nan, hi[3], nan]
    out.append(Case("overflow_test_product_2p31", 1.0,
                    [hi, points_round([(5.5, 6.5, 7.5), (0.25, 0.25, 0.25)], seed=9) + [nan],
                     points_round([(100.0, 100.0, 100.0)], seed=10)]))
    # div_b exceeds d on every axis: points just inside the first and the last cell (x * inv = k + 0.9 ... m + 0.1)
    leaf = f32(0.04)
    inv = inv_of(leaf)
    a, b = f32(0.9) / inv, f32(10.1) / inv
    pts = [(a, a, a), (b, b, b), (a, b, a), (b, a, b), ((a + b) / 2, a, b)]
    pts += [(f32(k + 0.5) / inv, f32(k + 0.25) / inv, f32(k + 0.75) / inv) for k in range(1, 10)]
    out.append(Case("div_b_exceeds_d_first_and_last_cells", leaf, [points_round(pts, seed=11)]))
    # a clean round, then a far point makes the second refilter overflow: the map is the first round's centroids and the
    # new finite points, in order; a third round continues from there
    rng = np.random.default_rng(12)
    r1 = points_round(rng.uniform(0.0, 0.3, (40, 3)), seed=12)
    r2 = points_round([(0.05, 0.05, 0.05), (2000.0, 2000.0, 0.1)], seed=13) + [nan]
    r3 = points_round(rng.uniform(0.0, 0.3, (5, 3)), seed=14)
    out.append(Case("overflow_after_a_clean_round", leaf, [r1, r2, r3]))
    # an overflowing grid whose div_b products, if formed, wrap the second point's 32-bit key onto the all-ones no-cell
    # key: div_b = (65536, 65536, 2), div_b[0] * div_b[1] wraps to 0, 65535 + 65535 * 65536 = 2^32 - 1.  PCL forms no
    # key here and keeps every point; a second round continues from all three
    wrap = points_round([(0.5, 0.5, 0.5), (65535.5, 65535.5, 1.5), (3.5, 3.5, 0.5)], seed=20)
    out.append(Case("overflow_key_wraps_to_no_cell", 1.0, [wrap + [nan], points_round([(7.5, 7.5, 1.25)], seed=21)]))
    return out


# --------------------------------------------------------------------------------------------------------------------
# a cell whose linear index is INT_MAX, the value of the old non-finite marker

def int_max_cell_points(leaf):
    """P1, P2 with div_b = (128, 2^23, 2) and P2 in the last cell: index 127 + (2^23 - 1) * 128 + 2^30 = 2^31 - 1, while
    dx * dy * dz stays <= INT_MAX."""
    inv = inv_of(leaf)

    def at(k, frac):   # a float x with floor(x * inv) == k and x * inv about k + frac
        x = f32(f32(k + frac) / inv)
        while np.floor(f32(x * inv)) > k:
            x = down(x)
        while np.floor(f32(x * inv)) < k:
            x = up(x)
        return x
    p1 = (at(0, 0.75), at(0, 0.75), at(0, 0.75))
    p2 = (at(127, 0.25), at(2 ** 23 - 1, 0.0), at(1, 0.25))
    return p1, p2


def int_max_cases():
    out = []
    for leaf in (f32(1.0), f32(0.04)):
        p1, p2 = int_max_cell_points(leaf)
        out.append(Case("cell_index_int_max_leaf%s" % ("%g" % leaf).replace(".", "p"), leaf, [points_round([p1, p2], seed=15)]))
    p1, p2 = int_max_cell_points(f32(1.0))
    nan = point_kf(0.0, 0.0, np.nan)
    kf = points_round([p1, p2, (0.5, 0.5, 0.5), p2], seed=16)
    out.append(Case("cell_index_int_max_next_to_nan", 1.0, [[nan, kf[0], nan, kf[1], kf[2], nan, kf[3], nan]]))
    return out


# --------------------------------------------------------------------------------------------------------------------
# non-finite points

def _kf(depth, fx=1.0, fy=1.0, cx=0.0, cy=0.0, t=(0.0, 0.0, 0.0), rgb=(10, 20, 30), R=None):
    T = np.eye(4, dtype=np.float32)
    T[:3, 3] = t
    if R is not None:
        T[:3, :3] = R
    return (np.array([[depth]], np.float32), np.array([[[rgb[2], rgb[1], rgb[0]]]], np.uint8), T, fx, fy, cx, cy)


def nonfinite_cases():
    nan = [_kf(np.nan), _kf(np.nan, t=(1.0, 2.0, 3.0))]
    # cx = cy = -1 makes (0 - cx) * d / fx = d, so depth +-inf gives px = py = pz = +-inf; every entry of R is 1, since a
    # zero entry times an infinity would be NaN: the points are (+-inf, +-inf, +-inf) with no NaN
    ones = np.ones((3, 3), np.float32)
    inf = [_kf(np.inf, cx=-1.0, cy=-1.0, R=ones), _kf(-np.inf, cx=-1.0, cy=-1.0, R=ones),
           _kf(np.inf, cx=-1.0, cy=-1.0, t=(4.0, 5.0, 6.0), R=ones)]
    # an infinite pixel offset: (0 - (-1)) * 3e38 / 0.5 overflows float, and through R = I the point is (inf, NaN, NaN)
    one_axis = [_kf(3.0e38, fx=0.5, cx=-1.0, t=(0.0, -1.0, 0.0))]
    fin = points_round([(0.1, 0.2, 0.3), (0.11, 0.21, 0.31), (-0.5, 0.5, 1.5), (2.0, -2.0, 0.5)], seed=17)
    mixed = [nan[0], fin[0], inf[0], one_axis[0], fin[1], fin[2], nan[1], inf[1], fin[3]]
    return [Case("only_nan_gives_no_points", 0.05, [nan]), Case("only_inf_gives_no_points", 0.05, [inf]),
            Case("mixed_nonfinite_dropped", 0.05, [mixed]),
            Case("only_nan_then_finite", 0.05, [nan, fin])]


# --------------------------------------------------------------------------------------------------------------------
# tiny maps, one large cell, chained refilters

def small_cases():
    single = points_round([(0.123, -4.5, 2.25)], seed=18)
    leaf = f32(0.05)
    inv = inv_of(leaf)
    c = [f32((k + 0.5) / inv) for k in (3, -2, 7)]
    # five points of one cell; colour sums 499 / 5 = 99.8 and 254 * 4 + 253 -> averages just below an integer
    pts = [(c[0] + f32(0.001) * i, c[1] - f32(0.002) * i, c[2] + f32(0.0015) * i) for i in range(5)]
    cols = [(100, 254, 7), (100, 254, 3), (100, 254, 1), (100, 254, 250), (99, 253, 0)]
    one = [point_kf(*p, rgb=cl) for p, cl in zip(pts, cols)]
    return [Case("single_point", 0.05, [single]), Case("single_cell_truncated_colour", leaf, [one])]


def big_cell_keyframe(side=363):
    """One keyframe of side^2 >= 2^17 pixels, every one in the cell [0, 1)^3 at leaf 1.0: x, y in (0.04, 0.96), so the
    float sums of x and y depend on their order; r averages just below 100, b holds odd values above 2^24 in its sum."""
    n = side * side
    depth = np.full((side, side), 0.5, np.float32)
    depth[::7, ::5] = np.float32(0.75)
    T = np.eye(4, dtype=np.float32)
    T[0, 3], T[1, 3] = -0.5, -0.5
    r = np.full(n, 100, np.uint8)
    r[n // 2] = 99
    g = np.full(n, 126, np.uint8)
    g[::3] = 125
    b = np.full(n, 255, np.uint8)
    b[1::2] = 253
    bgr = np.stack([b, g, r], 1).reshape(side, side, 3)
    return (depth, bgr, T, 300.0, 300.0, (side - 1) / 2.0, (side - 1) / 2.0)


def large_cases():
    kf = big_cell_keyframe()
    rng = np.random.default_rng(19)
    rows, cols = 24, 32
    rounds = []
    for k in range(3):
        depth = rng.uniform(0.8, 1.6, (rows, cols)).astype(np.float32)
        depth[3, 4 + k] = np.nan
        bgr = rng.integers(0, 256, (rows, cols, 3)).astype(np.uint8)
        T = np.eye(4, dtype=np.float32)
        T[:3, 3] = (0.01 * k, -0.02 * k, 0.03 * k)
        rounds.append([(depth, bgr, T, 40.0, 41.0, 15.5, 11.5)])
    return [Case("one_cell_of_131769_points", 1.0, [[kf]]), Case("chained_three_rounds", 0.05, rounds)]


def refilter_cases():
    out = [boundary_case(leaf, s) for leaf in (0.04, 0.05, 0.03, 1.0) for s in (1, -1)]
    out += negative_cases() + float_sub_cases() + overflow_cases() + int_max_cases() + nonfinite_cases()
    out += small_cases() + large_cases()
    return out


# --------------------------------------------------------------------------------------------------------------------
# the semantic clusters' per-box VoxelGrid: (name, leaf, depth, bgr, Tcw, fx, fy, cx, cy, objects)

def sem_int_max_box():
    """Box 0 of 7 x 8 band pixels: 28 at depth 0 (the camera centre A = (0.75, 0.5, 0)) and 28 at depth 0.25, which an
    affine Tcw (third row 506, 33554428, 5) sends to B = (127.25, 8388607.5, 1.25).  fx = fy = 1e30 keeps the pixel
    offsets below half an ulp.  Both groups are the other's 50 neighbours alike, so SOR keeps all 56, and at leaf 1 B's
    cell index is 127 + 8388607 * 128 + 2^30 = INT_MAX with dx*dy*dz = 127 * 2^23 * 2."""
    rows, cols = 8, 10
    depth = np.zeros((rows, cols), np.float32)
    depth[:7, 4:8] = 0.25
    bgr = np.full((rows, cols, 3), 60, np.uint8)
    T = np.eye(4, dtype=np.float32)
    T[2, :3] = (506.0, 33554428.0, 5.0)
    T[0, 3], T[1, 3] = -0.75, -0.5
    return ("sem_box0_cell_index_int_max", f32(1.0), depth, bgr, T, 1e30, 1e30, 0.0, 0.0, [(1.0, 1.0, 10.0, 8.0, 9, 0.9)])


def sem_negative_zero_overflow():
    """A tiny leaf overflows the box's grid, so PCL hands back its inliers themselves.  Depth -(c - cx) * 0.02 puts every
    point at x <= 0; column cx has depth -0.0 and back-projects to (-0, -0, -0) from the first band row on, so the box's
    max_pt.x is -0.0."""
    rows, cols, cx = 16, 24, 10
    c = np.arange(cols, dtype=np.float32)
    depth = np.tile(-(c - f32(cx)) * f32(0.02), (rows, 1)).astype(np.float32)
    depth[:, cx] = f32(-0.0)
    bgr = np.full((rows, cols, 3), 90, np.uint8)
    return ("sem_overflow_keeps_negative_zero", f32(1e-4), depth, bgr, np.eye(4, dtype=np.float32), 1.0, 1.0, float(cx), 0.0,
            [(1.0, 1.0, 24.0, 15.0, 15, 0.8)])


def sem_plane_on_boundaries():
    """A fronto-parallel plane at depth 2.0 with fx = fy = 40 at leaf 0.05 (inv 20): z * inv = 40 exactly, and x, y =
    float(k * 2 / 40) put x * inv on or next to the integer k -- every voxel centroid sits on a cell boundary."""
    rows, cols = 100, 140
    depth = np.full((rows, cols), 2.0, np.float32)
    bgr = np.full((rows, cols, 3), 30, np.uint8)
    T = np.eye(4, dtype=np.float32)
    return ("sem_plane_on_cell_boundaries", f32(0.05), depth, bgr, T, 40.0, 40.0, 70.0, 50.0,
            [(20.0, 15.0, 100.0, 70.0, 20, 0.9), (60.0, 40.0, 30.0, 30.0, 5, 0.7)])


def sem_tiny_leaf_room():
    depth, bgr, T, objs = sem_scenes.scene("overlap")
    from orb_slam2_ssd_semantic_b200 import synth
    return ("sem_tiny_leaf_every_box_overflows", f32(1e-6), depth, bgr, T, synth.FX, synth.FY, synth.CX, synth.CY, objs)


def sem_cases():
    return [sem_int_max_box(), sem_negative_zero_overflow(), sem_plane_on_boundaries(), sem_tiny_leaf_room()]


# --------------------------------------------------------------------------------------------------------------------
# what the reference's globalMap holds after each refilter

class Round:
    """One refilter round: the map before it (non-finite points included, as the device holds them), whether PCL's
    overflow test fires, and globalMap after it."""

    def __init__(self, xyz, rgb, overflow, out_xyz, out_rgb):
        self.xyz, self.rgb, self.overflow, self.out_xyz, self.out_rgb = xyz, rgb, overflow, out_xyz, out_rgb


def refilter_round(oracle, xyz, rgb, leaf):
    """VoxelGrid over the map; where the index space overflows PCL hands the input back, and the reference's input never
    held a non-finite point (removeNaNFromPointCloud before "*globalMap += ..."): its finite points, in order."""
    try:
        ox, oc = oracle.global_refilter(xyz, rgb, leaf)
        return Round(xyz, rgb, False, ox, oc)
    except ValueError:
        fin = np.isfinite(xyz).all(1)
        return Round(xyz, rgb, True, xyz[fin], rgb[fin])


def expected_rounds(oracle, case):
    acc_x, acc_c = np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8)
    out = []
    for rnd in case.rounds:
        for depth, bgr, T, fx, fy, cx, cy in rnd:
            acc_x = np.concatenate([acc_x, oracle.backproject_all(depth, T, fx, fy, cx, cy)])
            acc_c = np.concatenate([acc_c, bgr.reshape(-1, 3)[:, ::-1]])
        r = refilter_round(oracle, acc_x, acc_c, case.leaf)
        out.append(r)
        acc_x, acc_c = r.out_xyz, r.out_rgb
    return out
