"""Crafted keyframes for the occupancy path, shared by test_occupancy_geometry_cpu.py (C++ oracle against the Python
restatement) and test_occupancy_geometry_gpu.py (GPU against the C++ oracle).

Every scene is one keyframe whose geometry is exact in float32: a small image, fx = fy a power of two and an integer
principal point (so (n - cx) * z / fx is exact), the identity rotation, depth 0 except at the chosen pixels and an
explicit ground-label image.  With the identity rotation a world point is p_c - t, and the ray origin is t itself (the
sensor-origin quirk of UpdateOctomap: the translation of Tcw, not the camera centre).  Each scene asserts the premise it
exists for, so that it cannot silently stop testing it."""
from __future__ import annotations

import math

import numpy as np

from oracle.occ_py import PyOccupancy

F32 = np.float32
ROWS = COLS = 144
C0 = 72.0            # cx = cy of the standard camera
F = 64.0             # fx = fy of the standard camera
RES = 0.0625         # a power of two: voxel faces are exact, and so are the borders of computeRayKeys
NAN = F32(np.nan)


class Scene:
    def __init__(self, name, depth, label, t, params=None, f=F, c=C0, single_ray=False, capacity=1 << 16, seed=0):
        self.name = name
        self.depth = np.ascontiguousarray(depth, F32)
        rows, cols = self.depth.shape
        self.rgb = np.random.default_rng(seed).integers(0, 256, (rows, cols, 3), dtype=np.uint8)
        self.label = None if label is None else np.ascontiguousarray(label, np.uint8)
        self.T = np.eye(4, dtype=F32)
        self.T[:3, 3] = np.asarray(t, F32)
        self.fx = self.fy = float(f)
        self.cx = self.cy = float(c)
        self.params = dict(params or {})     # OcmParams fields other than the defaults
        self.single_ray = single_ray         # exactly one point, on a fresh map: the free leaves are oracle.ray(origin, end)
        self.capacity = capacity

    @property
    def origin(self):
        return self.T[:3, 3].copy()

    @property
    def cam(self):
        return self.fx, self.fy, self.cx, self.cy

    def camera_point(self, m, n):
        z = F32(self.depth[m, n])
        return np.array([F32(F32(F32(n) - F32(self.cx)) * z) / F32(self.fx),
                         F32(F32(F32(m) - F32(self.cy)) * z) / F32(self.fy), z], F32)

    def world_point(self, m, n):
        """p_c - t, asserted exact (the oracle transforms in double and rounds once)."""
        p = self.camera_point(m, n).astype(np.float64) - self.origin.astype(np.float64)
        assert (p.astype(F32).astype(np.float64) == p).all(), (self.name, m, n)
        return p.astype(F32)

    def py(self):
        """The Python restatement with this scene's parameters."""
        keep = ("resolution", "depth_min", "depth_max", "y_max", "leaf")
        return PyOccupancy(**{k: v for k, v in self.params.items() if k in keep})

    def res(self):
        return float(self.params.get("resolution", 0.05))


def _blank(rows=ROWS, cols=COLS):
    return np.zeros((rows, cols), F32), np.zeros((rows, cols), np.uint8)


def _key(s, p):
    return s.py().point_key(p)


def _on_face(s, c):
    """c lies on a voxel face: the double keyToCoord border of its cell, minus half a voxel, is c itself."""
    res = s.res()
    k = s.py().coord_to_key(c)
    return (float(k - 32768) + 0.5) * res - float(F32(res * 0.5)) == float(c)


def _single(name, m, n, d, t=(0.0, 0.0, 0.0), res=RES, **params):
    depth, label = _blank()
    depth[m, n] = d
    label[m, n] = 1
    s = Scene(name, depth, label, t, {"resolution": res, **params}, single_ray=True, seed=m * COLS + n)
    s.end = s.world_point(m, n)
    return s


# ---- rays (single ground point on a fresh map: the free leaves are exactly the oracle's computeRayKeys) -------------
def ray_axis_z(sign=1):
    if sign > 0:
        s = _single("ray+z", 72, 72, 2.0)                         # (0, 0, 0) -> (0, 0, 2)
    else:
        s = _single("ray-z", 72, 72, 1.0, t=(0.0, 0.0, 3.0))      # (0, 0, 3) -> (0, 0, -2)
    d = s.end - s.origin
    assert d[0] == 0 and d[1] == 0 and np.sign(d[2]) == sign     # step 0 on x and y: tMax = DBL_MAX, which overflows
    return s


def ray_plane(axis, sign):
    m, n = (72, 72 + sign * 32) if axis == "x" else (72 + sign * 32, 72)
    s = _single("ray-%s%s-plane" % ("+" if sign > 0 else "-", axis), m, n, 2.0)
    d = s.end - s.origin
    other = 1 if axis == "x" else 0
    assert d[other] == 0 and np.sign(d[0 if axis == "x" else 1]) == sign and d[2] > 0
    return s


def ray_diag2(sign, res=RES):
    s = _single("ray-diag2%s-res%g" % ("+" if sign > 0 else "-", res), 72 + sign * 32, 72 + sign * 32, 2.0, res=res)
    d = s.end - s.origin
    assert d[0] == d[1] and d[0] * sign > 0 and d[2] != d[0]    # dir_x == dir_y: tMax[0] and tMax[1] tie at every step
    return s


def ray_diag3(sign, res=RES):
    s = _single("ray-diag3%s-res%g" % ("+" if sign > 0 else "-", res), 72 + sign * 64, 72 + sign * 64, 2.0, res=res)
    d = s.end - s.origin
    assert abs(d[0]) == abs(d[1]) == abs(d[2]) and d[0] == d[1] and np.sign(d[0]) == sign   # n - cx = fx: a 3-way tie
    return s


def ray_origin_corner_negative():
    """Origin on a voxel corner, stepping down on x and y: both tMax start at exactly -0 (t = 0) and tie."""
    s = _single("ray-origin-corner-neg", 40, 40, 2.0)
    res = s.res()
    border = (float(s.py().coord_to_key(0.0) - 32768) + 0.5) * res + float(F32(-res * 0.5))
    assert (s.origin == 0).all() and border == 0.0 and (s.end[:2] < 0).all()
    return s


def ray_origin_on_face():
    s = _single("ray-origin-face", 72 + 16, 72 + 32, 2.0, t=(3 * RES, 2 ** -6, 2 ** -7))
    assert _on_face(s, s.origin[0]) and not _on_face(s, s.origin[1]) and not _on_face(s, s.origin[2])
    return s


def ray_end_on_corner():
    """Origin and end both on voxel corners (everything a multiple of the resolution)."""
    s = _single("ray-end-corner", 72 + 16, 72 + 48, 2.0, t=(2 * RES, RES, 4 * RES))
    assert all(_on_face(s, c) for c in s.end) and all(_on_face(s, c) for c in s.origin)
    return s


def ray_origin_inside_cell():
    s = _single("ray-origin-inside", 72 + 21, 72 + 38, 2.5, t=(2 ** -7, 2 ** -6, 3 * 2 ** -7), res=0.05)
    assert not any(_on_face(s, c) for c in s.origin)
    return s


def ray_end_in_origin_cell():
    s = _single("ray-end-in-origin-cell", 72, 72, 0.6, t=(0.0, 0.0, 0.3))
    assert _key(s, s.end) == _key(s, s.origin)                 # no ray at all
    return s


def ray_end_in_next_cell():
    s = _single("ray-end-in-next-cell", 72, 72, 0.6 + RES, t=(0.0, 0.0, 0.3))
    ko, ke = _key(s, s.origin), _key(s, s.end)
    assert sum(abs(a - b) for a, b in zip(ko, ke)) == 1         # the ray is the origin's cell alone
    return s


def ray_exits_on_distance():
    """The walk steps past the end cell: the loop ends on the distance test, not on reaching the end key."""
    s = _single("ray-exits-on-distance", 72 + 32, 72 + 32, 2.0, t=(RES, 0.0, 0.0))
    ray = s.py().ray_keys(s.origin, s.end)
    ke = _key(s, s.end)
    assert ray and sum(abs(a - b) for a, b in zip(ray[-1], ke)) != 1
    return s


def ray_long():
    """More cells than the scan kernel's per-CTA cache of free cells (SCAN_CACHE = 2048)."""
    s = _single("ray-long", 72 + 64, 72 + 64, 2.0, res=0.001)
    s.capacity = 1 << 20
    assert len(s.py().ray_keys(s.origin, s.end)) > 2048
    return s


def ray_long_axis():
    s = _single("ray-long-axis", 72, 72, 3.0, res=0.001)
    s.capacity = 1 << 20
    assert len(s.py().ray_keys(s.origin, s.end)) > 2048
    return s


def ray_end_outside_key_range():
    """resolution 5e-5: the key range is +-1.6384 m, the end lies beyond it, the origin inside."""
    s = _single("ray-end-outside-range", 72 + 8, 72, 2.0, res=5e-5)
    py = s.py()
    assert _key(s, s.origin) is not None and _key(s, s.end) is None and py.ray_keys(s.origin, s.end) is None
    return s


def _named(name, f, *args):
    g = lambda: f(*args)   # noqa: E731
    g.__name__ = name
    return g


# factories (scenes are built inside the tests, so a failing premise fails a test rather than the collection)
RAYS = [_named("ray_+z", ray_axis_z, 1), _named("ray_-z", ray_axis_z, -1), _named("ray_+x_plane", ray_plane, "x", 1),
        _named("ray_-x_plane", ray_plane, "x", -1), _named("ray_+y_plane", ray_plane, "y", 1),
        _named("ray_-y_plane", ray_plane, "y", -1), _named("ray_diag2_+", ray_diag2, 1), _named("ray_diag2_-", ray_diag2, -1),
        _named("ray_diag2_+_res0.05", ray_diag2, 1, 0.05), _named("ray_diag2_-_res0.05", ray_diag2, -1, 0.05),
        _named("ray_diag3_+", ray_diag3, 1), _named("ray_diag3_-", ray_diag3, -1),
        _named("ray_diag3_+_res0.05", ray_diag3, 1, 0.05), ray_origin_corner_negative, ray_origin_on_face,
        ray_end_on_corner, ray_origin_inside_cell, ray_end_in_origin_cell, ray_end_in_next_cell, ray_exits_on_distance,
        ray_long, ray_long_axis, ray_end_outside_key_range]


# ---- many rays ------------------------------------------------------------------------------------------------------
def rays_many(ground_all=False):
    """A grid of isolated pixels (>= 50 points): axis, plane and diagonal directions among them; ground-labelled
    pixels cast rays, the others are occupied endpoints."""
    depth, label = _blank()
    for m in range(8, 137, 8):
        for n in range(8, 137, 8):
            depth[m, n] = 1.0 + 0.25 * ((m // 8 + n // 8) % 7)
            label[m, n] = 1 if ground_all or (m // 8 + n // 8) % 3 != 2 else 0
    s = Scene("rays-many" + ("-all-ground" if ground_all else ""), depth, label, (0.0, 0.0, 0.0), {"resolution": RES}, seed=3)
    p = s.world_point(136, 136)
    assert (depth > 0).sum() >= 50 and label[72, 72] and label[136, 136] and label[16, 16] and p[0] == p[1] == p[2]
    assert 0 < (label[depth > 0] == 0).sum() or ground_all
    return s


def rays_sparse_nonground():
    """< 50 points, all labelled non-ground: the cloud is all ground anyway (MapDrawer.cc:676)."""
    depth, label = _blank()
    for i, (m, n) in enumerate([(8 + 11 * k, 136 - 11 * k) for k in range(12)] + [(72, 72)]):
        depth[m, n] = 0.75 + 0.125 * i
    s = Scene("rays-sparse-nonground", depth, label, (0.0, 0.0, 0.0), {"resolution": 0.05}, seed=4)
    assert 0 < (depth > 0).sum() < 50 and label.max() == 0
    return s


def origin_outside_key_range():
    """t = (0, 0, 1640) at resolution 0.05 (key range +-1638.4 m) with depth ~1641 m: the points lie near world z = 1,
    inside the key range, the origin outside it.  No free cells; the occupied endpoints are still inserted."""
    depth, label = _blank()
    for m in range(12, 133, 10):
        for n in range(12, 133, 10):
            depth[m, n] = 1640.5 + 0.25 * ((m + n) % 5)
            label[m, n] = (m // 10 + n // 10) % 3 == 0
    s = Scene("origin-outside-range", depth, label, (0.0, 0.0, 1640.0), {"depth_max": 2000.0, "y_max": 2000.0}, seed=5)
    py = s.py()
    assert py.point_key(s.origin) is None and (depth > 0).sum() >= 50 and 0 < label.sum() < (depth > 0).sum()
    assert all(py.point_key(s.world_point(m, n)) is not None for m, n in zip(*np.nonzero(depth)))
    return s


def ends_outside_key_range():
    depth, label = _blank()
    depth[8:136:8, 8:136:8] = 2.0           # outside +-1.6384 m
    depth[72, 72] = 0.5                     # inside: one ray of 10000 cells
    depth[72, 80] = 0.75
    label[::2, :] = 1
    s = Scene("ends-outside-range", depth, label, (0.0, 0.0, 0.0), {"resolution": 5e-5}, capacity=1 << 20, seed=6)
    py = s.py()
    assert py.point_key(s.world_point(8, 8)) is None and py.point_key(s.world_point(72, 72)) is not None
    assert label[72, 72] and not label[72 - 1, 72] and (depth > 0).sum() >= 50
    return s


# ---- gates ----------------------------------------------------------------------------------------------------------
def _fill_valid(depth, label, rows=range(20, 124, 6), cols=range(20, 124, 6)):
    for m in rows:
        for n in cols:
            depth[m, n] = 1.0 + 0.0625 * ((m + n) % 9)
            label[m, n] = (m * n) % 4 == 0


def gates_depth():
    depth, label = _blank()
    _fill_valid(depth, label)
    kept = {(10, 10): 0.5, (10, 20): 3.0}
    dropped = {(11, 10): np.nextafter(F32(0.5), F32(0)), (11, 20): np.nextafter(F32(3.0), F32(4)), (12, 10): 0.0,
               (12, 20): -1.0, (13, 10): np.inf, (13, 20): -np.inf, (14, 10): -0.0}
    for (m, n), d in {**kept, **dropped}.items():
        depth[m, n] = d
    s = Scene("gates-depth", depth, label, (0.0, 0.0, 0.0), seed=7)
    assert F32(np.nextafter(F32(0.5), F32(0))) < F32(0.5) and F32(np.nextafter(F32(3.0), F32(4))) > F32(3.0)
    s.expect_kept = [s.world_point(m, n) for m, n in kept]
    return s


def gates_y():
    """y exactly +-y_max (m - cy = +-fx, z = 3) is kept; one ULP beyond (z = 3 + ulp, so y = 3 + ulp) is dropped."""
    depth, label = _blank()
    _fill_valid(depth, label)
    z1 = np.nextafter(F32(3.0), F32(4))
    for m in (72 - 64, 72 + 64):
        depth[m, 30] = 3.0
        depth[m, 90] = z1
    s = Scene("gates-y", depth, label, (0.0, 0.0, 0.0), {"depth_max": 4.0}, seed=8)
    assert s.camera_point(8, 30)[1] == -3.0 and s.camera_point(136, 30)[1] == 3.0
    assert s.camera_point(136, 90)[1] == z1 > F32(3.0) and s.camera_point(8, 90)[1] == -z1
    return s


# ---- VoxelGrid cells --------------------------------------------------------------------------------------------------
def cells_around_zero():
    """Pixels on both sides of the principal point: x and y of both signs, floor of negatives."""
    depth, label = _blank()
    depth[60:85, 60:85] = 0.8
    depth[62, 70] = 0.8125
    label[60:85, 60:72] = 1
    s = Scene("cells-around-zero", depth, label, (0.0, 0.0, 0.0), seed=9)
    xs = [s.camera_point(72, n)[0] for n in range(60, 85)]
    assert min(xs) < 0 < max(xs) and any(x == 0 for x in xs)
    return s


def cells_integer_boundary():
    """x * inv_leaf, y * inv_leaf and z * inv_leaf exact integers (x = +-0.5, z = 2): points on cell faces."""
    depth, label = _blank()
    _fill_valid(depth, label)
    for m, n in ((72, 88), (72, 56), (88, 72), (56, 72), (88, 88), (56, 56)):
        depth[m, n] = 2.0
        depth[m + 1, n] = 2.0
    s = Scene("cells-integer-boundary", depth, label, (0.0, 0.0, 0.0), seed=10)
    inv = F32(1.0) / F32(0.01)
    for m, n in ((72, 88), (72, 56), (88, 72)):
        p = s.camera_point(m, n)
        assert all(float(F32(c * inv)) == math.floor(float(F32(c * inv))) for c in p)
    return s


def cells_crowded(rows=256, cols=256):
    """fx = fy = 4096 at z ~ 0.5: thousands of pixels per 1-cm cell, over many warps and CTAs, so the summation order of
    a cell decides its centroid's last bits."""
    rng = np.random.default_rng(12)
    depth = (0.5 + rng.integers(0, 8192, (rows, cols)) * F32(2 ** -20)).astype(F32)
    label = np.zeros((rows, cols), np.uint8)
    label[:, cols // 2:] = 1
    s = Scene("cells-crowded", depth, label, (0.0, 0.0, 0.0), f=4096.0, c=128.0, seed=11)
    ys, xs = np.mgrid[0:rows, 0:cols]
    x = ((xs.astype(F32) - F32(128)) * depth) / F32(4096)
    cell = np.floor(x * (F32(1) / F32(0.01))).astype(np.int64)
    sel = (cell == 0) & (np.floor((ys.astype(F32) - F32(128)) * depth / F32(4096) * (F32(1) / F32(0.01))) == 0)
    vals = x[sel]          # row-major order
    assert sel.sum() > 2000
    fwd = np.cumsum(vals, dtype=F32)[-1]
    rev = np.cumsum(vals[::-1], dtype=F32)[-1]
    assert fwd != rev      # the order of the sum shows in the centroid
    return s


# ---- non-finite depth and pose ----------------------------------------------------------------------------------------
T_OFF = (0.3125, 0.1875, 0.125)   # an origin whose key is not 32768 on any axis (the key NaN would convert to)


def nan_alone():
    depth, label = _blank()
    for m, n in ((20, 30), (20, 31), (90, 100), (130, 5)):
        depth[m, n] = NAN
    label[20, 30] = 1
    s = Scene("nan-alone", depth, label, T_OFF, seed=13)
    assert np.isnan(depth).sum() == 4 and (depth > 0).sum() == 0 and 32768 not in _key(s, s.origin)
    return s


def nan_mixed(first_ground):
    """>= 50 valid points plus NaN pixels; the NaN cell's label is that of its first pixel.  depth_min below 1 cm with a
    valid point in VoxelGrid cell (0, 0, 0): NaN pixels must not land in it."""
    depth, label = _blank()
    _fill_valid(depth, label)
    for m, n in ((5, 7), (5, 8), (60, 61), (140, 2)):
        depth[m, n] = NAN
    label[5, 7] = 1 if first_ground else 0
    label[60, 61] = 0 if first_ground else 1
    depth[72, 72] = 2 ** -8
    s = Scene("nan-mixed-%s" % ("ground" if first_ground else "nonground"), depth, label, T_OFF, {"depth_min": 0.001},
              seed=14 + first_ground)
    p = s.camera_point(72, 72)
    assert (np.floor(p * (F32(1) / F32(0.01))) == 0).all() and (depth > 0).sum() >= 50
    return s


def nan_sparse():
    depth, label = _blank()
    for k in range(10):
        depth[10 + 12 * k, 20 + 9 * k] = 0.75 + 0.125 * k
    depth[3, 3] = depth[100, 50] = NAN
    s = Scene("nan-sparse", depth, label, T_OFF, seed=16)
    assert (depth > 0).sum() + 1 < 50
    return s


def nan_pose():
    depth, label = _blank()
    _fill_valid(depth, label)
    s = Scene("nan-pose", depth, label, (0.0, np.nan, 0.5), seed=17)
    assert np.isnan(s.origin[1]) and (depth > 0).sum() >= 50 and 0 < label.sum()
    return s


NONFINITE = [nan_alone, _named("nan_mixed_ground", nan_mixed, True), _named("nan_mixed_nonground", nan_mixed, False),
             nan_sparse, nan_pose]


# ---- the VoxelGrid key range --------------------------------------------------------------------------------------------
LEAF_POW2 = 2.0 ** -6          # inv_leaf = 64 exactly
Z_AT_BOUND = float(np.nextafter(F32(2 ** 20 / 64), F32(0)))   # z * inv_leaf = 2^20 - 1/16: the largest accepted depth_max


def leaf_range_at_bound(depth_max=Z_AT_BOUND):
    """The largest depth_max whose VoxelGrid cells cannot alias (|z / leaf| < 2^20); x and y stay far below (8 x 8
    image, |n - cx| <= 4 < fx).  Resolution 1 m keeps the points inside the octree key range."""
    depth = np.full((8, 8), F32(depth_max), F32)
    depth[::3, ::2] = 1000.0
    label = np.zeros((8, 8), np.uint8)
    s = Scene("leaf-range-at-bound", depth, label, (0.0, 0.0, 0.0),
              {"resolution": 1.0, "leaf": LEAF_POW2, "depth_max": depth_max, "y_max": 1e9}, c=4.0, seed=18)
    assert F32(F32(depth_max) * F32(64)) < 2 ** 20 <= F32(np.nextafter(F32(depth_max), F32(np.inf)) * F32(64))
    assert (depth > 0).sum() >= 50
    return s


rays_many_all_ground = _named("rays_many_all_ground", rays_many, True)
SCENES = RAYS + [rays_many, rays_many_all_ground, rays_sparse_nonground, origin_outside_key_range, ends_outside_key_range,
                 gates_depth, gates_y, cells_around_zero, cells_integer_boundary, cells_crowded] + NONFINITE + \
    [leaf_range_at_bound]


def sequence():
    """> 32 keyframes of the standard camera, inserted under one parameter set (resolution RES) for the batched path:
    rays of every direction, repeated keyframes (hits and misses run into the clamps, so the replay order shows), gates
    and NaN pixels."""
    out = []
    for f in RAYS + [rays_many, rays_many_all_ground, gates_depth, cells_around_zero, cells_integer_boundary] + NONFINITE:
        s = f()
        if s.depth.shape == (ROWS, COLS) and s.fx == F and s.params.get("resolution", RES) == RES and \
                not (set(s.params) - {"resolution"}):
            out.append(s)
    out += [rays_many(), rays_many_all_ground(), rays_many()] * 4
    assert len(out) > 32
    return out
