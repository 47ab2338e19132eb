"""VoxelGrid binning against the C++ oracle, bit for bit (points as sets of byte rows with their rgb, leaves by key and by
the bits of their log-odds), on keyframes that stress k_ocm_bin's per-CTA pixel tiles: one cell spread over several
tiles and tile rows, tiles where every pixel is its own cell (with and without NaN speckle), a keyframe that is a single
cell, frame sizes that are not multiples of the tile, one launch of 32 keyframes with very different cell counts, and
clouds of 49 and 50 cells made of many more pixels (the all-ground rule of fewer than 50 points counts cells)."""
import numpy as np
import pytest

from tests import occ_scenes as S
from tests.test_occupancy_geometry_gpu import assert_same_map, point_rows

pytestmark = pytest.mark.gpu

F32 = np.float32
TILE_W, TILE_H = 32, 16   # k_ocm_bin's tile (BIN_TW x BIN_TH)
INV_LEAF = F32(1) / F32(0.01)


def cells(s):
    """VoxelGrid cell of every gated pixel (leaf_key with float32 arithmetic; all scenes here keep y inside y_max and
    NaN out unless asked), -> (rows, cols, 3) int64 with -1 where the pixel is gated out or not finite."""
    rows, cols = s.depth.shape
    m, n = np.mgrid[0:rows, 0:cols]
    z = s.depth
    x = ((n.astype(F32) - F32(s.cx)) * z) / F32(s.fx)
    y = ((m.astype(F32) - F32(s.cy)) * z) / F32(s.fy)
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(z) & (z >= F32(0.5)) & (z <= F32(3.0))
        c = np.stack([np.floor(v * INV_LEAF) for v in (x, y, z)], axis=-1)
    return np.where(ok[..., None], c, np.nan)


def distinct(c):
    v = c.reshape(-1, 3)
    v = v[~np.isnan(v).any(axis=1)]
    return len(np.unique(v, axis=0))


def check(oracle, s):
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    gpu = PointCloudMapping(map_capacity=s.capacity, **s.params)
    ref = oracle.RefOccupancy(**s.params)
    gpu.insertKeyFrame(s.T, s.depth, s.rgb, *s.cam, s.label)
    ref.insert_keyframe(s.T, s.depth, s.rgb, *s.cam, s.label)
    pg, cg = gpu.last_points()
    pr, cr, _ = ref.last_points()
    assert len(pg) == len(pr) > 0
    assert (point_rows(pg, cg) == point_rows(pr, cr)).all()
    assert_same_map(gpu, ref)
    return gpu, len(pr)


def _label(rng, shape):
    return rng.integers(0, 2, shape).astype(np.uint8)


def cell_over_many_tiles():
    """fx = 4096 at z ~ 0.5: a 1-cm cell is ~80 pixels wide, so each cell collects groups from several tiles and tile
    rows, joined by the atomicAdd of the leaf table in an arbitrary order; the summation order shows in the centroid."""
    rng = np.random.default_rng(31)
    rows, cols = 100, 150
    depth = (0.5 + rng.integers(0, 8192, (rows, cols)) * F32(2 ** -20)).astype(F32)
    s = S.Scene("cell-over-many-tiles", depth, _label(rng, (rows, cols)), (0.0, 0.0, 0.0), {"resolution": S.RES},
                f=4096.0, c=60.0, seed=31)
    c = cells(s)
    key = c[..., 0] * 1e6 + c[..., 1] * 1e3 + c[..., 2]
    m, n = np.mgrid[0:rows, 0:cols]
    spans = [(len(np.unique(n[key == k] // TILE_W)), len(np.unique(m[key == k] // TILE_H))) for k in np.unique(key)]
    assert max(a for a, _ in spans) >= 3 and max(b for _, b in spans) >= 3
    vals = ((n.astype(F32) - F32(60)) * depth / F32(4096))[key == key[50, 70]]   # row-major order
    assert np.cumsum(vals, dtype=F32)[-1] != np.cumsum(vals[::-1], dtype=F32)[-1]
    return s


def every_pixel_own_cell(nan_fraction=0.0):
    """fx = 64 at z ~ 2: neighbouring pixels are 3 cm apart, so every gated pixel of a tile is a cell of its own (and NaN
    pixels share one more)."""
    rng = np.random.default_rng(32)
    depth = (2.0 + rng.integers(0, 1024, (S.ROWS, S.COLS)) * F32(2 ** -10)).astype(F32)
    depth[rng.random((S.ROWS, S.COLS)) < nan_fraction] = S.NAN
    s = S.Scene("every-pixel-own-cell-nan%g" % nan_fraction, depth, _label(rng, depth.shape), (0.0, 0.0, 0.0),
                {"resolution": S.RES}, capacity=1 << 18, seed=32)
    finite = np.isfinite(depth)
    assert distinct(cells(s)) == finite.sum() and (nan_fraction == 0) == finite.all()
    return s


def one_cell():
    """fx = 65536, principal point at the corner: every pixel of the 40 x 48 keyframe falls into one cell, which is also a
    cloud of one point (all ground)."""
    rng = np.random.default_rng(33)
    depth = (0.505 + rng.integers(0, 64, (40, 48)) * F32(2 ** -20)).astype(F32)
    s = S.Scene("one-cell", depth, _label(rng, depth.shape), (0.0, 0.0, 0.0), {"resolution": S.RES}, f=65536.0, c=0.0,
                seed=33)
    assert distinct(cells(s)) == 1
    return s


def odd_size(rows, cols, seed):
    """Frame sizes that are not multiples of the tile: gated-out holes, depths over the whole gate."""
    rng = np.random.default_rng(seed)
    depth = rng.uniform(0.5, 3.0, (rows, cols)).astype(F32)
    depth[rng.random((rows, cols)) < 0.2] = 0.0
    s = S.Scene("odd-%dx%d" % (rows, cols), depth, _label(rng, depth.shape), (0.0, 0.0, 0.0), {"resolution": S.RES},
                f=40.0, c=cols / 2.0, seed=seed)
    assert rows % TILE_H and cols % TILE_W and distinct(cells(s)) >= 50
    return s


TILE_SCENES = [cell_over_many_tiles, every_pixel_own_cell, lambda: every_pixel_own_cell(0.3), one_cell,
               lambda: odd_size(37, 53, 34), lambda: odd_size(17, 100, 35), lambda: odd_size(49, 33, 36)]
TILE_IDS = ["cell_over_many_tiles", "every_pixel_own_cell", "every_pixel_own_cell_nan_speckle", "one_cell", "odd_37x53",
            "odd_17x100", "odd_49x33"]


@pytest.mark.parametrize("make", TILE_SCENES, ids=TILE_IDS)
def test_tile_scene_bit_equal_to_oracle(oracle, make):
    s = make()
    check(oracle, s)


def fifty_rule(ncells):
    """`ncells` cells of 9 pixels each (3 x 3 blocks at fx = 1024, z = 1: 1 mm apart), all labelled non-ground: below 50
    cells the cloud is all ground (free rays, no occupied leaf), at 50 it is not, although both have > 50 pixels."""
    depth = np.zeros((S.ROWS, S.COLS), F32)
    label = np.zeros((S.ROWS, S.COLS), np.uint8)
    s = S.Scene("fifty-rule-%d" % ncells, depth, label, (0.0, 0.0, 0.0), {"resolution": S.RES}, f=1024.0, seed=37)
    placed = 0
    for m0 in range(2, S.ROWS - 3, 12):
        for n0 in range(2, S.COLS - 3, 12):
            if placed == ncells:
                break
            depth[m0:m0 + 3, n0:n0 + 3] = 1.0
            if distinct(cells(s)) != placed + 1:   # the block straddles a cell face: leave it out
                depth[m0:m0 + 3, n0:n0 + 3] = 0.0
                continue
            placed += 1
    assert placed == ncells and distinct(cells(s)) == ncells and (depth > 0).sum() == 9 * ncells
    return s


@pytest.mark.parametrize("ncells", [49, 50])
def test_fewer_than_50_points_counts_cells_not_pixels(oracle, ncells):
    gpu, npts = check(oracle, fifty_rule(ncells))
    assert npts == ncells
    _, lo, _ = gpu.export_leaves()
    if ncells < 50:
        assert (lo < 0).all() and len(lo) > 0
    else:
        assert (lo > 0).all() and len(lo) > 0


def test_batch_of_32_keyframes_with_different_cell_counts(oracle):
    """One launch round of 32 keyframes (75 x 90, not a multiple of the tile) whose cell counts run from 1 to every
    pixel: the map equals the oracle's sequential inserts, the last keyframe's cloud equals the oracle's, and the round's
    point count is the sum of the oracle's."""
    import torch
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    rows, cols, n = 75, 90, 32
    rng = np.random.default_rng(38)
    depth = np.zeros((n, rows, cols), F32)
    for i in range(n):
        kind = i % 4
        if kind == 0:     # one flat patch: few cells
            depth[i, 10:10 + 2 * i, 20:40] = 1.5
        elif kind == 1:   # random depths over a fraction of the frame growing with i
            mask = rng.random((rows, cols)) < (i + 1) / n
            depth[i][mask] = rng.uniform(0.5, 3.0, mask.sum())
        elif kind == 2:   # every pixel valid, far apart
            depth[i] = rng.uniform(2.0, 3.0, (rows, cols))
        else:             # a handful of pixels
            depth[i, ::25, ::30] = 1.0 + 0.01 * i
    rgb = rng.integers(0, 256, (n, rows, cols, 3), dtype=np.uint8)
    label = rng.integers(0, 2, (n, rows, cols)).astype(np.uint8)
    cam = (40.0, 40.0, 45.0, 37.0)
    T = np.repeat(np.eye(4, dtype=F32)[None], n, axis=0)
    T[:, :3, 3] = rng.uniform(-0.5, 0.5, (n, 3)).astype(F32)
    ref = oracle.RefOccupancy(resolution=S.RES)
    counts = []
    for i in range(n):
        ref.insert_keyframe(T[i], depth[i], rgb[i], *cam, label[i])
        counts.append(len(ref.last_points()[0]))
    assert min(counts) <= 3 and max(counts) > 50 * min(counts) and len(set(counts)) > 10
    gpu = PointCloudMapping(S.RES, map_capacity=1 << 18)
    d, c, lb = (torch.from_numpy(x).cuda() for x in (depth, rgb, label))
    gpu.insert_keyframes_device(d.data_ptr(), c.data_ptr(), rows, cols, list(range(n)), T, *cam, d_label=lb.data_ptr())
    gpu.sync()
    assert_same_map(gpu, ref)
    pg, cg = gpu.last_points()
    pr, cr, _ = ref.last_points()
    assert (point_rows(pg, cg) == point_rows(pr, cr)).all()
    assert gpu.last_batch_stats()[0] == sum(counts)
