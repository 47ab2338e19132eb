"""GPU occupancy path against the C++ oracle, bit for bit, on the crafted scenes of occ_scenes.py: gates at their exact
bounds, VoxelGrid cells on both sides of 0, on integer boundaries and crowded over many warps, rays along the axes and
the exact diagonals (tMax ties), from voxel corners and faces, longer than the scan kernel's cache, with the origin or
the end outside the key range, and NaN depth or pose.  Points are compared as sets of rows of bytes (with their rgb),
leaves by key and by the bits of their log-odds; a single-ray keyframe on a fresh map must free exactly the cells of
the oracle's computeRayKeys."""
import numpy as np
import pytest

from tests import occ_scenes as S

pytestmark = pytest.mark.gpu


def canon(a):
    a = np.asarray(a, np.float32)
    return np.where(np.isnan(a), np.float32(np.nan), a).view(np.uint32)


def point_rows(xyz, rgb):
    rows = np.concatenate([canon(xyz).reshape(-1, 3), np.asarray(rgb, np.uint32).reshape(-1, 3)], axis=1)
    return rows[np.lexsort(rows.T[::-1])]


def leaf_bits(keys, lo):
    k = keys.astype(np.uint64)
    packed = k[:, 0] | (k[:, 1] << np.uint64(16)) | (k[:, 2] << np.uint64(32))
    o = np.argsort(packed)
    return packed[o], np.asarray(lo, np.float32)[o].view(np.uint32)


def assert_same_map(gpu, ref):
    (kg, vg), (kr, vr) = leaf_bits(*gpu.export_leaves()[:2]), leaf_bits(*ref.export_leaves())
    assert len(kg) == len(kr) and (kg == kr).all()
    assert (vg == vr).all()
    assert gpu.num_leaves() == len(kr)


def _gpu(s, **over):
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    return PointCloudMapping(map_capacity=s.capacity, **{**s.params, **over})


@pytest.mark.parametrize("make", S.SCENES, ids=lambda f: f.__name__)
def test_crafted_scene_bit_equal_to_oracle(oracle, make):
    s = make()
    gpu, ref = _gpu(s), oracle.RefOccupancy(**s.params)
    gpu.insertKeyFrame(s.T, s.depth, s.rgb, *s.cam, s.label)
    ref.insert_keyframe(s.T, s.depth, s.rgb, *s.cam, s.label)
    pg, cg = gpu.last_points()
    pr, cr, _ = ref.last_points()
    assert len(pg) == len(pr) > 0
    assert (point_rows(pg, cg) == point_rows(pr, cr)).all()
    assert_same_map(gpu, ref)
    keys, lo, _ = gpu.export_leaves()
    if s.single_ray:
        ray = ref.ray(s.origin, s.end)
        want = set() if ray is None else {tuple(k) for k in ray.tolist()}
        assert {tuple(k) for k in keys[lo < 0].tolist()} == want and (lo < 0).all()
    if np.isnan(pr).any() or np.isnan(s.origin).any():
        assert gpu.query(np.full(3, np.nan, np.float32)) is None
        for p in pr[np.isnan(pr).any(axis=1)]:
            assert gpu.query(p) is None
        assert not (keys == 32768).all(axis=1).any()      # the key a NaN coordinate converts to on the GPU


def test_batched_sequence_equals_sequential_inserts(oracle):
    """More than 32 crafted keyframes (two rounds of the batch masks) in one insert_keyframes_device call == the same
    keyframes one insertKeyFrame at a time == the oracle, bit for bit; repeated keyframes drive voxels into both
    clamps, so the keyframe-order replay of k_ocm_apply is what keeps the values equal."""
    import torch
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    seq = S.sequence()
    n = len(seq)
    seq_map = PointCloudMapping(S.RES, map_capacity=1 << 16)
    ref = oracle.RefOccupancy(resolution=S.RES)
    for s in seq:
        seq_map.insertKeyFrame(s.T, s.depth, s.rgb, *s.cam, s.label)
        ref.insert_keyframe(s.T, s.depth, s.rgb, *s.cam, s.label)
    assert_same_map(seq_map, ref)
    depth = torch.from_numpy(np.stack([s.depth for s in seq])).cuda()
    rgb = torch.from_numpy(np.stack([s.rgb for s in seq])).cuda()
    label = torch.from_numpy(np.stack([s.label for s in seq])).cuda()
    T = np.stack([s.T for s in seq])
    batch = PointCloudMapping(S.RES, map_capacity=1 << 16)
    batch.insert_keyframes_device(depth.data_ptr(), rgb.data_ptr(), S.ROWS, S.COLS, list(range(n)), T, *seq[0].cam,
                                  d_label=label.data_ptr())
    batch.sync()
    assert_same_map(batch, ref)
    pb, cb = batch.last_points()
    ps, cs = seq_map.last_points()
    assert (point_rows(pb, cb) == point_rows(ps, cs)).all()
    hit, miss, cmin, cmax = ref.constants()
    _, lo = ref.export_leaves()
    assert (lo == cmin).sum() > 100 and (lo == cmax).sum() > 10 and n > 32


def test_voxelgrid_key_range_is_refused_one_step_past_the_bound(oracle):
    """The VoxelGrid cell key has 21 bits per axis.  depth_max one float step below 2^20 leaves is accepted (and equal to
    the oracle: test_crafted_scene_bit_equal_to_oracle[leaf_range_at_bound]); 2^20 leaves exactly is refused, and so are
    intrinsics that let x reach it, a non-finite gate, and the batched device path."""
    import torch
    from orb_slam2_ssd_semantic_b200._lib import B200OrbError
    s = S.leaf_range_at_bound()
    past = dict(s.params, depth_max=2.0 ** 20 * S.LEAF_POW2)
    ok = _gpu(s)
    ok.insertKeyFrame(s.T, s.depth, s.rgb, *s.cam, s.label)
    assert ok.num_leaves() > 50
    for params, cam in ((past, s.cam), (s.params, (2.0 ** -10, s.fy, s.cx, s.cy)), (dict(s.params, depth_max=np.inf), s.cam),
                        (dict(s.params, depth_min=np.nan), s.cam)):
        with pytest.raises(B200OrbError) as e:
            _gpu(s, **params).insertKeyFrame(s.T, s.depth, s.rgb, *cam, s.label)
        assert e.value.code == -1 and "2^20" in str(e.value)
    g = _gpu(s, **past)
    d, c = torch.from_numpy(s.depth[None]).cuda(), torch.from_numpy(s.rgb[None]).cuda()
    with pytest.raises(B200OrbError) as e:
        g.insert_keyframes_device(d.data_ptr(), c.data_ptr(), 8, 8, [0], s.T[None], *s.cam)
    assert e.value.code == -1
    assert g.num_leaves() == 0
