"""The two CPU restatements of the occupancy path, oracle/occ_ref.cpp and oracle/occ_py.py, bit for bit on the crafted
scenes of occ_scenes.py: points, labels, leaf keys and log-odds, and for the single-ray scenes computeRayKeys itself.
These are the edges the GPU is compared on (test_occupancy_geometry_gpu.py), so the oracle is pinned there first."""
import numpy as np
import pytest

from tests import occ_scenes as S


def canon(a):
    """float32 bits with every NaN made the same NaN (x86 keeps a NaN's payload, the GPU writes the canonical one)."""
    a = np.asarray(a, np.float32)
    return np.where(np.isnan(a), np.float32(np.nan), a).view(np.uint32)


def ref_for(oracle, s):
    return oracle.RefOccupancy(**s.params)


@pytest.mark.parametrize("make", S.SCENES, ids=lambda f: f.__name__)
def test_oracle_restatements_agree_on_crafted_scene(oracle, make):
    s = make()
    ref, py = ref_for(oracle, s), s.py()
    n_ref = ref.insert_keyframe(s.T, s.depth, s.rgb, *s.cam, s.label)
    n_py = py.insert_keyframe(s.T, s.depth, *s.cam, s.label)
    pts, _, lab = ref.last_points()
    assert n_ref == n_py == len(pts) > 0
    assert (canon(pts) == canon(py.points)).all() and (lab == py.labels).all()
    keys, lo = ref.export_leaves()
    got = {tuple(int(v) for v in k): x for k, x in zip(keys, lo)}
    assert got.keys() == py.leaves.keys()
    assert all(canon(got[k]) == canon(py.leaves[k]) for k in got)
    if s.single_ray:
        r_ref, r_py = ref.ray(s.origin, s.end), py.ray_keys(s.origin, s.end)
        assert (r_ref is None) == (r_py is None)
        if r_py is not None:
            assert [tuple(int(v) for v in k) for k in r_ref] == r_py
            assert {k for k, v in got.items() if v < 0} == set(r_py)      # the ray's cells are the free leaves


def test_scene_expectations(oracle):
    """What each family of scenes is for, stated on the oracle's output."""
    # gates: the points at exactly depth_min / depth_max are kept, one ULP outside and 0, -1, +-inf are not
    s = S.gates_depth()
    ref = ref_for(oracle, s)
    ref.insert_keyframe(s.T, s.depth, s.rgb, *s.cam, s.label)
    pts = {tuple(p) for p in ref.last_points()[0].tolist()}
    assert all(tuple(p.tolist()) in pts for p in s.expect_kept)
    assert len(pts) == int(((s.depth >= 0.5) & (s.depth <= 3.0)).sum())
    s = S.gates_y()
    ref = ref_for(oracle, s)
    ref.insert_keyframe(s.T, s.depth, s.rgb, *s.cam, s.label)
    ys = ref.last_points()[0][:, 1]
    assert (ys == 3.0).sum() == 1 and (ys == -3.0).sum() == 1 and np.abs(ys).max() == 3.0
    # origin outside the key range: occupied endpoints, no free cells
    s = S.origin_outside_key_range()
    ref = ref_for(oracle, s)
    ref.insert_keyframe(s.T, s.depth, s.rgb, *s.cam, s.label)
    _, lo = ref.export_leaves()
    assert len(lo) == int(((s.depth > 0) & (s.label == 0)).sum()) and (lo > 0).all()
    # ends outside the key range: only the rays of the points inside it
    s = S.ends_outside_key_range()
    ref = ref_for(oracle, s)
    ref.insert_keyframe(s.T, s.depth, s.rgb, *s.cam, s.label)
    _, lo = ref.export_leaves()
    inside = {tuple(k) for n in (72, 80) for k in ref.ray(s.origin, s.world_point(72, n)).tolist()}
    assert (lo < 0).all() and len(lo) == len(inside) > 10000
    # NaN: never a key, never a leaf at the key NaN would convert to
    for make in S.NONFINITE:
        s = make()
        ref = ref_for(oracle, s)
        ref.insert_keyframe(s.T, s.depth, s.rgb, *s.cam, s.label)
        pts = ref.last_points()[0]
        keys, _ = ref.export_leaves()
        assert np.isnan(pts).any(axis=1).sum() == (len(pts) if s.name == "nan-pose" else 1), s.name
        assert not (keys == 32768).all(axis=1).any(), s.name
        if s.name in ("nan-alone", "nan-pose"):
            assert len(keys) == 0, s.name
    # the VoxelGrid cell (0, 0, 0) keeps its real point next to NaN pixels
    s = S.nan_mixed(True)
    ref = ref_for(oracle, s)
    ref.insert_keyframe(s.T, s.depth, s.rgb, *s.cam, s.label)
    assert (ref.last_points()[0] == s.world_point(72, 72)).all(axis=1).any()


def test_batch_sequence_is_long_enough():
    seq = S.sequence()
    assert len(seq) > 32 and len({s.name for s in seq}) > 20
    assert all(s.depth.shape == seq[0].depth.shape and s.cam == seq[0].cam for s in seq)
