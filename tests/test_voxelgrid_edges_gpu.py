"""GPU: the crafted VoxelGrid cases of tests/voxelgrid_cases.py bit for bit against the CPU oracle -- gcm_refilter
(csrc/gcm.cu) against occ_ref_global_refilter round by round, and the semantic clusters' per-box grids (csrc/gcm_sem.cu)
against oracle/sem_ref.cpp, every GcmCluster field.  Where PCL's overflow test fires, gcm_refilter returns
B200ORB_EGEOM and the map holds the reference's unfiltered globalMap: the finite points, in insertion order; a later
refilter continues from there as the reference does."""
import numpy as np
import pytest

from oracle import sem_py
from orb_slam2_ssd_semantic_b200 import GlobalCloudMapping
from orb_slam2_ssd_semantic_b200._lib import B200OrbError
from tests import voxelgrid_cases as V

pytestmark = pytest.mark.gpu
B200ORB_EGEOM = -5
CASES = V.refilter_cases()
SEM = V.sem_cases()
_SEM_REF = {}


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_cloud(gx, gc, xyz, rgb):
    """Equal point lists: finite values and infinities bit for bit, NaN where NaN (its payload is the platform's)."""
    nan = np.isnan(xyz)
    return gx.shape == xyz.shape and (np.isnan(gx) == nan).all() and (_bits(gx)[~nan] == _bits(xyz)[~nan]).all() and \
        (gc == rgb).all()


def _refilter_and_check(gm, r):
    if r.overflow:
        with pytest.raises(B200OrbError) as e:
            gm.refilter()
        assert e.value.code == B200ORB_EGEOM
    else:
        gm.refilter()
    gx, gc = gm.points()
    assert gm.size() == len(r.out_xyz) == len(gx)
    assert (_bits(gx) == _bits(r.out_xyz)).all() and (gc == r.out_rgb).all()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_refilter_matches_oracle_bits(oracle, case):
    gm = GlobalCloudMapping(case.leaf)
    for k, (rnd, r) in enumerate(zip(case.rounds, V.expected_rounds(oracle, case))):
        for depth, bgr, T, fx, fy, cx, cy in rnd:
            gm.insertKeyFrame(T, depth, bgr, fx, fy, cx, cy)
        assert gm.size() == len(r.xyz)
        if k == 0:                                          # the appended cloud, before any refilter
            assert _same_cloud(*gm.points(), r.xyz, r.rgb)
        _refilter_and_check(gm, r)


def _rec(r):
    return (r.status, r.n_band, r.n_inliers, r.n_voxels, tuple(_bits(list(r.centroid) + list(r.min_pt) + list(r.max_pt))))


def _sem_ref(case):
    name, leaf, depth, bgr, T, fx, fy, cx, cy, objs = case
    if name not in _SEM_REF:
        _SEM_REF[name] = sem_py.keyframe(depth, bgr, T, fx, fy, cx, cy, 1, objs, leaf)
    return _SEM_REF[name]


@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("case", SEM, ids=[c[0] for c in SEM])
def test_semantic_boxes_match_oracle_bits(oracle, case, entry):
    name, leaf, depth, bgr, T, fx, fy, cx, cy, objs = case
    gm = GlobalCloudMapping(leaf)
    if entry == "host":
        recs = gm.insertKeyFrameObjects(T, depth, bgr, fx, fy, cx, cy, 1, objs)
    else:
        import torch
        d, c = torch.from_numpy(depth).cuda(), torch.from_numpy(bgr).cuda()
        torch.cuda.synchronize()
        recs = gm.insert_keyframe_objects_device(d.data_ptr(), c.data_ptr(), depth.shape[0], depth.shape[1], T, fx, fy, cx,
                                                 cy, 1, objs)
    ref_recs, _, (xyz, rgb) = _sem_ref(case)
    assert [_rec(r) for r in recs] == [_rec(r) for r in ref_recs]
    assert _same_cloud(*gm.points(), xyz, rgb)
    _refilter_and_check(gm, V.refilter_round(oracle, xyz, rgb, leaf))
