"""Device == oracle, raw bits, on the crafted Frame-member cases of tests/frame_cases.py (the oracles are pinned to the
reference's own sources, to cv2 and to the DBoW2 stand-in by tests/test_frame_edges_cpu.py): orbm_is_in_frustum on all
six outputs, orbm_undistort_keypoints, the frame glue of track_batch / track_batch_u16 read back with
orbs_read_frame_glue, and orbv_transform raw and assembled.

One exception to raw bits: a float that is NaN on both sides counts as equal.  A case that reaches NaN (PcZ == +0.0
with PcX == 0 passes the u gate as NaN; +inf depth at u == cx) gets the device's canonical NaN 0x7fffffff there, and
x86 gives 0xffc00000."""
import os

import numpy as np
import pytest

from tests import frame_cases as FC
from tests.test_frame_edges_cpu import frustum_oracle, glue_inputs, glue_oracle
from tests.refpins import digest

pytestmark = pytest.mark.gpu

CASES = FC.all_cases()
FRUSTUM = [c for c in CASES if c.kind == "frustum"]
BOW = [c for c in CASES if c.kind == "bow"]


def _same_bits(name, got, ref):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape and got.dtype == ref.dtype, (name, got.shape, ref.shape, got.dtype, ref.dtype)
    if got.dtype.kind == "f":
        both_nan = np.isnan(got) & np.isnan(ref)
        bad = np.nonzero((got.view("u%d" % got.itemsize) != ref.view("u%d" % ref.itemsize)) & ~both_nan)
    else:
        bad = np.nonzero(got != ref)
    assert bad[0].size == 0, "%s: device %s, oracle %s at %s" % (name, got[bad], ref[bad], bad)


@pytest.fixture(scope="module")
def matcher():
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    return ORBmatcher(0.8, True)


@pytest.mark.parametrize("case", FRUSTUM, ids=[c.name for c in FRUSTUM])
def test_is_in_frustum_device_equals_oracle(oracle, matcher, case):
    kw = case.kw
    got = matcher.IsInFrustum(kw["F"], kw["xw"], kw["normal"], kw["mind"], kw["maxd"], float(kw["cos_limit"]), kw["lsf"])
    got = list(got[:4]) + [np.asarray(got[4])[~kw["undefined"]], got[5]]
    ref = frustum_oracle(oracle, case)
    for field, g, r in zip(("in_view", "proj_x", "proj_y", "proj_xr", "level", "view_cos"), got, ref):
        _same_bits("%s/%s" % (case.name, field), g, r)


@pytest.mark.parametrize("name,dist", FC.undistort_cases(), ids=[n for n, _ in FC.undistort_cases()])
def test_undistort_device_equals_oracle(oracle, matcher, name, dist):
    xy = FC.undistort_points()
    _same_bits(name, matcher.UndistortKeyPoints(xy, FC.UNDIST_K, dist), oracle.undistort(xy, FC.UNDIST_K, dist))


@pytest.mark.parametrize("u16", [False, True], ids=["float", "u16"])
def test_frame_glue_device_equals_oracle(oracle, u16):
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    gray, depth, d16, kps = glue_inputs(oracle, u16)
    st = StreamTracker(1000, 1.2, 8, 20, 7, FC.FX, FC.FY, FC.CX, FC.CY, FC.BF, 15.0, 0.9, True, 2)
    T = FC.GLUE_T[None]
    if u16:
        k, _, nkp, _, _ = st.track_batch_u16(gray[None], d16[None], FC.DEPTH_FACTOR, T)
    else:
        k, _, nkp, _, _ = st.track_batch(gray[None], depth[None], T)
    n = len(kps)
    assert nkp[0] == n and k[0, :n].tobytes() == kps.tobytes()
    ur, dp, xw, va = st.frame_glue(0, n)
    ref = glue_oracle(oracle, kps, depth)
    for field, g, r in zip(("uright", "depth", "valid", "xw"), (ur, dp, va, xw[va > 0]), ref):
        _same_bits("glue/%s" % field, g, r)


@pytest.mark.parametrize("case", BOW, ids=[c.name for c in BOW])
def test_bow_transform_device_equals_restatement(oracle, case):
    """orbv_transform per feature == the DBoW2 descent of tests/frame_cases.py at every levelsup the case names, and the
    assembled (BowVector, FeatureVector) == the same maps built from it; for word ids in leaf order also ==
    oracle.bow_transform_py, and at levelsup 4 == the reference's Frame::ComputeBoW on the shim ORBVocabulary where the
    shim library is built."""
    from orb_slam2_ssd_semantic_b200 import ORBVocabulary
    kw = case.kw
    voc = ORBVocabulary(kw["k"], kw["L"], kw["parent"], kw["node_desc"], kw["weight"], kw["word_id"])
    for ls in kw["levelsups"]:
        got = voc.transform_raw(kw["desc"], ls)
        want = FC.bow_expected_raw(case, ls)
        for field, g, r in zip(("word", "weight", "node"), got, want):
            _same_bits("%s/%d/%s" % (case.name, ls, field), g, r)
        maps = voc.transform(kw["desc"], ls)
        assert digest(maps) == digest(FC.assemble(*want)), (case.name, ls)
        if kw["word_id"] is None:
            args = (kw["k"], kw["L"], kw["parent"], kw["node_desc"], kw["weight"], kw["desc"])
            assert digest(maps) == digest(oracle.bow_transform_py(*args, levelsup=ls)), (case.name, ls)
            if ls == 4 and os.path.exists(oracle._SHIMSO):
                assert digest(oracle.src_bow_transform(*args, "shimsrc")) == digest(maps), case.name
