"""GPU: the semantic object clusters (gcm_add_keyframe_objects[_device], csrc/gcm_sem.cu) bit for bit against the CPU
oracle (oracle/sem_ref.cpp) on the crafted room scenes of tests/sem_scenes.py -- every GcmCluster field, the painted
colours and world points of the appended cloud (pixel order, before the refilter) and globalMap after the refilter --
plus the skip rule over a keyframe sequence and the C++ shim overload against the Python mirror's cluster database."""
import os
import struct
import subprocess

import numpy as np
import pytest

from oracle import sem_py
from orb_slam2_ssd_semantic_b200 import GlobalCloudMapping, SemanticClusters, synth
from orb_slam2_ssd_semantic_b200._abi import GCM_BELOW_PROB, GCM_CLUSTER, GCM_FEW_POINTS
from tests import sem_scenes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = (synth.FX, synth.FY, synth.CX, synth.CY)
LEAF = sem_scenes.LEAF
_REF = {}


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _rec(r):
    return (r.status, r.n_band, r.n_inliers, r.n_voxels, tuple(_bits(list(r.centroid) + list(r.min_pt) + list(r.max_pt))))


def _oracle(name, i=1):
    if (name, i) not in _REF:
        depth, bgr, T, objs = sem_scenes.scene(name)
        _REF[(name, i)] = sem_py.keyframe(depth, bgr, T, *K, i, objs, LEAF)
    return _REF[(name, i)]


def _insert(gm, entry, depth, bgr, T, i, objs):
    if entry == "host":
        return gm.insertKeyFrameObjects(T, depth, bgr, *K, i, objs)
    import torch
    d, c = torch.from_numpy(depth).cuda(), torch.from_numpy(bgr).cuda()
    torch.cuda.synchronize()
    return gm.insert_keyframe_objects_device(d.data_ptr(), c.data_ptr(), depth.shape[0], depth.shape[1], T, *K, i, objs)


@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("name", sem_scenes.NAMES)
def test_scene_matches_oracle(oracle, name, entry):
    depth, bgr, T, objs = sem_scenes.scene(name)
    gm = GlobalCloudMapping(LEAF)
    recs = _insert(gm, entry, depth, bgr, T, 1, objs)
    ref_recs, painted, (xyz, rgb) = _oracle(name)
    assert [_rec(r) for r in recs] == [_rec(r) for r in ref_recs]
    gx, gc = gm.points()                                    # the appended cloud, pixel order
    assert (gc == rgb).all() and (_bits(gx) == _bits(xyz)).all()
    assert (painted != bgr).any()
    st = [r.status for r in recs]
    if name == "small_missing":
        assert st == [GCM_FEW_POINTS, GCM_CLUSTER, GCM_FEW_POINTS, GCM_BELOW_PROB, GCM_CLUSTER]
        assert recs[1].n_voxels == 1 and recs[2].n_band == 0      # zero depth: one point at the camera; NaN: no band
    if name == "many":
        assert len(recs) == 32 and st.count(GCM_CLUSTER) >= 10
    if name == "big":
        assert recs[0].n_band >= 60000 and recs[0].n_inliers < recs[0].n_band
    if name == "edges":
        assert recs[3].n_band > 640                              # wider than the image: wrapped rows repeat indices
    gm.refilter()
    rx, rc = oracle.global_refilter(xyz, rgb, LEAF)
    gx, gc = gm.points()
    assert len(gx) == len(rx) > 1000 and (_bits(gx) == _bits(rx)).all() and (gc == rc).all()


def test_skip_rule_and_the_plain_overload_over_a_sequence():
    depth, bgr, T, objs = sem_scenes.scene("overlap")
    npix = depth.size
    gm = GlobalCloudMapping(LEAF)
    assert gm.insertKeyFrameObjects(T, depth, bgr, *K, 0, []) == [] and gm.size() == 0      # even, no objects: skipped
    gm.insertKeyFrameObjects(T, depth, bgr, *K, 1, [])
    assert gm.size() == npix
    low = [o[:5] + (0.5,) for o in objs]
    recs = gm.insertKeyFrameObjects(T, depth, bgr, *K, 2, low)                              # low prob still counts
    assert [r.status for r in recs] == [GCM_BELOW_PROB] * 3 and gm.size() == 2 * npix
    _, gc = gm.points()
    assert (gc[npix:] == bgr.reshape(-1, 3)[:, ::-1]).all()                                 # nothing painted
    gm.insertKeyFrame(T, depth, bgr, *K)                                                    # the plain overload: no skip
    assert gm.size() == 3 * npix


VOC = ["background", "aeroplane", "bicycle", "bird", "boat", "bottle", "bus", "car", "cat", "chair", "cow", "diningtable",
       "dog", "horse", "motorbike", "person", "pottedplant", "sheep", "sofa", "train", "tvmonitor"]


def _sequence():
    seq = []
    for i, t in enumerate(range(5, 13)):
        depth, bgr, T = sem_scenes.room_frame(t)
        s = 3.0 * i
        objs = [(100.0 + s, 80.0, 200.0, 150.0, 9, 0.9), (320.0 - s, 200.0, 120.0, 160.0, 15, 0.8),
                (400.0, 60.0 + s, 90.0, 70.0, 20, 0.7), (30.0, 300.0, 80.0, 60.0, 9, 0.6), (500.0, 300.0, 8.0, 8.0, 5, 0.9),
                (250.0, 250.0, 60.0, 50.0, 5, 0.3)]
        if i in (2, 3):
            objs = []                      # keyframe 2 is skipped (even, no objects); keyframe 3 is added unpainted
        seq.append((depth, bgr, T, objs))
    return seq


def test_shim_overload_matches_the_python_mirror(tmp_path):
    seq = _sequence()
    rows, cols = seq[0][0].shape
    with open(tmp_path / "seq.bin", "wb") as f:
        f.write(struct.pack("<3i5f", rows, cols, len(seq), *[float(np.float32(v)) for v in K], LEAF))
        for depth, bgr, T, objs in seq:
            f.write(np.ascontiguousarray(T, np.float32).tobytes() + depth.tobytes() + bgr.tobytes())
            f.write(struct.pack("<i", len(objs)))
            for x, y, w, h, c, p in objs:
                f.write(struct.pack("<4fif16s", x, y, w, h, c, p, VOC[c].encode()))
    shim = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200", "csrc", "shim")
    libdir = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200")
    exe = str(tmp_path / "shim_sem_check")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-o", exe, os.path.join(shim, "shim_sem_check.cpp"),
                           "-I" + os.path.join(ROOT, "oracle", "standin"), "-I" + os.path.join(ROOT, "include"), "-L" + libdir,
                           "-lb200orb", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe, str(tmp_path / "seq.bin")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    gm, db = GlobalCloudMapping(LEAF), SemanticClusters()
    merged = 0
    for i, (depth, bgr, T, objs) in enumerate(seq):
        for o, r in zip(objs, gm.insertKeyFrameObjects(T, depth, bgr, *K, i, objs)):
            if r.status == GCM_CLUSTER:
                db.merge_record(VOC[o[4]], o[4], np.float32(o[5]), r)
                merged += 1
    gm.refilter()
    want = ["cluster %s %d %s" % (c["object_name"], c["class_id"],
                                  " ".join("%08x" % b for b in _bits([c["prob"], *c["centroid"], *c["minPt"], *c["maxPt"]])))
            for c in db.clusters]
    want.append("globalMap %d" % gm.size())
    assert out.stdout.split("\n")[:-1] == want
    assert merged > len(db.clusters) >= 3           # some clusters were merged into earlier ones
