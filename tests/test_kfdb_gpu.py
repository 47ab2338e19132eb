"""Key-frame database on the GPU (orbv_db_*, csrc/orbv_db.cu): bit for bit -- candidates in order, the six database
members of every keyframe after every query --
  * the device through the Python mirror == the restatement (oracle/kfdb_py.py, pinned to the reference's source by
    tests/test_kfdb_cpu.py), and == the reference's own src/KeyFrameDatabase.cc where oracle/_ref is built;
  * the shim (shim/KeyFrameDatabase.h) on real KeyFrames (libkfdbshim.so) == the reference's source (libkfdbsrc.so);
and the device refuses malformed input."""
import ctypes as C

import numpy as np
import pytest

from oracle import kfdb_py
from tests import kfdb_cases
from tests.refpins import digest

pytestmark = pytest.mark.gpu
CRAFTED = kfdb_cases.crafted()
SCENES = dict(CRAFTED)
SCENES["random_scene"] = None
SCENES["growth_scene"] = None


def _scene(name):
    if name == "random_scene":
        return kfdb_cases.random_scene()
    if name == "growth_scene":
        return kfdb_cases.growth_scene()
    return CRAFTED[name]


def _ref_built():
    return kfdb_cases.src_available()


@pytest.mark.parametrize("name", sorted(SCENES))
def test_device_equals_restatement_and_reference(name):
    from orb_slam2_ssd_semantic_b200.keyframedb import KeyFrameDatabase
    scene = _scene(name)
    db = KeyFrameDatabase(scene.n_words)
    got = kfdb_cases.run_device(scene, db=db)
    want = kfdb_py.run(scene)
    assert digest(got) == digest(want), name
    for k in range(scene.n_kf):   # the device's mirror agrees with what was written back
        if k in db._added:
            m, _ = db.state(k)
            assert m.tobytes() == db.members[k].tobytes(), k
    if _ref_built():
        cands, members, neigh = kfdb_cases.run_src("refsrc", scene)
        assert digest((cands, members)) == digest(got) and neigh == scene.neigh


@pytest.mark.parametrize("name", sorted(SCENES))
def test_shim_on_reference_objects_equals_reference_source(name):
    if not _ref_built():
        pytest.skip("oracle/_ref is not built")
    scene = _scene(name)
    assert digest(kfdb_cases.run_src("shimsrc", scene)) == digest(kfdb_cases.run_src("refsrc", scene))


def test_one_sync_three_launches_per_query():
    from orb_slam2_ssd_semantic_b200.keyframedb import KeyFrameDatabase
    scene = CRAFTED["threshold_mult5"]
    db = KeyFrameDatabase(scene.n_words)
    for k in range(scene.n_kf):
        db.add(k, (scene.words[k], scene.weights[k]))
    n0 = db.launch_count()
    db.DetectRelocalizationCandidates(5, (scene.words[0], scene.weights[0]), scene.neigh)
    assert db.launch_count() - n0 == 3
    db.DetectRelocalizationCandidates(6, (np.array([63], np.uint32), np.ones(1)), scene.neigh)   # nobody shares word 63
    assert db.launch_count() - n0 == 6


def test_malformed_input_is_refused():
    from orb_slam2_ssd_semantic_b200 import B200OrbError, lib
    from orb_slam2_ssd_semantic_b200.keyframedb import HIT_DTYPE, KeyFrameDatabase
    db = KeyFrameDatabase(100)
    db.add(0, (np.array([1, 5, 9], np.uint32), np.full(3, 1 / 3)))
    bad = [np.array([1, 100], np.uint32), np.array([5, 1], np.uint32), np.array([1, 1], np.uint32)]
    for w in bad:
        with pytest.raises(B200OrbError) as e:
            db.add(1, (w, np.full(len(w), 0.5)))
        assert e.value.code == -1
        with pytest.raises(B200OrbError) as e:
            db.DetectRelocalizationCandidates(3, (w, np.full(len(w), 0.5)), [[]])
        assert e.value.code == -1
    for slot in (-1, 1 << 24):
        with pytest.raises(B200OrbError):
            db.add(slot, (np.array([1], np.uint32), np.ones(1)))
    L = lib()
    assert L.orbv_db_erase(db._h, 7) == -1 and L.orbv_db_state(db._h, 7, None, None, None) == -1
    hits = np.zeros(1, HIT_DTYPE)
    na, nm = C.c_int(), C.c_int()
    w, v = np.array([1], np.uint32), np.ones(1)
    assert L.orbv_db_query(db._h, 0, 3, w.ctypes.data, v.ctypes.data, 1, None, 0, hits.ctypes.data, 0, C.byref(na),
                           C.byref(nm)) == -2   # cap below the number of keyframes in the database: nothing changes
    assert db.state(0)[0]["reloc_query"] == 0
    assert db.DetectRelocalizationCandidates(3, (w, v), [[]]) == [0]
