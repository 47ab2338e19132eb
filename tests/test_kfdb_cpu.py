"""Key-frame database, CPU side: the restatement (oracle/kfdb_py.py) equals the reference's own
src/KeyFrameDatabase.cc on real KeyFrames (oracle/kfdb_harness.cpp, kfdb_run), bit for bit -- candidates in order,
the six database members of every keyframe after every query, and the GetBestCovisibilityKeyFrames(10) lists the scripts
assume -- pinned as digests in tests/golden/kfdb_pins.json (tests/refpins.py's format; REFSRC_RECORD=1 re-runs the
reference where oracle/_ref is built and rewrites them).  Without a GPU the device database refuses to start."""
import json
import os

import pytest

from oracle import kfdb_py
from tests import kfdb_cases
from tests.refpins import RECORD, Pins

CRAFTED = kfdb_cases.crafted()


PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kfdb_pins.json")


class KfdbPins(Pins):
    def __init__(self):
        with open(PINS) as f:
            self.d = json.load(f)

    def save(self):
        if RECORD:
            with open(PINS, "w") as f:
                json.dump(self.d, f, indent=0, sort_keys=True)
                f.write("\n")


@pytest.fixture(scope="module")
def pins():
    p = KfdbPins()
    yield p
    p.save()


def _check(pins, key, scene):
    cands, members = kfdb_py.run(scene)
    pins.check(key, (cands, members, scene.neigh), lambda: kfdb_cases.run_src("refsrc", scene))
    return cands


@pytest.mark.parametrize("name", sorted(CRAFTED))
def test_restatement_equals_reference_source(pins, name):
    _check(pins, "kfdb/" + name, CRAFTED[name])


def test_restatement_equals_reference_source_random_scene(pins):
    scene = kfdb_cases.random_scene()
    assert scene.n_kf >= 2000 and scene.n_words >= 100_000 and min(len(w) for w in scene.words) >= 300
    cands = _check(pins, "kfdb/random_scene", scene)
    assert sum(len(c) > 0 for c in cands) > len(cands) // 2


def test_growth_scene_pinned(pins):
    _check(pins, "kfdb/growth_scene", kfdb_cases.growth_scene())


def test_crafted_cases_reach_their_edges():
    """The crafted scripts land where they claim (checked on the restatement, which equals the reference source)."""
    F = kfdb_py.F32
    # threshold: 8 of 10 common words is not scored, 9 is; 5 of 7 is not, 6 is
    assert int(F(10) * F(0.8)) == 8 and int(F(7) * F(0.8)) == 5
    # equal scores: Z's accumulated 3.0 is exactly 0.75f * 4.0 and is not retained
    c, _ = kfdb_py.run(CRAFTED["equal_scores_acc_threshold"])
    assert list(c[0]) == [0] and F(0.75) * F(4) == F(3)
    # stale relocalisation score: the second query's candidate reads N's score from the first query
    c, m = kfdb_py.run(CRAFTED["reloc_stale_score"])
    assert m[1][3][0] == 12 and m[1][5][0] == m[0][5][0]   # N met again (query id 12), its score is the old one
    # loop: the connected keyframe that shares words ends at mnLoopWords 1 and is never marked
    c, m = kfdb_py.run(CRAFTED["loop_connected_min_score"])
    assert m[0][1][1] == 1 and m[0][0][1] == 0
    # the empty query, no shared word and every score under minScore give no candidate
    c, _ = kfdb_py.run(CRAFTED["empty_results"])
    assert [len(x) for x in c[:4]] == [0, 0, 0, 0]


def test_device_refuses_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from orb_slam2_ssd_semantic_b200 import B200OrbError, KeyFrameDatabase
    with pytest.raises(B200OrbError) as e:
        KeyFrameDatabase(64)
    assert e.value.code == -4 and "no CPU fallback" in str(e.value)
