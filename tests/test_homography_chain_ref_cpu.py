"""The TrackHomo step of the homography-batch restatement (tests/homography_chain_ref.track_homo: both searches, the
clear and retry at 2 th, the pair lists) against the perfect tree's own Frame / ORBmatcher code through
homo_cases.run_sequence (oracle/_ref/libhomoref.so), where oracle/_ref is built."""
import os

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth
from orb_slam2_ssd_semantic_b200._abi import FrameView
from tests import homo_cases
from tests import homography_chain_ref as HR


@pytest.mark.parametrize("shift", [0.0, 0.2])
def test_track_homo_step_equals_perfect_tree(shift):
    if not os.path.exists(homo_cases.REF_SO):
        pytest.skip("oracle/_ref is not built")
    from oracle import ref
    inp = homo_cases.sequence_inputs(shift=shift)
    R = ref.RefExtractor(1000, 1.2, 8, 20, 7)
    K, D = R(inp["gray"])
    ur, _, _, _ = ref.stereo_unproject(K, inp["depth"], inp["T"], synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
    rows, cols = inp["gray"].shape
    cur = FrameView(K["x"], K["y"], K["octave"], K["angle"], ur, D, inp["T"], synth.FX, synth.FY, synth.CX, synth.CY,
                    synth.BF, 0.0, float(cols), 0.0, float(rows), R.mvScaleFactor)
    xy = np.stack([K["x"], K["y"]], 1).astype(np.float32)
    nm, c2l, pl, pc, _ = HR.track_homo(cur, inp["last"], xy, inp["last_kxy"], 15.0)
    want = homo_cases.run_sequence(inp, homo_cases.harness(homo_cases.REF_SO, "refperfect_"), "refperfect_")
    assert nm == want[0] > 0
    assert np.asarray(c2l, np.int32).tobytes() == want[1].tobytes()
    assert pl.tobytes() == want[2].tobytes() and pc.tobytes() == want[3].tobytes()
