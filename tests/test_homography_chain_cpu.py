"""CPU checks of the homography batch's interface: OrbsBatch.homography sits in the struct's trailing padding (the size
stays 88 bytes), and the branch codes of include/b200orb.h are the ones StreamTracker.homography names."""
import ctypes as C
import os
import re

from orb_slam2_ssd_semantic_b200._abi import OrbsBatch
from orb_slam2_ssd_semantic_b200.pipeline import StreamTracker

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_homography_field_in_trailing_padding():
    assert OrbsBatch.homography.offset == OrbsBatch.binary_threshold.offset + 4
    assert C.sizeof(OrbsBatch) == 88


def test_branch_codes_match_header():
    with open(os.path.join(ROOT, "include", "b200orb.h")) as f:
        codes = dict((m.group(1).lower(), int(m.group(2)))
                     for m in re.finditer(r"#define ORBS_HOMO_(\w+) (\d+)", f.read()))
    assert [codes[k] for k in StreamTracker.HOMO_BRANCHES] == list(range(len(StreamTracker.HOMO_BRANCHES)))
