"""Device == oracle, bit for bit, on the crafted matcher cases of tests/match_cases.py (their oracle results are pinned to
the reference's own ORBmatcher.cc by tests/test_matcher_edges_cpu.py).  Every LAST case runs twice: as built (the fused
one-CTA kernel) and with the current frame padded at the front by keypoints outside the grid, which moves the crafted
indices above 4095 and the frame past the fused kernel's limit (the 4-launch path)."""
import numpy as np
import pytest

from tests import match_cases as M
from tests.test_boundaries_gpu import match_last_fused

pytestmark = pytest.mark.gpu

CASES = M.all_cases()
LAST = [c for c in CASES if c.kind == "last"]
OTHER = [c for c in CASES if c.kind != "last"]
PAD = 4200


def _assert_same(case, got, ref):
    assert len(got) == len(ref), case.name
    for g, r in zip(got, ref):
        g, r = np.asarray(g), np.asarray(r)
        bad = np.nonzero(np.atleast_1d(g != r))[0] if g.shape == r.shape else None
        assert bad is not None and bad.size == 0, "%s: device %s, oracle %s (differ at %s)" % (case.name, g, r, bad)


@pytest.mark.parametrize("pad", [0, PAD], ids=["fused", "padded"])
@pytest.mark.parametrize("case", LAST, ids=[c.name for c in LAST])
def test_last_device_equals_oracle(oracle, case, pad):
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    cur, last = M.last_views(case, pad)
    fused = match_last_fused(cur.n, last.n)
    assert fused == (pad == 0), (cur.n, last.n)
    m = ORBmatcher(M.LAST_NNRATIO, case.kw["ori"])
    before = m.launch_count()
    got = m.SearchByProjection(cur, last, case.kw["th"], case.kw["mono"])
    assert m.launch_count() - before == (1 if fused else 4)
    _assert_same(case, got, M.run(case, "oracle", oracle, pad))


@pytest.mark.parametrize("case", OTHER, ids=[c.name for c in OTHER])
def test_device_equals_oracle(oracle, case):
    _assert_same(case, M.run(case, "gpu"), M.run(case, "oracle", oracle))
