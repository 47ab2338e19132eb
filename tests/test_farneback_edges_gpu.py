"""The dense flow on the device on the crafted pairs of tests/flow_edge_cases.py: DynamicMask.farneback (dynm_farneback)
equal bit for bit to the restatement (oracle/farneback_py.py) and to cv2's flow stored in tests/golden/flow_edges.npz
(the array, or its digest for pairs too large to store); and dynm_flow_batch_device at the ends of the full-resolution
range it accepts, with and without the frame before the batch.

At most 3 full-resolution frames run at the large sizes: the scratch then stays near 1 GB (a full 64-pair chunk of
2048 x 2048 half-resolution images would take about 25 GB)."""
import functools
import os

import numpy as np
import pytest

from oracle import farneback_py as FB
from tests import flow_edge_cases as EC
from tests.refpins import digest
from tests.test_farneback_gpu import _flow_batch, _oracle_flows, _same

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flow_edges.npz")
Z = np.load(GOLDEN)
NAMES = [str(n) for n in Z["names"]]


@functools.lru_cache(maxsize=None)
def _cases():
    return {c.name: c for c in EC.cases()}


@functools.lru_cache(maxsize=None)
def _restated(name):
    c = _cases()[name]
    return FB.farneback(c.prev, c.cur)


@pytest.fixture(scope="module")
def dm():
    from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask
    return DynamicMask(0)


def test_golden_lists_every_case():
    assert NAMES == list(_cases())


@pytest.mark.parametrize("name", NAMES)
def test_case_equals_restatement_and_cv2(dm, name):
    c = _cases()[name]
    assert str(Z[name + "/inputs_sha256"]) == digest((c.prev, c.cur)), "tests/flow_edge_cases.py drifted"
    got = dm.farneback(c.prev, c.cur)
    _same(got, _restated(name))
    if name + "/flow" in Z:
        _same(got, Z[name + "/flow"])
    assert digest(got) == str(Z[name + "/flow_sha256"])


@pytest.mark.parametrize("rows,cols,n", [(32, 4097, 3), (4097, 33, 3), (33, 33, 3), (4097, 4097, 2)])
def test_flow_batch_device_at_accepted_extremes(dm, rows, cols, n):
    """Full-resolution sides 32 | 33 and 4097 halve to 16 and 2048, the ends of the half-resolution range."""
    seq = EC.sequence(rows, cols, n + 1, dy=2, dx=3, seed=rows + cols)
    want = _oracle_flows(seq[1:], seq[0])
    _same(_flow_batch(dm, seq[1:], seq[0]), want)
    got = _flow_batch(dm, seq[1:])
    assert not got[0].any()
    _same(got[1:], want[1:])
