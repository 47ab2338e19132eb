"""The homography branch's warp on the device (dynm_warp_perspective, dynm_warp_perspective_batch_device) against the
restatement oracle/homography_py.py (pinned to cv2 4.13 by tests/test_homography_cpu.py) and the goldens, bit for bit,
and the mirror's ComputeMask(GrayImg, Homo=H) overload (perfect/src/Flow.cc:73-80) against the plain ComputeMask of the
restated warp."""
import os

import numpy as np
import pytest

from oracle import farneback_py as FB
from oracle import homography_py as HP
from tests import warp_cases as WC

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "homography_warp.npz")


@pytest.fixture(scope="module")
def dm():
    from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask
    return DynamicMask(0)


@pytest.mark.parametrize("rows,cols", WC.SIZES + ((16, 2000), (7, 5), (1, 1)))
@pytest.mark.parametrize("case", WC.CASES)
def test_warp_equals_restatement(dm, case, rows, cols):
    src = WC.image(rows, cols)
    H = WC.homography(case, rows, cols)
    n0 = dm.launch_count()
    got = dm.warp_perspective(src, H)
    assert dm.launch_count() == n0 + 1
    want = HP.warp_perspective(src, H)
    assert (got == want).all(), "%d of %d bytes differ" % ((got != want).sum(), got.size)


def test_warp_equals_goldens(dm):
    z = np.load(GOLDEN)
    for c, H, dst in zip(z["cases"], z["H"], z["dst"]):
        assert (dm.warp_perspective(z["src"], H) == dst).all(), c


def test_warp_random_maps(dm):
    rng = np.random.Generator(np.random.PCG64(9))
    src = WC.image(480, 640, seed=2)
    for _ in range(10):
        H = np.eye(3) + rng.normal(0, 0.05, (3, 3))
        H[2, :2] *= 0.01
        H[:2, 2] += rng.normal(0, 10, 2)
        assert (dm.warp_perspective(src, H) == HP.warp_perspective(src, H)).all()


def test_warp_batch_device(dm):
    import torch
    rows, cols = 195, 323
    src = np.stack([WC.image(rows, cols, seed=s) for s in range(len(WC.CASES))])
    Hs = np.stack([WC.homography(c, rows, cols) for c in WC.CASES])
    g = torch.from_numpy(src).cuda()
    h = torch.from_numpy(Hs).cuda()
    out = torch.full_like(g, 77)
    torch.cuda.synchronize()
    dm.warp_perspective_batch_device(g.data_ptr(), len(src), rows, cols, h.data_ptr(), out.data_ptr())
    dm.sync()
    out = out.cpu().numpy()
    for t, c in enumerate(WC.CASES):
        assert (out[t] == HP.warp_perspective(src[t], Hs[t])).all(), c


def test_compute_mask_homography_overload(dm):
    """Flow.cc:73-80: ComputeMask(GrayImg, Homo) == ComputeMask(warpPerspective(GrayImg, Homo)), the previous half image
    kept in between as the plain call keeps it."""
    from orb_slam2_ssd_semantic_b200.dynmask import Flow
    from tests import flow_scenes as S
    g = S.frames("room", 480, 640, 3)
    Hs = [None, WC.homography("room", 480, 640), WC.homography("shift_sub", 480, 640)]
    a = Flow(flow_fn=dm.farneback, pyr_down_fn=lambda x: FB.pyr_down(x, x.shape[0] // 2, x.shape[1] // 2))
    b = Flow(flow_fn=dm.farneback, pyr_down_fn=lambda x: FB.pyr_down(x, x.shape[0] // 2, x.shape[1] // 2))
    for t in range(3):
        ma = a.ComputeMask(g[t], 40.0, Homo=Hs[t])
        mb = b.ComputeMask(g[t] if Hs[t] is None else HP.warp_perspective(g[t], Hs[t]), 40.0)
        assert (ma == mb).all(), t
        assert (a.mImGrayLast == b.mImGrayLast).all()


def test_bad_arguments_enqueue_nothing(dm):
    from orb_slam2_ssd_semantic_b200._lib import B200OrbError
    n0 = dm.launch_count()
    for shape in ((0, 8), (8, 0), (2, 32767), (32767, 2)):
        with pytest.raises(B200OrbError):
            dm.warp_perspective(np.zeros(shape, np.uint8), np.eye(3))
    with pytest.raises(ValueError):
        dm.warp_perspective(np.zeros((8, 8), np.uint8), np.eye(2))
    with pytest.raises(B200OrbError):
        dm.warp_perspective_batch_device(0, 1, 8, 8, 0, 0)
    with pytest.raises(B200OrbError):
        dm.warp_perspective_batch_device(0, -1, 8, 8, 0, 0)
    dm.warp_perspective_batch_device(0, 0, 8, 8, 0, 0)   # an empty batch is a no-op
    assert dm.launch_count() == n0
