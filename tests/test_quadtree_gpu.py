"""GPU parity of the quad-tree (DistributeOctTree, orbx_kernels.cuh K3) with the CPU oracle on inputs that drive each of
its round kinds: sweep rounds that run until every node holds one keypoint, largest-first rounds over many nodes of
equal size (the rank's list-order tie-break), levels with no or one candidate, and the largest list its shared memory
holds."""
import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth
from tests.test_boundaries_gpu import QT_LIMIT_8, _extract_and_compare, level_features, qt_fits

pytestmark = pytest.mark.gpu


def _lattice(step, h=480, w=640):
    """Single white pixels on black, `step` px apart: each is a FAST corner of the same response, and the quadrants of
    the initial node split the lattice evenly, so nodes tie on their keypoint counts round after round."""
    img = np.zeros((h, w), np.uint8)
    img[20:h - 20:step, 20:w - 20:step] = 255
    return img


def _squares(period, h=480, w=640):
    """A checkerboard of period x period squares: corners only at the square vertices, periodic in both axes."""
    yy, xx = np.mgrid[0:h, 0:w]
    return ((((yy // period) + (xx // period)) & 1) * 255).astype(np.uint8)


def _dots(points, h=480, w=640):
    img = np.zeros((h, w), np.uint8)
    for y, x in points:
        img[y, x] = 255
    return img


def _run(oracle, params, img, tag):
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    ex = ORBextractor(*params)
    K = _extract_and_compare(oracle, ex, params, img, tag)
    return K, ex.candidates_per_level()


@pytest.mark.parametrize("seed", [1, 2])
def test_sweep_rounds_until_every_node_is_single(oracle, seed):
    """Fewer candidates than the quota on every level: sweep rounds run until each node holds one keypoint and the
    list stops growing."""
    rng = np.random.default_rng(seed)
    pts = {(int(y), int(x)) for y, x in zip(rng.integers(24, 456, 400), rng.integers(24, 616, 400))}
    params = (QT_LIMIT_8, 1.2, 8, 20, 7)
    K, cand = _run(oracle, params, _dots(sorted(pts)), "scattered dots seed=%d" % seed)
    assert 100 < cand[0] < level_features(QT_LIMIT_8, 1.2, 8)[0], cand


def test_sweep_rounds_on_dense_noise(oracle):
    """Threshold 0 on uniform noise: a corner on most pixels, many sweep rounds before the quota is reached."""
    params = (3000, 1.2, 8, 0, 0)
    K, cand = _run(oracle, params, synth.adversarial_frames()["noise"], "noise th=0 nfeatures=3000")
    assert cand[0] > 5 * level_features(3000, 1.2, 8)[0] and len(K) >= 2700, cand


@pytest.mark.parametrize("step", [5, 6, 8, 12])
@pytest.mark.parametrize("nfeatures", [500, 1000, 2000])
def test_largest_first_with_tied_node_sizes(oracle, step, nfeatures):
    """Regular dot lattices: largest-first rounds pick among many nodes of equal size.  More candidates than the level's
    quota is what lets the sweep rounds hand over to largest-first rounds; the lattice makes the quadrant counts equal.
    Neither library reports its round kinds, so what catches a wrong rank or tie-break here is the bit-exact comparison
    of the keypoint list with the oracle's."""
    K, cand = _run(oracle, (nfeatures, 1.2, 8, 20, 7), _lattice(step), "lattice %d nfeatures=%d" % (step, nfeatures))
    assert cand[0] > level_features(nfeatures, 1.2, 8)[0], cand


@pytest.mark.parametrize("period", [4, 10, 16])
def test_largest_first_on_periodic_squares(oracle, period):
    _run(oracle, (1000, 1.2, 8, 20, 7), _squares(period), "squares %d" % period)


@pytest.mark.parametrize("points", [[], [(240, 320)], [(100, 100), (380, 540)]], ids=["none", "one", "two"])
def test_levels_with_zero_or_one_candidate(oracle, points):
    """One or two isolated dots: level 0 holds exactly that many candidates, an empty image none on any level."""
    K, cand = _run(oracle, (1000, 1.2, 8, 20, 7), _dots(points), "%d dots" % len(points))
    assert cand[0] == len(points) and (cand.any() if points else not cand.any()), cand


@pytest.mark.parametrize("nfeatures", [QT_LIMIT_8 - 1, QT_LIMIT_8])
@pytest.mark.parametrize("image", ["noise_th0", "lattice", "squares"])
def test_largest_list_the_shared_memory_holds(oracle, nfeatures, image):
    """nfeatures at the quad-tree's shared-memory limit and one below it."""
    assert qt_fits(480, 640, nfeatures, 1.2, 8)
    th = (0, 0) if image == "noise_th0" else (20, 7)
    img = {"noise_th0": synth.adversarial_frames()["noise"], "lattice": _lattice(5), "squares": _squares(4)}[image]
    _run(oracle, (nfeatures, 1.2, 8) + th, img, "%s nfeatures=%d" % (image, nfeatures))
