"""GPU parity of the orientation + descriptor stage at the edges of its patch tiles, bit-exact with the oracle.

Keypoints lie in [19, w-20] x [19, h-20] of their level; the stage reads 31x31 raw and 37x37 blurred patches around them
from word-aligned tiles.  These cases put keypoints on the first and last row and column of that range on every level, at
every byte phase of the level's width, through a level 0 whose pitch equals its width, and at angles where the rotated
pattern reaches 18 px."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PARAMS = (4000, 1.2, 8, 20, 7)   # many features: the quad-tree's nodes get small enough to keep keypoints on the edges


def _cmp(K, D, K2, D2, tag):
    assert len(K) == len(K2), "%s: keypoint count %d vs oracle %d" % (tag, len(K), len(K2))
    for name in K.dtype.names:
        bad = np.nonzero(K[name].view(np.int32) != K2[name].view(np.int32))[0]
        assert bad.size == 0, "%s: field %s differs at %s" % (tag, name, bad[:5])
    bad = np.nonzero((D != D2).any(axis=1))[0]
    assert bad.size == 0, "%s: %d descriptors differ, first %s" % (tag, bad.size, bad[:5])


def _border_noise(rows, cols, seed):
    """Uniform noise within 110 px of the image's sides, flat inside: corners crowd every level's border band."""
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, size=(rows, cols), dtype=np.uint8)
    yy, xx = np.mgrid[0:rows, 0:cols]
    d = np.minimum(np.minimum(xx, cols - 1 - xx), np.minimum(yy, rows - 1 - yy))
    img[d > 110] = 128
    return img


def _scale_factors(scale, nlevels):
    sf = [np.float32(1.0)]
    for _ in range(1, nlevels):
        sf.append(np.float32(sf[-1] * np.float32(scale)))
    return sf


def _edge_hits(ex, frames_kps, nlevels, scale):
    """hits[l] = set of the sides (left, right, top, bottom) of level l on whose extreme line some keypoint lies."""
    sf = _scale_factors(scale, nlevels)
    hits = [set() for _ in range(nlevels)]
    for K in frames_kps:
        for l in range(nlevels):
            h, w = ex.image_pyramid_level(l).shape
            k = K[K["octave"] == l]
            x = np.rint(k["x"] / sf[l]).astype(int)
            y = np.rint(k["y"] / sf[l]).astype(int)
            assert x.size == 0 or (x.min() >= 19 and x.max() <= w - 20 and y.min() >= 19 and y.max() <= h - 20)
            for side, on in (("left", x == 19), ("right", x == w - 20), ("top", y == 19), ("bottom", y == h - 20)):
                if on.any():
                    hits[l].add(side)
    return hits


@pytest.mark.parametrize("cols", [640, 641, 642, 643])
def test_keypoints_on_every_extreme_row_and_column(oracle, cols):
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    rows = 480
    imgs = np.stack([_border_noise(rows, cols, 1000 * cols + s) for s in range(4)])
    ex = ORBextractor(*PARAMS)
    res = ex.extract_batch(imgs)
    R = oracle.RefExtractor(*PARAMS)
    for f, (K, D) in enumerate(res):
        K2, D2 = R(imgs[f])
        _cmp(K, D, K2, D2, "cols %d frame %d" % (cols, f))
    hits = _edge_hits(ex, [K for K, _ in res], PARAMS[2], PARAMS[1])
    for l, h in enumerate(hits):
        assert h == {"left", "right", "top", "bottom"}, "cols %d level %d: keypoints only on %s" % (cols, l, sorted(h))


@pytest.mark.parametrize("cols", [640, 644])
def test_level0_pitch_equal_to_cols(oracle, cols):
    """orbx_extract_batch_device on a packed batch (pitch = cols, a multiple of 4): level 0 is read in place, and the
    last word of a tile row can be the last word of the caller's row."""
    import ctypes as C
    import types
    import torch
    from orb_slam2_ssd_semantic_b200 import ORBextractor, _lib
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE

    def to_host(ptr, nbytes):
        view = types.SimpleNamespace(__cuda_array_interface__={"shape": (nbytes,), "typestr": "|u1",
                                                               "data": (ptr, False), "version": 2})
        return torch.as_tensor(view, device="cuda").cpu().numpy()

    F, rows = 3, 480
    imgs = np.stack([_border_noise(rows, cols, 7000 * cols + s) for s in range(F)])
    d_imgs = torch.from_numpy(imgs).cuda()
    ex = ORBextractor(*PARAMS)
    L, h = _lib.lib(), ex.handle
    _lib.check(L.orbx_extract_batch_device(h, C.c_void_p(d_imgs.data_ptr()), F, rows, cols, cols, rows * cols))
    _lib.check(L.orbx_sync(h))
    d_kps, d_desc, d_n, cap = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int()
    _lib.check(L.orbx_device_results(h, C.byref(d_kps), C.byref(d_desc), C.byref(d_n), C.byref(cap)))
    cap = cap.value
    n = to_host(d_n.value, 4 * F).view(np.int32)
    kps = to_host(d_kps.value, KP_DTYPE.itemsize * cap * F).view(KP_DTYPE).reshape(F, cap)
    desc = to_host(d_desc.value, 32 * cap * F).reshape(F, cap, 32)
    R = oracle.RefExtractor(*PARAMS)
    for f in range(F):
        K2, D2 = R(imgs[f])
        _cmp(kps[f, :n[f]], desc[f, :n[f]], K2, D2, "pitch = cols = %d, frame %d" % (cols, f))
    hits = _edge_hits(ex, [kps[f, :n[f]] for f in range(F)], PARAMS[2], PARAMS[1])
    assert "right" in hits[0], "no level-0 keypoint on the last column"


def _ramp(rows, cols, deg, seed):
    """Triangle wave of period 256 px along direction `deg` plus noise: intensity centroids point along deg or deg+180."""
    yy, xx = np.mgrid[0:rows, 0:cols].astype(np.float64)
    th = np.deg2rad(deg)
    tri = np.abs(((xx * np.cos(th) + yy * np.sin(th)) / 128.0) % 2.0 - 1.0)
    rng = np.random.default_rng(seed)
    return np.clip(40 + 170 * tri + rng.normal(0, 12, (rows, cols)), 0, 255).astype(np.uint8)


def test_angles_near_multiples_of_45_degrees(oracle):
    """Near 45 + 90 j degrees the pattern point (-13, -13) lands 18 px from the keypoint: the blurred tile's edge."""
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    params = (1000, 1.2, 8, 20, 7)
    imgs = np.stack([_ramp(480, 641, 45 * k, k) for k in range(4)])
    res = ORBextractor(*params).extract_batch(imgs)
    R = oracle.RefExtractor(*params)
    for k, (K, D) in enumerate(res):
        K2, D2 = R(imgs[k])
        _cmp(K, D, K2, D2, "ramp at %d degrees" % (45 * k))
        a = K["angle"].astype(np.float64)
        assert np.mean(np.abs((a + 22.5) % 45.0 - 22.5) < 3.0) > 0.5, "ramp at %d degrees" % (45 * k)
        if k & 1:
            assert np.mean(np.abs(a % 90.0 - 45.0) < 10.0) > 0.5, "ramp at %d degrees" % (45 * k)
