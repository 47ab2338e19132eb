"""Stage-level GPU parity of the extractor on the crafted cases of tests/extractor_cases.py, bit for bit against the
oracle: per level and frame the raw pyramid level, its 7x7 blur (k_blur7_strip / k_blur7_edges) and the FAST candidates
of k_fast_cells in the quad-tree's input order, then the keypoints and descriptors.  Also batches of different cases in
one call, device batches with level 0 read in place and staged, and the read-backs' error returns."""
import ctypes as C

import numpy as np
import pytest

from oracle import ref
from tests import extractor_cases as E

pytestmark = pytest.mark.gpu

CASES = E.all_cases()
FAMILIES = sorted({c.name.split("/")[0] for c in CASES})


@pytest.fixture(scope="module")
def extractors():
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    cache = {}

    def get(params):
        if params not in cache:
            cache[params] = ORBextractor(*params)
        return cache[params]
    return get


def _compare_frame(ex, R, img, nlevels, frame, tag, K=None, D=None):
    """Every stage of frame `frame` of ex's last extract against the oracle R run on img; returns the differing items."""
    bad = []
    K2, D2 = R(img)
    for l in range(nlevels):
        lv = R.level(l)
        if not np.array_equal(ex.image_pyramid_level(l, frame), lv):
            bad.append("%s: raw level %d" % (tag, l))
        if not np.array_equal(ex.image_pyramid_level(l, frame, blurred=True), ref.blur(lv)):
            bad.append("%s: blurred level %d" % (tag, l))
        if not np.array_equal(ex.fast_candidates(l, frame), R.candidates(l)):
            bad.append("%s: candidates of level %d" % (tag, l))
    if K is not None and not (len(K) == len(K2) and K.tobytes() == K2.tobytes() and np.array_equal(D, D2)):
        bad.append("%s: keypoints / descriptors" % tag)
    return bad


@pytest.mark.parametrize("family", FAMILIES)
def test_stages_equal_oracle(extractors, family):
    bad = []
    for case in CASES:
        if case.name.split("/")[0] != family:
            continue
        ex = extractors(case.params)
        K, D = ex(case.img)
        R = ref.RefExtractor(*case.params)
        bad += _compare_frame(ex, R, case.img, case.params[2], 0, case.name, K, D)
    assert not bad, bad


def _batch_groups():
    """Three different cases of one geometry and parameters per batch."""
    groups = {}
    for case in CASES:
        groups.setdefault((case.img.shape, case.params), []).append(case)
    return [g[:3] for g in groups.values() if len(g) >= 3]


def test_batch_of_three_cases(extractors):
    groups = _batch_groups()
    assert len(groups) >= 10
    bad = []
    for group in groups:
        params = group[0].params
        ex = extractors(params)
        out = ex.extract_batch(np.stack([c.img for c in group]))
        for f, (case, (K, D)) in enumerate(zip(group, out)):
            bad += _compare_frame(ex, ref.RefExtractor(*params), case.img, params[2], f, "batch frame %d %s" % (f, case.name),
                                  K, D)
    assert not bad, bad


@pytest.mark.parametrize("staged", [False, True], ids=["in_place", "staged"])
def test_device_batch_level0_in_place_and_staged(extractors, staged):
    """orbx_extract_batch_device on three cases of 480 x 640: level 0 read where it lies (pitch = cols, aligned) or, from
    a pointer one byte off, staged into the internal plane first."""
    import torch
    from orb_slam2_ssd_semantic_b200 import _lib
    group = next(g for g in _batch_groups() if g[0].img.shape == (480, 640) and g[0].params[2] == 8)
    params = group[0].params
    ex = extractors(params)
    imgs = np.stack([c.img for c in group])
    F, rows, cols = imgs.shape
    buf = torch.zeros(F * rows * cols + 16, dtype=torch.uint8, device="cuda")
    off = 1 if staged else 0
    buf[off:off + F * rows * cols] = torch.from_numpy(imgs.reshape(-1)).cuda()
    torch.cuda.synchronize()
    _lib.check(_lib.lib().orbx_extract_batch_device(ex.handle, C.c_void_p(buf.data_ptr() + off), F, rows, cols, cols,
                                                    rows * cols))
    _lib.check(_lib.lib().orbx_sync(ex.handle))
    bad = []
    for f, case in enumerate(group):
        bad += _compare_frame(ex, ref.RefExtractor(*params), case.img, params[2], f, "device frame %d %s" % (f, case.name))
    assert not bad, bad


def test_readback_errors(extractors):
    from orb_slam2_ssd_semantic_b200 import ORBextractor, _lib
    L = _lib.lib()
    EINVAL, ECAP = -1, -2
    fresh = ORBextractor(1000, 1.2, 1, 20, 7)
    n = C.c_int(-7)
    buf = np.zeros((640, 3), np.int32)
    lvl = np.zeros((480, 640), np.uint8)
    ptr = buf.ctypes.data_as(C.c_void_p)
    assert L.orbx_get_candidates(fresh.handle, 0, 0, ptr, 640, C.byref(n)) == EINVAL   # nothing extracted yet
    assert L.orbx_get_level(fresh.handle, 0, 0, 2, lvl.ctypes.data_as(C.c_void_p), 640) == EINVAL
    case = next(c for c in CASES if c.name == "cells/straddle_49_50")
    ex = extractors(case.params)
    ex.extract_batch(np.stack([case.img, case.img]))
    for frame, level in ((-1, 0), (2, 0), (0, -1), (0, 1)):
        assert L.orbx_get_candidates(ex.handle, frame, level, ptr, 640, C.byref(n)) == EINVAL, (frame, level)
    for kind in (-1, 3):
        assert L.orbx_get_level(ex.handle, 0, 0, kind, lvl.ctypes.data_as(C.c_void_p), 640) == EINVAL
    assert L.orbx_get_level(ex.handle, 0, 0, 2, lvl.ctypes.data_as(C.c_void_p), 639) == EINVAL   # dst_stride < cols
    assert L.orbx_get_candidates(ex.handle, 1, 0, None, 0, None) == EINVAL
    buf[:] = -5
    n.value = -7
    assert L.orbx_get_candidates(ex.handle, 1, 0, ptr, 1, C.byref(n)) == ECAP
    assert n.value == 2 and (buf == -5).all()   # the count comes back, nothing is written
    assert L.orbx_get_candidates(ex.handle, 1, 0, ptr, 2, C.byref(n)) == 0
    assert n.value == 2 and buf[:2].tolist() == [[49, 100, 199], [50, 100, 199]] and (buf[2:] == -5).all()
