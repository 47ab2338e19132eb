"""One handle of each kind driven through a sequence that grows or replaces every one of its buffer blocks. Every call's
outputs must equal, bit for bit, those of a fresh handle given the same input (the maps: the oracle, as in
test_mapping_gpu.py, since a map's state is its whole history)."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth
from tests.helpers import frame_views

pytestmark = pytest.mark.gpu


def _leaf_dict(keys, lo):
    k = keys.astype(np.uint64)
    packed = k[:, 0] | (k[:, 1] << np.uint64(16)) | (k[:, 2] << np.uint64(32))
    o = np.argsort(packed)
    return packed[o], lo[o]


def _same_leaves(gpu, ref):
    (pg, lg), (pr, lr) = _leaf_dict(*gpu.export_leaves()[:2]), _leaf_dict(*ref.export_leaves())
    assert len(pr) > 500 and len(pg) == len(pr) and (pg == pr).all()
    assert (lg.view(np.uint32) == lr.view(np.uint32)).all()


def test_extractor_geometry_and_batch_changes():
    """Small geometry, a larger one, the small one again, then a larger batch: the geometry block is re-carved, the
    download staging and the bordered-level scratch grow."""
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    frames = np.stack([synth.synth_frame(77, t) for t in range(4)])
    small = np.ascontiguousarray(frames[:, :240, :320])
    args = (1000, 1.2, 8, 20, 7)
    ex = ORBextractor(*args)
    for imgs in (small[:1], frames[:2], small[:1], frames):
        fresh = ORBextractor(*args)
        got, want = ex.extract_batch(imgs), fresh.extract_batch(imgs)
        assert len(got) == len(want) == len(imgs)
        for (k, d), (k2, d2) in zip(got, want):
            assert len(k) > 100 and k.tobytes() == k2.tobytes() and d.tobytes() == d2.tobytes()
        for level in (0, 3):
            a = ex.image_pyramid_level(level, len(imgs) - 1, bordered=True)
            assert a.tobytes() == fresh.image_pyramid_level(level, len(imgs) - 1, bordered=True).tobytes()


def test_matcher_arena_grows(oracle):
    """SearchByProjection(cur, last) of increasing size on one matcher: its arena grows between the calls."""
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    ws = synth.WallStream(seed=1234, n=4)
    (g0, d0, _, T0), (g1, d1, _, T1) = ws.frame(0), ws.frame(1)
    m = ORBmatcher(0.9, True)
    for nfeat in (300, 1000, 3000):
        R = oracle.RefExtractor(nfeat, 1.2, 8, 20, 7)
        (Kl, Dl), (Kc, Dc) = R(g0), R(g1)
        cur, last = frame_views(oracle, Kc, Dc, d1, T1, Kl, Dl, d0, T0, R.mvScaleFactor)
        n, c2l = m.SearchByProjection(cur, last, 15.0, False)
        n2, c2l2 = ORBmatcher(0.9, True).SearchByProjection(cur, last, 15.0, False)
        assert n > 50 and n == n2 and c2l.tobytes() == c2l2.tobytes(), nfeat


def test_vocabulary_io_grows(oracle):
    """orbv_transform of increasing n on one vocabulary: the io block grows."""
    from orb_slam2_ssd_semantic_b200 import ORBVocabulary
    k, L = 10, 4
    parent, nd, w = oracle.synth_vocabulary(5, k, L)
    rng = np.random.default_rng(5)
    leaves = np.nonzero(w > 0)[0]
    voc = ORBVocabulary(k, L, parent, nd, w)
    for n in (10, 1000, 50000):
        desc = nd[rng.choice(leaves, n)].copy()
        desc[:, :2] ^= rng.integers(0, 256, size=(n, 2), dtype=np.uint8)
        got, want = voc.transform_raw(desc, 2), ORBVocabulary(k, L, parent, nd, w).transform_raw(desc, 2)
        for a, b in zip(got, want):
            assert a.tobytes() == b.tobytes(), n


def test_dynamic_mask_sizes_and_capacities():
    """Mask sizes and keypoint counts up and down on one handle: its block is re-carved for every entry's buffer list."""
    from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    rng = np.random.Generator(np.random.PCG64(3))
    dm = DynamicMask()
    masks = []
    for rows, cols, seed in ((60, 80, 1), (240, 320, 2), (120, 160, 3)):
        flow = synth.flow_field(seed, rows, cols)
        mask = dm.mask_from_flow(flow)
        assert mask.tobytes() == DynamicMask().mask_from_flow(flow).tobytes()
        masks.append(mask)
    for mask, n in ((masks[0], 100), (masks[1], 3000), (masks[2], 500), (masks[1], 20000)):
        h, w = mask.shape
        kps = np.zeros(n, KP_DTYPE)
        kps["x"] = rng.uniform(0, w - 1, n).astype(np.float32)
        kps["y"] = rng.uniform(0, h - 1, n).astype(np.float32)
        kps["octave"] = rng.integers(0, 8, n)
        desc = rng.integers(0, 256, (n, 32)).astype(np.uint8)
        k, d = dm.filter_keypoints(mask, kps, desc)
        k2, d2 = DynamicMask().filter_keypoints(mask, kps, desc)
        assert k.tobytes() == k2.tobytes() and d.tobytes() == d2.tobytes(), n


def test_global_cloud_grows_three_times_before_refilter(oracle):
    """Five keyframes grow the point block four times (capacity 1, 2, 4, 8 keyframes) before the first refilter; two
    more keyframes and a second refilter reuse the sort block."""
    from orb_slam2_ssd_semantic_b200 import GlobalCloudMapping
    ws = synth.WallStream(seed=5, n=8, depth0=2.0)
    leaf = 0.04
    gpu = GlobalCloudMapping(leaf)
    acc_xyz = np.zeros((0, 3), np.float32)
    acc_rgb = np.zeros((0, 3), np.uint8)
    for rnd in (range(5), range(5, 7)):
        for t in rnd:
            _, depth, bgr, T = ws.frame(3 * t)
            gpu.insertKeyFrame(T, depth, bgr, synth.FX, synth.FY, synth.CX, synth.CY)
            acc_xyz = np.concatenate([acc_xyz, oracle.backproject_all(depth, T, synth.FX, synth.FY, synth.CX, synth.CY)])
            acc_rgb = np.concatenate([acc_rgb, bgr.reshape(-1, 3)[:, ::-1]])
        assert gpu.size() == len(acc_xyz)
        gpu.refilter()
        acc_xyz, acc_rgb = oracle.global_refilter(acc_xyz, acc_rgb, leaf)
        gx, gc = gpu.points()
        assert len(gx) == len(acc_xyz) > 1000
        assert np.abs(gx - acc_xyz).max() <= 1e-5
        assert (gc == acc_rgb).all()


def test_occupancy_scratch_staging_export_and_merge(oracle):
    """A change of image size (scratch slots replaced), staging growth (1 then 3 host keyframes), ocm_export_leaves with
    cap 0, a cap one short and the exact cap.  A world-1 merge closes an epoch after the first, small keyframe and
    another after everything else, so the merge buffers grow; a world-1 merge leaves the map as it is."""
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping, _lib
    from orb_slam2_ssd_semantic_b200._abi import ptr
    ws = synth.WallStream(seed=99, n=12, depth0=2.0)
    frames = [ws.frame(5 * t) for t in range(7)]
    gpu, ref = PointCloudMapping(0.05), oracle.RefOccupancy()
    cam = (synth.FX, synth.FY, synth.CX, synth.CY)

    def insert_f32(depth, rgb, T):
        gpu.insertKeyFrame(T, depth, rgb, *cam)
        ref.insert_keyframe(T, depth, rgb, *cam)
        pg, pr = gpu.last_points()[0], ref.last_points()[0]
        assert len(pg) == len(pr) > 100
        rows = lambda p: p.view(np.uint32)[np.lexsort(p.view(np.uint32).T[::-1])]   # noqa: E731
        assert (rows(pg) == rows(pr)).all()

    def insert_u16(ts):
        factor = np.float32(1 / 5000.0)
        d16 = np.stack([np.round(frames[t][1] * 5000).astype(np.uint16) for t in ts])
        rgb = np.stack([frames[t][2] for t in ts])
        T = np.stack([frames[t][3] for t in ts])
        gpu.insert_keyframes_u16(d16, rgb, float(factor), T, *cam)
        gpu.sync()
        for i in range(len(ts)):
            ref.insert_keyframe(T[i], d16[i].astype(np.float32) * factor, rgb[i], *cam)

    _, depth, rgb, T = frames[0]
    insert_f32(np.ascontiguousarray(depth[:240, :320]), np.ascontiguousarray(rgb[:240, :320]), T)
    sent = [gpu.merge().records_sent]
    insert_f32(depth, rgb, T)
    insert_u16([1])
    insert_u16([2, 3, 4])
    _same_leaves(gpu, ref)

    L = _lib.lib()
    n = gpu.num_leaves()
    keys, lo, col = np.zeros((n, 3), np.uint16), np.zeros(n, np.float32), np.zeros((n, 3), np.uint8)
    cnt = C.c_int64(-1)
    for cap in (0, n - 1):
        assert L.ocm_export_leaves(gpu.handle, ptr(keys), ptr(lo), ptr(col), cap, C.byref(cnt)) == -2   # B200ORB_ECAP
        assert cnt.value == n
    assert L.ocm_export_leaves(gpu.handle, ptr(keys), ptr(lo), ptr(col), n, C.byref(cnt)) == 0 and cnt.value == n
    pg, lg = _leaf_dict(keys, lo)
    pr, lr = _leaf_dict(*ref.export_leaves())
    assert (pg == pr).all() and (lg.view(np.uint32) == lr.view(np.uint32)).all()

    for t in (5, 6):
        insert_f32(*frames[t][1:])
    sent.append(gpu.merge().records_sent)
    _same_leaves(gpu, ref)
    assert 0 < sent[0] < sent[1]
