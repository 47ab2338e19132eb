"""CPU suite for the semantic object clusters (src/pointcloudmapping.cc:197-322, :399-488): the quirks of the oracle
(oracle/sem_ref.cpp) pinned against an independent Python restatement of draw_rect_with_depth_threshold, its 51-NN
against a float32 brute force and scipy's cKDTree, the flip count of the two unpinned PCL readings, sem_merge's
min-of-maxima, and the class_id range check of the C-ABI."""
import ctypes as C

import numpy as np
import pytest

from oracle import sem_py
from orb_slam2_ssd_semantic_b200._abi import GCM_BELOW_PROB, GCM_CLUSTER, GCM_FEW_POINTS
from tests import sem_scenes


def py_band(depth, x, y, w, h):
    """draw_rect_with_depth_threshold (:206-241) in Python: int / double conversions as written, float32 sums; indices
    outside the image skipped.  -> (indices, mean depth)."""
    rows, cols = depth.shape
    flat = depth.reshape(-1)
    f32 = np.float32
    beg = int(np.float32(x)) + (int(np.float32(y)) - 1) * cols - 1
    hi, wi = int(np.float32(h)), int(np.float32(w))
    s, n = f32(0), 0
    k = int(hi * 0.3)
    while k < hi * 0.7:
        start = beg + k * cols
        for j in range(int(start + wi * 0.3), int(start + wi * 0.7)):
            if 0 <= j < flat.size:
                d = flat[j]
                if not (d < 0.5 or d > 6):
                    s = f32(s + d)
                    n += 1
        k += 1
    thr = f32(s / f32(n)) if n else f32(0)
    idx = []
    for k in range(0, hi - 1):
        start = beg + k * cols
        for j in range(start, start + wi - 2):
            if 0 <= j < flat.size and float(abs(f32(flat[j] - thr))) < 0.4:
                idx.append(j)
    return np.array(idx, np.int64), thr


def _band(depth, x, y, w, h, cls=9):
    return sem_py.band(depth, (x, y, w, h, cls, 0.9))


def test_band_is_shifted_one_row_up_and_one_column_left():
    depth = np.full((30, 40), 2.0, np.float32)
    idx, thr = _band(depth, 10.0, 20.0, 6.0, 5.0)
    assert thr == np.float32(2.0)
    r, c = np.divmod(idx, 40)
    assert sorted(set(r)) == [19, 20, 21, 22] and sorted(set(c)) == [9, 10, 11, 12]     # h-1 rows, w-2 columns from (y-1, x-1)
    assert (idx == py_band(depth, 10.0, 20.0, 6.0, 5.0)[0]).all()


def test_band_wraps_at_the_right_edge_and_repeats_when_wider_than_the_image():
    depth = np.full((10, 8), 1.5, np.float32)
    idx, _ = _band(depth, 5.0, 2.0, 12.0, 3.0)          # w - 2 = 10 > cols = 8: rows overlap
    assert idx.tolist() == list(range(12, 22)) + list(range(20, 30))
    idx, _ = _band(depth, 6.0, 3.0, 5.0, 4.0)           # 3 columns from column 5: the third wraps into the next row
    assert idx.tolist() == [21, 22, 23, 29, 30, 31, 37, 38, 39]


def test_mean_depth_rows_truncate_int_height_times_point_three():
    depth = np.full((40, 40), 1.0, np.float32)
    depth[:, :] = (1.0 + 0.1 * np.arange(40, dtype=np.float32))[:, None]   # one value per row
    # h = 9.9: (int)h = 9, rows k from (int)(9*0.3) = 2 while k < 6.3 -> k = 2..6 of the rectangle from row y - 1 = 4
    _, thr = _band(depth, 10.0, 5.0, 10.0, 9.9)
    _, py_thr = py_band(depth, 10.0, 5.0, 10.0, 9.9)
    rows = np.arange(4 + 2, 4 + 7)
    # columns (int)(start + 3.0) .. (int)(start + 7.0) - 1: 4 per row, 5 rows
    s = np.float32(0)
    for r in rows:
        for _ in range(4):
            s = np.float32(s + depth[r, 0])
    assert thr == py_thr == np.float32(s / np.float32(20))


def test_band_edge_is_a_float_difference_compared_with_double_point_four():
    # thr = 0 (no valid depth in the mean window): |d| < 0.4 in double -- 0.4f itself is 0.40000000596 and stays out
    depth = np.zeros((12, 12), np.float32)
    below = np.nextafter(np.float32(0.4), np.float32(0))
    depth[5, 5], depth[5, 6] = np.float32(0.4), below
    idx, thr = _band(depth, 2.0, 2.0, 10.0, 10.0)
    assert thr == 0 and 5 * 12 + 6 in idx and 5 * 12 + 5 not in idx
    # thr = 0.5: d - thr rounds in float for d near 0.1; find d where the float and the exact difference disagree
    d0 = np.float32(0.1)
    cands = [np.float32(d0 + np.float32(k) * np.float32(2 ** -27)) for k in range(-64, 64)]
    flip = [d for d in cands if (float(abs(np.float32(d - np.float32(0.5)))) < 0.4) != (abs(float(d) - 0.5) < 0.4)]
    assert flip
    d = flip[0]
    depth = np.full((12, 12), 0.5, np.float32)
    depth[1, 1] = d                                        # inside the band rows, outside the mean window
    idx, thr = _band(depth, 2.0, 2.0, 10.0, 10.0)
    assert thr == np.float32(0.5)
    assert (13 in idx) == (float(abs(np.float32(d - thr))) < 0.4)


def test_zero_mean_count_selects_missing_depth_pixels():
    depth = np.full((20, 20), 3.0, np.float32)
    depth[2:12, 2:12] = 0.0                                 # the whole box missing: the mean window counts nothing
    depth[3, 3] = 0.3
    idx, thr = _band(depth, 3.0, 3.0, 10.0, 10.0)
    py_idx, py_thr = py_band(depth, 3.0, 3.0, 10.0, 10.0)
    assert thr == py_thr == 0 and (idx == py_idx).all() and len(idx) == 9 * 8


def test_out_of_image_indices_are_skipped():
    depth = np.full((20, 30), 2.0, np.float32)
    for x, y, w, h in ((0.0, 0.0, 10.0, 6.0), (0.5, 0.9, 10.0, 6.0), (25.0, 17.0, 12.0, 9.0), (-4.0, 5.0, 8.0, 4.0)):
        idx, thr = _band(depth, x, y, w, h)
        py_idx, py_thr = py_band(depth, x, y, w, h)
        assert (idx == py_idx).all() and thr == py_thr and idx.min() >= 0 and idx.max() < depth.size


def test_crafted_scenes_match_the_python_band():
    for name in ("overlap", "edges", "small_missing"):
        depth, _, _, objs = sem_scenes.scene(name)
        for o in objs:
            idx, thr = sem_py.band(depth, o)
            py_idx, py_thr = py_band(depth, *o[:4])
            assert (idx == py_idx).all() and (thr == py_thr or (np.isnan(thr) and np.isnan(py_thr))), (name, o)


def test_prob_gate_and_the_skip_rule():
    depth, bgr, T, _ = sem_scenes.scene("overlap")
    fx, fy, cx, cy = 517.3, 516.5, 318.6, 255.3
    box = (100.0, 80.0, 60.0, 40.0, 9)
    recs, _, cloud = sem_py.keyframe(depth, bgr, T, fx, fy, cx, cy, 2, [box + (float(np.float32(0.54)),)], 0.04)
    assert recs[0].status == GCM_CLUSTER and cloud is not None          # 0.54f > 0.54 as double
    low = box + (float(np.nextafter(np.float32(0.54), np.float32(0))),)
    recs, painted, cloud = sem_py.keyframe(depth, bgr, T, fx, fy, cx, cy, 2, [low], 0.04)
    assert recs[0].status == GCM_BELOW_PROB and cloud is not None        # a low-prob object still prevents the skip
    assert (painted == bgr).all()
    assert sem_py.keyframe(depth, bgr, T, fx, fy, cx, cy, 2, [], 0.04)[2] is None
    assert sem_py.keyframe(depth, bgr, T, fx, fy, cx, cy, 3, [], 0.04)[2] is not None


def test_few_band_points_give_no_cluster():
    rng = np.random.Generator(np.random.PCG64(1))
    assert sem_py.cluster(rng.normal(size=(50, 3)), 0.04).status == GCM_FEW_POINTS
    assert sem_py.cluster(rng.normal(size=(51, 3)), 0.04).status == GCM_CLUSTER


def test_knn_matches_float32_brute_force_and_ckdtree():
    from scipy.spatial import cKDTree
    rng = np.random.Generator(np.random.PCG64(7))
    xyz = rng.normal(0, 0.3, (400, 3)).astype(np.float32) + np.float32(2.0)
    xyz[10:14] = xyz[3]                                     # repeated indices of a band are duplicate points
    nn = sem_py.knn(xyz, 51)
    d = xyz[:, None, :] - xyz[None, :, :]
    sq = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]     # float32, no FMA
    assert (nn == np.sort(sq, axis=1)[:, :51]).all()
    assert (nn[:, 0] == 0).all() and (nn[3, :5] == 0).all()
    _, ii = cKDTree(xyz.astype(np.float64)).query(xyz.astype(np.float64), 51)
    for q in range(len(xyz)):
        assert (np.sort(sq[q, ii[q]]) == nn[q]).all()


FLIPS = {"sqrt in float": 0, "sq_sum in double": 0}


def test_flip_count_of_the_unpinned_pcl_readings():
    """The keep decisions of every box of the scenes (tests/sem_scenes.py) under the chosen reading of PCL 1.7.2 and
    under the other reading of each unpinned line; DESIGN.md §2 reports these counts."""
    fx, fy, cx, cy = 517.3, 516.5, 318.6, 255.3
    counts = {"sqrt in float": 0, "sq_sum in double": 0}
    total = 0
    for name in sem_scenes.NAMES:
        depth, bgr, T, objs = sem_scenes.scene(name)
        _, _, cloud = sem_py.keyframe(depth, bgr, T, fx, fy, cx, cy, 1, [], sem_scenes.LEAF)
        xyz = cloud[0]
        for o in objs:
            if not o[5] > 0.54:
                continue
            idx, _ = sem_py.band(depth, o)
            if len(idx) < 51:
                continue
            pts = xyz[idx]
            d0, k0 = sem_py.sor(pts)
            d1, k1 = sem_py.sor(pts, sem_py.ALT_SQRT)
            d2, k2 = sem_py.sor(pts, sem_py.ALT_SQSUM)
            counts["sqrt in float"] += int((k0 != k1).sum())
            counts["sq_sum in double"] += int((k0 != k2).sum())
            total += len(pts)
    print("keep decisions over %d band points: %s" % (total, counts))
    assert total > 100000
    assert counts == FLIPS


def test_sem_merge_keeps_the_min_of_the_maxima():
    from orb_slam2_ssd_semantic_b200 import SemanticClusters
    db = SemanticClusters()
    db.merge("chair", 9, np.float32(0.8), [1.0, 0.0, 2.0], [0.5, -0.5, 1.5], [1.5, 0.5, 2.5])
    db.merge("chair", 9, np.float32(0.6), [1.2, 0.1, 2.1], [0.4, -0.2, 1.6], [1.9, 0.4, 2.9])   # 0.245 m < 0.5 m: merged
    assert len(db.clusters) == 1
    c = db.clusters[0]
    f = np.float32
    assert c["prob"] == f(np.float64(f(0.8) + f(0.6)) / 2.0)
    assert (c["centroid"] == (f([1.0, 0.0, 2.0]) + f([1.2, 0.1, 2.1])) / f(2)).all()
    assert (c["minPt"] == np.float32([0.4, -0.5, 1.5])).all()
    assert (c["maxPt"] == np.float32([1.5, 0.4, 2.5])).all()      # element-wise MIN of the maxima, as the reference writes it
    db.merge("chair", 9, np.float32(0.9), [3.0, 0.0, 2.0], [2.5, -0.5, 1.5], [3.5, 0.5, 2.5])   # too far: a new one
    db.merge("person", 15, np.float32(0.9), [1.1, 0.05, 2.05], [0, 0, 0], [1, 1, 1])            # other name: a new one
    assert [x["object_name"] for x in db.clusters] == ["chair", "chair", "person"]
    db.merge("bottle", 5, np.float32(0.9), [0, 0, 0], [0, 0, 0], [1, 1, 1])
    db.merge("bottle", 5, np.float32(0.9), [0.06, 0, 0], [0, 0, 0], [1, 1, 1])   # 0.06 is not < obj_size_[5] = 0.06f
    assert len(db.clusters) == 5


def test_abi_rejects_class_ids_outside_the_21_entry_tables():
    import orb_slam2_ssd_semantic_b200 as pkg
    from orb_slam2_ssd_semantic_b200._abi import GcmCluster, gcm_objects
    L = pkg.lib()
    depth = np.zeros((4, 4), np.float32)
    bgr = np.zeros((4, 4, 3), np.uint8)
    T = np.eye(4, dtype=np.float32)
    out = (GcmCluster * 1)()
    for cls, expect in ((21, "class_id 21"), (-1, "class_id -1"), (20, "bad argument"), (0, "bad argument")):
        o = gcm_objects([(1.0, 1.0, 2.0, 2.0, cls, 0.9)])
        for fn in (L.gcm_add_keyframe_objects, L.gcm_add_keyframe_objects_device):
            rc = fn(None, depth.ctypes.data_as(C.c_void_p), bgr.ctypes.data_as(C.c_void_p), 4, 4, T.ctypes.data_as(C.c_void_p),
                    1.0, 1.0, 1.0, 1.0, 1, o.ctypes.data_as(C.c_void_p), 1, out)
            assert rc == -1 and expect in L.b200orb_last_error().decode(), (cls, L.b200orb_last_error())
    o = gcm_objects([(float("nan"), 1.0, 2.0, 2.0, 3, 0.9)])
    rc = L.gcm_add_keyframe_objects(None, depth.ctypes.data_as(C.c_void_p), bgr.ctypes.data_as(C.c_void_p), 4, 4,
                                    T.ctypes.data_as(C.c_void_p), 1.0, 1.0, 1.0, 1.0, 1, o.ctypes.data_as(C.c_void_p), 1, out)
    assert rc == -1 and "rectangle" in L.b200orb_last_error().decode()
