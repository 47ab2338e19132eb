"""GPU parity of the keyframe -> point cloud -> occupancy path vs the CPU oracle, bit for bit: points (equal as sets of
float32 bit patterns), leaf sets, log-odds.  The library is built with --fmad=false and the oracle with -ffp-contract=off,
every cell sums its pixels in row-major order and every voxel replays its updates in keyframe order, so the two are
bit-equal by construction; a tolerance would hide a reordered sum."""
import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth

pytestmark = pytest.mark.gpu


def _sorted_pts(xyz):
    """Rows of float32 bit patterns, sorted: equal point clouds give equal arrays."""
    b = np.ascontiguousarray(xyz, np.float32).view(np.uint32)
    return b[np.lexsort(b.T[::-1])]


def _leaf_dict(keys, lo):
    k = keys.astype(np.uint64)
    packed = k[:, 0] | (k[:, 1] << np.uint64(16)) | (k[:, 2] << np.uint64(32))
    o = np.argsort(packed)
    return packed[o], lo[o]


def _scene(n):
    ws = synth.WallStream(seed=99, n=n, depth0=2.0)
    out = []
    for t in range(n):
        gray, depth, rgb, T = ws.frame(t * 7)
        # add relief so rays / voxels vary: a tilted depth ramp + a box in front
        yy, xx = np.mgrid[0:480, 0:640]
        depth = (depth + 0.3 * np.sin(xx / 90.0) * np.cos(yy / 70.0)).astype(np.float32)
        depth[100:200, 150:300] = 1.1
        depth[::50, ::60] = 0.0      # invalid pixels
        depth[300:320, 400:460] = 3.7   # beyond depth_max
        out.append((depth, rgb, T))
    return out


@pytest.mark.parametrize("mode", ["nonground", "floor_ground"])
def test_insert_keyframes_match_oracle(oracle, mode):
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    scene = _scene(5)
    gpu = PointCloudMapping(0.05)
    ref = oracle.RefOccupancy()
    for depth, rgb, T in scene:
        label = None
        if mode == "floor_ground":
            label = np.zeros(depth.shape, np.uint8)
            label[300:, :] = 1          # lower image part is "ground": exercises the ray casting
        gpu.insertKeyFrame(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, label)
        ref.insert_keyframe(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, label)
        pg, _ = gpu.last_points()
        pr, _, _ = ref.last_points()
        assert len(pg) == len(pr) and len(pr) > 1000
        assert (_sorted_pts(pg) == _sorted_pts(pr)).all()
    kg, lg, _ = gpu.export_leaves()
    kr, lr = ref.export_leaves()
    pk_g, lo_g = _leaf_dict(kg, lg)
    pk_r, lo_r = _leaf_dict(kr, lr)
    assert len(pk_r) > 500
    assert len(pk_g) == len(pk_r) and (pk_g == pk_r).all()
    assert (lo_g.view(np.uint32) == lo_r.view(np.uint32)).all()
    assert gpu.num_leaves() == len(pk_r)
    if mode == "floor_ground":
        assert (lo_r < 0).sum() > 100     # free cells were carved


def test_clamping_and_query(oracle):
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    depth, rgb, T = _scene(1)[0]
    gpu = PointCloudMapping(0.05)
    ref = oracle.RefOccupancy()
    for _ in range(8):   # same keyframe over and over: values must saturate at the clamp
        gpu.insertKeyFrame(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY)
        ref.insert_keyframe(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY)
    kg, lg, _ = gpu.export_leaves()
    kr, lr = ref.export_leaves()
    a, b = _leaf_dict(kg, lg), _leaf_dict(kr, lr)
    assert (a[0] == b[0]).all() and (a[1].view(np.uint32) == b[1].view(np.uint32)).all()
    hit, miss, cmin, cmax = ref.constants()
    assert np.isclose(lg.max(), cmax) and lg.max() <= cmax + 1e-6
    pts, _ = gpu.last_points()
    v = gpu.query(pts[0])
    assert v is not None and v > 0
    assert gpu.query(np.array([50.0, 50.0, 50.0], np.float32)) is None


def test_no_leaf_filter_and_other_resolution(oracle):
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    depth, rgb, T = _scene(2)[1]
    gpu = PointCloudMapping(0.1, leaf=0.0, depth_max=4.0)
    ref = oracle.RefOccupancy(resolution=0.1, leaf=0.0, depth_max=4.0)
    gpu.insertKeyFrame(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY)
    ref.insert_keyframe(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY)
    pg, _ = gpu.last_points()
    pr, _, _ = ref.last_points()
    assert len(pg) == len(pr)
    assert (_sorted_pts(pg) == _sorted_pts(pr)).all()
    a, b = _leaf_dict(*gpu.export_leaves()[:2]), _leaf_dict(*ref.export_leaves())
    assert (a[0] == b[0]).all() and (a[1].view(np.uint32) == b[1].view(np.uint32)).all()


def test_save_octomap_round_trip(oracle, tmp_path):
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    from orb_slam2_ssd_semantic_b200 import octree_io as O
    gpu = PointCloudMapping(0.05)
    for depth, rgb, T in _scene(3):
        gpu.insertKeyFrame(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY)
    path = str(tmp_path / "map.ot")
    nleaves, nnodes = gpu.SaveOctoMap(path)
    res, nodes, hdr = O.read_ot(path)
    assert hdr.startswith("# Octomap OcTree file") and "id ColorOcTree" in hdr and res == 0.05
    keys, depths, vals, cols, consistent, used = O.leaves_from_nodes(nodes)
    assert consistent and used == len(nodes) == nnodes
    k16, v16, _ = O.expand_to_max_depth(keys, depths, vals, cols)
    kg, lg, _ = gpu.export_leaves()
    a, b = _leaf_dict(k16, v16), _leaf_dict(kg, lg)
    assert len(a[0]) == nleaves and (a[0] == b[0]).all() and (a[1] == b[1]).all()


def test_host_u16_keyframe_batch_equals_per_keyframe_inserts(oracle):
    """ocm_insert_keyframes_u16_labeled (CV_16U depth + colour from host buffers, one asynchronous call) builds the same
    map as the per-keyframe float-depth inserts and as the oracle."""
    import torch
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    scene = _scene(4)
    d16 = np.stack([np.rint(d.astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16) for d, _, _ in scene])
    factor = np.float32(1.0 / synth.DEPTH_FACTOR)
    depth = d16.astype(np.float32) * factor
    rgb = np.ascontiguousarray(np.stack([c for _, c, _ in scene]))
    T = np.stack([t for _, _, t in scene]).astype(np.float32)
    a = PointCloudMapping(0.05)
    p16, prgb = torch.from_numpy(d16).pin_memory(), torch.from_numpy(rgb).pin_memory()
    a.insert_keyframes_u16(p16.numpy(), prgb.numpy(), factor, T, synth.FX, synth.FY, synth.CX, synth.CY)
    a.insert_keyframes_u16(p16.numpy()[:0], prgb.numpy()[:0], factor, T[:0], synth.FX, synth.FY, synth.CX, synth.CY)   # n = 0
    a.sync()
    b = PointCloudMapping(0.05)
    ref = oracle.RefOccupancy()
    for i in range(len(scene)):
        b.insertKeyFrame(T[i], depth[i], rgb[i], synth.FX, synth.FY, synth.CX, synth.CY)
        ref.insert_keyframe(T[i], depth[i], rgb[i], synth.FX, synth.FY, synth.CX, synth.CY, None)
    ka, la, _ = a.export_leaves()
    kb, lb, _ = b.export_leaves()
    kr, lr = ref.export_leaves()
    pa, va = _leaf_dict(ka, la)
    pb, vb = _leaf_dict(kb, lb)
    pr, vr = _leaf_dict(kr, lr)
    assert len(pr) > 500 and (pa == pb).all() and (va == vb).all()
    assert len(pa) == len(pr) and (pa == pr).all() and (va.view(np.uint32) == vr.view(np.uint32)).all()
    with pytest.raises(ValueError):
        a.insert_keyframes_u16(d16.astype(np.int32), rgb, factor, T, synth.FX, synth.FY, synth.CX, synth.CY)


def test_global_cloud_refilter_matches_oracle(oracle):
    """T variant (src/pointcloudmapping.cc:131-194, 482-493): every pixel back-projected (no gate), accumulated, and the
    whole map re-filtered by VoxelGrid(resolution) after each batch -- point for point (cell order) against the oracle;
    the second round filters the previous centroids together with the new keyframes."""
    from orb_slam2_ssd_semantic_b200 import GlobalCloudMapping
    scene = _scene(4)
    leaf = 0.04
    gpu = GlobalCloudMapping(leaf)
    acc_xyz = np.zeros((0, 3), np.float32)
    acc_rgb = np.zeros((0, 3), np.uint8)
    for rnd in range(2):
        for depth, bgr, T in scene[2 * rnd:2 * rnd + 2]:
            d = depth.copy()
            d[5, 7] = np.nan                       # removed by removeNaNFromPointCloud
            gpu.insertKeyFrame(T, d, bgr, synth.FX, synth.FY, synth.CX, synth.CY)
            pts = oracle.backproject_all(d, T, synth.FX, synth.FY, synth.CX, synth.CY)
            acc_xyz = np.concatenate([acc_xyz, pts])
            acc_rgb = np.concatenate([acc_rgb, bgr.reshape(-1, 3)[:, ::-1]])
        assert gpu.size() == len(acc_xyz)
        gpu.refilter()
        acc_xyz, acc_rgb = oracle.global_refilter(acc_xyz, acc_rgb, leaf)
        gx, gc = gpu.points()
        assert len(gx) == len(acc_xyz) and len(acc_xyz) > 1000
        assert (gx.view(np.uint32) == acc_xyz.view(np.uint32)).all()   # same order, same float sums: bit-equal
        assert (gc == acc_rgb).all()
    with pytest.raises(Exception):
        GlobalCloudMapping(0.0)


def test_more_keyframes_than_batch_slots(oracle):
    """One ocm_insert_keyframes_u16_labeled call with 40 keyframes (the batch masks hold 32: the call is split into rounds
    and the scratch slots are reused) builds the same map as 40 single inserts."""
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    base = _scene(5)
    n = 40
    d16 = np.stack([np.rint(base[i % 5][0].astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16) for i in range(n)])
    rgb = np.ascontiguousarray(np.stack([base[i % 5][1] for i in range(n)]))
    T = np.stack([base[i % 5][2] for i in range(n)]).astype(np.float32)
    factor = np.float32(1.0 / synth.DEPTH_FACTOR)
    a = PointCloudMapping(0.05)
    a.insert_keyframes_u16(d16, rgb, factor, T, synth.FX, synth.FY, synth.CX, synth.CY)
    a.sync()
    b = PointCloudMapping(0.05)
    depth = d16.astype(np.float32) * factor
    for i in range(n):
        b.insertKeyFrame(T[i], depth[i], rgb[i], synth.FX, synth.FY, synth.CX, synth.CY)
    pa, va = _leaf_dict(*a.export_leaves()[:2])
    pb, vb = _leaf_dict(*b.export_leaves()[:2])
    assert len(pa) > 500 and (pa == pb).all() and (va == vb).all()
    assert va.max() > 3.0     # repeated hits ran into the upper clamp: the replay order mattered


def test_config4_shape_120_keyframes_with_ground_rays(oracle):
    """BASELINE.json configs[3] shape at a size the CPU oracle finishes in seconds: 120 keyframes of the room stream (every
    3rd frame of a 360-frame path: walls, floor, ceiling enter and leave the 0.5 - 3 m gate), 0.05 m voxels, 1 cm
    pre-filter, both label modes -- A: all non-ground (no rays), B: GT floor as ground (free-space rays) -- inserted in
    batches of 40 (rounds of 32 mask bits + remainder): leaf set, log-odds and the points of the last keyframe bit-equal."""
    import torch
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    rs = synth.RoomStream(seed=77, n=361)
    fr = [rs.frame(3 * t, with_label=True) for t in range(120)]
    depth, rgb = np.stack([f[1] for f in fr]), np.stack([f[2] for f in fr])
    T, label = np.stack([f[3] for f in fr]).astype(np.float32), np.stack([f[4] for f in fr])
    d_depth, d_rgb, d_lab = torch.from_numpy(depth).cuda(), torch.from_numpy(rgb).cuda(), torch.from_numpy(label).cuda()
    for mode in ("A", "B"):
        pcm = PointCloudMapping(0.05)
        ref = oracle.RefOccupancy()
        for b in range(0, 120, 40):
            idx = list(range(b, b + 40))
            pcm.insert_keyframes_device(d_depth.data_ptr(), d_rgb.data_ptr(), 480, 640, idx, T[idx], synth.FX, synth.FY, synth.CX,
                                        synth.CY, d_label=d_lab.data_ptr() if mode == "B" else 0)
        pcm.sync()
        ref.insert_keyframes_mt(depth, rgb, label if mode == "B" else None, list(range(120)), T, synth.FX, synth.FY, synth.CX,
                                synth.CY, 8)
        kr, lr = ref.export_leaves()
        kg, lg, _ = pcm.export_leaves()
        pk = lambda k: k.astype(np.uint64)[:, 0] | (k.astype(np.uint64)[:, 1] << np.uint64(16)) | (k.astype(np.uint64)[:, 2] << np.uint64(32))
        og, orr = np.argsort(pk(kg)), np.argsort(pk(kr))
        assert len(kg) == len(kr) > 20000 and (pk(kg)[og] == pk(kr)[orr]).all(), mode
        assert (lg[og].view(np.uint32) == lr[orr].view(np.uint32)).all(), mode
        if mode == "B":
            assert (lr < 0).sum() > 10000
        xg, _ = pcm.last_points()
        xr, _, _ = ref.last_points()
        assert len(xg) == len(xr)
        assert (_sorted_pts(xg) == _sorted_pts(xr)).all()


def test_sparse_keyframe_under_50_points_is_all_ground(oracle):
    """perfect/src/MapDrawer.cc:676-680: a cloud of fewer than 50 points skips the plane extraction and becomes ALL ground:
    free-space rays only, no occupied endpoint -- whatever label is (or is not) supplied."""
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    rs = synth.RoomStream(seed=5, n=4)
    gray, depth, rgb, T, lab = rs.frame(1, with_label=True)
    sparse = np.zeros_like(depth)
    ys, xs = np.mgrid[60:420:60, 80:560:80]
    sparse[ys, xs] = np.clip(depth[ys, xs], 0.6, 2.9)          # 36 valid pixels, far apart: 36 points after the 1 cm filter
    for label in (None, np.zeros_like(lab)):
        pcm, ref = PointCloudMapping(0.05), oracle.RefOccupancy()
        pcm.insertKeyFrame(T, sparse, rgb, synth.FX, synth.FY, synth.CX, synth.CY, label)
        ref.insert_keyframe(T, sparse, rgb, synth.FX, synth.FY, synth.CX, synth.CY, label)
        kg, lg, _ = pcm.export_leaves()
        kr, lr = ref.export_leaves()
        assert len(ref.last_points()[0]) == 36
        a = {tuple(k): v for k, v in zip(kg.tolist(), lg.tolist())}
        b = {tuple(k): v for k, v in zip(kr.tolist(), lr.tolist())}
        assert a.keys() == b.keys() and len(a) > 100
        assert all(np.float32(a[k]).view(np.uint32) == np.float32(b[k]).view(np.uint32) for k in a)
        assert max(b.values()) < 0          # only misses: nothing became occupied
