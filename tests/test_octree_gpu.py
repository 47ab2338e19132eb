"""GPU: the pruned ColorOcTree built on the device (ocm_tree_build / ocm_write_ot / ocm_tree_leaves) equals
octree_io.build_ot -- the numpy oracle pinned to the reference's own octomap.ot -- byte for byte; `.ot` files load into a
map (ocm_read_ot) that continues exactly where the saved one stopped; whatever is refused leaves the map as it was."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import octree_io as O
from orb_slam2_ssd_semantic_b200 import synth
from tests import occ_scenes as S
from tests.test_octree_cpu import reference_bytes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, ECAP = -1, -2


def _pcm(res=0.05, **kw):
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping
    return PointCloudMapping(res, **kw)


def _sorted_cells(keys, vals, cols):
    """Cells as rows (packed key, log-odds bits, packed colour), sorted by key: equal maps give equal arrays."""
    k = keys.astype(np.uint64)
    packed = k[:, 0] | (k[:, 1] << np.uint64(16)) | (k[:, 2] << np.uint64(32))
    c = cols.astype(np.uint64)
    o = np.argsort(packed)
    return np.stack([packed, np.ascontiguousarray(vals, np.float32).view(np.uint32).astype(np.uint64),
                     c[:, 0] | (c[:, 1] << np.uint64(8)) | (c[:, 2] << np.uint64(16))], 1)[o]


def assert_tree_equals_oracle(pcm, res):
    """Device tree of the map == build_ot(export_leaves) byte for byte, pruned leaves == leaves_from_nodes.  -> bytes."""
    k, v, c = pcm.export_leaves()
    expect = O.build_ot(k, v, c, res, "%g" % res)
    nn, nl = pcm.tree_build()
    got = pcm.write_ot()
    _, nodes, _ = O.read_ot(expect)
    assert nn == len(nodes)
    assert got == expect
    tk, td, tv, tc = pcm.tree_leaves()
    if len(nodes) == 0:
        assert nl == 0 and len(tk) == 0
        return got
    keys, depths, vals, cols, consistent, used = O.leaves_from_nodes(nodes)
    assert consistent and used == len(nodes) and nl == len(keys)
    assert (tk == keys).all() and (td == depths).all() and (tc == cols).all()
    assert (tv.view(np.uint32) == vals.view(np.uint32)).all()
    return got


def test_reference_tree_round_trip():
    """read(reference bytes) -> the map holds exactly the tree's depth-16 cells -> write == the oracle's file, which
    test_oracle_cpu pins to the reference's octomap.ot (node count, order, values, child masks, leaf colours)."""
    data, nodes = reference_bytes()
    keys, depths, vals, cols, _, _ = O.leaves_from_nodes(nodes)
    k16, v16, c16 = O.expand_to_max_depth(keys, depths, vals, cols)
    assert len(k16) == 391387
    pcm = _pcm()
    pcm.read_ot(data)
    assert pcm.num_leaves() == len(k16)
    assert (_sorted_cells(*pcm.export_leaves()) == _sorted_cells(k16, v16, c16)).all()
    nn, nl = pcm.tree_build()
    assert (nn, nl) == (390133, 318930)
    out = pcm.write_ot()
    assert out == O.build_ot(k16, v16, c16, 0.05, "0.05")
    _, n2, hdr = O.read_ot(out)
    leaf = nodes["child"] == 0
    assert hdr == data[:len(hdr)].decode() and (n2["v"].view(np.uint32) == nodes["v"].view(np.uint32)).all()
    assert (n2["child"] == nodes["child"]).all() and (n2["rgb"][leaf] == nodes["rgb"][leaf]).all()
    tk, td, tv, tc = pcm.tree_leaves()
    assert (tk == keys).all() and (td == depths).all() and (tv == vals).all() and (tc == cols).all()


@pytest.mark.parametrize("make", S.SCENES, ids=lambda f: f.__name__)
def test_device_tree_equals_numpy_on_crafted_scenes(make):
    s = make()
    pcm = _pcm(s.res(), map_capacity=s.capacity, **{k: v for k, v in s.params.items() if k != "resolution"})
    pcm.insertKeyFrame(s.T, s.depth, s.rgb, *s.cam, s.label)
    assert_tree_equals_oracle(pcm, s.res())


def _room(n):
    """Keyframes of a wall with relief seen from a moving camera; the lower image part is ground: free-space rays."""
    ws = synth.WallStream(seed=7, n=n, depth0=2.0)
    yy, xx = np.mgrid[0:480, 0:640]
    label = np.zeros((480, 640), np.uint8)
    label[300:, :] = 1
    out = []
    for t in range(n):
        _, depth, rgb, T = ws.frame(t * 7)
        depth = (depth + 0.3 * np.sin(xx / 90.0) * np.cos(yy / 70.0)).astype(np.float32)
        depth[100:200, 150:300] = 1.1
        out.append((T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, label))
    return out


def test_device_tree_equals_numpy_on_a_room_sequence_and_is_repeatable():
    room = _room(5)
    pcm = _pcm()
    for kf in room[:4]:
        pcm.insertKeyFrame(*kf)
    first = assert_tree_equals_oracle(pcm, 0.05)
    _, nodes, _ = O.read_ot(first)
    assert len(nodes) > 1000
    pcm.tree_build()
    assert pcm.write_ot() == first                            # same map, same bytes
    pcm.insertKeyFrame(*room[4])
    assert pcm.write_ot() == first                            # the tree is a snapshot until the next build
    second = assert_tree_equals_oracle(pcm, 0.05)
    assert second != first


def _file(cells, res=0.05):
    """[(key, value, colour)] -> the oracle's `.ot` bytes."""
    keys = np.array([c[0] for c in cells], np.uint16).reshape(-1, 3)
    vals = np.array([c[1] for c in cells], np.float32)
    cols = np.array([c[2] for c in cells], np.uint8).reshape(-1, 3)
    return O.build_ot(keys, vals, cols, res, "%g" % res)


def _block(x0, y0, z0, side, v=0.5, col=(10, 20, 30)):
    return [((x0 + x, y0 + y, z0 + z), v, col) for z in range(side) for y in range(side) for x in range(side)]


def _unpruned_file(cells, col):
    """A valid file the writer would never produce: every cell its own depth-16 leaf of colour `col`, nothing pruned."""
    distinct = [(c[0], c[1], (i, 0, 0)) for i, c in enumerate(cells)]
    data = _file(distinct)
    res, nodes, hdr = O.read_ot(data)
    nodes = nodes.copy()
    nodes["rgb"][nodes["child"] == 0] = col
    return hdr.encode() + nodes.tobytes()


def _crafted():
    """name -> (file, the cells it holds, depths of the pruned leaves the device must find)."""
    eight = _block(100, 200, 300, 2)
    col = eight[0][2]
    zeros = [(c[0], (0.0, -0.0)[i % 2], col) for i, c in enumerate(eight)] + [((0, 0, 0), 1.0, col)]
    blocks = [c for c in _block(64, 64, 64, 4) if min(c[0]) < 66] + _block(66, 66, 66, 2, v=0.75)
    cases = {"eight_equal": (eight, [15]),
             "one_colour_differs": (eight[:5] + [(eight[5][0], 0.5, (10, 20, 31))] + eight[6:], [16] * 8),
             "one_value_differs": (eight[:7] + [(eight[7][0], np.nextafter(np.float32(0.5), np.float32(1)), col)], [16] * 8),
             "seven_siblings": (eight[:3] + eight[4:], [16] * 7),
             "two_level_cascade": (_block(4096, 8, 65532, 4), [14]),
             "unaligned_block": (_block(101, 200, 300, 2), [16] * 8),
             "pruned_blocks_one_differs": (blocks, [15] * 8),
             "block_and_far_corner": (_block(0, 0, 0, 8, v=-2.0) + [((65535, 65535, 65535), 3.5, (0, 255, 0))], [13, 16]),
             "one_cell": ([((32768, 32768, 32768), 0.25, (7, 7, 7))], [16]),
             "no_cell": ([], [])}
    out = {k: (_file(cells), cells, depths) for k, (cells, depths) in cases.items()}
    out["plus_and_minus_zero"] = (_unpruned_file(zeros, col), zeros, [15, 16])     # +0.0 == -0.0: the block prunes
    out["unpruned_file_of_equal_cells"] = (_unpruned_file(_block(8, 8, 8, 4), col), _block(8, 8, 8, 4), [14])
    return out


@pytest.mark.parametrize("name", sorted(_crafted()))
def test_crafted_pruning(name):
    data, cells, leaf_depths = _crafted()[name]
    assert len({c[0] for c in cells}) == len(cells)
    pcm = _pcm(map_capacity=1 << 12)
    pcm.read_ot(data)
    assert pcm.num_leaves() == len(cells)
    if cells:
        want = _sorted_cells(np.array([c[0] for c in cells], np.uint16), np.array([c[1] for c in cells], np.float32),
                             np.array([c[2] for c in cells], np.uint8))
        assert (_sorted_cells(*pcm.export_leaves()) == want).all()
    out = assert_tree_equals_oracle(pcm, 0.05)
    assert sorted(pcm.tree_leaves()[1].tolist()) == sorted(leaf_depths)
    if not name.startswith(("plus_and", "unpruned")):
        assert out == data                     # the writer's own files come back byte for byte


@pytest.mark.parametrize("merge", [False, True], ids=["inserts", "merge_epochs"])
def test_resume_equals_the_uninterrupted_map(tmp_path, merge):
    room = _room(5)
    k = 3
    a = _pcm()
    for kf in room[:k]:
        a.insertKeyFrame(*kf)
    if merge:
        a.merge()
    path = str(tmp_path / "saved.ot")
    cells, nodes = a.SaveOctoMap(path)
    assert cells == a.num_leaves() and nodes == len(O.read_ot(path)[1])
    b = _pcm()
    b.insertKeyFrame(*room[4])               # loading replaces whatever the map held
    b.LoadOctoMap(path)
    assert (_sorted_cells(*a.export_leaves()) == _sorted_cells(*b.export_leaves())).all()
    for pcm in (a, b):
        for kf in room[k:]:
            pcm.insertKeyFrame(*kf)
        if merge:
            st = pcm.merge()
            assert st.records_sent > 0
    ca, cb = _sorted_cells(*a.export_leaves()), _sorted_cells(*b.export_leaves())
    assert len(ca) > cells and ca.shape == cb.shape and (ca == cb).all()
    fa, fb = str(tmp_path / "a.ot"), str(tmp_path / "b.ot")
    a.SaveOctoMap(fa)
    b.SaveOctoMap(fb)
    assert open(fa, "rb").read() == open(fb, "rb").read()


def test_refusals_keep_the_map():
    from orb_slam2_ssd_semantic_b200 import B200OrbError, _lib
    s = S.rays_many()
    pcm = _pcm(S.RES, map_capacity=1 << 16)
    pcm.insertKeyFrame(s.T, s.depth, s.rgb, *s.cam, s.label)
    before = _sorted_cells(*pcm.export_leaves())
    assert 8 < len(before) < 1 << 16
    good = _file(_block(0, 0, 0, 2), S.RES)
    chain = np.zeros(11, O.NODE_DT)          # one leaf of depth 10: 64^3 cells, four times the map's capacity
    chain["child"][:10] = 1
    too_many = (O.HEADER % (11, "%g" % S.RES)).encode() + chain.tobytes()
    for data, code, word in ((_file(_block(0, 0, 0, 2), 0.05), EINVAL, "res"), (good[:-8], EINVAL, "size"),
                             (too_many, ECAP, "map_capacity"),
                             (good.replace(b"ColorOcTree", b"OcTree"), EINVAL, "ColorOcTree"), (b"", EINVAL, "first line")):
        with pytest.raises(B200OrbError) as e:
            pcm.read_ot(data)
        assert e.value.code == code and word in str(e.value)
        assert (_sorted_cells(*pcm.export_leaves()) == before).all()
    with pytest.raises(B200OrbError) as e:
        pcm.LoadOctoMap("/nonexistent/octomap.ot")
    assert e.value.code == EINVAL
    pcm.insertKeyFrame(s.T, s.depth, s.rgb, *s.cam, s.label)          # the map goes on
    after = _sorted_cells(*pcm.export_leaves())
    assert (after[:, 0] == before[:, 0]).all() and (after[:, 1] != before[:, 1]).any()
    # a buffer one byte short: B200ORB_ECAP and the size; nothing written
    L = _lib.lib()
    fresh = _pcm(S.RES, map_capacity=1 << 12)
    full = np.zeros(13, O.NODE_DT)           # one leaf of depth 12: 16^3 cells fill the 4096 slots exactly
    full["child"][:12] = 1
    fresh.read_ot((O.HEADER % (13, "%g" % S.RES)).encode() + full.tobytes())
    assert fresh.num_leaves() == 1 << 12 and fresh.tree_build() == (13, 1)
    fresh = _pcm(S.RES, map_capacity=1 << 12)
    n = C.c_int64(0)
    assert L.ocm_write_ot(fresh.handle, None, 0, C.byref(n)) == EINVAL      # no tree built yet
    pcm.tree_build()
    data = pcm.write_ot()
    buf = np.full(len(data), 0xEE, np.uint8)
    assert L.ocm_write_ot(pcm.handle, buf.ctypes.data_as(C.c_void_p), len(data) - 1, C.byref(n)) == ECAP
    assert n.value == len(data) and (buf == 0xEE).all()
    assert L.ocm_tree_leaves(pcm.handle, buf.ctypes.data_as(C.c_void_p), None, None, None, 1, C.byref(n)) == ECAP
    assert n.value == pcm.tree_build()[1] and (buf == 0xEE).all()
    pcm.read_ot(good)                                                    # and a good file still loads
    assert pcm.num_leaves() == 8 and pcm.last_points()[0].shape == (0, 3)


def test_ot_shim_program_saves_loads_and_resumes(tmp_path):
    shim = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200", "csrc", "shim")
    libdir = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200")
    exe = str(tmp_path / "shim_ot_check")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(shim, "shim_ot_check.cpp"),
                           "-I" + os.path.join(ROOT, "oracle", "standin"), "-I" + os.path.join(ROOT, "include"), "-L" + libdir,
                           "-lb200orb", "-Wl,-rpath," + libdir])
    files = [str(tmp_path / n) for n in ("first.ot", "kept.ot", "resumed.ot")]
    out = subprocess.run([exe] + files, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "resumed to" in out.stdout and "other resolution refused" in out.stdout
    first, kept, resumed = (open(f, "rb").read() for f in files)
    assert kept == resumed and kept != first
    for data in (first, kept):
        res, nodes, hdr = O.read_ot(data)
        keys, depths, vals, cols, consistent, used = O.leaves_from_nodes(nodes)
        assert res == 0.05 and "id ColorOcTree" in hdr and consistent and used == len(nodes) > 1000
        k16, v16, c16 = O.expand_to_max_depth(keys, depths, vals, cols)
        assert O.build_ot(k16, v16, c16, 0.05, "0.05") == data
