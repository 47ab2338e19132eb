"""CPU suite: the `.ot` parser of the library (ocm_ot_leaves: host only, no handle, no GPU) against octree_io, on the
reference's own tree and on malformed files; the octree entries are declared, exported and bound."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import octree_io as O
from orb_slam2_ssd_semantic_b200._abi import ptr

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ["ocm_tree_build", "ocm_write_ot", "ocm_tree_leaves", "ocm_save_ot", "ocm_read_ot", "ocm_load_ot", "ocm_ot_leaves"]
EINVAL, ECAP = -1, -2


def reference_bytes():
    z = np.load(os.path.join(G, "octomap_nodes.npz"))
    nodes = np.zeros(len(z["v"]), O.NODE_DT)
    nodes["v"], nodes["rgb"], nodes["child"] = z["v"], z["rgb"], z["child"]
    return str(z["header"]).encode() + nodes.tobytes(), nodes


def ot_leaves(data: bytes, cap=None):
    """ocm_ot_leaves -> (rc, res, n, keys, depth, logodds, rgb); the arrays keep a sentinel where nothing was written."""
    from orb_slam2_ssd_semantic_b200 import _lib
    L = _lib.lib()
    buf = np.frombuffer(data, np.uint8)
    n, res = C.c_int64(-7), C.c_double(-7.0)
    if cap is None:
        rc = L.ocm_ot_leaves(ptr(buf) if len(buf) else None, len(buf), C.byref(res), None, None, None, None, 0, C.byref(n))
        if rc != 0:
            return rc, res.value, n.value, None, None, None, None
        cap = n.value
    keys, depth = np.full((max(cap, 1), 3), 0xABCD, np.uint16), np.full(max(cap, 1), 0xEE, np.uint8)
    lo, rgb = np.full(max(cap, 1), -123.0, np.float32), np.full((max(cap, 1), 3), 0xEE, np.uint8)
    rc = L.ocm_ot_leaves(ptr(buf) if len(buf) else None, len(buf), C.byref(res), ptr(keys), ptr(depth), ptr(lo), ptr(rgb), cap,
                         C.byref(n))
    return rc, res.value, n.value, keys, depth, lo, rgb


def last_error():
    from orb_slam2_ssd_semantic_b200 import _lib
    return _lib.lib().b200orb_last_error().decode()


def test_parser_equals_octree_io_on_the_reference_tree():
    data, nodes = reference_bytes()
    keys, depths, vals, cols, consistent, used = O.leaves_from_nodes(nodes)
    rc, res, n, k, d, v, c = ot_leaves(data)
    assert rc == 0 and res == 0.05 and n == len(keys) == 318930
    assert np.bincount(d[:n], minlength=17)[13:].tolist() == [4, 187, 8376, 310363]
    assert (k[:n] == keys).all() and (d[:n] == depths).all() and (c[:n] == cols).all()
    assert (v[:n].view(np.uint32) == vals.view(np.uint32)).all()


def small_file():
    """Two levels of crafted tree through the oracle's writer: 8 equal cells (one pruned leaf of depth 15) and two loose
    cells."""
    keys = [(32768 + x, 32768 + y, 32768 + z) for z in (0, 1) for y in (0, 1) for x in (0, 1)] + [(10, 20, 30), (65535, 0, 7)]
    v = np.array([0.5] * 8 + [-1.25, 2.0], np.float32)
    rgb = np.array([[1, 2, 3]] * 8 + [[9, 8, 7], [255, 0, 128]], np.uint8)
    return O.build_ot(np.array(keys, np.uint16), v, rgb, 0.05, "0.05")


def test_parser_on_a_small_tree_and_capacity():
    data = small_file()
    _, nodes, _ = O.read_ot(data)
    keys, depths, vals, cols, _, _ = O.leaves_from_nodes(nodes)
    assert sorted(depths.tolist()) == [15, 16, 16]
    rc, res, n, k, d, v, c = ot_leaves(data)
    assert rc == 0 and n == 3 and res == 0.05
    assert (k[:3] == keys).all() and (d[:3] == depths).all() and (v[:3] == vals).all() and (c[:3] == cols).all()
    rc, _, n, k, d, v, c = ot_leaves(data, cap=2)
    assert rc == ECAP and n == 3 and "3 leaves" in last_error()
    assert (k == 0xABCD).all() and (d == 0xEE).all() and (v == -123.0).all() and (c == 0xEE).all()
    empty = (O.HEADER % (0, "0.05")).encode()
    rc, res, n, *_ = ot_leaves(empty)
    assert rc == 0 and n == 0 and res == 0.05


def _with_size(data: bytes, size: int) -> bytes:
    i = data.index(b"data\n") + 5
    return (O.HEADER % (size, "0.05")).encode() + data[i:]


MALFORMED = {
    "zero_bytes": lambda d: b"",
    "truncated_body": lambda d: d[:-8],
    "truncated_mid_node": lambda d: d[:-3],
    "trailing_bytes": lambda d: d + b"\0" * 8,
    "size_too_large": lambda d: _with_size(d, len(O.read_ot(d)[1]) + 1),
    "size_too_small": lambda d: _with_size(d, len(O.read_ot(d)[1]) - 1),
    "trailing_nodes": lambda d: _with_size(d + d[-8:], len(O.read_ot(d)[1]) + 1),
    "mask_past_the_end": lambda d: d[:-1] + b"\x01",
    "wrong_id": lambda d: d.replace(b"id ColorOcTree", b"id OcTree"),
    "missing_data_line": lambda d: d.replace(b"data\n", b"\n", 1),
    "first_line": lambda d: b"# Some other file\n" + d,
    "bad_res": lambda d: d.replace(b"res 0.05", b"res -1"),
    "bad_size": lambda d: d.replace(b"size ", b"size x"),
    "no_header_at_all": lambda d: d[d.index(b"data\n") + 5:],
}


@pytest.mark.parametrize("case", sorted(MALFORMED))
def test_malformed_files_are_refused_and_nothing_is_written(case):
    good = small_file()
    assert ot_leaves(good)[0] == 0
    bad = MALFORMED[case](good)
    assert bad != good
    rc, res, n, *_ = ot_leaves(bad)
    assert rc == EINVAL and res == -7.0 and n == -7 and last_error()
    rc, res, n, k, d, v, c = ot_leaves(bad, cap=16)
    assert rc == EINVAL and res == -7.0 and n == -7
    assert (k == 0xABCD).all() and (d == 0xEE).all() and (v == -123.0).all() and (c == 0xEE).all()


def test_tree_deeper_than_16_is_refused():
    """17 inner nodes in a chain: the node of depth 16 has a child."""
    nodes = np.zeros(18, O.NODE_DT)
    nodes["child"][:17] = 1
    rc, *_ = ot_leaves((O.HEADER % (18, "0.05")).encode() + nodes.tobytes())
    assert rc == EINVAL and "deeper than 16" in last_error()
    nodes = np.zeros(17, O.NODE_DT)      # 16 inner nodes and the cell of key (0, 0, 0)
    nodes["child"][:16] = 1
    rc, _, n, k, d, _, _ = ot_leaves((O.HEADER % (17, "0.05")).encode() + nodes.tobytes())
    assert rc == 0 and n == 1 and d[0] == 16 and (k[0] == 0).all()


def test_octree_entries_are_declared_exported_and_bound():
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping, _lib
    hdr = open(os.path.join(ROOT, "include", "b200orb.h")).read()
    L = _lib.lib()
    syms = subprocess.run(["nm", "-D", "--defined-only", _lib.library_path()], capture_output=True, text=True, check=True).stdout
    for name in ENTRIES:
        assert "int %s(" % name in hdr and name in _lib.EXPORTS and (" T %s\n" % name) in syms
        assert getattr(L, name).argtypes is not None
    for member in ("SaveOctoMap", "LoadOctoMap", "read_ot", "tree_build", "write_ot", "tree_leaves"):
        assert callable(getattr(PointCloudMapping, member))
    shim = open(os.path.join(ROOT, "orb_slam2_ssd_semantic_b200", "csrc", "shim", "pointcloudmapping.h")).read()
    assert "void SaveOctoMap(const char* filename)" in shim and "void LoadOctoMap()" in shim


def test_ot_shim_program_compiles_and_links(tmp_path):
    shim = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200", "csrc", "shim")
    libdir = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-o", str(tmp_path / "shim_ot_check"),
                           os.path.join(shim, "shim_ot_check.cpp"), "-I" + os.path.join(ROOT, "oracle", "standin"),
                           "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lb200orb", "-Wl,-rpath," + libdir])
