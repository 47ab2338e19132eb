"""CPU suite: the C-ABI library loads, exports every symbol include/b200orb.h declares, and refuses to run without a
GPU (no silent CPU fallback).  No compute calls here."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    txt = open(os.path.join(ROOT, "include", "b200orb.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b((?:orbx|orbm|orbs|orbv|ocm|gcm|dynm|b200orb)_[a-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    import orb_slam2_ssd_semantic_b200 as pkg
    L = pkg.lib()
    names = _declared()
    assert len(names) > 40
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, "declared in include/b200orb.h but not exported: %s" % missing


def test_python_binding_lists_match_header():
    from orb_slam2_ssd_semantic_b200._lib import EXPORTS
    assert set(EXPORTS) <= set(_declared())


def test_struct_layouts_match_header():
    from orb_slam2_ssd_semantic_b200 import _abi
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    assert KP_DTYPE.itemsize == 28 and C.sizeof(_abi.OrbxParams) == 20
    assert C.sizeof(_abi.OrbmFrame) == 8 + 7 * 8 + 64 + 10 * 4 + 8 + 8     # n(+pad), 7 ptrs, Tcw, 10 floats, ptr, nlevels(+pad)
    assert C.sizeof(_abi.OrbmLast) == 8 + 6 * 8 + 64
    assert C.sizeof(_abi.OcmParams) == 5 * 8 + 4 * 4 + 8
    # 4 ints, 3 ptrs, depth_factor(+pad), 2 ptrs, device_flow(+pad), prev_gray, binary_threshold(+pad)
    assert C.sizeof(_abi.OrbsBatch) == 4 * 4 + 3 * 8 + 8 + 2 * 8 + 8 + 8 + 8
    assert C.sizeof(_abi.OrbsResults) == 5 * 8 + 8                             # 5 ptrs, cap(+pad)


def test_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import orb_slam2_ssd_semantic_b200 as pkg
    from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask
    for ctor in (pkg.ORBextractor, pkg.ORBmatcher, pkg.StreamTracker, pkg.PointCloudMapping, pkg.GlobalCloudMapping, DynamicMask):
        with pytest.raises(pkg.B200OrbError) as e:
            ctor()
        assert e.value.code == -4 and "no CPU fallback" in str(e.value)


def test_hamming_host_inline():
    import numpy as np
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    a = np.arange(32, dtype=np.uint8)
    b = np.zeros(32, np.uint8)
    assert ORBmatcher.DescriptorDistance(a, b) == int(np.unpackbits(a).sum())
    assert ORBmatcher.TH_HIGH == 100 and ORBmatcher.TH_LOW == 50 and ORBmatcher.HISTO_LENGTH == 30


def test_cpp_shims_compile_link_and_fail_loudly(tmp_path):
    """The header-only C++ shims (class surface of the reference) compile against the stand-in cv:: types, link the
    C-ABI library, and -- on this GPU-less box -- refuse to construct."""
    import subprocess
    import torch
    shim = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200", "csrc", "shim")
    libdir = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200")
    exe = str(tmp_path / "shim_check")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(shim, "shim_check.cpp"),
                           "-I" + os.path.join(ROOT, "oracle", "standin"), "-I" + os.path.join(ROOT, "include"),
                           "-L" + libdir, "-lb200orb", "-Wl,-rpath," + libdir])
    if torch.cuda.is_available():
        pytest.skip("GPU present: exercised by tests/test_shim_gpu.py")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "loud failure" in out.stdout and "no CPU fallback" in out.stdout


def test_shims_compile_against_the_reference_sources():
    """All three shim headers in their one and only (production) form: shim/ORBextractor.h + shim/ORBmatcher.h are what
    the reference's own src/Frame.cc, KeyFrame.cc, MapPoint.cc, Map.cc are compiled against for oracle/_ref/libshimsrc.so
    (oracle/Makefile, target `shim`); the library must link against libb200orb.so and export every shimsrc_* entry."""
    import subprocess
    if not os.path.exists("/root/reference/src/Frame.cc"):
        pytest.skip("the reference is not on this box")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "shim"])
    L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libshimsrc.so"))
    for name in ("projection_last", "projection_points", "projection_kf", "projection_sim3", "bow", "bow_kf", "initialization",
                 "triangulation", "search_by_sim3", "fuse", "fuse_sim3", "frame_rgbd", "pipeline_run", "orb_extract"):
        assert hasattr(L, "shimsrc_" + name), name


def test_flow_shim_syntax():
    """shim/Flow.h (drop-in for perfect/include/Flow.h) compiles against the stand-in cv:: types; the three OpenCV calls it
    leaves on the host are declared by oracle/standin/flow_decls.hpp."""
    import subprocess
    shim = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200", "csrc", "shim")
    subprocess.check_call(["g++", "-std=c++14", "-fsyntax-only", "-Wall", "-x", "c++", "-include",
                           os.path.join(ROOT, "oracle", "standin", "flow_decls.hpp"), os.path.join(shim, "Flow.h"),
                           "-I" + os.path.join(ROOT, "oracle", "standin"), "-I" + os.path.join(ROOT, "include")])


def test_tuning_reports_fixed_selection():
    """b200orb_get_tuning is a read-only report (no GPU) of the extractor kernels this build runs, the selection chosen on
    an H100 (csrc/orbx.cu); nothing can switch them at run time: the library exports no b200orb_* entry that
    include/b200orb.h does not declare."""
    import subprocess
    import orb_slam2_ssd_semantic_b200 as pkg
    L = pkg.lib()
    m, w, q = C.c_int(), C.c_int(), C.c_int()
    assert L.b200orb_get_tuning(C.byref(m), C.byref(w), C.byref(q)) == 0
    assert (m.value, w.value, q.value) == (3, 8, 4)
    assert L.b200orb_get_tuning(None, None, None) == 0
    syms = subprocess.run(["nm", "-D", "--defined-only", pkg._lib.library_path()], capture_output=True, text=True,
                          check=True).stdout
    exported = set(re.findall(r"\sT (b200orb_\w+)", syms))
    assert "b200orb_get_tuning" in exported and exported <= set(_declared()), exported - set(_declared())
