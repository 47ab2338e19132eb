"""GPU: the C++ class-surface shims (ORBextractor / ORBmatcher / PointCloudMapping) run end to end on the device."""
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _shim_check(tmp_path):
    shim = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200", "csrc", "shim")
    libdir = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200")
    exe = str(tmp_path / "shim_check")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(shim, "shim_check.cpp"),
                           "-I" + os.path.join(ROOT, "oracle", "standin"), "-I" + os.path.join(ROOT, "include"), "-L" + libdir,
                           "-lb200orb", "-Wl,-rpath," + libdir])
    return exe


def test_cpp_shims_run(tmp_path):
    exe = _shim_check(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "keypoints" in out.stdout and "UpdateOctomap lag" in out.stdout and "leaves" in out.stdout


@pytest.mark.parametrize("rows,cols,nfeatures,nlevels", [(100, 4000, 10, 1), (200, 3000, 30, 4)])
def test_shim_extractor_fresh_on_wide_image(oracle, tmp_path, rows, cols, nfeatures, nlevels):
    """operator() of a fresh shim ORBextractor sizes its output for the image: levels with nIni > 4 return up to 4*nIni
    keypoints on the first frame, bit-exact with the oracle."""
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    from tests.test_quadtree_cases_cpu import wide_image
    exe = _shim_check(tmp_path)
    img = wide_image(rows, cols)
    img.tofile(tmp_path / "img.u8")
    out = subprocess.run([exe, "extract", str(nfeatures), str(nlevels), str(rows), str(cols), str(tmp_path / "img.u8"),
                          str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    raw = (tmp_path / "out.bin").read_bytes()
    n = int(np.frombuffer(raw[:4], np.int32)[0])
    K = np.frombuffer(raw[4:4 + 28 * n], KP_DTYPE)
    D = np.frombuffer(raw[4 + 28 * n:], np.uint8).reshape(n, 32)
    K2, D2 = oracle.RefExtractor(nfeatures, 1.2, nlevels, 20, 7)(img)
    assert n > nfeatures + 3 * nlevels + 64
    assert K.tobytes() == K2.tobytes() and np.array_equal(D, D2)
