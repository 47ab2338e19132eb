"""The owners of the handles' CUDA resources (csrc/common.cuh) on a machine without a GPU: every allocation fails, and a
failed allocation must leave an empty block that is never sized beyond what exists and is allocated again next time."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "orb_slam2_ssd_semantic_b200", "csrc")

PROGRAM = r"""
#include <cstdarg>
#include "common.cuh"

static int n_errors = 0;
void b200::set_error(const char*, ...) { ++n_errors; }
using namespace b200;

// One line per call: the return code, whether a CUDA call failed in it, the block afterwards, the buffer pointers.
template <class B>
static void report(const char* what, B& b, cudaStream_t st, bool grow) {
  float* a = (float*)&n_errors;
  int* i = (int*)&n_errors;
  auto list = [&](Carver& t) { a = t.take<float>(1000); i = t.take<int>(10); };
  const int before = n_errors;
  const int rc = grow ? b.reserve(st, list) : b.carve(st, list);
  const bool cuda_failed = cudaGetLastError() != cudaSuccess;
  printf("%s rc=%d cuda_failed=%d errors=%d p=%d bytes=%zu bufs=%d\n", what, rc, (int)cuda_failed, n_errors - before,
         b.p != nullptr, b.bytes, a != nullptr || i != nullptr);
}

int main() {
  DeviceBlock d;
  HostBlock h;
  report("device_carve", d, nullptr, false);
  report("device_reserve", d, nullptr, true);
  report("device_reserve", d, nullptr, true);
  report("host_carve", h, nullptr, false);
  report("host_reserve", h, nullptr, true);
  report("host_reserve", h, nullptr, true);
  Stream s;
  Event e;
  const int rs = s.create(), re = e.create();
  printf("stream rc=%d null=%d\nevent rc=%d null=%d\n", rs, (cudaStream_t)s == nullptr, re, (cudaEvent_t)e == nullptr);
  return 0;
}
"""


def test_failed_allocation_leaves_an_empty_block(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    src = tmp_path / "handles.cu"
    src.write_text(PROGRAM)
    exe = str(tmp_path / "handles")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-I" + CSRC, "-o", exe,
                           str(src)])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    lines = [ln.split() for ln in out.stdout.splitlines()]
    ecuda = "rc=-3"
    blocks = [ln for ln in lines if ln[0].endswith(("_carve", "_reserve"))]
    assert [ln[0] for ln in blocks] == ["device_carve", "device_reserve", "device_reserve", "host_carve", "host_reserve",
                                        "host_reserve"]
    for name, rc, cuda_failed, errors, p, nbytes, bufs in blocks:
        # every call, a later reserve included, tries the allocation again and reports B200ORB_ECUDA
        assert rc == ecuda and cuda_failed == "cuda_failed=1" and errors == "errors=1", (name, rc, cuda_failed, errors)
        # the block stays empty, with no size, and the caller's buffer pointers are null
        assert p == "p=0" and nbytes == "bytes=0" and bufs == "bufs=0", (name, p, nbytes, bufs)
    assert lines[-2] == ["stream", ecuda, "null=1"] and lines[-1] == ["event", ecuda, "null=1"]
