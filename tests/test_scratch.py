"""windflow_b200/csrc/wfb_scratch.h -- the grow-on-demand scratch buffers of libwfb200 -- on the CPU: no call within the capacity, the
waits before the free, the growth policy, the zero fill, a failed allocation that leaves the buffer null and reusable, and every
allocation freed exactly once (tests/cpp/test_scratch.cpp, over stubs of the CUDA runtime calls; no libcudart, no GPU)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
@pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime_api.h")), reason="cuda_runtime_api.h not available")
def test_scratch_unit(tmp_path):
    exe = str(tmp_path / "test_scratch")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + CUDA_INC, "-I" + os.path.join(ROOT, "windflow_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "test_scratch.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "scratch OK" in out.stdout, out.stdout + out.stderr
