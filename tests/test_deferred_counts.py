"""include/wf/deferred_counts.hpp -- the blocks of pinned words that carry deferred batch sizes to the consumer -- on the CPU: a block is
handed out again only when no batch points into it, a producer ahead of its consumers gets fresh blocks (a slab per allocation) and never
a held one, a failed allocation is reported, everything is freed once (tests/cpp/test_deferred_counts.cpp, over stubs of the CUDA
allocation calls; no libcudart, no GPU)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
@pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime_api.h")), reason="cuda_runtime_api.h not available")
def test_deferred_counts_unit(tmp_path):
    exe = str(tmp_path / "test_deferred_counts")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + CUDA_INC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "test_deferred_counts.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "deferred counts OK" in out.stdout, out.stdout + out.stderr
