"""The un-keyed Reduce_GPU in the builder API (include/wf/windflow_gpu.hpp): tests/cpp/test_facade_reduce.cu runs Source -> Reduce_GPU
without a key -> Sink and compares the Sink's rows, one per source batch, with a direct fold of each batch on the host (an
order-sensitive hash, from a default-constructed tuple). CPU: the application compiles for sm_90a. GPU: it runs and prints REDUCE_OK."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_facade_reduce.cu")
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_reduce.bin")
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")


def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(ROOT, "include", "wf", h) for h in ("windflow_gpu.hpp", "deferred_counts.hpp")] + \
        [os.path.join(ROOT, "windflow_b200", "csrc", h) for h in ("wfb_kernels.cuh", "wfb_launch.cuh")] + [SRC]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(h) for h in hdrs):
        return
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
                           "--expt-extended-lambda", "-diag-suppress", "186", "-I" + os.path.join(ROOT, "include"), "-o", EXE, SRC,
                           "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"])


@needs_nvcc
def test_facade_reduce_compiles():
    _compile()
    assert os.path.exists(EXE)


@pytest.mark.gpu
def test_facade_unkeyed_reduce_rows_match_direct_fold():
    _compile()
    out = subprocess.run([EXE], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "REDUCE_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
