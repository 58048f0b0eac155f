"""Operators over more than 65 536 keys in the builder API (include/wf/windflow_gpu.hpp). CPU: the test program
tests/cpp/test_facade_many_keys.cu compiles with nvcc for sm_90a. GPU: its graph -- keyed-stateful Map_GPU withMaxKeys(1 << 18), then
time-based windows withKeyGrowth() from 16 keys, over 200 000 keys -- gives the windows the host computes."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_facade_many_keys.cu")
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_many_keys.bin")
NVCC = ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "--expt-extended-lambda",
        "-I" + os.path.join(ROOT, "include")]
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")


def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(ROOT, "include", "wf", "windflow_gpu.hpp"), os.path.join(ROOT, "include", "wfb200.h")] + \
        [os.path.join(ROOT, "windflow_b200", "csrc", h) for h in ("wfb_kernels.cuh", "wfb_keys.cuh", "wfb_launch.cuh")] + [SRC]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(h) for h in hdrs):
        return
    subprocess.check_call(NVCC + ["-o", EXE, SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200",
                                  "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"])


@needs_nvcc
def test_facade_many_keys_compiles():
    _compile()
    assert os.path.exists(EXE)


@pytest.mark.gpu
def test_facade_many_keys_runs():
    _compile()
    out = subprocess.run([EXE], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "MANY_KEYS_OK" in out.stdout, out.stdout[-3000:]
