"""Keyed_Windows_GPU in the builder API (include/wf/windflow_gpu.hpp): the application tests/cpp/test_facade_keyed_windows.cu
(Source -> Map_GPU -> Filter_GPU [-> keyed-stateful Map_GPU] -> Keyed_Windows_GPU -> Sink) writes the source's tuples and the results
of three runs in Sink order; this test folds the tuples with the Python model of tests/test_gpu_keyed_windows.py and compares:
  K128  K = 128 batches per call, K1  one batch per call, KS  a keyed-stateful Map in front (ivalue += the key's running count)
Every run's results equal the model's, end-of-stream windows included, and each key's window ids arrive as 0, 1, 2, ... in Sink order.
CPU: the application compiles for sm_90a. GPU: it runs and its windows match."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_gpu_keyed_windows import TUPLE64, Model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_facade_keyed_windows.cu")
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_keyed_windows.bin")
WIN, SLIDE = 12, 5
RES = np.dtype([("key", "<u8"), ("id", "<u8"), ("hash", "<u8"), ("size", "<u8"), ("mid", "<u8"), ("front", "<u8"), ("back", "<u8"),
                ("distinct", "<u8"), ("fsum", "<f8")])


def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(ROOT, "include", "wf", "windflow_gpu.hpp"), os.path.join(ROOT, "windflow_b200", "csrc", "wfb_kernels.cuh"),
            os.path.join(ROOT, "windflow_b200", "csrc", "wfb_launch.cuh"), SRC]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(h) for h in hdrs):
        return
    libdir = os.path.join(ROOT, "windflow_b200")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
                           "--expt-extended-lambda", "-diag-suppress", "186", "-I" + os.path.join(ROOT, "include"), "-o", EXE, SRC,
                           "-L" + libdir, "-lwfb200", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"])


def expected(src, stateful):
    """The model's windows (fired, then end of stream) over the tuples that pass the Map and the Filter (and the keyed Map)."""
    t = src.copy()
    t["ivalue"] += 2
    t = t[(t["ivalue"] & 3) != 0]
    if stateful:
        cnt = {}
        for i in range(len(t)):
            k = int(t["key"][i])
            cnt[k] = cnt.get(k, 0) + 1
            t["ivalue"][i] += cnt[k]
    m = Model(0, WIN, SLIDE)
    rows = m.feed(t, np.arange(len(t), dtype=np.uint64)) + m.flush()
    return sorted(r[:-1] for r in rows)  # (the Sink sees no timestamps)


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
def test_facade_keyed_windows_compiles():
    _compile()
    assert os.path.exists(EXE)


@pytest.mark.gpu
def test_facade_keyed_windows(tmp_path):
    _compile()
    out = subprocess.run([EXE, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "KEYED_WINDOWS_OK" in out.stdout, out.stdout[-3000:]
    src = np.fromfile(tmp_path / "tuples.bin", dtype=TUPLE64)
    assert len(src) == 40000
    for name, stateful in (("K128", False), ("K1", False), ("KS", True)):
        r = np.fromfile(tmp_path / f"{name}.bin", dtype=RES)
        nxt = {}
        for k, g in zip(r["key"].tolist(), r["id"].tolist()):  # each key's windows in order, none missing or repeated
            assert g == nxt.get(k, 0), (name, k, g)
            nxt[k] = g + 1
        got = sorted((int(x["key"]), int(x["id"]), int(x["hash"]), int(x["size"]), int(x["mid"]), int(x["front"]), int(x["back"]),
                      int(x["distinct"]), float(x["fsum"])) for x in r)
        exp = expected(src, stateful)
        assert len(got) == len(exp) > 0, (name, len(got), len(exp))
        assert got == exp, name
        assert any(x[3] < WIN for x in got)  # the end-of-stream windows are there
