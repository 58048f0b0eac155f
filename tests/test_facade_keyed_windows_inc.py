"""The incremental Keyed_Windows_GPU in the builder API (include/wf/windflow_gpu.hpp): the application
tests/cpp/test_facade_keyed_windows_inc.cu (Source -> Map_GPU -> Filter_GPU -> Keyed_WindowsGPU_Builder(void(const tuple_t &, result_t &))
-> Sink) writes the source's tuples and the results of three runs in Sink order; this test folds the tuples with the incremental model of
tests/test_gpu_keyed_windows_inc.py and compares:
  K128  K = 128 batches per call, K1  one batch per call, NK  no withKeyBy (one key, results start as result_t(gwid))
Every run's results equal the model's, end-of-stream windows included, and each key's window ids arrive as 0, 1, 2, ... in Sink order.
CPU: the application compiles for sm_90a, and a functor matching neither signature stops the compilation with the builder's message.
GPU: it runs and its windows match."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_gpu_keyed_windows import TUPLE64
from test_gpu_keyed_windows_inc import RES, IncModel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_facade_keyed_windows_inc.cu")
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_keyed_windows_inc.bin")
WIN, SLIDE = 12, 5
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")


def nvcc(src, exe):
    libdir = os.path.join(ROOT, "windflow_b200")
    return ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "--expt-extended-lambda",
            "-diag-suppress", "186", "-I" + os.path.join(ROOT, "include"), "-o", exe, src, "-L" + libdir, "-lwfb200",
            "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"]


def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(ROOT, "include", "wf", "windflow_gpu.hpp"), os.path.join(ROOT, "windflow_b200", "csrc", "wfb_kernels.cuh"),
            os.path.join(ROOT, "windflow_b200", "csrc", "wfb_launch.cuh"), SRC]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(h) for h in hdrs):
        return
    subprocess.check_call(nvcc(SRC, EXE))


def expected(src, keyed):
    """The model's windows (fired, then end of stream) over the tuples that pass the Map and the Filter."""
    t = src.copy()
    t["ivalue"] += 2
    t = t[(t["ivalue"] & 3) != 0]
    if not keyed:
        t["key"] = 0
    m = IncModel(0, WIN, SLIDE)
    rows = m.feed(t, np.arange(len(t), dtype=np.uint64)) + m.flush()
    return sorted(r[:-1] for r in rows)  # (the Sink sees no timestamps)


@needs_nvcc
def test_facade_keyed_windows_inc_compiles():
    _compile()
    assert os.path.exists(EXE)


@needs_nvcc
def test_builder_refuses_other_signatures(tmp_path):
    """A functor that takes the tuple by non-const reference matches neither signature: the builder's static_assert names both."""
    src = tmp_path / "bad.cu"
    src.write_text("#include <wf/windflow_gpu.hpp>\n"
                   "struct T { uint64_t key, id; };\n"
                   "struct R { uint64_t key, id; __host__ __device__ R() : key(0), id(0) {} };\n"
                   "struct F { __host__ __device__ void operator()(T &t, R &r) const { r.id += t.id; } };\n"
                   "int main() { auto op = wf::Keyed_WindowsGPU_Builder(F()).withCBWindows(4, 2).build(); (void)op; return 0; }\n")
    p = subprocess.run(nvcc(str(src), str(tmp_path / "bad.bin")), capture_output=True, text=True)
    assert p.returncode != 0
    msg = p.stdout + p.stderr
    assert "unknown signature passed to the Keyed_WindowsGPU_Builder" in msg, msg[-3000:]
    assert "void(const tuple_t &, result_t &)" in msg and "void(const Iterable_GPU<tuple_t> &, result_t &)" in msg, msg[-3000:]


@pytest.mark.gpu
def test_facade_keyed_windows_inc(tmp_path):
    _compile()
    out = subprocess.run([EXE, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "KEYED_WINDOWS_INC_OK" in out.stdout, out.stdout[-3000:]
    src = np.fromfile(tmp_path / "tuples.bin", dtype=TUPLE64)
    assert len(src) == 40000
    for name, keyed in (("K128", True), ("K1", True), ("NK", False)):
        r = np.fromfile(tmp_path / f"{name}.bin", dtype=RES[0])
        nxt = {}
        for k, g in zip(r["key"].tolist(), r["id"].tolist()):  # each key's windows in order, none missing or repeated
            assert g == nxt.get(k, 0), (name, k, g)
            nxt[k] = g + 1
        got = sorted((int(x["key"]), int(x["id"]), int(x["hash"]), int(x["size"]), int(x["front"]), int(x["back"]), int(x["mask"]),
                      float(x["fsum"]), int(x["argmax"]), int(x["maxiv"])) for x in r)
        exp = expected(src, keyed)
        assert len(got) == len(exp) > 0, (name, len(got), len(exp))
        assert got == exp, name
        assert any(x[3] < WIN for x in got)  # the end-of-stream windows are there
