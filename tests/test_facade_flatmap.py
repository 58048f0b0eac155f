"""FlatMap_GPU in the builder API (include/wf/windflow_gpu.hpp): the WordCount-shaped application tests/cpp/test_facade_flatmap.cu
(Source of sentences -> FlatMap_GPU, one record per word -> keyed count-based Ffat_Windows_GPU -> Sink) writes its sentences and the
windows of three runs; this test expands the sentences with a numpy model and compares the windows with the oracle's count-based
windows (oracle/oracle.py) over the expanded stream:
  A  no prefix, position-weighted words: the oracle's windows exactly (the weights make every window depend on arrival order)
  F  Map -> Filter fused into the FlatMap's pass: the oracle's windows over the model's prefix, exactly
  B  the same Map -> Filter at another parallelism (not fused): the same multiset of windows as F
CPU: the application compiles for sm_90a. GPU: it runs and its windows match."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_facade_flatmap.cu")
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_flatmap.bin")

N, BATCH, MAXW, WIN, SLIDE, NWB = 40000, 1000, 6, 8, 4, 2
SENTENCE = np.dtype([("seq", "<u8"), ("nwords", "<u8"), ("words", "<u8", (MAXW,))])
WRES = np.dtype([("key", "<u8"), ("id", "<u8"), ("isum", "<i8"), ("fsum", "<f8")])


def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(ROOT, "include", "wf", "windflow_gpu.hpp"), os.path.join(ROOT, "windflow_b200", "csrc", "wfb_kernels.cuh"),
            os.path.join(ROOT, "windflow_b200", "csrc", "wfb_launch.cuh"), SRC]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(h) for h in hdrs):
        return
    libdir = os.path.join(ROOT, "windflow_b200")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr",
                           "--expt-extended-lambda", "-I" + os.path.join(ROOT, "include"), "-o", EXE, SRC, "-L" + libdir, "-lwfb200",
                           "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"])


def expand(s, prefix, weight):
    """The words of the sentences in stream order, per source batch: [(keys, isum)]; prefix: Map (drop the last word of every fifth
    sentence) -> Filter (drop every sentence with seq % 7 == 3)."""
    out = []
    for b in range(0, len(s), BATCH):
        x = s[b:b + BATCH].copy()
        if prefix:
            cut = (x["seq"] % np.uint64(5) == 0) & (x["nwords"] > 0)
            x["nwords"][cut] -= np.uint64(1)
            x = x[x["seq"] % np.uint64(7) != 3]
        c = x["nwords"].astype(np.int64)
        idx = np.repeat(np.arange(len(x)), c)
        j = np.arange(int(c.sum())) - np.repeat(np.cumsum(c) - c, c)
        keys = x["words"][idx, j]
        with np.errstate(over="ignore"):
            isum = (x["seq"][idx] * np.uint64(8) + j.astype(np.uint64)) if weight == "pos" else keys * np.uint64(3) + np.uint64(1)
        out.append((keys, isum.astype(np.int64), int(s["seq"][b])))
    return out


def oracle_windows(O, batches):
    go = O.FfatGpuOracle(WIN, SLIDE, NWB)
    res = []
    for keys, isum, wm in batches:
        r = np.zeros(len(keys), dtype=O.RES)
        r["key"], r["isum"] = keys, isum
        res.append(go.process_batch(r, wm)[0])
    return O.sort_results(np.concatenate(res))


def canon(r):
    r = r[np.lexsort((r["isum"], r["id"], r["key"]))]
    return np.stack([r["key"], r["id"], r["isum"].astype(np.uint64), r["fsum"].view(np.uint64)], axis=1)


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
def test_facade_flatmap_compiles():
    _compile()
    assert os.path.exists(EXE)


@pytest.mark.gpu
def test_facade_flatmap_wordcount_windows(oracle, tmp_path):
    _compile()
    out = subprocess.run([EXE, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "FLATMAP_OK" in out.stdout, out.stdout[-3000:]
    s = np.fromfile(tmp_path / "sentences.bin", dtype=SENTENCE)
    assert len(s) == N
    runs = {name: np.fromfile(tmp_path / f"{name}.bin", dtype=WRES) for name in ("A", "F", "B")}
    for name, prefix, weight in (("A", False, "pos"), ("F", True, "word")):
        exp = oracle_windows(oracle, expand(s, prefix, weight))
        got = oracle.sort_results(runs[name])
        assert len(got) == len(exp) > 0, (name, len(got), len(exp))
        for fld in ("key", "id", "isum"):
            assert np.array_equal(got[fld], exp[fld]), (name, fld)
        assert np.array_equal(got["fsum"], exp["fsum"]), name
    assert np.array_equal(canon(runs["B"]), canon(runs["F"]))
