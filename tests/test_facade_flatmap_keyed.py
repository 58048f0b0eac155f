"""The keyed-stateful FlatMap_GPU in the builder API (include/wf/windflow_gpu.hpp): the sessionising application
tests/cpp/test_facade_flatmap_keyed.cu (Source of events -> FlatMap_GPU keyed by user, m = 2: the closed session's summary, then the
event -> keyed count-based Ffat_Windows_GPU -> Sink) writes its events and the windows of four runs; this test sessionises the events
with a numpy model, in each user's arrival order, and compares the windows with the oracle's count-based windows over the records:
  P1  parallelism 1, K = 128 batches per call: the oracle's windows exactly
  K1  one batch per call, and G  a key table that grows from 16 keys: the same windows exactly
  P2  parallelism 2 (every user's events reach one replica, in order): the same multiset of windows
CPU: the application compiles for sm_90a. GPU: it runs and its windows match."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_facade_flatmap_keyed.cu")
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_flatmap_keyed.bin")

N, BATCH, GAP, WIN, SLIDE, NWB = 60000, 500, 700, 8, 4, 2
EVENT = np.dtype([("user", "<u8"), ("seq", "<u8"), ("time", "<u8"), ("value", "<i8")])
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


def sessionise(ev):
    """The records of every source batch, in input order: [(keys, isum of the lift, watermark)]."""
    state = {}
    out = []
    for b in range(0, len(ev), BATCH):
        keys, isum = [], []
        for e in ev[b:b + BATCH]:
            u, t = int(e["user"]), int(e["time"])
            last, start, count, s = state.get(u, (0, 0, 0, 0))
            if count > 0 and t - last > GAP:
                keys.append(u)
                isum.append(start * 7 + count * 1000 + s)
                count, s = 0, 0
            if count == 0:
                start = t
            count += 1
            s += int(e["value"])
            state[u] = (t, start, count, s)
            keys.append(u)
            isum.append(int(e["seq"]) * 3 + count)
        out.append((np.array(keys, dtype=np.uint64), np.array(isum, dtype=np.int64), int(ev["seq"][b])))
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
def test_facade_flatmap_keyed_compiles():
    _compile()
    assert os.path.exists(EXE)


@pytest.mark.gpu
def test_facade_flatmap_keyed_sessions(oracle, tmp_path):
    _compile()
    out = subprocess.run([EXE, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "FLATMAP_KEYED_OK" in out.stdout, out.stdout[-3000:]
    ev = np.fromfile(tmp_path / "events.bin", dtype=EVENT)
    assert len(ev) == N
    batches = sessionise(ev)
    assert sum(len(k) for k, _, _ in batches) > N  # some sessions closed
    exp = oracle_windows(oracle, batches)
    runs = {name: np.fromfile(tmp_path / f"{name}.bin", dtype=WRES) for name in ("P1", "K1", "G", "P2")}
    for name in ("P1", "K1", "G"):
        got = oracle.sort_results(runs[name])
        assert len(got) == len(exp) > 0, (name, len(got), len(exp))
        for fld in ("key", "id", "isum", "fsum"):
            assert np.array_equal(got[fld], exp[fld]), (name, fld)
    assert np.array_equal(canon(runs["P2"]), canon(runs["P1"]))
