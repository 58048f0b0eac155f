"""A builder-API application over a 256-byte tuple (tests/cpp/test_facade_big_tuple.cu): Map -> Filter -> count-based windows and a
keyed-stateful Map. The builder API registers programs whose result_t is the tuple itself, and the window kernels are instantiated for
every registered program, so the application only compiles when the window update and the tile pass accept 256-byte records.

CPU: the application compiles for sm_90a and the numpy model of its windows equals a plain fold. GPU: every window record and every
row of the stateful run equals the numpy model; the window set and ids come from the oracle."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import test_gpu_ordered_windows as ow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_facade_big_tuple.cu")
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_big_tuple.bin")
N, BATCH, NKEYS, WIN, SLIDE, NWB = 60000, 1000, 37, 24, 8, 2
MULT = ow.M
BIG = np.dtype([("key", "<u8"), ("seq", "<u8"), ("pad", "<u8", (30,))])
RES = np.dtype([("key", "<u8"), ("id", "<u8"), ("h", "<u8"), ("q", "<u8")])


def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(ROOT, "include", "wf", "windflow_gpu.hpp"), os.path.join(ROOT, "windflow_b200", "csrc", "wfb_kernels.cuh"),
            os.path.join(ROOT, "windflow_b200", "csrc", "wfb_launch.cuh"), SRC]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(h) for h in hdrs):
        return
    cmd = ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "--expt-extended-lambda",
           "-I" + os.path.join(ROOT, "include"), "-o", EXE, SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200",
           "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"]
    subprocess.check_call(cmd)


def mix64(x):
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(31)); x = x * np.uint64(0x7fb5d329728ea185)
        x = x ^ (x >> np.uint64(27)); x = x * np.uint64(0x81dadef4bc2dd44d)
        return x ^ (x >> np.uint64(33))


def ord_mix(a, k):
    with np.errstate(over="ignore"):
        x = ((a + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)) ^ (k * np.uint64(0xC2B2AE3D27D4EB4F))
        x ^= x >> np.uint64(29)
        return x | np.uint64(1)


def stream():
    i = np.arange(N, dtype=np.uint64)
    t = np.zeros(N, dtype=BIG)
    t["key"], t["seq"] = mix64(i) % np.uint64(NKEYS), i
    with np.errstate(over="ignore"):
        t["pad"] = mix64(i[:, None] * np.uint64(32) + np.arange(1, 31, dtype=np.uint64)[None, :])
    return t


def stir(t):
    t = t.copy()
    with np.errstate(over="ignore"):
        t["pad"] = (t["pad"] ^ (t["key"][:, None] * np.uint64(0xD6E8FEB86659FD93))) + \
            np.arange(1, 31, dtype=np.uint64)[None, :] * t["seq"][:, None]
    return t


def keep(t):
    return (t["seq"] % np.uint64(7) != np.uint64(3)) & ((t["pad"][:, 29] >> np.uint64(5)) % np.uint64(4) != np.uint64(0))


def expected_windows(O):
    u = stir(stream())
    s = u[keep(u)]
    go = O.FfatGpuOracle(WIN, SLIDE, NWB)
    e, _ = go.process_batch(ow._lift_res(np.rec.fromarrays([s["key"], s["seq"]], names="key,id")), 0)
    go.close()
    e = O.sort_results(e)
    order, a, b = ow.cb_ranges(s["key"], e["key"], e["id"], WIN, SLIDE)
    h = ord_mix(s["pad"][:, 29] ^ s["pad"][:, 0], s["key"])
    r = np.zeros(len(e), dtype=RES)
    r["key"], r["id"] = e["key"], e["id"]
    r["h"] = ow.hash_ranges(h[order], a, b, np.uint64)[0]
    r["q"] = b - a
    return r


def expected_stateful():
    u = stir(stream())
    m64 = (1 << 64) - 1
    st = {}
    x = ord_mix(u["pad"][:, 29], u["key"]).tolist()
    for i, k in enumerate(u["key"].tolist()):
        c, h = st.get(k, (0, 0))
        c, h = c + 1, (h * MULT + x[i]) & m64
        st[k] = (c, h)
        u["pad"][i, 0], u["pad"][i, 1] = h, c
    return u


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
def test_big_tuple_application_compiles():
    _compile()
    assert os.path.exists(EXE)


def test_window_model_equals_plain_fold(oracle):
    e = expected_windows(oracle)
    assert len(e) > 1000
    u = stir(stream())
    s = u[keep(u)]
    h = ord_mix(s["pad"][:, 29] ^ s["pad"][:, 0], s["key"])
    for r in e[::97]:
        items = h[s["key"] == r["key"]][int(r["id"]) * SLIDE:int(r["id"]) * SLIDE + WIN]
        acc = 0
        for v in items.tolist():
            acc = (acc * MULT + v) & ((1 << 64) - 1)
        assert acc == int(r["h"]) and len(items) == r["q"] == WIN


@pytest.mark.gpu
def test_big_tuple_application_matches_model(oracle, tmp_path):
    _compile()
    out = subprocess.run([EXE, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "BIG_TUPLE_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    got = np.fromfile(tmp_path / "cb.bin", dtype=RES)
    got = got[np.lexsort((got["id"], got["key"]))]
    exp = expected_windows(oracle)
    assert len(got) == len(exp)
    assert got.tobytes() == exp.tobytes()
    rows = np.fromfile(tmp_path / "stateful.bin", dtype=BIG)
    assert rows.tobytes() == expected_stateful().tobytes()
