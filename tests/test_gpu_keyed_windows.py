"""Keyed_Windows_GPU (wfb_kwin_*) against a direct Python fold of the count-based semantics, every field exact.

Per key, tuples get ids 0, 1, 2, ... in arrival order; window g holds ids [g*slide, g*slide + win) and fires with the first tuple after it,
id g*slide + win, carrying that tuple's timestamp (the reference's rule: tests/test_keyed_windows_golden.py pins it against the reference's
own outputs). At end of stream every window that opened (its first tuple arrived) and has not fired is evaluated
on the tuples of it that arrived, with the largest timestamp seen. The programs of tests/cpp/kwin_programs.cu hash the window's tuples in
order through the iterators and read size(), the middle element, front(), back() and the distinct ivalue % 16: a window missing a tuple,
holding another key's or seeing them out of order changes the result.

CPU (-m "not gpu"): the programs compile for sm_90a and the model agrees with a brute-force enumeration of the windows. GPU: the rest."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "windflow_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "cpp", "kwin_programs.cu")
SO = os.path.join(ROOT, "tests", "cpp", "kwin_programs.so")
NVCC = ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "--expt-extended-lambda",
        "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-Xcompiler", "-fPIC", "-shared", "-diag-suppress", "186"]
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")

TUPLE64 = np.dtype([("key", "<u8"), ("id", "<u8"), ("ivalue", "<i8"), ("fvalue", "<f8"), ("pad", "<u8", (4,))])
KEY16 = np.dtype([("key", "<u8"), ("a", "<u4"), ("b", "<u4")])
FIELDS = [("id", "<u8"), ("hash", "<u8"), ("size", "<u8"), ("mid", "<u8"), ("front", "<u8"), ("back", "<u8"), ("distinct", "<u8"), ("fsum", "<f8")]
RES = {0: np.dtype([("key", "<u8")] + FIELDS), 1: np.dtype([("key", KEY16)] + FIELDS)}
MIX, MUL, M64 = 0x9E3779B97F4A7C15, 0x100000001B3, (1 << 64) - 1
SENTINEL = 0xAB


# ---------------------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------------------
def win_fields(w):
    """The window function of kwin_programs.cu over a list of (id, ivalue, fvalue) in arrival order."""
    h, s, seen = 0, 0.0, 0
    for (i, iv, fv) in w:
        h = (h * MUL + (((i * MIX) & M64) ^ (iv & M64))) & M64
        s += fv
        seen |= 1 << (iv & 15)
    return (h, len(w), w[len(w) // 2][0], w[0][0], w[-1][0], bin(seen).count("1"), s)


def key_of(prog, row):
    if prog == 0:
        return int(row["key"])
    p0 = int(row["pad"][0])
    return (int(row["key"]), p0 & 0xFFFFFFFF, p0 >> 32)


class Model:
    """Count-based keyed windows, tuple after tuple (wf/window_replica.hpp:228-352, DETERMINISTIC mode)."""

    def __init__(self, prog, win, slide):
        self.prog, self.win, self.slide = prog, win, slide
        self.arch, self.last_ts = {}, 0

    def feed(self, rows, ts, drop=()):
        out = []
        for row, t in zip(rows, ts):
            k = key_of(self.prog, row)
            self.last_ts = max(self.last_ts, int(t))
            if k in drop:
                continue
            lst = self.arch.setdefault(k, [])
            i = len(lst)  # the tuple's id: it fires window g when i == g * slide + win (wf/window_structure.hpp:69-80)
            if i >= self.win and (i - self.win) % self.slide == 0:
                g = (i - self.win) // self.slide
                out.append((k, g) + win_fields(lst[g * self.slide:i]) + (int(t),))
            lst.append((int(row["id"]), int(row["ivalue"]), float(row["fvalue"])))
        return out

    def flush(self):
        out = []
        for k, lst in self.arch.items():
            c = len(lst)
            for g in range((c - 1) // self.slide + 1):
                if g * self.slide + self.win >= c:  # not fired: its firing tuple (id g * slide + win) never came
                    out.append((k, g) + win_fields(lst[g * self.slide:g * self.slide + self.win]) + (self.last_ts,))
        return out


def brute_windows(n, win, slide):
    """(fired windows as (g, trigger id), open windows) of one key with n tuples, by enumeration."""
    fired, opened = [], []
    for g in range(n + 1):
        first = g * slide
        if first >= n:
            break
        if first + win < n:
            fired.append((g, first + win))
        else:
            opened.append(g)
    return fired, opened


# ---------------------------------------------------------------------------------------------------------------------------------
# the test programs
# ---------------------------------------------------------------------------------------------------------------------------------
def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(CSRC, h) for h in ("wfb_kernels.cuh", "wfb_keys.cuh", "wfb_launch.cuh", "wfb_programs.cuh", "wfb_ptx.cuh")] + \
        [os.path.join(ROOT, "include", "wfb200.h"), SRC]
    if os.path.exists(SO) and all(os.path.getmtime(SO) > os.path.getmtime(h) for h in hdrs):
        return
    subprocess.check_call(NVCC + ["-o", SO, SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200",
                                  "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"])


_kw = None


def kwlib():
    global _kw
    if _kw is None:
        _compile()
        from windflow_b200 import _lib
        _lib.lib()
        L = C.CDLL(SO)
        L.kw_register.argtypes = [C.c_int]
        L.kw_register.restype = C.c_int
        _kw = L
    return _kw


@pytest.fixture(scope="module")
def progs(wfb):
    L = kwlib()
    ids = {w: L.kw_register(w) for w in range(2)}
    assert all(i >= 6 for i in ids.values()), ids
    return ids


# ---------------------------------------------------------------------------------------------------------------------------------
# streams
# ---------------------------------------------------------------------------------------------------------------------------------
def make_stream(n, nkeys, seed, zipf=False, key_list=None):
    rng = np.random.default_rng(seed)
    t = np.zeros(n, TUPLE64)
    if key_list is not None:
        t["key"] = key_list
    elif zipf:
        w = 1.0 / np.arange(1, nkeys + 1) ** 1.1
        t["key"] = rng.choice(nkeys, size=n, p=w / w.sum()).astype(np.uint64) * np.uint64(7919) + np.uint64(3)
    else:
        t["key"] = rng.integers(0, nkeys, n).astype(np.uint64) * np.uint64(7919) + np.uint64(3)
    t["id"] = np.arange(n, dtype=np.uint64)
    t["ivalue"] = rng.integers(-1000, 1000, n)
    t["fvalue"] = rng.random(n)
    t["pad"][:, 0] = (t["key"] * np.uint64(0x9E3779B1)) ^ np.uint64(0x1234)  # the 16-byte key's halves follow the integer key
    ts = np.cumsum(rng.integers(0, 5, n)).astype(np.uint64) + np.uint64(10)
    return t, ts


def split(n, sizes):
    """Cut [0, n) into consecutive batches whose sizes cycle through `sizes` (0 = an empty batch)."""
    out, i, j = [], 0, 0
    while i < n:
        m = min(sizes[j % len(sizes)], n - i)
        out.append((i, i + m))
        i += m
        j += 1
    return out


def results(kw, prog, out, out_ts, n_out):
    import torch
    torch.cuda.synchronize()
    n = int(n_out.cpu()[0])
    r = out.cpu().numpy().view(RES[prog])[:n]
    ts = out_ts.cpu().numpy().view(np.uint64)[:n]
    rows = []
    for x, t in zip(r, ts):
        k = int(x["key"]) if prog == 0 else (int(x["key"]["key"]), int(x["key"]["a"]), int(x["key"]["b"]))
        rows.append((k, int(x["id"]), int(x["hash"]), int(x["size"]), int(x["mid"]), int(x["front"]), int(x["back"]), int(x["distinct"]),
                     float(x["fsum"]), int(t)))
    return rows


def check_key_order(rows):
    """Results of one key come out in window order (within a call's output)."""
    last = {}
    for r in rows:
        assert last.get(r[0], -1) < r[1], ("window order", r[0], last.get(r[0]), r[1])
        last[r[0]] = r[1]


def run(wfb, prog_id, prog, t, ts, win, slide, max_keys, sizes, K, streams=None, drop=(), flush=True, dense=False):
    """Feeds the stream K batches per call; returns (gpu rows, model rows, handle)."""
    import torch
    kw = wfb.KeyedWindowsGPU(prog_id, win, slide, max_keys, dense_keys=dense)
    model = Model(prog, win, slide)
    cuts = split(len(t), sizes)
    batches = [wfb.DeviceBatch.from_host(t[a:b], ts[a:b]) if b > a else
               wfb.DeviceBatch(torch.empty(0, dtype=torch.uint8, device="cuda"), None, 0) for (a, b) in cuts]
    got, exp = [], []
    for c in range(0, len(batches), K):
        s = streams[(c // K) % len(streams)] if streams else None
        grp = batches[c:c + K]
        out, out_ts, n_out = kw.process(grp, stream=s)
        if s is not None:
            s.synchronize()
        rows = results(kw, prog, out, out_ts, n_out)
        check_key_order(rows)
        got += rows
        a, b = cuts[c][0], cuts[min(c + K, len(cuts)) - 1][1]
        exp += model.feed(t[a:b], ts[a:b], drop)
    if flush:
        cap = max_keys * (-(-win // slide) + 1)
        out, out_ts, n_out = kw.flush(cap)
        rows = results(kw, prog, out, out_ts, n_out)
        check_key_order(rows)
        got += rows
        exp += model.flush()
    return sorted(got), sorted(exp), kw


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------------
@needs_nvcc
def test_programs_compile_for_sm90a(tmp_path):
    from windflow_b200 import build
    build.build()
    subprocess.check_call(NVCC + ["-o", str(tmp_path / "kw.so"), SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200"])


@pytest.mark.parametrize("win,slide", [(1, 1), (1, 3), (3, 5), (8, 8), (10, 3), (16, 4), (5, 1)])
def test_model_matches_enumeration(win, slide):
    rng = np.random.default_rng(win * 100 + slide)
    t, ts = make_stream(500, 3, 11)
    m = Model(0, win, slide)
    got = m.feed(t, ts) + m.flush()
    for k in set(int(x) for x in t["key"]):
        sel = np.nonzero(t["key"] == k)[0]
        fired, opened = brute_windows(len(sel), win, slide)
        mine = sorted((r[1], r[-1]) for r in got if r[0] == k)
        expect = sorted([(g, int(ts[sel[i]])) for g, i in fired] + [(g, m.last_ts) for g in opened])
        assert mine == expect
        for r in got:
            if r[0] == k:
                ids = [int(t["id"][sel[i]]) for i in range(r[1] * slide, min(r[1] * slide + win, len(sel)))]
                assert r[3] == len(ids) and r[5] == ids[0] and r[6] == ids[-1] and r[4] == ids[len(ids) // 2]
    del rng


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------
GEOMS = [(1, 1), (1, 3), (4, 1), (3, 5), (8, 8), (10, 10), (10, 3), (16, 4), (64, 16), (100, 7)]


@pytest.mark.gpu
@pytest.mark.parametrize("prog", [0, 1])
@pytest.mark.parametrize("win,slide", GEOMS)
def test_geometries(progs, wfb, prog, win, slide):
    t, ts = make_stream(4000, 7, win * 31 + slide)
    got, exp, kw = run(wfb, progs[prog], prog, t, ts, win, slide, 64, [300, 0, 17, 1, 555, 64], 3)
    assert got == exp
    assert kw.stats() == (7, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("win,slide", [(10, 3), (16, 16), (5, 9)])
def test_more_than_ring_per_call(progs, wfb, win, slide):
    """One key receives hundreds of tuples per call (more than its ring holds): windows straddle the ring and the staging buffer."""
    t, ts = make_stream(5000, 1, 5)
    got, exp, _ = run(wfb, progs[0], 0, t, ts, win, slide, 4, [500, 37, 900], 1)
    assert got == exp and len(got) > 0


@pytest.mark.gpu
def test_few_tuples_per_call_wrap_the_ring(progs, wfb):
    """Fewer than slide tuples of a key per call over enough calls to wrap its ring many times."""
    t, ts = make_stream(1500, 3, 9)
    got, exp, _ = run(wfb, progs[0], 0, t, ts, 20, 16, 8, [5, 3, 7], 1)
    assert got == exp and len(got) > 50


@pytest.mark.gpu
@pytest.mark.parametrize("prog", [0, 1])
def test_batches_per_call(progs, wfb, prog):
    """K = 1, 7 and 128 batches per call give the results of the same stream one batch per call."""
    t, ts = make_stream(20000, 300, 21, zipf=True)
    runs = {}
    for K in (1, 7, 128):
        got, exp, _ = run(wfb, progs[prog], prog, t, ts, 24, 5, 512, [97, 0, 130, 3], K)
        assert got == exp
        runs[K] = got
    assert runs[1] == runs[7] == runs[128]


@pytest.mark.gpu
@pytest.mark.parametrize("nkeys,max_keys,dense", [(1, 1, False), (300, 300, False), (65536, 65536, False), (70000, 70000, False),
                                                  (70000, 70000, True)])
def test_key_counts(progs, wfb, nkeys, max_keys, dense):
    n = max(6000, 6 * nkeys)
    keys = None
    if dense:
        keys = np.random.default_rng(3).integers(0, nkeys, n).astype(np.uint64)
    t, ts = make_stream(n, nkeys, 33, key_list=keys)
    got, exp, kw = run(wfb, progs[0], 0, t, ts, 3, 2, max_keys, [4096, 0, 1000], 2, dense=dense)
    assert got == exp and len(got) > 0
    assert kw.stats()[1] == 0


@pytest.mark.gpu
def test_one_key_too_many(progs, wfb):
    """Every key takes a slot in the first calls; a new key arriving later finds none: bit 0, its tuples dropped, the others exact."""
    t, ts = make_stream(3000, 16, 41)
    extra = np.uint64(999983)
    t["key"][2000::5] = extra
    t["pad"][2000::5, 0] = (extra * np.uint64(0x9E3779B1)) ^ np.uint64(0x1234)
    for prog in (0, 1):
        drop = {key_of(prog, t[2000])}
        got, exp, kw = run(wfb, progs[prog], prog, t, ts, 6, 4, 16, [500], 1, drop=drop)
        assert got == exp
        nk, ef = kw.stats()
        assert ef & 1 and nk == 16


@pytest.mark.gpu
def test_output_capacity_too_small(progs, wfb):
    import torch
    t, ts = make_stream(3000, 5, 51)
    kw = wfb.KeyedWindowsGPU(progs[0], 10, 2, 8)
    model = Model(0, 10, 2)
    exp = model.feed(t, ts)
    cap = len(exp) - 17
    rb = RES[0].itemsize
    out = torch.full(((cap + 40) * rb,), SENTINEL, dtype=torch.uint8, device="cuda")
    out_ts = torch.full((cap + 40,), -1, dtype=torch.int64, device="cuda")
    out, out_ts, n_out = kw.process([wfb.DeviceBatch.from_host(t, ts)], capacity=cap, out=out, out_ts=out_ts)
    rows = results(kw, 0, out, out_ts, n_out)
    assert len(rows) == cap
    assert set(rows) <= set(exp)
    assert bool((out[cap * rb:].cpu() == SENTINEL).all()) and bool((out_ts[cap:].cpu() == -1).all())
    assert kw.stats()[1] & 2


@pytest.mark.gpu
def test_two_streams(progs, wfb):
    """Calls alternate between two streams with nothing synchronised in between (the inputs are uploaded first, every call writes its own
    output buffers, all are read at the end): only the handle's own stream ordering keeps the archive consistent."""
    import torch
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    t, ts = make_stream(8000, 40, 61)
    kw = wfb.KeyedWindowsGPU(progs[1], 12, 5, 64)
    model = Model(1, 12, 5)
    cuts = split(len(t), [333, 100])
    batches = [wfb.DeviceBatch.from_host(t[a:b], ts[a:b]) for (a, b) in cuts]
    torch.cuda.synchronize()
    outs = []
    for c in range(0, len(batches), 2):
        s = streams[(c // 2) % 2]
        grp = batches[c:c + 2]
        with torch.cuda.stream(s):
            outs.append(kw.process(grp, stream=s))
    outs.append(kw.flush(64 * 4, stream=streams[0]))
    torch.cuda.synchronize()
    got = []
    for o in outs:
        rows = results(kw, 1, *o)
        check_key_order(rows)
        got += rows
    exp = model.feed(t, ts) + model.flush()
    assert sorted(got) == sorted(exp) and len(got) > 0


@pytest.mark.gpu
def test_flush_only_open_windows(progs, wfb):
    """A stream whose every key ends inside open windows: flush returns exactly the model's."""
    t, ts = make_stream(997, 9, 71)
    got, exp, _ = run(wfb, progs[0], 0, t, ts, 50, 20, 16, [997], 1)
    assert got == exp
    assert any(r[-1] == int(ts.max()) and r[3] < 50 for r in got)


@pytest.mark.gpu
def test_refusals(progs, wfb):
    from windflow_b200 import _lib
    L = _lib.lib()
    h = C.c_void_p()
    assert L.wfb_kwin_create(C.byref(h), wfb.PROG_TUPLE64, 4, 2, 16, 0) == -5  # no win_func
    assert L.wfb_kwin_create(C.byref(h), progs[0], 0, 2, 16, 0) == -1
    assert L.wfb_kwin_create(C.byref(h), progs[0], 4, 0, 16, 0) == -1
    assert L.wfb_kwin_create(C.byref(h), progs[0], (1 << 24) + 1, 1, 16, 0) == -5  # ring longer than 2^24
    assert L.wfb_kwin_create(C.byref(h), progs[0], 4, 1, (1 << 30) + 1, 0) == -5
    assert L.wfb_kwin_create(C.byref(h), progs[0], 4, 1, 16, 4) == -5  # no growing key table
    assert L.wfb_kwin_create(C.byref(h), progs[1], 4, 1, 16, 1) == -1  # dense keys are integers
    assert L.wfb_kwin_create(C.byref(h), progs[0], 1 << 20, 1, 1 << 26, 1) == 2  # a 4 PiB ring: cudaErrorMemoryAllocation
    kw = wfb.KeyedWindowsGPU(progs[0], 4, 2, 16)
    assert L.wfb_kwin_process_cb(kw.h, None, 1, None, None, 0, None, None) == -1
    assert L.wfb_kwin_set_params(kw.h, None, 0) == -1
