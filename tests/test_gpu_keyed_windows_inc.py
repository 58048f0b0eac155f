"""Incremental Keyed_Windows_GPU (wfb_kwin_* with WFB_KWIN_INCREMENTAL) against a direct Python fold, every field exact.

Per key, tuples get ids 0, 1, 2, ... in arrival order; window g holds ids [g*slide, g*slide + win). Its accumulator starts as
make_result(key, g) when tuple g*slide arrives, every tuple IN the window is folded into it in arrival order, and it fires with tuple
g*slide + win (not folded), carrying that tuple's timestamp. At end of stream every window that opened and has not fired is emitted with
the largest timestamp seen. The programs of tests/cpp/kwin_inc_programs.cu fold an order-sensitive hash, the size, the first and last id,
the ivalue % 16 mask, the fvalue sum in order and the id of the first largest ivalue: a window that misses a tuple, folds another key's or
folds them out of order changes the result.

The handle keeps R = pow2ceil(ceil(win / slide)) accumulators per key. Within one call a window open before it can fire while a window
opened in the same call stays open in the same ring entry (test_ring_hazard drives exactly that).

CPU (-m "not gpu"): the programs compile for sm_90a and the model agrees with a brute-force enumeration of the windows. GPU: the rest."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_gpu_keyed_windows import KEY16, NVCC, brute_windows, key_of, make_stream, split

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "windflow_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "cpp", "kwin_inc_programs.cu")
SO = os.path.join(ROOT, "tests", "cpp", "kwin_inc_programs.so")
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")

TUPLE256 = np.dtype([("key", "<u8"), ("id", "<u8"), ("ivalue", "<i8"), ("fvalue", "<f8"), ("pad", "<u8", (28,))])
FIELDS = [("id", "<u8"), ("hash", "<u8"), ("size", "<u8"), ("front", "<u8"), ("back", "<u8"), ("mask", "<u8"), ("fsum", "<f8"),
          ("argmax", "<u8"), ("maxiv", "<i8")]
RES = {0: np.dtype([("key", "<u8")] + FIELDS), 1: np.dtype([("key", KEY16)] + FIELDS),
       2: np.dtype([("key", "<u8")] + FIELDS + [("pad_sum", "<u8"), ("pad", "<u8", (21,))])}
MIX, MUL, M64 = 0x9E3779B97F4A7C15, 0x100000001B3, (1 << 64) - 1
SENTINEL = 0xAB


# ---------------------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------------------
def new_acc():
    return [0, 0, None, None, 0, 0.0, None, None, 0]  # hash, size, front, back, mask, fsum, argmax, maxiv, pad_sum


def fold(a, row):
    i, iv, fv = int(row["id"]), int(row["ivalue"]), float(row["fvalue"])
    if a[1] == 0 or iv > a[7]:
        a[6], a[7] = i, iv
    if a[1] == 0:
        a[2] = i
    a[0] = (a[0] * MUL + (((i * MIX) & M64) ^ (iv & M64))) & M64
    a[1] += 1
    a[3] = i
    a[4] |= 1 << (iv & 15)
    a[5] += fv
    if "pad" in row.dtype.names and len(row["pad"]) == 28:
        a[8] = (a[8] + int(row["pad"][27])) & M64


def row_of(prog, k, g, a, ts):
    r = (k, g, a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7])
    return r + ((a[8],) if prog == 2 else ()) + (int(ts),)


class IncModel:
    """Count-based keyed windows with an incremental function, tuple after tuple (wf/window_replica.hpp:293-303, DETERMINISTIC mode)."""

    def __init__(self, prog, win, slide):
        self.prog, self.win, self.slide = prog, win, slide
        self.cnt, self.open, self.last_ts = {}, {}, 0

    def feed(self, rows, ts, drop=()):
        out = []
        for row, t in zip(rows, ts):
            k = key_of(0 if self.prog == 2 else self.prog, row)
            self.last_ts = max(self.last_ts, int(t))
            if k in drop:
                continue
            i = self.cnt.get(k, 0)
            opn = self.open.setdefault(k, {})
            if i >= self.win and (i - self.win) % self.slide == 0:  # tuple i fires window g: FIRED, not IN
                g = (i - self.win) // self.slide
                out.append(row_of(self.prog, k, g, opn.pop(g), t))
            if i % self.slide == 0:
                opn[i // self.slide] = new_acc()
            for g, a in opn.items():
                if g * self.slide <= i < g * self.slide + self.win:
                    fold(a, row)
            self.cnt[k] = i + 1
        return out

    def flush(self):
        return [row_of(self.prog, k, g, opn[g], self.last_ts) for k, opn in self.open.items() for g in sorted(opn)]


def rows_of_keys(t):
    by = {}
    for i in range(len(t)):
        by.setdefault(key_of(0, t[i]), []).append(i)
    return by


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


_kwi = None


def kwilib():
    global _kwi
    if _kwi is None:
        _compile()
        from windflow_b200 import _lib
        _lib.lib()
        L = C.CDLL(SO)
        L.kwi_register.argtypes = [C.c_int]
        L.kwi_register.restype = C.c_int
        _kwi = L
    return _kwi


@pytest.fixture(scope="module")
def progs(wfb):
    L = kwilib()
    ids = {w: L.kwi_register(w) for w in range(4)}
    assert all(i >= 6 for i in ids.values()), ids
    return ids


# ---------------------------------------------------------------------------------------------------------------------------------
# running a handle
# ---------------------------------------------------------------------------------------------------------------------------------
def make_stream256(n, nkeys, seed):
    t64, ts = make_stream(n, nkeys, seed)
    t = np.zeros(n, TUPLE256)
    for f in ("key", "id", "ivalue", "fvalue"):
        t[f] = t64[f]
    t["pad"][:, 27] = t["id"] * np.uint64(3) + np.uint64(11)
    return t, ts


def results(prog, out, out_ts, n_out):
    import torch
    torch.cuda.synchronize()
    n = int(n_out.cpu()[0])
    r = out.cpu().numpy().view(RES[prog])[:n]
    ts = out_ts.cpu().numpy().view(np.uint64)[:n]
    rows = []
    for x, t in zip(r, ts):
        k = (int(x["key"]["key"]), int(x["key"]["a"]), int(x["key"]["b"])) if prog == 1 else int(x["key"])
        row = (k, int(x["id"]), int(x["hash"]), int(x["size"]), int(x["front"]), int(x["back"]), int(x["mask"]), float(x["fsum"]),
               int(x["argmax"]), int(x["maxiv"]))
        rows.append(row + ((int(x["pad_sum"]),) if prog == 2 else ()) + (int(t),))
    return rows


def check_key_order(rows):
    last = {}
    for r in rows:
        assert last.get(r[0], -1) < r[1], ("window order", r[0], last.get(r[0]), r[1])
        last[r[0]] = r[1]


def run(wfb, prog_id, prog, t, ts, win, slide, max_keys, sizes, K, streams=None, drop=(), flush=True, dense=False):
    """Feeds the stream K batches per call to an incremental handle; returns (gpu rows, model rows, handle)."""
    import torch
    kw = wfb.KeyedWindowsGPU(prog_id, win, slide, max_keys, dense_keys=dense, incremental=True)
    model = IncModel(prog, win, slide)
    cuts = split(len(t), sizes)
    batches = [wfb.DeviceBatch.from_host(t[a:b], ts[a:b]) if b > a else
               wfb.DeviceBatch(torch.empty(0, dtype=torch.uint8, device="cuda"), None, 0) for (a, b) in cuts]
    got, exp = [], []
    for c in range(0, len(batches), K):
        s = streams[(c // K) % len(streams)] if streams else None
        out, out_ts, n_out = kw.process(batches[c:c + K], stream=s)
        rows = results(prog, out, out_ts, n_out)
        check_key_order(rows)
        got += rows
        a, b = cuts[c][0], cuts[min(c + K, len(cuts)) - 1][1]
        exp += model.feed(t[a:b], ts[a:b], drop)
    if flush:
        out, out_ts, n_out = kw.flush(max_keys * (-(-win // slide)))
        rows = results(prog, out, out_ts, n_out)
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
    subprocess.check_call(NVCC + ["-o", str(tmp_path / "kwi.so"), SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200"])


@pytest.mark.parametrize("win,slide", [(1, 1), (1, 3), (3, 5), (8, 8), (10, 3), (16, 4), (5, 1), (6, 9)])
def test_model_matches_enumeration(win, slide):
    t, ts = make_stream(500, 3, win * 100 + slide)
    m = IncModel(0, win, slide)
    got = sorted(m.feed(t, ts) + m.flush())
    exp = []
    for k, sel in rows_of_keys(t).items():
        fired, opened = brute_windows(len(sel), win, slide)
        for g, trig in fired + [(g, None) for g in opened]:
            a = new_acc()
            for i in range(g * slide, min(g * slide + win, len(sel))):
                fold(a, t[sel[i]])
            exp.append(row_of(0, k, g, a, ts[sel[trig]] if trig is not None else int(ts.max())))
    assert got == sorted(exp) and len(got) > 0


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
@pytest.mark.parametrize("win,slide", [(10, 3), (1024, 64)])
def test_ring_hazard(progs, wfb, win, slide):
    """One key, single calls of thousands of tuples (each one fires windows that were open before it while windows it opens stay open in
    the same ring entries), then small calls."""
    t, ts = make_stream(12000, 1, 7)
    got, exp, _ = run(wfb, progs[0], 0, t, ts, win, slide, 4, [5000, 3000, 7, 1, 30, 2, 100], 1)
    assert got == exp and len(got) > 0


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
    keys = np.random.default_rng(3).integers(0, nkeys, n).astype(np.uint64) if dense else None
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
    """Bit 1, nothing written past the capacity, and the windows that stay open are still exact afterwards (the flush)."""
    import torch
    t, ts = make_stream(3000, 5, 51)
    kw = wfb.KeyedWindowsGPU(progs[0], 10, 2, 8, incremental=True)
    model = IncModel(0, 10, 2)
    exp = model.feed(t, ts)
    cap = len(exp) - 17
    rb = RES[0].itemsize
    out = torch.full(((cap + 40) * rb,), SENTINEL, dtype=torch.uint8, device="cuda")
    out_ts = torch.full((cap + 40,), -1, dtype=torch.int64, device="cuda")
    out, out_ts, n_out = kw.process([wfb.DeviceBatch.from_host(t, ts)], capacity=cap, out=out, out_ts=out_ts)
    rows = results(0, out, out_ts, n_out)
    assert len(rows) == cap
    assert set(rows) <= set(exp)
    assert bool((out[cap * rb:].cpu() == SENTINEL).all()) and bool((out_ts[cap:].cpu() == -1).all())
    assert kw.stats()[1] & 2
    assert sorted(results(0, *kw.flush(8 * 5))) == sorted(model.flush())


@pytest.mark.gpu
def test_two_streams(progs, wfb):
    """Calls alternate between two streams with nothing synchronised in between: only the handle's own stream ordering keeps the
    accumulators consistent."""
    import torch
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    t, ts = make_stream(8000, 40, 61)
    kw = wfb.KeyedWindowsGPU(progs[1], 12, 5, 64, incremental=True)
    model = IncModel(1, 12, 5)
    cuts = split(len(t), [333, 100])
    batches = [wfb.DeviceBatch.from_host(t[a:b], ts[a:b]) for (a, b) in cuts]
    torch.cuda.synchronize()
    outs = []
    for c in range(0, len(batches), 2):
        s = streams[(c // 2) % 2]
        with torch.cuda.stream(s):
            outs.append(kw.process(batches[c:c + 2], stream=s))
    outs.append(kw.flush(64 * 3, stream=streams[0]))
    torch.cuda.synchronize()
    got = []
    for o in outs:
        rows = results(1, *o)
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
    inc = wfb.KWIN_INCREMENTAL
    assert L.wfb_kwin_create(C.byref(h), progs[3], 4, 2, 16, inc) == -5  # no win_func_inc
    assert L.wfb_kwin_create(C.byref(h), wfb.PROG_TUPLE64, 4, 2, 16, inc) == -5
    assert L.wfb_kwin_create(C.byref(h), progs[0], 4, 2, 16, inc | 4) == -5  # no growing key table
    assert L.wfb_kwin_create(C.byref(h), progs[0], 4, 2, 16, inc | 2) == -5
    assert L.wfb_kwin_create(C.byref(h), progs[1], 4, 2, 16, inc | 1) == -1  # dense keys are integers
    assert L.wfb_kwin_create(C.byref(h), progs[0], 0, 2, 16, inc) == -1
    assert L.wfb_kwin_create(C.byref(h), progs[0], (1 << 24) + 1, 1, 16, inc) == -5
    assert L.wfb_kwin_create(C.byref(h), progs[0], 1 << 24, 1, 1 << 26, inc | 1) == 2  # 2^26 keys x 2^24 accumulators: cudaErrorMemoryAllocation
    kw = wfb.KeyedWindowsGPU(progs[0], 4, 2, 16, dense_keys=True, incremental=True)  # the flag combines with dense keys
    assert L.wfb_kwin_process_cb(kw.h, None, 1, None, None, 0, None, None) == -1


@pytest.mark.gpu
def test_large_windows(progs, wfb):
    """win 2^20 / slide 2^18 on 65 536 keys: 4 accumulators of 80 bytes per key, 20 MiB (the tuple ring would be 2^20 x 64 bytes per key,
    4 TiB, and no test allocates it). Then win 2^16 / slide 2^14 on 3 keys, long enough for windows to fire, against the model."""
    big = wfb.KeyedWindowsGPU(progs[0], 1 << 20, 1 << 18, 65536, incremental=True)
    t, ts = make_stream(4096, 5, 3)
    out, out_ts, n_out = big.process([wfb.DeviceBatch.from_host(t, ts)])
    assert results(0, out, out_ts, n_out) == [] and big.stats() == (5, 0)
    big.close()
    t, ts = make_stream(400000, 3, 81)
    got, exp, kw = run(wfb, progs[0], 0, t, ts, 1 << 16, 1 << 14, 4, [65536, 40000, 7, 100000], 1)
    assert got == exp and sum(1 for r in got if r[3] == 1 << 16) >= 9
    assert kw.stats() == (3, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("win,slide", [(10, 3), (12, 12), (6, 9), (100, 7)])
def test_cross_check_with_noninc(progs, wfb, win, slide):
    """One stream through an incremental and a non-incremental handle of the same program: the same windows, keys, ids, timestamps and
    fields."""
    t, ts = make_stream(6000, 11, win + slide)
    inc = wfb.KeyedWindowsGPU(progs[0], win, slide, 16, incremental=True)
    non = wfb.KeyedWindowsGPU(progs[0], win, slide, 16)
    got = {0: [], 1: []}
    for a, b in split(len(t), [700, 13, 1900]):
        batch = [wfb.DeviceBatch.from_host(t[a:b], ts[a:b])]
        got[0] += results(0, *inc.process(batch))
        got[1] += results(0, *non.process(batch))
    got[0] += results(0, *inc.flush(16 * 40))
    got[1] += results(0, *non.flush(16 * 40))
    assert sorted(got[0]) == sorted(got[1]) and len(got[0]) > 0


@pytest.mark.gpu
def test_large_records(progs, wfb):
    t, ts = make_stream256(5000, 6, 91)
    got, exp, kw = run(wfb, progs[2], 2, t, ts, 20, 6, 16, [900, 1, 64], 2)
    assert got == exp and len(got) > 0
    assert kw.stats() == (6, 0)
