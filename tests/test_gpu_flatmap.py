"""FlatMap_GPU (wfb_flatmap_batches) against a numpy model of the expansion, byte for byte.

The programs of tests/cpp/flatmap_programs.cu (registered at run time, as an application registers its functors) read each tuple's
fan-out from the tuple itself, so a case sets every count: drawn from 0..m, all 0, all m, or above m (the pushes beyond the m-th of
a tuple are dropped and counted in n_out[K]). Records are placed per batch in input order and, per tuple, in push order, each with
the timestamp of the tuple that pushed it; the result of K batches in one call equals K single-batch calls. Record and tuple sizes:
64 -> 16 and 64 -> 32 bytes (64-byte tuples take the tensor-map load), 16 -> 48 bytes (the plain bulk load). A selection program
with m = 1 equals wfb_map_filter_batches of the built-in program.

CPU (-m "not gpu"): the programs compile for sm_90a and their host functors agree with the numpy model. GPU: everything else."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "windflow_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "cpp", "flatmap_programs.cu")
SO = os.path.join(ROOT, "tests", "cpp", "flatmap_programs.so")
NVCC = ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "--expt-extended-lambda",
        "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-Xcompiler", "-fPIC", "-shared", "-diag-suppress", "186"]
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")

TUPLE64 = np.dtype([("key", "<u8"), ("id", "<u8"), ("ivalue", "<i8"), ("fvalue", "<f8"), ("pad", "<u8", (4,))])
TUPLE16 = np.dtype([("key", "<u8"), ("value", "<i8")])
REC = {0: np.dtype([("key", "<u8"), ("value", "<i8")]),
       1: np.dtype([("key", "<u8"), ("id", "<u8"), ("j", "<u8"), ("value", "<i8")]),
       2: np.dtype([("key", "<u8"), ("id", "<u8"), ("value", "<i8"), ("j", "<u8"), ("a", "<u8"), ("b", "<u8")]),
       3: TUPLE64}
TUPLE = {0: TUPLE64, 1: TUPLE64, 2: TUPLE16, 3: TUPLE64}
MIX = np.uint64(0x9E3779B97F4A7C15)
SENTINEL = 0xAB


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


_fm = None


def fmlib():
    """The test programs' shared object, loaded after libwfb200.so so that it binds the same library instance."""
    global _fm
    if _fm is None:
        _compile()
        from windflow_b200 import _lib
        _lib.lib()
        L = C.CDLL(SO)
        L.fm_register.argtypes = [C.c_int]
        L.fm_register.restype = C.c_int
        vp, u64 = C.c_void_p, C.c_uint64
        L.fm_host.argtypes = [C.c_int, C.POINTER(_lib.Functors), vp, vp, u64, C.c_uint32, vp, vp, C.POINTER(u64), C.POINTER(u64)]
        L.fm_host.restype = C.c_int
        _fm = L
    return _fm


@pytest.fixture(scope="module")
def progs(wfb):
    """Program id of every test program (0: 64 -> 16 bytes, 1: 64 -> 32, 2: 16 -> 48, 3: 64 -> 64 selection)."""
    L = fmlib()
    ids = {w: L.fm_register(w) for w in range(4)}
    assert all(i >= 6 for i in ids.values()), ids
    return ids


def functors(map_kind=0, iadd=0, fscale=1.0, filt_kind=0, mod=1):
    from windflow_b200 import _lib
    return _lib.Functors(map_kind, filt_kind, iadd, fscale, mod)


# ---------------------------------------------------------------------------------------------------------------------------------
# inputs and the numpy model
# ---------------------------------------------------------------------------------------------------------------------------------
def gen(which, n, fan, seed):
    """n tuples of program `which` whose fan-out is fan[i]."""
    rng = np.random.default_rng(seed)
    fan = np.asarray(fan, dtype=np.uint64)
    ts = np.sort(rng.integers(0, 1 << 40, n, dtype=np.uint64))
    if TUPLE[which] is TUPLE16:
        t = np.zeros(n, dtype=TUPLE16)
        t["key"] = rng.integers(0, 1 << 63, n, dtype=np.uint64)
        t["value"] = (rng.integers(-(1 << 50), 1 << 50, n, dtype=np.int64) << 6) | fan.astype(np.int64)
        return t, ts
    t = np.zeros(n, dtype=TUPLE64)
    t["key"] = rng.integers(0, 1 << 63, n, dtype=np.uint64)
    t["id"] = np.arange(n, dtype=np.uint64) + np.uint64(seed << 32)
    t["ivalue"] = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    t["fvalue"] = rng.random(n)
    t["pad"][:, :3] = rng.integers(0, 1 << 63, (n, 3), dtype=np.uint64)
    t["pad"][:, 3] = fan
    return t, ts


def prefix(which, t, f):
    """The fused [map ->] [filter ->] slots (those of the built-in program over the same tuples): mapped tuples, kept mask."""
    t = t.copy()
    v = "value" if TUPLE[which] is TUPLE16 else "ivalue"
    with np.errstate(over="ignore"):
        if f.map_kind == 1:
            t[v] += np.int64(f.map_iadd)
            if v == "ivalue":
                t["fvalue"] *= f.map_fscale
    if f.filt_kind == 1:
        keep = (t[v] & 1) == 0
    elif f.filt_kind == 2:
        keep = np.fmod(t[v], np.int64(f.filt_mod)) == 0
    else:
        keep = np.ones(len(t), dtype=bool)
    return t, keep


def model(which, t, ts, f, m):
    """(records, record timestamps, dropped pushes) of one batch."""
    if which == 3:  # the selection functor runs map and filter itself; its own slots do nothing
        u, keep = prefix(3, t, f)
        return u[keep], (ts[keep] if ts is not None else None), 0
    u, keep = prefix(which, t, f)
    u = u[keep]
    fan = (u["value"].astype(np.uint64) & np.uint64(63)) if which == 2 else u["pad"][:, 3]
    c = np.minimum(fan, np.uint64(m)).astype(np.int64)
    dropped = int((fan - np.minimum(fan, np.uint64(m))).sum())
    idx = np.repeat(np.arange(len(u)), c)
    starts = np.cumsum(c) - c
    j = (np.arange(int(c.sum())) - np.repeat(starts, c)).astype(np.uint64)
    s = u[idx]
    r = np.zeros(len(idx), dtype=REC[which])
    with np.errstate(over="ignore"):
        if which == 0:
            r["key"] = s["key"] + j
            r["value"] = (s["ivalue"].astype(np.uint64) * np.uint64(3) + j).astype(np.int64)
        elif which == 1:
            r["key"], r["id"], r["j"] = s["key"], s["id"], j
            r["value"] = (s["ivalue"].astype(np.uint64) + j).astype(np.int64)
        else:
            r["key"], r["value"], r["j"] = s["key"], s["value"], j
            r["id"] = s["value"].astype(np.uint64) >> np.uint64(6)
            r["a"] = s["key"] ^ j
            r["b"] = j * MIX
    rts = ts[keep][idx] if ts is not None else None
    return r, rts, dropped


def host_run(which, t, ts, f, m):
    """The program's own functors on the host (fm_host)."""
    L = fmlib()
    cap = max(1, len(t) * m)
    out = np.zeros(cap, dtype=REC[which])
    ts_out = np.zeros(cap, dtype=np.uint64)
    n_out, dropped = C.c_uint64(0), C.c_uint64(0)
    t = np.ascontiguousarray(t)
    ts_arg = np.ascontiguousarray(ts).ctypes.data_as(C.c_void_p) if ts is not None else None
    assert L.fm_host(which, C.byref(f), t.ctypes.data_as(C.c_void_p), ts_arg, len(t), m, out.ctypes.data_as(C.c_void_p),
                     ts_out.ctypes.data_as(C.c_void_p), C.byref(n_out), C.byref(dropped)) == 0
    k = n_out.value
    return out[:k], (ts_out[:k] if ts is not None else None), dropped.value


# ---------------------------------------------------------------------------------------------------------------------------------
# the GPU call
# ---------------------------------------------------------------------------------------------------------------------------------
def run_gpu(ops, eng, which, batches, f, m, with_ts=True):
    """One wfb_flatmap_batches call over `batches` [(tuples, ts)]: [(records, ts or None, untouched tail ok)], dropped."""
    import torch
    rb = REC[which].itemsize
    ins, outs = [], []
    for t, ts in batches:
        n = len(t)
        ins.append(ops.DeviceBatch(ops.to_device(t) if n else torch.empty(TUPLE[which].itemsize, dtype=torch.uint8, device="cuda"),
                                   ops.ts_to_device(ts) if (with_ts and n) else None, n, int(ts[0]) if n else 0))
        cap = max(1, n * m)
        outs.append(ops.DeviceBatch(torch.full((cap * rb,), SENTINEL, dtype=torch.uint8, device="cuda"),
                                    torch.full((cap,), -1, dtype=torch.int64, device="cuda"), cap))
    n_out = torch.full((len(batches) + 1,), 0x7eadbeef, dtype=torch.int32, device="cuda")
    eng.flatmap_batches(ins, f, outs, n_out, m)
    torch.cuda.synchronize()
    counts = n_out.cpu().numpy().astype(np.int64)
    res = []
    for i, o in enumerate(outs):
        k = int(counts[i])
        raw = o.tuples.cpu().numpy()
        ots = ops.ts_to_host(o.ts)
        tail_ok = bool((raw[k * rb:] == SENTINEL).all()) and bool((ots[k:] == np.uint64(0xFFFFFFFFFFFFFFFF)).all())
        res.append((raw[:k * rb].tobytes(), ots[:k].copy() if with_ts else None, tail_ok, k))
    return res, int(counts[-1])


def check(which, batches, res, dropped, f, m, with_ts=True):
    exp_drop = 0
    for (t, ts), (got, got_ts, tail_ok, k) in zip(batches, res):
        r, rts, d = model(which, t, ts if with_ts else None, f, m)
        exp_drop += d
        assert k == len(r)
        assert got == r.tobytes()
        if with_ts:
            assert np.array_equal(got_ts, rts)
        assert tail_ok, "records or timestamps written beyond the batch's count (or a timestamp written without input timestamps)"
    assert dropped == exp_drop


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------------
@needs_nvcc
def test_programs_compile():
    _compile()
    assert os.path.exists(SO)


@needs_nvcc
@pytest.mark.parametrize("which", [0, 1, 2])
@pytest.mark.parametrize("m", [1, 3, 8, 32])
def test_host_functors_match_model(which, m):
    rng = np.random.default_rng(m * 10 + which)
    n = 3000
    fan = rng.integers(0, m + 1, n)
    over = rng.random(n) < 0.1
    fan[over] = m + rng.integers(1, 6, int(over.sum()))
    t, ts = gen(which, n, fan, seed=m + 7 * which)
    for f in (functors(), functors(map_kind=1, iadd=3, fscale=1.5, filt_kind=1), functors(filt_kind=2, mod=3)):
        r, rts, d = model(which, t, ts, f, m)
        hr, hts, hd = host_run(which, t, ts, f, m)
        assert hr.tobytes() == r.tobytes() and np.array_equal(hts, rts) and hd == d
        assert d > 0


@needs_nvcc
def test_host_selection_matches_model():
    t, ts = gen(3, 2000, np.zeros(2000), seed=3)
    f = functors(map_kind=1, iadd=2, fscale=1.0000001, filt_kind=2, mod=3)
    r, rts, _ = model(3, t, ts, f, 1)
    hr, hts, hd = host_run(3, t, ts, f, 1)
    assert hr.tobytes() == r.tobytes() and np.array_equal(hts, rts) and hd == 0 and 0 < len(r) < len(t)


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 2])
@pytest.mark.parametrize("m", [1, 3, 8, 32])
def test_fanout_drawn_from_0_to_m(wfb, progs, which, m):
    eng = wfb.Engine(progs[which])
    rng = np.random.default_rng(m)
    n = 70001
    batches = [gen(which, n, rng.integers(0, m + 1, n), seed=m)]
    res, dropped = run_gpu(wfb, eng, which, batches, functors(), m)
    check(which, batches, res, dropped, functors(), m)


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 1, 2])
def test_all_zero_and_all_m(wfb, progs, which):
    eng, m, n = wfb.Engine(progs[which]), 8, 5000
    batches = [gen(which, n, np.zeros(n), seed=1), gen(which, n, np.full(n, m), seed=2), gen(which, 300, np.zeros(300), seed=3)]
    res, dropped = run_gpu(wfb, eng, which, batches, functors(), m)
    check(which, batches, res, dropped, functors(), m)
    assert res[0][3] == 0 and res[1][3] == n * m and res[2][3] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("which", [1, 2])
def test_batch_sizes(wfb, progs, which):
    eng, m = wfb.Engine(progs[which]), 3
    rng = np.random.default_rng(11)
    batches = [gen(which, n, rng.integers(0, m + 1, n), seed=20 + i) for i, n in enumerate([0, 1, 255, 257, 65536])]
    res, dropped = run_gpu(wfb, eng, which, batches, functors(), m)
    check(which, batches, res, dropped, functors(), m)
    for b, r in zip(batches, res):  # each size alone
        r1, d1 = run_gpu(wfb, eng, which, [b], functors(), m)
        assert r1[0][0] == r[0] and np.array_equal(r1[0][1], r[1]) and d1 == 0


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 2])
@pytest.mark.parametrize("k", [1, 7, 128])
def test_k_batches_equal_single_calls(wfb, progs, which, k):
    eng, m = wfb.Engine(progs[which]), 8
    rng = np.random.default_rng(k)
    sizes = rng.integers(0, 3000, k)
    sizes[::5] = rng.choice([0, 1, 255, 256, 257], len(sizes[::5]))
    batches = [gen(which, int(n), rng.integers(0, m + 1, int(n)), seed=100 + i) for i, n in enumerate(sizes)]
    res, dropped = run_gpu(wfb, eng, which, batches, functors(), m)
    check(which, batches, res, dropped, functors(), m)
    for b, r in zip(batches, res):
        r1, _ = run_gpu(wfb, eng, which, [b], functors(), m)
        assert r1[0][0] == r[0] and np.array_equal(r1[0][1], r[1])


@pytest.mark.gpu
@pytest.mark.parametrize("which", [1, 2])
def test_without_timestamps(wfb, progs, which):
    eng, m, n = wfb.Engine(progs[which]), 4, 20000
    rng = np.random.default_rng(5)
    batches = [gen(which, n, rng.integers(0, m + 1, n), seed=5), gen(which, 999, rng.integers(0, m + 1, 999), seed=6)]
    res, dropped = run_gpu(wfb, eng, which, batches, functors(), m, with_ts=False)
    check(which, batches, res, dropped, functors(), m, with_ts=False)


@pytest.mark.gpu
@pytest.mark.parametrize("which", [1, 2])
def test_fused_map_filter_prefix(wfb, progs, which):
    eng, m = wfb.Engine(progs[which]), 8
    rng = np.random.default_rng(9)
    batches = [gen(which, n, rng.integers(0, m + 1, n), seed=40 + n) for n in (40000, 1, 257, 3000)]
    for f in (functors(map_kind=1, iadd=3, fscale=1.5, filt_kind=1), functors(map_kind=1, iadd=1, filt_kind=2, mod=3)):
        res, dropped = run_gpu(wfb, eng, which, batches, f, m)
        check(which, batches, res, dropped, f, m)
        u, keep = prefix(which, batches[0][0], f)
        assert 0 < keep.sum() < len(keep)


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 2])
@pytest.mark.parametrize("m", [1, 3, 32])
def test_pushes_beyond_m_are_dropped_and_counted(wfb, progs, which, m):
    eng = wfb.Engine(progs[which])
    rng = np.random.default_rng(77 + m)
    batches = []
    for i, n in enumerate((50000, 700, 1)):
        fan = rng.integers(0, m + 1, n)
        over = rng.random(n) < 0.2
        fan[over] = m + 1
        fan[over & (rng.random(n) < 0.3)] = m + 5
        if n == 1:
            fan[:] = m + 1
        batches.append(gen(which, n, fan, seed=60 + i))
    res, dropped = run_gpu(wfb, eng, which, batches, functors(), m)
    check(which, batches, res, dropped, functors(), m)
    assert dropped > 0


@pytest.mark.gpu
def test_m1_selection_equals_map_filter_batches(wfb, progs):
    import torch
    ops = wfb
    f = functors(map_kind=1, iadd=2, fscale=1.0000001, filt_kind=2, mod=3)
    batches = [gen(3, int(n), np.zeros(int(n)), seed=80 + i) for i, n in enumerate([65536, 1, 0, 257, 12345, 255, 70000])]
    res, dropped = run_gpu(ops, ops.Engine(progs[3]), 3, batches, f, 1)
    assert dropped == 0
    ins = [ops.DeviceBatch(ops.to_device(t) if len(t) else torch.empty(64, dtype=torch.uint8, device="cuda"),
                           ops.ts_to_device(ts) if len(t) else None, len(t)) for t, ts in batches]
    outs = [ops.DeviceBatch(torch.empty(max(1, len(t)) * 64, dtype=torch.uint8, device="cuda"),
                            torch.empty(max(1, len(t)), dtype=torch.int64, device="cuda"), len(t)) for t, _ in batches]
    n_out = torch.zeros(len(batches), dtype=torch.int32, device="cuda")
    ops.Engine(ops.PROG_TUPLE64).map_filter_batches(ins, f, outs, n_out, stream=None)
    torch.cuda.synchronize()
    counts = n_out.cpu().numpy()
    assert sum(r[3] for r in res) > 0
    for (got, got_ts, _, k), o, c in zip(res, outs, counts):
        assert k == int(c)
        assert got == o.tuples.cpu().numpy()[:k * 64].tobytes()
        assert np.array_equal(got_ts, ops.ts_to_host(o.ts)[:k])


@pytest.mark.gpu
def test_refusals(wfb, progs):
    import torch
    ops = wfb
    t, ts = gen(0, 10, np.ones(10), seed=1)
    b = [ops.DeviceBatch.from_host(t, ts)]
    o = [ops.DeviceBatch(torch.empty(64 * 10, dtype=torch.uint8, device="cuda"), torch.empty(10, dtype=torch.int64, device="cuda"), 10)]
    n_out = torch.zeros(2, dtype=torch.int32, device="cuda")
    with pytest.raises(ops.WfbError) as e:  # a program without a flatmap functor
        ops.Engine(ops.PROG_TUPLE64).flatmap_batches(b, functors(), o, n_out, 1)
    assert e.value.code == -5
    with pytest.raises(ops.WfbError) as e:  # m = 0
        ops.Engine(progs[0]).flatmap_batches(b, functors(), o, n_out, 0)
    assert e.value.code == -1
    big = [ops.DeviceBatch(b[0].tuples, b[0].ts, 1 << 20)]  # n * m >= 2^31 (refused before anything is read)
    with pytest.raises(ops.WfbError) as e:
        ops.Engine(progs[0]).flatmap_batches(big, functors(), o, n_out, 1 << 11)
    assert e.value.code == -1
