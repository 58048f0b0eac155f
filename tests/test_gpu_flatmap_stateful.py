"""Keyed-stateful FlatMap_GPU (wfb_flatmap_stateful) against a numpy model that walks each key's tuples in arrival order, byte for byte.

The programs of tests/cpp/stateful_flatmap_programs.cu (registered at run time) push (count + field) % mod records per tuple, count
being the number of the key's earlier tuples, and every record carries a position-weighted sum over the key's history: a wrong
per-key order or state changes the bytes. Records of batch i are in input order and, per tuple, in push order, each with its tuple's
timestamp; pushes beyond the m-th of a tuple are dropped and counted in n_out[K] (their state changes stand); a tuple whose key
finds no slot pushes nothing and touches no state; K batches in one call equal K single-batch calls. Programs: 64 -> 32 bytes with
an integer key (dense and hashed tables), 16 -> 48 bytes, 64 -> 32 bytes with a 16-byte key, and a selection whose m = 1 run equals
wfb_filter_stateful of the built-in program.

CPU (-m "not gpu"): the programs compile for sm_90a and their host functors agree with the model. GPU: everything else."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "windflow_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "cpp", "stateful_flatmap_programs.cu")
SO = os.path.join(ROOT, "tests", "cpp", "stateful_flatmap_programs.so")
NVCC = ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "--expt-extended-lambda",
        "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-Xcompiler", "-fPIC", "-shared", "-diag-suppress", "186"]
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")

TUPLE64 = np.dtype([("key", "<u8"), ("id", "<u8"), ("ivalue", "<i8"), ("fvalue", "<f8"), ("pad", "<u8", (4,))])
TUPLE16 = np.dtype([("key", "<u8"), ("value", "<i8")])
REC32 = np.dtype([("key", "<u8"), ("id", "<u8"), ("j", "<u8"), ("h", "<u8")])
REC48 = np.dtype([("key", "<u8"), ("id", "<u8"), ("j", "<u8"), ("h", "<u8"), ("count", "<u8"), ("x", "<u8")])
REC = {0: REC32, 1: REC48, 2: REC32, 3: TUPLE64}
TUPLE = {0: TUPLE64, 1: TUPLE16, 2: TUPLE64, 3: TUPLE64}
MIX = np.uint64(0x9E3779B97F4A7C15)
SENTINEL = 0xAB
ALL_ONES = -1  # key id of the all-ones 16-byte key (program 2), which the key table refuses


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


_sfm = None


def sfmlib():
    """The test programs' shared object, loaded after libwfb200.so so that it binds the same library instance."""
    global _sfm
    if _sfm is None:
        _compile()
        from windflow_b200 import _lib
        _lib.lib()
        L = C.CDLL(SO)
        L.sfm_register.argtypes = [C.c_int]
        L.sfm_register.restype = C.c_int
        vp, u64 = C.c_void_p, C.c_uint64
        L.sfm_host.argtypes = [C.c_int, C.POINTER(_lib.Functors), vp, vp, u64, C.c_uint32, vp, vp, C.POINTER(u64), C.POINTER(u64)]
        L.sfm_host.restype = C.c_int
        _sfm = L
    return _sfm


@pytest.fixture(scope="module")
def progs(wfb):
    """Program id of every test program (0: 64 -> 32 bytes, 1: 16 -> 48, 2: 64 -> 32 with a 16-byte key, 3: selection)."""
    L = sfmlib()
    ids = {w: L.sfm_register(w) for w in range(4)}
    assert all(i >= 6 for i in ids.values()), ids
    return ids


def functors(map_kind=0, iadd=0, fscale=1.0, filt_kind=0, mod=1):
    from windflow_b200 import _lib
    return _lib.Functors(map_kind, filt_kind, iadd, fscale, mod)


def drawn(m):
    """Fan-out (count + field) % (m + 2): from 0 to m + 1, so some tuples push more than m."""
    return functors(mod=m + 2)


def fixed(c):
    """Fan-out c for every tuple."""
    return functors(map_kind=1, iadd=c, mod=1)


# ---------------------------------------------------------------------------------------------------------------------------------
# inputs and the numpy model
# ---------------------------------------------------------------------------------------------------------------------------------
def key_words(which, kid, dense=False):
    """(key, pad[0]) of key id kid: dense keys are the ids; hashed ones spread over 64 bits; the 16-byte key shares its first word
    among four keys (kid ALL_ONES: the all-ones key)."""
    kid = np.asarray(kid, dtype=np.int64)
    u = kid.astype(np.uint64)
    with np.errstate(over="ignore"):
        if which == 2:
            key = (u >> np.uint64(2)) * MIX + np.uint64(7)
            pad0 = (u & np.uint64(3)) * np.uint64(0x100000001) + np.uint64(5)
            ones = kid == ALL_ONES
            key[ones] = np.uint64(0xFFFFFFFFFFFFFFFF)
            pad0[ones] = np.uint64(0xFFFFFFFFFFFFFFFF)
            return key, pad0
        return (u if dense else u * MIX + np.uint64(12345)), np.zeros(len(kid), dtype=np.uint64)


def gen(which, kid, seed, dense=False):
    """Tuples of program `which` with key ids kid (ids unique per seed), their timestamps and key ids."""
    rng = np.random.default_rng(seed)
    n = len(kid)
    ts = np.sort(rng.integers(0, 1 << 40, n, dtype=np.uint64))
    key, pad0 = key_words(which, kid, dense)
    ids = np.arange(n, dtype=np.uint64) + np.uint64(seed << 32)
    if which == 1:
        t = np.zeros(n, dtype=TUPLE16)
        t["key"] = key
        t["value"] = ids.astype(np.int64)
        return t, ts, np.asarray(kid, dtype=np.int64)
    t = np.zeros(n, dtype=TUPLE64)
    t["key"], t["id"] = key, ids
    t["ivalue"] = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    t["fvalue"] = rng.random(n)
    t["pad"][:, 0] = pad0
    t["pad"][:, 1:] = rng.integers(0, 1 << 63, (n, 3), dtype=np.uint64)
    return t, ts, np.asarray(kid, dtype=np.int64)


class ModelState:
    """The model's per-key state: (count, h) of programs 0-2, the counter of program 3; key ids index it (ALL_ONES: none)."""

    def __init__(self, nkeys):
        self.count = np.zeros(nkeys, dtype=np.uint64)
        self.h = np.zeros(nkeys, dtype=np.uint64)


def model(which, batches, st, f, m, skip=()):
    """One call over `batches` [(tuples, ts, kid)]: [(records, record ts)] per batch and the dropped pushes; st advances. Key ids in
    `skip` (and ALL_ONES) find no slot."""
    kid = np.concatenate([b[2] for b in batches]) if batches else np.zeros(0, dtype=np.int64)
    t = np.concatenate([b[0] for b in batches]) if batches else np.zeros(0, dtype=TUPLE[which])
    n = len(kid)
    valid = (kid != ALL_ONES) & ~np.isin(kid, np.asarray(list(skip), dtype=np.int64))
    pos = np.nonzero(valid)[0]
    k = kid[pos]
    o = np.argsort(k, kind="stable")
    ks, ps = k[o], pos[o]
    new = np.r_[True, ks[1:] != ks[:-1]] if len(ks) else np.zeros(0, dtype=bool)
    gstart = np.maximum.accumulate(np.where(new, np.arange(len(ks)), 0)) if len(ks) else np.zeros(0, dtype=np.int64)
    rank = (np.arange(len(ks)) - gstart).astype(np.uint64)
    last = np.r_[ks[1:] != ks[:-1], True] if len(ks) else np.zeros(0, dtype=bool)
    C_ = np.zeros(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        cnt = st.count[ks] + rank
        if which == 3:  # ProgTuple64::filter_stateful: counter++, ivalue += counter, then the predicate
            u = t.copy()
            u["ivalue"][ps] += (cnt + np.uint64(1)).astype(np.int64)
            st.count[ks[last]] = cnt[last] + np.uint64(1)
            keep = np.zeros(n, dtype=bool)
            iv = u["ivalue"]
            keep[ps] = True if f.filt_kind == 0 else ((iv[ps] & 1) == 0 if f.filt_kind == 1 else np.fmod(iv[ps], np.int64(f.filt_mod)) == 0)
            C_[keep] = 1
            src = u
        else:
            ids = (t["value"].astype(np.uint64) if which == 1 else t["id"])[ps]
            field = (t["value"].astype(np.uint64) if which == 1 else t["ivalue"].astype(np.uint64))[ps]
            w = ids * MIX * (cnt + np.uint64(1))
            cs = np.cumsum(w, dtype=np.uint64)
            excl = cs - w
            h = st.h[ks] + (excl - excl[gstart])
            c = np.full(len(ks), np.uint64(f.map_iadd)) if f.map_kind == 1 else (cnt + field) % np.uint64(f.filt_mod)
            st.count[ks[last]] = cnt[last] + np.uint64(1)
            st.h[ks[last]] = h[last] + w[last]
            C_[ps] = c
            H, CNT = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64)
            H[ps], CNT[ps] = h, cnt
    kept = np.minimum(C_, np.uint64(m)).astype(np.int64)
    dropped = int((C_ - kept.astype(np.uint64)).sum())
    out, b0 = [], 0
    for tb, tsb, _ in batches:
        sl = slice(b0, b0 + len(tb))
        b0 += len(tb)
        c = kept[sl]
        idx = np.repeat(np.arange(sl.start, sl.stop), c)
        j = (np.arange(int(c.sum())) - np.repeat(np.cumsum(c) - c, c)).astype(np.uint64)
        if which == 3:
            r = src[idx]
        else:
            r = np.zeros(len(idx), dtype=REC[which])
            with np.errstate(over="ignore"):
                r["id"] = t["value"][idx].astype(np.uint64) if which == 1 else t["id"][idx]
                r["j"], r["h"] = j, H[idx]
                r["key"] = (t["key"][idx] ^ t["pad"][idx, 0]) if which == 2 else t["key"][idx]
                if which == 1:
                    r["count"], r["x"] = CNT[idx], t["key"][idx] ^ H[idx]
        out.append((r, tsb[idx - sl.start] if tsb is not None else None))
    return out, dropped


def host_run(which, t, ts, f, m):
    """The program's own functors on the host over one call with fresh states (sfm_host)."""
    L = sfmlib()
    cap = max(1, len(t) * m)
    out = np.zeros(cap, dtype=REC[which])
    ts_out = np.zeros(cap, dtype=np.uint64)
    n_out, dropped = C.c_uint64(0), C.c_uint64(0)
    t = np.ascontiguousarray(t)
    ts = np.ascontiguousarray(ts)
    assert L.sfm_host(which, C.byref(f), t.ctypes.data_as(C.c_void_p), ts.ctypes.data_as(C.c_void_p), len(t), m,
                      out.ctypes.data_as(C.c_void_p), ts_out.ctypes.data_as(C.c_void_p), C.byref(n_out), C.byref(dropped)) == 0
    k = n_out.value
    return out[:k], ts_out[:k], dropped.value


# ---------------------------------------------------------------------------------------------------------------------------------
# the GPU call
# ---------------------------------------------------------------------------------------------------------------------------------
def run_gpu(ops, ks, which, batches, f, m, with_ts=True, stream=None):
    """One wfb_flatmap_stateful call over `batches` [(tuples, ts, kid)]: [(record bytes, ts or None, untouched tail ok, count)], dropped."""
    import torch
    rb = REC[which].itemsize
    ins, outs = [], []
    for t, ts, _ in batches:
        n = len(t)
        ins.append(ops.DeviceBatch(ops.to_device(t) if n else torch.empty(TUPLE[which].itemsize, dtype=torch.uint8, device="cuda"),
                                   ops.ts_to_device(ts) if (with_ts and n) else None, n, int(ts[0]) if n else 0))
        cap = max(1, n * m)
        outs.append(ops.DeviceBatch(torch.full((cap * rb,), SENTINEL, dtype=torch.uint8, device="cuda"),
                                    torch.full((cap,), -1, dtype=torch.int64, device="cuda"), cap))
    n_out = torch.full((len(batches) + 1,), 0x7eadbeef, dtype=torch.int32, device="cuda")
    if stream is not None:
        stream.wait_stream(torch.cuda.current_stream())
    ks.flatmap(ins, f, outs, n_out, m, stream=stream)
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


def check(batches, res, dropped, exp, exp_drop, with_ts=True):
    assert len(res) == len(exp)
    for (got, got_ts, tail_ok, k), (r, rts) in zip(res, exp):
        assert k == len(r)
        assert got == r.tobytes()
        if with_ts:
            assert np.array_equal(got_ts, rts)
        assert tail_ok, "records or timestamps written beyond the batch's count (or a timestamp written without input timestamps)"
    assert dropped == exp_drop


def call_and_check(ops, ks, which, batches, st, f, m, with_ts=True, skip=(), stream=None):
    exp, exp_drop = model(which, batches, st, f, m, skip)
    res, dropped = run_gpu(ops, ks, which, batches, f, m, with_ts, stream)
    check(batches, res, dropped, exp, exp_drop, with_ts)
    return res, dropped


def split(seq, sizes):
    out, b = [], 0
    for s in sizes:
        out.append(seq[b:b + s])
        b += s
    return out


def batches_of(which, kid, sizes, seed, dense=False):
    t, ts, k = gen(which, kid, seed, dense)
    return list(zip(split(t, sizes), split(ts, sizes), split(k, sizes)))


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------------
@needs_nvcc
def test_programs_compile():
    _compile()
    assert os.path.exists(SO)


@needs_nvcc
@pytest.mark.parametrize("which", [0, 1, 2, 3])
@pytest.mark.parametrize("m", [1, 3, 8])
def test_host_functors_match_model(which, m):
    rng = np.random.default_rng(m * 10 + which)
    n = 4000
    kid = rng.integers(0, 37, n)
    t, ts, k = gen(which, kid, seed=m + 7 * which)
    fs = (functors(filt_kind=2, mod=3), functors(filt_kind=1)) if which == 3 else (drawn(m), fixed(m + 2), fixed(0))
    for f in fs:
        exp, d = model(which, [(t, ts, k)], ModelState(37), f, m)
        hr, hts, hd = host_run(which, t, ts, f, m)
        assert hr.tobytes() == exp[0][0].tobytes() and np.array_equal(hts, exp[0][1]) and hd == d
        if which != 3 and f.map_kind == 0:
            assert d > 0 and len(hr) > 0


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------
KEY_CASES = [(0, 1, False), (0, 7, True), (0, 5000, False), (0, 60000, True), (0, 1 << 17, False), (0, 1 << 20, False),
             (1, 7, False), (1, 60000, False), (1, 1 << 17, False), (2, 5000, False), (2, 1 << 17, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("which,nkeys,dense", KEY_CASES)
def test_keys_on_both_paths(wfb, progs, which, nkeys, dense):
    """1 key (a run longer than a bucket chunk of KS_CAP = 2304 items), 7, 5 000 and 60 000 keys on the bucket path; 2^17 and 2^20
    keys on the full sort. Two calls of several batches: the state carries over."""
    m = 3
    ks = wfb.KeyedState(progs[which], nkeys, dense_keys=dense)
    st = ModelState(nkeys)
    rng = np.random.default_rng(nkeys + which)
    n = max(6000, 2 * nkeys)
    for call in range(2):
        kid = rng.integers(0, nkeys, n)
        sizes = [n // 3, 1, n - n // 3 - 1 - 1000, 0, 1000]
        call_and_check(wfb, ks, which, batches_of(which, kid, sizes, seed=10 * call + 1, dense=dense), st, drawn(m), m)


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 1])
def test_zipf_keys(wfb, progs, which):
    nkeys, n, m = 65536, 1 << 18, 4
    p = 1.0 / np.arange(1, nkeys + 1) ** 0.8
    rng = np.random.default_rng(3)
    ks, st = wfb.KeyedState(progs[which], nkeys), ModelState(nkeys)
    for call in range(2):
        kid = rng.choice(nkeys, n, p=p / p.sum())
        call_and_check(wfb, ks, which, batches_of(which, kid, [n // 2, n - n // 2], seed=20 + call), st, drawn(m), m)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 7, 128])
def test_k_batches_equal_single_calls(wfb, progs, k):
    """K batches of sizes 0, 1, ... 65 536 in one call give the bytes of K single-batch calls on another handle."""
    which, m, nkeys = 0, 4, 3000
    rng = np.random.default_rng(k)
    sizes = [int(x) for x in rng.integers(0, 3000, k)]
    sizes[::4] = [int(x) for x in rng.choice([0, 1, 255, 257], len(sizes[::4]))]
    if k > 1:
        sizes[1] = 65536
    kid = rng.integers(0, nkeys, sum(sizes))
    batches = batches_of(which, kid, sizes, seed=30 + k)
    one, st1 = wfb.KeyedState(progs[which], nkeys), ModelState(nkeys)
    res, _ = call_and_check(wfb, one, which, batches, st1, drawn(m), m)
    many, st2 = wfb.KeyedState(progs[which], nkeys), ModelState(nkeys)
    for b, r in zip(batches, res):
        r1, _ = call_and_check(wfb, many, which, [b], st2, drawn(m), m)
        assert r1[0][0] == r[0] and np.array_equal(r1[0][1], r[1])


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 1, 2])
def test_fanout_all_zero_all_m_and_above(wfb, progs, which):
    m, nkeys, n = 5, 4000, 30000
    ks, st = wfb.KeyedState(progs[which], nkeys), ModelState(nkeys)
    rng = np.random.default_rng(which)
    for i, (f, per) in enumerate(((fixed(0), 0), (fixed(m), m), (fixed(m + 3), m))):
        kid = rng.integers(0, nkeys, n)
        res, dropped = call_and_check(wfb, ks, which, batches_of(which, kid, [n - 700, 700], seed=40 + i), st, f, m)
        assert [r[3] for r in res] == [(n - 700) * per, 700 * per]
        assert dropped == (3 * n if i == 2 else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 1])
def test_without_timestamps(wfb, progs, which):
    m, nkeys, n = 4, 1000, 20000
    ks, st = wfb.KeyedState(progs[which], nkeys), ModelState(nkeys)
    kid = np.random.default_rng(5).integers(0, nkeys, n)
    call_and_check(wfb, ks, which, batches_of(which, kid, [n - 999, 999], seed=50), st, drawn(m), m, with_ts=False)


@pytest.mark.gpu
def test_state_carried_across_many_calls(wfb, progs):
    which, m, nkeys = 1, 3, 100
    ks, st = wfb.KeyedState(progs[which], nkeys), ModelState(nkeys)
    rng = np.random.default_rng(6)
    for call in range(24):
        n = int(rng.integers(1, 3000))
        call_and_check(wfb, ks, which, batches_of(which, rng.integers(0, nkeys, n), [n], seed=60 + call), st, drawn(m), m)
    assert st.count.sum() > 0


@pytest.mark.gpu
def test_growing_handle_equals_fixed_one(wfb, progs):
    """From 1 024 keys past 65 536 (bucket path, then the full sort) against a fixed handle of 2^17 keys and the model."""
    which, m, nkeys = 0, 3, 100000
    grow, fixed_h = wfb.KeyedState(progs[which], 1024, grow_keys=True), wfb.KeyedState(progs[which], 1 << 17)
    sg, sf = ModelState(nkeys), ModelState(nkeys)
    rng = np.random.default_rng(7)
    for call, hi in enumerate((800, 5000, 40000, 70000, nkeys, nkeys)):
        kid = rng.integers(0, hi, 60000)
        batches = batches_of(which, kid, [30000, 30000], seed=70 + call)
        a, _ = call_and_check(wfb, grow, which, batches, sg, drawn(m), m)
        b, _ = call_and_check(wfb, fixed_h, which, batches, sf, drawn(m), m)
        assert [x[0] for x in a] == [x[0] for x in b]
    assert grow.key_capacity > 65536


@pytest.mark.gpu
def test_fixed_table_one_key_short(wfb, progs):
    """The key that finds no slot pushes nothing, call after call; every other key is the model's."""
    which, m, nkeys = 0, 3, 300
    ks = wfb.KeyedState(progs[which], nkeys - 1)
    rng = np.random.default_rng(8)
    kid = np.concatenate([np.arange(nkeys), rng.integers(0, nkeys, 5000)])
    b = batches_of(which, kid, [len(kid)], seed=80)
    res, _ = run_gpu(wfb, ks, which, b, fixed(1), m)  # one record per tuple: the missing key is the one without records
    got = np.frombuffer(res[0][0], dtype=REC32)
    missing = np.setdiff1d(b[0][0]["key"], got["key"])
    assert len(missing) == 1
    skip = [int(kid[np.nonzero(b[0][0]["key"] == missing[0])[0][0]])]
    st = ModelState(nkeys)
    exp, _ = model(which, b, st, fixed(1), m, skip)
    assert res[0][0] == exp[0][0].tobytes() and res[0][3] == len(kid) - int((kid == skip[0]).sum())
    for call in range(3):
        kid = rng.integers(0, nkeys, 8000)
        call_and_check(wfb, ks, which, batches_of(which, kid, [4000, 4000], seed=81 + call), st, drawn(m), m, skip=skip)


@pytest.mark.gpu
def test_all_ones_16_byte_key_pushes_nothing(wfb, progs):
    which, m, nkeys = 2, 3, 500
    ks, st = wfb.KeyedState(progs[which], nkeys), ModelState(nkeys)
    rng = np.random.default_rng(9)
    for call in range(2):
        kid = rng.integers(0, nkeys, 9000)
        kid[rng.random(9000) < 0.05] = ALL_ONES
        call_and_check(wfb, ks, which, batches_of(which, kid, [9000], seed=90 + call), st, fixed(2), m)


@pytest.mark.gpu
def test_calls_alternating_between_two_streams(wfb, progs):
    import torch
    which, m, nkeys = 0, 4, 2000
    ks, st = wfb.KeyedState(progs[which], nkeys), ModelState(nkeys)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    rng = np.random.default_rng(10)
    for call in range(8):
        kid = rng.integers(0, nkeys, 20000)
        call_and_check(wfb, ks, which, batches_of(which, kid, [12000, 8000], seed=100 + call), st, drawn(m), m,
                       stream=s1 if call % 2 == 0 else s2)


@pytest.mark.gpu
def test_m1_selection_equals_filter_stateful(wfb, progs):
    import torch
    ops = wfb
    f = functors(filt_kind=2, mod=3)
    nkeys = 5000
    sel, flt = ops.KeyedState(progs[3], nkeys), ops.KeyedState(ops.PROG_TUPLE64, nkeys)
    rng = np.random.default_rng(11)
    total = 0
    for call in range(3):
        sizes = [65536, 1, 0, 257, 12345]
        kid = rng.integers(0, nkeys, sum(sizes))
        batches = batches_of(3, kid, sizes, seed=110 + call)
        res, dropped = run_gpu(ops, sel, 3, batches, f, 1)
        assert dropped == 0
        ins = [ops.DeviceBatch(ops.to_device(t) if len(t) else torch.empty(64, dtype=torch.uint8, device="cuda"),
                               ops.ts_to_device(ts) if len(t) else None, len(t)) for t, ts, _ in batches]
        outs = [ops.DeviceBatch(torch.empty(max(1, len(t)) * 64, dtype=torch.uint8, device="cuda"),
                                torch.empty(max(1, len(t)), dtype=torch.int64, device="cuda"), len(t)) for t, _, _ in batches]
        n_out = torch.zeros(len(batches), dtype=torch.int32, device="cuda")
        flt.filter(ins, f, outs, n_out)
        torch.cuda.synchronize()
        counts = n_out.cpu().numpy()
        for (got, got_ts, _, k), o, c in zip(res, outs, counts):
            assert k == int(c)
            assert got == o.tuples.cpu().numpy()[:k * 64].tobytes()
            assert np.array_equal(got_ts, ops.ts_to_host(o.ts)[:k])
            total += k
    assert total > 0


@pytest.mark.gpu
def test_refusals(wfb, progs):
    import torch
    ops = wfb
    t, ts, _ = gen(0, np.zeros(10, dtype=np.int64), seed=1)
    b = [ops.DeviceBatch.from_host(t, ts)]
    o = [ops.DeviceBatch(torch.empty(32 * 10, dtype=torch.uint8, device="cuda"), torch.empty(10, dtype=torch.int64, device="cuda"), 10)]
    n_out = torch.zeros(4, dtype=torch.int32, device="cuda")
    with pytest.raises(ops.WfbError) as e:  # a program without flatmap_stateful
        ops.KeyedState(ops.PROG_TUPLE64, 16).flatmap(b, functors(), o, n_out, 1)
    assert e.value.code == -5
    ks = ops.KeyedState(progs[0], 16)
    with pytest.raises(ops.WfbError) as e:  # m = 0
        ks.flatmap(b, functors(), o, n_out, 0)
    assert e.value.code == -1
    big = [ops.DeviceBatch(b[0].tuples, b[0].ts, 1 << 20)]  # n * m >= 2^31 (refused before anything is read)
    with pytest.raises(ops.WfbError) as e:
        ks.flatmap(big, functors(), o, n_out, 1 << 11)
    assert e.value.code == -1
    near = ops.DeviceBatch(b[0].tuples, b[0].ts, (1 << 30) - 1)  # every batch below 2^31 records, the call at 2^32 or more
    with pytest.raises(ops.WfbError) as e:
        ks.flatmap([near, near, near], functors(), o * 3, n_out, 2)
    assert e.value.code == -1
    with pytest.raises(ops.WfbError) as e:  # the output overlaps the input
        ks.flatmap(b, functors(), [ops.DeviceBatch(b[0].tuples, b[0].ts, 10)], n_out, 1)
    assert e.value.code == -1
    res, dropped = run_gpu(ops, ks, 0, [(t, ts, np.zeros(10, dtype=np.int64))], fixed(1), 1)  # the handle still works
    assert res[0][3] == 10 and dropped == 0
