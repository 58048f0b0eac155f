"""The window operators with a program whose combine reads its params, against a direct fold.

The program of tests/cpp/ordered_program_32p.cu folds the polynomial hash of tests/test_gpu_ordered_windows.py with the multiplier M
read in its combine: (h1, q1) o (h2, q2) = (h1 M^q2 + h2, q1 + q2), so a window's h is the same hash and its q is the window's
length. A window-update kernel launched without the handle's params folds with M^q2 = 0 and keeps only the right operand's h. Every
32-byte count-based case and both time-based cases of tests/test_gpu_ordered_windows.py run with it here, which pins each update launch
site (bucket, lanes, heavy, deferred, lazy, pipelined, bucket-move, time-based back end) to the handle's params. The windows that
fire, their ids and timestamps come from the oracle as there.

CPU (-m "not gpu"): the program compiles, its host comb / lift agree with the numpy model. GPU: the windows of every case."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import test_gpu_ordered_windows as ow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "ordered_program_32p.cu")
SO = os.path.join(ROOT, "tests", "cpp", "ordered_program_32p.so")
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
RES32 = ow.RES_DTYPE[32]
M = ow.M


def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(ow.CSRC, h) for h in ("wfb_kernels.cuh", "wfb_keys.cuh", "wfb_launch.cuh", "wfb_programs.cuh", "wfb_ptx.cuh")] + \
        [os.path.join(ROOT, "include", "wfb200.h"), SRC]
    if os.path.exists(SO) and all(os.path.getmtime(SO) > os.path.getmtime(h) for h in hdrs):
        return
    subprocess.check_call(ow.NVCC + ["-o", SO, SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200",
                                     "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"])


_so = None


def lib32p():
    """The program's shared object, loaded after libwfb200.so so that it binds the same library instance."""
    global _so
    if _so is None:
        _compile()
        from windflow_b200 import _lib
        _lib.lib()
        L = C.CDLL(SO)
        vp, u64 = C.c_void_p, C.c_uint64
        L.ord32p_register.restype = C.c_int
        L.ord32p_comb_host.argtypes = [u64, vp, vp, vp, vp, vp, vp, u64, C.c_int]
        L.ord32p_comb_host.restype = None
        L.ord32p_lift_host.argtypes = [u64, vp, u64, vp, vp, vp]
        L.ord32p_lift_host.restype = None
        _so = L
    return _so


def register(ops):
    """Program id of the program, its dtypes registered with ops."""
    prog = lib32p().ord32p_register()
    assert prog >= 6, prog
    ops.RESULT_DTYPE[prog], ops.TUPLE_DTYPE[prog] = RES32, ow.TUPLE64
    return prog


@pytest.fixture(scope="module")
def prog32p(wfb):
    prog = register(wfb)
    yield prog
    wfb.RESULT_DTYPE.pop(prog, None); wfb.TUPLE_DTYPE.pop(prog, None)


# ---------------------------------------------------------------------------------------------------------------------------------
# numpy model
# ---------------------------------------------------------------------------------------------------------------------------------
def np_pow(b, e):
    """b ** e per element, wrapping uint64 (squaring)."""
    e = np.array(e, dtype=np.uint64)
    r, b = np.ones_like(e), np.full_like(e, b)
    with np.errstate(over="ignore"):
        for _ in range(64):
            r = np.where(e & np.uint64(1), r * b, r)
            b = b * b
            e = e >> np.uint64(1)
    return r


def np_comb_p(h1, q1, h2, q2):
    with np.errstate(over="ignore"):
        return (h1 * np_pow(M, q2) + h2).astype(np.uint64), (q1 + q2).astype(np.uint64)


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------
CB_CASES = [c for c in ow.CASES if c.rec == 32]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CB_CASES, ids=lambda c: c.name)
def test_params_cb_windows_match_direct_fold(wfb, oracle, prog32p, monkeypatch, case):
    ops, O = wfb, oracle
    if case.move:
        monkeypatch.setenv("WFB_BUCKET_MOVE", "1")  # read when the handle is created
    t, calls = case.stream()
    if case.census:
        ow.assert_regimes(ow.census(ow._geometry(case), case.call_slots(calls)), case.expect)
    e, et, h, _, surv = ow._expected(O, case, t, calls)
    _, a, b = ow.cb_ranges(surv["key"], e["key"], e["id"], case.win, case.slide)
    got, gts, err = ow._run_cb(ops, ops._lib.lib(), prog32p, case, calls)
    assert err == 0
    ow._check(got, gts, e, et, h, (b - a).astype(np.uint64), 32)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ow.TB_CASES, ids=[c[0] for c in ow.TB_CASES])
def test_params_tb_windows_match_direct_fold(wfb, oracle, prog32p, case):
    import torch
    ops, O = wfb, oracle
    name, win, slide, nb, late, cap, nkeys, n, batch, group, div, jitter = case
    t, ts = ow._tb_stream(nkeys, n, div, jitter, seed=len(name))
    to = O.FfatTbOracle(win, slide, late, nb)
    L = ops._lib.lib()
    ff = ops.FfatWindowsGPU(prog32p, win, slide, nb, max_keys=cap, dense_keys=True, win_type=1, lateness=late)
    prm = C.c_uint64(M)
    ops.check(L.wfb_ffat_set_params(ff.h, C.byref(prm), C.sizeof(prm)), "wfb_ffat_set_params")
    exp, ets, got, gts, batches = [], [], [], [], []
    for b in range(0, n, batch):
        tb, tsb = t[b:b + batch], ts[b:b + batch]
        k = ow.keep_mask(tb)
        r, rt = to.process_batch(ow._lift_res(tb[k]), tsb[k], int(tsb[0]))
        exp.append(r); ets.append(rt)
        batches.append(ops.DeviceBatch.from_host(tb, tsb))
    assert to.ignored == 0
    for i in range(0, len(batches), group):
        out, out_ts, n_out = ff.process(batches[i:i + group])
        torch.cuda.synchronize()
        r, rt = ff.results_to_host(out, out_ts, n_out)
        got.append(r); gts.append(rt)
    assert ff.stats()[1] == 0
    e, et = O.sort_results(np.concatenate(exp), np.concatenate(ets))
    k = ow.keep_mask(t)
    surv, sts = t[k], ts[k]
    order, a, b = ow.tb_ranges(surv["key"], sts, e["key"], e["id"], win, slide, math.gcd(win, slide))
    h, _ = ow.hash_ranges(ow.np_lift_h(surv, 32)[order], a, b, np.uint64)
    assert np.count_nonzero(b - a > 1) > len(e) // 2  # (most windows fold several items)
    ow._check(np.concatenate(got), np.concatenate(gts), e, et, h, (b - a).astype(np.uint64), 32)


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU checks
# ---------------------------------------------------------------------------------------------------------------------------------
@needs_nvcc
def test_params_program_compiles():
    _compile()
    assert os.path.exists(SO)


def _host(h1, q1, h2, q2, alias=0, m=M):
    a = [np.ascontiguousarray(x, dtype=np.uint64) for x in (h1, q1, h2, q2)]
    ho, qo = np.zeros(len(h1), np.uint64), np.zeros(len(h1), np.uint64)
    lib32p().ord32p_comb_host(m, *map(ow._p, a), ow._p(ho), ow._p(qo), len(h1), alias)
    return ho, qo


@needs_nvcc
def test_host_comb_matches_numpy_model():
    """The program's comb on the host == the numpy model, out aliasing an operand or not, == a plain loop at small lengths; associative
    on triples, not commutative, zero is its identity; all-zero params keep the right operand's h wherever it is not empty."""
    rng = np.random.default_rng(320)
    n = 4096
    v = [rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n).astype(np.uint64) for _ in range(6)]
    v[1][:64] = 0; v[3][64:128] = 0  # zero lengths among the pairs
    for alias in (0, 1):
        ho, qo = _host(v[0], v[1], v[2], v[3], alias)
        eh, eq = np_comb_p(v[0], v[1], v[2], v[3])
        assert np.array_equal(ho, eh) and np.array_equal(qo, eq)
    q2 = np.arange(n, dtype=np.uint64) % np.uint64(50)
    eh = np_comb_p(v[0], v[1], v[2], q2)[0]
    for i in range(0, n, 41):
        x = int(v[0][i])
        for _ in range(int(q2[i])):
            x = x * M % 2**64
        assert int(eh[i]) == (x + int(v[2][i])) % 2**64
    h0 = _host(v[0], v[1], v[2], q2, m=0)[0]
    with np.errstate(over="ignore"):
        assert np.array_equal(h0[q2 != 0], v[2][q2 != 0]) and np.array_equal(h0[q2 == 0], (v[0] + v[2])[q2 == 0])
    ab = np_comb_p(v[0], v[1], v[2], v[3])
    left = _host(*ab, v[4], v[5], 1)
    right = _host(v[0], v[1], *np_comb_p(v[2], v[3], v[4], v[5]))
    assert np.array_equal(left[0], right[0]) and np.array_equal(left[1], right[1])
    ba = _host(v[2], v[3], v[0], v[1])
    assert np.count_nonzero(ba[0] != ab[0]) > n * 0.9
    z = np.zeros(n, dtype=np.uint64)
    assert all(np.array_equal(x, y) for x, y in zip(_host(z, z, v[0], v[1], 1), (v[0], v[1])))
    assert all(np.array_equal(x, y) for x, y in zip(_host(v[0], v[1], z, z), (v[0], v[1])))


@needs_nvcc
def test_host_lift_matches_numpy_model():
    """h is the hash of the 32-byte program of tests/cpp/ordered_programs.cu, q = 1, the same filter."""
    rng = np.random.default_rng(420)
    t = ow.make_tuples(rng.integers(0, 2**64 - 2, 5000, dtype=np.uint64), int(rng.integers(0, 2**40)), 32)
    h, q, keep = np.zeros(len(t), np.uint64), np.zeros(len(t), np.uint64), np.zeros(len(t), np.uint8)
    lib32p().ord32p_lift_host(M, ow._p(t), len(t), ow._p(h), ow._p(q), ow._p(keep))
    assert np.array_equal(h, ow.np_lift_h(t, 32)) and np.all(h != 0)
    assert np.all(q == 1)
    assert np.array_equal(keep.astype(bool), ow.keep_mask(t)) and 0 < keep.sum() < len(t)
