"""The builder API (include/wf/windflow_gpu.hpp) bit for bit against a direct fold, at a size where its host machinery cycles.

The application tests/cpp/test_facade_exact.cu sends 400 300 tuples of 24 bytes over 300 hashed, Zipf-distributed keys through Map /
Filter runs fused into count-based windows (through thunks and typed, K = 1, 7, 128 batches per call), a Map -> Filter run to a Sink,
keyed-stateful Map and Filter over a 24-byte state, keyed Reduce_GPU, time-based windows with out-of-order timestamps and idle gaps, and
three graphs whose producer of deferred batch sizes runs hundreds of calls ahead of a Sink that is slow at first. It writes its stream
and the rows every Sink received, in arrival order. Here the expected rows are rebuilt with numpy and every field is compared:
  * windows: the set of windows and their ids from the oracle (oracle/oracle.py), their (h, q) from the prefix hashes of
    tests/test_gpu_ordered_windows.py -- the combine is the polynomial hash (h1, q1) o (h2, q2) = (h1 M^q2 + h2, q1 + q2), associative and
    not commutative, so tuples, windows or batches that change places change the rows; per key the Sink must see ids 0, 1, 2, ...;
  * chain_sink, stateful_p1, reduce_*: the Sink's row SEQUENCE equals the model's;
  * stateful_p2 (two replicas per operator): every state update happened exactly once (see INTEGRATION.md, keyed-stateful operators);
  * the application is built twice, with the default WF_MAX_BATCHES_PER_CALL and with 3: both must give the same rows.
CPU (-m "not gpu"): the application compiles for sm_90a, its functors on the host equal the numpy models (--host-check), and the models
of the stateful and reduce functors equal plain per-key Python loops."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import test_gpu_ordered_params as op
import test_gpu_ordered_windows as ow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_facade_exact.cu")
EXE = {"default": os.path.join(ROOT, "tests", "cpp", "test_facade_exact.bin"), "k3": os.path.join(ROOT, "tests", "cpp", "test_facade_exact_k3.bin")}
DEFS = {"default": [], "k3": ["-DWF_MAX_BATCHES_PER_CALL=3"]}
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")

N, BATCH, WIN, SLIDE, NWB = 400300, 1000, 48, 16, 3
DROP_LO, DROP_HI = 37000, 41000
TB_WIN, TB_SLIDE, TB_NWB, TB_LATE = 400, 100, 2, 150
SLOW_BATCH, SLOW_BATCHES, SINKS_BATCH, SINKS_BATCHES = 500, 800, 64, 5000
M = ow.M
U = np.uint64
TUP = np.dtype([("key", "<u8"), ("seq", "<u8"), ("value", "<u8")])
RES = ow.RES_DTYPE[32]


def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(ROOT, "include", "wf", h) for h in ("windflow_gpu.hpp", "deferred_counts.hpp")] + \
        [os.path.join(ROOT, "windflow_b200", "csrc", h) for h in ("wfb_kernels.cuh", "wfb_launch.cuh")] + [SRC]
    procs = []
    for name, exe in EXE.items():
        if os.path.exists(exe) and all(os.path.getmtime(exe) > os.path.getmtime(h) for h in hdrs):
            continue
        procs.append(subprocess.Popen(
            ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "--expt-extended-lambda",
             "-diag-suppress", "186", "-I" + os.path.join(ROOT, "include")] + DEFS[name] +
            ["-o", exe, SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"]))
    for p in procs:
        assert p.wait() == 0


# ---------------------------------------------------------------------------------------------------------------------------------
# numpy models of the application's functors (wrapping 64-bit arithmetic)
# ---------------------------------------------------------------------------------------------------------------------------------
def map_a(t):
    t = t.copy()
    with np.errstate(over="ignore"):
        t["value"] = ((t["seq"] * t["seq"]) ^ (t["seq"] >> U(3))) * U(0x9E3779B97F4A7C15) + t["key"]
    return t


def keep_a(t):
    return ((t["value"] >> U(11)) % U(3) != 0) & ~((t["seq"] >= DROP_LO) & (t["seq"] < DROP_HI))


def map_b(t):
    t = t.copy()
    with np.errstate(over="ignore"):
        t["value"] = (t["value"] ^ (t["value"] >> U(17))) * U(0xD6E8FEB86659FD93) + t["seq"]
    return t


def keep_b(t):
    return (t["value"] >> U(9)) % U(5) != 0


def chain_a(t):
    t = map_a(t)
    return t[keep_a(t)]


def chain_ab(t):
    t = map_b(chain_a(t))
    return t[keep_b(t)]


def lift_h(t):
    """The lift's item hash: ord_mix of the tuple's value and key (the 32-byte program's of tests/cpp/ordered_programs.cu)."""
    x = np.zeros(len(t), dtype=[("id", "<u8"), ("key", "<u8")])
    x["id"], x["key"] = t["value"], t["key"]
    return ow.np_lift_h(x, 32)


def _by_key(keys):
    """Stable order by key, every item's rank among its key's items and the position of its key's first item in that order."""
    order = np.argsort(keys, kind="stable")
    _, start, cnt = np.unique(keys[order], return_index=True, return_counts=True)
    first = np.repeat(start, cnt)
    return order, np.arange(len(keys)) - first, first


def stateful_model(x):
    """Keyed-stateful Map then Filter of the application over the tuples x (arrival order): the Sink's rows, in order."""
    order, rank, first = _by_key(x["key"])
    s = x[order]
    n = len(s)
    upto = np.arange(n) + 1
    cnt = (rank + 1).astype(U)
    mh, _ = ow.hash_ranges(lift_h(s), first, upto, U)  # the map's running hash of the key
    last = np.where(rank == 0, U(0), np.roll(s["seq"], 1))
    with np.errstate(over="ignore"):
        v = mh + last
    fh, _ = ow.hash_ranges(v, first, upto, U)  # the filter's, over the map's values
    out = np.zeros(n, dtype=TUP)
    out["key"], out["value"] = s["key"], fh
    out["seq"] = s["seq"] | (cnt << U(20)) | (cnt << U(42))
    res, keep = np.zeros(n, dtype=TUP), np.zeros(n, dtype=bool)
    res[order], keep[order] = out, cnt % U(4) != 0
    return res[keep]


def stateful_loop(x):
    ms, fs, out = {}, {}, []
    for key, seq, value in x.tolist():
        c, h, last = ms.get(key, (0, 0, 0))
        c, h = c + 1, (h * M + int(lift_h(np.array([(key, seq, value)], dtype=TUP))[0])) % 2**64
        value, seq2 = (h + last) % 2**64, seq | (c << 20)
        ms[key] = (c, h, seq)
        c, h, _ = fs.get(key, (0, 0, 0))
        c, h = c + 1, (h * M + value) % 2**64
        fs[key] = (c, h, seq2)
        if c % 4 != 0:
            out.append((key, seq2 | (c << 42), h))
    return np.array(out, dtype=TUP)


def small_keys(t):
    t = t.copy()
    t["key"] %= U(65521)
    return t


def reduce_model(x, batch):
    """Keyed Reduce_GPU of the application: per batch one row per key, ascending, the fold of the key's tuples in arrival order."""
    n = len(x)
    b = np.arange(n) // batch
    order = np.lexsort((np.arange(n), x["key"], b))
    s = x[order]
    new = np.ones(n, dtype=bool)
    new[1:] = (s["key"][1:] != s["key"][:-1]) | (b[order][1:] != b[order][:-1])
    starts = np.flatnonzero(new)
    with np.errstate(over="ignore"):
        total = np.add.reduceat(s["seq"], starts)
        incl = np.cumsum(s["seq"], dtype=U)
        before = np.concatenate([[U(0)], incl[starts[1:] - 1]]).astype(U)  # the sum of everything in front of the group
        grp = np.cumsum(new) - 1
        after = total[grp] - (incl - before[grp])  # the seqs of the key's later tuples: the power their value is carried by
        h = np.add.reduceat(s["value"] * op.np_pow(M, after), starts)
    out = s[starts].copy()
    out["seq"], out["value"] = total, h
    return out


def reduce_loop(x, batch):
    out = []
    for b in range(0, len(x), batch):
        acc = {}
        for key, seq, value in x[b:b + batch].tolist():
            if key in acc:
                k, q, h = acc[key]
                acc[key] = (k, q + seq, (h * pow(M, seq, 2**64) + value) % 2**64)
            else:
                acc[key] = (key, seq, value)
        out += [acc[k] for k in sorted(acc)]
    return np.array(out, dtype=TUP)


def cb_expected(O, surv, batch_of):
    """Count-based windows over the survivors (arrival order; batch_of: their source batch): rows sorted by (key, id)."""
    go = O.FfatGpuOracle(WIN, SLIDE, NWB)
    exp = []
    cuts = np.flatnonzero(np.diff(batch_of)) + 1
    for part in np.split(np.arange(len(surv)), cuts):
        r = np.zeros(len(part), dtype=O.RES)
        r["key"], r["isum"] = surv["key"][part], surv["seq"][part].astype(np.int64)
        exp.append(go.process_batch(r, int(batch_of[part[0]]))[0])
    go.close()
    e = O.sort_results(np.concatenate(exp))
    order, a, b = ow.cb_ranges(surv["key"], e["key"], e["id"], WIN, SLIDE)
    A = np.concatenate([[0], np.cumsum(surv["seq"][order].astype(np.int64))])
    assert np.array_equal(A[b] - A[a], e["isum"])  # (the oracle's windows are these arrival ranks)
    h, _ = ow.hash_ranges(lift_h(surv)[order], a, b, U)
    out = np.zeros(len(e), dtype=RES)
    out["key"], out["id"], out["h"], out["q"] = e["key"], e["id"], h, (b - a).astype(U)
    return out


def tb_expected(O, t, ts, wm):
    to = O.FfatTbOracle(TB_WIN, TB_SLIDE, TB_LATE, TB_NWB)
    exp = []
    for b in range(0, len(t), BATCH):
        r = np.zeros(len(t[b:b + BATCH]), dtype=O.RES)
        r["key"] = t["key"][b:b + BATCH]
        exp.append(to.process_batch(r, ts[b:b + BATCH], int(wm[b:b + BATCH].min()))[0])
    assert to.ignored == 0  # nothing is late: every item is in its windows
    to.close()
    e = O.sort_results(np.concatenate(exp))
    uk, dense = np.unique(t["key"], return_inverse=True)  # (tb_ranges packs a key into 32 bits)
    rk = np.searchsorted(uk, e["key"])
    assert np.array_equal(uk[rk], e["key"])
    order, a, b = ow.tb_ranges(dense.astype(U), ts, rk.astype(U), e["id"], TB_WIN, TB_SLIDE, math.gcd(TB_WIN, TB_SLIDE))
    h, _ = ow.hash_ranges(lift_h(t)[order], a, b, U)
    assert np.count_nonzero(b - a > 1) > len(e) // 2  # (most windows fold several items)
    out = np.zeros(len(e), dtype=RES)
    out["key"], out["id"], out["h"], out["q"] = e["key"], e["id"], h, (b - a).astype(U)
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# comparisons
# ---------------------------------------------------------------------------------------------------------------------------------
def canon(r):
    return r[np.lexsort((r["id"], r["key"]))]


def check_windows(run, got, exp, ordered_ids=True):
    g = canon(got)
    assert len(g) == len(exp) > 0, f"{run}: {len(g)} windows, expected {len(exp)}"
    bad = np.flatnonzero(g != exp)
    assert len(bad) == 0, f"{run}: {len(bad)} of {len(g)} windows differ from the direct fold, first (key, id), got / expected: " + \
        "; ".join(f"({int(exp['key'][i]):#x}, {int(exp['id'][i])}) {g[i]} / {exp[i]}" for i in bad[:4])
    if ordered_ids:  # per key the Sink saw ids 0, 1, 2, ...
        order, rank, _ = _by_key(got["key"])
        bad = np.flatnonzero(got["id"][order] != rank.astype(U))
        assert len(bad) == 0, f"{run}: {len(bad)} windows reached the Sink out of their key's order, first (key, id): " \
                              f"{[(hex(int(got['key'][order][i])), int(got['id'][order][i])) for i in bad[:5]]}"


def check_rows(run, got, exp):
    """The Sink's row sequence equals the model's."""
    n = min(len(got), len(exp))
    bad = np.flatnonzero(got[:n] != exp[:n])
    assert len(bad) == 0 and len(got) == len(exp), \
        f"{run}: {len(got)} rows, expected {len(exp)}; {len(bad)} differ, first (position, got / expected): " + \
        "; ".join(f"{i}: {got[i]} / {exp[i]}" for i in bad[:4])


def check_stateful_p2(got, entering):
    """Two replicas per operator share the state behind a mutex: the order of a key's updates is not defined, their number is."""
    seq, mc, fc = got["seq"] & U((1 << 20) - 1), (got["seq"] >> U(20)) & U((1 << 22) - 1), got["seq"] >> U(42)
    keys, n_k = np.unique(entering["key"], return_counts=True)
    assert len(np.unique(seq)) == len(seq) and np.array_equal(got["key"], entering["key"][np.searchsorted(entering["seq"], seq)])
    for k, n in zip(keys, n_k):
        m = got["key"] == k
        exp_f = np.arange(1, n + 1)
        assert np.array_equal(np.sort(fc[m]), exp_f[exp_f % 4 != 0]), f"stateful_p2: the filter's updates of key {int(k):#x} are not 1..{n}, each once"
        assert len(np.unique(mc[m])) == m.sum() and mc[m].min() >= 1 and mc[m].max() <= n, f"stateful_p2: a doubled or lost map update of key {int(k):#x}"


def load(d, run, dtype):
    return np.fromfile(os.path.join(str(d), run + ".bin"), dtype=dtype)


def check_outputs(d, O):
    """Every run of the application's output directory d against its model."""
    t = load(d, "stream", TUP)
    assert len(t) == N and len(np.unique(t["key"])) > 250
    a = map_a(t)
    ka = keep_a(a)
    assert not ka[DROP_LO:DROP_HI].any() and 0.6 < ka.mean() < 0.7  # whole batches are dropped, and about a third of the rest
    sa = a[ka]
    exp = cb_expected(O, sa, sa["seq"] // U(BATCH))
    runs = {r: load(d, r, RES) for r in ("cb_thunk_K1", "cb_thunk_K7", "cb_thunk_K128", "cb_typed")}
    for r, got in runs.items():
        check_windows(r, got, exp)
        assert canon(got).tobytes() == canon(runs["cb_thunk_K1"]).tobytes()
    sab = chain_ab(t)
    exp = cb_expected(O, sab, sab["seq"] // U(BATCH))
    for r in ("cb_mmff_thunk", "cb_mmff_typed"):
        check_windows(r, load(d, r, RES), exp)
    check_rows("chain_sink", load(d, "chain_sink", TUP), sa)
    check_rows("stateful_p1", load(d, "stateful_p1", TUP), stateful_model(sa))
    check_stateful_p2(load(d, "stateful_p2", TUP), sa)
    exp = reduce_model(small_keys(t), BATCH)
    r16, r64 = load(d, "reduce_bits16", TUP), load(d, "reduce_bits64", TUP)
    check_rows("reduce_bits16", r16, exp)
    check_rows("reduce_bits64", r64, exp)
    assert r16.tobytes() == r64.tobytes()
    exp = tb_expected(O, t, load(d, "tb_ts", U), load(d, "tb_wm", U))
    check_windows("tb_ooo", load(d, "tb_ooo", RES), exp)
    check_slow(d, O, t, exp)


def check_slow(d, O, t, tb_exp):
    """The runs whose producer is far ahead of a Sink that is slow at first: a deferred size that another call overwrote shows as
    missing or stale rows."""
    s = t[:SLOW_BATCH * SLOW_BATCHES]
    s = s[keep_b(s)]
    exp = cb_expected(O, s, s["seq"] // U(SLOW_BATCH))
    per_call = np.bincount((np.sort(s["seq"]) // U(SLOW_BATCH)).astype(np.int64))
    assert len(np.unique(per_call)) > 5
    check_windows("slow_sink_cb", load(d, "slow_sink_cb", RES), exp)
    check_windows("slow_sink_tb", load(d, "slow_sink_tb", RES), tb_exp)
    s = t[:SINKS_BATCH * SINKS_BATCHES]
    s = s[keep_b(s)]
    got = load(d, "slow_sinks_filter", TUP)
    check_rows("slow_sinks_filter (rows sorted by seq)", got[np.argsort(got["seq"], kind="stable")], s)


# ---------------------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------------------
@needs_nvcc
def test_facade_exact_compiles():
    _compile()
    assert all(os.path.exists(e) for e in EXE.values())


@needs_nvcc
def test_host_functors_match_numpy_models(tmp_path):
    """The application's functors on the host (--host-check: no device) against the numpy models."""
    _compile()
    out = subprocess.run([EXE["default"], "--host-check", str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "HOST_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    t = load(tmp_path, "stream", TUP)
    sa = chain_a(t)
    check_rows("host_chain_sink", load(tmp_path, "host_chain_sink", TUP), sa)
    check_rows("host_chain2", load(tmp_path, "host_chain2", TUP), chain_ab(t))
    check_rows("host_stateful", load(tmp_path, "host_stateful", TUP), stateful_model(sa))
    check_rows("host_reduce", load(tmp_path, "host_reduce", TUP), reduce_model(small_keys(t), BATCH))
    lifted = load(tmp_path, "host_lift", RES)
    assert np.array_equal(lifted["h"], lift_h(t)) and np.all(lifted["q"] == 1) and np.array_equal(lifted["key"], t["key"])
    fold = load(tmp_path, "host_fold", RES)
    n = len(fold)
    h, _ = ow.hash_ranges(lift_h(t[:n]), np.zeros(n, dtype=np.int64), np.arange(n) + 1, U)
    assert n == 5000 and np.array_equal(fold["h"], h) and np.array_equal(fold["q"], np.arange(n) + 1)


def test_models_equal_plain_loops():
    rng = np.random.default_rng(5)
    x = np.zeros(3000, dtype=TUP)
    x["key"] = rng.integers(0, 2**63, 40, dtype=np.uint64)[rng.integers(0, 40, len(x))]
    x["seq"], x["value"] = np.arange(len(x)), rng.integers(0, 2**63, len(x), dtype=np.uint64) * U(2) + U(1)
    got, exp = stateful_model(x), stateful_loop(x)
    assert len(got) == len(exp) > 2000 and got.tobytes() == exp.tobytes()
    y = small_keys(x)
    got, exp = reduce_model(y, 170), reduce_loop(y, 170)
    assert len(got) == len(exp) > 500 and got.tobytes() == exp.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("binary", ["default", "k3"])
def test_facade_exact_rows_match_direct_fold(oracle, tmp_path, binary):
    _compile()
    out = subprocess.run([EXE[binary], str(tmp_path)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "EXACT_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    check_outputs(tmp_path, oracle)
