"""Every GPU handle called on a different stream from one call to the next, against a direct fold of the same calls.

A replica that binds each call to its batch's own stream (Batch_GPU_t creates one per batch, wf/batch_gpu_t.hpp:101) calls the
same handle on a different stream every time. A handle's scratch and state are shared by its calls, so each call has to wait on the
device for everything the handle issued before, and a query that takes a stream has to see every earlier call.

The schedule is adversarial and deterministic. The calls go, one after the other, to a cycle of three non-blocking streams and the
legacy default stream, in segments of two: a spin kernel (torch.cuda._sleep) on the stream of the first call, the first call, then
the second on the next stream, which has nothing pending. A library that does not order the second call behind the first runs it
while the first is still asleep, and the first after it: the result is wrong values. The two calls never overlap, so such a library
computes in the wrong order instead of racing on its scratch. After a segment the event recorded behind its second call is
synchronised, and the one behind its first call must be done. Inputs and outputs are allocated before the schedule, behind one
synchronisation, and read after another one, so the caching allocator never hands memory from one stream to another.

Every comparison is bit-exact, except floating-point sums against a direct fold that associates differently (1e-6 relative)."""
import ctypes as C
import threading
import types

import numpy as np
import pytest

import test_gpu_flatmap as fm
import test_gpu_ordered_windows as ow

pytestmark = pytest.mark.gpu

# spin length of the sleep at the head of a segment, chosen so that the control test below passes with a wide margin: on an H100
# SXM (700 W power limit, 1980 MHz max SM clock) it lasts 101 ms, while the twelve unordered calls of the control take 3 ms.
SLEEP_CYCLES = 200_000_000
FA = 1.0000001


# ---------------------------------------------------------------------------------------------------------------------------------
# the schedule
# ---------------------------------------------------------------------------------------------------------------------------------
class Hops:
    """Runs (name, call(stream)) on a cycle of streams, in segments of two; records the second calls that finished before the first."""

    def __init__(self):
        import torch
        legacy = torch.cuda.default_stream()
        assert legacy.cuda_stream == 0  # the legacy default stream (handle 0)
        pool = [torch.cuda.Stream() for _ in range(3)]
        self.cycle = [pool[0], pool[1], legacy, pool[2]]  # (in and out of the legacy stream)
        self.k = 0
        self.late = []

    def next_stream(self):
        s = self.cycle[self.k % len(self.cycle)]
        self.k += 1
        return s

    def run(self, calls):
        import torch
        for a in range(0, len(calls), 2):
            evs = []
            for j, (name, call) in enumerate(calls[a:a + 2]):
                s = self.next_stream()
                if j == 0:
                    with torch.cuda.stream(s):
                        torch.cuda._sleep(SLEEP_CYCLES)
                call(s)
                e = torch.cuda.Event()
                e.record(s)
                evs.append(e)
            if len(evs) == 2:
                evs[1].synchronize()
                if not evs[0].query():
                    self.late.append(f"{calls[a + 1][0]} finished before {calls[a][0]}")
            torch.cuda.synchronize()

    def assert_ordered(self):
        assert not self.late, f"{len(self.late)} calls were not ordered behind the call before them: {self.late[:6]}"


def _empty(ops, with_ts=True):
    import torch
    return ops.DeviceBatch(torch.empty(0, dtype=torch.uint8, device="cuda"),
                           torch.empty(0, dtype=torch.int64, device="cuda") if with_ts else None, 0, 0)


def _like(ops, b):
    import torch
    return ops.DeviceBatch(torch.empty_like(b.tuples), torch.empty_like(b.ts) if b.ts is not None else None, b.n, 0)


# ---------------------------------------------------------------------------------------------------------------------------------
# control
# ---------------------------------------------------------------------------------------------------------------------------------
def test_schedule_is_adversarial(wfb, oracle):
    """Unordered work on another stream finishes while the sleep still runs: twelve engine calls at 300 000 tuples (more than the
    second call of any segment does) issued on B after a sleep on A are done before A wakes up."""
    import torch
    ops, O = wfb, oracle
    n = 299999
    eng = ops.Engine(ops.PROG_TUPLE64)
    eng.set_key_bits(20)
    t, ts = O.gen_tuple64(0, n, O.KEY_UNIFORM, 5000)
    b = ops.DeviceBatch.from_host(t, ts)
    out, n_out = _like(ops, b), torch.zeros(1, dtype=torch.int32, device="cuda")
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    for s in (None, None):  # warm up: scratch at its size, modules loaded
        eng.map_filter(b, ops.functors(map_kind=1, iadd=1, filt_kind=2, mod=3), out=out, n_out=n_out, stream=s)
        eng.reduce_by_key(b, out=out, n_out=n_out, stream=s)
    torch.cuda.synchronize()
    t0, t1, b0, b1 = (torch.cuda.Event(enable_timing=True) for _ in range(4))
    eA, eB = torch.cuda.Event(), torch.cuda.Event()
    with torch.cuda.stream(A):
        t0.record()
        torch.cuda._sleep(SLEEP_CYCLES)
        t1.record()
    eA.record(A)
    b0.record(B)
    for _ in range(6):
        eng.map_filter(b, ops.functors(map_kind=1, iadd=1, filt_kind=2, mod=3), out=out, n_out=n_out, stream=B)
        eng.reduce_by_key(b, out=out, n_out=n_out, stream=B)
    b1.record(B)
    eB.record(B)
    eB.synchronize()
    assert not eA.query(), "the sleep ended before unordered work on another stream: the schedule would not be adversarial"
    torch.cuda.synchronize()
    sleep_ms, work_ms = t0.elapsed_time(t1), b0.elapsed_time(b1)
    print(f"sleep of {SLEEP_CYCLES} cycles: {sleep_ms:.1f} ms; 12 unordered calls at {n} tuples on another stream: {work_ms:.2f} ms")
    assert sleep_ms > 4 * work_ms


# ---------------------------------------------------------------------------------------------------------------------------------
# engines
# ---------------------------------------------------------------------------------------------------------------------------------
def _engine_calls(ops, O, eng, fme, n, seed):
    """The stateless and per-batch calls of one engine at n tuples (and FlatMap_GPU on a registered program): a list of (name, call)
    and the check of their results after the schedule."""
    import torch
    L = eng.L
    rng = np.random.default_rng(seed)
    f = ops.functors(map_kind=1, iadd=int(rng.integers(1, 9)), fscale=FA, filt_kind=2, mod=3)

    def gen(n, nkeys=5000):
        t, ts = O.gen_tuple64(int(rng.integers(0, 1 << 30)), n, O.KEY_UNIFORM, nkeys)
        t["pad"] = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
        ts = rng.permutation(n).astype(np.uint64) * np.uint64(7)  # not monotone: a reduced key's ts is the max
        return t, ts

    calls, checks = [], []
    dev = ops.DeviceBatch.from_host

    t_all, ts_all = gen(n)
    b_all = dev(t_all, ts_all)  # read-only input of the calls that do not write it

    # Reduce_GPU un-keyed
    ra_t = torch.empty(64, dtype=torch.uint8, device="cuda")
    ra_ts = torch.zeros(1, dtype=torch.int64, device="cuda")
    calls.append(("reduce_all", lambda s: ops.check(L.wfb_reduce_all(eng.h, ops._ptr(b_all.tuples), ops._ptr(b_all.ts), n, ops._ptr(ra_t),
                                                                     ops._ptr(ra_ts), ops._stream_ptr(s)), "wfb_reduce_all")))

    def check_reduce_all():
        r = ops.to_host(ra_t, ops.TUPLE64)[0]
        assert r["key"] == 0 and r["id"] == 0 and r["ivalue"] == t_all["ivalue"].sum()
        assert abs(r["fvalue"] - t_all["fvalue"].sum()) <= 1e-6 * abs(t_all["fvalue"].sum())
        assert int(ops.ts_to_host(ra_ts)[0]) == int(ts_all.max())
    checks.append(check_reduce_all)

    # Map_GPU in place
    t_m, ts_m = gen(n)
    b_m = dev(t_m, ts_m)
    calls.append(("map", lambda s: eng.map(b_m, f, stream=s)))

    def check_map():
        assert ops.to_host(b_m.tuples, ops.TUPLE64).tobytes() == O.map_filter_tuple64(t_m, ts_m, 1, f.map_iadd, FA, 0)[0].tobytes()
    checks.append(check_map)

    # [Map_GPU ->] Filter_GPU out of place and in place
    o_mf, n_mf = _like(ops, b_all), torch.full((1,), -1, dtype=torch.int32, device="cuda")
    calls.append(("map_filter", lambda s: eng.map_filter(b_all, f, out=o_mf, n_out=n_mf, stream=s)))
    t_mi, ts_mi = gen(n)
    b_mi = dev(t_mi, ts_mi)
    n_mi = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    calls.append(("map_filter in place", lambda s: eng.map_filter(b_mi, f, out=b_mi, n_out=n_mi, stream=s)))

    def check_mf(t, ts, out, n_out, what):
        exp, ets, _ = O.map_filter_tuple64(t, ts, 1, f.map_iadd, FA, 2, 3)
        k = int(n_out.item())
        assert k == len(exp), what
        assert ops.to_host(out.tuples, ops.TUPLE64)[:k].tobytes() == exp.tobytes(), what
        assert np.array_equal(ops.ts_to_host(out.ts)[:k], ets), what
    checks.append(lambda: check_mf(t_all, ts_all, o_mf, n_mf, "map_filter"))
    checks.append(lambda: check_mf(t_mi, ts_mi, b_mi, n_mi, "map_filter in place"))

    # the same over K queued batches (one empty)
    cut = [0, n // 3, n // 3, n]
    mfb_in = [dev(t_all[a:b], ts_all[a:b]) if b > a else _empty(ops) for a, b in zip(cut, cut[1:])]
    mfb_out = [_like(ops, x) for x in mfb_in]
    n_mfb = torch.full((3,), -1, dtype=torch.int32, device="cuda")
    calls.append(("map_filter_batches", lambda s: eng.map_filter_batches(mfb_in, f, mfb_out, n_mfb, stream=s)))

    def check_mfb():
        no = n_mfb.cpu().numpy()
        for i, (a, b) in enumerate(zip(cut, cut[1:])):
            exp, ets, _ = O.map_filter_tuple64(t_all[a:b], ts_all[a:b], 1, f.map_iadd, FA, 2, 3)
            assert no[i] == len(exp)
            if len(exp):
                assert ops.to_host(mfb_out[i].tuples, ops.TUPLE64)[:len(exp)].tobytes() == exp.tobytes()
                assert np.array_equal(ops.ts_to_host(mfb_out[i].ts)[:len(exp)], ets)
    checks.append(check_mfb)

    # Reduce_GPU keyed, one batch and K batches
    o_rk, n_rk = _like(ops, b_all), torch.full((1,), -1, dtype=torch.int32, device="cuda")
    calls.append(("reduce_by_key", lambda s: eng.reduce_by_key(b_all, out=o_rk, n_out=n_rk, stream=s)))
    cut2 = [0, n // 2 + 1, n]
    rkb_in = [dev(t_all[a:b], ts_all[a:b]) for a, b in zip(cut2, cut2[1:])]
    rkb_out = [_like(ops, x) for x in rkb_in]
    n_rkb = torch.full((2,), -1, dtype=torch.int32, device="cuda")
    calls.append(("reduce_by_key_batches", lambda s: eng.reduce_by_key_batches(rkb_in, rkb_out, n_rkb, stream=s)))

    def check_reduce(t, ts, out, k, what):
        exp, ets = O.reduce_tuple64(t, ts)
        assert k == len(exp), what
        got = ops.to_host(out.tuples, ops.TUPLE64)[:k]
        assert np.array_equal(got["key"], exp["key"]) and np.array_equal(got["ivalue"], exp["ivalue"]), what
        assert np.allclose(got["fvalue"], exp["fvalue"], rtol=1e-6, atol=0), what
        assert np.array_equal(got["id"], exp["id"]) and np.array_equal(got["pad"], exp["pad"]), what
        assert np.array_equal(ops.ts_to_host(out.ts)[:k], ets), what
    checks.append(lambda: check_reduce(t_all, ts_all, o_rk, int(n_rk.item()), "reduce_by_key"))
    checks.append(lambda: [check_reduce(t_all[a:b], ts_all[a:b], rkb_out[i], int(n_rkb[i].item()), f"reduce_by_key_batches {i}")
                           for i, (a, b) in enumerate(zip(cut2, cut2[1:]))])

    # KeyBy_Emitter_GPU grouping
    kg = [torch.full((n,), -7, dtype=torch.int32, device="cuda"), torch.full((n,), -7, dtype=torch.int32, device="cuda"),
          torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")]
    calls.append(("keyby_group", lambda s: ops.check(L.wfb_keyby_group(eng.h, ops._ptr(b_all.tuples), n, *map(ops._ptr, kg), ops._stream_ptr(s)),
                                                     "wfb_keyby_group")))

    def check_keyby():
        es, em, ek = O.keyby_group(t_all["key"], 1)
        k = int(kg[3].item())
        assert k == len(ek)
        assert np.array_equal(kg[2].cpu().numpy().view(np.uint64)[:k], ek)
        assert np.array_equal(kg[0].cpu().numpy()[:k], es) and np.array_equal(kg[1].cpu().numpy(), em)
    checks.append(check_keyby)

    # key -> shard partition, and the fused [map -> filter ->] lift -> partition
    shards = 4
    o_sh, seg = _like(ops, b_all), torch.full((shards + 1,), -1, dtype=torch.int32, device="cuda")
    calls.append(("shard_by_key", lambda s: ops.check(L.wfb_shard_by_key(eng.h, ops._ptr(b_all.tuples), ops._ptr(b_all.ts), n, shards,
                                                                         ops._ptr(o_sh.tuples), ops._ptr(o_sh.ts), ops._ptr(seg),
                                                                         ops._stream_ptr(s)), "wfb_shard_by_key")))

    def check_shard():
        dest = O.route(t_all["key"], shards)
        order = np.argsort(dest, kind="stable")
        assert ops.to_host(o_sh.tuples, ops.TUPLE64).tobytes() == t_all[order].tobytes()
        assert np.array_equal(ops.ts_to_host(o_sh.ts), ts_all[order])
        assert np.array_equal(seg.cpu().numpy(), np.concatenate([[0], np.cumsum(np.bincount(dest, minlength=shards))]))
    checks.append(check_shard)

    lshards = 3
    regions = torch.zeros(lshards * n * 32, dtype=torch.uint8, device="cuda")
    counts = torch.full((9,), -1, dtype=torch.int32, device="cuda")
    calls.append(("shard_lift", lambda s: eng.shard_lift(mfb_in, f, lshards, regions, n, counts, stream=s)))

    def check_lift():
        surv, _, _ = O.map_filter_tuple64(t_all, ts_all, 1, f.map_iadd, FA, 2, 3)
        lifted = O.lift_tuple64(surv)
        dest = O.route(surv["key"], lshards)
        c = counts.cpu().numpy()
        assert c[8] == 0
        got = ops.to_host(regions, ops.RESULT32).reshape(lshards, n)
        for d in range(lshards):
            exp = lifted[dest == d]
            assert c[d] == len(exp) and got[d][:c[d]].tobytes() == exp.tobytes()
    checks.append(check_lift)

    # FlatMap_GPU (program 1 of tests/cpp/flatmap_programs.cu: 64 -> 32 bytes, up to m records per tuple), two calls in a row
    m = 3
    ff = fm.functors(map_kind=1, iadd=3, fscale=1.5, filt_kind=1)
    for c in range(2):
        fm_batches = [fm.gen(1, k, rng.integers(0, m + 2, k), seed=seed * 10 + 3 * c + i) for i, k in enumerate((n - n // 4, 0, n // 4))]
        fm_in = [ops.DeviceBatch(ops.to_device(t), ops.ts_to_device(ts), len(t), int(ts[0])) if len(t) else _empty(ops)
                 for t, ts in fm_batches]
        fm_out = [ops.DeviceBatch(torch.full((max(1, len(t) * m) * 32,), fm.SENTINEL, dtype=torch.uint8, device="cuda"),
                                  torch.full((max(1, len(t) * m),), -1, dtype=torch.int64, device="cuda"), len(t) * m) for t, _ in fm_batches]
        n_fm = torch.full((len(fm_batches) + 1,), -1, dtype=torch.int32, device="cuda")
        calls.append((f"flatmap_batches {c}", lambda s, i=fm_in, o=fm_out, k=n_fm: fme.flatmap_batches(i, ff, o, k, m, stream=s)))

        def check_flatmap(fm_batches=fm_batches, fm_out=fm_out, n_fm=n_fm):
            counts = n_fm.cpu().numpy().astype(np.int64)
            dropped = 0
            for i, ((t, ts), o) in enumerate(zip(fm_batches, fm_out)):
                r, rts, d = fm.model(1, t, ts, ff, m)
                dropped += d
                assert counts[i] == len(r)
                assert o.tuples.cpu().numpy()[:len(r) * 32].tobytes() == r.tobytes()
                assert np.array_equal(ops.ts_to_host(o.ts)[:len(r)], rts)
            assert counts[-1] == dropped > 0
        checks.append(check_flatmap)
    return calls, checks


def test_engine_hops(wfb, oracle):
    """One Engine(PROG_TUPLE64) and one FlatMap_GPU engine through every per-batch call, at sizes that grow (1 003, 70 001, 299 999
    tuples: the first pass over a size grows the scratch on hops; the second, on the same sizes, hops without growing)."""
    import torch
    ops, O = wfb, oracle
    fm_prog = fm.fmlib().fm_register(1)
    assert fm_prog >= 6
    eng, fme = ops.Engine(ops.PROG_TUPLE64), ops.Engine(fm_prog)
    eng.set_key_bits(20)
    passes = [_engine_calls(ops, O, eng, fme, n, seed=i) for i, n in enumerate((1003, 1003, 70001, 70001, 299999, 299999))]
    torch.cuda.synchronize()
    hops = Hops()
    for calls, _ in passes:
        hops.run(calls)
    torch.cuda.synchronize()
    for _, checks in passes:
        for c in checks:
            c()
    hops.assert_ordered()


# ---------------------------------------------------------------------------------------------------------------------------------
# keyed-stateful Map_GPU / Filter_GPU
# ---------------------------------------------------------------------------------------------------------------------------------
KS_CASES = [  # name, max_keys, dense, grow, keys
    ("buckets_7", 16, False, False, "7"),
    ("buckets_5000", 8192, False, False, "5000"),
    ("full_sort_100000", 100000, True, False, "spread"),
    ("grow", 16, False, True, "5000"),
]
KS_SIZES = [3000, 1, 2700]  # every call, the warm-up too: no scratch grows under a pending call
KS_FUNCS = {"tuple64": [("map", 1), ("map", 2), ("filter", 2)], "wftest16": [("map", 1), ("map", 2)]}


def _ks_keys(kind, rng):
    if kind == "7":
        return rng.integers(0, 1 << 63, 7, dtype=np.uint64)
    if kind == "5000":
        return rng.choice(1 << 40, 5000, replace=False).astype(np.uint64) * np.uint64(977)
    return np.unique(np.concatenate([rng.choice(99999, 2999, replace=False), [99999]])).astype(np.uint64)  # dense, over the slot range


def _ks_call(ops, prog, keyset, rng, first=False):
    """One call's batches (host): KS_SIZES tuples whose keys are drawn from keyset (the warm-up call: every key at least once)."""
    n = sum(KS_SIZES)
    keys = keyset[rng.integers(0, len(keyset), n)]
    if first:
        keys[:len(keyset)] = rng.permutation(keyset)
    if prog == ops.PROG_WFTEST16:
        t = np.zeros(n, dtype=ops.WFTEST16)
        t["key"], t["value"] = keys, rng.integers(-1000, 1000, n)
    else:
        t = np.zeros(n, dtype=ops.TUPLE64)
        t["key"], t["id"] = keys, np.arange(n)
        t["ivalue"], t["fvalue"] = rng.integers(-1000, 1000, n), rng.random(n)
        t["pad"] = rng.integers(0, 1 << 63, (n, 4), dtype=np.uint64)
    ts = rng.integers(0, 1 << 40, n).astype(np.uint64)
    cut = np.cumsum([0] + KS_SIZES)
    return [(t[a:b], ts[a:b]) for a, b in zip(cut, cut[1:])]


@pytest.mark.parametrize("prog_name", ["wftest16", "tuple64"])
@pytest.mark.parametrize("case", KS_CASES, ids=[c[0] for c in KS_CASES])
def test_keyed_state_hops(wfb, oracle, prog_name, case):
    """Map (map_kind 1 and 2) and, on the 64-byte tuples, filter (filt_kind 2) calls on one KeyedState, each on the next stream:
    every key's state sequence is the per-key fold of the whole call sequence."""
    import torch
    ops, O = wfb, oracle
    name, max_keys, dense, grow, keykind = case
    prog = ops.PROG_WFTEST16 if prog_name == "wftest16" else ops.PROG_TUPLE64
    dt, field = (ops.WFTEST16, "value") if prog == ops.PROG_WFTEST16 else (ops.TUPLE64, "ivalue")
    rng = np.random.default_rng(len(name) * 7 + prog)
    keyset = _ks_keys(keykind, rng)
    ks = ops.KeyedState(prog, max_keys=max_keys, dense_keys=dense, grow_keys=grow)
    ncalls = 1 + 8
    host = [_ks_call(ops, prog, keyset, rng, first=(i == 0)) for i in range(ncalls)]
    funcs = [KS_FUNCS[prog_name][i % len(KS_FUNCS[prog_name])] for i in range(ncalls)]
    ins, outs, n_outs = [], [], []
    for i, bs in enumerate(host):
        ins.append([ops.DeviceBatch.from_host(t, ts) for t, ts in bs])
        outs.append([_like(ops, b) for b in ins[-1]] if funcs[i][0] == "filter" else None)
        n_outs.append(torch.full((len(bs),), -1, dtype=torch.int32, device="cuda"))

    def call(i):
        kind, k = funcs[i]
        if kind == "map":
            return lambda s: ks.map(ins[i], ops.functors(map_kind=k), stream=s)
        return lambda s: ks.filter(ins[i], ops.functors(filt_kind=k, mod=3), outs[i], n_outs[i], stream=s)
    torch.cuda.synchronize()
    call(0)(None)  # warm-up on one stream: every key in the table, the scratch at the size of every call
    torch.cuda.synchronize()
    cap0 = ks.key_capacity
    hops = Hops()
    hops.run([(f"call {i} ({funcs[i][0]} {funcs[i][1]})", call(i)) for i in range(1, ncalls)])
    torch.cuda.synchronize()
    assert ks.key_capacity == cap0 >= len(keyset)  # (no growth in the schedule)
    state, wrong = {}, []
    for i, bs in enumerate(host):
        kind, k = funcs[i]
        no = n_outs[i].cpu().numpy()
        for j, (t, ts) in enumerate(bs):
            if kind == "map":
                exp = O.stateful_map(t, field, state, k)
                got = ops.to_host(ins[i][j].tuples, dt)
            else:
                exp, ets, _ = O.stateful_filter(t, ts, field, state, k, 3)
                if no[j] != len(exp):
                    wrong.append(f"call {i} batch {j}: {no[j]} survivors, expected {len(exp)}")
                got = ops.to_host(outs[i][j].tuples, dt)[:len(exp)] if len(exp) else exp
                if no[j] == len(exp) and len(exp) and not np.array_equal(ops.ts_to_host(outs[i][j].ts)[:len(exp)], ets):
                    wrong.append(f"call {i} batch {j}: survivor timestamps")
            if len(got) == len(exp) and got.tobytes() != exp.tobytes():
                bad = np.flatnonzero(got[field] != exp[field])
                wrong.append(f"call {i} ({kind} {k}) batch {j}: {len(bad)} of {len(exp)} tuples differ")
    assert not wrong, "states applied out of call order: " + "; ".join(wrong[:8])
    hops.assert_ordered()


def test_keyed_state_shared_by_two_replica_threads(wfb, oracle):
    """Two replicas share one KeyedState, each on its own stream and thread with its own keys (key % 2): the calls overlap (ctypes
    releases the GIL), and every key's states are the per-key fold of its replica's calls in order."""
    import torch
    ops, O = wfb, oracle
    rng = np.random.default_rng(2)
    keyset = rng.choice(1 << 40, 2000, replace=False).astype(np.uint64)
    ks = ops.KeyedState(ops.PROG_WFTEST16, max_keys=4096)
    ncalls, n = 24, 4096

    def batch(keys):
        t = np.zeros(len(keys), dtype=ops.WFTEST16)
        t["key"], t["value"] = keys, rng.integers(-1000, 1000, len(keys))
        return t
    warm = batch(np.concatenate([keyset, keyset[rng.integers(0, len(keyset), n - len(keyset))]]))
    parts = [keyset[keyset % np.uint64(2) == np.uint64(r)] for r in (0, 1)]
    host = [[batch(parts[r][rng.integers(0, len(parts[r]), n)]) for _ in range(ncalls)] for r in (0, 1)]
    dev = [[ops.DeviceBatch.from_host(t, np.zeros(n, dtype=np.uint64)) for t in h] for h in host]
    d_warm = ops.DeviceBatch.from_host(warm, np.zeros(n, dtype=np.uint64))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    kinds = [[1 + (i % 2) for i in range(ncalls)], [1 + ((i + 1) % 2) for i in range(ncalls)]]
    torch.cuda.synchronize()
    ks.map([d_warm], ops.functors(map_kind=1))
    torch.cuda.synchronize()
    errors = []
    start = threading.Barrier(2)

    def replica(r):
        try:
            start.wait()
            for i in range(ncalls):
                ks.map([dev[r][i]], ops.functors(map_kind=kinds[r][i]), stream=streams[r])
        except Exception as e:  # (reported below)
            errors.append(e)
    th = [threading.Thread(target=replica, args=(r,)) for r in (0, 1)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    torch.cuda.synchronize()
    assert not errors, errors
    state = {}
    O.stateful_map(warm, "value", state, 1)
    for r in (0, 1):
        for i in range(ncalls):
            exp = O.stateful_map(host[r][i], "value", state, kinds[r][i])
            assert ops.to_host(dev[r][i].tuples, ops.WFTEST16).tobytes() == exp.tobytes(), f"replica {r} call {i}"


# ---------------------------------------------------------------------------------------------------------------------------------
# count-based windows
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ordered(wfb):
    """Program id of the 32-byte order-sensitive program of tests/cpp/ordered_programs.cu."""
    i = ow._ordlib().ord_register_32()
    assert i >= 6
    wfb.RESULT_DTYPE[i], wfb.TUPLE_DTYPE[i] = ow.RES_DTYPE[32], ow.TUPLE64
    yield i
    wfb.RESULT_DTYPE.pop(i, None); wfb.TUPLE_DTYPE.pop(i, None)


CB_CASES = [  # name, win, slide, nb, capacity, dense, grow, pipelined, keys of each call (count, key range)
    ("buckets_dense", 48, 16, 1, 65536, True, False, False, [(3001, 64), (70001, 64), (150001, 64), (150001, 64)]),
    ("buckets_hashed", 40, 10, 2, 65536, False, False, False, [(3001, 1000), (70001, 1000), (150001, 1000), (150001, 1000)]),
    ("full_sort", 40, 10, 2, 1 << 17, True, False, False, [(3001, 3000), (70001, 3000), (150001, 3000), (150001, 3000)]),
    ("grow_on_a_hop", 40, 10, 2, 64, False, True, False, [(3001, 40), (70001, 1000), (150001, 1000), (150001, 1000)]),
    ("buckets_pipelined", 48, 16, 1, 65536, True, False, True, [(3001, 64), (70001, 64), (150001, 64)]),
    ("full_sort_pipelined", 40, 10, 2, 1 << 17, True, False, True, [(3001, 3000), (70001, 3000), (150001, 3000)]),
]


def _cb_stream(calls_spec, cap, dense, seed, batch=4000):
    """Per call, its batches [(tuples, ts = id)], and all tuples; dense keys spread over the slot range (and its last slot)."""
    rng = np.random.default_rng(seed)
    keys = []
    for n, nk in calls_spec:
        ks = (np.linspace(0, cap - 1, nk).astype(np.uint64) if dense else np.arange(nk, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
        keys.append(ks[rng.integers(0, nk, n)])
    t = ow.make_tuples(np.concatenate(keys), 0, 32)
    calls, off = [], 0
    for n, _ in calls_spec:
        calls.append([(t[b:min(b + batch, off + n)], t["id"][b:min(b + batch, off + n)].copy()) for b in range(off, off + n, batch)])
        off += n
    return t, calls


def _window_buffers(ops, ff, cap_records, count):
    import torch
    rb = ff.res_dtype.itemsize
    return ([torch.empty(cap_records * rb, dtype=torch.uint8, device="cuda") for _ in range(count)],
            [torch.empty(cap_records, dtype=torch.int64, device="cuda") for _ in range(count)])


@pytest.mark.parametrize("case", CB_CASES, ids=[c[0] for c in CB_CASES])
def test_count_based_window_hops(wfb, oracle, ordered, case):
    """Ffat_Windows_GPU with an order-sensitive combine, every call (and a pipelined handle's flush) on the next stream: the windows
    are the oracle's, their values the direct fold of every key's items."""
    import torch
    ops, O = wfb, oracle
    name, win, slide, nb, cap, dense, grow, pipelined, spec = case
    t, calls = _cb_stream(spec, cap, dense, seed=len(name))
    c = types.SimpleNamespace(win=win, slide=slide, nb=nb, rec=32)
    e, et, h, q, _ = ow._expected(O, c, t, calls)
    ff = ops.FfatWindowsGPU(ordered, win, slide, nb, max_keys=cap, dense_keys=dense, pipelined=pipelined, grow_keys=grow)
    prm = C.c_uint64(ow.M)
    ops.check(ff.L.wfb_ffat_set_params(ff.h, C.byref(prm), C.sizeof(prm)), "wfb_ffat_set_params")
    ins = [[ops.DeviceBatch.from_host(tb, ts) for tb, ts in call] for call in calls]
    nkeys = max(nk for _, nk in spec)
    rcap = (max(n for n, _ in spec) // (slide * nb) + nkeys + 1) * nb * 2
    ncalls = len(calls) + (1 if pipelined else 0)
    outs, outs_ts = _window_buffers(ops, ff, rcap, ncalls)
    n_out = torch.full((ncalls,), -1, dtype=torch.int32, device="cuda")
    seg = [(f"process {i}", lambda s, i=i: ff.process(ins[i], out=outs[i], out_ts=outs_ts[i], n_out=n_out[i:i + 1], stream=s))
           for i in range(len(calls))]
    if pipelined:
        k = len(calls)
        seg.append(("flush", lambda s: ff.flush(out=outs[k], out_ts=outs_ts[k], n_out=n_out[k:k + 1], stream=s)))
    torch.cuda.synchronize()
    hops = Hops()
    hops.run(seg)
    torch.cuda.synchronize()
    no = n_out.cpu().numpy()
    assert np.all((no >= 0) & (no <= rcap)), no
    got = np.concatenate([ops.to_host(o, ff.res_dtype)[:k] for o, k in zip(outs, no)])
    gts = np.concatenate([ops.ts_to_host(o)[:k] for o, k in zip(outs_ts, no)])
    nk, err = ff.stats()
    assert err == 0 and (dense or nk == len(np.unique(t["key"])))  # (a dense-key handle keeps no key count)
    if grow:
        assert ff.key_capacity >= 1000
    ow._check(got, gts, e, et, h, q, 32)
    hops.assert_ordered()


def test_count_based_window_hops_tuple64(wfb, oracle):
    """The built-in program (sums) against O.FfatGpuOracle, calls of growing size on the next stream each."""
    import torch
    ops, O = wfb, oracle
    win, slide, nb, nkeys = 64, 16, 2, 300
    go = O.FfatGpuOracle(win, slide, nb)
    ff = ops.FfatWindowsGPU(ops.PROG_TUPLE64, win, slide, nb, max_keys=1024)
    calls, exp, ets, start = [], [], [], 0
    for n in (1003, 70001, 150001, 150001):
        bs = []
        for b in range(0, n, 25000):
            k = min(25000, n - b)
            t, ts = O.gen_tuple64(start, k, O.KEY_UNIFORM, nkeys)
            start += k
            r, rt = go.process_batch(O.lift_tuple64(t), int(ts[0]))
            exp.append(r); ets.append(rt)
            bs.append(ops.DeviceBatch.from_host(t, ts))
        calls.append(bs)
    rcap = (150001 // (slide * nb) + nkeys + 1) * nb * 2
    outs, outs_ts = _window_buffers(ops, ff, rcap, len(calls))
    n_out = torch.full((len(calls),), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    hops = Hops()
    hops.run([(f"process {i}", lambda s, i=i: ff.process(calls[i], out=outs[i], out_ts=outs_ts[i], n_out=n_out[i:i + 1], stream=s))
              for i in range(len(calls))])
    torch.cuda.synchronize()
    no = n_out.cpu().numpy()
    got, gts = O.sort_results(np.concatenate([ops.to_host(o, ops.RESULT32)[:k] for o, k in zip(outs, no)]),
                              np.concatenate([ops.ts_to_host(o)[:k] for o, k in zip(outs_ts, no)]))
    e, et = O.sort_results(np.concatenate(exp), np.concatenate(ets))
    assert len(got) == len(e) > 0 and ff.stats()[1] == 0
    assert np.array_equal(got["key"], e["key"]) and np.array_equal(got["id"], e["id"]) and np.array_equal(got["isum"], e["isum"])
    assert np.allclose(got["fsum"], e["fsum"], rtol=1e-6, atol=0)
    assert np.array_equal(gts, et)
    hops.assert_ordered()


# ---------------------------------------------------------------------------------------------------------------------------------
# time-based windows
# ---------------------------------------------------------------------------------------------------------------------------------
TB_CASES = [  # name, win, slide, nb, lateness, capacity (dense keys), keys, tuples, batch, batches per call, ts step divisor, jitter
    ("bucket_back_end", 400, 100, 2, 150, 65536, 300, 60000, 2000, 6, 20, 100),
    ("full_sort_back_end", 400, 100, 2, 150, 100000, 20000, 200000, 2000, 10, 250, 100),
]


@pytest.mark.parametrize("case", TB_CASES, ids=[c[0] for c in TB_CASES])
def test_time_based_window_hops(wfb, oracle, ordered, case):
    """Time-based windows with lateness and jittered timestamps, every call on the next stream: the oracle's windows, the direct
    fold's values."""
    import math
    import torch
    ops, O = wfb, oracle
    name, win, slide, nb, late, cap, nkeys, n, batch, group, div, jitter = case
    t, ts = ow._tb_stream(nkeys, n, div, jitter, seed=len(name) + 1)
    to = O.FfatTbOracle(win, slide, late, nb)
    ff = ops.FfatWindowsGPU(ordered, win, slide, nb, max_keys=cap, dense_keys=True, win_type=1, lateness=late)
    prm = C.c_uint64(ow.M)
    ops.check(ff.L.wfb_ffat_set_params(ff.h, C.byref(prm), C.sizeof(prm)), "wfb_ffat_set_params")
    exp, ets, batches = [], [], []
    for b in range(0, n, batch):
        tb, tsb = t[b:b + batch], ts[b:b + batch]
        k = ow.keep_mask(tb)
        r, rt = to.process_batch(ow._lift_res(tb[k]), tsb[k], int(tsb[0]))
        exp.append(r); ets.append(rt)
        batches.append(ops.DeviceBatch.from_host(tb, tsb))
    assert to.ignored == 0
    calls = [batches[i:i + group] for i in range(0, len(batches), group)]
    rcap = (batch * group + 8 * (nkeys + 1)) * nb
    outs, outs_ts = _window_buffers(ops, ff, rcap, len(calls))
    n_out = torch.full((len(calls),), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    hops = Hops()
    hops.run([(f"process {i}", lambda s, i=i: ff.process(calls[i], out=outs[i], out_ts=outs_ts[i], n_out=n_out[i:i + 1], stream=s))
              for i in range(len(calls))])
    torch.cuda.synchronize()
    no = n_out.cpu().numpy()
    assert np.all((no >= 0) & (no <= rcap)), no
    got = np.concatenate([ops.to_host(o, ff.res_dtype)[:k] for o, k in zip(outs, no)])
    gts = np.concatenate([ops.ts_to_host(o)[:k] for o, k in zip(outs_ts, no)])
    assert ff.stats()[1] == 0
    e, et = O.sort_results(np.concatenate(exp), np.concatenate(ets))
    k = ow.keep_mask(t)
    surv, sts = t[k], ts[k]
    order, a, b = ow.tb_ranges(surv["key"], sts, e["key"], e["id"], win, slide, math.gcd(win, slide))
    h, q = ow.hash_ranges(ow.np_lift_h(surv, 32)[order], a, b, np.uint64)
    ow._check(got, gts, e, et, h, q, 32)
    hops.assert_ordered()


# ---------------------------------------------------------------------------------------------------------------------------------
# queries
# ---------------------------------------------------------------------------------------------------------------------------------
def test_queries_see_earlier_calls(wfb, oracle):
    """stats() and results_total() on stream B right after a call on stream A (still asleep when B is queried) report that call's
    keys, error flags and results: for a count-based handle, with an output buffer too small for its results (err bit 1), and for a
    pipelined handle after a flush on A."""
    import torch
    ops, O = wfb, oracle
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    win, slide, nb, per_step = 8, 4, 1, 1000

    def step_batch(j, n=20000):
        t, ts = O.gen_tuple64(j * n, n, O.KEY_UNIFORM, per_step)
        t["key"] += np.uint64(j * per_step)  # new keys in every step
        return t, ts

    def asleep_then(call):
        with torch.cuda.stream(A):
            torch.cuda._sleep(SLEEP_CYCLES)
        call()
        return ff.stats(stream=B), ff.results_total(stream=B)

    # count-based: every step's keys and results, then a step whose results do not fit
    steps = [step_batch(j) for j in range(4)]
    go = O.FfatGpuOracle(win, slide, nb)
    totals = np.cumsum([len(go.process_batch(O.lift_tuple64(t), int(ts[0]))[0]) for t, ts in steps])
    ins = [ops.DeviceBatch.from_host(t, ts) for t, ts in steps]
    ff = ops.FfatWindowsGPU(ops.PROG_TUPLE64, win, slide, nb, max_keys=8192)
    rcap = ff.max_results(20000)
    outs, outs_ts = _window_buffers(ops, ff, rcap, len(steps))
    small, small_ts = _window_buffers(ops, ff, 4, 1)
    n_out = torch.full((len(steps),), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    seen = []
    for j in range(3):
        (nk, ef), tot = asleep_then(lambda: ff.process([ins[j]], out=outs[j], out_ts=outs_ts[j], n_out=n_out[j:j + 1], stream=A))
        seen.append((nk, ef, tot))
    (nk, ef), _ = asleep_then(lambda: ff.process([ins[3]], out=small[0], out_ts=small_ts[0], n_out=n_out[3:4], stream=A))
    seen.append((nk, ef, None))
    torch.cuda.synchronize()
    exp = [(per_step * (j + 1), 0, int(totals[j])) for j in range(3)] + [(per_step * 4, 2, None)]
    assert int(totals[0]) > 0
    assert seen == exp, f"stats / results_total on another stream (got, expected): {list(zip(seen, exp))}"

    # pipelined: two calls (the second delivers the first's results), then a flush on A into a buffer too small for the second's
    ff = ops.FfatWindowsGPU(ops.PROG_TUPLE64, win, slide, nb, max_keys=8192, pipelined=True)
    torch.cuda.synchronize()
    ff.process([ins[0]], out=outs[0], out_ts=outs_ts[0], n_out=n_out[0:1], stream=A)
    ff.process([ins[1]], out=outs[1], out_ts=outs_ts[1], n_out=n_out[1:2], stream=A)
    (nk, ef), tot = asleep_then(lambda: ff.flush(out=small[0], out_ts=small_ts[0], n_out=n_out[2:3], stream=A))
    torch.cuda.synchronize()
    assert (nk, ef, tot) == (2 * per_step, 2, int(totals[1])), "pipelined flush: (keys, err flags, results total) on another stream"
