"""Key tables that grow (WFB_KEYS_GROW): a handle created with a small capacity and the flag gives the same results as a fixed handle
created at the capacity the growing one ended with. Results are compared sorted by (key, id): keys, window ids, integer sums and result
timestamps exactly, floating-point sums within 1e-6 relative; window cases of PROG_TUPLE64 are also compared with the oracle. Covered:
count-based windows across the bucket -> onesweep switch at 65536 keys, keys arriving over many calls, one call that grows several times
and fills the key table, the double and 16-byte key programs (the all-ones 16-byte key still raises bit 0 and grows nothing),
time-based windows, keyed-stateful Map / Filter, the counters and the refusals. The refusals that need no device run without one."""
import ctypes as C

import numpy as np
import pytest

FP_RTOL = 1e-6
WFB_E_BADARG = -1
KEYS_GROW, DENSE, PIPELINED = 4, 1, 2
gpu = pytest.mark.gpu


def _sorted(prog, ops, res, ts):
    """Results (and timestamps) sorted by (key, id); the key as sortable columns."""
    if prog == ops.PROG_TUPLE64_K16:
        order = np.lexsort((res["id"], res["key"]["b"], res["key"]["a"], res["key"]["key"]))
    elif prog == ops.PROG_TUPLE64_FKEY:
        order = np.lexsort((res["id"], res["key"].view(np.uint64)))
    else:
        order = np.lexsort((res["id"], res["key"]))
    return res[order], ts[order]


def _check(prog, ops, got, gts, exp, ets):
    g, gt = _sorted(prog, ops, got, gts)
    e, et = _sorted(prog, ops, exp, ets)
    assert len(g) == len(e) > 0, (len(g), len(e))
    assert g["key"].tobytes() == e["key"].tobytes() and np.array_equal(g["id"], e["id"])
    assert np.array_equal(gt, et)
    assert np.array_equal(g["isum"], e["isum"])
    assert np.allclose(g["fsum"], e["fsum"], rtol=FP_RTOL, atol=0)


def _key_table(prog, nkeys):
    """pad[0] of key index 0 .. nkeys-1: a distinct double (FKEY), a high word (K16)."""
    import torch
    if prog == 4:  # PROG_TUPLE64_FKEY
        vals = np.arange(nkeys) * 0.25 - 1000.75
    else:
        vals = np.random.default_rng(5).integers(1, 1 << 62, nkeys, dtype=np.int64)
    return torch.from_numpy(np.ascontiguousarray(vals).view(np.int64).copy()).cuda()


def _segment(ops, prog, start, n, limit, table):
    """n device tuples of the bench stream from index `start` (watermark = start), key index = uniform key % limit; the program's key
    derived from the key index."""
    import torch
    b = ops.gen_tuple64(start, n, ops.KEY_UNIFORM, 1 << 20)
    v = b.tuples.view(torch.int64).view(-1, 8)
    v[:, 0] %= limit
    if table is not None:
        v[:, 4] = table[v[:, 0]]
    return b


def _pow2(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def _grown(cap, keys_per_call, ceiling=65536):
    """Capacity of a growing handle after calls that bring it to keys_per_call[i] distinct keys: a pass inserts keys until the key table
    (a power of two >= 2 * capacity entries) is full, then the capacity becomes a power of two >= 2 * max(keys inserted, capacity), but
    only the ceiling (65536: the bucket path, the limit of time-based and keyed-stateful handles) when it is below it and they fit it."""
    for keys in keys_per_call:
        while keys > cap:
            n = min(keys, _pow2(2 * cap))
            new = _pow2(2 * max(n, cap))
            cap = ceiling if new > ceiling and cap < ceiling and n <= ceiling else new
    return cap


def _run_cb(ops, prog, calls, max_keys, grow, win, slide, nb, pre):
    """Count-based windows over the calls (each a list of DeviceBatch); returns the results, their timestamps and the handle."""
    import torch
    ff = ops.FfatWindowsGPU(prog, win, slide, nb, max_keys=max_keys, grow_keys=grow)
    got, gts = [], []
    for batches in calls:
        out, out_ts, n_out = ff.process(batches, pre=pre)
        torch.cuda.synchronize()
        g, gt = ff.results_to_host(out, out_ts, n_out)
        got.append(g); gts.append(gt)
    return np.concatenate(got), np.concatenate(gts), ff


def _oracle_cb(O, calls, win, slide, nb, f):
    go = O.FfatGpuOracle(win, slide, nb)
    exp, ets = [], []
    for batches in calls:
        for b in batches:
            t = b.tuples.cpu().numpy().view(O.TUPLE64)[:b.n]
            ts = b.ts.cpu().numpy().view(np.uint64)[:b.n]
            surv, _, _ = O.map_filter_tuple64(t, ts, f.map_kind, f.map_iadd, f.map_fscale, f.filt_kind, f.filt_mod)
            r, rts = go.process_batch(O.lift_tuple64(surv), b.watermark)
            exp.append(r); ets.append(rts)
    return np.concatenate(exp), np.concatenate(ets)


def _cb_case(ops, O, prog, calls, init_keys, win, slide, nb, f):
    got, gts, ffg = _run_cb(ops, prog, calls, init_keys, True, win, slide, nb, f)
    cap = ffg.key_capacity
    exp, ets, fff = _run_cb(ops, prog, calls, cap, False, win, slide, nb, f)
    assert ffg.stats() == fff.stats() and ffg.stats()[1] == 0
    assert ffg.results_total() == fff.results_total() == len(got)
    _check(prog, ops, got, gts, exp, ets)
    if prog == ops.PROG_TUPLE64:
        oe, oet = _oracle_cb(O, calls, win, slide, nb, f)
        _check(prog, ops, got, gts, oe, oet)
    return ffg


@gpu
def test_cb_grows_across_the_bucket_limit(wfb, oracle):
    """70 000 uniform keys from a capacity of 16: the keys arrive over five calls, so the handle leaves the bucket path (at most 65536
    keys) in the middle of the stream, with every older key's windows open."""
    ops = wfb
    f = ops.functors(map_kind=1, iadd=3, fscale=1.5, filt_kind=2, mod=3)
    n = 1 << 20
    limits = [16, 5000, 40000, 70000, 70000, 70000]
    calls = [[_segment(ops, ops.PROG_TUPLE64, c * n, n, lim, None)] for c, lim in enumerate(limits)]
    ffg = _cb_case(ops, oracle, ops.PROG_TUPLE64, calls, 16, 16, 4, 3, f)
    assert ffg.key_capacity == _grown(16, limits) == 262144 and ffg.stats()[0] == 70000


@gpu
@pytest.mark.parametrize("prog", [0, 4, 5], ids=["u64", "f64", "k16"])
def test_cb_new_keys_over_many_calls(wfb, oracle, prog):
    """New keys arrive call after call (two batches each) while the windows of the older keys straddle every growth."""
    ops = wfb
    f = ops.functors(map_kind=1, iadd=2, fscale=1.25, filt_kind=1)
    table = None if prog == ops.PROG_TUPLE64 else _key_table(prog, 3000)
    n, limits = 20000, [min(3000, 16 + 100 * c) for c in range(30)]
    calls = [[_segment(ops, prog, (2 * c + h) * n, n, lim, table) for h in range(2)] for c, lim in enumerate(limits)]
    ffg = _cb_case(ops, oracle, prog, calls, 8, 64, 16, 3, f)
    assert ffg.stats()[0] == limits[-1] and ffg.key_capacity == _grown(8, limits)


@gpu
@pytest.mark.parametrize("prog", [0, 4, 5], ids=["u64", "f64", "k16"])
def test_cb_one_call_grows_several_times(wfb, oracle, prog):
    """One call brings 5000 new keys into a 16-key handle: the 32-entry key table fills, and the call grows 16 -> 64 -> 256 -> 1024 ->
    4096 -> 16384 before its pass takes every key."""
    ops = wfb
    f = ops.functors()
    table = None if prog == ops.PROG_TUPLE64 else _key_table(prog, 5000)
    calls = [[_segment(ops, prog, c * 400000, 400000, 5000, table)] for c in range(2)]
    ffg = _cb_case(ops, oracle, prog, calls, 16, 32, 8, 2, f)
    assert ffg.key_capacity == _grown(16, [5000]) == 16384 and ffg.stats()[0] == 5000


@gpu
@pytest.mark.parametrize("prog", [0, 5], ids=["u64", "k16"])
def test_cb_all_ones_key_grows_nothing(wfb, prog):
    """The all-ones key (8 or 16 bytes) marks a free entry: on a growing handle it raises bit 0, the other keys' windows are those of a
    stream without it, and the capacity is what those keys need."""
    import torch
    ops = wfb
    table = None if prog == ops.PROG_TUPLE64 else _key_table(prog, 100)
    b = _segment(ops, prog, 0, 200000, 100, table)
    v = b.tuples.view(torch.int64).view(-1, 8)
    bad = (torch.arange(200000, device="cuda") % 7) == 0
    v[bad, 0] = -1
    if table is not None:
        v[bad, 4] = -1
    clean = b.tuples.view(torch.int64).view(-1, 8)[~bad].contiguous().view(torch.uint8).view(-1)
    nclean = int((~bad).sum())
    cb = ops.DeviceBatch(clean, b.ts[~bad].contiguous(), nclean, 0)
    got, gts, ffg = _run_cb(ops, prog, [[b]], 4, True, 32, 8, 2, None)
    exp, ets, fff = _run_cb(ops, prog, [[cb]], 4, True, 32, 8, 2, None)
    assert ffg.stats() == (100, 1) and fff.stats() == (100, 0)
    assert ffg.key_capacity == fff.key_capacity == 256
    _check(prog, ops, got, gts, exp, ets)


TB_CASES = [(40, 10, 0, 3, "mono"), (64, 16, 100, 2, "jitter")]


@gpu
@pytest.mark.parametrize("case", TB_CASES, ids=[f"w{c[0]}_s{c[1]}_l{c[2]}_{c[4]}" for c in TB_CASES])
def test_tb_grows_across_batches(wfb, oracle, case):
    import torch
    O, ops = oracle, wfb
    win, slide, lateness, nb, mode = case
    n, batch = 9000, 300
    t, _ = O.gen_tuple64(11, n, O.KEY_RR, 1 << 20)
    for i, b in enumerate(range(0, n, batch)):
        t["key"][b:b + batch] %= min(100, 3 + 4 * i)  # new keys batch after batch (a new key fires every group since time 0)
    rng = np.random.default_rng(11)
    ts = np.arange(n, dtype=np.int64) * 3
    if mode == "jitter":
        ts = ts + rng.integers(-40, 41, n)
    ts = np.maximum(ts, 0).astype(np.uint64)

    def run(max_keys, grow):
        ff = ops.FfatWindowsGPU(ops.PROG_TUPLE64, win, slide, nb, max_keys=max_keys, win_type=1, lateness=lateness, grow_keys=grow)
        got, gts = [], []
        for b in range(0, n, batch):
            tb_, tsb = t[b:b + batch], ts[b:b + batch]
            wm = int(tsb.min()) if mode == "jitter" else int(tsb[0])
            out, out_ts, n_out = ff.process([ops.DeviceBatch.from_host(tb_, tsb, watermark=wm)])
            torch.cuda.synchronize()
            g_, gt_ = ff.results_to_host(out, out_ts, n_out)
            got.append(g_); gts.append(gt_)
        return np.concatenate(got), np.concatenate(gts), ff

    got, gts, ffg = run(4, True)
    cap = _grown(4, [min(100, 3 + 4 * i) for i in range(n // batch)])
    assert ffg.key_capacity == cap and ffg.stats() == (100, 0)
    exp, ets, fff = run(cap, False)
    assert fff.stats() == (100, 0) and ffg.results_total() == fff.results_total() == len(got)
    _check(ops.PROG_TUPLE64, ops, got, gts, exp, ets)
    tbo = O.FfatTbOracle(win, slide, lateness, nb)
    oe, oet = [], []
    for b in range(0, n, batch):
        tsb = ts[b:b + batch]
        r, rt = tbo.process_batch(O.lift_tuple64(t[b:b + batch]), tsb, int(tsb.min()) if mode == "jitter" else int(tsb[0]))
        oe.append(r); oet.append(rt)
    _check(ops.PROG_TUPLE64, ops, got, gts, np.concatenate(oe), np.concatenate(oet))


@gpu
@pytest.mark.parametrize("prog", [0, 5], ids=["u64", "k16"])
@pytest.mark.parametrize("op", ["map", "filter"])
def test_stateful_grows_and_keeps_state(wfb, prog, op):
    """Keyed-stateful Map / Filter: a growing handle (capacity 16) and a fixed one give the same tuples call after call, so the state of
    every key from before a growth survives it."""
    import torch
    ops = wfb
    f = ops.functors(map_kind=1, filt_kind=1)
    table = None if prog == ops.PROG_TUPLE64 else _key_table(prog, 4000)
    calls = [([5000, 3, 1025], 40), ([65536], 1000), ([100] * 5, 1200), ([30000, 30000], 4000), ([7000], 4000)]
    cap = _grown(16, [lim for _, lim in calls])
    ksg = ops.KeyedState(prog, max_keys=16, grow_keys=True)
    ksf = ops.KeyedState(prog, max_keys=cap)
    start = 0
    for sizes, lim in calls:
        res = []
        for ks in (ksg, ksf):
            ins, outs, s0 = [], [], start
            for n in sizes:
                b = _segment(ops, prog, s0, n, lim, table)
                s0 += n
                ins.append(b)
                outs.append(ops.DeviceBatch(torch.empty_like(b.tuples), torch.empty_like(b.ts), n, 0))
            if op == "map":
                ks.map(ins, f)
                torch.cuda.synchronize()
                res.append([ops.to_host(b.tuples, ops.TUPLE64)["ivalue"].copy() for b in ins])
            else:
                n_out = torch.zeros(len(ins), dtype=torch.int32, device="cuda")
                ks.filter(ins, f, outs, n_out)
                torch.cuda.synchronize()
                no = n_out.cpu().numpy()
                res.append([(int(no[i]), ops.to_host(outs[i].tuples, ops.TUPLE64)["ivalue"][:no[i]].copy(), ops.ts_to_host(outs[i].ts)[:no[i]].copy())
                            for i in range(len(ins))])
        start += sum(sizes)
        for a, b in zip(res[0], res[1]):
            if op == "map":
                assert np.array_equal(a, b)
            else:
                assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert ksg.key_capacity == ksf.key_capacity == cap


@gpu
def test_key_shard_refused_on_growing_handle(wfb):
    ff = wfb.FfatWindowsGPU(wfb.PROG_TUPLE64, 16, 4, 1, max_keys=64, grow_keys=True)
    assert ff.L.wfb_ffat_set_key_shard(ff.h, 2, 0) == WFB_E_BADARG
    assert ff.key_capacity == 64


def test_growth_refusals():
    """Growth with dense keys or with pipelining is refused before any device work (so this runs without a GPU as well)."""
    from windflow_b200 import build, _lib
    build.build()
    L = _lib.lib()
    h = C.c_void_p()
    for win_type in (0, 1):
        assert L.wfb_ffat_create(C.byref(h), 0, 16, 4, 1, 64, win_type, 0, KEYS_GROW | DENSE) == WFB_E_BADARG
        assert L.wfb_ffat_create(C.byref(h), 0, 16, 4, 1, 64, win_type, 0, KEYS_GROW | PIPELINED) == WFB_E_BADARG
    assert L.wfb_kstate_create(C.byref(h), 0, 64, KEYS_GROW | DENSE) == WFB_E_BADARG
    assert L.wfb_ffat_key_capacity(None) == 0 and L.wfb_kstate_key_capacity(None) == 0


CEILING_LIMITS = [1000, 1001, 2049, 8193, 32769, 40000]  # 1000 -> 2048 -> 8192 -> 32768, then 65536 rather than 131072


@gpu
@pytest.mark.parametrize("kind", ["cb", "tb", "stateful"])
def test_growth_stops_at_65536_on_the_way_past_32768(wfb, oracle, kind):
    """A handle created at 1000 keys whose keys arrive so that it reaches 32768: key 32769 takes it to 65536 (the limit of time-based
    and keyed-stateful handles, the last capacity of the bucket path), not to 131072. Compared with a fixed handle at 65536 keys."""
    import torch
    O, ops = oracle, wfb
    n = 1 << 16
    cap = _grown(1000, CEILING_LIMITS)
    assert cap == 65536
    if kind == "cb":  # round-robin keys: every key of the call's range in every call (no filter: every tuple reaches the key table)
        f = ops.functors(map_kind=1, iadd=3, fscale=1.5)
        calls = [[ops.gen_tuple64(c * n, n, ops.KEY_RR, lim)] for c, lim in enumerate(CEILING_LIMITS)]
        ffg = _cb_case(ops, O, ops.PROG_TUPLE64, calls, 1000, 16, 4, 3, f)
        assert ffg.key_capacity == cap and ffg.stats() == (40000, 0)
    elif kind == "tb":
        win = 1 << 17  # tumbling windows of two batches: a key fires a few windows per batch at most

        def run(max_keys, grow):
            ff = ops.FfatWindowsGPU(ops.PROG_TUPLE64, win, win, 1, max_keys=max_keys, win_type=1, grow_keys=grow)
            got, gts = [], []
            for c, lim in enumerate(CEILING_LIMITS):
                t, _ = O.gen_tuple64(c * n, n, O.KEY_RR, lim)
                ts = np.arange(c * n, (c + 1) * n, dtype=np.uint64)
                out, out_ts, n_out = ff.process([ops.DeviceBatch.from_host(t, ts, watermark=c * n)])
                torch.cuda.synchronize()
                g_, gt_ = ff.results_to_host(out, out_ts, n_out)
                got.append(g_); gts.append(gt_)
            return np.concatenate(got), np.concatenate(gts), ff

        got, gts, ffg = run(1000, True)
        assert ffg.key_capacity == cap and ffg.stats() == (40000, 0)
        exp, ets, fff = run(cap, False)
        assert ffg.results_total() == fff.results_total() == len(got)
        _check(ops.PROG_TUPLE64, ops, got, gts, exp, ets)
        tbo = O.FfatTbOracle(win, win, 0, 1)
        oe, oet = [], []
        for c, lim in enumerate(CEILING_LIMITS):
            t, _ = O.gen_tuple64(c * n, n, O.KEY_RR, lim)
            r, rt = tbo.process_batch(O.lift_tuple64(t), np.arange(c * n, (c + 1) * n, dtype=np.uint64), c * n)
            oe.append(r); oet.append(rt)
        _check(ops.PROG_TUPLE64, ops, got, gts, np.concatenate(oe), np.concatenate(oet))
    else:
        f = ops.functors(map_kind=1, filt_kind=1)
        ksg = ops.KeyedState(ops.PROG_TUPLE64, max_keys=1000, grow_keys=True)
        ksf = ops.KeyedState(ops.PROG_TUPLE64, max_keys=cap)
        for c, lim in enumerate(CEILING_LIMITS):
            res = []
            for ks in (ksg, ksf):
                b = ops.gen_tuple64(c * n, n, ops.KEY_RR, lim)
                ks.map([b], f)
                torch.cuda.synchronize()
                res.append(ops.to_host(b.tuples, ops.TUPLE64)["ivalue"].copy())
            assert np.array_equal(res[0], res[1])
        assert ksg.key_capacity == cap
