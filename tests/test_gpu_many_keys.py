"""More than 65 536 keys in keyed-stateful Map / Filter (the full-sort path: a stable sort of the (slot, position) pairs and one thread
per run of a slot) and in time-based windows (a count-based back end off the bucket path). Keyed-stateful results are compared bit for
bit with the oracle's per-key sequential restatement, with the state carried across calls; windows are compared sorted by (key, id):
keys, ids, integer sums and timestamps exactly, floating-point sums within 1e-6 relative. Also: the same stream through both paths gives
the same bytes, growth from 16 keys past the 65 536 ceiling, a key that finds no slot, and the slot whose low bits equal INVALID_SLOT's.
The refusal above 2^30 keys needs no device."""
import ctypes as C
import functools

import numpy as np
import pytest

gpu = pytest.mark.gpu
FP_RTOL = 1e-6
WFB_E_BADARG, WFB_E_UNSUPPORTED = -1, -5
KEYS_GROW, DENSE = 4, 1

# (program, dense keys): the bench tuple through the hash table, the reference's 16-byte test tuple with dense keys, a 16-byte key
PROGS = [(0, False), (1, True), (5, False)]
PROG_IDS = ["u64", "wftest16_dense", "k16"]
NKEYS = [100000, 1 << 20]
CALLS = ([100000, 1, 0, 30000], [0], [70000, 257, 0, 4096])  # several calls of several batches, empty batches in between


@functools.lru_cache(maxsize=None)
def _cdf(O, nkeys):
    return O.zipf_cdf(nkeys)


@functools.lru_cache(maxsize=None)
def _k16_table(nkeys):
    """pad[0] of key 0 .. nkeys-1 for the 16-byte key program: the key is (key, low and high half of pad[0])."""
    return np.random.default_rng(7).integers(1, 1 << 62, nkeys, dtype=np.int64).view(np.uint64)


def _stream(O, ops, prog, start, n, nkeys, dist):
    """n host tuples of the program from stream index `start`; returns (tuples, ts, the field the stateful functors add to)."""
    t, ts = O.gen_tuple64(start, n, dist, nkeys, cdf=_cdf(O, nkeys) if dist == O.KEY_ZIPF else None)
    if prog == ops.PROG_WFTEST16:
        w = np.zeros(n, dtype=ops.WFTEST16)
        w["key"], w["value"] = t["key"], t["ivalue"]
        return w, ts, "value"
    if prog == ops.PROG_TUPLE64_K16:
        t["pad"][:, 0] = _k16_table(nkeys)[t["key"]]
    return t, ts, "ivalue"


def _dev(ops, arr, ts):
    import torch
    if len(arr):
        return ops.DeviceBatch.from_host(arr, ts)
    return ops.DeviceBatch(torch.empty(0, dtype=torch.uint8, device="cuda"), torch.empty(0, dtype=torch.int64, device="cuda"), 0, 0)


def _map_call(ops, ks, prog, hosts, f):
    """One keyed-stateful Map call over the host batches; returns the tuples as they came back."""
    import torch
    devs = [_dev(ops, a, ts) for a, ts in hosts]
    ks.map(devs, f)
    torch.cuda.synchronize()
    return [ops.to_host(d.tuples, ops.TUPLE_DTYPE[prog])[:d.n].copy() for d in devs]


def _filter_call(ops, ks, prog, hosts, f):
    """One keyed-stateful Filter call; returns (survivors, their ts) per batch."""
    import torch
    ins = [_dev(ops, a, ts) for a, ts in hosts]
    outs = [ops.DeviceBatch(torch.empty_like(b.tuples), torch.empty_like(b.ts), b.n, 0) for b in ins]
    n_out = torch.full((len(ins),), 99, dtype=torch.int32, device="cuda")
    ks.filter(ins, f, outs, n_out)
    torch.cuda.synchronize()
    no = n_out.cpu().numpy()
    return [(ops.to_host(outs[i].tuples, ops.TUPLE_DTYPE[prog])[:no[i]].copy(), ops.ts_to_host(outs[i].ts)[:no[i]].copy()) for i in range(len(ins))]


@gpu
@pytest.mark.parametrize("dist", [1, 2], ids=["uniform", "zipf"])
@pytest.mark.parametrize("nkeys", NKEYS)
@pytest.mark.parametrize("prog,dense", PROGS, ids=PROG_IDS)
@pytest.mark.parametrize("kind", [1, 2])
def test_map_stateful_many_keys(wfb, oracle, prog, dense, nkeys, dist, kind):
    O, ops = oracle, wfb
    ks = ops.KeyedState(prog, max_keys=nkeys, dense_keys=dense)
    f = ops.functors(map_kind=kind)
    state, start = {}, 0
    for sizes in CALLS:
        hosts, field = [], "ivalue"
        for n in sizes:
            a, ts, field = _stream(O, ops, prog, start, n, nkeys, dist)
            start += n
            hosts.append((a, ts))
        got = _map_call(ops, ks, prog, hosts, f)
        for (a, _), g in zip(hosts, got):
            assert g.tobytes() == O.stateful_map(a, field, state, kind).tobytes()
    assert ks.key_capacity == nkeys


@gpu
@pytest.mark.parametrize("dist", [1, 2], ids=["uniform", "zipf"])
@pytest.mark.parametrize("nkeys", NKEYS)
@pytest.mark.parametrize("prog,dense", PROGS, ids=PROG_IDS)
@pytest.mark.parametrize("filt", [(0, 1), (1, 1), (2, 3)], ids=["all", "even", "mod3"])
def test_filter_stateful_many_keys(wfb, oracle, prog, dense, nkeys, dist, filt):
    O, ops = oracle, wfb
    kind, mod = filt
    ks = ops.KeyedState(prog, max_keys=nkeys, dense_keys=dense)
    f = ops.functors(filt_kind=kind, mod=mod)
    state, start = {}, 0
    for sizes in CALLS:
        hosts, field = [], "ivalue"
        for n in sizes:
            a, ts, field = _stream(O, ops, prog, start, n, nkeys, dist)
            start += n
            hosts.append((a, ts))
        got = _filter_call(ops, ks, prog, hosts, f)
        for (a, ts), (g, gts) in zip(hosts, got):
            exp, ets, _ = O.stateful_filter(a, ts, field, state, kind, mod)
            assert len(g) == len(exp) and g.tobytes() == exp.tobytes()
            assert np.array_equal(gts, ets)


@gpu
@pytest.mark.parametrize("op", ["map", "filter"])
def test_full_sort_and_bucket_paths_agree(wfb, oracle, op):
    """Keys below 65 536 through a handle of 2^17 keys (full sort) and one of 65 536 keys (buckets): the same bytes come out."""
    O, ops = oracle, wfb
    prog = ops.PROG_TUPLE64
    f = ops.functors(map_kind=2) if op == "map" else ops.functors(filt_kind=2, mod=3)
    handles = [ops.KeyedState(prog, max_keys=1 << 17), ops.KeyedState(prog, max_keys=1 << 16)]
    start = 0
    for c, sizes in enumerate(([65536, 0, 5000], [200000], [1, 30000, 30000])):
        outs = []
        for ks in handles:
            s0, hosts = start, []
            for n in sizes:
                a, ts, _ = _stream(O, ops, prog, s0, n, 60000, O.KEY_ZIPF if c == 1 else O.KEY_UNIFORM)
                s0 += n
                hosts.append((a, ts))
            if op == "map":
                outs.append(b"".join(g.tobytes() for g in _map_call(ops, ks, prog, hosts, f)))
            else:
                outs.append(b"".join(g.tobytes() + gts.tobytes() for g, gts in _filter_call(ops, ks, prog, hosts, f)))
        start += sum(sizes)
        assert outs[0] == outs[1]


def _pow2(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def _grown(cap, keys_per_call, ceiling=65536):
    """Capacity of a growing handle after calls that bring it to keys_per_call[i] distinct keys: a pass inserts keys until the key table
    (a power of two >= 2 * capacity entries) is full, then the capacity becomes a power of two >= 2 * max(keys inserted, capacity), but
    only the ceiling (65536, the last capacity of the bucket path) when it is below it and they fit it."""
    for keys in keys_per_call:
        while keys > cap:
            n = min(keys, _pow2(2 * cap))
            new = _pow2(2 * max(n, cap))
            cap = ceiling if new > ceiling and cap < ceiling and n <= ceiling else new
    return cap


GROW_LIMITS = [16, 5000, 40000, 70000, 200000, 200000]  # 16 -> 16384 -> 65536 (the ceiling) -> 262144


@gpu
@pytest.mark.parametrize("op", ["map", "filter"])
def test_stateful_grows_past_65536(wfb, oracle, op):
    """A keyed-stateful handle created at 16 keys meets up to 200 000 round-robin keys: it stops at 65 536 (bucket path), then doubles
    onto the full-sort path with every key's state. Its tuples equal a fixed handle's at the final capacity and the oracle's."""
    O, ops = oracle, wfb
    prog, n = ops.PROG_TUPLE64, 1 << 18
    cap = _grown(16, GROW_LIMITS)
    assert cap == 262144
    f = ops.functors(map_kind=2) if op == "map" else ops.functors(filt_kind=1)
    ksg = ops.KeyedState(prog, max_keys=16, grow_keys=True)
    ksf = ops.KeyedState(prog, max_keys=cap)
    state, caps = {}, []
    for c, lim in enumerate(GROW_LIMITS):
        t, ts = O.gen_tuple64(c * n, n, O.KEY_RR, lim)
        hosts = [(t[:n // 2], ts[:n // 2]), (t[n // 2:], ts[n // 2:])]
        if op == "map":
            got = [_map_call(ops, ks, prog, hosts, f) for ks in (ksg, ksf)]
            exp = [O.stateful_map(a, "ivalue", state, 2) for a, _ in hosts]
            for g, x, e in zip(got[0], got[1], exp):
                assert g.tobytes() == x.tobytes() == e.tobytes()
        else:
            got = [_filter_call(ops, ks, prog, hosts, f) for ks in (ksg, ksf)]
            for (a, ts_), (g, gts), (x, xts) in zip(hosts, got[0], got[1]):
                e, ets, _ = O.stateful_filter(a, ts_, "ivalue", state, 1, 1)
                assert g.tobytes() == x.tobytes() == e.tobytes()
                assert np.array_equal(gts, ets) and np.array_equal(xts, ets)
        caps.append(ksg.key_capacity)
    assert caps == [_grown(16, GROW_LIMITS[:i + 1]) for i in range(len(GROW_LIMITS))]
    assert caps[2] == 65536 and ksg.key_capacity == ksf.key_capacity == cap


def _check_windows(ops, got, gts, exp, ets):
    og, oe = np.lexsort((got["id"], got["key"])), np.lexsort((exp["id"], exp["key"]))
    g, gt, e, et = got[og], gts[og], exp[oe], ets[oe]
    assert len(g) == len(e) > 0, (len(g), len(e))
    assert np.array_equal(g["key"], e["key"]) and np.array_equal(g["id"], e["id"])
    assert np.array_equal(gt, et)
    assert np.array_equal(g["isum"], e["isum"])
    assert np.allclose(g["fsum"], e["fsum"], rtol=FP_RTOL, atol=0)


OUT_CAP = 1 << 17  # results one call may deliver here; the batches below are small enough that the oracle's 65 536 per batch suffice too


def _run_tb(ops, batches, win, slide, nb, max_keys, lateness=0, dense=False, grow=False):
    """Time-based windows over the host batches [(tuples, ts, watermark)], one call each; returns the results, their ts, the handle and
    the capacity after every call."""
    import torch
    ff = ops.FfatWindowsGPU(ops.PROG_TUPLE64, win, slide, nb, max_keys=max_keys, dense_keys=dense, win_type=1, lateness=lateness, grow_keys=grow)
    out = torch.empty(OUT_CAP * ops.RESULT32.itemsize, dtype=torch.uint8, device="cuda")
    out_ts = torch.empty(OUT_CAP, dtype=torch.int64, device="cuda")
    n_out = torch.zeros(1, dtype=torch.int32, device="cuda")
    got, gts, caps = [], [], []
    for t, ts, wm in batches:
        ff.process([ops.DeviceBatch.from_host(t, ts, watermark=wm)], out=out, out_ts=out_ts, n_out=n_out)
        n = int(n_out.item())
        assert n < OUT_CAP
        got.append(out[:n * ops.RESULT32.itemsize].cpu().numpy().view(ops.RESULT32).copy())
        gts.append(ops.ts_to_host(out_ts[:n]).copy())
        caps.append(ff.key_capacity)
    assert ff.stats()[1] == 0
    return np.concatenate(got), np.concatenate(gts), ff, caps


def _oracle_tb(O, batches, win, slide, nb, lateness=0):
    tbo = O.FfatTbOracle(win, slide, lateness, nb)
    exp, ets = [], []
    for t, ts, wm in batches:
        r, rt = tbo.process_batch(O.lift_tuple64(t), ts, wm)
        exp.append(r); ets.append(rt)
    return np.concatenate(exp), np.concatenate(ets)


TB_VARIANTS = [("monotone", 0, False), ("jitter", 500, False), ("dense", 0, True)]


@gpu
@pytest.mark.parametrize("variant", TB_VARIANTS, ids=[v[0] for v in TB_VARIANTS])
def test_tb_windows_100000_keys(wfb, oracle, variant):
    """Time-based windows over 100 000 uniform keys (the back end on the full-sort path), against the oracle: timestamps in order, jittered
    with lateness (watermark = the batch's smallest timestamp), and a dense-key handle."""
    O, ops = oracle, wfb
    mode, lateness, dense = variant
    nkeys, n, batch = 100000, 400000, 2000  # (a batch fires at most ~2000 keys x 5 groups x Nb windows)
    win, slide, nb = 80000, 20000, 3
    t, _ = O.gen_tuple64(0, n, O.KEY_UNIFORM, nkeys)
    ts = np.arange(n, dtype=np.int64)
    if mode == "jitter":
        ts = ts + np.random.default_rng(3).integers(-400, 401, n)
    ts = np.maximum(ts, 0).astype(np.uint64)
    batches = [(t[b:b + batch], ts[b:b + batch], int(ts[b:b + batch].min())) for b in range(0, n, batch)]
    got, gts, ff, _ = _run_tb(ops, batches, win, slide, nb, nkeys, lateness, dense)
    assert ff.key_capacity == nkeys
    exp, ets = _oracle_tb(O, batches, win, slide, nb, lateness)
    _check_windows(ops, got, gts, exp, ets)


@gpu
def test_tb_grows_past_65536(wfb, oracle):
    """A time-based handle created at 16 keys meets up to 200 000 round-robin keys, stretch after stretch of the stream: 65 536, then
    262 144. Its back end was created on the bucket path with lazy FlatFAT levels (win 4 panes, slide 1 pane, Nb 2: 16 leaves, built on
    chip per fired group), has fired windows there, and keeps that layout on the full-sort path. Results equal a fixed handle created at
    262 144 keys (eager levels) and the oracle."""
    O, ops = oracle, wfb
    n, pane, batch = 1 << 18, 1 << 16, 2048  # (a batch fires at most 2048 keys x 6 groups x Nb windows)
    win, slide, nb = 4 * pane, pane, 2
    batches, seen, known = [], [], np.zeros(max(GROW_LIMITS), dtype=bool)
    for c, lim in enumerate(GROW_LIMITS):
        t, _ = O.gen_tuple64(c * n, n, O.KEY_RR, lim)
        ts = np.arange(c * n, (c + 1) * n, dtype=np.uint64)
        for b in range(0, n, batch):
            batches.append((t[b:b + batch], ts[b:b + batch], int(ts[b])))
            known[t["key"][b:b + batch]] = True
            seen.append(int(known.sum()))  # distinct keys so far
    got, gts, ffg, caps = _run_tb(ops, batches, win, slide, nb, 16, grow=True)
    assert caps == [_grown(16, seen[:i + 1]) for i in range(len(seen))] and 65536 in caps and caps[-1] == 262144
    assert ffg.stats() == (200000, 0)
    exp, ets, fff, _ = _run_tb(ops, batches, win, slide, nb, caps[-1])
    assert fff.stats() == (200000, 0) and ffg.results_total() == fff.results_total() == len(got)
    _check_windows(ops, got, gts, exp, ets)
    oe, oet = _oracle_tb(O, batches, win, slide, nb)
    _check_windows(ops, got, gts, oe, oet)


@gpu
def test_key_without_slot_is_left_alone(wfb, oracle):
    """A fixed handle of 2^17 keys meets 2^17 + 1 round-robin keys: one key finds no slot, and its tuples come back unchanged from the
    map, call after call; every other key's tuples and state are the oracle's (as on the bucket path)."""
    O, ops = oracle, wfb
    prog, keys = ops.PROG_TUPLE64, (1 << 17) + 1
    ks = ops.KeyedState(prog, max_keys=1 << 17)
    f = ops.functors(map_kind=1)
    state, lost = {}, None
    for c in range(3):
        t, ts = O.gen_tuple64(c * 2 * keys, 2 * keys, O.KEY_RR, keys)
        (g,) = _map_call(ops, ks, prog, [(t, ts)], f)
        same = np.unique(t["key"][g["ivalue"] == t["ivalue"]])
        assert len(same) == 1 and (lost is None or same[0] == lost), same[:8]
        lost = same[0]
        mine = t["key"] == lost
        assert g[mine].tobytes() == t[mine].tobytes()
        assert g[~mine].tobytes() == O.stateful_map(t[~mine], "ivalue", state, 1).tobytes()


@gpu
def test_slot_with_invalid_low_bits(wfb, oracle):
    """Dense keys at 2^24 keys: slot 2^24 - 1 has the low 24 bits of INVALID_SLOT. The sort takes 4 passes there, so that key's run and the
    items of keys without a slot (2^24 and above) do not mix: the last slot's tuples are the oracle's, the others' are unchanged."""
    O, ops = oracle, wfb
    top = 1 << 24
    ks = ops.KeyedState(ops.PROG_WFTEST16, max_keys=top, dense_keys=True)
    f = ops.functors(map_kind=1)
    keyset = np.array([top - 1, top, 3, top - 1, top + 7, top - 2, top - 1, top], dtype=np.uint64)
    state = {}
    for c in range(2):
        w = np.zeros(40000, dtype=ops.WFTEST16)
        w["key"] = np.resize(keyset, len(w))
        w["value"] = np.arange(len(w)) + c * 1000000
        (g,) = _map_call(ops, ks, ops.PROG_WFTEST16, [(w, np.arange(len(w), dtype=np.uint64))], f)
        valid = w["key"] < top
        assert g[~valid].tobytes() == w[~valid].tobytes()
        assert g[valid].tobytes() == O.stateful_map(w[valid], "value", state, 1).tobytes()


def test_kstate_refusals():
    """More than 2^30 keys, and growth with dense keys, are refused before any device work (so this runs without a GPU as well)."""
    from windflow_b200 import build, _lib
    build.build()
    L = _lib.lib()
    h = C.c_void_p()
    for mk in ((1 << 30) + 1, 0xffffffff):
        for flags in (0, DENSE, KEYS_GROW):
            assert L.wfb_kstate_create(C.byref(h), 0, mk, flags) == WFB_E_UNSUPPORTED
    assert L.wfb_kstate_create(C.byref(h), 0, 1 << 20, KEYS_GROW | DENSE) == WFB_E_BADARG
    assert L.wfb_kstate_create(C.byref(h), 0, 1 << 30, KEYS_GROW | DENSE) == WFB_E_BADARG
