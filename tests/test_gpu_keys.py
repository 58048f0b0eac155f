"""GPU tests (-m gpu): the built-in programs keyed by a double (PROG_TUPLE64_FKEY, the bits of pad[0]) and by a 16-byte struct
(PROG_TUPLE64_K16, {key, pad[0]}). Renaming equivalence: every distinct key is renamed to a dense integer on the host and the
renamed stream goes through PROG_TUPLE64 (and the oracle for count-based windows); after mapping the keys back, keys, window ids,
integer sums and result timestamps match exactly, floating-point sums within 1e-6 relative. Also: the capacity error flag, the
order of Reduce_GPU's output and the refusals of the integer-only features."""
import ctypes as C

import numpy as np
import pytest

from windflow_b200.ops import PROG_TUPLE64_FKEY, PROG_TUPLE64_K16

pytestmark = pytest.mark.gpu
FP_RTOL = 1e-6
NAN_BITS = 0x7FF8000000000000
ALL_ONES = np.uint64(0xFFFFFFFFFFFFFFFF)


def _canon_f64(bits):
    """Host restatement of the double key codec: -0.0 -> +0.0, every NaN -> one quiet NaN, then the order-preserving transform."""
    bits = np.asarray(bits, dtype=np.uint64)
    x = bits.view(np.float64)
    bits = np.where(np.isnan(x), np.uint64(NAN_BITS), np.where(x == 0, np.uint64(0), bits))
    neg = (bits >> np.uint64(63)) != 0
    return np.where(neg, ~bits, bits | np.uint64(1 << 63))


def _rank(prog, ops, t):
    """Dense id of every tuple's key, in the key order Reduce_GPU emits (numeric for doubles, 128-bit little-endian for K16)."""
    if prog == ops.PROG_TUPLE64_FKEY:
        _, inv = np.unique(_canon_f64(t["pad"][:, 0]), return_inverse=True)
    else:
        _, inv = np.unique(np.stack([t["pad"][:, 0], t["key"]], axis=1), axis=0, return_inverse=True)
    return inv.reshape(-1).astype(np.uint64)


def _result_rank(prog, ops, res, t):
    """Dense id of every result's key, with the ranks of the stream `t`."""
    if prog == ops.PROG_TUPLE64_FKEY:
        u = np.unique(_canon_f64(t["pad"][:, 0]))
        r = np.searchsorted(u, _canon_f64(res["key"].view(np.uint64)))
        assert np.array_equal(u[r], _canon_f64(res["key"].view(np.uint64)))
    else:
        u = np.unique(np.stack([t["pad"][:, 0], t["key"]], axis=1), axis=0)
        hi = res["key"]["a"].astype(np.uint64) | (res["key"]["b"].astype(np.uint64) << np.uint64(32))
        packed = np.stack([hi, res["key"]["key"]], axis=1)
        lookup = {(int(a), int(b)): i for i, (a, b) in enumerate(u)}
        r = np.array([lookup[(int(a), int(b))] for a, b in packed], dtype=np.int64)
    return r.astype(np.uint64)


def _keys(prog, nkeys, seed):
    """Key values of key index 0 .. nkeys-1 (pad[0] for both programs): doubles with fractional parts, negatives, -0.0 and +0.0 and
    NaNs of several payloads; for K16 the high words, with key index pairs sharing the low word."""
    rng = np.random.default_rng(seed)
    if prog == PROG_TUPLE64_FKEY:
        base = (np.arange(nkeys) // 2) * 0.5 + np.where(np.arange(nkeys) % 2 == 0, 1.25, 1.75)
        vals = np.where(rng.random(nkeys) < 0.5, -base, base)
        if nkeys >= 8:
            vals[:4] = [0.0, -0.0, np.nan, -np.nan]
        bits = vals.astype(np.float64).view(np.uint64).copy()
        if nkeys >= 8:
            bits[4] = np.uint64(0x7FF0000000000123)  # another NaN payload: still one key
        return bits
    hi = rng.integers(0, 1 << 63, nkeys, dtype=np.uint64) | np.uint64(1)
    if nkeys >= 8:
        hi[6] = ALL_ONES  # a key whose high half is all ones (the empty marker of one half of a table entry)
    return hi


def _stream(O, prog, n, nkeys, seed, mode=None):
    """Tuples whose key index is t["key"] (uniform) -> program keys (one key table for every stream of nkeys keys); K16 folds key
    indexes pairwise onto one low word."""
    t, ts = O.gen_tuple64(seed, n, O.KEY_UNIFORM if mode is None else mode, nkeys)
    idx = t["key"].copy()
    t["pad"][:, 0] = _keys(prog, nkeys, 0)[idx]
    if prog == PROG_TUPLE64_K16:
        t["key"] = idx // np.uint64(2)  # equal low words that differ only in the high word
        if nkeys >= 10:
            t["key"][(idx == 8) | (idx == 9)] = ALL_ONES  # two keys whose low half is all ones
    return t, ts


def _renamed(ops, prog, t):
    r = t.copy()
    r["key"] = _rank(prog, ops, t)
    return r


def _check_windows(got, gts, exp, ets):
    assert len(got) == len(exp) > 0, (len(got), len(exp))
    assert np.array_equal(got["key"], exp["key"]) and np.array_equal(got["id"], exp["id"])
    assert np.array_equal(gts, ets)
    assert np.array_equal(got["isum"], exp["isum"])
    assert np.allclose(got["fsum"], exp["fsum"], rtol=FP_RTOL, atol=0)


def _run_ffat(ops, prog, t, ts, win, slide, nb, max_keys, batch, win_type=0, lateness=0, wm_fn=None, pre=None):
    import torch
    ff = ops.FfatWindowsGPU(prog, win, slide, nb, max_keys=max_keys, win_type=win_type, lateness=lateness)
    got, gts = [], []
    for b in range(0, len(t), batch):
        tb_, tsb = t[b:b + batch], ts[b:b + batch]
        wm = wm_fn(tsb) if wm_fn else int(tsb[0])
        out, out_ts, n_out = ff.process([ops.DeviceBatch.from_host(tb_, tsb, watermark=wm)], pre=pre)
        torch.cuda.synchronize()
        g, gt = ff.results_to_host(out, out_ts, n_out)
        got.append(g); gts.append(gt)
    flags = ff.stats()[1]
    return np.concatenate(got), np.concatenate(gts), flags


def _as_result32(ops, prog, res, t):
    r = np.zeros(len(res), dtype=ops.RESULT32)
    r["key"] = _result_rank(prog, ops, res, t)
    r["id"], r["isum"], r["fsum"] = res["id"], res["isum"], res["fsum"]
    return r


PROGS = [PROG_TUPLE64_FKEY, PROG_TUPLE64_K16]
CB_CASES = [(16, 4, 2, 40, 20000, 3000), (64, 16, 3, 300, 150000, 8192), (10, 3, 1, 7, 4000, 1000)]


@pytest.mark.parametrize("prog", PROGS, ids=["f64", "k16"])
@pytest.mark.parametrize("case", CB_CASES, ids=[f"w{c[0]}_s{c[1]}_nb{c[2]}_k{c[3]}" for c in CB_CASES])
def test_cb_windows_rename_equivalence(wfb, oracle, prog, case):
    O, ops = oracle, wfb
    win, slide, nb, nkeys, n, batch = case
    t, ts = _stream(O, prog, n, nkeys, 7)
    f = ops.functors(map_kind=1, iadd=3, fscale=1.5, filt_kind=2, mod=3)
    got, gts, fl = _run_ffat(ops, prog, t, ts, win, slide, nb, nkeys, batch, pre=f)
    rt = _renamed(ops, prog, t)
    exp, ets, fl2 = _run_ffat(ops, ops.PROG_TUPLE64, rt, ts, win, slide, nb, nkeys, batch, pre=f)
    assert fl == fl2 == 0
    g, gt = O.sort_results(_as_result32(ops, prog, got, t), gts)
    e, et = O.sort_results(exp, ets)
    _check_windows(g, gt, e, et)
    # the oracle on the renamed stream
    go = O.FfatGpuOracle(win, slide, nb)
    oexp, oets = [], []
    for b in range(0, n, batch):
        surv, _, _ = O.map_filter_tuple64(rt[b:b + batch], ts[b:b + batch], 1, 3, 1.5, 2, 3)
        r, rts = go.process_batch(O.lift_tuple64(surv), int(ts[b]))
        oexp.append(r); oets.append(rts)
    oe, oet = O.sort_results(np.concatenate(oexp), np.concatenate(oets))
    _check_windows(g, gt, oe, oet)


@pytest.mark.parametrize("prog", PROGS, ids=["f64", "k16"])
def test_cb_windows_bench_geometry(wfb, prog):
    """4096 / 64 / Nb 65 with 2000 keys, on the device: the K16 / double program and PROG_TUPLE64 over the same tuples (key index in
    `key`, the program's key derived from it one to one), so the renaming is the key table itself."""
    import torch
    ops = wfb
    nkeys, per_call, calls = 2000, 1 << 21, 12
    win, slide, nb = 4096, 64, 65
    table = torch.from_numpy(_keys(prog, nkeys, 3).view(np.int64).copy()).cuda()
    if prog == PROG_TUPLE64_FKEY:
        table = torch.from_numpy((np.arange(nkeys) * 0.5 - 400.25).view(np.int64).copy()).cuda()  # distinct, negative and fractional
    ff_new = ops.FfatWindowsGPU(prog, win, slide, nb, max_keys=nkeys)
    ff_ref = ops.FfatWindowsGPU(ops.PROG_TUPLE64, win, slide, nb, max_keys=nkeys)
    got, gts, exp, ets = [], [], [], []
    for c in range(calls):
        b = ops.gen_tuple64(c * per_call, per_call, ops.KEY_UNIFORM, nkeys)
        v = b.tuples.view(torch.int64).view(-1, 8)
        v[:, 4] = table[v[:, 0]]
        o, ot, no = ff_new.process([b])
        torch.cuda.synchronize()
        g_, gt_ = ff_new.results_to_host(o, ot, no)
        o, ot, no = ff_ref.process([b])
        torch.cuda.synchronize()
        e_, et_ = ff_ref.results_to_host(o, ot, no)
        got.append(g_); gts.append(gt_); exp.append(e_); ets.append(et_)
    got, gts, exp, ets = map(np.concatenate, (got, gts, exp, ets))
    tab = table.cpu().numpy().view(np.uint64)
    if prog == PROG_TUPLE64_FKEY:
        lookup = {int(x): i for i, x in enumerate(tab)}
        kidx = np.array([lookup[int(x)] for x in got["key"].view(np.uint64)], dtype=np.uint64)
    else:
        kidx = got["key"]["key"]
        hi = got["key"]["a"].astype(np.uint64) | (got["key"]["b"].astype(np.uint64) << np.uint64(32))
        assert np.array_equal(hi, tab[kidx])
    g = np.zeros(len(got), dtype=ops.RESULT32)
    g["key"], g["id"], g["isum"], g["fsum"] = kidx, got["id"], got["isum"], got["fsum"]
    order_g = np.lexsort((g["id"], g["key"]))
    order_e = np.lexsort((exp["id"], exp["key"]))
    assert len(g) == len(exp) > nkeys * nb
    _check_windows(g[order_g], gts[order_g], exp[order_e], ets[order_e])
    assert ff_new.stats() == ff_ref.stats()


TB_CASES = [(40, 10, 0, 3, 6, 8000, 777, "mono"), (64, 16, 100, 2, 9, 9000, 1000, "jitter")]


@pytest.mark.parametrize("prog", PROGS, ids=["f64", "k16"])
@pytest.mark.parametrize("case", TB_CASES, ids=[f"w{c[0]}_s{c[1]}_l{c[2]}_{c[7]}" for c in TB_CASES])
def test_tb_windows_rename_equivalence(wfb, oracle, prog, case):
    O, ops = oracle, wfb
    win, slide, lateness, nb, nkeys, n, batch, mode = case
    t, _ = _stream(O, prog, n, nkeys, 11, O.KEY_RR)
    rng = np.random.default_rng(11)
    ts = np.arange(n, dtype=np.int64) * 3
    if mode == "jitter":
        ts = ts + rng.integers(-40, 41, n)
    ts = np.maximum(ts, 0).astype(np.uint64)
    wm_fn = (lambda x: int(x.min())) if mode == "jitter" else None
    got, gts, fl = _run_ffat(ops, prog, t, ts, win, slide, nb, max(nkeys, 8), batch, 1, lateness, wm_fn)
    rt = _renamed(ops, prog, t)
    exp, ets, fl2 = _run_ffat(ops, ops.PROG_TUPLE64, rt, ts, win, slide, nb, max(nkeys, 8), batch, 1, lateness, wm_fn)
    assert fl == fl2 == 0
    g, gt = O.sort_results(_as_result32(ops, prog, got, t), gts)
    e, et = O.sort_results(exp, ets)
    _check_windows(g, gt, e, et)


@pytest.mark.parametrize("prog", PROGS, ids=["f64", "k16"])
@pytest.mark.parametrize("op", ["map", "filter"])
def test_stateful_rename_equivalence(wfb, oracle, prog, op):
    import torch
    O, ops = oracle, wfb
    nkeys = 300
    ks_new = ops.KeyedState(prog, max_keys=nkeys)
    ks_ref = ops.KeyedState(ops.PROG_TUPLE64, max_keys=nkeys)
    f = ops.functors(map_kind=1, filt_kind=1)
    calls, start = [], 0
    for sizes in ([5000, 3, 1025], [65536], [100] * 5):
        hosts = []
        for n in sizes:
            hosts.append(_stream(O, prog, n, nkeys, 100 + start))
            start += n
        calls.append(hosts)
    # one renaming over the whole stream: the handles keep their state from call to call
    ranks = _rank(prog, ops, np.concatenate([t for hosts in calls for t, _ in hosts]))
    roff = 0
    for hosts in calls:
        res = []
        for prg, ks in ((prog, ks_new), (ops.PROG_TUPLE64, ks_ref)):
            ins, outs, off = [], [], 0
            for t, ts in hosts:
                tt = t.copy()
                if prg == ops.PROG_TUPLE64:
                    tt["key"] = ranks[roff + off:roff + off + len(t)]
                off += len(t)
                b = ops.DeviceBatch.from_host(tt, ts)
                ins.append(b)
                outs.append(ops.DeviceBatch(torch.empty_like(b.tuples), torch.empty_like(b.ts), len(t), 0))
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
        roff += sum(len(t) for t, _ in hosts)
        for a, b in zip(res[0], res[1]):
            if op == "map":
                assert np.array_equal(a, b)
            else:
                assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def _reduce_expect(ops, prog, t, ts):
    """Reduce_GPU of the renamed stream through PROG_TUPLE64 (key bits 32)."""
    import torch
    eng = ops.Engine(ops.PROG_TUPLE64)
    out, n_out = eng.reduce_by_key(ops.DeviceBatch.from_host(_renamed(ops, prog, t), ts))
    torch.cuda.synchronize()
    k = int(n_out.item())
    return ops.to_host(out.tuples, ops.TUPLE64)[:k].copy(), ops.ts_to_host(out.ts)[:k].copy()


def _check_reduce(ops, prog, got, gts, t, exp, ets):
    assert len(got) == len(exp)
    r = _result_rank(prog, ops, _reduced_keys(ops, prog, got), t)
    assert np.array_equal(r, exp["key"])                       # ascending key order: the ranks are 0, 1, 2, ...
    assert np.array_equal(r, np.arange(len(r), dtype=np.uint64))
    assert np.array_equal(got["ivalue"], exp["ivalue"]) and np.array_equal(gts, ets)
    assert np.allclose(got["fvalue"], exp["fvalue"], rtol=FP_RTOL, atol=0)


def _reduced_keys(ops, prog, tup):
    """The program key of reduced tuples, as the key field of a result record (reduce keeps `key` and pad[0])."""
    if prog == ops.PROG_TUPLE64_FKEY:
        r = np.zeros(len(tup), dtype=ops.RESULT32D)
        r["key"] = tup["pad"][:, 0].view(np.float64)
    else:
        r = np.zeros(len(tup), dtype=ops.RESULT48K)
        r["key"]["key"] = tup["key"]
        r["key"]["a"] = (tup["pad"][:, 0] & np.uint64(0xFFFFFFFF)).astype(np.uint32)
        r["key"]["b"] = (tup["pad"][:, 0] >> np.uint64(32)).astype(np.uint32)
    return r


@pytest.mark.parametrize("prog", PROGS, ids=["f64", "k16"])
@pytest.mark.parametrize("n", [1, 33, 4097, 100001])
def test_reduce_by_key_order_and_rename(wfb, oracle, prog, n):
    import torch
    O, ops = oracle, wfb
    t, ts = _stream(O, prog, n, 500, 5)
    eng = ops.Engine(prog)
    out, n_out = eng.reduce_by_key(ops.DeviceBatch.from_host(t, ts))
    torch.cuda.synchronize()
    k = int(n_out.item())
    got, gts = ops.to_host(out.tuples, ops.TUPLE64)[:k].copy(), ops.ts_to_host(out.ts)[:k].copy()
    exp, ets = _reduce_expect(ops, prog, t, ts)
    _check_reduce(ops, prog, got, gts, t, exp, ets)
    if prog == ops.PROG_TUPLE64_FKEY:  # numeric order, NaN last
        keys = got["pad"][:, 0].view(np.float64)
        finite = keys[~np.isnan(keys)]
        assert np.all(np.diff(finite) > 0) and (np.isnan(keys).sum() <= 1) and (not np.isnan(keys).any() or np.isnan(keys[-1]))


@pytest.mark.parametrize("prog", PROGS, ids=["f64", "k16"])
def test_reduce_by_key_batches_rename(wfb, oracle, prog):
    import torch
    O, ops = oracle, wfb
    sizes = [3000, 1, 0, 4097, 20000]
    hosts, ins, outs = [], [], []
    for i, n in enumerate(sizes):
        t, ts = _stream(O, prog, n, 300, 40 + i)
        hosts.append((t, ts))
        b = ops.DeviceBatch.from_host(t, ts) if n else ops.DeviceBatch(torch.empty(0, dtype=torch.uint8, device="cuda"), torch.empty(0, dtype=torch.int64, device="cuda"), 0, 0)
        ins.append(b)
        outs.append(ops.DeviceBatch(torch.empty(max(n, 1) * 64, dtype=torch.uint8, device="cuda"), torch.empty(max(n, 1), dtype=torch.int64, device="cuda"), n, 0))
    eng = ops.Engine(prog)
    n_out = torch.full((len(sizes),), 7, dtype=torch.int32, device="cuda")
    eng.reduce_by_key_batches(ins, outs, n_out)
    torch.cuda.synchronize()
    no = n_out.cpu().numpy()
    for i, (t, ts) in enumerate(hosts):
        if len(t) == 0:
            assert no[i] == 0
            continue
        got, gts = ops.to_host(outs[i].tuples, ops.TUPLE64)[:no[i]].copy(), ops.ts_to_host(outs[i].ts)[:no[i]].copy()
        exp, ets = _reduce_expect(ops, prog, t, ts)
        _check_reduce(ops, prog, got, gts, t, exp, ets)


@pytest.mark.parametrize("prog", PROGS, ids=["f64", "k16"])
def test_capacity_flag_like_integer_keys(wfb, oracle, prog):
    """max_keys distinct keys fit; one key more raises the key-table-full flag, as it does for integer keys."""
    O, ops = oracle, wfb
    for extra in (0, 1):
        t, ts = _stream(O, prog, 20000, 64 + extra, 9, O.KEY_RR)
        flags = []
        for prg, tt in ((prog, t), (ops.PROG_TUPLE64, _renamed(ops, prog, t))):
            ff = ops.FfatWindowsGPU(prg, 16, 4, 1, max_keys=_distinct(ops, prog, t) - extra)
            ff.process([ops.DeviceBatch.from_host(tt, ts)])
            flags.append(ff.stats()[1] & 1)
        assert flags == [extra, extra], (extra, flags)


def _distinct(ops, prog, t):
    return int(_rank(prog, ops, t).max()) + 1


@pytest.mark.parametrize("prog", PROGS, ids=["f64", "k16"])
def test_integer_only_features_refused(wfb, prog):
    import torch
    ops = wfb
    from windflow_b200 import _lib
    L = _lib.lib()
    for kw in ({}, {"win_type": 1}):
        with pytest.raises(ops.WfbError) as e:
            ops.FfatWindowsGPU(prog, 16, 4, 1, max_keys=64, dense_keys=True, **kw)
        assert e.value.code == -1
    with pytest.raises(ops.WfbError) as e:
        ops.KeyedState(prog, max_keys=64, dense_keys=True)
    assert e.value.code == -1
    ff = ops.FfatWindowsGPU(prog, 16, 4, 1, max_keys=64)
    with pytest.raises(ops.WfbError) as e:
        ff.set_key_shard(2, 0)
    assert e.value.code == -1
    h = C.c_void_p()
    assert L.wfb_mg_create(C.byref(h), prog, 1, 0, None, 16, 4, 1, 64) == -5
    eng = ops.Engine(prog)
    with pytest.raises(ops.WfbError) as e:
        eng.set_key_bits(32)
    assert e.value.code == -1
    t = np.zeros(64, dtype=ops.TUPLE64)
    b = ops.DeviceBatch.from_host(t, np.arange(64, dtype=np.uint64))
    for call in (lambda: eng.keyby_group(b), lambda: eng.shard_by_key(b, 2),
                 lambda: eng.shard_lift([b], None, 2, torch.empty(2 * 64 * 64, dtype=torch.uint8, device="cuda"), 64,
                                        torch.zeros(9, dtype=torch.int32, device="cuda"))):
        with pytest.raises(ops.WfbError) as e:
            call()
        assert e.value.code == -5


@pytest.mark.parametrize("win_type", [0, 1], ids=["cb", "tb"])
def test_all_ones_16_byte_key_is_refused(wfb, oracle, win_type):
    """The all-ones 16-byte key marks a free table entry: tuples carrying it are dropped with the capacity flag (the call ends), and the
    other keys' windows are those of the stream without them."""
    O, ops = oracle, wfb
    t, ts = _stream(O, PROG_TUPLE64_K16, 12000, 12, 21, O.KEY_RR)
    bad = (np.arange(len(t)) % 7) == 3
    t["key"][bad] = ALL_ONES
    t["pad"][bad, 0] = ALL_ONES
    ts = np.arange(len(t), dtype=np.uint64)
    got, gts, fl = _run_ffat(ops, PROG_TUPLE64_K16, t, ts, 64, 16, 2, 16, 3000, win_type)
    assert fl & 1
    good = t[~bad]
    exp, ets, fl2 = _run_ffat(ops, PROG_TUPLE64_K16, good, ts[~bad], 64, 16, 2, 16, 3000, win_type)
    assert fl2 == 0
    if win_type == 0:  # count-based: the same windows per key (the dropped tuples never entered a window)
        g, gt = O.sort_results(_as_result32(ops, PROG_TUPLE64_K16, got, good), np.zeros(len(got), dtype=np.uint64))
        e, et = O.sort_results(_as_result32(ops, PROG_TUPLE64_K16, exp, good), np.zeros(len(exp), dtype=np.uint64))
        assert len(g) == len(e) > 0
        assert np.array_equal(g["key"], e["key"]) and np.array_equal(g["id"], e["id"]) and np.array_equal(g["isum"], e["isum"])
    else:  # time-based: the batches (and so the watermarks) differ once the tuples are removed; no window carries the refused key
        hi = got["key"]["a"].astype(np.uint64) | (got["key"]["b"].astype(np.uint64) << np.uint64(32))
        assert len(got) > 0 and not ((got["key"]["key"] == ALL_ONES) & (hi == ALL_ONES)).any()
