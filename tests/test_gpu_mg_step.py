"""The key-sharded step (wfb_mg_step / wfb_mg_flush) at one rank against a direct fold, the oracle and the single-GPU operator.

The step runs its own kernels and its own window-update entry point: on the bucketed exchange, the source's tile pass with the
destination-major virtual slots, the partition into bins and k_shard_bin_counts, then at the destination k_mg_count / k_mg_scan /
k_mg_split and the bucket update reading the receive buffer; on the fallback exchange (more than 65 536 slots, or WFB_MG_BUCKETED=0),
wfb_shard_lift and the window operator of the lifted program reading the received records in place. Results arrive three calls late
through a four-slot pipeline, and wfb_mg_flush appends the steps still in flight.

Every case folds the program of tests/cpp/ordered_program_32p.cu, whose combine reads its params ((h1, q1) o (h2, q2) =
(h1 M^q2 + h2, q1 + q2)), over ragged steps, and checks the windows of all steps and flushes against three references: the direct
fold of every key's surviving items in stream order (h and q bit for bit), the oracle fed one batch per step whose watermark is the
step's (window set, ids, result timestamps), and the single-GPU operator over the same steps (byte-identical records and timestamps).
The census of tests/test_gpu_ordered_windows.py states which branches of the window update every case reaches.

At one rank the exchange is a device copy. Only more ranks reach the sub-bucket split (nsub > 1), the virtual slots
(key % n) * L + key / n, the copy-engine push and the NCCL tokens; two processes cannot share a GPU in one NCCL communicator, so those
stay covered by bench.py's full-size check at N > 1 and by the numpy model of tests/test_multi_gpu.py."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import test_gpu_ordered_params as op
import test_gpu_ordered_windows as ow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WFB_E_CAPACITY = -3


class Step:
    """One step: its batch sizes (none: nbatches = 0), key draw ("u" uniform over the case's key set, "z" Zipf over it) and whether
    every tuple is filtered out (ids = 3 mod 7)."""

    def __init__(self, sizes, keys="u", filtered=False):
        self.sizes, self.keys, self.filtered = list(sizes), keys, filtered


FLUSH = "flush"


class MgCase:
    def __init__(self, name, cap, win, slide, nb, nkeys, steps, expect, shift=None, zipf=1.1, pre=True, seed=0):
        self.name, self.cap, self.win, self.slide, self.nb, self.nkeys = name, cap, win, slide, nb, nkeys
        self.steps, self.expect, self.shift, self.zipf, self.pre, self.seed = steps, expect, shift, zipf, pre, seed

    def stream(self):
        """Per entry of `steps`: FLUSH, or the step's list of batches (tuple arrays) in stream order."""
        rng = np.random.default_rng(self.seed)
        if self.nkeys >= self.cap:
            ks = np.arange(self.cap, dtype=np.uint64)
        else:  # a key set spread over the slot range, its last slot included
            ks = np.unique(np.concatenate([rng.choice(self.cap - 1, self.nkeys - 1, replace=False), [self.cap - 1]])).astype(np.uint64)
        w = 1.0 / np.arange(1, len(ks) + 1) ** self.zipf
        zk = rng.permutation(ks)
        out, nid = [], 0
        for st in self.steps:
            if st == FLUSH:
                out.append(FLUSH)
                continue
            n = sum(st.sizes)
            keys = ks[rng.integers(0, len(ks), n)] if st.keys == "u" else zk[rng.choice(len(ks), n, p=w / w.sum())]
            t = ow.make_tuples(keys, nid, 32)
            if st.filtered:
                base = (nid + 6) // 7 * 7
                t["id"] = np.uint64(base + 3) + np.uint64(7) * np.arange(n, dtype=np.uint64)
                nid = base + 7 * n
            else:
                nid += n
            bounds = np.cumsum([0] + st.sizes)
            out.append([t[bounds[i]:bounds[i + 1]] for i in range(len(st.sizes))])
        return out

    def update_calls(self, stream):
        """Survivors' keys (= slots: dense keys, one rank) of every window update, one per step."""
        res = []
        for st in stream:
            if st != FLUSH:
                k = [b["key"][ow.keep_mask(b)] for b in st]
                res.append(np.concatenate(k).astype(np.int64) if k else np.zeros(0, np.int64))
        return res


def S(*sizes, keys="u", filtered=False):
    return Step(sizes, keys, filtered)


MG_CASES = [
    # bps = 64, shift = 0: 40 keys with thousands of items per step (in-kernel evaluation, multi-chunk buckets, ring wrap); ragged K with
    # batches of 1, 255, 257 and 65536 tuples; a step of no batches; two steps before a flush, then the stream carries on
    MgCase("b64", 64, 48, 16, 1, 40,
           [S(4000, 4000, 4000), S(1, 255, 257, 6000), FLUSH, S(5000, 3000, 2000, 1000, 4000), S(), S(65536), S(3000, 2999),
            S(1, 1, 1, 1, 1, 1, 1, 9000), FLUSH, S(7000), S(6000, 255), S(257, 12000), S(100, 200), FLUSH],
           ("bucket_path", "eager", "inkernel_thread", "deferred", "multichunk_bucket", "open_pane_at_chunk", "window_wraps_ring",
            "ring_wrapped_twice"), shift=0, seed=1),
    # a key space that is not a power of two (L = 1024), Zipf keys with key 999 among them, lazy levels; a step whose tuples are all
    # filtered; a step 8x larger than all before it (grows the receive and region buffers)
    MgCase("b1000", 1000, 64, 16, 4, 400,
           [S(5000, keys="z"), S(3000, 2000, keys="z"), S(4000, filtered=True), S(5000), FLUSH, S(2500, 2500, keys="z"),
            S(*([5000] * 8), keys="z"), S(20000, 20000, keys="z"), S(1, 255), FLUSH],
           ("bucket_path", "lazy", "deferred_lazy", "inkernel_thread", "multichunk_bucket", "window_wraps_ring"), shift=0, seed=2),
    # shift = 2, bps = 1024: tiny panes (pane 3) whose buckets of four keys take the warp fold
    MgCase("b4096", 4096, 6, 3, 1, 200,
           [S(20000, 20000, 20000), S(65536), S(1, 255, 257), S(30000, 30000), FLUSH, S(40000, 1), FLUSH],
           ("bucket_path", ("max_keys_per_bucket", 2), "warp_fold", "warp_fold_multikey", "warp_subrange_split", "inkernel_warp",
            "key_warp_and_thread", "deferred_lazy", "window_wraps_ring"), shift=2, seed=3),
    # shift = 6: every slot of the bucketed exchange's largest key space, uniform and Zipf keys, about a million tuples
    MgCase("b65536", 65536, 4, 2, 2, 65536,
           [S(65536, 65536, 65536), S(200000, keys="z"), S(65536, 65536, 65536, 65536, keys="z"), FLUSH, S(200000), S(150000, 255, keys="z"),
            FLUSH],
           ("bucket_path", ("max_keys_per_bucket", 64), "multichunk_bucket", "inkernel_thread", "inkernel_warp", "deferred_lazy"),
           shift=6, zipf=1.0, seed=4),
    # more than 65536 slots: the fallback exchange, the destination's full sort over in-place lifted records, Zipf heavy keys; the
    # source side takes the engine's own params (pre = None)
    MgCase("fallback_full_sort", 100000, 40, 10, 2, 3000,
           [S(50000, 50000, keys="z"), S(100000, keys="z"), S(30000, filtered=True), S(80000, 20000, keys="z"), FLUSH,
            S(100000, keys="z"), S(1, 255, 257), FLUSH],
           ("full_sort", "lanes", "update", "inkernel_lanes", "inkernel_update", "deferred"), zipf=1.0, pre=False, seed=5),
]
# WFB_MG_BUCKETED=0 (latched by the first wfb_mg_create of a process): the fallback exchange on a key space the bucketed one would take
FORCED = MgCase("fallback_forced", 4096, 48, 16, 1, 300,
                [S(20000, 4000), S(), S(1, 255, 257, 30000), S(24000), FLUSH, S(10000, 10000), S(30000), FLUSH],
                ("bucket_path", "inkernel_thread", "deferred", "window_wraps_ring"), shift=2, seed=6)
ALL_CASES = MG_CASES + [FORCED]


def _geometry(c):
    return ow.Geometry(c.win, c.slide, c.nb, c.cap, 32)


@pytest.mark.parametrize("case", ALL_CASES, ids=lambda c: c.name)
def test_mg_case_reaches_its_regimes(case):
    """The census of every case (CPU): the window updates of its steps reach the branches it is there for; on the bucketed exchange at
    one rank the handle's bucket shift is the step's (slot >> shift, bps = L >> shift buckets)."""
    g = _geometry(case)
    if case.shift is not None:
        assert g.shift == case.shift
    assert g.buckets == (case.cap <= 65536)
    assert sum(len(b) for st in case.stream() if st != FLUSH for b in st) <= (1_100_000 if case.name == "b65536" else 600_000)
    ow.assert_regimes(ow.census(g, case.update_calls(case.stream())), case.expect)


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def prog32p(wfb):
    prog = op.register(wfb)
    yield prog
    wfb.RESULT_DTYPE.pop(prog, None); wfb.TUPLE_DTYPE.pop(prog, None)


def _params_as_pre(m):
    """OrdParams {M} in the `pre` argument of wfb_mg_step (typed wfb_functors_t in the binding: a registered program reads its own
    params_t there)."""
    from windflow_b200 import _lib
    buf = bytearray(C.sizeof(_lib.Functors))
    buf[:8] = int(m).to_bytes(8, "little")
    return _lib.Functors.from_buffer(buf)


def _watermark(i):
    return 1_000_000 + 1000 * i + 7  # (not a tuple id: the results must carry the step's argument)


def _oracle_step(go, res, wm, nb):
    """One step as one oracle batch of watermark wm, fed in pieces small enough for the oracle's output bound."""
    out, ots = [], []
    piece = max(1, 1024 // nb)
    for i in range(0, len(res), piece):
        r, rt = go.process_batch(res[i:i + piece], wm)
        out.append(r); ots.append(rt)
    return out, ots


def run_case(ops, O, prog, c):
    import torch
    from windflow_b200 import multigpu
    L = ops._lib.lib()
    stream = c.stream()
    prm = C.c_uint64(ow.M)
    pipe = multigpu.KeyShardedPipelineC(ops, _params_as_pre(ow.M) if c.pre else None, c.win, c.slide, c.nb, c.cap, 0, 1,
                                        torch.device("cuda", 0), prog=prog, params=prm)
    single = ops.FfatWindowsGPU(prog, c.win, c.slide, c.nb, max_keys=c.cap, dense_keys=True)
    ops.check(L.wfb_ffat_set_params(single.h, C.byref(prm), C.sizeof(prm)), "wfb_ffat_set_params")
    go = O.FfatGpuOracle(c.win, c.slide, c.nb)
    total = sum(len(b) for st in stream if st != FLUSH for b in st)
    cap = pipe.max_results(total)
    out = torch.empty(cap * 32, dtype=torch.uint8, device="cuda")
    out_ts = torch.empty(cap, dtype=torch.int64, device="cuda")
    n_out = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    got, gts, sgot, sgts, exp, ets = [], [], [], [], [], []
    since_flush, step_no = 0, 0
    for st in stream:
        if st == FLUSH:
            pipe.flush(out, out_ts, n_out)
            since_flush = 0
        else:
            wm = _watermark(step_no)
            step_no += 1
            dev = [ops.DeviceBatch.from_host(b, None, watermark=int(b["id"][0])) for b in st]  # (batch watermarks the step ignores)
            pipe.step(dev, wm, out, out_ts, n_out)
            since_flush += 1
            if dev:
                so, sts, sn = single.process([ops.DeviceBatch(d.tuples, None, d.n, wm) for d in dev])
                torch.cuda.synchronize()
                r, rt = single.results_to_host(so, sts, sn)
                sgot.append(r); sgts.append(rt)
            t = np.concatenate(st) if st else np.zeros(0, ow.TUPLE64)
            r, rt = _oracle_step(go, ow._lift_res(t[ow.keep_mask(t)]), wm, c.nb)
            exp += r; ets += rt
        torch.cuda.synchronize()
        r, rt = pipe.results_to_host(out, out_ts, n_out)
        if st != FLUSH and since_flush <= 3:
            assert len(r) == 0, f"a result {since_flush} calls after the start of the pipeline"
        got.append(r); gts.append(rt)
    assert pipe.stats()[1] == 0 and single.stats()[1] == 0
    assert pipe.results_total() == sum(len(x) for x in got)
    pipe.close(); single.close(); go.close()

    g, gt = O.sort_results(np.concatenate(got), np.concatenate(gts))
    e, et = O.sort_results(np.concatenate(exp), np.concatenate(ets))
    assert len(g) == len(e) > 0, (len(g), len(e))
    assert np.array_equal(g["key"], e["key"]) and np.array_equal(g["id"], e["id"])
    assert np.array_equal(gt, et)
    assert len(set(gt.tolist())) > 1
    t = np.concatenate([b for st in stream if st != FLUSH for b in st])
    surv = t[ow.keep_mask(t)]
    order, a, b = ow.cb_ranges(surv["key"], e["key"], e["id"], c.win, c.slide)
    h, _ = ow.hash_ranges(ow.np_lift_h(surv, 32)[order], a, b, np.uint64)
    bad = np.flatnonzero((g["h"] != h) | (g["q"] != (b - a).astype(np.uint64)))
    assert len(bad) == 0, f"{len(bad)} of {len(g)} windows differ from the direct fold in (h, q), first (key, id): " \
                          f"{[(int(g['key'][i]), int(g['id'][i])) for i in bad[:5]]}"
    s, stt = O.sort_results(np.concatenate(sgot), np.concatenate(sgts))
    assert s.tobytes() == g.tobytes() and np.array_equal(stt, gt), "the step's windows differ from the single-GPU operator's"
    return len(g)


def _outside_key_space(ops, prog, cap, bucketed):
    """A key equal to max_keys_total in the first step. Bucketed: WFB_E_CAPACITY from the call that exchanges that step (two calls
    later), or from the flush when fewer calls follow. Fallback: error bit 0 of wfb_mg_stats."""
    import torch
    from windflow_b200 import multigpu
    prm = C.c_uint64(ow.M)
    out = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    out_ts = torch.empty(1 << 15, dtype=torch.int64, device="cuda")
    n_out = torch.zeros(1, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(cap)

    def step_batches(i, bad):
        keys = rng.integers(0, min(cap, 64), 3000).astype(np.uint64)
        if bad:
            keys[1000] = cap
        return [ops.DeviceBatch.from_host(ow.make_tuples(keys, 3000 * i, 32), None, watermark=0)]
    for nsteps in (3, 1):
        pipe = multigpu.KeyShardedPipelineC(ops, None, 8, 4, 1, cap, 0, 1, torch.device("cuda", 0), prog=prog, params=prm)
        try:
            for i in range(nsteps):
                if bucketed and i == 2:
                    with pytest.raises(ops.WfbError) as ex:
                        pipe.step(step_batches(i, False), i, out, out_ts, n_out)
                    assert ex.value.code == WFB_E_CAPACITY
                    break
                pipe.step(step_batches(i, i == 0), i, out, out_ts, n_out)
            else:
                if bucketed:
                    with pytest.raises(ops.WfbError) as ex:
                        pipe.flush(out, out_ts, n_out)
                    assert ex.value.code == WFB_E_CAPACITY
                else:
                    pipe.flush(out, out_ts, n_out)
                    torch.cuda.synchronize()
                    assert pipe.stats()[1] & 1
                    assert np.all(pipe.results_to_host(out, out_ts, n_out)[0]["key"] < cap)
        finally:
            pipe.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", MG_CASES, ids=lambda c: c.name)
def test_mg_step_matches_direct_fold_oracle_and_single_gpu(wfb, oracle, prog32p, case):
    assert run_case(wfb, oracle, prog32p, case) > 0


@pytest.mark.gpu
def test_mg_step_forced_fallback_exchange():
    """WFB_MG_BUCKETED=0 is latched by the first wfb_mg_create of a process: the case runs in a child process. A key outside the key
    space then raises error bit 0 (the fallback's report) where the bucketed exchange would fail the call."""
    env = dict(os.environ, WFB_MG_BUCKETED="0")
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; import test_gpu_mg_step as T; T.child_main()"
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    p = subprocess.run(args, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, (p.stdout + p.stderr)[-4000:]
    assert "fallback_forced OK" in p.stdout


def child_main():
    from oracle import oracle as O
    from windflow_b200 import build, ops
    build.build()
    O.lib()
    prog = op.register(ops)
    n = run_case(ops, O, prog, FORCED)
    _outside_key_space(ops, prog, FORCED.cap, bucketed=False)
    print(f"fallback_forced OK: {n} windows")


@pytest.mark.gpu
def test_mg_key_outside_key_space_is_reported(wfb, prog32p):
    _outside_key_space(wfb, prog32p, 64, bucketed=True)
    _outside_key_space(wfb, prog32p, 100000, bucketed=False)
