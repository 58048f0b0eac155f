"""Every window of the bench's headline configuration against a direct fold, on each arm the bench reports.

bench.py's flagship workload -- PROG_TUPLE64 with its Map (ivalue += 2, fvalue *= 1.0000001) and Filter ((ivalue & 1) == 0) fused in
front, count-based windows 4096 / 64, Nb 65, 65 536 dense keys, 128 batches of 65 536 tuples per call -- takes paths no smaller case
reaches: the grouped scatter k_wide_scatter_ranked (2048 wide tiles per call, at least 4 per SM), lazy FlatFAT levels (256 leaves of
32 bytes), the bucket update over 1024 buckets of 64 keys with about one pane per key per call, and k_ffat_windows_lazy firing about a
thousand groups per call. bench.py's own check samples 52 keys over two steps; here every window of every call is compared.

The reference (DirectFold) is written in torch and shares nothing with the library: it takes the generated device tensors (the device
generator is pinned against the host one by test_device_generator_matches_host), applies the Map and Filter itself, gives every
survivor its per-key arrival rank, folds pane partials (pane = gcd(win, slide)) into a per-key ring with index_add_, and emits the
windows of every group whose triggering item arrived in the call. Two payloads:
  * sums: isum exact in int64, fsum in float64;
  * the order-sensitive hash of Prog32 (tests/cpp/ordered_programs.cu): h = ord_mix(id, key, 0) per item, filter id % 7 != 3, a
    window's h = sum_i h_i M^(win-1-i) over its arrival ranks, q = M^win - 1, all mod 2^64. Its records have the bench program's sizes
    (64-byte tuple in, 32-byte result out), so its kernels take the same paths, and a fold out of order, a duplicated or a lost item
    changes it where a sum does not.

The stream is the bench's (run_ours): the priming calls, the 65 stagger rounds (2 to 128 batches: the first ones take the per-tile
scatter, so per-key state crosses both scatters), then main calls of 128 batches, generated one segment at a time, until every key's
kernel ring of 256 leaves has wrapped at least twice (594 calls in all). Arms: sums through the direct, the pipelined and the
hashed-key handle and the multi-GPU step at one rank (the --mg-path arm); the hash through the direct and the pipelined handle. Each
compares every call, profiles one main call to prove the arm ran the path it is there for, and checks the error flags. The builder-API
arm (pipeline_bench.cu restated as tests/cpp/headline_facade.cu) replays the same batches through the reference and compares the whole
run as a set.

Cost, measured on an H100 80GB HBM3 at a 700 W power limit: the GPU tests of this file take about 55 s; the device memory in use
(every process on the device, CUDA context included) peaks at 6.7 GiB in the multi-GPU arm, 4.4 to 5.2 GiB in the others, of which
torch holds at most 2.6 GiB.

CPU (-m "not gpu"): the reference equals the oracle on small streams and the direct fold of test_gpu_ordered_windows in hash form, the
headline shape reaches the paths above and wraps every ring twice, and headline_facade.cu compiles for sm_90a."""
import ctypes as C
import math
import os
import shutil
import subprocess
import time

import numpy as np
import pytest
import torch

import test_gpu_ordered_windows as ow
from bench import BATCH, FILT, MAP, NKEYS, SIGMA, SLIDE, WIN, stagger_rounds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NB = 65                       # bench.py --nb default
BPS = 128                     # bench.py --batches-per-step default
SEG = BPS * BATCH
STAG_BASE = 1 << 44           # run_ours: the stagger rounds draw from their own part of the index space
H100_SMS = 132
WIDE_TILE = 4096              # OSW_TILE_POS (wfb_kernels.cuh): positions per wide tile
OSR_GROUP = 4                 # wide tiles per CTA of k_wide_scatter_ranked, taken from OSR_GROUP wide tiles per SM on
FSUM_RTOL = 1e-12
FACADE_SRC = os.path.join(ROOT, "tests", "cpp", "headline_facade.cu")
FACADE_EXE = os.path.join(ROOT, "tests", "cpp", "headline_facade.bin")
FACADE_K, FACADE_RING, FACADE_SINKS = 128, 64, 2
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")


def _s64(x):
    """An unsigned 64-bit constant as the int64 with the same bits."""
    x %= 1 << 64
    return x - (1 << 64) if x >= 1 << 63 else x


MIX = [_s64(int(m)) for m in ow.MIX]


# ---------------------------------------------------------------------------------------------------------------------------------
# the reference: a direct fold in torch
# ---------------------------------------------------------------------------------------------------------------------------------
def _powers(base, n):
    """[base^0, ..., base^(n-1)] mod 2^64, as int64 bits."""
    out, x = [], 1
    for _ in range(n):
        out.append(_s64(x))
        x = x * base % (1 << 64)
    return out


def ord_mix(ids, keys):
    """ord_mix(id, key, 0) of tests/cpp/ordered_programs.cu in int64 (wrapping); `>>` is arithmetic in torch, hence the mask."""
    x = ((ids + 1) * MIX[0]) ^ (keys * MIX[1])
    x = x ^ ((x >> 29) & ((1 << 35) - 1))
    return x | 1


class DirectFold:
    """Count-based windows (win, slide, Nb) of every key, folded directly from pane partials.

    A group g of a key fires when the key's item of arrival rank B + g slide Nb - 1 arrives (B = (Nb - 1) slide + win); its windows
    w = g Nb + j, j < Nb, cover the arrival ranks [w slide, w slide + win), i.e. the panes [w slide / pane, (w slide + win) / pane).
    Every key keeps a ring of R = B / pane + spare pane partials; a slot is zeroed when its pane starts. A call may bring a key at most
    (spare - 1) panes: the ring then still holds every pane of the groups not fired before the call (asserted per call).

    step() takes the survivors of one call in arrival order: keys, per-item result timestamp (the watermark the trigger rule assigns)
    and the payloads (isum, fsum) or h. It returns the windows fired in the call, in (key, id) order, as a dict of device tensors."""

    def __init__(self, win, slide, nb, nkeys, device, sums=True, hashed=False, spare=8):
        self.win, self.slide, self.nb, self.nkeys, self.dev = win, slide, nb, nkeys, device
        self.pane = math.gcd(win, slide)
        self.B = (nb - 1) * slide + win
        self.G = slide * nb
        self.wp, self.sp, self.bp = win // self.pane, slide // self.pane, self.B // self.pane
        self.spare = spare
        self.R = self.bp + spare
        self.sums, self.hashed = sums, hashed
        z = dict(device=device)
        self.cnt = torch.zeros(nkeys, dtype=torch.int64, **z)
        if sums:
            self.isum = torch.zeros(nkeys * self.R, dtype=torch.int64, **z)
            self.fsum = torch.zeros(nkeys * self.R, dtype=torch.float64, **z)
        if hashed:
            self.h = torch.zeros(nkeys * self.R, dtype=torch.int64, **z)
            # an item of rank j in its pane is carried by M^(pane-1-j); pane p of a window by M^(pane (Wp-1-p))
            self.item_pow = torch.tensor(_powers(ow.M, self.pane)[::-1], dtype=torch.int64, **z)
            self.pane_pow = torch.tensor(_powers(pow(ow.M, self.pane, 1 << 64), self.wp)[::-1], dtype=torch.int64, **z)
            self.q = _s64(pow(ow.M, win, 1 << 64) - 1)
        self.pane_off = torch.arange(self.wp, dtype=torch.int64, **z)
        self.j_off = torch.arange(nb, dtype=torch.int64, **z)

    CHUNK = 1 << 18  # windows folded at a time

    def _floordiv(self, a, b):
        return torch.div(a, b, rounding_mode="floor")

    def step(self, keys, ts, isum=None, fsum=None, h=None):
        n = keys.numel()
        sk, order = torch.sort(keys, stable=True)
        uk, counts = torch.unique_consecutive(sk, return_counts=True)
        starts = torch.cumsum(counts, 0) - counts
        c0 = self.cnt[uk]
        c1 = c0 + counts
        assert n == 0 or int(counts.max()) <= (self.spare - 1) * self.pane, "a key got more panes in one call than the ring spares"
        rank = torch.arange(n, dtype=torch.int64, device=self.dev) - torch.repeat_interleave(starts, counts) + torch.repeat_interleave(c0, counts)
        p = self._floordiv(rank, self.pane)
        j = rank - p * self.pane
        slot = sk * self.R + torch.remainder(p, self.R)
        fresh = slot[j == 0]
        if self.sums:
            self.isum[fresh] = 0
            self.fsum[fresh] = 0
            self.isum.index_add_(0, slot, isum[order])
            self.fsum.index_add_(0, slot, fsum[order])
        if self.hashed:
            self.h[fresh] = 0
            self.h.index_add_(0, slot, h[order] * self.item_pow[j])
        self.cnt[uk] = c1
        # groups whose trigger rank B + g G - 1 lies in [c0, c1)
        g_lo = torch.clamp(-self._floordiv(self.B - 1 - c0, self.G), min=0)
        g_hi = self._floordiv(c1 - self.B, self.G)
        ng = torch.clamp(g_hi - g_lo + 1, min=0)
        gk = torch.repeat_interleave(torch.arange(len(uk), device=self.dev), ng)
        first = torch.cumsum(ng, 0) - ng
        g = g_lo[gk] + torch.arange(gk.numel(), dtype=torch.int64, device=self.dev) - first[gk]
        trig = self.B + g * self.G - 1
        g_ts = ts[order[starts[gk] + trig - c0[gk]]]
        w = (g * self.nb)[:, None] + self.j_off[None, :]                           # (groups, Nb)
        key = uk[gk][:, None].expand_as(w).reshape(-1)
        w = w.reshape(-1)
        out = {"key": key, "id": w, "ts": g_ts[:, None].expand(-1, self.nb).reshape(-1)}
        if self.sums:
            out["isum"], out["fsum"] = torch.empty_like(w), torch.empty(w.numel(), dtype=torch.float64, device=self.dev)
        if self.hashed:
            out["h"], out["q"] = torch.empty_like(w), torch.full_like(w, self.q)
        for c in range(0, w.numel(), self.CHUNK):  # (a call where every key fires its first group has 65 windows per key)
            s = slice(c, c + self.CHUNK)
            panes = (w[s] * self.sp)[:, None] + self.pane_off[None, :]             # (windows, Wp)
            cells = key[s, None] * self.R + torch.remainder(panes, self.R)
            if self.sums:
                out["isum"][s] = self.isum[cells].sum(1)
                out["fsum"][s] = self.fsum[cells].sum(1)
            if self.hashed:
                out["h"][s] = (self.h[cells] * self.pane_pow[None, :]).sum(1)
        return out


def bench_survivors(tuples, wm):
    """Map then Filter of the bench functors over one call's tuples (uint8 tensor of 64-byte records) in torch: keys, per-item
    watermarks, isum, fsum of the survivors in arrival order. The Map is one IEEE multiply, as in the kernel."""
    t = tuples.view(torch.int64).view(-1, 8)
    iv = t[:, 2] + MAP["iadd"]
    keep = (iv & FILT["mod"]) == 0
    fv = t[:, 3].view(torch.float64) * MAP["fscale"]
    return t[:, 0][keep], wm[keep], iv[keep], fv[keep]


def hash_survivors(tuples, wm):
    """Prog32's filter (id % 7 != 3) and item hash over one call's tuples."""
    t = tuples.view(torch.int64).view(-1, 8)
    keep = torch.remainder(t[:, 1], 7) != 3
    k, ids = t[:, 0][keep], t[:, 1][keep]
    return k, wm[keep], ord_mix(ids, k)


# ---------------------------------------------------------------------------------------------------------------------------------
# the stream: bench.py's run_ours at one GPU
# ---------------------------------------------------------------------------------------------------------------------------------
def prime_calls():
    return int(np.ceil(((NB - 1) * SLIDE + WIN) * NKEYS / SIGMA / SEG)) + 2


def kernel_geometry():
    return ow.Geometry(WIN, SLIDE, NB, NKEYS, 32)


def main_calls():
    """Main calls after which every key's count exceeds twice its kernel ring of n leaves (panes), with the count of the key that
    gets the fewest stagger panes (one) at six standard deviations below its expectation."""
    g = kernel_geometry()
    c = 0
    while _least_count(c) - 6 * math.sqrt(_least_count(c)) < 2 * g.n * g.pane:
        c += 1
    return c


def _least_count(main):
    """Expected survivors of the key with the fewest stagger panes (one) after the priming calls, the stagger rounds and `main` calls."""
    return (prime_calls() + main) * SEG * SIGMA / NKEYS + SLIDE


def calls():
    """(kind, start, n, nkeys of the generator) of every call, in order."""
    out = [("prime", t * SEG, SEG, NKEYS) for t in range(prime_calls())]
    off = 0
    for nk, n in stagger_rounds(1):
        out.append(("stagger", STAG_BASE + off, n, nk))
        off += n
    t0 = prime_calls()
    out += [("main", (t0 + i) * SEG, SEG, NKEYS) for i in range(main_calls())]
    return out


def gen_call(ops, start, n, nkeys, buf):
    """The call's tuples, generated into the first n records of buf = (tuples, ts): one allocation for every call of a run."""
    b = ops.gen_tuple64(start, n, ops.KEY_UNIFORM, nkeys, tuples=buf[0][:n * 64], ts=buf[1][:n])
    batches = ops.Segment([ops.DeviceBatch(b.tuples[i * BATCH * 64:(i + 1) * BATCH * 64], b.ts[i * BATCH:(i + 1) * BATCH], BATCH,
                                           watermark=start + i * BATCH) for i in range(n // BATCH)])
    return b, batches


# ---------------------------------------------------------------------------------------------------------------------------------
# comparison
# ---------------------------------------------------------------------------------------------------------------------------------
def _canon(d):
    """Sort a dict of equal-length tensors by (key, id); also return the sorted composite (key << 40 | id)."""
    comp = (d["key"] << 40) | d["id"]
    comp, order = torch.sort(comp)
    return comp, {k: v[order] for k, v in d.items()}


def compare(arm, call, got, exp, fields, shift, dense):
    """got / exp: dicts of device tensors. Exact fields, fsum within FSUM_RTOL, no duplicate (key, id)."""
    assert got["key"].numel() == exp["key"].numel(), f"{arm}, call {call}: {got['key'].numel()} windows, expected {exp['key'].numel()}"
    if exp["key"].numel() == 0:
        return
    gc, g = _canon(got)
    ec, e = _canon(exp)
    dup = int((gc[1:] == gc[:-1]).sum())
    assert dup == 0, f"{arm}, call {call}: {dup} duplicate (key, id)"
    bad = gc != ec
    for f in fields:
        if f == "fsum":
            bad |= ~((g[f] - e[f]).abs() <= FSUM_RTOL * e[f].abs())
        else:
            bad |= g[f] != e[f]
    nbad = int(bad.sum())
    if nbad:
        idx = torch.nonzero(bad).flatten()[:5].cpu().numpy()
        gh = {f: g[f].cpu().numpy() for f in ["key", "id"] + list(fields)}
        eh = {f: e[f].cpu().numpy() for f in ["key", "id"] + list(fields)}
        lines = []
        for i in idx:
            k = int(eh["key"][i])
            where = f"bucket {k >> shift}" if dense else "bucket unknown (hashed keys: slot order varies)"
            lines.append(f"(key {k}, id {int(eh['id'][i])}; {where}) expected " +
                         ", ".join(f"{f}={eh[f][i]}" for f in fields) + " got " +
                         ", ".join(f"{f}={gh[f][i]}" for f in ["key", "id"] + list(fields)))
        raise AssertionError(f"{arm}, call {call}: {nbad} of {len(ec)} windows differ from the direct fold; first: " + "; ".join(lines))


def lib_results(out, out_ts, n, hashed):
    r = out[:n * 32].view(torch.int64).view(-1, 4)
    d = {"key": r[:, 0], "id": r[:, 1], "ts": out_ts[:n]}
    if hashed:
        d["h"], d["q"] = r[:, 2], r[:, 3]
    else:
        d["isum"], d["fsum"] = r[:, 2], r[:, 3].view(torch.float64)
    return d


def _cat(ds):
    return {k: torch.cat([d[k] for d in ds]) for k in ds[0]}


def kernel_names(prof):
    """Base names of the CUDA kernels of a trace: 'void k_x<...>(...)' -> 'k_x'."""
    names = set()
    for ev in prof.events():
        n = ev.name
        if n.startswith("void "):
            n = n[5:]
        n = n.split("(")[0].split("<")[0].split("::")[-1].strip()
        names.add(n)
    return names


# ---------------------------------------------------------------------------------------------------------------------------------
# the arms
# ---------------------------------------------------------------------------------------------------------------------------------
ARMS = {  # name: (payload, handle, delay in calls, kernels the arm exists to reach)
    "sum_direct": ("sum", "direct", 0, {"k_wide_scatter_ranked", "k_ffat_update_buckets", "k_ffat_windows_lazy"}),
    "sum_pipelined": ("sum", "pipelined", 1, {"k_wide_scatter_ranked", "k_ffat_update_buckets", "k_ffat_windows_lazy"}),
    "sum_hashed_keys": ("sum", "hashed", 0, {"k_wide_scatter_ranked", "k_ffat_update_buckets", "k_ffat_windows_lazy"}),
    "sum_mg_step": ("sum", "mg", 3, {"k_wide_scatter_ranked_tile", "k_ffat_update_buckets"}),
    "hash_direct": ("hash", "direct", 0, {"k_wide_scatter_ranked", "k_ffat_update_buckets", "k_ffat_windows_lazy"}),
    "hash_pipelined": ("hash", "pipelined", 1, {"k_wide_scatter_ranked", "k_ffat_update_buckets", "k_ffat_windows_lazy"}),
}
PROFILED_MAIN_CALL = 2


@pytest.fixture(scope="module")
def prog32(wfb):
    """Prog32 of tests/cpp/ordered_programs.cu, registered as an application registers its program."""
    L = ow._ordlib()
    pid = L.ord_register_32()
    assert pid >= 6, pid
    wfb.RESULT_DTYPE[pid], wfb.TUPLE_DTYPE[pid] = ow.RES_DTYPE[32], ow.TUPLE64
    yield pid
    wfb.RESULT_DTYPE.pop(pid, None); wfb.TUPLE_DTYPE.pop(pid, None)


def _make_handle(ops, arm, prog32, dev):
    from windflow_b200 import multigpu
    payload, kind, _, _ = ARMS[arm]
    prog = ops.PROG_TUPLE64 if payload == "sum" else prog32
    pre = ops.functors(**MAP, **FILT) if payload == "sum" else None
    if kind == "mg":
        pipe = multigpu.KeyShardedPipelineC(ops, pre, WIN, SLIDE, NB, NKEYS, 0, 1, dev)
        return pipe, pre
    ff = ops.FfatWindowsGPU(prog, WIN, SLIDE, NB, max_keys=NKEYS, dense_keys=kind != "hashed", pipelined=kind == "pipelined")
    if payload == "hash":
        prm = C.c_uint64(ow.M)
        ops.check(ops._lib.lib().wfb_ffat_set_params(ff.h, C.byref(prm), C.sizeof(prm)), "wfb_ffat_set_params")
    return ff, pre


def run_arm(ops, arm, prog32):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    handle, pre = _make_handle(ops, arm, prog32, torch.device("cuda", 0))
    try:
        return _run_arm(ops, arm, handle, pre)
    finally:
        handle.close()


def _run_arm(ops, arm, handle, pre):
    payload, kind, delay, _ = ARMS[arm]
    dev = torch.device("cuda", 0)
    ref = DirectFold(WIN, SLIDE, NB, NKEYS, dev, sums=payload == "sum", hashed=payload == "hash")
    fields = ("isum", "fsum", "ts") if payload == "sum" else ("h", "q", "ts")
    shift = kernel_geometry().shift
    cap = handle.max_results(SEG * (4 if kind == "mg" else 1))
    out = torch.empty(cap * 32, dtype=torch.uint8, device=dev)
    out_ts = torch.empty(cap, dtype=torch.int64, device=dev)
    n_out = torch.zeros(1, dtype=torch.int32, device=dev)
    pending = []          # reference windows of the calls whose results the handle has not delivered yet
    total0 = handle.results_total()
    windows = compared_calls = main_no = 0
    names = None
    peak = 0
    stream = calls()
    buf = (torch.empty(SEG * 64, dtype=torch.uint8, device=dev), torch.empty(SEG, dtype=torch.int64, device=dev))
    for i, (what, start, n, nk) in enumerate(stream):
        if what == "main" and main_no == 0:
            torch.cuda.empty_cache()  # (the stagger rounds leave cached blocks of many sizes)
        b, batches = gen_call(ops, start, n, nk, buf)
        profile = what == "main" and main_no == PROFILED_MAIN_CALL
        main_no += what == "main"
        if profile:
            torch.cuda.synchronize()
            prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
            prof.__enter__()
        if kind == "mg":
            handle.step(batches, b.watermark, out, out_ts, n_out)
        else:
            handle.process(batches, pre=pre, out=out, out_ts=out_ts, n_out=n_out)
        if profile:
            torch.cuda.synchronize()
            prof.__exit__(None, None, None)
            names = kernel_names(prof)
        # the reference of this call (multi-GPU step: every result carries the step's watermark)
        idx = torch.arange(n, dtype=torch.int64, device=dev)
        wm = torch.full_like(idx, start) if kind == "mg" else start + torch.div(idx, BATCH, rounding_mode="floor") * BATCH
        if payload == "sum":
            k, w, iv, fv = bench_survivors(b.tuples, wm)
            pending.append(ref.step(k, w, isum=iv, fsum=fv))
        else:
            k, w, h = hash_survivors(b.tuples, wm)
            pending.append(ref.step(k, w, h=h))
        del b, batches, k, w
        # results_total() counts a call's results where its window update runs: the pipelined handle's one call before it delivers them
        total1 = handle.results_total()
        counted = pending[-1] if kind == "pipelined" else (pending[0] if len(pending) > delay else None)
        want = 0 if counted is None else counted["key"].numel()
        assert total1 - total0 == want, f"{arm}, call {i}: results_total() grew by {total1 - total0}, expected {want}"
        total0 = total1
        if len(pending) > delay:
            got_n = int(n_out.item())
            exp = pending.pop(0)
            compare(arm, i - delay, lib_results(out, out_ts, got_n, payload == "hash"), exp, fields, shift, kind != "hashed")
            windows += got_n
            compared_calls += 1
        else:
            assert int(n_out.item()) == 0, f"{arm}, call {i}: results before the pipeline is full"
        free, tot = torch.cuda.mem_get_info()
        peak = max(peak, tot - free)
    if delay:
        handle.flush(out, out_ts, n_out)
        got_n = int(n_out.item())
        total1 = handle.results_total()
        assert total1 - total0 == (0 if kind == "pipelined" else got_n), f"{arm}, flush: results_total() grew by {total1 - total0}"
        compare(arm, f"flush (calls {len(stream) - delay}..)", lib_results(out, out_ts, got_n, payload == "hash"), _cat(pending), fields,
                shift, kind != "hashed")
        windows += got_n
        compared_calls += len(pending)
    assert handle.stats()[1] == 0, f"{arm}: error flags {handle.stats()[1]}"
    return {"calls": compared_calls, "windows": windows, "kernels": names, "least_key_count": int(ref.cnt.min()), "device_in_use": peak,
            "torch_reserved": torch.cuda.max_memory_reserved()}


@pytest.mark.gpu
@pytest.mark.parametrize("arm", list(ARMS))
def test_headline_arm_matches_direct_fold(wfb, prog32, arm):
    t0 = time.perf_counter()
    r = run_arm(wfb, arm, prog32)
    want = ARMS[arm][3]
    assert r["kernels"] is not None and want <= r["kernels"], \
        f"{arm} no longer reaches {sorted(want - (r['kernels'] or set()))}; kernels of a main call: {sorted(r['kernels'] or [])}"
    g = kernel_geometry()
    assert r["least_key_count"] >= 2 * g.n * g.pane, f"{arm}: a key's ring wrapped fewer than two times ({r['least_key_count']} items)"
    assert r["calls"] == len(calls()) and r["windows"] > 0
    r["seconds"] = time.perf_counter() - t0
    print(f"\n{arm}: {r['calls']} calls, {r['windows']} windows compared, {r['seconds']:.1f} s, "
          f"device memory in use at most {r['device_in_use'] / 2**30:.2f} GiB (of it held by torch at most {r['torch_reserved'] / 2**30:.2f} GiB)")


# ---------------------------------------------------------------------------------------------------------------------------------
# the builder-API arm: tests/cpp/headline_facade.cu
# ---------------------------------------------------------------------------------------------------------------------------------
FACADE_BATCHES = 20480        # source batches of a run: 4096 past the 16384 after which every key has fired its first group
FACADE_NVCC = ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "--expt-extended-lambda",
               "-diag-suppress", "186", "-I" + os.path.join(ROOT, "include")]


def _facade_compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(ROOT, "include", "wf", h) for h in ("windflow_gpu.hpp", "deferred_counts.hpp")] + \
        [os.path.join(ROOT, "windflow_b200", "csrc", h) for h in ("wfb_kernels.cuh", "wfb_launch.cuh")] + [FACADE_SRC]
    if os.path.exists(FACADE_EXE) and all(os.path.getmtime(FACADE_EXE) > os.path.getmtime(h) for h in hdrs):
        return
    subprocess.check_call(FACADE_NVCC + ["-o", FACADE_EXE, FACADE_SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200",
                                         "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"])


def facade_expected(ops, nbatches, ring):
    """The windows of the application's run: batch i of the source is batch i % ring of the stream, every window in (key, id) order."""
    dev = torch.device("cuda", 0)
    ref = DirectFold(WIN, SLIDE, NB, NKEYS, dev)
    ring_b = ops.gen_tuple64(0, ring * BATCH, ops.KEY_UNIFORM, NKEYS)
    outs = []
    for c0 in range(0, nbatches, FACADE_K):
        idx = [i % ring for i in range(c0, min(nbatches, c0 + FACADE_K))]
        tup = torch.cat([ring_b.tuples[r * BATCH * 64:(r + 1) * BATCH * 64] for r in idx])
        wm = torch.zeros(len(idx) * BATCH, dtype=torch.int64, device=dev)
        k, w, iv, fv = bench_survivors(tup, wm)
        o = ref.step(k, w, isum=iv, fsum=fv)
        del o["ts"]
        outs.append(o)
    return _cat(outs)


@pytest.mark.gpu
@pytest.mark.parametrize("style", ["fluent", "statements"])
def test_headline_facade_matches_direct_fold(wfb, tmp_path, style):
    """Whether the window replica's calls reach 128 batches depends on its queue, so this arm does not assert its path; a Sink sees no
    timestamps, so the comparison is of (key, id, isum, fsum), as a set over the whole run."""
    _facade_compile()
    t0 = time.perf_counter()
    p = subprocess.run([FACADE_EXE, str(FACADE_K), str(FACADE_BATCHES), str(FACADE_RING), str(FACADE_SINKS), style, str(tmp_path)],
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "FACADE_OK" in p.stdout, (p.stdout + p.stderr)[-3000:]
    rows = np.concatenate([np.fromfile(os.path.join(str(tmp_path), f"sink{s}.bin"), dtype=wfb.RESULT32) for s in range(FACADE_SINKS)])
    size = sum(os.path.getsize(os.path.join(str(tmp_path), f"sink{s}.bin")) for s in range(FACADE_SINKS))
    assert size < 0.5 * 2**30
    got = {f: torch.from_numpy(rows[f].astype(np.float64 if f == "fsum" else np.int64)).cuda() for f in ("key", "id", "isum", "fsum")}
    exp = facade_expected(wfb, FACADE_BATCHES, FACADE_RING)
    compare(f"facade {style}", "whole run", got, exp, ("isum", "fsum"), kernel_geometry().shift, True)
    print(f"\nfacade {style}: {len(rows)} windows compared, {time.perf_counter() - t0:.1f} s")


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------------
def _cpu_stream(nkeys, n, seed):
    from oracle import oracle as O
    t, _ = O.gen_tuple64(seed * 1000003, n, O.KEY_UNIFORM, nkeys)
    return t


@pytest.mark.parametrize("geom", [(10, 4, 3), (3, 5, 2), (48, 16, 1), (4096, 64, 65)], ids=["pane_lt_slide", "slide_gt_win", "nb1", "headline_nb65"])
@pytest.mark.parametrize("rule", ["batch", "step"])
def test_direct_fold_matches_oracle(oracle, geom, rule):
    """The reference on the CPU against oracle.FfatGpuOracle: window set, ids, isum exact, fsum within 1e-12, result timestamps by the
    batch-watermark rule (direct and pipelined handles) or the step-watermark rule (multi-GPU step)."""
    O = oracle
    win, slide, nb = geom
    big = win == 4096
    nkeys = 3 if big else 7
    batch = 4000 if big else 300
    per_call = 6 if big else 5
    t = _cpu_stream(nkeys, 120000 if big else 9000, win + slide)
    f = lambda x: O.map_filter_tuple64(x, np.zeros(len(x), np.uint64), 1, MAP["iadd"], MAP["fscale"], 1)  # noqa: E731
    ref = DirectFold(win, slide, nb, nkeys, "cpu", spare=(per_call * batch) // math.gcd(win, slide) + 2)
    go = O.FfatGpuOracle(win, slide, nb)
    got, exp = [], []
    nbat = len(t) // batch
    for c0 in range(0, nbat, per_call):
        step_wm = 10**9 + 17 * c0
        for bi in range(c0, min(nbat, c0 + per_call)):
            surv = f(t[bi * batch:(bi + 1) * batch])[0]
            wm = 5 + bi * batch if rule == "batch" else step_wm
            r, rt = go.process_batch(O.lift_tuple64(surv), wm)
            exp.append((r, rt))
        tt = torch.from_numpy(t[c0 * batch:min(nbat, c0 + per_call) * batch].view(np.uint8).reshape(-1).copy())
        idx = torch.arange(tt.numel() // 64, dtype=torch.int64)
        wm = 5 + c0 * batch + torch.div(idx, batch, rounding_mode="floor") * batch if rule == "batch" else torch.full_like(idx, step_wm)
        k, w, iv, fv = bench_survivors(tt, wm)
        got.append(ref.step(k, w, isum=iv, fsum=fv))
    go.close()
    e, et = O.sort_results(np.concatenate([x[0] for x in exp]), np.concatenate([x[1] for x in exp]))
    g = _cat(got)
    assert len(e) == g["key"].numel() > (50 if big else 200)
    o = np.lexsort((g["id"].numpy(), g["key"].numpy()))
    assert np.array_equal(g["key"].numpy()[o], e["key"].astype(np.int64)) and np.array_equal(g["id"].numpy()[o], e["id"].astype(np.int64))
    assert np.array_equal(g["isum"].numpy()[o], e["isum"])
    assert np.all(np.abs(g["fsum"].numpy()[o] - e["fsum"]) <= FSUM_RTOL * np.abs(e["fsum"]))
    assert np.array_equal(g["ts"].numpy()[o], et.astype(np.int64))
    assert len(np.unique(et)) > 1


@needs_nvcc
def test_hash_form_matches_host_program_and_direct_fold():
    """The reference's item hash == ord_lift_host of Prog32, its windows' (h, q) == test_gpu_ordered_windows.hash_ranges and, on a
    sample, a sequential fold with ord_comb_host."""
    L = ow._ordlib()
    t = _cpu_stream(5, 40000, 11)
    hh, qq, keep = np.zeros(len(t), np.uint64), np.zeros(len(t), np.uint64), np.zeros(len(t), np.uint8)
    assert L.ord_lift_host(32, ow.M, ow._p(t), len(t), ow._p(hh), ow._p(qq), ow._p(keep)) == 0
    tt = torch.from_numpy(t.view(np.uint8).reshape(-1).copy())
    k, _, h = hash_survivors(tt, torch.zeros(len(t), dtype=torch.int64))
    assert np.array_equal(h.numpy().view(np.uint64), hh[keep.astype(bool)])
    win, slide, nb = 96, 32, 3
    ref = DirectFold(win, slide, nb, 5, "cpu", sums=False, hashed=True, spare=300)
    outs = [ref.step(k[i:i + 4000], torch.zeros(len(k[i:i + 4000]), dtype=torch.int64), h=h[i:i + 4000]) for i in range(0, len(k), 4000)]
    g = _cat(outs)
    surv = t[keep.astype(bool)]
    order, a, b = ow.cb_ranges(surv["key"], g["key"].numpy().astype(np.uint64), g["id"].numpy().astype(np.uint64), win, slide)
    eh, eq = ow.hash_ranges(hh[keep.astype(bool)][order], a, b, np.uint64)
    assert len(eh) > 500
    assert np.array_equal(g["h"].numpy().view(np.uint64), eh) and np.array_equal(g["q"].numpy().view(np.uint64), eq)
    hs = np.ascontiguousarray(hh[keep.astype(bool)][order])
    for i in np.random.default_rng(2).choice(len(eh), 20, replace=False):
        x, y = np.zeros(1, np.uint64), np.zeros(1, np.uint64)
        for jj in range(a[i], b[i]):
            hv = hs[jj:jj + 1]
            assert L.ord_comb_host(32, ow.M, ow._p(x), ow._p(y), ow._p(hv), ow._p(np.array([ow.M - 1], np.uint64)), ow._p(x), ow._p(y), 1, 1) == 0
        assert x[0] == eh[i] and y[0] == eq[i]


def test_headline_shape_reaches_its_paths():
    """At the bench's shape: a main call has at least 4 wide tiles per SM of an H100 (the grouped scatter), the FlatFAT levels are lazy on
    the bucket path (1024 buckets of 64 keys), and the run is long enough that every key's ring wraps twice."""
    g = kernel_geometry()
    assert (BPS * (-(-BATCH // 256) * 256)) // WIDE_TILE >= OSR_GROUP * H100_SMS
    assert min(n for _, n in stagger_rounds(1)) // WIDE_TILE < OSR_GROUP * H100_SMS  # (the first stagger rounds take the per-tile scatter)
    assert g.buckets and g.lazy and g.shift == 6 and NKEYS >> g.shift == 1024 and g.n == 256
    assert SEG * SIGMA / NKEYS == SLIDE == g.pane  # about one pane per key per main call
    least = _least_count(main_calls())
    assert least - 6 * math.sqrt(least) >= 2 * g.n * g.pane > _least_count(0)
    assert 350 <= main_calls() <= 420
    # the reference's ring: a key's items of one call (binomial, mean 64 or 110 for the hash filter) stay far below its spare panes
    assert (DirectFold(WIN, SLIDE, NB, 1, "cpu").spare - 1) * g.pane >= 4 * (SEG * 6 / 7 / NKEYS)


@needs_nvcc
def test_headline_facade_compiles():
    _facade_compile()
    assert os.path.exists(FACADE_EXE)
