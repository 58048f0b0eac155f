#!/usr/bin/env python
"""Operators over more than 65536 keys: one JSON line per configuration, each with the card's name and power limit read in the same run.

  keyed-stateful Map_GPU / Filter_GPU (PROG_TUPLE64, the counter per key of tools/bench_configs.py): 64 queued batches of 65536 tuples
      per call, at 65536 keys (bucket path) and at 2^20 and 2^22 keys (full sort by slot), uniform and Zipf-0.8 keys, through the hash
      table and dense. tuples/s and ms per call from CUDA events around the timed calls; then, in a run of its own, the per-phase split
      from torch.profiler's kernel durations (the phases run inside one library call): slots (k_ks_slots), sort (the partition or the
      onesweep passes), apply (k_ks_apply / k_ks_apply_runs) and compaction (the filter's k_flag_* kernels and their scan).
  time-based Ffat_Windows_GPU: tools/bench_configs.py's geometry scaled by the key count (win 4096 nk, slide 64 nk timestamp units,
      Nb 65, nk round-robin dense keys, ts = tuple index, one batch of 65536 per call) at nk = 65536 and 2^20.

    python tools/many_keys_bench.py [--iters 20] [--only stateful|tb]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from windflow_b200 import build, ops  # noqa: E402

BATCH, RING = 65536, 64


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # (the numbers stand without it, but the report says so)
        return f"unknown ({e!r})"


def zipf_cdf(nkeys, s=0.8):  # the oracle's table (oracle/oracle.py)
    w = 1.0 / np.power(np.arange(1, nkeys + 1, dtype=np.float64), s)
    c = np.cumsum(w)
    c /= c[-1]
    return c


def timed(fn, iters, warm=3):
    for i in range(warm):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(warm + i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


PHASES = [("slots", ("k_ks_slots",)), ("apply", ("k_ks_apply",)), ("compaction", ("k_flag_", "k_scan_u32")),
          ("sort", ("k_wide_", "k_radix_", "k_onesweep_"))]


def phase_split(fn, calls=5):
    """ms per call of every phase: kernel durations from torch.profiler (CUDA activities), summed by kernel name."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(calls):
            fn(i)
        torch.cuda.synchronize()
    ms = {p: 0.0 for p, _ in PHASES}
    ms["other"] = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t <= 0:
            continue
        name = next((p for p, pre in PHASES if any(x in ev.key for x in pre)), "other")
        ms[name] += t / 1e3 / calls
    return ms


def stateful(args, gpu):
    f_map, f_filt = ops.functors(map_kind=1), ops.functors(filt_kind=1)
    ins = ops.Segment([ops.gen_tuple64(i * BATCH, BATCH, ops.KEY_UNIFORM, 1) for i in range(RING)])
    outs = ops.Segment([ops.DeviceBatch(torch.empty_like(b.tuples), torch.empty_like(b.ts), BATCH, 0) for b in ins])
    n_out = torch.zeros(RING, dtype=torch.int32, device="cuda")
    for nkeys in (1 << 16, 1 << 20, 1 << 22):
        for dist in ("uniform", "zipf"):
            cdf = torch.from_numpy(zipf_cdf(nkeys)).cuda() if dist == "zipf" else None
            for i, b in enumerate(ins):  # regenerate the ring in place with this key space
                ops.gen_tuple64(i * BATCH, BATCH, ops.KEY_ZIPF if cdf is not None else ops.KEY_UNIFORM, nkeys, zipf_cdf=cdf, tuples=b.tuples, ts=b.ts)
            for dense in (False, True):
                for op in ("map", "filter"):
                    ks = ops.KeyedState(ops.PROG_TUPLE64, max_keys=nkeys, dense_keys=dense)
                    call = (lambda i: ks.map(ins, f_map)) if op == "map" else (lambda i: ks.filter(ins, f_filt, outs, n_out))
                    ms = timed(call, args.iters)
                    split = phase_split(call)
                    print(json.dumps({"config": f"{'Map' if op == 'map' else 'Filter'}_GPU keyed-stateful, {nkeys} {dist} keys "
                                                f"({'dense' if dense else 'hashed'}), {RING} queued batches of {BATCH} per call",
                                      "path": "buckets" if nkeys <= 65536 else "full sort", "gpu": gpu, "tuples_per_s": RING * BATCH / (ms * 1e-3),
                                      "ms_per_call": ms, "phase_ms_per_call": split}), flush=True)
                    ks.close()
            del cdf
    del ins, outs
    torch.cuda.empty_cache()


def time_based(args, gpu):
    n_out = torch.zeros(1, dtype=torch.int32, device="cuda")
    cap = 1 << 22
    o = torch.empty(cap * 32, dtype=torch.uint8, device="cuda")
    ots = torch.empty(cap, dtype=torch.int64, device="cuda")
    ring = 8
    for nk in (1 << 16, 1 << 20):
        tbh = ops.FfatWindowsGPU(ops.PROG_TUPLE64, 4096 * nk, 64 * nk, 65, max_keys=nk, dense_keys=True, win_type=1)
        tbb = [ops.gen_tuple64(i * BATCH, BATCH, ops.KEY_RR, nk) for i in range(ring)]
        state = {"i": 0}

        def step(_):  # a fresh stretch of the stream every call (timestamps keep growing), regenerated into the ring slot
            i = state["i"]
            state["i"] += 1
            b = tbb[i % ring]
            ops.gen_tuple64(i * BATCH, BATCH, ops.KEY_RR, nk, tuples=b.tuples, ts=b.ts)
            b.watermark = i * BATCH
            tbh.process([b], out=o, out_ts=ots, n_out=n_out)
        ms = timed(step, max(20, args.iters * 4))
        gen_ms = timed(lambda i: ops.gen_tuple64(i * BATCH, BATCH, ops.KEY_RR, nk, tuples=tbb[0].tuples, ts=tbb[0].ts), 50)
        err = tbh.stats()[1]
        if err:
            raise SystemExit(f"many_keys_bench.py: time-based, {nk} keys: device error flags {err}")
        print(json.dumps({"config": f"Ffat_Windows_GPU time-based, win 4096*{nk} slide 64*{nk} ts units, Nb=65, {nk} round-robin dense keys, "
                                    f"one batch of {BATCH} per call",
                          "path": "buckets" if nk <= 65536 else "full sort", "gpu": gpu, "tuples_per_s": BATCH / ((ms - gen_ms) * 1e-3),
                          "ms_per_call": ms - gen_ms, "windows_last_call": int(n_out.item())}), flush=True)
        tbh.close()
        del tbb
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="timed calls per keyed-stateful configuration (time-based: 4x)")
    ap.add_argument("--only", choices=["stateful", "tb"], default=None)
    args = ap.parse_args()
    build.build()
    if not torch.cuda.is_available():
        raise SystemExit("many_keys_bench.py: no CUDA device (nothing here runs on the CPU)")
    torch.cuda.set_device(0)
    gpu = card()
    if args.only in (None, "stateful"):
        stateful(args, gpu)
    if args.only in (None, "tb"):
        time_based(args, gpu)


if __name__ == "__main__":
    main()
