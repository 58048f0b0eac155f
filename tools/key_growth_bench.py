"""Cost of a key table that grows (WFB_KEYS_GROW): the count-based Ffat_Windows_GPU bench configuration (Map -> Filter -> windows
4096 / 64, Nb 65, 65536 uniform keys, batches of 65536 tuples) through PROG_TUPLE64 on the hashed key table (as tools/keys_bench.py's
tuple64_hash), with

    fixed        a handle created at 65536 keys
    grow_same    a growing handle created at 65536 keys: it never grows, every call pays only the growth check (one 8-byte copy to the
                 host that the host waits for)
    grow_1024    a growing handle created at 1024 keys: it grows while the stream primes it

and prints one JSON line per variant: the per-call time over the timed steps (CUDA events around the whole run of calls) and, for
grow_1024, the time of every priming call that grew (CUDA events around that call) with the capacity before and after it. The first
call of every variant is timed as well: it also pays the handle's first-call setup, which a growth in the first call shares.

    python tools/key_growth_bench.py [--steps 130] [--warmup 8] [--bps 64]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH, NKEYS, WIN, SLIDE, NB = 65536, 65536, 4096, 64, 65
MAP = dict(map_kind=1, iadd=2, fscale=1.0000001, filt_kind=1, mod=1)
SIGMA = 0.5  # selectivity of the filter on the synthetic stream


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # (the numbers stand without it, but the report says so)
        return f"unknown ({e!r})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=130, help="timed steps (one wfb_ffat_process_cb call each)")
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--bps", type=int, default=64, help="batches of 65536 tuples per step")
    ap.add_argument("--ring", type=int, default=8, help="device-resident segments the steps cycle through")
    args = ap.parse_args()

    import torch
    from windflow_b200 import build, ops
    build.build()
    torch.cuda.set_device(0)
    seg_tuples = args.bps * BATCH
    f = ops.functors(**MAP)

    def segment(start):
        b = ops.gen_tuple64(start, seg_tuples, ops.KEY_UNIFORM, NKEYS)
        return ops.Segment([ops.DeviceBatch(b.tuples[i * BATCH * 64:(i + 1) * BATCH * 64], b.ts[i * BATCH:(i + 1) * BATCH], BATCH,
                                            watermark=start + i * BATCH) for i in range(args.bps)]), b

    gpu = card()
    B = (NB - 1) * SLIDE + WIN
    prime = int(np.ceil(B * NKEYS / SIGMA / seg_tuples)) + 2
    for name, max_keys, grow in (("fixed", NKEYS, False), ("grow_same", NKEYS, True), ("grow_1024", 1024, True)):
        ff = ops.FfatWindowsGPU(ops.PROG_TUPLE64, WIN, SLIDE, NB, max_keys=max_keys, grow_keys=grow)
        cap = (seg_tuples // (SLIDE * NB) + NKEYS + seg_tuples // B + 1) * NB  # the bound of the largest capacity the handle reaches
        out = torch.empty(cap * ff.res_dtype.itemsize, dtype=torch.uint8, device="cuda")
        out_ts = torch.empty(cap, dtype=torch.int64, device="cuda")
        n_out = torch.zeros(1, dtype=torch.int32, device="cuda")
        grew = []
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for t in range(prime):  # every key past its first trigger (untimed, except the calls that grow)
            seg, keep = segment(t * seg_tuples)
            before = ff.key_capacity
            torch.cuda.synchronize()
            e0.record()
            ff.process(seg, pre=f, out=out, out_ts=out_ts, n_out=n_out)
            e1.record()
            torch.cuda.synchronize()
            if t == 0:
                first_ms = e0.elapsed_time(e1)  # (the first call of every handle also pays its first-call setup)
            if ff.key_capacity != before:
                grew.append({"call": t, "capacity_before": before, "capacity_after": ff.key_capacity, "ms": e0.elapsed_time(e1)})
        ring = [segment((prime + i) * seg_tuples) for i in range(args.ring)]
        for i in range(args.warmup):
            ff.process(ring[i % args.ring][0], pre=f, out=out, out_ts=out_ts, n_out=n_out)
        torch.cuda.synchronize()
        r0 = ff.results_total()
        e0.record()
        for i in range(args.steps):
            ff.process(ring[i % args.ring][0], pre=f, out=out, out_ts=out_ts, n_out=n_out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        wins = ff.results_total() - r0
        nk, err = ff.stats()
        if err:
            raise SystemExit(f"key_growth_bench.py: {name}: device error flags {err}")
        print(json.dumps({"variant": name, "gpu": gpu, "call_ms": ms / args.steps, "tuples_per_s": args.steps * seg_tuples / (ms / 1e3),
                          "windows_per_call": wins / args.steps, "keys": nk, "key_capacity": ff.key_capacity, "first_call_ms": first_ms,
                          "growth_calls": grew}), flush=True)
        del ring, ff, out, out_ts
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
