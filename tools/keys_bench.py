"""Cost of keys that are not integers: the count-based Ffat_Windows_GPU bench configuration (Map -> Filter -> windows 4096 / 64,
Nb 65, 65536 uniform keys, batches of 65536 tuples) over the same device-resident stream with

    tuple64_dense  PROG_TUPLE64, dense keys (slot = key: what bench.py runs)
    tuple64_hash   PROG_TUPLE64 through the key table (8-byte entries)
    fkey_hash      PROG_TUPLE64_FKEY: a double key per key index (8-byte entries)
    k16_hash       PROG_TUPLE64_K16: {key, pad[0]}, a 16-byte key per key index (16-byte entries, 16-byte CAS)

and prints one JSON line per variant: tuples/s over the timed steps (CUDA events) and the per-call phase times of wfb_ffat_timing
(ingest = the tile pass that looks the keys up). Every key is first driven past its first trigger, so the timed steps fire windows.

    python tools/keys_bench.py [--steps 130] [--warmup 8] [--bps 64]
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
    ap.add_argument("--steps", type=int, default=130, help="timed steps (130 steps of 64 batches: every key fires about once)")
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--bps", type=int, default=64, help="batches of 65536 tuples per step (one wfb_ffat_process_cb call)")
    ap.add_argument("--ring", type=int, default=8, help="device-resident segments the steps cycle through")
    args = ap.parse_args()

    import torch
    from windflow_b200 import build, ops
    build.build()
    torch.cuda.set_device(0)
    seg_tuples = args.bps * BATCH
    rng = np.random.default_rng(1)
    hi = torch.from_numpy(rng.integers(1, 1 << 62, NKEYS, dtype=np.int64)).cuda()                 # K16: high word per key index
    fk = torch.from_numpy((np.arange(NKEYS) * 0.25 - 8191.75).view(np.int64).copy()).cuda()      # FKEY: a distinct double per key index
    f = ops.functors(**MAP)

    def segment(start, table):
        b = ops.gen_tuple64(start, seg_tuples, ops.KEY_UNIFORM, NKEYS)
        if table is not None:
            v = b.tuples.view(torch.int64).view(-1, 8)
            v[:, 4] = table[v[:, 0]]
        return ops.Segment([ops.DeviceBatch(b.tuples[i * BATCH * 64:(i + 1) * BATCH * 64], b.ts[i * BATCH:(i + 1) * BATCH], BATCH,
                                            watermark=start + i * BATCH) for i in range(args.bps)]), b

    variants = [("tuple64_dense", ops.PROG_TUPLE64, True, None), ("tuple64_hash", ops.PROG_TUPLE64, False, None),
                ("fkey_hash", ops.PROG_TUPLE64_FKEY, False, fk), ("k16_hash", ops.PROG_TUPLE64_K16, False, hi)]
    gpu = card()
    B = (NB - 1) * SLIDE + WIN
    prime = int(np.ceil(B * NKEYS / SIGMA / seg_tuples)) + 2
    for name, prog, dense, table in variants:
        ff = ops.FfatWindowsGPU(prog, WIN, SLIDE, NB, max_keys=NKEYS, dense_keys=dense)
        cap = ff.max_results(seg_tuples)
        out = torch.empty(cap * ff.res_dtype.itemsize, dtype=torch.uint8, device="cuda")
        out_ts = torch.empty(cap, dtype=torch.int64, device="cuda")
        n_out = torch.zeros(1, dtype=torch.int32, device="cuda")
        t = 0
        for _ in range(prime):  # every key past its first trigger (untimed)
            seg, keep = segment(t * seg_tuples, table)
            ff.process(seg, pre=f, out=out, out_ts=out_ts, n_out=n_out)
            t += 1
        ring = [segment((t + i) * seg_tuples, table) for i in range(args.ring)]
        for i in range(args.warmup):
            ff.process(ring[i % args.ring][0], pre=f, out=out, out_ts=out_ts, n_out=n_out)
        torch.cuda.synchronize()
        r0 = ff.results_total()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            ff.process(ring[i % args.ring][0], pre=f, out=out, out_ts=out_ts, n_out=n_out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        wins = ff.results_total() - r0
        ff.timing(True)
        for i in range(16):
            ff.process(ring[i % args.ring][0], pre=f, out=out, out_ts=out_ts, n_out=n_out)
        torch.cuda.synchronize()
        ing, srt, upd, tot, calls = ff.timing(False)
        nk, err = ff.stats()
        if err:
            raise SystemExit(f"keys_bench.py: {name}: device error flags {err}")
        print(json.dumps({"variant": name, "program": prog, "gpu": gpu, "tuples_per_s": args.steps * seg_tuples / (ms / 1e3),
                          "step_ms": ms / args.steps, "windows_per_step": wins / args.steps, "keys": nk,
                          "phase_ms_per_call": {"ingest_tile_pass": ing / calls, "sort": srt / calls, "update": upd / calls, "call": tot / calls}}),
              flush=True)
        del ring, ff, out, out_ts
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
