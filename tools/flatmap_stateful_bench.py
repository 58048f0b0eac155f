"""Keyed-stateful FlatMap_GPU (wfb_flatmap_stateful) throughput next to the keyed-stateful Filter_GPU (wfb_filter_stateful) at the same
configuration: calls of 64 or 128 batches of 65536 64-byte tuples (the bench stream of SURVEY.md 8d, device-generated) through the
test programs of tests/cpp/stateful_flatmap_programs.cu, one JSON line per configuration:

    keys     65536 uniform keys (the bucket path), 2^20 uniform keys (the full sort), 65536 Zipf-0.8 keys
    m = 1    the selection program (the tuple iff ProgTuple64::filter_stateful holds): the bytes of wfb_filter_stateful
    m = 4    64-byte tuples -> 32-byte records, (count + ivalue) % 5 records per tuple (2 on average)
    filter   wfb_filter_stateful of the built-in program with the selection's functors

Per call: the time (CUDA events around `--calls` calls after `--warmup` calls of the same shape, the key states carried from call to
call) and input tuples/s. `--profile` instead traces a few calls of each m at 65536 uniform keys and 128 batches with torch.profiler
and splits the kernel time into phases: slots, partition, count walk, offsets, emit walk. The card's name and power limit are printed
with the numbers.

    python tools/flatmap_stateful_bench.py [--calls 10] [--warmup 3] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BATCH = 65536
SEL = dict(map_kind=0, iadd=0, fscale=1.0, filt_kind=1, mod=1)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # (the numbers stand without it, but the report says so)
        return f"unknown ({e!r})"


def phase(name):
    if "k_ks_slots" in name:
        return "slots"
    if "k_ks_apply" in name:
        return "count walk" if name.split(">")[0].rstrip().endswith(", 2") else ("emit walk" if name.split(">")[0].rstrip().endswith(", 3") else "walk")
    if "k_flag_" in name or "k_scan_u32" in name or "k_fm_offsets" in name:
        return "offsets"
    if "emset" in name or "Memset" in name or "Memcpy" in name:
        return "memset / copy"
    return "partition"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()

    import torch
    from windflow_b200 import build, ops
    from oracle.oracle import zipf_cdf
    import test_gpu_flatmap_stateful as T
    build.build()
    torch.cuda.set_device(0)
    progs = {w: T.sfmlib().sfm_register(w) for w in (0, 3)}
    gpu = card()
    kmax = 128
    outs = {1: [ops.DeviceBatch(torch.empty(BATCH * 64, dtype=torch.uint8, device="cuda"), torch.empty(BATCH, dtype=torch.int64, device="cuda"), BATCH)
                for _ in range(kmax)],
            4: [ops.DeviceBatch(torch.empty(BATCH * 4 * 32, dtype=torch.uint8, device="cuda"), torch.empty(BATCH * 4, dtype=torch.int64, device="cuda"),
                                BATCH * 4) for _ in range(kmax)]}
    n_out = torch.zeros(kmax + 1, dtype=torch.int32, device="cuda")

    def stream_of(keys, dist):
        cdf = torch.from_numpy(zipf_cdf(keys)).cuda() if dist == "zipf" else None
        src = ops.gen_tuple64(0, kmax * BATCH, ops.KEY_ZIPF if cdf is not None else ops.KEY_UNIFORM, keys, zipf_cdf=cdf)
        return [ops.DeviceBatch(src.tuples[i * BATCH * 64:(i + 1) * BATCH * 64], src.ts[i * BATCH:(i + 1) * BATCH], BATCH) for i in range(kmax)]

    def op_call(arm, keys, ins):
        if arm == "filter":
            ks, f = ops.KeyedState(ops.PROG_TUPLE64, keys), ops.functors(**SEL)
            return lambda: ks.filter(ins, f, outs[1][:len(ins)], n_out)
        m = 1 if arm == "m1" else 4
        ks = ops.KeyedState(progs[3 if m == 1 else 0], keys)
        f = ops.functors(**SEL) if m == 1 else T.functors(mod=m + 1)
        return lambda: ks.flatmap(ins, f, outs[m][:len(ins)], n_out, m)

    def timed(call):
        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.calls):
            call()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.calls

    if args.profile:
        from torch.profiler import profile, ProfilerActivity
        ins = stream_of(65536, "uniform")
        for arm in ("m1", "m4", "filter"):
            call = op_call(arm, 65536, ins)
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.calls):
                    call()
                torch.cuda.synchronize()
            split = {}
            for ev in prof.key_averages():
                if ev.device_time_total > 0:
                    split[phase(ev.key)] = split.get(phase(ev.key), 0.0) + ev.device_time_total / 1e3 / args.calls
            print(json.dumps({"arm": arm, "keys": 65536, "batches": kmax, "ms_per_call_by_phase": {k: round(v, 4) for k, v in sorted(split.items())},
                              "gpu": gpu}), flush=True)
        return

    for keys, dist in ((65536, "uniform"), (1 << 20, "uniform"), (65536, "zipf")):
        stream = stream_of(keys, dist)
        for k in (64, 128):
            ins = stream[:k]
            for arm in ("m1", "m4", "filter"):
                ms = timed(op_call(arm, keys, ins))
                print(json.dumps({"arm": arm, "keys": keys, "dist": dist, "batches": k, "ms_per_call": round(ms, 3),
                                  "gtuples_per_s": round(k * BATCH / ms / 1e6, 3), "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
