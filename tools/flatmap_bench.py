"""FlatMap_GPU (wfb_flatmap_batches) throughput: calls of 128 batches of 65536 64-byte tuples (the bench stream of SURVEY.md 8d,
device-generated) through the test programs of tests/cpp/flatmap_programs.cu, one JSON line per configuration:

    fm64to32_m{1,4,16}   64-byte tuples -> 32-byte records, fan-out drawn uniformly from 0..m (mean m / 2)
    select64_m1          64-byte tuples -> the mapped tuple when the filter keeps it (m = 1, about half the tuples)
    map_filter           wfb_map_filter_batches of the built-in program with the same map and filter: the same bytes as select64_m1

Per call: the time (CUDA events around `--calls` calls after `--warmup` calls of the same shape; one call is one kernel plus a
memset of the counts and the copy of the batch table), input tuples/s, output records/s, and the algorithmic bytes (tuples +
timestamps read, records + timestamps written) over the call time as a fraction of 3.35 TB/s (H100 SXM HBM3, data sheet).
The card's name and power limit are printed with the numbers.

    python tools/flatmap_bench.py [--calls 20] [--warmup 3] [--batches 128]
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
HBM = 3.35e12
MAP = dict(map_kind=1, iadd=2, fscale=1.0000001, filt_kind=1, mod=1)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # (the numbers stand without it, but the report says so)
        return f"unknown ({e!r})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batches", type=int, default=128)
    args = ap.parse_args()

    import numpy as np
    import torch
    from windflow_b200 import build, ops
    import test_gpu_flatmap as T
    build.build()
    torch.cuda.set_device(0)
    L = T.fmlib()
    k, n_all = args.batches, args.batches * BATCH
    src = ops.gen_tuple64(0, n_all, ops.KEY_UNIFORM, 65536)
    words = src.tuples.view(torch.int64).view(n_all, 8)  # pad[3] is word 7: the fan-out of the FlatMap programs
    ins = [ops.DeviceBatch(src.tuples[i * BATCH * 64:(i + 1) * BATCH * 64], src.ts[i * BATCH:(i + 1) * BATCH], BATCH) for i in range(k)]
    gpu = card()

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
        return e0.elapsed_time(e1) / 1e3 / args.calls

    def outs(rb, m):
        return [ops.DeviceBatch(torch.empty(BATCH * m * rb, dtype=torch.uint8, device="cuda"),
                                torch.empty(BATCH * m, dtype=torch.int64, device="cuda"), BATCH * m) for _ in range(k)]

    def report(name, sec, records, rb):
        moved = n_all * (64 + 8) + records * (rb + 8)
        print(json.dumps({"config": name, "batches": k, "tuples": n_all, "records": int(records), "call_ms": round(sec * 1e3, 4),
                          "tuples_per_s": n_all / sec, "records_per_s": records / sec, "bytes": moved,
                          "hbm_fraction": round(moved / sec / HBM, 4), "gpu": gpu}), flush=True)

    f0 = ops.functors()
    for m in (1, 4, 16):
        gen = torch.Generator(device="cuda").manual_seed(m)
        words[:, 7] = torch.randint(0, m + 1, (n_all,), device="cuda", generator=gen)
        eng = ops.Engine(L.fm_register(1))
        o = outs(32, m)
        n_out = torch.zeros(k + 1, dtype=torch.int32, device="cuda")
        sec = timed(lambda: eng.flatmap_batches(ins, f0, o, n_out, m))
        c = n_out.cpu().numpy().astype(np.int64)
        assert c[-1] == 0
        report(f"fm64to32_m{m}", sec, int(c[:-1].sum()), 32)
        del o

    f = ops.functors(**MAP)
    eng = ops.Engine(L.fm_register(3))
    o = outs(64, 1)
    n_out = torch.zeros(k + 1, dtype=torch.int32, device="cuda")
    sec_fm = timed(lambda: eng.flatmap_batches(ins, f, o, n_out, 1))
    c_fm = n_out.cpu().numpy().astype(np.int64)[:-1]
    ref = ops.Engine(ops.PROG_TUPLE64)
    o2 = outs(64, 1)
    n2 = torch.zeros(k, dtype=torch.int32, device="cuda")
    sec_mf = timed(lambda: ref.map_filter_batches(ins, f, o2, n2))
    c_mf = n2.cpu().numpy().astype(np.int64)
    torch.cuda.synchronize()
    assert np.array_equal(c_fm, c_mf)
    same = all(torch.equal(a.tuples[:int(c) * 64], b.tuples[:int(c) * 64]) for a, b, c in zip(o, o2, c_mf))
    report("select64_m1", sec_fm, int(c_fm.sum()), 64)
    report("map_filter", sec_mf, int(c_mf.sum()), 64)
    print(json.dumps({"select64_m1_over_map_filter": round(sec_fm / sec_mf, 4), "identical_records": bool(same), "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
