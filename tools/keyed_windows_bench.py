"""Throughput of Keyed_Windows_GPU, three arms per workload, one JSON line each, with the GPU's name and power limit read in the same run:
  c_abi      wfb_kwin_process_cb on the program of tests/cpp/kwin_programs.cu (64-byte tuples, uint64_t key in the hashed key table,
             a window function that reads every tuple of the window); K = 8 batches of 65 536 tuples per call, keys uniform; the timed
             window is `calls` calls, ended by a device synchronise, after enough untimed calls for every key to hold a full window, plus
             `warmup`
  builder    windflow_b200/apps/keyed_windows_bench.bin: SourceGPU -> Map_GPU -> Filter_GPU -> Keyed_Windows_GPU -> Sink through the
             builder API, hashed keys, K = 128 batches per call, the same window function
  reference  the reference's CPU Keyed_Windows (oracle/_ref/ref_keyed_windows_cpu, built by tests/golden/make_golden_kw.py from a WindFlow
             checkout): Source -> Map -> Filter -> Keyed_Windows -> Sink, DETERMINISTIC mode, `par` replicas, the same window function, on
             this host's CPU (reported as unavailable when the program was not built)

    python tools/keyed_windows_bench.py [--calls N] [--warmup W] [--par P] [--ref-tuples N]

Workloads: 65 536 keys, win 1024 / slide 64 (a 4 GiB ring); 1 024 keys, win 64 / slide 16."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

WORKLOADS = [(65536, 1024, 64), (1024, 64, 16)]  # keys, win, slide
BATCH, K = 65536, 8
BUILDER = os.path.join(ROOT, "windflow_b200", "apps", "keyed_windows_bench.bin")
REFERENCE = os.path.join(ROOT, "oracle", "_ref", "ref_keyed_windows_cpu")


def gpu_card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--par", type=int, default=min(8, os.cpu_count() or 1), help="replicas of each reference CPU operator")
    ap.add_argument("--ref-tuples", type=int, default=1 << 22)
    a = ap.parse_args()
    import torch
    from windflow_b200 import ops
    import test_gpu_keyed_windows as T
    assert torch.cuda.is_available(), "the bench needs a CUDA device"
    prog = T.kwlib().kw_register(0)
    card = gpu_card()
    for keys, win, slide in WORKLOADS:
        kw = ops.KeyedWindowsGPU(prog, win, slide, keys)
        batches = []
        for i in range(K):
            batches.append(ops.gen_tuple64(i * BATCH, BATCH, key_mode=ops.KEY_UNIFORM, nkeys=keys))
        seg = ops.Segment(batches)
        cap = K * BATCH // slide + keys + 1
        out = torch.empty(cap * 72, dtype=torch.uint8, device="cuda")
        out_ts = torch.empty(cap, dtype=torch.int64, device="cuda")
        n_out = torch.zeros(1, dtype=torch.int32, device="cuda")
        # untimed: every key past its first window (win of its tuples) so that the timed calls fire windows at the steady rate
        prime = -(-win * keys // (K * BATCH)) + a.warmup
        for _ in range(prime):
            kw.process(seg, capacity=cap, out=out, out_ts=out_ts, n_out=n_out)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.calls):
            kw.process(seg, capacity=cap, out=out, out_ts=out_ts, n_out=n_out)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        nk, err = kw.stats()
        tuples = a.calls * K * BATCH
        print(json.dumps({"arm": "c_abi", "keys": keys, "win": win, "slide": slide, "batches_per_call": K, "batch": BATCH, "calls": a.calls,
                          "seconds": round(dt, 6), "tuples_per_s": round(tuples / dt, 1), "windows_last_call": int(n_out.cpu()[0]),
                          "ring_bytes": keys * (1 << (win - 1).bit_length()) * 64, "key_table": "hashed", "err_flags": err, "gpu": card}), flush=True)
        kw.close()
        del out, out_ts, batches, seg
        torch.cuda.empty_cache()
        arm("builder", [BUILDER, "128", "2048", str(keys), str(win), str(slide)], card)
        arm("reference", [REFERENCE, f"gen={a.ref_tuples}", f"keys={keys}", f"win={win}", f"slide={slide}", f"par={a.par}"], card,
            {"cpu_threads_available": os.cpu_count()})


def arm(name, cmd, card, extra=None):
    """Runs one arm's program and prints its JSON line with the card; an arm whose program was not built is reported as unavailable."""
    rec = {"arm": name, "gpu": card}
    if not os.path.exists(cmd[0]):
        rec["unavailable"] = f"{os.path.relpath(cmd[0], ROOT)} was not built"
    else:
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
        line = [x for x in p.stdout.splitlines() if x.startswith("{")]
        if p.returncode != 0 or not line:
            raise RuntimeError(f"{name} arm failed ({p.returncode}): {p.stdout[-2000:]}{p.stderr[-2000:]}")
        rec.update(json.loads(line[-1]))
    rec.update(extra or {})
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
