"""Throughput of Keyed_Windows_GPU, non-incremental and incremental, one JSON line per arm and workload, with the GPU's name, power
limit and max SM clock read in the same run:
  c_abi      wfb_kwin_process_cb on the program of tests/cpp/kwin_programs.cu (64-byte tuples, uint64_t key in the hashed key table,
             a window function that reads every tuple of the window); K = 8 batches of 65 536 tuples per call, keys uniform; the timed
             window is `calls` calls, ended by a device synchronise, after enough untimed calls for every key to hold a full window, plus
             `warmup`
  builder    windflow_b200/apps/keyed_windows_bench.bin: SourceGPU -> Map_GPU -> Filter_GPU -> Keyed_Windows_GPU -> Sink through the
             builder API, hashed keys, K = 128 batches per call, the same window function
  reference  the reference's CPU Keyed_Windows (oracle/_ref/ref_keyed_windows_cpu, built by tests/golden/make_golden_kw.py from a WindFlow
             checkout): Source -> Map -> Filter -> Keyed_Windows -> Sink, DETERMINISTIC mode, `par` replicas, the same window function, on
             this host's CPU (reported as unavailable when the program was not built)
  c_abi_inc, builder_inc, reference_inc
             the same three on an incremental handle (WFB_KWIN_INCREMENTAL) with the fold of tests/cpp/kwin_inc_programs.cu
             (80-byte results; the reference arm runs oracle/_ref/ref_keyed_windows_inc_cpu, built by tests/golden/make_golden_kwi.py).
             The C ABI arms of a workload alternate, `rounds` times each, on the same card.
             c_abi_inc also reports the windows fired during its timed calls.

    python tools/keyed_windows_bench.py [--calls N] [--warmup W] [--par P] [--ref-tuples N] [--rounds R]

Workloads: 65 536 keys, win 1024 / slide 64 (a 4 GiB ring); 1 024 keys, win 64 / slide 16; and, incremental only, 65 536 keys, win
2^20 / slide 2^18 (4 accumulators per key, 20 MiB; the ring of the non-incremental handle would be 4 TiB): a key fires its first window
after 2^20 of its own tuples, so that workload measures the fold into open windows."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

WORKLOADS = [(65536, 1024, 64, False), (1024, 64, 16, False), (65536, 1 << 20, 1 << 18, True)]  # keys, win, slide, incremental only
BATCH, K = 65536, 8
BUILDER = os.path.join(ROOT, "windflow_b200", "apps", "keyed_windows_bench.bin")
REFERENCE = os.path.join(ROOT, "oracle", "_ref", "ref_keyed_windows_cpu")
REFERENCE_INC = os.path.join(ROOT, "oracle", "_ref", "ref_keyed_windows_inc_cpu")


def gpu_card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--par", type=int, default=min(8, os.cpu_count() or 1), help="replicas of each reference CPU operator")
    ap.add_argument("--ref-tuples", type=int, default=1 << 22)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the two C ABI arms per workload")
    a = ap.parse_args()
    import torch
    from windflow_b200 import ops
    import test_gpu_keyed_windows as T
    import test_gpu_keyed_windows_inc as TI
    assert torch.cuda.is_available(), "the bench needs a CUDA device"
    progs = {False: (T.kwlib().kw_register(0), 72), True: (TI.kwilib().kwi_register(0), 80)}
    card = gpu_card()
    for keys, win, slide, inc_only in WORKLOADS:
        batches = [ops.gen_tuple64(i * BATCH, BATCH, key_mode=ops.KEY_UNIFORM, nkeys=keys) for i in range(K)]
        seg = ops.Segment(batches)
        for _ in range(a.rounds):
            for inc in ((True,) if inc_only else (False, True)):
                c_abi(ops, torch, seg, progs[inc], inc, keys, win, slide, a, card)
        del batches, seg
        torch.cuda.empty_cache()
        for inc in ((True,) if inc_only else (False, True)):
            sfx = "_inc" if inc else ""
            arm("builder" + sfx, [BUILDER, "128", "2048", str(keys), str(win), str(slide), "256", str(int(inc))], card)
            arm("reference" + sfx, [REFERENCE_INC if inc else REFERENCE, f"gen={a.ref_tuples}", f"keys={keys}", f"win={win}", f"slide={slide}", f"par={a.par}"],
                card, {"cpu_threads_available": os.cpu_count()})


def c_abi(ops, torch, seg, prog, inc, keys, win, slide, a, card):
    """`calls` timed calls of K batches on one handle, after enough untimed calls for every key to hold a full window (at most 256)."""
    prog_id, rb = prog
    kw = ops.KeyedWindowsGPU(prog_id, win, slide, keys, incremental=inc)
    cap = K * BATCH // slide + keys + 1
    out = torch.empty(cap * rb, dtype=torch.uint8, device="cuda")
    out_ts = torch.empty(cap, dtype=torch.int64, device="cuda")
    n_out = torch.zeros(1, dtype=torch.int32, device="cuda")
    fired = torch.zeros(1, dtype=torch.int64, device="cuda")
    prime = min(-(-win * keys // (K * BATCH)), 256) + a.warmup
    for _ in range(prime):
        kw.process(seg, capacity=cap, out=out, out_ts=out_ts, n_out=n_out)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.calls):
        kw.process(seg, capacity=cap, out=out, out_ts=out_ts, n_out=n_out)
        fired += n_out  # (on the device, in stream order: no host synchronisation inside the timed window)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    nk, err = kw.stats()
    tuples = a.calls * K * BATCH
    C = 1 << ((-(-win // slide) if inc else win) - 1).bit_length()
    print(json.dumps({"arm": "c_abi_inc" if inc else "c_abi", "keys": keys, "win": win, "slide": slide, "batches_per_call": K, "batch": BATCH,
                      "calls": a.calls, "primed_calls": prime, "seconds": round(dt, 6), "tuples_per_s": round(tuples / dt, 1),
                      "windows_timed": int(fired.cpu()[0]), "windows_last_call": int(n_out.cpu()[0]),
                      ("state_bytes" if inc else "ring_bytes"): keys * C * (rb if inc else 64), "key_table": "hashed", "err_flags": err,
                      "gpu": card}), flush=True)
    kw.close()


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
