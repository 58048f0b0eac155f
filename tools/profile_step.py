"""Per-kernel table of the bench step from torch.profiler, steady-state launches only.

Runs `bench.py` in this process under torch.profiler (CUDA activities) with the arguments given after `--`, then prints, for every
kernel of the window operator, the mean and median duration over its last `--last` launches (the priming launches at the start of
the run are left out). Example: `python tools/profile_step.py --last 64 -- --no-extras --steps 65`.
"""
import argparse
import collections
import json
import os
import re
import runpy
import statistics
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--last", type=int, default=64, help="launches per kernel to average, counted from the end of the run")
    ap.add_argument("--out", default=None, help="also write the table as JSON here")
    ap.add_argument("bench_args", nargs=argparse.REMAINDER)
    a = ap.parse_args()
    bargs = [x for x in a.bench_args if x != "--"]
    sys.argv = [os.path.join(ROOT, "bench.py")] + bargs
    sys.path.insert(0, ROOT)
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        try:
            runpy.run_path(sys.argv[0], run_name="__main__")
        except SystemExit as e:
            if e.code not in (None, 0):
                raise
        torch.cuda.synchronize()
    by_name = collections.defaultdict(list)
    events = prof.events()
    for ev in events:
        if ev.device_type != torch.autograd.DeviceType.CPU and re.match(r"(void )?(wfb::)?k_", ev.name):
            by_name[ev.name].append((ev.time_range.start, ev.time_range.end - ev.time_range.start))
    rows = []
    for name, evs in by_name.items():
        evs.sort()
        durs = [d for _, d in evs[-a.last:]]
        rows.append({"kernel": name[:140], "launches": len(evs), "averaged": len(durs), "mean_us": statistics.fmean(durs), "median_us": statistics.median(durs)})
    if not rows:
        raise SystemExit(f"profile_step.py: no kernel of the library among {len(events)} profiler events")
    rows.sort(key=lambda r: -r["mean_us"] * r["averaged"])
    for r in rows:
        print(f"{r['mean_us']:9.1f} {r['median_us']:9.1f}  {r['averaged']:4d}/{r['launches']:<5d} {r['kernel']}")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
