#!/usr/bin/env python
"""Phase timeline of k_ffat_update_buckets at the bench configuration (128 batches of 65 536 tuples per call).
Needs WFB_LIB=<build with -DWFB_BK_TRACE>: per CTA, the start and end (globaltimer) and the time thread 0 spends in each phase,
summed over the bucket's chunks."""
import ctypes as C, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from windflow_b200 import ops, _lib
BATCH, WIN, SLIDE, NB, BPS = 65536, 4096, 64, 65, 128
NKEYS = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
f = ops.functors(map_kind=1, iadd=2, fscale=1.0000001, filt_kind=1, mod=1)
ff = ops.FfatWindowsGPU(ops.PROG_TUPLE64, WIN, SLIDE, NB, max_keys=NKEYS, dense_keys=True)
cap = ff.max_results(BPS * BATCH)
out = torch.empty(cap * 32, dtype=torch.uint8, device="cuda"); out_ts = torch.empty(cap, dtype=torch.int64, device="cuda")
n_out = torch.zeros(1, dtype=torch.int32, device="cuda")
ff.timing(True)
for step in range(6 * (65536 // NKEYS)):
    b = ops.gen_tuple64(step * BPS * BATCH, BPS * BATCH, ops.KEY_UNIFORM, NKEYS)
    batches = [ops.DeviceBatch(b.tuples[i * BATCH * 64:(i + 1) * BATCH * 64], b.ts[i * BATCH:(i + 1) * BATCH], BATCH, watermark=i) for i in range(BPS)]
    ff.process(batches, pre=f, out=out, out_ts=out_ts, n_out=n_out)
torch.cuda.synchronize()
print('keys', NKEYS, 'phase ms (ingest, partition, update, call, calls):', [round(x, 3) for x in ff.timing(False)])
L = _lib.lib()
buf = (C.c_ulonglong * (1024 * 8))()
L.wfb_debug_bk_trace.restype = C.c_int
assert L.wfb_debug_bk_trace(buf) == 0
t = np.frombuffer(buf, dtype=np.uint64).reshape(1024, 8).astype(np.int64)
t = t[t[:, 7] > t[:, 0]]  # CTAs of the last launch (all of them, unless a bucket was empty)
t0 = t[:, 0].min()
names = ["prologue (range, key counts, state)", "split (bucket list, ranks)", "scans + place + gather", "fold (thread per segment)",
         "panes (leaves, paths, groups)", "tiny-pane warp fold + chunk end"]
print("kernel span us:", (t[:, 7].max() - t0) / 1e3)
for i, nme in enumerate(names):
    d = t[:, i + 1] / 1e3
    print(f"{nme:36s} mean {d.mean():7.2f}  p50 {np.median(d):7.2f}  p90 {np.percentile(d, 90):7.2f}  max {d.max():7.2f} us")
life = (t[:, 7] - t[:, 0]) / 1e3
wb = life - t[:, 1:7].sum(axis=1) / 1e3
print(f"{'write-back':36s} mean {wb.mean():7.2f} us")
print("CTA lifetime mean %.2f p50 %.2f max %.2f us" % (life.mean(), np.median(life), life.max()))
st = np.sort((t[:, 0] - t0) / 1e3)
print("CTA start times us: p10 %.1f p50 %.1f p60 %.1f p75 %.1f p90 %.1f max %.1f" % tuple(np.percentile(st, [10, 50, 60, 75, 90, 100])))
