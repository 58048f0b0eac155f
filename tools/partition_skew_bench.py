"""Count-based windows on the bucket path with few or skewed keys, where the wide partition's cells are long: ms per call of
64 batches of 65 536 24-byte records (`PROG_WFWIN24`, win 256, slide 64, Nb 1) for 16 uniform keys, Zipf-1.3 keys over 65 536 and
65 536 uniform keys. CUDA events around 20 calls after 3 warm-up calls; WFB_LIB selects another build of the library."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from windflow_b200 import ops  # noqa: E402

BATCH, BPC, CALLS, WARM = 65536, 64, 20, 3


def main():
    rng = np.random.default_rng(5)
    n = BATCH * BPC
    for name, keys_np, nkeys in (("16 uniform keys", rng.integers(0, 16, n), 16),
                                 ("Zipf-1.3 over 65536 keys", (rng.zipf(1.3, n) - 1) % 65536, 65536),
                                 ("65536 uniform keys", rng.integers(0, 65536, n), 65536)):
        keys = torch.from_numpy(keys_np.astype(np.int64)).cuda()
        idx = torch.arange(n, dtype=torch.int64, device="cuda")
        rec = torch.stack([keys, torch.zeros_like(idx), idx + 1], dim=1).contiguous().view(torch.uint8).reshape(-1)
        batches = [ops.DeviceBatch(rec[b * BATCH * 24:(b + 1) * BATCH * 24], None, BATCH, watermark=b) for b in range(BPC)]
        ff = ops.FfatWindowsGPU(ops.PROG_WFWIN24, 256, 64, 1, max_keys=nkeys, dense_keys=True)
        for _ in range(WARM):
            ff.process(batches)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(CALLS):
            ff.process(batches)
        e1.record()
        torch.cuda.synchronize()
        assert ff.stats()[1] == 0
        ms = e0.elapsed_time(e1) / CALLS
        print(json.dumps({"config": name, "ms_per_call": ms, "tuples_per_s": n / ms * 1e3}))


if __name__ == "__main__":
    main()
