"""GPU tests (-m gpu) of the wide partition's variants that the default configuration does not take: the bucket-move path
(WFB_BUCKET_MOVE=1: the partition moves the lifted records into their buckets, and the update reads the arrival position of a group's
triggering item from the partition's output to stamp its results) and the few-destination shard partition of an engine whose sorter
grows between calls (rows filed by the tile pass must survive when only the partition's chunk rows grow)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
FP_RTOL = 1e-6

MOVE_CASES = [  # win, slide, nb, nkeys, n, batch, batches per call
    (64, 16, 5, 600, 120000, 5000, 4),
    (4096, 64, 5, 20, 400000, 40000, 4),  # 160 000 positions per call: 40 wide tiles, two chunks of the partition
]


@pytest.mark.parametrize("pipelined", [False, True], ids=["direct", "pipelined"])
@pytest.mark.parametrize("case", MOVE_CASES, ids=[f"w{c[0]}_s{c[1]}_nb{c[2]}_k{c[3]}" for c in MOVE_CASES])
def test_bucket_move_results_and_timestamps_match_oracle(wfb, oracle, monkeypatch, case, pipelined):
    import torch
    O, ops = oracle, wfb
    win, slide, nb, nkeys, n, batch, group = case
    monkeypatch.setenv("WFB_BUCKET_MOVE", "1")  # read when the handle is created
    t, ts = O.gen_tuple64(0, n, O.KEY_UNIFORM, nkeys)
    ff = ops.FfatWindowsGPU(ops.PROG_TUPLE64, win, slide, nb, max_keys=nkeys, pipelined=pipelined)
    go = O.FfatGpuOracle(win, slide, nb)
    batches, exp, ets = [], [], []
    for b in range(0, n, batch):
        batches.append(ops.DeviceBatch.from_host(t[b:b + batch], ts[b:b + batch]))
        r, rt = go.process_batch(O.lift_tuple64(t[b:b + batch]), int(ts[b]))
        exp.append(r); ets.append(rt)
    got, gts = [], []
    calls = [batches[i:i + group] for i in range(0, len(batches), group)]
    for c in calls:
        out, out_ts, n_out = ff.process(c)
        torch.cuda.synchronize()
        r, rt = ff.results_to_host(out, out_ts, n_out)
        got.append(r); gts.append(rt)
    if pipelined:
        out, out_ts, n_out = ff.flush(device=batches[0].tuples.device)
        torch.cuda.synchronize()
        r, rt = ff.results_to_host(out, out_ts, n_out)
        got.append(r); gts.append(rt)
    g, gt = O.sort_results(np.concatenate(got), np.concatenate(gts))
    e, et = O.sort_results(np.concatenate(exp), np.concatenate(ets))
    assert len(g) == len(e) and len(e) > 0, (len(g), len(e))
    assert np.array_equal(g["key"], e["key"]) and np.array_equal(g["id"], e["id"])
    assert np.array_equal(g["isum"], e["isum"])
    assert np.allclose(g["fsum"], e["fsum"], rtol=FP_RTOL, atol=0)
    assert len(np.unique(et)) > 1  # the results come from several batches: a wrong triggering position shows in the timestamps
    assert np.array_equal(gt, et)
    assert ff.stats()[1] == 0


@pytest.mark.parametrize("shards", [1, 3])
def test_shard_partition_after_sorter_growth(wfb, oracle, shards):
    """One engine, a small call first and then one of 33 wide tiles: the tile pass files its rows for chunks of 32 tiles, the
    few-destination partition works on chunks of 16 and grows only its chunk rows."""
    import torch
    O, ops = oracle, wfb
    f = ops.functors(map_kind=1, iadd=2, fscale=1.0000001, filt_kind=1)
    eng = ops.Engine(ops.PROG_TUPLE64)
    start = 0
    for sizes in ([1000], [65536, 65536, 4097]):
        n = sum(sizes)
        t, ts = O.gen_tuple64(start, n, O.KEY_UNIFORM, 5000)
        start += n
        batches, off = [], 0
        for sz in sizes:
            batches.append(ops.DeviceBatch.from_host(t[off:off + sz], ts[off:off + sz]))
            off += sz
        regions = torch.zeros(shards * n * 32, dtype=torch.uint8, device="cuda")
        counts = torch.zeros(9, dtype=torch.int32, device="cuda")
        eng.shard_lift(batches, f, shards, regions, n, counts)
        torch.cuda.synchronize()
        surv, _, _ = O.map_filter_tuple64(t, ts, 1, 2, 1.0000001, 1)
        lifted = O.lift_tuple64(surv)
        dest = O.route(surv["key"], shards)
        c = counts.cpu().numpy()
        assert c[8] == 0
        got = ops.to_host(regions, ops.RESULT32).reshape(shards, n)
        for d in range(shards):
            exp = lifted[dest == d]
            assert c[d] == len(exp)
            assert got[d][:c[d]].tobytes() == exp.tobytes()
