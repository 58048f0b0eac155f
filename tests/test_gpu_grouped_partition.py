"""The wide partition's grouped scatter (k_wide_scatter_ranked: four wide tiles per CTA, used from 4 wide tiles per SM on) against the
per-tile scatter (k_wide_scatter_ranked_tile, which smaller calls take) and a direct computation of every window.

One stream is fed twice to count-based windows on the bucket path: as one call just below, at and above the switch to groups --
including a partial last group and a partial last wide tile -- and as calls of 64 Ki tuples, which stay per tile. The record's value
is its index in the stream, so an item placed out of arrival order moves across a window edge and changes a sum. Few keys (16: every
digit is one key, parts of hundreds of items) and Zipf-skewed keys over 65 536 exercise long parts; 4096 uniform keys short ones.
"""
import numpy as np
import pytest

WIN, SLIDE = 256, 64
SMALL = 65536


def _stream(dist, n, seed=3):
    rng = np.random.default_rng(seed)
    if dist == "few16":
        return rng.integers(0, 16, n), 16
    if dist == "zipf":
        return (rng.zipf(1.3, n) - 1) % 65536, 65536
    return rng.integers(0, 4096, n), 4096


def _records(torch, keys, b0, m):
    idx = torch.arange(b0, b0 + m, dtype=torch.int64, device="cuda")
    rec = torch.stack([keys[b0:b0 + m], torch.zeros_like(idx), idx + 1], dim=1).contiguous()
    return rec.view(torch.uint8).reshape(-1)


def _run(ops, torch, keys, n, nkeys, call):
    ff = ops.FfatWindowsGPU(ops.PROG_WFWIN24, WIN, SLIDE, 1, max_keys=nkeys, dense_keys=True)
    outs, outts = [], []
    for c0 in range(0, n, call):
        m = min(call, n - c0)
        out, out_ts, n_out = ff.process([ops.DeviceBatch(_records(torch, keys, c0, m), None, m, watermark=7)])
        torch.cuda.synchronize()
        r, rt = ff.results_to_host(out, out_ts, n_out)
        outs.append(r); outts.append(rt)
    assert ff.stats()[1] == 0
    got, ts = np.concatenate(outs), np.concatenate(outts)
    order = np.lexsort((got["id"], got["key"]))
    return got[order], ts[order]


def _expected(keys_np):
    """(key, window id, sum) of every complete window: values are stream index + 1, windows are arrival ranks [w*SLIDE, w*SLIDE+WIN)."""
    order = np.argsort(keys_np, kind="stable")
    k, v = keys_np[order], order.astype(np.int64) + 1
    heads = np.flatnonzero(np.r_[True, k[1:] != k[:-1]])
    ends = np.r_[heads[1:], len(k)]
    ek, ei, es = [], [], []
    for h, e in zip(heads, ends):
        cnt = e - h
        if cnt < WIN:
            continue
        cs = np.r_[0, np.cumsum(v[h:e])]
        w = np.arange((cnt - WIN) // SLIDE + 1)
        ek.append(np.full(len(w), k[h])); ei.append(w); es.append(cs[w * SLIDE + WIN] - cs[w * SLIDE])
    return np.concatenate(ek), np.concatenate(ei), np.concatenate(es)


@pytest.mark.gpu
@pytest.mark.parametrize("dist", ["few16", "zipf", "uniform"])
@pytest.mark.parametrize("tiles_over", [-1, 0, 2])
def test_grouped_scatter_matches_per_tile_and_direct_windows(wfb, dist, tiles_over):
    import torch
    ops = wfb
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    wide = 4 * sms + tiles_over                        # wide tiles of the one-call feed (4096 positions each); grouped from 4 per SM
    n = wide * 4096 - (0 if tiles_over <= 0 else 4096 - 123)  # tiles_over = 2: a partial last group whose last wide tile holds 123 tuples
    keys_np, nkeys = _stream(dist, n)
    keys = torch.from_numpy(keys_np.astype(np.int64)).cuda()
    big, big_ts = _run(ops, torch, keys, n, nkeys, n)
    small, small_ts = _run(ops, torch, keys, n, nkeys, SMALL)
    assert big.tobytes() == small.tobytes() and np.array_equal(big_ts, small_ts)
    ek, ei, es = _expected(keys_np)
    assert len(big) == len(ek) > 0
    assert np.array_equal(big["key"].astype(np.int64), ek) and np.array_equal(big["id"].astype(np.int64), ei)
    assert np.array_equal(big["value"].astype(np.int64), es)
