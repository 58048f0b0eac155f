"""Keyed_Windows_GPU pinned to the reference: tests/golden/ref_cpu_kw_*.npz hold what the unmodified reference's Source -> Map -> Filter ->
Keyed_Windows (count-based, DETERMINISTIC mode) -> Sink emitted on a seeded stream (tests/golden/make_golden_kw.py): the fired windows
with the timestamp of their firing tuple, then the end-of-stream windows with the largest timestamp seen. Geometries: sliding, tumbling
and hopping windows, win not a power of two.

CPU (-m "not gpu"): the stored outputs equal the Python model of tests/test_gpu_keyed_windows.py, and every key's windows arrived in
order. GPU: the same stream through Map_GPU -> Filter_GPU (wfb_map_filter_batches) -> Keyed_Windows_GPU (wfb_kwin_process_cb, then
wfb_kwin_flush) gives the stored results: integers and timestamps exact, sums within 1e-12 relative."""
import glob
import os

import numpy as np
import pytest

from test_gpu_keyed_windows import RES, Model, kwlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "ref_cpu_kw_*.npz")))
INT_FIELDS = ("key", "id", "hash", "size", "mid", "front", "back", "distinct")


def load(path):
    z = np.load(path)
    win, slide = (int(x) for x in z["geometry"])
    return z["tuples"], z["ts"], z["results"], win, slide


def map_filter(t, ts):
    """Map ivalue += 2, fvalue *= 1.0000001, then Filter (ivalue & 1) == 0 (the functors of the reference run)."""
    u = t.copy()
    u["ivalue"] += 2
    u["fvalue"] *= 1.0000001
    keep = (u["ivalue"] & 1) == 0
    return u[keep], ts[keep]


def rows(res, ts=None):
    ts = res["ts"] if ts is None else ts
    return sorted((int(r["key"]), int(r["id"])) + tuple(int(r[f]) for f in INT_FIELDS[2:]) + (float(r["fsum"]), int(t)) for r, t in zip(res, ts))


def same(got, exp):
    assert len(got) == len(exp) > 0
    for g, e in zip(got, exp):
        assert g[:8] == e[:8] and g[9] == e[9], (g, e)
        assert g[8] == pytest.approx(e[8], rel=1e-12, abs=0), (g, e)


def test_golden_files_present():
    names = [os.path.basename(f) for f in FILES]
    assert any("slide" in n for n in names) and any("tumble" in n for n in names) and any("hop" in n for n in names), names


@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(f)[:-4] for f in FILES])
def test_reference_matches_model(path):
    t, ts, res, win, slide = load(path)
    u, uts = map_filter(t, ts)
    m = Model(0, win, slide)
    exp = sorted(m.feed(u, uts) + m.flush())
    same(rows(res), exp)
    nxt = {}
    for k, g in zip(res["key"].tolist(), res["id"].tolist()):  # every key's windows reach the Sink in order
        assert g == nxt.get(k, 0), (k, g)
        nxt[k] = g + 1
    assert any(int(r["size"]) < win for r in res)  # end-of-stream windows are part of the outputs


@pytest.mark.gpu
@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(f)[:-4] for f in FILES])
@pytest.mark.parametrize("K", [1, 4])
def test_gpu_matches_reference(wfb, path, K):
    import torch
    t, ts, res, win, slide = load(path)
    prog = kwlib().kw_register(0)
    eng = wfb.Engine(wfb.PROG_TUPLE64)
    f = wfb.functors(map_kind=1, iadd=2, fscale=1.0000001, filt_kind=1)
    kw = wfb.KeyedWindowsGPU(prog, win, slide, 64)
    B = 257
    ins = [wfb.DeviceBatch.from_host(t[i:i + B], ts[i:i + B]) for i in range(0, len(t), B)]
    got_r, got_ts = [], []

    def collect(out, out_ts, n_out):
        torch.cuda.synchronize()
        n = int(n_out.cpu()[0])
        got_r.append(out.cpu().numpy().view(RES[0])[:n].copy())
        got_ts.append(out_ts.cpu().numpy().view(np.uint64)[:n].copy())

    for c in range(0, len(ins), K):
        grp = ins[c:c + K]
        outs = [wfb.DeviceBatch(torch.empty_like(b.tuples), torch.empty_like(b.ts), b.n, b.watermark) for b in grp]
        n_out = torch.zeros(len(grp), dtype=torch.int32, device="cuda")
        eng.map_filter_batches(grp, f, outs, n_out)
        counts = n_out.cpu().tolist()
        for o, n in zip(outs, counts):
            o.n = n
        collect(*kw.process(outs))
    collect(*kw.flush(64 * (-(-win // slide))))
    assert kw.stats()[1] == 0
    same(rows(np.concatenate(got_r), np.concatenate(got_ts)), rows(res))
