"""The incremental Keyed_Windows_GPU pinned to the reference: tests/golden/ref_cpu_kwi_*.npz hold what the unmodified reference's
Source -> Map -> Filter -> Keyed_Windows (count-based, DETERMINISTIC mode, the incremental function void(const tuple_t &, result_t &) of
tests/cpp/kwin_inc_programs.cu) -> Sink emitted (tests/golden/make_golden_kwi.py runs tests/golden/ref_keyed_windows_inc.cpp), on the
same streams as ref_cpu_kw_*.npz.

CPU (-m "not gpu"): the stored outputs equal the incremental model of tests/test_gpu_keyed_windows_inc.py, every key's windows arrived in
order with the end-of-stream windows present, and they equal the non-incremental reference run (ref_cpu_kw_*.npz) on every field both
carry: key, id, hash, size, front, back, fsum, timestamp, and popcount(mask) = distinct. GPU: the same stream through Map_GPU ->
Filter_GPU (wfb_map_filter_batches) -> incremental Keyed_Windows_GPU gives the stored results: integers and timestamps exact, sums
within 1e-12 relative."""
import glob
import os

import numpy as np
import pytest

from test_gpu_keyed_windows_inc import RES, IncModel, kwilib
from test_keyed_windows_golden import map_filter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "ref_cpu_kwi_*.npz")))
INT_FIELDS = ("key", "id", "hash", "size", "front", "back", "mask", "argmax", "maxiv")


def load(path):
    z = np.load(path)
    win, slide = (int(x) for x in z["geometry"])
    return z["tuples"], z["ts"], z["results"], win, slide


def rows(res, ts=None):
    """(key, id, hash, size, front, back, mask, argmax, maxiv, fsum, ts) per result, sorted."""
    ts = res["ts"] if ts is None else ts
    return sorted(tuple(int(r[f]) for f in INT_FIELDS) + (float(r["fsum"]), int(t)) for r, t in zip(res, ts))


def same(got, exp):
    assert len(got) == len(exp) > 0
    for g, e in zip(got, exp):
        assert g[:9] == e[:9] and g[10] == e[10], (g, e)
        assert g[9] == pytest.approx(e[9], rel=1e-12, abs=0), (g, e)


def model_rows(u, uts, win, slide):
    m = IncModel(0, win, slide)
    out = []
    for r in m.feed(u, uts) + m.flush():  # (k, g, hash, size, front, back, mask, fsum, argmax, maxiv, ts)
        out.append(tuple(r[:7]) + (r[8], r[9], r[7], r[10]))
    return sorted(out)


def test_golden_files_present():
    names = [os.path.basename(f) for f in FILES]
    assert len(names) == 4 and any("slide" in n for n in names) and any("tumble" in n for n in names) and any("hop" in n for n in names), names


@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(f)[:-4] for f in FILES])
def test_reference_matches_model(path):
    t, ts, res, win, slide = load(path)
    u, uts = map_filter(t, ts)
    same(rows(res), model_rows(u, uts, win, slide))
    nxt = {}
    for k, g in zip(res["key"].tolist(), res["id"].tolist()):  # every key's windows reach the Sink in order
        assert g == nxt.get(k, 0), (k, g)
        nxt[k] = g + 1
    assert any(int(r["size"]) < win for r in res)  # end-of-stream windows are part of the outputs


@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(f)[:-4] for f in FILES])
def test_reference_matches_noninc_run(path):
    """Both forms of the reference's Keyed_Windows pin the same windows, timestamps and shared fields, fsum bit for bit."""
    t, ts, res, win, slide = load(path)
    z = np.load(path.replace("ref_cpu_kwi_", "ref_cpu_kw_"))
    assert np.array_equal(z["tuples"], t) and np.array_equal(z["ts"], ts)
    non = z["results"]

    def shared(r, distinct):
        return sorted((int(x["key"]), int(x["id"]), int(x["hash"]), int(x["size"]), int(x["front"]), int(x["back"]), d, float(x["fsum"]),
                       int(x["ts"])) for x, d in zip(r, distinct))

    inc_distinct = [bin(int(m)).count("1") for m in res["mask"]]
    assert shared(res, inc_distinct) == shared(non, [int(d) for d in non["distinct"]])


@pytest.mark.gpu
@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(f)[:-4] for f in FILES])
@pytest.mark.parametrize("K", [1, 4])
def test_gpu_matches_reference(wfb, path, K):
    import torch
    t, ts, res, win, slide = load(path)
    prog = kwilib().kwi_register(0)
    eng = wfb.Engine(wfb.PROG_TUPLE64)
    f = wfb.functors(map_kind=1, iadd=2, fscale=1.0000001, filt_kind=1)
    kw = wfb.KeyedWindowsGPU(prog, win, slide, 64, incremental=True)
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
        for o, n in zip(outs, n_out.cpu().tolist()):
            o.n = n
        collect(*kw.process(outs))
    collect(*kw.flush(64 * (-(-win // slide))))
    assert kw.stats()[1] == 0
    same(rows(np.concatenate(got_r), np.concatenate(got_ts)), rows(res))
