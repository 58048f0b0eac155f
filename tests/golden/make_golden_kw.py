"""Generates tests/golden/ref_cpu_kw_*.npz from the REFERENCE itself: tests/golden/ref_keyed_windows.cpp drives the unmodified reference's
Source -> Map -> Filter -> Keyed_Windows (count-based, DETERMINISTIC mode, the order-sensitive window function of
tests/cpp/kwin_programs.cu) -> Sink over a seeded stream, and the stream and every result the Sink received (fired windows and the
end-of-stream windows, each with its timestamp, in Sink order) are stored, so that the tests compare with the reference without needing it.

    python tests/golden/make_golden_kw.py --ref <WindFlow checkout> [--out DIR]

The program is compiled (g++, CPU only) to oracle/_ref/ref_keyed_windows_cpu, where tools/keyed_windows_bench.py also finds it.
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "ref_keyed_windows.cpp")
EXE = os.path.join(ROOT, "oracle", "_ref", "ref_keyed_windows_cpu")
TUPLE64 = np.dtype([("key", "<u8"), ("id", "<u8"), ("ivalue", "<i8"), ("fvalue", "<f8"), ("pad", "<u8", (4,))])
RES72_TS = np.dtype([("key", "<u8"), ("id", "<u8"), ("hash", "<u8"), ("size", "<u8"), ("mid", "<u8"), ("front", "<u8"), ("back", "<u8"),
                     ("distinct", "<u8"), ("fsum", "<f8"), ("ts", "<u8")])
# (name, win, slide, nkeys, n, seed): sliding, tumbling and hopping windows, win not a power of two
CASES = [("ref_cpu_kw_slide_w10_s3_k5", 10, 3, 5, 3000, 1),
         ("ref_cpu_kw_tumble_w12_s12_k3", 12, 12, 3, 3000, 2),
         ("ref_cpu_kw_hop_w6_s9_k4", 6, 9, 4, 3000, 3),
         ("ref_cpu_kw_slide_w100_s7_k13", 100, 7, 13, 4000, 4)]


def stream(n, nkeys, seed):
    """The seeded input stream: keys, ids 0..n-1, ivalue in [0, 65536), fvalue in [0, 1), non-decreasing timestamps."""
    rng = np.random.default_rng(seed)
    t = np.zeros(n, TUPLE64)
    t["key"] = rng.integers(0, nkeys, n).astype(np.uint64) * np.uint64(7919) + np.uint64(3)
    t["id"] = np.arange(n, dtype=np.uint64)
    t["ivalue"] = rng.integers(0, 1 << 16, n)
    t["fvalue"] = rng.random(n)
    ts = (np.cumsum(rng.integers(0, 4, n)) + 5).astype(np.uint64)
    return t, ts


def compile_ref(ref):
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", "-x", "c++", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ref, "wf"),
                           "-o", EXE, SRC])
    return EXE


def run_ref(t, ts, win, slide, tmp):
    inp, out = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.uint64(len(t)).tobytes()); f.write(t.tobytes()); f.write(ts.tobytes()); f.write(np.zeros(len(t), np.uint64).tobytes())
    subprocess.run([EXE, f"in={inp}", f"out={out}", f"win={win}", f"slide={slide}", "par=1"], check=True, capture_output=True)
    raw = open(out, "rb").read()
    m = int(np.frombuffer(raw[:8], np.uint64)[0])
    return np.frombuffer(raw[8:], RES72_TS, count=m)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True, help="a WindFlow source tree (its wf/ directory holds windflow.hpp)")
    ap.add_argument("--out", default=HERE)
    a = ap.parse_args()
    compile_ref(a.ref)
    with tempfile.TemporaryDirectory() as tmp:
        for (name, win, slide, nkeys, n, seed) in CASES:
            t, ts = stream(n, nkeys, seed)
            res = run_ref(t, ts, win, slide, tmp)
            np.savez_compressed(os.path.join(a.out, name + ".npz"), tuples=t, ts=ts, results=res, geometry=np.array([win, slide], np.uint64))
            print(f"{name}: {len(res)} results", file=sys.stderr)


if __name__ == "__main__":
    main()
