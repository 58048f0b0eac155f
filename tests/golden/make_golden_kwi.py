"""Generates tests/golden/ref_cpu_kwi_*.npz from the REFERENCE itself: tests/golden/ref_keyed_windows_inc.cpp drives the unmodified
reference's Source -> Map -> Filter -> Keyed_Windows (count-based, DETERMINISTIC mode, the incremental fold of
tests/cpp/kwin_inc_programs.cu) -> Sink over the seeded streams of tests/golden/make_golden_kw.py (the same (win, slide, keys, n, seed)
rows, so each ref_cpu_kwi_* file shares its stream with a ref_cpu_kw_* file), and the stream and every result the Sink received (fired
windows and the end-of-stream windows, each with its timestamp, in Sink order) are stored. The ref_cpu_kw_*.npz files are not touched.

    python tests/golden/make_golden_kwi.py --ref <WindFlow checkout> [--out DIR]

The program is compiled (g++, CPU only) to oracle/_ref/ref_keyed_windows_inc_cpu, where tools/keyed_windows_bench.py also finds it.
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_kw import CASES, ROOT, stream  # noqa: E402

SRC = os.path.join(HERE, "ref_keyed_windows_inc.cpp")
EXE = os.path.join(ROOT, "oracle", "_ref", "ref_keyed_windows_inc_cpu")
RES80_TS = np.dtype([("key", "<u8"), ("id", "<u8"), ("hash", "<u8"), ("size", "<u8"), ("front", "<u8"), ("back", "<u8"), ("mask", "<u8"),
                     ("fsum", "<f8"), ("argmax", "<u8"), ("maxiv", "<i8"), ("ts", "<u8")])


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
    return np.frombuffer(raw[8:], RES80_TS, count=m)


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
            name = name.replace("ref_cpu_kw_", "ref_cpu_kwi_")
            np.savez_compressed(os.path.join(a.out, name + ".npz"), tuples=t, ts=ts, results=res, geometry=np.array([win, slide], np.uint64))
            print(f"{name}: {len(res)} results", file=sys.stderr)


if __name__ == "__main__":
    main()
