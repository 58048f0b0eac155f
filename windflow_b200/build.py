"""Builds libwfb200.so in-tree with nvcc for sm_90a (H100). Nothing is compiled at run time: the library loads as built."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libwfb200.so")
SOURCES = ["wfb_lib.cu"]
HEADERS = ["wfb_kernels.cuh", "wfb_keys.cuh", "wfb_launch.cuh", "wfb_programs.cuh", "wfb_ptx.cuh", "wfb_scratch.h", os.path.join("..", "..", "include", "wfb200.h")]

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared",
    "-diag-suppress", "186",  # "pointless comparison of unsigned integer with zero": loops whose bound is a template constant 0 (lazy FlatFAT levels)
]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build(force=False, verbose=False):
    """Compile every CUDA source of the package for sm_90a (nvcc cross-compiles without a GPU)."""
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + [os.path.join(CSRC, f) for f in SOURCES]
    subprocess.check_call(cmd, cwd=CSRC)
    return LIB


APPS = os.path.join(HERE, "apps")
INCLUDE = os.path.join(HERE, "..", "include")
FACADE_HEADERS = [os.path.join(INCLUDE, "wf", "windflow_gpu.hpp"), os.path.join(INCLUDE, "wf", "deferred_counts.hpp"), os.path.join(INCLUDE, "ff", "ff.hpp"), os.path.join(INCLUDE, "wfb200.h")]


def build_apps(force=False):
    """Applications written against the builder API (include/wf/windflow_gpu.hpp), linked with libwfb200.so: the application's own
    translation unit instantiates the kernels for its functors (nvcc, sm_90a)."""
    build()
    out = []
    for src in sorted(f for f in os.listdir(APPS) if f.endswith(".cu")):
        exe = os.path.join(APPS, src[:-3] + ".bin")
        deps = [os.path.join(APPS, src), LIB] + FACADE_HEADERS + [os.path.join(CSRC, h) for h in HEADERS if not h.startswith("..")]
        if force or not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
            cmd = [os.environ.get("NVCC", "nvcc"), "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "--expt-relaxed-constexpr",
                   "--expt-extended-lambda", "-diag-suppress", "186", "-I" + INCLUDE, "-o", exe, os.path.join(APPS, src), "-L" + HERE, "-lwfb200", "-lpthread",
                   "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/.."]
            subprocess.check_call(cmd)
        out.append(exe)
    return out


if __name__ == "__main__":
    print(build(force=True, verbose=True))
