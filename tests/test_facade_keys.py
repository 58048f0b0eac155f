"""Key types other than integers in the builder API (include/wf/windflow_gpu.hpp) and the C ABI. CPU: the test program
tests/cpp/test_facade_keys.cu compiles with nvcc for sm_90a, a key type with padding is refused at compile time with WindFlow's
message, and wfb_program_info reports the key width and kind of the built-in programs. GPU: the test program passes."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_facade_keys.cu")
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_keys.bin")
NVCC = ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "--expt-extended-lambda",
        "-I" + os.path.join(ROOT, "include")]
needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")


def _compile():
    from windflow_b200 import build
    build.build()
    hdrs = [os.path.join(ROOT, "include", "wf", "windflow_gpu.hpp")] + \
        [os.path.join(ROOT, "windflow_b200", "csrc", h) for h in ("wfb_kernels.cuh", "wfb_keys.cuh", "wfb_launch.cuh", "wfb_programs.cuh")] + [SRC]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(h) for h in hdrs):
        return
    subprocess.check_call(NVCC + ["-o", EXE, SRC, "-L" + os.path.join(ROOT, "windflow_b200"), "-lwfb200",
                                  "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../windflow_b200"])


@needs_nvcc
def test_facade_keys_compiles():
    _compile()
    assert os.path.exists(EXE)


@needs_nvcc
def test_padded_key_is_refused_at_compile_time(tmp_path):
    src = tmp_path / "padded_key.cu"
    src.write_text(
        "#include <wf/windflow_gpu.hpp>\n"
        "struct padded_t { uint32_t a; uint64_t b; };  // 4 bytes of padding: comparing bytes is not comparing members\n"
        "struct tuple_t { padded_t k; int64_t v; };\n"
        "struct result_t { padded_t key; uint64_t id; int64_t v; };\n"
        "struct KeyF { __host__ __device__ padded_t operator()(const tuple_t &t) const { return t.k; } };\n"
        "int main() { return wfb::register_program<wf::FacadeStatefulProgram<tuple_t, int64_t, wf::StatefulIdMap<tuple_t, int64_t>,\n"
        "                                            wf::StatefulKeepAll<tuple_t, int64_t>, KeyF>>(); }\n")
    out = subprocess.run(NVCC + ["-c", "-o", str(tmp_path / "padded_key.o"), str(src)], capture_output=True, text=True)
    assert out.returncode != 0
    assert "WindFlow Compilation Error - the key type of a GPU operator" in out.stdout + out.stderr, (out.stdout + out.stderr)[-3000:]


def test_program_info_key_width_and_kind():
    from windflow_b200 import build, _lib, ops
    build.build()
    L = _lib.lib()
    info = _lib.ProgramInfo()
    expect = {ops.PROG_TUPLE64: (64, 32, 8, 0), ops.PROG_LIFTED32: (32, 32, 8, 0),
              ops.PROG_TUPLE64_FKEY: (64, 32, 8, 1), ops.PROG_TUPLE64_K16: (64, 48, 16, 2)}
    for prog, (tb, rb, kb, kind) in expect.items():
        assert L.wfb_program_info(prog, C.byref(info)) == 0
        assert (info.tuple_bytes, info.result_bytes, info.key_bytes, info.key_kind) == (tb, rb, kb, kind), prog
    assert ops.RESULT_DTYPE[ops.PROG_TUPLE64_FKEY].itemsize == 32 and ops.RESULT_DTYPE[ops.PROG_TUPLE64_K16].itemsize == 48


@pytest.mark.gpu
def test_facade_keys_runs():
    _compile()
    out = subprocess.run([EXE], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "KEYS_OK" in out.stdout, out.stdout[-3000:]
