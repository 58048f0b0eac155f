"""ctypes binding of libwfb200.so (the C ABI of include/wfb200.h). Fails loudly: there is no CPU fallback."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("WFB_LIB") or os.path.join(HERE, "libwfb200.so")  # WFB_LIB: another build of the same library (kernel tuning)

u8p, vp = C.c_void_p, C.c_void_p
u32, u64, i32, i64, f64 = C.c_uint32, C.c_uint64, C.c_int32, C.c_int64, C.c_double


class Functors(C.Structure):
    """wfb_functors_t"""
    _fields_ = [("map_kind", i32), ("filt_kind", i32), ("map_iadd", i64), ("map_fscale", f64), ("filt_mod", i64)]


class ProgramInfo(C.Structure):
    _fields_ = [("tuple_bytes", u32), ("result_bytes", u32), ("key_bytes", u32), ("key_kind", u32)]


class Batch(C.Structure):
    """wfb_batch_t"""
    _fields_ = [("tuples", vp), ("ts", vp), ("watermark", u64), ("n", u32), ("reserved", u32)]


class WfbError(RuntimeError):
    def __init__(self, code, what):
        super().__init__(f"libwfb200: {what} failed with {code}: {error_string(code)}")
        self.code = code


_lib = None

# every symbol include/wfb200.h declares: (restype, argtypes)
SYMBOLS = {
    "wfb_abi_version": (C.c_int, []),
    "wfb_error_string": (C.c_char_p, [C.c_int]),
    "wfb_device_count": (C.c_int, []),
    "wfb_program_register": (C.c_int, [vp, C.c_size_t]),
    "wfb_program_info": (C.c_int, [C.c_int, C.POINTER(ProgramInfo)]),
    "wfb_engine_create": (C.c_int, [C.POINTER(vp), C.c_int]),
    "wfb_engine_destroy": (C.c_int, [vp]),
    "wfb_engine_launches": (u64, [vp]),
    "wfb_engine_set_params": (C.c_int, [vp, vp, C.c_size_t]),
    "wfb_ffat_set_params": (C.c_int, [vp, vp, C.c_size_t]),
    "wfb_ffat_set_key_shard": (C.c_int, [vp, u32, u32]),
    "wfb_engine_set_key_bits": (C.c_int, [vp, u32]),
    "wfb_map": (C.c_int, [vp, C.POINTER(Functors), vp, u32, vp]),
    "wfb_map_filter": (C.c_int, [vp, C.POINTER(Functors), vp, vp, u32, vp, vp, vp, vp]),
    "wfb_kstate_create": (C.c_int, [C.POINTER(vp), C.c_int, u32, u32]),
    "wfb_kstate_destroy": (C.c_int, [vp]),
    "wfb_kstate_key_capacity": (u32, [vp]),
    "wfb_map_stateful": (C.c_int, [vp, C.POINTER(Functors), C.POINTER(Batch), u32, vp]),
    "wfb_filter_stateful": (C.c_int, [vp, C.POINTER(Functors), C.POINTER(Batch), C.POINTER(Batch), u32, vp, vp]),
    "wfb_flatmap_stateful": (C.c_int, [vp, C.POINTER(Functors), C.POINTER(Batch), C.POINTER(Batch), u32, u32, vp, vp]),
    "wfb_kwin_create": (C.c_int, [C.POINTER(vp), C.c_int, u64, u64, u32, u32]),
    "wfb_kwin_destroy": (C.c_int, [vp]),
    "wfb_kwin_set_params": (C.c_int, [vp, vp, C.c_size_t]),
    "wfb_kwin_process_cb": (C.c_int, [vp, C.POINTER(Batch), u32, vp, vp, u32, vp, vp]),
    "wfb_kwin_flush": (C.c_int, [vp, vp, vp, u32, vp, vp]),
    "wfb_kwin_stats": (C.c_int, [vp, C.POINTER(u32), C.POINTER(u32), vp]),
    "wfb_kwin_key_capacity": (u32, [vp]),
    "wfb_kwin_launches": (u64, [vp]),
    "wfb_reduce_by_key_batches": (C.c_int, [vp, C.POINTER(Batch), C.POINTER(Batch), u32, vp, vp]),
    "wfb_map_filter_batches": (C.c_int, [vp, C.POINTER(Functors), C.POINTER(Batch), C.POINTER(Batch), u32, vp, vp]),
    "wfb_flatmap_batches": (C.c_int, [vp, C.POINTER(Functors), C.POINTER(Batch), C.POINTER(Batch), u32, u32, vp, vp]),
    "wfb_reduce_by_key": (C.c_int, [vp, vp, vp, u32, vp, vp, vp, vp]),
    "wfb_reduce_all": (C.c_int, [vp, vp, vp, u32, vp, vp, vp]),
    "wfb_keyby_group": (C.c_int, [vp, vp, u32, vp, vp, vp, vp, vp]),
    "wfb_shard_by_key": (C.c_int, [vp, vp, vp, u32, u32, vp, vp, vp, vp]),
    "wfb_shard_lift": (C.c_int, [vp, C.POINTER(Functors), C.POINTER(Batch), u32, u32, vp, u32, vp, vp]),
    "wfb_ffat_create": (C.c_int, [C.POINTER(vp), C.c_int, u64, u64, u32, u32, C.c_int, u64, u32]),
    "wfb_ffat_destroy": (C.c_int, [vp]),
    "wfb_ffat_launches": (u64, [vp]),
    "wfb_ffat_state_bytes": (u64, [vp]),
    "wfb_ffat_process_tb": (C.c_int, [vp, C.POINTER(Functors), C.POINTER(Batch), u32, vp, vp, u32, vp, vp]),
    "wfb_ffat_process_cb": (C.c_int, [vp, C.POINTER(Functors), C.POINTER(Batch), u32, vp, vp, u32, vp, vp]),
    "wfb_ffat_flush": (C.c_int, [vp, vp, vp, u32, vp, vp]),
    "wfb_ffat_timing": (C.c_int, [vp, C.c_int, C.POINTER(C.c_float), C.POINTER(u32)]),
    "wfb_ffat_stats": (C.c_int, [vp, C.POINTER(u32), C.POINTER(u32), vp]),
    "wfb_ffat_key_capacity": (u32, [vp]),
    "wfb_ffat_results_total": (C.c_int, [vp, C.POINTER(C.c_uint64), vp]),
    "wfb_gen_tuple64": (C.c_int, [u64, u64, u32, C.c_int, u64, vp, vp, vp, vp]),
    "wfb_mg_unique_id": (C.c_int, [vp]),
    "wfb_mg_create": (C.c_int, [C.POINTER(vp), C.c_int, C.c_int, C.c_int, vp, u64, u64, u32, u32]),
    "wfb_mg_destroy": (C.c_int, [vp]),
    "wfb_mg_set_params": (C.c_int, [vp, vp, C.c_size_t]),
    "wfb_mg_step": (C.c_int, [vp, C.POINTER(Functors), C.POINTER(Batch), u32, u64, vp, vp, u32, vp, vp]),
    "wfb_mg_flush": (C.c_int, [vp, vp, vp, u32, vp, vp]),
    "wfb_mg_launches": (u64, [vp]),
    "wfb_mg_stats": (C.c_int, [vp, C.POINTER(u32), C.POINTER(C.c_uint64), vp]),
}


def lib():
    """Load the CUDA library. Raises (never falls back) when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(windflow_b200 has no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def error_string(code):
    return lib().wfb_error_string(code).decode()


def check(code, what):
    if code != 0:
        raise WfbError(code, what)
