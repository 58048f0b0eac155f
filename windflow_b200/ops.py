"""Host-side handles over the C ABI (include/wfb200.h), used by tests/, bench.py and __graft_entry__.smoke().

PyTorch is only plumbing here: device memory (uint8 / int64 tensors), streams and torch.distributed. Every
compute call goes through libwfb200.so; nothing in this module computes on the CPU.

Naming follows the reference operators: Map_GPU (wf/map_gpu.hpp), Filter_GPU (wf/filter_gpu.hpp), Reduce_GPU
(wf/reduce_gpu.hpp), Ffat_Windows_GPU (wf/ffat_windows_gpu.hpp), KeyBy_Emitter_GPU (wf/keyby_emitter_gpu.hpp).
"""
import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from ._lib import WfbError, Batch as CBatch
from ._lib import Functors, check

PROG_TUPLE64, PROG_WFTEST16, PROG_WFWIN24, PROG_LIFTED32 = 0, 1, 2, 3
# the bench stream keyed by the double whose bits are pad[0] / by the 16-byte struct KEY16 {key, low and high half of pad[0]}
PROG_TUPLE64_FKEY, PROG_TUPLE64_K16 = 4, 5

TUPLE64 = np.dtype([("key", "<u8"), ("id", "<u8"), ("ivalue", "<i8"), ("fvalue", "<f8"), ("pad", "<u8", (4,))])
RESULT32 = np.dtype([("key", "<u8"), ("id", "<u8"), ("isum", "<i8"), ("fsum", "<f8")])
WFTEST16 = np.dtype([("key", "<u8"), ("value", "<i8")])
WFWIN24 = np.dtype([("key", "<u8"), ("id", "<u8"), ("value", "<i8")])
RESULT32D = np.dtype([("key", "<f8"), ("id", "<u8"), ("isum", "<i8"), ("fsum", "<f8")])
KEY16 = np.dtype([("key", "<u8"), ("a", "<u4"), ("b", "<u4")])
RESULT48K = np.dtype([("key", KEY16), ("id", "<u8"), ("isum", "<i8"), ("fsum", "<f8"), ("pad", "<u8")])

TUPLE_DTYPE = {PROG_TUPLE64: TUPLE64, PROG_WFTEST16: WFTEST16, PROG_WFWIN24: WFWIN24, PROG_LIFTED32: RESULT32,
               PROG_TUPLE64_FKEY: TUPLE64, PROG_TUPLE64_K16: TUPLE64}
RESULT_DTYPE = {PROG_TUPLE64: RESULT32, PROG_WFTEST16: WFWIN24, PROG_WFWIN24: WFWIN24, PROG_LIFTED32: RESULT32,
                PROG_TUPLE64_FKEY: RESULT32D, PROG_TUPLE64_K16: RESULT48K}

KEY_RR, KEY_UNIFORM, KEY_ZIPF = 0, 1, 2
KEYS_GROW = 4  # WFB_KEYS_GROW
SEED = 0x5EED5EED




def functors(map_kind=0, iadd=0, fscale=1.0, filt_kind=0, mod=1):
    return Functors(map_kind, filt_kind, iadd, fscale, mod)


def _stream_ptr(stream=None):
    s = stream if stream is not None else torch.cuda.current_stream()
    return C.c_void_p(s.cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def to_device(arr, device="cuda"):
    """numpy (structured) array -> flat uint8 CUDA tensor holding the same bytes."""
    a = np.ascontiguousarray(arr)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to(device)


def to_host(t, dtype, n=None):
    """uint8 CUDA tensor -> numpy array of `dtype` (first n records)."""
    a = t.cpu().numpy().view(dtype)
    return a if n is None else a[:n]


def ts_to_device(ts, device="cuda"):
    return torch.from_numpy(np.ascontiguousarray(ts, dtype=np.uint64).view(np.int64).copy()).to(device)


def ts_to_host(t, n=None):
    a = t.cpu().numpy().view(np.uint64)
    return a if n is None else a[:n]


class DeviceBatch:
    """Batch_GPU_t stand-in (wf/batch_gpu_t.hpp:50-243), structure-of-arrays: `tuples` (uint8, n*tuple_bytes) and
    `ts` (int64 holding uint64 bits), the number of meaningful items `n` and the batch watermark."""

    def __init__(self, tuples, ts, n, watermark=0):
        self.tuples, self.ts, self.n, self.watermark = tuples, ts, int(n), int(watermark)

    @staticmethod
    def from_host(arr, ts=None, watermark=None, device="cuda"):
        t = to_device(arr, device)
        d = ts_to_device(ts, device) if ts is not None else None
        wm = int(ts[0]) if (watermark is None and ts is not None and len(ts)) else int(watermark or 0)
        return DeviceBatch(t, d, len(arr), wm)


class Engine:
    """Per-replica scratch + the stateless / per-batch operators of one program."""

    def __init__(self, prog=PROG_TUPLE64):
        self.L = _lib.lib()
        if self.L.wfb_device_count() <= 0:
            raise RuntimeError("windflow_b200: no CUDA device (there is no CPU fallback)")
        self.prog = prog
        self.h = C.c_void_p()
        check(self.L.wfb_engine_create(C.byref(self.h), prog), "wfb_engine_create")
        info = _lib.ProgramInfo()
        check(self.L.wfb_program_info(prog, C.byref(info)), "wfb_program_info")
        self.tuple_bytes, self.result_bytes = info.tuple_bytes, info.result_bytes

    def close(self):
        if self.h:
            self.L.wfb_engine_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launches(self):
        return int(self.L.wfb_engine_launches(self.h))

    def set_key_bits(self, bits):
        check(self.L.wfb_engine_set_key_bits(self.h, bits), "wfb_engine_set_key_bits")

    # Map_GPU (stateless), in place
    def map(self, batch, f, stream=None):
        check(self.L.wfb_map(self.h, C.byref(f), _ptr(batch.tuples), batch.n, _stream_ptr(stream)), "wfb_map")
        return batch

    # [Map_GPU ->] Filter_GPU (stateless): returns (out batch, n_out device tensor). out may alias in.
    def map_filter(self, batch, f, out=None, n_out=None, stream=None):
        if out is None:
            out = DeviceBatch(torch.empty_like(batch.tuples), torch.empty_like(batch.ts) if batch.ts is not None else None,
                              batch.n, batch.watermark)
        if n_out is None:
            n_out = torch.zeros(1, dtype=torch.int32, device=batch.tuples.device)
        check(self.L.wfb_map_filter(self.h, C.byref(f), _ptr(batch.tuples), _ptr(batch.ts), batch.n,
                                    _ptr(out.tuples), _ptr(out.ts), _ptr(n_out), _stream_ptr(stream)), "wfb_map_filter")
        return out, n_out

    def map_filter_batches(self, batches, f, outs, n_out, stream=None):
        """[Map_GPU ->] Filter_GPU over K queued batches in one launch: batch i compacted into outs[i], n_out[i] survivors."""
        check(self.L.wfb_map_filter_batches(self.h, C.byref(f), _cbatches(batches), _cbatches(outs), len(batches), _ptr(n_out),
                                            _stream_ptr(stream)), "wfb_map_filter_batches")
        return outs, n_out

    def reduce_by_key(self, batch, out=None, n_out=None, stream=None):
        if out is None:
            out = DeviceBatch(torch.empty_like(batch.tuples), torch.empty_like(batch.ts), batch.n, batch.watermark)
        if n_out is None:
            n_out = torch.zeros(1, dtype=torch.int32, device=batch.tuples.device)
        check(self.L.wfb_reduce_by_key(self.h, _ptr(batch.tuples), _ptr(batch.ts), batch.n, _ptr(out.tuples), _ptr(out.ts),
                                       _ptr(n_out), _stream_ptr(stream)), "wfb_reduce_by_key")
        return out, n_out

    def reduce_by_key_batches(self, batches, outs, n_out, stream=None):
        """Reduce_GPU over K queued batches in one launch sequence: batch i reduced into outs[i], n_out[i] distinct keys."""
        check(self.L.wfb_reduce_by_key_batches(self.h, _cbatches(batches), _cbatches(outs), len(batches), _ptr(n_out), _stream_ptr(stream)),
              "wfb_reduce_by_key_batches")
        return outs, n_out

    def reduce_all(self, batch, stream=None):
        out_t = torch.empty(self.tuple_bytes, dtype=torch.uint8, device=batch.tuples.device)
        out_ts = torch.zeros(1, dtype=torch.int64, device=batch.tuples.device)
        check(self.L.wfb_reduce_all(self.h, _ptr(batch.tuples), _ptr(batch.ts), batch.n, _ptr(out_t), _ptr(out_ts),
                                    _stream_ptr(stream)), "wfb_reduce_all")
        return out_t, out_ts

    def keyby_group(self, batch, stream=None):
        dev = batch.tuples.device
        start = torch.empty(max(1, batch.n), dtype=torch.int32, device=dev)
        mp = torch.empty(max(1, batch.n), dtype=torch.int32, device=dev)
        dk = torch.empty(max(1, batch.n), dtype=torch.int64, device=dev)
        nk = torch.zeros(1, dtype=torch.int32, device=dev)
        check(self.L.wfb_keyby_group(self.h, _ptr(batch.tuples), batch.n, _ptr(start), _ptr(mp), _ptr(dk), _ptr(nk),
                                     _stream_ptr(stream)), "wfb_keyby_group")
        return start, mp, dk, nk

    def shard_lift(self, batches, pre, num_shards, regions, region_capacity, counts, stream=None):
        """Fused [Map -> Filter ->] lift + stable partition by key % num_shards (source side of the multi-GPU keyby).
        regions: uint8 tensor of num_shards * region_capacity * result_bytes; counts: int32 tensor of 9."""
        arr = _cbatches(batches)
        check(self.L.wfb_shard_lift(self.h, C.byref(pre) if pre is not None else None, arr, len(batches), num_shards,
                                    _ptr(regions), region_capacity, _ptr(counts), _stream_ptr(stream)), "wfb_shard_lift")
        return counts

    def shard_by_key(self, batch, num_shards, out=None, stream=None):
        dev = batch.tuples.device
        if out is None:
            out = DeviceBatch(torch.empty_like(batch.tuples), torch.empty_like(batch.ts) if batch.ts is not None else None,
                              batch.n, batch.watermark)
        seg = torch.zeros(num_shards + 1, dtype=torch.int32, device=dev)
        check(self.L.wfb_shard_by_key(self.h, _ptr(batch.tuples), _ptr(batch.ts), batch.n, num_shards, _ptr(out.tuples),
                                      _ptr(out.ts), _ptr(seg), _stream_ptr(stream)), "wfb_shard_by_key")
        return out, seg


class KeyedState:
    """Per-operator keyed state of a stateful Map_GPU / Filter_GPU (wf/map_gpu.hpp:212-299, wf/filter_gpu.hpp:247-355)."""

    def __init__(self, prog, max_keys, dense_keys=False, grow_keys=False):
        """grow_keys: max_keys is the initial capacity, the table grows with the keys (WFB_KEYS_GROW)."""
        self.L = _lib.lib()
        if self.L.wfb_device_count() <= 0:
            raise RuntimeError("windflow_b200: no CUDA device (there is no CPU fallback)")
        self.h = C.c_void_p()
        check(self.L.wfb_kstate_create(C.byref(self.h), prog, max_keys, (1 if dense_keys else 0) | (KEYS_GROW if grow_keys else 0)),
              "wfb_kstate_create")

    @property
    def key_capacity(self):
        """Keys the table holds now (max_keys, or what a growing table has grown to)."""
        return int(self.L.wfb_kstate_key_capacity(self.h))

    def close(self):
        if self.h:
            self.L.wfb_kstate_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def map(self, batches, f, stream=None):
        """func(tuple, state_of_key) in place, per-key arrival order over the queued batches."""
        check(self.L.wfb_map_stateful(self.h, C.byref(f), _cbatches(batches), len(batches), _stream_ptr(stream)), "wfb_map_stateful")
        return batches

    def filter(self, batches, f, outs, n_out, stream=None):
        """predicate(tuple, state_of_key); survivors of batch i compacted into outs[i], n_out[i] of them."""
        check(self.L.wfb_filter_stateful(self.h, C.byref(f), _cbatches(batches), _cbatches(outs), len(batches), _ptr(n_out), _stream_ptr(stream)),
              "wfb_filter_stateful")
        return outs, n_out


class Segment(list):
    """A list of DeviceBatch whose C descriptor array is built once: a replica that re-submits the same device buffers
    (a ring of input segments) does not pay the per-batch Python / ctypes cost on every call. Immutable by convention."""

    def __init__(self, batches):
        super().__init__(batches)
        self.carr = _cbatches(self, cache=False)
        self.total = sum(b.n for b in self)


def _cbatches(batches, cache=True):
    if cache and isinstance(batches, Segment):
        return batches.carr
    arr = (CBatch * len(batches))()
    for i, b in enumerate(batches):
        arr[i].tuples = b.tuples.data_ptr()
        arr[i].ts = b.ts.data_ptr() if b.ts is not None else None
        arr[i].watermark = b.watermark
        arr[i].n = b.n
    return arr


class FfatWindowsGPU:
    """Ffat_Windows_GPU replica state (wf/ffat_windows_gpu.hpp, wf/ffat_replica_gpu.hpp): count-based windows
    `withCBWindows(win, slide)`, `withNumWinPerBatch(nb)`."""

    def __init__(self, prog, win, slide, nb, max_keys, dense_keys=False, win_type=0, lateness=0, pipelined=False, grow_keys=False):
        """grow_keys: max_keys is the initial capacity, the key table grows with the keys (WFB_KEYS_GROW)."""
        self.L = _lib.lib()
        if self.L.wfb_device_count() <= 0:
            raise RuntimeError("windflow_b200: no CUDA device (there is no CPU fallback)")
        self.prog, self.win, self.slide, self.nb, self.max_keys = prog, win, slide, nb, max_keys
        self.win_type = win_type  # 0 count-based, 1 time-based (win / slide / lateness in timestamp units)
        self.h = C.c_void_p()
        self.pipelined, self.grow_keys = pipelined, grow_keys
        check(self.L.wfb_ffat_create(C.byref(self.h), prog, win, slide, nb, max_keys, win_type, lateness,
                                     (1 if dense_keys else 0) | (2 if pipelined else 0) | (KEYS_GROW if grow_keys else 0)), "wfb_ffat_create")
        self.res_dtype = RESULT_DTYPE[prog]
        self._keep = None
        self._max_items = 0  # largest segment seen: a pipelined handle delivers the previous call's results into this call's buffer

    def close(self):
        if self.h:
            self.L.wfb_ffat_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launches(self):
        return int(self.L.wfb_ffat_launches(self.h))

    @property
    def state_bytes(self):
        return int(self.L.wfb_ffat_state_bytes(self.h))

    def set_key_shard(self, num_shards, shard):
        """Dense-key handle of one keyby shard: keys with key % num_shards == shard, slot = key // num_shards."""
        check(self.L.wfb_ffat_set_key_shard(self.h, num_shards, shard), "wfb_ffat_set_key_shard")

    @property
    def key_capacity(self):
        """Keys the table holds now (max_keys, or what a growing table has grown to)."""
        return int(self.L.wfb_ffat_key_capacity(self.h))

    def max_results(self, n_items):
        """Upper bound on the results one call over n_items input items can produce (count-based windows; time-based
        callers size the output for the groups a watermark jump can complete)."""
        cap = self.key_capacity
        keys = cap if self.win_type == 0 else max(cap * 8, 65536)  # (time-based: a watermark jump completes several groups per key)
        groups = n_items // max(1, self.slide * self.nb) + keys + 1  # every key may fire one more group than its items alone account for
        if self.grow_keys:  # a key new in the call fires its first group after B = (Nb-1)*slide + win of its items (time-based: a key of
            groups += n_items if self.win_type else n_items // ((self.nb - 1) * self.slide + self.win)  # the call may fire with one item)
        return groups * self.nb

    def process(self, batches, pre=None, out=None, out_ts=None, n_out=None, stream=None):
        """One stream segment (list of DeviceBatch). Returns (out uint8 tensor, out_ts int64 tensor, n_out tensor)."""
        dev = batches[0].tuples.device
        total = batches.total if isinstance(batches, Segment) else sum(b.n for b in batches)
        self._max_items = max(self._max_items, total)
        if out is None:
            cap = self.max_results(self._max_items)
            out = torch.empty(cap * self.res_dtype.itemsize, dtype=torch.uint8, device=dev)
            out_ts = torch.empty(cap, dtype=torch.int64, device=dev)
        cap = out.numel() // self.res_dtype.itemsize
        if n_out is None:
            n_out = torch.zeros(1, dtype=torch.int32, device=dev)
        arr = _cbatches(batches)
        if self.win_type == 1:
            check(self.L.wfb_ffat_process_tb(self.h, C.byref(pre) if pre is not None else None, arr, len(batches),
                                             _ptr(out), _ptr(out_ts), cap, _ptr(n_out), _stream_ptr(stream)), "wfb_ffat_process_tb")
            return out, out_ts, n_out
        check(self.L.wfb_ffat_process_cb(self.h, C.byref(pre) if pre is not None else None, arr, len(batches),
                                         _ptr(out), _ptr(out_ts), cap, _ptr(n_out), _stream_ptr(stream)),
              "wfb_ffat_process_cb")
        return out, out_ts, n_out

    def flush(self, out=None, out_ts=None, n_out=None, stream=None, device="cuda"):
        """Pipelined handles: the results of the last segment (count 0 otherwise)."""
        if out is None:
            cap = self.max_results(max(1 << 16, self._max_items))
            out = torch.empty(cap * self.res_dtype.itemsize, dtype=torch.uint8, device=device)
            out_ts = torch.empty(cap, dtype=torch.int64, device=device)
        if n_out is None:
            n_out = torch.zeros(1, dtype=torch.int32, device=out.device)
        cap = out.numel() // self.res_dtype.itemsize
        check(self.L.wfb_ffat_flush(self.h, _ptr(out), _ptr(out_ts), cap, _ptr(n_out), _stream_ptr(stream)), "wfb_ffat_flush")
        return out, out_ts, n_out

    def results_to_host(self, out, out_ts, n_out):
        n = int(n_out.item())
        cap = out.numel() // self.res_dtype.itemsize
        if n > cap or (n == cap and (self.stats()[1] & 2)):
            raise WfbError(-3, "Ffat_Windows_GPU: more results than the output buffer holds (results were dropped)")
        return to_host(out, self.res_dtype)[:n].copy(), ts_to_host(out_ts)[:n].copy()

    def timing(self, enable=True):
        """(ingest_ms, sort_ms, update_ms, total_ms, calls) summed over the calls recorded since the last query."""
        ms = (C.c_float * 4)()
        calls = C.c_uint32(0)
        check(self.L.wfb_ffat_timing(self.h, 1 if enable else 0, ms, C.byref(calls)), "wfb_ffat_timing")
        return ms[0], ms[1], ms[2], ms[3], calls.value

    def results_total(self, stream=None):
        """Window results delivered since the handle was created (device-side counter; synchronises the stream)."""
        t = C.c_uint64(0)
        check(self.L.wfb_ffat_results_total(self.h, C.byref(t), _stream_ptr(stream)), "wfb_ffat_results_total")
        return t.value

    def stats(self, stream=None):
        nk, ef = C.c_uint32(0), C.c_uint32(0)
        check(self.L.wfb_ffat_stats(self.h, C.byref(nk), C.byref(ef), _stream_ptr(stream)), "wfb_ffat_stats")
        return nk.value, ef.value


def gen_tuple64(start, n, key_mode=KEY_UNIFORM, nkeys=65536, seed=SEED, zipf_cdf=None, device="cuda", stream=None,
                tuples=None, ts=None):
    """Device-side generator of the synthetic stream of SURVEY.md 8d."""
    L = _lib.lib()
    if tuples is None:
        tuples = torch.empty(n * 64, dtype=torch.uint8, device=device)
        ts = torch.empty(n, dtype=torch.int64, device=device)
    check(L.wfb_gen_tuple64(seed, start, n, key_mode, nkeys, _ptr(zipf_cdf), _ptr(tuples), _ptr(ts), _stream_ptr(stream)),
          "wfb_gen_tuple64")
    return DeviceBatch(tuples, ts, n, start)
