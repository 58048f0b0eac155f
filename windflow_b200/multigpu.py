"""Key-sharded execution of the pipeline across the GPUs of one box (one process per GPU, torch.distributed).

The reference is single-GPU (README.md:15); its keyed operators shard by `std::hash<key_t>()(key) % num_dests`
(wf/keyby_emitter.hpp:215-217, wf/keyby_emitter_gpu.hpp:621) -- the identity hash for integer keys -- and that is the
rule used here across ranks. Map_GPU / Filter_GPU are stateless replicas; the window state partitions by key:

  global step t covers world*K consecutive batches of the stream; rank r owns the K batches [r*K, (r+1)*K) of that span,
  runs the fused Map->Filter over them, partitions the survivors into `world` shard segments (stable), exchanges the
  segment sizes and then the segments (all-to-all over NVLink), and feeds what it receives -- one chunk per source rank,
  in source-rank order, which is global stream order -- to its Ffat_Windows_GPU replica (keys with key % world == rank).

Because every rank receives its keys' items in global arrival order, every count window is the one a single operator
would produce. Only host-side plumbing lives here (testable on CPU with the gloo backend); kernels stay behind the C ABI.
"""
import torch
import torch.distributed as dist


def owner_span(step, rank, world, seg_tuples):
    """[first, last) stream indices of the segment rank `rank` ingests at global step `step`."""
    first = (step * world + rank) * seg_tuples
    return first, first + seg_tuples


def exchange_counts(send_counts, watermark=0):
    """send_counts[d] = items this rank sends to rank d  ->  (recv_counts[s], watermark[s]) = what rank s sends to this
    rank and the watermark of rank s's segment (both travel in one small all-to-all)."""
    meta = torch.stack([send_counts, torch.full_like(send_counts, int(watermark))], dim=1).contiguous()
    recv = torch.empty_like(meta)
    dist.all_to_all_single(recv, meta)
    return recv[:, 0].contiguous(), recv[:, 1].contiguous()


def exchange_segments(send_buf, send_counts_h, recv_counts_h, item_bytes, recv_buf=None):
    """All-to-all of variable-size shard segments. send_buf holds the segments for rank 0..world-1 back to back
    (uint8, item_bytes per item). Returns (recv_buf, offsets) where chunk s = recv_buf[offsets[s]*item_bytes :
    offsets[s+1]*item_bytes] came from source rank s, in its arrival order."""
    n_recv = int(sum(recv_counts_h))
    if recv_buf is None or recv_buf.numel() < n_recv * item_bytes:
        recv_buf = torch.empty(max(1, n_recv) * item_bytes, dtype=torch.uint8, device=send_buf.device)
    n_send = int(sum(send_counts_h))
    dist.all_to_all_single(recv_buf[:n_recv * item_bytes], send_buf[:n_send * item_bytes],
                           output_split_sizes=[int(c) * item_bytes for c in recv_counts_h],
                           input_split_sizes=[int(c) * item_bytes for c in send_counts_h])
    offs = [0]
    for c in recv_counts_h:
        offs.append(offs[-1] + int(c))
    return recv_buf, offs


def exchange_regions(regions, region_cap, send_counts_h, recv_counts_h, item_bytes, recv_buf=None):
    """All-to-all of the shard regions written by wfb_shard_lift (region d starts at d*region_cap items). Returns
    (recv_buf, offsets): chunk s came from source rank s, in its arrival order."""
    world = len(send_counts_h)
    n_recv = int(sum(recv_counts_h))
    if recv_buf is None or recv_buf.numel() < max(1, n_recv) * item_bytes:
        recv_buf = torch.empty(max(1, n_recv) * item_bytes, dtype=torch.uint8, device=regions.device)
    offs = [0]
    for c in recv_counts_h:
        offs.append(offs[-1] + int(c))
    ins = [regions[d * region_cap * item_bytes:(d * region_cap + int(send_counts_h[d])) * item_bytes] for d in range(world)]
    outs = [recv_buf[offs[s] * item_bytes:offs[s + 1] * item_bytes] for s in range(world)]
    dist.all_to_all(outs, ins)
    return recv_buf, offs


TILE = 256  # positions per tile of the window operator's streaming pass (csrc/wfb_kernels.cuh)


def tile_layout(counts):
    """Record offsets that put chunk s of a segment at its tile position (the layout the window operator reads in place):
    chunk s starts at 256 * (tiles of the chunks before it). Returns (offsets, total records incl. padding)."""
    offs, tiles = [], 0
    for c in counts:
        offs.append(tiles * TILE)
        tiles += (int(c) + TILE - 1) // TILE
    return offs, tiles * TILE


class _Slot:
    """Buffers of one step in flight (two of them: the exchange of step i-1 overlaps the source pass of step i)."""

    def __init__(self, world, dev):
        self.regions = None
        self.region_cap = 0
        self.counts = torch.zeros(9, dtype=torch.int32, device=dev)
        self.send_meta = torch.zeros(world, 2, dtype=torch.int64, device=dev)
        self.recv_meta = torch.zeros(world, 2, dtype=torch.int64, device=dev)
        self.h_counts = torch.zeros(9, dtype=torch.int32).pin_memory() if dev.type == "cuda" else torch.zeros(9, dtype=torch.int32)
        self.h_recv = torch.zeros(world, 2, dtype=torch.int64).pin_memory() if dev.type == "cuda" else torch.zeros(world, 2, dtype=torch.int64)
        self.recv = None
        self.ev_src = torch.cuda.Event()
        self.ev_meta = torch.cuda.Event()
        self.ev_a2a = torch.cuda.Event()
        self.ev_done = torch.cuda.Event()
        self.used = False


class KeyShardedPipeline:
    """Map_GPU -> Filter_GPU -> (keyby across GPUs) -> Ffat_Windows_GPU on this rank's key shard.

    Source side (wfb_shard_lift): one streaming pass (map, filter, lift; no compaction chain) and one stable partition
    pass that moves the 32-byte lifted results into `world` destination regions. Exchange: sizes + watermarks in one
    small all-to-all, then the records (NCCL, NVLink), each source's chunk landing at its tile position of the receive
    buffer. Destination side: the window operator instantiated for already-lifted records (WFB_PROG_LIFTED32) reads the
    received records in place.

    pipelined=True: the exchange and the window update of step i-1 are issued behind the source pass of step i (the
    host never waits for the GPU: the sizes it needs were produced a step ago), so results arrive one step() late and
    flush() delivers the last ones."""

    def __init__(self, ops, functors, win, slide, nb, max_keys, rank, world, device, pipelined=True):
        self.ops, self.f, self.rank, self.world, self.dev = ops, functors, rank, world, device
        self.eng = ops.Engine(ops.PROG_TUPLE64)
        # the rank's replica owns the keys with key % world == rank: compact slots key // world
        self.ff = ops.FfatWindowsGPU(ops.PROG_LIFTED32, win, slide, nb, max_keys=(max_keys + world - 1) // world, dense_keys=True,
                                     pipelined=False)
        if world > 1:
            self.ff.set_key_shard(world, rank)
        self.rb = self.eng.result_bytes
        self.overlap = bool(pipelined)
        self.slots = [_Slot(world, device), _Slot(world, device)]
        self.comm = torch.cuda.Stream(device)
        self.step_no = 0
        self.pending = None

    # ---- source side of a step: fused pass + partition by destination, then the sizes travel ------------------------
    def _source(self, sl, batches, watermark):
        n = getattr(batches, "total", None) or sum(b.n for b in batches)
        if sl.region_cap < n:
            if sl.used:
                torch.cuda.synchronize(self.dev)
            sl.region_cap = n  # worst case: every item of the segment survives and goes to one shard
            sl.regions = torch.empty(self.world * n * self.rb, dtype=torch.uint8, device=self.dev)
        main = torch.cuda.current_stream(self.dev)
        self.eng.shard_lift(batches, self.f, self.world, sl.regions, sl.region_cap, sl.counts)
        sl.send_meta[:, 0].copy_(sl.counts[:self.world])
        sl.send_meta[:, 1].fill_(int(watermark))
        sl.ev_src.record(main)
        with torch.cuda.stream(self.comm):
            self.comm.wait_event(sl.ev_src)
            dist.all_to_all_single(sl.recv_meta, sl.send_meta)
            sl.h_counts.copy_(sl.counts, non_blocking=True)
            sl.h_recv.copy_(sl.recv_meta, non_blocking=True)
            sl.ev_meta.record(self.comm)
        sl.used = True

    # ---- exchange of the records (communication stream) -----------------------------------------------------------------
    def _exchange(self, sl):
        sl.ev_meta.synchronize()  # sizes of this step on the host (a step old when pipelined: no GPU stall)
        cnt = sl.h_counts.tolist()
        if cnt[8]:
            raise RuntimeError("wfb_shard_lift: shard region overflow")
        send = cnt[:self.world]
        rm = sl.h_recv.tolist()
        recv_counts, wms = [int(r[0]) for r in rm], [int(r[1]) for r in rm]
        offs, total = tile_layout(recv_counts)
        if sl.recv is None or sl.recv.numel() < max(1, total) * self.rb:
            torch.cuda.synchronize(self.dev)
            sl.recv = torch.empty(max(1, total) * self.rb * 5 // 4, dtype=torch.uint8, device=self.dev)
        rb, cap = self.rb, sl.region_cap
        ins = [sl.regions[d * cap * rb:(d * cap + send[d]) * rb] for d in range(self.world)]
        outs = [sl.recv[offs[s] * rb:(offs[s] + recv_counts[s]) * rb] for s in range(self.world)]
        with torch.cuda.stream(self.comm):
            self.comm.wait_event(sl.ev_done)  # the window update that read this receive buffer two steps ago
            dist.all_to_all(outs, ins)
            sl.ev_a2a.record(self.comm)
        return recv_counts, wms, offs

    # ---- destination side: window update on the received chunks (source-rank order = global stream order) ---------
    def _update(self, sl, recv_counts, wms, offs, out, out_ts, n_out):
        ops, rb = self.ops, self.rb
        main = torch.cuda.current_stream(self.dev)
        main.wait_event(sl.ev_a2a)
        chunks = [ops.DeviceBatch(sl.recv[offs[s] * rb:(offs[s] + recv_counts[s]) * rb], None, recv_counts[s], wms[s])
                  for s in range(self.world)]
        self.ff.process(chunks, pre=None, out=out, out_ts=out_ts, n_out=n_out)
        sl.ev_done.record(main)
        return sum(recv_counts)

    def step(self, batches, watermark, out, out_ts, n_out):
        """batches: this rank's K batches of the global step. Window results go to out (of the previous step when
        pipelined). Returns the number of records the window operator consumed in this call."""
        cur = self.slots[self.step_no & 1]
        self.step_no += 1
        if not self.overlap:
            self._source(cur, batches, watermark)
            return self._update(cur, *self._exchange(cur), out, out_ts, n_out)
        prev, ex = self.pending, None
        if prev is not None:
            ex = self._exchange(prev)       # records of step i-1 travel while ...
        self._source(cur, batches, watermark)  # ... the source pass of step i runs
        self.pending = cur
        if prev is None:
            n_out.zero_()
            return 0
        return self._update(prev, *ex, out, out_ts, n_out)

    def flush(self, out, out_ts, n_out):
        """Delivers the results of the step still in flight (pipelined mode)."""
        prev, self.pending = self.pending, None
        if prev is None:
            n_out.zero_()
            return 0
        return self._update(prev, *self._exchange(prev), out, out_ts, n_out)



class KeyShardedPipelineC:
    """The same pipeline with the whole step under the C ABI (wfb_mg_*): source pass, size exchange, NCCL all-to-all and window update
    are issued by ONE library call per step (NCCL send/recv groups from C on a communication stream; nothing of torch on the per-step
    path). Only the communicator's unique id travels through torch.distributed, once. Same interface as KeyShardedPipeline (always
    pipelined: results arrive THREE steps late, flush() delivers the rest, in step order). With at most 65536 slots over all ranks the
    exchange is the bucketed one (include/wfb200.h): the destination side runs no partition.

    params: the program's params_t as a ctypes object (wfb_mg_set_params), for a program whose combine, make_result or result_key
    reads it; `functors` is what every step passes as `pre` (None: the source side uses `params` too)."""

    def __init__(self, ops, functors, win, slide, nb, max_keys, rank, world, device, prog=None, params=None):
        import ctypes as C
        from . import _lib
        self.ops, self.f, self.rank, self.world, self.dev = ops, functors, rank, world, device
        self.L = _lib.lib()
        ident = torch.zeros(128, dtype=torch.uint8)
        if world > 1:
            if rank == 0:
                buf = (C.c_char * 128)()
                _lib.check(self.L.wfb_mg_unique_id(buf), "wfb_mg_unique_id")
                ident = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
            t = ident.to(device)
            dist.broadcast(t, src=0)
            ident = t.cpu()
        self._id = (C.c_char * 128).from_buffer_copy(bytes(ident.numpy().tobytes()))
        self.h = C.c_void_p()
        _lib.check(self.L.wfb_mg_create(C.byref(self.h), ops.PROG_TUPLE64 if prog is None else prog, world, rank, self._id, win, slide, nb, max_keys), "wfb_mg_create")
        if params is not None:
            _lib.check(self.L.wfb_mg_set_params(self.h, C.byref(params), C.sizeof(params)), "wfb_mg_set_params")
        self.res_dtype = ops.RESULT_DTYPE[ops.PROG_TUPLE64 if prog is None else prog]
        self.max_keys, self.slide, self.nb = max_keys, slide, nb
        self.ff = self  # (bench.py talks to `pipe.ff` for launches / stats / results)
        self.eng = _NoLaunches()

    # ---- the interface bench.py and the tests use ----------------------------------------------------------------------
    def step(self, batches, watermark, out, out_ts, n_out):
        import ctypes as C
        from . import _lib
        arr = self.ops._cbatches(batches)
        _lib.check(self.L.wfb_mg_step(self.h, C.byref(self.f) if self.f is not None else None, arr, len(batches), int(watermark),
                                      self.ops._ptr(out), self.ops._ptr(out_ts), out.numel() // self.res_dtype.itemsize, self.ops._ptr(n_out),
                                      self.ops._stream_ptr(None)), "wfb_mg_step")

    def flush(self, out, out_ts, n_out):
        from . import _lib
        _lib.check(self.L.wfb_mg_flush(self.h, self.ops._ptr(out), self.ops._ptr(out_ts), out.numel() // self.res_dtype.itemsize, self.ops._ptr(n_out),
                                       self.ops._stream_ptr(None)), "wfb_mg_flush")

    @property
    def launches(self):
        return int(self.L.wfb_mg_launches(self.h))

    def max_results(self, n_items):
        keys = (self.max_keys + self.world - 1) // self.world
        return (n_items // max(1, self.slide * self.nb) + keys + 1) * self.nb

    def stats(self):
        import ctypes as C
        from . import _lib
        ef, tot = C.c_uint32(0), C.c_uint64(0)
        _lib.check(self.L.wfb_mg_stats(self.h, C.byref(ef), C.byref(tot), self.ops._stream_ptr(None)), "wfb_mg_stats")
        return 0, ef.value

    def results_total(self):
        import ctypes as C
        from . import _lib
        ef, tot = C.c_uint32(0), C.c_uint64(0)
        _lib.check(self.L.wfb_mg_stats(self.h, C.byref(ef), C.byref(tot), self.ops._stream_ptr(None)), "wfb_mg_stats")
        return tot.value

    def results_to_host(self, out, out_ts, n_out):
        n = int(n_out.item())
        return self.ops.to_host(out, self.res_dtype)[:n].copy(), self.ops.ts_to_host(out_ts)[:n].copy()

    def timing(self, enable=True):
        return 0.0, 0.0, 0.0, 0.0, 0

    def close(self):
        if self.h:
            self.L.wfb_mg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _NoLaunches:
    launches = 0
