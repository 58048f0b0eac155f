/*
 * wfb200.h -- C ABI of libwfb200.so, the H100-native (sm_90a) GPU stream-operator kernels that sit
 * underneath the WindFlow GPU operator API (Map_GPU / Filter_GPU / Reduce_GPU / Ffat_Windows_GPU and the
 * KeyBy_Emitter_GPU grouping).
 *
 * The reference (ParaGroup/WindFlow) has no FFI: its GPU path is a set of C++ templates whose kernels are
 * launched from each replica's svc(). Every entry point below replaces one such launch sequence; the
 * reference interface it stands in for is cited as wf/<file>:<line> (relative to the reference repo).
 * INTEGRATION.md shows the binding a WindFlow maintainer adds inside those svc() bodies.
 *
 * Conventions
 *  - all functions return 0 on success, a cudaError_t value (>0) for CUDA failures, or a negative
 *    WFB_E_* code; they never throw and never synchronise the stream unless stated;
 *  - a call that cannot allocate the scratch memory it grows on demand returns the CUDA error and leaves the handle usable: a later
 *    call allocates again;
 *  - pointers are DEVICE pointers unless the name ends in _h; `stream` is a cudaStream_t passed as void*;
 *  - successive calls on one handle may pass different streams (a replica may bind every call to its batch's own stream): each call
 *    is ordered on the device behind everything the handle issued before, and a query that takes a stream sees every earlier call.
 *    The caller still orders its own input and output buffers with the stream it passes. Calls on a keyed-stateful handle
 *    (wfb_kstate_t) may come from several threads at once;
 *  - a batch is structure-of-arrays: `tuples` (n * tuple_bytes, 16-byte aligned) and `ts` (n * uint64_t);
 *    user functors only ever see `tuple_t &`, so this replaces wf/basic_gpu.hpp:132-140's 72-byte AoS item
 *    without touching the operator API;
 *  - record schemas and functors are compiled in ("programs"): the library pre-instantiates the programs
 *    below; user code instantiates its own with WFB_DEFINE_PROGRAM from windflow_b200/csrc/wfb_kernels.cuh
 *    and gets the same entry points for its functors (see INTEGRATION.md);
 *  - a program's tuple_t and result_t are multiples of 8 bytes of up to about 430 bytes (two tile-pass stages of 256 records must
 *    fit 227 KB of shared memory: larger records fail to compile in wfb::register_program); sizes up to 256 bytes are tested.
 *    Results above 160 bytes have no bucket window update: their count-based handles take the full-sort path at every key count
 *    (INTEGRATION.md section 3).
 */
#ifndef WFB200_H
#define WFB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WFB_ABI_VERSION 1

/* negative error codes (positive values are cudaError_t) */
#define WFB_E_BADARG    (-1)  /* null pointer, zero-size window, unknown program ... */
#define WFB_E_NOPROG    (-2)  /* program id not registered */
#define WFB_E_CAPACITY  (-3)  /* more distinct keys / results than the handle was created for */
#define WFB_E_NOGPU     (-4)  /* no CUDA device: the library has NO CPU fallback */
#define WFB_E_UNSUPPORTED (-5)

/* ---- built-in programs ------------------------------------------------------------------------- */
#define WFB_PROG_TUPLE64  0   /* bench stream of SURVEY.md 8d: wfb_tuple64_t -> wfb_result32_t            */
#define WFB_PROG_WFTEST16 1   /* reference tests/graph_tests_gpu/graph_common_gpu.hpp:40-49 {key,value}  */
#define WFB_PROG_WFWIN24  2   /* reference tests/win_tests_gpu/win_common_gpu.hpp:40-80 {key,id,value}   */
#define WFB_PROG_LIFTED32 3   /* already-lifted wfb_result32_t records (destination side of the multi-GPU keyby) */
#define WFB_PROG_TUPLE64_FKEY 4 /* wfb_tuple64_t keyed by the double whose bits are pad[0] -> wfb_result32d_t (a floating-point key) */
#define WFB_PROG_TUPLE64_K16  5 /* wfb_tuple64_t keyed by wfb_key16_t {key, low and high half of pad[0]} -> wfb_result48k_t (a 16-byte key) */

typedef struct { uint64_t key; uint64_t id; int64_t ivalue; double fvalue; uint64_t pad[4]; } wfb_tuple64_t;
typedef struct { uint64_t key; uint64_t id; int64_t isum; double fsum; } wfb_result32_t;
typedef struct { uint64_t key; int64_t value; } wfb_wftest16_t;
typedef struct { uint64_t key; uint64_t id; int64_t value; } wfb_wfwin24_t; /* tuple_t and result_t */
typedef struct { double key; uint64_t id; int64_t isum; double fsum; } wfb_result32d_t;
typedef struct { uint64_t key; uint32_t a, b; } wfb_key16_t;
typedef struct { wfb_key16_t key; uint64_t id; int64_t isum; double fsum; uint64_t pad; } wfb_result48k_t;
typedef struct { int64_t counter; } wfb_state8_t; /* per-key state of the built-in stateful functors (map_state_t / filter_state_t of the reference's tests) */

/* Parameters of the built-in functors (a user program carries its own functor objects instead).
 *   map_kind : 0 identity; 1 value += map_iadd, fvalue *= map_fscale   (Map_Functor_GPU "+2": iadd=2, fscale=1)
 *   filt_kind: 0 keep all; 1 (value & 1) == 0; 2 value % filt_mod == 0 (Filter_Functor_GPU(mod))
 * keyed-stateful variants (wfb_map_stateful / wfb_filter_stateful): a counter per key; map_kind 1: counter++, 2: counter-- on
 * odd keys, then value += counter (Map_Functor_GPU_KB); filter: counter++, value += counter, then the filt_kind predicate. */
typedef struct {
    int32_t map_kind;
    int32_t filt_kind;
    int64_t map_iadd;
    double  map_fscale;
    int64_t filt_mod;
} wfb_functors_t;

typedef struct {
    uint32_t tuple_bytes;   /* sizeof(tuple_t) */
    uint32_t result_bytes;  /* sizeof(result_t) of the window operators */
    uint32_t key_bytes;     /* bytes of the key's canonical words: 8 (key_t of at most 8 bytes) or 16 (9-16 bytes) */
    uint32_t key_kind;      /* 0 integral or enum, 1 float / double, 2 other bytes (windflow_b200/csrc/wfb_keys.cuh) */
} wfb_program_info_t;

/* One input batch of a multi-batch call (host-side descriptor array). */
typedef struct {
    const void     *tuples;     /* device, n * tuple_bytes */
    const uint64_t *ts;         /* device, n timestamps (may be NULL for count-based windows) */
    uint64_t        watermark;  /* Batch_GPU_t::getWatermark(id_replica), wf/batch_gpu_t.hpp:184-192 */
    uint32_t        n;
    uint32_t        reserved;
} wfb_batch_t;

typedef struct wfb_engine wfb_engine_t; /* per-replica scratch for the stateless / per-batch operators */
typedef struct wfb_ffat   wfb_ffat_t;   /* per-replica state of one Ffat_Windows_GPU */

/* ---- library ----------------------------------------------------------------------------------- */
int         wfb_abi_version(void);
const char *wfb_error_string(int code);
int         wfb_device_count(void);                    /* 0 => every compute entry point returns WFB_E_NOGPU */
int         wfb_program_info(int prog, wfb_program_info_t *info);
/* Adds an application-defined program (record schema + functors compiled in the application's own .cu): `ops` is the
 * launch table built by wfb::register_program<P>() of windflow_b200/csrc/wfb_launch.cuh. Returns the new program id
 * (>= 6) or a negative error. For such programs every `const wfb_functors_t *` parameter below points to the program's
 * own params_t (its functor objects) instead. */
int         wfb_program_register(const void *ops, size_t ops_bytes);

/* ---- per-replica scratch ------------------------------------------------------------------------
 * Replaces the per-replica records / Thrust allocator of wf/filter_gpu.hpp:401-470, wf/reduce_gpu.hpp:122-200,
 * wf/keyby_emitter_gpu.hpp:519-537: tile descriptors, sort buffers, counters. Grows on demand (cudaMalloc). */
int wfb_engine_create(wfb_engine_t **e, int prog);
int wfb_engine_destroy(wfb_engine_t *e);
/* launches issued by this engine so far (kernel launches only; bench.py reports it as gpu_launches) */
uint64_t wfb_engine_launches(const wfb_engine_t *e);
/* The program's params_t (functor objects) used by the calls that take no functor argument (key extraction, reduce).
 * Built-in programs need none; for a registered program pass its params_t (bytes must equal sizeof(params_t)). */
int wfb_engine_set_params(wfb_engine_t *e, const void *params, size_t bytes);

/* number of significant low bits of key_t for the per-batch keyed operators below (default 64): the stable LSD
 * radix sort that replaces thrust::sort_by_key runs ceil(bits/8) passes. Integral keys only (WFB_E_BADARG otherwise). */
int wfb_engine_set_key_bits(wfb_engine_t *e, uint32_t bits);

/* ---- Map_GPU, stateless: in-place func(tuple) over a batch --------------------------------------
 * replaces Stateless_MAPGPU_Kernel + launch, wf/map_gpu.hpp:61-76, :357-409. */
int wfb_map(wfb_engine_t *e, const wfb_functors_t *f, void *tuples, uint32_t n, void *stream);

/* ---- Filter_GPU, stateless (optionally fused with a preceding stateless Map_GPU) ------------------
 * out = stable compaction of { map(t) : filter(map(t)) }; *n_out_dev (device uint32) = survivors.
 * replaces Stateless_FILTERGPU_Kernel + thrust::copy_if + D2D copy-back, wf/filter_gpu.hpp:72-88, :497-589
 * (and, when f->map_kind != 0, the Map_GPU launch before it). in/out must not overlap unless identical
 * (in-place compaction is allowed: tuples_out == tuples_in, ts_out == ts_in). ts_in may be NULL. */
int wfb_map_filter(wfb_engine_t *e, const wfb_functors_t *f,
                   const void *tuples_in, const uint64_t *ts_in, uint32_t n,
                   void *tuples_out, uint64_t *ts_out, uint32_t *n_out_dev, void *stream);

/* The same operator over K queued batches in ONE launch (a replica that finds several batches on its input channel):
 * batch i is compacted into (out[i].tuples, out[i].ts) and its survivor count written to n_out_dev[i]; results are
 * identical to K wfb_map_filter calls. in[i].ts may be NULL (then out[i].ts is not written). out[i].tuples may be
 * in[i].tuples (in-place compaction of every batch). */
int wfb_map_filter_batches(wfb_engine_t *e, const wfb_functors_t *f, const wfb_batch_t *in_h, const wfb_batch_t *out_h,
                           uint32_t nbatches, uint32_t *n_out_dev, void *stream);

/* ---- FlatMap_GPU: [map ->] [filter ->] flatmap(tuple, shipper) pushing 0..max_per_tuple result_t records per tuple ---------
 * (wf/flatmap.hpp, wf/shipper.hpp). K queued batches in ONE launch: batch i expands into out[i] (capacity >= in[i].n *
 * max_per_tuple result records; out[i].ts written when in[i].ts and out[i].ts are both non-null, every record with the timestamp
 * of the tuple that pushed it), in input order and, per tuple, in push order; the results are identical to K single-batch calls.
 * n_out_dev[i] = records of batch i, n_out_dev[nbatches] = pushes dropped because a tuple exceeded max_per_tuple (0 when none):
 * n_out_dev holds nbatches + 1 words. max_per_tuple >= 1 and in[i].n * max_per_tuple < 2^31 (WFB_E_BADARG otherwise). The
 * functor may run more than once per tuple: it must push the same records every time. `f` is the program's params_t, whose
 * map / filter run in front as in wfb_map_filter_batches. Programs without a flatmap functor: WFB_E_UNSUPPORTED. */
int wfb_flatmap_batches(wfb_engine_t *e, const wfb_functors_t *f, const wfb_batch_t *in_h, const wfb_batch_t *out_h, uint32_t nbatches,
                        uint32_t max_per_tuple, uint32_t *n_out_dev, void *stream);

/* ---- Map_GPU / Filter_GPU, keyed-stateful ------------------------------------------------------------------------
 * func(tuple, state_of_key) applied in per-key arrival order; a key's state (the program's state_t, zero-initialised) lives
 * in the handle, which the replicas of one operator share (they see disjoint keys). K queued batches per call; arrival
 * order = batch order, then index order. max_keys up to 2^30 (WFB_E_UNSUPPORTED above): up to 65536 keys the items are
 * split into buckets of at most 64 keys, above that they are sorted by key slot; the results are the same. replaces
 * Stateful_MAPGPU_Kernel / Stateful_FILTERGPU_Kernel + the TBB key map, spinlock and per-key state allocation,
 * wf/map_gpu.hpp:80-102, :212-299, wf/filter_gpu.hpp:91-117, :247-355. */
typedef struct wfb_kstate wfb_kstate_t;
int wfb_kstate_create(wfb_kstate_t **h, int prog, uint32_t max_keys, uint32_t flags /* WFB_FFAT_DENSE_KEYS or WFB_KEYS_GROW */);
int wfb_kstate_destroy(wfb_kstate_t *h);
/* Current key capacity (max_keys, or what a WFB_KEYS_GROW handle has grown to). Host-side: does not synchronise. */
uint32_t wfb_kstate_key_capacity(const wfb_kstate_t *h);
/* Map_GPU: in place. */
int wfb_map_stateful(wfb_kstate_t *h, const wfb_functors_t *f, const wfb_batch_t *batches_h, uint32_t nbatches, void *stream);
/* Filter_GPU: the functor may modify the tuple; survivors of batch i are compacted (stable) into (out[i].tuples, out[i].ts),
 * n_out_dev[i] of them. out[i] must not alias in[i]. */
int wfb_filter_stateful(wfb_kstate_t *h, const wfb_functors_t *f, const wfb_batch_t *in_h, const wfb_batch_t *out_h, uint32_t nbatches,
                        uint32_t *n_out_dev, void *stream);

/* ---- Reduce_GPU, per batch -------------------------------------------------------------------------
 * keyed: one output item per distinct key, ascending key order (floating-point keys: numeric, NaN last; other keys that are not
 * integers: their bytes read as a little-endian unsigned integer), tuple = fold of the program's reduce functor
 * over the key's items, ts = max ts. replaces Extract_Keys_Kernel + sort_by_key + reduce_by_key + D2D,
 * wf/reduce_gpu.hpp:75-105, :226-262. */
int wfb_reduce_by_key(wfb_engine_t *e, const void *tuples, const uint64_t *ts, uint32_t n,
                      void *out_tuples, uint64_t *out_ts, uint32_t *n_out_dev, void *stream);
/* The same operator over K queued batches in ONE launch sequence: batch i reduced into (out[i].tuples, out[i].ts) with
 * n_out_dev[i] items (ascending key); results are identical to K wfb_reduce_by_key calls. Keys must fit the engine's
 * key_bits (wfb_engine_set_key_bits) and key_bits + ceil(log2 K) <= 64. */
int wfb_reduce_by_key_batches(wfb_engine_t *e, const wfb_batch_t *in_h, const wfb_batch_t *out_h, uint32_t nbatches,
                              uint32_t *n_out_dev, void *stream);
/* un-keyed: whole batch -> one item. replaces thrust::reduce, wf/reduce_gpu.hpp:264-286. */
int wfb_reduce_all(wfb_engine_t *e, const void *tuples, const uint64_t *ts, uint32_t n,
                   void *out_tuple, uint64_t *out_ts, void *stream);

/* ---- KeyBy_Emitter_GPU grouping (GPU->GPU) -----------------------------------------------------------
 * start_idxs[k] = first index of the k-th distinct key (ascending key order), map_idxs[i] = next index with
 * the same key or -1, dist_keys[k] = the key; *n_keys_dev = number of distinct keys.
 * replaces Extract_Dests_Kernel + sort_by_key + Compute_Mapping_Kernel + unique_by_key_copy,
 * wf/keyby_emitter_gpu.hpp:68-100, :519-583. */
/* integral keys only (WFB_E_UNSUPPORTED otherwise), as for wfb_shard_by_key, wfb_shard_lift and wfb_mg_create */
int wfb_keyby_group(wfb_engine_t *e, const void *tuples, uint32_t n,
                    int32_t *start_idxs, int32_t *map_idxs, uint64_t *dist_keys, uint32_t *n_keys_dev,
                    void *stream);

/* ---- key -> shard partition (stands in for keyby_emitter_gpu when the pipeline spans > 1 GPU) ---------
 * dest = key % num_shards (wf/keyby_emitter.hpp:215-217, wf/keyby_emitter_gpu.hpp:621). Stable: within a
 * shard segment items keep arrival order. seg_off_dev[num_shards + 1] = exclusive offsets (device). */
int wfb_shard_by_key(wfb_engine_t *e, const void *tuples, const uint64_t *ts, uint32_t n, uint32_t num_shards,
                     void *out_tuples, uint64_t *out_ts, uint32_t *seg_off_dev, void *stream);

/* Fused source side of the multi-GPU keyby: [Map_GPU -> Filter_GPU ->] lift of `nbatches` batches and stable partition
 * of the lifted results by key % num_shards (num_shards <= 8) in ONE pass. Shard d's records land, in arrival order, at
 * out_regions + d * region_capacity * result_bytes; counts_dev[d] = records of shard d, counts_dev[8] != 0 => a region
 * overflowed (records beyond region_capacity are dropped). counts_dev must hold 9 uint32. */
int wfb_shard_lift(wfb_engine_t *e, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches, uint32_t num_shards,
                   void *out_regions, uint32_t region_capacity, uint32_t *counts_dev, void *stream);

/* ---- Ffat_Windows_GPU ------------------------------------------------------------------------------------
 * Per-replica handle: owns the key table and, per key, the count, the open-pane accumulator and the FlatFAT
 * (pane ring + internal levels). replaces Key_Descriptor / FlatFAT_GPU allocation,
 * wf/ffat_replica_gpu.hpp:438-506, wf/flatfat_gpu.hpp:165-192.
 *   win_type: 0 count-based (win/slide in tuples, wfb_ffat_process_cb), 1 time-based (win/slide/lateness in timestamp
 *             units, wfb_ffat_process_tb)
 *   flags   : WFB_FFAT_DENSE_KEYS => keys are known to be < max_keys (slot = key, no hash probe); integral keys only (WFB_E_BADARG) */
#define WFB_FFAT_DENSE_KEYS 1u
/*   WFB_FFAT_PIPELINED  => results are delivered one call late: wfb_ffat_process_cb(segment k) returns the results of
 *                          segment k-1 (none on the first call) while sort + update of segment k run on an internal stream and
 *                          overlap the ingest pass of segment k+1; wfb_ffat_flush returns the last segment's results. The
 *                          set of results over the whole stream is identical to the non-pipelined mode. */
#define WFB_FFAT_PIPELINED 2u
/*   WFB_KEYS_GROW       => max_keys is the initial capacity: the key table and every per-key array grow on demand (the reference's
 *                          key maps grow on the host, wf/ffat_replica_gpu.hpp:783-790, wf/map_gpu.hpp:236-240). A call that meets more
 *                          keys than the capacity grows it to a power of two >= 2 * max(keys, capacity) and reruns its key lookup; slots
 *                          are kept, so every key's state survives. The only cost on calls that do not grow is one 8-byte device-to-host
 *                          copy the host waits for. A growth that cannot allocate returns WFB_E_CAPACITY and leaves the handle as it was.
 *                          Also accepted by wfb_kstate_create. Not with WFB_FFAT_DENSE_KEYS, WFB_FFAT_PIPELINED or a key shard
 *                          (WFB_E_BADARG). The doubling stops once at 65536 keys while the keys fit (the last capacity of the
 *                          bucket path), then doubles again up to 2^30, for every kind of handle. On a growing handle the integer key
 *                          2^64-1 (the free-entry marker) is refused with error bit 0, as the all-ones 16-byte key is. */
#define WFB_KEYS_GROW 4u
int wfb_ffat_create(wfb_ffat_t **h, int prog, uint64_t win, uint64_t slide, uint32_t wins_per_batch,
                    uint32_t max_keys, int win_type, uint64_t lateness, uint32_t flags);
int wfb_ffat_destroy(wfb_ffat_t *h);
uint64_t wfb_ffat_launches(const wfb_ffat_t *h);
/* params_t of a registered program used by the key extractor, lift and combine (see wfb_engine_set_params). */
int wfb_ffat_set_params(wfb_ffat_t *h, const void *params, size_t bytes);
uint64_t wfb_ffat_state_bytes(const wfb_ffat_t *h);
/* Dense-key handle that owns one shard of a keyby (keys with key % num_shards == shard, the routing rule of
 * wf/keyby_emitter.hpp:215-217 for integer keys): key -> slot key / num_shards, so max_keys counts the shard's keys only.
 * A key of another shard sets the capacity error flag. Call before the first batch. */
int wfb_ffat_set_key_shard(wfb_ffat_t *h, uint32_t num_shards, uint32_t shard);

/* Count-based windows over `nbatches` consecutive input batches (one stream segment). Per key, items are
 * appended in arrival order; whenever the key's count reaches the trigger (first (Nb-1)*slide+win, then every
 * slide*Nb) Nb results result_t(key, gwid) folded over [gwid*slide, gwid*slide+win) are emitted with
 * ts = watermark of the batch holding the triggering item. Nothing is flushed at end of stream.
 * `pre` (may be NULL) fuses a chain of stateless Map_GPU -> Filter_GPU in front of the lift.
 * Results are appended to out_results/out_ts (capacity out_capacity) in groups of Nb per key; the order of the
 * groups is unspecified. *n_out_dev (device uint32) = number of results of this call.
 * replaces Ffat_Replica_GPU::process_batch_cb + process_wins_cb and FlatFAT_GPU::add_cb/build/update/
 * computeResults, wf/ffat_replica_gpu.hpp:734-867, wf/flatfat_gpu.hpp:226-252, :338-419. */
int wfb_ffat_process_cb(wfb_ffat_t *h, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches,
                        void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev,
                        void *stream);

/* Time-based windows (handles created with win_type = 1; win / slide / lateness in timestamp units).
 * Every batch must carry its timestamps; batches are processed one after the other. Per batch: tuples are assigned to panes
 * ts / gcd(win, slide), per-(key, pane) partials are merged into the key's pending panes, and for every key PRESENT in the
 * batch the groups of panes the watermark has completed (panes < (watermark - lateness) / pane length; first (Nb-1)*slide+win
 * panes, then slide*Nb) fire Nb windows each, ts = the batch watermark. Tuples of panes already consumed are dropped.
 * replaces Ffat_Replica_GPU::process_batch_tb + process_wins_tb, PendingPanes_Queue and Lifting_Kernel_TB_Keyed,
 * wf/ffat_replica_gpu.hpp:150-171, :214-420, :870-1047. Synchronises the stream once per batch (so does the reference, :962). */
int wfb_ffat_process_tb(wfb_ffat_t *h, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches,
                        void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, void *stream);

/* Pipelined handles only: deliver the results of the last segment (a no-op with *n_out_dev = 0 otherwise). */
int wfb_ffat_flush(wfb_ffat_t *h, void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, void *stream);

/* Per-phase device timing of wfb_ffat_process_cb calls (CUDA events recorded on the launching stream).
 * enable != 0 starts recording (up to 512 calls); the call returns, for the calls recorded since the last query,
 * ms_h[0] = streaming ingest pass, ms_h[1] = key offsets + radix sort, ms_h[2] = window update, ms_h[3] = whole
 * call, and *calls_h = number of calls summed. Synchronises on the last recorded event. */
int wfb_ffat_timing(wfb_ffat_t *h, int enable, float *ms_h, uint32_t *calls_h);

/* Number of distinct keys seen so far / error flags raised on the device (synchronises the stream). Flags: bit 0 more keys than the
 * capacity (fixed handles), bit 1 more results than out_capacity, bit 2 pane id out of range (time-based), bit 3 the key table must
 * grow (growing handles: set only while a growth that returned WFB_E_CAPACITY is pending). */
int wfb_ffat_stats(wfb_ffat_t *h, uint32_t *n_keys_h, uint32_t *err_flags_h, void *stream);
/* Current key capacity (max_keys, or what a WFB_KEYS_GROW handle has grown to). Host-side: does not synchronise. */
uint32_t wfb_ffat_key_capacity(const wfb_ffat_t *h);
/* Window results delivered by the handle since it was created (summed on the device by the last kernel of every call; synchronises
 * the stream). Lets a caller account for results without reading *n_out_dev back after every call (the role of the
 * outputs_sent counter of wf/stats_record.hpp:80-82). A WFB_FFAT_PIPELINED handle counts a segment's results when its window update
 * runs, one call before it delivers them: after wfb_ffat_flush the total is what was delivered. */
int wfb_ffat_results_total(wfb_ffat_t *h, uint64_t *total_h, void *stream);

/* ---- the pipeline sharded by key across the GPUs of one box (no counterpart in the reference: it drives one device) ----------------
 * One process (or thread) per GPU, `nranks` of them. Global step t of the stream covers nranks * K consecutive batches; rank r
 * ingests the K batches [r K, (r+1) K) of that span. Per step and rank: [Map_GPU -> Filter_GPU ->] lift and a stable partition
 * of the lifted results by key % nranks (wf/keyby_emitter.hpp:215-217), an all-to-all of the partitions (NCCL send/recv over
 * NVLink), and the rank's Ffat_Windows_GPU replica on the keys with key % nranks == rank, fed the received chunks in source-rank
 * order = global stream order (every count window equals the single-GPU one). Stands in for KeyBy_Emitter_GPU between the
 * replicas of different devices. NCCL is looked up at run time (dlopen "libnccl.so.2"): WFB_E_UNSUPPORTED when it is missing.
 * Exchange: when every rank's slots fit 16 bits together (max_keys_total, rounded up per rank to a power of two, times nranks <= 65536)
 * the SOURCE partitions its surviving records by (destination, bucket of the destination's slot space) in its one partition pass, and
 * the destination only concatenates the runs it receives, source after source, bucket by bucket -- it runs no partition of its own;
 * otherwise the source partitions by destination and the destination partitions what it received (WFB_MG_BUCKETED=0 forces this).
 * Transport: at the first step every rank allocates its receive buffers (sized for the worst case of THAT step: a later step may not
 * carry more tuples than the first one, WFB_E_CAPACITY) and maps its peers' buffers (cudaIpc: the ranks are processes of one node);
 * the records are then pushed with device-to-device copies over NVLink and a 4-byte NCCL token round signals completion. When the
 * buffers cannot be mapped, or with WFB_MG_CE=0, an NCCL send/recv group carries the records instead (buffers then grow on demand).
 * WFB_MG_TRACE=1 prints the device timeline of a step and the host time spent issuing it, per rank, every 64 steps (stderr).
 * The exchange of step t is issued behind the source pass of step t+2 and its window update behind that of step t+3, so results arrive THREE steps late
 * (wfb_mg_flush delivers the rest, appended in step order). Neither the host nor the compute stream ever waits for an exchange: the sizes
 * the host needs are a step old when it reads them, and a step's records have a whole step to arrive before they are read. */
typedef struct wfb_mg wfb_mg_t;
int wfb_mg_unique_id(void *id128_h);   /* rank 0: an ncclUniqueId (128 bytes) to hand to the other ranks (broadcast it with the launcher's means) */
int wfb_mg_create(wfb_mg_t **h, int prog, int nranks, int rank, const void *id128_h, uint64_t win, uint64_t slide, uint32_t wins_per_batch,
                  uint32_t max_keys_total /* keys 0 .. max_keys_total-1 over all ranks */);
int wfb_mg_destroy(wfb_mg_t *h);
/* params_t of the program (see wfb_engine_set_params), on every rank: used by the source side of a step that passes no `pre` and, always,
 * by the destination side -- the key extractor on the received records and the window update's comb and make_result. Call before the
 * first step; until then both sides use all-zero params. */
int wfb_mg_set_params(wfb_mg_t *h, const void *params, size_t bytes);
/* this rank's K batches of the next global step; the window results of the step three calls back go to out_results / out_ts (none on the first three calls).
 * `watermark`: the watermark of the segment (result timestamps carry the watermark of the source segment that held the triggering item). */
int wfb_mg_step(wfb_mg_t *h, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches, uint64_t watermark,
                void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, void *stream);
int wfb_mg_flush(wfb_mg_t *h, void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, void *stream);
/* launches so far (source engine + window operator) / device error flags of the window operator and results delivered (synchronises) */
uint64_t wfb_mg_launches(const wfb_mg_t *h);
int wfb_mg_stats(wfb_mg_t *h, uint32_t *err_flags_h, uint64_t *results_total_h, void *stream);

/* ---- synthetic stream (SURVEY.md 8d), generated on the device for tests and bench --------------------------
 * key_mode: 0 i % nkeys, 1 splitmix64(i) % nkeys, 2 zipf via zipf_cdf (device, nkeys doubles) */
int wfb_gen_tuple64(uint64_t seed, uint64_t start, uint32_t n, int key_mode, uint64_t nkeys,
                    const double *zipf_cdf, void *tuples, uint64_t *ts, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* WFB200_H */
