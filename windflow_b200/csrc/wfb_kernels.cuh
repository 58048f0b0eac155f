// wfb_kernels.cuh -- hand-written sm_90a kernels of the WindFlow GPU operator hot path, templated on a
// "program" (record schema + functors, see wfb_programs.cuh).
//
// Kernel inventory (DESIGN.md sections 3-4 have the algorithms and the measured roofline of each):
//   k_tile_pass<P, MODE>     streaming tile pass, persistent warp-specialised CTAs: TMA load of a tile of tuples
//                            (cp.async.bulk.tensor / cp.async.bulk + mbarrier rings), per-tuple map / filter / lift / key->slot
//                            in registers, survivors staged in shared memory, TMA bulk store.
//                              MODE_MAP     in-place Map_GPU                 (wf/map_gpu.hpp:61-76)
//                              MODE_FILTER  [Map_GPU ->] Filter_GPU, compacted per batch with a decoupled look-back
//                                           (wf/filter_gpu.hpp:72-88, :555-570)
//                              MODE_INGEST  [Map -> Filter ->] lift + key->slot for Ffat_Windows_GPU, or -> destination for
//                                           wfb_shard_lift (wf/ffat_replica_gpu.hpp:94-121); chain-free ("sparse") on the bucket path
//                              MODE_FLATMAP [Map -> Filter ->] FlatMap_GPU: 0..m result records per tuple, stable per batch
//                                           (count pass, CTA scan, decoupled look-back, emit pass; wf/flatmap.hpp, wf/shipper.hpp)
//   k_wide_tile_hist / k_wide_scatter / k_shard_scatter   one stable partition pass on a 10-bit digit (window path: 1024
//                            buckets of slots; multi-GPU: destinations, with the records)
//   k_ffat_update_buckets<P> one CTA per bucket: split by key, ordered pane folds, FlatFAT leaf + path update, fired
//                            groups (wf/flatfat_gpu.hpp:62-139, wf/ffat_replica_gpu.hpp:830-867); k_ffat_windows<P> window queries
//   k_onesweep_pass / k_radix_ghist   LSD radix sort, 8 bits per pass, one kernel per pass: the replacement of
//                            thrust::sort_by_key for the per-batch keyed operators and the full-sort window path
//                            (wf/ffat_replica_gpu.hpp:751, wf/keyby_emitter_gpu.hpp:547, wf/reduce_gpu.hpp:239)
//   k_ffat_update_lanes / k_ffat_update   full-sort window path: one thread / one warp per key
//   k_extract_keys, k_seg_*, k_reduce_segments*, k_reduce_all, k_gather_tuples   KeyBy_Emitter_GPU grouping, Reduce_GPU
#pragma once
#include <type_traits>
#include <iterator>
#include <cstdint>
#include <cstring>
#include <cuda.h>
#include <cuda_runtime.h>
#include "wfb_ptx.cuh"
#include "wfb_keys.cuh"

namespace wfb {

// the canonical words of a program's key (wfb_keys.cuh): uint64_t for keys of at most 8 bytes, Key128 for 9-16 bytes
template <class P> using key_codec = KeyCodec<typename P::key_t>;
template <class P> using key_words_t = typename key_codec<P>::words_t;
template <class P>
__host__ __device__ __forceinline__ key_words_t<P> key_words(const typename P::tuple_t &t, const typename P::params_t &prm)
{
    return key_codec<P>::encode(P::key(t, prm));
}

constexpr int TILE = 256;    // tuples per tile == threads per CTA of k_tile_pass
constexpr uint32_t OSW_TILE_POS = 4096; // positions per tile of the wide partition pass (== OSW_TILE below)
#ifndef WFB_STAGES
#define WFB_STAGES 4
#endif
constexpr int STAGES = WFB_STAGES;    // TMA ring depth per CTA
constexpr uint32_t FULL = 0xffffffffu;

enum { MODE_MAP = 0, MODE_FILTER = 1, MODE_INGEST = 2, MODE_FLATMAP = 3 };
constexpr uint32_t MAX_SHARDS = 8;

// decoupled look-back tile state: [63:34] epoch, [33:32] status, [31:0] value
constexpr uint64_t ST_AGG = 1, ST_PREFIX = 2;
__host__ __device__ __forceinline__ uint64_t pack_state(uint32_t epoch, uint64_t status, uint32_t v)
{
    return (static_cast<uint64_t>(epoch & 0x3fffffffu) << 34) | (status << 32) | v;
}

// one input batch as the kernels see it
struct DevBatch {
    const unsigned char *tuples;
    const uint64_t *ts;
    unsigned char *out;        // MODE_FILTER/MAP: output tuples
    uint64_t *ts_out;          // MODE_FILTER: output timestamps (may be null)
    uint32_t *n_out;           // MODE_FILTER: survivors of this batch (device)
    uint64_t watermark;
    uint32_t n;
    uint32_t tile_begin;       // first global tile index of this batch
};

// one fired window group whose Nb window queries are evaluated after the update kernel. `key` holds the key of a one-word program;
// a group of a two-word program reads its key from FfatDev::slot_key[slot] (trig_key below).
struct Trigger { uint64_t key; uint64_t g; uint32_t slot; uint32_t last_pos; uint32_t obase; uint32_t pad; };

// key -> slot table (open addressing, linear probing) + per-key window state of one Ffat_Windows_GPU
struct FfatDev {
    // key table (entries and slot keys are key_codec<P>::words words wide: one 8-byte word, or two for a 16-byte key)
    uint64_t *ht_keys;         // capacity entries, EMPTY_KEY when free
    uint32_t *ht_slots;        // capacity entries, INVALID_SLOT until published
    uint32_t ht_mask;          // capacity - 1
    uint32_t max_keys;
    uint32_t *n_slots;         // number of keys inserted so far
    uint32_t *err_flags;       // bit0: key table full, bit1: output capacity exceeded, bit2: pane ring overflow (time-based), bit3: KEYS_GROW_FLAG
    unsigned long long *results_total; // window results delivered so far (added by the last kernel of every call)
    uint64_t defer_items;              // a fired group may wait for the deferred pass (k_ffat_windows*) while fewer than this many further items of
                                       // its key follow in the call: (spare ring leaves + 1) panes -- later panes then do not overwrite leaves it reads
    uint32_t dense;            // 1: slot = key (keys < max_keys), or key / key_div for one shard of a keyby
    uint32_t grow;             // 1: the key table grows (WFB_KEYS_GROW): a key beyond max_keys keeps its slot and raises KEYS_GROW_FLAG
    uint32_t key_div, key_rem; // dense: the handle owns the keys with key % key_div == key_rem (key_div <= 1: all keys)
    // per-slot state
    uint64_t *slot_key;        // key of each slot
    uint64_t *cnt;             // lifted results appended so far (Key_Descriptor::count)
    unsigned char *acc;        // open-pane accumulator, result_t per slot
    unsigned char *tree;       // FlatFAT per slot: (2*n_leaves-1) result_t, leaves first (level 0), root last
    uint32_t *seg_cnt;         // full-sort path only: items of the current stream segment per slot (TileArgs::count_keys; zeroed by the
                               // update kernels). The bucket path counts per key inside the bucket CTA instead.
    uint32_t *seg_off;         // exclusive offsets into the sorted segment, max_keys+1
    struct Trigger *trig;      // deferred window groups of the current segment (evaluated by k_ffat_windows)
    uint32_t *n_trig;          // number of deferred groups
    uint32_t trig_cap;
    uint32_t *heavy;           // slots with more than light_max items in the segment (handled warp-per-key)
    uint32_t *n_heavy;
    uint32_t light_max;        // 256 (a run-time value: as a constant, ptxas spills k_ffat_update_lanes)
    // window geometry (in tuples and in panes)
    uint64_t win, slide, B;    // B = (Nb-1)*slide + win  (ffat_replica_gpu.hpp:657)
    uint32_t nb;               // windows per trigger
    uint32_t pane;             // pane length P = gcd(win, slide) in tuples
    uint32_t wp, sp;           // window / slide in panes
    uint32_t n_leaves;         // power of two >= B / P
    uint32_t log_leaves;
    uint32_t lazy;             // 1: the update kernels only write the pane LEAVES of the key's FlatFAT; the internal levels a group of windows needs
                               // are built in shared memory when the group is evaluated (k_ffat_windows_lazy). A pane completes once per
                               // `pane` items but fires windows only once per slide * Nb items: maintaining log2(n) path nodes per pane in
                               // global memory costs more than rebuilding n - 1 nodes on chip per fired group.
};
constexpr uint64_t EMPTY_KEY = 0xffffffffffffffffull;
constexpr uint32_t INVALID_SLOT = 0xffffffffu;
// error flag of a growing handle: a key got a slot at or beyond max_keys, or found the key table full. Its items were not taken
// (INVALID_SLOT); the host grows the table and reruns the pass that inserts the keys (wfb_lib.cu, grow_keys). Cleared by the rebuild.
constexpr uint32_t KEYS_GROW_FLAG = 8u;

struct TileArgs {
    const DevBatch *batches;   // device array (nbatches entries) or null => use `one`
    DevBatch one;
    uint32_t nbatches;
    uint32_t num_tiles;
    uint64_t *tile_state;      // num_tiles words (epoch-tagged, never cleared)
    uint32_t *ticket;          // monotonically increasing ticket counter
    uint32_t ticket_base;      // value of *ticket when this launch starts
    uint32_t epoch;
    uint64_t tmap_base;        // global address the 2-D tensor map starts at (rows of 64 bytes)
    uint32_t use_tmap;         // 1: `tmap` is valid for this launch
    uint32_t max_ctas_per_sm;  // host-side launch hint (0 = no limit), not read by the kernel
    uint32_t sparse;           // MODE_INGEST, 1: no global compaction -- tile t owns lifted / slots [t*TILE, +TILE) (survivors first,
                               // INVALID_SLOT padding), so tiles are independent: no look-back chain, positions are tuple indices
    uint32_t count_keys;       // MODE_INGEST: 1 = per-key item counts of the segment (ff.seg_cnt) for the full-sort update kernels
    uint16_t *wide_h16;        // MODE_INGEST + sparse: per-tile digit counts of the wide partition ([position / 4096][1024], 16-bit rows), filed by
                               // the tile pass itself: with tiles_per_ticket = 16 a CTA owns whole wide tiles, counts their digits in shared
                               // memory and writes each row once -- the partition then needs no counting pass (k_wide_tile_hist) of its own
    uint32_t tiles_per_ticket; // consecutive tiles a producer claims per ticket (0 or 1: one; 16 with wide_h16)
    uint32_t pack_rank;        // with wide_h16 and at most 65536 slots: slots[pos] = slot | rank << 16, rank = what the digit counter of the wide
                               // tile held when this survivor was counted (any order among the survivors of one digit): k_wide_scatter_ranked
                               // places the pairs with it and then restores arrival order inside every (wide tile, digit) cell
    const uint32_t *ext_slots; // MODE_INGEST + in-place: slot of the record at every position, given by the caller (the time-based
                               // front end knows the key slot of every pane it pops); the program's key extractor is not used
    uint32_t inplace;          // MODE_INGEST + sparse, 1: the program passes records through unchanged (lift = identity, no map) and the
                               // batches lie at their tile positions in one buffer: nothing is copied, only the slots are written
    uint32_t l2_hints;         // 1: input tiles are loaded evict-first, lifted records stored evict-last (they are re-read by the update)
    // MODE_INGEST with nshards != 0 (wfb_shard_lift): the "slot" of a tuple is its destination key % nshards
    uint32_t nshards, region_cap;
    // ... and with shard_slots != 0 (bucketed exchange, wfb_mg_*): the "slot" is the VIRTUAL slot dest * shard_slots + key / nshards
    // (shard_slots a power of two, nshards * shard_slots <= 65536), so that ONE wide partition at the source leaves the records
    // grouped by (destination, bucket of the destination's slot space); keys at or above shard_keys * nshards raise *shard_err
    uint32_t shard_slots, shard_keys;
    uint32_t *shard_err;
    // MODE_INGEST: digit histograms of the slot sort that follows (RadixSorter ctl), accumulated per CTA in shared memory
    uint32_t *sort_ctl; uint32_t sort_passes, sort_shift, sort_dbits; // sort_dbits: digit width of a pass (8, or 10 for the wide pass)
    uint32_t max_per_tuple;    // MODE_FLATMAP: records kept per tuple (m >= 1; the word fills the padding before `lifted`)
    // MODE_INGEST outputs (compacted over the whole segment, arrival order)
    unsigned char *lifted;     // result_t per surviving tuple
    uint32_t *slots;           // slot per surviving tuple
    uint32_t *batch_off;       // nbatches+1: compact offset of the first survivor of each batch; [nbatches]=total
    uint32_t *n_total;         // == batch_off[nbatches]; MODE_FLATMAP: pushes dropped beyond max_per_tuple (added once per tile)
    FfatDev ff;
};

// The Shipper of a FlatMap functor: push(r) places record j (the j-th push of the tuple) at out[j] with the tuple's timestamp,
// for j < m; later pushes are only counted. With out == nullptr it only counts (the count pass of MODE_FLATMAP: the functor is
// inlined, so the stores vanish from that instance).
template <class R>
class Shipper {
    unsigned char *out; uint64_t *ts_out; uint64_t ts; uint32_t m, n;
public:
    __host__ __device__ Shipper(unsigned char *out_, uint64_t *ts_out_, uint64_t ts_, uint32_t m_): out(out_), ts_out(ts_out_), ts(ts_), m(m_), n(0) {}
    __host__ __device__ void push(const R &r)
    {
        if (out != nullptr && n < m) {
            store(out + static_cast<size_t>(n) * sizeof(R), r);
            if (ts_out != nullptr) ts_out[n] = ts;
        }
        n++;
    }
    __host__ __device__ uint32_t pushes() const { return n; } // every push, the dropped ones included
private:
    __host__ __device__ static void store(unsigned char *p, const R &r)
    {
        const unsigned char *src = reinterpret_cast<const unsigned char *>(&r);
        if constexpr (sizeof(R) % 16 == 0) {
            if ((reinterpret_cast<uintptr_t>(p) & 15u) == 0) { // (records of 16 * k bytes from a 16-byte aligned base: vector stores)
#pragma unroll
                for (uint32_t k = 0; k < sizeof(R) / 16; k++) { uint4 v; memcpy(&v, src + 16 * k, 16); reinterpret_cast<uint4 *>(p)[k] = v; }
                return;
            }
        }
#pragma unroll
        for (uint32_t k = 0; k < sizeof(R) / 8; k++) { uint64_t v; memcpy(&v, src + 8 * k, 8); reinterpret_cast<uint64_t *>(p)[k] = v; }
    }
};

// ------------------------------------------------------------------------------------------------------
// shared-memory tile access. A tuple of C = sizeof(T)/16 16-byte chunks is read/written with its chunks
// rotated by (idx*C/8)%C so that the 8 lanes of a quarter warp hit 8 different 16-byte bank groups
// (stride-64B LDS.128 would otherwise be a 4-way bank conflict).
// ------------------------------------------------------------------------------------------------------
template <class T>
struct TileIO {
    static constexpr int TB = sizeof(T);
    static constexpr bool V16 = (TB % 16 == 0) && (TB / 16 == 1 || TB / 16 == 2 || TB / 16 == 4 || TB / 16 == 8);
    static constexpr int C = V16 ? TB / 16 : TB / 8;

    __device__ __forceinline__ static void load(const unsigned char *base, uint32_t idx, T &out)
    {
        if constexpr (V16) {
            uint4 v[C];
            const uint4 *p = reinterpret_cast<const uint4 *>(base + static_cast<size_t>(idx) * TB);
            const uint32_t rot = (C > 1) ? ((idx * C / 8) % C) : 0;
#pragma unroll
            for (int j = 0; j < C; j++) v[j] = p[(j + rot) & (C - 1)];
            // v[j] holds chunk (j+rot)%C; rotate right by rot so that v[k] holds chunk k
#pragma unroll
            for (int s = 1; s < C; s <<= 1) {
                if (rot & s) {
                    uint4 t[C];
#pragma unroll
                    for (int k = 0; k < C; k++) t[k] = v[(k - s) & (C - 1)];
#pragma unroll
                    for (int k = 0; k < C; k++) v[k] = t[k];
                }
            }
            uint4 *o = reinterpret_cast<uint4 *>(&out);
#pragma unroll
            for (int k = 0; k < C; k++) o[k] = v[k];
        } else {
            const uint64_t *p = reinterpret_cast<const uint64_t *>(base + static_cast<size_t>(idx) * TB);
            uint64_t *o = reinterpret_cast<uint64_t *>(&out);
#pragma unroll
            for (int k = 0; k < C; k++) o[k] = p[k];
        }
    }

    __device__ __forceinline__ static void store(unsigned char *base, uint32_t idx, const T &in)
    {
        if constexpr (V16) {
            uint4 v[C];
            const uint4 *src = reinterpret_cast<const uint4 *>(&in);
#pragma unroll
            for (int k = 0; k < C; k++) v[k] = src[k];
            const uint32_t rot = (C > 1) ? ((idx * C / 8) % C) : 0;
            // rotate left by rot: v'[j] = chunk (j+rot)%C, then store v'[j] at position (j+rot)%C
#pragma unroll
            for (int s = 1; s < C; s <<= 1) {
                if (rot & s) {
                    uint4 t[C];
#pragma unroll
                    for (int k = 0; k < C; k++) t[k] = v[(k + s) & (C - 1)];
#pragma unroll
                    for (int k = 0; k < C; k++) v[k] = t[k];
                }
            }
            uint4 *p = reinterpret_cast<uint4 *>(base + static_cast<size_t>(idx) * TB);
#pragma unroll
            for (int j = 0; j < C; j++) p[(j + rot) & (C - 1)] = v[j];
        } else {
            uint64_t *p = reinterpret_cast<uint64_t *>(base + static_cast<size_t>(idx) * TB);
            const uint64_t *s = reinterpret_cast<const uint64_t *>(&in);
#pragma unroll
            for (int k = 0; k < C; k++) p[k] = s[k];
        }
    }
};

// global <-> shared tile movement: TMA bulk copy when size and address allow it, else coalesced 8-byte words
__device__ __forceinline__ bool bulk_ok(const void *g, uint32_t bytes)
{
    return ((reinterpret_cast<uintptr_t>(g) | bytes) & 15u) == 0;
}

// ------------------------------------------------------------------------------------------------------
// key -> slot lookup / insert (replaces the host unordered_map of ffat_replica_gpu.hpp:514, :783-795)
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t mix64(uint64_t x)
{
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}

template <class P>
__device__ __forceinline__ key_words_t<P> key_of_slot(const FfatDev &ff, uint32_t slot)
{
    if constexpr (key_codec<P>::words == 2) return reinterpret_cast<const Key128 *>(ff.slot_key)[slot]; // (never dense)
    else return ff.dense ? (ff.key_div > 1 ? static_cast<uint64_t>(slot) * ff.key_div + ff.key_rem : static_cast<uint64_t>(slot)) : ff.slot_key[slot];
}
// the key a Trigger carries (one-word keys only) and the key of a fired group
__device__ __forceinline__ uint64_t trig_word(uint64_t key) { return key; }
__device__ __forceinline__ uint64_t trig_word(const Key128 &) { return 0; }
template <class P>
__device__ __forceinline__ key_words_t<P> trig_key(const FfatDev &ff, const Trigger &tr)
{
    if constexpr (key_codec<P>::words == 2) return key_of_slot<P>(ff, tr.slot); else return tr.key;
}

// 16-byte keys: one 16-byte load per probe. The load may see an entry that a concurrent 16-byte CAS is writing half done, so an entry
// with an all-ones half -- free, half written, or a key with such a half -- is settled with the CAS (which returns the whole entry)
// before it is compared: a torn read never counts as a hit. The all-ones key itself marks a free entry: it is refused with the key
// table's capacity flag.
__device__ __forceinline__ uint32_t slot_of_key(const FfatDev &ff, const Key128 &key)
{
    if (key.lo == EMPTY_KEY && key.hi == EMPTY_KEY) { atomicOr(ff.err_flags, 1u); return INVALID_SLOT; }
    uint32_t h = static_cast<uint32_t>(mix64(key.lo ^ mix64(key.hi))) & ff.ht_mask;
    for (uint32_t probe = 0; probe <= ff.ht_mask; probe++) {
        uint64_t *e = ff.ht_keys + 2 * static_cast<size_t>(h);
        Key128 k;
        ld_relaxed_v2u64(e, k.lo, k.hi);
        if (k.lo == EMPTY_KEY || k.hi == EMPTY_KEY) {
            atom_cas_b128(e, EMPTY_KEY, EMPTY_KEY, key.lo, key.hi, k.lo, k.hi);
            if (k.lo == EMPTY_KEY && k.hi == EMPTY_KEY) { // we own the entry: allocate the slot and publish it
                uint32_t s = atomicAdd(ff.n_slots, 1u);
                if (s < ff.max_keys) reinterpret_cast<Key128 *>(ff.slot_key)[s] = key;
                else if (ff.grow) atomicOr(ff.err_flags, KEYS_GROW_FLAG); // (the rebuild at the new capacity writes slot_key[s])
                else { atomicOr(ff.err_flags, 1u); s = INVALID_SLOT - 1; }
                st_release_u32(&ff.ht_slots[h], s);
                return s >= ff.max_keys ? INVALID_SLOT : s;
            }
        }
        if (k == key) {
            uint32_t s;
            while ((s = ld_acquire_u32(&ff.ht_slots[h])) == INVALID_SLOT) { }
            if (s >= ff.max_keys) { if (ff.grow) atomicOr(ff.err_flags, KEYS_GROW_FLAG); return INVALID_SLOT; }
            return s;
        }
        h = (h + 1) & ff.ht_mask;
    }
    atomicOr(ff.err_flags, ff.grow ? KEYS_GROW_FLAG : 1u);
    return INVALID_SLOT;
}

__device__ __forceinline__ uint32_t slot_of_key(const FfatDev &ff, uint64_t key)
{
    if (ff.dense) {
        if (ff.key_div > 1) { // one shard of a keyby: keys with key % key_div == key_rem, compact slots
            if (key % ff.key_div != ff.key_rem) { atomicOr(ff.err_flags, 1u); return INVALID_SLOT; }
            key /= ff.key_div;
        }
        if (key >= ff.max_keys) { atomicOr(ff.err_flags, 1u); return INVALID_SLOT; }
        return static_cast<uint32_t>(key);
    }
    // the all-ones key marks a free entry: every insert of it would take a new slot. A growing table refuses it with the capacity flag
    // (as the 16-byte path does), so that it never grows the table
    if (ff.grow && key == EMPTY_KEY) { atomicOr(ff.err_flags, 1u); return INVALID_SLOT; }
    uint32_t h = static_cast<uint32_t>(mix64(key)) & ff.ht_mask;
    for (uint32_t probe = 0; probe <= ff.ht_mask; probe++) {
        uint64_t k = ld_relaxed_u64(&ff.ht_keys[h]);
        if (k == EMPTY_KEY) {
            unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long *>(&ff.ht_keys[h]),
                                               static_cast<unsigned long long>(EMPTY_KEY),
                                               static_cast<unsigned long long>(key));
            if (old == EMPTY_KEY) { // we own the entry: allocate the slot and publish it
                uint32_t s = atomicAdd(ff.n_slots, 1u);
                if (s < ff.max_keys) ff.slot_key[s] = key;
                else if (ff.grow) atomicOr(ff.err_flags, KEYS_GROW_FLAG); // (the rebuild at the new capacity writes slot_key[s])
                else { atomicOr(ff.err_flags, 1u); s = INVALID_SLOT - 1; }
                st_release_u32(&ff.ht_slots[h], s);
                return s >= ff.max_keys ? INVALID_SLOT : s;
            }
            k = old;
        }
        if (k == key) {
            uint32_t s;
            while ((s = ld_acquire_u32(&ff.ht_slots[h])) == INVALID_SLOT) { }
            if (s >= ff.max_keys) { if (ff.grow) atomicOr(ff.err_flags, KEYS_GROW_FLAG); return INVALID_SLOT; }
            return s;
        }
        h = (h + 1) & ff.ht_mask;
    }
    atomicOr(ff.err_flags, ff.grow ? KEYS_GROW_FLAG : 1u);
    return INVALID_SLOT;
}

// Rebuilds the key table of a growing handle at a new capacity (new_keys / new_slots all free, new_mask + 1 entries): every
// entry of the old table is inserted again with its slot -- slots are never renumbered, so the per-slot state moves with a prefix
// copy -- and slot_key (already the new, larger array) gets the keys of the slots at or beyond old_max_keys, which the old array
// had no room for. Keys are distinct: an insert claims the first free entry of its probe (16-byte entries with the 16-byte CAS,
// as slot_of_key does). Clears KEYS_GROW_FLAG.
static __global__ void __launch_bounds__(256) k_key_table_rebuild(const uint64_t *__restrict__ old_keys, const uint32_t *__restrict__ old_slots,
                                                           uint32_t old_mask, uint64_t *new_keys, uint32_t *__restrict__ new_slots, uint32_t new_mask,
                                                           uint64_t *__restrict__ slot_key, uint32_t old_max_keys, uint32_t words, uint32_t *err_flags)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAnd(err_flags, ~KEYS_GROW_FLAG);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= old_mask; i += gridDim.x * blockDim.x) {
        uint32_t h;
        const uint32_t s = old_slots[i];
        if (words == 2) {
            const Key128 k = reinterpret_cast<const Key128 *>(old_keys)[i];
            if (k.lo == EMPTY_KEY && k.hi == EMPTY_KEY) continue;
            h = static_cast<uint32_t>(mix64(k.lo ^ mix64(k.hi))) & new_mask;
            for (;; h = (h + 1) & new_mask) {
                uint64_t lo, hi;
                atom_cas_b128(new_keys + 2 * static_cast<size_t>(h), EMPTY_KEY, EMPTY_KEY, k.lo, k.hi, lo, hi);
                if (lo == EMPTY_KEY && hi == EMPTY_KEY) break;
            }
            if (s >= old_max_keys) reinterpret_cast<Key128 *>(slot_key)[s] = k;
        } else {
            const uint64_t k = old_keys[i];
            if (k == EMPTY_KEY) continue;
            h = static_cast<uint32_t>(mix64(k)) & new_mask;
            while (atomicCAS(reinterpret_cast<unsigned long long *>(&new_keys[h]), static_cast<unsigned long long>(EMPTY_KEY),
                             static_cast<unsigned long long>(k)) != EMPTY_KEY) h = (h + 1) & new_mask;
            if (s >= old_max_keys) slot_key[s] = k;
        }
        new_slots[h] = s;
    }
}

// ------------------------------------------------------------------------------------------------------
// k_tile_pass: persistent, warp-specialised CTAs (10 warps), dynamic tile tickets, STAGES-deep TMA ring.
//   warp 0      PRODUCER  (one lane): wait empty[s] | claim ticket | find the batch | TMA load of the tile:
//                         cp.async.bulk.tensor.2d with SWIZZLE_64B for full tiles of 64-byte tuples (bank-conflict
//                         free LDS.128 without register shuffling), cp.async.bulk (linear) otherwise; timestamps of
//                         the tile ride on the same mbarrier.
//   warps 1..8  CONSUMERS (one tuple per thread): wait full[s] | tuple -> registers | map | filter | [lift,
//                         key->slot, per-key count] | ballot + warp totals -> local offsets (one named barrier) |
//                         survivors -> shared (compacted, linear) | publish the tile count (look-back AGGREGATE) |
//                         arrive staged[s] and move on to the next tile.
//   warp 9      EPILOGUE: wait staged[s] | decoupled look-back -> tile base, publish PREFIX | one TMA bulk store of
//                         the compacted records, coalesced stores of the staged slots / timestamps | wait for the
//                         store to have read shared memory | arrive empty[s].
// Tickets: every CTA claims one ticket per processed tile plus the failing one, so a launch consumes exactly
// num_tiles + gridDim.x tickets (the host advances ticket_base by that amount). (Claiming several tiles per atomic was
// measured: it delays the aggregates the look-backs of the following tiles wait for, 0.10 -> 0.14 ms.)
// ------------------------------------------------------------------------------------------------------
constexpr uint32_t TP_THREADS = TILE + 64;         // producer warp + 8 consumer warps + epilogue warp
constexpr uint32_t TILE_SENTINEL = 0x7fffffffu;
enum { TF_SWZ = 1u, TF_FALLBACK = 2u, TF_TS_SMEM = 4u, TF_WIDE_LAST = 8u };

struct StageMeta {
    uint32_t tile, batch, first, cnt, flags, count; // count: survivors (written by the consumers)
    uint32_t wide, pad;                             // wide: ticket (= wide tile when tiles_per_ticket = 16)
};

constexpr uint32_t TP_SMEM_MAX = 232448; // opt-in dynamic shared memory of one block on sm_90 (227 KB)

// Shared memory of k_tile_pass<P, MODE>. The ring keeps STAGES stages while they fit TP_SMEM_MAX; larger records get 3, then 2
// (records of up to about 430 bytes); a record that does not fit twice fails to compile (launch_tile_pass).
template <class P, int MODE>
struct TilePassSmem {
    using T = typename P::tuple_t;
    using R = typename P::result_t;
    static constexpr uint32_t rec_bytes = (MODE == MODE_INGEST && sizeof(R) > sizeof(T)) ? sizeof(R) : sizeof(T);
    static constexpr uint32_t tile_bytes = (TILE * rec_bytes + 1023u) & ~1023u; // swizzled stages need 512-B alignment
    static constexpr uint32_t aux_bytes = (MODE == MODE_INGEST) ? TILE * 4u : (MODE == MODE_FILTER ? TILE * 16u : (MODE == MODE_FLATMAP ? TILE * 8u : 0u)); // slots | ts in + ts out | ts in
    static constexpr uint32_t stage_bytes = tile_bytes + aux_bytes;
    static constexpr uint32_t hist_bytes = (MODE == MODE_INGEST) ? 4u * 256u * 4u : 0u; // up to 4 sort passes of 8 bits or one of 10 | two buffers of 1024 packed 16-bit per-wide-tile counts
    static constexpr uint32_t total_at(uint32_t st) { return st * stage_bytes + 1024 /*alignment slack*/ + 1024 /*barriers, meta, scan*/ + hist_bytes; }
    static constexpr int stages = (STAGES <= 2 || total_at(STAGES) <= TP_SMEM_MAX) ? STAGES : ((STAGES > 3 && total_at(3) <= TP_SMEM_MAX) ? 3 : 2);
    static constexpr uint32_t total = total_at(stages);
};

__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const void *tmap, int32_t c0, int32_t c1, uint64_t *bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_2d_hint(void *smem_dst, const void *tmap, int32_t c0, int32_t c1, uint64_t *bar, uint64_t policy)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
                 ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const void *tmap, int32_t c0, int32_t c1, const void *smem_src)
{
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(tmap), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, %0;" ::"n"(TILE) : "memory"); }

// decoupled look-back of tile t > chain_begin (one whole warp): adds the sum of the published counts of tiles [chain_begin, t) to
// excl, read back from the nearest PREFIX (the chain's start acts as a PREFIX of 0)
__device__ __forceinline__ void lookback_exclusive(const TileArgs &a, uint32_t t, uint32_t chain_begin, uint32_t lane, uint32_t &excl)
{
    int64_t idx = static_cast<int64_t>(t) - 1;
    while (true) {
        const int64_t my = idx - lane;
        uint64_t w = pack_state(a.epoch, ST_PREFIX, 0); // virtual terminator below the chain start
        bool valid;
        do {
            valid = true;
            if (my >= static_cast<int64_t>(chain_begin)) {
                w = ld_relaxed_u64(&a.tile_state[my]);
                valid = ((w >> 34) == (a.epoch & 0x3fffffffu)) && (((w >> 32) & 3u) != 0);
            }
        } while (!__all_sync(FULL, valid));
        const uint32_t status = static_cast<uint32_t>(w >> 32) & 3u;
        const uint32_t pmask = __ballot_sync(FULL, status == ST_PREFIX);
        const uint32_t firstp = pmask ? (__ffs(pmask) - 1) : 32;
        uint32_t v = (lane <= firstp) ? static_cast<uint32_t>(w) : 0u;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
        excl += v;
        if (pmask) break;
        idx -= 32;
    }
}

template <class P, int MODE>
__global__ void __launch_bounds__(TP_THREADS) k_tile_pass(const __grid_constant__ CUtensorMap tmap, const TileArgs a,
                                                          const __grid_constant__ typename P::params_t prm)
{
    using T = typename P::tuple_t;
    using R = typename P::result_t;
    using SM = TilePassSmem<P, MODE>;
    constexpr uint32_t TB = sizeof(T);
    constexpr uint32_t RB = sizeof(R);
    static_assert(TB % 8 == 0 && RB % 8 == 0, "records must be multiples of 8 bytes");
    constexpr bool CAN_SWZ = (TB == 64);

    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    unsigned char *ctl = smem + SM::stages * SM::stage_bytes;        // (SM::stages: the ring depth of this record size)
    uint64_t *full = reinterpret_cast<uint64_t *>(ctl);              // stages  producer -> consumers (tx)
    uint64_t *staged = full + SM::stages;                            // stages  consumers -> epilogue
    uint64_t *empty = staged + SM::stages;                           // stages  epilogue -> producer
    StageMeta *meta = reinterpret_cast<StageMeta *>(empty + SM::stages);  // stages
    uint32_t *warp_tot = reinterpret_cast<uint32_t *>(meta + SM::stages); // 2 x 8 warp totals (double-buffered by iteration parity)
    uint32_t *fm_words = warp_tot + 2 * (TILE / 32);                  // MODE_FLATMAP: 2 x 8 warp drop counts, then 2 tile bases
    uint32_t *s_hist = reinterpret_cast<uint32_t *>(ctl + 1024);      // MODE_INGEST: [pass][1 << sort_dbits] digit counts of this CTA (1024 words)

    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    auto stage_buf = [&](uint32_t s) { return smem + s * SM::stage_bytes; };
    auto stage_aux = [&](uint32_t s) { return smem + s * SM::stage_bytes + SM::tile_bytes; };

    if (tid == 0) {
        for (int s = 0; s < SM::stages; s++) { mbar_init(&full[s], 1); mbar_init(&staged[s], TILE / 32); mbar_init(&empty[s], 1); }
        mbar_fence_init();
    }
    if constexpr (MODE == MODE_INGEST) { for (uint32_t i = tid; i < 4u * 256u; i += TP_THREADS) s_hist[i] = 0; }
    __syncthreads();

    if (warp == 0) {
        // ================================= PRODUCER =================================
        if (lane == 0) {
            const uint64_t pol_first = l2_policy_evict_first();
            DevBatch b = a.one; uint32_t bi = 0, b_end = 0; // batch of the previous tile, first tile after it
            bool have_batch = false;
            const uint32_t tpt = a.tiles_per_ticket ? a.tiles_per_ticket : 1u;
            uint32_t t_next = 0, t_end = 0, claim = 0; // tiles [t_next, t_end) of the current claim are still to load
            for (uint32_t it = 0;; it++) {
                const uint32_t s = it % SM::stages, par = (it / SM::stages) & 1u;
                mbar_wait(&empty[s], par ^ 1u); // a fresh barrier passes the wait on parity 1
                // claim only now: a claimed tile is loaded at once, so the look-backs of its successors never wait on a stalled ring
                StageMeta &m = meta[s];
                if (t_next == t_end) {
                    claim = atomicAdd(a.ticket, 1u) - a.ticket_base;
                    t_next = claim * tpt; // (claim <= (num_tiles + grid) / tpt: no overflow)
                    if (claim >= (a.num_tiles + tpt - 1) / tpt) { m.tile = TILE_SENTINEL; mbar_arrive(&full[s]); break; }
                    t_end = min(t_next + tpt, a.num_tiles);
                }
                const uint32_t t = t_next++;
                if (a.batches != nullptr && !(have_batch && t >= b.tile_begin && t < b_end)) {
                    uint32_t lo = 0, hi = a.nbatches - 1; // last batch with tile_begin <= t
                    while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (a.batches[mid].tile_begin <= t) lo = mid; else hi = mid - 1; }
                    bi = lo; b = a.batches[lo];
                    b_end = (lo + 1 < a.nbatches) ? a.batches[lo + 1].tile_begin : a.num_tiles;
                    have_batch = true;
                }
                const uint32_t first = (t - b.tile_begin) * TILE;
                const uint32_t cnt = min(static_cast<uint32_t>(TILE), b.n - first);
                const unsigned char *src = b.tuples + static_cast<size_t>(first) * TB;
                uint32_t flags = 0, tx = 0;
                const uint64_t off = reinterpret_cast<uint64_t>(src) - a.tmap_base;
                if (CAN_SWZ && a.use_tmap && cnt == TILE && (off & 63u) == 0 && (off >> 6) < 0x7fffff00ull) flags = TF_SWZ;
                else if (!bulk_ok(src, cnt * TB)) flags = TF_FALLBACK;
                if (!(flags & TF_FALLBACK)) tx += cnt * TB;
                const uint64_t *tsp = ((MODE == MODE_FILTER || MODE == MODE_FLATMAP) && b.ts != nullptr) ? b.ts + first : nullptr;
                if (tsp != nullptr && bulk_ok(tsp, cnt * 8u)) { flags |= TF_TS_SMEM; tx += cnt * 8u; }
                if (t_next == t_end) flags |= TF_WIDE_LAST;
                m.tile = t; m.batch = bi; m.first = first; m.cnt = cnt; m.flags = flags; m.wide = claim;
                if (tx) mbar_expect_tx(&full[s], tx); else mbar_arrive(&full[s]);
                if (a.l2_hints) { // read-once stream: first in line for eviction
                    if (flags & TF_SWZ) tma_load_2d_hint(stage_buf(s), &tmap, 0, static_cast<int32_t>(off >> 6), &full[s], pol_first);
                    else if (!(flags & TF_FALLBACK)) bulk_g2s_hint(stage_buf(s), src, cnt * TB, &full[s], pol_first);
                } else if (flags & TF_SWZ) tma_load_2d(stage_buf(s), &tmap, 0, static_cast<int32_t>(off >> 6), &full[s]);
                else if (!(flags & TF_FALLBACK)) bulk_g2s(stage_buf(s), src, cnt * TB, &full[s]);
                if (flags & TF_TS_SMEM) bulk_g2s(stage_aux(s), tsp, cnt * 8u, &full[s]);
            }
        }
    } else if (warp <= TILE / 32) {
        // ================================= CONSUMERS =================================
        const uint32_t ctid = tid - 32, cwarp = warp - 1;
        uint32_t wpar = 0; // which of the two digit-count buffers the current wide tile uses
        for (uint32_t it = 0;; it++) {
            const uint32_t s = it % SM::stages, par = (it / SM::stages) & 1u;
            unsigned char *buf = stage_buf(s);
            mbar_wait(&full[s], par);
            const StageMeta m = meta[s];
            if (m.tile == TILE_SENTINEL) { // pass the end-of-work marker on to the epilogue warp
                __syncwarp();
                if (lane == 0) mbar_arrive(&staged[s]);
                if constexpr (MODE == MODE_INGEST) {
                    if (a.sort_ctl != nullptr) { // every consumer is done counting: add this CTA's digit counts to the global ones
                        consumer_bar();
                        for (uint32_t i = ctid; i < (a.sort_passes << a.sort_dbits); i += TILE) { const uint32_t c = s_hist[i]; if (c) atomicAdd(&a.sort_ctl[i], c); }
                    }
                }
                break;
            }
            DevBatch b;
            if (a.batches == nullptr) b = a.one; else b = a.batches[m.batch];
            const uint32_t cnt = m.cnt;
            const bool active = ctid < cnt;
            if (m.flags & TF_FALLBACK) { // unaligned / odd-sized tile: coalesced 8-byte copies into the linear buffer
                const uint64_t *src = reinterpret_cast<const uint64_t *>(b.tuples + static_cast<size_t>(m.first) * TB);
                uint64_t *dst = reinterpret_cast<uint64_t *>(buf);
                for (uint32_t w = ctid; w < cnt * (TB / 8); w += TILE) dst[w] = src[w];
                consumer_bar();
            }
            // ---- per-tuple work in registers ---------------------------------------------------------------
            alignas(16) T tup;
            uint64_t ts = 0;
            bool keep = false;
            if (active) {
                if constexpr (CAN_SWZ) {
                    if (m.flags & TF_SWZ) { // SWIZZLE_64B: 16-byte chunk j of row r lives at chunk j ^ ((r >> 1) & 3)
                        const uint4 *p = reinterpret_cast<const uint4 *>(buf + static_cast<size_t>(ctid) * 64);
                        const uint32_t x = (ctid >> 1) & 3u;
                        uint4 *o = reinterpret_cast<uint4 *>(&tup);
#pragma unroll
                        for (uint32_t jj = 0; jj < 4; jj++) o[jj] = p[jj ^ x];
                    } else TileIO<T>::load(buf, ctid, tup);
                } else TileIO<T>::load(buf, ctid, tup);
                if constexpr (MODE == MODE_FILTER || MODE == MODE_FLATMAP) {
                    if (b.ts != nullptr)
                        ts = (m.flags & TF_TS_SMEM) ? reinterpret_cast<const uint64_t *>(stage_aux(s))[ctid] : b.ts[m.first + ctid];
                }
                P::map(tup, prm);
                keep = (MODE == MODE_MAP) ? true : P::filter(tup, prm);
            }
            uint32_t slot = INVALID_SLOT;
            alignas(16) R res;
            if constexpr (MODE == MODE_INGEST) {
                if (keep) {
                    P::lift(tup, res, prm);
                    if (a.nshards && a.shard_slots) { // keyby across GPUs, bucketed: destination-major virtual slot
                        // (integer keys only: the shard paths refuse other key types)
                        const uint64_t key = key_word0(key_words<P>(tup, prm)), q = key / a.nshards;
                        if (q < a.shard_keys) slot = static_cast<uint32_t>(key - q * a.nshards) * a.shard_slots + static_cast<uint32_t>(q);
                        else atomicOr(a.shard_err, 2u); // (a key outside the declared key space: the record is dropped, the step fails)
                    } else if (a.nshards) slot = static_cast<uint32_t>(key_word0(key_words<P>(tup, prm)) % a.nshards); // keyby across GPUs: the "slot" is the destination
                    else {
                        if (a.ext_slots != nullptr) { slot = a.ext_slots[m.tile * TILE + ctid]; if (slot >= a.ff.max_keys) slot = INVALID_SLOT; }
                        else slot = slot_of_key(a.ff, key_words<P>(tup, prm));
                        if (slot != INVALID_SLOT && a.count_keys) atomicAdd(&a.ff.seg_cnt[slot], 1u); // (full-sort path only)
                    }
                    if (a.wide_h16 != nullptr) { // digit counts of this wide tile (the CTA owns all of its tiles)
                        if (slot != INVALID_SLOT) { // two 16-bit counters per word (a wide tile holds 4096 positions: no carry)
                            const uint32_t d = (slot >> a.sort_shift) & 1023u;
                            const uint32_t before = atomicAdd(&s_hist[wpar * 512u + (d >> 1)], 1u << ((d & 1u) * 16u));
                            if (a.pack_rank) slot |= ((before >> ((d & 1u) * 16u)) & 0xffffu) << 16; // (slot < 65536: the rank rides in the upper half)
                        }
                    } else if (a.sort_ctl != nullptr && !(a.sparse && slot == INVALID_SLOT)) { // digit counts for the radix passes over the slots (invalid slots sort last / are skipped)
                        for (uint32_t ps = 0; ps < a.sort_passes; ps++)
                            atomicAdd(&s_hist[(ps << a.sort_dbits) + ((slot >> (a.sort_shift + a.sort_dbits * ps)) & ((1u << a.sort_dbits) - 1u))], 1u);
                    }
                }
            }
            if constexpr (MODE == MODE_MAP) {
                consumer_bar(); // every consumer has read its tuple: overwrite the stage with the results
                if (active) {
                    if constexpr (CAN_SWZ) {
                        if (m.flags & TF_SWZ) {
                            uint4 *p = reinterpret_cast<uint4 *>(buf + static_cast<size_t>(ctid) * 64);
                            const uint32_t x = (ctid >> 1) & 3u;
                            const uint4 *o = reinterpret_cast<const uint4 *>(&tup);
#pragma unroll
                            for (uint32_t jj = 0; jj < 4; jj++) p[jj ^ x] = o[jj];
                        } else TileIO<T>::store(buf, ctid, tup);
                    } else TileIO<T>::store(buf, ctid, tup);
                }
                if (ctid == 0) meta[s].count = cnt;
            } else if constexpr (MODE == MODE_FLATMAP) {
                // ---- count pass: the functor with a counting shipper, capped at m ------------------------------------
                const uint32_t mpt = a.max_per_tuple;
                uint32_t cnt_t = 0;
                if (keep) { Shipper<R> sh(nullptr, nullptr, 0, mpt); P::flatmap(tup, sh, prm); cnt_t = sh.pushes(); }
                const uint32_t dropped = cnt_t > mpt ? cnt_t - mpt : 0u;
                cnt_t -= dropped;
                // ---- CTA scan: warp inclusive scan + warp totals (double-buffered by iteration parity) ---------------
                uint32_t incl = cnt_t;
#pragma unroll
                for (uint32_t o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += v; }
                uint32_t *wt = warp_tot + (it & 1u) * (TILE / 32);
                uint32_t *wd = fm_words + (it & 1u) * (TILE / 32);
                const uint32_t wdrop = __reduce_add_sync(FULL, dropped);
                if (lane == 31) { wt[cwarp] = incl; wd[cwarp] = wdrop; }
                consumer_bar(); // warp totals visible; every consumer has read its tuple and timestamp
                uint32_t wbase = 0, total = 0, tdrop = 0;
#pragma unroll
                for (uint32_t w = 0; w < TILE / 32; w++) { const uint32_t c = wt[w]; if (w < cwarp) wbase += c; total += c; tdrop += wd[w]; }
                // ---- the tile's base in its batch's output: consumer warp 0 publishes the aggregate and looks back ----
                uint32_t *tile_base = fm_words + 2 * (TILE / 32) + (it & 1u);
                if (cwarp == 0) {
                    if (lane == 0) {
                        meta[s].count = total;
                        if (m.tile != b.tile_begin) st_relaxed_u64(&a.tile_state[m.tile], pack_state(a.epoch, ST_AGG, total));
                    }
                    uint32_t excl = 0;
                    if (m.tile != b.tile_begin) lookback_exclusive(a, m.tile, b.tile_begin, lane, excl);
                    if (lane == 0) {
                        st_relaxed_u64(&a.tile_state[m.tile], pack_state(a.epoch, ST_PREFIX, excl + total));
                        if (m.tile == b.tile_begin + (b.n + TILE - 1) / TILE - 1 && b.n_out != nullptr) *b.n_out = excl + total;
                        if (tdrop) atomicAdd(a.n_total, tdrop); // (one atomic per tile that dropped pushes)
                        *tile_base = excl;
                    }
                }
                consumer_bar(); // tile base visible
                // ---- emit pass: the functor again, record j of this tuple at batch base + tile excl + thread excl + j ---
                if (cnt_t) {
                    const uint32_t pos = *tile_base + wbase + incl - cnt_t;
                    Shipper<R> sh(b.out + static_cast<size_t>(pos) * RB, b.ts_out != nullptr ? b.ts_out + pos : nullptr, ts, mpt);
                    P::flatmap(tup, sh, prm);
                }
            } else {
                // ---- stable local offsets: ballot + warp totals (double-buffered), ONE named barrier ------------
                const uint32_t bal = __ballot_sync(FULL, keep);
                uint32_t *wt = warp_tot + (it & 1u) * (TILE / 32);
                if (lane == 0) wt[cwarp] = __popc(bal);
                consumer_bar(); // totals visible; every consumer has read its tuple (stage re-usable for staging)
                if constexpr (MODE == MODE_INGEST) {
                    if (a.wide_h16 != nullptr && (m.flags & TF_WIDE_LAST)) { // last tile of the wide tile: file its row, clear the buffer for the
                        uint32_t *hrow = s_hist + wpar * 512u;                 // wide tile after the next (a barrier per tile lies in between)
                        const uint2 c = reinterpret_cast<const uint2 *>(hrow)[ctid];
                        reinterpret_cast<uint2 *>(hrow)[ctid] = make_uint2(0, 0);
                        reinterpret_cast<uint2 *>(a.wide_h16 + static_cast<size_t>(m.wide) * 1024u)[ctid] = c; // (little endian: the packed words are the row)
                        wpar ^= 1u;
                    }
                }
                uint32_t wbase = 0, total = 0;
#pragma unroll
                for (uint32_t w = 0; w < TILE / 32; w++) { const uint32_t c = wt[w]; if (w < cwarp) wbase += c; total += c; }
                const uint32_t local = wbase + __popc(bal & lanemask_lt());
                if (ctid == 0) { // publish the aggregate right away so that other CTAs' look-backs never wait for us
                    meta[s].count = total;
                    const uint32_t chain_begin = (MODE == MODE_FILTER) ? b.tile_begin : 0u;
                    if (m.tile != chain_begin && !(MODE == MODE_INGEST && a.sparse)) st_relaxed_u64(&a.tile_state[m.tile], pack_state(a.epoch, ST_AGG, total));
                }
                if (keep) {
                    if constexpr (MODE == MODE_FILTER) {
                        TileIO<T>::store(buf, local, tup);
                        if (b.ts_out != nullptr) reinterpret_cast<uint64_t *>(stage_aux(s) + TILE * 8)[local] = ts;
                    } else if (MODE == MODE_INGEST && a.inplace) {
                        reinterpret_cast<uint32_t *>(stage_aux(s))[ctid] = slot; // the record stays where it is: position = tuple index
                    } else {
                        TileIO<R>::store(buf, local, res);
                        reinterpret_cast<uint32_t *>(stage_aux(s))[local] = slot;
                    }
                } else if (MODE == MODE_INGEST && a.inplace) reinterpret_cast<uint32_t *>(stage_aux(s))[ctid] = INVALID_SLOT;
            }
            fence_async_smem();
            __syncwarp();
            if (lane == 0) mbar_arrive(&staged[s]);
        }
    } else {
        // ================================= EPILOGUE =================================
        for (uint32_t it = 0;; it++) {
            const uint32_t s = it % SM::stages, par = (it / SM::stages) & 1u;
            unsigned char *buf = stage_buf(s);
            mbar_wait(&staged[s], par);
            const StageMeta m = meta[s];
            if (m.tile == TILE_SENTINEL) break;
            if constexpr (MODE == MODE_FLATMAP) { // the consumers placed the records themselves: only release the stage
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);
                continue;
            }
            DevBatch b;
            if (a.batches == nullptr) b = a.one; else b = a.batches[m.batch];
            const uint32_t t = m.tile, tile_count = m.count;
            uint32_t excl = 0;
            if (MODE == MODE_INGEST && a.sparse) {
                excl = t * TILE; // the tile's own region
                if (lane == 0 && t == 0 && a.ff.n_trig != nullptr) { *a.ff.n_trig = 0; *a.ff.n_heavy = 0; } // per-segment lists filled by the update kernels
            } else if constexpr (MODE != MODE_MAP) {
                const uint32_t chain_begin = (MODE == MODE_FILTER) ? b.tile_begin : 0u;
                if (t != chain_begin) lookback_exclusive(a, t, chain_begin, lane, excl);
                if (lane == 0) {
                    st_relaxed_u64(&a.tile_state[t], pack_state(a.epoch, ST_PREFIX, excl + tile_count));
                    if constexpr (MODE == MODE_FILTER) {
                        const uint32_t last_tile = b.tile_begin + (b.n + TILE - 1) / TILE - 1;
                        if (t == last_tile && b.n_out != nullptr) *b.n_out = excl + tile_count;
                    } else {
                        if (t == 0) { *a.ff.n_trig = 0; *a.ff.n_heavy = 0; } // per-segment lists filled by the update kernels
                        if (t == b.tile_begin) a.batch_off[m.batch] = excl;
                        if (t == a.num_tiles - 1) { a.batch_off[a.nbatches] = excl + tile_count; *a.n_total = excl + tile_count; }
                    }
                }
            }
            // ---- write out ---------------------------------------------------------------------------------------
            unsigned char *dst;
            uint32_t bytes;
            if constexpr (MODE == MODE_MAP) { dst = b.out + static_cast<size_t>(m.first) * TB; bytes = m.cnt * TB; }
            else if constexpr (MODE == MODE_FILTER) { dst = b.out + static_cast<size_t>(excl) * TB; bytes = tile_count * TB; }
            else { dst = a.lifted + static_cast<size_t>(excl) * RB; bytes = a.inplace ? 0u : tile_count * RB; }
            if (MODE == MODE_MAP && (m.flags & TF_SWZ)) {
                if (lane == 0) tma_store_2d(&tmap, 0, static_cast<int32_t>((reinterpret_cast<uint64_t>(dst) - a.tmap_base) >> 6), buf);
            } else if (bulk_ok(dst, bytes)) {
                if (lane == 0 && bytes) {
                    if ((MODE == MODE_INGEST) && a.l2_hints) bulk_s2g_hint(dst, buf, bytes, l2_policy_evict_last());
                    else bulk_s2g(dst, buf, bytes);
                }
            } else {
                uint64_t *d8 = reinterpret_cast<uint64_t *>(dst);
                const uint64_t *s8 = reinterpret_cast<const uint64_t *>(buf);
                for (uint32_t w = lane; w < bytes / 8; w += 32) d8[w] = s8[w];
            }
            if constexpr (MODE == MODE_FILTER) {
                if (b.ts_out != nullptr) {
                    const uint64_t *sts = reinterpret_cast<const uint64_t *>(stage_aux(s) + TILE * 8);
                    for (uint32_t i = lane; i < tile_count; i += 32) b.ts_out[excl + i] = sts[i];
                }
            }
            if constexpr (MODE == MODE_INGEST) {
                const uint32_t *ssl = reinterpret_cast<const uint32_t *>(stage_aux(s));
                if (a.sparse) for (uint32_t i = lane; i < TILE; i += 32) a.slots[excl + i] = i < (a.inplace ? m.cnt : tile_count) ? ssl[i] : INVALID_SLOT;
                else for (uint32_t i = lane; i < tile_count; i += 32) a.slots[excl + i] = ssl[i];
            }
            __syncwarp();
            if (lane == 0) {
                bulk_commit();
                bulk_wait_read<0>();   // the store has finished READING shared memory: the stage can be refilled
                mbar_arrive(&empty[s]);
            }
        }
        if (lane == 0) bulk_wait_all<0>();
    }
}

// ------------------------------------------------------------------------------------------------------
// record helpers (R = result_t): vectorised global load/store and warp shuffles of whole records
// ------------------------------------------------------------------------------------------------------
template <class R>
__device__ __forceinline__ void ld_rec(const unsigned char *p, R &r)
{
    if constexpr (sizeof(R) % 16 == 0) {
        const uint4 *s = reinterpret_cast<const uint4 *>(p);
        uint4 *d = reinterpret_cast<uint4 *>(&r);
#pragma unroll
        for (uint32_t k = 0; k < sizeof(R) / 16; k++) d[k] = s[k];
    } else {
        const uint64_t *s = reinterpret_cast<const uint64_t *>(p);
        uint64_t *d = reinterpret_cast<uint64_t *>(&r);
#pragma unroll
        for (uint32_t k = 0; k < sizeof(R) / 8; k++) d[k] = s[k];
    }
}
template <class R>
__device__ __forceinline__ void st_rec(unsigned char *p, const R &r)
{
    if constexpr (sizeof(R) % 16 == 0) {
        uint4 *d = reinterpret_cast<uint4 *>(p);
        const uint4 *s = reinterpret_cast<const uint4 *>(&r);
#pragma unroll
        for (uint32_t k = 0; k < sizeof(R) / 16; k++) d[k] = s[k];
    } else {
        uint64_t *d = reinterpret_cast<uint64_t *>(p);
        const uint64_t *s = reinterpret_cast<const uint64_t *>(&r);
#pragma unroll
        for (uint32_t k = 0; k < sizeof(R) / 8; k++) d[k] = s[k];
    }
}
template <class R>
__device__ __forceinline__ R shfl_down_rec(const R &r, uint32_t delta)
{
    alignas(16) R o;
    const uint32_t *s = reinterpret_cast<const uint32_t *>(&r);
    uint32_t *d = reinterpret_cast<uint32_t *>(&o);
#pragma unroll
    for (uint32_t k = 0; k < sizeof(R) / 4; k++) d[k] = __shfl_down_sync(FULL, s[k], delta);
    return o;
}
template <class R>
__device__ __forceinline__ R shfl_rec(const R &r, uint32_t src)
{
    alignas(16) R o;
    const uint32_t *s = reinterpret_cast<const uint32_t *>(&r);
    uint32_t *d = reinterpret_cast<uint32_t *>(&o);
#pragma unroll
    for (uint32_t k = 0; k < sizeof(R) / 4; k++) d[k] = __shfl_sync(FULL, s[k], src);
    return o;
}

// exclusive scan of `total` uint32 counters (in may alias out), one CTA of 1024 threads
static __global__ void __launch_bounds__(1024) k_scan_u32(const uint32_t *in, uint32_t *out, uint32_t total, uint32_t *sum_out)
{
    __shared__ uint32_t warp_sums[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t per = (total + 1023) / 1024;
    const uint32_t begin = min(tid * per, total), end = min(begin + per, total);
    uint32_t sum = 0;
    for (uint32_t i = begin; i < end; i++) sum += in[i];
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += v; }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = warp_sums[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, wi, o); if (lane >= o) wi += v; }
        warp_sums[lane] = wi - w; // exclusive
        if (lane == 31 && sum_out != nullptr) *sum_out = wi;
    }
    __syncthreads();
    uint32_t run = warp_sums[warp] + incl - sum;
    for (uint32_t i = begin; i < end; i++) { const uint32_t v = in[i]; out[i] = run; run += v; }
}


// ------------------------------------------------------------------------------------------------------
// Onesweep-style stable LSD radix pass (8-bit digits): ONE kernel per pass.
//   k_radix_ghist     digit histograms of every pass in one read of the keys   ghist[pass][256]
//   k_onesweep_pass   per tile (dynamic ticket order): stable in-tile ranks (warp match_any, warps in index order),
//                     per-digit decoupled look-back over the earlier tiles (thread d owns digit d, epoch-tagged
//                     64-bit state words), keys/values regrouped by digit in shared memory and written coalesced.
// ctl layout (uint32): [pass][256] histograms, then [pass] ticket counters; the host clears it once per sort.
// ------------------------------------------------------------------------------------------------------
constexpr int OS_THREADS = 256;
constexpr int OS_MAX_PASSES = 8;
constexpr int OS_ITEMS = 8; // elements per thread of a pass

template <class K>
__global__ void __launch_bounds__(256) k_radix_ghist(const K *__restrict__ keys, const uint32_t *__restrict__ n_ptr, uint32_t n_host,
                                                     uint32_t passes, uint32_t *__restrict__ ctl, uint32_t base_shift)
{
    __shared__ uint32_t h[OS_MAX_PASSES * 256];
    const uint32_t n = n_ptr ? *n_ptr : n_host;
    for (uint32_t i = threadIdx.x; i < passes * 256; i += blockDim.x) h[i] = 0;
    __syncthreads();
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const K k = keys[i];
        for (uint32_t p = 0; p < passes; p++) atomicAdd(&h[p * 256 + (static_cast<uint32_t>(k >> (base_shift + 8 * p)) & 255u)], 1u);
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < passes * 256; i += blockDim.x) if (h[i]) atomicAdd(&ctl[i], h[i]);
}

template <class K>
__global__ void __launch_bounds__(OS_THREADS) k_onesweep_pass(const K *__restrict__ keys_in, const uint32_t *__restrict__ vals_in,
                                                              K *__restrict__ keys_out, uint32_t *__restrict__ vals_out,
                                                              const uint32_t *__restrict__ n_ptr, uint32_t n_host, uint32_t pass,
                                                              uint32_t passes, uint32_t *__restrict__ ctl,
                                                              uint64_t *__restrict__ tile_state, uint32_t epoch,
                                                              uint32_t *__restrict__ seg_first, uint32_t seg_first_n,
                                                              uint32_t base_shift)
{
    __shared__ uint32_t cntw[OS_THREADS / 32][256]; // per-warp digit counts -> exclusive offsets over the warps
    __shared__ uint32_t dig_off[256];               // exclusive offset of each digit inside the tile
    __shared__ uint32_t bin_base[256];              // global position of the tile's first element of each digit
    __shared__ uint32_t wsum[OS_THREADS / 32];
    __shared__ uint32_t s_tile;
    constexpr int OS_TILE = OS_THREADS * OS_ITEMS;
    __shared__ K skeys[OS_TILE];
    __shared__ uint32_t svals[OS_TILE];

    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t n = n_ptr ? *n_ptr : n_host;
    const uint32_t num_tiles = (n + OS_TILE - 1) / OS_TILE;
    const uint32_t shift = base_shift + 8 * pass;
    if (tid == 0) s_tile = atomicAdd(&ctl[passes * 256 + pass], 1u);
#pragma unroll
    for (int w = 0; w < OS_THREADS / 32; w++) cntw[w][tid] = 0;
    __syncthreads();
    const uint32_t tile = s_tile;
    if (tile >= num_tiles) return;
    const uint32_t start = tile * OS_TILE;

    // ---- stable in-tile ranks: warp w owns [start + w*512, +512), 32 consecutive elements per round ------------
    K k[OS_ITEMS];
    uint32_t rk[OS_ITEMS];
#pragma unroll
    for (int r = 0; r < OS_ITEMS; r++) {
        const uint32_t idx = start + warp * (32 * OS_ITEMS) + r * 32 + lane;
        const bool valid = idx < n;
        k[r] = valid ? keys_in[idx] : K(0);
        const uint32_t d = valid ? (static_cast<uint32_t>(k[r] >> shift) & 255u) : 256u;
        const uint32_t mask = __match_any_sync(FULL, d);
        rk[r] = valid ? (cntw[warp][d] + __popc(mask & lanemask_lt())) : 0u;
        __syncwarp();
        if (valid && lane == static_cast<uint32_t>(__ffs(mask) - 1)) cntw[warp][d] += __popc(mask);
        __syncwarp();
    }
    __syncthreads();

    // ---- digit `tid`: tile total, exclusive offsets over warps, publish, look back -----------------------------------
    uint32_t total = 0;
#pragma unroll
    for (int w = 0; w < OS_THREADS / 32; w++) { const uint32_t c = cntw[w][tid]; cntw[w][tid] = total; total += c; }
    uint64_t *my_state = tile_state + static_cast<size_t>(tile) * 256 + tid;
    st_relaxed_u64(my_state, pack_state(epoch, tile == 0 ? ST_PREFIX : ST_AGG, total));
    // global base of digit tid = exclusive scan of the pass histogram over the digits
    const uint32_t gcount = ctl[pass * 256 + tid];
    uint32_t incl = gcount;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += v; }
    if (lane == 31) wsum[warp] = incl;
    // exclusive offset of the digit inside the tile (same scan over `total`)
    uint32_t tincl = total;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, tincl, o); if (lane >= o) tincl += v; }
    __shared__ uint32_t twsum[OS_THREADS / 32];
    if (lane == 31) twsum[warp] = tincl;
    __syncthreads();
    uint32_t gbase = incl - gcount, tbase = tincl - total;
#pragma unroll
    for (uint32_t w = 0; w < OS_THREADS / 32; w++) if (w < warp) { gbase += wsum[w]; tbase += twsum[w]; }
    uint32_t excl = 0;
    if (tile > 0) { // thread d walks digit d's chain back, 8 independent loads per step
        int64_t t2 = static_cast<int64_t>(tile) - 1;
        bool found = false;
        while (!found) {
            uint64_t w[8];
#pragma unroll
            for (int q = 0; q < 8; q++) w[q] = (t2 - q >= 0) ? ld_relaxed_u64(tile_state + static_cast<size_t>(t2 - q) * 256 + tid) : 0ull;
#pragma unroll
            for (int q = 0; q < 8; q++) {
                if (found || t2 - q < 0) continue;
                if ((w[q] >> 34) != (epoch & 0x3fffffffu) || ((w[q] >> 32) & 3u) == 0) { t2 -= q; goto next_round; } // not published yet: retry from here
                excl += static_cast<uint32_t>(w[q]);
                if (((w[q] >> 32) & 3u) == ST_PREFIX) found = true;
            }
            t2 -= 8;
        next_round:;
        }
        st_relaxed_u64(my_state, pack_state(epoch, ST_PREFIX, excl + total));
    }
    dig_off[tid] = tbase;
    bin_base[tid] = gbase + excl;
    __syncthreads();

    // ---- regroup by digit in shared memory, then coalesced writes ---------------------------------------------------
#pragma unroll
    for (int r = 0; r < OS_ITEMS; r++) {
        const uint32_t idx = start + warp * (32 * OS_ITEMS) + r * 32 + lane;
        if (idx < n) {
            const uint32_t d = static_cast<uint32_t>(k[r] >> shift) & 255u;
            const uint32_t lp = dig_off[d] + cntw[warp][d] + rk[r];
            skeys[lp] = k[r];
            svals[lp] = vals_in ? vals_in[idx] : idx;
        }
    }
    __syncthreads();
    const uint32_t cnt = min(static_cast<uint32_t>(OS_TILE), n - start);
    for (uint32_t i = tid; i < cnt; i += OS_THREADS) {
        const K kk = skeys[i];
        const uint32_t d = static_cast<uint32_t>(kk >> shift) & 255u;
        const uint32_t dst = bin_base[d] + (i - dig_off[d]);
        keys_out[dst] = kk;
        vals_out[dst] = svals[i];
        // last pass of the window operator's sort: first sorted position of every key (entries start at 0xffffffff)
        if (seg_first != nullptr && static_cast<uint64_t>(kk) < seg_first_n) atomicMin(&seg_first[static_cast<uint32_t>(kk)], dst);
    }
}

// ------------------------------------------------------------------------------------------------------
// k_slots_inplace: the streaming pass of a pass-through program whose records already sit at their tile positions
// (TileArgs::inplace): nothing is staged or copied, so a plain grid-stride kernel replaces k_tile_pass -- key -> slot (or the
// caller's slot), INVALID_SLOT padding, the 16-bit rows of the wide partition (TileArgs::wide_h16).
// 32-byte records make 8-KB tiles, too small to amortise the tile pass's per-tile machinery (measured 1.2 TB/s there).
// ------------------------------------------------------------------------------------------------------
template <class P>
__global__ void __launch_bounds__(256) k_slots_inplace(const TileArgs a, const typename P::params_t prm)
{
    using T = typename P::tuple_t;
    __shared__ uint32_t s_h[512];
    const uint32_t tid = threadIdx.x;
    const uint32_t npos = a.num_tiles * TILE;
    if (blockIdx.x == 0 && tid == 0 && a.ff.n_trig != nullptr) { *a.ff.n_trig = 0; *a.ff.n_heavy = 0; } // per-segment lists of the update kernels
    auto slot_at = [&](uint32_t p) -> uint32_t {
        const uint32_t t = p / TILE;
        uint32_t lo = 0, hi = a.nbatches - 1; // last batch with tile_begin <= t
        while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (a.batches[mid].tile_begin <= t) lo = mid; else hi = mid - 1; }
        const DevBatch &b = a.batches[lo];
        const uint32_t local = p - b.tile_begin * TILE;
        uint32_t slot = INVALID_SLOT;
        if (local < b.n) {
            if (a.ext_slots != nullptr) { slot = a.ext_slots[p]; if (slot >= a.ff.max_keys) slot = INVALID_SLOT; }
            else {
                const T *rec = reinterpret_cast<const T *>(b.tuples + static_cast<size_t>(local) * sizeof(T));
                slot = slot_of_key(a.ff, key_words<P>(*rec, prm));
            }
            if (slot != INVALID_SLOT && a.count_keys) atomicAdd(&a.ff.seg_cnt[slot], 1u);
        }
        return slot;
    };
    // a CTA owns whole wide tiles (4096 positions): digit counts in shared memory (two 16-bit counters per word), one row per wide tile,
    // and -- TileArgs::pack_rank -- every slot leaves with the count its digit had when it was counted (k_wide_scatter_ranked)
    const uint32_t nwide = (npos + OSW_TILE_POS - 1) / OSW_TILE_POS;
    for (uint32_t wt = blockIdx.x; wt < nwide; wt += gridDim.x) {
        for (uint32_t i = tid; i < 512; i += blockDim.x) s_h[i] = 0;
        __syncthreads();
        for (uint32_t p = wt * OSW_TILE_POS + tid; p < min(npos, (wt + 1) * OSW_TILE_POS); p += blockDim.x) {
            uint32_t slot = slot_at(p);
            if (slot != INVALID_SLOT) {
                const uint32_t d = (slot >> a.sort_shift) & 1023u;
                const uint32_t before = atomicAdd(&s_h[d >> 1], 1u << ((d & 1u) * 16u));
                if (a.pack_rank) slot |= ((before >> ((d & 1u) * 16u)) & 0xffffu) << 16;
            }
            a.slots[p] = slot;
        }
        __syncthreads();
        for (uint32_t i = tid; i < 512; i += blockDim.x) reinterpret_cast<uint32_t *>(a.wide_h16 + static_cast<size_t>(wt) * 1024u)[i] = s_h[i];
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------------
// Wide partition: ONE stable pass on a 10-bit digit (1024 bins) without a chained scan -- with 1024 bins a tile holds
// only a few elements per bin, so the look-back chains of k_onesweep_pass are long and cheap to avoid:
//   k_wide_tile_hist  per-tile digit counts H[tile][1024] (16-bit) + their sums over chunks of 2^chunk_shift tiles
//                     C[chunk][1024] (+ the global counts ctl[1024] unless the producer of the keys already made them)
//   k_wide_scatter    rank inside the tile (warp match_any, warps in index order), base of (tile, digit) =
//                     exclusive scan of ctl over the digits + C rows of the earlier chunks + H rows of the earlier
//                     tiles of the own chunk; elements go straight to their final position
// The window operator uses it to split a segment's (slot, arrival position) pairs into 1024 buckets of consecutive
// slots (k_ffat_update_buckets finishes the grouping inside each bucket).
// ------------------------------------------------------------------------------------------------------
#ifndef WFB_OSW_MINBLOCKS
#define WFB_OSW_MINBLOCKS 5
#endif
constexpr uint32_t OSW_BITS = 10, OSW_DIGITS = 1u << OSW_BITS;
constexpr uint32_t OSW_THREADS = 256, OSW_ITEMS = 16, OSW_TILE = OSW_THREADS * OSW_ITEMS; // 4096 elements per tile
static_assert(OSW_TILE == OSW_TILE_POS, "the tile pass files its digit counts per wide tile");
// wide tiles per CTA of k_wide_scatter_ranked (and per offset row T of k_wide_tile_bases): a chunk is a whole number of groups
constexpr uint32_t OSR_GROUP = 4, OSR_GROUP_POS = OSR_GROUP * OSW_TILE;
// The bucket list the partition leaves for k_ffat_update_buckets: ONE word per item, pos << BKL_KEY_BITS | local key. local key = slot -
// first slot of the item's bucket (a bucket holds at most 2^BKL_KEY_BITS consecutive slots; the bucket is the update's CTA), pos = the
// item's record index relative to the first position of its position range (moved records: the arrival position of the item whose
// record sits at that list index). The word holds positions below BKL_RANGE_POS, so a window phase over more positions runs in ranges
// of BKL_RANGE_POS positions: partition, update and window queries of one range, then the next (ffat_window_phase,
// ffat_process_prebucketed). A test build may lower WFB_BKL_RANGE_POS to cut small calls into many ranges.
#ifndef WFB_BKL_RANGE_POS
#define WFB_BKL_RANGE_POS (1u << 26)
#endif
constexpr uint32_t BKL_KEY_BITS = 6, BKL_RANGE_POS = WFB_BKL_RANGE_POS;
static_assert(BKL_RANGE_POS <= (1u << (32 - BKL_KEY_BITS)) && BKL_RANGE_POS >= OSR_GROUP_POS && BKL_RANGE_POS % OSR_GROUP_POS == 0,
              "a range is whole groups of wide tiles, and its positions fit the list word");
__device__ __forceinline__ uint32_t bkl_word(uint32_t pos, uint32_t local_key) { return pos << BKL_KEY_BITS | local_key; }

template <class K>
__global__ void __launch_bounds__(OSW_THREADS) k_wide_tile_hist(const K *__restrict__ keys, const uint32_t *__restrict__ n_ptr, uint32_t n_host,
                                                                uint32_t shift, uint32_t chunk_shift, uint16_t *__restrict__ H,
                                                                uint32_t *__restrict__ C, uint32_t *__restrict__ ctl_counts, uint32_t skip_invalid)
{
    static_assert(OSW_THREADS * 4 == OSW_DIGITS, "four digits per thread");
    __shared__ __align__(16) uint32_t h[OSW_DIGITS];
    const uint32_t tid = threadIdx.x, tile = blockIdx.x;
    const uint32_t n = n_ptr ? *n_ptr : n_host;
    const uint32_t start = tile * OSW_TILE;
    if (start >= n) return;
    reinterpret_cast<uint4 *>(h)[tid] = make_uint4(0, 0, 0, 0);
    __syncthreads();
#pragma unroll
    for (uint32_t r = 0; r < OSW_ITEMS; r++) {
        const uint32_t idx = start + r * OSW_THREADS + tid;
        if (idx < n) { const K kk = keys[idx]; if (!(skip_invalid && kk == static_cast<K>(~K(0)))) atomicAdd(&h[static_cast<uint32_t>(kk >> shift) & (OSW_DIGITS - 1u)], 1u); }
    }
    __syncthreads();
    const uint4 c = reinterpret_cast<const uint4 *>(h)[tid];
    reinterpret_cast<ushort4 *>(H + static_cast<size_t>(tile) * OSW_DIGITS)[tid] =
        make_ushort4(static_cast<uint16_t>(c.x), static_cast<uint16_t>(c.y), static_cast<uint16_t>(c.z), static_cast<uint16_t>(c.w));
    uint32_t *crow = C + static_cast<size_t>(tile >> chunk_shift) * OSW_DIGITS + tid * 4;
    if (c.x) atomicAdd(crow + 0, c.x);
    if (c.y) atomicAdd(crow + 1, c.y);
    if (c.z) atomicAdd(crow + 2, c.z);
    if (c.w) atomicAdd(crow + 3, c.w);
    if (ctl_counts != nullptr) {
        if (c.x) atomicAdd(ctl_counts + tid * 4 + 0, c.x);
        if (c.y) atomicAdd(ctl_counts + tid * 4 + 1, c.y);
        if (c.z) atomicAdd(ctl_counts + tid * 4 + 2, c.z);
        if (c.w) atomicAdd(ctl_counts + tid * 4 + 3, c.w);
    }
}

// C[chunk][digit] = sum of the 16-bit per-tile rows of the chunk that the tile pass files (TileArgs::wide_h16)
static __global__ void __launch_bounds__(OSW_THREADS) k_wide_chunk_sums16(const uint16_t *__restrict__ H, uint32_t tiles, uint32_t chunk_shift, uint32_t *__restrict__ C,
                                                                          uint32_t *__restrict__ ctl_counts = nullptr)
{
    // ctl_counts (optional): the global digit counts are accumulated there as well (callers that do not run k_wide_tile_bases)
    const uint32_t chunk = blockIdx.x, tid = threadIdx.x;
    const uint32_t t0 = chunk << chunk_shift, t1 = min(tiles, t0 + (1u << chunk_shift));
    uint4 acc = make_uint4(0, 0, 0, 0);
    const ushort4 *row = reinterpret_cast<const ushort4 *>(H) + tid;
#pragma unroll 16
    for (uint32_t t = t0; t < t1; t++) { const ushort4 v = row[static_cast<size_t>(t) * (OSW_DIGITS / 4)]; acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
    reinterpret_cast<uint4 *>(C + static_cast<size_t>(chunk) * OSW_DIGITS)[tid] = acc;
    if (ctl_counts != nullptr) {
        if (acc.x) atomicAdd(ctl_counts + tid * 4 + 0, acc.x);
        if (acc.y) atomicAdd(ctl_counts + tid * 4 + 1, acc.y);
        if (acc.z) atomicAdd(ctl_counts + tid * 4 + 2, acc.z);
        if (acc.w) atomicAdd(ctl_counts + tid * 4 + 3, acc.w);
    }
}

// The first output position of every (group of 2^gshift wide tiles, digit), in one launch, from the 16-bit rows the tile pass filed.
// CTA c adds the rows of chunk c and files, for every group of the chunk, the sum of the chunk's earlier rows (T[group][digit], 32-bit). The last CTA to
// finish turns the chunk sums C[chunk][digit] into the first output position of every (chunk, digit) -- exclusive scan over the digits
// of the totals + exclusive scan over the chunks, in place -- and sets ctl_counts[digit] = total of the digit. A group's first output
// position of digit d is then C[chunk][d] + T[group][d]: two rows per scatter CTA, whatever the group's place in its chunk.
// `done` (one word, zero between launches: the last CTA clears it) counts the finished chunks.
static __global__ void __launch_bounds__(OSW_THREADS) k_wide_tile_bases(const uint16_t *__restrict__ H, uint32_t tiles, uint32_t chunk_shift, uint32_t chunks,
                                                                        uint32_t *__restrict__ C, uint32_t *__restrict__ T, uint32_t *__restrict__ ctl_counts,
                                                                        uint32_t *__restrict__ done, uint32_t gshift)
{
    static_assert(OSW_THREADS * 4 == OSW_DIGITS, "four digits per thread");
    constexpr uint32_t NW = OSW_THREADS / 32;
    __shared__ uint32_t wsum[NW];
    __shared__ uint32_t s_last;
    const uint32_t chunk = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t t0 = chunk << chunk_shift, t1 = min(tiles, t0 + (1u << chunk_shift));
    uint4 acc = make_uint4(0, 0, 0, 0);
    const ushort4 *row = reinterpret_cast<const ushort4 *>(H) + tid;
    uint4 *trow = reinterpret_cast<uint4 *>(T) + tid;
#pragma unroll 8
    for (uint32_t t = t0; t < t1; t++) {
        const ushort4 v = row[static_cast<size_t>(t) * (OSW_DIGITS / 4)];
        if ((t & ((1u << gshift) - 1u)) == 0) trow[static_cast<size_t>(t >> gshift) * (OSW_DIGITS / 4)] = acc;
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    uint4 *C4 = reinterpret_cast<uint4 *>(C);
    C4[static_cast<size_t>(chunk) * (OSW_DIGITS / 4) + tid] = acc;
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(done, 1u) == chunks - 1u;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    uint4 tot = make_uint4(0, 0, 0, 0);
#pragma unroll 8
    for (uint32_t c = 0; c < chunks; c++) { const uint4 v = __ldcg(C4 + static_cast<size_t>(c) * (OSW_DIGITS / 4) + tid); tot.x += v.x; tot.y += v.y; tot.z += v.z; tot.w += v.w; }
    reinterpret_cast<uint4 *>(ctl_counts)[tid] = tot;
    const uint32_t sum = tot.x + tot.y + tot.z + tot.w;
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    uint32_t base = incl - sum;
#pragma unroll
    for (uint32_t q = 0; q < NW; q++) if (q < warp) base += wsum[q];
    uint4 run = make_uint4(base, base + tot.x, base + tot.x + tot.y, base + tot.x + tot.y + tot.z);
#pragma unroll 8
    for (uint32_t c = 0; c < chunks; c++) {
        uint4 *p = C4 + static_cast<size_t>(c) * (OSW_DIGITS / 4) + tid;
        const uint4 v = __ldcg(p);
        *p = run;
        run.x += v.x; run.y += v.y; run.z += v.z; run.w += v.w;
    }
    if (tid == 0) *done = 0;
}

// The scatter of the wide partition when the tile pass packed a rank with every slot (TileArgs::pack_rank): word = slot | rank << 16,
// rank = any numbering 0 .. count-1 of the survivors of one (wide tile, digit) cell. One CTA per GROUP of OSR_GROUP consecutive wide
// tiles, everything on chip:
//   1. the group's rows; the group's cells laid out back to back in shared memory (exclusive scan of the group's digit counts). The
//      cell of (group, digit) is the group's (wide tile, digit) cells -- its "parts" -- in tile order, which is arrival order, and it is
//      where they sit in the output as well,
//   2. every item files its position within the group (and its slot, at the same index) at its part's start + rank -- no ranking
//      rounds, no per-warp counters,
//   3. a sweep over the laid-out cells, consecutive threads on consecutive entries of a cell: ARRIVAL order inside each part (the count
//      windows need every key's items in stream order, and two items of one key may share a part; every entry of an earlier part is
//      earlier, every entry of a later part later) -- an entry's place in its part is the number of the part's entries with a smaller
//      position, two 16-bit compares per 4-byte load as in k_wide_scatter_ranked_tile -- and one write of the item's list word to the
//      final place: first output position of the group's cell (C[chunk] + T[group] of k_wide_tile_bases) + the earlier parts + that number.
// Why groups: a (wide tile, digit) cell holds about 2 items at the bench step (4096 positions, half of them survivors, 1024 digits), so
// with one wide tile per CTA a warp's store touched about 16 separate 32-byte sectors; a group cell of 4 tiles is about 8 items, whole
// sectors (tools/micro/bucket_store.cu replays both patterns). Used when there are enough groups to give every SM one (osr_group in
// wfb_lib.cu) and no records travel; otherwise k_wide_scatter_ranked_tile below (one wide tile per CTA) runs.
// Output: list_out[i] = bkl_word(position, slot - first slot of its bucket), stable by (digit, position). `packed` starts at the
// position range's first position (the positions in the words are relative to it), n < BKL_RANGE_POS. The tile pass wrote no word for
// an item without a slot (INVALID_SLOT is never counted in a row), and every slot is below the key capacity, 1024 << shift: every item
// lies inside its bucket's keys.
// OSR_SMEM = 74 KB of dynamic shared memory: 3 resident CTAs per SM. Positions within a group are < 2^14, slots < 2^16.
constexpr uint32_t OSR_SMEM = OSR_GROUP_POS * 2u * 2u + OSW_DIGITS * 8u + OSW_DIGITS * 2u;
static_assert(OSR_GROUP == 4 && OSR_GROUP_POS <= 0x8000u, "one ushort4 of part sizes per digit; 16-bit packed position compare");
static __global__ void __launch_bounds__(OSW_THREADS, 3) k_wide_scatter_ranked(const uint32_t *__restrict__ packed, uint32_t *__restrict__ list_out,
                                                                            uint32_t n, uint32_t shift, uint32_t chunk_shift,
                                                                            uint32_t tiles, const uint16_t *__restrict__ H, const uint32_t *__restrict__ Cx,
                                                                            const uint32_t *__restrict__ T)
{
    constexpr uint32_t NW = OSW_THREADS / 32;
    static_assert(OSW_THREADS * 4 == OSW_DIGITS, "four digits per thread");
    extern __shared__ __align__(16) unsigned char osr_smem_buf[];
    uint16_t *lpos = reinterpret_cast<uint16_t *>(osr_smem_buf);        // [OSR_GROUP_POS] position within the group, cells back to back
    uint16_t *lslot = lpos + OSR_GROUP_POS;                               // [OSR_GROUP_POS] the slot of the same entry
    ushort4 *part = reinterpret_cast<ushort4 *>(lslot + OSR_GROUP_POS);  // [OSW_DIGITS] sizes of the digit's parts, tile 0 .. 3
    uint16_t *cell = reinterpret_cast<uint16_t *>(part + OSW_DIGITS);     // [OSW_DIGITS] start of the digit's cell in lpos / lslot
    __shared__ uint32_t wsum[NW];
    __shared__ uint32_t s_total;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, group = blockIdx.x, tile0 = group * OSR_GROUP;
    const uint32_t start = tile0 * OSW_TILE;
    if (start >= n) return;
    {
        ushort4 h[OSR_GROUP]; // the group's rows, digits 4 tid .. 4 tid + 3 (a group past the last tile has empty rows)
#pragma unroll
        for (uint32_t k = 0; k < OSR_GROUP; k++)
            h[k] = tile0 + k < tiles ? reinterpret_cast<const ushort4 *>(H)[static_cast<size_t>(tile0 + k) * (OSW_DIGITS / 4) + tid] : make_ushort4(0, 0, 0, 0);
        part[4 * tid + 0] = make_ushort4(h[0].x, h[1].x, h[2].x, h[3].x);
        part[4 * tid + 1] = make_ushort4(h[0].y, h[1].y, h[2].y, h[3].y);
        part[4 * tid + 2] = make_ushort4(h[0].z, h[1].z, h[2].z, h[3].z);
        part[4 * tid + 3] = make_ushort4(h[0].w, h[1].w, h[2].w, h[3].w);
        uint32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
#pragma unroll
        for (uint32_t k = 0; k < OSR_GROUP; k++) { c0 += h[k].x; c1 += h[k].y; c2 += h[k].z; c3 += h[k].w; }
        const uint32_t sum = c0 + c1 + c2 + c3;
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        uint32_t base = incl - sum;
#pragma unroll
        for (uint32_t q = 0; q < NW; q++) if (q < warp) base += wsum[q];
        if (tid == OSW_THREADS - 1) s_total = base + sum;
        reinterpret_cast<ushort4 *>(cell)[tid] = make_ushort4(static_cast<uint16_t>(base), static_cast<uint16_t>(base + c0), static_cast<uint16_t>(base + c0 + c1),
                                                               static_cast<uint16_t>(base + c0 + c1 + c2));
    }
    __syncthreads();
    // parts of tile k of digit d start at cell[d] + the sizes of the digit's parts of tiles 0 .. k-1
    auto part_start = [&](uint32_t d, uint32_t k, uint32_t *size) {
        const ushort4 p = part[d];
        *size = k == 0 ? p.x : k == 1 ? p.y : k == 2 ? p.z : p.w;
        return (k > 0 ? p.x : 0u) + (k > 1 ? p.y : 0u) + (k > 2 ? p.z : 0u);
    };
#pragma unroll 1
    for (uint32_t k = 0; k < OSR_GROUP; k++) {
        uint32_t w[OSW_ITEMS];
#pragma unroll
        for (uint32_t r = 0; r < OSW_ITEMS; r++) {
            const uint32_t idx = start + k * OSW_TILE + r * OSW_THREADS + tid;
            w[r] = idx < n ? packed[idx] : INVALID_SLOT;
        }
#pragma unroll
        for (uint32_t r = 0; r < OSW_ITEMS; r++)
            if (w[r] != INVALID_SLOT) {
                const uint32_t slot = w[r] & 0xffffu, d = (slot >> shift) & (OSW_DIGITS - 1u);
                uint32_t size;
                const uint32_t i = cell[d] + part_start(d, k, &size) + (w[r] >> 16);
                lpos[i] = static_cast<uint16_t>(k * OSW_TILE + r * OSW_THREADS + tid);
                lslot[i] = static_cast<uint16_t>(slot);
            }
    }
    __syncthreads();
    const uint32_t total = s_total;
    const uint32_t *cbase = Cx + static_cast<size_t>(tile0 >> chunk_shift) * OSW_DIGITS, *tbase = T + static_cast<size_t>(group) * OSW_DIGITS;
#pragma unroll 2
    for (uint32_t e = tid; e < total; e += OSW_THREADS) {
        const uint32_t mine = lpos[e], slot = lslot[e], d = (slot >> shift) & (OSW_DIGITS - 1u);
        uint32_t size;
        const uint32_t before = part_start(d, mine / OSW_TILE, &size);
        uint32_t j = cell[d] + before;
        const uint32_t end = j + size;
        // entries of the part below `mine`: an odd head and tail one by one, the rest two per load -- per 16-bit half, bit 15 of
        // (0x8000 + mine - 1 - entry) says entry < mine (positions are < 2^14, so the halves never borrow from each other)
        uint32_t less = 0;
        if (j & 1u) { less += lpos[j] < mine ? 1u : 0u; j++; }
        const uint32_t mm = (mine | (mine << 16)) + 0x7fff7fffu;
        for (; j + 1 < end; j += 2) less += __popc((mm - *reinterpret_cast<const uint32_t *>(lpos + j)) & 0x80008000u);
        if (j < end) less += lpos[j] < mine ? 1u : 0u;
        const uint32_t dst = __ldg(cbase + d) + __ldg(tbase + d) + before + less;
        list_out[dst] = bkl_word(start + mine, slot - (d << shift));
    }
}

// The same scatter with one CTA per wide tile (k_wide_tile_bases files one offset row per tile, gshift = 0): calls with fewer wide
// tiles than 4 per SM and the payload variants (their L2 prefetch of a group's records would overrun the L2). Everything on chip:
//   1. the tile's words to shared memory; first output position of every digit for this tile (C[chunk] + T[tile] of k_wide_tile_bases)
//      and the tile's own cells laid out back to back in shared memory (exclusive scan of the tile's digit counts),
//   2. every item files its position within the tile at cell start + rank -- no ranking rounds, no per-warp counters,
//   3. a sweep over the laid-out cells, consecutive threads on consecutive entries of a cell: ARRIVAL order inside the cell (the count
//      windows need every key's items in stream order, and two items of one key may share a cell) -- an entry's place is the number of
//      the cell's entries with a smaller position -- and one write to the final place. The stores of a warp land in the few cells it
//      sweeps, and no per-thread array outlives a loop (nothing is indexed at run time: no local memory).
// Output, stable by (digit, position): list != 0, keys_out[i] = the item's bucket-list word (bkl_word, as k_wide_scatter_ranked); list
// = 0 (RBYTES != 0 only), keys_out[i] = slot.
// RBYTES != 0: the records travel as well (payload_in at the arrival positions -> payload_out at the final places): the source side of
// the bucketed multi-GPU exchange (list = 0: the destination splits its coarse buckets by slot), and WFB_BUCKET_MOVE=1 (list = 1: the
// record index is the list index, and the word's position is the arrival position the update needs for a group's triggering item).
// 34 KB of shared memory and at most 40 registers: 6 resident CTAs per SM, so the 2048 wide tiles of the bench step take 2.6 waves
// on 132 SMs.
#ifndef WFB_OSR_MINBLOCKS
#define WFB_OSR_MINBLOCKS 6
#endif
template <int RBYTES>
static __global__ void __launch_bounds__(OSW_THREADS, WFB_OSR_MINBLOCKS) k_wide_scatter_ranked_tile(const uint32_t *__restrict__ packed, uint32_t *__restrict__ keys_out,
                                                                            uint32_t list, uint32_t n, uint32_t shift, uint32_t chunk_shift,
                                                                            const uint16_t *__restrict__ H, const uint32_t *__restrict__ Cx, const uint32_t *__restrict__ T,
                                                                            const unsigned char *__restrict__ payload_in, unsigned char *__restrict__ payload_out)
{
    constexpr uint32_t NW = OSW_THREADS / 32;
    constexpr uint32_t LPOS = OSW_TILE + OSW_DIGITS;  // every cell padded to an even number of entries (4-byte loads in the repair loop)
    constexpr uint32_t LPAD = 0x0fffu;                // padding entry: never below a position of the tile (positions are < 4096)
    static_assert(OSW_TILE <= 4096 && LPOS % (2 * OSW_THREADS) == 0, "16-bit packed position compare");
    __shared__ __align__(16) uint32_t sw[OSW_TILE];   // the tile's words, arrival order
    __shared__ __align__(16) uint32_t bin_base[OSW_DIGITS];
    __shared__ __align__(8) uint16_t cnt_row[OSW_DIGITS], cell_start[OSW_DIGITS];
    __shared__ __align__(4) uint16_t lpos[LPOS];
    __shared__ uint32_t wsum[NW];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, tile = blockIdx.x;
    const uint32_t start = tile * OSW_TILE;
    if (start >= n) return;
#pragma unroll
    for (uint32_t r = 0; r < OSW_ITEMS; r++) {
        const uint32_t i = r * OSW_THREADS + tid, idx = start + i;
        const uint32_t w = idx < n ? packed[idx] : INVALID_SLOT;
        sw[i] = w;
        if constexpr (RBYTES != 0) // the records this CTA will move: on their way to L2 while the offsets are worked out below
            if (w != INVALID_SLOT) asm volatile("prefetch.global.L2 [%0];" ::"l"(payload_in + static_cast<size_t>(idx) * RBYTES));
    }
    {
        const uint4 cb = reinterpret_cast<const uint4 *>(Cx)[static_cast<size_t>(tile >> chunk_shift) * (OSW_DIGITS / 4) + tid];
        const uint4 tb = reinterpret_cast<const uint4 *>(T)[static_cast<size_t>(tile) * (OSW_DIGITS / 4) + tid];
        reinterpret_cast<uint4 *>(bin_base)[tid] = make_uint4(cb.x + tb.x, cb.y + tb.y, cb.z + tb.z, cb.w + tb.w);
        const ushort4 c = reinterpret_cast<const ushort4 *>(H)[static_cast<size_t>(tile) * (OSW_DIGITS / 4) + tid];
        reinterpret_cast<ushort4 *>(cnt_row)[tid] = c;
        // the tile's cells back to back: exclusive scan of its 1024 digit counts (thread tid owns digits 4 tid .. 4 tid + 3)
        const uint32_t p0 = (c.x + 1u) & ~1u, p1 = (c.y + 1u) & ~1u, p2 = (c.z + 1u) & ~1u, p3 = (c.w + 1u) & ~1u; // padded cell sizes
        const uint32_t sum = p0 + p1 + p2 + p3;
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
        if (lane == 31) wsum[warp] = incl;
#pragma unroll
        for (uint32_t i = 0; i < LPOS / (2 * OSW_THREADS); i++) reinterpret_cast<uint32_t *>(lpos)[i * OSW_THREADS + tid] = LPAD | (LPAD << 16);
        __syncthreads();
        uint32_t base = incl - sum;
#pragma unroll
        for (uint32_t q = 0; q < NW; q++) if (q < warp) base += wsum[q];
        reinterpret_cast<ushort4 *>(cell_start)[tid] = make_ushort4(static_cast<uint16_t>(base), static_cast<uint16_t>(base + p0), static_cast<uint16_t>(base + p0 + p1),
                                                                     static_cast<uint16_t>(base + p0 + p1 + p2));
    }
    __syncthreads();
#pragma unroll
    for (uint32_t r = 0; r < OSW_ITEMS; r++) {
        const uint32_t i = r * OSW_THREADS + tid, w = sw[i];
        if (w != INVALID_SLOT) lpos[cell_start[((w & 0xffffu) >> shift) & (OSW_DIGITS - 1u)] + (w >> 16)] = static_cast<uint16_t>(i);
    }
    __syncthreads();
#pragma unroll 2
    for (uint32_t e = tid; e < LPOS; e += OSW_THREADS) {
        const uint32_t mine = lpos[e], w = sw[mine];
        if (w == INVALID_SLOT) continue;
        const uint32_t slot = w & 0xffffu, d = (slot >> shift) & (OSW_DIGITS - 1u);
        const uint32_t cs = cell_start[d], cnt = cnt_row[d];
        if (e - cs >= cnt) continue; // padding (it reads as position 4095, which lives in another cell or not at all)
        // entries of the cell below `mine`, two per load: per 16-bit half, bit 15 of (0x8000 + mine - 1 - entry) says entry < mine
        // (all values are < 4096, so the halves never borrow from each other; padding entries are never below)
        const uint32_t mm = (mine | (mine << 16)) + 0x7fff7fffu;
        const uint32_t *cell = reinterpret_cast<const uint32_t *>(lpos + cs);
        uint32_t less = 0;
        for (uint32_t j = 0; j < cnt; j += 2) less += __popc((mm - cell[j >> 1]) & 0x80008000u);
        const uint32_t dst = bin_base[d] + less;
        keys_out[dst] = (RBYTES == 0 || list) ? bkl_word(start + mine, slot - (d << shift)) : slot;
        if constexpr (RBYTES != 0) {
            static_assert(RBYTES % 8 == 0, "record size");
            using W = typename std::conditional<RBYTES % 16 == 0, uint4, uint2>::type;
            const W *src = reinterpret_cast<const W *>(payload_in + static_cast<size_t>(start + mine) * RBYTES);
            W *dstp = reinterpret_cast<W *>(payload_out + static_cast<size_t>(dst) * RBYTES);
            W v[RBYTES / sizeof(W)];
#pragma unroll
            for (uint32_t q = 0; q < RBYTES / sizeof(W); q++) v[q] = src[q];
#pragma unroll
            for (uint32_t q = 0; q < RBYTES / sizeof(W); q++) dstp[q] = v[q];
        }
    }
}

// bucketed exchange, source side: records per destination = sums of the bins [d * bps, (d + 1) * bps) of the partition
// (send_meta != nullptr: also the (count, watermark) pair every destination is sent ahead of the records)
static __global__ void k_shard_bin_counts(const uint32_t *__restrict__ bin_counts, uint32_t nshards, uint32_t bps, uint32_t *__restrict__ counts_out,
                                          uint64_t *__restrict__ send_meta, uint64_t watermark)
{
    const uint32_t d = threadIdx.x >> 5, lane = threadIdx.x & 31; // one warp per destination
    uint32_t c = 0;
    if (d < nshards) for (uint32_t b = lane; b < bps; b += 32) c += bin_counts[d * bps + b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL, c, o);
    if (lane == 0 && d < MAX_SHARDS) counts_out[d] = d < nshards ? c : 0u; // ([MAX_SHARDS]: error flags, set by the tile pass)
    if (lane == 0 && d < nshards && send_meta != nullptr) { send_meta[2 * d] = c; send_meta[2 * d + 1] = watermark; }
}

// bucketed exchange, destination side: source s delivered, for every COARSE bucket b of this GPU's slot space (bps of them: the
// source's 1024 bins are shared by all destinations), a run of cnt[s][b] records in arrival order -- the runs of one source back to
// back from recv position off[s]. The update kernel wants all 1024 CTAs busy, so every coarse bucket is split into nsub = 1024 / bps
// sub-buckets by slot: the items of sub-bucket (b, j) are, source after source (= global stream order), the items of run (s, b) whose
// slot falls into j, in arrival order. Three small kernels write them as the bucket list + sizes k_ffat_update_buckets consumes:
// count per (b, j, s) | exclusive scan in that order | stable split of every run. A record's index is its receive position, and the
// kernels see only the items of one range of receive positions [lo, hi) (hi - lo <= BKL_RANGE_POS; the list words hold positions
// relative to lo). Sources' regions lie in source order and a key's run inside a region is in arrival order, so every key's items
// are in increasing receive position: consecutive ranges are consecutive parts of every key's stream.
struct MgRuns { uint32_t off[MAX_SHARDS + 1]; };
// the items [*i0, *i1) of a run of m items from receive position p0 that lie in [lo, hi)
__device__ __forceinline__ void mg_clip(uint32_t p0, uint32_t m, uint32_t lo, uint32_t hi, uint32_t *i0, uint32_t *i1)
{
    *i0 = min(m, max(p0, lo) - p0);
    *i1 = min(m, max(p0, hi) - p0);
}
constexpr uint32_t MG_THREADS = 256;
__device__ __forceinline__ uint32_t mg_run_start(const uint32_t *__restrict__ cnt, uint32_t s, uint32_t bps, uint32_t b, uint32_t *sh)
{   // records of source s in the coarse buckets before b (block-wide sum; sh: 8 words of shared memory)
    uint32_t c = 0;
    for (uint32_t q = threadIdx.x; q < b; q += MG_THREADS) c += cnt[s * bps + q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL, c, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = c;
    __syncthreads();
    uint32_t t = 0;
#pragma unroll
    for (uint32_t w = 0; w < MG_THREADS / 32; w++) t += sh[w];
    __syncthreads();
    return t;
}
static __global__ void __launch_bounds__(MG_THREADS) k_mg_count(const uint32_t *__restrict__ cnt, uint32_t nsrc, uint32_t bps, const MgRuns runs,
                                                                const uint32_t *__restrict__ recv_slots, uint32_t slot_mask, uint32_t shift2, uint32_t nsub,
                                                                uint32_t *__restrict__ cnt3, uint32_t *__restrict__ run_starts,
                                                                uint32_t *__restrict__ n_trig, uint32_t *__restrict__ n_heavy, uint32_t lo, uint32_t hi)
{
    __shared__ uint32_t sh[8], c[MAX_SHARDS];
    const uint32_t b = blockIdx.x, s = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
    if (b == 0 && s == 0 && tid == 0) { *n_trig = 0; *n_heavy = 0; } // per-segment lists filled by the update kernel
    if (tid < MAX_SHARDS) c[tid] = 0;
    const uint32_t rs = mg_run_start(cnt, s, bps, b, sh), m = cnt[s * bps + b];
    if (tid == 0) run_starts[s * bps + b] = rs;
    const uint32_t *sl = recv_slots + runs.off[s] + rs;
    uint32_t ib, ie;
    mg_clip(runs.off[s] + rs, m, lo, hi, &ib, &ie);
    for (uint32_t i0 = ib; i0 < ie; i0 += MG_THREADS) {
        const uint32_t i = i0 + tid;
        const uint32_t j = i < ie ? ((sl[i] & slot_mask) >> shift2) & (nsub - 1u) : nsub;
        for (uint32_t jj = 0; jj < nsub; jj++) { const uint32_t bal = __ballot_sync(FULL, j == jj); if (lane == 0 && bal) atomicAdd(&c[jj], __popc(bal)); }
    }
    __syncthreads();
    if (tid < nsub) cnt3[(b * nsub + tid) * nsrc + s] = c[tid];
}
// exclusive scan of cnt3 in (bucket, sub-bucket, source) order + the sub-bucket sizes (one CTA of 1024 threads; n <= 1024 * MAX_SHARDS)
static __global__ void __launch_bounds__(1024) k_mg_scan(const uint32_t *__restrict__ cnt3, uint32_t n, uint32_t nsrc, uint32_t *__restrict__ off3,
                                                         uint32_t *__restrict__ digit_counts)
{
    __shared__ uint32_t wsum[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t per = (n + 1023u) / 1024u, lo = tid * per;
    uint32_t v[MAX_SHARDS], sum = 0;
#pragma unroll
    for (uint32_t q = 0; q < MAX_SHARDS; q++) { v[q] = (q < per && lo + q < n) ? cnt3[lo + q] : 0u; sum += v[q]; }
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += x; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = wsum[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(FULL, wi, o); if (lane >= static_cast<uint32_t>(o)) wi += x; }
        wsum[lane] = wi - w;
    }
    __syncthreads();
    uint32_t run = wsum[warp] + incl - sum;
#pragma unroll
    for (uint32_t q = 0; q < MAX_SHARDS; q++) if (q < per && lo + q < n) { off3[lo + q] = run; run += v[q]; }
    for (uint32_t d = tid; d * nsrc < n; d += 1024) { uint32_t t = 0; for (uint32_t q = 0; q < nsrc; q++) t += cnt3[d * nsrc + q]; digit_counts[d] = t; }
}
static __global__ void __launch_bounds__(MG_THREADS) k_mg_split(const uint32_t *__restrict__ cnt, uint32_t nsrc, uint32_t bps, const MgRuns runs,
                                                                const uint32_t *__restrict__ recv_slots, uint32_t slot_mask, uint32_t shift2, uint32_t nsub,
                                                                const uint32_t *__restrict__ off3, const uint32_t *__restrict__ run_starts,
                                                                uint32_t *__restrict__ out_list, uint32_t lo, uint32_t hi)
{
    __shared__ uint32_t wc[MG_THREADS / 32][MAX_SHARDS], fill[MAX_SHARDS];
    const uint32_t b = blockIdx.x, s = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t m = cnt[s * bps + b], src0 = runs.off[s] + run_starts[s * bps + b];
    uint32_t ib, ie;
    mg_clip(src0, m, lo, hi, &ib, &ie);
    if (tid < nsub) fill[tid] = off3[(b * nsub + tid) * nsrc + s];
    __syncthreads();
    for (uint32_t i0 = ib; i0 < ie; i0 += MG_THREADS) {
        const uint32_t i = i0 + tid;
        uint32_t slot = 0, j = nsub, before = 0;
        if (i < ie) { slot = recv_slots[src0 + i] & slot_mask; j = (slot >> shift2) & (nsub - 1u); }
        for (uint32_t jj = 0; jj < nsub; jj++) {
            const uint32_t bal = __ballot_sync(FULL, j == jj);
            if (lane == 0) wc[warp][jj] = __popc(bal);
            if (j == jj) before = __popc(bal & lanemask_lt());
        }
        __syncthreads();
        if (i < ie) { // (slot >> shift2 is the update's bucket: the local key is the slot's low shift2 bits)
            uint32_t dst = fill[j] + before;
            for (uint32_t w = 0; w < warp; w++) dst += wc[w][j];
            out_list[dst] = bkl_word(src0 + i - lo, slot & ((1u << shift2) - 1u));
        }
        __syncthreads();
        if (tid < nsub) { uint32_t t = 0; for (uint32_t w = 0; w < MG_THREADS / 32; w++) t += wc[w][tid]; fill[tid] += t; }
        __syncthreads();
    }
}

// RBYTES: bytes of the payload record that travels with each element (payload_out[dst] = payload_in[index]); 0 = none,
// -1 = run-time size `payload_bytes` (multiple of 8)
template <class K, int RBYTES>
__global__ void __launch_bounds__(OSW_THREADS, WFB_OSW_MINBLOCKS) k_wide_scatter(const K *__restrict__ keys_in, K *__restrict__ keys_out, uint32_t *__restrict__ vals_out,
                                                              const uint32_t *__restrict__ n_ptr, uint32_t n_host, uint32_t shift,
                                                              uint32_t chunk_shift, const uint16_t *__restrict__ H, const uint32_t *__restrict__ C,
                                                              const uint32_t *__restrict__ ctl_counts,
                                                              const unsigned char *__restrict__ payload_in, unsigned char *__restrict__ payload_out,
                                                              uint32_t payload_bytes, uint32_t skip_invalid, uint32_t region_stride)
{
    // region_stride != 0: bin d starts at d * region_stride (fixed-capacity regions; elements beyond the capacity are dropped)
    constexpr uint32_t NW = OSW_THREADS / 32;
    __shared__ __align__(16) uint16_t cntw[NW][OSW_DIGITS]; // per-warp digit counts -> exclusive offsets over the warps
    __shared__ uint32_t bin_base[OSW_DIGITS];               // global position of the tile's first element of each digit
    __shared__ uint32_t wsum[NW];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, tile = blockIdx.x;
    const uint32_t n = n_ptr ? *n_ptr : n_host;
    const uint32_t start = tile * OSW_TILE;
    if (start >= n) return;
    {
        uint4 *z = reinterpret_cast<uint4 *>(&cntw[0][0]);
        for (uint32_t i = tid; i < NW * OSW_DIGITS / 8; i += OSW_THREADS) z[i] = make_uint4(0, 0, 0, 0);
    }
    // base of (tile, digit) for digits 4*tid .. 4*tid+3: rows of earlier chunks + rows of earlier tiles of this chunk
    uint32_t acc[4] = {0, 0, 0, 0};
    {
        const uint32_t chunk = tile >> chunk_shift;
        const uint4 *crow = reinterpret_cast<const uint4 *>(C) + tid;
#pragma unroll 8
        for (uint32_t c = 0; c < chunk; c++) { const uint4 v = crow[static_cast<size_t>(c) * (OSW_DIGITS / 4)]; acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w; }
        const ushort4 *hrow = reinterpret_cast<const ushort4 *>(H) + tid;
#pragma unroll 16
        for (uint32_t t = chunk << chunk_shift; t < tile; t++) { const ushort4 v = hrow[static_cast<size_t>(t) * (OSW_DIGITS / 4)]; acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w; }
    }
    const uint4 g4 = reinterpret_cast<const uint4 *>(ctl_counts)[tid];
    const uint32_t gsum = g4.x + g4.y + g4.z + g4.w;
    uint32_t incl = gsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();

    // ---- stable in-tile ranks: warp w owns [start + w*32*ITEMS, +32*ITEMS), 32 consecutive elements per round --------
    K k[OSW_ITEMS];
    uint32_t rk[OSW_ITEMS];
#pragma unroll
    for (uint32_t r = 0; r < OSW_ITEMS; r++) {
        const uint32_t idx = start + warp * (32 * OSW_ITEMS) + r * 32 + lane;
        k[r] = idx < n ? keys_in[idx] : K(0);
    }
#pragma unroll
    for (uint32_t r = 0; r < OSW_ITEMS; r++) {
        const uint32_t idx = start + warp * (32 * OSW_ITEMS) + r * 32 + lane;
        const bool valid = idx < n && !(skip_invalid && k[r] == static_cast<K>(~K(0)));
        rk[r] = 0xffffffffu; // 0xffffffff: not an element
        if (!__any_sync(FULL, valid)) continue; // (the survivors of the streaming pass sit at the front of every 256-position tile: half of the rounds are padding)
        const uint32_t d = valid ? (static_cast<uint32_t>(k[r] >> shift) & (OSW_DIGITS - 1u)) : OSW_DIGITS + lane;
        const uint32_t mask = __match_any_sync(FULL, d);
        const uint32_t leader = static_cast<uint32_t>(__ffs(mask) - 1);
        uint32_t before = 0;
        if (valid && lane == leader) { before = cntw[warp][d]; cntw[warp][d] = static_cast<uint16_t>(before + __popc(mask)); } // one lane per digit and round
        before = __shfl_sync(FULL, before, leader);
        if (valid) rk[r] = before + __popc(mask & lanemask_lt());
        __syncwarp(); // the next round's leaders read what this round's leaders wrote
    }
    __syncthreads();
    {
        uint32_t gb = incl - gsum;
#pragma unroll
        for (uint32_t w = 0; w < NW; w++) if (w < warp) gb += wsum[w];
        uint32_t run[4] = {0, 0, 0, 0};
#pragma unroll
        for (uint32_t w = 0; w < NW; w++) { // exclusive offsets over the warps
            ushort4 *row = reinterpret_cast<ushort4 *>(&cntw[w][0]);
            const ushort4 c = row[tid];
            row[tid] = make_ushort4(static_cast<uint16_t>(run[0]), static_cast<uint16_t>(run[1]), static_cast<uint16_t>(run[2]), static_cast<uint16_t>(run[3]));
            run[0] += c.x; run[1] += c.y; run[2] += c.z; run[3] += c.w;
        }
        const uint32_t gc[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
        for (int q = 0; q < 4; q++) { bin_base[tid * 4 + q] = (region_stride ? (tid * 4 + q) * region_stride : gb) + acc[q]; gb += gc[q]; }
    }
    __syncthreads();
#pragma unroll
    for (uint32_t r = 0; r < OSW_ITEMS; r++) {
        const uint32_t idx = start + warp * (32 * OSW_ITEMS) + r * 32 + lane;
        if (rk[r] != 0xffffffffu) {
            const uint32_t d = static_cast<uint32_t>(k[r] >> shift) & (OSW_DIGITS - 1u);
            const uint32_t dst = bin_base[d] + cntw[warp][d] + rk[r];
            if (region_stride && dst - d * region_stride >= region_stride) { rk[r] = 0xffffffffu; continue; } // region overflow (the caller sees the count)
            if (keys_out != nullptr) keys_out[dst] = k[r];
            if (vals_out != nullptr) vals_out[dst] = idx;
            rk[r] = dst;
        }
    }
    if constexpr (RBYTES > 0) { // records: read in index order (coalesced), written next to the other records of their bin
        using V = typename std::conditional<RBYTES % 16 == 0, uint4, uint2>::type;
        constexpr uint32_t NV = RBYTES / sizeof(V);
#pragma unroll
        for (uint32_t r = 0; r < OSW_ITEMS; r++) {
            const uint32_t idx = start + warp * (32 * OSW_ITEMS) + r * 32 + lane;
            if (rk[r] != 0xffffffffu) {
                const V *src = reinterpret_cast<const V *>(payload_in + static_cast<size_t>(idx) * RBYTES);
                V *dstp = reinterpret_cast<V *>(payload_out + static_cast<size_t>(rk[r]) * RBYTES);
                V tmp[NV];
#pragma unroll
                for (uint32_t q = 0; q < NV; q++) tmp[q] = src[q];
#pragma unroll
                for (uint32_t q = 0; q < NV; q++) dstp[q] = tmp[q];
            }
        }
    } else if constexpr (RBYTES < 0) {
#pragma unroll 1
        for (uint32_t r = 0; r < OSW_ITEMS; r++) {
            const uint32_t idx = start + warp * (32 * OSW_ITEMS) + r * 32 + lane;
            if (rk[r] != 0xffffffffu) {
                const uint64_t *src = reinterpret_cast<const uint64_t *>(payload_in + static_cast<size_t>(idx) * payload_bytes);
                uint64_t *dstp = reinterpret_cast<uint64_t *>(payload_out + static_cast<size_t>(rk[r]) * payload_bytes);
                for (uint32_t q = 0; q < payload_bytes / 8; q++) dstp[q] = src[q];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// k_shard_scatter: the partition pass of wfb_shard_lift when there are only a few bins (destination GPUs): stable
// partition of the lifted records by dest[i] (INVALID_SLOT = dropped) into fixed-capacity regions. Same tiles and the
// same per-tile counts (H rows, chunk sums C) as k_wide_scatter, but the ranks come from one ballot per bin and round
// and the records of a bin leave a warp in runs (coalesced). nbins <= 32.
// ------------------------------------------------------------------------------------------------------
template <int RBYTES>
__global__ void __launch_bounds__(OSW_THREADS) k_shard_scatter(const uint32_t *__restrict__ dest, uint32_t n, uint32_t nbins, uint32_t chunk_shift,
                                                               const uint16_t *__restrict__ H, const uint32_t *__restrict__ C,
                                                               const unsigned char *__restrict__ payload_in, unsigned char *__restrict__ payload_out,
                                                               uint32_t region_stride)
{
    constexpr uint32_t NW = OSW_THREADS / 32;
    __shared__ uint32_t base[32];        // first output position of bin b for this tile
    __shared__ uint32_t wtot[NW][32];    // items of bin b held by warp w -> exclusive over the warps
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, tile = blockIdx.x;
    const uint32_t start = tile * OSW_TILE;
    if (start >= n) return;
    if (tid < 32) {
        uint32_t acc = 0;
        if (tid < nbins) {
            const uint32_t chunk = tile >> chunk_shift;
            for (uint32_t c = 0; c < chunk; c++) acc += C[static_cast<size_t>(c) * OSW_DIGITS + tid];
            for (uint32_t t = chunk << chunk_shift; t < tile; t++) acc += H[static_cast<size_t>(t) * OSW_DIGITS + tid];
        }
        base[tid] = tid * region_stride + acc;
    }
    // warp w owns [start + w*32*ITEMS, +32*ITEMS), 32 consecutive positions per round; lane b keeps bin b's running count
    uint32_t running = 0;
    uint16_t code[OSW_ITEMS]; // bin (5 bits) | rank inside the warp << 5; 0xffff: dropped
#pragma unroll
    for (uint32_t r = 0; r < OSW_ITEMS; r++) {
        const uint32_t idx = start + warp * (32 * OSW_ITEMS) + r * 32 + lane;
        const uint32_t d = idx < n ? dest[idx] : INVALID_SLOT;
        const uint32_t any = __ballot_sync(FULL, d < nbins);
        code[r] = 0xffffu;
        if (any == 0) continue; // (survivors are at the front of every 256-position tile: the tail rounds are empty)
        uint32_t mine = 0, add = 0;
        for (uint32_t b = 0; b < nbins; b++) {
            const uint32_t bal = __ballot_sync(FULL, d == b);
            if (d == b) mine = __popc(bal & lanemask_lt());
            if (lane == b) add = __popc(bal);
        }
        const uint32_t before = __shfl_sync(FULL, running, d < nbins ? d : 0u);
        if (d < nbins) code[r] = static_cast<uint16_t>(d | ((before + mine) << 5));
        running += add;
    }
    wtot[warp][lane] = running;
    __syncthreads();
    if (tid < 32) { // exclusive offsets over the warps
        uint32_t run = 0;
#pragma unroll
        for (uint32_t w = 0; w < NW; w++) { const uint32_t c = wtot[w][tid]; wtot[w][tid] = run; run += c; }
    }
    __syncthreads();
    using V = typename std::conditional<RBYTES % 16 == 0, uint4, uint2>::type;
    constexpr uint32_t NV = RBYTES / sizeof(V);
#pragma unroll
    for (uint32_t r = 0; r < OSW_ITEMS; r++) {
        if (code[r] != 0xffffu) {
            const uint32_t idx = start + warp * (32 * OSW_ITEMS) + r * 32 + lane;
            const uint32_t b = code[r] & 31u, rank = code[r] >> 5;
            const uint32_t local = base[b] - b * region_stride + wtot[warp][b] + rank; // position inside the region
            if (local < region_stride) {
                const V *src = reinterpret_cast<const V *>(payload_in + static_cast<size_t>(idx) * RBYTES);
                V *dstp = reinterpret_cast<V *>(payload_out + (static_cast<size_t>(b) * region_stride + local) * RBYTES);
                V tmp[NV];
#pragma unroll
                for (uint32_t q = 0; q < NV; q++) tmp[q] = src[q];
#pragma unroll
                for (uint32_t q = 0; q < NV; q++) dstp[q] = tmp[q];
            }
        }
    }
}

// multi-GPU exchange, push with SMs: every peer's slice of records (16-byte words), slots and run lengths (4-byte words) is
// stored straight into that peer's mapped receive buffer over NVLink. MG_PUSH_CTAS CTAs per peer share a slice.
constexpr uint32_t MG_PUSH_CTAS = 16, MG_PUSH_THREADS = 256; // (one CTA moves ~10 GB/s over NVLink: stores to a peer are latency-bound)
struct MgPush {
    const uint4 *rec_src[MAX_SHARDS]; uint4 *rec_dst[MAX_SHARDS]; uint32_t rec_n16[MAX_SHARDS];
    const uint32_t *slot_src[MAX_SHARDS]; uint32_t *slot_dst[MAX_SHARDS]; uint32_t slot_n[MAX_SHARDS];
    const uint32_t *bin_src[MAX_SHARDS]; uint32_t *bin_dst[MAX_SHARDS]; uint32_t bin_n;
};
static __global__ void __launch_bounds__(MG_PUSH_THREADS) k_mg_push(const __grid_constant__ MgPush a)
{
    const uint32_t peer = blockIdx.x / MG_PUSH_CTAS, part = blockIdx.x % MG_PUSH_CTAS;
    const uint32_t t = part * MG_PUSH_THREADS + threadIdx.x, stride = MG_PUSH_CTAS * MG_PUSH_THREADS;
    {
        const uint4 *src = a.rec_src[peer]; uint4 *dst = a.rec_dst[peer]; const uint32_t n = a.rec_n16[peer];
        uint32_t i = t;
        for (; i + 7 * stride < n; i += 8 * stride) { // eight independent 16-byte loads, then eight stores in flight per thread
            uint4 v[8];
#pragma unroll
            for (uint32_t q = 0; q < 8; q++) v[q] = src[i + q * stride];
#pragma unroll
            for (uint32_t q = 0; q < 8; q++) dst[i + q * stride] = v[q];
        }
        for (; i < n; i += stride) dst[i] = src[i];
    }
    {
        const uint32_t *src = a.slot_src[peer]; uint32_t *dst = a.slot_dst[peer]; const uint32_t n = a.slot_n[peer];
        for (uint32_t i = t; i < n; i += stride) dst[i] = src[i];
    }
    if (part == 0) for (uint32_t i = threadIdx.x; i < a.bin_n; i += MG_PUSH_THREADS) a.bin_dst[peer][i] = a.bin_src[peer][i];
}

// counts of the destination partition (wfb_shard_lift): counts_out[0 .. nshards) + overflow flag at [MAX_SHARDS]
static __global__ void k_shard_counts(const uint32_t *__restrict__ digit_counts, uint32_t nshards, uint32_t region_cap, uint32_t *__restrict__ counts_out)
{
    const uint32_t d = threadIdx.x;
    const uint32_t c = d < nshards ? digit_counts[d] : 0u;
    if (d < MAX_SHARDS) counts_out[d] = c;
    const uint32_t over = __ballot_sync(FULL, c > region_cap);
    if (d == 0) counts_out[MAX_SHARDS] = over ? 1u : 0u;
}


// ------------------------------------------------------------------------------------------------------
// k_ffat_update_lanes: ONE THREAD per key for the (usual) keys with few items in the segment: 65 536 keys are 65 536
// independent, short sequential folds -- enough parallelism to hide the latency of the dependent loads that bound the
// warp-per-key kernel. Each thread walks its key's items in arrival order (4 loads in flight), folds them into the open
// pane; a completed pane is written as a FlatFAT leaf and its root path recomputed in a warp-converged step (all lanes
// leave the item loop together when any of them completes a pane), fired groups go to the deferred window list.
// Keys with more than ff.light_max items are put on the heavy list for k_ffat_update (warp per key).
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t level_off(uint32_t n_leaves, uint32_t level);
__device__ __forceinline__ uint64_t batch_watermark(const uint32_t *__restrict__ batch_off, const DevBatch *__restrict__ batches,
                                                    uint32_t nbatches, uint32_t pos);
template <class P>
__device__ __forceinline__ void ffat_eval_window(const FfatDev &ff, const unsigned char *tree, key_words_t<P> key, uint64_t gwid, uint64_t wm,
                                                 uint32_t opos, unsigned char *__restrict__ out_res, uint64_t *__restrict__ out_ts,
                                                 uint32_t out_cap, const typename P::params_t &prm);

template <class P>
__global__ void __launch_bounds__(128) k_ffat_update_lanes(const FfatDev ff, const unsigned char *__restrict__ lifted,
                                                           const uint32_t *__restrict__ sorted_pos,
                                                           const uint32_t *__restrict__ batch_off, const DevBatch *__restrict__ batches,
                                                           uint32_t nbatches, unsigned char *__restrict__ out_res,
                                                           uint64_t *__restrict__ out_ts, uint32_t out_cap, uint32_t *__restrict__ n_out,
                                                           const typename P::params_t prm)
{
    using R = typename P::result_t;
    constexpr uint32_t RB = sizeof(R);
    constexpr uint32_t U = 4; // item loads in flight per thread
    const uint32_t nslots = ff.dense ? ff.max_keys : min(*ff.n_slots, ff.max_keys);
    const uint32_t n = ff.n_leaves, logn = ff.log_leaves;
    const uint64_t P_ = ff.pane;
    const uint64_t group_items = ff.slide * ff.nb;
    const size_t tree_stride = static_cast<size_t>(2 * n - 1) * RB;

    for (uint32_t base = blockIdx.x * blockDim.x; base < nslots; base += gridDim.x * blockDim.x) { // block-uniform
        const uint32_t slot = base + threadIdx.x;
        uint32_t m = (slot < nslots) ? ff.seg_cnt[slot] : 0u;
        if (m > ff.light_max) { // heavy key: k_ffat_update takes it (its seg_cnt stays for that kernel)
            const uint32_t hi = atomicAdd(ff.n_heavy, 1u);
            if (hi < ff.max_keys) ff.heavy[hi] = slot;
            m = 0;
        }
        const bool act = m > 0;
        uint32_t off = 0; uint64_t c = 0, g = 0, trig = 0;
        key_words_t<P> key{};
        alignas(16) R acc;
        unsigned char *tree = ff.tree + static_cast<size_t>(slot) * tree_stride;
        if (act) {
            off = ff.seg_off[slot]; c = ff.cnt[slot];
            key = key_of_slot<P>(ff, slot);
            if (c % P_ != 0) ld_rec<R>(ff.acc + static_cast<size_t>(slot) * RB, acc);
            g = (c < ff.B) ? 0 : 1 + (c - ff.B) / group_items;
            trig = ff.B + g * group_items;
        }
        uint32_t j = 0;
        while (__any_sync(FULL, act && j < m)) {
            // ---- phase 1: fold items until the open pane completes (or the key runs out of items) -------------------
            bool completed = false;
            while (act && j < m && !completed) {
                uint32_t p[U];
                alignas(16) R it[U];
                const uint32_t k = min(U, m - j);
#pragma unroll
                for (uint32_t q = 0; q < U; q++) if (q < k) p[q] = sorted_pos[off + j + q];
#pragma unroll
                for (uint32_t q = 0; q < U; q++) if (q < k) ld_rec<R>(lifted + static_cast<size_t>(p[q]) * RB, it[q]);
#pragma unroll
                for (uint32_t q = 0; q < U; q++) {
                    if (q < k && !completed) {
                        if (c % P_ == 0) acc = it[q]; else P::comb(acc, it[q], acc, prm);
                        c++; j++;
                        completed = (c % P_ == 0);
                    }
                }
            }
            // ---- phase 2 (warp-converged): new leaf, root path, fired groups -----------------------------------------------
            if (completed) {
                const uint32_t leaf = static_cast<uint32_t>((c / P_ - 1) & (n - 1));
                const uint32_t plev = ff.lazy ? 0u : logn; // (lazy: only the leaf is written)
                for (uint32_t l = 0; l < plev; l++) // siblings towards L2 first: the sequential walk below then hits
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(tree + static_cast<size_t>(level_off(n, l) + ((leaf >> l) ^ 1u)) * RB));
                alignas(16) R cur = acc;
                st_rec<R>(tree + static_cast<size_t>(leaf) * RB, cur);
                for (uint32_t l = 0; l < plev; l++) {
                    alignas(16) R s;
                    ld_rec<R>(tree + static_cast<size_t>(level_off(n, l) + ((leaf >> l) ^ 1u)) * RB, s);
                    alignas(16) R parent = cur;
                    if ((leaf >> l) & 1u) P::comb(s, cur, parent, prm); else P::comb(cur, s, parent, prm);
                    cur = parent;
                    st_rec<R>(tree + static_cast<size_t>(level_off(n, l + 1) + (leaf >> (l + 1))) * RB, cur);
                }
                if (c == trig) {
                    const uint32_t last_pos = sorted_pos[off + j - 1]; // arrival position of the triggering item
                    const uint32_t obase = atomicAdd(n_out, ff.nb);
                    bool deferred = (m - j) < ff.defer_items; // the panes this key still completes in this segment fit the spare ring leaves
                    if (deferred) {
                        const uint32_t ti = atomicAdd(ff.n_trig, 1u);
                        if (ti < ff.trig_cap) { Trigger tr; tr.key = trig_word(key); tr.g = g; tr.slot = slot; tr.last_pos = last_pos; tr.obase = obase; tr.pad = 0; ff.trig[ti] = tr; }
                        else deferred = false;
                    }
                    if (!deferred) {
                        const uint64_t wm = batch_watermark(batch_off, batches, nbatches, last_pos);
                        for (uint32_t i = 0; i < ff.nb; i++)
                            ffat_eval_window<P>(ff, tree, key, g * ff.nb + i, wm, obase + i, out_res, out_ts, out_cap, prm);
                    }
                    g++; trig += group_items;
                }
            }
        }
        if (act) {
            ff.cnt[slot] = c;
            if (c % P_ != 0) st_rec<R>(ff.acc + static_cast<size_t>(slot) * RB, acc);
            ff.seg_cnt[slot] = 0;
            ff.seg_off[slot] = 0xffffffffu; // the next segment's sort records the key's first position with atomicMin
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// k_ffat_update_buckets: the window update after ONE wide partition pass (k_wide_scatter_ranked) on the top 10 bits of the
// slot. The pass leaves the bucket list of a position range -- one word per item, its position in the range and its key within
// the bucket (bkl_word) -- in 1024 buckets of at most BK_KEYS consecutive slots, arrival order inside a bucket. One CTA per
// bucket. The kernel's time is the random gather of the records and the
// dependent round trips in front of it, so every phase issues all of its global loads before it uses the first one:
//   0. the bucket's range (scan of the pass histogram), the keys' state, and the items of every key in the whole bucket
//      (BK_CNT_U independent loads of the bucket list per thread and round trip): the deferral of fired groups needs them,
// then per chunk of at most CAP items (arrival order is chunk order; CAP is sized so that the chunk's records take
// BK_REC_BYTES of shared memory). The chunk's part of the bucket list is already in shared memory: it was copied with
// cp.async while the previous chunk ran.
//   1. stable split by key: item r * BK_THREADS + t is thread t's r-th; a warp ranks its items of a key with match_any and
//      files their count per (round, warp) column; scans over the columns and over the keys give every item its place in
//      the key-major order,
//   2. every thread copies its items' records global -> shared in that order with cp.async (all of them in flight at once;
//      16-byte copies bypass L1, where a copy in flight would hold a line); eager FlatFAT levels also stage the siblings of
//      the first leaf each key completes,
//   3. ONE THREAD per segment (the items of a run that fall into one pane) folds them in arrival order from shared memory
//      and leaves the result in place of the segment's first record; then one thread per key walks its segments in order:
//      completed panes become FlatFAT leaves, their root paths are recomputed (staged siblings for the first) and fired
//      groups go to the deferred window list; the last partial segment is the new open pane,
//   4. a chunk with more segments than threads (tiny panes) is folded one warp per key instead (ordered shuffle-tree
//      fold of 32 staged records at a time).
// Per-key bookkeeping (count, position in the open pane, next leaf, next trigger, open-pane accumulator) is computed
// once per CTA by one thread per key and lives in shared memory across the chunks.
// `moved` = 1: the partition pass also moved the records (bucket b's records are lifted[boff[b] ..)); 0: records are
// gathered through the positions, and `lifted` points at the range's first record. pos_base = the range's first position: a
// triggering item's position in the call is pos_base + the position in its word.
// ------------------------------------------------------------------------------------------------------
#ifdef WFB_BK_TRACE
// debug build only, per CTA: start time, time thread 0 spent in phases 1..6 (summed over the chunks), end time (globaltimer ns)
__device__ unsigned long long g_bk_trace[1024 * 8];
__device__ __forceinline__ unsigned long long bk_now() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define BK_TRACE_STATE unsigned long long bk_t = 0
#define BK_MARK(i) do { if (threadIdx.x == 0) { const unsigned long long t_ = bk_now(); unsigned long long *r_ = g_bk_trace + blockIdx.x * 8; \
    if ((i) == 0) { r_[0] = t_; for (int q_ = 1; q_ < 8; q_++) r_[q_] = 0; } else if ((i) == 7) r_[7] = t_; else r_[i] += t_ - bk_t; bk_t = t_; } } while (0)
#else
#define BK_TRACE_STATE do { } while (0)
#define BK_MARK(i) do { } while (0)
#endif
constexpr uint32_t BK_KEYS = 64;      // keys per bucket (at most)
constexpr uint32_t BK_THREADS = 128;
#ifndef WFB_BK_REC_BYTES
#define WFB_BK_REC_BYTES 16384
#endif
constexpr uint32_t BK_REC_BYTES = WFB_BK_REC_BYTES; // shared memory for a chunk's records
constexpr uint32_t BK_CNT_U = 16;     // bucket-list loads in flight per thread (key counts)
// a copy of v the compiler cannot see through: keeps it from computing a shared-memory address from v before the chunk loop
// and holding it (in local memory, under the launch bound) until the write-back
__device__ __forceinline__ uint32_t bk_opaque(uint32_t v) { asm volatile("" : "+r"(v)); return v; }
template <uint32_t RB>                // items per thread and chunk: BK_REC_BYTES of records, 1..8
constexpr uint32_t bk_items_per_thread() { return BK_REC_BYTES / (BK_THREADS * RB) < 1 ? 1 : (BK_REC_BYTES / (BK_THREADS * RB) > 8 ? 8 : BK_REC_BYTES / (BK_THREADS * RB)); }
template <uint32_t RB>                // FlatFAT levels whose siblings k_ffat_update_buckets stages in shared memory
constexpr uint32_t bk_sibl_levels() { return RB <= 32 ? 8 : (RB <= 48 ? 4 : (RB <= 128 ? 2 : 1)); }
// static shared memory of k_ffat_update_buckets<P, LAZY> for results of RB bytes: its arrays below, plus 64 bytes for alignment
template <uint32_t RB, bool LAZY>
constexpr uint32_t bk_smem_bytes()
{
    constexpr uint32_t IT = bk_items_per_thread<RB>(), CAP = BK_THREADS * IT, CS = IT * (BK_THREADS / 32) + 2;
    // (CAP * 4 bytes of the sum are not used since the bucket list is one word per item: kept, so that results above 160 bytes keep
    // the full-sort path)
    return CAP * RB + 3 * CAP * 4 + BK_KEYS * CS * 2 + 5 * BK_KEYS * 4 + 3 * BK_KEYS * 8 + BK_KEYS * RB
         + (LAZY ? 16 : BK_KEYS * bk_sibl_levels<RB>() * RB) + 2 * BK_KEYS * 4 + BK_THREADS * 4 + (BK_THREADS / 32 + 5) * 4 + 64;
}
// The bucket update exists for results whose layout fits the 48 KB of static shared memory (RB <= 160 bytes): a program with larger
// results has no bucket kernel (ProgramOps::ffat_buckets is null) and its count-based handles take the full-sort path at every capacity
template <uint32_t RB>
constexpr bool bk_fits() { return bk_smem_bytes<RB, false>() <= (48u << 10) && bk_smem_bytes<RB, true>() <= (48u << 10); }
#ifndef WFB_BK_MINBLOCKS
#define WFB_BK_MINBLOCKS 4        // eager FlatFAT levels (16 KB of staged siblings on top of the lazy footprint)
#endif
#ifndef WFB_BK_MINBLOCKS_LAZY
#define WFB_BK_MINBLOCKS_LAZY 4   // lazy FlatFAT levels. Update + queries per bench step at 4 CTAs per SM: 153 us; at 6: 167 us; at 7:
#endif                            // 168 us (H100 SXM, 700 W): more resident CTAs only queue more gathers behind each other

template <class P, bool LAZY>
__global__ void __launch_bounds__(BK_THREADS, LAZY ? WFB_BK_MINBLOCKS_LAZY : WFB_BK_MINBLOCKS) k_ffat_update_buckets(const FfatDev ff, const unsigned char *__restrict__ lifted,
                                                                       const uint32_t *__restrict__ bk_list, uint32_t pos_base,
                                                                       const uint32_t *__restrict__ digit_counts, uint32_t shift, uint32_t moved,
                                                                       const uint32_t *__restrict__ batch_off, const DevBatch *__restrict__ batches,
                                                                       uint32_t nbatches, unsigned char *__restrict__ out_res,
                                                                       uint64_t *__restrict__ out_ts, uint32_t out_cap, uint32_t *__restrict__ n_out,
                                                                       const typename P::params_t prm)
{
    using R = typename P::result_t;
    constexpr uint32_t RB = sizeof(R);
    constexpr uint32_t NW = BK_THREADS / 32;
    constexpr uint32_t DPT = OSW_DIGITS / BK_THREADS;                  // digit counts per thread
    constexpr uint32_t IT = bk_items_per_thread<RB>();                 // items per thread and chunk
    constexpr uint32_t CAP = BK_THREADS * IT;                          // items per chunk
    constexpr uint32_t NCOL = IT * NW;                                 // (round, warp) columns of the split counts
    constexpr uint32_t CS = NCOL + 2;                                  // row stride of the split counts (odd in words: no bank conflicts)
    constexpr uint32_t CPB = (RB % 16 == 0) ? 16 : 8;                  // cp.async granule of a record
    constexpr uint32_t BK_SIBL = bk_sibl_levels<RB>();                 // FlatFAT levels whose siblings are staged in shared memory
    static_assert(DPT % 4 == 0 && BK_KEYS == 64 && BK_KEYS == (1u << BKL_KEY_BITS) && BK_THREADS == 128 && RB % 8 == 0, "layout");
    static_assert(bk_fits<RB>(), "the arrays below exceed 48 KB of static shared memory (bk_smem_bytes)");
    __shared__ __align__(16) unsigned char s_rec[CAP * RB]; // the chunk's records, key-major; a segment's fold replaces its first record
    __shared__ uint32_t s_idx[CAP];                    // record index of the items (into `lifted`), key-major
    __shared__ uint32_t s_list[CAP];                   // the bucket list of the next chunk, prefetched
    __shared__ __align__(16) uint16_t s_col[BK_KEYS][CS]; // items of key k in (round, warp) column c -> exclusive over the columns
    __shared__ uint32_t kcnt[BK_KEYS], koff[BK_KEYS];  // items / first index of key k in this chunk
    __shared__ uint32_t kleft[BK_KEYS];                // items of key k still to come in this segment
    __shared__ uint32_t kcp[BK_KEYS], kleaf[BK_KEYS];  // items in the open pane, leaf the open pane will be written to
    __shared__ uint64_t kc[BK_KEYS], kg[BK_KEYS], ktt[BK_KEYS]; // count, groups fired, items until the next trigger
    __shared__ __align__(16) unsigned char kacc[BK_KEYS * RB];   // open-pane accumulator of key k
    __shared__ __align__(16) unsigned char s_sib[LAZY ? 16 : BK_KEYS * BK_SIBL * RB]; // siblings of the leaf key k completes in this chunk (lazy levels: none)
    __shared__ uint32_t s_heavy[BK_KEYS];              // keys folded by a warp in this chunk
    __shared__ uint32_t ksegb[BK_KEYS];                // first segment of key k (a segment = the items of a run that fall into one pane)
    __shared__ uint32_t seg_desc[BK_THREADS];          // key | index of the segment in its run << 8
    __shared__ uint32_t misc[NW], s_boff[2], s_nheavy, s_hnext, s_nseg;

    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t bucket = blockIdx.x;
    const uint32_t kpc = min(BK_KEYS, 1u << shift);    // keys of this bucket
    const uint32_t key_lo = bucket << shift;
    const uint32_t n = ff.n_leaves, logn = ff.log_leaves;
    const uint32_t P32 = static_cast<uint32_t>(ff.pane);
    const uint64_t group_items = ff.slide * ff.nb;
    const size_t tree_stride = static_cast<size_t>(2 * n - 1) * RB;
    BK_TRACE_STATE;

    BK_MARK(0);
    // ---- 0. per-key bookkeeping, one thread per key (loads first: they overlap the histogram scan below) -----------------------
    uint32_t my_total = 0;
    uint64_t st_c = 0;
    const bool has_key = tid < kpc && key_lo + tid < ff.max_keys;
    if (has_key) { // the open-pane accumulator goes straight to shared memory (it has landed by the first fold's barrier)
        const uint32_t slot = key_lo + tid;
        st_c = ff.cnt[slot];
#pragma unroll
        for (uint32_t q = 0; q < RB / CPB; q++) cp_async<CPB>(kacc + tid * RB + q * CPB, ff.acc + static_cast<size_t>(slot) * RB + q * CPB);
    }
    if (tid < BK_KEYS) kleft[tid] = 0;
    // ---- bucket range = exclusive scan of the pass histogram --------------------------------------------------------------
    {
        uint32_t cc[DPT];
#pragma unroll
        for (uint32_t q = 0; q < DPT / 4; q++) {
            const uint4 v = reinterpret_cast<const uint4 *>(digit_counts)[tid * (DPT / 4) + q];
            cc[4 * q] = v.x; cc[4 * q + 1] = v.y; cc[4 * q + 2] = v.z; cc[4 * q + 3] = v.w;
        }
        uint32_t sum = 0;
#pragma unroll
        for (uint32_t q = 0; q < DPT; q++) sum += cc[q];
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
        if (lane == 31) misc[warp] = incl;
        __syncthreads();
        if (tid == bucket / DPT) {
            uint32_t base = incl - sum;
            for (uint32_t w = 0; w < warp; w++) base += misc[w];
            for (uint32_t q = bucket - bucket % DPT; q < bucket; q++) base += digit_counts[q]; // (L1 hits; indexing cc would put it in local memory)
            s_boff[0] = base; s_boff[1] = base + digit_counts[bucket];
        }
        __syncthreads();
    }
    const uint32_t bbeg = s_boff[0], bend = s_boff[1];
    // the bucket list of the chunk at `at` -> s_list, asynchronously. Item r * BK_THREADS + tid is copied and later read by thread
    // tid alone: its own cp.async.wait_all makes it visible, no barrier is needed.
    const auto fetch_list = [&](uint32_t at, uint32_t end) {
#pragma unroll
        for (uint32_t r = 0; r < IT; r++) {
            const uint32_t i = r * BK_THREADS + tid;
            if (at + i < end) cp_async<4>(s_list + i, bk_list + at + i);
        }
    };
    fetch_list(bbeg, bend); // the first chunk's list: in flight during the key counts
    // items of every key in this stream segment (the whole bucket, all chunks): the deferral of fired groups needs them. Counting
    // them here instead of one global RED per survivor in the streaming pass is what that pass is sensitive to (+17 us per RED).
    // BK_CNT_U loads per thread are in flight before the first count: a bucket of 4096 items costs two round trips.
    for (uint32_t base = bbeg; base < bend; base += BK_CNT_U * BK_THREADS) {
        uint32_t lk[BK_CNT_U];
#pragma unroll
        for (uint32_t q = 0; q < BK_CNT_U; q++) {
            const uint32_t i = base + q * BK_THREADS + tid;
            lk[q] = i < bend ? bk_list[i] & (BK_KEYS - 1u) : BK_KEYS;
        }
#pragma unroll
        for (uint32_t q = 0; q < BK_CNT_U; q++) if (lk[q] < BK_KEYS) atomicAdd(&kleft[lk[q]], 1u);
    }
    __syncthreads();
    if (tid < BK_KEYS) {
        const uint32_t m = has_key ? kleft[tid] : 0u;
        my_total = m;
        const uint64_t c = st_c;
        uint64_t g = 0, tt = 0; uint32_t cp = 0, leaf = 0;
        if (m) {
            cp = static_cast<uint32_t>(c % P32); leaf = static_cast<uint32_t>((c / P32) & (n - 1));
            if (c < ff.B) { g = 0; tt = ff.B - c; }
            else { g = 1 + (c - ff.B) / group_items; tt = ff.B + g * group_items - c; }
        }
        kleft[tid] = m; kc[tid] = c; kg[tid] = g; ktt[tid] = tt; kcp[tid] = cp; kleaf[tid] = leaf;
    }
    const uint32_t any_items = __syncthreads_or(my_total != 0);
    BK_MARK(1);
    if (!any_items) { cp_async_wait_all(); BK_MARK(7); return; }
    if (moved)
        for (size_t o = static_cast<size_t>(tid) * 128; o < static_cast<size_t>(bend - bbeg) * RB; o += BK_THREADS * 128) // the bucket's block -> L2
            asm volatile("prefetch.global.L2 [%0];" ::"l"(lifted + static_cast<size_t>(bbeg) * RB + o));

    // s_boff[0] is the chunk cursor: kept in shared memory, no register is held across the chunk
    for (uint32_t cursor = s_boff[0]; cursor < s_boff[1]; cursor = s_boff[0]) {
        const uint32_t nsel = min(CAP, s_boff[1] - cursor);
        // ---- 1. stable split of the chunk's items by key: item r * BK_THREADS + tid is this thread's r-th -------------------------
        uint32_t ek[IT], ep[IT]; // local key (BK_KEYS = none) | rank among the warp's items of the key << 8, record index
        cp_async_wait_all();     // (the first chunk's list; the later ones landed with the previous chunk's gather)
#pragma unroll
        for (uint32_t r = 0; r < IT; r++) {
            const uint32_t i = r * BK_THREADS + tid;
            ek[r] = BK_KEYS; ep[r] = cursor + i;
            if (i < nsel) {
                const uint32_t w = s_list[i];              // (every producer writes items of the bucket's keys only)
                if (!moved) ep[r] = w >> BKL_KEY_BITS;     // records still in arrival order: the index is the position
                ek[r] = w & (BK_KEYS - 1u);
            }
        }
        {
            uint32_t *z = reinterpret_cast<uint32_t *>(&s_col[0][0]);
            for (uint32_t i = tid; i < BK_KEYS * CS / 2; i += BK_THREADS) z[i] = 0;
        }
        __syncthreads();
        fetch_list(cursor + CAP, s_boff[1]); // the next chunk's list, in flight with this chunk's gather (this thread's reads are done)
#pragma unroll
        for (uint32_t r = 0; r < IT; r++) {
            const uint32_t k = ek[r];
            const uint32_t peers = __match_any_sync(FULL, k);
            const uint32_t rank = __popc(peers & lanemask_lt());
            if (k < BK_KEYS && rank == 0) s_col[k][r * NW + warp] = static_cast<uint16_t>(__popc(peers));
            ek[r] = k | rank << 8;
        }
        __syncthreads();
        BK_MARK(2);
        if (warp == 0) { // keys lane and lane+32: exclusive scan over the columns, chunk totals, exclusive scan over the keys, long runs
            uint32_t a0 = 0, a1 = 0;
#pragma unroll
            for (uint32_t c = 0; c < NCOL; c++) {
                const uint32_t v0 = s_col[lane][c], v1 = s_col[lane + 32][c];
                s_col[lane][c] = static_cast<uint16_t>(a0); s_col[lane + 32][c] = static_cast<uint16_t>(a1);
                a0 += v0; a1 += v1;
            }
            uint32_t i0 = a0, i1 = a1;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v0 = __shfl_up_sync(FULL, i0, o), v1 = __shfl_up_sync(FULL, i1, o);
                if (lane >= static_cast<uint32_t>(o)) { i0 += v0; i1 += v1; }
            }
            const uint32_t t0 = __shfl_sync(FULL, i0, 31);
            kcnt[lane] = a0; kcnt[lane + 32] = a1;
            koff[lane] = i0 - a0; koff[lane + 32] = t0 + i1 - a1;
            // segments of the runs: the items that complete the open pane, then one segment per further pane
            const uint32_t c0 = kcp[lane], c1 = kcp[lane + 32];
            const uint32_t f0 = min(a0, P32 - c0), f1 = min(a1, P32 - c1);
            const uint32_t n0 = a0 ? 1u + (a0 - f0 + P32 - 1) / P32 : 0u, n1 = a1 ? 1u + (a1 - f1 + P32 - 1) / P32 : 0u;
            uint32_t s0 = n0, s1 = n1;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v0 = __shfl_up_sync(FULL, s0, o), v1 = __shfl_up_sync(FULL, s1, o);
                if (lane >= static_cast<uint32_t>(o)) { s0 += v0; s1 += v1; }
            }
            const uint32_t st0 = __shfl_sync(FULL, s0, 31), nseg = st0 + __shfl_sync(FULL, s1, 31);
            ksegb[lane] = s0 - n0; ksegb[lane + 32] = st0 + s1 - n1;
            // more segments than threads (tiny panes): every run of the chunk is folded by a warp instead
            const bool fallback = nseg > BK_THREADS;
            const bool h0 = fallback && a0 != 0, h1 = fallback && a1 != 0;
            const uint32_t b0 = __ballot_sync(FULL, h0), b1 = __ballot_sync(FULL, h1);
            if (h0) s_heavy[__popc(b0 & lanemask_lt())] = lane;
            if (h1) s_heavy[__popc(b0) + __popc(b1 & lanemask_lt())] = lane + 32;
            if (lane == 0) { s_nheavy = __popc(b0) + __popc(b1); s_hnext = 0; s_nseg = fallback ? 0u : nseg; }
        }
        __syncthreads();
        // ---- 2. every item's place in the key-major order; its record -> shared memory there (asynchronous) ------------------------
#pragma unroll
        for (uint32_t r = 0; r < IT; r++) {
            const uint32_t k = ek[r] & 255u;
            if (k < BK_KEYS) {
                const uint32_t at = koff[k] + s_col[k][r * NW + warp] + (ek[r] >> 8);
                s_idx[at] = ep[r];
                const unsigned char *src = lifted + static_cast<size_t>(ep[r]) * RB;
#pragma unroll
                for (uint32_t q = 0; q < RB / CPB; q++) { // (16-byte granules bypass L1: the records are read once)
                    if constexpr (CPB == 16) cp_async_cg16(s_rec + at * RB + q * CPB, src + q * CPB);
                    else cp_async<CPB>(s_rec + at * RB + q * CPB, src + q * CPB);
                }
            }
        }
        // segment descriptors; siblings of the first leaf each key completes -> shared memory
        const uint32_t nseg = s_nseg;
        bool sib_staged = false;
        if (tid < BK_KEYS && nseg != 0) {
            const uint32_t m = kcnt[tid];
            if (m != 0) {
                const uint32_t cp0 = kcp[tid], first = min(m, P32 - cp0), ns = 1u + (m - first + P32 - 1) / P32, sb = ksegb[tid];
                for (uint32_t j = 0; j < ns; j++) seg_desc[sb + j] = tid | (j << 8);
                if (!LAZY && cp0 + first == P32) {
                    const uint32_t leaf = kleaf[tid];
                    const unsigned char *tr = ff.tree + static_cast<size_t>(key_lo + tid) * tree_stride;
                    for (uint32_t l = 0; l < min(logn, BK_SIBL); l++) {
                        const unsigned char *src = tr + static_cast<size_t>(level_off(n, l) + ((leaf >> l) ^ 1u)) * RB;
                        unsigned char *dst = s_sib + (tid * BK_SIBL + l) * RB;
#pragma unroll
                        for (uint32_t q = 0; q < RB / CPB; q++) cp_async<CPB>(dst + q * CPB, src + q * CPB);
                    }
                    sib_staged = true;
                }
            }
        }
        cp_async_wait_all();
        __syncthreads();
        BK_MARK(3);
        // ---- 3a. one thread per segment: ordered fold of at most one pane of staged records ------------------------------------
        if (tid < nseg) {
            const uint32_t d = seg_desc[tid], k = d & 255u, j = d >> 8;
            const uint32_t m = kcnt[k], cp0 = kcp[k], first = min(m, P32 - cp0);
            const uint32_t start = j == 0 ? 0u : first + (j - 1) * P32;
            const uint32_t seg = j == 0 ? first : min(P32, m - start);
            unsigned char *rp = s_rec + (koff[k] + start) * RB;
            alignas(16) R acc;
            uint32_t i = 1;
            if (j == 0 && cp0 != 0) { ld_rec<R>(kacc + k * RB, acc); i = 0; } // the open pane continues
            else ld_rec<R>(rp, acc);
#pragma unroll 4
            for (; i < seg; i++) { alignas(16) R it; ld_rec<R>(rp + i * RB, it); P::comb(acc, it, acc, prm); }
            st_rec<R>(rp, acc);
        }
        __syncthreads();
        BK_MARK(4);
        // ---- 3b. one thread per key, its segments in order: completed panes -> leaf + root path + fired group; the rest is the open
        // pane. The loop over the segments is warp-uniform: a group that cannot be deferred (another pane of the key completes
        // in this stream segment and would overwrite ring leaves the windows still need) is evaluated by the whole warp at once.
        if (tid < BK_KEYS && nseg != 0) { // warps 0 and 1, whole
            const uint32_t k = bk_opaque(tid), m = kcnt[k]; // (the key's slot, key_lo + k, and tree are recomputed where they are used)
            const uint32_t cp0 = kcp[k];
            uint32_t leafi = kleaf[k], new_cp = cp0, consumed = 0;
            uint64_t g = kg[k], tt = ktt[k]; // tt: index (1-based) of the run's item that fires the next group
            while (__any_sync(FULL, consumed < m)) {
                bool eval_now = false;
                uint32_t ev_obase = 0, ev_pos = 0;
                uint64_t ev_g = 0;
                if (consumed < m) {
                    const uint32_t open = consumed == 0 ? cp0 : 0u; // items already in the pane the segment continues
                    const uint32_t len = min(m - consumed, P32 - open);
                    alignas(16) R cur;
                    ld_rec<R>(s_rec + (koff[k] + consumed) * RB, cur); // the segment's fold
                    consumed += len;
                    const bool completes = open + len == P32;
                    if (!completes) { st_rec<R>(kacc + k * RB, cur); new_cp = open + len; } // (only the last segment)
                    else {
                        new_cp = 0;
                        const uint32_t slot = key_lo + k, leaf = leafi;
                        unsigned char *tree = ff.tree + static_cast<size_t>(slot) * tree_stride;
                        leafi = (leafi + 1) & (n - 1);
                        st_rec<R>(tree + static_cast<size_t>(leaf) * RB, cur);
                        for (uint32_t l0 = 0; l0 < (LAZY ? 0u : logn); l0 += 4) { // siblings of four levels per round trip (none of them is on the path)
                            alignas(16) R sbl[4];
#pragma unroll
                            for (uint32_t q = 0; q < 4; q++) {
                                const uint32_t l = l0 + q;
                                if (l < logn) {
                                    if (sib_staged && l < BK_SIBL) ld_rec<R>(s_sib + (k * BK_SIBL + l) * RB, sbl[q]);
                                    else ld_rec<R>(tree + static_cast<size_t>(level_off(n, l) + ((leaf >> l) ^ 1u)) * RB, sbl[q]);
                                }
                            }
#pragma unroll
                            for (uint32_t q = 0; q < 4; q++) {
                                const uint32_t l = l0 + q;
                                if (l < logn) {
                                    alignas(16) R parent = cur;
                                    if ((leaf >> l) & 1u) P::comb(sbl[q], cur, parent, prm); else P::comb(cur, sbl[q], parent, prm);
                                    cur = parent;
                                    st_rec<R>(tree + static_cast<size_t>(level_off(n, l + 1) + (leaf >> (l + 1))) * RB, cur);
                                }
                            }
                        }
                        sib_staged = false; // the next pane of the same run reads the tree it has just written
                        if (consumed == tt) {
                            const uint32_t lp = s_idx[koff[k] + consumed - 1];
                            const uint32_t last_pos = pos_base + (moved ? bk_list[lp] >> BKL_KEY_BITS : lp); // arrival position of the triggering item
                            const uint32_t obase = atomicAdd(n_out, ff.nb);
                            bool deferred = (kleft[k] - consumed) < ff.defer_items; // the panes this key still completes in this segment fit the spare ring leaves
                            if (deferred) {
                                const uint32_t ti = atomicAdd(ff.n_trig, 1u);
                                if (ti < ff.trig_cap) { Trigger tr; tr.key = trig_word(key_of_slot<P>(ff, slot)); tr.g = g; tr.slot = slot; tr.last_pos = last_pos; tr.obase = obase; tr.pad = 0; ff.trig[ti] = tr; }
                                else deferred = false;
                            }
                            if (!deferred) { eval_now = true; ev_obase = obase; ev_pos = last_pos; ev_g = g; }
                            g++; tt += group_items;
                        }
                    }
                }
                // groups to evaluate before their key's next pane: one after the other, the warp's lanes share the windows
                uint32_t pend = __ballot_sync(FULL, eval_now);
                while (pend) {
                    const int src = __ffs(pend) - 1;
                    pend &= pend - 1;
                    const uint32_t e_slot = key_lo + (warp << 5) + src, e_obase = __shfl_sync(FULL, ev_obase, src), e_pos = __shfl_sync(FULL, ev_pos, src);
                    const key_words_t<P> e_key = key_of_slot<P>(ff, e_slot);
                    const uint64_t e_g = __shfl_sync(FULL, ev_g, src);
                    const unsigned char *e_tree = ff.tree + static_cast<size_t>(e_slot) * tree_stride;
                    const uint64_t wm = batch_watermark(batch_off, batches, nbatches, e_pos);
                    for (uint32_t i = lane; i < ff.nb; i += 32)
                        ffat_eval_window<P>(ff, e_tree, e_key, e_g * ff.nb + i, wm, e_obase + i, out_res, out_ts, out_cap, prm);
                }
                __syncwarp(); // the evaluated windows read tree nodes another lane has just written, and it may overwrite them next
            }
            if (m != 0) { kc[k] += m; kg[k] = g; ktt[k] = tt - m; kcp[k] = new_cp; kleaf[k] = leafi; kleft[k] -= m; }
        }
        BK_MARK(5);
        // ---- 4. tiny panes: one warp per key, ordered shuffle-tree fold of 32 staged records at a time -----------------------------
        if (s_nheavy != 0) { // (block-uniform: written before the last barrier)
            __syncthreads();
            for (;;) { // a warp claims the next key (no loop counter is held across the fold)
                uint32_t h = 0;
                if (lane == 0) h = atomicAdd(&s_hnext, 1u);
                h = __shfl_sync(FULL, h, 0);
                if (h >= s_nheavy) break;
                const uint32_t k = s_heavy[h];
                const uint32_t m = kcnt[k], off = koff[k], slot = key_lo + k;
                uint64_t g = kg[k], tt = ktt[k];
                uint32_t cp = kcp[k], leafi = kleaf[k], left = kleft[k];
                unsigned char *tree = ff.tree + static_cast<size_t>(slot) * tree_stride;
                alignas(16) R acc;
                if (cp) ld_rec<R>(kacc + k * RB, acc);
                uint32_t j = 0;
                while (j < m) {
                    const uint32_t cnt = min(32u, m - j);
                    alignas(16) R cur_rec;
                    if (lane < cnt) ld_rec<R>(s_rec + (off + j + lane) * RB, cur_rec);
                    uint32_t lo = 0;
                    while (lo < cnt) { // sub-ranges of the 32 records that fall into one pane
                        const uint32_t hi = min(cnt, lo + (P32 - cp));
                        alignas(16) R r = cur_rec;
#pragma unroll
                        for (uint32_t o = 1; o < 32; o <<= 1) {
                            const R other = shfl_down_rec<R>(r, o);
                            if (lane >= lo && lane + o < hi) P::comb(r, other, r, prm);
                        }
                        r = shfl_rec<R>(r, lo);
                        if (cp == 0) acc = r; else P::comb(acc, r, acc, prm);
                        const uint32_t take = hi - lo;
                        cp += take; left -= take; tt -= take;
                        if (cp == P32) { // pane complete -> leaf + root path
                            cp = 0;
                            const uint32_t leaf = leafi;
                            leafi = (leafi + 1) & (n - 1);
                            alignas(16) R sib;
                            const uint32_t plev = LAZY ? 0u : logn; // (lazy: only the leaf is written)
                            if (lane < plev) ld_rec<R>(tree + static_cast<size_t>(level_off(n, lane) + ((leaf >> lane) ^ 1u)) * RB, sib);
                            alignas(16) R cur = acc;
                            if (lane == 0) st_rec<R>(tree + static_cast<size_t>(leaf) * RB, cur);
                            for (uint32_t l = 0; l < plev; l++) {
                                const R sb = shfl_rec<R>(sib, l);
                                alignas(16) R parent = cur;
                                if ((leaf >> l) & 1u) P::comb(sb, cur, parent, prm); else P::comb(cur, sb, parent, prm);
                                cur = parent;
                                if (lane == 0) st_rec<R>(tree + static_cast<size_t>(level_off(n, l + 1) + (leaf >> (l + 1))) * RB, cur);
                            }
                            __syncwarp();
                            if (tt == 0) {
                                const uint32_t lp = s_idx[off + j + hi - 1];
                                const uint32_t last_pos = pos_base + (moved ? bk_list[lp] >> BKL_KEY_BITS : lp); // arrival position of the triggering item
                                uint32_t obase = 0;
                                if (lane == 0) obase = atomicAdd(n_out, ff.nb);
                                obase = __shfl_sync(FULL, obase, 0);
                                bool deferred = left < ff.defer_items; // the panes this key still completes in this segment fit the spare ring leaves
                                if (deferred) {
                                    uint32_t ti = 0;
                                    if (lane == 0) ti = atomicAdd(ff.n_trig, 1u);
                                    ti = __shfl_sync(FULL, ti, 0);
                                    if (ti < ff.trig_cap) {
                                        if (lane == 0) { Trigger tr; tr.key = trig_word(key_of_slot<P>(ff, slot)); tr.g = g; tr.slot = slot; tr.last_pos = last_pos; tr.obase = obase; tr.pad = 0; ff.trig[ti] = tr; }
                                    } else deferred = false;
                                }
                                if (!deferred) {
                                    const uint64_t wm = batch_watermark(batch_off, batches, nbatches, last_pos);
                                    const key_words_t<P> key = key_of_slot<P>(ff, slot);
                                    for (uint32_t i = lane; i < ff.nb; i += 32)
                                        ffat_eval_window<P>(ff, tree, key, g * ff.nb + i, wm, obase + i, out_res, out_ts, out_cap, prm);
                                }
                                g++; tt = group_items;
                                __syncwarp();
                            }
                        }
                        lo = hi;
                    }
                    j += cnt;
                }
                if (lane == 0) {
                    kc[k] += m; kg[k] = g; ktt[k] = tt; kcp[k] = cp; kleaf[k] = leafi; kleft[k] = left;
                    if (cp) st_rec<R>(kacc + k * RB, acc);
                }
            }
        }
        if (tid == 0) s_boff[0] += CAP; // (every thread has read it before the chunk's first barrier)
        __syncthreads(); // the next chunk overwrites the shared buffers
        BK_MARK(6);
    }
    // ---- keys' state back as contiguous blocks (a key without items rewrites its count; its cp is 0: no accumulator) ------------
    if (tid < kpc && key_lo + tid < ff.max_keys) {
        const uint32_t k = bk_opaque(tid), slot = key_lo + k;
        ff.cnt[slot] = kc[k];
        if (kcp[k]) { alignas(16) R a; ld_rec<R>(kacc + k * RB, a); st_rec<R>(ff.acc + static_cast<size_t>(slot) * RB, a); }
    }
    BK_MARK(7);
}

// ------------------------------------------------------------------------------------------------------
// k_ffat_update: one warp per key that k_ffat_update_lanes put on the heavy list.
//   items of the key, in arrival order: lifted[sorted_pos[seg_off[slot] .. +seg_cnt[slot])]
//   -> ordered warp fold into the open pane (pane = gcd(win, slide) items)
//   -> completed pane = new FlatFAT leaf (ring of n_leaves panes) + recompute of its root path
//   -> when the key's count reaches the trigger: Nb window queries (greedy aligned-node fold, the same walk as
//      Compute_Results_Kernel, wf/flatfat_gpu.hpp:93-139, over panes instead of tuples)
// Window / trigger bookkeeping restates Ffat_Replica_GPU::process_wins_cb (wf/ffat_replica_gpu.hpp:830-867):
// groups fired so far G(c) = c < B ? 0 : 1 + (c - B) / (S*Nb); next_gwid = G*Nb; trigger = B + G*S*Nb.
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t level_off(uint32_t n_leaves, uint32_t level) { return 2u * n_leaves - ((2u * n_leaves) >> level); }

// watermark of the batch that holds compact position `pos` (batch_off has nbatches+1 ascending entries)
__device__ __forceinline__ uint64_t batch_watermark(const uint32_t *__restrict__ batch_off, const DevBatch *__restrict__ batches,
                                                    uint32_t nbatches, uint32_t pos)
{
    uint32_t lo = 0, hi = nbatches - 1;
    while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (batch_off[mid] <= pos) lo = mid; else hi = mid - 1; }
    return batches[lo].watermark;
}

// one window: result_t(key, gwid) folded left to right over the largest aligned FlatFAT nodes covering panes
// [gwid*sp, gwid*sp + wp) of the key's ring (the walk of Compute_Results_Kernel, wf/flatfat_gpu.hpp:109-136)
template <class P>
__device__ __forceinline__ void ffat_eval_window(const FfatDev &ff, const unsigned char *tree, key_words_t<P> key, uint64_t gwid, uint64_t wm,
                                                 uint32_t opos, unsigned char *__restrict__ out_res, uint64_t *__restrict__ out_ts,
                                                 uint32_t out_cap, const typename P::params_t &prm)
{
    using R = typename P::result_t;
    constexpr uint32_t RB = sizeof(R);
    const uint32_t n = ff.n_leaves;
    alignas(16) R res = P::make_result(key_codec<P>::decode(key), gwid, prm);
    uint32_t ws = static_cast<uint32_t>((gwid * ff.sp) & (n - 1));
    uint32_t remaining = ff.wp;
    if (ff.lazy) { // only the leaves are kept in global memory: fold them in order (the rare in-kernel evaluations; the deferred groups go
                   // through k_ffat_windows_lazy, which builds the levels on chip)
        for (; remaining > 0; remaining--) {
            alignas(16) R node;
            ld_rec<R>(tree + static_cast<size_t>(ws) * RB, node);
            P::comb(res, node, res, prm);
            ws = (ws + 1) & (n - 1);
        }
    }
    while (remaining > 0) {
        uint32_t range = (ws == 0) ? n : (ws & (0u - ws));
        const uint32_t pw = 1u << (31 - __clz(remaining));
        range = min(range, pw);
        const uint32_t level = 31 - __clz(range);
        alignas(16) R node;
        ld_rec<R>(tree + static_cast<size_t>(level_off(n, level) + (ws >> level)) * RB, node);
        P::comb(res, node, res, prm);
        ws = (ws + range) & (n - 1);
        remaining -= range;
    }
    if (opos < out_cap) {
        st_rec<R>(out_res + static_cast<size_t>(opos) * RB, res);
        if (out_ts != nullptr) out_ts[opos] = wm;
    } else atomicOr(ff.err_flags, 2u);
}

// deferred window groups: one thread per window
template <class P>
__global__ void __launch_bounds__(256) k_ffat_windows(const FfatDev ff, const uint32_t *__restrict__ batch_off,
                                                      const DevBatch *__restrict__ batches, uint32_t nbatches,
                                                      unsigned char *__restrict__ out_res, uint64_t *__restrict__ out_ts, uint32_t out_cap,
                                                      const typename P::params_t prm, uint32_t *__restrict__ n_out)
{
    using R = typename P::result_t;
    // the update kernels reserve output slots with atomicAdd(n_out, Nb) whether they fit or not: a count beyond the capacity is clamped
    // here (the last kernel of the call) and flagged, so that *n_out is always the number of results actually written
    if (blockIdx.x == 0 && threadIdx.x == 0 && n_out != nullptr) {
        if (*n_out > out_cap) { *n_out = out_cap; atomicOr(ff.err_flags, 2u); }
        if (ff.results_total != nullptr) *ff.results_total += *n_out;
    }
    const uint32_t nt = min(*ff.n_trig, ff.trig_cap);
    const uint64_t total = static_cast<uint64_t>(nt) * ff.nb;
    const size_t tree_stride = static_cast<size_t>(2 * ff.n_leaves - 1) * sizeof(R);
    for (uint64_t w = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; w < total; w += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
        const uint32_t ti = static_cast<uint32_t>(w / ff.nb), i = static_cast<uint32_t>(w % ff.nb);
        const Trigger tr = ff.trig[ti];
        const uint64_t wm = batch_watermark(batch_off, batches, nbatches, tr.last_pos);
        ffat_eval_window<P>(ff, ff.tree + static_cast<size_t>(tr.slot) * tree_stride, trig_key<P>(ff, tr), tr.g * ff.nb + i, wm, tr.obase + i,
                            out_res, out_ts, out_cap, prm);
    }
}

// deferred window groups of a handle that keeps only the pane leaves (FfatDev::lazy): ONE WARP per fired group. The warp copies the key's
// n leaves to shared memory (coalesced), builds the n - 1 internal nodes level by level -- the nodes of a level are independent: lanes take
// them round-robin, one __syncwarp per level ("the FlatFAT levels with warp-level primitives") -- and then every lane evaluates its share of
// the group's Nb windows with the same greedy aligned-node walk over the on-chip tree. Dynamic shared memory: warps per block x 2 n x sizeof(R).
template <class P>
__global__ void __launch_bounds__(128) k_ffat_windows_lazy(const FfatDev ff, const uint32_t *__restrict__ batch_off,
                                                           const DevBatch *__restrict__ batches, uint32_t nbatches,
                                                           unsigned char *__restrict__ out_res, uint64_t *__restrict__ out_ts, uint32_t out_cap,
                                                           const typename P::params_t prm, uint32_t *__restrict__ n_out)
{
    using R = typename P::result_t;
    constexpr uint32_t RB = sizeof(R);
    extern __shared__ __align__(16) unsigned char lazy_smem[];
    if (blockIdx.x == 0 && threadIdx.x == 0 && n_out != nullptr) {
        if (*n_out > out_cap) { *n_out = out_cap; atomicOr(ff.err_flags, 2u); }
        if (ff.results_total != nullptr) *ff.results_total += *n_out;
    }
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const uint32_t n = ff.n_leaves, logn = ff.log_leaves;
    unsigned char *t = lazy_smem + static_cast<size_t>(warp) * 2u * n * RB; // (2 n - 1) nodes, levels back to back as in the global layout
    const uint32_t nt = min(*ff.n_trig, ff.trig_cap);
    const size_t tree_stride = static_cast<size_t>(2 * n - 1) * RB;
    FfatDev fs = ff; fs.lazy = 0; // the on-chip tree has every level: the ordinary walk
    for (uint32_t ti = blockIdx.x * wpb + warp; ti < nt; ti += gridDim.x * wpb) {
        const Trigger tr = ff.trig[ti];
        const unsigned char *leaves = ff.tree + static_cast<size_t>(tr.slot) * tree_stride;
        for (uint32_t i = lane; i < n * (RB / 8); i += 32) reinterpret_cast<uint64_t *>(t)[i] = reinterpret_cast<const uint64_t *>(leaves)[i];
        __syncwarp();
        for (uint32_t l = 0; l < logn; l++) {
            const unsigned char *src = t + static_cast<size_t>(level_off(n, l)) * RB;
            unsigned char *dst = t + static_cast<size_t>(level_off(n, l + 1)) * RB;
            for (uint32_t i = lane; i < (n >> (l + 1)); i += 32) {
                alignas(16) R a, b, o;
                ld_rec<R>(src + static_cast<size_t>(2 * i) * RB, a); ld_rec<R>(src + static_cast<size_t>(2 * i + 1) * RB, b);
                o = a;
                P::comb(a, b, o, prm);
                st_rec<R>(dst + static_cast<size_t>(i) * RB, o);
            }
            __syncwarp();
        }
        const uint64_t wm = batch_watermark(batch_off, batches, nbatches, tr.last_pos);
        for (uint32_t i = lane; i < ff.nb; i += 32)
            ffat_eval_window<P>(fs, t, trig_key<P>(ff, tr), tr.g * ff.nb + i, wm, tr.obase + i, out_res, out_ts, out_cap, prm);
        __syncwarp(); // the next group overwrites the on-chip tree
    }
}

template <class P>
__global__ void __launch_bounds__(256) k_ffat_update(const FfatDev ff, const unsigned char *__restrict__ lifted,
                                                     const uint32_t *__restrict__ sorted_pos,
                                                     const uint32_t *__restrict__ batch_off, const DevBatch *__restrict__ batches,
                                                     uint32_t nbatches, unsigned char *__restrict__ out_res,
                                                     uint64_t *__restrict__ out_ts, uint32_t out_cap, uint32_t *__restrict__ n_out,
                                                     const typename P::params_t prm)
{
    using R = typename P::result_t;
    constexpr uint32_t RB = sizeof(R);
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t n = ff.n_leaves, logn = ff.log_leaves;
    const uint64_t P_ = ff.pane;
    const uint64_t group_items = ff.slide * ff.nb;
    const size_t tree_stride = static_cast<size_t>(2 * n - 1) * RB;

    const uint32_t nwork = min(*ff.n_heavy, ff.max_keys);
    for (uint32_t wi = gwarp; wi < nwork; wi += nwarps) {
        const uint32_t slot = ff.heavy[wi];
        const uint32_t m = ff.seg_cnt[slot];
        if (m == 0) continue;
        const uint32_t off = ff.seg_off[slot];
        uint64_t c = ff.cnt[slot];
        const key_words_t<P> key = key_of_slot<P>(ff, slot);
        unsigned char *tree = ff.tree + static_cast<size_t>(slot) * tree_stride;
        alignas(16) R acc;
        if (c % P_ != 0) ld_rec<R>(ff.acc + static_cast<size_t>(slot) * RB, acc); // every lane keeps a copy
        uint64_t g = (c < ff.B) ? 0 : 1 + (c - ff.B) / group_items;
        uint64_t trig = ff.B + g * group_items;

        uint32_t j = 0;
        while (j < m) {
            const uint32_t room = static_cast<uint32_t>(P_ - (c % P_));
            const uint32_t take = min(min(32u, m - j), room);
            alignas(16) R r;
            if (lane < take) {
                ld_rec<R>(lifted + static_cast<size_t>(sorted_pos[off + j + lane]) * RB, r);
            }
            // ordered fold: after the step with stride o, lane l holds items [l, l+2o) (clipped to take)
#pragma unroll
            for (uint32_t o = 1; o < 32; o <<= 1) {
                const R other = shfl_down_rec<R>(r, o);
                if (lane + o < take) P::comb(r, other, r, prm);
            }
            r = shfl_rec<R>(r, 0);
            if (c % P_ == 0) acc = r; else P::comb(acc, r, acc, prm);
            c += take; j += take;

            if (c % P_ == 0) { // pane complete -> leaf + root path
                const uint32_t leaf = static_cast<uint32_t>((c / P_ - 1) & (n - 1));
                alignas(16) R sib;
                const uint32_t plev = ff.lazy ? 0u : logn; // (lazy: only the leaf is written)
                if (lane < plev) { // lane l fetches the sibling of the path node at level l
                    const uint32_t idx = (leaf >> lane) ^ 1u;
                    ld_rec<R>(tree + static_cast<size_t>(level_off(n, lane) + idx) * RB, sib);
                }
                alignas(16) R cur = acc;
                if (lane == 0) st_rec<R>(tree + static_cast<size_t>(leaf) * RB, cur);
                for (uint32_t l = 0; l < plev; l++) {
                    const R s = shfl_rec<R>(sib, l);
                    alignas(16) R parent = cur; // key/id fields are don't-care in internal nodes
                    if ((leaf >> l) & 1u) P::comb(s, cur, parent, prm); else P::comb(cur, s, parent, prm);
                    cur = parent;
                    if (lane == 0) st_rec<R>(tree + static_cast<size_t>(level_off(n, l + 1) + (leaf >> (l + 1))) * RB, cur);
                }
                __syncwarp();

                if (c == trig) { // fire Nb windows: gwid = g*Nb + i
                    const uint32_t last_pos = sorted_pos[off + j - 1]; // arrival position of the triggering item
                    uint32_t obase = 0;
                    if (lane == 0) obase = atomicAdd(n_out, ff.nb);
                    obase = __shfl_sync(FULL, obase, 0);
                    // No further pane of this key can complete in this segment => the tree stays as it is now and the
                    // queries can run later, thread-per-window, in k_ffat_windows; otherwise evaluate them here.
                    bool deferred = (m - j) < ff.defer_items;
                    if (deferred) {
                        uint32_t ti = 0;
                        if (lane == 0) ti = atomicAdd(ff.n_trig, 1u);
                        ti = __shfl_sync(FULL, ti, 0);
                        if (ti < ff.trig_cap) {
                            if (lane == 0) { Trigger tr; tr.key = trig_word(key); tr.g = g; tr.slot = slot; tr.last_pos = last_pos; tr.obase = obase; tr.pad = 0; ff.trig[ti] = tr; }
                        } else deferred = false;
                    }
                    if (!deferred) {
                        const uint64_t wm = batch_watermark(batch_off, batches, nbatches, last_pos);
                        for (uint32_t i = lane; i < ff.nb; i += 32)
                            ffat_eval_window<P>(ff, tree, key, g * ff.nb + i, wm, obase + i, out_res, out_ts, out_cap, prm);
                    }
                    g++; trig += group_items;
                    __syncwarp();
                }
            }
        }
        if (lane == 0) {
            ff.cnt[slot] = c;
            if (c % P_ != 0) st_rec<R>(ff.acc + static_cast<size_t>(slot) * RB, acc);
            ff.seg_cnt[slot] = 0;
            ff.seg_off[slot] = 0xffffffffu;
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// Per-batch keyed operators built on the sort: KeyBy_Emitter_GPU grouping, Reduce_GPU, key -> shard partition
// ------------------------------------------------------------------------------------------------------
// keys[i] = key_extr(tuple_i)   (Extract_Keys_Kernel wf/reduce_gpu.hpp:75-86, Extract_Dests_Kernel wf/keyby_emitter_gpu.hpp:68-81)
template <class P>
__global__ void k_extract_keys(const unsigned char *__restrict__ tuples, uint32_t n, uint64_t *__restrict__ keys,
                               uint32_t *__restrict__ dest, uint32_t num_shards, const typename P::params_t prm)
{
    using T = typename P::tuple_t;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const T *t = reinterpret_cast<const T *>(tuples + static_cast<size_t>(i) * sizeof(T));
        const uint64_t k = key_word0(key_words<P>(*t, prm)); // (integer keys: other key types go through k_key_order_words)
        if (keys) keys[i] = k;
        if (dest) dest[i] = static_cast<uint32_t>(k % num_shards); // wf/keyby_emitter.hpp:215-217
    }
}

// head[i] = 1 when sorted position i starts a new key; map_idxs links equal neighbours
// (Compute_Mapping_Kernel, wf/keyby_emitter_gpu.hpp:84-100)
static __global__ void k_seg_heads(const uint64_t *__restrict__ skeys, const uint32_t *__restrict__ sidx, uint32_t n,
                            uint32_t *__restrict__ head, int32_t *__restrict__ map_idxs)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        head[i] = (i == 0 || skeys[i] != skeys[i - 1]) ? 1u : 0u;
        if (map_idxs) map_idxs[sidx[i]] = (i + 1 < n && skeys[i] == skeys[i + 1]) ? static_cast<int32_t>(sidx[i + 1]) : -1;
    }
}

// after the exclusive scan of head[] (seg[i] = index of the segment sorted position i belongs to, for heads):
// start_idxs[k] / dist_keys[k] of the k-th distinct key (unique_by_key_copy, wf/keyby_emitter_gpu.hpp:559-564),
// seg_begin[k] = first sorted position of segment k (used by the reduce), *n_keys = number of segments
static __global__ void k_seg_finish(const uint64_t *__restrict__ skeys, const uint32_t *__restrict__ sidx, const uint32_t *__restrict__ head_scan,
                             uint32_t n, int32_t *__restrict__ start_idxs, uint64_t *__restrict__ dist_keys,
                             uint32_t *__restrict__ seg_begin, uint32_t *__restrict__ n_keys)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const bool is_head = (i == 0 || skeys[i] != skeys[i - 1]);
        if (is_head) {
            const uint32_t k = head_scan[i];
            if (start_idxs) start_idxs[k] = static_cast<int32_t>(sidx[i]);
            if (dist_keys) dist_keys[k] = skeys[i];
            if (seg_begin) seg_begin[k] = i;
        }
        if (i == n - 1) {
            const uint32_t total = head_scan[i] + (is_head ? 1u : 0u); // exclusive scan value + own flag
            if (n_keys) *n_keys = total;
            if (seg_begin) seg_begin[total] = n;
        }
    }
}

// Reduce_GPU keyed: one warp per distinct key folds the key's items in arrival order with P::reduce, ts = max
// (thrust_reduce_func_gpu_t, wf/reduce_gpu.hpp:88-105; reduce_by_key :245-252). Output k = k-th smallest key.
template <class P>
__global__ void __launch_bounds__(256) k_reduce_segments(const unsigned char *__restrict__ tuples, const uint64_t *__restrict__ ts,
                                                         const uint32_t *__restrict__ sidx, const uint32_t *__restrict__ seg_begin,
                                                         const uint32_t *__restrict__ n_keys, unsigned char *__restrict__ out_tuples,
                                                         uint64_t *__restrict__ out_ts, const typename P::params_t prm)
{
    using T = typename P::tuple_t;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t nk = *n_keys;
    for (uint32_t k = gwarp; k < nk; k += nwarps) {
        const uint32_t b = seg_begin[k], e = seg_begin[k + 1];
        alignas(16) T acc; uint64_t mts = 0; bool have = false;
        for (uint32_t j = b; j < e; j += 32) {
            const uint32_t take = min(32u, e - j);
            alignas(16) T t; uint64_t tt = 0;
            if (lane < take) {
                const uint32_t i = sidx[j + lane];
                ld_rec<T>(tuples + static_cast<size_t>(i) * sizeof(T), t);
                tt = ts ? ts[i] : 0;
            }
#pragma unroll
            for (uint32_t o = 1; o < 32; o <<= 1) {
                const T other = shfl_down_rec<T>(t, o);
                const uint64_t ots = __shfl_down_sync(FULL, tt, o);
                if (lane + o < take) { t = P::reduce(t, other, prm); tt = tt < ots ? ots : tt; }
            }
            t = shfl_rec<T>(t, 0); tt = __shfl_sync(FULL, tt, 0);
            if (!have) { acc = t; mts = tt; have = true; }
            else { acc = P::reduce(acc, t, prm); mts = mts < tt ? tt : mts; }
        }
        if (lane == 0) {
            st_rec<T>(out_tuples + static_cast<size_t>(k) * sizeof(T), acc);
            if (out_ts) out_ts[k] = mts;
        }
    }
}

// ---- Reduce_GPU over K queued batches in one launch sequence: composite sort key (batch index << key_bits) | key ----------
// batch of global element index gi (boff has nb+1 ascending entries)
__device__ __forceinline__ uint32_t batch_of(const uint32_t *__restrict__ boff, uint32_t nb, uint32_t gi)
{
    uint32_t lo = 0, hi = nb - 1;
    while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (boff[mid] <= gi) lo = mid; else hi = mid - 1; }
    return lo;
}

template <class P>
__global__ void k_extract_keys_batches(const DevBatch *__restrict__ batches, const uint32_t *__restrict__ boff, uint32_t nb, uint32_t total,
                                       uint32_t key_bits, uint64_t *__restrict__ keys, const typename P::params_t prm)
{
    using T = typename P::tuple_t;
    const uint64_t mask = key_bits >= 64 ? ~0ull : ((1ull << key_bits) - 1ull);
    for (uint32_t gi = blockIdx.x * blockDim.x + threadIdx.x; gi < total; gi += gridDim.x * blockDim.x) {
        const uint32_t b = batch_of(boff, nb, gi);
        const T *t = reinterpret_cast<const T *>(batches[b].tuples + static_cast<size_t>(gi - boff[b]) * sizeof(T));
        keys[gi] = (key_bits >= 64 ? 0ull : (static_cast<uint64_t>(b) << key_bits)) | (key_word0(key_words<P>(*t, prm)) & mask);
    }
}

// ---- Reduce_GPU over keys that are not integers: the keys are first replaced by their dense rank in the sort order ----------------
// lo[gi] / hi[gi] = the order words (KeyCodec::order) of element gi's key; hi only for two-word keys. `tuples` is the one batch when
// `batches` is null.
template <class P>
__global__ void k_key_order_words(const DevBatch *__restrict__ batches, const uint32_t *__restrict__ boff, uint32_t nb,
                                  const unsigned char *__restrict__ tuples, uint32_t total, uint64_t *__restrict__ lo, uint64_t *__restrict__ hi,
                                  const typename P::params_t prm)
{
    using T = typename P::tuple_t;
    for (uint32_t gi = blockIdx.x * blockDim.x + threadIdx.x; gi < total; gi += gridDim.x * blockDim.x) {
        const unsigned char *src = tuples + static_cast<size_t>(gi) * sizeof(T);
        if (batches != nullptr) { const uint32_t b = batch_of(boff, nb, gi); src = batches[b].tuples + static_cast<size_t>(gi - boff[b]) * sizeof(T); }
        const key_words_t<P> w = key_codec<P>::order(key_words<P>(*reinterpret_cast<const T *>(src), prm));
        if constexpr (key_codec<P>::words == 2) { lo[gi] = w.lo; hi[gi] = w.hi; } else lo[gi] = w;
    }
}

// out[i] = in[perm[i]]
static __global__ void k_gather_u64(const uint64_t *__restrict__ in, const uint32_t *__restrict__ perm, uint32_t n, uint64_t *__restrict__ out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = in[perm[i]];
}
// out[i] = a[b[i]]
static __global__ void k_compose_perm(const uint32_t *__restrict__ a, const uint32_t *__restrict__ b, uint32_t n, uint32_t *__restrict__ out)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = a[b[i]];
}
// head[i] = 1 when sorted position i (element perm[i]) has other order words than its predecessor (hi may be null: one word)
__device__ __forceinline__ bool rank_head(const uint64_t *__restrict__ lo, const uint64_t *__restrict__ hi, const uint32_t *__restrict__ perm, uint32_t i)
{
    if (i == 0) return true;
    const uint32_t a = perm[i], b = perm[i - 1];
    return lo[a] != lo[b] || (hi != nullptr && hi[a] != hi[b]);
}
static __global__ void k_rank_heads(const uint64_t *__restrict__ lo, const uint64_t *__restrict__ hi, const uint32_t *__restrict__ perm, uint32_t n,
                                    uint32_t *__restrict__ head)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) head[i] = rank_head(lo, hi, perm, i) ? 1u : 0u;
}
// after the exclusive scan of head[]: keys[e] = (batch of e << 32) | dense rank of e's key (boff null: the rank alone)
static __global__ void k_rank_scatter(const uint64_t *__restrict__ lo, const uint64_t *__restrict__ hi, const uint32_t *__restrict__ perm,
                                      const uint32_t *__restrict__ head_scan, uint32_t n, const uint32_t *__restrict__ boff, uint32_t nb,
                                      uint64_t *__restrict__ keys)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t e = perm[i];
        const uint64_t rank = head_scan[i] - (rank_head(lo, hi, perm, i) ? 0u : 1u);
        keys[e] = (boff != nullptr ? (static_cast<uint64_t>(batch_of(boff, nb, e)) << 32) : 0ull) | rank;
    }
}

constexpr uint32_t SEGT = 2048; // sorted positions per tile of the head count / finish kernels (256 threads x 8)

// counts[tile] = segment heads (sorted position whose key differs from its predecessor) in the tile
static __global__ void __launch_bounds__(256) k_head_tile_counts(const uint64_t *__restrict__ skeys, uint32_t n, uint32_t *__restrict__ counts)
{
    __shared__ uint32_t wsum[8];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, base = blockIdx.x * SEGT;
    uint32_t c = 0;
#pragma unroll
    for (uint32_t r = 0; r < SEGT / 256; r++) {
        const uint32_t i = base + r * 256 + tid;
        if (i < n && (i == 0 || skeys[i] != skeys[i - 1])) c++;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL, c, o);
    if (lane == 0) wsum[warp] = c;
    __syncthreads();
    if (tid == 0) { uint32_t t = 0; for (int w = 0; w < 8; w++) t += wsum[w]; counts[blockIdx.x] = t; }
}

// tile_base = exclusive scan of the tile counts. seg_begin[k] = first sorted position of the k-th segment (global numbering),
// first_seg[b] = number of the first segment of batch b (0xffffffff when the batch has none), *n_segs = total, seg_begin[total] = n
static __global__ void __launch_bounds__(256) k_seg_finish_batches(const uint64_t *__restrict__ skeys, uint32_t n, uint32_t key_bits,
                                                            const uint32_t *__restrict__ tile_base, uint32_t *__restrict__ seg_begin,
                                                            uint32_t *__restrict__ first_seg, uint32_t *__restrict__ n_segs)
{
    __shared__ uint32_t wsum[8];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t first = blockIdx.x * SEGT + tid * (SEGT / 256); // thread t owns 8 consecutive positions
    bool head[SEGT / 256];
    uint32_t mine = 0;
#pragma unroll
    for (uint32_t r = 0; r < SEGT / 256; r++) {
        const uint32_t i = first + r;
        head[r] = i < n && (i == 0 || skeys[i] != skeys[i - 1]);
        mine += head[r] ? 1u : 0u;
    }
    uint32_t incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    uint32_t k = tile_base[blockIdx.x] + incl - mine;
    for (uint32_t w = 0; w < warp; w++) k += wsum[w];
#pragma unroll
    for (uint32_t r = 0; r < SEGT / 256; r++) {
        const uint32_t i = first + r;
        if (head[r]) {
            seg_begin[k] = i;
            const uint64_t b = key_bits >= 64 ? 0ull : (skeys[i] >> key_bits);
            if (i == 0 || (key_bits < 64 && (skeys[i - 1] >> key_bits) != b)) first_seg[b] = k;
            k++;
        }
        if (i == n - 1) { *n_segs = k; seg_begin[k] = n; }
    }
}

// n_out[b] = segments of batch b (first_seg[] is ascending over the batches that have segments)
static __global__ void k_batch_seg_counts(const uint32_t *__restrict__ first_seg, uint32_t nb, const uint32_t *__restrict__ n_segs,
                                          const DevBatch *__restrict__ batches)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        uint32_t next = *n_segs;
        for (uint32_t b = nb; b-- > 0;) {
            uint32_t c = 0;
            if (first_seg[b] != 0xffffffffu) { c = next - first_seg[b]; next = first_seg[b]; }
            if (batches[b].n_out != nullptr) *batches[b].n_out = c;
        }
    }
}

constexpr uint32_t RB_LONG = 48; // segments longer than this are folded by a warp (k_reduce_segments_batches), the others by one thread

// one THREAD per segment (most keys of a batch occur once or twice): sequential fold, 4 tuples in flight; long segments
// are put on a list for the warp kernel
template <class P>
__global__ void __launch_bounds__(128) k_reduce_segments_batches_short(const DevBatch *__restrict__ batches, const uint32_t *__restrict__ boff,
                                                                       const uint64_t *__restrict__ skeys, const uint32_t *__restrict__ sidx,
                                                                       const uint32_t *__restrict__ seg_begin, const uint32_t *__restrict__ first_seg,
                                                                       const uint32_t *__restrict__ n_segs, uint32_t key_bits,
                                                                       uint32_t *__restrict__ long_list, uint32_t *__restrict__ n_long,
                                                                       const typename P::params_t prm)
{
    using T = typename P::tuple_t;
    const uint32_t nk = *n_segs;
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < nk; k += gridDim.x * blockDim.x) {
        const uint32_t sb = seg_begin[k], se = seg_begin[k + 1];
        if (se - sb > RB_LONG) { long_list[atomicAdd(n_long, 1u)] = k; continue; }
        const uint32_t b = key_bits >= 64 ? 0u : static_cast<uint32_t>(skeys[sb] >> key_bits);
        const unsigned char *tuples = batches[b].tuples;
        const uint64_t *ts = batches[b].ts;
        const uint32_t base = boff[b];
        alignas(16) T acc; uint64_t mts = 0;
        {
            const uint32_t i = sidx[sb] - base;
            ld_rec<T>(tuples + static_cast<size_t>(i) * sizeof(T), acc);
            mts = ts ? ts[i] : 0;
        }
        for (uint32_t j = sb + 1; j < se; j += 2) { // two tuples in flight
            const uint32_t i0 = sidx[j] - base, i1 = (j + 1 < se) ? sidx[j + 1] - base : i0;
            alignas(16) T t0, t1;
            ld_rec<T>(tuples + static_cast<size_t>(i0) * sizeof(T), t0);
            if (j + 1 < se) ld_rec<T>(tuples + static_cast<size_t>(i1) * sizeof(T), t1);
            const uint64_t s0 = ts ? ts[i0] : 0, s1 = (ts && j + 1 < se) ? ts[i1] : 0;
            acc = P::reduce(acc, t0, prm); mts = mts < s0 ? s0 : mts;
            if (j + 1 < se) { acc = P::reduce(acc, t1, prm); mts = mts < s1 ? s1 : mts; }
        }
        const uint32_t o = k - first_seg[b];
        st_rec<T>(batches[b].out + static_cast<size_t>(o) * sizeof(T), acc);
        if (batches[b].ts_out) batches[b].ts_out[o] = mts;
    }
}

// one warp per long segment (list filled by the kernel above; long_list == nullptr: every segment): ordered fold with
// P::reduce, ts = max; output = the batch's out buffers
template <class P>
__global__ void __launch_bounds__(256) k_reduce_segments_batches(const DevBatch *__restrict__ batches, const uint32_t *__restrict__ boff,
                                                                 const uint64_t *__restrict__ skeys, const uint32_t *__restrict__ sidx,
                                                                 const uint32_t *__restrict__ seg_begin, const uint32_t *__restrict__ first_seg,
                                                                 const uint32_t *__restrict__ n_segs, uint32_t key_bits,
                                                                 const uint32_t *__restrict__ long_list, const uint32_t *__restrict__ n_long,
                                                                 const typename P::params_t prm)
{
    using T = typename P::tuple_t;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t nk = long_list ? *n_long : *n_segs;
    for (uint32_t kk = gwarp; kk < nk; kk += nwarps) {
        const uint32_t k = long_list ? long_list[kk] : kk;
        const uint32_t sb = seg_begin[k], se = seg_begin[k + 1];
        const uint32_t b = key_bits >= 64 ? 0u : static_cast<uint32_t>(skeys[sb] >> key_bits);
        const DevBatch bt = batches[b];
        const uint32_t base = boff[b];
        alignas(16) T acc; uint64_t mts = 0; bool have = false;
        for (uint32_t j = sb; j < se; j += 32) {
            const uint32_t take = min(32u, se - j);
            alignas(16) T t; uint64_t tt = 0;
            if (lane < take) {
                const uint32_t i = sidx[j + lane] - base;
                ld_rec<T>(bt.tuples + static_cast<size_t>(i) * sizeof(T), t);
                tt = bt.ts ? bt.ts[i] : 0;
            }
#pragma unroll
            for (uint32_t o = 1; o < 32; o <<= 1) {
                const T other = shfl_down_rec<T>(t, o);
                const uint64_t ots = __shfl_down_sync(FULL, tt, o);
                if (lane + o < take) { t = P::reduce(t, other, prm); tt = tt < ots ? ots : tt; }
            }
            t = shfl_rec<T>(t, 0); tt = __shfl_sync(FULL, tt, 0);
            if (!have) { acc = t; mts = tt; have = true; }
            else { acc = P::reduce(acc, t, prm); mts = mts < tt ? tt : mts; }
        }
        if (lane == 0) {
            const uint32_t o = k - first_seg[b];
            st_rec<T>(bt.out + static_cast<size_t>(o) * sizeof(T), acc);
            if (bt.ts_out) bt.ts_out[o] = mts;
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// Time-based windows, front end (Ffat_Replica_GPU::process_batch_tb, wf/ffat_replica_gpu.hpp:870-1019; PendingPanes_Queue
// :263-420; Aggregate_Panes_Kernel :214-260). Per input batch: lift + (slot, pane) composite key -> stable sort ->
// per-(key, pane) partial in arrival order -> merged into the key's ring of pending panes -> for every key present in the
// batch, the panes of the groups the watermark has completed are popped, in pane order, into an array of lifted records
// that the count-based back end (a second handle over the "lifted" program, window / slide in panes) consumes as one
// batch: it fires exactly one group of Nb windows per popped group, with ts = the batch watermark.
// ------------------------------------------------------------------------------------------------------

struct TbDev {
    uint64_t pane_len, Bp, group;      // pane length (timestamp units), panes of the first group, panes of every further group
    uint32_t capq;                     // ring capacity per key (panes)
    uint32_t kbits;                    // this batch: sort key = (slot << kbits) | (pane - first pending pane of the key); 2^kbits - 1 = late
                                       // pane (already consumed), slot >= max_keys = no tuple (filtered out)
    uint64_t *first;                   // id of the first pending pane of every key
    uint32_t *num, *num_new;           // pending panes (before / after this batch)
    uint64_t *trig;                    // pane_id_triggerer
    uint32_t *done;                    // firstWinDone
    unsigned char *ring;               // max_keys x capq results, pane p of key s at (s * capq + p % capq)
    uint32_t *present, *n_present;     // slots of the keys of this batch
    uint32_t *cnt;                     // panes to pop per present key -> exclusive offsets
    uint32_t *ignored;                 // tuples older than the first incomplete pane (statistic)
    uint32_t *need;                    // ring capacity this batch needs: max over its tuples of pane - first pending pane + 2
    uint32_t *err;                     // bit 2: ring overflow / pane id out of range
};

template <class P>
__global__ void k_tb_lift(const unsigned char *__restrict__ tuples, const uint64_t *__restrict__ ts, uint32_t n, const FfatDev ff,
                          const TbDev tb, uint64_t first_incomplete, unsigned char *__restrict__ lifted, uint64_t *__restrict__ ckeys,
                          const typename P::params_t prm)
{
    using T = typename P::tuple_t;
    using R = typename P::result_t;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        alignas(16) T t;
        ld_rec<T>(tuples + static_cast<size_t>(i) * sizeof(T), t);
        P::map(t, prm);
        uint64_t ck = ~0ull;
        if (P::filter(t, prm)) {
            alignas(16) R r;
            P::lift(t, r, prm);
            st_rec<R>(lifted + static_cast<size_t>(i) * sizeof(R), r);
            const uint32_t slot = slot_of_key(ff, key_words<P>(t, prm));
            const uint64_t pane = ts[i] / tb.pane_len;                 // Lifting_Kernel_TB_Keyed :164
            if (pane < first_incomplete) atomicAdd(tb.ignored, 1u);    // :165-167
            if (slot != INVALID_SLOT) { // raw key: slot, pane relative to the key's first pending pane (0xffffffff: older = late)
                const uint64_t f0 = tb.first[slot];
                uint32_t rel = 0xffffffffu;
                if (pane >= f0) {
                    if (pane - f0 >= 0xfffffff0ull) atomicOr(tb.err, 4u);
                    else { rel = static_cast<uint32_t>(pane - f0); atomicMax(tb.need, rel + 2u); } // push_panes :367-372
                }
                ck = (static_cast<uint64_t>(slot) << 32) | rel;
            }
        }
        ckeys[i] = ck;
    }
}

// sort keys of the batch once the number of pane bits it needs is known: (slot << kbits) | relative pane
static __global__ void k_tb_pack(uint64_t *__restrict__ ckeys, uint32_t n, uint32_t kbits, uint32_t invalid_slot)
{
    const uint64_t late = (1ull << kbits) - 1ull;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint64_t c = ckeys[i];
        if (c == ~0ull) { ckeys[i] = static_cast<uint64_t>(invalid_slot) << kbits; continue; }
        const uint32_t rel = static_cast<uint32_t>(c);
        ckeys[i] = ((c >> 32) << kbits) | (rel == 0xffffffffu ? late : static_cast<uint64_t>(rel));
    }
}

// partial of every (key, pane) of the batch: fold of the lifted results in arrival order (thrust::reduce_by_key :925-935)
template <class P>
__global__ void k_tb_reduce(const unsigned char *__restrict__ lifted, const uint64_t *__restrict__ skeys, const uint32_t *__restrict__ sidx,
                            const uint32_t *__restrict__ seg_begin, const uint32_t *__restrict__ n_segs, unsigned char *__restrict__ part,
                            uint32_t kbits, uint32_t max_keys, const typename P::params_t prm)
{
    using R = typename P::result_t;
    const uint32_t nk = *n_segs;
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < nk; k += gridDim.x * blockDim.x) {
        const uint32_t sb = seg_begin[k], se = seg_begin[k + 1];
        if ((skeys[sb] >> kbits) >= max_keys || (skeys[sb] & ((1ull << kbits) - 1ull)) == (1ull << kbits) - 1ull) continue; // no tuple / late pane
        alignas(16) R acc;
        ld_rec<R>(lifted + static_cast<size_t>(sidx[sb]) * sizeof(R), acc);
        for (uint32_t j = sb + 1; j < se; j++) {
            alignas(16) R r;
            ld_rec<R>(lifted + static_cast<size_t>(sidx[j]) * sizeof(R), r);
            P::comb(acc, r, acc, prm);
        }
        st_rec<R>(part + static_cast<size_t>(k) * sizeof(R), acc);
    }
}

// partials (ascending slot, ascending pane) -> the keys' rings of pending panes; the last partial of a key records the
// new number of pending panes and lists the key as present
template <class P>
__global__ void k_tb_merge(const uint64_t *__restrict__ skeys, const uint32_t *__restrict__ seg_begin, const uint32_t *__restrict__ n_segs,
                           const unsigned char *__restrict__ part, const FfatDev ff, const TbDev tb, const typename P::params_t prm)
{
    using R = typename P::result_t;
    const uint32_t nk = *n_segs;
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < nk; k += gridDim.x * blockDim.x) {
        const uint64_t ck = skeys[seg_begin[k]];
        const uint64_t relmask = (1ull << tb.kbits) - 1ull;
        if ((ck >> tb.kbits) >= ff.max_keys) continue;                // filtered tuples
        const uint32_t slot = static_cast<uint32_t>(ck >> tb.kbits);
        const uint64_t first_id = tb.first[slot];
        const bool late = (ck & relmask) == relmask;                  // pane already consumed (:232-234)
        const uint64_t pane = late ? 0 : first_id + (ck & relmask);
        const uint32_t num = tb.num[slot];
        const uint64_t have_end = first_id + num;                      // first pane id that is not in the ring yet
        unsigned char *ring = tb.ring + static_cast<size_t>(slot) * tb.capq * sizeof(R);
        const uint64_t ckn = (k + 1 < nk) ? skeys[seg_begin[k + 1]] : ~0ull;
        const bool last_of_key = (ckn >> tb.kbits) != slot; // (ckn = ~0 past the end: never a slot)
        bool stored = false;
        if (!late) {
            if (pane - first_id >= tb.capq) atomicOr(tb.err, 4u);
            else {
                alignas(16) R v;
                ld_rec<R>(part + static_cast<size_t>(k) * sizeof(R), v);
                unsigned char *dst = ring + (pane % tb.capq) * sizeof(R);
                if (pane < have_end) { alignas(16) R old; ld_rec<R>(dst, old); P::comb(old, v, old, prm); st_rec<R>(dst, old); } // :236
                else {
                    st_rec<R>(dst, v);
                    uint64_t lower = have_end;                          // missing panes below this one become empty panes (:239-257)
                    if (k > 0) {
                        const uint64_t ckp = skeys[seg_begin[k - 1]];
                        if ((ckp >> tb.kbits) == slot && first_id + (ckp & relmask) + 1 > lower) lower = first_id + (ckp & relmask) + 1;
                    }
                    const typename P::key_t key = key_codec<P>::decode(key_of_slot<P>(ff, slot));
                    for (uint64_t m = lower; m < pane; m++) {
                        alignas(16) R e = P::make_result(key, 0, prm);
                        st_rec<R>(ring + (m % tb.capq) * sizeof(R), e);
                    }
                }
                stored = true;
            }
        }
        if (last_of_key) {
            uint32_t nn = num;
            if (stored && pane >= have_end) nn = static_cast<uint32_t>(pane - first_id + 1);
            tb.num_new[slot] = nn;
            tb.present[atomicAdd(tb.n_present, 1u)] = slot;
        }
    }
}

// the rings grow (PendingPanes_Queue::resize :326-357): pending pane p of key s moves from p % old_cap to p % new_cap
static __global__ void k_tb_ring_resize(const TbDev tb, const unsigned char *__restrict__ old_ring, uint32_t old_cap, unsigned char *__restrict__ new_ring,
                                        uint32_t new_cap, uint32_t max_keys, uint32_t rbytes)
{
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < max_keys; s += gridDim.x * blockDim.x) {
        const uint64_t f0 = tb.first[s];
        const uint32_t num = tb.num[s];
        for (uint32_t j = 0; j < num; j++) {
            const uint64_t *src = reinterpret_cast<const uint64_t *>(old_ring + (static_cast<size_t>(s) * old_cap + (f0 + j) % old_cap) * rbytes);
            uint64_t *dst = reinterpret_cast<uint64_t *>(new_ring + (static_cast<size_t>(s) * new_cap + (f0 + j) % new_cap) * rbytes);
            for (uint32_t q = 0; q < rbytes / 8; q++) dst[q] = src[q];
        }
    }
}

// panes every present key pops now: groups completed by the watermark (process_wins_tb :1029-1046), first Bp then `group` each
static __global__ void k_tb_pop_count(const TbDev tb, uint64_t first_incomplete)
{
    const uint32_t np = *tb.n_present;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < np; i += gridDim.x * blockDim.x) {
        const uint32_t slot = tb.present[i];
        uint64_t trig = tb.trig[slot];
        bool done = tb.done[slot] != 0;
        uint64_t c = 0;
        while (trig < first_incomplete) { c += done ? tb.group : tb.Bp; done = true; trig += tb.group; }
        tb.cnt[i] = static_cast<uint32_t>(c > 0x7fffffffull ? 0x7fffffffull : c);
    }
}

// exclusive scan of the pop counts of the *n_present keys of the batch (one CTA), total to *total_out
static __global__ void __launch_bounds__(1024) k_tb_scan_present(uint32_t *__restrict__ cnt, const uint32_t *__restrict__ n_present, uint32_t *__restrict__ total_out)
{
    __shared__ uint32_t warp_sums[32];
    const uint32_t total = *n_present;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t per = (total + 1023) / 1024;
    const uint32_t begin = min(tid * per, total), end = min(begin + per, total);
    uint32_t sum = 0;
    for (uint32_t i = begin; i < end; i++) sum += cnt[i];
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = warp_sums[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, wi, o); if (lane >= static_cast<uint32_t>(o)) wi += v; }
        warp_sums[lane] = wi - w;
        if (lane == 31) *total_out = wi;
    }
    __syncthreads();
    uint32_t run = warp_sums[warp] + incl - sum;
    for (uint32_t i = begin; i < end; i++) { const uint32_t v = cnt[i]; cnt[i] = run; run += v; }
}

template <class P>
__global__ void k_tb_pop_write(const FfatDev ff, const TbDev tb, uint64_t first_incomplete, const uint32_t *__restrict__ offs,
                               unsigned char *__restrict__ popped, uint32_t *__restrict__ popped_slots, uint32_t popped_cap,
                               const typename P::params_t prm)
{
    using R = typename P::result_t;
    const uint32_t np = *tb.n_present;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < np; i += gridDim.x * blockDim.x) {
        const uint32_t slot = tb.present[i];
        uint64_t trig = tb.trig[slot], first_id = tb.first[slot];
        uint32_t num = tb.num_new[slot];
        bool done = tb.done[slot] != 0;
        const typename P::key_t key = key_codec<P>::decode(key_of_slot<P>(ff, slot));
        const unsigned char *ring = tb.ring + static_cast<size_t>(slot) * tb.capq * sizeof(R);
        uint32_t w = offs[i];
        while (trig < first_incomplete) {
            const uint64_t need = done ? tb.group : tb.Bp;
            for (uint64_t m = 0; m < need; m++, w++) {                  // pop_and_add :394-415; a missing pane is an empty pane
                alignas(16) R v;
                if (m < num) ld_rec<R>(ring + ((first_id + m) % tb.capq) * sizeof(R), v);
                else v = P::make_result(key, 0, prm);
                if (w < popped_cap) { st_rec<R>(popped + static_cast<size_t>(w) * sizeof(R), v); popped_slots[w] = slot; }
            }
            first_id += need; num = num > need ? static_cast<uint32_t>(num - need) : 0u;
            done = true; trig += tb.group;
        }
        tb.first[slot] = first_id; tb.num[slot] = num; tb.trig[slot] = trig; tb.done[slot] = done ? 1u : 0u;
    }
}

// ------------------------------------------------------------------------------------------------------
// Keyed-stateful Map_GPU / Filter_GPU (wf/map_gpu.hpp:80-102, :212-299; wf/filter_gpu.hpp:91-117, :247-355): the same
// shape as the window update -- slots of the segment's tuples, ONE wide partition pass into 1024 buckets of consecutive
// slots, one CTA per bucket splits its items by key (stable) and ONE THREAD per key walks its run in arrival order with
// the key's state in registers (above 65536 keys: a full sort by slot and k_ks_apply_runs). Stateful filter: keep flags,
// then a stable per-batch compaction. Keyed-stateful FlatMap_GPU: two walks over the same partition -- KS_FM_COUNT runs the
// functor with a counting Shipper and keeps neither records nor state, a per-batch scan of the counts gives every tuple its
// first record's index (k_fm_offsets), and KS_FM_EMIT runs it again from the same states, writing the records in place.
// ------------------------------------------------------------------------------------------------------
enum { KS_MAP = 0, KS_FILTER = 1, KS_FM_COUNT = 2, KS_FM_EMIT = 3 };
// the flatmap walks' arrays: records kept per position (min(pushes, m); written by KS_FM_COUNT), the record index of every
// position's first record within its batch (read by KS_FM_EMIT), and the word that sums the pushes dropped beyond m
struct KsFlatMap { uint32_t *cnt; const uint32_t *off; uint32_t m; uint32_t *drop; };

// one tuple of a key's run (global position gi) with the key's state `st`
template <class P, int KM>
__device__ __forceinline__ void ks_visit(uint32_t gi, const DevBatch *__restrict__ batches, const uint32_t *__restrict__ boff, uint32_t nb,
                                         typename P::state_t &st, unsigned char *__restrict__ keep, const KsFlatMap fm, uint32_t &excess,
                                         const typename P::params_t &prm)
{
    using T = typename P::tuple_t;
    const uint32_t b = batch_of(boff, nb, gi);
    unsigned char *tp = const_cast<unsigned char *>(batches[b].tuples) + static_cast<size_t>(gi - boff[b]) * sizeof(T);
    if constexpr (KM == KS_MAP || KM == KS_FILTER) {
        alignas(16) T t;
        ld_rec<T>(tp, t);
        if constexpr (KM == KS_FILTER) keep[gi] = P::filter_stateful(t, st, prm) ? 1 : 0;
        else P::map_stateful(t, st, prm);
        st_rec<T>(tp, t);
    } else {
        using R = typename P::result_t;
        if constexpr (KM == KS_FM_COUNT) {
            alignas(16) T t;
            ld_rec<T>(tp, t);
            Shipper<R> sh(nullptr, nullptr, 0, fm.m);
            P::flatmap_stateful(t, sh, st, prm);
            const uint32_t c = sh.pushes();
            fm.cnt[gi] = min(c, fm.m);
            excess += c > fm.m ? c - fm.m : 0u;
        } else {
            const uint32_t o = fm.off[gi]; // (issued with the tuple's load: no longer chain of dependent loads)
            const uint32_t li = gi - boff[b];
            unsigned char *out = batches[b].out;
            uint64_t *ts_out = batches[b].ts_out;
            alignas(16) T t;
            ld_rec<T>(tp, t);
            const uint64_t ts = ts_out != nullptr ? batches[b].ts[li] : 0;
            Shipper<R> sh(out + static_cast<size_t>(o) * sizeof(R), ts_out != nullptr ? ts_out + o : nullptr, ts, fm.m);
            P::flatmap_stateful(t, sh, st, prm);
        }
    }
}
template <class P>
__global__ void k_ks_slots(const DevBatch *__restrict__ batches, const uint32_t *__restrict__ boff, uint32_t nb, uint32_t total, const FfatDev ff,
                           uint32_t *__restrict__ slots, const typename P::params_t prm)
{
    using T = typename P::tuple_t;
    for (uint32_t gi = blockIdx.x * blockDim.x + threadIdx.x; gi < total; gi += gridDim.x * blockDim.x) {
        const uint32_t b = batch_of(boff, nb, gi);
        const T *t = reinterpret_cast<const T *>(batches[b].tuples + static_cast<size_t>(gi - boff[b]) * sizeof(T));
        slots[gi] = slot_of_key(ff, key_words<P>(*t, prm));
    }
}

constexpr uint32_t KS_KEYS = 64, KS_THREADS = 128, KS_IT = 18, KS_CAP = KS_THREADS * KS_IT;

template <class P, int KM>
__global__ void __launch_bounds__(KS_THREADS) k_ks_apply(const FfatDev ff, const DevBatch *__restrict__ batches, const uint32_t *__restrict__ boff,
                                                         uint32_t nb, const uint32_t *__restrict__ bk_slots, const uint32_t *__restrict__ bk_pos,
                                                         const uint32_t *__restrict__ digit_counts, uint32_t shift, unsigned char *__restrict__ states,
                                                         unsigned char *__restrict__ keep, const typename P::params_t prm, const KsFlatMap fm)
{
    using S = typename P::state_t;
    constexpr uint32_t NW = KS_THREADS / 32, DPT = OSW_DIGITS / KS_THREADS, HS = KS_THREADS + 2;
    __shared__ uint32_t s_idx[KS_CAP];                 // positions (global tuple index in the segment), key-major
    __shared__ uint16_t hist[KS_KEYS][HS];             // private key counts of every thread -> exclusive over the threads
    __shared__ uint32_t htot[2][KS_KEYS], kcnt[KS_KEYS], koff[KS_KEYS];
    __shared__ uint32_t misc[NW], s_boff[2];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, bucket = blockIdx.x;
    const uint32_t kpc = min(KS_KEYS, 1u << shift), key_lo = bucket << shift;
    { // bucket range = exclusive scan of the pass histogram (as in k_ffat_update_buckets)
        uint32_t cc[DPT];
#pragma unroll
        for (uint32_t q = 0; q < DPT / 4; q++) {
            const uint4 v = reinterpret_cast<const uint4 *>(digit_counts)[tid * (DPT / 4) + q];
            cc[4 * q] = v.x; cc[4 * q + 1] = v.y; cc[4 * q + 2] = v.z; cc[4 * q + 3] = v.w;
        }
        uint32_t sum = 0;
#pragma unroll
        for (uint32_t q = 0; q < DPT; q++) sum += cc[q];
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
        if (lane == 31) misc[warp] = incl;
        __syncthreads();
        if (tid == bucket / DPT) {
            uint32_t base = incl - sum;
            for (uint32_t w = 0; w < warp; w++) base += misc[w];
            uint32_t own = 0;
#pragma unroll
            for (uint32_t q = 0; q < DPT; q++) { if (q < bucket % DPT) base += cc[q]; if (q == bucket % DPT) own = cc[q]; }
            s_boff[0] = base; s_boff[1] = base + own;
        }
        __syncthreads();
    }
    uint32_t cursor = s_boff[0];
    const uint32_t bend = s_boff[1];
    if (cursor == bend) return;
    // the key's state stays in registers across the chunks of the bucket
    alignas(8) S st;
    const bool has_key = tid < kpc && key_lo + tid < ff.max_keys;
    bool touched = false;
    uint32_t excess = 0; // KS_FM_COUNT: pushes of this thread's key dropped beyond m
    if (has_key) st = *reinterpret_cast<const S *>(states + static_cast<size_t>(key_lo + tid) * sizeof(S));
    while (cursor < bend) {
        const uint32_t nsel = min(KS_CAP, bend - cursor);
        uint32_t ek[KS_IT], ep[KS_IT];
#pragma unroll
        for (uint32_t r = 0; r < KS_IT; r++) {
            const uint32_t i = tid * KS_IT + r;
            ek[r] = KS_KEYS; ep[r] = 0;
            if (i < nsel) {
                const uint32_t lk = bk_slots[cursor + i] - key_lo; // slots outside the bucket's keys (invalid slots) are dropped
                ep[r] = bk_pos[cursor + i];
                if (lk < kpc) ek[r] = lk;
            }
        }
        {
            uint32_t *z = reinterpret_cast<uint32_t *>(&hist[0][0]);
            for (uint32_t i = tid; i < KS_KEYS * HS / 2; i += KS_THREADS) z[i] = 0;
        }
        __syncthreads();
#pragma unroll
        for (uint32_t r = 0; r < KS_IT; r++) if (ek[r] < KS_KEYS) hist[ek[r]][tid]++;
        __syncthreads();
        {
            const uint32_t k = tid & 63u, half = tid >> 6;
            uint16_t *row = &hist[k][half * 64];
            uint32_t run = 0;
#pragma unroll 16
            for (uint32_t i = 0; i < 64; i++) { const uint32_t c = row[i]; row[i] = static_cast<uint16_t>(run); run += c; }
            htot[half][k] = run;
        }
        __syncthreads();
        if (warp == 0) {
            const uint32_t a0 = htot[0][lane] + htot[1][lane], a1 = htot[0][lane + 32] + htot[1][lane + 32];
            uint32_t i0 = a0, i1 = a1;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v0 = __shfl_up_sync(FULL, i0, o), v1 = __shfl_up_sync(FULL, i1, o);
                if (lane >= static_cast<uint32_t>(o)) { i0 += v0; i1 += v1; }
            }
            const uint32_t t0 = __shfl_sync(FULL, i0, 31);
            kcnt[lane] = a0; kcnt[lane + 32] = a1;
            koff[lane] = i0 - a0; koff[lane + 32] = t0 + i1 - a1;
        }
        __syncthreads();
        {
            const uint32_t hb = tid >> 6;
#pragma unroll
            for (uint32_t r = 0; r < KS_IT; r++) {
                const uint32_t k = ek[r];
                if (k < KS_KEYS) {
                    const uint32_t rank = hist[k][tid];
                    hist[k][tid] = static_cast<uint16_t>(rank + 1);
                    s_idx[koff[k] + (hb ? htot[0][k] : 0u) + rank] = ep[r];
                }
            }
        }
        __syncthreads();
        if (has_key) { // one thread per key: the run in arrival order
            const uint32_t m = kcnt[tid], off = koff[tid];
            for (uint32_t j = 0; j < m; j++) ks_visit<P, KM>(s_idx[off + j], batches, boff, nb, st, keep, fm, excess, prm);
            touched |= m != 0;
        }
        cursor += nsel;
        __syncthreads();
    }
    if constexpr (KM == KS_FM_COUNT) { // the count walk keeps no state; one atomic per warp for the drops
        const uint32_t w = __reduce_add_sync(FULL, excess);
        if (lane == 0 && w != 0) atomicAdd(fm.drop, w);
    } else if (has_key && touched) *reinterpret_cast<S *>(states + static_cast<size_t>(key_lo + tid) * sizeof(S)) = st;
}

// More than 65536 keys: the (slot, arrival position) pairs come fully sorted by slot (stable onesweep passes with 8·passes > log2
// capacity, so INVALID_SLOT sorts behind every real slot). The thread whose item starts a run -- its slot differs from its
// predecessor's -- walks that run in arrival order with the key's state in registers: work follows the call's items, not the capacity.
template <class P, int KM>
__global__ void __launch_bounds__(256) k_ks_apply_runs(const FfatDev ff, const DevBatch *__restrict__ batches, const uint32_t *__restrict__ boff,
                                                       uint32_t nb, uint32_t n, const uint32_t *__restrict__ sorted_slots,
                                                       const uint32_t *__restrict__ sorted_pos, unsigned char *__restrict__ states,
                                                       unsigned char *__restrict__ keep, const typename P::params_t prm, const KsFlatMap fm)
{
    using S = typename P::state_t;
    uint32_t excess = 0; // KS_FM_COUNT: pushes of this thread's runs dropped beyond m
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t slot = sorted_slots[i];
        if (slot >= ff.max_keys || (i > 0 && sorted_slots[i - 1] == slot)) continue; // (no slot: the item is not applied)
        S *sp = reinterpret_cast<S *>(states + static_cast<size_t>(slot) * sizeof(S));
        alignas(8) S st = *sp;
        uint32_t j = i;
        do ks_visit<P, KM>(sorted_pos[j], batches, boff, nb, st, keep, fm, excess, prm);
        while (++j < n && sorted_slots[j] == slot);
        if constexpr (KM != KS_FM_COUNT) *sp = st; // (the count walk keeps no state)
    }
    if constexpr (KM == KS_FM_COUNT) {
        const uint32_t w = __reduce_add_sync(FULL, excess);
        if ((threadIdx.x & 31u) == 0 && w != 0) atomicAdd(fm.drop, w);
    }
}

// stable per-batch compaction by the keep flags of a stateful filter (E = unsigned char): tile counts, scan, scatter. The same
// tile counts and batch starts over the kept record counts of a stateful flatmap (E = uint32_t) give its per-batch offsets.
template <class E> __device__ __forceinline__ uint32_t flag_count(E v) { if constexpr (sizeof(E) == 1) return v ? 1u : 0u; else return v; }

template <class E>
static __global__ void __launch_bounds__(256) k_flag_tile_counts(const E *__restrict__ keep, uint32_t n, uint32_t *__restrict__ counts)
{
    __shared__ uint32_t wsum[8];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, base = blockIdx.x * SEGT;
    uint32_t c = 0;
#pragma unroll
    for (uint32_t r = 0; r < SEGT / 256; r++) {
        const uint32_t i = base + r * 256 + tid;
        if constexpr (sizeof(E) == 1) { if (i < n && keep[i]) c++; } else { if (i < n) c += keep[i]; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL, c, o);
    if (lane == 0) wsum[warp] = c;
    __syncthreads();
    if (tid == 0) { uint32_t t = 0; for (int w = 0; w < 8; w++) t += wsum[w]; counts[blockIdx.x] = t; }
}

// rank_start[b] = survivors before batch b (global rank of its first tuple); n_out of every batch
template <class E>
static __global__ void k_flag_batch_starts(const E *__restrict__ keep, const uint32_t *__restrict__ tile_base, const uint32_t *__restrict__ boff,
                                           uint32_t nb, uint32_t n, uint32_t *__restrict__ rank_start, const DevBatch *__restrict__ batches)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b > nb) return;
    const uint32_t gi = boff[b]; // boff[nb] = n
    uint32_t r;
    if (gi >= n) { // total survivors
        const uint32_t lt = (n - 1) / SEGT;
        r = tile_base[lt];
        for (uint32_t i = lt * SEGT; i < n; i++) r += flag_count(keep[i]);
    } else {
        const uint32_t t = gi / SEGT;
        r = tile_base[t];
        for (uint32_t i = t * SEGT; i < gi; i++) r += flag_count(keep[i]);
    }
    rank_start[b] = r;
}
static __global__ void k_flag_batch_counts(const uint32_t *__restrict__ rank_start, uint32_t nb, const DevBatch *__restrict__ batches)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < nb && batches[b].n_out != nullptr) *batches[b].n_out = rank_start[b + 1] - rank_start[b];
}

template <class P>
__global__ void __launch_bounds__(256) k_flag_scatter(const unsigned char *__restrict__ keep, const uint32_t *__restrict__ tile_base,
                                                      const uint32_t *__restrict__ boff, uint32_t nb, uint32_t n,
                                                      const uint32_t *__restrict__ rank_start, const DevBatch *__restrict__ batches)
{
    using T = typename P::tuple_t;
    __shared__ uint32_t wsum[8];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t first = blockIdx.x * SEGT + tid * (SEGT / 256);
    bool k[SEGT / 256];
    uint32_t mine = 0;
#pragma unroll
    for (uint32_t r = 0; r < SEGT / 256; r++) { const uint32_t i = first + r; k[r] = i < n && keep[i]; mine += k[r] ? 1u : 0u; }
    uint32_t incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    uint32_t rank = tile_base[blockIdx.x] + incl - mine;
    for (uint32_t w = 0; w < warp; w++) rank += wsum[w];
#pragma unroll
    for (uint32_t r = 0; r < SEGT / 256; r++) {
        if (k[r]) {
            const uint32_t gi = first + r, b = batch_of(boff, nb, gi);
            const DevBatch bt = batches[b];
            const uint32_t li = gi - boff[b], o = rank - rank_start[b];
            alignas(16) T t;
            ld_rec<T>(bt.tuples + static_cast<size_t>(li) * sizeof(T), t);
            st_rec<T>(bt.out + static_cast<size_t>(o) * sizeof(T), t);
            if (bt.ts_out) bt.ts_out[o] = bt.ts[li];
            rank++;
        }
    }
}

// keyed-stateful FlatMap_GPU: off[gi] = the records of the tuples before gi in its batch (the exclusive scan of the kept counts,
// per batch), laid out as k_flag_scatter ranks its survivors
static __global__ void __launch_bounds__(256) k_fm_offsets(const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ tile_base,
                                                           const uint32_t *__restrict__ boff, uint32_t nb, uint32_t n,
                                                           const uint32_t *__restrict__ rank_start, uint32_t *__restrict__ off)
{
    __shared__ uint32_t wsum[8];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t first = blockIdx.x * SEGT + tid * (SEGT / 256);
    uint32_t c[SEGT / 256];
    uint32_t mine = 0;
#pragma unroll
    for (uint32_t r = 0; r < SEGT / 256; r++) { const uint32_t i = first + r; c[r] = i < n ? cnt[i] : 0u; mine += c[r]; }
    uint32_t incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    uint32_t rank = tile_base[blockIdx.x] + incl - mine;
    for (uint32_t w = 0; w < warp; w++) rank += wsum[w];
#pragma unroll
    for (uint32_t r = 0; r < SEGT / 256; r++) {
        const uint32_t gi = first + r;
        if (gi < n) off[gi] = rank - rank_start[batch_of(boff, nb, gi)];
        rank += c[r];
    }
}

// ------------------------------------------------------------------------------------------------------
// Keyed_Windows_GPU, count-based (wf/keyed_windows.hpp, wf/window_replica.hpp:230-407): a window function that iterates every
// tuple of the window. Per key, tuple ids 0, 1, 2, ... in arrival order; window g holds ids [g*slide, g*slide + win) and fires with the
// first tuple after it, id g*slide + win (wf/window_structure.hpp:69-80: that tuple is FIRED, not IN). The key's last C = pow2ceil(win)
// tuples live in its ring (ring + slot * C, id & (C - 1)): a window that has not fired has at most win of its tuples already. Per call the items come sorted by slot (stable: each key's run in arrival order)
// and are gathered into a staging buffer in that order, so that a window firing in the call reads its older tuples from the ring and
// the call's own from the staging buffer. Then: windows per run (k_kw_count) -> exclusive scan -> one thread per fired window
// (k_kw_eval) -> the last C tuples of every run into the ring and the key's count (k_kw_archive).
// ------------------------------------------------------------------------------------------------------

// Read-only view of one window (wf/iterable.hpp without the mutating overloads): the older part in the key's ring, ids
// [first_id, first_id + n_ring), then n_stage contiguous tuples of the current call.
template <class T>
class Iterable_GPU {
public:
    class const_iterator {
    public:
        using iterator_category = std::random_access_iterator_tag;
        using value_type = T; using difference_type = long long; using reference = const T &; using pointer = const T *;
        __host__ __device__ const_iterator(const Iterable_GPU *it, size_t i) : it_(it), i_(i) {}
        __host__ __device__ const T &operator*() const { return (*it_)[i_]; }
        __host__ __device__ const T *operator->() const { return &(*it_)[i_]; }
        __host__ __device__ const T &operator[](difference_type d) const { return (*it_)[i_ + d]; }
        __host__ __device__ const_iterator &operator++() { ++i_; return *this; }
        __host__ __device__ const_iterator operator++(int) { const_iterator o = *this; ++i_; return o; }
        __host__ __device__ const_iterator &operator--() { --i_; return *this; }
        __host__ __device__ const_iterator operator--(int) { const_iterator o = *this; --i_; return o; }
        __host__ __device__ const_iterator &operator+=(difference_type d) { i_ += d; return *this; }
        __host__ __device__ const_iterator &operator-=(difference_type d) { i_ -= d; return *this; }
        __host__ __device__ const_iterator operator+(difference_type d) const { return const_iterator(it_, i_ + d); }
        __host__ __device__ friend const_iterator operator+(difference_type d, const const_iterator &x) { return x + d; }
        __host__ __device__ const_iterator operator-(difference_type d) const { return const_iterator(it_, i_ - d); }
        __host__ __device__ difference_type operator-(const const_iterator &o) const { return static_cast<difference_type>(i_) - static_cast<difference_type>(o.i_); }
        __host__ __device__ bool operator==(const const_iterator &o) const { return i_ == o.i_; }
        __host__ __device__ bool operator!=(const const_iterator &o) const { return i_ != o.i_; }
        __host__ __device__ bool operator<(const const_iterator &o) const { return i_ < o.i_; }
        __host__ __device__ bool operator<=(const const_iterator &o) const { return i_ <= o.i_; }
        __host__ __device__ bool operator>(const const_iterator &o) const { return i_ > o.i_; }
        __host__ __device__ bool operator>=(const const_iterator &o) const { return i_ >= o.i_; }
    private:
        const Iterable_GPU *it_; size_t i_;
    };
    using iterator = const_iterator;

    __host__ __device__ Iterable_GPU(const T *ring, uint32_t mask, uint64_t first_id, uint32_t n_ring, const T *stage, uint32_t n_stage)
        : ring_(ring), mask_(mask), first_(first_id), n_ring_(n_ring), stage_(stage), n_stage_(n_stage) {}
    __host__ __device__ size_t size() const { return static_cast<size_t>(n_ring_) + n_stage_; }
    __host__ __device__ const T &operator[](size_t i) const
    {
        return i < n_ring_ ? ring_[(first_ + i) & mask_] : stage_[i - n_ring_];
    }
    __host__ __device__ const T &at(size_t i) const { return (*this)[i < size() ? i : size() - 1]; } // (no exceptions on the device: clamped)
    __host__ __device__ const T &front() const { return (*this)[0]; }
    __host__ __device__ const T &back() const { return (*this)[size() - 1]; }
    __host__ __device__ const_iterator begin() const { return const_iterator(this, 0); }
    __host__ __device__ const_iterator end() const { return const_iterator(this, size()); }

private:
    const T *ring_; uint32_t mask_; uint64_t first_; uint32_t n_ring_; const T *stage_; uint32_t n_stage_;
};

// state and geometry of one Keyed_Windows_GPU handle as its kernels see it
struct KwinDev {
    unsigned char *ring;     // max_keys * C tuples (incremental: max_keys * C accumulators)
    uint64_t *cnt;           // tuples of each slot so far
    uint64_t *last_ts;       // largest timestamp seen (the end-of-stream windows carry it)
    uint64_t win, slide;
    uint32_t C;              // ring length (power of two >= win; incremental: >= ceil(win / slide))
    uint32_t max_keys;
    uint32_t *err_flags;     // bit 0: a key found no slot, bit 1: more results than the output capacity
    uint32_t *n_slots;       // slots taken (a dense table takes none: slot = key, every slot may hold a key)
    uint32_t dense;
};

// the windows g whose firing id g*slide + win lies in [c, c + m) (fired by a run of m tuples on a key that had c): [*g_lo, *g_lo + count)
__device__ __forceinline__ uint64_t kw_fired(uint64_t c, uint64_t m, uint64_t win, uint64_t slide, uint64_t *g_lo)
{
    const uint64_t lo = c > win ? (c - win + slide - 1) / slide : 0;
    *g_lo = lo;
    if (c + m <= win) return 0;
    const uint64_t hi = (c + m - 1 - win) / slide;
    return hi >= lo ? hi - lo + 1 : 0;
}

// first index in [lo, hi) whose sorted slot is >= v
__device__ __forceinline__ uint32_t kw_lower_bound(const uint32_t *__restrict__ a, uint32_t lo, uint32_t hi, uint32_t v)
{
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (a[mid] < v) lo = mid + 1; else hi = mid; }
    return lo;
}

// staging: tuple and timestamp of every sorted position; the largest timestamp of the call into last_ts
template <class P>
__global__ void __launch_bounds__(256) k_kw_stage(const DevBatch *__restrict__ batches, const uint32_t *__restrict__ boff, uint32_t nb, uint32_t n,
                                                  const uint32_t *__restrict__ sorted_pos, unsigned char *__restrict__ stage,
                                                  uint64_t *__restrict__ stage_ts, uint64_t *__restrict__ last_ts)
{
    using T = typename P::tuple_t;
    uint64_t mx = 0;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t gi = sorted_pos[j], b = batch_of(boff, nb, gi), li = gi - boff[b];
        alignas(16) T t;
        ld_rec<T>(batches[b].tuples + static_cast<size_t>(li) * sizeof(T), t);
        st_rec<T>(stage + static_cast<size_t>(j) * sizeof(T), t);
        const uint64_t ts = batches[b].ts != nullptr ? batches[b].ts[li] : 0;
        stage_ts[j] = ts;
        mx = ts > mx ? ts : mx;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const uint64_t v = __shfl_xor_sync(FULL, mx, o); mx = v > mx ? v : mx; }
    if ((threadIdx.x & 31u) == 0 && mx != 0) atomicMax(reinterpret_cast<unsigned long long *>(last_ts), static_cast<unsigned long long>(mx));
}

// per sorted position: the windows its run fires (run heads only; 0 elsewhere), and the run's length and starting count at its head
static __global__ void __launch_bounds__(256) k_kw_count(const KwinDev kw, const uint32_t *__restrict__ sorted_slots, uint32_t n,
                                                         uint32_t *__restrict__ wcnt, uint32_t *__restrict__ run_m, uint64_t *__restrict__ run_c)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t slot = sorted_slots[j];
        uint32_t w = 0;
        if (slot < kw.max_keys && (j == 0 || sorted_slots[j - 1] != slot)) {
            const uint32_t m = kw_lower_bound(sorted_slots, j, n, slot + 1) - j;
            const uint64_t c = kw.cnt[slot];
            uint64_t g_lo;
            w = static_cast<uint32_t>(kw_fired(c, m, kw.win, kw.slide, &g_lo));
            run_m[j] = m; run_c[j] = c;
        }
        wcnt[j] = w;
    }
}

// woff[j] = windows of the positions before j (tile_base: the exclusive scan of the SEGT-position tile sums); total -> *n_total
static __global__ void __launch_bounds__(256) k_kw_offsets(const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ tile_base, uint32_t n,
                                                           uint32_t *__restrict__ off)
{
    __shared__ uint32_t wsum[8];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t first = blockIdx.x * SEGT + tid * (SEGT / 256);
    uint32_t c[SEGT / 256];
    uint32_t mine = 0;
#pragma unroll
    for (uint32_t r = 0; r < SEGT / 256; r++) { const uint32_t i = first + r; c[r] = i < n ? cnt[i] : 0u; mine += c[r]; }
    uint32_t incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, o); if (lane >= static_cast<uint32_t>(o)) incl += v; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    uint32_t rank = tile_base[blockIdx.x] + incl - mine;
    for (uint32_t w = 0; w < warp; w++) rank += wsum[w];
#pragma unroll
    for (uint32_t r = 0; r < SEGT / 256; r++) {
        const uint32_t i = first + r;
        if (i < n) off[i] = rank;
        rank += c[r];
    }
}

// *n_out = min(total, cap); bit 1 when the results exceed the capacity
static __global__ void k_kw_clamp(const uint32_t *__restrict__ total, uint32_t cap, uint32_t *__restrict__ n_out, uint32_t *__restrict__ err_flags)
{
    const uint32_t t = *total;
    *n_out = t < cap ? t : cap;
    if (t > cap) atomicOr(err_flags, 2u);
}

// one thread per fired window (the first min(total, cap)): its run by binary search over the offsets, its view, the user's function
template <class P>
__global__ void __launch_bounds__(128) k_kw_eval(const KwinDev kw, const uint32_t *__restrict__ sorted_slots, uint32_t n,
                                                 const uint32_t *__restrict__ woff, const uint32_t *__restrict__ run_m, const uint64_t *__restrict__ run_c,
                                                 const unsigned char *__restrict__ stage, const uint64_t *__restrict__ stage_ts,
                                                 const uint32_t *__restrict__ n_out, unsigned char *__restrict__ out, uint64_t *__restrict__ out_ts,
                                                 const typename P::params_t prm)
{
    using T = typename P::tuple_t; using R = typename P::result_t;
    const uint32_t total = *n_out;
    const T *st = reinterpret_cast<const T *>(stage);
    for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < total; w += gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = n; // last j with woff[j] <= w: the run head whose windows include w
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (woff[mid] <= w) lo = mid; else hi = mid; }
        const uint32_t j = lo, slot = sorted_slots[j];
        const uint64_t c = run_c[j];
        uint64_t g_lo;
        kw_fired(c, run_m[j], kw.win, kw.slide, &g_lo);
        const uint64_t g = g_lo + (w - woff[j]), first = g * kw.slide, last = first + kw.win; // ids [first, last)
        const uint32_t n_ring = first < c ? static_cast<uint32_t>(c - first) : 0u;
        const uint32_t s0 = j + static_cast<uint32_t>(first > c ? first - c : 0); // staging index of the window's first id of this call
        const Iterable_GPU<T> it(reinterpret_cast<const T *>(kw.ring) + static_cast<size_t>(slot) * kw.C, kw.C - 1, first, n_ring,
                                 st + s0, static_cast<uint32_t>(kw.win) - n_ring);
        R r = P::make_result(P::key(st[j], prm), g, prm);
        P::win_func(it, r, prm);
        st_rec<R>(out + static_cast<size_t>(w) * sizeof(R), r);
        if (out_ts != nullptr) out_ts[w] = stage_ts[j + static_cast<uint32_t>(last - c)]; // (the firing tuple, id `last`, is of this call)
    }
}

// after k_kw_eval: the last C tuples of every run into the key's ring; the run's head stores the key's new count
template <class P>
__global__ void __launch_bounds__(256) k_kw_archive(const KwinDev kw, const uint32_t *__restrict__ sorted_slots, uint32_t n,
                                                    const uint32_t *__restrict__ run_m, const uint64_t *__restrict__ run_c,
                                                    const unsigned char *__restrict__ stage)
{
    using T = typename P::tuple_t;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t slot = sorted_slots[j];
        if (slot >= kw.max_keys) continue;
        const uint32_t head = kw_lower_bound(sorted_slots, 0, j, slot), r = j - head, m = run_m[head];
        const uint64_t c = run_c[head];
        if (static_cast<uint64_t>(r) + kw.C >= m) {
            alignas(16) T t;
            ld_rec<T>(stage + static_cast<size_t>(j) * sizeof(T), t);
            st_rec<T>(kw.ring + (static_cast<size_t>(slot) * kw.C + ((c + r) & (kw.C - 1))) * sizeof(T), t);
        }
        if (r == 0) kw.cnt[slot] = c + m;
    }
}

// end of stream (wf/window_replica.hpp:356-407): every window of every key that opened (g*slide < count) and has not fired
// (g*slide + win >= count: also a complete window whose firing tuple never came), on the tuples of it that arrived, with the largest
// timestamp seen. One thread per key; a key's windows take consecutive results.
template <class P>
__global__ void __launch_bounds__(128) k_kw_flush(const KwinDev kw, uint32_t *__restrict__ total, uint32_t cap, unsigned char *__restrict__ out,
                                                  uint64_t *__restrict__ out_ts, const typename P::params_t prm)
{
    using T = typename P::tuple_t; using R = typename P::result_t;
    const uint32_t nk = kw.dense ? kw.max_keys : min(*kw.n_slots, kw.max_keys);
    const uint64_t ts = *kw.last_ts;
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < nk; s += gridDim.x * blockDim.x) {
        const uint64_t c = kw.cnt[s];
        if (c == 0) continue;
        const uint64_t g_lo = c > kw.win ? (c - kw.win + kw.slide - 1) / kw.slide : 0, g_hi = (c - 1) / kw.slide; // g*slide <= c-1
        if (g_hi < g_lo) continue;
        const T *ring = reinterpret_cast<const T *>(kw.ring) + static_cast<size_t>(s) * kw.C;
        const uint32_t k = static_cast<uint32_t>(g_hi - g_lo + 1), base = atomicAdd(total, k);
        for (uint32_t q = 0; q < k && base + q < cap; q++) {
            const uint64_t g = g_lo + q, first = g * kw.slide;
            const Iterable_GPU<T> it(ring, kw.C - 1, first, static_cast<uint32_t>(min(c, first + kw.win) - first), nullptr, 0);
            R r = P::make_result(P::key(it.front(), prm), g, prm);
            P::win_func(it, r, prm);
            st_rec<R>(out + static_cast<size_t>(base + q) * sizeof(R), r);
            if (out_ts != nullptr) out_ts[base + q] = ts;
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// Keyed_Windows_GPU, incremental (WFB_KWIN_INCREMENTAL; wf/window_replica.hpp:293-303): win_func_inc(t, acc, params) folds every tuple
// that is IN window g into its accumulator, in arrival order. Per key the handle keeps its count and a ring of C = pow2ceil(ceil(win /
// slide)) accumulators (kw.ring + slot * C results, entry g & (C - 1)): at most ceil(win / slide) windows are open at once, and windows
// open together never share an entry. A call reuses the staging gather, then per run (a key's m tuples of the call, count c before it)
// the windows it touches, g with g*slide <= c + m - 1 and g*slide + win >= c, are [g_lo, g_lo + fired + open): the fired ones first
// (k_kwi_count), each count scanned on its own (fired -> output index, open -> pending index, their sum -> the run of a thread). Then
// one thread per touched window (k_kwi_eval) and the copy of the windows opened in the call that stay open into the ring (k_kwi_writeback).
// The ring hazard: a window open before the call can fire in it while a window opened in the same call stays open in the same entry, so
// the latter is written to the pending buffer and copied after every read of the call. A window open before the call that stays open
// is written in place: no other window open before the call, and none open after it, shares its entry.
// ------------------------------------------------------------------------------------------------------

// one record from src to dst, both aligned as ld_rec / st_rec require
template <class R>
__device__ __forceinline__ void copy_rec(unsigned char *__restrict__ dst, const unsigned char *__restrict__ src)
{
    if constexpr (sizeof(R) % 16 == 0) {
#pragma unroll
        for (uint32_t k = 0; k < sizeof(R) / 16; k++) reinterpret_cast<uint4 *>(dst)[k] = reinterpret_cast<const uint4 *>(src)[k];
    } else {
#pragma unroll
        for (uint32_t k = 0; k < sizeof(R) / 8; k++) reinterpret_cast<uint64_t *>(dst)[k] = reinterpret_cast<const uint64_t *>(src)[k];
    }
}

// per sorted position: the windows its run fires and those it leaves open (run heads only; 0 elsewhere), the run's length and starting
// count at its head; the head also stores the key's new count (the call's later kernels read the starting count from run_c)
static __global__ void __launch_bounds__(256) k_kwi_count(const KwinDev kw, const uint32_t *__restrict__ sorted_slots, uint32_t n,
                                                          uint32_t *__restrict__ wcnt, uint32_t *__restrict__ ocnt, uint32_t *__restrict__ run_m,
                                                          uint64_t *__restrict__ run_c)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t slot = sorted_slots[j];
        uint32_t w = 0, o = 0;
        if (slot < kw.max_keys && (j == 0 || sorted_slots[j - 1] != slot)) {
            const uint32_t m = kw_lower_bound(sorted_slots, j, n, slot + 1) - j;
            const uint64_t c = kw.cnt[slot];
            uint64_t g_lo;
            w = static_cast<uint32_t>(kw_fired(c, m, kw.win, kw.slide, &g_lo));
            const uint64_t g_hi = (c + m - 1) / kw.slide; // the last window whose first id is of this call or earlier
            o = g_hi + 1 >= g_lo + w ? static_cast<uint32_t>(g_hi + 1 - g_lo - w) : 0u;
            run_m[j] = m; run_c[j] = c;
            kw.cnt[slot] = c + m;
        }
        wcnt[j] = w; ocnt[j] = o;
    }
}

// one thread per touched window: its run by binary search over the summed offsets, its accumulator (the ring entry when it opened before
// the call, else make_result(key, g)), the fold of the call's tuples IN it; then the result (fired, among the first *n_out) or the
// accumulator (open: in place, or to the pending buffer when it opened in this call)
template <class P>
__global__ void __launch_bounds__(128) k_kwi_eval(const KwinDev kw, const uint32_t *__restrict__ sorted_slots, uint32_t n,
                                                  const uint32_t *__restrict__ woff, const uint32_t *__restrict__ ooff, const uint32_t *__restrict__ n_open,
                                                  const uint32_t *__restrict__ run_m, const uint64_t *__restrict__ run_c,
                                                  const unsigned char *__restrict__ stage, const uint64_t *__restrict__ stage_ts,
                                                  const uint32_t *__restrict__ n_fired, const uint32_t *__restrict__ n_out, unsigned char *__restrict__ out,
                                                  uint64_t *__restrict__ out_ts, unsigned char *__restrict__ pending, const typename P::params_t prm)
{
    using T = typename P::tuple_t; using R = typename P::result_t;
    const uint32_t total = *n_fired + *n_open, cap = *n_out; // (the host keeps fired + open below 2^32)
    const T *st = reinterpret_cast<const T *>(stage);
    for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < total; w += gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = n; // last j with woff[j] + ooff[j] <= w: the run head whose windows include w
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (woff[mid] + ooff[mid] <= w) lo = mid; else hi = mid; }
        const uint32_t j = lo, slot = sorted_slots[j], q = w - (woff[j] + ooff[j]);
        const uint64_t c = run_c[j], m = run_m[j];
        uint64_t g_lo;
        const uint32_t nf = static_cast<uint32_t>(kw_fired(c, m, kw.win, kw.slide, &g_lo));
        const bool fired = q < nf;
        if (fired && woff[j] + q >= cap) continue; // (beyond the output capacity: error bit 1; a fired window keeps no state)
        const uint64_t g = g_lo + q, first = g * kw.slide, last = first + kw.win; // ids [first, last)
        unsigned char *entry = kw.ring + (static_cast<size_t>(slot) * kw.C + (g & (kw.C - 1))) * sizeof(R);
        alignas(16) R r = P::make_result(P::key(st[j], prm), g, prm);
        if (first < c) ld_rec<R>(entry, r);
        const uint64_t a = first > c ? first : c, b = last < c + m ? last : c + m;
        for (uint64_t id = a; id < b; id++) P::win_func_inc(st[j + static_cast<uint32_t>(id - c)], r, prm);
        if (fired) {
            st_rec<R>(out + static_cast<size_t>(woff[j] + q) * sizeof(R), r);
            if (out_ts != nullptr) out_ts[woff[j] + q] = stage_ts[j + static_cast<uint32_t>(last - c)]; // (the firing tuple, id `last`, is of this call)
        } else if (first < c) {
            st_rec<R>(entry, r);
        } else {
            st_rec<R>(pending + static_cast<size_t>(ooff[j] + (q - nf)) * sizeof(R), r);
        }
    }
}

// after k_kwi_eval: the accumulators of the windows opened in the call that stay open, from the pending buffer into their ring entries
template <class P>
__global__ void __launch_bounds__(256) k_kwi_writeback(const KwinDev kw, const uint32_t *__restrict__ sorted_slots, uint32_t n,
                                                       const uint32_t *__restrict__ ooff, const uint32_t *__restrict__ n_open,
                                                       const uint32_t *__restrict__ run_m, const uint64_t *__restrict__ run_c,
                                                       const unsigned char *__restrict__ pending)
{
    using R = typename P::result_t;
    const uint32_t total = *n_open;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = n; // last j with ooff[j] <= i
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (ooff[mid] <= i) lo = mid; else hi = mid; }
        const uint32_t j = lo;
        const uint64_t c = run_c[j];
        uint64_t g_lo;
        const uint64_t nf = kw_fired(c, run_m[j], kw.win, kw.slide, &g_lo), g = g_lo + nf + (i - ooff[j]);
        if (g * kw.slide < c) continue; // (opened before the call: k_kwi_eval wrote it in place)
        copy_rec<R>(kw.ring + (static_cast<size_t>(sorted_slots[j]) * kw.C + (g & (kw.C - 1))) * sizeof(R), pending + static_cast<size_t>(i) * sizeof(R));
    }
}

// end of stream: the accumulator of every window of every key that opened and has not fired, in window order, with the largest
// timestamp seen (the window set of k_kw_flush). One thread per key; a key's windows take consecutive results.
template <class P>
__global__ void __launch_bounds__(128) k_kwi_flush(const KwinDev kw, uint32_t *__restrict__ total, uint32_t cap, unsigned char *__restrict__ out,
                                                   uint64_t *__restrict__ out_ts)
{
    using R = typename P::result_t;
    const uint32_t nk = kw.dense ? kw.max_keys : min(*kw.n_slots, kw.max_keys);
    const uint64_t ts = *kw.last_ts;
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < nk; s += gridDim.x * blockDim.x) {
        const uint64_t c = kw.cnt[s];
        if (c == 0) continue;
        const uint64_t g_lo = c > kw.win ? (c - kw.win + kw.slide - 1) / kw.slide : 0, g_hi = (c - 1) / kw.slide;
        if (g_hi < g_lo) continue;
        const uint32_t k = static_cast<uint32_t>(g_hi - g_lo + 1), base = atomicAdd(total, k);
        for (uint32_t q = 0; q < k && base + q < cap; q++) {
            const uint64_t g = g_lo + q;
            copy_rec<R>(out + static_cast<size_t>(base + q) * sizeof(R), kw.ring + (static_cast<size_t>(s) * kw.C + (g & (kw.C - 1))) * sizeof(R));
            if (out_ts != nullptr) out_ts[base + q] = ts;
        }
    }
}

// Reduce_GPU un-keyed: the whole batch folded into one item, starting from a default-constructed item
// (thrust::reduce with init = batch_item_gpu_t<tuple_t>(), wf/reduce_gpu.hpp:264-273). One CTA of 1024 threads.
template <class P>
__global__ void __launch_bounds__(1024) k_reduce_all(const unsigned char *__restrict__ tuples, const uint64_t *__restrict__ ts, uint32_t n,
                                                     unsigned char *__restrict__ out_tuple, uint64_t *__restrict__ out_ts,
                                                     const typename P::params_t prm)
{
    using T = typename P::tuple_t;
    __shared__ __align__(16) unsigned char sm[32 * sizeof(T)];
    __shared__ uint64_t smts[32];
    __shared__ uint32_t smhave[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // thread t folds the contiguous chunk [t*per, (t+1)*per): order preserved
    const uint32_t per = (n + 1023) / 1024;
    const uint32_t b = min(tid * per, n), e = min(b + per, n);
    alignas(16) T acc; uint64_t mts = 0; bool have = false;
    for (uint32_t i = b; i < e; i++) {
        alignas(16) T t; ld_rec<T>(tuples + static_cast<size_t>(i) * sizeof(T), t);
        const uint64_t tt = ts ? ts[i] : 0;
        if (!have) { acc = t; mts = tt; have = true; } else { acc = P::reduce(acc, t, prm); mts = mts < tt ? tt : mts; }
    }
    // ordered combine across lanes, then across warps (a lane/warp without items is skipped)
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
        const T other = shfl_down_rec<T>(acc, o);
        const uint64_t ots = __shfl_down_sync(FULL, mts, o);
        const bool ohave = __shfl_down_sync(FULL, have ? 1u : 0u, o) != 0;
        if (lane + o < 32 && ohave) {
            if (have) { acc = P::reduce(acc, other, prm); mts = mts < ots ? ots : mts; } else { acc = other; mts = ots; have = true; }
        }
    }
    if (lane == 0) { st_rec<T>(sm + warp * sizeof(T), acc); smts[warp] = mts; smhave[warp] = have ? 1u : 0u; }
    __syncthreads();
    if (tid == 0) {
        T init{};                 // default-constructed tuple, timestamp 0
        alignas(16) T r = init; uint64_t rts = 0;
        for (uint32_t w = 0; w < 32; w++) if (smhave[w]) {
            alignas(16) T t; ld_rec<T>(sm + w * sizeof(T), t);
            r = P::reduce(r, t, prm); rts = rts < smts[w] ? smts[w] : rts;
        }
        st_rec<T>(out_tuple, r);
        if (out_ts) *out_ts = rts;
    }
}

// payload gather after a stable partition: out[j] = in[perm[j]] (tuples and timestamps)
template <class P>
__global__ void k_gather_tuples(const unsigned char *__restrict__ tuples, const uint64_t *__restrict__ ts, const uint32_t *__restrict__ perm,
                                uint32_t n, unsigned char *__restrict__ out_tuples, uint64_t *__restrict__ out_ts)
{
    using T = typename P::tuple_t;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t i = perm[j];
        alignas(16) T t; ld_rec<T>(tuples + static_cast<size_t>(i) * sizeof(T), t);
        st_rec<T>(out_tuples + static_cast<size_t>(j) * sizeof(T), t);
        if (ts && out_ts) out_ts[j] = ts[i];
    }
}

// seg_off[d] for d in [0, num_shards]: first sorted position whose destination is >= d (sorted dest array)
static __global__ void k_shard_offsets(const uint32_t *__restrict__ sdest, uint32_t n, uint32_t num_shards, uint32_t *__restrict__ seg_off)
{
    for (uint32_t d = blockIdx.x * blockDim.x + threadIdx.x; d <= num_shards; d += gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = n; // lower_bound(sdest, d)
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (sdest[mid] < d) lo = mid + 1; else hi = mid; }
        seg_off[d] = lo;
    }
}

// pipelined window operator: hand the results of a finished segment over to the caller's buffers
static __global__ void k_copy_results(const unsigned char *__restrict__ src, const uint64_t *__restrict__ src_ts, const uint32_t *__restrict__ src_n,
                               uint32_t rec_bytes, unsigned char *__restrict__ dst, uint64_t *__restrict__ dst_ts, uint32_t dst_cap,
                               uint32_t *__restrict__ n_out, uint32_t *__restrict__ err_flags)
{
    const uint32_t n = *src_n;
    const uint32_t m = min(n, dst_cap);
    const uint64_t words = static_cast<uint64_t>(m) * (rec_bytes / 8);
    const uint64_t *s8 = reinterpret_cast<const uint64_t *>(src);
    uint64_t *d8 = reinterpret_cast<uint64_t *>(dst);
    const uint64_t gtid = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x, gsz = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t w = gtid; w < words; w += gsz) d8[w] = s8[w];
    if (dst_ts != nullptr) for (uint64_t i = gtid; i < m; i += gsz) dst_ts[i] = src_ts[i];
    if (gtid == 0) { *n_out = m; if (n > dst_cap) atomicOr(err_flags, 2u); }
}

// ------------------------------------------------------------------------------------------------------
// synthetic stream of SURVEY.md 8d (integer arithmetic specified there; the tests check it bit for bit)
// ------------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x)
{
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

static __global__ void k_gen_tuple64(uint64_t seed, uint64_t start, uint32_t n, int key_mode, uint64_t nkeys,
                              const double *__restrict__ zipf_cdf, wfb_tuple64_t *__restrict__ out, uint64_t *__restrict__ ts)
{
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint64_t i = start + j;
        uint64_t key;
        if (key_mode == 0) key = i % nkeys;
        else if (key_mode == 1) key = splitmix64(i) % nkeys;
        else {
            const double u = static_cast<double>(splitmix64(i ^ 0xA5A5A5A5A5A5A5A5ull) >> 11) * (1.0 / 9007199254740992.0);
            uint64_t lo = 0, hi = nkeys - 1;
            while (lo < hi) { const uint64_t mid = (lo + hi) >> 1; if (zipf_cdf[mid] > u) hi = mid; else lo = mid + 1; }
            key = lo;
        }
        const int64_t iv = static_cast<int64_t>(splitmix64(seed ^ i) & 0xFFFFull);
        const double fv = static_cast<double>(splitmix64(seed ^ ~i) >> 11) * (1.0 / 9007199254740992.0);
        uint4 *o = reinterpret_cast<uint4 *>(out + j);
        uint4 c0, c1;
        c0.x = static_cast<uint32_t>(key); c0.y = static_cast<uint32_t>(key >> 32);
        c0.z = static_cast<uint32_t>(i); c0.w = static_cast<uint32_t>(i >> 32);
        const uint64_t ivb = static_cast<uint64_t>(iv);
        const uint64_t fvb = static_cast<uint64_t>(__double_as_longlong(fv));
        c1.x = static_cast<uint32_t>(ivb); c1.y = static_cast<uint32_t>(ivb >> 32);
        c1.z = static_cast<uint32_t>(fvb); c1.w = static_cast<uint32_t>(fvb >> 32);
        o[0] = c0; o[1] = c1; o[2] = make_uint4(0, 0, 0, 0); o[3] = make_uint4(0, 0, 0, 0);
        if (ts != nullptr) ts[j] = i;
    }
}

} // namespace wfb
