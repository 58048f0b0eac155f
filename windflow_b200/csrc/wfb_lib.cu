// wfb_lib.cu -- libwfb200.so: the extern "C" layer of include/wfb200.h over the kernels of wfb_kernels.cuh,
// instantiated for the built-in programs of wfb_programs.cuh. No Thrust, no unified memory, no CPU fallback:
// every compute entry point fails with WFB_E_NOGPU when there is no CUDA device.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <mutex>
#include <vector>
#include <algorithm>
#include <atomic>
#include <new>
#include <cuda.h>
#include <cuda_runtime.h>
#include "../../include/wfb200.h"
#include "wfb_kernels.cuh"
#include "wfb_launch.cuh"
#include "wfb_programs.cuh"
#include "wfb_scratch.h"

using namespace wfb;

#define CK(call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) return static_cast<int>(e__); } while (0)

namespace {

int g_num_sms = 0;

int device_ready()
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { cudaGetLastError(); return WFB_E_NOGPU; }
    if (g_num_sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return WFB_E_NOGPU;
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    return 0;
}

std::mutex &registry_mutex() { static std::mutex m; return m; } // replicas of different operators may register programs concurrently

std::vector<ProgramOps> &registry()
{
    static std::vector<ProgramOps> table; if (table.empty()) { table.reserve(4096); table = { make_ops<ProgTuple64>(), make_ops<ProgWfTest16>(), make_ops<ProgWfWin24>(), make_ops<ProgLifted32>(),
                                                                 make_ops<ProgTuple64FKey>(), make_ops<ProgTuple64K16>() }; table.reserve(4096); }
    return table;
}

const ProgramOps *program(int prog)
{
    std::lock_guard<std::mutex> lock(registry_mutex());
    std::vector<ProgramOps> &t = registry();
    if (prog < 0 || prog >= static_cast<int>(t.size())) return nullptr;
    return &t[prog];
}

// ---- host -> device staging of the small per-call tables (batch descriptors, offsets): a ring of pinned buffers, so that the
// copy is a real asynchronous DMA (a cudaMemcpyAsync from pageable memory is staged by the driver and serialises with the stream) ----
struct PinnedStage {
    static constexpr int SLOTS = 8;
    PinnedScratch<unsigned char> buf[SLOTS]; cudaEvent_t ev[SLOTS] = {}; bool used[SLOTS] = {}; int next = 0;
    int h2d(void *dst, const void *src, size_t bytes, cudaStream_t s)
    {
        if (bytes == 0) return 0;
        const int i = next; next = (next + 1) % SLOTS;
        if (used[i]) CK(cudaEventSynchronize(ev[i])); // the copy that used this slot SLOTS calls ago has long finished
        CK(buf[i].ensure(bytes, ScratchWaits(), std::max<size_t>(bytes, 4096) * 2));
        if (!ev[i]) CK(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
        std::memcpy(buf[i], src, bytes);
        CK(cudaMemcpyAsync(dst, buf[i], bytes, cudaMemcpyHostToDevice, s));
        CK(cudaEventRecord(ev[i], s)); used[i] = true;
        return 0;
    }
    void destroy() { for (int i = 0; i < SLOTS; i++) { if (ev[i]) cudaEventDestroy(ev[i]); ev[i] = nullptr; } }
};

// ---- stream order of one handle: a call on a new stream waits for everything the handle issued on the previous one ----------
// A handle's scratch and state are shared by its consecutive calls, and the reference launches on each batch's own stream
// (wf/map_gpu.hpp:399-405), so a caller may hop between streams from one call to the next.
struct StreamOrder {
    cudaStream_t last_stream = nullptr; bool used = false; cudaEvent_t ev = nullptr;

    int init() { CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); return 0; }
    void destroy() { if (ev) cudaEventDestroy(ev); ev = nullptr; }
    int enter(cudaStream_t s)
    {
        if (used && s != last_stream) { CK(cudaEventRecord(ev, last_stream)); CK(cudaStreamWaitEvent(s, ev, 0)); }
        last_stream = s; used = true;
        return 0;
    }
};

// ---- scratch shared by the tile passes: ticket counter, epoch-tagged tile states, batch descriptors -----------
struct TileScratch {
    PinnedStage stage;
    Scratch<uint64_t> tile_state;
    Scratch<uint32_t> ticket; uint32_t ticket_base = 0; uint32_t epoch = 0;
    Scratch<DevBatch> d_batches;
    StreamOrder order;

    int init()
    {
        CK(ticket.ensure(1));
        CK(cudaMemset(ticket, 0, sizeof(uint32_t)));
        return order.init();
    }
    void destroy()
    {
        stage.destroy();
        order.destroy();
    }
    int enter(cudaStream_t s) { return order.enter(s); }
    int ensure_tiles(uint32_t num_tiles) { return tile_state.ensure_zeroed(num_tiles, order.last_stream, order.last_stream); } // epoch 0 is never used by a launch
    int ensure_batches(uint32_t nb) { return d_batches.ensure(nb, order.last_stream); }
    void next_launch(TileArgs &a) { epoch = (epoch + 1) & 0x3fffffffu; if (epoch == 0) epoch = 1; a.epoch = epoch; a.ticket = ticket; a.ticket_base = ticket_base; a.tile_state = tile_state; }
    void launched(uint32_t num_claims, uint32_t grid) { ticket_base += num_claims + grid; } // one failing claim per CTA
};

inline uint32_t tiles_of(uint32_t n) { return (n + TILE - 1) / TILE; }

// wide tiles per CTA of k_wide_scatter_ranked (and per row T of k_wide_tile_bases): OSR_GROUP when no records travel and every SM gets a
// group, else 1
inline uint32_t osr_group(uint32_t tiles, bool payload) { return !payload && tiles >= OSR_GROUP * static_cast<uint32_t>(g_num_sms) ? OSR_GROUP : 1u; }

// k_wide_scatter_ranked takes more than 48 KB of dynamic shared memory: opt in once per device (bit = device ordinal)
cudaError_t osr_smem_attr()
{
    static std::atomic<uint64_t> done{0};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const uint64_t bit = 1ull << (dev & 63);
    if (done.load(std::memory_order_relaxed) & bit) return cudaSuccess;
    e = cudaFuncSetAttribute(k_wide_scatter_ranked, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(OSR_SMEM));
    if (e == cudaSuccess) done.fetch_or(bit, std::memory_order_relaxed);
    return e;
}

// scratch + launcher of the onesweep radix sort (one per engine / window handle)
struct RadixSorter {
    Scratch<uint32_t> ctl;          // [passes][256] histograms + [passes] tickets
    Scratch<uint64_t> state;        // [tiles][digits] look-back words
    uint32_t epoch = 0;
    uint64_t launches = 0;

    // stable sort of (kA[i], i) by the low 8*passes bits; n on the device (n_ptr) or the host (n_host), cap = upper bound
    // clears the histograms / tickets of the next sort; call it BEFORE a producer that fills the histograms itself
    static constexpr size_t CTL_WORDS = OS_MAX_PASSES * 256 + OS_MAX_PASSES > OSW_DIGITS + 1 ? OS_MAX_PASSES * 256 + OS_MAX_PASSES : OSW_DIGITS + 1;
    static int prepare(uint32_t *ctl_buf, uint32_t passes, cudaStream_t s)
    {
        passes = std::min<uint32_t>(std::max(1u, passes), OS_MAX_PASSES);
        WFB_CK(cudaMemsetAsync(ctl_buf, 0, sizeof(uint32_t) * (passes * 256 + passes), s));
        return 0;
    }

    // wide pass (10-bit digit): ctl = [1024 counts][ticket]
    static int prepare_wide(uint32_t *ctl_buf, cudaStream_t s)
    {
        WFB_CK(cudaMemsetAsync(ctl_buf, 0, sizeof(uint32_t) * (OSW_DIGITS + 1), s));
        return 0;
    }
    // ONE stable partition pass of (kin[i], i) on the digit (key >> shift) & 1023 into (kout, vout): per-tile counts, then
    // the scatter (no chained scan). *counts = the 1024 digit counts (ready_ctl if the producer of the keys made them).
    Scratch<uint16_t> wideH; Scratch<uint32_t> wideC;
    Scratch<uint32_t> wideT;    // [groups of osr_group() tiles][1024]: sum of the earlier rows of the group's chunk (k_wide_tile_bases)
    Scratch<uint32_t> wideDone; // finished chunks of k_wide_tile_bases (zero between launches)
    // tiles of the wide pass over `cap` positions and their chunks. prefix = false: about sqrt(tiles) chunks of >= 16 tiles, every
    // scatter CTA sums the rows of the earlier chunks itself; true (rows filed by the tile pass): chunks of 32 tiles; one kernel
    // (k_wide_tile_bases) computes the first output positions of every chunk and the in-chunk offsets of every tile, so a scatter
    // CTA reads two rows
    static void wide_geometry(uint32_t cap, bool prefix, uint32_t *tiles, uint32_t *chunk_shift, uint32_t *chunks)
    {
        *tiles = std::max(1u, (cap + OSW_TILE - 1) / OSW_TILE);
        uint32_t cs = prefix ? 5 : 4; // (prefix: 32 tiles per chunk -- the scan over the chunks, done by one CTA, stays short)
        if (!prefix) while ((1u << (2 * cs)) < *tiles) cs++;
        *chunk_shift = cs;
        *chunks = (*tiles + (1u << cs) - 1) >> cs;
    }
    // grows the rows and chunk rows of the wide pass; the chunk rows alone when only they are short, so that rows a producer has
    // already filed (ensure_wide, whose chunks of 32 tiles may be fewer than sort_wide's without a prefix) survive
    int ensure_wide_buffers(uint32_t tiles, uint32_t chunks, ScratchWaits waits)
    {
        const size_t rows = static_cast<size_t>(OSW_DIGITS) * tiles, chunk_rows = static_cast<size_t>(OSW_DIGITS) * chunks;
        CK(wideH.ensure(rows, waits, rows));
        CK(wideT.ensure(rows, waits, rows)); // (one row per group: as many as tiles at a group of 1)
        CK(wideC.ensure(chunk_rows, waits, chunk_rows));
        return 0;
    }
    // rows of the wide partition for `cap` positions, allocated before the producer of the keys files them (TileArgs::wide_h16);
    // waits: the streams that may still read the rows (a pipelined handle's sort stream too)
    int ensure_wide(uint32_t cap, ScratchWaits waits, uint16_t **rows)
    {
        uint32_t tiles, chunk_shift, chunks;
        wide_geometry(cap, true, &tiles, &chunk_shift, &chunks);
        { int rc = ensure_wide_buffers(tiles, chunks, waits); if (rc) return rc; }
        *rows = wideH;
        return 0;
    }
    template <class K, int RBYTES>
    void launch_wide_scatter(uint32_t tiles, const K *kin, K *kout, uint32_t *vout, const uint32_t *n_ptr, uint32_t n_host, uint32_t shift,
                             uint32_t chunk_shift, const uint32_t *c, cudaStream_t s, const unsigned char *pin, unsigned char *pout, uint32_t pbytes,
                             uint32_t skip_invalid, uint32_t region_stride)
    {
        k_wide_scatter<K, RBYTES><<<tiles, OSW_THREADS, 0, s>>>(kin, kout, vout, n_ptr, n_host, shift, chunk_shift, wideH, wideC, c, pin, pout, pbytes, skip_invalid, region_stride);
    }
    // payload_in / payload_out (optional): payload_bytes-sized records that travel with the elements (multiple of 8 bytes)
    // ready_ctl: the producer of the keys (the tile pass) cleared it and filed the 16-bit rows of the wide tiles (TileArgs::wide_h16) --
    // in h16_rows when they do not live in this sorter (a pipelined handle keeps one set per segment in flight) -- and, without few_bins,
    // packed a rank with every key (TileArgs::pack_rank), by which k_wide_scatter_ranked places them. Null: k_wide_tile_hist counts.
    // list (ranked only): kout receives the bucket list of k_ffat_update_buckets (bkl_word; kin starts at the first position of a
    // range of fewer than BKL_RANGE_POS positions) instead of the slots; vout is not written. Without records travelling the ranked
    // pass writes the bucket list only.
    template <class K>
    int sort_wide(const K *kin, K *kout, uint32_t *vout, const uint32_t *n_ptr, uint32_t n_host, uint32_t cap, uint32_t shift,
                  cudaStream_t s, uint32_t *ready_ctl, const uint32_t **counts, const unsigned char *payload_in = nullptr,
                  unsigned char *payload_out = nullptr, uint32_t payload_bytes = 0, bool skip_invalid = false, uint32_t region_stride = 0, uint32_t few_bins = 0,
                  const uint16_t *h16_rows = nullptr, bool list = false)
    {
        if (payload_in && (payload_bytes == 0 || (payload_bytes & 7u))) return WFB_E_BADARG;
        CK(ctl.ensure(CTL_WORDS));
        const bool ranked = ready_ctl && !few_bins;
        const uint16_t *rows = h16_rows ? h16_rows : wideH;
        uint32_t tiles, chunk_shift, chunks;
        wide_geometry(cap, ranked, &tiles, &chunk_shift, &chunks);
        { int rc = ensure_wide_buffers(tiles, chunks, s); if (rc) return rc; }
        uint32_t *c = ready_ctl ? ready_ctl : ctl;
        if (!ready_ctl) { int rc = prepare_wide(c, s); if (rc) return rc; }
        if (ranked) { // first output position of every (chunk, digit) and (tile, digit) + digit counts
            CK(wideDone.ensure_zeroed(1, s));
            k_wide_tile_bases<<<chunks, OSW_THREADS, 0, s>>>(rows, tiles, chunk_shift, chunks, wideC, wideT, c, wideDone,
                                                             osr_group(tiles, payload_in != nullptr) == OSR_GROUP ? 2u : 0u); // (log2 OSR_GROUP)
        } else if (ready_ctl) { // a few bins (destinations): chunk sums + the global counts
            k_wide_chunk_sums16<<<chunks, OSW_THREADS, 0, s>>>(rows, tiles, chunk_shift, wideC, c);
        } else {
            CK(cudaMemsetAsync(wideC, 0, sizeof(uint32_t) * OSW_DIGITS * chunks, s));
            k_wide_tile_hist<K><<<tiles, OSW_THREADS, 0, s>>>(kin, n_ptr, n_host, shift, chunk_shift, wideH, wideC, c, skip_invalid ? 1u : 0u);
        }
        if (region_stride && few_bins && payload_in && few_bins <= 32 && (payload_bytes == 16 || payload_bytes == 24 || payload_bytes == 32 || payload_bytes == 64)) {
            // a few fixed-capacity regions (destination GPUs): ranks from ballots, records leave in runs
            const uint32_t *d32 = reinterpret_cast<const uint32_t *>(kin);
            static_assert(sizeof(K) == 4 || sizeof(K) == 8, "key width");
            if (sizeof(K) == 4) {
                switch (payload_bytes) {
                    case 16: k_shard_scatter<16><<<tiles, OSW_THREADS, 0, s>>>(d32, n_host, few_bins, chunk_shift, wideH, wideC, payload_in, payload_out, region_stride); break;
                    case 24: k_shard_scatter<24><<<tiles, OSW_THREADS, 0, s>>>(d32, n_host, few_bins, chunk_shift, wideH, wideC, payload_in, payload_out, region_stride); break;
                    case 32: k_shard_scatter<32><<<tiles, OSW_THREADS, 0, s>>>(d32, n_host, few_bins, chunk_shift, wideH, wideC, payload_in, payload_out, region_stride); break;
                    default: k_shard_scatter<64><<<tiles, OSW_THREADS, 0, s>>>(d32, n_host, few_bins, chunk_shift, wideH, wideC, payload_in, payload_out, region_stride); break;
                }
                CK(cudaGetLastError());
                launches += 2;
                *counts = c;
                return 0;
            }
        }
        if (ranked) {
            if (sizeof(K) != 4 || !kout || (payload_in ? !payload_out || region_stride : !list) || (list && n_host > BKL_RANGE_POS)) return WFB_E_UNSUPPORTED;
            if (!payload_in && osr_group(tiles, false) == OSR_GROUP) {
                CK(osr_smem_attr());
                k_wide_scatter_ranked<<<(tiles + OSR_GROUP - 1) / OSR_GROUP, OSW_THREADS, OSR_SMEM, s>>>(reinterpret_cast<const uint32_t *>(kin), reinterpret_cast<uint32_t *>(kout),
                                                                                                       n_host, shift, chunk_shift, tiles, rows, wideC, wideT);
            }
#define WFB_WSRT(RB_) k_wide_scatter_ranked_tile<RB_><<<tiles, OSW_THREADS, 0, s>>>(reinterpret_cast<const uint32_t *>(kin), reinterpret_cast<uint32_t *>(kout), list ? 1u : 0u, \
                                                                                  n_host, shift, chunk_shift, rows, wideC, wideT, payload_in, payload_out)
            else if (!payload_in) WFB_WSRT(0);
            else switch (payload_bytes) { // the records travel with their slots (bucketed exchange)
                case 16: WFB_WSRT(16); break; case 24: WFB_WSRT(24); break; case 32: WFB_WSRT(32); break; case 48: WFB_WSRT(48); break; case 64: WFB_WSRT(64); break;
                default: return WFB_E_UNSUPPORTED;
            }
#undef WFB_WSRT
            CK(cudaGetLastError());
            launches += 2;
            *counts = c;
            return 0;
        }
#define WFB_WS(RB_) launch_wide_scatter<K, RB_>(tiles, kin, kout, vout, n_ptr, n_host, shift, chunk_shift, c, s, payload_in, payload_out, payload_bytes, skip_invalid ? 1u : 0u, region_stride)
        if (!payload_in) WFB_WS(0);
        else switch (payload_bytes) {
            case 8: WFB_WS(8); break;   case 16: WFB_WS(16); break; case 24: WFB_WS(24); break; case 32: WFB_WS(32); break;
            case 48: WFB_WS(48); break; case 64: WFB_WS(64); break; default: WFB_WS(-1); break;
        }
#undef WFB_WS
        CK(cudaGetLastError());
        launches += 2;
        *counts = c;
        return 0;
    }

    template <class K>
    int sort(K *kA, K *kB, uint32_t *vA, uint32_t *vB, const uint32_t *n_ptr, uint32_t n_host, uint32_t cap, uint32_t passes,
             cudaStream_t s, const K **skeys, const uint32_t **svals, uint32_t *ready_ctl = nullptr, uint32_t *seg_first = nullptr, uint32_t seg_first_n = 0, uint32_t base_shift = 0)
    {
        // ready_ctl != nullptr: histograms already accumulated there by the producer of the keys (after prepare())
        const bool hist_ready = ready_ctl != nullptr;
        if (!hist_ready) CK(ctl.ensure(CTL_WORDS));
        uint32_t *const c = hist_ready ? ready_ctl : static_cast<uint32_t *>(ctl);
        const uint32_t TE = OS_THREADS * OS_ITEMS;
        const uint64_t state_words = static_cast<uint64_t>((cap + OS_THREADS * 4 - 1) / (OS_THREADS * 4)) * 256;
        CK(state.ensure_zeroed(state_words, s, s, state_words));
        passes = std::min<uint32_t>(std::max(1u, passes), OS_MAX_PASSES);
        const uint32_t tiles = std::max(1u, (cap + TE - 1) / TE);
        if (!hist_ready) {
            CK(cudaMemsetAsync(c, 0, sizeof(uint32_t) * (passes * 256 + passes), s));
            k_radix_ghist<K><<<std::min(tiles, static_cast<uint32_t>(g_num_sms) * 4u), 256, 0, s>>>(kA, n_ptr, n_host, passes, c, base_shift);
            launches++;
        }
        const K *kin = kA; const uint32_t *vin = nullptr;
        K *kout = kB; uint32_t *vout = vB;
        for (uint32_t p = 0; p < passes; p++) {
            epoch = (epoch + 1) & 0x3fffffffu; if (epoch == 0) epoch = 1;
            uint32_t *sf = (p + 1 == passes) ? seg_first : nullptr;
            k_onesweep_pass<K><<<tiles, OS_THREADS, 0, s>>>(kin, vin, kout, vout, n_ptr, n_host, p, passes, c, state, epoch, sf, seg_first_n, base_shift);
            kin = kout; vin = vout;
            if (kout == kB) { kout = kA; vout = vA; } else { kout = kB; vout = vB; }
        }
        CK(cudaGetLastError());
        launches += passes;
        *skeys = kin; *svals = vin;
        return 0;
    }
};

// ---- key tables that grow (WFB_KEYS_GROW) -----------------------------------------------------------------------------------
// The arrays one growth replaces. Every new array is allocated before any old one is freed, so that a failed allocation leaves the
// handle as it was.
struct GrowPlan {
    struct Array { void **ptr; size_t old_bytes, bytes; bool copy; int fill; bool counted; void *fresh; };
    std::vector<Array> arrays;
    // *p (old_bytes) becomes `bytes` bytes: the old ones copied when `copy`, the rest set to the byte `fill` (-1: uninitialised, as
    // create leaves it). counted: part of wfb_ffat_state_bytes
    template <class T> void add(T *&p, size_t old_bytes, size_t bytes, bool copy, int fill, bool counted = true)
    {
        arrays.push_back({reinterpret_cast<void **>(&p), old_bytes, bytes, copy, fill, counted, nullptr});
    }
    template <class T> T *fresh(T *const &p) const
    {
        for (const Array &a : arrays) if (a.ptr == reinterpret_cast<void *const *>(&p)) return static_cast<T *>(a.fresh);
        return nullptr;
    }
    int64_t grown_bytes() const { int64_t d = 0; for (const Array &a : arrays) if (a.counted) d += static_cast<int64_t>(a.bytes) - static_cast<int64_t>(a.old_bytes); return d; }
    int alloc()
    {
        for (Array &a : arrays)
            if (cudaMalloc(&a.fresh, a.bytes) != cudaSuccess) { cudaGetLastError(); release(); return WFB_E_CAPACITY; }
        return 0;
    }
    void release() { for (Array &a : arrays) { cudaFree(a.fresh); a.fresh = nullptr; } }
    int fill(cudaStream_t s)
    {
        for (Array &a : arrays) {
            const size_t keep = a.copy ? a.old_bytes : 0;
            if (keep) CK(cudaMemcpyAsync(a.fresh, *a.ptr, keep, cudaMemcpyDeviceToDevice, s));
            if (a.fill >= 0 && a.bytes > keep) CK(cudaMemsetAsync(static_cast<unsigned char *>(a.fresh) + keep, a.fill, a.bytes - keep, s));
        }
        return 0;
    }
    void commit() { for (Array &a : arrays) { cudaFree(*a.ptr); *a.ptr = a.fresh; a.fresh = nullptr; } }
};

// pinned words the growth check reads the key count and the error flags into, and the event it waits on
struct GrowCheck {
    uint32_t *host = nullptr; cudaEvent_t ev = nullptr;
    int init() { CK(cudaMallocHost(reinterpret_cast<void **>(&host), 2 * sizeof(uint32_t))); CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); return 0; }
    void destroy() { if (host) cudaFreeHost(host); if (ev) cudaEventDestroy(ev); host = nullptr; ev = nullptr; }
};

// The growth step of every handle kind, run after the pass that inserts the keys of a call. It reads the key count and the error
// flags (the one synchronisation growth adds, on growing handles only). When the pass raised KEYS_GROW_FLAG, the capacity becomes a
// power of two >= 2 * max(keys, capacity), but not beyond `ceiling` (a power of two) while the capacity is below it and the keys fit it:
// the largest capacity that keeps the handle's path (time-based and keyed-stateful handles: their only path; count-based: the bucket
// path). It is at most `limit` (else WFB_E_CAPACITY). add_state(plan, cap) lists the handle's own arrays sized by the capacity, the key
// table is rebuilt at the new size, and derive(cap, plan) recomputes what create derived from the capacity. *grew = true: the caller
// reruns its key-inserting pass (it has no other state than the inserts, which are idempotent), and so on until a pass raises no flag;
// every growth but the one that stops at the ceiling at least doubles the capacity.
template <class AddState, class Derive>
int grow_keys(FfatDev &ff, uint32_t key_bytes, GrowCheck &gc, uint32_t ceiling, uint32_t limit, cudaStream_t s, bool *grew, AddState add_state,
              Derive derive)
{
    *grew = false;
    CK(cudaMemcpyAsync(gc.host, ff.n_slots, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s)); // n_slots, err_flags (adjacent)
    CK(cudaEventRecord(gc.ev, s));
    CK(cudaEventSynchronize(gc.ev));
    if (!(gc.host[1] & KEYS_GROW_FLAG)) return 0;
    const uint32_t old = ff.max_keys;
    uint64_t cap = 1; while (cap < 2ull * std::max(gc.host[0], old)) cap <<= 1;
    if (cap > ceiling && old < ceiling && gc.host[0] <= ceiling) cap = ceiling; // (every slot handed out so far, < n_slots, fits)
    if (cap > limit) return WFB_E_CAPACITY;
    uint64_t entries = 1; while (entries < 2 * cap) entries <<= 1;
    GrowPlan plan;
    plan.add(ff.ht_keys, static_cast<size_t>(key_bytes) * (ff.ht_mask + 1ull), key_bytes * entries, false, 0xff);
    plan.add(ff.ht_slots, sizeof(uint32_t) * (ff.ht_mask + 1ull), sizeof(uint32_t) * entries, false, 0xff);
    plan.add(ff.slot_key, static_cast<size_t>(key_bytes) * old, static_cast<size_t>(key_bytes) * cap, true, -1);
    int rc = add_state(plan, static_cast<uint32_t>(cap)); if (rc) return rc;
    rc = plan.alloc(); if (rc) return rc;
    rc = plan.fill(s);
    if (!rc) {
        k_key_table_rebuild<<<grid_for(ff.ht_mask + 1, 256), 256, 0, s>>>(ff.ht_keys, ff.ht_slots, ff.ht_mask, plan.fresh(ff.ht_keys), plan.fresh(ff.ht_slots),
                                                                        static_cast<uint32_t>(entries - 1), plan.fresh(ff.slot_key), old, key_bytes / 8, ff.err_flags);
        rc = static_cast<int>(cudaGetLastError());
    }
    if (!rc) rc = static_cast<int>(cudaStreamSynchronize(s)); // (the old arrays are read until here)
    if (rc) { cudaStreamSynchronize(s); plan.release(); return rc; }
    plan.commit();
    ff.ht_mask = static_cast<uint32_t>(entries - 1); ff.max_keys = static_cast<uint32_t>(cap);
    rc = derive(static_cast<uint32_t>(cap), plan); if (rc) return rc;
    *grew = true;
    return 0;
}

} // namespace

struct wfb_engine {
    int prog = 0;
    const ProgramOps *ops = nullptr;
    std::vector<unsigned char> params; // the program's params_t used by key / reduce (zeros unless wfb_engine_set_params)
    const void *pp() const { return params.empty() ? nullptr : params.data(); }
    TileScratch ts;
    uint64_t launches = 0;
    // scratch of the per-batch keyed operators (sort buffers), grown on demand
    uint32_t key_bits = 64;
    Scratch<uint64_t> keysA, keysB;
    Scratch<uint32_t> idxA, idxB, destA, destB;
    Scratch<uint32_t> head, seg_begin;
    // wfb_shard_lift: lifted records / destinations of one segment, tile t owns positions [t*TILE, +TILE)
    Scratch<unsigned char> sh_lifted; Scratch<uint32_t> sh_dest, sh_ctl;
    // wfb_reduce_by_key_batches: element offset of every batch, first segment of every batch, segment total
    Scratch<uint32_t> rb_off, rb_first, rb_total;
    Scratch<uint32_t> rb_long; // segments folded by a warp; rb_total[1] = their number
    RadixSorter sorter;
    // Reduce_GPU over keys that are not integers: the order words of the keys (whi: two-word keys) and the permutation of the first sort
    Scratch<uint64_t> wlo, whi; Scratch<uint32_t> wperm;

    // the sort buffers, all of keysA's capacity (seg_begin: one more)
    int ensure_sort(uint32_t n, cudaStream_t s)
    {
        CK(keysA.ensure(n, s));
        const size_t cap = keysA.capacity();
        CK(keysB.ensure(n, s, cap)); CK(idxA.ensure(n, s, cap)); CK(idxB.ensure(n, s, cap));
        CK(destA.ensure(n, s, cap)); CK(destB.ensure(n, s, cap));
        CK(head.ensure(n, s, cap)); CK(seg_begin.ensure(n + 1ull, s, cap + 1));
        return 0;
    }
    // stable LSD radix sort of (keysA[i], i) by key over `bits` bits; returns the buffers holding the result
    int sort64(uint32_t n, uint32_t bits, cudaStream_t s, const uint64_t **skeys, const uint32_t **sidx)
    {
        const uint64_t before = sorter.launches;
        int rc = sorter.sort<uint64_t>(keysA, keysB, idxA, idxB, nullptr, n, n, (bits + 7) / 8, s, skeys, sidx);
        launches += sorter.launches - before;
        return rc;
    }
    // Keys that are not integers (after ensure_sort(n)): keysA[i] = (batch of i << 32) | dense rank of element i's key in the key order
    // (the rank alone when boff is null), so that the integer path that follows sorts 32 (+ batch) bits. The order words are sorted
    // LSD over the bits the key type has (8 * sizeof(key_t)), low word first, then the high word of a two-word key; equal neighbours
    // share a rank. `tuples` is the batch when `batches` is null.
    int rank_keys(const DevBatch *batches, const uint32_t *boff, uint32_t nb, const void *tuples, uint32_t n, cudaStream_t s)
    {
        const bool two = ops->key_bytes == 16;
        const uint32_t bits = 8u * ops->key_size, lo_bits = std::min(bits, 64u), hi_bits = two ? bits - 64u : 0u;
        const size_t wcap = std::max<size_t>(n, keysA.capacity());
        CK(wlo.ensure(n, s, wcap));
        if (two) { CK(whi.ensure(n, s, wcap)); CK(wperm.ensure(n, s, wcap)); }
        int rc = ops->key_order_words(batches, boff, nb, static_cast<const unsigned char *>(tuples), n, wlo, whi, s, pp()); if (rc) return rc;
        CK(cudaMemcpyAsync(keysA, wlo, sizeof(uint64_t) * n, cudaMemcpyDeviceToDevice, s));
        const uint64_t *sk; const uint32_t *perm;
        rc = sort64(n, lo_bits, s, &sk, &perm); if (rc) return rc;
        const uint32_t g = grid_for(n, 256);
        if (two) { // sort the high words in the order of the low words, then compose the two permutations
            CK(cudaMemcpyAsync(wperm, perm, sizeof(uint32_t) * n, cudaMemcpyDeviceToDevice, s));
            k_gather_u64<<<g, 256, 0, s>>>(whi, wperm, n, keysA);
            const uint32_t *p2;
            rc = sort64(n, hi_bits, s, &sk, &p2); if (rc) return rc;
            k_compose_perm<<<g, 256, 0, s>>>(wperm, p2, n, destA);
            perm = destA;
            launches += 2;
        }
        k_rank_heads<<<g, 256, 0, s>>>(wlo, whi, perm, n, head);
        k_scan_u32<<<1, 1024, 0, s>>>(head, head, n, nullptr);
        k_rank_scatter<<<g, 256, 0, s>>>(wlo, whi, perm, head, n, boff, nb, keysA);
        CK(cudaGetLastError());
        launches += 4;
        return 0;
    }
};

// per-segment scratch of one Ffat_Windows_GPU; two sets when the handle is pipelined (the ingest pass of segment k+1
// overlaps sort + update of segment k)
struct SegScratch {
    Scratch<uint32_t> slotsA, slotsB, posA, posB; // the segment's capacity in records: slotsA's. Bucket path: slotsB holds the bucket
                                                  // list (posA / posB are the full sort's and stay unallocated)
    Scratch<unsigned char> lifted, lifted_sorted;
    Scratch<uint32_t> batch_off; Scratch<DevBatch> d_batches;
    uint32_t *n_total = nullptr;
    Scratch<uint16_t> h16; // pipelined handles: this segment's own rows (the next segment's tile pass files its rows while this segment's
                           // partition still reads these)
    const unsigned char *lifted_src = nullptr; // records of this segment: `lifted`, or the caller's buffer (in-place ingest)
    uint32_t *seg_cnt = nullptr;          // per-slot item counts of the segment (max_keys)
    Scratch<Trigger> trig; uint32_t *n_trig = nullptr;
    uint32_t *n_heavy = nullptr;
    uint32_t *sort_ctl = nullptr;         // digit histograms + tickets of this segment's slot sort
    // pipelined mode: results of the segment wait here until the next call / flush delivers them
    Scratch<unsigned char> res; Scratch<uint64_t> res_ts; uint32_t *res_n = nullptr;
    cudaEvent_t ev_ingest = nullptr, ev_done = nullptr;
    bool pending = false;
    uint32_t nbatches = 0, total = 0;

    void destroy()
    {
        if (ev_ingest) cudaEventDestroy(ev_ingest);
        if (ev_done) cudaEventDestroy(ev_done);
    }
};

struct wfb_ffat {
    int prog = 0;
    const ProgramOps *ops = nullptr;
    std::vector<unsigned char> params; // the program's params_t used by key / lift / comb (zeros unless wfb_ffat_set_params)
    const void *pp() const { return params.empty() ? nullptr : params.data(); }
    FfatDev ff{};
    TileScratch ts;
    uint32_t sort_passes = 1;
    SegScratch seg[2];
    RadixSorter sorter;
    bool pipelined = false;
    uint64_t call_no = 0;
    cudaStream_t s2 = nullptr;            // pipelined mode: sort + update + window queries run here
    uint64_t launches = 0;
    size_t state_bytes = 0;
    int win_type = 0;
    // time-based windows (win_type 1): this handle is the front end (key table, rings of pending panes); the popped panes go to
    // `cb`, a count-based handle over the lifted program with window / slide in panes
    TbDev tb{};
    wfb_ffat *cb = nullptr;
    uint64_t tb_lateness = 0;
    Scratch<uint64_t> tb_kA, tb_kB; Scratch<uint32_t> tb_iA, tb_iB; // scratch of a batch (capacity in tuples: tb_kA's)
    Scratch<unsigned char> tb_lifted, tb_part;
    Scratch<unsigned char> tb_popped; Scratch<uint32_t> tb_popped_slots; // the popped panes (capacity in records: tb_popped's / result bytes)
    bool shares_slot_key = false;                   // back end of a time-based handle: ff.slot_key / ff.n_slots belong to the front end
    uint32_t *own_n_slots = nullptr;                // the allocation behind ff.n_slots / ff.err_flags of this handle
    Scratch<uint32_t> tb_head, tb_seg;
    uint32_t *tb_misc = nullptr;    // [0] n_segs [1] first_seg dummy [2] n_present [3] popped total [4] ignored [5] ring capacity needed [6] ignored before the batch (growing handles)
    GrowCheck growc;                // WFB_KEYS_GROW (ff.grow): the growth check after the key-inserting pass
    Scratch<uint32_t> mg_scratch;   // (internal, ffat_process_prebucketed) per-(bucket, sub-bucket, source) counts, their scan, run starts
    bool append_results = false;  // (internal, wfb_mg_flush) the next call's results follow the ones already in the output buffer
    bool buckets = true;          // one wide radix pass + per-bucket CTAs (<= 65536 keys); else the full sort + thread-per-key update
    uint32_t bucket_shift = 0;    // the wide pass partitions on (slot >> bucket_shift) & 1023
    bool bucket_move = false;     // WFB_BUCKET_MOVE=1: the wide pass also moves the lifted records into their buckets
    // optional per-phase timing (wfb_ffat_timing)
    bool timing = false;
    std::vector<cudaEvent_t> tev; // 4 events per recorded call
    uint32_t tev_used = 0;        // recorded calls since the last query
    static constexpr uint32_t TEV_MAX = 512;
    void mark(int which, cudaStream_t s)
    {
        if (!timing || tev_used >= TEV_MAX) return;
        cudaEventRecord(tev[tev_used * 4 + which], s);
    }
};

extern "C" {

int wfb_abi_version(void) { return WFB_ABI_VERSION; }

const char *wfb_error_string(int code)
{
    switch (code) {
    case 0: return "success";
    case WFB_E_BADARG: return "wfb: bad argument";
    case WFB_E_NOPROG: return "wfb: unknown program id";
    case WFB_E_CAPACITY: return "wfb: capacity exceeded (keys or results)";
    case WFB_E_NOGPU: return "wfb: no CUDA device (libwfb200 has no CPU fallback)";
    case WFB_E_UNSUPPORTED: return "wfb: not supported";
    }
    if (code > 0) return cudaGetErrorString(static_cast<cudaError_t>(code));
    return "wfb: unknown error";
}

int wfb_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int wfb_program_register(const void *ops, size_t ops_bytes)
{
    if (!ops || ops_bytes != sizeof(ProgramOps)) return WFB_E_BADARG;
    std::lock_guard<std::mutex> lock(registry_mutex());
    std::vector<ProgramOps> &t = registry();
    if (t.size() >= 4096) return WFB_E_CAPACITY;
    t.reserve(4096); // handles keep pointers into the table: never reallocate it
    t.push_back(*static_cast<const ProgramOps *>(ops));
    return static_cast<int>(t.size()) - 1;
}

int wfb_program_info(int prog, wfb_program_info_t *info)
{
    const ProgramOps *o = program(prog);
    if (!o) return WFB_E_NOPROG;
    if (!info) return WFB_E_BADARG;
    info->tuple_bytes = o->tuple_bytes; info->result_bytes = o->result_bytes; info->key_bytes = o->key_bytes; info->key_kind = o->key_kind;
    return 0;
}

// ---- engine -------------------------------------------------------------------------------------------------
int wfb_engine_create(wfb_engine_t **e, int prog)
{
    if (!e) return WFB_E_BADARG;
    const ProgramOps *o = program(prog);
    if (!o) return WFB_E_NOPROG;
    int rc = device_ready(); if (rc) return rc;
    wfb_engine *g = new (std::nothrow) wfb_engine();
    if (!g) return WFB_E_BADARG;
    g->prog = prog; g->ops = o;
    rc = g->ts.init(); if (rc) { delete g; return rc; }
    *e = g;
    return 0;
}

int wfb_engine_destroy(wfb_engine_t *e)
{
    if (!e) return 0;
    cudaDeviceSynchronize();
    e->ts.destroy();
    delete e;
    return 0;
}

uint64_t wfb_engine_launches(const wfb_engine_t *e) { return e ? e->launches : 0; }

int wfb_engine_set_params(wfb_engine_t *e, const void *params, size_t bytes)
{
    if (!e || !params || bytes != e->ops->params_bytes) return WFB_E_BADARG;
    e->params.assign(static_cast<const unsigned char *>(params), static_cast<const unsigned char *>(params) + bytes);
    return 0;
}

static int run_single(wfb_engine_t *e, int mode, const wfb_functors_t *f, const DevBatch &b, cudaStream_t s)
{
    const uint32_t num_tiles = tiles_of(b.n);
    int rc = e->ts.enter(s); if (rc) return rc;
    rc = e->ts.ensure_tiles(num_tiles); if (rc) return rc;
    TileArgs a; std::memset(&a, 0, sizeof(a));
    a.batches = nullptr; a.one = b; a.nbatches = 1; a.num_tiles = num_tiles;
    e->ts.next_launch(a);
    uint32_t grid = 0;
    const uint64_t sb = reinterpret_cast<uint64_t>(b.tuples);
    rc = e->ops->tile_pass(mode, a, f, num_tiles, s, &grid, sb, sb + static_cast<uint64_t>(b.n) * e->ops->tuple_bytes); if (rc) return rc;
    e->ts.launched(num_tiles, grid);
    e->launches++;
    return 0;
}

int wfb_map(wfb_engine_t *e, const wfb_functors_t *f, void *tuples, uint32_t n, void *stream)
{
    if (!e || !f || (!tuples && n)) return WFB_E_BADARG;
    if (n == 0) return 0;
    DevBatch b; std::memset(&b, 0, sizeof(b));
    b.tuples = static_cast<const unsigned char *>(tuples); b.out = static_cast<unsigned char *>(tuples); b.n = n;
    return run_single(e, MODE_MAP, f, b, static_cast<cudaStream_t>(stream));
}

int wfb_map_filter(wfb_engine_t *e, const wfb_functors_t *f, const void *tuples_in, const uint64_t *ts_in, uint32_t n,
                   void *tuples_out, uint64_t *ts_out, uint32_t *n_out_dev, void *stream)
{
    if (!e || !f || !n_out_dev || (n && (!tuples_in || !tuples_out))) return WFB_E_BADARG;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (n == 0) { CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t), s)); return 0; }
    DevBatch b; std::memset(&b, 0, sizeof(b));
    b.tuples = static_cast<const unsigned char *>(tuples_in); b.ts = ts_in;
    b.out = static_cast<unsigned char *>(tuples_out); b.ts_out = ts_in ? ts_out : nullptr; b.n_out = n_out_dev; b.n = n;
    return run_single(e, MODE_FILTER, f, b, s);
}

int wfb_map_filter_batches(wfb_engine_t *e, const wfb_functors_t *f, const wfb_batch_t *in_h, const wfb_batch_t *out_h, uint32_t nbatches,
                           uint32_t *n_out_dev, void *stream)
{
    if (!e || !f || !n_out_dev || (nbatches && (!in_h || !out_h))) return WFB_E_BADARG;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (nbatches == 0) return 0;
    int rc = e->ts.enter(s); if (rc) return rc;
    CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t) * nbatches, s)); // empty batches keep 0
    std::vector<DevBatch> hb; hb.reserve(nbatches);
    uint32_t tiles = 0; uint64_t span_begin = ~0ull, span_end = 0;
    for (uint32_t i = 0; i < nbatches; i++) {
        if (in_h[i].n == 0) continue;
        if (!in_h[i].tuples || !out_h[i].tuples) return WFB_E_BADARG;
        DevBatch b; std::memset(&b, 0, sizeof(b));
        b.tuples = static_cast<const unsigned char *>(in_h[i].tuples); b.ts = in_h[i].ts;
        b.out = static_cast<unsigned char *>(const_cast<void *>(out_h[i].tuples));
        b.ts_out = in_h[i].ts ? const_cast<uint64_t *>(out_h[i].ts) : nullptr;
        b.n_out = n_out_dev + i; b.n = in_h[i].n; b.tile_begin = tiles;
        tiles += tiles_of(b.n);
        const uint64_t p0 = reinterpret_cast<uint64_t>(b.tuples);
        span_begin = std::min(span_begin, p0); span_end = std::max(span_end, p0 + static_cast<uint64_t>(b.n) * e->ops->tuple_bytes);
        hb.push_back(b);
    }
    if (hb.empty()) return 0;
    rc = e->ts.ensure_tiles(tiles); if (rc) return rc;
    rc = e->ts.ensure_batches(static_cast<uint32_t>(hb.size())); if (rc) return rc;
    { int rc_ = e->ts.stage.h2d(e->ts.d_batches, hb.data(), sizeof(DevBatch) * hb.size(), s); if (rc_) return rc_; }
    TileArgs a; std::memset(&a, 0, sizeof(a));
    a.batches = e->ts.d_batches; a.nbatches = static_cast<uint32_t>(hb.size()); a.num_tiles = tiles; a.l2_hints = 1;
    e->ts.next_launch(a);
    uint32_t grid = 0;
    rc = e->ops->tile_pass(MODE_FILTER, a, f, tiles, s, &grid, span_begin, span_end); if (rc) return rc;
    e->ts.launched(tiles, grid);
    e->launches++;
    return 0;
}

int wfb_flatmap_batches(wfb_engine_t *e, const wfb_functors_t *f, const wfb_batch_t *in_h, const wfb_batch_t *out_h, uint32_t nbatches,
                        uint32_t max_per_tuple, uint32_t *n_out_dev, void *stream)
{
    if (!e || !f || !n_out_dev || max_per_tuple == 0 || (nbatches && (!in_h || !out_h))) return WFB_E_BADARG;
    if (!e->ops->flatmap) return WFB_E_UNSUPPORTED;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc = e->ts.enter(s); if (rc) return rc;
    std::vector<DevBatch> hb; hb.reserve(nbatches);
    uint32_t tiles = 0; uint64_t span_begin = ~0ull, span_end = 0;
    for (uint32_t i = 0; i < nbatches; i++) {
        if (in_h[i].n == 0) continue;
        if (!in_h[i].tuples || !out_h[i].tuples) return WFB_E_BADARG;
        if (static_cast<uint64_t>(in_h[i].n) * max_per_tuple >= (1ull << 31)) return WFB_E_BADARG; // (positions of a batch are 32-bit)
        DevBatch b; std::memset(&b, 0, sizeof(b));
        b.tuples = static_cast<const unsigned char *>(in_h[i].tuples); b.ts = in_h[i].ts;
        b.out = static_cast<unsigned char *>(const_cast<void *>(out_h[i].tuples));
        b.ts_out = in_h[i].ts ? const_cast<uint64_t *>(out_h[i].ts) : nullptr;
        b.n_out = n_out_dev + i; b.n = in_h[i].n; b.tile_begin = tiles;
        tiles += tiles_of(b.n);
        const uint64_t p0 = reinterpret_cast<uint64_t>(b.tuples);
        span_begin = std::min(span_begin, p0); span_end = std::max(span_end, p0 + static_cast<uint64_t>(b.n) * e->ops->tuple_bytes);
        hb.push_back(b);
    }
    CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t) * (nbatches + 1), s)); // empty batches keep 0; the drop counter starts at 0
    if (hb.empty()) return 0;
    rc = e->ts.ensure_tiles(tiles); if (rc) return rc;
    rc = e->ts.ensure_batches(static_cast<uint32_t>(hb.size())); if (rc) return rc;
    { int rc_ = e->ts.stage.h2d(e->ts.d_batches, hb.data(), sizeof(DevBatch) * hb.size(), s); if (rc_) return rc_; }
    TileArgs a; std::memset(&a, 0, sizeof(a));
    a.batches = e->ts.d_batches; a.nbatches = static_cast<uint32_t>(hb.size()); a.num_tiles = tiles; a.l2_hints = 1;
    a.max_per_tuple = max_per_tuple; a.n_total = n_out_dev + nbatches;
    e->ts.next_launch(a);
    uint32_t grid = 0;
    rc = e->ops->flatmap(a, f, tiles, s, &grid, span_begin, span_end); if (rc) return rc;
    e->ts.launched(tiles, grid);
    e->launches++;
    return 0;
}

int wfb_engine_set_key_bits(wfb_engine_t *e, uint32_t bits)
{
    if (!e || bits == 0 || bits > 64 || e->ops->key_kind != KEY_KIND_INTEGRAL) return WFB_E_BADARG;
    e->key_bits = bits;
    return 0;
}

// sort the batch's (key, index) pairs and derive the key segments; shared by reduce_by_key and keyby_group
static int keyed_prepare(wfb_engine_t *e, const void *tuples, uint32_t n, int32_t *map_idxs, int32_t *start_idxs, uint64_t *dist_keys,
                         uint32_t *n_keys_dev, cudaStream_t s, const uint32_t **sidx_out)
{
    int rc = e->ts.enter(s); if (rc) return rc;
    rc = e->ensure_sort(n, s); if (rc) return rc;
    const bool ranked = e->ops->key_kind != KEY_KIND_INTEGRAL; // (reduce_by_key only: keyby_group refuses such keys)
    if (ranked) rc = e->rank_keys(nullptr, nullptr, 1, tuples, n, s);
    else { rc = e->ops->extract_keys(static_cast<const unsigned char *>(tuples), n, e->keysA, nullptr, 1, s, e->pp()); e->launches++; }
    if (rc) return rc;
    const uint64_t *skeys; const uint32_t *sidx;
    rc = e->sort64(n, ranked ? 32u : e->key_bits, s, &skeys, &sidx); if (rc) return rc;
    const uint32_t g = grid_for(n, 256);
    k_seg_heads<<<g, 256, 0, s>>>(skeys, sidx, n, e->head, map_idxs);
    k_scan_u32<<<1, 1024, 0, s>>>(e->head, e->head, n, nullptr);
    k_seg_finish<<<g, 256, 0, s>>>(skeys, sidx, e->head, n, start_idxs, dist_keys, e->seg_begin, n_keys_dev);
    CK(cudaGetLastError());
    e->launches += 3;
    *sidx_out = sidx;
    return 0;
}

int wfb_reduce_by_key(wfb_engine_t *e, const void *tuples, const uint64_t *ts, uint32_t n,
                      void *out_tuples, uint64_t *out_ts, uint32_t *n_out_dev, void *stream)
{
    if (!e || !n_out_dev || (n && (!tuples || !out_tuples))) return WFB_E_BADARG;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (n == 0) { CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t), s)); return 0; }
    const uint32_t *sidx;
    int rc = keyed_prepare(e, tuples, n, nullptr, nullptr, nullptr, n_out_dev, s, &sidx); if (rc) return rc;
    rc = e->ops->reduce_segments(static_cast<const unsigned char *>(tuples), ts, sidx, e->seg_begin, n_out_dev,
                                 static_cast<unsigned char *>(out_tuples), ts ? out_ts : nullptr, n, s, e->pp());
    if (rc) return rc;
    e->launches++;
    return 0;
}

int wfb_reduce_by_key_batches(wfb_engine_t *e, const wfb_batch_t *in_h, const wfb_batch_t *out_h, uint32_t nbatches, uint32_t *n_out_dev,
                              void *stream)
{
    if (!e || !n_out_dev || (nbatches && (!in_h || !out_h))) return WFB_E_BADARG;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (nbatches == 0) return 0;
    uint32_t bbits = 0; while ((1ull << bbits) < nbatches) bbits++;
    const bool ranked = e->ops->key_kind != KEY_KIND_INTEGRAL; // keys replaced by their 32-bit rank (wfb_engine::rank_keys)
    const uint32_t key_bits = ranked ? 32u : e->key_bits;
    if (key_bits + bbits > 64) return WFB_E_BADARG;
    int rc = e->ts.enter(s); if (rc) return rc;
    CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t) * nbatches, s));
    std::vector<DevBatch> hb(nbatches);
    std::vector<uint32_t> boff(nbatches + 1);
    uint64_t total = 0;
    for (uint32_t i = 0; i < nbatches; i++) { // (empty batches keep their index: the composite key carries it)
        if (in_h[i].n && (!in_h[i].tuples || !out_h[i].tuples)) return WFB_E_BADARG;
        DevBatch b; std::memset(&b, 0, sizeof(b));
        b.tuples = static_cast<const unsigned char *>(in_h[i].tuples); b.ts = in_h[i].ts;
        b.out = static_cast<unsigned char *>(const_cast<void *>(out_h[i].tuples));
        b.ts_out = in_h[i].ts ? const_cast<uint64_t *>(out_h[i].ts) : nullptr;
        b.n_out = n_out_dev + i; b.n = in_h[i].n;
        hb[i] = b; boff[i] = static_cast<uint32_t>(total); total += b.n;
    }
    boff[nbatches] = static_cast<uint32_t>(total);
    if (total == 0) return 0;
    if (total > 0x7fffffffull) return WFB_E_BADARG;
    const uint32_t n = static_cast<uint32_t>(total);
    rc = e->ensure_sort(n, s); if (rc) return rc;
    rc = e->ts.ensure_batches(nbatches); if (rc) return rc;
    CK(e->rb_first.ensure(nbatches, s));
    CK(e->rb_off.ensure(nbatches + 1ull, s, e->rb_first.capacity() + 1));
    CK(e->rb_total.ensure(2));
    { int rc_ = e->ts.stage.h2d(e->ts.d_batches, hb.data(), sizeof(DevBatch) * nbatches, s); if (rc_) return rc_; }
    { int rc_ = e->ts.stage.h2d(e->rb_off, boff.data(), sizeof(uint32_t) * (nbatches + 1), s); if (rc_) return rc_; }
    CK(cudaMemsetAsync(e->rb_first, 0xff, sizeof(uint32_t) * nbatches, s));
    CK(cudaMemsetAsync(e->rb_total, 0, sizeof(uint32_t) * 2, s));
    CK(e->rb_long.ensure(n / RB_LONG + 1, s));
    const uint32_t kb = nbatches == 1 ? 64u : key_bits; // a single batch needs no composite key
    if (ranked) rc = e->rank_keys(e->ts.d_batches, e->rb_off, nbatches, nullptr, n, s);
    else rc = e->ops->extract_keys_batches(e->ts.d_batches, e->rb_off, nbatches, n, kb, e->keysA, s, e->pp());
    if (rc) return rc;
    const uint64_t *skeys; const uint32_t *sidx;
    const uint64_t before = e->sorter.launches;
    const uint32_t sort_bits = nbatches == 1 ? key_bits : key_bits + bbits;
    rc = e->sorter.sort<uint64_t>(e->keysA, e->keysB, e->idxA, e->idxB, nullptr, n, n, (sort_bits + 7) / 8, s, &skeys, &sidx); if (rc) return rc;
    const uint32_t tiles = (n + SEGT - 1) / SEGT;
    k_head_tile_counts<<<tiles, 256, 0, s>>>(skeys, n, e->head);
    k_scan_u32<<<1, 1024, 0, s>>>(e->head, e->head, tiles, nullptr);
    k_seg_finish_batches<<<tiles, 256, 0, s>>>(skeys, n, kb, e->head, e->seg_begin, e->rb_first, e->rb_total);
    k_batch_seg_counts<<<1, 32, 0, s>>>(e->rb_first, nbatches, e->rb_total, e->ts.d_batches);
    CK(cudaGetLastError());
    rc = e->ops->reduce_segments_batches(e->ts.d_batches, e->rb_off, skeys, sidx, e->seg_begin, e->rb_first, e->rb_total, kb, n, e->rb_long,
                                         e->rb_total + 1, s, e->pp());
    if (rc) return rc;
    e->launches += 7 + (e->sorter.launches - before);
    return 0;
}

int wfb_reduce_all(wfb_engine_t *e, const void *tuples, const uint64_t *ts, uint32_t n, void *out_tuple, uint64_t *out_ts, void *stream)
{
    if (!e || !out_tuple || (n && !tuples)) return WFB_E_BADARG;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc = e->ts.enter(s); if (rc) return rc;
    rc = e->ops->reduce_all(static_cast<const unsigned char *>(tuples), ts, n, static_cast<unsigned char *>(out_tuple), out_ts, s, e->pp());
    if (rc) return rc;
    e->launches++;
    return 0;
}

int wfb_keyby_group(wfb_engine_t *e, const void *tuples, uint32_t n, int32_t *start_idxs, int32_t *map_idxs, uint64_t *dist_keys,
                    uint32_t *n_keys_dev, void *stream)
{
    if (!e || !n_keys_dev || (n && (!tuples || !start_idxs || !map_idxs || !dist_keys))) return WFB_E_BADARG;
    if (e->ops->key_kind != KEY_KIND_INTEGRAL) return WFB_E_UNSUPPORTED; // dist_keys holds 8-byte integer keys
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (n == 0) { CK(cudaMemsetAsync(n_keys_dev, 0, sizeof(uint32_t), s)); return 0; }
    const uint32_t *sidx;
    return keyed_prepare(e, tuples, n, map_idxs, start_idxs, dist_keys, n_keys_dev, s, &sidx);
}

int wfb_shard_by_key(wfb_engine_t *e, const void *tuples, const uint64_t *ts, uint32_t n, uint32_t num_shards,
                     void *out_tuples, uint64_t *out_ts, uint32_t *seg_off_dev, void *stream)
{
    if (!e || !seg_off_dev || num_shards == 0 || num_shards > 256 || (n && (!tuples || !out_tuples))) return WFB_E_BADARG;
    if (e->ops->key_kind != KEY_KIND_INTEGRAL) return WFB_E_UNSUPPORTED; // shard = key % num_shards
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (n == 0) { CK(cudaMemsetAsync(seg_off_dev, 0, sizeof(uint32_t) * (num_shards + 1), s)); return 0; }
    int rc = e->ts.enter(s); if (rc) return rc;
    rc = e->ensure_sort(n, s); if (rc) return rc;
    rc = e->ops->extract_keys(static_cast<const unsigned char *>(tuples), n, nullptr, e->destA, num_shards, s, e->pp()); if (rc) return rc;
    const uint32_t *sdest, *perm;
    const uint64_t before = e->sorter.launches;
    rc = e->sorter.sort<uint32_t>(e->destA, e->destB, e->idxA, e->idxB, nullptr, n, n, 1, s, &sdest, &perm); if (rc) return rc;
    k_shard_offsets<<<1, 288, 0, s>>>(sdest, n, num_shards, seg_off_dev);
    CK(cudaGetLastError());
    rc = e->ops->gather(static_cast<const unsigned char *>(tuples), ts, perm, n, static_cast<unsigned char *>(out_tuples),
                        ts ? out_ts : nullptr, s);
    if (rc) return rc;
    e->launches += 3 + (e->sorter.launches - before);
    return 0;
}

// bucketed mode (wfb_mg_*): shard_slots != 0 -- the partition is the full 1024-bin one on the destination-major virtual slot
// (dest * shard_slots + key / num_shards) >> shift: out_regions gets the records bin after bin (capacity: the segment's positions),
// out_slots their virtual slots, bins_ctl (OSW_DIGITS + 1 words, the caller's) the bin sizes, counts_dev the records per destination
static int shard_lift_impl(wfb_engine_t *e, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches, uint32_t num_shards,
                           void *out_regions, uint32_t region_capacity, uint32_t *counts_dev, void *stream,
                           uint32_t shard_slots, uint32_t shard_keys, uint32_t shift, uint32_t *out_slots, uint32_t *bins_ctl,
                           uint64_t *send_meta = nullptr, uint64_t watermark = 0);

int wfb_shard_lift(wfb_engine_t *e, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches, uint32_t num_shards,
                   void *out_regions, uint32_t region_capacity, uint32_t *counts_dev, void *stream)
{
    return shard_lift_impl(e, pre, batches_h, nbatches, num_shards, out_regions, region_capacity, counts_dev, stream, 0, 0, 0, nullptr, nullptr);
}

static int shard_lift_impl(wfb_engine_t *e, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches, uint32_t num_shards,
                           void *out_regions, uint32_t region_capacity, uint32_t *counts_dev, void *stream,
                           uint32_t shard_slots, uint32_t shard_keys, uint32_t shift, uint32_t *out_slots, uint32_t *bins_ctl,
                           uint64_t *send_meta, uint64_t watermark)
{
    // Map -> Filter -> lift in one streaming pass (no compaction chain: tile t owns positions [t*TILE, +TILE)), then one
    // stable partition pass on the destination (key % num_shards) that moves the lifted records into the shard regions.
    if (!e || !counts_dev || !out_regions || num_shards == 0 || num_shards > MAX_SHARDS || (nbatches && !batches_h)) return WFB_E_BADARG;
    if (e->ops->key_kind != KEY_KIND_INTEGRAL) return WFB_E_UNSUPPORTED; // shard = key % num_shards
    const bool bucketed = shard_slots != 0;
    if (bucketed && (!out_slots || !bins_ctl || (shard_slots & (shard_slots - 1)) || static_cast<uint64_t>(num_shards) * shard_slots > 65536u ||
                     shard_keys > shard_slots || (shard_slots >> shift) == 0)) return WFB_E_BADARG;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc = e->ts.enter(s); if (rc) return rc;
    CK(cudaMemsetAsync(counts_dev, 0, sizeof(uint32_t) * (MAX_SHARDS + 1), s));
    std::vector<DevBatch> hb; hb.reserve(nbatches);
    uint64_t total = 0; uint32_t tiles = 0; uint64_t span_begin = ~0ull, span_end = 0;
    for (uint32_t i = 0; i < nbatches; i++) {
        if (batches_h[i].n == 0) continue;
        if (!batches_h[i].tuples) return WFB_E_BADARG;
        DevBatch b; std::memset(&b, 0, sizeof(b));
        b.tuples = static_cast<const unsigned char *>(batches_h[i].tuples); b.watermark = batches_h[i].watermark;
        b.n = batches_h[i].n; b.tile_begin = tiles;
        tiles += tiles_of(b.n); total += b.n;
        const uint64_t p0 = reinterpret_cast<uint64_t>(b.tuples);
        span_begin = std::min(span_begin, p0); span_end = std::max(span_end, p0 + static_cast<uint64_t>(b.n) * e->ops->tuple_bytes);
        hb.push_back(b);
    }
    if (total == 0) { if (bucketed) CK(cudaMemsetAsync(bins_ctl, 0, sizeof(uint32_t) * (OSW_DIGITS + 1), s)); return 0; }
    const uint64_t positions = static_cast<uint64_t>(tiles) * TILE;
    if (positions > 0x7fffffffull || (bucketed && positions > region_capacity)) return WFB_E_BADARG;
    nbatches = static_cast<uint32_t>(hb.size());
    const size_t RB = e->ops->result_bytes;
    CK(e->sh_dest.ensure(positions, s));
    CK(e->sh_lifted.ensure(positions * RB, s, e->sh_dest.capacity() * RB));
    CK(e->sh_ctl.ensure(RadixSorter::CTL_WORDS));
    rc = e->ts.ensure_tiles(tiles); if (rc) return rc;
    rc = e->ts.ensure_batches(nbatches); if (rc) return rc;
    { int rc_ = e->ts.stage.h2d(e->ts.d_batches, hb.data(), sizeof(DevBatch) * nbatches, s); if (rc_) return rc_; }
    uint32_t *ctl = bucketed ? bins_ctl : e->sh_ctl;
    rc = RadixSorter::prepare_wide(ctl, s); if (rc) return rc;
    TileArgs a; std::memset(&a, 0, sizeof(a));
    a.batches = e->ts.d_batches; a.nbatches = nbatches; a.num_tiles = tiles;
    a.lifted = e->sh_lifted; a.slots = e->sh_dest; a.nshards = num_shards; a.sparse = 1; a.l2_hints = 1;
    a.sort_ctl = ctl; a.sort_passes = 1; a.sort_shift = 0; a.sort_dbits = OSW_BITS;
    if (bucketed) { a.shard_slots = shard_slots; a.shard_keys = shard_keys; a.shard_err = counts_dev + MAX_SHARDS; a.sort_shift = shift; a.pack_rank = 1; }
    // the tile pass claims whole wide tiles and files the per-tile destination counts itself (no counting pass in the partition)
    rc = e->sorter.ensure_wide(static_cast<uint32_t>(positions), s, &a.wide_h16); if (rc) return rc;
    a.tiles_per_ticket = OSW_TILE_POS / TILE; a.sort_ctl = nullptr;
    const uint32_t claims = (tiles + a.tiles_per_ticket - 1) / a.tiles_per_ticket;
    e->ts.next_launch(a);
    uint32_t grid = 0;
    rc = e->ops->tile_pass(MODE_INGEST, a, pre ? static_cast<const void *>(pre) : e->pp(), claims, s, &grid, span_begin, span_end); if (rc) return rc;
    e->ts.launched(claims, grid);
    e->launches++;
    const uint32_t *counts = nullptr;
    const uint64_t before = e->sorter.launches;
    if (bucketed) {
        rc = e->sorter.sort_wide<uint32_t>(e->sh_dest, out_slots, nullptr, nullptr, static_cast<uint32_t>(positions), static_cast<uint32_t>(positions), shift, s,
                                           ctl, &counts, e->sh_lifted, static_cast<unsigned char *>(out_regions), static_cast<uint32_t>(RB), true);
        if (rc) return rc;
        k_shard_bin_counts<<<1, 32 * MAX_SHARDS, 0, s>>>(counts, num_shards, shard_slots >> shift, counts_dev, send_meta, watermark);
    } else {
        rc = e->sorter.sort_wide<uint32_t>(e->sh_dest, nullptr, nullptr, nullptr, static_cast<uint32_t>(positions), static_cast<uint32_t>(positions), 0, s,
                                           e->sh_ctl, &counts, e->sh_lifted, static_cast<unsigned char *>(out_regions), static_cast<uint32_t>(RB), true,
                                           region_capacity, num_shards);
        if (rc) return rc;
        k_shard_counts<<<1, 32, 0, s>>>(counts, num_shards, region_capacity, counts_dev);
    }
    CK(cudaGetLastError());
    e->launches += e->sorter.launches - before + 1;
    return 0;
}

// ---- Ffat_Windows_GPU ------------------------------------------------------------------------------------------
static uint64_t gcd_u64(uint64_t a, uint64_t b) { while (b) { uint64_t t = a % b; a = b; b = t; } return a; }

// ---- keyed-stateful Map_GPU / Filter_GPU ---------------------------------------------------------------------------------
} // extern "C" (the struct below is C++)
struct wfb_kstate {
    int prog = 0;
    const ProgramOps *ops = nullptr;
    FfatDev ff{};                 // key table only (dense or open addressing)
    unsigned char *states = nullptr;
    RadixSorter sorter;
    bool buckets = true;          // at most 65536 keys: buckets of at most 64 keys (k_ks_apply); else a full sort (k_ks_apply_runs)
    uint32_t bucket_shift = 0, sort_passes = 0;
    Scratch<DevBatch> d_batches; Scratch<uint32_t> d_boff, rank_start; // capacity in batches: d_batches'
    Scratch<uint32_t> slotsA, slotsB, posA, posB, tile_cnt;           // capacity in tuples per call: slotsA's
    Scratch<unsigned char> keep;
    uint64_t launches = 0;
    PinnedStage stage;
    GrowCheck growc;              // WFB_KEYS_GROW (ff.grow)
    StreamOrder order;            // a call on another stream waits for the previous call: the scratch and the states are shared
    std::mutex mu;                // the replicas of an operator share the handle: one call at a time (the reference's spinlock)
};
extern "C" {

// what the key capacity decides: up to 65536 keys, 1024 buckets of at most 64 keys; above, a full sort by slot over 8-bit passes with
// 8·passes > log2(capacity), so that the low bits of INVALID_SLOT sort behind every real slot instead of aliasing one
static void kstate_derive_paths(wfb_kstate *h, uint32_t cap)
{
    uint32_t bits = 0; while ((1ull << bits) < cap) bits++;
    h->buckets = bits <= OSW_BITS + 6;
    h->bucket_shift = bits > OSW_BITS ? bits - OSW_BITS : 0;
    h->sort_passes = bits / 8 + 1;
}

int wfb_kstate_create(wfb_kstate_t **hh, int prog, uint32_t max_keys, uint32_t flags)
{
    if (!hh || max_keys == 0) return WFB_E_BADARG;
    const ProgramOps *o = program(prog);
    if (!o) return WFB_E_NOPROG;
    if (o->state_bytes == 0) return WFB_E_UNSUPPORTED; // the program has no state_t / stateful functors
    if ((flags & WFB_FFAT_DENSE_KEYS) && o->key_kind != KEY_KIND_INTEGRAL) return WFB_E_BADARG; // dense keys are integers
    if ((flags & WFB_KEYS_GROW) && (flags & WFB_FFAT_DENSE_KEYS)) return WFB_E_BADARG;       // (slot = key: nothing to grow)
    if (max_keys > (1u << 30)) return WFB_E_UNSUPPORTED;  // (the count-based limit)
    int rc = device_ready(); if (rc) return rc;
    wfb_kstate *h = new (std::nothrow) wfb_kstate();
    if (!h) return WFB_E_BADARG;
    h->prog = prog; h->ops = o;
    kstate_derive_paths(h, max_keys);
    FfatDev &ff = h->ff;
    ff.max_keys = max_keys; ff.dense = (flags & WFB_FFAT_DENSE_KEYS) ? 1u : 0u;
    rc = h->order.init(); if (rc) { wfb_kstate_destroy(h); return rc; }
    if (flags & WFB_KEYS_GROW) { ff.grow = 1; rc = h->growc.init(); if (rc) { wfb_kstate_destroy(h); return rc; } }
    uint32_t cap = 1; while (cap < 2ull * max_keys) cap <<= 1;
    ff.ht_mask = cap - 1;
#define ALLOC(ptr, bytes) do { cudaError_t e_ = cudaMalloc(reinterpret_cast<void **>(&(ptr)), (bytes)); if (e_ != cudaSuccess) { wfb_kstate_destroy(h); return static_cast<int>(e_); } } while (0)
    if (!ff.dense) {
        ALLOC(ff.ht_keys, static_cast<size_t>(o->key_bytes) * cap); ALLOC(ff.ht_slots, sizeof(uint32_t) * cap);
        CK(cudaMemset(ff.ht_keys, 0xff, static_cast<size_t>(o->key_bytes) * cap)); CK(cudaMemset(ff.ht_slots, 0xff, sizeof(uint32_t) * cap));
    }
    ALLOC(ff.n_slots, sizeof(uint32_t) * 4); ff.err_flags = ff.n_slots + 1;
    CK(cudaMemset(ff.n_slots, 0, sizeof(uint32_t) * 4));
    ALLOC(ff.slot_key, static_cast<size_t>(o->key_bytes) * max_keys);
    ALLOC(h->states, static_cast<size_t>(o->state_bytes) * max_keys);
    CK(cudaMemset(h->states, 0, static_cast<size_t>(o->state_bytes) * max_keys)); // state_t(): zero-initialised
#undef ALLOC
    *hh = h;
    return 0;
}

int wfb_kstate_destroy(wfb_kstate_t *h)
{
    if (!h) return 0;
    cudaDeviceSynchronize();
    cudaFree(h->ff.ht_keys); cudaFree(h->ff.ht_slots); cudaFree(h->ff.n_slots); cudaFree(h->ff.slot_key); cudaFree(h->states);
    h->stage.destroy(); h->growc.destroy(); h->order.destroy();
    delete h;
    cudaGetLastError();
    return 0;
}

uint32_t wfb_kstate_key_capacity(const wfb_kstate_t *h) { return h ? h->ff.max_keys : 0; }

static int kstate_run(wfb_kstate_t *h, const wfb_functors_t *f, const wfb_batch_t *in_h, const wfb_batch_t *out_h, uint32_t nbatches,
                      uint32_t *n_out_dev, bool filter, cudaStream_t s)
{
    if (!h || !f || (nbatches && !in_h) || (filter && (!out_h || !n_out_dev))) return WFB_E_BADARG;
    if (nbatches == 0) return 0;
    std::lock_guard<std::mutex> lock(h->mu);
    int rc = h->order.enter(s); if (rc) return rc;
    if (filter) CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t) * nbatches, s));
    std::vector<DevBatch> hb(nbatches);
    std::vector<uint32_t> boff(nbatches + 1);
    uint64_t total = 0;
    for (uint32_t i = 0; i < nbatches; i++) {
        if (in_h[i].n && (!in_h[i].tuples || (filter && !out_h[i].tuples))) return WFB_E_BADARG;
        DevBatch b; std::memset(&b, 0, sizeof(b));
        b.tuples = static_cast<const unsigned char *>(in_h[i].tuples); b.ts = in_h[i].ts; b.n = in_h[i].n;
        if (filter) {
            b.out = static_cast<unsigned char *>(const_cast<void *>(out_h[i].tuples));
            b.ts_out = in_h[i].ts ? const_cast<uint64_t *>(out_h[i].ts) : nullptr;
            b.n_out = n_out_dev + i;
        }
        hb[i] = b; boff[i] = static_cast<uint32_t>(total); total += b.n;
    }
    boff[nbatches] = static_cast<uint32_t>(total);
    if (total == 0) return 0;
    if (total > 0x7fffffffull) return WFB_E_BADARG;
    const uint32_t n = static_cast<uint32_t>(total);
    CK(h->d_batches.ensure(nbatches, s));
    const size_t bcap = h->d_batches.capacity();
    CK(h->d_boff.ensure(nbatches + 1ull, s, bcap + 1)); CK(h->rank_start.ensure(nbatches + 1ull, s, bcap + 1));
    CK(h->slotsA.ensure(n, s));
    const size_t cap = h->slotsA.capacity();
    CK(h->slotsB.ensure(n, s, cap)); CK(h->posA.ensure(n, s, cap)); CK(h->posB.ensure(n, s, cap)); CK(h->keep.ensure(n, s, cap));
    const size_t cnt_cap = (cap + SEGT - 1) / SEGT + 1;
    CK(h->tile_cnt.ensure(cnt_cap, s, cnt_cap));
    { int rc_ = h->stage.h2d(h->d_batches, hb.data(), sizeof(DevBatch) * nbatches, s); if (rc_) return rc_; }
    { int rc_ = h->stage.h2d(h->d_boff, boff.data(), sizeof(uint32_t) * (nbatches + 1), s); if (rc_) return rc_; }
    // 1. slots; 2. one wide partition pass into 1024 buckets of consecutive slots; 3. per-bucket CTAs, one thread per key
    // (more than 65536 keys: 2. a stable sort by slot; 3. one thread per run of a slot)
    rc = h->ops->ks_slots(h->d_batches, h->d_boff, nbatches, n, h->ff, h->slotsA, s, f); if (rc) return rc;
    for (bool grew = h->ff.grow != 0; grew; ) { // (a growing handle stops at 65536 keys, the last capacity of the bucket path, on its way up)
        rc = grow_keys(h->ff, h->ops->key_bytes, h->growc, 1u << (OSW_BITS + 6), 1u << 30, s, &grew,
                       [h](GrowPlan &plan, uint32_t cap) {
                           const size_t sb = h->ops->state_bytes;
                           plan.add(h->states, sb * h->ff.max_keys, sb * cap, true, 0); // state_t(): zero-initialised
                           return 0;
                       },
                       [h](uint32_t cap, const GrowPlan &) { kstate_derive_paths(h, cap); return 0; });
        if (rc) return rc;
        if (grew) { rc = h->ops->ks_slots(h->d_batches, h->d_boff, nbatches, n, h->ff, h->slotsA, s, f); if (rc) return rc; h->launches += 2; }
    }
    const uint64_t before = h->sorter.launches;
    if (h->buckets) {
        const uint32_t *counts = nullptr;
        rc = h->sorter.sort_wide<uint32_t>(h->slotsA, h->slotsB, h->posB, nullptr, n, n, h->bucket_shift, s, nullptr, &counts, nullptr, nullptr, 0, true);
        if (rc) return rc;
        rc = h->ops->ks_apply(filter ? 1 : 0, h->ff, h->d_batches, h->d_boff, nbatches, h->slotsB, h->posB, counts, h->bucket_shift, h->states,
                              h->keep, s, f);
    } else {
        const uint32_t *sorted_slots, *sorted_pos;
        rc = h->sorter.sort<uint32_t>(h->slotsA, h->slotsB, h->posA, h->posB, nullptr, n, n, h->sort_passes, s, &sorted_slots, &sorted_pos);
        if (rc) return rc;
        rc = h->ops->ks_apply_runs(filter ? 1 : 0, h->ff, h->d_batches, h->d_boff, nbatches, n, sorted_slots, sorted_pos, h->states, h->keep, s, f);
    }
    if (rc) return rc;
    h->launches += 2 + (h->sorter.launches - before);
    if (filter) { // stable per-batch compaction by the keep flags
        const uint32_t tiles = (n + SEGT - 1) / SEGT;
        k_flag_tile_counts<<<tiles, 256, 0, s>>>(h->keep, n, h->tile_cnt);
        k_scan_u32<<<1, 1024, 0, s>>>(h->tile_cnt, h->tile_cnt, tiles, nullptr);
        k_flag_batch_starts<<<(nbatches + 1 + 127) / 128, 128, 0, s>>>(h->keep, h->tile_cnt, h->d_boff, nbatches, n, h->rank_start, h->d_batches);
        k_flag_batch_counts<<<(nbatches + 127) / 128, 128, 0, s>>>(h->rank_start, nbatches, h->d_batches);
        CK(cudaGetLastError());
        rc = h->ops->flag_scatter(h->keep, h->tile_cnt, h->d_boff, nbatches, n, h->rank_start, h->d_batches, s); if (rc) return rc;
        h->launches += 5;
    }
    return 0;
}

int wfb_map_stateful(wfb_kstate_t *h, const wfb_functors_t *f, const wfb_batch_t *batches_h, uint32_t nbatches, void *stream)
{
    return kstate_run(h, f, batches_h, nullptr, nbatches, nullptr, false, static_cast<cudaStream_t>(stream));
}

int wfb_filter_stateful(wfb_kstate_t *h, const wfb_functors_t *f, const wfb_batch_t *in_h, const wfb_batch_t *out_h, uint32_t nbatches,
                        uint32_t *n_out_dev, void *stream)
{
    return kstate_run(h, f, in_h, out_h, nbatches, n_out_dev, true, static_cast<cudaStream_t>(stream));
}

static int ffat_process_cb_impl(wfb_ffat_t *h, const void *pre, const wfb_batch_t *batches_h, uint32_t nbatches, void *out_results, uint64_t *out_ts,
                                uint32_t out_capacity, uint32_t *n_out_dev, void *stream, const uint32_t *ext_slots);

// ---- time-based windows: front-end handle + count-based back end over the lifted program ------------------------------------
// id of the lifted variant of a program (LiftedOf<P>, registered on first use)
static int lifted_program_of(int prog)
{
    static std::vector<int> cache; // by program id
    static std::mutex cache_mutex;
    const ProgramOps *o = program(prog);
    if (!o || !o->lifted_ops) return -1;
    std::lock_guard<std::mutex> lock(cache_mutex);
    if (static_cast<size_t>(prog) < cache.size() && cache[prog] > 0) return cache[prog];
    const int id = wfb_program_register(o->lifted_ops(), sizeof(ProgramOps));
    if (id < 0) return id;
    if (cache.size() <= static_cast<size_t>(prog)) cache.resize(prog + 1, 0);
    cache[prog] = id;
    return id;
}

// what create derives from the key capacity: the sort passes over the slots and the bucket / onesweep path. The full sort takes
// 8·passes > log2(capacity) bits, so that the low bits of INVALID_SLOT (an item whose key found no slot) sort behind every real slot
// instead of aliasing the last one (at a capacity of exactly 2^24, three passes would see 0xffffff = slot 2^24 - 1)
static void ffat_derive_paths(wfb_ffat *h)
{
    uint32_t bits = 0; while ((1ull << bits) < h->ff.max_keys) bits++;
    h->sort_passes = bits / 8 + 1;
    h->bucket_shift = bits > OSW_BITS ? bits - OSW_BITS : 0;
    // bucket path: every bucket holds at most BK_KEYS keys, the pane length fits 32 bits and the program has a bucket kernel (a
    // result_t above 160 bytes has none: bk_fits)
    h->buckets = (1u << h->bucket_shift) <= BK_KEYS && h->ff.pane < (1ull << 32) && h->ops->ffat_buckets != nullptr;
}

// deferred window groups a segment of seg_cap records can fire: one per slide * Nb records, and one more per key
static uint32_t ffat_trig_cap(const wfb_ffat *h, uint32_t seg_cap, uint32_t keys)
{
    const uint64_t per_group = std::max<uint64_t>(1, h->ff.slide * h->ff.nb);
    return static_cast<uint32_t>(std::min<uint64_t>(seg_cap / per_group + keys + 1, 0x7fffffffull));
}

// growth of a count-based handle (also the back end of a time-based one) to `cap` keys: its per-key arrays, tails as create leaves
// them (slot-major: the state of slot s stays at s), then what create derives from the capacity
static void ffat_plan_state(wfb_ffat *h, GrowPlan &plan, uint32_t cap)
{
    FfatDev &ff = h->ff;
    const size_t old = ff.max_keys, RB = h->ops->result_bytes, tree = (2ull * ff.n_leaves - 1) * RB;
    plan.add(ff.cnt, sizeof(uint64_t) * old, sizeof(uint64_t) * cap, true, 0);
    plan.add(ff.acc, RB * old, RB * cap, true, 0);
    plan.add(ff.tree, tree * old, tree * cap, true, 0);
    plan.add(ff.seg_off, sizeof(uint32_t) * (old + 1), sizeof(uint32_t) * (cap + 1ull), true, 0xff);
    plan.add(ff.heavy, sizeof(uint32_t) * old, sizeof(uint32_t) * cap, false, -1);
    SegScratch &g = h->seg[0]; // (growing handles are not pipelined: one segment scratch)
    plan.add(g.seg_cnt, sizeof(uint32_t) * old, sizeof(uint32_t) * cap, false, 0); // (a rerun pass counts the segment's items again)
}
static void ffat_derive(wfb_ffat *h, uint32_t cap)
{
    h->ff.max_keys = cap;
    ffat_derive_paths(h); // (the rerun pass sizes the window groups for the new capacity: ffat_ensure_segment)
}
static int ffat_grow(wfb_ffat *h, cudaStream_t s, bool *grew)
{
    return grow_keys(h->ff, h->ops->key_bytes, h->growc, BK_KEYS << OSW_BITS, 1u << 30, s, grew,
                     [h](GrowPlan &plan, uint32_t cap) { ffat_plan_state(h, plan, cap); return 0; },
                     [h](uint32_t cap, const GrowPlan &plan) { ffat_derive(h, cap); h->state_bytes += plan.grown_bytes(); return 0; });
}

// growth of a time-based front end: its rings of pending panes and per-key pane bookkeeping, and its count-based back end (which
// leaves the bucket path above 65536 keys, as a count-based handle does)
static int tb_grow(wfb_ffat *h, cudaStream_t s, bool *grew)
{
    return grow_keys(h->ff, h->ops->key_bytes, h->growc, BK_KEYS << OSW_BITS, 1u << 30, s, grew,
        [h](GrowPlan &plan, uint32_t cap) {
            TbDev &tb = h->tb;
            const size_t old = h->ff.max_keys, RB = h->ops->result_bytes;
            if (static_cast<uint64_t>(tb.capq) * cap * RB > (32ull << 30)) return WFB_E_CAPACITY; // (the guard of tb_create)
            plan.add(tb.first, sizeof(uint64_t) * old, sizeof(uint64_t) * cap, true, 0);
            plan.add(tb.num, sizeof(uint32_t) * old, sizeof(uint32_t) * cap, true, 0);
            plan.add(tb.num_new, sizeof(uint32_t) * old, sizeof(uint32_t) * cap, false, -1);
            plan.add(tb.trig, sizeof(uint64_t) * old, sizeof(uint64_t) * cap, true, -1); // (tail: Bp - 1, below)
            plan.add(tb.done, sizeof(uint32_t) * old, sizeof(uint32_t) * cap, true, 0);
            plan.add(tb.ring, RB * tb.capq * old, RB * tb.capq * cap, true, -1);
            plan.add(tb.present, sizeof(uint32_t) * old, sizeof(uint32_t) * cap, false, -1);
            plan.add(tb.cnt, sizeof(uint32_t) * (old + 1), sizeof(uint32_t) * (cap + 1ull), false, -1);
            ffat_plan_state(h->cb, plan, cap);
            return 0;
        },
        [h, s](uint32_t cap, const GrowPlan &plan) {
            const uint32_t old = h->cb->ff.max_keys; // (the back end still has the old capacity)
            std::vector<uint64_t> t0(cap - old, h->tb.Bp - 1); // :463
            CK(cudaMemcpyAsync(h->tb.trig + old, t0.data(), sizeof(uint64_t) * t0.size(), cudaMemcpyHostToDevice, s));
            CK(cudaStreamSynchronize(s)); // (t0 lives until here)
            ffat_derive(h->cb, cap);
            h->cb->ff.slot_key = h->ff.slot_key;
            h->state_bytes += plan.grown_bytes();
            return 0;
        });
}

static int tb_create(wfb_ffat_t **hh, int prog, uint64_t win, uint64_t slide, uint32_t nb, uint32_t max_keys, uint64_t lateness, uint32_t flags)
{
    const ProgramOps *o = program(prog);
    if (!o) return WFB_E_NOPROG;
    const int lp = lifted_program_of(prog);
    if (lp < 0 || (flags & WFB_FFAT_PIPELINED)) return WFB_E_UNSUPPORTED;
    if ((flags & WFB_FFAT_DENSE_KEYS) && o->key_kind != KEY_KIND_INTEGRAL) return WFB_E_BADARG; // dense keys are integers
    int rc = device_ready(); if (rc) return rc;
    const uint64_t pane_len = gcd_u64(win, slide);                   // wf/ffat_replica_gpu.hpp:639-642
    const uint64_t win_p = win / pane_len, slide_p = slide / pane_len;
    const uint64_t Bp = static_cast<uint64_t>(nb - 1) * slide_p + win_p, group = slide_p * nb;
    uint64_t capq = 1; while (capq < 2 * Bp + group + lateness / pane_len + 8) capq <<= 1;
    const size_t RB = o->result_bytes;
    if (Bp > (1ull << 24) || capq * max_keys * RB > (32ull << 30)) return WFB_E_BADARG;
    wfb_ffat *h = new (std::nothrow) wfb_ffat();
    if (!h) return WFB_E_BADARG;
    h->prog = prog; h->ops = o; h->win_type = 1; h->tb_lateness = lateness; h->pipelined = false;
    FfatDev &ff = h->ff;
    ff.max_keys = max_keys; ff.dense = (flags & WFB_FFAT_DENSE_KEYS) ? 1u : 0u; ff.nb = nb;
    uint32_t cap = 1; while (cap < 2ull * max_keys) cap <<= 1;
    ff.ht_mask = cap - 1;
    size_t total = 0;
#define ALLOC(ptr, bytes) do { cudaError_t e_ = cudaMalloc(reinterpret_cast<void **>(&(ptr)), (bytes)); if (e_ != cudaSuccess) { wfb_ffat_destroy(h); return static_cast<int>(e_); } total += (bytes); } while (0)
    if (!ff.dense) {
        ALLOC(ff.ht_keys, static_cast<size_t>(o->key_bytes) * cap);
        ALLOC(ff.ht_slots, sizeof(uint32_t) * cap);
        CK(cudaMemset(ff.ht_keys, 0xff, static_cast<size_t>(o->key_bytes) * cap));
        CK(cudaMemset(ff.ht_slots, 0xff, sizeof(uint32_t) * cap));
    }
    ALLOC(ff.n_slots, sizeof(uint32_t) * 4);
    h->own_n_slots = ff.n_slots;
    ff.err_flags = ff.n_slots + 1;
    CK(cudaMemset(ff.n_slots, 0, sizeof(uint32_t) * 4));
    ALLOC(ff.slot_key, static_cast<size_t>(o->key_bytes) * max_keys);
    TbDev &tb = h->tb;
    tb.pane_len = pane_len; tb.Bp = Bp; tb.group = group; tb.capq = static_cast<uint32_t>(capq);
    ALLOC(tb.first, sizeof(uint64_t) * max_keys); CK(cudaMemset(tb.first, 0, sizeof(uint64_t) * max_keys));
    ALLOC(tb.num, sizeof(uint32_t) * max_keys); CK(cudaMemset(tb.num, 0, sizeof(uint32_t) * max_keys));
    ALLOC(tb.num_new, sizeof(uint32_t) * max_keys);
    ALLOC(tb.trig, sizeof(uint64_t) * max_keys);
    { std::vector<uint64_t> t0(max_keys, Bp - 1); CK(cudaMemcpy(tb.trig, t0.data(), sizeof(uint64_t) * max_keys, cudaMemcpyHostToDevice)); } // :463
    ALLOC(tb.done, sizeof(uint32_t) * max_keys); CK(cudaMemset(tb.done, 0, sizeof(uint32_t) * max_keys));
    ALLOC(tb.ring, RB * capq * max_keys);
    ALLOC(tb.present, sizeof(uint32_t) * max_keys);
    ALLOC(tb.cnt, sizeof(uint32_t) * (static_cast<size_t>(max_keys) + 1));
    ALLOC(h->tb_misc, sizeof(uint32_t) * 8); CK(cudaMemset(h->tb_misc, 0, sizeof(uint32_t) * 8));
    tb.n_present = h->tb_misc + 2; tb.ignored = h->tb_misc + 4; tb.need = h->tb_misc + 5; tb.err = ff.err_flags;
#undef ALLOC
    rc = h->ts.init(); if (rc) { wfb_ffat_destroy(h); return rc; }
    if (flags & WFB_KEYS_GROW) { ff.grow = 1; rc = h->growc.init(); if (rc) { wfb_ffat_destroy(h); return rc; } } // (the back end grows with it)
    rc = wfb_ffat_create(&h->cb, lp, win_p, slide_p, nb, max_keys, 0, 0, flags & WFB_FFAT_DENSE_KEYS);
    if (rc) { wfb_ffat_destroy(h); return rc; }
    // the front end hands the popped panes to the back end with the slot of every record. On the bucket path (at most 65536 keys) the
    // back end reads them in place, which WFB_BUCKET_MOVE=1 does not do: refuse that here, before any pane has been consumed, rather than
    // at the first firing batch. Above 65536 keys the full-sort path's streaming pass takes the slots as they are.
    if (h->cb->buckets && h->cb->bucket_move) { wfb_ffat_destroy(h); return WFB_E_UNSUPPORTED; }
    // the back end never looks keys up (the front end hands it the slot of every record): it only needs slot -> key for the results
    if (!ff.dense) { cudaFree(h->cb->ff.slot_key); h->cb->ff.slot_key = ff.slot_key; h->cb->ff.n_slots = ff.n_slots; h->cb->shares_slot_key = true; }
    h->state_bytes = total + h->cb->state_bytes;
    *hh = h;
    return 0;
}

static int tb_ensure(wfb_ffat *h, uint32_t n, cudaStream_t s)
{
    CK(h->tb_kA.ensure(n, s));
    const size_t RB = h->ops->result_bytes, c = h->tb_kA.capacity(), head_cap = (c + SEGT - 1) / SEGT + 1;
    CK(h->tb_kB.ensure(n, s, c)); CK(h->tb_iA.ensure(n, s, c)); CK(h->tb_iB.ensure(n, s, c));
    CK(h->tb_lifted.ensure(RB * n, s, RB * c)); CK(h->tb_part.ensure(RB * n, s, RB * c));
    CK(h->tb_head.ensure(head_cap, s, head_cap)); CK(h->tb_seg.ensure(n + 1ull, s, c + 1));
    return 0;
}

int wfb_ffat_process_tb(wfb_ffat_t *h, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches,
                        void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, void *stream)
{
    if (!h || h->win_type != 1 || !n_out_dev || (nbatches && !batches_h) || (out_capacity && !out_results)) return WFB_E_BADARG;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t RB = h->ops->result_bytes;
    const void *prm = pre ? static_cast<const void *>(pre) : h->pp();
    uint32_t produced = 0;
    for (uint32_t bi = 0; bi < nbatches; bi++) {
        const wfb_batch_t &b = batches_h[bi];
        if (b.n == 0) continue;
        if (!b.tuples || !b.ts) return WFB_E_BADARG;            // time-based windows need the timestamps
        int rc = tb_ensure(h, b.n, s); if (rc) return rc;
        const uint64_t wm = b.watermark;
        const uint64_t F = wm >= h->tb_lateness ? (wm - h->tb_lateness) / h->tb.pane_len : 0; // first_pane_not_complete :875-881
        uint32_t *misc = h->tb_misc;
        CK(cudaMemsetAsync(misc, 0, sizeof(uint32_t) * 4, s));
        CK(cudaMemsetAsync(misc + 5, 0, sizeof(uint32_t), s));
        // 1. lift + composite (slot, pane) keys; 2. stable sort; 3. (key, pane) segments; 4. partials; 5. merge into the rings
        if (h->ff.grow) CK(cudaMemcpyAsync(misc + 6, misc + 4, sizeof(uint32_t), cudaMemcpyDeviceToDevice, s)); // (ignored tuples before this batch)
        rc = h->ops->tb_lift(static_cast<const unsigned char *>(b.tuples), b.ts, b.n, h->ff, h->tb, F, h->tb_lifted, h->tb_kA, s, prm); if (rc) return rc;
        for (bool grew = h->ff.grow != 0; grew; ) { // more keys than the capacity: grow, then lift the batch again
            rc = tb_grow(h, s, &grew); if (rc) return rc;
            if (!grew) break;
            CK(cudaMemsetAsync(misc + 5, 0, sizeof(uint32_t), s));
            CK(cudaMemcpyAsync(misc + 4, misc + 6, sizeof(uint32_t), cudaMemcpyDeviceToDevice, s)); // (the rerun counts this batch's late tuples again)
            rc = h->ops->tb_lift(static_cast<const unsigned char *>(b.tuples), b.ts, b.n, h->ff, h->tb, F, h->tb_lifted, h->tb_kA, s, prm); if (rc) return rc;
            h->launches += 2;
        }
        uint32_t tb_need_bits = 2;
        { // the rings must hold every pane from a key's first pending one to its newest (PendingPanes_Queue::push_panes :367-372)
            uint32_t need = 0;
            CK(cudaMemcpyAsync(&need, misc + 5, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            tb_need_bits = std::max(2u, need);
            if (need > h->tb.capq) {
                uint64_t ncap = h->tb.capq; while (ncap < need) ncap <<= 1;
                if (ncap * h->ff.max_keys * RB > (32ull << 30)) return WFB_E_CAPACITY;
                unsigned char *nr = nullptr;
                CK(cudaMalloc(&nr, RB * ncap * h->ff.max_keys));
                k_tb_ring_resize<<<grid_for(h->ff.max_keys, 128), 128, 0, s>>>(h->tb, h->tb.ring, h->tb.capq, nr, static_cast<uint32_t>(ncap), h->ff.max_keys,
                                                                                static_cast<uint32_t>(RB));
                CK(cudaStreamSynchronize(s));
                cudaFree(h->tb.ring);
                h->tb.ring = nr; h->tb.capq = static_cast<uint32_t>(ncap);
                h->launches++;
            }
        }
        // sort keys (slot << kbits) | relative pane, with just the bits this batch needs; filtered tuples sort behind every slot
        uint32_t sbits = 0; while ((1ull << sbits) < static_cast<uint64_t>(h->ff.max_keys) + 1) sbits++;
        uint32_t kbits = 1; while ((1ull << kbits) < tb_need_bits) kbits++;
        h->tb.kbits = kbits;
        k_tb_pack<<<grid_for(b.n, 256), 256, 0, s>>>(h->tb_kA, b.n, kbits, h->ff.max_keys);
        const uint64_t *skeys; const uint32_t *sidx;
        const uint64_t before = h->sorter.launches;
        rc = h->sorter.sort<uint64_t>(h->tb_kA, h->tb_kB, h->tb_iA, h->tb_iB, nullptr, b.n, b.n, (kbits + sbits + 7) / 8, s, &skeys, &sidx); if (rc) return rc;
        const uint32_t tiles = (b.n + SEGT - 1) / SEGT;
        k_head_tile_counts<<<tiles, 256, 0, s>>>(skeys, b.n, h->tb_head);
        k_scan_u32<<<1, 1024, 0, s>>>(h->tb_head, h->tb_head, tiles, nullptr);
        k_seg_finish_batches<<<tiles, 256, 0, s>>>(skeys, b.n, 64u, h->tb_head, h->tb_seg, misc + 1, misc + 0);
        CK(cudaGetLastError());
        rc = h->ops->tb_reduce(h->tb_lifted, skeys, sidx, h->tb_seg, misc + 0, h->tb_part, b.n, kbits, h->ff.max_keys, s, prm); if (rc) return rc;
        rc = h->ops->tb_merge(skeys, h->tb_seg, misc + 0, h->tb_part, h->ff, h->tb, b.n, s, prm); if (rc) return rc;
        // 6. panes to pop per present key, offsets, total
        const uint32_t maxp = std::min<uint32_t>(b.n, h->ff.max_keys);
        k_tb_pop_count<<<grid_for(maxp, 128), 128, 0, s>>>(h->tb, F);
        k_tb_scan_present<<<1, 1024, 0, s>>>(h->tb.cnt, h->tb.n_present, misc + 3);
        CK(cudaGetLastError());
        uint32_t total = 0;
        CK(cudaMemcpyAsync(&total, misc + 3, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));                           // (the reference synchronises here as well, :962)
        CK(h->tb_popped.ensure(RB * total));
        const size_t pop_cap = h->tb_popped.capacity() / RB, slots_cap = (pop_cap + TILE - 1) / TILE * TILE;
        CK(h->tb_popped_slots.ensure(slots_cap, ScratchWaits(), slots_cap));
        rc = h->ops->tb_pop_write(h->ff, h->tb, F, h->tb.cnt, h->tb_popped, h->tb_popped_slots, static_cast<uint32_t>(pop_cap), maxp, s, prm); if (rc) return rc;
        h->launches += 10 + (h->sorter.launches - before);
        // 7. the count-based back end consumes the popped panes as one batch with this batch's watermark
        if (total) {
            wfb_batch_t pb; std::memset(&pb, 0, sizeof(pb));
            pb.tuples = h->tb_popped; pb.ts = nullptr; pb.watermark = wm; pb.n = total;
            const uint64_t lb = h->cb->launches;
            rc = ffat_process_cb_impl(h->cb, prm, &pb, 1, static_cast<unsigned char *>(out_results) + static_cast<size_t>(produced) * RB,
                                      out_ts ? out_ts + produced : nullptr, out_capacity - produced, n_out_dev, s, h->tb_popped_slots);
            if (rc) return rc;
            h->launches += h->cb->launches - lb;
            uint32_t got = 0;
            CK(cudaMemcpyAsync(&got, n_out_dev, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            produced += std::min(got, out_capacity - produced);
        }
    }
    CK(cudaMemcpyAsync(n_out_dev, &produced, sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s)); // `produced` lives on this stack frame
    return 0;
}

int wfb_ffat_create(wfb_ffat_t **hh, int prog, uint64_t win, uint64_t slide, uint32_t wins_per_batch,
                    uint32_t max_keys, int win_type, uint64_t lateness, uint32_t flags)
{
    if (!hh || win == 0 || slide == 0 || wins_per_batch == 0 || max_keys == 0) return WFB_E_BADARG;
    if ((flags & WFB_KEYS_GROW) && (flags & (WFB_FFAT_DENSE_KEYS | WFB_FFAT_PIPELINED))) return WFB_E_BADARG; // (dense: slot = key, nothing to grow)
    if (win_type == 1) return tb_create(hh, prog, win, slide, wins_per_batch, max_keys, lateness, flags);
    if (win_type != 0) return WFB_E_UNSUPPORTED;
    const ProgramOps *o = program(prog);
    if (!o) return WFB_E_NOPROG;
    if ((flags & WFB_FFAT_DENSE_KEYS) && o->key_kind != KEY_KIND_INTEGRAL) return WFB_E_BADARG; // dense keys are integers
    int rc = device_ready(); if (rc) return rc;
    wfb_ffat *h = new (std::nothrow) wfb_ffat();
    if (!h) return WFB_E_BADARG;
    h->prog = prog; h->ops = o; h->win_type = win_type;
    rc = h->ts.init(); if (rc) { delete h; return rc; }
    FfatDev &ff = h->ff;
    ff.win = win; ff.slide = slide; ff.nb = wins_per_batch;
    ff.B = static_cast<uint64_t>(wins_per_batch - 1) * slide + win;
    const uint64_t pane = gcd_u64(win, slide);
    const uint64_t bp = ff.B / pane;
    if (pane > 0xffffffffull || bp > (1ull << 30)) { delete h; return WFB_E_BADARG; }
    ff.pane = static_cast<uint32_t>(pane); ff.wp = static_cast<uint32_t>(win / pane); ff.sp = static_cast<uint32_t>(slide / pane);
    // ring of n leaves (a power of two) for the bp panes a group reads + spare leaves: a key that completes up to `spare` further panes in
    // the call that fires a group leaves the group's leaves alone, so the group can wait for the deferred pass (one warp per group, levels
    // built on chip) instead of being evaluated inside the update kernel. At least min(bp, 32) spare leaves.
    const uint64_t spare_min = std::min<uint64_t>(bp, 32);
    uint32_t n = 1, lg = 0; while (n < bp + spare_min) { n <<= 1; lg++; }
    ff.n_leaves = n; ff.log_leaves = lg;
    ff.defer_items = (static_cast<uint64_t>(n) - bp + 1) * pane;
    ff.max_keys = max_keys; ff.dense = (flags & WFB_FFAT_DENSE_KEYS) ? 1u : 0u;
    uint32_t cap = 1; while (cap < 2ull * max_keys) cap <<= 1;
    ff.ht_mask = cap - 1;
    const size_t RB = o->result_bytes;
    const size_t tree_bytes = static_cast<size_t>(max_keys) * (2ull * n - 1) * RB;
    size_t total = 0;
#define ALLOC(ptr, bytes) do { cudaError_t e_ = cudaMalloc(reinterpret_cast<void **>(&(ptr)), (bytes)); if (e_ != cudaSuccess) { wfb_ffat_destroy(h); return static_cast<int>(e_); } total += (bytes); } while (0)
    if (!ff.dense) {
        ALLOC(ff.ht_keys, static_cast<size_t>(o->key_bytes) * cap);
        ALLOC(ff.ht_slots, sizeof(uint32_t) * cap);
        CK(cudaMemset(ff.ht_keys, 0xff, static_cast<size_t>(o->key_bytes) * cap));
        CK(cudaMemset(ff.ht_slots, 0xff, sizeof(uint32_t) * cap));
    }
    ALLOC(ff.n_slots, sizeof(uint32_t) * 4);
    h->own_n_slots = ff.n_slots;
    ff.err_flags = ff.n_slots + 1;
    ff.results_total = reinterpret_cast<unsigned long long *>(ff.n_slots + 2);
    CK(cudaMemset(ff.n_slots, 0, sizeof(uint32_t) * 4));
    ALLOC(ff.slot_key, static_cast<size_t>(o->key_bytes) * max_keys);
    ALLOC(ff.cnt, sizeof(uint64_t) * max_keys);
    CK(cudaMemset(ff.cnt, 0, sizeof(uint64_t) * max_keys));
    ALLOC(ff.acc, RB * max_keys);
    CK(cudaMemset(ff.acc, 0, RB * max_keys));
    ALLOC(ff.tree, tree_bytes);
    CK(cudaMemset(ff.tree, 0, tree_bytes));
    ALLOC(ff.seg_off, sizeof(uint32_t) * (static_cast<size_t>(max_keys) + 1));
    CK(cudaMemset(ff.seg_off, 0xff, sizeof(uint32_t) * (static_cast<size_t>(max_keys) + 1)));
    ALLOC(ff.heavy, sizeof(uint32_t) * max_keys);
    ff.light_max = 256;
    h->pipelined = (flags & WFB_FFAT_PIPELINED) != 0;
    for (int p = 0; p < (h->pipelined ? 2 : 1); p++) {
        SegScratch &g = h->seg[p];
        ALLOC(g.seg_cnt, sizeof(uint32_t) * max_keys);
        CK(cudaMemset(g.seg_cnt, 0, sizeof(uint32_t) * max_keys));
        ALLOC(g.n_total, sizeof(uint32_t) * 4);
        CK(cudaMemset(g.n_total, 0, sizeof(uint32_t) * 4));
        g.n_trig = g.n_total + 1; g.res_n = h->pipelined ? g.n_total + 2 : nullptr; g.n_heavy = g.n_total + 3;
        ALLOC(g.sort_ctl, sizeof(uint32_t) * RadixSorter::CTL_WORDS);
        CK(cudaEventCreateWithFlags(&g.ev_ingest, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&g.ev_done, cudaEventDisableTiming));
    }
    if (h->pipelined) CK(cudaStreamCreateWithFlags(&h->s2, cudaStreamNonBlocking));
#undef ALLOC
    if (flags & WFB_KEYS_GROW) { ff.grow = 1; rc = h->growc.init(); if (rc) { wfb_ffat_destroy(h); return rc; } }
    { const char *e = std::getenv("WFB_BUCKET_MOVE"); h->bucket_move = e && std::atoi(e) != 0; }
    ffat_derive_paths(h);
    { // lazy FlatFAT levels (FfatDev::lazy): bucket path, the on-chip tree of one group must fit 32 KB, and building the n - 1 internal
      // nodes once per fired group must be cheaper than a root path (log n nodes) per completed pane: a group fires every sp * Nb panes.
      // (Nb = 1 with slide = pane fires on every pane: eager levels there.) A growing handle keeps the layout it was created with when
      // it leaves the bucket path: the update kernels of both paths read and write either one.
        const bool fits = h->buckets && static_cast<size_t>(2) * ff.n_leaves * RB <= (32u << 10);
        const bool pays = static_cast<uint64_t>(ff.n_leaves) <= 2ull * std::max(1u, ff.log_leaves) * ff.sp * ff.nb;
        ff.lazy = (fits && pays) ? 1u : 0u;
    }
    h->state_bytes = total;
    *hh = h;
    return 0;
}

int wfb_ffat_destroy(wfb_ffat_t *h)
{
    if (!h) return 0;
    cudaDeviceSynchronize();
    FfatDev &ff = h->ff;
    cudaFree(ff.ht_keys); cudaFree(ff.ht_slots); cudaFree(h->own_n_slots); if (!h->shares_slot_key) cudaFree(ff.slot_key); cudaFree(ff.cnt);
    cudaFree(ff.acc); cudaFree(ff.tree); cudaFree(ff.seg_off); cudaFree(ff.heavy);
    for (SegScratch &g : h->seg) { cudaFree(g.n_total); cudaFree(g.seg_cnt); cudaFree(g.sort_ctl); g.destroy(); } // (n_trig, n_heavy, res_n: inside n_total)
    if (h->cb) wfb_ffat_destroy(h->cb);
    cudaFree(h->tb.first); cudaFree(h->tb.num); cudaFree(h->tb.num_new); cudaFree(h->tb.trig); cudaFree(h->tb.done); cudaFree(h->tb.ring);
    cudaFree(h->tb.present); cudaFree(h->tb.cnt); cudaFree(h->tb_misc);
    if (h->s2) cudaStreamDestroy(h->s2);
    for (auto &e : h->tev) cudaEventDestroy(e);
    h->ts.destroy(); h->growc.destroy();
    delete h;
    cudaGetLastError();
    return 0;
}

uint64_t wfb_ffat_launches(const wfb_ffat_t *h) { return h ? h->launches : 0; }

int wfb_ffat_set_params(wfb_ffat_t *h, const void *params, size_t bytes)
{
    if (!h || !params || bytes != h->ops->params_bytes) return WFB_E_BADARG;
    h->params.assign(static_cast<const unsigned char *>(params), static_cast<const unsigned char *>(params) + bytes);
    if (h->cb) h->cb->params = h->params; // the lifted variant shares the program's params_t (its comb / make_result)
    return 0;
}
uint64_t wfb_ffat_state_bytes(const wfb_ffat_t *h) { return h ? h->state_bytes : 0; }
uint32_t wfb_ffat_key_capacity(const wfb_ffat_t *h) { return h ? h->ff.max_keys : 0; }
int wfb_ffat_set_key_shard(wfb_ffat_t *h, uint32_t num_shards, uint32_t shard)
{
    if (!h || num_shards == 0 || shard >= num_shards || !h->ff.dense || h->call_no != 0) return WFB_E_BADARG;
    if (h->win_type == 1) { // time-based: the front end maps keys to slots, the back end turns slots back into keys for the results
        if (h->cb == nullptr || h->cb->call_no != 0) return WFB_E_BADARG;
        h->cb->ff.key_div = num_shards; h->cb->ff.key_rem = shard;
    }
    h->ff.key_div = num_shards; h->ff.key_rem = shard;
    return 0;
}

static double host_now_us() { timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec * 1e6 + t.tv_nsec * 1e-3; }
static int ffat_ensure_segment(wfb_ffat *h, SegScratch &g, uint32_t total, uint32_t nbatches, cudaStream_t s)
{
    const ScratchWaits w = h->s2 ? ScratchWaits(s, h->s2) : ScratchWaits(s);
    CK(g.slotsA.ensure(total, w));
    const size_t cap = g.slotsA.capacity(), RB = h->ops->result_bytes;
    CK(g.slotsB.ensure(total, w, cap));
    if (!h->buckets) { CK(g.posA.ensure(total, w, cap)); CK(g.posB.ensure(total, w, cap)); }
    CK(g.lifted.ensure(RB * total, w, RB * cap));
    if (h->bucket_move) CK(g.lifted_sorted.ensure(RB * total, w, RB * cap));
    // the window groups the segment can fire, for the current key capacity (key growth raises it before the pass runs again)
    const uint32_t trig_cap = ffat_trig_cap(h, static_cast<uint32_t>(cap), h->ff.max_keys);
    CK(g.trig.ensure(trig_cap, w, trig_cap));
    if (h->pipelined) { // every group that can fire in one segment: trig_cap groups of Nb results
        const size_t res_cap = std::min<uint64_t>(static_cast<uint64_t>(trig_cap) * h->ff.nb, 0x7fffffffull);
        CK(g.res_ts.ensure(res_cap, w, res_cap)); CK(g.res.ensure(RB * res_cap, w, RB * res_cap));
    }
    CK(g.batch_off.ensure(nbatches + 1ull, w));
    CK(g.d_batches.ensure(nbatches + 1ull, w, g.batch_off.capacity()));
    return 0;
}

// the last kernel of a call adds *n_out to results_total: a call (or position range) whose results follow the ones already in the
// output buffer takes those out of the total first
__global__ void k_results_pre_append(unsigned long long *results_total, const uint32_t *n_out) { if (results_total) *results_total -= *n_out; }

// sort + update + deferred window queries of the segment held in `g`, results to (out, out_ts, n_out)
static int ffat_window_phase(wfb_ffat *h, SegScratch &g, const FfatDev &ff, unsigned char *out, uint64_t *out_ts, uint32_t out_cap,
                             uint32_t *n_out, cudaStream_t s)
{
    const uint32_t *sorted_slots, *sorted_pos;
    const uint64_t before = h->sorter.launches;
    int rc;
    if (h->buckets) {
        // The bucket list holds positions below BKL_RANGE_POS: a segment of more positions is partitioned, updated and queried one range
        // of BKL_RANGE_POS positions (whole wide tiles) at a time. The ranges are consecutive in arrival order, so every key's state
        // carries over from one range to the next as it does from call to call, and the windows a range fires are evaluated before
        // the next range writes leaves. Results of all ranges are appended to `out`.
        const size_t RB = h->ops->result_bytes;
        const uint16_t *rows = h->pipelined ? static_cast<const uint16_t *>(g.h16) : static_cast<const uint16_t *>(h->sorter.wideH);
        for (uint32_t base = 0; base < g.total; base += BKL_RANGE_POS) {
            const uint32_t n = std::min(BKL_RANGE_POS, g.total - base);
            if (base != 0) { // (the first range's trigger list: cleared by the tile pass)
                CK(cudaMemsetAsync(g.n_trig, 0, sizeof(uint32_t), s));
                k_results_pre_append<<<1, 1, 0, s>>>(ff.results_total, n_out);
                CK(cudaGetLastError());
                h->launches++;
            }
            // ONE wide radix pass on the top 10 slot bits: 1024 buckets of consecutive keys, arrival order inside a bucket ...
            const uint32_t *counts = nullptr;
            const uint64_t before_r = h->sorter.launches;
            rc = h->sorter.sort_wide<uint32_t>(g.slotsA + base, g.slotsB, nullptr, nullptr, n, n, h->bucket_shift, s, g.sort_ctl, &counts,
                                               h->bucket_move ? static_cast<unsigned char *>(g.lifted) + base * RB : nullptr,
                                               h->bucket_move ? static_cast<unsigned char *>(g.lifted_sorted) : nullptr,
                                               static_cast<uint32_t>(RB), true, 0, 0, rows + static_cast<size_t>(base / OSW_TILE) * OSW_DIGITS, true);
            if (rc) return rc;
            h->launches += h->sorter.launches - before_r;
            h->mark(2, s);
            // ... then one CTA per bucket finishes the job (local split by key, per-key ordered fold, FlatFAT update)
            rc = h->ops->ffat_buckets(ff, h->bucket_move ? static_cast<const unsigned char *>(g.lifted_sorted) : g.lifted_src + base * RB, g.slotsB, base, counts,
                                      h->bucket_shift, h->bucket_move ? 1u : 0u, g.batch_off, g.d_batches, g.nbatches, out, out_ts, out_cap, n_out, s, h->pp());
            if (rc) return rc;
            // deferred window groups: one thread per window
            rc = h->ops->ffat_windows(ff, g.batch_off, g.d_batches, g.nbatches, out, out_ts, out_cap, static_cast<uint32_t>(g_num_sms) * 4u, s, h->pp(), n_out);
            if (rc) return rc;
            h->launches += 2;
        }
        return 0;
    } else {
        // stable sort of (slot, arrival position) by slot: onesweep radix, 8 bits per pass
        rc = h->sorter.sort<uint32_t>(g.slotsA, g.slotsB, g.posA, g.posB, g.n_total, 0, g.total, h->sort_passes, s, &sorted_slots,
                                      &sorted_pos, g.sort_ctl, ff.seg_off, ff.max_keys);
        if (rc) return rc;
        h->launches += h->sorter.launches - before;
        h->mark(2, s);
        // one thread per key (one warp per heavy key): pane fold, FlatFAT update
        uint32_t ugrid = std::max(1u, std::min((ff.max_keys + 7) / 8, static_cast<uint32_t>(g_num_sms) * 8u));
        rc = h->ops->ffat_update(ff, g.lifted, sorted_pos, g.batch_off, g.d_batches, g.nbatches, out, out_ts, out_cap, n_out, ugrid, s, h->pp(),
                                 std::max(1u, std::min((ff.max_keys + 127u) / 128u, static_cast<uint32_t>(g_num_sms) * 16u)));
        if (rc) return rc;
        h->launches += 2;
    }
    // deferred window groups: one thread per window
    rc = h->ops->ffat_windows(ff, g.batch_off, g.d_batches, g.nbatches, out, out_ts, out_cap, static_cast<uint32_t>(g_num_sms) * 4u, s, h->pp(), n_out);
    if (rc) return rc;
    h->launches += 1;
    return 0;
}

// pipelined mode: hand the finished results of the segment in `g` to the caller (stream-ordered on s)
static int ffat_deliver(wfb_ffat *h, SegScratch &g, unsigned char *out, uint64_t *out_ts, uint32_t out_cap, uint32_t *n_out, cudaStream_t s)
{
    if (!g.pending) { CK(cudaMemsetAsync(n_out, 0, sizeof(uint32_t), s)); return 0; }
    CK(cudaStreamWaitEvent(s, g.ev_done, 0));
    k_copy_results<<<static_cast<uint32_t>(g_num_sms) * 2u, 256, 0, s>>>(g.res, g.res_ts, g.res_n, h->ops->result_bytes, out, out_ts,
                                                                          out_cap, n_out, h->ff.err_flags);
    CK(cudaGetLastError());
    h->launches++;
    g.pending = false;
    return 0;
}

int wfb_ffat_process_cb(wfb_ffat_t *h, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches,
                        void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, void *stream)
{
    return ffat_process_cb_impl(h, pre, batches_h, nbatches, out_results, out_ts, out_capacity, n_out_dev, stream, nullptr);
}

// ext_slots != nullptr: the key slot of the record at every position is given (one batch, read in place on the bucket path; used by
// the time-based front end, whose programs' lifted variants have no key extractor)
static int ffat_process_cb_impl(wfb_ffat_t *h, const void *pre, const wfb_batch_t *batches_h, uint32_t nbatches,
                                void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, void *stream,
                                const uint32_t *ext_slots)
{
    if (!h || !n_out_dev || (nbatches && !batches_h) || (out_capacity && !out_results)) return WFB_E_BADARG;
    if (h->win_type != 0) return WFB_E_BADARG; // time-based handles: wfb_ffat_process_tb
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc = h->ts.enter(s); if (rc) return rc;
    unsigned char *out = static_cast<unsigned char *>(out_results);
    const uint32_t par = h->pipelined ? static_cast<uint32_t>(h->call_no & 1u) : 0u;
    SegScratch &g = h->seg[par];
    SegScratch &prev = h->seg[h->pipelined ? (par ^ 1u) : 0u];

    std::vector<DevBatch> hb; // empty batches trigger nothing: only the non-empty ones reach the device
    hb.reserve(nbatches);
    uint64_t total = 0; uint32_t tiles = 0;
    uint64_t span_begin = ~0ull, span_end = 0; // address span of the segment's tuples (for the 2-D tensor map)
    for (uint32_t i = 0; i < nbatches; i++) {
        if (batches_h[i].n == 0) continue;
        if (!batches_h[i].tuples) return WFB_E_BADARG;
        DevBatch b; std::memset(&b, 0, sizeof(b));
        b.tuples = static_cast<const unsigned char *>(batches_h[i].tuples); b.ts = batches_h[i].ts;
        b.watermark = batches_h[i].watermark; b.n = batches_h[i].n; b.tile_begin = tiles;
        tiles += tiles_of(b.n); total += b.n;
        const uint64_t p0 = reinterpret_cast<uint64_t>(b.tuples);
        span_begin = std::min(span_begin, p0); span_end = std::max(span_end, p0 + static_cast<uint64_t>(b.n) * h->ops->tuple_bytes);
        hb.push_back(b);
    }
    if (total > 0x7fffffffull) return WFB_E_BADARG;
    if (total == 0) { // nothing to ingest: (pipelined) still deliver what is pending
        if (h->pipelined) return ffat_deliver(h, prev, out, out_ts, out_capacity, n_out_dev, s);
        if (!h->append_results) CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t), s));
        return 0;
    }
    nbatches = static_cast<uint32_t>(hb.size());
    FfatDev ff; // this call's view of the state: per-segment buffers of parity `par`
    // the pass that inserts the call's keys into the key table; a growing handle runs it again after the table grew
    const auto ingest = [&]() -> int {
        // bucket path: no global compaction in the streaming pass -- tile t owns positions [t*TILE, +TILE) of the segment
        const bool sparse = h->buckets;
        const uint64_t seg_cap = sparse ? static_cast<uint64_t>(tiles) * TILE : total;
        if (seg_cap > 0x7fffffffull) return WFB_E_BADARG;
        rc = ffat_ensure_segment(h, g, static_cast<uint32_t>(seg_cap), nbatches, s); if (rc) return rc;
        rc = h->ts.ensure_tiles(tiles); if (rc) return rc;
        { int rc_ = h->ts.stage.h2d(g.d_batches, hb.data(), sizeof(DevBatch) * nbatches, s); if (rc_) return rc_; }
        g.nbatches = nbatches; g.total = static_cast<uint32_t>(seg_cap);
        if (sparse) { // first position of every batch (the compacting pass writes the compact offsets itself)
            std::vector<uint32_t> boff(nbatches + 1);
            for (uint32_t i = 0; i < nbatches; i++) boff[i] = hb[i].tile_begin * TILE;
            boff[nbatches] = tiles * TILE;
            { int rc_ = h->ts.stage.h2d(g.batch_off, boff.data(), sizeof(uint32_t) * (nbatches + 1), s); if (rc_) return rc_; }
        }

        ff = h->ff;
        ff.seg_cnt = g.seg_cnt; ff.trig = g.trig; ff.n_trig = g.n_trig; ff.trig_cap = static_cast<uint32_t>(g.trig.capacity()); ff.n_heavy = g.n_heavy;

        // the streaming pass also counts the digits of the slot sort that follows
        const uint32_t npasses = h->buckets ? 1u : h->sort_passes;
        rc = h->buckets ? RadixSorter::prepare_wide(g.sort_ctl, s) : RadixSorter::prepare(g.sort_ctl, npasses, s); if (rc) return rc;
        h->mark(0, s);
        // 1. streaming pass: [map -> filter ->] lift, key -> slot, stable compaction over the whole segment
        TileArgs a; std::memset(&a, 0, sizeof(a));
        a.sort_ctl = g.sort_ctl; a.sort_passes = npasses; a.sort_shift = h->buckets ? h->bucket_shift : 0u; a.sort_dbits = h->buckets ? OSW_BITS : 8u;
        a.batches = g.d_batches; a.nbatches = nbatches; a.num_tiles = tiles;
        a.lifted = g.lifted; a.slots = g.slotsA; a.batch_off = g.batch_off; a.n_total = g.n_total; a.ff = ff;
        g.lifted_src = g.lifted;
        if (sparse && !h->pipelined && !h->bucket_move && (h->ops->reserved & 1u)) {
            // pass-through program and every batch at its tile position inside one buffer: read the records where they are
            const unsigned char *base = hb[0].tuples;
            bool ok = (reinterpret_cast<uintptr_t>(base) & 15u) == 0;
            for (uint32_t i = 0; ok && i < nbatches; i++) ok = hb[i].tuples == base + static_cast<size_t>(hb[i].tile_begin) * TILE * h->ops->tuple_bytes;
            if (ok) { a.inplace = 1; g.lifted_src = base; a.ext_slots = ext_slots; }
        }
        if (ext_slots != nullptr && !a.inplace) {
            // full-sort path: the compacting pass reads the slot of position tile·TILE + thread. The time-based front end hands over one
            // batch from tile 0 whose records all pass (a lifted program filters nothing): compacted position = popped index = position
            if (sparse) return WFB_E_UNSUPPORTED; // (the front end always meets the in-place conditions on the bucket path)
            if (nbatches != 1 || !(h->ops->reserved & 1u)) return WFB_E_BADARG;
            a.ext_slots = ext_slots;
        }
        h->ts.next_launch(a);
        a.max_ctas_per_sm = h->pipelined ? 2u : 0u; // (pipelined: leave room for the concurrent sort / update kernels)
        a.l2_hints = 1;
        a.sparse = sparse ? 1u : 0u;
        a.count_keys = h->buckets ? 0u : 1u;
        uint32_t claims = tiles;
        if (sparse) {
            // a CTA claims the 16 tiles of a wide tile at once, counts its digits in shared memory and files the row itself, and packs a
            // rank with every slot (bucket-path slots fit 16 bits): the partition that follows needs neither a counting pass nor the
            // per-CTA global digit counts
            const ScratchWaits w = h->pipelined ? ScratchWaits(s, h->s2) : ScratchWaits(s);
            rc = h->sorter.ensure_wide(g.total, w, &a.wide_h16); if (rc) return rc; // (also sizes the chunk rows the partition needs)
            if (h->pipelined) {
                const size_t wt = (g.total + OSW_TILE - 1) / OSW_TILE;
                CK(g.h16.ensure(OSW_DIGITS * wt, w));
                a.wide_h16 = g.h16;
            }
            a.tiles_per_ticket = OSW_TILE_POS / TILE;
            a.sort_ctl = nullptr; // (the partition accumulates the global counts into g.sort_ctl, cleared above)
            a.pack_rank = 1;
            claims = (tiles + a.tiles_per_ticket - 1) / a.tiles_per_ticket;
        }
        if (a.inplace && h->ops->slots_inplace) {
            // records read in place: only the slots and the rows are produced -- no tiles to stage, a plain kernel does it
            rc = h->ops->slots_inplace(a, pre ? static_cast<const void *>(pre) : h->pp(), s); if (rc) return rc;
        } else {
            uint32_t grid = 0;
            rc = h->ops->tile_pass(MODE_INGEST, a, pre ? static_cast<const void *>(pre) : h->pp(), claims, s, &grid, span_begin, span_end); if (rc) return rc;
            h->ts.launched(claims, grid);
        }
        h->launches++;
        h->mark(1, s);
        return 0;
    };
    rc = ingest(); if (rc) return rc;
    for (bool grew = h->ff.grow != 0; grew; ) { // more keys than the capacity: grow, then run the pass again
        rc = ffat_grow(h, s, &grew); if (rc) return rc;
        if (grew) { rc = ingest(); if (rc) return rc; h->launches++; }
    }

    if (!h->pipelined) {
        if (!h->append_results) CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t), s));
        rc = ffat_window_phase(h, g, ff, out, out_ts, out_capacity, n_out_dev, s); if (rc) return rc;
        h->mark(3, s);
    } else {
        // the ingest pass of this segment is queued: now hand over the previous segment's results, then start this
        // segment's sort + update on the internal stream, where it overlaps the NEXT call's ingest pass
        CK(cudaEventRecord(g.ev_ingest, s));
        rc = ffat_deliver(h, prev, out, out_ts, out_capacity, n_out_dev, s); if (rc) return rc;
        CK(cudaStreamWaitEvent(h->s2, g.ev_ingest, 0));
        CK(cudaMemsetAsync(g.res_n, 0, sizeof(uint32_t), h->s2));
        rc = ffat_window_phase(h, g, ff, g.res, g.res_ts, static_cast<uint32_t>(g.res_ts.capacity()), g.res_n, h->s2); if (rc) return rc;
        h->mark(3, h->s2);
        CK(cudaEventRecord(g.ev_done, h->s2));
        g.pending = true;
    }
    if (h->timing && h->tev_used < wfb_ffat::TEV_MAX) h->tev_used++;
    h->call_no++;
    return 0;
}

// Window update on records that arrive grouped by bucket (destination side of the bucketed multi-GPU exchange): source s delivered
// offs_h[s+1] - offs_h[s] records from position offs_h[s] of `records`, bucket after bucket of this handle's slot space (buckets of
// 2^shift slots, bps of them; bins = the run lengths [nsrc][bps], recv_slots = the records' slots before masking). No partition pass:
// the runs of a bucket, in source order, ARE its items in stream order.
static int ffat_process_prebucketed(wfb_ffat *h, const unsigned char *records, const uint32_t *recv_slots, const uint32_t *bins, uint32_t nsrc,
                                    uint32_t bps, const uint32_t *offs_h, const uint64_t *wms_h, uint32_t slot_mask, uint32_t shift,
                                    void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, cudaStream_t s, bool append, uint32_t items)
{   // items: records delivered in all (the runs of a source need not be back to back with the next source's: offs_h[nsrc] only bounds the positions)
    if (!h || !n_out_dev || nsrc == 0 || nsrc > MAX_SHARDS || bps == 0 || bps > OSW_DIGITS || (1u << shift) > BK_KEYS) return WFB_E_BADARG;
    if (h->win_type != 0 || h->pipelined || !h->buckets) return WFB_E_UNSUPPORTED;
    int rc = h->ts.enter(s); if (rc) return rc;
    SegScratch &g = h->seg[0];
    const uint32_t total = items;
    if (!append) CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t), s)); // (append: the results follow the ones already in the buffer)
    if (total == 0) return 0;
    rc = ffat_ensure_segment(h, g, total, nsrc, s); if (rc) return rc;
    std::vector<DevBatch> hb(nsrc);
    for (uint32_t i = 0; i < nsrc; i++) {
        std::memset(&hb[i], 0, sizeof(DevBatch));
        hb[i].tuples = records + static_cast<size_t>(offs_h[i]) * h->ops->result_bytes; hb[i].n = offs_h[i + 1] - offs_h[i]; hb[i].watermark = wms_h[i];
    }
    { int rc_ = h->ts.stage.h2d(g.d_batches, hb.data(), sizeof(DevBatch) * nsrc, s); if (rc_) return rc_; }
    { int rc_ = h->ts.stage.h2d(g.batch_off, offs_h, sizeof(uint32_t) * (nsrc + 1), s); if (rc_) return rc_; }
    g.nbatches = nsrc; g.total = total; g.lifted_src = records;
    FfatDev ff = h->ff;
    ff.seg_cnt = g.seg_cnt; ff.trig = g.trig; ff.n_trig = g.n_trig; ff.trig_cap = static_cast<uint32_t>(g.trig.capacity()); ff.n_heavy = g.n_heavy;
    rc = RadixSorter::prepare_wide(g.sort_ctl, s); if (rc) return rc; // (buckets at or above bps stay empty)
    h->mark(0, s); h->mark(1, s);
    MgRuns runs;
    for (uint32_t i = 0; i <= MAX_SHARDS; i++) runs.off[i] = offs_h[std::min(i, nsrc)];
    // the sources' 1024 bins are shared by all destinations: split every coarse bucket so that the update kernel gets (up to) 1024 buckets
    uint32_t nsub = 1, shift2 = shift;
    while (nsub * 2 * bps <= OSW_DIGITS && nsub * 2 <= MAX_SHARDS && shift2 > 0) { nsub *= 2; shift2--; }
    CK(h->mg_scratch.ensure(3 * OSW_DIGITS * MAX_SHARDS));
    uint32_t *cnt3 = h->mg_scratch, *off3 = cnt3 + OSW_DIGITS * MAX_SHARDS, *run_starts = off3 + OSW_DIGITS * MAX_SHARDS;
    const dim3 grid(bps, nsrc);
    // a record's index is its receive position, and the bucket list holds positions below BKL_RANGE_POS: ranges of receive positions,
    // each split, updated and queried before the next (every key's items are in increasing receive position: k_mg_split)
    const uint64_t npos = offs_h[nsrc];
    for (uint64_t lo = 0; lo < npos; lo += BKL_RANGE_POS) {
        const uint32_t lo32 = static_cast<uint32_t>(lo), hi32 = static_cast<uint32_t>(std::min<uint64_t>(npos, lo + BKL_RANGE_POS));
        if (lo != 0) { k_results_pre_append<<<1, 1, 0, s>>>(ff.results_total, n_out_dev); h->launches++; }
        k_mg_count<<<grid, MG_THREADS, 0, s>>>(bins, nsrc, bps, runs, recv_slots, slot_mask, shift2, nsub, cnt3, run_starts, g.n_trig, g.n_heavy, lo32, hi32);
        k_mg_scan<<<1, 1024, 0, s>>>(cnt3, bps * nsub * nsrc, nsrc, off3, g.sort_ctl);
        k_mg_split<<<grid, MG_THREADS, 0, s>>>(bins, nsrc, bps, runs, recv_slots, slot_mask, shift2, nsub, off3, run_starts, g.slotsB, lo32, hi32);
        CK(cudaGetLastError());
        h->mark(2, s);
        rc = h->ops->ffat_buckets(ff, records + lo * h->ops->result_bytes, g.slotsB, lo32, g.sort_ctl, shift2, 0u, g.batch_off, g.d_batches, nsrc,
                                  static_cast<unsigned char *>(out_results), out_ts, out_capacity, n_out_dev, s, h->pp());
        if (rc) return rc;
        rc = h->ops->ffat_windows(ff, g.batch_off, g.d_batches, nsrc, static_cast<unsigned char *>(out_results), out_ts, out_capacity, static_cast<uint32_t>(g_num_sms) * 4u, s,
                                  h->pp(), n_out_dev);
        if (rc) return rc;
        h->launches += 5;
    }
    h->mark(3, s);
    if (h->timing && h->tev_used < wfb_ffat::TEV_MAX) h->tev_used++;
    h->call_no++;
    return 0;
}

int wfb_ffat_flush(wfb_ffat_t *h, void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, void *stream)
{
    if (!h || !n_out_dev || (out_capacity && !out_results)) return WFB_E_BADARG;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (!h->pipelined) { CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t), s)); return 0; }
    int rc = h->ts.enter(s); if (rc) return rc;
    // at most one segment is pending: the one of the last call
    SegScratch &last = h->seg[(h->call_no + 1) & 1u];
    return ffat_deliver(h, last, static_cast<unsigned char *>(out_results), out_ts, out_capacity, n_out_dev, s);
}

int wfb_ffat_timing(wfb_ffat_t *h, int enable, float *ms_h, uint32_t *calls_h)
{
    if (!h) return WFB_E_BADARG;
    float acc[4] = {0, 0, 0, 0};
    if (h->tev_used) {
        CK(cudaEventSynchronize(h->tev[(h->tev_used - 1) * 4 + 3]));
        for (uint32_t i = 0; i < h->tev_used; i++) {
            float a = 0, b = 0, c = 0, d = 0;
            cudaEvent_t *e = &h->tev[i * 4];
            CK(cudaEventElapsedTime(&a, e[0], e[1]));
            CK(cudaEventElapsedTime(&b, e[1], e[2]));
            CK(cudaEventElapsedTime(&c, e[2], e[3]));
            CK(cudaEventElapsedTime(&d, e[0], e[3]));
            acc[0] += a; acc[1] += b; acc[2] += c; acc[3] += d;
        }
    }
    if (ms_h) for (int i = 0; i < 4; i++) ms_h[i] = acc[i];
    if (calls_h) *calls_h = h->tev_used;
    h->tev_used = 0;
    if (enable && h->tev.empty()) {
        h->tev.resize(wfb_ffat::TEV_MAX * 4);
        for (auto &e : h->tev) CK(cudaEventCreate(&e));
    }
    h->timing = enable != 0;
    return 0;
}

int wfb_ffat_stats(wfb_ffat_t *h, uint32_t *n_keys_h, uint32_t *err_flags_h, void *stream)
{
    if (!h) return WFB_E_BADARG;
    uint32_t v[2] = {0, 0};
    int rc = h->ts.enter(static_cast<cudaStream_t>(stream)); if (rc) return rc; // (the counters of a call issued on another stream)
    if (h->s2) CK(cudaStreamSynchronize(h->s2));
    CK(cudaMemcpyAsync(v, h->ff.n_slots, sizeof(v), cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(stream)));
    CK(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
    if (n_keys_h) *n_keys_h = v[0];
    if (err_flags_h) *err_flags_h = v[1];
    if (h->cb && err_flags_h) { uint32_t e2 = 0; rc = wfb_ffat_stats(h->cb, nullptr, &e2, stream); if (rc) return rc; *err_flags_h |= e2; }
    return 0;
}

int wfb_ffat_results_total(wfb_ffat_t *h, uint64_t *total_h, void *stream)
{
    if (!h || !total_h) return WFB_E_BADARG;
    wfb_ffat *src = h->cb ? h->cb : h; // time-based handles: the count-based back end emits the results
    int rc = h->ts.enter(static_cast<cudaStream_t>(stream)); if (rc) return rc;
    if (src != h) { rc = src->ts.enter(static_cast<cudaStream_t>(stream)); if (rc) return rc; }
    unsigned long long v = 0;
    if (src->s2) CK(cudaStreamSynchronize(src->s2));
    if (src->ff.results_total == nullptr) { *total_h = 0; return 0; }
    CK(cudaMemcpyAsync(&v, src->ff.results_total, sizeof(v), cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(stream)));
    CK(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
    *total_h = v;
    return 0;
}

// ---- key-sharded pipeline across GPUs ------------------------------------------------------------------------------------------------
} // extern "C"
#include <dlfcn.h>
namespace {
// the few NCCL entry points used, resolved at run time (the library a torch process has already loaded, or the system one)
struct Nccl {
    struct Id { char b[128]; }; // ncclUniqueId (passed by value)
    typedef int (*GetUniqueId_t)(void *);
    typedef int (*CommInitRank_t)(void **, int, Id, int);
    typedef int (*CommDestroy_t)(void *);
    typedef int (*SendRecv_t)(void *, size_t, int, int, void *, cudaStream_t);
    typedef int (*Group_t)();
    typedef const char *(*ErrStr_t)(int);
    void *lib = nullptr;
    GetUniqueId_t GetUniqueId = nullptr; CommInitRank_t CommInitRank = nullptr; CommDestroy_t CommDestroy = nullptr;
    SendRecv_t Send = nullptr, Recv = nullptr; Group_t GroupStart = nullptr, GroupEnd = nullptr;
    bool ok = false;
    Nccl()
    {
        const char *names[] = {std::getenv("WFB_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char *n : names) { if (n && (lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL))) break; }
        if (!lib) return;
        GetUniqueId = reinterpret_cast<GetUniqueId_t>(dlsym(lib, "ncclGetUniqueId"));
        CommInitRank = reinterpret_cast<CommInitRank_t>(dlsym(lib, "ncclCommInitRank"));
        CommDestroy = reinterpret_cast<CommDestroy_t>(dlsym(lib, "ncclCommDestroy"));
        Send = reinterpret_cast<SendRecv_t>(dlsym(lib, "ncclSend")); Recv = reinterpret_cast<SendRecv_t>(dlsym(lib, "ncclRecv"));
        GroupStart = reinterpret_cast<Group_t>(dlsym(lib, "ncclGroupStart")); GroupEnd = reinterpret_cast<Group_t>(dlsym(lib, "ncclGroupEnd"));
        ok = GetUniqueId && CommInitRank && CommDestroy && Send && Recv && GroupStart && GroupEnd;
    }
};
Nccl &nccl() { static Nccl n; return n; }
constexpr int NCCL_UINT8 = 1; // ncclUint8
#define NK(call) do { int r__ = (call); if (r__ != 0) return 1000 + r__; } while (0) // (NCCL errors: 1000 + ncclResult_t)

__global__ void k_mg_meta(const uint32_t *__restrict__ counts, uint64_t watermark, uint32_t nranks, uint64_t *__restrict__ send_meta)
{
    const uint32_t d = threadIdx.x;
    if (d < nranks) { send_meta[2 * d] = counts[d]; send_meta[2 * d + 1] = watermark; }
}

// appended results (wfb_mg_flush): the call about to run adds the WHOLE count of the output buffer to the handle's total

struct MgSlot { // buffers of one step in flight (three: the exchange of step i-2 overlaps the source pass of step i)
    Scratch<unsigned char> regions;            // records by destination (bucketed: bin after bin, as many as the segment's positions)
    uint32_t region_cap = 0;                   // not bucketed: records per destination region (the stride of `regions`)
    Scratch<uint32_t> vslots;                  // bucketed: virtual slot of every record of `regions`
    uint32_t *bins = nullptr;                  // bucketed: OSW_DIGITS + 1 words, the bin sizes of this step's partition
    uint32_t *recv_slots = nullptr, *recv_bins = nullptr; size_t recv_slots_cap = 0; // bucketed: what the sources delivered ([nranks][bps] run lengths)
    unsigned char *ce_buf = nullptr;           // copy-engine exchange: the receive buffers of this slot in ONE allocation other ranks map (cudaIpc):
                                               // [records n x cap][slots n x cap][run lengths n x bps], source s at stride cap
    unsigned char *peer[MAX_SHARDS] = {};      // every rank's ce_buf of this slot, mapped here
    uint32_t offs[MAX_SHARDS + 1] = {}; uint64_t wms[MAX_SHARDS] = {}; // where every source's records start in `recv` / their watermarks (host, set by the exchange)
    uint32_t *counts = nullptr;                // MAX_SHARDS + 1 (device)
    uint64_t *send_meta = nullptr, *recv_meta = nullptr; // [nranks][2] (device)
    uint32_t *h_counts = nullptr; uint64_t *h_recv = nullptr; // pinned copies
    unsigned char *recv = nullptr; size_t recv_bytes = 0;
    cudaEvent_t ev_src = nullptr, ev_meta = nullptr, ev_a2a = nullptr, ev_done = nullptr, ev_self = nullptr, ev_fork = nullptr;
    bool used = false, done_recorded = false, exchanged = false;
    cudaEvent_t tr[8] = {}; bool tr_valid = false; // WFB_MG_TRACE: source begin/end, update begin/end (caller's stream); exchange begin/end, sizes begin/end (communication stream)
};
} // namespace

struct wfb_mg {
    int nranks = 1, rank = 0;
    void *comm = nullptr;
    wfb_engine_t *eng = nullptr;
    wfb_ffat_t *ffat = nullptr;
    size_t rb = 0;
    MgSlot slot[4];            // four steps in flight: step i's source pass, step i-1 waiting, step i-2 travelling, step i-3 being updated
    cudaStream_t cs = nullptr; // communication stream
    cudaStream_t cs2 = nullptr; // the rank's own share of an exchange: device-to-device copies (copy engine), next to the NCCL group
    uint64_t step_no = 0;
    MgSlot *pend[3] = {nullptr, nullptr, nullptr}; int npend = 0; // steps not yet updated, oldest first (the oldest of three has been exchanged)
    std::vector<wfb_batch_t> chunks;
    // bucketed exchange: the source partitions by (destination, bucket of the destination's slot space), the destination only concatenates runs
    // copy-engine exchange (bucketed mode, all ranks on one node): records are PUSHED into the peers' receive buffers with plain
    // device-to-device copies over NVLink (no SM, no NCCL channel limit); the next step's size exchange is the completion signal
    bool ce = false, ce_tried = false; uint64_t ce_cap = 0, peer_cap[MAX_SHARDS] = {};
    unsigned char *ce_msg = nullptr; // device staging of the handle exchange
    cudaEvent_t ev_flush = nullptr;
    static constexpr int CE_STREAMS = 4;
    cudaStream_t ce_s[CE_STREAMS] = {}; cudaEvent_t ce_ev[CE_STREAMS] = {}; // peer copies of one exchange are spread over these (several copy engines)
    uint32_t *tok = nullptr;            // device words of the completion tokens: [0] sent, [1 + p] received from p
    cudaEvent_t last_done = nullptr;    // end of the most recently issued window update (caller's stream)
    double host_acc[3] = {}; uint64_t host_n = 0;
    bool trace = false; double tr_acc[8] = {}; uint64_t tr_n = 0; // WFB_MG_TRACE=1: device timeline of a step, printed every 64 steps (tuning aid)
    bool bucketed = false;
    uint32_t shard_slots = 0, shard_keys = 0, shift = 0, bps = 0; // slots per destination (power of two), keys per destination, bucket = slot >> shift, buckets per destination
};

extern "C" {

int wfb_mg_unique_id(void *id128_h)
{
    if (!id128_h) return WFB_E_BADARG;
    if (!nccl().ok) return WFB_E_UNSUPPORTED;
    NK(nccl().GetUniqueId(id128_h));
    return 0;
}

int wfb_mg_destroy(wfb_mg_t *h)
{
    if (!h) return 0;
    cudaDeviceSynchronize();
    if (h->comm && nccl().ok) nccl().CommDestroy(h->comm);
    if (h->eng) wfb_engine_destroy(h->eng);
    if (h->ffat) wfb_ffat_destroy(h->ffat);
    for (MgSlot &sl : h->slot) {
        cudaFree(sl.counts); cudaFree(sl.send_meta); cudaFree(sl.recv_meta); if (!sl.ce_buf) cudaFree(sl.recv);
        cudaFree(sl.bins);
        if (sl.ce_buf) { // (recv / recv_slots / recv_bins point into ce_buf)
            for (int p = 0; p < h->nranks; p++) if (p != h->rank && sl.peer[p]) cudaIpcCloseMemHandle(sl.peer[p]);
            cudaFree(sl.ce_buf); sl.recv = nullptr;
        } else { cudaFree(sl.recv_slots); cudaFree(sl.recv_bins); }
        if (sl.h_counts) cudaFreeHost(sl.h_counts);
        if (sl.h_recv) cudaFreeHost(sl.h_recv);
        for (cudaEvent_t e : {sl.ev_src, sl.ev_meta, sl.ev_a2a, sl.ev_done, sl.ev_self, sl.ev_fork}) if (e) cudaEventDestroy(e);
        for (cudaEvent_t e : sl.tr) if (e) cudaEventDestroy(e);
    }
    if (h->cs) cudaStreamDestroy(h->cs);
    if (h->cs2) cudaStreamDestroy(h->cs2);
    cudaFree(h->ce_msg); cudaFree(h->tok);
    if (h->ev_flush) cudaEventDestroy(h->ev_flush);
    for (cudaStream_t st : h->ce_s) if (st) cudaStreamDestroy(st);
    for (cudaEvent_t e : h->ce_ev) if (e) cudaEventDestroy(e);
    delete h;
    cudaGetLastError();
    return 0;
}

int wfb_mg_create(wfb_mg_t **hh, int prog, int nranks, int rank, const void *id128_h, uint64_t win, uint64_t slide, uint32_t wins_per_batch,
                  uint32_t max_keys_total)
{
    if (!hh || nranks < 1 || nranks > static_cast<int>(MAX_SHARDS) || rank < 0 || rank >= nranks || (nranks > 1 && !id128_h) || max_keys_total == 0) return WFB_E_BADARG;
    const ProgramOps *o = program(prog);
    if (!o) return WFB_E_NOPROG;
    const int lp = lifted_program_of(prog);
    if (lp < 0 || !(program(lp)->reserved2 & 1u)) return WFB_E_UNSUPPORTED; // the lifted records must carry their key (Program::result_key)
    if (o->key_kind != KEY_KIND_INTEGRAL) return WFB_E_UNSUPPORTED;            // shards are key % nranks: integer keys only
    int rc = device_ready(); if (rc) return rc;
    if (nranks > 1 && !nccl().ok) return WFB_E_UNSUPPORTED;
    wfb_mg *h = new (std::nothrow) wfb_mg();
    if (!h) return WFB_E_BADARG;
    h->nranks = nranks; h->rank = rank; h->rb = o->result_bytes;
    h->trace = std::getenv("WFB_MG_TRACE") && std::atoi(std::getenv("WFB_MG_TRACE")) != 0;
#define MGCK(call) do { int r__ = (call); if (r__) { wfb_mg_destroy(h); return r__; } } while (0)
    MGCK(wfb_engine_create(&h->eng, prog));
    // the rank's replica owns the keys with key % nranks == rank: compact slots key / nranks, records read in place
    MGCK(wfb_ffat_create(&h->ffat, lp, win, slide, wins_per_batch, (max_keys_total + nranks - 1) / nranks, 0, 0, WFB_FFAT_DENSE_KEYS));
    if (nranks > 1) MGCK(wfb_ffat_set_key_shard(h->ffat, static_cast<uint32_t>(nranks), static_cast<uint32_t>(rank)));
    MGCK(static_cast<int>(cudaStreamCreateWithFlags(&h->cs, cudaStreamNonBlocking)));
    MGCK(static_cast<int>(cudaStreamCreateWithFlags(&h->cs2, cudaStreamNonBlocking)));
    MGCK(static_cast<int>(cudaEventCreateWithFlags(&h->ev_flush, cudaEventDisableTiming)));
    {   // bucketed exchange when the destination-major virtual slots fit 16 bits (they travel packed with a 16-bit rank)
        const uint32_t keys = (max_keys_total + nranks - 1) / nranks;
        uint32_t L = 1; while (L < keys) L <<= 1;
        static const bool off = std::getenv("WFB_MG_BUCKETED") && std::atoi(std::getenv("WFB_MG_BUCKETED")) == 0;
        const size_t rb = o->result_bytes;
        if (!off && static_cast<uint64_t>(L) * nranks <= 65536u && h->ffat->buckets && (rb == 16 || rb == 24 || rb == 32 || rb == 48 || rb == 64)) {
            uint32_t span = 1; while (span < L * static_cast<uint32_t>(nranks)) span <<= 1; // virtual slot space, rounded up
            uint32_t sh = 0; while ((span >> sh) > OSW_DIGITS) sh++;
            if ((L >> sh) >= 1) { h->bucketed = true; h->shard_slots = L; h->shard_keys = keys; h->shift = sh; h->bps = L >> sh; }
        }
    }
    for (MgSlot &sl : h->slot) {
        if (h->bucketed) {
            MGCK(static_cast<int>(cudaMalloc(&sl.bins, sizeof(uint32_t) * (OSW_DIGITS + 1))));
            MGCK(static_cast<int>(cudaMalloc(&sl.recv_bins, sizeof(uint32_t) * MAX_SHARDS * OSW_DIGITS)));
        }
        MGCK(static_cast<int>(cudaMalloc(&sl.counts, sizeof(uint32_t) * (MAX_SHARDS + 1))));
        MGCK(static_cast<int>(cudaMalloc(&sl.send_meta, sizeof(uint64_t) * 2 * MAX_SHARDS)));
        MGCK(static_cast<int>(cudaMalloc(&sl.recv_meta, sizeof(uint64_t) * 2 * MAX_SHARDS)));
        MGCK(static_cast<int>(cudaMallocHost(&sl.h_counts, sizeof(uint32_t) * (MAX_SHARDS + 1))));
        MGCK(static_cast<int>(cudaMallocHost(&sl.h_recv, sizeof(uint64_t) * 2 * MAX_SHARDS)));
        for (cudaEvent_t *e : {&sl.ev_src, &sl.ev_meta, &sl.ev_a2a, &sl.ev_done, &sl.ev_self, &sl.ev_fork}) MGCK(static_cast<int>(cudaEventCreateWithFlags(e, cudaEventDisableTiming)));
        if (h->trace) for (cudaEvent_t &e : sl.tr) MGCK(static_cast<int>(cudaEventCreate(&e)));
    }
    if (nranks > 1) {
        Nccl::Id id; std::memcpy(id.b, id128_h, sizeof(id.b));
        int r = nccl().CommInitRank(&h->comm, nranks, id, rank);
        if (r != 0) { wfb_mg_destroy(h); return 1000 + r; }
    }
#undef MGCK
    *hh = h;
    return 0;
}

int wfb_mg_set_params(wfb_mg_t *h, const void *params, size_t bytes)
{
    if (!h) return WFB_E_BADARG;
    // the source engine (map / filter / key / lift when a step passes no `pre`) and the destination window operator (its key
    // extractor on the lifted records, comb and make_result): LiftedOf<P> shares P's params_t, so one size fits both
    int rc = wfb_engine_set_params(h->eng, params, bytes); if (rc) return rc;
    return wfb_ffat_set_params(h->ffat, params, bytes);
}

// ---- copy-engine exchange: setup (collective, at the first step) ---------------------------------------------------------------
struct CeLayout { size_t slots_off, bins_off, bytes; };
static CeLayout ce_layout(uint64_t cap, int n, size_t rb, uint32_t bps)
{
    CeLayout l; l.slots_off = static_cast<size_t>(n) * cap * rb; l.bins_off = (l.slots_off + static_cast<size_t>(n) * cap * 4 + 255) & ~static_cast<size_t>(255);
    l.bytes = l.bins_off + static_cast<size_t>(n) * bps * 4; return l;
}
constexpr int MG_SLOTS = 4;
struct CeMsg { cudaIpcMemHandle_t h[MG_SLOTS]; uint64_t cap; uint64_t ok; };
// one small message to / from every other rank (communication stream, synchronous)
static int mg_all_exchange(wfb_mg *h, const void *mine_h, void *all_h, size_t bytes)
{
    const int n = h->nranks;
    if (!h->ce_msg) CK(cudaMalloc(&h->ce_msg, sizeof(CeMsg) * (MAX_SHARDS + 1)));
    if (bytes > sizeof(CeMsg)) return WFB_E_BADARG;
    unsigned char *snd = h->ce_msg, *rcv = h->ce_msg + sizeof(CeMsg);
    CK(cudaMemcpyAsync(snd, mine_h, bytes, cudaMemcpyHostToDevice, h->cs));
    NK(nccl().GroupStart());
    for (int p = 0; p < n; p++) {
        if (p == h->rank) continue;
        NK(nccl().Send(snd, bytes, NCCL_UINT8, p, h->comm, h->cs));
        NK(nccl().Recv(rcv + static_cast<size_t>(p) * bytes, bytes, NCCL_UINT8, p, h->comm, h->cs));
    }
    NK(nccl().GroupEnd());
    CK(cudaMemcpyAsync(all_h, rcv, bytes * n, cudaMemcpyDeviceToHost, h->cs));
    CK(cudaStreamSynchronize(h->cs));
    std::memcpy(static_cast<unsigned char *>(all_h) + static_cast<size_t>(h->rank) * bytes, mine_h, bytes);
    return 0;
}
static int mg_ce_setup(wfb_mg *h, uint64_t positions)
{
    h->ce_tried = true;
    static const bool off = std::getenv("WFB_MG_CE") && std::atoi(std::getenv("WFB_MG_CE")) == 0;
    if (off || !h->bucketed || h->nranks < 2) return 0;
    const int n = h->nranks;
    const uint64_t cap = (positions + 1023) & ~1023ull; // worst case: every survivor of a source's step goes to one destination
    const CeLayout l = ce_layout(cap, n, h->rb, h->bps);
    CeMsg mine; std::memset(&mine, 0, sizeof(mine)); mine.cap = cap; mine.ok = 1;
    for (int i = 0; i < MG_SLOTS && mine.ok; i++) {
        if (cudaMalloc(&h->slot[i].ce_buf, l.bytes) != cudaSuccess || cudaIpcGetMemHandle(&mine.h[i], h->slot[i].ce_buf) != cudaSuccess) mine.ok = 0;
    }
    cudaGetLastError();
    CeMsg all[MAX_SHARDS];
    int rc = mg_all_exchange(h, &mine, all, sizeof(CeMsg)); if (rc) return rc;
    uint64_t ok = 1;
    for (int p = 0; p < n; p++) ok &= all[p].ok;
    if (ok) {
        for (int p = 0; p < n && ok; p++) {
            h->peer_cap[p] = all[p].cap;
            for (int i = 0; i < MG_SLOTS && ok; i++) {
                if (p == h->rank) { h->slot[i].peer[p] = h->slot[i].ce_buf; continue; }
                void *ptr = nullptr;
                if (cudaIpcOpenMemHandle(&ptr, all[p].h[i], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = 0; cudaGetLastError(); }
                else h->slot[i].peer[p] = static_cast<unsigned char *>(ptr);
            }
        }
    }
    // second round: every rank could map every buffer, or nobody uses the path
    uint64_t st_mine = ok, st_all[MAX_SHARDS];
    rc = mg_all_exchange(h, &st_mine, st_all, sizeof(uint64_t)); if (rc) return rc;
    for (int p = 0; p < n; p++) ok &= st_all[p];
    if (!ok) {
        for (MgSlot &sl : h->slot) {
            for (int p = 0; p < n; p++) { if (p != h->rank && sl.peer[p]) cudaIpcCloseMemHandle(sl.peer[p]); sl.peer[p] = nullptr; }
            cudaFree(sl.ce_buf); sl.ce_buf = nullptr;
        }
        cudaGetLastError();
        if (h->trace) std::fprintf(stderr, "[wfb_mg rank %d] copy-engine exchange not available (cudaIpc): NCCL exchange\n", h->rank);
        return 0; // (the NCCL exchange stays in use)
    }
    for (int i = 0; i < wfb_mg::CE_STREAMS; i++) { CK(cudaStreamCreateWithFlags(&h->ce_s[i], cudaStreamNonBlocking)); CK(cudaEventCreateWithFlags(&h->ce_ev[i], cudaEventDisableTiming)); }
    CK(cudaMalloc(&h->tok, sizeof(uint32_t) * (MAX_SHARDS + 1)));
    CK(cudaMemset(h->tok, 0, sizeof(uint32_t) * (MAX_SHARDS + 1)));
    h->ce = true; h->ce_cap = cap;
    if (h->trace) std::fprintf(stderr, "[wfb_mg rank %d] copy-engine exchange enabled (capacity %llu records per source)\n", h->rank, static_cast<unsigned long long>(cap));
    for (MgSlot &sl : h->slot) {
        cudaFree(sl.recv); cudaFree(sl.recv_slots); cudaFree(sl.recv_bins);
        sl.recv = sl.ce_buf; sl.recv_slots = reinterpret_cast<uint32_t *>(sl.ce_buf + l.slots_off); sl.recv_bins = reinterpret_cast<uint32_t *>(sl.ce_buf + l.bins_off);
        sl.recv_bytes = l.slots_off; sl.recv_slots_cap = static_cast<size_t>(n) * cap;
    }
    return 0;
}

// source side of a step: fused pass + partition by destination; the sizes travel (and reach the host a step later)
static int mg_source(wfb_mg *h, MgSlot &sl, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches, uint64_t watermark, cudaStream_t s)
{
    uint64_t n = 0;
    for (uint32_t i = 0; i < nbatches; i++) n += batches_h[i].n;
    if (n > 0x7fffffffull) return WFB_E_BADARG;
    int rc;
    if (h->trace) {
        if (sl.tr_valid) { // this slot's previous step (three calls ago) is complete: add its timeline
            CK(cudaEventSynchronize(sl.tr[3]));
            float ms; const int pairs[6][2] = {{0, 1}, {2, 3}, {4, 5}, {6, 7}, {4, 2}, {5, 2}};
            for (int i = 0; i < 6; i++) if (cudaEventElapsedTime(&ms, sl.tr[pairs[i][0]], sl.tr[pairs[i][1]]) == cudaSuccess) h->tr_acc[i] += ms;
            if (++h->tr_n % 64 == 0) {
                std::fprintf(stderr, "[wfb_mg rank %d] us/step over 64 steps: source %.0f | update %.0f | exchange %.0f | sizes %.0f | exchange begin -> update begin %.0f | exchange end -> update begin %.0f\n",
                             h->rank, h->tr_acc[0] / 64 * 1e3, h->tr_acc[1] / 64 * 1e3, h->tr_acc[2] / 64 * 1e3, h->tr_acc[3] / 64 * 1e3, h->tr_acc[4] / 64 * 1e3, h->tr_acc[5] / 64 * 1e3);
                for (double &a : h->tr_acc) a = 0;
            }
            sl.tr_valid = false;
        }
        CK(cudaEventRecord(sl.tr[0], s));
    }
    const ScratchWaits waits = sl.used ? ScratchWaits::device() : ScratchWaits(); // (the exchange of the slot's last step reads the regions)
    if (h->bucketed) {
        uint64_t positions = 0;
        for (uint32_t i = 0; i < nbatches; i++) positions += static_cast<uint64_t>(tiles_of(batches_h[i].n)) * TILE;
        if (!h->ce_tried) { rc = mg_ce_setup(h, std::max<uint64_t>(positions, 1)); if (rc) return rc; } // (collective: every rank is in its first step)
        // (at least one tile: a step without tuples on a slot that never held any still hands the partition buffers it accepts)
        const uint64_t room = std::max<uint64_t>(positions, TILE);
        CK(sl.vslots.ensure(room, waits, room));
        CK(sl.regions.ensure(room * h->rb, waits, room * h->rb));
        rc = shard_lift_impl(h->eng, pre, batches_h, nbatches, static_cast<uint32_t>(h->nranks), sl.regions, static_cast<uint32_t>(sl.vslots.capacity()), sl.counts, s,
                             h->shard_slots, h->shard_keys, h->shift, sl.vslots, sl.bins, n ? sl.send_meta : nullptr, watermark);
    } else {
        const size_t region_bytes = static_cast<size_t>(h->nranks) * h->rb; // worst case: every item of the segment survives and goes to one shard
        const uint64_t room = std::max<uint64_t>(n, 1); // (a step without tuples: regions of one record, not none)
        CK(sl.regions.ensure(room * region_bytes, waits, room * region_bytes));
        sl.region_cap = static_cast<uint32_t>(sl.regions.capacity() / region_bytes);
        rc = wfb_shard_lift(h->eng, pre, batches_h, nbatches, static_cast<uint32_t>(h->nranks), sl.regions, sl.region_cap, sl.counts, s);
    }
    if (rc) return rc;
    if (!(h->bucketed && n)) { // (bucketed: the kernel that sums the bins per destination wrote the pairs)
        k_mg_meta<<<1, 32, 0, s>>>(sl.counts, watermark, static_cast<uint32_t>(h->nranks), sl.send_meta);
        CK(cudaGetLastError());
    }
    CK(cudaEventRecord(sl.ev_src, s));
    if (h->trace) CK(cudaEventRecord(sl.tr[1], s));
    CK(cudaStreamWaitEvent(h->cs, sl.ev_src, 0));
    if (h->trace) CK(cudaEventRecord(sl.tr[6], h->cs));
    if (h->nranks > 1) {
        NK(nccl().GroupStart());
        for (int p = 0; p < h->nranks; p++) {
            NK(nccl().Send(sl.send_meta + 2 * p, 16, NCCL_UINT8, p, h->comm, h->cs));
            NK(nccl().Recv(sl.recv_meta + 2 * p, 16, NCCL_UINT8, p, h->comm, h->cs));
        }
        NK(nccl().GroupEnd());
    } else CK(cudaMemcpyAsync(sl.recv_meta, sl.send_meta, 16, cudaMemcpyDeviceToDevice, h->cs));
    CK(cudaMemcpyAsync(sl.h_counts, sl.counts, sizeof(uint32_t) * (MAX_SHARDS + 1), cudaMemcpyDeviceToHost, h->cs));
    CK(cudaMemcpyAsync(sl.h_recv, sl.recv_meta, sizeof(uint64_t) * 2 * h->nranks, cudaMemcpyDeviceToHost, h->cs));
    CK(cudaEventRecord(sl.ev_meta, h->cs));
    if (h->trace) CK(cudaEventRecord(sl.tr[7], h->cs));
    sl.used = true;
    return 0;
}

// exchange of the records of a step, on the communication stream (issued BEFORE the next step's source pass so that it runs next to it)
static int mg_exchange(wfb_mg *h, MgSlot &sl)
{
    CK(cudaEventSynchronize(sl.ev_meta)); // the sizes of this step on the host (a step old: no stall)
    if (sl.h_counts[MAX_SHARDS]) return WFB_E_CAPACITY; // a shard region overflowed / a key outside the declared key space
    const int n = h->nranks;
    if (h->bucketed) {
        // records, their slots and the run lengths of every source; source-rank order = global stream order
        uint64_t tot = 0;
        for (int p = 0; p < n; p++) { sl.offs[p] = static_cast<uint32_t>(tot); tot += sl.h_recv[2 * p]; sl.wms[p] = sl.h_recv[2 * p + 1]; }
        if (tot > 0x7fffffffull) return WFB_E_CAPACITY;
        sl.offs[n] = static_cast<uint32_t>(tot);
        if (h->ce) {
            // push: this rank's records for peer p go straight into p's receive buffer of this slot, at the stride-cap region of source `rank`
            const uint64_t cap = h->ce_cap;
            if (static_cast<uint64_t>(n) * cap > 0x7fffffffull) return WFB_E_CAPACITY;
            for (int p = 0; p <= n; p++) sl.offs[p] = static_cast<uint32_t>(p * cap);
            size_t send_off[MAX_SHARDS + 1]; send_off[0] = 0;
            for (int p = 0; p < n; p++) {
                send_off[p + 1] = send_off[p] + sl.h_counts[p];
                if (sl.h_recv[2 * p] > cap || sl.h_counts[p] > h->peer_cap[p]) return WFB_E_CAPACITY; // (a step larger than the first one: WFB_MG_CE=0)
            }
            const int slot_idx = static_cast<int>(&sl - h->slot);
            const size_t bin_bytes = sizeof(uint32_t) * h->bps;
            if (h->trace) CK(cudaEventRecord(sl.tr[4], h->cs));
            CK(cudaStreamWaitEvent(h->cs2, sl.ev_src, 0));
            if (sl.done_recorded) CK(cudaStreamWaitEvent(h->cs2, sl.ev_done, 0));
            // the peers' shares: plain copies (copy engines, no SM; 450 GB/s to one peer, ~250 GB/s aggregate with 7 peers x 3 pieces each), or --
            // WFB_MG_PUSH=sm -- one kernel that stores into the mapped buffers (16 CTAs per peer; 205 instead of 465 us at N = 8, same step time:
            // the exchange is hidden behind the source pass either way)
            static const char *push_env = std::getenv("WFB_MG_PUSH");
            const bool use_sm = push_env && std::strcmp(push_env, "sm") == 0 && h->rb % 16 == 0;
            {   // own share: a local copy next to the rest
                const int p = h->rank;
                const CeLayout l = ce_layout(h->peer_cap[p], n, h->rb, h->bps);
                unsigned char *dst = h->slot[slot_idx].peer[p];
                const uint64_t me = static_cast<uint64_t>(h->rank), pc = h->peer_cap[p];
                CK(cudaMemcpyAsync(dst + me * pc * h->rb, sl.regions + send_off[p] * h->rb, static_cast<size_t>(sl.h_counts[p]) * h->rb, cudaMemcpyDeviceToDevice, h->cs2));
                CK(cudaMemcpyAsync(dst + l.slots_off + me * pc * 4, sl.vslots + send_off[p], static_cast<size_t>(sl.h_counts[p]) * 4, cudaMemcpyDeviceToDevice, h->cs2));
                CK(cudaMemcpyAsync(dst + l.bins_off + me * bin_bytes, sl.bins + static_cast<size_t>(p) * h->bps, bin_bytes, cudaMemcpyDeviceToDevice, h->cs2));
                CK(cudaEventRecord(sl.ev_self, h->cs2));
            }
            if (use_sm) {
                MgPush a; std::memset(&a, 0, sizeof(a));
                int k = 0;
                for (int p = 0; p < n; p++) {
                    if (p == h->rank) continue;
                    const CeLayout l = ce_layout(h->peer_cap[p], n, h->rb, h->bps);
                    unsigned char *dst = h->slot[slot_idx].peer[p];
                    const uint64_t me = static_cast<uint64_t>(h->rank), pc = h->peer_cap[p];
                    a.rec_src[k] = reinterpret_cast<const uint4 *>(sl.regions + send_off[p] * h->rb); a.rec_dst[k] = reinterpret_cast<uint4 *>(dst + me * pc * h->rb);
                    a.rec_n16[k] = static_cast<uint32_t>(static_cast<size_t>(sl.h_counts[p]) * h->rb / 16);
                    a.slot_src[k] = sl.vslots + send_off[p]; a.slot_dst[k] = reinterpret_cast<uint32_t *>(dst + l.slots_off + me * pc * 4); a.slot_n[k] = sl.h_counts[p];
                    a.bin_src[k] = sl.bins + static_cast<size_t>(p) * h->bps; a.bin_dst[k] = reinterpret_cast<uint32_t *>(dst + l.bins_off + me * bin_bytes);
                    k++;
                }
                a.bin_n = h->bps;
                k_mg_push<<<static_cast<uint32_t>(k) * MG_PUSH_CTAS, MG_PUSH_THREADS, 0, h->cs>>>(a);
                CK(cudaGetLastError());
            } else { // several streams (copy engines, different NVLink destinations), forked from the communication stream and joined back
                CK(cudaEventRecord(sl.ev_fork, h->cs));
                const int nst = std::min(wfb_mg::CE_STREAMS, n - 1);
                for (int i = 0; i < nst; i++) CK(cudaStreamWaitEvent(h->ce_s[i], sl.ev_fork, 0));
                int k = 0;
                for (int p = 0; p < n; p++) {
                    if (p == h->rank) continue;
                    const CeLayout l = ce_layout(h->peer_cap[p], n, h->rb, h->bps);
                    unsigned char *dst = h->slot[slot_idx].peer[p];
                    const uint64_t me = static_cast<uint64_t>(h->rank), pc = h->peer_cap[p];
                    cudaStream_t st = h->ce_s[k++ % nst];
                    CK(cudaMemcpyAsync(dst + me * pc * h->rb, sl.regions + send_off[p] * h->rb, static_cast<size_t>(sl.h_counts[p]) * h->rb, cudaMemcpyDeviceToDevice, st));
                    CK(cudaMemcpyAsync(dst + l.slots_off + me * pc * 4, sl.vslots + send_off[p], static_cast<size_t>(sl.h_counts[p]) * 4, cudaMemcpyDeviceToDevice, st));
                    CK(cudaMemcpyAsync(dst + l.bins_off + me * bin_bytes, sl.bins + static_cast<size_t>(p) * h->bps, bin_bytes, cudaMemcpyDeviceToDevice, st));
                }
                for (int i = 0; i < nst; i++) { CK(cudaEventRecord(h->ce_ev[i], h->ce_s[i])); CK(cudaStreamWaitEvent(h->cs, h->ce_ev[i], 0)); }
            }
            if (h->trace) CK(cudaEventRecord(sl.tr[5], h->cs));
            // completion tokens: a peer's token arrives after its copies (its stream order) and after the window update it issued last
            // (so that what this rank pushes NEXT into that peer's buffers overwrites nothing still being read)
            if (h->last_done) CK(cudaStreamWaitEvent(h->cs, h->last_done, 0));
            NK(nccl().GroupStart());
            for (int p = 0; p < n; p++) {
                if (p == h->rank) continue;
                NK(nccl().Send(h->tok, 4, NCCL_UINT8, p, h->comm, h->cs));
                NK(nccl().Recv(h->tok + 1 + p, 4, NCCL_UINT8, p, h->comm, h->cs));
            }
            NK(nccl().GroupEnd());
            CK(cudaEventRecord(sl.ev_a2a, h->cs));
            return 0;
        }
        const size_t need = std::max<size_t>(1, tot);
        if (sl.recv_bytes < need * h->rb || sl.recv_slots_cap < need) {
            CK(cudaDeviceSynchronize());
            cudaFree(sl.recv); cudaFree(sl.recv_slots);
            sl.recv = nullptr; sl.recv_slots = nullptr; sl.recv_bytes = 0; sl.recv_slots_cap = 0; // (as a failed allocation leaves them)
            const size_t cap = need * 5 / 4;
            CK(cudaMalloc(&sl.recv, cap * h->rb)); sl.recv_bytes = cap * h->rb;
            CK(cudaMalloc(&sl.recv_slots, sizeof(uint32_t) * cap)); sl.recv_slots_cap = cap;
        }
        if (sl.done_recorded) CK(cudaStreamWaitEvent(h->cs, sl.ev_done, 0)); // the window update that read these receive buffers two steps ago
        if (h->trace) CK(cudaEventRecord(sl.tr[4], h->cs));
        size_t send_off[MAX_SHARDS + 1]; send_off[0] = 0;
        for (int p = 0; p < n; p++) send_off[p + 1] = send_off[p] + sl.h_counts[p];
        const size_t bin_bytes = sizeof(uint32_t) * h->bps;
        if (n > 1) {
            {   // this rank's own share does not go through NCCL: plain copies on the copy engine, next to the group
                const int p = h->rank;
                CK(cudaStreamWaitEvent(h->cs2, sl.ev_src, 0));
                if (sl.done_recorded) CK(cudaStreamWaitEvent(h->cs2, sl.ev_done, 0));
                CK(cudaMemcpyAsync(sl.recv + static_cast<size_t>(sl.offs[p]) * h->rb, sl.regions + send_off[p] * h->rb, static_cast<size_t>(sl.h_counts[p]) * h->rb, cudaMemcpyDeviceToDevice, h->cs2));
                CK(cudaMemcpyAsync(sl.recv_slots + sl.offs[p], sl.vslots + send_off[p], static_cast<size_t>(sl.h_counts[p]) * 4, cudaMemcpyDeviceToDevice, h->cs2));
                CK(cudaMemcpyAsync(sl.recv_bins + static_cast<size_t>(p) * h->bps, sl.bins + static_cast<size_t>(p) * h->bps, bin_bytes, cudaMemcpyDeviceToDevice, h->cs2));
                CK(cudaEventRecord(sl.ev_self, h->cs2));
            }
            NK(nccl().GroupStart());
            for (int p = 0; p < n; p++) {
                if (p == h->rank) continue;
                NK(nccl().Send(sl.regions + send_off[p] * h->rb, static_cast<size_t>(sl.h_counts[p]) * h->rb, NCCL_UINT8, p, h->comm, h->cs));
                NK(nccl().Recv(sl.recv + static_cast<size_t>(sl.offs[p]) * h->rb, static_cast<size_t>(sl.h_recv[2 * p]) * h->rb, NCCL_UINT8, p, h->comm, h->cs));
                NK(nccl().Send(sl.vslots + send_off[p], static_cast<size_t>(sl.h_counts[p]) * 4, NCCL_UINT8, p, h->comm, h->cs));
                NK(nccl().Recv(sl.recv_slots + sl.offs[p], static_cast<size_t>(sl.h_recv[2 * p]) * 4, NCCL_UINT8, p, h->comm, h->cs));
                NK(nccl().Send(sl.bins + static_cast<size_t>(p) * h->bps, bin_bytes, NCCL_UINT8, p, h->comm, h->cs));
                NK(nccl().Recv(sl.recv_bins + static_cast<size_t>(p) * h->bps, bin_bytes, NCCL_UINT8, p, h->comm, h->cs));
            }
            NK(nccl().GroupEnd());
        } else {
            CK(cudaMemcpyAsync(sl.recv, sl.regions, static_cast<size_t>(sl.h_counts[0]) * h->rb, cudaMemcpyDeviceToDevice, h->cs));
            CK(cudaMemcpyAsync(sl.recv_slots, sl.vslots, static_cast<size_t>(sl.h_counts[0]) * 4, cudaMemcpyDeviceToDevice, h->cs));
            CK(cudaMemcpyAsync(sl.recv_bins, sl.bins, bin_bytes, cudaMemcpyDeviceToDevice, h->cs));
        }
        CK(cudaEventRecord(sl.ev_a2a, h->cs));
        if (h->trace) CK(cudaEventRecord(sl.tr[5], h->cs));
        return 0;
    }
    size_t tiles = 0; // every source's chunk at its tile position of the receive buffer (read in place)
    for (int p = 0; p < n; p++) { sl.offs[p] = static_cast<uint32_t>(tiles * TILE); tiles += (static_cast<size_t>(sl.h_recv[2 * p]) + TILE - 1) / TILE; sl.wms[p] = sl.h_recv[2 * p + 1]; }
    if (tiles * TILE > 0x7fffffffull) return WFB_E_CAPACITY;
    const size_t need = std::max<size_t>(1, tiles * TILE) * h->rb;
    if (sl.recv_bytes < need) {
        CK(cudaDeviceSynchronize());
        cudaFree(sl.recv);
        sl.recv = nullptr; sl.recv_bytes = 0; // (as a failed allocation leaves them)
        CK(cudaMalloc(&sl.recv, need * 5 / 4)); sl.recv_bytes = need * 5 / 4;
    }
    if (sl.done_recorded) CK(cudaStreamWaitEvent(h->cs, sl.ev_done, 0)); // the window update that read this receive buffer two steps ago
    if (h->trace) CK(cudaEventRecord(sl.tr[4], h->cs));
    if (n > 1) {
        NK(nccl().GroupStart());
        for (int p = 0; p < n; p++) {
            NK(nccl().Send(sl.regions + static_cast<size_t>(p) * sl.region_cap * h->rb, static_cast<size_t>(sl.h_counts[p]) * h->rb, NCCL_UINT8, p, h->comm, h->cs));
            NK(nccl().Recv(sl.recv + static_cast<size_t>(sl.offs[p]) * h->rb, static_cast<size_t>(sl.h_recv[2 * p]) * h->rb, NCCL_UINT8, p, h->comm, h->cs));
        }
        NK(nccl().GroupEnd());
    } else CK(cudaMemcpyAsync(sl.recv, sl.regions, static_cast<size_t>(sl.h_counts[0]) * h->rb, cudaMemcpyDeviceToDevice, h->cs));
    CK(cudaEventRecord(sl.ev_a2a, h->cs));
    if (h->trace) CK(cudaEventRecord(sl.tr[5], h->cs));
    return 0;
}

// window update on what mg_exchange delivered (caller's stream)
static int mg_update(wfb_mg *h, MgSlot &sl, void *out, uint64_t *out_ts, uint32_t out_cap, uint32_t *n_out_dev, cudaStream_t s, bool append = false)
{
    const int n = h->nranks;
    CK(cudaStreamWaitEvent(s, sl.ev_a2a, 0));
    if (h->bucketed && n > 1) CK(cudaStreamWaitEvent(s, sl.ev_self, 0));
    if (h->trace) CK(cudaEventRecord(sl.tr[2], s));
    uint64_t items = 0;
    for (int p = 0; p < n; p++) items += sl.h_recv[2 * p];
    if (append && items != 0) { k_results_pre_append<<<1, 1, 0, s>>>(h->ffat->ff.results_total, n_out_dev); CK(cudaGetLastError()); }
    int rc;
    if (h->bucketed) {
        rc = ffat_process_prebucketed(h->ffat, sl.recv, sl.recv_slots, sl.recv_bins, static_cast<uint32_t>(n), h->bps, sl.offs, sl.wms, h->shard_slots - 1u, h->shift,
                                      out, out_ts, out_cap, n_out_dev, s, append, static_cast<uint32_t>(items));
    } else {
        h->chunks.resize(n);
        for (int p = 0; p < n; p++) { // source-rank order = global stream order
            wfb_batch_t &b = h->chunks[p];
            b.tuples = sl.recv + static_cast<size_t>(sl.offs[p]) * h->rb; b.ts = nullptr; b.watermark = sl.wms[p]; b.n = static_cast<uint32_t>(sl.h_recv[2 * p]); b.reserved = 0;
        }
        h->ffat->append_results = append;
        rc = wfb_ffat_process_cb(h->ffat, nullptr, h->chunks.data(), static_cast<uint32_t>(n), out, out_ts, out_cap, n_out_dev, s);
        h->ffat->append_results = false;
    }
    if (rc) return rc;
    CK(cudaEventRecord(sl.ev_done, s));
    h->last_done = sl.ev_done;
    if (h->trace) { CK(cudaEventRecord(sl.tr[3], s)); sl.tr_valid = true; }
    sl.done_recorded = true;
    return 0;
}

int wfb_mg_step(wfb_mg_t *h, const wfb_functors_t *pre, const wfb_batch_t *batches_h, uint32_t nbatches, uint64_t watermark,
                void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, void *stream)
{
    if (!h || !n_out_dev || (nbatches && !batches_h)) return WFB_E_BADARG;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    MgSlot &cur = h->slot[h->step_no % 4];
    h->step_no++;
    // call i: the records of step i-2 start travelling (communication stream; their sizes reached the host a step ago), the source pass
    // of step i runs next to them, then the window update of step i-3 -- whose records arrived during the previous call, so the compute
    // stream never waits for an exchange, and no rank waits for the slowest peer of the step in flight
    MgSlot *ex = h->npend >= 2 ? h->pend[h->npend - 2] : nullptr, *upd = h->npend == 3 ? h->pend[0] : nullptr;
    int rc;
    const double t0 = h->trace ? host_now_us() : 0;
    if (ex != nullptr && !ex->exchanged) { rc = mg_exchange(h, *ex); if (rc) return rc; ex->exchanged = true; }
    const double t1 = h->trace ? host_now_us() : 0;
    rc = mg_source(h, cur, pre, batches_h, nbatches, watermark, s); if (rc) return rc;
    const double t2 = h->trace ? host_now_us() : 0;
    cur.exchanged = false;
    if (upd != nullptr) { h->pend[0] = h->pend[1]; h->pend[1] = h->pend[2]; h->pend[2] = &cur; } else h->pend[h->npend++] = &cur;
    if (upd == nullptr) { CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t), s)); return 0; }
    rc = mg_update(h, *upd, out_results, out_ts, out_capacity, n_out_dev, s);
    upd->exchanged = false;
    if (h->trace) { // host time spent ISSUING the three parts of a step (includes any wait for a pinned staging slot)
        const double t3 = host_now_us();
        h->host_acc[0] += t1 - t0; h->host_acc[1] += t2 - t1; h->host_acc[2] += t3 - t2;
        if (++h->host_n % 64 == 0) {
            std::fprintf(stderr, "[wfb_mg rank %d] host us/step over 64 steps: issue exchange %.0f | issue source + sizes %.0f | issue update %.0f\n", h->rank,
                         h->host_acc[0] / 64, h->host_acc[1] / 64, h->host_acc[2] / 64);
            h->host_acc[0] = h->host_acc[1] = h->host_acc[2] = 0;
        }
    }
    return rc;
}

int wfb_mg_flush(wfb_mg_t *h, void *out_results, uint64_t *out_ts, uint32_t out_capacity, uint32_t *n_out_dev, void *stream)
{
    if (!h || !n_out_dev) return WFB_E_BADARG;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (h->npend == 0) { CK(cudaMemsetAsync(n_out_dev, 0, sizeof(uint32_t), s)); return 0; }
    const int n = h->npend; h->npend = 0;
    int rc;
    for (int i = 0; i < n; i++) { // oldest first; the results of the later steps follow the first one's in the buffer
        MgSlot &sl = *h->pend[i];
        if (!sl.exchanged) { rc = mg_exchange(h, sl); if (rc) return rc; }
        rc = mg_update(h, sl, out_results, out_ts, out_capacity, n_out_dev, s, i != 0); if (rc) return rc;
        sl.exchanged = false;
        h->pend[i] = nullptr;
    }
    return 0;
}

uint64_t wfb_mg_launches(const wfb_mg_t *h) { return h ? wfb_engine_launches(h->eng) + wfb_ffat_launches(h->ffat) : 0; }

int wfb_mg_stats(wfb_mg_t *h, uint32_t *err_flags_h, uint64_t *results_total_h, void *stream)
{
    if (!h) return WFB_E_BADARG;
    uint32_t nk = 0, ef = 0; uint64_t tot = 0;
    int rc = wfb_ffat_stats(h->ffat, &nk, &ef, stream); if (rc) return rc;
    rc = wfb_ffat_results_total(h->ffat, &tot, stream); if (rc) return rc;
    if (err_flags_h) *err_flags_h = ef;
    if (results_total_h) *results_total_h = tot;
    return 0;
}

int wfb_gen_tuple64(uint64_t seed, uint64_t start, uint32_t n, int key_mode, uint64_t nkeys, const double *zipf_cdf,
                    void *tuples, uint64_t *ts, void *stream)
{
    int rc = device_ready(); if (rc) return rc;
    if ((n && !tuples) || nkeys == 0 || (key_mode == 2 && !zipf_cdf)) return WFB_E_BADARG;
    if (n == 0) return 0;
    const uint32_t grid = std::min((n + 255) / 256, static_cast<uint32_t>(g_num_sms) * 16u);
    k_gen_tuple64<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(seed, start, n, key_mode, nkeys, zipf_cdf,
                                                                       static_cast<wfb_tuple64_t *>(tuples), ts);
    CK(cudaGetLastError());
    return 0;
}

} // extern "C"

#ifdef WFB_BK_TRACE
// debug build only: phase timestamps (globaltimer ns) of the last k_ffat_update_buckets launch, 8 per CTA
extern "C" int wfb_debug_bk_trace(unsigned long long *out) { return cudaMemcpyFromSymbol(out, wfb::g_bk_trace, sizeof(unsigned long long) * 1024 * 8) == cudaSuccess ? 0 : -1; }
#endif
