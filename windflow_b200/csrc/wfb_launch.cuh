// wfb_launch.cuh -- host-side launchers of the kernels of wfb_kernels.cuh for ONE program, and the table of function
// pointers (ProgramOps) through which libwfb200's C ABI reaches them. libwfb200.so instantiates it for the built-in
// programs; an application instantiates it for its own functors with wfb::register_program<MyProgram>() (see
// INTEGRATION.md section 3) and then uses the same C ABI with the returned program id.
#pragma once
#include <type_traits>
#include <algorithm>
#include <cstring>
#include <cuda.h>
#include <cuda_runtime.h>
#include "../../include/wfb200.h"
#include "wfb_kernels.cuh"

#define WFB_CK(call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) return static_cast<int>(e__); } while (0)

namespace wfb {

inline int num_sms()
{
    static int n = 0;
    if (n == 0) { int dev = 0; if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); }
    return n;
}


// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline PFN_encodeTiled get_encode_tiled()
{
    static PFN_encodeTiled fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
        cudaGetLastError();
    }
    return fn;
}

// 2-D view [rows][64 bytes] of a span of device memory holding 64-byte tuples, box = one tile, SWIZZLE_64B
inline bool make_tuple_tmap(CUtensorMap *m, uint64_t base, uint64_t end)
{
    std::memset(m, 0, sizeof(*m));
    PFN_encodeTiled enc = get_encode_tiled();
    if (!enc || (base & 63u) || end <= base) return false;
    const uint64_t rows = (end - base) / 64;
    if (rows == 0 || rows > 0xffffffffull) return false;
    cuuint64_t gdim[2] = {64, rows};
    cuuint64_t gstr[1] = {64};
    cuuint32_t box[2] = {64, TILE};
    cuuint32_t estr[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, reinterpret_cast<void *>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// ---- per-program launch table ------------------------------------------------------------------------------
struct ProgramOps {
    uint32_t tuple_bytes, result_bytes, params_bytes, reserved;
    int (*tile_pass)(int mode, TileArgs &a, const void *params, uint32_t want_grid, cudaStream_t s, uint32_t *grid_used,
                     uint64_t span_begin, uint64_t span_end);
    int (*ffat_update)(const FfatDev &ff, const unsigned char *lifted, const uint32_t *sorted_pos, const uint32_t *batch_off,
                       const DevBatch *batches, uint32_t nbatches, unsigned char *out_res, uint64_t *out_ts,
                       uint32_t out_cap, uint32_t *n_out, uint32_t grid, cudaStream_t s, const void *params, uint32_t lanes_grid);
    int (*ffat_buckets)(const FfatDev &ff, const unsigned char *lifted, const uint32_t *bk_list, uint32_t pos_base,
                        const uint32_t *digit_counts, uint32_t shift, uint32_t moved, const uint32_t *batch_off, const DevBatch *batches,
                        uint32_t nbatches, unsigned char *out_res, uint64_t *out_ts, uint32_t out_cap, uint32_t *n_out, cudaStream_t s,
                        const void *params);
    int (*ffat_windows)(const FfatDev &ff, const uint32_t *batch_off, const DevBatch *batches, uint32_t nbatches,
                        unsigned char *out_res, uint64_t *out_ts, uint32_t out_cap, uint32_t grid, cudaStream_t s, const void *params, uint32_t *n_out);
    int (*extract_keys)(const unsigned char *tuples, uint32_t n, uint64_t *keys, uint32_t *dest, uint32_t num_shards, cudaStream_t s,
                        const void *params);
    int (*reduce_segments)(const unsigned char *tuples, const uint64_t *ts, const uint32_t *sidx, const uint32_t *seg_begin,
                           const uint32_t *n_keys, unsigned char *out_tuples, uint64_t *out_ts, uint32_t n, cudaStream_t s, const void *params);
    int (*reduce_all)(const unsigned char *tuples, const uint64_t *ts, uint32_t n, unsigned char *out_tuple, uint64_t *out_ts, cudaStream_t s,
                      const void *params);
    int (*gather)(const unsigned char *tuples, const uint64_t *ts, const uint32_t *perm, uint32_t n, unsigned char *out_tuples,
                  uint64_t *out_ts, cudaStream_t s);
    // time-based windows, front end
    int (*tb_lift)(const unsigned char *tuples, const uint64_t *ts, uint32_t n, const FfatDev &ff, const TbDev &tb, uint64_t first_incomplete,
                   unsigned char *lifted, uint64_t *ckeys, cudaStream_t s, const void *params);
    int (*tb_reduce)(const unsigned char *lifted, const uint64_t *skeys, const uint32_t *sidx, const uint32_t *seg_begin, const uint32_t *n_segs,
                     unsigned char *part, uint32_t n, uint32_t kbits, uint32_t max_keys, cudaStream_t s, const void *params);
    int (*tb_merge)(const uint64_t *skeys, const uint32_t *seg_begin, const uint32_t *n_segs, const unsigned char *part, const FfatDev &ff,
                    const TbDev &tb, uint32_t n, cudaStream_t s, const void *params);
    int (*tb_pop_write)(const FfatDev &ff, const TbDev &tb, uint64_t first_incomplete, const uint32_t *offs, unsigned char *popped,
                        uint32_t *popped_slots, uint32_t popped_cap, uint32_t max_present, cudaStream_t s, const void *params);
    // launch table of the program's lifted variant (LiftedOf<P>: the count-based back end of time-based windows); null for lifted programs
    const void *(*lifted_ops)();
    // streaming pass of a pass-through program whose records are read in place (TileArgs::inplace)
    int (*slots_inplace)(const TileArgs &a, const void *params, cudaStream_t s);
    // keyed-stateful Map_GPU / Filter_GPU (null when the program has no state_t)
    uint32_t state_bytes, reserved2;
    int (*ks_slots)(const DevBatch *batches, const uint32_t *boff, uint32_t nb, uint32_t total, const FfatDev &ff, uint32_t *slots, cudaStream_t s,
                    const void *params);
    int (*ks_apply)(int filter, const FfatDev &ff, const DevBatch *batches, const uint32_t *boff, uint32_t nb, const uint32_t *bk_slots,
                    const uint32_t *bk_pos, const uint32_t *digit_counts, uint32_t shift, unsigned char *states, unsigned char *keep, cudaStream_t s,
                    const void *params);
    // (more than 65536 keys) the same over the n (slot, position) pairs sorted by slot
    int (*ks_apply_runs)(int filter, const FfatDev &ff, const DevBatch *batches, const uint32_t *boff, uint32_t nb, uint32_t n,
                         const uint32_t *sorted_slots, const uint32_t *sorted_pos, unsigned char *states, unsigned char *keep, cudaStream_t s,
                         const void *params);
    int (*flag_scatter)(const unsigned char *keep, const uint32_t *tile_base, const uint32_t *boff, uint32_t nb, uint32_t n,
                        const uint32_t *rank_start, const DevBatch *batches, cudaStream_t s);
    // Reduce_GPU over K queued batches
    int (*extract_keys_batches)(const DevBatch *batches, const uint32_t *boff, uint32_t nb, uint32_t total, uint32_t key_bits, uint64_t *keys,
                                cudaStream_t s, const void *params);
    int (*reduce_segments_batches)(const DevBatch *batches, const uint32_t *boff, const uint64_t *skeys, const uint32_t *sidx,
                                   const uint32_t *seg_begin, const uint32_t *first_seg, const uint32_t *n_segs, uint32_t key_bits,
                                   uint32_t total, uint32_t *long_list, uint32_t *n_long, cudaStream_t s, const void *params);
    // key_t (wfb_keys.cuh): bytes of its canonical words (8 or 16), KEY_KIND_* and sizeof(key_t) (the order words of a key that is not
    // an integer have no bits above 8 * key_size: a float's fit in 32)
    uint32_t key_bytes, key_kind, key_size;
    // Reduce_GPU over keys that are not integers: the order words of every element (k_key_order_words; batches null: `tuples` is the batch)
    int (*key_order_words)(const DevBatch *batches, const uint32_t *boff, uint32_t nb, const unsigned char *tuples, uint32_t total, uint64_t *lo,
                           uint64_t *hi, cudaStream_t s, const void *params);
    // FlatMap_GPU: the tile pass in MODE_FLATMAP (null when the program has no flatmap)
    int (*flatmap)(TileArgs &a, const void *params, uint32_t want_grid, cudaStream_t s, uint32_t *grid_used, uint64_t span_begin, uint64_t span_end);
};

// P::passthrough (optional): map is a no-op and lift the identity (tuple_t == result_t)
template <class P, class = void> struct program_passthrough : std::false_type {};
template <class P> struct program_passthrough<P, std::void_t<decltype(P::passthrough)>> : std::integral_constant<bool, P::passthrough && std::is_same<typename P::tuple_t, typename P::result_t>::value> {};

template <class P>
inline typename P::params_t load_params(const void *params)
{
    typename P::params_t prm;
    if (params) std::memcpy(&prm, params, sizeof(prm)); else std::memset(&prm, 0, sizeof(prm));
    return prm;
}

template <class P, int MODE>
int launch_tile_pass(TileArgs &a, const void *params, uint32_t want_grid, cudaStream_t s, uint32_t *grid_used,
                     uint64_t span_begin, uint64_t span_end)
{
    static_assert(TilePassSmem<P, MODE>::total <= TP_SMEM_MAX, "tuple_t / result_t too large for the tile pass: two stages of 256 records "
                  "must fit TP_SMEM_MAX (232448 bytes) of shared memory (records of up to about 430 bytes)");
    static int max_grid = -1;
    constexpr uint32_t smem = TilePassSmem<P, MODE>::total;
    if (max_grid < 0) {
        WFB_CK(cudaFuncSetAttribute(k_tile_pass<P, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        int per_sm = 0;
        WFB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_tile_pass<P, MODE>, TP_THREADS, smem));
        if (per_sm < 1) per_sm = 1;
        max_grid = per_sm * wfb::num_sms();
    }
    uint32_t grid = std::max(1u, std::min(want_grid, static_cast<uint32_t>(max_grid)));
    if (a.max_ctas_per_sm) grid = std::max(1u, std::min(grid, a.max_ctas_per_sm * static_cast<uint32_t>(wfb::num_sms())));
    const typename P::params_t prm = load_params<P>(params);
    alignas(64) CUtensorMap tmap;
    a.use_tmap = 0; a.tmap_base = span_begin;
    if (sizeof(typename P::tuple_t) == 64 && make_tuple_tmap(&tmap, span_begin, span_end)) a.use_tmap = 1;
    else std::memset(&tmap, 0, sizeof(tmap));
    k_tile_pass<P, MODE><<<grid, TP_THREADS, smem, s>>>(tmap, a, prm);
    WFB_CK(cudaGetLastError());
    *grid_used = grid;
    return 0;
}

template <class P>
int tile_pass_dispatch(int mode, TileArgs &a, const void *params, uint32_t want_grid, cudaStream_t s, uint32_t *grid_used,
                       uint64_t span_begin, uint64_t span_end)
{
    switch (mode) {
    case MODE_MAP: return launch_tile_pass<P, MODE_MAP>(a, params, want_grid, s, grid_used, span_begin, span_end);
    case MODE_FILTER: return launch_tile_pass<P, MODE_FILTER>(a, params, want_grid, s, grid_used, span_begin, span_end);
    case MODE_INGEST: return launch_tile_pass<P, MODE_INGEST>(a, params, want_grid, s, grid_used, span_begin, span_end);
    }
    return WFB_E_BADARG;
}

template <class P>
int ffat_update_dispatch(const FfatDev &ff, const unsigned char *lifted, const uint32_t *sorted_pos, const uint32_t *batch_off,
                         const DevBatch *batches, uint32_t nbatches, unsigned char *out_res, uint64_t *out_ts,
                         uint32_t out_cap, uint32_t *n_out, uint32_t grid, cudaStream_t s, const void *params, uint32_t lanes_grid)
{
    // thread-per-key pass for the light keys, then warp-per-key only for the heavy list it produced
    const typename P::params_t prm = load_params<P>(params);
    k_ffat_update_lanes<P><<<lanes_grid, 128, 0, s>>>(ff, lifted, sorted_pos, batch_off, batches, nbatches, out_res, out_ts, out_cap, n_out, prm);
    k_ffat_update<P><<<std::max(1u, std::min(grid, static_cast<uint32_t>(wfb::num_sms()) * 2u)), 256, 0, s>>>(
        ff, lifted, sorted_pos, batch_off, batches, nbatches, out_res, out_ts, out_cap, n_out, prm);
    WFB_CK(cudaGetLastError());
    return 0;
}

template <class P>
int ffat_buckets_dispatch(const FfatDev &ff, const unsigned char *lifted, const uint32_t *bk_list, uint32_t pos_base,
                          const uint32_t *digit_counts, uint32_t shift, uint32_t moved, const uint32_t *batch_off, const DevBatch *batches,
                          uint32_t nbatches, unsigned char *out_res, uint64_t *out_ts, uint32_t out_cap, uint32_t *n_out, cudaStream_t s,
                          const void *params)
{
    if (ff.lazy) k_ffat_update_buckets<P, true><<<OSW_DIGITS, BK_THREADS, 0, s>>>(ff, lifted, bk_list, pos_base, digit_counts, shift, moved, batch_off, batches,
                                                                                 nbatches, out_res, out_ts, out_cap, n_out, load_params<P>(params));
    else k_ffat_update_buckets<P, false><<<OSW_DIGITS, BK_THREADS, 0, s>>>(ff, lifted, bk_list, pos_base, digit_counts, shift, moved, batch_off, batches,
                                                                          nbatches, out_res, out_ts, out_cap, n_out, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
// the bucket update of P, or null when its results are too large for it (the handles then take the full-sort path): the kernel is
// instantiated only for results that fit (bk_fits)
template <class P>
constexpr decltype(ProgramOps::ffat_buckets) ffat_buckets_of()
{
    if constexpr (bk_fits<sizeof(typename P::result_t)>()) return &ffat_buckets_dispatch<P>; else return nullptr;
}

template <class P>
int ffat_windows_dispatch(const FfatDev &ff, const uint32_t *batch_off, const DevBatch *batches, uint32_t nbatches,
                          unsigned char *out_res, uint64_t *out_ts, uint32_t out_cap, uint32_t grid, cudaStream_t s, const void *params, uint32_t *n_out)
{
    if (ff.lazy) { // one warp per fired group, the internal levels built on chip: warps per block x 2 n x sizeof(result_t) of dynamic shared memory
        const size_t per_warp = static_cast<size_t>(2) * ff.n_leaves * sizeof(typename P::result_t);
        const uint32_t wpb = static_cast<uint32_t>(std::max<size_t>(1, std::min<size_t>(4, (32u << 10) / per_warp)));
        k_ffat_windows_lazy<P><<<grid, 32 * wpb, wpb * per_warp, s>>>(ff, batch_off, batches, nbatches, out_res, out_ts, out_cap, load_params<P>(params), n_out);
    } else
    k_ffat_windows<P><<<grid, 256, 0, s>>>(ff, batch_off, batches, nbatches, out_res, out_ts, out_cap, load_params<P>(params), n_out);
    WFB_CK(cudaGetLastError());
    return 0;
}

inline uint32_t grid_for(uint32_t n, uint32_t per_block) { return std::max(1u, std::min((n + per_block - 1) / per_block, static_cast<uint32_t>(wfb::num_sms()) * 16u)); }

template <class P>
int extract_keys_dispatch(const unsigned char *tuples, uint32_t n, uint64_t *keys, uint32_t *dest, uint32_t num_shards, cudaStream_t s,
                          const void *params)
{
    k_extract_keys<P><<<grid_for(n, 256), 256, 0, s>>>(tuples, n, keys, dest, num_shards, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int reduce_segments_dispatch(const unsigned char *tuples, const uint64_t *ts, const uint32_t *sidx, const uint32_t *seg_begin,
                             const uint32_t *n_keys, unsigned char *out_tuples, uint64_t *out_ts, uint32_t n, cudaStream_t s,
                             const void *params)
{
    k_reduce_segments<P><<<grid_for(n, 8), 256, 0, s>>>(tuples, ts, sidx, seg_begin, n_keys, out_tuples, out_ts, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int slots_inplace_dispatch(const TileArgs &a, const void *params, cudaStream_t s)
{
    const uint32_t npos = a.num_tiles * TILE;
    k_slots_inplace<P><<<std::max(1u, std::min((npos + 2047u) / 2048u, static_cast<uint32_t>(wfb::num_sms()) * 8u)), 256, 0, s>>>(a, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}

template <class P, class = void> struct program_has_state : std::false_type {};
template <class P> struct program_has_state<P, std::void_t<typename P::state_t>> : std::true_type {};

template <class P>
int ks_slots_dispatch(const DevBatch *batches, const uint32_t *boff, uint32_t nb, uint32_t total, const FfatDev &ff, uint32_t *slots, cudaStream_t s,
                      const void *params)
{
    k_ks_slots<P><<<grid_for(total, 256), 256, 0, s>>>(batches, boff, nb, total, ff, slots, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int ks_apply_dispatch(int filter, const FfatDev &ff, const DevBatch *batches, const uint32_t *boff, uint32_t nb, const uint32_t *bk_slots,
                      const uint32_t *bk_pos, const uint32_t *digit_counts, uint32_t shift, unsigned char *states, unsigned char *keep, cudaStream_t s,
                      const void *params)
{
    if constexpr (program_has_state<P>::value) {
        if (filter) k_ks_apply<P, true><<<OSW_DIGITS, KS_THREADS, 0, s>>>(ff, batches, boff, nb, bk_slots, bk_pos, digit_counts, shift, states, keep, load_params<P>(params));
        else k_ks_apply<P, false><<<OSW_DIGITS, KS_THREADS, 0, s>>>(ff, batches, boff, nb, bk_slots, bk_pos, digit_counts, shift, states, keep, load_params<P>(params));
        WFB_CK(cudaGetLastError());
        return 0;
    } else return WFB_E_UNSUPPORTED;
}
template <class P>
int ks_apply_runs_dispatch(int filter, const FfatDev &ff, const DevBatch *batches, const uint32_t *boff, uint32_t nb, uint32_t n,
                           const uint32_t *sorted_slots, const uint32_t *sorted_pos, unsigned char *states, unsigned char *keep, cudaStream_t s,
                           const void *params)
{
    if constexpr (program_has_state<P>::value) {
        if (filter) k_ks_apply_runs<P, true><<<grid_for(n, 256), 256, 0, s>>>(ff, batches, boff, nb, n, sorted_slots, sorted_pos, states, keep, load_params<P>(params));
        else k_ks_apply_runs<P, false><<<grid_for(n, 256), 256, 0, s>>>(ff, batches, boff, nb, n, sorted_slots, sorted_pos, states, keep, load_params<P>(params));
        WFB_CK(cudaGetLastError());
        return 0;
    } else return WFB_E_UNSUPPORTED;
}
template <class P>
int flag_scatter_dispatch(const unsigned char *keep, const uint32_t *tile_base, const uint32_t *boff, uint32_t nb, uint32_t n,
                          const uint32_t *rank_start, const DevBatch *batches, cudaStream_t s)
{
    k_flag_scatter<P><<<(n + SEGT - 1) / SEGT, 256, 0, s>>>(keep, tile_base, boff, nb, n, rank_start, batches);
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P> constexpr uint32_t program_state_bytes() { if constexpr (program_has_state<P>::value) return sizeof(typename P::state_t); else return 0; }

// P::flatmap(const tuple_t &, Shipper<result_t> &, const params_t &) (optional: FlatMap_GPU)
template <class P, class = void> struct program_has_flatmap : std::false_type {};
template <class P> struct program_has_flatmap<P, std::void_t<decltype(P::flatmap(std::declval<const typename P::tuple_t &>(),
    std::declval<Shipper<typename P::result_t> &>(), std::declval<const typename P::params_t &>()))>> : std::true_type {};
template <class P>
int flatmap_dispatch(TileArgs &a, const void *params, uint32_t want_grid, cudaStream_t s, uint32_t *grid_used, uint64_t span_begin, uint64_t span_end)
{
    return launch_tile_pass<P, MODE_FLATMAP>(a, params, want_grid, s, grid_used, span_begin, span_end);
}

template <class P>
int tb_lift_dispatch(const unsigned char *tuples, const uint64_t *ts, uint32_t n, const FfatDev &ff, const TbDev &tb, uint64_t first_incomplete,
                     unsigned char *lifted, uint64_t *ckeys, cudaStream_t s, const void *params)
{
    k_tb_lift<P><<<grid_for(n, 256), 256, 0, s>>>(tuples, ts, n, ff, tb, first_incomplete, lifted, ckeys, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int tb_reduce_dispatch(const unsigned char *lifted, const uint64_t *skeys, const uint32_t *sidx, const uint32_t *seg_begin, const uint32_t *n_segs,
                       unsigned char *part, uint32_t n, uint32_t kbits, uint32_t max_keys, cudaStream_t s, const void *params)
{
    k_tb_reduce<P><<<grid_for(n, 128), 128, 0, s>>>(lifted, skeys, sidx, seg_begin, n_segs, part, kbits, max_keys, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int tb_merge_dispatch(const uint64_t *skeys, const uint32_t *seg_begin, const uint32_t *n_segs, const unsigned char *part, const FfatDev &ff,
                      const TbDev &tb, uint32_t n, cudaStream_t s, const void *params)
{
    k_tb_merge<P><<<grid_for(n, 128), 128, 0, s>>>(skeys, seg_begin, n_segs, part, ff, tb, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int tb_pop_write_dispatch(const FfatDev &ff, const TbDev &tb, uint64_t first_incomplete, const uint32_t *offs, unsigned char *popped,
                          uint32_t *popped_slots, uint32_t popped_cap, uint32_t max_present, cudaStream_t s, const void *params)
{
    k_tb_pop_write<P><<<grid_for(max_present, 128), 128, 0, s>>>(ff, tb, first_incomplete, offs, popped, popped_slots, popped_cap, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int extract_keys_batches_dispatch(const DevBatch *batches, const uint32_t *boff, uint32_t nb, uint32_t total, uint32_t key_bits, uint64_t *keys,
                                  cudaStream_t s, const void *params)
{
    k_extract_keys_batches<P><<<grid_for(total, 256), 256, 0, s>>>(batches, boff, nb, total, key_bits, keys, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int key_order_words_dispatch(const DevBatch *batches, const uint32_t *boff, uint32_t nb, const unsigned char *tuples, uint32_t total, uint64_t *lo,
                             uint64_t *hi, cudaStream_t s, const void *params)
{
    k_key_order_words<P><<<grid_for(total, 256), 256, 0, s>>>(batches, boff, nb, tuples, total, lo, hi, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int reduce_segments_batches_dispatch(const DevBatch *batches, const uint32_t *boff, const uint64_t *skeys, const uint32_t *sidx,
                                     const uint32_t *seg_begin, const uint32_t *first_seg, const uint32_t *n_segs, uint32_t key_bits,
                                     uint32_t total, uint32_t *long_list, uint32_t *n_long, cudaStream_t s, const void *params)
{
    // short segments: one thread each; long ones (listed by the first kernel): one warp each
    k_reduce_segments_batches_short<P><<<grid_for(total, 128), 128, 0, s>>>(batches, boff, skeys, sidx, seg_begin, first_seg, n_segs, key_bits,
                                                                            long_list, n_long, load_params<P>(params));
    k_reduce_segments_batches<P><<<std::max(1u, std::min(grid_for(total / RB_LONG + 1, 8), static_cast<uint32_t>(wfb::num_sms()) * 8u)), 256, 0, s>>>(
        batches, boff, skeys, sidx, seg_begin, first_seg, n_segs, key_bits, long_list, n_long, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int reduce_all_dispatch(const unsigned char *tuples, const uint64_t *ts, uint32_t n, unsigned char *out_tuple, uint64_t *out_ts, cudaStream_t s,
                        const void *params)
{
    k_reduce_all<P><<<1, 1024, 0, s>>>(tuples, ts, n, out_tuple, out_ts, load_params<P>(params));
    WFB_CK(cudaGetLastError());
    return 0;
}
template <class P>
int gather_dispatch(const unsigned char *tuples, const uint64_t *ts, const uint32_t *perm, uint32_t n, unsigned char *out_tuples,
                    uint64_t *out_ts, cudaStream_t s)
{
    k_gather_tuples<P><<<grid_for(n, 256), 256, 0, s>>>(tuples, ts, perm, n, out_tuples, out_ts);
    WFB_CK(cudaGetLastError());
    return 0;
}

// The lifted variant of a program: its records are the program's results (pane aggregates), combined with the program's comb;
// the key slot of every record comes from the caller (TileArgs::ext_slots), so the program needs no key inside result_t.
template <class P, class = void> struct program_has_result_key : std::false_type {};
template <class P> struct program_has_result_key<P, std::void_t<decltype(P::result_key(std::declval<const typename P::result_t &>(), std::declval<const typename P::params_t &>()))>> : std::true_type {};

template <class P>
struct LiftedOf {
    using tuple_t = typename P::result_t; using result_t = typename P::result_t; using key_t = typename P::key_t; using params_t = typename P::params_t;
    static constexpr bool passthrough = true;
    static constexpr bool is_lifted = true;
    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &, const params_t &) { return true; }
    // the key of a lifted record: P::result_key where the program names it (the destination side of the multi-GPU keyby reads it);
    // the time-based front end hands the slots over itself (TileArgs::ext_slots) and never asks
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &p)
    {
        if constexpr (program_has_result_key<P>::value) return P::result_key(t, p); else return key_t{};
    }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &) { r = t; }
    __host__ __device__ static void comb(const result_t &a, const result_t &b, result_t &o, const params_t &p) { P::comb(a, b, o, p); }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &p) { return P::make_result(k, gwid, p); }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
};
template <class P, class = void> struct program_is_lifted : std::false_type {};
template <class P> struct program_is_lifted<P, std::void_t<decltype(P::is_lifted)>> : std::integral_constant<bool, P::is_lifted> {};

template <class P>
int tile_pass_ingest_dispatch(int mode, TileArgs &a, const void *params, uint32_t want_grid, cudaStream_t s, uint32_t *grid_used,
                              uint64_t span_begin, uint64_t span_end)
{
    if (mode != MODE_INGEST) return WFB_E_UNSUPPORTED;
    return launch_tile_pass<P, MODE_INGEST>(a, params, want_grid, s, grid_used, span_begin, span_end);
}
template <class P>
const void *lifted_ops_of()
{
    static const ProgramOps o = [] {
        using L = LiftedOf<P>;
        ProgramOps t; std::memset(&t, 0, sizeof(t));
        t.tuple_bytes = sizeof(typename L::tuple_t); t.result_bytes = sizeof(typename L::result_t);
        t.params_bytes = sizeof(typename L::params_t); t.reserved = 1u; // pass-through
        t.tile_pass = &tile_pass_ingest_dispatch<L>; t.slots_inplace = &slots_inplace_dispatch<L>;
        t.ffat_update = &ffat_update_dispatch<L>; t.ffat_buckets = ffat_buckets_of<L>(); t.ffat_windows = &ffat_windows_dispatch<L>;
        t.key_bytes = 8u * key_codec<L>::words; t.key_kind = key_codec<L>::kind; t.key_size = sizeof(typename L::key_t);
        t.reserved2 = program_has_result_key<P>::value ? 1u : 0u; // bit 0: the lifted records carry their key (usable behind an exchange)
        return t;
    }();
    return &o;
}

template <class P>
ProgramOps make_ops()
{
    ProgramOps o;
    o.tuple_bytes = sizeof(typename P::tuple_t);
    o.result_bytes = sizeof(typename P::result_t);
    o.params_bytes = sizeof(typename P::params_t); o.reserved = program_passthrough<P>::value ? 1u : 0u; // bit 0: records pass through unchanged
    o.tile_pass = &tile_pass_dispatch<P>;
    o.ffat_update = &ffat_update_dispatch<P>;
    o.ffat_buckets = ffat_buckets_of<P>();
    o.ffat_windows = &ffat_windows_dispatch<P>;
    o.extract_keys = &extract_keys_dispatch<P>;
    o.reduce_segments = &reduce_segments_dispatch<P>;
    o.reduce_all = &reduce_all_dispatch<P>;
    o.gather = &gather_dispatch<P>;
    o.slots_inplace = &slots_inplace_dispatch<P>;
    o.state_bytes = program_state_bytes<P>(); o.reserved2 = 0;
    o.ks_slots = &ks_slots_dispatch<P>; o.ks_apply = &ks_apply_dispatch<P>; o.ks_apply_runs = &ks_apply_runs_dispatch<P>; o.flag_scatter = &flag_scatter_dispatch<P>;
    o.tb_lift = &tb_lift_dispatch<P>; o.tb_reduce = &tb_reduce_dispatch<P>; o.tb_merge = &tb_merge_dispatch<P>; o.tb_pop_write = &tb_pop_write_dispatch<P>;
    o.extract_keys_batches = &extract_keys_batches_dispatch<P>;
    o.reduce_segments_batches = &reduce_segments_batches_dispatch<P>;
    o.key_bytes = 8u * key_codec<P>::words; o.key_kind = key_codec<P>::kind; o.key_size = sizeof(typename P::key_t);
    o.key_order_words = &key_order_words_dispatch<P>;
    if constexpr (program_is_lifted<P>::value) o.lifted_ops = nullptr; else o.lifted_ops = &lifted_ops_of<P>;
    if constexpr (program_has_flatmap<P>::value) o.flatmap = &flatmap_dispatch<P>; else o.flatmap = nullptr;
    return o;
}


// registers the launch table of program P with libwfb200 and returns its program id (>= 6), or a negative error
template <class P>
int register_program()
{
    static int id = -1;
    if (id < 0) { const ProgramOps o = make_ops<P>(); id = wfb_program_register(&o, sizeof(o)); }
    return id;
}

} // namespace wfb
