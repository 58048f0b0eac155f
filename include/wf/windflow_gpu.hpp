// wf/windflow_gpu.hpp -- header-only C++17 host side of the H100-native GPU operators, keeping WindFlow's builder API
// (MapGPU_Builder / FilterGPU_Builder / ReduceGPU_Builder / Ffat_WindowsGPU_Builder, wf/builders_gpu.hpp) and the
// PipeGraph / MultiPipe wiring calls (wf/pipegraph.hpp:594-764, wf/multipipe.hpp:953-1330) for the GPU path:
//
//     PipeGraph graph("app", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
//     MultiPipe &mp = graph.add_source(Source_Builder(src).withOutputBatchSize(65536).build());
//     mp.chain(MapGPU_Builder(map_f).build());
//     mp.chain(FilterGPU_Builder(filter_f).build());
//     mp.add(Ffat_WindowsGPU_Builder(lift_f, comb_f).withKeyBy(key_f).withCBWindows(4096, 64).withNumWinPerBatch(65).build());
//     mp.chain_sink(Sink_Builder(sink_f).build());
//     graph.run();
//
// How it runs (DESIGN.md section 7):
//   * every operator replica is an ff_node of the FastFlow-compatible runtime in include/ff/ (one thread per replica, bounded
//     lock-free queues between them), as in the reference (wf/basic_operator.hpp:54, wf/multipipe.hpp:428-590);
//   * a GPU replica that finds K batches queued on its input takes all of them (up to withMaxBatchesPerCall) and issues ONE
//     launch sequence through the extern "C" layer of include/wfb200.h (wfb_*_batches / wfb_ffat_process_cb with nbatches = K);
//   * chained stateless Map_GPU / Filter_GPU operators are FUSED: a run of them becomes one streaming pass, and when a
//     Ffat_Windows_GPU follows, the run is folded into the window operator's own ingest pass (its `pre` stage) -- the analogue of
//     MultiPipe::chain fusing chained replicas into one thread (wf/multipipe.hpp:538-590). The user's functors keep their
//     types: each one is reached through a __device__ function thunk compiled in the application's translation unit;
//   * no operator waits for the GPU: result sizes stay on the device, every batch carries the CUDA event after which it is
//     valid, and only the Sink (or an operator that needs a size on the host) waits for it;
//   * the CPU Source stages tuples in pinned buffers, several batches in flight (wf/forward_emitter_gpu.hpp:254-305); a
//     device-side source (SourceGPU_Builder) hands over batches that already live in HBM.
// Compile the application with nvcc (-std=c++17 --expt-relaxed-constexpr --expt-extended-lambda), link with -lwfb200 -lpthread.
// Errors follow the reference convention: a red "WindFlow Error:" line and exit.
#pragma once
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <iostream>
#include <limits>
#include <memory>
#include <mutex>
#include <optional>
#include <string>
#include <tuple>
#include <type_traits>
#include <typeindex>
#include <utility>
#include <vector>
#include <cuda_runtime.h>
#include "../ff/ff.hpp"
#include "deferred_counts.hpp"
#include "../wfb200.h"
#include "../../windflow_b200/csrc/wfb_launch.cuh"

namespace wf {

// ---- basic types (wf/basic.hpp) ----------------------------------------------------------------------------------
enum class Execution_Mode_t { DEFAULT, DETERMINISTIC, PROBABILISTIC };
enum class Time_Policy_t { INGRESS_TIME, EVENT_TIME };
enum class Routing_Mode_t { NONE, FORWARD, KEYBY, BROADCAST, REBALANCING };
enum class Win_Type_t { CB, TB };
enum class op_type_t { SOURCE, SINK, BASIC, BASIC_GPU, WIN, WIN_PANED, WIN_MR, WIN_GPU };
struct empty_key_t {};
#define WF_RED "\033[31m"
#define WF_GREEN "\033[32m"
#define WF_DEFAULT_COLOR "\033[0m"

[[noreturn]] inline void wf_fatal(const std::string &msg)
{
    std::cerr << WF_RED << "WindFlow Error: " << msg << WF_DEFAULT_COLOR << std::endl;
    std::exit(EXIT_FAILURE);
}
inline void wfbAssert(int rc, const char *file, int line) // gpuErrChk of wf/basic_gpu.hpp:99-113 for the C ABI
{
    if (rc != 0) {
        std::cerr << WF_RED << "WindFlow Error: libwfb200 => " << wfb_error_string(rc) << ", file => " << file << ", at line => " << line
                  << WF_DEFAULT_COLOR << std::endl;
        std::exit(rc > 0 ? rc : EXIT_FAILURE);
    }
}
#define wfbErrChk(ans) { ::wf::wfbAssert((ans), __FILE__, __LINE__); }
#define gpuErrChk(ans) { ::wf::wfbAssert(static_cast<int>(ans), __FILE__, __LINE__); }

// ---- functor signature sniffing (the role of wf/meta_gpu.hpp) ---------------------------------------------------------
template <class F> struct fn_sig : fn_sig<decltype(&F::operator())> {};
template <class C, class R, class... A> struct fn_sig<R (C::*)(A...) const> { using ret = R; using args = std::tuple<A...>; };
template <class C, class R, class... A> struct fn_sig<R (C::*)(A...)> { using ret = R; using args = std::tuple<A...>; };
template <class R, class... A> struct fn_sig<R (*)(A...)> { using ret = R; using args = std::tuple<A...>; };
template <class F, size_t I> using fn_arg_t = std::decay_t<std::tuple_element_t<I, typename fn_sig<F>::args>>;
template <class F> using fn_ret_t = typename fn_sig<F>::ret;

// ---- fused chains of stateless functors ----------------------------------------------------------------------------------------
// A run of chained Map_GPU / Filter_GPU operators over the same tuple type executes inside ONE streaming pass: stage i is a
// __device__ thunk (instantiated for the user's functor type in this translation unit, so the functor body is compiled as
// written) plus the functor object's bytes; the kernel walks the stages per tuple and stops at the first predicate that fails.
using stage_fn_t = bool (*)(void *, const void *);
constexpr uint32_t WF_MAX_FUSED = 6;      // stateless operators per fused run (a longer chain starts a new run)
constexpr uint32_t WF_FUNCTOR_BYTES = 48; // largest functor object that travels in a fused stage
struct StageChain {
    stage_fn_t fn[WF_MAX_FUSED];
    alignas(8) unsigned char blob[WF_MAX_FUSED][WF_FUNCTOR_BYTES];
    uint32_t n, has_filter;
};
template <class F, class T> __device__ bool wf_map_thunk(void *t, const void *f) { F fn(*static_cast<const F *>(f)); fn(*static_cast<T *>(t)); return true; }
template <class F, class T> __device__ bool wf_filter_thunk(void *t, const void *f) { F fn(*static_cast<const F *>(f)); return fn(*static_cast<T *>(t)); }
template <class F, class T> __device__ stage_fn_t wf_map_thunk_ptr = wf_map_thunk<F, T>;
template <class F, class T> __device__ stage_fn_t wf_filter_thunk_ptr = wf_filter_thunk<F, T>;
template <class T> struct ChainStages { // both the "map" and the "filter" slot of a program are chains; an empty one does nothing
    StageChain c;
    __host__ __device__ bool operator()(T &t) const
    {
#if defined(__CUDA_ARCH__)
        for (uint32_t i = 0; i < c.n; i++) if (!c.fn[i](&t, c.blob[i])) return false;
#else
        (void) t;
#endif
        return true;
    }
};
template <class X> struct is_chain : std::false_type {};
template <class T> struct is_chain<ChainStages<T>> : std::true_type {};
// The same run with the functor TYPES known where the program is instantiated (a fluent pipe.chain(map).chain(filter).add(ffat):
// FusedPipe below): the functors are called directly and inlined into the tile pass -- no thunks, no tuple in local memory.
template <class F, bool IS_FILTER> struct TypedStage { F f; };
template <class T, class... S> struct TypedChain { __host__ __device__ bool operator()(T &) const { return true; } };
template <class T, class F, bool IS_FILTER, class... Rest>
struct TypedChain<T, TypedStage<F, IS_FILTER>, Rest...> {
    F f; TypedChain<T, Rest...> rest;
    __host__ __device__ bool operator()(T &t) const
    {
        F fn(f);
        if constexpr (IS_FILTER) { if (!fn(t)) return false; } else fn(t);
        return rest(t);
    }
};
template <class T> inline TypedChain<T> make_typed_chain() { return {}; }
template <class T, class F, bool IS_FILTER, class... Rest>
inline TypedChain<T, TypedStage<F, IS_FILTER>, Rest...> make_typed_chain(TypedStage<F, IS_FILTER> s, Rest... rest) { return {s.f, make_typed_chain<T>(rest...)}; }

// ---- default functors of the slots an operator does not use -------------------------------------------------------------
template <class T> struct NoKey { __host__ __device__ uint64_t operator()(const T &) const { return 0; } };
template <class T, class R> struct NoLift { __host__ __device__ void operator()(const T &, R &) const {} };
template <class R> struct NoComb { __host__ __device__ void operator()(const R &, const R &, R &) const {} };
template <class T> struct NoReduce { __host__ __device__ T operator()(const T &a, const T &) const { return a; } };

// The key type of an operator is what its key extractor returns (as in the reference, wf/keyby_emitter_gpu.hpp:108): an integral or
// enum type, float, double, or a trivially copyable type of at most 16 bytes without padding or floating-point members (such as a
// struct { uint32_t src, dst; }). windflow_b200/csrc/wfb_keys.cuh maps it to the words the device key table stores; any other type
// fails to compile there.
template <class KeyF> using key_of_t = std::decay_t<fn_ret_t<KeyF>>;
template <class KeyF> constexpr bool integral_key_v = wfb::KeyCodec<key_of_t<KeyF>>::kind == wfb::KEY_KIND_INTEGRAL;

// The program the kernels are instantiated for: the user's functor objects travel by value in params_t; the map / filter slots
// hold the fused chain that runs in front of the operator.
template <class T, class R, class KeyF, class LiftF, class CombF, class RedF, bool KEYED, class PreF = ChainStages<T>>
struct FacadeProgram {
    using tuple_t = T; using result_t = R; using key_t = key_of_t<KeyF>;
    // (a typed run leaves no stage that is called through a pointer: the tuple then stays in registers)
    using map_slot_t = std::conditional_t<is_chain<PreF>::value, ChainStages<T>, TypedChain<T>>;
    struct params_t { map_slot_t map; PreF filt; KeyF key; LiftF lift; CombF comb; RedF red; };
    static_assert(std::is_trivially_copyable<T>::value && std::is_trivially_copyable<R>::value, "tuple_t / result_t must be trivially copyable");
    static_assert(sizeof(T) % 8 == 0 && sizeof(R) % 8 == 0, "tuple_t / result_t sizes must be multiples of 8 bytes");
    __host__ __device__ static void map(tuple_t &t, const params_t &p) { p.map(t); }
    __host__ __device__ static bool filter(tuple_t &t, const params_t &p) { return p.filt(t); }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &p) { KeyF f = p.key; return f(t); }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &p) { LiftF f = p.lift; f(t, r); }
    __host__ __device__ static void comb(const result_t &a, const result_t &b, result_t &o, const params_t &p) { CombF f = p.comb; f(a, b, o); }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &)
    {   // create_win_result_t_gpu, wf/basic_gpu.hpp:236-247: result_t(key, gwid) when keyed, result_t(gwid) otherwise
        if constexpr (KEYED && std::is_constructible<result_t, key_t, uint64_t>::value) { result_t r(k, gwid); return r; }
        else if constexpr (!KEYED && std::is_constructible<result_t, uint64_t>::value) { result_t r(gwid); return r; }
        else { (void) k; (void) gwid; return result_t(); } // programs of operators without windows never call this
    }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &b, const params_t &p) { RedF f = p.red; return f(a, b); }
};
template <class T> using ChainProgram = FacadeProgram<T, T, NoKey<T>, NoLift<T, T>, NoComb<T>, NoReduce<T>, false>;

// The program of a keyed-stateful Map_GPU / Filter_GPU: func(tuple_t &, state_t &) in per-key arrival order
// (API: __host__ __device__ void(tuple_t &, state_t &) / bool(tuple_t &, state_t &), wf/map_gpu.hpp:104-310, wf/filter_gpu.hpp:120-399).
template <class T, class S, class MapF2, class FiltF2, class KeyF>
struct FacadeStatefulProgram {
    using tuple_t = T; using result_t = T; using key_t = key_of_t<KeyF>; using state_t = S;
    struct params_t { MapF2 map; FiltF2 filt; KeyF key; };
    static_assert(std::is_trivially_copyable<T>::value && std::is_trivially_copyable<S>::value, "tuple_t / state_t must be trivially copyable");
    static_assert(sizeof(T) % 8 == 0, "tuple_t size must be a multiple of 8 bytes");
    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &, const params_t &) { return true; }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &p) { KeyF f = p.key; return f(t); }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &) { r = t; }
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t(); }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
    __host__ __device__ static void map_stateful(tuple_t &t, state_t &st, const params_t &p) { MapF2 f = p.map; f(t, st); }
    __host__ __device__ static bool filter_stateful(tuple_t &t, state_t &st, const params_t &p) { FiltF2 f = p.filt; return f(t, st); }
};
// The program of a FlatMap_GPU: func(const tuple_t &, Shipper_GPU<result_t> &) after the fused run of stateless operators in front
// (the filter slot runs maps and predicates in order). The window slots are never launched for it.
template <class R> using Shipper_GPU = wfb::Shipper<R>; // push(const result_t &): the shipper of a FlatMap_GPU functor (wf/shipper.hpp)
template <class T, class R, class FlatF>
struct FacadeFlatMapProgram {
    using tuple_t = T; using result_t = R; using key_t = uint64_t;
    struct params_t { ChainStages<T> map; ChainStages<T> filt; FlatF fm; };
    static_assert(std::is_trivially_copyable<T>::value && std::is_trivially_copyable<R>::value, "tuple_t / result_t must be trivially copyable");
    static_assert(sizeof(T) % 8 == 0 && sizeof(R) % 8 == 0, "tuple_t / result_t sizes must be multiples of 8 bytes");
    __host__ __device__ static void map(tuple_t &t, const params_t &p) { p.map(t); }
    __host__ __device__ static bool filter(tuple_t &t, const params_t &p) { return p.filt(t); }
    __host__ __device__ static void flatmap(const tuple_t &t, Shipper_GPU<result_t> &sh, const params_t &p) { FlatF f = p.fm; f(t, sh); }
    __host__ __device__ static key_t key(const tuple_t &, const params_t &) { return 0; }
    __host__ __device__ static void lift(const tuple_t &, result_t &, const params_t &) {}
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t(); }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
};
// The program of a keyed-stateful FlatMap_GPU: func(const tuple_t &, Shipper_GPU<result_t> &, state_t &) in per-key arrival order
// (nothing runs in front of it: a stateless run before it is materialised, as before the keyed Map / Filter)
template <class T, class R, class S, class FlatF, class KeyF>
struct FacadeStatefulFlatMapProgram {
    using tuple_t = T; using result_t = R; using key_t = key_of_t<KeyF>; using state_t = S;
    struct params_t { FlatF fm; KeyF key; };
    static_assert(std::is_trivially_copyable<T>::value && std::is_trivially_copyable<R>::value && std::is_trivially_copyable<S>::value,
                  "tuple_t / result_t / state_t must be trivially copyable");
    static_assert(sizeof(T) % 8 == 0 && sizeof(R) % 8 == 0, "tuple_t / result_t sizes must be multiples of 8 bytes");
    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &, const params_t &) { return true; }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &p) { KeyF f = p.key; return f(t); }
    __host__ __device__ static void lift(const tuple_t &, result_t &, const params_t &) {}
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t(); }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
    __host__ __device__ static void map_stateful(tuple_t &, state_t &, const params_t &) {}
    __host__ __device__ static bool filter_stateful(tuple_t &, state_t &, const params_t &) { return true; }
    __host__ __device__ static void flatmap_stateful(const tuple_t &t, Shipper_GPU<result_t> &sh, state_t &st, const params_t &p)
    {
        FlatF f = p.fm; f(t, sh, st);
    }
};
// The program of a Keyed_Windows_GPU: func(const Iterable_GPU<tuple_t> &, result_t &) over each count-based window of a key, or,
// INC, func(const tuple_t &, result_t &) folding each tuple into every open window it is IN (wf/keyed_windows.hpp, non-riched); the
// result starts as result_t(key, gwid) when that constructor exists. Only the member matching the functor is defined (win_func or
// win_func_inc), so that the launch table takes the matching path.
template <class T> using Iterable_GPU = wfb::Iterable_GPU<T>; // size(), operator[], at(), front(), back(), begin() / end() (wf/iterable.hpp)
template <class T, class R, class WinF, class KeyF, bool KEYED, bool INC>
struct FacadeKeyedWindowsProgram {
    using tuple_t = T; using result_t = R; using key_t = key_of_t<KeyF>;
    struct params_t { WinF win; KeyF key; };
    static_assert(std::is_trivially_copyable<T>::value && std::is_trivially_copyable<R>::value, "tuple_t / result_t must be trivially copyable");
    static_assert(sizeof(T) % 8 == 0 && sizeof(R) % 8 == 0, "tuple_t / result_t sizes must be multiples of 8 bytes");
    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &, const params_t &) { return true; }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &p) { KeyF f = p.key; return f(t); }
    __host__ __device__ static void lift(const tuple_t &, result_t &, const params_t &) {}
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &p)
    {
        return FacadeProgram<T, R, KeyF, NoLift<T, R>, NoComb<R>, NoReduce<T>, KEYED>::make_result(k, gwid, {{}, {}, p.key, {}, {}, {}});
    }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
    template <bool I = INC, std::enable_if_t<!I, int> = 0>
    __host__ __device__ static void win_func(const Iterable_GPU<tuple_t> &w, result_t &r, const params_t &p) { WinF f = p.win; f(w, r); }
    template <bool I = INC, std::enable_if_t<I, int> = 0>
    __host__ __device__ static void win_func_inc(const tuple_t &t, result_t &r, const params_t &p) { WinF f = p.win; f(t, r); }
};
// the tuple type of a window function's first argument: T from const Iterable_GPU<T> & (non-incremental) or from const T & (incremental)
template <class X> struct window_tuple { using type = X; static constexpr bool incremental = true; };
template <class T> struct window_tuple<wfb::Iterable_GPU<T>> { using type = T; static constexpr bool incremental = false; };

template <class T, class S> struct StatefulIdMap { __host__ __device__ void operator()(T &, S &) const {} };
template <class T, class S> struct StatefulKeepAll { __host__ __device__ bool operator()(T &, S &) const { return true; } };

// ---- Batch_GPU_t (wf/batch_gpu_t.hpp:50-243) as structure of arrays ---------------------------------------------------
// `size` may be DEFERRED: the producing kernel leaves the count on the device, an asynchronous copy brings it to the pinned
// word `count_h`, and it is valid once `valid_after` has fired -- getSize() waits for it, nothing else does. The word belongs to a
// block of the producing replica (wf/deferred_counts.hpp) that is not rewritten while this batch still points into it.
struct Batch_Base {
    ff::MPMC_Ptr_Queue *home = nullptr; // the producer's recycling queue (the reference's batch->queue, wf/recycling_gpu.hpp:88-141)
    virtual ~Batch_Base() {}
};
template <class tuple_t>
struct Batch_GPU_t: Batch_Base {
    tuple_t *tuples_gpu = nullptr;      // capacity * sizeof(tuple_t)
    uint64_t *ts_gpu = nullptr;         // capacity timestamps
    tuple_t *pinned_tuples_cpu = nullptr;
    uint64_t *pinned_ts_cpu = nullptr;
    bool owns_device = true;            // false: the arrays belong to the application (device-side source)
    size_t size = 0, original_size = 0; // items (upper bound while deferred) | capacity
    bool deferred = false;              // size = *count_h once valid_after has fired
    uint32_t *count_h = nullptr; CountBlock *count_blk = nullptr; // deferred count: the pinned word and the producing replica's block it lies in
    std::vector<uint64_t> watermarks{std::numeric_limits<uint64_t>::max()};
    cudaStream_t cudaStream = nullptr;  // per-batch stream of the host->device copy (wf/batch_gpu_t.hpp:83-101)
    cudaEvent_t own_ev = nullptr;       // recorded by the producer behind the work that fills this batch ...
    cudaEvent_t valid_after = nullptr;  // ... or the event of the group this batch was produced with (consumers wait for this one)
    cudaEvent_t reuse_after = nullptr;  // recorded by the last consumer behind its reads: the producer's next write waits for it

    explicit Batch_GPU_t(size_t n, bool device_arrays = true): size(n), original_size(n), owns_device(device_arrays)
    {
        if (device_arrays) {
            gpuErrChk(cudaMalloc(&tuples_gpu, sizeof(tuple_t) * (n ? n : 1)));
            gpuErrChk(cudaMalloc(&ts_gpu, sizeof(uint64_t) * (n ? n : 1)));
            gpuErrChk(cudaStreamCreateWithFlags(&cudaStream, cudaStreamNonBlocking));
        }
        gpuErrChk(cudaEventCreateWithFlags(&own_ev, cudaEventDisableTiming));
    }
    ~Batch_GPU_t() override
    {
        release_count();
        if (own_ev) { cudaEventSynchronize(own_ev); cudaEventDestroy(own_ev); }
        if (owns_device) { cudaFree(tuples_gpu); cudaFree(ts_gpu); }
        if (pinned_tuples_cpu) cudaFreeHost(pinned_tuples_cpu);
        if (pinned_ts_cpu) cudaFreeHost(pinned_ts_cpu);
        if (cudaStream) cudaStreamDestroy(cudaStream);
    }
    Batch_GPU_t(const Batch_GPU_t &) = delete;
    Batch_GPU_t &operator=(const Batch_GPU_t &) = delete;
    size_t getSize() // resolves a deferred size (waits for the producing work)
    {
        if (deferred) { gpuErrChk(cudaEventSynchronize(valid_after)); size = *count_h; deferred = false; release_count(); }
        return size;
    }
    // the size is word i of `blk`, at most `bound`, valid after `e`
    void defer(size_t bound, CountBlock *blk, size_t i, cudaEvent_t e) { size = bound; deferred = true; count_blk = blk; count_h = blk->h + i; valid_after = e; }
    void release_count() { if (count_blk) { count_blk->release(); count_blk = nullptr; } }
    uint64_t getWatermark(size_t id = 0) const { return id < watermarks.size() ? watermarks[id] : watermarks[0]; }
    void setWatermark(uint64_t wm, size_t id = 0) { if (id < watermarks.size()) watermarks[id] = wm; else watermarks[0] = wm; }
    void updateWatermark(uint64_t wm) { if (watermarks[0] > wm) watermarks[0] = wm; }
    size_t pinned_cap = 0;
    void ensureHost(size_t n = 0) // pinned staging for n items (the whole capacity when n = 0); grows, never shrinks
    {
        if (n == 0) n = original_size ? original_size : 1;
        if (n <= pinned_cap) return;
        if (pinned_tuples_cpu) { cudaFreeHost(pinned_tuples_cpu); cudaFreeHost(pinned_ts_cpu); }
        pinned_cap = std::max(n, 2 * pinned_cap);
        gpuErrChk(cudaMallocHost(&pinned_tuples_cpu, sizeof(tuple_t) * pinned_cap));
        gpuErrChk(cudaMallocHost(&pinned_ts_cpu, sizeof(uint64_t) * pinned_cap));
    }
    void transfer2CPU(cudaStream_t s) // :154-165 (after getSize())
    {
        ensureHost(size ? size : 1);
        if (valid_after) gpuErrChk(cudaStreamWaitEvent(s, valid_after, 0));
        gpuErrChk(cudaMemcpyAsync(pinned_tuples_cpu, tuples_gpu, sizeof(tuple_t) * size, cudaMemcpyDeviceToHost, s));
        if (ts_gpu) gpuErrChk(cudaMemcpyAsync(pinned_ts_cpu, ts_gpu, sizeof(uint64_t) * size, cudaMemcpyDeviceToHost, s));
        gpuErrChk(cudaStreamSynchronize(s));
    }
    tuple_t &getTupleAtPos(size_t pos) { return pinned_tuples_cpu[pos]; }
    uint64_t getTimestampAtPos(size_t pos) { return pinned_ts_cpu[pos]; }
    void reset(size_t n) { release_count(); size = n; deferred = false; valid_after = nullptr; watermarks.assign(1, std::numeric_limits<uint64_t>::max()); }
};

// returns a batch to its producer (deleteBatch_t, wf/recycling.hpp:66-85); batches that do not fit the queue are freed
inline void recycleBatch(Batch_Base *b)
{
    if (b == nullptr) return;
    if (b->home == nullptr || !b->home->push(b)) delete b;
}

// per-replica pool of batches of one type: the recycling queue + allocation on a miss (allocateBatch_GPU_t, wf/recycling_gpu.hpp:88-141)
template <class tuple_t>
class BatchPool {
    ff::MPMC_Ptr_Queue queue;
    size_t allocated = 0, max_live;
public:
    explicit BatchPool(size_t max_live_ = 64): max_live(max_live_) { queue.init(DEFAULT_BUFFER_CAPACITY); }
    ~BatchPool() { void *p; while (queue.pop(&p)) delete static_cast<Batch_Base *>(p); }
    // a recycled batch of capacity >= n, or a new one; with `bounded`, at most max_live batches exist (the caller waits for a
    // consumer to return one: back-pressure on the source)
    Batch_GPU_t<tuple_t> *get(size_t n, bool device_arrays = true, bool bounded = false)
    {
        unsigned spins = 0;
        for (;;) {
            void *p = nullptr;
            if (queue.pop(&p)) {
                auto *b = static_cast<Batch_GPU_t<tuple_t> *>(p);
                if (b->original_size >= n && b->owns_device == device_arrays) { b->reset(n); return b; }
                delete b; allocated--;
                continue;
            }
            if (!bounded || allocated < max_live) break;
            ff::rt::backoff(spins);
        }
        auto *b = new Batch_GPU_t<tuple_t>(n, device_arrays);
        b->home = &queue; allocated++;
        return b;
    }
};

// ---- replicas: nodes of the thread runtime ---------------------------------------------------------------------------------------
class Basic_Replica: public ff::ff_monode { // wf/basic_operator.hpp:54-235
protected:
    std::string opName; bool terminated = false;
    cudaStream_t stream = nullptr; // the replica's own stream: every launch sequence of its svc() goes here
    std::vector<cudaEvent_t> evs; size_t ev_next = 0; // events recorded behind the launch sequences (a small ring)
    cudaEvent_t next_event()
    {
        if (evs.empty()) { evs.resize(16); for (auto &e : evs) gpuErrChk(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); }
        cudaEvent_t e = evs[ev_next]; ev_next = (ev_next + 1) % evs.size();
        return e;
    }
    // the launch sequence about to be issued reads these batches: order the replica's stream behind their producers
    template <class B> void wait_inputs(const std::vector<B *> &in)
    {
        cudaEvent_t last = nullptr;
        for (auto *b : in) if (b->valid_after && b->valid_after != last) { gpuErrChk(cudaStreamWaitEvent(stream, b->valid_after, 0)); last = b->valid_after; }
    }
public:
    explicit Basic_Replica(std::string n): opName(std::move(n)) {}
    ~Basic_Replica() override { for (auto e : evs) cudaEventDestroy(e); if (stream) cudaStreamDestroy(stream); }
    int svc_init() override { gpuErrChk(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)); return 0; }
    void eosnotify(ssize_t) override { terminated = true; }
    bool isTerminated() const { return terminated; }
    // up to `maxk` batches: the one svc() was called with and whatever else is already queued on the input
    template <class B> void drain(void *first, size_t maxk, std::vector<B *> &out)
    {
        out.clear();
        out.push_back(reinterpret_cast<B *>(first));
        void *more;
        while (out.size() < maxk && this->ff_poll(&more)) out.push_back(reinterpret_cast<B *>(more));
    }
};

class Basic_Operator {
protected:
    std::string name; size_t parallelism; Routing_Mode_t input_routing_mode; size_t outputBatchSize;
public:
    Basic_Operator(std::string n, size_t p, Routing_Mode_t r, size_t obs): name(std::move(n)), parallelism(p ? p : 1), input_routing_mode(r), outputBatchSize(obs) {}
    virtual ~Basic_Operator() {}
    std::string getName() const { return name; }
    size_t getParallelism() const { return parallelism; }
    Routing_Mode_t getInputRoutingMode() const { return input_routing_mode; }
    size_t getOutputBatchSize() const { return outputBatchSize; }
    virtual bool isGPUOperator() const { return true; }
    virtual std::string getType() const = 0;
    void setExecutionMode(Execution_Mode_t m) { if (m != Execution_Mode_t::DEFAULT) wf_fatal(getType() + " can only be used in DEFAULT mode"); }
};

// ---- Source (CPU side) -----------------------------------------------------------------------------------------------------------------
template <class tuple_t> class Source_Shipper;

// Source_Replica + Forward_Emitter_GPU<..., false, true> (wf/forward_emitter_gpu.hpp:254-305): tuples are written into the pinned
// buffer of the open batch; a full batch goes to the device with an asynchronous copy on its own stream and is sent on at once --
// WF_SOURCE_BATCHES_IN_FLIGHT batches (the reference keeps 2) are in flight before push() waits for a consumer to return one.
#ifndef WF_SOURCE_BATCHES_IN_FLIGHT
#define WF_SOURCE_BATCHES_IN_FLIGHT 8
#endif
template <class tuple_t>
class SourceReplica: public Basic_Replica {
    friend class Source_Shipper<tuple_t>;
    std::function<void(Source_Shipper<tuple_t> &)> func;
    size_t batch_size;
    BatchPool<tuple_t> pool{WF_SOURCE_BATCHES_IN_FLIGHT};
    Batch_GPU_t<tuple_t> *cur = nullptr;
    size_t fill = 0;
    uint64_t next_wm = 0;
    void open()
    {
        cur = pool.get(batch_size, true, true);
        cur->ensureHost();
        gpuErrChk(cudaEventSynchronize(cur->own_ev)); // the previous copy out of this pinned buffer is over
        fill = 0;
    }
public:
    SourceReplica(std::string n, std::function<void(Source_Shipper<tuple_t> &)> f, size_t bs): Basic_Replica(std::move(n)), func(std::move(f)), batch_size(bs) {}
    void push(const tuple_t &t, uint64_t ts)
    {
        if (!cur) open();
        cur->pinned_tuples_cpu[fill] = t; cur->pinned_ts_cpu[fill] = ts; cur->updateWatermark(next_wm);
        if (++fill == batch_size) flush();
    }
    void flush()
    {
        if (!cur || fill == 0) return;
        cur->size = fill;
        if (cur->reuse_after) gpuErrChk(cudaStreamWaitEvent(cur->cudaStream, cur->reuse_after, 0)); // the last reader of the device arrays
        gpuErrChk(cudaMemcpyAsync(cur->tuples_gpu, cur->pinned_tuples_cpu, sizeof(tuple_t) * fill, cudaMemcpyHostToDevice, cur->cudaStream));
        gpuErrChk(cudaMemcpyAsync(cur->ts_gpu, cur->pinned_ts_cpu, sizeof(uint64_t) * fill, cudaMemcpyHostToDevice, cur->cudaStream));
        gpuErrChk(cudaEventRecord(cur->own_ev, cur->cudaStream));
        cur->valid_after = cur->own_ev;
        Batch_GPU_t<tuple_t> *b = cur; cur = nullptr; fill = 0;
        this->ff_send_out(b); // ownership moves downstream; the last consumer returns it with recycleBatch()
    }
    void *svc(void *) override;
};

template <class tuple_t>
class Source_Shipper { // wf/source_shipper.hpp:289-322
    SourceReplica<tuple_t> *st;
public:
    explicit Source_Shipper(SourceReplica<tuple_t> *s): st(s) {}
    void push(const tuple_t &t) { st->push(t, std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now().time_since_epoch()).count()); }
    void pushWithTimestamp(const tuple_t &t, uint64_t ts) { st->push(t, ts); }
    void setNextWatermark(uint64_t wm) { st->next_wm = wm; }
};
template <class tuple_t> void *SourceReplica<tuple_t>::svc(void *) { Source_Shipper<tuple_t> sh(this); func(sh); flush(); terminated = true; return this->EOS; }

template <class source_func_t>
class Source: public Basic_Operator {
public:
    source_func_t func;
    static constexpr op_type_t op_type = op_type_t::SOURCE;
    Source(source_func_t f, std::string n, size_t p, size_t obs): Basic_Operator(std::move(n), p, Routing_Mode_t::NONE, obs), func(f) {}
    bool isGPUOperator() const override { return false; }
    std::string getType() const override { return "Source"; }
};
template <class F> struct shipper_tuple;
template <class T> struct shipper_tuple<Source_Shipper<T>> { using type = T; };

template <class source_func_t>
class Source_Builder {
    source_func_t func; std::string name = "source"; size_t parallelism = 1, obs = 0;
public:
    explicit Source_Builder(source_func_t f): func(f) {}
    auto &withName(std::string n) { name = std::move(n); return *this; }
    auto &withParallelism(size_t p) { parallelism = p; return *this; }
    auto &withOutputBatchSize(size_t n) { obs = n; return *this; }
    auto build() { return Source<source_func_t>(func, name, parallelism, obs); }
};

// ---- device-side source (SURVEY.md 8 f3): batches that already live in HBM ------------------------------------------------------------------
// The functor receives a SourceGPU_Shipper and hands over device arrays it owns: pushBatch() wraps them in a Batch_GPU_t without
// copying. `valid_after` (optional) is the event behind the work that fills the arrays; consecutive batches may share one.
template <class tuple_t> class SourceGPU_Shipper;
template <class tuple_t>
class SourceGPUReplica: public Basic_Replica {
    friend class SourceGPU_Shipper<tuple_t>;
    std::function<void(SourceGPU_Shipper<tuple_t> &)> func;
    BatchPool<tuple_t> pool{1024};
public:
    SourceGPUReplica(std::string n, std::function<void(SourceGPU_Shipper<tuple_t> &)> f): Basic_Replica(std::move(n)), func(std::move(f)) {}
    void *svc(void *) override;
};
template <class tuple_t>
class SourceGPU_Shipper {
    SourceGPUReplica<tuple_t> *st;
public:
    explicit SourceGPU_Shipper(SourceGPUReplica<tuple_t> *s): st(s) {}
    void pushBatch(tuple_t *tuples_dev, uint64_t *ts_dev, size_t n, uint64_t watermark, cudaEvent_t valid_after = nullptr)
    {
        Batch_GPU_t<tuple_t> *b = st->pool.get(n, false, true);
        b->tuples_gpu = tuples_dev; b->ts_gpu = ts_dev; b->size = n; b->original_size = n; b->setWatermark(watermark); b->valid_after = valid_after;
        st->ff_send_out(b);
    }
    cudaStream_t stream() const { return st->stream; } // a stream of the replica for the application's generator kernels
};
template <class tuple_t> void *SourceGPUReplica<tuple_t>::svc(void *) { SourceGPU_Shipper<tuple_t> sh(this); func(sh); terminated = true; return this->EOS; }
template <class source_func_t>
class SourceGPU: public Basic_Operator {
public:
    source_func_t func;
    static constexpr op_type_t op_type = op_type_t::SOURCE;
    SourceGPU(source_func_t f, std::string n, size_t obs): Basic_Operator(std::move(n), 1, Routing_Mode_t::NONE, obs), func(f) {}
    std::string getType() const override { return "Source_GPU"; }
};
template <class T> struct shipper_tuple<SourceGPU_Shipper<T>> { using type = T; };
template <class source_func_t>
class SourceGPU_Builder {
    source_func_t func; std::string name = "source_gpu";
public:
    explicit SourceGPU_Builder(source_func_t f): func(f) {}
    auto &withName(std::string n) { name = std::move(n); return *this; }
    auto build() { return SourceGPU<source_func_t>(func, name, 1); }
};

// ---- Sink (CPU side) ---------------------------------------------------------------------------------------------------------------------
template <class sink_func_t>
class Sink: public Basic_Operator {
public:
    sink_func_t func;
    std::atomic<uint64_t> *wm_probe = nullptr;
    static constexpr op_type_t op_type = op_type_t::SINK;
    Sink(sink_func_t f, std::string n, size_t p, std::atomic<uint64_t> *probe = nullptr): Basic_Operator(std::move(n), p, Routing_Mode_t::FORWARD, 0), func(f), wm_probe(probe) {}
    Sink(const Sink &o): Basic_Operator(o), func(o.func), wm_probe(o.wm_probe) {}
    bool isGPUOperator() const override { return false; }
    std::string getType() const override { return "Sink"; }
};
template <class sink_func_t>
class Sink_Builder {
    sink_func_t func; std::string name = "sink"; size_t parallelism = 1; std::atomic<uint64_t> *probe = nullptr;
public:
    explicit Sink_Builder(sink_func_t f): func(f) {}
    auto &withName(std::string n) { name = std::move(n); return *this; }
    auto &withParallelism(size_t p) { parallelism = p; return *this; }
    // extension: the sink stores the watermark of every batch it has finished with (how far the stream has been processed end to end)
    auto &withWatermarkProbe(std::atomic<uint64_t> *p) { probe = p; return *this; }
    auto build() { return Sink<sink_func_t>(func, name, parallelism, probe); }
};

// Forward_Emitter_GPU<..., true, false> (transfer2CPU) + Sink_Replica::svc (wf/sink.hpp:102-111). The only place that waits for the GPU.
template <class tuple_t, class sink_func_t>
class SinkReplica: public Basic_Replica {
    sink_func_t func; std::atomic<uint64_t> *wm_probe;
public:
    SinkReplica(std::string n, sink_func_t f, std::atomic<uint64_t> *probe = nullptr): Basic_Replica(std::move(n)), func(f), wm_probe(probe) {}
    void *svc(void *msg) override
    {
        auto *b = reinterpret_cast<Batch_GPU_t<tuple_t> *>(msg);
        if (b->getSize() != 0) {
            b->transfer2CPU(stream);
            for (size_t i = 0; i < b->size; i++) { std::optional<tuple_t> o(b->getTupleAtPos(i)); func(o); }
        }
        if (wm_probe) { // the highest watermark finished so far (several sink replicas finish batches out of order)
            b->getSize();
            uint64_t wm = b->getWatermark(), cur = wm_probe->load(std::memory_order_relaxed);
            while (cur < wm && !wm_probe->compare_exchange_weak(cur, wm, std::memory_order_release)) { }
        }
        recycleBatch(b);
        return this->GO_ON;
    }
    void svc_end() override { std::optional<tuple_t> o; func(o); } // the reference's end-of-stream call with an empty optional
};

// ---- GPU operators ------------------------------------------------------------------------------------------------------
#ifndef WF_MAX_BATCHES_PER_CALL
#define WF_MAX_BATCHES_PER_CALL 128
#endif

// The drop counts of a FlatMap_GPU replica's calls: every call leaves its count in the word after its batches' sizes, in a block the
// replica holds until the host has read that word.
class FlatMapDrops {
    struct Pending { CountBlock *blk; size_t word; cudaEvent_t ev; };
    std::vector<Pending> pending; uint64_t dropped = 0; // drop counts of calls the host has not read yet / the sum of those it read
public:
    void add(CountBlock *blk, size_t word, cudaEvent_t ev) { pending.push_back(Pending{blk, word, ev}); }
    // adds the drop counts of finished calls (all of them with `wait`)
    void read(bool wait)
    {
        size_t i = 0;
        for (; i < pending.size(); i++) {
            if (wait || pending.size() - i > 8) { gpuErrChk(cudaEventSynchronize(pending[i].ev)); } // (events of the ring are re-recorded after 16 calls)
            else if (cudaEventQuery(pending[i].ev) != cudaSuccess) { cudaGetLastError(); break; }
            dropped += pending[i].blk->h[pending[i].word];
            pending[i].blk->release();
        }
        pending.erase(pending.begin(), pending.begin() + static_cast<std::ptrdiff_t>(i));
    }
    // end of stream: stops the program when a push was dropped
    void check(const std::string &op_name, uint32_t max_out)
    {
        read(true);
        if (dropped) wf_fatal("FlatMap_GPU [" + op_name + "]: " + std::to_string(dropped) + " records pushed beyond withMaxOutputsPerTuple(" +
                              std::to_string(max_out) + ") were dropped");
    }
};

// The call of every GPU replica: svc() takes the batches queued on its input (up to maxk) and hands them to ONE launch sequence.
// take() is the input half. The operator then sends its results in one of two shapes: send_in_place() (the inputs, changed in place,
// move on) or send_deferred() (input i becomes output batch i, whose size stays on the device).
template <class in_t, class out_t = in_t>
class Batch_Replica: public Basic_Replica {
protected:
    using in_batch_t = Batch_GPU_t<in_t>;
    using out_batch_t = Batch_GPU_t<out_t>;
    size_t maxk;
    DeferredCounts counts; // (before the pool: its batches point into it)
    BatchPool<out_t> pool;
    std::vector<in_batch_t *> in;     // the batches of the call
    std::vector<wfb_batch_t> bi, bo;  // their descriptors, and those of their output batches
    std::vector<out_batch_t *> outs;
    Batch_Replica(std::string n, size_t maxk_, size_t pool_size = 4 * WF_MAX_BATCHES_PER_CALL): Basic_Replica(std::move(n)), maxk(maxk_ ? maxk_ : 1), pool(pool_size) {}
    // the batches queued on the input (those of size 0 recycled with `skip_empty`), the stream ordered behind their producers, their
    // descriptors in bi; false: nothing to launch
    bool take(void *msg, bool skip_empty)
    {
        drain(msg, maxk, in);
        size_t k = 0;
        for (auto *b : in) { if (b->getSize() == 0 && skip_empty) recycleBatch(b); else in[k++] = b; }
        in.resize(k);
        if (k == 0) return false;
        wait_inputs(in);
        bi.resize(k);
        for (size_t i = 0; i < k; i++) bi[i] = wfb_batch_t{in[i]->tuples_gpu, in[i]->ts_gpu, in[i]->getWatermark(), static_cast<uint32_t>(in[i]->size), 0};
        return true;
    }
    // a batch of capacity >= cap for the results of input b, which the stream may write
    out_batch_t *output_for(const in_batch_t *b, size_t cap)
    {
        out_batch_t *o = pool.get(cap);
        o->watermarks = b->watermarks;
        if (o->reuse_after) gpuErrChk(cudaStreamWaitEvent(stream, o->reuse_after, 0));
        return o;
    }
    // the inputs, changed in place by the launches just issued, move on
    void send_in_place()
    {
        cudaEvent_t e = next_event();
        gpuErrChk(cudaEventRecord(e, stream));
        for (auto *b : in) { b->valid_after = e; this->ff_send_out(b); }
    }
    // input i becomes output batch i, of capacity original_size * mult and at most size * mult results: call(counts_d) issues the
    // launches, which leave the size of output i in counts_d[i] and `extra` words of the operator's after the k sizes. Those words are
    // the replica's to read and release. Returns the call's block and the event behind the call.
    template <class Call> std::pair<CountBlock *, cudaEvent_t> send_deferred(size_t mult, size_t extra, Call &&call)
    {
        const size_t k = in.size();
        bo.resize(k); outs.resize(k);
        for (size_t i = 0; i < k; i++) {
            outs[i] = output_for(in[i], in[i]->original_size * mult);
            bo[i] = wfb_batch_t{outs[i]->tuples_gpu, outs[i]->ts_gpu, in[i]->getWatermark(), static_cast<uint32_t>(outs[i]->original_size), 0};
        }
        CountBlock *blk; uint32_t *counts_d;
        gpuErrChk(counts.acquire(static_cast<uint32_t>(k + extra), blk, counts_d));
        call(counts_d);
        gpuErrChk(cudaMemcpyAsync(blk->h, counts_d, sizeof(uint32_t) * (k + extra), cudaMemcpyDeviceToHost, stream));
        cudaEvent_t e = next_event();
        gpuErrChk(cudaEventRecord(e, stream));
        for (size_t i = 0; i < k; i++) {
            outs[i]->defer(in[i]->size * mult, blk, i, e);
            in[i]->reuse_after = e; recycleBatch(in[i]); // (the reference drops empty batches here, wf/filter_gpu.hpp:572-581: the
            this->ff_send_out(outs[i]);                   // size is not known on the host yet, the consumer skips an empty one)
        }
        return {blk, e};
    }
    // send_deferred() of a FlatMap_GPU: outputs of original_size * m records, and the call's drop count in the word after the sizes
    template <class Call> void send_expanded(FlatMapDrops &drops, uint32_t m, Call &&call)
    {
        drops.read(false);
        const auto sent = send_deferred(m, 1, call);
        drops.add(sent.first, in.size(), sent.second);
    }
};

// A fused run of stateless Map_GPU / Filter_GPU operators over tuple_t (wf/map_gpu.hpp:313-420, wf/filter_gpu.hpp:401-600): ONE
// streaming pass per svc() over the K batches found queued. A run of maps only works in place (wfb_map per batch: same batch
// moves on); with a filter in the run the survivors are compacted, stable, into K spare batches whose sizes stay on the device.
template <class tuple_t>
class ChainReplica: public Batch_Replica<tuple_t> {
    using base_t = Batch_Replica<tuple_t>; using base_t::in; using base_t::bi; using base_t::bo; using base_t::stream;
    using prog_t = ChainProgram<tuple_t>;
    wfb_engine_t *eng = nullptr; typename prog_t::params_t prm{};
public:
    ChainReplica(std::string n, const StageChain &c, size_t maxk): base_t(std::move(n), maxk)
    {
        if (c.has_filter) prm.filt.c = c; else prm.map.c = c; // (the filter slot runs maps and predicates in order)
    }
    ~ChainReplica() override { if (eng) wfb_engine_destroy(eng); }
    int svc_init() override
    {
        Basic_Replica::svc_init();
        wfbErrChk(wfb_engine_create(&eng, wfb::register_program<prog_t>()));
        if (prm.filt.c.n) gpuErrChk(this->counts.init(this->maxk));
        return 0;
    }
    void *svc(void *msg) override
    {
        if (!this->take(msg, false)) return this->GO_ON;
        const wfb_functors_t *f = reinterpret_cast<const wfb_functors_t *>(&prm);
        if (prm.filt.c.n == 0) { // maps only: in place, the same batches move on
            for (auto *b : in) if (b->size) wfbErrChk(wfb_map(eng, f, b->tuples_gpu, static_cast<uint32_t>(b->size), stream));
            this->send_in_place();
        } else {
            this->send_deferred(1, 0, [&](uint32_t *counts_d) {
                wfbErrChk(wfb_map_filter_batches(eng, f, bi.data(), bo.data(), static_cast<uint32_t>(in.size()), counts_d, stream));
            });
        }
        return this->GO_ON;
    }
};

// description of a stateless GPU operator before it is placed: the thunk, the functor bytes, the tuple type
template <class func_t, bool IS_FILTER>
class Stateless_GPU: public Basic_Operator {
public:
    using tuple_t = fn_arg_t<func_t, 0>;
    using result_t = tuple_t;
    static constexpr op_type_t op_type = op_type_t::BASIC_GPU;
    static constexpr bool is_filter = IS_FILTER;
    func_t func;
    Stateless_GPU(func_t f, size_t p, std::string n, Routing_Mode_t r): Basic_Operator(std::move(n), p, r, 1), func(f)
    {
        static_assert(std::is_trivially_copyable<func_t>::value, "GPU functors must be trivially copyable");
    }
    std::string getType() const override { return IS_FILTER ? "Filter_GPU" : "Map_GPU"; }
    bool append_to(StageChain &c) const // false: the run is full or the functor object too large to travel in a fused stage
    {
        if (c.n >= WF_MAX_FUSED || sizeof(func_t) > WF_FUNCTOR_BYTES) return false;
        stage_fn_t fn = nullptr;
        if constexpr (IS_FILTER) { gpuErrChk(cudaMemcpyFromSymbol(&fn, wf_filter_thunk_ptr<func_t, tuple_t>, sizeof(fn))); }
        else { gpuErrChk(cudaMemcpyFromSymbol(&fn, wf_map_thunk_ptr<func_t, tuple_t>, sizeof(fn))); }
        c.fn[c.n] = fn;
        std::memset(c.blob[c.n], 0, WF_FUNCTOR_BYTES);
        std::memcpy(c.blob[c.n], &func, sizeof(func_t));
        c.n++; if (IS_FILTER) c.has_filter = 1;
        return true;
    }
};
template <class F> using Map_GPU = Stateless_GPU<F, false>;
template <class F> using Filter_GPU = Stateless_GPU<F, true>;

// FlatMap_GPU (wf/flatmap.hpp with wf/shipper.hpp on the GPU): func(const tuple_t &, Shipper_GPU<result_t> &) pushes 0..m records per
// tuple, m = withMaxOutputsPerTuple(m). ONE wfb_flatmap_batches call per svc() over the K batches found queued, with the fused run of
// stateless operators in front of it: input batch i becomes output batch i (records in input order, per tuple in push order, each
// with its tuple's timestamp), of capacity original_size * m, whose size stays on the device. The functor may run more than once per
// tuple (it must push the same records every time). Pushes beyond the m-th of a tuple are dropped and counted on the device; a
// non-zero count stops the program at the end of the stream with the operator's name and m.
template <class shipper_t> struct shipper_result;
template <class R> struct shipper_result<wfb::Shipper<R>> { using type = R; };

template <class tuple_t, class result_t, class func_t>
class FlatMapReplica: public Batch_Replica<tuple_t, result_t> {
    using base_t = Batch_Replica<tuple_t, result_t>; using base_t::in; using base_t::bi; using base_t::bo; using base_t::stream;
    using prog_t = FacadeFlatMapProgram<tuple_t, result_t, func_t>;
    wfb_engine_t *eng = nullptr; typename prog_t::params_t prm{};
    uint32_t max_out;
    FlatMapDrops drops; // (the replica holds every call's block until it has read the drop count)
public:
    FlatMapReplica(std::string n, const StageChain &pre, func_t f, uint32_t m, size_t maxk): base_t(std::move(n), maxk), max_out(m)
    {
        prm.filt.c = pre; prm.fm = f;
    }
    ~FlatMapReplica() override { if (eng) wfb_engine_destroy(eng); }
    int svc_init() override
    {
        Basic_Replica::svc_init();
        wfbErrChk(wfb_engine_create(&eng, wfb::register_program<prog_t>()));
        gpuErrChk(this->counts.init(this->maxk + 1));
        return 0;
    }
    void *svc(void *msg) override
    {
        if (!this->take(msg, false)) return this->GO_ON;
        this->send_expanded(drops, max_out, [&](uint32_t *counts_d) {
            wfbErrChk(wfb_flatmap_batches(eng, reinterpret_cast<const wfb_functors_t *>(&prm), bi.data(), bo.data(), static_cast<uint32_t>(in.size()),
                                          max_out, counts_d, stream));
        });
        return this->GO_ON;
    }
    void eosnotify(ssize_t id) override
    {
        drops.check(this->opName, max_out);
        Basic_Replica::eosnotify(id);
    }
};

template <class func_t>
class FlatMap_GPU: public Basic_Operator {
public:
    using tuple_t = fn_arg_t<func_t, 0>;
    using result_t = typename shipper_result<fn_arg_t<func_t, 1>>::type;
    static constexpr op_type_t op_type = op_type_t::BASIC_GPU;
    func_t func; uint32_t max_outputs;
    FlatMap_GPU(func_t f, size_t p, std::string n, Routing_Mode_t r, uint32_t m): Basic_Operator(std::move(n), p, r, 1), func(f), max_outputs(m)
    {
        static_assert(std::is_trivially_copyable<func_t>::value, "GPU functors must be trivially copyable");
    }
    std::string getType() const override { return "FlatMap_GPU"; }
    // a replica with the fused run `pre` of stateless operators over tuple_t in front (empty: none)
    FlatMapReplica<tuple_t, result_t, func_t> *make_replica(const StageChain &pre) const
    {
        return new FlatMapReplica<tuple_t, result_t, func_t>(name, pre, func, max_outputs, parallelism > 1 ? 1 : WF_MAX_BATCHES_PER_CALL);
    }
};

// Map_GPU / Filter_GPU / FlatMap_GPU, keyed-stateful (wf/map_gpu.hpp:104-310, wf/filter_gpu.hpp:120-399, FlatMap_Builder(f).withKeyBy(k)
// of wf/flatmap.hpp): func(tuple_t &, state_t &), or func(const tuple_t &, Shipper_GPU<result_t> &, state_t &) for a FlatMap, in per-key
// arrival order. The key -> state table is one wfb_kstate_t per operator, shared by its replicas behind a mutex (the reference's TBB
// map + spinlock, wf/map_gpu.hpp:551-559); a replica hands the K batches it finds queued to one launch sequence. A Map works in place,
// a Filter compacts the survivors into output batches whose sizes stay on the device, and a FlatMap has the outputs and the drop count
// of FlatMap_GPU: input batch i becomes output batch i of capacity original_size * m whose size stays on the device, and a push beyond
// the m-th of a tuple stops the program at the end of the stream.
struct SharedKState { wfb_kstate_t *h = nullptr; std::mutex mu; ~SharedKState() { if (h) wfb_kstate_destroy(h); } };
enum class Stateful_Kind_t { MAP, FILTER, FLATMAP };
template <class F, Stateful_Kind_t KIND> struct stateful_result { using type = fn_arg_t<F, 0>; };
template <class F> struct stateful_result<F, Stateful_Kind_t::FLATMAP> { using type = typename shipper_result<fn_arg_t<F, 1>>::type; };

template <class func_t, class keyextr_func_gpu_t, Stateful_Kind_t KIND>
class Stateful_GPU: public Basic_Operator {
public:
    static constexpr bool is_flatmap = KIND == Stateful_Kind_t::FLATMAP;
    using tuple_t = fn_arg_t<func_t, 0>;
    using result_t = typename stateful_result<func_t, KIND>::type;
    using state_t = fn_arg_t<func_t, is_flatmap ? 2 : 1>;
    using prog_t = std::conditional_t<is_flatmap, FacadeStatefulFlatMapProgram<tuple_t, result_t, state_t, func_t, keyextr_func_gpu_t>,
                   std::conditional_t<KIND == Stateful_Kind_t::FILTER,
                                      FacadeStatefulProgram<tuple_t, state_t, StatefulIdMap<tuple_t, state_t>, func_t, keyextr_func_gpu_t>,
                                      FacadeStatefulProgram<tuple_t, state_t, func_t, StatefulKeepAll<tuple_t, state_t>, keyextr_func_gpu_t>>>;
    static constexpr op_type_t op_type = op_type_t::BASIC_GPU;
    func_t func; keyextr_func_gpu_t key_extr; uint32_t max_keys, max_outputs; size_t maxk = WF_MAX_BATCHES_PER_CALL;
    bool grow_keys = false; // withKeyGrowth(): max_keys is the initial capacity of the table (WFB_KEYS_GROW), which grows under the replicas' mutex
    Stateful_GPU(func_t f, keyextr_func_gpu_t k, size_t p, std::string n, uint32_t mk, uint32_t m)
        : Basic_Operator(std::move(n), p, Routing_Mode_t::KEYBY, 1), func(f), key_extr(k), max_keys(mk), max_outputs(m)
    {
        static_assert(!is_flatmap || std::is_trivially_copyable<func_t>::value, "GPU functors must be trivially copyable");
    }
    std::string getType() const override { return KIND == Stateful_Kind_t::MAP ? "Map_GPU" : KIND == Stateful_Kind_t::FILTER ? "Filter_GPU" : "FlatMap_GPU"; }
    keyextr_func_gpu_t getKeyExtractor() const { return key_extr; }
    class Replica: public Batch_Replica<tuple_t, result_t> {
        using base_t = Batch_Replica<tuple_t, result_t>; using base_t::in; using base_t::bi; using base_t::bo; using base_t::stream;
        std::shared_ptr<SharedKState> ks; typename prog_t::params_t prm; uint32_t max_out;
        FlatMapDrops drops; // (FlatMap)
        // the replicas of the operator share the state table: one launch sequence at a time
        template <class Launch> void locked(Launch &&launch)
        {
            std::lock_guard<std::mutex> lock(ks->mu);
            wfbErrChk(launch());
            gpuErrChk(cudaStreamSynchronize(stream)); // another replica's launches on its own stream must see this call's state
        }
    public:
        Replica(std::string n, std::shared_ptr<SharedKState> h, typename prog_t::params_t p, uint32_t m, size_t maxk)
            : base_t(std::move(n), maxk), ks(std::move(h)), prm(p), max_out(m) {}
        int svc_init() override
        {
            Basic_Replica::svc_init();
            if constexpr (KIND == Stateful_Kind_t::FILTER) gpuErrChk(this->counts.init(this->maxk));
            if constexpr (is_flatmap) gpuErrChk(this->counts.init(this->maxk + 1));
            return 0;
        }
        void *svc(void *msg) override
        {
            if (!this->take(msg, !is_flatmap)) return this->GO_ON;
            const wfb_functors_t *f = reinterpret_cast<const wfb_functors_t *>(&prm);
            const uint32_t k = static_cast<uint32_t>(in.size());
            if constexpr (KIND == Stateful_Kind_t::MAP) {
                locked([&] { return wfb_map_stateful(ks->h, f, bi.data(), k, stream); });
                this->send_in_place();
            } else if constexpr (KIND == Stateful_Kind_t::FILTER) {
                this->send_deferred(1, 0, [&](uint32_t *counts_d) {
                    locked([&] { return wfb_filter_stateful(ks->h, f, bi.data(), bo.data(), k, counts_d, stream); });
                });
            } else {
                this->send_expanded(drops, max_out, [&](uint32_t *counts_d) {
                    locked([&] { return wfb_flatmap_stateful(ks->h, f, bi.data(), bo.data(), k, max_out, counts_d, stream); });
                });
            }
            return this->GO_ON;
        }
        void eosnotify(ssize_t id) override
        {
            if constexpr (is_flatmap) drops.check(this->opName, max_out);
            Basic_Replica::eosnotify(id);
        }
    };
    typename prog_t::params_t params() const
    {
        if constexpr (KIND == Stateful_Kind_t::MAP) return {func, {}, key_extr};
        else if constexpr (KIND == Stateful_Kind_t::FILTER) return {{}, func, key_extr};
        else return {func, key_extr};
    }
    std::shared_ptr<SharedKState> kstate;
    Replica *make_replica()
    {
        if (!kstate) { kstate = std::make_shared<SharedKState>(); wfbErrChk(wfb_kstate_create(&kstate->h, wfb::register_program<prog_t>(), max_keys, grow_keys ? WFB_KEYS_GROW : 0u)); }
        return new Replica(name, kstate, params(), max_outputs, parallelism > 1 ? 1 : maxk);
    }
};
template <class F, class K> using Map_GPU_KB = Stateful_GPU<F, K, Stateful_Kind_t::MAP>;
template <class F, class K> using Filter_GPU_KB = Stateful_GPU<F, K, Stateful_Kind_t::FILTER>;
template <class F, class K> using FlatMap_GPU_KB = Stateful_GPU<F, K, Stateful_Kind_t::FLATMAP>;

// Reduce_GPU (wf/reduce_gpu.hpp:109-289): per batch, one item per distinct key (ascending) or one item for the batch.
template <class reduce_func_gpu_t, class keyextr_func_gpu_t>
class Reduce_GPU: public Basic_Operator {
public:
    using tuple_t = fn_arg_t<reduce_func_gpu_t, 0>;
    using result_t = tuple_t;
    static constexpr bool isKeyed = !std::is_same<keyextr_func_gpu_t, NoKey<tuple_t>>::value;
    using prog_t = FacadeProgram<tuple_t, tuple_t, keyextr_func_gpu_t, NoLift<tuple_t, tuple_t>, NoComb<tuple_t>, reduce_func_gpu_t, false>;
    static constexpr op_type_t op_type = op_type_t::BASIC_GPU;
    reduce_func_gpu_t func; keyextr_func_gpu_t key_extr; uint32_t key_bits = 64; size_t maxk = WF_MAX_BATCHES_PER_CALL;
    Reduce_GPU(reduce_func_gpu_t f, keyextr_func_gpu_t k, size_t p, std::string n, Routing_Mode_t r): Basic_Operator(std::move(n), p, r, 1), func(f), key_extr(k) {}
    std::string getType() const override { return "Reduce_GPU"; }
    class Replica: public Batch_Replica<tuple_t> {
        using base_t = Batch_Replica<tuple_t>; using base_t::in; using base_t::bi; using base_t::bo; using base_t::outs; using base_t::stream;
        wfb_engine_t *eng = nullptr; typename prog_t::params_t prm; uint32_t key_bits;
    public:
        Replica(std::string n, reduce_func_gpu_t f, keyextr_func_gpu_t k, uint32_t kb, size_t mk): base_t(std::move(n), mk), prm{{}, {}, k, {}, {}, f}, key_bits(kb) {}
        ~Replica() override { if (eng) wfb_engine_destroy(eng); }
        int svc_init() override
        {
            Basic_Replica::svc_init();
            wfbErrChk(wfb_engine_create(&eng, wfb::register_program<prog_t>()));
            wfbErrChk(wfb_engine_set_params(eng, &prm, sizeof(prm)));
            if (key_bits != 64) wfbErrChk(wfb_engine_set_key_bits(eng, key_bits)); // (integral keys: ReduceGPU_Builder::build checks)
            if (isKeyed) gpuErrChk(this->counts.init(this->maxk));
            return 0;
        }
        void *svc(void *msg) override
        {
            if (!this->take(msg, true)) return this->GO_ON;
            const size_t k = in.size();
            if constexpr (isKeyed) {
                uint32_t kbits = 0; while ((1ull << kbits) < k) kbits++;
                const uint32_t sort_bits = integral_key_v<keyextr_func_gpu_t> ? key_bits : 32u; // other keys are sorted by their 32-bit rank
                this->send_deferred(1, 0, [&](uint32_t *counts_d) {
                    if (k > 1 && sort_bits + kbits <= 64) { wfbErrChk(wfb_reduce_by_key_batches(eng, bi.data(), bo.data(), static_cast<uint32_t>(k), counts_d, stream)); }
                    else for (size_t i = 0; i < k; i++)
                        wfbErrChk(wfb_reduce_by_key(eng, bi[i].tuples, bi[i].ts, bi[i].n, const_cast<void *>(bo[i].tuples), const_cast<uint64_t *>(bo[i].ts), counts_d + i, stream));
                });
            } else { // one item per batch: the output's size, 1, is known on the host
                outs.resize(k);
                for (size_t i = 0; i < k; i++) outs[i] = this->output_for(in[i], 1);
                for (size_t i = 0; i < k; i++) wfbErrChk(wfb_reduce_all(eng, bi[i].tuples, bi[i].ts, bi[i].n, outs[i]->tuples_gpu, outs[i]->ts_gpu, stream));
                cudaEvent_t e = this->next_event();
                gpuErrChk(cudaEventRecord(e, stream));
                for (size_t i = 0; i < k; i++) {
                    outs[i]->valid_after = e;
                    in[i]->reuse_after = e; recycleBatch(in[i]);
                    this->ff_send_out(outs[i]);
                }
            }
            return this->GO_ON;
        }
    };
    Replica *make_replica() { return new Replica(name, func, key_extr, key_bits, maxk); }
};

// Ffat_Windows_GPU, count-based and time-based (wf/ffat_windows_gpu.hpp:59-274, wf/ffat_replica_gpu.hpp:707-1047). svc(): the K
// batches found queued go to ONE wfb_ffat_process_cb call, with the fused run of stateless operators in front of it as `pre`;
// the results of the call form one output batch whose size stays on the device.
template <class lift_func_gpu_t, class comb_func_gpu_t, class keyextr_func_gpu_t, class pre_t = ChainStages<fn_arg_t<lift_func_gpu_t, 0>>>
class Ffat_Windows_GPU: public Basic_Operator {
public:
    using tuple_t = fn_arg_t<lift_func_gpu_t, 0>;
    using result_t = fn_arg_t<lift_func_gpu_t, 1>;
    static constexpr bool isKeyed = !std::is_same<keyextr_func_gpu_t, NoKey<tuple_t>>::value;
    static constexpr bool typed_pre = !is_chain<pre_t>::value; // the run in front is part of the program's type (FusedPipe)
    using prog_t = FacadeProgram<tuple_t, result_t, keyextr_func_gpu_t, lift_func_gpu_t, comb_func_gpu_t, NoReduce<tuple_t>, isKeyed, pre_t>;
    static constexpr op_type_t op_type = op_type_t::WIN_GPU;
    lift_func_gpu_t lift; comb_func_gpu_t comb; keyextr_func_gpu_t key_extr;
    uint64_t win_len, slide_len, lateness; Win_Type_t winType; size_t numWinPerBatch; uint32_t max_keys; bool dense_keys;
    size_t maxk = WF_MAX_BATCHES_PER_CALL;
    bool grow_keys = false; // withKeyGrowth(): max_keys is the initial capacity of the key table (WFB_KEYS_GROW)
    pre_t pre{}; // the fused run of stateless operators chained in front of this operator (MultiPipe / FusedPipe fill it)
    bool has_pre() const { if constexpr (typed_pre) return true; else return pre.c.n != 0; }
    // the same operator with the typed run `p` in front (FusedPipe)
    template <class other_pre_t>
    Ffat_Windows_GPU(const Ffat_Windows_GPU<lift_func_gpu_t, comb_func_gpu_t, keyextr_func_gpu_t, other_pre_t> &o, pre_t p):
        Basic_Operator(o), lift(o.lift), comb(o.comb), key_extr(o.key_extr), win_len(o.win_len), slide_len(o.slide_len), lateness(o.lateness), winType(o.winType),
        numWinPerBatch(o.numWinPerBatch), max_keys(o.max_keys), dense_keys(o.dense_keys), maxk(o.maxk), grow_keys(o.grow_keys), pre(p) {}
    Ffat_Windows_GPU(lift_func_gpu_t l, comb_func_gpu_t c, keyextr_func_gpu_t k, std::string n, uint64_t w, uint64_t s, uint64_t late,
                     Win_Type_t wt, size_t nwb, uint32_t mk, bool dense, size_t mbpc):
        Basic_Operator(std::move(n), 1 /* forced to 1, wf/ffat_windows_gpu.hpp:197 */, isKeyed ? Routing_Mode_t::KEYBY : Routing_Mode_t::FORWARD, nwb), lift(l), comb(c), key_extr(k),
        win_len(w), slide_len(s), lateness(late), winType(wt), numWinPerBatch(nwb), max_keys(mk), dense_keys(dense), maxk(mbpc ? mbpc : 1)
    {
        if (win_len == 0 || slide_len == 0) wf_fatal("Ffat_Windows_GPU used with window length or slide equal to zero");
        if (numWinPerBatch == 0) wf_fatal("Ffat_Windows_GPU used with zero windows per batch");
    }
    std::string getType() const override { return "Ffat_Windows_GPU"; }
    keyextr_func_gpu_t getKeyExtractor() const { return key_extr; }
    class Replica: public Batch_Replica<tuple_t, result_t> {
        using base_t = Batch_Replica<tuple_t, result_t>; using base_t::in; using base_t::bi; using base_t::stream;
        Ffat_Windows_GPU op;
        wfb_ffat_t *ffat = nullptr; typename prog_t::params_t prm;
        const bool tb; uint64_t last_wm = 0; size_t cap_hint = 0;
    public:
        // (time-based windows fire per batch watermark: one batch per call)
        explicit Replica(const Ffat_Windows_GPU &o): base_t(o.name, o.winType == Win_Type_t::TB ? 1 : o.maxk, 64), op(o), prm{{}, o.pre, o.key_extr, o.lift, o.comb, {}},
            tb(o.winType == Win_Type_t::TB) {}
        ~Replica() override { if (ffat) wfb_ffat_destroy(ffat); }
        int svc_init() override
        {
            Basic_Replica::svc_init();
            wfbErrChk(wfb_ffat_create(&ffat, wfb::register_program<prog_t>(), op.win_len, op.slide_len, static_cast<uint32_t>(op.numWinPerBatch),
                                      op.max_keys, tb ? 1 : 0, op.lateness, (op.dense_keys ? WFB_FFAT_DENSE_KEYS : 0u) | (op.grow_keys ? WFB_KEYS_GROW : 0u)));
            wfbErrChk(wfb_ffat_set_params(ffat, &prm, sizeof(prm)));
            gpuErrChk(this->counts.init(1)); // (one word per call)
            return 0;
        }
        void *svc(void *msg) override
        {
            if (!this->take(msg, true)) return this->GO_ON;
            const size_t k = in.size();
            uint64_t total = 0;
            for (auto *b : in) total += b->size;
            // every group that can fire in this call: per key, count-based one per slide*Nb items (+1: the first group); time-based one
            // per slide*Nb time units the watermark advanced since the key was last seen -- bounded here by the whole advance. A growing
            // key table may take new keys in the call: count-based, a new key fires its first group after B = (Nb-1)*slide+win of its
            // items; time-based, one item may be enough, so every item counts as a key
            const uint64_t wm = in.back()->getWatermark();
            const uint64_t nb = op.numWinPerBatch, per = op.slide_len * nb, B = (nb - 1) * op.slide_len + op.win_len;
            const uint64_t keys = wfb_ffat_key_capacity(ffat) + (op.grow_keys ? (tb ? total : total / B) : 0);
            const uint64_t groups = tb ? keys * ((wm > last_wm ? wm - last_wm : 0) / per + 2) + (wm / per + 2)
                                       : total / per + keys + 1;
            if (tb && last_wm == 0) last_wm = wm; // (the bound above for the first batch: wm / per groups of one key)
            cap_hint = std::max(cap_hint, static_cast<size_t>(std::min<uint64_t>(groups * nb, 0x7fffffffull))); // (never shrinks: recycled batches keep fitting)
            const size_t cap = cap_hint;
            if (tb) last_wm = wm;
            Batch_GPU_t<result_t> *out = this->output_for(in.back(), cap); // (with the watermark of the call's last batch)
            CountBlock *blk; uint32_t *count_d;
            gpuErrChk(this->counts.acquire(1, blk, count_d));
            const wfb_functors_t *pre = op.has_pre() ? reinterpret_cast<const wfb_functors_t *>(&prm) : nullptr;
            if (tb) { wfbErrChk(wfb_ffat_process_tb(ffat, pre, bi.data(), static_cast<uint32_t>(k), out->tuples_gpu, out->ts_gpu, static_cast<uint32_t>(cap), count_d, stream)); }
            else { wfbErrChk(wfb_ffat_process_cb(ffat, pre, bi.data(), static_cast<uint32_t>(k), out->tuples_gpu, out->ts_gpu, static_cast<uint32_t>(cap), count_d, stream)); }
            if (tb) check_errors(); // (the time-based path synchronises per batch anyway: a result that did not fit is reported, not lost silently)
            gpuErrChk(cudaMemcpyAsync(blk->h, count_d, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
            cudaEvent_t e = this->next_event();
            gpuErrChk(cudaEventRecord(e, stream));
            out->defer(cap, blk, 0, e);
            for (auto *b : in) { b->reuse_after = e; recycleBatch(b); }
            this->ff_send_out(out);
            return this->GO_ON;
        }
        void check_errors()
        {
            uint32_t nkeys = 0, err = 0;
            if (ffat) wfbErrChk(wfb_ffat_stats(ffat, &nkeys, &err, stream));
            if (err & 1u) wf_fatal("Ffat_Windows_GPU [" + this->opName + "]: more distinct keys than withMaxKeys(" + std::to_string(op.max_keys) + ")");
            if (err & ~1u) wf_fatal("Ffat_Windows_GPU [" + this->opName + "]: more window results in one call than the output batch holds");
        }
        void eosnotify(ssize_t id) override
        {   // nothing is flushed at end of stream (wf/ffat_replica_gpu.hpp:1050-1056); errors raised on the device surface here
            check_errors();
            Basic_Replica::eosnotify(id);
        }
    };
    Replica *make_replica() { return new Replica(*this); }
};

// Keyed_Windows_GPU, count-based (wf/keyed_windows.hpp, wf/window_replica.hpp): func(const Iterable_GPU<tuple_t> &, result_t &) over
// every window of every key, the key's last pow2ceil(win) tuples kept on the device; or func(const tuple_t &, result_t &) folding each
// tuple into the accumulator of every open window it is IN, the key's open accumulators kept on the device (a WFB_KWIN_INCREMENTAL
// handle). svc(): the K batches found queued go to ONE
// wfb_kwin_process_cb call, whose results form one output batch whose size stays on the device; at end of stream the windows that
// opened and did not fire are evaluated on the tuples they have (wf/window_replica.hpp:356-407) and sent as one more batch.
template <class win_func_gpu_t, class keyextr_func_gpu_t>
class Keyed_Windows_GPU: public Basic_Operator {
public:
    using tuple_t = typename window_tuple<fn_arg_t<win_func_gpu_t, 0>>::type;
    using result_t = fn_arg_t<win_func_gpu_t, 1>;
    static constexpr bool isKeyed = !std::is_same<keyextr_func_gpu_t, NoKey<tuple_t>>::value;
    static constexpr bool isIncremental = window_tuple<fn_arg_t<win_func_gpu_t, 0>>::incremental;
    using prog_t = FacadeKeyedWindowsProgram<tuple_t, result_t, win_func_gpu_t, keyextr_func_gpu_t, isKeyed, isIncremental>;
    static constexpr op_type_t op_type = op_type_t::WIN_GPU;
    win_func_gpu_t func; keyextr_func_gpu_t key_extr; uint64_t win_len, slide_len; uint32_t max_keys; size_t maxk;
    Keyed_Windows_GPU(win_func_gpu_t f, keyextr_func_gpu_t k, std::string n, uint64_t w, uint64_t s, uint32_t mk, size_t mbpc):
        Basic_Operator(std::move(n), 1, isKeyed ? Routing_Mode_t::KEYBY : Routing_Mode_t::FORWARD, 1), func(f), key_extr(k),
        win_len(w), slide_len(s), max_keys(mk), maxk(mbpc ? mbpc : 1)
    {
        static_assert(std::is_trivially_copyable<win_func_gpu_t>::value, "GPU functors must be trivially copyable");
        if (win_len == 0 || slide_len == 0) wf_fatal("Keyed_Windows_GPU used with window length or slide equal to zero");
    }
    std::string getType() const override { return "Keyed_Windows_GPU"; }
    keyextr_func_gpu_t getKeyExtractor() const { return key_extr; }
    class Replica: public Batch_Replica<tuple_t, result_t> {
        using base_t = Batch_Replica<tuple_t, result_t>; using base_t::in; using base_t::bi; using base_t::stream;
        Keyed_Windows_GPU op;
        wfb_kwin_t *kw = nullptr; typename prog_t::params_t prm;
        size_t cap_hint = 0, eos_seen = 0; uint64_t last_wm = 0;
        // one output batch of capacity `cap` whose size `call(count_d)` leaves on the device
        template <class Call> void send_results(size_t cap, uint64_t wm, Call &&call)
        {
            Batch_GPU_t<result_t> *out = this->pool.get(cap);
            out->setWatermark(wm);
            if (out->reuse_after) gpuErrChk(cudaStreamWaitEvent(stream, out->reuse_after, 0));
            CountBlock *blk; uint32_t *count_d;
            gpuErrChk(this->counts.acquire(1, blk, count_d));
            wfbErrChk(call(out, count_d));
            gpuErrChk(cudaMemcpyAsync(blk->h, count_d, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
            cudaEvent_t e = this->next_event();
            gpuErrChk(cudaEventRecord(e, stream));
            out->defer(cap, blk, 0, e);
            for (auto *b : in) { b->reuse_after = e; recycleBatch(b); }
            in.clear();
            this->ff_send_out(out);
        }
    public:
        explicit Replica(const Keyed_Windows_GPU &o): base_t(o.name, o.maxk, 64), op(o), prm{o.func, o.key_extr} {}
        ~Replica() override { if (kw) wfb_kwin_destroy(kw); }
        int svc_init() override
        {
            Basic_Replica::svc_init();
            wfbErrChk(wfb_kwin_create(&kw, wfb::register_program<prog_t>(), op.win_len, op.slide_len, op.max_keys, isIncremental ? WFB_KWIN_INCREMENTAL : 0u));
            wfbErrChk(wfb_kwin_set_params(kw, &prm, sizeof(prm)));
            gpuErrChk(this->counts.init(1)); // (one word per call)
            return 0;
        }
        void *svc(void *msg) override
        {
            if (!this->take(msg, true)) return this->GO_ON;
            uint64_t total = 0;
            for (auto *b : in) total += b->size;
            // every window the call can fire: per key, at most one per slide items of its run, plus one
            const uint64_t groups = total / op.slide_len + wfb_kwin_key_capacity(kw) + 1;
            cap_hint = std::max(cap_hint, static_cast<size_t>(std::min<uint64_t>(groups, 0x7fffffffull))); // (never shrinks: recycled batches keep fitting)
            const size_t cap = cap_hint, k = in.size();
            last_wm = in.back()->getWatermark();
            send_results(cap, last_wm, [&](Batch_GPU_t<result_t> *out, uint32_t *count_d) {
                return wfb_kwin_process_cb(kw, bi.data(), static_cast<uint32_t>(k), out->tuples_gpu, out->ts_gpu, static_cast<uint32_t>(cap), count_d, stream);
            });
            return this->GO_ON;
        }
        void check_errors()
        {
            uint32_t nkeys = 0, err = 0;
            if (kw) wfbErrChk(wfb_kwin_stats(kw, &nkeys, &err, stream));
            if (err & 1u) wf_fatal("Keyed_Windows_GPU [" + this->opName + "]: more distinct keys than withMaxKeys(" + std::to_string(op.max_keys) + ")");
            if (err & ~1u) wf_fatal("Keyed_Windows_GPU [" + this->opName + "]: more window results in one call than the output batch holds");
        }
        void eosnotify(ssize_t id) override
        {   // once every input has ended: the open windows of every key (at most ceil(win / slide) each), then the errors raised on the device
            const size_t nin = this->worker_ ? this->worker_->in.size() : 1;
            if (id >= 0 && ++eos_seen < nin) return;
            uint32_t nkeys = 0, err = 0;
            wfbErrChk(wfb_kwin_stats(kw, &nkeys, &err, stream));
            const size_t cap = std::max<size_t>(1, static_cast<size_t>(nkeys) * ((op.win_len + op.slide_len - 1) / op.slide_len));
            in.clear();
            send_results(cap, last_wm, [&](Batch_GPU_t<result_t> *out, uint32_t *count_d) {
                return wfb_kwin_flush(kw, out->tuples_gpu, out->ts_gpu, static_cast<uint32_t>(cap), count_d, stream);
            });
            check_errors();
            Basic_Replica::eosnotify(id);
        }
    };
    Replica *make_replica() { return new Replica(*this); }
};

// ---- builders (wf/builders_gpu.hpp)----------------------------------------------------------------------------------------
// MapGPU_Builder / FilterGPU_Builder / FlatMapGPU_Builder(func).withKeyBy(key_extr): the keyed-stateful operator
template <class func_t, class keyextr_func_gpu_t, Stateful_Kind_t KIND>
class StatefulGPU_Builder {
    func_t func; keyextr_func_gpu_t key; std::string name; size_t parallelism; uint32_t max_keys = 1u << 16; bool grow = false;
    uint32_t max_outputs; // (FlatMap)
public:
    StatefulGPU_Builder(func_t f, keyextr_func_gpu_t k, std::string n, size_t p, uint32_t m = 0): func(f), key(k), name(std::move(n)), parallelism(p), max_outputs(m) {}
    auto &withName(std::string n) { name = std::move(n); return *this; }
    auto &withParallelism(size_t p) { parallelism = p; return *this; }
    auto &withMaxKeys(uint32_t mk) { max_keys = mk; return *this; } // capacity of the device key -> state table (the initial one withKeyGrowth())
    auto &withKeyGrowth() { grow = true; return *this; } // extension: the table grows with the keys, as the reference's map does on the host
    auto &withMaxOutputsPerTuple(uint32_t m) // required by a FlatMap: the output batches hold original_size * m records
    {
        static_assert(KIND == Stateful_Kind_t::FLATMAP, "WindFlow Compilation Error - withMaxOutputsPerTuple() belongs to FlatMapGPU_Builder");
        max_outputs = m; return *this;
    }
    auto build()
    {
        if (KIND == Stateful_Kind_t::FLATMAP && max_outputs == 0) wf_fatal("FlatMapGPU_Builder [" + name + "]: withMaxOutputsPerTuple(m >= 1) is required");
        Stateful_GPU<func_t, keyextr_func_gpu_t, KIND> op(func, key, parallelism, name, max_keys, max_outputs);
        op.grow_keys = grow;
        return op;
    }
};

template <class map_func_gpu_t>
class MapGPU_Builder {
    map_func_gpu_t func; std::string name = "map_gpu"; size_t parallelism = 1; Routing_Mode_t mode = Routing_Mode_t::FORWARD;
    static constexpr size_t arity = std::tuple_size<typename fn_sig<map_func_gpu_t>::args>::value;
public:
    explicit MapGPU_Builder(map_func_gpu_t f): func(f)
    {
        static_assert(arity == 1 || arity == 2,
                      "WindFlow Compilation Error - MapGPU_Builder: __host__ __device__ void(tuple_t &) or void(tuple_t &, state_t &)");
    }
    auto &withName(std::string n) { name = std::move(n); return *this; }
    auto &withParallelism(size_t p) { parallelism = p; return *this; }
    auto &withRebalancing() { mode = Routing_Mode_t::REBALANCING; return *this; }
    template <class keyextr_t> auto withKeyBy(keyextr_t k)
    {
        static_assert(arity == 2, "WindFlow Compilation Error - MapGPU_Builder: withKeyBy() needs the stateful signature void(tuple_t &, state_t &)");
        return StatefulGPU_Builder<map_func_gpu_t, keyextr_t, Stateful_Kind_t::MAP>(func, k, name, parallelism);
    }
    auto build()
    {
        static_assert(arity == 1, "WindFlow Compilation Error - MapGPU_Builder: a stateful functor needs withKeyBy()");
        return Map_GPU<map_func_gpu_t>(func, parallelism, name, mode);
    }
};

template <class filter_func_gpu_t>
class FilterGPU_Builder {
    filter_func_gpu_t func; std::string name = "filter_gpu"; size_t parallelism = 1; Routing_Mode_t mode = Routing_Mode_t::FORWARD;
    static constexpr size_t arity = std::tuple_size<typename fn_sig<filter_func_gpu_t>::args>::value;
public:
    explicit FilterGPU_Builder(filter_func_gpu_t f): func(f)
    {
        static_assert(arity == 1 || arity == 2,
                      "WindFlow Compilation Error - FilterGPU_Builder: __host__ __device__ bool(tuple_t &) or bool(tuple_t &, state_t &)");
    }
    auto &withName(std::string n) { name = std::move(n); return *this; }
    auto &withParallelism(size_t p) { parallelism = p; return *this; }
    auto &withRebalancing() { mode = Routing_Mode_t::REBALANCING; return *this; }
    template <class keyextr_t> auto withKeyBy(keyextr_t k)
    {
        static_assert(arity == 2, "WindFlow Compilation Error - FilterGPU_Builder: withKeyBy() needs the stateful signature bool(tuple_t &, state_t &)");
        return StatefulGPU_Builder<filter_func_gpu_t, keyextr_t, Stateful_Kind_t::FILTER>(func, k, name, parallelism);
    }
    auto build()
    {
        static_assert(arity == 1, "WindFlow Compilation Error - FilterGPU_Builder: a stateful functor needs withKeyBy()");
        return Filter_GPU<filter_func_gpu_t>(func, parallelism, name, mode);
    }
};

template <class flatmap_func_gpu_t>
class FlatMapGPU_Builder {
    flatmap_func_gpu_t func; std::string name = "flatmap_gpu"; size_t parallelism = 1; Routing_Mode_t mode = Routing_Mode_t::FORWARD;
    uint32_t max_outputs = 0;
    using args_t = typename fn_sig<flatmap_func_gpu_t>::args;
    static constexpr size_t arity = std::tuple_size<args_t>::value;
public:
    explicit FlatMapGPU_Builder(flatmap_func_gpu_t f): func(f)
    {
        static_assert(arity == 3 || (arity == 2 &&
                      std::is_same<fn_ret_t<flatmap_func_gpu_t>, void>::value &&
                      std::is_same<std::tuple_element_t<1, args_t>,
                                   Shipper_GPU<typename shipper_result<fn_arg_t<flatmap_func_gpu_t, 1>>::type> &>::value),
                      "WindFlow Compilation Error - FlatMapGPU_Builder: __host__ __device__ void(const tuple_t &, Shipper_GPU<result_t> &)");
        if constexpr (arity == 3)
            static_assert(std::is_same<fn_ret_t<flatmap_func_gpu_t>, void>::value &&
                          std::is_same<std::tuple_element_t<1, args_t>, Shipper_GPU<typename shipper_result<fn_arg_t<flatmap_func_gpu_t, 1>>::type> &>::value &&
                          std::is_same<std::tuple_element_t<2, args_t>, fn_arg_t<flatmap_func_gpu_t, 2> &>::value,
                          "WindFlow Compilation Error - FlatMapGPU_Builder: __host__ __device__ void(const tuple_t &, Shipper_GPU<result_t> &, state_t &)");
    }
    auto &withName(std::string n) { name = std::move(n); return *this; }
    auto &withParallelism(size_t p) { parallelism = p; return *this; }
    auto &withRebalancing() { mode = Routing_Mode_t::REBALANCING; return *this; }
    auto &withMaxOutputsPerTuple(uint32_t m) { max_outputs = m; return *this; } // required: the output batches hold original_size * m records
    template <class keyextr_t> auto withKeyBy(keyextr_t k)
    {
        static_assert(arity == 3, "WindFlow Compilation Error - FlatMapGPU_Builder: withKeyBy() needs the stateful signature "
                                  "void(const tuple_t &, Shipper_GPU<result_t> &, state_t &)");
        return StatefulGPU_Builder<flatmap_func_gpu_t, keyextr_t, Stateful_Kind_t::FLATMAP>(func, k, name, parallelism, max_outputs);
    }
    auto build()
    {
        static_assert(arity == 2, "WindFlow Compilation Error - FlatMapGPU_Builder: a stateful functor needs withKeyBy()");
        if (max_outputs == 0) wf_fatal("FlatMapGPU_Builder [" + name + "]: withMaxOutputsPerTuple(m >= 1) is required");
        return FlatMap_GPU<flatmap_func_gpu_t>(func, parallelism, name, mode, max_outputs);
    }
};

template <class reduce_func_gpu_t, class keyextr_func_gpu_t = NoKey<fn_arg_t<reduce_func_gpu_t, 0>>>
class ReduceGPU_Builder {
    template <class A, class B> friend class ReduceGPU_Builder;
    reduce_func_gpu_t func; keyextr_func_gpu_t key_extr; std::string name = "reduce_gpu"; size_t parallelism = 1;
    Routing_Mode_t mode = Routing_Mode_t::FORWARD; uint32_t key_bits = 64;
    ReduceGPU_Builder(reduce_func_gpu_t f, keyextr_func_gpu_t k): func(f), key_extr(k) {}
public:
    explicit ReduceGPU_Builder(reduce_func_gpu_t f): func(f), key_extr() {}
    auto &withName(std::string n) { name = std::move(n); return *this; }
    auto &withParallelism(size_t p) { parallelism = p; return *this; }
    auto &withKeyBits(uint32_t b) { key_bits = b; return *this; } // extension: significant low bits of an integral key (fewer radix passes)
    template <class new_keyextr_t> auto withKeyBy(new_keyextr_t k)
    {
        ReduceGPU_Builder<reduce_func_gpu_t, new_keyextr_t> nb(func, k);
        nb.name = name; nb.parallelism = parallelism; nb.mode = Routing_Mode_t::KEYBY; nb.key_bits = key_bits;
        return nb;
    }
    auto build()
    {   // (withKeyBits may precede withKeyBy: the key type is known here)
        if (key_bits != 64 && !integral_key_v<keyextr_func_gpu_t>) wf_fatal("ReduceGPU_Builder: withKeyBits() needs an integral or enum key type");
        Reduce_GPU<reduce_func_gpu_t, keyextr_func_gpu_t> r(func, key_extr, parallelism, name, mode); r.key_bits = key_bits; return r;
    }
};

template <class lift_func_gpu_t, class comb_func_gpu_t, class keyextr_func_gpu_t = NoKey<fn_arg_t<lift_func_gpu_t, 0>>>
class Ffat_WindowsGPU_Builder {
    template <class A, class B, class C> friend class Ffat_WindowsGPU_Builder;
    lift_func_gpu_t lift; comb_func_gpu_t comb; keyextr_func_gpu_t key_extr; std::string name = "ffat_windows_gpu";
    size_t numWinPerBatch = 0, max_batches = WF_MAX_BATCHES_PER_CALL; uint64_t win_len = 0, slide_len = 0, lateness = 0; Win_Type_t winType = Win_Type_t::CB;
    uint32_t max_keys = 65536; bool dense = false, grow = false;
    Ffat_WindowsGPU_Builder(lift_func_gpu_t l, comb_func_gpu_t c, keyextr_func_gpu_t k): lift(l), comb(c), key_extr(k) {}
public:
    Ffat_WindowsGPU_Builder(lift_func_gpu_t l, comb_func_gpu_t c): lift(l), comb(c), key_extr() {}
    auto &withName(std::string n) { name = std::move(n); return *this; }
    template <class new_keyextr_t> auto withKeyBy(new_keyextr_t k)
    {
        Ffat_WindowsGPU_Builder<lift_func_gpu_t, comb_func_gpu_t, new_keyextr_t> nb(lift, comb, k);
        nb.name = name; nb.numWinPerBatch = numWinPerBatch; nb.win_len = win_len; nb.slide_len = slide_len; nb.lateness = lateness;
        nb.winType = winType; nb.max_keys = max_keys; nb.dense = dense; nb.grow = grow; nb.max_batches = max_batches;
        return nb;
    }
    auto &withCBWindows(uint64_t w, uint64_t s) { win_len = w; slide_len = s; winType = Win_Type_t::CB; lateness = 0; return *this; }
    auto &withTBWindows(std::chrono::microseconds w, std::chrono::microseconds s) { win_len = w.count(); slide_len = s.count(); winType = Win_Type_t::TB; return *this; }
    auto &withLateness(std::chrono::microseconds l) { lateness = l.count(); return *this; }
    auto &withNumWinPerBatch(size_t n) { numWinPerBatch = n; return *this; }
    auto &withMaxKeys(uint32_t n) { max_keys = n; return *this; }       // extension: capacity of the device-resident key table (the initial one withKeyGrowth())
    auto &withKeyGrowth() { grow = true; return *this; }                // extension: the key table grows with the keys (not with withDenseKeys)
    auto &withDenseKeys()                                               // extension: keys are 0 .. max_keys-1 (slot = key, no hash probe)
    {
        static_assert(integral_key_v<keyextr_func_gpu_t>, "WindFlow Compilation Error - Ffat_WindowsGPU_Builder: withDenseKeys() needs an integral or enum key type:\n");
        dense = true; return *this;
    }
    auto &withMaxBatchesPerCall(size_t k) { max_batches = k; return *this; } // extension: queued batches one svc() hands to one launch sequence
    auto build()
    {   // (withDenseKeys before withKeyBy: the key type is known here)
        if (dense && !integral_key_v<keyextr_func_gpu_t>) wf_fatal("Ffat_WindowsGPU_Builder: withDenseKeys() needs an integral or enum key type");
        if (dense && grow) wf_fatal("Ffat_WindowsGPU_Builder: withKeyGrowth() cannot be combined with withDenseKeys()");
        Ffat_Windows_GPU<lift_func_gpu_t, comb_func_gpu_t, keyextr_func_gpu_t> w(lift, comb, key_extr, name, win_len, slide_len, lateness, winType, numWinPerBatch, max_keys, dense, max_batches);
        w.grow_keys = grow;
        return w;
    }
};

// Keyed_WindowsGPU_Builder(win_func).withKeyBy(k).withCBWindows(w, s): win_func is __host__ __device__
// void(const Iterable_GPU<tuple_t> &, result_t &) or, incremental, __host__ __device__ void(const tuple_t &, result_t &)
// (wf/builders.hpp, Keyed_Windows_Builder); without withKeyBy every tuple has one key (and withMaxKeys is ignored)
template <class win_func_gpu_t, class keyextr_func_gpu_t = NoKey<typename window_tuple<fn_arg_t<win_func_gpu_t, 0>>::type>>
class Keyed_WindowsGPU_Builder {
    template <class A, class B> friend class Keyed_WindowsGPU_Builder;
    win_func_gpu_t func; keyextr_func_gpu_t key_extr; std::string name = "keyed_windows_gpu";
    uint64_t win_len = 0, slide_len = 0; uint32_t max_keys = 65536; size_t max_batches = WF_MAX_BATCHES_PER_CALL;
    Keyed_WindowsGPU_Builder(win_func_gpu_t f, keyextr_func_gpu_t k): func(f), key_extr(k) {}
    using args_t = typename fn_sig<win_func_gpu_t>::args;
public:
    explicit Keyed_WindowsGPU_Builder(win_func_gpu_t f): func(f), key_extr()
    {
        using T = typename window_tuple<fn_arg_t<win_func_gpu_t, 0>>::type;
        static_assert(std::tuple_size<args_t>::value == 2 && std::is_same<fn_ret_t<win_func_gpu_t>, void>::value &&
                      (std::is_same<std::tuple_element_t<0, args_t>, const Iterable_GPU<T> &>::value ||
                       std::is_same<std::tuple_element_t<0, args_t>, const T &>::value) &&
                      std::is_same<std::tuple_element_t<1, args_t>, fn_arg_t<win_func_gpu_t, 1> &>::value,
                      "WindFlow Compilation Error - unknown signature passed to the Keyed_WindowsGPU_Builder:\n"
                      "  Candidate 1 : __host__ __device__ void(const Iterable_GPU<tuple_t> &, result_t &)\n"
                      "  Candidate 2 : __host__ __device__ void(const tuple_t &, result_t &)\n");
    }
    auto &withName(std::string n) { name = std::move(n); return *this; }
    template <class new_keyextr_t> auto withKeyBy(new_keyextr_t k)
    {
        Keyed_WindowsGPU_Builder<win_func_gpu_t, new_keyextr_t> nb(func, k);
        nb.name = name; nb.win_len = win_len; nb.slide_len = slide_len; nb.max_keys = max_keys; nb.max_batches = max_batches;
        return nb;
    }
    auto &withCBWindows(uint64_t w, uint64_t s) { win_len = w; slide_len = s; return *this; }
    auto &withMaxKeys(uint32_t n) { max_keys = n; return *this; }            // extension: capacity of the device key table and archive
    auto &withMaxBatchesPerCall(size_t k) { max_batches = k; return *this; } // extension: queued batches one svc() hands to one launch sequence
    auto build()
    {   // (without withKeyBy every tuple has the one key: a table, a ring and an output bound for one key)
        using op_t = Keyed_Windows_GPU<win_func_gpu_t, keyextr_func_gpu_t>;
        return op_t(func, key_extr, name, win_len, slide_len, op_t::isKeyed ? max_keys : 1u, max_batches);
    }
};

// ---- MultiPipe / PipeGraph (wf/multipipe.hpp, wf/pipegraph.hpp) ------------------------------------------------------------------------
// A MultiPipe is a sequence of stages; a stage is the group of replicas of one operator (ff_group), consecutive stages are connected
// all-to-all by the runtime (a producer sends a batch to ONE consumer replica, round-robin: batches are the unit of routing on the
// GPU path, wf/keyby_emitter_gpu.hpp:519-583). A run of stateless Map_GPU / Filter_GPU operators stays pending until the next
// operator arrives: a Ffat_Windows_GPU over the same tuple type absorbs it as its `pre` stage, anything else turns it into ONE
// replica group running one fused streaming pass.
class PipeGraph;
template <class... Ops> class FusedPipe;
class MultiPipe {
    friend class PipeGraph;
    template <class... Ops> friend class FusedPipe;
    ff::ff_pipeline pipe;
    std::vector<std::string> op_names;
    bool has_sink = false, tail_is_gpu = false; size_t prevOutputBatchSize = 0;
    // the pending fused run
    StageChain pending{}; std::type_index pending_type{typeid(void)}; size_t pending_par = 1; std::string pending_name;
    std::function<void()> materialize_pending; // creates the ChainReplica group for the pending run

    void add_stage(ff::ff_group *g) { pipe.add_stage(g, true); }
    template <class op_t> void attach(op_t &op)
    {
        if (has_sink) wf_fatal("MultiPipe is already terminated by a Sink");
        if (!tail_is_gpu && prevOutputBatchSize == 0)  // wf/multipipe.hpp:486-488
            wf_fatal(op.getType() + " cannot be added after a CPU operator without withOutputBatchSize()");
        op.setExecutionMode(Execution_Mode_t::DEFAULT);
        op_names.push_back(op.getName());
    }
    void flush_pending() { if (pending.n) { materialize_pending(); pending = StageChain{}; pending_type = std::type_index(typeid(void)); materialize_pending = nullptr; } }
    template <class func_t, bool F> MultiPipe &chain_stateless(Stateless_GPU<func_t, F> op)
    {
        using T = typename Stateless_GPU<func_t, F>::tuple_t;
        attach(op);
        const bool same_run = pending.n && pending_type == std::type_index(typeid(T)) && pending_par == op.getParallelism();
        if (!same_run) flush_pending();
        if (!op.append_to(pending)) { flush_pending(); if (!op.append_to(pending)) wf_fatal(op.getType() + " functor object larger than " + std::to_string(WF_FUNCTOR_BYTES) + " bytes"); }
        if (pending.n == 1) { pending_type = std::type_index(typeid(T)); pending_par = op.getParallelism(); pending_name = op.getName(); }
        else pending_name += "+" + op.getName();
        materialize_pending = [this]() {
            auto *g = new ff::ff_group();
            for (size_t i = 0; i < pending_par; i++) g->add(new ChainReplica<T>(pending_name, pending, pending_par > 1 ? 1 : WF_MAX_BATCHES_PER_CALL), true);
            add_stage(g);
        };
        tail_is_gpu = true;
        return *this;
    }
    template <class op_t> MultiPipe &add_replicated(op_t &op)
    {
        attach(op);
        flush_pending();
        auto *g = new ff::ff_group();
        for (size_t i = 0; i < op.getParallelism(); i++) g->add(op.make_replica(), true);
        add_stage(g);
        tail_is_gpu = true;
        return *this;
    }
public:
    // chain == add here: an operator that cannot be fused into its neighbour runs on its own thread, so that its input queue
    // can fill while it works (the replica then takes everything queued in one call)
    // (stateless operators return a proxy that remembers the functor types while the expression goes on: FusedPipe below)
    template <class F, bool IS> FusedPipe<Stateless_GPU<F, IS>> chain(Stateless_GPU<F, IS> op);
    template <class F, class K, Stateful_Kind_t KIND> MultiPipe &chain(Stateful_GPU<F, K, KIND> op) { return add_replicated(op); }
    template <class F, class K> MultiPipe &chain(Reduce_GPU<F, K> op) { return add_replicated(op); }
    template <class F, class K> MultiPipe &chain(Keyed_Windows_GPU<F, K> op) { return add_replicated(op); } // (a pending stateless run is materialised in front)
    template <class F> MultiPipe &chain(FlatMap_GPU<F> op)
    {
        using T = typename FlatMap_GPU<F>::tuple_t;
        attach(op);
        StageChain pre{}; // a pending run over the same tuples with the same parallelism runs in the FlatMap's own pass
        if (pending.n && pending_type == std::type_index(typeid(T)) && pending_par == op.getParallelism()) {
            pre = pending;
            pending = StageChain{}; pending_type = std::type_index(typeid(void)); materialize_pending = nullptr;
        } else flush_pending();
        auto *g = new ff::ff_group();
        for (size_t i = 0; i < op.getParallelism(); i++) g->add(op.make_replica(pre), true);
        add_stage(g);
        tail_is_gpu = true;
        return *this;
    }
    template <class L, class C, class K> MultiPipe &chain(Ffat_Windows_GPU<L, C, K> op)
    {
        using T = typename Ffat_Windows_GPU<L, C, K>::tuple_t;
        if (pending.n && pending_type == std::type_index(typeid(T))) { // the run in front becomes the window operator's own ingest stage
            op.pre.c = pending;
            pending = StageChain{}; pending_type = std::type_index(typeid(void)); materialize_pending = nullptr;
        }
        return add_replicated(op);
    }
    template <class op_t> auto add(op_t op) -> decltype(this->chain(op)) { return chain(op); }
    template <class sink_f> MultiPipe &chain_sink(Sink<sink_f> op)
    {
        if (has_sink) wf_fatal("MultiPipe is already terminated by a Sink");
        flush_pending();
        using T = std::decay_t<decltype(*std::declval<fn_arg_t<sink_f, 0>>())>; // std::optional<tuple_t> & -> tuple_t
        auto *g = new ff::ff_group();
        for (size_t i = 0; i < op.getParallelism(); i++) g->add(new SinkReplica<T, sink_f>(op.getName(), op.func, op.wm_probe), true);
        add_stage(g);
        op_names.push_back(op.getName()); has_sink = true;
        return *this;
    }
    template <class sink_f> MultiPipe &add_sink(Sink<sink_f> op) { return chain_sink(op); }
    size_t getNumThreads() const { return static_cast<size_t>(pipe.cardinality()); }
    const std::vector<std::string> &getOperatorNames() const { return op_names; }
};

// What pipe.chain(map_or_filter) returns: the MultiPipe plus the stateless operators of the expression so far, with their types.
//   .chain(another Map_GPU / Filter_GPU)   -> a longer FusedPipe
//   .chain / .add(Ffat_Windows_GPU)        -> the run becomes part of the window operator's PROGRAM TYPE (TypedChain): its functors are
//                                             inlined into the tile pass -- the pipeline of BASELINE.json is one kernel with no indirect call
//   anything else, conversion to MultiPipe &, or the end of the statement -> the operators are handed to the MultiPipe as usual (the
//                                             run stays open there: a window operator chained by a later statement still absorbs it, through thunks)
template <class... Ops>
class FusedPipe {
    MultiPipe *mp; std::tuple<Ops...> ops; bool done = false;
    template <class... O> friend class FusedPipe;
public:
    FusedPipe(MultiPipe &m, std::tuple<Ops...> o): mp(&m), ops(std::move(o)) {}
    FusedPipe(FusedPipe &&o) noexcept: mp(o.mp), ops(std::move(o.ops)), done(o.done) { o.done = true; }
    FusedPipe(const FusedPipe &) = delete;
    ~FusedPipe() { if (!done) materialize(); }
    MultiPipe &materialize()
    {
        if (!done) { done = true; std::apply([this](auto &...op) { (mp->chain_stateless(op), ...); }, ops); }
        return *mp;
    }
    operator MultiPipe &() { return materialize(); }
    template <class F, bool IS> FusedPipe<Ops..., Stateless_GPU<F, IS>> chain(Stateless_GPU<F, IS> op)
    {
        if (done) wf_fatal("FusedPipe used after it was handed over");
        done = true;
        return FusedPipe<Ops..., Stateless_GPU<F, IS>>(*mp, std::tuple_cat(std::move(ops), std::make_tuple(op)));
    }
    template <class L, class C, class K> MultiPipe &chain(Ffat_Windows_GPU<L, C, K> op)
    {
        using T = typename Ffat_Windows_GPU<L, C, K>::tuple_t;
        constexpr bool same_type = (std::is_same<typename Ops::tuple_t, T>::value && ...);
        if constexpr (!same_type) return materialize().chain(op);
        else {
            if (done) wf_fatal("FusedPipe used after it was handed over");
            if (mp->pending.n) return materialize().chain(op); // (an open run of earlier statements goes first: thunks for all of it)
            done = true;
            std::apply([this](auto &...o) { (mp->attach(o), ...); }, ops);
            using pre_t = TypedChain<T, TypedStage<decltype(std::declval<Ops>().func), Ops::is_filter>...>;
            pre_t pre = std::apply([](auto &...o) { return make_typed_chain<T>(TypedStage<decltype(o.func), std::decay_t<decltype(o)>::is_filter>{o.func}...); }, ops);
            Ffat_Windows_GPU<L, C, K, pre_t> fop(op, pre);
            mp->tail_is_gpu = true;
            return mp->add_replicated(fop);
        }
    }
    template <class Op> decltype(auto) chain(Op op) { return materialize().chain(op); }
    template <class Op> decltype(auto) add(Op op) { return this->chain(op); }
    template <class sink_f> MultiPipe &chain_sink(Sink<sink_f> op) { return materialize().chain_sink(op); }
    template <class sink_f> MultiPipe &add_sink(Sink<sink_f> op) { return materialize().chain_sink(op); }
    size_t getNumThreads() { return materialize().getNumThreads(); }
    const std::vector<std::string> &getOperatorNames() { return materialize().getOperatorNames(); }
};
template <class F, bool IS> FusedPipe<Stateless_GPU<F, IS>> MultiPipe::chain(Stateless_GPU<F, IS> op) { return FusedPipe<Stateless_GPU<F, IS>>(*this, std::make_tuple(op)); }

class PipeGraph {
    std::string name; Execution_Mode_t mode; Time_Policy_t policy;
    std::vector<std::unique_ptr<MultiPipe>> pipes;
public:
    PipeGraph(std::string n, Execution_Mode_t m = Execution_Mode_t::DEFAULT, Time_Policy_t p = Time_Policy_t::INGRESS_TIME): name(std::move(n)), mode(m), policy(p)
    {
        if (wfb_device_count() <= 0) wf_fatal("no CUDA device: the GPU operators have no CPU fallback");
    }
    template <class src_f> MultiPipe &add_source(Source<src_f> src)
    {
        using T = typename shipper_tuple<std::decay_t<fn_arg_t<src_f, 0>>>::type;
        if (src.getOutputBatchSize() == 0) wf_fatal("Source feeding GPU operators must be built withOutputBatchSize(n > 0)"); // multipipe.hpp:486-488
        auto mp = std::make_unique<MultiPipe>();
        auto *g = new ff::ff_group();
        for (size_t i = 0; i < src.getParallelism(); i++)
            g->add(new SourceReplica<T>(src.getName(), std::function<void(Source_Shipper<T> &)>(src.func), src.getOutputBatchSize()), true);
        mp->add_stage(g);
        mp->prevOutputBatchSize = src.getOutputBatchSize();
        mp->op_names.push_back(src.getName());
        pipes.push_back(std::move(mp));
        return *pipes.back();
    }
    template <class src_f> MultiPipe &add_source(SourceGPU<src_f> src)
    {
        using T = typename shipper_tuple<std::decay_t<fn_arg_t<src_f, 0>>>::type;
        auto mp = std::make_unique<MultiPipe>();
        auto *g = new ff::ff_group();
        g->add(new SourceGPUReplica<T>(src.getName(), std::function<void(SourceGPU_Shipper<T> &)>(src.func)), true);
        mp->add_stage(g);
        mp->prevOutputBatchSize = 1; mp->tail_is_gpu = true;
        mp->op_names.push_back(src.getName());
        pipes.push_back(std::move(mp));
        return *pipes.back();
    }
    size_t getNumThreads() const { size_t n = 0; for (auto &p : pipes) n += p->getNumThreads(); return n; }
    int start()
    {
        if (mode != Execution_Mode_t::DEFAULT) wf_fatal("GPU operators can only be used in DEFAULT mode");
        for (auto &p : pipes) { if (!p->has_sink) wf_fatal("MultiPipe without a Sink"); }
        for (auto &p : pipes) if (p->pipe.run() < 0) return -1;
        return 0;
    }
    int wait_end()
    {
        for (auto &p : pipes) p->pipe.wait();
        gpuErrChk(cudaDeviceSynchronize());
        return 0;
    }
    int run() { if (start() < 0) return -1; return wait_end(); }
};

} // namespace wf
