// keyed_windows_bench.cu -- Keyed_Windows_GPU written against the builder API (include/wf/windflow_gpu.hpp), driven as an application
// drives it:
//
//     SourceGPU (a ring of batches resident in HBM) -> Map_GPU -> Filter_GPU -> Keyed_Windows_GPU (count-based, hashed keys) -> Sink
//
// 64-byte tuples of the seeded synthetic stream (batch 65536, uniform keys), map ivalue += 2 / fvalue *= 1.0000001, filter
// (ivalue & 1) == 0, and a window function that reads every tuple of its window (the one of tests/cpp/kwin_programs.cu), or with
// inc=1 the incremental function of tests/cpp/kwin_inc_programs.cu, void(const tuple64_t &, result80_t &).
// tools/keyed_windows_bench.py runs it as the builder arms.
//   usage: keyed_windows_bench.bin [K=128] [timed_batches=2048] [keys=65536] [win=1024] [slide=64] [ring_batches=256] [inc=0]
// prints one JSON line.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <functional>
#include <optional>
#include <thread>
#include <wf/windflow_gpu.hpp>

using namespace wf;

struct tuple64_t { uint64_t key, id; int64_t ivalue; double fvalue; uint64_t pad[4]; };
struct result72_t {
    uint64_t key, id, hash, size, mid, front, back, distinct; double fsum;
    __host__ __device__ result72_t(): key(0), id(0), hash(0), size(0), mid(0), front(0), back(0), distinct(0), fsum(0) {}
    __host__ __device__ result72_t(uint64_t k, uint64_t g): key(k), id(g), hash(0), size(0), mid(0), front(0), back(0), distinct(0), fsum(0) {}
};
struct result80_t {
    uint64_t key, id, hash, size, front, back, mask; double fsum; uint64_t argmax; int64_t maxiv;
    __host__ __device__ result80_t(): key(0), id(0), hash(0), size(0), front(0), back(0), mask(0), fsum(0), argmax(0), maxiv(0) {}
    __host__ __device__ result80_t(uint64_t k, uint64_t g): result80_t() { key = k; id = g; }
};
struct MapF { __host__ __device__ void operator()(tuple64_t &t) { t.ivalue += 2; t.fvalue *= 1.0000001; } };
struct FiltF { __host__ __device__ bool operator()(tuple64_t &t) { return (t.ivalue & 1) == 0; } };
struct KeyF { __host__ __device__ uint64_t operator()(const tuple64_t &t) { return t.key; } };
struct WinF {
    __host__ __device__ void operator()(const Iterable_GPU<tuple64_t> &w, result72_t &r) const
    {
        constexpr uint64_t MIX = 0x9E3779B97F4A7C15ull, MUL = 0x100000001B3ull;
        uint64_t h = 0; double s = 0.0; uint32_t seen = 0;
        for (auto it = w.begin(); it != w.end(); ++it) {
            h = h * MUL + (it->id * MIX ^ static_cast<uint64_t>(it->ivalue));
            s += it->fvalue;
            seen |= 1u << (static_cast<uint64_t>(it->ivalue) & 15u);
        }
        r.hash = h; r.fsum = s; r.size = w.size(); r.mid = w[w.size() / 2].id; r.front = w.front().id; r.back = w.back().id;
        r.distinct = static_cast<uint64_t>(__builtin_popcount(seen));
    }
};

struct WinIncF {
    __host__ __device__ void operator()(const tuple64_t &t, result80_t &r) const
    {
        constexpr uint64_t MIX = 0x9E3779B97F4A7C15ull, MUL = 0x100000001B3ull;
        if (r.size == 0 || t.ivalue > r.maxiv) { r.maxiv = t.ivalue; r.argmax = t.id; }
        if (r.size == 0) r.front = t.id;
        r.hash = r.hash * MUL + (t.id * MIX ^ static_cast<uint64_t>(t.ivalue));
        r.size++; r.back = t.id;
        r.mask |= 1ull << (static_cast<uint64_t>(t.ivalue) & 15u);
        r.fsum += t.fvalue;
    }
};

static std::atomic<uint64_t> g_seen_wm{0}; // watermark (= index of the last input batch) of the newest result batch the sink has seen
static std::atomic<uint64_t> g_windows{0};
template <class R> struct SinkF {
    uint64_t windows = 0;
    void operator()(std::optional<R> &r) { if (r) windows++; else g_windows.fetch_add(windows); }
};

template <class Win, class R>
static size_t run_graph(Win winf, size_t K, uint64_t nkeys, uint64_t win, uint64_t slide, std::function<void(SourceGPU_Shipper<tuple64_t> &)> source)
{
    PipeGraph graph("keyed_windows_bench", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(SourceGPU_Builder(source).withName("source").build());
    mp.chain(MapGPU_Builder(MapF()).withName("map").build());
    mp.chain(FilterGPU_Builder(FiltF()).withName("filter").build());
    mp.add(Keyed_WindowsGPU_Builder(winf).withName("keyed_windows").withKeyBy(KeyF()).withCBWindows(win, slide)
               .withMaxKeys(static_cast<uint32_t>(nkeys)).withMaxBatchesPerCall(K).build());
    mp.chain_sink(Sink_Builder(SinkF<R>()).withName("sink").withWatermarkProbe(&g_seen_wm).build());
    const size_t threads = graph.getNumThreads();
    graph.run();
    return threads;
}

int main(int argc, char **argv)
{
    const size_t K = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 128;
    const uint64_t timed = argc > 2 ? std::strtoull(argv[2], nullptr, 10) : 2048;
    const uint64_t nkeys = argc > 3 ? std::strtoull(argv[3], nullptr, 10) : 65536;
    const uint64_t win = argc > 4 ? std::strtoull(argv[4], nullptr, 10) : 1024;
    const uint64_t slide = argc > 5 ? std::strtoull(argv[5], nullptr, 10) : 64;
    const uint64_t ring = argc > 6 ? std::strtoull(argv[6], nullptr, 10) : 256;
    const bool inc = argc > 7 && std::strtoull(argv[7], nullptr, 10) != 0;
    const uint64_t BATCH = 65536;
    // every key past its first window before the clock starts: win + 1 surviving tuples per key at selectivity 0.5 (at most 8192
    // batches: with longer windows the timed batches mostly fold into windows that stay open)
    const uint64_t prime = std::min<uint64_t>((2 * (win + 1) * nkeys + BATCH - 1) / BATCH, 8192) + ring;

    tuple64_t *d_tuples = nullptr; uint64_t *d_ts = nullptr;
    gpuErrChk(cudaMalloc(&d_tuples, ring * BATCH * sizeof(tuple64_t)));
    gpuErrChk(cudaMalloc(&d_ts, ring * BATCH * sizeof(uint64_t)));
    for (uint64_t r = 0; r < ring; r++)
        wfbErrChk(wfb_gen_tuple64(0x5EED5EEDull, r * BATCH, static_cast<uint32_t>(BATCH), 1, nkeys, nullptr, d_tuples + r * BATCH, d_ts + r * BATCH, nullptr));
    gpuErrChk(cudaDeviceSynchronize());

    std::chrono::steady_clock::time_point t0, t1;
    auto source = [&](SourceGPU_Shipper<tuple64_t> &sh) {
        auto push = [&](uint64_t i) { const uint64_t r = i % ring; sh.pushBatch(d_tuples + r * BATCH, d_ts + r * BATCH, BATCH, i + 1); };
        auto drained = [&](uint64_t upto) { while (g_seen_wm.load(std::memory_order_acquire) < upto) std::this_thread::sleep_for(std::chrono::microseconds(50)); };
        for (uint64_t i = 0; i < prime; i++) push(i);
        drained(prime);
        t0 = std::chrono::steady_clock::now();
        for (uint64_t i = prime; i < prime + timed; i++) push(i);
        drained(prime + timed);
        t1 = std::chrono::steady_clock::now();
    };
    const size_t threads = inc ? run_graph<WinIncF, result80_t>(WinIncF(), K, nkeys, win, slide, source)
                               : run_graph<WinF, result72_t>(WinF(), K, nkeys, win, slide, source);
    const double sec = std::chrono::duration<double>(t1 - t0).count();
    std::printf("{\"arm\": \"%s\", \"max_batches_per_call\": %zu, \"tuples\": %llu, \"seconds\": %.6f, \"tuples_per_s\": %.1f, \"windows\": %llu, "
                "\"threads\": %zu, \"keys\": %llu, \"win\": %llu, \"slide\": %llu, \"primed_batches\": %llu}\n",
                inc ? "builder_inc" : "builder", K, static_cast<unsigned long long>(timed * BATCH), sec, timed * BATCH / sec,
                static_cast<unsigned long long>(g_windows.load()), threads,
                static_cast<unsigned long long>(nkeys), static_cast<unsigned long long>(win), static_cast<unsigned long long>(slide),
                static_cast<unsigned long long>(prime));
    cudaFree(d_tuples); cudaFree(d_ts);
    return 0;
}
