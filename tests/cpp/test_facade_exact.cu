// Exact, order-sensitive application-level test of the builder API (include/wf/windflow_gpu.hpp) at a size where its machinery cycles:
// batch pools recycle, deferred sizes travel (also of batches a filter emptied), replicas drain K batches per call, a producer runs
// hundreds of calls ahead of a slow Sink. 400 300 tuples of 24 bytes {key, seq, value} over 300 hashed, Zipf-distributed keys go through
//   cb_thunk_K{1,7,128}  Source -> Map -> Filter -> count-based Ffat_Windows_GPU (one chain per statement: fused through thunks)
//   cb_typed             the same as one fluent expression (the functor types reach the window operator's program)
//   cb_mmff_thunk/_typed Map -> Filter -> Map -> Filter -> windows on both routes
//   chain_sink           Source -> Map -> Filter -> Sink
//   stateful_p1 / _p2    Source -> Map -> Filter -> keyed-stateful Map -> keyed-stateful Filter -> Sink over a 24-byte state
//   reduce_bits16/_64    Source -> keyed Reduce_GPU
//   tb_ooo               Source -> time-based Ffat_Windows_GPU, out-of-order timestamps within the lateness, idle gaps
//   slow_sink_cb/_tb, slow_sinks_filter   the producer of deferred sizes far ahead of a Sink that is slow at first
// Every window folds a polynomial hash (associative, not commutative), so two tuples, windows or batches swapped change the output.
// The program writes its stream and the rows every Sink received, in arrival order, to the directory argv[1];
// tests/test_facade_exact.py rebuilds the expected rows with numpy and compares every field. `--host-check DIR` applies the same
// functors on the host (no device needed) and writes the rows in the same formats. Prints EXACT_OK on success.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <optional>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>
#include <wf/windflow_gpu.hpp>

using namespace wf;

constexpr uint64_t N = 400300, BATCH = 1000, NKEYS = 300, WIN = 48, SLIDE = 16, NWB = 3, MAXKEYS = 512;
constexpr uint64_t DROP_LO = 37000, DROP_HI = 41000;                       // the filter drops every tuple of these whole batches
constexpr uint64_t TB_WIN = 400, TB_SLIDE = 100, TB_NWB = 2, TB_LATE = 150; // time-based: timestamp units
constexpr uint64_t SLOW_BATCH = 500, SLOW_BATCHES = 800, SINKS_BATCH = 64, SINKS_BATCHES = 5000;
constexpr uint64_t MULT = 0x5851F42D4C957F2Dull;

struct tuple_t { uint64_t key, seq, value; };
struct result_t {
    uint64_t key, id, h, q;
    __host__ __device__ result_t(): key(0), id(0), h(0), q(0) {}
    __host__ __device__ result_t(uint64_t k, uint64_t i): key(k), id(i), h(0), q(0) {}
};
struct state_t { uint64_t count, hash, last; };
static_assert(sizeof(tuple_t) == 24 && sizeof(result_t) == 32 && sizeof(state_t) == 24, "record sizes");

// ---- functors, as an application writes them ------------------------------------------------------------------------------------------
// nonzero item hash of two words (the lift of the programs of tests/cpp/ordered_programs.cu, restated)
__host__ __device__ inline uint64_t ord_mix(uint64_t id, uint64_t k0)
{
    uint64_t x = ((id + 1) * 0x9E3779B97F4A7C15ull) ^ (k0 * 0xC2B2AE3D27D4EB4Full);
    x ^= x >> 29;
    return x | 1u;
}
__host__ __device__ inline uint64_t ord_pow(uint64_t b, uint64_t e)
{
    uint64_t r = 1;
    for (; e; e >>= 1, b *= b) if (e & 1) r *= b;
    return r;
}
struct MapA { __host__ __device__ void operator()(tuple_t &t) const { t.value = ((t.seq * t.seq) ^ (t.seq >> 3)) * 0x9E3779B97F4A7C15ull + t.key; } };
struct FiltA { __host__ __device__ bool operator()(tuple_t &t) const { return (t.value >> 11) % 3 != 0 && !(t.seq >= DROP_LO && t.seq < DROP_HI); } };
struct MapB { __host__ __device__ void operator()(tuple_t &t) const { t.value = (t.value ^ (t.value >> 17)) * 0xD6E8FEB86659FD93ull + t.seq; } };
struct FiltB { __host__ __device__ bool operator()(tuple_t &t) const { return (t.value >> 9) % 5 != 0; } };
struct KeyF { __host__ __device__ uint64_t operator()(const tuple_t &t) const { return t.key; } };
struct Lift { __host__ __device__ void operator()(const tuple_t &t, result_t &r) const { r.key = t.key; r.id = 0; r.h = ord_mix(t.value, t.key); r.q = 1; } };
struct Comb { // (h1, q1) o (h2, q2) = (h1 M^q2 + h2, q1 + q2): q is the length of the folded sequence
    __host__ __device__ void operator()(const result_t &a, const result_t &b, result_t &o) const
    {
        const uint64_t h = a.h * ord_pow(MULT, b.q) + b.h, q = a.q + b.q;
        o.h = h; o.q = q; // (after both reads: o may alias an operand)
    }
};
// keyed-stateful: the tuple leaves with the running hash of its key and with the state's count stamped above its seq
struct SMap {
    __host__ __device__ void operator()(tuple_t &t, state_t &st) const
    {
        st.count++; st.hash = st.hash * MULT + ord_mix(t.value, t.key);
        t.value = st.hash + st.last; st.last = t.seq; t.seq |= st.count << 20;
    }
};
struct SFilt {
    __host__ __device__ bool operator()(tuple_t &t, state_t &st) const
    {
        st.count++; st.hash = st.hash * MULT + t.value; st.last = t.seq;
        t.value = st.hash; t.seq |= st.count << 42;
        return st.count % 4 != 0;
    }
};
struct Red { // the same hash on tuples: (value, seq) as (h, q)
    __host__ __device__ tuple_t operator()(const tuple_t &a, const tuple_t &b) const
    {
        tuple_t r = a;
        r.value = a.value * ord_pow(MULT, b.seq) + b.value; r.seq = a.seq + b.seq;
        return r;
    }
};

// ---- the stream ------------------------------------------------------------------------------------------------------------------------
static uint64_t mix64(uint64_t x) { x ^= x >> 31; x *= 0x7fb5d329728ea185ull; x ^= x >> 27; x *= 0x81dadef4bc2dd44dull; x ^= x >> 33; return x; }
static std::vector<tuple_t> stream;   // hashed 64-bit keys, rank r with probability ~ 1 / r
static std::vector<uint64_t> tb_ts, tb_wm; // time-based runs: timestamp and watermark of every tuple
static void make_stream()
{
    stream.resize(N); tb_ts.resize(N); tb_wm.resize(N);
    uint64_t gap = 0;
    for (uint64_t i = 0; i < N; i++) {
        const double u = static_cast<double>(mix64(i * 2 + 1) >> 11) / 9007199254740992.0;
        const uint64_t rank = std::min<uint64_t>(NKEYS - 1, static_cast<uint64_t>(std::pow(static_cast<double>(NKEYS), u)) - 1);
        stream[i] = tuple_t{mix64(0xABCDull + rank) | (1ull << 40), i, mix64(i * 2 + 2)};
        if (i % 90000 == 89999) gap += 3000; // idle: the watermark jumps over several groups of windows
        tb_wm[i] = i / 20 + gap;
        tb_ts[i] = tb_wm[i] + mix64(i + 77) % 100; // out of order, within the lateness
    }
}

static void write_file(const std::string &path, const void *p, size_t bytes)
{
    FILE *f = std::fopen(path.c_str(), "wb");
    if (!f || std::fwrite(p, 1, bytes, f) != bytes) { std::printf("FAILED writing %s\n", path.c_str()); std::exit(1); }
    std::fclose(f);
}
template <class R> static void write_rows(const std::string &dir, const std::string &name, const std::vector<R> &rows)
{
    write_file(dir + "/" + name + ".bin", rows.data(), rows.size() * sizeof(R));
}
[[noreturn]] static void fail(const std::string &msg) { std::printf("FAILED %s\n", msg.c_str()); std::exit(1); }

// ---- sources and sinks -----------------------------------------------------------------------------------------------------------------
static std::atomic<bool> g_source_done{false};
// batches pushed | batches the Sinks have finished (their watermark probe; a device-side source numbers its batches) | the most between the two
static std::atomic<uint64_t> g_pushed{0}, g_finished{0}, g_max_depth{0};
static bool g_numbered = false;
static void note_depth()
{
    const uint64_t p = g_pushed.load(), f = g_numbered ? g_finished.load() : 0, d = p > f ? p - f : 0;
    uint64_t cur = g_max_depth.load();
    while (cur < d && !g_max_depth.compare_exchange_weak(cur, d)) { }
}
enum class Feed { PLAIN, SMALL_KEYS, TB };
struct Source_Functor {
    Feed feed;
    void operator()(Source_Shipper<tuple_t> &sh)
    {
        for (uint64_t i = 0; i < N; i++) {
            tuple_t t = stream[i];
            if (feed == Feed::SMALL_KEYS) t.key %= 65521;
            if (feed == Feed::TB) { sh.setNextWatermark(tb_wm[i]); sh.pushWithTimestamp(t, tb_ts[i]); }
            else { sh.setNextWatermark(i); sh.pushWithTimestamp(t, i); }
            if (i % BATCH == BATCH - 1) g_pushed.fetch_add(1);
        }
        g_source_done.store(true, std::memory_order_release);
    }
};
// batches of `bs` tuples that already lie in device memory; the watermark of batch i is i + 1
struct SourceGPU_Functor {
    tuple_t *d_tuples; uint64_t *d_ts; uint64_t bs, nbatches;
    void operator()(SourceGPU_Shipper<tuple_t> &sh)
    {
        for (uint64_t i = 0; i < nbatches; i++) { sh.pushBatch(d_tuples + i * bs, d_ts + i * bs, bs, i + 1); g_pushed.fetch_add(1); note_depth(); }
        g_source_done.store(true, std::memory_order_release);
    }
};
// Every replica of a Sink appends to its own rows and hands them over at the end of the stream. A slow Sink blocks in its first call:
// `until_source_done` until the source has pushed its last batch and 200 ms more, otherwise for `first_sleep_ms`.
template <class R> struct Collected { static std::mutex mu; static std::vector<R> rows; };
template <class R> std::mutex Collected<R>::mu;
template <class R> std::vector<R> Collected<R>::rows;
template <class R> struct Sink_Functor {
    bool until_source_done = false; int first_sleep_ms = 0;
    bool first = true; std::vector<R> mine;
    void operator()(std::optional<R> &r)
    {
        if (first) {
            first = false;
            if (until_source_done) { while (!g_source_done.load(std::memory_order_acquire)) std::this_thread::sleep_for(std::chrono::milliseconds(1)); first_sleep_ms = 200; }
            if (r && first_sleep_ms) { note_depth(); std::this_thread::sleep_for(std::chrono::milliseconds(first_sleep_ms)); note_depth(); }
        }
        if (r) mine.push_back(*r);
        else { std::lock_guard<std::mutex> lock(Collected<R>::mu); Collected<R>::rows.insert(Collected<R>::rows.end(), mine.begin(), mine.end()); }
    }
};
template <class R> static auto sink(bool until_done = false, int sleep_ms = 0, size_t par = 1)
{
    Sink_Functor<R> f; f.until_source_done = until_done; f.first_sleep_ms = sleep_ms;
    return Sink_Builder(f).withName("sink").withParallelism(par).withWatermarkProbe(&g_finished).build();
}
template <class R> static void begin_run(bool numbered = false) { g_numbered = numbered; Collected<R>::rows.clear(); g_source_done = false; g_pushed = 0; g_finished = 0; g_max_depth = 0; }
template <class R> static void end_run(PipeGraph &graph, const std::string &dir, const std::string &name, bool may_be_empty = false)
{
    graph.run();
    write_rows(dir, name, Collected<R>::rows);
    std::printf("run %s: %zu rows, %zu threads, %llu batches ahead of a slow Sink at most\n", name.c_str(), Collected<R>::rows.size(),
                graph.getNumThreads(), static_cast<unsigned long long>(g_max_depth.load()));
    if (Collected<R>::rows.empty() && !may_be_empty) fail("run " + name + ": no rows");
}
static void expect_graph(MultiPipe &mp, const std::string &run, const std::vector<std::string> &names, size_t threads)
{
    std::string got, exp;
    for (auto &n : mp.getOperatorNames()) got += n + " ";
    for (auto &n : names) exp += n + " ";
    if (got != exp || mp.getNumThreads() != threads)
        fail("run " + run + ": operators [" + got + "] on " + std::to_string(mp.getNumThreads()) + " threads, expected [" + exp + "] on " + std::to_string(threads));
}

static auto cb_windows(size_t K)
{
    return Ffat_WindowsGPU_Builder(Lift(), Comb()).withName("windows").withKeyBy(KeyF()).withCBWindows(WIN, SLIDE).withNumWinPerBatch(NWB)
        .withMaxKeys(MAXKEYS).withMaxBatchesPerCall(K).build();
}
static auto tb_windows()
{
    return Ffat_WindowsGPU_Builder(Lift(), Comb()).withName("windows").withKeyBy(KeyF())
        .withTBWindows(std::chrono::microseconds(TB_WIN), std::chrono::microseconds(TB_SLIDE)).withLateness(std::chrono::microseconds(TB_LATE))
        .withNumWinPerBatch(TB_NWB).withMaxKeys(MAXKEYS).build();
}
static auto source(Feed feed) { return Source_Builder(Source_Functor{feed}).withName("source").withOutputBatchSize(BATCH).build(); }
static auto map_a() { return MapGPU_Builder(MapA()).withName("map_a").build(); }
static auto filt_a() { return FilterGPU_Builder(FiltA()).withName("filt_a").build(); }
static auto map_b() { return MapGPU_Builder(MapB()).withName("map_b").build(); }
static auto filt_b() { return FilterGPU_Builder(FiltB()).withName("filt_b").build(); }

// Map -> Filter (-> Map -> Filter) -> count-based windows; thunks: one chain per statement, typed: one fluent expression. On both
// routes the run is part of the window operator's pass: source, windows and Sink are the only threads.
static void run_cb(const std::string &dir, const std::string &name, size_t K, bool typed, bool two)
{
    begin_run<result_t>();
    PipeGraph graph(name, Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(source(Feed::PLAIN));
    if (typed && two) mp.chain(map_a()).chain(filt_a()).chain(map_b()).chain(filt_b()).add(cb_windows(K));
    else if (typed) mp.chain(map_a()).chain(filt_a()).add(cb_windows(K));
    else {
        mp.chain(map_a());
        mp.chain(filt_a());
        if (two) { mp.chain(map_b()); mp.chain(filt_b()); }
        mp.add(cb_windows(K));
    }
    mp.chain_sink(sink<result_t>());
    if (two) expect_graph(mp, name, {"source", "map_a", "filt_a", "map_b", "filt_b", "windows", "sink"}, 3);
    else expect_graph(mp, name, {"source", "map_a", "filt_a", "windows", "sink"}, 3);
    end_run<result_t>(graph, dir, name);
}
static void run_chain_sink(const std::string &dir)
{
    begin_run<tuple_t>();
    PipeGraph graph("chain_sink", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(source(Feed::PLAIN));
    mp.chain(map_a());
    mp.chain(filt_a());
    mp.chain_sink(sink<tuple_t>());
    expect_graph(mp, "chain_sink", {"source", "map_a", "filt_a", "sink"}, 3); // (the run is one replica)
    end_run<tuple_t>(graph, dir, "chain_sink");
}
static void run_stateful(const std::string &dir, const std::string &name, size_t par)
{
    begin_run<tuple_t>();
    PipeGraph graph(name, Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(source(Feed::PLAIN));
    mp.chain(map_a());
    mp.chain(filt_a());
    mp.chain(MapGPU_Builder(SMap()).withName("smap").withKeyBy(KeyF()).withParallelism(par).withMaxKeys(64).withKeyGrowth().build());
    mp.chain(FilterGPU_Builder(SFilt()).withName("sfilt").withKeyBy(KeyF()).withParallelism(par).withMaxKeys(512).build());
    mp.chain_sink(sink<tuple_t>());
    expect_graph(mp, name, {"source", "map_a", "filt_a", "smap", "sfilt", "sink"}, 3 + 2 * par);
    end_run<tuple_t>(graph, dir, name);
}
static void run_reduce(const std::string &dir, const std::string &name, uint32_t bits)
{
    begin_run<tuple_t>();
    PipeGraph graph(name, Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(source(Feed::SMALL_KEYS));
    if (bits != 64) mp.chain(ReduceGPU_Builder(Red()).withName("reduce").withKeyBy(KeyF()).withKeyBits(bits).build());
    else mp.chain(ReduceGPU_Builder(Red()).withName("reduce").withKeyBy(KeyF()).build());
    mp.chain_sink(sink<tuple_t>());
    end_run<tuple_t>(graph, dir, name);
}
static void run_tb(const std::string &dir, const std::string &name, bool slow)
{
    begin_run<result_t>();
    PipeGraph graph(name, Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(source(Feed::TB));
    mp.add(tb_windows());
    mp.chain_sink(sink<result_t>(slow));
    end_run<result_t>(graph, dir, name);
}
// the first `nbatches * bs` tuples of the stream, resident on the device
struct DeviceStream {
    tuple_t *d_tuples = nullptr; uint64_t *d_ts = nullptr;
    explicit DeviceStream(uint64_t n)
    {
        std::vector<uint64_t> ts(n);
        for (uint64_t i = 0; i < n; i++) ts[i] = i;
        gpuErrChk(cudaMalloc(&d_tuples, n * sizeof(tuple_t))); gpuErrChk(cudaMalloc(&d_ts, n * sizeof(uint64_t)));
        gpuErrChk(cudaMemcpy(d_tuples, stream.data(), n * sizeof(tuple_t), cudaMemcpyHostToDevice));
        gpuErrChk(cudaMemcpy(d_ts, ts.data(), n * sizeof(uint64_t), cudaMemcpyHostToDevice));
    }
    ~DeviceStream() { cudaFree(d_tuples); cudaFree(d_ts); }
};
static void run_slow_sink_cb(const std::string &dir)
{
    begin_run<result_t>(true);
    DeviceStream ds(SLOW_BATCH * SLOW_BATCHES);
    {
        PipeGraph graph("slow_sink_cb", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
        MultiPipe &mp = graph.add_source(SourceGPU_Builder(SourceGPU_Functor{ds.d_tuples, ds.d_ts, SLOW_BATCH, SLOW_BATCHES}).withName("source").build());
        mp.chain(FilterGPU_Builder(FiltB()).withName("filt_b").build());
        mp.add(cb_windows(1));
        mp.chain_sink(sink<result_t>(true));
        end_run<result_t>(graph, dir, "slow_sink_cb");
    }
}
static void run_slow_sinks_filter(const std::string &dir)
{
    begin_run<tuple_t>(true);
    DeviceStream ds(SINKS_BATCH * SINKS_BATCHES);
    {
        PipeGraph graph("slow_sinks_filter", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
        MultiPipe &mp = graph.add_source(SourceGPU_Builder(SourceGPU_Functor{ds.d_tuples, ds.d_ts, SINKS_BATCH, SINKS_BATCHES}).withName("source").build());
        mp.chain(FilterGPU_Builder(FiltB()).withName("filt_b").build());
        mp.chain_sink(sink<tuple_t>(false, 400, 3)); // (5000 batches do not fit the queues in front of the Sinks: they are slow for a fixed time)
        end_run<tuple_t>(graph, dir, "slow_sinks_filter");
    }
}

// ---- the functors on the host ------------------------------------------------------------------------------------------------------------
static void host_check(const std::string &dir)
{
    std::vector<tuple_t> chain, chain2, st, red; std::vector<result_t> lifted, folded;
    std::unordered_map<uint64_t, state_t> ms, fs;
    result_t acc;
    for (uint64_t i = 0; i < N; i++) {
        tuple_t t = stream[i];
        result_t r; Lift()(t, r); lifted.push_back(r);
        if (i < 5000) { Comb()(acc, r, acc); folded.push_back(acc); }
        MapA()(t);
        if (!FiltA()(t)) continue;
        chain.push_back(t);
        tuple_t s = t;
        SMap()(s, ms[s.key]);
        if (SFilt()(s, fs[s.key])) st.push_back(s);
        MapB()(t);
        if (FiltB()(t)) chain2.push_back(t);
    }
    for (uint64_t b = 0; b < N; b += BATCH) {
        std::map<uint64_t, tuple_t> keys; // ascending; the fold of a key's tuples in arrival order
        for (uint64_t i = b; i < std::min(N, b + BATCH); i++) {
            tuple_t t = stream[i]; t.key %= 65521;
            auto it = keys.find(t.key);
            if (it == keys.end()) keys[t.key] = t; else it->second = Red()(it->second, t);
        }
        for (auto &kv : keys) red.push_back(kv.second);
    }
    write_rows(dir, "host_chain_sink", chain); write_rows(dir, "host_chain2", chain2); write_rows(dir, "host_stateful", st);
    write_rows(dir, "host_reduce", red); write_rows(dir, "host_lift", lifted); write_rows(dir, "host_fold", folded);
    std::printf("HOST_OK\n");
}

int main(int argc, char **argv)
{
    const bool host = argc > 1 && std::strcmp(argv[1], "--host-check") == 0;
    if (argc < (host ? 3 : 2)) { std::printf("usage: %s [--host-check] OUTPUT_DIR [run ...]\n", argv[0]); return 2; }
    const std::string dir = argv[host ? 2 : 1];
    make_stream();
    write_rows(dir, "stream", stream); write_rows(dir, "tb_ts", tb_ts); write_rows(dir, "tb_wm", tb_wm);
    if (host) { host_check(dir); return 0; }
    auto wanted = [&](const char *run) { if (argc == 2) return true; for (int i = 2; i < argc; i++) if (std::strcmp(argv[i], run) == 0) return true; return false; };
    std::printf("WF_MAX_BATCHES_PER_CALL %d\n", static_cast<int>(WF_MAX_BATCHES_PER_CALL));
    for (size_t K : {size_t(1), size_t(7), size_t(128)}) if (wanted("cb")) run_cb(dir, "cb_thunk_K" + std::to_string(K), K, false, false);
    if (wanted("cb")) { run_cb(dir, "cb_typed", 128, true, false); run_cb(dir, "cb_mmff_thunk", 128, false, true); run_cb(dir, "cb_mmff_typed", 128, true, true); }
    if (wanted("chain_sink")) run_chain_sink(dir);
    if (wanted("stateful")) { run_stateful(dir, "stateful_p1", 1); run_stateful(dir, "stateful_p2", 2); }
    if (wanted("reduce")) { run_reduce(dir, "reduce_bits16", 16); run_reduce(dir, "reduce_bits64", 64); }
    if (wanted("tb")) run_tb(dir, "tb_ooo", false);
    if (wanted("slow")) { run_slow_sink_cb(dir); run_tb(dir, "slow_sink_tb", true); run_slow_sinks_filter(dir); }
    std::printf("EXACT_OK\n");
    return 0;
}
