// Application-level test of key tables that grow (withKeyGrowth() in include/wf/windflow_gpu.hpp). Thousands of keys go through
// operators built withMaxKeys(16).withKeyGrowth(): Map -> Filter -> Ffat_Windows_GPU with count-based and with time-based windows, and a
// keyed-stateful Map_GPU. The Sinks check closed-form sums per key. Prints GROWTH_OK on success.
// With the argument "fixed" it runs the count-based graph without withKeyGrowth(): the program must stop with the capacity message.
#include <cstdio>
#include <cstring>
#include <optional>
#include <vector>
#include <wf/windflow_gpu.hpp>

using namespace wf;

struct tuple_t {
    uint64_t key; int64_t value;
    __host__ __device__ tuple_t(): key(0), value(0) {}
};
struct result_t {
    uint64_t key; uint64_t id; int64_t value;
    __host__ __device__ result_t(): key(0), id(0), value(0) {}
    __host__ __device__ result_t(uint64_t k, uint64_t i): key(k), id(i), value(0) {}
};

constexpr size_t KEYS = 3000, LEN = 120, BATCH = 1000;

struct Source_Functor { // for i = 1 .. LEN, one tuple of value i for every key: key k's i-th tuple has ts (i - 1) * KEYS + k
    void operator()(Source_Shipper<tuple_t> &shipper)
    {
        uint64_t ts = 0;
        for (size_t i = 1; i <= LEN; i++)
            for (size_t k = 0; k < KEYS; k++) {
                tuple_t t; t.key = k; t.value = static_cast<int64_t>(i);
                shipper.pushWithTimestamp(t, ts); shipper.setNextWatermark(ts); ts++;
            }
    }
};
struct Key { __host__ __device__ uint64_t operator()(const tuple_t &t) const { return t.key; } };
struct Double { __host__ __device__ void operator()(tuple_t &t) const { t.value *= 2; } };
struct Positive { __host__ __device__ bool operator()(tuple_t &t) const { return t.value > 0; } };
struct Lift { __host__ __device__ void operator()(const tuple_t &t, result_t &r) const { r.value = t.value; } };
struct Comb { __host__ __device__ void operator()(const result_t &a, const result_t &b, result_t &o) const { o.value = a.value + b.value; } };
struct state_t { int64_t counter; __host__ __device__ state_t(): counter(0) {} };
struct MapKB { __host__ __device__ void operator()(tuple_t &t, state_t &s) const { s.counter++; t.value += s.counter; } };

static long win_sum[KEYS], win_cnt[KEYS]; static bool order_ok = true, unknown_key = false;
static void reset() { for (size_t k = 0; k < KEYS; k++) win_sum[k] = win_cnt[k] = 0; order_ok = true; unknown_key = false; }
struct WinSink { // the windows of a key arrive with consecutive ids 0, 1, 2, ...
    void operator()(std::optional<result_t> &r)
    {
        if (!r) return;
        if (r->key >= KEYS) { unknown_key = true; return; }
        if (r->id != static_cast<uint64_t>(win_cnt[r->key])) order_ok = false;
        win_sum[r->key] += r->value; win_cnt[r->key]++;
    }
};
struct TupleSink { void operator()(std::optional<tuple_t> &t) { if (!t) return; if (t->key >= KEYS) { unknown_key = true; return; } win_sum[t->key] += t->value; win_cnt[t->key]++; } };

static void fail(const char *what) { std::printf("FAILED %s\n", what); std::exit(1); }

static void run_cb(bool grow)
{
    const uint64_t win = 16, slide = 4, nwb = 3, B = (nwb - 1) * slide + win;
    reset();
    PipeGraph graph("growth_cb", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor()).withName("source").withOutputBatchSize(BATCH).build());
    auto fb0 = Ffat_WindowsGPU_Builder(Lift(), Comb()).withName("ffat").withMaxKeys(16);
    if (grow) fb0.withKeyGrowth(); // (before withKeyBy: the builder carries it over)
    auto fb = fb0.withKeyBy(Key()).withCBWindows(win, slide).withNumWinPerBatch(nwb);
    mp.chain(MapGPU_Builder(Double()).withName("map").build())
      .chain(FilterGPU_Builder(Positive()).withName("filter").build())
      .add(fb.build());
    mp.chain_sink(Sink_Builder(WinSink()).withName("sink").build());
    graph.run();
    if (unknown_key || !order_ok) fail("cb windows: unknown key or window ids out of order");
    // every key: items 2, 4, ..., 2 LEN; groups of nwb windows fire after B items, then every slide * nwb
    const uint64_t groups = LEN >= B ? 1 + (LEN - B) / (slide * nwb) : 0;
    long exp = 0;
    for (uint64_t w = 0; w < groups * nwb; w++) for (uint64_t j = w * slide; j < w * slide + win; j++) exp += 2 * static_cast<long>(j + 1);
    for (size_t k = 0; k < KEYS; k++)
        if (win_sum[k] != exp || win_cnt[k] != static_cast<long>(groups * nwb)) {
            std::printf("FAILED cb windows of key %zu: sum %ld count %ld, expected %ld over %lu\n", k, win_sum[k], win_cnt[k], exp, static_cast<unsigned long>(groups * nwb));
            std::exit(1);
        }
    std::printf("map -> filter -> ffat cb windows OK (%lu windows per key)\n", static_cast<unsigned long>(groups * nwb));
}

static void run_tb()
{
    const uint64_t win = 4 * KEYS, slide = 2 * KEYS; // microseconds; a key sees one tuple every KEYS us
    reset();
    PipeGraph graph("growth_tb", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor()).withName("source").withOutputBatchSize(BATCH).build());
    mp.chain(MapGPU_Builder(Double()).withName("map").build())
      .chain(FilterGPU_Builder(Positive()).withName("filter").build())
      .add(Ffat_WindowsGPU_Builder(Lift(), Comb()).withName("ffat_tb").withKeyBy(Key())
               .withTBWindows(std::chrono::microseconds(win), std::chrono::microseconds(slide)).withNumWinPerBatch(2).withMaxKeys(16).withKeyGrowth().build());
    mp.chain_sink(Sink_Builder(WinSink()).withName("sink").build());
    graph.run();
    if (unknown_key || !order_ok) fail("tb windows: unknown key or window ids out of order");
    long fired = 0;
    for (size_t k = 0; k < KEYS; k++) { // window g of key k = the sum of its values with ts in [g * slide, g * slide + win)
        long exp = 0;
        for (long g = 0; g < win_cnt[k]; g++)
            for (size_t i = 1; i <= LEN; i++) { const uint64_t ts = (i - 1) * KEYS + k; if (ts >= g * slide && ts < g * slide + win) exp += 2 * static_cast<long>(i); }
        if (exp != win_sum[k]) { std::printf("FAILED tb windows of key %zu: got %ld expected %ld over %ld windows\n", k, win_sum[k], exp, win_cnt[k]); std::exit(1); }
        fired += win_cnt[k];
    }
    // the stream spans LEN * KEYS us: every key fires all but its last few groups of 2 windows (about LEN / 2 windows)
    if (fired < static_cast<long>(KEYS) * (LEN / 2 - 6) || fired % 2 != 0) { std::printf("FAILED tb windows: %ld fired\n", fired); std::exit(1); }
    std::printf("map -> filter -> ffat tb windows OK (%ld windows)\n", fired);
}

static void run_stateful()
{
    reset();
    PipeGraph graph("growth_stateful", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor()).withName("source").withOutputBatchSize(BATCH).build());
    mp.chain(MapGPU_Builder(MapKB()).withName("map_kb").withKeyBy(Key()).withMaxKeys(16).withKeyGrowth().build());
    mp.chain_sink(Sink_Builder(TupleSink()).withName("sink").build());
    graph.run();
    if (unknown_key) fail("stateful map: unknown key");
    const long exp = static_cast<long>(LEN * (LEN + 1)); // sum over i of (i + counter i)
    for (size_t k = 0; k < KEYS; k++)
        if (win_sum[k] != exp || win_cnt[k] != static_cast<long>(LEN)) { std::printf("FAILED stateful map of key %zu: %ld over %ld\n", k, win_sum[k], win_cnt[k]); std::exit(1); }
    std::printf("keyed-stateful map OK\n");
}

int main(int argc, char **argv)
{
    if (argc > 1 && std::strcmp(argv[1], "fixed") == 0) { run_cb(false); std::printf("FIXED_DID_NOT_STOP\n"); return 0; }
    run_cb(true);
    run_tb();
    run_stateful();
    std::printf("GROWTH_OK\n");
    return 0;
}
