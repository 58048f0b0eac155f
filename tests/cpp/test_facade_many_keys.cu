// Application-level test of operators over more than 65536 keys (include/wf/windflow_gpu.hpp): Source -> keyed-stateful Map_GPU
// withMaxKeys(1 << 18) (the full-sort path from the start) -> time-based Ffat_Windows_GPU withMaxKeys(16).withKeyGrowth() (grows past
// 65536 keys) -> Sink, over 200 000 keys. The Sink checks every key's windows against sums computed on the host. Prints MANY_KEYS_OK on
// success.
#include <cstdio>
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

constexpr size_t KEYS = 200000, LEN = 12, BATCH = 10000;

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
struct state_t { int64_t counter; __host__ __device__ state_t(): counter(0) {} };
struct MapKB { __host__ __device__ void operator()(tuple_t &t, state_t &s) const { s.counter++; t.value += s.counter; } }; // i-th tuple: 2 i
struct Lift { __host__ __device__ void operator()(const tuple_t &t, result_t &r) const { r.value = t.value; } };
struct Comb { __host__ __device__ void operator()(const result_t &a, const result_t &b, result_t &o) const { o.value = a.value + b.value; } };

static std::vector<long> win_sum(KEYS), win_cnt(KEYS); static bool order_ok = true, unknown_key = false;
struct WinSink { // the windows of a key arrive with consecutive ids 0, 1, 2, ...
    void operator()(std::optional<result_t> &r)
    {
        if (!r) return;
        if (r->key >= KEYS) { unknown_key = true; return; }
        if (r->id != static_cast<uint64_t>(win_cnt[r->key])) order_ok = false;
        win_sum[r->key] += r->value; win_cnt[r->key]++;
    }
};

int main()
{
    const uint64_t win = 4 * KEYS, slide = 2 * KEYS; // microseconds; a key sees one tuple every KEYS us
    PipeGraph graph("many_keys", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor()).withName("source").withOutputBatchSize(BATCH).build());
    mp.chain(MapGPU_Builder(MapKB()).withName("map_kb").withKeyBy(Key()).withMaxKeys(1u << 18).build())
      .add(Ffat_WindowsGPU_Builder(Lift(), Comb()).withName("ffat_tb").withKeyBy(Key())
               .withTBWindows(std::chrono::microseconds(win), std::chrono::microseconds(slide)).withNumWinPerBatch(2).withMaxKeys(16).withKeyGrowth().build());
    mp.chain_sink(Sink_Builder(WinSink()).withName("sink").build());
    graph.run();
    if (unknown_key || !order_ok) { std::printf("FAILED: unknown key or window ids out of order\n"); return 1; }
    long fired = 0;
    for (size_t k = 0; k < KEYS; k++) { // window g of key k = the sum of 2 i over its tuples with ts in [g * slide, g * slide + win)
        long exp = 0;
        for (long g = 0; g < win_cnt[k]; g++)
            for (size_t i = 1; i <= LEN; i++) { const uint64_t ts = (i - 1) * KEYS + k; if (ts >= g * slide && ts < g * slide + win) exp += 2 * static_cast<long>(i); }
        if (exp != win_sum[k]) { std::printf("FAILED windows of key %zu: got %ld expected %ld over %ld windows\n", k, win_sum[k], exp, win_cnt[k]); return 1; }
        fired += win_cnt[k];
    }
    // the stream spans LEN * KEYS us: every key fires all but its last few groups of 2 windows
    if (fired < static_cast<long>(KEYS) * (LEN / 2 - 3) || fired % 2 != 0) { std::printf("FAILED: %ld windows fired\n", fired); return 1; }
    std::printf("keyed-stateful map -> ffat tb windows over %zu keys OK (%ld windows)\n", KEYS, fired);
    std::printf("MANY_KEYS_OK\n");
    return 0;
}
