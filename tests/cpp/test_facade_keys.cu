// Application-level test of key types other than integers in the builder API (include/wf/windflow_gpu.hpp): the key type of an
// operator is what its key extractor returns. Graphs keyed by a double (with 1.25 / 1.75, a negative key, and -0.0 / +0.0, which
// compare equal and are one key), by an 8-byte struct flow_t { src, dst } and by a 16-byte struct flow16_t run count-based
// Ffat_Windows_GPU, keyed Reduce_GPU and keyed-stateful Map_GPU; the Sinks check closed-form sums per key. It also checks that
// wfb_mg_create refuses a double key even when the lifted records carry their key. Prints KEYS_OK on success.
#include <cstdio>
#include <cstdlib>
#include <optional>
#include <vector>
#include <wf/windflow_gpu.hpp>
#include "../../windflow_b200/csrc/wfb_programs.cuh"

using namespace wf;

struct flow_t { uint32_t src, dst; };
struct flow16_t { uint32_t src, dst; uint32_t ports, proto; };
__host__ __device__ inline bool operator==(const flow_t &a, const flow_t &b) { return a.src == b.src && a.dst == b.dst; }
__host__ __device__ inline bool operator==(const flow16_t &a, const flow16_t &b) { return a.src == b.src && a.dst == b.dst && a.ports == b.ports && a.proto == b.proto; }

struct tuple_t {
    double dkey; flow_t flow; flow16_t flow16; int64_t value;
    __host__ __device__ tuple_t(): dkey(0), flow{0, 0}, flow16{0, 0, 0, 0}, value(0) {}
};
template <class K> struct result_t {
    K key; uint64_t id; int64_t value;
    __host__ __device__ result_t(): key{}, id(0), value(0) {}
    __host__ __device__ result_t(K k, uint64_t i): key(k), id(i), value(0) {}
};

// the key table of every graph: key index k of the source -> the key value; `group` maps k to its distinct key
static const double DKEYS[] = {1.25, 1.75, -1.25, 0.0, -0.0};
static const int DGROUP[] = {0, 1, 2, 3, 3};
static const flow_t FKEYS[] = {{1, 2}, {2, 1}, {1, 3}, {0xffffffffu, 0}};
static const flow16_t F16KEYS[] = {{1, 2, 80, 6}, {1, 2, 80, 17}, {2, 1, 80, 6}}; // equal low words, different high words
constexpr size_t LEN = 2000, BATCH = 700, MAXG = 8;

struct Source_Functor { // for i = 1 .. LEN, one tuple of value i for every key index
    size_t nkeys;
    void operator()(Source_Shipper<tuple_t> &shipper)
    {
        uint64_t ts = 0;
        for (size_t i = 1; i <= LEN; i++)
            for (size_t k = 0; k < nkeys; k++) {
                tuple_t t;
                t.dkey = DKEYS[k % 5]; t.flow = FKEYS[k % 4]; t.flow16 = F16KEYS[k % 3]; t.value = static_cast<int64_t>(i);
                shipper.pushWithTimestamp(t, ts); shipper.setNextWatermark(ts); ts++;
            }
    }
};
struct DKey { __host__ __device__ double operator()(const tuple_t &t) const { return t.dkey; } };
struct FKey { __host__ __device__ flow_t operator()(const tuple_t &t) const { return t.flow; } };
struct F16Key { __host__ __device__ flow16_t operator()(const tuple_t &t) const { return t.flow16; } };
template <class K> struct Lift { __host__ __device__ void operator()(const tuple_t &t, result_t<K> &r) const { r.value = t.value; } };
template <class K> struct Comb { __host__ __device__ void operator()(const result_t<K> &a, const result_t<K> &b, result_t<K> &o) const { o.value = a.value + b.value; } };
struct Reduce { __host__ __device__ tuple_t operator()(const tuple_t &a, const tuple_t &b) const { tuple_t r = a; r.value = a.value + b.value; return r; } };
struct state_t { int64_t counter; __host__ __device__ state_t(): counter(0) {} };
struct MapKB { __host__ __device__ void operator()(tuple_t &t, state_t &s) const { s.counter++; t.value += s.counter; } };

static long got_sum[MAXG], got_cnt[MAXG]; static bool unknown_key = false;
template <class K> static int group_of(const K &key, const K *keys, const int *group, size_t n)
{
    for (size_t k = 0; k < n; k++) if (key == keys[k]) return group ? group[k] : static_cast<int>(k);
    return -1;
}
static void add(int g, long v) { if (g < 0) { unknown_key = true; return; } got_sum[g] += v; got_cnt[g]++; }
static void reset() { for (size_t g = 0; g < MAXG; g++) got_sum[g] = got_cnt[g] = 0; unknown_key = false; }

template <class K, size_t N> struct WinSink {
    const K *keys; const int *group;
    void operator()(std::optional<result_t<K>> &r) { if (r) add(group_of(r->key, keys, group, N), r->value); }
};
struct DTupleSink { void operator()(std::optional<tuple_t> &t) { if (t) add(group_of(t->dkey, DKEYS, DGROUP, 5), t->value); } };
struct FTupleSink { void operator()(std::optional<tuple_t> &t) { if (t) add(group_of(t->flow, FKEYS, nullptr, 4), t->value); } };
struct F16TupleSink { void operator()(std::optional<tuple_t> &t) { if (t) add(group_of(t->flow16, F16KEYS, nullptr, 3), t->value); } };

// the values of one distinct key in arrival order: `mult` source key indexes share it
static std::vector<long> sequence(size_t mult)
{
    std::vector<long> s;
    for (size_t i = 1; i <= LEN; i++) for (size_t m = 0; m < mult; m++) s.push_back(static_cast<long>(i));
    return s;
}
enum Kind { WINDOWS, REDUCE, STATEFUL };
static const uint64_t WIN = 64, SLIDE = 16, NWB = 3;
static void expect(const char *what, size_t g, const std::vector<long> &s, Kind kind)
{
    long sum = 0, cnt = 0;
    if (kind == WINDOWS) { // count-based windows fire in groups of NWB: first after (NWB-1)*SLIDE+WIN items, then every SLIDE*NWB
        const uint64_t B = (NWB - 1) * SLIDE + WIN, c = s.size(), groups = c >= B ? 1 + (c - B) / (SLIDE * NWB) : 0;
        for (uint64_t w = 0; w < groups * NWB; w++) { for (uint64_t j = w * SLIDE; j < w * SLIDE + WIN; j++) sum += s[j]; cnt++; }
    } else if (kind == REDUCE) { for (long v : s) sum += v; cnt = -1; } // (outputs per batch: not checked)
    else { for (size_t j = 0; j < s.size(); j++) sum += s[j] + static_cast<long>(j + 1); cnt = static_cast<long>(s.size()); }
    if (unknown_key) { std::printf("FAILED %s: a result carries a key the source never produced\n", what); std::exit(1); }
    if (got_sum[g] != sum || (cnt >= 0 && got_cnt[g] != cnt)) {
        std::printf("FAILED %s, key %zu: sum %ld count %ld, expected sum %ld count %ld\n", what, g, got_sum[g], got_cnt[g], sum, cnt);
        std::exit(1);
    }
    std::printf("%s key %zu OK (sum %ld)\n", what, g, sum);
}

template <class KeyF, class K, class TSink, size_t N>
static void run_all(const char *name, size_t nkeys, KeyF kf, const K *keys, const int *group, size_t ngroups, const std::vector<size_t> &mult)
{
    { // Ffat_Windows_GPU, count-based
        reset();
        PipeGraph graph(std::string(name) + "_win", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
        MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor{nkeys}).withName("source").withOutputBatchSize(BATCH).build());
        mp.add(Ffat_WindowsGPU_Builder(Lift<K>(), Comb<K>()).withName("ffat").withKeyBy(kf).withCBWindows(WIN, SLIDE).withNumWinPerBatch(NWB)
                   .withMaxKeys(16).build());
        mp.chain_sink(Sink_Builder(WinSink<K, N>{keys, group}).withName("sink").build());
        graph.run();
        for (size_t g = 0; g < ngroups; g++) expect((std::string(name) + " ffat cb windows").c_str(), g, sequence(mult[g]), WINDOWS);
    }
    { // Reduce_GPU, keyed
        reset();
        PipeGraph graph(std::string(name) + "_reduce", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
        MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor{nkeys}).withName("source").withOutputBatchSize(BATCH).build());
        mp.chain(ReduceGPU_Builder(Reduce()).withName("reduce").withKeyBy(kf).build());
        mp.chain_sink(Sink_Builder(TSink()).withName("sink").build());
        graph.run();
        for (size_t g = 0; g < ngroups; g++) expect((std::string(name) + " reduce_by_key").c_str(), g, sequence(mult[g]), REDUCE);
    }
    { // Map_GPU, keyed-stateful
        reset();
        PipeGraph graph(std::string(name) + "_stateful", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
        MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor{nkeys}).withName("source").withOutputBatchSize(BATCH).build());
        mp.chain(MapGPU_Builder(MapKB()).withName("map_kb").withKeyBy(kf).withMaxKeys(64).build());
        mp.chain_sink(Sink_Builder(TSink()).withName("sink").build());
        graph.run();
        for (size_t g = 0; g < ngroups; g++) expect((std::string(name) + " stateful map").c_str(), g, sequence(mult[g]), STATEFUL);
    }
}

// the double-key built-in program with a result_key: its lifted records carry their key, so only the key type keeps it off the
// multi-GPU path (shards are key % nranks)
struct FKeyCarried : wfb::ProgTuple64FKey {
    __host__ __device__ static key_t result_key(const result_t &r, const params_t &) { return r.key; }
};

int main()
{
    {
        wfb_mg_t *mg = nullptr;
        const int rc = wfb_mg_create(&mg, wfb::register_program<FKeyCarried>(), 1, 0, nullptr, 16, 4, 1, 64);
        if (rc != WFB_E_UNSUPPORTED) { std::printf("FAILED wfb_mg_create with a double key: %d\n", rc); return 1; }
        std::printf("wfb_mg_create refuses a double key OK\n");
    }
    run_all<DKey, double, DTupleSink, 5>("double key", 5, DKey(), DKEYS, DGROUP, 4, {1, 1, 1, 2});
    run_all<FKey, flow_t, FTupleSink, 4>("flow_t key", 4, FKey(), FKEYS, nullptr, 4, {1, 1, 1, 1});
    run_all<F16Key, flow16_t, F16TupleSink, 3>("flow16_t key", 3, F16Key(), F16KEYS, nullptr, 3, {1, 1, 1});
    std::printf("KEYS_OK\n");
    return 0;
}
