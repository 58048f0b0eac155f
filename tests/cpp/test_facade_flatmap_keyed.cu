// Application-level test of the keyed-stateful FlatMap_GPU in the builder API (include/wf/windflow_gpu.hpp): a sessionising pipeline.
// A Source of events {user, seq, time, value} -> FlatMap_GPU keyed by user (m = 2: when the gap since the user's last event exceeds GAP,
// the closed session's summary, then the event's own record) -> keyed count-based Ffat_Windows_GPU over the records -> Sink, run as
//   P1    parallelism 1, K = 128 batches per call
//   K1    parallelism 1, one batch per call
//   G     parallelism 1, a key table of 16 keys that grows (withKeyGrowth)
//   P2    parallelism 2: the source alternates the batches between the replicas, and a user's events all lie in batches of one parity,
//         so every user's events reach one replica in order and the windows are those of P1 (emitted in another order)
// and writes the events and the windows of every run to the directory argv[1]; tests/test_facade_flatmap_keyed.py sessionises the
// events with its numpy model and compares the windows with the oracle's. Prints FLATMAP_KEYED_OK on success.
#include <cstdio>
#include <cstdlib>
#include <optional>
#include <string>
#include <vector>
#include <wf/windflow_gpu.hpp>

using namespace wf;

constexpr uint64_t N = 60000, BATCH = 500, USERS = 40, GAP = 700, WIN = 8, SLIDE = 4, NWB = 2;

struct event_t { uint64_t user, seq, time; int64_t value; };
struct session_t { uint64_t last, start, count; int64_t sum; };
struct rec_t { uint64_t key, kind, a; int64_t b; };
struct wres_t {
    uint64_t key, id; int64_t isum; double fsum;
    __host__ __device__ wres_t(): key(0), id(0), isum(0), fsum(0) {}
    __host__ __device__ wres_t(uint64_t k, uint64_t i): key(k), id(i), isum(0), fsum(0) {}
};
static_assert(sizeof(event_t) == 32 && sizeof(rec_t) == 32 && sizeof(wres_t) == 32, "record sizes");

static uint64_t mix(uint64_t x) { x ^= x >> 31; x *= 0x7fb5d329728ea185ull; x ^= x >> 27; x *= 0x81dadef4bc2dd44dull; x ^= x >> 33; return x; }
static event_t event(uint64_t seq)
{
    event_t e; e.seq = seq; e.time = seq * 10;
    e.user = 2 * (mix(seq) % (USERS / 2)) + (seq / BATCH) % 2; // (a user's events lie in batches of one parity)
    e.value = static_cast<int64_t>(mix(seq + 77) % 1000) - 500;
    return e;
}

struct Source_Functor {
    void operator()(Source_Shipper<event_t> &sh)
    {
        for (uint64_t seq = 0; seq < N; seq++) { sh.setNextWatermark(seq); sh.pushWithTimestamp(event(seq), seq); }
    }
};
struct Sessionise { // the closed session's summary (kind 1: start, count * 1000 + sum), then the event (kind 0: seq, position in its session)
    __host__ __device__ void operator()(const event_t &e, Shipper_GPU<rec_t> &sh, session_t &st) const
    {
        if (st.count > 0 && e.time - st.last > GAP) {
            sh.push(rec_t{e.user, 1, st.start, static_cast<int64_t>(st.count) * 1000 + st.sum});
            st.count = 0; st.sum = 0;
        }
        if (st.count == 0) st.start = e.time;
        st.count++; st.sum += e.value; st.last = e.time;
        sh.push(rec_t{e.user, 0, e.seq, static_cast<int64_t>(st.count)});
    }
};
struct UserKey { __host__ __device__ uint64_t operator()(const event_t &e) const { return e.user; } };
struct RecKey { __host__ __device__ uint64_t operator()(const rec_t &r) const { return r.key; } };
struct Lift { __host__ __device__ void operator()(const rec_t &r, wres_t &w) const { w.isum = static_cast<int64_t>(r.a * (r.kind ? 7 : 3)) + r.b; w.fsum = 0; } };
struct Comb { __host__ __device__ void operator()(const wres_t &a, const wres_t &b, wres_t &o) const { o.isum = a.isum + b.isum; o.fsum = a.fsum + b.fsum; } };

static std::vector<wres_t> got;
struct WinSink { void operator()(std::optional<wres_t> &r) { if (r) got.push_back(*r); } };

static void write_file(const std::string &path, const void *p, size_t bytes)
{
    FILE *f = std::fopen(path.c_str(), "wb");
    if (!f || std::fwrite(p, 1, bytes, f) != bytes) { std::printf("FAILED writing %s\n", path.c_str()); std::exit(1); }
    std::fclose(f);
}

static void run(const std::string &name, size_t par, size_t k, bool grow, const std::string &dir)
{
    got.clear();
    PipeGraph graph(name, Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor()).withName("source").withOutputBatchSize(BATCH).build());
    auto b = FlatMapGPU_Builder(Sessionise()).withName("sessions").withKeyBy(UserKey()).withMaxOutputsPerTuple(2).withParallelism(par)
                 .withMaxKeys(grow ? 16 : 64);
    if (grow) b.withKeyGrowth();
    auto op = b.build();
    op.maxk = k;
    mp.chain(op);
    mp.add(Ffat_WindowsGPU_Builder(Lift(), Comb()).withName("count").withKeyBy(RecKey()).withCBWindows(WIN, SLIDE).withNumWinPerBatch(NWB)
               .withMaxKeys(64).build());
    mp.chain_sink(Sink_Builder(WinSink()).withName("sink").build());
    graph.run();
    write_file(dir + "/" + name + ".bin", got.data(), got.size() * sizeof(wres_t));
    std::printf("run %s: %zu windows\n", name.c_str(), got.size());
    if (got.empty()) { std::printf("FAILED run %s: no windows\n", name.c_str()); std::exit(1); }
}

int main(int argc, char **argv)
{
    if (argc < 2) { std::printf("usage: %s OUTPUT_DIR\n", argv[0]); return 2; }
    const std::string dir = argv[1];
    std::vector<event_t> src(N);
    for (uint64_t seq = 0; seq < N; seq++) src[seq] = event(seq);
    write_file(dir + "/events.bin", src.data(), src.size() * sizeof(event_t));
    run("P1", 1, WF_MAX_BATCHES_PER_CALL, false, dir);
    run("K1", 1, 1, false, dir);
    run("G", 1, WF_MAX_BATCHES_PER_CALL, true, dir);
    run("P2", 2, WF_MAX_BATCHES_PER_CALL, false, dir);
    std::printf("FLATMAP_KEYED_OK\n");
    return 0;
}
