// headline_facade.cu -- the builder-API pipeline of windflow_b200/apps/pipeline_bench.cu with every window result recorded:
//
//     SourceGPU (a ring of batches resident in HBM) -> Map_GPU -> Filter_GPU -> Ffat_Windows_GPU (count-based) -> Sink
//
// The same functors, builders and configuration (64-byte tuples of the seeded synthetic stream, batch 65536, 65536 dense keys, map
// ivalue += 2 / fvalue *= 1.0000001, filter (ivalue & 1) == 0, windows 4096 / 64, Nb 65, K batches per call, two Sink replicas), in
// both styles: "fluent" (one chain expression: the functor types reach the window operator's program) and "statements" (one chain
// call per statement: fused through device function pointers). Batch i of the source is batch i % ring of the stream, with watermark
// i + 1. Every Sink replica writes the (key, id, isum, fsum) records it received to <dir>/sink<r>.bin; tests/test_gpu_headline.py
// replays the same batches through a direct fold and compares the whole run as a set.
//   usage: headline_facade.bin K batches ring sinks fluent|statements dir
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <optional>
#include <string>
#include <vector>
#include <wf/windflow_gpu.hpp>

using namespace wf;

struct tuple64_t { uint64_t key, id; int64_t ivalue; double fvalue; uint64_t pad[4]; };
struct result32_t {
    uint64_t key, id; int64_t isum; double fsum;
    __host__ __device__ result32_t(): key(0), id(0), isum(0), fsum(0) {}
    __host__ __device__ result32_t(uint64_t k, uint64_t i): key(k), id(i), isum(0), fsum(0) {}
};
static_assert(sizeof(result32_t) == 32, "record size");
struct MapF { __host__ __device__ void operator()(tuple64_t &t) { t.ivalue += 2; t.fvalue *= 1.0000001; } };
struct FiltF { __host__ __device__ bool operator()(tuple64_t &t) { return (t.ivalue & 1) == 0; } };
struct LiftF { __host__ __device__ void operator()(const tuple64_t &t, result32_t &r) { r.key = t.key; r.id = 0; r.isum = t.ivalue; r.fsum = t.fvalue; } };
struct CombF { __host__ __device__ void operator()(const result32_t &a, const result32_t &b, result32_t &o) { o.isum = a.isum + b.isum; o.fsum = a.fsum + b.fsum; } };
struct KeyF { __host__ __device__ uint64_t operator()(const tuple64_t &t) { return t.key; } };

static std::string g_dir;
static std::atomic<int> g_files{0};
static std::atomic<uint64_t> g_rows{0};
static std::atomic<bool> g_write_failed{false};

// every Sink replica (a copy of this functor) keeps its records and writes them to a file of its own at the end of the stream
struct SinkF {
    std::vector<result32_t> mine;
    void operator()(std::optional<result32_t> &r)
    {
        if (r) { mine.push_back(*r); return; }
        const std::string path = g_dir + "/sink" + std::to_string(g_files.fetch_add(1)) + ".bin";
        FILE *f = std::fopen(path.c_str(), "wb");
        if (!f || std::fwrite(mine.data(), sizeof(result32_t), mine.size(), f) != mine.size()) g_write_failed = true;
        if (f) std::fclose(f);
        g_rows.fetch_add(mine.size());
    }
};

int main(int argc, char **argv)
{
    if (argc != 7) { std::fprintf(stderr, "usage: %s K batches ring sinks fluent|statements dir\n", argv[0]); return 2; }
    const size_t K = std::strtoull(argv[1], nullptr, 10);
    const uint64_t nbatches = std::strtoull(argv[2], nullptr, 10);
    const uint64_t ring = std::strtoull(argv[3], nullptr, 10);
    const size_t sinks = std::strtoull(argv[4], nullptr, 10);
    const bool fluent = std::strcmp(argv[5], "statements") != 0;
    g_dir = argv[6];
    const uint64_t BATCH = 65536, WIN = 4096, SLIDE = 64, NKEYS = 65536;
    const size_t NB = 65;

    tuple64_t *d_tuples = nullptr; uint64_t *d_ts = nullptr;
    gpuErrChk(cudaMalloc(&d_tuples, ring * BATCH * sizeof(tuple64_t)));
    gpuErrChk(cudaMalloc(&d_ts, ring * BATCH * sizeof(uint64_t)));
    for (uint64_t r = 0; r < ring; r++)
        wfbErrChk(wfb_gen_tuple64(0x5EED5EEDull, r * BATCH, static_cast<uint32_t>(BATCH), 1, NKEYS, nullptr, d_tuples + r * BATCH, d_ts + r * BATCH, nullptr));
    gpuErrChk(cudaDeviceSynchronize());

    auto source = [&](SourceGPU_Shipper<tuple64_t> &sh) {
        for (uint64_t i = 0; i < nbatches; i++) { const uint64_t r = i % ring; sh.pushBatch(d_tuples + r * BATCH, d_ts + r * BATCH, BATCH, i + 1); }
    };
    {
        PipeGraph graph("headline_facade", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
        MultiPipe &mp = graph.add_source(SourceGPU_Builder(source).withName("source").build());
        auto ffat = Ffat_WindowsGPU_Builder(LiftF(), CombF()).withName("ffat").withKeyBy(KeyF()).withCBWindows(WIN, SLIDE).withNumWinPerBatch(NB)
                        .withMaxKeys(static_cast<uint32_t>(NKEYS)).withDenseKeys().withMaxBatchesPerCall(K).build();
        if (fluent) mp.chain(MapGPU_Builder(MapF()).withName("map").build()).chain(FilterGPU_Builder(FiltF()).withName("filter").build()).add(ffat);
        else {
            mp.chain(MapGPU_Builder(MapF()).withName("map").build());
            mp.chain(FilterGPU_Builder(FiltF()).withName("filter").build());
            mp.add(ffat);
        }
        mp.chain_sink(Sink_Builder(SinkF()).withName("sink").withParallelism(sinks).build());
        graph.run();
    }
    cudaFree(d_tuples); cudaFree(d_ts);
    if (g_write_failed || g_files.load() != static_cast<int>(sinks)) { std::printf("FACADE_FAILED: %d files written\n", g_files.load()); return 1; }
    std::printf("FACADE_OK style %s: %llu windows in %d files\n", fluent ? "fluent" : "statements", static_cast<unsigned long long>(g_rows.load()), g_files.load());
    return 0;
}
