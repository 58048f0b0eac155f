// Application-level test of FlatMap_GPU in the builder API (include/wf/windflow_gpu.hpp): a WordCount-shaped pipeline. A Source of
// 64-byte "sentences" (0..6 word ids each) -> FlatMap_GPU (one record per word) -> keyed count-based Ffat_Windows_GPU -> Sink, run as
//   A  without a prefix, each word weighted by its position in the stream (seq * 8 + j): the windows depend on the arrival order
//   F  with Map_GPU -> Filter_GPU chained in front and fused into the FlatMap's pass, each word weighted by its word id
//   B  the same with the Map / Filter at parallelism 2: the run is not fused, and its two replicas may reorder batches
// and writes the sentences and the windows of every run to the directory argv[1]; tests/test_facade_flatmap.py expands the sentences
// with its numpy model and compares the windows with the oracle's. It also checks that run F has the two Map / Filter replicas of
// run B fewer. Prints FLATMAP_OK on success.
#include <cstdio>
#include <cstdlib>
#include <optional>
#include <string>
#include <vector>
#include <wf/windflow_gpu.hpp>

using namespace wf;

constexpr uint64_t N = 40000, BATCH = 1000, VOCAB = 97, MAXW = 6, WIN = 8, SLIDE = 4, NWB = 2;

struct sentence_t { uint64_t seq; uint64_t nwords; uint64_t words[MAXW]; };
struct word_t { uint64_t key; uint64_t weight; };
struct wres_t {
    uint64_t key, id; int64_t isum; double fsum;
    __host__ __device__ wres_t(): key(0), id(0), isum(0), fsum(0) {}
    __host__ __device__ wres_t(uint64_t k, uint64_t i): key(k), id(i), isum(0), fsum(0) {}
};
static_assert(sizeof(sentence_t) == 64 && sizeof(word_t) == 16 && sizeof(wres_t) == 32, "record sizes");

static uint64_t mix(uint64_t x) { x ^= x >> 31; x *= 0x7fb5d329728ea185ull; x ^= x >> 27; x *= 0x81dadef4bc2dd44dull; x ^= x >> 33; return x; }
static sentence_t sentence(uint64_t seq)
{
    sentence_t s{}; s.seq = seq; s.nwords = mix(seq) % (MAXW + 1);
    for (uint64_t j = 0; j < MAXW; j++) s.words[j] = j < s.nwords ? mix(seq * 8 + j + 1) % VOCAB : 0;
    return s;
}

struct Source_Functor {
    void operator()(Source_Shipper<sentence_t> &sh)
    {
        for (uint64_t seq = 0; seq < N; seq++) { sh.setNextWatermark(seq); sh.pushWithTimestamp(sentence(seq), seq); }
    }
};
struct Split { // one record per word, weighted by its position in the stream
    __host__ __device__ void operator()(const sentence_t &s, Shipper_GPU<word_t> &sh) const
    {
        for (uint64_t j = 0; j < s.nwords; j++) { word_t w; w.key = s.words[j]; w.weight = s.seq * 8 + j; sh.push(w); }
    }
};
struct DropLast { __host__ __device__ void operator()(sentence_t &s) const { if (s.seq % 5 == 0 && s.nwords > 0) s.nwords--; } };
struct Keep { __host__ __device__ bool operator()(sentence_t &s) const { return s.seq % 7 != 3; } };
struct WordKey { __host__ __device__ uint64_t operator()(const word_t &w) const { return w.key; } };
struct LiftPos { __host__ __device__ void operator()(const word_t &w, wres_t &r) const { r.isum = static_cast<int64_t>(w.weight); r.fsum = 0; } };
struct LiftWord { __host__ __device__ void operator()(const word_t &w, wres_t &r) const { r.isum = static_cast<int64_t>(w.key * 3 + 1); r.fsum = 0; } };
struct Comb { __host__ __device__ void operator()(const wres_t &a, const wres_t &b, wres_t &o) const { o.isum = a.isum + b.isum; o.fsum = a.fsum + b.fsum; } };

static std::vector<wres_t> got;
struct WinSink { void operator()(std::optional<wres_t> &r) { if (r) got.push_back(*r); } };

static void write_file(const std::string &path, const void *p, size_t bytes)
{
    FILE *f = std::fopen(path.c_str(), "wb");
    if (!f || std::fwrite(p, 1, bytes, f) != bytes) { std::printf("FAILED writing %s\n", path.c_str()); std::exit(1); }
    std::fclose(f);
}

template <class LiftF>
static size_t run(const std::string &name, int prefix_par, const std::string &dir)
{
    got.clear();
    PipeGraph graph(name, Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor()).withName("source").withOutputBatchSize(BATCH).build());
    if (prefix_par > 0) {
        mp.chain(MapGPU_Builder(DropLast()).withName("drop_last").withParallelism(prefix_par).build());
        mp.chain(FilterGPU_Builder(Keep()).withName("keep").withParallelism(prefix_par).build());
    }
    mp.chain(FlatMapGPU_Builder(Split()).withName("split").withMaxOutputsPerTuple(MAXW).build());
    mp.add(Ffat_WindowsGPU_Builder(LiftF(), Comb()).withName("count").withKeyBy(WordKey()).withCBWindows(WIN, SLIDE).withNumWinPerBatch(NWB)
               .withMaxKeys(128).build());
    mp.chain_sink(Sink_Builder(WinSink()).withName("sink").build());
    const size_t threads = graph.getNumThreads();
    graph.run();
    write_file(dir + "/" + name + ".bin", got.data(), got.size() * sizeof(wres_t));
    std::printf("run %s: %zu windows, %zu threads\n", name.c_str(), got.size(), threads);
    if (got.empty()) { std::printf("FAILED run %s: no windows\n", name.c_str()); std::exit(1); }
    return threads;
}

int main(int argc, char **argv)
{
    if (argc < 2) { std::printf("usage: %s OUTPUT_DIR\n", argv[0]); return 2; }
    const std::string dir = argv[1];
    std::vector<sentence_t> src(N);
    for (uint64_t seq = 0; seq < N; seq++) src[seq] = sentence(seq);
    write_file(dir + "/sentences.bin", src.data(), src.size() * sizeof(sentence_t));
    run<LiftPos>("A", 0, dir);
    const size_t fused = run<LiftWord>("F", 1, dir);
    const size_t unfused = run<LiftWord>("B", 2, dir);
    if (unfused != fused + 2) { std::printf("FAILED: %zu threads with the run fused, %zu without\n", fused, unfused); return 1; }
    std::printf("FLATMAP_OK\n");
    return 0;
}
