// Application-level test of the incremental Keyed_Windows_GPU in the builder API (include/wf/windflow_gpu.hpp): Source -> Map_GPU ->
// Filter_GPU -> Keyed_Windows_GPU (count-based, an order-sensitive function void(const tuple_t &, result_t &) folding each tuple into
// every open window it is IN) -> Sink, run as
//   K128  K = 128 batches per call
//   K1    one batch per call
//   NK    no withKeyBy: every tuple has the one key, the result starts as result_t(gwid)
// and writes the source's tuples and every run's results, in Sink order, to the directory argv[1]; tests/test_facade_keyed_windows_inc.py
// folds the tuples with its Python model and compares. Prints KEYED_WINDOWS_INC_OK on success.
#include <cstdio>
#include <cstdlib>
#include <optional>
#include <string>
#include <vector>
#include <wf/windflow_gpu.hpp>

using namespace wf;

constexpr uint64_t N = 40000, BATCH = 500, KEYS = 50, WIN = 12, SLIDE = 5;
constexpr uint64_t MIX = 0x9E3779B97F4A7C15ull, MUL = 0x100000001B3ull;

struct tup_t { uint64_t key, id; int64_t ivalue; double fvalue; uint64_t pad[4]; };
struct res_t {
    uint64_t key, id, hash, size, front, back, mask; double fsum; uint64_t argmax; int64_t maxiv;
    __host__ __device__ res_t(): key(0), id(0), hash(0), size(0), front(0), back(0), mask(0), fsum(0), argmax(0), maxiv(0) {}
    __host__ __device__ explicit res_t(uint64_t g): res_t() { id = g; }
    __host__ __device__ res_t(uint64_t k, uint64_t g): res_t() { key = k; id = g; }
};
static_assert(sizeof(tup_t) == 64 && sizeof(res_t) == 80, "record sizes");

static uint64_t mix(uint64_t x) { x ^= x >> 31; x *= 0x7fb5d329728ea185ull; x ^= x >> 27; x *= 0x81dadef4bc2dd44dull; x ^= x >> 33; return x; }
static tup_t make_tuple(uint64_t i)
{
    tup_t t{};
    t.key = mix(i) % KEYS; t.id = i;
    t.ivalue = static_cast<int64_t>(mix(i + 99) % 2000) - 1000;
    t.fvalue = static_cast<double>(mix(i + 7) >> 11) * (1.0 / 9007199254740992.0);
    return t;
}

struct Source_Functor {
    void operator()(Source_Shipper<tup_t> &sh)
    {
        for (uint64_t i = 0; i < N; i++) { sh.setNextWatermark(i); sh.pushWithTimestamp(make_tuple(i), i * 3); }
    }
};
struct AddTwo { __host__ __device__ void operator()(tup_t &t) const { t.ivalue += 2; } };
struct KeepSome { __host__ __device__ bool operator()(tup_t &t) const { return (t.ivalue & 3) != 0; } };
struct Key { __host__ __device__ uint64_t operator()(const tup_t &t) const { return t.key; } };
// the incremental window function: a polynomial hash over (id, ivalue), the size, the first and last id, the mask of the ivalue % 16
// seen, the in-order sum of fvalue and the id of the first tuple with the largest ivalue
struct WinIncF {
    __host__ __device__ void operator()(const tup_t &t, res_t &r) const
    {
        if (r.size == 0 || t.ivalue > r.maxiv) { r.maxiv = t.ivalue; r.argmax = t.id; }
        if (r.size == 0) r.front = t.id;
        r.hash = r.hash * MUL + (t.id * MIX ^ static_cast<uint64_t>(t.ivalue));
        r.size++; r.back = t.id;
        r.mask |= 1ull << (static_cast<uint64_t>(t.ivalue) & 15u);
        r.fsum += t.fvalue;
    }
};

static std::vector<res_t> got;
struct ResSink { void operator()(std::optional<res_t> &r) { if (r) got.push_back(*r); } };

static void write_file(const std::string &path, const void *p, size_t bytes)
{
    FILE *f = std::fopen(path.c_str(), "wb");
    if (!f || std::fwrite(p, 1, bytes, f) != bytes) { std::printf("FAILED writing %s\n", path.c_str()); std::exit(1); }
    std::fclose(f);
}

template <class Windows>
static void run(const std::string &name, Windows &&windows, const std::string &dir)
{
    got.clear();
    PipeGraph graph(name, Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor()).withName("source").withOutputBatchSize(BATCH).build());
    mp.chain(MapGPU_Builder(AddTwo()).withName("add").build());
    mp.chain(FilterGPU_Builder(KeepSome()).withName("keep").build());
    mp.add(windows);
    mp.chain_sink(Sink_Builder(ResSink()).withName("sink").build());
    graph.run();
    write_file(dir + "/" + name + ".bin", got.data(), got.size() * sizeof(res_t));
    std::printf("run %s: %zu windows\n", name.c_str(), got.size());
    if (got.empty()) { std::printf("FAILED run %s: no windows\n", name.c_str()); std::exit(1); }
}

int main(int argc, char **argv)
{
    if (argc < 2) { std::printf("usage: %s OUTPUT_DIR\n", argv[0]); return 2; }
    const std::string dir = argv[1];
    std::vector<tup_t> src(N);
    for (uint64_t i = 0; i < N; i++) src[i] = make_tuple(i);
    write_file(dir + "/tuples.bin", src.data(), src.size() * sizeof(tup_t));
    run("K128", Keyed_WindowsGPU_Builder(WinIncF()).withName("windows").withKeyBy(Key()).withCBWindows(WIN, SLIDE).withMaxKeys(64)
                    .withMaxBatchesPerCall(128).build(), dir);
    run("K1", Keyed_WindowsGPU_Builder(WinIncF()).withName("windows").withKeyBy(Key()).withCBWindows(WIN, SLIDE).withMaxKeys(64)
                  .withMaxBatchesPerCall(1).build(), dir);
    run("NK", Keyed_WindowsGPU_Builder(WinIncF()).withName("windows").withCBWindows(WIN, SLIDE).withMaxBatchesPerCall(128).build(), dir);
    std::printf("KEYED_WINDOWS_INC_OK\n");
    return 0;
}
