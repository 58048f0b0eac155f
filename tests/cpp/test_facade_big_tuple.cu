// Application-level test of the builder API (include/wf/windflow_gpu.hpp) with a 256-byte tuple. Map_GPU, Filter_GPU and keyed-stateful
// operators register a program whose result_t is the tuple itself, and the window kernels are instantiated for every program: a tuple of
// 256 bytes needs the tile pass with fewer stages and the full-sort window path. Two runs, each writing its Sink's rows to argv[1]:
//   cb        Source -> Map -> Filter -> count-based Ffat_Windows_GPU -> Sink (window records)
//   stateful  Source -> Map -> keyed-stateful Map -> Sink (tuples, in stream order)
// The Map rewrites every pad word, the Filter and the lift read the last one, the window combine is an order-sensitive hash and the
// stateful functor stamps its running hash and count into the tuple. tests/test_facade_big_tuple.py compares the rows with its numpy
// model. Prints BIG_TUPLE_OK on success.
#include <cstdio>
#include <cstdlib>
#include <optional>
#include <string>
#include <vector>
#include <wf/windflow_gpu.hpp>

using namespace wf;

constexpr uint64_t N = 60000, BATCH = 1000, NKEYS = 37, WIN = 24, SLIDE = 8, NWB = 2, MULT = 0x5851F42D4C957F2Dull;

struct big_t { uint64_t key, seq; uint64_t pad[30]; };
struct result_t {
    uint64_t key, id, h, q;
    __host__ __device__ result_t(): key(0), id(0), h(0), q(0) {}
    __host__ __device__ result_t(uint64_t k, uint64_t i): key(k), id(i), h(0), q(0) {}
};
struct state_t { uint64_t count, hash; };
static_assert(sizeof(big_t) == 256 && sizeof(result_t) == 32 && sizeof(state_t) == 16, "record sizes");

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
struct Stir {
    __host__ __device__ void operator()(big_t &t) const
    {
        for (uint64_t j = 0; j < 30; j++) t.pad[j] = (t.pad[j] ^ (t.key * 0xD6E8FEB86659FD93ull)) + (j + 1) * t.seq;
    }
};
struct Keep { __host__ __device__ bool operator()(big_t &t) const { return t.seq % 7 != 3 && (t.pad[29] >> 5) % 4 != 0; } };
struct KeyF { __host__ __device__ uint64_t operator()(const big_t &t) const { return t.key; } };
struct Lift { __host__ __device__ void operator()(const big_t &t, result_t &r) const { r.key = t.key; r.id = 0; r.h = ord_mix(t.pad[29] ^ t.pad[0], t.key); r.q = 1; } };
struct Comb { // (h1, q1) o (h2, q2) = (h1 M^q2 + h2, q1 + q2)
    __host__ __device__ void operator()(const result_t &a, const result_t &b, result_t &o) const
    {
        const uint64_t h = a.h * ord_pow(MULT, b.q) + b.h, q = a.q + b.q;
        o.h = h; o.q = q;
    }
};
struct SMap { // the key's running hash and count go into pad[0] and pad[1]
    __host__ __device__ void operator()(big_t &t, state_t &st) const
    {
        st.count++; st.hash = st.hash * MULT + ord_mix(t.pad[29], t.key);
        t.pad[0] = st.hash; t.pad[1] = st.count;
    }
};

static uint64_t mix64(uint64_t x) { x ^= x >> 31; x *= 0x7fb5d329728ea185ull; x ^= x >> 27; x *= 0x81dadef4bc2dd44dull; x ^= x >> 33; return x; }
static big_t make(uint64_t i)
{
    big_t t{}; t.key = mix64(i) % NKEYS; t.seq = i;
    for (uint64_t j = 0; j < 30; j++) t.pad[j] = mix64(i * 32 + j + 1);
    return t;
}
struct Source_Functor {
    void operator()(Source_Shipper<big_t> &sh) { for (uint64_t i = 0; i < N; i++) { sh.setNextWatermark(i); sh.pushWithTimestamp(make(i), i); } }
};
template <class R> struct Rows { static std::vector<R> v; };
template <class R> std::vector<R> Rows<R>::v;
template <class R> struct Collect { void operator()(std::optional<R> &r) { if (r) Rows<R>::v.push_back(*r); } };

static void write_file(const std::string &path, const void *p, size_t bytes)
{
    FILE *f = std::fopen(path.c_str(), "wb");
    if (!f || std::fwrite(p, 1, bytes, f) != bytes) { std::printf("FAILED writing %s\n", path.c_str()); std::exit(1); }
    std::fclose(f);
}

int main(int argc, char **argv)
{
    if (argc < 2) { std::printf("usage: %s OUTPUT_DIR\n", argv[0]); return 2; }
    const std::string dir = argv[1];
    {
        PipeGraph graph("cb", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
        MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor()).withName("source").withOutputBatchSize(BATCH).build());
        mp.chain(MapGPU_Builder(Stir()).withName("stir").build());
        mp.chain(FilterGPU_Builder(Keep()).withName("keep").build());
        mp.add(Ffat_WindowsGPU_Builder(Lift(), Comb()).withName("windows").withKeyBy(KeyF()).withCBWindows(WIN, SLIDE).withNumWinPerBatch(NWB)
                   .withMaxKeys(64).build());
        mp.chain_sink(Sink_Builder(Collect<result_t>()).withName("sink").build());
        graph.run();
        write_file(dir + "/cb.bin", Rows<result_t>::v.data(), Rows<result_t>::v.size() * sizeof(result_t));
        std::printf("run cb: %zu windows\n", Rows<result_t>::v.size());
    }
    {
        PipeGraph graph("stateful", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
        MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor()).withName("source").withOutputBatchSize(BATCH).build());
        mp.chain(MapGPU_Builder(Stir()).withName("stir").build());
        mp.chain(MapGPU_Builder(SMap()).withName("smap").withKeyBy(KeyF()).withMaxKeys(64).build());
        mp.chain_sink(Sink_Builder(Collect<big_t>()).withName("sink").build());
        graph.run();
        write_file(dir + "/stateful.bin", Rows<big_t>::v.data(), Rows<big_t>::v.size() * sizeof(big_t));
        std::printf("run stateful: %zu rows\n", Rows<big_t>::v.size());
    }
    if (Rows<result_t>::v.empty() || Rows<big_t>::v.size() != N) { std::printf("FAILED: %zu windows, %zu rows\n", Rows<result_t>::v.size(), Rows<big_t>::v.size()); return 1; }
    std::printf("BIG_TUPLE_OK\n");
    return 0;
}
