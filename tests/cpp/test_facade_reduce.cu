// Application-level test of the un-keyed Reduce_GPU in the builder API (include/wf/windflow_gpu.hpp): Source (withOutputBatchSize(BATCH),
// parallelism 1) -> ReduceGPU_Builder(f).build() -> Sink. Each source batch must reach the Sink as one row: the fold of the batch's tuples
// in arrival order, starting from a default-constructed tuple. The functor is a polynomial hash (associative, not commutative), so two
// tuples that change places change the row. The rows are compared with a direct fold on the host. Prints REDUCE_OK on success.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <optional>
#include <string>
#include <vector>
#include <wf/windflow_gpu.hpp>

using namespace wf;

constexpr uint64_t N = 400300, BATCH = 1000, MULT = 0x5851F42D4C957F2Dull; // (the last batch holds 300 tuples)

struct tuple_t { uint64_t key, seq, value; };

__host__ __device__ inline uint64_t pow_mod64(uint64_t b, uint64_t e)
{
    uint64_t r = 1;
    for (; e; e >>= 1, b *= b) if (e & 1) r *= b;
    return r;
}
struct Red { // (value, seq) as (h, q): (h1, q1) o (h2, q2) = (h1 M^q2 + h2, q1 + q2); the left operand's key is kept
    __host__ __device__ tuple_t operator()(const tuple_t &a, const tuple_t &b) const
    {
        tuple_t r = a;
        r.value = a.value * pow_mod64(MULT, b.seq) + b.value; r.seq = a.seq + b.seq;
        return r;
    }
};

static uint64_t mix64(uint64_t x) { x ^= x >> 31; x *= 0x7fb5d329728ea185ull; x ^= x >> 27; x *= 0x81dadef4bc2dd44dull; x ^= x >> 33; return x; }
static tuple_t item(uint64_t i) { return tuple_t{mix64(i * 2 + 1) % 300, i % 7, mix64(i * 2 + 2)}; }

struct Source_Functor {
    void operator()(Source_Shipper<tuple_t> &sh)
    {
        for (uint64_t i = 0; i < N; i++) { sh.setNextWatermark(i); sh.pushWithTimestamp(item(i), i); }
    }
};
static std::vector<tuple_t> rows;
struct Sink_Functor { void operator()(std::optional<tuple_t> &t) { if (t) rows.push_back(*t); } };

int main()
{
    PipeGraph graph("reduce_all", Execution_Mode_t::DEFAULT, Time_Policy_t::EVENT_TIME);
    MultiPipe &mp = graph.add_source(Source_Builder(Source_Functor()).withName("source").withOutputBatchSize(BATCH).build());
    mp.chain(ReduceGPU_Builder(Red()).withName("reduce").build());
    mp.chain_sink(Sink_Builder(Sink_Functor()).withName("sink").build());
    graph.run();
    std::vector<tuple_t> exp;
    for (uint64_t b = 0; b < N; b += BATCH) {
        tuple_t acc{};
        for (uint64_t i = b; i < std::min(N, b + BATCH); i++) acc = Red()(acc, item(i));
        exp.push_back(acc);
    }
    std::printf("%zu rows, %zu expected\n", rows.size(), exp.size());
    if (rows.size() != exp.size()) { std::printf("FAILED: one row per source batch expected\n"); return 1; }
    for (size_t r = 0; r < rows.size(); r++)
        if (rows[r].key != exp[r].key || rows[r].seq != exp[r].seq || rows[r].value != exp[r].value) {
            std::printf("FAILED row %zu: (%llu, %llu, %llx), expected (%llu, %llu, %llx)\n", r, (unsigned long long) rows[r].key,
                        (unsigned long long) rows[r].seq, (unsigned long long) rows[r].value, (unsigned long long) exp[r].key,
                        (unsigned long long) exp[r].seq, (unsigned long long) exp[r].value);
            return 1;
        }
    std::printf("REDUCE_OK\n");
    return 0;
}
