// tests/golden/ref_keyed_windows_inc.cpp -- TEST INFRASTRUCTURE: the UNMODIFIED reference (wf/windflow.hpp, included from a WindFlow
// checkout at build time; FastFlow's API comes from include/ff/) running
//
//     Source -> Map -> Filter -> Keyed_Windows (count-based, INCREMENTAL window function, DETERMINISTIC mode) -> Sink
//
// on the bench schema, with the order-sensitive fold of tests/cpp/kwin_inc_programs.cu, void(const tuple64_t &, result80_t &), which the
// reference calls once per tuple for every open window the tuple is IN. It is the incremental counterpart of
// tests/golden/ref_keyed_windows.cpp, with the same arguments, stream file and synthetic stream. tests/golden/make_golden_kwi.py
// compiles it (g++, CPU only), runs it on the streams of ref_cpu_kw_*.npz and stores its outputs as tests/golden/ref_cpu_kwi_*.npz;
// tools/keyed_windows_bench.py runs it as the incremental reference CPU arm. Nothing of the product links or loads this program.
//
//   ref_keyed_windows_inc key=value ...
//     in=<file>   stream to replay: u64 n, then n x tuple64, n x u64 timestamps, n x u64 watermarks
//     gen=<n>     instead of in=: n tuples of the synthetic stream (seed 0x5EED5EED, keys splitmix64(i) % keys, ts = i)
//     out=<file>  results: u64 m, then m x {result80, u64 ts}, in Sink order
//     win= slide= keys= par= (replicas of Map, Filter and Keyed_Windows; default 1)
//   prints one JSON line {"mode","tuples","seconds","tuples_per_s","results","threads"}.
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <mutex>
#include <optional>
#include <string>
#include <vector>
#include <windflow.hpp>

using namespace wf;

struct tuple64_t {
    uint64_t key, id; int64_t ivalue; double fvalue; uint64_t pad[4];
    tuple64_t(): key(0), id(0), ivalue(0), fvalue(0) { pad[0] = pad[1] = pad[2] = pad[3] = 0; }
};
struct result80_t {
    uint64_t key, id, hash, size, front, back, mask; double fsum; uint64_t argmax; int64_t maxiv;
    result80_t(): key(0), id(0), hash(0), size(0), front(0), back(0), mask(0), fsum(0), argmax(0), maxiv(0) {}
    result80_t(uint64_t k, uint64_t g): result80_t() { key = k; id = g; }
};
static_assert(sizeof(tuple64_t) == 64 && sizeof(result80_t) == 80, "record sizes");

constexpr uint64_t MIX = 0x9E3779B97F4A7C15ull, MUL = 0x100000001B3ull;

struct MapC { void operator()(tuple64_t &t) { t.ivalue += 2; t.fvalue *= 1.0000001; } };
struct FiltC { bool operator()(tuple64_t &t) { return (t.ivalue & 1) == 0; } };
// the incremental window function of tests/cpp/kwin_inc_programs.cu: hash over (id, ivalue), size, first and last id, the mask of the
// ivalue % 16 seen, the in-order sum of fvalue, the id of the first tuple with the largest ivalue
struct WinIncC {
    void operator()(const tuple64_t &t, result80_t &r)
    {
        if (r.size == 0 || t.ivalue > r.maxiv) { r.maxiv = t.ivalue; r.argmax = t.id; }
        if (r.size == 0) r.front = t.id;
        r.hash = r.hash * MUL + (t.id * MIX ^ static_cast<uint64_t>(t.ivalue));
        r.size++; r.back = t.id;
        r.mask |= 1ull << (static_cast<uint64_t>(t.ivalue) & 15u);
        r.fsum += t.fvalue;
    }
};

static uint64_t splitmix64(uint64_t x) { x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; return x ^ (x >> 31); }

struct Stream { std::vector<tuple64_t> t; std::vector<uint64_t> ts; };
struct SourceF {
    const Stream *s;
    void operator()(Source_Shipper<tuple64_t> &sh)
    {
        for (size_t i = 0; i < s->t.size(); i++) { tuple64_t t = s->t[i]; sh.pushWithTimestamp(std::move(t), s->ts[i]); }
    }
};
struct Collected { std::mutex mu; std::vector<result80_t> res; std::vector<uint64_t> ts; };
struct SinkF {
    Collected *c;
    void operator()(std::optional<result80_t> &o, RuntimeContext &ctx)
    {
        if (!o) return;
        std::lock_guard<std::mutex> l(c->mu);
        c->res.push_back(*o); c->ts.push_back(ctx.getCurrentTimestamp());
    }
};

int main(int argc, char **argv)
{
    std::map<std::string, std::string> kv;
    for (int i = 1; i < argc; i++) { const char *e = std::strchr(argv[i], '='); if (e) kv[std::string(argv[i], e - argv[i])] = e + 1; }
    auto num = [&](const char *k, uint64_t d) { return kv.count(k) ? std::strtoull(kv[k].c_str(), nullptr, 10) : d; };
    const uint64_t win = num("win", 64), slide = num("slide", 16), nkeys = num("keys", 1024), par = num("par", 1);
    if (win == 0 || slide == 0) { std::fprintf(stderr, "ref_keyed_windows_inc: win and slide must be positive\n"); return 2; }
    Stream s;
    if (kv.count("in")) {
        std::ifstream f(kv["in"], std::ios::binary);
        uint64_t n = 0;
        f.read(reinterpret_cast<char *>(&n), 8);
        s.t.resize(n); s.ts.resize(n);
        std::vector<uint64_t> wm(n);
        f.read(reinterpret_cast<char *>(s.t.data()), n * 64); f.read(reinterpret_cast<char *>(s.ts.data()), n * 8); f.read(reinterpret_cast<char *>(wm.data()), n * 8);
        if (!f) { std::fprintf(stderr, "ref_keyed_windows_inc: short read of %s\n", kv["in"].c_str()); return 2; }
    } else {
        const uint64_t n = num("gen", 1 << 20), seed = 0x5EED5EEDull;
        s.t.resize(n); s.ts.resize(n);
        for (uint64_t i = 0; i < n; i++) {
            tuple64_t &t = s.t[i];
            t.key = splitmix64(i) % nkeys; t.id = i;
            t.ivalue = static_cast<int64_t>(splitmix64(seed ^ i) & 0xFFFF);
            t.fvalue = static_cast<double>(splitmix64(seed ^ ~i) >> 11) * (1.0 / 9007199254740992.0);
            s.ts[i] = i;
        }
    }
    Collected c;
    size_t threads = 0;
    const auto t0 = std::chrono::steady_clock::now();
    {
        PipeGraph graph("ref_keyed_windows_inc", Execution_Mode_t::DETERMINISTIC, Time_Policy_t::EVENT_TIME);
        SourceF src{&s};
        Source source = Source_Builder(src).withName("source").withParallelism(1).build();
        MultiPipe &mp = graph.add_source(source);
        MapC mf; FiltC ff_;
        Map map = Map_Builder(mf).withName("map").withParallelism(par).build();
        mp.chain(map);
        Filter filter = Filter_Builder(ff_).withName("filter").withParallelism(par).build();
        mp.chain(filter);
        WinIncC wf_;
        Keyed_Windows kwin = Keyed_Windows_Builder(wf_).withName("keyed_windows").withParallelism(par)
                                 .withKeyBy([](const tuple64_t &t) -> uint64_t { return t.key; }).withCBWindows(win, slide).build();
        mp.add(kwin);
        SinkF sf{&c};
        Sink sink = Sink_Builder(sf).withName("sink").withParallelism(1).build();
        mp.chain_sink(sink);
        threads = graph.getNumThreads();
        graph.run();
    }
    const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    if (kv.count("out")) {
        std::ofstream f(kv["out"], std::ios::binary);
        const uint64_t m = c.res.size();
        f.write(reinterpret_cast<const char *>(&m), 8);
        for (uint64_t i = 0; i < m; i++) { f.write(reinterpret_cast<const char *>(&c.res[i]), sizeof(result80_t)); f.write(reinterpret_cast<const char *>(&c.ts[i]), 8); }
    }
    std::printf("{\"mode\": \"cpu_kwi\", \"tuples\": %zu, \"seconds\": %.6f, \"tuples_per_s\": %.1f, \"results\": %zu, \"threads\": %zu}\n", s.t.size(), sec,
                s.t.size() / sec, c.res.size(), threads);
    return 0;
}
