// FlatMap programs registered at run time, as an application registers its own functors (wfb::register_program, INTEGRATION.md
// section 3). tests/test_gpu_flatmap.py builds this file into a shared object linked against libwfb200.so, compares the programs'
// host functors with its numpy model of the expansion, and the GPU's wfb_flatmap_batches with the same model byte for byte;
// tools/flatmap_bench.py measures them.
//
// The fan-out of a tuple is part of the tuple (pad[3] of a 64-byte tuple, the low 6 bits of `value` of a 16-byte one), so a test
// chooses every tuple's count, including counts above the operator's bound. The map / filter slots are those of the built-in
// programs over the same tuples (ProgTuple64, ProgWfTest16): wfb_functors_t selects them, as for wfb_map_filter_batches.
#include <cstdint>
#include "wfb_launch.cuh"
#include "wfb_programs.cuh"

namespace {

struct Rec16 { uint64_t key; int64_t value; };
struct Rec32 { uint64_t key; uint64_t id; uint64_t j; int64_t value; };
struct Rec48 { uint64_t key; uint64_t id; int64_t value; uint64_t j; uint64_t a, b; };
static_assert(sizeof(Rec16) == 16 && sizeof(Rec32) == 32 && sizeof(Rec48) == 48, "record sizes");
constexpr uint64_t MIX = 0x9E3779B97F4A7C15ull;

// 64-byte tuples -> pad[3] records of 16 bytes: (key + j, 3 * ivalue + j)
struct Fm64to16 {
    using tuple_t = wfb_tuple64_t; using result_t = Rec16; using key_t = uint64_t; using params_t = wfb_functors_t;
    __host__ __device__ static void map(tuple_t &t, const params_t &p) { wfb::ProgTuple64::map(t, p); }
    __host__ __device__ static bool filter(tuple_t &t, const params_t &p) { return wfb::ProgTuple64::filter(t, p); }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static void lift(const tuple_t &, result_t &r, const params_t &) { r = result_t{}; }
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t{}; }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
    __host__ __device__ static void flatmap(const tuple_t &t, wfb::Shipper<result_t> &sh, const params_t &)
    {
        for (uint64_t j = 0; j < t.pad[3]; j++) {
            Rec16 r; r.key = t.key + j; r.value = static_cast<int64_t>(static_cast<uint64_t>(t.ivalue) * 3u + j);
            sh.push(r);
        }
    }
};

// 64-byte tuples -> pad[3] records of 32 bytes: (key, id, j, ivalue + j)
struct Fm64to32: Fm64to16 {
    using result_t = Rec32;
    __host__ __device__ static void lift(const tuple_t &, result_t &r, const params_t &) { r = result_t{}; }
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t{}; }
    __host__ __device__ static void flatmap(const tuple_t &t, wfb::Shipper<result_t> &sh, const params_t &)
    {
        for (uint64_t j = 0; j < t.pad[3]; j++) {
            Rec32 r; r.key = t.key; r.id = t.id; r.j = j; r.value = static_cast<int64_t>(static_cast<uint64_t>(t.ivalue) + j);
            sh.push(r);
        }
    }
};

// 16-byte tuples {key, value} -> (value & 63) records of 48 bytes: (key, value >> 6, value, j, key ^ j, j * MIX)
struct Fm16to48 {
    using tuple_t = wfb_wftest16_t; using result_t = Rec48; using key_t = uint64_t; using params_t = wfb_functors_t;
    __host__ __device__ static void map(tuple_t &t, const params_t &p) { wfb::ProgWfTest16::map(t, p); }
    __host__ __device__ static bool filter(tuple_t &t, const params_t &p) { return wfb::ProgWfTest16::filter(t, p); }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static void lift(const tuple_t &, result_t &r, const params_t &) { r = result_t{}; }
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t{}; }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
    __host__ __device__ static void flatmap(const tuple_t &t, wfb::Shipper<result_t> &sh, const params_t &)
    {
        const uint64_t n = static_cast<uint64_t>(t.value) & 63u;
        for (uint64_t j = 0; j < n; j++) {
            Rec48 r; r.key = t.key; r.id = static_cast<uint64_t>(t.value) >> 6; r.value = t.value; r.j = j; r.a = t.key ^ j; r.b = j * MIX;
            sh.push(r);
        }
    }
};

// 64-byte tuples -> at most one 64-byte tuple: map(t) when filter(map(t)) holds, with the built-in program's functors applied INSIDE
// the flatmap (its own map / filter slots do nothing), so that m = 1 reproduces wfb_map_filter_batches of ProgTuple64
struct FmSelect64 {
    using tuple_t = wfb_tuple64_t; using result_t = wfb_tuple64_t; using key_t = uint64_t; using params_t = wfb_functors_t;
    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &, const params_t &) { return true; }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &) { r = t; }
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t{}; }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
    __host__ __device__ static void flatmap(const tuple_t &t, wfb::Shipper<result_t> &sh, const params_t &p)
    {
        tuple_t u = t;
        wfb::ProgTuple64::map(u, p);
        if (wfb::ProgTuple64::filter(u, p)) sh.push(u);
    }
};

// the whole operator on the host, tuple after tuple: [map ->] [filter ->] flatmap, records at consecutive positions
template <class P>
void host_run(const wfb_functors_t &f, const void *tuples, const uint64_t *ts, uint64_t n, uint32_t m, void *out, uint64_t *ts_out,
              uint64_t *n_out, uint64_t *dropped)
{
    const typename P::tuple_t *in = static_cast<const typename P::tuple_t *>(tuples);
    uint64_t pos = 0, drop = 0;
    for (uint64_t i = 0; i < n; i++) {
        typename P::tuple_t t = in[i];
        P::map(t, f);
        if (!P::filter(t, f)) continue;
        wfb::Shipper<typename P::result_t> sh(static_cast<unsigned char *>(out) + pos * sizeof(typename P::result_t),
                                              ts_out != nullptr ? ts_out + pos : nullptr, ts != nullptr ? ts[i] : 0, m);
        P::flatmap(t, sh, f);
        const uint32_t c = sh.pushes();
        pos += c < m ? c : m; drop += c > m ? c - m : 0;
    }
    *n_out = pos; *dropped = drop;
}

} // namespace

extern "C" {

// 0: 64 -> 16 bytes, 1: 64 -> 32, 2: 16 -> 48, 3: 64 -> 64 (selection); the program id, or -1 for another index
int fm_register(int which)
{
    switch (which) {
    case 0: return wfb::register_program<Fm64to16>();
    case 1: return wfb::register_program<Fm64to32>();
    case 2: return wfb::register_program<Fm16to48>();
    case 3: return wfb::register_program<FmSelect64>();
    }
    return -1;
}

int fm_host(int which, const wfb_functors_t *f, const void *tuples, const uint64_t *ts, uint64_t n, uint32_t m, void *out, uint64_t *ts_out,
            uint64_t *n_out, uint64_t *dropped)
{
    switch (which) {
    case 0: host_run<Fm64to16>(*f, tuples, ts, n, m, out, ts_out, n_out, dropped); return 0;
    case 1: host_run<Fm64to32>(*f, tuples, ts, n, m, out, ts_out, n_out, dropped); return 0;
    case 2: host_run<Fm16to48>(*f, tuples, ts, n, m, out, ts_out, n_out, dropped); return 0;
    case 3: host_run<FmSelect64>(*f, tuples, ts, n, m, out, ts_out, n_out, dropped); return 0;
    }
    return -1;
}

} // extern "C"
