// Keyed_Windows_GPU programs registered at run time, as an application registers its own functors (wfb::register_program,
// INTEGRATION.md section 3). tests/test_gpu_keyed_windows.py builds this file into a shared object linked against libwfb200.so and
// compares wfb_kwin_process_cb / wfb_kwin_flush with its Python model field by field; tools/keyed_windows_bench.py measures them.
//
// The window function is order-sensitive and uses every accessor of Iterable_GPU: a polynomial hash over (id, ivalue) through the
// iterators, size(), operator[](size() / 2), front() and back(), the number of distinct ivalue % 16, and the sum of fvalue in order.
// A window that misses a tuple, holds one of another key, or sees its tuples out of order changes the result.
#include <cstdint>
#include <cstring>
#include "wfb_launch.cuh"
#include "wfb_programs.cuh"

namespace {

constexpr uint64_t MIX = 0x9E3779B97F4A7C15ull, MUL = 0x100000001B3ull;

// the fields every result carries after its key
struct KwFields { uint64_t id, hash, size, mid_id, front_id, back_id, distinct; double fsum; };
struct KwRes64 { uint64_t key; KwFields f; };
struct KwRes80 { wfb_key16_t key; KwFields f; };
static_assert(sizeof(KwRes64) == 72 && sizeof(KwRes80) == 80, "result sizes");

template <class It>
__host__ __device__ inline void win_fields(const It &win, KwFields &f)
{
    uint64_t h = 0; double s = 0.0; uint32_t seen = 0;
    for (auto it = win.begin(); it != win.end(); ++it) {
        h = h * MUL + (it->id * MIX ^ static_cast<uint64_t>(it->ivalue));
        s += it->fvalue;
        seen |= 1u << (static_cast<uint64_t>(it->ivalue) & 15u);
    }
    f.hash = h; f.fsum = s; f.size = win.size();
    f.mid_id = win[win.size() / 2].id; f.front_id = win.front().id; f.back_id = win.back().id;
    f.distinct = static_cast<uint64_t>(__builtin_popcount(seen));
}

// the slots every program carries (the other operators' functors); these programs only use key, make_result and win_func
template <class R>
struct KwBase {
    using tuple_t = wfb_tuple64_t; using result_t = R; using params_t = wfb_functors_t;
    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &, const params_t &) { return true; }
    __host__ __device__ static void lift(const tuple_t &, result_t &r, const params_t &) { r = result_t{}; }
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
    __host__ __device__ static void win_func(const wfb::Iterable_GPU<tuple_t> &win, result_t &r, const params_t &) { win_fields(win, r.f); }
};

// 64-byte bench tuples keyed by their uint64_t key
struct Kw64: KwBase<KwRes64> {
    using key_t = uint64_t;
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &)
    {
        result_t r{}; r.key = k; r.f.id = gwid; return r;
    }
};

// the same tuples keyed by the 16-byte struct {key, low and high half of pad[0]}
struct Kw64K16: KwBase<KwRes80> {
    using key_t = wfb_key16_t;
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &)
    {
        key_t k; k.key = t.key; k.a = static_cast<uint32_t>(t.pad[0]); k.b = static_cast<uint32_t>(t.pad[0] >> 32); return k;
    }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &)
    {
        result_t r{}; r.key = k; r.f.id = gwid; return r;
    }
};

} // namespace

extern "C" {

// 0: 64-byte tuples, uint64_t key -> 72-byte results; 1: 64-byte tuples, 16-byte key -> 80-byte results; -1 for another index
int kw_register(int which)
{
    switch (which) {
    case 0: return wfb::register_program<Kw64>();
    case 1: return wfb::register_program<Kw64K16>();
    }
    return -1;
}

} // extern "C"
