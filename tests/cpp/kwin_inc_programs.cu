// Incremental Keyed_Windows_GPU programs registered at run time, as an application registers its own functors (wfb::register_program,
// INTEGRATION.md section 3). tests/test_gpu_keyed_windows_inc.py builds this file into a shared object linked against libwfb200.so and
// compares wfb_kwin_process_cb / wfb_kwin_flush on WFB_KWIN_INCREMENTAL handles with its Python model field by field;
// tools/keyed_windows_bench.py measures them.
//
// win_func_inc is an order-sensitive fold: a polynomial hash over (id, ivalue), the size, the first and last id, the mask of the
// ivalue % 16 seen, the sum of fvalue in arrival order, and the id of the FIRST tuple with the largest ivalue. A window that misses a
// tuple, folds one of another key, or folds them out of order changes the result. Every program also defines win_func, the same
// fields computed over the whole window, so that one program drives an incremental and a non-incremental handle.
#include <cstdint>
#include <cstring>
#include "wfb_launch.cuh"
#include "wfb_programs.cuh"

namespace {

constexpr uint64_t MIX = 0x9E3779B97F4A7C15ull, MUL = 0x100000001B3ull;

// the fields every result carries after its key
struct IncFields { uint64_t id, hash, size, front_id, back_id, mask; double fsum; uint64_t argmax_id; int64_t max_ivalue; };
struct IncRes64 { uint64_t key; IncFields f; };
struct IncRes88 { wfb_key16_t key; IncFields f; };
static_assert(sizeof(IncRes64) == 80 && sizeof(IncRes88) == 88, "result sizes");

// 256-byte records: the large-record path (pad_sum folds the tuple's last word, so the whole record travels)
struct Tuple256 { uint64_t key, id; int64_t ivalue; double fvalue; uint64_t pad[28]; };
struct IncRes256 { uint64_t key; IncFields f; uint64_t pad_sum; uint64_t pad[21]; };
static_assert(sizeof(Tuple256) == 256 && sizeof(IncRes256) == 256, "record sizes");

template <class T>
__host__ __device__ inline void fold(const T &t, IncFields &f)
{
    if (f.size == 0 || t.ivalue > f.max_ivalue) { f.max_ivalue = t.ivalue; f.argmax_id = t.id; }
    if (f.size == 0) f.front_id = t.id;
    f.hash = f.hash * MUL + (t.id * MIX ^ static_cast<uint64_t>(t.ivalue));
    f.size++;
    f.back_id = t.id;
    f.mask |= 1ull << (static_cast<uint64_t>(t.ivalue) & 15u);
    f.fsum += t.fvalue;
}

template <class Tup, class R>
struct IncBase {
    using tuple_t = Tup; using result_t = R; using params_t = wfb_functors_t;
    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &, const params_t &) { return true; }
    __host__ __device__ static void lift(const tuple_t &, result_t &r, const params_t &) { r = result_t{}; }
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
    __host__ __device__ static void win_func_inc(const tuple_t &t, result_t &r, const params_t &) { fold(t, r.f); }
    __host__ __device__ static void win_func(const wfb::Iterable_GPU<tuple_t> &win, result_t &r, const params_t &)
    {
        for (auto it = win.begin(); it != win.end(); ++it) fold(*it, r.f);
    }
};

// 64-byte bench tuples keyed by their uint64_t key
struct Inc64: IncBase<wfb_tuple64_t, IncRes64> {
    using key_t = uint64_t;
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &) { result_t r{}; r.key = k; r.f.id = gwid; return r; }
};

// the same tuples keyed by the 16-byte struct {key, low and high half of pad[0]}
struct Inc64K16: IncBase<wfb_tuple64_t, IncRes88> {
    using key_t = wfb_key16_t;
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &)
    {
        key_t k; k.key = t.key; k.a = static_cast<uint32_t>(t.pad[0]); k.b = static_cast<uint32_t>(t.pad[0] >> 32); return k;
    }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &) { result_t r{}; r.key = k; r.f.id = gwid; return r; }
};

// 256-byte tuples and results keyed by their uint64_t key
struct Inc256: IncBase<Tuple256, IncRes256> {
    using key_t = uint64_t;
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &) { result_t r{}; r.key = k; r.f.id = gwid; return r; }
    __host__ __device__ static void win_func_inc(const tuple_t &t, result_t &r, const params_t &) { fold(t, r.f); r.pad_sum += t.pad[27]; }
    __host__ __device__ static void win_func(const wfb::Iterable_GPU<tuple_t> &win, result_t &r, const params_t &p)
    {
        for (auto it = win.begin(); it != win.end(); ++it) win_func_inc(*it, r, p);
    }
};

// a program with win_func only: an incremental handle refuses it
struct NonInc64: Inc64 {
    static void win_func_inc() = delete;
};

} // namespace

extern "C" {

// 0: 64-byte tuples, uint64_t key -> 80-byte results; 1: 64-byte tuples, 16-byte key -> 88-byte results; 2: 256-byte tuples and
// results; 3: program 0 without win_func_inc; -1 for another index
int kwi_register(int which)
{
    switch (which) {
    case 0: return wfb::register_program<Inc64>();
    case 1: return wfb::register_program<Inc64K16>();
    case 2: return wfb::register_program<Inc256>();
    case 3: return wfb::register_program<NonInc64>();
    }
    return -1;
}

} // extern "C"
