// A window program whose combine reads its params, registered at run time as an application registers its own functors
// (wfb::register_program, INTEGRATION.md section 3). tests/test_gpu_ordered_params.py and tests/test_gpu_mg_step.py build this file into a
// shared object linked against libwfb200.so.
//
// It folds the polynomial hash of tests/cpp/ordered_programs.cu with the multiplier M read in the combine instead of the lift:
// (h1, q1) o (h2, q2) = (h1 M^q2 + h2, q1 + q2), wrapping 64-bit arithmetic, q the length of the folded sequence (lift: q = 1). Its h
// therefore equals the 32-byte program's there, and all-zero bits are its identity. M (odd) is the program's params_t, set with
// wfb_ffat_set_params / wfb_engine_set_params / wfb_mg_set_params: a window-update kernel launched without the handle's params folds
// with M^q2 = 0 and keeps only the right operand's h. result_key lets its lifted records travel through the key-sharded step (wfb_mg_*).
#include <cstdint>
#include "wfb_launch.cuh"

namespace {

struct OrdParams { uint64_t M; };
struct Ord32 { uint64_t key; uint64_t id; uint64_t h, q; };
static_assert(sizeof(Ord32) == 32, "record size");

// nonzero item hash of the tuple's id and key (the 32-byte program's of ordered_programs.cu)
__host__ __device__ inline uint64_t ord_mix(uint64_t id, uint64_t k0)
{
    uint64_t x = ((id + 1) * 0x9E3779B97F4A7C15ull) ^ (k0 * 0xC2B2AE3D27D4EB4Full);
    x ^= x >> 29;
    return x | 1u;
}

__host__ __device__ inline uint64_t ord_pow(uint64_t b, uint64_t e)
{
    uint64_t r = 1;
    for (; e; e >>= 1, b *= b)
        if (e & 1) r *= b;
    return r;
}

struct Prog32P {
    using tuple_t = wfb_tuple64_t;
    using result_t = Ord32;
    using key_t = uint64_t;
    using params_t = OrdParams;

    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &t, const params_t &) { return t.id % 7 != 3; } // gaps in every batch
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &)
    {
        r = result_t{};
        r.key = t.key; r.id = 0; r.h = ord_mix(t.id, t.key); r.q = 1;
    }
    __host__ __device__ static void comb(const result_t &a, const result_t &b, result_t &out, const params_t &p)
    {
        const uint64_t h = a.h * ord_pow(p.M, b.q) + b.h, q = a.q + b.q;
        out.h = h; out.q = q; // (after both reads: out may alias either operand)
    }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &)
    {
        result_t r{}; r.key = k; r.id = gwid; return r;
    }
    __host__ __device__ static key_t result_key(const result_t &r, const params_t &) { return r.key; }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
};

} // namespace

extern "C" {

int ord32p_register() { return wfb::register_program<Prog32P>(); }

// the program's comb (out aliasing the left operand when alias != 0) and lift / filter on the host
void ord32p_comb_host(uint64_t M, const uint64_t *h1, const uint64_t *q1, const uint64_t *h2, const uint64_t *q2, uint64_t *ho, uint64_t *qo,
                      uint64_t n, int alias)
{
    const OrdParams prm{M};
    for (uint64_t i = 0; i < n; i++) {
        Ord32 a{}, b{}, o{};
        a.h = h1[i]; a.q = q1[i]; b.h = h2[i]; b.q = q2[i];
        if (alias) { Prog32P::comb(a, b, a, prm); o = a; } else Prog32P::comb(a, b, o, prm);
        ho[i] = o.h; qo[i] = o.q;
    }
}

void ord32p_lift_host(uint64_t M, const void *tuples, uint64_t n, uint64_t *h, uint64_t *q, uint8_t *keep)
{
    const OrdParams prm{M};
    const wfb_tuple64_t *t = static_cast<const wfb_tuple64_t *>(tuples);
    for (uint64_t i = 0; i < n; i++) {
        wfb_tuple64_t c = t[i];
        Ord32 r{};
        Prog32P::lift(c, r, prm);
        h[i] = r.h; q[i] = r.q; keep[i] = Prog32P::filter(c, prm) ? 1 : 0;
    }
}

} // extern "C"
