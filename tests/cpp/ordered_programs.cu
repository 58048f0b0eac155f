// Window programs with an order-sensitive combine, registered at run time as an application registers its own functors
// (wfb::register_program, INTEGRATION.md section 3). tests/test_gpu_ordered_windows.py builds this file into a shared object linked
// against libwfb200.so and compares the windows with a direct fold of every key's items in arrival order.
//
// Payload (h, q) and combine (h1, q1) o (h2, q2) = (h1 (q2 + 1) + h2, (q1 + 1)(q2 + 1) - 1), wrapping unsigned arithmetic: a polynomial
// hash with multiplier M, the length of the folded sequence carried as q = M^len - 1. It is associative and not commutative, all-zero
// bits are its identity (the trees and panes start zeroed, make_result starts a window with a zero payload), and any reordering,
// duplication or omission of items changes it. M (odd) is the program's params_t, set with wfb_ffat_set_params /
// wfb_engine_set_params: a kernel launched without the handle's params folds with M = 0 and shows.
#include <cstdint>
#include "wfb_launch.cuh"

namespace {

struct OrdParams { uint64_t M; };

struct Ord24 { uint64_t key; uint64_t id; uint32_t h, q; };                     // arithmetic mod 2^32
struct Ord32 { uint64_t key; uint64_t id; uint64_t h, q; };                     // mod 2^64
struct Ord48 { wfb_key16_t key; uint64_t id; uint64_t h, q; uint64_t pad; };    // 16-byte key, mod 2^64
static_assert(sizeof(Ord24) == 24 && sizeof(Ord32) == 32 && sizeof(Ord48) == 48, "record sizes");

// nonzero item hash of the tuple's id and key words
__host__ __device__ inline uint64_t ord_mix(uint64_t id, uint64_t k0, uint64_t k1)
{
    uint64_t x = ((id + 1) * 0x9E3779B97F4A7C15ull) ^ (k0 * 0xC2B2AE3D27D4EB4Full) ^ (k1 * 0x165667B19E3779F9ull);
    x ^= x >> 29;
    return x | 1u;
}

template <class W>
__host__ __device__ inline void ord_comb(W h1, W q1, W h2, W q2, W &ho, W &qo)
{
    const W h = static_cast<W>(h1 * static_cast<W>(q2 + 1u) + h2);
    const W q = static_cast<W>(static_cast<W>(q1 + 1u) * static_cast<W>(q2 + 1u) - 1u);
    ho = h; qo = q; // (after both reads: out may alias either operand)
}

template <class R, class K, class W>
struct OrdProgram {
    using tuple_t = wfb_tuple64_t;
    using result_t = R;
    using key_t = K;
    using params_t = OrdParams;

    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &t, const params_t &) { return t.id % 7 != 3; } // gaps in every batch
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &)
    {
        if constexpr (sizeof(K) == 8) return t.key;
        else { K k; k.key = t.key; k.a = static_cast<uint32_t>(t.pad[0]); k.b = static_cast<uint32_t>(t.pad[0] >> 32); return k; }
    }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &p)
    {
        r = result_t{};
        r.key = key(t, p); r.id = 0;
        r.h = static_cast<W>(ord_mix(t.id, t.key, sizeof(K) == 8 ? 0ull : t.pad[0]));
        r.q = static_cast<W>(p.M - 1u);
    }
    __host__ __device__ static void comb(const result_t &a, const result_t &b, result_t &out, const params_t &)
    {
        W h, q;
        ord_comb<W>(a.h, a.q, b.h, b.q, h, q);
        out.h = h; out.q = q;
    }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &)
    {
        result_t r{}; r.key = k; r.id = gwid; return r;
    }
    // Reduce_GPU: the same combine over (h, q) = (ivalue, pad[1]) of the tuples; the rest of the first tuple is kept
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &b, const params_t &)
    {
        tuple_t r = a;
        uint64_t h, q;
        ord_comb<uint64_t>(static_cast<uint64_t>(a.ivalue), a.pad[1], static_cast<uint64_t>(b.ivalue), b.pad[1], h, q);
        r.ivalue = static_cast<int64_t>(h); r.pad[1] = q;
        return r;
    }
};

using Prog24 = OrdProgram<Ord24, uint64_t, uint32_t>;
using Prog32 = OrdProgram<Ord32, uint64_t, uint64_t>;
using Prog48 = OrdProgram<Ord48, wfb_key16_t, uint64_t>;

template <class P>
void comb_arrays(uint64_t M, const uint64_t *h1, const uint64_t *q1, const uint64_t *h2, const uint64_t *q2, uint64_t *ho, uint64_t *qo,
                 uint64_t n, int alias)
{
    const OrdParams prm{M};
    for (uint64_t i = 0; i < n; i++) {
        typename P::result_t a{}, b{}, o{};
        a.h = h1[i]; a.q = q1[i]; b.h = h2[i]; b.q = q2[i];
        if (alias) { P::comb(a, b, a, prm); o = a; } else P::comb(a, b, o, prm);
        ho[i] = o.h; qo[i] = o.q;
    }
}

template <class P>
void lift_arrays(uint64_t M, const wfb_tuple64_t *t, uint64_t n, uint64_t *h, uint64_t *q, uint8_t *keep)
{
    const OrdParams prm{M};
    for (uint64_t i = 0; i < n; i++) {
        wfb_tuple64_t c = t[i];
        typename P::result_t r{};
        P::lift(c, r, prm);
        h[i] = r.h; q[i] = r.q; keep[i] = P::filter(c, prm) ? 1 : 0;
    }
}

} // namespace

extern "C" {

int ord_register_24() { return wfb::register_program<Prog24>(); }
int ord_register_32() { return wfb::register_program<Prog32>(); }
int ord_register_48() { return wfb::register_program<Prog48>(); }

// the programs' comb / lift / filter on the host (rec: record size 24, 32 or 48); -1 for another size
int ord_comb_host(int rec, uint64_t M, const uint64_t *h1, const uint64_t *q1, const uint64_t *h2, const uint64_t *q2, uint64_t *ho, uint64_t *qo,
                  uint64_t n, int alias)
{
    if (rec == 24) comb_arrays<Prog24>(M, h1, q1, h2, q2, ho, qo, n, alias);
    else if (rec == 32) comb_arrays<Prog32>(M, h1, q1, h2, q2, ho, qo, n, alias);
    else if (rec == 48) comb_arrays<Prog48>(M, h1, q1, h2, q2, ho, qo, n, alias);
    else return -1;
    return 0;
}

int ord_lift_host(int rec, uint64_t M, const void *tuples, uint64_t n, uint64_t *h, uint64_t *q, uint8_t *keep)
{
    const wfb_tuple64_t *t = static_cast<const wfb_tuple64_t *>(tuples);
    if (rec == 24) lift_arrays<Prog24>(M, t, n, h, q, keep);
    else if (rec == 32) lift_arrays<Prog32>(M, t, n, h, q, keep);
    else if (rec == 48) lift_arrays<Prog48>(M, t, n, h, q, keep);
    else return -1;
    return 0;
}

} // extern "C"
