// Programs of one shape at many record sizes, registered at run time as an application registers its own functors
// (wfb::register_program, INTEGRATION.md section 3). tests/test_gpu_record_sizes.py builds this file into a shared object linked
// against libwfb200.so and compares every GPU operator with a direct fold of each key's items in arrival order.
//
// Geo<TB, RB, SB>: tuple_t of TB bytes, result_t of RB bytes, state_t of SB bytes. The kernels branch on these sizes (16-byte or
// 8-byte tile access, bulk or word copies, items per thread, cp.async granule, staged FlatFAT levels, tile-pass stages), so every
// geometry takes a different set of branches. Every byte of every record is checked:
//  - tuple {key, id, pad[]} (TB = 8: a 32-bit key and id); map rewrites every pad word from itself, the key and the id;
//  - result {key, id, h, q, pad[]} (RB = 16: 32-bit words, no pad). Window combine: (h, q) is the polynomial hash of
//    ordered_programs.cu, (h1, q1) o (h2, q2) = (h1 (q2 + 1) + h2, (q1 + 1)(q2 + 1) - 1), associative, not commutative, zero its
//    identity; the pad words add up. lift copies the tuple's pad words into the result's pad, so a torn or short copy shows;
//  - state {h, pad[]} (SB = 4: a 32-bit h): h = h * M + item hash (a running hash of the key's items), pad[i] += id * (2i + 1) + key.
//    The stateful functors write the state into the tuple (TB = 8: into id), so every intermediate state reaches the output; the
//    stateful filter keeps a tuple when bits 13-14 of the new h are not both zero.
//  - Reduce_GPU: (pad[0], pad[1]) fold with the same hash, pad[2..] add up, key and id of the first item (TB = 8: id holds a 16-bit
//    (h, q) pair).
#include <cstdint>
#include <unordered_map>
#include "wfb_launch.cuh"

namespace {

struct GeoParams { uint64_t M; };

template <uint32_t TB> struct GTuple { uint64_t key, id; uint64_t pad[(TB - 16) / 8]; };
template <> struct GTuple<8> { uint32_t key, id; };
template <uint32_t RB> struct GResult { uint64_t key, id, h, q; uint64_t pad[(RB - 32) / 8]; };
template <> struct GResult<16> { uint32_t key, id, h, q; };
template <uint32_t SB> struct GState { uint64_t h; uint64_t pad[(SB - 8) / 8]; };
template <> struct GState<8> { uint64_t h; };
template <> struct GState<4> { uint32_t h; };

__host__ __device__ inline uint64_t geo_mix(uint64_t id, uint64_t key)
{
    uint64_t x = ((id + 1) * 0x9E3779B97F4A7C15ull) ^ (key * 0xC2B2AE3D27D4EB4Full);
    x ^= x >> 29;
    return x | 1u;
}

template <class W>
__host__ __device__ inline void geo_comb(W h1, W q1, W h2, W q2, W &ho, W &qo)
{
    const W h = static_cast<W>(h1 * static_cast<W>(q2 + 1u) + h2);
    const W q = static_cast<W>(static_cast<W>(q1 + 1u) * static_cast<W>(q2 + 1u) - 1u);
    ho = h; qo = q;
}

template <uint32_t TB_, uint32_t RB_, uint32_t SB_>
struct Geo {
    static constexpr uint32_t TB = TB_, RB = RB_, SB = SB_;
    static constexpr uint32_t TP = TB == 8 ? 0 : (TB - 16) / 8; // pad words of a tuple / result / state
    static constexpr uint32_t RP = RB == 16 ? 0 : (RB - 32) / 8;
    static constexpr uint32_t SP = SB <= 8 ? 0 : (SB - 8) / 8;
    static_assert(TB == 8 || TP >= 2, "Reduce and the stateful functors use pad[0] and pad[1]");
    static_assert(RB == 16 || RP == 0 || TP > 0, "lift fills the result pad from the tuple pad");
    using tuple_t = GTuple<TB>;
    using result_t = GResult<RB>;
    using state_t = GState<SB>;
    using key_t = uint64_t;
    using params_t = GeoParams;
    using WR = std::conditional_t<RB == 16, uint32_t, uint64_t>; // hash words of the result
    using WS = std::conditional_t<SB == 4, uint32_t, uint64_t>;  // hash word of the state
    static_assert(sizeof(tuple_t) == TB && sizeof(result_t) == RB && sizeof(state_t) == SB, "record sizes");

    __host__ __device__ static void map(tuple_t &t, const params_t &)
    {
        if constexpr (TP > 0) {
            for (uint32_t j = 0; j < TP; j++) t.pad[j] = (t.pad[j] ^ (t.key * 0xD6E8FEB86659FD93ull)) + (j + 1) * t.id;
        }
    }
    __host__ __device__ static bool filter(tuple_t &t, const params_t &) { return t.id % 7 != 3; }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &p)
    {
        r = result_t{};
        r.key = t.key; r.id = 0;
        r.h = static_cast<WR>(geo_mix(t.id, t.key));
        r.q = static_cast<WR>(p.M - 1u);
        if constexpr (RP > 0) {
            for (uint32_t i = 0; i < RP; i++) r.pad[i] = t.pad[i % TP] + i;
        }
    }
    __host__ __device__ static void comb(const result_t &a, const result_t &b, result_t &out, const params_t &)
    {
        WR h, q;
        geo_comb<WR>(a.h, a.q, b.h, b.q, h, q);
        if constexpr (RP > 0) {
            for (uint32_t i = 0; i < RP; i++) { const uint64_t s = a.pad[i] + b.pad[i]; out.pad[i] = s; } // (element i of out read before written)
        }
        out.h = h; out.q = q;
    }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &)
    {
        result_t r{};
        r.key = static_cast<decltype(r.key)>(k); r.id = static_cast<decltype(r.id)>(gwid);
        return r;
    }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &b, const params_t &)
    {
        tuple_t r = a;
        if constexpr (TB == 8) { // id = (h, q) of 16 bits each
            uint16_t h, q;
            geo_comb<uint16_t>(static_cast<uint16_t>(a.id), static_cast<uint16_t>(a.id >> 16), static_cast<uint16_t>(b.id),
                               static_cast<uint16_t>(b.id >> 16), h, q);
            r.id = static_cast<uint32_t>(h) | (static_cast<uint32_t>(q) << 16);
        } else {
            geo_comb<uint64_t>(a.pad[0], a.pad[1], b.pad[0], b.pad[1], r.pad[0], r.pad[1]);
            for (uint32_t j = 2; j < TP; j++) r.pad[j] = a.pad[j] + b.pad[j];
        }
        return r;
    }
    __host__ __device__ static void map_stateful(tuple_t &t, state_t &st, const params_t &p)
    {
        st.h = static_cast<WS>(st.h * static_cast<WS>(p.M) + static_cast<WS>(geo_mix(t.id, t.key)));
        if constexpr (SP > 0) {
            for (uint32_t i = 0; i < SP; i++) st.pad[i] += t.id * (2 * i + 1) + t.key;
        }
        if constexpr (TB == 8) t.id = static_cast<uint32_t>(st.h);
        else {
            t.pad[0] = st.h;
            for (uint32_t j = 1; j < TP; j++) t.pad[j] += st.h * j;
            if constexpr (SP > 0) {
                for (uint32_t i = 0; i < SP; i++) t.pad[1 + i % (TP - 1)] ^= st.pad[i];
            }
        }
    }
    __host__ __device__ static bool filter_stateful(tuple_t &t, state_t &st, const params_t &p)
    {
        map_stateful(t, st, p);
        return ((st.h >> 13) & 3u) != 0;
    }
    // FlatMap_GPU: id % 3 records per tuple, record j = lift(tuple) with id = j
    __host__ __device__ static void flatmap(const tuple_t &t, wfb::Shipper<result_t> &sh, const params_t &p)
    {
        for (uint32_t j = 0; j < t.id % 3; j++) {
            result_t r;
            lift(t, r, p);
            r.id = static_cast<decltype(r.id)>(j);
            sh.push(r);
        }
    }
};

// ---- host side: the functors over arrays, and what the launch tables derive from the record sizes ----------------------------
template <class G>
int host_op(int op, uint64_t M, void *a, const void *b, void *out, uint64_t n)
{
    using T = typename G::tuple_t; using R = typename G::result_t; using S = typename G::state_t;
    const GeoParams prm{M};
    T *t = static_cast<T *>(a);
    switch (op) {
    case 0: for (uint64_t i = 0; i < n; i++) G::map(t[i], prm); return 0;                                   // map, in place
    case 1: for (uint64_t i = 0; i < n; i++) static_cast<uint8_t *>(out)[i] = G::filter(t[i], prm); return 0; // filter flags
    case 2: for (uint64_t i = 0; i < n; i++) G::lift(t[i], static_cast<R *>(out)[i], prm); return 0;          // lift
    case 3: for (uint64_t i = 0; i < n; i++) G::comb(static_cast<R *>(a)[i], static_cast<const R *>(b)[i], static_cast<R *>(out)[i], prm); return 0;
    case 4: for (uint64_t i = 0; i < n; i++) G::comb(static_cast<R *>(a)[i], static_cast<const R *>(b)[i], static_cast<R *>(a)[i], prm); return 0; // out = a
    case 5: for (uint64_t i = 0; i < n; i++) static_cast<T *>(out)[i] = G::reduce(t[i], static_cast<const T *>(b)[i], prm); return 0;
    case 6: case 7: { // keyed-stateful map / filter over the sequence (per-key states from zero), in place; filter: flags into out
        std::unordered_map<uint64_t, S> states;
        for (uint64_t i = 0; i < n; i++) {
            auto it = states.find(static_cast<uint64_t>(t[i].key));
            if (it == states.end()) it = states.emplace(static_cast<uint64_t>(t[i].key), S{}).first;
            if (op == 6) G::map_stateful(t[i], it->second, prm);
            else static_cast<uint8_t *>(out)[i] = G::filter_stateful(t[i], it->second, prm);
        }
        return 0;
    }
    }
    return -1;
}

template <class G>
void info(uint32_t *o)
{
    using L = wfb::LiftedOf<G>;
    o[0] = G::TB; o[1] = G::RB; o[2] = G::SB;
    o[3] = wfb::TilePassSmem<G, wfb::MODE_MAP>::total; o[4] = wfb::TilePassSmem<G, wfb::MODE_FILTER>::total;
    o[5] = wfb::TilePassSmem<G, wfb::MODE_INGEST>::total; o[6] = wfb::TilePassSmem<G, wfb::MODE_FLATMAP>::total;
    o[7] = wfb::TilePassSmem<L, wfb::MODE_INGEST>::total;
    o[8] = wfb::TilePassSmem<G, wfb::MODE_MAP>::stages; o[9] = wfb::TilePassSmem<G, wfb::MODE_FILTER>::stages;
    o[10] = wfb::TilePassSmem<G, wfb::MODE_INGEST>::stages; o[11] = wfb::TilePassSmem<G, wfb::MODE_FLATMAP>::stages;
    o[12] = wfb::TilePassSmem<L, wfb::MODE_INGEST>::stages;
    o[13] = wfb::bk_fits<G::RB>() ? 1u : 0u; o[14] = wfb::TP_SMEM_MAX;
    o[15] = wfb::bk_smem_bytes<G::RB, false>(); o[16] = wfb::bk_smem_bytes<G::RB, true>();
}

using G0 = Geo<8, 16, 4>;
using G1 = Geo<40, 40, 8>;
using G2 = Geo<72, 56, 40>;
using G3 = Geo<128, 128, 128>;
using G4 = Geo<136, 160, 136>;
using G5 = Geo<256, 256, 16>;

} // namespace

extern "C" {

#define GEO_SWITCH(g, EXPR) \
    switch (g) { case 0: { using G = G0; EXPR; } case 1: { using G = G1; EXPR; } case 2: { using G = G2; EXPR; } \
                 case 3: { using G = G3; EXPR; } case 4: { using G = G4; EXPR; } case 5: { using G = G5; EXPR; } }

int geo_count() { return 6; }
// program id of geometry g (>= 6), or a negative error
int geo_register(int g) { GEO_SWITCH(g, return wfb::register_program<G>()); return -1; }
// what the launch tables derive from the record sizes (17 words, see info())
int geo_info(int g, uint32_t *out) { GEO_SWITCH(g, info<G>(out); return 0); return -1; }
// the functors on the host (op: see host_op)
int geo_host(int g, int op, uint64_t M, void *a, const void *b, void *out, uint64_t n) { GEO_SWITCH(g, return host_op<G>(op, M, a, b, out, n)); return -1; }

} // extern "C"
