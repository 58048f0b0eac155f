// Keyed-stateful FlatMap programs registered at run time, as an application registers its own functors (wfb::register_program,
// INTEGRATION.md section 3). tests/test_gpu_flatmap_stateful.py builds this file into a shared object linked against libwfb200.so,
// compares the programs' host functors with its numpy model, and the GPU's wfb_flatmap_stateful with the same model byte for byte;
// tools/flatmap_stateful_bench.py measures them.
//
// The fan-out of a tuple depends on its key's state: (count + field) % filt_mod, where count is the number of the key's tuples
// before it and field a value of the tuple (map_kind == 1: map_iadd for every tuple instead, so a test can ask for all 0, all m or
// more than m). Record j of a tuple carries (key, tuple id, j, h), h being a position-weighted sum over the key's history before the
// tuple: a wrong per-key order, a lost state or a state shared by two keys changes the bytes.
#include <cstdint>
#include <cstring>
#include <map>
#include <utility>
#include "wfb_launch.cuh"
#include "wfb_programs.cuh"

namespace {

struct SfmState { uint64_t count, h; };
struct Rec32 { uint64_t key, id, j, h; };
struct Rec48 { uint64_t key, id, j, h, count, x; };
static_assert(sizeof(Rec32) == 32 && sizeof(Rec48) == 48 && sizeof(SfmState) == 16, "record sizes");
constexpr uint64_t MIX = 0x9E3779B97F4A7C15ull;

__host__ __device__ inline uint64_t fanout(const SfmState &st, uint64_t field, const wfb_functors_t &p)
{
    return p.map_kind == 1 ? static_cast<uint64_t>(p.map_iadd) : (st.count + field) % static_cast<uint64_t>(p.filt_mod);
}
__host__ __device__ inline void advance(SfmState &st, uint64_t id) { st.h += id * MIX * (st.count + 1); st.count++; }

// the slots every program with a state_t carries (the keyed Map / Filter walks); these programs only use flatmap_stateful
template <class T, class R>
struct SfmBase {
    using tuple_t = T; using result_t = R; using params_t = wfb_functors_t; using state_t = SfmState;
    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &, const params_t &) { return true; }
    __host__ __device__ static void lift(const tuple_t &, result_t &r, const params_t &) { r = result_t{}; }
    __host__ __device__ static void comb(const result_t &, const result_t &, result_t &, const params_t &) {}
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &, const params_t &) { return a; }
    __host__ __device__ static void map_stateful(tuple_t &, state_t &, const params_t &) {}
    __host__ __device__ static bool filter_stateful(tuple_t &, state_t &, const params_t &) { return true; }
};

// 64-byte tuples -> 32-byte records, integer key
struct Sfm64to32: SfmBase<wfb_tuple64_t, Rec32> {
    using key_t = uint64_t;
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t{}; }
    __host__ __device__ static void flatmap_stateful(const tuple_t &t, wfb::Shipper<result_t> &sh, state_t &st, const params_t &p)
    {
        const uint64_t c = fanout(st, static_cast<uint64_t>(t.ivalue), p);
        for (uint64_t j = 0; j < c; j++) sh.push(Rec32{t.key, t.id, j, st.h});
        advance(st, t.id);
    }
};

// 16-byte tuples {key, value} -> 48-byte records (the value is the tuple's id)
struct Sfm16to48: SfmBase<wfb_wftest16_t, Rec48> {
    using key_t = uint64_t;
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t{}; }
    __host__ __device__ static void flatmap_stateful(const tuple_t &t, wfb::Shipper<result_t> &sh, state_t &st, const params_t &p)
    {
        const uint64_t id = static_cast<uint64_t>(t.value);
        const uint64_t c = fanout(st, id, p);
        for (uint64_t j = 0; j < c; j++) sh.push(Rec48{t.key, id, j, st.h, st.count, t.key ^ st.h});
        advance(st, id);
    }
};

// 64-byte tuples keyed by the 16-byte struct {key, low and high half of pad[0]} -> 32-byte records
struct Sfm64K16: SfmBase<wfb_tuple64_t, Rec32> {
    using key_t = wfb_key16_t;
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &)
    {
        key_t k; k.key = t.key; k.a = static_cast<uint32_t>(t.pad[0]); k.b = static_cast<uint32_t>(t.pad[0] >> 32); return k;
    }
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t{}; }
    __host__ __device__ static void flatmap_stateful(const tuple_t &t, wfb::Shipper<result_t> &sh, state_t &st, const params_t &p)
    {
        const uint64_t c = fanout(st, static_cast<uint64_t>(t.ivalue), p);
        for (uint64_t j = 0; j < c; j++) sh.push(Rec32{t.key ^ t.pad[0], t.id, j, st.h});
        advance(st, t.id);
    }
};

// 64-byte tuples -> the tuple iff ProgTuple64::filter_stateful holds (which updates the tuple and the key's counter): with m = 1 this
// is wfb_filter_stateful of the built-in program
struct SfmSelect64: SfmBase<wfb_tuple64_t, wfb_tuple64_t> {
    using key_t = uint64_t; using state_t = wfb_state8_t;
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static result_t make_result(key_t, uint64_t, const params_t &) { return result_t{}; }
    __host__ __device__ static void map_stateful(tuple_t &, state_t &, const params_t &) {}
    __host__ __device__ static bool filter_stateful(tuple_t &, state_t &, const params_t &) { return true; }
    __host__ __device__ static void flatmap_stateful(const tuple_t &t, wfb::Shipper<result_t> &sh, state_t &st, const params_t &p)
    {
        tuple_t u = t;
        if (wfb::ProgTuple64::filter_stateful(u, st, p)) sh.push(u);
    }
};

// the operator on the host, tuple after tuple with one state per key (std::map over the key's bytes), records at consecutive positions
template <class P>
void host_run(const wfb_functors_t &f, const void *tuples, const uint64_t *ts, uint64_t n, uint32_t m, void *out, uint64_t *ts_out,
              uint64_t *n_out, uint64_t *dropped)
{
    using K = typename P::key_t;
    const typename P::tuple_t *in = static_cast<const typename P::tuple_t *>(tuples);
    std::map<std::pair<uint64_t, uint64_t>, typename P::state_t> states;
    uint64_t pos = 0, drop = 0;
    for (uint64_t i = 0; i < n; i++) {
        const K k = P::key(in[i], f);
        uint64_t w[2] = {0, 0};
        std::memcpy(w, &k, sizeof(K));
        auto it = states.find({w[0], w[1]});
        if (it == states.end()) { typename P::state_t z; std::memset(&z, 0, sizeof(z)); it = states.emplace(std::make_pair(w[0], w[1]), z).first; }
        wfb::Shipper<typename P::result_t> sh(static_cast<unsigned char *>(out) + pos * sizeof(typename P::result_t),
                                              ts_out != nullptr ? ts_out + pos : nullptr, ts != nullptr ? ts[i] : 0, m);
        P::flatmap_stateful(in[i], sh, it->second, f);
        const uint32_t c = sh.pushes();
        pos += c < m ? c : m; drop += c > m ? c - m : 0;
    }
    *n_out = pos; *dropped = drop;
}

} // namespace

extern "C" {

// 0: 64 -> 32 bytes, 1: 16 -> 48, 2: 64 -> 32 with a 16-byte key, 3: 64 -> 64 (selection); the program id, or -1 for another index
int sfm_register(int which)
{
    switch (which) {
    case 0: return wfb::register_program<Sfm64to32>();
    case 1: return wfb::register_program<Sfm16to48>();
    case 2: return wfb::register_program<Sfm64K16>();
    case 3: return wfb::register_program<SfmSelect64>();
    }
    return -1;
}

int sfm_host(int which, const wfb_functors_t *f, const void *tuples, const uint64_t *ts, uint64_t n, uint32_t m, void *out, uint64_t *ts_out,
             uint64_t *n_out, uint64_t *dropped)
{
    switch (which) {
    case 0: host_run<Sfm64to32>(*f, tuples, ts, n, m, out, ts_out, n_out, dropped); return 0;
    case 1: host_run<Sfm16to48>(*f, tuples, ts, n, m, out, ts_out, n_out, dropped); return 0;
    case 2: host_run<Sfm64K16>(*f, tuples, ts, n, m, out, ts_out, n_out, dropped); return 0;
    case 3: host_run<SfmSelect64>(*f, tuples, ts, n, m, out, ts_out, n_out, dropped); return 0;
    }
    return -1;
}

} // extern "C"
