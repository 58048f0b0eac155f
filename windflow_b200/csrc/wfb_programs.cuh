// wfb_programs.cuh -- the built-in "programs": record schemas + functors compiled into libwfb200.so.
//
// A program is a traits struct with
//   tuple_t, result_t, key_t, params_t (functor objects / parameters, passed by value to kernels)
//   (key_t: an integral or enum type, float, double, or a trivially copyable type of at most 16 bytes without padding or
//    floating-point members; wfb_keys.cuh maps it to the words the key table stores)
//   map(tuple_t&, params)            Map_GPU functor      __host__ __device__ void(tuple_t &)           (API:50-52)
//   filter(tuple_t&, params)->bool   Filter_GPU functor   __host__ __device__ bool(tuple_t &)           (API:34-36)
//   key(const tuple_t&, params)->key_t       key extractor    __host__ __device__ key_t(const tuple_t &)    (API:213)
//   lift(const tuple_t&, result_t&, params)  FFAT lift        (API:150-151)
//   comb(a, b, out, params)                  FFAT combine (associative; must tolerate out aliasing a)  (API:153-154)
//   make_result(key, gwid, params)           result_t(key, gwid) constructor (wf/basic_gpu.hpp:236-247)
//   reduce(t1, t2, params)->tuple_t          Reduce_GPU functor   (API:78-79)
// (every function receives the program's params_t, i.e. the functor objects, which the kernels carry by value)
// User code writes the same struct around its own functors and instantiates the kernels with
// WFB_DEFINE_PROGRAM (wfb_kernels.cuh); see INTEGRATION.md.
#pragma once
#include <cstdint>
#include <cstring>
#include "../../include/wfb200.h"

namespace wfb {

// ---- program 0: bench stream of SURVEY.md 8d --------------------------------------------------------
struct ProgTuple64 {
    using tuple_t = wfb_tuple64_t;
    using result_t = wfb_result32_t;
    using key_t = uint64_t;
    using params_t = wfb_functors_t;
    static constexpr int id = WFB_PROG_TUPLE64;

    __host__ __device__ static void map(tuple_t &t, const params_t &p)
    {
        if (p.map_kind == 1) { t.ivalue += p.map_iadd; t.fvalue *= p.map_fscale; }
    }
    __host__ __device__ static bool filter(tuple_t &t, const params_t &p)
    {
        if (p.filt_kind == 1) return (t.ivalue & 1) == 0;
        if (p.filt_kind == 2) return (t.ivalue % p.filt_mod) == 0;
        return true;
    }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &)
    {
        r.key = t.key; r.id = 0; r.isum = t.ivalue; r.fsum = t.fvalue;
    }
    __host__ __device__ static void comb(const result_t &a, const result_t &b, result_t &out, const params_t &)
    {
        int64_t is = a.isum + b.isum; double fs = a.fsum + b.fsum;
        out.isum = is; out.fsum = fs;
    }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &)
    {
        result_t r; r.key = k; r.id = gwid; r.isum = 0; r.fsum = 0.0; return r;
    }
    __host__ __device__ static key_t result_key(const result_t &r, const params_t &) { return r.key; } // (optional: lets lifted records travel, wfb_mg_*)
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &b, const params_t &)
    {
        tuple_t r; r.key = a.key; r.id = 0; r.ivalue = a.ivalue + b.ivalue; r.fvalue = a.fvalue + b.fvalue;
        r.pad[0] = r.pad[1] = r.pad[2] = r.pad[3] = 0; return r;
    }
    // keyed-stateful Map_GPU / Filter_GPU functors (API:54-56, :38-40): a running counter per key
    using state_t = wfb_state8_t;
    __host__ __device__ static void map_stateful(tuple_t &t, state_t &st, const params_t &p)
    {
        if (p.map_kind == 2 && (t.key & 1)) st.counter--; else st.counter++;
        t.ivalue += st.counter;
    }
    __host__ __device__ static bool filter_stateful(tuple_t &t, state_t &st, const params_t &p)
    {
        st.counter++; t.ivalue += st.counter;
        if (p.filt_kind == 1) return (t.ivalue & 1) == 0;
        if (p.filt_kind == 2) return (t.ivalue % p.filt_mod) == 0;
        return true;
    }
};

// ---- program 1: reference tests/graph_tests_gpu/graph_common_gpu.hpp ({key, value}) ------------------
struct ProgWfTest16 {
    using tuple_t = wfb_wftest16_t;
    using result_t = wfb_wfwin24_t; // windows over this schema reuse the {key,id,value} result
    using key_t = uint64_t;
    using params_t = wfb_functors_t;
    static constexpr int id = WFB_PROG_WFTEST16;

    __host__ __device__ static void map(tuple_t &t, const params_t &p)          // Map_Functor_GPU :245-253
    {
        if (p.map_kind == 1) t.value += p.map_iadd;
    }
    __host__ __device__ static bool filter(tuple_t &t, const params_t &p)       // Filter_Functor_GPU :198-215
    {
        if (p.filt_kind == 1) return (t.value & 1) == 0;
        if (p.filt_kind == 2) return (t.value % p.filt_mod) == 0;
        return true;
    }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &) { r.key = t.key; r.id = 0; r.value = t.value; }
    __host__ __device__ static void comb(const result_t &a, const result_t &b, result_t &out, const params_t &) { out.value = a.value + b.value; }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &) { result_t r; r.key = k; r.id = gwid; r.value = 0; return r; }
    __host__ __device__ static key_t result_key(const result_t &r, const params_t &) { return r.key; }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &b, const params_t &) // Reduce_Functor_GPU :268-279
    {
        tuple_t r; r.key = a.key; r.value = a.value + b.value; return r;
    }
    // Map_Functor_GPU_KB :256-265 (kind 1) / tests/merge_tests_gpu/merge_common_gpu_kb.hpp:153-168 (kind 2, on the key's parity),
    // Filter_Functor_GPU_KB :221-231 (kind 0 keeps everything, as the reference's does)
    using state_t = wfb_state8_t;
    __host__ __device__ static void map_stateful(tuple_t &t, state_t &st, const params_t &p)
    {
        if (p.map_kind == 2 && (t.key & 1)) st.counter--; else st.counter++;
        t.value += st.counter;
    }
    __host__ __device__ static bool filter_stateful(tuple_t &t, state_t &st, const params_t &p)
    {
        st.counter++; t.value += st.counter;
        if (p.filt_kind == 1) return (t.value & 1) == 0;
        if (p.filt_kind == 2) return (t.value % p.filt_mod) == 0;
        return true;
    }
};

// ---- program 2: reference tests/win_tests_gpu/win_common_gpu.hpp ({key, id, value}) ------------------
struct ProgWfWin24 {
    using tuple_t = wfb_wfwin24_t;
    using result_t = wfb_wfwin24_t;
    using key_t = uint64_t;
    using params_t = wfb_functors_t;
    static constexpr int id = WFB_PROG_WFWIN24;

    __host__ __device__ static void map(tuple_t &t, const params_t &p)          // Map_Functor_GPU :221-229
    {
        if (p.map_kind == 1) t.value += p.map_iadd;
    }
    __host__ __device__ static bool filter(tuple_t &t, const params_t &p)       // Filter_Functor :190-203
    {
        if (p.filt_kind == 1) return (t.value & 1) == 0;
        if (p.filt_kind == 2) return (t.value % p.filt_mod) == 0;
        return true;
    }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &) { r.key = t.key; r.id = 0; r.value = t.value; } // :295-303
    __host__ __device__ static void comb(const result_t &a, const result_t &b, result_t &out, const params_t &) { out.value = a.value + b.value; } // :306-314
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &) { result_t r; r.key = k; r.id = gwid; r.value = 0; return r; }
    __host__ __device__ static key_t result_key(const result_t &r, const params_t &) { return r.key; }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &b, const params_t &)
    {
        tuple_t r; r.key = a.key; r.id = 0; r.value = a.value + b.value; return r;
    }
};

// ---- program 3: already-lifted bench records (multi-GPU keyby: the source GPU ran Map -> Filter -> lift and shipped
// 32-byte results; the destination GPU only looks up the key slot and runs the window operator) -----------------
struct ProgLifted32 {
    using tuple_t = wfb_result32_t;
    using result_t = wfb_result32_t;
    using key_t = uint64_t;
    using params_t = wfb_functors_t;
    static constexpr int id = WFB_PROG_LIFTED32;
    static constexpr bool is_lifted = true;    // (no lifted variant of a lifted program)
    static constexpr bool passthrough = true; // map is a no-op and lift the identity: the window operator may read the records in place

    __host__ __device__ static void map(tuple_t &, const params_t &) {}
    __host__ __device__ static bool filter(tuple_t &, const params_t &) { return true; }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &) { return t.key; }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &) { r = t; }
    __host__ __device__ static void comb(const result_t &a, const result_t &b, result_t &out, const params_t &p) { ProgTuple64::comb(a, b, out, p); }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &p) { return ProgTuple64::make_result(k, gwid, p); }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &b, const params_t &)
    {
        tuple_t r; r.key = a.key; r.id = 0; r.isum = a.isum + b.isum; r.fsum = a.fsum + b.fsum; return r;
    }
};

// ---- programs 4 and 5: the bench stream keyed by a double / by a 16-byte struct -------------------------------------------------
// The functors of ProgTuple64 over the same tuples; only the key extractor and the result record differ (and reduce keeps pad[0],
// which holds part of the key).
template <class K, class R, int ID>
struct ProgTuple64Keyed {
    using tuple_t = wfb_tuple64_t;
    using result_t = R;
    using key_t = K;
    using params_t = wfb_functors_t;
    using state_t = wfb_state8_t;
    static constexpr int id = ID;
    __host__ __device__ static void map(tuple_t &t, const params_t &p) { ProgTuple64::map(t, p); }
    __host__ __device__ static bool filter(tuple_t &t, const params_t &p) { return ProgTuple64::filter(t, p); }
    __host__ __device__ static key_t key(const tuple_t &t, const params_t &)
    {
        if constexpr (sizeof(K) == 8) { K k; std::memcpy(&k, &t.pad[0], sizeof(k)); return k; } // the double whose bits are pad[0]
        else { K k; k.key = t.key; k.a = static_cast<uint32_t>(t.pad[0]); k.b = static_cast<uint32_t>(t.pad[0] >> 32); return k; }
    }
    __host__ __device__ static void lift(const tuple_t &t, result_t &r, const params_t &p)
    {
        r.key = key(t, p); r.id = 0; r.isum = t.ivalue; r.fsum = t.fvalue;
    }
    __host__ __device__ static void comb(const result_t &a, const result_t &b, result_t &out, const params_t &)
    {
        int64_t is = a.isum + b.isum; double fs = a.fsum + b.fsum;
        out.isum = is; out.fsum = fs;
    }
    __host__ __device__ static result_t make_result(key_t k, uint64_t gwid, const params_t &)
    {
        result_t r{}; r.key = k; r.id = gwid; r.isum = 0; r.fsum = 0.0; return r;
    }
    __host__ __device__ static tuple_t reduce(const tuple_t &a, const tuple_t &b, const params_t &p)
    {
        tuple_t r = ProgTuple64::reduce(a, b, p); r.pad[0] = a.pad[0]; return r;
    }
    __host__ __device__ static void map_stateful(tuple_t &t, state_t &st, const params_t &p) { ProgTuple64::map_stateful(t, st, p); }
    __host__ __device__ static bool filter_stateful(tuple_t &t, state_t &st, const params_t &p) { return ProgTuple64::filter_stateful(t, st, p); }
};
using ProgTuple64FKey = ProgTuple64Keyed<double, wfb_result32d_t, WFB_PROG_TUPLE64_FKEY>;
using ProgTuple64K16 = ProgTuple64Keyed<wfb_key16_t, wfb_result48k_t, WFB_PROG_TUPLE64_K16>;

} // namespace wfb
