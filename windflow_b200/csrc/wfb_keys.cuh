// wfb_keys.cuh -- the canonical words of a program's key_t. Every kernel that needs a key goes through KeyCodec: the key table
// stores these words, window results decode them back to key_t, and Reduce_GPU sorts on their order transform.
//   integral / enum   one word: static_cast<uint64_t>(key)
//   float / double    one word: the bit pattern (zero-extended for float), -0.0 stored as +0.0 and every NaN as one quiet NaN,
//                     so that keys equal under == share one state (DESIGN.md section 5: NaN keys)
//   other types       trivially copyable, at most 16 bytes, std::has_unique_object_representations (no padding, no floating-point
//                     members: comparing bytes is comparing members): the bytes, zero-padded to one word (<= 8 bytes) or two
// The all-ones pattern (every word 2^64-1) is reserved as the empty marker of the key table.
#pragma once
#include <cstdint>
#include <cstring>
#include <type_traits>

namespace wfb {

// a key of 9-16 bytes: lo = bytes 0-7, hi = bytes 8-15 (zero-padded)
struct alignas(16) Key128 { uint64_t lo, hi; };
__host__ __device__ __forceinline__ bool operator==(const Key128 &a, const Key128 &b) { return a.lo == b.lo && a.hi == b.hi; }
__host__ __device__ __forceinline__ bool operator!=(const Key128 &a, const Key128 &b) { return !(a == b); }
__host__ __device__ __forceinline__ uint64_t key_word0(uint64_t w) { return w; }
__host__ __device__ __forceinline__ uint64_t key_word0(const Key128 &w) { return w.lo; }

enum : uint32_t { KEY_KIND_INTEGRAL = 0, KEY_KIND_FLOATING = 1, KEY_KIND_BYTES = 2 }; // wfb_program_info_t::key_kind

template <class K>
struct KeyCodec {
    static constexpr bool integral = (std::is_integral<K>::value || std::is_enum<K>::value) && sizeof(K) <= 8;
    static constexpr bool floating = std::is_same<K, float>::value || std::is_same<K, double>::value;
    static constexpr bool bytes = !std::is_integral<K>::value && !std::is_enum<K>::value && !std::is_floating_point<K>::value &&
                                  std::is_trivially_copyable<K>::value && std::has_unique_object_representations<K>::value && sizeof(K) <= 16;
    static_assert(integral || floating || bytes,
                  "WindFlow Compilation Error - the key type of a GPU operator must be an integral or enum type, float, double, or a "
                  "trivially copyable type of at most 16 bytes without padding or floating-point members "
                  "(std::has_unique_object_representations):\n");
    static constexpr uint32_t words = sizeof(K) > 8 ? 2u : 1u;
    static constexpr uint32_t kind = integral ? KEY_KIND_INTEGRAL : (floating ? KEY_KIND_FLOATING : KEY_KIND_BYTES);
    using words_t = std::conditional_t<words == 1, uint64_t, Key128>;

    __host__ __device__ __forceinline__ static words_t encode(const K &k)
    {
        if constexpr (integral) return static_cast<uint64_t>(k);
        else if constexpr (std::is_same<K, double>::value) {
            if (k != k) return 0x7ff8000000000000ull;
            const double d = (k == 0.0) ? 0.0 : k;
            uint64_t u; std::memcpy(&u, &d, sizeof(u)); return u;
        } else if constexpr (std::is_same<K, float>::value) {
            if (k != k) return 0x7fc00000ull;
            const float f = (k == 0.0f) ? 0.0f : k;
            uint32_t u; std::memcpy(&u, &f, sizeof(u)); return u;
        } else {
            words_t w{};
            std::memcpy(&w, &k, sizeof(K));
            return w;
        }
    }
    __host__ __device__ __forceinline__ static K decode(const words_t &w)
    {
        if constexpr (integral) return static_cast<K>(w);
        else if constexpr (std::is_same<K, float>::value) { const uint32_t u = static_cast<uint32_t>(w); K k; std::memcpy(&k, &u, sizeof(k)); return k; }
        else { K k; std::memcpy(&k, &w, sizeof(K)); return k; }
    }
    // the words as unsigned integers whose ascending order is the order Reduce_GPU emits: numeric for floating-point keys (non-negatives
    // get the sign bit set, negatives are inverted; the canonical NaN sorts last), the words themselves otherwise
    __host__ __device__ __forceinline__ static words_t order(const words_t &w)
    {
        if constexpr (std::is_same<K, double>::value) return (w >> 63) ? ~w : (w | 0x8000000000000000ull);
        else if constexpr (std::is_same<K, float>::value) return (w >> 31) ? (~w & 0xffffffffull) : (w | 0x80000000ull);
        else return w;
    }
};

} // namespace wfb
