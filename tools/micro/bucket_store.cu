// micro-benchmark: the store pattern of the wide partition's scatter (k_wide_scatter_ranked) at the bench step's sizes.
// 2048 wide tiles of 4096 positions, half of them survivors with a uniform slot of 65 536 (digit = slot >> 6, 1024 digits): 4.2 M items.
// Output order is (digit, position), so the cell of (wide tile, digit) holds about 2 items. A CTA owns G consecutive wide tiles; its
// threads sweep the group's cells laid out back to back (digit-major, the G tiles' cells of a digit in tile order) and store every
// item at its final place -- consecutive threads on consecutive entries, as the scatter does. The destinations are precomputed and
// read coalesced (the scatter reads its packed words the same way). Variants: two u32 arrays (slot, position) or one u32 array
// (position << 6 | local key), G = 1, 2, 4, 8. Cold L2: 134 MB (the tile pass's lifted records) are written just before every launch.
#include <cstdio>
#include <cstdint>
#include <vector>
#include <algorithm>
#include <random>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)

template <int ARRAYS>
__global__ void __launch_bounds__(256) k_store(const uint32_t *__restrict__ dst, const uint32_t *__restrict__ gstart, uint32_t *__restrict__ a,
                                               uint32_t *__restrict__ b)
{
    const uint32_t g0 = gstart[blockIdx.x], g1 = gstart[blockIdx.x + 1];
#pragma unroll 4
    for (uint32_t e = g0 + threadIdx.x; e < g1; e += blockDim.x) {
        const uint32_t d = dst[e];
        a[d] = e << 6 | (d & 63u);
        if (ARRAYS == 2) b[d] = e;
    }
}

int main()
{
    constexpr uint32_t TILES = 2048, POS = 4096, DIGITS = 1024;
    std::mt19937 rng(7);
    // per (tile, digit) counts of a uniform stream with selectivity 1/2
    std::vector<uint32_t> cnt(static_cast<size_t>(TILES) * DIGITS, 0);
    uint64_t items = 0;
    for (uint32_t t = 0; t < TILES; t++)
        for (uint32_t p = 0; p < POS; p++)
            if (rng() & 1u) { cnt[static_cast<size_t>(t) * DIGITS + ((rng() & 0xffffu) >> 6)]++; items++; }
    // first output position of (tile, digit): exclusive scan in (digit, tile) order
    std::vector<uint32_t> base(static_cast<size_t>(TILES) * DIGITS);
    uint32_t run = 0;
    for (uint32_t d = 0; d < DIGITS; d++)
        for (uint32_t t = 0; t < TILES; t++) { base[static_cast<size_t>(t) * DIGITS + d] = run; run += cnt[static_cast<size_t>(t) * DIGITS + d]; }
    uint32_t *d_dst, *d_gs, *d_a, *d_b; unsigned char *flush;
    const size_t flush_bytes = 134u << 20;
    CK(cudaMalloc(&d_dst, items * 4)); CK(cudaMalloc(&d_gs, (TILES + 1) * 4)); CK(cudaMalloc(&d_a, items * 4)); CK(cudaMalloc(&d_b, items * 4));
    CK(cudaMalloc(&flush, flush_bytes));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    printf("%llu items over %u wide tiles x %u digits (%.2f per cell)\n", (unsigned long long)items, TILES, DIGITS, double(items) / TILES / DIGITS);
    for (uint32_t G : {1u, 2u, 4u, 8u}) {
        std::vector<uint32_t> dst; dst.reserve(items);
        std::vector<uint32_t> gs;
        for (uint32_t g = 0; g < TILES / G; g++) {
            gs.push_back(static_cast<uint32_t>(dst.size()));
            for (uint32_t d = 0; d < DIGITS; d++)
                for (uint32_t t = g * G; t < (g + 1) * G; t++) {
                    const size_t c = static_cast<size_t>(t) * DIGITS + d;
                    for (uint32_t k = 0; k < cnt[c]; k++) dst.push_back(base[c] + k);
                }
        }
        gs.push_back(static_cast<uint32_t>(dst.size()));
        CK(cudaMemcpy(d_dst, dst.data(), dst.size() * 4, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_gs, gs.data(), gs.size() * 4, cudaMemcpyHostToDevice));
        for (int arrays = 2; arrays >= 1; arrays--) {
            std::vector<float> t_ms;
            for (int rep = 0; rep < 12; rep++) {
                CK(cudaMemset(flush, rep, flush_bytes));
                cudaEventRecord(e0);
                if (arrays == 2) k_store<2><<<TILES / G, 256>>>(d_dst, d_gs, d_a, d_b);
                else k_store<1><<<TILES / G, 256>>>(d_dst, d_gs, d_a, d_b);
                cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
                float ms; cudaEventElapsedTime(&ms, e0, e1);
                if (rep >= 2) t_ms.push_back(ms);
            }
            std::sort(t_ms.begin(), t_ms.end());
            const double med = t_ms[t_ms.size() / 2], bytes = double(items) * (4 + 4 * arrays);
            printf("G = %u (%.1f items per cell), %d u32 array%s, cold L2: median %.1f us, min %.1f us (%.0f GB/s of destinations read + items written)\n",
                   G, double(items) * G / TILES / DIGITS, arrays, arrays == 2 ? "s" : "", med * 1e3, t_ms[0] * 1e3, bytes / med / 1e6);
        }
    }
    { // reference: the same bytes written in order
        std::vector<float> t_ms;
        for (int rep = 0; rep < 12; rep++) {
            CK(cudaMemset(flush, rep, flush_bytes));
            cudaEventRecord(e0); CK(cudaMemsetAsync(d_a, rep, items * 4)); CK(cudaMemsetAsync(d_b, rep, items * 4)); cudaEventRecord(e1);
            CK(cudaEventSynchronize(e1));
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            if (rep >= 2) t_ms.push_back(ms);
        }
        std::sort(t_ms.begin(), t_ms.end());
        printf("memset of the two arrays (%.1f MB), cold L2: median %.1f us\n", items * 8 / 1e6, t_ms[t_ms.size() / 2] * 1e3);
    }
    return 0;
}
