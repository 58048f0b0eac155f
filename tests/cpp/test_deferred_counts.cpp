// Unit test of include/wf/deferred_counts.hpp (the blocks of pinned words that carry deferred batch sizes) on the CPU: the four CUDA
// allocation calls the header makes are stubbed below. A block is handed out again only when nobody holds it; when the oldest block is
// still held the next call gets a fresh one (one pinned allocation per slab of blocks), never a wait and never a held block.
// Build: g++ -std=c++17 -I$CUDA_HOME/include -I include tests/cpp/test_deferred_counts.cpp -o test_deferred_counts (no libcudart)
#include "wf/deferred_counts.hpp"
#include <cstdio>
#include <cstdlib>
#include <set>

#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "CHECK failed: %s (line %d)\n", #c, __LINE__); std::exit(1); } } while (0)

namespace {
int host_allocs = 0, dev_allocs = 0, frees = 0, bad_frees = 0;
std::set<void *> live;
cudaError_t fail_next = cudaSuccess;
cudaError_t alloc(void **p, size_t bytes, int &n)
{
    if (fail_next != cudaSuccess) { const cudaError_t e = fail_next; fail_next = cudaSuccess; return e; }
    *p = std::malloc(bytes); live.insert(*p); n++;
    return cudaSuccess;
}
cudaError_t release(void *p)
{
    if (p == nullptr) return cudaSuccess;
    if (live.erase(p) != 1) bad_frees++; else { std::free(p); frees++; }
    return cudaSuccess;
}
} // namespace

extern "C" {
cudaError_t cudaMalloc(void **p, size_t bytes) { return alloc(p, bytes, dev_allocs); }
cudaError_t cudaFree(void *p) { return release(p); }
cudaError_t cudaMallocHost(void **p, size_t bytes) { return alloc(p, bytes, host_allocs); }
cudaError_t cudaFreeHost(void *p) { return release(p); }
}

using wf::CountBlock;
using wf::DeferredCounts;

int main()
{
    {
        DeferredCounts c;
        CHECK(c.init(4) == cudaSuccess && dev_allocs == 1 && host_allocs == 0);
        CountBlock *b; uint32_t *d, *d0 = nullptr;
        // a consumer that keeps up: the first slab serves every call, the device words cycle
        std::set<uint32_t *> words;
        for (int i = 0; i < 1000; i++) {
            CHECK(c.acquire(3, b, d) == cudaSuccess && b->refs.load() == 3);
            if (i == 0) d0 = d;
            if (i == 16) CHECK(d == d0);
            words.insert(b->h);
            for (int j = 0; j < 4; j++) b->h[j] = 0; // (the whole block is this call's)
            b->release(); b->release(); b->release();
        }
        CHECK(host_allocs == 1 && c.blocks() == 64 && words.size() == 64);
        // a consumer that falls behind: held blocks are never handed out, fresh ones are allocated a slab at a time
        std::set<CountBlock *> held;
        for (int i = 0; i < 300; i++) {
            CHECK(c.acquire(2, b, d) == cudaSuccess);
            CHECK(held.insert(b).second);
            b->h[0] = static_cast<uint32_t>(i); b->release(); // one of the two holders reads at once
        }
        CHECK(host_allocs == 5 && c.blocks() == 320);
        for (auto *h : held) CHECK(h->refs.load() == 1);
        // the consumer catches up, oldest first: the blocks serve again without another allocation
        for (auto *h : held) h->release();
        std::set<CountBlock *> again;
        for (int i = 0; i < 320; i++) { CHECK(c.acquire(1, b, d) == cudaSuccess); CHECK(again.insert(b).second); b->release(); }
        CHECK(host_allocs == 5 && c.blocks() == 320);
        // the oldest still held, younger ones free: a fresh slab goes in front of it and the held one keeps its word
        CHECK(c.acquire(1, b, d) == cudaSuccess);
        CountBlock *old = b; old->h[0] = 77;
        for (int i = 0; i < 319; i++) { CHECK(c.acquire(1, b, d) == cudaSuccess); b->release(); }
        CHECK(c.acquire(1, b, d) == cudaSuccess && b != old && host_allocs == 6 && old->h[0] == 77);
        b->release();
        // a failed pinned allocation is reported and leaves the object usable
        for (int i = 0; i < 63; i++) { CHECK(c.acquire(1, b, d) == cudaSuccess); CHECK(b != old); b->release(); }
        fail_next = cudaErrorMemoryAllocation;
        CHECK(c.acquire(1, b, d) == cudaErrorMemoryAllocation);
        old->release();
        CHECK(c.acquire(1, b, d) == cudaSuccess && b == old);
    }
    CHECK(live.empty() && bad_frees == 0 && frees == 7);
    std::printf("deferred counts OK\n");
    return 0;
}
