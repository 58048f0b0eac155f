// wf/deferred_counts.hpp -- the words that carry deferred batch sizes from the device to the consumer (include/wf/windflow_gpu.hpp).
//
// A replica whose kernels leave the sizes of its K output batches on the device copies them, once per call, into a BLOCK of pinned
// words and points every output batch at its word; the consumer reads the word in getSize(), on its own thread, any time later. A
// block therefore counts the batches that still point into it (`refs`) and is handed out again only when that count is back to zero:
// however far the producer runs ahead of its consumers, a size is never overwritten before it was read. When the oldest block is still
// referenced the producer does not wait: it takes a fresh one (pinned memory is allocated a slab of blocks at a time, on a miss, and
// kept). The device-side words cycle through a small ring: the replica's stream orders their reuse behind the copy of the call before.
// No CUDA call besides the four allocation calls: the bookkeeping is tested without a device (tests/cpp/test_deferred_counts.cpp).
#pragma once
#include <atomic>
#include <cstddef>
#include <cstdint>
#include <vector>
#include <cuda_runtime_api.h>

namespace wf {

struct CountBlock {
    uint32_t *h = nullptr;             // the call's pinned words
    std::atomic<uint32_t> refs{0};     // holders that have not read their word yet
    void release() { refs.fetch_sub(1, std::memory_order_release); } // (after the holder's read of its word)
};

class DeferredCounts {
    static constexpr size_t SLAB = 64, DEV_BLOCKS = 16;
    size_t words = 0;                  // words per block: the most sizes one call produces
    uint32_t *dev = nullptr; size_t dev_next = 0;
    std::vector<CountBlock *> ring; size_t next = 0; // in the order they are handed out; ring[next] is the oldest
    std::vector<CountBlock *> slabs; std::vector<uint32_t *> pinned;
    cudaError_t grow() // a slab of fresh blocks in front of the oldest one
    {
        uint32_t *h = nullptr;
        const cudaError_t rc = cudaMallocHost(reinterpret_cast<void **>(&h), sizeof(uint32_t) * words * SLAB);
        if (rc != cudaSuccess) return rc;
        CountBlock *s = new CountBlock[SLAB];
        pinned.push_back(h); slabs.push_back(s);
        std::vector<CountBlock *> fresh(SLAB);
        for (size_t i = 0; i < SLAB; i++) { s[i].h = h + i * words; fresh[i] = s + i; }
        ring.insert(ring.begin() + static_cast<std::ptrdiff_t>(next), fresh.begin(), fresh.end());
        return cudaSuccess;
    }
public:
    DeferredCounts() = default;
    DeferredCounts(const DeferredCounts &) = delete;
    DeferredCounts &operator=(const DeferredCounts &) = delete;
    ~DeferredCounts()
    {
        cudaFree(dev);
        for (auto *h : pinned) cudaFreeHost(h);
        for (auto *s : slabs) delete[] s;
    }
    cudaError_t init(size_t words_per_call)
    {
        words = words_per_call ? words_per_call : 1;
        return cudaMalloc(reinterpret_cast<void **>(&dev), sizeof(uint32_t) * words * DEV_BLOCKS);
    }
    // the block of the next call, held by `holders` readers from now on, and the device words the call's kernels write
    cudaError_t acquire(uint32_t holders, CountBlock *&blk, uint32_t *&d)
    {
        if (ring.empty() || ring[next]->refs.load(std::memory_order_acquire) != 0) {
            const cudaError_t rc = grow();
            if (rc != cudaSuccess) return rc;
        }
        blk = ring[next]; next = (next + 1) % ring.size();
        blk->refs.store(holders, std::memory_order_relaxed); // (published with the batches: the queue to the consumer releases)
        d = dev + (dev_next++ % DEV_BLOCKS) * words;
        return cudaSuccess;
    }
    size_t blocks() const { return ring.size(); }
};

} // namespace wf
