// Unit test of windflow_b200/csrc/wfb_scratch.h (the grow-on-demand scratch buffers of libwfb200) on the CPU: the CUDA runtime calls
// the header makes are stubbed below, log every call and can fail the next allocation.
// Build: g++ -std=c++17 -I$CUDA_HOME/include -I windflow_b200/csrc tests/cpp/test_scratch.cpp -o test_scratch (no libcudart)
#include "wfb_scratch.h"
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <set>
#include <string>
#include <utility>
#include <vector>

#define CHECK(c) do { if (!(c)) { std::fprintf(stderr, "CHECK failed: %s (line %d)\n", #c, __LINE__); std::exit(1); } } while (0)

namespace {
std::vector<std::string> calls;   // every runtime call, in order
std::set<uintptr_t> live_dev, live_host;
uintptr_t next_addr = 0x10000;
cudaError_t fail_next_alloc = cudaSuccess, fail_next_memset = cudaSuccess, last_error = cudaSuccess;
int bad_frees = 0;

std::string hex(uintptr_t v) { char b[32]; std::snprintf(b, sizeof(b), "%llx", static_cast<unsigned long long>(v)); return b; }
std::string hex(const void *p) { return hex(reinterpret_cast<uintptr_t>(p)); }

cudaError_t alloc(std::set<uintptr_t> &live, const char *name, void **p, size_t bytes)
{
    calls.push_back(std::string(name) + " " + std::to_string(bytes));
    if (fail_next_alloc != cudaSuccess) { const cudaError_t e = fail_next_alloc; fail_next_alloc = cudaSuccess; last_error = e; return e; }
    *p = reinterpret_cast<void *>(next_addr); live.insert(next_addr); next_addr += 0x10000;
    return cudaSuccess;
}
cudaError_t release(std::set<uintptr_t> &live, const char *name, void *p)
{
    calls.push_back(std::string(name) + " " + hex(p));
    if (live.erase(reinterpret_cast<uintptr_t>(p)) != 1) bad_frees++; // never allocated, or freed already
    return cudaSuccess;
}
} // namespace

extern "C" {
cudaError_t cudaMalloc(void **p, size_t bytes) { return alloc(live_dev, "malloc", p, bytes); }
cudaError_t cudaFree(void *p) { return release(live_dev, "free", p); }
cudaError_t cudaMallocHost(void **p, size_t bytes) { return alloc(live_host, "mallochost", p, bytes); }
cudaError_t cudaFreeHost(void *p) { return release(live_host, "freehost", p); }
cudaError_t cudaStreamSynchronize(cudaStream_t s) { calls.push_back("sync " + hex(s)); return cudaSuccess; }
cudaError_t cudaDeviceSynchronize(void) { calls.push_back("devsync"); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void *p, int v, size_t bytes, cudaStream_t s)
{
    calls.push_back("memset " + hex(p) + " " + std::to_string(v) + " " + std::to_string(bytes) + " " + hex(s));
    if (fail_next_memset != cudaSuccess) { const cudaError_t e = fail_next_memset; fail_next_memset = cudaSuccess; last_error = e; return e; }
    return cudaSuccess;
}
cudaError_t cudaGetLastError(void) { calls.push_back("getlasterror"); const cudaError_t e = last_error; last_error = cudaSuccess; return e; }
}

using wfb::Scratch;
using wfb::PinnedScratch;
using wfb::ScratchWaits;

static std::vector<std::string> take() { std::vector<std::string> c; c.swap(calls); return c; }
static bool log_is(const std::vector<std::string> &want) { const std::vector<std::string> got = take(); if (got == want) return true;
    for (const std::string &g : got) std::fprintf(stderr, "  got: %s\n", g.c_str());
    for (const std::string &w : want) std::fprintf(stderr, "  want: %s\n", w.c_str());
    return false; }

int main()
{
    const cudaStream_t s1 = reinterpret_cast<cudaStream_t>(0x51), s2 = reinterpret_cast<cudaStream_t>(0x52);
    {   // 1. the first allocation, then calls within the capacity make no runtime call
        Scratch<uint32_t> b;
        CHECK(static_cast<uint32_t *>(b) == nullptr && b.capacity() == 0);
        CHECK(b.ensure(100, s1) == cudaSuccess);
        CHECK(b.capacity() == 100 && static_cast<uint32_t *>(b) != nullptr);
        CHECK(log_is({"sync 51", "malloc 400"}));
        CHECK(b.ensure(100, s1) == cudaSuccess && b.ensure(1, ScratchWaits(s1, s2)) == cudaSuccess && b.ensure(0) == cudaSuccess);
        CHECK(b.ensure_zeroed(50, s2, s1) == cudaSuccess);
        CHECK(log_is({}));
        CHECK(b.capacity() == 100);

        // 2. growth: every given stream is waited for before the old allocation is freed (once), then max(n, 2 * capacity) elements
        const uintptr_t old = reinterpret_cast<uintptr_t>(static_cast<uint32_t *>(b));
        CHECK(b.ensure(150, ScratchWaits(s1, s2)) == cudaSuccess);
        CHECK(log_is({"sync 51", "sync 52", "free " + hex(old), "malloc 800"}));
        CHECK(b.capacity() == 200);
        CHECK(b.ensure(1000, s2) == cudaSuccess); // more than twice the capacity: n
        CHECK(b.capacity() == 1000);
        const std::string cur = hex(static_cast<uint32_t *>(b));
        take();
        CHECK(b.ensure(1001, ScratchWaits::device()) == cudaSuccess); // the whole device instead of streams
        CHECK(b.capacity() == 2000);
        CHECK(log_is({"devsync", "free " + cur, "malloc 8000"}));
    }
    CHECK(live_dev.empty() && bad_frees == 0); // the destructor freed the last allocation, once
    take();
    {   // a capacity the caller asks for, and no stream to wait for
        Scratch<uint64_t> b;
        CHECK(b.ensure(3, ScratchWaits(), 64) == cudaSuccess);
        CHECK(b.capacity() == 64);
        CHECK(log_is({"malloc 512"}));
        CHECK(b.ensure(65, s1, 65) == cudaSuccess);
        CHECK(b.capacity() == 65);
        CHECK(b.ensure(66, s1, 10) == cudaSuccess); // (never less than n)
        CHECK(b.capacity() == 66);
        take();
    }
    take();
    {   // zero-filled growth: the new allocation, all of it, on the given stream
        Scratch<uint64_t> b;
        CHECK(b.ensure_zeroed(10, s2, s1) == cudaSuccess);
        const std::string p = hex(static_cast<uint64_t *>(b));
        CHECK(log_is({"sync 51", "malloc 80", "memset " + p + " 0 80 52"}));
        CHECK(b.ensure_zeroed(11, s2) == cudaSuccess);
        const std::string q = hex(static_cast<uint64_t *>(b));
        CHECK(log_is({"free " + p, "malloc 160", "memset " + q + " 0 160 52"}));
    }
    CHECK(live_dev.empty() && bad_frees == 0);
    take();
    {   // 3. a failed allocation: the error, the buffer null with capacity 0, the old allocation freed once; then a smaller call allocates
        Scratch<uint32_t> b;
        CHECK(b.ensure(100, s1) == cudaSuccess);
        const std::string old = hex(static_cast<uint32_t *>(b));
        take();
        fail_next_alloc = cudaErrorMemoryAllocation;
        CHECK(b.ensure(300, s1) == cudaErrorMemoryAllocation);
        CHECK(static_cast<uint32_t *>(b) == nullptr && b.capacity() == 0);
        CHECK(log_is({"sync 51", "free " + old, "malloc 1200", "getlasterror"}));
        CHECK(last_error == cudaSuccess); // (the error is returned, not left for the next launch check to find)
        CHECK(live_dev.empty() && bad_frees == 0);
        CHECK(b.ensure(10, s1) == cudaSuccess);
        CHECK(b.capacity() == 10 && static_cast<uint32_t *>(b) != nullptr);
        CHECK(log_is({"sync 51", "malloc 40"}));
        // a failed zero fill: the new allocation is freed as well
        const std::string cur = hex(static_cast<uint32_t *>(b));
        fail_next_memset = cudaErrorInvalidValue;
        CHECK(b.ensure_zeroed(20, s2) == cudaErrorInvalidValue);
        CHECK(static_cast<uint32_t *>(b) == nullptr && b.capacity() == 0);
        const std::vector<std::string> c = take();
        CHECK(c.size() == 5 && c[0] == "free " + cur && c[1] == "malloc 80" && c[2].rfind("memset ", 0) == 0 && c[3].rfind("free ", 0) == 0 &&
              c[4] == "getlasterror");
        CHECK(live_dev.empty() && bad_frees == 0);
    }
    // 4. ... and its destructor, after the failure, frees nothing
    CHECK(log_is({}));
    {   // the destructor frees a live allocation once
        Scratch<unsigned char> b;
        CHECK(b.ensure(7) == cudaSuccess);
        take();
    }
    CHECK(calls.size() == 1 && calls[0].rfind("free ", 0) == 0 && live_dev.empty() && bad_frees == 0);
    take();
    {   // 5. a moved-from buffer frees nothing; a move assignment frees what the target held
        Scratch<uint32_t> a;
        CHECK(a.ensure(8) == cudaSuccess);
        const std::string pa = hex(static_cast<uint32_t *>(a));
        {
            Scratch<uint32_t> b(std::move(a));
            CHECK(static_cast<uint32_t *>(a) == nullptr && a.capacity() == 0 && b.capacity() == 8 && hex(static_cast<uint32_t *>(b)) == pa);
            Scratch<uint32_t> c;
            CHECK(c.ensure(4) == cudaSuccess);
            const std::string pc = hex(static_cast<uint32_t *>(c));
            take();
            c = std::move(b);
            CHECK(log_is({"free " + pc}));
            CHECK(c.capacity() == 8 && hex(static_cast<uint32_t *>(c)) == pa && static_cast<uint32_t *>(b) == nullptr);
        } // c frees pa; b frees nothing
        CHECK(log_is({"free " + pa}));
    } // a frees nothing
    CHECK(log_is({}));
    CHECK(live_dev.empty() && bad_frees == 0);
    {   // pinned host memory: the same rules over cudaMallocHost / cudaFreeHost
        PinnedScratch<unsigned char> h;
        CHECK(h.ensure(100, ScratchWaits(), 8192) == cudaSuccess);
        CHECK(h.capacity() == 8192);
        const std::string p = hex(static_cast<unsigned char *>(h));
        CHECK(log_is({"mallochost 8192"}));
        fail_next_alloc = cudaErrorMemoryAllocation;
        CHECK(h.ensure(9000, ScratchWaits(), 18000) == cudaErrorMemoryAllocation);
        CHECK(static_cast<unsigned char *>(h) == nullptr && h.capacity() == 0);
        CHECK(log_is({"freehost " + p, "mallochost 18000", "getlasterror"}));
        CHECK(h.ensure(9000, ScratchWaits(), 18000) == cudaSuccess);
        take();
    }
    CHECK(calls.size() == 1 && calls[0].rfind("freehost ", 0) == 0);
    CHECK(live_dev.empty() && live_host.empty() && bad_frees == 0);
    std::printf("scratch OK\n");
    return 0;
}
