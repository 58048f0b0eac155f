// wfb_scratch.h -- scratch memory that grows on demand: one allocation and its capacity, kept in agreement. Host code only (the
// CUDA runtime API, no nvcc needed).
#ifndef WFB_SCRATCH_H
#define WFB_SCRATCH_H

#include <cuda_runtime_api.h>

namespace wfb {

// what a growth waits for before it frees the old allocation: the streams that may still read it, or the whole device
struct ScratchWaits {
    cudaStream_t s[2] = {nullptr, nullptr};
    int n = 0; // streams in s; -1: the whole device
    ScratchWaits() = default;
    ScratchWaits(cudaStream_t a) : s{a, nullptr}, n(1) {}
    ScratchWaits(cudaStream_t a, cudaStream_t b) : s{a, b}, n(2) {}
    static ScratchWaits device() { ScratchWaits w; w.n = -1; return w; }
};

// capacity() elements of T, used as a T *. The allocation is freed exactly once: by the growth that replaces it or by the destructor
// (the owner's destroy entry point synchronises the device first). A growth that cannot allocate leaves the buffer null with capacity 0,
// so the next ensure() allocates again.
template <class T, cudaError_t (*Alloc)(void **, size_t) = cudaMalloc, cudaError_t (*Free)(void *) = cudaFree>
class Scratch {
public:
    Scratch() = default;
    Scratch(const Scratch &) = delete;
    Scratch &operator=(const Scratch &) = delete;
    Scratch(Scratch &&o) noexcept : p_(o.p_), cap_(o.cap_) { o.p_ = nullptr; o.cap_ = 0; }
    Scratch &operator=(Scratch &&o) noexcept
    {
        if (this != &o) { release(); p_ = o.p_; cap_ = o.cap_; o.p_ = nullptr; o.cap_ = 0; }
        return *this;
    }
    ~Scratch() { release(); }

    operator T *() const { return p_; }
    size_t capacity() const { return cap_; }

    // room for n elements: nothing when they fit; else wait for `waits`, free the old allocation and allocate max(n, want) elements
    // (want = 0: twice the old capacity)
    cudaError_t ensure(size_t n, ScratchWaits waits = ScratchWaits(), size_t want = 0) { return grow(n, waits, want, nullptr); }
    // the same, with the new allocation zero-filled on stream `fill`
    cudaError_t ensure_zeroed(size_t n, cudaStream_t fill, ScratchWaits waits = ScratchWaits(), size_t want = 0) { return grow(n, waits, want, &fill); }

private:
    T *p_ = nullptr;
    size_t cap_ = 0;

    void release()
    {
        if (p_) Free(p_);
        p_ = nullptr; cap_ = 0;
    }
    cudaError_t grow(size_t n, const ScratchWaits &w, size_t want, const cudaStream_t *fill)
    {
        if (n <= cap_) return cudaSuccess;
        cudaError_t e = w.n < 0 ? cudaDeviceSynchronize() : cudaSuccess;
        for (int i = 0; i < w.n && e == cudaSuccess; i++) e = cudaStreamSynchronize(w.s[i]);
        if (e != cudaSuccess) return e; // (the old allocation is still whole)
        if (want == 0) want = 2 * cap_;
        const size_t c = n > want ? n : want;
        release();
        void *p = nullptr;
        e = Alloc(&p, sizeof(T) * c);
        if (e == cudaSuccess && fill) {
            e = cudaMemsetAsync(p, 0, sizeof(T) * c, *fill);
            if (e != cudaSuccess) Free(p);
        }
        if (e != cudaSuccess) { cudaGetLastError(); return e; } // (the error is returned here, not left for a later launch check)
        p_ = static_cast<T *>(p); cap_ = c;
        return cudaSuccess;
    }
};

template <class T> using PinnedScratch = Scratch<T, cudaMallocHost, cudaFreeHost>;

} // namespace wfb

#endif
