// wfb_ptx.cuh -- sm_90a inline-PTX helpers: mbarrier, TMA bulk copies (cp.async.bulk -> SASS UBLKCP),
// scoped loads/stores for decoupled look-back. No CUTLASS/CuTe dependency.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace wfb {

__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier --------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    while (!mbar_try_wait(bar, parity)) { }
}

// ---- TMA 1-D bulk copies ---------------------------------------------------------------------------
// global -> shared, completion signalled on an mbarrier (bytes % 16 == 0, both addresses 16-B aligned)
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// ---- LDGSTS: asynchronous global -> shared copies of one thread (no registers in between) -------------------------------
template <int BYTES>
__device__ __forceinline__ void cp_async(void *smem_dst, const void *gmem_src)
{
    static_assert(BYTES == 4 || BYTES == 8 || BYTES == 16, "cp.async copies 4, 8 or 16 bytes");
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "n"(BYTES) : "memory");
}
// the same, 16 bytes, bypassing L1: a copy in flight holds no L1 line (random gathers with many copies in flight per SM)
__device__ __forceinline__ void cp_async_cg16(void *smem_dst, const void *gmem_src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); } // at most N groups of this thread pending

// ---- L2 eviction-priority policies (createpolicy) and the TMA copies that carry them -----------------------------------
__device__ __forceinline__ uint64_t l2_policy_evict_first()
{
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last()
{
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p;
}
__device__ __forceinline__ void bulk_g2s_hint(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar, uint64_t policy)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}
__device__ __forceinline__ void bulk_s2g_hint(void *gmem_dst, const void *smem_src, uint32_t bytes, uint64_t policy)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
                 ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes), "l"(policy) : "memory");
}
// shared -> global (bulk async-group completion)
__device__ __forceinline__ void bulk_s2g(void *gmem_dst, const void *smem_src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// make generic-proxy shared-memory writes visible to the async proxy (before a bulk store reads them)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- scoped global accesses for inter-CTA flags ----------------------------------------------------
__device__ __forceinline__ uint64_t ld_relaxed_u64(const uint64_t *p)
{
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u64(uint64_t *p, uint64_t v)
{
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t ld_acquire_u64(const uint64_t *p)
{
    uint64_t v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t *p, uint32_t v)
{
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// one 16-byte load of two words (not guaranteed single-copy atomic: a concurrent 16-byte CAS may be seen half written)
__device__ __forceinline__ void ld_relaxed_v2u64(const uint64_t *p, uint64_t &lo, uint64_t &hi)
{
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(lo), "=l"(hi) : "l"(p) : "memory");
}
// 16-byte compare-and-swap (sm_90): returns the words found at p
__device__ __forceinline__ void atom_cas_b128(uint64_t *p, uint64_t cmp_lo, uint64_t cmp_hi, uint64_t val_lo, uint64_t val_hi,
                                              uint64_t &old_lo, uint64_t &old_hi)
{
    asm volatile("{\n\t.reg .b128 c, v, d;\n\t"
                 "mov.b128 c, {%2, %3};\n\t"
                 "mov.b128 v, {%4, %5};\n\t"
                 "atom.relaxed.gpu.global.cas.b128 d, [%6], c, v;\n\t"
                 "mov.b128 {%0, %1}, d;\n\t}"
                 : "=l"(old_lo), "=l"(old_hi)
                 : "l"(cmp_lo), "l"(cmp_hi), "l"(val_lo), "l"(val_hi), "l"(p)
                 : "memory");
}

// streaming (read-once) 128-bit global load / store
__device__ __forceinline__ uint4 ld_stream_u4(const void *p)
{
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_stream_u4(void *p, uint4 v)
{
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }
__device__ __forceinline__ uint32_t lanemask_lt()
{
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

} // namespace wfb
