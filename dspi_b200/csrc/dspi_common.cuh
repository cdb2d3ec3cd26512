// dspi_common.cuh — sm_90a device helpers: mbarrier, TMA (cp.async.bulk.tensor), proxies.
#pragma once
#ifdef __CUDACC_RTC__
// runtime compilation (eq_jit.cu): no host headers; the tensor map is an opaque 128-byte parameter
typedef unsigned char uint8_t;
typedef unsigned short uint16_t;
typedef unsigned int uint32_t;
typedef int int32_t;
typedef unsigned long long uint64_t;
typedef long long int64_t;
typedef unsigned long long size_t_rtc;
struct alignas(64) CUtensorMap { unsigned long long opaque[16]; };
#else
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#endif

namespace dspi {

__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

// make mbarrier initialisation visible to the async (TMA) proxy
__device__ __forceinline__ void fence_mbar_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// generic-proxy smem writes -> visible to the async proxy (needed before a TMA store reads them)
__device__ __forceinline__ void fence_proxy_async_smem()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}

// 2-D tiled TMA load: box at element coordinates (x = innermost, y) -> smem, completes on `bar`
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int32_t x, int32_t y)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(x), "r"(y)
        : "memory");
}

// 1-D bulk load: `bytes` contiguous bytes global -> smem, completes on `bar`.  Both addresses and the size are multiples of 16.
__device__ __forceinline__ void bulk_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gsrc),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// 1-D bulk store: `bytes` contiguous bytes smem -> global, tracked by the issuing thread's bulk async-group.  Same multiples of 16.
__device__ __forceinline__ void bulk_store_1d(void *gdst, const void *smem_src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}

// 2-D tiled TMA store: smem -> box at (x, y); tracked by the issuing thread's bulk async-group
__device__ __forceinline__ void tma_store_2d(const CUtensorMap *map, const void *smem_src, int32_t x, int32_t y)
{
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(map)),
                 "r"(smem_u32(smem_src)), "r"(x), "r"(y)
                 : "memory");
}

__device__ __forceinline__ void tma_store_commit()
{
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}

// wait until at most N of this thread's bulk groups still READ their smem source
template <int N>
__device__ __forceinline__ void tma_store_wait_read()
{
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all()
{
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// 4-byte asynchronous copy global -> shared (LDGSTS): no register, completion by cp_async_wait_all()
__device__ __forceinline__ void cp_async_4(void *smem_dst, const void *gsrc)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit()
{
    asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait()                      // at most N of this thread's groups still pending
{
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all()
{
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *map)
{
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

}  // namespace dspi
