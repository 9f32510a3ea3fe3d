// Shared helpers: mbarrier / TMA / L2-policy PTX wrappers for sm_90a, error plumbing, TMA descriptors and kernel launch set-up.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <atomic>
#include <mutex>
#include "../../include/fiery_b200.h"

namespace fiery {

// ------------------------------------------------------------------------------------------------------------
// host-side error plumbing (definitions in c_api.cu)
// ------------------------------------------------------------------------------------------------------------
int set_error(int code, const char* fmt, ...);

#define FIERY_CUDA_CHECK(expr)                                                                              \
    do {                                                                                                    \
        cudaError_t _e = (expr);                                                                            \
        if (_e != cudaSuccess)                                                                              \
            return ::fiery::set_error(FIERY_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                                      __FILE__, __LINE__);                                                  \
    } while (0)

#define FIERY_REQUIRE(cond, ...)                                             \
    do {                                                                     \
        if (!(cond)) return ::fiery::set_error(FIERY_E_INVALID, __VA_ARGS__); \
    } while (0)

// cuTensorMapEncodeTiled (definition in c_api.cu) without interleave and with FLOAT_OOB_FILL_NONE: coordinates outside the tensor
// read as zero, which the convolutions use as their padding.  elem_strides: nullptr for all 1.  A failure is reported through
// set_error, naming the map by `what`.
int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, int rank, const void* base, const cuuint64_t* dims,
                      const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* elem_strides,
                      CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2_promotion, const char* what);

// ------------------------------------------------------------------------------------------------------------
// host-side launch set-up
// ------------------------------------------------------------------------------------------------------------
// One-time per-device set-up of a kernel (function attributes are per device), safe when several host threads call in.
struct OncePerDevice {
    std::atomic<int> done[64];
    std::mutex mu;
    template <typename F>
    int run(F&& configure) {
        int dev = 0;
        FIERY_CUDA_CHECK(cudaGetDevice(&dev));
        std::atomic<int>& flag = done[dev & 63];
        if (flag.load(std::memory_order_acquire)) return FIERY_OK;
        std::lock_guard<std::mutex> lock(mu);
        if (flag.load(std::memory_order_relaxed)) return FIERY_OK;
        const int rc = configure();
        if (rc == FIERY_OK) flag.store(1, std::memory_order_release);
        return rc;
    }
};

template <typename Kernel>
int set_dynamic_smem(Kernel kernel, int bytes) {
    FIERY_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    return FIERY_OK;
}

// Persistent grid: at most one CTA per SM of the current device, the n_tiles (>= 1) tiles spread evenly over them.
inline int persistent_grid(long long n_tiles, unsigned* grid) {
    int dev = 0, sms = 0;
    FIERY_CUDA_CHECK(cudaGetDevice(&dev));
    FIERY_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const long long waves = (n_tiles + sms - 1) / sms;
    *grid = static_cast<unsigned>((n_tiles + waves - 1) / waves);
    return FIERY_OK;
}

// ------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}

// make the barrier initialisation visible to the async (TMA) proxy
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_addr(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}

// Bounded wait: a TMA that never completes (bad descriptor) traps instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 24)) __trap();
    }
}

// A ring of `stages` shared-memory stages that TMA fills and the consumers read in order: iteration `it` uses stage it % stages for
// the (it / stages)-th time.  full[s] (count 1) completes when the producer has armed it and the stage's bytes have landed; empty[s]
// completes when every consumer warp has released the stage.  The barriers lie in one array, full[stages] then empty[stages].  A
// ring initialised with no consumer warps has no empty side: its kernels arm() a stage only after a CTA-wide barrier has shown every
// consumer done with it.
struct MbarRing {
    uint64_t* full;
    uint64_t* empty;
    int stages;

    __device__ __forceinline__ MbarRing(uint64_t* bars, int n) : full(bars), empty(bars + n), stages(n) {}

    // one thread, before a CTA barrier
    __device__ __forceinline__ void init(uint32_t consumer_warps) const {
        for (int s = 0; s < stages; ++s) {
            mbar_init(full + s, 1);
            if (consumer_warps) mbar_init(empty + s, consumer_warps);
        }
        fence_mbar_init();
    }
    // announce the bytes that iteration it's loads bring into its stage; returns the stage
    __device__ __forceinline__ int arm(int it, uint32_t bytes) const {
        const int st = it % stages;
        mbar_arrive_expect_tx(full + st, bytes);
        return st;
    }
    // producer: wait until the consumers have released the stage's previous use, then arm it
    __device__ __forceinline__ int produce(int it, uint32_t bytes) const {
        const int st = it % stages, use = it / stages;
        if (use > 0) mbar_wait(empty + st, (use - 1) & 1);
        mbar_arrive_expect_tx(full + st, bytes);
        return st;
    }
    // consumer: wait until iteration it's stage has landed; returns the stage
    __device__ __forceinline__ int consume(int it) const {
        const int st = it % stages;
        mbar_wait(full + st, (it / stages) & 1);
        return st;
    }
    // consumer warp: every lane is done reading iteration it's stage
    __device__ __forceinline__ void release(int it) const {
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(empty + it % stages);
    }
};

// The dynamic shared memory, realigned to the 1024 bytes the 128-byte swizzle atoms need: the window itself is only guaranteed
// 16-byte aligned, so launches reserve 1024 bytes of slack.
__device__ __forceinline__ unsigned char* dynamic_smem_1024() {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    return reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
}

// Named barrier `id` (1..15; 0 is __syncthreads) over n threads, for code paths that only some warps take
__device__ __forceinline__ void named_barrier(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// L2 eviction-priority policies (createpolicy: a 64-bit descriptor covering the whole access) for the .L2::cache_hint forms:
// evict_first for data used once (it streams past what should stay), evict_last for data that is used again soon,
// evict_normal to hand lines back to the default priority.
__device__ __forceinline__ uint64_t l2_evict_first() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_evict_last() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_evict_normal() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
    return p;
}

// 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP); 16-byte aligned, size a multiple of 16
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)), "l"(policy) : "memory");
}

// 2-D and 3-D tiled TMA loads global -> shared, completion signalled on an mbarrier (SASS: UTMALDG)
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_addr(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_addr(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

// 4-D variants: (column, row, channel-within-image, image)
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_addr(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3,
                                            uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
        ::"r"(smem_addr(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
          "l"(policy)
        : "memory");
}

// 5-D variants: (column, channel lane, channel within lane, row, image) of the lift's context tile
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(smem_addr(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3, int c4,
                                            uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5, %6, %7}], [%2], %8;"
        ::"r"(smem_addr(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4),
          "l"(policy)
        : "memory");
}

// shared -> global tiled TMA store (SASS: UTMASTG); out-of-range parts of the box are clipped
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3, int c4) {
    asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
                 : "memory");
}

__device__ __forceinline__ void tma_store_commit_and_wait() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// inclusive prefix sum of v over the block (every thread must call it); warp_sums: >= 32 ints of shared memory
__device__ __forceinline__ int block_inclusive_scan(int v, int* warp_sums) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    if (lane == 31) warp_sums[warp] = v;
    __syncthreads();
    if (warp == 0) {
        int w = (lane < (blockDim.x >> 5)) ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += t;
        }
        warp_sums[lane] = w;
    }
    __syncthreads();
    const int base = warp > 0 ? warp_sums[warp - 1] : 0;
    __syncthreads();
    return v + base;
}

}  // namespace fiery
