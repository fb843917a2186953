// Shared helpers for the b200asr sm_90a kernels (error plumbing, launch accounting, warp/block
// reductions, mbarrier + bulk-copy wrappers).  Everything in csrc/ is compiled into ONE shared
// library (libb200asr.so) whose only exported symbols are the extern "C" entry points declared in
// include/b200asr.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>

namespace b200asr {

// ---- error plumbing (thread-local message, C-ABI returns <0) -------------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define B200_OK 0
#define B200_EINVAL (-1)
#define B200_ECUDA (-2)

#define B200_REQUIRE(cond, ...)                         \
    do {                                                \
        if (!(cond)) {                                  \
            ::b200asr::set_error(__VA_ARGS__);          \
            return B200_EINVAL;                         \
        }                                               \
    } while (0)

#define B200_CUDA(expr)                                                                   \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            ::b200asr::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),  \
                                 __FILE__, __LINE__);                                     \
            return B200_ECUDA;                                                            \
        }                                                                                 \
    } while (0)

// check the launch that was just enqueued (does not synchronise)
#define B200_LAUNCH_CHECK(name)                                                           \
    do {                                                                                  \
        cudaError_t _e = cudaGetLastError();                                              \
        if (_e != cudaSuccess) {                                                          \
            ::b200asr::set_error("launch of %s failed: %s", name, cudaGetErrorString(_e)); \
            return B200_ECUDA;                                                            \
        }                                                                                 \
        ::b200asr::count_launch();                                                        \
    } while (0)

int sm_count();
int max_optin_smem();

// ---- device helpers ---------------------------------------------------------------------
#define NEG_INF (-INFINITY)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide reductions through a 32-float shared scratch. All threads must call; result is
// broadcast to all threads. blockDim.x must be a multiple of 32 and <= 1024.
__device__ __forceinline__ float block_sum(float v, float* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = warp_sum(v);
    __syncthreads();  // protect scratch from a previous use
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    float r = (lane < nw) ? scratch[lane] : 0.f;
    r = warp_sum(r);
    return r;
}
__device__ __forceinline__ float block_max(float v, float* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    float r = (lane < nw) ? scratch[lane] : NEG_INF;
    r = warp_max(r);
    return r;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ---- mbarrier / bulk async copy (TMA 1-D) ------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// global -> shared bulk copy (bytes multiple of 16, both addresses 16-B aligned); completion is
// signalled on `bar` via complete_tx.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// order earlier generic-proxy accesses (made visible to this thread) before later async-proxy ones
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_add_u32(unsigned* p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

}  // namespace b200asr
