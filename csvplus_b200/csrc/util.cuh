// util.cuh — device-side helpers (sm_90a): the one-thread-per-row launcher, mbarrier + bulk-async (TMA 1-D) staging,
// gpu-scope acquire/release for the decoupled look-back chains, warp scans, key-image compare.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "core.hpp"

namespace cpb {

// ---- one thread per row: f(i) for every i in [0, n)
template <class F>
__global__ void __launch_bounds__(256) each_row_kernel(uint64_t n, F f) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) f(i);
}
// Launches each_row_kernel on c's stream and checks the launch; nothing is launched for n == 0 (a grid of no blocks is a
// launch error).  f is a [=] __device__ (uint64_t i) lambda that captures plain values and device pointers.
template <class F>
void each_row(Ctx* c, uint64_t n, F f) {
    if (n == 0) return;
    each_row_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(n, f);
    CPB_CUDA(cudaGetLastError());
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier / cp.async.bulk (SASS: SYNCS.*, UBLKCP)
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// asks the bulk-copy engine to pull [src, src + bytes) into L2 (no shared memory, no completion to wait for)
__device__ __forceinline__ void bulk_prefetch_l2(const void* src_gmem, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src_gmem), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra LAB_DONE;\n"
        "bra LAB_WAIT;\n"
        "LAB_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(phase)
        : "memory");
}

// ---- gpu-scope ordering for tile-state words
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t ld_relaxed_u64(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u64(uint64_t* p, uint64_t v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// ---- warp helpers
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}
__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, v, d);
        if (lane_id() >= (uint32_t)d) v += t;
    }
    return v;
}
__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

// ---- key images (sort.cu): word w of row r of an image of n rows is img[w * n + r], first byte most significant
// the first pbytes bytes of row ra of image a equal those of row rb of image b
__device__ __forceinline__ bool prefix_equal(const uint64_t* a, uint64_t na, uint64_t ra, const uint64_t* b, uint64_t nb, uint64_t rb,
                                             uint32_t pbytes) {
    uint32_t full = pbytes >> 3, rem = pbytes & 7;
    for (uint32_t w = 0; w < full; w++) if (a[(uint64_t)w * na + ra] != b[(uint64_t)w * nb + rb]) return false;
    if (rem) {
        uint64_t m = ~0ull << (8 * (8 - rem));
        if ((a[(uint64_t)full * na + ra] & m) != (b[(uint64_t)full * nb + rb] & m)) return false;
    }
    return true;
}

// the first pbytes of row r of image a (na rows) against those of row i of image b (nb rows): <0, 0, >0
__device__ __forceinline__ int prefix_cmp(const uint64_t* a, uint64_t na, uint64_t r, const uint64_t* b, uint64_t nb, uint64_t i, uint32_t pbytes) {
    const uint32_t full = pbytes >> 3, rem = pbytes & 7;
    for (uint32_t w = 0; w < full; w++) {
        const uint64_t x = a[(uint64_t)w * na + r], y = b[(uint64_t)w * nb + i];
        if (x != y) return x < y ? -1 : 1;
    }
    if (rem) {
        const uint64_t m = ~0ull << (8 * (8 - rem));
        const uint64_t x = a[(uint64_t)full * na + r] & m, y = b[(uint64_t)full * nb + i] & m;
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}
// ---- SWAR byte classification
// exact per-byte equality flags: bit 7 of every byte of the result is set iff that byte of w == c
__device__ __forceinline__ uint32_t eq_flags(uint32_t w, uint32_t c4) {
    uint32_t x = w ^ c4;
    uint32_t y = (x & 0x7f7f7f7fu) + 0x7f7f7f7fu;
    return ~(y | x) & 0x80808080u;
}
// nonzero iff some byte of w == c (inexact per byte, exact as an any-test)
__device__ __forceinline__ uint32_t eq_any(uint32_t w, uint32_t c4) {
    uint32_t x = w ^ c4;
    return (x - 0x01010101u) & ~x & 0x80808080u;
}
// gather the 4 flag bits (7,15,23,31) into the top nibble: bits 28..31
__device__ __forceinline__ uint32_t flags_top(uint32_t z) { return z * 0x00204081u; }
// 16 flag bits of a uint4 worth of flags -> 16-bit mask (byte i of the vector -> bit i)
__device__ __forceinline__ uint32_t flags16(uint32_t z0, uint32_t z1, uint32_t z2, uint32_t z3) {
    uint32_t acc = flags_top(z3) >> 28;
    acc = __funnelshift_l(flags_top(z2), acc, 4);  // (acc << 4) | top nibble
    acc = __funnelshift_l(flags_top(z1), acc, 4);
    acc = __funnelshift_l(flags_top(z0), acc, 4);
    return acc;
}

}  // namespace cpb
