// keyhash.cuh — the byte-value hash and equality of codes.cu and groupby.cu.  The hash of a value is the sum of
// word_mix(word i, i) over its 8-byte little-endian words (the last one zero-padded), finished with the length
// (hash_finish).  A sum does not depend on which lane added which word, so one thread or a whole warp computes the same
// hash.  A value of at most LONG_BYTES is hashed and compared by one thread; a longer one by a whole warp.  GroupBy
// chains the hashes hk of a row's key columns k = 0, 1, ... from h = 0 as h = fmix64(h + word_mix(hk, k)) (row_hash_step).
// tests/hash_ref.py restates every function here, and tests/hash_harness.cu checks that restatement on the device.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "util.cuh"

namespace cpb {

constexpr uint32_t LONG_BYTES = 128;

__device__ __forceinline__ uint64_t fmix64(uint64_t k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return k;
}
__device__ __forceinline__ uint64_t word_mix(uint64_t w, uint32_t i) { return fmix64(w ^ ((uint64_t)(i + 1) * 0x9E3779B97F4A7C15ull)); }
__device__ __forceinline__ uint64_t hash_finish(uint64_t sum, uint32_t len) { return fmix64(sum + (uint64_t)len * 0xC2B2AE3D27D4EB4Full); }

// word i (bytes [8i, min(8i + 8, len)), little-endian, zero-padded) of the len bytes at sp, from aligned 8-byte loads:
// the aligned word holding a byte of the value never crosses a page, so nothing past the value's last word is read
__device__ __forceinline__ uint64_t word_at(const uint8_t* sp, uint32_t len, uint32_t i) {
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(sp) & 7u), sh = mis * 8, rem = len - 8 * i;
    const unsigned long long* wp = reinterpret_cast<const unsigned long long*>(sp - mis) + i;
    uint64_t v = __ldg(wp) >> sh;
    if (sh && mis + rem > 8) v |= (uint64_t)__ldg(wp + 1) << (64 - sh);
    if (rem < 8) v &= (1ull << (8 * rem)) - 1;
    return v;
}
// the hash of the len bytes at sp, by one thread
__device__ __forceinline__ uint64_t hash_thread(const uint8_t* sp, uint32_t len) {
    uint64_t sum = 0;
    for (uint32_t w = 0; w * 8 < len; w++) sum += word_mix(word_at(sp, len, w), w);
    return hash_finish(sum, len);
}
// the same hash by the whole warp: every lane calls it with the same sp and len; the hash is valid on lane `owner`
__device__ __forceinline__ uint64_t hash_warp(const uint8_t* sp, uint32_t len, int lane, int owner, uint64_t h) {
    uint64_t sum = 0;
    for (uint32_t w = lane; w * 8 < len; w += 32) sum += word_mix(word_at(sp, len, w), w);
    sum = warp_sum_u64(sum);
    if (lane == owner) h = hash_finish(sum, len);
    return h;
}
// one key column's hash hk folded into GroupBy's row hash h (column k, counted from 0; h starts at 0)
__device__ __forceinline__ uint64_t row_hash_step(uint64_t h, uint64_t hk, uint32_t k) { return fmix64(h + word_mix(hk, k)); }
__device__ __forceinline__ bool equal_thread(const uint8_t* a, const uint8_t* b, uint32_t len) {
    const uint32_t nw = (len + 7) / 8;
    for (uint32_t w = 0; w < nw; w++) if (word_at(a, len, w) != word_at(b, len, w)) return false;
    return true;
}
// every lane of the warp calls it with the same a, b and len
__device__ __forceinline__ bool equal_warp(const uint8_t* a, const uint8_t* b, uint32_t len, int lane) {
    const uint32_t nw = (len + 7) / 8;
    bool diff = false;
    for (uint32_t w0 = 0; w0 < nw; w0 += 32) {
        const uint32_t w = w0 + lane;
        if (w < nw) diff = word_at(a, len, w) != word_at(b, len, w);
        if (__any_sync(0xffffffffu, diff)) return false;
    }
    return true;
}

}  // namespace cpb
