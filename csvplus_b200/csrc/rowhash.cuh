// rowhash.cuh — device-side key hashing shared by the probe tables (join.cu) and the row-carrying hash table's fused
// probe / length scan (gather.cu): the probe key packed in registers, its hash, the 128-bit slot claims (global and
// shared memory), and the 32-byte row-carrying slot with its region-wrapped probe sequence.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "core.hpp"

namespace cpb {

__device__ __forceinline__ uint64_t mix64(uint64_t h) {
    h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
    return h;
}
__device__ __forceinline__ uint64_t hash3(unsigned long long a, unsigned long long b, unsigned long long c) {
    return mix64(mix64(mix64(0x9E3779B97F4A7C15ull ^ a) ^ b) ^ c);
}
__device__ __forceinline__ uint64_t slot_of(uint64_t h, uint64_t nslots) { return __umul64hi(h, nslots); }
// the hash of the first pbytes bytes of row r of a key image of n rows (word w at img[w * n + r]): the ordinal probe
// tables of join.cu (smem, global) start at hash_prefix & (nslots - 1)
__device__ __forceinline__ uint64_t hash_prefix(const uint64_t* img, uint64_t n, uint64_t r, uint32_t pbytes) {
    uint32_t full = pbytes >> 3, rem = pbytes & 7;
    uint64_t h = 0x9E3779B97F4A7C15ull;
    for (uint32_t w = 0; w < full; w++) h = mix64(h ^ img[(uint64_t)w * n + r]);
    if (rem) h = mix64(h ^ (img[(uint64_t)full * n + r] & (~0ull << (8 * (8 - rem)))));
    return h;
}

__device__ __forceinline__ unsigned long long bswap64(unsigned long long x) {
    return ((unsigned long long)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | __byte_perm((uint32_t)(x >> 32), 0, 0x0123);
}
// the first min(len,16) bytes of a string, little-endian in (a, b), the rest zero: aligned 8-byte loads only (the
// probe rows of a warp are ~one sector apart, a byte loop costs one L1 request per byte)
__device__ __forceinline__ void load16(const uint8_t* p, uint32_t len, unsigned long long& a, unsigned long long& b) {
    a = b = 0;
    if (len == 0) return;
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 7u), sh = mis * 8;
    const unsigned long long* wp = reinterpret_cast<const unsigned long long*>(p - mis);
    const uint32_t need = mis + (len < 16u ? len : 16u);
    const unsigned long long w0 = __ldg(wp), w1 = need > 8 ? __ldg(wp + 1) : 0ull, w2 = need > 16 ? __ldg(wp + 2) : 0ull;
    a = sh ? (w0 >> sh) | (w1 << (64 - sh)) : w0;
    b = sh ? (w1 >> sh) | (w2 << (64 - sh)) : w1;
    if (len < 8) { a &= (1ull << (8 * len)) - 1; b = 0; }
    else if (len < 16) b &= (1ull << (8 * (len - 8))) - 1;
}
// packs the probe key exactly like key_pack_kernel (sort.cu), but into three registers
__device__ __forceinline__ void pack3(const KeyDesc& kd, uint64_t r, unsigned long long& w0, unsigned long long& w1, unsigned long long& w2) {
    unsigned long long cur = 0; int cnt = 0, word = 0;
    w0 = w1 = w2 = 0;
    auto flush = [&](unsigned long long v) { if (word == 0) w0 = v; else if (word == 1) w1 = v; else w2 = v; word++; };
    auto push = [&](uint32_t b) { cur = (cur << 8) | b; if (++cnt == 8) { flush(cur); cnt = 0; cur = 0; } };
    for (int k = 0; k < kd.nkeys; k++) {
        const uint32_t s = kd.off[k][r], len = kd.off[k][r + 1] - s, wd = kd.width[k];
        const uint8_t* p = kd.data[k] + s;
        unsigned long long a, b;
        load16(p, len < wd ? len : wd, a, b);
        uint32_t i = 0;
        if (cnt == 0 && wd >= 8) { flush(bswap64(a)); i = 8; if (wd >= 16) { flush(bswap64(b)); i = 16; } }
        for (; i < wd; i++)
            push(i < 8 ? (uint32_t)(a >> (8 * i)) & 255u : i < 16 ? (uint32_t)(b >> (8 * (i - 8))) & 255u : (i < len ? p[i] : 0u));
        const uint32_t lf = len > wd ? 0xffffffffu : len;
        for (int i2 = (int)kd.lenbytes[k] - 1; i2 >= 0; i2--) push((lf >> (8 * i2)) & 0xffu);
    }
    if (cnt) flush(cur << (8 * (8 - cnt)));
}

// (a slot is claimed and filled by ONE 128-bit compare-and-swap — SASS ATOMG.E.CAS.128 — so a slot is never seen half
// written and an insert that meets its own key knows it)
__device__ __forceinline__ void cas128(void* addr, unsigned long long vl, unsigned long long vh, unsigned long long& ol, unsigned long long& oh) {
    asm volatile("{\n.reg .b128 c, v, o;\nmov.b128 c, {%3, %4};\nmov.b128 v, {%5, %6};\natom.global.cas.b128 o, [%2], c, v;\nmov.b128 {%0, %1}, o;\n}"
                 : "=l"(ol), "=l"(oh) : "l"(addr), "l"(0ull), "l"(0ull), "l"(vl), "l"(vh) : "memory");
}
// the same claim on a shared-memory slot (SASS ATOMS.CAS.128)
__device__ __forceinline__ void cas128_shared(void* addr, unsigned long long vl, unsigned long long vh, unsigned long long& ol, unsigned long long& oh) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(addr);
    asm volatile("{\n.reg .b128 c, v, o;\nmov.b128 c, {%3, %4};\nmov.b128 v, {%5, %6};\natom.shared.cas.b128 o, [%2], c, v;\nmov.b128 {%0, %1}, o;\n}"
                 : "=l"(ol), "=l"(oh) : "r"(a), "l"(0ull), "l"(0ull), "l"(vl), "l"(vh) : "memory");
}

// ------------------------------------------------------------------ row-carrying slot (Index::derived.rowhash)
// One 32-byte slot = one DRAM sector: a 16-byte header {12 key bytes, hdr}, then the payload columns' values back to
// back.  hdr = RH_OCCUPIED | length of payload column j in bits 5j..5j+4 (a value is at most 16 bytes): the occupied
// bit keeps the header of an empty key (an all-zero image) from reading as an empty slot.
struct __align__(32) RowSlot { unsigned long long k0; uint32_t k1; uint32_t hdr; uint4 pay; };
constexpr uint32_t RH_OCCUPIED = 0x80000000u;
constexpr int RH_MAXC = 4;         // payload columns
constexpr uint32_t RH_PAY = 16;    // payload bytes
// The table is cut into regions of RowHash::region slots (a power of two, RH_REGION for all but small tables): a key's
// probe sequence starts at slot_of(hash, nslots) and wraps from its region's last slot to the region's first, so each
// region is built on its own in shared memory (join.cu: rowhash_build).
constexpr uint32_t RH_REGION = 1024;

// the packed key of probe row r (12 bytes: k0, k1) and the first slot of its probe sequence
__device__ __forceinline__ uint64_t rh_start(const KeyDesc& kd, uint64_t r, uint64_t nslots, unsigned long long& k0, uint32_t& k1) {
    unsigned long long w0, w1, w2;
    pack3(kd, r, w0, w1, w2);
    k0 = w0; k1 = (uint32_t)(w1 >> 32);
    return slot_of(hash3(w0, w1, 0ull), nslots);
}
__device__ __forceinline__ uint4 rh_header(const RowSlot* slots, uint64_t s) { return __ldg(reinterpret_cast<const uint4*>(&slots[s])); }
// the slot after s in s's region (rmask = region - 1)
__device__ __forceinline__ uint64_t rh_next(uint64_t s, uint64_t rmask) { return (s & ~rmask) | ((s + 1) & rmask); }
// linear probing from slot s, whose header h is loaded, inside s's region: true when the key is found, s and h then are
// its slot's
__device__ __forceinline__ bool rh_walk(const RowSlot* slots, uint64_t rmask, unsigned long long k0, uint32_t k1, uint64_t& s, uint4& h) {
    for (;;) {
        if (h.w == 0u) return false;
        if (h.x == (uint32_t)k0 && h.y == (uint32_t)(k0 >> 32) && h.z == k1) return true;
        s = rh_next(s, rmask);
        h = rh_header(slots, s);
    }
}

// bytes of a 16-byte value held little-endian in (a, b): OR (x, y) in at byte pos; bytes shifted past byte 15 are dropped
__device__ __forceinline__ void or_at16(unsigned long long& a, unsigned long long& b, uint32_t pos, unsigned long long x, unsigned long long y) {
    if (pos == 0) { a |= x; b |= y; }
    else if (pos < 8) { const uint32_t s = 8 * pos; a |= x << s; b |= (y << s) | (x >> (64 - s)); }
    else if (pos < 16) b |= x << (8 * (pos - 8));
}
// bytes [pos, pos + len) of (a, b) moved to byte 0, the rest zero
__device__ __forceinline__ void take16(unsigned long long a, unsigned long long b, uint32_t pos, uint32_t len, unsigned long long& x,
                                       unsigned long long& y) {
    if (pos == 0) { x = a; y = b; }
    else if (pos < 8) { const uint32_t s = 8 * pos; x = (a >> s) | (b << (64 - s)); y = b >> s; }
    else { x = pos < 16 ? b >> (8 * (pos - 8)) : 0ull; y = 0; }
    if (len < 8) { x &= (1ull << (8 * len)) - 1; y = 0; }
    else if (len < 16) y &= (1ull << (8 * (len - 8))) - 1;
}

}  // namespace cpb
