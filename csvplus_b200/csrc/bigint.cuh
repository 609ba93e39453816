// bigint.cuh — the little-endian big integers of the exact (rare) paths: numeric_rare (ParseFloat) and format_rare
// (FormatFloat).  A Big is a view of caller-provided 32-bit limbs, normally a warp's slice of shared memory; one lane
// runs the sequential carries.
#pragma once
#include <cstdint>

namespace cpb {

constexpr int BIGL = 128;  // 32-bit limbs: 4096 bits, above the 3808 the largest ParseFloat operand needs (DESIGN §3.6)

struct Big { uint32_t* w; int n; };

__device__ inline void big_mul_add(Big& b, uint32_t m, uint32_t a) {  // b = b * m + a
    uint64_t carry = a;
    for (int i = 0; i < b.n; i++) {
        const uint64_t t = (uint64_t)b.w[i] * m + carry;
        b.w[i] = (uint32_t)t; carry = t >> 32;
    }
    if (carry && b.n < BIGL) b.w[b.n++] = (uint32_t)carry;
}

__device__ inline void big_pow10(Big& b, int e) {
    b.w[0] = 1; b.n = 1;
    for (; e >= 9; e -= 9) big_mul_add(b, 1000000000u, 0);
    uint32_t m = 1;
    for (; e > 0; e--) m *= 10;
    big_mul_add(b, m, 0);
}

__device__ inline void big_mul_u64(const Big& a, uint64_t x, Big& o) {  // o = a * x
    const uint32_t xm[2] = {(uint32_t)x, (uint32_t)(x >> 32)};
    for (int i = 0; i < a.n + 2 && i < BIGL; i++) o.w[i] = 0;
    for (int pass = 0; pass < 2; pass++) {
        if (!xm[pass]) continue;
        uint64_t carry = 0;
        for (int i = 0; i < a.n; i++) {
            const uint64_t t = (uint64_t)a.w[i] * xm[pass] + o.w[i + pass] + carry;
            o.w[i + pass] = (uint32_t)t; carry = t >> 32;
        }
        for (int k = a.n + pass; carry && k < BIGL; k++) {
            const uint64_t t = (uint64_t)o.w[k] + carry;
            o.w[k] = (uint32_t)t; carry = t >> 32;
        }
    }
    o.n = min(a.n + 2, BIGL);
    while (o.n > 0 && o.w[o.n - 1] == 0) o.n--;
}

__device__ inline int big_bits(const Big& a) { return a.n ? 32 * (a.n - 1) + (32 - __clz(a.w[a.n - 1])) : 0; }

__device__ inline void big_shl(const Big& a, int s, Big& o) {  // o = a << s; the caller guarantees the result fits
    const int q = s >> 5, r = s & 31;
    const int on = a.n + q + 1;
    for (int i = 0; i < on; i++) o.w[i] = 0;
    for (int i = 0; i < a.n; i++) {
        o.w[i + q] |= a.w[i] << r;
        if (r) o.w[i + q + 1] |= a.w[i] >> (32 - r);
    }
    o.n = on;
    while (o.n > 0 && o.w[o.n - 1] == 0) o.n--;
}

__device__ inline int big_cmp(const Big& a, const Big& b) {
    if (a.n != b.n) return a.n < b.n ? -1 : 1;
    for (int i = a.n - 1; i >= 0; i--)
        if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
    return 0;
}

// sign of A * 2^d - C (d may be negative), via bit lengths first: the shifted operand then never outgrows the other
__device__ inline int big_cmp_shifted(const Big& a, int d, const Big& c, Big& t) {
    const int la = big_bits(a) + (a.n ? d : 0), lc = big_bits(c);
    if (la != lc) return la < lc ? -1 : 1;
    if (d >= 0) { big_shl(a, d, t); return big_cmp(t, c); }
    big_shl(c, -d, t);
    return big_cmp(a, t);
}

// b = b / d, returning the remainder (d > 0)
__device__ inline uint32_t big_divmod(Big& b, uint32_t d) {
    uint64_t rem = 0;
    for (int i = b.n - 1; i >= 0; i--) {
        const uint64_t cur = rem << 32 | b.w[i];
        b.w[i] = (uint32_t)(cur / d); rem = cur % d;
    }
    while (b.n > 0 && b.w[b.n - 1] == 0) b.n--;
    return (uint32_t)rem;
}

}  // namespace cpb
