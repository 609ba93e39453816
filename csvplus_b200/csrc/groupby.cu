// groupby.cu — GroupBy: per-key count / sum / min / max / first / last of int64 (Row.ValueAsInt) and float64
// (Row.ValueAsFloat64) inputs, folded batch by batch into state that persists across pushes.
//
// Semantics (those of a Go RowFunc folding the rows in plan order): two rows are in one group when every key column
// holds equal bytes; groups are numbered in order of first appearance.  count: rows; sum int: int64 += (wrapping);
// sum float: acc = acc + v in row order from +0.0, each addition rounded to nearest (__dadd_rn: no reassociation, no
// FMA), a NaN result keeping the NaN operand, or the x86 default NaN for Inf - Inf, as Go's ADDSD does; min / max int:
// the least / greatest value; min / max float: a fold with Go's math.Min / math.Max (-Inf / +Inf wins, then NaN, and
// Min(-0, +0) = -0), which makes the result independent of row order; first / last: the value of the group's first / last row.
//
// State (struct Groups): per group its 64-bit hash and, per key column, a pointer to and the length of its key bytes.
// The pointers point into the tables of the new groups' key rows that earlier pushes gathered (kept alive here, and
// concatenated into the result's key table).  An open-addressing slot table of uint32 group ids (0xFFFFFFFF = empty,
// linear probing from hash & (nslots - 1), load factor <= 1/2) is rebuilt from the stored hashes when it grows.  One
// 8-byte accumulator per group per aggregate.  Every per-group array grows by doubling.
//
// A push of n rows:
//   1. every aggregate input converted with column_as_number (numeric.cu); the lowest failing row (ties to the earlier
//      aggregate) cuts the push: the rows before it are folded, then its error is thrown;
//   2. groupby_hash: each row's hash over its key columns: per column keyhash.cuh's word hash (length included), the
//      columns chained with fmix64.  A value over LONG_BYTES is hashed by the whole warp;
//   3. groupby_probe: the persistent slot table probed read-only; a slot whose group has the row's hash is compared byte
//      for byte in every key column (a hash is never taken as equality; a row with a value over LONG_BYTES compares with
//      the whole warp).  gid[r] = the group, or a miss;
//   4. the misses (scan_flags / compact_flags into their rows) get codes.cu's first-appearance treatment: a temporary
//      table of miss ids, atomicCAS to claim a slot, atomicMin to keep the lowest miss of equal keys (groupby_first); the
//      first misses, scanned and compacted, are the new groups ngroups + position.  Their key rows are appended with
//      gather_rows, their hashes stored, and their ids inserted into the persistent table (groupby_insert);
//   5. the fold: the group ids sorted stably (sort_by_image over a one-word image of the id: only the id's non-constant
//      bytes are passed over), then groupby_fold, one thread per run of equal ids in (group, row) order, folds the run
//      into the group's accumulators.  A float sum is therefore one dependent chain of additions per group per push:
//      the cost of matching the reference bit for bit (one group of every row is one thread's serial loop).
// Host synchronisations per push: one per converted aggregate input (column_as_number), the miss count, and the sort's
// digit histogram; when some row misses, the new-group count and gather_rows' byte totals too.
// Device memory: per group 8 B of hash + 12 B per key column + 8 B per aggregate + 8-16 B of slots + its key bytes; per
// pushed row 8 B per aggregate input (+ 4 B of float rare-path ids) + 52 B (hash, id, miss flag, its scan, the sort's
// image, keys and ids), freed when the push returns.
#include <algorithm>

#include "core.hpp"
#include "keyhash.cuh"
#include "util.cuh"

namespace cpb {

constexpr uint32_t NO_GROUP = 0xFFFFFFFFu;
constexpr int GB_WARPS = 8;
constexpr int MAXAGGS = 32;
constexpr uint64_t GO_NAN = 0x7FF8000000000001ull;  // math.NaN(), what math.Min / Max return for a NaN operand
constexpr uint64_t X86_NAN = 0xFFF8000000000000ull; // the default NaN of an x86 addition such as Inf + -Inf

struct KeyCols { int n; const uint32_t* off[MAXKEYS]; const uint8_t* data[MAXKEYS]; };
// the stored keys: column k of group g at ptr[k * cap + g], len[k * cap + g]
struct StoredKeys { int n; uint64_t cap; const uint64_t* hash; const uint8_t* const* ptr; const uint32_t* len; };

__device__ __forceinline__ bool row_is_long(const KeyCols& kc, uint64_t r) {
    bool l = false;
    for (int k = 0; k < kc.n; k++) l |= kc.off[k][r + 1] - kc.off[k][r] > LONG_BYTES;
    return l;
}
// row r's key against stored group g / row s of the same table: one thread, or (warp) every lane with the same arguments
template <bool WARP>
__device__ __forceinline__ bool key_equals_group(const KeyCols& kc, uint64_t r, const StoredKeys& sk, uint32_t g, int lane) {
    for (int k = 0; k < kc.n; k++) {
        const uint32_t s = kc.off[k][r], len = kc.off[k][r + 1] - s;
        if (sk.len[k * sk.cap + g] != len) return false;
        const uint8_t* a = sk.ptr[k * sk.cap + g];
        if (!(WARP ? equal_warp(a, kc.data[k] + s, len, lane) : equal_thread(a, kc.data[k] + s, len))) return false;
    }
    return true;
}
template <bool WARP>
__device__ __forceinline__ bool key_equals_row(const KeyCols& kc, uint64_t r, uint64_t q, int lane) {
    for (int k = 0; k < kc.n; k++) {
        const uint32_t s = kc.off[k][r], len = kc.off[k][r + 1] - s, t = kc.off[k][q];
        if (kc.off[k][q + 1] - t != len) return false;
        if (!(WARP ? equal_warp(kc.data[k] + t, kc.data[k] + s, len, lane) : equal_thread(kc.data[k] + t, kc.data[k] + s, len))) return false;
    }
    return true;
}

__global__ void __launch_bounds__(GB_WARPS * 32) groupby_hash_kernel(const KeyCols kc, uint64_t n, uint64_t* __restrict__ hashes) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t nwarps = (uint64_t)gridDim.x * GB_WARPS;
    for (uint64_t g = (uint64_t)blockIdx.x * GB_WARPS + warp; g * 32 < n; g += nwarps) {
        const uint64_t i = g * 32 + lane;
        const bool valid = i < n;
        uint64_t h = 0;
        for (int k = 0; k < kc.n; k++) {
            uint32_t len = 0;
            const uint8_t* sp = kc.data[k];
            if (valid) { const uint32_t s = kc.off[k][i]; len = kc.off[k][i + 1] - s; sp += s; }
            const bool is_long = valid && len > LONG_BYTES;
            uint64_t hk = 0;
            if (valid && !is_long) hk = hash_thread(sp, len);
            for (uint32_t m = __ballot_sync(0xffffffffu, is_long); m; m &= m - 1) {
                const int l = __ffs(m) - 1;
                const uint8_t* lp = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(sp), l));
                const uint32_t ll = __shfl_sync(0xffffffffu, len, l);
                hk = hash_warp(lp, ll, lane, l, hk);
            }
            h = row_hash_step(h, hk, (uint32_t)k);
        }
        if (valid) hashes[i] = h;
    }
}

// gid[r] = the stored group of row r's key, NO_GROUP when there is none; miss[r] = (gid[r] == NO_GROUP)
__global__ void __launch_bounds__(GB_WARPS * 32) groupby_probe_kernel(const KeyCols kc, uint64_t n, const uint64_t* __restrict__ hashes,
                                                                      const StoredKeys sk, const uint32_t* __restrict__ slots, uint64_t mask,
                                                                      uint32_t* __restrict__ gid, uint32_t* __restrict__ miss) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t nwarps = (uint64_t)gridDim.x * GB_WARPS;
    for (uint64_t g = (uint64_t)blockIdx.x * GB_WARPS + warp; g * 32 < n; g += nwarps) {
        const uint64_t i = g * 32 + lane;
        const bool valid = i < n;
        const uint64_t h = valid ? hashes[i] : 0;
        const bool is_long = valid && row_is_long(kc, i);
        uint32_t found = NO_GROUP;
        if (valid && !is_long) {
            for (uint64_t p = h & mask;; p = (p + 1) & mask) {
                const uint32_t s = slots[p];
                if (s == NO_GROUP) break;
                if (sk.hash[s] == h && key_equals_group<false>(kc, i, sk, s, lane)) { found = s; break; }
            }
        }
        for (uint32_t m = __ballot_sync(0xffffffffu, is_long); m; m &= m - 1) {
            const int l = __ffs(m) - 1;
            const uint64_t r = g * 32 + l, lh = __shfl_sync(0xffffffffu, h, l);
            uint32_t f = NO_GROUP;
            for (uint64_t p = lh & mask;; p = (p + 1) & mask) {
                const uint32_t s = slots[p];  // (every lane reads the same words: the branches stay warp-uniform)
                if (s == NO_GROUP) break;
                if (sk.hash[s] == lh && key_equals_group<true>(kc, r, sk, s, lane)) { f = s; break; }
            }
            if (lane == l) found = f;
        }
        if (valid) { gid[i] = found; miss[i] = found == NO_GROUP; }
    }
}

// codes_insert over the m misses (rows mrow[j]): slot of miss j in rep[j]; when the kernel ends every slot holds the
// lowest miss of its key
__global__ void __launch_bounds__(GB_WARPS * 32) groupby_first_kernel(const KeyCols kc, uint64_t m, const uint32_t* __restrict__ mrow,
                                                                      const uint64_t* __restrict__ hashes, uint32_t* slots, uint64_t mask,
                                                                      uint32_t* __restrict__ rep) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t nwarps = (uint64_t)gridDim.x * GB_WARPS;
    for (uint64_t g = (uint64_t)blockIdx.x * GB_WARPS + warp; g * 32 < m; g += nwarps) {
        const uint64_t j = g * 32 + lane;
        const bool valid = j < m;
        const uint32_t r = valid ? mrow[j] : 0;
        const uint64_t h = valid ? hashes[r] : 0;
        const bool is_long = valid && row_is_long(kc, r);
        if (valid && !is_long) {
            for (uint64_t p = h & mask;; p = (p + 1) & mask) {
                uint32_t s = slots[p];
                if (s == NO_GROUP && (s = atomicCAS(&slots[p], NO_GROUP, (uint32_t)j)) == NO_GROUP) { rep[j] = (uint32_t)p; break; }
                const uint32_t rs = mrow[s];
                if (hashes[rs] != h) continue;
                if (key_equals_row<false>(kc, r, rs, lane)) {
                    if ((uint32_t)j < s) atomicMin(&slots[p], (uint32_t)j);
                    rep[j] = (uint32_t)p;
                    break;
                }
            }
        }
        for (uint32_t b = __ballot_sync(0xffffffffu, is_long); b; b &= b - 1) {
            const int l = __ffs(b) - 1;
            const uint32_t lj = (uint32_t)(g * 32 + l), lr = __shfl_sync(0xffffffffu, r, l);
            const uint64_t lh = __shfl_sync(0xffffffffu, h, l);
            for (uint64_t p = lh & mask;; p = (p + 1) & mask) {
                uint32_t s = 0;
                if (lane == 0) {
                    s = slots[p];
                    if (s == NO_GROUP) s = atomicCAS(&slots[p], NO_GROUP, lj);
                }
                s = __shfl_sync(0xffffffffu, s, 0);
                if (s == NO_GROUP) { if (lane == 0) rep[lj] = (uint32_t)p; break; }
                const uint32_t rs = mrow[s];
                if (hashes[rs] != lh) continue;
                if (key_equals_row<true>(kc, lr, rs, lane)) {
                    if (lane == 0) { if (lj < s) atomicMin(&slots[p], lj); rep[lj] = (uint32_t)p; }
                    break;
                }
            }
        }
    }
}

// ------------------------------------------------------------------ the fold
struct AggArgs {
    int n;
    int op[MAXAGGS], kind[MAXAGGS];
    uint64_t* acc[MAXAGGS];
    const uint64_t* val[MAXAGGS];  // the converted inputs (null for count)
};

__device__ __forceinline__ double go_min(double x, double y) {  // math.Min
    if ((isinf(x) && x < 0) || (isinf(y) && y < 0)) return -INFINITY;
    if (isnan(x) || isnan(y)) return __longlong_as_double((long long)GO_NAN);
    if (x == 0 && x == y) return signbit(x) ? x : y;
    return x < y ? x : y;
}
__device__ __forceinline__ double go_max(double x, double y) {  // math.Max
    if ((isinf(x) && x > 0) || (isinf(y) && y > 0)) return INFINITY;
    if (isnan(x) || isnan(y)) return __longlong_as_double((long long)GO_NAN);
    if (x == 0 && x == y) return signbit(x) ? y : x;
    return x > y ? x : y;
}
__device__ __forceinline__ double go_add(double a, double b) {  // acc += v as Go on amd64 computes it
    const double r = __dadd_rn(a, b);
    if (!isnan(r)) return r;
    return isnan(a) ? a : isnan(b) ? b : __longlong_as_double((long long)X86_NAN);
}

// f(v[perm[i]]) for i in [lo, hi) in order, the loads issued 16 at a time: a long run is one thread's serial fold, and
// its pace is set by how many loads it has in flight
template <class F>
__device__ __forceinline__ void each_value(const uint32_t* __restrict__ perm, const uint64_t* __restrict__ v, uint64_t lo, uint64_t hi, F f) {
    uint64_t i = lo;
    for (; i + 16 <= hi; i += 16) {
        uint64_t x[16];
#pragma unroll
        for (int u = 0; u < 16; u++) x[u] = v[perm[i + u]];
#pragma unroll
        for (int u = 0; u < 16; u++) f(x[u]);
    }
    for (; i < hi; i++) f(v[perm[i]]);
}

// one thread per run of equal ids in the sorted order: gid[perm[lo .. hi)] = g; groups >= g0 are new in this push
__global__ void __launch_bounds__(256) groupby_fold_kernel(const uint32_t* __restrict__ gid, const uint32_t* __restrict__ perm, uint64_t n,
                                                           uint32_t g0, const AggArgs a) {
    const uint64_t lo = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (lo >= n) return;
    const uint32_t g = gid[perm[lo]];
    if (lo > 0 && gid[perm[lo - 1]] == g) return;
    uint64_t hi = lo + 1;
    while (hi < n && gid[perm[hi]] == g) hi++;
    for (int k = 0; k < a.n; k++) {
        uint64_t* acc = a.acc[k] + g;
        const uint64_t* v = a.val[k];
        const bool is_int = a.kind[k] == CPB_AGG_INT;
        switch (a.op[k]) {
            case CPB_AGG_COUNT: *acc += hi - lo; break;
            case CPB_AGG_FIRST: if (g >= g0) *acc = v[perm[lo]]; break;
            case CPB_AGG_LAST: *acc = v[perm[hi - 1]]; break;
            case CPB_AGG_SUM:
                if (is_int) {
                    uint64_t s = *acc;
                    each_value(perm, v, lo, hi, [&](uint64_t x) { s += x; });
                    *acc = s;
                } else {
                    double s = __longlong_as_double((long long)*acc);
                    each_value(perm, v, lo, hi, [&](uint64_t x) { s = go_add(s, __longlong_as_double((long long)x)); });
                    *acc = (uint64_t)__double_as_longlong(s);
                }
                break;
            case CPB_AGG_MIN:
            case CPB_AGG_MAX: {
                const bool mn = a.op[k] == CPB_AGG_MIN;
                if (is_int) {
                    int64_t s = (int64_t)*acc;
                    each_value(perm, v, lo, hi, [&](uint64_t x) { s = mn ? min(s, (int64_t)x) : max(s, (int64_t)x); });
                    *acc = (uint64_t)s;
                } else {
                    double s = __longlong_as_double((long long)*acc);
                    each_value(perm, v, lo, hi, [&](uint64_t x) {
                        const double d = __longlong_as_double((long long)x);
                        s = mn ? go_min(s, d) : go_max(s, d);
                    });
                    *acc = (uint64_t)__double_as_longlong(s);
                }
                break;
            }
        }
    }
}

// ------------------------------------------------------------------ state
struct Groups {
    Ctx* ctx = nullptr;
    std::vector<std::string> keys;
    std::vector<GroupAgg> aggs;
    uint64_t ngroups = 0, cap = 0, nslots = 0;
    Buf hash, ptr, len, slots;             // uint64[cap], (const uint8_t*)[nkeys][cap], uint32[nkeys][cap], uint32[nslots]
    std::vector<Buf> acc;                  // per aggregate: 8 B [cap]
    std::vector<std::shared_ptr<Table>> rows;  // the key rows of the groups, push by push
};

Groups* groups_open(Ctx* c, const std::vector<std::string>& keys, const std::vector<GroupAgg>& aggs) {
    if (keys.empty() || (int)keys.size() > MAXKEYS)
        throw ArgError{CPB_ERR_ARG, "GroupBy: 1 to " + std::to_string(MAXKEYS) + " key columns"};
    for (size_t i = 0; i < keys.size(); i++)
        for (size_t j = i + 1; j < keys.size(); j++)
            if (keys[i] == keys[j]) throw ArgError{CPB_ERR_ARG, "GroupBy: duplicate key column " + go_quote(keys[i])};
    if ((int)aggs.size() > MAXAGGS) throw ArgError{CPB_ERR_ARG, "GroupBy: more than " + std::to_string(MAXAGGS) + " aggregates"};
    for (const GroupAgg& a : aggs) {
        if (a.op < CPB_AGG_COUNT || a.op > CPB_AGG_LAST) throw ArgError{CPB_ERR_ARG, "GroupBy: unknown aggregate op " + std::to_string(a.op)};
        if (a.op != CPB_AGG_COUNT && a.kind != CPB_AGG_INT && a.kind != CPB_AGG_FLOAT64)
            throw ArgError{CPB_ERR_ARG, "GroupBy: unknown input kind " + std::to_string(a.kind)};
    }
    auto* g = new Groups;
    g->ctx = c; g->keys = keys; g->aggs = aggs;
    g->nslots = 64;
    g->slots = dev_alloc(c, g->nslots * 4);
    CPB_CUDA(cudaMemsetAsync(g->slots->p, 0xff, g->nslots * 4, c->stream));
    return g;
}

void groups_free(Groups* g) { delete g; }

// the accumulator a group starts from: the identity of its fold
static uint64_t agg_init(const GroupAgg& a) {
    if (a.op == CPB_AGG_MIN) return a.kind == CPB_AGG_INT ? 0x7FFFFFFFFFFFFFFFull : 0x7FF0000000000000ull;  // +Inf
    if (a.op == CPB_AGG_MAX) return a.kind == CPB_AGG_INT ? 0x8000000000000000ull : 0xFFF0000000000000ull;  // -Inf
    return 0;
}

// room for `need` groups: every per-group array doubled until it fits, the old contents copied
static void grow(Ctx* c, Groups& G, uint64_t need) {
    if (need <= G.cap) return;
    uint64_t cap = std::max<uint64_t>(G.cap, 1024);
    while (cap < need) cap *= 2;
    const size_t nk = G.keys.size();
    auto regrow = [&](Buf& b, size_t width, size_t parts) {
        Buf nb = dev_alloc(c, cap * width * parts);
        for (size_t k = 0; b && k < parts && G.ngroups; k++)
            CPB_CUDA(cudaMemcpyAsync(nb->as<uint8_t>() + k * cap * width, b->as<uint8_t>() + k * G.cap * width, G.ngroups * width,
                                     cudaMemcpyDeviceToDevice, c->stream));
        b = nb;
    };
    regrow(G.hash, 8, 1);
    regrow(G.ptr, 8, nk);
    regrow(G.len, 4, nk);
    G.acc.resize(G.aggs.size());
    for (Buf& a : G.acc) regrow(a, 8, 1);
    G.cap = cap;
}

// the slot table holds every group: rebuilt from the stored hashes (grown) when 2 * groups exceed it, else the groups
// [from, ngroups) inserted
static void insert_groups(Ctx* c, Groups& G, uint64_t from) {
    if (2 * G.ngroups > G.nslots) {
        while (2 * G.ngroups > G.nslots) G.nslots *= 2;
        G.slots = dev_alloc(c, G.nslots * 4);
        CPB_CUDA(cudaMemsetAsync(G.slots->p, 0xff, G.nslots * 4, c->stream));
        from = 0;
    }
    KernelTimer kt(c, "groupby_insert", (G.ngroups - from) * 16);
    const uint64_t* h = G.hash->as<uint64_t>();
    uint32_t* sl = G.slots->as<uint32_t>();
    const uint64_t mask = G.nslots - 1;
    each_row(c, G.ngroups - from, [=] __device__(uint64_t i) {
        const uint32_t g = (uint32_t)(from + i);
        for (uint64_t p = h[g] & mask;; p = (p + 1) & mask)
            if (atomicCAS(&sl[p], NO_GROUP, g) == NO_GROUP) break;
    });
}

// steps 3 and 4 for the misses of a push: new groups for their distinct keys, gid[] of every miss set
static void add_groups(Ctx* c, Groups& G, const Table& T, const KeyCols& kc, const std::vector<int>& kidx, const uint64_t* hashes,
                       uint32_t* gid, const FlagScan& ms, uint32_t blocks_for_m) {
    const uint64_t m = ms.count;
    Buf mrow = dev_alloc(c, (m + 1) * 4);
    {
        KernelTimer kt(c, "compact_ids", ms.n * 8 + m * 4);
        compact_flags(c, ms, 0, mrow->as<uint32_t>());
    }
    uint64_t nts = 64;
    while (nts < 2 * m) nts <<= 1;
    Buf tslots = dev_alloc(c, nts * 4), rep = dev_alloc(c, m * 4), first = dev_alloc(c, m * 4);
    CPB_CUDA(cudaMemsetAsync(tslots->p, 0xff, nts * 4, c->stream));
    {
        KernelTimer kt(c, "groupby_first", m * 24);
        groupby_first_kernel<<<blocks_for_m, GB_WARPS * 32, 0, c->stream>>>(kc, m, mrow->as<uint32_t>(), hashes, tslots->as<uint32_t>(), nts - 1,
                                                                             rep->as<uint32_t>());
        CPB_CUDA(cudaGetLastError());
    }
    uint32_t* rp = rep->as<uint32_t>();
    {
        KernelTimer kt(c, "groupby_flags", m * 16);
        const uint32_t* ts = tslots->as<uint32_t>();
        uint32_t* fl = first->as<uint32_t>();
        each_row(c, m, [=] __device__(uint64_t j) {
            const uint32_t f = ts[rp[j]];
            rp[j] = f;
            fl[j] = f == (uint32_t)j;
        });
    }
    const FlagScan fs = scan_flags(c, first->as<uint32_t>(), m);
    const uint64_t g0 = G.ngroups, ng = fs.count;
    if (g0 + ng > 0xFFFFFFFFull)
        throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "GroupBy: more than 2^32 - 1 groups"};
    Buf firsts = dev_alloc(c, (ng + 1) * 4);
    {
        KernelTimer kt(c, "compact_ids", m * 8 + ng * 4);
        compact_flags(c, fs, 0, firsts->as<uint32_t>());
    }
    grow(c, G, g0 + ng);
    {
        // gid of every miss; the new groups' source rows (into firsts) and hashes
        KernelTimer kt(c, "groupby_new", m * 20 + ng * 24);
        const uint32_t* pos = fs.pos->as<uint32_t>();
        const uint32_t* mr = mrow->as<uint32_t>();
        each_row(c, m, [=] __device__(uint64_t j) { gid[mr[j]] = (uint32_t)g0 + pos[rp[j]]; });
        uint32_t* fr = firsts->as<uint32_t>();
        uint64_t* gh = G.hash->as<uint64_t>() + g0;
        each_row(c, ng, [=] __device__(uint64_t i) {
            const uint32_t r = mr[fr[i]];
            fr[i] = r;
            gh[i] = hashes[r];
        });
    }
    auto view = table_view(c, T, 0, T.nrows, &kidx);
    for (size_t k = 0; k < kidx.size(); k++) view->cols[k].name = G.keys[k];
    auto rows = gather_rows(c, *view, firsts->as<uint32_t>(), (int64_t)ng);
    {
        KernelTimer kt(c, "groupby_keys", ng * 16 * kidx.size());
        const uint64_t cap = G.cap;
        for (size_t k = 0; k < kidx.size(); k++) {
            const uint32_t* off = rows->cols[k].off();
            const uint8_t* data = rows->cols[k].bytes();
            const uint8_t** pp = G.ptr->as<const uint8_t*>() + k * cap + g0;
            uint32_t* lp = G.len->as<uint32_t>() + k * cap + g0;
            each_row(c, ng, [=] __device__(uint64_t i) { pp[i] = data + off[i]; lp[i] = off[i + 1] - off[i]; });
        }
        for (size_t a = 0; a < G.aggs.size(); a++) {
            uint64_t* ac = G.acc[a]->as<uint64_t>() + g0;
            const uint64_t init = agg_init(G.aggs[a]);
            each_row(c, ng, [=] __device__(uint64_t i) { ac[i] = init; });
        }
    }
    G.rows.push_back(rows);
    G.ngroups = g0 + ng;
    insert_groups(c, G, g0);
}

void groups_push(Ctx* c, Groups& G, const Table& T) {
    const uint64_t n = (uint64_t)T.nrows;
    if (n == 0) return;
    if (n > 0xFFFFFFFFull) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "GroupBy: a push of 2^32 rows or more: push row-range slices"};
    KeyCols kc{};
    kc.n = (int)G.keys.size();
    std::vector<int> kidx;
    for (const std::string& k : G.keys) {
        const int i = T.find(k);
        if (i < 0) throw DataError{CPB_E_MISSING_COLUMN, -1, 0, false, "missing column " + go_quote(k)};
        kidx.push_back(i);
        kc.off[kidx.size() - 1] = T.cols[i].off();
        kc.data[kidx.size() - 1] = T.cols[i].bytes();
    }
    // 1. the inputs; the lowest failing row (ties to the earlier aggregate) ends the rows folded
    AggArgs aa{};
    aa.n = (int)G.aggs.size();
    std::vector<Buf> vals(G.aggs.size());
    std::optional<DataError> bad;
    for (size_t a = 0; a < G.aggs.size(); a++) {
        const GroupAgg& ag = G.aggs[a];
        aa.op[a] = ag.op; aa.kind[a] = ag.kind;
        if (ag.op == CPB_AGG_COUNT) continue;
        const int col = T.find(ag.column);
        if (col < 0) {
            if (!bad || bad->line > 0) bad = DataError{CPB_E_MISSING_COLUMN, -1, 0, false, "missing column " + go_quote(ag.column)};
            continue;
        }
        vals[a] = dev_alloc(c, n * 8);
        aa.val[a] = vals[a]->as<uint64_t>();
        const NumKind kind = ag.kind == CPB_AGG_INT ? NumKind::Int64 : NumKind::Float64;
        const NumResult r = column_as_number(c, T, col, kind, vals[a]->p, nullptr);
        if (r.nbad && (!bad || r.first_row < bad->line)) bad = number_error(ag.column, kind, r);
    }
    const uint64_t nf = bad ? bad->line : n;  // rows folded
    if (nf > 0) {
        const uint32_t blocks = (uint32_t)std::min<uint64_t>((nf + GB_WARPS * 32 - 1) / (GB_WARPS * 32), (uint64_t)c->sm_count * 16);
        Buf hashes = dev_alloc(c, nf * 8), gid = dev_alloc(c, nf * 4), miss = dev_alloc(c, nf * 4);
        {
            KernelTimer kt(c, "groupby_hash", nf * (8 + 4 * (uint64_t)kc.n));  // algorithmic bytes: offsets and hashes
            groupby_hash_kernel<<<blocks, GB_WARPS * 32, 0, c->stream>>>(kc, nf, hashes->as<uint64_t>());
            CPB_CUDA(cudaGetLastError());
        }
        {
            const StoredKeys sk{kc.n, G.cap, G.hash ? G.hash->as<uint64_t>() : nullptr, G.ptr ? G.ptr->as<const uint8_t*>() : nullptr,
                                G.len ? G.len->as<uint32_t>() : nullptr};
            KernelTimer kt(c, "groupby_probe", nf * 20);
            groupby_probe_kernel<<<blocks, GB_WARPS * 32, 0, c->stream>>>(kc, nf, hashes->as<uint64_t>(), sk, G.slots->as<uint32_t>(), G.nslots - 1,
                                                                          gid->as<uint32_t>(), miss->as<uint32_t>());
            CPB_CUDA(cudaGetLastError());
        }
        const uint64_t g0 = G.ngroups;
        const FlagScan ms = scan_flags(c, miss->as<uint32_t>(), nf);
        if (ms.count) {
            const uint32_t mb = (uint32_t)std::min<uint64_t>((ms.count + GB_WARPS * 32 - 1) / (GB_WARPS * 32), (uint64_t)c->sm_count * 16);
            add_groups(c, G, T, kc, kidx, hashes->as<uint64_t>(), gid->as<uint32_t>(), ms, mb);
        }
        // 5. (group, row) order, then one thread per run
        Buf image = dev_alloc(c, nf * 8);
        {
            KernelTimer kt(c, "groupby_image", nf * 12);
            const uint32_t* gp = gid->as<uint32_t>();
            uint64_t* im = image->as<uint64_t>();
            each_row(c, nf, [=] __device__(uint64_t i) { im[i] = gp[i]; });
        }
        uint64_t traffic = 0;
        Buf perm = sort_by_image(c, image->as<uint64_t>(), 1, nf, &traffic);
        for (size_t a = 0; a < G.aggs.size(); a++) aa.acc[a] = G.acc[a]->as<uint64_t>();
        {
            KernelTimer kt(c, "groupby_fold", nf * (8 + 8 * (uint64_t)aa.n));
            groupby_fold_kernel<<<nblk(nf, 256), 256, 0, c->stream>>>(gid->as<uint32_t>(), perm->as<uint32_t>(), nf, (uint32_t)g0, aa);
            CPB_CUDA(cudaGetLastError());
        }
    }
    if (bad) throw *bad;
}

std::shared_ptr<Table> groups_keys(Ctx* c, const Groups& G) {
    if (G.rows.empty()) {
        auto t = std::make_shared<Table>(); t->ctx = c;
        for (const std::string& k : G.keys) { Column col = empty_column(c); col.name = k; t->cols.push_back(col); }
        return t;
    }
    if (G.rows.size() == 1) return G.rows[0];
    std::vector<const Table*> parts;
    for (auto& r : G.rows) parts.push_back(r.get());
    return concat_tables(c, parts);
}

uint64_t groups_count(const Groups& G) { return G.ngroups; }

void groups_values(Ctx* c, const Groups& G, int i, void* dst) {
    need(i >= 0 && (size_t)i < G.aggs.size(), "aggregate index out of range");
    need(dst || G.ngroups == 0, "null destination");
    if (G.ngroups) CPB_CUDA(cudaMemcpyAsync(dst, G.acc[i]->p, G.ngroups * 8, cudaMemcpyDeviceToDevice, c->stream));
    sync_stream(c);
}

Ctx* groups_ctx(const Groups& G) { return G.ctx; }

}  // namespace cpb
