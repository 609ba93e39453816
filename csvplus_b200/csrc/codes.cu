// codes.cu — categorical codes of a string column (pandas.factorize(sort=False)) and the column rebuilt from codes.
//   codes[r] = the rank of row r's value among the column's distinct values in order of first appearance; the
//   dictionary is one column whose row k holds the value of code k.  Values are equal when their bytes are: any
//   length, any bytes, the empty value included.
//
// Distinct pass.  An open-addressing table of uint32 row ids in HBM: nslots = the power of two >= 2 n (load factor
// between 1/4 and 1/2, at least 64 slots), 0xFFFFFFFF = empty, linear probing from hash & (nslots - 1).  The hash
// (keyhash.cuh) is 64 bits over the value's 8-byte little-endian words (the last one zero-padded): the sum of fmix64(word ^ (i + 1) *
// golden) over the words, finished with the length.  A sum does not depend on which lane added which word, so one
// thread or a whole warp computes the same hash.  A row claims an empty slot with atomicCAS; a slot whose row has the
// same hash is compared byte for byte (a hash is never taken as equality), and on equal bytes the row is folded in
// with atomicMin, skipped when the slot already showed a lower row (slots only decrease, so a stale read can only
// cause a needless atomic: on a column of few values every row would otherwise hit the same few words).  A slot, once claimed, only ever holds rows of one value (a row never passes an empty slot, and
// atomicMin only runs on equal bytes), so every value owns exactly one slot, and when the kernel ends that slot holds
// the value's lowest row: its first appearance.
// Codes.  A row is a first row when its slot holds its own id.  The 0/1 flags are scanned (scan_flags) and compacted
// (compact_flags) into the first rows in ascending order: the code of a first row is its position in the scan, every
// other row takes the code of its slot's row.  Determinism: the slot contents after the kernel (the lowest row of each
// value), the flags, the scan and so the codes depend only on the bytes and their order, never on which thread won a
// CAS, on the grid or on the number of SMs.  The dictionary is gather_rows of the compacted first rows, or, when every
// row is a first row, a view of the column itself (no copy).
//
// Kernels (one warp per 32 consecutive rows, grid-stride):
//   codes_hash: the row's hash into hashes[r].  A value of at most LONG_BYTES = 128 bytes (16 words) is hashed by its
//     own lane; a longer one by the whole warp, 32 words (256 bytes) per round with aligned 8-byte loads, the warp
//     taking its long values one after the other.  At 128 bytes a warp round keeps at least half the lanes busy, and
//     below it the per-lane loop (at most 16 loads) costs less than the ballot / shuffle / reduction of a warp round;
//     a long value never holds 31 lanes idle while one thread walks kilobytes.
//   codes_insert: the probe of each row, with the same split: a short row probes and compares on its own lane; for a
//     long row lane 0 reads / claims the slot and the warp compares the bytes (one __any_sync per 256 bytes).  The
//     row's slot goes to rep[r].
//   codes_flags: rep[r] = the row its slot holds (its value's first row); flags[r] = rep[r] == r.
//   codes_write: codes[r] = pos[rep[r]] (pos: the exclusive scan of the flags).
// Reverse step (table_set_codes): codes_check narrows the codes to uint32 row ids of the dictionary in one pass and
// takes the lowest row whose code lies outside [0, rows of the dictionary) with atomicMin (read back once, as
// first_false_row reads its row); the column is then gather_rows of the dictionary by those ids.
// Host synchronisations: codes two (the flag count, then the dictionary's byte total, or the end of codes_write when
// the dictionary is the column), set_codes two (the check, the gathered column's byte total).  Memory of column_codes: 4 B per slot + 24 B per row besides the codes.
#include <algorithm>

#include "core.hpp"
#include "keyhash.cuh"
#include "util.cuh"

namespace cpb {

constexpr uint32_t EMPTY_SLOT = 0xFFFFFFFFu;
constexpr int CW_WARPS = 8;

struct ValCol { const uint32_t* off; const uint8_t* data; };

__global__ void __launch_bounds__(CW_WARPS * 32) codes_hash_kernel(const ValCol v, uint64_t n, uint64_t* __restrict__ hashes) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t nwarps = (uint64_t)gridDim.x * CW_WARPS;
    for (uint64_t g = (uint64_t)blockIdx.x * CW_WARPS + warp; g * 32 < n; g += nwarps) {
        const uint64_t i = g * 32 + lane;
        const bool valid = i < n;
        uint32_t len = 0;
        const uint8_t* sp = v.data;
        if (valid) { const uint32_t s = v.off[i]; len = v.off[i + 1] - s; sp += s; }
        const bool is_long = valid && len > LONG_BYTES;
        uint64_t h = 0;
        if (valid && !is_long) h = hash_thread(sp, len);
        for (uint32_t m = __ballot_sync(0xffffffffu, is_long); m; m &= m - 1) {
            const int l = __ffs(m) - 1;
            const uint8_t* lp = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(sp), l));
            const uint32_t ll = __shfl_sync(0xffffffffu, len, l);
            h = hash_warp(lp, ll, lane, l, h);
        }
        if (valid) hashes[i] = h;
    }
}

__global__ void __launch_bounds__(CW_WARPS * 32) codes_insert_kernel(const ValCol v, uint64_t n, const uint64_t* __restrict__ hashes,
                                                                     uint32_t* slots, uint64_t mask, uint32_t* __restrict__ rep) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t nwarps = (uint64_t)gridDim.x * CW_WARPS;
    for (uint64_t g = (uint64_t)blockIdx.x * CW_WARPS + warp; g * 32 < n; g += nwarps) {
        const uint64_t i = g * 32 + lane;
        const bool valid = i < n;
        uint32_t len = 0;
        uint64_t h = 0;
        const uint8_t* sp = v.data;
        if (valid) { const uint32_t s = v.off[i]; len = v.off[i + 1] - s; sp += s; h = hashes[i]; }
        const bool is_long = valid && len > LONG_BYTES;
        if (valid && !is_long) {
            const uint32_t r = (uint32_t)i;
            for (uint64_t p = h & mask;; p = (p + 1) & mask) {
                uint32_t s = slots[p];
                if (s == EMPTY_SLOT && (s = atomicCAS(&slots[p], EMPTY_SLOT, r)) == EMPTY_SLOT) { rep[r] = (uint32_t)p; break; }
                if (hashes[s] != h) continue;
                const uint32_t so = v.off[s];
                if (v.off[s + 1] - so == len && equal_thread(v.data + so, sp, len)) {
                    if (r < s) atomicMin(&slots[p], r);
                    rep[r] = (uint32_t)p;
                    break;
                }
            }
        }
        for (uint32_t m = __ballot_sync(0xffffffffu, is_long); m; m &= m - 1) {
            const int l = __ffs(m) - 1;
            const uint8_t* lp = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(sp), l));
            const uint32_t ll = __shfl_sync(0xffffffffu, len, l);
            const uint64_t lh = __shfl_sync(0xffffffffu, h, l);
            const uint32_t r = (uint32_t)(g * 32 + l);
            for (uint64_t p = lh & mask;; p = (p + 1) & mask) {
                uint32_t s = 0;
                if (lane == 0) {
                    s = slots[p];
                    if (s == EMPTY_SLOT) s = atomicCAS(&slots[p], EMPTY_SLOT, r);
                }
                s = __shfl_sync(0xffffffffu, s, 0);
                if (s == EMPTY_SLOT) { if (lane == 0) rep[r] = (uint32_t)p; break; }
                if (hashes[s] != lh) continue;  // (every lane reads the same words: the branches stay warp-uniform)
                const uint32_t so = v.off[s];
                if (v.off[s + 1] - so == ll && equal_warp(v.data + so, lp, ll, lane)) {
                    if (lane == 0) { if (r < s) atomicMin(&slots[p], r); rep[r] = (uint32_t)p; }
                    break;
                }
            }
        }
    }
}

std::shared_ptr<Table> column_codes(Ctx* c, const Table& t, int col, int64_t* codes) {
    const uint64_t n = (uint64_t)t.nrows;
    const std::vector<int> pick{col};
    auto view = table_view(c, t, 0, t.nrows, &pick);
    if (n == 0) return gather_rows(c, *view, nullptr, 0);
    if (n >= 0x80000000ull)
        throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "codes of a table of 2^31 rows or more: take codes of row-range slices"};
    const Column& cc = t.cols[col];
    const ValCol v{cc.off(), cc.bytes()};
    uint64_t nslots = 64;
    while (nslots < 2 * n) nslots <<= 1;
    Buf slots = dev_alloc(c, nslots * 4), hashes = dev_alloc(c, n * 8), rep = dev_alloc(c, n * 4), flags = dev_alloc(c, n * 4);
    CPB_CUDA(cudaMemsetAsync(slots->p, 0xff, nslots * 4, c->stream));
    const uint32_t blocks = (uint32_t)std::min<uint64_t>((n + CW_WARPS * 32 - 1) / (CW_WARPS * 32), (uint64_t)c->sm_count * 16);
    {
        KernelTimer kt(c, "codes_hash", n * 12);  // algorithmic bytes: the offsets and hashes (the value bytes are not known here)
        codes_hash_kernel<<<blocks, CW_WARPS * 32, 0, c->stream>>>(v, n, hashes->as<uint64_t>());
        CPB_CUDA(cudaGetLastError());
    }
    {
        KernelTimer kt(c, "codes_insert", n * 20);
        codes_insert_kernel<<<blocks, CW_WARPS * 32, 0, c->stream>>>(v, n, hashes->as<uint64_t>(), slots->as<uint32_t>(), nslots - 1,
                                                                      rep->as<uint32_t>());
        CPB_CUDA(cudaGetLastError());
    }
    uint32_t* r = rep->as<uint32_t>();
    {
        // r[i] = the first row of row i's value; flags: the rows that are first
        KernelTimer kt(c, "codes_flags", n * 16);
        const uint32_t* sl = slots->as<uint32_t>();
        uint32_t* fl = flags->as<uint32_t>();
        each_row(c, n, [=] __device__(uint64_t i) {
            const uint32_t f = sl[r[i]];
            r[i] = f;
            fl[i] = f == (uint32_t)i;
        });
    }
    const FlagScan s = scan_flags(c, flags->as<uint32_t>(), n);
    Buf first = dev_alloc(c, (s.count + 1) * 4);
    {
        KernelTimer kt(c, "compact_ids", n * 8 + s.count * 4);
        compact_flags(c, s, 0, first->as<uint32_t>());
    }
    {
        KernelTimer kt(c, "codes_write", n * 16);
        const uint32_t* pos = s.pos->as<uint32_t>();
        each_row(c, n, [=] __device__(uint64_t i) { codes[i] = pos[r[i]]; });
    }
    if (s.count == n) {  // every value distinct: the column is its own dictionary; the codes are complete on return
        sync_stream(c);
        return view;
    }
    return gather_rows(c, *view, first->as<uint32_t>(), (int64_t)s.count);
}

std::shared_ptr<Table> table_set_codes(Ctx* c, const Table& t, const std::string& name, const int64_t* codes, const Table& dict) {
    if (dict.cols.size() != 1)
        throw ArgError{CPB_ERR_ARG, "set_codes: the dictionary has " + std::to_string(dict.cols.size()) + " columns (want one)"};
    const uint64_t n = (uint64_t)t.nrows, nd = (uint64_t)dict.nrows;
    if (n == 0) return with_column(t, name, empty_column(c));
    if (!codes) throw ArgError{CPB_ERR_ARG, "no codes for a table with rows"};
    if (n > 0xFFFFFFFFull) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "set_codes: a table of 2^32 rows or more"};
    Buf ids = dev_alloc(c, n * 4), bad = dev_alloc(c, 8);
    CPB_CUDA(cudaMemsetAsync(bad->p, 0xff, 8, c->stream));
    {
        // ids[i] = code i, or 0 where it is outside the dictionary; *first_bad = the first such row
        KernelTimer kt(c, "codes_check", n * 12);
        uint32_t* id = ids->as<uint32_t>();
        unsigned long long* first_bad = (unsigned long long*)bad->p;
        each_row(c, n, [=] __device__(uint64_t i) {
            const int64_t k = codes[i];
            const bool ok = k >= 0 && (uint64_t)k < nd;
            id[i] = ok ? (uint32_t)k : 0;
            if (!ok) atomicMin(first_bad, (unsigned long long)i);
        });
    }
    const uint64_t row = read_back<uint64_t>(c, bad->p);
    if (row != ~0ull) {
        const int64_t k = read_back<int64_t>(c, codes + row);
        throw DataError{CPB_E_BAD_CODE, -1, row, false,
                        "row " + std::to_string(row) + ": code " + std::to_string(k) + " outside a dictionary of " + std::to_string(nd) + " values"};
    }
    auto g = gather_rows(c, dict, ids->as<uint32_t>(), (int64_t)n);
    return with_column(t, name, g->cols[0]);
}

}  // namespace cpb
