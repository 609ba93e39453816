// gather.cu — column-level primitives shared by Filter / IndexOn / Join:
//   * device-wide exclusive scans (single pass, one decoupled look-back chain for every scan);
//   * string-column gather by row ids (lengths -> scan -> byte copy) = the columnar form of the
//     per-row map copies the reference makes (Row.Select csvplus.go:122-134, mergeRows :571-583);
//   * Filter(Like/All/Any/Not) over a materialised table (csvplus.go:276-286, :1243-1293);
//   * row-wise concatenation of tables (assembling all-gathered shards).
#include <algorithm>

#include "core.hpp"
#include "pred.cuh"
#include "rowhash.cuh"
#include "util.cuh"

namespace cpb {

// ------------------------------------------------------------------ exclusive scan (uint32 in, uint32 out, uint64 total)
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 16;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// The look-back chain of one tile, run by a whole warp.  Tile t's state word is st[t * stride] (stride NC: the words of
// NC columns interleaved): bits 63:62 status (0 none, 1 aggregate, 2 inclusive prefix), bits 61:0 the value.  Publishes
// the tile's total tot, walks the predecessors 32 at a time until one holds its inclusive prefix, publishes this tile's
// and returns its exclusive prefix (every lane).
__device__ __forceinline__ unsigned long long lookback(unsigned long long* st, uint32_t stride, uint64_t tile, uint32_t tot) {
    const int lane = threadIdx.x & 31;
    if (tile == 0) {
        if (lane == 0) atomicExch(&st[0], (2ull << 62) | tot);
        return 0;
    }
    if (lane == 0) atomicExch(&st[tile * stride], (1ull << 62) | tot);
    unsigned long long excl = 0;
    for (int64_t b = (int64_t)tile - 1;; b -= 32) {
        const int64_t p = b - lane;
        unsigned long long s = 2ull << 62;
        if (p >= 0) { do { s = ld_relaxed_u64((const uint64_t*)&st[p * stride]); } while ((s >> 62) == 0); }
        const int f = __ffs(__ballot_sync(0xffffffffu, (s >> 62) == 2)) - 1;
        excl += warp_sum_u64((f < 0 || lane <= f) ? (s & ((1ull << 62) - 1)) : 0ull);
        if (f >= 0) break;
    }
    if (lane == 0) atomicExch(&st[tile * stride], (2ull << 62) | (excl + tot));
    return excl;
}

// GATHER: the scanned values are the lengths of the strings picked by `ids` (identity when null) from the offsets
// array `in` -- the length array of a gather is never materialised.
template <bool GATHER>
__global__ void __launch_bounds__(SCAN_THREADS) scan_u32_kernel(const uint32_t* __restrict__ in, const uint32_t* __restrict__ ids,
                                                                uint32_t* out, uint64_t n, unsigned long long* state,
                                                                uint32_t* ticket, unsigned long long* total) {
    __shared__ uint32_t s_tile;
    __shared__ uint32_t s_warp[SCAN_THREADS / 32];
    __shared__ unsigned long long s_prefix;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    for (;;) {
        if (tid == 0) s_tile = atomicAdd(ticket, 1u);
        __syncthreads();
        const uint64_t tile = s_tile;
        if (tile >= ntiles) break;
        const uint64_t base = tile * SCAN_TILE + (uint64_t)tid * SCAN_ITEMS;
        uint32_t v[SCAN_ITEMS];
        uint32_t sum = 0;
#pragma unroll
        for (int i = 0; i < SCAN_ITEMS; i++) {
            v[i] = 0;
            if (base + i < n) {
                if (GATHER) { const uint32_t r = ids ? ids[base + i] : (uint32_t)(base + i); v[i] = in[r + 1] - in[r]; }
                else v[i] = in[base + i];
            }
            sum += v[i];
        }
        uint32_t inc = warp_incl_scan(sum);
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        uint32_t woff = 0, tot = 0;
#pragma unroll
        for (int i = 0; i < SCAN_THREADS / 32; i++) { uint32_t t = s_warp[i]; if (i < warp) woff += t; tot += t; }
        if (warp == 0) {
            const unsigned long long excl = lookback(state, 1, tile, tot);
            if (lane == 0) { s_prefix = excl; if (tile == ntiles - 1) { *total = excl + tot; out[n] = (uint32_t)(excl + tot); } }
        }
        __syncthreads();
        uint32_t run = (uint32_t)s_prefix + woff + (inc - sum);
#pragma unroll
        for (int i = 0; i < SCAN_ITEMS; i++) { if (base + i < n) out[base + i] = run; run += v[i]; }
        __syncthreads();
    }
}

__global__ void scan_empty_kernel(uint32_t* out, unsigned long long* total) { out[0] = 0; *total = 0; }

// out may alias in; out has n+1 entries (out[n] = total, truncated to 32 bits); *total_dev holds the 64-bit total.
// gather_off != nullptr: scan the lengths off[ids[i]+1]-off[ids[i]] instead of `in` (ids may be null = identity).
static void scan_impl(Ctx* c, const uint32_t* in, const uint32_t* gather_off, const uint32_t* ids, uint32_t* out, uint64_t n,
                      uint64_t* total_dev) {
    if (n == 0) {
        KernelTimer kt(c, "scan_u32", 0);
        scan_empty_kernel<<<1, 1, 0, c->stream>>>(out, (unsigned long long*)total_dev);
        return;
    }
    uint64_t ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    Buf st = dev_alloc(c, ntiles * 8 + 64);
    CPB_CUDA(cudaMemsetAsync(st->p, 0, ntiles * 8 + 64, c->stream));
    unsigned long long* state = st->as<unsigned long long>() + 8;
    uint32_t* ticket = st->as<uint32_t>();
    uint32_t grid = (uint32_t)std::min<uint64_t>(ntiles, (uint64_t)c->sm_count * 8);
    if (gather_off) {
        KernelTimer kt(c, "scan_gather_len", n * (ids ? 16 : 12));
        scan_u32_kernel<true><<<grid, SCAN_THREADS, 0, c->stream>>>(gather_off, ids, out, n, state, ticket, (unsigned long long*)total_dev);
    } else {
        KernelTimer kt(c, "scan_u32", n * 8);
        scan_u32_kernel<false><<<grid, SCAN_THREADS, 0, c->stream>>>(in, nullptr, out, n, state, ticket, (unsigned long long*)total_dev);
    }
    CPB_CUDA(cudaGetLastError());
}
void exclusive_scan_u32(Ctx* c, const uint32_t* in, uint32_t* out, uint64_t n, uint64_t* total_dev) {
    scan_impl(c, in, nullptr, nullptr, out, n, total_dev);
}

// ------------------------------------------------------------------ compaction of flags (scan_flags / compact_flags)
__global__ void compact_kernel(const uint32_t* __restrict__ flags, const uint32_t* __restrict__ pos, uint32_t* out, uint64_t n, uint32_t add) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && flags[i]) out[pos[i]] = (uint32_t)i + add;
    if (i == 0) out[pos[n]] = (uint32_t)n + add;  // sentinel: the end of the last run when the flags mark run heads
}
FlagScan scan_flags(Ctx* c, const uint32_t* flags, uint64_t n) {
    FlagScan s{flags, n, dev_alloc(c, (n + 1) * 4), 0};
    Buf tot = dev_alloc(c, 8);
    exclusive_scan_u32(c, flags, s.pos->as<uint32_t>(), n, tot->as<uint64_t>());
    s.count = read_back<uint64_t>(c, tot->p);
    return s;
}
void compact_flags(Ctx* c, const FlagScan& s, uint32_t add, uint32_t* out) {
    if (s.n == 0) return;
    compact_kernel<<<nblk(s.n, 256), 256, 0, c->stream>>>(s.flags, s.pos->as<uint32_t>(), out, s.n, add);
    CPB_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------ gather by row ids
// One warp gathers 32 consecutive output values.  Their destination bytes are contiguous, so the lanes first
// copy their (randomly placed) source strings into a per-warp shared-memory stage laid out like the
// destination, then the warp writes the stage with aligned 16-byte stores: HBM/L2 see full sectors instead of one
// scattered byte store per lane.  ids==nullptr means identity (compaction of a view).
// Copies len bytes from an arbitrarily aligned global source with aligned 8-byte loads (two per 8 bytes at most, the
// second carried over to the next round): the lanes of a warp read unrelated strings, so every load instruction
// costs 32 L1 wavefronts and a byte-wise loop is wavefront-bound.  Source buffers are allocated in multiples of
// 512 bytes (DevBuf), so the aligned word holding the last byte is always readable.
__device__ __forceinline__ void copy_unaligned(uint8_t* q, const uint8_t* sp, uint32_t len) {
    if (len == 0) return;
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(sp) & 7u), sh = mis * 8;
    const unsigned long long* wp = reinterpret_cast<const unsigned long long*>(sp - mis);
    unsigned long long lo = __ldg(wp);
    for (uint32_t k = 0; k < len; k += 8) {
        const uint32_t rem = len - k;
        unsigned long long v = lo >> sh;
        if (mis + rem > 8) {  // bytes beyond the current word are needed (this round or the next)
            const unsigned long long hi = __ldg(++wp);
            if (sh) v |= hi << (64 - sh);
            lo = hi;
        }
#pragma unroll
        for (uint32_t b = 0; b < 8; b++) if (b < rem) q[k + b] = (uint8_t)(v >> (8 * b));
    }
}
// Writes stage bytes [sh, end) to gb (16-byte aligned, laid out like the stage): whole vectors with 16-byte
// stores, the partial first / last vector one byte per lane (lanes 0-15 / 16-31) -- no lane loops over bytes.
__device__ __forceinline__ void warp_store_stage(uint8_t* gb, const uint8_t* stage, uint32_t sh, uint32_t end, int lane) {
    for (uint32_t x = lane * 16; x + 16 <= end; x += 32 * 16)
        if (x >= sh) *reinterpret_cast<uint4*>(gb + x) = *reinterpret_cast<const uint4*>(stage + x);
    const uint32_t t0 = end & ~15u;
    const bool head = lane < 16;
    const uint32_t y = head ? (uint32_t)lane : t0 + (uint32_t)(lane - 16);
    const bool on = head ? sh != 0 : ((end & 15u) != 0 && (t0 != 0 || sh == 0));
    if (on && y >= sh && y < end) gb[y] = stage[y];
}
constexpr int GW_WARPS = 8;
constexpr int GW_STAGE = 2048;  // bytes staged per warp; longer groups take the direct path
__global__ void __launch_bounds__(GW_WARPS * 32) gather_copy_kernel(const uint32_t* __restrict__ src_off, const uint8_t* __restrict__ src,
                                                                    const uint32_t* __restrict__ ids, const uint32_t* __restrict__ dst_off,
                                                                    uint8_t* __restrict__ dst, uint64_t n) {
    __shared__ __align__(16) uint8_t stage_all[GW_WARPS][GW_STAGE + 16];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t* stage = stage_all[warp];
    const uint64_t nwarps = (uint64_t)gridDim.x * GW_WARPS;
    for (uint64_t g = (uint64_t)blockIdx.x * GW_WARPS + warp; g * 32 < n; g += nwarps) {
        const uint64_t i = g * 32 + lane;
        uint32_t s = 0, len = 0, d = 0;
        if (i < n) {
            const uint32_t r = ids ? ids[i] : (uint32_t)i;
            s = src_off[r]; len = src_off[r + 1] - s; d = dst_off[i];
        }
        const uint32_t d0 = __shfl_sync(0xffffffffu, d, 0);
        const uint64_t last = (g * 32 + 31 < n ? g * 32 + 31 : n - 1) - g * 32;
        const uint32_t dl = __shfl_sync(0xffffffffu, d + len, (int)last);
        const uint32_t total = dl - d0, sh = d0 & 15u;
        const uint8_t* sp = src + s;
        if (sh + total <= GW_STAGE) {
            copy_unaligned(stage + sh + (d - d0), sp, len);
            __syncwarp();
            warp_store_stage(dst + (d0 - sh), stage, sh, sh + total, lane);
            __syncwarp();
        } else {
            copy_unaligned(dst + d, sp, len);
        }
    }
}

// gathers several columns with ONE host synchronisation (totals of all columns read back together)
static std::vector<Column> gather_columns(Ctx* c, const std::vector<const Column*>& srcs, const uint32_t* ids, int64_t nout) {
    std::vector<Column> out(srcs.size());
    if (srcs.empty()) return out;
    Buf totals = dev_alloc(c, srcs.size() * 8);
    for (size_t k = 0; k < srcs.size(); k++) {
        out[k].name = srcs[k]->name;
        out[k].offsets = dev_alloc(c, ((size_t)nout + 1) * 4);
        uint32_t* o = out[k].offsets->as<uint32_t>();
        scan_impl(c, nullptr, srcs[k]->off(), ids, o, (uint64_t)nout, totals->as<uint64_t>() + k);
    }
    const std::vector<uint64_t> tot = read_back<uint64_t>(c, totals->p, srcs.size());
    for (size_t k = 0; k < srcs.size(); k++) {
        if (tot[k] > 0xffffffffull) throw DataError{CPB_E_TOO_LARGE, (int)k, 0, false, "a result column exceeds 4 GiB; process in smaller batches"};
        out[k].data = dev_alloc(c, tot[k] + 16);
        if (nout && tot[k]) {
            KernelTimer kt(c, "gather_copy", 2 * tot[k] + (uint64_t)nout * 12);
            const uint32_t gblocks = (uint32_t)std::min<uint64_t>(((uint64_t)nout + GW_WARPS * 32 - 1) / (GW_WARPS * 32), (uint64_t)c->sm_count * 16);
            gather_copy_kernel<<<gblocks, GW_WARPS * 32, 0, c->stream>>>(srcs[k]->off(), srcs[k]->bytes(), ids,
                                                                              out[k].offsets->as<uint32_t>(), out[k].data->as<uint8_t>(), (uint64_t)nout);
            CPB_CUDA(cudaGetLastError());
        }
    }
    return out;
}

std::shared_ptr<Table> gather_rows(Ctx* c, const Table& t, const uint32_t* row_ids, int64_t nout) {
    auto r = std::make_shared<Table>(); r->ctx = c; r->nrows = nout; r->first_line = t.first_line;
    // columns sharing buffers (AssumeHeader aliases) are gathered once
    std::vector<const Column*> uniq; std::vector<int> which(t.cols.size());
    for (size_t i = 0; i < t.cols.size(); i++) {
        int f = -1;
        for (size_t u = 0; u < uniq.size(); u++)
            if (uniq[u]->offsets == t.cols[i].offsets && uniq[u]->data == t.cols[i].data && uniq[u]->row0 == t.cols[i].row0) f = (int)u;
        if (f < 0) { f = (int)uniq.size(); uniq.push_back(&t.cols[i]); }
        which[i] = f;
    }
    auto g = gather_columns(c, uniq, row_ids, nout);
    for (size_t i = 0; i < t.cols.size(); i++) { Column col = g[which[i]]; col.name = t.cols[i].name; r->cols.push_back(col); }
    return r;
}

// the rows of t whose flag is set: the flags scanned and counted (one host synchronisation), compacted to row ids
// (timed as compact_ids) and the rows gathered
std::shared_ptr<Table> rows_where(Ctx* c, const Table& t, const uint32_t* flags, uint64_t* first) {
    const uint64_t n = (uint64_t)t.nrows;
    const FlagScan s = scan_flags(c, flags, n);
    Buf ids = dev_alloc(c, (s.count + 1) * 4);
    {
        KernelTimer kt(c, "compact_ids", n * 8 + s.count * 4);
        compact_flags(c, s, 0, ids->as<uint32_t>());
    }
    if (first) *first = s.count ? read_back<uint32_t>(c, ids->p) : 0;
    return gather_rows(c, t, ids->as<uint32_t>(), (int64_t)s.count);
}

// ------------------------------------------------------------------ row slots: one random access per gathered index row
// A join reads index rows in probe order, i.e. at random: per output column that is one access to the offsets and
// one to the bytes, each a 64-byte DRAM granule once the index outgrows L2 (many times the
// DRAM traffic of the bytes gathered).  Short rows are therefore re-laid once per index as fixed-size slots (all output columns back to back) +
// one packed word of lengths; a gather then costs one L2-friendly 4-byte read (lengths -> offsets of all columns in
// one scan) and one slot read (bytes of all columns in one pass).
constexpr int RS_MAXC = 4;       // columns per slot set (lengths are 8 bits each in one word)
constexpr uint32_t RS_MAXS = 64; // bytes per slot
struct SlotCols { int nc; const uint32_t* off[RS_MAXC]; const uint8_t* data[RS_MAXC]; };
struct SlotOut { uint32_t* off[RS_MAXC]; uint8_t* data[RS_MAXC]; };

// (`perm`: slot r holds source row perm[r] — the slots are laid out in sorted order straight from the unsorted rows
// of the index source; null = identity)
__global__ void __launch_bounds__(256) slot_lens_kernel(SlotCols sc, const uint32_t* __restrict__ perm, uint64_t n, uint32_t* lens, uint32_t* stat) {  // stat: [0] max row bytes, [1] a value > 255 bytes
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t tot = 0, packed = 0, bad = 0;
    if (r < n) {
        const uint64_t sr = perm ? perm[r] : r;
        for (int c = 0; c < sc.nc; c++) {
            const uint32_t l = sc.off[c][sr + 1] - sc.off[c][sr];
            bad |= l > 255u;
            packed |= (l & 255u) << (8 * c);
            tot += l;
        }
        lens[r] = packed;
    }
    // one global atomic per block (every block hits the same word: same-address atomics serialise in L2)
    __shared__ uint32_t s_max[8], s_bad[8];
    tot = __reduce_max_sync(0xffffffffu, tot);
    bad = __any_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0) { s_max[threadIdx.x >> 5] = tot; s_bad[threadIdx.x >> 5] = bad; }
    __syncthreads();
    if (threadIdx.x < 32) {
        const bool in = threadIdx.x < (blockDim.x >> 5);
        tot = __reduce_max_sync(0xffffffffu, in ? s_max[threadIdx.x] : 0u);
        bad = __any_sync(0xffffffffu, in && s_bad[threadIdx.x]);
        if (threadIdx.x == 0) { atomicMax(&stat[0], tot); if (bad) stat[1] = 1u; }
    }
}
// one block lays out 256 consecutive slots in shared memory (row stride padded to an odd number of words: no bank
// conflicts) and writes them with coalesced 16-byte stores
constexpr uint32_t RS_PAD = 4;
__global__ void __launch_bounds__(256) slot_fill_kernel(SlotCols sc, const uint32_t* __restrict__ perm, uint64_t n, uint32_t S, uint8_t* slots) {
    __shared__ __align__(16) uint8_t sm[256 * (RS_MAXS + RS_PAD)];
    const uint64_t r0 = (uint64_t)blockIdx.x * 256, r = r0 + threadIdx.x;
    uint8_t* q = sm + threadIdx.x * (S + RS_PAD);
    if (r < n) {
        const uint64_t sr = perm ? perm[r] : r;
        uint32_t pos = 0;
        for (int c = 0; c < sc.nc; c++) {
            const uint32_t s = sc.off[c][sr], l = sc.off[c][sr + 1] - s;
            copy_unaligned(q + pos, sc.data[c] + s, l);
            pos += l;
        }
        for (; pos < S; pos++) q[pos] = 0;
    }
    __syncthreads();
    const uint32_t rows = (uint32_t)(n - r0 < 256 ? n - r0 : 256), wps = S / 4;  // words per slot
    uint32_t* g = reinterpret_cast<uint32_t*>(slots + r0 * S);
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(sm);
    for (uint32_t x = threadIdx.x; x < rows * wps; x += 256) g[x] = sw[(x / wps) * (wps + RS_PAD / 4) + x % wps];
}

// Row-carrying hash table: probe row i looks its key up with one 32-byte slot read; the lengths of the output columns
// (8 bits each, as row slots pack them) go to lens[i], their bytes back to back to scratch[i] (zero on a miss), both
// written sequentially, and the hits are counted into *matches.  (Probing inside the length scan, 8 rows per thread,
// needs ~170 registers: one CTA per SM, and the kernel ran latency-bound at 3.6x this one + the scan.)
__global__ void __launch_bounds__(256) rowhash_probe_kernel(KeyDesc kd, uint64_t np, const RowSlot* __restrict__ slots, uint64_t nslots,
                                                            uint64_t rmask, int npay, uint32_t sel, uint32_t* lens, uint4* scratch,
                                                            unsigned long long* matches) {
    unsigned long long hits = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (uint64_t)gridDim.x * blockDim.x) {
        unsigned long long k0; uint32_t k1;
        uint64_t s = rh_start(kd, i, nslots, k0, k1);
        uint4 h = rh_header(slots, s), v = __ldg(&slots[s].pay);  // one sector, both halves
        const uint64_t s0 = s;
        const bool found = rh_walk(slots, rmask, k0, k1, s, h);
        if (found && s != s0) v = __ldg(&slots[s].pay);
        unsigned long long a = 0, b = 0;
        uint32_t p = 0;
        if (found) {
            const unsigned long long pa = ((unsigned long long)v.y << 32) | v.x, pb = ((unsigned long long)v.w << 32) | v.z;
            uint32_t pos = 0, opos = 0;
            int oc = 0;
#pragma unroll
            for (int j = 0; j < RH_MAXC; j++) {
                if (j >= npay) break;
                const uint32_t l = (h.w >> (5 * j)) & 31u;
                if (sel >> j & 1u) {
                    unsigned long long x, y;
                    take16(pa, pb, pos, l, x, y);
                    or_at16(a, b, opos, x, y);
                    p |= l << (8 * oc);
                    opos += l; oc++;
                }
                pos += l;
            }
            hits++;
        }
        lens[i] = p;
        scratch[i] = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
    }
    hits = warp_sum_u64(hits);
    if ((threadIdx.x & 31) == 0 && hits) atomicAdd(matches, hits);
}

// exclusive scans of the NC length fields (8 bits each) of row i's packed lengths in one pass (warp c runs column c's
// look-back).  Src::load(base, n, p) gives the packed lengths of rows [base, base + LS_ITEMS) (0 past n).  A body of its
// own: folded into one kernel with scan_u32_kernel, the scan_gather_len instantiation took 40 registers instead of 32.
constexpr int LS_ITEMS = 8;
constexpr int LS_TILE = SCAN_THREADS * LS_ITEMS;
struct LensById {  // row slots: lens[ids[i]]
    const uint32_t* __restrict__ lens;
    const uint32_t* __restrict__ ids;
    __device__ __forceinline__ void load(uint64_t base, uint64_t n, uint32_t (&p)[LS_ITEMS]) const {
        if (base + LS_ITEMS <= n) {
            const uint4 a = *reinterpret_cast<const uint4*>(ids + base), b = *reinterpret_cast<const uint4*>(ids + base + 4);
            p[0] = lens[a.x]; p[1] = lens[a.y]; p[2] = lens[a.z]; p[3] = lens[a.w];
            p[4] = lens[b.x]; p[5] = lens[b.y]; p[6] = lens[b.z]; p[7] = lens[b.w];
        } else {
#pragma unroll
            for (int i = 0; i < LS_ITEMS; i++) p[i] = base + i < n ? lens[ids[base + i]] : 0u;
        }
    }
};
struct LensSeq {  // row-carrying hash table: lens[i], written by rowhash_probe_kernel
    const uint32_t* __restrict__ lens;
    __device__ __forceinline__ void load(uint64_t base, uint64_t n, uint32_t (&p)[LS_ITEMS]) const {
        if (base + LS_ITEMS <= n) {
            const uint4 a = *reinterpret_cast<const uint4*>(lens + base), b = *reinterpret_cast<const uint4*>(lens + base + 4);
            p[0] = a.x; p[1] = a.y; p[2] = a.z; p[3] = a.w; p[4] = b.x; p[5] = b.y; p[6] = b.z; p[7] = b.w;
        } else {
#pragma unroll
            for (int i = 0; i < LS_ITEMS; i++) p[i] = base + i < n ? lens[base + i] : 0u;
        }
    }
};
template <int NC, class Src>
__global__ void __launch_bounds__(SCAN_THREADS) scan_lens_kernel(const Src src, uint64_t n, SlotOut out, unsigned long long* state, uint32_t* ticket,
                                                                 unsigned long long* totals) {
    __shared__ uint32_t s_tile;
    __shared__ uint32_t s_warp[NC][SCAN_THREADS / 32];
    __shared__ unsigned long long s_prefix[NC];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t ntiles = (n + LS_TILE - 1) / LS_TILE;
    for (;;) {
        if (tid == 0) s_tile = atomicAdd(ticket, 1u);
        __syncthreads();
        const uint64_t tile = s_tile;
        if (tile >= ntiles) break;
        const uint64_t base = tile * LS_TILE + (uint64_t)tid * LS_ITEMS;
        uint32_t p[LS_ITEMS];
        src.load(base, n, p);
        uint32_t sum[NC], inc[NC];
#pragma unroll
        for (int c = 0; c < NC; c++) {
            sum[c] = 0;
#pragma unroll
            for (int i = 0; i < LS_ITEMS; i++) sum[c] += (p[i] >> (8 * c)) & 255u;
            inc[c] = warp_incl_scan(sum[c]);
            if (lane == 31) s_warp[c][warp] = inc[c];
        }
        __syncthreads();
        if (warp < NC) {
            const int c = warp;
            uint32_t tot = 0;
#pragma unroll
            for (int i = 0; i < SCAN_THREADS / 32; i++) tot += s_warp[c][i];
            const unsigned long long excl = lookback(state + c, NC, tile, tot);  // state[tile * NC + c]
            if (lane == 0) {
                s_prefix[c] = excl;
                if (tile == ntiles - 1) totals[c] = excl + tot;
            }
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < NC; c++) {
            uint32_t run = (uint32_t)s_prefix[c] + (inc[c] - sum[c]);
#pragma unroll
            for (int i = 0; i < SCAN_THREADS / 32; i++) if (i < warp) run += s_warp[c][i];
            uint32_t* o = out.off[c];
            if (base + LS_ITEMS <= n) {
                uint32_t v[LS_ITEMS];
#pragma unroll
                for (int i = 0; i < LS_ITEMS; i++) { v[i] = run; run += (p[i] >> (8 * c)) & 255u; }
                *reinterpret_cast<uint4*>(o + base) = make_uint4(v[0], v[1], v[2], v[3]);
                *reinterpret_cast<uint4*>(o + base + 4) = make_uint4(v[4], v[5], v[6], v[7]);
            } else {
#pragma unroll
                for (int i = 0; i < LS_ITEMS; i++) { if (base + i < n) o[base + i] = run; run += (p[i] >> (8 * c)) & 255u; }
            }
            if (base < n && n <= base + LS_ITEMS) o[n] = run;  // (the thread holding the last row: the total; a column index
                                                                // taken from the warp number would put `out` on the stack)
        }
        __syncthreads();
    }
}

// Stores bytes [lo, hi) (lo < hi <= 16) of the vector v to gb (16-byte aligned) with naturally aligned 8/4/2/1-byte
// stores (at most 6): the partial first / last vector of a warp's destination range, whose other bytes belong to the
// neighbouring groups.
__device__ __forceinline__ void store_part16(uint8_t* gb, uint4 v, uint32_t lo, uint32_t hi) {
    const unsigned long long h0 = ((unsigned long long)v.y << 32) | v.x, h1 = ((unsigned long long)v.w << 32) | v.z;
    for (uint32_t x = lo; x < hi;) {
        const unsigned long long w = (x < 8 ? h0 : h1) >> (8 * (x & 7));
        if ((x & 7) == 0 && x + 8 <= hi) { *reinterpret_cast<unsigned long long*>(gb + x) = w; x += 8; }
        else if ((x & 3) == 0 && x + 4 <= hi) { *reinterpret_cast<uint32_t*>(gb + x) = (uint32_t)w; x += 4; }
        else if ((x & 1) == 0 && x + 2 <= hi) { *reinterpret_cast<uint16_t*>(gb + x) = (uint16_t)w; x += 2; }
        else { gb[x] = (uint8_t)w; x += 1; }
    }
}
// ORs the len bytes at slot[pos..] into the zeroed stage at byte q, one aligned 4-byte word at a time: each word is
// two slot words funnel-shifted into place and masked to the value's bytes.  A word the value shares with its
// neighbours' values is completed by their ORs.  Reads the slot word before and after the value (never used).
__device__ __forceinline__ void or_value(uint8_t* stage, uint32_t q, const uint8_t* slot, uint32_t pos, uint32_t len) {
    if (len == 0) return;
    const uint32_t b = q & 3u, e = (pos & 3u) + 4u - b;  // target word j = slot bytes from (pos & ~3) + 4j + e - 4
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(slot + (pos & ~3u)) + (e >> 2) - 1;
    uint32_t* tw = reinterpret_cast<uint32_t*>(stage + (q & ~3u));
    const uint32_t shift = 8 * (e & 3u), nw = (b + len + 3) >> 2, endb = b + len - 4 * (nw - 1);  // endb in 1..4
    uint32_t cur = sw[0];
    for (uint32_t j = 0; j < nw; j++) {
        const uint32_t nxt = sw[j + 1];
        uint32_t m = j == 0 ? 0xffffffffu << (8 * b) : 0xffffffffu;
        if (j == nw - 1 && endb < 4) m &= (1u << (8 * endb)) - 1u;
        atomicOr(tw + j, __funnelshift_r(cur, nxt, shift) & m);
        cur = nxt;
    }
}
// One warp gathers 32 consecutive output rows: every lane pulls its row's slot into shared memory with 16-byte
// loads (the one random access).  The lanes then OR their values, word by word, into a zeroed staging buffer laid
// out like the destination (all columns of the group, one 16-byte aligned region each), and the warp writes every
// column's region in ONE pass of aligned 16-byte stores, the partial first / last vector of a column with a few
// aligned narrower stores.  No lane loops over the bytes of a value.  A column whose region does not fit the stage
// any more is copied straight to its destination.  Row i's slot is slots[ids[i]], or slots[i] when ids is null.
constexpr uint32_t SC_STRIDE_PAD = 12;  // slot stride S + 12 bytes: an odd number of words, and room for or_value's over-read
template <int NC, int SV>  // SV: 16-byte vectors held per prefetched slot (S <= 16 SV)
__global__ void __launch_bounds__(GW_WARPS * 32) slot_copy_kernel(const uint8_t* __restrict__ slots, uint32_t S, const uint32_t* __restrict__ ids,
                                                                  SlotOut out, uint64_t n) {
    // (16 bytes ahead of the first slot: or_value may read the word before a value)
    __shared__ __align__(16) uint8_t slot_sm[16 + GW_WARPS * 32 * (RS_MAXS + SC_STRIDE_PAD)];
    __shared__ __align__(16) uint8_t stage_all[GW_WARPS][GW_STAGE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t* stage = stage_all[warp];
    uint8_t* myslot = slot_sm + 16 + (warp * 32 + lane) * (S + SC_STRIDE_PAD);
    const uint64_t nwarps = (uint64_t)gridDim.x * GW_WARPS;
    // the slot and the destination offsets of a lane's row are fetched one round ahead, so that the random slot read
    // of the next group is in flight while this group is laid out and stored
    uint4 v[SV];
    uint32_t nd[NC], nlen[NC];
    auto fetch = [&](uint64_t g) {
        const uint64_t i = g * 32 + lane;
#pragma unroll
        for (int c = 0; c < NC; c++) { nd[c] = 0; nlen[c] = 0; }
        if (i < n) {
            const uint4* sp = reinterpret_cast<const uint4*>(slots + (ids ? (uint64_t)ids[i] : i) * S);
#pragma unroll
            for (int j = 0; j < SV; j++) if (j < (int)(S / 16)) v[j] = __ldg(sp + j);
#pragma unroll
            for (int c = 0; c < NC; c++) { nd[c] = out.off[c][i]; nlen[c] = out.off[c][i + 1] - nd[c]; }
        }
    };
    uint64_t g = (uint64_t)blockIdx.x * GW_WARPS + warp;
    fetch(g);
    for (; g * 32 < n; g += nwarps) {
        const uint64_t i = g * 32 + lane;
        const bool valid = i < n;
        if (valid) {
#pragma unroll
            for (int j = 0; j < SV; j++)
                if (j < (int)(S / 16)) {
                    uint32_t* w = reinterpret_cast<uint32_t*>(myslot) + 4 * j;
                    w[0] = v[j].x; w[1] = v[j].y; w[2] = v[j].z; w[3] = v[j].w;
                }
        }
        // per column: this lane's destination offset and length; the group's stage region [base, base + 16 nv), head
        // shift sh (stage byte sh = destination byte d0) and byte count
        uint32_t d[NC], len[NC], d0[NC], sh[NC], total[NC], base[NC], nv[NC];
#pragma unroll
        for (int c = 0; c < NC; c++) { d[c] = nd[c]; len[c] = nlen[c]; }
        fetch(g + nwarps);
        const uint64_t last = (g * 32 + 31 < n ? g * 32 + 31 : n - 1) - g * 32;
        uint32_t used = 0;
#pragma unroll
        for (int c = 0; c < NC; c++) {
            d0[c] = __shfl_sync(0xffffffffu, d[c], 0);
            total[c] = __shfl_sync(0xffffffffu, d[c] + len[c], (int)last) - d0[c];
            sh[c] = d0[c] & 15u;
            nv[c] = total[c] ? (sh[c] + total[c] + 15) / 16 : 0;
            base[c] = used;
            if (used + nv[c] * 16 <= GW_STAGE) used += nv[c] * 16;
            else nv[c] = ~0u;  // direct
        }
        for (uint32_t x = lane * 16; x < used; x += 32 * 16) *reinterpret_cast<uint4*>(stage + x) = make_uint4(0, 0, 0, 0);
        __syncwarp();
        uint32_t pos = 0;
#pragma unroll
        for (int c = 0; c < NC; c++) {
            if (nv[c] != ~0u) {
                or_value(stage, base[c] + sh[c] + (d[c] - d0[c]), myslot, pos, len[c]);
            } else {
                uint8_t* dp = out.data[c] + d[c];
                for (uint32_t k = 0; k < len[c]; k++) dp[k] = myslot[pos + k];
            }
            pos += len[c];
        }
        __syncwarp();
        for (uint32_t x = lane * 16; x < used; x += 32 * 16) {
            uint8_t* gb = nullptr;
            uint32_t lo = 0, hi = 0;
#pragma unroll
            for (int c = 0; c < NC; c++)
                if (nv[c] != ~0u && x >= base[c] && x < base[c] + nv[c] * 16) {
                    const uint32_t r = x - base[c];  // vector r / 16 of column c's region
                    gb = out.data[c] + (d0[c] - sh[c]) + r;
                    lo = sh[c] > r ? sh[c] - r : 0;
                    hi = min(sh[c] + total[c] - r, 16u);
                }
            const uint4 v = *reinterpret_cast<const uint4*>(stage + x);
            if (lo == 0 && hi == 16) *reinterpret_cast<uint4*>(gb) = v;
            else store_part16(gb, v, lo, hi);
        }
        __syncwarp();  // the slots and the stage are overwritten by the next round
    }
}

static RowSlots& ensure_row_slots(Ctx* c, Index& ix, const std::vector<int>& cols, RowOrder order) {
    std::lock_guard<std::mutex> lk(ix.mu);
    auto& smap = ix.derived.row_slots;
    auto it = smap.find({order, cols});
    if (it != smap.end()) { wait_ready(c, it->second.ready); return it->second; }
    RowSlots rs;
    // source order: slot r = source row r (filled sequentially); sorted order: the sorted rows if they exist, else the
    // source rows through the permutation
    const bool by_src = order == RowOrder::source;
    const Table& t = by_src ? *ix.src : (ix.table ? *ix.table : *ix.src);
    const uint32_t* perm = (by_src || ix.table) ? nullptr : ix.perm->as<uint32_t>();
    const uint64_t n = (uint64_t)ix.nrows;
    if (n > 0 && !cols.empty() && cols.size() <= (size_t)RS_MAXC) {
        SlotCols sc{};
        sc.nc = (int)cols.size();
        for (int k = 0; k < sc.nc; k++) { sc.off[k] = t.cols[cols[k]].off(); sc.data[k] = t.cols[cols[k]].bytes(); }
        Buf lens = dev_alloc_owned(ix.ctx, c, n * 4), stat = dev_alloc(c, 8);  // kept structures: the index owner's pool
        CPB_CUDA(cudaMemsetAsync(stat->p, 0, 8, c->stream));
        uint64_t col_bytes = n * 4 * sc.nc;
        {
            KernelTimer kt(c, "slot_build", col_bytes + n * 4);
            slot_lens_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(sc, perm, n, lens->as<uint32_t>(), stat->as<uint32_t>());
            CPB_CUDA(cudaGetLastError());
        }
        const std::vector<uint32_t> hs = read_back<uint32_t>(c, stat->p, 2);
        if (hs[1] == 0 && hs[0] <= RS_MAXS) {
            rs.S = std::max<uint32_t>(16, (hs[0] + 15) & ~15u);
            rs.slots = dev_alloc_owned(ix.ctx, c, n * rs.S);
            rs.lens = lens;
            KernelTimer kt(c, "slot_build", n * rs.S * 2);
            slot_fill_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(sc, perm, n, rs.S, rs.slots->as<uint8_t>());
            CPB_CUDA(cudaGetLastError());
            rs.usable = true;
        }
    }
    rs.ready = record_ready(c);  // another context (stream) that finds it in the map waits for this event, not the host
    return smap.emplace(std::make_pair(order, cols), std::move(rs)).first->second;
}

// Columns `names` of n rows from slots of S bytes: the offsets scanned from the packed lengths `src` gives
// (scan_lens_kernel), ONE host synchronisation for the column totals and *counter (the 64-bit count at counter_dev,
// when given), then the bytes copied by slot_copy_kernel from slot ids[i] (slot i when ids is null).
template <class Src>
static std::vector<Column> slot_gather(Ctx* c, const std::vector<std::string>& names, uint64_t n, const Src& src, const char* scan_name,
                                       uint64_t scan_bytes, const uint8_t* slots, uint32_t S, const uint32_t* ids,
                                       const unsigned long long* counter_dev, uint64_t* counter) {
    const int nc = (int)names.size();
    SlotOut so{};
    std::vector<Column> out(nc);
    for (int k = 0; k < nc; k++) {
        out[k].name = names[k];
        out[k].offsets = dev_alloc(c, (n + 1) * 4);
        so.off[k] = out[k].offsets->as<uint32_t>();
    }
    const uint64_t ntiles = (n + LS_TILE - 1) / LS_TILE;
    Buf st = dev_alloc(c, ntiles * nc * 8 + 64 + RS_MAXC * 8);
    CPB_CUDA(cudaMemsetAsync(st->p, 0, ntiles * nc * 8 + 64 + RS_MAXC * 8, c->stream));
    uint32_t* ticket = st->as<uint32_t>();
    unsigned long long* totals = st->as<unsigned long long>() + 1;  // [RS_MAXC]: *counter_dev
    unsigned long long* state = st->as<unsigned long long>() + 8 + RS_MAXC;
    {
        KernelTimer kt(c, scan_name, scan_bytes);
        const uint32_t grid = (uint32_t)std::min<uint64_t>(ntiles, (uint64_t)c->sm_count * 8);
#define CPB_LS(NC) scan_lens_kernel<NC, Src><<<grid, SCAN_THREADS, 0, c->stream>>>(src, n, so, state, ticket, totals)
        switch (nc) { case 1: CPB_LS(1); break; case 2: CPB_LS(2); break; case 3: CPB_LS(3); break; default: CPB_LS(4); break; }
#undef CPB_LS
        CPB_CUDA(cudaGetLastError());
    }
    if (counter_dev) CPB_CUDA(cudaMemcpyAsync(totals + RS_MAXC, counter_dev, 8, cudaMemcpyDeviceToDevice, c->stream));
    const std::vector<uint64_t> ht = read_back<uint64_t>(c, totals, RS_MAXC + 1);
    if (counter) *counter = ht[RS_MAXC];
    uint64_t all = 0;
    for (int k = 0; k < nc; k++) {
        if (ht[k] > 0xffffffffull) throw DataError{CPB_E_TOO_LARGE, k, 0, false, "a result column exceeds 4 GiB; process in smaller batches"};
        out[k].data = dev_alloc(c, ht[k] + 16);
        so.data[k] = out[k].data->as<uint8_t>();
        all += ht[k];
    }
    {
        KernelTimer kt(c, "slot_copy", 2 * all + n * (4 + 4 * (uint64_t)nc));
        const uint32_t gblocks = (uint32_t)std::min<uint64_t>((n + GW_WARPS * 32 - 1) / (GW_WARPS * 32), (uint64_t)c->sm_count * 16);
#define CPB_SC2(NC, SV) slot_copy_kernel<NC, SV><<<gblocks, GW_WARPS * 32, 0, c->stream>>>(slots, S, ids, so, n)
#define CPB_SC(NC) (S <= 16 ? CPB_SC2(NC, 1) : S <= 32 ? CPB_SC2(NC, 2) : CPB_SC2(NC, 4))
        switch (nc) { case 1: CPB_SC(1); break; case 2: CPB_SC(2); break; case 3: CPB_SC(3); break; default: CPB_SC(4); break; }
#undef CPB_SC
#undef CPB_SC2
        CPB_CUDA(cudaGetLastError());
    }
    return out;
}

std::shared_ptr<Table> gather_index_rows(Ctx* c, Index& ix, const std::vector<int>& cols, const uint32_t* ids, int64_t nout, RowOrder order) {
    if (cols.empty()) {  // nothing to gather (a join whose index columns are all key columns): no slots, no sorted rows
        auto r = std::make_shared<Table>(); r->ctx = c; r->nrows = nout; r->first_line = ix.schema().first_line;
        return r;
    }
    auto plain = [&]() {  // per-column gather: from the source rows (ids = source rows), or from the physically sorted rows
        std::shared_ptr<Table> keep = order == RowOrder::source ? ix.src : sorted_table(c, ix);
        const Table& st = *keep;
        Table sub; sub.ctx = c; sub.nrows = st.nrows; sub.first_line = st.first_line;
        for (int ci : cols) sub.cols.push_back(st.cols[ci]);
        return gather_rows(c, sub, ids, nout);
    };
    bool use = ids != nullptr && nout > 0 && cols.size() <= (size_t)RS_MAXC;
    if (use) {
        bool built;
        { std::lock_guard<std::mutex> lk(ix.mu); built = ix.derived.row_slots.count({order, cols}) != 0; }
        if (!built && nout < ix.nrows) use = false;  // laying the slots out costs about one gather of the whole index
    }
    if (!use) return plain();
    RowSlots& rs = ensure_row_slots(c, ix, cols, order);
    if (!rs.usable) return plain();
    const Table& t = ix.schema();
    std::vector<std::string> names;
    for (int ci : cols) names.push_back(t.cols[ci].name);
    auto r = std::make_shared<Table>(); r->ctx = c; r->nrows = nout; r->first_line = t.first_line;
    const uint64_t n = (uint64_t)nout;
    r->cols = slot_gather(c, names, n, LensById{rs.lens->as<uint32_t>(), ids}, "slot_scan_lens", n * (8 + 4 * (uint64_t)cols.size()),
                          rs.slots->as<uint8_t>(), rs.S, ids, nullptr, nullptr);
    return r;
}

std::shared_ptr<Table> rowhash_gather(Ctx* c, Index& ix, const Table& probe, const std::vector<int>& pidx, const std::vector<int>& cols,
                                      uint64_t* matches) {
    const RowHash& rh = ix.derived.rowhash;
    const Table& t = ix.schema();
    const uint64_t np = (uint64_t)probe.nrows;
    KeyDesc kd{};
    describe_keys(c, probe, pidx, ix.key_width, kd);
    std::vector<std::string> names;
    uint32_t sel = 0;
    for (int ci : cols) {  // cols is a subset of the payload in payload order (both in schema order)
        names.push_back(t.cols[ci].name);
        sel |= 1u << (int)(std::find(rh.cols.begin(), rh.cols.end(), ci) - rh.cols.begin());
    }
    Buf lens = dev_alloc(c, np * 4), scratch = dev_alloc(c, np * RH_PAY), cnt = dev_alloc(c, 8);
    CPB_CUDA(cudaMemsetAsync(cnt->p, 0, 8, c->stream));
    {
        KernelTimer kt(c, "rowhash_probe", np * ((uint64_t)kd.words * 8 + 4 * (uint64_t)kd.nkeys + sizeof(RowSlot) + RH_PAY + 4));
        const uint32_t grid = (uint32_t)std::min<uint64_t>(nblk(np, 256), (uint64_t)c->sm_count * 16);
        rowhash_probe_kernel<<<grid, 256, 0, c->stream>>>(kd, np, rh.slots->as<RowSlot>(), rh.nslots, rh.region - 1ull, (int)rh.cols.size(), sel,
                                                          lens->as<uint32_t>(), scratch->as<uint4>(), cnt->as<unsigned long long>());
        CPB_CUDA(cudaGetLastError());
    }
    auto r = std::make_shared<Table>(); r->ctx = c; r->nrows = (int64_t)np; r->first_line = t.first_line;
    r->cols = slot_gather(c, names, np, LensSeq{lens->as<uint32_t>()}, "rowhash_scan_lens", np * (4 + 4 * (uint64_t)cols.size()),
                          scratch->as<uint8_t>(), RH_PAY, nullptr, cnt->as<unsigned long long>(), matches);
    return r;
}

// ------------------------------------------------------------------ Filter over a table
struct FilterCols { const uint32_t* off[MAXTERMS]; const uint8_t* data[MAXTERMS]; };

// the eq word of row i over the literal terms (the terms in `skip`, set terms, are left 0)
__device__ __forceinline__ uint32_t literal_terms(const FilterCols& cols, const PredProg& prog, const uint8_t* __restrict__ lits, uint64_t i,
                                                  uint32_t skip) {
    uint32_t eq = 0;
    for (int t = 0; t < prog.nterms; t++) {
        if ((skip >> t) & 1u) continue;
        const uint32_t* off = cols.off[t];
        uint32_t s = off[i], len = off[i + 1] - s;
        if (len != prog.term_len[t]) continue;
        const uint8_t* p = cols.data[t] + s;
        const uint8_t* l = lits + prog.term_off[t];
        bool ok = true;
        for (uint32_t k = 0; k < len; k++) if (p[k] != l[k]) { ok = false; break; }
        if (ok) eq |= 1u << t;
    }
    return eq;
}
__global__ void filter_flags_kernel(FilterCols cols, PredProg prog, const uint8_t* __restrict__ lits, uint32_t* flags, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    flags[i] = eval_pred(prog, literal_terms(cols, prog, lits, i, 0u)) ? 1u : 0u;
}
// A program with set terms: term t of `sets` takes its bit from hit[t][i], the probe of the term's index (key_flags).
// (__grid_constant__: the arrays indexed by term are read where the parameters are, not copied to each thread's stack)
struct SetHits { const uint32_t* hit[MAXTERMS]; };
__global__ void filter_set_kernel(const __grid_constant__ FilterCols cols, const __grid_constant__ PredProg prog, const uint8_t* __restrict__ lits,
                                  const __grid_constant__ SetHits hits, uint32_t sets, uint32_t* flags, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t eq = literal_terms(cols, prog, lits, i, sets);
    for (uint32_t m = sets; m; m &= m - 1) {
        const int t = __ffs(m) - 1;
        eq |= (hits.hit[t][i] & 1u) << t;
    }
    flags[i] = eval_pred(prog, eq) ? 1u : 0u;
}

static Compiled compile_for(const Table& t, const cpb_pred* pred) {
    if (!pred) throw ArgError{CPB_ERR_ARG, "nil predicate"};
    Compiled comp;
    compile_pred(pred, [&](const std::string& key) { return t.find(key); }, comp);
    return comp;
}
// the literal terms' columns and the literal pool on the device
static Buf literal_args(Ctx* c, const Table& t, const Compiled& comp, FilterCols& fc) {
    for (int i = 0; i < comp.prog.nterms; i++)
        if (comp.prog.term_col[i] >= 0) { fc.off[i] = t.cols[comp.prog.term_col[i]].off(); fc.data[i] = t.cols[comp.prog.term_col[i]].bytes(); }
    Buf lits = dev_alloc(c, comp.lits.size() + 16);
    if (!comp.lits.empty()) CPB_CUDA(cudaMemcpyAsync(lits->p, comp.lits.data(), comp.lits.size(), cudaMemcpyHostToDevice, c->stream));
    return lits;
}
// flags[i] = 1 when the program of a tree without set terms holds for row i of a non-empty t
static Buf predicate_flags(Ctx* c, const Table& t, const Compiled& comp) {
    const uint64_t n = (uint64_t)t.nrows;
    FilterCols fc{};
    Buf lits = literal_args(c, t, comp, fc);
    Buf flags = dev_alloc(c, n * 4);
    filter_flags_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(fc, comp.prog, lits->as<uint8_t>(), flags->as<uint32_t>(), n);
    CPB_CUDA(cudaGetLastError());
    return flags;
}
// IndexOn(keys) over the literal tuples of a set term; the host copy of the literals is released once they are uploaded
static std::shared_ptr<Index> set_index(Ctx* c, SetTerm& s) {
    auto lt = std::make_shared<Table>(); lt->ctx = c; lt->nrows = (int64_t)s.rows;
    uint64_t bytes = 0;
    for (size_t j = 0; j < s.keys.size(); j++) bytes += s.data[j].size() + s.off[j].size() * 4;
    {
        KernelTimer kt(c, "pred_set_upload", bytes, 0);
        for (size_t j = 0; j < s.keys.size(); j++) {
            Column col; col.name = s.keys[j];
            col.offsets = dev_alloc(c, s.off[j].size() * 4);
            col.data = dev_alloc(c, s.data[j].size() + 16);
            // (pageable sources: the runtime has staged them when the call returns)
            CPB_CUDA(cudaMemcpyAsync(col.offsets->p, s.off[j].data(), s.off[j].size() * 4, cudaMemcpyHostToDevice, c->stream));
            if (!s.data[j].empty()) CPB_CUDA(cudaMemcpyAsync(col.data->p, s.data[j].data(), s.data[j].size(), cudaMemcpyHostToDevice, c->stream));
            lt->cols.push_back(col);
        }
    }
    s.off.clear(); s.off.shrink_to_fit(); s.data.clear(); s.data.shrink_to_fit();
    return build_index(c, lt, s.keys, false);
}
// flags of a program with set terms over a non-empty t: per set term its index (built on first use) probed with t's
// columns, then the literal terms and the program in filter_set
static Buf set_predicate_flags(Ctx* c, const Table& t, Compiled& comp) {
    const uint64_t n = (uint64_t)t.nrows;
    SetHits sh{};
    uint32_t sets = 0;
    std::vector<Buf> hits;
    for (SetTerm& s : comp.sets) {
        if (!s.index) s.index = set_index(c, s);
        hits.push_back(key_flags(c, t, s.cols, *s.index, true));
        sh.hit[s.term] = hits.back()->as<uint32_t>();
        sets |= 1u << s.term;
    }
    FilterCols fc{};
    Buf lits = literal_args(c, t, comp, fc);
    Buf flags = dev_alloc(c, n * 4);
    KernelTimer kt(c, "filter_set", n * (4 + 4 * (uint64_t)comp.sets.size() + 4 * (uint64_t)(comp.prog.nterms - (int)comp.sets.size())));
    filter_set_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(fc, comp.prog, lits->as<uint8_t>(), sh, sets, flags->as<uint32_t>(), n);
    CPB_CUDA(cudaGetLastError());
    return flags;
}

// TakeWhile / DropWhile (csvplus.go:346-374) with a recognisable predicate: the index of the first row for which the
// predicate is FALSE (nrows when there is none) — TakeWhile is then the row range before it, DropWhile the range from it.
__global__ void first_false_kernel(const uint32_t* __restrict__ flags, uint64_t n, unsigned long long* out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && flags[i] == 0) atomicMin(out, (unsigned long long)i);
}
// The predicate is compiled against t's columns first, so a bad one throws whether or not t has rows.
int64_t first_false_row(Ctx* c, const Table& t, const cpb_pred* pred) {
    Compiled comp = compile_for(t, pred);
    const uint64_t n = (uint64_t)t.nrows;
    if (n == 0) return 0;
    Buf out = dev_alloc(c, 8);
    CPB_CUDA(cudaMemsetAsync(out->p, 0xff, 8, c->stream));
    if (comp.sets.empty()) {
        KernelTimer kt(c, "filter_like", n * 12, 2);
        Buf flags = predicate_flags(c, t, comp);
        first_false_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(flags->as<uint32_t>(), n, (unsigned long long*)out->p);
        CPB_CUDA(cudaGetLastError());
    } else {
        Buf flags = set_predicate_flags(c, t, comp);
        KernelTimer kt(c, "first_false", n * 4);
        first_false_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(flags->as<uint32_t>(), n, (unsigned long long*)out->p);
        CPB_CUDA(cudaGetLastError());
    }
    const uint64_t first = read_back<uint64_t>(c, out->p);
    return first == ~0ull ? (int64_t)n : (int64_t)first;
}

// the rows of t for which comp holds; *first (when given) = the position of the first of them in t
static std::shared_ptr<Table> filter_compiled(Ctx* c, const Table& t, Compiled& comp, uint64_t* first = nullptr) {
    const uint64_t n = (uint64_t)t.nrows;
    if (n == 0) { if (first) *first = 0; return gather_rows(c, t, nullptr, 0); }
    Buf flags;
    if (comp.sets.empty()) {
        KernelTimer kt(c, "filter_like", n * 12);
        flags = predicate_flags(c, t, comp);
    } else flags = set_predicate_flags(c, t, comp);
    return rows_where(c, t, flags->as<uint32_t>(), first);
}

std::shared_ptr<Table> filter_table(Ctx* c, const Table& t, const cpb_pred* pred) {
    Compiled comp = compile_for(t, pred);
    return filter_compiled(c, t, comp);
}

void filter_parsed(Ctx* c, Parsed& p, const cpb_pred* pred, std::shared_ptr<Compiled>& comp) {
    const Table& t = *p.table;
    if (t.nrows == 0) return;
    std::vector<std::string> names;
    for (const Column& col : t.cols) names.push_back(col.name);
    if (!comp || comp->columns != names) {
        comp = std::make_shared<Compiled>(compile_for(t, pred));
        comp->columns = std::move(names);
    }
    uint64_t first = 0;
    auto r = filter_compiled(c, t, *comp, &first);
    r->first_line = t.first_line + first;
    r->src_field = t.src_field;
    r->record_fields = t.record_fields;
    p.table = r;
}

// ------------------------------------------------------------------ concat
__global__ void rebase_offsets_kernel(const uint32_t* __restrict__ in, uint32_t* out, uint64_t n, uint32_t add) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n) out[i] = in[i] - in[0] + add;  // also writes the sentinel (overwritten by the next part's first entry: same value)
}

std::shared_ptr<Table> concat_tables(Ctx* c, const std::vector<const Table*>& parts) {
    const Table& first = *parts[0];
    for (auto* p : parts) {
        if (p->cols.size() != first.cols.size()) throw ArgError{CPB_ERR_ARG, "concat: column count mismatch"};
        for (size_t k = 0; k < first.cols.size(); k++) if (p->cols[k].name != first.cols[k].name) throw ArgError{CPB_ERR_ARG, "concat: column name mismatch"};
    }
    int64_t nrows = 0;
    for (auto* p : parts) nrows += p->nrows;
    const size_t K = first.cols.size(), NPARTS = parts.size();
    // byte extents of every (part, column): one D2H round trip
    std::vector<uint32_t> ext(2 * K * NPARTS);
    uint32_t* hp = (uint32_t*)c->pinned_scratch(ext.size() * 4);
    for (size_t p = 0; p < NPARTS; p++)
        for (size_t k = 0; k < K; k++) {
            const uint32_t* off = parts[p]->cols[k].off();
            CPB_CUDA(cudaMemcpyAsync(hp + 2 * (p * K + k), off, 4, cudaMemcpyDeviceToHost, c->stream));
            CPB_CUDA(cudaMemcpyAsync(hp + 2 * (p * K + k) + 1, off + parts[p]->nrows, 4, cudaMemcpyDeviceToHost, c->stream));
        }
    sync_stream(c);
    memcpy(ext.data(), hp, ext.size() * 4);
    auto r = std::make_shared<Table>(); r->ctx = c; r->nrows = nrows; r->first_line = first.first_line;
    for (size_t k = 0; k < K; k++) {
        uint64_t total = 0;
        for (size_t p = 0; p < NPARTS; p++) total += ext[2 * (p * K + k) + 1] - ext[2 * (p * K + k)];
        if (total > 0xffffffffull) throw DataError{CPB_E_TOO_LARGE, (int)k, 0, false, "concatenated column exceeds 4 GiB"};
        Column col; col.name = first.cols[k].name;
        col.offsets = dev_alloc(c, ((size_t)nrows + 1) * 4);
        col.data = dev_alloc(c, total + 16);
        uint64_t row = 0, byte = 0;
        for (size_t p = 0; p < NPARTS; p++) {
            uint32_t b0 = ext[2 * (p * K + k)], b1 = ext[2 * (p * K + k) + 1];
            uint64_t pr = (uint64_t)parts[p]->nrows;
            KernelTimer kt(c, "concat", (uint64_t)(b1 - b0) * 2 + pr * 8);
            rebase_offsets_kernel<<<nblk(pr + 1, 256), 256, 0, c->stream>>>(parts[p]->cols[k].off(), col.offsets->as<uint32_t>() + row, pr, (uint32_t)byte);
            CPB_CUDA(cudaGetLastError());
            if (b1 > b0) CPB_CUDA(cudaMemcpyAsync(col.data->as<uint8_t>() + byte, parts[p]->cols[k].bytes() + b0, b1 - b0, cudaMemcpyDeviceToDevice, c->stream));
            row += pr; byte += b1 - b0;
        }
        r->cols.push_back(col);
    }
    return r;
}

}  // namespace cpb
