// join.cu — K8/K9 of SURVEY §2: the probe side of DataSource.Join / Except and Index.Find.
//
// Replaces (reference): Join csvplus.go:545-569 (per probe row: SelectValues, indexImpl.first =
// sort.Search lower bound :893-897 with cmp :907-920, then a forward scan while equal), mergeRows
// :571-583, Except :588-608 (indexImpl.has :899-905) and indexImpl.find :870-891.
//
// The index keeps its sorted key image (sort.cu).  For a join on the first nk key columns the
// distinct nk-column prefixes ("heads") of the sorted image are inserted into an open-addressing
// hash table that maps a prefix to its run [heads[j], heads[j+1]) of sorted rows — exactly the
// [lower_bound, upper_bound) range the reference finds by binary search, so output order (probe
// order, then index order) is unchanged.  Small tables are staged into shared memory per CTA; large
// ones are probed in L2/HBM.  Probe keys are packed with the index's column widths so equality of
// images is equality of keys.
#include <algorithm>

#include "core.hpp"
#include "rowhash.cuh"
#include "util.cuh"

namespace cpb {

constexpr uint32_t EMPTY = 0xffffffffu;

__global__ void hash_insert_kernel(const uint64_t* __restrict__ image, uint64_t n, uint32_t pbytes, const uint32_t* __restrict__ heads,
                                   uint64_t nheads, uint32_t* slots, uint64_t mask) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nheads) return;
    uint64_t s = hash_prefix(image, n, heads[j], pbytes) & mask;
    for (;;) {
        uint32_t old = atomicCAS(&slots[s], EMPTY, (uint32_t)j);
        if (old == EMPTY) return;
        s = (s + 1) & mask;
    }
}

// total number of matches (= join result rows), one atomic per warp: flags layout [0..1] scan total, [2] not_one,
// [4..5] matches.  With it a join whose probe rows all match exactly once needs no scan of the counts at all.
__device__ __forceinline__ void add_matches(uint32_t* not_one, unsigned long long matches) {
    matches = warp_sum_u64(matches);
    if ((threadIdx.x & 31) == 0 && matches) atomicAdd(reinterpret_cast<unsigned long long*>(not_one + 2), matches);
}
// probe: per probe row the matching run of sorted index rows: lo[i], cnt[i] (cnt 0 = no match)
template <bool SMEM>
__global__ void __launch_bounds__(256) join_probe_kernel(const uint64_t* __restrict__ pimg, uint64_t np, const uint64_t* __restrict__ iimg,
                                                         uint64_t ni, uint32_t pbytes, const uint32_t* __restrict__ slots_g, uint64_t nslots,
                                                         const uint32_t* __restrict__ heads_g, uint64_t nheads, uint32_t* lo, uint32_t* cnt,
                                                         uint32_t* not_one) {
    extern __shared__ uint32_t sh[];
    const uint32_t* slots = slots_g;
    const uint32_t* heads = heads_g;
    if (SMEM) {  // stage the build-side table (slots + heads) into shared memory once per CTA
        for (uint64_t i = threadIdx.x; i < nslots; i += blockDim.x) sh[i] = slots_g[i];
        for (uint64_t i = threadIdx.x; i <= nheads; i += blockDim.x) sh[nslots + i] = heads_g[i];
        __syncthreads();
        slots = sh; heads = sh + nslots;
    }
    const uint64_t mask = nslots - 1;
    unsigned long long matches = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t s = hash_prefix(pimg, np, i, pbytes) & mask;
        uint32_t l = 0, c = 0;
        for (;;) {
            uint32_t j = slots[s];
            if (j == EMPTY) break;
            uint32_t r = heads[j];
            if (prefix_equal(pimg, np, i, iimg, ni, r, pbytes)) { l = r; c = heads[j + 1] - r; break; }
            s = (s + 1) & mask;
        }
        lo[i] = l; cnt[i] = c; matches += c;
        if (__any_sync(__activemask(), c != 1) && c != 1) *not_one = 1u;  // benign race: every writer stores 1
    }
    add_matches(not_one, matches);
}

// ------------------------------------------------------------------ embedded-key table (key prefixes <= 24 bytes)
// One 32-byte slot = one DRAM sector: the whole key prefix (3 image words) + (first sorted row, run length).
// A probe is resolved by the sector it hashes to — no dependent reads of heads[] / the key image — and the probe
// key is packed in registers straight from the probe column (no materialised probe image).
struct __align__(32) Slot32 { unsigned long long k[3]; unsigned long long payload; };  // payload = lo | cnt << 32; 0 = empty

__global__ void hash32_insert_kernel(const uint64_t* __restrict__ image, uint64_t n, uint32_t pbytes, const uint32_t* __restrict__ heads,
                                     uint64_t nheads, Slot32* slots, uint64_t nslots) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nheads) return;
    const uint32_t r = heads[j], full = pbytes >> 3, rem = pbytes & 7;
    unsigned long long w[3] = {0, 0, 0};
    for (uint32_t i = 0; i < full; i++) w[i] = image[(uint64_t)i * n + r];
    if (rem) w[full] = image[(uint64_t)full * n + r] & (~0ull << (8 * (8 - rem)));
    const unsigned long long payload = (unsigned long long)r | ((unsigned long long)(heads[j + 1] - r) << 32);
    uint64_t s = slot_of(hash3(w[0], w[1], w[2]), nslots);
    for (;;) {
        if (atomicCAS(&slots[s].payload, 0ull, payload) == 0ull) { slots[s].k[0] = w[0]; slots[s].k[1] = w[1]; slots[s].k[2] = w[2]; return; }
        if (++s == nslots) s = 0;
    }
}

__global__ void __launch_bounds__(256) join_probe32_kernel(KeyDesc kd, uint64_t np, const Slot32* __restrict__ slots, uint64_t nslots,
                                                           uint32_t* lo, uint32_t* cnt, uint32_t* not_one) {
    unsigned long long matches = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (uint64_t)gridDim.x * blockDim.x) {
        unsigned long long w0, w1, w2;
        pack3(kd, i, w0, w1, w2);
        uint64_t s = slot_of(hash3(w0, w1, w2), nslots);
        uint32_t l = 0, c = 0;
        for (;;) {
            const ulonglong4 sl = *reinterpret_cast<const ulonglong4*>(&slots[s]);  // one 32-byte sector
            if (sl.w == 0ull) break;
            if (sl.x == w0 && sl.y == w1 && sl.z == w2) { l = (uint32_t)sl.w; c = (uint32_t)(sl.w >> 32); break; }
            if (++s == nslots) s = 0;
        }
        lo[i] = l; cnt[i] = c; matches += c;
        if (c != 1) *not_one = 1u;  // benign race: every writer stores 1
    }
    add_matches(not_one, matches);
}

// 16-byte slots for key prefixes <= 12 bytes whose runs all have length 1 (unique keys): four slots per 64-byte
// DRAM granule at load factor 1/2, so a probe costs about one granule (a 32-byte slot at 2/3 costs about two).
struct __align__(16) Slot16 { unsigned long long k0; uint32_t k1; uint32_t row1; };  // row1 = sorted row + 1; 0 = empty
// (claimed by cas128: `dup`, when given, is set if any key is inserted twice.  That is the whole duplicate check of
// UniqueIndexOn for keys <= 12 bytes: the second inserter of a key walks the same probe sequence as the first and
// reaches its slot.)
__global__ void hash16_insert_kernel(const uint64_t* __restrict__ image, uint64_t n, uint32_t pbytes, const uint32_t* __restrict__ heads,
                                     uint64_t nheads, Slot16* slots, uint64_t nslots, uint32_t* dup) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nheads) return;
    const uint32_t r = heads[j], full = pbytes >> 3, rem = pbytes & 7;
    unsigned long long w[2] = {0, 0};
    for (uint32_t i = 0; i < full; i++) w[i] = image[(uint64_t)i * n + r];
    if (rem) w[full] = image[(uint64_t)full * n + r] & (~0ull << (8 * (8 - rem)));
    const unsigned long long lo = w[0], hi = (w[1] >> 32) | ((unsigned long long)(r + 1u) << 32);  // {k0, k1 | row1 << 32}
    uint64_t s = slot_of(hash3(w[0], w[1], 0ull), nslots);
    for (;;) {
        unsigned long long ol, oh;
        cas128(&slots[s], lo, hi, ol, oh);
        if ((ol | oh) == 0ull) return;
        if (dup && ol == lo && (uint32_t)oh == (uint32_t)hi) { *dup = 1u; return; }  // benign race: every writer stores 1
        if (++s == nslots) s = 0;
    }
}
__global__ void __launch_bounds__(256) join_probe16_kernel(KeyDesc kd, uint64_t np, const Slot16* __restrict__ slots, uint64_t nslots,
                                                           uint32_t* lo, uint32_t* cnt, uint32_t* not_one) {
    unsigned long long matches = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (uint64_t)gridDim.x * blockDim.x) {
        unsigned long long w0, w1, w2;
        pack3(kd, i, w0, w1, w2);
        uint64_t s = slot_of(hash3(w0, w1, 0ull), nslots);
        uint32_t l = 0, c = 0;
        for (;;) {
            const uint4 sl = __ldg(reinterpret_cast<const uint4*>(&slots[s]));
            if (sl.w == 0u) break;
            if (sl.x == (uint32_t)w0 && sl.y == (uint32_t)(w0 >> 32) && sl.z == (uint32_t)(w1 >> 32)) { l = sl.w - 1u; c = 1u; break; }
            if (++s == nslots) s = 0;
        }
        lo[i] = l; cnt[i] = c; matches += c;
        if (c != 1) *not_one = 1u;  // benign race: every writer stores 1
    }
    add_matches(not_one, matches);
}

// The order a join on the first nk key columns uses: a lazily sorted unique index joined on its full key is probed
// over the rows as they were given (no sort needed); everything else over the sorted rows.
static RowOrder join_order(const Index& ix, int nk) {
    return ix.unique && ix.derived.uimage && nk == (int)ix.key_cols.size() ? RowOrder::source : RowOrder::sorted;
}
static const Buf& key_image(const Index& ix, RowOrder order) { return order == RowOrder::source ? ix.derived.uimage : ix.image; }

// ordinal slots for nheads runs: a power of two, load factor at most 1/2
static uint64_t ordinal_slots(uint64_t nheads) {
    const uint64_t want = std::max<uint64_t>(16, nheads * 2);
    uint64_t s = 1;
    while (s < want) s <<= 1;
    return s;
}
static ProbeTable::Kind probe_kind(uint64_t nheads, uint32_t pbytes, uint64_t nrows) {
    if ((ordinal_slots(nheads) + nheads + 1) * 4 <= 200 * 1024) return ProbeTable::Kind::smem;
    if (pbytes <= 12 && nheads == nrows) return ProbeTable::Kind::unique16;
    if (pbytes <= 24) return ProbeTable::Kind::run32;
    return ProbeTable::Kind::global;
}

// The probe table over the first nk key columns of the rows in `order` (payload = position in that order).  dup_flag,
// when given, is set by a unique16 insert that meets a key twice.
static ProbeTable& ensure_hash(Ctx* c, Index& ix, RowOrder order, int nk, uint32_t* dup_flag = nullptr) {
    std::lock_guard<std::mutex> lk(ix.mu);
    auto& tables = ix.derived.probe;
    const Buf& image = key_image(ix, order);
    auto it = tables.find({order, nk});
    if (it != tables.end()) { wait_ready(c, it->second.ready); return it->second; }
    ProbeTable ht;
    ht.pbytes = prefix_bytes(ix, nk);
    const uint64_t n = (uint64_t)ix.nrows;
    if (ix.unique && nk == (int)ix.key_cols.size()) {
        // a verified unique index probed on its full key: every row is its own run — no adjacent compare, no scan,
        // no host round trip for the number of distinct keys
        ht.nheads = n;
        ht.heads = dev_alloc_owned(ix.ctx, c, (n + 1) * 4);
        iota_u32(c, ht.heads->as<uint32_t>(), n + 1);
    } else {
        Buf head = dev_alloc(c, (n + 1) * 4);
        {
            KernelTimer kt(c, "hash_heads", (uint64_t)ix.image_words * n * 8 + n * 4);
            head_flags(c, image->as<uint64_t>(), n, ht.pbytes, head->as<uint32_t>());
        }
        const FlagScan s = scan_flags(c, head->as<uint32_t>(), n);  // (its temporaries: this context's pool)
        ht.nheads = s.count;
        // what stays in the index comes from the index owner's pool: the probing context may be shut down first
        ht.heads = dev_alloc_owned(ix.ctx, c, (ht.nheads + 1) * 4);
        compact_flags(c, s, 0, ht.heads->as<uint32_t>());  // heads[nheads] = nrows: the end of the last run
    }
    ht.kind = probe_kind(ht.nheads, ht.pbytes, n);
    const bool ordinal = ht.kind == ProbeTable::Kind::smem || ht.kind == ProbeTable::Kind::global, u16 = ht.kind == ProbeTable::Kind::unique16;
    const size_t slot = ordinal ? 4 : u16 ? sizeof(Slot16) : sizeof(Slot32);
    ht.nslots = ordinal ? ordinal_slots(ht.nheads) : u16 ? ht.nheads * 2 + 16 : ht.nheads + ht.nheads / 2 + 16;
    ht.slots = dev_alloc_owned(ix.ctx, c, ht.nslots * slot);
    CPB_CUDA(cudaMemsetAsync(ht.slots->p, ordinal ? 0xff : 0, ht.nslots * slot, c->stream));  // all slots empty
    {
        KernelTimer kt(c, "hash_build", ht.nheads * (ht.pbytes + 8) + (ordinal ? 0 : ht.nslots * slot));
        const uint64_t* img = image->as<uint64_t>();
        const uint32_t* heads = ht.heads->as<uint32_t>();
        const uint32_t grid = nblk(ht.nheads, 256);
        if (ordinal) hash_insert_kernel<<<grid, 256, 0, c->stream>>>(img, n, ht.pbytes, heads, ht.nheads, ht.slots->as<uint32_t>(), ht.nslots - 1);
        else if (u16) hash16_insert_kernel<<<grid, 256, 0, c->stream>>>(img, n, ht.pbytes, heads, ht.nheads, ht.slots->as<Slot16>(), ht.nslots, dup_flag);
        else hash32_insert_kernel<<<grid, 256, 0, c->stream>>>(img, n, ht.pbytes, heads, ht.nheads, ht.slots->as<Slot32>(), ht.nslots);
        CPB_CUDA(cudaGetLastError());
    }
    ht.ready = record_ready(c);  // another context (stream) that finds it in the map waits for this event, not the host
    return tables.emplace(std::make_pair(order, nk), std::move(ht)).first->second;
}

// per probe row the matching run [lo, lo+cnt) of the index rows in `order`, through the probe table ht over nk columns
static void probe_dispatch(Ctx* c, const Table& probe, const std::vector<int>& pidx, Index& ix, const ProbeTable& ht, RowOrder order, int nk,
                           uint32_t* lo, uint32_t* cnt, uint32_t* not_one) {
    const uint64_t np = (uint64_t)probe.nrows, ni = (uint64_t)ix.nrows;
    std::vector<uint32_t> widths(ix.key_width.begin(), ix.key_width.begin() + nk);
    // the ordinal tables compare a packed probe image with the index's key image; the others pack the probe key in registers
    const bool ordinal = ht.kind == ProbeTable::Kind::smem || ht.kind == ProbeTable::Kind::global;
    uint32_t pwords = (ht.pbytes + 7) / 8;
    KeyDesc kd{};
    const Buf pimg = ordinal ? pack_with_widths(c, probe, pidx, widths, &pwords) : nullptr;
    if (!ordinal) describe_keys(c, probe, pidx, widths, kd);
    const uint64_t* pi = ordinal ? pimg->as<uint64_t>() : nullptr;
    const uint64_t* ii = ordinal ? key_image(ix, order)->as<uint64_t>() : nullptr;
    // algorithmic bytes (SURVEY §8d): probe keys once + build table once (counted as the ordinal table for every kind)
    const uint64_t algo = np * ((uint64_t)pwords * 8 + 8) + ordinal_slots(ht.nheads) * 4 + ht.nheads * ((uint64_t)ht.pbytes + 4);
    const uint32_t grid = (uint32_t)std::min<uint64_t>(nblk(np, 256), (uint64_t)c->sm_count * 16);
    KernelTimer kt(c, "join_probe", algo);
    switch (ht.kind) {
    case ProbeTable::Kind::smem:
        // (per device, and cheap: set on every launch rather than cached per process)
        CPB_CUDA(cudaFuncSetAttribute(join_probe_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        join_probe_kernel<true><<<(uint32_t)std::min<uint64_t>(nblk(np, 256), (uint64_t)c->sm_count), 256, (ht.nslots + ht.nheads + 1) * 4, c->stream>>>(
            pi, np, ii, ni, ht.pbytes, ht.slots->as<uint32_t>(), ht.nslots, ht.heads->as<uint32_t>(), ht.nheads, lo, cnt, not_one);
        break;
    case ProbeTable::Kind::global:
        join_probe_kernel<false><<<grid, 256, 0, c->stream>>>(pi, np, ii, ni, ht.pbytes, ht.slots->as<uint32_t>(), ht.nslots, ht.heads->as<uint32_t>(),
                                                              ht.nheads, lo, cnt, not_one);
        break;
    case ProbeTable::Kind::unique16:
        join_probe16_kernel<<<grid, 256, 0, c->stream>>>(kd, np, ht.slots->as<Slot16>(), ht.nslots, lo, cnt, not_one);
        break;
    case ProbeTable::Kind::run32:
        join_probe32_kernel<<<grid, 256, 0, c->stream>>>(kd, np, ht.slots->as<Slot32>(), ht.nslots, lo, cnt, not_one);
        break;
    }
    CPB_CUDA(cudaGetLastError());
}

// An index whose rows are not in key order: per probe row what the reference computes, on any order of rows.
// first = sort.Search(n, row >= v) (indexImpl.first, csvplus.go:893-897), then Join takes every row from there while
// row <= v (:557); Except keeps the probe row when that run is empty (has, :899-905: the row at first equals v).
__global__ void __launch_bounds__(256) join_search_kernel(const uint64_t* __restrict__ pimg, uint64_t np, const uint64_t* __restrict__ iimg,
                                                          uint64_t ni, uint32_t pbytes, uint32_t* lo, uint32_t* cnt, uint32_t* not_one) {
    unsigned long long matches = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t a = 0, b = ni;
        while (a < b) { const uint64_t h = a + (b - a) / 2; if (prefix_cmp(iimg, ni, h, pimg, np, i, pbytes) < 0) a = h + 1; else b = h; }
        uint64_t e = a;
        while (e < ni && prefix_cmp(iimg, ni, e, pimg, np, i, pbytes) <= 0) e++;
        const uint32_t c = (uint32_t)(e - a);
        lo[i] = (uint32_t)a; cnt[i] = c; matches += c;
        if (c != 1) *not_one = 1u;  // benign race: every writer stores 1
    }
    add_matches(not_one, matches);
}
static void search_probe(Ctx* c, const Table& probe, const std::vector<int>& pidx, Index& ix, int nk, uint32_t* lo, uint32_t* cnt,
                         uint32_t* not_one) {
    const uint64_t np = (uint64_t)probe.nrows, ni = (uint64_t)ix.nrows;
    std::vector<uint32_t> widths(ix.key_width.begin(), ix.key_width.begin() + nk);
    uint32_t pwords = 0;
    Buf pimg = pack_with_widths(c, probe, pidx, widths, &pwords);
    KernelTimer kt(c, "join_search", np * ((uint64_t)pwords * 8 + 8));
    const uint32_t grid = (uint32_t)std::min<uint64_t>(nblk(np, 256), (uint64_t)c->sm_count * 16);
    join_search_kernel<<<grid, 256, 0, c->stream>>>(pimg->as<uint64_t>(), np, ix.image->as<uint64_t>(), ni, prefix_bytes(ix, nk), lo, cnt, not_one);
    CPB_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------ row-carrying hash table (Index::derived.rowhash)
// Built region by region in two passes, so that no insert is a random read-modify-write of DRAM:
//  1. rowhash_scatter, one thread per source row: the key packed straight from the key columns, the payload columns'
//     lengths and bytes gathered in registers, and the row's slot image {k0, k1, hdr, payload} appended to its region's
//     part of the table itself (fill[g] counts region g's rows).  A region's appends are consecutive sectors, so the
//     writes of a warp's rows merge in L2 and reach DRAM as whole sectors.
//  2. rowhash_region, one CTA per region: the region's staged images read, inserted into the region built in shared
//     memory with one 128-bit CAS per claim, and the whole region, empty slots included, written back over them.  So
//     the table needs no zeroing.  A key that meets itself sets flags[0]: that is the whole duplicate check of
//     UniqueIndexOn for such an index (equal keys hash to one region).  A region given more than region - 1 rows is
//     not built and sets flags[1] (its images past `region` were dropped by the scatter).
struct PayCols { int nc; const uint32_t* off[RH_MAXC]; const uint8_t* data[RH_MAXC]; };
__global__ void __launch_bounds__(256) rowhash_scatter_kernel(KeyDesc kd, PayCols pc, uint64_t n, RowSlot* slots, uint64_t nslots,
                                                              uint32_t rshift, uint32_t* fill) {
    const uint64_t r0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r0 - (threadIdx.x & 31u) >= n) return;  // whole warps only: pairs of lanes exchange their images below
    const uint64_t r = r0 < n ? r0 : n - 1;     // (a row past n is read, not stored)
    unsigned long long w0, w1, w2;
    pack3(kd, r, w0, w1, w2);
    unsigned long long pa = 0, pb = 0;
    uint32_t hdr = RH_OCCUPIED, pos = 0;
#pragma unroll
    for (int j = 0; j < RH_MAXC; j++) {
        if (j >= pc.nc) break;
        const uint32_t s = pc.off[j][r], l = pc.off[j][r + 1] - s;
        unsigned long long a, b;
        load16(pc.data[j] + s, l, a, b);
        or_at16(pa, pb, pos, a, b);
        hdr |= l << (5 * j);
        pos += l;
    }
#ifdef RH_DIAG_NO_PAYLOAD  // diagnostic (tools/prof_rowhash.py): the key alone
    pa = pb = 0; hdr = RH_OCCUPIED;
#endif
    const uint64_t g = slot_of(hash3(w0, w1, 0ull), nslots) >> rshift;
#ifdef RH_DIAG_NO_ATOMIC  // diagnostic: the position from the row number, the fill counts untouched
    const uint32_t p = (uint32_t)r & ((1u << rshift) - 1u);
#else
    const uint32_t p = r0 < n ? atomicAdd(&fill[g], 1u) : ~0u;
#endif
    bool ok = r0 < n && !(p >> rshift);  // a region given more than it holds: rowhash_region reports it
#ifdef RH_DIAG_NO_STORE  // diagnostic: no image store (kept live by a store no row makes)
    ok = ok && ((pa ^ pb ^ w0) + hdr) == 0x9E3779B97F4A7C15ull;
#endif
    // A row's image is one 32-byte sector.  Written as two 16-byte halves by one lane, each store instruction of a warp
    // sends 32 half sectors to L2; instead lanes 2i and 2i + 1 write lane 2i's image in the first store and lane
    // 2i + 1's in the second, so each store is 16 whole sectors (one shuffle of the half each lane lacks).  Evict-last:
    // a region's frontier line stays in L2 until its later images fill it.
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    uint4* d = reinterpret_cast<uint4*>(&slots[(g << rshift) + p]);
    const uint4 h4 = make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)(w1 >> 32), hdr);
    const uint4 p4 = make_uint4((uint32_t)pa, (uint32_t)(pa >> 32), (uint32_t)pb, (uint32_t)(pb >> 32));
    const bool odd = threadIdx.x & 1u;
    uint4 x = odd ? h4 : p4;  // what the other lane of the pair stores: the odd lane's header, the even lane's payload
    x.x = __shfl_xor_sync(~0u, x.x, 1); x.y = __shfl_xor_sync(~0u, x.y, 1); x.z = __shfl_xor_sync(~0u, x.z, 1); x.w = __shfl_xor_sync(~0u, x.w, 1);
    uint4* dp = reinterpret_cast<uint4*>(__shfl_xor_sync(~0u, reinterpret_cast<unsigned long long>(d), 1));
    const bool okp = __shfl_xor_sync(~0u, ok ? 1u : 0u, 1) != 0u;
    uint4* d1 = odd ? dp + 1 : d; const uint4 v1 = odd ? x : h4; const bool ok1 = odd ? okp : ok;  // the even lane's row
    uint4* d2 = odd ? d + 1 : dp; const uint4 v2 = odd ? p4 : x; const bool ok2 = odd ? ok : okp;  // the odd lane's row
    if (ok1) asm volatile("st.global.L2::cache_hint.v4.u32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(d1), "r"(v1.x), "r"(v1.y), "r"(v1.z), "r"(v1.w), "l"(pol) : "memory");
    if (ok2) asm volatile("st.global.L2::cache_hint.v4.u32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(d2), "r"(v2.x), "r"(v2.y), "r"(v2.z), "r"(v2.w), "l"(pol) : "memory");
}
constexpr int RH_THREADS = 256, RH_UNROLL = 2;  // staged images in flight per thread
__global__ void __launch_bounds__(RH_THREADS) rowhash_region_kernel(RowSlot* slots, uint64_t nslots, uint64_t nregions, uint32_t rshift,
                                                                    const uint32_t* __restrict__ fill, uint32_t* flags) {
    extern __shared__ uint4 sm[];  // the region: 2 x uint4 per slot
    const uint32_t rs = 1u << rshift, rmask = rs - 1;
    for (uint64_t g = blockIdx.x; g < nregions; g += gridDim.x) {
        const uint32_t cnt = fill[g];
        if (cnt >= rs) {  // at most rs - 1 keys: a probe for a missing key must meet an empty slot
            if (threadIdx.x == 0) flags[1] = 1u;
            continue;
        }
        for (uint32_t i = threadIdx.x; i < 2 * rs; i += RH_THREADS) sm[i] = make_uint4(0, 0, 0, 0);
        __syncthreads();
        uint4* reg = reinterpret_cast<uint4*>(slots + (g << rshift));
        for (uint32_t i0 = 0; i0 < cnt; i0 += RH_THREADS * RH_UNROLL) {
            uint4 hd[RH_UNROLL], pay[RH_UNROLL];
#pragma unroll
            for (int u = 0; u < RH_UNROLL; u++) {
                const uint32_t i = i0 + u * RH_THREADS + threadIdx.x;
                if (i < cnt) { hd[u] = __ldcs(reg + 2 * i); pay[u] = __ldcs(reg + 2 * i + 1); }
            }
#pragma unroll
            for (int u = 0; u < RH_UNROLL; u++) {
                if (i0 + u * RH_THREADS + threadIdx.x >= cnt) break;
                const unsigned long long lo = ((unsigned long long)hd[u].y << 32) | hd[u].x, hi = ((unsigned long long)hd[u].w << 32) | hd[u].z;
                uint32_t s = (uint32_t)slot_of(hash3(lo, (unsigned long long)hd[u].z << 32, 0ull), nslots) & rmask;
                for (;;) {
                    unsigned long long ol, oh;
                    cas128_shared(&sm[2 * s], lo, hi, ol, oh);
                    if ((ol | oh) == 0ull) { sm[2 * s + 1] = pay[u]; break; }
                    if (ol == lo && (uint32_t)oh == (uint32_t)hi) { flags[0] = 1u; break; }  // benign race: every writer stores 1
                    s = (s + 1) & rmask;
                }
            }
        }
        __syncthreads();  // every staged image is read: the region is written over them
        for (uint32_t i = threadIdx.x; i < 2 * rs; i += RH_THREADS) __stcs(reg + i, sm[i]);
        __syncthreads();
    }
}
RhBuild rowhash_build(Ctx* c, Index& ix) {
    RowHash& rh = ix.derived.rowhash;
    const uint64_t n = (uint64_t)ix.nrows;
    const Table& t = *ix.src;
    KeyDesc kd{};
    describe_keys(c, t, ix.key_col_idx, ix.key_width, kd);
    PayCols pc{};
    pc.nc = (int)rh.cols.size();
    for (int j = 0; j < pc.nc; j++) { pc.off[j] = t.cols[rh.cols[j]].off(); pc.data[j] = t.cols[rh.cols[j]].bytes(); }
    // at least 2n + 16 slots (load factor about 1/2) in whole regions; a table smaller than RH_REGION is one region
    const uint64_t want = n * 2 + 16;
    uint32_t rshift = 0;
    while ((1ull << rshift) < want && (1u << rshift) < RH_REGION) rshift++;
    rh.region = 1u << rshift;
    const uint64_t nregions = (want + rh.region - 1) >> rshift;
    rh.nslots = nregions << rshift;
    rh.slots = dev_alloc(c, rh.nslots * sizeof(RowSlot));
    Buf fill = dev_alloc(c, nregions * 4), flags = dev_alloc(c, 8);
    CPB_CUDA(cudaMemsetAsync(fill->p, 0, nregions * 4, c->stream));
    CPB_CUDA(cudaMemsetAsync(flags->p, 0, 8, c->stream));
    {
        KernelTimer kt(c, "rowhash_scatter", n * ((uint64_t)kd.words * 8 + RH_PAY + 4 * (uint64_t)(kd.nkeys + pc.nc) + sizeof(RowSlot)));
        rowhash_scatter_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(kd, pc, n, rh.slots->as<RowSlot>(), rh.nslots, rshift, fill->as<uint32_t>());
        CPB_CUDA(cudaGetLastError());
    }
    {
        KernelTimer kt(c, "rowhash_build", n * sizeof(RowSlot) + rh.nslots * sizeof(RowSlot));
        const size_t smem = (size_t)rh.region * sizeof(RowSlot);
        // (per device, and cheap: set on every launch rather than cached per process)
        CPB_CUDA(cudaFuncSetAttribute(rowhash_region_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int per_sm = 0;
        CPB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rowhash_region_kernel, RH_THREADS, smem));
        const uint32_t grid = (uint32_t)std::min<uint64_t>(nregions, (uint64_t)c->sm_count * std::max(per_sm, 1));
        rowhash_region_kernel<<<grid, RH_THREADS, smem, c->stream>>>(rh.slots->as<RowSlot>(), rh.nslots, nregions, rshift, fill->as<uint32_t>(),
                                                                     flags->as<uint32_t>());
        CPB_CUDA(cudaGetLastError());
    }
    const uint64_t f = read_back<uint64_t>(c, flags->p);
    return (uint32_t)f ? RhBuild::duplicate : (f >> 32) ? RhBuild::overflow : RhBuild::built;
}
// flag[i] = whether probe row i finds its key (want 1) / finds nothing (want 0): the slot headers only
__global__ void __launch_bounds__(256) rowhash_flags_kernel(KeyDesc kd, uint64_t np, const RowSlot* __restrict__ slots, uint64_t nslots,
                                                            uint64_t rmask, uint32_t want, uint32_t* flag) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (uint64_t)gridDim.x * blockDim.x) {
        unsigned long long k0; uint32_t k1;
        uint64_t s = rh_start(kd, i, nslots, k0, k1);
        uint4 h = rh_header(slots, s);
        flag[i] = rh_walk(slots, rmask, k0, k1, s, h) == (want != 0) ? 1u : 0u;
    }
}
static Buf rowhash_flags(Ctx* c, const Table& probe, const std::vector<int>& pidx, const Index& ix, bool want) {
    const uint64_t np = (uint64_t)probe.nrows;
    KeyDesc kd{};
    describe_keys(c, probe, pidx, ix.key_width, kd);
    Buf flag = dev_alloc(c, np * 4);
    KernelTimer kt(c, "rowhash_flags", np * ((uint64_t)kd.words * 8 + 4 * (uint64_t)kd.nkeys + 16 + 4));
    const uint32_t grid = (uint32_t)std::min<uint64_t>(nblk(np, 256), (uint64_t)c->sm_count * 16);
    const RowHash& rh = ix.derived.rowhash;
    rowhash_flags_kernel<<<grid, 256, 0, c->stream>>>(kd, np, rh.slots->as<RowSlot>(), rh.nslots, rh.region - 1ull, want ? 1u : 0u, flag->as<uint32_t>());
    CPB_CUDA(cudaGetLastError());
    return flag;
}

// per probe row the run of index rows matching its key on the first nk key columns: lo / cnt (cnt 0: none), and in
// flags (32 bytes, zeroed here) the scan total slot [0..1], not_one [2] and the match count [4..5]
static RowOrder probe_runs(Ctx* c, const Table& probe, const std::vector<int>& pidx, Index& ix, uint32_t* lo, uint32_t* cnt, const Buf& flags) {
    const uint64_t np = (uint64_t)probe.nrows, ni = (uint64_t)ix.nrows;
    const int nk = (int)pidx.size();
    CPB_CUDA(cudaMemsetAsync(flags->p, 0, 32, c->stream));
    uint32_t* not_one = flags->as<uint32_t>() + 2;  // [0..1] = scan total
    const RowOrder order = join_order(ix, nk);
    if (ni != 0 && order == RowOrder::sorted) ensure_sorted(c, ix);
    if (ni == 0) {
        CPB_CUDA(cudaMemsetAsync(cnt, 0, (np + 1) * 4, c->stream));
    } else if (!ix.in_order) {
        search_probe(c, probe, pidx, ix, nk, lo, cnt, not_one);
    } else {
        const ProbeTable& ht = ensure_hash(c, ix, order, nk);
        probe_dispatch(c, probe, pidx, ix, ht, order, nk, lo, cnt, not_one);
    }
    return order;
}

Buf key_flags(Ctx* c, const Table& probe, const std::vector<int>& pidx, Index& ix, bool hit) {
    const uint64_t np = (uint64_t)probe.nrows;
    if (np == 0) return dev_alloc(c, 4);
    if (ix.derived.rowhash.slots && pidx.size() == ix.key_cols.size()) return rowhash_flags(c, probe, pidx, ix, hit);
    Buf lo = dev_alloc(c, np * 4), cnt = dev_alloc(c, (np + 1) * 4), flags = dev_alloc(c, 32);
    probe_runs(c, probe, pidx, ix, lo->as<uint32_t>(), cnt->as<uint32_t>(), flags);
    Buf flag = dev_alloc(c, np * 4);
    nonzero_flags(c, cnt->as<uint32_t>(), np, hit, flag->as<uint32_t>());
    return flag;
}

// LeftJoin (mode left) keeps Join's path up to the point where Join drops the probe rows that found nothing; there it keeps
// them, with every index-only column empty:
//  * row-carrying table: rowhash_gather's full-length columns are already empty on a miss, so nothing is compacted; the
//    index key columns Join takes from the probe are gathered from it again with the miss rows' ids NO_ROW;
//  * run routes: every probe row gives max(cnt, 1) pairs (one more host synchronisation: their total), a miss one pair
//    whose index id is NO_ROW, and the index side (key columns included) is gathered with empty values for it.
// Every probe row matching exactly once returns Join's result on Join's kernels; no match at all (an empty index
// included) returns the probe's columns shared and each index-only column as zeroed offsets, with no gather.
std::shared_ptr<Table> join_tables(Ctx* c, const Table& probe, Index& ix, const std::vector<std::string>& cols, JoinMode mode) {
    const bool anti = mode == JoinMode::anti, left = mode == JoinMode::left;
    const uint64_t np = (uint64_t)probe.nrows, ni = (uint64_t)ix.nrows;
    const int nk = (int)cols.size();
    std::vector<int> pidx;
    for (int k = 0; k < nk; k++) {
        int ci = probe.find(cols[k]);
        if (ci < 0 && np > 0)  // row.SelectValues(columns...) fails on the first probe row (csvplus.go:556, :145)
            throw DataError{CPB_E_MISSING_COLUMN, k, probe.first_line, true, "missing column " + go_quote(cols[k])};
        pidx.push_back(ci);
    }
    // output schema: mergeRows(indexRow, probeRow) — probe wins name collisions (csvplus.go:571-583)
    std::vector<const Column*> icols, pcols;
    // An index column that is one of the nk joined key columns is not gathered: a match means equal key images, and
    // equal images mean equal bytes (value zero-padded to the index's width, then its length), so the index value IS
    // the probe value.  icol_key[j] = k takes output column j from probe key column pidx[k]; -1 gathers it from the
    // index (gather_idx: those index columns, in order).  Rows out of key order are searched as the reference does
    // (join_search_kernel): a run there can hold rows whose keys are below the probe's, so every index column is gathered.
    // (all_idx: every index-only column, key columns included, in order)
    std::vector<int> icol_key, gather_idx, all_idx;
    const Table& ischema = ix.schema();  // names only: the sorted columns may not be materialised
    if (!anti) for (size_t q = 0; q < ischema.cols.size(); q++) {
        if (probe.find(ischema.cols[q].name) >= 0) continue;
        int key = -1;
        for (int k = 0; k < nk && key < 0 && ix.in_order; k++) if (ix.key_col_idx[k] == (int)q) key = k;
        icols.push_back(&ischema.cols[q]);
        icol_key.push_back(key);
        if (key < 0) gather_idx.push_back((int)q);
        all_idx.push_back((int)q);
    }
    for (auto& col : probe.cols) pcols.push_back(&col);

    auto out = std::make_shared<Table>(); out->ctx = c; out->first_line = probe.first_line;
    // appends the index-side output columns: the gathered ones in order from `gi`, the key columns as keycol(k)
    auto put_index_cols = [&](const Table& gi, auto keycol) {
        size_t g = 0;
        for (size_t j = 0; j < icols.size(); j++) {
            Column col = icol_key[j] >= 0 ? keycol(icol_key[j]) : gi.cols[g++];
            col.name = icols[j]->name;
            out->cols.push_back(col);
        }
    };
    auto empty_result = [&]() {
        Table e; e.ctx = c; e.nrows = 0;
        for (auto* p : icols) e.cols.push_back(*p);
        for (auto* p : pcols) e.cols.push_back(*p);
        return gather_rows(c, e, nullptr, 0);
    };
    if (np == 0) return empty_result();
    // the probe rows whose flag is set (Except's result)
    auto flagged_rows = [&](const Table& t, const FlagScan& s) {
        Buf ids = dev_alloc(c, (s.count + 1) * 4);
        compact_flags(c, s, 0, ids->as<uint32_t>());
        auto r = gather_rows(c, t, ids->as<uint32_t>(), (int64_t)s.count);
        r->first_line = probe.first_line;
        return r;
    };
    if (anti) {
        Buf miss = key_flags(c, probe, pidx, ix, false);
        return flagged_rows(probe, scan_flags(c, miss->as<uint32_t>(), np));
    }
    // LeftJoin where no probe row matches: the probe's columns shared, each index-only column np empty values
    auto all_missed = [&]() {
        Buf zero = dev_alloc(c, (np + 1) * 4), none = dev_alloc(c, 16);
        CPB_CUDA(cudaMemsetAsync(zero->p, 0, (np + 1) * 4, c->stream));
        out->nrows = (int64_t)np;
        for (auto* p : icols) out->cols.push_back(Column{p->name, zero, none, 0});
        for (auto* p : pcols) out->cols.push_back(*p);
        return out;
    };
    if (ix.derived.rowhash.slots && nk == (int)ix.key_cols.size()) {
        // a unique index with a row-carrying table joined on its full key: one random access per probe row
        Buf hit;
        FlagScan hits{};  // hits.pos stays null until the hit rows are needed
        std::shared_ptr<Table> gi;
        uint64_t m = 0;
        if (gather_idx.empty()) {  // no index column to fetch: only the matches
            hit = rowhash_flags(c, probe, pidx, ix, true);
            hits = scan_flags(c, hit->as<uint32_t>(), np);
            m = hits.count;
            gi = std::make_shared<Table>(); gi->ctx = c; gi->nrows = (int64_t)np;
        } else {
            gi = rowhash_gather(c, ix, probe, pidx, gather_idx, &m);
        }
        if (m == 0) return left ? all_missed() : empty_result();
        out->nrows = (int64_t)np;
        put_index_cols(*gi, [&](int k) { return probe.cols[pidx[k]]; });
        for (auto* p : pcols) out->cols.push_back(*p);
        if (m == np) return out;  // every probe row matched: the probe columns are shared as they are
        if (left) {
            // the full-length result is LeftJoin's once the key columns taken from the probe are empty on the miss rows
            std::vector<size_t> keyed;
            Table kt; kt.ctx = c; kt.nrows = (int64_t)np;
            for (size_t j = 0; j < icols.size(); j++)
                if (icol_key[j] >= 0) { keyed.push_back(j); kt.cols.push_back(probe.cols[pidx[icol_key[j]]]); }
            if (keyed.empty()) return out;
            if (!hit) hit = rowhash_flags(c, probe, pidx, ix, true);
            Buf ids = dev_alloc(c, np * 4);
            {
                KernelTimer kt_ids(c, "left_ids", np * 8);
                const uint32_t* h = hit->as<uint32_t>();
                uint32_t* id = ids->as<uint32_t>();
                each_row(c, np, [=] __device__(uint64_t i) { id[i] = h[i] ? (uint32_t)i : NO_ROW; });
            }
            auto g = gather_rows(c, kt, ids->as<uint32_t>(), (int64_t)np, true);
            for (size_t x = 0; x < keyed.size(); x++) { Column col = g->cols[x]; col.name = icols[keyed[x]]->name; out->cols[keyed[x]] = col; }
            return out;
        }
        // probe rows that found nothing: the full-length result (empty index values there) compacted to the rows that did
        if (!hits.pos) {
            hit = rowhash_flags(c, probe, pidx, ix, true);
            hits = scan_flags(c, hit->as<uint32_t>(), np);
        }
        return flagged_rows(*out, hits);
    }
    Buf lo = dev_alloc(c, np * 4), cnt = dev_alloc(c, (np + 1) * 4), flags = dev_alloc(c, 32);
    const RowOrder order = probe_runs(c, probe, pidx, ix, lo->as<uint32_t>(), cnt->as<uint32_t>(), flags);
    const std::vector<uint32_t> hf = read_back<uint32_t>(c, flags->p, 8);
    const uint64_t m = (uint64_t)hf[4] | ((uint64_t)hf[5] << 32);  // counted by the probe kernel (0 when ni == 0)
    // every probe row matched exactly one index row (the usual foreign-key join): the probe-side columns of the
    // result ARE the probe columns, in order — share their buffers instead of copying them; no scan of the counts
    const bool probe_identity = ni != 0 && hf[2] == 0 && m == np;
    if (m > 0xfffffffeull) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "join result exceeds 2^32-2 rows; probe in smaller batches"};
    if (m == 0) return left ? all_missed() : empty_result();
    if (probe_identity) {
        auto gi = gather_index_rows(c, ix, gather_idx, lo->as<uint32_t>(), (int64_t)m, order);  // lo[i] is the single matching index row
        out->nrows = (int64_t)m;
        put_index_cols(*gi, [&](int k) { return probe.cols[pidx[k]]; });
        for (auto* p : pcols) out->cols.push_back(*p);
        return out;
    }
    Buf pos = dev_alloc(c, (np + 1) * 4);
    Table pt; pt.ctx = c; pt.nrows = (int64_t)np;
    for (auto* p : pcols) pt.cols.push_back(*p);
    if (left) {
        // max(cnt[i], 1) pairs per probe row, a miss as one pair (i, NO_ROW); the pair count is read back
        {
            KernelTimer kt(c, "left_counts", np * 8);
            const uint32_t* run_cnt = cnt->as<uint32_t>();
            uint32_t* at = pos->as<uint32_t>();
            each_row(c, np, [=] __device__(uint64_t i) { at[i] = run_cnt[i] ? run_cnt[i] : 1u; });
        }
        exclusive_scan_u32(c, pos->as<uint32_t>(), pos->as<uint32_t>(), np, flags->as<uint64_t>());
        const uint64_t ml = read_back<uint64_t>(c, flags->p);
        if (ml > 0xfffffffeull) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "join result exceeds 2^32-2 rows; probe in smaller batches"};
        Buf pid = dev_alloc(c, ml * 4), iid = dev_alloc(c, ml * 4);
        {
            KernelTimer kt(c, "join_pairs", np * 12 + ml * 8);
            const uint32_t *run_lo = lo->as<uint32_t>(), *run_cnt = cnt->as<uint32_t>(), *at = pos->as<uint32_t>();
            uint32_t *probe_id = pid->as<uint32_t>(), *index_id = iid->as<uint32_t>();
            each_row(c, np, [=] __device__(uint64_t i) {
                const uint32_t k = run_cnt[i], p = at[i], l = run_lo[i];
                if (k == 0) { probe_id[p] = (uint32_t)i; index_id[p] = NO_ROW; }
                for (uint32_t j = 0; j < k; j++) { probe_id[p + j] = (uint32_t)i; index_id[p + j] = l + j; }
            });
        }
        // every index-only column from the index: a key column taken from the probe would be a value on a miss row
        auto gi = gather_index_rows(c, ix, all_idx, iid->as<uint32_t>(), (int64_t)ml, order, true);
        auto gp = gather_rows(c, pt, pid->as<uint32_t>(), (int64_t)ml);
        out->nrows = (int64_t)ml;
        for (size_t j = 0; j < icols.size(); j++) { Column col = gi->cols[j]; col.name = icols[j]->name; out->cols.push_back(col); }
        for (auto& col : gp->cols) out->cols.push_back(col);
        return out;
    }
    exclusive_scan_u32(c, cnt->as<uint32_t>(), pos->as<uint32_t>(), np, flags->as<uint64_t>());
    Buf pid = dev_alloc(c, m * 4), iid = dev_alloc(c, m * 4);
    {
        // probe row i's run of index rows [lo[i], lo[i] + cnt[i]) as the pairs pos[i] onwards
        KernelTimer kt(c, "join_pairs", np * 12 + m * 8);
        const uint32_t *run_lo = lo->as<uint32_t>(), *run_cnt = cnt->as<uint32_t>(), *at = pos->as<uint32_t>();
        uint32_t *probe_id = pid->as<uint32_t>(), *index_id = iid->as<uint32_t>();
        each_row(c, np, [=] __device__(uint64_t i) {
            const uint32_t k = run_cnt[i], p = at[i], l = run_lo[i];
            for (uint32_t j = 0; j < k; j++) { probe_id[p + j] = (uint32_t)i; index_id[p + j] = l + j; }
        });
    }
    auto gi = gather_index_rows(c, ix, gather_idx, iid->as<uint32_t>(), (int64_t)m, order);
    auto gp = gather_rows(c, pt, pid->as<uint32_t>(), (int64_t)m);
    out->nrows = (int64_t)m;
    put_index_cols(*gi, [&](int k) { return gp->cols[pidx[k]]; });
    for (auto& col : gp->cols) out->cols.push_back(col);
    return out;
}

// ------------------------------------------------------------------ UniqueIndexOn without sorting
// Every row probes the full-key table built over the rows themselves: with unique keys row r finds r.  Two rows with
// the same key occupy two slots of one probe sequence, so at least one of them finds the other: a duplicate exists
// iff some row does not find itself.
bool index_has_duplicates(Ctx* c, Index& ix) {
    const uint64_t n = (uint64_t)ix.nrows;
    const int nk = (int)ix.key_cols.size();
    Buf flags = dev_alloc(c, 64);
    CPB_CUDA(cudaMemsetAsync(flags->p, 0, 64, c->stream));
    const ProbeTable& ht = ensure_hash(c, ix, RowOrder::source, nk, flags->as<uint32_t>() + 8);
    if (ht.kind == ProbeTable::Kind::unique16)  // the insert saw every key it met twice: no self probe needed
        return read_back<uint32_t>(c, flags->as<uint32_t>() + 8) != 0;
    Buf lo = dev_alloc(c, n * 4), cnt = dev_alloc(c, (n + 1) * 4);
    probe_dispatch(c, *ix.src, ix.key_col_idx, ix, ht, RowOrder::source, nk, lo->as<uint32_t>(), cnt->as<uint32_t>(), flags->as<uint32_t>() + 2);
    {
        KernelTimer kt(c, "unique_check", n * 8);
        const uint32_t *run_lo = lo->as<uint32_t>(), *run_cnt = cnt->as<uint32_t>();
        uint32_t* dup = flags->as<uint32_t>() + 8;
        each_row(c, n, [=] __device__(uint64_t i) {
            if (run_cnt[i] != 1u || run_lo[i] != (uint32_t)i) *dup = 1u;  // benign race: every writer stores 1
        });
    }
    return read_back<uint32_t>(c, flags->as<uint32_t>() + 8) != 0;
}

// ------------------------------------------------------------------ Index.Find: [lower, upper) of a key prefix
// val: the key image of one row (the lookup values)
__global__ void find_range_kernel(const uint64_t* __restrict__ image, uint64_t n, const uint64_t* __restrict__ val, uint32_t pbytes,
                                  unsigned long long* out) {
    // in the reference's order (:882-888), which decides the result when the rows are not in key order (in_order):
    uint64_t i = 0, j = n;  // upper = sort.Search(n, row > val)
    while (i < j) { uint64_t h = i + (j - i) / 2; if (prefix_cmp(image, n, h, val, 1, 0, pbytes) <= 0) i = h + 1; else j = h; }
    out[1] = i;
    j = i; i = 0;           // lower = sort.Search(upper, row >= val)
    while (i < j) { uint64_t h = i + (j - i) / 2; if (prefix_cmp(image, n, h, val, 1, 0, pbytes) < 0) i = h + 1; else j = h; }
    out[0] = i;
}

void find_range(Ctx* c, Index& ix, const std::vector<std::string>& values, int64_t* lo, int64_t* hi) {
    const uint64_t n = (uint64_t)ix.nrows;
    *lo = 0; *hi = 0;
    if (n == 0) return;
    ensure_sorted(c, ix);
    // the lookup values as a one-row table: value k is column k, a view at row k of one offsets / bytes pair
    std::vector<uint32_t> off(1, 0);
    std::string bytes;
    std::vector<int> kidx;
    for (const std::string& v : values) { bytes += v; off.push_back((uint32_t)bytes.size()); kidx.push_back((int)kidx.size()); }
    Buf doff = dev_alloc(c, off.size() * 4), dbytes = dev_alloc(c, bytes.size()), out = dev_alloc(c, 16);
    CPB_CUDA(cudaMemcpyAsync(doff->p, off.data(), off.size() * 4, cudaMemcpyHostToDevice, c->stream));
    if (!bytes.empty()) CPB_CUDA(cudaMemcpyAsync(dbytes->p, bytes.data(), bytes.size(), cudaMemcpyHostToDevice, c->stream));
    Table t; t.ctx = c; t.nrows = 1;
    for (int k : kidx) t.cols.push_back(Column{"", doff, dbytes, k});
    uint32_t words = 0;
    const Buf val = pack_with_widths(c, t, kidx, std::vector<uint32_t>(ix.key_width.begin(), ix.key_width.begin() + kidx.size()), &words);
    {
        KernelTimer kt(c, "index_find", 0);
        find_range_kernel<<<1, 1, 0, c->stream>>>(ix.image->as<uint64_t>(), n, val->as<uint64_t>(), prefix_bytes(ix, (int)kidx.size()),
                                                  (unsigned long long*)out->p);
        CPB_CUDA(cudaGetLastError());
    }
    const std::vector<uint64_t> h = read_back<uint64_t>(c, out->p, 2);
    *lo = (int64_t)h[0]; *hi = (int64_t)h[1];
}

}  // namespace cpb
