// sort.cu — K5/K6/K7 of SURVEY §2: IndexOn / UniqueIndexOn / ResolveDuplicates.
//
// Replaces (reference): createIndex csvplus.go:707-738 (sort.Sort with indexImpl.Less :794-807),
// createUniqueIndex :740-756 (adjacent equalRows scan), indexImpl.dedup :810-867.
//
// Order = per key column bytewise strings.Compare, columns left to right.  Each row's key is
// packed into an order-preserving fixed-width big-endian image (per column: value zero-padded to
// the column's longest value, then the value length), so comparing images as unsigned integers is
// exactly the reference's comparator (DESIGN.md §index).  The image is sorted with a stable LSD
// radix sort, one 64-bit image word at a time, 8-bit digits, skipping digits that are constant
// over the whole column.  Ties keep input order (the reference's pdqsort is unstable: SURVEY §Q2).
#include <algorithm>

#include "core.hpp"
#include "rowhash.cuh"
#include "util.cuh"

namespace cpb {

// ------------------------------------------------------------------ key widths
__global__ void max_len_kernel(const uint32_t* __restrict__ off, uint64_t n, uint32_t* out) {
    uint32_t m = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        m = max(m, off[i + 1] - off[i]);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, d));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// ------------------------------------------------------------------ key image
// image[w * n + r] = bytes [8w, 8w+8) of row r's key image, first byte most significant.  A value
// longer than the column width (possible for probe / lookup values only) keeps its first `width`
// bytes and gets the all-ones length, which orders it after every real key sharing those bytes and
// never compares equal.
__global__ void key_pack_kernel(KeyDesc kd, uint64_t n, uint64_t* image) {
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    uint64_t cur = 0; int cnt = 0; uint32_t word = 0;
    auto push = [&](uint32_t b) {
        cur = (cur << 8) | b;
        if (++cnt == 8) { image[(uint64_t)word * n + r] = cur; word++; cnt = 0; cur = 0; }
    };
    for (int k = 0; k < kd.nkeys; k++) {
        uint32_t s = kd.off[k][r], len = kd.off[k][r + 1] - s;
        const uint8_t* p = kd.data[k] + s;
        uint32_t w = kd.width[k];
        for (uint32_t i = 0; i < w; i++) push(i < len ? p[i] : 0u);
        uint32_t lf = len > w ? 0xffffffffu : len;
        for (int i = (int)kd.lenbytes[k] - 1; i >= 0; i--) push((lf >> (8 * i)) & 0xffu);
    }
    if (cnt) { cur <<= 8 * (8 - cnt); image[(uint64_t)word * n + r] = cur; }
}

// ------------------------------------------------------------------ radix sort of (u64 key, u32 value)
constexpr int RS_THREADS = 256;
constexpr int RS_ITEMS = 8;
constexpr int RS_TILE = RS_THREADS * RS_ITEMS;

void iota_u32(Ctx* c, uint32_t* p, uint64_t n) {
    each_row(c, n, [=] __device__(uint64_t i) { p[i] = (uint32_t)i; });
}
// dst[i] = src[idx[i]]
static void gather_u64(Ctx* c, const uint64_t* src, const uint32_t* idx, uint64_t* dst, uint64_t n) {
    each_row(c, n, [=] __device__(uint64_t i) { dst[i] = src[idx[i]]; });
}
// histogram of all 8 bytes of every key: hist[b * 256 + v]
__global__ void hist8_kernel(const uint64_t* __restrict__ keys, uint64_t n, uint32_t* hist) {
    __shared__ uint32_t sh[8 * 256];
    for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t k = keys[i];
#pragma unroll
        for (int b = 0; b < 8; b++) atomicAdd(&sh[b * 256 + ((k >> (8 * b)) & 0xff)], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) if (sh[i]) atomicAdd(&hist[i], sh[i]);
}
// per-block digit counts over the block's contiguous tile range: counts[d * nblocks + block]
__global__ void __launch_bounds__(RS_THREADS) radix_count_kernel(const uint64_t* __restrict__ keys, uint64_t n, int shift,
                                                                 uint64_t tiles_per_block, uint32_t* counts) {
    __shared__ uint32_t sh[256];
    sh[threadIdx.x] = 0;
    __syncthreads();
    uint64_t lo = (uint64_t)blockIdx.x * tiles_per_block * RS_TILE;
    uint64_t hi = min(n, lo + tiles_per_block * RS_TILE);
    for (uint64_t i = lo + threadIdx.x; i < hi; i += RS_THREADS) atomicAdd(&sh[(keys[i] >> shift) & 0xff], 1u);
    __syncthreads();
    counts[(uint64_t)threadIdx.x * gridDim.x + blockIdx.x] = sh[threadIdx.x];
}
__global__ void __launch_bounds__(RS_THREADS) radix_scatter_kernel(const uint64_t* __restrict__ kin, const uint32_t* __restrict__ vin,
                                                                   uint64_t* kout, uint32_t* vout, uint64_t n, int shift,
                                                                   uint64_t tiles_per_block, const uint32_t* __restrict__ bases) {
    __shared__ uint32_t cnt[RS_THREADS / 32][256];
    __shared__ uint32_t base[256];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    base[tid] = bases[(uint64_t)tid * gridDim.x + blockIdx.x];
    uint64_t lo = (uint64_t)blockIdx.x * tiles_per_block * RS_TILE;
    uint64_t hi = min(n, lo + tiles_per_block * RS_TILE);
    for (uint64_t t0 = lo; t0 < hi; t0 += RS_TILE) {
        for (int i = tid; i < (RS_THREADS / 32) * 256; i += RS_THREADS) (&cnt[0][0])[i] = 0;
        __syncthreads();
        uint64_t k[RS_ITEMS]; uint32_t v[RS_ITEMS], rank[RS_ITEMS];
        const uint64_t wbase = t0 + (uint64_t)warp * 32 * RS_ITEMS;
#pragma unroll
        for (int i = 0; i < RS_ITEMS; i++) {
            uint64_t idx = wbase + i * 32 + lane;
            bool ok = idx < hi;
            k[i] = ok ? kin[idx] : 0; v[i] = ok ? vin[idx] : 0;
            uint32_t d = ok ? (uint32_t)((k[i] >> shift) & 0xff) : 0x100u;
            uint32_t peers = __match_any_sync(0xffffffffu, d);
            uint32_t pre = ok ? cnt[warp][d] : 0;
            __syncwarp();
            if (ok && lane == __ffs(peers) - 1) cnt[warp][d] = pre + __popc(peers);
            __syncwarp();
            rank[i] = pre + __popc(peers & lanemask_lt());
        }
        __syncthreads();
        {  // thread tid owns digit tid: exclusive prefix over warps, advance the running base
            uint32_t run = base[tid];
#pragma unroll
            for (int w = 0; w < RS_THREADS / 32; w++) { uint32_t c = cnt[w][tid]; cnt[w][tid] = run; run += c; }
            base[tid] = run;
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < RS_ITEMS; i++) {
            uint64_t idx = wbase + i * 32 + lane;
            if (idx < hi) {
                uint32_t d = (uint32_t)((k[i] >> shift) & 0xff);
                uint32_t pos = cnt[warp][d] + rank[i];
                kout[pos] = k[i]; vout[pos] = v[i];
            }
        }
        __syncthreads();
    }
}

// skip[w * 8 + b] = 1 when byte b (0 = least significant) of image word w is the same in every row, so that a radix pass
// over it would be the identity.  Which digits are constant does not depend on the order of the rows: the byte
// histograms of ALL image words are taken up front and read back with one host round trip.
static std::vector<uint8_t> constant_digits(Ctx* c, const uint64_t* image, uint32_t words, uint64_t n, uint64_t* traffic) {
    Buf hist = dev_alloc(c, (size_t)words * 8 * 256 * 4);
    CPB_CUDA(cudaMemsetAsync(hist->p, 0, (size_t)words * 8 * 256 * 4, c->stream));
    {
        KernelTimer kt(c, "sort_hist", n * 8 * words, (int)words);
        for (uint32_t w = 0; w < words; w++)
            hist8_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(image + (uint64_t)w * n, n, hist->as<uint32_t>() + (size_t)w * 8 * 256);
        CPB_CUDA(cudaGetLastError());
    }
    *traffic += n * 8 * words;
    const std::vector<uint32_t> hh = read_back<uint32_t>(c, hist->p, (size_t)words * 8 * 256);
    std::vector<uint8_t> skip((size_t)words * 8, 0);
    for (uint32_t w = 0; w < words; w++)
        for (int b = 0; b < 8; b++)
            for (int v = 0; v < 256; v++) if (hh[((size_t)w * 8 + b) * 256 + v] == n) skip[(size_t)w * 8 + b] = 1;
    return skip;
}

// Stable sort of `perm` (row ids) by image words [0, words): returns the buffer holding the sorted ids.  Constant digits
// (constant_digits) are not passed over (round 1: one host round trip per image word).
Buf sort_by_image(Ctx* c, const uint64_t* image, uint32_t words, uint64_t n, uint64_t* traffic) {
    Buf permA = dev_alloc(c, n * 4), permB = dev_alloc(c, n * 4), keyA = dev_alloc(c, n * 8), keyB = dev_alloc(c, n * 8);
    iota_u32(c, permA->as<uint32_t>(), n);
    const uint64_t ntiles = (n + RS_TILE - 1) / RS_TILE;
    const uint32_t nblocks = (uint32_t)std::min<uint64_t>(ntiles, (uint64_t)c->sm_count * 4);
    const uint64_t tpb = (ntiles + nblocks - 1) / nblocks;
    Buf counts = dev_alloc(c, (256ull * nblocks + 1) * 4), tot = dev_alloc(c, 8);
    const std::vector<uint8_t> skip = constant_digits(c, image, words, n, traffic);
    for (int w = (int)words - 1; w >= 0; w--) {
        bool any = false;
        for (int b = 0; b < 8; b++) any = any || !skip[(size_t)w * 8 + b];
        if (!any) continue;  // the whole word is constant
        {
            KernelTimer kt(c, "sort_gather_word", n * 20);
            gather_u64(c, image + (uint64_t)w * n, permA->as<uint32_t>(), keyA->as<uint64_t>(), n);
        }
        *traffic += n * 20;
        for (int b = 0; b < 8; b++) {
            if (skip[(size_t)w * 8 + b]) continue;  // every key has the same byte here: the pass would be the identity
            KernelTimer kt(c, "radix_pass", n * 32, 3);
            radix_count_kernel<<<nblocks, RS_THREADS, 0, c->stream>>>(keyA->as<uint64_t>(), n, 8 * b, tpb, counts->as<uint32_t>());
            exclusive_scan_u32(c, counts->as<uint32_t>(), counts->as<uint32_t>(), 256ull * nblocks, tot->as<uint64_t>());
            radix_scatter_kernel<<<nblocks, RS_THREADS, 0, c->stream>>>(keyA->as<uint64_t>(), permA->as<uint32_t>(), keyB->as<uint64_t>(),
                                                                        permB->as<uint32_t>(), n, 8 * b, tpb, counts->as<uint32_t>());
            CPB_CUDA(cudaGetLastError());
            std::swap(keyA, keyB); std::swap(permA, permB);
            *traffic += n * 32;
        }
    }
    return permA;
}

// ------------------------------------------------------------------ top-k selection: MSD radix select
// The threshold is found digit by digit, most significant first, on the device: a pass histograms one digit of the rows
// still in the running (their higher digits equal the threshold's so far) and a one-block step picks the bucket that
// holds the need-th of them.  st[r] holds row r's digit of the last pass, or SEL_OUT once the row left the running: pass
// p + 1 keeps the rows whose digit is the bucket pass p chose, so no pass reads an earlier word again.
constexpr uint16_t SEL_OUT = 0xFFFF;
struct SelState {
    uint64_t need;    // rows still to take among those equal to the threshold so far
    uint32_t choice;  // the bucket the last pass chose
    uint32_t first;   // no pass has run yet: every row is in the running
    uint32_t done;    // the chosen bucket is taken whole: the threshold is known as far as it matters
};
__global__ void __launch_bounds__(256) select_hist_kernel(const uint64_t* __restrict__ word, uint64_t n, int shift, uint16_t* __restrict__ st,
                                                          const SelState* __restrict__ s, uint32_t* __restrict__ hist) {
    if (s->done) return;
    __shared__ uint32_t sh[256];
    sh[threadIdx.x] = 0;
    __syncthreads();
    const bool first = s->first != 0;
    const uint32_t prev = s->choice;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (!first) {
            const uint16_t v = st[i];
            if (v != prev) {
                if (v != SEL_OUT) st[i] = SEL_OUT;
                continue;
            }
        }
        const uint32_t d = (uint32_t)(word[i] >> shift) & 0xffu;
        st[i] = (uint16_t)d;
        atomicAdd(&sh[d], 1u);
    }
    __syncthreads();
    if (sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], sh[threadIdx.x]);
}
// one block of 256 threads: the bucket d holding the need-th row in the running; its digit goes into the threshold and
// its mask, need becomes the rank within d, and hist is cleared for the next pass
__global__ void __launch_bounds__(256) select_choose_kernel(uint32_t* __restrict__ hist, SelState* __restrict__ s, uint64_t* __restrict__ thr,
                                                            uint64_t* __restrict__ mask, int shift) {
    __shared__ uint32_t sc[256];
    const uint32_t t = threadIdx.x, h = hist[t];
    const bool live = !s->done;
    const uint64_t need = s->need;
    sc[t] = h;
    __syncthreads();
    for (uint32_t d = 1; d < 256; d <<= 1) {  // inclusive scan
        const uint32_t v = t >= d ? sc[t - d] : 0;
        __syncthreads();
        sc[t] += v;
        __syncthreads();
    }
    const uint64_t below = sc[t] - h;
    if (live && h && below < need && need <= below + h) {
        s->need = need - below;
        s->choice = t;
        s->first = 0;
        s->done = need - below == h;
        *thr |= (uint64_t)t << shift;
        *mask |= 0xffull << shift;
    }
    hist[t] = 0;
}

// The first k rows (0 < k < n) of the order (image words [0, words) as unsigned integers, then row), as ascending row
// ids uint32[k + 1] (the last entry is n).  One host synchronisation (constant_digits).
Buf select_by_image(Ctx* c, const uint64_t* image, uint32_t words, uint64_t n, uint64_t k, uint64_t* traffic) {
    const std::vector<uint8_t> skip = constant_digits(c, image, words, n, traffic);
    Buf st = dev_alloc(c, n * 2), state = dev_alloc(c, sizeof(SelState)), hist = dev_alloc(c, 256 * 4),
        thr = dev_alloc(c, (size_t)words * 16);
    uint64_t* th = thr->as<uint64_t>();
    uint64_t* mk = th + words;  // the digits of the threshold that are known (constant digits never are: every row has them)
    const SelState s0{k, 0, 1, 0};
    CPB_CUDA(cudaMemcpyAsync(state->p, &s0, sizeof s0, cudaMemcpyHostToDevice, c->stream));
    CPB_CUDA(cudaMemsetAsync(hist->p, 0, 256 * 4, c->stream));
    CPB_CUDA(cudaMemsetAsync(thr->p, 0, (size_t)words * 16, c->stream));
    SelState* sp = state->as<SelState>();
    {
        int passes = 0;
        for (uint32_t w = 0; w < words; w++)
            for (int b = 0; b < 8; b++) passes += !skip[(size_t)w * 8 + b];
        KernelTimer kt(c, "select_pass", n * 12 * (uint64_t)passes, 2 * passes);
        for (uint32_t w = 0; w < words; w++)
            for (int b = 7; b >= 0; b--) {
                if (skip[(size_t)w * 8 + b]) continue;
                select_hist_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(image + (uint64_t)w * n, n, 8 * b, st->as<uint16_t>(), sp,
                                                                            hist->as<uint32_t>());
                select_choose_kernel<<<1, 256, 0, c->stream>>>(hist->as<uint32_t>(), sp, th + w, mk + w, 8 * b);
            }
        CPB_CUDA(cudaGetLastError());
    }
    st.reset();
    // the rows below the threshold, and the first `need` rows equal to it in row order: k rows, as the choices made sure
    Buf lt = dev_alloc(c, n * 4), eq = dev_alloc(c, n * 4), pos = dev_alloc(c, (n + 1) * 4), tot = dev_alloc(c, 8), ids = dev_alloc(c, (k + 1) * 4);
    {
        KernelTimer kt(c, "select_take", n * (8 * (uint64_t)words + 40), 4);
        uint32_t *l = lt->as<uint32_t>(), *e = eq->as<uint32_t>(), *ep = pos->as<uint32_t>();
        each_row(c, n, [=] __device__(uint64_t i) {
            int r = 0;
            for (uint32_t w = 0; w < words && r == 0; w++) {
                const uint64_t m = mk[w], x = image[(uint64_t)w * n + i] & m, y = th[w] & m;
                r = x < y ? -1 : x > y ? 1 : 0;
            }
            l[i] = r < 0; e[i] = r == 0;
        });
        exclusive_scan_u32(c, e, ep, n, tot->as<uint64_t>());
        each_row(c, n, [=] __device__(uint64_t i) { l[i] = l[i] || (e[i] && ep[i] < sp->need); });
        exclusive_scan_u32(c, l, ep, n, tot->as<uint64_t>());  // (the ranks among the equal rows are used up)
        compact_flags(c, FlagScan{l, n, pos, k}, 0, ids->as<uint32_t>());
    }
    *traffic += n * 12 * 8 * (uint64_t)words + n * (8 * (uint64_t)words + 40);
    return ids;
}

// ------------------------------------------------------------------ adjacent compare (unique check, groups)
void head_flags(Ctx* c, const uint64_t* image, uint64_t n, uint32_t pbytes, uint32_t* head) {
    each_row(c, n, [=] __device__(uint64_t i) { head[i] = (i == 0 || !prefix_equal(image, n, i, image, n, i - 1, pbytes)) ? 1u : 0u; });
}
// nonzero when the row after row i starts a run of equal keys; past the last row, one always starts
__device__ __forceinline__ uint32_t next_head(const uint32_t* head, uint64_t last, uint64_t i) { return i == last ? 1u : head[i + 1]; }

void describe_keys(Ctx* c, const Table& t, const std::vector<int>& kidx, const std::vector<uint32_t>& width, KeyDesc& kd) {
    kd.nkeys = (int)kidx.size();
    uint32_t bytes = 0;
    for (int k = 0; k < kd.nkeys; k++) {
        kd.off[k] = t.cols[kidx[k]].off(); kd.data[k] = t.cols[kidx[k]].bytes();
        kd.width[k] = width[k];
        kd.lenbytes[k] = len_field_bytes(width[k]);
        bytes += kd.width[k] + kd.lenbytes[k];
    }
    kd.words = (bytes + 7) / 8;
    (void)c;
}

// bytes of the image covered by the first nk key columns
uint32_t prefix_bytes(const Index& ix, int nk) {
    uint32_t b = 0;
    for (int k = 0; k < nk; k++) b += ix.key_width[k] + len_field_bytes(ix.key_width[k]);
    return b;
}

// packs rows of `t` (columns kidx) with the widths of an existing index: probe / lookup images
Buf pack_with_widths(Ctx* c, const Table& t, const std::vector<int>& kidx, const std::vector<uint32_t>& width, uint32_t* words_out) {
    KeyDesc kd{};
    describe_keys(c, t, kidx, width, kd);
    *words_out = kd.words;
    Buf img = dev_alloc(c, std::max<uint64_t>(1, (uint64_t)kd.words * (uint64_t)t.nrows) * 8);
    pack_into(c, t, kidx, width, img->as<uint64_t>());
    return img;
}
void pack_into(Ctx* c, const Table& t, const std::vector<int>& kidx, const std::vector<uint32_t>& width, uint64_t* dst) {
    KeyDesc kd{};
    describe_keys(c, t, kidx, width, kd);
    const uint64_t n = (uint64_t)t.nrows;
    if (n && kd.words) {
        KernelTimer kt(c, "key_pack", n * kd.words * 8);
        key_pack_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(kd, n, dst);
        CPB_CUDA(cudaGetLastError());
    }
}

// the longest row of up to 4 columns taken together (the bytes of all their values in one row)
struct RowCols { int nc; const uint32_t* off[4]; };
__global__ void max_row_bytes_kernel(RowCols rc, uint64_t n, uint32_t* out) {
    uint32_t m = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t t = 0;
#pragma unroll
        for (int c = 0; c < 4; c++) if (c < rc.nc) t += rc.off[c][i + 1] - rc.off[c][i];
        m = max(m, t);
    }
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// per key column the longest value of rows [0, n) of t: the column widths of the key image.  With `row_cols` (at most
// 4 columns), *row_max = their longest row, from the same readback.
std::vector<uint32_t> key_widths(Ctx* c, const Table& t, const std::vector<int>& key_cols, uint64_t n, const std::vector<int>* row_cols,
                                 uint32_t* row_max) {
    const size_t nk = key_cols.size();
    Buf wd = dev_alloc(c, (nk + 1) * 4);
    CPB_CUDA(cudaMemsetAsync(wd->p, 0, (nk + 1) * 4, c->stream));
    for (size_t k = 0; k < nk && n; k++)
        max_len_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(t.cols[key_cols[k]].off(), n, wd->as<uint32_t>() + k);
    if (row_cols && !row_cols->empty() && n) {
        RowCols rc{};
        rc.nc = (int)row_cols->size();
        for (int j = 0; j < rc.nc; j++) rc.off[j] = t.cols[(*row_cols)[j]].off();
        max_row_bytes_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(rc, n, wd->as<uint32_t>() + nk);
    }
    CPB_CUDA(cudaGetLastError());
    std::vector<uint32_t> w = read_back<uint32_t>(c, wd->p, nk + 1);
    if (row_max) *row_max = w[nk];
    w.pop_back();
    return w;
}

// rows ids[0..m) of a key image of n_src rows, as an image of m rows
Buf gather_image(Ctx* c, const uint64_t* image, uint32_t words, uint64_t n_src, const uint32_t* ids, uint64_t m) {
    Buf out = dev_alloc(c, std::max<uint64_t>(1, (uint64_t)words * m) * 8);
    for (uint32_t w = 0; w < words; w++) gather_u64(c, image + (uint64_t)w * n_src, ids, out->as<uint64_t>() + (uint64_t)w * m, m);
    return out;
}

// while in scope, what c allocates stays inside an index: it comes from the pool of the index's owner (dev_alloc)
struct OwnerPool {
    Ctx* c; Ctx* prev;
    OwnerPool(Ctx* ctx, Ctx* owner) : c(ctx), prev(ctx->alloc_for) { c->alloc_for = owner; }
    ~OwnerPool() { c->alloc_for = prev; }
    OwnerPool(const OwnerPool&) = delete; OwnerPool& operator=(const OwnerPool&) = delete;
};

static void ensure_sorted_locked(Ctx* c, Index& ix) {
    if (ix.sorted) return;
    const uint64_t n = (uint64_t)ix.nrows;
    OwnerPool scope(c, ix.ctx);
    uint32_t words = ix.image_words;
    const Buf uimg = ix.derived.uimage ? ix.derived.uimage : pack_with_widths(c, *ix.src, ix.key_col_idx, ix.key_width, &words);  // (row-carrying table)
    uint64_t traffic = 0;
    Buf perm = sort_by_image(c, uimg->as<uint64_t>(), ix.image_words, n, &traffic);
    Buf simg;
    {
        KernelTimer kt(c, "image_gather", (uint64_t)ix.image_words * n * 20, (int)ix.image_words);
        simg = gather_image(c, uimg->as<uint64_t>(), ix.image_words, n, perm->as<uint32_t>(), n);
    }
    sync_stream(c);  // complete before another context (stream) can see it
    ix.perm = perm; ix.image = simg; ix.sorted = true;
}
void ensure_sorted(Ctx* c, Index& ix) {
    std::lock_guard<std::mutex> lk(ix.mu);
    ensure_sorted_locked(c, ix);
}

std::shared_ptr<Table> sorted_table(Ctx* c, Index& ix) {
    std::lock_guard<std::mutex> lk(ix.mu);
    if (ix.table) return ix.table;
    ensure_sorted_locked(c, ix);
    OwnerPool scope(c, ix.ctx);
    ix.table = gather_rows(c, *ix.src, ix.perm->as<uint32_t>(), ix.nrows);
    ix.table->first_line = 0;  // iterating an Index reports 0-based rows (csvplus.go:243)
    sync_stream(c);  // complete before another context (stream) can see it
    return ix.table;
}

std::shared_ptr<Index> build_index(Ctx* c, std::shared_ptr<Table> tp, const std::vector<std::string>& keys, bool unique) {
    const Table& t = *tp;
    if ((int)keys.size() > MAXKEYS) throw ArgError{CPB_ERR_UNSUPPORTED, "more than 16 index key columns"};
    auto ix = std::make_shared<Index>();
    ix->ctx = c; ix->key_cols = keys;
    const uint64_t n = (uint64_t)t.nrows;
    for (size_t k = 0; k < keys.size(); k++) {
        int ci = t.find(keys[k]);
        if (ci < 0) {
            if (n == 0) { ci = -1; }
            else  // csvplus.go:723-727, raised for the first row pulled
                throw DataError{CPB_E_MISSING_INDEX_COLUMN, (int)k, t.first_line, true, "missing column " + go_quote(keys[k]) + " while creating an index"};
        }
        ix->key_col_idx.push_back(ci);
    }
    if (n == 0) {
        auto e = std::make_shared<Table>(t); e->nrows = 0;
        ix->table = e; ix->src = e; ix->nrows = 0; ix->key_width.assign(keys.size(), 0); ix->image_words = 0; ix->image = dev_alloc(c, 8);
        for (auto& ci : ix->key_col_idx) if (ci < 0) ci = 0;
        return ix;
    }
    if (n > 0xfffffffeull) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "an index holds at most 2^32-2 rows"};
    const bool lazy = unique && n >= 2;
    // 1. key widths; for a UniqueIndexOn with at most 4 other columns also their longest row: whether the row-carrying
    //    hash table can hold the index
    std::vector<int> pay;  // the non-key columns, in schema order
    for (int q = 0; q < (int)t.cols.size(); q++)
        if (std::find(ix->key_col_idx.begin(), ix->key_col_idx.end(), q) == ix->key_col_idx.end()) pay.push_back(q);
    uint32_t pay_max = ~0u;
    {
        KernelTimer kt(c, "key_width", n * 4 * keys.size(), (int)keys.size());
        ix->key_width = key_widths(c, t, ix->key_col_idx, n, lazy && (int)pay.size() <= RH_MAXC ? &pay : nullptr, &pay_max);
    }
    const uint32_t kbytes = prefix_bytes(*ix, (int)keys.size()), words = (kbytes + 7) / 8;
    ix->image_words = words;
    if ((uint64_t)words * 8 > MAX_KEY_IMAGE_BYTES) throw ArgError{CPB_ERR_UNSUPPORTED, "index keys longer than 4 KiB are not supported"};
    // 2. UniqueIndexOn: the duplicate check does not need the order — a probe table over the rows as they are, in which
    //    every key must find itself.  When it passes (the usual case) the sort is left for whoever needs the order.
    Buf img;  // image of the unsorted rows
    if (lazy) {
        ix->src = tp; ix->nrows = (int64_t)n; ix->sorted = false; ix->unique = true;
        bool dup_seen = false;
        if (kbytes <= 12 && (int)pay.size() <= RH_MAXC && pay_max <= RH_PAY) {
            // key, lengths and payload fit one 32-byte slot: the row-carrying table is the index's probe structure (and
            // its build the duplicate check); no key image until something needs the order
            ix->derived.rowhash.cols = pay;
            const RhBuild rb = rowhash_build(c, *ix);
            if (rb == RhBuild::built) return ix;
            ix->derived.rowhash = RowHash{};
            dup_seen = rb == RhBuild::duplicate;
        }
        // no row-carrying table, or one of its regions overflowed (keys crafted to collide): a probe table over the key
        // image in source order and the row slots, exact for any input
        if (!dup_seen) {
            img = pack_with_widths(c, t, ix->key_col_idx, ix->key_width, &ix->image_words);
            ix->derived.uimage = img;
            if (!index_has_duplicates(c, *ix)) return ix;
        }
        // a duplicate exists: sort, so that the error names the key the reference would name (the lowest in sort order)
        ix->reset_derived(); ix->unique = false; ix->sorted = true;
    }
    if (!img) img = pack_with_widths(c, t, ix->key_col_idx, ix->key_width, &ix->image_words);
    // 3. stable LSD radix sort -> permutation
    uint64_t traffic = 0;
    Buf perm = sort_by_image(c, img->as<uint64_t>(), words, n, &traffic);
    // 4. the sorted key image; the sorted rows themselves stay virtual (src + perm) until something needs them
    ix->src = tp; ix->perm = perm; ix->nrows = (int64_t)n;
    {
        KernelTimer kt(c, "image_gather", (uint64_t)words * n * 20, (int)words);
        ix->image = gather_image(c, img->as<uint64_t>(), words, n, perm->as<uint32_t>(), n);
    }
    const uint64_t* simg = ix->image->as<uint64_t>();
    // 5. uniqueness (createUniqueIndex, csvplus.go:740-756)
    if (unique && n >= 2) {
        Buf head = dev_alloc(c, n * 4), first = dev_alloc(c, 8);
        CPB_CUDA(cudaMemsetAsync(first->p, 0xff, 8, c->stream));
        {
            KernelTimer kt(c, "unique_check", (uint64_t)words * n * 8, 2);
            uint32_t* hd = head->as<uint32_t>();
            unsigned long long* fd = (unsigned long long*)first->p;
            head_flags(c, simg, n, words * 8, hd);
            each_row(c, n, [=] __device__(uint64_t i) { if (i >= 1 && hd[i] == 0) atomicMin(fd, (unsigned long long)i); });
        }
        const uint64_t fd = read_back<uint64_t>(c, first->p);
        if (fd != ~0ull) {
            // "duplicate value while creating unique index: " + rows[i].SelectExisting(columns...).String()  (:751, :90-104)
            std::vector<std::pair<std::string, std::string>> kv;
            for (size_t k = 0; k < keys.size(); k++) {
                const Column& col = sorted_table(c, *ix)->cols[ix->key_col_idx[k]];
                const std::vector<uint32_t> oo = read_back<uint32_t>(c, col.off() + fd, 2);
                const std::vector<char> v = read_back<char>(c, col.bytes() + oo[0], oo[1] - oo[0]);
                kv.emplace_back(keys[k], std::string(v.begin(), v.end()));
            }
            std::sort(kv.begin(), kv.end());
            std::string s = "{ ";
            for (size_t i = 0; i < kv.size(); i++) { if (i) s += ", "; s += "\"" + kv[i].first + "\" : \"" + kv[i].second + "\""; }
            s += " }";
            throw DataError{CPB_E_DUPLICATE_KEY, -1, 0, false, "duplicate value while creating unique index: " + s};
        }
    }
    ix->unique = unique;
    return ix;
}

// ------------------------------------------------------------------ ResolveDuplicates support
// indexImpl.dedup's walk (csvplus.go:814-859) over rows in any order, one thread: a group starts at the first adjacent
// equal pair (i - 1, i) with i >= lower (pairs: those i, ascending) and ends at upper = lower + sort.Search(n - lower,
// row > key) (:831), which on rows out of key order can take in rows with other keys; the next search starts at
// upper + 1.  Groups [lo, hi) come out ascending and disjoint.
__global__ void dup_walk_kernel(const uint64_t* __restrict__ image, uint64_t n, uint32_t pbytes, const uint32_t* __restrict__ pairs,
                                uint64_t npairs, uint32_t* lo, uint32_t* hi, unsigned long long* ngroups) {
    uint64_t g = 0, lower = 1, p = 0;
    for (;;) {
        uint64_t a = p, b = npairs;
        while (a < b) { const uint64_t h = a + (b - a) / 2; if (pairs[h] < lower) a = h + 1; else b = h; }
        if (a == npairs) break;
        p = a; lower = pairs[a];
        uint64_t i = lower, j = n;  // (the midpoints of sort.Search over [0, n - lower), offset by lower)
        while (i < j) { const uint64_t h = i + (j - i) / 2; if (prefix_cmp(image, n, h, image, n, lower, pbytes) <= 0) i = h + 1; else j = h; }
        lo[g] = (uint32_t)(lower - 1); hi[g] = (uint32_t)i; g++;
        lower = i + 1;
    }
    *ngroups = g;
}
void index_dup_groups(Ctx* c, Index& ix, std::vector<int64_t>& lo, std::vector<int64_t>& hi) {
    lo.clear(); hi.clear();
    const uint64_t n = (uint64_t)ix.nrows;
    if (n < 2 || ix.unique) return;  // (a verified unique index has no duplicate group)
    auto compact = [&](const Buf& flags, uint32_t add, uint64_t* count) {
        const FlagScan s = scan_flags(c, flags->as<uint32_t>(), n);
        Buf out = dev_alloc(c, (s.count + 1) * 4);
        compact_flags(c, s, add, out->as<uint32_t>());
        *count = s.count;
        return out;
    };
    Buf head = dev_alloc(c, n * 4), gs = dev_alloc(c, n * 4);
    uint32_t* hd = head->as<uint32_t>();
    uint64_t ng = 0, ne = 0;
    Buf los, his;
    if (ix.in_order) {  // a group is a run of equal keys: its first row is a head followed by a non-head, and so on
        Buf ge = dev_alloc(c, n * 4);
        {
            KernelTimer kt(c, "dedup_segments", (uint64_t)ix.image_words * n * 8 + n * 12, 2);
            head_flags(c, ix.image->as<uint64_t>(), n, ix.image_words * 8, hd);
            // group start: a head followed by a non-head; group end (exclusive hi = i + 1): a non-head followed by a head
            uint32_t *s = gs->as<uint32_t>(), *e = ge->as<uint32_t>();
            const uint64_t last = n - 1;
            each_row(c, n, [=] __device__(uint64_t i) {
                const bool h = hd[i] != 0, nh = next_head(hd, last, i) != 0;
                s[i] = (h && !nh) ? 1u : 0u;
                e[i] = (!h && nh) ? 1u : 0u;
            });
        }
        los = compact(gs, 0, &ng);
        his = compact(ge, 1, &ne);
        if (ng != ne) throw ArgError{CPB_ERR_CUDA, "internal: group start/end mismatch"};
    } else {
        {
            KernelTimer kt(c, "dedup_segments", (uint64_t)ix.image_words * n * 8 + n * 8, 2);
            head_flags(c, ix.image->as<uint64_t>(), n, ix.image_words * 8, hd);
            nonzero_flags(c, hd, n, false, gs->as<uint32_t>());
        }
        uint64_t npairs = 0;
        Buf pairs = compact(gs, 0, &npairs);
        if (npairs == 0) return;
        los = dev_alloc(c, npairs * 4); his = dev_alloc(c, npairs * 4);
        Buf cnt = dev_alloc(c, 8);
        {
            KernelTimer kt(c, "dedup_walk", 0);
            dup_walk_kernel<<<1, 1, 0, c->stream>>>(ix.image->as<uint64_t>(), n, ix.image_words * 8, pairs->as<uint32_t>(), npairs,
                                                    los->as<uint32_t>(), his->as<uint32_t>(), (unsigned long long*)cnt->p);
            CPB_CUDA(cudaGetLastError());
        }
        ng = read_back<uint64_t>(c, cnt->p);
    }
    std::vector<uint32_t> a(ng), b(ng);
    if (ng) {
        CPB_CUDA(cudaMemcpyAsync(a.data(), los->p, ng * 4, cudaMemcpyDeviceToHost, c->stream));
        CPB_CUDA(cudaMemcpyAsync(b.data(), his->p, ng * 4, cudaMemcpyDeviceToHost, c->stream));
        sync_stream(c);
    }
    lo.assign(a.begin(), a.end()); hi.assign(b.begin(), b.end());
}

void index_adopt_rows(Ctx* c, Index& ix, std::shared_ptr<Table> nt) {
    const uint64_t m = (uint64_t)nt->nrows;
    nt->first_line = 0;
    ix.table = nt; ix.src = nullptr; ix.perm = nullptr; ix.sorted = true; ix.nrows = (int64_t)m; ix.unique = false;
    ix.reset_derived();
    for (size_t k = 0; k < ix.key_cols.size(); k++) ix.key_col_idx[k] = nt->find(ix.key_cols[k]);
    ix.key_width = key_widths(c, *nt, ix.key_col_idx, m);
    uint32_t words = 0;
    ix.image = pack_with_widths(c, *nt, ix.key_col_idx, ix.key_width, &words);
    ix.image_words = words;
    ix.in_order = true;
    if (m >= 2 && words) {
        Buf flag = dev_alloc(c, 8);
        CPB_CUDA(cudaMemsetAsync(flag->p, 0, 8, c->stream));
        {
            // *out = 1 when some row's key image is below the previous row's
            KernelTimer kt(c, "order_check", m * words * 8);
            const uint64_t* image = ix.image->as<uint64_t>();
            uint32_t* out = flag->as<uint32_t>();
            each_row(c, m, [=] __device__(uint64_t i) {
                if (i == 0) return;
                for (uint32_t w = 0; w < words; w++) {
                    const uint64_t a = image[(uint64_t)w * m + i - 1], b = image[(uint64_t)w * m + i];
                    if (a != b) { if (a > b) *out = 1u; return; }  // benign race: every writer stores 1
                }
            });
        }
        ix.in_order = read_back<uint32_t>(c, flag->p) == 0;
    }
}

// indexImpl.dedup (csvplus.go:810-867) with the resolver's choices already made on the host.
// keep[g] >= 0: stored position of the row kept for group g; -1: the group is dropped (the resolver returned an "empty"
// row, :845); <= -2: the resolver returned a row that is not one of the group's rows — row (-2 - keep[g]) of `repl`
// takes the place of the group (:846 stores whatever row came back; the index is NOT re-sorted, exactly like the reference).
// The rows kept: every row outside the groups, the chosen row of each group, in stored order — except that the walk
// never copies the last row when no group covers it (SURVEY §Q1, bug_compatible).
void index_dedup_apply(Ctx* c, Index& ix, const std::vector<int64_t>& keep_in, bool bug_compatible, const Table* repl) {
    const uint64_t n = (uint64_t)ix.nrows;
    if (n < 2 || keep_in.empty()) return;  // no duplicate group: the reference returns early (:820-822)
    sorted_table(c, ix);
    std::vector<int64_t> keep = keep_in;
    // groups answered with a replacement row keep their first position as the slot the new row goes to
    std::vector<int64_t> rpos; std::vector<uint32_t> rid;
    bool any_repl = false;
    for (auto k : keep) if (k <= -2) any_repl = true;
    std::vector<int64_t> lo, hi;
    if (any_repl || !ix.in_order) index_dup_groups(c, ix, lo, hi);
    if (any_repl) {
        if (!repl) throw ArgError{CPB_ERR_ARG, "replacement rows referenced but no replacement table given"};
        if (repl->cols.size() != ix.table->cols.size()) throw ArgError{CPB_ERR_UNSUPPORTED, "a replacement row must have the columns of the index rows"};
        for (auto& col : ix.table->cols) if (repl->find(col.name) < 0) throw ArgError{CPB_ERR_UNSUPPORTED, "a replacement row must have the columns of the index rows"};
        if (lo.size() != keep.size()) throw ArgError{CPB_ERR_ARG, "keep[] does not match the duplicate groups of the index"};
        for (size_t g = 0; g < keep.size(); g++)
            if (keep[g] <= -2) {
                const int64_t j = -2 - keep[g];
                if (j >= repl->nrows) throw ArgError{CPB_ERR_ARG, "replacement row out of range"};
                rpos.push_back(lo[g]); rid.push_back((uint32_t)(n + (uint64_t)j));
                keep[g] = lo[g];
            }
    }
    // flag = the rows outside the groups.  In key order the groups are the runs of equal keys, so those are the rows
    // that are heads of runs of one; out of key order they come from the groups the walk found.
    Buf flag = dev_alloc(c, n * 4);
    uint32_t* fl = flag->as<uint32_t>();
    bool last_outside = false;
    if (ix.in_order) {
        Buf head = dev_alloc(c, n * 4);
        uint32_t* hd = head->as<uint32_t>();
        head_flags(c, ix.image->as<uint64_t>(), n, ix.image_words * 8, hd);
        const uint64_t last = n - 1;
        each_row(c, n, [=] __device__(uint64_t i) {
            const bool h = hd[i] != 0, nh = next_head(hd, last, i) != 0;
            fl[i] = (h && nh) ? 1u : 0u;
        });
        if (bug_compatible) last_outside = read_back<uint32_t>(c, hd + (n - 1)) != 0;
    } else {
        std::vector<uint32_t> lh(lo.begin(), lo.end()), hh(hi.begin(), hi.end());
        Buf dlo = dev_alloc(c, (lh.size() + 1) * 4), dhi = dev_alloc(c, (hh.size() + 1) * 4);
        if (!lh.empty()) {
            CPB_CUDA(cudaMemcpyAsync(dlo->p, lh.data(), lh.size() * 4, cudaMemcpyHostToDevice, c->stream));
            CPB_CUDA(cudaMemcpyAsync(dhi->p, hh.data(), hh.size() * 4, cudaMemcpyHostToDevice, c->stream));
        }
        // the rows outside the groups [lo, hi) (ascending, disjoint)
        const uint32_t *glo = dlo->as<uint32_t>(), *ghi = dhi->as<uint32_t>();
        const uint64_t ng = lh.size();
        each_row(c, n, [=] __device__(uint64_t i) {
            uint64_t a = 0, b = ng;  // groups starting at or before i
            while (a < b) { const uint64_t h = a + (b - a) / 2; if (glo[h] <= i) a = h + 1; else b = h; }
            fl[i] = (a == 0 || i >= ghi[a - 1]) ? 1u : 0u;
        });
        last_outside = hi.empty() || (uint64_t)hi.back() < n;
        sync_stream(c);  // lh / hh are pageable host vectors
    }
    Buf kd = dev_alloc(c, keep.size() * 8);
    CPB_CUDA(cudaMemcpyAsync(kd->p, keep.data(), keep.size() * 8, cudaMemcpyHostToDevice, c->stream));
    const int64_t* rows = kd->as<int64_t>();
    each_row(c, keep.size(), [=] __device__(uint64_t i) { if (rows[i] >= 0 && (uint64_t)rows[i] < n) fl[rows[i]] = 1u; });
    if (bug_compatible && last_outside) CPB_CUDA(cudaMemsetAsync(fl + (n - 1), 0, 4, c->stream));
    // compaction of the kept positions (the scanned positions are needed again to patch replacement ids in)
    const FlagScan kept = scan_flags(c, flag->as<uint32_t>(), n);
    const uint64_t m = kept.count;
    Buf ids = dev_alloc(c, (m + 1) * 4);
    compact_flags(c, kept, 0, ids->as<uint32_t>());
    std::shared_ptr<Table> nt;
    if (!rpos.empty()) {
        Buf dp = dev_alloc(c, rpos.size() * 8), dr = dev_alloc(c, rid.size() * 4);
        CPB_CUDA(cudaMemcpyAsync(dp->p, rpos.data(), rpos.size() * 8, cudaMemcpyHostToDevice, c->stream));
        CPB_CUDA(cudaMemcpyAsync(dr->p, rid.data(), rid.size() * 4, cudaMemcpyHostToDevice, c->stream));
        const uint32_t *pos = kept.pos->as<uint32_t>(), *with = dr->as<uint32_t>();
        const int64_t* at = dp->as<int64_t>();
        uint32_t* id = ids->as<uint32_t>();
        each_row(c, rpos.size(), [=] __device__(uint64_t i) { id[pos[at[i]]] = with[i]; });
        // rows [0, n) = the index, rows [n, n + repl) = the replacement rows in the index's column order
        Table rsel; rsel.ctx = c; rsel.nrows = repl->nrows;
        for (auto& col : ix.table->cols) rsel.cols.push_back(repl->cols[repl->find(col.name)]);
        auto both = concat_tables(c, {ix.table.get(), &rsel});
        nt = gather_rows(c, *both, ids->as<uint32_t>(), (int64_t)m);
        sync_stream(c);  // rpos / rid are pageable host vectors
        // keys may have changed (even their widths): the image is rebuilt from the new rows, their order is kept
        index_adopt_rows(c, ix, nt);
        return;
    }
    nt = gather_rows(c, *ix.table, ids->as<uint32_t>(), (int64_t)m);
    Buf simg = gather_image(c, ix.image->as<uint64_t>(), ix.image_words, n, ids->as<uint32_t>(), m);
    nt->first_line = 0;
    ix.table = nt; ix.src = nullptr; ix.perm = nullptr; ix.nrows = (int64_t)m; ix.image = simg;
    ix.reset_derived();
}

}  // namespace cpb
