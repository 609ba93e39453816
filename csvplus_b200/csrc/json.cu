// json.cu — DataSource.ToJSON (csvplus.go:446-474): json.Encoder with SetEscapeHTML(false), an empty indent and Encode's
// trailing '\n', over every column of a device table.
//
// The document is '[', then per row: ',' before every row but the first, '{', the pairs enc(name) ':' enc(value) joined
// by ',' with the columns in bytewise name order (strings.Compare, the order encoding/json gives map keys; computed once
// on the host), '}' '\n'; then ']'.  An empty source gives "[]", a row without columns "{}".
//
// enc(s) is encoding/json's appendString (go 1.23): '"', then the bytes from position i:
//   byte < 0x80:  '"' -> \"  and '\' -> \\ ;  0x0a 0x0d 0x09 -> \n \r \t ;  0x08 0x0c -> \b \f ;  any other byte < 0x20
//                 -> \u00xx (lowercase hex);  everything else verbatim, 0x7f and < > & included.
//   byte >= 0x80: if a complete sequence utf8.DecodeRune accepts starts at i (C2-DF +1 continuation byte; E0 A0-BF +1;
//                 E1-EC +2; ED 80-9F +1; EE-EF +2; F0 90-BF +2; F1-F3 +3; F4 80-8F +2) it is copied, except that
//                 E2 80 A8 / E2 80 A9 become \u2028 / \u2029; otherwise \ufffd is written and i advances ONE byte.
// then '"'.
//
// One call serialises one table or one row-range batch of a larger result: first_batch puts '[' before its first row
// (else ','), last_batch appends ']'.  An empty batch writes only those brackets, so first = last = 1 gives "[]".
// Kernels: json_row_len (bytes per row) -> exclusive_scan_u32 -> json_write (one warp per 32 rows through a shared
// stage, as csv_row_write_kernel).  Column descriptors live in a device array, so there is no column limit.
#include <algorithm>
#include <numeric>

#include "core.hpp"
#include "util.cuh"

namespace cpb {

struct JsonCol {
    const uint32_t* off; const uint8_t* data;
    uint32_t key, key_len;  // the column's prefix in the key blob: [","] enc(name) ':' '"'
};

// true when no byte of p[0..n) needs attention (< 0x20, '"', '\', >= 0x80): such a value is written as '"' p '"'.
// Reads the aligned 8-byte words covering the value; the word holding the last byte lies inside its allocation.
__device__ __forceinline__ bool json_plain(const uint8_t* p, uint32_t n) {
    if (n == 0) return true;
    constexpr uint64_t L = 0x0101010101010101ull, H = 0x8080808080808080ull;
    const uint32_t head = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 7u);
    const uint64_t* w = reinterpret_cast<const uint64_t*>(p - head);
    const uint64_t span = (uint64_t)head + n;
    for (uint64_t i = 0; i < span; i += 8) {
        uint64_t x = __ldg(w + i / 8);
        uint64_t valid = ~0ull;
        if (i == 0) valid <<= head * 8;
        if (span - i < 8) valid &= ~0ull >> ((8 - (span - i)) * 8);
        x = (x & valid) | (0x4141414141414141ull & ~valid);  // bytes outside the value read as 'A'
        const uint64_t q = x ^ (0x22 * L), b = x ^ (0x5c * L);
        if ((x | ((x - 0x20 * L) & ~x) | ((q - L) & ~q) | ((b - L) & ~b)) & H) return false;
    }
    return true;
}

// length of the valid UTF-8 sequence (utf8.DecodeRune) starting at p, 0 if none; p[0] >= 0x80, rem >= 1 bytes readable
__host__ __device__ inline uint32_t utf8_seq(const uint8_t* p, uint64_t rem) {
    const uint8_t c = p[0];
    uint32_t w;
    uint8_t lo = 0x80, hi = 0xBF;
    if (c < 0xC2) return 0;
    if (c < 0xE0) w = 2;
    else if (c < 0xF0) { w = 3; if (c == 0xE0) lo = 0xA0; else if (c == 0xED) hi = 0x9F; }
    else if (c < 0xF5) { w = 4; if (c == 0xF0) lo = 0x90; else if (c == 0xF4) hi = 0x8F; }
    else return 0;
    if (rem < w || p[1] < lo || p[1] > hi) return 0;
    for (uint32_t j = 2; j < w; j++) if ((p[j] & 0xC0) != 0x80) return 0;
    return w;
}

__host__ __device__ inline void put6(uint8_t* d, uint8_t a, uint8_t b, uint8_t c, uint8_t e) {
    d[0] = '\\'; d[1] = 'u'; d[2] = a; d[3] = b; d[4] = c; d[5] = e;
}

// the bytes of p[0..n) between enc's quotes; written to d unless d is null; returns their count
__host__ __device__ inline uint64_t json_escape(const uint8_t* p, uint64_t n, uint8_t* d) {
    uint64_t k = 0;
    for (uint64_t i = 0; i < n;) {
        const uint8_t c = p[i];
        if (c < 0x80) {
            i++;
            uint8_t e = 0;
            if (c == '"' || c == '\\') e = c;
            else if (c == '\n') e = 'n';
            else if (c == '\r') e = 'r';
            else if (c == '\t') e = 't';
            else if (c == 0x08) e = 'b';
            else if (c == 0x0c) e = 'f';
            if (e) { if (d) { d[k] = '\\'; d[k + 1] = e; } k += 2; }
            else if (c < 0x20) { if (d) put6(d + k, '0', '0', "0123456789abcdef"[c >> 4], "0123456789abcdef"[c & 15]); k += 6; }
            else { if (d) d[k] = c; k++; }
            continue;
        }
        const uint32_t w = utf8_seq(p + i, n - i);
        if (w == 0) { if (d) put6(d + k, 'f', 'f', 'f', 'd'); k += 6; i++; }
        else if (w == 3 && c == 0xE2 && p[i + 1] == 0x80 && (p[i + 2] == 0xA8 || p[i + 2] == 0xA9)) {
            if (d) put6(d + k, '2', '0', '2', p[i + 2] == 0xA8 ? '8' : '9');
            k += 6; i += 3;
        } else {
            if (d) for (uint32_t j = 0; j < w; j++) d[k + j] = p[i + j];
            k += w; i += w;
        }
    }
    return k;
}

// len[r] = output bytes of row r, saturated at 0xFFFFFFFF (the host then reports CPB_E_TOO_LARGE)
__global__ void json_row_len_kernel(const JsonCol* __restrict__ cols, int ncols, uint64_t row_const, uint64_t n, uint32_t* len) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    uint64_t total = row_const;
    for (int k = 0; k < ncols; k++) {
        const uint32_t* off = cols[k].off;
        const uint32_t s = off[r], l = off[r + 1] - s;
        const uint8_t* p = cols[k].data + s;
        total += json_plain(p, l) ? l : json_escape(p, l, nullptr);
    }
    len[r] = total > 0xffffffffull ? 0xffffffffu : (uint32_t)total;
}

// One warp serialises 32 consecutive rows into a per-warp shared stage laid out like the destination, then stores it
// with aligned 16-byte vectors (see csv_row_write_kernel).  A JSON row repeats every key, so it is several times longer
// than the CSV line of the same row (about 120-150 B for a joined orders x customers row): the stage holds 32 rows of
// up to 190 B, where ToCsv's 4 KB would send most such groups down the direct path.  Longer groups are written directly.
// The column descriptors and key prefixes are copied to shared memory when they fit (meta_smem), else read from global.
constexpr int JW_WARPS = 8;
constexpr int JW_STAGE = 6144;
constexpr uint32_t JW_STAGE_BYTES = JW_WARPS * (JW_STAGE + 16);
constexpr uint32_t JW_META_SMEM = 16384;
__global__ void __launch_bounds__(JW_WARPS * 32) json_write_kernel(const JsonCol* gcols, const uint8_t* gkeys, int ncols, uint32_t meta_bytes,
                                                                   int meta_smem, uint8_t first_byte, uint64_t n,
                                                                   const uint32_t* __restrict__ pos, uint8_t* out) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t* stage = smem + warp * (JW_STAGE + 16);
    const JsonCol* cols = gcols;
    const uint8_t* keys = gkeys;
    if (meta_smem) {  // descriptors then key blob, contiguous in global memory as in shared
        uint8_t* sm = smem + JW_STAGE_BYTES;
        const uint8_t* gm = reinterpret_cast<const uint8_t*>(gcols);
        for (uint32_t i = threadIdx.x; i < meta_bytes; i += blockDim.x) sm[i] = gm[i];
        __syncthreads();
        cols = reinterpret_cast<const JsonCol*>(sm);
        keys = sm + (gkeys - gm);
    }
    const uint64_t nwarps = (uint64_t)gridDim.x * JW_WARPS;
    for (uint64_t g = (uint64_t)blockIdx.x * JW_WARPS + warp; g * 32 < n; g += nwarps) {
        const uint64_t r = g * 32 + lane;
        const bool valid = r < n;
        const uint32_t d = valid ? pos[r] : 0u;
        const uint64_t lastr = g * 32 + 31 < n ? g * 32 + 31 : n - 1;
        const uint32_t d0 = __shfl_sync(0xffffffffu, d, 0);
        const uint32_t dend = pos[lastr + 1];
        const uint32_t sh = (uint32_t)((reinterpret_cast<uintptr_t>(out) + d0) & 15u), total = dend - d0;
        const bool staged = (uint64_t)sh + total <= JW_STAGE;
        if (valid) {
            uint8_t* q = staged ? stage + sh + (d - d0) : out + d;
            *q++ = r == 0 ? first_byte : ',';
            *q++ = '{';
            for (int k = 0; k < ncols; k++) {
                const JsonCol c = cols[k];
                for (uint32_t j = 0; j < c.key_len; j++) q[j] = keys[c.key + j];
                q += c.key_len;
                const uint32_t s = c.off[r], l = c.off[r + 1] - s;
                const uint8_t* p = c.data + s;
                if (json_plain(p, l)) { for (uint32_t j = 0; j < l; j++) q[j] = p[j]; q += l; }
                else q += json_escape(p, l, q);
                *q++ = '"';
            }
            q[0] = '}'; q[1] = '\n';
        }
        if (staged) {
            __syncwarp();
            uint8_t* gb = out + d0 - sh;
            for (uint32_t x = lane * 16; x < sh + total; x += 32 * 16) {
                if (x >= sh && x + 16 <= sh + total) *reinterpret_cast<uint4*>(gb + x) = *reinterpret_cast<const uint4*>(stage + x);
                else for (uint32_t y = x; y < x + 16; y++) if (y >= sh && y < sh + total) gb[y] = stage[y];
            }
            __syncwarp();
        }
    }
}

__global__ void json_value_bytes_kernel(const JsonCol* cols, int ncols, uint64_t n, unsigned long long* out) {
    unsigned long long s = 0;
    for (int k = 0; k < ncols; k++) s += cols[k].off[n] - cols[k].off[0];
    *out = s;
}

Buf table_to_json(Ctx* c, const Table& t, bool first, bool last, uint64_t room, uint64_t* nbytes) {
    const uint64_t n = (uint64_t)t.nrows;
    if (n == 0) {
        std::string s = std::string(first ? "[" : "") + (last ? "]" : "");
        *nbytes = s.size();
        if (*nbytes > room) return nullptr;
        Buf out = dev_alloc(c, 16);
        if (!s.empty()) CPB_CUDA(cudaMemcpyAsync(out->p, s.data(), s.size(), cudaMemcpyHostToDevice, c->stream));
        sync_stream(c);  // s is pageable stack memory
        return out;
    }
    const int ncols = (int)t.cols.size();
    std::vector<int> order(ncols);
    std::iota(order.begin(), order.end(), 0);
    std::sort(order.begin(), order.end(), [&](int a, int b) { return t.cols[a].name < t.cols[b].name; });  // bytewise
    // metadata blob: JsonCol[ncols] then the key prefixes
    std::vector<JsonCol> hc(ncols);
    std::vector<uint8_t> keys;
    uint64_t row_const = 4;  // '['/',' '{' '}' '\n'
    for (int k = 0; k < ncols; k++) {
        const Column& col = t.cols[order[k]];
        std::vector<uint8_t> e(col.name.size() * 6 + 2);
        const uint64_t m = json_escape((const uint8_t*)col.name.data(), col.name.size(), e.data());
        const uint32_t at = (uint32_t)keys.size();
        if (k) keys.push_back(',');
        keys.push_back('"');
        keys.insert(keys.end(), e.begin(), e.begin() + m);
        keys.push_back('"'); keys.push_back(':'); keys.push_back('"');
        hc[k] = JsonCol{col.off(), col.bytes(), at, (uint32_t)(keys.size() - at)};
        row_const += hc[k].key_len + 1;  // + the closing quote of the value
    }
    const uint32_t keys_at = (uint32_t)(ncols * sizeof(JsonCol)), meta_bytes = keys_at + (uint32_t)keys.size();
    std::vector<uint8_t> meta(meta_bytes);
    if (ncols) memcpy(meta.data(), hc.data(), keys_at);
    if (!keys.empty()) memcpy(meta.data() + keys_at, keys.data(), keys.size());
    Buf md = dev_alloc(c, meta_bytes);
    if (meta_bytes) CPB_CUDA(cudaMemcpyAsync(md->p, meta.data(), meta_bytes, cudaMemcpyHostToDevice, c->stream));
    const JsonCol* dcols = md->as<JsonCol>();
    const uint8_t* dkeys = md->as<uint8_t>() + keys_at;

    Buf len = dev_alloc(c, (n + 1) * 4), tot = dev_alloc(c, 16);
    {
        KernelTimer kt(c, "json_row_len", n * 4 * (ncols + 1));
        json_row_len_kernel<<<nblk(n, 256), 256, 0, c->stream>>>(dcols, ncols, row_const, n, len->as<uint32_t>());
        CPB_CUDA(cudaGetLastError());
    }
    json_value_bytes_kernel<<<1, 1, 0, c->stream>>>(dcols, ncols, n, tot->as<unsigned long long>() + 1);
    CPB_CUDA(cudaGetLastError());
    exclusive_scan_u32(c, len->as<uint32_t>(), len->as<uint32_t>(), n, tot->as<uint64_t>());
    const std::vector<uint64_t> ht = read_back<uint64_t>(c, tot->p, 2);
    const uint64_t body = ht[0], value_bytes = ht[1];
    if (body >= 0xffffffffull) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "ToJSON output exceeds 4 GiB; write in smaller batches"};
    *nbytes = body + (last ? 1 : 0);
    if (*nbytes > room) return nullptr;
    Buf out = dev_alloc(c, body + 1 + 16);
    {
        KernelTimer kt(c, "json_write", value_bytes + n * 4 * (ncols + 1) + body);
        const bool meta_smem = meta_bytes <= JW_META_SMEM;
        const uint32_t smem = JW_STAGE_BYTES + (meta_smem ? meta_bytes : 0);
        CPB_CUDA(cudaFuncSetAttribute(json_write_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, JW_STAGE_BYTES + JW_META_SMEM));
        const uint32_t blocks = (uint32_t)std::min<uint64_t>((n + JW_WARPS * 32 - 1) / (JW_WARPS * 32), (uint64_t)c->sm_count * 8);
        json_write_kernel<<<blocks, JW_WARPS * 32, smem, c->stream>>>(dcols, dkeys, ncols, meta_bytes, meta_smem, first ? '[' : ',', n,
                                                                      len->as<uint32_t>(), out->as<uint8_t>());
        CPB_CUDA(cudaGetLastError());
    }
    if (last) CPB_CUDA(cudaMemsetAsync(out->as<uint8_t>() + body, ']', 1, c->stream));
    return out;
}

}  // namespace cpb
