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
// The row type JsonRows through the row serialiser driver of rowwrite.cuh (json_row_len -> exclusive_scan_u32 ->
// json_write).  The columns are a keyed-column table (rowwrite.cuh) whose names are the key prefixes, so there is no
// column limit.
#include <algorithm>
#include <numeric>

#include "core.hpp"
#include "rowwrite.cuh"

namespace cpb {

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

// A JSON row repeats every key, so it is several times longer than the CSV line of the same row (about 120-150 B for a
// joined orders x customers row): the stage holds 32 rows of up to 190 B, where ToCsv's 4 KB would send most such
// groups down the direct path.
constexpr uint32_t JW_STAGE = 6144;
// a row: first_byte ('[' or ',') for row 0, else ','; then the pairs between braces, and '\n'
struct JsonRows : KeyedRows {
    uint8_t first_byte;
    __device__ uint64_t len(uint64_t r) const {
        uint64_t total = row_const;
        for (int k = 0; k < ncols; k++) {
            const uint32_t* off = cols[k].off;
            const uint32_t s = off[r], l = off[r + 1] - s;
            const uint8_t* p = cols[k].data + s;
            total += json_plain(p, l) ? l : json_escape(p, l, nullptr);
        }
        return total;
    }
    __device__ void write(uint64_t r, uint8_t* q, const Tables& t) const {
        *q++ = r == 0 ? first_byte : ',';
        *q++ = '{';
        for (int k = 0; k < ncols; k++) {
            const KeyedCol c = t.cols[k];
            for (uint32_t j = 0; j < c.key_len; j++) q[j] = t.keys[c.key + j];
            q += c.key_len;
            const uint32_t s = c.off[r], l = c.off[r + 1] - s;
            const uint8_t* p = c.data + s;
            if (json_plain(p, l)) { for (uint32_t j = 0; j < l; j++) q[j] = p[j]; q += l; }
            else q += json_escape(p, l, q);
            *q++ = '"';
        }
        q[0] = '}'; q[1] = '\n';
    }
};

// ---- the keyed-column table of rowwrite.cuh (ToJSON and Index.WriteTo)
__global__ void keyed_value_bytes_kernel(const KeyedCol* cols, int ncols, uint64_t n, unsigned long long* out) {
    unsigned long long s = 0;
    for (int k = 0; k < ncols; k++) s += cols[k].off[n] - cols[k].off[0];
    *out = s;
}

void keyed_value_bytes(Ctx* c, const KeyedCols& kc, uint64_t n, unsigned long long* out) {
    keyed_value_bytes_kernel<<<1, 1, 0, c->stream>>>(kc.md->as<KeyedCol>(), kc.ncols, n, out);
    CPB_CUDA(cudaGetLastError());
}

KeyedCols keyed_cols(Ctx* c, const Table& t, uint64_t lo, void (*enc)(std::string& keys, const std::string& name, int k)) {
    KeyedCols kc;
    kc.ncols = (int)t.cols.size();
    std::vector<int> order(kc.ncols);
    std::iota(order.begin(), order.end(), 0);
    std::sort(order.begin(), order.end(), [&](int a, int b) { return t.cols[a].name < t.cols[b].name; });  // bytewise
    std::vector<KeyedCol> hc(kc.ncols);
    std::string keys;
    for (int k = 0; k < kc.ncols; k++) {
        const Column& col = t.cols[order[k]];
        const uint32_t at = (uint32_t)keys.size();
        enc(keys, col.name, k);
        hc[k] = KeyedCol{col.off() + lo, col.bytes(), at, (uint32_t)(keys.size() - at)};
    }
    kc.keys_at = (uint32_t)(kc.ncols * sizeof(KeyedCol));
    kc.meta_bytes = kc.keys_at + (uint32_t)keys.size();
    std::string meta(reinterpret_cast<const char*>(hc.data()), kc.keys_at);
    meta += keys;
    kc.md = dev_alloc(c, kc.meta_bytes);
    // (pageable source: the call returns once the bytes are staged, so meta may go away)
    if (kc.meta_bytes) CPB_CUDA(cudaMemcpyAsync(kc.md->p, meta.data(), kc.meta_bytes, cudaMemcpyHostToDevice, c->stream));
    return kc;
}

// a column's key prefix: [","] '"' enc(name) '"' ':' '"'
static void json_key(std::string& keys, const std::string& name, int k) {
    std::vector<uint8_t> e(name.size() * 6 + 2);
    const uint64_t m = json_escape((const uint8_t*)name.data(), name.size(), e.data());
    if (k) keys += ',';
    keys += '"';
    keys.append((const char*)e.data(), m);
    keys += "\":\"";
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
    const KeyedCols kc = keyed_cols(c, t, 0, json_key);
    const int ncols = kc.ncols;
    // '['/',' '{' '}' '\n', the key prefixes and the closing quote of every value
    const JsonRows rows{KeyedRows(kc, 4 + (kc.meta_bytes - kc.keys_at) + ncols), (uint8_t)(first ? '[' : ',')};
    Buf len = dev_alloc(c, (n + 1) * 4), tot = dev_alloc(c, 16);
    row_lengths(c, rows, n, len->as<uint32_t>(), "json_row_len", n * 4 * (ncols + 1));
    keyed_value_bytes(c, kc, n, tot->as<unsigned long long>() + 1);
    const std::vector<uint64_t> ht = row_offsets(c, len->as<uint32_t>(), n, tot->as<uint64_t>(), 2, MAX_BODY - 1,
                                                 "ToJSON output exceeds 4 GiB; write in smaller batches");
    const uint64_t body = ht[0], value_bytes = ht[1];
    *nbytes = body + (last ? 1 : 0);
    if (*nbytes > room) return nullptr;
    Buf out = dev_alloc(c, body + 1 + 16);
    row_write<JW_STAGE>(c, rows, n, len->as<uint32_t>(), out->as<uint8_t>(), "json_write", value_bytes + n * 4 * (ncols + 1) + body, 8);
    if (last) CPB_CUDA(cudaMemsetAsync(out->as<uint8_t>() + body, ']', 1, c->stream));
    return out;
}

}  // namespace cpb
