// gob.cu — Index.WriteTo / LoadIndex (csvplus.go:655-705): the index file is an encoding/gob stream of two values sent
// by one encoder, `columns []string` (the key columns) then `rows []Row` (Row = map[string]string).  Every rule of the
// format the project relies on lives in this file.
//
//   stream   messages: uint(byte count of the rest) int(type id) ...; a negative id -t defines type t (a wireType struct
//            value follows), a positive id is a value of that type.
//   uint     x < 128: one byte; else one byte holding the negated byte count (0xFF = 1, 0xFE = 2, ...) then x big-endian
//            in the fewest bytes (256 -> FE 01 00).  int: x >= 0 -> uint(x << 1), x < 0 -> uint(^x << 1 | 1).
//   string   uint(len) bytes.   struct: (uint field delta from -1, value) pairs, zero fields omitted, 0 ends it.
//   top-level non-struct value: a 0 byte (singleton field delta) first.  slice: uint(count) then every element.
//   map      uint(count) then key / value pairs (Go's random iteration order).
//   ids      built-ins: string 6; user types from 65 in a fresh process.  wireType = {ArrayT 0, SliceT 1, StructT 2,
//            MapT 3, ...}; CommonType = {Name, Id}; sliceType = {CommonType, Elem}; mapType = {CommonType, Key, Elem}.
//
// What WriteTo writes (gob's encoder sends a type before its first value, the outer type's definition before its
// element's; ids in registration order, the element of []Row registered first):
//   def []string (65)   value of 65: the key columns
//   def []Row (67)      def Row = "Row" (66) map[string]string      value of 67: 0 uint(nrows) then per row
//   uint(k) and the k pairs uint(len name) name uint(len value) value, names in bytewise order (deterministic; the
//   reference's own files have them in random order).
// The rows of the index are taken in its stored order (sorted_table).  A message of 8 GiB or more (encoding/gob's tooBig
// on 64-bit), or a rows slice above 8 GiB of Go maps, is refused before anything is written, as gob's encoder refuses it.
//
// Encode: the row type GobRows through the row serialiser driver of rowwrite.cuh (gob_row_len, which also sums the
// lengths exactly -> exclusive_scan_u32 -> gob_write) over a keyed-column table whose names are uint(len name) name.
// The prefix (type definitions, columns, rows header) is built here on the host; the rows are written in row-range
// batches (each < 4 GiB) by cpb_index_gob_into.
//
// Decode: the host parses the type definitions (any ids, any order), the columns value, the rows message header and the
// first row (k and the column set).  The rows body is uploaded once.  A row has no marker and its start depends on every
// length before it, so the row starts are recovered in parallel, window by window: a window is at most GOB_WINDOW bytes
// of the body starting at a known row start (the first at 0), positions inside it are 32-bit offsets, and rows are
// parsed against the whole body with 64-bit positions.  In each window:
//   gob_cand    position x is a candidate if a whole row parses there: uint(k), then k pairs whose keys are the k
//               column names, each once, all inside the body.  Most bytes fail at the first byte.
//   compact     the candidates in position order (scan_flags / compact_flags); succ(x) = candidate index of the end of
//               x's row, END when that end is at or past the window's end, DEAD when it is not a candidate.
//   exits       candidates in chunks of GOB_CHUNK; one thread per chunk walks its candidates last to first: since
//               succ(x) > x, exit(x) (the first node past the chunk on x's path) is succ(x) or exit(succ(x)).
//   stitch      one thread follows exits chunk to chunk from the window's first row and records where the path enters
//               each chunk; then one thread per entered chunk walks forward from its entry and marks the rows.  The row
//               whose successor is END gives the start of the next window.
// True rows tile the body, so the path from a row start visits true rows only, whatever bytes the values hold.  A path
// that does not end at END, or a row count other than nrows, is an error: a corrupt file, or rows whose column sets
// differ (which a device table cannot hold).  gob_extract writes each row's value lengths and 64-bit starts,
// gob_sum_kernel gives every column's exact total (a column holds less than 4 GiB), the offsets are scanned per column,
// and gob_copy gathers the bytes.
#include <algorithm>

#include "core.hpp"
#include "rowwrite.cuh"
#include "util.cuh"

namespace cpb {

constexpr uint64_t GOB_TOO_BIG = 8ull << 30;  // encoding/gob tooBig on 64-bit: messages (and slice bytes) must stay below
constexpr int64_t GOB_STRING = 6;             // built-in type id of string
constexpr int64_t GOB_ID_STRINGS = 65, GOB_ID_ROW = 66, GOB_ID_ROWS = 67;
constexpr uint64_t GOB_MAP_SIZE = 8;          // bytes of one Go map value: gob's decoder bounds count * size by tooBig
constexpr uint32_t GOB_MAXCOLS = 256;         // columns of a row the decoder tracks (four 64-bit masks)
constexpr uint32_t GOB_CHUNK = 1024;          // candidates per chunk of the exit walk
constexpr uint32_t GOB_DEAD = 0xffffffffu;
constexpr uint64_t GOB_WINDOW = 256ull << 20;  // body bytes per decode window: its per-byte flags and their scan take 8 B per byte

__host__ __device__ inline uint32_t gob_uint_len(uint64_t x) {
    if (x < 128) return 1;
    uint32_t n = 1;
    for (; x; x >>= 8) n++;
    return n;
}
__host__ __device__ inline uint32_t gob_put_uint(uint8_t* d, uint64_t x) {
    if (x < 128) { d[0] = (uint8_t)x; return 1; }
    const uint32_t n = gob_uint_len(x) - 1;
    d[0] = (uint8_t)(256u - n);
    for (uint32_t i = 0; i < n; i++) d[1 + i] = (uint8_t)(x >> (8 * (n - 1 - i)));
    return n + 1;
}
// the uint at p (avail bytes readable) -> *x; its width, 0 when it is malformed (more than 8 value bytes) or cut off.
// Non-minimal encodings are accepted, as gob's decoder accepts them.
__host__ __device__ inline uint32_t gob_get_uint(const uint8_t* p, uint64_t avail, uint64_t* x) {
    if (avail == 0) return 0;
    const uint8_t b = p[0];
    if (b < 128) { *x = b; return 1; }
    const uint32_t n = 256u - b;
    if (n > 8 || avail < 1ull + n) return 0;
    uint64_t v = 0;
    for (uint32_t i = 0; i < n; i++) v = (v << 8) | p[1 + i];
    *x = v;
    return n + 1;
}

// ------------------------------------------------------------------ host-side encoding (prefix)
static void put_uint(std::string& s, uint64_t x) { uint8_t b[9]; s.append((const char*)b, gob_put_uint(b, x)); }
static void put_int(std::string& s, int64_t x) { put_uint(s, x < 0 ? ((uint64_t)~x << 1) | 1u : (uint64_t)x << 1); }
static void put_str(std::string& s, const std::string& v) { put_uint(s, v.size()); s += v; }
static void put_msg(std::string& out, const std::string& body) { put_uint(out, body.size()); out += body; }
static std::string common_type(const std::string& name, int64_t id) {  // CommonType{Name, Id}: an empty Name is omitted
    std::string s;
    if (!name.empty()) { put_uint(s, 1); put_str(s, name); put_uint(s, 1); }
    else put_uint(s, 2);
    put_int(s, id);
    s += '\0';
    return s;
}
static std::string slice_def(int64_t id, int64_t elem) {  // -id, wireType{SliceT: sliceType{CommonType{"", id}, elem}}
    std::string b;
    put_int(b, -id);
    put_uint(b, 2);
    put_uint(b, 1); b += common_type("", id);
    put_uint(b, 1); put_int(b, elem);
    b += '\0'; b += '\0';
    return b;
}
static std::string map_def(const std::string& name, int64_t id, int64_t key, int64_t elem) {  // wireType{MapT: mapType{...}}
    std::string b;
    put_int(b, -id);
    put_uint(b, 4);
    put_uint(b, 1); b += common_type(name, id);
    put_uint(b, 1); put_int(b, key);
    put_uint(b, 1); put_int(b, elem);
    b += '\0'; b += '\0';
    return b;
}

// ------------------------------------------------------------------ encode kernels
// a row: uint(k), then every pair uint(len name) name (pre-encoded) uint(len value) value
struct GobRows : KeyedRows {
    __device__ uint64_t len(uint64_t r) const {
        uint64_t total = row_const;
        for (int k = 0; k < ncols; k++) {
            const uint32_t* off = cols[k].off;
            const uint32_t l = off[r + 1] - off[r];
            total += gob_uint_len(l) + l;
        }
        return total;
    }
    __device__ void write(uint64_t r, uint8_t* q, const Tables& t) const {
        q += gob_put_uint(q, (uint64_t)ncols);
        for (int k = 0; k < ncols; k++) {
            const KeyedCol c = t.cols[k];
            for (uint32_t j = 0; j < c.key_len; j++) q[j] = t.keys[c.key + j];
            q += c.key_len;
            const uint32_t s = c.off[r], l = c.off[r + 1] - s;
            q += gob_put_uint(q, l);
            const uint8_t* p = c.data + s;
            for (uint32_t j = 0; j < l; j++) q[j] = p[j];
            q += l;
        }
    }
};
// out[y] += the exact 64-bit sum of v[y * stride + i], i < n (blockIdx.y = y)
__global__ void gob_sum_kernel(const uint32_t* __restrict__ v, uint64_t n, uint64_t stride, unsigned long long* out) {
    const uint32_t* p = v + (uint64_t)blockIdx.y * stride;
    uint64_t s = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) s += p[i];
    s = warp_sum_u64(s);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(out + blockIdx.y, (unsigned long long)s);
}

// the keyed columns of rows [lo, hi) of the index's stored rows
struct GobMeta {
    std::shared_ptr<Table> t;  // the stored rows, kept alive while the kernels read them
    KeyedCols kc;
};
static GobMeta gob_meta(Ctx* c, Index& ix, uint64_t lo) {
    GobMeta m;
    m.t = sorted_table(c, ix);
    m.kc = keyed_cols(c, *m.t, lo, [](std::string& keys, const std::string& name, int) { put_str(keys, name); });
    return m;
}
// uint(k) + every pre-encoded name: the bytes of a row besides its values
static GobRows gob_row_type(const KeyedCols& kc) { return GobRows{KeyedRows(kc, gob_uint_len((uint64_t)kc.ncols) + (kc.meta_bytes - kc.keys_at))}; }

// row lengths of rows [lo, lo + n) into len (n + 1 entries, not yet scanned); *out = {exact total bytes, value bytes}.
// The 32-bit scan of the lengths is run only when that total is below 4 GiB, so no partial sum of it can wrap.
static void gob_lengths(Ctx* c, const GobMeta& m, uint64_t n, Buf& len, uint64_t out[2]) {
    len = dev_alloc(c, (n + 1) * 4);
    Buf tot = dev_alloc(c, 16);
    CPB_CUDA(cudaMemsetAsync(tot->p, 0, 16, c->stream));
    row_lengths<true>(c, gob_row_type(m.kc), n, len->as<uint32_t>(), "gob_row_len", n * 4 * (m.kc.ncols + 1), tot->as<unsigned long long>());
    keyed_value_bytes(c, m.kc, n, tot->as<unsigned long long>() + 1);
    const std::vector<uint64_t> h = read_back<uint64_t>(c, tot->p, 2);
    out[0] = h[0]; out[1] = h[1];
}

std::string gob_prefix(Ctx* c, Index& ix, uint64_t* total) {
    const uint64_t n = (uint64_t)ix.nrows;
    GobMeta m = gob_meta(c, ix, 0);
    Buf len;
    uint64_t t[2];
    gob_lengths(c, m, n, len, t);
    // the rows message: int(67) 0 uint(nrows) rows
    std::string head;
    put_int(head, GOB_ID_ROWS); head += '\0'; put_uint(head, n);
    const uint64_t body = head.size() + t[0];
    if (body >= GOB_TOO_BIG || n * GOB_MAP_SIZE > GOB_TOO_BIG)
        throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "gob: encoder: message too big"};
    std::string out;
    put_msg(out, slice_def(GOB_ID_STRINGS, GOB_STRING));
    std::string cv;
    put_int(cv, GOB_ID_STRINGS); cv += '\0'; put_uint(cv, ix.key_cols.size());
    for (auto& k : ix.key_cols) put_str(cv, k);
    put_msg(out, cv);
    put_msg(out, slice_def(GOB_ID_ROWS, GOB_ID_ROW));
    put_msg(out, map_def("Row", GOB_ID_ROW, GOB_STRING, GOB_STRING));
    put_uint(out, body);
    out += head;
    *total = out.size() + t[0];
    return out;
}

Buf gob_rows(Ctx* c, Index& ix, uint64_t lo, uint64_t hi, uint64_t room, uint64_t* nbytes) {
    const uint64_t n = hi - lo;
    GobMeta m = gob_meta(c, ix, lo);
    Buf len;
    uint64_t t[2];
    gob_lengths(c, m, n, len, t);
    check_body(t[0], n, MAX_BODY - 1, "index rows batch exceeds 4 GiB; write in smaller batches");
    *nbytes = t[0];
    if (*nbytes > room) return nullptr;
    Buf tot = dev_alloc(c, 8);
    exclusive_scan_u32(c, len->as<uint32_t>(), len->as<uint32_t>(), n, tot->as<uint64_t>());  // every partial sum < 4 GiB
    Buf out = dev_alloc(c, t[0] + 16);
    row_write<4096>(c, gob_row_type(m.kc), n, len->as<uint32_t>(), out->as<uint8_t>(), "gob_write", t[1] + n * 4 * (m.kc.ncols + 1) + t[0], 8);
    return out;
}

// ------------------------------------------------------------------ decode kernels
struct GobKeys {  // the column names of the rows, bytewise sorted: name j = blob[off[j], off[j + 1])
    const uint8_t* blob; const uint32_t* off; uint32_t k;
};

// The row that parses at x of the body b[0, L): its end, or 0 when no row parses there (a row is never empty, so its
// end is > x >= 0).  With lens / vpos given, the length and start of the value of column j go to lens[j * stride + r] /
// vpos[j * stride + r].
__device__ __forceinline__ uint64_t gob_row_end(const uint8_t* __restrict__ b, uint64_t L, uint64_t x, const GobKeys& ks,
                                                uint32_t* lens, uint64_t* vpos, uint64_t stride, uint64_t r) {
    uint64_t v;
    uint32_t w = gob_get_uint(b + x, L - x, &v);
    if (w == 0 || v != ks.k) return 0;
    uint64_t p = x + w;
    uint64_t m0 = 0, m1 = 0, m2 = 0, m3 = 0;  // columns seen in this row
    for (uint32_t i = 0; i < ks.k; i++) {
        w = gob_get_uint(b + p, L - p, &v);
        if (w == 0 || v > L - p - w) return 0;
        const uint32_t kl = (uint32_t)v;
        const uint64_t ks0 = p + w;
        uint32_t j = 0;
        for (; j < ks.k; j++) {  // the name: one of the k column names
            const uint32_t o = ks.off[j];
            if (ks.off[j + 1] - o != kl) continue;
            uint32_t q = 0;
            while (q < kl && ks.blob[o + q] == b[ks0 + q]) q++;
            if (q == kl) break;
        }
        if (j == ks.k) return 0;
        const uint64_t bit = 1ull << (j & 63);
        const uint32_t q = j >> 6;
        const uint64_t m = q == 0 ? m0 : q == 1 ? m1 : q == 2 ? m2 : m3;
        if (m & bit) return 0;  // a name twice
        if (q == 0) m0 |= bit; else if (q == 1) m1 |= bit; else if (q == 2) m2 |= bit; else m3 |= bit;
        p = ks0 + kl;
        w = gob_get_uint(b + p, L - p, &v);
        if (w == 0 || v > L - p - w || v > 0xffffffffull) return 0;
        if (lens) { lens[j * stride + r] = (uint32_t)v; vpos[j * stride + r] = p + w; }
        p += w + v;
    }
    return p;
}

// The body is decoded in windows [s, s + w) of at most GOB_WINDOW bytes, each starting at a known row start; positions
// inside a window are 32-bit offsets from s, rows are parsed against the whole body.
__global__ void gob_cand_kernel(const uint8_t* __restrict__ b, uint64_t L, uint64_t s, uint32_t w, GobKeys ks, uint32_t* flag) {
    for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < w; x += (uint64_t)gridDim.x * blockDim.x)
        flag[x] = gob_row_end(b, L, s + x, ks, nullptr, nullptr, 0, 0) != 0 ? 1u : 0u;
}
// exit[i] = the first node past i's chunk on i's path (a later candidate, END or DEAD)
__global__ void gob_exit_kernel(const uint32_t* __restrict__ succ, uint64_t C, uint32_t* exit) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t lo = t * GOB_CHUNK;
    if (lo >= C) return;
    const uint64_t hi = lo + GOB_CHUNK < C ? lo + GOB_CHUNK : C;
    for (uint64_t i = hi; i-- > lo;) {
        const uint32_t s = succ[i];
        exit[i] = (s == GOB_DEAD || s >= hi) ? s : exit[s];
    }
}
// from candidate 0 (the window's first row, at offset 0), chunk to chunk: entry[chunk] = the candidate the path enters
// it at; *ok = 1 when the path ends at END
__global__ void gob_stitch_kernel(const uint32_t* __restrict__ cpos, const uint32_t* __restrict__ exit, uint64_t C, uint32_t* entry,
                                  unsigned long long* ok) {
    *ok = 0;
    if (C == 0 || cpos[0] != 0) return;
    uint64_t cur = 0;
    while (cur < C) {
        entry[cur / GOB_CHUNK] = (uint32_t)cur;
        cur = exit[cur];
    }
    *ok = cur == C ? 1u : 0u;
}
// marks the rows on the path; the last one (its successor is END) writes where the next window starts
__global__ void gob_mark_kernel(const uint8_t* __restrict__ b, uint64_t L, uint64_t s, GobKeys ks, const uint32_t* __restrict__ cpos,
                                const uint32_t* __restrict__ succ, const uint32_t* __restrict__ entry, uint64_t C, uint32_t* mark,
                                unsigned long long* next) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t lo = t * GOB_CHUNK;
    if (lo >= C || entry[t] == GOB_DEAD) return;
    const uint64_t hi = lo + GOB_CHUNK < C ? lo + GOB_CHUNK : C;
    for (uint64_t x = entry[t]; x < hi; x = succ[x]) {
        mark[x] = 1u;
        if (succ[x] == C) *next = gob_row_end(b, L, s + cpos[x], ks, nullptr, nullptr, 0, 0);
    }
}
struct GobOut { uint32_t* off; uint8_t* data; };

// ------------------------------------------------------------------ decode, host side
[[noreturn]] static void gob_fail(const std::string& msg) { throw DataError{CPB_E_GOB, -1, 0, false, msg}; }

struct GobReader {
    const uint8_t* p; uint64_t n, i = 0;
    uint64_t end = 0;  // end of the current message
    uint64_t get_uint() {
        uint64_t x;
        const uint32_t w = gob_get_uint(p + i, end - i, &x);
        if (w == 0) gob_fail("gob: corrupted data: bad uint");
        i += w;
        return x;
    }
    int64_t get_int() { const uint64_t u = get_uint(); return (u & 1) ? (int64_t)~(u >> 1) : (int64_t)(u >> 1); }
    std::string get_str() {
        const uint64_t l = get_uint();
        if (l > end - i) gob_fail("gob: corrupted data: string length beyond the message");
        std::string s((const char*)p + i, (size_t)l);
        i += l;
        return s;
    }
    // the next message: false at the end of the input (io.EOF when nothing of it was read), its bytes must be there
    void next_message() {
        if (i == n) gob_fail("EOF");
        uint64_t len;
        const uint32_t w = gob_get_uint(p + i, n - i, &len);
        if (w == 0) gob_fail(p[i] >= 128 && 256u - p[i] > 8 ? "gob: invalid message length" : "unexpected EOF");
        if (len >= GOB_TOO_BIG) gob_fail("gob: invalid message length");
        i += w;
        if (len > n - i) gob_fail("unexpected EOF");
        end = i + len;
    }
};

struct GobType { int kind = -1; int64_t elem = 0, key = 0; };  // kind: wireType field (1 SliceT, 3 MapT, ...)

// a CommonType struct; only its presence matters here
static void skip_common(GobReader& r) {
    for (int64_t f = -1;;) {
        const uint64_t d = r.get_uint();
        if (d == 0) return;
        f += (int64_t)d;
        if (f == 0) r.get_str();
        else if (f == 1) r.get_int();
        else gob_fail("gob: corrupted data: CommonType field");
    }
}
// reads type definitions until a value message; returns its type id with the reader at its value
static int64_t gob_value(GobReader& r, std::map<int64_t, GobType>& types) {
    for (;;) {
        r.next_message();
        const int64_t id = r.get_int();
        if (id >= 0) return id;
        GobType t;
        const uint64_t d = r.get_uint();  // the one field of wireType this definition sets
        if (d == 0) gob_fail("gob: corrupted data: empty wireType");
        t.kind = (int)d - 1;
        if (t.kind == 1 || t.kind == 3) {  // sliceType{CommonType, Elem} / mapType{CommonType, Key, Elem}
            for (int64_t f = -1;;) {
                const uint64_t e = r.get_uint();
                if (e == 0) break;
                f += (int64_t)e;
                if (f == 0) skip_common(r);
                else if (t.kind == 1 && f == 1) t.elem = r.get_int();
                else if (t.kind == 3 && f == 1) t.key = r.get_int();
                else if (t.kind == 3 && f == 2) t.elem = r.get_int();
                else gob_fail("gob: corrupted data: type field");
            }
        }
        types[-id] = t;
        r.i = r.end;  // anything else of the definition is not needed
    }
}
static void gob_singleton(GobReader& r) {
    if (r.get_uint() != 0) gob_fail("gob: decode: corrupted data: non-zero delta for singleton");
}

std::shared_ptr<Index> gob_load(Ctx* c, const uint8_t* bytes, uint64_t nbytes, std::vector<std::string>* key_cols) {
    GobReader r{bytes, nbytes};
    std::map<int64_t, GobType> types;
    auto is = [&](int64_t id, int kind) { auto it = types.find(id); return it != types.end() && it->second.kind == kind ? &it->second : nullptr; };
    // columns []string
    int64_t id = gob_value(r, types);
    const GobType* ct = is(id, 1);
    if (!ct || ct->elem != GOB_STRING) gob_fail("gob: type mismatch: the first value of an index file is not a []string");
    gob_singleton(r);
    const uint64_t ncols = r.get_uint();
    if (ncols > r.end - r.i) gob_fail("gob: corrupted data: column count beyond the message");
    for (uint64_t k = 0; k < ncols; k++) key_cols->push_back(r.get_str());
    // rows []map[string]string
    id = gob_value(r, types);
    const GobType* rt = is(id, 1);
    const GobType* mt = rt ? is(rt->elem, 3) : nullptr;
    if (!mt || mt->key != GOB_STRING || mt->elem != GOB_STRING)
        gob_fail("gob: type mismatch: the second value of an index file is not a []map[string]string");
    gob_singleton(r);
    const uint64_t nrows = r.get_uint();
    const uint64_t b0 = r.i, L = r.end - r.i;
    if (nrows > L || nrows * GOB_MAP_SIZE > GOB_TOO_BIG) gob_fail("gob: corrupted data: row count beyond the message");
    if (nrows > 0xfffffffeull) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "an index holds at most 2^32-2 rows"};
    if ((int)key_cols->size() > MAXKEYS) throw ArgError{CPB_ERR_UNSUPPORTED, "more than 16 index key columns"};
    // the first row: k and the column names
    std::vector<std::string> names;
    if (nrows) {
        const uint64_t k = r.get_uint();
        if (k > GOB_MAXCOLS) throw ArgError{CPB_ERR_UNSUPPORTED, "index rows with more than 256 columns"};
        for (uint64_t j = 0; j < k; j++) { names.push_back(r.get_str()); r.get_str(); }
        std::sort(names.begin(), names.end());
        if (std::adjacent_find(names.begin(), names.end()) != names.end()) gob_fail("gob: corrupted data: a column twice in a row");
    } else {
        if (L) gob_fail("gob: corrupted data: extra data after the rows");
        names = *key_cols;  // an empty index: a table of its key columns
        std::sort(names.begin(), names.end());
        names.erase(std::unique(names.begin(), names.end()), names.end());
    }
    for (auto& kc : *key_cols)
        if (!std::binary_search(names.begin(), names.end(), kc)) gob_fail("index file: key column " + go_quote(kc) + " is not a column of the rows");
    const uint32_t k = (uint32_t)names.size();
    auto t = std::make_shared<Table>(); t->ctx = c; t->first_line = 0;
    std::vector<GobOut> houts(k);
    for (uint32_t j = 0; j < k; j++) { Column col; col.name = names[j]; t->cols.push_back(col); }
    uint64_t R = 0;
    if (nrows) {
        // names and body on the device
        std::vector<uint32_t> koff(k + 1, 0);
        std::string blob;
        for (uint32_t j = 0; j < k; j++) { blob += names[j]; koff[j + 1] = (uint32_t)blob.size(); }
        Buf kb = dev_alloc(c, blob.size() + 16), ko = dev_alloc(c, (k + 1) * 4);
        CPB_CUDA(cudaMemcpyAsync(kb->p, blob.data(), blob.size(), cudaMemcpyHostToDevice, c->stream));
        CPB_CUDA(cudaMemcpyAsync(ko->p, koff.data(), (k + 1) * 4, cudaMemcpyHostToDevice, c->stream));
        const GobKeys ks{kb->as<uint8_t>(), ko->as<uint32_t>(), k};
        Buf body = dev_alloc(c, L + 16);
        {
            KernelTimer kt(c, "h2d_input", L, 0);
            CPB_CUDA(cudaMemcpyAsync(body->p, bytes + b0, L, cudaMemcpyHostToDevice, c->stream));
        }
        const uint8_t* b = body->as<uint8_t>();
        // 1.-5. per window: candidates (compacted in position order, cpos[C] = w), successors, chunk exits, stitch from
        // the window's first row, the rows on the path; the row that ends at or past the window's end starts the next
        Buf start = dev_alloc(c, nrows * 8 + 8);
        const uint64_t W = std::min<uint64_t>(L, GOB_WINDOW);
        Buf flag = dev_alloc(c, W * 4 + 4), st = dev_alloc(c, 16);
        for (uint64_t s = 0; s < L;) {
            const uint32_t w = (uint32_t)std::min<uint64_t>(W, L - s);
            {
                KernelTimer kt(c, "gob_cand", (uint64_t)w * 5);
                gob_cand_kernel<<<(uint32_t)std::min<uint64_t>(nblk(w, 256), (uint64_t)c->sm_count * 32), 256, 0, c->stream>>>(b, L, s, w, ks,
                                                                                                                         flag->as<uint32_t>());
                CPB_CUDA(cudaGetLastError());
            }
            const FlagScan cs = scan_flags(c, flag->as<uint32_t>(), w);
            const uint64_t C = cs.count;
            Buf cpos = dev_alloc(c, (C + 1) * 4);
            compact_flags(c, cs, 0, cpos->as<uint32_t>());
            const uint64_t nchunks = (C + GOB_CHUNK - 1) / GOB_CHUNK;
            Buf succ = dev_alloc(c, C * 4 + 4), exits = dev_alloc(c, C * 4 + 4), entry = dev_alloc(c, nchunks * 4 + 4);
            Buf mark = dev_alloc(c, C * 4 + 4);
            CPB_CUDA(cudaMemsetAsync(entry->p, 0xff, nchunks * 4 + 4, c->stream));
            CPB_CUDA(cudaMemsetAsync(mark->p, 0, C * 4 + 4, c->stream));
            CPB_CUDA(cudaMemsetAsync(st->p, 0, 16, c->stream));
            unsigned long long* ok = st->as<unsigned long long>();
            const uint32_t* cp = cpos->as<uint32_t>();
            {
                KernelTimer kt(c, "gob_path", C * 28, 4);
                // sc[i] = candidate index of the end of candidate i's row: END = C when the row ends at or past the window's
                // end (cp[C] = w is the compaction's sentinel), DEAD when its end is not a candidate
                uint32_t* sc = succ->as<uint32_t>();
                each_row(c, C, [=] __device__(uint64_t i) {
                    const uint64_t e = gob_row_end(b, L, s + cp[i], ks, nullptr, nullptr, 0, 0) - s;
                    if (e >= w) { sc[i] = (uint32_t)C; return; }
                    uint64_t lo = i + 1, hi = C;  // e > cp[i]: the lower bound of e in cp(i, C]
                    while (lo < hi) { const uint64_t h = lo + (hi - lo) / 2; if (cp[h] < e) lo = h + 1; else hi = h; }
                    sc[i] = cp[lo] == e ? (uint32_t)lo : GOB_DEAD;
                });
                if (C) gob_exit_kernel<<<nblk(nchunks, 128), 128, 0, c->stream>>>(succ->as<uint32_t>(), C, exits->as<uint32_t>());
                gob_stitch_kernel<<<1, 1, 0, c->stream>>>(cpos->as<uint32_t>(), exits->as<uint32_t>(), C, entry->as<uint32_t>(), ok);
                if (C)
                    gob_mark_kernel<<<nblk(nchunks, 128), 128, 0, c->stream>>>(b, L, s, ks, cpos->as<uint32_t>(), succ->as<uint32_t>(),
                                                                               entry->as<uint32_t>(), C, mark->as<uint32_t>(), ok + 1);
                CPB_CUDA(cudaGetLastError());
            }
            const FlagScan ms = scan_flags(c, mark->as<uint32_t>(), C);
            const std::vector<uint64_t> h = read_back<uint64_t>(c, st->p, 2);  // {path ends at END, next window start}
            if (h[0] != 1u || h[1] <= s || R + ms.count > nrows)
                gob_fail("index file: the rows do not decode as " + std::to_string(nrows) + " rows of one column set");
            Buf rid = dev_alloc(c, (ms.count + 1) * 4);
            compact_flags(c, ms, 0, rid->as<uint32_t>());
            const uint32_t* row = rid->as<uint32_t>();
            uint64_t* at = start->as<uint64_t>() + R;
            each_row(c, ms.count, [=] __device__(uint64_t j) { at[j] = s + cp[row[j]]; });
            R += ms.count;
            s = h[1];
        }
        if (R != nrows) gob_fail("index file: " + std::to_string(R) + " rows decoded, the file declares " + std::to_string(nrows));
        // 6. value lengths and starts, exact 64-bit column totals (a column holds < 4 GiB), offsets, bytes
        Buf lens = dev_alloc(c, R * k * 4 + 4), vpos = dev_alloc(c, R * k * 8 + 8), tots = dev_alloc(c, k * 8 + 8);
        CPB_CUDA(cudaMemsetAsync(tots->p, 0, k * 8 + 8, c->stream));
        {
            KernelTimer kt(c, "gob_extract", L + R * (8 + 12 * (uint64_t)k));
            const uint64_t* row_start = start->as<uint64_t>();
            uint32_t* ln = lens->as<uint32_t>();
            uint64_t* vp = vpos->as<uint64_t>();
            each_row(c, R, [=] __device__(uint64_t r) { gob_row_end(b, L, row_start[r], ks, ln, vp, R, r); });
            if (k) gob_sum_kernel<<<dim3((uint32_t)std::min<uint64_t>(nblk(R, 256), (uint64_t)c->sm_count * 4), k), 256, 0, c->stream>>>(
                lens->as<uint32_t>(), R, R, tots->as<unsigned long long>());
            CPB_CUDA(cudaGetLastError());
        }
        const std::vector<uint64_t> tot = read_back<uint64_t>(c, tots->p, k);
        for (uint32_t j = 0; j < k; j++) {
            if (tot[j] > 0xffffffffull) throw DataError{CPB_E_TOO_LARGE, (int)j, 0, false, "index file: column " + go_quote(names[j]) + " exceeds 4 GiB"};
            t->cols[j].offsets = dev_alloc(c, (R + 1) * 4);
            exclusive_scan_u32(c, lens->as<uint32_t>() + (uint64_t)j * R, t->cols[j].offsets->as<uint32_t>(), R, tots->as<uint64_t>() + j);
        }
        uint64_t all = 0;
        for (uint32_t j = 0; j < k; j++) {
            t->cols[j].data = dev_alloc(c, tot[j] + 16);
            houts[j] = GobOut{t->cols[j].offsets->as<uint32_t>(), t->cols[j].data->as<uint8_t>()};
            all += tot[j];
        }
        if (k) {
            Buf douts = dev_alloc(c, k * sizeof(GobOut));
            CPB_CUDA(cudaMemcpyAsync(douts->p, houts.data(), k * sizeof(GobOut), cudaMemcpyHostToDevice, c->stream));
            KernelTimer kt(c, "gob_copy", 2 * all + R * k * 12);
            // thread t copies the value of column t / R of row t % R
            const uint32_t* ln = lens->as<uint32_t>();
            const uint64_t* vp = vpos->as<uint64_t>();
            const GobOut* outs = douts->as<GobOut>();
            each_row(c, R * k, [=] __device__(uint64_t t) {
                const uint64_t j = t / R, r = t - j * R;
                const uint32_t l = ln[t];
                const uint8_t* src = b + vp[t];
                uint8_t* d = outs[j].data + outs[j].off[r];
                for (uint32_t i = 0; i < l; i++) d[i] = src[i];
            });
            sync_stream(c);  // houts is pageable host memory
        }
    } else {
        for (auto& col : t->cols) {
            col.offsets = dev_alloc(c, 4);
            col.data = dev_alloc(c, 16);
            CPB_CUDA(cudaMemsetAsync(col.offsets->p, 0, 4, c->stream));
        }
    }
    t->nrows = (int64_t)R;
    auto ix = std::make_shared<Index>();
    ix->ctx = c; ix->key_cols = *key_cols; ix->key_col_idx.assign(key_cols->size(), 0);
    index_adopt_rows(c, *ix, t);
    if ((uint64_t)ix->image_words * 8 > 4096) throw ArgError{CPB_ERR_UNSUPPORTED, "index keys longer than 4 KiB are not supported"};
    return ix;
}

}  // namespace cpb
