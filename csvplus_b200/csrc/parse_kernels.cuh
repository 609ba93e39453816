// parse_kernels.cuh — device code of the fused CSV scan (see parse.cu for the design notes).
//
// v2 layout of one 32 KiB tile (window = tile + 16 B look-behind + 2 KiB look-ahead, staged by TMA):
//   classify   SWAR compares -> newline bitmap T and structural bitmap S (delimiter | newline)
//   quotes     tiles holding a quote (or entered inside one) build the exact quote bitmap, carry the
//              parity across tiles (look-back chain 1) and clear T inside quoted regions
//   index      the set bits of S are expanded, in order, into a flat shared-memory array of byte
//              positions (sidx); the structural ordinal of every terminator goes to `ord`.
//              Line i then spans structurals (ord[i-1], ord[i]] and field j of it is found in O(1):
//              [sidx[ord[i-1]+j]+1, sidx[ord[i-1]+j+1])  — no per-record searching, no divergence.
//   pass 1     one thread per line (blocked): field extents of the selected columns, Like terms,
//              field-count check -> (records, rows, bytes per column)
//   scan       block scan + decoupled look-back (chain 2) -> global output positions
//   pass 2     offsets written, field bytes gathered into the column buffers
// Lines containing quotes, or running past the window, go through the exact sequential state machine.
// Tiles whose structural density exceeds the shared-memory index fall back to a per-thread walk.
#pragma once
#include "core.hpp"
#include "pred.cuh"
#include "subst.hpp"
#include "util.cuh"

// Variants tried and removed because they were slower (timings taken on an earlier GPU target; not re-measured on H100):
//   * drawing the next tile's ticket early (it lengthens the look-back distance);
//   * word-wise staging copies instead of the byte loop (short fields);
//   * one stage for all columns with direct offset stores -- the barriers are not the cost, the byte loop is;
//   * folding the parity verification and the any-slow vote into the block scan's barrier;
//   * 16 KiB tiles with 128-thread CTAs (-DCPB_TILE=16384 -DCPB_THREADS=128) -- the per-tile fixed costs win;
//   * a line-end list + per-line walk of the structural bitmap instead of the flat index: the per-line ffs walk costs
//     what the expansion + O(1) look-ups cost, with longer dependent chains;
//   * a separate "lean" path for quote-free regular tiles (thread owns the lines starting in its 128-byte slice): slice
//     ownership leaves most lanes idle and the unrolled body overflows the instruction cache;
//   * the tile body as a __noinline__ function: shared memory and kernel parameters are then reached through generic
//     pointers.
namespace cpb {

#ifndef CPB_TILE
#define CPB_TILE 32768
#endif
#ifndef CPB_THREADS
#define CPB_THREADS 256
#endif
constexpr int TILE = CPB_TILE;
constexpr int PRE = 16;
constexpr int HALO = 2048;
constexpr int WIN = TILE + HALO;
constexpr int THREADS = CPB_THREADS;
constexpr int WIN_WORDS = WIN / 32;        // 1088
constexpr int TILE_WORDS = TILE / 32;      // 1024
constexpr int HALO_WORDS = HALO / 32;      // 64
constexpr int WPT = TILE_WORDS / THREADS;  // bitmap words per thread (4)
constexpr int SCAP = TILE / 4;             // structural index capacity per window (8192)
constexpr int LCAP = TILE / 16;            // terminator capacity per window (2048)
static_assert(TILE_WORDS == 4 * THREADS, "every thread owns one uint4 of each bitmap");
constexpr int LITS_SMEM = 256;
constexpr int MAXSEL = CPB_MAX_PARSE_COLS;
constexpr int HDR_MAX_FIELDS = 1024;
constexpr int HDR_MAX_BYTES = 16384;
constexpr int HDR_SAMPLE_FIELDS = 64;

enum { K_OK = 0, K_BARE = CPB_E_BARE_QUOTE, K_QUOTE = CPB_E_QUOTE, K_FIELDS = CPB_E_FIELD_COUNT, K_COLIDX = CPB_E_COLUMN_INDEX };

struct ParseResult {  // device -> host
    uint64_t totals[2 + MAXSEL];  // records, rows, bytes per slot
    unsigned long long err_key;   // (record ordinal << 16) | (kind << 8) | slot ; ~0 = none
    unsigned long long err_rows;  // rows delivered before the failing record
    unsigned long long first_row_ordinal;  // record ordinal of output row 0 (~0 if no rows)
    uint32_t fallback_tiles;      // tiles that took the dense fallback
    uint32_t eof_hit;             // a record of this shard was closed by the end of the buffer, not by a terminator
    uint32_t need_general;        // a comment line that may hold a quote was seen: the quote-parity shortcut does not hold, rerun on the general path
    uint32_t pad_;
};

struct ParseParams {
    const uint8_t* in;
    uint64_t n;
    uint64_t data_start;  // records starting before this byte are not data (header row)
    uint32_t ntiles;
    uint32_t delim;
    int32_t expect_fields;  // >0: every record must have exactly this many fields
    int32_t pad_missing;    // numFields < 0: short records pad selected columns with ""
    int32_t nsel;
    int32_t sel_field[MAXSEL];  // ascending, distinct
    uint32_t* out_off[MAXSEL];
    uint8_t* out_data[MAXSEL];
    uint64_t data_cap[MAXSEL];
    uint64_t row_cap;
    const uint8_t* lits;
    uint32_t lits_len;
    PredProg pred;
    uint32_t slot_terms[MAXSEL];  // per slot: mask of Like terms comparing that slot
    // look-back state
    uint32_t* st1;   // [ntiles] quote-parity chain: bits1:0 status (1 aggregate, 2 inclusive), bit2 value
    unsigned long long* words;  // [ntiles][2+nsel] totals chain: bits 63:62 status, bits 61:0 value (self-validating)
    uint32_t* ticket;
    ParseResult* result;
    const SubTable* subs;  // stand-in bytes of multi-byte reader runes (subst.cu), null when there are none
    // byte-range shards of one file (cpb_parse_csv_shard): the quote parity the buffer starts with, and the last byte
    // position at which a record may START to belong to this shard (later ones are the next shard's; ~0: no limit)
    uint32_t pin0;
    uint32_t l2_ahead;     // 1: prefetch the tile one grid-width ahead into L2
    uint32_t ds_is_start;  // data_start is itself the first byte of a record (after a header row); 0 for shards after the first
    uint64_t own_end;
    // reader options csv_scan_kernel's guarded instantiations take optimistically (parse.cu): TrimLeadingSpace, and the
    // CommentChar byte (0: none).  The kernels specialised on the column count never read them.
    uint32_t trim, comment;
};

// ------------------------------------------------------------------ byte source: staged window or HBM
struct ByteSrc {
    const uint8_t* g; uint64_t n;
    const uint8_t* s; uint64_t s_lo, s_hi;  // smem copy of absolute [s_lo, s_hi)
    __device__ __forceinline__ int get(uint64_t pos) const {
        if (pos >= n) return -1;
        if (pos >= s_lo && pos < s_hi) return s[pos - s_lo];
        return g[pos];
    }
};

struct SeqResult { int err; int nfields; uint64_t next; };

// Exact sequential restatement of encoding/csv readRecord (+readLine's \r\n and trailing-\r rules)
// for one record starting at `start` (a non-empty line start), default options, single-byte comma.
// Sink: begin_field(f) / put(byte) / unput() / end_field().
template <class Sink>
__device__ SeqResult seq_parse_record(const ByteSrc& src, uint64_t start, int delim, Sink& sink) {
    uint64_t pos = start;
    int f = 0;
    for (;;) {  // parseField
        sink.begin_field(f);
        int c = src.get(pos);
        if (c != '"') {
            // non-quoted field: up to the next comma or end of line
            uint64_t fb = pos;
            for (;;) {
                c = src.get(pos);
                if (c == delim) { sink.end_field(); pos++; f++; break; }
                if (c == '\n' || c < 0) {
                    // "\r\n" -> "\n" normalisation / trailing \r before EOF: the \r was already fed; retract it
                    if (pos > fb && src.get(pos - 1) == '\r') sink.unput();
                    sink.end_field();
                    return {K_OK, f + 1, c < 0 ? src.n : pos + 1};
                }
                if (c == '"') return {K_BARE, f + 1, pos};
                sink.put(c);
                pos++;
            }
        } else {
            pos++;  // opening quote
            for (;;) {
                c = src.get(pos);
                if (c < 0) return {K_QUOTE, f + 1, pos};  // EOF inside quotes (non-lazy)
                if (c == '"') {
                    int c2 = src.get(pos + 1);
                    if (c2 == '"') { sink.put('"'); pos += 2; continue; }
                    if (c2 == delim) { sink.end_field(); pos += 2; f++; break; }
                    if (c2 == '\n') { sink.end_field(); return {K_OK, f + 1, pos + 2}; }
                    if (c2 < 0) { sink.end_field(); return {K_OK, f + 1, src.n}; }
                    if (c2 == '\r') {
                        int c3 = src.get(pos + 2);
                        if (c3 == '\n') { sink.end_field(); return {K_OK, f + 1, pos + 3}; }
                        if (c3 < 0) { sink.end_field(); return {K_OK, f + 1, src.n}; }
                    }
                    return {K_QUOTE, f + 1, pos};
                }
                if (c == '\r') {
                    int c2 = src.get(pos + 1);
                    if (c2 == '\n') { sink.put('\n'); pos += 2; continue; }  // \r\n -> \n on every physical line
                    if (c2 < 0) return {K_QUOTE, f + 1, pos};               // trailing \r dropped, then EOF in quotes
                }
                sink.put(c);
                pos++;
            }
        }
    }
}

// Exact sequential restatement of encoding/csv readRecord with LazyQuotes / TrimLeadingSpace (single-byte comma).
template <class Sink>
__device__ SeqResult seq_parse_record_gen(const ByteSrc& src, uint64_t start, int delim, bool lazy, bool trim, const uint32_t* sp_bits, Sink& sink) {
    uint64_t pos = start;
    int f = 0;
    auto is_sp = [&](int c) { return c == ' ' || c == '\t' || c == '\v' || c == '\f' || c == '\r' || sub_is(sp_bits, c); };
    for (;;) {  // parseField
        sink.begin_field(f);
        if (trim) {
            // bytes.IndexFunc(line, !unicode.IsSpace): the line's own "\n" is white space too, so a field of
            // spaces up to the end of the line is empty and ends the record
            for (;;) {
                int c = src.get(pos);
                if (c == '\n') { sink.end_field(); return {K_OK, f + 1, pos + 1}; }
                if (c < 0) { sink.end_field(); return {K_OK, f + 1, src.n}; }
                if (!is_sp(c)) break;
                pos++;
            }
        }
        int c = src.get(pos);
        if (c != '"') {
            uint64_t fb = pos;
            for (;;) {
                c = src.get(pos);
                if (c == delim) { sink.end_field(); pos++; f++; break; }
                if (c == '\n' || c < 0) {
                    if (pos > fb && src.get(pos - 1) == '\r') sink.unput();
                    sink.end_field();
                    return {K_OK, f + 1, c < 0 ? src.n : pos + 1};
                }
                if (c == '"' && !lazy) return {K_BARE, f + 1, pos};
                sink.put(c);
                pos++;
            }
        } else {
            pos++;
            for (;;) {
                c = src.get(pos);
                if (c < 0) {  // abrupt end of file inside quotes
                    if (!lazy) return {K_QUOTE, f + 1, pos};
                    sink.end_field();
                    return {K_OK, f + 1, src.n};
                }
                if (c == '"') {
                    int c2 = src.get(pos + 1);
                    if (c2 == '"') { sink.put('"'); pos += 2; continue; }
                    if (c2 == delim) { sink.end_field(); pos += 2; f++; break; }
                    if (c2 == '\n') { sink.end_field(); return {K_OK, f + 1, pos + 2}; }
                    if (c2 < 0) { sink.end_field(); return {K_OK, f + 1, src.n}; }
                    if (c2 == '\r') {
                        int c3 = src.get(pos + 2);
                        if (c3 == '\n') { sink.end_field(); return {K_OK, f + 1, pos + 3}; }
                        if (c3 < 0) { sink.end_field(); return {K_OK, f + 1, src.n}; }
                    }
                    if (!lazy) return {K_QUOTE, f + 1, pos};
                    sink.put('"');  // `"` sequence (bare quote) under LazyQuotes
                    pos++;
                    continue;
                }
                if (c == '\r') {
                    int c2 = src.get(pos + 1);
                    if (c2 == '\n') { sink.put('\n'); pos += 2; continue; }
                    if (c2 < 0) {  // trailing \r before EOF is dropped, then EOF inside quotes
                        if (!lazy) return {K_QUOTE, f + 1, pos};
                        sink.end_field();
                        return {K_OK, f + 1, src.n};
                    }
                }
                sink.put(c);
                pos++;
            }
        }
    }
}

// the ASCII white space TrimLeadingSpace trims inside a line (unicode.IsSpace minus '\n'; the multi-byte spaces go
// through stand-in bytes and the general path)
__device__ __forceinline__ bool is_space_byte(int c) { return c == ' ' || c == '\t' || c == '\v' || c == '\f' || c == '\r'; }

// ------------------------------------------------------------------ header kernel
struct HeaderOut {
    int32_t err;        // K_* of the first record (0 ok)
    int32_t nfields;
    int32_t eof;        // 1: no record at all
    int32_t truncated;  // names did not fit
    uint64_t rec_start, data_start;
    uint64_t sample_bytes, sample_newlines;
    unsigned long long samp_lines;                            // lines split naively for the capacity estimate
    unsigned long long samp_field_bytes[HDR_SAMPLE_FIELDS];   // their bytes per field index
    uint32_t field_len[HDR_MAX_FIELDS];
    uint8_t bytes[HDR_MAX_BYTES];
};
struct HeaderSink {
    HeaderOut* o; const SubTable* subs = nullptr; int f = 0; uint32_t len = 0; uint32_t used = 0;
    __device__ void begin_field(int fi) { f = fi; len = 0; }
    __device__ void put1(int c) { if (used < HDR_MAX_BYTES) o->bytes[used] = (uint8_t)c; else o->truncated = 1; used++; len++; }
    __device__ void put(int c) {
        if (subs && sub_is(subs->bits, c)) { for (int j = 0; j < subs->len[c]; j++) put1(subs->seq[c][j]); }
        else put1(c);
    }
    __device__ void unput() { used--; len--; }
    __device__ void end_field() { if (f < HDR_MAX_FIELDS) o->field_len[f] = len; else o->truncated = 1; }
};

// Parses the first record (makeHeader's reader.Read(), csvplus.go:1150) and samples newline density
// in three 64 KiB windows for the row-capacity estimate.  The first 8 KiB are staged in shared memory
// so that the sequential parse of a normal header never waits on HBM.
// sample_only: the first record was parsed by the options-aware g_header_kernel (parse_general.cu); only the sampling runs.
static __global__ void csv_header_kernel(const uint8_t* in, uint64_t n, int delim, const SubTable* subs, HeaderOut* out, int sample_only = 0) {
    __shared__ unsigned long long s_nl;
    __shared__ uint8_t s_head[8192];
    const uint64_t staged = n < 8192 ? n : 8192;
    for (uint64_t i = threadIdx.x; i < staged; i += blockDim.x) s_head[i] = in[i];
    if (threadIdx.x == 0) s_nl = 0;
    __syncthreads();
    if (threadIdx.x == 0 && !sample_only) {
        ByteSrc src{in, n, s_head, 0, staged};
        uint64_t pos = 0;
        // skip empty lines: "\n", "\r\n", and a lone trailing "\r" before EOF
        for (;;) {
            int c = src.get(pos);
            if (c == '\n') { pos++; continue; }
            if (c == '\r') {
                int c2 = src.get(pos + 1);
                if (c2 == '\n') { pos += 2; continue; }
                if (c2 < 0) { pos += 1; continue; }
            }
            break;
        }
        out->truncated = 0;
        out->rec_start = pos;
        if (pos >= n) { out->eof = 1; out->err = 0; out->nfields = 0; out->data_start = n; }
        else {
            HeaderSink sink{out, subs};
            SeqResult r = seq_parse_record(src, pos, delim, sink);
            out->eof = 0; out->err = r.err; out->nfields = r.nfields; out->data_start = r.next;
        }
    }
    const uint64_t S = 65536;
    unsigned long long cnt = 0, tot = 0;
    for (int w = 0; w < 3; w++) {
        uint64_t lo = w == 0 ? 0 : (w == 1 ? (n / 2) : (n > S ? n - S : 0));
        uint64_t hi = lo + S < n ? lo + S : n;
        // 16 bytes per thread per step, several loads in flight (a byte-at-a-time loop is latency-bound: ~0.3 ms)
        const uint64_t lo16 = (lo + 15) & ~15ull, hi16 = hi & ~15ull;
        if (lo16 < hi16) {
            const uint4* v = reinterpret_cast<const uint4*>(in + lo16);
            const uint64_t nv = (hi16 - lo16) / 16;
#pragma unroll 4
            for (uint64_t i = threadIdx.x; i < nv; i += blockDim.x) {
                const uint4 x = v[i];
                cnt += __popc(eq_flags(x.x, 0x0a0a0a0au)) + __popc(eq_flags(x.y, 0x0a0a0a0au)) + __popc(eq_flags(x.z, 0x0a0a0a0au)) +
                       __popc(eq_flags(x.w, 0x0a0a0a0au));
            }
            tot += hi16 - lo16;
        }
    }
    atomicAdd(&s_nl, cnt);
    // mean field lengths: every thread splits one line (naively: quotes ignored — this only sizes buffers) in each window
    __shared__ unsigned long long s_lines, s_fb[HDR_SAMPLE_FIELDS];
    if (threadIdx.x == 0) s_lines = 0;
    if (threadIdx.x < HDR_SAMPLE_FIELDS) s_fb[threadIdx.x] = 0;
    __syncthreads();
    for (int w = 0; w < 3; w++) {
        uint64_t lo = w == 0 ? 0 : (w == 1 ? (n / 2) : (n > S ? n - S : 0));
        uint64_t p = lo + (uint64_t)threadIdx.x * (S / blockDim.x);
        uint64_t lim = p + 4096 < n ? p + 4096 : n;
        while (p < lim && in[p] != '\n') p++;
        p++;  // first byte of the next line
        if (p >= n || p >= lim) continue;
        lim = p + 4096 < n ? p + 4096 : n;
        int f = 0; uint32_t len = 0; bool done = false;
        for (; p < lim; p++) {
            uint8_t ch = in[p];
            if (ch == delim || ch == '\n') {
                if (f < HDR_SAMPLE_FIELDS) atomicAdd(&s_fb[f], (unsigned long long)len);
                f++; len = 0;
                if (ch == '\n') { done = true; break; }
            } else len++;
        }
        if (done) atomicAdd(&s_lines, 1ull);
        else for (int g = 0; g < f && g < HDR_SAMPLE_FIELDS; g++) {}  // partial line: its complete fields stay counted (slight overestimate)
    }
    __syncthreads();
    if (threadIdx.x == 0) { out->sample_bytes = tot; out->sample_newlines = s_nl; out->samp_lines = s_lines; }
    if (threadIdx.x < HDR_SAMPLE_FIELDS) out->samp_field_bytes[threadIdx.x] = s_fb[threadIdx.x];
}

// ------------------------------------------------------------------ main kernel
struct __align__(16) ParseSmem {
    uint8_t data[PRE + WIN + 16];
    uint32_t Tb[WIN_WORDS + 4];  // record terminators: '\n' outside quotes (+ a virtual one at EOF)
    uint32_t Sb[WIN_WORDS + 4];  // structural bytes: delimiter | terminator
    uint32_t Qb[WIN_WORDS + 4];  // quote bytes (exact; only built for tiles that contain quotes)
    uint16_t sidx[SCAP];         // byte position of every structural, in order
    uint16_t ord[LCAP];          // structural ordinal of every terminator, in order
    __align__(16) uint8_t lits[LITS_SMEM + 16];  // Like literals (word-wise compares read up to 7 bytes past the end)
    uint64_t mbar;
    uint64_t tile_prefix[2 + MAXSEL];
    uint32_t wtot[1 + MAXSEL][THREADS / 32];
    uint32_t wpar[THREADS / 32];
    uint64_t col_total[2 + MAXSEL];  // last tile: grand totals (records, rows, bytes per column)
    uint32_t ticket;
    uint32_t pin;
    uint32_t nstruct, nterm;     // totals of the window
};

__device__ __forceinline__ int next_set(const uint32_t* bm, int from, int lim) {
    int wi = from >> 5;
    uint32_t m = bm[wi] & (0xffffffffu << (from & 31));
    for (;;) {
        if (m) { int i = (wi << 5) + __ffs(m) - 1; return i < lim ? i : lim; }
        wi++;
        if ((wi << 5) >= lim) return lim;
        m = bm[wi];
    }
}
// (out of line: only tiles that contain quotes call it, and it would be inlined once per cached line)
static __device__ __noinline__ int count_bits(const uint32_t* bm, int a, int b) {  // bits set in [a,b)
    if (a >= b) return 0;
    int wa = a >> 5, wb = b >> 5;
    uint32_t ma = 0xffffffffu << (a & 31);
    uint32_t mb = (b & 31) ? (0xffffffffu >> (32 - (b & 31))) : 0u;
    if (wa == wb) return __popc(bm[wa] & ma & mb);
    int c = __popc(bm[wa] & ma);
    for (int w = wa + 1; w < wb; w++) c += __popc(bm[w]);
    if (mb) c += __popc(bm[wb] & mb);
    return c;
}
__device__ __forceinline__ bool bytes_eq(const uint8_t* a, const uint8_t* lit, uint32_t n) {
    for (uint32_t i = 0; i < n; i++) if (a[i] != lit[i]) return false;
    return true;
}
// 4 bytes starting at an arbitrary byte offset of a 4-byte aligned shared-memory array (reads 8 aligned bytes)
__device__ __forceinline__ uint32_t lds_u32_at(const uint8_t* base, uint32_t off) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(base + (off & ~3u));
    return __funnelshift_r(w[0], w[1], (off & 3u) * 8);
}
// field (in the staged window) == literal (in shared memory), both read a word at a time
__device__ __forceinline__ bool field_eq_smem(const uint8_t* data, uint32_t foff, const uint8_t* lits, uint32_t loff, uint32_t n) {
    uint32_t i = 0;
    for (; i + 4 <= n; i += 4) if (lds_u32_at(data, foff + i) != lds_u32_at(lits, loff + i)) return false;
    if (i < n) {
        const uint32_t m = (1u << (8 * (n - i))) - 1;
        if ((lds_u32_at(data, foff + i) ^ lds_u32_at(lits, loff + i)) & m) return false;
    }
    return true;
}
// Sink of the slow path inside the main kernel: tracks the selected slots of one record.
struct SlowSink {
    const ParseParams& P;
    bool emit;
    int next_slot = 0, cur = -1;
    uint32_t len = 0, present = 0, alive = 0, eq = 0;
    uint32_t alive_before = 0;  // count: alive before the last put1, restored by unput (a retracted '\r' must not kill a term)
    uint32_t ulen[MAXSEL];
    uint8_t* dst[MAXSEL];
    uint32_t maxlen[MAXSEL];  // emit: value lengths known from pass 1 (a retracted '\r' must never be stored)
    __device__ SlowSink(const ParseParams& p, bool e) : P(p), emit(e) {}
    __device__ void begin_field(int f) {
        cur = -1;
        if (next_slot < P.nsel && P.sel_field[next_slot] == f) { cur = next_slot++; len = 0; alive = P.slot_terms[cur]; }
    }
    __device__ void put(int c) {
        if (cur < 0) return;
        if (P.subs && sub_is(P.subs->bits, c)) {  // a stand-in byte that is data here: its original UTF-8 sequence
            const int n = P.subs->len[c];
            for (int j = 0; j < n; j++) put1(P.subs->seq[c][j]);
        } else put1(c);
    }
    __device__ void put1(int c) {
        if (emit) { if (dst[cur] && len < maxlen[cur]) dst[cur][len] = (uint8_t)c; }
        else {
            alive_before = alive;
            uint32_t m = alive;
            while (m) {
                int t = __ffs(m) - 1; m &= m - 1;
                if (len >= P.pred.term_len[t] || __ldg(P.lits + P.pred.term_off[t] + len) != (uint8_t)c) alive &= ~(1u << t);
            }
        }
        len++;
    }
    __device__ void unput() { if (cur >= 0) { len--; alive = alive_before; } }
    __device__ void end_field() {
        if (cur < 0) return;
        ulen[cur] = len; present |= 1u << cur;
        uint32_t m = alive;
        while (m) { int t = __ffs(m) - 1; m &= m - 1; if (len == P.pred.term_len[t]) eq |= 1u << t; }
    }
};

struct SlowOut { uint32_t ulen[MAXSEL]; uint32_t present, eq; int nf, err; };

// count mode (emit=false): lengths / predicate terms / error of one record; emit mode: store the unescaped values.
// (TRIM: the options-aware machine with TrimLeadingSpace — only the guarded kernel instantiations reference it, so the
// kernels specialised on the column count carry exactly the code they carried before)
template <bool TRIM>
static __device__ __noinline__ void slow_record_t(const ParseParams& P, const ByteSrc& src, uint64_t start, bool emit,
                                                  const uint64_t* dst_off, const uint32_t* maxlen, SlowOut* o) {
    SlowSink sink(P, emit);
    if (emit) {
        for (int k = 0; k < P.nsel; k++) {
            bool fits = dst_off[k] + maxlen[k] <= P.data_cap[k];
            sink.dst[k] = fits ? P.out_data[k] + dst_off[k] : nullptr;
            sink.maxlen[k] = maxlen[k];
        }
    }
    SeqResult s;
    if (TRIM) {
        const uint32_t no_sp[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        s = seq_parse_record_gen(src, start, (int)P.delim, false, true, no_sp, sink);
    } else s = seq_parse_record(src, start, (int)P.delim, sink);
    o->err = s.err; o->nf = s.nfields; o->present = sink.present; o->eq = sink.eq;
    // (shards: a record closed by the end of the buffer instead of a terminator — benign race, every writer stores 1)
    if (!emit && s.err == K_OK && s.next >= src.n && src.n > 0 && src.get(src.n - 1) != '\n') P.result->eof_hit = 1u;
    for (int k = 0; k < P.nsel; k++) o->ulen[k] = ((sink.present >> k) & 1) ? sink.ulen[k] : 0;
}

template <bool EXACT>
__device__ __forceinline__ void slow_record(const ParseParams& P, const ByteSrc& src, uint64_t start, bool emit,
                                            const uint64_t* dst_off, const uint32_t* maxlen, SlowOut* o) {
    if (!EXACT && P.trim) slow_record_t<true>(P, src, start, emit, dst_off, maxlen, o);
    else slow_record_t<false>(P, src, start, emit, dst_off, maxlen, o);
}

template <int KMAX>
struct Rec {
    uint32_t f[KMAX];  // fast: beg | len << 16 (window-relative); slow: unescaped length
    uint32_t present, eq;
    int nf, err, err_slot;
    bool slow;
};

// record-level checks in the reference's order: parse error (already set) > field count > missing column
// HP ("has predicate") = false compiles every Like comparison out: the kernels of unfiltered parses carry no
// literal-compare code between their hot loops (the kernel is instruction-fetch sensitive).
template <int KMAX, bool EXACT, bool HP>
__device__ __forceinline__ void finish_record(const ParseParams& P, Rec<KMAX>& r) {
    if (r.err != K_OK) return;
    if (P.expect_fields > 0 && r.nf != P.expect_fields) { r.err = K_FIELDS; return; }
    uint32_t want = (1u << (EXACT ? KMAX : P.nsel)) - 1;
    uint32_t missing = want & ~r.present;
    if (missing) {
        if (P.pad_missing) {  // padded "" values still take part in Like comparisons against empty literals
            uint32_t m = HP ? missing : 0u;
            while (m) {
                int k = __ffs(m) - 1; m &= m - 1;
                uint32_t tm = P.slot_terms[k];
                while (tm) { int t = __ffs(tm) - 1; tm &= tm - 1; if (P.pred.term_len[t] == 0) r.eq |= 1u << t; }
            }
        } else { r.err = K_COLIDX; r.err_slot = __ffs(missing) - 1; }
    }
}

template <int KMAX, bool EXACT>
__device__ __forceinline__ void run_slow(const ParseParams& P, const ByteSrc& src, uint64_t start_abs, Rec<KMAX>& r) {
    SlowOut so;
    slow_record<EXACT>(P, src, start_abs, false, nullptr, nullptr, &so);
    r.err = so.err; r.nf = so.nf; r.present = so.present; r.eq = so.eq; r.slow = true; r.err_slot = 0;
#pragma unroll
    for (int k = 0; k < KMAX; k++) r.f[k] = k < (EXACT ? KMAX : P.nsel) ? so.ulen[k] : 0;
}

// Line `i` of the window through the flat structural index.  Returns false when it is not a record.
template <int KMAX, bool EXACT, bool HP>
__device__ __forceinline__ bool flat_line(const ParseParams& P, const ParseSmem& sm, const ByteSrc& src, const uint8_t* lits,
                                          bool lits_in_smem, uint64_t tile_base, int i, int nterm, int rel_n, int64_t rel_ds, bool tile_has_q,
                                          Rec<KMAX>& r) {
    const int a = i == 0 ? -1 : (int)sm.ord[i - 1];
    const int start = i == 0 ? 0 : (int)sm.sidx[a] + 1;
    if (start >= rel_n || start < rel_ds) return false;
    r.present = 0; r.eq = 0; r.err = K_OK; r.err_slot = 0; r.slow = false;
    bool to_slow = i >= nterm;  // no terminator inside the window: runs past it
    int b = 0, e_nl = 0, e = 0;
    if (!to_slow) {
        b = sm.ord[i]; e_nl = sm.sidx[b];
        e = e_nl;
        if (e > start && sm.data[PRE + e - 1] == '\r') e--;  // \r\n -> \n ; trailing \r before EOF
        if (e == start) return false;                          // empty line: not a record
        if (tile_has_q && count_bits(sm.Qb, start, e_nl) != 0) to_slow = true;
    }
    if (!EXACT && P.comment != 0 && sm.data[PRE + start] == (uint8_t)P.comment) {
        // a comment line (checked on the raw line, before any trimming): not a record.  Its quotes, if it has any, were
        // counted by the parity chain though — the parse is then redone on the general path (rare; parse.cu)
        if (to_slow) P.result->need_general = 1u;
        return false;
    }
    if (to_slow) {
        run_slow<KMAX, EXACT>(P, src, tile_base + start, r);
    } else {
        const int nf = b - a;
        r.nf = nf;
#pragma unroll
        for (int k = 0; k < KMAX; k++) {
            r.f[k] = 0;
            if (k < (EXACT ? KMAX : P.nsel)) {
                const int target = P.sel_field[k];
                if (target < nf) {
                    int fb = target == 0 ? start : (int)sm.sidx[a + target] + 1;
                    const int fe = target + 1 < nf ? (int)sm.sidx[a + target + 1] : e;
                    if (!EXACT && P.trim) while (fb < fe && is_space_byte(sm.data[PRE + fb])) fb++;  // TrimLeadingSpace
                    const uint32_t len = (uint32_t)(fe - fb);
                    r.f[k] = (uint32_t)fb | (len << 16);
                    r.present |= 1u << k;
                    uint32_t tm = HP ? P.slot_terms[k] : 0u;
                    while (tm) {
                        int t = __ffs(tm) - 1; tm &= tm - 1;
                        if (len == P.pred.term_len[t]) {
                            const bool eq = lits_in_smem ? field_eq_smem(sm.data, PRE + fb, sm.lits, P.pred.term_off[t], len)
                                                         : bytes_eq(sm.data + PRE + fb, lits + P.pred.term_off[t], len);
                            if (eq) r.eq |= 1u << t;  // (inline: an out-of-line compare was slower)
                        }
                    }
                }
            }
        }
    }
    finish_record<KMAX, EXACT, HP>(P, r);
    return true;
}

// Dense-tile fallback: the record starting at window offset ws, always through the sequential machine.
template <int KMAX, bool EXACT, bool HP>
__device__ __forceinline__ bool generic_record(const ParseParams& P, const ParseSmem& sm, const ByteSrc& src, uint64_t tile_base,
                                               int ws, int rel_n, Rec<KMAX>& r) {
    // empty line: "\n", "\r\n", or a lone "\r" right before EOF
    if (!EXACT && tile_base + (uint64_t)ws > P.own_end) return false;
    int c0 = sm.data[PRE + ws];
    if (c0 == '\n') return false;
    if (c0 == '\r' && (sm.data[PRE + ws + 1] == '\n' || ws + 1 >= rel_n)) return false;
    if (!EXACT && P.comment != 0 && c0 == (int)P.comment) { P.result->need_general = 1u; return false; }  // (dense tiles do not look for its quotes)
    r.present = 0; r.eq = 0; r.err = K_OK; r.err_slot = 0;
    run_slow<KMAX, EXACT>(P, src, tile_base + ws, r);
    finish_record<KMAX, EXACT, HP>(P, r);
    return true;
}


// ------------------------------------------------------------------ decoupled look-back (one warp)
// In steady state the nearest inclusive predecessor is a few tiles back, so one 32-wide round (one L2 round trip)
// resolves the look-back while the other warps wait at a single barrier.  (A block-wide, 256-predecessors-per-round
// version was measured slower.)
constexpr unsigned long long LB_AGG = 1ull << 62, LB_INCL = 2ull << 62, LB_VAL = (1ull << 62) - 1;

__device__ __forceinline__ uint32_t lookback_parity_w0(const uint32_t* st1, uint32_t tile) {
    const int lane = threadIdx.x & 31;
    uint32_t acc = 0;
    int64_t base = (int64_t)tile - 1;
    for (;;) {
        const int64_t p = base - lane;
        uint32_t s = 2u;
        if (p >= 0) { do { s = ld_relaxed_u32(&st1[p]); } while ((s & 3u) == 0); }
        const uint32_t incl = __ballot_sync(0xffffffffu, (s & 3u) == 2u);
        const uint32_t vals = __ballot_sync(0xffffffffu, (s >> 2) & 1u);
        if (incl) { const int f = __ffs(incl) - 1; acc ^= __popc(vals & (0xffffffffu >> (31 - f))) & 1; break; }
        acc ^= __popc(vals) & 1;
        base -= 32;
    }
    return acc;
}
template <int KMAX>
__device__ __forceinline__ void lookback_totals_w0(const unsigned long long* words, uint32_t tile, int NP, ParseSmem& sm) {
    const int lane = threadIdx.x & 31;
    unsigned long long excl = 0;  // lane c accumulates component c
    int64_t base = (int64_t)tile - 1;
    for (;;) {
        const int64_t p = base - lane;
        unsigned long long v[KMAX + 2];
        bool is_incl = true;
        if (p >= 0) {
            const unsigned long long* w = words + (uint64_t)p * NP;
            for (;;) {  // re-read until all words are valid and carry the same status
#pragma unroll
                for (int c = 0; c < KMAX + 2; c++) v[c] = c < NP ? ld_relaxed_u64((const uint64_t*)(w + c)) : 0ull;
                const unsigned long long f0 = v[0] >> 62;
                bool ok = f0 != 0;
#pragma unroll
                for (int c = 1; c < KMAX + 2; c++) if (c < NP) ok = ok && (v[c] >> 62) == f0;
                if (ok) break;
            }
            is_incl = (v[0] >> 62) == 2;
        } else {
#pragma unroll
            for (int c = 0; c < KMAX + 2; c++) v[c] = 0ull;  // before the first tile: inclusive zero
        }
        const uint32_t incl = __ballot_sync(0xffffffffu, is_incl);
        const int f = __ffs(incl) - 1;
        const bool take = p >= 0 && (f < 0 || lane <= f);
#pragma unroll
        for (int c = 0; c < KMAX + 2; c++) {
            if (c < NP) {
                const unsigned long long x = warp_sum_u64(take ? (v[c] & LB_VAL) : 0ull);
                if (lane == c) excl += x;
            }
        }
        if (f >= 0) break;
        base -= 32;
    }
    if (lane < NP) sm.tile_prefix[lane] = excl;
}

// Byte-range shards (not the file's last): the tile that holds own_end keeps only the lines that start at or before it
// — starts ascend with the line index, so that is a prefix — and the tile that sees the end of the buffer reports
// whether the line closed by the virtual terminator there is one of this shard's records (look-ahead too small).
// Cold and out of line: the hot per-line code carries none of it.
static __device__ __noinline__ int shard_tile_tail(const ParseParams& P, const ParseSmem& sm, uint32_t tile, uint64_t tile_base, int i0, int m_last,
                                                   int nterm, int rel_n, int64_t rel_ds) {
    int m_last_v = m_last;
    if (tile == P.ntiles - 1) {
        const int64_t rel_oe = (int64_t)(P.own_end - tile_base);
        int lo = i0 - 1, hi = m_last;  // invariant: line lo starts <= rel_oe (or lo = i0 - 1); lines after hi start > rel_oe
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            const int st = mid == 0 ? 0 : (int)sm.sidx[sm.ord[mid - 1]] + 1;
            if (st <= rel_oe) lo = mid; else hi = mid - 1;
        }
        m_last_v = lo;
    }
    if (rel_n < WIN && threadIdx.x == 0 && nterm >= 1) {
        const int il = nterm - 1;
        const int st = il == 0 ? 0 : (int)sm.sidx[sm.ord[il - 1]] + 1;
        if (il >= i0 && il <= m_last_v && st < rel_n && st >= rel_ds && (int)sm.sidx[sm.ord[il]] == rel_n) P.result->eof_hit = 1u;
    }
    return m_last_v;
}

template <int KMAX, bool EXACT, bool HP>
__global__ void __launch_bounds__(THREADS, KMAX <= 8 ? 768 / THREADS : 1) csv_scan_kernel(const __grid_constant__ ParseParams P) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    ParseSmem& sm = *reinterpret_cast<ParseSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int NP = 2 + (EXACT ? KMAX : P.nsel);
    const uint32_t NL4 = 0x0a0a0a0au, Q4 = 0x22222222u, D4 = P.delim * 0x01010101u;

    if (tid == 0) { mbar_init(&sm.mbar, 1); fence_mbar_init(); }
    const bool lits_in_smem = P.lits_len <= LITS_SMEM;
    if (lits_in_smem) for (uint32_t i = tid; i < P.lits_len; i += THREADS) sm.lits[i] = P.lits[i];
    const uint8_t* lits = lits_in_smem ? sm.lits : P.lits;
    __syncthreads();
    uint32_t phase = 0;

    for (;;) {
        if (tid == 0) sm.ticket = atomicAdd(P.ticket, 1u);
        __syncthreads();
        const uint32_t tile = sm.ticket;
        if (tile >= P.ntiles) break;
        const uint64_t tile_base = (uint64_t)tile * TILE;
        // ---- stage the window [tile_base-PRE, tile_base+WIN) with one bulk copy
        const uint64_t w_lo = tile_base >= PRE ? tile_base - PRE : 0;
        const uint64_t n16 = (P.n + 15) & ~15ull;
        const uint64_t w_hi = tile_base + WIN < n16 ? tile_base + WIN : n16;
        const uint32_t lead = (uint32_t)(PRE - (tile_base - w_lo));  // 0, or PRE for tile 0
        const uint32_t nbytes = (uint32_t)(w_hi - w_lo);
        if (tid == 0) {
            fence_proxy_async();
            mbar_expect_tx(&sm.mbar, nbytes);
            bulk_g2s(sm.data + lead, P.in + w_lo, nbytes, &sm.mbar);
            // the tile one grid-width ahead is taken (by some CTA) about one tile time from now: pull it into L2 so that its
            // bulk load finds it there
            if (P.l2_ahead) {
                const uint64_t pf = tile_base + (uint64_t)gridDim.x * TILE;
                if (pf + TILE <= (P.n & ~15ull)) bulk_prefetch_l2(P.in + pf, TILE);
            }
        }
        mbar_wait(&sm.mbar, phase);
        phase ^= 1;
        // bytes at absolute positions >= n are zeroed so that they classify as nothing
        const int64_t rel_n64 = (int64_t)(P.n - tile_base);  // > 0
        if (rel_n64 < WIN) {
            for (int i = (int)rel_n64 + tid; i < WIN + 16; i += THREADS) sm.data[PRE + i] = 0;
            __syncthreads();
        }
        const int rel_n = rel_n64 < WIN ? (int)rel_n64 : WIN;  // also the limit of valid window bytes
        const bool eof_in_win = rel_n64 < WIN;
        const int64_t rel_ds = (int64_t)P.data_start - (int64_t)tile_base;

        // ---- classify: newline / structural bitmaps, quote presence
        const uint4* d4 = reinterpret_cast<const uint4*>(sm.data + PRE);
        uint16_t* T16 = reinterpret_cast<uint16_t*>(sm.Tb);
        uint16_t* S16 = reinterpret_cast<uint16_t*>(sm.Sb);
        uint32_t anyq = 0;
        for (int v = tid; v < WIN / 16; v += THREADS) {
            uint4 x = d4[v];
            uint32_t nl = flags16(eq_flags(x.x, NL4), eq_flags(x.y, NL4), eq_flags(x.z, NL4), eq_flags(x.w, NL4));
            uint32_t dl = flags16(eq_flags(x.x, D4), eq_flags(x.y, D4), eq_flags(x.z, D4), eq_flags(x.w, D4));
            T16[v] = (uint16_t)nl;
            S16[v] = (uint16_t)(dl | nl);
            anyq |= eq_any(x.x, Q4) | eq_any(x.y, Q4) | eq_any(x.z, Q4) | eq_any(x.w, Q4);
        }
        if (tid < 4) { sm.Tb[WIN_WORDS + tid] = 0; sm.Sb[WIN_WORDS + tid] = 0; sm.Qb[WIN_WORDS + tid] = 0; }
        const bool hasq = __syncthreads_or(anyq != 0);
        uint32_t tile_par = 0;
        if (hasq) {
            uint16_t* Q16 = reinterpret_cast<uint16_t*>(sm.Qb);
            for (int v = tid; v < WIN / 16; v += THREADS) {
                uint4 x = d4[v];
                Q16[v] = (uint16_t)flags16(eq_flags(x.x, Q4), eq_flags(x.y, Q4), eq_flags(x.z, Q4), eq_flags(x.w, Q4));
            }
            __syncthreads();
            uint32_t par = 0;
            for (int w = tid; w < TILE_WORDS; w += THREADS) par ^= __popc(sm.Qb[w]);
            tile_par = __syncthreads_count(par & 1) & 1;
        }
        // ---- chain 1: quote parity at the tile start.  The tile's own parity is published at once; a tile
        // without quotes does not wait for its predecessors here: it proceeds assuming it starts outside
        // quotes and verifies that after pass 1 (the rare miss redoes the tile from `retry`).
        const uint32_t pin0 = EXACT ? 0u : P.pin0;
        if (tid == 0) st_release_u32(&P.st1[tile], tile == 0 ? (2u | ((pin0 ^ tile_par) << 2)) : (1u | (tile_par << 2)));
        uint32_t pin = tile == 0 ? pin0 : 0;
        bool pin_known = tile == 0;
        if (hasq && !pin_known) {
            if (warp == 0) {
                const uint32_t pv = lookback_parity_w0(P.st1, tile);
                if (lane == 0) { sm.pin = pv; st_release_u32(&P.st1[tile], 2u | ((pv ^ tile_par) << 2)); }
            }
            __syncthreads();
            pin = sm.pin;
            pin_known = true;
        }
    retry:
        if (hasq || pin) {
            // in-quote mask by prefix-XOR of the quote bitmap; terminators are newlines outside quotes
            uint32_t carry = pin;
            for (int r0 = 0; r0 < WIN_WORDS; r0 += THREADS) {
                int w = r0 + tid;
                uint32_t q = (w < WIN_WORDS && hasq) ? sm.Qb[w] : 0;
                uint32_t px = q; px ^= px << 1; px ^= px << 2; px ^= px << 4; px ^= px << 8; px ^= px << 16;
                uint32_t bal = __ballot_sync(0xffffffffu, px >> 31);
                uint32_t before = __popc(bal & lanemask_lt()) & 1;
                if (lane == 0) sm.wpar[warp] = __popc(bal) & 1;
                __syncthreads();
                uint32_t c = carry, tot = 0;
                for (int i = 0; i < THREADS / 32; i++) { if (i < warp) c ^= sm.wpar[i]; tot ^= sm.wpar[i]; }
                uint32_t cin = c ^ before;
                uint32_t iq = (px ^ q) ^ (0u - cin);
                if (w < WIN_WORDS) sm.Tb[w] &= ~iq;  // (Sb keeps quoted newlines/delimiters: only lines with quotes see them)
                carry ^= tot;
                __syncthreads();
            }
        }
        // a virtual terminator at EOF closes a last line that has no newline
        if (eof_in_win && tid == 0) { sm.Tb[rel_n >> 5] |= 1u << (rel_n & 31); sm.Sb[rel_n >> 5] |= 1u << (rel_n & 31); }
        if (eof_in_win) __syncthreads();

        // ---- flat structural index
        uint4 tw = reinterpret_cast<const uint4*>(sm.Tb)[tid];
        {
            const uint4 sw = reinterpret_cast<const uint4*>(sm.Sb)[tid];
            const uint32_t tws[4] = {tw.x, tw.y, tw.z, tw.w}, sws[4] = {sw.x, sw.y, sw.z, sw.w};
            uint32_t cs = __popc(sw.x) + __popc(sw.y) + __popc(sw.z) + __popc(sw.w);
            uint32_t ct = __popc(tw.x) + __popc(tw.y) + __popc(tw.z) + __popc(tw.w);
            uint32_t v = cs | (ct << 16);
            uint32_t inc = warp_incl_scan(v);
            if (lane == 31) sm.wtot[0][warp] = inc;
            // the 64 halo words: one per thread of warps 0-1
            uint32_t hs = 0, ht = 0, hv = 0, hinc = 0;
            if (tid < HALO_WORDS) { hs = sm.Sb[TILE_WORDS + tid]; ht = sm.Tb[TILE_WORDS + tid]; hv = __popc(hs) | (__popc(ht) << 16); }
            if (warp < HALO_WORDS / 32) { hinc = warp_incl_scan(hv); if (lane == 31) sm.wtot[1][warp] = hinc; }
            __syncthreads();
            uint32_t ex = inc - v, tile_tot = 0;
#pragma unroll
            for (int i = 0; i < THREADS / 32; i++) { uint32_t t = sm.wtot[0][i]; if (i < warp) ex += t; tile_tot += t; }
            uint32_t o = ex & 0xffffu, tc = ex >> 16;
            uint32_t halo_tot = 0;
            for (int i = 0; i < HALO_WORDS / 32; i++) halo_tot += sm.wtot[1][i];
            // the totals are known before the expansion: a window that does not fit skips it (dense fallback), one
            // that fits needs no bounds checks
            const bool fits = (tile_tot & 0xffffu) + (halo_tot & 0xffffu) <= (uint32_t)SCAP && (tile_tot >> 16) + (halo_tot >> 16) <= (uint32_t)LCAP;
            if (fits) {
#pragma unroll
                for (int j = 0; j < WPT; j++) {
                    uint32_t m = sws[j];
                    const int pos0 = (tid * WPT + j) * 32;
                    uint32_t tm = tws[j];
                    while (tm) {  // terminators are ~7x sparser than structurals: their ordinals come from a popcount
                        int bpos = __ffs(tm) - 1; tm &= tm - 1;
                        sm.ord[tc++] = (uint16_t)(o + __popc(m & ((1u << bpos) - 1)));
                    }
                    while (m) {
                        int bpos = __ffs(m) - 1; m &= m - 1;
                        sm.sidx[o++] = (uint16_t)(pos0 + bpos);
                    }
                }
            }
            if (fits && tid < HALO_WORDS) {
                uint32_t hex = hinc - hv;
                for (int i = 0; i < warp; i++) hex += sm.wtot[1][i];
                uint32_t o2 = (tile_tot & 0xffffu) + (hex & 0xffffu), tc2 = (tile_tot >> 16) + (hex >> 16);
                uint32_t m = hs;
                const int pos0 = (TILE_WORDS + tid) * 32;
                while (m) {
                    int bpos = __ffs(m) - 1; m &= m - 1;
                    sm.sidx[o2] = (uint16_t)(pos0 + bpos);
                    if ((ht >> bpos) & 1) sm.ord[tc2++] = (uint16_t)o2;
                    o2++;
                }
            }
            if (tid == 0) { sm.nstruct = (tile_tot & 0xffffu) + (halo_tot & 0xffffu); sm.nterm = (tile_tot >> 16) + (halo_tot >> 16); }
            // terminators of the tile proper (tile_tot >> 16) are needed below: stash in wpar[0]
            if (tid == 0) sm.wpar[0] = tile_tot >> 16;
            __syncthreads();
        }
        const int nterm = (int)sm.nterm;
        const bool flat_ok = sm.nstruct <= SCAP && sm.nterm <= LCAP;
        const bool first_owned = tile_base == 0 || (sm.data[PRE - 1] == '\n' && pin == 0);
        // lines 1..m start inside the tile proper (terminator i-1 at position <= TILE-2); line 0 iff first_owned
        const int m_last = (int)sm.wpar[0] - (int)((sm.Tb[TILE_WORDS - 1] >> 31) & 1);
        const int i0 = first_owned ? 0 : 1;
        // (byte-range shards run the guarded 16-column instantiation only: the kernels specialised on the column count —
        // the hot ones — carry none of the shard logic; even its few registers cost them 3-5 %)
        int m_last_v = m_last;
        if (!EXACT && P.own_end != ~0ull && flat_ok)  // a shard that is not the file's last (uniform, cold, out of line)
            m_last_v = shard_tile_tail(P, sm, tile, tile_base, i0, m_last, nterm, rel_n, rel_ds);
        const int nown = m_last_v - i0 + 1;
        const int L = (nown + THREADS - 1) / THREADS;
        ByteSrc src{P.in, P.n, sm.data + PRE, tile_base, tile_base + (uint64_t)rel_n};

        // record-start bits of this thread's 4 words (dense fallback only)
        uint32_t rs[WPT] = {0, 0, 0, 0};
        if (!flat_ok) {
            uint32_t prev = tid == 0 ? (first_owned && tile_base > 0 ? 0x80000000u : 0u) : sm.Tb[tid * WPT - 1];
            rs[0] = (tw.x << 1) | (prev >> 31);
            rs[1] = (tw.y << 1) | (tw.x >> 31);
            rs[2] = (tw.z << 1) | (tw.y >> 31);
            rs[3] = (tw.w << 1) | (tw.z >> 31);
#pragma unroll
            for (int j = 0; j < WPT; j++) {
                const int64_t b0 = (int64_t)(tid * WPT + j) * 32;
                uint32_t keep = 0xffffffffu;
                if (rel_ds > b0) keep = rel_ds >= b0 + 32 ? 0u : (0xffffffffu << (rel_ds - b0));
                if (rel_n64 < b0 + 32) keep &= rel_n64 <= b0 ? 0u : (0xffffffffu >> (32 - (rel_n64 - b0)));
                rs[j] &= keep;
                if ((EXACT || P.ds_is_start) && rel_ds >= b0 && rel_ds < b0 + 32 && rel_ds < rel_n64) rs[j] |= 1u << (rel_ds - b0);
            }
            if (tid == 0 && tile_base == 0 && rel_ds <= 0) rs[0] |= 1u;  // file start
            if (tid == 0) atomicAdd(&P.result->fallback_tiles, 1u);
        }

        // ---- pass 1: count records / surviving rows / bytes per column
        uint32_t nrec = 0, nrow = 0, cb[KMAX];
        uint32_t my_err = 0xffffffffu;  // (local record idx << 16) | kind << 8 | slot
        uint32_t err_rows_local = 0, first_surv_rec = 0;
#pragma unroll
        for (int k = 0; k < KMAX; k++) cb[k] = 0;
        auto account = [&](const Rec<KMAX>& r) -> bool {
            bool survived = false;
            if (r.err != K_OK) {
                if (my_err == 0xffffffffu) { my_err = (nrec << 16) | ((uint32_t)r.err << 8) | (uint32_t)r.err_slot; err_rows_local = nrow; }
            } else if (!HP || eval_pred(P.pred, r.eq)) {
                if (nrow == 0) first_surv_rec = nrec;
                nrow++;
                survived = true;
#pragma unroll
                for (int k = 0; k < KMAX; k++) if (k < (EXACT ? KMAX : P.nsel)) cb[k] += r.slow ? r.f[k] : (r.f[k] >> 16);
            }
            nrec++;
            return survived;
        };
        // pass-1 results of the first RC lines of a thread stay in registers so that pass 2 only writes
        constexpr int RC = KMAX <= 4 ? 6 : (KMAX <= 8 ? 3 : 1);
        uint32_t cf[RC][KMAX];
        uint32_t cmask = 0;
        bool any_slow = false;
        if (flat_ok) {
#pragma unroll
            for (int q = 0; q < RC; q++) {
#pragma unroll
                for (int k = 0; k < KMAX; k++) cf[q][k] = 0;
                const int i = i0 + tid * L + q;
                if (q < L && i <= m_last_v) {
                    Rec<KMAX> r;
                    if (flat_line<KMAX, EXACT, HP>(P, sm, src, lits, lits_in_smem, tile_base, i, nterm, rel_n, rel_ds, hasq, r)) {
                        const bool surv = account(r);
                        if (r.slow) any_slow = true;
                        else if (surv) {
                            cmask |= 1u << q;
#pragma unroll
                            for (int k = 0; k < KMAX; k++) cf[q][k] = r.f[k];
                        }
                    }
                }
            }
            for (int q = RC; q < L; q++) {
                const int i = i0 + tid * L + q;
                if (i > m_last_v) break;
                Rec<KMAX> r;
                if (flat_line<KMAX, EXACT, HP>(P, sm, src, lits, lits_in_smem, tile_base, i, nterm, rel_n, rel_ds, hasq, r)) account(r);
            }
        } else {
#pragma unroll 1
            for (int j = 0; j < WPT; j++) {
                uint32_t m = rs[j];
                while (m) {
                    int b = __ffs(m) - 1; m &= m - 1;
                    Rec<KMAX> r;
                    if (generic_record<KMAX, EXACT, HP>(P, sm, src, tile_base, (tid * WPT + j) * 32 + b, rel_n, r)) account(r);
                }
            }
        }
        if (!pin_known) {  // verify the optimistic assumption "this tile starts outside quotes"
            if (warp == 0) {
                const uint32_t pv = lookback_parity_w0(P.st1, tile);
                if (lane == 0) { sm.pin = pv; st_release_u32(&P.st1[tile], 2u | ((pv ^ tile_par) << 2)); }
            }
            __syncthreads();
            pin = sm.pin;
            pin_known = true;
            if (pin) goto retry;
        }
        // staged output (coalesced stores) needs every row of the tile cached and on the fast path
        const bool staged_pre = !__syncthreads_or(any_slow) && flat_ok && L <= RC;
        // ---- block scan of (records | rows << 16, bytes[k])
        uint32_t v0 = nrec | (nrow << 16);
        uint32_t i0s = warp_incl_scan(v0);
        uint32_t ik[KMAX];
#pragma unroll
        for (int k = 0; k < KMAX; k++) if (k < (EXACT ? KMAX : P.nsel)) ik[k] = warp_incl_scan(cb[k]);
        if (lane == 31) {
            sm.wtot[0][warp] = i0s;
#pragma unroll
            for (int k = 0; k < KMAX; k++) if (k < (EXACT ? KMAX : P.nsel)) sm.wtot[1 + k][warp] = ik[k];
        }
        __syncthreads();
        uint32_t ex0 = i0s - v0, tot0 = 0;
        uint32_t exk[KMAX], totk[KMAX];
#pragma unroll
        for (int i = 0; i < THREADS / 32; i++) { uint32_t t = sm.wtot[0][i]; if (i < warp) ex0 += t; tot0 += t; }
#pragma unroll
        for (int k = 0; k < KMAX; k++) {
            exk[k] = 0; totk[k] = 0;
            if (k < (EXACT ? KMAX : P.nsel)) {
                exk[k] = ik[k] - cb[k];
#pragma unroll
                for (int i = 0; i < THREADS / 32; i++) { uint32_t t = sm.wtot[1 + k][i]; if (i < warp) exk[k] += t; totk[k] += t; }
            }
        }
        const bool staged = staged_pre && (tot0 >> 16) <= (uint32_t)LCAP;
        // ---- chain 2: global prefix of (records, rows, bytes[k])
        {
            unsigned long long mine = 0;  // component `tid` of this tile's totals
            if (tid == 0) mine = tot0 & 0xffffu;
            else if (tid == 1) mine = tot0 >> 16;
#pragma unroll
            for (int k = 0; k < KMAX; k++) if (tid == 2 + k) mine = totk[k];
            unsigned long long* wt = P.words + (uint64_t)tile * NP;
            if (tile == 0) {
                if (tid < NP) { st_relaxed_u64((uint64_t*)(wt + tid), LB_INCL | mine); sm.tile_prefix[tid] = 0; }
                __syncthreads();
            } else {
                if (tid < NP) st_relaxed_u64((uint64_t*)(wt + tid), LB_AGG | mine);
                if (warp == 0) {
                    lookback_totals_w0<KMAX>(P.words, tile, NP, sm);
                    if (lane < NP) st_relaxed_u64((uint64_t*)(wt + lane), LB_INCL | (sm.tile_prefix[lane] + mine));
                }
                __syncthreads();
            }
            if (tile == P.ntiles - 1 && tid < NP) {  // totals + end-of-column sentinels
                const unsigned long long total = sm.tile_prefix[tid] + mine;
                P.result->totals[tid] = total;
                sm.col_total[tid] = total;
            }
            if (tile == P.ntiles - 1) {
                __syncthreads();
                const unsigned long long rows = sm.col_total[1];
                if (tid >= 2 && tid < NP && rows <= P.row_cap) P.out_off[tid - 2][rows] = (uint32_t)sm.col_total[tid];
            }
        }

        // ---- pass 2: write offsets, gather field bytes
        {
            const uint64_t rec0 = sm.tile_prefix[0] + (ex0 & 0xffffu);
            uint64_t row = sm.tile_prefix[1] + (ex0 >> 16);
            if (my_err != 0xffffffffu) {
                unsigned long long key = ((rec0 + (my_err >> 16)) << 16) | (my_err & 0xffffu);
                atomicMin(&P.result->err_key, key);
                atomicMin(&P.result->err_rows, (unsigned long long)(row + err_rows_local));
            }
            if (staged) {
                // Tb|Sb|Qb|sidx|ord are dead once pass 1 has cached every row: their 33 KB hold, per column, the
                // row list (source extent, destination offset) and a staging buffer, so that rows are copied by
                // all threads evenly and HBM sees full, aligned 16-byte stores.
                uint32_t* ost = reinterpret_cast<uint32_t*>(sm.Tb);  // [LCAP + 4] destination offsets of the tile's rows
                uint32_t* wl = ost + (LCAP + 4);                      // [LCAP]     beg | len << 16 of the field
                uint8_t* stage = reinterpret_cast<uint8_t*>(wl + LCAP);
                constexpr uint32_t REGION = 3 * (WIN_WORDS + 4) * 4 + SCAP * 2 + LCAP * 2;
                constexpr uint32_t CH = ((REGION - (2 * LCAP + 4) * 4) / 16) * 16;
                const uint32_t tile_rows = tot0 >> 16;
                const uint64_t row_base = sm.tile_prefix[1];
                const uint32_t osh = (uint32_t)(row_base & 3);
                if (nrow != 0 && row == 0) P.result->first_row_ordinal = rec0 + first_surv_rec;
                // (a run-time column loop -- one copy of the staging code instead of KMAX -- was slower)
#pragma unroll
                for (int k = 0; k < KMAX; k++) {
                    if (k < (EXACT ? KMAX : P.nsel)) {
                        const uint64_t dbase = sm.tile_prefix[2 + k];
                        uint32_t myf[RC], exk_k = 0, totk_k = 0;
#pragma unroll
                        for (int kk = 0; kk < KMAX; kk++) if (kk == k) { exk_k = exk[kk]; totk_k = totk[kk]; }
#pragma unroll
                        for (int q = 0; q < RC; q++) {
                            myf[q] = 0;
#pragma unroll
                            for (int kk = 0; kk < KMAX; kk++) if (kk == k) myf[q] = cf[q][kk];
                        }
                        {
                            uint32_t j = ex0 >> 16, run = exk_k;
#pragma unroll
                            for (int q = 0; q < RC; q++)
                                if ((cmask >> q) & 1) { ost[osh + j] = (uint32_t)(dbase + run); wl[j] = myf[q]; j++; run += myf[q] >> 16; }
                        }
                        __syncthreads();
                        // ---- offsets of this tile's rows
                        {
                            uint32_t* gout = P.out_off[k] + (row_base - osh);
                            const uint64_t rows_ok = P.row_cap > row_base ? P.row_cap - row_base : 0;  // rows of this tile that fit
                            const uint32_t lim_e = osh + (uint32_t)(tile_rows < rows_ok ? tile_rows : rows_ok);
                            for (uint32_t e = tid * 4; e < lim_e; e += THREADS * 4)
                                if (e >= osh && e + 4 <= lim_e) *reinterpret_cast<uint4*>(gout + e) = *reinterpret_cast<const uint4*>(ost + e);
                            if (tid < 8) {  // partial first / last vector: one element per lane
                                const uint32_t tv0 = lim_e & ~3u;
                                const uint32_t x = tid < 4 ? (uint32_t)tid : tv0 + (uint32_t)(tid - 4);
                                const bool head = tid < 4 && osh != 0;
                                const bool tail = tid >= 4 && (lim_e & 3u) != 0 && !(tv0 == 0 && osh != 0);
                                if ((head || tail) && x >= osh && x < lim_e) gout[x] = ost[x];
                            }
                        }
                        // ---- field bytes
                        const uint32_t B = totk_k;
                        const uint32_t r16 = (uint32_t)(dbase & 15);
                        const uint64_t room = P.data_cap[k] > dbase ? P.data_cap[k] - dbase : 0;
                        const uint32_t hi_ok = r16 + (uint32_t)(B < room ? B : room);  // shifted local end of writable bytes
                        uint8_t* gbase = P.out_data[k] + (dbase - r16);
                        for (uint32_t c0 = 0; c0 < r16 + B; c0 += CH) {
                            for (uint32_t j = tid; j < tile_rows; j += THREADS) {
                                const uint32_t f = wl[j], len = f >> 16;
                                const uint32_t st = ost[osh + j] - (uint32_t)dbase + r16;  // shifted tile-local start
                                const uint32_t lo = st > c0 ? st : c0, hi = st + len < c0 + CH ? st + len : c0 + CH;
                                const uint8_t* sp = sm.data + PRE + (f & 0xffffu) - st;
                                for (uint32_t x = lo; x < hi; x++) stage[x - c0] = sp[x];  // (word-wise copies measured slower)
                            }
                            __syncthreads();
                            const uint32_t cend = c0 + CH < r16 + B ? c0 + CH : r16 + B;
                            for (uint32_t x0 = c0 + tid * 16; x0 < cend; x0 += THREADS * 16)
                                if (x0 >= r16 && x0 + 16 <= hi_ok) *reinterpret_cast<uint4*>(gbase + x0) = *reinterpret_cast<const uint4*>(stage + (x0 - c0));
                            // the (at most two) partial vectors at the column's first and last byte: one byte per lane
                            if (tid < 32) {
                                const uint32_t tv0 = hi_ok & ~15u;
                                const uint32_t x = tid < 16 ? (uint32_t)tid : tv0 + (uint32_t)(tid - 16);
                                const bool head = tid < 16 && c0 == 0 && r16 != 0;
                                const bool tail = tid >= 16 && (hi_ok & 15u) != 0 && tv0 >= c0 && tv0 < cend && !(tv0 == 0 && r16 != 0);
                                if ((head || tail) && x >= r16 && x < hi_ok) gbase[x] = stage[x - c0];
                            }
                            __syncthreads();
                        }
                        __syncthreads();
                    }
                }
            } else if (nrow != 0) {
                uint64_t off[KMAX];
#pragma unroll
                for (int k = 0; k < KMAX; k++) off[k] = k < (EXACT ? KMAX : P.nsel) ? sm.tile_prefix[2 + k] + exk[k] : 0;
                uint32_t rec_local = 0;
                auto emit = [&](const Rec<KMAX>& r, uint64_t start_abs) {
                    if (r.err != K_OK || (HP && !eval_pred(P.pred, r.eq))) { rec_local++; return; }
                    if (row == 0) P.result->first_row_ordinal = rec0 + rec_local;
                    const bool row_ok = row < P.row_cap;
                    if (r.slow) {
                        uint64_t dst_off[MAXSEL];
                        uint32_t maxlen[MAXSEL];
                        SlowOut so;
#pragma unroll
                        for (int k = 0; k < KMAX; k++) { dst_off[k] = off[k]; maxlen[k] = r.f[k]; }
                        slow_record<EXACT>(P, src, start_abs, true, dst_off, maxlen, &so);
                    }
#pragma unroll
                    for (int k = 0; k < KMAX; k++) {
                        if (k < (EXACT ? KMAX : P.nsel)) {
                            uint32_t len = r.slow ? r.f[k] : (r.f[k] >> 16);
                            if (row_ok) P.out_off[k][row] = (uint32_t)off[k];
                            if (!r.slow && off[k] + len <= P.data_cap[k]) {
                                const uint8_t* s = sm.data + PRE + (r.f[k] & 0xffffu);
                                uint8_t* d = P.out_data[k] + off[k];
                                for (uint32_t i = 0; i < len; i++) d[i] = s[i];
                            }
                            off[k] += len;
                        }
                    }
                    row++; rec_local++;
                };
                if (flat_ok) {
                    for (int q = 0; q < L; q++) {
                        const int i = i0 + tid * L + q;
                        if (i > m_last_v) break;
                        Rec<KMAX> r;
                        if (flat_line<KMAX, EXACT, HP>(P, sm, src, lits, lits_in_smem, tile_base, i, nterm, rel_n, rel_ds, hasq, r))
                            emit(r, tile_base + (i == 0 ? 0 : (uint64_t)sm.sidx[sm.ord[i - 1]] + 1));
                    }
                } else {
#pragma unroll 1
                    for (int j = 0; j < WPT; j++) {
                        uint32_t m = rs[j];
                        while (m) {
                            int b = __ffs(m) - 1; m &= m - 1;
                            const int ws = (tid * WPT + j) * 32 + b;
                            Rec<KMAX> r;
                            if (generic_record<KMAX, EXACT, HP>(P, sm, src, tile_base, ws, rel_n, r)) emit(r, tile_base + ws);
                        }
                    }
                }
            }
        }
        __syncthreads();  // smem is reused by the next tile
    }
}

// ------------------------------------------------------------------ general reader path (parse_general.cu)
struct GenResult {
    uint64_t nrec_eff = 0, rows = 0;
    uint64_t nrec = 0;  // data records of the input (before filtering)
    unsigned long long err_key = ~0ull;
    std::vector<Buf> offs, datas;
};
void general_header(Ctx* c, const uint8_t* in, uint64_t n, const cpb_reader_opts& o, const Substitution* sub, HeaderOut* dev_out);
void general_parse(Ctx* c, ParseParams P, const cpb_reader_opts& o, const Substitution* sub, uint64_t data_start, GenResult* out);

}  // namespace cpb
