// parse_general.cu — the general (multi-pass) reader path for CommentChar / LazyQuotes / TrimLeadingSpace
// (csvplus.go:976-993 -> encoding/csv Reader.Comment / LazyQuotes / TrimLeadingSpace, SURVEY App. A).
//
// Since round 2 this is the FALLBACK: parse.cu first lets the single-pass scan stand in for it (DESIGN.md §3.4) and comes
// here only when the input needs it — a quote inside a comment line, a real lazy quote, TrimLeadingSpace with a
// white-space delimiter, stand-in bytes of multi-byte runes (subst.cu) — or when CPB_GENERAL_PATH=dfa asks for it.
//
// With these options "inside a quoted field" is no longer the parity of the quote bytes (a comment line
// may contain quotes, lazy quotes are literal), so record boundaries come from a small byte-level DFA
// evaluated in parallel by transition-vector composition (SURVEY App. A.4):
//   g_chunk_vec    one thread per 1 KiB chunk: the composed transition vector of the chunk (8 states x 3 bits)
//   g_block_vec    one vector per block of 256 chunks;  g_chain: the true state at every block start
//   g_chunk_state  the true state at every chunk start
//   g_count/g_emit record starts per chunk -> exclusive scan -> start positions (uint64)
//   g_rec_count    one thread per record: the exact sequential machine (options aware; seq_parse_record_gen lives in
//                  parse_kernels.cuh, the scan's guarded instantiations use it too) -> lengths, Like terms, errors
//   g_rec_emit     offsets + unescaped field bytes
//   g_cut_chunk / g_cut_pick   the stream cut under CommentChar / LazyQuotes (stream.cu, general_cut): per chunk and
//                  entry state the last line end, then the one of the chunk's true entry state
// Exact sizes are known before anything is written (multi-pass: this path trades bandwidth for generality).
// Delimiter / comment are single bytes here: multi-byte runes and the multi-byte Unicode spaces arrive as stand-in bytes.
#include <algorithm>

#include "core.hpp"
#include "pred.cuh"
#include "util.cuh"
#include "parse_kernels.cuh"

namespace cpb {

enum { S_RS = 0, S_RSR = 1, S_CM = 2, S_FS = 3, S_UQ = 4, S_QF = 5, S_QQ = 6, S_QQR = 7 };
enum { C_Q = 0, C_D = 1, C_N = 2, C_R = 3, C_C = 4, C_S = 5, C_O = 6, NCLASS = 7 };
constexpr int GCHUNK = 1024;
constexpr int GBLOCK = 256;  // chunks per block vector

struct CutTokens {  // multi-byte runes the stream cut matches as byte sequences (general_cut)
    int n;
    uint8_t len[MAX_SUB_SEQ], cls[MAX_SUB_SEQ];
    uint8_t b[MAX_SUB_SEQ][4];
};

struct GenOpts {
    uint8_t delim, comment, lazy, trim;
    uint32_t T[NCLASS];  // transition vector per byte class: bits [3s, 3s+3) = next state from state s
    uint32_t sp_bits[8]; // stand-in bytes of the multi-byte Unicode spaces (subst.cu): white space like ' '
    uint32_t has_sp;     // any bit of sp_bits set (the per-byte classifier skips the table otherwise)
    const SubTable* subs;
};

__host__ __device__ inline int gen_class(uint8_t b, const GenOpts& o) {
    if (b == '"') return C_Q;
    if (b == o.delim) return C_D;
    if (b == '\n') return C_N;
    if (b == '\r') return C_R;
    if (o.comment && b == o.comment) return C_C;
    if (b == ' ' || b == '\t' || b == '\v' || b == '\f') return C_S;
    if (o.has_sp && ((o.sp_bits[b >> 5] >> (b & 31)) & 1u)) return C_S;
    return C_O;
}
static int gen_delta(int s, int c, bool trim) {
    switch (s) {
        case S_RS: switch (c) { case C_N: return S_RS; case C_R: return S_RSR; case C_C: return S_CM; case C_Q: return S_QF; case C_D: return S_FS;
                                case C_S: return trim ? S_FS : S_UQ; default: return S_UQ; }
        case S_RSR: return c == C_N ? S_RS : gen_delta(trim ? S_FS : S_UQ, c, trim);
        case S_CM: return c == C_N ? S_RS : S_CM;
        case S_FS: switch (c) { case C_N: return S_RS; case C_D: return S_FS; case C_Q: return S_QF; case C_S: case C_R: return trim ? S_FS : S_UQ; default: return S_UQ; }
        case S_UQ: switch (c) { case C_N: return S_RS; case C_D: return S_FS; default: return S_UQ; }
        case S_QF: return c == C_Q ? S_QQ : S_QF;
        case S_QQ: switch (c) { case C_Q: return S_QF; case C_D: return S_FS; case C_N: return S_RS; case C_R: return S_QQR; default: return S_QF; }
        default: /* S_QQR */ return c == C_N ? S_RS : (c == C_Q ? S_QQ : S_QF);
    }
}
__device__ __forceinline__ uint32_t vec_compose(uint32_t v, uint32_t t) {  // first v, then t
    uint32_t r = 0;
#pragma unroll
    for (int s = 0; s < 8; s++) r |= ((t >> (3 * ((v >> (3 * s)) & 7))) & 7) << (3 * s);
    return r;
}
constexpr uint32_t VEC_ID = 0 | (1 << 3) | (2 << 6) | (3 << 9) | (4 << 12) | (5 << 15) | (6 << 18) | (7 << 21);

__global__ void g_chunk_vec(const uint8_t* __restrict__ in, uint64_t n, GenOpts o, uint32_t* vec) {
    uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t lo = c * GCHUNK;
    if (lo >= n) return;
    uint64_t hi = lo + GCHUNK < n ? lo + GCHUNK : n;
    uint32_t v = VEC_ID;
    for (uint64_t i = lo; i < hi; i++) v = vec_compose(v, o.T[gen_class(in[i], o)]);
    vec[c] = v;
}
__global__ void g_block_vec(const uint32_t* __restrict__ vec, uint64_t nchunks, uint32_t* bvec) {
    uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t lo = b * GBLOCK;
    if (lo >= nchunks) return;
    uint64_t hi = lo + GBLOCK < nchunks ? lo + GBLOCK : nchunks;
    uint32_t v = VEC_ID;
    for (uint64_t i = lo; i < hi; i++) v = vec_compose(v, vec[i]);
    bvec[b] = v;
}
__global__ void g_chain(const uint32_t* __restrict__ bvec, uint64_t nblocks, uint8_t* bstate) {  // one thread
    uint32_t s = S_RS;
    for (uint64_t b = 0; b < nblocks; b++) { bstate[b] = (uint8_t)s; s = (bvec[b] >> (3 * s)) & 7; }
    bstate[nblocks] = (uint8_t)s;  // state at EOF
}
__global__ void g_chunk_state(const uint32_t* __restrict__ vec, uint64_t nchunks, const uint8_t* __restrict__ bstate, uint8_t* cstate) {
    uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t lo = b * GBLOCK;
    if (lo >= nchunks) return;
    uint64_t hi = lo + GBLOCK < nchunks ? lo + GBLOCK : nchunks;
    uint32_t s = bstate[b];
    for (uint64_t i = lo; i < hi; i++) { cstate[i] = (uint8_t)s; s = (vec[i] >> (3 * s)) & 7; }
}
// record starts of one chunk (WRITE: positions, else count).  A line starting with '\r' is a record only if the
// next byte is not '\n' (RSR resolution): its start is the '\r' position, possibly the last byte of the previous chunk.
template <bool WRITE>
__global__ void g_starts(const uint8_t* __restrict__ in, uint64_t n, GenOpts o, const uint8_t* __restrict__ cstate, uint32_t* counts,
                         const uint32_t* __restrict__ offs, unsigned long long* starts) {
    uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t lo = c * GCHUNK;
    if (lo >= n) return;
    uint64_t hi = lo + GCHUNK < n ? lo + GCHUNK : n;
    uint32_t s = cstate[c], k = 0;
    uint64_t w = WRITE ? offs[c] : 0;
    for (uint64_t i = lo; i < hi; i++) {
        int cl = gen_class(in[i], o);
        bool st = (s == S_RS && cl != C_N && cl != C_R && cl != C_C) || (s == S_RSR && cl != C_N);
        if (st) { if (WRITE) starts[w + k] = s == S_RSR ? i - 1 : i; k++; }
        s = (o.T[cl] >> (3 * s)) & 7;
    }
    if (!WRITE) counts[c] = k;
}

struct GenRec { uint32_t lazy, trim; };

// first record (header row / field-count seed), honouring comment and empty lines
__global__ void g_header_kernel(const uint8_t* in, uint64_t n, GenOpts o, HeaderOut* out) {
    ByteSrc src{in, n, nullptr, 0, 0};
    uint64_t pos = 0;
    for (;;) {  // skip comment lines and empty lines (readRecord's loop, SURVEY App. A.2.2)
        int c = src.get(pos);
        if (c < 0) break;
        if (o.comment && c == o.comment) { while (src.get(pos) >= 0 && src.get(pos) != '\n') pos++; if (src.get(pos) == '\n') pos++; continue; }
        if (c == '\n') { pos++; continue; }
        if (c == '\r') {
            int c2 = src.get(pos + 1);
            if (c2 == '\n') { pos += 2; continue; }
            if (c2 < 0) { pos += 1; continue; }
        }
        break;
    }
    out->truncated = 0; out->rec_start = pos; out->sample_bytes = 0; out->sample_newlines = 0; out->samp_lines = 0;
    if (pos >= n) { out->eof = 1; out->err = 0; out->nfields = 0; out->data_start = n; return; }
    HeaderSink sink{out, o.subs};
    SeqResult r = seq_parse_record_gen(src, pos, o.delim, o.lazy, o.trim, o.sp_bits, sink);
    out->eof = 0; out->err = r.err; out->nfields = r.nfields; out->data_start = r.next;
}

// per record: lengths of the selected fields, Like terms, record-level checks; the first failing ordinal
__global__ void g_rec_count(ParseParams P, GenOpts o, const unsigned long long* __restrict__ starts, uint64_t nrec, uint64_t first,
                            uint32_t* flag, uint32_t* lens /*[nsel][nrec]*/) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nrec) return;
    ByteSrc src{P.in, P.n, nullptr, 0, 0};
    SlowSink sink(P, false);
    SeqResult s = seq_parse_record_gen(src, starts[first + i], (int)P.delim, o.lazy, o.trim, o.sp_bits, sink);
    Rec<MAXSEL> r;
    r.err = s.err; r.nf = s.nfields; r.present = sink.present; r.eq = sink.eq; r.slow = true; r.err_slot = 0;
    for (int k = 0; k < MAXSEL; k++) r.f[k] = (k < P.nsel && ((sink.present >> k) & 1)) ? sink.ulen[k] : 0;
    finish_record<MAXSEL, false, true>(P, r);
    bool ok = r.err == K_OK && eval_pred(P.pred, r.eq);
    if (r.err != K_OK) atomicMin(&P.result->err_key, (unsigned long long)((i << 16) | ((uint32_t)r.err << 8) | (uint32_t)r.err_slot));
    flag[i] = ok ? 1u : 0u;
    for (int k = 0; k < P.nsel; k++) lens[(uint64_t)k * nrec + i] = ok ? r.f[k] : 0u;
}
__global__ void g_rec_emit(ParseParams P, GenOpts o, const unsigned long long* __restrict__ starts, uint64_t nrec_eff, uint64_t nrec, uint64_t first,
                           const uint32_t* __restrict__ flag, const uint32_t* __restrict__ rowpos, const uint32_t* __restrict__ lens,
                           const uint32_t* __restrict__ offs /*[nsel][nrec+1] exclusive scans of lens*/) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nrec_eff || !flag[i]) return;
    ByteSrc src{P.in, P.n, nullptr, 0, 0};
    SlowSink sink(P, true);
    const uint32_t row = rowpos[i];
    for (int k = 0; k < P.nsel; k++) {
        const uint32_t off = offs[(uint64_t)k * (nrec + 1) + i];
        sink.dst[k] = P.out_data[k] + off;
        sink.maxlen[k] = lens[(uint64_t)k * nrec + i];
        P.out_off[k][row] = off;
    }
    seq_parse_record_gen(src, starts[first + i], (int)P.delim, o.lazy, o.trim, o.sp_bits, sink);
}
__global__ void g_sentinel(ParseParams P, const uint32_t* __restrict__ offs, uint64_t nrec, uint64_t nrec_eff, uint64_t rows) {
    int k = threadIdx.x;
    if (k < P.nsel) P.out_off[k][rows] = offs[(uint64_t)k * (nrec + 1) + nrec_eff];
}

// Returns the raw pieces of the general parse; parse.cu turns them into a Table and error (shared logic).

// the transition table T of g's trim option; without a comment byte (has_comment false) the comment class is ordinary data
static void gen_transitions(GenOpts& g, bool has_comment) {
    for (int cl = 0; cl < NCLASS; cl++) {
        uint32_t v = 0;
        for (int s = 0; s < 8; s++) v |= (uint32_t)gen_delta(s, (cl == C_C && !has_comment) ? C_O : cl, g.trim) << (3 * s);
        g.T[cl] = v;
    }
}

// the machine of the (single-byte, after subst.cu) reader options and the substitution's stand-in bytes
static GenOpts gen_opts(const cpb_reader_opts& o, const Substitution* sub) {
    GenOpts g{};
    g.delim = (uint8_t)o.delimiter; g.comment = (uint8_t)o.comment; g.lazy = o.lazy_quotes; g.trim = o.trim_leading_space;
    if (sub && sub->table) {
        g.subs = sub->table->as<SubTable>();
        memcpy(g.sp_bits, sub->host_table.space_bits, sizeof g.sp_bits);
        for (int i = 0; i < 8; i++) if (g.sp_bits[i]) g.has_sp = 1;
    }
    gen_transitions(g, g.comment != 0);
    return g;
}

void general_header(Ctx* c, const uint8_t* in, uint64_t n, const cpb_reader_opts& o, const Substitution* sub, HeaderOut* dev_out) {
    const GenOpts g = gen_opts(o, sub);
    KernelTimer kt(c, "csv_header_general", 0);
    g_header_kernel<<<1, 1, 0, c->stream>>>(in, n, g, dev_out);
    CPB_CUDA(cudaGetLastError());
}

void general_parse(Ctx* c, ParseParams P, const cpb_reader_opts& o, const Substitution* sub, uint64_t data_start, GenResult* out) {
    const GenOpts g = gen_opts(o, sub);
    const uint64_t n = P.n;
    const uint64_t nchunks = (n + GCHUNK - 1) / GCHUNK, nblocks = (nchunks + GBLOCK - 1) / GBLOCK;
    Buf vec = dev_alloc(c, nchunks * 4), bvec = dev_alloc(c, nblocks * 4), bstate = dev_alloc(c, nblocks + 1), cstate = dev_alloc(c, nchunks);
    Buf counts = dev_alloc(c, (nchunks + 1) * 4), tot = dev_alloc(c, 8);
    {
        KernelTimer kt(c, "general_boundaries", n * 3, 6);
        g_chunk_vec<<<nblk(nchunks, 128), 128, 0, c->stream>>>(P.in, n, g, vec->as<uint32_t>());
        g_block_vec<<<nblk(nblocks, 128), 128, 0, c->stream>>>(vec->as<uint32_t>(), nchunks, bvec->as<uint32_t>());
        g_chain<<<1, 1, 0, c->stream>>>(bvec->as<uint32_t>(), nblocks, bstate->as<uint8_t>());
        g_chunk_state<<<nblk(nblocks, 128), 128, 0, c->stream>>>(vec->as<uint32_t>(), nchunks, bstate->as<uint8_t>(), cstate->as<uint8_t>());
        g_starts<false><<<nblk(nchunks, 128), 128, 0, c->stream>>>(P.in, n, g, cstate->as<uint8_t>(), counts->as<uint32_t>(), nullptr, nullptr);
        CPB_CUDA(cudaGetLastError());
    }
    exclusive_scan_u32(c, counts->as<uint32_t>(), counts->as<uint32_t>(), nchunks, tot->as<uint64_t>());
    const uint64_t nstarts = read_back<uint64_t>(c, tot->p);
    if (nstarts > 0xfffffff0ull) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "more than 2^32 records in one batch"};
    Buf starts = dev_alloc(c, (nstarts + 1) * 8);
    g_starts<true><<<nblk(nchunks, 128), 128, 0, c->stream>>>(P.in, n, g, cstate->as<uint8_t>(), nullptr, counts->as<uint32_t>(),
                                                             (unsigned long long*)starts->p);
    CPB_CUDA(cudaGetLastError());
    // records before data_start (the header row) are not data: they are the first `first` starts
    uint64_t first = 0;
    if (data_start > 0 && nstarts > 0) first = 1;  // exactly one record (the header) starts before data_start
    const uint64_t nrec = nstarts - first;
    out->nrec = nrec;
    const int nsel = P.nsel;
    out->offs.resize(nsel); out->datas.resize(nsel);
    Buf res = dev_alloc(c, sizeof(ParseResult));
    CPB_CUDA(cudaMemsetAsync(res->p, 0xff, sizeof(ParseResult), c->stream));
    P.result = res->as<ParseResult>();
    if (nrec == 0) {
        for (int k = 0; k < nsel; k++) { out->offs[k] = dev_alloc(c, 4); out->datas[k] = dev_alloc(c, 16); CPB_CUDA(cudaMemsetAsync(out->offs[k]->p, 0, 4, c->stream)); }
        return;
    }
    Buf flag = dev_alloc(c, (nrec + 1) * 4), rowpos = dev_alloc(c, (nrec + 1) * 4), lens = dev_alloc(c, (uint64_t)nsel * nrec * 4 + 4);
    Buf offs = dev_alloc(c, (uint64_t)nsel * (nrec + 1) * 4 + 4), tots = dev_alloc(c, (nsel + 1) * 8);
    {
        KernelTimer kt(c, "general_rec_count", n);
        g_rec_count<<<nblk(nrec, 128), 128, 0, c->stream>>>(P, g, (const unsigned long long*)starts->p, nrec, first, flag->as<uint32_t>(), lens->as<uint32_t>());
        CPB_CUDA(cudaGetLastError());
    }
    out->err_key = read_back<ParseResult>(c, res->p).err_key;
    const uint64_t nrec_eff = out->err_key == ~0ull ? nrec : (uint64_t)(out->err_key >> 16);  // rows before the first failing record
    out->nrec_eff = nrec_eff;
    exclusive_scan_u32(c, flag->as<uint32_t>(), rowpos->as<uint32_t>(), nrec_eff, tots->as<uint64_t>());
    for (int k = 0; k < nsel; k++)
        exclusive_scan_u32(c, lens->as<uint32_t>() + (uint64_t)k * nrec, offs->as<uint32_t>() + (uint64_t)k * (nrec + 1), nrec_eff, tots->as<uint64_t>() + 1 + k);
    const std::vector<uint64_t> ht = read_back<uint64_t>(c, tots->p, nsel + 1);
    out->rows = ht[0];
    for (int k = 0; k < nsel; k++) {
        if (ht[1 + k] > 0xffffffffull) throw DataError{CPB_E_TOO_LARGE, k, 0, false, "a column of this batch exceeds 4 GiB; parse the input in smaller batches"};
        out->offs[k] = dev_alloc(c, (out->rows + 1) * 4);
        out->datas[k] = dev_alloc(c, ht[1 + k] + 16);
        P.out_off[k] = out->offs[k]->as<uint32_t>(); P.out_data[k] = out->datas[k]->as<uint8_t>(); P.data_cap[k] = ht[1 + k];
    }
    {
        KernelTimer kt(c, "general_rec_emit", n);
        if (nrec_eff) g_rec_emit<<<nblk(nrec_eff, 128), 128, 0, c->stream>>>(P, g, (const unsigned long long*)starts->p, nrec_eff, nrec, first, flag->as<uint32_t>(),
                                                                            rowpos->as<uint32_t>(), lens->as<uint32_t>(), offs->as<uint32_t>());
        g_sentinel<<<1, 32, 0, c->stream>>>(P, offs->as<uint32_t>(), nrec, nrec_eff, out->rows);
        CPB_CUDA(cudaGetLastError());
    }
    sync_stream(c);
}

// ------------------------------------------------------------------ stream cut (stream.cu) under CommentChar / LazyQuotes
// The end of the last complete record of a buffer that starts at a record start: 1 + the position of the last '\n' after
// which the machine above is at a record start.  A multi-byte Delimiter / CommentChar / Unicode space (TrimLeadingSpace)
// is matched as its byte sequence: its first byte takes the rune's class and the rest of the sequence is skipped, which
// is what the transcoding of subst.cu gives the general parse.
__device__ __forceinline__ int cut_token_at(const uint8_t* __restrict__ in, uint64_t n, uint64_t i, const CutTokens& tk) {
    for (int q = 0; q < tk.n; q++) {
        if (tk.b[q][0] != in[i] || i + tk.len[q] > n) continue;
        bool ok = true;
        for (int j = 1; j < tk.len[q]; j++) ok = ok && in[i + j] == tk.b[q][j];
        if (ok) return q;
    }
    return -1;
}
// per chunk: its transition vector, and per entry state 1 + the chunk offset of the last '\n' that ends a line (0: none)
__global__ void g_cut_chunk(const uint8_t* __restrict__ in, uint64_t n, GenOpts o, CutTokens tk, uint32_t* vec, uint16_t* last) {
    const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t lo = c * GCHUNK;
    if (lo >= n) return;
    const uint64_t hi = lo + GCHUNK < n ? lo + GCHUNK : n;
    uint64_t i = lo;
    for (uint64_t back = 1; back <= 3 && back <= lo && tk.n; back++) {  // a sequence that started before the chunk covers its first bytes
        const int q = in[lo - back] >= 0x80 ? cut_token_at(in, n, lo - back, tk) : -1;
        if (q >= 0 && lo - back + tk.len[q] > i) i = lo - back + tk.len[q];
    }
    uint32_t v = VEC_ID;
    uint16_t l[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    while (i < hi) {
        const uint8_t b = in[i];
        int cl, step = 1;
        const int q = (b >= 0x80 && tk.n) ? cut_token_at(in, n, i, tk) : -1;
        if (q >= 0) { cl = tk.cls[q]; step = tk.len[q]; }
        else cl = gen_class(b, o);
        v = vec_compose(v, o.T[cl]);
        if (cl == C_N) {
#pragma unroll
            for (int s = 0; s < 8; s++) if (((v >> (3 * s)) & 7) == S_RS) l[s] = (uint16_t)(i - lo + 1);
        }
        i += step;
    }
    vec[c] = v;
#pragma unroll
    for (int s = 0; s < 8; s++) last[c * 8 + s] = l[s];
}
__global__ void g_cut_pick(const uint16_t* __restrict__ last, uint64_t nchunks, const uint8_t* __restrict__ cstate, unsigned long long* cut) {
    const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const uint16_t l = last[c * 8 + cstate[c]];
    if (l) atomicMax(cut, (unsigned long long)(c * GCHUNK + l));
}

void general_cut(Ctx* c, const uint8_t* in, uint64_t n, const cpb_reader_opts& o, uint64_t* cut_dev) {
    GenOpts g{};
    g.delim = o.delimiter < 0x80 ? (uint8_t)o.delimiter : (uint8_t)'"';  // '"' classifies first: a multi-byte delimiter is a token
    g.comment = o.comment < 0x80 ? (uint8_t)o.comment : 0;
    g.lazy = o.lazy_quotes; g.trim = o.trim_leading_space;
    gen_transitions(g, o.comment != 0);
    CutTokens tk{};
    auto add = [&](uint32_t r, int cls) {
        if (r < 0x80 || tk.n >= MAX_SUB_SEQ) return;
        const std::string u = utf8_rune(r);
        tk.len[tk.n] = (uint8_t)u.size();
        for (size_t j = 0; j < u.size(); j++) tk.b[tk.n][j] = (uint8_t)u[j];
        tk.cls[tk.n++] = (uint8_t)cls;
    };
    add(o.delimiter, C_D);
    add(o.comment, C_C);
    if (o.trim_leading_space)
        for (uint32_t r : kUnicodeSpaces) if (r != o.delimiter && r != o.comment) add(r, C_S);
    CPB_CUDA(cudaMemsetAsync(cut_dev, 0, 8, c->stream));
    if (n == 0) return;
    const uint64_t nchunks = (n + GCHUNK - 1) / GCHUNK, nblocks = (nchunks + GBLOCK - 1) / GBLOCK;
    Buf vec = dev_alloc(c, nchunks * 4), last = dev_alloc(c, nchunks * 16), bvec = dev_alloc(c, nblocks * 4), bstate = dev_alloc(c, nblocks + 1),
        cstate = dev_alloc(c, nchunks);
    KernelTimer kt(c, "stream_cut_dfa", n, 5);
    g_cut_chunk<<<nblk(nchunks, 128), 128, 0, c->stream>>>(in, n, g, tk, vec->as<uint32_t>(), last->as<uint16_t>());
    g_block_vec<<<nblk(nblocks, 128), 128, 0, c->stream>>>(vec->as<uint32_t>(), nchunks, bvec->as<uint32_t>());
    g_chain<<<1, 1, 0, c->stream>>>(bvec->as<uint32_t>(), nblocks, bstate->as<uint8_t>());
    g_chunk_state<<<nblk(nblocks, 128), 128, 0, c->stream>>>(vec->as<uint32_t>(), nchunks, bstate->as<uint8_t>(), cstate->as<uint8_t>());
    g_cut_pick<<<nblk(nchunks, 128), 128, 0, c->stream>>>(last->as<uint16_t>(), nchunks, cstate->as<uint8_t>(), (unsigned long long*)cut_dev);
    CPB_CUDA(cudaGetLastError());
}

}  // namespace cpb
