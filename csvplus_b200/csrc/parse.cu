// parse.cu — K1..K4 of SURVEY §2: single-pass CSV scan -> column offsets -> per-column gather into
// string columns, fused with the Like/All/Any/Not filter and row compaction.
//
// Replaces (reference): Reader.Iterate csvplus.go:1080-1146 (hot loop :1117-1138), the stdlib
// encoding/csv.Reader it drives (readRecord/readLine, SURVEY App. A), Row construction
// csvplus.go:1118-1122, Filter csvplus.go:276-286 and Like csvplus.go:1279-1293.
//
// Design (DESIGN.md §parse): the input is read from HBM exactly once.  A persistent grid walks
// 32 KiB tiles in ticket order; each tile (+16 B look-behind, +2 KiB look-ahead) is staged into
// shared memory with one bulk-async copy (TMA 1-D, cp.async.bulk + mbarrier).  Bytes are classified
// with SWAR compares into newline / delimiter bitmaps; quote parity and the running
// (records, rows, bytes-per-column) totals are carried across tiles by two decoupled look-back
// chains.  The set bits of the structural bitmap are expanded into a flat index, so that field j of
// line i is found in O(1); one thread per line counts (pass 1), a block scan + look-back turns counts
// into global output positions, pass 2 writes offsets and gathers field bytes through a staging buffer
// into aligned 16-byte stores.  Records containing quotes (or running past the staged window) take an
// exact sequential state machine that restates Go's readRecord byte for byte.  CommentChar /
// LazyQuotes / TrimLeadingSpace ride on the same scan whenever the input allows (DESIGN.md §3.4);
// parse_general.cu is their multi-pass fallback.
#include <algorithm>
#include <functional>
#include <mutex>

#include "core.hpp"
#include "pred.cuh"
#include "util.cuh"
#include "parse_kernels.cuh"

namespace cpb {

// ------------------------------------------------------------------ host driver
namespace {

const char* kind_text(int k) {
    switch (k) {
        case CPB_E_BARE_QUOTE: return "bare \" in non-quoted-field";
        case CPB_E_QUOTE: return "extraneous or missing \" in quoted-field";
        case CPB_E_FIELD_COUNT: return "wrong number of fields";
        default: return "";
    }
}

template <int KMAX, bool EXACT, bool HP>
void launch_scan_hp(Ctx* c, const ParseParams& P, uint64_t algo_bytes) {
    // function attributes and occupancy are per device: cached per (kernel, device) so that one process may drive
    // several GPUs through several contexts
    static std::mutex mu;
    static int occ_of[64];
    const size_t smem = sizeof(ParseSmem);
    int occ;
    {
        std::lock_guard<std::mutex> lk(mu);
        int& cached = occ_of[c->device & 63];
        if (cached == 0) {
            CPB_CUDA(cudaFuncSetAttribute(csv_scan_kernel<KMAX, EXACT, HP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            int o = 0;
            CPB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, csv_scan_kernel<KMAX, EXACT, HP>, THREADS, smem));
            cached = o < 1 ? 1 : o;
        }
        occ = cached;
    }
    uint32_t grid = (uint32_t)std::min<uint64_t>((uint64_t)c->sm_count * occ, P.ntiles);
    KernelTimer kt(c, "csv_scan", algo_bytes);
    csv_scan_kernel<KMAX, EXACT, HP><<<grid, THREADS, smem, c->stream>>>(P);
    CPB_CUDA(cudaGetLastError());
}

// unfiltered parses run kernels compiled without any Like-comparison code
template <int KMAX, bool EXACT>
void launch_scan(Ctx* c, const ParseParams& P, uint64_t algo_bytes) {
    if (EXACT && P.pred.nops == 0) launch_scan_hp<KMAX, EXACT, false>(c, P, algo_bytes);
    else launch_scan_hp<KMAX, EXACT, true>(c, P, algo_bytes);
}

}  // namespace

bool valid_delim(uint32_t r) {
    return r != 0 && r != '"' && r != '\r' && r != '\n' && r != 0xFFFD && r <= 0x10FFFF && !(r >= 0xD800 && r <= 0xDFFF);
}

// parity of the '"' bytes of [0, n): what a byte-range shard contributes to the quote state of the shards after it
__global__ void quote_parity_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t* out) {
    uint32_t cnt = 0;
    const uint64_t nv = n / 16;
    const uint4* v = reinterpret_cast<const uint4*>(in);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint4 x = v[i];
        cnt += __popc(eq_flags(x.x, 0x22222222u)) + __popc(eq_flags(x.y, 0x22222222u)) + __popc(eq_flags(x.z, 0x22222222u)) +
               __popc(eq_flags(x.w, 0x22222222u));
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) for (uint64_t i = nv * 16; i < n; i++) cnt += in[i] == '"';
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if ((threadIdx.x & 31) == 0 && (cnt & 1)) atomicXor(out, 1u);
}
uint32_t quote_parity(Ctx* c, const uint8_t* in, uint64_t n) {
    Buf out = dev_alloc(c, 4);
    CPB_CUDA(cudaMemsetAsync(out->p, 0, 4, c->stream));
    if (n) {
        KernelTimer kt(c, "quote_parity", n);
        quote_parity_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(in, n, out->as<uint32_t>());
        CPB_CUDA(cudaGetLastError());
    }
    return read_back<uint32_t>(c, out->p) & 1u;
}

std::shared_ptr<Table> parse_csv(Ctx* c, const uint8_t* in_arg, uint64_t n_arg, const cpb_reader_opts& o_arg,
                                 const std::vector<std::pair<std::string, int>>& spec, const cpb_pred* filter,
                                 bool* had_error, DataError* derr, const ShardArgs* sh, const BatchArgs* ba) {
    const uint8_t* in = in_arg;
    uint64_t n = n_arg;
    cpb_reader_opts o = o_arg;
    *had_error = false;
    auto fail = [&](int kind, int col, uint64_t line, const std::string& msg) {
        *had_error = true; *derr = DataError{kind, col, line, true, msg};
    };
    auto empty_table = [&](const std::vector<std::string>& names) {
        auto t = std::make_shared<Table>(); t->ctx = c; t->nrows = 0;
        for (auto& nm : names) {
            Column col; col.name = nm; col.offsets = dev_alloc(c, 4); col.data = dev_alloc(c, 1);
            CPB_CUDA(cudaMemsetAsync(col.offsets->p, 0, 4, c->stream));
            t->cols.push_back(col);
        }
        return t;
    };
    std::vector<std::string> spec_names;
    for (auto& s : spec) spec_names.push_back(s.first);

    // encoding/csv readRecord's option validation (SURVEY App. A.2.1)
    if (o.delimiter == o.comment || !valid_delim(o.delimiter) || (o.comment != 0 && !valid_delim(o.comment))) {
        fail(CPB_E_INVALID_DELIM, -1, 1, "csv: invalid field or comment delimiter");
        return empty_table(spec_names);
    }
    if ((reinterpret_cast<uintptr_t>(in) & 15) != 0) throw ArgError{CPB_ERR_ARG, "device input must be 16-byte aligned"};
    // Multi-byte Delimiter / CommentChar runes and the multi-byte Unicode spaces of TrimLeadingSpace: every occurrence
    // is transcoded to a single byte value the input does not use (subst.cu); from here on the options are single-byte
    Substitution sub;
    if (needs_substitution(o)) {
        sub = substitute_runes(c, in, n, o);
        o.delimiter = sub.delimiter; o.comment = sub.comment;
        if (sub.buffer) { in = sub.buffer->as<uint8_t>(); n = sub.nbytes; }
    }
    const SubTable* subs_dev = sub.table ? sub.table->as<SubTable>() : nullptr;  // (reset below when no stand-in byte is in play)
    // CommentChar / LazyQuotes / TrimLeadingSpace change what "inside quotes" means: they take the general
    // (DFA-composition, multi-pass) path of parse_general.cu; the default options take the single-pass scan.
    const bool special = o.comment != 0 || o.lazy_quotes || o.trim_leading_space;
    // ... unless the input lets the single-pass scan stand in for it (the common case: no stand-in bytes in play, a
    // delimiter TrimLeadingSpace would not eat).  The scan then runs *optimistically*:
    //   * TrimLeadingSpace is exact in it: leading white space of a quote-free line's fields is skipped where the field
    //     extents are computed, lines with quotes take the options-aware sequential machine (seq_parse_record_gen);
    //   * CommentChar: a line whose first byte is the comment byte is not a record; if such a line holds a quote (which the
    //     quote-parity chain has counted) the kernel says so and the parse is redone on the general path;
    //   * LazyQuotes only ever turns ErrBareQuote / ErrQuote of the strict rules into data: the strict scan runs, and only
    //     if its first error is one of those two is the parse redone on the general path.
    // CPB_GENERAL_PATH=dfa forces the general path (tests / timing).
    bool any_standin = false;
    for (int i = 0; i < 8; i++) any_standin = any_standin || sub.host_table.bits[i] != 0;
    const bool delim_is_space = o.delimiter == ' ' || o.delimiter == '\t' || o.delimiter == '\v' || o.delimiter == '\f';
    static const bool force_dfa = getenv("CPB_GENERAL_PATH") != nullptr && !strcmp(getenv("CPB_GENERAL_PATH"), "dfa");
    const bool optimistic = special && !sh && !any_standin && !sub.buffer && !(o.trim_leading_space && delim_is_space) && !force_dfa;
    bool general = special && !optimistic;
    if (sh) {  // a byte-range shard of one file (cpb_parse_csv_shard)
        if (special || sub.table) throw ArgError{CPB_ERR_UNSUPPORTED, "byte-range shards take the default reader options only"};
        if (sh->index > 0 && (o.header_from_first_row || o.num_fields == 0))
            throw ArgError{CPB_ERR_ARG, "shards after the first need the resolved header (name -> index) and an explicit field count"};
        if (sh->own_bytes > n) throw ArgError{CPB_ERR_ARG, "own_bytes exceeds the buffer"};
    }
    if ((reinterpret_cast<uintptr_t>(in) & 15) != 0) throw ArgError{CPB_ERR_ARG, "device input must be 16-byte aligned"};

    // ---- header kernel (first record + sampling)
    Buf hbuf = dev_alloc(c, sizeof(HeaderOut));
    if (special) {
        general_header(c, in, n, o, &sub, hbuf->as<HeaderOut>());
        if (optimistic) {  // the capacity estimate of the single-pass scan needs the newline / field-length samples too
            KernelTimer kt(c, "csv_header", 0);
            csv_header_kernel<<<1, 256, 0, c->stream>>>(in, n, (int)o.delimiter, nullptr, hbuf->as<HeaderOut>(), 1);
            CPB_CUDA(cudaGetLastError());
        }
    } else {
        KernelTimer kt(c, "csv_header", 0);
        csv_header_kernel<<<1, 256, 0, c->stream>>>(in, n, (int)o.delimiter, subs_dev, hbuf->as<HeaderOut>());
        CPB_CUDA(cudaGetLastError());
    }
    HeaderOut* h = (HeaderOut*)c->pinned_scratch(sizeof(HeaderOut));
    // only the fixed part + what is needed: copy the whole struct (≈80 KB) — small next to the input
    CPB_CUDA(cudaMemcpyAsync(h, hbuf->p, sizeof(HeaderOut), cudaMemcpyDeviceToHost, c->stream));
    sync_stream(c);
    // the first record's bytes are kept only for its names: its field count and end are exact at any size, so a long first
    // record matters only when it is the header row (not for AssumeHeader, nor for a later batch of a stream)
    if (h->truncated && o.header_from_first_row) throw ArgError{CPB_ERR_UNSUPPORTED, "header row larger than 16 KiB / 1024 fields"};
    if (ba) { *ba->records = 0; *ba->no_record = h->eof != 0; }

    // ---- header resolution: makeHeader, csvplus.go:1149-1206
    std::vector<std::pair<std::string, int>> cols;  // output columns (name, field index)
    uint64_t data_start = 0;
    const bool hdr = o.header_from_first_row != 0;
    int first_nfields = h->eof ? 0 : h->nfields;
    if (hdr) {
        if (h->eof) { fail(CPB_E_EOF, -1, 1, "EOF"); return empty_table(spec_names); }
        if (h->err) { fail(h->err, -1, 1, kind_text(h->err)); return empty_table(spec_names); }
        if (o.num_fields > 0 && h->nfields != o.num_fields) { fail(CPB_E_FIELD_COUNT, -1, 1, kind_text(CPB_E_FIELD_COUNT)); return empty_table(spec_names); }
        std::vector<std::string> line;
        size_t offb = 0;
        for (int i = 0; i < h->nfields; i++) { line.emplace_back((const char*)h->bytes + offb, h->field_len[i]); offb += h->field_len[i]; }
        if (spec.empty()) {  // :1160-1168: later duplicates overwrite earlier ones
            for (size_t i = 0; i < line.size(); i++) {
                bool found = false;
                for (auto& cc : cols) if (cc.first == line[i]) { cc.second = (int)i; found = true; }
                if (!found) cols.emplace_back(line[i], (int)i);
            }
        } else {
            std::vector<int> got(spec.size(), -1);
            for (size_t i = 0; i < line.size(); i++) {  // :1174-1183
                for (size_t s = 0; s < spec.size(); s++) {
                    if (spec[s].first != line[i]) continue;
                    if (spec[s].second == -1 || spec[s].second == (int)i) got[s] = (int)i;
                    else {
                        fail(CPB_E_MISPLACED_COLUMN, (int)s, 1,
                             "misplaced column " + go_quote(line[i]) + ": expected at pos. " + std::to_string(spec[s].second) +
                                 ", but found at pos. " + std::to_string(i));
                        return empty_table(spec_names);
                    }
                }
            }
            std::vector<std::string> missing; int first_missing = -1;
            for (size_t s = 0; s < spec.size(); s++) if (got[s] < 0) { missing.push_back(spec[s].first); if (first_missing < 0) first_missing = (int)s; }
            if (!missing.empty()) {  // :1186-1202
                std::string m = missing.size() > 1 ? "columns not found: " : "column not found: ";
                for (size_t i = 0; i < missing.size(); i++) { if (i) m += ", "; m += missing[i]; }
                fail(CPB_E_COLUMN_NOT_FOUND, first_missing, 1, m);
                return empty_table(spec_names);
            }
            for (size_t s = 0; s < spec.size(); s++) cols.emplace_back(spec[s].first, got[s]);
        }
        data_start = h->data_start;
    } else {
        if (spec.empty()) throw ArgError{CPB_ERR_ARG, "Empty header spec"};  // csvplus.go:999-1001
        for (auto& s : spec) { if (s.second < 0) throw ArgError{CPB_ERR_ARG, "header spec: negative index for column " + s.first}; cols.push_back(s); }
        data_start = sh && sh->index > 0 ? 1 : 0;  // a record starting at byte 0 of a later shard belongs to the shard before it
    }
    std::vector<std::string> names;
    for (auto& cc : cols) names.push_back(cc.first);
    // DataSourceError.Line of data record 0 (csvplus.go:1102-1109); a later batch of a stream continues the count
    const uint64_t line_base = ba ? ba->line_base : (hdr ? 2 : 1);

    // ---- slots: distinct field indices, ascending
    std::vector<int> fields;
    for (auto& cc : cols) fields.push_back(cc.second);
    std::sort(fields.begin(), fields.end());
    fields.erase(std::unique(fields.begin(), fields.end()), fields.end());
    if ((int)fields.size() > MAXSEL) {
        // More than 16 distinct fields (e.g. Take(FromFile(x)) of a wide file, csvplus.go:1160-1168 takes every column):
        // the scan runs once per group of columns over the same input — each pass extracts its group plus the columns
        // the predicate compares, so every pass delivers the same rows (and the same error) — and the groups' columns are
        // put together in the caller's order.  The reference handles any width; so does this, at one read per 16 columns.
        std::vector<std::string> pred_names;
        {
            std::function<void(const cpb_pred*)> walk = [&](const cpb_pred* p) {
                if (!p) return;
                if (p->op == CPB_PRED_LIKE) { for (int i = 0; i < p->n; i++) pred_names.push_back(to_string(p->keys[i])); }
                else for (int i = 0; i < p->n; i++) walk(p->children[i]);
            };
            walk(filter);
        }
        std::vector<std::pair<std::string, int>> pred_cols;
        for (auto& cc : cols)
            if (std::find(pred_names.begin(), pred_names.end(), cc.first) != pred_names.end()) pred_cols.push_back(cc);
        std::vector<int> pf;
        for (auto& pc : pred_cols) pf.push_back(pc.second);
        std::sort(pf.begin(), pf.end()); pf.erase(std::unique(pf.begin(), pf.end()), pf.end());
        if ((int)pf.size() >= MAXSEL) throw ArgError{CPB_ERR_UNSUPPORTED, "a predicate over 16 or more columns of one fused parse"};
        auto merged = std::make_shared<Table>();
        std::vector<Column> out_cols(cols.size());
        std::vector<char> have(cols.size(), 0);
        size_t next = 0;
        bool first_pass = true;
        while (next < cols.size()) {
            std::vector<std::pair<std::string, int>> group = pred_cols;
            std::vector<int> gf = pf;
            std::vector<size_t> members;
            for (; next < cols.size(); next++) {
                if (have[next]) continue;
                const bool known = std::find(gf.begin(), gf.end(), cols[next].second) != gf.end();
                if (!known && (int)gf.size() >= MAXSEL) break;
                if (!known) gf.push_back(cols[next].second);
                if (std::find_if(group.begin(), group.end(), [&](auto& g) { return g.first == cols[next].first; }) == group.end()) group.push_back(cols[next]);
                members.push_back(next);
            }
            bool he = false; DataError de{};
            auto part = parse_csv(c, in_arg, n_arg, o_arg, group, filter, &he, &de, sh, ba);
            if (first_pass) {
                *had_error = he; *derr = de;
                merged->ctx = c; merged->nrows = part->nrows; merged->first_line = part->first_line; merged->record_fields = part->record_fields;
                first_pass = false;
            } else if (part->nrows != merged->nrows) throw ArgError{CPB_ERR_CUDA, "internal: column groups of one parse disagree on the row count"};
            for (size_t m : members) {
                const int k = part->find(cols[m].first);
                if (k < 0) throw ArgError{CPB_ERR_CUDA, "internal: column group lost a column"};
                out_cols[m] = part->cols[k]; have[m] = 1;
            }
        }
        for (size_t i = 0; i < cols.size(); i++) { merged->cols.push_back(out_cols[i]); merged->src_field.push_back(cols[i].second); }
        return merged;
    }
    std::vector<int> col_slot;
    for (auto& cc : cols) col_slot.push_back((int)(std::lower_bound(fields.begin(), fields.end(), cc.second) - fields.begin()));
    const int nsel = (int)fields.size();

    Compiled comp;
    compile_pred(filter, [&](const std::string& key) {
        int col = -1;
        for (size_t i = 0; i < names.size(); i++) if (names[i] == key) col = (int)i;
        return col < 0 ? -1 : col_slot[col];
    }, comp);

    ParseParams P{};
    P.in = in; P.n = n; P.data_start = data_start; P.delim = o.delimiter;
    P.expect_fields = o.num_fields > 0 ? o.num_fields : (o.num_fields == 0 ? first_nfields : 0);
    P.pad_missing = o.num_fields < 0;
    P.nsel = nsel;
    for (int k = 0; k < nsel; k++) P.sel_field[k] = fields[k];
    P.pred = comp.prog;
    for (int t = 0; t < comp.prog.nterms; t++) P.slot_terms[comp.prog.term_col[t]] |= 1u << t;
    P.ntiles = data_start >= n ? 0 : (uint32_t)((n + TILE - 1) / TILE);
    P.own_end = ~0ull;
    { static const bool off = getenv("CPB_NO_L2_AHEAD") != nullptr; P.l2_ahead = off ? 0u : 1u; }
    P.ds_is_start = !(sh && sh->index > 0);
    if (sh) {
        P.pin0 = sh->pin0 & 1u;
        if (!sh->is_last) {  // records that start after own_bytes are the next shard's; the tiles past that byte are never visited
            P.own_end = sh->own_bytes;
            if (P.ntiles) P.ntiles = (uint32_t)std::min<uint64_t>(P.ntiles, sh->own_bytes / TILE + 1);
        }
    }
    P.subs = optimistic ? nullptr : subs_dev;
    P.trim = optimistic && o.trim_leading_space ? 1u : 0u;
    P.comment = optimistic ? o.comment : 0u;

    if (P.ntiles == 0) {
        if (sh && sh->records) *sh->records = 0;
        auto t = empty_table(names);
        for (auto& cc : cols) t->src_field.push_back(cc.second);
        t->record_fields = first_nfields;
        return t;
    }

    Buf lits = dev_alloc(c, comp.lits.size() + 16);
    if (!comp.lits.empty())  // pageable source: the runtime stages it before returning
        CPB_CUDA(cudaMemcpyAsync(lits->p, comp.lits.data(), comp.lits.size(), cudaMemcpyHostToDevice, c->stream));
    P.lits = lits->as<uint8_t>();
    P.lits_len = (uint32_t)comp.lits.size();

    // the result of either path: the table of the slot buffers, and the error err_key names (ordinal << 16 | kind << 8 |
    // slot of the first failing record, ~0 = none)
    auto finish = [&](int64_t nrows, uint64_t first_line, uint64_t err_key, const std::vector<Buf>& offs, const std::vector<Buf>& datas) {
        auto t = std::make_shared<Table>();
        t->ctx = c; t->nrows = nrows; t->first_line = first_line; t->record_fields = first_nfields;
        if (err_key != ~0ull) {
            uint64_t ordinal = err_key >> 16;
            int kind = (int)((err_key >> 8) & 0xff), slot = (int)(err_key & 0xff);
            if (kind == CPB_E_COLUMN_INDEX) {
                int ci = 0;
                for (size_t i = 0; i < cols.size(); i++) if (col_slot[i] == slot) { ci = (int)i; break; }
                fail(kind, ci, line_base + ordinal,
                     "column not found: " + go_quote(cols[ci].first) + " (" + std::to_string(cols[ci].second) + ")");  // csvplus.go:1128
            } else fail(kind, -1, line_base + ordinal, kind_text(kind));
        }
        for (size_t i = 0; i < cols.size(); i++) {
            Column col; col.name = cols[i].first; col.offsets = offs[col_slot[i]]; col.data = datas[col_slot[i]];
            t->cols.push_back(col);
            t->src_field.push_back(cols[i].second);
        }
        return t;
    };
    auto run_general = [&]() -> std::shared_ptr<Table> {
        GenResult gr;
        P.subs = subs_dev; P.trim = 0; P.comment = 0;
        general_parse(c, P, o, &sub, data_start, &gr);
        if (ba) *ba->records = gr.nrec;
        return finish((int64_t)gr.rows, line_base, gr.err_key, gr.offs, gr.datas);
    };
    if (general) return run_general();

    // ---- capacities (exact totals always come back; overflow => one exact rerun)
    const int NP = 2 + nsel;
    const uint64_t sample_bytes = h->sample_bytes, sample_newlines = h->sample_newlines;  // h aliases pinned scratch
    double avg = sample_newlines ? (double)sample_bytes / (double)sample_newlines : (double)n;
    if (avg < 2) avg = 2;
    // Capacities are rounded up to size classes so that successive batches of slightly different sizes request
    // identical blocks and are served from the stream-ordered pool instead of mapping fresh memory.
    auto size_class = [](uint64_t v, uint64_t gran) { return (v + gran - 1) / gran * gran; };
    const uint64_t body = n - data_start;
    uint64_t row_cap = (uint64_t)((double)body / avg * 1.10) + 4096;
    if (row_cap > body / 2 + 2) row_cap = body / 2 + 2;
    row_cap = size_class(row_cap, 1u << 20);
    // per-column bytes from the sampled mean field lengths (naive split of ~768 sampled lines); the worst case
    // (all of the input) when a field was not sampled.  An underestimate costs one exact rerun, never correctness.
    std::vector<uint64_t> data_cap(nsel, std::min<uint64_t>(body, 0xffffffffull));
    const uint64_t samp_lines = h->samp_lines;
    for (int k = 0; k < nsel && samp_lines >= 16; k++) {
        if (fields[k] >= HDR_SAMPLE_FIELDS) continue;
        double mean = (double)h->samp_field_bytes[fields[k]] / (double)samp_lines;
        uint64_t est = (uint64_t)((double)row_cap * mean * 1.25) + (4u << 20);
        data_cap[k] = std::min<uint64_t>(data_cap[k], size_class(est, 32u << 20));
    }

    Buf state = dev_alloc(c, (size_t)P.ntiles * (8 + 16ull * NP) + 64 + sizeof(ParseResult));
    std::vector<Buf> offs(nsel), datas(nsel);
    ParseResult res{};
    for (int attempt = 0; attempt < 2; attempt++) {
        for (int k = 0; k < nsel; k++) {
            offs[k] = dev_alloc(c, (row_cap + 1) * 4);
            datas[k] = dev_alloc(c, data_cap[k] + 16);
            P.out_off[k] = offs[k]->as<uint32_t>(); P.out_data[k] = datas[k]->as<uint8_t>(); P.data_cap[k] = data_cap[k];
        }
        P.row_cap = row_cap;
        uint8_t* sp = state->as<uint8_t>();
        P.result = reinterpret_cast<ParseResult*>(sp); sp += sizeof(ParseResult);
        P.ticket = reinterpret_cast<uint32_t*>(sp); sp += 64;
        P.words = reinterpret_cast<unsigned long long*>(sp); sp += (size_t)P.ntiles * NP * 8;
        P.st1 = reinterpret_cast<uint32_t*>(sp);
        // zero: result totals, ticket, status words; err fields = ~0
        CPB_CUDA(cudaMemsetAsync(state->p, 0, sizeof(ParseResult) + 64, c->stream));
        CPB_CUDA(cudaMemsetAsync(&P.result->err_key, 0xff, 24, c->stream));
        CPB_CUDA(cudaMemsetAsync(P.words, 0, (size_t)P.ntiles * (NP * 8 + 4), c->stream));
        uint64_t algo = n;  // S_in; S_out added by the caller of stats from the totals
        if (P.trim || P.comment) {  // optimistic TrimLeadingSpace / CommentChar: the guarded instantiations carry the extra checks
            if (nsel <= 4) launch_scan<4, false>(c, P, algo);
            else if (nsel <= 8) launch_scan<8, false>(c, P, algo);
            else launch_scan<16, false>(c, P, algo);
        } else
        switch (sh ? 99 : nsel) {  // kernels specialised on the exact number of extracted columns (no per-column guards); shards: the guarded one
            case 1: launch_scan<1, true>(c, P, algo); break;
            case 2: launch_scan<2, true>(c, P, algo); break;
            case 3: launch_scan<3, true>(c, P, algo); break;
            case 4: launch_scan<4, true>(c, P, algo); break;
            case 5: launch_scan<5, true>(c, P, algo); break;
            case 6: launch_scan<6, true>(c, P, algo); break;
            case 7: launch_scan<7, true>(c, P, algo); break;
            case 8: launch_scan<8, true>(c, P, algo); break;
            default: launch_scan<16, false>(c, P, algo); break;
        }
        res = read_back<ParseResult>(c, P.result);
        if (optimistic) {  // did the shortcut hold?
            const int ekind = res.err_key == ~0ull ? 0 : (int)((res.err_key >> 8) & 0xff);
            const bool lazy_matters = o.lazy_quotes && (ekind == CPB_E_BARE_QUOTE || ekind == CPB_E_QUOTE);
            if (res.need_general || lazy_matters) {
                offs.clear(); datas.clear();
                return run_general();
            }
        }
        bool overflow = res.totals[1] > row_cap;
        for (int k = 0; k < nsel; k++) {
            if (res.totals[2 + k] > 0xffffffffull)
                throw DataError{CPB_E_TOO_LARGE, k, 0, false, "a column of this batch exceeds 4 GiB; parse the input in smaller batches"};
            if (res.totals[2 + k] > data_cap[k]) overflow = true;
        }
        if (!overflow) break;
        if (attempt == 1) throw ArgError{CPB_ERR_CUDA, "parse capacity overflow after exact resize"};
        row_cap = res.totals[1] + 1;
        for (int k = 0; k < nsel; k++) data_cap[k] = res.totals[2 + k];
    }
    if (ba) *ba->records = res.totals[0];
    if (sh) {
        if (sh->records) *sh->records = res.totals[0];
        if (!sh->is_last && res.eof_hit)
            throw ArgError{CPB_ERR_ARG, "shard look-ahead too small: a record that starts in this shard runs past the end of the buffer"};
    }
    // fold S_out into the algorithmic bytes of the scan record
    if (c->stats_on) {
        uint64_t s_out = 0;
        for (int k = 0; k < nsel; k++) s_out += res.totals[2 + k] + 4 * (res.totals[1] + 1);
        c->drain_events();
        c->stats["csv_scan"].bytes += s_out;
    }

    return finish((int64_t)(res.err_key != ~0ull ? res.err_rows : res.totals[1]),
                  line_base + (res.first_row_ordinal == ~0ull ? 0 : res.first_row_ordinal), res.err_key, offs, datas);
}

}  // namespace cpb
