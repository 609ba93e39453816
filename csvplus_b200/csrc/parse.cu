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
//
// Host driver (parse_csv), one step per function: option validation and the multi-byte rune substitution; the route
// (the scan, the scan checking the options on the fly, or the general path), chosen once; the header pass and its
// readback; the column resolution of makeHeader / AssumeHeader; for more than 16 columns, one parse per group of
// columns; the scan with its capacity estimate and exact rerun, or the general path; the table and error of the result.
// Every call returns one Parsed value: the rows before the first data error, that error and the record counts.
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

// ------------------------------------------------------------------ parse_csv, step by step
namespace {

using Spec = std::vector<std::pair<std::string, int>>;  // (column name, field index; -1: wherever the header row has it)

enum class Route {
    scan,          // the single-pass scan
    checked_scan,  // the single-pass scan checks the options on the fly; the general path redoes the parse if they matter
    general,       // the general (DFA-composition, multi-pass) path of parse_general.cu
};

// CommentChar / LazyQuotes / TrimLeadingSpace change what "inside quotes" means: they take the general path; the
// default options take the scan.  Unless the input lets the scan stand in for the general path (the common case: no
// stand-in bytes in play, a delimiter TrimLeadingSpace would not eat): the scan then runs *optimistically*:
//   * TrimLeadingSpace is exact in it: leading white space of a quote-free line's fields is skipped where the field
//     extents are computed, lines with quotes take the options-aware sequential machine (seq_parse_record_gen);
//   * CommentChar: a line whose first byte is the comment byte is not a record; if such a line holds a quote (which the
//     quote-parity chain has counted) the kernel says so and the parse is redone on the general path;
//   * LazyQuotes only ever turns ErrBareQuote / ErrQuote of the strict rules into data: the strict scan runs, and only
//     if its first error is one of those two is the parse redone on the general path.
// CPB_GENERAL_PATH=dfa forces the general path (tests / timing).  o: the options after the rune substitution.
Route choose_route(const cpb_reader_opts& o, const Substitution& sub, bool shard) {
    if (o.comment == 0 && !o.lazy_quotes && !o.trim_leading_space) return Route::scan;
    bool any_standin = false;
    for (int i = 0; i < 8; i++) any_standin = any_standin || sub.host_table.bits[i] != 0;
    const bool delim_is_space = o.delimiter == ' ' || o.delimiter == '\t' || o.delimiter == '\v' || o.delimiter == '\f';
    static const bool force_dfa = getenv("CPB_GENERAL_PATH") != nullptr && !strcmp(getenv("CPB_GENERAL_PATH"), "dfa");
    const bool checked = !shard && !any_standin && !sub.buffer && !(o.trim_leading_space && delim_is_space) && !force_dfa;
    return checked ? Route::checked_scan : Route::general;
}

const SubTable* dev_subs(const Substitution& sub) { return sub.table ? sub.table->as<SubTable>() : nullptr; }

std::shared_ptr<Table> empty_table(Ctx* c, const Spec& cols) {
    auto t = std::make_shared<Table>(); t->ctx = c; t->nrows = 0;
    for (auto& cc : cols) {
        Column col; col.name = cc.first; col.offsets = dev_alloc(c, 4); col.data = dev_alloc(c, 1);
        CPB_CUDA(cudaMemsetAsync(col.offsets->p, 0, 4, c->stream));
        t->cols.push_back(col);
    }
    return t;
}

// The header pass: the first record (its field count and end, its fields for a header row) and the samples of the
// capacity estimate, read back with one synchronisation.  What it returns is a host copy: the pinned scratch it was read
// through is reused by the next readback.
HeaderOut read_header(Ctx* c, const uint8_t* in, uint64_t n, const cpb_reader_opts& o, const Substitution& sub, Route route) {
    Buf hbuf = dev_alloc(c, sizeof(HeaderOut));
    if (route != Route::scan) general_header(c, in, n, o, &sub, hbuf->as<HeaderOut>());
    if (route != Route::general) {  // (the checked scan's capacity estimate needs the newline / field-length samples too)
        KernelTimer kt(c, "csv_header", 0);
        if (route == Route::scan) csv_header_kernel<<<1, 256, 0, c->stream>>>(in, n, (int)o.delimiter, dev_subs(sub), hbuf->as<HeaderOut>());
        else csv_header_kernel<<<1, 256, 0, c->stream>>>(in, n, (int)o.delimiter, nullptr, hbuf->as<HeaderOut>(), 1);
        CPB_CUDA(cudaGetLastError());
    }
    HeaderOut h = read_back<HeaderOut>(c, hbuf->p);
    // the first record's bytes are kept only for its names: its field count and end are exact at any size, so a long first
    // record matters only when it is the header row (not for AssumeHeader, nor for a later batch of a stream)
    if (h.truncated && o.header_from_first_row) throw ArgError{CPB_ERR_UNSUPPORTED, "header row larger than 16 KiB / 1024 fields"};
    return h;
}

// The output columns (name, field index) into cols: makeHeader (csvplus.go:1149-1206) over the header row, or the
// columns AssumeHeader names.  Returns the error the reference reports for the header row.
std::optional<DataError> resolve_columns(const HeaderOut& h, const cpb_reader_opts& o, const Spec& spec, Spec& cols) {
    if (!o.header_from_first_row) {
        if (spec.empty()) throw ArgError{CPB_ERR_ARG, "Empty header spec"};  // csvplus.go:999-1001
        for (auto& s : spec) { if (s.second < 0) throw ArgError{CPB_ERR_ARG, "header spec: negative index for column " + s.first}; cols.push_back(s); }
        return std::nullopt;
    }
    auto fail = [](int kind, int col, const std::string& msg) { return DataError{kind, col, 1, true, msg}; };
    if (h.eof) return fail(CPB_E_EOF, -1, "EOF");
    if (h.err) return fail(h.err, -1, kind_text(h.err));
    if (o.num_fields > 0 && h.nfields != o.num_fields) return fail(CPB_E_FIELD_COUNT, -1, kind_text(CPB_E_FIELD_COUNT));
    std::vector<std::string> line;
    size_t offb = 0;
    for (int i = 0; i < h.nfields; i++) { line.emplace_back((const char*)h.bytes + offb, h.field_len[i]); offb += h.field_len[i]; }
    if (spec.empty()) {  // :1160-1168: later duplicates overwrite earlier ones
        for (size_t i = 0; i < line.size(); i++) {
            bool found = false;
            for (auto& cc : cols) if (cc.first == line[i]) { cc.second = (int)i; found = true; }
            if (!found) cols.emplace_back(line[i], (int)i);
        }
        return std::nullopt;
    }
    std::vector<int> got(spec.size(), -1);
    for (size_t i = 0; i < line.size(); i++) {  // :1174-1183
        for (size_t s = 0; s < spec.size(); s++) {
            if (spec[s].first != line[i]) continue;
            if (spec[s].second == -1 || spec[s].second == (int)i) got[s] = (int)i;
            else
                return fail(CPB_E_MISPLACED_COLUMN, (int)s, "misplaced column " + go_quote(line[i]) + ": expected at pos. " +
                                                                std::to_string(spec[s].second) + ", but found at pos. " + std::to_string(i));
        }
    }
    std::vector<std::string> missing; int first_missing = -1;
    for (size_t s = 0; s < spec.size(); s++) if (got[s] < 0) { missing.push_back(spec[s].first); if (first_missing < 0) first_missing = (int)s; }
    if (!missing.empty()) {  // :1186-1202
        std::string m = missing.size() > 1 ? "columns not found: " : "column not found: ";
        for (size_t i = 0; i < missing.size(); i++) { if (i) m += ", "; m += missing[i]; }
        return fail(CPB_E_COLUMN_NOT_FOUND, first_missing, m);
    }
    for (size_t s = 0; s < spec.size(); s++) cols.emplace_back(spec[s].first, got[s]);
    return std::nullopt;
}

// More than 16 distinct fields (e.g. Take(FromFile(x)) of a wide file, csvplus.go:1160-1168 takes every column): the
// parse runs once per group of columns over the same input — each pass extracts its group plus the columns the predicate
// compares, so every pass delivers the same rows (and the same error) — and the groups' columns are put together in the
// caller's order.  The reference handles any width; so does this, at one read per 16 columns.
Parsed parse_column_groups(Ctx* c, const uint8_t* in, uint64_t n, const cpb_reader_opts& o, const Spec& cols, const cpb_pred* filter,
                           uint64_t line_base, const ShardArgs* sh) {
    std::vector<std::string> pred_names;
    std::function<void(const cpb_pred*)> walk = [&](const cpb_pred* p) {
        if (!p) return;
        if (p->op == CPB_PRED_LIKE) { for (int i = 0; i < p->n; i++) pred_names.push_back(to_string(p->keys[i])); }
        else for (int i = 0; i < p->n; i++) walk(p->children[i]);
    };
    walk(filter);
    Spec pred_cols;
    for (auto& cc : cols)
        if (std::find(pred_names.begin(), pred_names.end(), cc.first) != pred_names.end()) pred_cols.push_back(cc);
    std::vector<int> pf;
    for (auto& pc : pred_cols) pf.push_back(pc.second);
    std::sort(pf.begin(), pf.end()); pf.erase(std::unique(pf.begin(), pf.end()), pf.end());
    if ((int)pf.size() >= MAXSEL) throw ArgError{CPB_ERR_UNSUPPORTED, "a predicate over 16 or more columns of one fused parse"};
    Parsed out;  // the first pass's error and record counts, with the merged table
    std::vector<Column> out_cols(cols.size());
    std::vector<char> have(cols.size(), 0);
    size_t next = 0;
    while (next < cols.size()) {
        Spec group = pred_cols;
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
        const Parsed part = parse_csv(c, in, n, o, group, filter, line_base, sh);
        if (!out.table) {
            out = part;
            out.table = std::make_shared<Table>();
            out.table->ctx = c; out.table->nrows = part.table->nrows; out.table->first_line = part.table->first_line;
            out.table->record_fields = part.table->record_fields;
        } else if (part.table->nrows != out.table->nrows) throw ArgError{CPB_ERR_CUDA, "internal: column groups of one parse disagree on the row count"};
        for (size_t m : members) {
            const int k = part.table->find(cols[m].first);
            if (k < 0) throw ArgError{CPB_ERR_CUDA, "internal: column group lost a column"};
            out_cols[m] = part.table->cols[k]; have[m] = 1;
        }
    }
    for (size_t i = 0; i < cols.size(); i++) { out.table->cols.push_back(out_cols[i]); out.table->src_field.push_back(cols[i].second); }
    return out;
}

int slot_of(const ParseParams& P, int field) { return (int)(std::lower_bound(P.sel_field, P.sel_field + P.nsel, field) - P.sel_field); }

// The result of either path: the table of the slot buffers, and the error err_key names (ordinal << 16 | kind << 8 |
// slot of the first failing record, ~0 = none).
Parsed finish(Ctx* c, const HeaderOut& h, const Spec& cols, const ParseParams& P, uint64_t line_base, int64_t nrows, uint64_t first_line,
              uint64_t err_key, const std::vector<Buf>& offs, const std::vector<Buf>& datas) {
    Parsed out{std::make_shared<Table>()};
    Table& t = *out.table;
    t.ctx = c; t.nrows = nrows; t.first_line = first_line; t.record_fields = h.eof ? 0 : h.nfields;
    out.no_record = h.eof != 0;
    if (err_key != ~0ull) {
        const uint64_t line = line_base + (err_key >> 16);
        const int kind = (int)((err_key >> 8) & 0xff), slot = (int)(err_key & 0xff);
        if (kind == CPB_E_COLUMN_INDEX) {
            int ci = 0;
            for (size_t i = 0; i < cols.size(); i++) if (slot_of(P, cols[i].second) == slot) { ci = (int)i; break; }
            out.error = DataError{kind, ci, line, true,
                                  "column not found: " + go_quote(cols[ci].first) + " (" + std::to_string(cols[ci].second) + ")"};  // csvplus.go:1128
        } else out.error = DataError{kind, -1, line, true, kind_text(kind)};
    }
    for (auto& cc : cols) {
        Column col; col.name = cc.first; col.offsets = offs[slot_of(P, cc.second)]; col.data = datas[slot_of(P, cc.second)];
        t.cols.push_back(col);
        t.src_field.push_back(cc.second);
    }
    return out;
}

// the scan kernel for P: the checked scan's TrimLeadingSpace / CommentChar need the guarded instantiations; otherwise
// kernels specialised on the exact number of extracted columns (no per-column guards), except for shards
void launch_scan_for(Ctx* c, const ParseParams& P, bool shard, uint64_t algo_bytes) {
    if (P.trim || P.comment) {
        if (P.nsel <= 4) launch_scan<4, false>(c, P, algo_bytes);
        else if (P.nsel <= 8) launch_scan<8, false>(c, P, algo_bytes);
        else launch_scan<16, false>(c, P, algo_bytes);
        return;
    }
    switch (shard ? 99 : P.nsel) {
        case 1: launch_scan<1, true>(c, P, algo_bytes); break;
        case 2: launch_scan<2, true>(c, P, algo_bytes); break;
        case 3: launch_scan<3, true>(c, P, algo_bytes); break;
        case 4: launch_scan<4, true>(c, P, algo_bytes); break;
        case 5: launch_scan<5, true>(c, P, algo_bytes); break;
        case 6: launch_scan<6, true>(c, P, algo_bytes); break;
        case 7: launch_scan<7, true>(c, P, algo_bytes); break;
        case 8: launch_scan<8, true>(c, P, algo_bytes); break;
        default: launch_scan<16, false>(c, P, algo_bytes); break;
    }
}

// The single-pass scan.  Its output is sized from the header pass's samples; the exact totals always come back, and an
// overflow costs one exact rerun.  nullopt: the checked scan found that its options matter to this input, and the
// general path parses it.
std::optional<Parsed> run_scan(Ctx* c, ParseParams& P, const HeaderOut& h, Route route, bool lazy_quotes, const ShardArgs* sh,
                               const Spec& cols, uint64_t line_base) {
    const int nsel = P.nsel, NP = 2 + nsel;
    double avg = h.sample_newlines ? (double)h.sample_bytes / (double)h.sample_newlines : (double)P.n;
    if (avg < 2) avg = 2;
    // Capacities are rounded up to size classes so that successive batches of slightly different sizes request
    // identical blocks and are served from the stream-ordered pool instead of mapping fresh memory.
    auto size_class = [](uint64_t v, uint64_t gran) { return (v + gran - 1) / gran * gran; };
    const uint64_t body = P.n - P.data_start;
    uint64_t row_cap = (uint64_t)((double)body / avg * 1.10) + 4096;
    if (row_cap > body / 2 + 2) row_cap = body / 2 + 2;
    row_cap = size_class(row_cap, 1u << 20);
    // per-column bytes from the sampled mean field lengths (naive split of ~768 sampled lines); the worst case
    // (all of the input) when a field was not sampled.  An underestimate costs one exact rerun, never correctness.
    std::vector<uint64_t> data_cap(nsel, std::min<uint64_t>(body, 0xffffffffull));
    for (int k = 0; k < nsel && h.samp_lines >= 16; k++) {
        if (P.sel_field[k] >= HDR_SAMPLE_FIELDS) continue;
        double mean = (double)h.samp_field_bytes[P.sel_field[k]] / (double)h.samp_lines;
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
        launch_scan_for(c, P, sh != nullptr, P.n);  // S_in; S_out added below from the totals
        res = read_back<ParseResult>(c, P.result);
        if (route == Route::checked_scan) {  // did the shortcut hold?
            const int ekind = res.err_key == ~0ull ? 0 : (int)((res.err_key >> 8) & 0xff);
            if (res.need_general || (lazy_quotes && (ekind == CPB_E_BARE_QUOTE || ekind == CPB_E_QUOTE))) return std::nullopt;
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
    if (sh && !sh->is_last && res.eof_hit)
        throw ArgError{CPB_ERR_ARG, "shard look-ahead too small: a record that starts in this shard runs past the end of the buffer"};
    // fold S_out into the algorithmic bytes of the scan record
    if (c->stats_on) {
        uint64_t s_out = 0;
        for (int k = 0; k < nsel; k++) s_out += res.totals[2 + k] + 4 * (res.totals[1] + 1);
        c->drain_events();
        c->stats["csv_scan"].bytes += s_out;
    }
    Parsed p = finish(c, h, cols, P, line_base, (int64_t)(res.err_key != ~0ull ? res.err_rows : res.totals[1]),
                      line_base + (res.first_row_ordinal == ~0ull ? 0 : res.first_row_ordinal), res.err_key, offs, datas);
    p.records = res.totals[0];
    return p;
}

// the general path (parse_general.cu): the route of the options the scan cannot check, and the fallback of the checked scan
Parsed run_general(Ctx* c, ParseParams P, const cpb_reader_opts& o, const Substitution& sub, const HeaderOut& h, const Spec& cols,
                   uint64_t line_base) {
    P.subs = dev_subs(sub); P.trim = 0; P.comment = 0;
    GenResult gr;
    general_parse(c, P, o, &sub, P.data_start, &gr);
    Parsed p = finish(c, h, cols, P, line_base, (int64_t)gr.rows, line_base, gr.err_key, gr.offs, gr.datas);
    p.records = gr.nrec;
    return p;
}

}  // namespace

Parsed parse_csv(Ctx* c, const uint8_t* in_arg, uint64_t n_arg, const cpb_reader_opts& o_arg, const Spec& spec, const cpb_pred* filter,
                 uint64_t line_base, const ShardArgs* sh) {
    // encoding/csv readRecord's option validation (SURVEY App. A.2.1)
    if (o_arg.delimiter == o_arg.comment || !valid_delim(o_arg.delimiter) || (o_arg.comment != 0 && !valid_delim(o_arg.comment)))
        return {empty_table(c, spec), DataError{CPB_E_INVALID_DELIM, -1, 1, true, "csv: invalid field or comment delimiter"}};
    if ((reinterpret_cast<uintptr_t>(in_arg) & 15) != 0) throw ArgError{CPB_ERR_ARG, "device input must be 16-byte aligned"};
    // Multi-byte Delimiter / CommentChar runes and the multi-byte Unicode spaces of TrimLeadingSpace: every occurrence
    // is transcoded to a single byte value the input does not use (subst.cu); from here on the options are single-byte
    const uint8_t* in = in_arg;
    uint64_t n = n_arg;
    cpb_reader_opts o = o_arg;
    Substitution sub;
    if (needs_substitution(o)) {
        sub = substitute_runes(c, in, n, o);
        o.delimiter = sub.delimiter; o.comment = sub.comment;
        if (sub.buffer) { in = sub.buffer->as<uint8_t>(); n = sub.nbytes; }
    }
    const Route route = choose_route(o, sub, sh != nullptr);
    if (sh) {  // a byte-range shard of one file (cpb_parse_csv_shard)
        if (route != Route::scan || sub.table) throw ArgError{CPB_ERR_UNSUPPORTED, "byte-range shards take the default reader options only"};
        if (sh->index > 0 && (o.header_from_first_row || o.num_fields == 0))
            throw ArgError{CPB_ERR_ARG, "shards after the first need the resolved header (name -> index) and an explicit field count"};
        if (sh->own_bytes > n) throw ArgError{CPB_ERR_ARG, "own_bytes exceeds the buffer"};
    }

    const HeaderOut h = read_header(c, in, n, o, sub, route);
    Spec cols;
    if (std::optional<DataError> e = resolve_columns(h, o, spec, cols)) return {empty_table(c, spec), e, 0, h.eof != 0};

    // slots: the distinct field indices, ascending
    std::vector<int> fields;
    for (auto& cc : cols) fields.push_back(cc.second);
    std::sort(fields.begin(), fields.end());
    fields.erase(std::unique(fields.begin(), fields.end()), fields.end());
    if ((int)fields.size() > MAXSEL) return parse_column_groups(c, in_arg, n_arg, o_arg, cols, filter, line_base, sh);

    ParseParams P{};
    P.in = in; P.n = n; P.delim = o.delimiter;
    // a record starting at byte 0 of a later shard belongs to the shard before it
    P.data_start = o.header_from_first_row ? h.data_start : (sh && sh->index > 0 ? 1 : 0);
    const int first_nfields = h.eof ? 0 : h.nfields;
    P.expect_fields = o.num_fields > 0 ? o.num_fields : (o.num_fields == 0 ? first_nfields : 0);
    P.pad_missing = o.num_fields < 0;
    P.nsel = (int)fields.size();
    for (int k = 0; k < P.nsel; k++) P.sel_field[k] = fields[k];
    Compiled comp;
    compile_pred(filter, [&](const std::string& key) {
        int slot = -1;
        for (auto& cc : cols) if (cc.first == key) slot = slot_of(P, cc.second);
        return slot;
    }, comp);
    P.pred = comp.prog;
    for (int t = 0; t < comp.prog.nterms; t++) P.slot_terms[comp.prog.term_col[t]] |= 1u << t;
    P.ntiles = P.data_start >= n ? 0 : (uint32_t)((n + TILE - 1) / TILE);
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
    P.subs = route == Route::checked_scan ? nullptr : dev_subs(sub);
    P.trim = route == Route::checked_scan && o.trim_leading_space ? 1u : 0u;
    P.comment = route == Route::checked_scan ? o.comment : 0u;
    if (P.ntiles == 0) {
        Parsed p{empty_table(c, cols), std::nullopt, 0, h.eof != 0};
        for (auto& cc : cols) p.table->src_field.push_back(cc.second);
        p.table->record_fields = first_nfields;
        return p;
    }
    Buf lits = dev_alloc(c, comp.lits.size() + 16);
    if (!comp.lits.empty())  // pageable source: the runtime stages it before returning
        CPB_CUDA(cudaMemcpyAsync(lits->p, comp.lits.data(), comp.lits.size(), cudaMemcpyHostToDevice, c->stream));
    P.lits = lits->as<uint8_t>();
    P.lits_len = (uint32_t)comp.lits.size();

    if (route != Route::general)
        if (std::optional<Parsed> p = run_scan(c, P, h, route, o.lazy_quotes, sh, cols, line_base)) return std::move(*p);
    return run_general(c, P, o, sub, h, cols, line_base);
}

}  // namespace cpb
