// sprintf.cu — fmt.Sprintf(format, values...) of string columns, row by row: a computed column (the reference's
//   Map(func(row Row) Row { v, _ := row.SelectValues(cols...); row[name] = fmt.Sprintf(format, v[0], ...); return row }))
// and a text sink (src(func(row Row) error { ...; _, err = fmt.Fprintf(out, format, v[0], ...); return err })), whose
// output is every row's text in row order, with no header and no separator.
//
// The format language is the subset of Go's fmt whose output for string operands is fixed and never an error text:
//   literal bytes (any bytes, NUL and invalid UTF-8 included), %% (bare), and %[-...][width][.[prec]]s / v with width and
//   precision decimal and at most 1 000 000.  Precision keeps the first prec runes (fmt's truncateString), width pads
//   with spaces to width runes (padString: on the left, on the right with '-').  Runes are utf8.DecodeRune's: a byte that
//   does not start a valid sequence is one rune of one byte.  Everything else (another verb, the flags 0 + # and space,
//   '*', argument indexes, a lone trailing '%', a verb count other than the column count, more than SP_MAXV verbs, a
//   format longer than SP_MAXLIT bytes) is refused by sprintf_compile with CPB_ERR_UNSUPPORTED before any launch.
//
// The format compiles once, on the host, into pieces: a literal slice of the format's bytes (adjacent literals and %%
// merged) or a verb (its column, width, precision, alignment).  The row type SprintfRows runs through the row serialiser
// driver of rowwrite.cuh, as ToCsv's does:
//   sprintf_len:   one thread per row: the literal bytes (a constant) plus each verb's bytes; a verb with a precision walks
//                  at most prec runes, a verb with a width counts the runes of its (truncated) value unless the value has at
//                  least 4 * width bytes (then it has at least width runes and needs no padding).
//   exclusive_scan_u32 of the lengths (the offsets) and its exact 64-bit total, read back once: a total of 2^32 or more,
//                  or one row of exactly 0xFFFFFFFF bytes (which may be a saturated longer one), is CPB_E_TOO_LARGE before
//                  anything else is allocated.
//   sprintf_write: the warp-staged row writer; every block first copies the piece table and the literal bytes into
//                  shared memory.
#include "core.hpp"
#include "rowwrite.cuh"

namespace cpb {

constexpr int SP_MAXV = 64;                   // verbs per format
constexpr int SP_MAXP = 2 * SP_MAXV + 1;      // pieces: literals between the verbs
constexpr uint32_t SP_MAXLIT = 4096;          // bytes of a format
constexpr uint32_t SP_MAXNUM = 1000000;       // the largest width or precision
constexpr uint32_t SP_NO_PREC = 0xFFFFFFFFu;  // a verb without a precision

// the bytes of the rune utf8.DecodeRune reads at p (n > 0 bytes left): 1 for a byte that starts no valid sequence
__host__ __device__ __forceinline__ uint32_t rune_bytes(const uint8_t* p, uint32_t n) {
    const uint32_t w = utf8_seq(p, n);
    return w ? w : 1;
}

// one verb of a row: *keep = the value's bytes that are written (truncateString), returns the padding spaces (padString)
__host__ __device__ __forceinline__ uint32_t verb_layout(const uint8_t* p, uint32_t l, uint32_t width, uint32_t prec, uint32_t* keep) {
    uint32_t b = l, runes = 0;
    bool counted = false;
    if (prec != SP_NO_PREC) {
        uint32_t i = 0;
        while (i < l && runes < prec) { i += rune_bytes(p + i, l - i); runes++; }
        b = i; counted = true;
    }
    *keep = b;
    if (width == 0) return 0;
    if (!counted) {
        if (l >= 4 * width) return 0;  // at least l / 4 >= width runes
        for (uint32_t i = 0; i < l; runes++) i += rune_bytes(p + i, l - i);
    }
    return runes < width ? width - runes : 0;
}

// a piece of the format: verb >= 0, or the literal bytes [lit, lit + len) of the literal blob
struct SpPiece { int32_t verb; uint32_t lit, len, pad_; };

struct SpFormat {
    std::vector<SpPiece> pieces;
    std::string lit;                // the literal bytes, piece after piece
    std::vector<uint32_t> width, prec;
    uint64_t left = 0;
    int nverbs = 0;
};

[[noreturn]] static void refuse(size_t at, const std::string& what) {
    throw ArgError{CPB_ERR_UNSUPPORTED, "Sprintf format: " + what + " at byte " + std::to_string(at)};
}

// the format as Go's fmt.doPrintf reads it, restricted to the accepted subset; nargs: the columns it is given
static SpFormat sprintf_compile(const std::string& f, int nargs) {
    if (f.size() > SP_MAXLIT) refuse(SP_MAXLIT, "a format longer than " + std::to_string(SP_MAXLIT) + " bytes");
    SpFormat r;
    auto literal = [&](const char* p, size_t n) {
        if (!n) return;
        if (r.pieces.empty() || r.pieces.back().verb >= 0) r.pieces.push_back(SpPiece{-1, (uint32_t)r.lit.size(), 0, 0});
        r.lit.append(p, n);
        r.pieces.back().len += (uint32_t)n;
    };
    const size_t end = f.size();
    size_t i = 0;
    while (i < end) {
        size_t j = i;
        while (j < end && f[j] != '%') j++;
        literal(f.data() + i, j - i);
        if (j >= end) break;
        const size_t at = j++;  // the '%'
        if (j >= end) refuse(at, "a lone '%' at the end of the format");
        bool minus = false;
        for (; j < end; j++) {
            const char c = f[j];
            if (c == '-') minus = true;
            else if (c == '0' || c == '+' || c == '#' || c == ' ') refuse(j, std::string("the flag '") + c + "'");
            else break;
        }
        auto number = [&](uint32_t* v) {  // decimal digits from j; false when there are none
            const size_t s = j;
            uint64_t x = 0;
            for (; j < end && f[j] >= '0' && f[j] <= '9'; j++) {
                x = x * 10 + (uint64_t)(f[j] - '0');
                if (x > SP_MAXNUM) refuse(s, "a width or precision above " + std::to_string(SP_MAXNUM));
            }
            *v = (uint32_t)x;
            return j > s;
        };
        uint32_t width = 0, prec = SP_NO_PREC;
        if (j < end && f[j] == '[') refuse(j, "an explicit argument index");
        if (j < end && f[j] == '*') refuse(j, "a '*' width");
        const bool has_width = number(&width);
        if (j < end && f[j] == '.') {
            j++;
            if (j < end && f[j] == '[') refuse(j, "an explicit argument index");
            if (j < end && f[j] == '*') refuse(j, "a '*' precision");
            number(&prec);  // a bare '.' is precision 0
        }
        if (j < end && f[j] == '[') refuse(j, "an explicit argument index");
        if (j >= end) refuse(at, "a verb missing at the end of the format");
        const unsigned char verb = (unsigned char)f[j];
        if (verb == '%') {
            if (minus || has_width || prec != SP_NO_PREC) refuse(at, "flags, width or precision on %%");
            literal("%", 1);
        } else if (verb == 's' || verb == 'v') {
            if (r.nverbs == SP_MAXV) refuse(at, "more than " + std::to_string(SP_MAXV) + " verbs");
            if (r.nverbs >= nargs) refuse(at, "verb " + std::to_string(r.nverbs + 1) + " without a column (" + std::to_string(nargs) + " given)");
            if (minus) r.left |= 1ull << r.nverbs;
            r.width.push_back(width); r.prec.push_back(prec);
            r.pieces.push_back(SpPiece{r.nverbs++, 0, 0, 0});
        } else if (verb >= 0x80) {
            refuse(j, "a non-ASCII verb");
        } else {
            refuse(j, std::string("the verb '") + (char)verb + "' (want s, v or %%)");
        }
        i = j + 1;
    }
    if (r.nverbs != nargs) refuse(end, std::to_string(nargs) + " columns for " + std::to_string(r.nverbs) + " verbs");
    return r;
}

constexpr uint32_t SW_STAGE = 4096;
// a row: the pieces of a compiled format; verb v reads column off[v] / data[v].  Every block copies the piece table and
// the literal bytes into shared memory, at their largest size whatever the format.
struct SprintfRows {
    int n;
    uint32_t lit_total;  // literal bytes of a row
    const uint32_t* off[SP_MAXV];
    const uint8_t* data[SP_MAXV];
    uint32_t width[SP_MAXV], prec[SP_MAXV];
    uint64_t left;       // bit v: verb v is left-aligned ('-')
    const SpPiece* pieces; int npieces;
    const uint8_t* lit;

    __device__ uint64_t len(uint64_t r) const {
        uint64_t total = lit_total;
        for (int v = 0; v < n; v++) {
            const uint32_t s = off[v][r], l = off[v][r + 1] - s;
            uint32_t keep;
            const uint32_t pad = verb_layout(data[v] + s, l, width[v], prec[v], &keep);
            total += (uint64_t)keep + pad;
        }
        return total;
    }

    struct Tables { const SpPiece* pieces; const uint8_t* lit; };
    static constexpr uint32_t TABLE_BYTES = SP_MAXP * sizeof(SpPiece) + SP_MAXLIT;
    static constexpr bool TAIL_VARIES = false;
    uint32_t tail() const { return TABLE_BYTES; }
    __device__ Tables stage(uint8_t* sm) const {
        SpPiece* sp = reinterpret_cast<SpPiece*>(sm);
        uint8_t* sl = sm + SP_MAXP * sizeof(SpPiece);
        for (int i = threadIdx.x; i < npieces; i += blockDim.x) sp[i] = pieces[i];
        for (uint32_t i = threadIdx.x; i < lit_total; i += blockDim.x) sl[i] = lit[i];
        __syncthreads();
        return {sp, sl};
    }

    __device__ void write(uint64_t r, uint8_t* q, const Tables& t) const {
        for (int k = 0; k < npieces; k++) {
            const SpPiece pc = t.pieces[k];
            if (pc.verb < 0) {
                for (uint32_t i = 0; i < pc.len; i++) *q++ = t.lit[pc.lit + i];
                continue;
            }
            const int v = pc.verb;
            const uint32_t s = off[v][r], l = off[v][r + 1] - s;
            const uint8_t* p = data[v] + s;
            uint32_t keep;
            const uint32_t pad = verb_layout(p, l, width[v], prec[v], &keep);
            const bool left_aligned = (left >> v) & 1;
            if (!left_aligned) for (uint32_t i = 0; i < pad; i++) *q++ = ' ';
            for (uint32_t i = 0; i < keep; i++) *q++ = p[i];
            if (left_aligned) for (uint32_t i = 0; i < pad; i++) *q++ = ' ';
        }
    }
};

// the lengths of the n rows into len (n + 1 entries), which then holds the offsets; returns the exact total
static uint64_t sprintf_sizes(Ctx* c, const SprintfRows& rows, uint64_t n, uint32_t* len, const std::string& what) {
    Buf tot = dev_alloc(c, 8);
    row_lengths(c, rows, n, len, "sprintf_len", n * 4 * (rows.n + 1));
    return row_offsets(c, len, n, tot->as<uint64_t>(), 1, MAX_BODY, what + " would hold 4 GiB or more: format row-range slices")[0];
}

static void sprintf_write(Ctx* c, const SpFormat& f, SprintfRows rows, uint64_t n, const uint32_t* pos, uint64_t body, uint8_t* out) {
    if (!n) return;
    const size_t pbytes = f.pieces.size() * sizeof(SpPiece);
    Buf meta = dev_alloc(c, pbytes + f.lit.size());
    // (pageable source: the copy is staged before the call returns, so the host table may go away)
    CPB_CUDA(cudaMemcpyAsync(meta->p, f.pieces.data(), pbytes, cudaMemcpyHostToDevice, c->stream));
    if (!f.lit.empty()) CPB_CUDA(cudaMemcpyAsync(meta->as<uint8_t>() + pbytes, f.lit.data(), f.lit.size(), cudaMemcpyHostToDevice, c->stream));
    rows.pieces = meta->as<SpPiece>();
    rows.npieces = (int)f.pieces.size();
    rows.lit = meta->as<uint8_t>() + pbytes;
    row_write<SW_STAGE>(c, rows, n, pos, out, "sprintf_write", 2 * body + n * 4 * (rows.n + 1), 16);
}

// the format compiled for the columns `names` of t, and their positions in t.  A column t lacks is Row.SelectValues's
// `missing column %q` (csvplus.go:138-149), for a table with rows only: as ToCsv reports it (column index, row 0) for a
// sink, as column_as_int64 does (no row) for a computed column.
static SprintfRows sprintf_prepare(const Table& t, const std::string& format, const std::vector<std::string>& names, bool sink, SpFormat& f) {
    f = sprintf_compile(format, (int)names.size());
    SprintfRows sv{};
    sv.n = f.nverbs;
    sv.lit_total = (uint32_t)f.lit.size();
    sv.left = f.left;
    for (int v = 0; v < f.nverbs; v++) {
        sv.width[v] = f.width[v]; sv.prec[v] = f.prec[v];
        const int k = t.find(names[v]);
        if (t.nrows == 0) continue;
        if (k < 0) {
            if (sink) throw DataError{CPB_E_MISSING_COLUMN, v, t.first_line, true, "missing column " + go_quote(names[v])};
            throw DataError{CPB_E_MISSING_COLUMN, -1, 0, false, "missing column " + go_quote(names[v])};
        }
        sv.off[v] = t.cols[k].off(); sv.data[v] = t.cols[k].bytes();
    }
    return sv;
}

std::shared_ptr<Table> table_set_sprintf(Ctx* c, const Table& t, const std::string& name, const std::string& format,
                                         const std::vector<std::string>& cols) {
    SpFormat f;
    const SprintfRows sv = sprintf_prepare(t, format, cols, false, f);
    const uint64_t n = (uint64_t)t.nrows;
    if (n == 0) return with_column(t, name, empty_column(c));
    Column col;
    col.offsets = dev_alloc(c, (n + 1) * 4);
    const uint64_t body = sprintf_sizes(c, sv, n, col.offsets->as<uint32_t>(), "column " + go_quote(name));
    col.data = dev_alloc(c, body + 16);
    sprintf_write(c, f, sv, n, col.offsets->as<uint32_t>(), body, col.data->as<uint8_t>());
    return with_column(t, name, col);
}

Buf table_sprintf(Ctx* c, const Table& t, const std::string& format, const std::vector<std::string>& cols, uint64_t room, uint64_t* nbytes) {
    SpFormat f;
    const SprintfRows sv = sprintf_prepare(t, format, cols, true, f);
    const uint64_t n = (uint64_t)t.nrows;
    Buf len = dev_alloc(c, (n + 1) * 4);
    const uint64_t body = sprintf_sizes(c, sv, n, len->as<uint32_t>(), "Sprintf output");
    *nbytes = body;
    if (body > room) return nullptr;
    Buf out = dev_alloc(c, body + 16);
    sprintf_write(c, f, sv, n, len->as<uint32_t>(), body, out->as<uint8_t>());
    return out;
}

}  // namespace cpb
