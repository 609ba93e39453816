// oracle.cpp — CPU restatement of the maxim2266/csvplus hot path.
//
// TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
// legs may load this library, and only as the checker / timed CPU baseline.
// The product path (csvplus_b200/libcsvplus_b200.so) never links or calls it.
//
// PARITY STATUS: "parity unpinned by execution".  The reference is pure Go and no
// Go toolchain exists in this image, so the reference cannot be run here.  The
// oracle is pinned against (a) every literal known-answer vector in the
// reference's own tests (csvplus_test.go: TestRow :49-116, TestIndexImpl :198-246,
// TestErrors :808-909 message strings) and (b) a restatement of Go's
// encoding/csv reader_test table (SURVEY.md App. A.3) — see tests/test_oracle_kat.py.
//
// Every function cites the reference lines it restates (csvplus.go = the single
// source file of the reference; "encoding/csv" = Go 1.23 stdlib, go.mod:3, which
// is not vendored with the reference — its published algorithm is restated).
//
// Data model mirrors the reference: Row = hash map string->string
// (csvplus.go:59), a DataSource result = vector of Rows + optional error
// (row-at-a-time evaluation, one map allocation per row per stage, like the
// reference's closure chain), Index = sorted vector<Row> + key columns
// (csvplus.go:785-788).

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

namespace {

using Row = std::unordered_map<std::string, std::string>;

// ---------------------------------------------------------------- errors
enum ErrKind : int {
    E_NONE = 0,
    E_BARE_QUOTE = 1,   // encoding/csv ErrBareQuote  `bare " in non-quoted-field`
    E_QUOTE = 2,        // encoding/csv ErrQuote      `extraneous or missing " in quoted-field`
    E_FIELD_COUNT = 3,  // encoding/csv ErrFieldCount `wrong number of fields`
    E_INVALID_DELIM = 4,// `csv: invalid field or comment delimiter`
    E_EOF = 5,          // io.EOF surfaced through mapError (empty input with header expected)
    E_OTHER = 6,        // message carried verbatim
};

const char* csv_err_text(int k) {
    switch (k) {
        case E_BARE_QUOTE: return "bare \" in non-quoted-field";
        case E_QUOTE: return "extraneous or missing \" in quoted-field";
        case E_FIELD_COUNT: return "wrong number of fields";
        case E_INVALID_DELIM: return "csv: invalid field or comment delimiter";
        case E_EOF: return "EOF";
        default: return "";
    }
}

struct Result {            // what a DataSource pull produced
    std::vector<Row> rows; // rows delivered before the error (streaming semantics)
    bool failed = false;
    uint64_t line = 0;     // DataSourceError.Line (csvplus.go:1230-1233)
    std::string msg;       // DataSourceError.Err text
    int kind = 0;
    std::string error() const {  // csvplus.go:1236-1238  `row %d: %s`
        return failed ? ("row " + std::to_string(line) + ": " + msg) : std::string();
    }
};

// ---------------------------------------------------------------- UTF-8 helpers (Go runes)
// utf8.DecodeRune restated: returns rune and width; invalid => (0xFFFD, 1); empty => (0xFFFD, 0).
static uint32_t decode_rune(const uint8_t* p, size_t n, int* w) {
    if (n == 0) { *w = 0; return 0xFFFD; }
    uint8_t c = p[0];
    if (c < 0x80) { *w = 1; return c; }
    auto cont = [&](size_t i) { return i < n && (p[i] & 0xC0) == 0x80; };
    if (c >= 0xC2 && c <= 0xDF && cont(1)) { *w = 2; return ((c & 0x1F) << 6) | (p[1] & 0x3F); }
    if (c >= 0xE0 && c <= 0xEF && cont(1) && cont(2)) {
        uint32_t r = ((c & 0x0F) << 12) | ((p[1] & 0x3F) << 6) | (p[2] & 0x3F);
        if (r >= 0x800 && !(r >= 0xD800 && r <= 0xDFFF)) { *w = 3; return r; }
    }
    if (c >= 0xF0 && c <= 0xF4 && cont(1) && cont(2) && cont(3)) {
        uint32_t r = ((c & 0x07) << 18) | ((p[1] & 0x3F) << 12) | ((p[2] & 0x3F) << 6) | (p[3] & 0x3F);
        if (r >= 0x10000 && r <= 0x10FFFF) { *w = 4; return r; }
    }
    *w = 1; return 0xFFFD;
}
static int rune_len(uint32_t r) {  // utf8.RuneLen
    if (r < 0x80) return 1; if (r < 0x800) return 2;
    if (r >= 0xD800 && r <= 0xDFFF) return -1;
    if (r < 0x10000) return 3; if (r <= 0x10FFFF) return 4; return -1;
}
static std::string encode_rune(uint32_t r) {
    std::string s;
    if (r < 0x80) s += char(r);
    else if (r < 0x800) { s += char(0xC0 | (r >> 6)); s += char(0x80 | (r & 0x3F)); }
    else if (r < 0x10000) { s += char(0xE0 | (r >> 12)); s += char(0x80 | ((r >> 6) & 0x3F)); s += char(0x80 | (r & 0x3F)); }
    else { s += char(0xF0 | (r >> 18)); s += char(0x80 | ((r >> 12) & 0x3F)); s += char(0x80 | ((r >> 6) & 0x3F)); s += char(0x80 | (r & 0x3F)); }
    return s;
}
// unicode.IsSpace restated (Latin-1 fast path + the Unicode White_Space set).
static bool is_space_rune(uint32_t r) {
    switch (r) {
        case '\t': case '\n': case '\v': case '\f': case '\r': case ' ': case 0x85: case 0xA0:
        case 0x1680: case 0x2028: case 0x2029: case 0x202F: case 0x205F: case 0x3000: return true;
    }
    return r >= 0x2000 && r <= 0x200A;
}

// ---------------------------------------------------------------- encoding/csv.Reader restated
// Options csvplus sets on the stdlib reader: csvplus.go:1091-1097.
struct CsvOpts {
    uint32_t comma = ',';
    uint32_t comment = 0;
    bool lazy_quotes = false;
    bool trim_leading_space = false;
    int fields_per_record = 0;  // 0 auto (first record), >0 exact, <0 any
};

// encoding/csv validDelim: r != 0 && r != '"' && r != '\r' && r != '\n' && utf8.ValidRune(r) && r != utf8.RuneError
static bool valid_delim(uint32_t r) {
    return r != 0 && r != '"' && r != '\r' && r != '\n' && rune_len(r) > 0 && r != 0xFFFD;
}

class CsvReader {
public:
    CsvReader(const uint8_t* p, size_t n, const CsvOpts& o) : p_(p), n_(n), o_(o), fpr_(o.fields_per_record) {}

    // encoding/csv (*Reader).readRecord.  Returns: 0 ok, 1 io.EOF, 2 error (kind in *err);
    // like Go, a record with ErrFieldCount is still produced (rec filled) together with the error.
    int read(std::vector<std::string>& rec, int* err) {
        rec.clear();
        *err = E_NONE;
        if (o_.comma == o_.comment || !valid_delim(o_.comma) || (o_.comment != 0 && !valid_delim(o_.comment))) {
            *err = E_INVALID_DELIM;
            return 2;
        }
        // Read line (automatically skipping past empty lines and any comments).
        std::string line;
        bool have = false, err_eof = false;
        for (;;) {
            have = read_line(line, &err_eof);
            if (o_.comment != 0) {
                int w; uint32_t r = decode_rune((const uint8_t*)line.data(), line.size(), &w);
                if (r == o_.comment) { line.clear(); if (err_eof) break; continue; }
            }
            if (!err_eof && line.size() == length_nl(line)) { line.clear(); continue; }
            break;
        }
        (void)have;
        if (err_eof) return 1;  // errRead == io.EOF

        const std::string comma = encode_rune(o_.comma);
        const size_t comma_len = comma.size();
        std::string buf;                 // r.recordBuffer
        std::vector<size_t> idx;         // r.fieldIndexes
        size_t lp = 0;                   // cursor into `line` (Go reslices line)
        bool read_err_eof = false;       // errRead inside the quoted-field loop
        for (;;) {  // parseField
            if (o_.trim_leading_space) {
                size_t i = lp; bool found = false;
                while (i < line.size()) {
                    int w; uint32_t r = decode_rune((const uint8_t*)line.data() + i, line.size() - i, &w);
                    if (!is_space_rune(r)) { found = true; break; }
                    i += w;
                }
                if (!found) i = line.size();
                lp = i;
            }
            if (lp >= line.size() || line[lp] != '"') {
                // Non-quoted string field
                size_t i = line.find(comma, lp);
                size_t fend;
                if (i != std::string::npos) fend = i;
                else fend = line.size() - length_nl_at(line, lp);
                if (!o_.lazy_quotes) {
                    for (size_t j = lp; j < fend; j++)
                        if (line[j] == '"') { *err = E_BARE_QUOTE; goto done; }
                }
                buf.append(line, lp, fend - lp);
                idx.push_back(buf.size());
                if (i != std::string::npos) { lp = i + comma_len; continue; }
                break;
            } else {
                // Quoted string field
                lp += 1;
                for (;;) {
                    size_t i = line.find('"', lp);
                    if (i != std::string::npos) {
                        // Hit next quote.
                        buf.append(line, lp, i - lp);
                        lp = i + 1;
                        int w; uint32_t rn = decode_rune((const uint8_t*)line.data() + lp, line.size() - lp, &w);
                        if (lp < line.size() && rn == '"') {          // `""` sequence (append quote)
                            buf += '"'; lp += 1;
                        } else if (lp < line.size() && rn == o_.comma) {  // `",` sequence (end of field)
                            lp += comma_len;
                            idx.push_back(buf.size());
                            goto next_field;
                        } else if (length_nl_at(line, lp) == line.size() - lp) {  // `"\n` (end of line)
                            idx.push_back(buf.size());
                            goto done;
                        } else if (o_.lazy_quotes) {                  // `"` sequence (bare quote)
                            buf += '"';
                        } else {                                      // `"*` sequence (invalid non-escaped quote)
                            *err = E_QUOTE; goto done;
                        }
                    } else if (lp < line.size()) {
                        // Hit end of line (copy all data so far).
                        buf.append(line, lp, std::string::npos);
                        if (read_err_eof) goto done;  // (errRead != nil) — unreachable: EOF is cleared below
                        bool e2 = false;
                        read_line(line, &e2);
                        lp = 0;
                        // Go: if errRead == io.EOF { errRead = nil }
                        (void)e2;
                    } else {
                        // Abrupt end of file (EOF or error).
                        if (!o_.lazy_quotes) { *err = E_QUOTE; goto done; }
                        idx.push_back(buf.size());
                        goto done;
                    }
                }
            }
        next_field:;
        }
    done:
        // Create a single string and create slices out of it.
        {
            size_t pre = 0;
            for (size_t e : idx) { rec.emplace_back(buf, pre, e - pre); pre = e; }
        }
        if (*err != E_NONE) return 2;
        // Check or update the expected fields per record.
        if (fpr_ > 0) {
            if ((int)rec.size() != fpr_) { *err = E_FIELD_COUNT; return 2; }
        } else if (fpr_ == 0) {
            fpr_ = (int)rec.size();
        }
        return 0;
    }

private:
    static size_t length_nl(const std::string& b) { return (!b.empty() && b.back() == '\n') ? 1 : 0; }
    static size_t length_nl_at(const std::string& b, size_t from) {
        return (b.size() > from && b.back() == '\n') ? 1 : 0;
    }
    // encoding/csv (*Reader).readLine: returns false + *eof when no bytes remain.
    bool read_line(std::string& line, bool* eof) {
        line.clear();
        *eof = false;
        if (pos_ >= n_) { *eof = true; return false; }
        const uint8_t* s = p_ + pos_;
        const uint8_t* nl = (const uint8_t*)memchr(s, '\n', n_ - pos_);
        size_t len = nl ? (size_t)(nl - s) + 1 : n_ - pos_;
        line.assign((const char*)s, len);
        pos_ += len;
        if (!nl) {  // readSize > 0 && err == io.EOF  => err = nil; drop trailing \r before EOF
            if (line.back() == '\r') line.pop_back();
        }
        // Normalize \r\n to \n on all input lines.
        size_t n = line.size();
        if (n >= 2 && line[n - 2] == '\r' && line[n - 1] == '\n') { line[n - 2] = '\n'; line.pop_back(); }
        return true;
    }

    const uint8_t* p_; size_t n_; size_t pos_ = 0;
    CsvOpts o_; int fpr_;
};

// ---------------------------------------------------------------- csvplus Reader (csvplus.go:922-1227)
struct HeaderSpec {                 // Reader.header map[string]int (csvplus.go:929)
    std::vector<std::pair<std::string, int>> cols;  // name -> index (-1 = search)
    bool from_first_row = true;     // headerFromFirstRow (csvplus.go:930)
};

static std::string go_quote(const std::string& s) {  // fmt %q for the plain strings used in tests
    std::string r = "\"";
    for (unsigned char c : s) {
        if (c == '"' || c == '\\') { r += '\\'; r += char(c); }
        else if (c == '\n') r += "\\n"; else if (c == '\r') r += "\\r"; else if (c == '\t') r += "\\t";
        else if (c < 0x20 || c == 0x7f) { char b[8]; snprintf(b, sizeof b, "\\x%02x", c); r += b; }
        else r += char(c);
    }
    return r + "\"";
}

// Reader.makeHeader, csvplus.go:1149-1206.  Returns "" on success else the error text.
static std::string make_header(CsvReader& rd, const HeaderSpec& spec, std::vector<std::pair<std::string, int>>& header,
                               int* kind) {
    std::vector<std::string> line; int err;
    int rc = rd.read(line, &err);
    if (rc == 1) { *kind = E_EOF; return "EOF"; }
    if (rc == 2) { *kind = err; return csv_err_text(err); }
    if (line.empty()) { *kind = E_OTHER; return "empty header"; }
    header.clear();
    if (spec.cols.empty()) {  // :1160-1168 — later duplicates overwrite earlier ones (map assignment)
        std::unordered_map<std::string, size_t> pos;
        for (size_t i = 0; i < line.size(); i++) {
            auto it = pos.find(line[i]);
            if (it == pos.end()) { pos[line[i]] = header.size(); header.emplace_back(line[i], (int)i); }
            else header[it->second].second = (int)i;
        }
        return "";
    }
    std::unordered_map<std::string, int> want(spec.cols.begin(), spec.cols.end());
    std::unordered_map<std::string, int> got;
    for (size_t i = 0; i < line.size(); i++) {  // :1174-1183
        auto it = want.find(line[i]);
        if (it != want.end()) {
            if (it->second == -1 || it->second == (int)i) got[line[i]] = (int)i;
            else {
                *kind = E_OTHER;
                return "misplaced column " + go_quote(line[i]) + ": expected at pos. " + std::to_string(it->second) +
                       ", but found at pos. " + std::to_string(i);
            }
        }
    }
    if (got.size() < want.size()) {  // :1186-1202 (order of names is Go-map-random; we use spec order)
        std::vector<std::string> list;
        for (auto& c : spec.cols) if (!got.count(c.first)) list.push_back(c.first);
        *kind = E_OTHER;
        if (list.size() > 1) {
            std::string s = "columns not found: ";
            for (size_t i = 0; i < list.size(); i++) { if (i) s += ", "; s += list[i]; }
            return s;
        }
        return "column not found: " + list[0];
    }
    for (auto& c : spec.cols) header.emplace_back(c.first, got[c.first]);
    return "";
}

// Reader.Iterate, csvplus.go:1080-1146.  `fn` returns "" to continue, or an error text
// (kind E_OTHER); a special value "\x01EOF" plays io.EOF (clean stop, csvplus.go:1141).
using RowFn = std::function<std::string(Row&)>;
static void reader_iterate(const uint8_t* p, size_t n, const CsvOpts& o, const HeaderSpec& spec, Result& res,
                           const RowFn& fn) {
    CsvReader rd(p, n, o);
    std::vector<std::pair<std::string, int>> header;
    uint64_t line_no = 1;                                   // :1102
    auto fail = [&](int kind, const std::string& msg) { res.failed = true; res.line = line_no; res.kind = kind; res.msg = msg; };
    if (spec.from_first_row) {                              // :1104-1112
        int kind = 0;
        std::string e = make_header(rd, spec, header, &kind);
        if (!e.empty()) { fail(kind, e); return; }
        line_no++;
    } else header = spec.cols;
    std::vector<std::string> line; int err;
    for (;;) {                                              // :1117
        int rc = rd.read(line, &err);
        if (rc == 1) return;                                // io.EOF => nil (:1141-1145)
        if (rc == 2) { fail(err, csv_err_text(err)); return; }  // mapError :1209-1227 keeps ParseError.Err
        Row row; row.reserve(header.size());                // :1118
        for (auto& h : header) {                            // :1120-1131
            if (h.second < (int)line.size()) row[h.first] = line[h.second];
            else if (o.fields_per_record < 0) row[h.first] = "";
            else { fail(E_OTHER, "column not found: " + go_quote(h.first) + " (" + std::to_string(h.second) + ")"); return; }
        }
        std::string e = fn(row);                            // :1133
        if (!e.empty()) { if (e != "\x01""EOF") fail(E_OTHER, e); return; }
        line_no++;                                          // :1137
    }
}

// ---------------------------------------------------------------- Row helpers (csvplus.go:62-161)
static std::string row_string(const Row& row) {  // Row.String, csvplus.go:90-104 (keys sorted, :78-87)
    if (row.empty()) return "{}";
    std::map<std::string, std::string> s(row.begin(), row.end());
    std::string b = "{ ";
    bool first = true;
    for (auto& kv : s) { if (!first) b += ", "; first = false; b += "\"" + kv.first + "\" : \"" + kv.second + "\""; }
    return b + " }";
}
// Row.Select, csvplus.go:122-134
static std::string row_select(const Row& row, const std::vector<std::string>& cols, Row& out) {
    out.clear(); out.reserve(cols.size());
    for (auto& c : cols) { auto it = row.find(c); if (it == row.end()) return "missing column " + go_quote(c); out[c] = it->second; }
    return "";
}
// Row.SelectValues, csvplus.go:138-150
static std::string row_select_values(const Row& row, const std::vector<std::string>& cols, std::vector<std::string>& out) {
    out.assign(cols.size(), std::string());
    for (size_t i = 0; i < cols.size(); i++) { auto it = row.find(cols[i]); if (it == row.end()) return "missing column " + go_quote(cols[i]); out[i] = it->second; }
    return "";
}
// Like, csvplus.go:1279-1293
static bool like(const Row& row, const Row& match) {
    for (auto& kv : match) { auto it = row.find(kv.first); if (it == row.end() || it->second != kv.second) return false; }
    return true;
}

// predicate AST mirroring All/Any/Not/Like (csvplus.go:1243-1293); serialised form is parsed in orc_pred_*.
struct Pred {
    int op = 0;  // 0 LIKE, 1 ALL, 2 ANY, 3 NOT
    Row match;
    std::vector<Pred> kids;
    bool eval(const Row& r) const {
        switch (op) {
            case 0: return like(r, match);
            case 1: for (auto& k : kids) if (!k.eval(r)) return false; return true;   // :1243-1253
            case 2: for (auto& k : kids) if (k.eval(r)) return true; return false;    // :1258-1268
            default: return !kids[0].eval(r);                                         // :1271-1275
        }
    }
};

// ---------------------------------------------------------------- Index (csvplus.go:610-920)
struct Index { std::vector<Row> rows; std::vector<std::string> columns; };

static const std::string kEmpty;
static const std::string& getv(const Row& r, const std::string& c) { auto it = r.find(c); return it == r.end() ? kEmpty : it->second; }
static int str_cmp(const std::string& a, const std::string& b) {  // strings.Compare: bytewise, shorter prefix first
    int c = memcmp(a.data(), b.data(), std::min(a.size(), b.size()));
    if (c) return c < 0 ? -1 : 1;
    return a.size() < b.size() ? -1 : (a.size() > b.size() ? 1 : 0);
}
// indexImpl.Less, csvplus.go:794-807
static bool index_less(const std::vector<std::string>& cols, const Row& l, const Row& r) {
    for (auto& c : cols) { int k = str_cmp(getv(l, c), getv(r, c)); if (k < 0) return true; if (k > 0) return false; }
    return false;
}
// equalRows, csvplus.go:759-767
static bool equal_rows(const std::vector<std::string>& cols, const Row& a, const Row& b) {
    for (auto& c : cols) if (getv(a, c) != getv(b, c)) return false;
    return true;
}
// indexImpl.cmp, csvplus.go:907-920
static bool index_cmp(const Index& ix, size_t i, const std::vector<std::string>& values, bool eq) {
    const Row& row = ix.rows[i];
    for (size_t j = 0; j < values.size(); j++) {
        int k = str_cmp(getv(row, ix.columns[j]), values[j]);
        if (k > 0) return true; if (k < 0) return false;
    }
    return eq;
}
// sort.Search restated: smallest i in [0,n) with f(i) true, else n.
template <class F> static size_t go_search(size_t n, F f) {
    size_t i = 0, j = n;
    while (i < j) { size_t h = i + (j - i) / 2; if (!f(h)) i = h + 1; else j = h; }
    return i;
}
// indexImpl.first, csvplus.go:893-897
static size_t index_first(const Index& ix, const std::vector<std::string>& values) {
    return go_search(ix.rows.size(), [&](size_t i) { return index_cmp(ix, i, values, true); });
}
// indexImpl.find, csvplus.go:870-891
static std::pair<size_t, size_t> index_find(const Index& ix, const std::vector<std::string>& values) {
    if (values.empty()) return {0, ix.rows.size()};
    size_t upper = go_search(ix.rows.size(), [&](size_t i) { return index_cmp(ix, i, values, false); });
    size_t lower = go_search(upper, [&](size_t i) { return index_cmp(ix, i, values, true); });
    return {lower, upper};
}

// createIndex, csvplus.go:707-738.  `stable`: the reference's sort.Sort is an unstable pdqsort
// (SURVEY §Q2); order inside equal-key runs is unspecified there.  stable=true gives the
// by-input-ordinal tie order the CUDA path defines; stable=false (std::sort, introsort) is the
// timing proxy for sort.Sort.
static std::string create_index(const Result& src, const std::vector<std::string>& cols, bool stable, Index& ix) {
    ix.columns = cols; ix.rows.clear();
    for (auto& row : src.rows) {
        for (auto& c : cols) if (!row.count(c)) return "missing column " + go_quote(c) + " while creating an index";  // :723-727
        ix.rows.push_back(row);
    }
    auto less = [&](const Row& a, const Row& b) { return index_less(cols, a, b); };
    if (stable) std::stable_sort(ix.rows.begin(), ix.rows.end(), less); else std::sort(ix.rows.begin(), ix.rows.end(), less);
    return "";
}
// createUniqueIndex, csvplus.go:740-756
static std::string check_unique(const Index& ix) {
    for (size_t i = 1; i < ix.rows.size(); i++)
        if (equal_rows(ix.columns, ix.rows[i - 1], ix.rows[i])) {
            Row key;  // rows[i].SelectExisting(columns...) :751, :108-118
            for (auto& c : ix.columns) { auto it = ix.rows[i].find(c); if (it != ix.rows[i].end()) key[c] = it->second; }
            return "duplicate value while creating unique index: " + row_string(key);
        }
    return "";
}
// mergeRows, csvplus.go:571-583 (right/probe wins collisions)
static Row merge_rows(const Row& l, const Row& r) {
    Row m; m.reserve(l.size() + r.size());
    for (auto& kv : l) m[kv.first] = kv.second;
    for (auto& kv : r) m[kv.first] = kv.second;
    return m;
}

// indexImpl.dedup, csvplus.go:810-867 — bug-compatible with the trailing-singleton loss (SURVEY §Q1).
// resolve(lo, hi) returns the chosen absolute row position in [lo,hi), or -1 for "empty row".
static void index_dedup(Index& ix, const std::function<long(size_t, size_t)>& resolve) {
    auto& rows = ix.rows;
    size_t lower;
    for (lower = 1; lower < rows.size(); lower++) if (equal_rows(ix.columns, rows[lower - 1], rows[lower])) break;
    if (lower >= rows.size()) return;
    size_t dest = lower - 1;
    while (lower < rows.size()) {
        std::vector<std::string> values; row_select_values(rows[lower], ix.columns, values);
        size_t upper = lower + go_search(rows.size() - lower, [&](size_t i) { return index_cmp(ix, lower + i, values, false); });
        long pick = resolve(lower - 1, upper);
        Row row; if (pick >= 0) row = rows[(size_t)pick];
        lower = upper + 1;
        if (row.size() >= ix.columns.size()) { rows[dest] = row; dest++; }
        while (lower < rows.size()) {
            if (equal_rows(ix.columns, rows[lower - 1], rows[lower])) break;
            rows[dest] = rows[lower - 1]; lower++; dest++;
        }
    }
    rows.resize(dest);
}

// ---------------------------------------------------------------- encoding/csv.Writer restated (SURVEY App. B)
static bool field_needs_quotes(const std::string& f, uint32_t comma) {  // (*Writer).fieldNeedsQuotes
    if (f.empty()) return false;
    if (f == "\\.") return true;
    if (comma < 0x80) { if (f.find(char(comma)) != std::string::npos) return true; }
    else if (f.find(encode_rune(comma)) != std::string::npos) return true;
    if (f.find_first_of("\"\r\n") != std::string::npos) return true;
    int w; uint32_t r1 = decode_rune((const uint8_t*)f.data(), f.size(), &w);
    return is_space_rune(r1);
}
static void csv_write_record(std::string& out, const std::vector<std::string>& rec) {  // (*Writer).Write, UseCRLF=false
    for (size_t n = 0; n < rec.size(); n++) {
        if (n > 0) out += ',';
        const std::string& f = rec[n];
        if (!field_needs_quotes(f, ',')) { out += f; continue; }
        out += '"';
        for (char c : f) { if (c == '"') out += "\"\""; else out += c; }  // \r and \n written as is
        out += '"';
    }
    out += '\n';
}

// parse a serialised string list: "a\0b\0c\0" with count
static std::vector<std::string> unpack_list(const char* buf, const int64_t* lens, int n) {
    std::vector<std::string> v; size_t off = 0;
    for (int i = 0; i < n; i++) { v.emplace_back(buf + off, (size_t)lens[i]); off += lens[i]; }
    return v;
}

}  // namespace

// =================================================================== C API (ctypes)
extern "C" {

struct orc_opts {
    uint32_t comma, comment;
    int32_t fields_per_record;
    uint8_t lazy_quotes, trim_leading_space, header_from_first_row, _pad;
};

typedef struct Result orc_result;
typedef struct Index orc_index;
typedef struct Pred orc_pred;

// low-level: encoding/csv records only (KAT tests for App. A.3).  Output: records serialised as
// fields joined by \x1f and records by \x1e into `out` (caller-sized); returns #records, err kind in *err.
int64_t orc_csv_records(const uint8_t* p, uint64_t n, const orc_opts* o, char* out, uint64_t cap, uint64_t* out_len, int* err) {
    CsvOpts c; c.comma = o->comma; c.comment = o->comment; c.lazy_quotes = o->lazy_quotes; c.trim_leading_space = o->trim_leading_space;
    c.fields_per_record = o->fields_per_record;
    CsvReader rd(p, n, c);
    std::vector<std::string> rec; std::string s; int64_t cnt = 0; *err = 0;
    for (;;) {
        int e; int rc = rd.read(rec, &e);
        if (rc == 1) break;
        if (rc == 2) { *err = e; break; }
        for (size_t i = 0; i < rec.size(); i++) { if (i) s += '\x1f'; s += rec[i]; }
        s += '\x1e'; cnt++;
    }
    *out_len = s.size();
    if (s.size() <= cap) memcpy(out, s.data(), s.size());
    return cnt;
}

// Take(FromFile(...)[.SelectColumns/.ExpectHeader/.AssumeHeader]) pulled to completion (csvplus.go:1080-1146).
// header spec: names packed back-to-back with lens, idx[i] = -1 search / >=0 fixed; nspec==0 => header from file.
orc_result* orc_reader_rows(const uint8_t* p, uint64_t n, const orc_opts* o, const char* names, const int64_t* name_lens,
                            const int32_t* idx, int nspec) {
    CsvOpts c; c.comma = o->comma; c.comment = o->comment; c.lazy_quotes = o->lazy_quotes; c.trim_leading_space = o->trim_leading_space;
    c.fields_per_record = o->fields_per_record;
    HeaderSpec spec; spec.from_first_row = o->header_from_first_row;
    auto nm = unpack_list(names, name_lens, nspec);
    for (int i = 0; i < nspec; i++) spec.cols.emplace_back(nm[i], idx[i]);
    auto* r = new Result();
    reader_iterate(p, n, c, spec, *r, [&](Row& row) { r->rows.push_back(std::move(row)); return std::string(); });
    return r;
}

// fused pull used by the CPU baseline: Reader(+SelectColumns) -> Filter(pred) -> ToRows in one streaming pass,
// exactly the reference's closure chain for BASELINE config 1/2 (csvplus.go:276-286, :483-490).
orc_result* orc_reader_filter_rows(const uint8_t* p, uint64_t n, const orc_opts* o, const char* names, const int64_t* name_lens,
                                   const int32_t* idx, int nspec, const orc_pred* pred) {
    CsvOpts c; c.comma = o->comma; c.comment = o->comment; c.lazy_quotes = o->lazy_quotes; c.trim_leading_space = o->trim_leading_space;
    c.fields_per_record = o->fields_per_record;
    HeaderSpec spec; spec.from_first_row = o->header_from_first_row;
    auto nm = unpack_list(names, name_lens, nspec);
    for (int i = 0; i < nspec; i++) spec.cols.emplace_back(nm[i], idx[i]);
    auto* r = new Result();
    reader_iterate(p, n, c, spec, *r, [&](Row& row) { if (!pred || pred->eval(row)) r->rows.push_back(std::move(row)); return std::string(); });
    return r;
}

void orc_result_free(orc_result* r) { delete r; }
int64_t orc_result_nrows(const orc_result* r) { return (int64_t)r->rows.size(); }
int orc_result_failed(const orc_result* r) { return r->failed; }
uint64_t orc_result_line(const orc_result* r) { return r->line; }
int orc_result_kind(const orc_result* r) { return r->kind; }
int64_t orc_result_error(const orc_result* r, char* out, uint64_t cap) {
    std::string e = r->error();
    if (e.size() < cap) { memcpy(out, e.data(), e.size()); out[e.size()] = 0; }
    return (int64_t)e.size();
}
// sorted column names of row i joined by \x1f
int64_t orc_result_row_header(const orc_result* r, int64_t i, char* out, uint64_t cap) {
    std::vector<std::string> h; for (auto& kv : r->rows[(size_t)i]) h.push_back(kv.first);
    std::sort(h.begin(), h.end());
    std::string s; for (size_t k = 0; k < h.size(); k++) { if (k) s += '\x1f'; s += h[k]; }
    if (s.size() < cap) { memcpy(out, s.data(), s.size()); out[s.size()] = 0; }
    return (int64_t)s.size();
}
// export one column Arrow-style: offsets[nrows+1] (int64) + data.  present[i]=0 where the row lacks the column.
// Call with data==NULL to size.  Returns total data bytes.
int64_t orc_result_column(const orc_result* r, const char* name, int64_t name_len, int64_t* offsets, uint8_t* data, uint8_t* present) {
    std::string col(name, (size_t)name_len);
    int64_t off = 0;
    for (size_t i = 0; i < r->rows.size(); i++) {
        auto it = r->rows[i].find(col);
        if (offsets) offsets[i] = off;
        if (present) present[i] = it != r->rows[i].end();
        if (it != r->rows[i].end()) { if (data) memcpy(data + off, it->second.data(), it->second.size()); off += (int64_t)it->second.size(); }
    }
    if (offsets) offsets[r->rows.size()] = off;
    return off;
}
int64_t orc_row_string(const orc_result* r, int64_t i, char* out, uint64_t cap) {
    std::string s = row_string(r->rows[(size_t)i]);
    if (s.size() < cap) { memcpy(out, s.data(), s.size()); out[s.size()] = 0; }
    return (int64_t)s.size();
}

// build a Result from columns (TakeRows of literal rows): ncols columns, each Arrow-style.
orc_result* orc_result_from_columns(int ncols, const char* names, const int64_t* name_lens, const int64_t* const* offsets,
                                    const uint8_t* const* data, int64_t nrows) {
    auto nm = unpack_list(names, name_lens, ncols);
    auto* r = new Result(); r->rows.resize((size_t)nrows);
    for (int c = 0; c < ncols; c++)
        for (int64_t i = 0; i < nrows; i++)
            r->rows[(size_t)i][nm[c]] = std::string((const char*)data[c] + offsets[c][i], (size_t)(offsets[c][i + 1] - offsets[c][i]));
    return r;
}

// ---- predicates
orc_pred* orc_pred_like(int n, const char* keys, const int64_t* key_lens, const char* vals, const int64_t* val_lens) {
    auto k = unpack_list(keys, key_lens, n); auto v = unpack_list(vals, val_lens, n);
    auto* p = new Pred(); p->op = 0; for (int i = 0; i < n; i++) p->match[k[i]] = v[i];
    return p;
}
orc_pred* orc_pred_combine(int op, int n, orc_pred* const* kids) {  // op 1 ALL, 2 ANY, 3 NOT; copies children
    auto* p = new Pred(); p->op = op; for (int i = 0; i < n; i++) p->kids.push_back(*kids[i]);
    return p;
}
void orc_pred_free(orc_pred* p) { delete p; }

// DataSource.Filter, csvplus.go:276-286
orc_result* orc_filter(const orc_result* src, const orc_pred* pred) {
    auto* r = new Result();
    for (auto& row : src->rows) if (pred->eval(row)) r->rows.push_back(row);
    r->failed = src->failed; r->line = src->line; r->msg = src->msg; r->kind = src->kind;
    return r;
}
// DataSource.SelectColumns, csvplus.go:511-525 (errors wrap with the 0-based iterate() index, csvplus.go:243,
// when the source is a row slice; through a Reader the record ordinal applies — callers pass `line_base`:
// line = line_base + i).
orc_result* orc_select(const orc_result* src, int n, const char* names, const int64_t* name_lens, uint64_t line_base) {
    auto cols = unpack_list(names, name_lens, n);
    auto* r = new Result();
    for (size_t i = 0; i < src->rows.size(); i++) {
        Row out; std::string e = row_select(src->rows[i], cols, out);
        if (!e.empty()) { r->failed = true; r->line = line_base + i; r->msg = e; r->kind = E_OTHER; return r; }
        r->rows.push_back(std::move(out));
    }
    r->failed = src->failed; r->line = src->line; r->msg = src->msg; r->kind = src->kind;
    return r;
}

// DataSource.Top / Drop / TakeWhile / DropWhile, csvplus.go:313-374, and DropColumns :493-507.  A source that stops early
// (Top, TakeWhile return io.EOF) never reaches an error further down the input.
// mode 0 Top(n), 1 Drop(n), 2 TakeWhile(pred), 3 DropWhile(pred)
orc_result* orc_cut(const orc_result* src, int mode, uint64_t n, const orc_pred* pred) {
    auto* r = new Result();
    bool stopped = false, yield = false;
    uint64_t counter = n;
    for (auto& row : src->rows) {
        if (mode == 0) { if (counter == 0) { stopped = true; break; } counter--; r->rows.push_back(row); }
        else if (mode == 1) { if (counter == 0) r->rows.push_back(row); else counter--; }
        else if (mode == 2) { if (!pred->eval(row)) { stopped = true; break; } r->rows.push_back(row); }
        else { if ((yield = yield || !pred->eval(row))) r->rows.push_back(row); }
    }
    // Top(n) asks for one more row before it stops (csvplus.go:317-323): with exactly n rows delivered before an error
    // of the source the error still surfaces; TakeWhile stops on the first failing row it SEES
    if (!stopped) { r->failed = src->failed; r->line = src->line; r->msg = src->msg; r->kind = src->kind; }
    return r;
}
orc_result* orc_drop_columns(const orc_result* src, int n, const char* names, const int64_t* name_lens) {
    auto cols = unpack_list(names, name_lens, n);
    auto* r = new Result();
    for (auto& row : src->rows) {
        Row out = row;
        for (auto& c : cols) out.erase(c);
        r->rows.push_back(std::move(out));
    }
    r->failed = src->failed; r->line = src->line; r->msg = src->msg; r->kind = src->kind;
    return r;
}

// ---- index
// IndexOn / UniqueIndexOn, csvplus.go:527-537.  err text (if any) copied to errbuf; returns NULL on error.
orc_index* orc_index_create(const orc_result* src, int n, const char* names, const int64_t* name_lens, int unique, int stable,
                            char* errbuf, uint64_t cap) {
    auto cols = unpack_list(names, name_lens, n);
    auto* ix = new Index();
    std::string e = create_index(*src, cols, stable != 0, *ix);
    if (e.empty() && unique && ix->rows.size() >= 2) e = check_unique(*ix);
    if (!e.empty()) { if (e.size() < cap) { memcpy(errbuf, e.data(), e.size()); errbuf[e.size()] = 0; } delete ix; return nullptr; }
    if (cap) errbuf[0] = 0;
    return ix;
}
void orc_index_free(orc_index* ix) { delete ix; }
int64_t orc_index_nrows(const orc_index* ix) { return (int64_t)ix->rows.size(); }
// Index.Iterate as a Result (sorted rows), csvplus.go:618-620
orc_result* orc_index_rows(const orc_index* ix) { auto* r = new Result(); r->rows = ix->rows; return r; }
// Index.Find, csvplus.go:625-627
orc_result* orc_index_find(const orc_index* ix, int n, const char* vals, const int64_t* val_lens) {
    auto v = unpack_list(vals, val_lens, n);
    auto lu = index_find(*ix, v);
    auto* r = new Result(); r->rows.assign(ix->rows.begin() + lu.first, ix->rows.begin() + lu.second);
    return r;
}
// DataSource.Join, csvplus.go:545-569.  n==0 => natural join on index columns.
orc_result* orc_join(const orc_result* src, const orc_index* ix, int n, const char* names, const int64_t* name_lens, uint64_t line_base) {
    auto cols = n ? unpack_list(names, name_lens, n) : ix->columns;
    auto* r = new Result();
    std::vector<std::string> values;
    for (size_t k = 0; k < src->rows.size(); k++) {
        std::string e = row_select_values(src->rows[k], cols, values);
        if (!e.empty()) { r->failed = true; r->line = line_base + k; r->msg = e; r->kind = E_OTHER; return r; }
        size_t nn = ix->rows.size();
        for (size_t i = index_first(*ix, values); i < nn && !index_cmp(*ix, i, values, false); i++)
            r->rows.push_back(merge_rows(ix->rows[i], src->rows[k]));
    }
    r->failed = src->failed; r->line = src->line; r->msg = src->msg; r->kind = src->kind;
    return r;
}
// DataSource.Except, csvplus.go:588-608
orc_result* orc_except(const orc_result* src, const orc_index* ix, int n, const char* names, const int64_t* name_lens) {
    auto cols = n ? unpack_list(names, name_lens, n) : ix->columns;
    auto* r = new Result();
    std::vector<std::string> values;
    for (auto& row : src->rows) {
        std::string e = row_select_values(row, cols, values);
        if (!e.empty()) { r->failed = true; r->msg = e; r->kind = E_OTHER; return r; }
        size_t i = index_first(*ix, values);
        bool has = i < ix->rows.size() && !index_cmp(*ix, i, values, false);  // indexImpl.has :899-905
        if (!has) r->rows.push_back(row);
    }
    return r;
}
// Index.ResolveDuplicates with a built-in tie-order-independent resolver family (SURVEY §8d cfg 5):
// mode 0: keep the row whose `col` value is bytewise smallest (ties: any — values equal);
// mode 1: return an empty row (drop the whole group);  mode 2: keep first row of the run as sorted.
void orc_index_dedup(orc_index* ix, int mode, const char* col, int64_t col_len) {
    std::string c(col ? col : "", (size_t)col_len);
    index_dedup(*ix, [&](size_t lo, size_t hi) -> long {
        if (mode == 1) return -1;
        if (mode == 2) return (long)lo;
        size_t best = lo;
        for (size_t i = lo + 1; i < hi; i++) if (str_cmp(getv(ix->rows[i], c), getv(ix->rows[best], c)) < 0) best = i;
        return (long)best;
    });
}

// DataSource.ToCsv, csvplus.go:379-406 (+ encoding/csv.Writer).  Returns bytes; err text to errbuf.
int64_t orc_to_csv(const orc_result* src, int n, const char* names, const int64_t* name_lens, uint8_t* out, uint64_t cap,
                   char* errbuf, uint64_t ecap) {
    auto cols = unpack_list(names, name_lens, n);
    std::string s; csv_write_record(s, cols);
    std::vector<std::string> values;
    if (ecap) errbuf[0] = 0;
    for (size_t k = 0; k < src->rows.size(); k++) {
        std::string e = row_select_values(src->rows[k], cols, values);
        if (!e.empty()) { if (e.size() < ecap) { memcpy(errbuf, e.data(), e.size()); errbuf[e.size()] = 0; } break; }
        csv_write_record(s, values);
    }
    if (out && s.size() <= cap) memcpy(out, s.data(), s.size());
    return (int64_t)s.size();
}

}  // extern "C"
