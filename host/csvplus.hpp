// csvplus.hpp — header-only C++ mirror of the csvplus Go API (csvplus.go) over the C ABI of
// include/csvplus_b200.h.  The reference's language (Go) has no toolchain in this image; the reference
// is compiled code, so the host side above the C ABI is written in C++ with the reference's names,
// argument meaning and error text.  A DataSource is a plan; sinks lower it to C-ABI calls (CUDA kernels).
// Opaque std::function closures (Filter(func), Map) run on the host at a materialisation boundary
// and the rows are uploaded again with TakeRows semantics — exactly what the cgo wrapper does for Go
// closures (INTEGRATION.md).  There is no CPU fallback: without a GPU every sink throws.
#pragma once
#include <sys/stat.h>

#include <algorithm>
#include <cerrno>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <fstream>
#include <ostream>
#include <stdexcept>
#include <string>
#include <variant>
#include <vector>

#include "../include/csvplus_b200.h"

namespace csvplus {

using Row = std::map<std::string, std::string>;  // map[string]string, csvplus.go:59
using RowFunc = std::function<void(const Row&)>;

struct DataSourceError : std::runtime_error {  // csvplus.go:1230-1238
    uint64_t Line; std::string Err;
    DataSourceError(uint64_t line, const std::string& err)
        : std::runtime_error("row " + std::to_string(line) + ": " + err), Line(line), Err(err) {}
};
struct Error : std::runtime_error { using std::runtime_error::runtime_error; };

namespace detail {
inline cpb_ctx* ctx() {
    static cpb_ctx* c = [] {
        cpb_ctx* h = nullptr;
        if (cpb_init(0, &h) != CPB_OK) throw Error("csvplus: no usable CUDA device (there is no CPU fallback)");
        return h;
    }();
    return c;
}
inline void check(int st, const cpb_error& e) {
    if (st == CPB_OK) return;
    if (st == CPB_ERR_DATA && e.has_line) throw DataSourceError(e.line, e.msg);
    throw Error(e.msg[0] ? e.msg : cpb_last_error(ctx()));
}
struct Strs {
    std::vector<std::string> keep; std::vector<cpb_str> v;
    explicit Strs(const std::vector<std::string>& s) : keep(s) { for (auto& x : keep) v.push_back(cpb_str{x.data(), x.size()}); if (v.empty()) v.push_back(cpb_str{nullptr, 0}); }
};
// the pinned host buffer a sink serialises its batches into.  write(out, into): into(buf, cap, &n, &err) is a
// cpb_table_to_*_into call, which writes nothing when its n exceeds cap: the buffer then grows and the call is repeated.
struct Pinned {
    void* p = nullptr; uint64_t cap = 0;
    ~Pinned() { if (p) cpb_host_free(ctx(), p); }
    void reserve(uint64_t n) {  // at least n bytes (the contents are not kept)
        if (n <= cap) return;
        if (p) cpb_host_free(ctx(), p);
        p = nullptr; cap = 0;
        if (cpb_host_alloc(ctx(), n, &p) != CPB_OK) throw Error(cpb_last_error(ctx()));
        cap = n;
    }
    template <class Into> void write(std::ostream& out, const Into& into) {
        for (;;) {
            uint64_t n = 0; cpb_error e{};
            const int st = into(p, cap, &n, &e);
            if (st == CPB_ERR_ARG && n > cap) {
                if (p) cpb_host_free(ctx(), p);
                p = nullptr; cap = 0;
                if (cpb_host_alloc(ctx(), n + n / 4 + 64, &p) != CPB_OK) throw Error(cpb_last_error(ctx()));
                cap = n + n / 4 + 64;
                continue;
            }
            check(st, e);
            out.write((const char*)p, (std::streamsize)n);
            return;
        }
    }
};
}  // namespace detail

// bytes per push of an input (cpb_stream_*): FromFile / FromString inputs larger than this are parsed in batches of whole
// records, smaller ones are one push
inline uint64_t& StreamBatchBytes() { static uint64_t v = 128ull << 20; return v; }

// maps nbytes of device memory into the context's pool ahead of time (cpb_pool_reserve); optional
inline void Reserve(uint64_t nbytes) { if (cpb_pool_reserve(detail::ctx(), nbytes) != CPB_OK) throw Error(cpb_last_error(detail::ctx())); }

// ---------------------------------------------------------------- predicates (csvplus.go:1243-1293)
struct Predicate {
    int op = -1;  // CPB_PRED_*; -1 = opaque host function
    Row match; std::vector<Predicate> kids; std::function<bool(const Row&)> fn;
    bool operator()(const Row& r) const {
        switch (op) {
            case CPB_PRED_LIKE: for (auto& kv : match) { auto it = r.find(kv.first); if (it == r.end() || it->second != kv.second) return false; } return true;
            case CPB_PRED_ALL: for (auto& k : kids) if (!k(r)) return false; return true;
            case CPB_PRED_ANY: for (auto& k : kids) if (k(r)) return true; return false;
            case CPB_PRED_NOT: return !kids[0](r);
            default: return fn(r);
        }
    }
    // the device compiles the tree: no opaque function in it, within the CPB_PRED_MAX_* limits (every Like pair counted
    // as a term, a set term as one); a declined tree runs on host rows
    bool lowerable() const { int terms = 0, ops = 0; return fits(0, terms, ops) && terms <= CPB_PRED_MAX_TERMS && ops <= CPB_PRED_MAX_OPS; }
    bool fits(int depth, int& terms, int& ops) const {
        if (op < 0 || depth > CPB_PRED_MAX_DEPTH) return false;
        if (op == CPB_PRED_LIKE) { terms += (int)match.size(); ops += 2 * (int)match.size() - 1; return true; }
        if (kids.empty()) { ops += 1; return true; }
        const std::vector<int> set = set_of();
        int nsets = 0, grouped = 0;
        for (size_t i = 0; i < kids.size(); i++) if (set[i] >= 0) { grouped++; if (set[i] >= nsets) nsets = set[i] + 1; }
        terms += nsets; ops += nsets;  // one term each; its Likes add no depth
        ops += op == CPB_PRED_NOT ? 1 : (int)kids.size() - grouped + nsets - 1;
        for (size_t i = 0; i < kids.size(); i++) if (set[i] < 0 && !kids[i].fits(depth + 1, terms, ops)) return false;
        return true;
    }
    // The set terms of an Any node (CPB_PRED_SET_MIN, include/csvplus_b200.h): per child the set term it belongs to (0, 1, ...
    // in the order of their first children), -1 for none.  A group of Likes over one set of column names is a set term when
    // it has CPB_PRED_SET_MIN children or more and its literals fit an index key image.
    std::vector<int> set_of() const {
        std::vector<int> out(kids.size(), -1);
        if (op != CPB_PRED_ANY || kids.size() < CPB_PRED_SET_MIN) return out;
        std::map<std::vector<std::string>, std::vector<size_t>> groups;  // key names (sorted: Row is an ordered map) -> children
        for (size_t i = 0; i < kids.size(); i++) {
            const Predicate& k = kids[i];
            if (k.op != CPB_PRED_LIKE || k.match.empty() || k.match.size() > 16) continue;
            std::vector<std::string> names;
            for (auto& kv : k.match) names.push_back(kv.first);
            groups[names].push_back(i);
        }
        std::vector<const std::vector<size_t>*> sets;
        for (auto& g : groups) {
            if (g.second.size() < CPB_PRED_SET_MIN) continue;
            uint64_t image = 0;  // the key image of an index over the literals: every value padded to w, then its length
            for (auto& name : g.first) {
                uint64_t w = 0;
                for (size_t i : g.second) w = std::max<uint64_t>(w, kids[i].match.at(name).size());
                image += w + (w < 255 ? 1 : w < 65535 ? 2 : 4);
            }
            if (image <= 4096) sets.push_back(&g.second);
        }
        std::sort(sets.begin(), sets.end(), [](auto a, auto b) { return (*a)[0] < (*b)[0]; });
        for (size_t s = 0; s < sets.size(); s++) for (size_t i : *sets[s]) out[i] = (int)s;
        return out;
    }
    // the distinct columns the Like terms compare
    void columns(std::vector<std::string>& out) const {
        for (auto& kv : match) if (std::find(out.begin(), out.end(), kv.first) == out.end()) out.push_back(kv.first);
        for (auto& k : kids) k.columns(out);
    }
};
inline Predicate Like(const Row& match) {
    if (match.empty()) throw std::logic_error("empty match row in Like() predicate");
    Predicate p; p.op = CPB_PRED_LIKE; p.match = match; return p;
}
inline Predicate All(std::vector<Predicate> k) { Predicate p; p.op = CPB_PRED_ALL; p.kids = std::move(k); return p; }
inline Predicate Any(std::vector<Predicate> k) { Predicate p; p.op = CPB_PRED_ANY; p.kids = std::move(k); return p; }
inline Predicate Not(Predicate k) { Predicate p; p.op = CPB_PRED_NOT; p.kids = {std::move(k)}; return p; }
inline Predicate Func(std::function<bool(const Row&)> f) { Predicate p; p.fn = std::move(f); return p; }

namespace detail {
// owns the cpb_pred tree.  The Likes of a set term are lowered in bulk: one keys array for all of them, their values in one
// array pointing at the Predicate's strings (so the Predicate must outlive the CPred), their nodes in one array.
struct CPred {
    std::vector<std::unique_ptr<CPred>> kids; std::vector<const cpb_pred*> kid_ptrs;
    std::vector<std::string> ks, vs; std::vector<cpb_str> kstr, vstr; cpb_pred p{};
    struct Set { std::vector<cpb_str> keys, values; std::vector<cpb_pred> nodes; };
    std::vector<Set> sets;
    explicit CPred(const Predicate& q) {
        p.op = q.op;
        if (q.op == CPB_PRED_LIKE) {
            for (auto& kv : q.match) { ks.push_back(kv.first); vs.push_back(kv.second); }
            for (size_t i = 0; i < ks.size(); i++) { kstr.push_back(cpb_str{ks[i].data(), ks[i].size()}); vstr.push_back(cpb_str{vs[i].data(), vs[i].size()}); }
            p.n = (int)ks.size(); p.keys = kstr.data(); p.values = vstr.data();
        } else {
            const std::vector<int> set = q.set_of();
            std::vector<size_t> nodes, values;  // per set: reserved up front, the nodes and values must not move once pointed at
            for (size_t i = 0; i < set.size(); i++) {
                if (set[i] < 0) continue;
                if (set[i] >= (int)nodes.size()) { nodes.resize(set[i] + 1); values.resize(set[i] + 1); }
                nodes[set[i]]++; values[set[i]] += q.kids[i].match.size();
            }
            sets.resize(nodes.size());
            for (size_t s = 0; s < sets.size(); s++) { sets[s].nodes.reserve(nodes[s]); sets[s].values.reserve(values[s]); }
            for (size_t i = 0; i < q.kids.size(); i++) {
                if (set[i] < 0) { kids.emplace_back(new CPred(q.kids[i])); kid_ptrs.push_back(&kids.back()->p); continue; }
                Set& s = sets[set[i]];
                const Row& m = q.kids[i].match;  // (a Row is ordered: every Like of the set has its keys in one order)
                if (s.keys.empty()) for (auto& kv : m) s.keys.push_back(cpb_str{kv.first.data(), kv.first.size()});
                cpb_pred node{};
                node.op = CPB_PRED_LIKE; node.n = (int)m.size(); node.keys = s.keys.data(); node.values = s.values.data() + s.values.size();
                for (auto& kv : m) s.values.push_back(cpb_str{kv.second.data(), kv.second.size()});
                s.nodes.push_back(node);
                kid_ptrs.push_back(&s.nodes.back());
            }
            p.n = (int)kid_ptrs.size(); p.children = kid_ptrs.data();
        }
    }
};
}  // namespace detail

// ---------------------------------------------------------------- Table / Index handles
class Index;
class Table {
public:
    explicit Table(cpb_table* h = nullptr) : h_(h, cpb_table_free) {}
    cpb_table* get() const { return h_.get(); }
    int64_t size() const { return h_ ? cpb_table_num_rows(h_.get()) : 0; }
    std::vector<std::string> columns() const {
        std::vector<std::string> out;
        for (int i = 0; h_ && i < cpb_table_num_cols(h_.get()); i++) { cpb_str s; cpb_table_col_name(h_.get(), i, &s); out.emplace_back(s.ptr, s.len); }
        return out;
    }
    std::vector<Row> rows() const {
        std::vector<Row> out((size_t)size());
        auto cols = columns();
        for (size_t c = 0; c < cols.size(); c++) {
            uint64_t nb = 0;
            cpb_table_col_bytes(detail::ctx(), h_.get(), (int)c, 0, size(), &nb);
            std::vector<int64_t> off((size_t)size() + 1); std::vector<uint8_t> data(nb + 1);
            if (cpb_table_fetch_column(detail::ctx(), h_.get(), (int)c, 0, size(), off.data(), data.data(), data.size()) != CPB_OK) throw Error("fetch failed");
            for (size_t i = 0; i < out.size(); i++) out[i][cols[c]] = std::string((const char*)data.data() + off[i], (size_t)(off[i + 1] - off[i]));
        }
        return out;
    }
    Table slice(int64_t lo, int64_t hi) const {  // a row-range view (cpb_table_slice)
        cpb_table* out = nullptr;
        if (cpb_table_slice(detail::ctx(), h_.get(), lo, hi, &out) != CPB_OK) throw Error(cpb_last_error(detail::ctx()));
        return Table(out);
    }
    static Table from_rows(const std::vector<Row>& rows) {  // TakeRows, csvplus.go:218
        std::vector<std::string> cols;
        if (!rows.empty()) for (auto& kv : rows[0]) cols.push_back(kv.first);
        std::vector<std::vector<int64_t>> offs(cols.size()); std::vector<std::string> datas(cols.size());
        for (size_t c = 0; c < cols.size(); c++) {
            offs[c].push_back(0);
            for (auto& r : rows) { auto it = r.find(cols[c]); if (it == r.end()) throw Error("TakeRows on the device requires rows with identical column sets"); datas[c] += it->second; offs[c].push_back((int64_t)datas[c].size()); }
            datas[c] += '\0';
        }
        detail::Strs names(cols);
        std::vector<const int64_t*> op; std::vector<const uint8_t*> dp;
        for (size_t c = 0; c < cols.size(); c++) { op.push_back(offs[c].data()); dp.push_back((const uint8_t*)datas[c].data()); }
        cpb_table* h = nullptr;
        if (cpb_table_from_host(detail::ctx(), (int)cols.size(), names.v.data(), op.data(), dp.data(), (int64_t)rows.size(), &h) != CPB_OK) throw Error("from_host failed");
        return Table(h);
    }
    // Row.ValueAsInt / ValueAsFloat64 (csvplus.go:163-205: strconv.Atoi / ParseFloat(s, 64)) of every row of a column,
    // converted on the GPU into caller-owned device memory: values[size()] (Go's value on error too), status[size()]
    // nullable (CPB_NUM_OK / _SYNTAX / _RANGE).  Returns the failing rows; strict: the first one throws Error with the
    // reference's text, as a RowFunc returning the helper's error.  An absent column throws in both modes.
    uint64_t ValuesAsInt(const std::string& column, int64_t* dev_values, uint8_t* dev_status = nullptr, bool strict = true) const {
        return convert(column, false, dev_values, dev_status, strict);
    }
    uint64_t ValuesAsFloat64(const std::string& column, double* dev_values, uint8_t* dev_status = nullptr, bool strict = true) const {
        return convert(column, true, dev_values, dev_status, strict);
    }
    // Map(func(row) Row { row[column] = value; return row }) on the GPU: a table with `column` set (replaced in place, else
    // appended; every other column shares this table's buffers).  dev_values[size()] is device memory read on the ctx
    // stream: strconv.FormatInt(v, 10), strconv.FormatFloat(x, fmt, prec, 64) (fmt e E f g G, prec -1..64), or one
    // literal value in every row.  A column of 4 GiB or more throws.
    Table WithColumn(const std::string& column, const int64_t* dev_values) const {
        return set(column, [&](cpb_str c, cpb_table** out, cpb_error* e) { return cpb_table_set_int64(detail::ctx(), h_.get(), c, dev_values, out, e); });
    }
    Table WithColumn(const std::string& column, const double* dev_values, char fmt = 'g', int prec = -1) const {
        return set(column, [&](cpb_str c, cpb_table** out, cpb_error* e) {
            return cpb_table_set_float64(detail::ctx(), h_.get(), c, dev_values, fmt, prec, out, e);
        });
    }
    Table WithColumn(const std::string& column, const std::string& value) const {
        const cpb_str v{value.data(), value.size()};
        return set(column, [&](cpb_str c, cpb_table** out, cpb_error* e) { return cpb_table_set_literal(detail::ctx(), h_.get(), c, v, out, e); });
    }
    // the rows whose dev_keep[row] byte (device memory, size() bytes) is nonzero, in order
    Table FilterMask(const uint8_t* dev_keep) const {
        cpb_table* out = nullptr; cpb_error e{};
        detail::check(cpb_table_filter_flags(detail::ctx(), h_.get(), dev_keep, &out, &e), e);
        return Table(out);
    }
private:
    template <class F> Table set(const std::string& column, F call) const {
        cpb_table* out = nullptr; cpb_error e{};
        detail::check(call(cpb_str{column.data(), column.size()}, &out, &e), e);
        return Table(out);
    }
    uint64_t convert(const std::string& column, bool is_float, void* values, uint8_t* status, bool strict) const {
        cpb_error e{}; uint64_t nbad = 0;
        const cpb_str c{column.data(), column.size()};
        const int st = is_float ? cpb_table_column_as_float64(detail::ctx(), h_.get(), c, (double*)values, status, &nbad, &e)
                                : cpb_table_column_as_int64(detail::ctx(), h_.get(), c, (int64_t*)values, status, &nbad, &e);
        if (st == CPB_ERR_DATA && (strict || e.kind == CPB_E_MISSING_COLUMN)) throw Error(e.msg);
        if (st != CPB_OK && st != CPB_ERR_DATA) throw Error(e.msg[0] ? e.msg : cpb_last_error(detail::ctx()));
        return nbad;
    }
    std::shared_ptr<cpb_table> h_;
};

class DataSource;
class Index {  // csvplus.go:610-653
public:
    Index(cpb_index* h, std::vector<std::string> cols) : h_(h, cpb_index_free), columns_(std::move(cols)) {}
    cpb_index* get() const { return h_.get(); }
    const std::vector<std::string>& columns() const { return columns_; }
    int64_t size() const { return cpb_index_num_rows(h_.get()); }
    Table table() const { cpb_table* t = nullptr; cpb_index_table(detail::ctx(), h_.get(), &t); return Table(t); }
    inline DataSource Find(const std::vector<std::string>& values) const;
    Index SubIndex(const std::vector<std::string>& values) const {
        if (values.size() >= columns_.size()) throw std::logic_error("too many values in SubIndex()");
        detail::Strs v(values); cpb_index* s = nullptr;
        if (cpb_index_sub(detail::ctx(), h_.get(), v.v.data(), (int)values.size(), &s) != CPB_OK) throw Error(cpb_last_error(detail::ctx()));
        return Index(s, std::vector<std::string>(columns_.begin() + values.size(), columns_.end()));
    }
    // ResolveDuplicates, csvplus.go:651: resolve returns the position (within the group) of the row to keep, or -1
    void ResolveDuplicates(const std::function<long(const std::vector<Row>&)>& resolve, bool bug_compatible = true) {
        int64_t ng = 0, *lo = nullptr, *hi = nullptr;
        if (cpb_index_dup_groups(detail::ctx(), h_.get(), &ng, &lo, &hi) != CPB_OK) throw Error(cpb_last_error(detail::ctx()));
        std::vector<int64_t> keep((size_t)ng + 1);
        Table t = table();
        auto all = t.rows();
        for (int64_t g = 0; g < ng; g++) {
            std::vector<Row> grp(all.begin() + lo[g], all.begin() + hi[g]);
            long pick = resolve(grp);
            keep[(size_t)g] = pick < 0 ? -1 : lo[g] + pick;
        }
        cpb_free(lo); cpb_free(hi);
        if (cpb_index_dedup_apply(detail::ctx(), h_.get(), ng, keep.data(), bug_compatible) != CPB_OK) throw Error(cpb_last_error(detail::ctx()));
    }
    // WriteTo, csvplus.go:655-680: the reference's encoding/gob index file, encoded on the GPU and written in row-range
    // batches through one pinned buffer.  A path that cannot be created throws and leaves no file; any later error
    // removes the file.
    void WriteTo(const std::string& name) const {
        std::ofstream f(name, std::ios::binary | std::ios::trunc);
        if (!f) throw Error("open " + name + ": " + strerror(errno));
        try {
            // one pinned buffer sized up front: the prefix (the key column names and about 100 bytes more) and then every
            // batch (at most the rows' total, and less than 4 GiB) are serialised in one call each
            detail::Pinned buf;
            uint64_t bound = 256, total = 0, plen = 0;
            for (auto& c : columns_) bound += c.size() + 10;
            buf.reserve(bound);
            buf.write(f, [&](void* p, uint64_t cap, uint64_t* n, cpb_error* e) {
                const int st = cpb_index_gob_begin(detail::ctx(), h_.get(), p, cap, n, &total, e);
                plen = *n;
                return st;
            });
            buf.reserve(std::min<uint64_t>(total - plen, uint64_t(1) << 32) + 64);
            const int64_t n = size();
            for (int64_t lo = 0, step = int64_t(1) << 24; lo < n;) {
                const int64_t hi = std::min(n, lo + step);
                bool too_large = false;  // CPB_E_TOO_LARGE: the batch is 4 GiB or more
                try {
                    buf.write(f, [&](void* dst, uint64_t cap, uint64_t* w, cpb_error* e) {
                        const int st = cpb_index_gob_into(detail::ctx(), h_.get(), lo, hi, dst, cap, w, e);
                        too_large = st == CPB_ERR_DATA && e->kind == CPB_E_TOO_LARGE;
                        return st;
                    });
                } catch (const Error&) {
                    if (!too_large || hi - lo < 2) throw;
                    step = (hi - lo) / 2;  // halve the batch
                    continue;
                }
                lo = hi;
            }
            f.close();
            if (!f) throw Error("write " + name + " failed");
        } catch (...) { f.close(); std::remove(name.c_str()); throw; }
    }
private:
    std::shared_ptr<cpb_index> h_; std::vector<std::string> columns_;
};

// ---------------------------------------------------------------- Reader (csvplus.go:922-1076)
class Reader {
public:
    // fills the next piece of the input; true when it is the last one
    using Pieces = std::function<bool(std::string&)>;
    // pieces: a function that starts reading the input and returns its pieces
    explicit Reader(std::function<Pieces()> pieces) : pieces_(std::move(pieces)) {}
    Reader& Delimiter(char32_t c) { delimiter_ = c; return *this; }
    Reader& CommentChar(char32_t c) { comment_ = c; return *this; }
    Reader& LazyQuotes() { lazy_ = true; return *this; }
    Reader& TrimLeadingSpace() { trim_ = true; return *this; }
    Reader& NumFields(int n) { num_fields_ = n; return *this; }
    Reader& NumFieldsAuto() { return NumFields(0); }
    Reader& NumFieldsAny() { return NumFields(-1); }
    Reader& SelectColumns(const std::vector<std::string>& names) {
        if (names.empty()) throw std::logic_error("empty header spec");
        header_.clear();
        for (auto& n : names) { for (auto& h : header_) if (h.first == n) throw std::logic_error("header spec: duplicate column name: " + n); header_.emplace_back(n, -1); }
        from_first_row_ = true; return *this;
    }
    Reader& ExpectHeader(const std::map<std::string, int>& spec) {
        if (spec.empty()) throw std::logic_error("empty header spec");
        header_.assign(spec.begin(), spec.end()); from_first_row_ = true; return *this;
    }
    Reader& AssumeHeader(const std::map<std::string, int>& spec) {
        if (spec.empty()) throw std::logic_error("Empty header spec");
        for (auto& kv : spec) if (kv.second < 0) throw std::logic_error("header spec: negative index for column " + kv.first);
        header_.assign(spec.begin(), spec.end()); from_first_row_ = false; return *this;
    }
    // one batch of Reader.Iterate: its rows, the DataSourceError raised after them (last batch only) and whether the
    // input was pushed in more than one piece.  fn returns false to stop reading the input.
    using BatchFn = std::function<bool(Table, std::unique_ptr<DataSourceError>, bool several)>;
    // Reader.Iterate lowered to cpb_stream_*: an input that fits one piece is one push, parsed as one batch
    void batches(const Predicate* pred, const BatchFn& fn) const {
        Pieces next = pieces_();
        cpb_reader_opts o{}; o.delimiter = delimiter_; o.comment = comment_; o.num_fields = num_fields_;
        o.lazy_quotes = lazy_; o.trim_leading_space = trim_; o.header_from_first_row = from_first_row_;
        std::vector<cpb_header_col> spec;
        for (auto& h : header_) spec.push_back(cpb_header_col{cpb_str{h.first.data(), h.first.size()}, h.second, 0});
        std::unique_ptr<detail::CPred> cp; if (pred) cp.reset(new detail::CPred(*pred));
        cpb_stream* sp = nullptr; cpb_error e{};
        detail::check(cpb_stream_open(detail::ctx(), &o, spec.data(), (int)spec.size(), cp ? &cp->p : nullptr, &sp, &e), e);
        std::unique_ptr<cpb_stream, void (*)(cpb_stream*)> st(sp, cpb_stream_free);
        // One cpb_stream_next per push parses every complete record pushed so far.  A batch is delivered after the next
        // piece has been pushed: that piece's host-to-device copy (the stream's copy stream) overlaps what fn does with
        // the batch on the context's stream, and it is parsed only after fn has returned.
        Table pending; bool have = false;
        bool several = false;  // known from the first piece, so every batch, the first one included, reports it
        auto deliver = [&]() -> bool { if (!have) return true; have = false; return fn(pending, nullptr, several); };
        std::string piece;  // untouched until the cpb_stream_next after its push has returned
        for (bool first = true, last = false, done = false; !last && !done; first = false) {
            last = next(piece);
            if (first) several = !last;
            if (cpb_stream_push(st.get(), piece.data(), piece.size(), last) != CPB_OK) throw Error(cpb_last_error(detail::ctx()));
            if (!deliver()) return;
            cpb_table* bt = nullptr; int fin = 0;
            const int s = cpb_stream_next(st.get(), &bt, &fin, &e);
            if (s == CPB_ERR_DATA && bt && e.has_line) {
                fn(Table(bt), std::unique_ptr<DataSourceError>(new DataSourceError(e.line, e.msg)), several);
                return;
            }
            detail::check(s, e);
            if (bt) { pending = Table(bt); have = true; }
            done = fin != 0;
        }
        deliver();
    }
private:
    std::function<Pieces()> pieces_;
    uint32_t delimiter_ = ',', comment_ = 0; int num_fields_ = 0; bool lazy_ = false, trim_ = false, from_first_row_ = true;
    std::vector<std::pair<std::string, int>> header_;
};
Reader FromFile(const std::string& name);  // csvplus.go:950 (defined below)
inline Reader FromString(std::string data) {
    auto d = std::make_shared<std::string>(std::move(data));
    return Reader([d]() -> Reader::Pieces {
        auto pos = std::make_shared<size_t>(0);
        return [d, pos](std::string& piece) {
            piece.assign(*d, *pos, (size_t)StreamBatchBytes());
            *pos += piece.size();
            return *pos >= d->size();
        };
    });
}

// ---------------------------------------------------------------- DataSource (csvplus.go:207-608)
class DataSource {
    struct Op { int kind; Predicate pred; std::vector<std::string> cols; std::shared_ptr<Index> index; uint64_t n = 0; std::function<Row(const Row&)> map; };
    enum { FILTER, SELECT, DROPCOLS, JOIN, EXCEPT, TOP, DROP, MAP };
public:
    explicit DataSource(Reader r) : reader_(new Reader(std::move(r))) {}
    explicit DataSource(Table t) : table_(new Table(std::move(t))) {}
    DataSource Filter(Predicate p) const { return with({FILTER, std::move(p)}); }
    DataSource Map(std::function<Row(const Row&)> f) const { Op o{MAP}; o.map = std::move(f); return with(std::move(o)); }
    DataSource Top(uint64_t n) const { Op o{TOP}; o.n = n; return with(std::move(o)); }
    DataSource Drop(uint64_t n) const { Op o{DROP}; o.n = n; return with(std::move(o)); }
    DataSource SelectColumns(const std::vector<std::string>& c) const { if (c.empty()) throw std::logic_error("no columns specified in SelectColumns()"); Op o{SELECT}; o.cols = c; return with(std::move(o)); }
    DataSource DropColumns(const std::vector<std::string>& c) const { if (c.empty()) throw std::logic_error("no columns specified in DropColumns()"); Op o{DROPCOLS}; o.cols = c; return with(std::move(o)); }
    DataSource Join(const Index& ix, const std::vector<std::string>& c = {}) const {
        if (c.size() > ix.columns().size()) throw std::logic_error("too many source columns in Join()");
        Op o{JOIN}; o.cols = c; o.index.reset(new Index(ix)); return with(std::move(o));
    }
    DataSource Except(const Index& ix, const std::vector<std::string>& c = {}) const {
        if (c.size() > ix.columns().size()) throw std::logic_error("too many source columns in Except()");
        Op o{EXCEPT}; o.cols = c; o.index.reset(new Index(ix)); return with(std::move(o));
    }
    // sinks: each batch of a streamed input is delivered before the next one is parsed
    void operator()(const RowFunc& fn) const {
        each([&](Table& t, std::unique_ptr<DataSourceError>& err, bool) {
            for (auto& r : t.rows()) fn(r);
            if (err) throw *err;
            return true;
        });
    }
    std::vector<Row> ToRows() const { std::vector<Row> out; (*this)([&](const Row& r) { out.push_back(r); }); return out; }
    // the plan's rows as a device table (an extension beyond the reference API, like TakeTable): the input of
    // Table::ValuesAsInt / ValuesAsFloat64.  A source error is thrown.
    Table ToTable() const { std::unique_ptr<DataSourceError> err; Table t = run(&err); if (err) throw *err; return t; }
    // ToCsv, csvplus.go:379-406: the header line once, then every batch's rows; delivered rows are written before a source
    // error is thrown
    void ToCsv(std::ostream& out, const std::vector<std::string>& columns) const {
        if (columns.empty()) throw std::logic_error("empty column list in ToCsv() function");
        detail::Strs c(columns);
        detail::Pinned buf;
        bool header = true;  // the header line once, before the first batch (csvplus.go:387)
        each([&](Table& t, std::unique_ptr<DataSourceError>& err, bool) {
            buf.write(out, [&](void* p, uint64_t cap, uint64_t* n, cpb_error* e) {
                return cpb_table_to_csv_into(detail::ctx(), t.get(), c.v.data(), (int)columns.size(), header, p, cap, n, e);
            });
            header = false;
            if (err) throw *err;
            return true;
        });
    }
    // ToCsvFile, csvplus.go:411-443: the file is removed on error
    void ToCsvFile(const std::string& name, const std::vector<std::string>& columns) const {
        try {
            std::ofstream f(name, std::ios::binary | std::ios::trunc);
            if (!f) throw Error("open " + name + ": " + strerror(errno));
            ToCsv(f, columns);
            f.close();
            if (!f) throw Error("write " + name + " failed");
        } catch (...) { std::remove(name.c_str()); throw; }
    }
    // ToJSON, csvplus.go:446-474: the GPU serialises the result in row-range batches (each < 4 GiB) into one reused
    // pinned buffer.  On a source error nothing is written when the input was pushed in one piece; an input pushed in
    // several keeps what its batches wrote (a prefix of the array without ']'), as the reference's encoder has flushed it.
    void ToJSON(std::ostream& out) const {
        detail::Pinned buf;
        bool opened = false;
        each([&](Table& t, std::unique_ptr<DataSourceError>& err, bool several) {
            if (err && !several) throw *err;
            const int64_t n = t.size(), step = int64_t(1) << 24;
            for (int64_t lo = 0; lo < n; lo += step) {
                Table p = t.slice(lo, std::min(n, lo + step));
                const bool first = !opened;
                buf.write(out, [&](void* dst, uint64_t cap, uint64_t* w, cpb_error* e) {
                    return cpb_table_to_json_into(detail::ctx(), p.get(), first, 0, dst, cap, w, e);
                });
                opened = true;
            }
            if (err) throw *err;
            return true;
        });
        out << (opened ? "]" : "[]");
    }
    Index IndexOn(const std::vector<std::string>& cols) const { return index(cols, false); }
    Index UniqueIndexOn(const std::vector<std::string>& cols) const { return index(cols, true); }
private:
    DataSource with(Op o) const { DataSource d = *this; d.ops_.push_back(std::move(o)); return d; }
    Index index(const std::vector<std::string>& cols, bool unique) const {
        if (cols.empty()) throw std::logic_error("empty column list in CreateIndex()");
        for (size_t i = 0; i < cols.size(); i++) for (size_t j = i + 1; j < cols.size(); j++) if (cols[i] == cols[j]) throw std::logic_error("duplicate column name(s) in CreateIndex()");
        std::unique_ptr<DataSourceError> err; Table t = run(&err); if (err) throw *err;
        detail::Strs c(cols); cpb_index* ix = nullptr; cpb_error e{};
        detail::check(cpb_index_build(detail::ctx(), t.get(), c.v.data(), (int)cols.size(), unique, &ix, &e), e);
        return Index(ix, cols);
    }
    // the batches' tables concatenated (cpb_table_concat); *err: the source error after them
    Table run(std::unique_ptr<DataSourceError>* err) const {
        std::vector<Table> parts;
        each([&](Table& t, std::unique_ptr<DataSourceError>& e, bool) { parts.push_back(t); *err = std::move(e); return true; });
        if (parts.size() == 1) return parts[0];
        std::vector<const cpb_table*> hs;
        for (auto& p : parts) hs.push_back(p.get());
        cpb_table* out = nullptr;
        if (cpb_table_concat(detail::ctx(), hs.data(), (int)hs.size(), &out) != CPB_OK) throw Error(cpb_last_error(detail::ctx()));
        return Table(out);
    }
    // the operations over every batch of the source, in order: fn(rows, error after them, several) returns false to stop;
    // several: the input was pushed in more than one piece.
    // Top / Drop count rows across batches; once Top has pulled n + 1 rows the input is no longer read.
    using EachFn = std::function<bool(Table&, std::unique_ptr<DataSourceError>&, bool)>;
    void each(const EachFn& fn) const {
        size_t first = 0;
        std::vector<uint64_t> seen(ops_.size(), 0);
        auto apply = [&](Table t, std::unique_ptr<DataSourceError> err, bool several) -> bool {
            bool stop = false;
            for (size_t i = first; i < ops_.size(); i++) {
                const Op& o = ops_[i]; cpb_table* out = nullptr; cpb_error e{}; detail::Strs c(o.cols);
                const uint64_t n = (uint64_t)t.size();
                switch (o.kind) {
                    case FILTER:
                        if (o.pred.lowerable()) { detail::CPred cp(o.pred); detail::check(cpb_table_filter(detail::ctx(), t.get(), &cp.p, &out), e); }
                        else { std::vector<Row> keep; for (auto& r : t.rows()) if (o.pred(r)) keep.push_back(r); t = Table::from_rows(keep); continue; }
                        break;
                    case MAP: { std::vector<Row> m; for (auto& r : t.rows()) m.push_back(o.map(r)); t = Table::from_rows(m); continue; }
                    case SELECT: detail::check(cpb_table_select(detail::ctx(), t.get(), c.v.data(), (int)o.cols.size(), &out, &e), e); break;
                    case DROPCOLS: detail::check(cpb_table_drop(detail::ctx(), t.get(), c.v.data(), (int)o.cols.size(), &out), e); break;
                    case JOIN: detail::check(cpb_join(detail::ctx(), t.get(), o.index->get(), c.v.data(), (int)o.cols.size(), &out, &e), e); break;
                    case EXCEPT: detail::check(cpb_except(detail::ctx(), t.get(), o.index->get(), c.v.data(), (int)o.cols.size(), &out, &e), e); break;
                    case TOP: {  // the reference pulls n + 1 rows then stops (io.EOF): a later error is never met
                        const uint64_t keep = o.n > seen[i] ? std::min(n, o.n - seen[i]) : 0;
                        seen[i] += n;
                        if (seen[i] > o.n) { err.reset(); stop = true; }
                        detail::check(cpb_table_slice(detail::ctx(), t.get(), 0, (int64_t)keep, &out), e);
                        break;
                    }
                    case DROP: {
                        const uint64_t lo = o.n > seen[i] ? std::min(n, o.n - seen[i]) : 0;
                        seen[i] += n;
                        detail::check(cpb_table_slice(detail::ctx(), t.get(), (int64_t)lo, (int64_t)n, &out), e);
                        break;
                    }
                }
                t = Table(out);
            }
            const bool failed = err != nullptr;
            return fn(t, err, several) && !stop && !failed;
        };
        if (reader_) {
            // a predicate over CPB_MAX_PARSE_COLS or more columns filters the parsed table instead of the parse
            std::vector<std::string> pcols;
            if (!ops_.empty() && ops_[0].kind == FILTER) ops_[0].pred.columns(pcols);
            const Predicate* fused = (!ops_.empty() && ops_[0].kind == FILTER && ops_[0].pred.lowerable() && (int)pcols.size() < CPB_MAX_PARSE_COLS)
                                         ? &ops_[0].pred : nullptr;
            if (fused) first = 1;
            reader_->batches(fused, apply);
        } else apply(*table_, nullptr, false);
    }
    std::shared_ptr<Reader> reader_; std::shared_ptr<Table> table_; std::vector<Op> ops_;
};

inline DataSource Take(const Reader& r) { return DataSource(r); }                          // csvplus.go:252
inline DataSource Take(const Index& ix) { return DataSource(ix.table()); }
inline DataSource TakeRows(const std::vector<Row>& rows) { return DataSource(Table::from_rows(rows)); }  // :218
inline DataSource Index::Find(const std::vector<std::string>& values) const {
    if (values.size() > columns_.size()) throw std::logic_error("too many columns in indexImpl.find()");
    detail::Strs v(values); cpb_table* t = nullptr;
    if (cpb_index_find(detail::ctx(), h_.get(), v.v.data(), (int)values.size(), &t) != CPB_OK) throw Error(cpb_last_error(detail::ctx()));
    return DataSource(Table(t));
}
// LoadIndex, csvplus.go:683-705: the index in a file WriteTo (or the reference) wrote, decoded on the GPU; its rows in
// file order.  A missing file throws the OS error, an empty one Error("EOF"), a cut one Error("unexpected EOF").
inline Index LoadIndex(const std::string& name) {
    std::shared_ptr<FILE> f(fopen(name.c_str(), "rb"), [](FILE* p) { if (p) fclose(p); });
    if (!f) throw Error("open " + name + ": " + strerror(errno));
    struct stat sb;
    if (fstat(fileno(f.get()), &sb) != 0) throw Error("stat " + name + ": " + strerror(errno));
    detail::Pinned buf;  // the rows are copied to the device from pinned memory
    const uint64_t size = (uint64_t)sb.st_size;
    buf.reserve(size ? size : 1);
    if (size && fread(buf.p, 1, (size_t)size, f.get()) != size) throw Error("read " + name + ": short read");
    cpb_index* ix = nullptr; cpb_error e{};
    detail::check(cpb_index_load_gob(detail::ctx(), buf.p, size, &ix, &e), e);
    std::vector<std::string> cols;
    for (int k = 0; k < cpb_index_num_keys(ix); k++) { cpb_str s; cpb_index_key_col(ix, k, &s); cols.emplace_back(s.ptr, s.len); }
    return Index(ix, cols);
}

// the file in pieces of StreamBatchBytes(): a file that fits one piece is read whole and is one push.  A regular file's
// pieces are read at their exact size, another file's (a pipe) in steps of 64 KiB: a piece is never sized above the
// bytes it holds.
inline Reader FromFile(const std::string& name) {
    return Reader([name]() -> Reader::Pieces {
        std::shared_ptr<FILE> f(fopen(name.c_str(), "rb"), [](FILE* p) { if (p) fclose(p); });
        if (!f) throw DataSourceError(1, std::string("open: ") + strerror(errno));  // mapError, csvplus.go:1216-1220
        struct stat sb;
        const bool regular = fstat(fileno(f.get()), &sb) == 0 && S_ISREG(sb.st_mode);
        auto left = std::make_shared<uint64_t>(regular ? (uint64_t)sb.st_size : 0);
        return [f, regular, left](std::string& piece) {
            const uint64_t cap = StreamBatchBytes();
            if (regular) {
                piece.resize((size_t)std::min(*left, cap));
                piece.resize(fread(&piece[0], 1, piece.size(), f.get()));
                const bool short_read = piece.size() < std::min(*left, cap);
                *left -= piece.size();
                return short_read || *left == 0;
            }
            piece.clear();
            char buf[1 << 16]; size_t n;
            while (piece.size() < cap && (n = fread(buf, 1, (size_t)std::min<uint64_t>(sizeof buf, cap - piece.size()), f.get())) > 0)
                piece.append(buf, n);
            const int c = fgetc(f.get());
            if (c == EOF) return true;
            ungetc(c, f.get());
            return false;
        };
    });
}

}  // namespace csvplus
