// order.cu — OrderBy: a stable multi-key order of a table's rows by string, int and float64 keys, and its first `limit`
// rows by radix select (DESIGN §3.16).
//
// Order (that of Go's slices.SortStableFunc with cmp.Or of one cmp.Compare per key): each key is turned into whole
// 64-bit words of one order-preserving image, the keys' words concatenated in key order, so that comparing images as
// unsigned integers word by word is the comparator.
//   str:     sort.cu's key image of the one column (value zero-padded to the column's longest value, then its length):
//            strings.Compare, IndexOn's order
//   int:     Row.ValueAsInt as int64, u ^ 2^63
//   float64: Row.ValueAsFloat64 as cmp.Compare orders it: every NaN is 0 (below everything, all equal), -0 is +0's image,
//            a negative value ~u, any other value u | 2^63
//   desc:    the key's words complemented (cmp.Compare(b, a): NaNs last); a string key's zero padding stays constant
// Ties in every key keep row order: the radix sort is stable, and the select takes equal rows in row order.
//
// Routes for the first k of n rows: k * SELECT_RATIO <= n selects the k rows (select_by_image), sorts only those and
// gathers them; otherwise the whole image is sorted and the first k gathered.  With `before`, t's own first k rows are
// picked the same way and before ‖ those are ordered again: a row of t outside t's first k has k rows of t ahead of it.
#include <algorithm>

#include "core.hpp"
#include "util.cuh"

namespace cpb {

// select when limit * SELECT_RATIO <= rows: the crossover measured on an H100 (DESIGN §3.16).  (-D for an A/B build of
// tools/build_variant.sh.)
#ifndef ORDER_SELECT_RATIO
#define ORDER_SELECT_RATIO 2
#endif
constexpr uint64_t SELECT_RATIO = ORDER_SELECT_RATIO;
constexpr uint64_t SIGN = 0x8000000000000000ull;

static void check_keys(const std::vector<OrderKey>& keys) {
    if (keys.empty() || (int)keys.size() > MAXKEYS) throw ArgError{CPB_ERR_ARG, "OrderBy: 1 to " + std::to_string(MAXKEYS) + " keys"};
    for (size_t i = 0; i < keys.size(); i++) {
        if (keys[i].kind < CPB_ORDER_STR || keys[i].kind > CPB_ORDER_FLOAT64)
            throw ArgError{CPB_ERR_ARG, "OrderBy: unknown key kind " + std::to_string(keys[i].kind)};
        for (size_t j = i + 1; j < keys.size(); j++)
            if (keys[i].column == keys[j].column) throw ArgError{CPB_ERR_ARG, "OrderBy: duplicate key column " + go_quote(keys[i].column)};
    }
}

// the image of t's keys (word w of row r at [w * rows + r]); *words = its words per row.  Host synchronisations: one
// per numeric key (the conversion), one for the string keys' widths when there is a string key.
static Buf order_image(Ctx* c, const Table& t, const std::vector<OrderKey>& keys, uint32_t* words) {
    const uint64_t n = (uint64_t)t.nrows;
    std::vector<int> col(keys.size());
    std::vector<Buf> vals(keys.size());
    std::optional<DataError> bad;
    for (size_t k = 0; k < keys.size(); k++) {
        col[k] = t.find(keys[k].column);
        std::optional<DataError> e;
        if (col[k] < 0) {
            e = DataError{CPB_E_MISSING_COLUMN, -1, 0, false, "missing column " + go_quote(keys[k].column)};
        } else if (keys[k].kind != CPB_ORDER_STR) {
            const NumKind kind = keys[k].kind == CPB_ORDER_INT ? NumKind::Int64 : NumKind::Float64;
            vals[k] = dev_alloc(c, n * 8);
            const NumResult r = column_as_number(c, t, col[k], kind, vals[k]->p, nullptr);
            if (r.nbad) e = number_error(keys[k].column, kind, r);
        }
        if (e && (!bad || e->line < bad->line)) bad = e;
    }
    if (bad) throw *bad;
    std::vector<int> scols;
    for (size_t k = 0; k < keys.size(); k++) if (keys[k].kind == CPB_ORDER_STR) scols.push_back(col[k]);
    std::vector<uint32_t> width;
    if (!scols.empty()) {
        KernelTimer kt(c, "key_width", n * 4 * scols.size(), (int)scols.size());
        width = key_widths(c, t, scols, n);
    }
    std::vector<uint32_t> kw(keys.size());
    uint64_t total = 0;
    for (size_t k = 0, s = 0; k < keys.size(); k++) {
        kw[k] = keys[k].kind == CPB_ORDER_STR ? (width[s] + len_field_bytes(width[s]) + 7) / 8 : 1;
        s += keys[k].kind == CPB_ORDER_STR;
        total += kw[k];
    }
    if (total * 8 > MAX_KEY_IMAGE_BYTES) throw ArgError{CPB_ERR_UNSUPPORTED, "order keys longer than 4 KiB are not supported"};
    *words = (uint32_t)total;
    Buf img = dev_alloc(c, std::max<uint64_t>(1, total * n) * 8);
    KernelTimer kt(c, "order_image", n * 16 * keys.size(), (int)keys.size());
    uint64_t w0 = 0;
    for (size_t k = 0, s = 0; k < keys.size(); k++) {
        uint64_t* dst = img->as<uint64_t>() + w0 * n;
        if (keys[k].kind == CPB_ORDER_STR) {
            pack_into(c, t, {col[k]}, {width[s++]}, dst);
        } else {
            const uint64_t* v = vals[k]->as<uint64_t>();
            if (keys[k].kind == CPB_ORDER_INT)
                each_row(c, n, [=] __device__(uint64_t i) { dst[i] = v[i] ^ SIGN; });
            else
                each_row(c, n, [=] __device__(uint64_t i) {
                    const uint64_t u = v[i];
                    const bool nan = (u & 0x7FF0000000000000ull) == 0x7FF0000000000000ull && (u & 0x000FFFFFFFFFFFFFull) != 0;
                    dst[i] = nan ? 0 : u == SIGN ? SIGN : (u & SIGN) ? ~u : (u | SIGN);
                });
            vals[k].reset();
        }
        if (keys[k].descending) each_row(c, kw[k] * n, [=] __device__(uint64_t i) { dst[i] = ~dst[i]; });
        w0 += kw[k];
    }
    return img;
}

// the first k rows (0 < k <= n) of t in image order: row ids of t, uint32[k].  sorted = false: any order will do (the
// select route then leaves them in row order).  Host synchronisations: select 2 (1 unsorted), full sort 1.
static Buf first_rows(Ctx* c, const uint64_t* img, uint32_t words, uint64_t n, uint64_t k, bool sorted) {
    uint64_t traffic = 0;
    if (k * SELECT_RATIO > n) return sort_by_image(c, img, words, n, &traffic);
    Buf ids = select_by_image(c, img, words, n, k, &traffic);
    if (!sorted) return ids;
    Buf simg;
    {
        KernelTimer kt(c, "image_gather", (uint64_t)words * k * 20, (int)words);
        simg = gather_image(c, img, words, n, ids->as<uint32_t>(), k);
    }
    Buf perm = sort_by_image(c, simg->as<uint64_t>(), words, k, &traffic);
    uint32_t* p = perm->as<uint32_t>();
    const uint32_t* id = ids->as<uint32_t>();
    each_row(c, k, [=] __device__(uint64_t i) { p[i] = id[p[i]]; });
    return perm;
}

static std::shared_ptr<Table> no_rows(Ctx* c, const Table& t) {
    auto r = table_view(c, t, 0, 0);
    r->first_line = 0;
    return r;
}

std::shared_ptr<Table> order_table(Ctx* c, const Table& t, const std::vector<OrderKey>& keys, uint64_t limit, const Table* before) {
    check_keys(keys);
    const uint64_t n = (uint64_t)t.nrows;
    if (n > 0xFFFFFFFFull) throw DataError{CPB_E_TOO_LARGE, -1, 0, false, "OrderBy: a table of 2^32 rows or more: order row-range slices"};
    if (before) {
        if (before->cols.size() != t.cols.size()) throw ArgError{CPB_ERR_ARG, "OrderBy: the rows before have other columns"};
        for (size_t i = 0; i < t.cols.size(); i++)
            if (before->cols[i].name != t.cols[i].name) throw ArgError{CPB_ERR_ARG, "OrderBy: the rows before have other columns"};
    }
    if (n == 0) return before ? order_table(c, *before, keys, limit, nullptr) : no_rows(c, t);
    uint32_t words = 0;
    Buf img = order_image(c, t, keys, &words);
    const uint64_t k = std::min(limit, n);
    if (before) {
        std::shared_ptr<Table> mine;
        if (k == 0) {
            mine = no_rows(c, t);
        } else if (k < n) {
            Buf ids = first_rows(c, img->as<uint64_t>(), words, n, k, false);
            img.reset();
            mine = gather_rows(c, t, ids->as<uint32_t>(), (int64_t)k);
        }
        auto both = concat_tables(c, {before, mine ? mine.get() : &t});
        return order_table(c, *both, keys, limit, nullptr);
    }
    if (k == 0) return no_rows(c, t);
    Buf ids = first_rows(c, img->as<uint64_t>(), words, n, k, true);
    img.reset();
    auto r = gather_rows(c, t, ids->as<uint32_t>(), (int64_t)k);
    r->first_line = 0;
    return r;
}

}  // namespace cpb
