// pred.cuh — the recognisable predicates Like / All / Any / Not (csvplus.go:1243-1293) lowered to a
// tiny postfix program over "term" bits (term t = column term_col[t] equals literal t, or, for a set term, the row's
// tuple of the term's columns is one of its literal tuples: CPB_PRED_SET_MIN, csvplus_b200.h).
#pragma once
#include <algorithm>
#include <cstring>
#include <functional>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "core.hpp"

namespace cpb {

constexpr int MAXTERMS = CPB_PRED_MAX_TERMS;
constexpr int MAXOPS = CPB_PRED_MAX_OPS;
enum { OP_TERM = 0, OP_AND = 1, OP_OR = 2, OP_NOT = 3, OP_FALSE = 4, OP_TRUE = 5 };

struct PredProg {
    int32_t nops;
    int32_t nterms;
    uint8_t op[MAXOPS];
    uint8_t arg[MAXOPS];          // OP_TERM: term id
    uint32_t term_off[MAXTERMS];  // literal offset in the literal pool
    uint32_t term_len[MAXTERMS];
    int32_t term_col[MAXTERMS];   // column (table filter) or extracted slot (fused parse); -1 for a set term
};

// general case out of line (the parse kernel would inline the interpreter once per cached line)
static __device__ __noinline__ bool eval_pred_general(const PredProg& pr, uint32_t eq) {
    uint64_t st = 0;  // bit stack
    for (int i = 0; i < pr.nops; i++) {
        switch (pr.op[i]) {
            case OP_TERM: st = (st << 1) | ((eq >> pr.arg[i]) & 1); break;
            case OP_FALSE: st = st << 1; break;
            case OP_TRUE: st = (st << 1) | 1; break;
            case OP_NOT: st ^= 1; break;
            case OP_AND: { uint64_t a = st & 1; st >>= 1; st = (st & ~1ull) | (st & a & 1); } break;
            default: { uint64_t a = st & 1; st >>= 1; st |= a; } break;  // OP_OR
        }
    }
    return st & 1;
}
__device__ __forceinline__ bool eval_pred(const PredProg& pr, uint32_t eq) {
    if (pr.nops == 0) return true;
    if (pr.nops == 1 && pr.op[0] == OP_TERM) return (eq >> pr.arg[0]) & 1;
    return eval_pred_general(pr, eq);
}

// One set term: the literal tuples of its group as a table, one row per Like of the group, the columns in the group's key
// order (its first Like's).  Its term bit is whether the row's tuple is in IndexOn(keys) over that table.
struct SetTerm {
    int term = 0;
    std::vector<std::string> keys;
    std::vector<int> cols;                   // the keys' columns in the table the predicate was compiled against
    uint64_t rows = 0;
    std::vector<std::vector<uint32_t>> off;  // per key: offsets[rows + 1] into data (emptied once the index is built)
    std::vector<std::vector<uint8_t>> data;  // per key: the literals back to back
    std::shared_ptr<Index> index;            // built on first use (gather.cu)
};

struct Compiled {
    PredProg prog{};
    std::vector<uint8_t> lits;
    std::vector<SetTerm> sets;
    std::vector<std::string> columns;  // filter_parsed: the column names it was compiled against
};

// ------------------------------------------------------------------ the set-term rule (csvplus_b200.h, CPB_PRED_SET_MIN)
inline bool same_name(cpb_str a, cpb_str b) { return a.len == b.len && (a.len == 0 || memcmp(a.ptr, b.ptr, a.len) == 0); }
inline uint64_t name_hash(cpb_str s) {  // FNV-1a, then a final mix so that the sum over a key set spreads
    uint64_t h = 0xcbf29ce484222325ull;
    for (uint64_t i = 0; i < s.len; i++) h = (h ^ (uint8_t)s.ptr[i]) * 0x100000001b3ull;
    h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33;
    return h;
}
// pos[j] = the pair of Like `c` that compares key j of Like `f`; false when their key names differ as sets.  Both name each
// column once.  Likes that share one keys array (the host layers lower a group that way) are matched without a compare.
inline bool match_keys(const cpb_pred* f, const cpb_pred* c, uint8_t* pos) {
    if (c->n != f->n) return false;
    if (c->keys == f->keys) { for (int j = 0; j < f->n; j++) pos[j] = (uint8_t)j; return true; }
    for (int j = 0; j < f->n; j++) {
        int i = 0;
        while (i < c->n && !same_name(f->keys[j], c->keys[i])) i++;
        if (i == c->n) return false;
        pos[j] = (uint8_t)i;
    }
    return true;
}
inline bool distinct_names(const cpb_pred* c) {
    for (int i = 0; i < c->n; i++)
        for (int j = i + 1; j < c->n; j++) if (same_name(c->keys[i], c->keys[j])) return false;
    return true;
}

// The direct Like children of one Any node grouped by the set of column names they compare.  Linear in the children:
// a child joins the group of its hashed key set (consecutive children with one keys array are looked up once).
struct LikeGroups {
    struct Group {
        int first = 0;                // its first child
        uint64_t members = 0;
        std::vector<uint32_t> width;  // per key: the longest literal
        std::vector<uint64_t> bytes;  // per key: all literals
        bool set = false;             // it compiles to one set term
    };
    std::vector<int> of;  // per child: its group, -1 for none
    std::vector<Group> groups;
};
inline LikeGroups group_likes(const cpb_pred* any) {
    LikeGroups out;
    out.of.assign(any->n > 0 ? any->n : 0, -1);
    if (any->n < CPB_PRED_SET_MIN) return out;  // no group can reach the threshold
    std::unordered_map<uint64_t, std::vector<int>> by_hash;
    const cpb_str* last_keys = nullptr;
    int last_n = -1, last_g = -1;
    uint8_t pos[MAXKEYS];
    for (int i = 0; i < any->n; i++) {
        const cpb_pred* c = any->children[i];
        if (!c || c->op != CPB_PRED_LIKE || c->n <= 0 || c->n > MAXKEYS) continue;
        int g = -1;
        if (c->keys == last_keys && c->n == last_n) g = last_g;
        else {
            if (distinct_names(c)) {
                uint64_t h = 0;
                for (int k = 0; k < c->n; k++) h += name_hash(c->keys[k]);
                std::vector<int>& cand = by_hash[h];
                for (int x : cand) if (match_keys(any->children[out.groups[x].first], c, pos)) { g = x; break; }
                if (g < 0) {
                    g = (int)out.groups.size();
                    LikeGroups::Group ng; ng.first = i; ng.width.assign(c->n, 0); ng.bytes.assign(c->n, 0);
                    out.groups.push_back(std::move(ng));
                    cand.push_back(g);
                }
            }
            last_keys = c->keys; last_n = c->n; last_g = g;
        }
        if (g < 0) continue;
        LikeGroups::Group& gr = out.groups[g];
        out.of[i] = g;
        gr.members++;
        match_keys(any->children[gr.first], c, pos);
        for (int j = 0; j < c->n; j++) {
            const uint64_t len = c->values[pos[j]].len;
            gr.width[j] = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(gr.width[j], len), 0xffffffffull);
            gr.bytes[j] += len;
        }
    }
    for (auto& gr : out.groups) {
        uint64_t image = 0;  // the key image of IndexOn over the group's literals (sort.cu)
        for (uint32_t w : gr.width) image += (uint64_t)w + len_field_bytes(w);
        gr.set = gr.members >= CPB_PRED_SET_MIN && image <= MAX_KEY_IMAGE_BYTES;
    }
    return out;
}

// whether the tree compiles to a program with a set term, whatever the row type (a group's columns decide only whether its
// term is a constant false)
inline bool has_set_terms(const cpb_pred* p, int depth = 0) {
    if (!p || depth > CPB_PRED_MAX_DEPTH || p->op == CPB_PRED_LIKE) return false;
    if (p->op != CPB_PRED_ALL && p->op != CPB_PRED_ANY && p->op != CPB_PRED_NOT) return false;
    if (p->op == CPB_PRED_ANY)
        for (const auto& gr : group_likes(p).groups) if (gr.set) return true;
    for (int i = 0; i < p->n; i++) if (has_set_terms(p->children[i], depth + 1)) return true;
    return false;
}

// resolve(name) -> column/slot id or -1 when the row type lacks the column (Like => false, csvplus.go:1286)
inline void compile_pred(const cpb_pred* p, const std::function<int(const std::string&)>& resolve, Compiled& out, int depth = 0) {
    if (!p) return;
    auto push = [&](uint8_t op, uint8_t arg = 0) {
        if (out.prog.nops >= MAXOPS) throw ArgError{CPB_ERR_UNSUPPORTED, "predicate too large"};
        out.prog.op[out.prog.nops] = op; out.prog.arg[out.prog.nops] = arg; out.prog.nops++;
    };
    auto new_term = [&]() {
        if (out.prog.nterms >= MAXTERMS) throw ArgError{CPB_ERR_UNSUPPORTED, "too many Like terms"};
        return out.prog.nterms++;
    };
    // group g of Any node p as one set term (a constant false when the row type lacks one of its columns)
    auto set_term = [&](const LikeGroups& lg, int g) {
        const LikeGroups::Group& gr = lg.groups[g];
        const cpb_pred* f = p->children[gr.first];
        SetTerm st;
        for (int j = 0; j < f->n; j++) {
            st.keys.push_back(to_string(f->keys[j]));
            st.cols.push_back(resolve(st.keys.back()));
            if (st.cols.back() < 0) { push(OP_FALSE); return; }
        }
        const int t = new_term();
        out.prog.term_off[t] = 0; out.prog.term_len[t] = 0; out.prog.term_col[t] = -1;
        st.term = t;
        st.rows = gr.members;
        st.off.resize(f->n); st.data.resize(f->n);
        for (int j = 0; j < f->n; j++) {
            if (gr.bytes[j] > 0xffffffffull) throw ArgError{CPB_ERR_UNSUPPORTED, "the literals of one set term column exceed 4 GiB"};
            st.off[j].reserve(gr.members + 1); st.off[j].push_back(0);
            st.data[j].reserve(gr.bytes[j]);
        }
        uint8_t pos[MAXKEYS];
        for (int i = gr.first; i < p->n; i++) {
            if (lg.of[i] != g) continue;
            const cpb_pred* c = p->children[i];
            match_keys(f, c, pos);
            for (int j = 0; j < f->n; j++) {
                const cpb_str v = c->values[pos[j]];
                if (v.len) st.data[j].insert(st.data[j].end(), (const uint8_t*)v.ptr, (const uint8_t*)v.ptr + v.len);
                st.off[j].push_back((uint32_t)st.data[j].size());
            }
        }
        out.sets.push_back(std::move(st));
        push(OP_TERM, (uint8_t)t);
    };
    if (depth > CPB_PRED_MAX_DEPTH) throw ArgError{CPB_ERR_UNSUPPORTED, "predicate too deep"};
    switch (p->op) {
        case CPB_PRED_LIKE: {
            if (p->n <= 0) throw ArgError{CPB_ERR_ARG, "empty match row in Like() predicate"};  // csvplus.go:1280-1282
            for (int i = 0; i < p->n; i++) {
                int col = resolve(to_string(p->keys[i]));
                if (col < 0) push(OP_FALSE);
                else {
                    const int t = new_term();
                    out.prog.term_off[t] = (uint32_t)out.lits.size();
                    out.prog.term_len[t] = (uint32_t)p->values[i].len;
                    out.prog.term_col[t] = col;
                    const uint8_t* v = (const uint8_t*)p->values[i].ptr;
                    out.lits.insert(out.lits.end(), v, v + p->values[i].len);
                    push(OP_TERM, (uint8_t)t);
                }
                if (i > 0) push(OP_AND);
            }
        } break;
        case CPB_PRED_ALL:
            if (p->n == 0) { push(OP_TRUE); break; }
            for (int i = 0; i < p->n; i++) {
                compile_pred(p->children[i], resolve, out, depth + 1);
                if (i > 0) push(OP_AND);
            }
            break;
        case CPB_PRED_ANY: {
            if (p->n == 0) { push(OP_FALSE); break; }
            const LikeGroups lg = group_likes(p);
            int operands = 0;
            for (int i = 0; i < p->n; i++) {
                const int g = lg.of[i];
                if (g >= 0 && lg.groups[g].set) {
                    if (lg.groups[g].first != i) continue;  // the group is one operand, at its first child
                    set_term(lg, g);
                } else compile_pred(p->children[i], resolve, out, depth + 1);
                if (operands++ > 0) push(OP_OR);
            }
        } break;
        case CPB_PRED_NOT:
            if (p->n != 1) throw ArgError{CPB_ERR_ARG, "Not() takes one predicate"};
            compile_pred(p->children[0], resolve, out, depth + 1);
            push(OP_NOT);
            break;
        default: throw ArgError{CPB_ERR_ARG, "bad predicate op"};
    }
}

}  // namespace cpb
