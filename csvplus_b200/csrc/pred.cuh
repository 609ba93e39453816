// pred.cuh — the recognisable predicates Like / All / Any / Not (csvplus.go:1243-1293) lowered to a
// tiny postfix program over "term" bits (term t = column term_col[t] equals literal t).
#pragma once
#include <functional>
#include <string>
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
    int32_t term_col[MAXTERMS];   // column (table filter) or extracted slot (fused parse)
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

struct Compiled {
    PredProg prog{};
    std::vector<uint8_t> lits;
};

// resolve(name) -> column/slot id or -1 when the row type lacks the column (Like => false, csvplus.go:1286)
inline void compile_pred(const cpb_pred* p, const std::function<int(const std::string&)>& resolve, Compiled& out, int depth = 0) {
    if (!p) return;
    auto push = [&](uint8_t op, uint8_t arg = 0) {
        if (out.prog.nops >= MAXOPS) throw ArgError{CPB_ERR_UNSUPPORTED, "predicate too large"};
        out.prog.op[out.prog.nops] = op; out.prog.arg[out.prog.nops] = arg; out.prog.nops++;
    };
    if (depth > CPB_PRED_MAX_DEPTH) throw ArgError{CPB_ERR_UNSUPPORTED, "predicate too deep"};
    switch (p->op) {
        case CPB_PRED_LIKE: {
            if (p->n <= 0) throw ArgError{CPB_ERR_ARG, "empty match row in Like() predicate"};  // csvplus.go:1280-1282
            for (int i = 0; i < p->n; i++) {
                int col = resolve(to_string(p->keys[i]));
                if (col < 0) push(OP_FALSE);
                else {
                    if (out.prog.nterms >= MAXTERMS) throw ArgError{CPB_ERR_UNSUPPORTED, "too many Like terms"};
                    int t = out.prog.nterms++;
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
        case CPB_PRED_ANY: {
            if (p->n == 0) { push(p->op == CPB_PRED_ALL ? OP_TRUE : OP_FALSE); break; }
            for (int i = 0; i < p->n; i++) {
                compile_pred(p->children[i], resolve, out, depth + 1);
                if (i > 0) push(p->op == CPB_PRED_ALL ? OP_AND : OP_OR);
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
