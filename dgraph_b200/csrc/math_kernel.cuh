// math_kernel.cuh -- math() over value variables (query/math.go evalMathTree, transformVars' leaf rule and
// valueVarAggregation's math branch, query/query.go :1239-1361) in one call.
//
// Real uids are never 0, so every node of a program is one of two kinds.  A scalar node depends only on constants,
// empty or nil maps and {0: v} aggregates: its key set is a subset of {0}, and one thread evaluates it exactly.  A
// vector node has its keys in U, the union of the general leaves' keys (which exclude 0), and is evaluated by a thread
// per key of U.  A vector binary node sees each scalar child as a broadcast constant or as a missing entry.
//   mt_check_kernel   thread per leaf entry and range uid: count words within their room, keys and range strictly
//                     ascending, entry tags known
//   mt_plan_kernel    one thread: classifies the leaves (nil, empty, {MaxUint64: v} constant, {0: v} aggregate,
//                     general; key 0 among other keys is refused), evaluates every scalar node with Go's rules
//                     (checkAggrResult left first) and records, for each vector node, where each child's value comes
//                     from; the general leaves' row offsets for the key union
//   mt_gather_kernel  thread per leaf entry: the general leaves' keys as the rows of one matrix
//   merge_matrix_impl the existing matrix merge: the rows' union U, ascending and de-duplicated
//   mt_eval_kernel    thread per key of U: the vector nodes in post-order, each a presence, a tag and a word kept in
//                     thread-local arrays; per-node present and error counts, the root's tag set
//   scan_u64_kernel   the root's present keys -> output positions
//   mt_finish_kernel  one thread: the order-dependent refusals from the counts, the result's kind, length and tags
//   mt_write_kernel   thread per key: the root's entries (ints promoted to float when both are present), or the
//                     constant over the range
// 7 launches plus the merge's, whatever the tree and map sizes.  Float arithmetic uses the _rn intrinsics: nothing
// contracts to FMA, so every result is the IEEE one Go computes.
#pragma once

#include "merge_matrix.cuh"

namespace dgx {

using u8 = uint8_t;

constexpr int kLaneErrMath = 512;  // lane error flag bit: a math() input is malformed or Go's answer is an error
constexpr int MT_MAX_NODES = 64, MT_MAX_LEAVES = 16;
// entry tags (DGX_VAL_*); 0 is a missing entry
constexpr u8 MT_ABS = 0, MT_INT = 1, MT_FLT = 2, MT_BOOL = 3, MT_NIL = 4;
// ops (DGX_MATH_*)
constexpr int MO_CONST = 0, MO_VAR = 1, MO_ADD = 2, MO_SUB = 3, MO_MUL = 4, MO_DIV = 5, MO_MOD = 6, MO_MIN = 7,
              MO_MAX = 8, MO_NEG = 9, MO_SQRT = 10, MO_FLOOR = 11, MO_CEIL = 12, MO_LT = 13, MO_GT = 14, MO_LE = 15,
              MO_GE = 16, MO_EQ = 17, MO_NE = 18, MO_COND = 19;
// a node's kind after the plan: a constant, no map (Go's nil), an empty map, {0: v}, or keys in U
constexpr u8 MK_CONST = 0, MK_NIL = 1, MK_EMPTY = 2, MK_MAP0 = 3, MK_VEC = 4;
// where a vector node reads a child: its per-key result, a broadcast constant, or a missing entry at every key of U
constexpr u8 MS_VEC = 0, MS_CONST = 1, MS_NONE = 2;
// words: the result's kind, whether ints are promoted, the capacity overflow
constexpr int MT_W_KIND = 0, MT_W_PROMOTE = 1, MT_W_OVER = 2, MT_W_TAGS = 3, MT_WORDS = 4;

__host__ __device__ constexpr bool mt_binary(int op) { return op >= MO_ADD && op <= MO_MAX; }
__host__ __device__ constexpr bool mt_unary(int op) { return op >= MO_NEG && op <= MO_CEIL; }
__host__ __device__ constexpr bool mt_compare(int op) { return op >= MO_LT && op <= MO_NE; }
__host__ __device__ constexpr int mt_arity(int op) {
    return op == MO_COND ? 3 : mt_binary(op) || mt_compare(op) ? 2 : mt_unary(op) ? 1 : 0;
}

// dgx_math_node (include/dgx.h)
struct MtProg {
    u8 op, ctag;
    uint16_t child[3];
    u32 leaf;
    u64 cword;
};

// A leaf with device pointers: entries n (room), *d_len (count) when d_len is set.
struct MtLeaf {
    const u64* key;
    const u64* word;
    const u8* tag;
    const u64* d_len;
    u64 n;
    int type, nil;
};

// The plan of one node: its kind and (scalar) value; for a vector node each child's source and constant.
struct MtPlan {
    u8 kind, tag, op, nilc_n;
    u8 src[3];
    u8 ctag[3];
    u8 nilc[2];  // COND over a vector binary node: that node's vector children (nil when all are empty)
    uint16_t child[3];
    u32 leaf;
    u64 word;
    u64 cword[3];
};

struct MtParams {
    const MtProg* prog;   // nn
    u32 nn, nl;
    const MtLeaf* leaf;   // nl
    const u64* cap_off;   // nl + 1: prefix of the leaves' rooms (the thread space of check and gather)
    u64 cap_total;
    const u64* range;     // nrange, or null: no range
    u64 nrange;
    MtPlan* plan;         // nn
    u64* llen;            // nl: entry counts
    u64* row_off;         // nl + 1: the general leaves' rows in cat
    u64* cat;             // cap_total
    const u64* U;         // the key union and its length word
    const u64* ulen;
    u32* cnt;             // nn present keys, zeroed
    u32* nerr;            // nn failed keys, zeroed
    u8* rtag;             // per key of U: the root's entry
    u64* rword;
    u64* flag;            // per key of U: the root is present
    u64* pos;             // cap + 1
    u64* words;           // MT_WORDS, zeroed
    int* bad;             // zeroed
    int* err;
    u64* out_key;
    u64* out_word;
    u8* out_tag;
    u64 out_cap;
    u64* info;
};

__device__ __forceinline__ void mt_refuse(const MtParams& P) {
    atomicOr(P.bad, 1);
    atomicOr(P.err, kLaneErrMath);
}

__device__ __forceinline__ double mt_d(u64 x) { return __longlong_as_double((long long)x); }
__device__ __forceinline__ u64 mt_u(double x) { return (u64)__double_as_longlong(x); }

// aggregator.Value: +Inf -> MaxFloat64, -Inf -> -MaxFloat64, NaN -> +0.0.
__device__ __forceinline__ u64 mt_clamp(u64 w) {
    const double x = mt_d(w);
    if (x != x) return 0;
    if (w == 0x7ff0000000000000ull) return 0x7fefffffffffffffull;
    if (w == 0xfff0000000000000ull) return 0xffefffffffffffffull;
    return w;
}

// Go's int64 / and %: MinInt64 / -1 wraps to MinInt64, MinInt64 % -1 is 0 (both undefined in C).
__device__ __forceinline__ long long mt_idiv(long long a, long long b) { return b == -1 ? (long long)(0ull - (u64)a) : a / b; }
__device__ __forceinline__ long long mt_imod(long long a, long long b) { return b == -1 ? 0 : a % b; }

// processBinary's f for one key: ApplyVal(l), ApplyVal(r) (a missing or nil value is int64 0), matchType, apply*,
// Value().  Returns false where Go's f errs (the key is dropped).
__device__ bool mt_bin(int op, u8 ta, u64 a, u8 tb, u64 b, u8* tr, u64* r) {
    if (ta == MT_ABS || ta == MT_NIL) { ta = MT_INT; a = 0; }
    if (tb == MT_ABS || tb == MT_NIL) { tb = MT_INT; b = 0; }
    if (ta != tb) {  // matchType: bool is DEFAULT and meets nothing else; an int meeting a float becomes one
        if (ta == MT_BOOL || tb == MT_BOOL) return false;
        if (ta == MT_INT) { a = mt_u(__ll2double_rn((long long)a)); ta = MT_FLT; }
        else { b = mt_u(__ll2double_rn((long long)b)); tb = MT_FLT; }
    }
    if (ta == MT_BOOL) return false;  // every apply* (and types.Less) refuses DEFAULT operands
    *tr = ta;
    if (ta == MT_INT) {
        const long long x = (long long)a, y = (long long)b;
        switch (op) {
            case MO_ADD:
                if ((x > 0 && y > LLONG_MAX - x) || (x < 0 && y < LLONG_MIN - x)) return false;
                *r = a + b;
                return true;
            case MO_SUB:
                if ((y < 0 && x > LLONG_MAX + y) || (y > 0 && x < LLONG_MIN + y)) return false;
                *r = a - b;
                return true;
            case MO_MUL: {
                const long long c = (long long)(a * b);  // wraps; Go detects overflow by c / y != x
                if (x != 0 && y != 0 && mt_idiv(c, y) != x) return false;
                *r = (u64)c;
                return true;
            }
            case MO_DIV:
                if (y == 0) return false;
                *r = (u64)mt_idiv(x, y);
                return true;
            case MO_MOD:
                if (y == 0) return false;
                *r = (u64)mt_imod(x, y);
                return true;
            case MO_MIN: *r = x < y ? a : b; return true;
            default: *r = x < y ? b : a; return true;  // MO_MAX
        }
    }
    const double x = mt_d(a), y = mt_d(b);
    double z;
    switch (op) {
        case MO_ADD: z = __dadd_rn(x, y); break;
        case MO_SUB: z = __dsub_rn(x, y); break;
        case MO_MUL: z = __dmul_rn(x, y); break;
        case MO_DIV:
            if (y == 0) return false;
            z = __ddiv_rn(x, y);
            break;
        case MO_MOD:
            if (y == 0) return false;
            z = fmod(x, y);  // exact, as math.Mod: NaN for an infinite x or a NaN operand, x for an infinite y
            break;
        case MO_MIN: *r = mt_clamp(x < y ? a : b); return true;
        default: *r = mt_clamp(x < y ? b : a); return true;  // MO_MAX
    }
    *r = mt_clamp(mt_u(z));
    return true;
}

// processUnary for one value (a missing or nil value is int64 0); false where apply* errs.
__device__ bool mt_un(int op, u8 ta, u64 a, u8* tr, u64* r) {
    if (ta == MT_ABS || ta == MT_NIL) { ta = MT_INT; a = 0; }
    if (ta == MT_BOOL) return false;
    if (ta == MT_INT) {
        const long long x = (long long)a;
        switch (op) {
            case MO_NEG:
                if (x == LLONG_MIN) return false;
                *tr = MT_INT;
                *r = 0ull - a;
                return true;
            case MO_SQRT:
                if (x < 0) return false;
                *tr = MT_FLT;
                *r = mt_clamp(mt_u(__dsqrt_rn(__ll2double_rn(x))));
                return true;
            default:  // floor, ceil of an int: the int
                *tr = MT_INT;
                *r = a;
                return true;
        }
    }
    const double x = mt_d(a);
    *tr = MT_FLT;
    switch (op) {
        case MO_NEG: *r = mt_clamp(a ^ 0x8000000000000000ull); return true;
        case MO_SQRT:
            if (x < 0) return false;
            *r = mt_clamp(mt_u(__dsqrt_rn(x)));
            return true;
        case MO_FLOOR: *r = mt_clamp(mt_u(floor(x))); return true;
        default: *r = mt_clamp(mt_u(ceil(x))); return true;  // MO_CEIL
    }
}

// compareValues(op, a, b): b missing is Val{} (nil).  Numbers compare as floats when their types differ; nil against
// nil is neither ordered nor equal; every other pair errs (false).
__device__ bool mt_cmp(int op, u8 ta, u64 a, u8 tb, u64 b, u64* r) {
    if (tb == MT_ABS) tb = MT_NIL;
    bool lt, gt, eq;
    if (ta == MT_NIL && tb == MT_NIL) {
        lt = gt = eq = false;
    } else if ((ta == MT_INT || ta == MT_FLT) && (tb == MT_INT || tb == MT_FLT)) {
        if (ta == MT_INT && tb == MT_INT) {
            lt = (long long)a < (long long)b;
            gt = (long long)b < (long long)a;
            eq = a == b;
        } else {
            const double x = ta == MT_INT ? __ll2double_rn((long long)a) : mt_d(a);
            const double y = tb == MT_INT ? __ll2double_rn((long long)b) : mt_d(b);
            lt = x < y;
            gt = y < x;
            eq = x == y;
        }
    } else {
        return false;
    }
    bool v;
    switch (op) {
        case MO_LT: v = lt; break;
        case MO_GT: v = gt; break;
        case MO_LE: v = lt || eq; break;
        case MO_GE: v = gt || eq; break;
        case MO_EQ: v = eq; break;
        default: v = !eq; break;  // MO_NE
    }
    *r = v;
    return true;
}

// The count word's low 32 bits: a dgx_var_propagate length, or the info word of a previous math() call.
__device__ __forceinline__ u64 mt_len(const MtLeaf& L) { return L.d_len ? (*L.d_len & 0xffffffffull) : L.n; }
__device__ __forceinline__ u8 mt_etag(const MtLeaf& L, u64 i) { return L.tag ? L.tag[i] : (u8)L.type; }

// Grid over cap_total + nrange threads.
__global__ void __launch_bounds__(256) mt_check_kernel(const MtParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    if (t < P.cap_total) {
        u32 j = 0;
        while (P.cap_off[j + 1] <= t) ++j;
        const MtLeaf& L = P.leaf[j];
        const u64 i = t - P.cap_off[j], n = mt_len(L);
        if (i < n && i < L.n) {
            if (i > 0 && L.key[i - 1] >= L.key[i]) bad = true;
            const u8 g = mt_etag(L, i);
            if (g < MT_INT || g > MT_NIL) bad = true;
        }
    } else if (P.range && t - P.cap_total < P.nrange) {
        const u64 i = t - P.cap_total;
        if (i > 0 && P.range[i - 1] >= P.range[i]) bad = true;
    }
    if (bad) mt_refuse(P);
}

// One thread.  The scalar rules of processBinary / processUnary / processBinaryBoolean / processTernary over values
// whose key set is a subset of {0}; Go's errors refuse the call.
__global__ void __launch_bounds__(32) mt_plan_kernel(const MtParams P) {
    if (threadIdx.x != 0) return;
    u64 off = 0;
    bool bad = *P.bad != 0;
    u8 lk[MT_MAX_LEAVES], lt[MT_MAX_LEAVES];
    u64 lw[MT_MAX_LEAVES];
    for (u32 j = 0; j < P.nl; ++j) {
        const MtLeaf& L = P.leaf[j];
        u64 n = bad ? 0 : mt_len(L);
        if (n > L.n) {  // a count word past the leaf's room
            bad = true;
            n = 0;
        }
        P.llen[j] = n;
        P.row_off[j] = off;
        lt[j] = MT_ABS;
        lw[j] = 0;
        if (L.nil) {
            lk[j] = MK_NIL;
        } else if (n == 0) {
            lk[j] = MK_EMPTY;
        } else if (n == 1 && (L.key[0] == ~0ull || L.key[0] == 0)) {
            lt[j] = mt_etag(L, 0);
            lw[j] = L.word[0];
            // transformVars: {MaxUint64: v} is the constant v (a nil v sets no constant and no map)
            lk[j] = L.key[0] == 0 ? MK_MAP0 : lt[j] == MT_NIL ? MK_NIL : MK_CONST;
        } else if (L.key[0] == 0) {
            bad = true;  // key 0 among other keys: neither an aggregate nor a map over uids
            lk[j] = MK_EMPTY;
        } else {
            lk[j] = MK_VEC;
            off += n;
        }
    }
    P.row_off[P.nl] = off;
    for (u32 i = 0; i < P.nn && !bad; ++i) {
        const MtProg& g = P.prog[i];
        MtPlan& N = P.plan[i];
        N.op = g.op;
        N.leaf = g.leaf;
        N.nilc_n = 0;
        N.tag = MT_ABS;
        N.word = 0;
        for (int c = 0; c < 3; ++c) {
            N.child[c] = g.child[c];
            N.src[c] = MS_NONE;
            N.ctag[c] = MT_ABS;
            N.cword[c] = 0;
        }
        const int op = g.op;
        if (op == MO_CONST) {
            N.kind = MK_CONST;
            N.tag = g.ctag;
            N.word = g.cword;
            continue;
        }
        if (op == MO_VAR) {
            N.kind = lk[g.leaf];
            N.tag = lt[g.leaf];
            N.word = lw[g.leaf];
            continue;
        }
        const MtPlan& A = P.plan[g.child[0]];
        if (mt_binary(op)) {
            const MtPlan& B = P.plan[g.child[1]];
            // checkAggrResult: the left {0: v} becomes a constant, else the right one
            const bool lconv = A.kind == MK_MAP0, rconv = !lconv && B.kind == MK_MAP0;
            const bool lc = A.kind == MK_CONST || (lconv && A.tag != MT_NIL);
            const bool rc = B.kind == MK_CONST || (rconv && B.tag != MT_NIL);
            if (A.kind == MK_VEC || B.kind == MK_VEC) {
                N.kind = MK_VEC;
                N.src[0] = A.kind == MK_VEC ? MS_VEC : lc ? MS_CONST : MS_NONE;
                N.src[1] = B.kind == MK_VEC ? MS_VEC : rc ? MS_CONST : MS_NONE;
                N.ctag[0] = A.tag;
                N.cword[0] = A.word;
                N.ctag[1] = B.tag;
                N.cword[1] = B.word;
            } else if (B.kind == MK_MAP0 && !rconv) {  // the right {0: v} stays a map: key 0 alone
                u8 t;
                u64 w;
                if (mt_bin(op, lc ? A.tag : MT_ABS, lc ? A.word : 0, B.tag, B.word, &t, &w)) {
                    N.kind = MK_MAP0;
                    N.tag = t;
                    N.word = w;
                } else {
                    N.kind = MK_EMPTY;
                }
            } else if (lc && rc) {
                u8 t;
                u64 w;
                if (!mt_bin(op, A.tag, A.word, B.tag, B.word, &t, &w)) bad = true;  // returned by evalMathTree
                N.kind = MK_CONST;
                N.tag = t;
                N.word = w;
            } else {
                N.kind = MK_NIL;
            }
        } else if (mt_unary(op)) {
            u8 t;
            u64 w;
            if (A.kind == MK_VEC) {
                N.kind = MK_VEC;
                N.src[0] = MS_VEC;
            } else if (A.kind == MK_CONST) {
                if (!mt_un(op, A.tag, A.word, &t, &w)) bad = true;
                N.kind = MK_CONST;
                N.tag = t;
                N.word = w;
            } else if (A.kind == MK_MAP0 && mt_un(op, A.tag, A.word, &t, &w)) {
                N.kind = MK_MAP0;
                N.tag = t;
                N.word = w;
            } else {
                N.kind = MK_EMPTY;  // a new map: empty, or its only key failed
            }
        } else if (mt_compare(op)) {
            const MtPlan& B = P.plan[g.child[1]];
            const u8 rs = B.kind == MK_VEC ? MS_VEC : B.kind == MK_CONST ? MS_CONST : MS_NONE;
            u64 w;
            if (A.kind == MK_VEC) {
                N.kind = MK_VEC;
                N.src[0] = MS_VEC;
                N.src[1] = rs;
                N.ctag[1] = B.tag;
                N.cword[1] = B.word;
            } else if (A.kind == MK_MAP0 &&
                       mt_cmp(op, A.tag, A.word, B.kind == MK_CONST || B.kind == MK_MAP0 ? B.tag : MT_ABS, B.word, &w)) {
                N.kind = MK_MAP0;
                N.tag = MT_BOOL;
                N.word = w;
            } else {
                N.kind = MK_EMPTY;
            }
        } else {  // MO_COND
            const MtPlan& B = P.plan[g.child[1]];
            const MtPlan& C = P.plan[g.child[2]];
            if (A.kind == MK_CONST || A.kind == MK_NIL) {
                bad = true;  // "Expected a value variable in cond but missing."
            } else if (A.kind == MK_VEC) {
                N.kind = MK_VEC;
                N.src[0] = MS_VEC;
                N.src[1] = B.kind == MK_VEC ? MS_VEC : B.kind == MK_CONST ? MS_CONST : MS_NONE;
                N.src[2] = C.kind == MK_VEC ? MS_VEC : C.kind == MK_CONST ? MS_CONST : MS_NONE;
                N.ctag[1] = B.tag;
                N.cword[1] = B.word;
                N.ctag[2] = C.tag;
                N.cword[2] = C.word;
                if (mt_binary(A.op))  // nil when every vector child of it comes out empty
                    for (int c = 0; c < 2; ++c)
                        if (A.src[c] == MS_VEC) N.nilc[N.nilc_n++] = (u8)A.child[c];
            } else if (A.kind == MK_MAP0 && A.tag == MT_BOOL) {
                const MtPlan& X = A.word ? B : C;
                N.kind = MK_MAP0;
                N.tag = X.kind == MK_CONST || X.kind == MK_MAP0 ? X.tag : MT_NIL;
                N.word = X.kind == MK_CONST || X.kind == MK_MAP0 ? X.word : 0;
            } else {
                N.kind = MK_EMPTY;  // empty, or its only value is not a bool
            }
        }
    }
    if (bad) {
        for (u32 j = 0; j <= P.nl; ++j) P.row_off[j] = 0;  // nothing reaches the merge
        mt_refuse(P);
    }
}

// Grid over cap_total threads: the general leaves' keys as rows.
__global__ void __launch_bounds__(256) mt_gather_kernel(const MtParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.cap_total || *P.bad) return;
    u32 j = 0;
    while (P.cap_off[j + 1] <= t) ++j;
    const u64 i = t - P.cap_off[j], a = P.row_off[j];
    if (i < P.row_off[j + 1] - a) P.cat[a + i] = P.leaf[j].key[i];
}

// Thread per key of U (grid over cap_total): every vector node in post-order.  Children's results are read from the
// thread-local tag / word arrays, broadcast constants from the plan.
__global__ void __launch_bounds__(256) mt_eval_kernel(const MtParams P) {
    __shared__ MtPlan sp[MT_MAX_NODES];
    __shared__ MtLeaf sl[MT_MAX_LEAVES];
    __shared__ u64 sn[MT_MAX_LEAVES];
    __shared__ u32 s_cnt[MT_MAX_NODES], s_err[MT_MAX_NODES], s_tags;
    const u32 nn = P.nn;
    for (u32 i = threadIdx.x; i < nn; i += blockDim.x) {
        sp[i] = P.plan[i];
        s_cnt[i] = s_err[i] = 0;
    }
    for (u32 j = threadIdx.x; j < P.nl; j += blockDim.x) {
        sl[j] = P.leaf[j];
        sn[j] = P.llen[j];
    }
    if (threadIdx.x == 0) s_tags = 0;
    __syncthreads();
    if (*P.bad) return;
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const bool on = t < *P.ulen;
    const u64 u = on ? P.U[t] : 0;
    const int lane = threadIdx.x & 31;
    u8 tg[MT_MAX_NODES];
    u64 wd[MT_MAX_NODES];
    for (u32 i = 0; i < nn; ++i) {
        const MtPlan& N = sp[i];
        if (N.kind != MK_VEC) continue;
        u8 rt = MT_ABS;
        u64 rw = 0;
        bool fail = false;
        if (on) {
            u8 ct[3];
            u64 cw[3];
            const int ar = mt_arity(N.op);
            for (int c = 0; c < ar; ++c) {
                const u8 s = N.src[c];
                ct[c] = s == MS_VEC ? tg[N.child[c]] : s == MS_CONST ? N.ctag[c] : MT_ABS;
                cw[c] = s == MS_VEC ? wd[N.child[c]] : s == MS_CONST ? N.cword[c] : 0;
            }
            if (N.op == MO_VAR) {
                const MtLeaf& L = sl[N.leaf];
                const u64 n = sn[N.leaf], j = lower_bound_g(L.key, n, u);
                if (j < n && L.key[j] == u) {
                    rt = mt_etag(L, j);
                    rw = L.word[j];
                }
            } else if (mt_binary(N.op)) {
                // the union of the maps' keys: present when a vector child holds the key
                const bool any = (N.src[0] == MS_VEC && ct[0] != MT_ABS) || (N.src[1] == MS_VEC && ct[1] != MT_ABS);
                if (any && !mt_bin(N.op, ct[0], cw[0], ct[1], cw[1], &rt, &rw)) rt = MT_ABS;
                if (!any) rt = MT_ABS;
            } else if (ct[0] != MT_ABS) {  // unary, comparison and cond range over the first child's keys
                if (mt_unary(N.op)) {
                    fail = !mt_un(N.op, ct[0], cw[0], &rt, &rw);
                } else if (mt_compare(N.op)) {
                    fail = !mt_cmp(N.op, ct[0], cw[0], ct[1], cw[1], &rw);
                    rt = MT_BOOL;
                } else if (ct[0] != MT_BOOL) {
                    fail = true;
                } else {
                    const int c = cw[0] ? 1 : 2;
                    rt = ct[c] == MT_ABS ? MT_NIL : ct[c];  // a missing branch entry is stored as Val{}
                    rw = ct[c] == MT_ABS ? 0 : cw[c];
                }
                if (fail) rt = MT_ABS;
            }
        }
        tg[i] = rt;
        wd[i] = rw;
        const u32 pc = __popc(__ballot_sync(0xffffffffu, rt != MT_ABS));
        const u32 ec = __popc(__ballot_sync(0xffffffffu, fail));
        if (lane == 0) {
            if (pc) atomicAdd(&s_cnt[i], pc);
            if (ec) atomicAdd(&s_err[i], ec);
        }
    }
    const u8 r = tg[nn - 1];
    if (on && sp[nn - 1].kind == MK_VEC) {  // a scalar root is the plan's; its tg entry is never written
        P.flag[t] = r != MT_ABS;
        P.rtag[t] = r;
        P.rword[t] = wd[nn - 1];
        if (r != MT_ABS) atomicOr(&s_tags, 1u << r);
    }
    __syncthreads();
    for (u32 i = threadIdx.x; i < nn; i += blockDim.x) {
        if (s_cnt[i]) atomicAdd(P.cnt + i, s_cnt[i]);
        if (s_err[i]) atomicAdd(P.nerr + i, s_err[i]);
    }
    if (threadIdx.x == 0 && s_tags) atomicOr((unsigned long long*)(P.words + MT_W_TAGS), (unsigned long long)s_tags);
}

// One thread: refusals where Go's answer depends on map order (a unary, comparison or cond node failing on some but not
// all of more than one key; cond over a binary node all of whose maps came out empty, a nil map), then the result's
// kind, length and tags into *info.  A result longer than out_cap sets only *info (DGX_ERR_CAP).
__global__ void __launch_bounds__(32) mt_finish_kernel(const MtParams P) {
    if (threadIdx.x != 0 || *P.bad) return;
    const u32 nn = P.nn;
    for (u32 i = 0; i < nn; ++i) {
        const MtPlan& N = P.plan[i];
        if (N.kind != MK_VEC || N.op == MO_VAR || mt_binary(N.op)) continue;
        const u32 keys = P.cnt[N.child[0]], e = P.nerr[i];
        bool refuse = e > 0 && e < keys;
        if (N.op == MO_COND && N.nilc_n) {
            bool all_empty = true;
            for (int c = 0; c < N.nilc_n; ++c) all_empty = all_empty && P.cnt[N.nilc[c]] == 0;
            refuse = refuse || all_empty;
        }
        if (refuse) {
            mt_refuse(P);
            return;
        }
    }
    const MtPlan& R = P.plan[nn - 1];
    u64 kind = 0, len = 0, tags = 0;
    if (R.kind == MK_CONST) {
        kind = 2;
        len = P.range ? P.nrange : 1;
        tags = 1u << R.tag;
    } else if (R.kind == MK_MAP0) {
        kind = 1;
        len = 1;
        tags = 1u << R.tag;
    } else if (R.kind == MK_VEC && P.cnt[nn - 1]) {
        kind = 1;
        len = P.cnt[nn - 1];
        tags = P.words[MT_W_TAGS];
        if ((tags & (1u << MT_INT)) && (tags & (1u << MT_FLT))) {  // Go converts every int to float
            P.words[MT_W_PROMOTE] = 1;
            tags &= ~(u64)(1u << MT_INT);
        }
    }
    if (len == 0) tags = 0;  // a constant over an empty range
    P.words[MT_W_KIND] = kind;
    *P.info = len | kind << 32 | tags << 40;
    if (len > P.out_cap) {
        P.words[MT_W_OVER] = 1;
        atomicOr(P.err, 1);
    }
}

// Grid over max(cap_total, nrange, 1) threads.
__global__ void __launch_bounds__(256) mt_write_kernel(const MtParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || P.words[MT_W_OVER]) return;
    const u64 kind = P.words[MT_W_KIND];
    const MtPlan& R = P.plan[P.nn - 1];
    if (kind == 2) {
        if (t < (P.range ? P.nrange : 1)) {
            P.out_key[t] = P.range ? P.range[t] : 0;
            P.out_word[t] = R.word;
            P.out_tag[t] = R.tag;
        }
    } else if (kind == 1 && R.kind == MK_MAP0) {
        if (t == 0) {
            P.out_key[0] = 0;
            P.out_word[0] = R.word;
            P.out_tag[0] = R.tag;
        }
    } else if (kind == 1 && t < *P.ulen && P.flag[t]) {
        const u64 p = P.pos[t];
        u8 g = P.rtag[t];
        u64 w = P.rword[t];
        if (g == MT_INT && P.words[MT_W_PROMOTE]) {
            g = MT_FLT;
            w = mt_u(__ll2double_rn((long long)w));
        }
        P.out_key[p] = P.U[t];
        P.out_word[p] = w;
        P.out_tag[p] = g;
    }
}

}  // namespace dgx
