/* math_oracle.c -- math() restated line by line from the reference (query/math.go evalMathTree, processBinary,
 * processUnary, processBinaryBoolean, processTernary; query/aggregator.go ApplyVal, matchType, applyAdd .. applyCeil,
 * Value, compareValues; types/sort.go Less, Equal, mismatchedLess; types/scalar_types.go Safe; math.Mod; query/query.go
 * transformVars' leaf rule and valueVarAggregation's math branch).  TEST INFRASTRUCTURE ONLY: the checker of
 * dgx_math_eval in tests/ and in smoke().
 *
 * A types.Val is a type id, a nil bit (Value == nil) and a 64-bit word.  A ShardedMap is 30 shards keyed uid % 30;
 * Go visits the shards in index order and each shard's entries in an order of its own: here a shuffle drawn from
 * `seed` at every range statement, so one seed is one of Go's possible iteration orders.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { DEFAULT_ID = 0, INT_ID = 2, FLOAT_ID = 3, BOOL_ID = 4 };      /* types.TypeID */
enum { TAG_INT = 1, TAG_FLOAT = 2, TAG_BOOL = 3, TAG_NIL = 4 };       /* DGX_VAL_* */
enum { OP_CONST, OP_VAR, OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_MOD, OP_MIN, OP_MAX, OP_NEG, OP_SQRT, OP_FLOOR, OP_CEIL,
       OP_LT, OP_GT, OP_LE, OP_GE, OP_EQ, OP_NE, OP_COND };
enum { NSHARDS = 30, MAXN = 64 };

typedef struct { uint8_t tid, nil; uint64_t w; } Val;
static const Val NILVAL = {DEFAULT_ID, 1, 0};

static double as_f(uint64_t w) { double d; memcpy(&d, &w, 8); return d; }
static uint64_t as_w(double d) { uint64_t w; memcpy(&w, &d, 8); return w; }

/* ---- random iteration orders ---- */
static uint64_t g_rng;
static uint64_t rnd(void) {
    g_rng ^= g_rng << 13; g_rng ^= g_rng >> 7; g_rng ^= g_rng << 17;
    return g_rng;
}

/* ---- ShardedMap ---- */
/* A shard: its entries in insertion order and an open-addressing index over them (slot = entry + 1, 0 empty). */
typedef struct { uint64_t* k; Val* v; size_t n, cap; uint32_t* h; size_t hcap; } Shard;
typedef struct { Shard s[NSHARDS]; } SMap;

static SMap* smap_new(void) { return calloc(1, sizeof(SMap)); }
static void smap_free(SMap* m) {
    if (!m) return;
    for (int i = 0; i < NSHARDS; ++i) { free(m->s[i].k); free(m->s[i].v); free(m->s[i].h); }
    free(m);
}
static size_t hslot(const Shard* s, uint64_t k) {
    size_t h = (size_t)((k * 0x9E3779B97F4A7C15ull) >> 20) & (s->hcap - 1);
    while (s->h[h] && s->k[s->h[h] - 1] != k) h = (h + 1) & (s->hcap - 1);
    return h;
}
static long shard_find(const Shard* s, uint64_t k) {
    if (!s->hcap) return -1;
    const uint32_t e = s->h[hslot(s, k)];
    return e ? (long)e - 1 : -1;
}
static void shard_index(Shard* s) {  /* room for twice the entries */
    if (2 * (s->n + 1) <= s->hcap) return;
    free(s->h);
    s->hcap = s->hcap ? 2 * s->hcap : 16;
    while (s->hcap < 2 * (s->n + 1)) s->hcap *= 2;
    s->h = calloc(s->hcap, 4);
    for (size_t i = 0; i < s->n; ++i) s->h[hslot(s, s->k[i])] = (uint32_t)(i + 1);
}
static int smap_get(const SMap* m, uint64_t k, Val* out) {  /* a nil map holds nothing */
    if (!m) { *out = NILVAL; return 0; }
    const Shard* s = &m->s[k % NSHARDS];
    long i = shard_find(s, k);
    if (i < 0) { *out = NILVAL; return 0; }
    *out = s->v[i];
    return 1;
}
static void smap_set(SMap* m, uint64_t k, Val v) {
    Shard* s = &m->s[k % NSHARDS];
    long i = shard_find(s, k);
    if (i >= 0) { s->v[i] = v; return; }
    if (s->n == s->cap) {
        s->cap = s->cap ? 2 * s->cap : 8;
        s->k = realloc(s->k, s->cap * 8);
        s->v = realloc(s->v, s->cap * sizeof(Val));
    }
    shard_index(s);
    s->h[hslot(s, k)] = (uint32_t)(s->n + 1);
    s->k[s->n] = k;
    s->v[s->n++] = v;
}
static size_t smap_len(const SMap* m) {
    size_t n = 0;
    if (m) for (int i = 0; i < NSHARDS; ++i) n += m->s[i].n;
    return n;
}
/* One shard's keys in a fresh random order (a range statement over a Go map). */
static uint64_t* shard_order(const Shard* s) {
    uint64_t* o = malloc((s->n + 1) * 8);
    memcpy(o, s->k, s->n * 8);
    for (size_t i = s->n; i > 1; --i) {
        size_t j = rnd() % i;
        uint64_t t = o[i - 1]; o[i - 1] = o[j]; o[j] = t;
    }
    return o;
}
typedef int (*IterFn)(void* ctx, uint64_t k, Val v);
/* Not part of the restatement: set when an Iterate stopped by an error would have succeeded on some other key, the
 * case whose outcome depends on the iteration order (found by trying the remaining keys with g_dry set: no writes). */
static int g_partial, g_dry;
/* ShardedMap.Iterate: shards in index order, stops at (and returns) the first error. */
static int smap_iterate(const SMap* m, IterFn f, void* ctx) {
    if (!m) return 0;
    for (int i = 0; i < NSHARDS; ++i) {
        uint64_t* o = shard_order(&m->s[i]);
        for (size_t j = 0; j < m->s[i].n; ++j) {
            Val v;
            smap_get(m, o[j], &v);
            if (f(ctx, o[j], v)) {
                free(o);
                size_t ok = 0;
                g_dry = 1;
                for (int s = 0; s < NSHARDS; ++s)
                    for (size_t e = 0; e < m->s[s].n; ++e) ok += f(ctx, m->s[s].k[e], m->s[s].v[e]) == 0;
                g_dry = 0;
                if (ok) g_partial = 1;
                return 1;
            }
        }
        free(o);
    }
    return 0;
}

/* ---- aggregator ---- */
enum { VT_INT, VT_FLOAT, VT_DEFAULT };
static int getValType(const Val* v) { return v->tid == INT_ID ? VT_INT : v->tid == FLOAT_ID ? VT_FLOAT : VT_DEFAULT; }

static int matchType(Val* left, Val* right) {
    int lt = getValType(left), rt = getValType(right);
    if (lt == rt) return 0;
    if (lt == VT_DEFAULT || rt == VT_DEFAULT) return 1;
    if (lt == VT_INT) { left->tid = FLOAT_ID; left->w = as_w((double)(int64_t)left->w); }
    else { right->tid = FLOAT_ID; right->w = as_w((double)(int64_t)right->w); }  /* lt == FLOAT, rt == INT */
    return 0;
}

/* Go's int64 / and %: defined for MinInt64 / -1 (MinInt64) and MinInt64 % -1 (0). */
static int64_t go_div(int64_t a, int64_t b) { return b == -1 ? (int64_t)(0 - (uint64_t)a) : a / b; }
static int64_t go_mod(int64_t a, int64_t b) { return b == -1 ? 0 : a % b; }

/* math.Mod (src/math/mod.go) */
static double go_mathmod(double x, double y) {
    if (y == 0 || isinf(x) || isnan(x) || isnan(y)) return NAN;
    y = fabs(y);
    int yexp;
    double yfr = frexp(y, &yexp);
    double r = x;
    if (x < 0) r = -x;
    while (r >= y) {
        int rexp;
        double rfr = frexp(r, &rexp);
        if (rfr < yfr) rexp = rexp - 1;
        r = r - ldexp(y, rexp - yexp);
    }
    if (x < 0) r = -r;
    return r;
}

/* types.Less for the in-scope types: Int, Float, Default (through Safe(): "" < "" is false); Bool errs. */
static int types_less(Val a, Val b, int* r) {
    if (a.tid != b.tid) return 1;
    switch (a.tid) {
        case INT_ID: *r = (int64_t)a.w < (int64_t)b.w; return 0;
        case FLOAT_ID: *r = as_f(a.w) < as_f(b.w); return 0;
        case DEFAULT_ID: *r = 0; return 0;  /* a nil Val's Safe() is "" */
        default: return 1;
    }
}
/* types.Equal: a nil Default value is not a string, so it equals nothing. */
static int types_equal(Val a, Val b, int* r) {
    if (a.tid != b.tid) return 1;
    switch (a.tid) {
        case INT_ID: *r = a.w == b.w; return 0;
        case FLOAT_ID: *r = as_f(a.w) == as_f(b.w); return 0;
        case BOOL_ID: *r = !a.nil && !b.nil && a.w == b.w; return 0;
        case DEFAULT_ID: *r = 0; return 0;
        default: return 1;
    }
}

static int apply_binary(int op, Val* a, Val* b, Val* c) {
    int vb = getValType(a);
    if (op == OP_MIN || op == OP_MAX) {
        int r;
        if (types_less(*a, *b, &r)) return 1;
        *c = (op == OP_MIN) == (r != 0) ? *a : *b;
        return 0;
    }
    if (vb == VT_DEFAULT) return 1;
    if (vb == VT_INT) {
        int64_t x = (int64_t)a->w, y = (int64_t)b->w;
        switch (op) {
            case OP_ADD:
                if ((x > 0 && y > INT64_MAX - x) || (x < 0 && y < INT64_MIN - x)) return 1;
                c->w = (uint64_t)x + (uint64_t)y; break;
            case OP_SUB:
                if ((y < 0 && x > INT64_MAX + y) || (y > 0 && x < INT64_MIN + y)) return 1;
                c->w = (uint64_t)x - (uint64_t)y; break;
            case OP_MUL:
                c->tid = INT_ID;
                c->w = (uint64_t)x * (uint64_t)y;
                c->nil = 0;
                if (x == 0 || y == 0) return 0;
                if (go_div((int64_t)c->w, y) != x) return 1;
                break;
            case OP_DIV:
                if (y == 0) return 1;
                c->w = (uint64_t)go_div(x, y); c->tid = INT_ID; break;
            case OP_MOD:
                if (y == 0) return 1;
                c->w = (uint64_t)go_mod(x, y); break;
        }
        c->nil = 0;
        return 0;
    }
    double x = as_f(a->w), y = as_f(b->w), z = 0;
    switch (op) {
        case OP_ADD: z = x + y; break;
        case OP_SUB: z = x - y; break;
        case OP_MUL: z = x * y; c->tid = FLOAT_ID; break;
        case OP_DIV: if (y == 0) return 1; z = x / y; c->tid = FLOAT_ID; break;
        case OP_MOD: if (y == 0) return 1; z = go_mathmod(x, y); break;
    }
    c->w = as_w(z);
    c->nil = 0;
    return 0;
}

static int apply_unary(int op, Val* a, Val* res) {
    int vb = getValType(a);
    if (vb == VT_DEFAULT) return 1;
    res->nil = 0;
    if (vb == VT_INT) {
        int64_t x = (int64_t)a->w;
        switch (op) {
            case OP_NEG: if (x == INT64_MIN) return 1; res->w = 0 - (uint64_t)x; res->tid = INT_ID; return 0;
            case OP_SQRT: if (x < 0) return 1; res->w = as_w(sqrt((double)x)); res->tid = FLOAT_ID; return 0;
            default: res->w = a->w; return 0;  /* floor, ceil */
        }
    }
    double x = as_f(a->w);
    switch (op) {
        case OP_NEG: res->w = as_w(-x); res->tid = FLOAT_ID; return 0;
        case OP_SQRT: if (x < 0) return 1; res->w = as_w(sqrt(x)); return 0;
        case OP_FLOOR: res->w = as_w(floor(x)); return 0;
        default: res->w = as_w(ceil(x)); return 0;
    }
}

typedef struct { int op; Val result; } Agg;

/* ag.ApplyVal */
static int ApplyVal(Agg* ag, Val v) {
    if (v.nil) { v.nil = 0; v.w = 0; v.tid = INT_ID; }  /* a missing value is int64(0) */
    Val res = {0, 1, 0};
    if (ag->op >= OP_NEG && ag->op <= OP_CEIL) {
        res.tid = v.tid;
        if (apply_unary(ag->op, &v, &res)) return 1;
        ag->result = res;
        return 0;
    }
    if (ag->result.nil) { ag->result = v; return 0; }
    Val left = ag->result;
    if (matchType(&left, &v)) return 1;
    res.tid = left.tid;
    if (apply_binary(ag->op, &left, &v, &res)) return 1;
    ag->result = res;
    return 0;
}

/* ag.Value */
static int Value(Agg* ag, Val* out) {
    if (ag->result.nil) { *out = ag->result; return 1; }
    if (ag->result.tid == FLOAT_ID) {
        double x = as_f(ag->result.w);
        if (isinf(x) && x > 0) ag->result.w = as_w(1.7976931348623157e308);
        else if (isinf(x)) ag->result.w = as_w(-1.7976931348623157e308);
        else if (isnan(x)) ag->result.w = as_w(0.0);
    }
    *out = ag->result;
    return 0;
}

static int compareValues(int op, Val va, Val vb, int* out) {
    int r;
    if (types_less(va, vb, &r)) {
        if (va.tid == INT_ID) { va.tid = FLOAT_ID; va.w = as_w((double)(int64_t)va.w); }
        else if (vb.tid == INT_ID) { vb.tid = FLOAT_ID; vb.w = as_w((double)(int64_t)vb.w); }
        else return 1;
    }
    int isLess, isMore, isEqual;
    if (types_less(va, vb, &isLess) || types_less(vb, va, &isMore) || types_equal(va, vb, &isEqual)) return 1;
    switch (op) {
        case OP_LT: *out = isLess; break;
        case OP_GT: *out = isMore; break;
        case OP_LE: *out = isLess || isEqual; break;
        case OP_GE: *out = isMore || isEqual; break;
        case OP_EQ: *out = isEqual; break;
        default: *out = !isEqual; break;
    }
    return 0;
}

/* ---- mathTree ---- */
typedef struct { int fn, var, nchild, child[3]; Val cnst; SMap* val; } Node;
static Node g_n[MAXN];

static int is_const(const Val* v) { return !v->nil; }

/* processBinary's f */
static void bin_f(int op, uint64_t k, SMap* mpl, SMap* mpr, Val cl, Val cr, SMap* dest) {
    Agg ag = {op, NILVAL};
    Val lVal, rVal, out;
    smap_get(mpl, k, &lVal);
    if (is_const(&cl)) lVal = cl;
    smap_get(mpr, k, &rVal);
    if (is_const(&cr)) rVal = cr;
    if (ApplyVal(&ag, lVal) || ApplyVal(&ag, rVal) || Value(&ag, &out)) return;  /* the error is ignored */
    smap_set(dest, k, out);
}

static int checkAggrResult(const SMap* m, Val* v) {
    if (smap_len(m) != 1) return 0;
    return smap_get(m, 0, v);
}

static int processBinary(Node* n) {
    SMap *mpl = g_n[n->child[0]].val, *mpr = g_n[n->child[1]].val;
    Val cl = g_n[n->child[0]].cnst, cr = g_n[n->child[1]].cnst, v;
    if (checkAggrResult(mpl, &v)) { cl = v; mpl = NULL; }
    else if (checkAggrResult(mpr, &v)) { cr = v; mpr = NULL; }
    if (smap_len(mpl) != 0 || smap_len(mpr) != 0) {
        SMap* ret = smap_new();
        for (int i = 0; i < NSHARDS; ++i) {
            Shard empty = {0};
            const Shard* ls = mpl ? &mpl->s[i] : &empty;
            const Shard* rs = mpr ? &mpr->s[i] : &empty;
            uint64_t* o = shard_order(ls);
            for (size_t j = 0; j < ls->n; ++j) bin_f(n->fn, o[j], mpl, mpr, cl, cr, ret);
            free(o);
            o = shard_order(rs);
            for (size_t j = 0; j < rs->n; ++j) {
                if (shard_find(ls, o[j]) >= 0) continue;
                bin_f(n->fn, o[j], mpl, mpr, cl, cr, ret);
            }
            free(o);
        }
        n->val = ret;
        return 0;
    }
    if (is_const(&cl) && is_const(&cr)) {
        Agg ag = {n->fn, NILVAL};
        if (ApplyVal(&ag, cl) || ApplyVal(&ag, cr)) return 1;
        return Value(&ag, &n->cnst);
    }
    return 0;
}

typedef struct { Agg* ag; SMap* dest; } UnCtx;
static int un_f(void* c, uint64_t k, Val val) {
    UnCtx* u = c;
    Val value;
    if (ApplyVal(u->ag, val) || Value(u->ag, &value)) return 1;
    if (!g_dry) smap_set(u->dest, k, value);
    return 0;
}
static int processUnary(Node* n) {
    Node* ch = &g_n[n->child[0]];
    SMap* dest = smap_new();
    Agg ag = {n->fn, NILVAL};
    if (is_const(&ch->cnst)) {
        smap_free(dest);
        if (ApplyVal(&ag, ch->cnst)) return 1;
        return Value(&ag, &n->cnst);
    }
    UnCtx u = {&ag, dest};
    smap_iterate(ch->val, un_f, &u);  /* the error that stops Iterate is discarded */
    n->val = dest;
    return 0;
}

typedef struct { int op; Node* ch; SMap* dest; } CmpCtx;
static int cmp_f(void* c, uint64_t k, Val val) {
    CmpCtx* u = c;
    Val curVal;
    smap_get(u->ch->val, k, &curVal);
    if (is_const(&u->ch->cnst)) curVal = u->ch->cnst;
    int res;
    if (compareValues(u->op, val, curVal, &res)) return 1;
    Val b = {BOOL_ID, 0, (uint64_t)res};
    if (!g_dry) smap_set(u->dest, k, b);
    return 0;
}
static int processBinaryBoolean(Node* n) {
    CmpCtx u = {n->fn, &g_n[n->child[1]], smap_new()};
    smap_iterate(g_n[n->child[0]].val, cmp_f, &u);
    n->val = u.dest;
    return 0;
}

typedef struct { Node *one, *two; SMap* dest; } CondCtx;
static int cond_f(void* c, uint64_t k, Val val) {
    CondCtx* u = c;
    Val res;
    if (val.tid != BOOL_ID || val.nil) return 1;
    Node* b = val.w ? u->one : u->two;
    if (is_const(&b->cnst)) res = b->cnst;
    else smap_get(b->val, k, &res);
    if (!g_dry) smap_set(u->dest, k, res);
    return 0;
}
static int processTernary(Node* n) {
    SMap* condMap = g_n[n->child[0]].val;
    if (!condMap) return 1;  /* IsEmpty: a nil map */
    CondCtx u = {&g_n[n->child[1]], &g_n[n->child[2]], smap_new()};
    smap_iterate(condMap, cond_f, &u);
    n->val = u.dest;
    return 0;
}

static int evalMathTree(int i) {
    Node* n = &g_n[i];
    if (is_const(&n->cnst)) return 0;
    if (n->var >= 0) return 0;
    for (int c = 0; c < n->nchild; ++c)
        if (evalMathTree(n->child[c])) return 1;
    if (n->fn >= OP_NEG && n->fn <= OP_CEIL) return processUnary(n);
    if (n->fn >= OP_ADD && n->fn <= OP_MAX) return processBinary(n);
    if (n->fn >= OP_LT && n->fn <= OP_NE) return processBinaryBoolean(n);
    return processTernary(n);
}

static Val tag_val(uint8_t tag, uint64_t w) {
    Val v = {0, 0, w};
    switch (tag) {
        case TAG_INT: v.tid = INT_ID; break;
        case TAG_FLOAT: v.tid = FLOAT_ID; break;
        case TAG_BOOL: v.tid = BOOL_ID; break;
        default: v = NILVAL; break;
    }
    return v;
}
static uint8_t val_tag(Val v) {
    if (v.nil) return TAG_NIL;
    return v.tid == INT_ID ? TAG_INT : v.tid == FLOAT_ID ? TAG_FLOAT : v.tid == BOOL_ID ? TAG_BOOL : TAG_NIL;
}

static int cmp_u64(const void* a, const void* b) {
    uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
    return x < y ? -1 : x > y;
}

typedef struct { int* isInt; int* isFloat; SMap* m; } TopCtx;
static int top_scan(void* c, uint64_t k, Val v) {
    TopCtx* t = c;
    (void)k;
    if (v.tid == FLOAT_ID && !v.nil) *t->isFloat = 1;
    if (v.tid == INT_ID && !v.nil) *t->isInt = 1;
    return 0;
}
static int top_promote(void* c, uint64_t k, Val v) {
    TopCtx* t = c;
    if (v.tid == INT_ID) { v.tid = FLOAT_ID; v.w = as_w((double)(int64_t)v.w); }
    smap_set(t->m, k, v);
    return 0;
}

/* One math() evaluation.  Program arrays as dgx_math_node (op, const_tag, child[3], leaf, const_word), leaves as
 * (keys, words, tags) with lengths and nil bits; range (nrange uids) or has_range 0.  Returns -1 where evalMathTree
 * returns an error, else the kind (0 none, 1 map, 2 const) with the result sorted by key into out_* (*out_len);
 * *partial as g_partial. */
int64_t orc_math(const uint8_t* op, const uint8_t* ctag, const uint16_t* child, const uint32_t* leaf,
                 const uint64_t* cword, size_t nn, const uint64_t* const* lkey, const uint64_t* const* lword,
                 const uint8_t* const* ltag, const uint64_t* llen, const uint8_t* lnil, const uint64_t* range,
                 size_t nrange, int has_range, uint64_t seed, uint64_t* out_key, uint64_t* out_word, uint8_t* out_tag,
                 uint64_t* out_len, int* partial) {
    g_partial = 0;
    g_rng = seed * 0x9E3779B97F4A7C15ull + 0x2545F4914F6CDD1Dull;
    if (!g_rng) g_rng = 1;
    for (size_t i = 0; i < nn; ++i) {
        Node* n = &g_n[i];
        memset(n, 0, sizeof *n);
        n->fn = op[i];
        n->var = -1;
        n->cnst = NILVAL;
        n->nchild = op[i] == OP_COND ? 3 : op[i] >= OP_NEG && op[i] <= OP_CEIL ? 1 : op[i] >= OP_ADD ? 2 : 0;
        for (int c = 0; c < 3; ++c) n->child[c] = child[3 * i + c];
        if (op[i] == OP_CONST) n->cnst = tag_val(ctag[i], cword[i]);
        if (op[i] == OP_VAR) {
            /* transformVars: the leaf's map; {MaxUint64: v} alone is the constant v */
            const uint32_t j = leaf[i];
            n->var = (int)j;
            if (lnil[j]) continue;
            if (llen[j] == 1 && lkey[j][0] == UINT64_MAX) { n->cnst = tag_val(ltag[j][0], lword[j][0]); continue; }
            n->val = smap_new();
            for (uint64_t e = 0; e < llen[j]; ++e) smap_set(n->val, lkey[j][e], tag_val(ltag[j][e], lword[j][e]));
        }
    }
    int64_t kind = 0;
    *out_len = 0;
    if (evalMathTree((int)nn - 1)) {
        kind = -1;
    } else {
        Node* r = &g_n[nn - 1];
        if (smap_len(r->val) != 0) {
            int isInt = 0, isFloat = 0;
            TopCtx t = {&isInt, &isFloat, r->val};
            smap_iterate(r->val, top_scan, &t);
            if (isInt && isFloat) smap_iterate(r->val, top_promote, &t);
            kind = 1;
            size_t m = 0;
            for (int s = 0; s < NSHARDS; ++s)
                for (size_t e = 0; e < r->val->s[s].n; ++e) out_key[m++] = r->val->s[s].k[e];
            qsort(out_key, m, 8, cmp_u64);
            for (size_t e = 0; e < m; ++e) {
                Val v;
                smap_get(r->val, out_key[e], &v);
                out_word[e] = v.nil ? 0 : v.w;
                out_tag[e] = val_tag(v);
            }
            *out_len = m;
        } else if (is_const(&r->cnst)) {
            kind = 2;
            const size_t m = has_range ? nrange : 1;
            for (size_t e = 0; e < m; ++e) {
                out_key[e] = has_range ? range[e] : 0;
                out_word[e] = r->cnst.w;
                out_tag[e] = val_tag(r->cnst);
            }
            *out_len = m;
        }
    }
    for (size_t i = 0; i < nn; ++i) smap_free(g_n[i].val);
    *partial = g_partial;
    return kind;
}
