/* valvar_oracle.c -- value variables restated line by line from the reference (query/query.go transformTo
 * :1143-1236, evalLevelAgg :1042-1125; query/aggregator.go Apply :794-854, divideByCount, Value :905-921;
 * types/sort.go Less; types/sharded_map.go Merge).  TEST INFRASTRUCTURE ONLY: the checker of dgx_var_propagate and
 * dgx_var_level_agg in tests/ and the CPU leg of tools/bench_ops.py C17.
 *
 * A types.Val of IntID or FloatID is a 64-bit word and the map's type; a ShardedMap is an open-addressing hash map.
 * Go runs transformTo's four chunks as goroutines and merges each tempMap into resultMap as it finishes: `order` is
 * that completion order (a permutation of 0..3).
 */
#include <math.h>
#include <float.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { INT64 = 1, FLOAT64 = 2 };
enum { MIN = 0, MAX = 1, SUM = 2, AVG = 3 };

static double as_f(uint64_t w) { double d; memcpy(&d, &w, 8); return d; }
static uint64_t as_w(double d) { uint64_t w; memcpy(&w, &d, 8); return w; }

/* ---- ShardedMap: uid -> 64-bit word ---- */
typedef struct { uint64_t* k; uint64_t* v; uint8_t* used; size_t cap, n; } Map;

static int map_init(Map* m, size_t hint) {
    size_t cap = 16;
    while (cap < 2 * hint + 2) cap <<= 1;
    m->k = calloc(cap, 8); m->v = calloc(cap, 8); m->used = calloc(cap, 1);
    m->cap = cap; m->n = 0;
    return m->k && m->v && m->used ? 0 : -1;
}
static void map_free(Map* m) { free(m->k); free(m->v); free(m->used); memset(m, 0, sizeof *m); }
static size_t map_slot(const Map* m, uint64_t key) {
    size_t h = (size_t)((key * 0x9E3779B97F4A7C15ull) >> 17) & (m->cap - 1);
    while (m->used[h] && m->k[h] != key) h = (h + 1) & (m->cap - 1);
    return h;
}
static int map_get(const Map* m, uint64_t key, uint64_t* val) {
    const size_t h = map_slot(m, key);
    if (!m->used[h]) return 0;
    *val = m->v[h];
    return 1;
}
static void map_set(Map* m, uint64_t key, uint64_t val) {  /* room for every key is reserved by map_init */
    const size_t h = map_slot(m, key);
    if (!m->used[h]) { m->used[h] = 1; m->k[h] = key; m->n++; }
    m->v[h] = val;
}

/* ---- aggregator ---- */
typedef struct { int name, typ, has; uint64_t result; uint64_t count; } Agg;

/* types.Less on one type */
static int less(int typ, uint64_t a, uint64_t b) { return typ == FLOAT64 ? as_f(a) < as_f(b) : (int64_t)a < (int64_t)b; }

static void apply(Agg* ag, uint64_t val) {
    if (!ag->has) { ag->result = val; ag->has = 1; ag->count++; return; }
    const uint64_t va = ag->result, vb = val;
    uint64_t res;
    switch (ag->name) {
    case MIN: res = less(ag->typ, va, vb) ? va : vb; break;
    case MAX: res = less(ag->typ, va, vb) ? vb : va; break;
    default:  /* sum, avg */
        res = ag->typ == INT64 ? (uint64_t)((int64_t)va + (int64_t)vb)  /* int64 wraps in Go */
                               : as_w(as_f(va) + as_f(vb));
    }
    ag->count++;
    ag->result = res;
}

/* Value(): divideByCount for avg (the result becomes FloatID), then the float clamp.  *typ gets the result type. */
static uint64_t value(Agg* ag, int* typ) {
    int t = ag->typ;
    uint64_t r = ag->result;
    if (ag->name == AVG && ag->count) {
        const double v = t == INT64 ? (double)(int64_t)r : as_f(r);
        r = as_w(v / (double)ag->count);
        t = FLOAT64;
    }
    if (t == FLOAT64) {
        const double f = as_f(r);
        if (isinf(f) && f > 0) r = as_w(DBL_MAX);
        else if (isinf(f)) r = as_w(-1 * DBL_MAX);
        else if (isnan(f)) r = as_w(0.0);
    }
    if (typ) *typ = t;
    return r;
}

static uint64_t sum2(int typ, uint64_t a, uint64_t b) {  /* the Merge callback: Apply(a), Apply(b), Value() */
    Agg ag = {SUM, typ, 0, 0, 0};
    apply(&ag, a);
    apply(&ag, b);
    return value(&ag, NULL);
}

static int cmp_u64(const void* a, const void* b) {
    const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
    return x < y ? -1 : x > y;
}

/* Writes newMap's entries into out_key / out_val ascending by key; returns the count. */
static size_t map_sorted(const Map* m, uint64_t* out_key, uint64_t* out_val) {
    size_t n = 0;
    for (size_t h = 0; h < m->cap; ++h) if (m->used[h]) out_key[n++] = m->k[h];
    qsort(out_key, n, 8, cmp_u64);
    for (size_t i = 0; i < n; ++i) map_get(m, out_key[i], &out_val[i]);
    return n;
}

/* transformTo from the first level of the path on (the caller skips index 0).  Level l has nrows[l] rows: row i is
 * v[l][v_off[l][i] .. v_off[l][i+1]) of src[l][i].  Returns the last map's size (entries into out_key / out_val,
 * ascending), or -1 when an allocation fails. */
int64_t orc_propagate(int typ, const uint64_t* key, const uint64_t* val, size_t n, size_t nlevels,
                      const uint64_t* const* src, const uint64_t* nrows, const uint64_t* const* v_off,
                      const uint64_t* const* v, const int* order, uint64_t* out_key, uint64_t* out_val) {
    Map newMap;
    if (map_init(&newMap, n)) return -1;
    for (size_t i = 0; i < n; ++i) map_set(&newMap, key[i], val[i]);
    for (size_t l = 0; l < nlevels; ++l) {
        const size_t R = nrows[l];
        const uint64_t* off = v_off[l];
        Map temp[4];
        /* width := len(curNode.uidMatrix) / numThreadsVariablePropogation */
        const size_t width = R / 4;
        for (int c = 0; c < 4; ++c) {
            const size_t start = c * width, end = c == 3 ? R : (c + 1) * width;
            if (map_init(&temp[c], off[end] - off[start])) return -1;
            for (size_t i = start; i < end; ++i) {  /* calculate(start, end) */
                uint64_t curVal;
                if (!map_get(&newMap, src[l][i], &curVal)) continue;
                Agg ag = {SUM, typ, 0, 0, 0};
                for (uint64_t j = off[i]; j < off[i + 1]; ++j) {
                    ag.has = 0;  /* ag.result = types.Val{} */
                    const uint64_t dstUid = v[l][j];
                    apply(&ag, curVal);
                    uint64_t tempVal;
                    if (map_get(&temp[c], dstUid, &tempVal)) apply(&ag, tempVal);
                    map_set(&temp[c], dstUid, value(&ag, NULL));
                }
            }
        }
        /* the chunks finish in `order`: the first becomes resultMap, the others Merge into it */
        Map* resultMap = &temp[order[0]];
        for (int q = 1; q < 4; ++q) {
            Map* other = &temp[order[q]];
            Map grown;  /* room for both */
            if (map_init(&grown, resultMap->n + other->n)) return -1;
            for (size_t h = 0; h < resultMap->cap; ++h)
                if (resultMap->used[h]) map_set(&grown, resultMap->k[h], resultMap->v[h]);
            for (size_t h = 0; h < other->cap; ++h) {
                if (!other->used[h]) continue;
                uint64_t a;
                if (map_get(&grown, other->k[h], &a)) map_set(&grown, other->k[h], sum2(typ, a, other->v[h]));
                else map_set(&grown, other->k[h], other->v[h]);
            }
            map_free(resultMap);
            *resultMap = grown;
        }
        map_free(&newMap);
        newMap = *resultMap;
        for (int c = 0; c < 4; ++c) if (&temp[c] != resultMap) map_free(&temp[c]);
    }
    const size_t m = map_sorted(&newMap, out_key, out_val);
    map_free(&newMap);
    return (int64_t)m;
}

/* evalLevelAgg's loop over relSG's uid matrix: returns the entries written (keys src[i] in row order), or -1. */
int64_t orc_level_agg(int typ, int fn, const uint64_t* key, const uint64_t* val, size_t n, const uint64_t* src,
                      size_t nrows, const uint64_t* v_off, const uint64_t* v, uint64_t* out_key, uint64_t* out_val) {
    Map vals;
    if (map_init(&vals, n)) return -1;
    for (size_t i = 0; i < n; ++i) map_set(&vals, key[i], val[i]);
    size_t m = 0;
    for (size_t i = 0; i < nrows; ++i) {
        Agg ag = {fn, typ, 0, 0, 0};
        for (uint64_t j = v_off[i]; j < v_off[i + 1]; ++j) {
            uint64_t x;
            if (map_get(&vals, v[j], &x)) apply(&ag, x);
        }
        if (!ag.has) continue;  /* ErrEmptyVal: nothing set */
        out_key[m] = src[i];
        out_val[m] = value(&ag, NULL);
        m++;
    }
    map_free(&vals);
    return (int64_t)m;
}
