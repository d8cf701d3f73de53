/*
 * sg_filter_oracle.c -- a subgraph's @filter tree and first / offset restated line by line from the reference:
 *   filterCopy (query/query.go :458-489): the filter tree hangs under the node as sg.Filters = [root];
 *   ProcessGraph's filter block (:2310-2373): every filter runs with SrcUIDs = the node's DestUIDs and is skipped,
 *     its DestUIDs left nil, when that is empty; an op node's DestUIDs starts as a copy of its SrcUIDs (:2219-2224);
 *     "or" MergeSorted, "not" Difference(DestUIDs, child), "and" IntersectSorted, and the node itself (no FilterOp)
 *     IntersectSorted(append(lists, DestUIDs));
 *   applyPagination (:2492-2507) with updateUidMatrix (:1425-1439, uid-sorted rows: IntersectWith(l, DestUIDs, l)) and
 *     x.PageRange (x/x.go:738-767); without pagination the rows meet DestUIDs in populateVarMap (:1461-1463);
 *   the DoCount block (:2402-2413): updateUidMatrix, then counts[i] = len(row i);
 *   handleUidPostings' compareScalarFn / hasFn / uidInFn branches (worker/task.go:880-948) with evalCompare
 *     (worker/compare.go): a COUNT leaf's DestUIDs are the SrcUIDs whose count compares true, in order.
 * The set operations are oracle/oracle.c's restatements of algo/uidlist.go.  TEST INFRASTRUCTURE ONLY.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

enum { OP_LEAF = 0, OP_AND = 1, OP_OR = 2, OP_NOT = 3 };
enum { K_LIST = 0, K_COUNT = 1 };

typedef struct {
    uint64_t* u; /* malloc'ed, or NULL */
    size_t n;
    int nil;     /* Go's nil *pb.List */
} List;

typedef struct {
    size_t nnodes;
    const uint8_t* op;
    const uint32_t* parent;
    const uint32_t* leaf;
    const int* kind;
    const int* cmp;
    const int64_t* thr;
    const uint64_t* lists;
    const uint64_t* list_off;  /* per leaf: LIST uids */
    const int64_t* cvals;
    const uint64_t* cval_off;  /* per leaf: c_i of each SrcUIDs value (COUNT) */
    int oom;
} Ctx;

/* worker/compare.go evalCompare: le ge lt gt eq */
static int eval_compare(int cmp, int64_t lv, int64_t rv) {
    switch (cmp) {
        case 0: return lv <= rv;
        case 1: return lv >= rv;
        case 2: return lv < rv;
        case 3: return lv > rv;
        default: return lv == rv;
    }
}

/* x.PageRange */
static void page_range(long long count, long long offset, long long n, long long* s, long long* e) {
    if (n == 0) { *s = 0; *e = 0; return; }
    if (count == 0 && offset == 0) { *s = 0; *e = n; return; }
    if (count < 0) {
        if (count * -1 > n) count = -n;
        *s = (((n + count) % n) + n) % n;
        *e = n;
        return;
    }
    long long start = offset;
    if (start < 0) start = 0;
    if (start > n) { *s = n; *e = n; return; }
    if (count == 0) { *s = start; *e = n; return; }
    long long end = start + count;
    if (end > n) end = n;
    *s = start;
    *e = end;
}

static uint64_t* alloc_u64(Ctx* c, size_t n) {
    uint64_t* p = (uint64_t*)malloc((n ? n : 1) * sizeof(uint64_t));
    if (!p) c->oom = 1;
    return p;
}

static List copy_list(Ctx* c, const uint64_t* u, size_t n) {
    List l = {alloc_u64(c, n), n, 0};
    if (l.u && n) memcpy(l.u, u, n * sizeof(uint64_t));
    return l;
}

/* ProcessGraph of filter node k with SrcUIDs src (the parent's DestUIDs): its DestUIDs. */
static List process(Ctx* c, uint32_t k, const List* src) {
    List none = {NULL, 0, 1};
    if (c->oom) return none;
    if (c->op[k] == OP_LEAF) {
        const uint32_t j = c->leaf[k];
        if (c->kind[j] == K_LIST)  /* the leaf's DestUIDs: a function's result, uid(var) or literal uids */
            return copy_list(c, c->lists + c->list_off[j], (size_t)(c->list_off[j + 1] - c->list_off[j]));
        /* handleUidPostings: a row [uid] per SrcUIDs value whose count compares true; DestUIDs = their merge */
        List d = {alloc_u64(c, src->n), 0, 0};
        if (!d.u) return none;
        const int64_t* cv = c->cvals + c->cval_off[j];
        for (size_t i = 0; i < src->n; ++i)
            if (eval_compare(c->cmp[j], cv[i], c->thr[j])) d.u[d.n++] = src->u[i];
        return d;
    }
    /* an op node: DestUIDs starts as a copy of SrcUIDs; its filters run with SrcUIDs = DestUIDs */
    List dest = copy_list(c, src->u, src->n);
    size_t nk = 0;
    for (size_t q = k + 1; q < c->nnodes; ++q)
        if (c->parent[q] == k) ++nk;
    List* kids = (List*)calloc(nk ? nk : 1, sizeof(List));
    if (!kids || !dest.u) { c->oom = 1; free(kids); free(dest.u); return none; }
    size_t i = 0;
    for (size_t q = k + 1; q < c->nnodes; ++q) {
        if (c->parent[q] != k) continue;
        if (dest.n == 0) kids[i++] = none;  /* skipped: filter.DestUIDs stays nil */
        else kids[i++] = process(c, (uint32_t)q, &dest);
    }
    List r = {NULL, 0, 0};
    const uint64_t** ptrs = (const uint64_t**)malloc((nk ? nk : 1) * sizeof(uint64_t*));
    size_t* lens = (size_t*)malloc((nk ? nk : 1) * sizeof(size_t));
    if (!ptrs || !lens) c->oom = 1;
    size_t tot = 0, mn = SIZE_MAX;
    for (i = 0; i < nk && !c->oom; ++i) {
        ptrs[i] = kids[i].u;
        lens[i] = kids[i].n;
        tot += kids[i].n;
        if (kids[i].n < mn) mn = kids[i].n;
    }
    if (!c->oom) {
        if (c->op[k] == OP_OR) {
            r.u = alloc_u64(c, tot);
            if (r.u) r.n = orc_merge_sorted(ptrs, lens, nk, r.u);
        } else if (c->op[k] == OP_NOT) {  /* x.AssertTrue(len(sg.Filters) == 1) */
            r.u = alloc_u64(c, dest.n);
            /* Difference(u, nil) is empty (algo/uidlist.go:332-335) */
            if (r.u) r.n = kids[0].nil ? 0 : orc_difference(dest.u, dest.n, kids[0].u, kids[0].n, r.u);
        } else {
            r.u = alloc_u64(c, nk ? mn : 0);
            if (r.u) r.n = orc_intersect_sorted(ptrs, lens, nk, r.u);
        }
    }
    for (i = 0; i < nk; ++i) free(kids[i].u);
    free(kids);
    free(ptrs);
    free(lens);
    free(dest.u);
    return r;
}

/* One node with DestUIDs d0 and uid matrix (v, v_off): its new DestUIDs, rows and counts.  Returns 0, or -1 when an
 * allocation failed.  dest_out holds n0 values, out v_off[nrows]. */
int orc_sg_filter(size_t nnodes, const uint8_t* op, const uint32_t* parent, const uint32_t* leaf, const int* kind,
                  const int* cmp, const int64_t* thr, const uint64_t* lists, const uint64_t* list_off,
                  const int64_t* cvals, const uint64_t* cval_off, const uint64_t* d0, size_t n0, const uint64_t* v,
                  const uint64_t* v_off, size_t nrows, int32_t count, int32_t offset, uint64_t* dest_out,
                  size_t* dest_len, uint64_t* out, uint64_t* out_off, uint32_t* counts) {
    Ctx c = {nnodes, op, parent, leaf, kind, cmp, thr, lists, list_off, cvals, cval_off, 0};
    List D = copy_list(&c, d0, n0);
    if (c.oom) return -1;
    /* the filter block: sg.Filters = [root], no FilterOp -> IntersectSorted(append(lists, sg.DestUIDs)) */
    List f = {NULL, 0, 1};
    if (D.n != 0) f = process(&c, 0, &D);
    if (c.oom) { free(D.u); free(f.u); return -1; }
    {
        const uint64_t* ptrs[2] = {f.u, D.u};
        size_t lens[2] = {f.n, D.n};
        List d1 = {alloc_u64(&c, D.n), 0, 0};
        if (!d1.u) { free(D.u); free(f.u); return -1; }
        d1.n = orc_intersect_sorted(ptrs, lens, 2, d1.u);
        free(f.u);
        free(D.u);
        D = d1;
    }
    /* updateUidMatrix: every row meets the new DestUIDs (in place), then applyPagination's cut */
    uint64_t* rows = alloc_u64(&c, v_off[nrows]);
    size_t* rs = (size_t*)malloc((nrows ? nrows : 1) * sizeof(size_t));
    size_t* rn = (size_t*)malloc((nrows ? nrows : 1) * sizeof(size_t));
    if (!rows || !rs || !rn) { free(rows); free(rs); free(rn); free(D.u); return -1; }
    if (v_off[nrows]) memcpy(rows, v, v_off[nrows] * sizeof(uint64_t));
    for (size_t i = 0; i < nrows; ++i) {
        uint64_t* l = rows + v_off[i];
        rs[i] = 0;
        rn[i] = orc_intersect_with(l, (size_t)(v_off[i + 1] - v_off[i]), D.u, D.n, l);
    }
    if (count != 0 || offset != 0) {
        for (size_t i = 0; i < nrows; ++i) {
            long long s, e;
            page_range(count, offset, (long long)rn[i], &s, &e);
            rs[i] = (size_t)s;
            rn[i] = (size_t)(e - s);
        }
        /* sg.DestUIDs = algo.MergeSorted(sg.uidMatrix) */
        const uint64_t** ptrs = (const uint64_t**)malloc((nrows ? nrows : 1) * sizeof(uint64_t*));
        if (!ptrs) { free(rows); free(rs); free(rn); free(D.u); return -1; }
        size_t tot = 0;
        for (size_t i = 0; i < nrows; ++i) { ptrs[i] = rows + v_off[i] + rs[i]; tot += rn[i]; }
        List d2 = {alloc_u64(&c, tot), 0, 0};
        if (d2.u) d2.n = orc_merge_sorted(ptrs, rn, nrows, d2.u);
        free(ptrs);
        free(D.u);
        D = d2;
        if (!D.u) { free(rows); free(rs); free(rn); return -1; }
    }
    /* the DoCount block's updateUidMatrix meets rows that already lie in DestUIDs: counts are the row lengths */
    size_t k = 0;
    out_off[0] = 0;
    for (size_t i = 0; i < nrows; ++i) {
        if (out) memcpy(out + k, rows + v_off[i] + rs[i], rn[i] * sizeof(uint64_t));
        k += rn[i];
        out_off[i + 1] = k;
        counts[i] = (uint32_t)rn[i];
    }
    if (D.n) memcpy(dest_out, D.u, D.n * sizeof(uint64_t));
    *dest_len = D.n;
    free(rows);
    free(rs);
    free(rn);
    free(D.u);
    return 0;
}
