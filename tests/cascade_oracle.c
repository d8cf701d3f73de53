/*
 * cascade_oracle.c -- @cascade restated line by line: query/query.go populateVarMap :1445-1527 for every node of a
 * forest, updateUidMatrix :1425-1439 without facets, x.PageRange (x/x.go:738-767) and ProcessQuery's root pagination
 * :3004-3011.  TEST INFRASTRUCTURE ONLY: the checker of dgx_cascade in tests/ and the CPU leg of tools/bench_ops.py
 * C15.  cascade_oracle.py compiles it together with oracle/oracle.c.
 *
 * The forest is the CSR of dgx_cascade (include/dgx.h): node n has parent[n] (UINT32_MAX for a query root), flags[n]
 * (DGX_CASCADE_* bits, values repeated below), first[n] / offset[n] (Params.Cascade.First / Offset), counts_len[n]
 * (len(n.counts)), DestUIDs dest[dest_off[n] .. dest_off[n+1]), uidMatrix rows row_off[n] .. row_off[n+1] of (v, v_off)
 * and valueMatrix lengths as has_val[hv_off[n] .. hv_off[n+1]).  The flags stand for what the Go code reads:
 *   CASCADE   len(sg.Params.Cascade.Fields) > 0
 *   CHECKED   (cascadeAllPreds || cascadeArgMap[child.Attr]) && !child.IsInternal(), and child.Attr != "uid"
 *   FILTERED  len(sg.Filters) > 0
 *   ORDERED   len(sg.Params.Order) > 0 || len(sg.Params.FacetsOrder) > 0
 *   SKIP      sg.IsGroupBy() (return nil) or sg.Params.Alias == "shortest" (goto AssignStep)
 * orc_cascade writes every node's rows after the call to (out, out_off) and its DestUIDs to (dest_out, dest_out_off),
 * both in node order.  Returns 0, or -1 when an allocation fails.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

enum { CASCADE = 1, CHECKED = 2, FILTERED = 4, ORDERED = 8, SKIP = 16 };

typedef struct {
    uint64_t* u;
    size_t n;
} list;

typedef struct {
    size_t nnodes;
    const uint32_t* parent;
    const uint8_t* flags;
    const int32_t* first;
    const int32_t* offset;
    const uint64_t* counts_len;
    list* dest;         /* sg.DestUIDs */
    list** rows;        /* sg.uidMatrix */
    size_t* nrows;
    const uint8_t** hv; /* len(sg.valueMatrix[i].Values) > 0 */
    size_t* nhv;
} forest;

int orc_cascade(size_t nnodes, const uint32_t* parent, const uint8_t* flags, const int32_t* first,
                const int32_t* offset, const uint64_t* counts_len, const uint64_t* v, const uint64_t* v_off,
                const uint64_t* row_off, const uint64_t* dest, const uint64_t* dest_off, const uint8_t* has_val,
                const uint64_t* hv_off, uint64_t* out, uint64_t* out_off, uint64_t* dest_out, uint64_t* dest_out_off);

/* algo.IndexOf (algo/uidlist.go): sort.Search, then the equality test */
static long index_of(const list* l, uint64_t uid) {
    size_t lo = 0, hi = l->n;
    while (lo < hi) {
        size_t mid = lo + (hi - lo) / 2;
        if (l->u[mid] >= uid) hi = mid; else lo = mid + 1;
    }
    return lo < l->n && l->u[lo] == uid ? (long)lo : -1;
}

/* x.PageRange (x/x.go:738-767) */
static void page_range(long count, long offset, long n, long* start, long* end) {
    if (n == 0) { *start = 0; *end = 0; return; }
    if (count == 0 && offset == 0) { *start = 0; *end = n; return; }
    if (count < 0) {
        if (count * -1 > n) count = -n;
        *start = (((n + count) % n) + n) % n;
        *end = n;
        return;
    }
    long s = offset;
    if (s < 0) s = 0;
    if (s > n) { *start = n; *end = n; return; }
    if (count == 0) { *start = s; *end = n; return; }
    long e = s + count;
    if (e > n) e = n;
    *start = s;
    *end = e;
}

/* updateUidMatrix (:1425-1439) without updateFacetMatrix */
static void update_uid_matrix(forest* f, size_t sg) {
    for (size_t i = 0; i < f->nrows[sg]; ++i) {
        list* l = &f->rows[sg][i];
        if (f->flags[sg] & ORDERED) {
            /* algo.ApplyFilter(l, func(uid, idx) bool { return algo.IndexOf(sg.DestUIDs, uid) >= 0 }) */
            size_t k = 0;
            for (size_t j = 0; j < l->n; ++j)
                if (index_of(&f->dest[sg], l->u[j]) >= 0) l->u[k++] = l->u[j];
            l->n = k;
        } else {
            /* algo.IntersectWith(l, sg.DestUIDs, l) */
            l->n = orc_intersect_with(l->u, l->n, f->dest[sg].u, f->dest[sg].n, l->u);
        }
    }
}

static void page_rows(forest* f, size_t sg) {
    for (size_t i = 0; i < f->nrows[sg]; ++i) {
        long start, end;
        page_range(f->first[sg], f->offset[sg], (long)f->rows[sg][i].n, &start, &end);
        f->rows[sg][i].u += start; /* uidMatrix[i].Uids = uidMatrix[i].Uids[start:end] */
        f->rows[sg][i].n = (size_t)(end - start);
    }
}

static void populate_var_map(forest* f, size_t sg) {
    /* :1449  if sg.DestUIDs == nil || sg.IsGroupBy() { return nil }  and  :1460  Alias == "shortest": goto AssignStep */
    if (f->flags[sg] & SKIP) return;
    /* :1464 */
    if (f->flags[sg] & FILTERED) update_uid_matrix(f, sg);
    /* :1468  children in order: the forest is in pre-order, so they are the later nodes naming sg as parent */
    for (size_t child = sg + 1; child < f->nnodes; ++child) {
        if (f->parent[child] != sg) continue;
        populate_var_map(f, child);
        if (!(f->flags[child] & CASCADE)) continue;
        update_uid_matrix(f, child);
        if (f->first[child] != 0 || f->offset[child] != 0) page_rows(f, child);
    }
    /* :1494 */
    if (!(f->flags[sg] & CASCADE)) return;
    /* :1499  filter out UIDs that don't have at least one UID in every child */
    list* d = &f->dest[sg];
    size_t k = 0;
    for (size_t i = 0; i < d->n; ++i) {
        int exclude = 0;
        for (size_t child = sg + 1; child < f->nnodes && !exclude; ++child) {
            if (f->parent[child] != sg || !(f->flags[child] & CHECKED)) continue;
            if ((f->nhv[child] <= i || f->hv[child][i] == 0) && f->counts_len[child] <= i &&
                (f->nrows[child] <= i || f->rows[child][i].n == 0))
                exclude = 1;
        }
        if (!exclude) d->u[k++] = d->u[i]; /* out = append(out, uid); sg.DestUIDs = &pb.List{Uids: out} */
    }
    d->n = k;
}

int orc_cascade(size_t nnodes, const uint32_t* parent, const uint8_t* flags, const int32_t* first,
                const int32_t* offset, const uint64_t* counts_len, const uint64_t* v, const uint64_t* v_off,
                const uint64_t* row_off, const uint64_t* dest, const uint64_t* dest_off, const uint8_t* has_val,
                const uint64_t* hv_off, uint64_t* out, uint64_t* out_off, uint64_t* dest_out, uint64_t* dest_out_off) {
    forest f = {nnodes, parent, flags, first, offset, counts_len, NULL, NULL, NULL, NULL, NULL};
    const size_t nr = nnodes ? row_off[nnodes] : 0, m = nr ? v_off[nr] : 0, nd = nnodes ? dest_off[nnodes] : 0;
    uint64_t* vals = malloc((m + 1) * sizeof(uint64_t));
    uint64_t* dvals = malloc((nd + 1) * sizeof(uint64_t));
    list* rows = malloc((nr + 1) * sizeof(list));
    f.dest = malloc((nnodes + 1) * sizeof(list));
    f.rows = malloc((nnodes + 1) * sizeof(list*));
    f.nrows = malloc((nnodes + 1) * sizeof(size_t));
    f.hv = malloc((nnodes + 1) * sizeof(uint8_t*));
    f.nhv = malloc((nnodes + 1) * sizeof(size_t));
    int rc = -1;
    if (!vals || !dvals || !rows || !f.dest || !f.rows || !f.nrows || !f.hv || !f.nhv) goto done;
    if (m) memcpy(vals, v, m * sizeof(uint64_t));
    if (nd) memcpy(dvals, dest, nd * sizeof(uint64_t));
    for (size_t r = 0; r < nr; ++r) rows[r] = (list){vals + v_off[r], (size_t)(v_off[r + 1] - v_off[r])};
    for (size_t n = 0; n < nnodes; ++n) {
        f.dest[n] = (list){dvals + dest_off[n], (size_t)(dest_off[n + 1] - dest_off[n])};
        f.rows[n] = rows + row_off[n];
        f.nrows[n] = (size_t)(row_off[n + 1] - row_off[n]);
        f.hv[n] = has_val + hv_off[n];
        f.nhv[n] = (size_t)(hv_off[n + 1] - hv_off[n]);
    }
    for (size_t sg = 0; sg < nnodes; ++sg) {
        if (parent[sg] != UINT32_MAX) continue;
        populate_var_map(&f, sg);
        /* ProcessQuery :3004-3011: apply pagination at the root after @cascade */
        if ((flags[sg] & CASCADE) && (first[sg] != 0 || offset[sg] != 0)) {
            update_uid_matrix(&f, sg);
            page_rows(&f, sg);
        }
    }
    size_t w = 0;
    out_off[0] = 0;
    for (size_t r = 0; r < nr; ++r) {
        memmove(out + w, rows[r].u, rows[r].n * sizeof(uint64_t));
        w += rows[r].n;
        out_off[r + 1] = w;
    }
    w = 0;
    dest_out_off[0] = 0;
    for (size_t n = 0; n < nnodes; ++n) {
        memmove(dest_out + w, f.dest[n].u, f.dest[n].n * sizeof(uint64_t));
        w += f.dest[n].n;
        dest_out_off[n + 1] = w;
    }
    rc = 0;
done:
    free(vals);
    free(dvals);
    free(rows);
    free(f.dest);
    free(f.rows);
    free(f.nrows);
    free(f.hv);
    free(f.nhv);
    return rc;
}
