/*
 * recurse_oracle.c -- one sg of one level of @recurse (query/recurse.go expandRecurse :96-135) restated line by line.
 * TEST INFRASTRUCTURE ONLY: the checker of dgx_recurse_filter in tests/ and the CPU leg of tools/bench_ops.py C14.
 * recurse_oracle.py compiles it together with oracle/oracle.c.
 *
 * reachMap (:21) is a set of keys "attr|fromUID|toUID"; here a key is the triple (attr, from, to) with attr an integer
 * the caller gives each distinct sg.Attr string, so equal strings share keys exactly as the formatted strings do.
 *
 * orc_recurse_sg(set, attr, src, nrows, v, v_off, has_filters, dest, ndest, allow_loop, out, out_off, dest_out,
 * &dest_len) runs the body of the `for _, sg := range exec` loop for one sg whose uidMatrix is the CSR (v, v_off):
 *   :106-109  with filters, updateUidMatrix: algo.IntersectWith(l, sg.DestUIDs, l) on every row (query.go:1425-1439)
 *   :111-130  for every row, in SrcUIDs order: loop: true adds len(ul.Uids) of EVERY row for each fromUID; otherwise
 *             algo.ApplyFilter keeps uid iff its key is not in reachMap, inserting it and counting the edge
 *   :134      sg.DestUIDs = algo.MergeSorted(sg.uidMatrix)
 * The rows after the step go to (out, out_off), the DestUIDs to dest_out; returns the step's numEdges, or
 * (uint64_t)-1 when an allocation fails.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

typedef struct {
    uint64_t a, f, t;
} key3;

typedef struct {
    key3* slot;
    unsigned char* used;
    size_t n, cap; /* cap is a power of two */
} reach;

reach* orc_reach_new(void);
void orc_reach_free(reach* r);
int orc_reach_insert(reach* r, uint64_t attr, uint64_t from, uint64_t to);
size_t orc_reach_size(const reach* r);
size_t orc_reach_export(const reach* r, uint64_t attr, uint64_t* from, uint64_t* to);
uint64_t orc_recurse_sg(reach* r, uint64_t attr, const uint64_t* src, size_t nrows, const uint64_t* v,
                        const uint64_t* v_off, int has_filters, const uint64_t* dest, size_t ndest, int allow_loop,
                        uint64_t* out, uint64_t* out_off, uint64_t* dest_out, size_t* dest_len);

static size_t hash3(key3 k, size_t mask) {
    uint64_t h = k.a * 0x9e3779b97f4a7c15ull ^ k.f * 0xc2b2ae3d27d4eb4full ^ k.t * 0x165667b19e3779f9ull;
    h ^= h >> 33;
    h *= 0xff51afd7ed558ccdull;
    h ^= h >> 33;
    return (size_t)h & mask;
}

reach* orc_reach_new(void) { return calloc(1, sizeof(reach)); }

void orc_reach_free(reach* r) {
    if (!r) return;
    free(r->slot);
    free(r->used);
    free(r);
}

static int grow(reach* r) {
    size_t nc = r->cap ? 2 * r->cap : 1024;
    key3* s = malloc(nc * sizeof(key3));
    unsigned char* u = calloc(nc, 1);
    if (!s || !u) {
        free(s);
        free(u);
        return -1;
    }
    for (size_t i = 0; i < r->cap; ++i)
        if (r->used[i]) {
            size_t j = hash3(r->slot[i], nc - 1);
            while (u[j]) j = (j + 1) & (nc - 1);
            u[j] = 1;
            s[j] = r->slot[i];
        }
    free(r->slot);
    free(r->used);
    r->slot = s;
    r->used = u;
    r->cap = nc;
    return 0;
}

/* 1: inserted, 0: already there (`_, seen := reachMap[key]`), -1: out of memory */
int orc_reach_insert(reach* r, uint64_t attr, uint64_t from, uint64_t to) {
    if (2 * (r->n + 1) > r->cap && grow(r)) return -1;
    key3 k = {attr, from, to};
    size_t j = hash3(k, r->cap - 1);
    while (r->used[j]) {
        if (r->slot[j].a == attr && r->slot[j].f == from && r->slot[j].t == to) return 0;
        j = (j + 1) & (r->cap - 1);
    }
    r->used[j] = 1;
    r->slot[j] = k;
    r->n += 1;
    return 1;
}

size_t orc_reach_size(const reach* r) { return r->n; }

/* The keys of one attr, in table order (the caller sorts); from / to need room for orc_reach_size. */
size_t orc_reach_export(const reach* r, uint64_t attr, uint64_t* from, uint64_t* to) {
    size_t n = 0;
    for (size_t i = 0; i < r->cap; ++i)
        if (r->used[i] && r->slot[i].a == attr) {
            from[n] = r->slot[i].f;
            to[n] = r->slot[i].t;
            ++n;
        }
    return n;
}

uint64_t orc_recurse_sg(reach* r, uint64_t attr, const uint64_t* src, size_t nrows, const uint64_t* v,
                        const uint64_t* v_off, int has_filters, const uint64_t* dest, size_t ndest, int allow_loop,
                        uint64_t* out, uint64_t* out_off, uint64_t* dest_out, size_t* dest_len) {
    uint64_t num_edges = 0;
    size_t m = nrows ? v_off[nrows] : 0;
    /* the uid matrix, one owned slice per row: out is the rows' storage, len[i] each row's length */
    size_t* len = malloc((nrows + 1) * sizeof(size_t));
    if (!len) return (uint64_t)-1;
    memcpy(out, v, m * sizeof(uint64_t));
    for (size_t i = 0; i < nrows; ++i) len[i] = v_off[i + 1] - v_off[i];
    if (has_filters) /* sg.updateUidMatrix(): IntersectWith(l, sg.DestUIDs, l) */
        for (size_t i = 0; i < nrows; ++i) {
            uint64_t* l = out + v_off[i];
            len[i] = orc_intersect_with(l, len[i], dest, ndest, l);
        }
    for (size_t mIdx = 0; mIdx < nrows; ++mIdx) { /* for mIdx, fromUID := range sg.SrcUIDs.Uids */
        uint64_t fromUID = src[mIdx];
        if (allow_loop) {
            for (size_t i = 0; i < nrows; ++i) num_edges += len[i];
        } else { /* algo.ApplyFilter(sg.uidMatrix[mIdx], ...): kept values move to the front in order */
            uint64_t* l = out + v_off[mIdx];
            size_t w = 0;
            for (size_t i = 0; i < len[mIdx]; ++i) {
                int ins = orc_reach_insert(r, attr, fromUID, l[i]);
                if (ins < 0) {
                    free(len);
                    return (uint64_t)-1;
                }
                if (ins == 0) continue; /* seen: return false */
                num_edges++;
                l[w++] = l[i];
            }
            len[mIdx] = w;
        }
    }
    /* sg.DestUIDs = algo.MergeSorted(sg.uidMatrix) */
    const uint64_t** lists = malloc((nrows + 1) * sizeof(uint64_t*));
    if (!lists) {
        free(len);
        return (uint64_t)-1;
    }
    for (size_t i = 0; i < nrows; ++i) lists[i] = out + v_off[i];
    *dest_len = orc_merge_sorted(lists, len, nrows, dest_out);
    free(lists);
    /* the rows packed as CSR */
    size_t w = 0;
    out_off[0] = 0;
    for (size_t i = 0; i < nrows; ++i) {
        memmove(out + w, out + v_off[i], len[i] * sizeof(uint64_t));
        w += len[i];
        out_off[i + 1] = w;
    }
    free(len);
    return num_edges;
}
