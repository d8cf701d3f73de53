/*
 * groupby_oracle.c -- @groupby over one uid attribute (query/groupby.go) restated line by line.  TEST INFRASTRUCTURE
 * ONLY: the checker of dgx_groupby_uid in tests/ and the CPU leg of tools/bench_ops.py C13.  groupby_oracle.py compiles
 * it into a temporary directory.
 *
 * orc_groupby_uid(src, nrows, v, v_off, par, par_off, npar, ...): for every parent row ul, formResult's "UID node"
 * branch (groupby.go:208-221) for a child with IgnoreResult set: child row i takes part iff IndexOf(ul, SrcUIDs[i]) >= 0
 * (a binary search of ul), and each of its values d appends SrcUIDs[i] to d's entity list through dedup.addValue
 * (groupby.go:104-128: a map from the key to the group, a new group appended at the end of dedup.groups).  formGroups
 * then keeps every group (one attribute: no IntersectWith cross product), aggregateChild gives it count(uid) = the size
 * of its entity list (groupby.go:33-48), and the groups are ordered with groupLess (groupby.go:385-430): the entity
 * counts, then the aggregate counts (one each), then the keys with types.Less on UidID (uint64 <).
 * fillGroupedVars (groupby.go:265-361) is the same computation over every child row: one parent equal to SrcUIDs.
 *
 * Output per parent p, in order: its groups grp_off[p] .. grp_off[p+1]; group g's key keys[g], its count(uid) agg[g]
 * and its entity list members[mem_off[g] .. mem_off[g+1]).  keys / agg need room for every group and members for every
 * entity; returns the number of groups, or (size_t)-1 when an allocation fails.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

size_t orc_groupby_uid(const uint64_t* src, size_t nrows, const uint64_t* v, const uint64_t* v_off,
                       const uint64_t* par, const uint64_t* par_off, size_t npar, uint64_t* keys, uint64_t* agg,
                       uint64_t* grp_off, uint64_t* mem_off, uint64_t* members);

/* algo.IndexOf (algo/uidlist.go): sort.Search for the first uid >= x, -1 unless it is x. */
static long index_of(const uint64_t* ul, size_t n, uint64_t x) {
    size_t lo = 0, hi = n;
    while (lo < hi) {
        size_t mid = lo + (hi - lo) / 2;
        if (ul[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo < n && ul[lo] == x ? (long)lo : -1;
}

typedef struct { /* groupResult: one key, its entity list */
    uint64_t key;
    uint64_t* uids;
    size_t n, cap;
} group;

typedef struct { /* dedup: groups in the order they were made, and a map from key to group */
    group* groups;
    size_t n, cap;
    size_t* slot; /* open addressing over keys: group index + 1, 0 empty */
    size_t nslot;
} dedup;

static size_t hash_key(uint64_t k, size_t mask) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    return (size_t)k & mask;
}

static int grow_map(dedup* d) {
    size_t ns = d->nslot ? 2 * d->nslot : 64;
    size_t* s = calloc(ns, sizeof(size_t));
    if (!s) return -1;
    for (size_t g = 0; g < d->n; ++g) {
        size_t h = hash_key(d->groups[g].key, ns - 1);
        while (s[h]) h = (h + 1) & (ns - 1);
        s[h] = g + 1;
    }
    free(d->slot);
    d->slot = s;
    d->nslot = ns;
    return 0;
}

/* dedup.addValue(attr, value, uid): find the key's group, or make one at the end; append uid to its list. */
static int add_value(dedup* d, uint64_t key, uint64_t uid) {
    if (2 * (d->n + 1) > d->nslot && grow_map(d)) return -1;
    size_t h = hash_key(key, d->nslot - 1);
    while (d->slot[h] && d->groups[d->slot[h] - 1].key != key) h = (h + 1) & (d->nslot - 1);
    if (!d->slot[h]) {
        if (d->n == d->cap) {
            size_t nc = d->cap ? 2 * d->cap : 16;
            group* ng = realloc(d->groups, nc * sizeof(group));
            if (!ng) return -1;
            d->groups = ng;
            d->cap = nc;
        }
        d->groups[d->n] = (group){key, NULL, 0, 0};
        d->slot[h] = ++d->n;
    }
    group* g = &d->groups[d->slot[h] - 1];
    if (g->n == g->cap) {
        size_t nc = g->cap ? 2 * g->cap : 4;
        uint64_t* nu = realloc(g->uids, nc * sizeof(uint64_t));
        if (!nu) return -1;
        g->uids = nu;
        g->cap = nc;
    }
    g->uids[g->n++] = uid;
    return 0;
}

/* groupLess(a, b): len(uids), then len(aggregates) (one count(uid) each: equal), then the keys (types.Less, UidID). */
static int group_less(const void* pa, const void* pb) {
    const group *a = pa, *b = pb;
    if (a->n != b->n) return a->n < b->n ? -1 : 1;
    if (a->key != b->key) return a->key < b->key ? -1 : 1;
    return 0;
}

size_t orc_groupby_uid(const uint64_t* src, size_t nrows, const uint64_t* v, const uint64_t* v_off,
                       const uint64_t* par, const uint64_t* par_off, size_t npar, uint64_t* keys, uint64_t* agg,
                       uint64_t* grp_off, uint64_t* mem_off, uint64_t* members) {
    size_t ng = 0, nm = 0;
    mem_off[0] = 0;
    for (size_t p = 0; p < npar; ++p) {
        grp_off[p] = ng;
        const uint64_t* ul = par + par_off[p];
        const size_t nul = par_off[p + 1] - par_off[p];
        dedup d = {0};
        int bad = 0;
        /* formResult: for i, srcUid := range child.SrcUIDs.Uids { if algo.IndexOf(ul, srcUid) < 0 { continue } ... } */
        for (size_t i = 0; i < nrows && !bad; ++i) {
            if (index_of(ul, nul, src[i]) < 0) continue;
            for (uint64_t k = v_off[i]; k < v_off[i + 1] && !bad; ++k) bad = add_value(&d, v[k], src[i]);
        }
        if (!bad) {
            /* formGroups: one attribute, every group kept with its aggregate count(uid); then sort.Slice(groupLess) */
            qsort(d.groups, d.n, sizeof(group), group_less);
            for (size_t g = 0; g < d.n; ++g) {
                keys[ng] = d.groups[g].key;
                agg[ng] = d.groups[g].n;
                memcpy(members + nm, d.groups[g].uids, d.groups[g].n * sizeof(uint64_t));
                nm += d.groups[g].n;
                mem_off[++ng] = nm;
            }
        }
        for (size_t g = 0; g < d.n; ++g) free(d.groups[g].uids);
        free(d.groups);
        free(d.slot);
        if (bad) return (size_t)-1;
    }
    grp_off[npar] = ng;
    return ng;
}
