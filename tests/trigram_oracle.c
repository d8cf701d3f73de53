/*
 * trigram_oracle.c -- uidsForRegex (worker/trigram.go:24-102) restated line by line.  TEST INFRASTRUCTURE ONLY: the
 * checker of dgx_trigram_query in tests/ and the CPU legs of tools/bench_ops.py C12.  It includes
 * list_uids_unfiltered_oracle.c (which includes list_uids_oracle.c), so that every trigram read is the same List.Uids
 * restatement the List.Uids row calls are checked against; trigram_oracle.py compiles it together with oracle/oracle.c
 * into a temporary directory.
 *
 * orc_uids_for_regex(tree..., packs, mut..., approx, npacks, lists, list_off, nlists, after_uid, out): the root call
 * uidsForRegex(attr, arg, query, &pb.List{}) (worker/task.go:1288) with arg.q.First = MaxInt32 (query/query.go:989-1019
 * leaves regexp out of the pagination parameters) and arg.q.AfterUid = after_uid.  The tree is the ABI's: node 0 the
 * root, op 2 = QAnd, 3 = QOr, each node's trigrams and subs as CSR.  Leaves 0 .. npacks-1 are unsplit posting lists
 * (pack, resolved REF layer, ApproxLen), read with List.Uids and the branch the reference picks: IntersectCompressedWith
 * without a mutable layer, findPostingWithItr per uid when len(Intersect) < ApproxLen, iterate otherwise
 * (posting/list.go:1795-1822).  Leaves npacks .. are lists the caller already read (a split list's pl.Uids without
 * Intersect): their filtered read is IntersectWith(list, Intersect).  out must hold the root's bound.  Returns the
 * result length, or (size_t)-1 for a node that is neither QAnd nor QOr (errRegexTooWide).
 */
#include "list_uids_unfiltered_oracle.c"

size_t orc_uids_for_regex(const uint8_t* op, const uint32_t* leaf_off, const uint32_t* leaf_idx, const uint32_t* sub_off,
                          const uint32_t* sub_idx, const orc_pack* const* packs, const uint64_t* mu, const uint8_t* mf,
                          const uint64_t* mut_off, const uint64_t* approx, size_t npacks, const uint64_t* lists,
                          const uint64_t* list_off, size_t nlists, uint64_t after_uid, uint64_t* out);

enum { ORC_QAND = 2, ORC_QOR = 3 };

typedef struct { /* *pb.List: nil, or Uids[0 .. n) */
    uint64_t* u;
    size_t n;
    int nil;
} tg_list;

typedef struct {
    const uint8_t* op;
    const uint32_t *leaf_off, *leaf_idx, *sub_off, *sub_idx;
    const orc_pack* const* packs;
    const uint64_t* mu;
    const uint8_t* mf;
    const uint64_t *mut_off, *approx;
    size_t npacks;
    const uint64_t *lists, *list_off;
    uint64_t after_uid;
    int err;
} tg_ctx;

static tg_list tg_alloc(size_t cap) {
    tg_list r = {(uint64_t*)malloc((cap + 1) * sizeof(uint64_t)), 0, 0};
    return r;
}

static tg_list tg_copy(const tg_list* x) {
    tg_list r = tg_alloc(x->n);
    memcpy(r.u, x->u, x->n * sizeof(uint64_t));
    r.n = x->n;
    r.nil = x->nil;
    return r;
}

/* uidsForTrigram (:35-42): pl.Uids(opts) with opts.Intersect = X (NULL: nil), First = MaxInt32 */
static tg_list uids_for_trigram(const tg_ctx* c, uint32_t leaf, const tg_list* X) {
    if (leaf >= c->npacks) { /* a list the caller read without Intersect; Uids then applies IntersectWith */
        const size_t j = leaf - c->npacks;
        const uint64_t* l = c->lists + c->list_off[j];
        const size_t n = (size_t)(c->list_off[j + 1] - c->list_off[j]);
        tg_list r = tg_alloc(n);
        if (X) r.n = orc_intersect_with(l, n, X->u, X->n, r.u);
        else { memcpy(r.u, l, n * sizeof(uint64_t)); r.n = n; }
        return r;
    }
    const orc_pack* p = c->packs[leaf];
    const size_t m0 = (size_t)c->mut_off[leaf], nmut = (size_t)(c->mut_off[leaf + 1] - m0);
    if (!X) {
        tg_list r = tg_alloc(orc_exact_len(p) + nmut);
        r.n = orc_list_uids_unfiltered(p, c->mu + m0, c->mf + m0, nmut, c->after_uid, 0x7fffffff, r.u);
        return r;
    }
    /* posting/list.go:1795-1822: no mutable layer -> compressed; len(Intersect) < ApproxLen -> probe; else iterate */
    const int mode = nmut == 0 ? 0 : (X->n < c->approx[leaf] ? 1 : 2);
    tg_list r = tg_alloc(X->n);
    r.n = orc_list_uids(p, mode, c->mu + m0, c->mf + m0, nmut, c->after_uid, X->u, X->n, r.u);
    return r;
}

static tg_list merge2(tg_list* a, tg_list* b) { /* algo.MergeSorted([]*pb.List{a, b}) */
    const uint64_t* ls[2] = {a->u, b->u};
    size_t lens[2] = {a->n, b->n};
    tg_list r = tg_alloc(a->n + b->n);
    r.n = orc_merge_sorted(ls, lens, 2, r.u);
    free(a->u);
    free(b->u);
    return r;
}

static tg_list uids_for_regex(tg_ctx* c, uint32_t q, const tg_list* intersect) {
    tg_list results = {NULL, 0, 1}; /* var results *pb.List */
    const tg_list* X = intersect->n > 0 ? intersect : NULL; /* :32-34 proto.Size(intersect) > 0 */
    switch (c->op[q]) {
    case ORC_QAND:
        for (uint32_t k = c->leaf_off[q]; k < c->leaf_off[q + 1]; k++) { /* :46-61 */
            tg_list t = uids_for_trigram(c, c->leaf_idx[k], X);
            if (results.nil) results = t;
            else {
                results.n = orc_intersect_with(results.u, results.n, t.u, t.n, results.u);
                free(t.u);
            }
            if (results.n == 0) return results;
        }
        for (uint32_t k = c->sub_off[q]; k < c->sub_off[q + 1]; k++) { /* :62-75 */
            if (results.nil) results = tg_copy(intersect);
            tg_list r = uids_for_regex(c, c->sub_idx[k], &results);
            free(results.u);
            results = r;
            if (results.n == 0) return results;
        }
        break;
    case ORC_QOR: { /* :76-96 */
        const size_t nt = c->leaf_off[q + 1] - c->leaf_off[q];
        tg_list* matrix = (tg_list*)malloc((nt + 1) * sizeof(tg_list));
        const uint64_t** ls = (const uint64_t**)malloc((nt + 1) * sizeof(uint64_t*));
        size_t* lens = (size_t*)malloc((nt + 1) * sizeof(size_t));
        size_t total = 0;
        for (size_t i = 0; i < nt; i++) {
            matrix[i] = uids_for_trigram(c, c->leaf_idx[c->leaf_off[q] + i], X);
            ls[i] = matrix[i].u;
            lens[i] = matrix[i].n;
            total += matrix[i].n;
        }
        results = tg_alloc(total);
        results.n = orc_merge_sorted(ls, lens, nt, results.u);
        for (size_t i = 0; i < nt; i++) free(matrix[i].u);
        free(matrix);
        free(ls);
        free(lens);
        for (uint32_t k = c->sub_off[q]; k < c->sub_off[q + 1]; k++) {
            if (results.nil) results = tg_copy(intersect);
            tg_list s = uids_for_regex(c, c->sub_idx[k], intersect);
            results = merge2(&results, &s);
        }
        break;
    }
    default:
        c->err = 1; /* errRegexTooWide */
    }
    return results;
}

size_t orc_uids_for_regex(const uint8_t* op, const uint32_t* leaf_off, const uint32_t* leaf_idx, const uint32_t* sub_off,
                          const uint32_t* sub_idx, const orc_pack* const* packs, const uint64_t* mu, const uint8_t* mf,
                          const uint64_t* mut_off, const uint64_t* approx, size_t npacks, const uint64_t* lists,
                          const uint64_t* list_off, size_t nlists, uint64_t after_uid, uint64_t* out) {
    (void)nlists;
    tg_ctx c = {op, leaf_off, leaf_idx, sub_off, sub_idx, packs, mu, mf, mut_off, approx, npacks, lists, list_off,
                after_uid, 0};
    uint64_t none = 0;
    tg_list empty = {&none, 0, 0}; /* &pb.List{} */
    tg_list r = uids_for_regex(&c, 0, &empty);
    if (c.err) {
        free(r.u);
        return (size_t)-1;
    }
    if (r.n) memcpy(out, r.u, r.n * sizeof(uint64_t));
    free(r.u);
    return r.n;
}
