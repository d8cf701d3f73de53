/*
 * list_uids_unfiltered_oracle.c -- posting.List.Uids with opts.Intersect == nil and the count of List.Postings, for one
 * unsplit list, restated line by line.  TEST INFRASTRUCTURE ONLY: the checker of dgx_list_uids_unfiltered_rows and
 * dgx_list_count_rows in tests/ and smoke(), and the CPU legs of tools/bench_ops.py C10.  It includes
 * list_uids_oracle.c, so that the pIterator and mutable-layer restatement is the same code as for List.Uids with a
 * filter; list_uids_unfiltered_oracle.py compiles it together with oracle/oracle.c into a temporary directory.
 *
 * orc_list_uids_unfiltered(p, mut_uids, mut_flags, nmut, after_uid, first, out): List.Uids(opts) with
 * opts.Intersect == nil (posting/list.go:1758-1874): iterate with the REF filter and no bounds (:1822-1852), then the
 * First cut (:1864-1872); first is opts.First as the int32 the worker receives.  out must hold orc_exact_len(p) + nmut
 * values.  orc_list_count(p, mut_uids, mut_flags, nmut, after_uid): the REF postings List.Postings (:1878-1890) passes
 * to countForUidPostings with a nil facets tree (worker/task.go:743-755).  p and the resolved layer are as for
 * orc_list_uids.
 */
#include "list_uids_oracle.c"

size_t orc_list_uids_unfiltered(const orc_pack* p, const uint64_t* mu, const uint8_t* mf, size_t nmut,
                                uint64_t after_uid, int32_t first, uint64_t* out);
size_t orc_list_count(const orc_pack* p, const uint64_t* mu, const uint8_t* mf, size_t nmut, uint64_t after_uid);

/* iterate (:1116-1232) over the resolved layer: fn(ctx, posting) for every posting it yields, uid ascending, until fn
 * returns 1 (ErrStopIteration).  A posting is (uid, is_ref): pack uids are REF postings (pIterator.posting, :688-704). */
typedef int (*orc_posting_fn)(void* ctx, uint64_t uid, int is_ref);
static void iterate(const orc_pack* p, const uint64_t* mu, const uint8_t* mf, size_t nmut, uint64_t after_uid,
                    orc_posting_fn fn, void* ctx) {
    size_t midx = 0;
    if (after_uid > 0) midx = search_gt(mu, nmut, after_uid); /* :1126-1131 */
    orc_pitr it = {0};
    pitr_seek(&it, p, after_uid);
    uint64_t prev_uid = 0;
    for (;;) {
        uint64_t mp = midx < nmut ? mu[midx] : 0; /* emptyPosting: Uid 0 */
        uint8_t mflag = midx < nmut ? mf[midx] : 0;
        uint64_t pp = pitr_valid(&it) ? it.uids[it.uidx] : 0;
        if (mp > 0 && mp == prev_uid) {
            midx++;
        } else if (pp == 0 && mp == 0) {
            break;
        } else if (mp == 0 || (pp > 0 && pp < mp)) {
            if (fn(ctx, pp, 1)) break;
            pitr_next(&it);
        } else if (pp == 0 || (mp > 0 && mp < pp)) {
            if (!(mflag & ORC_MUT_DEL) && fn(ctx, mp, !(mflag & ORC_MUT_VALUE))) break;
            prev_uid = mp;
            midx++;
        } else { /* pp == mp */
            if (!(mflag & ORC_MUT_DEL) && fn(ctx, mp, !(mflag & ORC_MUT_VALUE))) break;
            prev_uid = mp;
            pitr_next(&it);
            midx++;
        }
    }
    if (it.dec) orc_decoder_free(it.dec);
}

/* the callback of :1830-1845 with uidMin = uidMax = 0 */
typedef struct {
    uint64_t* res;
    size_t n;
    int64_t first;
} orc_uids_ctx;
static int uids_fn(void* c, uint64_t uid, int is_ref) {
    orc_uids_ctx* x = (orc_uids_ctx*)c;
    if (!is_ref) return 0;
    x->res[x->n++] = uid;
    return x->first != 0 && (int64_t)x->n > x->first;
}

size_t orc_list_uids_unfiltered(const orc_pack* p, const uint64_t* mu, const uint8_t* mf, size_t nmut,
                                uint64_t after_uid, int32_t first, uint64_t* out) {
    int64_t f = first == 0 ? 0x7fffffff : first; /* :1759-1761 (opt.First is a Go int) */
    orc_uids_ctx x = {out, 0, f};
    iterate(p, mu, mf, nmut, after_uid, uids_fn, &x);
    /* :1864-1872: Intersect is nil, so no IntersectWith */
    if (f < 0) {
        if ((int64_t)x.n > -f) {
            size_t from = (size_t)((int64_t)x.n + f);
            memmove(out, out + from, (x.n - from) * sizeof(uint64_t));
            x.n -= from;
        }
    } else if ((int64_t)x.n > f) {
        x.n = (size_t)f;
    }
    return x.n;
}

static int count_fn(void* c, uint64_t uid, int is_ref) {
    (void)uid;
    if (is_ref) ++*(size_t*)c; /* Postings passes REF postings only (:1884-1886) */
    return 0;
}

size_t orc_list_count(const orc_pack* p, const uint64_t* mu, const uint8_t* mf, size_t nmut, uint64_t after_uid) {
    size_t n = 0;
    iterate(p, mu, mf, nmut, after_uid, count_fn, &n);
    return n;
}
