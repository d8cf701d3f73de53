/*
 * list_uids_oracle.c -- posting.List.Uids (posting/list.go:1758-1874) of one unsplit list, restated line by line on
 * top of the CPU oracle's codec and algo functions (oracle/oracle.h).  TEST INFRASTRUCTURE ONLY: it is the checker of
 * dgx_list_uids_rows in tests/ and the CPU legs of tools/bench_ops.py C9; list_uids_oracle.py compiles it together
 * with oracle/oracle.c into a temporary directory.
 *
 * orc_list_uids(p, mode, mut_uids, mut_flags, nmut, after_uid, v, m, out): List.Uids(opts) with opts.Intersect = v
 * (m > 0) and opts.First 0 or MaxInt32, branch `mode`:
 *   0 IntersectCompressedWith (:1795-1800), 1 findPostingWithItr per uid of v (:1805-1820),
 *   2 iterate with the REF filter (:1822-1852) then IntersectWith and the First cut (:1860-1872).
 * The mutable layer is passed resolved: mut_uids strictly ascending and nonzero, one entry per uid -- the posting
 * List.Uids sees for that uid -- with flags ORC_MUT_DEL (Op == Del) and ORC_MUT_VALUE (PostingType != REF).
 * p == NULL with mode 1 / 2 is a list whose delete-all marker hides the immutable layer.
 * out must hold m values.  Returns the result length.
 */
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

enum { ORC_MUT_DEL = 1, ORC_MUT_VALUE = 2 };

size_t orc_list_uids(const orc_pack* p, int mode, const uint64_t* mu, const uint8_t* mf, size_t nmut,
                     uint64_t after_uid, const uint64_t* v, size_t m, uint64_t* out);

/* sort.Search for the first a[i] >= val / > val */
static size_t search_ge(const uint64_t* a, size_t n, uint64_t val) {
    size_t lo = 0, hi = n;
    while (lo < hi) {
        size_t h = lo + (hi - lo) / 2;
        if (a[h] < val) lo = h + 1; else hi = h;
    }
    return lo;
}
static size_t search_gt(const uint64_t* a, size_t n, uint64_t val) {
    size_t lo = 0, hi = n;
    while (lo < hi) {
        size_t h = lo + (hi - lo) / 2;
        if (a[h] <= val) lo = h + 1; else hi = h;
    }
    return lo;
}


/* MutableLayer.findPosting (:418-490) over the resolved layer: *searchFurther = 0 when the entry decides (or the
 * delete-all marker hides the immutable layer); returns 1 with a non-deleted posting found. */
static int mut_find(const orc_pack* p, const uint64_t* mu, const uint8_t* mf, size_t nmut, uint64_t uid,
                    int* search_further) {
    size_t i = search_ge(mu, nmut, uid);
    if (i < nmut && mu[i] == uid) {
        *search_further = 0;
        return !(mf[i] & ORC_MUT_DEL); /* :476-480 */
    }
    *search_further = p != NULL; /* :484-486: deleteAllMarker > 0 */
    return 0;
}

/* pIterator (:520-704) of an unsplit list: the decoder's current slice and the position in it */
typedef struct {
    orc_decoder* dec;
    const uint64_t* uids;
    size_t len, uidx;
    int delete_all;
} orc_pitr;

static void pitr_seek(orc_pitr* it, const orc_pack* p, uint64_t after_uid) { /* :530-578 */
    it->delete_all = p == NULL;
    it->len = it->uidx = 0;
    it->uids = NULL;
    if (it->delete_all) return; /* :561-565 */
    it->dec = orc_decoder_new(p);
    it->uids = orc_decoder_seek(it->dec, after_uid, ORC_SEEK_CURRENT, &it->len); /* :569 */
}
static int pitr_valid(const orc_pitr* it) { return !it->delete_all && it->len > 0; } /* :667-686 */
static void pitr_next(orc_pitr* it) {                                                  /* :648-663 */
    if (it->delete_all) { it->len = 0; return; }
    it->uidx++;
    if (it->uidx < it->len) return;
    it->uidx = 0;
    it->uids = orc_decoder_next(it->dec, &it->len);
}

/* findPostingWithItr (:2167-2199).  pitr is passed by value there, so every call seeks a fresh iterator. */
static int find_posting_with_itr(const orc_pack* p, orc_decoder* dec, const uint64_t* mu, const uint8_t* mf,
                                 size_t nmut, uint64_t uid) {
    int further = 0;
    if (mut_find(p, mu, mf, nmut, uid, &further)) return 1;
    if (!further) return 0;
    size_t len = 0;
    const uint64_t* uids = orc_decoder_seek(dec, uid - 1, ORC_SEEK_CURRENT, &len); /* pitr.seek(l, uid-1, 0) */
    return len > 0 && uids[0] == uid;
}

size_t orc_list_uids(const orc_pack* p, int mode, const uint64_t* mu, const uint8_t* mf, size_t nmut,
                     uint64_t after_uid, const uint64_t* v, size_t m, uint64_t* out) {
    if (mode == 0) return orc_intersect_compressed_with(p, after_uid, v, m, out); /* :1795-1800 */
    const uint64_t first = 0x7fffffff; /* opt.First 0 -> math.MaxInt32 (:1759-1761) */
    if (mode == 1) {                   /* :1805-1820 */
        orc_decoder* dec = orc_decoder_new(p);
        size_t n = 0;
        for (size_t k = 0; k < m; k++)
            if (find_posting_with_itr(p, dec, mu, mf, nmut, v[k])) out[n++] = v[k];
        orc_decoder_free(dec);
        return n;
    }
    /* :1824-1828 */
    uint64_t uid_min = m ? v[0] : 0, uid_max = m ? v[m - 1] : 0;
    /* iterate (:1116-1232) */
    size_t midx = 0;
    if (after_uid > 0) midx = search_gt(mu, nmut, after_uid); /* :1126-1131 */
    orc_pitr it = {0};
    pitr_seek(&it, p, after_uid);
    size_t cap = orc_exact_len(p) + nmut + 1, n = 0;
    uint64_t* res = (uint64_t*)malloc(cap * sizeof(uint64_t));
    uint64_t prev_uid = 0;
    int stop = 0;
    /* f of :1830-1845 for a posting of uid u: 1 = ErrStopIteration */
#define ORC_EMIT(u, is_ref)                                                           \
    do {                                                                              \
        if (is_ref) {                                                                 \
            if ((u) < uid_min) break;                                                 \
            if ((u) > uid_max && uid_max > 0) { stop = 1; break; }                    \
            res[n++] = (u);                                                           \
            if (n > first) { stop = 1; break; }                                       \
        }                                                                             \
    } while (0)
    while (!stop) {
        uint64_t mp = midx < nmut ? mu[midx] : 0; /* emptyPosting: Uid 0 */
        uint8_t mflag = midx < nmut ? mf[midx] : 0;
        uint64_t pp = pitr_valid(&it) ? it.uids[it.uidx] : 0;
        if (mp > 0 && mp == prev_uid) {
            midx++;
        } else if (pp == 0 && mp == 0) {
            break;
        } else if (mp == 0 || (pp > 0 && pp < mp)) {
            ORC_EMIT(pp, 1); /* pIterator.posting: a REF uid posting (:688-704) */
            if (stop) break;
            pitr_next(&it);
        } else if (pp == 0 || (mp > 0 && mp < pp)) {
            if (!(mflag & ORC_MUT_DEL)) ORC_EMIT(mp, !(mflag & ORC_MUT_VALUE));
            if (stop) break;
            prev_uid = mp;
            midx++;
        } else { /* pp == mp */
            if (!(mflag & ORC_MUT_DEL)) ORC_EMIT(mp, !(mflag & ORC_MUT_VALUE));
            if (stop) break;
            prev_uid = mp;
            pitr_next(&it);
            midx++;
        }
    }
#undef ORC_EMIT
    if (it.dec) orc_decoder_free(it.dec);
    /* :1860-1872: IntersectWith(out, v, out), then the First cut */
    n = orc_intersect_with(res, n, v, m, res);
    if (n > first) n = first;
    memcpy(out, res, n * sizeof(uint64_t));
    free(res);
    return n;
}
