/*
 * match_oracle.c -- handleMatchFunction (worker/task.go:1526-1620) with uidsForMatch, matchFuzzy and
 * levenshteinDistance (worker/match.go:24-100) restated line by line.  TEST INFRASTRUCTURE ONLY: the checker of
 * dgx_match / dgx_dev_match in tests/ and smoke(), and the CPU legs of tools/bench_ops.py C21.  It includes
 * list_uids_unfiltered_oracle.c, so that every trigram read is the same List.Uids restatement the trigram query is
 * checked against; match_oracle.py compiles it together with oracle/oracle.c into a temporary directory.
 *
 * orc_match(packs, mu, mf, mut_off, npacks, lists, list_off, nlists, after_uid, uids, nuids, col..., query, qlen, max,
 * out): the candidates are uids when nuids > 0 (arg.q.UidList), otherwise uidsForMatch: every trigram row read with
 * pl.Uids(ListOptions{First: MaxInt32, AfterUid}) -- leaves 0 .. npacks-1 unsplit posting lists with their resolved REF
 * layer, leaves npacks .. lists a caller already read -- and algo.MergeSorted of them.  For every candidate in order
 * its values are looked up in the column (absent: ErrNoValue, skipped), and the uid is kept when matchFuzzy(query,
 * val, max) holds for any of them.  out must hold the candidates' count.  Returns the kept count.
 * orc_levenshtein(s, slen, t, tlen): levenshteinDistance(s, t).
 */
#include "list_uids_unfiltered_oracle.c"

size_t orc_match(const orc_pack* const* packs, const uint64_t* mu, const uint8_t* mf, const uint64_t* mut_off,
                 size_t npacks, const uint64_t* lists, const uint64_t* list_off, size_t nlists, uint64_t after_uid,
                 const uint64_t* uids, size_t nuids, const uint64_t* col_uid, const uint64_t* val_off,
                 const uint64_t* byte_off, const uint8_t* bytes, size_t ncol, const uint8_t* query, size_t qlen,
                 int64_t max, uint64_t* out);
int64_t orc_levenshtein(const uint8_t* s, size_t slen, const uint8_t* t, size_t tlen);

#define RUNE_ERROR 0xFFFDu

/* utf8.DecodeRuneInString (unicode/utf8/utf8.go): the first / accept tables written out per lead byte. */
static uint32_t decode_rune(const uint8_t* p, size_t n, uint32_t* width) {
    const uint8_t s0 = p[0];
    *width = 1;
    if (s0 < 0x80) return s0;             /* as: ASCII */
    if (s0 < 0xC2 || s0 > 0xF4) return RUNE_ERROR; /* xx: invalid lead byte */
    size_t sz;
    uint8_t lo = 0x80, hi = 0xBF;         /* locb, hicb */
    if (s0 < 0xE0) sz = 2;
    else if (s0 < 0xF0) {
        sz = 3;
        if (s0 == 0xE0) lo = 0xA0;        /* s2: accept range 1 */
        if (s0 == 0xED) hi = 0x9F;        /* s3: accept range 2 */
    } else {
        sz = 4;
        if (s0 == 0xF0) lo = 0x90;        /* s5: accept range 3 */
        if (s0 == 0xF4) hi = 0x8F;        /* s7: accept range 4 */
    }
    if (n < sz) return RUNE_ERROR;
    const uint8_t s1 = p[1];
    if (s1 < lo || hi < s1) return RUNE_ERROR;
    if (sz <= 2) { *width = 2; return (uint32_t)(s0 & 0x1F) << 6 | (uint32_t)(s1 & 0x3F); }
    const uint8_t s2 = p[2];
    if (s2 < 0x80 || 0xBF < s2) return RUNE_ERROR;
    if (sz <= 3) { *width = 3; return (uint32_t)(s0 & 0x0F) << 12 | (uint32_t)(s1 & 0x3F) << 6 | (uint32_t)(s2 & 0x3F); }
    const uint8_t s3 = p[3];
    if (s3 < 0x80 || 0xBF < s3) return RUNE_ERROR;
    *width = 4;
    return (uint32_t)(s0 & 0x07) << 18 | (uint32_t)(s1 & 0x3F) << 12 | (uint32_t)(s2 & 0x3F) << 6 | (uint32_t)(s3 & 0x3F);
}

/* []rune(s): the runes of a range loop over s. */
static uint32_t* to_runes(const uint8_t* s, size_t n, size_t* len) {
    uint32_t* r = (uint32_t*)malloc((n + 1) * sizeof(uint32_t));
    size_t k = 0;
    for (size_t i = 0; i < n;) {
        uint32_t w;
        r[k++] = decode_rune(s + i, n - i, &w);
        i += w;
    }
    *len = k;
    return r;
}

static int64_t min3(int64_t a, int64_t b, int64_t c) { /* min(a, b, c) */
    if (a < b && a < c) return a;
    if (b < c) return b;
    return c;
}

int64_t orc_levenshtein(const uint8_t* s, size_t slen, const uint8_t* t, size_t tlen) {
    if (slen > tlen) { /* if len(s) > len(t) { s, t = t, s } */
        const uint8_t* x = s; s = t; t = x;
        size_t y = slen; slen = tlen; tlen = y;
    }
    size_t n1, n2;
    uint32_t* r1 = to_runes(s, slen, &n1);
    uint32_t* r2 = to_runes(t, tlen, &n2);
    int64_t* column = (int64_t*)calloc(n1 + 1, sizeof(int64_t));
    for (size_t y = 1; y <= n1; y++) column[y] = (int64_t)y;
    for (size_t x = 1; x <= n2; x++) {
        column[0] = (int64_t)x;
        int64_t lastDiag = (int64_t)x - 1;
        for (size_t y = 1; y <= n1; y++) {
            const int64_t oldDiag = column[y];
            int64_t cost = 0;
            if (r1[y - 1] != r2[x - 1]) cost = 1;
            column[y] = min3(column[y] + 1, column[y - 1] + 1, lastDiag + cost);
            lastDiag = oldDiag;
        }
    }
    const int64_t d = column[n1];
    free(r1);
    free(r2);
    free(column);
    return d;
}

/* matchFuzzy(query, val, max) */
static int match_fuzzy(const uint8_t* query, size_t qlen, const uint8_t* val, size_t vlen, int64_t max) {
    if (vlen == 0) return 0;
    return orc_levenshtein(val, vlen, query, qlen) <= max;
}

size_t orc_match(const orc_pack* const* packs, const uint64_t* mu, const uint8_t* mf, const uint64_t* mut_off,
                 size_t npacks, const uint64_t* lists, const uint64_t* list_off, size_t nlists, uint64_t after_uid,
                 const uint64_t* uids_in, size_t nuids, const uint64_t* col_uid, const uint64_t* val_off,
                 const uint64_t* byte_off, const uint8_t* bytes, size_t ncol, const uint8_t* query, size_t qlen,
                 int64_t max, uint64_t* out) {
    const uint64_t* uids = uids_in;
    size_t n = nuids;
    uint64_t* merged = NULL;
    if (nuids == 0) { /* uidsForMatch */
        const size_t k = npacks + nlists;
        const uint64_t** ls = (const uint64_t**)malloc((k + 1) * sizeof(uint64_t*));
        size_t* lens = (size_t*)malloc((k + 1) * sizeof(size_t));
        uint64_t** rows = (uint64_t**)malloc((k + 1) * sizeof(uint64_t*));
        size_t total = 0;
        for (size_t i = 0; i < npacks; i++) { /* uidsForNgram: pl.Uids(opts) */
            const size_t m0 = (size_t)mut_off[i], nmut = (size_t)(mut_off[i + 1] - m0);
            rows[i] = (uint64_t*)malloc((orc_exact_len(packs[i]) + nmut + 1) * sizeof(uint64_t));
            lens[i] = orc_list_uids_unfiltered(packs[i], mu + m0, mf + m0, nmut, after_uid, 0x7fffffff, rows[i]);
            ls[i] = rows[i];
            total += lens[i];
        }
        for (size_t j = 0; j < nlists; j++) {
            rows[npacks + j] = NULL;
            ls[npacks + j] = lists + list_off[j];
            lens[npacks + j] = (size_t)(list_off[j + 1] - list_off[j]);
            total += lens[npacks + j];
        }
        merged = (uint64_t*)malloc((total + 1) * sizeof(uint64_t));
        n = orc_merge_sorted(ls, lens, k, merged); /* algo.MergeSorted(uidMatrix) */
        for (size_t i = 0; i < k; i++) free(rows[i]);
        free(rows);
        free(ls);
        free(lens);
        uids = merged;
    }
    size_t kept = 0;
    for (size_t u = 0; u < n; u++) {
        const uint64_t uid = uids[u];
        size_t lo = 0, hi = ncol; /* qs.cache.Get(x.DataKey(attr, uid)) */
        while (lo < hi) {
            const size_t mid = lo + (hi - lo) / 2;
            if (col_uid[mid] < uid) lo = mid + 1; else hi = mid;
        }
        if (lo == ncol || col_uid[lo] != uid) continue; /* ErrNoValue */
        for (uint64_t j = val_off[lo]; j < val_off[lo + 1]; j++) {
            if (match_fuzzy(query, qlen, bytes + byte_off[j], (size_t)(byte_off[j + 1] - byte_off[j]), max)) {
                out[kept++] = uid;
                break; /* We only add the uid once. */
            }
        }
    }
    free(merged);
    return kept; /* IntersectWith(UidMatrix[0], filtered): filtered is a subsequence of the candidates */
}
