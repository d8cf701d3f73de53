/*
 * pred_order_oracle.c -- a uid matrix ordered by a predicate without its index, restated line by line from the
 * reference:
 *   applyOrderAndPagination (query/query.go :2511-2592), predicate branch: updateUidMatrix (:1425-1439) with an order
 *     keeps, in row order, the row uids IndexOf(DestUIDs, uid) >= 0 finds (U); processSort's sortWithoutIndex result
 *     replaces the matrix; updateDestUids (:2594-2609) keeps the DestUIDs some row still holds;
 *   processSort (worker/sort.go :494-564): a negative count is an error; a list predicate is an error;
 *   sortWithoutIndex (:139-187): per row sortByValue, then paginate and the row cut to [start, end);
 *   sortByValue (:775-822): fetchValue per uid in row order; an error (no value, a failed conversion) sends the uid to
 *     nullsList, otherwise to (uids, values); types.Sort(values, &uids, []bool{desc}, ""); the row becomes uids ++
 *     nullsList;
 *   paginate (:740-773) with one order key: x.PageRange(count, offset, len(row)) (x/x.go :738-767);
 *   types.Sort -> SortWithFacet (types/sort.go :142-166), sort.Sort(byValue) with byValue.Less (:49-82), less
 *     (:188-214) and equal (:249-): int64 <, float64 < and ==, datetime Before / Equal, string bytes.Compare;
 *   sort.Sort: Go's pdqsort, the same driver var_order_oracle.c restates.
 * The column is dgx_val_column's: uid[n] ascending, val_off[n + 1], per value a word (int64, float64 bits, datetime
 * seconds), nsec (datetime) or bytes[byte_off[j] .. byte_off[j + 1]) (string), and an optional bad byte (the value's
 * conversion failed: fetchValue's error).  TEST INFRASTRUCTURE ONLY.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { T_INT = 1, T_FLOAT = 2, T_BOOL = 3, T_TIME = 5, T_STR = 6 };

typedef struct {
    uint64_t w; /* int64, float64 bits, datetime seconds; string: first byte offset */
    uint64_t x; /* datetime nanoseconds; string: end byte offset */
} Val;

static double f64(uint64_t w) {
    double d;
    memcpy(&d, &w, 8);
    return d;
}

typedef struct {
    uint64_t insertion, heap, partition, partition_equal, partial_insertion, partial_insertion_ok, break_patterns,
        reverse;
} OrcPoStats;
static __thread OrcPoStats g_pst;

void orc_pred_order_stats(OrcPoStats* s, int reset) {
    if (s) *s = g_pst;
    if (reset) memset(&g_pst, 0, sizeof g_pst);
}

typedef struct {
    Val* v;
    uint64_t* u;
    int desc;
    int type;
    const uint8_t* bytes;
} Data;

/* bytes.Compare */
static int bytes_compare(const uint8_t* a, uint64_t la, const uint8_t* b, uint64_t lb) {
    const uint64_t m = la < lb ? la : lb;
    for (uint64_t i = 0; i < m; i++)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return la < lb ? -1 : la > lb ? 1 : 0;
}

/* types.less for one type (string without a collator) */
static int less(const Data* d, Val a, Val b) {
    switch (d->type) {
        case T_INT: return (int64_t)a.w < (int64_t)b.w;
        case T_FLOAT: return f64(a.w) < f64(b.w);
        case T_TIME: return (int64_t)a.w < (int64_t)b.w || ((int64_t)a.w == (int64_t)b.w && a.x < b.x); /* Before */
    }
    return bytes_compare(d->bytes + a.w, a.x - a.w, d->bytes + b.w, b.x - b.w) < 0;
}

/* types.equal */
static int equal(const Data* d, Val a, Val b) {
    switch (d->type) {
        case T_INT: return (int64_t)a.w == (int64_t)b.w;
        case T_FLOAT: return f64(a.w) == f64(b.w);
        case T_TIME: return a.w == b.w && a.x == b.x; /* Equal */
    }
    return bytes_compare(d->bytes + a.w, a.x - a.w, d->bytes + b.w, b.x - b.w) == 0;
}

/* byValue.Less with one value per uid, none of them nil */
static int Less(const Data* d, long i, long j) {
    const Val a = d->v[i], b = d->v[j];
    if (equal(d, a, b)) return 0;
    const int l = less(d, a, b);
    return d->desc ? !l : l;
}

static void Swap(const Data* d, long i, long j) {
    const Val t = d->v[i];
    d->v[i] = d->v[j];
    d->v[j] = t;
    const uint64_t x = d->u[i];
    d->u[i] = d->u[j];
    d->u[j] = x;
}

/* ---- sort/zsortinterface.go ---- */
static int bits_len(uint64_t x) { return x ? 64 - __builtin_clzll(x) : 0; }

static void insertion_sort(const Data* d, long a, long b) {
    g_pst.insertion++;
    for (long i = a + 1; i < b; i++)
        for (long j = i; j > a && Less(d, j, j - 1); j--) Swap(d, j, j - 1);
}

static void sift_down(const Data* d, long lo, long hi, long first) {
    long root = lo;
    for (;;) {
        long child = 2 * root + 1;
        if (child >= hi) return;
        if (child + 1 < hi && Less(d, first + child, first + child + 1)) child++;
        if (!Less(d, first + root, first + child)) return;
        Swap(d, first + root, first + child);
        root = child;
    }
}

static void heap_sort(const Data* d, long a, long b) {
    g_pst.heap++;
    const long first = a, lo = 0, hi = b - a;
    for (long i = (hi - 1) / 2; i >= 0; i--) sift_down(d, i, hi, first);
    for (long i = hi - 1; i >= 0; i--) {
        Swap(d, first, first + i);
        sift_down(d, lo, i, first);
    }
}

enum { UNKNOWN_HINT = 0, INCREASING_HINT = 1, DECREASING_HINT = 2 };

static long partition(const Data* d, long a, long b, long pivot, int* already) {
    g_pst.partition++;
    Swap(d, a, pivot);
    long i = a + 1, j = b - 1;
    while (i <= j && Less(d, i, a)) i++;
    while (i <= j && !Less(d, j, a)) j--;
    if (i > j) {
        Swap(d, j, a);
        *already = 1;
        return j;
    }
    Swap(d, i, j);
    i++;
    j--;
    for (;;) {
        while (i <= j && Less(d, i, a)) i++;
        while (i <= j && !Less(d, j, a)) j--;
        if (i > j) break;
        Swap(d, i, j);
        i++;
        j--;
    }
    Swap(d, j, a);
    *already = 0;
    return j;
}

static long partition_equal(const Data* d, long a, long b, long pivot) {
    g_pst.partition_equal++;
    Swap(d, a, pivot);
    long i = a + 1, j = b - 1;
    for (;;) {
        while (i <= j && !Less(d, a, i)) i++;
        while (i <= j && Less(d, a, j)) j--;
        if (i > j) break;
        Swap(d, i, j);
        i++;
        j--;
    }
    return i;
}

static int partial_insertion_sort(const Data* d, long a, long b) {
    g_pst.partial_insertion++;
    const int max_steps = 5;
    const long shortest_shifting = 50;
    long i = a + 1;
    for (int j = 0; j < max_steps; j++) {
        while (i < b && !Less(d, i, i - 1)) i++;
        if (i == b) {
            g_pst.partial_insertion_ok++;
            return 1;
        }
        if (b - a < shortest_shifting) return 0;
        Swap(d, i, i - 1);
        if (i - a >= 2) {
            for (long k = i - 1; k >= 1; k--) { /* Go's bound: k >= 1, not k > a */
                if (!Less(d, k, k - 1)) break;
                Swap(d, k, k - 1);
            }
        }
        if (b - i >= 2) {
            for (long k = i + 1; k < b; k++) {
                if (!Less(d, k, k - 1)) break;
                Swap(d, k, k - 1);
            }
        }
    }
    return 0;
}

static void break_patterns(const Data* d, long a, long b) {
    const long length = b - a;
    if (length >= 8) {
        g_pst.break_patterns++;
        uint64_t random = (uint64_t)length; /* xorshift seeded by the length */
        const uint64_t modulus = (uint64_t)1 << bits_len((uint64_t)length); /* nextPowerOfTwo */
        const long idx = a + (length / 4) * 2 - 1;
        for (int i = 0; i < 3; i++) {
            random ^= random << 13;
            random ^= random >> 7;
            random ^= random << 17;
            long other = (long)(random & (modulus - 1));
            if (other >= length) other -= length;
            Swap(d, idx - 1 + i, a + other);
        }
    }
}

static void order2(const Data* d, long a, long b, int* swaps, long* x, long* y) {
    if (Less(d, b, a)) {
        (*swaps)++;
        *x = b;
        *y = a;
        return;
    }
    *x = a;
    *y = b;
}

static long median(const Data* d, long a, long b, long c, int* swaps) {
    order2(d, a, b, swaps, &a, &b);
    order2(d, b, c, swaps, &b, &c);
    order2(d, a, b, swaps, &a, &b);
    return b;
}

static long median_adjacent(const Data* d, long a, int* swaps) { return median(d, a - 1, a, a + 1, swaps); }

static long choose_pivot(const Data* d, long a, long b, int* hint) {
    const long shortest_ninther = 50;
    const int max_swaps = 4 * 3;
    const long l = b - a;
    int swaps = 0;
    long i = a + l / 4 * 1, j = a + l / 4 * 2, k = a + l / 4 * 3;
    if (l >= 8) {
        if (l >= shortest_ninther) {
            i = median_adjacent(d, i, &swaps);
            j = median_adjacent(d, j, &swaps);
            k = median_adjacent(d, k, &swaps);
        }
        j = median(d, i, j, k, &swaps);
    }
    *hint = swaps == 0 ? INCREASING_HINT : swaps == max_swaps ? DECREASING_HINT : UNKNOWN_HINT;
    return j;
}

static void reverse_range(const Data* d, long a, long b) {
    g_pst.reverse++;
    long i = a, j = b - 1;
    while (i < j) {
        Swap(d, i, j);
        i++;
        j--;
    }
}

static void pdqsort(const Data* d, long a, long b, int limit) {
    const long max_insertion = 12;
    int was_balanced = 1, was_partitioned = 1;
    for (;;) {
        const long length = b - a;
        if (length <= max_insertion) {
            insertion_sort(d, a, b);
            return;
        }
        if (limit == 0) {
            heap_sort(d, a, b);
            return;
        }
        if (!was_balanced) {
            break_patterns(d, a, b);
            limit--;
        }
        int hint;
        long pivot = choose_pivot(d, a, b, &hint);
        if (hint == DECREASING_HINT) {
            reverse_range(d, a, b);
            pivot = (b - 1) - (pivot - a);
            hint = INCREASING_HINT;
        }
        if (was_balanced && was_partitioned && hint == INCREASING_HINT) {
            if (partial_insertion_sort(d, a, b)) return;
        }
        if (a > 0 && !Less(d, a - 1, pivot)) {
            const long mid = partition_equal(d, a, b, pivot);
            a = mid;
            continue;
        }
        int already;
        const long mid = partition(d, a, b, pivot, &already);
        was_partitioned = already;
        const long left_len = mid - a, right_len = b - mid;
        const long balance_threshold = length / 8;
        if (left_len < right_len) {
            was_balanced = left_len >= balance_threshold;
            pdqsort(d, a, mid, limit);
            a = mid + 1;
        } else {
            was_balanced = right_len >= balance_threshold;
            pdqsort(d, mid + 1, b, limit);
            b = mid;
        }
    }
}

/* sort.Sort */
static void go_sort(const Data* d, long n) {
    if (n <= 1) return;
    pdqsort(d, 0, n, bits_len((uint64_t)n));
}

/* x.PageRange */
static void page_range(long long count, long long offset, long long n, long long* s, long long* e) {
    if (n == 0) { *s = 0; *e = 0; return; }
    if (count == 0 && offset == 0) { *s = 0; *e = n; return; }
    if (count < 0) {
        if (-count > n) count = -n;
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

/* algo.IndexOf: binary search of a strictly ascending list */
static long index_of(const uint64_t* a, size_t n, uint64_t x) {
    size_t lo = 0, hi = n;
    while (lo < hi) {
        const size_t mid = lo + (hi - lo) / 2;
        if (a[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && a[lo] == x ? (long)lo : -1;
}

/* The whole node: the column (type, uid[n], val_off[n + 1], word / nsec / byte_off + bytes, bad or NULL), the node's
 * DestUIDs dest[ndest] and rows v[v_off[i] .. v_off[i+1]).  Writes the rows to out / out_off and the new DestUIDs to
 * dest_out / *dest_len.  Returns 0, 1 (a bool column: SortWithFacet's "isn't sortable"), 2 (a negative count), 3 (a
 * row uid with several values: a list predicate) or -1 (allocation). */
int orc_pred_order(int type, const uint64_t* uid, const uint64_t* val_off, size_t n, const uint64_t* word,
                   const uint32_t* nsec, const uint64_t* byte_off, const uint8_t* bytes, const uint8_t* bad, int desc,
                   const uint64_t* dest, size_t ndest, const uint64_t* v, const uint64_t* v_off, size_t nrows,
                   int32_t count, int32_t offset, uint64_t* out, uint64_t* out_off, uint64_t* dest_out,
                   size_t* dest_len) {
    if (count < 0) return 2;
    const size_t m = nrows ? v_off[nrows] : 0;
    uint64_t* row = (uint64_t*)malloc((m ? m : 1) * sizeof(uint64_t));
    uint64_t* wu = (uint64_t*)malloc((m ? m : 1) * sizeof(uint64_t));
    uint64_t* nu = (uint64_t*)malloc((m ? m : 1) * sizeof(uint64_t));
    Val* wv = (Val*)malloc((m ? m : 1) * sizeof(Val));
    uint8_t* included = (uint8_t*)calloc(ndest ? ndest : 1, 1);
    if (!row || !wu || !nu || !wv || !included) {
        free(row); free(wu); free(nu); free(wv); free(included);
        return -1;
    }
    int rc = 0;
    size_t o = 0;
    out_off[0] = 0;
    for (size_t r = 0; r < nrows && rc == 0; r++) {
        /* updateUidMatrix, order branch */
        size_t un = 0;
        for (uint64_t t = v_off[r]; t < v_off[r + 1]; t++)
            if (index_of(dest, ndest, v[t]) >= 0) row[un++] = v[t];
        /* sortByValue: fetchValue per uid */
        size_t wn = 0, nn = 0;
        for (size_t t = 0; t < un; t++) {
            const long k = index_of(uid, n, row[t]);
            const uint64_t c = k < 0 ? 0 : val_off[k + 1] - val_off[k];
            if (c > 1) { rc = 3; break; } /* the schema's list flag, which processSort refuses */
            if (c == 0 || (bad && bad[val_off[k]])) { nu[nn++] = row[t]; continue; }
            const uint64_t j = val_off[k];
            if (type == T_BOOL) { rc = 1; break; }
            Val x = {0, 0};
            if (type == T_STR) { x.w = byte_off[j]; x.x = byte_off[j + 1]; }
            else { x.w = word[j]; x.x = type == T_TIME ? nsec[j] : 0; }
            wv[wn] = x;
            wu[wn++] = row[t];
        }
        if (rc) break;
        const Data d = {wv, wu, desc, type, bytes};
        go_sort(&d, (long)wn);
        memcpy(row, wu, wn * sizeof(uint64_t));
        memcpy(row + wn, nu, nn * sizeof(uint64_t));
        /* paginate */
        long long s, e;
        page_range(count, offset, (long long)un, &s, &e);
        for (long long t = s; t < e; t++) out[o++] = row[t];
        out_off[r + 1] = o;
    }
    if (rc == 0) {
        /* updateDestUids */
        for (size_t t = 0; t < o; t++) {
            const long k = index_of(dest, ndest, out[t]);
            if (k >= 0) included[k] = 1;
        }
        size_t dn = 0;
        for (size_t k = 0; k < ndest; k++)
            if (included[k]) dest_out[dn++] = dest[k];
        *dest_len = dn;
    }
    free(row); free(wu); free(nu); free(wv); free(included);
    return rc;
}
