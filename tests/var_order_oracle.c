/*
 * var_order_oracle.c -- ordering a uid matrix by a value variable, restated line by line from the reference:
 *   applyOrderAndPagination (query/query.go :2511-2530), value-variable branch: updateUidMatrix (:1425-1439) with an
 *     order keeps, in row order, the row uids IndexOf(DestUIDs, uid) >= 0 finds;
 *   sortAndPaginateUsingVar (:2697-2738): a nil UidToVal is an error; per row W is the uids with a map entry, in row
 *     order; an empty W leaves the row as it is; otherwise types.Sort(values, &uids, []bool{desc}, "") and the row
 *     becomes the sorted uids; then x.PageRange (x/x.go:738-767) when Count or Offset is set;
 *   updateDestUids (:2594-2609): DestUIDs keeps the values some row still holds;
 *   types.Sort -> SortWithFacet (types/sort.go :142-166): IsSortable on the first entry's type, then sort.Sort(byValue)
 *     with byValue.Less (:49-82), less / mismatchedLess (:188-232) and equal (:249-);
 *   sort.Sort (Go >= 1.19, sort/sort.go and sort/zsortinterface.go): pdqsort(data, 0, n, bits.Len(n)) with
 *     insertionSort, heapSort / siftDown, pdqsort, partition, partitionEqual, partialInsertionSort, breakPatterns
 *     (xorshift, nextPowerOfTwo), choosePivot, order2, median, medianAdjacent and reverseRange.
 * Map entries carry the library's tags: 1 int64, 2 float64, 3 bool, 4 nil (Go's Val{}).  TEST INFRASTRUCTURE ONLY.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { T_INT = 1, T_FLOAT = 2, T_BOOL = 3, T_NIL = 4 };

/* Go's TypeIDs (protos/pb.proto Posting.ValType): DEFAULT 0, INT 2, FLOAT 3, BOOL 4 */
static int go_tid(uint8_t t) { return t == T_INT ? 2 : t == T_FLOAT ? 3 : t == T_BOOL ? 4 : 0; }

typedef struct {
    uint8_t tag;
    uint64_t w;
} Val;

static double f64(uint64_t w) {
    double d;
    memcpy(&d, &w, 8);
    return d;
}

/* which helpers ran, for the tests' coverage checks */
typedef struct {
    uint64_t insertion, heap, partition, partition_equal, partial_insertion, partial_insertion_ok, break_patterns,
        reverse;
} OrcVoStats;
static __thread OrcVoStats g_st;

void orc_var_order_stats(OrcVoStats* s, int reset) {
    if (s) *s = g_st;
    if (reset) memset(&g_st, 0, sizeof g_st);
}

/* ---- types/sort.go ---- */
static int mismatched_less(Val a, Val b) {
    const int at = go_tid(a.tag), bt = go_tid(b.tag);
    if ((a.tag != T_INT && a.tag != T_FLOAT) || (b.tag != T_INT && b.tag != T_FLOAT)) return at < bt;
    if (a.tag == T_FLOAT) return f64(a.w) < (double)(int64_t)b.w;
    return (double)(int64_t)a.w < f64(b.w);
}

static int less(Val a, Val b) {
    if (a.tag != b.tag) return mismatched_less(a, b);
    switch (a.tag) {
        case T_INT: return (int64_t)a.w < (int64_t)b.w;
        case T_FLOAT: return f64(a.w) < f64(b.w);
    }
    return 0; /* bool: no case in less */
}

static int equal(Val a, Val b) {
    if (a.tag != b.tag) return 0;
    switch (a.tag) {
        case T_INT: return (int64_t)a.w == (int64_t)b.w;
        case T_FLOAT: return f64(a.w) == f64(b.w);
        case T_BOOL: return a.w == b.w;
    }
    return 0;
}

typedef struct {
    Val* v;
    uint64_t* u;
    int desc;
} Data;

/* byValue.Less with one value per uid */
static int Less(const Data* d, long i, long j) {
    const Val a = d->v[i], b = d->v[j];
    if (a.tag == T_NIL && b.tag == T_NIL) return d->desc;
    if (a.tag == T_NIL) return 0;
    if (b.tag == T_NIL) return 1;
    if (equal(a, b)) return 0;
    const int l = less(a, b);
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
    g_st.insertion++;
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
    g_st.heap++;
    const long first = a, lo = 0, hi = b - a;
    for (long i = (hi - 1) / 2; i >= 0; i--) sift_down(d, i, hi, first);
    for (long i = hi - 1; i >= 0; i--) {
        Swap(d, first, first + i);
        sift_down(d, lo, i, first);
    }
}

enum { UNKNOWN_HINT = 0, INCREASING_HINT = 1, DECREASING_HINT = 2 };

static long partition(const Data* d, long a, long b, long pivot, int* already) {
    g_st.partition++;
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
    g_st.partition_equal++;
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
    g_st.partial_insertion++;
    const int max_steps = 5;
    const long shortest_shifting = 50;
    long i = a + 1;
    for (int j = 0; j < max_steps; j++) {
        while (i < b && !Less(d, i, i - 1)) i++;
        if (i == b) {
            g_st.partial_insertion_ok++;
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
        g_st.break_patterns++;
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
    g_st.reverse++;
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

/* types.Sort over one W: 0, or 2 when the first entry is a bool ("isn't sortable"). */
static int types_sort(Val* v, uint64_t* u, long n, int desc) {
    if (n == 0) return 0;
    if (v[0].tag == T_BOOL) return 2; /* IsSortable(v[0][0].Tid): nil (DefaultID), int and float pass */
    const Data d = {v, u, desc};
    go_sort(&d, n);
    return 0;
}

/* sort.Sort(byValue) of n values in place, with their uids: for pinning the tie order against Go. */
int orc_var_order_sort(const uint8_t* tag, uint64_t* word, uint64_t* uid, size_t n, int desc) {
    Val* v = (Val*)malloc((n ? n : 1) * sizeof(Val));
    if (!v) return -1;
    for (size_t i = 0; i < n; i++) v[i] = (Val){tag[i], word[i]};
    const int rc = types_sort(v, uid, (long)n, desc);
    for (size_t i = 0; i < n; i++) word[i] = v[i].w;
    free(v);
    return rc;
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

/* The whole node: rows v[v_off[i] .. v_off[i+1]), the map key[n] / word[n] / tag[n] (nil = Go's nil UidToVal), the
 * node's DestUIDs dest[ndest].  Writes the rows to out / out_off and the new DestUIDs to dest_out / *dest_len.
 * Returns 0, 1 (a nil map: "used before definition"), 2 (a row's first entry is a bool) or -1 (allocation). */
int orc_var_order(const uint64_t* key, const uint64_t* word, const uint8_t* tag, size_t n, int nil, int desc,
                  const uint64_t* dest, size_t ndest, const uint64_t* v, const uint64_t* v_off, size_t nrows,
                  int32_t count, int32_t offset, uint64_t* out, uint64_t* out_off, uint64_t* dest_out,
                  size_t* dest_len) {
    if (nil) return 1;
    const size_t m = nrows ? v_off[nrows] : 0;
    uint64_t* row = (uint64_t*)malloc((m ? m : 1) * sizeof(uint64_t));
    uint64_t* wu = (uint64_t*)malloc((m ? m : 1) * sizeof(uint64_t));
    Val* wv = (Val*)malloc((m ? m : 1) * sizeof(Val));
    uint8_t* included = (uint8_t*)calloc(ndest ? ndest : 1, 1);
    if (!row || !wu || !wv || !included) {
        free(row); free(wu); free(wv); free(included);
        return -1;
    }
    int rc = 0;
    size_t o = 0;
    out_off[0] = 0;
    for (size_t r = 0; r < nrows; r++) {
        /* updateUidMatrix, order branch */
        size_t un = 0;
        for (uint64_t t = v_off[r]; t < v_off[r + 1]; t++)
            if (index_of(dest, ndest, v[t]) >= 0) row[un++] = v[t];
        /* sortAndPaginateUsingVar */
        size_t wn = 0;
        for (size_t t = 0; t < un; t++) {
            const long k = index_of(key, n, row[t]);
            if (k < 0) continue;
            wv[wn] = (Val){tag[k], word[k]};
            wu[wn++] = row[t];
        }
        if (wn > 0) {
            if ((rc = types_sort(wv, wu, (long)wn, desc))) break;
            memcpy(row, wu, wn * sizeof(uint64_t));
            un = wn;
        }
        long long s = 0, e = (long long)un;
        if (count != 0 || offset != 0) page_range(count, offset, (long long)un, &s, &e);
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
    free(row); free(wu); free(wv); free(included);
    return rc;
}
