/* compare_oracle.c -- the compare functions eq / le / lt / ge / gt / between restated line by line from Go.  TEST
 * INFRASTRUCTURE ONLY: the checker of dgx_compare_uids / dgx_compare_rows and their device forms.
 *
 *   orc_less / orc_equal      types.Less / types.Equal (types/sort.go), both operands of one type
 *   orc_compare_vals          types.CompareVals (types/compare.go): ge !Less(v, a), gt Less(a, v), le !Less(a, v),
 *                             lt Less(v, a), eq Equal(v, a), each false when Less / Equal errors
 *   orc_compare_uids          handleValuePostings' compareAttrFn branch (worker/task.go:540-575): row i holds
 *                             UidList[i] once per matching value; any conversion error fails the task (-1)
 *   orc_compare_rows          handleCompareFunction's filterRow (worker/task.go:1395-1520) over the rows row_arg selects
 *
 * Types are DGX_VAL_*: 1 int64, 2 float64, 3 bool, 5 datetime (seconds, nanoseconds), 6 string. */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

enum { T_INT = 1, T_FLOAT = 2, T_BOOL = 3, T_TIME = 5, T_STR = 6 };
enum { OP_LE = 0, OP_GE = 1, OP_LT = 2, OP_GT = 3, OP_EQ = 4, OP_BETWEEN = 5 };

typedef struct {
    int type;
    const uint64_t* uid;
    const uint64_t* val_off;
    const uint64_t* word;
    const uint32_t* nsec;
    const uint8_t* bad;
    const uint64_t* byte_off;
    const uint8_t* bytes;
    size_t n;
} orc_col;

typedef struct {
    const uint64_t* word;
    const uint32_t* nsec;
    const uint8_t* bytes;
    const uint64_t* byte_off;
    size_t n;
} orc_args;

typedef struct {  /* types.Val */
    int tid;
    uint64_t w;
    uint32_t ns;
    const uint8_t* s;
    size_t len;
} val;

static val col_val(const orc_col* c, uint64_t j) {
    val v = {c->type, 0, 0, NULL, 0};
    if (c->type == T_STR) {
        v.s = c->bytes + c->byte_off[j];
        v.len = (size_t)(c->byte_off[j + 1] - c->byte_off[j]);
    } else {
        v.w = c->word[j];
        if (c->type == T_TIME) v.ns = c->nsec[j];
    }
    return v;
}

static val arg_val(int type, const orc_args* a, size_t k) {
    val v = {type, 0, 0, NULL, 0};
    if (type == T_STR) {
        v.s = a->bytes + a->byte_off[k];
        v.len = (size_t)(a->byte_off[k + 1] - a->byte_off[k]);
    } else {
        v.w = a->word[k];
        if (type == T_TIME) v.ns = a->nsec[k];
    }
    return v;
}

static double f64(uint64_t w) {
    double d;
    memcpy(&d, &w, 8);
    return d;
}

/* Go's string < : bytewise, unsigned, a proper prefix less. */
static int str_less(const val* a, const val* b) {
    size_t m = a->len < b->len ? a->len : b->len;
    int c = m ? memcmp(a->s, b->s, m) : 0;
    return c != 0 ? c < 0 : a->len < b->len;
}

/* Less returns true if a is strictly less than b; *err for a type it cannot sort (bool). */
static int orc_less(const val* a, const val* b, int* err) {
    *err = 0;
    switch (a->tid) {
        case T_TIME: /* a.Value.(time.Time).Before(b.Value.(time.Time)) */
            return (int64_t)a->w < (int64_t)b->w || ((int64_t)a->w == (int64_t)b->w && a->ns < b->ns);
        case T_INT: return (int64_t)a->w < (int64_t)b->w;
        case T_FLOAT: return f64(a->w) < f64(b->w);
        case T_STR: return str_less(a, b);
        default: *err = 1; return 0;  /* "Compare not supported for type" */
    }
}

static int orc_equal(const val* a, const val* b) {
    switch (a->tid) {
        case T_TIME: return a->w == b->w && a->ns == b->ns;  /* aVal.Equal(bVal): the instant */
        case T_INT: return (int64_t)a->w == (int64_t)b->w;
        case T_FLOAT: return f64(a->w) == f64(b->w);
        case T_STR: return a->len == b->len && (a->len == 0 || memcmp(a->s, b->s, a->len) == 0);
        case T_BOOL: return (a->w != 0) == (b->w != 0);
    }
    return 0;
}

/* CompareVals(op, arg1, arg2): arg1 the stored value, arg2 the argument. */
int orc_compare_vals(int op, const val* arg1, const val* arg2) {
    int err, b;
    switch (op) {
        case OP_GE: b = orc_less(arg1, arg2, &err); return !b && !err;
        case OP_GT: b = orc_less(arg2, arg1, &err); return b && !err;
        case OP_LE: b = orc_less(arg2, arg1, &err); return !b && !err;
        case OP_LT: b = orc_less(arg1, arg2, &err); return b && !err;
        case OP_EQ: return orc_equal(arg1, arg2);
    }
    return 0;
}

static int compare_between(const val* dst, const val* v1, const val* v2) {
    return orc_compare_vals(OP_GE, dst, v1) && orc_compare_vals(OP_LE, dst, v2);
}

/* The column's values of uid: [*lo, *hi), none when it is absent (posting.ErrNoValue). */
static void values_of(const orc_col* c, uint64_t uid, uint64_t* lo, uint64_t* hi) {
    size_t a = 0, b = c->n;
    while (a < b) {
        size_t m = (a + b) / 2;
        if (c->uid[m] < uid) a = m + 1; else b = m;
    }
    *lo = *hi = 0;
    if (a < c->n && c->uid[a] == uid) { *lo = c->val_off[a]; *hi = c->val_off[a + 1]; }
}

/* The value path: rowlen[i] = len(UidMatrix[i]); dest the uids with a non-empty row (algo.MergeSorted of the rows).
 * Returns the dest length, or -1 where Go returns the conversion error. */
long orc_compare_uids(int op, const orc_args* args, const orc_col* c, const uint64_t* uids, size_t nuids,
                      uint64_t* dest, uint32_t* rowlen) {
    long nd = 0;
    for (size_t i = 0; i < nuids; ++i) {
        uint64_t lo, hi;
        values_of(c, uids[i], &lo, &hi);
        uint32_t row = 0;
        for (uint64_t j = lo; j < hi; ++j) {
            if (c->bad && c->bad[j]) return -1;  /* convertToType / types.Convert: return err */
            const val v = col_val(c, j);
            switch (op) {
                case OP_EQ:
                    for (size_t k = 0; k < args->n; ++k) {
                        const val t = arg_val(c->type, args, k);
                        if (orc_compare_vals(OP_EQ, &v, &t)) { row++; break; }
                    }
                    break;
                case OP_BETWEEN: {
                    const val a0 = arg_val(c->type, args, 0), a1 = arg_val(c->type, args, 1);
                    if (compare_between(&v, &a0, &a1)) row++;
                    break;
                }
                default: {
                    const val a0 = arg_val(c->type, args, 0);
                    if (orc_compare_vals(op, &v, &a0)) row++;
                }
            }
        }
        rowlen[i] = row;
        if (row) dest[nd++] = uids[i];
    }
    return nd;
}

/* The index path: row r filtered by algo.ApplyFilter when row_arg[r] != UINT32_MAX, a value that fails conversion
 * never matching.  Writes the rows to out / out_off; returns the value count. */
size_t orc_compare_rows(int op, const orc_args* args, const orc_col* c, const uint64_t* v, const uint64_t* v_off,
                        size_t nrows, const uint32_t* row_arg, uint64_t* out, uint64_t* out_off) {
    size_t w = 0;
    out_off[0] = 0;
    for (size_t r = 0; r < nrows; ++r) {
        for (uint64_t i = v_off[r]; i < v_off[r + 1]; ++i) {
            int keep = 1;
            if (row_arg[r] != UINT32_MAX) {
                const size_t k = row_arg[r];
                uint64_t lo, hi;
                values_of(c, v[i], &lo, &hi);
                keep = 0;
                for (uint64_t j = lo; j < hi && !keep; ++j) {
                    if (c->bad && c->bad[j]) continue;  /* types.Convert failed: not this value */
                    const val d = col_val(c, j), a0 = arg_val(c->type, args, k);
                    if (op == OP_BETWEEN) {
                        const val a1 = arg_val(c->type, args, k + 1);
                        keep = compare_between(&d, &a0, &a1);
                    } else {
                        keep = orc_compare_vals(op, &d, &a0);
                    }
                }
            }
            if (keep) out[w++] = v[i];
        }
        out_off[r + 1] = w;
    }
    return w;
}
