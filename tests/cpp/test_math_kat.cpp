// Known-answer tests of algo::EvalMath in the C++ host mirror (include/dgx_algo.hpp), on the reference's math cases:
// TestProcessBinary's + and * over two maps, TestProcessBinaryBoolean's <, TestProcessTernary's cond with a missing
// branch entry stored as nil, checkAggrResult's {0: s} + {0: t} kept as a map and s + 1 set over the range,
// TestMathCeil's ceil of an int, the MinInt64 boundaries and the int / float promotion at the top.  Built and run by
// tests/test_cpp_math_mirror.py on a GPU box.
#include <cstdio>
#include <cstring>

#include "dgx_algo.hpp"

using V = std::vector<uint64_t>;
using T = std::vector<uint8_t>;
using dgx::algo::MathMap;

static int failures = 0;
#define REQUIRE_EQ(got, want, what)                                                                  \
    do {                                                                                             \
        if ((got) != (want)) { ++failures; std::printf("FAIL %s (line %d)\n", what, __LINE__); }    \
    } while (0)

static uint64_t w(double d) { uint64_t x; std::memcpy(&x, &d, 8); return x; }
static uint64_t w(int64_t i) { return (uint64_t)i; }

static dgx_math_node var(uint32_t leaf) { dgx_math_node n{}; n.op = DGX_MATH_VAR; n.leaf = leaf; return n; }
static dgx_math_node cst(int64_t v) {
    dgx_math_node n{}; n.op = DGX_MATH_CONST; n.const_tag = DGX_VAL_INT64; n.const_word = w(v); return n;
}
static dgx_math_node op(int o, uint16_t a, uint16_t b = 0, uint16_t c = 0) {
    dgx_math_node n{}; n.op = (uint8_t)o; n.child[0] = a; n.child[1] = b; n.child[2] = c; return n;
}
static MathMap ints(V k, std::vector<int64_t> v) {
    MathMap m; m.keys = k; for (int64_t x : v) m.words.push_back(w(x)); m.tags.assign(k.size(), DGX_VAL_INT64); return m;
}
static MathMap flts(V k, std::vector<double> v) {
    MathMap m; m.keys = k; for (double x : v) m.words.push_back(w(x)); m.tags.assign(k.size(), DGX_VAL_FLOAT64); return m;
}

int main() {
    if (dgx_init(-1) != DGX_OK) { std::printf("no device: %s\n", dgx_last_error()); return 2; }
    using dgx::algo::EvalMath;
    const V two = {1, 2};
    auto r = EvalMath({var(0), var(1), op(DGX_MATH_ADD, 0, 1)}, {ints(two, {2, 3}), ints(two, {4, 5})}, nullptr);
    REQUIRE_EQ(r.kind, DGX_MATH_KIND_MAP, "a + b is a map");
    REQUIRE_EQ(r.map.words, V({w(int64_t(6)), w(int64_t(8))}), "2 + 4, 3 + 5");
    r = EvalMath({var(0), var(1), op(DGX_MATH_MUL, 0, 1)}, {flts(two, {2.0, 3.0}), ints(two, {4, 5})}, nullptr);
    REQUIRE_EQ(r.map.words, V({w(8.0), w(15.0)}), "float * int");
    REQUIRE_EQ(r.map.tags, T({DGX_VAL_FLOAT64, DGX_VAL_FLOAT64}), "float * int is float");
    r = EvalMath({var(0), var(1), op(DGX_MATH_LT, 0, 1)}, {ints(two, {1, 5}), flts(two, {2.0, 5.0})}, nullptr);
    REQUIRE_EQ(r.map.words, V({1, 0}), "1 < 2.0, 5 < 5.0");
    REQUIRE_EQ(r.map.tags, T({DGX_VAL_BOOL, DGX_VAL_BOOL}), "comparisons are bools");
    r = EvalMath({var(0), cst(3), op(DGX_MATH_LT, 0, 1), var(1), cst(9), op(DGX_MATH_COND, 2, 3, 4)},
                 {ints(two, {1, 5}), ints({2}, {7})}, nullptr);
    REQUIRE_EQ(r.map.tags, T({DGX_VAL_NIL, DGX_VAL_INT64}), "cond: a missing branch entry is nil");
    REQUIRE_EQ(r.map.words[1], w(int64_t(9)), "cond: the constant branch");
    r = EvalMath({var(0), var(1), op(DGX_MATH_ADD, 0, 1)}, {ints({0}, {2}), ints({0}, {5})}, nullptr);
    REQUIRE_EQ(r.kind, DGX_MATH_KIND_MAP, "{0: s} + {0: t} stays a map");
    REQUIRE_EQ(r.map.keys, V({0}), "on key 0");
    REQUIRE_EQ(r.map.words, V({w(int64_t(7))}), "s + t");
    const V range = {4, 8};
    r = EvalMath({var(0), cst(1), op(DGX_MATH_ADD, 0, 1)}, {ints({0}, {2})}, &range);
    REQUIRE_EQ(r.kind, DGX_MATH_KIND_CONST, "s + 1 is a constant");
    REQUIRE_EQ(r.map.keys, range, "set over the range");
    r = EvalMath({var(0), op(DGX_MATH_CEIL, 0)}, {ints(two, {1, -1})}, nullptr);
    REQUIRE_EQ(r.map.words, V({w(int64_t(1)), w(int64_t(-1))}), "ceil of an int");
    r = EvalMath({cst(INT64_MIN), cst(-1), op(DGX_MATH_DIV, 0, 1)}, {}, nullptr);
    REQUIRE_EQ(r.map.words, V({w(INT64_MIN)}), "MinInt64 / -1");
    bool refused = false;
    try {
        EvalMath({cst(-1), cst(INT64_MIN), op(DGX_MATH_MUL, 0, 1)}, {}, nullptr);
    } catch (const dgx::Error& e) {
        refused = true;
    }
    REQUIRE_EQ(refused, true, "-1 * MinInt64 overflows: evalMathTree's error");
    r = EvalMath({var(0), var(1), op(DGX_MATH_ADD, 0, 1)}, {ints({1}, {1}), flts({2}, {0.5})}, nullptr);
    REQUIRE_EQ(r.map.words, V({w(1.0), w(0.5)}), "ints promoted when floats are present");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
