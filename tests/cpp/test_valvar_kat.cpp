// Known-answer tests of algo::PropagateVar and algo::LevelAgg in the C++ host mirror (include/dgx_algo.hpp), on
// query/common_test.go's data: TestLevelBasedFacetVarSum1's propagation of L1 = {1001: 0.1, 1002: 0.7} through
// `path` (1001 -> {1002, 1003}, 1002 -> {1003}), TestLevelBasedSumMix1's int map {1: 38} through 1 -> {24, 31},
// TestLevelBasedFacetVarAggSum's sum 0.7999999999999999, and TestQueryVarValAggMinMax's min / max of the ages over
// the friend rows.  Built and run by tests/test_cpp_valvar_mirror.py on a GPU box.
#include <cstdio>
#include <cstring>

#include "dgx_algo.hpp"

using dgx::pb::List;
using V = std::vector<uint64_t>;

static int failures = 0;
#define REQUIRE_EQ(got, want, what)                                                                  \
    do {                                                                                             \
        if ((got) != (want)) { ++failures; std::printf("FAIL %s (line %d)\n", what, __LINE__); }    \
    } while (0)

static uint64_t w(double d) { uint64_t x; std::memcpy(&x, &d, 8); return x; }
static uint64_t w(int64_t i) { return (uint64_t)i; }

int main() {
    if (dgx_init(-1) != DGX_OK) { std::printf("no device: %s\n", dgx_last_error()); return 2; }
    using dgx::algo::ValueMap;
    const ValueMap L1{DGX_VAL_FLOAT64, {1001, 1002}, {w(0.1), w(0.7)}};
    const auto p = dgx::algo::PropagateVar(L1, {{{1001, 1002}, {List{1002, 1003}, List{1003}}, {1002, 1003}}});
    REQUIRE_EQ(p.type, DGX_VAL_FLOAT64, "float map stays float");
    REQUIRE_EQ(p.keys, V({1002, 1003}), "propagated keys");
    REQUIRE_EQ(p.words, V({w(0.1), w(0.7999999999999999)}), "0.1 and 0.1 + 0.7");
    const ValueMap age{DGX_VAL_INT64, {1}, {w(int64_t(38))}};
    const auto a = dgx::algo::PropagateVar(age, {{{1}, {List{24, 31}}, {24, 31}}});
    REQUIRE_EQ(a.keys, V({24, 31}), "int map keys");
    REQUIRE_EQ(a.words, V({w(int64_t(38)), w(int64_t(38))}), "int map values");
    const auto s = dgx::algo::LevelAgg(DGX_AGG_SUM, L1, {1000}, {List{1001, 1002}});
    REQUIRE_EQ(s.keys, V({1000}), "sumw key");
    REQUIRE_EQ(s.words, V({w(0.7999999999999999)}), "sumw");
    const ValueMap x{DGX_VAL_INT64, {1, 23, 24, 25, 31}, {w(int64_t(38)), w(int64_t(15)), w(int64_t(15)),
                                                          w(int64_t(17)), w(int64_t(19))}};
    const V roots = {1, 23, 31, 240};
    const std::vector<List> friends = {List{23, 24, 25, 31, 101}, List{1}, List{24}, List{}};
    const auto n = dgx::algo::LevelAgg(DGX_AGG_MIN, x, roots, friends);
    const auto m = dgx::algo::LevelAgg(DGX_AGG_MAX, x, roots, friends);
    REQUIRE_EQ(n.keys, V({1, 23, 31}), "rows with a value");
    REQUIRE_EQ(n.words, V({w(int64_t(15)), w(int64_t(38)), w(int64_t(15))}), "min(val(x))");
    REQUIRE_EQ(m.words, V({w(int64_t(19)), w(int64_t(38)), w(int64_t(15))}), "max(val(x))");
    const auto avg = dgx::algo::LevelAgg(DGX_AGG_AVG, x, roots, friends);
    REQUIRE_EQ(avg.type, DGX_VAL_FLOAT64, "avg is float");
    REQUIRE_EQ(avg.words[0], w(16.5), "avg of 15, 15, 17, 19");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
