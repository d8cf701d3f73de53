// Known-answer tests of algo::OrderByVar in the C++ host mirror (include/dgx_algo.hpp over dgx_var_order), on the
// published answers of two reference tests (query/common_test.go uids: Michonne 1, Rick Grimes 23, Glenn Rhee 24,
// Daryl Dixon 25, Andrea 31, "Andrea With no friends" 240, and 101 without a name):
//   TestMultiCountSort:     uid(f), orderasc: val(n), n = count(friend) = {1: 5, 23: 1, 31: 1, 240: 0}
//                           -> Andrea With no friends, Rick Grimes, Andrea, Michonne (the tie at 1 in uid order)
//   TestQueryVarValAggMul:  uid(f), orderdesc: val(mul), mul = {23: 15, 24: 0, 25: 0, 31: 19, 101: 0}
//                           -> Andrea, Rick Grimes, Glenn Rhee, Daryl Dixon, 101 (the tie at 0 in uid order)
// plus the nil map of TestUseVariableBeforeDefinitionError, a math() map holding nils and a page cut.
// Built and run by tests/test_cpp_var_order_mirror.py on a GPU box.
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

static dgx::algo::ValueMap int_map(const V& keys, const std::vector<int64_t>& vals) {
    dgx::algo::ValueMap m;
    m.type = DGX_VAL_INT64;
    m.keys = keys;
    for (int64_t x : vals) m.words.push_back((uint64_t)x);
    return m;
}

int main() {
    if (dgx_init(-1) != DGX_OK) { std::printf("no device: %s\n", dgx_last_error()); return 2; }
    const V f = {1, 23, 31, 240};
    auto cs = dgx::algo::OrderByVar(int_map(f, {5, 1, 1, 0}), false, List(f), {List(f)});
    REQUIRE_EQ(cs.rows[0].Uids, V({240, 23, 31, 1}), "TestMultiCountSort rows");
    REQUIRE_EQ(cs.dest.Uids, f, "TestMultiCountSort dest");
    const V fr = {23, 24, 25, 31, 101};
    auto mul = dgx::algo::OrderByVar(int_map(fr, {15, 0, 0, 19, 0}), true, List(fr), {List(fr)});
    REQUIRE_EQ(mul.rows[0].Uids, V({31, 23, 24, 25, 101}), "TestQueryVarValAggMul rows");
    // first: 2 keeps the two largest; the new dest is theirs
    auto page = dgx::algo::OrderByVar(int_map(fr, {15, 0, 0, 19, 0}), true, List(fr), {List(fr)}, 2, 0);
    REQUIRE_EQ(page.rows[0].Uids, V({31, 23}), "orderdesc first: 2 rows");
    REQUIRE_EQ(page.dest.Uids, V({23, 31}), "orderdesc first: 2 dest");
    // a math() map: nils sort last both ways, a float and an int of one value tie
    dgx::algo::MathMap mm;
    mm.keys = {1, 23, 31, 240};
    const double two = 2.0;
    uint64_t w2;
    std::memcpy(&w2, &two, 8);
    mm.words = {0, 2, w2, 0};
    mm.tags = {DGX_VAL_NIL, DGX_VAL_INT64, DGX_VAL_FLOAT64, DGX_VAL_NIL};
    auto mo = dgx::algo::OrderByVar(mm, false, List(f), {List(f)});
    REQUIRE_EQ(V(mo.rows[0].Uids.begin(), mo.rows[0].Uids.begin() + 2), V({23, 31}), "math map, nils last");
    // TestUseVariableBeforeDefinitionError: the nil map is Go's error
    dgx::algo::MathMap nil;
    nil.nil = true;
    bool refused = false;
    try {
        dgx::algo::OrderByVar(nil, false, List(f), {List(f)});
    } catch (const dgx::Error& e) {
        refused = e.code == DGX_ERR_ARG;
    }
    REQUIRE_EQ(refused, true, "nil map refused");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
