// Known-answer tests of algo::OrderByPred in the C++ host mirror (include/dgx_algo.hpp over dgx_pred_order): the
// published answers of tests/golden/pred_order_common.json (query/common_test.go values: uid 1's friends 23, 24, 25,
// 31, 101 and their alias; Michonne 1, Rick Grimes 23 and Glenn Rhee 24 and their dob), and cases worked by hand from
// sortWithoutIndex's rules: the uids with a value sorted by it (ties in row order up to 12 entries), then those
// without one in row order, then x.PageRange; a bool column and a list value refused as Go refuses them.
// Built and run by tests/test_cpp_pred_order_mirror.py on a GPU box.
#include <cstdio>
#include <string>

#include "dgx_algo.hpp"

using dgx::pb::List;
using V = std::vector<uint64_t>;

static int failures = 0;
#define REQUIRE_EQ(got, want, what)                                                                  \
    do {                                                                                             \
        if ((got) != (want)) { ++failures; std::printf("FAIL %s (line %d)\n", what, __LINE__); }    \
    } while (0)

static bool refused(const dgx::algo::ValColumn& col, const V& dest, int32_t count = 0) {
    try {
        dgx::algo::OrderByPred(col, false, List(dest), {List(dest)}, count);
    } catch (const dgx::Error& e) {
        return e.code == DGX_ERR_ARG;
    }
    return false;
}

int main() {
    if (dgx_init(-1) != DGX_OK) { std::printf("no device: %s\n", dgx_last_error()); return 2; }
    // TestToFastJSONOrderName / ...Desc: friend(orderasc / orderdesc: alias) of uid 1
    dgx::algo::ValColumn alias;
    alias.type = DGX_VAL_STRING;
    alias.uids = {23, 24, 25, 31, 101};
    alias.strs = {{"Zambo Alice"}, {"John Alice"}, {"Bob Joe"}, {"Allan Matt"}, {"John Oliver"}};
    const V fr = {23, 24, 25, 31, 101};
    REQUIRE_EQ(dgx::algo::OrderByPred(alias, false, List(fr), {List(fr)}, 1000).rows[0].Uids, V({31, 25, 24, 101, 23}),
               "TestToFastJSONOrderName");
    REQUIRE_EQ(dgx::algo::OrderByPred(alias, true, List(fr), {List(fr)}, 1000).rows[0].Uids, V({23, 101, 24, 25, 31}),
               "TestToFastJSONOrderNameDesc");
    // TestGeneratorMultiRootOrder / ...Orderdesc / ...VarOrderOffset1: me(func: anyofterms(name, "Michonne Rick
    // Glenn"), orderasc / orderdesc: dob[, offset: 2]), the dob days as UTC seconds
    dgx::algo::ValColumn rdob;
    rdob.type = DGX_VAL_DATETIME;
    rdob.uids = {1, 23, 24};
    rdob.words = {{(uint64_t)-1893456000LL}, {(uint64_t)-1893369600LL}, {(uint64_t)-1914278400LL}};
    rdob.nsec = {{0}, {0}, {0}};
    const V mrg = {1, 23, 24};
    REQUIRE_EQ(dgx::algo::OrderByPred(rdob, false, List(mrg), {List(mrg)}, 1000).rows[0].Uids, V({24, 1, 23}),
               "TestGeneratorMultiRootOrder");
    REQUIRE_EQ(dgx::algo::OrderByPred(rdob, true, List(mrg), {List(mrg)}, 1000).rows[0].Uids, V({23, 1, 24}),
               "TestGeneratorMultiRootOrderdesc");
    REQUIRE_EQ(dgx::algo::OrderByPred(rdob, false, List(mrg), {List(mrg)}, 1000, 2).rows[0].Uids, V({23}),
               "TestGeneratorMultiRootVarOrderOffset1");
    // orderasc: name over 1, 23, 24, 25, 31 and 101, where 101 has no name and 25's name did not convert
    dgx::algo::ValColumn names;
    names.type = DGX_VAL_STRING;
    names.uids = {1, 23, 24, 25, 31};
    names.strs = {{"Michonne"}, {"Rick Grimes"}, {"Glenn Rhee"}, {"Daryl Dixon"}, {"Andrea"}};
    names.bad = {{0}, {0}, {0}, {1}, {0}};
    const V all = {1, 23, 24, 25, 31, 101};
    auto asc = dgx::algo::OrderByPred(names, false, List(all), {List(all)});
    REQUIRE_EQ(asc.rows[0].Uids, V({31, 24, 1, 23, 25, 101}), "orderasc: name, nulls last in row order");
    auto desc = dgx::algo::OrderByPred(names, true, List(all), {List(all)}, 3, 1);
    REQUIRE_EQ(desc.rows[0].Uids, V({1, 24, 31}), "orderdesc: name, first: 3, offset: 1");
    REQUIRE_EQ(desc.dest.Uids, V({1, 24, 31}), "orderdesc dest");
    // orderasc: age with a tie kept in row order, a uid outside dest dropped
    dgx::algo::ValColumn age;
    age.type = DGX_VAL_INT64;
    age.uids = {1, 23, 24, 31};
    age.words = {{38}, {15}, {38}, {19}};
    auto a = dgx::algo::OrderByPred(age, false, List(V({1, 23, 24})), {List(V({1, 23, 24, 31}))});
    REQUIRE_EQ(a.rows[0].Uids, V({23, 1, 24}), "orderasc: age");
    // orderdesc: dob, two instants in one second
    dgx::algo::ValColumn dob;
    dob.type = DGX_VAL_DATETIME;
    dob.uids = {1, 23, 24};
    dob.words = {{(uint64_t)-100}, {(uint64_t)-100}, {5}};
    dob.nsec = {{7}, {8}, {0}};
    auto d = dgx::algo::OrderByPred(dob, true, List(V({1, 23, 24})), {List(V({1, 23, 24}))});
    REQUIRE_EQ(d.rows[0].Uids, V({24, 23, 1}), "orderdesc: dob");
    // refusals
    dgx::algo::ValColumn alive;
    alive.type = DGX_VAL_BOOL;
    alive.uids = {1};
    alive.words = {{1}};
    REQUIRE_EQ(refused(alive, {1}), true, "bool refused");
    REQUIRE_EQ(refused(age, {1}, -1), true, "negative count refused");
    dgx::algo::ValColumn list = age;
    list.words[0] = {38, 39};
    REQUIRE_EQ(refused(list, {1, 23}), true, "list value refused");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
