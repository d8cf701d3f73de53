// Known-answer tests of algo::GroupByUid in the C++ host mirror (include/dgx_algo.hpp): the reference's
// TestGroupByFriendsMultipleParents and TestGroupByFriendsMultipleParentsVar (query/query0_test.go:1798-1836) over the
// friend edges 1 -> {23, 24, 25, 31, 101}, 23 -> {1}, 31 -> {24}.  Built and run by tests/test_cpp_groupby_mirror.py on
// a GPU box.
#include <cstdio>

#include "dgx_algo.hpp"

using dgx::pb::List;
using V = std::vector<uint64_t>;

static int failures = 0;
#define REQUIRE_EQ(got, want, what)                                                                  \
    do {                                                                                             \
        if ((got) != (want)) { ++failures; std::printf("FAIL %s (line %d)\n", what, __LINE__); }    \
    } while (0)

int main() {
    if (dgx_init(-1) != DGX_OK) { std::printf("no device: %s\n", dgx_last_error()); return 2; }
    const V src = {1, 23, 31}, dest = {1, 23, 24, 25, 31, 101};
    const std::vector<List> rows = {List{23, 24, 25, 31, 101}, List{1}, List{24}};
    // three parents: {23, 24, 25, 31, 101}, {1}, {24}
    const auto g = dgx::algo::GroupByUid({List{23, 24, 25, 31, 101}, List{1}, List{24}}, src, rows, dest);
    REQUIRE_EQ(g.size(), size_t(3), "parents");
    REQUIRE_EQ(g[0].keys, V({1, 24}), "parent 0 keys");
    REQUIRE_EQ(g[0].members, V({23, 31}), "parent 0 members");
    REQUIRE_EQ(g[1].keys, V({23, 24, 25, 31, 101}), "parent 1 keys");
    REQUIRE_EQ(g[1].counts, V({1, 1, 1, 1, 1}), "parent 1 counts");
    REQUIRE_EQ(g[2].keys, V(), "parent 2 has no groups");
    // fillGroupedVars: one parent equal to SrcUIDs, counts only; 24 -> 2 orders last
    const auto vars = dgx::algo::GroupByUid({List{1, 23, 31}}, src, rows, dest, false);
    REQUIRE_EQ(vars[0].keys, V({1, 23, 25, 31, 101, 24}), "var keys");
    REQUIRE_EQ(vars[0].counts, V({1, 1, 1, 1, 1, 2}), "var counts");
    REQUIRE_EQ(vars[0].members, V(), "counts only");
    const auto full = dgx::algo::GroupByUid({List{1, 23, 31}}, src, rows, dest);
    REQUIRE_EQ(V(full[0].members.end() - 2, full[0].members.end()), V({1, 31}), "group 24's members");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
