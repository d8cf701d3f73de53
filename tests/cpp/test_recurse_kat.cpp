// Known-answer tests of algo::ReachSet in the C++ host mirror (include/dgx_algo.hpp): @recurse { friend follow } from
// uid 1 over the friend edges 1 -> {23, 24, 25, 31, 101}, 31 -> 24, 23 -> 1 and the follow edges 1 -> {24, 31},
// 31 -> 1001, 1001 -> {1000, 1003}, 1002 -> 1000, 1003 -> 1002 (query/common_test.go), one sg at a time in exec order.
// Built and run by tests/test_cpp_recurse_mirror.py on a GPU box.
#include <cstdio>
#include <map>

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
    std::map<std::string, std::map<uint64_t, V>> g;
    g["friend"] = {{1, {23, 24, 25, 31, 101}}, {23, {1}}, {31, {24}}};
    g["follow"] = {{1, {24, 31}}, {31, {1001}}, {1001, {1000, 1003}}, {1002, {1000}}, {1003, {1002}}};
    const std::vector<std::string> preds = {"friend", "follow"};
    std::map<std::string, dgx::algo::ReachSet> sets;
    for (const auto& p : preds) sets.emplace(p, dgx::algo::ReachSet());
    std::vector<std::pair<std::string, V>> exec = {{"friend", {1}}, {"follow", {1}}};
    uint64_t edges = 0;
    int levels = 0;
    std::map<std::string, V> unions;
    std::vector<uint64_t> level2;
    while (!exec.empty()) {
        ++levels;
        std::vector<std::pair<std::string, V>> next;
        for (const auto& [attr, src] : exec) {
            std::vector<List> rows;
            for (uint64_t u : src) rows.emplace_back(g[attr].count(u) ? g[attr][u] : V());
            const auto st = sets.at(attr).Filter(src, rows);
            edges += st.kept;
            if (levels == 2) level2.push_back(st.kept);
            V& un = unions[attr];
            un.insert(un.end(), st.dest.Uids.begin(), st.dest.Uids.end());
            if (!st.dest.Uids.empty())
                for (const auto& p : preds) next.push_back({p, st.dest.Uids});
        }
        exec = next;
    }
    REQUIRE_EQ(edges, uint64_t(14), "kept edges");
    REQUIRE_EQ(levels, 6, "levels");
    REQUIRE_EQ(level2, V({2, 1, 0, 0}), "level 2: the third sg's only edge (31, 24) was kept by the first");
    for (auto& [a, u] : unions) {
        std::sort(u.begin(), u.end());
        u.erase(std::unique(u.begin(), u.end()), u.end());
    }
    REQUIRE_EQ(unions["friend"], V({1, 23, 24, 25, 31, 101}), "friend DestUIDs");
    REQUIRE_EQ(unions["follow"], V({24, 31, 1000, 1001, 1002, 1003}), "follow DestUIDs");
    REQUIRE_EQ(sets.at("friend").Size(), size_t(7), "friend set");
    // hand the friend set over and back: the copy holds the same edges and refuses them again
    const auto e = sets.at("friend").Export();
    REQUIRE_EQ(e.first, V({1, 1, 1, 1, 1, 23, 31}), "export from");
    REQUIRE_EQ(e.second, V({23, 24, 25, 31, 101, 1, 24}), "export to");
    dgx::algo::ReachSet copy(e.first, e.second);
    const List f1({23, 24, 25, 31, 101}), f31({24, 26});
    const List only24({24, 26});
    const auto st = copy.Filter({1, 31}, {f1, f31}, &only24);
    REQUIRE_EQ(st.kept, uint64_t(1), "only (31, 26) is new and passes the filter");
    REQUIRE_EQ(st.dest.Uids, V({26}), "DestUIDs after the handoff");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
