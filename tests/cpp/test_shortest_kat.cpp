// Known-answer tests of algo::PathSearch in the C++ host mirror (include/dgx_algo.hpp): shortest(from: 1, to: 1003)
// { path follow } and shortest(from: 1, to: 1002) { path @filter(not anyofterms(name, "alice")) follow } over the
// path and follow edges of query/common_test.go, with Go's exec structure (every sg with a DestUIDs spawns one sg per
// child), against the answers of TestShortestPath4 and TestShortestPath_filter (query/query3_test.go).
// Built and run by tests/test_cpp_shortest_mirror.py on a GPU box.
#include <cstdio>
#include <map>
#include <set>

#include "dgx_algo.hpp"

using dgx::pb::List;
using V = std::vector<uint64_t>;
using Sg = dgx::algo::PathSearch::Sg;

static int failures = 0;
#define REQUIRE_EQ(got, want, what)                                                                  \
    do {                                                                                             \
        if ((got) != (want)) { ++failures; std::printf("FAIL %s (line %d)\n", what, __LINE__); }    \
    } while (0)

using Graph = std::map<uint64_t, V>;

// ProcessGraph + updateUidMatrix for one child: rows of src, DestUIDs = their union minus the excluded uids.
static Sg process(const Graph& g, uint32_t attr, const V& src, const std::set<uint64_t>& exclude) {
    Sg sg;
    sg.attr = attr;
    sg.src = src;
    std::set<uint64_t> dest;
    for (uint64_t u : src) {
        auto it = g.find(u);
        V row = it == g.end() ? V() : it->second;
        for (uint64_t x : row) if (!exclude.count(x)) dest.insert(x);
        sg.rows.emplace_back(row);
    }
    sg.dest = List(V(dest.begin(), dest.end()));
    for (List& r : sg.rows) {
        V kept;
        for (uint64_t x : r.Uids) if (dest.count(x)) kept.push_back(x);
        r = List(kept);
    }
    return sg;
}

static std::pair<V, std::vector<uint32_t>> shortest(const std::vector<Graph>& children,
                                                    const std::vector<std::set<uint64_t>>& exclude, uint64_t from,
                                                    uint64_t to, std::vector<dgx_path_stats>* levels) {
    dgx::algo::PathSearch ps(from, to);
    std::vector<std::pair<uint32_t, V>> exec;
    for (uint32_t c = 0; c < children.size(); ++c) exec.push_back({c, V{from}});
    while (!exec.empty()) {
        std::vector<Sg> sgs;
        for (const auto& [c, src] : exec) sgs.push_back(process(children[c], c, src, exclude[c]));
        const auto lv = ps.Expand(sgs);
        levels->push_back(lv.stats);
        if (lv.stats.to_level || lv.stats.discovered == 0) break;
        exec.clear();
        for (size_t i = 0; i < sgs.size(); ++i)
            if (!sgs[i].dest.Uids.empty())
                for (uint32_t c = 0; c < children.size(); ++c) exec.push_back({c, lv.next[i].Uids});
    }
    return ps.Path();
}

int main() {
    if (dgx_init(-1) != DGX_OK) { std::printf("no device: %s\n", dgx_last_error()); return 2; }
    const Graph path = {{1, {24, 31}}, {31, {1000}}, {1000, {1001, 1002}}, {1001, {1002, 1003}}, {1002, {1003}},
                        {1003, {1001}}};
    const Graph follow = {{1, {24, 31}}, {31, {1001}}, {1001, {1000, 1003}}, {1002, {1000}}, {1003, {1002}}};
    std::vector<dgx_path_stats> lv;
    auto r = shortest({path, follow}, {{}, {}}, 1, 1003, &lv);
    REQUIRE_EQ(r.first, V({1, 31, 1001, 1003}), "TestShortestPath4 uids");
    REQUIRE_EQ(r.second, std::vector<uint32_t>({1, 1, 1}), "TestShortestPath4: every hop says follow");
    REQUIRE_EQ(lv.size(), size_t(3), "three levels");
    REQUIRE_EQ(lv[0].edges, uint64_t(4), "level 1 counts (1, 24) and (1, 31) once per sg");
    REQUIRE_EQ(lv[2].to_level, uint64_t(3), "To at level 3");
    lv.clear();
    r = shortest({path, follow}, {{1000}, {}}, 1, 1002, &lv);  // 1000 is Alice
    REQUIRE_EQ(r.first, V({1, 31, 1001, 1002}), "TestShortestPath_filter uids");
    REQUIRE_EQ(r.second, std::vector<uint32_t>({1, 1, 0}), "TestShortestPath_filter: follow, follow, path");
    lv.clear();
    r = shortest({path, follow}, {{1000}, {1001}}, 1, 1002, &lv);  // and 1001 is Bob
    REQUIRE_EQ(r.first.size(), size_t(0), "TestShortestPath_filter2: no path");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
