// Known-answer tests of algo::SubgraphFilter in the C++ host mirror (include/dgx_algo.hpp), on the friend edges of uid 1
// (query/common_test.go: 1 -> {23, 24, 25, 31, 101}; names Rick Grimes, Glenn Rhee, Daryl Dixon, Andrea on 23, 24, 25,
// 31; 101 has none).  Each anyofterms(name, ...) leaf is the name index's row for its terms:
//   TestToFastJSONFilterOrFirst:  friend(first: 2) @filter(anyofterms(name, "Andrea") or anyofterms(name, "Glenn
//                                 SomethingElse") or anyofterms(name, "Daryl"))  -> Glenn Rhee, Daryl Dixon
//   TestToFastJSONFilterOrOffset: friend(offset: 1) @filter(... "Andrea" or "Glenn Rhee" or "Daryl Dixon")
//                                                                                  -> Daryl Dixon, Andrea
//   TestToFastJSONFilterOrCount:  count(friend @filter(anyofterms(name, "Andrea") or anyofterms(name, "Andrea
//                                 Rhee")))                                         -> 2
// Built and run by tests/test_cpp_sg_filter_mirror.py on a GPU box.
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
    const V friends = {23, 24, 25, 31, 101}, andrea = {31, 240}, glenn = {24}, daryl = {25};
    auto list = [](const V& u) {
        dgx_sg_filter_leaf l{};
        l.kind = DGX_SGF_LIST;
        l.uids = u.data();
        l.n = u.size();
        return l;
    };
    const std::vector<dgx_sg_filter_leaf> leaves = {list(andrea), list(glenn), list(daryl)};
    const std::vector<uint8_t> op = {DGX_SGF_OR, DGX_SGF_LEAF, DGX_SGF_LEAF, DGX_SGF_LEAF};
    const std::vector<uint32_t> parent = {UINT32_MAX, 0, 0, 0}, leaf = {0, 0, 1, 2};
    const std::vector<List> rows = {List(friends)};
    auto first = dgx::algo::SubgraphFilter(op, parent, leaf, leaves, List(friends), rows, 2, 0);
    REQUIRE_EQ(first.rows[0].Uids, V({24, 25}), "FilterOrFirst rows");
    REQUIRE_EQ(first.dest.Uids, V({24, 25}), "FilterOrFirst dest");
    auto off = dgx::algo::SubgraphFilter(op, parent, leaf, leaves, List(friends), rows, 0, 1);
    REQUIRE_EQ(off.rows[0].Uids, V({25, 31}), "FilterOrOffset rows");
    // count(friend @filter(anyofterms(name, "Andrea") or anyofterms(name, "Andrea Rhee"))): the term rows are
    // {31, 240} and {24, 31, 240} ("Andrea With no friends" is 240)
    const V andrea_row = {31, 240}, andrea_rhee = {24, 31, 240};
    const std::vector<dgx_sg_filter_leaf> or2 = {list(andrea_row), list(andrea_rhee)};
    auto cnt = dgx::algo::SubgraphFilter({DGX_SGF_OR, DGX_SGF_LEAF, DGX_SGF_LEAF}, {UINT32_MAX, 0, 0}, {0, 0, 1}, or2,
                                         List(friends), rows, 0, 0, true);
    REQUIRE_EQ(cnt.counts, std::vector<uint32_t>({2}), "FilterOrCount");
    REQUIRE_EQ(cnt.dest.Uids, V({24, 31}), "FilterOrCount dest");
    // has(friend)-style COUNT leaf: NOT(count > 0) over per-uid counts keeps the uids without friends
    dgx_sg_filter_leaf c{};
    const std::vector<uint32_t> fc = {1, 0, 0, 1, 0};
    c.kind = DGX_SGF_COUNT;
    c.cmp = DGX_SGF_CMP_GT;
    c.threshold = 0;
    c.counts = fc.data();
    auto nf = dgx::algo::SubgraphFilter({DGX_SGF_NOT, DGX_SGF_LEAF}, {UINT32_MAX, 0}, {0, 0}, {c}, List(friends), rows);
    REQUIRE_EQ(nf.dest.Uids, V({24, 25, 101}), "not has(friend)");
    REQUIRE_EQ(nf.rows[0].Uids, V({24, 25, 101}), "not has(friend) row");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
