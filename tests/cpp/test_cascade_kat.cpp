// Known-answer tests of algo::Cascade in the C++ host mirror (include/dgx_algo.hpp): the reference's
// TestCascadeWithPaginationDeep shape over the friend edges 1 -> {23, 24, 25, 31, 101}, 23 -> {1}, 31 -> {24},
// 101 -> {} and names on 1, 23, 24, 25, 31 (query/common_test.go):
//   me(func: uid(1, 23, 24, 25, 31)) @cascade { name friend { name friend(first: 2, offset: 1) { name } } }
// Built and run by tests/test_cpp_cascade_mirror.py on a GPU box.
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
    const uint8_t C = DGX_CASCADE_CASCADE | DGX_CASCADE_CHECKED;
    const V people = {1, 23, 24, 25, 31}, friends1 = {1, 23, 24, 25, 31, 101}, friends2 = {1, 24};
    auto named = [](const V& u) {  // has_val of name over a dest list
        std::vector<uint8_t> h;
        for (uint64_t x : u) h.push_back(x != 101);
        return h;
    };
    std::vector<dgx::algo::CascadeNode> t(6);
    t[0] = {-1, DGX_CASCADE_CASCADE, 0, 0, 0, List(people), {List(people)}, {}};
    t[1] = {0, C, 0, 0, 0, List(V{}), {}, named(people)};
    t[2] = {0, C, 0, 0, 0, List(friends1), {List(V{23, 24, 25, 31, 101}), List(V{1}), List(V{}), List(V{}),
                                             List(V{24})}, {}};
    t[3] = {2, C, 0, 0, 0, List(V{}), {}, named(friends1)};
    // friend rows of friends1: 1 -> {23, 24, 25, 31, 101}, 23 -> {1}, 24, 25 -> {}, 31 -> {24}, 101 -> {}
    t[4] = {2, C, 2, 1, 0, List(friends1), {List(V{23, 24, 25, 31, 101}), List(V{1}), List(V{}), List(V{}),
                                            List(V{24}), List(V{})}, {}};
    t[5] = {4, C, 0, 0, 0, List(V{}), {}, named(friends1)};
    const auto r = dgx::algo::Cascade(t);
    // level 2: friend(first: 2, offset: 1) keeps 101 out (no name), so uid 1's row [23 24 25 31] pages to [24 25]; the
    // rows of 23 and 31 hold one friend each and page to nothing
    REQUIRE_EQ(r.first[4][0].Uids, V({24, 25}), "friend of friend of 1, paged");
    REQUIRE_EQ(r.first[4][1].Uids, V({}), "friend of friend of 23, paged away");
    REQUIRE_EQ(r.second[4].Uids, V({1, 23, 24, 25, 31}), "friend.friend dest: 101 has no name");
    // level 1: only friend 1 keeps a row after the paging, so friend's dest is {1}
    REQUIRE_EQ(r.second[2].Uids, V({1}), "friend dest");
    REQUIRE_EQ(r.first[2][0].Uids, V({}), "friend row of 1 filtered by {1}");
    REQUIRE_EQ(r.second[0].Uids, V({23}), "root: only 23 has a friend left");
    REQUIRE_EQ(r.first[0][0].Uids, people, "root row without root pagination");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
