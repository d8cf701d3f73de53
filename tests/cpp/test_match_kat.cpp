// Known-answer tests of algo::MatchFuzzy in the C++ host mirror (include/dgx_algo.hpp over dgx_match), on published
// answers: worker/match_test.go TestDistance's distances as one-uid columns tested at the distance and one below it,
// and TestMatchFuncWithAfterWithValidUid (match(name, Ali, 5), after: 0x2710 -> 0x2712, 0x2714) over the Alice uids of
// query/common_test.go, the "Ali" trigram row read from after.  Built and run by tests/test_cpp_match_mirror.py on a
// GPU box.
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

int main() {
    const struct { const char* a; const char* b; int d; } dist[] = {
        {"detour", "detour", 0}, {"detour", "det.our", 1}, {"detour", "det..our", 2}, {"detour", "..det..our", 4},
        {"detour", "detour..", 2}, {"detour", "detour...", 3}, {"detour", "...detour", 3}, {"detour", "..detour.", 3},
        {"detour", "detoar", 1}, {"detour", "DETOUR", 6}};
    for (const auto& t : dist) {
        dgx::algo::StrColumn col{{7}, {{t.b}}};
        REQUIRE_EQ(dgx::algo::MatchFuzzy(col, t.a, t.d, List(V{7})).Uids, V{7}, t.b);
        if (t.d > 0) REQUIRE_EQ(dgx::algo::MatchFuzzy(col, t.a, t.d - 1, List(V{7})).Uids, V{}, t.b);
    }
    // name values of the uids the "Ali" trigram row holds; the row is read from after = 0x2710
    dgx::algo::StrColumn names{{110, 1000, 2301, 10000, 10002, 10004},
                               {{"Alice"}, {"Alice"}, {"Alice\""}, {"Alice"}, {"Alice"}, {"Alice"}}};
    const V row{10002, 10004};
    REQUIRE_EQ(dgx::algo::MatchFuzzy(names, "Ali", 5, List(V{}), {List(row)}).Uids, (V{0x2712, 0x2714}),
               "TestMatchFuncWithAfterWithValidUid");
    REQUIRE_EQ(dgx::algo::MatchFuzzy(names, "Ali", 5, List(V{}), {List(V{})}).Uids, V{},
               "TestMatchFuncWithAfterWithLastUid");
    // the UidList branch wins over the rows; an invalid byte is one rune
    dgx::algo::StrColumn bad{{3, 5}, {{"al\xff\xff" "e"}, {"", "alice"}}};
    REQUIRE_EQ(dgx::algo::MatchFuzzy(bad, "alice", 2, List(V{3, 5, 9}), {List(V{9})}).Uids, (V{3, 5}), "UidList");
    REQUIRE_EQ(dgx::algo::MatchFuzzy(bad, "alice", 1, List(V{3, 5})).Uids, (V{5}), "invalid bytes");
    bool refused = false;
    try {
        dgx::algo::MatchFuzzy(bad, "alice", -1, List(V{3}));
    } catch (const dgx::Error& e) {
        refused = e.code == DGX_ERR_ARG;
    }
    REQUIRE_EQ(refused, true, "max < 0");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
