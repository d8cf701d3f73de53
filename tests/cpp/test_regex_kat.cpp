// Known-answer tests of algo::MatchRegex in the C++ host mirror (include/dgx_algo.hpp over dgx_regex_match), on
// published answers: query/query3_test.go TestFilterRegex6-13, regexp(value, /.../) over the 24 `value` strings
// query/common_test.go gives the `pattern` children 0x2000, 0x2001, ... of uid 0x1234, plus the refusals.  Built and
// run by tests/test_cpp_regex_mirror.py on a GPU box.
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
    const char* values[] = {"mississippi", "missouri", "mission", "missionary", "whissle", "transmission", "zipped",
                            "monosiphonic", "vasopressin", "vapoured", "virtuously", "zurich", "synopsis",
                            "subsensuously", "admission", "commission", "submission", "subcommission",
                            "retransmission", "omission", "permission", "intermission", "dimission", "discommission"};
    dgx::algo::StrColumn col;
    V all;
    for (uint64_t i = 0; i < 24; ++i) {
        col.uids.push_back(0x2000 + i);
        col.vals.push_back({values[i]});
        all.push_back(0x2000 + i);
    }
    const struct { const char* test; const char* pat; bool fold; V want; } cases[] = {
        {"TestFilterRegex6", "miss((issippi)|(ouri))", false, {0x2000, 0x2001}},
        {"TestFilterRegex7", "[aeiou]mission", false, {0x2013, 0x2016}},
        {"TestFilterRegex8", "^(trans)?mission", false, {0x2002, 0x2003, 0x2005}},
        {"TestFilterRegex9", "s.{2,5}mission", false, {0x2010, 0x2011, 0x2017}},
        {"TestFilterRegex10", "[^m]iss", false, {0x2000, 0x2004}},
        {"TestFilterRegex11", "SUB[cm]", true, {0x2010, 0x2011}},
        {"TestFilterRegex12", "(?i)SUB[cm]", false, {0x2010, 0x2011}},
        {"TestFilterRegex13", "(?i)SUB[cm](?-i)ISSION", false, {}}};
    for (const auto& c : cases) {
        const dgx::algo::RegexProg prog(c.pat, c.fold);
        REQUIRE_EQ(dgx::algo::MatchRegex(col, prog, List(all)).Uids, c.want, c.test);
        // the trigram branch: the same candidates as one row
        REQUIRE_EQ(dgx::algo::MatchRegex(col, prog, List(V{}), {List(all)}).Uids, c.want, c.test);
    }
    // a uid without a value, and (?-m): ^ is \A
    const dgx::algo::RegexProg anchored("(?-m)^b");
    dgx::algo::StrColumn lines{{3, 5}, {{"a\nb"}, {"b\na"}}};
    REQUIRE_EQ(dgx::algo::MatchRegex(lines, anchored, List(V{3, 5, 9})).Uids, V{5}, "(?-m)^");
    const std::string too_many_states(5000, 'a');  // a literal's DFA has a state per byte
    const struct { std::string pat; int code; } refused[] = {{"\\bx", DGX_ERR_ARG}, {"a**", DGX_ERR_ARG},
                                                              {"a{1001}", DGX_ERR_ARG}, {too_many_states, DGX_ERR_CAP}};
    for (const auto& r : refused) {
        int code = 0;
        try {
            dgx::algo::RegexProg p(r.pat);
        } catch (const dgx::Error& e) {
            code = e.code;
        }
        REQUIRE_EQ(code, r.code, r.pat.substr(0, 16).c_str());
    }
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
