// Known-answer tests of algo::CompareUids / algo::CompareRows in the C++ host mirror (include/dgx_algo.hpp over
// dgx_compare_uids / dgx_compare_rows), on Go's rules for types.CompareVals: NaN and -0 for floats, signed int64,
// datetimes before 1970, bool only under eq, bytewise strings, a list value's row length, the conversion error, and
// Go's index-path row cases.  Built and run by tests/test_cpp_compare_mirror.py on a GPU box.
#include <cmath>
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

static uint64_t f(double d) {
    uint64_t w;
    std::memcpy(&w, &d, 8);
    return w;
}
static uint64_t i(int64_t x) { return (uint64_t)x; }

int main() {
    using dgx::algo::ValColumn;
    using dgx::algo::ValArgs;
    const V all{1, 2, 3, 4};
    ValColumn fl{DGX_VAL_FLOAT64, {1, 2, 3, 4}, {{f(NAN)}, {f(-0.0)}, {f(0.0)}, {f(1.0)}}, {}, {}, {}};
    REQUIRE_EQ(dgx::algo::CompareUids(fl, DGX_SGF_CMP_GE, {{f(0.5)}, {}, {}}, List(all)).Uids, (V{1, 4}), "ge NaN value");
    REQUIRE_EQ(dgx::algo::CompareUids(fl, DGX_SGF_CMP_GT, {{f(0.5)}, {}, {}}, List(all)).Uids, (V{4}), "gt");
    REQUIRE_EQ(dgx::algo::CompareUids(fl, DGX_SGF_CMP_LE, {{f(NAN)}, {}, {}}, List(all)).Uids, all, "le NaN argument");
    REQUIRE_EQ(dgx::algo::CompareUids(fl, DGX_SGF_CMP_EQ, {{f(-0.0), f(NAN)}, {}, {}}, List(all)).Uids, (V{2, 3}), "eq -0");
    REQUIRE_EQ(dgx::algo::CompareUids(fl, DGX_SGF_CMP_BETWEEN, {{f(1.0), f(0.0)}, {}, {}}, List(all)).Uids, (V{1}),
               "between a > b keeps only NaN");
    ValColumn in{DGX_VAL_INT64, {1, 2, 3}, {{i(INT64_MIN)}, {i(INT64_MAX)}, {i(5), i(7), i(5)}}, {}, {}, {}};
    std::vector<uint32_t> rl;
    REQUIRE_EQ(dgx::algo::CompareUids(in, DGX_SGF_CMP_EQ, {{i(5), i(7)}, {}, {}}, List(V{1, 2, 3}), &rl).Uids, (V{3}),
               "eq list");
    REQUIRE_EQ(rl, (std::vector<uint32_t>{0, 0, 3}), "row lengths");
    REQUIRE_EQ(dgx::algo::CompareUids(in, DGX_SGF_CMP_LT, {{i(0)}, {}, {}}, List(V{1, 2, 3})).Uids, (V{1}), "signed");
    ValColumn dt{DGX_VAL_DATETIME, {1, 2}, {{i(-14516064000)}, {0}}, {{0}, {5}}, {}, {}};
    REQUIRE_EQ(dgx::algo::CompareUids(dt, DGX_SGF_CMP_LE, {{0}, {0}, {}}, List(V{1, 2})).Uids, (V{1}), "datetime");
    ValColumn bo{DGX_VAL_BOOL, {1, 2}, {{1}, {0}}, {}, {}, {}};
    REQUIRE_EQ(dgx::algo::CompareUids(bo, DGX_SGF_CMP_GE, {{0}, {}, {}}, List(V{1, 2})).Uids, V{}, "bool ge");
    REQUIRE_EQ(dgx::algo::CompareUids(bo, DGX_SGF_CMP_EQ, {{0}, {}, {}}, List(V{1, 2})).Uids, (V{2}), "bool eq");
    ValColumn st{DGX_VAL_STRING, {1, 2, 3}, {}, {}, {{"a"}, {"ab"}, {std::string("\xff", 1)}}, {}};
    REQUIRE_EQ(dgx::algo::CompareUids(st, DGX_SGF_CMP_LT, {{}, {}, {"ab"}}, List(V{1, 2, 3})).Uids, (V{1}), "string");
    // a conversion error on a candidate is Go's error; off the candidates it is not read
    ValColumn bd{DGX_VAL_INT64, {1, 2}, {{i(1)}, {i(2)}}, {}, {}, {{0}, {1}}};
    REQUIRE_EQ(dgx::algo::CompareUids(bd, DGX_SGF_CMP_GE, {{i(0)}, {}, {}}, List(V{1})).Uids, (V{1}), "bad off");
    try {
        dgx::algo::CompareUids(bd, DGX_SGF_CMP_GE, {{i(0)}, {}, {}}, List(V{1, 2}));
        REQUIRE_EQ(0, 1, "bad on a candidate is refused");
    } catch (const dgx::Error& e) {
        REQUIRE_EQ(e.code, DGX_ERR_ARG, "bad code");
    }
    // the index path: between filters rows 0 and last; a bad value never passes
    const auto rows = dgx::algo::CompareRows(bd, DGX_SGF_CMP_BETWEEN, {{i(0), i(5)}, {}, {}},
                                             {List(V{2, 1}), List(V{2}), List(V{1, 2})}, {0, UINT32_MAX, 0});
    REQUIRE_EQ(rows.size(), 3u, "rows");
    REQUIRE_EQ(rows[0].Uids, (V{1}), "row 0");
    REQUIRE_EQ(rows[1].Uids, (V{2}), "row 1 unchanged");
    REQUIRE_EQ(rows[2].Uids, (V{1}), "row 2");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
