// Known-answer tests of algo::UidsForRegex in the C++ host mirror (include/dgx_algo.hpp): the trees of /abcd/,
// /abc|def/ and /abc(de|fg)h/ over pack and list leaves, after 0 and after a uid.  Built and run by
// tests/test_cpp_trigram_mirror.py on a GPU box.
#include <cstdio>

#include "dgx_algo.hpp"

using dgx::algo::QueryNode;
using dgx::algo::TrigramLeaf;
using dgx::pb::List;
using V = std::vector<uint64_t>;

static int failures = 0;
#define REQUIRE_EQ(got, want, what)                                                                  \
    do {                                                                                             \
        if ((got) != (want)) { ++failures; std::printf("FAIL %s (line %d)\n", what, __LINE__); }    \
    } while (0)

// a pack from its uvarint deltas (every delta below 128 is one byte)
static dgx::pb::UidPack pack_of(const V& uids) {
    std::vector<uint8_t> b;
    uint64_t last = 0;
    for (uint64_t u : uids) { b.push_back((uint8_t)(u - last)); last = u; }
    return dgx::codec::EncodeFromBuffer(b, 256);
}

int main() {
    if (dgx_init(-1) != DGX_OK) { std::printf("no device: %s\n", dgx_last_error()); return 2; }
    const auto abc = pack_of({1, 2, 5, 8, 9, 12}), bcd = pack_of({2, 3, 5, 9, 11});
    List def_{V{2, 4, 9, 20}}, bcf{V{5, 12}};
    const std::vector<TrigramLeaf> leaves = {{&abc, nullptr}, {&bcd, nullptr}, {nullptr, &def_}, {nullptr, &bcf},
                                             {nullptr, nullptr}};
    // /abcd/: abc AND bcd
    REQUIRE_EQ(dgx::algo::UidsForRegex({{DGX_QAND, {0, 1}, {}}}, leaves, 0).Uids, V({2, 5, 9}), "abcd");
    REQUIRE_EQ(dgx::algo::UidsForRegex({{DGX_QAND, {0, 1}, {}}}, leaves, 2).Uids, V({5, 9}), "abcd after 2");
    // /abc|def/: abc OR def
    REQUIRE_EQ(dgx::algo::UidsForRegex({{DGX_QOR, {0, 2}, {}}}, leaves, 0).Uids, V({1, 2, 4, 5, 8, 9, 12, 20}), "abc|def");
    // /abc(de|fg)h/ written as abc AND (bcd OR bcf), an empty leaf in the OR
    const std::vector<QueryNode> t = {{DGX_QAND, {0}, {1}}, {DGX_QOR, {1, 3, 4}, {}}};
    REQUIRE_EQ(dgx::algo::UidsForRegex(t, leaves, 0).Uids, V({2, 5, 9, 12}), "abc(de|fg)h");
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
