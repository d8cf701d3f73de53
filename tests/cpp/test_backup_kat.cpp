// Known-answer tests of codec::DecodeToBuffer / codec::EncodeFromBuffer in the C++ host mirror (include/dgx_algo.hpp):
// a pack whose first uid is 0, a block whose running sum wraps past 2^64, the nil pack and a malformed stream.
// Built and run by tests/test_cpp_backup_mirror.py on a GPU box.
#include <cstdio>

#include "dgx_algo.hpp"

using dgx::pb::UidPack;
using B = std::vector<uint8_t>;
using V = std::vector<uint64_t>;

static int failures = 0;
#define REQUIRE_EQ(got, want, what)                                                                  \
    do {                                                                                             \
        if ((got) != (want)) { ++failures; std::printf("FAIL %s (line %d)\n", what, __LINE__); }    \
    } while (0)

static UidPack one_block(uint64_t base, uint32_t num, B deltas) {
    UidPack p;
    p.block_size = 256;
    p.base = {base};
    p.num_uids = {num};
    p.delta_off = {0, deltas.size()};
    p.deltas = deltas;
    return p;
}

int main() {
    if (dgx_init(-1) != DGX_OK) { std::printf("no device: %s\n", dgx_last_error()); return 2; }
    const uint64_t M = ~0ull;
    {   // uids {0, 1, 2}: the first uid 0 is written as 00
        const UidPack p = one_block(0, 3, {0x00, 1, 1, 0, 0});
        const B bytes = dgx::codec::DecodeToBuffer(&p);
        REQUIRE_EQ(bytes, B({0x00, 0x01, 0x01}), "DecodeToBuffer {0,1,2}");
        const UidPack q = dgx::codec::EncodeFromBuffer(bytes, 256);
        REQUIRE_EQ(q.base, V({0}), "EncodeFromBuffer {0,1,2} base");
        REQUIRE_EQ(q.num_uids, std::vector<uint32_t>({3}), "EncodeFromBuffer {0,1,2} num");
        REQUIRE_EQ(q.deltas, p.deltas, "EncodeFromBuffer {0,1,2} deltas");
    }
    {   // base 2^64 - 3, delta 5: the running sum wraps to uid 2; the stream's second delta wraps back to 5
        const UidPack p = one_block(M - 2, 2, {0x00, 5, 0, 0, 0});
        const B bytes = dgx::codec::DecodeToBuffer(&p);
        REQUIRE_EQ(bytes, B({0xfd, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0xff, 0x01, 0x05}), "DecodeToBuffer wrap");
        const UidPack q = dgx::codec::EncodeFromBuffer(bytes, 256);  // the upper 32 bits change: two blocks
        REQUIRE_EQ(q.base, V({M - 2, 2}), "EncodeFromBuffer wrap base");
        REQUIRE_EQ(q.num_uids, std::vector<uint32_t>({1, 1}), "EncodeFromBuffer wrap num");
        REQUIRE_EQ(q.delta_off, V({0, 5, 10}), "EncodeFromBuffer wrap delta_off");
        REQUIRE_EQ(q.deltas, B(10, 0), "EncodeFromBuffer wrap deltas");
    }
    {   // nil pack, empty buffer, non-minimal zero
        REQUIRE_EQ(dgx::codec::DecodeToBuffer(nullptr).empty(), true, "DecodeToBuffer nil");
        REQUIRE_EQ(dgx::codec::EncodeFromBuffer(B(), 256).base.empty(), true, "EncodeFromBuffer empty");
        REQUIRE_EQ(dgx::codec::EncodeFromBuffer(B({0x80, 0x00}), 256).base, V({0}), "EncodeFromBuffer 80 00");
    }
    {   // a 10th byte of 02 overflows: where the Go function panics, the mirror throws DGX_ERR_ARG
        int code = 0;
        try {
            dgx::codec::EncodeFromBuffer(B({0x80, 0x80, 0x80, 0x80, 0x80, 0x80, 0x80, 0x80, 0x80, 0x02}), 256);
        } catch (const dgx::Error& e) {
            code = e.code;
        }
        REQUIRE_EQ(code, (int)DGX_ERR_ARG, "EncodeFromBuffer overflow");
    }
    std::printf("%s: %d failure(s)\n", failures ? "FAILED" : "OK", failures);
    return failures ? 1 : 0;
}
