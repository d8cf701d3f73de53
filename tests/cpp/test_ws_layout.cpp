// Known-answer tests of dgraph_b200/csrc/ws_layout.hpp, the byte layout of a call's device workspace.
#include <cstdint>
#include <cstdio>
#include <initializer_list>

#include "ws_layout.hpp"

using dgx::WsLayout;

static int failures = 0;
#define EXPECT(c)                                                  \
    do {                                                           \
        if (!(c)) {                                                \
            std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c); \
            ++failures;                                            \
        }                                                          \
    } while (0)

struct Job { uint64_t a, b, c; uint32_t d; };          // 32 bytes, 8-aligned
struct alignas(32) Wide { unsigned char b[40]; };       // 64 bytes, 32-aligned

static void mixed_layout() {
    WsLayout L;
    const size_t jobs = L.add<Job>(WsLayout::kCopied, 3);           // [0, 96)
    const size_t rows = L.add<uint64_t>(WsLayout::kCopied, 5);      // [96, 136)
    const size_t mode = L.add<unsigned char>(WsLayout::kCopied, 7); // [144, 151)
    const size_t vlo = L.add<uint32_t>(WsLayout::kZeroed, 5);       // [160, 180)
    const size_t none = L.add<uint64_t>(WsLayout::kZeroed, 0);      // [192, 192)
    const size_t tick = L.add<uint32_t>(WsLayout::kZeroed, 2);      // [192, 200)
    const size_t stop = L.add<uint64_t>(WsLayout::kOnes, 3);        // [208, 232)
    const size_t wide = L.add<Wide>(WsLayout::kPlain, 1);           // [256, 320)
    const size_t last = L.add<uint64_t>(WsLayout::kPlain, 9);       // [320, 392)
    EXPECT(L.ok);
    EXPECT(jobs == 0 && rows == 96 && mode == 144);
    EXPECT(vlo == 160 && none == 192 && tick == 192);
    EXPECT(stop == 208 && wide == 256 && last == 320);
    EXPECT(L.bytes == 392);
    for (size_t off : {jobs, rows, mode, vlo, none, tick, stop, last}) EXPECT(off % 16 == 0);
    EXPECT(wide % alignof(Wide) == 0);
    // the copy covers the tables, each memset its section, and nothing else
    EXPECT(L.begin(WsLayout::kCopied) == 0 && L.end(WsLayout::kCopied) == 151);
    EXPECT(L.begin(WsLayout::kZeroed) == 160 && L.end(WsLayout::kZeroed) == 200);
    EXPECT(L.begin(WsLayout::kOnes) == 208 && L.end(WsLayout::kOnes) == 232);
    EXPECT(L.begin(WsLayout::kPlain) == 256 && L.end(WsLayout::kPlain) == 392);
}

static void empty_sections() {
    WsLayout L;  // nothing copied, nothing set to ones
    EXPECT(L.add<uint64_t>(WsLayout::kZeroed, 4) == 0);
    EXPECT(L.add<uint32_t>(WsLayout::kPlain, 3) == 32);
    EXPECT(L.ok && L.bytes == 44);
    EXPECT(L.end(WsLayout::kCopied) == 0);
    EXPECT(L.begin(WsLayout::kZeroed) == 0 && L.end(WsLayout::kZeroed) == 32);
    EXPECT(L.begin(WsLayout::kOnes) == L.end(WsLayout::kOnes));
    EXPECT(L.begin(WsLayout::kPlain) == 32 && L.end(WsLayout::kPlain) == 44);

    WsLayout Z;  // only zero-count regions
    Z.add<uint64_t>(WsLayout::kCopied, 0);
    Z.add<uint32_t>(WsLayout::kZeroed, 0);
    Z.add<unsigned char>(WsLayout::kPlain, 0);
    EXPECT(Z.ok && Z.bytes == 0);
    for (int s = 0; s < WsLayout::kSections; ++s) EXPECT(Z.begin(s) == 0 && Z.end(s) == 0);

    WsLayout E;  // no region at all
    EXPECT(E.ok && E.bytes == 0 && E.end(WsLayout::kCopied) == 0 && E.end(WsLayout::kPlain) == 0);
}

static void trailing_sections() {
    WsLayout L;  // a copied table alone: later sections are empty at its end
    L.add<uint64_t>(WsLayout::kCopied, 3);
    EXPECT(L.ok && L.bytes == 24 && L.end(WsLayout::kCopied) == 24);
    for (int s = WsLayout::kZeroed; s < WsLayout::kSections; ++s) EXPECT(L.begin(s) == 24 && L.end(s) == 24);
}

static void section_order() {
    WsLayout A;
    A.add<uint64_t>(WsLayout::kPlain, 1);
    A.add<uint64_t>(WsLayout::kZeroed, 1);  // zeroed after plain
    EXPECT(!A.ok);

    WsLayout B;
    B.add<uint64_t>(WsLayout::kOnes, 1);
    B.add<uint64_t>(WsLayout::kCopied, 1);  // copied after ones
    B.add<uint64_t>(WsLayout::kPlain, 1);   // in order again: the layout stays refused
    EXPECT(!B.ok);

    WsLayout C;
    C.add<uint64_t>(WsLayout::kSections, 1);  // no such section
    EXPECT(!C.ok);

    WsLayout D;  // repeated sections and skipped ones are in order
    D.add<uint64_t>(WsLayout::kCopied, 1);
    D.add<uint64_t>(WsLayout::kCopied, 1);
    D.add<uint64_t>(WsLayout::kPlain, 1);
    D.add<uint64_t>(WsLayout::kPlain, 1);
    EXPECT(D.ok);
}

int main() {
    mixed_layout();
    empty_sections();
    trailing_sections();
    section_order();
    std::printf("OK: %d failure(s)\n", failures);
    return failures ? 1 : 0;
}
