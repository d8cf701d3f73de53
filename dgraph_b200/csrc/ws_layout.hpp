// ws_layout.hpp -- byte layout of one call's device workspace (host only: no CUDA, so CPU tests compile it).
//
// A call states each scratch array once, as an element type, a count and a section; the offsets and the total byte
// count follow from those statements.  Sections come in a fixed order:
//   copied  a table the host fills, then uploads in one copy
//   zeroed  cleared by one memset
//   ones    every byte 0xff, set by one memset
//   plain   left uninitialised
// Every region starts at a multiple of 16 bytes, or of alignof(T) when that is larger.  A region declared after a
// later section has begun is a programming error: `ok` turns false and stays so.
#pragma once
#include <cstddef>

namespace dgx {

struct WsLayout {
    enum Section { kCopied, kZeroed, kOnes, kPlain, kSections };
    size_t bytes = 0;       // end of the last region: the workspace's size
    int section = kCopied;  // section of the last region
    bool ok = true;

    // Byte offset of a new region of n elements of `size` bytes, aligned to max(16, align).
    size_t add(int sec, size_t n, size_t size, size_t align) {
        if (sec < section || sec >= kSections) {
            ok = false;
            sec = section;
        }
        const size_t a = align > 16 ? align : 16;
        const size_t off = (bytes + a - 1) / a * a;
        for (int s = section + 1; s <= sec; ++s) begin_[s] = end_[s] = off;
        section = sec;
        bytes = end_[sec] = off + n * size;
        return off;
    }
    template <class T>
    size_t add(int sec, size_t n) { return add(sec, n, sizeof(T), alignof(T)); }

    // [begin(s), end(s)) spans the regions of section s, empty when it has none: what its copy or memset covers.
    size_t begin(int s) const { return s > section ? bytes : begin_[s]; }
    size_t end(int s) const { return s > section ? bytes : end_[s]; }

  private:
    size_t begin_[kSections] = {}, end_[kSections] = {};
};

}  // namespace dgx
