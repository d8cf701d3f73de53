// regex_compile.hpp -- regexp()'s pattern compiled to a line-oriented byte DFA (host only: no CUDA).
//
// handleRegexFunction (worker/task.go:1240-1356) tests each value with matchRegex: len(s) > 0 &&
// re.MatchString(s, true, true) > 0, where re is codesearch's regexp over "(?m)" + pattern (plus "i" for /.../i),
// parsed by Go's regexp/syntax with Perl flags and run as a byte-level DFA one line at a time.  This file restates that
// for a declared subset of the syntax and refuses everything else (DGX_ERR_ARG), so a caller keeps its own path:
//   parse    (the "(?m)" prefix clears Go's OneLine; a later (?-m) sets it again, and ^ / $ then read as \A / \z)
//            literals and escapes, '.', bracket classes (ranges, negation, Perl and ASCII classes inside), \d \w \s and
//            negations, [[:name:]], groups ( (?: (?flags) (?flags:, alternation, * + ? and lazy forms, {n} {n,}
//            {n,m} up to 1000 with Go's nested-repeat limit, ^ $ \A \z.  (?i) folds ASCII letters and the two
//            non-ASCII runes in an ASCII letter's orbit (K U+212A, long s U+017F); a folded item holding any other
//            non-ASCII rune is refused, as are \p, \b, \B, \Q, octal escapes, named groups and a literal '{'.
//   NFA      Thompson construction over bytes: a rune range becomes the UTF-8 byte sequences of its scalar values
//            (surrogates excluded), so an invalid UTF-8 byte matches nothing, not even '.' or a negated class.
//   DFA      subset construction, unanchored, one line at a time: a state is a set of NFA nodes plus the assertions
//            that hold there (^ and \A only at a line's start state).  '\n' ends the line: $ holds, and the line either
//            matched or the walk restarts at the line start state.  codesearch reports a match at the end of its line,
//            so a match in an empty first line reports offset 0, which matchRegex counts as no match: that edge goes
//            to the dead state.  A match anywhere else is final, so the accepting state absorbs.
// States: 0 dead, 1 accept (both absorbing), 2 the text's start, 3 a later line's start.  Bytes fall into classes
// that every state treats alike; '\n' is a class of its own.
#pragma once
#include <algorithm>
#include <cctype>
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <vector>

namespace dgx {
namespace rx {

constexpr int kMaxStates = 4096;      // DGX_REGEX_MAX_STATES
constexpr int kMaxNfa = 200000;       // byte-level NFA nodes (a bound far below Go's own size limit)
constexpr int kMaxDepth = 500;        // group / repetition nesting
constexpr uint64_t kMaxWork = 4000000;  // NFA nodes visited while building the DFA: bounds the compile's host time
constexpr int kMaxRepeat = 1000;      // Go's repeat count limit
constexpr uint8_t kTermAbsorb = 2;    // term[s]: the walk can stop here
constexpr uint8_t kTermAccept = 4;    // term[s]: the value matches if its bytes end here
constexpr uint16_t kDead = 0, kAccept = 1, kStartText = 2, kStartLine = 3;

enum RC { kOK = 0, kRefuse = 1, kTooBig = 2 };

struct Range { uint32_t lo, hi; };

enum Op { OpClass, OpEmpty, OpCat, OpAlt, OpRepeat, OpBOL, OpEOL, OpBOT, OpEOT };

struct Node {
    Op op;
    std::vector<Range> cls;  // OpClass: sorted, disjoint
    int min = 0, max = 0;    // OpRepeat: max -1 is unbounded
    std::vector<int> sub;
};

// Canonical class: sorted, merged.
inline void normalize(std::vector<Range>& c) {
    std::sort(c.begin(), c.end(), [](const Range& a, const Range& b) { return a.lo < b.lo; });
    std::vector<Range> o;
    for (const Range& r : c) {
        if (!o.empty() && r.lo <= o.back().hi + 1) o.back().hi = std::max(o.back().hi, r.hi);
        else o.push_back(r);
    }
    c.swap(o);
}
inline std::vector<Range> negate(const std::vector<Range>& c) {
    std::vector<Range> o;
    uint32_t next = 0;
    for (const Range& r : c) {
        if (r.lo > next) o.push_back({next, r.lo - 1});
        next = r.hi + 1;
    }
    if (next <= 0x10FFFF) o.push_back({next, 0x10FFFF});
    return o;
}

class Parser {
  public:
    std::vector<Node> nodes;
    int rc = kOK;

    Parser(const uint8_t* p, size_t n) : s_(p), n_(n) {}

    // The root, or -1 with rc set.
    int parse(bool fold) {
        if (!valid_utf8()) return fail();
        flags_ = (fold ? kFold : 0);
        const int r = alt(0);
        if (rc) return -1;
        if (i_ != n_) return fail();  // an unmatched ')'
        for (size_t k = 0; k < nodes.size(); ++k)
            if (nodes[k].op == OpRepeat && (nodes[k].min >= 2 || nodes[k].max >= 2) && !repeat_ok((int)k, kMaxRepeat))
                return fail();
        return r;
    }

  private:
    enum { kFold = 1, kDotNL = 2, kOneLine = 4 };  // kOneLine: Go's OneLine, set by (?-m): ^ is \A and $ is \z
    const uint8_t* s_;
    size_t n_, i_ = 0;
    int flags_ = 0;

    int fail() {
        if (!rc) rc = kRefuse;
        return -1;
    }
    int add(Node nd) {
        nodes.push_back(std::move(nd));
        return (int)nodes.size() - 1;
    }
    bool valid_utf8() const {
        for (size_t i = 0; i < n_;) {
            uint32_t r;
            const size_t w = decode(i, &r);
            if (!w) return false;
            i += w;
        }
        return true;
    }
    // A valid UTF-8 rune at i: its width, 0 if invalid.
    size_t decode(size_t i, uint32_t* r) const {
        const uint32_t b0 = s_[i];
        if (b0 < 0x80) { *r = b0; return 1; }
        if (b0 < 0xC2 || b0 > 0xF4) return 0;
        const size_t need = b0 < 0xE0 ? 1 : (b0 < 0xF0 ? 2 : 3);
        if (i + need >= n_) return 0;
        uint32_t lo = 0x80, hi = 0xBF;
        if (b0 == 0xE0) lo = 0xA0;
        else if (b0 == 0xED) hi = 0x9F;
        else if (b0 == 0xF0) lo = 0x90;
        else if (b0 == 0xF4) hi = 0x8F;
        if (s_[i + 1] < lo || s_[i + 1] > hi) return 0;
        for (size_t k = 2; k <= need; ++k)
            if (s_[i + k] < 0x80 || s_[i + k] > 0xBF) return 0;
        uint32_t v = b0 & (need == 1 ? 0x1F : need == 2 ? 0x0F : 0x07);
        for (size_t k = 1; k <= need; ++k) v = (v << 6) | (s_[i + k] & 0x3F);
        *r = v;
        return need + 1;
    }
    uint32_t next_rune() {
        uint32_t r;
        i_ += decode(i_, &r);
        return r;
    }
    // Go's repeatIsValid: nested {n,m} counts multiply to at most 1000.
    bool repeat_ok(int k, int n) const {
        const Node& nd = nodes[k];
        if (nd.op == OpRepeat) {
            int m = nd.max;
            if (m == 0) return true;
            if (m < 0) m = nd.min;
            if (m > n) return false;
            if (m > 0) n /= m;
        }
        for (int c : nd.sub)
            if (!repeat_ok(c, n)) return false;
        return true;
    }

    // (?i) over a class: ASCII letters gain their other case, k / s their non-ASCII orbit member; any other non-ASCII
    // rune would need Unicode's fold tables, so it is refused.
    bool fold(std::vector<Range>& c) {
        std::vector<Range> add;
        for (const Range& r : c) {
            if (r.hi >= 0x80) {
                if (!(r.lo == r.hi && (r.lo == 0x212A || r.lo == 0x17F))) return false;
            }
            for (uint32_t x = r.lo; x <= std::min<uint32_t>(r.hi, 0x7F); ++x) {
                if (x >= 'a' && x <= 'z') add.push_back({x - 32, x - 32});
                if (x >= 'A' && x <= 'Z') add.push_back({x + 32, x + 32});
            }
            auto has = [&](uint32_t x) { return r.lo <= x && x <= r.hi; };
            if (has('k') || has('K') || has(0x212A)) add.insert(add.end(), {{'k', 'k'}, {'K', 'K'}, {0x212A, 0x212A}});
            if (has('s') || has('S') || has(0x17F)) add.insert(add.end(), {{'s', 's'}, {'S', 'S'}, {0x17F, 0x17F}});
        }
        c.insert(c.end(), add.begin(), add.end());
        normalize(c);
        return true;
    }
    int cls_node(std::vector<Range> c, bool neg) {
        normalize(c);
        if ((flags_ & kFold) && !fold(c)) return fail();
        if (neg) c = negate(c);
        Node nd{OpClass};
        nd.cls = std::move(c);
        return add(std::move(nd));
    }

    static void perl(char k, std::vector<Range>& c) {
        switch (k | 0x20) {
            case 'd': c.push_back({'0', '9'}); break;
            case 's': c.insert(c.end(), {{'\t', '\n'}, {'\f', '\r'}, {' ', ' '}}); break;
            case 'w': c.insert(c.end(), {{'0', '9'}, {'A', 'Z'}, {'_', '_'}, {'a', 'z'}}); break;
        }
    }
    static bool posix(const std::string& name, std::vector<Range>& c) {
        static const std::map<std::string, std::vector<Range>> tab = {
            {"alnum", {{'0', '9'}, {'A', 'Z'}, {'a', 'z'}}}, {"alpha", {{'A', 'Z'}, {'a', 'z'}}},
            {"ascii", {{0, 0x7F}}}, {"blank", {{'\t', '\t'}, {' ', ' '}}}, {"cntrl", {{0, 0x1F}, {0x7F, 0x7F}}},
            {"digit", {{'0', '9'}}}, {"graph", {{'!', '~'}}}, {"lower", {{'a', 'z'}}}, {"print", {{' ', '~'}}},
            {"punct", {{'!', '/'}, {':', '@'}, {'[', '`'}, {'{', '~'}}}, {"space", {{'\t', '\r'}, {' ', ' '}}},
            {"upper", {{'A', 'Z'}}}, {"word", {{'0', '9'}, {'A', 'Z'}, {'a', 'z'}, {'_', '_'}}},
            {"xdigit", {{'0', '9'}, {'A', 'F'}, {'a', 'f'}}}};
        auto it = tab.find(name);
        if (it == tab.end()) return false;
        c.insert(c.end(), it->second.begin(), it->second.end());
        return true;
    }

    // One escaped rune after '\\' (the '\\' consumed): its value, or -1 refused.
    int64_t escape_rune() {
        if (i_ >= n_) return -1;
        const uint32_t c = s_[i_];
        if (c < 0x80 && !isalnum((int)c)) { ++i_; return c; }  // escaped punctuation
        ++i_;
        switch (c) {
            case 'a': return 7;
            case 'f': return 12;
            case 't': return 9;
            case 'n': return 10;
            case 'r': return 13;
            case 'v': return 11;
            case 'x': {
                if (i_ >= n_) return -1;
                uint64_t v = 0;
                if (s_[i_] == '{') {
                    ++i_;
                    size_t d = 0;
                    while (i_ < n_ && isxdigit(s_[i_]) && d < 8) { v = v * 16 + hexv(s_[i_++]); ++d; }
                    if (!d || i_ >= n_ || s_[i_] != '}' || v > 0x10FFFF) return -1;
                    ++i_;
                    return (int64_t)v;
                }
                if (i_ + 1 >= n_ || !isxdigit(s_[i_]) || !isxdigit(s_[i_ + 1])) return -1;
                v = hexv(s_[i_]) * 16 + hexv(s_[i_ + 1]);
                i_ += 2;
                return (int64_t)v;
            }
        }
        return -1;
    }
    static uint32_t hexv(uint8_t c) { return c <= '9' ? c - '0' : (c | 0x20) - 'a' + 10; }

    int bracket() {  // after '['
        bool neg = false;
        if (i_ < n_ && s_[i_] == '^') { neg = true; ++i_; }
        std::vector<Range> c;
        bool first = true;
        for (;;) {
            if (i_ >= n_) return fail();  // missing ']'
            if (s_[i_] == ']' && !first) { ++i_; break; }
            first = false;
            if (s_[i_] == '[' && i_ + 1 < n_ && s_[i_ + 1] == ':') {
                size_t e = i_ + 2;
                while (e + 1 < n_ && !(s_[e] == ':' && s_[e + 1] == ']')) ++e;
                if (e + 1 >= n_) return fail();
                std::string name((const char*)s_ + i_ + 2, e - i_ - 2);
                bool pn = !name.empty() && name[0] == '^';
                if (pn) name.erase(0, 1);
                std::vector<Range> sub;
                if (!posix(name, sub)) return fail();
                normalize(sub);
                if (pn) sub = negate(sub);
                c.insert(c.end(), sub.begin(), sub.end());
                i_ = e + 2;
                continue;
            }
            uint32_t lo;
            if (s_[i_] == '\\') {
                ++i_;
                if (i_ < n_ && strchr("dDsSwW", s_[i_]) && s_[i_]) {
                    std::vector<Range> sub;
                    perl((char)s_[i_], sub);
                    normalize(sub);
                    if (isupper(s_[i_])) sub = negate(sub);
                    ++i_;
                    c.insert(c.end(), sub.begin(), sub.end());
                    continue;
                }
                const int64_t r = escape_rune();
                if (r < 0) return fail();
                lo = (uint32_t)r;
            } else {
                lo = next_rune();
            }
            uint32_t hi = lo;
            if (i_ + 1 < n_ && s_[i_] == '-' && s_[i_ + 1] != ']') {
                ++i_;
                if (s_[i_] == '\\') {
                    ++i_;
                    const int64_t r = escape_rune();
                    if (r < 0) return fail();
                    hi = (uint32_t)r;
                } else {
                    hi = next_rune();
                }
                if (hi < lo) return fail();  // invalid character class range
            }
            c.push_back({lo, hi});
        }
        return cls_node(std::move(c), neg);
    }

    // {n}, {n,}, {n,m} at i_ ('{' there): true with min / max set, i_ past '}'.
    bool counts(int* mn, int* mx) {
        size_t j = i_ + 1;
        auto num = [&](int* v) {
            const size_t b = j;
            long long x = 0;
            while (j < n_ && isdigit(s_[j]) && j - b < 9) x = x * 10 + (s_[j++] - '0');
            if (j == b || (j - b > 1 && s_[b] == '0') || (j < n_ && isdigit(s_[j]))) return false;
            *v = (int)x;
            return true;
        };
        if (!num(mn)) return false;
        *mx = *mn;
        if (j < n_ && s_[j] == ',') {
            ++j;
            if (j < n_ && s_[j] == '}') *mx = -1;
            else if (!num(mx)) return false;
        }
        if (j >= n_ || s_[j] != '}') return false;
        i_ = j + 1;
        return true;
    }

    int alt(int depth) {
        if (depth > kMaxDepth) return fail();
        std::vector<int> alts{concat(depth)};
        while (!rc && i_ < n_ && s_[i_] == '|') {
            ++i_;
            alts.push_back(concat(depth));
        }
        if (rc) return -1;
        if (alts.size() == 1) return alts[0];
        Node nd{OpAlt};
        nd.sub = alts;
        return add(std::move(nd));
    }

    int concat(int depth) {
        std::vector<int> items;
        bool last_flags = false;  // a flag group just ended: a repetition operator next is refused
        while (!rc && i_ < n_ && s_[i_] != '|' && s_[i_] != ')') {
            const uint8_t c = s_[i_];
            if (c == '*' || c == '+' || c == '?' || c == '{') {
                if (items.empty() || last_flags) return fail();  // missing argument to repetition operator
                int mn, mx;
                if (c == '{') {
                    if (!counts(&mn, &mx)) return fail();  // Go takes a malformed '{' as a literal: refused here
                    if (mn > kMaxRepeat || mx > kMaxRepeat || (mx >= 0 && mn > mx)) return fail();
                } else {
                    ++i_;
                    mn = c == '+' ? 1 : 0;
                    mx = c == '?' ? 1 : -1;
                }
                if (i_ < n_ && s_[i_] == '?') ++i_;  // lazy: the same set of matches
                if (i_ < n_ && (s_[i_] == '*' || s_[i_] == '+' || s_[i_] == '?' || s_[i_] == '{'))
                    return fail();  // invalid nested repetition operator
                Node nd{OpRepeat};
                nd.min = mn;
                nd.max = mx;
                nd.sub = {items.back()};
                items.back() = add(std::move(nd));
                continue;
            }
            last_flags = false;
            int a = -1;
            if (c == '(') {
                ++i_;
                const int saved = flags_;
                if (i_ < n_ && s_[i_] == '?') {
                    ++i_;
                    int f = flags_, sign = 1;
                    bool saw = false;
                    for (;;) {
                        if (i_ >= n_) return fail();
                        const uint8_t k = s_[i_++];
                        if (k == 'i' || k == 'm' || k == 's' || k == 'U') {
                            const int bit = k == 'i' ? kFold : k == 's' ? kDotNL : k == 'm' ? kOneLine : 0;  // U: no effect
                            const bool on = k == 'm' ? sign < 0 : sign > 0;  // m clears OneLine, -m sets it
                            f = on ? (f | bit) : (f & ~bit);
                            saw = true;
                        } else if (k == '-') {
                            if (sign < 0) return fail();
                            sign = -1;
                            saw = false;
                        } else if (k == ':' || k == ')') {
                            if (sign < 0 && !saw) return fail();
                            if (k == ')') {  // (?flags): the rest of the enclosing group
                                flags_ = f;
                                last_flags = true;
                                break;
                            }
                            flags_ = f;
                            a = alt(depth + 1);
                            flags_ = saved;
                            if (rc) return -1;
                            if (i_ >= n_ || s_[i_] != ')') return fail();
                            ++i_;
                            break;
                        } else {
                            return fail();  // named groups and anything else
                        }
                    }
                    if (a < 0) continue;
                } else {
                    a = alt(depth + 1);
                    flags_ = saved;
                    if (rc) return -1;
                    if (i_ >= n_ || s_[i_] != ')') return fail();  // missing ')'
                    ++i_;
                }
            } else if (c == '[') {
                ++i_;
                a = bracket();
            } else if (c == '.') {
                ++i_;
                std::vector<Range> r = (flags_ & kDotNL) ? std::vector<Range>{{0, 0x10FFFF}}
                                                         : std::vector<Range>{{0, 9}, {11, 0x10FFFF}};
                Node nd{OpClass};
                nd.cls = r;
                a = add(std::move(nd));
            } else if (c == '^') {
                ++i_;
                a = add(Node{(flags_ & kOneLine) ? OpBOT : OpBOL});
            } else if (c == '$') {
                ++i_;
                a = add(Node{(flags_ & kOneLine) ? OpEOT : OpEOL});
            } else if (c == '\\') {
                ++i_;
                if (i_ >= n_) return fail();  // trailing backslash
                const uint8_t e = s_[i_];
                if (e == 'A') { ++i_; a = add(Node{OpBOT}); }
                else if (e == 'z') { ++i_; a = add(Node{OpEOT}); }
                else if (strchr("dDsSwW", e) && e) {
                    ++i_;
                    std::vector<Range> r;
                    perl((char)e, r);
                    a = cls_node(r, isupper(e));
                } else {
                    const int64_t r = escape_rune();
                    if (r < 0) return fail();
                    a = cls_node({{(uint32_t)r, (uint32_t)r}}, false);
                }
            } else {
                const uint32_t r = next_rune();
                a = cls_node({{r, r}}, false);
            }
            if (rc) return -1;
            items.push_back(a);
        }
        if (rc) return -1;
        if (items.empty()) return add(Node{OpEmpty});
        if (items.size() == 1) return items[0];
        Node nd{OpCat};
        nd.sub = items;
        return add(std::move(nd));
    }
};

// ----- byte NFA -----
enum NKind : uint8_t { NByte, NSplit, NEps, NAssert, NMatch };
enum Assert : uint8_t { AsBOL = 1, AsEOL = 2, AsBOT = 4, AsEOT = 8 };

struct NNode {
    NKind k;
    uint8_t lo = 0, hi = 0;  // NByte
    uint8_t as = 0;          // NAssert
    int out = -1, out2 = -1;
};

class Nfa {
  public:
    std::vector<NNode> n;
    int rc = kOK;

    int node(NNode x) {
        if ((int)n.size() >= kMaxNfa) { rc = kTooBig; return 0; }
        n.push_back(x);
        return (int)n.size() - 1;
    }

    // The fragment of AST node k whose exit is `next`: its entry.
    int comp(const std::vector<Node>& ast, int k, int next) {
        if (rc) return next;
        const Node& a = ast[k];
        switch (a.op) {
            case OpEmpty: return next;
            case OpBOL: case OpEOL: case OpBOT: case OpEOT: {
                NNode x{NAssert};
                x.as = a.op == OpBOL ? AsBOL : a.op == OpEOL ? AsEOL : a.op == OpBOT ? AsBOT : AsEOT;
                x.out = next;
                return node(x);
            }
            case OpCat: {
                int e = next;
                for (size_t i = a.sub.size(); i-- > 0;) e = comp(ast, a.sub[i], e);
                return e;
            }
            case OpAlt: {
                int e = comp(ast, a.sub.back(), next);
                for (size_t i = a.sub.size() - 1; i-- > 0;) {
                    NNode s{NSplit};
                    s.out = comp(ast, a.sub[i], next);
                    s.out2 = e;
                    e = node(s);
                }
                return e;
            }
            case OpRepeat: {
                int e = next;
                if (a.max < 0) {  // x{min,}: x* after min copies
                    NNode s{NSplit};
                    const int sp = node(s);
                    if (rc) return next;
                    const int body = comp(ast, a.sub[0], sp);
                    n[sp].out = body;
                    n[sp].out2 = next;
                    e = sp;
                } else {
                    for (int i = 0; i < a.max - a.min && !rc; ++i) {  // (x(x(...)?)?)?
                        NNode s{NSplit};
                        s.out = comp(ast, a.sub[0], e);
                        s.out2 = next;
                        e = node(s);
                    }
                }
                for (int i = 0; i < a.min && !rc; ++i) e = comp(ast, a.sub[0], e);
                return e;
            }
            case OpClass: {
                // every UTF-8 byte sequence of the class's scalar values, as alternatives into `next`
                std::vector<std::vector<std::pair<uint8_t, uint8_t>>> seqs;
                for (const Range& r : a.cls) {
                    if (r.lo <= 0xD7FF) utf8_seqs(r.lo, std::min<uint32_t>(r.hi, 0xD7FF), seqs);
                    if (r.hi >= 0xE000) utf8_seqs(std::max<uint32_t>(r.lo, 0xE000), r.hi, seqs);
                }
                int e = -1;
                for (const auto& sq : seqs) {
                    int in = next;
                    for (size_t i = sq.size(); i-- > 0;) {
                        NNode b{NByte};
                        b.lo = sq[i].first;
                        b.hi = sq[i].second;
                        b.out = in;
                        in = node(b);
                    }
                    if (e < 0) { e = in; continue; }
                    NNode s{NSplit};
                    s.out = in;
                    s.out2 = e;
                    e = node(s);
                }
                if (e < 0) {  // an empty class matches nothing: a byte range no byte is in
                    NNode b{NByte};
                    b.lo = 1;
                    b.hi = 0;
                    b.out = next;
                    e = node(b);
                }
                return e;
            }
        }
        return next;
    }

  private:
    static int ulen(uint32_t r) { return r < 0x80 ? 1 : r < 0x800 ? 2 : r < 0x10000 ? 3 : 4; }
    static void enc(uint32_t r, uint8_t* b) {
        const int n = ulen(r);
        if (n == 1) { b[0] = (uint8_t)r; return; }
        for (int i = n - 1; i > 0; --i) { b[i] = (uint8_t)(0x80 | (r & 0x3F)); r >>= 6; }
        b[0] = (uint8_t)((n == 2 ? 0xC0 : n == 3 ? 0xE0 : 0xF0) | r);
    }
    // [lo, hi] (no surrogates) as byte-range sequences, each byte position an independent range.
    static void utf8_seqs(uint32_t lo, uint32_t hi, std::vector<std::vector<std::pair<uint8_t, uint8_t>>>& out) {
        if (lo > hi) return;
        static const uint32_t lim[3] = {0x7F, 0x7FF, 0xFFFF};
        for (uint32_t m : lim)
            if (lo <= m && hi > m) {
                utf8_seqs(lo, m, out);
                utf8_seqs(m + 1, hi, out);
                return;
            }
        const int n = ulen(lo);
        for (int i = 1; i < n; ++i) {
            const uint32_t m = (1u << (6 * i)) - 1;
            if ((lo & ~m) != (hi & ~m)) {
                if ((lo & m) != 0) {
                    utf8_seqs(lo, lo | m, out);
                    utf8_seqs((lo | m) + 1, hi, out);
                    return;
                }
                if ((hi & m) != m) {
                    utf8_seqs(lo, (hi & ~m) - 1, out);
                    utf8_seqs(hi & ~m, hi, out);
                    return;
                }
            }
        }
        uint8_t a[4], b[4];
        enc(lo, a);
        enc(hi, b);
        std::vector<std::pair<uint8_t, uint8_t>> sq;
        for (int i = 0; i < n; ++i) sq.push_back({a[i], b[i]});
        out.push_back(sq);
    }
};

// ----- the DFA -----
struct Prog {
    uint32_t nstates = 0, nclasses = 0;
    uint8_t cls[256] = {};
    std::vector<uint16_t> trans;  // nstates x nclasses
    std::vector<uint8_t> term;    // nstates
};

class Builder {
  public:
    Builder(const Nfa& nfa, int start) : N_(nfa.n), start_(start), seen_(nfa.n.size(), 0) {}

    int build(Prog* P) {
        // byte classes: bytes no NByte range separates, '\n' alone
        std::vector<uint8_t> cut(257, 0);
        cut[0] = cut['\n'] = cut['\n' + 1] = 1;
        for (const NNode& x : N_)
            if (x.k == NByte && x.lo <= x.hi) { cut[x.lo] = 1; cut[x.hi + 1] = 1; }
        std::vector<int> rep;  // a byte of each contiguous class
        int cl = -1;
        uint8_t raw[256];
        for (int b = 0; b < 256; ++b) {
            if (cut[b]) { ++cl; rep.push_back(b); }
            raw[b] = (uint8_t)cl;
        }
        const int nc = cl + 1;
        states_.clear();
        index_.clear();
        add_state({}, 0);  // 0 dead
        add_state({}, 0);  // 1 accept
        std::vector<int> s0 = closure({start_}, AsBOL | AsBOT);
        std::vector<int> s1 = closure({start_}, AsBOL);
        add_state(s0, AsBOL | AsBOT);
        add_state(s1, AsBOL);
        const std::vector<int> restart = closure({start_}, 0);
        std::vector<uint16_t> T;
        std::vector<uint8_t> term;
        for (size_t s = 0; s < states_.size(); ++s) {
            if ((int)states_.size() > kMaxStates) return kTooBig;
            T.resize((s + 1) * nc);
            term.resize(s + 1);
            if (s < 2) {
                for (int c = 0; c < nc; ++c) T[s * nc + c] = (uint16_t)s;
                term[s] = s == kAccept ? (kTermAbsorb | kTermAccept) : kTermAbsorb;
                continue;
            }
            const std::vector<int> set = states_[s].first;  // copy: states_ grows
            const int fl = states_[s].second;
            const bool matched = has_match(set);
            term[s] = has_match(closure(set, fl | AsEOL | AsEOT)) ? kTermAccept : 0;
            for (int c = 0; c < nc; ++c) {
                const int b = rep[c];
                uint16_t to;
                if (b == '\n') {
                    const bool m = matched || has_match(closure(set, fl | AsEOL));
                    to = m ? (s == kStartText ? kDead : kAccept) : kStartLine;
                } else if (matched) {
                    to = kAccept;
                } else {
                    std::vector<int> seeds;
                    work_ += set.size();
                    if (work_ > kMaxWork) return kTooBig;
                    for (int x : set)
                        if (N_[x].k == NByte && N_[x].lo <= b && b <= N_[x].hi) seeds.push_back(N_[x].out);
                    std::vector<int> nx = closure(seeds, 0);
                    nx.insert(nx.end(), restart.begin(), restart.end());
                    std::sort(nx.begin(), nx.end());
                    nx.erase(std::unique(nx.begin(), nx.end()), nx.end());
                    if (work_ > kMaxWork) return kTooBig;
                    to = has_match(nx) ? kAccept : (uint16_t)add_state(nx, 0);
                    if ((int)states_.size() > kMaxStates) return kTooBig;
                }
                T[s * nc + c] = to;
            }
        }
        // merge classes every state treats alike
        std::vector<int> col_of(nc, -1);
        std::vector<int> keep;
        const size_t ns = states_.size();
        for (int c = 0; c < nc; ++c) {
            for (size_t k = 0; k < keep.size() && col_of[c] < 0; ++k) {
                bool same = true;
                for (size_t s = 0; s < ns && same; ++s) same = T[s * nc + c] == T[s * nc + keep[k]];
                if (same) col_of[c] = (int)k;
            }
            if (col_of[c] < 0) { col_of[c] = (int)keep.size(); keep.push_back(c); }
        }
        P->nstates = (uint32_t)ns;
        P->nclasses = (uint32_t)keep.size();
        for (int b = 0; b < 256; ++b) P->cls[b] = (uint8_t)col_of[raw[b]];
        P->trans.resize(ns * keep.size());
        for (size_t s = 0; s < ns; ++s)
            for (size_t k = 0; k < keep.size(); ++k) P->trans[s * keep.size() + k] = T[s * nc + keep[k]];
        P->term = term;
        return kOK;
    }

  private:
    const std::vector<NNode>& N_;
    int start_;
    std::vector<uint32_t> seen_;
    uint32_t epoch_ = 0;
    uint64_t work_ = 0;  // NFA nodes visited so far (kMaxWork)
    std::vector<std::pair<std::vector<int>, int>> states_;
    std::map<std::pair<std::vector<int>, int>, int> index_;

    int add_state(const std::vector<int>& set, int fl) {
        auto key = std::make_pair(set, fl);
        if (states_.size() >= 2) {
            auto it = index_.find(key);
            if (it != index_.end()) return it->second;
        }
        states_.push_back(key);
        const int id = (int)states_.size() - 1;
        if (id >= 2) index_[key] = id;
        return id;
    }
    bool has_match(const std::vector<int>& set) const {
        for (int x : set)
            if (N_[x].k == NMatch) return true;
        return false;
    }
    // Every node reachable from seeds through splits, epsilons and the assertions in fl; sorted.
    std::vector<int> closure(const std::vector<int>& seeds, int fl) {
        ++epoch_;
        std::vector<int> out, stack(seeds.begin(), seeds.end());
        while (!stack.empty()) {
            const int x = stack.back();
            stack.pop_back();
            if (x < 0 || seen_[x] == epoch_) continue;
            seen_[x] = epoch_;
            out.push_back(x);
            ++work_;
            const NNode& nd = N_[x];
            if (nd.k == NSplit) { stack.push_back(nd.out2); stack.push_back(nd.out); }
            else if (nd.k == NEps) stack.push_back(nd.out);
            else if (nd.k == NAssert && (nd.as & fl)) stack.push_back(nd.out);
        }
        std::sort(out.begin(), out.end());
        return out;
    }
};

// pattern -> Prog: kOK, kRefuse (outside the subset, or rejected by Go) or kTooBig (NFA or state cap).
inline int compile(const uint8_t* pat, size_t len, bool fold, Prog* P) {
    Parser ps(pat, len);
    const int root = ps.parse(fold);
    if (root < 0) return ps.rc ? ps.rc : kRefuse;
    Nfa nfa;
    const int m = nfa.node(NNode{NMatch});
    const int start = nfa.comp(ps.nodes, root, m);
    if (nfa.rc) return nfa.rc;
    Builder b(nfa, start);
    return b.build(P);
}

}  // namespace rx
}  // namespace dgx
