// regex_kernel.cuh -- handleRegexFunction (worker/task.go:1240-1356): regexp(attr, /pattern/)'s candidates tested
// with matchRegex (:1809-1811) over a string value column, in one call.
//
// The candidates are the UidList, or uidsForRegex's trigram rows (trigram_kernel.cuh), and their values are read from
// the same caller-owned column as match() (dgx_str_column).  A candidate is kept when one of its values is not empty
// and the pattern's line-oriented byte DFA (regex_compile.hpp) ends that value in an accepting state.  The device runs:
//   fz_lookup_kernel   match_kernel.cuh's lookup and order checks, unchanged
//   scan_u64_kernel    value counts -> pair offsets: (candidate, value) pairs flattened
//   rx_test_kernel     fixed grid, thread per pair: an empty value fails; a value longer than RX_LONG_BYTES of a DFA
//                      with at most RX_WARP_STATES states is queued for the warp tier; otherwise the thread walks the
//                      value's bytes, read as aligned 16-byte vectors, through the table (in shared memory when it
//                      fits), and stops at an absorbing state
//   rx_long_kernel     fixed grid, warp per queued value: the value's 16-byte segments are cut into 32 chunks, lane l
//                      computes its chunk's map from every DFA state (a state vector, until its live entries agree,
//                      then one walk) and lane 0 composes the 32 maps from the text's start state
//   compact_kernel     the kept candidates, in order (compressed_kernel.cuh's look-back compaction)
// A malformed input sets the call's bad word and the lane's kLaneErrMatch bit, as in match(): every later stage then
// keeps nothing, so the call writes only a zero length.
#pragma once

#include "match_kernel.cuh"

namespace dgx {

constexpr int RX_NT = 256;               // rx_test_kernel and rx_long_kernel: 8 warps per CTA
constexpr int RX_WARP_STATES = 64;       // the warp tier's state bound: a u16 per state and lane in shared memory
constexpr u64 RX_LONG_BYTES = 4096;      // longer values of a small DFA go to the warp tier
constexpr u32 RX_SMEM_TABLE = 32768;     // rx_test_kernel keeps the table in shared memory up to this many bytes
constexpr u32 RX_ABSORB = 2, RX_ACCEPT = 4;  // term[] bits (regex_compile.hpp kTermAbsorb / kTermAccept)
constexpr u32 RX_START = 2;              // the text's start state

struct RxParams {
    FzParams F;  // candidates, column and workspace, as match() lays them out (the query fields unused)
    const unsigned char* cls;  // 256: byte -> class
    const unsigned short* trans;  // nstates x nclasses
    const unsigned char* term;    // nstates
    u32 nstates, nclasses;
    u32 warp;  // nstates <= RX_WARP_STATES: long values take the warp tier
};

// The value's bytes as aligned 16-byte segments: the column's base rounded down, and the value's span inside it.
// Segments are read whole, except the column's first and last, which may hold bytes outside [bytes, bytes + nbytes):
// those are read byte by byte, so no call reads outside the caller's column.
struct RxSpan {
    const uint4* seg;
    u64 lo, hi;      // the value's byte offsets from seg
    u64 clo, chi;    // the column's
};
__device__ __forceinline__ RxSpan rx_span(const unsigned char* bytes, u64 nbytes, u64 b0, u64 len) {
    const uintptr_t a = (uintptr_t)bytes;
    const uintptr_t base = a & ~(uintptr_t)15;
    const u64 off = (u64)(a - base);
    return RxSpan{(const uint4*)base, off + b0, off + b0 + len, off, off + nbytes};
}
__device__ __forceinline__ uint4 rx_load(const RxSpan& sp, u64 g) {
    if (g * 16 >= sp.clo && g * 16 + 16 <= sp.chi) return __ldg(sp.seg + g);
    const unsigned char* p = (const unsigned char*)(sp.seg + g);
    u32 w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 16; ++k)
        if (g * 16 + k >= sp.clo && g * 16 + k < sp.chi) w[k >> 2] |= (u32)__ldg(p + k) << (8 * (k & 3));
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// Walk bytes [q, q + 4) of word x, those inside [lo, hi), from state s.
template <class Tab>
__device__ __forceinline__ u32 rx_word(const Tab& tab, u32 x, u64 q, u64 lo, u64 hi, u32 s) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (q + k >= lo && q + k < hi) s = tab.next(s, (x >> (8 * k)) & 0xFFu);
    return s;
}
// The same over the 16 bytes [q, q + 16) of segment v.
template <class Tab>
__device__ __forceinline__ u32 rx_seg(const Tab& tab, uint4 v, u64 q, u64 lo, u64 hi, u32 s) {
    s = rx_word(tab, v.x, q, lo, hi, s);
    s = rx_word(tab, v.y, q + 4, lo, hi, s);
    s = rx_word(tab, v.z, q + 8, lo, hi, s);
    return rx_word(tab, v.w, q + 12, lo, hi, s);
}

struct RxTab {
    const unsigned char* cls;
    const unsigned short* trans;
    const unsigned char* term;
    u32 nc;
    __device__ __forceinline__ u32 next(u32 s, u32 b) const { return trans[s * nc + cls[b]]; }
};

// Fixed grid, thread per pair; dynamic shared memory holds the table, the class map and term when SMEM.
template <bool SMEM>
__global__ void __launch_bounds__(RX_NT) rx_test_kernel(const RxParams P) {
    extern __shared__ __align__(16) unsigned char rx_smem[];
    RxTab tab{P.cls, P.trans, P.term, P.nclasses};
    if (SMEM) {
        const u32 nt = P.nstates * P.nclasses;
        unsigned short* t = (unsigned short*)rx_smem;
        unsigned char* c = rx_smem + ((nt * 2 + 15) & ~15u);
        for (u32 i = threadIdx.x; i < nt; i += blockDim.x) t[i] = P.trans[i];
        for (u32 i = threadIdx.x; i < 256; i += blockDim.x) c[i] = P.cls[i];
        for (u32 i = threadIdx.x; i < P.nstates; i += blockDim.x) c[256 + i] = P.term[i];
        __syncthreads();
        tab = RxTab{c, t, c + 256, P.nclasses};
    }
    const FzParams& F = P.F;
    if (*(volatile u64*)(F.words + FZ_W_BAD)) return;
    const u64 nc = F.words[FZ_W_N], np = F.words[FZ_W_PAIRS];
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < np && p < F.nvals; p += stride) {
        const u64 c = lower_bound_g(F.pair_off, nc + 1, p + 1) - 1;  // the candidate owning pair p
        const u64 j = F.vlo[c] + (p - F.pair_off[c]);
        const u64 b0 = F.byte_off[j], len = F.byte_off[j + 1] - b0;
        if (len == 0) continue;  // matchRegex: an empty value never matches
        if (P.warp && len > RX_LONG_BYTES) {
            F.longq[atomicAdd((unsigned long long*)(F.words + FZ_W_LONG), 1ull)] = (c << 32) | (j - F.vlo[c]);
            continue;
        }
        const RxSpan sp = rx_span(F.bytes, F.nbytes, b0, len);
        u32 s = RX_START;
        for (u64 q = sp.lo & ~15ull; q < sp.hi && !(tab.term[s] & RX_ABSORB); q += 16)
            s = rx_seg(tab, rx_load(sp, q / 16), q, sp.lo, sp.hi, s);
        if (tab.term[s] & RX_ACCEPT) F.keep[c] = 1;
    }
}

// Fixed grid, warp per queued value (a DFA of at most RX_WARP_STATES states).  maps[w][s][l]: the state lane l's chunk
// leads DFA state s to.
__global__ void __launch_bounds__(RX_NT, 1) rx_long_kernel(const RxParams P) {
    __shared__ unsigned short maps[RX_NT / 32][RX_WARP_STATES][32];
    const FzParams& F = P.F;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const u32 nwarps = gridDim.x * (RX_NT / 32);
    if (*(volatile u64*)(F.words + FZ_W_BAD)) return;
    const u32 nq = (u32)F.words[FZ_W_LONG];  // at most nvals < 2^32
    const RxTab tab{P.cls, P.trans, P.term, P.nclasses};
    const u32 S = P.nstates;
    for (u32 q = blockIdx.x * (RX_NT / 32) + wid; q < nq; q += nwarps) {
        const u64 e = F.longq[q], c = e >> 32, j = F.vlo[c] + (e & 0xFFFFFFFFull);
        const u64 b0 = F.byte_off[j], len = F.byte_off[j + 1] - b0;
        const RxSpan sp = rx_span(F.bytes, F.nbytes, b0, len);
        const u64 g0 = sp.lo / 16, nseg = (sp.hi + 15) / 16 - g0, per = (nseg + 31) / 32;
        const u64 s0 = g0 + (u64)lane * per, s1 = min(s0 + per, g0 + nseg);
        // lane 0 starts at the text's start: one walk; every other lane a vector over all states until it converges
        bool single = lane == 0;
        u32 v = RX_START;
        for (u32 s = 0; s < S; ++s) maps[wid][s][lane] = (unsigned short)s;
        for (u64 g = s0; g < s1; ++g) {
            const uint4 w = rx_load(sp, g);
            if (single) {
                if (tab.term[v] & RX_ABSORB) break;
                v = rx_seg(tab, w, g * 16, sp.lo, sp.hi, v);
                continue;
            }
#pragma unroll 1
            for (u32 s = 0; s < S; ++s) {
                u32 x = maps[wid][s][lane];
                x = rx_word(tab, w.x, g * 16, sp.lo, sp.hi, x);
                x = rx_word(tab, w.y, g * 16 + 4, sp.lo, sp.hi, x);
                x = rx_word(tab, w.z, g * 16 + 8, sp.lo, sp.hi, x);
                maps[wid][s][lane] = (unsigned short)rx_word(tab, w.w, g * 16 + 12, sp.lo, sp.hi, x);
            }
            // converged: every entry not yet absorbed is one state, which one walk carries on
            u32 live = 0xFFFFu;
            bool conv = true;
            for (u32 s = 0; s < S && conv; ++s) {
                const u32 x = maps[wid][s][lane];
                if (tab.term[x] & RX_ABSORB) continue;
                if (live == 0xFFFFu) live = x;
                else conv = x == live;
            }
            if (conv && live != 0xFFFFu) { single = true; v = live; }
            else if (conv) break;  // every entry absorbed
        }
        if (single && lane != 0)
            for (u32 s = 0; s < S; ++s)
                if (!(tab.term[maps[wid][s][lane]] & RX_ABSORB)) maps[wid][s][lane] = (unsigned short)v;
        __syncwarp();
        if (lane == 0) {
            u32 st = v;
            for (int l = 1; l < 32 && !(tab.term[st] & RX_ABSORB); ++l) st = maps[wid][st][l];
            if (tab.term[st] & RX_ACCEPT) F.keep[c] = 1;
        }
        __syncwarp();
    }
}

}  // namespace dgx
