// recurse_kernel.cuh -- one step of @recurse with loop: false (query/recurse.go expandRecurse :96-135) for one
// subgraph: its uid matrix filtered against the edges already taken, the kept edges added to them, and the kept rows
// merged into DestUIDs.
//
// The taken edges of one sg.Attr (a reach set) live in HBM as two u64 arrays from[] / to[], sorted by (from, to), in
// two ping-pong buffers; which buffer is current and its size are two device words (state[0], state[1]) that only the
// last kernel of a step changes, and only when the step was accepted and kept an edge.  A refused step therefore leaves
// the set as it was without any host round trip.  Row i holds the values v[v_off[i] .. v_off[i+1]) of source src[i];
// edge (src[i], x) is kept iff x is in dest (when there is a dest: updateUidMatrix's IntersectWith) and is not in the
// set.  Rows and src strictly ascend, so the kept edges of one step are distinct and already sorted by (from, to).
//   rc_check_kernel     thread per index: src, rows and dest strictly ascend, offsets start at 0, do not decrease and
//                       end inside v
//   rc_locate_kernel    thread per row: the row's slice of the set, equal_range(src[i]) on from[]
//   rc_flags_kernel     thread per value: its row (a search of v_off) and whether it is kept (a search of dest, a
//                       search of the row's slice of to[])
//   scan_u64_kernel     the keep flags -> output positions, the kept count K
//   rc_gather_kernel    thread per value and row: out, out_off, the kept edges' from[], and the offsets the merge reads
//   merge_matrix_impl   DestUIDs = MergeSorted(kept rows) (merge_matrix.cuh)
//   rc_insert_kernel    grid-stride over size + K records: the set and the kept edges merged into the other buffer.
//                       Both sequences are sorted and disjoint, so a record's new place is its own index plus its rank
//                       in the other sequence (a binary search)
//   rc_commit_kernel    one thread: flips the current buffer and adds K to the size when the step was accepted and kept
//                       an edge; writes sizes = {K, |DestUIDs|}, or {0, 0} for a refused step
#pragma once

#include "encode_kernel.cuh"  // scan_u64_kernel, EN_NT, EN_TILE

namespace dgx {

constexpr int kLaneErrRecurse = 32;  // lane error flag bit: a recurse step's input is malformed (DGX_ERR_ARG at sync)
// words of one step: the value count, the kept count, the DestUIDs length
constexpr int RC_W_M = 0, RC_W_K = 1, RC_W_D = 2, RC_WORDS = 3;

struct RcParams {
    const u64* src;
    u64 nrows;
    const u64* v;
    const u64* v_off;   // nrows + 1
    u64 v_cap;
    const u64* dest;    // null: the sg has no filters
    u64 ndest;
    u64* sfrom[2];      // the set's two buffers
    u64* sto[2];
    u64* state;         // [current buffer, size]
    int* bad;           // zeroed
    u64* words;         // RC_WORDS, zeroed
    u64* lo;            // nrows: each row's slice of the current buffer
    u64* hi;
    u32* row;           // v_cap: the row of each value
    u64* keep;          // v_cap
    u64* kex;           // v_cap + 1
    u64* kfrom;         // v_cap: from of each kept edge (its to is out[k])
    u64* out;
    u64* out_off;       // nrows + 1
    u64* w_off;         // nrows + 1: out_off, or zeros for a refused step (what the merge reads)
    u64* sizes;         // [kept, dest_len]
    int* err;
};

__device__ __forceinline__ void rc_refuse(const RcParams& P) {
    atomicOr(P.bad, 1);
    atomicOr(P.err, kLaneErrRecurse);
}

// First index in [0, n) with (f[i], t[i]) >= (a, b) (n if none).
__device__ __forceinline__ u64 rc_lower_pair(const u64* f, const u64* t, u64 n, u64 a, u64 b) {
    u64 lo = 0, hi = n;
    while (lo < hi) {
        const u64 mid = lo + ((hi - lo) >> 1);
        const u64 fm = ld_probe(f + mid);
        if (fm < a || (fm == a && ld_probe(t + mid) < b)) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// Grid over max(nrows + 1, v_cap, ndest) threads.
__global__ void __launch_bounds__(256) rc_check_kernel(const RcParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    const u64 m = P.v_off[P.nrows];
    const bool off_ok = P.v_off[0] == 0 && m <= P.v_cap;
    if (t == 0) {
        bad = !off_ok;
        P.words[RC_W_M] = off_ok ? m : 0;
    }
    if (t < P.nrows) {
        if (t > 0 && P.src[t - 1] >= P.src[t]) bad = true;
        if (P.v_off[t] > P.v_off[t + 1]) bad = true;
    }
    if (P.dest && t > 0 && t < P.ndest && P.dest[t - 1] >= P.dest[t]) bad = true;
    if (off_ok && t > 0 && t < m) {
        const u64 r = lower_bound_g(P.v_off, P.nrows + 1, t + 1) - 1;  // the row holding value t
        if (P.v_off[r] != t && P.v[t - 1] >= P.v[t]) bad = true;
    }
    if (bad) rc_refuse(P);
}

// Thread per row (grid over nrows).
__global__ void __launch_bounds__(256) rc_locate_kernel(const RcParams P) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || i >= P.nrows) return;
    const u64 cur = P.state[0], n = P.state[1];
    const u64* f = P.sfrom[cur];
    const u64 x = P.src[i];
    const u64 lo = lower_bound_g(f, n, x);
    u64 hi = lo;  // first from > x
    for (u64 len = n - lo; len > 0;) {
        const u64 half = len >> 1;
        if (ld_probe(f + hi + half) <= x) { hi += half + 1; len -= half + 1; } else len = half;
    }
    P.lo[i] = lo;
    P.hi[i] = hi;
}

// Thread per value (grid over v_cap).  A refused step keeps nothing.
__global__ void __launch_bounds__(256) rc_flags_kernel(const RcParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 m = P.words[RC_W_M];
    if (t >= m) return;
    if (*P.bad) {
        P.keep[t] = 0;
        return;
    }
    const u64 r = lower_bound_g(P.v_off, P.nrows + 1, t + 1) - 1;
    const u64 x = P.v[t];
    bool k = true;
    if (P.dest) {
        const u64 j = lower_bound_g(P.dest, P.ndest, x);
        k = j < P.ndest && P.dest[j] == x;
    }
    if (k) {
        const u64 lo = P.lo[r], hi = P.hi[r];
        const u64* to = P.sto[P.state[0]];
        const u64 j = lo + lower_bound_g(to + lo, hi - lo, x);
        k = !(j < hi && to[j] == x);
    }
    P.keep[t] = k;
    P.row[t] = (u32)r;
}

// Grid over max(v_cap, nrows + 1) threads.  A refused step writes nothing to out / out_off and zeros to w_off.
__global__ void __launch_bounds__(256) rc_gather_kernel(const RcParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) {
        if (t <= P.nrows) P.w_off[t] = 0;
        return;
    }
    if (t <= P.nrows) {
        const u64 o = P.kex[P.v_off[t]];
        P.w_off[t] = o;
        P.out_off[t] = o;
    }
    if (t < P.words[RC_W_M] && P.keep[t]) {
        const u64 k = P.kex[t];
        P.out[k] = P.v[t];
        P.kfrom[k] = P.src[P.row[t]];
    }
}

// Grid-stride over size + K records: the current buffer and the kept edges (kfrom[k], out[k]) into the other buffer.
// Nothing runs for a refused step or one that kept nothing.
__global__ void __launch_bounds__(256) rc_insert_kernel(const RcParams P) {
    const u64 K = P.words[RC_W_K];
    if (*P.bad || K == 0) return;
    const u64 cur = P.state[0], n = P.state[1];
    const u64 *f = P.sfrom[cur], *to = P.sto[cur];
    u64 *nf = P.sfrom[cur ^ 1], *nt = P.sto[cur ^ 1];
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n + K; i += stride) {
        u64 a, b, pos;
        if (i < n) {
            a = f[i];
            b = to[i];
            pos = i + rc_lower_pair(P.kfrom, P.out, K, a, b);
        } else {
            const u64 k = i - n;
            a = P.kfrom[k];
            b = P.out[k];
            pos = k + rc_lower_pair(f, to, n, a, b);
        }
        nf[pos] = a;
        nt[pos] = b;
    }
}

__global__ void rc_commit_kernel(const RcParams P) {
    if (*P.bad) {
        P.sizes[0] = P.sizes[1] = 0;
        return;
    }
    const u64 K = P.words[RC_W_K];
    if (K) {
        P.state[0] ^= 1;
        P.state[1] += K;
    }
    P.sizes[0] = K;
    P.sizes[1] = P.words[RC_W_D];
}

}  // namespace dgx
