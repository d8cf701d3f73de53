// merge_kernel.cuh -- batched 2-way sorted union with de-duplication (sm_90a).
//
// Building block of algo.MergeSorted (algo/uidlist.go:448-542): the reference
// pops a k-way heap and drops a value equal to the last one written (:409-412),
// i.e. a sorted union with GLOBAL de-duplication (in-list and cross-list).  Here
// a level of the merge tree is one launch over all pairs of the level; a pair is
// split into balanced merge-path tiles, each tile is merged from shared memory,
// values equal to their predecessor in merged order are dropped, and tile
// outputs are concatenated with a single-pass decoupled look-back that also
// yields the CSR offsets the next level reads its (now shorter) inputs through.
#pragma once

#include "common.cuh"

namespace dgx {

constexpr int M_NT = 256;           // threads per CTA
constexpr int M_VT = 8;             // merged values per thread
constexpr int M_T = M_NT * M_VT;    // merged values per tile

// A sorted run: either a plain array (off == nullptr) or the slice
// base[off[0] .. off[1]) of a previous level's compact output.
struct MRef {
    const u64* base;
    const u64* off;
    u64 len;  // length, or an upper bound when off != nullptr
};
struct MTask {
    u64 tile_base;
    MRef a, b;
};
struct MParams {
    const MTask* tasks;
    u32 ntasks;
    u32 ntiles;
    u64* out;
    u64 out_cap;
    u64* out_off;  // ntasks + 1
    u64* status;
    u32* ticket;
    int* err;
};

__device__ __forceinline__ void mref_resolve(const MRef& r, const u64*& p, u64& n) {
    if (r.off) {
        u64 s = ld_relaxed(r.off), e = ld_relaxed(r.off + 1);
        p = r.base + s;
        n = e - s;
    } else {
        p = r.base;
        n = r.len;
    }
}

// Merge-path split of diagonal d (A first on ties): number of A values among the
// first d merged values.  Warp-cooperative 32-ary search over global memory.
__device__ __forceinline__ u64 warp_merge_path_g(const u64* __restrict__ A, u64 la,
                                                 const u64* __restrict__ B, u64 lb, u64 d, int lane) {
    u64 lo = d > lb ? d - lb : 0;
    u64 hi = d < la ? d : la;  // answer in [lo, hi]; "before(i)" = A[i] <= B[d-1-i]
    while (hi - lo > 32) {
        u64 stride = (hi - lo) >> 5;
        u64 i = lo + (u64)(lane + 1) * stride - 1;
        bool before = ld_probe(A + i) <= ld_probe(B + (d - 1 - i));
        unsigned c = __popc(__ballot_sync(0xffffffffu, before));
        u64 nlo = lo + (u64)c * stride;
        if (c < 32) hi = lo + (u64)(c + 1) * stride - 1;
        lo = nlo;
    }
    u64 i = lo + lane;
    bool before = false;
    if (i < hi) before = ld_probe(A + i) <= ld_probe(B + (d - 1 - i));
    return lo + __popc(__ballot_sync(0xffffffffu, before));
}

__global__ void __launch_bounds__(M_NT) merge_kernel(const MParams P) {
    __shared__ __align__(16) u64 s_in[M_T + 2];
    __shared__ u64 s_split[2];
    __shared__ u64 s_prefix;
    __shared__ u32 s_scan[M_NT / 32 + 1];
    __shared__ u32 s_tile;

    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(P.ticket, 1u);
    __syncthreads();
    const u32 tile = s_tile;

    u32 q;
    {
        u32 lo = 0, hi = P.ntasks;
        while (hi - lo > 1) {
            u32 mid = (lo + hi) >> 1;
            if (P.tasks[mid].tile_base <= (u64)tile) lo = mid; else hi = mid;
        }
        q = lo;
    }
    const u64 tile_base = P.tasks[q].tile_base;
    const u64* A; const u64* B; u64 la, lb;
    mref_resolve(P.tasks[q].a, A, la);
    mref_resolve(P.tasks[q].b, B, lb);
    const u64 total = la + lb;
    u64 d0 = (u64)(tile - tile_base) * M_T;
    u64 d1 = d0 + M_T;
    if (d0 > total) d0 = total;
    if (d1 > total) d1 = total;

    if (wid < 2) {
        u64 d = wid == 0 ? d0 : d1;
        u64 s = warp_merge_path_g(A, la, B, lb, d, lane);
        if (lane == 0) s_split[wid] = s;
    }
    __syncthreads();
    const u64 ai0 = s_split[0], ai1 = s_split[1];
    const u64 bi0 = d0 - ai0, bi1 = d1 - ai1;
    const int na = (int)(ai1 - ai0), nb = (int)(bi1 - bi0), nt = na + nb;

    // predecessor (in merged order) of the tile's first value
    bool has_pred = false;
    u64 pred = 0;
    if (tid == 0) {
        if (ai0 > 0) { pred = ld_probe(A + ai0 - 1); has_pred = true; }
        if (bi0 > 0) { u64 pb = ld_probe(B + bi0 - 1); if (!has_pred || pb > pred) pred = pb; has_pred = true; }
    }
    for (int i = tid; i < na; i += M_NT) s_in[i] = ld_stream(A + ai0 + i);
    for (int i = tid; i < nb; i += M_NT) s_in[na + i] = ld_stream(B + bi0 + i);
    __syncthreads();

    const u64* sA = s_in;
    const u64* sB = s_in + na;
    // per-thread merge path over shared memory
    int diag = tid * M_VT; if (diag > nt) diag = nt;
    int lo = diag > nb ? diag - nb : 0, hi = diag < na ? diag : na;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (sA[mid] <= sB[diag - 1 - mid]) lo = mid + 1; else hi = mid;
    }
    int ai = lo, bi = diag - lo;
    if (tid > 0 && diag > 0) {
        has_pred = true;
        if (ai > 0) pred = sA[ai - 1];
        if (bi > 0) { u64 pb = sB[bi - 1]; if (ai == 0 || pb > pred) pred = pb; }
    }
    u64 vals[M_VT];
    unsigned keep = 0;
    u64 last = pred;
    bool have_last = has_pred;
#pragma unroll
    for (int s = 0; s < M_VT; ++s) {
        if (diag + s < nt) {
            bool takeA = (bi >= nb) || (ai < na && sA[ai] <= sB[bi]);
            u64 v = takeA ? sA[ai] : sB[bi];
            if (takeA) ++ai; else ++bi;
            vals[s] = v;
            if (!have_last || v != last) keep |= 1u << s;
            last = v;
            have_last = true;
        }
    }
    u32 tile_total;
    u32 off = block_exclusive_scan<M_NT>(__popc(keep), s_scan, &tile_total);
    // scan barriers: all reads of s_in are complete; reuse it as output staging
#pragma unroll
    for (int s = 0; s < M_VT; ++s)
        if ((keep >> s) & 1u) s_in[off++] = vals[s];

    if (wid == 0) {
        u64 ex = lookback_exclusive(P.status, tile, (u64)tile_total, lane);
        if (lane == 0) s_prefix = ex;
    }
    __syncthreads();
    const u64 base = s_prefix;
    if (tid == 0) {
        if ((u64)tile == tile_base) P.out_off[q] = base;
        if (tile == P.ntiles - 1) P.out_off[P.ntasks] = base + (u64)tile_total;
    }
    if (base + (u64)tile_total > P.out_cap) {
        if (tid == 0) atomicExch(P.err, 1);
    } else {
        for (int i = tid; i < (int)tile_total; i += M_NT) st_stream(P.out + base + i, s_in[i]);
    }
}

}  // namespace dgx
