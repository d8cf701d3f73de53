// sg_filter_kernel.cuh -- a subgraph's @filter tree and its first/offset (query/query.go ProcessGraph :2310-2413 with
// applyPagination :2492-2507 and updateUidMatrix :1425-1439, without order or facets) over its uid matrix in one call.
//
// D0 is the node's DestUIDs as processTask left it, rows its uid matrix.  Every filter runs with SrcUIDs = D0 and the
// node's new dest is D1 = f(root) ∩ D0, so each set only matters inside D0: D0[i] is in D1 iff the tree holds at D0[i],
// with f(LIST leaf) a binary search of the leaf's list, f(COUNT leaf) evalCompare(cmp, c_i, thr) on the count aligned
// with D0[i], AND / OR their children's conjunction / disjunction and NOT the negation of its one child.  The rows are
// then filtered by D1 and cut by x.PageRange(count, offset, len), and the new dest D2 is D1 (no pagination) or the
// D1 values some kept row value hits (MergeSorted of the paged rows: each kept value lies in D1).
//
// The row filter and the page cut are cascade's level kernels (cascade_kernel.cuh) driven as one NEW node whose old
// dest is D0 and whose keep flags are the tree's verdicts: its kept values and row offsets are the outputs themselves.
//   sf_check_kernel    thread per slot: D0, LIST leaves and rows strictly ascend, COUNT offsets and row offsets do not
//                      decrease, row offsets start at 0 and end inside v_cap; the size words of the scans
//   sf_eval_kernel     thread per D0 slot: the pre-order program without a stack -> keep
//   scan_u64_kernel    keep -> D1 ranks
//   cc_filter_kernel   D1 compacted, its length; thread per value: its row and whether it lies in D1
//   scan_u64_kernel    value flags -> ranks in rows
//   cc_page_kernel     the PageRange cut
//   scan_u64_kernel    the paged flags -> output positions
//   cc_compact_kernel  the kept values (not in counts-only mode) and the row offsets
//   sf_mark_kernel     the D1 positions of D2: every D1 value, or those a kept row value hits when paging
//   scan_u64_kernel    marks -> D2 positions
//   sf_out_kernel      D2, its length word and the row counts; a refused call writes the length word 0 and nothing else
// Launches: 11, whatever the rows, values, |D0|, leaves and tree.
#pragma once

#include "cascade_kernel.cuh"  // CcParams, CcNode, CcLevel and the level kernels; scan_u64_kernel

namespace dgx {

constexpr int kLaneErrSgFilter = 1024;  // lane error flag bit: an @filter input is malformed (DGX_ERR_ARG at sync)
constexpr u32 SF_LIST = 0, SF_COUNT = 1;
constexpr u32 SF_LE = 0, SF_GE = 1, SF_LT = 2, SF_GT = 3, SF_EQ = 4;  // worker/compare.go evalCompare

struct SfLeaf {
    const u64* p;        // LIST: the uids
    const u64* len;      // LIST: null, or a device word whose low 32 bits are the length (at most room)
    u64 room;            // LIST: the length when len is null, else the room of p
    const u32* cnt;      // COUNT: c_i = cnt[i] ...
    const u64* off;      // ... or off[i + 1] - off[i]
    u64 sb;              // first check slot: room + 1 slots for a LIST, d0_cap for a COUNT over off, none otherwise
    long long thr;
    u32 kind, cmp;
};

// One word pair per program entry, in pre-order.  An op node: w0 = kSfNode | its op << 28 | the index one past its
// subtree, w1 = its parent's index (kSfNoParent for the root).  A leaf: w0 = the leaf index, w1 = its parent.
constexpr u32 kSfNode = 1u << 31, kSfEndMask = (1u << 28) - 1, kSfNoParent = 0xffffffffu;
constexpr u32 SF_AND = 1, SF_OR = 2, SF_NOT = 3;
struct SfOp {
    u32 w0, w1;
};

struct SfParams {
    const SfLeaf* leaf;
    u32 nleaves;
    const SfOp* prog;
    const u64* d0;
    const u64* d0_len;  // null: d0_cap values; else a device word whose low 32 bits are |D0| (at most d0_cap)
    u64 d0_cap;
    const u64* v_off;   // nrows + 1
    const u64* v;
    u64 nrows, v_cap;
    u64 slots;          // sum of the leaves' check slots
    CcNode* node;       // cascade's one node: ndest receives |D0|
    u64* words;         // [|D0|, v_off[nrows]] for the scans
    int counts_only;
    int paged;          // count or offset set: D2 is the merge of the kept rows
    u64* keep;          // d0_cap
    const u64* d1;      // D1 (cascade's ND) ...
    const u64* n1;      // ... and its length (cascade's NDE[0])
    const u64* fv;      // the kept-value flags after the page cut
    const u64* oo;      // the output row offsets
    u64* mark;          // d0_cap, zeroed
    const u64* mx;      // their scan
    int* bad;
    int* err;
    u64* dest_out;
    u64* dest_len;
    u32* counts;
};

__device__ __forceinline__ void sf_refuse(const SfParams& P) {
    atomicOr(P.bad, 1);
    atomicOr(P.err, kLaneErrSgFilter);
}

__device__ __forceinline__ u64 sf_word_len(const u64* w, u64 room, bool& over) {
    if (!w) return room;
    const u64 n = *w & 0xffffffffull;
    over = n > room;
    return over ? 0 : n;
}

// Grid over max(d0_cap, slots, nrows + 1, v_cap) threads.
__global__ void __launch_bounds__(256) sf_check_kernel(const SfParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool over = false;
    const u64 n0 = sf_word_len(P.d0_len, P.d0_cap, over);
    if (t == 0) {
        if (over) sf_refuse(P);
        P.node->ndest = n0;
        P.words[0] = n0;
        P.words[1] = P.v_off[P.nrows];
    }
    if (t > 0 && t < n0 && P.d0[t - 1] >= P.d0[t]) sf_refuse(P);
    if (t < P.slots) {
        u32 lo = 0, hi = P.nleaves;  // the last leaf whose first slot is <= t
        while (hi - lo > 1) {
            const u32 mid = (lo + hi) >> 1;
            if (P.leaf[mid].sb <= t) lo = mid; else hi = mid;
        }
        const SfLeaf L = P.leaf[lo];
        const u64 j = t - L.sb;
        if (L.kind == SF_LIST) {
            bool lover = false;
            const u64 n = sf_word_len(L.len, L.room, lover);
            if (lover && j == 0) sf_refuse(P);
            if (j > 0 && j < n && L.p[j - 1] >= L.p[j]) sf_refuse(P);
        } else if (j < n0 && L.off[j + 1] < L.off[j]) {
            sf_refuse(P);
        }
    }
    if (t <= P.nrows) {
        const u64 x = P.v_off[t];
        if (t == 0 ? x != 0 : x < P.v_off[t - 1]) sf_refuse(P);
        if (t == P.nrows && x > P.v_cap) sf_refuse(P);
    }
    const u64 nv = min(P.v_off[P.nrows], P.v_cap);
    // only a row start may descend; with v_off[0] != 0 (refused above) the row search could land before the array
    if (t > 0 && t < nv && P.v_off[0] == 0 && P.v[t - 1] >= P.v[t]) {
        const u64 r = lower_bound_g(P.v_off, P.nrows + 1, t + 1) - 1;
        if (P.v_off[r] != t) sf_refuse(P);
    }
}

__device__ __forceinline__ bool sf_leaf_holds(const SfLeaf& L, u64 i, u64 x) {
    if (L.kind == SF_LIST) {
        bool over = false;
        const u64 n = sf_word_len(L.len, L.room, over);
        const u64 j = lower_bound_g(L.p, n, x);
        return j < n && L.p[j] == x;
    }
    const long long c = L.cnt ? (long long)L.cnt[i] : (long long)(L.off[i + 1] - L.off[i]);
    switch (L.cmp) {
        case SF_LE: return c <= L.thr;
        case SF_GE: return c >= L.thr;
        case SF_LT: return c < L.thr;
        case SF_GT: return c > L.thr;
        default: return c == L.thr;
    }
}

// Thread per D0 slot: keep[i] = the root's value at D0[i] (0 past |D0|).  A node's entry holds its end and its parent,
// so closing a node goes back to its parent's entry: an AND stops at its first miss, an OR at its first hit.
__global__ void __launch_bounds__(256) sf_eval_kernel(const SfParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.d0_cap) return;
    if (*P.bad || t >= P.node->ndest) {
        P.keep[t] = 0;
        return;
    }
    const u64 x = P.d0[t];
    u32 cur = kSfNoParent, pc = 0;
    bool r = false;
    for (;;) {
        const SfOp e = P.prog[pc];
        if (e.w0 & kSfNode) {  // open the node: its first child is next (every op node has one)
            cur = pc++;
            continue;
        }
        r = sf_leaf_holds(P.leaf[e.w0], t, x);
        ++pc;
        for (;;) {  // close every node the value r decides or completes
            if (cur == kSfNoParent) {
                P.keep[t] = r;
                return;
            }
            const SfOp f = P.prog[cur];
            const u32 op = (f.w0 >> 28) & 7u, end = f.w0 & kSfEndMask;
            if (op == SF_NOT) r = !r;
            else if ((op == SF_AND) == r && pc != end) break;  // an AND after a hit or an OR after a miss goes on
            pc = end;
            cur = f.w1;
        }
    }
}

// Grid over max(d0_cap, v_cap) threads.
__global__ void __launch_bounds__(256) sf_mark_kernel(const SfParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    const u64 n1 = *P.n1;
    if (!P.paged) {
        if (t < n1) P.mark[t] = 1;
        return;
    }
    if (t < P.v_cap && P.fv[t]) P.mark[lower_bound_g(P.d1, n1, P.v[t])] = 1;
}

// Grid over max(d0_cap, nrows) threads.
__global__ void __launch_bounds__(256) sf_out_kernel(const SfParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) {
        if (t == 0) *P.dest_len = 0;
        return;
    }
    const u64 n1 = *P.n1;
    if (t < n1 && P.mark[t]) P.dest_out[P.mx[t]] = P.d1[t];
    if (t == 0) *P.dest_len = P.mx[n1];
    if (t < P.nrows) P.counts[t] = (u32)(P.oo[t + 1] - P.oo[t]);
}

}  // namespace dgx
