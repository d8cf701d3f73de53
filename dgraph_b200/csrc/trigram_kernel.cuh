// trigram_kernel.cuh -- uidsForRegex (worker/trigram.go:24-102): a regexp()'s AND / OR tree of trigram posting lists
// evaluated in one call.
//
// codesearch turns the pattern into a cindex.Query tree; every trigram of a node is an index posting list read with
// List.Uids, an AND node intersects its trigrams and subs, an OR node unions them.  With the reads' filters folded in,
// the tree is the set formula f(leaf) = S_leaf, f(AND) = ∩ children, f(OR) = ∪ children (DESIGN section 5), where
// S_leaf is the unfiltered List.Uids row of the leaf.  The host plans from bounds alone (bound(AND) = min of its
// children, bound(OR) = their sum): the root's result lies inside the union of its DRIVING leaves (an AND is driven by
// its smallest child, an OR by all of them).  The device then runs:
//   (the unfiltered rows call)  pack leaves decoded as rows, mutable layers resolved (list_uids_unfiltered_kernel.cuh)
//   tg_leaves_kernel            one CTA: every leaf's row (pointer, length) from the rows' device offsets or the list
//                               leaves' offsets, the DGX_MUT_VALUE check of the layers, and the driving rows' offsets
//   tg_gather_kernel            thread per value: the driving rows back to back
//   (merge_matrix.cuh)          the union of the driving rows: the candidates (skipped with one driving leaf)
//   tg_eval_kernel              thread per candidate (a warp per 32 consecutive ones): the tree's pre-order program,
//                               an AND testing its children smallest bound first and stopping at the first miss, an OR
//                               stopping at the first hit; membership is a binary search in the leaf's row -> keep
//   compact_kernel              the kept candidates, in order (compressed_kernel.cuh's look-back compaction)
// When every node is an OR the candidates are the result: the last two stages are skipped, and with one driving leaf
// the gather writes the result itself.
#pragma once

#include "compressed_kernel.cuh"
#include "list_uids_kernel.cuh"

namespace dgx {

struct TgLeaf {  // a leaf's decoded row on the device
    const u64* p;
    u64 n;
};

// One word pair per program entry, in pre-order.  A node: w0 = kTgNode | (kTgAnd for an AND) | the index one past its
// subtree, w1 = its parent's index (kTgNoParent for the root).  A leaf: w0 = the leaf index.
constexpr u32 kTgNode = 1u << 30, kTgAnd = 1u << 31, kTgEndMask = kTgNode - 1, kTgNoParent = 0xffffffffu;
struct TgOp {
    u32 w0, w1;
};

constexpr int TG_NT = 1024;  // tg_leaves_kernel: one CTA

struct TgParams {
    u32 npacks;                  // leaves [0, npacks) are the rows of the unfiltered rows call ...
    u32 nleaves;                 // ... and [npacks, nleaves) the list leaves
    const u64* rows;             // the rows call's values
    const u64* row_off;          // npacks + 1, written on the device by the rows call
    const u64* lists;            // the list leaves, back to back
    const u64* list_off;         // nleaves - npacks + 1
    const unsigned char* flags;  // nmut flags of the layers: DGX_MUT_VALUE is refused
    u64 nmut;
    TgLeaf* leaf;                // nleaves
    const u32* drive;            // ndrive distinct driving leaves
    u32 ndrive;
    u64* drive_off;              // ndrive + 1: the driving rows' offsets in `gathered`
    u64* len_word;               // or null: receives drive_off[ndrive] (the result length when the gather is the result)
    u64 dcap;                    // sum of the driving leaves' bounds: room of gathered, cand and keep
    u64* gathered;
    const TgOp* prog;
    const u64* cand;             // the candidates ...
    const u64* ncand;            // ... and their number (a device word)
    unsigned char* keep;         // dcap: candidate i is in the result
    int* err;
};

// One CTA.  A layer holding a DGX_MUT_VALUE entry empties every leaf and sets the lane's malformed-layer flag.
__global__ void __launch_bounds__(TG_NT) tg_leaves_kernel(const TgParams P) {
    __shared__ u32 warp_sums[TG_NT / 32 + 1];
    const int tid = threadIdx.x;
    int bad = 0;
    for (u64 k = tid; k < P.nmut; k += TG_NT)
        if (P.flags[k] & LU_VALUE) bad = 1;
    bad = __syncthreads_or(bad);
    if (bad && tid == 0) atomicOr(P.err, kLaneErrMut);
    for (u32 i = tid; i < P.nleaves; i += TG_NT) {
        TgLeaf L;
        if (i < P.npacks) {
            L.p = P.rows + P.row_off[i];
            L.n = P.row_off[i + 1] - P.row_off[i];
        } else {
            const u32 j = i - P.npacks;
            L.p = P.lists + P.list_off[j];
            L.n = P.list_off[j + 1] - P.list_off[j];
        }
        if (bad) L.n = 0;
        P.leaf[i] = L;
    }
    __syncthreads();
    // the driving rows' offsets: a block scan per TG_NT leaves (every sum is below 2^32: the plan bounds it)
    u64 carry = 0;
    for (u32 b = 0; b < P.ndrive; b += TG_NT) {
        const u32 i = b + tid;
        const u32 n = i < P.ndrive ? (u32)P.leaf[P.drive[i]].n : 0u;
        u32 total;
        const u32 ex = block_exclusive_scan<TG_NT>(n, warp_sums, &total);
        if (i < P.ndrive) P.drive_off[i] = carry + ex;
        carry += total;
        __syncthreads();  // warp_sums is reused by the next chunk
    }
    if (tid == 0) {
        P.drive_off[P.ndrive] = carry;
        if (P.len_word) *P.len_word = carry;
    }
}

// Thread per value of the driving rows (grid over dcap).
__global__ void __launch_bounds__(256) tg_gather_kernel(const TgParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.dcap || t >= P.drive_off[P.ndrive]) return;
    const u64 d = lower_bound_g(P.drive_off, (u64)P.ndrive + 1, t + 1) - 1;  // the row holding position t
    const TgLeaf L = P.leaf[P.drive[d]];
    P.gathered[t] = L.p[t - P.drive_off[d]];
}

__device__ __forceinline__ bool tg_member(const TgLeaf& L, u64 x) {
    const u64 i = lower_bound_g(L.p, L.n, x);
    return i < L.n && ld_probe(L.p + i) == x;
}

// Thread per candidate (grid over dcap): keep[t] = the root's value at cand[t].  The program is walked without a stack:
// a node's entry holds its end and its parent, so closing a node goes back to its parent's entry.
__global__ void __launch_bounds__(256) tg_eval_kernel(const TgParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.dcap) return;
    if (t >= *P.ncand) {
        P.keep[t] = 0;
        return;
    }
    const u64 x = P.cand[t];
    u32 cur = 0, pc = 1;  // prog[0] is the root, which has a child (a root of bound 0 never reaches the device)
    bool r = false;
    for (;;) {
        const TgOp e = P.prog[pc];
        if (e.w0 & kTgNode) {
            const u32 end = e.w0 & kTgEndMask;
            if (end != pc + 1) {  // open the node: its first child is next
                cur = pc++;
                continue;
            }
            r = false;  // an OR without children is empty (an AND always has one)
            pc = end;
        } else {
            r = tg_member(P.leaf[e.w0], x);
            ++pc;
        }
        // close every node the value r decides or completes
        for (;;) {
            const TgOp f = P.prog[cur];
            const bool is_and = f.w0 & kTgAnd;
            const u32 end = f.w0 & kTgEndMask;
            if (is_and == r && pc != end) break;  // an AND after a hit or an OR after a miss goes on to the next child
            pc = end;
            if (f.w1 == kTgNoParent) {
                P.keep[t] = r;
                return;
            }
            cur = f.w1;
        }
    }
}

}  // namespace dgx
