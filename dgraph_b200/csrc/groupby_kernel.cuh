// groupby_kernel.cuh -- @groupby over one uid predicate (query/groupby.go formResult / formGroups / fillGroupedVars):
// the child's uid matrix inverted into `dest uid -> ascending source uids`, restricted to every parent row, each
// parent's groups ordered by (size, key), in one call.
//
// Child row i holds the values v[v_off[i] .. v_off[i+1]) of source src[i]; parent p holds par[par_off[p] ..
// par_off[p+1]).  Row i takes part in parent p iff src[i] is in parent p (IndexOf with the roles swapped: both lists
// strictly ascend), and then every value d of row i adds src[i] to the group (p, d).  The device runs:
//   gb_check_kernel     thread per index: src, rows and dest strictly ascend, offsets do not decrease and end inside
//                       their arrays
//   gb_pairs_kernel     thread per parent value: its parent, that its parent row ascends, its source row (a binary
//                       search of src) and that row's length
//   scan_u64_kernel     the lengths -> edge offsets, the restricted edge count E
//   gb_expand_kernel    thread per edge: key = parent << b_d | rank of the value in dest (not found: refused),
//                       payload = source row; edges are written in (parent, source) order
//   3 x P1 launches     stable LSD radix sort of the edges by key, 8-bit digits: gb_hist_kernel (a tile's digit
//                       counts), scan_u64_kernel (digit-major, so the scan is the scatter base), gb_scatter_kernel
//                       (stable ranks inside the tile).  P1 = ceil((b_p + b_d) / 8)
//   gb_heads_kernel     thread per edge: a group starts where the key changes
//   scan_u64_kernel     the starts -> group indices, the group count G
//   gb_groups_kernel    thread per edge: each group's first edge
//   gb_gkeys_kernel     thread per group: order key parent << b_s | size, payload = group
//   3 x P2 launches     the same radix sort over the groups.  P2 = ceil((b_p + b_s) / 8); they already ascend by key
//                       inside a parent, so the stable sort leaves ties in key order
//   gb_sizes_kernel     thread per ordered group: its size, its position
//   scan_u64_kernel     the sizes -> member offsets
//   gb_write_kernel     thread per edge, group and parent: keys, grp_off, mem_off and the members, or nothing at all
//                       when the input was refused or an output does not fit
// b_p, b_d and b_s are the bit widths of npar - 1, ndest - 1 and nrows: the launch count is 11 + 3 (P1 + P2), set by
// the call's sizes alone.
#pragma once

#include "encode_kernel.cuh"  // scan_u64_kernel, EN_NT, EN_TILE

namespace dgx {

constexpr int kLaneErrGroupBy = 16;  // lane error flag bit: a groupby input is malformed (DGX_ERR_ARG at sync)
constexpr int GB_NT = 256, GB_VT = 8, GB_TILE = GB_NT * GB_VT;  // radix sort tile
constexpr int GB_RADIX = 256, GB_DIGIT_BITS = 8;
constexpr int GB_WARPS = GB_NT / 32;
constexpr int kGbBadArg = 1, kGbBadCap = 2;  // the call's own error word
constexpr u32 kGbNoRow = 0xffffffffu;
// words: the parent value count, the edge count, the group count, the length of a hist scan
constexpr int GB_W_PV = 0, GB_W_E = 1, GB_W_G = 2, GB_W_H = 3, GB_WORDS = 4;

struct GbParams {
    const u64* src;
    u64 nrows;
    const u64* v;
    const u64* v_off;   // nrows + 1
    u64 v_cap;
    const u64* dest;
    u64 ndest;
    const u64* par;
    const u64* par_off; // npar + 1
    u64 npar, par_cap;
    u32 b_d, b_s;       // bits of a dest rank and of a group size
    u64 e_cap;          // room for edges (and groups)
    u64 tiles;          // radix tiles over e_cap: the hist's row length
    u64* words;         // GB_WORDS
    int* bad;           // kGbBadArg | kGbBadCap, zeroed
    u32* prow;          // par_cap: source row of a parent value, kGbNoRow if none
    u32* ppar;          // par_cap: parent of a parent value
    u64* plen;          // par_cap: length of that row
    u64* eoff;          // par_cap + 1
    u64* ek;            // e_cap: edge keys, sorted (where sort 1 leaves them)
    u32* ep;            // e_cap: edge source rows, in the same order
    u64* head;          // e_cap
    u64* gidx;          // e_cap + 1
    u64* gstart;        // e_cap + 1
    u64* gk;            // e_cap: groups' order keys, sorted
    u32* gp;            // e_cap: group of each ordered position
    u64* gsz;           // e_cap
    u64* moff;          // e_cap + 1
    u32* inv;           // e_cap: ordered position of each group
    u64* keys;
    u64* grp_off;
    u64* mem_off;
    u64* members;       // null: counts only
    u64 grp_cap, mem_cap;
    u64* sizes;         // [groups, members]
    int* err;
};

__device__ __forceinline__ void gb_refuse(const GbParams& P) {
    atomicOr(P.bad, kGbBadArg);
    atomicOr(P.err, kLaneErrGroupBy);
}

// Grid over max(nrows + 1, npar + 1, ndest, v_cap) threads.
__global__ void __launch_bounds__(256) gb_check_kernel(const GbParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    if (t == 0) {
        bad = P.v_off[0] != 0 || P.par_off[0] != 0 || P.v_off[P.nrows] > P.v_cap || P.par_off[P.npar] > P.par_cap;
        P.words[GB_W_PV] = bad ? 0 : P.par_off[P.npar];
    }
    if (t < P.nrows) {
        if (t > 0 && P.src[t - 1] >= P.src[t]) bad = true;
        if (P.v_off[t] > P.v_off[t + 1]) bad = true;
    }
    if (t < P.npar && P.par_off[t] > P.par_off[t + 1]) bad = true;
    if (t > 0 && t < P.ndest && P.dest[t - 1] >= P.dest[t]) bad = true;
    const u64 m = P.v_off[P.nrows];
    if (t > 0 && t < m && m <= P.v_cap && P.v_off[0] == 0) {  // offsets from 0: the search lands on a row
        const u64 r = lower_bound_g(P.v_off, P.nrows + 1, t + 1) - 1;  // the row holding value t
        if (P.v_off[r] != t && P.v[t - 1] >= P.v[t]) bad = true;
    }
    if (bad) gb_refuse(P);
}

// Thread per parent value (grid over par_cap).
__global__ void __launch_bounds__(256) gb_pairs_kernel(const GbParams P) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || j >= P.words[GB_W_PV]) return;
    const u64 p = lower_bound_g(P.par_off, P.npar + 1, j + 1) - 1;
    const u64 x = P.par[j];
    if (j > P.par_off[p] && P.par[j - 1] >= x) gb_refuse(P);
    const u64 i = lower_bound_g(P.src, P.nrows, x);
    const bool hit = i < P.nrows && P.src[i] == x;
    P.prow[j] = hit ? (u32)i : kGbNoRow;
    P.ppar[j] = (u32)p;
    P.plen[j] = hit ? P.v_off[i + 1] - P.v_off[i] : 0;
}

// Thread per edge (grid over e_cap).  The edge count is checked here: 2^32 or more is refused, more than e_cap does
// not fit.
__global__ void __launch_bounds__(256) gb_expand_kernel(const GbParams P) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0) P.words[GB_W_H] = (u64)GB_RADIX * P.tiles;
    if (*P.bad) return;
    const u64 E = P.words[GB_W_E];
    if (E >> 32 || E > P.e_cap) {
        if (k == 0) {
            if (E >> 32) gb_refuse(P);
            else atomicOr(P.bad, kGbBadCap);
        }
        return;
    }
    if (k >= E) return;
    const u64 npv = P.words[GB_W_PV];
    const u64 j = lower_bound_g(P.eoff, npv + 1, k + 1) - 1;  // the parent value holding edge k
    const u64 i = P.prow[j];
    const u64 d = P.v[P.v_off[i] + (k - P.eoff[j])];
    const u64 r = lower_bound_g(P.dest, P.ndest, d);
    if (r == P.ndest || P.dest[r] != d) gb_refuse(P);
    P.ek[k] = ((u64)P.ppar[j] << P.b_d) | r;
    P.ep[k] = (u32)i;
}

// ---- stable LSD radix sort, 8-bit digits ----------------------------------------------------------------------------
// Tile t holds items [t * GB_TILE, (t + 1) * GB_TILE); thread x of round r holds item r * GB_NT + x of the tile, so the
// tile's order is (round, warp, lane).  hist[d * tiles + t] is tile t's count of digit d: its exclusive scan is where
// the tile's first item of digit d goes.

// CTA per tile (grid over tiles); every CTA writes its 256 counts, zeros past n.
__global__ void __launch_bounds__(GB_NT) gb_hist_kernel(const u64* __restrict__ key, const u64* n_word, const int* bad,
                                                        u32 shift, u64 tiles, u64* __restrict__ hist) {
    __shared__ u32 cnt[GB_RADIX];
    const int tid = threadIdx.x;
    cnt[tid] = 0;
    __syncthreads();
    const u64 n = *bad ? 0 : *n_word;
    const u64 t0 = (u64)blockIdx.x * GB_TILE;
#pragma unroll
    for (int r = 0; r < GB_VT; ++r) {
        const u64 e = t0 + (u64)r * GB_NT + tid;
        if (e < n) atomicAdd(&cnt[(u32)(key[e] >> shift) & (GB_RADIX - 1)], 1u);
    }
    __syncthreads();
    hist[(u64)tid * tiles + blockIdx.x] = cnt[tid];
}

__device__ __forceinline__ u32 lanemask_lt() {
    u32 m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// CTA per tile: the items to base[digit] + their stable rank among the tile's items of that digit.
__global__ void __launch_bounds__(GB_NT) gb_scatter_kernel(const u64* __restrict__ key, const u32* __restrict__ pay,
                                                           const u64* n_word, const int* bad, u32 shift, u64 tiles,
                                                           const u64* __restrict__ hoff, u64* __restrict__ key_out,
                                                           u32* __restrict__ pay_out) {
    __shared__ u64 s_base[GB_RADIX];
    __shared__ u32 s_warp[GB_WARPS][GB_RADIX];
    const int tid = threadIdx.x, wid = tid >> 5;
    const u64 n = *bad ? 0 : *n_word;
    const u64 t0 = (u64)blockIdx.x * GB_TILE;
    if (t0 >= n) return;
    s_base[tid] = hoff[(u64)tid * tiles + blockIdx.x];
    for (int r = 0; r < GB_VT; ++r) {
#pragma unroll
        for (int w = 0; w < GB_WARPS; ++w) s_warp[w][tid] = 0;
        __syncthreads();
        const u64 e = t0 + (u64)r * GB_NT + tid;
        const bool ok = e < n;
        const u64 k = ok ? key[e] : 0;
        const u32 d = ok ? (u32)(k >> shift) & (GB_RADIX - 1) : GB_RADIX;
        const u32 same = __match_any_sync(0xffffffffu, d);
        const u32 rank = __popc(same & lanemask_lt());
        if (ok && rank == 0) s_warp[wid][d] = __popc(same);
        __syncthreads();
        u32 run = 0;  // digit tid: each warp's exclusive offset inside this round
#pragma unroll
        for (int w = 0; w < GB_WARPS; ++w) {
            const u32 c = s_warp[w][tid];
            s_warp[w][tid] = run;
            run += c;
        }
        __syncthreads();
        if (ok) {
            const u64 pos = s_base[d] + s_warp[wid][d] + rank;
            key_out[pos] = k;
            pay_out[pos] = pay[e];
        }
        __syncthreads();
        s_base[tid] += run;
    }
}

// ---- groups ----------------------------------------------------------------------------------------------------------

// Thread per edge (grid over e_cap): 1 where a group starts.
__global__ void __launch_bounds__(256) gb_heads_kernel(const GbParams P) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || k >= P.words[GB_W_E]) return;
    P.head[k] = k == 0 || P.ek[k] != P.ek[k - 1];
}

// Thread per edge: gstart[g] = the first edge of group g; gstart[G] = E.
__global__ void __launch_bounds__(256) gb_groups_kernel(const GbParams P) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0) P.words[GB_W_H] = (u64)GB_RADIX * P.tiles;
    if (*P.bad) return;
    const u64 E = P.words[GB_W_E];
    if (k == 0) P.gstart[P.words[GB_W_G]] = E;
    if (k < E && P.head[k]) P.gstart[P.gidx[k]] = k;
}

// Thread per group (grid over e_cap): the order key parent << b_s | size, and the group itself as the payload.
__global__ void __launch_bounds__(256) gb_gkeys_kernel(const GbParams P, u64* gk, u32* gp) {
    const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || g >= P.words[GB_W_G]) return;
    const u64 s = P.gstart[g];
    gk[g] = ((P.ek[s] >> P.b_d) << P.b_s) | (P.gstart[g + 1] - s);
    gp[g] = (u32)g;
}

// Thread per ordered group: its size, and the position of each group in the order.
__global__ void __launch_bounds__(256) gb_sizes_kernel(const GbParams P) {
    const u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || o >= P.words[GB_W_G]) return;
    const u32 g = P.gp[o];
    P.gsz[o] = P.gstart[g + 1] - P.gstart[g];
    P.inv[g] = (u32)o;
}

// Grid over max(e_cap + 1, npar + 1) threads: thread G writes mem_off[G] even when every edge is its own group.  Nothing is written but the sizes when the input was refused or an output
// does not fit: G > grp_cap, or E > mem_cap with members.
__global__ void __launch_bounds__(256) gb_write_kernel(const GbParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const int bad = *P.bad;
    const u64 E = P.words[GB_W_E], G = bad ? 0 : P.words[GB_W_G];
    const bool fit = G <= P.grp_cap && (!P.members || E <= P.mem_cap);
    if (t == 0) {
        P.sizes[0] = G;
        P.sizes[1] = bad & kGbBadArg ? 0 : E;
        if ((bad & kGbBadCap) || (!bad && !fit)) atomicOr(P.err, 1);
    }
    if (bad || !fit) return;
    if (t < G) {
        P.keys[t] = P.dest[P.ek[P.gstart[P.gp[t]]] & ((1ull << P.b_d) - 1)];
        P.mem_off[t] = P.moff[t];
    }
    if (t == G) P.mem_off[G] = E;
    if (t <= P.npar) {  // the first ordered group of parent t
        u64 lo = 0, hi = G;
        while (lo < hi) {
            const u64 mid = lo + ((hi - lo) >> 1);
            if ((P.gk[mid] >> P.b_s) < t) lo = mid + 1; else hi = mid;
        }
        P.grp_off[t] = lo;
    }
    if (P.members && t < E) {
        const u64 g = P.gidx[t] + P.head[t] - 1;
        P.members[P.moff[P.inv[g]] + (t - P.gstart[g])] = P.src[P.ep[t]];
    }
}

}  // namespace dgx
