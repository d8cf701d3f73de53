// path_kernel.cuh -- one expansion level of shortest() without weights (query/shortest.go expandOut :141-273 with
// shortestPath's Dijkstra loop :518-586 at unit cost), over every exec sg of the level at once.
//
// A search (dgx_path_search) lives in HBM as two sorted sets in ping-pong buffers:
//   seen      the discovered nodes: uid (u64, ascending), parent (u64), the attr index of the hop into it (u32) and its
//             level (u32).  From is at level 0.
//   expanded  the sources that have had a kept edge (adjacencyMap's keys), ascending.
// Which buffer is current, the sizes, the level count and To's level are device words (state[]) that only the last
// kernel of a level changes, and only when the level was accepted, so a refused level leaves the search as it was
// without a host round trip.
//
// Level layout: sg s (exec order) has rows src_off[s] .. src_off[s+1]; row r holds v[v_off[r] .. v_off[r+1]) of source
// src[r]; dest[dest_off[s] .. dest_off[s+1]) is the sg's DestUIDs.  An edge (src[r], x) is kept iff x is in its sg's
// dest (updateUidMatrix).  A kept edge reaches a new node iff x is not in seen.
//   ps_check_kernel    thread per index: offsets start at 0, do not decrease and end inside their arrays; src, rows and
//                      dests strictly ascend within their sg / row
//   ps_flags_kernel    thread per value: its row and sg, kept (dest), new (not in seen), the row's has-edge flag, the
//                      level's kept count, and the refusal of a source with a kept edge that was not discovered at the
//                      previous level (which covers one already expanded)
//   scan_u64_kernel    x2: new values -> positions; rows with an edge -> positions
//   ps_gather_kernel   the new values as a matrix over the rows, the sources with an edge as a matrix over the sgs
//   merge_matrix_impl  x2: the distinct new nodes N and the distinct new expanded sources E (merge_matrix.cuh)
//   ps_parent_kernel   thread per value: atomicMin of the source over the edges into each new node (its parent);
//                      thread per dest value: is it outside expanded and E (the next frontier)
//   ps_attr_kernel     thread per value: atomicMax of the sg index over the edges from that parent into the node
//   scan_u64_kernel    the next-frontier flags -> positions
//   ps_insert_kernel   grid-stride: seen and N, expanded and E merged by rank into the other buffers
//   ps_write_kernel    thread per dest value and sg: next / next_off
//   ps_commit_kernel   one thread: flips the buffers, adds the sizes, the level, To's level, and writes the stats
// ps_walk_kernel (one thread) reads the path from To back to From for dgx_path_result.
#pragma once

#include "encode_kernel.cuh"  // scan_u64_kernel, EN_NT, EN_TILE

namespace dgx {

constexpr int kLaneErrPath = 128;  // lane error flag bit: a shortest-path level's input is malformed (DGX_ERR_ARG at sync)
// words of one level: rows, values, dest values, new values, rows with an edge, |N|, |E|, next frontier, kept edges
constexpr int PS_W_R = 0, PS_W_M = 1, PS_W_D = 2, PS_W_NV = 3, PS_W_NR = 4, PS_W_NN = 5, PS_W_NE = 6, PS_W_NX = 7,
              PS_W_EDGES = 8, PS_WORDS = 9;
// the search's device words
constexpr int PS_S_CUR = 0, PS_S_N = 1, PS_E_CUR = 2, PS_E_N = 3, PS_LEVEL = 4, PS_TO_LEVEL = 5, PS_TO = 6,
              PS_STATE = 7;

struct PsParams {
    u64 nsg;
    const u32* attr;      // nsg
    const u64* src_off;   // nsg + 1
    const u64* src;
    u64 r_cap;
    const u64* v_off;     // rows + 1
    const u64* v;
    u64 v_cap;
    const u64* dest_off;  // nsg + 1
    const u64* dest;
    u64 d_cap;
    // the search
    u64* su[2];           // seen: uid, parent, attr, level
    u64* sp[2];
    u32* sa[2];
    u32* sl[2];
    u64* ex[2];           // expanded
    u64* state;           // PS_STATE words
    // workspace
    int* bad;             // zeroed
    u64* words;           // PS_WORDS, zeroed
    u32* vrow;            // v_cap: the row of each value
    u32* vsg;             // v_cap: its sg
    u64* vflag;           // v_cap: kept and new
    u64* vpos;            // v_cap + 1
    u64* rflag;           // r_cap + 1, zeroed: the row has a kept edge
    u64* rpos;            // r_cap + 2
    u64* nv;              // v_cap: the new values, row by row
    u64* nv_off;          // r_cap + 2 (the merge reads max(r_cap, 1) rows)
    u64* es;              // r_cap + 1: the sources with an edge, sg by sg
    u64* es_off;          // nsg + 1
    u64* nn;              // v_cap: N
    u64* ne;              // r_cap + 1: E
    u64* npar;            // v_cap, all ones: each new node's parent
    u32* nsgi;            // v_cap, zeroed: the largest sg index holding (parent, node)
    u64* dflag;           // d_cap
    u64* dpos;            // d_cap + 1
    // outputs
    u64* next;
    u64* next_off;        // nsg + 1
    u64* stats;           // {edges, discovered, to_level}
    int* err;
};

__device__ __forceinline__ void ps_refuse(const PsParams& P) {
    atomicOr(P.bad, 1);
    atomicOr(P.err, kLaneErrPath);
}

__device__ __forceinline__ bool ps_has(const u64* a, u64 n, u64 x) {
    const u64 j = lower_bound_g(a, n, x);
    return j < n && ld_probe(a + j) == x;
}

// The segment of off[0 .. n] holding index t (off[0] == 0 <= t).
__device__ __forceinline__ u64 ps_seg(const u64* off, u64 n, u64 t) { return lower_bound_g(off, n + 1, t + 1) - 1; }

// Grid over max(nsg + 1, r_cap + 1, v_cap, d_cap) threads.
__global__ void __launch_bounds__(256) ps_check_kernel(const PsParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 S = P.nsg;
    const u64 R = P.src_off[S], D = P.dest_off[S];
    const bool r_ok = P.src_off[0] == 0 && R <= P.r_cap;
    const bool d_ok = P.dest_off[0] == 0 && D <= P.d_cap;
    const u64 M = r_ok ? P.v_off[R] : 0;
    const bool v_ok = r_ok && P.v_off[0] == 0 && M <= P.v_cap;
    bool bad = false;
    if (t == 0) {
        bad = !(r_ok && d_ok && v_ok);
        P.words[PS_W_R] = r_ok ? R : 0;
        P.words[PS_W_M] = v_ok ? M : 0;
        P.words[PS_W_D] = d_ok ? D : 0;
    }
    if (t < S && (P.src_off[t] > P.src_off[t + 1] || P.dest_off[t] > P.dest_off[t + 1])) bad = true;
    if (r_ok && t < R) {
        if (P.v_off[t] > P.v_off[t + 1]) bad = true;
        if (t > 0 && P.src_off[ps_seg(P.src_off, S, t)] != t && P.src[t - 1] >= P.src[t]) bad = true;
    }
    if (v_ok && t > 0 && t < M && P.v_off[ps_seg(P.v_off, R, t)] != t && P.v[t - 1] >= P.v[t]) bad = true;
    if (d_ok && t > 0 && t < D && P.dest_off[ps_seg(P.dest_off, S, t)] != t && P.dest[t - 1] >= P.dest[t]) bad = true;
    if (bad) ps_refuse(P);
}

// Thread per value (grid over v_cap).  A refused level flags nothing.
__global__ void __launch_bounds__(256) ps_flags_kernel(const PsParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 M = P.words[PS_W_M];
    bool kept = false;
    if (t < M) {
        P.vflag[t] = 0;
        if (!*P.bad) {
            const u64 r = ps_seg(P.v_off, P.words[PS_W_R], t);
            const u64 s = ps_seg(P.src_off, P.nsg, r);
            const u64 x = P.v[t];
            const u64 d0 = P.dest_off[s];
            kept = ps_has(P.dest + d0, P.dest_off[s + 1] - d0, x);
            P.vrow[t] = (u32)r;
            P.vsg[t] = (u32)s;
            if (kept) {
                P.rflag[r] = 1;
                // the source must be a node discovered at the previous level: then it is not expanded yet, and the
                // path walk finds every parent one level up
                const u64* st = P.state;
                const u64 sc = st[PS_S_CUR], ns = st[PS_S_N], u = P.src[r];
                const u64 j = lower_bound_g(P.su[sc], ns, u);
                if (j == ns || P.su[sc][j] != u || P.sl[sc][j] != (u32)st[PS_LEVEL]) ps_refuse(P);
                P.vflag[t] = !ps_has(P.su[sc], ns, x);
            }
        }
    }
    const unsigned n = __popc(__ballot_sync(0xffffffffu, kept));
    if ((threadIdx.x & 31) == 0 && n) atomicAdd((unsigned long long*)(P.words + PS_W_EDGES), (unsigned long long)n);
}

// Grid over max(v_cap, r_cap + 2, nsg + 1) threads.  A refused level gathers nothing and gives both merges empty rows.
__global__ void __launch_bounds__(256) ps_gather_kernel(const PsParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 R = P.words[PS_W_R];
    if (*P.bad) {
        if (t < P.r_cap + 2) P.nv_off[t] = 0;
        if (t <= P.nsg) P.es_off[t] = 0;
        return;
    }
    if (t < P.r_cap + 2) P.nv_off[t] = P.vpos[P.v_off[t < R ? t : R]];  // rows past R are empty
    if (t <= P.nsg) P.es_off[t] = P.rpos[P.src_off[t]];
    if (t < P.words[PS_W_M] && P.vflag[t]) P.nv[P.vpos[t]] = P.v[t];
    if (t < R && P.rflag[t]) P.es[P.rpos[t]] = P.src[t];
}

// Grid over max(v_cap, d_cap) threads.  Nothing runs for a refused level.
__global__ void __launch_bounds__(256) ps_parent_kernel(const PsParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    if (t < P.words[PS_W_M] && P.vflag[t]) {
        const u64 k = lower_bound_g(P.nn, P.words[PS_W_NN], P.v[t]);
        atomicMin((unsigned long long*)(P.npar + k), (unsigned long long)P.src[P.vrow[t]]);
    }
    if (t < P.words[PS_W_D]) {
        const u64 x = P.dest[t];
        const u64* st = P.state;
        P.dflag[t] = !ps_has(P.ex[st[PS_E_CUR]], st[PS_E_N], x) && !ps_has(P.ne, P.words[PS_W_NE], x);
    }
}

// Grid over v_cap threads.
__global__ void __launch_bounds__(256) ps_attr_kernel(const PsParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || t >= P.words[PS_W_M] || !P.vflag[t]) return;
    const u64 k = lower_bound_g(P.nn, P.words[PS_W_NN], P.v[t]);
    if (P.src[P.vrow[t]] == P.npar[k]) atomicMax(P.nsgi + k, P.vsg[t]);
}

// Grid-stride over |seen| + |N| + |expanded| + |E| records: both sets and their new members into the other buffers.
// Each pair is sorted and disjoint, so a record's new place is its own index plus its rank in the other sequence.
__global__ void __launch_bounds__(256) ps_insert_kernel(const PsParams P) {
    if (*P.bad) return;
    const u64* st = P.state;
    const u64 sc = st[PS_S_CUR], ns = st[PS_S_N], ec = st[PS_E_CUR], ne = st[PS_E_N];
    const u64 NN = P.words[PS_W_NN], NE = P.words[PS_W_NE];
    const u32 level = (u32)st[PS_LEVEL] + 1;
    const u64 n1 = NN ? ns + NN : 0, n2 = NE ? ne + NE : 0;  // a set that gains nothing keeps its buffer
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2; i += stride) {
        if (i < n1) {
            u64 pos, uid, par;
            u32 a, l;
            if (i < ns) {
                uid = P.su[sc][i];
                pos = i + lower_bound_g(P.nn, NN, uid);
                par = P.sp[sc][i];
                a = P.sa[sc][i];
                l = P.sl[sc][i];
            } else {
                const u64 k = i - ns;
                uid = P.nn[k];
                pos = k + lower_bound_g(P.su[sc], ns, uid);
                par = P.npar[k];
                a = P.attr[P.nsgi[k]];
                l = level;
            }
            P.su[sc ^ 1][pos] = uid;
            P.sp[sc ^ 1][pos] = par;
            P.sa[sc ^ 1][pos] = a;
            P.sl[sc ^ 1][pos] = l;
        } else {
            const u64 j = i - n1;
            const u64 x = j < ne ? P.ex[ec][j] : P.ne[j - ne];
            const u64 pos = j < ne ? j + lower_bound_g(P.ne, NE, x) : (j - ne) + lower_bound_g(P.ex[ec], ne, x);
            P.ex[ec ^ 1][pos] = x;
        }
    }
}

// Grid over max(d_cap, nsg + 1) threads.  A refused level writes nothing.
__global__ void __launch_bounds__(256) ps_write_kernel(const PsParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    if (t <= P.nsg) P.next_off[t] = P.dpos[P.dest_off[t]];
    if (t < P.words[PS_W_D] && P.dflag[t]) P.next[P.dpos[t]] = P.dest[t];
}

__global__ void ps_commit_kernel(const PsParams P) {
    if (*P.bad) return;
    u64* st = P.state;
    const u64 NN = P.words[PS_W_NN], NE = P.words[PS_W_NE];
    const u64 level = st[PS_LEVEL] + 1;
    if (st[PS_TO_LEVEL] == 0 && ps_has(P.nn, NN, st[PS_TO])) st[PS_TO_LEVEL] = level;
    if (NN) {
        st[PS_S_CUR] ^= 1;
        st[PS_S_N] += NN;
    }
    if (NE) {
        st[PS_E_CUR] ^= 1;
        st[PS_E_N] += NE;
    }
    st[PS_LEVEL] = level;
    P.stats[0] = P.words[PS_W_EDGES];
    P.stats[1] = NN;
    P.stats[2] = st[PS_TO_LEVEL];
}

// One thread: the path To -> From by parents, written From first: uids[0 .. L], attrs[0 .. L) (attrs[i] is the hop
// into uids[i + 1]).  L is To's level, which the host read from state after the last level.
__global__ void ps_walk_kernel(const u64* su, const u64* sp, const u32* sa, const u64* state, u64 L, u64* uids,
                               u32* attrs) {
    const u64 n = state[PS_S_N];
    u64 cur = state[PS_TO];
    for (u64 i = L;; --i) {
        uids[i] = cur;
        if (i == 0) break;
        const u64 j = lower_bound_g(su, n, cur);
        attrs[i - 1] = sa[j];
        cur = sp[j];
    }
}

}  // namespace dgx
