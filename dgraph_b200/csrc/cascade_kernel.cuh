// cascade_kernel.cuh -- @cascade (query/query.go populateVarMap :1445-1527 with updateUidMatrix :1425-1439, and the root
// pagination of ProcessQuery :3004-3011) over a whole forest of subgraph nodes in one call.
//
// Each node n has its old DestUIDs (dest, strictly ascending), its uid matrix (rows; row i belongs to parent.dest[i]),
// has_val (one byte per row: the row has values) and counts_len.  What happens to a node is resolved on the host:
//   prune  (CASCADE and not SKIP)  dest[i] survives unless a CHECKED child has an empty or missing row i, an empty or
//                                  missing has_val[i] and i >= counts_len
//   rows   KEEP: left as they are; OLD (FILTERED, not SKIP, and not NEW): filtered by the dest the node came with;
//          NEW (CASCADE and not a root, or a root with first or offset): filtered by the node's new dest, then every
//          row cut with PageRange(first, offset, len) (x/x.go:738-767)
// A node's new dest depends on its children's final rows, and its final rows on its new dest only, so the forest is
// processed level by level from the deepest up, every node of a level in the same launches.
//
// Layout: every array of every node is gathered into flat slots in level order (deepest level first, node index
// order inside a level): values [vb, vb + vcap), row offsets [ob, ob + nrows + 1) (flat value indices), dest
// [db, db + ndest), has_val [hb, hb + nhv).  A node's kept values and new dest go to the front of its own slots.
//   cc_gather_kernel    thread per slot: the node's arrays into the flat slots; checks the offsets
//   per level (the nodes [a, b)):
//     cc_keep_kernel    thread per dest slot: dest strictly ascends; the keep flag (its checked children's final rows)
//     scan_u64_kernel   keep flags -> each kept dest value's rank in its node
//     cc_filter_kernel  thread per dest slot: the new dest compacted; thread per node: its length; thread per value:
//                       its row (a search of the offsets), the order check of unordered rows, and whether it survives
//                       the filter (a search of the node's old dest, then the keep flag for NEW)
//     scan_u64_kernel   value flags -> each surviving value's rank in its row, prefix(v) - prefix(row start)
//     cc_page_kernel    thread per surviving value: the PageRange cut from its row's surviving count
//     scan_u64_kernel   the paged flags -> output positions
//     cc_compact_kernel thread per value: the kept values; thread per offset slot: the new row offsets
//   cc_count_kernel     thread per node: its kept values and new dest length, in node order
//   scan_u64_kernel     both counts -> each node's place in the node-order outputs
//   cc_place_kernel     thread per slot: values, row offsets, new dest and dest offsets into the outputs, and sizes;
//                       a refused call writes sizes = {0, 0} and nothing else
// Launches: 4 + 7 * D, D the levels that hold a dest or a value slot.
#pragma once

#include "encode_kernel.cuh"  // scan_u64_kernel, EN_NT, EN_TILE

namespace dgx {

constexpr int kLaneErrCascade = 64;  // lane error flag bit: a cascade input is malformed (DGX_ERR_ARG at sync)
constexpr u32 CC_ROWS_KEEP = 0, CC_ROWS_OLD = 1, CC_ROWS_NEW = 2;

struct CcNode {                // one node, in level order
    const u64* v;              // its values (room for vcap)
    const u64* v_off;          // nrows + 1 offsets into v, plus v_base
    const u64* dest;           // ndest
    const unsigned char* hv;   // nhv
    u64 v_base;
    u64 vb, vcap;              // flat value slots
    u64 ob, nrows;             // flat offset slots: nrows + 1 of them
    u64 db, ndest;             // flat dest slots
    u64 hb, nhv;               // flat has_val slots
    u64 counts_len;
    u64 out_row;               // its first row in the node-order output
    u32 id;                    // node-order index
    u32 mode;                  // CC_ROWS_*
    u32 prune;                 // dest pruned by its checked children
    u32 ordered;               // rows not uid-sorted: not checked for order
    int first, offset;         // PageRange arguments of a NEW node (0, 0 otherwise)
    u32 ck_b, ck_e;            // its checked children ck[ck_b .. ck_e), level-order indices
};

struct CcLevel {               // the nodes [a, b) of one level and their slots
    u32 a, b;
    u64 va, nv, da, nd, oa, no;
    const u64* n_dest;         // device words holding nd and nv, for the scans
    const u64* n_val;
};

struct CcParams {
    const CcNode* node;        // nnodes, level order
    const u32* ck;
    u32 nnodes;
    u64 nv, no, nd, nh;        // flat slot totals
    u64 out_rows;              // rows of the whole forest
    u64* V;                    // gathered values (nv)
    u64* VO;                   // gathered row offsets (no)
    u64* D;                    // gathered dest (nd)
    unsigned char* H;          // gathered has_val (nh)
    u64* OV;                   // kept values, at the front of each node's value slots (nv)
    u64* OO;                   // their row offsets (no)
    u64* ND;                   // new dest, at the front of each node's dest slots (nd)
    u64* NDE;                  // new dest length per node (nnodes, level order)
    u64* keep;                 // per level: dest keep flags, then their scan (max nd + 1)
    u64* kx;
    u64* fv;                   // per level: value flags, their scan, the paged flags' scan (max nv + 1)
    u64* fx;
    u64* fy;
    u32* rw;                   // per level: each value's row in its node
    u64* cnt;                  // 2 * nnodes: node-order kept values, then new dest lengths; cx its scan
    u64* cx;
    int* bad;
    int* err;
    u64* out;
    u64* out_off;              // out_rows + 1
    u64* dest_out;
    u64* dest_off;             // nnodes + 1
    u64* sizes;                // [values, dest]
};

__device__ __forceinline__ void cc_refuse(const CcParams& P) {
    atomicOr(P.bad, 1);
    atomicOr(P.err, kLaneErrCascade);
}

// The last node in [a, b) whose slot base (field f) is <= t: the node owning slot t, since bases ascend in level order.
template <u64 CcNode::*F>
__device__ __forceinline__ u32 cc_node_of(const CcNode* N, u32 a, u32 b, u64 t) {
    u32 lo = a, hi = b;  // answer in [lo, hi)
    while (hi - lo > 1) {
        const u32 mid = lo + ((hi - lo) >> 1);
        if (N[mid].*F <= t) lo = mid; else hi = mid;
    }
    return lo;
}

// x.PageRange(count, offset, n) -> [s, e)
__device__ __forceinline__ void cc_page_range(long long count, long long offset, long long n, long long& s,
                                              long long& e) {
    s = 0;
    e = n;
    if (n == 0 || (count == 0 && offset == 0)) return;
    if (count < 0) {
        if (-count > n) count = -n;
        s = (((n + count) % n) + n) % n;
        return;
    }
    s = offset < 0 ? 0 : offset;
    if (s > n) { s = n; return; }
    if (count == 0) return;
    if (s + count < n) e = s + count;
}

// Grid over max(nv, no, nd, nh, nnodes) threads.
__global__ void __launch_bounds__(256) cc_gather_kernel(const CcParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const CcNode* N = P.node;
    if (t < P.nv) {
        const CcNode& n = N[cc_node_of<&CcNode::vb>(N, 0, P.nnodes, t)];
        P.V[t] = n.v[t - n.vb];
    }
    if (t < P.no) {
        const CcNode& n = N[cc_node_of<&CcNode::ob>(N, 0, P.nnodes, t)];
        const u64 r = t - n.ob, x = n.v_off[r];
        bool bad = r == 0 ? x != n.v_base : x < n.v_off[r - 1];
        if (r == n.nrows && x - n.v_base > n.vcap) bad = true;
        if (bad) cc_refuse(P);
        P.VO[t] = P.OO[t] = n.vb + (x - n.v_base);  // a level without work keeps its (empty) rows
    }
    if (t < P.nd) {
        const CcNode& n = N[cc_node_of<&CcNode::db>(N, 0, P.nnodes, t)];
        P.D[t] = n.dest[t - n.db];
    }
    if (t < P.nh) {
        const CcNode& n = N[cc_node_of<&CcNode::hb>(N, 0, P.nnodes, t)];
        P.H[t] = n.hv[t - n.hb];
    }
    if (t < P.nnodes) P.NDE[t] = N[t].ndest;
}

// Grid over L.nd threads.
__global__ void __launch_bounds__(256) cc_keep_kernel(const CcParams P, const CcLevel L) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || t >= L.nd) return;
    const u64 p = L.da + t;
    const CcNode* N = P.node;
    const CcNode& n = N[cc_node_of<&CcNode::db>(N, L.a, L.b, p)];
    const u64 i = p - n.db;
    if (i > 0 && P.D[p - 1] >= P.D[p]) cc_refuse(P);
    u64 keep = 1;
    if (n.prune)
        for (u32 k = n.ck_b; k < n.ck_e && keep; ++k) {
            const CcNode& c = N[P.ck[k]];
            const bool no_row = i >= c.nrows || P.OO[c.ob + i + 1] == P.OO[c.ob + i];
            const bool no_val = i >= c.nhv || P.H[c.hb + i] == 0;
            if (no_row && no_val && i >= c.counts_len) keep = 0;
        }
    P.keep[t] = keep;
}

// Grid over max(L.nd, L.nv, L.b - L.a) threads.
__global__ void __launch_bounds__(256) cc_filter_kernel(const CcParams P, const CcLevel L) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    const CcNode* N = P.node;
    if (t < L.nd && P.keep[t]) {
        const u64 p = L.da + t;
        const CcNode& n = N[cc_node_of<&CcNode::db>(N, L.a, L.b, p)];
        P.ND[n.db + P.kx[t] - P.kx[n.db - L.da]] = P.D[p];
    }
    if (t < L.b - L.a) {
        const CcNode& n = N[L.a + t];
        P.NDE[L.a + t] = P.kx[n.db + n.ndest - L.da] - P.kx[n.db - L.da];
    }
    if (t < L.nv) {
        const u64 p = L.va + t;
        const CcNode& n = N[cc_node_of<&CcNode::vb>(N, L.a, L.b, p)];
        u64 f = 0;
        if (p < P.VO[n.ob + n.nrows]) {  // past it: slack of the node's value room
            const u64 r = lower_bound_g(P.VO + n.ob, n.nrows + 1, p + 1) - 1;
            const u64 x = P.V[p];
            if (!n.ordered && P.VO[n.ob + r] != p && P.V[p - 1] >= x) cc_refuse(P);
            f = 1;
            if (n.mode != CC_ROWS_KEEP) {
                const u64 j = lower_bound_g(P.D + n.db, n.ndest, x);
                f = j < n.ndest && P.D[n.db + j] == x && (n.mode == CC_ROWS_OLD || P.keep[n.db - L.da + j]);
            }
            P.rw[t] = (u32)r;
        }
        P.fv[t] = f;
    }
}

// Grid over L.nv threads: a surviving value of a NEW node stays iff its rank in its row is inside the row's page.
__global__ void __launch_bounds__(256) cc_page_kernel(const CcParams P, const CcLevel L) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || t >= L.nv || !P.fv[t]) return;
    const u64 p = L.va + t;
    const CcNode& n = P.node[cc_node_of<&CcNode::vb>(P.node, L.a, L.b, p)];
    if (n.mode != CC_ROWS_NEW) return;
    const u64 r = P.rw[t];
    const u64 rs = P.VO[n.ob + r] - L.va, re = P.VO[n.ob + r + 1] - L.va;
    long long s, e;
    cc_page_range(n.first, n.offset, (long long)(P.fx[re] - P.fx[rs]), s, e);
    const long long rank = (long long)(P.fx[t] - P.fx[rs]);
    if (rank < s || rank >= e) P.fv[t] = 0;
}

// Grid over max(L.nv, L.no) threads.
__global__ void __launch_bounds__(256) cc_compact_kernel(const CcParams P, const CcLevel L) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    const CcNode* N = P.node;
    if (t < L.nv && P.fv[t]) {
        const u64 p = L.va + t;
        const CcNode& n = N[cc_node_of<&CcNode::vb>(N, L.a, L.b, p)];
        P.OV[n.vb + P.fy[t] - P.fy[n.vb - L.va]] = P.V[p];
    }
    if (t < L.no) {
        const u64 q = L.oa + t;
        const CcNode& n = N[cc_node_of<&CcNode::ob>(N, L.a, L.b, q)];
        P.OO[q] = n.vb + P.fy[P.VO[q] - L.va] - P.fy[n.vb - L.va];
    }
}

// Grid over nnodes threads.
__global__ void __launch_bounds__(256) cc_count_kernel(const CcParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || t >= P.nnodes) return;
    const CcNode& n = P.node[t];
    P.cnt[n.id] = P.OO[n.ob + n.nrows] - n.vb;
    P.cnt[P.nnodes + n.id] = P.NDE[t];
}

// Grid over max(nv, no, nd, nnodes + 1) threads.
__global__ void __launch_bounds__(256) cc_place_kernel(const CcParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) {
        if (t == 0) P.sizes[0] = P.sizes[1] = 0;
        return;
    }
    const CcNode* N = P.node;
    const u64 NN = P.nnodes, dbase = P.cx[NN];
    if (t < P.nv) {
        const CcNode& n = N[cc_node_of<&CcNode::vb>(N, 0, P.nnodes, t)];
        if (t < P.OO[n.ob + n.nrows]) P.out[P.cx[n.id] + t - n.vb] = P.OV[t];
    }
    if (t < P.no) {
        const CcNode& n = N[cc_node_of<&CcNode::ob>(N, 0, P.nnodes, t)];
        const u64 r = t - n.ob;
        if (r < n.nrows) P.out_off[n.out_row + r] = P.cx[n.id] + P.OO[t] - n.vb;
    }
    if (t < P.nd) {
        const u32 k = cc_node_of<&CcNode::db>(N, 0, P.nnodes, t);
        const CcNode& n = N[k];
        if (t - n.db < P.NDE[k]) P.dest_out[P.cx[NN + n.id] - dbase + t - n.db] = P.ND[t];
    }
    if (t < NN) P.dest_off[t] = P.cx[NN + t] - dbase;
    if (t == NN) {
        P.dest_off[NN] = P.cx[2 * NN] - dbase;
        P.out_off[P.out_rows] = dbase;
        P.sizes[0] = dbase;
        P.sizes[1] = P.cx[2 * NN] - dbase;
    }
}

}  // namespace dgx
