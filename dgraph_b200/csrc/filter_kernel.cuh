// filter_kernel.cuh -- batched "A-driven" sorted-set filter for sm_90a.
//
// One kernel covers algo.IntersectWith (algo/uidlist.go:142), the whole chain of
// algo.IntersectSorted (:297-329, k lists in ONE pass), algo.Difference (:332)
// and the batched row-filter shape of worker/task.go:783 / query/query.go:1425.
//
// Work unit ("tile"): F_TA consecutive values of a query's driving list A (its
// shortest list for intersections, u for Difference), held in registers (four
// per thread, warp-striped).  Every other list L_j of the query contributes only
// the slice [lower_bound(L_j, first), upper_bound(L_j, last)):
//   1. one warp per list finds both slice bounds with interleaved 32-ary
//      searches (log32 dependent rounds, all lists in parallel);
//   2. the slices of as many lists as fit are staged in shared memory together
//      with coalesced 16-byte loads, re-based to the tile's first value: when the
//      tile spans < 2^32 the staged keys are 32-bit (half the shared memory and
//      single-instruction compares), otherwise 64-bit;
//   3. each warp pushes its live candidates through the staged lists without
//      block barriers, using a branch-light "binary lifting" search whose step
//      sequence depends only on the slice length (no divergence).  After the
//      first list the block re-packs its survivors once; later lists only pay
//      for live rows;
//   4. survivors are counted per warp, tile outputs are concatenated with a
//      single-pass decoupled look-back (which also yields a batch's CSR offsets)
//      and written straight from registers, in order.
// Slices too large for shared memory are streamed in chunks (dense candidates)
// or binary-searched in global memory (sparse candidates).  Intermediates of the
// k-way chain never touch HBM and a list is read at most once.
//
// Duplicate semantics (pinned by algo/uidlist_test.go:329-348): a candidate that
// is the r-th copy of x in A survives list L_j iff L_j holds more than r copies
// of x, i.e. L_j[lower_bound(x) + r] == x -- multiset-min for intersections and
// multiset difference, exactly what the reference's two-pointer merges produce.
// Tiles that contain repeated values keep their candidates in place (no
// re-packing) so the rank can be recovered from the tile.
#pragma once

#include "common.cuh"

namespace dgx {

constexpr int F_NT = 256;            // threads per CTA
constexpr int F_VA = 4;              // candidates per thread (rows of a warp)
constexpr int F_TA = F_NT * F_VA;    // candidates per tile
constexpr int F_WC = 32 * F_VA;      // candidates per warp
constexpr int F_NW = F_NT / 32;      // warps per CTA
constexpr int F_LB = F_NW;           // lists whose slice bounds are searched per batch (one warp each)

struct FList {
    const u64* ptr;
    u64 len;             // length, or an upper bound when dyn_len != nullptr
    const u64* dyn_len;  // optional: device word holding the actual length
};
struct FTask {
    u64 tile_base;   // index of the task's first tile
    u32 list_first;  // lists[list_first] is A, followed by k-1 filter lists
    u32 k;
};
struct FParams {
    const FTask* tasks;
    const FList* lists;
    u32 ntasks;
    u32 ntiles;
    int op;               // 0 intersect, 1 difference
    u32 stream_ratio;     // oversized slice: stream when slice_len <= stream_ratio * live candidates
    u32 scap_bytes;       // shared-memory staging capacity for slices, in bytes
    u64* out;
    u64 out_cap;
    u64* out_off;         // ntasks + 1
    u64* status;          // ntiles words, zeroed
    u32* ticket;          // zeroed
    int* err;             // set to 1 on out_cap overflow
};

__device__ __forceinline__ u64 flist_len(const FList& L) {
    u64 n = L.len;
    if (L.dyn_len) {
        u64 d = ld_relaxed(L.dyn_len);
        if (d < n) n = d;
    }
    return n;
}

// Both slice bounds of one list in one pass: r0 = first i with a[i] >= xlo,
// r1 = first i with a[i] > xhi.  The two 32-ary searches advance in lock step so
// their global loads overlap (latency of one search).  Full warp, uniform args.
__device__ __forceinline__ void warp_bounds2_g(const u64* __restrict__ a, u64 n, u64 xlo, u64 xhi, int lane,
                                               u64& r0, u64& r1) {
    u64 lo0 = 0, hi0 = n, lo1 = 0, hi1 = n;
    while ((hi0 - lo0 > 32) || (hi1 - lo1 > 32)) {
        const bool a0 = hi0 - lo0 > 32, a1 = hi1 - lo1 > 32;
        const u64 st0 = (hi0 - lo0) >> 5, st1 = (hi1 - lo1) >> 5;
        u64 v0 = 0, v1 = 0;
        if (a0) v0 = ld_probe(a + lo0 + (u64)(lane + 1) * st0 - 1);
        if (a1) v1 = ld_probe(a + lo1 + (u64)(lane + 1) * st1 - 1);
        const unsigned c0 = __popc(__ballot_sync(0xffffffffu, a0 && v0 < xlo));
        const unsigned c1 = __popc(__ballot_sync(0xffffffffu, a1 && v1 <= xhi));
        if (a0) {
            const u64 nlo = lo0 + (u64)c0 * st0;
            if (c0 < 32) hi0 = lo0 + (u64)(c0 + 1) * st0 - 1;
            lo0 = nlo;
        }
        if (a1) {
            const u64 nlo = lo1 + (u64)c1 * st1;
            if (c1 < 32) hi1 = lo1 + (u64)(c1 + 1) * st1 - 1;
            lo1 = nlo;
        }
    }
    bool b0 = false, b1 = false;
    if (lo0 + lane < hi0) b0 = ld_probe(a + lo0 + lane) < xlo;
    if (lo1 + lane < hi1) b1 = ld_probe(a + lo1 + lane) <= xhi;
    r0 = lo0 + __popc(__ballot_sync(0xffffffffu, b0));
    r1 = lo1 + __popc(__ballot_sync(0xffffffffu, b1));
}

// Rank of tile candidate idx (value c) among equal values of A: copies before it
// in the tile plus, when the run reaches the tile start, copies before the tile.
__device__ __noinline__ u64 cand_rank(const u64* s_cand, int idx, u64 c, bool has_prev, u64 prev,
                                      const u64* A, u64 a0) {
    int s = idx;
    while (s > 0 && s_cand[s - 1] == c) --s;
    u64 r = (u64)(idx - s);
    if (s == 0 && has_prev && prev == c) r += a0 - lower_bound_g(A, a0, c);
    return r;
}

// Coalesced copy of n values from global src (8-byte aligned) to shared dst,
// re-based to `ref` and narrowed to KT.
template <typename KT>
__device__ __forceinline__ void stage_keys(KT* dst, const u64* __restrict__ src, int n, u64 ref, int tid) {
    if (n <= 0) return;
    const int head = (int)((reinterpret_cast<uintptr_t>(src) >> 3) & 1);
    if (tid == 0 && head) dst[0] = (KT)(ld_stream(src) - ref);
    const int npairs = (n - head) >> 1;
    KT* d = dst + head;
    const u64* s = src + head;
    for (int i = tid; i < npairs; i += F_NT) {
        ulonglong2 v = ld_stream2(s + 2 * i);
        d[2 * i] = (KT)(v.x - ref);
        d[2 * i + 1] = (KT)(v.y - ref);
    }
    if (tid == 32 && ((n - head) & 1)) dst[n - 1] = (KT)(ld_stream(src + n - 1) - ref);
}

// First index in sb[0..n) (1 <= n < 2^15) with sb[i] >= x, by binary lifting: the
// step ladder is entered at the largest power of two <= n, so the instruction
// sequence depends only on n and a warp searching one slice never diverges.
template <typename KT>
__device__ __forceinline__ int lower_bound_lift(const KT* sb, int n, KT x) {
    int base = 0;
#define DGX_LIFT(H) { const int t_ = base + (H); if (t_ <= n && sb[t_ - 1] < x) base = t_; }
    switch (31 - __clz(n)) {
        case 14: DGX_LIFT(16384)
        case 13: DGX_LIFT(8192)
        case 12: DGX_LIFT(4096)
        case 11: DGX_LIFT(2048)
        case 10: DGX_LIFT(1024)
        case 9: DGX_LIFT(512)
        case 8: DGX_LIFT(256)
        case 7: DGX_LIFT(128)
        case 6: DGX_LIFT(64)
        case 5: DGX_LIFT(32)
        case 4: DGX_LIFT(16)
        case 3: DGX_LIFT(8)
        case 2: DGX_LIFT(4)
        case 1: DGX_LIFT(2)
        default: DGX_LIFT(1)
    }
#undef DGX_LIFT
    return base;
}

struct FSlice {       // one filter list of the current batch (shared memory)
    const u64* ptr;
    u64 r0, r1, len;
};

struct FTileCtx {       // per-thread view of the tile
    const u64* s_cand;  // the tile's original candidates (for duplicate ranks)
    const u64* A;
    u64 a0, prev, tlo;
    bool has_prev;
    int cidx0;          // tile index of this lane's row-0 candidate while candidates are in place
    int op;
};

// Resolve this lane's live candidates against staged keys sb[0..n), n >= 1, whose
// first value is element g0 of list B.  kChunked: only candidates <= the chunk's
// last value (or all, in the last chunk) are decided now and recorded in `resolved`.
template <typename KT, bool kChunked>
__device__ __forceinline__ void probe_rows(const FTileCtx& X, const u64 (&c)[F_VA], unsigned& alive, unsigned dup,
                                           int rows, unsigned& resolved, const KT* sb, int n, u64 g0,
                                           bool last_chunk, const u64* __restrict__ B, u64 lenB) {
    const KT chunk_last = kChunked ? sb[n - 1] : (KT)0;
#pragma unroll
    for (int i = 0; i < F_VA; ++i) {
        if (i < rows) {  // warp-uniform
            const KT x = (KT)(c[i] - X.tlo);
            bool todo = (alive >> i) & 1u;
            if (kChunked) todo = todo && !((resolved >> i) & 1u) && (last_chunk || x <= chunk_last);
            const int p = lower_bound_lift<KT>(sb, n, x);  // whole warp, no divergence
            if (todo) {
                bool h;
                if (!((dup >> i) & 1u)) {
                    h = (p < n) && (sb[p] == x);
                } else {
                    const u64 g = g0 + (u64)p + cand_rank(X.s_cand, X.cidx0 + 32 * i, c[i], X.has_prev, X.prev, X.A, X.a0);
                    h = (g < lenB) && (ld_probe(B + g) == c[i]);
                }
                if ((X.op == 0) != h) alive &= ~(1u << i);  // intersect drops misses, difference drops hits
                if (kChunked) resolved |= 1u << i;
            }
        }
    }
}

// Re-pack a warp's survivors into rows 0..ceil(live/32)-1 (order preserved).
__device__ __forceinline__ void warp_repack(u64 (&c)[F_VA], unsigned& alive, int& rows, u64* s_w, int lane) {
    unsigned b[F_VA];
    int tot = 0;
#pragma unroll
    for (int i = 0; i < F_VA; ++i) {
        b[i] = __ballot_sync(0xffffffffu, (i < rows) && ((alive >> i) & 1u));
        tot += __popc(b[i]);
    }
    const int nrows = (tot + 31) >> 5;
    if (nrows >= rows) return;  // warp-uniform
    if (nrows == 0) { rows = 0; alive = 0; return; }
    const unsigned lt = (1u << lane) - 1u;
    int before = 0;
#pragma unroll
    for (int i = 0; i < F_VA; ++i) {
        if ((b[i] >> lane) & 1u) s_w[before + __popc(b[i] & lt)] = c[i];
        before += __popc(b[i]);
    }
    __syncwarp();
    alive = 0;
#pragma unroll
    for (int i = 0; i < F_VA; ++i) {
        if (i < nrows && 32 * i + lane < tot) {
            c[i] = s_w[32 * i + lane];
            alive |= 1u << i;
        }
    }
    __syncwarp();
    rows = nrows;
}

struct FShared {
    FSlice sl[F_LB];
    u64 prefix;
    u32 wcnt[F_NW];
    u32 tile, task;
};

template <typename KT>
__device__ __forceinline__ void filter_tile(const FParams& P, const FTask& T, FShared& S, u64* s_cand, u64* s_work,
                                            KT* s_l, FTileCtx& X, int na, u64 tlo, u64 thi,
                                            u64 (&c)[F_VA], unsigned& alive) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int scap = (int)(P.scap_bytes / sizeof(KT));
    unsigned dup = 0;
    int rows = 0;             // live rows of this warp (warp-uniform)
    bool have_c = false;      // block-uniform
    bool tile_dup = false;    // block-uniform: the tile holds repeated values -> candidates stay in place
    bool packed_once = false; // block-uniform: the one block-level re-pack has happened
    u64* s_w = s_work + F_WC * wid;

    for (u32 j = 1; j < T.k; j += F_LB) {
        // ---- slice bounds of lists j .. j+F_LB-1: one warp per list ------------------
        if (j + wid < T.k) {
            const FList Lq = P.lists[T.list_first + j + wid];
            const u64 ln = flist_len(Lq);
            u64 r0, r1;
            warp_bounds2_g(Lq.ptr, ln, tlo, thi, lane, r0, r1);
            if (lane == 0) { S.sl[wid].ptr = Lq.ptr; S.sl[wid].r0 = r0; S.sl[wid].r1 = r1; S.sl[wid].len = ln; }
        }
        __syncthreads();  // bounds visible; candidate staging complete
        const bool first_batch = !have_c;
        if (first_batch) {
            const int wn = na - F_WC * wid;  // candidates of this warp
            rows = wn <= 0 ? 0 : (wn >= F_WC ? F_VA : (wn + 31) >> 5);
#pragma unroll
            for (int i = 0; i < F_VA; ++i) {
                const int idx = X.cidx0 + 32 * i;
                if (idx < na) {
                    c[i] = s_cand[idx];
                    alive |= 1u << i;
                    const u64 before = idx > 0 ? s_cand[idx - 1] : X.prev;
                    if ((idx > 0 || X.has_prev) && before == c[i]) dup |= 1u << i;
                }
            }
            have_c = true;
        }
        const int nb = (int)((T.k - j < (u32)F_LB) ? (T.k - j) : (u32)F_LB);  // lists in this batch
        int jj = 0;
        bool dead = false;
        bool need_dup_vote = first_batch;
        while (jj < nb && !dead) {
            const u64 sz0 = S.sl[jj].r1 - S.sl[jj].r0;
            if (sz0 > (u64)scap) {
                // ---- oversized slice: stream in chunks, or probe global memory --------
                const u64* __restrict__ B = S.sl[jj].ptr;
                const u64 lenB = S.sl[jj].len, r0 = S.sl[jj].r0, r1 = S.sl[jj].r1;
                if (need_dup_vote) { tile_dup = __syncthreads_or(dup != 0) != 0; need_dup_vote = false; }
                const int live_threads = __syncthreads_count(alive != 0);
                if (live_threads == 0) { dead = true; break; }
                if (sz0 <= (u64)P.stream_ratio * (u64)(F_VA * live_threads)) {
                    unsigned resolved = 0;
                    for (u64 cs = r0; cs < r1; cs += (u64)scap) {
                        const int n = (int)((r1 - cs < (u64)scap) ? (r1 - cs) : (u64)scap);
                        const bool last = cs + (u64)n >= r1;
                        stage_keys<KT>(s_l, B + cs, n, tlo, tid);
                        __syncthreads();
                        probe_rows<KT, true>(X, c, alive, dup, rows, resolved, s_l, n, cs, last, B, lenB);
                        __syncthreads();
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < F_VA; ++i) {
                        if ((alive >> i) & 1u) {
                            const u64 x = c[i];
                            u64 g = r0 + lower_bound_g(B + r0, sz0, x);
                            if ((dup >> i) & 1u) g += cand_rank(s_cand, X.cidx0 + 32 * i, x, X.has_prev, X.prev, X.A, X.a0);
                            const bool h = (g < lenB) && (ld_probe(B + g) == x);
                            if ((P.op == 0) != h) alive &= ~(1u << i);
                        }
                    }
                }
                if (!tile_dup) warp_repack(c, alive, rows, s_w, lane);
                ++jj;
                continue;
            }
            // ---- stage as many whole slices as fit, then probe them barrier-free ------
            int je = jj, used = 0;
            while (je < nb) {
                const u64 sz = S.sl[je].r1 - S.sl[je].r0;
                if (sz > (u64)(scap - used)) break;
                used += (int)((sz + 3) & ~3ull);  // keep every slice 16-byte aligned in shared memory
                if (used > scap) { used = scap; }
                ++je;
            }
            {
                int o = 0;
                for (int t = jj; t < je; ++t) {
                    const int n = (int)(S.sl[t].r1 - S.sl[t].r0);
                    stage_keys<KT>(s_l + o, S.sl[t].ptr + S.sl[t].r0, n, tlo, tid);
                    o += (n + 3) & ~3;
                }
            }
            if (need_dup_vote) { tile_dup = __syncthreads_or(dup != 0) != 0; need_dup_vote = false; }
            else __syncthreads();
            {
                int o = 0;
                for (int t = jj; t < je; ++t) {
                    const int n = (int)(S.sl[t].r1 - S.sl[t].r0);
                    if (rows > 0) {
                        if (n == 0) {
                            if (P.op == 0) { alive = 0; rows = 0; }  // nothing of L_t in range: every candidate misses
                        } else {
                            unsigned dummy = 0;
                            probe_rows<KT, false>(X, c, alive, dup, rows, dummy, s_l + o, n, S.sl[t].r0, true,
                                                  S.sl[t].ptr, S.sl[t].len);
                        }
                    }
                    o += (n + 3) & ~3;
                    const bool more = (t + 1 < je) || (je < nb) || (j + F_LB < T.k);
                    if (!more || tile_dup) continue;
                    if (!packed_once) {
                        // ---- one block-level re-pack after the first list (block-uniform path) ----
                        packed_once = true;
                        unsigned b[F_VA];
                        int wtot = 0;
#pragma unroll
                        for (int i = 0; i < F_VA; ++i) {
                            b[i] = __ballot_sync(0xffffffffu, (alive >> i) & 1u);
                            wtot += __popc(b[i]);
                        }
                        if (lane == 0) S.wcnt[wid] = (u32)wtot;
                        __syncthreads();
                        int woff = 0, total = 0;
#pragma unroll
                        for (int w = 0; w < F_NW; ++w) {
                            const int v = (int)S.wcnt[w];
                            if (w < wid) woff += v;
                            total += v;
                        }
                        if (total == 0) { dead = true; alive = 0; rows = 0; break; }
                        if (total <= F_TA / 2) {
                            const unsigned lt = (1u << lane) - 1u;
                            int before = woff;
#pragma unroll
                            for (int i = 0; i < F_VA; ++i) {
                                if ((b[i] >> lane) & 1u) s_work[before + __popc(b[i] & lt)] = c[i];
                                before += __popc(b[i]);
                            }
                            __syncthreads();
                            const int R = (total + F_NT - 1) / F_NT;  // rows per warp afterwards (1 or 2)
                            const int start = wid * 32 * R;
                            alive = 0;
                            rows = 0;
#pragma unroll
                            for (int i = 0; i < F_VA; ++i) {
                                const int idx = start + 32 * i + lane;
                                if (i < R && start + 32 * i < total) {
                                    rows = i + 1;
                                    if (idx < total) { c[i] = s_work[idx]; alive |= 1u << i; }
                                }
                            }
                            __syncthreads();  // s_work is reused for warp re-packs from here on
                        }
                    } else {
                        warp_repack(c, alive, rows, s_w, lane);
                    }
                }
            }
            if (dead) break;
            jj = je;
            if (jj < nb || j + F_LB < T.k) {
                // more lists follow: everyone is done with the staging area; stop if nothing is alive
                if (__syncthreads_count(alive != 0) == 0) dead = true;
            }
        }
        if (dead) { alive = 0; break; }
    }
    if (!have_c) {  // k == 1: plain copy of A (IntersectSorted of one list, algo/uidlist.go:313-316)
        __syncthreads();
#pragma unroll
        for (int i = 0; i < F_VA; ++i) {
            const int idx = X.cidx0 + 32 * i;
            if (idx < na) { c[i] = s_cand[idx]; alive |= 1u << i; }
        }
    }
}

__global__ void __launch_bounds__(F_NT) filter_kernel(const FParams P) {
    extern __shared__ __align__(16) u64 s_dyn[];   // [F_TA tile | F_TA re-pack area | staged slice keys]
    u64* s_cand = s_dyn;
    u64* s_work = s_dyn + F_TA;
    __shared__ FShared S;

    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;

    if (tid == 0) {
        const u32 t = atomicAdd(P.ticket, 1u);
        // tile -> task: last task with tile_base <= tile
        u32 lo = 0, hi = P.ntasks;
        while (hi - lo > 1) {
            u32 mid = (lo + hi) >> 1;
            if (P.tasks[mid].tile_base <= (u64)t) lo = mid; else hi = mid;
        }
        S.tile = t;
        S.task = lo;
    }
    __syncthreads();
    const u32 tile = S.tile, q = S.task;
    const FTask T = P.tasks[q];
    const FList LA = P.lists[T.list_first];
    const u64 lenA = flist_len(LA);
    const u64* __restrict__ A = LA.ptr;
    const u64 a0 = (u64)(tile - T.tile_base) * F_TA;
    const int na = a0 < lenA ? (int)((lenA - a0 < (u64)F_TA) ? (lenA - a0) : (u64)F_TA) : 0;

    stage_keys<u64>(s_cand, A + a0, na, 0, tid);
    FTileCtx X;
    X.s_cand = s_cand; X.A = A; X.a0 = a0; X.op = P.op;
    X.has_prev = (a0 > 0) && (na > 0);
    X.prev = 0;
    X.cidx0 = F_WC * wid + lane;
    u64 tlo = 0, thi = 0;  // tile's first / last value straight from global (no wait on staging)
    if (na > 0) {
        tlo = ld_probe(A + a0);
        thi = ld_probe(A + a0 + na - 1);
        if (X.has_prev) X.prev = ld_probe(A + a0 - 1);
    }
    X.tlo = tlo;

    u64 c[F_VA] = {0, 0, 0, 0};
    unsigned alive = 0;
    if (na > 0) {
        if (thi - tlo < 0xffffffffull)
            filter_tile<u32>(P, T, S, s_cand, s_work, reinterpret_cast<u32*>(s_dyn + 2 * F_TA), X, na, tlo, thi, c, alive);
        else
            filter_tile<u64>(P, T, S, s_cand, s_work, s_dyn + 2 * F_TA, X, na, tlo, thi, c, alive);
    }

    // ---- output: per-warp counts -> tile prefix (look-back) -> ordered stores -----------
    unsigned b[F_VA];
    int wtot = 0;
#pragma unroll
    for (int i = 0; i < F_VA; ++i) {
        b[i] = __ballot_sync(0xffffffffu, (alive >> i) & 1u);
        wtot += __popc(b[i]);
    }
    __syncthreads();  // S.wcnt may still be read by the block re-pack
    if (lane == 0) S.wcnt[wid] = (u32)wtot;
    __syncthreads();
    u32 woff = 0, total = 0;
#pragma unroll
    for (int w = 0; w < F_NW; ++w) {
        const u32 v = S.wcnt[w];
        if (w < wid) woff += v;
        total += v;
    }
    if (wid == 0) {
        u64 ex = lookback_exclusive(P.status, tile, (u64)total, lane);
        if (lane == 0) S.prefix = ex;
    }
    __syncthreads();
    const u64 base = S.prefix;
    if (tid == 0) {
        if ((u64)tile == T.tile_base) P.out_off[q] = base;
        if (tile == P.ntiles - 1) P.out_off[P.ntasks] = base + (u64)total;
    }
    if (base + (u64)total > P.out_cap) {
        if (tid == 0) atomicExch(P.err, 1);
    } else {
        u64* dst = P.out + base + woff;
        const unsigned lt = (1u << lane) - 1u;
        int before = 0;
#pragma unroll
        for (int i = 0; i < F_VA; ++i) {
            if ((b[i] >> lane) & 1u) st_stream(dst + before + __popc(b[i] & lt), c[i]);
            before += __popc(b[i]);
        }
    }
}

}  // namespace dgx
