// merge_matrix.cuh -- algo.MergeSorted over the rows of a uid matrix, as a sample sort (sm_90a).
//
// sg.DestUIDs = algo.MergeSorted(result.UidMatrix) (query/query.go:2290) unions many short sorted rows.  The pairwise
// merge tree makes ceil(log2 nrows) passes over the whole matrix and the multiway merge stops at 64 runs, so the rows are
// first cut into tiles of fixed size, whatever their lengths, and the tiles are sample-sorted into disjoint value ranges:
//   xm_tile_kernel       CTA per tile of XM_T consecutive positions of v: the rows-ascend check (each element's row by
//                        a search of v_off narrowed to the tile's rows), a bitonic sort of the tile in shared memory,
//                        de-duplication; writes the tile's sorted distinct run, its length and every XM_S-th value as a
//                        sample
//   merge_tree_impl      (merge_kernel.cuh, unchanged) the sorted sample runs -> the distinct sorted samples, the
//                        splitters s_0 < s_1 < ... (their count stays on the device)
//   xm_count_kernel      CTA per run: every value's key -- 2b for the open bucket (s_{b-1}, s_b), 2b + 1 for the
//                        equality bucket {s_b} -- counted per warp segment of equal keys (a run is sorted, so equal keys
//                        are adjacent); an equality bucket only records presence (it is emitted once, never sorted)
//   scan_u64_kernel      key sizes -> key offsets: the buckets in value order
//   xm_scatter_kernel    CTA per run: values to their bucket; the present splitters to their equality slots
//   xm_chunk_kernel      CTA per chunk of XM_H positions: the whole buckets that start in it (fewer than XM_H plus one
//                        bucket of values) are sorted in shared memory and de-duplicated in place.  A chunk larger than
//                        shared memory (a bucket of more than XM_H values, which regular samples allow on adversarial
//                        input) takes the overflow path: a bitonic sort of the chunk in global memory by the same CTA,
//                        counted in the lane's overflow word
//   scan_u64_kernel      distinct counts per chunk -> output positions and the result length
//   xm_gather_kernel     CTA per chunk: its distinct values to out
// Buckets hold disjoint value ranges in ascending order, so the concatenated chunks are the sorted union, and a value
// occurs in one bucket only, so de-duplicating inside a chunk de-duplicates globally.  Launches: 7 plus the sample tree's
// ceil(log2 (number of tiles)) levels, whatever nrows is.
#pragma once

#include "common.cuh"
#include "compressed_kernel.cuh"  // kLaneErrOrder

namespace dgx {

constexpr int XM_NT = 256, XM_VT = 8, XM_T = XM_NT * XM_VT;  // tile pass: 2048 positions per CTA
constexpr int XM_S = 32;                                     // every XM_S-th distinct value of a run is a sample
constexpr int XM_SPR = XM_T / XM_S;                          // sample slots per run
constexpr int XM_CNT = 512, XM_CAP = 4096, XM_H = XM_CAP / 2;  // chunk pass: threads, shared capacity, chunk stride
constexpr u32 XM_EQ_NONE = 0xffffffffu;                      // key of a value that sits in an equality bucket
constexpr int kLaneOverflowWord = 4;                         // u32 index in the lane's error block: overflow chunks

struct XmParams {
    const u64* v;        // values, rows concatenated
    const u64* v_off;    // nrows + 1 (device)
    u64 nrows;
    u64 v_cap;           // values readable behind v; d_v_off[nrows] > v_cap is DGX_ERR_CAP
    u64* runs;           // ntiles * XM_T: tile t's sorted distinct run at t * XM_T
    u32* rlen;           // ntiles: run lengths
    u64* samples;        // ntiles * XM_SPR
    u64* soff;           // 2 * ntiles: [first, end) of tile t's samples (MRef::off of the sample tree)
    u32 ntiles;
    const u64* split;    // distinct sorted samples (the splitters)
    const u64* nsplit;   // device word: their count
    u32* key;            // per run slot: bucket key, XM_EQ_NONE for an equality value
    u64* kcnt;           // 2 * nsplit_cap + 1: open-bucket sizes (even), equality presence (odd); zero-initialised
    u64* koff;           // 2 * nsplit_cap + 2: exclusive scan of kcnt
    u64* kfill;          // 2 * nsplit_cap + 1: values placed so far; zero-initialised
    u64* nkeys;          // device word: 2 * nsplit + 1
    u64* nch;            // device word: nchunks (the length of the chunk scan)
    u64* bucketed;       // values in bucket order (<= number of run values), de-duplicated in place per chunk
    u32 nchunks;
    u64* cstart;         // per chunk: first position in bucketed
    u64* ccount;         // per chunk: distinct values
    u64* cpos;           // nchunks + 1: exclusive scan of ccount
    u64* out;
    u64 out_cap;
    int* err;
};

// Bitonic sort of a[0 .. n) in ascending order with every compare-exchange ascending (first step of each merge compares
// mirrored positions), so positions >= n act as +infinity and are never touched.  Called by all NT threads of a CTA.
template <int NT, typename Idx, typename Ptr>
__device__ __forceinline__ void xm_bitonic(Ptr a, Idx n) {
    Idx np2 = 1;
    while (np2 < n) np2 <<= 1;
    for (Idx k = 2; k <= np2; k <<= 1) {
        for (Idx j = k >> 1; j > 0; j >>= 1) {
            for (Idx p = threadIdx.x; p < (np2 >> 1); p += NT) {
                const Idx i = ((p & ~(j - 1)) << 1) | (p & (j - 1));  // p with a zero bit inserted at j
                const Idx q = (j == (k >> 1)) ? (i ^ (k - 1)) : (i | j);
                if (q < n) {
                    const u64 x = a[i], y = a[q];
                    if (y < x) { a[i] = y; a[q] = x; }
                }
            }
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(XM_NT) xm_tile_kernel(const XmParams P) {
    __shared__ u64 s[XM_T];
    __shared__ u32 s_scan[XM_NT / 32 + 1];
    __shared__ u64 s_row[2];
    const int tid = threadIdx.x;
    const u32 t = blockIdx.x;
    u64 m = P.v_off[P.nrows];
    if (m > P.v_cap) {
        if (t == 0 && tid == 0) atomicOr(P.err, 1);
        m = 0;
    }
    const u64 start = (u64)t * XM_T;
    const int n = m <= start ? 0 : (m - start < (u64)XM_T ? (int)(m - start) : XM_T);
    if (n == 0) {
        if (tid == 0) { P.rlen[t] = 0; P.soff[2 * t] = P.soff[2 * t + 1] = (u64)t * XM_SPR; }
        return;
    }
    if (tid < 2) {  // rows of the first / last position: last r with v_off[r] <= pos
        const u64 pos = tid == 0 ? start : start + n - 1;
        u64 lo = 0, hi = P.nrows;
        while (lo < hi) {
            const u64 mid = lo + ((hi - lo + 1) >> 1);
            if (ld_probe(P.v_off + mid) <= pos) lo = mid; else hi = mid - 1;
        }
        s_row[tid] = lo;
    }
    __syncthreads();
    const u64 r0 = s_row[0], r1 = s_row[1];
    bool bad = false;
    for (int i = tid; i < n; i += XM_NT) {
        const u64 j = start + i;
        const u64 x = ld_stream(P.v + j);
        s[i] = x;
        u64 lo = r0, hi = r1;
        while (lo < hi) {
            const u64 mid = lo + ((hi - lo + 1) >> 1);
            if (ld_probe(P.v_off + mid) <= j) lo = mid; else hi = mid - 1;
        }
        if (j > 0 && ld_probe(P.v_off + lo) != j && x < ld_probe(P.v + j - 1)) bad = true;  // inside a row: no descent
    }
    if (bad) atomicOr(P.err, kLaneErrOrder);
    __syncthreads();
    xm_bitonic<XM_NT, int>(s, n);
    // thread k owns sorted positions [k * XM_VT, k * XM_VT + XM_VT)
    u64 vals[XM_VT];
    u32 keep = 0;
#pragma unroll
    for (int q = 0; q < XM_VT; ++q) {
        const int i = tid * XM_VT + q;
        if (i < n) {
            vals[q] = s[i];
            if (i == 0 || vals[q] != s[i - 1]) keep |= 1u << q;
        }
    }
    u32 total;
    u32 pos = block_exclusive_scan<XM_NT>(__popc(keep), s_scan, &total);
    u64* run = P.runs + (u64)t * XM_T;
    u64* smp = P.samples + (u64)t * XM_SPR;
#pragma unroll
    for (int q = 0; q < XM_VT; ++q)
        if ((keep >> q) & 1u) {
            run[pos] = vals[q];
            if (pos % XM_S == 0) smp[pos / XM_S] = vals[q];
            ++pos;
        }
    if (tid == 0) {
        P.rlen[t] = total;
        P.soff[2 * t] = (u64)t * XM_SPR;
        P.soff[2 * t + 1] = (u64)t * XM_SPR + (total + XM_S - 1) / XM_S;
    }
}

// Key of x: 2b + 1 when x == s_b, else 2b for the open bucket below s_b (b = nsplit: above the last splitter).
__device__ __forceinline__ u32 xm_key(const u64* split, u64 lo, u64 hi, u64 nsplit, u64 x, bool* eq) {
    while (lo < hi) {
        const u64 mid = lo + ((hi - lo) >> 1);
        if (ld_probe(split + mid) < x) lo = mid + 1; else hi = mid;
    }
    *eq = lo < nsplit && ld_probe(split + lo) == x;
    return (u32)(2 * lo + (*eq ? 1 : 0));
}

__global__ void __launch_bounds__(XM_NT) xm_count_kernel(const XmParams P) {
    __shared__ u64 s_rng[2];
    const int tid = threadIdx.x, lane = tid & 31;
    const u32 t = blockIdx.x;
    const u64 nsplit = *P.nsplit;
    if (t == 0 && tid == 0) { *P.nkeys = 2 * nsplit + 1; *P.nch = P.nchunks; }
    const int n = (int)P.rlen[t];
    if (n == 0) return;
    const u64* run = P.runs + (u64)t * XM_T;
    if (tid < 2) {  // the run's splitter range: the first value's lower bound .. the last value's
        const u64 x = run[tid == 0 ? 0 : n - 1];
        u64 lo = 0, hi = nsplit;
        while (lo < hi) {
            const u64 mid = lo + ((hi - lo) >> 1);
            if (ld_probe(P.split + mid) < x) lo = mid + 1; else hi = mid;
        }
        s_rng[tid] = lo;
    }
    __syncthreads();
    const u64 lo = s_rng[0], hi = s_rng[1];  // every key of the run lies in [lo, hi]
    u32* key = P.key + (u64)t * XM_T;
    for (int i0 = 0; i0 < n; i0 += XM_NT) {  // warp-uniform trip count: __match_any_sync needs whole warps
        const int i = i0 + tid;
        const bool live = i < n;
        const u64 x = run[live ? i : n - 1];
        // the warp's 32 sorted values narrow every lane's search: a 32-ary warp search for the first and the last
        // value, then each lane searches only between them (a few cached sectors instead of the run's whole range)
        const u64 wlo = lo + warp_bound_g(P.split + lo, hi - lo, __shfl_sync(0xffffffffu, x, 0), false, lane);
        const u64 whi = lo + warp_bound_g(P.split + lo, hi - lo, __shfl_sync(0xffffffffu, x, 31), false, lane);
        bool eq = false;
        const u32 k = live ? xm_key(P.split, wlo, whi, nsplit, x, &eq) : XM_EQ_NONE;
        if (live) key[i] = eq ? XM_EQ_NONE : k;
        if (live && eq) P.kcnt[k] = 1;  // presence only
        const u32 grp = __match_any_sync(0xffffffffu, (live && !eq) ? k : XM_EQ_NONE);
        if (live && !eq && lane == __ffs(grp) - 1) atomicAdd(P.kcnt + k, (u64)__popc(grp));
    }
}

__global__ void __launch_bounds__(XM_NT) xm_scatter_kernel(const XmParams P) {
    const int tid = threadIdx.x, lane = tid & 31;
    const u32 t = blockIdx.x;
    const u64 g = (u64)t * XM_NT + tid;
    if (g < *P.nsplit && P.kcnt[2 * g + 1]) P.bucketed[P.koff[2 * g + 1]] = P.split[g];  // present splitters
    const int n = (int)P.rlen[t];
    const u64* run = P.runs + (u64)t * XM_T;
    const u32* key = P.key + (u64)t * XM_T;
    for (int i0 = 0; i0 < n; i0 += XM_NT) {
        const int i = i0 + tid;
        const u32 k = i < n ? key[i] : XM_EQ_NONE;
        const u32 grp = __match_any_sync(0xffffffffu, k);
        if (k == XM_EQ_NONE) continue;
        const int leader = __ffs(grp) - 1;
        u64 base = 0;
        if (lane == leader) base = atomicAdd(P.kfill + k, (u64)__popc(grp));
        base = __shfl_sync(grp, base, leader);
        P.bucketed[P.koff[k] + base + __popc(grp & ((1u << lane) - 1))] = run[i];
    }
}

// Sorted, de-duplicated a[0 .. n) compacted in place by one CTA (global memory); returns the distinct count.
__device__ u64 xm_dedup_global(u64* a, u64 n, u32* s_scan, u64* s_last) {
    u64 w = 0;
    for (u64 b = 0; b < n; b += XM_CNT) {
        const u64 i = b + threadIdx.x;
        const u64 x = i < n ? a[i] : 0;
        const u64 prev = i == 0 ? 0 : (threadIdx.x == 0 ? *s_last : a[i - 1]);
        const u32 keep = (i < n && (i == 0 || x != prev)) ? 1u : 0u;
        u32 total;
        const u32 pos = block_exclusive_scan<XM_CNT>(keep, s_scan, &total);  // barriers: every read above is done
        if (i < n && (threadIdx.x == XM_CNT - 1 || i == n - 1)) *s_last = x;
        if (keep) a[w + pos] = x;
        w += total;
        __syncthreads();
    }
    return w;
}

__global__ void __launch_bounds__(XM_CNT) xm_chunk_kernel(const XmParams P, u32* overflow) {
    __shared__ u64 s[XM_CAP];
    __shared__ u32 s_scan[XM_CNT / 32 + 1];
    __shared__ u64 s_last;
    const int tid = threadIdx.x;
    const u32 c = blockIdx.x;
    const u64 nk = *P.nkeys, total = P.koff[nk];
    const u64 a = (u64)c * XM_H;
    u64 p0 = total, p1 = total;
    if (a < total) {  // the keys that start in [a, a + XM_H): [first key with koff >= a, first key with koff >= a + XM_H)
        u64 lo = 0, hi = nk;
        while (lo < hi) { const u64 mid = lo + ((hi - lo) >> 1); if (P.koff[mid] < a) lo = mid + 1; else hi = mid; }
        p0 = P.koff[lo];
        hi = nk;
        while (lo < hi) { const u64 mid = lo + ((hi - lo) >> 1); if (P.koff[mid] < a + XM_H) lo = mid + 1; else hi = mid; }
        p1 = P.koff[lo];
    }
    const u64 n = p1 - p0;
    u64* buf = P.bucketed + p0;
    if (tid == 0) P.cstart[c] = p0;
    if (n == 0) {
        if (tid == 0) P.ccount[c] = 0;
        return;
    }
    if (n > (u64)XM_CAP) {  // overflow path: the chunk is sorted where it lies
        if (tid == 0) atomicAdd(overflow, 1u);
        xm_bitonic<XM_CNT, u64>(buf, n);
        const u64 d = xm_dedup_global(buf, n, s_scan, &s_last);
        if (tid == 0) P.ccount[c] = d;
        return;
    }
    const int nn = (int)n;
    for (int i = tid; i < nn; i += XM_CNT) s[i] = buf[i];
    __syncthreads();
    xm_bitonic<XM_CNT, int>(s, nn);
    u64 vals[XM_CAP / XM_CNT];
    u32 keep = 0;
#pragma unroll
    for (int q = 0; q < XM_CAP / XM_CNT; ++q) {
        const int i = tid * (XM_CAP / XM_CNT) + q;
        if (i < nn) {
            vals[q] = s[i];
            if (i == 0 || vals[q] != s[i - 1]) keep |= 1u << q;
        }
    }
    u32 cnt;
    u32 pos = block_exclusive_scan<XM_CNT>(__popc(keep), s_scan, &cnt);
#pragma unroll
    for (int q = 0; q < XM_CAP / XM_CNT; ++q)
        if ((keep >> q) & 1u) buf[pos++] = vals[q];
    if (tid == 0) P.ccount[c] = cnt;
}

__global__ void __launch_bounds__(256) xm_gather_kernel(const XmParams P) {
    const u32 c = blockIdx.x;
    const u64 n = P.ccount[c], o = P.cpos[c];
    if (o + n > P.out_cap && threadIdx.x == 0) atomicOr(P.err, 1);
    const u64* src = P.bucketed + P.cstart[c];
    for (u64 i = threadIdx.x; i < n && o + i < P.out_cap; i += 256) P.out[o + i] = src[i];
}

}  // namespace dgx
