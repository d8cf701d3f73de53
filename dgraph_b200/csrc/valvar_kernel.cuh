// valvar_kernel.cuh -- value variables over uid matrices: transformTo (query/query.go :1143-1236) over a whole path
// and evalLevelAgg's per-row branch (query/query.go :1042-1125), each in one call.
//
// A value map is key[n] (strictly ascending uids) and val[n] (64-bit words: int64 two's complement or IEEE binary64,
// one type per map).  Level k of a path has src (nrows, strictly ascending), rows v[v_off[i] .. v_off[i+1]) and dest
// (strictly ascending, every row value in it).  One level of the propagation, for every map, runs:
//   vv_check_kernel    thread per index: offsets from 0, not decreasing, inside v_cap; src, dest (and the input map's
//                      keys, first level) strictly ascend
//   vv_flags_kernel    thread per value: its row, its rank in dest (absent: refused), whether the row's source is a
//                      key of the current map; a contributing value gets key rank << 2 | range and payload map index
//   scan_u64_kernel    contributing flags -> positions, the count E
//   vv_compact_kernel  the contributing keys and payloads, in value (row-major) order
//   3 x P launches     the groupby stable LSD radix sort (gb_hist_kernel, scan_u64_kernel, gb_scatter_kernel) by
//                      rank << 2 | range: P = ceil((b_d + 2) / 8), b_d the bit width of ndest - 1.  Stable, so each
//                      (rank, range) segment keeps row-major order
//   vv_heads_kernel    thread per item: segment start (low word) and rank start (high word) packed in one u64
//   scan_u64_kernel    both counts at once: segment index and rank index of every item, S and G
//   vv_starts_kernel   each segment's first item
//   vv_fold_kernel     float64: thread per segment, the ordered fold of Go's per-range loop; int64 (order-free):
//                      thread per item, a warp-segmented sum and one atomicAdd per run of a segment
//   vv_combine_kernel  thread per rank head: the ranges merged in ascending order into the next map (key dest[rank]),
//                      or into the outputs at the last level
// The launch count is 9 + 3 P per level, set by nlevels and the dest sizes alone.
//
// The level aggregation runs la_check_kernel, la_fold_kernel (warp per row: lanes look the values up, every lane folds
// the present ones in row order through shuffles), scan_u64_kernel and la_write_kernel: 4 launches.
#pragma once

#include "groupby_kernel.cuh"  // gb_hist_kernel, gb_scatter_kernel; scan_u64_kernel via encode_kernel.cuh

namespace dgx {

constexpr int kLaneErrVar = 256;  // lane error flag bit: a value-variable input is malformed (DGX_ERR_ARG at sync)
constexpr int kVvInt64 = 1, kVvFloat64 = 2;                      // DGX_VAL_*
constexpr int kVaMin = 0, kVaMax = 1, kVaSum = 2, kVaAvg = 3;    // DGX_AGG_*
constexpr int VV_RANGES = 4, VV_RANGE_BITS = 2;                  // numThreadsVariablePropogation
// words of one level: values, contributing values, packed segment | rank totals, hist length, the first map's size,
// the size of the map it makes
constexpr int VV_W_M = 0, VV_W_E = 1, VV_W_SG = 2, VV_W_H = 3, VV_W_N0 = 4, VV_W_NX = 5, VV_WORDS = 6;

struct VvParams {
    const u64* mk;      // the map this level reads: keys, values, size word
    const u64* mv;
    const u64* mn;
    const u64* src;
    u64 nrows;
    const u64* v_off;   // nrows + 1
    const u64* v;
    u64 v_cap;
    const u64* dest;
    u64 ndest;
    u64 n0;             // first level: the input map's size (written to words[VV_W_N0] for mn)
    int first, is_float;
    u64 tiles;          // radix tiles over max(v_cap, 1)
    u64* words;         // VV_WORDS, zeroed
    int* bad;           // zeroed, shared by every level of the call
    int* err;
    u64* flag;          // v_cap
    u64* pos;           // v_cap + 1
    u64* ek;            // v_cap: the sorted keys (where the sort leaves them)
    u64* ek_raw;        // v_cap: keys in value order
    u32* ep;            // v_cap: sorted payloads
    u32* ep_raw;        // v_cap
    u64* ek_in;         // v_cap: compacted keys, the sort's input
    u32* ep_in;
    u64* head;          // v_cap
    u64* hidx;          // v_cap + 1
    u64* sstart;        // v_cap + 1
    u64* part;          // v_cap
    u64* ok;            // the next map (or the outputs): keys, values, size word, room
    u64* ov;
    u64* on;
    u64 o_cap;
};

__device__ __forceinline__ void vv_refuse(int* bad, int* err) {
    atomicOr(bad, 1);
    atomicOr(err, kLaneErrVar);
}

// aggregator.Value: +Inf -> MaxFloat64, -Inf -> -MaxFloat64, NaN -> +0.0.
__device__ __forceinline__ double vv_clamp(double x) {
    if (x != x) return 0.0;
    if (x == __longlong_as_double(0x7ff0000000000000ll)) return 1.7976931348623157e308;
    if (x == __longlong_as_double((long long)0xfff0000000000000ull)) return -1.7976931348623157e308;
    return x;
}

// One step of transformTo's sum with Value() after it: clamp(a + b) for floats, a wrapping add for ints.
__device__ __forceinline__ u64 vv_add(u64 a, u64 b, int is_float) {
    if (!is_float) return a + b;
    return (u64)__double_as_longlong(vv_clamp(__dadd_rn(__longlong_as_double((long long)a),
                                                         __longlong_as_double((long long)b))));
}

__device__ __forceinline__ u64 vv_first(u64 a, int is_float) {
    return is_float ? (u64)__double_as_longlong(vv_clamp(__longlong_as_double((long long)a))) : a;
}

// Go's range of row r: width = nrows / 4, the last range running to nrows.
__device__ __forceinline__ u32 vv_range(u64 r, u64 nrows) {
    const u64 w = nrows / VV_RANGES;
    if (w == 0) return VV_RANGES - 1;
    const u64 q = r / w;
    return q < VV_RANGES - 1 ? (u32)q : VV_RANGES - 1;
}

// Grid over max(nrows + 1, v_cap, ndest, first ? n0 : 0) threads.
__global__ void __launch_bounds__(256) vv_check_kernel(const VvParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    if (t == 0) {
        const bool ok = P.v_off[0] == 0 && P.v_off[P.nrows] <= P.v_cap;
        bad = !ok;
        P.words[VV_W_M] = ok ? P.v_off[P.nrows] : 0;
        if (P.first) P.words[VV_W_N0] = P.n0;
    }
    if (t < P.nrows) {
        if (t > 0 && P.src[t - 1] >= P.src[t]) bad = true;
        if (P.v_off[t] > P.v_off[t + 1]) bad = true;
    }
    if (t > 0 && t < P.ndest && P.dest[t - 1] >= P.dest[t]) bad = true;
    if (P.first && t > 0 && t < P.n0 && P.mk[t - 1] >= P.mk[t]) bad = true;
    if (bad) vv_refuse(P.bad, P.err);
}

// Thread per value (grid over v_cap).  A refused call flags nothing.
__global__ void __launch_bounds__(256) vv_flags_kernel(const VvParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.words[VV_W_M]) return;
    P.flag[t] = 0;
    if (*P.bad) return;
    const u64 r = lower_bound_g(P.v_off, P.nrows + 1, t + 1) - 1;
    const u64 x = P.v[t];
    const u64 d = lower_bound_g(P.dest, P.ndest, x);
    if (d == P.ndest || P.dest[d] != x) {
        vv_refuse(P.bad, P.err);
        return;
    }
    const u64 n = *P.mn, s = P.src[r];
    const u64 j = lower_bound_g(P.mk, n, s);
    if (j == n || P.mk[j] != s) return;
    P.flag[t] = 1;
    P.ek_raw[t] = (d << VV_RANGE_BITS) | vv_range(r, P.nrows);
    P.ep_raw[t] = (u32)j;
}

// Grid over v_cap threads: the contributing values at their positions, in value order.
__global__ void __launch_bounds__(256) vv_compact_kernel(const VvParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t == 0) P.words[VV_W_H] = (u64)GB_RADIX * P.tiles;
    if (*P.bad || t >= P.words[VV_W_M] || !P.flag[t]) return;
    P.ek_in[P.pos[t]] = P.ek_raw[t];
    P.ep_in[P.pos[t]] = P.ep_raw[t];
}

// Thread per sorted item: 1 where a (rank, range) segment starts, 1 << 32 where a rank starts.
__global__ void __launch_bounds__(256) vv_heads_kernel(const VvParams P) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || k >= P.words[VV_W_E]) return;
    const u64 key = P.ek[k];
    const u64 prev = k ? P.ek[k - 1] : ~0ull;
    P.head[k] = (u64)(key != prev) | ((u64)((key >> VV_RANGE_BITS) != (prev >> VV_RANGE_BITS)) << 32);
}

// Thread per sorted item: sstart[s] = the first item of segment s; sstart[S] = E.
__global__ void __launch_bounds__(256) vv_starts_kernel(const VvParams P) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    const u64 E = P.words[VV_W_E];
    if (k == 0) P.sstart[P.words[VV_W_SG] & 0xffffffffull] = E;
    if (k < E && (P.head[k] & 1)) {
        P.sstart[P.hidx[k] & 0xffffffffull] = k;
        if (!P.is_float) P.part[P.hidx[k] & 0xffffffffull] = 0;  // the int sums accumulate into it
    }
}

// int64: wrapping adds give the same sum in any order, so a thread per item adds its map value into its segment's
// part: a segmented scan across the warp (the items are sorted, so a segment is a run of lanes) and one atomicAdd per
// run.  A hub then costs its items over the whole grid, not one thread's chain.
__device__ __forceinline__ void vv_sum_items(const VvParams& P) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const bool ok = k < P.words[VV_W_E];
    const u64 seg = ok ? ((P.hidx[k] + P.head[k]) & 0xffffffffull) - 1 : ~0ull;  // hidx counts the heads before k
    u64 x = ok ? __ldg(P.mv + __ldg(P.ep + k)) : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u64 y = __shfl_up_sync(0xffffffffu, x, d), sy = __shfl_up_sync(0xffffffffu, seg, d);
        if (lane >= d && sy == seg) x += y;
    }
    const u64 next = __shfl_down_sync(0xffffffffu, seg, 1);
    if (ok && (lane == 31 || next != seg)) atomicAdd((unsigned long long*)(P.part + seg), (unsigned long long)x);
}

// float64: thread per segment, calculate()'s loop for one dst in one range, its contributions in row-major order.
// The map values are gathered eight ahead of the dependent chain of adds.  int64: vv_sum_items (grid over v_cap).
__global__ void __launch_bounds__(256) vv_fold_kernel(const VvParams P) {
    if (*P.bad) return;
    if (!P.is_float) {
        vv_sum_items(P);
        return;
    }
    const u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= (P.words[VV_W_SG] & 0xffffffffull)) return;
    const u64 a = P.sstart[s], b = P.sstart[s + 1];
    const int fl = 1;  // float64: the int64 path returned above
    u64 acc = vv_first(__ldg(P.mv + P.ep[a]), fl);
    u64 k = a + 1;
    for (; k + 8 <= b; k += 8) {
        u64 c[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) c[j] = __ldg(P.mv + __ldg(P.ep + k + j));
#pragma unroll
        for (int j = 0; j < 8; ++j) acc = vv_add(c[j], acc, fl);
    }
    for (; k < b; ++k) acc = vv_add(__ldg(P.mv + __ldg(P.ep + k)), acc, fl);
    P.part[s] = acc;
}

// Thread per segment: a rank's first segment merges the rank's later ranges into it in ascending order (Merge with
// the chunks finishing in index order) and writes the rank's entry.  Nothing but the size is written when the next
// map does not fit (the outputs at the last level: DGX_ERR_CAP).
__global__ void __launch_bounds__(256) vv_combine_kernel(const VvParams P) {
    const u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    const u64 sg = P.words[VV_W_SG], S = sg & 0xffffffffull, G = sg >> 32;
    if (s == 0) {
        *P.on = G;
        if (G > P.o_cap) atomicOr(P.err, 1);
    }
    if (G > P.o_cap || s >= S) return;
    const u64 h = P.head[P.sstart[s]];
    if (!(h >> 32)) return;
    u64 acc = P.part[s];
    for (u64 q = s + 1; q < S && !(P.head[P.sstart[q]] >> 32); ++q) acc = vv_add(acc, P.part[q], P.is_float);
    const u64 g = P.hidx[P.sstart[s]] >> 32;
    P.ok[g] = P.dest[P.ek[P.sstart[s]] >> VV_RANGE_BITS];
    P.ov[g] = acc;
}

// ---- level aggregation ------------------------------------------------------------------------------------------------

constexpr int VA_W_R = 0, VA_W_G = 1, VA_WORDS = 2;

struct VaParams {
    const u64* mk;
    const u64* mv;
    u64 n;
    const u64* src;
    u64 nrows;
    const u64* v_off;  // nrows + 1
    const u64* v;
    u64 v_cap;
    int fn, is_float;
    u64* words;        // VA_WORDS, zeroed
    int* bad;          // zeroed
    int* err;
    u64* rval;         // nrows
    u64* rflag;        // nrows
    u64* rpos;         // nrows + 1
    u64* out_key;
    u64* out_val;
    u64 out_cap;
    u64* out_len;
};

// Grid over max(nrows + 1, n) threads.
__global__ void __launch_bounds__(256) la_check_kernel(const VaParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    if (t == 0) {
        bad = P.v_off[0] != 0 || P.v_off[P.nrows] > P.v_cap;
        P.words[VA_W_R] = P.nrows;
    }
    if (t < P.nrows) {
        if (t > 0 && P.src[t - 1] >= P.src[t]) bad = true;
        if (P.v_off[t] > P.v_off[t + 1]) bad = true;
    }
    if (t > 0 && t < P.n && P.mk[t - 1] >= P.mk[t]) bad = true;
    if (bad) vv_refuse(P.bad, P.err);
}

__device__ __forceinline__ double va_d(u64 x) { return __longlong_as_double((long long)x); }
__device__ __forceinline__ u64 va_u(double x) { return (u64)__double_as_longlong(x); }

// aggregator.Apply for min / max / sum / avg on one type: types.Less is `<` on int64 and on float64.
__device__ __forceinline__ u64 va_apply(u64 acc, u64 x, int fn, int fl) {
    if (fn == kVaMin || fn == kVaMax) {
        const bool lt = fl ? va_d(acc) < va_d(x) : (long long)acc < (long long)x;
        return (fn == kVaMin) == lt ? acc : x;
    }
    return fl ? va_u(__dadd_rn(va_d(acc), va_d(x))) : acc + x;
}

// Warp per row (grid over nrows warps).  A refused call folds nothing.
__global__ void __launch_bounds__(256) la_fold_kernel(const VaParams P) {
    const u64 r = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= P.nrows) return;
    if (*P.bad) {
        if (lane == 0) P.rflag[r] = 0;
        return;
    }
    const u64 a = P.v_off[r], b = P.v_off[r + 1];
    const int fn = P.fn, fl = P.is_float;
    u64 acc = 0, cnt = 0;
    for (u64 base = a; base < b; base += 32) {
        const u64 k = base + lane;
        u64 x = 0;
        bool present = false;
        if (k < b) {
            const u64 u = P.v[k];
            const u64 j = lower_bound_g(P.mk, P.n, u);
            present = j < P.n && P.mk[j] == u;
            if (present) x = __ldg(P.mv + j);
        }
        for (u32 m = __ballot_sync(0xffffffffu, present); m; m &= m - 1) {
            const u64 xi = __shfl_sync(0xffffffffu, x, __ffs(m) - 1);
            acc = cnt ? va_apply(acc, xi, fn, fl) : xi;
            ++cnt;
        }
    }
    if (lane) return;
    P.rflag[r] = cnt != 0;
    if (!cnt) return;
    if (fn == kVaAvg) {
        const double s = fl ? va_d(acc) : __ll2double_rn((long long)acc);
        acc = va_u(vv_clamp(__ddiv_rn(s, __ull2double_rn(cnt))));
    } else {
        acc = vv_first(acc, fl);
    }
    P.rval[r] = acc;
}

// Grid over nrows threads (at least one).  Nothing but the size is written when the result does not fit.
__global__ void __launch_bounds__(256) la_write_kernel(const VaParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    const u64 G = P.words[VA_W_G];
    if (t == 0) {
        *P.out_len = G;
        if (G > P.out_cap) atomicOr(P.err, 1);
    }
    if (G > P.out_cap || t >= P.nrows || !P.rflag[t]) return;
    P.out_key[P.rpos[t]] = P.src[t];
    P.out_val[P.rpos[t]] = P.rval[t];
}

}  // namespace dgx
