// common.cuh -- shared device helpers for the dgx kernels (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace dgx {

typedef unsigned long long u64;
typedef unsigned int u32;

constexpr u64 kU64Max = 0xFFFFFFFFFFFFFFFFull;

// ---- memory access -------------------------------------------------------

// Streaming read of list data: read-only path, do not allocate in L1 (each
// element of a streamed slice is touched once per tile).
__device__ __forceinline__ u64 ld_stream(const u64* p) {
    u64 v;
    asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
}
// Probe read (binary searches): cached, neighbouring probes share sectors.
__device__ __forceinline__ u64 ld_probe(const u64* p) { return __ldg(p); }

__device__ __forceinline__ void st_stream(u64* p, u64 v) {
    asm volatile("st.global.L1::no_allocate.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_stream2(u64* p, u64 a, u64 b) {  // 16-byte aligned
    asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}

// Tile status words for the decoupled look-back are single 64-bit words, read
// and written with relaxed gpu-scope accesses (the value travels in the word).
__device__ __forceinline__ u64 ld_relaxed(const u64* p) {
    u64 v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(u64* p, u64 v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Bytes of the metadata of a flat pack image (dgx_pack_image_view): [base u64 x nb | delta_off u64 x (nb+1) |
// num_uids u32 x nb | pad to 16]; the delta bytes follow, padded to 16.
__host__ __device__ __forceinline__ u64 pack_image_meta_bytes(u64 nb) { return (nb * 8 + (nb + 1) * 8 + nb * 4 + 15) & ~15ull; }

// ---- searches --------------------------------------------------------------

// First index in [0, n) with a[i] >= x (n if none).  Per-thread, global memory.
__device__ __forceinline__ u64 lower_bound_g(const u64* __restrict__ a, u64 n, u64 x) {
    u64 lo = 0, hi = n;
    while (lo < hi) {
        u64 mid = lo + ((hi - lo) >> 1);
        if (ld_probe(a + mid) < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// Warp-cooperative 32-ary search in global memory: log32(n) dependent rounds
// instead of log2(n).  All 32 lanes must call with identical (a, n, x).
// upper == false: first i with a[i] >= x;  upper == true: first i with a[i] > x.
__device__ __forceinline__ u64 warp_bound_g(const u64* __restrict__ a, u64 n, u64 x, bool upper, int lane) {
    u64 lo = 0, hi = n;  // answer in [lo, hi]
    while (hi - lo > 32) {
        u64 stride = (hi - lo) >> 5;
        u64 p = lo + (u64)(lane + 1) * stride - 1;
        u64 v = ld_probe(a + p);
        bool before = upper ? (v <= x) : (v < x);
        unsigned c = __popc(__ballot_sync(0xffffffffu, before));
        u64 nlo = lo + (u64)c * stride;
        if (c < 32) hi = lo + (u64)(c + 1) * stride - 1;
        lo = nlo;
    }
    u64 p = lo + lane;
    bool before = false;
    if (p < hi) {
        u64 v = ld_probe(a + p);
        before = upper ? (v <= x) : (v < x);
    }
    return lo + __popc(__ballot_sync(0xffffffffu, before));
}

// First index in [lo, n) of the shared-memory array with s[i] >= x.
__device__ __forceinline__ int lower_bound_s(const u64* s, int lo, int n, u64 x) {
    int hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (s[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// ---- block scan -------------------------------------------------------------

// Exclusive scan of one u32 per thread over a block of NT threads (NT multiple
// of 32, <= 1024).  Returns the exclusive prefix; *total gets the block sum.
// `warp_sums` is NT/32 + 1 words of shared memory.  Contains two barriers.
template <int NT>
__device__ __forceinline__ u32 block_exclusive_scan(u32 v, u32* warp_sums, u32* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    u32 inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        u32 t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += t;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        u32 w = (lane < NT / 32) ? warp_sums[lane] : 0;
        u32 winc = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            u32 t = __shfl_up_sync(0xffffffffu, winc, d);
            if (lane >= d) winc += t;
        }
        if (lane < NT / 32) warp_sums[lane] = winc - w;
        if (lane == NT / 32 - 1) warp_sums[NT / 32] = winc;
    }
    __syncthreads();
    *total = warp_sums[NT / 32];
    return warp_sums[wid] + inc - v;
}

// ---- decoupled look-back ------------------------------------------------------
// status word: bits 63..62 = flag (0 not ready, 1 tile aggregate, 2 inclusive
// prefix), bits 61..0 = value.  Tiles are numbered by an atomic ticket so every
// predecessor of a running tile has already started (no deadlock).

constexpr u64 kFlagAgg = 1ull << 62;
constexpr u64 kFlagPrefix = 2ull << 62;
constexpr u64 kValMask = (1ull << 62) - 1;

// Called by one full warp.  Publishes this tile's aggregate, walks back to the
// nearest inclusive prefix and publishes this tile's inclusive prefix.
// Returns the exclusive prefix of the tile (same value in every lane).
// kPublished: the tile's aggregate word has already been stored by someone else.
// kBackoff: sleep between polls (the caller is a helper warp that must not steal issue slots).
template <bool kPublished = false, unsigned kBackoff = 0>  // kBackoff: ns to sleep between polls (0 = spin)
__device__ __forceinline__ u64 lookback_exclusive(u64* status, u32 tile, u64 aggregate, int lane) {
    if (tile == 0) {
        if (lane == 0) st_relaxed(status, kFlagPrefix | aggregate);
        return 0;
    }
    if (!kPublished && lane == 0) st_relaxed(status + tile, kFlagAgg | aggregate);
    u64 exclusive = 0;
    long long idx = (long long)tile - 1;
    while (true) {
        long long my = idx - lane;
        u64 w;
        if (my >= 0) {
            while (((w = ld_relaxed(status + my)) >> 62) == 0) { if (kBackoff) __nanosleep(kBackoff); }
        } else {
            w = kFlagPrefix;  // virtual tile before the first: prefix 0
        }
        unsigned pm = __ballot_sync(0xffffffffu, (w >> 62) == 2);
        u64 val = w & kValMask;
        if (pm) {
            int first = __ffs(pm) - 1;  // nearest predecessor holding a prefix
            if (lane > first) val = 0;
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) val += __shfl_xor_sync(0xffffffffu, val, d);
        exclusive += val;
        if (pm) break;
        idx -= 32;
    }
    if (lane == 0) st_relaxed(status + tile, kFlagPrefix | (exclusive + aggregate));
    return exclusive;
}

}  // namespace dgx
