// encode_kernel.cuh -- codec.Encode (Encoder.Add / packBlock / Done, codec/codec.go:57-136, 393-399) on the device.
//
// Block rule (:116-120): a new block starts where the upper 32 bits of the uid change, or when the current block
// holds BlockSize uids (BlockSize 0 behaves like 1: the length test follows the append).  Payload (:76-96): Base =
// first uid, then uint32 deltas in groups of four (last group zero-padded; a 1-uid block still emits one all-zero
// group), each group a go-groupvarint Encode4: tag byte (value j's length-1 in bits 2j+1:2j) + the four values,
// little-endian, 1..4 bytes each.
//
// Data-parallel formulation: the uids fall into SEGMENTS of equal upper 32 bits; inside a segment blocks start
// every BlockSize uids.  So
//   enc_segments_kernel   compacts the indices where the upper word changes (single-pass look-back)
//   enc_segscan_kernel    blocks per segment -> first block of every segment (one CTA; segments are few:
//                         a sorted list crosses a multiple of 2^32 rarely)
//   enc_sizes_kernel      warp per block: Base, NumUids, byte length of the block's groups
//   scan_u64_kernel       exclusive scan of the byte lengths -> delta_off (single-pass look-back)
//   enc_write_kernel      warp per block: lane g encodes group g at its offset inside the block
// Bound: HBM (8 B/uid in, ~1.3-2.6 B/uid out).
// Limit: a list of 2^32 uids or more, or a block of 2^32 - 2 uids or more, wraps the u32 num, ngroups and per-round
// totals; that is 32 GB of uids in one call, far past any posting list, and is not supported.
#pragma once

#include "common.cuh"

namespace dgx {

constexpr int EN_NT = 256, EN_VT = 8, EN_TILE = EN_NT * EN_VT;

struct EncParams {
    const u64* u;        // n ascending uids
    u64 n;               // number of uids, or an upper bound when n_dyn != nullptr
    const u64* n_dyn;    // optional device word holding the actual count (result of a previous kernel)
    u32 bsz;             // max(BlockSize, 1)
    u64* seg_start;      // seg_cap entries: index of the first uid of every segment, then n
    u64 seg_cap;
    u64* seg_blk;        // nseg + 1: first block of every segment
    u64* counts;         // [0] = nseg, [1] = nblocks, [2] = delta bytes
    u64* status;         // look-back words (segments pass, then scan pass), zeroed
    u32* ticket;         // two tickets, zeroed
    u64 nblocks_cap;     // capacity of base / num / blk_start / blk_bytes / delta_off
    u64* base;           // out: nblocks
    u32* num;            // out: nblocks
    u64* blk_start;      // scratch: first uid index of every block
    u64* blk_bytes;      // scratch: byte length of every block
    u64* delta_off;      // out: nblocks + 1
    unsigned char* deltas;  // out
    u64 delta_cap;
    int* err;            // 2 = nblocks_cap too small, 3 = delta_cap too small
};

__device__ __forceinline__ u64 enc_n(const EncParams& P);

// Indices i with i == 0 or (u[i] >> 32) != (u[i-1] >> 32), compacted in order.
__global__ void __launch_bounds__(EN_NT) enc_segments_kernel(const EncParams P) {
    __shared__ u32 warp_sums[EN_NT / 32 + 1];
    __shared__ u64 s_base;
    __shared__ u32 s_tile;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(P.ticket, 1u);
    __syncthreads();
    const u32 tile = s_tile;
    const u64 n = enc_n(P);
    if ((u64)tile * EN_TILE >= n && tile != 0) return;  // grid sized for the bound: nothing here
    const u64 e0 = (u64)tile * EN_TILE + (u64)tid * EN_VT;
    u32 flags = 0, cnt = 0;
    u32 prev_hi = 0;
    bool have_prev = false;
    if (e0 > 0 && e0 <= n) { prev_hi = (u32)(P.u[e0 - 1] >> 32); have_prev = true; }
#pragma unroll
    for (int i = 0; i < EN_VT; ++i)
        if (e0 + i < n) {
            const u32 hi = (u32)(P.u[e0 + i] >> 32);
            if (!have_prev || hi != prev_hi) { flags |= 1u << i; ++cnt; }
            prev_hi = hi;
            have_prev = true;
        }
    u32 total;
    const u32 ex = block_exclusive_scan<EN_NT>(cnt, warp_sums, &total);
    if (wid == 0) {
        const u64 b = lookback_exclusive(P.status, tile, (u64)total, lane);
        if (lane == 0) {
            s_base = b;
            if ((u64)(tile + 1) * EN_TILE >= n) {  // last tile: close the list with n
                P.counts[0] = b + total;
                if (b + total < P.seg_cap) P.seg_start[b + total] = n;
            }
        }
    }
    __syncthreads();
    u64 w = s_base + ex;
#pragma unroll
    for (int i = 0; i < EN_VT; ++i)
        if ((flags >> i) & 1u) { if (w < P.seg_cap) P.seg_start[w] = e0 + i; ++w; }
}

// One CTA: blocks per segment, exclusive scan.
__global__ void __launch_bounds__(1024) enc_segscan_kernel(const EncParams P) {
    __shared__ u32 s_warp[1024 / 32 + 1];
    __shared__ u64 s_carry;
    const u64 nseg = P.counts[0];
    if (nseg + 1 > P.seg_cap) {  // more segments than the arrays hold: report a block count that suffices
        if (threadIdx.x == 0) {
            // a segment of len uids takes ceil(len / bsz) <= floor(len / bsz) + 1 blocks, and every block holds a uid:
            // with this capacity the next call's segment array holds nseg + 1 entries and the exact count fits.  It
            // exceeds nblocks_cap, as nseg does (min(n, nblocks_cap) + 2 < nseg + 1 <= n + 1)
            const u64 n = enc_n(P), nb = n / P.bsz + nseg;
            P.counts[1] = nb < n ? nb : n;
            atomicExch(P.err, 2);
        }
        return;
    }
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (u64 start = 0; start < nseg; start += 1024) {
        const u64 s = start + threadIdx.x;
        u64 nblk = 0;
        if (s < nseg) nblk = (P.seg_start[s + 1] - P.seg_start[s] + P.bsz - 1) / P.bsz;
        // segments hold < 2^32 blocks each in any list that fits a GPU; the scan runs on 32-bit partials per round
        u32 total;
        const u32 off = block_exclusive_scan<1024>((u32)nblk, s_warp, &total);
        const u64 carry = s_carry;
        if (s < nseg) P.seg_blk[s] = carry + off;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + total;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        P.seg_blk[nseg] = s_carry;
        P.counts[1] = s_carry;
        if (s_carry > P.nblocks_cap) atomicExch(P.err, 2);
    }
}

__device__ __forceinline__ u64 enc_n(const EncParams& P) {
    u64 n = P.n;
    if (P.n_dyn) { const u64 d = ld_relaxed(P.n_dyn); if (d < n) n = d; }
    return n;
}

__device__ __forceinline__ u32 gv_len(u32 v) { return v < (1u << 8) ? 1u : (v < (1u << 16) ? 2u : (v < (1u << 24) ? 3u : 4u)); }

// The four deltas of group g of the block starting at uid index `start` with `num` uids (zero-padded).
__device__ __forceinline__ void enc_group(const u64* __restrict__ u, u64 start, u32 num, u32 g, u32 (&d)[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const u32 pos = 1u + 4u * g + (u32)j;  // uid position inside the block
        d[j] = pos < num ? (u32)(u[start + pos] - u[start + pos - 1]) : 0u;
    }
}

// Warp per block: Base, NumUids, bytes.
__global__ void __launch_bounds__(256) enc_sizes_kernel(const EncParams P) {
    const u64 nblocks = P.counts[1];
    if (nblocks > P.nblocks_cap) return;
    const int lane = threadIdx.x & 31;
    const u64 b = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= nblocks) return;
    const u64 nseg = P.counts[0];
    u64 lo = 0, hi = nseg;  // segment of block b: last s with seg_blk[s] <= b
    while (hi - lo > 1) {
        const u64 mid = (lo + hi) >> 1;
        if (P.seg_blk[mid] <= b) lo = mid; else hi = mid;
    }
    const u64 start = P.seg_start[lo] + (b - P.seg_blk[lo]) * (u64)P.bsz;
    const u64 seg_end = P.seg_start[lo + 1];
    const u32 num = (u32)((seg_end - start) < (u64)P.bsz ? (seg_end - start) : (u64)P.bsz);
    const u32 ngroups = num > 1 ? (num + 2) / 4 : 1;  // max(1, ceil((num-1)/4))
    u32 bytes = 0;
    for (u32 g = lane; g < ngroups; g += 32) {
        u32 d[4];
        enc_group(P.u, start, num, g, d);
        bytes += 1u + gv_len(d[0]) + gv_len(d[1]) + gv_len(d[2]) + gv_len(d[3]);
    }
#pragma unroll
    for (int dl = 16; dl > 0; dl >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, dl);
    if (lane == 0) {
        P.base[b] = P.u[start];
        P.num[b] = num;
        P.blk_start[b] = start;
        P.blk_bytes[b] = bytes;
    }
}

// Exclusive scan of in[0..n) into out[0..n], out[n] = total (single pass, look-back); n read from a device word.
__global__ void __launch_bounds__(EN_NT) scan_u64_kernel(const u64* __restrict__ in, u64* __restrict__ out,
                                                         const u64* __restrict__ n_word, u64 n_cap, u64* status,
                                                         u32* ticket, u64* total_out) {
    __shared__ u64 s_part[EN_NT / 32];
    __shared__ u64 s_base;
    __shared__ u32 s_tile;
    const u64 n = *n_word;
    if (n > n_cap) return;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    const u32 tile = s_tile;
    const u64 t0 = (u64)tile * EN_TILE;
    if (t0 >= n && !(n == 0 && tile == 0)) return;
    const u64 e0 = t0 + (u64)tid * EN_VT;
    u64 v[EN_VT];
    u64 sum = 0;
#pragma unroll
    for (int i = 0; i < EN_VT; ++i) { v[i] = e0 + i < n ? in[e0 + i] : 0; sum += v[i]; }
    u64 inc = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u64 t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += t;
    }
    if (lane == 31) s_part[wid] = inc;
    __syncthreads();
    u64 wbase = 0, total = 0;
#pragma unroll
    for (int w = 0; w < EN_NT / 32; ++w) { if (w < wid) wbase += s_part[w]; total += s_part[w]; }
    if (wid == 0) {
        const u64 b = lookback_exclusive(status, tile, total, lane);
        if (lane == 0) {
            s_base = b;
            if (t0 + EN_TILE >= n) { out[n] = b + total; if (total_out) *total_out = b + total; }
        }
    }
    __syncthreads();
    u64 run = s_base + wbase + inc - sum;
#pragma unroll
    for (int i = 0; i < EN_VT; ++i)
        if (e0 + i < n) { out[e0 + i] = run; run += v[i]; }
}

// Warp per block: lane g writes group g.
__global__ void __launch_bounds__(256) enc_write_kernel(const EncParams P) {
    const u64 nblocks = P.counts[1];
    if (nblocks > P.nblocks_cap) return;
    if (P.counts[2] > P.delta_cap) { if (threadIdx.x == 0 && blockIdx.x == 0) atomicExch(P.err, 3); return; }
    const int lane = threadIdx.x & 31;
    const u64 b = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= nblocks) return;
    const u64 start = P.blk_start[b];
    const u32 num = P.num[b];
    const u32 ngroups = num > 1 ? (num + 2) / 4 : 1;
    unsigned char* dst = P.deltas + P.delta_off[b];
    u32 carry = 0;
    for (u32 g0 = 0; g0 < ngroups; g0 += 32) {
        const u32 g = g0 + lane;
        u32 d[4] = {0, 0, 0, 0};
        u32 l[4] = {0, 0, 0, 0};
        u32 bytes = 0;
        if (g < ngroups) {
            enc_group(P.u, start, num, g, d);
#pragma unroll
            for (int j = 0; j < 4; ++j) l[j] = gv_len(d[j]);
            bytes = 1u + l[0] + l[1] + l[2] + l[3];
        }
        u32 inc = bytes;
#pragma unroll
        for (int dl = 1; dl < 32; dl <<= 1) {
            const u32 t = __shfl_up_sync(0xffffffffu, inc, dl);
            if (lane >= dl) inc += t;
        }
        if (g < ngroups) {
            unsigned char* p = dst + carry + inc - bytes;
            *p++ = (unsigned char)((l[0] - 1u) | ((l[1] - 1u) << 2) | ((l[2] - 1u) << 4) | ((l[3] - 1u) << 6));
#pragma unroll
            for (int j = 0; j < 4; ++j)
                for (u32 t = 0; t < l[j]; ++t) *p++ = (unsigned char)(d[j] >> (8u * t));
        }
        carry += __shfl_sync(0xffffffffu, inc, 31);
    }
}

}  // namespace dgx
