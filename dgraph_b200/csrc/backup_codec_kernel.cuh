// backup_codec_kernel.cuh -- the uid path of backup and restore on the device, batched over keys:
//   codec.DecodeToBuffer (codec/codec.go:456-467)   pack -> BackupPostingList.uid_bytes
//   codec.EncodeFromBuffer (codec/codec.go:402-414) uid_bytes -> pack
// uid_bytes is a stream of unsigned LEB128 varints (encoding/binary PutUvarint / Uvarint): uid u is written as
// PutUvarint(u - last), the subtraction on u64 (it wraps), last starting at 0.
//
// Packs -> bytes (tb_*), four launches whatever the row count, uid count and pack sizes are:
//   tb_blocks_kernel   thread per block: walks it with gv_walk_block (decode_kernel.cuh), records its last uid and the
//                      varint bytes of its internal deltas (= its group-varint u32 values); a block with NumUids 0 marks
//                      its row's stop (the reference's `for len(uids) > 0` loop ends there)
//   tb_sizes_kernel    adds the varint of the boundary delta base[b] - last[b-1] (base - 0 at a row's first block);
//                      blocks at or after the row's stop take no bytes
//   scan_u64_kernel    block byte counts -> byte offsets (single-pass look-back)
//   tb_write_kernel    row offsets, and thread per block: every varint at its final byte
//
// Bytes -> packs (bf_*), nine launches whatever the row count, byte count and block size are:
//   bf_values_kernel   byte tiles: flag the terminators (< 0x80), validate every value's length, assemble the values
//                      and compact them; two look-backs per tile: value count, and the wrapping u64 sum of all values
//   bf_segments_kernel uid = (prefix sum through the value) - (prefix sum before its row's first value) on u64, which is
//                      the running sum restarted at every row; a segment starts at a row's first value or where the upper
//                      32 bits change; segment starts compacted (look-back)
//   bf_segcount_kernel blocks per segment: ceil(len / BlockSize)
//   scan_u64_kernel    first block of every segment (multi-CTA look-back: every row starts a segment)
//   bf_sizes_kernel    warp per block: byte length of its groups (enc_block_bytes, encode_kernel.cuh), its row
//   scan_u64_kernel    block byte offsets
//   bf_rows_kernel     thread per row: first block, block count, delta bytes, image bytes; a row whose last byte has the
//                      high bit set is a truncated value
//   scan_u64_kernel    image offsets
//   bf_write_kernel    warp per block: Base, NumUids, delta_off and the groups (enc_block_write) into the row's flat
//                      image; a malformed stream zeroes the offset and size arrays instead and writes nothing
// Uids are recomputed from the prefix sums wherever they are read, never stored.
#pragma once

#include "common.cuh"
#include "decode_kernel.cuh"
#include "encode_kernel.cuh"

namespace dgx {

constexpr int kLaneErrVarint = 8;  // lane error flag bit: a uid_bytes stream is not a sequence of valid uvarints

// Bytes of PutUvarint(x): max(1, ceil(bits / 7)).
__device__ __forceinline__ u32 uvarint_len(u64 x) { return x ? (u32)(70 - __clzll((long long)x)) / 7u : 1u; }
__device__ __forceinline__ unsigned char* uvarint_put(unsigned char* p, u64 x) {
    while (x >= 0x80) { *p++ = (unsigned char)(x | 0x80); x >>= 7; }
    *p++ = (unsigned char)x;
    return p;
}

// ---- decoupled look-back over full u64 values (wrapping sums) -----------------------------------------------------
// The value does not leave room for the flag in its word, so the two travel apart: val[2t] the tile's aggregate,
// val[2t+1] its inclusive prefix, flag[t] 1 / 2 once the respective value is published (release / acquire).
__device__ __forceinline__ u32 ld_acquire_u32(const u32* p) {
    u32 v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(u32* p, u32 v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ u64 lookback_wide(u32* flag, u64* val, u32 tile, u64 aggregate, int lane) {
    if (tile == 0) {
        if (lane == 0) { st_relaxed(val + 1, aggregate); st_release_u32(flag, 2); }
        return 0;
    }
    if (lane == 0) { st_relaxed(val + 2 * (u64)tile, aggregate); st_release_u32(flag + tile, 1); }
    u64 exclusive = 0;
    long long idx = (long long)tile - 1;
    while (true) {
        const long long my = idx - lane;
        u32 f = 2;
        u64 v = 0;
        if (my >= 0) {
            while ((f = ld_acquire_u32(flag + my)) == 0) {}
            v = ld_relaxed(val + 2 * (u64)my + (f == 2 ? 1 : 0));
        }
        const unsigned pm = __ballot_sync(0xffffffffu, f == 2);
        if (pm && lane > __ffs(pm) - 1) v = 0;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
        exclusive += v;
        if (pm) break;
        idx -= 32;
    }
    if (lane == 0) { st_relaxed(val + 2 * (u64)tile + 1, exclusive + aggregate); st_release_u32(flag + tile, 2); }
    return exclusive;
}

// Exclusive block scan of one u64 per thread (EN_NT threads); *total gets the block's sum.  Two barriers.
__device__ __forceinline__ u64 block_exclusive_scan_u64(u64 v, u64* warp_sums, u64* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    u64 inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u64 t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += t;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    u64 wbase = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < EN_NT / 32; ++w) { if (w < wid) wbase += warp_sums[w]; tot += warp_sums[w]; }
    __syncthreads();
    *total = tot;
    return wbase + inc - v;
}

// ---- packs -> bytes ------------------------------------------------------------------------------------------------
struct TbJob {
    DPack pk;
    u64 blk0;  // the call's index of the pack's first block
    u64 row;
};
struct TbParams {
    const TbJob* jobs;
    u32 njobs;
    u64 nblk;              // blocks of all packs
    const u64* row_blk;    // nrows + 1: the call's index of every row's first block, nblk at the end
    u64 nrows;
    u64* stop;             // nrows: first block of the row with NumUids 0 (all ones: none)
    u64* last;             // nblk: last uid of every block
    u64* bytes;            // nblk: varint bytes of every block
    u64* boff;             // nblk + 1: their exclusive scan
    unsigned char* out;    // nullptr: offsets only
    u64 out_cap;
    u64* out_off;          // nrows + 1
    int* err;              // lane error flag (nullptr: the host checks the capacity)
};

__device__ __forceinline__ void tb_block(const TbParams& P, u64 g, u32& j, u64& b) {
    j = job_of<TbJob, &TbJob::blk0>(P.jobs, P.njobs, g);
    b = g - P.jobs[j].blk0;
}

__global__ void __launch_bounds__(256) tb_blocks_kernel(const TbParams P) {
    const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= P.nblk) return;
    u32 j;
    u64 b;
    tb_block(P, g, j, b);
    const DPack& pk = P.jobs[j].pk;
    const u32 num = pk.num[b];
    const u64 base = pk.base[b];
    if (num == 0) atomicMin(P.stop + P.jobs[j].row, b);
    u64 prev = base;
    u64 ib = 0;
    gv_walk_block(pk.deltas + pk.delta_off[b], base, num, [&](u32 i, u64 uid) {
        if (i) ib += uvarint_len(uid - prev);
        prev = uid;
        return true;
    });
    P.last[g] = prev;
    P.bytes[g] = ib;
}

__global__ void __launch_bounds__(256) tb_sizes_kernel(const TbParams P) {
    const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= P.nblk) return;
    u32 j;
    u64 b;
    tb_block(P, g, j, b);
    if (b >= P.stop[P.jobs[j].row]) { P.bytes[g] = 0; return; }
    const u64 prev = b ? P.last[g - 1] : 0;
    P.bytes[g] += uvarint_len(P.jobs[j].pk.base[b] - prev);
}

__global__ void __launch_bounds__(256) tb_write_kernel(const TbParams P) {
    const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (g <= P.nrows) P.out_off[g] = P.boff[P.row_blk[g]];
    if (!P.out || g >= P.nblk) return;
    if (P.boff[P.nblk] > P.out_cap) {
        if (g == 0 && P.err) atomicOr(P.err, 1);
        return;
    }
    u32 j;
    u64 b;
    tb_block(P, g, j, b);
    if (b >= P.stop[P.jobs[j].row]) return;
    const DPack& pk = P.jobs[j].pk;
    const u64 base = pk.base[b];
    unsigned char* p = uvarint_put(P.out + P.boff[g], base - (b ? P.last[g - 1] : 0));
    u64 prev = base;
    gv_walk_block(pk.deltas + pk.delta_off[b], base, pk.num[b], [&](u32 i, u64 uid) {
        if (i) p = uvarint_put(p, uid - prev);
        prev = uid;
        return true;
    });
}

// ---- bytes -> packs ------------------------------------------------------------------------------------------------
struct BfParams {
    const unsigned char* buf;  // every row's bytes, back to back
    u64 n;                     // bytes
    const u64* row_off;        // nrows + 1 byte offsets
    u64 nrows;
    u32 bsz;                   // max(BlockSize, 1)
    u64* counts;               // [0] values, [1] segments, [2] blocks, [3] delta bytes, [4] image bytes, [5] nrows
    u64* status;               // look-back words, zeroed: values, segments, segment scan, byte scan, image scan
    u32* ticket;               // five tickets, zeroed
    u32* sum_flag;             // wide look-back of the value sums, zeroed
    u64* sum_val;
    int* bad;                  // a malformed stream, zeroed
    u64* pre;                  // values: inclusive prefix (wrapping) of all values of the call
    u32* vrow;                 // values: row
    u64* rowbase;              // nrows: prefix before the row's first value
    u32* seg_start;            // segments + 1: first value of every segment, then the value count
    u64* seg_cnt;              // segments: blocks
    u64* seg_blk;              // segments + 1: first block
    u64* blk_bytes;            // blocks: group bytes
    u64* blk_doff;             // blocks + 1: the call's offset of every block's deltas
    u32* brow;                 // blocks: row
    u64* row_blk;              // nrows + 1: first block of every row
    u64* img_bytes;            // nrows
    unsigned char* img;        // nullptr: sizes only
    u64 img_cap;
    u64* img_off;              // nrows + 1
    u64* nblocks;              // nrows
    u64* delta_bytes;          // nrows
    int* err;                  // lane error flag (nullptr: the host reads `bad` and checks the capacity)
};

// uid i = the running sum of its row's values through value i
struct BfUid {
    const u64* pre;
    const u32* vrow;
    const u64* rowbase;
    __device__ __forceinline__ u64 operator()(u64 i) const { return pre[i] - rowbase[vrow[i]]; }
};

// Last index r of the ascending a[0..n) with a[r] <= x (a[0] <= x).
template <class T>
__device__ __forceinline__ u64 last_le(const T* a, u64 n, u64 x) {
    u64 lo = 0, hi = n;
    while (hi - lo > 1) {
        const u64 mid = (lo + hi) >> 1;
        if ((u64)a[mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
}
// First index of the ascending a[0..n) with a[i] >= x (n if none).
__device__ __forceinline__ u64 first_ge_u32(const u32* a, u64 n, u64 x) {
    u64 lo = 0, hi = n;
    while (lo < hi) {
        const u64 mid = (lo + hi) >> 1;
        if ((u64)a[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// binary.Uvarint rules: a byte < 0x80 ends a value; at most 10 bytes, the 10th <= 1.  The continuation bytes before a
// terminator never reach into the previous row unless that row ends in one, which bf_rows_kernel reports.
__global__ void __launch_bounds__(EN_NT) bf_values_kernel(const BfParams P) {
    __shared__ u32 s_wc[EN_NT / 32 + 1];
    __shared__ u64 s_ws[EN_NT / 32];
    __shared__ u64 s_cbase, s_sbase;
    __shared__ u32 s_tile;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(P.ticket, 1u);
    __syncthreads();
    const u32 tile = s_tile;
    const u64 e0 = (u64)tile * EN_TILE + (u64)tid * EN_VT;
    u64 x[EN_VT];
    u64 start[EN_VT];
    u32 flags = 0, cnt = 0;
    u64 sum = 0;
    bool bad = false;
#pragma unroll
    for (int i = 0; i < EN_VT; ++i) {
        x[i] = 0;
        start[i] = 0;
        const u64 k = e0 + i;
        if (k < P.n && P.buf[k] < 0x80) {
            u32 c = 0;
            while (c < 10 && k > c && P.buf[k - 1 - c] >= 0x80) ++c;
            if (c >= 10 || (c == 9 && P.buf[k] > 1)) bad = true;
            const u64 s = k - c;
            u64 v = 0;
            for (u32 t = 0; t <= c && t < 10; ++t) v |= (u64)(P.buf[s + t] & 0x7f) << (7 * t);
            x[i] = v;
            start[i] = s;
            flags |= 1u << i;
            ++cnt;
            sum += v;
        }
    }
    if (bad) atomicExch(P.bad, 1);
    u32 ctotal;
    const u32 cex = block_exclusive_scan<EN_NT>(cnt, s_wc, &ctotal);
    u64 stotal;
    const u64 sex = block_exclusive_scan_u64(sum, s_ws, &stotal);
    if (wid == 0) {
        const u64 cb = lookback_exclusive(P.status, tile, (u64)ctotal, lane);
        const u64 sb = lookback_wide(P.sum_flag, P.sum_val, tile, stotal, lane);
        if (lane == 0) {
            s_cbase = cb;
            s_sbase = sb;
            if ((u64)(tile + 1) * EN_TILE >= P.n) P.counts[0] = cb + ctotal;
        }
    }
    __syncthreads();
    u64 w = s_cbase + cex, run = s_sbase + sex;
#pragma unroll
    for (int i = 0; i < EN_VT; ++i)
        if ((flags >> i) & 1u) {
            run += x[i];
            const u64 row = last_le(P.row_off, P.nrows + 1, start[i]);
            P.pre[w] = run;
            P.vrow[w] = (u32)row;
            if (P.row_off[row] == start[i]) P.rowbase[row] = run - x[i];
            ++w;
        }
}

__global__ void __launch_bounds__(EN_NT) bf_segments_kernel(const BfParams P) {
    __shared__ u32 warp_sums[EN_NT / 32 + 1];
    __shared__ u64 s_base;
    __shared__ u32 s_tile;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(P.ticket + 1, 1u);
    __syncthreads();
    const u32 tile = s_tile;
    const u64 m = P.counts[0];
    if ((u64)tile * EN_TILE >= m && tile != 0) return;  // grid sized for the byte count: nothing here
    const BfUid uid{P.pre, P.vrow, P.rowbase};
    const u64 e0 = (u64)tile * EN_TILE + (u64)tid * EN_VT;
    u32 flags = 0, cnt = 0;
    u32 prow = 0;
    u64 prev = 0;
    if (e0 > 0 && e0 <= m) { prow = P.vrow[e0 - 1]; prev = uid(e0 - 1); }
#pragma unroll
    for (int i = 0; i < EN_VT; ++i)
        if (e0 + i < m) {
            const u64 j = e0 + i;
            const u32 row = P.vrow[j];
            const u64 u = uid(j);
            if (j == 0 || row != prow || (u >> 32) != (prev >> 32)) { flags |= 1u << i; ++cnt; }
            prow = row;
            prev = u;
        }
    u32 total;
    const u32 ex = block_exclusive_scan<EN_NT>(cnt, warp_sums, &total);
    if (wid == 0) {
        const u64 b = lookback_exclusive(P.status + 1 * (P.n / EN_TILE + 1), tile, (u64)total, lane);
        if (lane == 0) {
            s_base = b;
            if ((u64)(tile + 1) * EN_TILE >= m) {
                P.counts[1] = b + total;
                P.seg_start[b + total] = (u32)m;
            }
        }
    }
    __syncthreads();
    u64 w = s_base + ex;
#pragma unroll
    for (int i = 0; i < EN_VT; ++i)
        if ((flags >> i) & 1u) P.seg_start[w++] = (u32)(e0 + i);
}

__global__ void __launch_bounds__(256) bf_segcount_kernel(const BfParams P) {
    const u64 nseg = P.counts[1];
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < nseg; s += (u64)gridDim.x * blockDim.x)
        P.seg_cnt[s] = ((u64)P.seg_start[s + 1] - P.seg_start[s] + P.bsz - 1) / P.bsz;
}

// Block b: its first value and NumUids.
__device__ __forceinline__ void bf_block(const BfParams& P, u64 b, u64& start, u32& num) {
    const u64 s = last_le(P.seg_blk, P.counts[1], b);
    start = (u64)P.seg_start[s] + (b - P.seg_blk[s]) * (u64)P.bsz;
    const u64 left = (u64)P.seg_start[s + 1] - start;
    num = (u32)(left < (u64)P.bsz ? left : (u64)P.bsz);
}

__global__ void __launch_bounds__(256) bf_sizes_kernel(const BfParams P) {
    const u64 nblk = P.counts[2];
    const int lane = threadIdx.x & 31;
    const BfUid uid{P.pre, P.vrow, P.rowbase};
    const u64 nw = ((u64)gridDim.x * blockDim.x) >> 5;
    for (u64 b = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < nblk; b += nw) {
        u64 start;
        u32 num;
        bf_block(P, b, start, num);
        const u32 bytes = enc_block_bytes(uid, start, num, lane);
        if (lane == 0) {
            P.blk_bytes[b] = bytes;
            P.brow[b] = P.vrow[start];
        }
    }
}

__global__ void __launch_bounds__(256) bf_rows_kernel(const BfParams P) {
    const u64 nblk = P.counts[2];
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r <= P.nrows; r += (u64)gridDim.x * blockDim.x) {
        const u64 b0 = first_ge_u32(P.brow, nblk, r);
        P.row_blk[r] = b0;
        if (r == P.nrows) continue;
        const u64 b1 = first_ge_u32(P.brow, nblk, r + 1);
        const u64 nb = b1 - b0, db = P.blk_doff[b1] - P.blk_doff[b0];
        P.nblocks[r] = nb;
        P.delta_bytes[r] = db;
        P.img_bytes[r] = nb ? pack_image_meta_bytes(nb) + ((db + 15) & ~15ull) : 0;
        const u64 o0 = P.row_off[r], o1 = P.row_off[r + 1];
        if (o1 > o0 && P.buf[o1 - 1] >= 0x80) atomicExch(P.bad, 1);  // the row ends inside a value
    }
}

__global__ void __launch_bounds__(256) bf_write_kernel(const BfParams P) {
    const u64 gid = (u64)blockIdx.x * blockDim.x + threadIdx.x, gsz = (u64)gridDim.x * blockDim.x;
    if (*(volatile int*)P.bad) {
        for (u64 r = gid; r <= P.nrows; r += gsz) {
            P.img_off[r] = 0;
            if (r < P.nrows) { P.nblocks[r] = 0; P.delta_bytes[r] = 0; }
        }
        if (gid == 0 && P.err) atomicOr(P.err, kLaneErrVarint);
        return;
    }
    if (!P.img) return;
    if (P.img_off[P.nrows] > P.img_cap) {
        if (gid == 0 && P.err) atomicOr(P.err, 1);
        return;
    }
    const u64 nblk = P.counts[2];
    const int lane = threadIdx.x & 31;
    const BfUid uid{P.pre, P.vrow, P.rowbase};
    for (u64 b = gid >> 5; b < nblk; b += gsz >> 5) {
        const u32 r = P.brow[b];
        const u64 rb = P.row_blk[r], lb = b - rb, nb = P.nblocks[r], db = P.delta_bytes[r];
        unsigned char* im = P.img + P.img_off[r];
        const u64 meta = pack_image_meta_bytes(nb);
        u64 start;
        u32 num;
        bf_block(P, b, start, num);
        const u64 doff = P.blk_doff[b] - P.blk_doff[rb];
        if (lane == 0) {
            reinterpret_cast<u64*>(im)[lb] = uid(start);
            reinterpret_cast<u64*>(im + nb * 8)[lb] = doff;
            reinterpret_cast<u32*>(im + nb * 16 + 8)[lb] = num;
            if (lb == nb - 1) {
                reinterpret_cast<u64*>(im + nb * 8)[nb] = db;
                for (u64 z = nb * 20 + 8; z < meta; ++z) im[z] = 0;
                for (u64 z = meta + db; z < meta + ((db + 15) & ~15ull); ++z) im[z] = 0;
            }
        }
        enc_block_write(uid, start, num, im + meta + doff, lane);
    }
}

}  // namespace dgx
