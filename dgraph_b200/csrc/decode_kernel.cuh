// decode_kernel.cuh -- group-varint UidPack decode for sm_90a, and the block-format helpers every pack reader uses.
//
// codec.Decode / Decoder.UnpackBlock (codec/codec.go:154-200, 444-452): block b
// yields Base, then running sums of its group-varint u32 deltas, truncated to
// NumUids.  A group is 1 tag byte + 4 little-endian values of 1..4 bytes
// (go-groupvarint; value j's length-1 in tag bits [2j+1:2j]).
//
// The block format is read in this file only; compressed_kernel.cuh calls the same helpers:
//   gv_walk_block      one thread's walk of one block from global memory (blocks of more than 256 uids, seeks)
//   pack_block_of      the block whose value range holds x
//   warp_mbar_init / warp_window_load / warp_tag_walk / expand_block
//                      the shared-memory path of one warp, below
//
// Mapping: a warp owns a run of consecutive blocks and streams it in batches of
// up to 32 blocks.  Per batch: (1) ONE TMA bulk copy (cp.async.bulk + mbarrier)
// brings the batch's contiguous delta bytes into the warp's shared-memory
// window; (2) lane i walks block i's tag bytes (the only serial dependence:
// group g+1 starts BytesUsed[tag_g] after group g) and records group offsets;
// (3) all lanes decode a block's groups in parallel -- unaligned 16-byte read,
// four extractions, warp prefix sum of deltas (64-bit, `last + uint64(delta)` as in
// codec.go:191-196) -- into a staging row that is written out as coalesced 16-byte stores.
#pragma once

#include "common.cuh"

namespace dgx {

constexpr int D_WARPS = 4;                  // warps per CTA
constexpr int D_NT = D_WARPS * 32;
constexpr int D_BPW = 64;                   // blocks owned by one warp
constexpr int D_WB = 4096;                  // payload window per warp (bytes)
constexpr int D_MAXG = 64;                  // groups per block at BlockSize 256
constexpr int D_TSTRIDE = 33;               // group-offset table row stride (u16)
constexpr int D_STAGE = 260;                // staging row (u64)

struct DPack {
    u64 nblocks;
    const u64* base;       // nblocks
    const u32* num;        // nblocks
    const u64* delta_off;  // nblocks + 1
    const unsigned char* deltas;  // 16-byte aligned, >= 32 bytes of slack after the end
    const u64* uid_off;    // nblocks + 1: exclusive prefix of num
    u32 max_num;           // largest NumUids of any block
    u32 sysmem;            // base / num / delta_off / deltas are mapped pinned HOST memory (zero-copy decode):
                           // the window is filled with plain vector loads over PCIe instead of a TMA bulk copy
};
struct DSeek {            // written by decode_seek_kernel
    u64 first_block;
    u64 skip;             // uids (in pack order) before the first emitted one
    u64 out_len;
};

__device__ __forceinline__ u32 gv_bytes_used(u32 t) {
    return 5u + (t & 3u) + ((t >> 2) & 3u) + ((t >> 4) & 3u) + (t >> 6);
}
// groups of a block of num uids: ceil((num-1)/4) carry data
__device__ __forceinline__ u32 gv_groups(u32 num) { return num > 1 ? (num + 2) / 4 : 0; }

// One block walked by one thread straight from global memory, from its Base `last`, NumUids `num` and delta bytes p:
// fn(i, uid) for Base (i = 0), then for every running sum, i < num.  The sum is 64-bit like the reference's
// `last + uint64(delta)` (codec.go:191-196): packs produced by the Encoder never carry more than 2^32 per block,
// hand-built ones may.  fn returns false to stop.  Returns num.  (The callers pass what they have already loaded:
// reloading it here costs decode_batch_kernel registers.)
template <class Fn>
__device__ __forceinline__ u32 gv_walk_block(const unsigned char* p, u64 last, u32 num, Fn&& fn) {
    if (num == 0 || !fn(0u, last)) return num;
    u32 produced = 1;
    while (produced < num) {
        const u32 tag = p[0];
        const unsigned char* d = p + 1;
        for (int j = 0; j < 4 && produced < num; ++j) {
            const u32 l = ((tag >> (2 * j)) & 3u) + 1u;
            u32 v = 0;
            for (u32 k = 0; k < l; ++k) v |= (u32)d[k] << (8 * k);
            d += l;
            last += v;
            if (!fn(produced++, last)) return num;
        }
        p += gv_bytes_used(tag);
    }
    return num;
}

// Last block b with base[b] <= x, or -1 when x is below the first block.
__device__ __forceinline__ long long pack_block_of(const DPack& pk, u64 x) {
    u64 lo = 0, hi = pk.nblocks;  // first b with base[b] > x
    while (lo < hi) {
        const u64 mid = lo + ((hi - lo) >> 1);
        if (ld_probe(pk.base + mid) <= x) lo = mid + 1; else hi = mid;
    }
    return (long long)lo - 1;
}

// Last job whose field F is <= x (F ascends over the jobs).
template <class Job, u64 Job::*F>
__device__ __forceinline__ u32 job_of(const Job* __restrict__ jobs, u32 njobs, u64 x) {
    u32 lo = 0, hi = njobs;
    while (hi - lo > 1) {
        const u32 mid = (lo + hi) >> 1;
        if (jobs[mid].*F <= x) lo = mid; else hi = mid;
    }
    return lo;
}

// Decoder.Seek(seek, SeekStart), codec/codec.go:279-337, restated for one thread.
__global__ void decode_seek_kernel(const DPack pk, u64 seek, DSeek* out, u64* out_len_word, u64 out_cap, int* err) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    u64 first = 0, trim = 0;
    const u64 nb = pk.nblocks;
    if (nb > 0 && seek != 0) {
        u64 idx = lower_bound_g(pk.base, nb, seek);  // first block with Base >= seek
        if (idx == 0) {
            first = 0;
        } else if (idx < nb && pk.base[idx] == seek) {
            first = idx;
        } else {
            const u64 b = idx - 1;  // unpack the previous block, count uids < seek
            u32 below = 0;
            const u32 num = gv_walk_block(pk.deltas + pk.delta_off[b], pk.base[b], pk.num[b], [&](u32, u64 uid) {
                below += uid < seek;
                return true;
            });
            if (below < num) { first = b; trim = below; }
            else { first = idx; }  // Next(): nothing >= seek in that block
        }
    }
    DSeek s;
    s.first_block = first;
    const u64 total = nb ? pk.uid_off[nb] : 0;
    s.skip = (first < nb ? pk.uid_off[first] : total) + trim;
    s.out_len = total - s.skip;
    *out = s;
    *out_len_word = s.out_len;
    if (s.out_len > out_cap) atomicExch(err, 1);
}

__device__ __forceinline__ u32 smem_u32(const void* p) { return (u32)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(u32 bar, u32 count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(u32 bar, u32 bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(u32 dst, const void* src, u32 bytes, u32 bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(u32 bar, u32 parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}

// Same wait for the pipeline's helper warps: the try_wait carries a suspend-time hint and a miss
// backs off with nanosleep, so a waiting warp does not compete with working warps for issue slots.
template <unsigned kSleepNs = 128>
__device__ __forceinline__ void mbar_wait_relaxed(u32 bar, u32 parity) {
    u32 done = 0;
    while (true) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n" : "=r"(done) : "r"(bar), "r"(parity), "r"(2000u) : "memory");
        if (done) break;
        __nanosleep(kSleepNs);
    }
}

struct __align__(128) DWarpSmem {
    unsigned char payload[D_WB + 64];
    unsigned short goff[D_MAXG * D_TSTRIDE + 2];
    u64 stage[D_STAGE];
    u64 mbar;
};

// ---- one warp's shared-memory path over a batch of blocks; every helper is called by the whole warp -----------

__device__ __forceinline__ void warp_mbar_init(DWarpSmem& S, int lane) {
    if (lane == 0) {
        mbar_init(smem_u32(&S.mbar), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
}

// TMA bulk copy of delta bytes [win0, wend) of pk, win0 16-byte aligned, into S.payload (rounded up to 16 bytes);
// returns when they are there.  parity is the phase of S.mbar the copy completes and flips with every copy.
__device__ __forceinline__ void warp_window_load(const DPack& pk, u64 win0, u64 wend, DWarpSmem& S, u32& parity,
                                                 int lane) {
    const u32 bytes = (u32)(((wend - win0) + 15ull) & ~15ull);
    const u32 bar = smem_u32(&S.mbar);
    if (lane == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_expect_tx(bar, bytes);
        if (bytes) tma_bulk_g2s(smem_u32(S.payload), pk.deltas + win0, bytes, bar);  // blocks of one uid have none
    }
    mbar_wait(bar, parity);
    parity ^= 1u;
}

// Every lane with `walk` set records the payload offsets of its block's ngroups groups in column `lane` of S.goff;
// the block's delta bytes are [doff, dnext) of the pack, in the window that starts at win0.  A corrupt tag may claim
// more bytes than the block holds: the walk stops at the block's end (the reference zero-pads a short tail,
// codec.go:176-188; here the next block's bytes are read instead -- garbage in, garbage out, but never outside the
// window).
__device__ __forceinline__ void warp_tag_walk(DWarpSmem& S, bool walk, u64 doff, u64 dnext, u64 win0, u32 ngroups,
                                              int lane) {
    if (walk) {
        u32 off = (u32)(doff - win0);
        const u32 off_end = (u32)(dnext - win0);
        for (u32 g = 0; g < ngroups; ++g) {
            S.goff[g * D_TSTRIDE + lane] = (unsigned short)off;
            off += gv_bytes_used(S.payload[off]);
            off = off < off_end ? off : off_end;
        }
    }
    __syncwarp();
}

// Block i of the batch, its ng_i group offsets in column i of S.goff, expanded into S.stage[0, NumUids): Base, then
// the running sums of its deltas -- lane g decodes group g (unaligned 16-byte read, four extractions), and a 64-bit
// warp prefix sum (`last + uint64(delta)`, codec.go:191-196) carries the sums across lanes and rounds of 32 groups.
__device__ __forceinline__ void expand_block(DWarpSmem& S, int i, u32 ng_i, u64 base_i, int lane) {
    const u32* pl32 = reinterpret_cast<const u32*>(S.payload);
    if (lane == 0) S.stage[0] = base_i;
    u64 carry = 0;
    for (u32 g0 = 0; g0 < ng_i; g0 += 32) {
        const u32 g = g0 + lane;
        u32 d0 = 0, d1 = 0, d2 = 0, d3 = 0;
        if (g < ng_i) {
            const u32 off = S.goff[g * D_TSTRIDE + i];
            const u32 tag = S.payload[off];
            const u32 a = off + 1;
            const u32 wb = a >> 2, sh = (a & 3u) * 8u;
            const u32 w0 = pl32[wb], w1 = pl32[wb + 1], w2 = pl32[wb + 2], w3 = pl32[wb + 3], w4 = pl32[wb + 4];
            const u32 D0 = __funnelshift_r(w0, w1, sh), D1 = __funnelshift_r(w1, w2, sh);
            const u32 D2 = __funnelshift_r(w2, w3, sh), D3 = __funnelshift_r(w3, w4, sh);
            const u32 l0 = (tag & 3u) + 1u, l1 = ((tag >> 2) & 3u) + 1u;
            const u32 l2 = ((tag >> 4) & 3u) + 1u, l3 = (tag >> 6) + 1u;
            auto extract = [&](u32 s, u32 l) -> u32 {
                const u32 wi = s >> 2, sh2 = (s & 3u) * 8u;
                const u32 lo = wi == 0 ? D0 : (wi == 1 ? D1 : (wi == 2 ? D2 : D3));
                const u32 hi = wi == 0 ? D1 : (wi == 1 ? D2 : (wi == 2 ? D3 : 0u));
                return __funnelshift_r(lo, hi, sh2) & (0xffffffffu >> (32u - 8u * l));
            };
            d0 = extract(0, l0);
            d1 = extract(l0, l1);
            d2 = extract(l0 + l1, l2);
            d3 = extract(l0 + l1 + l2, l3);
        }
        const u64 p1 = d0, p2 = p1 + d1, p3 = p2 + d2, p4 = p3 + d3;
        u64 inc = p4;
#pragma unroll
        for (int dlt = 1; dlt < 32; dlt <<= 1) {
            u64 t = __shfl_up_sync(0xffffffffu, inc, dlt);
            if (lane >= dlt) inc += t;
        }
        const u64 ex = base_i + carry + inc - p4;
        if (g < ng_i) {
            const u32 idx = 1u + 4u * g;  // uid index of this group's first value
            S.stage[idx] = ex + p1;
            S.stage[idx + 1] = ex + p2;
            S.stage[idx + 2] = ex + p3;
            S.stage[idx + 3] = ex + p4;
        }
        carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    __syncwarp();
}

// One warp decodes blocks [first_block + gw*D_BPW, +D_BPW) of `pk` into out[uid_off - skip ...].
__device__ __forceinline__ void decode_warp_run(const DPack& pk, u64 first_block, u64 skip, u64* __restrict__ out,
                                                u64 gw, DWarpSmem& S, int lane) {
    u64 b = first_block + gw * D_BPW;
    const u64 bend = (b + D_BPW < pk.nblocks) ? b + D_BPW : pk.nblocks;
    if (b >= bend) return;  // whole warp
    warp_mbar_init(S, lane);
    u32 parity = 0;

    while (b < bend) {
        // ---- batch geometry ----------------------------------------------------
        const u64 bi = b + lane;
        const bool in = bi < bend;
        const u64 doff = in ? pk.delta_off[bi] : 0;
        const u64 dnext = in ? pk.delta_off[bi + 1] : 0;
        const u64 win0 = __shfl_sync(0xffffffffu, doff, 0) & ~15ull;  // 16-byte aligned window start
        const bool fits = in && (dnext - win0 <= (u64)D_WB);
        const unsigned fm = __ballot_sync(0xffffffffu, fits);
        // leading run of blocks that fit (at least one: a block is <= 1088 B at BlockSize 256)
        int nb = __ffs(~fm) - 1;
        if (fm == 0xffffffffu) nb = 32;
        if (nb == 0) nb = 1;  // oversize block (BlockSize > 256*7): handled by the slow path below
        const u64 wend = __shfl_sync(0xffffffffu, dnext, nb - 1);
        const u32 num = in ? pk.num[bi] : 0;
        const u64 base = in ? pk.base[bi] : 0;
        const u64 uoff = in ? pk.uid_off[bi] : 0;
        const u32 ngroups = gv_groups(num);

        const bool oversize = (wend - win0 > (u64)D_WB) || (num > 256u && lane < nb);
        if (__any_sync(0xffffffffu, oversize)) {
            // Generic slow path (BlockSize > 256 packs): lane-serial decode straight from
            // global memory, one block per lane.  Never taken at the reference's BlockSize 256.
            if (lane < nb && in)
                gv_walk_block(pk.deltas + doff, base, num, [&](u32 i, u64 uid) {
                    if (uoff + i >= skip) st_stream(out + (uoff + i - skip), uid);
                    return true;
                });
            b += nb;
            continue;
        }

        // ---- (1) TMA bulk copy of the batch's delta bytes ------------------------
        if (pk.sysmem) {
            // Zero-copy: the pack's bytes are read straight from pinned host memory by the lanes (16 bytes each,
            // all requests of the window in flight together); thousands of resident warps keep PCIe full without
            // the per-copy set-up a DMA of every small pack costs, and nothing compressed is staged in HBM.
            const u32 bytes = (u32)(((wend - win0) + 15ull) & ~15ull);
            const uint4* src = reinterpret_cast<const uint4*>(pk.deltas + win0);
            uint4* dstw = reinterpret_cast<uint4*>(S.payload);
            for (u32 o = lane; o < bytes / 16u; o += 32) {
                uint4 q;
                asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                             : "=r"(q.x), "=r"(q.y), "=r"(q.z), "=r"(q.w) : "l"(src + o));
                dstw[o] = q;
            }
            __syncwarp();
        } else {
            warp_window_load(pk, win0, wend, S, parity, lane);
        }

        // ---- (2) tag walk: lane i records the byte offset of every group of block i
        warp_tag_walk(S, lane < nb, doff, dnext, win0, ngroups, lane);

        // ---- (3) cooperative decode, block by block --------------------------------
        for (int i = 0; i < nb; ++i) {
            const u32 n_i = __shfl_sync(0xffffffffu, num, i);
            const u64 base_i = __shfl_sync(0xffffffffu, base, i);
            const u64 uoff_i = __shfl_sync(0xffffffffu, uoff, i);
            const u32 ng_i = __shfl_sync(0xffffffffu, ngroups, i);
            expand_block(S, i, ng_i, base_i, lane);
            // coalesced write-out of uids [e0, n_i) of the block
            const u64 e0 = skip > uoff_i ? skip - uoff_i : 0;  // trimmed head (first block only)
            if (e0 < (u64)n_i) {
                u64* dst = out + (uoff_i + e0 - skip);
                const u64* src = S.stage + e0;
                const int cnt = (int)((u64)n_i - e0);
                const int head = (int)((reinterpret_cast<uintptr_t>(dst) >> 3) & 1);
                if (lane == 0 && head) st_stream(dst, src[0]);
                const int npairs = (cnt - head) >> 1;
                for (int p = lane; p < npairs; p += 32)
                    st_stream2(dst + head + 2 * p, src[head + 2 * p], src[head + 2 * p + 1]);
                if (lane == 31 && ((cnt - head) & 1)) st_stream(dst + cnt - 1, src[cnt - 1]);
            }
            __syncwarp();
        }
        b += nb;
    }
}

__global__ void __launch_bounds__(D_NT) decode_kernel(const DPack pk, const DSeek* __restrict__ seekp,
                                                      u64* __restrict__ out, u64 out_cap) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    DWarpSmem& S = reinterpret_cast<DWarpSmem*>(smem_raw)[wid];
    if (seekp->out_len > out_cap) return;  // error already flagged by decode_seek_kernel
    decode_warp_run(pk, seekp->first_block, seekp->skip, out, (u64)blockIdx.x * D_WARPS + wid, S, lane);
}

// Several packs decoded in full (seek 0) by ONE launch: the k posting lists of a query arrive as
// UidPacks (1.3-1.6 B/UID over PCIe) and are expanded side by side.  Job j owns warps
// [warp_base[j], warp_base[j+1]) of the grid.
struct DJob {
    DPack pk;
    u64* out;
    u64 warp_base;
};
__global__ void __launch_bounds__(D_NT) decode_batch_kernel(const DJob* __restrict__ jobs, u32 njobs, u64 nwarps) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    DWarpSmem& S = reinterpret_cast<DWarpSmem*>(smem_raw)[wid];
    const u64 gw = (u64)blockIdx.x * D_WARPS + wid;
    if (gw >= nwarps) return;
    const u32 j = job_of<DJob, &DJob::warp_base>(jobs, njobs, gw);
    const DPack pk = jobs[j].pk;
    decode_warp_run(pk, 0, 0, jobs[j].out, gw - jobs[j].warp_base, S, lane);
}

}  // namespace dgx
