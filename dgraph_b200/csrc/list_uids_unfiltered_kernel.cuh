// list_uids_unfiltered_kernel.cuh -- posting.List.Uids without a filter for a task's rows, and the count of the same
// postings, the mutable layer included.
//
// handleUidPostings (worker/task.go:783-987) reads a plain edge traversal (`{ friend { name } }`) and `count(friend)`
// with opts.Intersect == nil.  Then List.Uids (posting/list.go:1758-1874) runs iterate(readTs, AfterUid) with the REF
// filter and no bounds for every key, and the First cut; Postings (:1878-1890) counts what the same iterate yields.
// Row i, with pack P_i (NULL: delete-all marker or empty immutable layer) and resolved entries mut_i (as for
// list_uids_kernel.cuh):
//   S_i = {x > after : mut_i(x) exists ? mut_i(x) has no flag : x in P_i}
//   row i = the min(|S_i|, first) smallest values of S_i, count i = |S_i|
// where `first` is the most values a row keeps (opts.First: 0 is MaxInt32; a negative First stops the callback after
// one value, so it keeps one).  Every pack uid above after and every inserting entry lands at
//   row start + (pack uids above after below it) - (drops below it) + (inserts below it)
// and nothing decoded is kept in HBM:
//   luu_classify_kernel  thread per entry: its row (search of mut_off), the order / zero / flag checks, the block of the
//                        row's pack that can hold it (pack_block_of), walked to find whether it is a pack uid and how many
//                        pack uids lie below it; an entry INSERTS (emits, not in the pack) or DROPS (does not emit, in
//                        the pack), above after only.  Then thread per row: the pack-starts-at-uid-0 check
//   scan_u64_kernel      drop | insert << 31 per entry -> counts of drops and inserts before every entry
//   luu_rows_kernel      thread per row: the seek block of after (walked once), the pack uids above after, |S_i|, the
//                        row length and the count
//   scan_u64_kernel      row lengths -> out_off
//   luu_write_kernel     warp per 64 blocks of the task's flat block space, as icw_rows_probe_kernel: blocks before the
//                        seek block, or whose first position is past the row's length, are never loaded; the others
//                        are expanded in shared memory and every kept uid is written at its position.  Then thread per
//                        inserting entry.
// The count entry points stop after luu_rows_kernel: they walk only the seek block of every row and the block every
// entry lands in.
#pragma once

#include "list_uids_kernel.cuh"

namespace dgx {

constexpr u32 kLuuNoJob = 0xffffffffu;  // row_job of a row with a NULL or empty pack

struct LuuJob {      // one row with a non-empty pack
    DPack pk;
    u64 row;
    u64 warp_base;   // its first warp in the write launch
};

struct LuuParams {
    const LuuJob* jobs;
    u32 njobs;
    u64 nwarps;                 // block warps of the write launch
    const u32* row_job;         // nrows: the row's job, kLuuNoJob without a pack
    const u64* mut_off;         // nrows + 1
    u64 nrows;
    const u64* mut;             // nmut resolved entries, rows concatenated
    const unsigned char* flags; // nmut
    u64 nmut;
    u64 after;
    u64 first;                  // the most values a row keeps (>= 1)
    u64* cls;                   // nmut: drop | insert << 31
    u64* cls_ex;                // nmut + 1: exclusive scan of cls
    u64* rank;                  // nmut: pack uids below the entry's uid (written for entries above after)
    u64* skip;                  // nrows: pack uids <= after
    u64* sblk;                  // nrows: the block holding the first pack uid above after
    u64* len;                   // nrows: row length, min(|S_i|, first)
    u32* counts;                // nrows, or null: |S_i|
    u64* out;
    u64 out_cap;
    u64* out_off;               // nrows + 1: exclusive scan of len
    int* bad;                   // workspace word, zero-initialised: some entry or pack is malformed
    int* err;
};

struct LuuPos {
    long long b;  // pack_block_of(x)
    u64 le;       // pack uids <= x
    bool hit;     // x is a pack uid
};

// Where x falls in a non-empty pack: the one block that can hold it, walked by this thread.
__device__ __forceinline__ LuuPos luu_locate(const DPack& pk, u64 x) {
    LuuPos s{pack_block_of(pk, x), 0, false};
    if (s.b < 0) return s;
    u32 le = 0;
    bool hit = false;
    gv_walk_block(pk.deltas + pk.delta_off[s.b], pk.base[s.b], pk.num[s.b], [&](u32, u64 y) {
        if (y > x) return false;
        ++le;
        hit = y == x;
        return !hit;
    });
    s.le = pk.uid_off[s.b] + le;
    s.hit = hit;
    return s;
}

// Thread k < nmut classifies entry k; thread nmut + r checks that row r's pack does not start at uid 0 (iterate reads
// uid 0 as the end of the list, :1178-1196).
__global__ void __launch_bounds__(256) luu_classify_kernel(const LuuParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.nmut) {
        const u64 r = t - P.nmut;
        if (r >= P.nrows) return;
        const u32 j = P.row_job[r];
        if (j != kLuuNoJob && ld_probe(P.jobs[j].pk.base) == 0) {
            *P.bad = 1;
            atomicOr(P.err, kLaneErrMut);
        }
        return;
    }
    const u64 k = t;
    const u64 r = lu_row_of(P.mut_off, P.nrows, k);
    const u64 x = P.mut[k];
    const unsigned f = P.flags[k];
    lu_check_entry(P, r, k, x, f);
    u64 c = 0, rank = 0;
    if (x > P.after) {  // iterate starts the mutable side at the first entry above after (:1126-1131)
        bool in_pack = false;
        const u32 j = P.row_job[r];
        if (j != kLuuNoJob) {
            const LuuPos s = luu_locate(P.jobs[j].pk, x);
            in_pack = s.hit;
            rank = s.le - (s.hit ? 1 : 0);
        }
        const bool emits = f == 0;  // a SET of a REF posting
        if (in_pack && !emits) c = kLuDrop;
        if (!in_pack && emits) c = kLuInsert;
    }
    P.cls[k] = c;
    P.rank[k] = rank;
}

// Thread per row: Seek(after, SeekCurrent) on the row's pack (:569), |S_i|, the row length and the count.  A malformed
// entry or pack empties every row.
__global__ void __launch_bounds__(256) luu_rows_kernel(const LuuParams P) {
    const u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= P.nrows) return;
    if (*P.bad) {
        P.len[r] = 0;
        if (P.counts) P.counts[r] = 0;
        return;
    }
    u64 skip = 0, sb = 0, above = 0;
    const u32 j = P.row_job[r];
    if (j != kLuuNoJob) {
        const DPack pk = P.jobs[j].pk;
        const LuuPos s = luu_locate(pk, P.after);
        skip = s.le;
        if (s.b >= 0) sb = s.le - pk.uid_off[s.b] < pk.num[s.b] ? (u64)s.b : (u64)s.b + 1;
        above = pk.uid_off[pk.nblocks] - skip;
    }
    const u64 d = P.cls_ex[P.mut_off[r + 1]] - P.cls_ex[P.mut_off[r]];
    const u64 n = lu_apply(above, d);
    P.skip[r] = skip;
    P.sblk[r] = sb;
    P.len[r] = n < P.first ? n : P.first;
    if (P.counts) P.counts[r] = (u32)n;
}

// Position in its row of a kept pack uid y of pack rank q (q >= skip): the row's entries of y's block are
// mut[js, je), and ms is the row's first entry.  kU64Max when an entry drops y.
__device__ __forceinline__ u64 luu_pos_of(const LuuParams& P, u64 y, u64 q, u64 skip, u64 ms, u64 js, u64 je) {
    const u64 j = js + lower_bound_g(P.mut + js, je - js, y);
    if (j < je && ld_probe(P.mut + j) == y && lu_drops(P.cls[j])) return kU64Max;
    const u64 below = P.cls_ex[j] - P.cls_ex[ms];
    return lu_apply(q - skip, below);
}

// One warp writes the kept uids of blocks [b, b + D_BPW) of row r's pack.  Per batch of 32 blocks: every lane finds
// its block's entries and the number of values of S below the block's base; the blocks whose values all lie past the
// row's length, and every block after them, are dropped before any delta byte is read; the rest is one window copy,
// the tag walk and each block expanded into S.stage and written.
__device__ __forceinline__ void luu_write_blocks(const LuuParams& P, const DPack& pk, u64 r, u64 b, DWarpSmem& S,
                                                 int lane) {
    const u64 skip = P.skip[r], sb = P.sblk[r], len = P.len[r], o0 = P.out_off[r];
    const u64 ms = P.mut_off[r], me = P.mut_off[r + 1];
    const u64 bend = (b + D_BPW < pk.nblocks) ? b + D_BPW : pk.nblocks;
    if (b < sb) b = sb;
    if (b >= bend || len == 0) return;
    warp_mbar_init(S, lane);
    u32 parity = 0;

    while (b < bend) {
        const u64 bi = b + lane;
        const bool in = bi < bend;
        u64 base = 0, uoff = 0, js = me, je = me, lower = 0;
        if (in) {
            base = pk.base[bi];
            uoff = pk.uid_off[bi];
            js = ms + lower_bound_g(P.mut + ms, me - ms, base);
            je = bi + 1 < pk.nblocks ? ms + lower_bound_g(P.mut + ms, me - ms, pk.base[bi + 1]) : me;
            if (bi > sb) {  // values of S below base: pack uids in (after, base) - drops + inserts below base
                const u64 d = P.cls_ex[js] - P.cls_ex[ms];
                lower = lu_apply(uoff - skip, d);
            }
        }
        // lower ascends with the block: the live blocks are lanes [0, last]
        const unsigned live = __ballot_sync(0xffffffffu, in && lower < len);
        if (live == 0) return;
        const int last = 31 - __clz(live);
        const u64 doff = in ? pk.delta_off[bi] : 0;
        const u64 dnext = in ? pk.delta_off[bi + 1] : 0;
        const u32 num = in ? pk.num[bi] : 0;
        const u64 win0 = __shfl_sync(0xffffffffu, doff, 0) & ~15ull;
        const bool fits = lane <= last && (dnext - win0 <= (u64)D_WB);
        const unsigned fm = __ballot_sync(0xffffffffu, fits);
        int run = __ffs(~fm) - 1;  // leading run of live blocks whose bytes fit the window together
        if (fm == 0xffffffffu) run = 32;
        const bool oversize = run == 0 || (num > 256u && lane < run);
        if (__any_sync(0xffffffffu, oversize)) {
            // Generic slow path (non-reference BlockSize): each live block of the run walked by its own lane.
            const int n = run ? run : 1;
            if (lane < n)
                gv_walk_block(pk.deltas + doff, base, num, [&](u32 e, u64 y) {
                    const u64 q = uoff + e;
                    if (q < skip) return true;
                    const u64 pos = luu_pos_of(P, y, q, skip, ms, js, je);
                    if (pos != kU64Max && pos < len) P.out[o0 + pos] = y;
                    return pos == kU64Max || pos < len;
                });
            b += n;
            continue;
        }
        const u64 wend = __shfl_sync(0xffffffffu, dnext, run - 1);
        warp_window_load(pk, win0, wend, S, parity, lane);
        warp_tag_walk(S, lane < run, doff, dnext, win0, gv_groups(num), lane);
        for (int i = 0; i < run; ++i) {
            const u32 n_i = __shfl_sync(0xffffffffu, num, i);
            const u64 base_i = __shfl_sync(0xffffffffu, base, i);
            const u64 uoff_i = __shfl_sync(0xffffffffu, uoff, i);
            const u64 js_i = __shfl_sync(0xffffffffu, js, i), je_i = __shfl_sync(0xffffffffu, je, i);
            expand_block(S, i, gv_groups(n_i), base_i, lane);
            for (u32 e = lane; e < n_i; e += 32) {
                const u64 q = uoff_i + e;
                if (q < skip) continue;
                const u64 y = S.stage[e];
                const u64 pos = luu_pos_of(P, y, q, skip, ms, js_i, je_i);
                if (pos != kU64Max && pos < len) st_stream(P.out + o0 + pos, y);
            }
            __syncwarp();
        }
        b += run;
    }
}

// CTAs [0, ceil(nwarps / D_WARPS)) write pack uids, a warp per 64 blocks; the CTAs after them write the inserting
// entries, a thread each.  A malformed entry or pack has emptied every row (out untouched); past out_cap nothing of out
// is written.
__global__ void __launch_bounds__(D_NT, 4) luu_write_kernel(const LuuParams P) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    if (*P.bad) return;
    if (P.out_off[P.nrows] > P.out_cap) {
        if (blockIdx.x == 0 && threadIdx.x == 0) atomicExch(P.err, 1);
        return;
    }
    const u64 g_blk = (P.nwarps + D_WARPS - 1) / D_WARPS;
    if (blockIdx.x < g_blk) {
        const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
        const u64 gw = (u64)blockIdx.x * D_WARPS + wid;
        if (gw >= P.nwarps) return;
        DWarpSmem& S = reinterpret_cast<DWarpSmem*>(smem_raw)[wid];
        const LuuJob& J = P.jobs[job_of<LuuJob, &LuuJob::warp_base>(P.jobs, P.njobs, gw)];
        const DPack pk = J.pk;
        luu_write_blocks(P, pk, J.row, (gw - J.warp_base) * D_BPW, S, lane);
        return;
    }
    const u64 k = (u64)(blockIdx.x - g_blk) * blockDim.x + threadIdx.x;
    if (k >= P.nmut || !lu_inserts(P.cls[k])) return;
    const u64 r = lu_row_of(P.mut_off, P.nrows, k);
    const u64 below = P.cls_ex[k] - P.cls_ex[ld_probe(P.mut_off + r)];
    const u64 pos = lu_apply(P.rank[k] - P.skip[r], below);
    if (pos < P.len[r]) P.out[P.out_off[r] + pos] = P.mut[k];
}

}  // namespace dgx
