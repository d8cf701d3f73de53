// compressed_kernel.cuh -- algo.IntersectCompressedWith fused on the device, and the Decoder's seeks.
//
// algo.IntersectCompressedWith(pack, afterUID, v, o) (algo/uidlist.go:33-138) intersects a UidPack with a
// plain list WITHOUT decoding the whole pack: the reference walks block bases (Decoder.SeekToBlock /
// LinearSeek, codec/codec.go:219-271, 349-359) and unpacks only blocks that can hold an element of v.
// Same idea here, data-parallel:
//   icw_ranges_*     block b can only match v[j] with base[b] <= v[j] < base[b+1]: the v-range of every
//                    block (searching the block bases with v, or v with the bases, whichever side is
//                    shorter: icw_range_by_v / icw_range_by_block, shared with the rows form).  Blocks with
//                    an empty range are never touched again.
//   icw_probe_kernel a warp owns 64 consecutive blocks (as in decode_kernel): per batch of 32 it TMA-copies
//                    only the delta bytes between the first and last touched block, walks the tags of
//                    touched blocks, expands each into the warp's shared-memory row and probes it with
//                    the block's slice of v (or probes that slice with the row when the slice is the
//                    longer side).  A match sets keep[j]; nothing decoded ever reaches HBM.  The walk is
//                    icw_probe_blocks, shared with the rows form, which differs only in where a match goes.
//   compact_kernel   o.Uids = v[keep], order preserved, single pass (decoupled look-back).
// The block format itself (window copy, tag walk, block expansion, lane-serial walk) is read through the helpers
// of decode_kernel.cuh.
// Defined, like the reference's own tests (algo/uidlist_test.go:607-681), for duplicate-free inputs.
#pragma once

#include "decode_kernel.cuh"

namespace dgx {

struct IcwParams {
    DPack pk;
    const u64* v;      // the plain list, ascending
    u64 m;
    u64 after;         // Decoder.Seek(after, SeekStart): only pack uids >= after take part (0: all)
    u32* vlo;          // per block: first index of v inside the block's value range ...
    u32* vhi;          // ... and one past the last (vlo == vhi: block not touched); zero-initialised
    unsigned char* keep;  // per v element: 1 when present in the pack; zero-initialised
};

// Element j of v: the block whose range holds v[j]; the first and the last element of a block's run write its
// vlo / vhi.
__device__ __forceinline__ void icw_range_by_v(const DPack& pk, const u64* v, u64 m, u64 after, u64 j, u32* vlo,
                                               u32* vhi) {
    const u64 x = v[j];
    if (x < after) return;
    const long long b = pack_block_of(pk, x);
    if (b < 0) return;  // before the pack's range
    long long bp = -2, bn = -2;
    if (j > 0) { const u64 xp = v[j - 1]; if (xp >= after) bp = pack_block_of(pk, xp); }
    if (j + 1 < m) bn = pack_block_of(pk, v[j + 1]);
    if (bp != b) vlo[b] = (u32)j;
    if (bn != b) vhi[b] = (u32)(j + 1);
}

// Block b: [lower_bound(v, max(base[b], after)), lower_bound(v, base[b+1])), written when not empty.
__device__ __forceinline__ void icw_range_by_block(const DPack& pk, const u64* v, u64 m, u64 after, u64 b, u32* vlo,
                                                   u32* vhi) {
    const u64 first = pk.base[b];
    const u64 lo = lower_bound_g(v, m, first > after ? first : after);
    const u64 hi = (b + 1 < pk.nblocks) ? lower_bound_g(v, m, pk.base[b + 1]) : m;
    if (hi > lo) { vlo[b] = (u32)lo; vhi[b] = (u32)hi; }
}

__global__ void __launch_bounds__(256) icw_ranges_by_v_kernel(const IcwParams P) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < P.m) icw_range_by_v(P.pk, P.v, P.m, P.after, j, P.vlo, P.vhi);
}

__global__ void __launch_bounds__(256) icw_ranges_by_block_kernel(const IcwParams P) {
    const u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (b < P.pk.nblocks) icw_range_by_block(P.pk, P.v, P.m, P.after, b, P.vlo, P.vhi);
}

// Where icw_probe_blocks puts a match.  Per batch, batch() reads what each lane's block needs; a block of more than 256
// uids is walked by its own lane, which reports each match with walk_hit() and ends with walk_done(); any other
// block is probed by the whole warp between open() and close(), which receives the matches of 32 probes at a time
// through hit().
template <class Flag>
struct IcwKeepSink {  // a match sets keep[j]
    Flag* keep;
    __device__ __forceinline__ void batch(u64, bool) {}
    __device__ __forceinline__ void walk_hit(u64 j, u64) { keep[j] = 1; }
    __device__ __forceinline__ void walk_done(u64) {}
    __device__ __forceinline__ void open(int) {}
    __device__ __forceinline__ void hit(bool h, u64 j, u64) { if (h) keep[j] = 1; }
    __device__ __forceinline__ void close(u64, int) {}
};
struct IcwSlotSink {  // rows form: matches go in ascending order to the block's slot, with a count per block
    u64* slots;
    const u64* slot_off;  // the pack's blocks: slot of block b = slots[slot_off[b], slot_off[b+1])
    u64* cnt;             // the pack's blocks: matches written
    unsigned below;       // lanes before this one
    u64 s0, scap;         // the lane's block of the batch
    u64 s0_i, scap_i;     // the block between open() and close()
    u64 w;                // matches so far in the block
    __device__ __forceinline__ void batch(u64 bi, bool touched) {
        s0 = touched ? slot_off[bi] : 0;
        scap = touched ? slot_off[bi + 1] - s0 : 0;
        w = 0;
    }
    __device__ __forceinline__ void walk_hit(u64, u64 y) {
        if (w < scap) slots[s0 + w] = y;
        ++w;
    }
    __device__ __forceinline__ void walk_done(u64 bi) { cnt[bi] = w < scap ? w : scap; }
    __device__ __forceinline__ void open(int i) {
        s0_i = __shfl_sync(0xffffffffu, s0, i);
        scap_i = __shfl_sync(0xffffffffu, scap, i);
        w = 0;
    }
    __device__ __forceinline__ void hit(bool h, u64, u64 x) {
        const unsigned hm = __ballot_sync(0xffffffffu, h);
        const u64 k = w + __popc(hm & below);
        if (h && k < scap_i) slots[s0_i + k] = x;
        w += __popc(hm);
    }
    __device__ __forceinline__ void close(u64 b, int lane) {
        if (lane == 0) cnt[b] = w < scap_i ? w : scap_i;
    }
};

// The block expanded in S.stage[0, n) probed with v[lo, hi) by the whole warp, the shorter side searching the longer
// one; matches go to the sink 32 probes at a time.
template <class Sink>
__device__ __forceinline__ void icw_probe_slice(const DWarpSmem& S, u32 n, const u64* v, u32 lo, u32 hi, Sink& sink,
                                                int lane) {
    if (hi - lo <= 4u * n) {
        for (u32 j0 = lo; j0 < hi; j0 += 32) {
            const u32 j = j0 + lane;
            u64 x = 0;
            bool h = false;
            if (j < hi) {
                x = ld_stream(v + j);
                const int pos = lower_bound_s(S.stage, 0, (int)n, x);
                h = pos < (int)n && S.stage[pos] == x;
            }
            sink.hit(h, j, x);
        }
    } else {
        for (u32 e0 = 0; e0 < n; e0 += 32) {
            const u32 e = e0 + lane;
            u64 y = 0, pos = 0;
            bool h = false;
            if (e < n) {
                y = S.stage[e];
                pos = lo + lower_bound_g(v + lo, (u64)(hi - lo), y);
                h = pos < hi && ld_probe(v + pos) == y;
            }
            sink.hit(h, pos, y);
        }
    }
}

// One warp probes blocks [b, b + D_BPW) of pk with their v-ranges [vlo, vhi): per batch of 32 blocks, one window
// copy from the first touched block to the last one that fits, the tag walk of the touched blocks, then each touched
// block expanded into S.stage and probed, the shorter side searching the longer one.
template <class Sink>
__device__ __forceinline__ void icw_probe_blocks(const DPack& pk, const u32* vlo, const u32* vhi, const u64* v, u64 b,
                                                 Sink& sink, DWarpSmem& S, int lane) {
    const u64 bend = (b + D_BPW < pk.nblocks) ? b + D_BPW : pk.nblocks;
    if (b >= bend) return;
    warp_mbar_init(S, lane);
    u32 parity = 0;

    while (b < bend) {
        const u64 bi = b + lane;
        const bool in = bi < bend;
        const u32 lo = in ? vlo[bi] : 0u, hi = in ? vhi[bi] : 0u;
        const bool tch = in && hi > lo;
        const unsigned touched = __ballot_sync(0xffffffffu, tch);
        if (touched == 0) { b += 32; continue; }  // nothing of v falls into these 32 blocks
        const int f = __ffs(touched) - 1;          // first touched block of the batch
        const u64 doff = in ? pk.delta_off[bi] : 0;
        const u64 dnext = in ? pk.delta_off[bi + 1] : 0;
        sink.batch(bi, tch);
        const u64 win0 = __shfl_sync(0xffffffffu, doff, f) & ~15ull;
        // blocks f .. l whose bytes fit the window together (l >= f: one block is at most 1088 B at BlockSize 256)
        const bool fits = in && lane >= f && (dnext - win0 <= (u64)D_WB);
        const unsigned fm = __ballot_sync(0xffffffffu, fits) >> f;
        int run = __ffs(~fm) - 1;                  // leading run of fitting blocks, counted from f
        if (fm == (0xffffffffu >> f)) run = 32 - f;
        const u32 num = in ? pk.num[bi] : 0;
        const bool oversize = run == 0 || (num > 256u && lane >= f && lane < f + (run ? run : 1));
        if (__any_sync(0xffffffffu, oversize)) {
            // Generic slow path (non-reference BlockSize): lane-serial walk of the touched blocks from global
            // memory, every decoded uid binary-searched in the block's slice of v.
            const int r = run ? run : 1;
            if (tch && lane >= f && lane < f + r) {
                gv_walk_block(pk.deltas + doff, pk.base[bi], num, [&](u32, u64 y) {
                    const u64 pos = lo + lower_bound_g(v + lo, (u64)(hi - lo), y);
                    if (pos < hi && ld_probe(v + pos) == y) sink.walk_hit(pos, y);
                    return true;
                });
                sink.walk_done(bi);
            }
            b += f + r;
            continue;
        }
        // last touched block inside the run: nothing behind it needs copying
        const unsigned in_run = (run >= 32 ? 0xffffffffu : ((1u << run) - 1u)) << f;
        const unsigned want = touched & in_run;
        const int last_t = 31 - __clz(want);
        const u64 wend = __shfl_sync(0xffffffffu, dnext, last_t);
        const u64 base = in ? pk.base[bi] : 0;
        const u32 ngroups = gv_groups(num);
        warp_window_load(pk, win0, wend, S, parity, lane);
        warp_tag_walk(S, (want >> lane) & 1u, doff, dnext, win0, ngroups, lane);  // touched blocks only

        for (unsigned rest = want; rest; rest &= rest - 1) {
            const int i = __ffs(rest) - 1;
            const u32 n_i = __shfl_sync(0xffffffffu, num, i);
            const u64 base_i = __shfl_sync(0xffffffffu, base, i);
            const u32 ng_i = __shfl_sync(0xffffffffu, ngroups, i);
            const u32 lo_i = __shfl_sync(0xffffffffu, lo, i), hi_i = __shfl_sync(0xffffffffu, hi, i);
            sink.open(i);
            expand_block(S, i, ng_i, base_i, lane);
            icw_probe_slice(S, n_i, v, lo_i, hi_i, sink, lane);
            sink.close(b + i, lane);
            __syncwarp();
        }
        b += f + run;
    }
}

__global__ void __launch_bounds__(D_NT) icw_probe_kernel(const IcwParams P) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    DWarpSmem& S = reinterpret_cast<DWarpSmem*>(smem_raw)[wid];
    IcwKeepSink<unsigned char> sink{P.keep};
    icw_probe_blocks(P.pk, P.vlo, P.vhi, P.v, ((u64)blockIdx.x * D_WARPS + wid) * D_BPW, sink, S, lane);
}

// ---- order-preserving compaction of v by keep[] (single pass, decoupled look-back) ------------
constexpr int CP_NT = 256, CP_VT = 8, CP_TILE = CP_NT * CP_VT;
struct CompactParams {
    const u64* v;
    const unsigned char* keep;
    u64 m;
    u64* out;
    u64 out_cap;
    u64* out_len;
    u64* status;   // ceil(m / CP_TILE) words, zeroed
    u32* ticket;   // zeroed: tiles are numbered in the order their CTAs start (no look-back deadlock)
    int* err;
};
__global__ void __launch_bounds__(CP_NT) compact_kernel(const CompactParams P) {
    __shared__ u32 warp_sums[CP_NT / 32 + 1];
    __shared__ u64 s_base;
    __shared__ u32 s_tile;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(P.ticket, 1u);
    __syncthreads();
    const u32 tile = s_tile;
    const u64 t0 = (u64)tile * CP_TILE;
    // thread owns CP_VT consecutive elements: order inside the tile is thread order
    u32 flags = 0, cnt = 0;
    const u64 e0 = t0 + (u64)tid * CP_VT;
#pragma unroll
    for (int i = 0; i < CP_VT; ++i)
        if (e0 + i < P.m && P.keep[e0 + i]) { flags |= 1u << i; ++cnt; }
    u32 total;
    const u32 ex = block_exclusive_scan<CP_NT>(cnt, warp_sums, &total);
    if (wid == 0) {
        const u64 base = lookback_exclusive(P.status, tile, (u64)total, lane);
        if (lane == 0) {
            s_base = base;
            if (t0 + CP_TILE >= P.m) {
                *P.out_len = base + total;
                if (base + total > P.out_cap) atomicExch(P.err, 1);
            }
        }
    }
    __syncthreads();
    u64 w = s_base + ex;
#pragma unroll
    for (int i = 0; i < CP_VT; ++i)
        if ((flags >> i) & 1u) {
            if (w < P.out_cap) P.out[w] = P.v[e0 + i];
            ++w;
        }
}

// ---- many packs, one v, one afterUID: the rows of a task's uid matrix -----------------------------
// handleUidPostings (worker/task.go:783-987) intersects every key's pack with the same v from the same afterUID.
// The blocks of all non-empty packs form ONE flat block space (pack after pack) and the batch runs a fixed number
// of launches whatever the row count; the workspace is a few words per flat block plus one slot buffer:
//   icw_rows_ranges_kernel  per-block v-ranges of every pack, the shorter side searched per row (as above)
//   icw_rows_slots_kernel   slot of block b = min(vhi - vlo, NumUids_b): at most that many of its v match
//   scan_u64_kernel         slot offsets (flat block order = row order, then block order)
//   icw_rows_probe_kernel   icw_probe_kernel's warp-per-64-blocks walk; matches go in order to the block's slot
//                           (warp ballot + popc) with a per-block count
//   scan_u64_kernel         counts -> final positions; out_off[i] = position of row i's first block
//   icw_rows_gather_kernel  slots -> out, CSR
// Slots of one row sum to at most min(m, ExactLen): their total stays within the caller's out_cap bound.
struct IcwJob {              // one non-empty pack
    DPack pk;
    u64 blk_base;            // its first block in the flat block space
    u64 thr_base;            // its first thread in the ranges launch
    u64 warp_base;           // its first warp in the probe launch
    u32 by_v;                // nblocks > m: ranges from v's side (m threads) instead of the blocks' (nblocks threads)
};
struct IcwRowsParams {
    const IcwJob* jobs;
    u32 njobs;
    const u64* v;
    u64 m;
    u64 after;
    u64 nblocks;             // flat blocks
    u64 nthreads;            // ranges launch
    u64 nwarps;              // probe launch
    u32* vlo;                // per flat block, zero-initialised (vlo == vhi: not touched)
    u32* vhi;
    u64* slot;               // per flat block: slot size; scanned into slot_off (nblocks + 1)
    u64* slot_off;
    u64* cnt;                // per flat block: matches; scanned into cnt_off (nblocks + 1)
    u64* cnt_off;
    u64* slots;              // slots_cap values
    u64 slots_cap;
    const u64* row_blk;      // nrows + 1: first flat block of each row (row_blk[nrows] = nblocks)
    u64 nrows;
    u64* out;
    u64 out_cap;
    u64* out_off;            // nrows + 1
    int* err;
};

__global__ void __launch_bounds__(256) icw_rows_ranges_kernel(const IcwRowsParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.nthreads) return;
    const IcwJob& J = P.jobs[job_of<IcwJob, &IcwJob::thr_base>(P.jobs, P.njobs, t)];
    const u64 k = t - J.thr_base;
    const DPack pk = J.pk;  // in registers: the searches read base and nblocks again and again
    u32* vlo = P.vlo + J.blk_base;
    u32* vhi = P.vhi + J.blk_base;
    if (J.by_v) icw_range_by_v(pk, P.v, P.m, P.after, k, vlo, vhi);
    else icw_range_by_block(pk, P.v, P.m, P.after, k, vlo, vhi);
}

__global__ void __launch_bounds__(256) icw_rows_slots_kernel(const IcwRowsParams P) {
    const u64 fb = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (fb >= P.nblocks) return;
    const IcwJob& J = P.jobs[job_of<IcwJob, &IcwJob::blk_base>(P.jobs, P.njobs, fb)];
    const u32 lo = P.vlo[fb], hi = P.vhi[fb];
    const u32 num = J.pk.num[fb - J.blk_base];
    const u32 n = hi > lo ? hi - lo : 0u;
    P.slot[fb] = n < num ? n : num;
    P.cnt[fb] = 0;
}

__global__ void __launch_bounds__(D_NT) icw_rows_probe_kernel(const IcwRowsParams P) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    DWarpSmem& S = reinterpret_cast<DWarpSmem*>(smem_raw)[wid];
    const u64 gw = (u64)blockIdx.x * D_WARPS + wid;
    // slots beyond the buffer only arise from a pack whose bases do not ascend: nothing is written then
    if (gw >= P.nwarps || P.slot_off[P.nblocks] > P.slots_cap) return;
    const IcwJob& J = P.jobs[job_of<IcwJob, &IcwJob::warp_base>(P.jobs, P.njobs, gw)];
    const DPack pk = J.pk;
    IcwSlotSink sink{P.slots, P.slot_off + J.blk_base, P.cnt + J.blk_base, (1u << lane) - 1u};
    icw_probe_blocks(pk, P.vlo + J.blk_base, P.vhi + J.blk_base, P.v, (gw - J.warp_base) * D_BPW, sink, S, lane);
}

// Thread t <= nrows writes out_off[t]; warp w moves block w's matches from its slot to their final place.
__global__ void __launch_bounds__(256) icw_rows_gather_kernel(const IcwRowsParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t <= P.nrows) P.out_off[t] = P.cnt_off[P.row_blk[t]];
    const bool bad = P.cnt_off[P.nblocks] > P.out_cap || P.slot_off[P.nblocks] > P.slots_cap;
    if (bad) {
        if (t == 0) atomicExch(P.err, 1);
        return;  // past out_cap nothing is written
    }
    const u64 fb = t >> 5;
    if (fb >= P.nblocks) return;
    const u64 c = P.cnt[fb];
    const u64* src = P.slots + P.slot_off[fb];
    u64* dst = P.out + P.cnt_off[fb];
    for (u64 k = t & 31; k < c; k += 32) dst[k] = src[k];
}

// ---- one pack, many v: the rows of a uid matrix against one posting list -------------------------
// intersectBucket (worker/sort.go:605-700) intersects every row of a uid matrix with the same index bucket's pack
// (afterUID 0).  The rows are the concatenation v[0 .. M), row i = v[v_off[i] .. v_off[i+1]).  A UNIT is the run of
// one row's elements inside one block's value range.  Membership of v[j] in the pack is all the result needs: keep[j]
// is set on a match, and the CSR result is v compacted by keep (row i starts at the count of matches before v_off[i]).
//   icw_mx_locate_kernel  thread per element: its row (search of v_off), the rows-ascend check, its block (search of
//                         the bases); the first element of a unit finds the unit's end by a search of its row and
//                         counts the unit for its block
//   scan_u64_kernel       units per block -> each block's first position in block order
//   icw_mx_place_kernel   thread per element: every unit takes a position in its block's range (block order)
//   icw_mx_probe_kernel   warp per 32 positions: one TMA window over the touched blocks, each distinct block expanded
//                         ONCE into shared memory and probed by all of its units in the warp; blocks of more than
//                         256 uids are walked lane-serially from global memory, one unit per lane
//   scan_u64_kernel       keep -> output positions
//   icw_mx_gather_kernel  out_off and out
// Work and workspace are linear in M + units + nrows + nblocks (units <= M); a block touched by every row is cut into
// pieces of 32 units, one per warp.  Every row must ascend strictly; the locate pass checks it (each thread reads its
// predecessor anyway), and a violation sets kLaneErrOrder in the lane's error flag and empties the result.
constexpr int kLaneErrOrder = 2;  // lane error flag bit: a row of a matrix call does not ascend (DGX_ERR_ARG at sync);
                                  // the flag's value 1 (result past out_cap, DGX_ERR_CAP) is unchanged
constexpr u32 MX_SERIAL = 8;      // units of at most this many elements are probed by their own lane
struct IcwMatrixParams {
    DPack pk;
    const u64* v;            // m values, rows concatenated
    u64 m;
    const u64* v_off;        // nrows + 1
    u64 nrows;
    u64* head;               // per element: (block << 32 | unit end) where a unit starts, else kU64Max
    u64* bcount;             // per block: units; zero-initialised
    u32* bfill;              // per block: units placed so far; zero-initialised
    u64* boff;               // nblocks + 1: first position of each block's units
    u64* unit;               // per position: lo | hi << 32 (v indices)
    u32* ublk;               // per position: block
    u64 unit_cap;            // positions allocated (= sum_i min(|row i|, nblocks) units of ascending rows)
    u64* keep;               // per element: 1 when in the pack
    u64* kex;                // m + 1: exclusive scan of keep
    u64* out;
    u64 out_cap;
    u64* out_off;            // nrows + 1
    int* bad;                // workspace word, zero-initialised: some row does not ascend
    int* err;
};

__global__ void __launch_bounds__(256) icw_mx_locate_kernel(const IcwMatrixParams P) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P.m) return;
    P.keep[k] = 0;
    u64 lo = 1, hi = P.nrows;  // row: last r with v_off[r] <= k (first r >= 1 with v_off[r] > k, minus one)
    while (lo < hi) {
        const u64 mid = lo + ((hi - lo) >> 1);
        if (ld_probe(P.v_off + mid) <= k) lo = mid + 1; else hi = mid;
    }
    const u64 s = ld_probe(P.v_off + lo - 1), e = ld_probe(P.v_off + lo);
    const u64 x = P.v[k];
    const u64 xp = k > s ? P.v[k - 1] : 0;
    if (k > s && xp >= x) {
        *P.bad = 1;
        atomicOr(P.err, kLaneErrOrder);
    }
    u64 hd = kU64Max;
    const long long b = pack_block_of(P.pk, x);
    if (b >= 0 && (k == s || xp < ld_probe(P.pk.base + b))) {  // the row's first element in block b
        const u64 end = (u64)b + 1 < P.pk.nblocks ? k + lower_bound_g(P.v + k, e - k, ld_probe(P.pk.base + b + 1)) : e;
        hd = ((u64)b << 32) | end;
        atomicAdd(P.bcount + b, 1ull);
    }
    P.head[k] = hd;
}

__global__ void __launch_bounds__(256) icw_mx_place_kernel(const IcwMatrixParams P) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P.m) return;
    const u64 hd = P.head[k];
    if (hd == kU64Max) return;
    const u32 b = (u32)(hd >> 32);
    const u64 pos = P.boff[b] + atomicAdd(P.bfill + b, 1u);
    if (pos >= P.unit_cap) return;  // only when a row does not ascend: the result is discarded then
    P.unit[pos] = k | (hd << 32);
    P.ublk[pos] = b;
}

__global__ void __launch_bounds__(D_NT) icw_mx_probe_kernel(const IcwMatrixParams P) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    DWarpSmem& S = reinterpret_cast<DWarpSmem*>(smem_raw)[wid];
    const DPack& pk = P.pk;
    const u64 nu = min(P.boff[pk.nblocks], P.unit_cap);
    const u64 p0 = ((u64)blockIdx.x * D_WARPS + wid) * 32;
    if (p0 >= nu) return;
    const int nin = (int)min(nu - p0, (u64)32);
    const bool in = lane < nin;
    const u64 lh = in ? P.unit[p0 + lane] : 0;
    const u32 blk = in ? P.ublk[p0 + lane] : 0u;
    const u32 lo = (u32)lh, hi = (u32)(lh >> 32);
    const u64 doff = in ? pk.delta_off[blk] : 0, dnext = in ? pk.delta_off[blk + 1] : 0;
    const u32 num = in ? pk.num[blk] : 0u;
    const u64 base = in ? pk.base[blk] : 0;
    const u32 ngroups = gv_groups(num);
    const u32 bup = __shfl_up_sync(0xffffffffu, blk, 1);
    IcwKeepSink<u64> sink{P.keep};
    warp_mbar_init(S, lane);
    u32 parity = 0;

    int f = 0;  // lanes [0, f) are done; positions are in block order, so a block's units are adjacent lanes
    while (f < nin) {
        const u64 win0 = __shfl_sync(0xffffffffu, doff, f) & ~15ull;
        const bool ok = in && lane >= f && num <= 256u && (dnext - win0 <= (u64)D_WB);
        const unsigned om = __ballot_sync(0xffffffffu, ok) >> f;
        const int run = om == (0xffffffffu >> f) ? 32 - f : __ffs(~om) - 1;  // leading lanes whose blocks fit the window
        if (run == 0) {
            // block of more than 256 uids (non-reference BlockSize): every unit of it walks it from global memory
            const u32 bf = __shfl_sync(0xffffffffu, blk, f);
            const unsigned grp = __ballot_sync(0xffffffffu, in && lane >= f && blk == bf);
            if ((grp >> lane) & 1u) {
                u32 q = lo;
                gv_walk_block(pk.deltas + doff, base, num, [&](u32, u64 uid) {  // merge step: both sides ascend
                    while (q < hi && ld_probe(P.v + q) < uid) ++q;
                    if (q < hi && ld_probe(P.v + q) == uid) P.keep[q] = 1;
                    return q < hi;
                });
            }
            f += __popc(grp);
            continue;
        }
        const int rend = f + run;
        const bool mine = lane >= f && lane < rend;
        // one leader per distinct block of the run; it walks the block's tags into its goff column
        const bool lead = mine && (lane == f || bup != blk);
        const unsigned leaders = __ballot_sync(0xffffffffu, lead);
        warp_window_load(pk, win0, __shfl_sync(0xffffffffu, dnext, rend - 1), S, parity, lane);
        warp_tag_walk(S, lead, doff, dnext, win0, ngroups, lane);

        for (unsigned rest = leaders; rest; rest &= rest - 1) {
            const int i = __ffs(rest) - 1;
            const unsigned later = (rest & (rest - 1));
            const int iend = later ? __ffs(later) - 1 : rend;  // units of this block: lanes [i, iend)
            const u32 n_i = __shfl_sync(0xffffffffu, num, i);
            const u64 base_i = __shfl_sync(0xffffffffu, base, i);
            const u32 ng_i = __shfl_sync(0xffffffffu, ngroups, i);
            expand_block(S, i, ng_i, base_i, lane);
            const bool grp = lane >= i && lane < iend;
            const u32 c = hi - lo;
            if (grp && c <= MX_SERIAL) {  // short units, side by side: each lane searches the block with its own
                for (u32 j = lo; j < hi; ++j) {
                    const u64 x = ld_probe(P.v + j);
                    const int pos = lower_bound_s(S.stage, 0, (int)n_i, x);
                    if (pos < (int)n_i && S.stage[pos] == x) P.keep[j] = 1;
                }
            }
            // longer units one after another with the whole warp, the shorter side searching the longer one
            for (unsigned big = __ballot_sync(0xffffffffu, grp && c > MX_SERIAL); big; big &= big - 1) {
                const int t = __ffs(big) - 1;
                const u32 lo_t = __shfl_sync(0xffffffffu, lo, t), hi_t = __shfl_sync(0xffffffffu, hi, t);
                icw_probe_slice(S, n_i, P.v, lo_t, hi_t, sink, lane);
            }
            __syncwarp();  // the next block's expansion overwrites S.stage
        }
        f = rend;
    }
}

// Thread t < m moves v[t] to its place when kept; thread t <= nrows writes out_off[t].  A row that does not ascend
// empties the result (out untouched, every offset 0); past out_cap nothing of out is written.
__global__ void __launch_bounds__(256) icw_mx_gather_kernel(const IcwMatrixParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) {
        if (t <= P.nrows) P.out_off[t] = 0;
        return;
    }
    if (t <= P.nrows) P.out_off[t] = P.kex[P.v_off[t]];
    if (P.kex[P.m] > P.out_cap) {
        if (t == 0) atomicExch(P.err, 1);
        return;
    }
    if (t < P.m && P.keep[t]) P.out[P.kex[t]] = P.v[t];
}

// ---- Decoder seeks on the device (codec/codec.go:219-384) --------------------------------------
// One thread restates the control flow of the reference's iterator for ONE call and expands the block it
// lands on; what comes back is what the Go call returns: the uid slice and the decoder's new block index.
// State carried between calls is the block index only (the current block counts as fully unpacked).
enum { SK_SEEK = 0, SK_SEEK_TO_BLOCK = 1, SK_LINEAR_SEEK = 2, SK_NEXT = 3, SK_UNPACK = 4 };
struct SeekParams {
    DPack pk;
    u64 uid;
    int whence;     // 0 SeekStart (>=), 1 SeekCurrent (>)
    int kind;
    u64 block_idx;  // the decoder's blockIdx before the call
    u64* out;       // up to max_num uids
    u64* out_meta;  // [0] = length, [1] = blockIdx after the call
};
__device__ __forceinline__ u32 sk_unpack(const DPack& pk, u64 b, u64* out) {  // Decoder.UnpackBlock (:154-200)
    if (b >= pk.nblocks) return 0;
    return gv_walk_block(pk.deltas + pk.delta_off[b], pk.base[b], pk.num[b], [&](u32 i, u64 uid) {
        out[i] = uid;
        return true;
    });
}
__global__ void pack_seek_kernel(const SeekParams P) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const DPack& pk = P.pk;
    const u64 nb = pk.nblocks;
    const bool gt = P.whence == 1;
    // sort.Search over Blocks[from:] for Base >= uid (SeekStart) / Base > uid (SeekCurrent)
    auto search_base = [&](u64 from) -> u64 {
        u64 lo = from, hi = nb;
        while (lo < hi) {
            const u64 mid = lo + ((hi - lo) >> 1);
            const u64 bs = pk.base[mid];
            if (gt ? (bs > P.uid) : (bs >= P.uid)) hi = mid; else lo = mid + 1;
        }
        return lo;
    };
    u64 blk = 0, len = 0, start = 0;
    auto next = [&]() { blk += 1; len = sk_unpack(pk, blk, P.out); start = 0; };  // Decoder.Next (:370-376)
    switch (P.kind) {
        case SK_UNPACK: blk = P.block_idx; len = sk_unpack(pk, blk, P.out); break;
        case SK_NEXT: blk = P.block_idx; next(); break;
        case SK_LINEAR_SEEK: {  // :349-359: advance while seek >= PeekNextBase (MaxUint64 past the last block)
            blk = P.block_idx;
            while (true) {
                const u64 nxt = (blk + 1 < nb) ? pk.base[blk + 1] : kU64Max;
                if (P.uid < nxt || blk >= nb) break;  // (the reference would spin forever on seek == MaxUint64)
                blk += 1;
            }
            len = sk_unpack(pk, blk, P.out);
            break;
        }
        case SK_SEEK: {  // :279-337
            if (P.uid == 0) { len = sk_unpack(pk, 0, P.out); break; }
            const u64 idx = search_base(0);
            if (idx == 0) { len = sk_unpack(pk, 0, P.out); break; }
            if (idx < nb && pk.base[idx] == P.uid) { blk = idx; len = sk_unpack(pk, blk, P.out); break; }
            blk = idx - 1;
            len = sk_unpack(pk, blk, P.out);
            u64 u = 0;
            while (u < len && (gt ? (P.out[u] <= P.uid) : (P.out[u] < P.uid))) ++u;
            if (u < len) { start = u; len -= u; } else next();
            break;
        }
        default: {  // SK_SEEK_TO_BLOCK, :219-271
            u64 prev = P.block_idx;
            if (P.uid == 0) { len = sk_unpack(pk, 0, P.out); break; }
            if (prev > 0 && prev < nb && P.uid < pk.base[prev]) prev = 0;
            if (prev > nb) prev = nb;
            const u64 idx = search_base(prev);
            if (idx == 0) { len = sk_unpack(pk, 0, P.out); break; }
            if (idx < nb && pk.base[idx] == P.uid) { blk = idx; len = sk_unpack(pk, blk, P.out); break; }
            blk = idx - 1;
            // `if d.blockIdx != prevBlockIdx { d.UnpackBlock() }` (:262-264): when the search was restarted from
            // block 0 for an older uid and lands on block 0, the reference keeps the slice it already held --
            // the block the decoder stood on before the call -- and tests uid against THAT slice.
            len = sk_unpack(pk, blk != prev ? blk : P.block_idx, P.out);
            if (!(len > 0 && P.uid <= P.out[len - 1])) next();
            break;
        }
    }
    if (start) for (u64 i = 0; i < len; ++i) P.out[i] = P.out[start + i];
    P.out_meta[0] = len;
    P.out_meta[1] = blk;
}

}  // namespace dgx
