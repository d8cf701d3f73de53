// filter_kernel.cuh -- the batch descriptors of the sorted-set filter, shared by the
// host (dgx_api.cu) and the kernels of filter_pipe.cuh.
//
// A batch of queries covers algo.IntersectWith (algo/uidlist.go:142), the whole chain
// of algo.IntersectSorted (:297-329, k lists in ONE pass), algo.Difference (:332) and
// the batched row-filter shape of worker/task.go:783 / query/query.go:1425.  Query q
// is a task: its lists are lists[list_first .. list_first + k), the first one the
// driving list A (its shortest list for intersections, u for Difference), cut into
// tiles numbered from tile_base.  FParams carries the batch and its outputs.
//
// Duplicate semantics (pinned by algo/uidlist_test.go:329-348): a candidate that
// is the r-th copy of x in A survives list L_j iff L_j holds more than r copies
// of x, i.e. L_j[lower_bound(x) + r] == x -- multiset-min for intersections and
// multiset difference, exactly what the reference's two-pointer merges produce.
// cand_rank recovers r from the tile, so tiles that contain repeated values keep
// their candidates in place (no re-packing).
#pragma once

#include "common.cuh"

namespace dgx {

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

}  // namespace dgx
