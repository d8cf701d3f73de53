// dgx_algo.hpp -- C++ host-side mirror of dgraph's `algo` and `codec` packages over
// the libdgx C ABI (include/dgx.h).
//
// The reference is compiled Go and its toolchain is absent from this image, so the
// host layer above the C ABI is mirrored in C++: same function names, argument
// meaning, aliasing rules and nil/empty result shapes as
//   /root/reference/algo/uidlist.go   (IntersectWith :142, IntersectSorted :297,
//                                      MergeSorted :448, Difference :332)
//   /root/reference/codec/codec.go    (Decode :444, ApproxLen :418, ExactLen :427, DecodeToBuffer :456,
//                                      EncodeFromBuffer :402)
// Every body is one libdgx call -- exactly what the cgo shim (go/algo_dgx.go) does.
// Errors: the Go functions cannot fail; here a non-zero dgx status throws
// dgx::Error so callers (the shim: fall back to the Go code) can react.
#pragma once

#include <algorithm>
#include <cstdint>
#include <memory>
#include <numeric>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "dgx.h"

namespace dgx {

struct Error : std::runtime_error {
    int code;
    Error(int c, const char* msg) : std::runtime_error(std::string(msg)), code(c) {}
};
inline void check(int rc) {
    if (rc != DGX_OK) throw Error(rc, dgx_last_error());
}

namespace pb {
// pb.List (protos/pb.proto:22-24).  `nil` models a nil Uids slice.
struct List {
    std::vector<uint64_t> Uids;
    bool nil = false;
    List() = default;
    List(std::initializer_list<uint64_t> v) : Uids(v) {}
    explicit List(std::vector<uint64_t> v) : Uids(std::move(v)) {}
    static List Nil() { List l; l.nil = true; return l; }
};
// pb.UidPack flattened (protos/pb.proto:379-400): block b = {base[b], num_uids[b],
// deltas[delta_off[b] .. delta_off[b+1])}.
struct UidPack {
    uint32_t block_size = 0;
    std::vector<uint64_t> base;
    std::vector<uint32_t> num_uids;
    std::vector<uint64_t> delta_off{0};
    std::vector<uint8_t> deltas;
    dgx_pack_view view() const {
        dgx_pack_view v;
        v.block_size = block_size;
        v.nblocks = base.size();
        v.base = base.data();
        v.num_uids = num_uids.data();
        v.delta_off = delta_off.data();
        v.deltas = deltas.data();
        return v;
    }
};
}  // namespace pb

namespace algo {

// IntersectWith(u, v, o): o.Uids = u ∩ v.  `o` may be `u` (in place); `v` is never modified.
inline void IntersectWith(const pb::List& u, const pb::List& v, pb::List& o) {
    const size_t cap = std::min(u.Uids.size(), v.Uids.size());
    std::vector<uint64_t> out(std::max<size_t>(cap, 1));
    size_t n = 0;
    check(dgx_intersect2(u.Uids.data(), u.Uids.size(), v.Uids.data(), v.Uids.size(), out.data(), cap, &n));
    out.resize(n);
    o.Uids.swap(out);  // after the call: `u` may alias `o`
    o.nil = false;
}

// IntersectSorted(lists): no lists -> &pb.List{} (nil Uids); one list -> a copy.
inline pb::List IntersectSorted(const std::vector<const pb::List*>& lists) {
    if (lists.empty()) return pb::List::Nil();
    std::vector<const uint64_t*> ptrs;
    std::vector<size_t> lens;
    size_t cap = SIZE_MAX;
    for (const pb::List* l : lists) {
        ptrs.push_back(l->Uids.data());
        lens.push_back(l->Uids.size());
        cap = std::min(cap, l->Uids.size());
    }
    pb::List out;
    out.Uids.resize(std::max<size_t>(cap, 1));
    size_t n = 0;
    check(dgx_intersect_sorted(ptrs.data(), lens.data(), lists.size(), out.Uids.data(), cap, &n));
    out.Uids.resize(n);
    return out;
}

// MergeSorted(lists): sorted union, globally de-duplicated; nil / empty lists are skipped.
inline pb::List MergeSorted(const std::vector<const pb::List*>& lists) {
    std::vector<const uint64_t*> ptrs;
    std::vector<size_t> lens;
    size_t total = 0;
    for (const pb::List* l : lists) {
        const bool skip = (l == nullptr) || l->Uids.empty();
        ptrs.push_back(skip ? nullptr : l->Uids.data());
        lens.push_back(skip ? 0 : l->Uids.size());
        total += lens.back();
    }
    pb::List out;
    out.Uids.resize(std::max<size_t>(total, 1));
    size_t n = 0;
    check(dgx_merge_sorted(ptrs.data(), lens.data(), lists.size(), out.Uids.data(), total, &n));
    out.Uids.resize(n);
    return out;
}

// Difference(u, v): u \ v; nil u or v -> empty non-nil list (algo/uidlist.go:333-335).
inline pb::List Difference(const pb::List* u, const pb::List* v) {
    pb::List out;
    if (u == nullptr || v == nullptr) return out;
    out.Uids.resize(std::max<size_t>(u->Uids.size(), 1));
    size_t n = 0;
    check(dgx_difference(u->Uids.data(), u->Uids.size(), v->Uids.data(), v->Uids.size(), out.Uids.data(),
                         u->Uids.size(), &n));
    out.Uids.resize(n);
    return out;
}

}  // namespace algo

namespace codec {

inline size_t ApproxLen(const pb::UidPack* p) { return p ? p->base.size() * (size_t)p->block_size : 0; }
inline size_t ExactLen(const pb::UidPack* p) {
    return p ? std::accumulate(p->num_uids.begin(), p->num_uids.end(), (size_t)0) : 0;
}
// Decode(pack, seek): uids from Decoder.Seek(seek, SeekStart) onward; nil pack -> empty non-nil slice.
inline std::vector<uint64_t> Decode(const pb::UidPack* p, uint64_t seek) {
    std::vector<uint64_t> out;
    if (p == nullptr || p->base.empty()) return out;
    const size_t cap = ExactLen(p);
    out.resize(std::max<size_t>(cap, 1));
    size_t n = 0;
    const dgx_pack_view v = p->view();
    check(dgx_decode(&v, seek, out.data(), cap, &n));
    out.resize(n);
    return out;
}

// DecodeToBuffer(pack) (codec.go:456-467): binary.PutUvarint(u - last) for every uid of Decode(pack, 0), the
// subtraction on uint64; nil pack -> no bytes.  One dgx_decode_to_buffer_rows call (a uvarint is at most 10 bytes).
inline std::vector<uint8_t> DecodeToBuffer(const pb::UidPack* p) {
    std::vector<uint8_t> out;
    if (p == nullptr || p->base.empty()) return out;
    const size_t cap = 10 * ExactLen(p);
    out.resize(std::max<size_t>(cap, 1));
    const dgx_pack_view v = p->view();
    const dgx_pack_ref ref{&v, 0, 0};
    uint64_t off[2] = {0, 0};
    check(dgx_decode_to_buffer_rows(&ref, 1, out.data(), off, cap));
    out.resize(off[1]);
    return out;
}

// EncodeFromBuffer(buf, blockSize) (codec.go:402-414): the pack of the uvarint-delta stream; an empty buf is the nil
// pack (no blocks).  A buf that is not a sequence of valid uvarints (where the Go function panics or never returns)
// throws dgx::Error with DGX_ERR_ARG.  One dgx_encode_from_buffer_rows call to size, one to write.
inline pb::UidPack EncodeFromBuffer(const std::vector<uint8_t>& buf, uint32_t block_size) {
    pb::UidPack p;
    p.block_size = block_size;
    if (buf.empty()) return p;
    const uint64_t buf_off[2] = {0, buf.size()};
    uint64_t img_off[2] = {0, 0}, nb = 0, db = 0;
    check(dgx_encode_from_buffer_rows(buf.data(), buf_off, 1, block_size, nullptr, 0, img_off, &nb, &db));
    std::vector<uint64_t> img((img_off[1] + 7) / 8 + 2);  // 8-byte aligned storage; the image needs 16
    char* a = reinterpret_cast<char*>(img.data());
    a += (16 - reinterpret_cast<uintptr_t>(a) % 16) % 16;
    check(dgx_encode_from_buffer_rows(buf.data(), buf_off, 1, block_size, a, img_off[1], img_off, &nb, &db));
    dgx_pack_view v;
    check(dgx_pack_image_view(a, block_size, nb, db, &v));
    p.base.assign(v.base, v.base + nb);
    p.num_uids.assign(v.num_uids, v.num_uids + nb);
    p.delta_off.assign(v.delta_off, v.delta_off + nb + 1);
    p.deltas.assign(v.deltas, v.deltas + db);
    return p;
}

}  // namespace codec

namespace algo {

// A node of a regexp()'s trigram query tree (cindex.Query): op DGX_QAND / DGX_QOR, its trigrams as leaf indices and its
// sub-nodes (indices above its own).  A leaf is an unsplit list's pack (nullptr: empty; no pending postings) or a list
// the caller decoded.
struct QueryNode {
    uint8_t op;
    std::vector<uint32_t> leaves, subs;
};
struct TrigramLeaf {
    const pb::UidPack* pack = nullptr;
    const pb::List* list = nullptr;  // set: a list leaf
};

// uidsForRegex(attr, arg, query, &pb.List{}) (worker/trigram.go:24-102) with AfterUid = afterUID: one
// dgx_trigram_query call, pack leaves passed first as the ABI numbers them.
inline pb::List UidsForRegex(const std::vector<QueryNode>& tree, const std::vector<TrigramLeaf>& leaves,
                             uint64_t afterUID) {
    std::vector<uint32_t> order(leaves.size());
    std::vector<dgx_pack_view> views;
    std::vector<uint64_t> lists, list_off{0}, bound(leaves.size());
    uint32_t k = 0;
    for (size_t j = 0; j < leaves.size(); ++j)
        if (!leaves[j].list) {
            order[j] = k++;
            bound[j] = codec::ExactLen(leaves[j].pack);
            views.push_back(leaves[j].pack ? leaves[j].pack->view() : dgx_pack_view{});
        }
    std::vector<dgx_pack_ref> refs(views.size());
    for (size_t i = 0; i < views.size(); ++i) refs[i] = {views[i].nblocks ? &views[i] : nullptr, 0, 0};
    for (size_t j = 0; j < leaves.size(); ++j)
        if (leaves[j].list) {
            order[j] = k++;
            lists.insert(lists.end(), leaves[j].list->Uids.begin(), leaves[j].list->Uids.end());
            list_off.push_back(lists.size());
            bound[j] = leaves[j].list->Uids.size();
        }
    std::vector<uint8_t> op;
    std::vector<uint32_t> leaf_off{0}, leaf_idx, sub_off{0}, sub_idx;
    std::vector<uint64_t> nb(tree.size());  // the root's bound is the out_cap the call needs
    for (size_t i = tree.size(); i-- > 0;) {
        uint64_t b = tree[i].op == DGX_QAND ? ~0ull : 0;
        for (uint32_t j : tree[i].leaves) b = tree[i].op == DGX_QAND ? std::min(b, bound[j]) : b + bound[j];
        for (uint32_t s : tree[i].subs) b = tree[i].op == DGX_QAND ? std::min(b, nb[s]) : b + nb[s];
        nb[i] = b == ~0ull ? 0 : b;
    }
    for (const QueryNode& q : tree) {
        op.push_back(q.op);
        for (uint32_t j : q.leaves) leaf_idx.push_back(order[j]);
        leaf_off.push_back(leaf_idx.size());
        sub_idx.insert(sub_idx.end(), q.subs.begin(), q.subs.end());
        sub_off.push_back(sub_idx.size());
    }
    const dgx_query_tree t{tree.size(), op.data(), leaf_off.data(), leaf_idx.data(), sub_off.data(), sub_idx.data()};
    const std::vector<uint64_t> mut_off(refs.size() + 1, 0);
    const uint64_t cap = tree.empty() ? 0 : nb[0];
    pb::List out;
    out.Uids.resize(std::max<uint64_t>(cap, 1));
    size_t n = 0;
    check(dgx_trigram_query(&t, refs.data(), refs.size(), nullptr, nullptr, mut_off.data(), lists.data(),
                            list_off.data(), list_off.size() - 1, afterUID, out.Uids.data(), cap, &n));
    out.Uids.resize(n);
    return out;
}

// One parent row's groups of a @groupby over a uid predicate, ordered by (count, key): group g has key keys[g],
// count(uid) counts[g] and, unless counts only, the ascending source uids members[mem_off[g] .. mem_off[g+1]).
struct ParentGroups {
    std::vector<uint64_t> keys, counts, members, mem_off{0};
};

// formResult (query/groupby.go:208-221) for every parent row at once: one dgx_groupby_uid call, sized again from the
// exact counts when the first guess (the number of row values) is short.
inline std::vector<ParentGroups> GroupByUid(const std::vector<pb::List>& parents, const std::vector<uint64_t>& src,
                                            const std::vector<pb::List>& rows, const std::vector<uint64_t>& dest,
                                            bool withMembers = true) {
    if (src.size() != rows.size()) throw Error(DGX_ERR_ARG, "one source per row");
    std::vector<uint64_t> v, v_off{0}, par, par_off{0};
    for (const pb::List& r : rows) { v.insert(v.end(), r.Uids.begin(), r.Uids.end()); v_off.push_back(v.size()); }
    for (const pb::List& p : parents) { par.insert(par.end(), p.Uids.begin(), p.Uids.end()); par_off.push_back(par.size()); }
    size_t gcap = v.size(), mcap = v.size(), ng = 0, nm = 0;
    std::vector<uint64_t> keys, grp_off(parents.size() + 1), mem_off, mem;
    int rc = DGX_OK;
    for (int attempt = 0; attempt < 2; ++attempt) {
        keys.assign(std::max<size_t>(gcap, 1), 0);
        mem_off.assign(gcap + 1, 0);
        mem.assign(withMembers ? std::max<size_t>(mcap, 1) : 0, 0);
        rc = dgx_groupby_uid(src.data(), src.size(), v.data(), v_off.data(), dest.data(), dest.size(), par.data(),
                             par_off.data(), parents.size(), keys.data(), grp_off.data(), mem_off.data(), gcap,
                             withMembers ? mem.data() : nullptr, mcap, &ng, &nm);
        if (rc != DGX_ERR_CAP) break;
        gcap = ng;
        mcap = nm;
    }
    check(rc);
    std::vector<ParentGroups> out(parents.size());
    for (size_t p = 0; p < parents.size(); ++p) {
        ParentGroups& g = out[p];
        for (uint64_t i = grp_off[p]; i < grp_off[p + 1]; ++i) {
            g.keys.push_back(keys[i]);
            g.counts.push_back(mem_off[i + 1] - mem_off[i]);
            if (withMembers) g.members.insert(g.members.end(), mem.begin() + mem_off[i], mem.begin() + mem_off[i + 1]);
            g.mem_off.push_back(g.mem_off.back() + g.counts.back());
        }
    }
    return out;
}

// The edges one sg.Attr has taken during one @recurse (query/recurse.go expandRecurse's reachMap, loop: false), held
// in device memory (dgx_reach_set).  One per distinct Attr for the life of one recursion; move-only.
class ReachSet {
public:
    ReachSet() { check(dgx_reach_create(nullptr, nullptr, 0, &s_)); }
    // A set holding the edges (from[k], to[k]), strictly ascending by (from, to): a recursion continued from the host.
    ReachSet(const std::vector<uint64_t>& from, const std::vector<uint64_t>& to) {
        if (from.size() != to.size()) throw Error(DGX_ERR_ARG, "one to per from");
        check(dgx_reach_create(from.data(), to.data(), from.size(), &s_));
    }
    ReachSet(ReachSet&& o) noexcept : s_(o.s_) { o.s_ = nullptr; }
    ReachSet& operator=(ReachSet&& o) noexcept {
        std::swap(s_, o.s_);
        return *this;
    }
    ReachSet(const ReachSet&) = delete;
    ReachSet& operator=(const ReachSet&) = delete;
    ~ReachSet() { dgx_reach_destroy(s_); }

    struct Step {
        std::vector<pb::List> rows;  // the kept rows
        pb::List dest;               // sg.DestUIDs: their sorted union
        uint64_t kept = 0;           // the step's numEdges
    };
    // One sg (:105-134): rows[i] belongs to src[i]; dest is sg.DestUIDs after its filters, or nullptr without filters.
    Step Filter(const std::vector<uint64_t>& src, const std::vector<pb::List>& rows, const pb::List* dest = nullptr) {
        if (src.size() != rows.size()) throw Error(DGX_ERR_ARG, "one source per row");
        std::vector<uint64_t> v, v_off{0};
        for (const pb::List& r : rows) { v.insert(v.end(), r.Uids.begin(), r.Uids.end()); v_off.push_back(v.size()); }
        const size_t m = v.size();
        std::vector<uint64_t> out(std::max<size_t>(m, 1)), out_off(rows.size() + 1), dout(std::max<size_t>(m, 1));
        static const uint64_t none = 0;
        size_t dlen = 0;
        check(dgx_recurse_filter(s_, src.data(), src.size(), v.data(), v_off.data(),
                                 dest ? (dest->Uids.empty() ? &none : dest->Uids.data()) : nullptr,
                                 dest ? dest->Uids.size() : 0, out.data(), out_off.data(), m, dout.data(), m, &dlen));
        Step st;
        for (size_t i = 0; i < rows.size(); ++i)
            st.rows.emplace_back(std::vector<uint64_t>(out.begin() + out_off[i], out.begin() + out_off[i + 1]));
        st.dest = pb::List(std::vector<uint64_t>(dout.begin(), dout.begin() + dlen));
        st.kept = out_off[rows.size()];
        return st;
    }
    size_t Size() {
        size_t n = 0;
        check(dgx_reach_size(s_, &n));
        return n;
    }
    // (from, to) of every edge, ascending: how a recursion hands back to the host.
    std::pair<std::vector<uint64_t>, std::vector<uint64_t>> Export() {
        const size_t n = Size();
        std::vector<uint64_t> f(std::max<size_t>(n, 1)), t(std::max<size_t>(n, 1));
        size_t got = 0;
        check(dgx_reach_export(s_, f.data(), t.data(), n, &got));
        f.resize(got);
        t.resize(got);
        return {f, t};
    }
    dgx_reach_set* handle() const { return s_; }

private:
    dgx_reach_set* s_ = nullptr;
};

// The result of SubgraphFilter: the filtered and paged rows (empty in counts-only mode), their lengths and the new
// DestUIDs.
struct SgFilterResult {
    std::vector<pb::List> rows;
    std::vector<uint32_t> counts;
    pb::List dest;
};

// A subgraph's @filter tree and first / offset (query/query.go ProcessGraph's filter block, applyPagination and the
// DoCount block) in one call (dgx_sg_filter).  op / parent / leaf form the flat tree of dgx_sg_filter_tree; leaves'
// arrays are host memory with n0 counts or n0 + 1 offsets for a COUNT leaf.
inline SgFilterResult SubgraphFilter(const std::vector<uint8_t>& op, const std::vector<uint32_t>& parent,
                                     const std::vector<uint32_t>& leaf, const std::vector<dgx_sg_filter_leaf>& leaves,
                                     const pb::List& d0, const std::vector<pb::List>& rows, int32_t count = 0,
                                     int32_t offset = 0, bool counts_only = false) {
    std::vector<uint64_t> v, v_off{0};
    for (const pb::List& r : rows) { v.insert(v.end(), r.Uids.begin(), r.Uids.end()); v_off.push_back(v.size()); }
    const dgx_sg_filter_tree tree{op.size(), op.data(), parent.data(), leaf.data()};
    const size_t n0 = d0.Uids.size(), nrows = rows.size();
    std::vector<uint64_t> dest(std::max<size_t>(n0, 1)), out(std::max<size_t>(v.size(), 1)), out_off(nrows + 1);
    std::vector<uint32_t> counts(std::max<size_t>(nrows, 1));
    size_t n = 0;
    check(dgx_sg_filter(&tree, leaves.data(), leaves.size(), d0.Uids.data(), n0, v.data(), v_off.data(), nrows, count,
                        offset, dest.data(), n0, &n, counts_only ? nullptr : out.data(), out_off.data(), v.size(),
                        counts.data()));
    SgFilterResult res;
    if (!counts_only)
        for (size_t r = 0; r < nrows; ++r)
            res.rows.emplace_back(std::vector<uint64_t>(out.begin() + out_off[r], out.begin() + out_off[r + 1]));
    res.counts.assign(counts.begin(), counts.begin() + nrows);
    res.dest = pb::List(std::vector<uint64_t>(dest.begin(), dest.begin() + n));
    return res;
}

// One subgraph node of a @cascade forest, in pre-order (dgx_cascade): parent index (-1 for a query root), DGX_CASCADE_*
// flags, Params.Cascade.First / Offset, len(counts), DestUIDs, uidMatrix rows and has_val (one byte per row).
struct CascadeNode {
    int64_t parent = -1;
    uint8_t flags = 0;
    int32_t first = 0, offset = 0;
    uint64_t counts_len = 0;
    pb::List dest;
    std::vector<pb::List> rows;
    std::vector<uint8_t> has_val;
};

// @cascade over a forest (query/query.go populateVarMap :1445-1527 and ProcessQuery's root pagination :3004-3011) in
// one call: every node's rows and DestUIDs after the cascade, in node order.
inline std::pair<std::vector<std::vector<pb::List>>, std::vector<pb::List>> Cascade(const std::vector<CascadeNode>& nodes) {
    const size_t n = nodes.size();
    std::vector<uint32_t> parent(n);
    std::vector<uint8_t> flags(n), hv;
    std::vector<int32_t> first(n), offset(n);
    std::vector<uint64_t> counts(n), v, v_off{0}, row_off{0}, dest, dest_off{0}, hv_off{0};
    for (size_t k = 0; k < n; ++k) {
        const CascadeNode& c = nodes[k];
        parent[k] = c.parent < 0 ? UINT32_MAX : (uint32_t)c.parent;
        flags[k] = c.flags;
        first[k] = c.first;
        offset[k] = c.offset;
        counts[k] = c.counts_len;
        for (const pb::List& r : c.rows) { v.insert(v.end(), r.Uids.begin(), r.Uids.end()); v_off.push_back(v.size()); }
        row_off.push_back(v_off.size() - 1);
        dest.insert(dest.end(), c.dest.Uids.begin(), c.dest.Uids.end());
        dest_off.push_back(dest.size());
        hv.insert(hv.end(), c.has_val.begin(), c.has_val.end());
        hv_off.push_back(hv.size());
    }
    const dgx_cascade_tree tree{n, parent.data(), flags.data(), first.data(), offset.data(), counts.data()};
    std::vector<uint64_t> out(std::max<size_t>(v.size(), 1)), out_off(row_off.back() + 1),
        dout(std::max<size_t>(dest.size(), 1)), dout_off(n + 1);
    check(dgx_cascade(&tree, v.data(), v_off.data(), row_off.data(), dest.data(), dest_off.data(), hv.data(),
                      hv_off.data(), out.data(), out_off.data(), v.size(), dout.data(), dout_off.data(), dest.size()));
    std::pair<std::vector<std::vector<pb::List>>, std::vector<pb::List>> res;
    for (size_t k = 0; k < n; ++k) {
        std::vector<pb::List> rows;
        for (uint64_t r = row_off[k]; r < row_off[k + 1]; ++r)
            rows.emplace_back(std::vector<uint64_t>(out.begin() + out_off[r], out.begin() + out_off[r + 1]));
        res.first.push_back(std::move(rows));
        res.second.emplace_back(std::vector<uint64_t>(dout.begin() + dout_off[k], dout.begin() + dout_off[k + 1]));
    }
    return res;
}

// shortest() with numpaths <= 1 and no facets (query/shortest.go expandOut + shortestPath at unit cost): a
// breadth-first search from `from` to `to` held in device memory (dgx_path_search), one Expand per level; move-only.
class PathSearch {
public:
    PathSearch(uint64_t from, uint64_t to) { check(dgx_path_create(from, to, &ps_)); }
    PathSearch(PathSearch&& o) noexcept : ps_(o.ps_) { o.ps_ = nullptr; }
    PathSearch& operator=(PathSearch&& o) noexcept {
        std::swap(ps_, o.ps_);
        return *this;
    }
    PathSearch(const PathSearch&) = delete;
    PathSearch& operator=(const PathSearch&) = delete;
    ~PathSearch() { dgx_path_destroy(ps_); }

    // One exec sg: the child index, SrcUIDs (strictly ascending), one row per source, and DestUIDs.
    struct Sg {
        uint32_t attr = 0;
        std::vector<uint64_t> src;
        std::vector<pb::List> rows;
        pb::List dest;
    };
    struct Level {
        std::vector<pb::List> next;  // each sg's next SrcUIDs
        dgx_path_stats stats{};      // {numEdges of the level, nodes discovered, To's level or 0}
    };
    // One level over the exec sgs in exec order.
    Level Expand(const std::vector<Sg>& sgs) {
        std::vector<uint32_t> attr;
        std::vector<uint64_t> src_off{0}, src, v_off{0}, v, dest_off{0}, dest;
        for (const Sg& sg : sgs) {
            if (sg.src.size() != sg.rows.size()) throw Error(DGX_ERR_ARG, "one source per row");
            attr.push_back(sg.attr);
            src.insert(src.end(), sg.src.begin(), sg.src.end());
            src_off.push_back(src.size());
            for (const pb::List& r : sg.rows) {
                v.insert(v.end(), r.Uids.begin(), r.Uids.end());
                v_off.push_back(v.size());
            }
            dest.insert(dest.end(), sg.dest.Uids.begin(), sg.dest.Uids.end());
            dest_off.push_back(dest.size());
        }
        const dgx_path_level lv{sgs.size(), attr.data(), src_off.data(), src.data(), v_off.data(), v.data(),
                                dest_off.data(), dest.data()};
        std::vector<uint64_t> next(std::max<size_t>(dest.size(), 1)), next_off(sgs.size() + 1);
        Level out;
        check(dgx_path_expand(ps_, &lv, next.data(), next_off.data(), dest.size(), &out.stats));
        for (size_t i = 0; i < sgs.size(); ++i)
            out.next.emplace_back(std::vector<uint64_t>(next.begin() + next_off[i], next.begin() + next_off[i + 1]));
        return out;
    }
    // The path From .. To and the child index of each hop; both empty when To was not reached.
    std::pair<std::vector<uint64_t>, std::vector<uint32_t>> Path() {
        size_t n = 0;
        const int rc = dgx_path_result(ps_, nullptr, nullptr, 0, &n);
        if (rc != DGX_OK && rc != DGX_ERR_CAP) check(rc);
        std::vector<uint64_t> uids(std::max<size_t>(n, 1));
        std::vector<uint32_t> attrs(std::max<size_t>(n, 1));
        check(dgx_path_result(ps_, uids.data(), attrs.data(), n, &n));
        uids.resize(n);
        attrs.resize(n ? n - 1 : 0);
        return {uids, attrs};
    }
    dgx_path_search* handle() const { return ps_; }

private:
    dgx_path_search* ps_ = nullptr;
};

// A value variable's map (query/query.go varValue.Vals for IntID or FloatID values): strictly ascending keys and one
// 64-bit word per key, the int64 or binary64 bit pattern of type DGX_VAL_INT64 or DGX_VAL_FLOAT64.
struct ValueMap {
    int type = DGX_VAL_INT64;
    std::vector<uint64_t> keys, words;
};

// One node of a value variable's path: SrcUIDs, uidMatrix (one row per source, in stored order) and DestUIDs.
struct VarLevel {
    std::vector<uint64_t> src;
    std::vector<pb::List> rows;
    std::vector<uint64_t> dest;
};

// transformTo (query/query.go:1143-1236) over `levels` (the path from len(fromNode.path) on, index 0 skipped) in one
// dgx_var_propagate call: the map at the last level.
inline ValueMap PropagateVar(const ValueMap& m, const std::vector<VarLevel>& levels) {
    if (m.keys.size() != m.words.size()) throw Error(DGX_ERR_ARG, "one word per key");
    std::vector<std::vector<uint64_t>> v(levels.size()), v_off(levels.size());
    std::vector<dgx_var_level> lv(levels.size());
    for (size_t k = 0; k < levels.size(); ++k) {
        const VarLevel& L = levels[k];
        if (L.src.size() != L.rows.size()) throw Error(DGX_ERR_ARG, "one source per row");
        v_off[k].push_back(0);
        for (const pb::List& r : L.rows) {
            v[k].insert(v[k].end(), r.Uids.begin(), r.Uids.end());
            v_off[k].push_back(v[k].size());
        }
        lv[k] = dgx_var_level{L.src.data(), v_off[k].data(), v[k].data(), L.dest.data(), L.src.size(), 0,
                              L.dest.size()};
    }
    const size_t cap = levels.empty() ? 0 : levels.back().dest.size();
    ValueMap out;
    out.type = m.type;
    out.keys.assign(std::max<size_t>(cap, 1), 0);
    out.words.assign(std::max<size_t>(cap, 1), 0);
    size_t n = 0;
    check(dgx_var_propagate(m.type, m.keys.data(), m.words.data(), m.keys.size(), lv.data(), lv.size(),
                            out.keys.data(), out.words.data(), cap, &n));
    out.keys.resize(n);
    out.words.resize(n);
    return out;
}

// evalLevelAgg's per-row branch (query/query.go:1088-1123) in one dgx_var_level_agg call: fn (DGX_AGG_*) of the map
// over every row of relSG's uidMatrix, keyed by src; DGX_VAL_FLOAT64 for DGX_AGG_AVG, the map's type otherwise.
inline ValueMap LevelAgg(int fn, const ValueMap& m, const std::vector<uint64_t>& src,
                         const std::vector<pb::List>& rows) {
    if (m.keys.size() != m.words.size()) throw Error(DGX_ERR_ARG, "one word per key");
    if (src.size() != rows.size()) throw Error(DGX_ERR_ARG, "one source per row");
    std::vector<uint64_t> v, v_off{0};
    for (const pb::List& r : rows) { v.insert(v.end(), r.Uids.begin(), r.Uids.end()); v_off.push_back(v.size()); }
    ValueMap out;
    out.type = fn == DGX_AGG_AVG ? DGX_VAL_FLOAT64 : m.type;
    out.keys.assign(std::max<size_t>(rows.size(), 1), 0);
    out.words.assign(std::max<size_t>(rows.size(), 1), 0);
    size_t n = 0;
    check(dgx_var_level_agg(m.type, fn, m.keys.data(), m.words.data(), m.keys.size(), src.data(), src.size(),
                            v_off.data(), v.data(), out.keys.data(), out.words.data(), rows.size(), &n));
    out.keys.resize(n);
    out.words.resize(n);
    return out;
}

// A math() leaf or result: strictly ascending keys, one 64-bit word and one DGX_VAL_* tag per key.  nil is a variable
// with no map at all (Go's nil ShardedMap), which cond tells apart from an empty one.
struct MathMap {
    std::vector<uint64_t> keys, words;
    std::vector<uint8_t> tags;
    bool nil = false;
};

// The result of EvalMath: kind DGX_MATH_KIND_MAP (the map), DGX_MATH_KIND_CONST (the constant set on every uid of the
// range, or on uid 0 without one) or DGX_MATH_KIND_NONE (Go assigns nothing).
struct MathResult {
    int kind = DGX_MATH_KIND_NONE;
    MathMap map;
};

// evalMathTree (query/math.go) and valueVarAggregation's math branch (query/query.go:1290-1361) in one dgx_math_eval
// call: prog in post-order, leaves indexed by its VAR nodes, range SrcUIDs (DestUIDs at the root) or null.
inline MathResult EvalMath(const std::vector<dgx_math_node>& prog, const std::vector<MathMap>& leaves,
                           const std::vector<uint64_t>* range) {
    std::vector<dgx_math_leaf> lv(leaves.size());
    size_t cap = 1;
    for (size_t j = 0; j < leaves.size(); ++j) {
        const MathMap& m = leaves[j];
        if (m.keys.size() != m.words.size() || m.keys.size() != m.tags.size())
            throw Error(DGX_ERR_ARG, "one word and one tag per key");
        const size_t n = m.nil ? 0 : m.keys.size();
        lv[j] = dgx_math_leaf{m.keys.data(), m.words.data(), m.tags.data(), nullptr, n, DGX_VAL_INT64, m.nil ? 1 : 0};
        cap += n;
    }
    const size_t nr = range ? range->size() : 0;
    cap = std::max(cap, nr);
    MathResult out;
    out.map.keys.assign(cap, 0);
    out.map.words.assign(cap, 0);
    out.map.tags.assign(cap, 0);
    uint64_t info = 0;
    static const uint64_t kNoUid = 0;
    check(dgx_math_eval(prog.data(), prog.size(), lv.data(), lv.size(),
                        range ? (nr ? range->data() : &kNoUid) : nullptr, nr, out.map.keys.data(),
                        out.map.words.data(), out.map.tags.data(), cap, &info));
    const size_t n = DGX_MATH_INFO_LEN(info);
    out.kind = DGX_MATH_INFO_KIND(info);
    out.map.keys.resize(n);
    out.map.words.resize(n);
    out.map.tags.resize(n);
    return out;
}

// The result of OrderByVar: the ordered and paged rows and the new DestUIDs.
struct OrderResult {
    std::vector<pb::List> rows;
    pb::List dest;
};

namespace detail {
inline OrderResult order_by_var(const dgx_math_leaf& leaf, bool desc, const pb::List& dest,
                                const std::vector<pb::List>& rows, int32_t count, int32_t offset) {
    std::vector<uint64_t> v, v_off{0};
    for (const pb::List& r : rows) { v.insert(v.end(), r.Uids.begin(), r.Uids.end()); v_off.push_back(v.size()); }
    const size_t nd = dest.Uids.size(), nrows = rows.size();
    std::vector<uint64_t> out(std::max<size_t>(v.size(), 1)), out_off(nrows + 1), dout(std::max<size_t>(nd, 1));
    size_t n = 0;
    check(dgx_var_order(&leaf, desc ? 1 : 0, dest.Uids.data(), nd, v.data(), v_off.data(), nrows, count, offset,
                        out.data(), out_off.data(), v.size(), dout.data(), nd, &n));
    OrderResult res;
    for (size_t r = 0; r < nrows; ++r)
        res.rows.emplace_back(std::vector<uint64_t>(out.begin() + out_off[r], out.begin() + out_off[r + 1]));
    res.dest = pb::List(std::vector<uint64_t>(dout.begin(), dout.begin() + n));
    return res;
}
}  // namespace detail

// orderasc / orderdesc by a value variable (query/query.go applyOrderAndPagination's value-variable branch:
// updateUidMatrix, sortAndPaginateUsingVar with types.Sort and x.PageRange, updateDestUids) in one dgx_var_order call,
// in Go's exact order, ties included.  dest: the node's DestUIDs after its filters; rows: its uidMatrix; count /
// offset: Params.Count / Offset.  A PropagateVar / LevelAgg map, or a math() map (MathMap; nil is Go's nil map, which
// the call refuses with DGX_ERR_ARG as Go returns an error).
inline OrderResult OrderByVar(const ValueMap& m, bool desc, const pb::List& dest, const std::vector<pb::List>& rows,
                              int32_t count = 0, int32_t offset = 0) {
    if (m.keys.size() != m.words.size()) throw Error(DGX_ERR_ARG, "one word per key");
    const dgx_math_leaf leaf{m.keys.data(), m.words.data(), nullptr, nullptr, m.keys.size(), m.type, 0};
    return detail::order_by_var(leaf, desc, dest, rows, count, offset);
}
inline OrderResult OrderByVar(const MathMap& m, bool desc, const pb::List& dest, const std::vector<pb::List>& rows,
                              int32_t count = 0, int32_t offset = 0) {
    if (m.keys.size() != m.words.size() || m.keys.size() != m.tags.size())
        throw Error(DGX_ERR_ARG, "one word and one tag per key");
    const dgx_math_leaf leaf{m.keys.data(), m.words.data(), m.tags.data(), nullptr, m.nil ? 0 : m.keys.size(),
                             DGX_VAL_INT64, m.nil ? 1 : 0};
    return detail::order_by_var(leaf, desc, dest, rows, count, offset);
}

// A predicate's string values for MatchFuzzy: uids strictly ascending, vals[i] the values of uids[i] as Go's match
// loop reads them (Value, ValueForTag or AllUntaggedValues); a uid without a value is left out.
struct StrColumn {
    std::vector<uint64_t> uids;
    std::vector<std::vector<std::string>> vals;
};

namespace detail {
// A StrColumn as the flat arrays of dgx_str_column; `c` points into this object, so it is neither copied nor moved.
struct StrColumnCsr {
    std::vector<uint64_t> val_off{0}, byte_off{0};
    std::string data;
    dgx_str_column c{};
    explicit StrColumnCsr(const StrColumn& col) {
        if (col.uids.size() != col.vals.size()) throw Error(DGX_ERR_ARG, "one list of values per uid");
        for (const auto& vs : col.vals) {
            for (const std::string& v : vs) { data += v; byte_off.push_back(data.size()); }
            val_off.push_back(byte_off.size() - 1);
        }
        c = dgx_str_column{col.uids.data(), val_off.data(), byte_off.data(), (const uint8_t*)data.data(),
                           col.uids.size(), byte_off.size() - 1, data.size()};
    }
    StrColumnCsr(const StrColumnCsr&) = delete;
    StrColumnCsr& operator=(const StrColumnCsr&) = delete;
};
// The candidates as dgx_match / dgx_regex_match take them: uids when not empty, otherwise rows as list leaves.
struct Candidates {
    std::vector<uint64_t> lists, list_off{0};
    size_t bound;
    Candidates(const pb::List& uids, const std::vector<pb::List>& rows) {
        if (uids.Uids.empty())
            for (const pb::List& r : rows) { lists.insert(lists.end(), r.Uids.begin(), r.Uids.end()); list_off.push_back(lists.size()); }
        bound = uids.Uids.empty() ? lists.size() : uids.Uids.size();
    }
};
}  // namespace detail

// match(attr, query, max) (worker/task.go handleMatchFunction, worker/match.go uidsForMatch / matchFuzzy) in one
// dgx_match call: the candidates are uids when it is not empty (the filter's UidList), otherwise the union of rows,
// the query's trigram rows as pl.Uids read them; a candidate is kept when one of its values is within max edits of
// the query over Go's []rune conversion.  Returns the kept candidates.
inline pb::List MatchFuzzy(const StrColumn& col, const std::string& query, int64_t max, const pb::List& uids,
                           const std::vector<pb::List>& rows = {}) {
    const detail::StrColumnCsr c(col);
    const detail::Candidates k(uids, rows);
    std::vector<uint64_t> out(std::max<size_t>(k.bound, 1));
    size_t n = 0;
    check(dgx_match(nullptr, 0, nullptr, nullptr, nullptr, k.lists.data(), k.list_off.data(), k.list_off.size() - 1, 0,
                    uids.Uids.data(), uids.Uids.size(), &c.c, (const uint8_t*)query.data(), query.size(), max,
                    out.data(), k.bound, &n));
    out.resize(n);
    return pb::List(out);
}

// A predicate's values converted to one type for CompareUids / CompareRows (dgx_val_column): type is DGX_VAL_INT64,
// DGX_VAL_FLOAT64 (IEEE bits), DGX_VAL_BOOL, DGX_VAL_DATETIME (Unix seconds in words, nanoseconds in nsec) or
// DGX_VAL_STRING (strs); uids strictly ascending, the values of uids[i] at index i; bad, when not empty, flags the
// values whose conversion failed or gave nil.
struct ValColumn {
    int type = DGX_VAL_INT64;
    std::vector<uint64_t> uids;
    std::vector<std::vector<uint64_t>> words;
    std::vector<std::vector<uint32_t>> nsec;
    std::vector<std::vector<std::string>> strs;
    std::vector<std::vector<uint8_t>> bad;
};
// A compare function's arguments of the column's type: words (and nsec) or strs.
struct ValArgs {
    std::vector<uint64_t> words;
    std::vector<uint32_t> nsec;
    std::vector<std::string> strs;
};

namespace detail {
// A ValColumn and its arguments as dgx_val_column / dgx_val_args; the structs point into this object.
struct ValCall {
    std::vector<uint64_t> val_off{0}, word, arg_off{0};
    std::vector<uint32_t> nsec;
    std::vector<uint8_t> bad;
    std::string arg_bytes;
    StrColumn sc;
    std::unique_ptr<StrColumnCsr> str;
    dgx_val_column c{};
    dgx_val_args a{};
    ValCall(const ValColumn& col, const ValArgs& args) {
        const bool is_str = col.type == DGX_VAL_STRING;
        const size_t n = col.uids.size();
        if ((is_str ? col.strs.size() : col.words.size()) != n) throw Error(DGX_ERR_ARG, "one list of values per uid");
        for (size_t i = 0; i < n; ++i) {
            const size_t k = is_str ? col.strs[i].size() : col.words[i].size();
            if (!is_str) word.insert(word.end(), col.words[i].begin(), col.words[i].end());
            if (col.type == DGX_VAL_DATETIME) nsec.insert(nsec.end(), col.nsec[i].begin(), col.nsec[i].end());
            if (!col.bad.empty()) bad.insert(bad.end(), col.bad[i].begin(), col.bad[i].end());
            val_off.push_back(val_off.back() + k);
        }
        if (is_str) {
            sc = StrColumn{col.uids, col.strs};
            str.reset(new StrColumnCsr(sc));
        }
        c = dgx_val_column{col.type, col.uids.data(), val_off.data(), word.data(), nsec.data(),
                           col.bad.empty() ? nullptr : bad.data(), is_str ? &str->c : nullptr, n, val_off.back()};
        for (const std::string& s : args.strs) { arg_bytes += s; arg_off.push_back(arg_bytes.size()); }
        a = dgx_val_args{args.words.data(), args.nsec.data(), (const uint8_t*)arg_bytes.data(), arg_off.data(),
                         is_str ? args.strs.size() : args.words.size()};
    }
    ValCall(const ValCall&) = delete;
    ValCall& operator=(const ValCall&) = delete;
};
}  // namespace detail

// eq / le / lt / ge / gt / between (op DGX_SGF_CMP_*) over the filter's UidList (worker/task.go handleValuePostings,
// compareAttrFn branch) in one dgx_compare_uids call: the candidates with a value passing types.CompareVals, and in
// *counts, when given, Go's row lengths.  A candidate's bad value throws Error(DGX_ERR_ARG), Go's conversion error.
inline pb::List CompareUids(const ValColumn& col, int op, const ValArgs& args, const pb::List& uids,
                            std::vector<uint32_t>* counts = nullptr) {
    const detail::ValCall v(col, args);
    std::vector<uint64_t> out(std::max<size_t>(uids.Uids.size(), 1));
    std::vector<uint32_t> cnt(std::max<size_t>(uids.Uids.size(), 1));
    size_t n = 0;
    check(dgx_compare_uids(op, &v.a, &v.c, uids.Uids.data(), uids.Uids.size(), out.data(), uids.Uids.size(), &n,
                           counts ? cnt.data() : nullptr));
    out.resize(n);
    if (counts) { cnt.resize(uids.Uids.size()); *counts = cnt; }
    return pb::List(out);
}

// handleCompareFunction's filterRow over the index rows (worker/task.go :1395-1520) in one dgx_compare_rows call:
// row r unchanged when row_arg[r] is UINT32_MAX, otherwise filtered by value against argument row_arg[r].
inline std::vector<pb::List> CompareRows(const ValColumn& col, int op, const ValArgs& args,
                                         const std::vector<pb::List>& rows, const std::vector<uint32_t>& row_arg) {
    const detail::ValCall v(col, args);
    if (row_arg.size() != rows.size()) throw Error(DGX_ERR_ARG, "one row_arg per row");
    std::vector<uint64_t> flat, off{0};
    for (const pb::List& r : rows) { flat.insert(flat.end(), r.Uids.begin(), r.Uids.end()); off.push_back(flat.size()); }
    std::vector<uint64_t> out(std::max<size_t>(flat.size(), 1)), out_off(rows.size() + 1);
    check(dgx_compare_rows(op, &v.a, &v.c, flat.data(), off.data(), rows.size(), row_arg.data(), out.data(),
                           out_off.data(), flat.size()));
    std::vector<pb::List> res;
    for (size_t r = 0; r < rows.size(); ++r)
        res.push_back(pb::List(std::vector<uint64_t>(out.begin() + out_off[r], out.begin() + out_off[r + 1])));
    return res;
}

// orderasc / orderdesc by a predicate with no sortable index (query/query.go applyOrderAndPagination's predicate
// branch with worker/sort.go sortWithoutIndex) in one dgx_pred_order call, in Go's exact order, ties included: each
// row's dest uids with a value sorted by it, then those without one (absent, or bad) in row order, cut by
// x.PageRange(count, offset, |row|).  col: DGX_VAL_INT64, DGX_VAL_FLOAT64, DGX_VAL_DATETIME or DGX_VAL_STRING, one
// value per uid.  A bool column, a negative count or a list value throws Error(DGX_ERR_ARG), where Go errs.
inline OrderResult OrderByPred(const ValColumn& col, bool desc, const pb::List& dest, const std::vector<pb::List>& rows,
                               int32_t count = 0, int32_t offset = 0) {
    const detail::ValCall c(col, ValArgs{});
    std::vector<uint64_t> v, v_off{0};
    for (const pb::List& r : rows) { v.insert(v.end(), r.Uids.begin(), r.Uids.end()); v_off.push_back(v.size()); }
    const size_t nd = dest.Uids.size(), nrows = rows.size();
    std::vector<uint64_t> out(std::max<size_t>(v.size(), 1)), out_off(nrows + 1), dout(std::max<size_t>(nd, 1));
    size_t n = 0;
    check(dgx_pred_order(&c.c, desc ? 1 : 0, dest.Uids.data(), nd, v.data(), v_off.data(), nrows, count, offset,
                         out.data(), out_off.data(), v.size(), dout.data(), nd, &n));
    OrderResult res;
    for (size_t r = 0; r < nrows; ++r)
        res.rows.emplace_back(std::vector<uint64_t>(out.begin() + out_off[r], out.begin() + out_off[r + 1]));
    res.dest = pb::List(std::vector<uint64_t>(dout.begin(), dout.begin() + n));
    return res;
}

// A regexp() pattern compiled once (dgx_regex_compile; fold is the /i modifier).  Throws Error with DGX_ERR_ARG for a
// pattern outside the compiled subset or one Go rejects, DGX_ERR_CAP past DGX_REGEX_MAX_STATES: keep Go's matcher then.
class RegexProg {
  public:
    explicit RegexProg(const std::string& pattern, bool fold = false) {
        check(dgx_regex_compile(pattern.data(), pattern.size(), fold ? DGX_REGEX_FOLD : 0, &p_));
    }
    ~RegexProg() { dgx_regex_free(p_); }
    RegexProg(const RegexProg&) = delete;
    RegexProg& operator=(const RegexProg&) = delete;
    const dgx_regex_prog* get() const { return p_; }

  private:
    dgx_regex_prog* p_ = nullptr;
};

// regexp(attr, /pattern/) (worker/task.go handleRegexFunction, matchRegex) in one dgx_regex_match call: the
// candidates as MatchFuzzy takes them, kept when one of their values matches prog.  Returns the kept candidates.
inline pb::List MatchRegex(const StrColumn& col, const RegexProg& prog, const pb::List& uids,
                           const std::vector<pb::List>& rows = {}) {
    const detail::StrColumnCsr c(col);
    const detail::Candidates k(uids, rows);
    std::vector<uint64_t> out(std::max<size_t>(k.bound, 1));
    size_t n = 0;
    check(dgx_regex_match(nullptr, 0, nullptr, nullptr, nullptr, k.lists.data(), k.list_off.data(),
                          k.list_off.size() - 1, 0, uids.Uids.data(), uids.Uids.size(), &c.c, prog.get(), out.data(),
                          k.bound, &n));
    out.resize(n);
    return pb::List(out);
}

}  // namespace algo

// Wire-format adjacency (dgx_wire_*, host only): the bytes proto.Unmarshal sees at posting/list.go:1045 and
// the pb.List messages of pb.Result.uid_matrix (protos/pb.proto:22-24, 76-78).
namespace wire {

// Serialized pb.UidPack -> the struct-of-arrays pb::UidPack.
inline pb::UidPack ParseUidPack(const uint8_t* buf, size_t len) {
    size_t nb = 0, db = 0;
    check(dgx_wire_pack_measure(buf, len, &nb, &db));
    pb::UidPack p;
    p.base.resize(nb);
    p.num_uids.resize(nb);
    p.delta_off.assign(nb + 1, 0);
    p.deltas.resize(db);
    dgx_pack_view v;
    check(dgx_wire_pack_parse(buf, len, p.base.data(), p.num_uids.data(), p.delta_off.data(), p.deltas.data(), nb, db, &v));
    p.block_size = v.block_size;
    return p;
}

// Serialized pb.PostingList -> its pb.UidPack; `found` is false when the posting list has no pack (nil).
inline pb::UidPack PostingListPack(const uint8_t* buf, size_t len, bool* found) {
    const uint8_t* sub = nullptr;
    size_t sub_len = 0;
    check(dgx_wire_posting_list_pack(buf, len, &sub, &sub_len));
    if (found) *found = sub != nullptr;
    return sub ? ParseUidPack(sub, sub_len) : pb::UidPack();
}

// pb.List -> its serialized message (header followed by the little-endian uids).
inline std::vector<uint8_t> ListToWire(const pb::List& l) {
    uint8_t hdr[16];
    const size_t h = dgx_wire_list_header(l.Uids.size(), hdr);
    std::vector<uint8_t> out(h + l.Uids.size() * 8);
    std::copy(hdr, hdr + h, out.begin());
    if (!l.Uids.empty()) std::copy((const uint8_t*)l.Uids.data(), (const uint8_t*)l.Uids.data() + l.Uids.size() * 8, out.begin() + h);
    return out;
}

inline pb::List ListFromWire(const uint8_t* buf, size_t len) {
    size_t n = 0;
    check(dgx_wire_list_decode(buf, len, nullptr, 0, &n));
    pb::List l;
    l.Uids.resize(n);
    if (n) check(dgx_wire_list_decode(buf, len, l.Uids.data(), n, &n));
    return l;
}

}  // namespace wire
}  // namespace dgx
