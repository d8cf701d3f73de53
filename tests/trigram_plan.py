"""The host plan of dgx_trigram_query (dgx_api.cu tg_plan / trigram_impl) restated in Python: the checks, the bounds,
the driving leaves, the all-OR skip, the capacities and the launch count of one call.  Its constants are read from the
CUDA sources and the statements it restates are matched as text, so a rewrite fails loudly here instead of drifting.
"""
from __future__ import annotations

import os
import re
from collections import namedtuple

from merge_geometry import tree_launches
from merge_matrix_geometry import K as XM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
QAND, QOR = 2, 3
OK, ERR_ARG, ERR_CAP = 0, -3, -4


def _src(fn):
    with open(os.path.join(CSRC, fn)) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the trigram plan model (tests/trigram_plan.py)")
    return m


def read_constants() -> dict:
    api, tk = _src("dgx_api.cu"), _src("trigram_kernel.cuh")
    m = _one(r"constexpr size_t kTgMaxNodes = size_t\(1\) << (\d+), kTgMaxLeaves = size_t\(1\) << (\d+), "
             r"kTgMaxRefs = size_t\(1\) << (\d+);", api, "the tree limits")
    K = {"MAX_NODES": 1 << int(m.group(1)), "MAX_LEAVES": 1 << int(m.group(2)), "MAX_REFS": 1 << int(m.group(3))}
    K["MAX_DEPTH"] = int(_one(r"constexpr uint32_t kTgMaxDepth = (\d+);", api, "kTgMaxDepth").group(1))
    K["TG_NT"] = int(_one(r"constexpr int TG_NT = (\d+);", tk, "TG_NT").group(1))
    # the launches of each stage
    K["ROWS"] = int(_one(r"launches = (\d+);\s*\}\s*l->launches \+= launches;", api,
                         "list_unfiltered_impl's launches").group(1))
    body = _one(r"(?s)static int trigram_impl\(.*?\n\}\n", api, "trigram_impl").group(0)
    counts = [int(x) for x in re.findall(r"count_launches\(l, (\d+)\);", body)]
    if counts != [2, 2] or body.count("<<<") != 4:
        raise ValueError("trigram_impl's launches changed: restate them in the trigram plan model")
    _one(r"const bool merge = nd >= 2;", body, "the merge condition")
    _one(r"if \(!T\.all_or\) \{", body, "the all-OR skip")
    _one(r"std::stable_sort\(ch\.begin\(\), ch\.end\(\), \[\]\(const auto& a, const auto& b\) \{ return a\.first < "
         r"b\.first; \}\);", api, "the AND children's order")
    _one(r"const size_t n = t->op\[i\] == DGX_QAND \? 1 : ch\.size\(\);", api, "the driving children")
    K["MERGE"] = XM["LAUNCHES"]
    K["XM_T"] = XM["XM_T"]
    return K


K = read_constants()

Plan = namedtuple("Plan", "rc bound root_bound drive dcap all_or launches merge")


def _check(tree, nleaves):
    nn = len(tree)
    if nn == 0 or nn >= K["MAX_NODES"] or nleaves >= K["MAX_LEAVES"]:
        return "size"
    if sum(len(t[1]) for t in tree) >= K["MAX_REFS"]:
        return "refs"
    parent, depth = [None] * nn, [1] * nn
    for i, (op, ls, subs) in enumerate(tree):
        if op not in (QAND, QOR):
            return "op"
        if op == QAND and not ls and not subs:
            return "empty AND"
        if i > 0 and parent[i] is None:
            return "no parent"
        if any(j < 0 or j >= nleaves for j in ls):
            return "leaf index"
        for s in subs:
            if s <= i or s >= nn:
                return "sub index"
            if parent[s] is not None:
                return "two parents"
            parent[s], depth[s] = i, depth[i] + 1
            if depth[s] > K["MAX_DEPTH"]:
                return "depth"
    return None


def plan(tree, leaf_bounds, out_cap=None) -> Plan:
    """One call's plan: rc (OK, ERR_ARG for a tree the library refuses, ERR_CAP for out_cap below the root's bound),
    every node's bound, the root's distinct driving leaves and their bound sum, the all-OR skip and the launches."""
    nleaves = len(leaf_bounds)
    if _check(tree, nleaves) or sum(leaf_bounds) >= 1 << 32:
        return Plan(ERR_ARG, None, None, None, None, None, 0, False)
    nn = len(tree)
    bound = [0] * nn

    def children(i):
        op, ls, subs = tree[i]
        ch = [(leaf_bounds[j], ("leaf", j)) for j in ls] + [(bound[s], ("node", s)) for s in subs]
        return sorted(ch, key=lambda c: c[0]) if op == QAND else ch  # Python's sort is stable

    for i in reversed(range(nn)):
        ch = [c[0] for c in children(i)]
        bound[i] = min(ch) if tree[i][0] == QAND else sum(ch)
    all_or = all(t[0] == QOR for t in tree)
    root = bound[0]
    if out_cap is not None and out_cap < root:
        return Plan(ERR_CAP, bound, root, None, None, all_or, 0, False)
    if root == 0:
        return Plan(OK, bound, 0, [], 0, all_or, 0, False)
    drive: list = []

    def walk(i):
        ch = children(i)
        for _, (kind, j) in (ch[:1] if tree[i][0] == QAND else ch):
            if kind == "node":
                walk(j)
            elif j not in drive:
                drive.append(j)

    walk(0)
    dcap = sum(leaf_bounds[j] for j in drive)
    return Plan(OK, bound, root, drive, dcap, all_or, None, len(drive) >= 2)


def launches(p: Plan, npacks: int) -> int:
    """Kernel launches of the call: the unfiltered rows' when there are pack leaves, the leaves and gather kernels, the
    matrix merge's (its sample tree has ceil(log2 ntiles) levels) when two or more leaves drive, evaluation and
    compaction unless every node is an OR.  Nothing runs for a root bound of 0."""
    if p.rc != OK or p.root_bound == 0:
        return 0
    n = (K["ROWS"] if npacks else 0) + 2
    if p.merge:
        n += K["MERGE"] + tree_launches(-(-p.dcap // K["XM_T"]))
    if not p.all_or:
        n += 2
    return n
