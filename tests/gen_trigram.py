"""Seeded trigram queries for dgx_trigram_query (tests/test_trigram_host.py, tests/test_gpu_trigram_query.py,
tools/bench_ops.py C12): random query trees over pack and list leaves with mutable layers, hand-written trees of a few
regexp patterns, a synthetic trigram index, and the set formula of the tree in numpy -- a second opinion on the
line-by-line restatement of uidsForRegex (trigram_oracle.c).

A raw leaf is ("pack", uids or None, (mut_uids, mut_flags) or None, approx_len) or ("list", uids); to_oracle / to_algo
turn raw leaves into the leaves trigram_oracle.py and algo.UidsForRegex take.
"""
from __future__ import annotations

import numpy as np

from gen_mut import MUT_DEL, layer

QAND, QOR = 2, 3
U64 = (1 << 64) - 1
MAX_DEPTH = 32


# ---- the set formula -------------------------------------------------------------------------------------------------

def leaf_set(leaf, after: int) -> np.ndarray:
    """S_leaf: the unfiltered List.Uids row of a pack leaf, {x > after : mut(x) exists ? mut(x) has no flag : x in
    pack}; a list leaf is its list."""
    if leaf[0] == "list":
        return np.asarray(leaf[1], np.uint64)
    pk = np.zeros(0, np.uint64) if leaf[1] is None else np.asarray(leaf[1], np.uint64)
    mu, mf = (np.zeros(0, np.uint64), np.zeros(0, np.uint8)) if leaf[2] is None else leaf[2]
    s = np.union1d(pk[~np.isin(pk, mu)], mu[mf == 0]).astype(np.uint64)
    return s[s > np.uint64(after)]


def want(tree, leaves, after: int) -> np.ndarray:
    """f(root) with f(leaf) = S_leaf, f(AND) = the intersection of its children, f(OR) = their union."""
    sets = [leaf_set(lf, after) for lf in leaves]
    val = [None] * len(tree)
    for i in reversed(range(len(tree))):
        op, ls, subs = tree[i]
        ch = [sets[j] for j in ls] + [val[s] for s in subs]
        if op == QAND:
            r = ch[0]
            for c in ch[1:]:
                r = np.intersect1d(r, c, assume_unique=True)
        else:
            r = np.unique(np.concatenate(ch)) if ch else np.zeros(0, np.uint64)
        val[i] = r.astype(np.uint64)
    return val[0]


def leaf_bound(leaf) -> int:
    if leaf[0] == "list":
        return len(leaf[1])
    return (0 if leaf[1] is None else len(leaf[1])) + (0 if leaf[2] is None else len(leaf[2][0]))


# ---- conversions -------------------------------------------------------------------------------------------------

def to_oracle(leaves):
    from oracle import pyoracle as orc

    out = []
    for lf in leaves:
        if lf[0] == "list":
            out.append(np.asarray(lf[1], np.uint64))
        else:
            p = orc.encode(np.asarray(lf[1], np.uint64), 256) if lf[1] is not None and len(lf[1]) else None
            out.append((p, lf[2], lf[3]))
    return out


def to_algo(leaves, block_size: int = 256):
    from dgraph_b200 import pb
    from oracle import pyoracle as orc

    out = []
    for lf in leaves:
        if lf[0] == "list":
            out.append(np.asarray(lf[1], np.uint64))
        elif lf[1] is None or not len(lf[1]):
            out.append((None, lf[2]))
        else:
            o = orc.encode(np.asarray(lf[1], np.uint64), block_size)
            out.append((pb.UidPack(o.block_size, o.base, o.num_uids, o.delta_off, o.deltas), lf[2]))
    return out


# ---- random trees ------------------------------------------------------------------------------------------------

def random_tree(rng, nleaves: int, nnodes: int, p_and: float = 0.5, max_depth: int = MAX_DEPTH):
    """nnodes nodes, every node's parent drawn among the earlier ones (depth at most max_depth), every node given a few
    leaves (shared leaves allowed); an AND with no child gets a leaf, an OR may stay empty."""
    parent, depth = [-1], [1]
    for i in range(1, nnodes):
        cands = [j for j in range(i) if depth[j] < max_depth]
        p = int(rng.choice(cands))
        parent.append(p)
        depth.append(depth[p] + 1)
    ops = [QAND if rng.random() < p_and else QOR for _ in range(nnodes)]
    tree = []
    for i in range(nnodes):
        subs = [j for j in range(i + 1, nnodes) if parent[j] == i]
        k = int(rng.integers(0, 4))
        ls = [int(x) for x in rng.integers(0, nleaves, k)] if nleaves else []
        if ops[i] == QAND and not ls and not subs:
            ls = [int(rng.integers(0, nleaves))]
        tree.append((ops[i], ls, subs))
    return tree


def random_leaves(rng, nleaves: int, universe: int, branch: str = "mixed", p_list: float = 0.2, after: int = 0):
    """Leaves over uids 1 .. universe: packs of random density with layers of REF postings (SET and DEL only), lists.
    branch: where every filtered read of a pack leaf lands -- "compressed" (no layer), "probe" (ApproxLen above every
    filter), "iterate" (ApproxLen 0) or "mixed".  List leaves lie above after, as a pl.Uids read returns them."""
    leaves = []
    for _ in range(nleaves):
        dens = float(rng.choice([0.0, 0.02, 0.1, 0.3, 0.7]))
        uids = np.flatnonzero(rng.random(universe) < dens).astype(np.uint64) + np.uint64(1)
        if rng.random() < p_list:
            leaves.append(("list", uids[uids > np.uint64(after)]))
            continue
        b = branch if branch != "mixed" else str(rng.choice(["compressed", "probe", "iterate"]))
        pk = None if (uids.size == 0 or rng.random() < 0.05) else uids
        mut = None
        if b != "compressed":
            pool = np.arange(1, universe + 1, dtype=np.uint64)
            mut = layer(rng, uids if uids.size else pool, pool, int(rng.integers(1, 12)), p_flags=(0.55, 0.45, 0.0, 0.0))
            if pk is None and rng.random() < 0.5:
                mut = (mut[0], np.full(mut[0].size, MUT_DEL, np.uint8))
        approx = {"compressed": 0, "probe": 1 << 40, "iterate": 0}[b]
        if pk is None and mut is None and b != "compressed":
            mut = (np.array([1], np.uint64), np.array([MUT_DEL], np.uint8))
        leaves.append(("pack", pk, mut, approx))
    return leaves


# ---- hand-written trees of regexp patterns ------------------------------------------------------------------------
# No Go toolchain is available to run codesearch's RegexpQuery, so these trees are written by hand from its rules: a
# literal is the AND of its trigrams, an alternation the OR of its branches, `.*` splits a pattern into ANDed parts, a
# small character class or a group expands into the OR of the exact strings, and a common prefix is factored out as an
# AND over an OR sub-node.  Each is a list of nodes (op, trigrams, subs).

def _and(*tris):
    return (QAND, list(tris), [])


PATTERNS = {
    "abcd": [_and("abc", "bcd")],
    "abc|def": [(QOR, ["abc", "def"], [])],
    "abc.*def": [_and("abc", "def")],
    "ab[cd]e": [(QOR, [], [1, 2]), _and("abc", "bce"), _and("abd", "bde")],
    "(abc|xyz)def": [(QOR, [], [1, 2]), _and("abc", "bcd", "cde", "def"), _and("xyz", "yzd", "zde", "def")],
    "abc(de|fg)h": [(QAND, ["abc"], [1]), (QOR, [], [2, 3]), _and("bcd", "cde", "deh"), _and("bcf", "cfg", "fgh")],
    "(ab|cd)(ef|gh)": [(QOR, [], [1, 2, 3, 4]), _and("abe", "bef"), _and("abg", "bgh"), _and("cde", "def"),
                       _and("cdg", "dgh")],
    "abc[0-9]+": [_and("abc")],
    "abc.*xyz|def": [(QOR, ["def"], [1]), _and("abc", "xyz")],
    "qu[aeiou]ck": [(QOR, [], [1, 2, 3, 4, 5])] + [_and(f"qu{v}", f"u{v}c", f"{v}ck") for v in "aeiou"],
}

# words the small index always holds, so that every pattern above matches some value and misses others
SEED_WORDS = ["abcdef", "xyzdef", "abcdeh", "abcfgh", "abce", "abde", "abef", "cdgh", "quack", "quick", "abc123",
              "abcxyz", "defy", "bcde", "qck", "uacu", "abcd"]


def tree_of_pattern(nodes):
    """(tree over leaf indices, the trigrams naming the leaves): every distinct trigram becomes one leaf."""
    tris: list = []
    tree = []
    for op, ts, subs in nodes:
        idx = []
        for t in ts:
            if t not in tris:
                tris.append(t)
            idx.append(tris.index(t))
        tree.append((op, idx, list(subs)))
    return tree, tris


def trigrams(word: str):
    return {word[i:i + 3] for i in range(len(word) - 2)}


# ---- a synthetic trigram index ------------------------------------------------------------------------------------

class TrigramIndex:
    """n_nodes string values, each a few words drawn Zipf-like from a seeded random vocabulary (SEED_WORDS first).
    Node i has uid i + 1.  A trigram's posting list is the union of the node lists of the words that hold it, built
    with numpy from a (word, node) table."""

    def __init__(self, seed: int, n_nodes: int, n_words: int = 4000, words_per_node: int = 3, zipf_a: float = 1.3):
        rng = np.random.default_rng(seed)
        letters = np.array(list("abcdefghijklmnopqrstuvwxyz"))
        vocab = list(SEED_WORDS)
        while len(vocab) < n_words:
            vocab.append("".join(rng.choice(letters, int(rng.integers(3, 9)))))
        self.vocab = vocab
        w = np.minimum(rng.zipf(zipf_a, n_nodes * words_per_node) - 1, n_words - 1)
        # SEED_WORDS are ranked first by the Zipf draw; shuffle ranks so that they are not all the most common
        perm = rng.permutation(n_words)
        w = perm[w]
        w[: len(SEED_WORDS) * words_per_node: words_per_node] = np.arange(len(SEED_WORDS))  # every seed word is used
        node = np.repeat(np.arange(n_nodes, dtype=np.int64), words_per_node)
        key = np.unique(w.astype(np.int64) * n_nodes + node)
        self.word_of, self.node_of = key // n_nodes, key % n_nodes
        self.word_off = np.searchsorted(self.word_of, np.arange(n_words + 1))
        self.tri_words: dict = {}
        for wi, word in enumerate(vocab):
            for t in trigrams(word):
                self.tri_words.setdefault(t, []).append(wi)
        self.n_nodes = n_nodes
        self._cache: dict = {}

    def words_of_node(self, i: int):
        return [self.vocab[w] for w in self.word_of[self.node_of == i]]

    def posting(self, tri: str) -> np.ndarray:
        if tri not in self._cache:
            parts = [self.node_of[self.word_off[w]:self.word_off[w + 1]] for w in self.tri_words.get(tri, [])]
            nodes = np.unique(np.concatenate(parts)) if parts else np.zeros(0, np.int64)
            self._cache[tri] = (nodes + 1).astype(np.uint64)
        return self._cache[tri]


def eval_on_value(nodes, tris_of_value: set, i: int = 0) -> bool:
    """The query of a pattern's nodes on one value's trigram set, node by node: what the index should return."""
    op, ts, subs = nodes[i]
    ch = [t in tris_of_value for t in ts] + [eval_on_value(nodes, tris_of_value, s) for s in subs]
    return all(ch) if op == QAND else any(ch)
