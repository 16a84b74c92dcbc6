"""Place-recognition inputs at the sizes and values where the CUDA kernels change behaviour — vocabulary shapes for the tree
descent, ComputeBoW sizes, keyframe-database queries and database SearchByBoW jobs — and a coverage report of which of those
paths a case reaches.  Test tooling: tests/test_oracle_bow_envelope.py pins the port to the verbatim DBoW2, KeyFrameDatabase.cc
and ORBmatcher.cc on every case where the reference is defined, tests/test_gpu_bow_envelope.py pins the CUDA library to the port.

The kernel constants are restated here (as tests/match_envelope.py restates the matcher's), each next to the line it exists
for.  Nothing in this module calls the CUDA library."""
import functools
import os

import numpy as np

from orb_slam2_b200._lib import KP_DTYPE
from orb_slam2_b200.matcher import FeatureVector, KeyFrameView, bow_and_featvec

# ---- vocabulary descent and ComputeBoW (k_match.cu)
CHILD_RANK_BITS = 23               # k_match.cu:757 — (distance << 23) | child rank; borb_voc_create refuses 2^23 children or more
DESCENT_LANES = 32                 # k_match.cu:754 — a warp per feature, children taken 32 at a time
BUILD_THREADS = 1024               # k_match.cu:818 — bow_build_kernel: one CTA per frame
def build_K(n):                    # k_match.cu:825-826 — key slots: next power of two >= n, at least 32
    K = 32
    while K < n:
        K <<= 1
    return K
def build_chunk(n):                # k_match.cu:830 — the contiguous slice of sorted keys each thread scans
    return (build_K(n) + BUILD_THREADS - 1) // BUILD_THREADS
# ---- keyframe-database score (k_match.cu)
KFDB_U = 8                         # k_match.cu:426 — keyframe words per lane in flight: a pass covers 32 * U = 256 words
KFDB_SMEM_LIMIT = 160 * 1024       # k_match.cu:911 — the query stays in shared memory while nq * 12 + 16 <= 160 KB
KFDB_GLOBAL_NQ = (KFDB_SMEM_LIMIT - 16) // 12 + 1     # 13,652: the first query size read from global memory
# ---- database SearchByBoW (k_bowdb.cu)
MATCH_MAX_FEATURES = 8192          # borb_match.h:45
BDB_WARPS = 32                     # k_bowdb.cu:36
BDB_QCAP = 64                      # k_bowdb.cu:38 — pending-row ring per warp
BDB_CLAIM_WORDS = MATCH_MAX_FEATURES // 32
BDB_WARP_BYTES = BDB_CLAIM_WORDS * 4 + 32 * 24 + BDB_QCAP * 48     # k_bowdb.cu:40
BDB_SMEM_BUDGET = 226 * 1024       # k_bowdb.cu:423
BDB_ITEM_TARGET = 8192             # k_bowdb.cu:569 — keyframes per work item = clamp(BDB_ITEM_TARGET / nt^2, 1, 32)
FIN_THREADS, FIN_REG = 128, 16     # k_bowdb.cu:337-338 — a row stays in registers up to FIN_THREADS * FIN_REG positions
TH_LOW = 50                        # ORBmatcher.cc:15
HISTO_LENGTH = 30
FRAME_HDR_BYTES = 64               # borb_match.h:155 — sizeof(FrameBlockHdr)


def frame_block_layout(nn, m):
    """borb_match.h:158-168: bytes of the packed query frame with nn FeatureVector nodes holding m features."""
    off = FRAME_HDR_BYTES
    for b in (nn * 4, (nn + 1) * 4, m * 2, m * 4, m * 32, nn * 4, nn * 4, (nn + 1) * 4):
        off = ((off + 15) & ~15) + b
    return (off + 15) & ~15


def bowdb_warps(frame_bytes):
    """k_bowdb.cu:421-427 for a block in shared memory: warps per CTA, 0 when fewer than 8 fit."""
    frame = (frame_bytes + 127) & ~127
    if frame + 8 * BDB_WARP_BYTES > BDB_SMEM_BUDGET:
        return 0
    return min(BDB_WARPS, (BDB_SMEM_BUDGET - frame) // BDB_WARP_BYTES)


def frame_fits_smem(nn, m):
    return bowdb_warps(frame_block_layout(nn, m)) >= 8      # k_bowdb.cu:429


def smem_fit_edge(nn=1):
    """The largest m whose block (nn nodes) still fits next to 8 warps of scratch."""
    m = 1
    while frame_fits_smem(nn, m + 1):
        m += 1
    return m


def fin_in_regs(mf):
    per_warp = (((mf + FIN_THREADS // 32 - 1) // (FIN_THREADS // 32)) + 31) & ~31         # k_bowdb.cu:355
    return per_warp <= 32 * FIN_REG                                                       # k_bowdb.cu:357


# coverage classes -> the kernel line each exists for
CLASSES = {
    # descent
    "children_gt_32": "k_match.cu:754 a node wider than a warp: the lane loop takes a second stride",
    "children_32": "k_match.cu:754 a node of exactly 32 children: one full stride",
    "children_33": "k_match.cu:754 a node of 33 children: a second stride of one lane",
    "children_gt_65536": "k_match.cu:757,760 child ranks above 16 bits (the flat vocabulary)",
    "single_child": "k_match.cu:749-762 a node with one child: the warp minimum of one candidate",
    "uneven_depth": "k_match.cu:751 leaves at different depths: the loop ends on children.empty()",
    "tie_lanes": "k_match.cu:757 tied children in different lanes and strides: the lowest rank wins",
    "nid_level_is_L": "k_match.cu:761 levelsup 0: the node is the leaf itself",
    "nid_level_le_0": "k_match.cu:747 levelsup >= L: every feature in node 0",
    "leaf_above_nid_level": "k_match.cu:761 a leaf reached above L - levelsup: node 0 (the reference reads an uninitialised NodeId)",
    # ComputeBoW bookkeeping
    "weight_zero": "k_match.cu:833 a stop word (weight 0) drops out of both vectors",
    "weight_negative": "k_match.cu:833 a negative weight drops out like a stop word",
    "weight_tiny": "k_match.cu:856 a 1e-300 weight kept, lost in the norm",
    "all_stopped": "k_match.cu:836-839 m = 0: both vectors empty, norm 0",
    "n_zero": "borb_compute_bow / bow_build_kernel with no features",
    "K_boundary": "k_match.cu:825 n = 32 / 33 and 1024 / 1025: K doubles",
    "chunk_gt_1": "k_match.cu:829-830 more than one key per thread (n > 1024)",
    "run_spans_chunks": "k_match.cu:842-846 one word run across every thread's chunk",
    "run_sum_order": "k_match.cu:846 a run whose sequential sum differs from a pairwise sum",
    "norm_order": "k_match.cu:853-858 an L1 norm whose sequential chain differs from a pairwise sum",
    # database query
    "kf_words_256": "k_match.cu:431 a keyframe of exactly one 256-word pass",
    "kf_words_257": "k_match.cu:431 a keyframe of 257 words: a second pass of one word",
    "nq_zero": "k_match.cu:424 an empty query (steps = 0)",
    "nq_global": "k_match.cu:910-911 a query too large for shared memory (in_smem == 0)",
    "score_order": "k_match.cu:461-471 score terms whose sequential sum differs from a pairwise one in the float score",
    "cand_ties": "host candidate order: tied scores and tied first shared words",
    # database search
    "nt_1": "k_bowdb.cu:196 a one-column bucket: bestDist2 = 256",
    "nt_32": "k_bowdb.cu:109,174 a 32-column bucket claimed in registers",
    "nt_33": "k_bowdb.cu:109,172-174 a 33-column bucket claimed through the shared-memory bitset",
    "stale_tied": "k_bowdb.cu:175-192 a rescan past a claimed column onto a tied one",
    "ring_wrap": "k_bowdb.cu:231-241 more than BDB_QCAP pending rows in one item",
    "empty_runs": "k_bowdb.cu:216-217 keyframes without the node inside a 32-keyframe batch",
    "rank_guess_miss": "k_bowdb.cu:123-127 the keyframe's node sits at another rank than the frame's",
    "dist_0": "k_bowdb.cu:159 distance 0",
    "dist_256": "k_bowdb.cu:159 distance 256",
    "th_low_eq": "k_bowdb.cu:195 bestDist1 == TH_LOW",
    "th_low_plus_1": "k_bowdb.cu:195 bestDist1 == TH_LOW + 1",
    "ratio_eq": "k_bowdb.cu:197 bestDist1 == nnratio * bestDist2 exactly",
    "hist_boundary": "match_rules.cuh:47 max2 exactly a tenth of max1",
    "one_node_8192": "k_bowdb.cu:106-110 an 8192-column bucket against an 8192-row keyframe",
    "smem_fit_below": "k_bowdb.cu:421-429 the largest block that fits beside 8 warps",
    "smem_fit_above": "k_bowdb.cu:421-429 one feature more: the block is read from global memory",
    "fin_2048": "k_bowdb.cu:357 mf = 2048: the row in registers",
    "fin_2049": "k_bowdb.cu:357 mf = 2049: the row re-read from global memory",
}


# ---------------------------------------------------------------------------------------------------------------------------
# vocabularies: built as node arrays, written as text WITHOUT a trailing newline (tests/test_oracle_dbow_ref.py: the reference's
# `while(!f.eof())` loader turns a final newline into a garbage node), so that the same file loads in DBoW2, the port and the library
class Tree:
    def __init__(self, L, k=10):
        self.L, self.k = L, k
        self.parent, self.desc, self.weight = [0], [np.zeros(32, np.uint8)], [0.0]

    def add(self, parent, desc, weight=0.0):
        self.parent.append(int(parent)); self.desc.append(np.asarray(desc, np.uint8)); self.weight.append(float(weight))
        return len(self.parent) - 1

    def arrays(self):
        parent = np.array(self.parent, np.int32)
        has_child = np.zeros(len(parent), bool)
        has_child[parent[1:]] = True
        # leaf flags equal "has no children": the port tests the flag, DBoW2 and the library test children.empty()
        return dict(parent=parent, is_leaf=(~has_child).astype(np.uint8), desc=np.stack(self.desc), weight=np.array(self.weight, np.float64),
                    k=self.k, L=self.L)


def voc_text(a):
    lines = [f"{a['k']} {a['L']} 0 0"]
    for i in range(1, len(a["parent"])):
        lines.append(f"{a['parent'][i]} {int(a['is_leaf'][i])} " + " ".join(map(str, a["desc"][i].tolist())) + f" {float(a['weight'][i])!r}")
    return "\n".join(lines)                                  # no trailing newline


def write_voc(a, path):
    with open(path, "w") as f:
        f.write(voc_text(a))
    return path


def depths(a):
    d = np.zeros(len(a["parent"]), np.int32)
    for i in range(1, len(d)):
        d[i] = d[a["parent"][i]] + 1
    return d


def child_counts(a):
    return np.bincount(a["parent"][1:], minlength=len(a["parent"]))


def _flip(rng, d, nbits):
    bits = np.unpackbits(np.asarray(d, np.uint8)).copy()
    bits[rng.choice(256, int(nbits), replace=False)] ^= 1
    return np.packbits(bits)


def _grow(t, rng, parent, pdesc, width, depth_left, flips=24, weight=lambda rng: 0.5 + rng.random() * 9.5):
    """Children of `parent` near its descriptor (so that a feature near a leaf descends to it), recursively."""
    for _ in range(width):
        d = _flip(rng, pdesc, flips) if parent else rng.integers(0, 256, 32, dtype=np.uint8)
        if depth_left == 1:
            t.add(parent, d, weight(rng))
        else:
            c = t.add(parent, d)
            _grow(t, rng, c, d, width, depth_left - 1, flips, weight)


@functools.lru_cache(maxsize=None)
def vocabulary(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "k40":                                        # 40 children per node (header k = 10: the loaders read it only)
        t = Tree(2)
        _grow(t, rng, 0, None, 40, 2)
    elif name == "w32_33":                                   # nodes of exactly 32 and 33 children, others of 1 to 3
        t = Tree(2)
        for i, w in enumerate([32, 33] + [1 + i % 3 for i in range(31)]):
            d = rng.integers(0, 256, 32, dtype=np.uint8)
            c = t.add(0, d)
            for _ in range(w):
                t.add(c, _flip(rng, d, 24), 0.5 + rng.random())
    elif name == "flat70000":                                # header "10 1 0 0", 70,000 leaves under the root
        t = Tree(1)
        for d in rng.integers(0, 256, (70000, 32), dtype=np.uint8):
            t.add(0, d, 0.25 + rng.random())
    elif name == "uneven":                                   # leaves at depths 1-4, single-child chains
        t = Tree(4)
        t.add(0, rng.integers(0, 256, 32, dtype=np.uint8), 1.5)              # a leaf at depth 1
        p = 0
        d = rng.integers(0, 256, 32, dtype=np.uint8)
        for depth in range(1, 5):                                            # a chain of single children down to depth 4
            p = t.add(p, d, 0.0 if depth < 4 else 2.5)
            d = _flip(rng, d, 20)
        d = rng.integers(0, 256, 32, dtype=np.uint8)
        b = t.add(0, d)
        for j in range(10):                                                  # depth-2 leaves and depth-3 subtrees side by side
            dj = _flip(rng, d, 24)
            if j % 2:
                t.add(b, dj, 0.5 + j)
            else:
                c = t.add(b, dj)
                for _ in range(1 + j // 2):
                    t.add(c, _flip(rng, dj, 24), 0.25 + rng.random())
        _grow(t, rng, t.add(0, rng.integers(0, 256, 32, dtype=np.uint8)), t.desc[-1], 3, 3)   # a full depth-4 subtree
    elif name == "tied":                                     # 100 children of the root, equal descriptors at ranks in other lanes / strides
        t = Tree(2)
        X, Y = rng.integers(0, 256, (2, 32), dtype=np.uint8)
        for r in range(100):
            d = X if r in (3, 35, 67, 99) else (Y if r in (10, 90) else rng.integers(0, 256, 32, dtype=np.uint8))
            c = t.add(0, d)
            for _ in range(2 + r % 3):
                t.add(c, _flip(rng, d, 30), 0.5 + rng.random())
    elif name == "weights":                                  # order-sensitive, zero, negative and tiny positive weights
        t = Tree(2)
        ws = [1.0] + [2.0 ** -55] * 120 + [0.1] * 20 + [0.0] * 10 + [-0.5] * 10 + [1e-300] * 10
        d = rng.integers(0, 256, (len(ws) // 10 + 1, 32), dtype=np.uint8)
        inner = [t.add(0, x) for x in d]
        for i, w in enumerate(ws):
            t.add(inner[i // 10], _flip(rng, d[i // 10], 24), w)
    elif name == "all_stop":                                 # every word a stop word
        t = Tree(2)
        _grow(t, rng, 0, None, 10, 2, weight=lambda rng: 0.0)
    else:
        raise KeyError(name)
    return t.arrays()


VOCABS = ["k40", "w32_33", "flat70000", "uneven", "tied", "weights", "all_stop"]
LEVELSUP = {"k40": [0, 1, 2, 3], "w32_33": [0, 1, 2], "flat70000": [0, 1, 2], "uneven": [0, 1, 2, 3, 4, 5], "tied": [0, 1, 2],
            "weights": [0, 1, 2], "all_stop": [0, 1]}


def near_leaves(a, rng, n, flips=(0, 1, 2, 3), leaves=None):
    """n descriptors near leaves of the tree (copies with a few flipped bits), cycling through `leaves`."""
    if leaves is None:
        leaves = np.nonzero(a["is_leaf"])[0]
        leaves = leaves[rng.permutation(len(leaves))]
    out = np.zeros((n, 32), np.uint8)
    for i in range(n):
        out[i] = _flip(rng, a["desc"][leaves[i % len(leaves)]], flips[i % len(flips)])
    return out


@functools.lru_cache(maxsize=None)
def descriptors(name):
    """Descriptor sets per vocabulary: features near its leaves, random ones, and the ones aimed at its edge."""
    a = vocabulary(name)
    rng = np.random.default_rng(len(name) * 7919)
    leaves = np.nonzero(a["is_leaf"])[0]
    small = name == "flat70000"                              # 70,000 distances per feature in the CPU descents: fewer features
    sets = {"near": near_leaves(a, rng, 80 if small else 400), "random": rng.integers(0, 256, (40 if small else 300, 32), dtype=np.uint8)}
    if small:                                                # exact copies of leaves ranked above 65,536 and below
        hi = leaves[leaves > 65536 + 1][:120]
        sets["high_ranks"] = np.concatenate([a["desc"][hi], near_leaves(a, rng, 40, leaves=leaves[:100])])
    if name == "tied":
        X = a["desc"][np.nonzero(a["parent"] == 0)[0][3]]; Y = a["desc"][np.nonzero(a["parent"] == 0)[0][10]]
        sets["ties"] = np.stack([X, Y] * 20 + [_flip(rng, X, 1), _flip(rng, Y, 2)] * 10)
    if name == "weights":
        by_w = {w: leaves[a["weight"][leaves] == w] for w in (1.0, 2.0 ** -55, 0.1)}
        # one feature on the heavy word, then one on each tiny word (their sum is lost in a sequential norm, not in a pairwise one),
        # and runs of ten features on the 0.1 words (a sequential run sum differs from a pairwise one)
        sets["order"] = np.concatenate([a["desc"][by_w[1.0]], a["desc"][by_w[2.0 ** -55]], np.repeat(a["desc"][by_w[0.1]], 10, 0),
                                        near_leaves(a, rng, 60)])
    return sets


# ComputeBoW sizes: n features on the "weights" vocabulary, chosen near its leaves; "one_word" puts every feature on one 0.1 word
COMPUTE_SIZES = [0, 1, 32, 33, 1024, 1025, 4097, 8192]


@functools.lru_cache(maxsize=None)
def compute_set(n, one_word=False):
    a = vocabulary("weights")
    rng = np.random.default_rng(n + 17 * one_word)
    leaves = np.nonzero(a["is_leaf"])[0]
    if one_word:
        return np.repeat(a["desc"][leaves[a["weight"][leaves] == 0.1][:1]], n, 0)
    heavy = leaves[a["weight"][leaves] == 1.0]
    order = np.concatenate([heavy, leaves[rng.permutation(len(leaves))]])
    return near_leaves(a, rng, n, flips=(0, 0, 1), leaves=order) if n else np.zeros((0, 32), np.uint8)


def leaf_depth_of_words(a):
    """depth of the leaf of each word id (word ids in leaf order, as every loader numbers them)."""
    return depths(a)[np.nonzero(a["is_leaf"])[0]]


def reference_defined(a, levelsup, words):
    """DBoW2 leaves NodeId uninitialised when a feature's leaf lies above level L - levelsup (TemplatedVocabulary.h:1227-1257):
    the reference is undefined for such features, so only the port and the library are compared there."""
    nid_level = a["L"] - levelsup
    return nid_level <= 0 or bool((leaf_depth_of_words(a)[np.asarray(words)] >= nid_level).all())


def descent_coverage(a, levelsup, words):
    """Classes a descent of features ending at `words` reaches on tree `a` at `levelsup`."""
    hit = set()
    cc = child_counts(a)
    dep = depths(a)
    leaves = np.nonzero(a["is_leaf"])[0]
    wl = leaves[np.asarray(words, np.int64)] if len(words) else np.zeros(0, np.int64)
    path = set()
    for leaf in set(wl.tolist()):                           # every inner node on the way to a reached leaf
        p = a["parent"][leaf]
        while True:
            path.add(int(p))
            if p == 0:
                break
            p = a["parent"][p]
    widths = cc[list(path)] if path else np.zeros(0, int)
    if (widths > 32).any(): hit.add("children_gt_32")
    if (widths == 32).any(): hit.add("children_32")
    if (widths == 33).any(): hit.add("children_33")
    if (widths == 1).any(): hit.add("single_child")
    if len(wl) and (wl - 1 >= 65536).any() and (widths > 65536).any(): hit.add("children_gt_65536")
    if len(wl) and len(set(dep[wl].tolist())) > 1: hit.add("uneven_depth")
    nid_level = a["L"] - levelsup
    if len(wl):
        if nid_level == a["L"]: hit.add("nid_level_is_L")
        if nid_level <= 0: hit.add("nid_level_le_0")
        if nid_level > 0 and (dep[wl] < nid_level).any(): hit.add("leaf_above_nid_level")
    # ties: a reached node whose children share a descriptor at ranks in different lanes and strides
    for p in path:
        ch = np.nonzero(a["parent"][1:] == p)[0] + 1
        if len(ch) > 32:
            _, inv, cnt = np.unique(a["desc"][ch], axis=0, return_inverse=True, return_counts=True)
            for g in np.nonzero(cnt > 1)[0]:
                r = np.nonzero(inv.ravel() == g)[0]
                if len(set((r // 32).tolist())) > 1 and len(set((r % 32).tolist())) > 1:
                    hit.add("tie_lanes")
    return hit


def _pairwise(x):
    x = list(x)
    while len(x) > 1:
        x = [x[i] + x[i + 1] if i + 1 < len(x) else x[i] for i in range(0, len(x), 2)]
    return x[0] if x else 0.0


def bow_coverage(a, words, weights, n):
    """ComputeBoW classes of one descriptor set: per-feature (word, weight) of the descent, n features."""
    hit = set()
    words = np.asarray(words); weights = np.asarray(weights, np.float64)
    if n == 0: hit.add("n_zero")
    if n in (32, 33, 1024, 1025): hit.add("K_boundary")
    if build_chunk(n) > 1: hit.add("chunk_gt_1")
    if (weights == 0).any(): hit.add("weight_zero")
    if (weights < 0).any(): hit.add("weight_negative")
    if ((weights > 0) & (weights < 1e-200)).any(): hit.add("weight_tiny")
    if n and not (weights > 0).any(): hit.add("all_stopped")
    kept = weights > 0
    runs = {}
    for w, v in zip(words[kept].tolist(), weights[kept].tolist()):
        runs.setdefault(w, []).append(v)
    for vs in runs.values():
        if len(vs) == n and -(-n // build_chunk(n)) >= BUILD_THREADS:     # the run's keys reach into every thread's chunk
            hit.add("run_spans_chunks")
        if sum_seq(vs) != _pairwise(vs):
            hit.add("run_sum_order")
    if runs:
        sums = [abs(sum_seq(v)) for _, v in sorted(runs.items())]
        if sum_seq(sums) != _pairwise(sums):
            hit.add("norm_order")
    return hit


def sum_seq(vs):
    s = 0.0
    for v in vs:
        s += v
    return s


# ---------------------------------------------------------------------------------------------------------------------------
# keyframe-database queries: BowVectors as {word: value}; the query's words are drawn below FLAT_WORDS so that the verbatim
# KeyFrameDatabase can be built over the flat vocabulary's inverted file
FLAT_WORDS = 70000
BIG = 1.0 + 2.0 ** -24             # term -2 * BIG: -acc / 2 is a float midpoint (ties to even: 1.0f)
TINY = 2.0 ** -56                  # term -2^-55: lost after BIG in a sequential sum, 64 of them tip the float score up


def _bow(words, values):
    o = np.argsort(words)
    return dict(zip(np.asarray(words)[o].tolist(), np.asarray(values, np.float64)[o].tolist()))


@functools.lru_cache(maxsize=None)
def query_world():
    """Keyframe BowVectors (256 and 257 words, identical keyframes for tied scores and first words, order-sensitive values) and
    queries of 0, 1, 8192 and 20,000 words."""
    rng = np.random.default_rng(41)
    kfs = []
    base = np.sort(rng.choice(FLAT_WORDS, 4000, replace=False))
    for i in range(24):
        nw = [256, 257, 255, 512, 1, 300][i % 6]
        w = np.sort(rng.choice(base, nw, replace=False))
        v = rng.random(nw); v /= v.sum()
        kfs.append(_bow(w, v))
    kfs.append(dict(kfs[3])); kfs.append(dict(kfs[3]))      # identical keyframes: tied scores and tied first shared words
    # order-sensitive keyframes: BIG at the first shared word (sequential sum keeps 1.0f) and BIG after 300 tiny terms
    ow = np.sort(rng.choice(base, 400, replace=False))
    v1 = np.full(400, TINY); v1[0] = BIG
    v2 = np.full(400, TINY); v2[300] = BIG
    kfs.append(_bow(ow, v1)); kfs.append(_bow(ow, v2))
    q_order = _bow(ow, v1)                                  # shares the order-sensitive words with both, same values: terms -2x
    q_order2 = _bow(ow, v2)
    queries = {
        "nq0": {},
        "nq1": _bow(base[:1], [1.0]),
        "nq8192": _bow(np.sort(rng.choice(FLAT_WORDS, 8192, replace=False)), rng.random(8192) / 8192),
        "nq20000": _bow(np.sort(np.concatenate([base, rng.choice(np.setdiff1d(np.arange(FLAT_WORDS), base), 16000, replace=False)])),
                        rng.random(20000) / 20000),
        "order_first": q_order,
        "order_mid": q_order2,
        "near3": dict(kfs[3]),
    }
    n_kf = len(kfs)
    neigh = np.full((n_kf, 10), -1, np.int32)
    for s in range(n_kf):
        nb = [x for x in dict.fromkeys([(s + 1) % n_kf, (s + 2) % n_kf, (s * 7) % n_kf, 25, 24]) if x != s][:10]
        neigh[s, :len(nb)] = nb
    return kfs, queries, neigh


def float_score_orders(q, b):
    """(sequential float score, pairwise float score) of two BowVectors: the L1 terms in word order, summed both ways."""
    terms = [abs(q[w] - b[w]) - abs(q[w]) - abs(b[w]) for w in sorted(set(q) & set(b))]
    return np.float32(-sum_seq(terms) / 2.0), np.float32(-_pairwise(terms) / 2.0)


def query_coverage(kfs, qname, q):
    hit = set()
    sizes = [len(b) for b in kfs]
    if 256 in sizes and any(set(b) & set(q) for b in kfs if len(b) == 256): hit.add("kf_words_256")
    if 257 in sizes and any(set(b) & set(q) for b in kfs if len(b) == 257): hit.add("kf_words_257")
    if len(q) == 0: hit.add("nq_zero")
    if len(q) * 12 + 16 > KFDB_SMEM_LIMIT: hit.add("nq_global")
    if any(len(set(q) & set(b)) and float_score_orders(q, b)[0] != float_score_orders(q, b)[1] for b in kfs): hit.add("score_order")
    shared = [b for b in kfs if set(b) & set(q)]
    keys = [(min(set(q) & set(b)), tuple(sorted(b.items()))) for b in shared]
    if len(keys) != len(set(keys)): hit.add("cand_ties")
    return hit


# ---------------------------------------------------------------------------------------------------------------------------
# database searches: frames and keyframes with explicit FeatureVectors (node ids chosen by the case), so that every bucket width
# and row distance is set on purpose
def _keys(rng, n, angles=None):
    k = np.zeros(n, KP_DTYPE)
    k["x"] = rng.uniform(10, 630, n); k["y"] = rng.uniform(10, 470, n); k["size"] = 31.0; k["class_id"] = -1
    k["angle"] = rng.uniform(0, 360, n) if angles is None else angles
    return k


def _view(keys, desc, nodes, has_mp=None):
    """KeyFrameView whose FeatureVector puts feature i in node nodes[i] (< 0: in no node)."""
    nodes = np.asarray(nodes, np.int64)
    keep = nodes >= 0
    fv = FeatureVector.from_nodes(np.where(keep, nodes, 0), keep)
    return KeyFrameView(mvKeysUn=keys, mDescriptors=np.ascontiguousarray(desc, np.uint8), mFeatVec=fv, has_mp=has_mp)


def _dist(a, b):
    return int(np.unpackbits(np.bitwise_xor(a, b)).sum())


def _at(rng, base, d, avoid=None):
    """A descriptor at exactly distance d from base (bits chosen outside `avoid`, a bit mask of 256)."""
    bits = np.unpackbits(base).copy()
    pool = np.arange(256) if avoid is None else np.nonzero(~avoid)[0]
    sel = rng.choice(pool, d, replace=False)
    bits[sel] ^= 1
    return np.packbits(bits), sel


@functools.lru_cache(maxsize=None)
def edges_case():
    """One frame with buckets of 1, 2, 32, 33 and 96 columns (and two nodes the keyframes lack), against 40 keyframes (more than
    one 32-keyframe batch) that lack some nodes, carry extra ones, and whose rows sit at chosen distances from the columns:
    0, 256, TH_LOW, TH_LOW + 1, best == 0.75 * second exactly, tied duplicate columns claimed in turn, and enough good rows in the
    96-column bucket to wrap the pending-row ring."""
    rng = np.random.default_rng(5)
    widths = {10: 1, 20: 2, 30: 32, 40: 33, 50: 96, 60: 1, 70: 3}
    fnodes = np.concatenate([np.full(w, nd) for nd, w in widths.items()])
    nF = len(fnodes)
    fdesc = rng.integers(0, 256, (nF, 32), dtype=np.uint8)
    col = {nd: np.nonzero(fnodes == nd)[0] for nd in widths}
    # tied columns in the 32- and 33-wide buckets: c1 is 20 bits from c0, and the tie rows below sit 10 bits from both
    tie_row = {}
    for nd in (30, 40):
        c = col[nd]
        fdesc[c[1]], s = _at(rng, fdesc[c[0]], 20)
        bits = np.unpackbits(fdesc[c[0]]).copy(); bits[s[:10]] ^= 1
        tie_row[nd] = np.packbits(bits)
    # a row 30 bits from column a and 40 bits (disjoint ones) from column b: bestDist1 == 0.75 * bestDist2
    a_col, b_col = col[50][0], col[50][1]
    ratio_row, s1 = _at(rng, fdesc[a_col], 30)
    mask = np.zeros(256, bool); mask[s1] = True
    fdesc[b_col] = _at(rng, ratio_row, 40, avoid=mask)[0]
    F = _view(_keys(rng, nF), fdesc, fnodes)
    kfs = []
    for k in range(40):
        rows, nodes = [], []
        for nd, w in widths.items():
            if nd in (60, 70) or (k % 5 == 2 and nd != 50):        # nodes the keyframe lacks: empty runs inside the batch
                continue
            c = col[nd]
            nr = 30 if nd == 50 else min(w + 2, 6)
            for r in range(nr):
                j = c[(r + k) % w]
                kind = (r + k) % 7
                if kind == 0: d = fdesc[j].copy()                                   # distance 0
                elif kind == 1: d = ~fdesc[j]                                       # distance 256 to its column
                elif kind == 2: d = _at(rng, fdesc[j], TH_LOW)[0]
                elif kind == 3: d = _at(rng, fdesc[j], TH_LOW + 1)[0]
                else: d = _at(rng, fdesc[j], int(rng.integers(0, 45)))[0]
                rows.append(d); nodes.append(nd)
            if nd in (30, 40):                                      # c0 claimed by its copy; then a row tied between c0 and c1
                rows.append(fdesc[c[0]].copy()); nodes.append(nd)   # is stale and rescans onto c1
                rows.append(tie_row[nd]); nodes.append(nd)
        rows.append(ratio_row); nodes.append(50)
        for extra in (5, 15, 45):                                   # nodes the frame lacks: the rank guess misses
            rows.append(rng.integers(0, 256, 32, dtype=np.uint8)); nodes.append(extra)
        rows = np.stack(rows)
        n = len(rows)
        hm = np.ones(n, np.uint8); hm[(np.arange(n) + k) % 9 == 4] = 0
        kfs.append(_view(_keys(rng, n), rows, nodes, hm))
    return dict(F=F, kfs=kfs, ratio=0.75, ori=True)


def hist_case():
    """One keyframe whose rows are exact copies of single-column buckets, rotated so the histogram is {1: 40, 3: 4, 5: 3}:
    max2 == 0.1 * max1 exactly (kept), max3 below (culled)."""
    rng = np.random.default_rng(9)
    bins = np.concatenate([np.full(40, 1), np.full(4, 3), np.full(3, 5)])
    n = len(bins)
    fdesc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    fang = rng.uniform(0, 360, n).astype(np.float32)
    F = _view(_keys(rng, n, fang), fdesc, np.arange(n) * 3 + 1)
    kang = np.mod(fang + 30.0 * bins + 5.0, 360.0).astype(np.float32)
    kf = _view(_keys(rng, n, kang), fdesc, np.arange(n) * 3 + 1, np.ones(n, np.uint8))
    return dict(F=F, kfs=[kf], ratio=0.75, ori=True)


def one_node_case(nF, n_kf=2, nK=None, seed=13, nodes=1):
    """A frame of nF features in `nodes` nodes against keyframes whose rows are noisy copies of the frame's columns."""
    rng = np.random.default_rng(seed + nF)
    fdesc = rng.integers(0, 256, (nF, 32), dtype=np.uint8)
    fnodes = np.arange(nF) % nodes
    F = _view(_keys(rng, nF), fdesc, fnodes)
    kfs = []
    for k in range(n_kf):
        nk = nK or nF
        src = rng.choice(nF, nk, replace=nk > nF)
        flip = rng.random((nk, 256)) < rng.choice([0.0, 0.02, 0.08, 0.2], nk)[:, None]
        rows = np.packbits(np.unpackbits(fdesc[src], axis=1) ^ flip, axis=1)
        kang = (F.mvKeysUn["angle"][src] + rng.choice([0.0, 0.0, 0.0, 100.0], nk)).astype(np.float32) % np.float32(360)
        kfs.append(_view(_keys(rng, nk, kang), rows, fnodes[src], (rng.random(nk) < 0.7).astype(np.uint8)))
    return dict(F=F, kfs=kfs, ratio=0.75, ori=True)


SMEM_EDGE = smem_fit_edge(1)

SEARCH_BUILDERS = {
    "edges": edges_case,
    "hist_tenth": hist_case,
    "one_node_8192": lambda: one_node_case(MATCH_MAX_FEATURES, n_kf=2),
    "smem_fit_below": lambda: one_node_case(SMEM_EDGE, n_kf=2, nK=1500),
    "smem_fit_above": lambda: one_node_case(SMEM_EDGE + 1, n_kf=2, nK=1500),
    "fin_2048": lambda: one_node_case(2048, n_kf=3, nK=1200, nodes=64),
    "fin_2049": lambda: one_node_case(2049, n_kf=3, nK=1200, nodes=64),
}
SEARCH_NAMES = sorted(SEARCH_BUILDERS)


@functools.lru_cache(maxsize=None)
def search_case(name):
    return SEARCH_BUILDERS[name]()


def _hamming_rows(A, b):
    return np.unpackbits(np.bitwise_xor(A, b), axis=1).sum(1)


def search_coverage(c, port_results, port_no_ori):
    """Classes a database search case reaches, from its inputs and the port's SearchByBoW of each keyframe (with and without the
    rotation check)."""
    hit = set()
    F = c["F"]
    fv = F.mFeatVec.as_dict()
    widths = {nd: len(v) for nd, v in fv.items()}
    m = len(F.mFeatVec.feat_idx)
    if m == MATCH_MAX_FEATURES and len(widths) == 1 and any(len(k.mFeatVec.feat_idx) == MATCH_MAX_FEATURES for k in c["kfs"]):
        hit.add("one_node_8192")
    nn = len(widths)
    if frame_fits_smem(nn, m) and not frame_fits_smem(nn, m + 1): hit.add("smem_fit_below")
    if not frame_fits_smem(nn, m) and frame_fits_smem(nn, m - 1): hit.add("smem_fit_above")
    if m == 2048 and fin_in_regs(m): hit.add("fin_2048")
    if m == 2049 and not fin_in_regs(m): hit.add("fin_2049")
    fnode_rank = {nd: i for i, nd in enumerate(F.mFeatVec.node_id.tolist())}
    for kb in range(0, len(c["kfs"]), 32):
        batch = c["kfs"][kb:kb + 32]
        for nd, cols in fv.items():
            have = [nd in set(k.mFeatVec.node_id.tolist()) for k in batch]
            if any(have) and not all(have): hit.add("empty_runs")
            good = sum(int(k.has_mp[k.mFeatVec.as_dict().get(nd, [])].sum()) for k in batch if nd in set(k.mFeatVec.node_id.tolist()))
            if good > BDB_QCAP: hit.add("ring_wrap")
    for k, (n_p, match), (_, match_all) in zip(c["kfs"], port_results, port_no_ori):
        kfv = k.mFeatVec.as_dict()
        knodes = k.mFeatVec.node_id.tolist()
        for nd in knodes:
            if nd in fnode_rank:
                r = fnode_rank[nd]
                if min(r, len(knodes) - 1) != knodes.index(nd): hit.add("rank_guess_miss")
        matched_rows = set(match_all[match_all >= 0].tolist())
        for nd, rows in kfv.items():
            cols = fv.get(nd)
            if not cols or len(cols) > 256:                     # the row-distance classes are set up in narrow buckets
                continue
            fd = F.mDescriptors[cols]
            nt = len(cols)
            for i in rows:
                if not k.has_mp[i]:
                    continue
                d = np.sort(_hamming_rows(fd, k.mDescriptors[i]))
                b1, b2 = int(d[0]), (int(d[1]) if nt > 1 else 256)
                if nt == 1 and b1 <= TH_LOW: hit.add("nt_1")
                if b1 == 0: hit.add("dist_0")
                if d[-1] == 256: hit.add("dist_256")
                if b1 == TH_LOW: hit.add("th_low_eq")
                if b1 == TH_LOW + 1: hit.add("th_low_plus_1")
                if b1 <= TH_LOW and np.float32(b1) == np.float32(c["ratio"]) * np.float32(b2): hit.add("ratio_eq")
                # a row whose best distance ties can match only after a claim made it stale and the rescan took the tied column
                if nt > 1 and b1 == b2 <= TH_LOW and i in matched_rows: hit.add("stale_tied")
        # buckets that matched at least one row, by width
        node_of = {f: nd for nd, cols in fv.items() for f in cols}
        for f in np.nonzero(match_all >= 0)[0]:
            nt = widths[node_of[int(f)]]
            if nt == 32: hit.add("nt_32")
            if nt == 33: hit.add("nt_33")
        # rotation histogram of the matches before the cull
        if c["ori"]:
            hist = np.zeros(HISTO_LENGTH, int)
            for f in np.nonzero(match_all >= 0)[0]:
                hist[_rot_bin(k.mvKeysUn["angle"][match_all[f]], F.mvKeysUn["angle"][f])] += 1
            srt = np.sort(hist)[::-1]
            if srt[0] and (np.float32(srt[1]) == np.float32(0.1) * np.float32(srt[0]) or np.float32(srt[2]) == np.float32(0.1) * np.float32(srt[0])):
                hit.add("hist_boundary")
    return hit


def _rot_bin(a1, a2):
    rot = np.float32(np.float32(a1) - np.float32(a2))
    if rot < 0:
        rot = np.float32(rot + np.float32(360.0))
    b = int(np.floor(np.float32(rot * np.float32(1.0 / 30)) + 0.5))
    return 0 if b == 30 else b


# ---------------------------------------------------------------------------------------------------------------------------
# the port on a case, in comparable form
def port_transform(O, pv, desc, levelsup):
    """(bow dict, FeatureVector, words, weights) of the port."""
    w, wt, nd = pv.transform_raw(desc, levelsup)
    bow, fv = bow_and_featvec(w, wt, nd)
    return bow, fv, w, wt, nd


def port_search(O, c, ori=None):
    ori = c["ori"] if ori is None else ori
    return [O.port_search_by_bow(k, c["F"], c["ratio"], ori) for k in c["kfs"]]


def dense_from_pairs(nm, off, pairs, n_f):
    out = np.full((len(nm), n_f), -1, np.int32)
    for k in range(len(nm)):
        pr = pairs[off[k]:off[k] + nm[k]]
        out[k, (pr & 0xFFFF).astype(np.int64)] = (pr >> 16).astype(np.int32)
    return out
