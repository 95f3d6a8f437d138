"""Pin the oracle's pinned X-drop aligner against the reference's own unit vectors
(src/unittest/xdrop_aligner.cpp, pinned cases; tests/golden/xdrop_pinned.json)."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
from vg_b200 import capi

GOLD = H.load_golden("xdrop_pinned.json")


def oracle_xdrop(index, parents, nodes, root_trim, read, scores, max_gap):
    lib = H.oracle_lib()
    par = np.asarray(parents, dtype=np.int32)
    nd = np.asarray(nodes, dtype=np.uint32)
    q = np.frombuffer(read.encode() + b"\0", dtype=np.uint8).copy()
    score = C.c_int32()
    maps = np.zeros(256, dtype=H.mapping_dt)
    edits = np.zeros(1024, dtype=np.uint32)
    nm, ne = C.c_uint32(), C.c_uint32()
    rc = lib.oracle_xdrop_pinned(C.byref(index.view), C.byref(scores), capi.ptr(par), capi.ptr(nd), len(nd), root_trim,
                                 capi.ptr(q), len(read), max_gap, C.byref(score), capi.ptr(maps), 256, C.byref(nm),
                                 capi.ptr(edits), 1024, C.byref(ne))
    assert rc == 0
    return score.value, capi.decode_path(maps, edits, nm.value)


def case_index(case):
    seqs = case["nodes"]
    # one haplotype per root-to-leaf walk so every node has a GBWT record
    parents = case["parents"]
    children = {i: [] for i in range(len(seqs))}
    for i, p in enumerate(parents):
        if p >= 0:
            children[p].append(i)
    paths = []
    for leaf in range(len(seqs)):
        if children[leaf]:
            continue
        walk = []
        x = leaf
        while x >= 0:
            walk.append(2 * (x + 1))
            x = parents[x]
        paths.append(walk[::-1])
    return capi.HostIndex(seqs, paths, None, k=5, w=3)


@pytest.mark.parametrize("case", GOLD["cases"], ids=[c["name"] for c in GOLD["cases"]])
def test_oracle_xdrop_matches_reference_vectors(case):
    index = case_index(case)
    sc = capi.Scores(*case["scores"])
    nodes = [2 * (i + 1) for i in range(len(case["nodes"]))]
    score, path = oracle_xdrop(index, case["parents"], nodes, 0, case["read"], sc, case["max_gap"])
    want = case["score"] if "score" in case else eval(case["score_expr"], {"len": len(case["read"])})
    assert score == want
    if "path" in case:
        assert path == case["path"]
    # every alignment accounts for the whole query
    qlen = sum(ed[1] for m in path for ed in m[2] if ed[0] in "MSI")
    assert qlen == len(case["read"])


def _random_tree_problem(rng, n_nodes, qlen, err):
    """A random haplotype tree with a query that follows one root-to-leaf walk with errors."""
    seqs, parents = [], []
    for i in range(n_nodes):
        L = int(rng.integers(1, 33))
        seqs.append("".join("ACGT"[x] for x in rng.integers(0, 4, size=L)))
        parents.append(-1 if i == 0 else int(rng.integers(max(0, i - 3), i)))
    # DFS-renumber so that parents precede children in visit order
    children = {i: [] for i in range(n_nodes)}
    for i, p in enumerate(parents):
        if p >= 0:
            children[p].append(i)
    order, stack = [], [0]
    while stack:
        x = stack.pop()
        order.append(x)
        stack.extend(reversed(children[x]))
    remap = {old: new for new, old in enumerate(order)}
    seqs = [seqs[o] for o in order]
    parents = [(-1 if parents[o] < 0 else remap[parents[o]]) for o in order]
    # walk
    leaf = int(rng.integers(0, n_nodes))
    walk = []
    x = leaf
    while x >= 0:
        walk.append(x)
        x = parents[x]
    ref = "".join(seqs[i] for i in reversed(walk))
    trim = int(rng.integers(0, len(seqs[0])))
    ref = ref[trim:]
    q = []
    for c in ref[:qlen + 8]:
        r = rng.random()
        if r < err:
            q.append("ACGT"[int(rng.integers(0, 4))])
        elif r < 1.5 * err:
            continue
        elif r < 2 * err:
            q.append(c); q.append("ACGT"[int(rng.integers(0, 4))])
        else:
            q.append(c)
    q = "".join(q)[:qlen]
    if not q:
        q = "A"
    return seqs, parents, trim, q


@pytest.mark.gpu
def test_cuda_xdrop_matches_reference_vectors_and_oracle():
    problems, wants = [], []
    for case in GOLD["cases"]:
        index = case_index(case)
        dev = capi.Device(index, scores=capi.Scores(*case["scores"]))
        nodes = [2 * (i + 1) for i in range(len(case["nodes"]))]
        got = dev.xdrop_pinned_batch([(case["parents"], nodes, 0, case["read"].encode(), case["max_gap"])])[0]
        want = oracle_xdrop(index, case["parents"], nodes, 0, case["read"], capi.Scores(*case["scores"]), case["max_gap"])
        assert got[0] == want[0] and got[1] == want[1], case["name"]
        exp = case["score"] if "score" in case else eval(case["score_expr"], {"len": len(case["read"])})
        assert got[0] == exp
        dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed,qlen,err,gap", [(1, 40, 0.03, 20), (2, 150, 0.05, 60), (3, 250, 0.08, 40), (4, 97, 0.15, 54),
                                               (5, 33, 0.3, 5)])
def test_cuda_xdrop_parity_random_trees(seed, qlen, err, gap):
    rng = np.random.default_rng(seed)
    for rep in range(6):
        seqs, parents, trim, q = _random_tree_problem(rng, int(rng.integers(1, 40)), qlen, err)
        case = {"nodes": seqs, "parents": parents}
        index = case_index(case)
        dev = capi.Device(index)
        nodes = [2 * (i + 1) for i in range(len(seqs))]
        qs = [q, q[: max(1, len(q) // 2)], q[::-1]]
        got = dev.xdrop_pinned_batch([(parents, nodes, trim, s.encode(), gap) for s in qs])
        for s, g in zip(qs, got):
            want = oracle_xdrop(index, parents, nodes, trim, s, capi.DEFAULT_SCORES, gap)
            assert g[0] == want[0] and g[1] == want[1], (seed, rep, s)
        dev.close()
