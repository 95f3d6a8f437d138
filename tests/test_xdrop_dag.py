"""Seeded two-pass X-drop alignment on a DAG (Aligner::align_xdrop, dozeu_interface.cpp:608-722):
the oracle's DAG pass against its own pinned aligner on trees, end-to-end properties of the two
passes, and the CUDA stage seam gb_xdrop_dag_batch against the oracle."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
from vg_b200 import capi
import test_xdrop_golden as TX
import test_sw_golden as TS

NO_SEED = 0xFFFFFFFF


def _csr(preds):
    pred = np.asarray([p for ps in preds for p in ps] + [0], dtype=np.uint32)
    off = np.zeros(len(preds) + 1, dtype=np.uint32)
    off[1:] = np.cumsum([len(ps) for ps in preds])
    return pred, off


def oracle_dag_pass(index, nodes, preds, read, scores, start_u, start_o, max_gap):
    lib = H.oracle_lib()
    lib.oracle_xdrop_dag_pass.restype = C.c_int
    lib.oracle_xdrop_dag_pass.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    node = np.asarray(nodes, dtype=np.uint32); pred, off = _csr(preds)
    q = np.frombuffer(read.encode() + b"\0", dtype=np.uint8).copy()
    score = C.c_int32(); n_ops = C.c_uint32(); ops = np.zeros(8192, dtype=np.uint32)
    rc = lib.oracle_xdrop_dag_pass(C.byref(index.view), C.byref(scores), capi.ptr(node), len(node), capi.ptr(pred), capi.ptr(off),
                                   capi.ptr(q), len(read), start_u, start_o, max_gap, C.byref(score), capi.ptr(ops), 8192, C.byref(n_ops))
    assert rc == 0
    return score.value, [(int(w) >> 8, chr(int(w) & 0xFF)) for w in ops[: n_ops.value]]


def oracle_xdrop_dag(index, nodes, preds, read, scores, seed, max_gap):
    """seed = (node index, node offset, query offset) or None."""
    lib = H.oracle_lib()
    lib.oracle_xdrop_dag.restype = C.c_int
    lib.oracle_xdrop_dag.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                     C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    node = np.asarray(nodes, dtype=np.uint32); pred, off = _csr(preds)
    q = np.frombuffer(read.encode() + b"\0", dtype=np.uint8).copy()
    score = C.c_int32(); nm, ne = C.c_uint32(), C.c_uint32(); cells = C.c_uint64()
    maps = np.zeros(1024, dtype=H.mapping_dt); edits = np.zeros(4096, dtype=np.uint32)
    su, so, sq = (NO_SEED, 0, 0) if seed is None else seed
    rc = lib.oracle_xdrop_dag(C.byref(index.view), C.byref(scores), capi.ptr(node), len(node), capi.ptr(pred), capi.ptr(off),
                              capi.ptr(q), len(read), su, so, sq, max_gap, C.byref(score), capi.ptr(maps), 1024, C.byref(nm),
                              capi.ptr(edits), 4096, C.byref(ne), C.byref(cells))
    assert rc == 0
    return score.value, capi.decode_path(maps, edits, nm.value)


@pytest.mark.parametrize("seed,qlen,err,gap", [(1, 40, 0.03, 20), (2, 150, 0.05, 60), (3, 250, 0.08, 40), (4, 97, 0.15, 54), (5, 64, 0.3, 30)])
def test_oracle_dag_pass_equals_the_pinned_aligner_on_trees(seed, qlen, err, gap):
    rng = np.random.default_rng(seed)
    sc = capi.Scores(1, 4, 6, 1, 5)
    for _ in range(25):
        seqs, parents, trim, q = TX._random_tree_problem(rng, int(rng.integers(1, 24)), qlen, err)
        index = TX.case_index({"nodes": seqs, "parents": parents})
        nodes = [2 * (i + 1) for i in range(len(seqs))]
        want_score, want_path = TX.oracle_xdrop(index, parents, nodes, trim, q, sc, gap)
        preds = [[p] if p >= 0 else [] for p in parents]
        got_score, steps = oracle_dag_pass(index, nodes, preds, q, sc, 0, trim, gap)
        assert got_score == want_score
        # the pinned aligner's path as (tree index, op) steps, trailing soft clip dropped
        flat = []
        for node, _, edits in want_path:
            for op, ln, _b in edits:
                flat += [(node - 1, {"M": "M", "S": "X", "I": "I", "D": "D"}[op])] * ln
        aligned_q = sum(1 for _, op in steps if op != "D")
        if want_score > 0:
            keep, used = [], 0
            for st in flat:
                if st[1] != "D" and used == aligned_q:
                    break
                keep.append(st); used += st[1] != "D"
            assert steps == keep


def _linear_case():
    seqs = ["ACGTTGCA", "GGATCCAT", "TTGACCGTA", "CATGCATGG", "ATATCGCGAT", "GGCCTTAAGC"]
    index = capi.HostIndex(seqs, [[2 * (i + 1) for i in range(len(seqs))]], None, k=5, w=3)
    nodes = [2 * (i + 1) for i in range(len(seqs))]
    preds = [[i - 1] if i else [] for i in range(len(seqs))]
    return seqs, index, nodes, preds


def test_oracle_two_pass_properties_on_a_linear_graph():
    seqs, index, nodes, preds = _linear_case()
    ref = "".join(seqs)
    sc = capi.Scores(1, 4, 6, 1, 5)
    read = ref[10:40]
    # seed in the middle of the read: node 2 ("TTGACCGTA") starts at ref offset 16 = read offset 6
    score, path = oracle_xdrop_dag(index, nodes, preds, read, sc, (2, 0, 6), 20)
    assert score == len(read) + 5                      # pass 2 spans the whole read and earns the left bonus
    assert path[0][0] == 1 and path[0][1] == 2         # starts 2 bases into node 1 (ref offset 10)
    assert sum(e[1] for m in path for e in m[2] if e[0] in "MSI") == len(read)
    assert all(e[0] == "M" for m in path for e in m[2])
    # junk in front: soft clipped on the left; junk behind: soft clipped on the right
    score2, path2 = oracle_xdrop_dag(index, nodes, preds, "TTTTT" + read + "AAAAAA", sc, (2, 0, 11), 20)
    assert path2[0][2][0] == ["I", 5, ""] and path2[-1][2][-1] == ["I", 6, ""]
    assert score2 == len(read)
    # no seed: the scan of the last 15 bases finds the same placement
    score3, path3 = oracle_xdrop_dag(index, nodes, preds, read, sc, None, 20)
    assert (score3, path3) == (score, path)
    # a read that is not in the graph at all
    assert oracle_xdrop_dag(index, nodes, preds, "N" * 30, sc, None, 20) == (0, [])


def _random_dag_case(rng):
    seqs, preds, walk, q = TS._random_dag_problem(rng, int(rng.integers(2, 30)), int(rng.integers(20, 120)), 0.05)
    # a seed: an exact 8-mer shared by the query and a node of the walk, when there is one
    seed = None
    for u in walk:
        s = seqs[u]
        for o in range(0, max(0, len(s) - 7)):
            k = q.find(s[o:o + 8])
            if k >= 0:
                seed = (u, o, k); break
        if seed:
            break
    return seqs, preds, q, seed


@pytest.mark.gpu
@pytest.mark.parametrize("bonus,gap", [(5, 30), (0, 12)])
def test_cuda_xdrop_dag_parity_random_dags(bonus, gap):
    rng = np.random.default_rng(300 + bonus)
    sc = capi.Scores(1, 4, 6, 1, bonus)
    for batch in range(4):
        all_seqs, srcs, problems = [], [], []
        for _ in range(40):
            seqs, preds, q, seed = _random_dag_case(rng)
            base = len(all_seqs)
            all_seqs += seqs
            srcs.append((base, preds))
            problems.append(([2 * (base + i + 1) for i in range(len(seqs))], preds, q.encode(), seed, gap))
        paths = [[2 * (base + x + 1) for x in walk] for base, preds in srcs for walk in TS._dag_walks(preds)]
        index = capi.HostIndex(all_seqs, paths, None, k=5, w=3)
        dev = capi.Device(index, scores=sc)
        got = dev.xdrop_dag_batch(problems)
        n_seeded = 0
        for i, (nodes, preds, q, seed, g) in enumerate(problems):
            want = oracle_xdrop_dag(index, nodes, preds, q.decode(), sc, seed, g)
            assert got[i] == want, (i, q, seed, got[i], want)
            n_seeded += seed is not None
        assert 0 < n_seeded < len(problems) or batch > 0
        dev.close()


@pytest.mark.gpu
def test_cuda_xdrop_dag_linear_properties():
    seqs, index, nodes, preds = _linear_case()
    ref = "".join(seqs)
    sc = capi.Scores(1, 4, 6, 1, 5)
    dev = capi.Device(index, scores=sc)
    read = ref[10:40]
    problems = [(nodes, preds, read.encode(), (2, 0, 6), 20), (nodes, preds, ("TTTTT" + read + "AAAAAA").encode(), (2, 0, 11), 20),
                (nodes, preds, read.encode(), None, 20), (nodes, preds, b"N" * 30, None, 20)]
    got = dev.xdrop_dag_batch(problems)
    for p, g in zip(problems, got):
        assert g == oracle_xdrop_dag(index, p[0], p[1], p[2].decode(), sc, p[3], p[4])
    dev.close()


# ---- the reference's own align_xdrop vectors (src/unittest/xdrop_aligner.cpp:21-265, forward mode) ----------------
# graph of :27-38 (a SNP bubble) and of :218-228 (a long homopolymer node in front of the true locus)
_BUBBLE = {"nodes": ["AGTG", "C", "A", "TGAAGT"], "paths": [[1, 2, 4], [1, 3, 4]]}
_BUBBLE_PREDS = [[], [0], [0], [1, 2]]
_PINNED = {"nodes": ["GAAAAAAAAAAAAAAAAAAAAA", "C", "A", "TGATTACAT"], "paths": [[1, 2, 4], [1, 3, 4]]}


def _ref_align_xdrop(case, read, scores, seed, max_gap=40):
    index = TS.case_index(case)
    nodes = [2 * (i + 1) for i in range(len(case["nodes"]))]
    return oracle_xdrop_dag(index, nodes, _BUBBLE_PREDS, read, capi.Scores(*scores), seed, max_gap)


def test_reference_align_xdrop_with_no_mems():
    """:21-56 "can compute an alignment with no MEMs": score = read length, path n0, n1, n3."""
    read = "AGTGCTGAAGT"
    score, path = _ref_align_xdrop(_BUBBLE, read, (1, 4, 6, 1, 0), None)
    assert score == len(read)
    assert [m[0] for m in path] == [0, 1, 3]           # positions in the topological order: n0, n1, n3


def test_reference_align_xdrop_with_a_mem_in_the_middle():
    """:101-141: a MEM on the "GT" of the first node (read offset 1, node offset 1) seeds the same alignment."""
    read = "AGTGCTGAAGT"
    score, path = _ref_align_xdrop(_BUBBLE, read, (1, 4, 6, 1, 0), (0, 1, 1))
    assert score == len(read)
    assert [m[0] for m in path] == [0, 1, 3]           # positions in the topological order: n0, n1, n3


@pytest.mark.parametrize("seed", [(0, 1, 1), None], ids=["with a MEM", "no MEM"])
def test_reference_align_xdrop_applies_the_full_length_bonus_at_one_end_only(seed):
    """:143-209 "still incorrectly applies the full length bonus at only one end": read length + ONE bonus of 10."""
    read = "AGTGCTGAAGT"
    score, _ = _ref_align_xdrop(_BUBBLE, read, (1, 4, 6, 1, 10), seed)
    assert score == len(read) + 10


def test_reference_align_xdrop_can_be_induced_to_pin_with_mems():
    """:211-265: without a MEM the optimal alignment (one mapping on the last node, score 7) is found; a MEM on the
    initial G of the homopolymer node forces the alignment onto that node."""
    read = "GATTACA"
    score, path = _ref_align_xdrop(_PINNED, read, (1, 4, 6, 1, 0), None)
    assert score == len(read) and [m[0] for m in path] == [3]
    score, path = _ref_align_xdrop(_PINNED, read, (1, 4, 6, 1, 0), (0, 0, 0))
    assert [m[0] for m in path] == [0]


def test_reference_align_xdrop_hard_to_find_a_seed_does_not_crash():
    """:764-779: a 150 bp read against 27 TA-rich 32 bp nodes in a line, no MEMs: any outcome, no crash."""
    seqs = ["ATTTATATATATATTTATATATATATTTATAT", "ATATATTTATATATTTTTATATATTATATATT", "TATATATATATTTATATATTATATATATATTT", "ATATATTTATATATATATTTATATATATTTAT",
            "ATATATATTTATATATATTTATATATATATTT", "ATATATATATATTTATATATATTTATATATTA", "TTTATATATATTTATATATATATTTATATATA", "TTTATATATATATATTTATATATATATATTTA",
            "TATATATATTTATATATATATTTATATATATA", "TTTATATATATATTTATATATATATTTATATA", "TATATTTATATATATATATTATATATATATAT", "TTATATATATATTTATATATATATTTATATAT",
            "ATATATATATATTTATATATATATTTATATAT", "ATATTTATATATATATATTTATATATATATTT", "ATATATATATTTATATATATATTATTTATATA", "TATATTTATATATATATTATATATATATTTAT",
            "ATATATATATTATATATATATTTATATATATA", "TTTATATATATATTTATATATATATATTATAT", "ATATATTTATATATATATTTATATATATATTT", "ATATATATATTTATATATATATTTATATATAT",
            "ATTTATATATATATTTATATATATATTTATAT", "ATATATTATATATATATTTATATATATATTTA", "TATATATATTTATATATATATTTATATATATA", "TTTATATATATTTATATATATATTTATATATA",
            "TATTTATATATATATTTATATATATTTATATA", "TATATTTATATATATATATATATATTTATATA", "TATATTTATATATATTTATATATATATTTATA"]
    case = {"nodes": seqs, "paths": [list(range(1, len(seqs) + 1))]}
    read = ("CAGCACTTTGGGAGGCCAAGGTGGGTGGATCATCTGAGGTCAGGAGTTTGAGACCAGCCTGACCAACATGGTGAAATCCTGTCTCTACTGAAAATACTAAAATTAGCCAGGCGTGGCGGCCAGTGCCTGTAATCCCGGCTACTGGGGAGG")
    index = TS.case_index(case)
    nodes = [2 * (i + 1) for i in range(len(seqs))]
    preds = [[]] + [[i] for i in range(len(seqs) - 1)]
    score, path = oracle_xdrop_dag(index, nodes, preds, read, capi.Scores(1, 4, 6, 1, 10), None, 40)
    if path:
        assert sum(ed[1] for m in path for ed in m[2] if ed[0] in "MSI") == len(read)
