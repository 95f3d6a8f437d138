"""Pin the oracle's banded global aligner (Aligner::align_global_banded, oracle/banded_global.cpp)
against the reference's own unit vectors (src/unittest/banded_global_aligner.cpp, regular scoring
1/4/6/1 unless stated), and the CUDA stage seam gb_banded_global_batch against the oracle.

Transcribed (31 vectors):
  * all edit types (:22): every section but the doubly-reversing edge;
  * graph structures (:827): path lengths, singleton, masked node, multiple sources, multiple sinks,
    multiple sources and sinks, separated graph;
  * banding edge cases (:1194): all three (the 100s case as its own test: it asserts a score bound);
  * permissive banding (:1342): both sections;
  * big indel on a tiny graph (:1635, its own test, with its empty end nodes dropped);
  * Ns (:2372): Ns to letters and Ns to Ns;
  * empty reads (:3229): the graph with one path and the graph with multiple paths.
Not transcribed:
  * the doubly-reversing edge (:75): a problem lists each node in one orientation;
  * the graph that is not topologically sorted (:913): the caller gives the topological order;
  * letters to Ns (:2410): the section rewrites the graph's sequences in ways this table cannot pose;
  * quality-adjusted alignment (:1456): giraffe never uses the quality-adjusted aligners;
  * alternate alignments (:1672): align_global_banded here returns one alignment;
  * empty nodes (:2480, :3338, :3407, :3516) and the int-width edge (:3545, whose graph is two empty
    nodes joined by an edge plus a path of letters): flat-index nodes are never empty.
"""
import ctypes as C

import numpy as np
import pytest

import helpers as H
from test_sw_golden import _dag_walks, _random_dag_problem
from vg_b200 import capi

SCORES = capi.Scores(1, 4, 6, 1, 0)
DIAMOND = [(0, 1), (0, 2), (1, 3), (2, 3)]


def M(n): return ["M", n, ""]
def D(n): return ["D", n, ""]
def I(n): return ["I", n, ""]
def S(b): return ["S", 1, b]


# (name, node sequences, edges, read, band padding, permissive, expected path [[node, [edits]]] or None, score or None)
CASES = [
    ("exact_match", ["AGTG", "C", "A", "TGAAGT"], DIAMOND, "AGTGCTGAAGT", 1, False, [[0, [M(4)]], [1, [M(1)]], [3, [M(6)]]], 11),
    ("mismatch", ["CCCAGTT", "C", "A", "TGAAGT"], DIAMOND, "CCCAGTGCTGAAGT", 1, True, [[0, [M(6), S("G")]], [1, [M(1)]], [3, [M(6)]]], 9),
    ("single_deletion", ["CCCAGATG", "C", "A", "TGAAGT"], DIAMOND, "CCCAGTGCTGAAGT", 2, False,
     [[0, [M(5), D(1), M(2)]], [1, [M(1)]], [3, [M(6)]]], 14 - 6),
    ("multi_deletion", ["AACCCAGATG", "C", "A", "TGAAGT"], DIAMOND, "AACCCAGGCTGAAGT", 2, False,
     [[0, [M(7), D(2), M(1)]], [1, [M(1)]], [3, [M(6)]]], 15 - 7),
    ("lead_insertion", ["AACCCAGG", "CA", "AT", "TGAAGT"], DIAMOND, "TAACCCAGGCATGAAGT", 2, False,
     [[0, [I(1), M(8)]], [1, [M(2)]], [3, [M(6)]]], 16 - 6),
    ("lead_multi_deletion", ["AACCCAGG", "CA", "AT", "TGAAGT"], DIAMOND, "CCCAGGCATGAAGT", 2, False,
     [[0, [D(2), M(6)]], [1, [M(2)]], [3, [M(6)]]], 14 - 7),
    ("multiple_sources", ["AGTG", "CGCC", "ATTA"], [(0, 2), (1, 2)], "AGTGATTA", 1, False, [[0, [M(4)]], [2, [M(4)]]], 8),
    ("band_one_base_wide", ["AGTG", "C", "A", "TGAAGT"], DIAMOND, "AGTGCTGAAGT", 0, False, [[0, [M(4)]], [1, [M(1)]], [3, [M(6)]]], 11),
    ("permissive_outside_band", ["AGTG", "CTGGTGTAGTA", "AATTCCCCCGG", "TGAAGT"], DIAMOND, "AGTGAATTGGTGAAGT", 0, True,
     [[0, [M(4)]], [2, [M(4), D(5), M(2)]], [3, [M(6)]]], 16 - 10),
    ("single_insertion", ["AACCCAGG", "C", "A", "TGAAGT"], DIAMOND, "AACCCAGAGCTGAAGT", 2, False,
     [[0, [M(7), I(1), M(1)]], [1, [M(1)]], [3, [M(6)]]], 15 - 6),
    ("multi_insertion", ["AACCCAGG", "C", "A", "TGAAGT"], DIAMOND, "AACCCAGATGCTGAAGT", 2, False,
     [[0, [M(7), I(2), M(1)]], [1, [M(1)]], [3, [M(6)]]], 15 - 7),
    ("deletion_across_node_boundary", ["AACCCAGG", "CA", "AT", "TGAAGT"], DIAMOND, "AACCCAGATGAAGT", 2, False,
     [[0, [M(7), D(1)]], [1, [D(1), M(1)]], [3, [M(6)]]], 14 - 7),
    ("lead_multi_insertion", ["AACCCAGG", "CA", "AT", "TGAAGT"], DIAMOND, "TGAACCCAGGCATGAAGT", 2, False,
     [[0, [I(2), M(8)]], [1, [M(2)]], [3, [M(6)]]], 16 - 7),
    ("lead_single_deletion", ["AACCCAGG", "CA", "AT", "TGAAGT"], DIAMOND, "ACCCAGGCATGAAGT", 2, False,
     [[0, [D(1), M(7)]], [1, [M(2)]], [3, [M(6)]]], 15 - 6),
    ("lead_deletion_across_node_boundary", ["AA", "CCCAGGCA", "GTGCTATA", "TGAAGT"], DIAMOND, "CCAGGCATGAAGT", 3, False,
     [[0, [D(2)]], [1, [D(1), M(7)]], [3, [M(6)]]], 13 - 8),
    ("lead_deletion_ending_at_node_boundary", ["A", "C"], [(0, 1)], "C", 1, True, [[0, [D(1)]], [1, [M(1)]]], 1 - 6),
    ("long_lead_deletion_ending_at_node_boundary", ["AATG", "C"], [(0, 1)], "C", 1, True, [[0, [D(4)]], [1, [M(1)]]], 1 - 9),
    ("paths_of_different_lengths", ["TG", "TGGC", "AAA", "AGT"], DIAMOND, "TGTGGCAGT", 1, False, [[0, [M(2)]], [1, [M(4)]], [3, [M(3)]]], 9),
    ("singleton_graph", ["C"], [], "A", 1, True, [[0, [S("A")]]], -4),
    ("masked_node", ["TG", "TGGC", "A", "AGT"], DIAMOND, "TGTGGCAGT", 1, False, [[0, [M(2)]], [1, [M(4)]], [3, [M(3)]]], 9),
    ("multiple_sinks", ["AGTG", "C", "A"], [(0, 1), (0, 2)], "AGTGC", 1, False, [[0, [M(4)]], [1, [M(1)]]], 5),
    ("multiple_sources_and_sinks", ["AGTG", "CGCC", "T", "TGGG", "GTTA"], [(0, 2), (1, 2), (2, 3), (2, 4)], "AGTGTTGGG", 1, False,
     [[0, [M(4)]], [2, [M(1)]], [3, [M(4)]]], 9),
    ("separated_graph", ["AGTG", "CGCC", "GTTA", "TGGG"], [(0, 1), (2, 3)], "AGTGCGCC", 1, False, [[0, [M(4)]], [1, [M(4)]]], 8),
    ("band_wider_than_read", ["CAGGA", "AA", "GTGTATA", "TGAAGT"], DIAMOND, "CAGGAAATGAAGT", 20, False,
     [[0, [M(5)]], [1, [M(2)]], [3, [M(6)]]], 13),
    ("runs_with_permissive_banding", ["AGTG", "C", "A", "TGAAGT"], DIAMOND, "AGTGCTGAAGT", 1, True, [[0, [M(4)]], [1, [M(1)]], [3, [M(6)]]], 11),
    ("ns_to_ns", ["NNNG", "C", "A", "TGANNN"], DIAMOND, "NNNGCTGANNN", 1, True, [[0, [M(4)]], [1, [M(1)]], [3, [M(6)]]], 5),
    ("empty_read_one_path", ["A", "G", "T"], [(0, 1), (1, 2)], "", 1, True, [[0, [D(1)]], [1, [D(1)]], [2, [D(1)]]], -8),
    ("ns_to_letters", ["AGTG", "C", "A", "TGAAGT"], DIAMOND, "NNNGCTGANNN", 1, True, None, 5),
    ("empty_read_multiple_paths", ["A", "G", "TC", "C"], DIAMOND, "", 1, True, [[0, [D(1)]], [1, [D(1)]], [3, [D(1)]]], -8),
]


def problem_of(nodes, edges):
    preds = [[] for _ in nodes]
    for a, b in edges:
        preds[b].append(a)
    return [2 * (i + 1) for i in range(len(nodes))], preds


def oracle_banded(index, node, preds, read, pad, permissive, scores=SCORES):
    lib = H.oracle_lib()
    lib.oracle_banded_global.restype = C.c_int
    lib.oracle_banded_global.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), C.c_void_p, C.c_uint32, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32, C.c_int, C.c_void_p, C.c_void_p, C.c_uint32,
                                         C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    node = np.asarray(node, dtype=np.uint32)
    pred = np.asarray([p for ps in preds for p in ps] + [0], dtype=np.uint32)
    pred_off = np.zeros(len(node) + 1, dtype=np.uint32)
    pred_off[1:] = np.cumsum([len(ps) for ps in preds])
    q = np.frombuffer(read.encode() + b"\0", dtype=np.uint8).copy()
    score = C.c_int32(); nm, ne = C.c_uint32(), C.c_uint32(); cells = C.c_uint64()
    maps = np.zeros(1024, dtype=H.mapping_dt); edits = np.zeros(8192, dtype=np.uint32)
    rc = lib.oracle_banded_global(C.byref(index.view), C.byref(scores), capi.ptr(node), len(node), capi.ptr(pred), capi.ptr(pred_off),
                                  capi.ptr(q), len(read), pad, int(permissive), C.byref(score), capi.ptr(maps), 1024, C.byref(nm),
                                  capi.ptr(edits), 8192, C.byref(ne), C.byref(cells))
    assert rc in (0, 1)
    status = capi.GB_ITEM_NO_BAND if rc == 1 else capi.GB_ITEM_OK
    return status, score.value, capi.decode_path(maps, edits, nm.value)


def path_score(path, seqs, node_of, read, sc):
    """Rescore a global path independently: matches / mismatches (N pairs 0) and affine gaps."""
    match, mismatch, go, ge = sc[0], sc[1], sc[2], sc[3]
    total, q, prev = 0, 0, None
    for node, off, edits in path:
        ref = seqs[node_of[node]]
        r = off
        for op, n, _ in edits:
            cont = prev == op
            prev = op
            if op in "ID" and cont:
                # the same gap continuing into the next node
                total -= n * ge; q += n if op == "I" else 0; r += n if op == "D" else 0
            elif op in "MS":
                for _ in range(n):
                    a, b = read[q], ref[r]
                    total += 0 if (a not in "ACGT" or b not in "ACGT") else (match if a == b else -mismatch)
                    q += 1; r += 1
            elif op == "I":
                total -= go + (n - 1) * ge; q += n
            else:
                total -= go + (n - 1) * ge; r += n
        assert r == len(ref), "global alignment covers whole nodes"
    assert q == len(read)
    return total


def _index_for(nodes, edges):
    node, preds = problem_of(nodes, edges)
    paths = [[node[x] for x in w] for w in _dag_walks(preds)] or [[node[0]]]
    return capi.HostIndex(nodes, paths, None, k=5, w=3), node, preds


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_banded_matches_reference_vectors(case):
    name, nodes, edges, read, pad, permissive, want_path, want_score = case
    index, node, preds = _index_for(nodes, edges)
    status, score, path = oracle_banded(index, node, preds, read, pad, permissive)
    assert status == capi.GB_ITEM_OK
    if want_score is not None:
        assert score == want_score
    if want_path is not None:
        assert [[p[0], p[2]] for p in path] == want_path
    assert all(p[1] == 0 for p in path)
    if read:
        assert path_score(path, nodes, list(range(len(nodes))), read, [1, 4, 6, 1]) == score


def test_oracle_banded_big_indel_on_tiny_graph():
    """banded_global_aligner.cpp:1635: GT -> G between two empty nodes (dropped here: flat-index nodes
    are never empty and they carry no sequence), scores 10 / 40 / 61 / 10: 3 matches, one gap of 8."""
    nodes, edges = ["GT", "G"], [(0, 1)]
    index, node, preds = _index_for(nodes, edges)
    status, score, path = oracle_banded(index, node, preds, "GTGTGTGTGTG", 1, True, capi.Scores(10, 40, 61, 10, 50))
    assert status == capi.GB_ITEM_OK
    assert score == 3 * 10 + 1 * -61 + 7 * -10
    assert path_score(path, nodes, [0, 1], "GTGTGTGTGTG", [10, 40, 61, 10]) == score


def test_oracle_banded_scores_in_the_100s():
    """banded_global_aligner.cpp:1299: one base against 300 A's in six nodes (an int8 score would wrap)."""
    nodes = ["A" * 50] * 6
    index, node, preds = _index_for(nodes, [(i, i + 1) for i in range(5)])
    status, score, path = oracle_banded(index, node, preds, "C", 1, True)
    assert status == capi.GB_ITEM_OK
    assert score < -128
    assert path_score(path, nodes, list(range(6)), "C", [1, 4, 6, 1]) == score


def test_oracle_banded_refuses_a_band_that_reaches_no_sink():
    nodes, edges = ["AGTG", "CTGGTGTAGTA", "AATTCCCCCGG", "TGAAGT"], DIAMOND
    index, node, preds = _index_for(nodes, edges)
    status, score, path = oracle_banded(index, node, preds, "AGTGAATTGGTGAAGT", 0, False)
    assert (status, score, path) == (capi.GB_ITEM_NO_BAND, 0, [])


def _py_global_score(ref, q, sc):
    """Independent unbanded global Gotoh of q against a linear reference (all gap adjacencies open anew)."""
    match, mismatch, go, ge = sc
    NEG = -10 ** 9
    n, m = len(ref), len(q)
    Mx = [[NEG] * (m + 1) for _ in range(n + 1)]
    Ix = [[NEG] * (m + 1) for _ in range(n + 1)]
    Dx = [[NEG] * (m + 1) for _ in range(n + 1)]
    Mx[0][0] = 0
    for c in range(n + 1):
        for j in range(m + 1):
            if c == 0 and j == 0:
                continue
            if c > 0 and j > 0:
                a, b = q[j - 1], ref[c - 1]
                s = 0 if (a not in "ACGT" or b not in "ACGT") else (match if a == b else -mismatch)
                Mx[c][j] = s + max(Mx[c - 1][j - 1], Ix[c - 1][j - 1], Dx[c - 1][j - 1])
            if c > 0:
                Dx[c][j] = max(Mx[c - 1][j] - go, Ix[c - 1][j] - go, Dx[c - 1][j] - ge)
            if j > 0:
                Ix[c][j] = max(Mx[c][j - 1] - go, Ix[c][j - 1] - ge, Dx[c][j - 1] - go)
    return max(Mx[n][m], Ix[n][m], Dx[n][m])


def test_oracle_banded_wide_band_equals_an_independent_global_dp_on_linear_graphs():
    rng = np.random.default_rng(31)
    for trial in range(60):
        k = int(rng.integers(1, 6))
        seqs = ["".join(rng.choice(list("ACGTN"), p=[0.24, 0.24, 0.24, 0.24, 0.04], size=int(rng.integers(1, 12)))) for _ in range(k)]
        ref = "".join(seqs)
        q = list(ref)
        for i in range(len(q)):
            if rng.random() < 0.1:
                q[i] = str(rng.choice(list("ACGT")))
        if rng.random() < 0.5 and len(q) > 3:
            del q[int(rng.integers(1, len(q) - 1))]
        if rng.random() < 0.5:
            q.insert(int(rng.integers(0, len(q) + 1)), "T")
        q = "".join(q)
        if not q:
            continue
        index, node, preds = _index_for(seqs, [(i, i + 1) for i in range(k - 1)])
        status, score, path = oracle_banded(index, node, preds, q, len(ref) + len(q) + 2, False)
        assert status == capi.GB_ITEM_OK
        assert score == _py_global_score(ref, q, [1, 4, 6, 1]), (seqs, q)
        assert path_score(path, seqs, list(range(k)), q, [1, 4, 6, 1]) == score


@pytest.mark.gpu
def test_cuda_banded_matches_reference_vectors_and_oracle():
    extra = [("big_indel_on_tiny_graph", ["GT", "G"], [(0, 1)], "GTGTGTGTGTG", 1, True, capi.Scores(10, 40, 61, 10, 50)),
             ("scores_in_the_100s", ["A" * 50] * 6, [(i, i + 1) for i in range(5)], "C", 1, True, SCORES)]
    for name, nodes, edges, read, pad, permissive, sc in [c[:6] + (SCORES,) for c in CASES] + extra:
        index, node, preds = _index_for(nodes, edges)
        dev = capi.Device(index, scores=sc)
        # a padding far beyond the graph and the read gives the same alignment as one that just covers them
        for p in (pad, 2 ** 31 - 1):
            got = dev.banded_global_batch([(node, preds, read.encode(), p, permissive)])[0]
            assert got == oracle_banded(index, node, preds, read, p, permissive, sc), (name, p)
        dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("permissive", [False, True])
def test_cuda_banded_parity_random_dags(permissive):
    rng = np.random.default_rng(101 + int(permissive))
    n_ok = n_refused = 0
    for batch in range(4):
        all_seqs, sources, problems = [], [], []
        for _ in range(60):
            seqs, preds, walk, q = _random_dag_problem(rng, int(rng.integers(2, 30)), int(rng.integers(5, 150)), 0.05)
            base = len(all_seqs)
            all_seqs += seqs
            sources.append((base, preds))
            pad = int(rng.choice([0, 1, 3, 8, 20, 200, 2 ** 31 - 1]))
            if rng.random() < 0.1:
                q = ""
            problems.append(([2 * (base + i + 1) for i in range(len(seqs))], preds, q.encode(), pad, permissive))
        paths = [[2 * (base + x + 1) for x in w] for base, preds in sources for w in _dag_walks(preds)]
        index = capi.HostIndex(all_seqs, paths, None, k=5, w=3)
        dev = capi.Device(index, scores=SCORES)
        got = dev.banded_global_batch(problems)
        for i, (nodes, preds, q, pad, perm) in enumerate(problems):
            want = oracle_banded(index, nodes, preds, q.decode(), pad, perm)
            assert got[i] == want, (i, q, pad, got[i], want)
            n_ok += want[0] == capi.GB_ITEM_OK
            n_refused += want[0] == capi.GB_ITEM_NO_BAND
        dev.close()
    assert n_ok > 100
    if not permissive:
        assert n_refused > 0
