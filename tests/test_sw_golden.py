"""Pin the oracle's full-DP local aligner (the GSSW replacement, oracle/full_dp.cpp) against the
reference's own unit vectors (src/unittest/aligner.cpp; tests/golden/sw_local.json), and the CUDA
stage seam gb_sw_batch against the oracle."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
from vg_b200 import capi

GOLD = H.load_golden("sw_local.json")


def oracle_sw(index, problem, read, scores):
    lib = H.oracle_lib()
    lib.oracle_sw_local.restype = C.c_int
    lib.oracle_sw_local.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                    C.c_void_p, C.c_void_p]
    node = np.asarray(problem["node"], dtype=np.uint32)
    pred = np.asarray([p for ps in problem["pred"] for p in ps] + [0], dtype=np.uint32)
    pred_off = np.zeros(len(node) + 1, dtype=np.uint32)
    pred_off[1:] = np.cumsum([len(ps) for ps in problem["pred"]])
    q = np.frombuffer(read.encode() + b"\0", dtype=np.uint8).copy()
    score = C.c_int32(); nm, ne = C.c_uint32(), C.c_uint32(); cells = C.c_uint64()
    maps = np.zeros(1024, dtype=H.mapping_dt); edits = np.zeros(4096, dtype=np.uint32)
    rc = lib.oracle_sw_local(C.byref(index.view), C.byref(scores), capi.ptr(node), len(node), capi.ptr(pred), capi.ptr(pred_off),
                             capi.ptr(q), len(read), C.byref(score), capi.ptr(maps), 1024, C.byref(nm), capi.ptr(edits), 4096,
                             C.byref(ne), C.byref(cells))
    assert rc == 0
    return score.value, capi.decode_path(maps, edits, nm.value), cells.value


def case_index(case):
    return capi.HostIndex(case["nodes"], [[2 * i for i in p] for p in case["paths"]], None, k=5, w=3)


def check_consistency(path, read):
    assert sum(ed[1] for m in path for ed in m[2] if ed[0] in "MSI") == len(read)


@pytest.mark.parametrize("case", GOLD["cases"], ids=[c["name"] for c in GOLD["cases"]])
def test_oracle_sw_matches_reference_vectors(case):
    index = case_index(case)
    score, path, _ = oracle_sw(index, case["problem"], case["read"], capi.Scores(*case["scores"]))
    assert score == case["score"]
    if "path" in case:
        assert path == case["path"]
    if "lengths" in case:
        got = [[sum(e[1] for e in m[2] if e[0] in "MSD"), sum(e[1] for e in m[2] if e[0] in "MSI")] for m in path]
        assert got == case["lengths"]
    if path:
        check_consistency(path, case["read"])


def _py_local_score(ref, q, sc):
    """Independent O(n m) Gotoh local alignment of q against the linear sequence ref with the same
    scoring rules (N pairs score 0, bonus at each attached read end); score only."""
    match, mismatch, go, ge, bonus = sc
    NEG = -10 ** 9
    m = len(q)
    Hp = [0] * (m + 1); Ep = [NEG] * (m + 1)
    best = 0
    for r in ref:
        H = [0] * (m + 1); E = [NEG] * (m + 1); F = NEG
        for j in range(1, m + 1):
            s = 0 if (r not in "ACGT" or q[j - 1] not in "ACGT") else (match if r == q[j - 1] else -mismatch)
            d = (bonus if j == 1 else max(Hp[j - 1], 0)) + s
            e = max(Hp[j] - go, Ep[j] - ge)
            F = max(H[j - 1] - go, F - ge)
            H[j] = max(d, e, F, 0); E[j] = e
            best = max(best, H[j], d + bonus if j == m else 0)
        Hp, Ep = H, E
    return best


def _random_dag_problem(rng, n_nodes, qlen, err):
    """A random layered DAG (bubbles) with a query following one walk with errors and soft-clipped junk."""
    seqs, preds, layer_of = [], [], []
    prev_layer = []
    walk = []
    while len(seqs) < n_nodes:
        width = int(rng.integers(1, 4))
        layer = []
        for _ in range(width):
            if len(seqs) >= n_nodes:
                break
            ln = int(rng.integers(1, 12))
            seqs.append("".join(rng.choice(list("ACGT"), size=ln)))
            preds.append(sorted(set(int(x) for x in rng.choice(prev_layer, size=min(len(prev_layer), int(rng.integers(1, 3))), replace=False))) if prev_layer else [])
            layer.append(len(seqs) - 1)
        prev_layer = layer
    # a walk: follow predecessor links backwards from a random last-layer node
    x = int(rng.choice(prev_layer))
    while True:
        walk.append(x)
        if not preds[x]:
            break
        x = int(rng.choice(preds[x]))
    walk.reverse()
    hap = "".join(seqs[i] for i in walk)
    start = int(rng.integers(0, max(1, len(hap) - qlen)))
    q = list(hap[start:start + qlen])
    for i in range(len(q)):
        if rng.random() < err:
            q[i] = str(rng.choice(list("ACGTN")))
    if rng.random() < 0.3 and len(q) > 8:
        del q[int(rng.integers(2, len(q) - 2))]
    if rng.random() < 0.3 and len(q) > 8:
        q.insert(int(rng.integers(2, len(q) - 2)), str(rng.choice(list("ACGT"))))
    if rng.random() < 0.3:
        q = list(rng.choice(list("ACGT"), size=int(rng.integers(1, 6)))) + q
    return seqs, preds, walk, "".join(q)


def _dag_walks(preds):
    """Walks (lists of node indices) that together cover every node and every edge of the DAG."""
    n = len(preds)
    succ = {i: [] for i in range(n)}
    for v, ps in enumerate(preds):
        for p in ps:
            succ[p].append(v)

    def back(v):
        w = [v]
        while preds[w[-1]]:
            w.append(preds[w[-1]][0])
        return w[::-1]

    def fwd(v):
        w = []
        while succ[v]:
            v = succ[v][0]; w.append(v)
        return w
    walks = []
    for v, ps in enumerate(preds):
        if not ps:
            walks.append([v] + fwd(v))
        for p in ps:
            walks.append(back(p) + [v] + fwd(v))
    return walks


def test_oracle_sw_score_matches_an_independent_dp_on_linear_graphs():
    rng = np.random.default_rng(12)
    for trial in range(60):
        n_nodes = int(rng.integers(1, 8))
        seqs = ["".join(rng.choice(list("ACGTN"), p=[0.24, 0.24, 0.24, 0.24, 0.04], size=int(rng.integers(1, 20)))) for _ in range(n_nodes)]
        ref = "".join(seqs)
        start = int(rng.integers(0, max(1, len(ref) - 5)))
        q = list(ref[start:start + int(rng.integers(1, 40))])
        for i in range(len(q)):
            if rng.random() < 0.1:
                q[i] = str(rng.choice(list("ACGTN")))
        if rng.random() < 0.4 and len(q) > 6:
            del q[len(q) // 2]
        if rng.random() < 0.4:
            q = ["T", "T"] + q
        q = "".join(q)
        sc = [1, 4, 6, 1, int(rng.choice([0, 5, 10]))]
        index = capi.HostIndex(seqs, [[2 * (i + 1) for i in range(n_nodes)]], None, k=5, w=3)
        problem = {"node": [2 * (i + 1) for i in range(n_nodes)], "pred": [[i - 1] if i else [] for i in range(n_nodes)]}
        score, path, _ = oracle_sw(index, problem, q, capi.Scores(*sc))
        assert score == _py_local_score(ref, q, sc), (seqs, q, sc)
        if path:
            check_consistency(path, q)


@pytest.mark.gpu
def test_cuda_sw_matches_reference_vectors_and_oracle():
    for case in GOLD["cases"]:
        index = case_index(case)
        dev = capi.Device(index, scores=capi.Scores(*case["scores"]))
        want = oracle_sw(index, case["problem"], case["read"], capi.Scores(*case["scores"]))
        got = dev.sw_batch([(case["problem"]["node"], case["problem"]["pred"], case["read"].encode())])[0]
        assert got[0] == case["score"], case["name"]
        assert (got[0], got[1]) == (want[0], want[1]), case["name"]
        dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bonus", [0, 5])
def test_cuda_sw_parity_random_dags(bonus):
    rng = np.random.default_rng(77 + bonus)
    sc = capi.Scores(1, 4, 6, 1, bonus)
    for batch in range(4):
        # each problem gets its own small index: build one graph holding all the batch's DAGs side by side
        all_seqs, all_paths_src, problems, queries = [], [], [], []
        for _ in range(40):
            seqs, preds, walk, q = _random_dag_problem(rng, int(rng.integers(2, 30)), int(rng.integers(5, 120)), 0.05)
            base = len(all_seqs)
            all_seqs += seqs
            all_paths_src.append((base, preds))
            problems.append(([2 * (base + i + 1) for i in range(len(seqs))], preds, q.encode()))
        paths = [[2 * (base + x + 1) for x in walk] for base, preds in all_paths_src for walk in _dag_walks(preds)]
        index = capi.HostIndex(all_seqs, paths, None, k=5, w=3)
        dev = capi.Device(index, scores=sc)
        got = dev.sw_batch(problems)
        for i, (nodes, preds, q) in enumerate(problems):
            want = oracle_sw(index, {"node": nodes, "pred": preds}, q.decode(), sc)
            assert got[i] == (want[0], want[1]), (i, q, got[i], want[:2])
        dev.close()
