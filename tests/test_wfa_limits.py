"""gb_wfa_batch (WFAExtender::connect / suffix / prefix) at every limit of its fixed per-problem workspace, and
against a plain gap-affine DP that shares no code with the kernel or the oracle.

The oracle (oracle/wfa.cpp) follows the kernel statement by statement, so GPU == oracle alone cannot catch a
mistake both make.  Here:
- a numpy Gotoh DP in WFA penalty units over every haplotype string a problem admits decides whether an alignment
  within the score bound exists and what it costs (tie-proof: no particular optimal path is compared);
- oracle_wfa_workspace reports what the kernel's workspace needs for a problem; `predict` turns that into the
  status (-1 / 0 / 1) the kernel must return, and the GPU must return exactly that;
- output caps set to exactly the answer's counts must fit, one below must not.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np
import pytest

import helpers as H
from vg_b200 import capi, synth

OPS = "MXID"
DEFAULT_SCORES = (1, 4, 6, 1, 5)
DEFAULT_MODEL = [0.03, 1, 6, 0.05, 1, 10, 0.1, 1, 20, 0.1, 10, 200]      # WFAExtender::ErrorModel defaults
NO_PRUNE = [0, 100000, 100000]                                             # distance band that never prunes

# gb_wfa_batch's per-problem workspace (giraffe_b200.h): field of the oracle's report -> largest value that fits
# (and min_diagonal >= -1024, checked in over_limits)
WORKSPACE_FIELDS = ["trie_nodes", "seq_bytes", "path_entries", "points", "scores", "max_score", "min_diagonal",
                    "max_diagonal", "max_seq_offset", "max_node_offset", "max_successors"]
LIMITS = {"trie_nodes": 64, "seq_bytes": 24576, "path_entries": 2048, "points": 3071, "scores": 512, "max_score": 8191,
          "max_diagonal": 1023, "max_seq_offset": 0xFFFF, "max_node_offset": 0xFFFF, "max_successors": 32}
SMALL_TABLE_POINTS = 191


def revcomp(s: str) -> str:
    return s[::-1].translate(str.maketrans("ACGT", "TGCA"))


class Graph:
    """Node sequences (node id i + 1) and haplotypes as oriented node walks (2 * id + reverse)."""

    def __init__(self, node_seqs, paths, index=None, acyclic=True, name=""):
        self.node_seqs, self.paths, self.acyclic, self.name = list(node_seqs), [list(p) for p in paths], acyclic, name
        self._index = index

    @classmethod
    def of(cls, sg: synth.SynthGraph):
        g = cls(sg.node_seqs, sg.paths, name=sg.name)
        g.synth = sg
        return g

    @property
    def index(self):
        if self._index is None:
            self._index = capi.HostIndex(self.node_seqs, self.paths, None, k=5, w=3)
        return self._index

    def seq(self, v):
        s = self.node_seqs[(v >> 1) - 1]
        return revcomp(s) if v & 1 else s

    @functools.cached_property
    def walks(self):
        """Every haplotype in both orientations."""
        return self.paths + [[v ^ 1 for v in reversed(p)] for p in self.paths]

    @functools.cached_property
    def edges(self):
        return {(a, b) for w in self.walks for a, b in zip(w, w[1:])}

    def valid(self, v):
        return 2 <= v < 2 * (len(self.node_seqs) + 1)


# ---------------------------------------------------------------------------------------------------------------
# oracle bindings
# ---------------------------------------------------------------------------------------------------------------
def _lib():
    lib = H.oracle_lib()
    vp, u32 = C.c_void_p, C.c_uint32
    head = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), vp, C.c_int, vp, u32, u32, u32, u32, u32]
    lib.oracle_wfa.restype = C.c_int
    lib.oracle_wfa.argtypes = head + [vp] * 5 + [vp, u32, vp, vp, u32, vp]
    lib.oracle_wfa_workspace.restype = None
    lib.oracle_wfa_workspace.argtypes = head + [vp]
    return lib


def _args(g, scores, em, prob):
    mode, seq, frm, to = prob
    q = np.frombuffer(bytes(seq) + b"\0", dtype=np.uint8).copy()
    e = None if em is None else np.asarray(em, dtype=np.float64)
    frm, to = frm or (0, 0), to or (0, 0)
    return (q, e), [C.byref(g.index.view), C.byref(capi.Scores(*scores)), None if e is None else capi.ptr(e), mode, capi.ptr(q),
                    len(seq), frm[0], frm[1], to[0], to[1]]


_CAP = 1 << 17
_PATH, _EDITS = np.zeros(_CAP, dtype=np.uint32), np.zeros(_CAP, dtype=np.uint32)


def oracle_run(g, scores, em, prob):
    """The oracle's answer in Device.wfa_batch's format (ok 0 / 1)."""
    keep, args = _args(g, scores, em, prob)
    ok, score = C.c_int32(), C.c_int32()
    noff, soff, length, npath, nedits = (C.c_uint32() for _ in range(5))
    rc = _lib().oracle_wfa(*args, C.byref(ok), C.byref(score), C.byref(noff), C.byref(soff), C.byref(length),
                           capi.ptr(_PATH), _CAP, C.byref(npath), capi.ptr(_EDITS), _CAP, C.byref(nedits))
    assert rc == 0
    if not ok.value:
        return {"ok": 0, "score": 0, "node_offset": 0, "seq_offset": 0, "length": 0, "path": [], "edits": []}
    return {"ok": 1, "score": score.value, "node_offset": noff.value, "seq_offset": soff.value, "length": length.value,
            "path": [int(x) for x in _PATH[: npath.value]], "edits": [(OPS[int(w) & 3], int(w) >> 2) for w in _EDITS[: nedits.value]]}


def oracle_workspace(g, scores, em, prob):
    keep, args = _args(g, scores, em, prob)
    out = np.zeros(len(WORKSPACE_FIELDS), dtype=np.int32)
    _lib().oracle_wfa_workspace(*args, capi.ptr(out))
    return dict(zip(WORKSPACE_FIELDS, (int(x) for x in out)))


def over_limits(ws):
    """The workspace limits a problem exceeds (the kernel follows the oracle's trajectory until it stops, so these
    are exactly the limits it meets)."""
    bad = [f for f, cap in LIMITS.items() if ws[f] > cap]
    if ws["min_diagonal"] < -1024:
        bad.append("min_diagonal")
    return bad


def predict(ws, want, path_cap=512, edit_cap=512):
    """The kernel's status for a problem: -1 when the workspace or an output cap does not hold it."""
    if over_limits(ws):
        return -1
    if want["ok"] and (len(want["path"]) > path_cap or len(want["edits"]) > edit_cap):
        return -1
    return want["ok"]


# ---------------------------------------------------------------------------------------------------------------
# independent reference: Gotoh over the haplotype strings a problem admits
# ---------------------------------------------------------------------------------------------------------------
_BIG = 1 << 40


def penalties(scores):
    m, x, o, e, _ = scores
    return 2 * (m + x), 2 * (o - e), 2 * e + m          # mismatch, gap open (beyond the first base), per gap base


def score_bound(em, n, scores):
    em = DEFAULT_MODEL if em is None else em
    ev = lambda k: min(int(em[3 * k + 2]), int(em[3 * k] * n) + int(em[3 * k + 1]))
    X, O, E = penalties(scores)
    return ev(0) * X + ev(1) * O + ev(2) * E


def masked(seq: bytes) -> np.ndarray:
    q = np.frombuffer(bytes(seq), dtype=np.uint8).copy()
    q[~np.isin(q, np.frombuffer(b"ACGT", dtype=np.uint8))] = ord("X")      # never equal to a graph base
    return q


def gotoh(q: np.ndarray, t: np.ndarray, X, O, E, free_end):
    """Cost of aligning all of q to all of t (free_end: to the best prefix of t); a gap of length L costs O + L * E."""
    j = np.arange(len(t) + 1, dtype=np.int64)
    h = np.where(j == 0, 0, O + E * j)
    ins = np.full(len(t) + 1, _BIG, dtype=np.int64)
    for i in range(len(q)):
        ins = np.minimum(h + O + E, ins + E)
        diag = np.full(len(t) + 1, _BIG, dtype=np.int64)
        diag[1:] = h[:-1] + np.where(t == q[i], 0, X)
        g = np.minimum(diag, ins)
        run = np.minimum.accumulate(g - E * j)
        dele = np.full(len(t) + 1, _BIG, dtype=np.int64)
        dele[1:] = run[:-1] + O + E * j[1:]
        h = np.minimum(g, dele)
    return int(h.min() if free_end else h[-1])


def admitted_strings(g: Graph, prob, limit):
    """Connect: the bases strictly between from and to on every haplotype through from that reaches to.
    Suffix: what follows from (its prefixes are the strings).  Prefix: what precedes to, reversed (so its
    prefixes are the suffixes of the real strings).  limit: longer strings cannot fit the score bound."""
    mode, seq, frm, to = prob
    out = set()
    for w in g.walks:
        for k, v in enumerate(w):
            if mode == 2:
                if v != to[0]:
                    continue
                before = "".join(g.seq(u) for u in w[max(0, k - limit - 1):k]) + g.seq(v)[:to[1]]
                out.add(before[::-1][:limit])
                continue
            if v != frm[0]:
                continue
            first = g.seq(v)[frm[1] + 1:]
            if mode == 1:
                rest = first + "".join(g.seq(u) for u in w[k + 1:k + 2 + limit])
                out.add(rest[:limit])
                continue
            if to[0] == v and to[1] > frm[1]:
                out.add(g.seq(v)[frm[1] + 1:to[1]])
                continue
            between = first
            for u in w[k + 1:]:
                if u == to[0]:
                    out.add(between + g.seq(u)[:to[1]])
                    break
                between += g.seq(u)
                if len(between) > limit:
                    break
    return out


def dp_cost(g: Graph, scores, em, prob):
    """The least cost of an alignment the problem admits, or None when none fits the score bound."""
    mode, seq, frm, to = prob
    X, O, E = penalties(scores)
    bound = score_bound(em, len(seq), scores)
    limit = len(seq) + bound // E + 1
    q = masked(seq)
    if mode == 2:
        q = q[::-1]
    best = None
    for s in admitted_strings(g, prob, limit):
        if len(s) > limit:
            continue
        c = gotoh(q, np.frombuffer(s.encode(), dtype=np.uint8), X, O, E, free_end=mode != 0)
        best = c if best is None else min(best, c)
    return best if best is not None and best <= bound else None


def edit_cost(aln, scores):
    X, O, E = penalties(scores)
    return sum(n * X if op == "X" else (O + n * E if op in "ID" else 0) for op, n in aln["edits"])


def bonus(mode, aln, n, scores):
    ends = {1: -1, 2: 0}
    if mode not in ends or not aln["edits"] or aln["length"] != n:
        return 0
    return scores[4] if aln["edits"][ends[mode]][0] in "MX" else 0


def replay(g: Graph, scores, prob, aln):
    """Walk the edits along the returned path base by base; return the score they give (bonus included)."""
    mode, seq, frm, to = prob
    m, x, o, e, _ = scores
    q = masked(seq).tobytes().decode()
    path = aln["path"]
    for a, b in zip(path, path[1:]):
        assert (a, b) in g.edges, (a, b)
    if path:
        assert aln["node_offset"] < len(g.seq(path[0]))
        if mode != 2:
            assert (path[0] == frm[0] and aln["node_offset"] == frm[1] + 1) or \
                   (aln["node_offset"] == 0 and frm[1] + 1 == len(g.seq(frm[0])) and (frm[0], path[0]) in g.edges)
    assert all(n > 0 for _, n in aln["edits"])
    for (a, _), (b, _) in zip(aln["edits"], aln["edits"][1:]):
        assert a != b
    so, no, pi, score = aln["seq_offset"], aln["node_offset"], 0, 0
    for op, n in aln["edits"]:
        if op == "I":
            so += n; score -= o + (n - 1) * e; continue
        if op == "D":
            score -= o + (n - 1) * e
        for _ in range(n):
            if no == len(g.seq(path[pi])):
                pi, no = pi + 1, 0
            base = g.seq(path[pi])[no]
            if op == "M":
                assert q[so] == base; so += 1; score += m
            elif op == "X":
                assert q[so] != base; so += 1; score -= x
            no += 1
    assert so == aln["seq_offset"] + aln["length"]
    if path:
        assert pi == len(path) - 1 and no > 0, "unused trailing nodes"
        if mode != 1:
            end = path[-1]
            assert (end == to[0] and no == to[1]) or (to[1] == 0 and no == len(g.seq(end)) and (end, to[0]) in g.edges)
    return score + bonus(mode, aln, len(seq), scores)


def dp_applies(g: Graph, prob):
    """The DP poses acyclic problems with a start in the graph; connect with destination node 0 is a suffix without
    the bonus and is left to the oracle."""
    mode, seq, frm, to = prob
    return g.acyclic and g.valid((to if mode == 2 else frm)[0]) and not (mode == 0 and to[0] == 0)


def check_against_dp(g: Graph, scores, em, prob, aln):
    mode, seq, frm, to = prob
    cost = dp_cost(g, scores, em, prob)
    if mode == 0:
        assert aln["ok"] == (cost is not None), (cost, aln)
    else:
        assert aln["ok"] == 1
        assert (aln["length"] == len(seq)) == (cost is not None), (cost, aln)
    if not aln["ok"]:
        return
    if cost is not None:
        assert edit_cost(aln, scores) == cost, (cost, aln)
        graph_len = sum(n for op, n in aln["edits"] if op != "I")
        assert aln["score"] - bonus(mode, aln, len(seq), scores) == (scores[0] * (len(seq) + graph_len) - cost) // 2
    assert replay(g, scores, prob, aln) == aln["score"], aln


# ---------------------------------------------------------------------------------------------------------------
# graphs and problems
# ---------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def variant_graph(max_node, seed=9, length=4000):
    sg = synth.make_variant_graph(length=length, n_snp=40, n_ins=5, n_del=5, n_haps=6, seed=seed, max_node=max_node,
                                  name=f"variants-{max_node}bp")
    g = Graph.of(sg)
    g._index = sg.build_index()
    return g


@functools.lru_cache(maxsize=None)
def branchy_graph(n_haps=16):
    sg = synth.make_branchy_graph(n_layers=400, n_haps=n_haps, seed=4, name=f"branchy-{n_haps}")
    g = Graph.of(sg); g._index = sg.build_index()
    return g


@functools.lru_cache(maxsize=None)
def nested_graph():
    return Graph.of(synth.make_nested_graph(n_items=80, n_haps=10, seed=7))


@functools.lru_cache(maxsize=None)
def edge_graph():
    """Hand-made acyclic graph: a SNP (2 / 3), an insertion (5), and node 7 only on a haplotype that avoids 2."""
    seqs = ["GATTACA", "C", "T", "GGCATTAG", "AC", "TTGCAAT", "CCGA"]
    paths = [[2, 4, 8, 10, 12], [2, 6, 8, 12], [2, 4, 8, 12], [14, 8, 10, 12]]
    return Graph(seqs, paths, name="edges")


@functools.lru_cache(maxsize=None)
def cyclic_graph():
    seqs = ["ACGTTG", "CA", "GGTCA"]
    paths = [[2, 4, 6, 2, 4, 6, 2, 4, 6, 2], [2, 6, 2, 6, 2, 6], [4, 6, 2, 4]]
    return Graph(seqs, paths, acyclic=False, name="cyclic")


def pool_connect(o):
    """From the first base of the chain to base 500 of its 24th trie node."""
    end = 23 * 1024 + (1 if o.name.endswith("1") else 0) + 500
    return (0, o.hap[1:end].encode(), (2, 0), (2 * len(o.node_seqs) - 6, 500))


def linear_graph(n, node_len, seed=3):
    rng = np.random.default_rng(seed)
    seq = bytes(synth.BASES[rng.integers(0, 4, size=n * node_len)]).decode()
    return Graph([seq[i:i + node_len] for i in range(0, len(seq), node_len)], [[2 * i for i in range(1, n + 1)]],
                 name=f"linear-{node_len}bp")


def star_graph(k):
    """Node 1 followed by k one-haplotype leaves: expanding node 1 meets k successors."""
    rng = np.random.default_rng(k)
    seqs = ["ACGTTGCA"] + [bytes(synth.BASES[rng.integers(0, 4, size=6)]).decode() for _ in range(k)]
    return Graph(seqs, [[2, 2 * (i + 2)] for i in range(k)], name=f"star-{k}")


def pool_graph(extra, seed=5):
    """A haplotype of 1024-base nodes (the longest the index accepts), with a 1-base node before the 24th when extra:
    a connect into the 24th trie node then needs 24 576 + extra bytes of trie sequence."""
    rng = np.random.default_rng(seed)
    lens = [1024] * 23 + ([1] if extra else []) + [1024] * 4
    seq = bytes(synth.BASES[rng.integers(0, 4, size=sum(lens))]).decode()
    cut = np.concatenate([[0], np.cumsum(lens)])
    g = Graph([seq[a:b] for a, b in zip(cut, cut[1:])], [[2 * i for i in range(1, len(lens) + 1)]], name=f"pool+{extra}")
    g.hap = seq
    return g


def random_problems(g: Graph, n, seed, max_len=90, sub=0.03, modes=(0, 1, 2), flip=0.3, min_len=0):
    """Cut from a random haplotype, mutated, on a random strand."""
    sg = g.synth
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        h = int(rng.integers(0, len(sg.paths)))
        hs = sg.hap_seq[h]
        ln = int(rng.integers(min_len, max_len + 1))
        a = int(rng.integers(0, len(hs) - ln - 2))
        seq = hs[a + 1:a + 1 + ln].copy()
        mut = rng.random(ln) < sub
        seq[mut] = synth.BASES[rng.integers(0, 4, size=int(mut.sum()))]
        seq = bytes(seq)
        if rng.random() < 0.2 and len(seq) > 10:
            k = int(rng.integers(2, len(seq) - 2)); seq = seq[:k] + seq[k + int(rng.integers(1, 4)):]
        if rng.random() < 0.2 and len(seq) > 10:
            k = int(rng.integers(2, len(seq) - 2)); seq = seq[:k] + b"ACGT"[: int(rng.integers(1, 4))] + seq[k:]
        frm = (2 * int(sg.hap_node[h][a]), int(sg.hap_off[h][a]))
        to = (2 * int(sg.hap_node[h][a + 1 + ln]), int(sg.hap_off[h][a + 1 + ln]))
        if rng.random() < flip:
            seq = revcomp(seq.decode()).encode()
            nlen = lambda v: len(g.seq(v))
            frm, to = (to[0] ^ 1, nlen(to[0]) - 1 - to[1]), (frm[0] ^ 1, nlen(frm[0]) - 1 - frm[1])
        mode = int(modes[int(rng.integers(0, len(modes)))])
        out.append((mode, seq, frm if mode != 2 else None, to if mode != 1 else None))
    return out


SCORE_SETS = [(1, 4, 6, 1, 5), (2, 4, 6, 1, 5), (3, 2, 5, 2, 0), (1, 3, 2, 2, 10), (1, 20, 6, 1, 5)]


def model(mismatches=(0.03, 1, 6), gaps=(0.05, 1, 10), gap_length=(0.1, 1, 20), distance=tuple(NO_PRUNE)):
    return [*mismatches, *gaps, *gap_length, *distance]


DP_MODELS = {"default": model(), "all-zero": model((0, 0, 0), (0, 0, 0), (0, 0, 0)), "per-base": model((0.05, 0, 100), (0.05, 0, 100), (0.1, 0, 100)),
             "wide": model((0.2, 2, 40), (0.1, 2, 20), (0.3, 2, 60))}
PRUNING_MODELS = {"band-0": model(distance=(0, 0, 0)), "band-1": model(distance=(0, 1, 1)), "default": None}


def edge_problems():
    """(graph, problem) pairs for the hand-written edges."""
    E = edge_graph()
    out = []
    for seq in (b"", b"A", b"C", b"T"):
        out += [(E, (0, seq, (2, 6), (8, 0))), (E, (0, seq, (2, 3), (2, 4))), (E, (1, seq, (2, 3), None)), (E, (1, seq, (8, 7), None)),
                (E, (2, seq, None, (8, 0))), (E, (2, seq, None, (12, 0))), (E, (1, seq, (9, 0), None)), (E, (2, seq, None, (3, 0)))]
    odd = [b"GGCnTTAG", b"NNNNN", b"ggcattag", b"GG\x00ATT-G", b"GGCAT\xffAG", b"TTAGACTTGCA"]
    for seq in odd:
        out += [(E, (1, seq, (2, 6), None)), (E, (0, seq, (2, 6), (12, 4))), (E, (2, seq, None, (12, 4)))]
    out += [
        (E, (0, b"CGGCATTAGACTTG", (2, 6), (12, 3))),          # from at the last base: the first node is dropped
        (E, (0, b"TGGCATTAG", (2, 6), (10, 0))),              # to at offset 0
        (E, (0, b"TTA", (8, 2), (8, 6))), (E, (0, b"", (8, 2), (8, 3))), (E, (0, b"A", (8, 2), (8, 3))),   # from == to node
        (E, (0, b"TTA", (8, 2), (8, 2))), (E, (0, b"TTA", (8, 4), (8, 1))),                                # to before from: 0
        (E, (0, b"GGCATTAGAC", (4, 0), (10, 1))),             # 5 only on haplotypes that avoid 2
        (E, (0, b"GGCATTAG", (14, 3), (10, 0))), (E, (0, b"GGCATTAG", (14, 3), (12, 0))),
        (E, (0, b"ACG", (0, 0), (8, 0))), (E, (0, b"ACG", (1, 0), (8, 0))), (E, (0, b"ACG", (16, 0), (8, 0))),
        (E, (0, b"ACG", (99, 0), (8, 0))), (E, (2, b"ACG", None, (0, 0))), (E, (2, b"ACG", None, (1, 0))),
        (E, (2, b"ACG", None, (16, 0))), (E, (1, b"ACG", (0, 0), None)), (E, (1, b"ACG", (1, 0), None)),
        (E, (0, b"GGCATTAG", (2, 6), (0, 0))),               # connect without a destination
        (E, (0, b"GGCATTAG", (2, 6), (99, 0))),              # destination not in the graph
        (E, (1, b"GGCAGGGGGGGGGGGGTTTTTTTTTTTTT", (2, 6), None)),   # needs trim
        (E, (1, b"GGCATTAGAGTTTTTTTTTTTTTTTTTTTTTTTTT", (2, 6), None)),   # trim ties across the 5 / no-5 branches
        (E, (2, b"TTTTTTTTTTTTTTTTTTTTTTTTGCAAT", None, (12, 6))),
    ]
    # both strands of everything with a valid start
    flipped = []
    for G, (mode, seq, frm, to) in out:
        if G is E and mode == 0 and frm and to and G.valid(frm[0]) and G.valid(to[0]) and frm[0] != to[0] and to[1] > 0:
            nl = lambda v: len(G.seq(v))
            flipped.append((G, (0, revcomp(seq.decode("latin1")).encode("latin1"), (to[0] ^ 1, nl(to[0]) - to[1]),
                                (frm[0] ^ 1, nl(frm[0]) - 1 - frm[1]))))
    return out + flipped


def cyclic_problems():
    Y = cyclic_graph()
    hs = "".join(Y.seq(v) for v in Y.paths[0])
    out = []
    for ln in (0, 1, 5, 13, 20, 30, 40):
        out += [(1, hs[6:6 + ln].encode(), (2, 5), None), (0, hs[6:6 + ln].encode(), (2, 5), (2, 0)),
                (0, hs[7:7 + ln].encode(), (4, 0), (6, 2)), (2, hs[10:10 + ln].encode(), None, (2, 3)),
                (1, revcomp(hs[6:6 + ln]).encode(), (3, 2), None)]
    return [(Y, p) for p in out]


# ---------------------------------------------------------------------------------------------------------------
# CPU: the oracle against the DP, the workspace report and the predictor
# ---------------------------------------------------------------------------------------------------------------
def dp_cases():
    """(graph, scores, error model, problems) sets checked against the DP, first on the oracle and then on the GPU."""
    cases = []
    for mn in (1, 2, 4, 32):
        g = variant_graph(mn)
        cases.append((g, DEFAULT_SCORES, model(), random_problems(g, 60, seed=100 + mn)))
    g = variant_graph(32)
    for i, sc in enumerate(SCORE_SETS[1:]):
        cases.append((g, sc, model(), random_problems(g, 40, seed=200 + i)))
    for i, (name, em) in enumerate(DP_MODELS.items()):
        cases.append((g, DEFAULT_SCORES, em, random_problems(g, 40, seed=300 + i, sub=0.06)))
    cases.append((branchy_graph(), DEFAULT_SCORES, model(), random_problems(branchy_graph(), 50, seed=400)))
    cases.append((nested_graph(), DEFAULT_SCORES, model(), random_problems(nested_graph(), 50, seed=401)))
    for sc in (DEFAULT_SCORES, (2, 4, 6, 1, 5)):
        cases.append((edge_graph(), sc, model(), [p for G, p in edge_problems()]))
    return cases


@pytest.mark.parametrize("k", range(len(dp_cases())))
def test_oracle_matches_the_gotoh_dp(k):
    g, sc, em, probs = dp_cases()[k]
    full = 0
    for p in probs:
        aln = oracle_run(g, sc, em, p)
        if not g.valid((p[3] if p[0] == 2 else p[2])[0]):
            assert aln["ok"] == 0
            continue
        if not dp_applies(g, p):
            continue
        check_against_dp(g, sc, em, p, aln)
        full += aln["ok"] == 1 and aln["length"] == len(p[1])
    assert full > 0


def test_gotoh_dp_hand_values():
    X, O, E = penalties(DEFAULT_SCORES)          # 10, 10, 3
    q = lambda s: masked(s.encode())
    t = lambda s: np.frombuffer(s.encode(), dtype=np.uint8)
    assert gotoh(q("ACGT"), t("ACGT"), X, O, E, False) == 0
    assert gotoh(q("ACCT"), t("ACGT"), X, O, E, False) == X
    assert gotoh(q("ACNT"), t("ACNT"), X, O, E, False) == X          # a masked base never matches
    assert gotoh(q("ACGT"), t("ACGGGT"), X, O, E, False) == O + 2 * E
    assert gotoh(q("AGGGCT"), t("ACT"), X, O, E, False) == O + 3 * E
    assert gotoh(q(""), t("ACG"), X, O, E, False) == O + 3 * E
    assert gotoh(q("ACG"), t("ACGTTT"), X, O, E, True) == 0
    assert gotoh(q("AAAAACCCCC"), t("AAAAAGCCCCC"), X, O, E, False) == O + E


def test_workspace_report_at_hand_computed_edges():
    # a 1-bp linear graph: the root trie node grows to 1024 graph nodes, the alignment uses 20 of them
    g = linear_graph(3000, 1)
    hs = "".join(g.node_seqs)
    prob = (1, hs[1:21].encode(), (2, 0), None)
    ws, want = oracle_workspace(g, DEFAULT_SCORES, None, prob), oracle_run(g, DEFAULT_SCORES, None, prob)
    assert (ws["trie_nodes"], ws["path_entries"], ws["seq_bytes"]) == (1, 1024, 1024)
    assert want["ok"] and len(want["path"]) == 20 and want["node_offset"] == 0
    assert predict(ws, want) == 1 and predict(ws, want, path_cap=20) == 1 and predict(ws, want, path_cap=19) == -1
    # its prefix mirror
    prob = (2, hs[1000:1020].encode(), None, (2 * 1021, 0))
    ws, want = oracle_workspace(g, DEFAULT_SCORES, None, prob), oracle_run(g, DEFAULT_SCORES, None, prob)
    assert ws["path_entries"] == 1021 and want["ok"] and len(want["path"]) == 20 and predict(ws, want) == 1     # the haplotype starts 1021 nodes back
    # 32 vs 33 successors of one trie node
    for k in (32, 33):
        s = star_graph(k)
        prob = (1, b"GAC", (2, 7), None)
        ws, want = oracle_workspace(s, DEFAULT_SCORES, None, prob), oracle_run(s, DEFAULT_SCORES, None, prob)
        assert ws["max_successors"] == k and ws["trie_nodes"] == k + 1
        assert over_limits(ws) == ([] if k == 32 else ["max_successors"])
    # a 24 576- vs 24 577-byte trie: a connect into the 24th trie node of a chain of 1024-base nodes
    for extra in (0, 1):
        o = pool_graph(extra)
        prob = pool_connect(o)
        ws, want = oracle_workspace(o, DEFAULT_SCORES, None, prob), oracle_run(o, DEFAULT_SCORES, None, prob)
        assert (ws["seq_bytes"], ws["trie_nodes"], ws["path_entries"]) == (24576 + extra, 24, 24 + extra)
        assert over_limits(ws) == ([] if extra == 0 else ["seq_bytes"]) and want["ok"] and len(want["path"]) == 24 + extra
    # the start point alone, for an empty suffix
    ws = oracle_workspace(edge_graph(), DEFAULT_SCORES, None, (1, b"", (2, 3), None))
    assert ws == {**dict.fromkeys(WORKSPACE_FIELDS, 0), "trie_nodes": 1, "seq_bytes": 7, "path_entries": 1, "points": 1,
                  "scores": 1, "max_node_offset": 4}
    # nothing runs for a start that is not in the graph
    assert oracle_workspace(edge_graph(), DEFAULT_SCORES, None, (1, b"ACG", (1, 0), None)) == dict.fromkeys(WORKSPACE_FIELDS, 0)


def test_predictor_edges():
    ws0 = dict.fromkeys(WORKSPACE_FIELDS, 0)
    ok = {"ok": 1, "path": [2] * 7, "edits": [("M", 1)] * 3}
    assert predict(ws0, ok) == 1 and predict(ws0, {"ok": 0, "path": [], "edits": []}) == 0
    assert predict(ws0, ok, path_cap=7, edit_cap=3) == 1
    assert predict(ws0, ok, path_cap=6) == -1 and predict(ws0, ok, edit_cap=2) == -1
    assert predict(ws0, {"ok": 0, "path": [], "edits": []}, path_cap=1, edit_cap=1) == 0
    for f, cap in LIMITS.items():
        assert predict({**ws0, f: cap}, ok) == 1 and predict({**ws0, f: cap + 1}, ok) == -1
    assert predict({**ws0, "min_diagonal": -1024}, ok) == 1 and predict({**ws0, "min_diagonal": -1025}, ok) == -1


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
_DEVICES = {}


def device(g, scores):
    key = (id(g), scores)
    if key not in _DEVICES:
        _DEVICES[key] = capi.Device(g.index, scores=capi.Scores(*scores))
    return _DEVICES[key]


@pytest.fixture(scope="module", autouse=True)
def _close_devices():
    yield
    for d in _DEVICES.values():
        d.close()
    _DEVICES.clear()


def gpu_run(g, scores, em, probs, path_cap=512, edit_cap=512):
    return device(g, scores).wfa_batch(probs, error_model=em, path_cap=path_cap, edit_cap=edit_cap, with_status=True)


def check_gpu(g, scores, em, probs, got, path_cap=512, edit_cap=512):
    """GPU status == predicted status; every field equal to the oracle's where the kernel answered."""
    stats = {-1: 0, 0: 0, 1: 0}
    for p, gt in zip(probs, got):
        want = oracle_run(g, scores, em, p)
        st = predict(oracle_workspace(g, scores, em, p), want, path_cap, edit_cap)
        assert gt["ok"] == st, (g.name, p, gt, want, oracle_workspace(g, scores, em, p))
        if st >= 0:
            assert gt == want, (g.name, p, gt, want)
        stats[st] += 1
    return stats


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(dp_cases())))
def test_gpu_matches_the_gotoh_dp_and_the_oracle(k):
    g, sc, em, probs = dp_cases()[k]
    got = gpu_run(g, sc, em, probs)
    check_gpu(g, sc, em, probs, got)
    for p, gt in zip(probs, got):
        if dp_applies(g, p) and gt["ok"] >= 0:          # -1 was checked against the prediction above
            check_against_dp(g, sc, em, p, gt)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRUNING_MODELS))
def test_gpu_pruning_error_models(name):
    g = variant_graph(32)
    probs = random_problems(g, 150, seed=500, sub=0.05)
    check_gpu(g, DEFAULT_SCORES, PRUNING_MODELS[name], probs, gpu_run(g, DEFAULT_SCORES, PRUNING_MODELS[name], probs))


@pytest.mark.gpu
def test_gpu_edges_and_cyclic_graphs():
    for g, probs in ((edge_graph(), [p for _, p in edge_problems()]), (cyclic_graph(), [p for _, p in cyclic_problems()])):
        for sc in (DEFAULT_SCORES, (2, 4, 6, 1, 5)):
            stats = check_gpu(g, sc, model(), probs, gpu_run(g, sc, model(), probs))
            assert stats[1] > 0 and stats[0] > 0


def long_connects():
    sg = synth.make_variant_graph(length=30000, n_snp=30, n_ins=3, n_del=3, n_haps=4, seed=21, name="30kb")
    g = Graph.of(sg); g._index = sg.build_index()
    rng = np.random.default_rng(6)
    probs = []
    for ln in (1000, 4000, 8000, 12000, 16000, 20000, 22000, 23500, 24000, 24500, 25000, 25000):
        probs += [p for p in random_problems(g, 1, seed=int(rng.integers(1 << 30)), min_len=ln, max_len=ln, sub=0.001, modes=(0,))]
    return g, probs


@functools.lru_cache(maxsize=None)
def limit_sets():
    """(family, graph, scores, error model, problems) on both sides of every workspace limit."""
    sets = []
    for mn in (1, 2, 4):
        g = variant_graph(mn, seed=31)
        sets.append((f"variants {mn}-bp nodes", g, DEFAULT_SCORES, None, random_problems(g, 250, seed=mn, max_len=300, sub=0.05)))
    sets.append(("branchy", branchy_graph(), DEFAULT_SCORES, None, random_problems(branchy_graph(), 200, seed=7, max_len=300, sub=0.05)))
    sets.append(("branchy, 64 haplotypes", branchy_graph(64), DEFAULT_SCORES, None,
                 random_problems(branchy_graph(64), 150, seed=9, max_len=200, sub=0.05)))
    sets.append(("branchy, 256 haplotypes", branchy_graph(256), DEFAULT_SCORES, model((0.1, 2, 30), (0.05, 1, 10), (0.1, 1, 20)),
                 random_problems(branchy_graph(256), 60, seed=10, max_len=150, sub=0.08)))
    g = variant_graph(4, seed=31)
    sets.append(("variants 4-bp nodes, noisy", g, DEFAULT_SCORES, model((0.2, 2, 60), (0.1, 2, 20), (0.2, 2, 40)),
                 random_problems(g, 80, seed=11, max_len=300, min_len=100, sub=0.15)))
    sets.append(("nested", nested_graph(), DEFAULT_SCORES, None, random_problems(nested_graph(), 200, seed=8, max_len=250, sub=0.05)))
    g, probs = long_connects()
    sets.append(("connects 1-25 kb", g, DEFAULT_SCORES, None, probs))
    # a wide error model and unrelated queries: scores past 8191, diagonals past -1024, many scores and points
    g = variant_graph(32)
    rng = np.random.default_rng(12)
    wide = [1, 0, 20000, 1, 0, 20000, 2, 0, 40000, 0, 100000, 100000]
    probs = []
    for ln in (1, 5, 20, 60, 150, 250):
        q = bytes(synth.BASES[rng.integers(0, 4, size=ln)])
        probs += [(1, q, (2 * 5, 3), None), (0, q[:3], (2 * 5, 3), (2 * 60, 0)), (0, q, (2 * 5, 3), (2 * 9, 1))]
    sets.append(("wide error model", g, DEFAULT_SCORES, wide, probs))
    # every penalty 256 in WFA units: few distinct scores, and a connect across k graph bases stores scores near 256 k
    lin = linear_graph(100, 4)
    sets.append(("scores past 8191", lin, (2, 126, 127, 127, 0), [0, 1, 1, 0, 1, 1, 0, 60, 60, 0, 100000, 100000],
                 [(0, b"A", (2 * 3, 1), (2 * (3 + k // 4), k % 4)) for k in range(24, 44)]))
    # the sequence pool exactly full and one byte over; 30 kb of 1024-base nodes (the index refuses longer nodes)
    for extra in (0, 1):
        o = pool_graph(extra)
        far = (0, o.hap[1:26 * 1024 + 300].encode(), (2, 0), (2 * len(o.node_seqs), 300))
        sets.append((f"1024-base nodes, pool + {extra}", o, DEFAULT_SCORES, None,
                     [pool_connect(o), far, (1, o.hap[1:41].encode(), (2, 0), None), (2, o.hap[-40:].encode(), None, (2 * len(o.node_seqs), 1023)),
                      (1, o.hap[5000:5040].encode(), (2 * 5, 903), None)]))
    for k in (31, 32, 33, 40):
        s = star_graph(k)
        sets.append((f"star {k}", s, DEFAULT_SCORES, None, [(1, s.seq(2 * (i + 2))[:4].encode(), (2, 7), None) for i in range(k)]))
    return sets


@pytest.mark.gpu
def test_gpu_status_equals_prediction_at_every_limit(capsys):
    bands = {"small table": 0, "retry": 0, "over": 0}
    exceeded = {}
    for family, g, sc, em, probs in limit_sets():
        stats = check_gpu(g, sc, em, probs, gpu_run(g, sc, em, probs))
        for p in probs:
            ws = oracle_workspace(g, sc, em, p)
            bands["small table" if ws["points"] <= SMALL_TABLE_POINTS else "retry" if ws["points"] <= LIMITS["points"] else "over"] += 1
            for f in over_limits(ws):
                exceeded[f] = exceeded.get(f, 0) + 1
        with capsys.disabled():
            print(f"\n{family}: {len(probs)} problems, -1 rate {stats[-1] / len(probs):.3f}, ok {stats[1]}, no alignment {stats[0]}")
    with capsys.disabled():
        print(f"point bands {bands}; limits exceeded {exceeded}")
    assert bands["retry"] >= 36 and bands["over"] >= 36 and bands["small table"] >= 36
    # The diagonal and offset limits stay in the predictor but cannot decide a problem: each step along a diagonal is a
    # distinct score, so 512 scores run out before diagonal -1024, and offsets are bounded by the 24 576-byte pool and
    # the 60 000-base sequence limit.
    for f in ("trie_nodes", "seq_bytes", "path_entries", "points", "scores", "max_score", "max_successors"):
        assert exceeded.get(f, 0) > 0, f


def cap_cases():
    import test_wfa_golden as TW
    cases = []
    by_key = {}
    for c in TW.GOLD["cases"]:
        key = (c["graph"], None if c["error_model"] is None else tuple(c["error_model"]))
        by_key.setdefault(key, []).append(c)
    for (graph, em), cs in by_key.items():
        gg = TW.GOLD["graphs"][graph]
        ids = sorted(int(k) for k in gg["nodes"])
        g = Graph([gg["nodes"][str(i)] for i in ids], [[2 * i for i in p] for p in gg["paths"]], index=TW.index_of(graph), name=graph)
        cases.append((g, TW.SCORES, None if em is None else list(em), [TW._problem_of(c) for c in cs]))
    for mn in (1, 2, 32):
        g = variant_graph(mn)
        cases.append((g, DEFAULT_SCORES, None, random_problems(g, 120, seed=600 + mn, max_len=120)))
    return cases


@pytest.mark.gpu
def test_gpu_output_caps_at_and_below_the_answer():
    checked = below = 0
    for g, sc, em, probs in cap_cases():
        wants = [oracle_run(g, sc, em, p) for p in probs]
        fits = [not over_limits(oracle_workspace(g, sc, em, p)) for p in probs]
        groups = {}
        for i, w in enumerate(wants):
            if w["ok"] and fits[i]:
                groups.setdefault((max(1, len(w["path"])), max(1, len(w["edits"]))), []).append(i)
        for (pc, ec), idx in groups.items():
            sub = [probs[i] for i in idx]
            for gt, i in zip(gpu_run(g, sc, em, sub, path_cap=pc, edit_cap=ec), idx):
                assert gt == wants[i], (g.name, probs[i], pc, ec, gt, wants[i])
                checked += 1
            if pc > 1:
                for gt in gpu_run(g, sc, em, sub, path_cap=pc - 1, edit_cap=ec):
                    assert gt["ok"] == -1 and gt["path"] == [] and gt["edits"] == []
                    below += 1
            if ec > 1:
                for gt in gpu_run(g, sc, em, sub, path_cap=pc, edit_cap=ec - 1):
                    assert gt["ok"] == -1
                    below += 1
    assert checked > 400 and below > 400


@pytest.mark.gpu
def test_gpu_batch_larger_than_the_grid_and_permuted():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    threads = 4 * sms * 32
    g = variant_graph(1, seed=31)
    base = random_problems(g, 300, seed=2, max_len=300, sub=0.05) + random_problems(g, 100, seed=3, max_len=40)
    wants = []
    for p in base:
        want = oracle_run(g, DEFAULT_SCORES, None, p)
        wants.append((predict(oracle_workspace(g, DEFAULT_SCORES, None, p), want), want))
    assert sum(w[0] == 1 for w in wants) > 100 and sum(w[0] == -1 for w in wants) > 10
    n = threads + 1500
    rng = np.random.default_rng(0)
    pick = rng.integers(0, len(base), size=n)
    got = gpu_run(g, DEFAULT_SCORES, None, [base[i] for i in pick])
    for i, gt in zip(pick, got):
        st, want = wants[i]
        assert gt["ok"] == st and (st < 0 or gt == want)
    perm = rng.permutation(n)
    got2 = gpu_run(g, DEFAULT_SCORES, None, [base[pick[j]] for j in perm])
    assert all(got2[k] == got[perm[k]] for k in range(n))


def all_gpu_sets():
    out = [(g, sc, em, probs) for g, sc, em, probs in dp_cases()]
    out += [(g, sc, em, probs) for _, g, sc, em, probs in limit_sets()]
    out += [(g, sc, model(), [p for _, p in edge_problems()]) for g in (edge_graph(),) for sc in (DEFAULT_SCORES,)]
    out += [(cyclic_graph(), DEFAULT_SCORES, model(), [p for _, p in cyclic_problems()])]
    return out


@pytest.mark.gpu
def test_gpu_input_checks():
    g = edge_graph()
    dev = device(g, DEFAULT_SCORES)
    with pytest.raises(capi.GbError) as e:
        dev.wfa_batch([(3, b"ACG", (2, 3), None)], with_status=True)
    assert e.value.code == capi.GB_ERR_ARG
    long_ok = dev.wfa_batch([(1, b"A" * 60000, (2, 3), None)], with_status=True)
    assert long_ok[0]["ok"] in (-1, 1)
    with pytest.raises(capi.GbError) as e:
        dev.wfa_batch([(1, b"ACG", (2, 3), None), (1, b"A" * 60001, (2, 3), None)], with_status=True)
    assert e.value.code == capi.GB_ERR_ARG
    for pc, ec in ((0, 8), (8, 0)):
        with pytest.raises(capi.GbError) as e:
            dev.wfa_batch([(1, b"ACG", (2, 3), None)], path_cap=pc, edit_cap=ec, with_status=True)
        assert e.value.code == capi.GB_ERR_ARG
    before = dev.launches()
    assert dev.wfa_batch([], with_status=True) == []
    assert dev.launches() == before
    dev.wfa_batch([(1, b"ACG", (2, 3), None)])
    assert dev.launches() == before + 1


@pytest.mark.gpu
def test_gpu_whole_table_from_the_start_gives_identical_outputs(monkeypatch):
    first = [gpu_run(g, sc, em, probs) for g, sc, em, probs in all_gpu_sets()]
    monkeypatch.setenv("GIRAFFE_B200_WFA_SMALL_TABLE", "0")
    second = [gpu_run(g, sc, em, probs) for g, sc, em, probs in all_gpu_sets()]
    assert first == second
