"""The DAG alignment seams gb_sw_batch, gb_xdrop_dag_batch and gb_banded_global_batch at their limits, against a
reference that computes the answer another way than the oracle.

Any alignment of a read to a DAG lies on one source-to-sink walk, so the DAG optimum is the maximum over walks of a
string DP.  The CPU part lists the walks, runs three numpy DPs along the query (local Gotoh with the gb_sw_batch rules,
global Gotoh with the gb_banded_global_batch rules, the pinned semi-global pass of the X-drop aligner) and rescores a
returned path from its mappings and edits alone.  It checks the oracle against them on DAG families and pins each DP on
hand-computed cases.

The GPU part runs one problem generator through the three seams: query widths around every 32-lane chunk edge up to
1024, node lengths 1 to 1024, long chains of 1-bp nodes, bubbles, fan-in and fan-out of 255, rescue-sized subgraphs,
N bases, seven scoring schemes, exact and short output caps, a batch larger than the resident warps, X-drop seeds and
max_gap values at their edges, and band paddings.  Every problem must equal the oracle, its path must rescore to its
score, and where the walk DP defines the answer the score must equal it.
"""
import numpy as np
import pytest

from vg_b200 import capi
import test_xdrop_dag as TD
from test_banded_global_golden import oracle_banded
from test_sw_golden import _dag_walks, oracle_sw

NEG = -(1 << 40)
ALIVE = NEG // 2
ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
WALK_LIMIT = 256

# (match, mismatch, gap_open, gap_extend, full_length_bonus)
SCHEMES = {"default": (1, 4, 6, 1, 5), "no-bonus": (1, 4, 6, 1, 0), "all-ones": (1, 1, 1, 1, 0), "go=ge": (2, 3, 2, 2, 4),
           "ge=0": (1, 4, 6, 0, 5), "int8-max": (127, 127, 127, 127, 127), "int8-mixed": (127, 1, 127, 1, 127)}


# ---- walks ---------------------------------------------------------------------------------------------------------
class TooManyWalks(Exception):
    pass


def successors(preds):
    succ = [[] for _ in preds]
    for v, ps in enumerate(preds):
        for p in sorted(set(ps)):
            succ[p].append(v)
    return succ


def walks_from(nxt, u, limit=WALK_LIMIT):
    """Every walk that starts at node u and follows nxt (successor or predecessor lists) until a node without any."""
    out, stack = [], [[u]]
    while stack:
        w = stack.pop()
        ahead = sorted(set(nxt[w[-1]]))
        if not ahead:
            out.append(w)
            if len(out) > limit:
                raise TooManyWalks
        stack += [w + [v] for v in ahead]
    return out


def walks(preds, limit=WALK_LIMIT):
    """Every source-to-sink walk of the problem."""
    succ, out = successors(preds), []
    for s in (u for u, ps in enumerate(preds) if not ps):
        out += walks_from(succ, s, limit - len(out))
    return out


# ---- string DPs, vectorised along the query ------------------------------------------------------------------------
def _qarr(q):
    qa = np.frombuffer(bytes(q), dtype=np.uint8)
    return qa, np.isin(qa, ACGT)


def _scan_insertions(src, go, ge):
    """F(j) = max over k < j of src(k) - go - (j - 1 - k) ge (dead sources at NEG)."""
    j = np.arange(len(src), dtype=np.int64)
    g = np.where(src > ALIVE, src + j * ge, NEG)
    excl = np.full(len(src), NEG, dtype=np.int64)
    excl[1:] = np.maximum.accumulate(g)[:-1]
    return np.where(excl > ALIVE, excl - go - (j - 1) * ge, NEG)


def local_best(ref, q, sc):
    """gb_sw_batch on a string: local Gotoh, pairs with N score 0, the bonus at each read end that is aligned."""
    match, mism, go, ge, bonus = sc
    m = len(q)
    if m == 0 or not ref:
        return 0
    qa, qok = _qarr(q)
    Hp = np.zeros(m + 1, dtype=np.int64)            # "no predecessor" behaves like H = 0: d takes max(H, 0), E needs H > 0
    Ep = np.full(m + 1, NEG, dtype=np.int64)
    best = 0
    for r in bytes(ref):
        s = np.where(qok & (r in b"ACGT"), np.where(qa == r, match, -mism), 0)
        d = np.full(m + 1, NEG, dtype=np.int64)
        d[1] = bonus + s[0]
        d[2:] = np.maximum(Hp[1:m], 0) + s[1:]
        e = np.maximum(np.where(Hp > 0, Hp - go, NEG), np.where(Ep > ALIVE, Ep - ge, NEG))
        e[(e <= 0) | (np.arange(m + 1) == 0)] = NEG
        hp = np.maximum(d, e)
        f = _scan_insertions(np.where(hp > 0, hp, NEG), go, ge)
        f[f <= 0] = NEG
        H = np.maximum(np.maximum(d, 0), np.maximum(e, f))
        H[0] = 0
        best = max(best, int(H.max()), int(d[m]) + bonus)
        Hp, Ep = H, e
    return best


def global_best(ref, q, sc):
    """gb_banded_global_batch without a band on a string: global Gotoh, N pairs 0, no bonus, every gap adjacency opens."""
    match, mism, go, ge = sc[:4]
    m = len(q)
    qa, qok = _qarr(q)
    j = np.arange(m + 1, dtype=np.int64)
    M = np.full(m + 1, NEG, dtype=np.int64); M[0] = 0
    I = np.where(j > 0, -(go + (j - 1) * ge), NEG)
    D = np.full(m + 1, NEG, dtype=np.int64)
    for r in bytes(ref):
        s = np.where(qok & (r in b"ACGT"), np.where(qa == r, match, -mism), 0)
        prev = np.maximum(np.maximum(M, I), D)
        Mn = np.full(m + 1, NEG, dtype=np.int64)
        Mn[1:] = np.where(prev[:-1] > ALIVE, prev[:-1] + s, NEG)
        Dn = np.maximum(np.where(np.maximum(M, I) > ALIVE, np.maximum(M, I) - go, NEG), np.where(D > ALIVE, D - ge, NEG))
        M, D, I = Mn, Dn, _scan_insertions(np.maximum(Mn, Dn), go, ge)
    return int(max(M[m], I[m], D[m]))


def pinned_rows(ref, q, sc, max_gap):
    """The pinned pass of gb_xdrop_dag_batch on a string, without X-drop pruning: H for every graph base and query prefix
    (rows = graph bases).  N is a mismatch, the bonus goes on the last query base, leading insertions <= max_gap."""
    match, mism, go, ge, bonus = sc
    assert go >= ge
    m = len(q)
    max_gap = max(max_gap, 1)
    qa, qok = _qarr(q)
    j = np.arange(m + 1, dtype=np.int64)
    Hp = np.where((j > 0) & (j <= max_gap), -(go + (j - 1) * ge), NEG)
    Hp[0] = 0
    Ep = np.full(m + 1, NEG, dtype=np.int64)
    rows = np.empty((len(ref), m + 1), dtype=np.int64)
    for c, r in enumerate(bytes(ref)):
        s = np.where(qok & (qa == r), match, -mism)
        if m:
            s[m - 1] += bonus
        d = np.full(m + 1, NEG, dtype=np.int64)
        d[1:] = np.where(Hp[:-1] > ALIVE, Hp[:-1] + s, NEG)
        e = np.maximum(np.where(Hp > ALIVE, Hp - go, NEG), np.where(Ep > ALIVE, Ep - ge, NEG))
        hp = np.maximum(d, e)
        H = np.maximum(hp, _scan_insertions(hp, go, ge))      # opening from an insertion never beats extending it (go >= ge)
        rows[c] = H
        Hp, Ep = H, e
    return rows


# ---- DAG optima over walks -----------------------------------------------------------------------------------------
def sw_optimum(seqs, preds, q, sc):
    return max(local_best("".join(seqs[u] for u in w).encode(), q, sc) for w in walks(preds))


def global_optimum(seqs, preds, q, sc):
    return max(global_best("".join(seqs[u] for u in w).encode(), q, sc) for w in walks(preds))


def pinned_cells(seqs, preds, start, q, sc, max_gap, backward=False):
    """The pinned pass from `start` = (node, offset) over every walk from there, without pruning: {(node, column): H row}
    with the maximum over walks.  Forward: the walk continues right of the offset; backward: left of it, mirrored."""
    u0, o0 = start
    nxt = preds if backward else successors(preds)
    cells = {}
    for w in walks_from(nxt, u0):
        pos = [(u0, c) for c in (range(o0 - 1, -1, -1) if backward else range(o0, len(seqs[u0])))]
        for u in w[1:]:
            pos += [(u, c) for c in (range(len(seqs[u]) - 1, -1, -1) if backward else range(len(seqs[u])))]
        if not pos:
            continue
        ref = bytes(seqs[u][c].encode()[0] for u, c in pos)
        for p, row in zip(pos, pinned_rows(ref, q, sc, max_gap)):
            cells[p] = np.maximum(cells[p], row) if p in cells else row
    return cells


def xdrop_expected(seqs, preds, q, sc, seed, max_gap):
    """(score, head) of the two passes of gb_xdrop_dag_batch without pruning: pass 1 from the seed picks the first
    maximum in (node, column, query offset) order as the head, pass 2 is the best pinned alignment ending there."""
    su, so, sq = seed
    m = len(q)
    cells = pinned_cells(seqs, preds, (su, so), q[sq:], sc, max_gap)
    head = (su, so, sq)
    if cells:
        best = max(int(r.max()) for r in cells.values())
        if best > 0:
            u, c = min(p for p, r in cells.items() if r.max() == best)
            head = (u, c + 1, sq + int(np.argmax(cells[(u, c)] == best)))
    hu, ho, hq = head
    if hq == 0:
        return 0, head
    cells2 = pinned_cells(seqs, preds, (hu, ho), q[:hq][::-1], sc, max_gap, backward=True)
    best2 = max((int(r.max()) for r in cells2.values()), default=0)
    return max(best2, 0), head


def no_drop(seqs, q, sc, max_gap):
    """True when no cell of either pass can fall below the X-drop threshold: a cell is never below -(2 go + ge (bases +
    m)) (delete, then insert) and the running maximum never above m match + bonus."""
    match, mism, go, ge, bonus = sc
    m, bases = len(q), sum(len(s) for s in seqs)
    return go + ge * (max(max_gap, 1) - 1) > m * match + bonus + 2 * go + ge * (bases + m)


# ---- path rescorer -------------------------------------------------------------------------------------------------
def rescore(path, seqs, preds, q, sc, rules, right_clip=None):
    """The score of a returned path under a seam's rules, from the path alone; asserts that it is a path of the problem.
    rules: "local" (gb_sw_batch), "global" (gb_banded_global_batch) or "pinned" (gb_xdrop_dag_batch, whose trailing
    insertion edit holds the right soft clip of right_clip bases after any insertion at the head)."""
    match, mism, go, ge, bonus = sc
    q = bytes(q)
    assert path
    for k, (u, off, edits) in enumerate(path):
        assert 0 <= u < len(seqs) and edits and all(n > 0 for _, n, _ in edits)
        used = sum(n for op, n, _ in edits if op in "MSD")
        assert off + used <= len(seqs[u])
        if k + 1 < len(path):
            assert off + used == len(seqs[u]), "a mapping followed by another ends at its node's end"
            assert u in preds[path[k + 1][0]], "consecutive mappings are joined by an edge"
            assert path[k + 1][1] == 0
    flat = []                                           # (node, column, op, length, base) in query order
    for u, off, edits in path:
        c = off
        for op, n, b in edits:
            flat.append((u, c, op, n, b))
            c += n if op in "MSD" else 0
    left = right = 0
    if rules == "global":
        assert path[0][1] == 0 and not preds[path[0][0]] and not successors(preds)[path[-1][0]]
        assert path_end(path, seqs)[1] == len(seqs[path[-1][0]]), "a global path ends at a sink's end"
    else:
        if flat[0][2] == "I":
            left = flat[0][3]; flat = flat[1:]
        if rules == "local" and flat and flat[-1][2] == "I":
            right = flat[-1][3]; flat = flat[:-1]
        if rules == "pinned" and right_clip:
            assert flat and flat[-1][2] == "I" and flat[-1][3] >= right_clip
            right = right_clip
            u, c, op, n, b = flat[-1]
            flat = flat[:-1] + ([(u, c, op, n - right, b)] if n > right else [])
        assert flat and flat[0][2] in "MS" and (rules == "pinned" or flat[-1][2] in "MS"), "soft clips only at the ends"
    qpos, score, prev = left, 0, None
    for u, c, op, n, b in flat:
        if op in "MS":
            for x in range(n):
                qc, rc = q[qpos], seqs[u][c + x].encode()[0]
                n_pair = qc not in b"ACGT" or rc not in b"ACGT"
                if op == "M":
                    assert qc == rc and (rules != "pinned" or not n_pair)
                    score += 0 if (n_pair and rules != "pinned") else match
                else:
                    assert n == 1 and b == ("ACGT"[b"ACGT".index(qc)] if qc in b"ACGT" else "A")
                    assert rules == "pinned" or qc != rc
                    score += 0 if (n_pair and rules != "pinned") else -mism
                qpos += 1
        else:
            score -= n * ge + (go - ge if prev != op else 0)
            qpos += n if op == "I" else 0
        prev = op
    assert qpos + right == len(q), "the path consumes the query exactly"
    if rules == "local":
        score += bonus * ((left == 0) + (right == 0))
    elif rules == "pinned":
        score += bonus * (left == 0 and flat[0][2] in "MS")
    return score


def path_end(path, seqs):
    """(node, offset) right after the last graph base the path consumes."""
    u, off, edits = path[-1]
    return u, off + sum(n for op, n, _ in edits if op in "MSD")


def trailing_insertion(path):
    op, n, _ = path[-1][2][-1]
    return n if op == "I" else 0


# ---- CPU: the DPs on hand-computed cases ---------------------------------------------------------------------------
def test_local_dp_hand_cases():
    sc = SCHEMES["default"]
    assert local_best(b"ACGT", b"ACGT", sc) == 4 + 2 * 5
    assert local_best(b"ACGT", b"TTACGT", sc) == 4 + 5                    # left end soft clipped: one bonus
    assert local_best(b"ANGT", b"ACGT", sc) == 3 + 2 * 5                  # an N pair scores 0
    assert local_best(b"ACGTTTACGT", b"ACGTACGT", sc) == 8 - 6 - 1 + 10   # a 2-base deletion
    assert local_best(b"GGGG", b"A", SCHEMES["no-bonus"]) == 0
    assert local_best(b"GGGG", b"A", sc) == -4 + 2 * 5                   # both bonuses outweigh one mismatch
    assert local_best(b"A", b"A", sc) == 1 + 10                           # a 1-base read earns both bonuses
    assert local_best(b"ACGTACGT", b"ACGTTTACGT", (1, 4, 6, 1, 0)) == 5          # TACGT beats 8 matches with a 2-base insertion
    assert local_best(b"GATTACAGGCCTAGATCCATG", b"GATTACAGGCTTCTAGATCCATG", (1, 4, 6, 1, 0)) == 21 - 7
    assert local_best(b"AAAA", b"AAAA", (1, 1, 1, 1, 0)) == 4


def test_global_dp_hand_cases():
    sc = SCHEMES["no-bonus"]
    assert global_best(b"ACGT", b"ACGT", sc) == 4
    assert global_best(b"ACGT", b"AGT", sc) == 3 - 6
    assert global_best(b"ACG", b"", sc) == -(6 + 2)
    assert global_best(b"AC", b"ACTT", sc) == 2 - 7
    assert global_best(b"ACGT", b"ANGT", sc) == 3
    assert global_best(b"A", b"C", sc) == -4
    assert global_best(b"AAAAAA", b"T", sc) == -4 - 6 - 4                 # one mismatch and a 5-base deletion


def test_pinned_dp_hand_cases():
    sc = SCHEMES["default"]
    assert pinned_rows(b"ACGT", b"ACGT", sc, 30).max() == 4 + 5           # the bonus on the last query base
    assert pinned_rows(b"ACGT", b"ACGA", sc, 30).max() == 3 - 4 + 5
    assert pinned_rows(b"ACNT", b"ACNT", sc, 30).max() == 3 - 4 + 5        # N is a mismatch
    # a leading insertion of one base is allowed at max_gap 1, and at max_gap 0 (taken as 1)
    for gap in (0, 1):
        assert pinned_rows(b"CGT", b"ACGT", sc, gap).max() == -6 + 3 + 5
    assert pinned_rows(b"CGT", b"AACGT", sc, 1).max() < 0
    assert pinned_rows(b"CGT", b"AACGT", sc, 2).max() == -7 + 3 + 5
    rows = pinned_rows(b"ACGT", b"AC", sc, 30)
    assert rows[1, 2] == 2 + 5 and rows[0, 0] == -6 and rows[3, 0] == -9


def test_walk_enumerator():
    preds = [[], [0], [0], [1, 2], [3], [3], [4, 5]]                      # two nested bubbles
    assert sorted(walks(preds)) == [[0, 1, 3, 4, 6], [0, 1, 3, 5, 6], [0, 2, 3, 4, 6], [0, 2, 3, 5, 6]]
    assert sorted(walks_from(preds, 6)) == sorted(w[::-1] for w in walks(preds))
    assert walks([[], [], [0, 1]]) == [[0, 2], [1, 2]]
    assert len(walks([[]] + [[i] for i in range(20)])) == 1
    # ten bubbles in a row: 2^10 walks, refused above the limit
    seqs, preds = bubbles(np.random.default_rng(0), 21, 1, 2, False)
    assert len(walks(preds, limit=1024)) == 1024
    with pytest.raises(TooManyWalks):
        walks(preds, limit=1023)


def test_rescorer_hand_cases():
    seqs, preds = ["ACGT", "T", "G", "CCA"], [[], [0], [0], [1, 2]]
    sc = SCHEMES["default"]
    path = [[0, 0, [["M", 4, ""]]], [2, 0, [["S", 1, "T"]]], [3, 0, [["M", 2, ""], ["I", 2, ""]]]]
    assert rescore(path, seqs, preds, b"ACGTTCCGG", sc, "local") == 6 - 4 + 5
    with pytest.raises(AssertionError):                                   # no edge 1 -> 1
        rescore([[0, 0, [["M", 4, ""]]], [1, 0, [["M", 1, ""]]], [1, 0, [["M", 1, ""]]]], seqs, preds, b"ACGTTT", sc, "local")
    with pytest.raises(AssertionError):                                   # a match on a different base
        rescore([[0, 0, [["M", 4, ""]]], [2, 0, [["M", 1, ""]]]], seqs, preds, b"ACGTT", sc, "local")
    with pytest.raises(AssertionError):                                   # the query is not consumed
        rescore([[0, 0, [["M", 3, ""]]]], seqs, preds, b"ACGT", sc, "local")
    gpath = [[0, 0, [["M", 2, ""], ["D", 2, ""]]], [1, 0, [["D", 1, ""]]], [3, 0, [["M", 3, ""]]]]
    assert rescore(gpath, seqs, preds, b"ACCCA", sc, "global") == 5 - 8
    ppath = [[0, 1, [["I", 1, ""], ["M", 3, ""]]], [1, 0, [["M", 1, ""], ["I", 3, ""]]]]
    assert rescore(ppath, seqs, preds, b"GCGTTAAA", sc, "pinned", right_clip=2) == 4 - 6
    assert rescore(ppath, seqs, preds, b"GCGTTAAA", sc, "pinned", right_clip=3) == 4


# ---- problem families ----------------------------------------------------------------------------------------------
def _rand_seq(rng, n, alphabet="ACGT"):
    return "".join(rng.choice(list(alphabet), size=n))


def mutate(rng, s, sub, indel):
    out = []
    for ch in s:
        r = rng.random()
        if r < sub:
            out.append(str(rng.choice([b for b in "ACGT" if b != ch])))
        elif r < sub + indel / 2:
            continue
        elif r < sub + indel:
            out += [ch, str(rng.choice(list("ACGT")))]
        else:
            out.append(ch)
    return "".join(out)


def bubbles(rng, n_layers, node_len, width=2, nested=False):
    """Layers of `width` parallel nodes between single nodes; nested: each branch is itself a small bubble."""
    seqs, preds, prev = [], [], []
    for layer in range(n_layers):
        if layer % 2 == 0:
            seqs.append(_rand_seq(rng, node_len)); preds.append(list(prev)); prev = [len(seqs) - 1]
            continue
        ends = []
        for _ in range(width):
            seqs.append(_rand_seq(rng, node_len)); preds.append(list(prev)); a = len(seqs) - 1
            if nested:
                seqs += [_rand_seq(rng, 1), _rand_seq(rng, 2)]; preds += [[a], [a]]
                seqs.append(_rand_seq(rng, node_len)); preds.append([a + 1, a + 2]); a = len(seqs) - 1
            ends.append(a)
        prev = ends
    if len(prev) > 1:
        seqs.append(_rand_seq(rng, node_len)); preds.append(list(prev))
    return seqs, preds


def read_on(rng, seqs, preds, m, sub=0.02, indel=0.01, clip=True):
    """A query of length m from a random walk (repeated if short), with errors and sometimes junk at an end."""
    succ = successors(preds)
    u = int(rng.choice([x for x, ps in enumerate(preds) if not ps]))
    hap = seqs[u]
    while succ[u]:
        u = int(rng.choice(succ[u])); hap += seqs[u]
    start = int(rng.integers(0, max(1, len(hap) - m)))
    q = mutate(rng, hap[start:start + m], sub, indel)
    if clip and rng.random() < 0.3:
        q = _rand_seq(rng, int(rng.integers(1, 6))) + q
    q = (q * (m // max(1, len(q)) + 1))[:m] if len(q) < m else q[:m]
    return q


def seed_for(seqs, q, walk_nodes, k=8):
    for u in walk_nodes:
        s = seqs[u]
        for o in range(0, max(0, len(s) - k + 1)):
            x = q.find(s[o:o + k])
            if x >= 0:
                return (u, o, x)
    return None


# ---- CPU: the oracle against the walk DPs and the rescorer ---------------------------------------------------------
def _cpu_families(rng):
    out = []
    for n_layers, node_len, width, nested in [(5, 3, 2, False), (7, 2, 3, False), (5, 4, 2, True), (9, 1, 2, False), (3, 12, 3, True)]:
        for _ in range(4):
            seqs, preds = bubbles(rng, n_layers, node_len, width, nested)
            q = read_on(rng, seqs, preds, int(rng.integers(1, 40)))
            out.append((seqs, preds, q))
    seqs = [_rand_seq(rng, 1, "ACGTN") for _ in range(40)]
    out.append((seqs, [[]] + [[i] for i in range(39)], "".join(seqs[5:30]).replace("C", "N")))
    return out


def _index_of(problems):
    """One index holding every problem's nodes side by side; returns it and the problems' node id lists."""
    all_seqs, ids, paths = [], [], []
    for seqs, preds, *_ in problems:
        base = len(all_seqs)
        all_seqs += seqs
        ids.append([2 * (base + i + 1) for i in range(len(seqs))])
        paths += [[ids[-1][x] for x in w] for w in _dag_walks(preds)]
    return capi.HostIndex(all_seqs, paths, None, k=5, w=3), ids


@pytest.mark.parametrize("scheme", SCHEMES)
def test_oracle_equals_the_walk_dps_on_dag_families(scheme):
    sc = SCHEMES[scheme]
    rng = np.random.default_rng(sorted(SCHEMES).index(scheme))
    problems = _cpu_families(rng)
    index, ids = _index_of(problems)
    scores = capi.Scores(*sc)
    for (seqs, preds, q), nodes in zip(problems, ids):
        got, path, _ = oracle_sw(index, {"node": nodes, "pred": preds}, q, scores)
        assert got == sw_optimum(seqs, preds, q.encode(), sc), (seqs, preds, q)
        if path:
            assert rescore(path, seqs, preds, q.encode(), sc, "local") == got
        status, got, path = oracle_banded(index, nodes, preds, q, len(q) + sum(map(len, seqs)) + 1, False, scores)
        assert status == capi.GB_ITEM_OK and got == global_optimum(seqs, preds, q.encode(), sc)
        assert rescore(path, seqs, preds, q.encode(), sc, "global") == got
        for seed in {seed_for(seqs, q, range(len(seqs)), 3), (0, 0, 0), (len(seqs) - 1, len(seqs[-1]), len(q))} - {None}:
            for gap in (0, 1, 65535):
                got, path = TD.oracle_xdrop_dag(index, nodes, preds, q, scores, seed, gap)
                if gap == 65535 and no_drop(seqs, q, sc, gap):
                    want, head = xdrop_expected(seqs, preds, q.encode(), sc, seed, gap)
                    assert got == want, (seqs, preds, q, seed)
                if path:
                    clip = trailing_insertion(path)
                    assert any(rescore(path, seqs, preds, q.encode(), sc, "pinned", right_clip=k) == got for k in range(clip + 1))


def test_oracle_pinned_pass_equals_the_walk_dp():
    rng = np.random.default_rng(5)
    for scheme, sc in SCHEMES.items():
        for _ in range(6):
            seqs, preds = bubbles(rng, int(rng.integers(3, 8)), int(rng.integers(1, 5)), 2, bool(rng.random() < 0.5))
            q = read_on(rng, seqs, preds, int(rng.integers(1, 30)))
            index, (nodes,) = _index_of([(seqs, preds)])
            u = int(rng.integers(0, len(seqs)))
            o = int(rng.integers(0, len(seqs[u]) + 1))
            for gap in (0, 1, 65535):
                got, _ = TD.oracle_dag_pass(index, nodes, preds, q, capi.Scores(*sc), u, o, gap)
                cells = pinned_cells(seqs, preds, (u, o), q.encode(), sc, gap)
                want = max([int(r.max()) for r in cells.values()] + [0])
                if no_drop(seqs, q, sc, gap):
                    assert got == want, (scheme, seqs, preds, q, u, o, gap)
                else:
                    assert got <= want


def test_oracle_max_gap_zero_allows_a_one_base_leading_insertion():
    """At max_gap 0 the oracle uses the kernels' rule (max_gap 1): a one-base leading insertion, X-drop threshold go."""
    seqs, preds = ["CGT"], [[]]
    index, (nodes,) = _index_of([(seqs, preds)])
    sc = SCHEMES["default"]
    for gap in (0, 1):
        assert TD.oracle_dag_pass(index, nodes, preds, "ACGT", capi.Scores(*sc), 0, 0, gap)[0] == -6 + 3 + 5


# ---- GPU -----------------------------------------------------------------------------------------------------------
MAP_CAP, EDIT_CAP = 2048, 4096


class Runner:
    """Runs problems (seqs, preds, query, seed, max_gap, pad) through the three seams on one device per index and checks
    every answer."""

    def __init__(self):
        self.checked = {"sw": 0, "xdrop_dag": 0, "banded_global": 0, "walk": 0}

    def run(self, problems, sc, seams=("sw", "xdrop_dag", "banded_global"), walk=True, caps=(MAP_CAP, EDIT_CAP)):
        index, ids = _index_of(problems)
        dev = capi.Device(index, scores=capi.Scores(*sc))
        try:
            return self._run(dev, index, ids, problems, sc, seams, walk, caps)
        finally:
            dev.close()

    def _run(self, dev, index, ids, problems, sc, seams, walk, caps):
        scores = capi.Scores(*sc)
        got = {}
        if "sw" in seams:
            got["sw"] = dev.sw_batch([(ids[i], p[1], p[2].encode()) for i, p in enumerate(problems)], *caps, with_status=True)
        if "xdrop_dag" in seams:
            got["xdrop_dag"] = dev.xdrop_dag_batch([(ids[i], p[1], p[2].encode(), p[3], p[4]) for i, p in enumerate(problems)],
                                                   *caps, with_status=True)
        if "banded_global" in seams:
            got["banded_global"] = dev.banded_global_batch([(ids[i], p[1], p[2].encode(), p[5], False) for i, p in enumerate(problems)],
                                                           *caps)
        for i, (seqs, preds, q, seed, gap, pad) in enumerate(problems):
            qb = q.encode()
            try:
                use_walks = walk and len(walks(preds)) <= WALK_LIMIT
            except TooManyWalks:
                use_walks = False
            if "sw" in got:
                st, score, path = got["sw"][i]
                want = oracle_sw(index, {"node": ids[i], "pred": preds}, q, scores)
                assert (st, score, path) == (capi.GB_ITEM_OK, want[0], want[1]), ("sw", i, seqs, preds, q)
                if path:
                    assert rescore(path, seqs, preds, qb, sc, "local") == score
                if use_walks:
                    assert score == sw_optimum(seqs, preds, qb, sc), ("sw walk", i)
                self.checked["sw"] += 1
            if "xdrop_dag" in got:
                st, score, path = got["xdrop_dag"][i]
                want = TD.oracle_xdrop_dag(index, ids[i], preds, q, scores, seed, gap)
                assert (st, score, path) == (capi.GB_ITEM_OK, *want), ("xdrop_dag", i, seqs, preds, q, seed, gap, (st, score, path), want)
                if path:
                    clip = trailing_insertion(path)
                    rescored = {k: rescore(path, seqs, preds, qb, sc, "pinned", right_clip=k) for k in range(clip + 1)}
                    assert score in rescored.values()
                if use_walks and seed is not None:
                    if no_drop(seqs, q, sc, gap):
                        want_score, (hu, ho, hq) = xdrop_expected(seqs, preds, qb, sc, seed, gap)
                        assert score == want_score, ("xdrop walk", i, seqs, preds, q, seed, gap)
                        if path:
                            # the path ends at the head, and its trailing insertion holds the right soft clip
                            end = path_end(path, seqs)
                            assert end == (hu, ho) or (ho == 0 and end[0] in preds[hu] and end[1] == len(seqs[end[0]]))
                            assert rescored[len(q) - hq] == score
                    elif path and trailing_insertion(path) <= 8:
                        u, o = path_end(path, seqs)
                        bound = max(max([int(r.max()) for r in pinned_cells(seqs, preds, (u, o), qb[:hq][::-1], sc, gap, True).values()] + [0])
                                    for hq in range(len(q) - trailing_insertion(path), len(q) + 1))
                        assert score <= bound
                    self.checked["walk"] += 1
                self.checked["xdrop_dag"] += 1
            if "banded_global" in got:
                st, score, path = got["banded_global"][i]
                want = oracle_banded(index, ids[i], preds, q, pad, False, scores)
                assert (st, score, path) == want, ("banded_global", i, seqs, preds, q, pad)
                full = pad >= len(q) + sum(map(len, seqs)) + 1
                if st == capi.GB_ITEM_OK:
                    assert rescore(path, seqs, preds, qb, sc, "global") == score
                else:
                    assert st == capi.GB_ITEM_NO_BAND and not full
                if use_walks:
                    opt = global_optimum(seqs, preds, qb, sc)
                    assert score == opt if full else (st != capi.GB_ITEM_OK or score <= opt)
                    self.checked["walk"] += 1
                self.checked["banded_global"] += 1
        return got


def problem(seqs, preds, q, seed="auto", gap=65535, pad=None):
    if seed == "auto":
        seed = seed_for(seqs, q, range(len(seqs)))
    return (seqs, preds, q, seed, gap, len(q) + sum(map(len, seqs)) + 1 if pad is None else pad)


WIDTHS = [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 511, 512, 513, 1008, 1009, 1023, 1024]


def _width_problem(rng, m):
    # three bubbles (eight walks) holding at least m + 40 bases on every walk
    seqs, preds = bubbles(rng, 7, -(-(m + 40) // 7), 2, False)
    return problem(seqs, preds, read_on(rng, seqs, preds, m, 0.02, 0.01))


@pytest.fixture(scope="module")
def runner():
    return Runner()


@pytest.mark.gpu
def test_query_widths_alone_and_mixed(runner):
    rng = np.random.default_rng(1)
    mixed = []
    for m in WIDTHS:
        p = _width_problem(rng, m)
        runner.run([p], SCHEMES["default"])
        mixed.append(p)
    # one batch: the batch-wide query width puts the short problems in 1024-column warp buffers
    small = [_width_problem(rng, m) for m in WIDTHS if m <= 129]
    runner.run(mixed + small, SCHEMES["default"], walk=False)
    runner.run(small + [mixed[-1]], SCHEMES["default"])


@pytest.mark.gpu
@pytest.mark.parametrize("scheme", SCHEMES)
def test_node_lengths_chains_bubbles_and_n(runner, scheme):
    rng = np.random.default_rng(10 + sorted(SCHEMES).index(scheme))
    problems = []
    for node_len in (1, 2, 31, 32, 33):
        for nested in (False, True):
            seqs, preds = bubbles(rng, 7, node_len, 2, nested)
            problems.append(problem(seqs, preds, read_on(rng, seqs, preds, int(rng.integers(5, 80)))))
    seqs = [_rand_seq(rng, 1024), _rand_seq(rng, 1024), _rand_seq(rng, 1024)]
    preds = [[], [0], [0]]
    problems.append(problem(seqs, preds, mutate(rng, seqs[0][900:] + seqs[2][:100], 0.02, 0.01)))
    # a chain of 600 1-bp nodes and a 1-bp bubble chain
    seqs = [_rand_seq(rng, 1) for _ in range(600)]
    problems.append(problem(seqs, [[]] + [[i] for i in range(599)], mutate(rng, "".join(seqs[100:500]), 0.02, 0.01)))
    seqs, preds = bubbles(rng, 301, 1, 2, False)
    problems.append(problem(seqs, preds, read_on(rng, seqs, preds, 200), gap=40))
    # N in the graph, in the query, and an all-N query
    seqs, preds = bubbles(rng, 9, 6, 2, True)
    seqs = [s[:2] + "N" + s[3:] if i % 3 == 0 else s for i, s in enumerate(seqs)]
    q = read_on(rng, seqs, preds, 40)
    problems.append(problem(seqs, preds, q))
    problems.append(problem(seqs, preds, q[:10] + "NN" + q[12:]))
    problems.append(problem(seqs, preds, "N" * 30, seed=(0, 0, 0)))
    problems.append(problem(seqs, preds, "N" * 30, seed=None))
    runner.run(problems, SCHEMES[scheme])


def _fan(best_at, tie, into):
    """255 four-base branches between a head and a tail node; the branch that matches the read sits at list position
    best_at, or every branch is the same (tie).  into: branches merge into the tail (fan-in), else they end (fan-out)."""
    seqs = ["ACGTAC"] + [("TTGA" if tie or k == best_at else "CCCC") for k in range(255)]
    preds = [[]] + [[0]] * 255
    if into:
        seqs.append("GATCCA")
        preds.append(list(range(1, 256)))
    return seqs, preds


@pytest.mark.gpu
def test_fan_in_and_fan_out_of_255(runner):
    problems = []
    for into in (True, False):
        for tie in (False, True):
            seqs, preds = _fan(254, tie, into)
            q = "ACGTAC" + "TTGA" + ("GATCCA" if into else "")
            for gap in (65535, 3):
                problems.append(problem(seqs, preds, q, seed=(0, 0, 0), gap=gap))
                problems.append(problem(seqs, preds, q, seed=(len(seqs) - 1, len(seqs[-1]), len(q)), gap=gap))
            problems.append(problem(seqs, preds, q, seed=None))
    got = runner.run(problems, SCHEMES["default"])
    # the matching branch (position 254, node 255) or, with every branch alike, the first one (node 1)
    for (seqs, preds, *_), (_, _, path) in zip(problems[::5], got["sw"][::5]):
        assert path[1][0] == (1 if seqs[1] == seqs[255] else 255)


def rescue_problem(rng, n_nodes=640, max_bases=6144, read_len=200, err=0.02, absent=False):
    """A rescue-sized subgraph: nodes in topological order, up to 8 in- and out-edges each among the next 20 nodes."""
    seqs, preds, outdeg = [], [], []
    bases = 0
    for u in range(n_nodes):
        ln = int(rng.integers(1, 2 * max_bases // n_nodes))
        ln = min(ln, max_bases - bases - (n_nodes - u - 1))
        seqs.append(_rand_seq(rng, max(1, ln))); bases += len(seqs[-1])
        cand = [p for p in range(max(0, u - 20), u) if outdeg[p] < 8]
        k = min(len(cand), int(rng.integers(1, 9))) if u else 0
        ps = sorted(int(x) for x in rng.choice(cand, size=k, replace=False)) if k else ([] if not u else [u - 1])
        for p in ps:
            outdeg[p] += 1
        preds.append(ps)
        outdeg.append(0)
    if absent:
        q = _rand_seq(rng, read_len)
    else:
        q = read_on(rng, seqs, preds, read_len, err, err / 2)
    return seqs, preds, q


@pytest.mark.gpu
def test_rescue_sized_subgraphs(runner):
    rng = np.random.default_rng(7)
    problems = []
    for k in range(12):
        seqs, preds, q = rescue_problem(rng, read_len=int(rng.integers(150, 251)), err=float(rng.choice([0.005, 0.02, 0.05])),
                                        absent=k % 4 == 3)
        assert sum(map(len, seqs)) <= 6144 and max(map(len, preds)) <= 8
        problems.append(problem(seqs, preds, q, gap=int(rng.choice([40, 125]))))
        problems.append(problem(seqs, preds, q, seed=None, gap=125))
    runner.run(problems, SCHEMES["default"], walk=False)


@pytest.mark.gpu
def test_xdrop_seeds_seedless_widths_and_max_gap(runner):
    rng = np.random.default_rng(11)
    problems = []
    seqs, preds = bubbles(rng, 9, 5, 2, True)
    q = read_on(rng, seqs, preds, 40, clip=False)
    last = len(seqs) - 1
    for seed in [(0, 0, 0), (0, len(seqs[0]), 0), (last, 0, 0), (last, len(seqs[last]), len(q)), (2, 1, 0), (2, len(seqs[2]), len(q)),
                 seed_for(seqs, q, range(len(seqs)), 4)]:
        for gap in (0, 1, len(q) - 1, len(q), len(q) + 1, 65535):
            problems.append(problem(seqs, preds, q, seed=seed, gap=gap))
    for m in (14, 15, 16):
        for gap in (0, 30):
            problems.append(problem(seqs, preds, read_on(rng, seqs, preds, m), seed=None, gap=gap))
    for scheme in SCHEMES.values():
        runner.run(problems, scheme, seams=("xdrop_dag",))


@pytest.mark.gpu
def test_banded_global_paddings(runner):
    rng = np.random.default_rng(12)
    problems = []
    for _ in range(20):
        seqs, preds = bubbles(rng, int(rng.integers(3, 9)), int(rng.integers(1, 9)), 2, bool(rng.random() < 0.5))
        q = read_on(rng, seqs, preds, int(rng.integers(0, 60)), 0.03, 0.03, clip=False)
        full = len(q) + sum(map(len, seqs)) + 1
        for pad in (0, 1, 4, 16, full - 1, full, 2 ** 31 - 1):
            problems.append(problem(seqs, preds, q, pad=pad))
    for scheme in ("default", "all-ones", "int8-mixed"):
        runner.run(problems, SCHEMES[scheme], seams=("banded_global",))


def _oracle_counts(index, nodes, preds, q, sc, seam, seed=None, gap=30):
    s = capi.Scores(*sc)
    if seam == "sw":
        path = oracle_sw(index, {"node": nodes, "pred": preds}, q, s)[1]
    elif seam == "xdrop_dag":
        path = TD.oracle_xdrop_dag(index, nodes, preds, q, s, seed, gap)[1]
    else:
        path = oracle_banded(index, nodes, preds, q, 10 ** 6, False, s)[2]
    return len(path), sum(len(mp[2]) for mp in path)


@pytest.mark.gpu
def test_output_caps_exact_and_one_below(runner):
    rng = np.random.default_rng(13)
    for k in range(6):
        seqs, preds = bubbles(rng, 11, int(rng.choice([1, 3])), 2, k % 2 == 1)
        q = read_on(rng, seqs, preds, 50, 0.05, 0.04, clip=False)
        index, (nodes,) = _index_of([(seqs, preds)])
        dev = capi.Device(index, scores=capi.Scores(*SCHEMES["default"]))
        seed = seed_for(seqs, q, range(len(seqs)), 4)
        calls = {"sw": lambda mc, ec: dev.sw_batch([(nodes, preds, q.encode())], mc, ec, with_status=True)[0],
                 "xdrop_dag": lambda mc, ec: dev.xdrop_dag_batch([(nodes, preds, q.encode(), seed, 30)], mc, ec, with_status=True)[0],
                 "banded_global": lambda mc, ec: dev.banded_global_batch([(nodes, preds, q.encode(), 10 ** 6, False)], mc, ec)[0]}
        for seam, call in calls.items():
            nm, ne = _oracle_counts(index, nodes, preds, q, SCHEMES["default"], seam, seed)
            if nm == 0:
                continue
            ok = call(nm, ne)
            assert ok[0] == capi.GB_ITEM_OK and len(ok[2]) == nm, seam
            # one below either cap: GB_ITEM_OUT_FULL with score 0 and no mappings
            for mc, ec in ((nm - 1, ne), (nm, ne - 1)):
                if mc and ec:
                    assert call(mc, ec) == (capi.GB_ITEM_OUT_FULL, 0, []), (seam, mc, ec)
        dev.close()


@pytest.mark.gpu
def test_large_batch_and_its_permutation():
    rng = np.random.default_rng(14)
    problems = []
    for k in range(10_000):
        seqs, preds = bubbles(rng, int(rng.integers(1, 6)), int(rng.integers(1, 6)), 2, k % 3 == 0)
        problems.append(problem(seqs, preds, read_on(rng, seqs, preds, int(rng.integers(1, 31))), gap=30))
    index, ids = _index_of(problems)
    sc = SCHEMES["default"]
    dev = capi.Device(index, scores=capi.Scores(*sc))
    perm = rng.permutation(len(problems))
    for seam in ("sw", "xdrop_dag", "banded_global"):
        def call(order):
            if seam == "sw":
                return dev.sw_batch([(ids[i], problems[i][1], problems[i][2].encode()) for i in order], with_status=True)
            if seam == "xdrop_dag":
                return dev.xdrop_dag_batch([(ids[i], problems[i][1], problems[i][2].encode(), problems[i][3], 30) for i in order],
                                           with_status=True)
            return dev.banded_global_batch([(ids[i], problems[i][1], problems[i][2].encode(), problems[i][5], False) for i in order])
        a = call(range(len(problems)))
        b = call(perm)
        assert all(b[k] == a[int(i)] for k, i in enumerate(perm)), seam
        assert all(r[0] == capi.GB_ITEM_OK for r in a)
        # a sample against the oracle
        for i in range(0, len(problems), 97):
            seqs, preds, q, seed, gap, pad = problems[i]
            s = capi.Scores(*sc)
            if seam == "sw":
                want = oracle_sw(index, {"node": ids[i], "pred": preds}, q, s)[:2]
            elif seam == "xdrop_dag":
                want = TD.oracle_xdrop_dag(index, ids[i], preds, q, s, seed, gap)
            else:
                want = oracle_banded(index, ids[i], preds, q, pad, False, s)[1:]
            assert a[i][1:] == tuple(want), (seam, i)
    dev.close()
