"""The pinned X-drop seam (gb_xdrop_pinned_batch) at the edges of its two kernels: the int16 tile kernel
(xdrop_tile_kernel<R>, R = 2, 4, 6, 8, 12, 16 rows per lane) and the int32 column sweep (xdrop_kernel).

Every batch runs on a device with the tiles and on one created with GIRAFFE_B200_TILES=0 (the sweep alone); both
must return the oracle's score and path.  Which kernel a problem takes follows tile_eligible (xdrop_tile.cuh),
restated below and pinned at its edges without a GPU; on the GPU the launch count shows the route."""
import contextlib
import ctypes as C

import numpy as np
import pytest

import helpers as H
from vg_b200 import capi

# ---- xdrop_tile.cuh: tile_class, tile_scores_fit_int16, tile_eligible, with the same constants ----------------------
TILE_MAX_ROWS, TILE_MAX_NODES, TILE_D_CAP, TILE_TB_BYTES, TILE_SMEM_BYTES = 512, 1024, 256, 512 * 1024, 4096
TILE_MAP_CAP, TILE_EDIT_CAP = 96, 192


def tile_class(m):
    rows = m + 1
    for cls, limit in enumerate((64, 128, 192, 256, 384)):
        if rows <= limit:
            return cls
    return 5


def tile_class_rows(cls):
    return (2, 4, 6, 8, 12, 16)[cls]


def tile_tb_stride(P):
    return 1 if P == 1 else 2 if P == 2 else 4 if P <= 4 else 8


def tile_scores_fit_int16(sc, m, max_gap):
    if m == 0 or m + 1 > TILE_MAX_ROWS:
        return False
    ge, go = sc.gap_extend, sc.gap_open
    if sc.match < 0 or sc.mismatch < 0 or ge < 0 or go < ge or sc.full_length_bonus < 0:
        return False
    xt = go + ge * (max_gap - 1)
    top = m * sc.match + sc.full_length_bonus
    drop = xt + go + (m + 1) * ge + sc.mismatch + sc.match + sc.full_length_bonus
    return top < 12000 and drop < 7000 and top + (m + 1) * ge < 24000


def tile_eligible(sc, m, max_gap, n_nodes, n_bases, max_depth):
    if not tile_scores_fit_int16(sc, m, max_gap):
        return False
    if n_nodes == 0 or n_nodes > TILE_MAX_NODES or max_depth >= TILE_D_CAP or n_bases == 0 or n_bases > 0xffff:
        return False
    R = tile_class_rows(tile_class(m))
    return n_bases * 32 * tile_tb_stride(R // 2) <= TILE_TB_BYTES


def tile_bytes(n_nodes, n_bases, m):
    return 32 + 8 * ((n_nodes + 1) & ~1) + ((n_bases + 15) & ~15) + ((m + 15) & ~15)


def tb_budget(m):
    """The most bases a tree may have for a query of length m to fit the per-warp traceback workspace."""
    return TILE_TB_BYTES // (32 * tile_tb_stride(tile_class_rows(tile_class(m)) // 2))


DEFAULT = capi.DEFAULT_SCORES


# ---- the Python copy at hand-computed values (no GPU) --------------------------------------------------------------
@pytest.mark.parametrize("m,cls", [(1, 0), (63, 0), (64, 1), (127, 1), (128, 2), (191, 2), (192, 3), (255, 3),
                                   (256, 4), (383, 4), (384, 5), (510, 5), (511, 5)])
def test_tile_class_boundaries(m, cls):
    assert tile_class(m) == cls


def test_traceback_budget_per_class():
    # bytes per base and lane: 1, 2, 4, 4, 8, 8 (tile_tb_stride of R / 2 packed registers)
    assert [tb_budget(m) for m in (63, 127, 191, 255, 383, 511)] == [16384, 8192, 4096, 4096, 2048, 2048]
    for m in (1, 63, 64, 127, 128, 191, 192, 255, 256, 383, 384, 511):
        assert tile_eligible(DEFAULT, m, 30, 10, tb_budget(m), 9)
        assert not tile_eligible(DEFAULT, m, 30, 10, tb_budget(m) + 1, 9)


def test_int16_score_limits():
    # top = m match + bonus < 12000: 499 * 24 + 23 = 11999, + 1 = 12000; 255 * 47 + 14 = 11999
    assert tile_scores_fit_int16(capi.Scores(24, 4, 6, 1, 23), 499, 30)
    assert not tile_scores_fit_int16(capi.Scores(24, 4, 6, 1, 24), 499, 30)
    assert tile_scores_fit_int16(capi.Scores(47, 4, 6, 1, 14), 255, 30)
    assert not tile_scores_fit_int16(capi.Scores(47, 4, 6, 1, 15), 255, 30)
    # drop = go + (gap - 1) ge + go + (m + 1) ge + mismatch + match + bonus < 7000: default scores, m = 511:
    # gap + 533 (6999 at gap 6466); m = 255: gap + 277 (6999 at gap 6722)
    assert tile_scores_fit_int16(DEFAULT, 511, 6466) and not tile_scores_fit_int16(DEFAULT, 511, 6467)
    assert tile_scores_fit_int16(DEFAULT, 255, 6722) and not tile_scores_fit_int16(DEFAULT, 255, 6723)
    # query length: 1 .. 511
    assert not tile_scores_fit_int16(DEFAULT, 0, 30) and not tile_scores_fit_int16(DEFAULT, 512, 30)
    # the third inequality never decides: drop >= (m + 1) ge, so top < 12000 and drop < 7000 imply it
    rng = np.random.default_rng(3)
    for _ in range(20000):
        sc = capi.Scores(*(int(x) for x in rng.integers(0, 128, size=5)))
        m, gap = int(rng.integers(1, 512)), int(rng.integers(1, 8000))
        if sc.gap_open < sc.gap_extend:
            continue
        top = m * sc.match + sc.full_length_bonus
        drop = sc.gap_open + sc.gap_extend * (gap - 1) + sc.gap_open + (m + 1) * sc.gap_extend + sc.mismatch + sc.match + sc.full_length_bonus
        assert tile_scores_fit_int16(sc, m, gap) == (top < 12000 and drop < 7000)


def test_structural_limits():
    assert tile_eligible(DEFAULT, 100, 30, 1024, 2000, 10) and not tile_eligible(DEFAULT, 100, 30, 1025, 2000, 10)
    assert tile_eligible(DEFAULT, 100, 30, 300, 2000, 255) and not tile_eligible(DEFAULT, 100, 30, 300, 2000, 256)
    assert not tile_eligible(DEFAULT, 100, 30, 0, 2000, 0) and not tile_eligible(DEFAULT, 100, 30, 1, 0, 0)
    assert tile_bytes(1024, 1536, 60) > TILE_SMEM_BYTES and tile_bytes(200, 3600, 250) > TILE_SMEM_BYTES
    assert tile_bytes(256, 384, 250) <= TILE_SMEM_BYTES


# ---- problems -----------------------------------------------------------------------------------------------------
def _rand_seq(rng, n):
    return "".join("ACGT"[x] for x in rng.integers(0, 4, size=n))


def _revcomp(s):
    return s[::-1].translate(str.maketrans("ACGTN", "TGCAN"))


class Pool:
    """One index whose nodes every problem draws from: 24 random nodes of each length 1 .. 32, 8 nodes of 24 bp with
    an N and 160 more nodes of 32 bp; a problem uses them in either orientation, a node may appear more than once in a
    tree."""

    def __init__(self, seed=7):
        rng = np.random.default_rng(seed)
        self.seqs, self.by_len, self.with_n = [], {L: [] for L in range(1, 33)}, []
        for L in range(1, 33):
            for _ in range(24):
                self.seqs.append(_rand_seq(rng, L))
                self.by_len[L].append(2 * len(self.seqs))
        for _ in range(8):
            s = list(_rand_seq(rng, 24))
            for x in rng.integers(0, 24, size=2):
                s[x] = "N"
            self.seqs.append("".join(s))
            self.with_n.append(2 * len(self.seqs))
        self.distinct = []                  # 160 more of 32 bp: a chain of them repeats no node
        for _ in range(160):
            self.seqs.append(_rand_seq(rng, 32))
            self.distinct.append(2 * len(self.seqs))
        self.index = capi.HostIndex(self.seqs, [[2 * (i + 1) for i in range(len(self.seqs))]], None, k=5, w=3)

    def seq(self, node):
        s = self.seqs[node // 2 - 1]
        return _revcomp(s) if node & 1 else s

    def pick(self, rng, lo, hi=None):
        L = int(rng.integers(lo, (hi if hi is not None else lo) + 1))
        return int(rng.choice(self.by_len[L])) | int(rng.integers(0, 2))


class Tree:
    """A haplotype tree in DFS visit order, built spine first: root .. leaf, each spine node optionally followed by a
    side chain, then further chains hung off the root."""

    def __init__(self):
        self.parents, self.nodes, self.spine = [], [], []

    def add(self, node, parent):
        self.parents.append(parent)
        self.nodes.append(node)
        return len(self.nodes) - 1

    def depth(self):
        d = []
        for p in self.parents:
            d.append(0 if p < 0 else d[p] + 1)
        return max(d)

    def bases(self, pool, trim=0):
        return sum(len(pool.seq(v)) for v in self.nodes) - trim

    def ref(self, pool, trim=0):
        return "".join(pool.seq(self.nodes[i]) for i in self.spine)[trim:]


def spine_tree(pool, rng, need, lo=1, hi=32, side=0.3, side_len=3):
    t, prev, bases = Tree(), -1, 0
    while bases < need:
        x = t.add(pool.pick(rng, lo, hi), prev)
        t.spine.append(x)
        bases += len(pool.seq(t.nodes[x]))
        if prev >= 0 and rng.random() < side:
            p = x
            for _ in range(int(rng.integers(1, side_len + 1))):
                p = t.add(pool.pick(rng, lo, hi), p)
        prev = x
    return t


def chain(pool, rng, n, lo, hi):
    t = Tree()
    for i in range(n):
        t.spine.append(t.add(pool.pick(rng, lo, hi), i - 1))
    return t


def hang_chains(t, pool, rng, lo, hi, chain_len, n_nodes=None, n_bases=None):
    """Chains of chain_len nodes off the root until the tree has n_nodes nodes or exactly n_bases bases."""
    bases = t.bases(pool)
    while (n_nodes is not None and len(t.nodes) < n_nodes) or (n_bases is not None and bases < n_bases):
        p = 0
        for _ in range(chain_len):
            if n_nodes is not None and len(t.nodes) >= n_nodes:
                break
            L = int(rng.integers(lo, hi + 1))
            if n_bases is not None:
                if bases >= n_bases:
                    break
                L = min(L, n_bases - bases)
            p = t.add(int(rng.choice(pool.by_len[L])), p)
            bases += L
    return t


def mutate(rng, ref, m, sub=0.0, ins=0.0, dele=0.0):
    q = []
    for c in ref:
        if len(q) >= m:
            break
        r = rng.random()
        if r < sub:
            q.append("ACGT".replace(c, "")[int(rng.integers(0, 3))] if c in "ACGT" else "A")
        elif r < sub + dele:
            continue
        elif r < sub + dele + ins:
            q += [c, "ACGT"[int(rng.integers(0, 4))]]
        else:
            q.append(c)
    while len(q) < m:
        q.append("ACGT"[int(rng.integers(0, 4))])
    return "".join(q[:m])


def mismatch_all(s):
    return "".join("CGTAA"["ACGTN".index(c)] for c in s)


def problem(t, q, gap, trim=0):
    return (list(t.parents), list(t.nodes), trim, q.encode(), gap)


def eligible(pool, p, sc):
    parents, nodes, trim, q, gap = p
    t = Tree()
    t.parents, t.nodes = parents, nodes
    return tile_eligible(sc, len(q), max(gap, 1), len(nodes), t.bases(pool, trim), t.depth())


# ---- GPU plumbing -------------------------------------------------------------------------------------------------
def oracle_xdrop(index, p, scores):
    """The oracle's pinned X-drop, outputs sized 1024 mappings / 4096 edits.  Its mappings name tree index + 1, as
    Device.xdrop_pinned_batch reports them."""
    lib = H.oracle_lib()
    parents, nodes, trim, q, gap = p
    par = np.asarray(parents, dtype=np.int32)
    nd = np.asarray(nodes, dtype=np.uint32)
    qb = np.frombuffer(bytes(q) + b"\0", dtype=np.uint8).copy()
    score, nm, ne = C.c_int32(), C.c_uint32(), C.c_uint32()
    maps = np.zeros(1024, dtype=H.mapping_dt)
    edits = np.zeros(4096, dtype=np.uint32)
    rc = lib.oracle_xdrop_pinned(C.byref(index.view), C.byref(scores), capi.ptr(par), capi.ptr(nd), len(nd), trim,
                                 capi.ptr(qb), len(q), gap, C.byref(score), capi.ptr(maps), 1024, C.byref(nm),
                                 capi.ptr(edits), 4096, C.byref(ne))
    assert rc == 0
    return score.value, capi.decode_path(maps, edits, nm.value)


def set_scores(dev, sc):
    assert capi.load_library().gb_set_scores(dev.handle, C.byref(sc)) == capi.GB_OK


@pytest.fixture(scope="module")
def pool():
    return Pool()


@pytest.fixture(scope="module")
def devs(pool):
    """{"tiles": the default device, "sweep": a device created with GIRAFFE_B200_TILES=0} on the same index."""
    with contextlib.ExitStack() as stack:
        tiles = capi.Device(pool.index)
        stack.callback(tiles.close)
        with pytest.MonkeyPatch.context() as mp:
            mp.setenv("GIRAFFE_B200_TILES", "0")
            sweep = capi.Device(pool.index)
        stack.callback(sweep.close)
        yield {"tiles": tiles, "sweep": sweep}


def tile_route(launches):
    """The int32 route is one launch (xdrop_kernel); the tile route adds pack_tiles_kernel, one xdrop_tile_kernel per row
    class and unpack_tile_results_kernel."""
    return launches > 1


def run(devs, problems, sc=DEFAULT, map_cap=256, edit_cap=1024):
    """Both devices' (status, score, path) per problem and launches per device."""
    out, launches = {}, {}
    for name, dev in devs.items():
        set_scores(dev, sc)
        before = dev.launches()
        out[name] = dev.xdrop_pinned_batch(problems, map_cap, edit_cap, with_status=True)
        launches[name] = dev.launches() - before
    return out, launches


def check(devs, pool, problems, sc=DEFAULT, what=""):
    """Both devices equal the oracle on every problem; returns the oracle's results and the launches per device."""
    want = [oracle_xdrop(pool.index, p, sc) for p in problems]
    got, launches = run(devs, problems, sc)
    for name in devs:
        for i, (g, w) in enumerate(zip(got[name], want)):
            assert g == (capi.GB_ITEM_OK, w[0], w[1]), (what, name, i, len(problems[i][3]), g[:2], w[0])
    assert launches["sweep"] == 1
    assert tile_route(launches["tiles"]) == any(eligible(pool, p, sc) for p in problems)
    return want, launches


# ---- a. row classes --------------------------------------------------------------------------------------------------
TILE_MS = [1, 63, 64, 127, 128, 191, 192, 255, 256, 383, 384, 510, 511]
SWEEP_MS = [512, 700, 1024]


@pytest.mark.gpu
def test_row_class_boundaries(devs, pool):
    rng = np.random.default_rng(11)
    problems = []
    for m in TILE_MS + SWEEP_MS:
        t = spine_tree(pool, rng, m + 64)
        ref = t.ref(pool)
        for sub, ins, dele in ((0.01, 0, 0), (0.03, 0.01, 0.01), (0.01, 0.04, 0), (0.01, 0, 0.04)):
            problems.append(problem(t, mutate(rng, ref, m, sub, ins, dele), 40))
        q = mutate(rng, ref, m, 0.03, 0.01, 0.01)
        problems.append(problem(t, q[: max(1, m // 2)], 40))
        problems.append(problem(t, q[::-1], 40))
    for p in problems:
        assert eligible(pool, p, DEFAULT) == (len(p[3]) < 512)
    check(devs, pool, problems, what="row classes")


# ---- b. the route of each problem ------------------------------------------------------------------------------------
def _edge_cases():
    """(name, build(pool, rng) -> (problem, scores), tile-eligible)."""
    cases = []

    def spine(m, gap, sc=DEFAULT, sub=0.01):
        def build(pool, rng):
            t = spine_tree(pool, rng, m + 64)
            return problem(t, mutate(rng, t.ref(pool), m, sub, 0.005, 0.005), gap), sc
        return build

    cases += [("m511", spine(511, 30), True), ("m512", spine(512, 30), False)]

    def deep(n):
        def build(pool, rng):
            t = chain(pool, rng, n, 2, 2)
            return problem(t, mutate(rng, t.ref(pool), 300, 0.01), 30), DEFAULT
        return build

    cases += [("depth255", deep(256), True), ("depth256", deep(257), False)]

    def wide(n):
        def build(pool, rng):
            t = spine_tree(pool, rng, 140, 32, 32, side=0)
            hang_chains(t, pool, rng, 1, 1, 10, n_nodes=n)
            return problem(t, mutate(rng, t.ref(pool), 100, 0.01), 30), DEFAULT
        return build

    cases += [("nodes1024", wide(1024), True), ("nodes1025", wide(1025), False)]

    def bases(m, extra):
        def build(pool, rng):
            t = spine_tree(pool, rng, m + 40, 32, 32, side=0)
            hang_chains(t, pool, rng, 24, 32, 20, n_bases=tb_budget(m) + extra)
            return problem(t, mutate(rng, t.ref(pool), m, 0.01), 30), DEFAULT
        return build

    for m in (60, 100, 150, 250, 300, 450):
        R = tile_class_rows(tile_class(m))
        cases += [(f"R{R}-bases{tb_budget(m)}", bases(m, 0), True), (f"R{R}-bases{tb_budget(m) + 1}", bases(m, 1), False)]
    cases += [("top11999-m499", spine(499, 30, capi.Scores(24, 4, 6, 1, 23)), True),
              ("top12000-m499", spine(499, 30, capi.Scores(24, 4, 6, 1, 24)), False),
              ("top11999-m255", spine(255, 30, capi.Scores(47, 4, 6, 1, 14)), True),
              ("top12000-m255", spine(255, 30, capi.Scores(47, 4, 6, 1, 15)), False),
              ("drop6999-m511", spine(511, 6466), True), ("drop7000-m511", spine(511, 6467), False),
              ("drop6999-m255", spine(255, 6722), True), ("drop7000-m255", spine(255, 6723), False)]
    return cases


EDGE_CASES = _edge_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("name,build,is_tile", EDGE_CASES, ids=[c[0] for c in EDGE_CASES])
def test_route_follows_tile_eligible(devs, pool, name, build, is_tile):
    rng = np.random.default_rng(sum(map(ord, name)))
    p, sc = build(pool, rng)
    assert eligible(pool, p, sc) == is_tile
    _, launches = check(devs, pool, [p], sc, what=name)
    assert tile_route(launches["tiles"]) == is_tile


# ---- c. values at the int16 extremes ---------------------------------------------------------------------------------
EXTREME_SCHEMES = [("top11999-m499", 499, capi.Scores(24, 4, 6, 1, 23), 30),
                   ("top11999-m255", 255, capi.Scores(47, 4, 6, 1, 14), 30),
                   ("drop6999-m511", 511, DEFAULT, 6466),
                   ("drop6999-m255", 255, DEFAULT, 6722)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,m,sc,gap", EXTREME_SCHEMES, ids=[s[0] for s in EXTREME_SCHEMES])
def test_values_at_the_int16_extremes(devs, pool, name, m, sc, gap):
    rng = np.random.default_rng(m + gap)
    t = spine_tree(pool, rng, m + 200, side=0.5)
    ref = t.ref(pool)
    g = 40
    problems = [problem(t, ref[:m], gap),                                        # exact copy: score = top
                problem(t, _rand_seq(rng, g) + ref[: m - g], g),                 # leading insertion of max_gap bases
                problem(t, _rand_seq(rng, g + 1) + ref[: m - g - 1], g),         # and one more
                problem(t, mismatch_all(ref[:m]), gap),                          # every column dies
                problem(t, ref[:m // 2] + mismatch_all(ref[m // 2: m]), gap)]
    for d in (g - 1, g, g + 1):                                                  # middle deletions near max_gap
        problems.append(problem(t, ref[: m // 2] + ref[m // 2 + d: m + d], g))
    problems += [problem(t, mutate(rng, ref, m, 0.02, 0.01, 0.01), gap), problem(t, mutate(rng, ref, m, 0.02, 0.01, 0.01), 400)]
    for p in problems:
        assert eligible(pool, p, sc)
    want, _ = check(devs, pool, problems, sc, what=name)
    assert want[0][0] == m * sc.match + sc.full_length_bonus


# ---- d. tile layout: staged and in-place tiles in one class, the double buffer ----------------------------------------
def _in_place_r2(pool, rng):
    t = spine_tree(pool, rng, 80, 1, 2, side=0)
    hang_chains(t, pool, rng, 1, 2, 50, n_nodes=1024)
    return problem(t, mutate(rng, t.ref(pool), 60, 0.02, 0.01, 0.01), 30)


def _in_place_r8(pool, rng):
    t = spine_tree(pool, rng, 280, 18, 18, side=0)
    hang_chains(t, pool, rng, 18, 18, 20, n_nodes=200)
    return problem(t, mutate(rng, t.ref(pool), 250, 0.02, 0.01, 0.01), 30)


def _staged(pool, rng, m):
    t = spine_tree(pool, rng, m + 40, 24, 32)
    return problem(t, mutate(rng, t.ref(pool), m, 0.02, 0.01, 0.01), 30)


def _is_staged(pool, p):
    return tile_bytes(len(p[1]), sum(len(pool.seq(v)) for v in p[1]) - p[2], len(p[3])) <= TILE_SMEM_BYTES


@pytest.mark.gpu
def test_staged_and_in_place_tiles_share_a_class(devs, pool):
    rng = np.random.default_rng(21)
    problems = []
    for big, m in ((_in_place_r2, 60), (_in_place_r8, 250)):
        for pattern in ("BSSBBSBS", "SBBSSBSB"):
            problems += [big(pool, rng) if c == "B" else _staged(pool, rng, m) for c in pattern]
    # a depth-255 chain is still a staged tile
    t = chain(pool, rng, 256, 1, 2)
    problems.append(problem(t, mutate(rng, t.ref(pool), 250, 0.02), 30))
    staged = [_is_staged(pool, p) for p in problems]
    assert staged.count(False) == 16 and staged[-1]
    assert all(eligible(pool, p, DEFAULT) for p in problems)
    check(devs, pool, problems, what="layout")


@pytest.mark.gpu
def test_more_tiles_than_warps(devs, pool):
    """Thousands of small tiles of one class (every resident warp claims several, so each alternates its two stage
    buffers) with in-place tiles among them."""
    rng = np.random.default_rng(22)
    problems = []
    for i in range(3000):
        if i % 75 == 37:
            problems.append(_in_place_r2(pool, rng))
        else:
            t = spine_tree(pool, rng, 90, 4, 32)
            problems.append(problem(t, mutate(rng, t.ref(pool), int(rng.integers(20, 64)), 0.03, 0.01, 0.01), 30))
    assert all(tile_class(len(p[3])) == 0 and eligible(pool, p, DEFAULT) for p in problems)
    check(devs, pool, problems, what="many tiles")


# ---- e. inputs -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_unusual_inputs(devs, pool):
    rng = np.random.default_rng(31)
    problems = []
    for m in (50, 200, 450, 600):
        t = spine_tree(pool, rng, m + 64)
        ref = t.ref(pool)
        q = list(mutate(rng, ref, m, 0.01))
        for x in rng.integers(0, m, size=4):
            q[x] = "N"
        problems.append(problem(t, "".join(q), 30))                              # N in the query
        tn = Tree()
        for i, v in enumerate(t.nodes):                                          # N in the graph
            tn.add(int(rng.choice(pool.with_n)) if i in t.spine[1::3] else v, t.parents[i])
        tn.spine = t.spine
        problems.append(problem(tn, mutate(rng, tn.ref(pool), m, 0.01), 30))
        for gap in (0, 1, m, m + 7, 1000):                                       # max_gap 0 (taken as 1), 1 and >= m
            problems.append(problem(t, mutate(rng, ref, m, 0.01, 0.01, 0.01), gap))
    for L in (1, 32):                                                            # root_trim 0 and len - 1
        for trim in (0, L - 1):
            t = Tree()
            t.spine.append(t.add(int(rng.choice(pool.by_len[L])), -1))
            while t.bases(pool, trim) < 200:
                t.spine.append(t.add(pool.pick(rng, 8, 32), t.spine[-1]))
            problems.append(problem(t, mutate(rng, t.ref(pool, trim), 150, 0.02), 30, trim))
    t = spine_tree(pool, rng, 40)
    ref = t.ref(pool)
    problems += [problem(t, q, 30) for q in (ref[0], mismatch_all(ref[0]), "N")]  # 1-base queries
    check(devs, pool, problems, what="inputs")


# ---- f. paths longer than a tile holds -------------------------------------------------------------------------------
SCHEME_F = capi.Scores(4, 2, 6, 1, 5)       # one mismatch in three bases still scores


def _long_paths(pool):
    rng = np.random.default_rng(41)
    t = chain(pool, rng, 150, 2, 2)          # 150 mappings
    many_maps = problem(t, t.ref(pool)[:300], 30)
    t = spine_tree(pool, rng, 500, 32, 32, side=0)
    ref = t.ref(pool)
    many_edits = problem(t, "".join(mismatch_all(c) if i % 3 == 2 else c for i, c in enumerate(ref[:450])), 30)
    return many_maps, many_edits


@pytest.mark.gpu
def test_paths_longer_than_a_tile_holds(devs, pool):
    many_maps, many_edits = _long_paths(pool)
    assert eligible(pool, many_maps, SCHEME_F) and eligible(pool, many_edits, SCHEME_F)
    want, _ = check(devs, pool, [many_maps, many_edits], SCHEME_F, what="long paths")
    assert len(want[0][1]) > TILE_MAP_CAP
    assert sum(len(mp[2]) for mp in want[1][1]) > TILE_EDIT_CAP


def _steps(path):
    """Traceback steps of a path: query bases plus deleted bases."""
    return sum(ed[1] for mp in path for ed in mp[2])


def _long_deletion(pool, m, d):
    """A chain of distinct 32-bp nodes and a query made of its first m - m // 2 bases and the m // 2 bases after a d-base gap."""
    t = Tree()
    for i, v in enumerate(pool.distinct[: (m + d) // 32 + 2]):
        t.spine.append(t.add(v, i - 1))
    ref = t.ref(pool)
    a = m - m // 2
    return problem(t, ref[:a] + ref[a + d: a + d + m // 2], 4000)


SCHEME_DEL = capi.Scores(20, 127, 100, 1, 127)      # gaps open at 100 and mismatches cost 127: one long deletion wins


@pytest.mark.gpu
def test_traceback_step_limit_is_the_same_on_both_routes(devs, pool):
    """Both kernels follow at most 4096 traceback steps (query bases plus deleted bases).  A 1800-base deletion at
    m = 255 (2055 steps) fits a tile and the sweep alike; at m = 383 (the sweep, within its 2^21 traceback cells),
    4096 steps are aligned and 4097 are GB_ITEM_OUT_FULL on both devices."""
    p = _long_deletion(pool, 255, 1800)
    assert eligible(pool, p, SCHEME_DEL)
    want, _ = check(devs, pool, [p], SCHEME_DEL, what="1800-base deletion")
    assert _steps(want[0][1]) == 255 + 1800
    at_cap, over = (_long_deletion(pool, 383, d) for d in (4096 - 383, 4097 - 383))
    want, _ = check(devs, pool, [at_cap], SCHEME_DEL, what="4096 steps")
    assert _steps(want[0][1]) == 4096
    assert _steps(oracle_xdrop(pool.index, over, SCHEME_DEL)[1]) == 4097
    got, _ = run(devs, [over], SCHEME_DEL)
    for name in devs:
        assert got[name][0][0] == capi.GB_ITEM_OUT_FULL, name


@pytest.mark.gpu
def test_paths_longer_than_the_callers_caps(devs, pool):
    many_maps, many_edits = _long_paths(pool)
    rng = np.random.default_rng(42)
    t = chain(pool, rng, 20, 16, 16)          # 20 mappings: the tile holds it, the caller's cap of 10 does not
    short = problem(t, t.ref(pool)[:300], 30)
    for p, map_cap, edit_cap in ((many_maps, 100, 1024), (many_edits, 256, 250), (short, 10, 1024), (short, 256, 1)):
        got, _ = run(devs, [p], SCHEME_F, map_cap, edit_cap)
        for name in devs:
            assert got[name][0][0] == capi.GB_ITEM_OUT_FULL, (name, map_cap, edit_cap)


# ---- g. input checks -------------------------------------------------------------------------------------------------
def refused(dev, problems, code=capi.GB_ERR_ARG):
    before = dev.launches()
    with pytest.raises(capi.GbError) as e:
        dev.xdrop_pinned_batch(problems)
    assert e.value.code == code
    assert dev.launches() == before


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["tiles", "sweep"])
def test_refuses_malformed_trees(devs, pool, which):
    dev = devs[which]
    set_scores(dev, DEFAULT)
    a, b, c = pool.by_len[32][:3]
    q = (pool.seq(a) + pool.seq(b)).encode()
    good = ([-1, 0, 1], [a, b, c], 0, q, 30)
    for bad in (0, 1, pool.index.view.n_nodes, pool.index.view.n_nodes + 1):        # unknown node
        refused(dev, [good, ([-1, 0, 1], [a, bad, c], 0, q, 30)])
    refused(dev, [([-1, 1, 1], [a, b, c], 0, q, 30)])                             # parent not below its own index
    refused(dev, [([-1, 0, 3], [a, b, c], 0, q, 30)])
    refused(dev, [([0, -1, 1], [a, b, c], 0, q, 30)])                             # first node not a root
    refused(dev, [([-1, 0, -1], [a, b, c], 0, q, 30)])                            # a second root
    refused(dev, [([-1, 0, 0, 1], [a, b, c, a], 0, q, 30)])                        # not in DFS visit order
    refused(dev, [([], [], 0, q, 30)])                                            # no nodes
    refused(dev, [([-1, 0, 1], [a, b, c], 32, q, 30)])                            # root_trim >= root length
    deep = ([-1] + list(range(512)), [a] * 513, 0, q, 30)                         # a node 512 levels down
    refused(dev, [deep])
    refused(dev, [([-1, 0, 1], [a, b, c], 0, (q * 20)[:1025], 30)])               # a 1025-base query
    # the accepted neighbours
    before = dev.launches()
    dev.xdrop_pinned_batch([([-1, 0, 1], [a, b, c], 31, q, 30), ([-1, 0, 0], [a, b, c], 0, q, 30),
                            ([-1] + list(range(511)), [a] * 512, 0, q, 30),
                            ([-1, 0, 1], [a, b, c], 0, (q * 20)[:1024], 30)])
    assert dev.launches() > before


def _raw_call(dev, n, map_cap, edit_cap):
    lib = capi.load_library()
    par = np.full(16, -1, dtype=np.int32); u32 = np.full(16, 2, dtype=np.uint32); off = np.zeros(16, dtype=np.uint64)
    q = np.zeros(16, dtype=np.uint8)
    outs = capi._seam_outputs(16, 16, 16)
    return lib.gb_xdrop_pinned_batch(dev.handle, n, capi.ptr(par), capi.ptr(u32), capi.ptr(off), capi.ptr(np.zeros(16, dtype=np.uint32)),
                                     capi.ptr(q), capi.ptr(off), capi.ptr(u32), map_cap, edit_cap, *map(capi.ptr, outs))


@pytest.mark.gpu
def test_empty_batch_and_zero_caps(devs):
    dev = devs["tiles"]
    before = dev.launches()
    assert _raw_call(dev, 0, 16, 16) == capi.GB_OK
    assert _raw_call(dev, 1, 0, 16) == capi.GB_ERR_ARG
    assert _raw_call(dev, 1, 16, 0) == capi.GB_ERR_ARG
    assert dev.launches() == before
