"""gb_extend_batch at every workspace, output-stride and read-length limit.

Two references:
  * HaplotypeModel, below: GaplessExtender::extend (vg src/gbwt_extender.cpp:186-737) restated in plain Python over the
    haplotypes themselves, without the GBWT.  Every haplotype and its reverse complement is a list of oriented nodes; a
    search state is the list of occurrences of the current path in those lists, follow_paths groups them by the next
    (or previous) node, and the state size is the occurrence count.  It follows oracle/extend.cpp's canonical order:
    seeds in ascending (node, diag) order, stable sorts.  CPU tests hold the oracle to it.
  * oracle_extend / oracle_extend_limits (oracle/extend.cpp): the GPU is held to them field for field, BWT ranges
    included, and to the GB_ITEM_* status the oracle derives for each capacity, checked in the kernel's order.

The kernel's fixed limits (vg_b200/csrc/device_state.cuh, capi.cu launch_extend) are restated here on purpose: a test
that read them from the code could not notice them change.
"""
from __future__ import annotations

import ctypes as C
import heapq

import numpy as np
import pytest

import helpers as H
from vg_b200 import capi, synth

Q_CAP = 512           # EXTEND_Q_CAP: frontier entries per warp; a push that would fill the last one is refused
A_CAP = 4096          # EXTEND_A_CAP: path-arena nodes per warp, per seed
MAX_READ = 25600      # 8 warps x read length of shared memory must fit in 200 KiB
OK, QUEUE_FULL, OUT_FULL = capi.GB_ITEM_OK, capi.GB_ITEM_QUEUE_FULL, capi.GB_ITEM_OUT_FULL
U32 = 0xFFFFFFFF
_RC = bytes.maketrans(b"ACGT", b"TGCA")


# ---------------------------------------------------------------------------------------------------------------------
# independent model
# ---------------------------------------------------------------------------------------------------------------------
class _Ext:
    __slots__ = ("path", "offset", "lo", "hi", "occ", "score", "lfull", "rfull", "lmax", "rmax", "internal", "old", "mism")

    def copy(self):
        e = _Ext()
        for f in _Ext.__slots__:
            setattr(e, f, getattr(self, f))
        return e


class HaplotypeModel:
    """GaplessExtender::extend over explicit haplotype occurrences (see the module docstring)."""

    def __init__(self, node_seqs, paths):
        self.seq = {}
        for i, s in enumerate(node_seqs, 1):
            b = s.encode() if isinstance(s, str) else bytes(s)
            self.seq[2 * i], self.seq[2 * i + 1] = b, b.translate(_RC)[::-1]
        self.n_handles = 2 * (len(node_seqs) + 1)
        self.hap = []
        for p in paths:
            self.hap.append(list(p))
            self.hap.append([v ^ 1 for v in reversed(p)])
        self.where = {}
        for s, q in enumerate(self.hap):
            for i, v in enumerate(q):
                self.where.setdefault(v, []).append((s, i, i))
        self.visits = None            # set to a list to record every follow_paths call: (path, backward, [(node, size)])

    def length(self, v):
        return len(self.seq[v])

    def occurrences(self, path):
        occ = list(self.where.get(path[0], ()))
        for v in path[1:]:
            occ = [(s, i, j + 1) for s, i, j in occ if j + 1 < len(self.hap[s]) and self.hap[s][j + 1] == v]
        return occ

    def follow(self, path, occ, backward):
        """Successor states in flat GBWT record order: records list their edges by ascending successor, and the backward
        direction walks the record of the reversed first node, so predecessors p come in ascending p ^ 1."""
        groups = {}
        for s, i, j in occ:
            if backward and i > 0:
                groups.setdefault(self.hap[s][i - 1], []).append((s, i - 1, j))
            elif not backward and j + 1 < len(self.hap[s]):
                groups.setdefault(self.hap[s][j + 1], []).append((s, i, j + 1))
        out = sorted(groups.items(), key=lambda kv: (kv[0] ^ 1) if backward else kv[0])
        if self.visits is not None:
            self.visits.append((tuple(path), backward, [(v, len(o)) for v, o in out]))
        return out

    # ---- GaplessExtension helpers, gbwt_extender.cpp:23-117 ----
    def contains(self, e, node, diag):
        ro, no = e.lo, e.offset
        for h in e.path:
            ln = min(self.length(h) - no, e.hi - ro)
            if h == node and ro - no == diag:
                return True
            ro += ln
            no = 0
        return False

    def overlap(self, a, b):
        res, ap, bp, ai, bi, ao, bo = 0, a.lo, b.lo, 0, 0, a.offset, b.offset
        while ap < a.hi and bp < b.hi:
            if ap == bp and a.path[ai] == b.path[bi] and ao == bo:
                ln = min(self.length(a.path[ai]) - ao, a.hi - ap, b.hi - bp)
                res += ln; ap += ln; bp += ln; ai += 1; bi += 1; ao = bo = 0
            elif ap <= bp:
                ap += self.length(a.path[ai]) - ao; ai += 1; ao = 0
            else:
                bp += self.length(b.path[bi]) - bo; bi += 1; bo = 0
        return res

    @staticmethod
    def _score(e, sc):
        e.score = (e.hi - e.lo) * sc.match - e.internal * (sc.match + sc.mismatch) + \
            (e.lfull + e.rfull) * sc.full_length_bonus

    def extend(self, read, seeds, max_mismatches=4, overlap_threshold=0.8, trim=True, scores=None):
        sc = scores or capi.DEFAULT_SCORES
        read = bytes(read)
        if not seeds or not read:
            return []
        seq = bytes(c if c in b"ACGT" else ord("X") for c in read)
        L = len(seq)
        result, best_alignment = [], None
        for node, diag in sorted(set((int(n), int(d)) for n, d in seeds)):
            ro, no = max(diag, 0), max(-diag, 0)
            if not (2 <= node < self.n_handles) or not self.seq[node] or ro > L or no > self.length(node):
                continue
            if best_alignment is not None and result[best_alignment].internal == 0 and \
                    self.contains(result[best_alignment], node, diag):
                continue
            m = _Ext()
            m.path, m.offset, m.lo, m.hi, m.occ = [node], no, ro, ro, self.occurrences([node])
            m.lfull = m.rfull = m.lmax = m.rmax = False
            m.mism = []
            target = self.seq[node]
            m.internal = sum(seq[ro + k] != target[no + k] for k in range(min(L - ro, len(target) - no)))
            m.hi = ro + min(L - ro, len(target) - no)
            m.old = m.internal
            if m.lo == 0:
                m.lfull = m.lmax = True
            if m.hi >= L:
                m.rfull = m.rmax = True
            self._score(m, sc)
            heap, number, best = [(-m.score, 0, m)], 1, None
            while heap:
                curr = heapq.heappop(heap)[2]
                limit = max((max_mismatches + 1) & U32, (max_mismatches // 2 + curr.old + 1) & U32)
                if not curr.rmax:
                    num = 0
                    for v, occ in self.follow(curr.path, curr.occ, False):
                        nx, t, k = curr.copy(), self.seq[v], 0
                        left = min(L - curr.hi, len(t))
                        while k < left:
                            if seq[nx.hi] != t[k]:
                                if nx.internal + 1 >= limit:
                                    break
                                nx.internal += 1
                            nx.hi += 1; k += 1
                        if k == 0:
                            continue
                        nx.path, nx.occ = curr.path + [v], occ
                        if nx.hi >= L:
                            nx.rfull = nx.rmax = True; nx.old = nx.internal
                        elif k < len(t):
                            nx.rmax = True; nx.old = nx.internal
                        self._score(nx, sc)
                        num += len(occ)
                        heapq.heappush(heap, (-nx.score, -number, nx)); number += 1
                    if num < len(curr.occ):
                        curr.rmax = True; curr.old = curr.internal
                        heapq.heappush(heap, (-curr.score, -number, curr)); number += 1
                    continue
                if not curr.lmax:
                    found = False
                    for v, occ in self.follow(curr.path, curr.occ, True):
                        nx, t = curr.copy(), self.seq[v]
                        nx.offset = len(t)
                        while min(nx.lo, nx.offset) > 0:
                            if seq[nx.lo - 1] != t[nx.offset - 1]:
                                if nx.internal + 1 >= limit:
                                    break
                                nx.internal += 1
                            nx.lo -= 1; nx.offset -= 1
                        if nx.offset >= len(t):
                            continue
                        nx.path, nx.occ = [v] + curr.path, occ
                        if nx.lo == 0:
                            nx.lfull = nx.lmax = True
                        elif nx.offset > 0:
                            nx.lmax = True
                        self._score(nx, sc)
                        heapq.heappush(heap, (-nx.score, -number, nx)); number += 1
                        found = True
                    if found:
                        continue
                    curr.lmax = True
                if best is None or best.score < curr.score:
                    best = curr
            if best is not None and best.hi > best.lo:
                best.mism = []
                if best.lfull and best.rfull and (best_alignment is None or best.internal < result[best_alignment].internal):
                    best_alignment = len(result)
                result.append(best)

        if best_alignment is not None and result[best_alignment].internal <= max_mismatches:
            # handle_full_length, gbwt_extender.cpp:301-329 (stable sort)
            result.sort(key=lambda e: (0, e.internal) if (e.lfull and e.rfull) else (1, 0))
            kept = []
            for e in result:
                if not (e.lfull and e.rfull):
                    break
                if not any(self.overlap(e, p) > overlap_threshold * (p.hi - p.lo) for p in kept):
                    kept.append(e)
            result = kept
            self._find_mismatches(seq, result)
        else:
            result = self._remove_duplicates(result)
            self._find_mismatches(seq, result)
            if trim:
                trimmed = [self._trim(e, sc) for e in result]
                if any(trimmed):
                    result = self._remove_duplicates(result)
        return [self._record(e) for e in result]

    @staticmethod
    def _dup_key(e):
        # gbwt_extender.cpp:333-350 orders ties of (interval, end nodes) by GBWT ranges, which this model does not have:
        # it breaks them by path, and compare() treats such runs as sets
        return (e.lo, e.hi, e.path[0] ^ 1 if e.path else -1, e.path[-1] if e.path else -1, tuple(e.path), e.offset)

    def _remove_duplicates(self, result):
        out = []
        for e in sorted(result, key=self._dup_key):
            if e.hi == e.lo:
                continue
            if not out or (out[-1].lo, out[-1].hi, out[-1].offset, out[-1].path) != (e.lo, e.hi, e.offset, e.path):
                out.append(e)
        return out

    def _find_mismatches(self, seq, result):
        for e in result:
            e.mism = []
            if e.internal == 0:
                continue
            no, ro = e.offset, e.lo
            for h in e.path:
                t = self.seq[h]
                while no < len(t) and ro < e.hi:
                    if t[no] != seq[ro]:
                        e.mism.append(ro)
                    no += 1; ro += 1
                no = 0

    def _trim(self, e, sc):
        # gbwt_extender.cpp:421-529
        if not e.mism:
            return False
        mm = e.mism
        cur = [e.lo, mm[0]]
        cs = (cur[1] - cur[0]) * sc.match + (sc.full_length_bonus if e.lfull else 0)
        best, bs = list(cur), cs
        for i in range(len(mm)):
            if cs >= sc.mismatch:
                cur[1] += 1; cs -= sc.mismatch
            else:
                cur = [mm[i] + 1, mm[i] + 1]; cs = 0
            if i + 1 == len(mm):
                cs += (e.hi - cur[1]) * sc.match + (sc.full_length_bonus if e.rfull else 0)
                cur[1] = e.hi
            else:
                cs += (mm[i + 1] - cur[1]) * sc.match
                cur[1] = mm[i + 1]
            if cs > bs or (cs > 0 and cs == bs and cur[1] - cur[0] > best[1] - best[0]):
                best, bs = list(cur), cs
        if best == [e.lo, e.hi]:
            return False
        if best[0] == best[1]:
            e.path, e.lo, e.hi, e.mism, e.score, e.lfull, e.rfull = [], best[0], best[1], [], 0, False, False
            return True
        if best[0] > e.lo:
            e.lfull = False
        if best[1] < e.hi:
            e.rfull = False
        no, ro = e.offset, e.lo
        e.lo, e.hi, e.score = best[0], best[1], bs
        head = 0
        while head < len(e.path):
            ln = self.length(e.path[head])
            ro += ln - no
            no = 0
            if ro > e.lo:
                e.offset = ln - (ro - e.lo)
                break
            head += 1
        tail = head + 1
        while ro < e.hi:
            ro += self.length(e.path[tail]); tail += 1
        if head > 0 or tail < len(e.path):
            e.path = e.path[head:tail]
            e.occ = self.occurrences(e.path)
        e.mism = [p for p in e.mism if e.lo <= p < e.hi]
        return True

    @staticmethod
    def _record(e):
        return {"path": list(e.path), "offset": e.offset, "read_lo": e.lo, "read_hi": e.hi, "score": e.score,
                "left_full": e.lfull, "right_full": e.rfull, "mismatches": list(e.mism), "mismatch_count": len(e.mism),
                "fwd_node": e.path[-1], "bwd_node": e.path[0] ^ 1, "size": len(e.occ)}


def _model_view(ext):
    """An oracle / GPU record in the model's terms: BWT ranges become the state size, which must agree on both sides."""
    s = ext["state"]
    assert s[2] - s[1] == s[5] - s[4], ext
    return {k: ext[k] for k in ("path", "offset", "read_lo", "read_hi", "score", "left_full", "right_full", "mismatches",
                                "mismatch_count")} | {"fwd_node": s[0], "bwd_node": s[3], "size": s[2] - s[1] + 1}


def _same_records(model, oracle):
    """Equal, in order, except that a run of records with the same (read interval, end nodes) is compared as a set
    (remove_duplicates orders such a run by GBWT ranges)."""
    if len(model) != len(oracle):
        return False
    key = lambda r: (r["read_lo"], r["read_hi"], r["bwd_node"], r["fwd_node"])
    if [key(r) for r in model] != [key(r) for r in oracle]:
        return False
    srt = lambda rs: sorted(rs, key=lambda r: (key(r), r["path"], r["offset"]))
    return srt(model) == srt(oracle)


def _model_graphs():
    yield "tiny", synth.make_tiny_graph()
    yield "branchy", synth.make_branchy_graph(n_layers=300, n_haps=6, seed=8)
    for mn in (1, 2, 7, 32, 33, 64):
        yield f"variant max_node={mn}", synth.make_variant_graph(length=3000, n_snp=8, n_ins=3, n_del=3, n_haps=4,
                                                                 seed=30 + mn, max_node=mn)
    yield "variant max_node=1024", synth.make_variant_graph(length=12000, n_snp=4, n_ins=1, n_del=1, n_haps=3, seed=31,
                                                            max_node=1024, min_spacing=1200)


MODEL_GRAPHS = dict(_model_graphs())


def _model_items(g, n, seed):
    rs = synth.simulate_reads(g, n, length=150, sub_rate=0.03, seed=seed)
    items = synth.truth_seeds(g, rs, read_offsets=(0, 41, 90, 149), false_seeds=2, seed=seed)
    return [(bytes(rs.reads[i]), seeds) for i, seeds in items]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the model against the oracle, the oracle's limit report against itself
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(MODEL_GRAPHS))
def test_model_matches_oracle(name):
    g = MODEL_GRAPHS[name]
    index = g.build_index()
    model = HaplotypeModel(g.node_seqs, g.paths)
    settings = [dict(), dict(max_mismatches=1, trim=False), dict(max_mismatches=0, overlap_threshold=0.5),
                dict(max_mismatches=8, scores=capi.Scores(2, 3, 6, 1, 0))]
    items = _model_items(g, 72, seed=len(name))
    n_full = n_trimmed = 0
    for k, (read, seeds) in enumerate(items):
        kw = settings[k % len(settings)]
        want = [_model_view(e) for e in H.oracle_extend(index, read, seeds, max_ext=256, path_cap=65536, mism_cap=8192, **kw)]
        got = model.extend(read, seeds, **kw)
        assert _same_records(got, want), f"{name} item {k} {kw}:\nmodel ={got}\noracle={want}"
        n_full += any(e["left_full"] and e["right_full"] for e in got)
        n_trimmed += any(not (e["left_full"] and e["right_full"]) and e["mismatch_count"] == 0 for e in got)
    assert n_full > len(items) // 3 and n_trimmed > 0, (n_full, n_trimmed)


def test_model_successor_order_matches_flat_gbwt():
    """Every state the model visits has the successors, in the order and with the sizes, that the flat GBWT's
    follow_paths gives the same path (this order sets the extension_number tie-break of the search)."""
    lib = H.oracle_lib()
    for name in ("branchy", "variant max_node=2", "variant max_node=33"):
        g = MODEL_GRAPHS[name]
        index = g.build_index()
        model = HaplotypeModel(g.node_seqs, g.paths)
        model.visits = []
        for read, seeds in _model_items(g, 12, seed=5):
            model.extend(read, seeds)
        assert len(model.visits) > 100
        state = np.zeros(6, dtype=np.int64)
        out = np.zeros(6 * 64, dtype=np.int64)
        for path, backward, succ in model.visits:
            lib.oracle_bd_state(C.byref(index.view), path[0], capi.ptr(state))
            for v in path[1:]:
                n = lib.oracle_follow_paths(C.byref(index.view), capi.ptr(state), 0, capi.ptr(out), 64)
                nxt = [out[6 * j: 6 * j + 6].copy() for j in range(n) if out[6 * j] == v]
                assert len(nxt) == 1, (name, path)
                state[:] = nxt[0]
            assert state[2] - state[1] + 1 == len(model.occurrences(list(path)))
            n = lib.oracle_follow_paths(C.byref(index.view), capi.ptr(state), int(backward), capi.ptr(out), 64)
            gbwt = [(int(out[6 * j + 3]) ^ 1 if backward else int(out[6 * j]), int(out[6 * j + 2] - out[6 * j + 1] + 1))
                    for j in range(n)]
            assert gbwt == succ, (name, path, backward)


@pytest.mark.parametrize("name", ["tiny", "variant max_node=1", "variant max_node=1024"])
def test_model_exact_placement(name):
    """A read copied from a haplotype, seeded once on its true placement: exactly one full-length extension, no
    mismatches, on both the model and the oracle."""
    g = MODEL_GRAPHS[name]
    index = g.build_index()
    model = HaplotypeModel(g.node_seqs, g.paths)
    rs = synth.simulate_reads(g, 40, length=150, sub_rate=0.0, seed=4)
    for k, (i, seeds) in enumerate(synth.truth_seeds(g, rs, read_offsets=(0, 63, 149))):
        seeds = [seeds[k % 3]]
        for res in (model.extend(rs.reads[i], seeds), [_model_view(e) for e in H.oracle_extend(index, rs.reads[i], seeds)]):
            assert len(res) == 1
            e = res[0]
            assert e["left_full"] and e["right_full"] and e["mismatch_count"] == 0 and e["mismatches"] == []
            assert (e["read_lo"], e["read_hi"], e["score"]) == (0, 150, 150 + 2 * capi.DEFAULT_SCORES.full_length_bonus)


def _needs_caps(need):
    """Output strides that hold exactly what the oracle says an item needs (gb_extend_batch refuses a zero stride)."""
    return max(1, need["records"]), max(1, need["path_nodes"]), max(1, need["mismatches"])


@pytest.mark.parametrize("name", ["branchy", "variant max_node=2", "variant max_node=1024"])
def test_oracle_extend_limits_self_consistent(name):
    """At its own needs an item is OK and oracle_extend fits; one below any of them it is refused with the status of
    that capacity; with no capacities the needs never change what oracle_extend returns."""
    g = MODEL_GRAPHS[name]
    index = g.build_index()
    n_checked = 0
    for read, seeds in _model_items(g, 40, seed=9):
        st, need, skip = H.oracle_extend_limits(index, read, seeds)
        assert st == OK and len(skip) == len(seeds)
        q, a = need["frontier"] + 1, need["arena"]
        e, p, m = _needs_caps(need)
        assert H.oracle_extend_limits(index, read, seeds, q, a, e, p, m)[0] == OK
        want = H.oracle_extend(index, read, seeds, max_ext=e, path_cap=p, mism_cap=m)
        assert len(want) <= need["records"] and sum(len(x["path"]) for x in want) <= need["path_nodes"]
        assert sum(x["mismatch_count"] for x in want) <= need["mismatches"]
        if q > 2:                      # the first entry of a seed is pushed without a check
            assert H.oracle_extend_limits(index, read, seeds, q - 1, a, e, p, m)[0] == QUEUE_FULL
        if a > 0:
            assert H.oracle_extend_limits(index, read, seeds, q, a - 1, e, p, m)[0] == QUEUE_FULL
        for k, c in enumerate((e, p, m)):
            if need[("records", "path_nodes", "mismatches")[k]] == c and c > 0:
                caps = [e, p, m]
                caps[k] -= 1
                assert H.oracle_extend_limits(index, read, seeds, q, a, *caps)[0] == OUT_FULL
                n_checked += 1
    assert n_checked > 60


# ---------------------------------------------------------------------------------------------------------------------
# frontier and arena corpus: junk reads on graphs of 1-2 bp nodes and many haplotypes
# ---------------------------------------------------------------------------------------------------------------------
def _dense_graph(n_haps):
    """120 layers of two 1-2 bp alleles, n_haps haplotypes choosing uniformly: every extension step branches."""
    rng = np.random.default_rng(3)
    node_seqs, slots = [], []
    for _ in range(120):
        slots.append([])
        for _ in range(2):
            node_seqs.append(bytes(synth.BASES[rng.integers(0, 4, size=int(rng.integers(1, 3)))]).decode())
            slots[-1].append(len(node_seqs))
    choice = rng.integers(0, 2, size=(n_haps, 120))
    return synth.SynthGraph(node_seqs, [[2 * slots[l][int(choice[h, l])] for l in range(120)] for h in range(n_haps)],
                            None, slots=slots)


def _junk_item(g, i, n_haps):
    """Candidate i: a random read, one seed on a random allele in either orientation, max_mismatches 8, 16 or 60."""
    rng = np.random.default_rng(1000 + i)
    mm, lo, hi = ((8, 16, 100), (16, 14, 40), (60, 10, 30))[i % 3] if n_haps > 500 else \
        ((8, 16, 150), (16, 14, 80), (60, 10, 50))[i % 3]
    L = int(rng.integers(lo, hi + 1))
    read = bytes(synth.BASES[rng.integers(0, 4, size=L)])
    node = 2 * g.slots[int(rng.integers(20, 100))][int(rng.integers(0, 2))] + int(rng.integers(0, 2))
    return mm, read, [(node, int(rng.integers(0, L)))]


# candidates whose peak frontier / arena sits exactly at a bound (found by scanning candidates 0..16000 with the oracle)
_AT_BOUND = {1200: (22, 139, 370, 484), 400: (3860, 5477, 9632)}
_CORPUS_CAPS = (4, 256, 128)


def _bound_corpus():
    """{max_mismatches: (index, [(read, seeds, status, needs)])} over both graphs, as the oracle sees them with the
    kernel's Q_CAP / A_CAP."""
    out = []
    for n_haps, exact in _AT_BOUND.items():
        g = _dense_graph(n_haps)
        index = g.build_index()
        by_mm = {}
        for i in list(range(90)) + list(exact):
            mm, read, seeds = _junk_item(g, i, n_haps)
            st, need, _ = H.oracle_extend_limits(index, read, seeds, Q_CAP, A_CAP, *_CORPUS_CAPS, max_mismatches=mm)
            by_mm.setdefault(mm, []).append((read, seeds, st, need))
        out.append((index, by_mm))
    return out


def _assert_corpus_reaches_bounds(corpus):
    rows = [(st, need) for _, by_mm in corpus for items in by_mm.values() for _, _, st, need in items]
    f_ok = lambda need: need["frontier"] <= Q_CAP - 1
    a_ok = lambda need: need["arena"] <= A_CAP
    assert any(st == OK and n["frontier"] == Q_CAP - 1 and a_ok(n) for st, n in rows)
    assert any(st == QUEUE_FULL and n["frontier"] == Q_CAP and a_ok(n) for st, n in rows)
    assert any(st == OK and n["arena"] == A_CAP and f_ok(n) for st, n in rows)
    assert any(st == QUEUE_FULL and n["arena"] == A_CAP + 1 and f_ok(n) for st, n in rows)
    assert all((st == OK) == (f_ok(n) and a_ok(n)) for st, n in rows)
    assert sum(st == OK for st, _ in rows) > 50 and sum(st == QUEUE_FULL for st, _ in rows) > 25


def test_frontier_and_arena_corpus_reaches_both_sides():
    _assert_corpus_reaches_bounds(_bound_corpus())


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _gpu_run(dev, reads, items, caps, **kw):
    out = dev.extend_batch(reads, items, max_ext=caps[0], path_cap=caps[1], mism_cap=caps[2], **kw)
    return H.gpu_extensions(*out, max_ext=caps[0], with_status=True)


def _oracle_run(index, reads, items, caps, **kw):
    """Per item (status, extensions) as gb_extend_batch must return them: a refused item has no extensions."""
    out = []
    for r, seeds in items:
        st, _, _ = H.oracle_extend_limits(index, reads[r], seeds, Q_CAP, A_CAP, *caps, **kw)
        exts = H.oracle_extend(index, reads[r], seeds, max_ext=caps[0], path_cap=caps[1], mism_cap=caps[2], **kw) \
            if st == OK and seeds and len(reads[r]) else []
        out.append((st, exts))
    return out


def _compare(dev, index, reads, items, caps, what="", **kw):
    got = _gpu_run(dev, reads, items, caps, **{k: v for k, v in kw.items() if k != "scores"})     # scores: the device's
    want = _oracle_run(index, reads, items, caps, **kw)
    bad = [i for i in range(len(items)) if got[i] != want[i]]
    assert not bad, f"{what}: {len(bad)} of {len(items)} items differ; first: item {bad[0]}\n got={got[bad[0]]}\nwant={want[bad[0]]}"
    return got


@pytest.mark.gpu
def test_output_strides_at_need_and_one_below():
    """Each target item run at exactly its record / path-node / mismatch needs is OK; one below any of them it is
    GB_ITEM_OUT_FULL with count 0.  Every item of each batch shares the target's strides, so the neighbours that fit
    (and the others that do not) are checked in the same launch."""
    g = synth.make_variant_graph(length=20000, n_snp=60, n_ins=8, n_del=8, n_haps=6, seed=41, max_node=4)
    index = g.build_index()
    rs = synth.simulate_reads(g, 160, length=150, sub_rate=0.04, seed=42)
    items = synth.truth_seeds(g, rs, read_offsets=(0, 30, 61, 99, 128, 149), false_seeds=4, seed=43)
    reads = [bytes(r) for r in rs.reads]
    needs = [H.oracle_extend_limits(index, reads[r], s)[1] for r, s in items]
    usable = [i for i, n in enumerate(needs) if min(n["records"], n["path_nodes"], n["mismatches"]) >= 2]
    assert len(usable) > 40
    targets = set(max(usable, key=lambda i: needs[i][k]) for k in ("records", "path_nodes", "mismatches"))
    targets |= set(usable[:: max(1, len(usable) // 6)])
    dev = capi.Device(index)
    n_mixed = 0
    for t in sorted(targets):
        caps = _needs_caps(needs[t])
        for k in range(4):
            c = list(caps)
            if k:
                c[k - 1] -= 1
            got = _compare(dev, index, reads, items, tuple(c), what=f"target {t} caps {c}")
            assert got[t][0] == (OK if k == 0 else OUT_FULL) and (k == 0 or got[t][1] == [])
            n_mixed += 0 < sum(s == OK for s, _ in got) < len(items)
    assert n_mixed >= 2 * len(targets), n_mixed
    dev.close()


@pytest.mark.gpu
def test_frontier_and_arena_bounds():
    """The kernel's fixed frontier (Q_CAP entries, one kept free) and per-seed arena (A_CAP nodes): items at the
    bound are OK and equal the oracle, items one past it are GB_ITEM_QUEUE_FULL, as oracle_extend_limits predicts."""
    corpus = _bound_corpus()
    _assert_corpus_reaches_bounds(corpus)
    for index, by_mm in corpus:
        dev = capi.Device(index)
        for mm, rows in by_mm.items():
            reads = [r for r, _, _, _ in rows]
            items = [(i, s) for i, (_, s, _, _) in enumerate(rows)]
            got = _compare(dev, index, reads, items, _CORPUS_CAPS, what=f"max_mismatches {mm}", max_mismatches=mm)
            assert [s for s, _ in got] == [st for _, _, st, _ in rows]
        dev.close()


def _tandem_item(n_seeds, seed):
    """A tandem repeat (a 48 bp unit, 40 copies, every copy but the first with two substitutions) on one haplotype of
    16 bp nodes; the read is exact on copies 0-2.  Seeds: every copy at every read offset (duplicates included), false
    seeds, shuffled, n_seeds in all."""
    rng = np.random.default_rng(seed)
    unit = synth.BASES[np.random.default_rng(77).integers(0, 4, size=48)]
    copies = []
    for c in range(40):
        u = unit.copy()
        if c >= 3:
            at = np.random.default_rng(100 + c).choice(48, size=2, replace=False)
            u[at] = synth.BASES[(np.searchsorted(synth.BASES, u[at]) + 1) % 4]
        copies.append(u)
    hap = np.concatenate(copies)
    node_seqs = [bytes(hap[i:i + 16]).decode() for i in range(0, len(hap), 16)]
    g = synth.SynthGraph(node_seqs, [[2 * (i + 1) for i in range(len(node_seqs))]], None).finish()
    L = 144
    read = bytes(hap[:L])
    pool = [(2 * int(g.hap_node[0][48 * c + o]), o - int(g.hap_off[0][48 * c + o]))
            for c in range(0, 40 - 3) for o in range(L)]
    seeds = [pool[int(j)] for j in rng.integers(0, len(pool), size=n_seeds)]
    for j in range(min(n_seeds, 8)):                       # copy 0 present whatever the sample
        seeds[j] = pool[int(rng.integers(0, L)) if j else 0]
    for j in rng.choice(n_seeds, size=n_seeds // 10, replace=False):
        seeds[int(j)] = (2 * int(rng.integers(1, len(node_seqs) + 1)) + int(rng.integers(0, 2)), int(rng.integers(-16, L)))
    rng.shuffle(seeds)
    for j in range(n_seeds - 1, 0, -97):                   # and in late chunks (the last node of copy 0: never the
        seeds[j] = pool[L - 1]                             # seed that finds the exact extension)
    return g, read, seeds


@pytest.mark.gpu
@pytest.mark.parametrize("n_seeds", [1, 31, 32, 33, 1023, 1024, 1025, 3000])
def test_seed_counts(n_seeds):
    """Seeds inside the first exact full-length extension are skipped: by a bit per 32-seed chunk up to 1024 seeds, by
    GaplessExtension::contains above.  The oracle reports which input positions it skipped."""
    g, read, seeds = _tandem_item(n_seeds, seed=n_seeds)
    index = g.build_index()
    st, need, skip = H.oracle_extend_limits(index, read, seeds, max_mismatches=4)
    assert st == OK and len(skip) == n_seeds
    skipped = [j for j, s in enumerate(skip) if s == 1]
    if n_seeds > 1:
        assert skipped and (n_seeds <= 32 or max(skipped) >= 32), skipped
    if n_seeds > 1024:
        assert max(skipped) >= 1024
    caps = _needs_caps(need)
    dev = capi.Device(index)
    # the item alone, then between two copies of itself with the seeds reversed (same set, other input positions)
    _compare(dev, index, [read], [(0, seeds)], caps, what=f"{n_seeds} seeds", max_mismatches=4)
    _compare(dev, index, [read], [(0, seeds), (0, seeds[::-1]), (0, seeds)], caps, what=f"{n_seeds} seeds x3",
             max_mismatches=4)
    dev.close()


def _truth_seed(g, h, p, L, rev, ro):
    """(node, diag) of read offset ro for a read copied from haplotype h at p (reverse-complemented if rev)."""
    if not rev:
        return 2 * int(g.hap_node[h][p + ro]), ro - int(g.hap_off[h][p + ro])
    hb = p + L - 1 - ro
    nid = int(g.hap_node[h][hb])
    return 2 * nid + 1, ro - (len(g.node_seqs[nid - 1]) - 1 - int(g.hap_off[h][hb]))


def _placed_read(g, rng, L, rev, mutate):
    """A read copied from a haplotype; with mutate, substitutions at both sides of the 32-base warp chunks and at the
    first and last base of the nodes it crosses."""
    h = int(rng.integers(0, len(g.paths)))
    p = int(rng.integers(0, len(g.hap_seq[h]) - L + 1))
    r = g.hap_seq[h][p:p + L].copy()
    if rev:
        r = synth.revcomp_bytes(r)
    if mutate:
        starts = [ro for ro in range(1, L) if g.hap_off[h][p + (L - 1 - ro if rev else ro)] == 0][:6]
        at = sorted({x for x in (31, 32, 63, 64, 511, 512, L - 1) if x < L} | set(starts) | {x - 1 for x in starts})
        r[at] = synth.BASES[(np.searchsorted(synth.BASES, r[at]) + 1) % 4]
    seeds = [_truth_seed(g, h, p, L, rev, ro) for ro in sorted({0, L // 2, L - 1})]
    return bytes(r), seeds


READ_LENGTHS = [1, 31, 32, 33, 64, 150, 512, 513, 1000, 6144, 6145, MAX_READ]


@pytest.fixture(scope="module")
def long_graph():
    g = synth.make_variant_graph(length=60000, n_snp=30, n_ins=4, n_del=4, n_haps=2, seed=51, max_node=1024,
                                 min_spacing=600)
    return g, g.build_index()


@pytest.mark.gpu
def test_read_lengths(long_graph):
    """Every read length class of the kernel: one warp chunk and its neighbours, 512, the last length that fits the
    default 48 KiB of shared memory (6144) and the first that needs the opt-in (6145), and the longest accepted read.
    Then one batch where a single 25600-base read puts every other item on the opt-in path too."""
    g, index = long_graph
    rng = np.random.default_rng(52)
    dev = capi.Device(index)
    short_reads, short_items = [], []
    for L in READ_LENGTHS:
        reads = []
        for rev in (False, True):
            for mutate in (False, True):
                reads.append(_placed_read(g, rng, L, rev, mutate))
        items = [(i, s) for i, (_, s) in enumerate(reads)]
        reads = [r for r, _ in reads]
        for mm in (4, 64):
            caps = tuple(max(c) for c in zip(*(_needs_caps(H.oracle_extend_limits(index, reads[r], s, max_mismatches=mm)[1])
                                              for r, s in items)))
            got = _compare(dev, index, reads, items, caps, what=f"read length {L}, max_mismatches {mm}", max_mismatches=mm)
            assert all(st == OK for st, _ in got)
            if L >= 32:
                assert got[0][1][0]["left_full"] and got[0][1][0]["right_full"] and got[0][1][0]["mismatch_count"] == 0
        if L <= 1000:
            short_items += [(len(short_reads) + r, s) for r, s in items]
            short_reads += reads
    long_read, long_seeds = _placed_read(g, rng, MAX_READ, False, True)
    reads = short_reads + [long_read]
    items = short_items + [(len(short_reads), long_seeds)]
    _compare(dev, index, reads, items, (8, 4096, 1024), what="mixed batch with one 25600-base read", max_mismatches=64)
    dev.close()


@pytest.mark.gpu
def test_read_longer_than_shared_memory_is_refused(long_graph):
    g, index = long_graph
    rng = np.random.default_rng(53)
    read, seeds = _placed_read(g, rng, MAX_READ + 1, False, False)
    dev = capi.Device(index)
    with pytest.raises(capi.GbError) as err:
        dev.extend_batch([b"ACGT", read], [(0, []), (1, seeds)])
    assert err.value.code == capi.GB_ERR_ARG
    assert capi.load_library().gb_last_error().decode() == "read too long for the extension kernel"
    # the device is still usable
    short, sseeds = _placed_read(g, rng, 150, True, True)
    _compare(dev, index, [short], [(0, sseeds)], (8, 256, 128))
    dev.close()


@pytest.mark.gpu
def test_read_masking(long_graph):
    """N, lowercase and IUPAC codes are masked to 'X' (ReadMasker): they never match, and a read carrying them extends
    exactly as the read with 'X' in their place."""
    g, index = long_graph
    rng = np.random.default_rng(54)
    reads, items = [], []
    for k, junk in enumerate((b"N", b"n", b"a", b"c", b"R", b"Y", b"K", b"M", b"S", b"W", b"-", b"*")):
        read, seeds = _placed_read(g, rng, 150, bool(k & 1), False)
        r = bytearray(read)
        for at in sorted({0, 31, 32, 75, 149, 3 * k + 1}):
            r[at] = junk[0]
        reads += [bytes(r), bytes(c if c in b"ACGT" else ord("X") for c in r)]
        items += [(2 * k, seeds), (2 * k + 1, seeds)]
    dev = capi.Device(index)
    for mm in (4, 8):
        got = _compare(dev, index, reads, items, (8, 512, 256), what=f"masking, max_mismatches {mm}", max_mismatches=mm)
        assert all(got[2 * k] == got[2 * k + 1] for k in range(len(items) // 2))
    dev.close()


SWEEP_SCORES = {"default": capi.DEFAULT_SCORES, "no bonus": capi.Scores(1, 4, 6, 1, 0),
                "large bonus": capi.Scores(2, 3, 6, 1, 120)}


@pytest.mark.gpu
@pytest.mark.parametrize("scores", list(SWEEP_SCORES))
def test_parameter_sweep(scores):
    """max_mismatches across the uint32 range (the limit max(mm + 1, mm / 2 + old + 1) wraps at 2^32 - 1), trimming on
    and off, the overlap threshold at both ends, with the default scores and two gb_set_scores sets."""
    sc = SWEEP_SCORES[scores]
    g = synth.make_variant_graph(length=20000, n_snp=60, n_ins=8, n_del=8, n_haps=6, seed=71, max_node=32)
    index = g.build_index()
    rs = synth.simulate_reads(g, 90, length=150, sub_rate=0.05, seed=72)
    items = synth.truth_seeds(g, rs, read_offsets=(0, 40, 80, 120, 149), false_seeds=3, seed=73)
    reads = [bytes(r) for r in rs.reads]
    dev = capi.Device(index, 0, sc)
    n_trimmed = n_full = 0
    for mm in (0, 1, 2, 4, 8, 33, 100, 2 ** 31, 2 ** 32 - 1):
        for trim in (True, False):
            for ov in (0.0, 0.5, 0.8, 1.0):
                got = _compare(dev, index, reads, items, (24, 1024, 512), what=f"mm {mm} trim {trim} overlap {ov}",
                               max_mismatches=mm, trim=trim, overlap_threshold=ov, scores=sc)
                n_full += sum(len(x) > 1 and all(e["left_full"] and e["right_full"] for e in x) for _, x in got)
                n_trimmed += sum(any(not (e["left_full"] or e["right_full"]) for e in x) for _, x in got)
    assert n_full > 0 and n_trimmed > 0
    dev.close()


@pytest.mark.gpu
def test_boundary_seeds():
    """Seeds at the edges of what is valid: diag = read length, diag = -node length, the last base of a node, reverse
    strand; and seeds that are skipped on both sides (node 0, handles past the graph, an empty node, offsets past the
    read or the node), alone or mixed with valid seeds, which must then extend as if the invalid ones were absent."""
    base = synth.make_variant_graph(length=4000, n_snp=10, n_ins=2, n_del=2, n_haps=3, seed=81, max_node=32)
    empty_id = len(base.node_seqs) + 1
    g = synth.SynthGraph(base.node_seqs + [""], base.paths, None).finish()
    index = g.build_index()
    n_handles = 2 * (empty_id + 1)
    rng = np.random.default_rng(82)
    reads, items, valid_only = [], [], []
    for k in range(40):
        L = (150, 33, 1)[k % 3]
        read, seeds = _placed_read(g, rng, L, bool(k & 1), k % 4 == 0)
        v, d = seeds[len(seeds) // 2]
        nlen = len(g.node_seqs[(v >> 1) - 1])
        edge = [(v, L), (v, -nlen), (v ^ 1, L), (seeds[0][0], -nlen)]
        # last base of the node under read offset 0: diag = 0 - (nlen - 1)
        edge.append((seeds[0][0], -(len(g.node_seqs[(seeds[0][0] >> 1) - 1]) - 1)))
        bad = [(0, 0), (1, 0), (n_handles, 0), (n_handles + 1, 3), (0xFFFFFFFF, 0), (2 * empty_id, 0),
               (2 * empty_id + 1, 0), (v, L + 1), (v, -nlen - 1), (v, 2 ** 31 - 1), (v, -2 ** 31)]
        reads.append(read)
        mixed = seeds + edge + bad
        rng.shuffle(mixed)
        items += [(k, mixed), (k, bad), (k, seeds + edge)]
        _, _, skip = H.oracle_extend_limits(index, read, mixed)
        assert [s == 2 for s in skip] == [sd in bad for sd in mixed]
    dev = capi.Device(index)
    got = _compare(dev, index, reads, items, (16, 512, 256), what="boundary seeds")
    for j in range(0, len(items), 3):
        assert got[j] == got[j + 2] and got[j + 1] == (OK, [])
    dev.close()


def _repeat_edge_reads():
    """A 9000-base haplotype (twice) of 32 bp nodes with a 2400-base tandem repeat of a 29-base unit at 3000-5400, and
    150-base reads across either edge of the repeat plus reads elsewhere."""
    rng = np.random.default_rng(61)
    ref = synth.BASES[rng.integers(0, 4, size=9000)]
    unit = synth.BASES[rng.integers(0, 4, size=29)]
    ref[3000:5400] = np.tile(unit, 2400 // 29 + 1)[:2400]
    node_seqs = [bytes(ref[i:i + 32]).decode() for i in range(0, len(ref), 32)]
    g = synth.SynthGraph(node_seqs, [[2 * (i + 1) for i in range(len(node_seqs))]] * 2, None).finish()
    starts = np.concatenate([rng.integers(2880, 2960, size=90), rng.integers(5280, 5360, size=90),
                             rng.integers(0, 2700, size=30), rng.integers(5600, 8850, size=30)])
    reads = np.stack([ref[p:p + 150] for p in starts])
    rev = rng.random(len(starts)) < 0.5
    reads[rev] = synth.revcomp_bytes(reads[rev])
    sub = rng.random(reads.shape) < 0.01
    reads[sub] = synth.BASES[(np.searchsorted(synth.BASES, reads[sub]) + 1) % 4]
    return g, reads, np.full(reads.shape, 30, dtype=np.uint8)


@pytest.mark.gpu
def test_mapper_large_extension_strides():
    """gb_map_batch redoes items whose extensions overflow its regular per-item strides (48 records, 384 path nodes,
    192 mismatches) with large ones (512 / 12288 / 2048), and the align stage reads them from the large pools.

    Reads across an edge of a tandem repeat give clusters with one extension per repeat copy their seeds hit; only the
    true placement is full length.  The oracle's stage dump, fed to oracle_extend_limits, must show items above the
    regular strides.  Reads wholly inside the repeat are left out: each of their copies is a full-length candidate,
    and the align stage's bounded candidate slots, not the extension strides, refuse them.
    No item here exceeds the large strides (asserted from the same counts: at most a few hundred raw records of a few
    path nodes each); a read with such an item would have to carry GB_ITEM_OUT_FULL, which is checked when one occurs."""
    g, reads, quals = _repeat_edge_reads()
    index = g.build_index()
    n = len(reads)
    p = H.default_map_params()
    rr, _, _, _, stage_items, item_seeds = H.oracle_seed_stage(index, reads, quals, p)
    read_class = []
    for r in range(n):
        cls = 0
        for k in range(int(rr[r]["item_cnt"])):
            it = stage_items[int(rr[r]["item_off"]) + k]
            sd = [(int(s["node"]), int(s["diag"])) for s in item_seeds[int(it["seed_off"]): int(it["seed_off"]) + int(it["seed_cnt"])]]
            kw = dict(max_mismatches=p.max_extension_mismatches)
            if H.oracle_extend_limits(index, reads[r], sd, Q_CAP, A_CAP, 48, 384, 192, **kw)[0] != OK:
                st = H.oracle_extend_limits(index, reads[r], sd, Q_CAP, A_CAP, 512, 12288, 2048, **kw)[0]
                cls = max(cls, 1 if st == OK else 2)
        read_class.append(cls)
    assert sum(c == 1 for c in read_class) >= 20, read_class
    assert sum(c == 2 for c in read_class) == 0
    dev = capi.Device(index)
    got = H.gpu_map(dev, reads, quals, p)
    assert any(name == "extend_kernel(large strides)" for name, _ in dev.kernel_times())
    want = H.oracle_map(index, reads, quals, p)
    fits = [r for r in range(n) if read_class[r] < 2]
    bad = H.compare_alignments(got, want, n, indices=fits)
    assert not bad, f"{len(bad)} reads differ; first: {bad[0]}"
    assert all(int(got[3][r]) == OUT_FULL for r in range(n) if read_class[r] == 2)
    dev.close()
