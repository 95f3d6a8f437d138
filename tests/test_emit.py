"""gb_emit_gaf / gb_emit_json: host-side text emission of alignment records (the AlignmentEmitter stand-in,
giraffe_main.cpp:2209-2226).  libvgio is absent from the reference tree, so these tests check the text against
the records and the graph: replaying a GAF line's cs string along its path must reproduce the aligned part of the
read, and a JSON line must decode to the same path / edits as the binary record (vg.proto field names)."""
import base64
import ctypes as C
import json
import re
import types

import numpy as np

import helpers as H
from vg_b200 import capi, synth

COMP = {"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}
MAPPED, SEC, PAIRED, RESCUED, ABSENT = capi.GB_ALN_MAPPED, capi.GB_ALN_SECONDARY, capi.GB_ALN_PAIRED, capi.GB_ALN_RESCUED, capi.GB_ALN_ABSENT


def _oriented_seq(g, v):
    s = g.node_seqs[(v >> 1) - 1]
    return "".join(COMP[c] for c in reversed(s)) if v & 1 else s


def _records(paired):
    g = synth.make_variant_graph(length=60000, n_snp=100, n_ins=12, n_del=12, n_haps=4, seed=8)
    index = g.build_index()
    if paired:
        rs = synth.simulate_pairs(g, 150, sub_rate=0.02, seed=5)
    else:
        rs = synth.simulate_reads(g, 300, length=150, sub_rate=0.02, ins_rate=0.004, del_rate=0.004, seed=6)
    rng = np.random.default_rng(1)
    for i in rng.integers(0, rs.n, size=20):                   # soft clips: garbage at one end
        rs.reads[i, :12] = synth.BASES[rng.integers(0, 4, size=12)]
    rs.reads[7] = synth.BASES[rng.integers(0, 4, size=rs.length)]      # an unmapped read
    if paired:
        res = H.oracle_map_paired(index, rs.reads, rs.quals, H.paired_params(), threads=8)
    else:
        res = H.oracle_map(index, rs.reads, rs.quals, threads=8)
    return g, index, rs, res


def _replay_gaf(f, tags, read, oriented, real=True):
    """Walks the cs string of the mapped GAF line f along its path: every base and column must agree with the read and the
    graph.  real=False for hand-made records, whose match runs are not real matches: those are not compared with the read.
    -> (path steps, cs tokens)"""
    steps = [(int(x[1:]) << 1) | (x[0] == "<") for x in re.findall(r"[<>]\d+", f[5])]
    ref = "".join(oriented(v) for v in steps)
    assert int(f[6]) == len(ref)
    pos, q, matches, block = int(f[7]), 0, 0, 0
    tokens = [(m[0] or m[2] or m[4] or m[6], m[1] or m[3] or m[5] or m[7])
              for m in re.findall(r"(:)(\d+)|(\*)([A-Z]{2})|(\+)([A-Z]+)|(-)([A-Z]+)", tags["cs"])]
    assert "".join(op + arg for op, arg in tokens) == tags["cs"]
    assert not any(a[0] == ":" and b[0] == ":" for a, b in zip(tokens, tokens[1:]))     # match runs are merged
    for op, arg in tokens:
        if op == ":":
            n = int(arg)
            assert not real or ref[pos:pos + n] == read[q:q + n]
            pos += n; q += n; matches += n; block += n
        elif op == "*":
            assert ref[pos] == arg[0] and read[q] == arg[1] and (not real or arg[0] != arg[1])
            pos += 1; q += 1; block += 1
        elif op == "+":
            assert read[q:q + len(arg)] == arg
            q += len(arg); block += len(arg)
        else:
            assert ref[pos:pos + len(arg)] == arg
            pos += len(arg); block += len(arg)
    assert q == len(read), (q, len(read))
    assert pos == int(f[8]) and matches == int(f[9]) and block == int(f[10])
    assert abs(float(tags["dv"]) - (1 - matches / block)) < 1e-5
    return steps, tokens


def _check_gaf(g, rs, res, text, paired, names):
    lines = text.splitlines()
    assert len(lines) == rs.n
    n_clipped = n_indel = 0
    for i, line in enumerate(lines):
        f = line.split("\t")
        read = bytes(rs.reads[i]).decode()
        assert f[0] == names[i] and int(f[1]) == rs.length
        assert (int(f[2]), int(f[3])) == (0, rs.length)                  # the whole read, soft clips included
        score, mapq, path = H.decode_alignment(res[0][i], res[1], res[2])
        tags = {t[:2]: t[5:] for t in f[12:]}
        if paired:
            assert tags["fn" if i % 2 == 0 else "fp"] == names[i ^ 1]
        if not path:
            assert f[4:12] == ["*"] * 7 + ["255"] and tags["cs"] == "+" + read
            continue
        assert f[4] == "+" and int(f[11]) == mapq and int(tags["AS"]) == score
        steps, tokens = _replay_gaf(f, tags, read, lambda v: _oriented_seq(g, v))
        assert steps == [m[0] for m in path if any(e[0] != "I" for e in m[2])]
        assert tags["bq"] == "".join(chr(int(c) + 33) for c in rs.quals[i])
        n_indel += sum(op in "+-" for op, _ in tokens)
        n_clipped += tokens[0][0] == "+" or tokens[-1][0] == "+"
    return n_clipped, n_indel


def _hand_record(mappings):
    """mappings: [(oriented node, offset, [(op, length, base2)...])] -> (aln[1], maps, edits) as the library lays them out."""
    aln = np.zeros(1, dtype=capi.alignment_dt)
    maps = np.zeros(len(mappings), dtype=capi.mapping_dt)
    words = []
    for i, (node, off, eds) in enumerate(mappings):
        maps[i]["node"] = node; maps[i]["offset"] = off; maps[i]["n_edits"] = len(eds)
        for op, ln, base in eds:
            words.append((ln << 4) | (base << 2) | "MSID".index(op))
    aln[0]["read_id"] = 0; aln[0]["flags"] = capi.GB_ALN_MAPPED if mappings else 0
    aln[0]["n_mappings"] = len(mappings); aln[0]["n_edits"] = len(words); aln[0]["score"] = 7; aln[0]["mapq"] = 60
    return aln, maps if len(maps) else np.zeros(1, dtype=capi.mapping_dt), np.array(words + [0], dtype=np.uint32)


def test_gaf_reference_vector_unused_final_node_is_removed():
    """unittest/alignment.cpp:398-470: GATTACA -> CAT -> GATTA, read TACACTTAC = TACA on 1:3, C *AT T on 2:0, AC soft-clipped
    onto node 3: query 0..9, path >1>2 of length 10, start 3, end 10, cs ":5*AT:1+AC"."""
    index = capi.HostIndex(["GATTACA", "CAT", "GATTA"], [[2, 4, 6]], None, k=5, w=3)
    aln, maps, edits = _hand_record([(2, 3, [("M", 4, 0)]), (4, 0, [("M", 1, 0), ("S", 1, 3), ("M", 1, 0)]), (6, 0, [("I", 2, 0)])])
    rbuf, qbuf, read_off = H.pack_reads(np.frombuffer(b"TACACTTAC", dtype=np.uint8).reshape(1, -1).copy(), None)
    f = capi.emit_text("gaf", index.view, aln, maps, edits, rbuf, None, read_off, ["softclip-at-end"]).rstrip("\n").split("\t")
    assert f[:9] == ["softclip-at-end", "9", "0", "9", "+", ">1>2", "10", "3", "10"]
    assert dict(t.split(":", 2)[::2] for t in f[12:])["cs"] == ":5*AT:1+AC"


def test_gaf_reference_vector_unaligned_read():
    """unittest/alignment.cpp:793-820: no path, query 0..9, cs "+TACACTTAC"."""
    index = capi.HostIndex(["GATTACA", "CAT", "GATTA"], [[2, 4, 6]], None, k=5, w=3)
    aln, maps, edits = _hand_record([])
    rbuf, qbuf, read_off = H.pack_reads(np.frombuffer(b"TACACTTAC", dtype=np.uint8).reshape(1, -1).copy(), None)
    f = capi.emit_text("gaf", index.view, aln, maps, edits, rbuf, None, read_off, ["unaligned"]).rstrip("\n").split("\t")
    assert f[:4] == ["unaligned", "9", "0", "9"] and f[5] == "*"
    assert dict(t.split(":", 2)[::2] for t in f[12:])["cs"] == "+TACACTTAC"


def test_gaf_lines_replay_to_the_reads_single_end():
    g, index, rs, res = _records(paired=False)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    names = [f"frag{i}" for i in range(rs.n)]
    text = capi.emit_text("gaf", index.view, res[0], res[1], res[2], rbuf, qbuf, read_off, names)
    n_clipped, n_indel = _check_gaf(g, rs, res, text, False, names)
    assert n_clipped >= 5 and n_indel >= 20          # soft clips and gapped alignments were exercised


def test_gaf_lines_replay_to_the_reads_paired():
    g, index, rs, res = _records(paired=True)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    names = [f"pair{i // 2}/{i % 2 + 1}" for i in range(rs.n)]
    text = capi.emit_text("gaf", index.view, res[0], res[1], res[2], rbuf, qbuf, read_off, names)
    _check_gaf(g, rs, res, text, True, names)
    # default names, a subset of the records in another order
    sub = res[0][[5, 2, 9]]
    lines = capi.emit_text("gaf", index.view, sub, res[1], res[2], rbuf, qbuf, read_off).splitlines()
    assert [l.split("\t")[0] for l in lines] == ["read5", "read2", "read9"]


def test_json_lines_decode_to_the_records():
    g, index, rs, res = _records(paired=True)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    names = [f"pair{i // 2}/{i % 2 + 1}" for i in range(rs.n)]
    text = capi.emit_text("json", index.view, res[0], res[1], res[2], rbuf, qbuf, read_off, names)
    lines = text.splitlines()
    assert len(lines) == rs.n
    for i, line in enumerate(lines):
        d = json.loads(line)
        read = bytes(rs.reads[i]).decode()
        score, mapq, path = H.decode_alignment(res[0][i], res[1], res[2])
        assert d["sequence"] == read and d["name"] == names[i]
        assert base64.b64decode(d["quality"]) == bytes(rs.quals[i])
        assert d.get("score", 0) == score and d.get("mapping_quality", 0) == mapq
        assert d["fragment_next" if i % 2 == 0 else "fragment_prev"]["name"] == names[i ^ 1]
        if not path:
            assert "path" not in d
            continue
        q = 0
        assert len(d["path"]["mapping"]) == len(path)
        for rank, (mj, (node, offset, edits)) in enumerate(zip(d["path"]["mapping"], path), 1):
            pos = mj["position"]
            assert int(pos["node_id"]) == node >> 1 and int(pos.get("offset", "0")) == offset and pos.get("is_reverse", False) == bool(node & 1)
            assert mj["rank"] == str(rank) and len(mj["edit"]) == len(edits)
            for ej, (op, length, base) in zip(mj["edit"], edits):
                fl, tl = ej.get("from_length", 0), ej.get("to_length", 0)
                if op == "M":
                    assert (fl, tl) == (length, length) and "sequence" not in ej
                elif op == "S":
                    assert (fl, tl) == (1, 1) and ej["sequence"] == read[q]
                elif op == "I":
                    assert (fl, tl) == (0, length) and ej["sequence"] == read[q:q + length]
                else:
                    assert (fl, tl) == (length, 0)
                q += tl
        assert q == rs.length
        assert 0.0 < d["identity"] <= 1.0


def test_emit_reports_a_short_buffer():
    import ctypes as C
    g, index, rs, res = _records(paired=False)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    out = np.zeros(64, dtype=np.uint8); used = C.c_uint64()
    lib = capi.load_library()
    args = lambda aln, n_maps, n_edits, n_reads: (C.byref(index.view), len(aln), capi.ptr(aln), capi.ptr(res[1]), n_maps, capi.ptr(res[2]), n_edits, n_reads,
                                                  capi.ptr(rbuf), capi.ptr(qbuf), capi.ptr(read_off), None, None, capi.ptr(out), 64, C.byref(used))
    ten = np.ascontiguousarray(res[0][:10])
    assert lib.gb_emit_gaf(*args(ten, len(res[1]), len(res[2]), rs.n)) == capi.GB_ERR_CAPACITY


def test_emit_refuses_records_that_point_outside_their_pools():
    import ctypes as C
    g, index, rs, res = _records(paired=False)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    lib = capi.load_library()
    out = np.zeros(1 << 20, dtype=np.uint8); used = C.c_uint64()

    def emit(fn, aln, n_maps=len(res[1]), n_edits=len(res[2]), n_reads=rs.n):
        aln = np.ascontiguousarray(aln)
        return fn(C.byref(index.view), len(aln), capi.ptr(aln), capi.ptr(res[1]), n_maps, capi.ptr(res[2]), n_edits, n_reads, capi.ptr(rbuf), capi.ptr(qbuf),
                  capi.ptr(read_off), None, None, capi.ptr(out), len(out), C.byref(used))

    mapped = res[0][(res[0]["flags"] & 1) != 0][:20]
    for fn in (lib.gb_emit_gaf, lib.gb_emit_json, lib.gb_emit_gam):
        assert emit(fn, mapped) == capi.GB_OK
        assert emit(fn, mapped, n_maps=int(mapped["mapping_off"].max())) == capi.GB_ERR_ARG                  # mapping pool shorter than a record needs
        assert emit(fn, mapped, n_edits=int(mapped["edit_off"].max())) == capi.GB_ERR_ARG
        assert emit(fn, mapped, n_reads=int(mapped["read_id"].max())) == capi.GB_ERR_ARG                     # read id outside the batch
        bad = mapped.copy(); bad[3]["n_edits"] += 1                                                          # edits no longer add up to the read
        assert emit(fn, bad) == capi.GB_ERR_ARG
        bad = mapped.copy(); bad[5]["mapping_off"] = bad[6]["mapping_off"]                                   # another record's mappings
        assert emit(fn, bad) == capi.GB_ERR_ARG


# ---- hand-made records (test_emit_device.py sends the same records through the device emitters) ----------------------
def _names_t(names):
    enc = [s.encode() for s in names]
    off = np.concatenate([[0], np.cumsum([len(b) for b in enc])]).astype(np.int64)
    return np.frombuffer(b"".join(enc) + b"\0", dtype=np.uint8).copy(), off


def _host(kind, view, aln, maps, edits, rbuf, qbuf, read_off, names=None, cap=None):
    """gb_emit_gaf / gb_emit_gam into a buffer of `cap` bytes (default: generous for short reads)."""
    lib = capi.load_library()
    fn = {"gaf": lib.gb_emit_gaf, "gam": lib.gb_emit_gam}[kind]
    nbuf, noff = _names_t(names) if names is not None else (None, None)
    aln = np.ascontiguousarray(aln)
    cap = cap or 4096 + len(aln) * 4096
    out = np.zeros(cap, dtype=np.uint8); used = C.c_uint64()
    rc = fn(C.byref(view), len(aln), capi.ptr(aln), capi.ptr(maps), len(maps), capi.ptr(edits), len(edits), len(read_off) - 1, capi.ptr(rbuf),
            capi.ptr(qbuf) if qbuf is not None else None, capi.ptr(read_off), capi.ptr(nbuf) if nbuf is not None else None,
            capi.ptr(noff) if noff is not None else None, capi.ptr(out), cap, C.byref(used))
    assert rc == capi.GB_OK, rc
    return out[: used.value].tobytes()


def _build(recs):
    """recs: [(read_id, flags, score, [(oriented node, offset, [(op "MSID", length, base)...])...])] -> aln, maps, edits."""
    n = len(recs)
    cols = {k: np.zeros(n, dtype=capi.alignment_dt[k]) for k in capi.alignment_dt.names}
    mnode, moff, mne, words = [], [], [], []
    for x, (rid, flags, score, mp) in enumerate(recs):
        cols["read_id"][x] = rid; cols["flags"][x] = flags; cols["score"][x] = score
        cols["mapping_off"][x] = len(mnode); cols["edit_off"][x] = len(words); cols["n_mappings"][x] = len(mp)
        for node, off, eds in mp:
            mnode.append(node); moff.append(off); mne.append(len(eds))
            words.extend((ln << 4) | (b << 2) | "MSID".index(op) for op, ln, b in eds)
        cols["n_edits"][x] = len(words) - cols["edit_off"][x]
    cols["mapq"][:] = np.arange(n) % 61
    cols["mapq_uncapped"][:] = np.arange(n, dtype=np.float32) * 0.37
    cols["mapq_explored_cap"][:] = np.where(np.arange(n) % 3 == 0, np.inf, np.arange(n) * 1.5)
    aln = np.zeros(n, dtype=capi.alignment_dt)
    for k, v in cols.items():
        aln[k] = v
    maps = np.zeros(len(mnode) + 1, dtype=capi.mapping_dt)
    maps["node"][:-1] = mnode; maps["offset"][:-1] = moff; maps["n_edits"][:-1] = mne
    return aln, maps, np.array(words + [0], dtype=np.uint32)


def _hand_seqs():
    rng = np.random.default_rng(12)
    return ["".join("ACGT"[c] for c in rng.integers(0, 4, size=1000)) for _ in range(3)]


def _hand_graph():
    return capi.HostIndex(_hand_seqs(), [[2, 4, 6]], None, k=15, w=5)


def _reads(lengths, seed=5, n_frac=0.0):
    rng = np.random.default_rng(seed)
    reads = [bytes(synth.BASES[rng.integers(0, 4, size=ln)]) for ln in lengths]
    if n_frac:
        reads = [bytes(ord("N") if rng.random() < n_frac else c for c in r) for r in reads]
    rbuf, _, read_off = H.pack_reads(reads)
    qbuf = (np.arange(len(rbuf)) % 41).astype(np.uint8)
    return rbuf, qbuf, read_off


def _corner_batch():
    """Records at the formatting corners, on _hand_graph().  -> rbuf, qbuf, read_off, recs, aln, maps, edits"""
    rbuf, qbuf, read_off = _reads([40, 40, 20, 0, 25000, 30001, 40, 40], n_frac=0.05)
    recs = [
        (0, MAPPED, 31, [(2, 5, [("I", 4, 0), ("M", 30, 0), ("S", 1, 2), ("M", 5, 0)])]),                  # leading soft clip
        (1, MAPPED, -17, [(3, 990, [("M", 10, 0)]), (6, 0, [("I", 7, 0)]), (4, 0, [("D", 12, 0), ("M", 23, 0)])]),  # insertion-only mapping, <id
        (2, MAPPED, -2147483648, [(4, 0, [("I", 20, 0)])]),                                                  # all-insertion path: '*'
        (3, 0, 0, []),                                                                                       # empty read, unmapped
        (4, MAPPED | SEC, 5, [(2, 0, [("M", 1000, 0)])] * 25 + [(4, 0, [("D", 1, 0)])]),                      # dv 1/25001: exponent form
        (5, MAPPED | RESCUED, 77, [(2, 0, [("M", 1000, 0)])] * 30 + [(4, 0, [("M", 1, 0), ("D", 2, 0)])]),    # dv 2/30003
        (6, MAPPED | PAIRED, 0, [(2, 0, [("M", 39, 0), ("S", 1, 1)])]),
        (7, PAIRED | RESCUED, 9, []),
        (6, ABSENT, 0, []),
        (0, MAPPED, 1, [(2, 0, []), (2, 5, [("I", 4, 0), ("M", 36, 0)])]),                                   # a mapping without edits
    ]
    return (rbuf, qbuf, read_off, recs) + _build(recs)


def _dv_sweep():
    """One record per (matches, block): every pair with block <= 1100, and long deletions with block up to ~3e5, on
    _hand_graph().  -> rbuf, read_off, (aln, maps, edits), and Python's '%.6g' % (1.0 - m / b) for each record, which is
    correctly rounded like glibc."""
    B = 1100
    large_m = [10007, 24999, 99999, 123457, 299990]
    large_d = [1, 2, 3, 7, 19, 29, 30, 31, 97, 500, 999]
    rbuf, _, read_off = _reads(list(range(B + 1)) + large_m)
    recs, want = [], []
    for b in range(1, B + 1):
        for m in range(b + 1):
            ins = b - m
            m1, m2 = min(m, 1000), m - min(m, 1000)
            if m == 0:
                mp = [(2, 0, [("I", ins, 0)])]
            elif m2 == 0:
                mp = [(2, 0, [("M", m1, 0)] + ([("I", ins, 0)] if ins else []))]
            else:
                mp = [(2, 0, [("M", m1, 0)]), (4, 0, [("M", m2, 0)] + ([("I", ins, 0)] if ins else []))]
            recs.append((b, MAPPED, 0, mp)); want.append("%.6g" % (1.0 - m / b))
    for j, m in enumerate(large_m):
        for d in large_d:
            mp = [(2, 0, [("M", 1000, 0)])] * (m // 1000) + [(4, 0, [("M", m % 1000, 0)])] + [(6, 0, [("D", d, 0)])]
            recs.append((B + 1 + j, MAPPED, 0, mp)); want.append("%.6g" % (1.0 - m / (m + d)))
    assert sum("e-" in w for w in want) >= 10
    return rbuf, read_off, _build(recs), want


def test_dv_matches_printf_g6_over_a_dense_range():
    index = _hand_graph()
    rbuf, read_off, (aln, maps, edits), want = _dv_sweep()
    cap = int((edits >> 4)[(edits & 3) == "MSID".index("I")].sum()) + 1024 * len(aln)     # insertions are spelled out in cs
    got = _host("gaf", index.view, aln, maps, edits, rbuf, None, read_off, cap=cap).decode()
    dv = [line.rsplit("\tdv:f:", 1)[1] for line in got.splitlines()]
    bad = [(i, g, w) for i, (g, w) in enumerate(zip(dv, want)) if g != w]
    assert len(dv) == len(want) and not bad, bad[:10]


def test_hand_made_formatting_corners():
    """The corner records through gb_emit_gaf and gb_emit_gam: the GAF lines replay against the reads and the graph, and the
    GAM messages decode back to the records."""
    import test_gam as TG
    index, hand = _hand_graph(), types.SimpleNamespace(node_seqs=_hand_seqs())
    rbuf, qbuf, read_off, recs, aln, maps, edits = _corner_batch()
    reads = [rbuf[read_off[r]:read_off[r + 1]].tobytes().decode() for r in range(len(read_off) - 1)]
    present = [x for x, rec in enumerate(recs) if not rec[1] & ABSENT]
    gaf = _host("gaf", index.view, aln, maps, edits, rbuf, qbuf, read_off, cap=1 << 22).decode().splitlines()
    assert gaf[2].split("\t")[5] == "*" and "AS:i:-2147483648" in gaf[2]
    assert re.search(r"\tdv:f:[1-9](\.\d+)?e-05(\t|$)", gaf[4]) and re.search(r"\tdv:f:6\.6\d*e-05(\t|$)", gaf[5])
    assert len(gaf) == len(present) == len(recs) - 1
    for line, x in zip(gaf, present):
        rid, flags, score, mp = recs[x]
        read = reads[rid]
        f = line.split("\t")
        tags = {t[:2]: t[5:] for t in f[12:]}
        assert f[:4] == [f"read{rid}", str(len(read)), "0", str(len(read))]
        if flags & PAIRED:
            assert tags["fn" if rid % 2 == 0 else "fp"] == f"read{rid ^ 1}"
        if not flags & MAPPED or not mp:
            assert f[4:12] == ["*"] * 7 + ["255"] and tags["cs"] == "+" + read
            continue
        assert f[4] == "+" and int(f[11]) == aln[x]["mapq"] and int(tags["AS"]) == score
        steps, _ = _replay_gaf(f, tags, read, lambda v: _oriented_seq(hand, v), real=False)
        assert steps == [node for node, _, eds in mp if any(op != "I" for op, _, _ in eds)]
        assert tags["bq"] == "".join(chr(int(c) + 33) for c in qbuf[read_off[rid]:read_off[rid + 1]])

    msgs, tagged = TG.read_stream(_host("gam", index.view, aln, maps, edits, rbuf, qbuf, read_off, cap=1 << 22))
    assert len(msgs) == len(present) and tagged == 1
    for m, x in zip(msgs, present):
        rid, flags, score, mp = recs[x]
        read, a, fs = reads[rid], TG.decode_alignment(m), TG._fields(m)
        assert a["sequence"] == read and a["name"] == f"read{rid}"
        assert a["quality"] == (qbuf[read_off[rid]:read_off[rid + 1]].tobytes() if read else None)
        assert a["mapq"] == aln[x]["mapq"] and a["score"] == score % (1 << 64)          # a negative score is a 10-byte varint
        assert (TG._one(fs, 15) == 1) == bool(flags & SEC)
        if flags & PAIRED:
            assert a["fragment_next" if rid % 2 == 0 else "fragment_prev"] == f"read{rid ^ 1}"
        path = mp if flags & MAPPED else []
        assert [(p["node_id"], p["offset"], p["is_reverse"], p["rank"]) for p in a["path"]] == \
            [(node >> 1, off, bool(node & 1), rank) for rank, (node, off, _) in enumerate(path, 1)]
        q = matches = 0
        for p, (_, _, eds) in zip(a["path"], path):
            want = []
            for op, ln, _ in eds:
                want.append({"M": (ln, ln, ""), "S": (1, 1, read[q:q + 1]), "I": (0, ln, read[q:q + ln]), "D": (ln, 0, "")}[op])
                q += want[-1][1]; matches += ln if op == "M" else 0
            assert p["edits"] == want
        assert a["identity"] == (matches / len(read) if path and read else None)
        ann = {"mapq_uncapped": (2, float(aln[x]["mapq_uncapped"])), "mapq_explored_cap": (2, float(aln[x]["mapq_explored_cap"]))}
        if flags & RESCUED:
            ann["rescued"] = (4, 1)
        assert a["annotation"] == ann
