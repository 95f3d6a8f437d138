"""Surjection onto reference paths and SAM output: gb_ref_paths_build / gb_sam_header on the host, gb_surject_device and
gb_emit_sam_device on the GPU, against the host restatement in surject_oracle.py.  Haplotype 0 is the reference path:
reads sampled from it take the direct route; reads from the other haplotypes leave it at variant sites."""
from pathlib import Path

import numpy as np
import pytest

import helpers as H
import surject_oracle as O
import vcf_graph
from vg_b200 import capi, synth

SAM_DIR = Path(__file__).parent / "golden" / "sam"


def _node_len(index):
    return index.array("nodes")["len"].astype(np.int64)


def _linear_paths_index(names, length=1001, seed=0):
    """One linear path of `length` bases per name, nodes of 32 bp, as one graph."""
    rng = np.random.default_rng(seed)
    seqs, paths = [], []
    for _ in names:
        s = "".join("ACGT"[i] for i in rng.integers(0, 4, size=length))
        ids = []
        for i in range(0, length, 32):
            seqs.append(s[i:i + 32]); ids.append(2 * len(seqs))
        paths.append(ids)
    return capi.HostIndex(seqs, paths), paths


# ---- host: reference paths and the header ----------------------------------------------------------------------------

@pytest.mark.parametrize("order", [("x", "y"), ("y", "x")])
def test_header_matches_the_sequence_dictionaries(order):
    """50_vg_giraffe.t:226-233: the @HD / @SQ lines follow the caller's path order (the dictionaries carry no M5)."""
    index, paths = _linear_paths_index(["x", "y"])
    by_name = dict(zip(["x", "y"], paths))
    rp = capi.RefPaths(index.view, [(n, by_name[n]) for n in order])
    want = (SAM_DIR / ("".join(order) + ".dict")).read_text()
    assert rp.sam_header() == want
    rp.close()


def test_builder_refusals():
    index, paths = _linear_paths_index(["x", "y"])
    n_ids = len(index.array("nodes")) // 2
    cases = {
        "node past the graph": [("x", paths[0] + [2 * n_ids])],
        "node occurs twice in one path": [("x", paths[0] + [paths[0][3]])],
        "node occurs twice across paths": [("x", paths[0]), ("y", paths[1] + [paths[0][0] | 1])],
        "empty path": [("x", [])],
        "empty name": [("", paths[0])],
        "name with a tab": [("x\ty", paths[0])],
    }
    for what, spec in cases.items():
        with pytest.raises(capi.GbError) as e:
            capi.RefPaths(index.view, spec)
        assert e.value.code == capi.GB_ERR_FORMAT, what
    # an id without sequence (ids need not be dense)
    seqs = ["ACGTACGTAC", "", "GGGTTTCCCA"]
    sparse = capi.HostIndex(seqs, [[2, 6]])
    with pytest.raises(capi.GbError) as e:
        capi.RefPaths(sparse.view, [("x", [2, 4, 6])])
    assert e.value.code == capi.GB_ERR_FORMAT
    capi.RefPaths(sparse.view, [("x", [2, 6])]).close()


# ---- host: the oracle on the reference's own pins ----------------------------------------------------------------------

def _small_x():
    g, _ = vcf_graph.small_x()
    ref = vcf_graph.read_fasta(vcf_graph.GOLD / "x.fa.gz")
    assert bytes(g.hap_seq[0]).decode() == ref                 # haplotype 0 is the reference walk: x.fa
    return g, g.build_index()


def _oracle_sam(g, index, res, names, reads, quals, tlen_max=0):
    recs = O.surject(res[0], res[1], res[2], [("x", g.paths[0])], _node_len(index), tlen_max=tlen_max)
    return recs, None if reads is None else O.sam_text(recs, names, reads, quals, ["x"])


def _perfect_reads(g, n, L, seed):
    rng = np.random.default_rng(seed)
    ref = g.hap_seq[0]
    starts = rng.integers(0, len(ref) - L, size=n)
    rev = rng.random(n) < 0.5
    reads = [synth.revcomp_bytes(ref[s:s + L]) if r else ref[s:s + L].copy() for s, r in zip(starts, rev)]
    return np.stack(reads), starts, rev


def test_perfect_reads_and_strand_invariance():
    """15_vg_surject.t:23-34 and :95: reads sampled from the reference give <L>M, AS = L + 2 x bonus and the sampled POS;
    a read and its reverse complement give the same columns 1 and 3-11."""
    g, index = _small_x()
    L = 100
    reads, starts, rev = _perfect_reads(g, 60, L, 1)
    res = H.oracle_map(index, reads)
    recs, _ = _oracle_sam(g, index, res, None, None, None)
    for r, s, rv in zip(recs, starts, rev):
        assert r["route"] == 0 and r["cigar"] == [(L, "M")] and r["score"] == L + 10 and r["pos"] == s and r["rev"] == bool(rv)
    both = np.concatenate([reads, synth.revcomp_bytes(reads)])
    res = H.oracle_map(index, both)
    strs = [bytes(r).decode() for r in both]
    _, text = _oracle_sam(g, index, res, [f"r{i % len(reads)}" for i in range(len(both))], strs, None)
    lines = text.splitlines()
    for i in range(len(reads)):
        a, b = lines[i].split("\t"), lines[i + len(reads)].split("\t")
        assert a[0] == b[0] and a[2:11] == b[2:11] and int(a[1]) ^ int(b[1]) == 16


def _variant_reads(g, index, n=300, seed=4):
    rs = synth.simulate_reads(g, n, length=150, sub_rate=0.01, ins_rate=0.003, del_rate=0.003, seed=seed)
    return rs, H.oracle_map(index, rs.reads, rs.quals, threads=8)


def test_oracle_cigars_replay_against_the_reference():
    """Every direct-route CIGAR, replayed against the reference path and the read, spells the read and rescores to AS."""
    g = synth.make_variant_graph(length=20000, n_snp=60, n_ins=8, n_del=8, n_haps=4, seed=3)
    index = g.build_index()
    rs, res = _variant_reads(g, index)
    recs = O.surject(res[0], res[1], res[2], [("ref", g.paths[0])], _node_len(index))
    ref = bytes(g.hap_seq[0]).decode()
    routes = [r["route"] for r in recs]
    assert routes.count(0) > len(recs) // 3 and routes.count(2) > 10
    for r in recs:
        if r["route"] != 0:
            continue
        read = bytes(rs.reads[r["read_id"]]).decode()
        if r["rev"]:
            read = read[::-1].translate(str.maketrans("ACGT", "TGCA"))
        q, t, score = 0, r["pos"], 0
        for i, (n, op) in enumerate(r["cigar"]):
            if op == "M":
                score += sum(1 if read[q + k] == ref[t + k] else -4 for k in range(n)); q += n; t += n
            elif op == "I":
                score -= 6 + (n - 1); q += n
            elif op == "D":
                score -= 6 + (n - 1); t += n
            else:
                q += n
        assert q == len(read)
        score += (0 if r["cigar"][0][1] == "S" else 5) + (0 if r["cigar"][-1][1] == "S" else 5)
        assert score == r["score"]


# ---- GPU -------------------------------------------------------------------------------------------------------------

def _t(a, dtype=None):
    import torch
    a = np.ascontiguousarray(a if dtype is None else a.astype(dtype))
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy() if dtype is None else a.copy()).cuda()


def _check_device(dev, index, g, res, rbuf, qbuf, read_off, reads, quals, names, tlen_max=0, paths=None):
    """Every record field and CIGAR op of gb_surject_device, the deferred count and the SAM text equal the oracle's;
    returns (the oracle's records, the SAM text)."""
    paths = paths or [("ref", g.paths[0])]
    want = O.surject(res[0], res[1], res[2], paths, _node_len(index), tlen_max=tlen_max)
    rec, cigar, n_realign = dev.surject_device(_t(res[0]), _t(res[1]), _t(res[2], np.uint32), _t(read_off, np.int64), tlen_max)
    got = O.decode_device(rec.cpu().numpy().tobytes(), cigar.cpu().numpy().view(np.uint32))
    assert len(got) == len(want) and n_realign == sum(r["route"] == 2 for r in want)
    for i, (a, b) in enumerate(zip(got, want)):
        b = {k: v for k, v in b.items() if k != "rev"}
        assert a == b, f"record {i}: device {a} oracle {b}"
    nm = None
    if names is not None:
        nb = [n.encode() for n in names]
        off = np.zeros(len(nb) + 1, dtype=np.int64); off[1:] = np.cumsum([len(n) for n in nb])
        nm = (_t(np.frombuffer(b"".join(nb) + b"\0", np.uint8)), _t(off, np.int64))
    text = dev.emit_sam_device(rec, cigar, _t(rbuf), _t(read_off, np.int64), None if qbuf is None else _t(qbuf),
                               *(nm or (None, None))).cpu().numpy().tobytes().decode()
    assert text == O.sam_text(want, names, reads, quals, [n for n, _ in paths])
    return want, text


def _graph_cases():
    yield "variant", synth.make_variant_graph(length=60000, n_snp=100, n_ins=12, n_del=12, n_haps=4, seed=8)
    yield "small_x", vcf_graph.small_x()[0]
    yield "kgp_100k", vcf_graph.kgp_100k()[0]
    yield "nested", synth.make_nested_graph()


@pytest.mark.gpu
@pytest.mark.parametrize("paired", [False, True])
def test_device_matches_oracle_on_oracle_records(paired):
    for gname, g in _graph_cases():
        index = g.build_index()
        if paired:
            rs = synth.simulate_pairs(g, 150, sub_rate=0.02, seed=5)
            res = H.oracle_map_paired(index, rs.reads, rs.quals, H.paired_params(), threads=8)
        else:
            rs = synth.simulate_reads(g, 300, length=150, sub_rate=0.02, ins_rate=0.004, del_rate=0.004, seed=6)
            res = H.oracle_map(index, rs.reads, rs.quals, threads=8)
        dev = capi.Device(index, 0)
        rp = capi.RefPaths(index.view, [("ref", g.paths[0])])
        dev.set_ref_paths(rp)
        rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
        reads = [bytes(r).decode() for r in rs.reads]
        names = [f"q{i // 2}/{i % 2 + 1}" if paired else f"q{i}" for i in range(rs.n)]
        want, _ = _check_device(dev, index, g, res, rbuf, qbuf, read_off, reads, list(rs.quals), names, tlen_max=700 if paired else 0)
        _check_device(dev, index, g, res, rbuf, None, read_off, reads, None, None)
        routes = [r["route"] for r in want]
        assert routes.count(0) > 0, gname
        dev.close(); rp.close()


@pytest.mark.gpu
@pytest.mark.parametrize("paired", [False, True])
def test_device_matches_oracle_with_multimaps(paired):
    from test_multimap import repeat_graph
    g = repeat_graph(); index = g.build_index()
    p = H.paired_params() if paired else H.default_map_params()
    p.max_multimaps = 3
    if paired:
        p.max_rescue_attempts = 15
        rs = synth.simulate_pairs(g, 150, sub_rate=0.01, seed=37)
        res = H.oracle_map_paired(index, rs.reads, rs.quals, p, threads=8)
    else:
        rs = synth.simulate_reads(g, 300, length=150, sub_rate=0.01, seed=36)
        res = H.oracle_map(index, rs.reads, rs.quals, p, threads=8)
    dev = capi.Device(index, 0)
    rp = capi.RefPaths(index.view, [("ref", g.paths[0])])
    dev.set_ref_paths(rp)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    want, _ = _check_device(dev, index, g, res, rbuf, qbuf, read_off, [bytes(r).decode() for r in rs.reads], list(rs.quals), None)
    assert sum(1 for r in want if r["flag"] & 0x100 and r["route"] == 0) > 5
    dev.close(); rp.close()


@pytest.mark.gpu
@pytest.mark.parametrize("paired", [False, True])
def test_device_on_records_from_map_batch_device(paired):
    g, index = _small_x()
    dev = capi.Device(index, 0)
    rp = capi.RefPaths(index.view, [("ref", g.paths[0])])
    dev.set_ref_paths(rp)
    if paired:
        rs = synth.simulate_pairs(g, 200, sub_rate=0.01, seed=9)
    else:
        rs = synth.simulate_reads(g, 400, length=150, sub_rate=0.01, ins_rate=0.003, del_rate=0.003, seed=9)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    res = dev.map_arrays(rbuf, qbuf, read_off, H.paired_params() if paired else None, paired=paired)
    want, _ = _check_device(dev, index, g, res, rbuf, qbuf, read_off, [bytes(r).decode() for r in rs.reads], list(rs.quals),
                            [f"p{i // 2}_{i % 2 + 1}" for i in range(rs.n)], tlen_max=700 if paired else 0)
    assert sum(r["route"] == 0 for r in want) > rs.n // 10          # small_x has a variant every ~20 bp
    dev.close(); rp.close()


@pytest.mark.gpu
def test_refusals_and_capacity():
    import torch
    from vg_b200.capi import load_library
    import ctypes as C
    g, index = _small_x()
    dev = capi.Device(index, 0)
    lib = load_library()
    reads, _, _ = _perfect_reads(g, 8, 100, 2)
    res = H.oracle_map(index, reads)
    rbuf, _, read_off = H.pack_reads(reads)
    aln, maps, edits, ro = _t(res[0]), _t(res[1]), _t(res[2], np.uint32), _t(read_off, np.int64)
    out = torch.empty(8 * 40, dtype=torch.uint8, device="cuda")
    cig = torch.empty(4096, dtype=torch.int32, device="cuda")
    used = C.c_uint64()
    vp = lambda t: C.c_void_p(t.data_ptr())
    call = lambda a=aln, cap=4096, n=8: lib.gb_surject_device(dev.handle, n, vp(a), vp(maps), maps.numel() // 8, vp(edits), edits.numel(),
                                                              8, vp(ro), 0, vp(out), vp(cig), cap, C.byref(used), None)
    assert call() == capi.GB_ERR_ARG                                   # no reference paths yet
    rp = capi.RefPaths(index.view, [("x", g.paths[0])])
    dev.set_ref_paths(rp)
    assert call(cap=0) == capi.GB_ERR_CAPACITY and used.value == 8      # one M op per perfect read
    assert call(cap=used.value) == capi.GB_OK
    bad = res[0].copy(); bad[3]["read_id"] = 99
    assert call(a=_t(bad)) == capi.GB_ERR_ARG
    bad = res[0].copy(); bad[2]["flags"] |= 4                          # paired, but its neighbour is not its mate
    assert call(a=_t(bad)) == capi.GB_ERR_ARG
    assert call(a=aln, n=0xffffffff) == capi.GB_ERR_ARG
    # the SAM emitter: capacity, then a record pointing past the cigar pool
    assert call() == capi.GB_OK
    torch.cuda.synchronize()
    so = torch.empty(1, dtype=torch.uint8, device="cuda")
    rc = lib.gb_emit_sam_device(dev.handle, 8, vp(out), vp(cig), 8, 8, vp(_t(rbuf)), None, vp(ro), None, None, vp(so), 1, C.byref(used))
    assert rc == capi.GB_ERR_CAPACITY and used.value > 8 * 100
    rc = lib.gb_emit_sam_device(dev.handle, 8, vp(out), vp(cig), 4, 8, vp(_t(rbuf)), None, vp(ro), None, None, vp(so), 1, C.byref(used))
    assert rc == capi.GB_ERR_ARG
    dev.close(); rp.close()


def _pairs_on_variant_graph():
    g = synth.make_variant_graph(length=60000, n_snp=100, n_ins=12, n_del=12, n_haps=4, seed=8)
    index = g.build_index()
    rs = synth.simulate_pairs(g, 200, sub_rate=0.01, seed=21)
    res = H.oracle_map_paired(index, rs.reads, rs.quals, H.paired_params(), threads=8)
    dev = capi.Device(index, 0)
    rp = capi.RefPaths(index.view, [("ref", g.paths[0])])
    dev.set_ref_paths(rp)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    return g, index, rs, res, dev, rp, rbuf, qbuf, read_off, [bytes(r).decode() for r in rs.reads]


@pytest.mark.gpu
def test_pairs_proper_at_tlen_max_deferred_together_and_unmapped_mate_location():
    g, index, rs, res, dev, rp, rbuf, qbuf, read_off, reads = _pairs_on_variant_graph()
    want, _ = _check_device(dev, index, g, res, rbuf, None, read_off, reads, None, None)
    # a pair with one mate off the reference path is deferred whole: both records, no SAM line for either
    split = [x for x in range(0, len(want), 2) if {want[x]["route"], want[x + 1]["route"]} == {2}
             and {O.surject_one(int(res[0][y]["flags"]), H.decode_alignment(res[0][y], res[1], res[2]),
                                O.ref_index([("ref", g.paths[0])], _node_len(index))[0], _node_len(index), (1, 4, 6, 1, 5))["route"]
                  for y in (x, x + 1)} == {0, 2}]
    assert split
    # proper pair exactly at tlen_max, not at tlen_max - 1 (|TLEN| <= tlen_max, alignment.cpp:732)
    x = next(i for i, r in enumerate(want) if r["flag"] & 0x2)
    t = abs(want[x]["tlen"])
    at, _ = _check_device(dev, index, g, res, rbuf, None, read_off, reads, None, None, tlen_max=t)
    below, _ = _check_device(dev, index, g, res, rbuf, None, read_off, reads, None, None, tlen_max=t - 1)
    assert at[x]["flag"] & 0x2 and not below[x]["flag"] & 0x2 and at[x ^ 1]["flag"] & 0x2 and not below[x ^ 1]["flag"] & 0x2
    # an unmapped mate takes its mate's RNAME and POS (SAMv1 2.4.1); the mapped mate gets 0x8 and RNEXT '*'
    aln = res[0].copy()
    mx = x | 1
    aln["flags"][mx] &= ~np.uint8(1); aln["n_mappings"][mx] = 0
    want2, text = _check_device(dev, index, g, (aln, res[1], res[2]), rbuf, None, read_off, reads, None, None)
    lines = {int(l.split("\t")[0][4:]): l.split("\t") for l in text.splitlines()}
    um, mm = lines[int(aln[mx]["read_id"])], lines[int(aln[mx ^ 1]["read_id"])]
    assert int(um[1]) & 0x4 and um[2] == "ref" and int(um[3]) == want2[mx ^ 1]["pos"] + 1 and um[5] == "*"
    assert int(mm[1]) & 0x8 and mm[6] == "*" and mm[7] == "0"
    dev.close(); rp.close()


@pytest.mark.gpu
def test_two_reference_paths_cut_from_one_walk():
    """Haplotype 0 cut in two paths: reads inside either get its name and a position counted from its start; a read across
    the cut lies on two paths, which is the realigning route's choice (choose_primary_strand), so it is deferred."""
    g = synth.make_variant_graph(length=60000, n_snp=100, n_ins=12, n_del=12, n_haps=4, seed=8)
    index = g.build_index()
    cut = len(g.paths[0]) // 2
    paths = [("a", g.paths[0][:cut]), ("b", g.paths[0][cut:])]
    ref = g.hap_seq[0]
    a_len = int(sum(_node_len(index)[v] for v in paths[0][1]))
    rng = np.random.default_rng(5)
    starts = np.concatenate([rng.integers(0, len(ref) - 150, size=100), a_len - rng.integers(10, 140, size=20)])
    reads = np.stack([ref[s:s + 150].copy() for s in starts])
    res = H.oracle_map(index, reads)
    dev = capi.Device(index, 0)
    rp = capi.RefPaths(index.view, paths)
    dev.set_ref_paths(rp)
    rbuf, _, read_off = H.pack_reads(reads)
    want, text = _check_device(dev, index, g, res, rbuf, None, read_off, [bytes(r).decode() for r in reads], None, None, paths=paths)
    for r, s in zip(want, starts):
        if s + 150 <= a_len:
            assert (r["route"], r["ref"], r["pos"]) == (0, 0, s)
        elif s >= a_len:
            assert (r["route"], r["ref"], r["pos"]) == (0, 1, s - a_len)
    assert all(want[i]["route"] == 2 for i in range(100, 120))
    assert rp.sam_header() == f"@HD\tVN:1.5\tSO:unknown\n@SQ\tSN:a\tLN:{a_len}\n@SQ\tSN:b\tLN:{len(ref) - a_len}\n"
    dev.close(); rp.close()
