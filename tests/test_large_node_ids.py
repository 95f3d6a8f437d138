"""Node ids past 2^22: the mapping entry points on graphs whose ids reach 2^22 - 1, 2^22, 2^22 + 1 and 2^24.

The graphs are the config-2 variant family and the nested family with every id shifted up by prepending unused ids (empty
sequences), so the node arrays grow to the shifted size while the graph itself stays small.  Each mapping result must equal
the unshifted run record for record once the shift is taken off the node handles, and the oracle's on the shifted index."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
from vg_b200 import capi, synth

TOPS = [(1 << 22) - 1, 1 << 22, (1 << 22) + 1, (1 << 24) + 3]


def _graph(family):
    if family == "variants":
        return synth.make_variant_graph(length=60000, n_snp=100, n_ins=12, n_del=12, n_haps=8, seed=21), (29, 11)
    return synth.make_nested_graph(n_items=120, n_haps=10, seed=5), (11, 5)


def _shifted(g, shift, k, w):
    """The index of g with every node id raised by `shift` (ids 1 .. shift carry no sequence)."""
    seqs = [""] * shift + list(g.node_seqs)
    paths = [[v + 2 * shift for v in p] for p in g.paths]
    dist = None
    if g.dist is not None:
        dist = np.zeros(len(seqs) + 1, dtype=capi.dist_dt); dist["allele"] = 0xFFFF
        dist[shift + 1:] = np.asarray(g.dist)[1:]
    return capi.HostIndex(seqs, paths, dist, k=k, w=w)


def _unshift(res, used, shift):
    """(aln, maps[:used], edits[:used]) with the shift taken off every mapped node handle."""
    aln, maps, edits = res[0], res[1][: used[0]].copy(), res[2][: used[1]]
    maps["node"] -= np.uint32(2 * shift)
    return aln, maps, edits


def _same_records(a, b):
    assert a[0].tobytes() == b[0].tobytes(), "alignment records differ"
    assert a[1].tobytes() == b[1].tobytes(), "mappings differ"
    assert a[2].tobytes() == b[2].tobytes(), "edits differ"


class Family:
    """One graph family: the unshifted index and the shifted ones, built once per top id."""

    def __init__(self, name):
        self.name = name
        self.g, (self.k, self.w) = _graph(name)
        self.base = capi.HostIndex(self.g.node_seqs, self.g.paths, self.g.dist, k=self.k, w=self.w)
        self._shifted = {}

    def shift(self, top):
        return top - len(self.g.node_seqs)

    def index(self, top):
        if top not in self._shifted:
            self._shifted[top] = _shifted(self.g, self.shift(top), self.k, self.w)
        return self._shifted[top]

    def close(self):
        for ix in [self.base, *self._shifted.values()]:
            ix.close()


@pytest.fixture(scope="module", params=["variants", "nested"])
def family(request):
    f = Family(request.param)
    yield f
    f.close()


def _cases():
    return [pytest.param(top, id=f"top{top}") for top in TOPS]


def test_shifted_builds_keep_arrays_past_2_22(family):
    """From paths and from the flat GBWT, the shifted index is the unshifted one moved up: same sequences, records, table."""
    g, top = family.g, (1 << 22) + 1
    shift, ix, base = family.shift(top), family.index(top), family.base
    assert int(ix.view.n_nodes) == int(base.view.n_nodes) + 2 * shift
    hits, bhits = ix.array("hits"), base.array("hits")
    assert ((hits["pos"] >> np.uint64(10)) == (bhits["pos"] >> np.uint64(10)) + np.uint64(2 * shift)).all()
    assert ix.array("table").tobytes() == base.array("table").tobytes()
    seqs = [""] * shift + list(g.node_seqs)
    again = capi.HostIndex.from_gbwt(seqs, len(g.paths), ix.array("gbwt"), ix.array("nodes")["rec_off"],
                                     None if g.dist is None else ix.array("dist"), k=family.k, w=family.w)
    for name in ("nodes", "seq", "gbwt", "dist", "slots", "site_dist", "table", "hits"):
        assert again.array(name).tobytes() == ix.array(name).tobytes(), name
    again.close()


def test_oracle_maps_shifted_graph_like_the_unshifted_one(family):
    top = (1 << 22) + 1
    shift, ix = family.shift(top), family.index(top)
    rs = synth.simulate_reads(family.g, 200, length=150, sub_rate=0.01, seed=8)
    a = H.oracle_map(family.base, rs.reads, rs.quals, threads=4)
    b = H.oracle_map(ix, rs.reads, rs.quals, threads=4)
    for i in range(rs.n):
        pa, pb = H.decode_alignment(a[0][i], a[1], a[2]), H.decode_alignment(b[0][i], b[1], b[2])
        assert pa[:2] == pb[:2] and [(n + 2 * shift, o, e) for n, o, e in pa[2]] == pb[2]


# ---- GPU -----------------------------------------------------------------------------------------------------------

def _map(ix, reads, quals, p, paired=False):
    dev = capi.Device(ix)
    try:
        res = H.gpu_map(dev, reads, quals, p, paired=paired)
        return res, dev.last_used
    finally:
        dev.close()


def _check_mode(family, top, reads, quals, p, paired, oracle):
    shift, ix = family.shift(top), family.index(top)
    want, wused = _map(family.base, reads, quals, p, paired)
    got, gused = _map(ix, reads, quals, p, paired)
    n = len(reads); K = max(1, int(p.max_multimaps))
    assert (got[3] == 0).all()
    _same_records(_unshift(got, gused, shift), _unshift(want, wused, 0))
    ref = oracle(ix, reads, quals, p)
    bad = H.compare_alignments(got, ref, n, k=K)
    assert not bad, f"{len(bad)} of {n * K} records differ from the oracle; first {bad[0]}"
    return ref


@pytest.mark.gpu
@pytest.mark.parametrize("top", _cases())
def test_single_end_past_2_22(family, top):
    rs = synth.simulate_reads(family.g, 400, length=150, sub_rate=0.01, ins_rate=0.001, del_rate=0.001, seed=3)
    _check_mode(family, top, rs.reads, rs.quals, H.default_map_params(), False,
                lambda ix, r, q, p: H.oracle_map(ix, r, q, p, threads=8))


@pytest.mark.gpu
@pytest.mark.parametrize("top", _cases())
def test_multimaps_past_2_22(family, top):
    rs = synth.simulate_reads(family.g, 300, length=150, sub_rate=0.01, seed=5)
    p = H.default_map_params(); p.max_multimaps = 3
    _check_mode(family, top, rs.reads, rs.quals, p, False, lambda ix, r, q, pp: H.oracle_map(ix, r, q, pp, threads=8))


def _pairs(g, n_pairs, seed, garble=0, rate=0.12):
    rs = synth.simulate_pairs(g, n_pairs, frag_mean=380, frag_sd=45, sub_rate=0.004, seed=seed)
    rng = np.random.default_rng(seed)
    for i in rng.choice(n_pairs, size=garble, replace=False):
        # mate 2 too damaged to seed well: found by rescue from mate 1
        m = rng.random(rs.length) < rate
        rs.reads[2 * i + 1, m] = synth.BASES[rng.integers(0, 4, size=int(m.sum()))]
    return rs


@pytest.mark.gpu
@pytest.mark.parametrize("rescue", [False, True], ids=["no-rescue", "rescue"])
@pytest.mark.parametrize("top", _cases())
def test_paired_past_2_22(family, top, rescue):
    # k = 11 on the nested graph seeds through 12 % substitutions: its mates need more damage to need rescue
    rs = _pairs(family.g, 200, seed=7, garble=40 if rescue else 0, rate=0.12 if family.name == "variants" else 0.3)
    p = H.paired_params(380.0, 45.0)
    if rescue:
        p.max_rescue_attempts = H.default_map_params().max_rescue_attempts
    ref = _check_mode(family, top, rs.reads, rs.quals, p, True, lambda ix, r, q, pp: H.oracle_map_paired(ix, r, q, pp, threads=8))
    if rescue:
        assert ref[4]["rescues"] > 0, "no mate was rescued: the test does not reach rescue"


@pytest.mark.gpu
@pytest.mark.parametrize("top", _cases())
def test_seed_stage_past_2_22(family, top):
    shift, ix = family.shift(top), family.index(top)
    rs = _pairs(family.g, 150, seed=9)
    p = H.paired_params(380.0, 45.0)
    rbuf, qbuf, off = H.pack_reads(rs.reads, rs.quals)
    dev = capi.Device(ix)
    got = dev.seed_stage(rbuf, qbuf, off, p, paired=True)
    dev.close()
    want = H.oracle_seed_stage(ix, rs.reads, rs.quals, p, paired=True)
    bad = H.compare_stage_dumps(got, want, rs.n)
    assert not bad, bad[:3]
    # against the unshifted run: seeds and item seeds move up by the shift, nothing else changes
    dev = capi.Device(family.base)
    un = dev.seed_stage(rbuf, qbuf, off, p, paired=True)
    dev.close()
    for name, x, y in zip(("reads", "minimizers", "seeds", "clusters", "items", "item_seeds"), got, un):
        if name in ("seeds", "item_seeds"):                       # the buffers' unused tails stay zero
            x = x.copy(); x["node"] = np.where(x["node"] != 0, x["node"] - np.uint32(2 * shift), 0).astype(np.uint32)
        assert x.tobytes() == y.tobytes(), name


def _device_job(dev, f, p, rbuf, qbuf, off, max_len):
    import torch
    n = len(off) - 1
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t_r, t_q, t_o = t(rbuf), t(qbuf), t(off.astype(np.int64))
    t_aln = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
    t_maps = torch.zeros(n * p.mapping_cap_per_read * 8, dtype=torch.uint8, device="cuda")
    t_edits = torch.zeros(n * p.edit_cap_per_read * 4, dtype=torch.uint8, device="cuda")
    t_status = torch.zeros(n, dtype=torch.uint8, device="cuda")
    t_route = torch.zeros(n // 2, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rc, nm, ne = dev.map_paired_job_device(f, n, t_r.data_ptr(), t_q.data_ptr(), t_o.data_ptr(), max_len, t_aln.data_ptr(),
                                           t_maps.data_ptr(), n * p.mapping_cap_per_read, t_edits.data_ptr(), n * p.edit_cap_per_read,
                                           t_status.data_ptr(), t_route.data_ptr(), params=p)
    assert rc == capi.GB_OK, capi.load_library().gb_last_error()
    return (t_aln.cpu().numpy().view(capi.alignment_dt), t_maps.cpu().numpy().view(capi.mapping_dt), t_edits.cpu().numpy().view(np.uint32),
            t_status.cpu().numpy(), t_route.cpu().numpy()), (nm, ne)


@pytest.mark.gpu
@pytest.mark.parametrize("top", _cases())
def test_paired_job_device_past_2_22(family, top):
    shift, ix = family.shift(top), family.index(top)
    rs = _pairs(family.g, 600, seed=11)
    p = H.default_map_params(); p.fragment_mean = 0.0; p.fragment_stdev = 0.0
    rbuf, qbuf, off = H.pack_reads(rs.reads, rs.quals)
    runs = []
    for index in (family.base, ix):
        dev = capi.Device(index)
        f = capi.FragmentDistribution(1000, 1000, 0.95)
        runs.append(_device_job(dev, f, p, rbuf, qbuf, off, rs.length))
        f.close(); dev.close()
    (want, wused), (got, gused) = runs
    _same_records(_unshift(got, gused, shift), _unshift(want, wused, 0))
    assert (got[4] == want[4]).all(), "pair routes differ"
    oracle = H.oracle_map_paired_job(ix, rs.reads, rs.quals, p, threads=8)
    bad = H.compare_alignments(got, oracle, rs.n)
    assert not bad, f"{len(bad)} records differ from the oracle; first {bad[0]}"


@pytest.mark.gpu
def test_emitters_print_ids_past_2_22(family):
    import torch
    top = (1 << 24) + 3
    shift, ix = family.shift(top), family.index(top)
    rs = synth.simulate_reads(family.g, 200, length=150, sub_rate=0.01, seed=13)
    dev = capi.Device(ix)
    aln, maps, edits, status = H.gpu_map(dev, rs.reads, rs.quals)
    nm, ne = dev.last_used
    maps, edits = maps[:nm], edits[:ne]
    rbuf, qbuf, off = H.pack_reads(rs.reads, rs.quals)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
    for kind in ("gaf", "gam"):
        host = capi.emit_text(kind, ix.view, aln, maps, edits, rbuf, qbuf, off)
        got = capi.emit_device_text(dev, kind, t(aln), t(maps), t(edits), t(rbuf), torch.from_numpy(off.astype(np.int64)).cuda(), quals=t(qbuf))
        assert got == host, kind
    dev.close()
    gaf = capi.emit_text("gaf", ix.view, aln, maps, edits, rbuf, qbuf, off)
    paths = [line.split("\t")[5] for line in gaf.splitlines()]
    ids = [int(x) for path in paths if path != "*" for x in path.replace("<", " ").replace(">", " ").split()]
    assert ids and min(ids) > shift and max(ids) <= top


@pytest.mark.gpu
def test_chain_coordinates_past_int32_are_refused():
    """A hand-made payload whose coordinates leave int32 is refused before any launch; the same graph one step lower maps."""
    g = synth.make_variant_graph(length=6000, n_snp=10, n_ins=2, n_del=2, n_haps=4, seed=3)
    rs = synth.simulate_reads(g, 20, length=150, sub_rate=0.0, seed=2)
    lens = np.array([0] + [len(s) for s in g.node_seqs], dtype=np.int64)
    top = int((np.asarray(g.dist)["x_in"].astype(np.int64) + lens).max())
    for lift, ok in (((1 << 31) - 1 - top, True), ((1 << 31) - top, False)):
        dist = np.asarray(g.dist).copy()
        for f in ("x_in", "x_out"):
            dist[f] = (dist[f].astype(np.int64) + lift).astype(np.uint32).view(np.int32)
        ix = capi.HostIndex(g.node_seqs, g.paths, dist)
        dev = capi.Device(ix)
        if ok:
            aln = H.gpu_map(dev, rs.reads, rs.quals)[0]
            assert (aln["flags"] & 1).all()
        else:
            with pytest.raises(capi.GbError) as e:
                H.gpu_map(dev, rs.reads, rs.quals)
            assert e.value.code == capi.GB_ERR_CAPACITY and dev.launches() == 0
        dev.close(); ix.close()


# ---- more than 2^22 real nodes ----------------------------------------------------------------------------------------

def _chopped(g, max_node=2):
    """g with every node cut into pieces of at most max_node bp: (node_seqs, paths, piece) where piece[new id] =
    (old id, start of the piece in the old node's forward sequence)."""
    seqs, piece, new_ids = [], [(0, 0)], [None]
    for old, s in enumerate(g.node_seqs, start=1):
        ids = []
        for at in range(0, len(s), max_node):
            seqs.append(s[at:at + max_node]); piece.append((old, at)); ids.append(len(seqs))
        new_ids.append(ids)
    paths = [[2 * n for v in p for n in new_ids[v >> 1]] for p in g.paths]
    return seqs, paths, piece


def _canonical(path, piece, old_len, chopped):
    """An alignment path as the graph positions it visits, per reference base, and its edit operations per base: the same
    for a path on the chopped graph and on the original one whenever they differ only at node boundaries."""
    pos, ops = [], []
    for node, off, edits in path:
        nid, rev = node >> 1, node & 1
        if chopped:
            old, at = piece[nid]
            plen = len_of_piece(piece, nid, old_len)
            start = (old_len[old] - at - plen if rev else at) + off
        else:
            old, start = nid, off
        p = start
        for op, n, base in edits:
            for _ in range(n):
                ops.append(op + base)
                if op != "I":
                    pos.append((2 * old + rev, p)); p += 1
    return pos, ops


def len_of_piece(piece, nid, old_len):
    old, at = piece[nid]
    nxt = piece[nid + 1] if nid + 1 < len(piece) else (None, None)
    return (nxt[1] if nxt[0] == old else old_len[old]) - at


@pytest.fixture(scope="module")
def chopped():
    """A config-2-density variant graph of 8.6 Mbp with nodes of at most 2 bp: more than 2^22 real node ids."""
    g = synth.make_variant_graph(length=8_600_000, n_snp=6800, n_ins=850, n_del=850, n_haps=4, seed=2)
    seqs, paths, piece = _chopped(g)
    assert len(seqs) > (1 << 22)
    whole = capi.HostIndex(g.node_seqs, g.paths, None)
    ix = capi.HostIndex(seqs, paths, None)
    old_len = [0] + [len(s) for s in g.node_seqs]
    yield g, whole, ix, piece, old_len
    ix.close(); whole.close()


def _chopped_params(p=None):
    p = p or H.default_map_params()
    p.mapping_cap_per_read = 256; p.edit_cap_per_read = 512          # 150 bp over 2 bp nodes: ~76 mappings per read
    return p


def _assert_same_up_to_boundaries(a, b, n, piece, old_len):
    for i in range(n):
        sa, qa, pa = H.decode_alignment(a[0][i], a[1], a[2])
        sb, qb, pb = H.decode_alignment(b[0][i], b[1], b[2])
        assert sa == sb and abs(qa - qb) <= 1, (i, sa, sb, qa, qb)
        assert _canonical(pa, piece, old_len, False) == _canonical(pb, piece, old_len, True), i


def test_oracle_maps_chopped_graph_like_the_32bp_one(chopped):
    g, whole, ix, piece, old_len = chopped
    rs = synth.simulate_reads(g, 150, length=150, sub_rate=0.01, seed=4)
    p = _chopped_params()
    a = H.oracle_map(whole, rs.reads, rs.quals, p, threads=8)
    b = H.oracle_map(ix, rs.reads, rs.quals, p, threads=8)
    assert (a[0]["flags"] & 1).mean() > 0.95
    _assert_same_up_to_boundaries(a, b, rs.n, piece, old_len)


@pytest.mark.gpu
def test_single_end_on_more_than_2_22_nodes(chopped, monkeypatch):
    # indels on 2 bp nodes: extensions outgrow the regular per-read stride, so chunks of 128 reads and the caps of
    # test_map_parity's 2 bp test keep every read inside the large-stride extension pool
    monkeypatch.setenv("GIRAFFE_B200_MAP_CHUNK", "128")
    g, whole, ix, piece, old_len = chopped
    rs = synth.simulate_reads(g, 600, length=150, sub_rate=0.01, ins_rate=0.001, del_rate=0.001, seed=6)
    p = _chopped_params()
    p.mapping_cap_per_read = 512; p.edit_cap_per_read = 1024
    dev = capi.Device(ix)
    got = H.gpu_map(dev, rs.reads, rs.quals, p)
    dev.close()
    want = H.oracle_map(ix, rs.reads, rs.quals, p, threads=8)
    bad = H.compare_alignments(got, want, rs.n)
    assert not bad, f"{len(bad)} of {rs.n} reads differ from the oracle; first {bad[0]}"
    on_high = sum(any((node >> 1) >= (1 << 22) for node, _, _ in H.decode_alignment(got[0][i], got[1], got[2])[2]) for i in range(rs.n))
    assert on_high > 0, "no read maps to a node id above 2^22"


@pytest.mark.gpu
@pytest.mark.parametrize("rescue", [False, True], ids=["no-rescue", "rescue"])
def test_paired_on_more_than_2_22_nodes(chopped, rescue):
    g, whole, ix, piece, old_len = chopped
    rs = _pairs(g, 300, seed=12, garble=60 if rescue else 0)
    p = _chopped_params(H.paired_params(380.0, 45.0))
    if rescue:
        p.max_rescue_attempts = H.default_map_params().max_rescue_attempts
    dev = capi.Device(ix)
    got = H.gpu_map(dev, rs.reads, rs.quals, p, paired=True)
    dev.close()
    want = H.oracle_map_paired(ix, rs.reads, rs.quals, p, threads=8)
    bad = H.compare_alignments(got, want, rs.n)
    assert not bad, f"{len(bad)} of {rs.n} reads differ from the oracle; first {bad[0]}"
    if rescue:
        assert want[4]["rescues"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("top", [pytest.param((1 << 22) + 1, id="top4194305"), pytest.param((1 << 24) + 3, id="top16777219")])
def test_device_index_builder_on_shifted_graphs(family, top):
    """gb_index_build_from_gbwt_device gives the host builder's arrays byte for byte on ids past 2^22."""
    shift, ix = family.shift(top), family.index(top)
    seqs = [""] * shift + list(family.g.node_seqs)
    dist = None if family.g.dist is None else ix.array("dist")
    nodes = ix.array("nodes")
    host = capi.HostIndex.from_gbwt(seqs, len(family.g.paths), ix.array("gbwt"), nodes["rec_off"], dist, k=family.k, w=family.w)
    dev = capi.HostIndex.from_gbwt(seqs, len(family.g.paths), ix.array("gbwt"), nodes["rec_off"], dist, k=family.k, w=family.w, device=0)
    for name in ("nodes", "seq", "gbwt", "dist", "slots", "site_dist", "table", "hits"):
        assert dev.array(name).tobytes() == host.array(name).tobytes(), name
    host.close(); dev.close()


def _fastq(reads, quals, mate):
    return b"".join(b"@p%d/%d\n" % (i, mate) + bytes(r) + b"\n+\n" + bytes(q + 33) + b"\n" for i, (r, q) in enumerate(zip(reads, quals)))


@pytest.mark.gpu
def test_fastq_gz_to_bgzf_gam_past_2_22(family):
    """FASTQ.gz inflated and parsed in HBM, mapped device-resident, emitted as GAM and compressed to BGZF on the GPU, on a
    graph whose ids reach 2^24: the container holds the host emitter's GAM of the host-buffer mapping."""
    import gzip
    import torch
    top = (1 << 24) + 3
    ix = family.index(top)
    rs = _pairs(family.g, 200, seed=14)
    r1, r2 = (_fastq(rs.reads[m::2], rs.quals[m::2], m + 1) for m in (0, 1))
    d = capi.Device(ix)
    t = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    t1, _ = d.bgzf_decompress_device(t(capi.bgzf_compress(r1, 6)))
    t2, _ = d.bgzf_decompress_device(t(capi.bgzf_compress(r2, 6)))
    fq = d.fastq_parse_device([t1, t2])
    n = fq["n_reads"]
    assert n == rs.n
    params = H.paired_params(380.0, 45.0)
    MAP_PER, EDIT_PER = 24, 64
    d_aln = torch.zeros((n, 32), dtype=torch.uint8, device="cuda")
    d_maps = torch.zeros((n * MAP_PER, 8), dtype=torch.uint8, device="cuda")
    d_edits = torch.zeros(n * EDIT_PER, dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_tot = torch.zeros(2, dtype=torch.int64, device="cuda")
    vp = lambda x: C.c_void_p(x.data_ptr())
    lib = capi.load_library()
    rc = lib.gb_map_batch_device(d.handle, C.byref(params), 1, n, vp(fq["reads"]), vp(fq["quals"]), vp(fq["read_off"]), fq["max_read_len"],
                                 vp(d_aln), vp(d_maps), n * MAP_PER, vp(d_edits), n * EDIT_PER, vp(d_status), vp(d_tot))
    assert rc == capi.GB_OK, lib.gb_last_error()
    lib.gb_device_synchronize(d.handle)
    gam = d.emit_device("gam", d_aln, d_maps, d_edits, fq["reads"], fq["read_off"], fq["quals"], fq["names"], fq["name_off"])
    bgzf = d.bgzf_compress_device(gam).cpu().numpy().tobytes()
    reads = [bytes(x) for x in rs.reads]; quals = [bytes(x) for x in rs.quals]
    rbuf, qbuf, off = H.pack_reads(reads, quals)
    aln, maps, edits, status = d.map_arrays(rbuf, qbuf, off, params, paired=True)
    assert (status == 0).all()
    nb, no = fq["names"].cpu().numpy().tobytes(), fq["name_off"].cpu().numpy()
    names = [nb[no[i]:no[i + 1]].decode() for i in range(n)]
    want = capi.emit_text("gam", ix.view, aln, maps, edits, rbuf, qbuf, off, names=names)
    assert gzip.decompress(bgzf) == want
    d.close()


def test_index_file_with_a_hit_payload_off_its_node_is_refused(tmp_path):
    """The seeding kernels take two seeds on one node to share x_in, so a file whose hit payload is not its node's is refused."""
    g = synth.make_variant_graph(length=6000, n_snp=10, n_ins=2, n_del=2, n_haps=4, seed=3)
    ix = g.build_index()
    path = tmp_path / "ix.gbflat"
    ix.save(str(path))
    capi.HostIndex.load(str(path)).close()
    pad = lambda b: (b + 15) // 16 * 16
    v = ix.view
    hits_at = 80 + pad(v.n_nodes * 16) + pad(v.seq_bytes) + pad(v.gbwt_words * 4) + pad(v.n_nodes // 2 * 16) + pad(v.table_cells * 16)
    data = bytearray(path.read_bytes())
    data[hits_at + 8] ^= 1                                    # x_in of the first hit's payload
    path.write_bytes(bytes(data))
    with pytest.raises(capi.GbError) as e:
        capi.HostIndex.load(str(path))
    assert e.value.code == capi.GB_ERR_FORMAT
    ix.close()
