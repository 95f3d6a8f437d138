"""gb_emit_gaf_device / gb_emit_gam_device: GAF and GAM formatted on the GPU from records in HBM must be the bytes the host
emitters gb_emit_gaf / gb_emit_gam write for the same records — oracle records, records straight out of
gb_map_batch_device, and hand-made records at the formatting corners (insertion-only mappings, empty paths, negative
scores, dv:f in exponent form, GAM group boundaries).  Refusals: the records the host emitter refuses, and a short
output buffer, which reports the bytes needed."""
import ctypes as C
import re

import numpy as np
import pytest

import helpers as H
from test_emit import ABSENT, MAPPED, PAIRED, RESCUED, SEC, _build, _corner_batch, _dv_sweep, _hand_graph, _host, _names_t, _reads
from vg_b200 import capi, synth

pytestmark = pytest.mark.gpu


def _t(a, dtype=None):
    import torch
    a = np.ascontiguousarray(a if dtype is None else a.astype(dtype))
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy() if dtype is None else a.copy()).cuda()


def _device(dev, kind, aln, maps, edits, rbuf, qbuf, read_off, names=None):
    nt = None if names is None else [_t(a, a.dtype) if a.dtype == np.int64 else _t(a) for a in _names_t(names)]
    return dev.emit_device(kind, _t(aln), _t(maps), _t(edits, np.uint32), _t(rbuf), _t(read_off, np.int64), None if qbuf is None else _t(qbuf),
                           *(nt or (None, None))).cpu().numpy().tobytes()


def _same(dev, view, aln, maps, edits, rbuf, qbuf, read_off, names=None, kinds=("gaf", "gam")):
    for kind in kinds:
        got = _device(dev, kind, aln, maps, edits, rbuf, qbuf, read_off, names)
        want = _host(kind, view, aln, maps, edits, rbuf, qbuf, read_off, names, cap=4096 + 2 * len(got) + 4096 * len(aln))
        assert got == want, f"{kind}: {len(got)} vs {len(want)} bytes, first difference at {_first_diff(got, want)}"


def _first_diff(a, b):
    n = min(len(a), len(b))
    d = np.flatnonzero(np.frombuffer(a[:n], np.uint8) != np.frombuffer(b[:n], np.uint8))
    return int(d[0]) if len(d) else n


def _mapped_records(paired, rescue=False, with_n=True):
    g = synth.make_variant_graph(length=60000, n_snp=100, n_ins=12, n_del=12, n_haps=4, seed=8)
    index = g.build_index()
    rng = np.random.default_rng(3)
    if paired:
        rs = synth.simulate_pairs(g, 150, sub_rate=0.02, seed=5)
    else:
        rs = synth.simulate_reads(g, 300, length=150, sub_rate=0.02, ins_rate=0.004, del_rate=0.004, seed=6)
    for i in rng.integers(0, rs.n, size=20):                   # soft clips: garbage at one end
        rs.reads[i, :12] = synth.BASES[rng.integers(0, 4, size=12)]
    rs.reads[7] = synth.BASES[rng.integers(0, 4, size=rs.length)]      # an unmapped read
    if with_n:
        for i in range(10, rs.n, 17):
            rs.reads[i, rng.integers(0, rs.length, size=3)] = ord("N")
    if rescue:
        for i in range(1, rs.n, 8):                            # mates too noisy to seed: rescued from their partners
            m = rng.random(rs.length) < 0.12
            rs.reads[i, m] = synth.BASES[rng.integers(0, 4, size=int(m.sum()))]
    if paired:
        p = H.paired_params(); p.max_rescue_attempts = 15 if rescue else 0
        res = H.oracle_map_paired(index, rs.reads, rs.quals, p, threads=8)
    else:
        res = H.oracle_map(index, rs.reads, rs.quals, threads=8)
    return g, index, rs, res


@pytest.mark.parametrize("paired", [False, True])
def test_oracle_records_match_the_host_emitters(paired):
    g, index, rs, res = _mapped_records(paired)
    dev = capi.Device(index, 0)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    aln, maps, edits = res[0], res[1], res[2]
    assert ((aln["flags"] & MAPPED) == 0).any() and ((aln["flags"] & MAPPED) != 0).sum() > rs.n // 2
    names = [f"pair{i // 2}/{i % 2 + 1}" if paired else f"frag{i}" for i in range(rs.n)]
    for q in (qbuf, None):
        for nm in (names, None):
            _same(dev, index.view, aln, maps, edits, rbuf, q, read_off, nm)
    # a permuted subset of the records
    sub = aln[np.random.default_rng(4).permutation(rs.n)[: rs.n // 3]]
    _same(dev, index.view, sub, maps, edits, rbuf, qbuf, read_off, names)
    dev.close()


def test_rescued_pairs_match_the_host_emitters():
    g, index, rs, res = _mapped_records(True, rescue=True)
    assert ((res[0]["flags"] & RESCUED) != 0).sum() >= 3
    dev = capi.Device(index, 0)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    _same(dev, index.view, res[0], res[1], res[2], rbuf, qbuf, read_off, [f"p{i // 2}.{i % 2}" for i in range(rs.n)])
    dev.close()


@pytest.mark.parametrize("paired", [False, True])
def test_multimaps_secondary_and_absent_ranks(paired):
    from test_multimap import repeat_graph
    g = repeat_graph(); index = g.build_index()
    p = H.paired_params() if paired else H.default_map_params()
    p.max_multimaps = 3
    if paired:
        rs = synth.simulate_pairs(g, 150, sub_rate=0.01, seed=37)
        res = H.oracle_map_paired(index, rs.reads, rs.quals, p, threads=8)
    else:
        rs = synth.simulate_reads(g, 300, length=150, sub_rate=0.01, seed=36)
        res = H.oracle_map(index, rs.reads, rs.quals, p, threads=8)
    aln = res[0]
    assert ((aln["flags"] & SEC) != 0).sum() > 20 and ((aln["flags"] & ABSENT) != 0).sum() > 20
    dev = capi.Device(index, 0)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    _same(dev, index.view, aln, res[1], res[2], rbuf, qbuf, read_off)
    _same(dev, index.view, aln, res[1], res[2], rbuf, None, read_off, [f"r{i}" for i in range(rs.n)])
    dev.close()


def test_records_straight_from_map_batch_device():
    import torch
    g = synth.make_variant_graph(length=60000, n_snp=100, n_ins=12, n_del=12, n_haps=4, seed=8)
    index = g.build_index()
    dev = capi.Device(index, 0)
    rs = synth.simulate_pairs(g, 500, sub_rate=0.01, seed=9)
    n, L = rs.n, rs.length
    p = H.paired_params()
    d_reads = torch.from_numpy(rs.reads.reshape(-1).copy()).cuda()
    d_quals = torch.from_numpy(rs.quals.reshape(-1).copy()).cuda()
    d_off = torch.arange(n + 1, dtype=torch.int64, device="cuda") * L
    d_aln = torch.zeros((n, 32), dtype=torch.uint8, device="cuda")
    d_maps = torch.zeros((n * 14, 8), dtype=torch.uint8, device="cuda")
    d_edits = torch.zeros(n * 20, dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_tot = torch.zeros(2, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    lib = capi.load_library()
    vp = lambda t: C.c_void_p(t.data_ptr())
    rc = lib.gb_map_batch_device(dev.handle, C.byref(p), 1, n, vp(d_reads), vp(d_quals), vp(d_off), L, vp(d_aln), vp(d_maps), n * 14,
                                 vp(d_edits), n * 20, vp(d_status), vp(d_tot))
    assert rc == capi.GB_OK
    # emitted from HBM before anything is read back
    gaf = dev.emit_device("gaf", d_aln, d_maps, d_edits, d_reads, d_off, d_quals).cpu().numpy().tobytes()
    gam = dev.emit_device("gam", d_aln, d_maps, d_edits, d_reads, d_off, d_quals).cpu().numpy().tobytes()
    tot = d_tot.cpu().numpy()
    aln = d_aln.cpu().numpy().view(capi.alignment_dt).reshape(-1)
    maps = d_maps.cpu().numpy().view(capi.mapping_dt).reshape(-1)[: int(tot[0]) + 1]
    edits = d_edits.cpu().numpy().view(np.uint32)[: int(tot[1]) + 1]
    assert (d_status.cpu().numpy() == 0).all() and ((aln["flags"] & MAPPED) != 0).mean() > 0.9
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    assert gaf == _host("gaf", index.view, aln, maps, edits, rbuf, qbuf, read_off)
    assert gam == _host("gam", index.view, aln, maps, edits, rbuf, qbuf, read_off)
    dev.close()


# ---- hand-made records -------------------------------------------------------------------------------------------------
def test_hand_made_formatting_corners():
    index = _hand_graph()
    dev = capi.Device(index, 0)
    rbuf, qbuf, read_off, recs, aln, maps, edits = _corner_batch()
    gaf = _host("gaf", index.view, aln, maps, edits, rbuf, qbuf, read_off, cap=1 << 22).decode().splitlines()
    assert gaf[2].split("\t")[5] == "*" and "AS:i:-2147483648" in gaf[2]
    assert re.search(r"\tdv:f:[1-9](\.\d+)?e-05(\t|$)", gaf[4]) and re.search(r"\tdv:f:6\.6\d*e-05(\t|$)", gaf[5])
    assert len(gaf) == len(recs) - 1
    names = [f"hand{i}" for i in range(len(read_off) - 1)]
    for q in (qbuf, None):
        for nm in (names, None):
            _same(dev, index.view, aln, maps, edits, rbuf, q, read_off, nm)
    dev.close()


@pytest.mark.parametrize("n_present", [0, 999, 1000, 1001, 2001])
def test_gam_group_boundaries(n_present):
    index = _hand_graph()
    dev = capi.Device(index, 0)
    rbuf, qbuf, read_off = _reads([40] * 64)
    rng = np.random.default_rng(n_present)
    recs = []
    for i in range(n_present):
        if i % 7 == 3:
            recs.append((i % 64, ABSENT, 0, []))                                        # absent ranks between present ones
        r = i % 64
        recs.append((r, MAPPED | (PAIRED if i % 5 == 0 else 0), int(rng.integers(-50, 60)),
                     [(2 + 2 * (i % 3), int(rng.integers(0, 900)), [("M", 20, 0), ("S", 1, int(rng.integers(0, 4))), ("M", 19, 0)])]))
    aln, maps, edits = _build(recs) if recs else _build([(0, ABSENT, 0, [])])
    names = [f"g{i}" * (1 + i % 4) for i in range(64)]
    _same(dev, index.view, aln, maps, edits, rbuf, qbuf, read_off, names, kinds=("gam",))
    gam = _device(dev, "gam", aln, maps, edits, rbuf, qbuf, read_off, names)
    import test_gam as TG
    if n_present:
        msgs, tagged = TG.read_stream(gam)
        assert len(msgs) == n_present
    else:
        assert gam == b""
    dev.close()


def test_dv_matches_printf_g6_over_a_dense_range():
    """every (matches, block) pair with block <= 1100 and long deletions (test_emit._dv_sweep): the dv:f field must read as
    Python's '%.6g' % (1.0 - m / b), which is correctly rounded like glibc."""
    index = _hand_graph()
    dev = capi.Device(index, 0)
    rbuf, read_off, (aln, maps, edits), want = _dv_sweep()
    got = _device(dev, "gaf", aln, maps, edits, rbuf, None, read_off).decode()
    dv = [line.rsplit("\tdv:f:", 1)[1] for line in got.splitlines()]
    bad = [(i, g, w) for i, (g, w) in enumerate(zip(dv, want)) if g != w]
    assert len(dv) == len(want) and not bad, bad[:10]
    assert got.encode() == _host("gaf", index.view, aln, maps, edits, rbuf, None, read_off, cap=2 * len(got) + (1 << 20))
    dev.close()


# ---- refusals ------------------------------------------------------------------------------------------------------------
def _raw(dev, kind, aln, maps, edits, rbuf, qbuf, read_off, n_maps, n_edits, n_reads, out, cap, names=None, name_off=None, maps_null=False):
    lib = capi.load_library()
    fn = {"gaf": lib.gb_emit_gaf_device, "gam": lib.gb_emit_gam_device}[kind]
    vp = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    used = C.c_uint64(12345)
    rc = fn(dev.handle, aln.numel() // 32, vp(aln), None if maps_null else vp(maps), n_maps, vp(edits), n_edits, n_reads, vp(rbuf), vp(qbuf),
            vp(read_off), vp(names), vp(name_off), vp(out), cap, C.byref(used))
    return rc, used.value


def test_refusals_write_nothing():
    import torch
    g, index, rs, res = _mapped_records(False, with_n=False)
    dev = capi.Device(index, 0)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    mapped = res[0][(res[0]["flags"] & MAPPED) != 0][:20].copy()
    tr, tq, to, tm, te = _t(rbuf), _t(qbuf), _t(read_off, np.int64), _t(res[1]), _t(res[2], np.uint32)
    nm, ne = len(res[1]), len(res[2])
    out = torch.full((1 << 20,), 0xAB, dtype=torch.uint8, device="cuda")
    nbuf, noff = _names_t([f"n{i}" for i in range(rs.n)])
    for kind in ("gaf", "gam"):
        assert _raw(dev, kind, _t(mapped), tm, te, tr, tq, to, nm, ne, rs.n, out, len(out))[0] == capi.GB_OK
        capi.load_library().gb_device_synchronize(dev.handle); out.fill_(0xAB)
        cases = [dict(n_maps=int(mapped["mapping_off"].max())), dict(n_edits=int(mapped["edit_off"].max())),
                 dict(n_reads=int(mapped["read_id"].max())), dict(maps_null=True)]
        bad_records = []
        b = mapped.copy(); b[3]["n_edits"] += 1; bad_records.append(b)                               # edits no longer add up to the read
        b = mapped.copy(); b[5]["mapping_off"] = b[6]["mapping_off"]; bad_records.append(b)           # another record's mappings
        b = mapped.copy(); b[2]["read_id"] = rs.n; bad_records.append(b)                             # read outside the batch
        for rec in bad_records:
            assert _raw(dev, kind, _t(rec), tm, te, tr, tq, to, nm, ne, rs.n, out, len(out))[0] == capi.GB_ERR_ARG
        # a paired record whose mate lies outside the batch (n_reads cut just behind the record's own read)
        b = mapped[mapped["read_id"] < rs.n - 2].copy(); b[0]["read_id"] = rs.n - 2
        assert _raw(dev, kind, _t(b), tm, te, tr, tq, to, nm, ne, rs.n - 1, out, len(out))[0] == capi.GB_OK
        capi.load_library().gb_device_synchronize(dev.handle); out.fill_(0xAB)
        b[0]["flags"] |= PAIRED
        assert _raw(dev, kind, _t(b), tm, te, tr, tq, to, nm, ne, rs.n - 1, out, len(out))[0] == capi.GB_ERR_ARG
        for c in cases:
            args = dict(n_maps=nm, n_edits=ne, n_reads=rs.n, maps_null=False); args.update(c)
            assert _raw(dev, kind, _t(mapped), tm, te, tr, tq, to, args["n_maps"], args["n_edits"], args["n_reads"], out, len(out),
                        maps_null=args["maps_null"])[0] == capi.GB_ERR_ARG
        # a node outside the graph, an offset past the end of its node
        maps_bad = res[1].copy(); maps_bad[int(mapped[0]["mapping_off"])]["node"] = index.view.n_nodes
        assert _raw(dev, kind, _t(mapped), _t(maps_bad), te, tr, tq, to, nm, ne, rs.n, out, len(out))[0] == capi.GB_ERR_ARG
        maps_bad = res[1].copy(); maps_bad[int(mapped[1]["mapping_off"])]["offset"] = 1020
        assert _raw(dev, kind, _t(mapped), _t(maps_bad), te, tr, tq, to, nm, ne, rs.n, out, len(out))[0] == capi.GB_ERR_ARG
        # name offsets that go backwards, read offsets that go backwards
        noff_bad = noff.copy(); noff_bad[5] = noff_bad[7]
        assert _raw(dev, kind, _t(mapped), tm, te, tr, tq, to, nm, ne, rs.n, out, len(out), _t(nbuf), _t(noff_bad, np.int64))[0] == capi.GB_ERR_ARG
        off_bad = read_off.astype(np.int64).copy(); r = int(mapped[0]["read_id"]); off_bad[r + 1] = off_bad[r] - 1
        assert _raw(dev, kind, _t(mapped), tm, te, tr, tq, _t(off_bad, np.int64), nm, ne, rs.n, out, len(out))[0] == capi.GB_ERR_ARG
        torch.cuda.synchronize()
        assert (out == 0xAB).all(), "a refused call wrote output"
    dev.close()


def test_capacity_reports_the_bytes_needed():
    import torch
    g, index, rs, res = _mapped_records(True, with_n=False)
    dev = capi.Device(index, 0)
    rbuf, qbuf, read_off = H.pack_reads(rs.reads, rs.quals)
    tr, tq, to, tm, te, ta = _t(rbuf), _t(qbuf), _t(read_off, np.int64), _t(res[1]), _t(res[2], np.uint32), _t(res[0])
    for kind in ("gaf", "gam"):
        want = _host(kind, index.view, res[0], res[1], res[2], rbuf, qbuf, read_off)
        need = len(want)
        out = torch.full((need + 64,), 0xAB, dtype=torch.uint8, device="cuda")
        rc, used = _raw(dev, kind, ta, tm, te, tr, tq, to, len(res[1]), len(res[2]), rs.n, out, need - 1)
        torch.cuda.synchronize()
        assert rc == capi.GB_ERR_CAPACITY and used == need and (out == 0xAB).all()
        rc, used = _raw(dev, kind, ta, tm, te, tr, tq, to, len(res[1]), len(res[2]), rs.n, out, need)
        assert capi.load_library().gb_device_synchronize(dev.handle) == capi.GB_OK
        assert rc == capi.GB_OK and used == need
        got = out.cpu().numpy().tobytes()
        assert got[:need] == want and got[need:] == b"\xab" * 64
    dev.close()
