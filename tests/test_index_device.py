"""gb_index_from_gbz_device / gb_index_build_from_gbwt_device: the minimizer step of the index builder on the GPU.  The host
builder is the oracle: on every graph below the device-built index must equal the host-built one array by array, and
gb_index_save must write the same file."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import helpers as H
import vcf_graph as V
from vg_b200 import capi, synth

GBZ = Path(__file__).parent / "golden" / "gbz" / "y.giraffe.gbz"
ARRAYS = ("nodes", "seq", "gbwt", "dist", "slots", "site_dist", "table", "hits")


def _gpu_present():
    import torch
    return torch.cuda.is_available()


def _has_model(index):
    return capi.load_library().gb_index_has_distance_model(index._h)


def assert_identical(host, dev, tmp_path):
    for name in ARRAYS:
        assert np.array_equal(host.array(name), dev.array(name)), name
    for field in ("n_nodes", "k", "w", "n_paths"):
        assert getattr(host.view, field) == getattr(dev.view, field), field
    assert _has_model(host) == _has_model(dev)
    host.save(tmp_path / "host.gbflat"); dev.save(tmp_path / "dev.gbflat")
    assert (tmp_path / "host.gbflat").read_bytes() == (tmp_path / "dev.gbflat").read_bytes()


def both_from_gbwt(seqs, paths, k, w, dist=None):
    """The flat GBWT of the path-built index, handed to the host and the device builder."""
    ref = capi.HostIndex(seqs, paths, dist, k=k, w=w)
    words, rec_off = ref.array("gbwt").copy(), ref.array("nodes")["rec_off"].copy()
    ref.close()
    host = capi.HostIndex.from_gbwt(seqs, len(paths), words, rec_off, dist, k=k, w=w)
    dev = capi.HostIndex.from_gbwt(seqs, len(paths), words, rec_off, dist, k=k, w=w, device=0)
    return host, dev


def check_from_gbwt(tmp_path, seqs, paths, k=29, w=11, dist=None, min_hits=1):
    host, dev = both_from_gbwt(seqs, paths, k, w, dist)
    assert int(host.view.n_hits) >= min_hits
    assert_identical(host, dev, tmp_path)
    t_host, t_dev = host.timing(), dev.timing()
    for name in ("start_nodes", "continuations", "raw_pairs", "unique_pairs"):
        assert t_host[name] == t_dev[name], name
    host.close(); dev.close()
    return t_dev


def _random_seq(rng, n):
    return "".join("ACGT"[i] for i in rng.integers(0, 4, size=n))


# ---- without a device ------------------------------------------------------------------------------------------------------

def test_arguments_are_refused_before_the_device_is_looked_at():
    lib = capi.load_library()
    h = C.c_void_p()
    g = synth.make_tiny_graph()
    ref = g.build_index()
    seq = np.frombuffer("".join(g.node_seqs).encode(), dtype=np.uint8).copy()
    node_off = np.zeros(len(g.node_seqs) + 1, dtype=np.uint64); node_off[1:] = np.cumsum([len(s) for s in g.node_seqs])
    words, ro = ref.array("gbwt").copy(), ref.array("nodes")["rec_off"].copy()

    def gbwt(k=29, w=11, dev=0, out=True, node_seq=True):
        return lib.gb_index_build_from_gbwt_device(len(g.node_seqs), capi.ptr(seq) if node_seq else None, capi.ptr(node_off),
                                                   len(g.paths), capi.ptr(words), len(words), capi.ptr(ro), None, k, w, 0, None,
                                                   None, dev, C.byref(h) if out else None)
    for k, w in ((0, 11), (32, 11), (29, 0)):
        assert lib.gb_index_from_gbz_device(str(GBZ).encode(), k, w, 0, C.byref(h)) == capi.GB_ERR_ARG
        assert gbwt(k, w) == capi.GB_ERR_ARG
    assert lib.gb_index_from_gbz_device(None, 29, 11, 0, C.byref(h)) == capi.GB_ERR_ARG
    assert lib.gb_index_from_gbz_device(str(GBZ).encode(), 29, 11, 0, None) == capi.GB_ERR_ARG
    assert lib.gb_index_from_gbz_device(str(GBZ).encode(), 29, 11, -1, C.byref(h)) == capi.GB_ERR_ARG
    assert gbwt(out=False) == capi.GB_ERR_ARG and gbwt(node_seq=False) == capi.GB_ERR_ARG and gbwt(dev=-1) == capi.GB_ERR_ARG
    ref.close()


def test_no_host_fallback_without_a_device():
    if _gpu_present():
        pytest.skip("a GPU is present")
    with pytest.raises(capi.GbError) as e:
        capi.HostIndex.from_gbz(GBZ, k=31, w=50, device=0)
    assert e.value.code == capi.GB_ERR_NO_DEVICE
    g = synth.make_tiny_graph()
    ref = g.build_index()
    with pytest.raises(capi.GbError) as e:
        capi.HostIndex.from_gbwt(g.node_seqs, len(g.paths), ref.array("gbwt"), ref.array("nodes")["rec_off"], g.dist, device=0)
    assert e.value.code == capi.GB_ERR_NO_DEVICE
    ref.close()


def test_the_host_build_reports_its_steps():
    g = synth.make_variant_graph(length=20000, n_snp=40, n_ins=5, n_del=5, n_haps=4, seed=12)
    ref = g.build_index()
    again = capi.HostIndex.from_gbwt(g.node_seqs, len(g.paths), ref.array("gbwt"), ref.array("nodes")["rec_off"], g.dist)
    t = again.timing()
    assert t["start_nodes"] == int((ref.array("nodes")["size"][2::2] > 0).sum())        # forward-only haplotypes: forward starts
    assert t["continuations"] >= t["start_nodes"] and t["raw_pairs"] >= t["unique_pairs"] == int(ref.view.n_hits)
    assert all(t[s] >= 0 for s in ("sequences_s", "distance_s", "gbwt_s", "minimizers_s", "table_s"))
    ref.close(); again.close()


# ---- on the GPU: the device-built index equals the host-built one -----------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("k,w", [(31, 50), (29, 11)])
def test_reference_gbz(k, w, tmp_path):
    host, dev = capi.HostIndex.from_gbz(GBZ, k=k, w=w), capi.HostIndex.from_gbz(GBZ, k=k, w=w, device=0)
    assert_identical(host, dev, tmp_path)
    if (k, w) == (31, 50):
        d = GBZ.parent
        from_min = capi.HostIndex.from_gbz_min(GBZ, d / "y.min", d / "y.zipcodes")
        for name in ("table", "hits"):
            assert np.array_equal(from_min.array(name), dev.array(name)), name
        from_min.close()
    host.close(); dev.close()


FAMILIES = {
    "variants": (lambda: synth.make_variant_graph(length=40000, n_snp=120, n_ins=15, n_del=15, n_haps=8, seed=4), 29, 11),
    "repeats": (lambda: synth.make_variant_graph(length=24000, n_snp=40, n_ins=4, n_del=4, n_haps=4, seed=23, repeat_unit=600,
                                                 repeat_copies=6), 29, 11),
    "nested": (lambda: synth.make_nested_graph(n_items=120, n_haps=10, seed=5), 11, 5),
    "branchy": (lambda: synth.make_branchy_graph(n_layers=600, n_haps=16, seed=4), 29, 11),
    "config-2": (lambda: synth.make_variant_graph(), 29, 11),
    "config-4 branchy": (lambda: synth.make_branchy_graph(), 29, 11),
    "1000 Genomes slice": (lambda: V.kgp_100k()[0], 29, 11),
    "x.vcf.gz": (lambda: V.small_x()[0], 29, 11),
    "variants k31 w1": (lambda: synth.make_variant_graph(length=20000, n_snp=60, n_ins=8, n_del=8, n_haps=6, seed=7), 31, 1),
    "variants k31 w32": (lambda: synth.make_variant_graph(length=20000, n_snp=60, n_ins=8, n_del=8, n_haps=6, seed=7), 31, 32),
    "variants k15 w5": (lambda: synth.make_variant_graph(length=20000, n_snp=60, n_ins=8, n_del=8, n_haps=6, seed=7), 15, 5),
}


@pytest.mark.gpu
@pytest.mark.parametrize("which", list(FAMILIES))
def test_graph_families(which, tmp_path):
    make, k, w = FAMILIES[which]
    g = make()
    check_from_gbwt(tmp_path, g.node_seqs, g.paths, k, w, g.dist, min_hits=50)


@pytest.mark.gpu
def test_haplotypes_on_reverse_strands_enumerate_every_start_node(tmp_path):
    """No distance model (a haplotype steps onto a reverse strand), so reverse start nodes are enumerated too."""
    rng = np.random.default_rng(11)
    seqs = [_random_seq(rng, int(n)) for n in rng.integers(5, 40, size=40)]
    paths = []
    for h in range(6):
        p = [2 * (i + 1) + int(rng.random() < 0.3) for i in range(40)]
        paths.append(p if h % 2 == 0 else [v ^ 1 for v in reversed(p)])
    t = check_from_gbwt(tmp_path, seqs, paths, 15, 5)
    nodes = capi.HostIndex(seqs, paths, k=15, w=5)
    assert t["start_nodes"] == int((nodes.array("nodes")["size"][2:] > 0).sum()) and not _has_model(nodes)
    nodes.close()


@pytest.mark.gpu
def test_cycle(tmp_path):
    rng = np.random.default_rng(12)
    seqs = [_random_seq(rng, int(n)) for n in rng.integers(3, 30, size=12)]
    loop = [2 * i for i in range(3, 7)]
    paths = [[2, 4, 6] + loop * 3 + [16, 18], [2, 4, 6] + loop + [16, 18, 20], [4, 6] + loop * 5 + [22, 24]]
    check_from_gbwt(tmp_path, seqs, paths, 15, 5)


@pytest.mark.gpu
def test_nodes_of_1024_bp(tmp_path):
    rng = np.random.default_rng(13)
    seqs = [_random_seq(rng, 1024) for _ in range(8)]
    paths = [[2, 4, 8, 10, 14, 16], [2, 6, 8, 12, 14, 16], [2, 4, 8, 12, 14]]
    check_from_gbwt(tmp_path, seqs, paths, 29, 11)
    check_from_gbwt(tmp_path, seqs, paths, 31, 32)


@pytest.mark.gpu
def test_haplotypes_around_one_window(tmp_path):
    """k = 15, w = 5: a window is 19 bases.  Haplotypes of 10, 18 (one base short), 19 and 20 (one base over) bases on their
    own nodes, and haplotypes that end early after a shared start node."""
    rng = np.random.default_rng(14)
    seqs, paths = [], []
    for total in (10, 18, 19, 20):
        a = len(seqs) + 1
        seqs += [_random_seq(rng, total // 2), _random_seq(rng, total - total // 2)]
        paths.append([2 * a, 2 * a + 2])
    a = len(seqs) + 1
    seqs += [_random_seq(rng, 6), _random_seq(rng, 12), _random_seq(rng, 13), _random_seq(rng, 30)]
    paths += [[2 * a, 2 * a + 2], [2 * a, 2 * a + 4], [2 * a, 2 * a + 6], [2 * a, 2 * a + 2, 2 * a + 6]]
    check_from_gbwt(tmp_path, seqs, paths, 15, 5)


@pytest.mark.gpu
def test_n_runs_inside_and_across_nodes(tmp_path):
    rng = np.random.default_rng(15)
    seqs = []
    for i in range(30):
        s = list(_random_seq(rng, int(rng.integers(10, 32))))
        if i % 3 == 0:
            at = int(rng.integers(0, len(s) - 3)); s[at:at + 3] = "NNN"
        if i % 4 == 1:
            s[-2:] = "NN"
        if i % 4 == 2:
            s[:2] = "NN"
        seqs.append("".join(s))
    paths = [[2 * (i + 1) for i in range(30) if i % 5 != h] for h in range(5)]
    check_from_gbwt(tmp_path, seqs, paths, 15, 5)


@pytest.mark.gpu
def test_unused_low_node_ids(tmp_path):
    shift = 100
    g = synth.make_variant_graph(length=20000, n_snp=40, n_ins=5, n_del=5, n_haps=4, seed=12)
    seqs = [""] * shift + list(g.node_seqs)
    paths = [[v + 2 * shift for v in p] for p in g.paths]
    dist = np.zeros(len(seqs) + 1, dtype=capi.dist_dt); dist["allele"] = 0xFFFF
    dist[shift + 1:] = np.asarray(g.dist)[1:]
    check_from_gbwt(tmp_path, seqs, paths, 29, 11, dist, min_hits=50)


@pytest.mark.gpu
def test_several_batches_of_start_nodes(tmp_path, monkeypatch):
    g = synth.make_variant_graph(length=40000, n_snp=120, n_ins=15, n_del=15, n_haps=8, seed=4)
    monkeypatch.setenv("GIRAFFE_B200_INDEX_POOL_PAIRS", "1000")
    t = check_from_gbwt(tmp_path, g.node_seqs, g.paths, 29, 11, g.dist, min_hits=50)
    assert t["raw_pairs"] > 5 * 1000


@pytest.mark.gpu
def test_damaged_gbwt_records_give_the_host_codes():
    g = synth.make_variant_graph(length=6000, n_snp=20, n_ins=3, n_del=3, n_haps=4, seed=9)
    ref = g.build_index()
    words, rec_off = ref.array("gbwt").copy(), ref.array("nodes")["rec_off"].copy()
    v = int(np.flatnonzero(rec_off)[5]); off = int(rec_off[v])
    n_edges = int(words[off])
    damage = [lambda w2, r2: r2.__setitem__(v, len(w2) + 5),
              lambda w2, r2: w2.__setitem__(off, 5000),
              lambda w2, r2: w2.__setitem__(off + 2, 2 * (len(g.node_seqs) + 9)),
              lambda w2, r2: w2.__setitem__(off + 3, 1 << 30),
              lambda w2, r2: w2.__setitem__(off + 2 + 2 * n_edges, (1 << 10) | 900)]
    for mut in damage:
        w2, r2 = words.copy(), rec_off.copy(); mut(w2, r2)
        codes = []
        for device in (None, 0):
            with pytest.raises(capi.GbError) as e:
                capi.HostIndex.from_gbwt(g.node_seqs, len(g.paths), w2, r2, g.dist, device=device)
            codes.append(e.value.code)
        assert codes[0] == codes[1] == capi.GB_ERR_FORMAT
    ref.close()


@pytest.mark.gpu
def test_two_calls_give_the_same_bytes(tmp_path):
    g = synth.make_branchy_graph(n_layers=600, n_haps=16, seed=4)
    ref = g.build_index()
    args = (g.node_seqs, len(g.paths), ref.array("gbwt").copy(), ref.array("nodes")["rec_off"].copy(), g.dist)
    a, b = capi.HostIndex.from_gbwt(*args, device=0), capi.HostIndex.from_gbwt(*args, device=0)
    assert_identical(a, b, tmp_path)
    for x in (ref, a, b):
        x.close()


@pytest.mark.gpu
def test_reads_map_identically_on_either_index():
    g = synth.make_variant_graph(length=40000, n_snp=120, n_ins=15, n_del=15, n_haps=8, seed=4)
    host, dev_built = both_from_gbwt(g.node_seqs, g.paths, 29, 11, g.dist)
    rs = synth.simulate_reads(g, 2000, length=150, sub_rate=0.01, seed=6)
    results = []
    for index in (host, dev_built):
        dev = capi.Device(index)
        results.append(H.gpu_map(dev, rs.reads, rs.quals))
        dev.close()
    assert not H.compare_alignments(results[1], results[0], rs.n, mapq_tol=0)
    assert (results[0][0]["flags"] & 1).mean() > 0.9
    host.close(); dev_built.close()
