"""MinimizerMapper::map parity (single-end): gb_map_batch on the GPU vs the oracle restatement
of map_from_extensions, on the BASELINE.json config families at oracle-sized inputs."""
import numpy as np
import pytest

import helpers as H
from vg_b200 import capi, synth


def _run(g, rs, params=None):
    index = g.build_index()
    dev = capi.Device(index)
    got = H.gpu_map(dev, rs.reads, rs.quals, params)
    want = H.oracle_map(index, rs.reads, rs.quals, params, threads=8)
    bad = H.compare_alignments(got, want, rs.n)
    dev.close()
    assert not bad, f"{len(bad)} of {rs.n} reads differ; first: read {bad[0][0]}\n got={bad[0][1]}\nwant={bad[0][2]}"
    return got, want


def test_oracle_maps_clean_reads_to_their_origin():
    g = synth.make_tiny_graph()
    index = g.build_index()
    rs = synth.simulate_reads(g, 200, length=150, sub_rate=0.0, seed=31)
    aln, maps, edits, status, counters = H.oracle_map(index, rs.reads, rs.quals)
    assert (aln["flags"] & 1).all()
    assert (aln["score"] == 160).all()
    assert counters["direct"] == 200 and counters["tail_dps"] == 0
    for i in range(rs.n):
        score, mapq, path = H.decode_alignment(aln[i], maps, edits)
        node, off = path[0][0], path[0][1]
        h, p = int(rs.hap[i]), int(rs.pos[i])
        if not rs.rev[i]:
            assert (node >> 1, off) == (int(g.hap_node[h][p]), int(g.hap_off[h][p])) and (node & 1) == 0
        else:
            assert (node & 1) == 1


@pytest.mark.gpu
def test_map_parity_config1_tiny():
    # BASELINE.json configs[0]: ~1 kbp graph, 1k SE 150 bp reads at 1 % substitutions
    g = synth.make_tiny_graph()
    rs = synth.simulate_reads(g, 1000, length=150, sub_rate=0.01, seed=11)
    got, want = _run(g, rs)
    assert (got[0]["flags"] & 1).mean() > 0.99


@pytest.mark.gpu
@pytest.mark.parametrize("sub_rate,ins_rate,del_rate,length", [(0.002, 0.0002, 0.0002, 150), (0.02, 0.002, 0.002, 150),
                                                               (0.03, 0.01, 0.01, 250)])
def test_map_parity_variant_graph(sub_rate, ins_rate, del_rate, length):
    # configs[1]/[4] family: SNP+indel graph; the last row is the 250 bp / 5 % error tail-DP stress
    g = synth.make_variant_graph(length=200000, n_snp=320, n_ins=40, n_del=40, n_haps=8, seed=2)
    rs = synth.simulate_reads(g, 3000, length=length, sub_rate=sub_rate, ins_rate=ins_rate, del_rate=del_rate, seed=55)
    _run(g, rs)


@pytest.mark.gpu
def test_map_parity_branchy_graph():
    # configs[3] family: 8-bp nodes, 4-way bubbles
    g = synth.make_branchy_graph(n_layers=4000, n_haps=16, seed=4)
    rs = synth.simulate_reads(g, 2000, length=150, sub_rate=0.005, seed=44)
    _run(g, rs)


@pytest.mark.gpu
def test_map_edge_cases():
    g = synth.make_tiny_graph()
    index = g.build_index()
    dev = capi.Device(index)
    hs = g.hap_seq[0]
    reads = [bytes(hs[100:250]), b"ACGT", b"N" * 150, bytes(hs[300:339]) , bytes(hs[10:160]).replace(b"A", b"N", 3),
             bytes(synth.revcomp_bytes(hs[400:550])), b"A" * 150, bytes(hs[0:150]), bytes(hs[-150:])]
    quals = [bytes([30] * len(r)) for r in reads]
    got = H.gpu_map(dev, reads, quals)
    want = H.oracle_map(index, reads, quals)
    bad = H.compare_alignments(got, want, len(reads))
    assert not bad, bad[0]
    # no qualities: explored cap is +inf on both sides
    got = H.gpu_map(dev, reads, None)
    want = H.oracle_map(index, reads, None)
    bad = H.compare_alignments(got, want, len(reads))
    assert not bad, bad[0]
    dev.close()


@pytest.mark.gpu
def test_map_parity_through_the_seeding_retry_pass(monkeypatch):
    """First-pass seeding tables too small for most reads -> second launch at full size."""
    monkeypatch.setenv("GIRAFFE_B200_SEED_TABLES", "16,1")
    g = synth.make_variant_graph(length=100000, n_snp=160, n_ins=20, n_del=20, n_haps=8, seed=5)
    rs = synth.simulate_reads(g, 1500, length=150, sub_rate=0.01, seed=52)
    _run(g, rs)


@pytest.mark.gpu
def test_map_parity_across_host_chunks(monkeypatch):
    monkeypatch.setenv("GIRAFFE_B200_MAP_CHUNK", "200")
    g = synth.make_variant_graph(length=100000, n_snp=160, n_ins=20, n_del=20, n_haps=8, seed=5)
    rs = synth.simulate_reads(g, 1501, length=150, sub_rate=0.02, seed=54)
    _run(g, rs)


@pytest.mark.gpu
def test_map_parity_with_read_coverage_filter_active():
    """max_unique_min below the minimizer count: the max-min||num-bp-per-min stage consults the
    read-coverage vector (find_seeds :4312-4355) instead of being a pass-through."""
    g = synth.make_variant_graph(length=100000, n_snp=160, n_ins=20, n_del=20, n_haps=8, seed=5)
    rs = synth.simulate_reads(g, 1200, length=150, sub_rate=0.01, seed=55)
    p = capi.default_map_params()
    p.max_unique_min = 6
    p.num_bp_per_min = 50
    p.minimizer_coverage_flank = 10
    _run(g, rs, p)


@pytest.mark.gpu
def test_map_parity_tail_alignment_with_non_acgt_bases():
    """N bases inside aligned tails: they never match (DP query staging masks them)."""
    g = synth.make_variant_graph(length=100000, n_snp=160, n_ins=20, n_del=20, n_haps=8, seed=21)
    rs = synth.simulate_reads(g, 1200, length=200, sub_rate=0.02, ins_rate=0.01, del_rate=0.01, seed=56)
    rng = np.random.default_rng(4)
    for i in rng.integers(0, rs.n, size=600):
        rs.reads[i, rng.integers(0, rs.length, size=3)] = ord("N")
    _run(g, rs)


def _run_scored(g, rs, scores):
    index = g.build_index()
    dev = capi.Device(index, scores=scores)
    got = H.gpu_map(dev, rs.reads, rs.quals)
    plan = dev.plan_stats()
    want = H.oracle_map(index, rs.reads, rs.quals, scores=scores, threads=8)
    bad = H.compare_alignments(got, want, rs.n)
    dev.close()
    assert not bad, f"{len(bad)} of {rs.n} reads differ; first: read {bad[0][0]}\n got={bad[0][1]}\nwant={bad[0][2]}"
    return plan, want


@pytest.mark.gpu
def test_map_parity_with_the_tile_kernels_switched_off(monkeypatch):
    """GIRAFFE_B200_TILES=0: every tail DP runs the int32 column sweep inside the align kernels (the path a tile the
    int16 kernel cannot take falls back to); same records as with the tiles."""
    monkeypatch.setenv("GIRAFFE_B200_TILES", "0")
    g = synth.make_variant_graph(length=200000, n_snp=320, n_ins=40, n_del=40, n_haps=8, seed=2)
    rs = synth.simulate_reads(g, 2000, length=250, sub_rate=0.03, ins_rate=0.01, del_rate=0.01, seed=58)
    plan, want = _run_scored(g, rs, None)
    assert want[4]["tail_dps"] > 1000 and plan["cells"] == 0 and plan["tails"] == 0


def _reads_with_one_indel(g, n, lengths, dist, seed):
    """n reads of lengths[0] .. lengths[1] bp copied from the haplotypes, each with one 1-3 bp insertion or deletion
    dist[0] .. dist[1] bases from its left or right end, half of them reverse complemented."""
    rng = np.random.default_rng(seed)
    reads = []
    for _ in range(n):
        hs = g.hap_seq[int(rng.integers(0, len(g.hap_seq)))]
        L = int(rng.integers(lengths[0], lengths[1] + 1))
        s = int(rng.integers(0, len(hs) - L - 8))
        seq = hs[s: s + L + 8]
        d = int(rng.integers(dist[0], dist[1] + 1))
        at = d if rng.random() < 0.5 else L - d
        k = int(rng.integers(1, 4))
        if rng.random() < 0.5:
            seq = np.concatenate([seq[:at], synth.BASES[rng.integers(0, 4, size=k)], seq[at:]])
        else:
            seq = np.concatenate([seq[:at], seq[at + k:]])
        seq = seq[:L]
        reads.append(bytes(synth.revcomp_bytes(seq) if rng.random() < 0.5 else seq))
    return reads, [bytes([30] * len(r)) for r in reads]


def _run_tiles_on_and_off(monkeypatch, index, reads, quals, params):
    """The records with the tile kernels and with GIRAFFE_B200_TILES=0 both equal the oracle's; plan stats of the
    tiled run."""
    want = H.oracle_map(index, reads, quals, params, threads=8)
    plan = None
    for tiles in ("1", "0"):
        monkeypatch.setenv("GIRAFFE_B200_TILES", tiles)
        dev = capi.Device(index)
        got = H.gpu_map(dev, reads, quals, params)
        if tiles == "1":
            plan = dev.plan_stats()
        dev.close()
        bad = H.compare_alignments(got, want, len(reads))
        assert not bad, f"tiles={tiles}: {len(bad)} of {len(reads)} reads differ; first: read {bad[0][0]}\n got={bad[0][1]}\nwant={bad[0][2]}"
    return plan, want


@pytest.mark.gpu
def test_map_parity_with_tails_longer_than_a_tile_path(monkeypatch):
    """2-bp nodes and 300-400 bp reads with an indel 100-150 bases from one end: the far tail's path has more mappings
    than a tile's result holds (96).  With the read's caps raised to 512 mappings / 1024 edits such a tail is aligned
    in place, and the records are the same with and without the tile kernels.  Chunks of 128 reads keep the
    extensions of every read within the large-stride extension pool (n_reads / 128 + 256 work items per chunk): nearly
    every read here outgrows the regular 384-node extension stride."""
    monkeypatch.setenv("GIRAFFE_B200_MAP_CHUNK", "128")
    g = synth.make_variant_graph(length=60000, n_snp=100, n_ins=12, n_del=12, n_haps=8, seed=6, max_node=2)
    reads, quals = _reads_with_one_indel(g, 600, (300, 400), (100, 150), seed=61)
    p = capi.default_map_params()
    p.mapping_cap_per_read = 512
    p.edit_cap_per_read = 1024
    plan, want = _run_tiles_on_and_off(monkeypatch, g.build_index(), reads, quals, p)
    assert want[4]["tail_dps"] > 500 and plan["cells"] > 0
    assert (want[0]["n_mappings"] > 96).sum() > 300


@pytest.mark.gpu
def test_map_parity_long_reads_with_long_tails(monkeypatch):
    """400-512 bp reads with an indel 40-80 bases from either end on 32-bp nodes: the extension on the short side has a
    tail of at least 320 bases (the 12- and 16-row tile classes when tail_plan plans it; left tails through the
    reverse-complement translation, GB_TILE_LEFT)."""
    g = synth.make_variant_graph(length=200000, n_snp=320, n_ins=40, n_del=40, n_haps=8, seed=2)
    reads, quals = _reads_with_one_indel(g, 1000, (400, 512), (40, 80), seed=62)
    plan, want = _run_tiles_on_and_off(monkeypatch, g.build_index(), reads, quals, None)
    assert want[4]["tail_dps"] > 500 and plan["tails"] > 500 and plan["cells"] > 0


@pytest.mark.gpu
def test_map_parity_with_scaled_scores_on_tiles_and_sweeps():
    """Scoring parameters x20: tile_scores_fit_int16 accepts the short tails and rejects the long ones, so one batch mixes
    int16 tiles with int32 sweeps under non-default scores; the records still equal the oracle's under the same scores."""
    g = synth.make_variant_graph(length=200000, n_snp=320, n_ins=40, n_del=40, n_haps=8, seed=2)
    rs = synth.simulate_reads(g, 2000, length=250, sub_rate=0.03, ins_rate=0.01, del_rate=0.01, seed=59)
    plan, want = _run_scored(g, rs, capi.Scores(20, 80, 120, 20, 100))
    assert want[4]["tail_dps"] > 1000 and plan["cells"] > 0
