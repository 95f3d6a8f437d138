"""gb_map_paired_job_device: the paired job (fragment-length training, map_paired with the learned distribution, the
ambiguous-pair buffer) on reads already in HBM.  Both jobs train through the same window step, so the training rule is
checked against the oracle job (here and in test_fragment_distribution.py); here the device job must also reproduce the
host job gb_map_paired_job byte for byte: records, both pools up to the used counts, status, pair routes and the
distribution afterwards.  The CPU tests rehearse the driver's window cut and pool order with a host-side model."""
import ctypes as C
import os

import numpy as np
import pytest

import helpers as H
from vg_b200 import capi, synth


# ---- CPU: a model of the driver's arithmetic -------------------------------------------------------------------------------
def sequential_window(elig, lengths, budget):
    """The host job's loop over one window: pairs in order until the sample is full."""
    consumed, kept, buffered = 0, [], []
    for i, e in enumerate(elig):
        if len(kept) == budget:
            break
        consumed += 1
        (kept if e else buffered).append(i)
    return consumed, [lengths[i] for i in kept], kept, buffered


def scan_window(elig, lengths, budget):
    """train_cut_kernel's rule: one inclusive scan over eligibility; pair i is consumed while fewer than `budget` eligible
    pairs precede it; a non-eligible consumed pair goes to buffer slot i - (eligible pairs before it)."""
    elig = np.asarray(elig, dtype=np.uint64)
    incl = np.cumsum(elig)
    before = incl - elig
    consumed_mask = before < budget
    cut = len(elig) if incl[-1] < budget else int(np.nonzero((elig == 1) & (incl == budget))[0][0]) + 1
    out_len = [None] * int(min(incl[-1], budget))
    buffered = {}
    for i in np.nonzero(consumed_mask)[0]:
        if elig[i]:
            out_len[int(before[i])] = lengths[i]
        else:
            buffered[int(i - before[i])] = int(i)
    keep = [int(i) for i in np.nonzero(consumed_mask & (elig == 1))[0]]
    return cut, out_len, keep, [buffered[k] for k in range(len(buffered))]


def pool_order_model(routes, n_maps):
    """Where the job appends each read's mappings: training pairs window by window in input order, then the remaining
    pairs, then the buffered pairs in buffer order.  Returns mapping_off per read and the total."""
    n_pairs = len(routes)
    off, total = [0] * (2 * n_pairs), 0
    training_end = max((i + 1 for i, r in enumerate(routes) if r != capi.GB_PAIR_PAIRED), default=0)
    order = [p for p in range(training_end) if routes[p] == capi.GB_PAIR_TRAINING]
    order += list(range(training_end, n_pairs))
    order += [p for p in range(training_end) if routes[p] == capi.GB_PAIR_BUFFERED]
    for p in order:
        for r in (0, 1):
            off[2 * p + r] = total
            total += n_maps[2 * p + r]
    return off, total


def append_model(keep_pairs, n_maps, base):
    """record_append's sizes -> exclusive scan over n + 1 items -> offsets (the last one the total)."""
    sizes = [n_maps[i] if (i >> 1) in keep_pairs else 0 for i in range(len(n_maps))] + [0]
    scan = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    return [base + int(scan[i]) for i in range(len(n_maps)) if (i >> 1) in keep_pairs], base + int(scan[-1])


@pytest.mark.parametrize("seed", range(12))
def test_window_cut_model_equals_the_sequential_loop(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 300))
    elig = (rng.random(n) < rng.random()).astype(int).tolist()
    lengths = rng.integers(-1, 2000, n).tolist()
    for budget in (1, 2, int(rng.integers(1, n + 2)), n, n + 5):
        a, b = sequential_window(elig, lengths, budget), scan_window(elig, lengths, budget)
        assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2] and a[3] == b[3]


@pytest.mark.parametrize("seed", range(6))
def test_append_offsets_follow_the_host_pool_order(seed):
    """Appending window by window (kept pairs only), then the remaining block, then the buffer, with the running totals as
    bases, gives the host job's pool order on synthetic record sizes."""
    rng = np.random.default_rng(100 + seed)
    n_pairs, window, budget = int(rng.integers(20, 200)), int(rng.integers(1, 40)), int(rng.integers(1, 60))
    elig = (rng.random(n_pairs) < 0.7).astype(int).tolist()
    n_maps = rng.integers(0, 9, 2 * n_pairs).tolist()
    # the device driver, window by window
    off_dev, total, nxt, buffered, left = [0] * (2 * n_pairs), 0, 0, [], budget
    routes = [capi.GB_PAIR_PAIRED] * n_pairs
    while left > 0 and nxt < n_pairs:
        wp = min(window, n_pairs - nxt)
        cut, lens, keep, buf = scan_window(elig[nxt:nxt + wp], [0] * wp, left)
        sub = n_maps[2 * nxt: 2 * (nxt + wp)]
        offs, total = append_model(set(keep), sub, total)
        i = 0
        for p in keep:
            for r in (0, 1):
                off_dev[2 * (nxt + p) + r] = offs[i]; i += 1
            routes[nxt + p] = capi.GB_PAIR_TRAINING
        for p in buf:
            routes[nxt + p] = capi.GB_PAIR_BUFFERED
        buffered += [nxt + p for p in buf]
        left -= len(lens); nxt += cut
    for block in (list(range(nxt, n_pairs)), buffered):
        sub = [n_maps[2 * p + r] for p in block for r in (0, 1)]
        offs, total = append_model(set(range(len(block))), sub, total)
        for i, p in enumerate(block):
            off_dev[2 * p], off_dev[2 * p + 1] = offs[2 * i], offs[2 * i + 1]
    want_off, want_total = pool_order_model(routes, n_maps)
    assert total == want_total
    assert off_dev == want_off


# ---- GPU ------------------------------------------------------------------------------------------------------------------
def _job_inputs(n_pairs, seed):
    g = synth.make_variant_graph(length=150000, n_snp=240, n_ins=30, n_del=30, n_haps=8, seed=12)
    rs = synth.simulate_pairs(g, n_pairs, frag_mean=380, frag_sd=45, sub_rate=0.004, seed=seed)
    rng = np.random.default_rng(seed)
    for i in rng.integers(0, rs.n, size=n_pairs // 8):
        m = rng.random(rs.length) < 0.06
        rs.reads[i, m] = synth.BASES[rng.integers(0, 4, size=int(m.sum()))]
    for i in rng.integers(0, rs.n, size=n_pairs // 40):
        rs.reads[i] = synth.BASES[rng.integers(0, 4, size=rs.length)]
    return g, rs


@pytest.fixture(scope="module")
def graph():
    g = synth.make_variant_graph(length=150000, n_snp=240, n_ins=30, n_del=30, n_haps=8, seed=12)
    index = g.build_index()
    yield g, index


@pytest.fixture(scope="module")
def dev(graph):
    d = capi.Device(graph[1])
    yield d
    d.close()


def learn_params():
    p = H.default_map_params()
    p.fragment_mean = 0.0; p.fragment_stdev = 0.0
    return p


def host_job(dev, reads, quals, f, p, window=0):
    return host_job_on(dev, H.pack_reads(list(reads), None if quals is None else list(quals)), f, p, window)


def host_job_on(dev, bufs, f, p, window=0):
    """gb_map_paired_job on (reads, quals, read_off) in host memory."""
    aln, maps, edits, status, route = dev.map_paired_job(*bufs, f, p, training_window=window)
    nm, ne = dev.last_used
    return aln, maps[:nm], edits[:ne], status, route


class DeviceReads:
    """Reads uploaded once: after `prefix` bytes, with `gap` bytes between reads (offsets int64)."""

    def __init__(self, reads, quals=None, prefix=0, gap=0):
        import torch
        reads = [bytes(r) for r in reads]
        quals = None if quals is None else [bytes(q) for q in quals]
        starts = list(prefix + np.cumsum([0] + [len(x) + gap for x in reads[:-1]])) if reads else []
        off = [int(s) for s in starts] + [int(starts[-1]) + len(reads[-1]) if reads else prefix]
        rb = bytearray(b"\x5a" * (off[-1] + 1)); qb = bytearray(len(rb))
        for s, r in zip(starts, reads):
            rb[s:s + len(r)] = r
        if quals is not None:
            for s, q in zip(starts, quals):
                qb[s:s + len(q)] = q
        self.n = len(reads)
        self.max_len = max((len(r) for r in reads), default=0)
        # the same buffers in host memory, for the host job
        self.host = (np.frombuffer(bytes(rb), np.uint8), None if quals is None else np.frombuffer(bytes(qb), np.uint8), np.array(off, np.uint64))
        self.reads = torch.frombuffer(rb, dtype=torch.uint8).cuda()
        self.quals = None if quals is None else torch.frombuffer(qb, dtype=torch.uint8).cuda()
        self.off = torch.tensor(off, dtype=torch.int64).cuda()


def device_job(dev, dr, f, p, window=0, route=True, map_cap=None, edit_cap=None, max_read_len=None):
    """Returns rc and (aln, maps[:used], edits[:used], status, route) as numpy, plus the sentinel tails of the pools."""
    import torch
    n = dr.n
    map_cap = n * p.mapping_cap_per_read if map_cap is None else map_cap
    edit_cap = n * p.edit_cap_per_read if edit_cap is None else edit_cap
    SENT = 64
    t_aln = torch.zeros(max(n, 1) * 32, dtype=torch.uint8, device="cuda")
    t_maps = torch.full(((map_cap + SENT) * 8,), 0xA5, dtype=torch.uint8, device="cuda")
    t_edits = torch.full(((edit_cap + SENT) * 4,), 0xA5, dtype=torch.uint8, device="cuda")
    t_status = torch.zeros(max(n, 1), dtype=torch.uint8, device="cuda")
    t_route = torch.full((max(n // 2, 1),), 0xEE, dtype=torch.uint8, device="cuda")
    vp = lambda t: None if t is None else t.data_ptr()
    torch.cuda.synchronize()
    rc, nm, ne = dev.map_paired_job_device(f, n, vp(dr.reads), vp(dr.quals), vp(dr.off), dr.max_len if max_read_len is None else max_read_len,
                                           vp(t_aln), vp(t_maps), map_cap, vp(t_edits), edit_cap, vp(t_status),
                                           vp(t_route) if route else None, params=p, training_window=window)
    maps = t_maps.cpu().numpy(); edits = t_edits.cpu().numpy()
    out = (t_aln.cpu().numpy()[: n * 32].view(capi.alignment_dt), maps[: nm * 8].view(capi.mapping_dt), edits[: ne * 4].view(np.uint32),
           t_status.cpu().numpy()[:n], t_route.cpu().numpy()[: n // 2])
    tails = (maps[map_cap * 8:], edits[edit_cap * 4:])
    return rc, out, tails


def assert_same(got, want, routes=True):
    assert got[0].tobytes() == want[0].tobytes(), "records differ"
    assert got[1].tobytes() == want[1].tobytes(), "mapping pools differ"
    assert got[2].tobytes() == want[2].tobytes(), "edit pools differ"
    assert (got[3] == want[3]).all(), "status differs"
    if routes:
        assert (got[4] == want[4]).all(), "pair routes differ"


def fstate(f):
    return f.mean(), f.std_dev(), f.curr_sample_size(), f.is_finalized()


def assert_oracle_job(got, f, index, reads, quals, max_n, freq):
    """Routes, (mean, stdev, sample size) and records of the oracle job on the same reads."""
    orc = H.oracle_map_paired_job(index, reads, quals, learn_params(), max_n, freq, 0.95, threads=8)
    assert (got[4] == orc[4]).all(), "pair routes differ from the oracle job"
    assert (f.mean(), f.std_dev(), f.curr_sample_size()) == orc[5]
    full = (got[0], np.concatenate([got[1], np.zeros(1, capi.mapping_dt)]), np.concatenate([got[2], np.zeros(1, np.uint32)]), got[3])
    bad = H.compare_alignments(full, orc, len(got[0]))
    assert not bad, f"{len(bad)} reads differ from the oracle job; first: {bad[0]}"


def both_jobs(dev, reads, quals, max_n, freq, window, p=None, **kw):
    p = p or learn_params()
    fh, fd = capi.FragmentDistribution(max_n, freq, 0.95), capi.FragmentDistribution(max_n, freq, 0.95)
    want = host_job(dev, reads, quals, fh, p, window)
    rc, got, _ = device_job(dev, DeviceReads(reads, quals, **kw), fd, p, window)
    assert rc == capi.GB_OK, capi.load_library().gb_last_error()
    return got, want, fh, fd


@pytest.mark.gpu
@pytest.mark.parametrize("n_pairs,max_n,freq,window", [(2500, 1000, 1000, 0), (1500, 300, 100, 128), (400, 1000, 1000, 64),
                                                       (600, 150, 50, 1), (600, 150, 50, 5000)])
def test_equals_host_job(dev, graph, n_pairs, max_n, freq, window):
    g, index = graph
    _, rs = _job_inputs(n_pairs, seed=70 + n_pairs)
    got, want, fh, fd = both_jobs(dev, rs.reads, rs.quals, max_n, freq, window)
    assert_same(got, want)
    assert fstate(fd) == fstate(fh) and fd.is_finalized()
    assert_oracle_job(got, fd, index, rs.reads, rs.quals, max_n, freq)


@pytest.mark.gpu
def test_window_independence(dev):
    _, rs = _job_inputs(700, seed=91)
    outs = []
    for window in (1, 7, 2048, 700):
        f = capi.FragmentDistribution(200, 50, 0.95)
        rc, got, _ = device_job(dev, DeviceReads(rs.reads, rs.quals), f, learn_params(), window)
        assert rc == capi.GB_OK
        outs.append((got, fstate(f)))
        fh = capi.FragmentDistribution(200, 50, 0.95)
        outs.append((host_job(dev, rs.reads, rs.quals, fh, learn_params(), window), fstate(fh)))
    for got, st in outs[1:]:
        assert_same(got, outs[0][0])
        assert st == outs[0][1]


@pytest.mark.gpu
def test_already_finalized_maps_everything_paired(dev):
    import torch
    _, rs = _job_inputs(500, seed=5)
    f = capi.FragmentDistribution(1000, 1000, 0.95)
    f.force_parameters(385.0, 47.0)
    dr = DeviceReads(rs.reads, rs.quals)
    rc, got, _ = device_job(dev, dr, f, learn_params())
    assert rc == capi.GB_OK and (got[4] == capi.GB_PAIR_PAIRED).all()
    p = H.default_map_params(); p.fragment_mean = 385.0; p.fragment_stdev = 47.0
    n = rs.n
    d_aln = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
    d_maps = torch.zeros(n * p.mapping_cap_per_read * 8, dtype=torch.uint8, device="cuda")
    d_edits = torch.zeros(n * p.edit_cap_per_read, dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_tot = torch.zeros(2, dtype=torch.int64, device="cuda")
    vp = lambda t: C.c_void_p(t.data_ptr())
    lib = capi.load_library()
    assert lib.gb_map_batch_device(dev.handle, C.byref(p), 1, n, vp(dr.reads), vp(dr.quals), vp(dr.off), dr.max_len, vp(d_aln), vp(d_maps),
                                   n * p.mapping_cap_per_read, vp(d_edits), n * p.edit_cap_per_read, vp(d_status), vp(d_tot)) == capi.GB_OK
    lib.gb_device_synchronize(dev.handle)
    tot = d_tot.cpu().numpy()
    direct = (d_aln.cpu().numpy().view(capi.alignment_dt), d_maps.cpu().numpy().view(capi.mapping_dt)[: tot[0]],
              d_edits.cpu().numpy().view(np.uint32)[: tot[1]], d_status.cpu().numpy())
    assert_same(got, direct, routes=False)
    assert not H.compare_alignments(got[:4], direct, n, mapq_tol=0)


@pytest.mark.gpu
def test_input_ending_before_the_sample_fills_and_the_fallback_limit(dev):
    # 0 +- 1: every pair takes the single-end fallback, flagged PAIRED
    _, rs = _job_inputs(300, seed=33)
    got, want, fh, fd = both_jobs(dev, rs.reads, rs.quals, 1000, 1000, 0)
    assert_same(got, want)
    assert fstate(fd) == fstate(fh)
    assert ((got[0]["flags"] & capi.GB_ALN_PAIRED) != 0).all()
    # read-1 lengths straddling the limit of a forced distribution: refused exactly when the host job refuses
    g = synth.make_variant_graph(length=150000, n_snp=240, n_ins=30, n_del=30, n_haps=8, seed=12)
    long = synth.simulate_pairs(g, 200, length=220, frag_mean=500, frag_sd=40, seed=4)
    p = learn_params()
    for lens1 in ([150] * 200, [150] * 100 + [220] * 100, [220] * 200):
        reads = [bytes(long.reads[i][: lens1[i // 2]] if i % 2 == 0 else long.reads[i][:150]) for i in range(long.n)]
        quals = [bytes(long.quals[i][: len(reads[i])]) for i in range(long.n)]
        fh, fd = capi.FragmentDistribution(), capi.FragmentDistribution()
        fh.force_parameters(170.0, 25.0); fd.force_parameters(170.0, 25.0)        # fragment limit 220: read 1 of 220 bp fails
        try:
            want = host_job(dev, reads, quals, fh, p); rc_h = capi.GB_OK
        except capi.GbError as e:
            rc_h = e.code
        rc_d, got, _ = device_job(dev, DeviceReads(reads, quals), fd, p)
        assert rc_d == rc_h
        if rc_h == capi.GB_OK:
            assert_same(got, want)


@pytest.mark.gpu
def test_unreachable_mates_register_minus_one(dev, graph):
    """Mate 2 replaced by a forward-strand read from elsewhere: both ends map uniquely at full score, but the flipped mate 2
    lies on the other strand, so the distance is unreachable (-1), which is below max_fragment_length and is registered.
    Both jobs train through one window step, so the oracle job is what checks that rule here."""
    g, index = graph
    rs = synth.simulate_pairs(g, 300, sub_rate=0.0, seed=17)
    other = synth.simulate_pairs(g, 300, sub_rate=0.0, seed=18)
    reads = [bytes(rs.reads[i]) if i % 2 == 0 or (i // 2) % 3 else bytes(other.reads[i - 1]) for i in range(rs.n)]
    got, want, fh, fd = both_jobs(dev, reads, list(rs.quals), 100, 100, 0)
    assert_same(got, want)
    assert fstate(fd) == fstate(fh) and fd.curr_sample_size() == 100
    assert_oracle_job(want, fh, index, reads, list(rs.quals), 100, 100)
    assert_oracle_job(got, fd, index, reads, list(rs.quals), 100, 100)


@pytest.mark.gpu
def test_pool_overflow_is_redone(dev, graph):
    _, rs = _job_inputs(600, seed=44)
    f0 = capi.FragmentDistribution(200, 100, 0.95)
    rc, want, _ = device_job(dev, DeviceReads(rs.reads, rs.quals), f0, learn_params())
    assert rc == capi.GB_OK
    os.environ["GIRAFFE_B200_POOL_SCALE"] = "0.01"
    try:
        small = capi.Device(graph[1])
    finally:
        del os.environ["GIRAFFE_B200_POOL_SCALE"]
    f1 = capi.FragmentDistribution(200, 100, 0.95)
    rc, got, _ = device_job(small, DeviceReads(rs.reads, rs.quals), f1, learn_params())
    assert rc == capi.GB_OK
    assert_same(got, want)
    assert fstate(f1) == fstate(f0)
    small.close()


@pytest.mark.gpu
def test_capacity(dev):
    _, rs = _job_inputs(400, seed=12)
    p = learn_params()
    f = capi.FragmentDistribution(150, 50, 0.95)
    rc, full, _ = device_job(dev, DeviceReads(rs.reads, rs.quals), f, p)
    assert rc == capi.GB_OK
    nm, ne = len(full[1]), len(full[2])
    f = capi.FragmentDistribution(150, 50, 0.95)
    rc, got, tails = device_job(dev, DeviceReads(rs.reads, rs.quals), f, p, map_cap=nm, edit_cap=ne)
    assert rc == capi.GB_OK
    assert_same(got, full)
    assert (tails[0] == 0xA5).all() and (tails[1] == 0xA5).all()
    for mc, ec in ((nm - 1, ne), (nm, ne - 1)):
        f = capi.FragmentDistribution(150, 50, 0.95)
        rc, _, tails = device_job(dev, DeviceReads(rs.reads, rs.quals), f, p, map_cap=mc, edit_cap=ec)
        assert rc == capi.GB_ERR_CAPACITY
        assert (tails[0] == 0xA5).all() and (tails[1] == 0xA5).all()


@pytest.mark.gpu
def test_refusals_and_optional_arrays(dev):
    import torch
    _, rs = _job_inputs(100, seed=2)
    dr = DeviceReads(rs.reads, rs.quals)
    lib = capi.load_library()
    f = capi.FragmentDistribution()
    t = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    x = t.data_ptr()
    p = learn_params()
    p2 = learn_params(); p2.max_multimaps = 2
    cases = [dict(reads=None), dict(n=dr.n - 1), dict(params=p2), dict(max_len=513), dict(aln=None), dict(status=None)]
    for c in cases:
        before = lib.gb_launch_count(dev.handle)
        rc, _, _ = dev.map_paired_job_device(f, c.get("n", dr.n), c.get("reads", dr.reads.data_ptr()), None, dr.off.data_ptr(), c.get("max_len", 150),
                                             c.get("aln", x), x, 10, x, 10, c.get("status", x), None, params=c.get("params", p))
        assert rc == capi.GB_ERR_ARG, c
        assert lib.gb_launch_count(dev.handle) == before
    rc, _, _ = dev.map_paired_job_device(f, 0, None, None, None, 150, None, None, 0, None, 0, None, None, params=p)
    assert rc == capi.GB_OK and not f.is_finalized() and f.curr_sample_size() == 0
    # no qualities, no routes: the host job's records
    fh, fd = capi.FragmentDistribution(150, 50, 0.95), capi.FragmentDistribution(150, 50, 0.95)
    want = host_job(dev, rs.reads, None, fh, p)
    rc, got, _ = device_job(dev, DeviceReads(rs.reads, None), fd, p, route=False)
    assert rc == capi.GB_OK
    assert_same(got, want, routes=False)
    assert fstate(fd) == fstate(fh)


@pytest.mark.gpu
def test_offsets_with_a_base_and_gaps(dev):
    """Offsets that start after a prefix give the records of zero-based ones, in both jobs (the host job uploads each
    training window and rebases its offsets).  Bytes between reads belong to the read before them (read r is
    [off[r], off[r + 1])), so reads with gaps are compared with the host job on those longer reads."""
    _, rs = _job_inputs(500, seed=8)
    outs = []
    for prefix in (0, 1000, 37):
        f = capi.FragmentDistribution(150, 50, 0.95)
        dr = DeviceReads(rs.reads, rs.quals, prefix=prefix)
        rc, got, _ = device_job(dev, dr, f, learn_params(), 64)
        assert rc == capi.GB_OK
        outs.append((got, fstate(f)))
        fh = capi.FragmentDistribution(150, 50, 0.95)
        outs.append((host_job_on(dev, dr.host, fh, learn_params(), 64), fstate(fh)))
    for got, st in outs[1:]:
        assert_same(got, outs[0][0])
        assert st == outs[0][1]
    gap = 13
    reads = [bytes(r) + (b"Z" * gap if i < rs.n - 1 else b"") for i, r in enumerate(rs.reads)]
    quals = [bytes(q) + (b"\0" * gap if i < rs.n - 1 else b"") for i, q in enumerate(rs.quals)]      # DeviceReads' filler bytes
    fh, fd = capi.FragmentDistribution(150, 50, 0.95), capi.FragmentDistribution(150, 50, 0.95)
    want = host_job(dev, reads, quals, fh, learn_params(), 64)
    dr = DeviceReads(rs.reads, rs.quals, prefix=37, gap=gap)
    rc, got, _ = device_job(dev, dr, fd, learn_params(), 64, max_read_len=150 + gap)
    assert rc == capi.GB_OK
    assert_same(got, want)
    assert fstate(fd) == fstate(fh)
    fb = capi.FragmentDistribution(150, 50, 0.95)
    assert_same(host_job_on(dev, dr.host, fb, learn_params(), 64), want)
    assert fstate(fb) == fstate(fh)
    # max_read_len below the longest read is refused
    rc, _, _ = device_job(dev, dr, capi.FragmentDistribution(150, 50, 0.95), learn_params(), 64, max_read_len=150)
    assert rc == capi.GB_ERR_ARG



@pytest.mark.gpu
def test_streaming_two_calls(dev):
    _, rs = _job_inputs(1200, seed=21)
    fh, fd = capi.FragmentDistribution(300, 100, 0.95), capi.FragmentDistribution(300, 100, 0.95)
    for lo, hi in ((0, 800), (800, 1200)):
        r, q = rs.reads[2 * lo: 2 * hi], rs.quals[2 * lo: 2 * hi]
        want = host_job(dev, r, q, fh, learn_params())
        rc, got, _ = device_job(dev, DeviceReads(r, q), fd, learn_params())
        assert rc == capi.GB_OK
        assert_same(got, want)
        assert fstate(fd) == fstate(fh)
    assert (got[4] == capi.GB_PAIR_PAIRED).all()


def fastq_of(reads, quals, mate):
    return b"".join(b"@p%d/%d extra\n" % (i, mate) + bytes(r) + b"\n+\n" + bytes(q + 33) + b"\n" for i, (r, q) in enumerate(zip(reads, quals)))


@pytest.mark.gpu
def test_end_to_end_fastq_gz_to_gam_with_a_learned_distribution(dev, graph):
    import torch
    g, index = graph
    rs = synth.simulate_pairs(g, 1500, frag_mean=380, frag_sd=45, sub_rate=0.002, seed=8, indel_rate=0.0002)
    rng = np.random.default_rng(2)
    quals = rng.choice(np.array([2, 12, 23, 37], np.uint8), size=rs.reads.shape, p=[0.02, 0.08, 0.2, 0.7])
    r1, r2 = (fastq_of(rs.reads[m::2], quals[m::2], m + 1) for m in (0, 1))
    z1, z2 = capi.bgzf_compress(r1, 6), capi.bgzf_compress(r2, 6)
    up = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    t1, _ = dev.bgzf_decompress_device(up(z1))
    t2, _ = dev.bgzf_decompress_device(up(z2))
    pr = dev.fastq_parse_device([t1, t2])
    n = pr["n_reads"]
    assert n == rs.n
    p = learn_params()
    fd = capi.FragmentDistribution(500, 100, 0.95)
    d_aln = torch.zeros((n, 32), dtype=torch.uint8, device="cuda")
    d_maps = torch.zeros((n * p.mapping_cap_per_read, 8), dtype=torch.uint8, device="cuda")
    d_edits = torch.zeros(n * p.edit_cap_per_read, dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.uint8, device="cuda")
    rc, nm, ne = dev.map_paired_job_device(fd, n, pr["reads"].data_ptr(), pr["quals"].data_ptr(), pr["read_off"].data_ptr(), pr["max_read_len"],
                                           d_aln.data_ptr(), d_maps.data_ptr(), n * p.mapping_cap_per_read, d_edits.data_ptr(),
                                           n * p.edit_cap_per_read, d_status.data_ptr(), None, params=p)
    assert rc == capi.GB_OK
    gam = dev.emit_device("gam", d_aln, d_maps[:nm], d_edits[:ne], pr["reads"], pr["read_off"], pr["quals"], pr["names"], pr["name_off"])
    z = dev.bgzf_compress_device(gam).cpu().numpy().tobytes()
    import gzip
    inflated = gzip.decompress(z)
    # host: parse on the host, the host job, the host emitter
    rbuf, qbuf, roff = H.pack_reads(list(rs.reads), list(quals))
    fh = capi.FragmentDistribution(500, 100, 0.95)
    aln, maps, edits, _, _ = dev.map_paired_job(rbuf, qbuf, roff, fh, p)
    names = [b"p%d/%d" % (i // 2, i % 2 + 1) for i in range(n)]
    want = capi.emit_text("gam", index.view, aln, maps, edits, rbuf, qbuf, roff, names=[x.decode() for x in names])
    assert inflated == want
    assert fstate(fd) == fstate(fh) and fd.curr_sample_size() == 500
