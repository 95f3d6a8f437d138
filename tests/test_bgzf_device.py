"""gb_bgzf_compress_device: BGZF compressed on the GPU.  The container must be the one gb_bgzf_compress writes (same
block cuts, headers, BSIZE, CRC32, ISIZE and EOF block), the deflate payloads must pass a strict RFC 1951 parser written
here independently of zlib (zlib itself accepts some streams other inflaters refuse), the output must be deterministic
and independent of the input's alignment, and on config-2-like GAM and GAF it must compress within 10 % of zlib level 1."""
import ctypes as C
import gzip
import heapq
import struct
import zlib

import numpy as np
import pytest

import helpers as H
from test_gam import _bgzf_blocks, decode_alignment, read_stream
from vg_b200 import capi

BLOCK = 0xff00


# ---- a strict deflate parser (RFC 1951) --------------------------------------------------------------------------------
class DeflateError(Exception):
    pass


class _Bits:
    def __init__(self, data):
        self.v = int.from_bytes(data, "little")
        self.n = 8 * len(data)
        self.pos = 0

    def get(self, k):
        if self.pos + k > self.n:
            raise DeflateError("read past the end of the payload")
        x = (self.v >> self.pos) & ((1 << k) - 1)
        self.pos += k
        return x


def _code(lengths, what, allow_single=False):
    """Canonical decoding table {(length, code): symbol}; refuses over-subscribed and (unless allowed) incomplete codes."""
    used = [n for n in lengths if n]
    kraft = sum(1 << (15 - n) for n in used)
    if kraft > 1 << 15:
        raise DeflateError(f"{what}: over-subscribed code")
    if kraft < 1 << 15:
        single = allow_single and (len(used) == 0 or (len(used) == 1 and used[0] == 1))
        if not single:
            raise DeflateError(f"{what}: incomplete code {sorted(used)}")
    bl = [0] * 16
    for n in used:
        bl[n] += 1
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    table = {}
    for s, n in enumerate(lengths):
        if n:
            table[(n, nxt[n])] = s
            nxt[n] += 1
    return table


def _decode(bits, table):
    code = 0
    for n in range(1, 16):
        code = (code << 1) | bits.get(1)
        s = table.get((n, code))
        if s is not None:
            return s
    raise DeflateError("no such code")


LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
         8193, 12289, 16385, 24577]
DEXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


def strict_inflate(payload, stats=None):
    """Inflate one raw deflate stream, refusing anything outside RFC 1951's strict reading.  stats (dict) collects the
    block types, the longest code lengths, the largest distance and, per dynamic block, its code lengths and the symbols
    it decoded ("trees")."""
    bits, out = _Bits(payload), bytearray()
    stats = {} if stats is None else stats
    stats.setdefault("btypes", []); stats.setdefault("max_len", 0); stats.setdefault("max_cl_len", 0); stats.setdefault("max_dist", 0)
    while True:
        final, btype = bits.get(1), bits.get(2)
        stats["btypes"].append(btype)
        if btype == 3:
            raise DeflateError("BTYPE 11")
        if btype == 0:
            bits.pos = (bits.pos + 7) & ~7
            ln, nln = bits.get(16), bits.get(16)
            if ln != nln ^ 0xffff:
                raise DeflateError("stored LEN / NLEN")
            for _ in range(ln):
                out.append(bits.get(8))
        else:
            if btype == 1:
                ll = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
                dl = [5] * 30
                lt, dt = _code(ll, "fixed litlen"), _code(dl + [5, 5], "fixed dist")
            else:
                hlit, hdist, hclen = bits.get(5) + 257, bits.get(5) + 1, bits.get(4) + 4
                if hlit > 286 or hdist > 30:
                    raise DeflateError(f"HLIT {hlit} / HDIST {hdist}")
                cl = [0] * 19
                for i in range(hclen):
                    cl[CL_ORDER[i]] = bits.get(3)
                stats["max_cl_len"] = max(stats["max_cl_len"], max(cl))
                ct = _code(cl, "code-length code")
                lens = []
                while len(lens) < hlit + hdist:
                    s = _decode(bits, ct)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        if not lens:
                            raise DeflateError("repeat with no previous length")
                        lens += [lens[-1]] * (3 + bits.get(2))
                    elif s == 17:
                        lens += [0] * (3 + bits.get(3))
                    else:
                        lens += [0] * (11 + bits.get(7))
                if len(lens) != hlit + hdist:
                    raise DeflateError("code lengths overrun HLIT + HDIST")
                ll, dl = lens[:hlit], lens[hlit:]
                if ll[256] == 0:
                    raise DeflateError("no end-of-block code")
                stats["max_len"] = max(stats["max_len"], max(lens))
                lt, dt = _code(ll, "litlen"), _code(dl, "dist", allow_single=True)
                stats.setdefault("trees", []).append({"ll": ll, "dl": dl, "lit": [0] * 286, "dist": [0] * 30})
            counts = stats["trees"][-1] if btype == 2 else {"lit": [0] * 286, "dist": [0] * 30}
            while True:
                s = _decode(bits, lt)
                if s < 286:
                    counts["lit"][s] += 1
                if s < 256:
                    out.append(s)
                    continue
                if s == 256:
                    break
                if s > 285:
                    raise DeflateError(f"litlen symbol {s}")
                length = LBASE[s - 257] + bits.get(LEXTRA[s - 257])
                if not 3 <= length <= 258:
                    raise DeflateError(f"length {length}")
                d = _decode(bits, dt)
                if d > 29:
                    raise DeflateError(f"distance code {d}")
                counts["dist"][d] += 1
                dist = DBASE[d] + bits.get(DEXTRA[d])
                if dist > min(32768, len(out)):
                    raise DeflateError(f"distance {dist} with {len(out)} bytes so far")
                stats["max_dist"] = max(stats["max_dist"], dist)
                for _ in range(length):
                    out.append(out[-dist])
        if final:
            return bytes(out)


def min_huffman_depth(counts):
    """The depth of the shallowest optimal (unlimited) prefix code for these counts: ties merge the shallower subtree
    first, so no Huffman code for them is shallower."""
    h = [(w, 0, i) for i, w in enumerate(counts) if w]
    heapq.heapify(h)
    k = len(h)
    while len(h) > 1:
        w1, d1, _ = heapq.heappop(h)
        w2, d2, _ = heapq.heappop(h)
        heapq.heappush(h, (w1 + w2, max(d1, d2) + 1, k)); k += 1
    return h[0][1] if h else 0


def test_strict_parser_reads_zlib():
    """The parser itself: zlib's own streams at several levels and strategies parse and decode to the input."""
    rng = np.random.default_rng(1)
    for data in (b"", b"a", bytes(rng.integers(0, 4, size=20000, dtype=np.uint8) + 65), bytes(range(256)) * 40,
                 bytes(rng.integers(0, 256, size=3000, dtype=np.uint8))):
        for level, strategy in ((1, zlib.Z_DEFAULT_STRATEGY), (9, zlib.Z_DEFAULT_STRATEGY), (6, zlib.Z_FIXED), (0, zlib.Z_DEFAULT_STRATEGY)):
            c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
            assert strict_inflate(c.compress(data) + c.flush()) == data
    with pytest.raises(DeflateError):
        strict_inflate(bytes([0b111]))                          # BTYPE 11


# ---- helpers -----------------------------------------------------------------------------------------------------------
def _members(raw):
    """[(offset, bsize)] of a BGZF stream."""
    i, out = 0, []
    while i < len(raw):
        bsize = struct.unpack("<H", raw[i + 16:i + 18])[0] + 1
        out.append((i, bsize)); i += bsize
    return out


def _zlib_level1_size(data):
    """zlib level 1 on the same 0xff00 cuts, with BGZF's 26 bytes per block and the 28-byte EOF block."""
    total = 28
    for at in range(0, len(data), BLOCK):
        c = zlib.compressobj(1, zlib.DEFLATED, -15)
        total += 26 + len(c.compress(data[at:at + BLOCK]) + c.flush())
    return total


def _check_container(raw, data, strict=True):
    """raw against gb_bgzf_compress on the same bytes: block by block, then whole-stream inflation.  Returns the strict
    parser's statistics over all members."""
    host = _bgzf_blocks(capi.bgzf_compress(data, 6))
    got = _bgzf_blocks(raw)
    assert len(got) == len(host) == (len(data) + BLOCK - 1) // BLOCK + 1
    assert raw[-28:] == capi.bgzf_compress(b"", 6)
    for (gh, gsize, gpay), (hh, _, hpay) in zip(got, host):
        assert gh == hh and len(gpay) == len(hpay) and gsize <= 0x10000
    assert b"".join(p for _, _, p in got) == data
    assert gzip.decompress(raw) == data
    rest, inflated = raw, b""
    while rest:
        d = zlib.decompressobj(31); inflated += d.decompress(rest); rest = d.unused_data
    assert inflated == data
    stats = {}
    if strict:
        for (off, bsize), (_, _, pay) in zip(_members(raw), got):
            assert strict_inflate(raw[off + 18:off + bsize - 8], stats) == pay
        assert stats["max_len"] <= 15 and stats["max_cl_len"] <= 7
    return stats


def _lib():
    return capi.load_library()


def test_null_handle_is_refused():
    used = C.c_uint64(7)
    buf = (C.c_uint8 * 64)()
    assert _lib().gb_bgzf_compress_device(None, C.cast(buf, C.c_void_p), 16, C.cast(buf, C.c_void_p), 64, C.byref(used)) == capi.GB_ERR_ARG
    assert used.value == 7


# ---- on the GPU --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    from vg_b200 import synth
    d = capi.Device(synth.make_tiny_graph().build_index(), 0)
    yield d
    d.close()


def _compress(dev, data):
    import torch
    t = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda() if data else torch.empty(0, dtype=torch.uint8, device="cuda")
    return dev.bgzf_compress_device(t).cpu().numpy().tobytes()


def _text(n, seed):
    """Compressible bytes: records of ACGT with repeated field names and numbers, like the emitters' output."""
    rng = np.random.default_rng(seed)
    parts, size = [], 0
    while size < n:
        seq = bytes(rng.integers(0, 4, size=int(rng.integers(40, 160)), dtype=np.uint8) + 65).translate(bytes.maketrans(b"ABCD", b"ACGT"))
        s = b"read%d\t%d\t+\t%s\tAS:i:%d\n" % (int(rng.integers(0, 10 ** 6)), len(seq), seq, int(rng.integers(0, 160)))
        parts.append(s); size += len(s)
    return b"".join(parts)[:n]


@pytest.mark.gpu
@pytest.mark.parametrize("size", [0, 1, 2, 3, BLOCK - 1, BLOCK, BLOCK + 1, 5 * BLOCK + 17])
def test_container_matches_the_host(dev, size):
    data = _text(size, size)
    raw = _compress(dev, data)
    _check_container(raw, data)
    if size >= BLOCK:
        assert len(raw) < len(data) / 2                        # text this redundant compresses


@pytest.mark.gpu
def test_random_bytes_are_stored(dev):
    data = bytes(np.random.default_rng(5).integers(0, 256, size=300000, dtype=np.uint8))
    raw = _compress(dev, data)
    _check_container(raw, data, strict=False)
    for off, bsize in _members(raw)[:-1]:
        assert raw[off + 18] & 7 == 1                          # BFINAL 1, BTYPE 00


def _skewed_lengths_block(seed=3, n_codes=16):
    """One full block whose parse has Fibonacci-skewed match lengths: copies of 3, 4, 5, ... bytes (the first length of
    each of the first n_codes length symbols) made 1597, 987, 610, ..., 2, 1 times between fresh bytes.  Every 3-gram of
    the fresh bytes is new, a copy's neighbours never extend it, and no copy crosses a 255-byte parse segment, so the
    greedy parse sees exactly those matches.  With the end-of-block code as the last 1 the litlen counts are
    Fibonacci-like and an optimal code for them is deeper than 15 bits: the encoder must limit the lengths."""
    fib = [1, 1]
    while len(fib) < n_codes + 1:
        fib.append(fib[-1] + fib[-2])
    first = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43][:n_codes]
    rng = np.random.default_rng(seed)
    copies = [ln for ln, c in zip(first, fib[1:][::-1]) for _ in range(c)]
    rng.shuffle(copies)
    rand = iter(rng.integers(0, 256, size=8 * BLOCK).tolist())
    b, fresh, seen, ci = bytearray(), [], set(), 0
    while len(b) < BLOCK:
        p = len(b)
        if ci < len(copies) and p >= 2 and fresh[p - 1]:
            L = copies[ci]
            if p + L <= BLOCK and p // 255 == (p + L - 1) // 255:
                for D in rng.integers(600, 3000, size=8).tolist():
                    s = p - D
                    if s < 0 or not all(fresh[s:s + L]):
                        continue
                    g0, g1 = (b[p - 2], b[p - 1], b[s]), (b[p - 1], b[s], b[s + 1])
                    if g0 in seen or g1 in seen:
                        continue
                    b += b[s:s + L]; fresh += [False] * L; seen.update((g0, g1)); ci += 1
                    break
                else:
                    L = 0
                if L:
                    continue
        v = next(rand)
        while p >= 2 and (b[p - 2], b[p - 1], v) in seen:
            v = next(rand)
        if p >= 2:
            seen.add((b[p - 2], b[p - 1], v))
        b.append(v); fresh.append(True)
    assert ci == len(copies)
    return bytes(b)


def _adversarial():
    rng = np.random.default_rng(9)
    periodic = b"".join((bytes(rng.integers(0, 256, size=p, dtype=np.uint8)) * (400 // p + 2))[:max(400, 2 * p)] for p in range(1, 301))
    far = []
    for back in (32768, 32769):
        a = bytearray(rng.integers(0, 64, size=40000, dtype=np.uint8) + 32)
        a[back:back + 300] = a[0:300]
        far.append((f"only repeat {back} back", bytes(a), back))
    cases = [("one byte repeated", b"a" * 100000, None), ("a single distinct symbol", b"\0" * 5000, None), ("single symbol, short", b"\0" * 5, None),
             ("periods 1..300", periodic, None), ("all 256 byte values", bytes(range(256)) * 200 + bytes(rng.permutation(256).astype(np.uint8)), None),
             ("Fibonacci-skewed match lengths", _skewed_lengths_block(), None),
             ("ACGT only", bytes(rng.integers(0, 4, size=150000, dtype=np.uint8)).translate(bytes.maketrans(bytes(range(4)), b"ACGT")), None)]
    return cases + far


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(9))
def test_adversarial_inputs_pass_the_strict_parser(dev, case):
    name, data, back = _adversarial()[case]
    raw = _compress(dev, data)
    stats = _check_container(raw, data)
    if len(data) >= 1000:                                      # a few bytes are cheaper stored
        assert 2 in stats["btypes"], f"{name}: no dynamic block"
    if back == 32768:
        assert stats["max_dist"] == 32768, f"{name}: the repeat 32768 back was not used"
    # back == 32769: the parser refuses any distance over 32768, so parsing is the check
    if name.startswith("Fibonacci"):
        (tree,) = stats["trees"]
        assert min_huffman_depth(tree["lit"]) > 15, "the input no longer needs the 15-bit limit"
        assert max(tree["ll"]) == 15                           # limited to exactly 15, and the stream still decodes


@pytest.mark.gpu
def test_deterministic_and_independent_of_alignment(dev):
    import torch
    data = _text(5 * BLOCK + 17, 3)
    first = _compress(dev, data)
    assert _compress(dev, data) == first
    src = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    for k in range(1, 16):
        buf = torch.zeros(len(data) + 32, dtype=torch.uint8, device="cuda")
        buf[k:k + len(data)] = src
        assert dev.bgzf_compress_device(buf[k:k + len(data)]).cpu().numpy().tobytes() == first, f"offset {k}"


@pytest.mark.gpu
def test_short_output_reports_the_size_and_writes_nothing(dev):
    import torch
    data = _text(3 * BLOCK + 5, 4)
    want = _compress(dev, data)
    src = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    lib, used = _lib(), C.c_uint64()
    for cap in (0, 27, len(want) - 1):
        out = torch.full((max(cap, 1),), 0xA5, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = lib.gb_bgzf_compress_device(dev.handle, C.c_void_p(src.data_ptr()), len(data), C.c_void_p(out.data_ptr()), cap, C.byref(used))
        assert rc == capi.GB_ERR_CAPACITY and used.value == len(want)
        lib.gb_device_synchronize(dev.handle)
        assert (out.cpu().numpy() == 0xA5).all()
    out = torch.full((len(want),), 0xA5, dtype=torch.uint8, device="cuda")
    rc = lib.gb_bgzf_compress_device(dev.handle, C.c_void_p(src.data_ptr()), len(data), C.c_void_p(out.data_ptr()), len(want), C.byref(used))
    assert rc == capi.GB_OK and used.value == len(want)
    lib.gb_device_synchronize(dev.handle)
    assert out.cpu().numpy().tobytes() == want
    assert lib.gb_bgzf_compress_device(dev.handle, None, 5, C.c_void_p(out.data_ptr()), len(want), C.byref(used)) == capi.GB_ERR_ARG


# ---- the emitters' output: round trip and ratio ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mapped_config2():
    """20,000 reads (10,000 pairs) of bench.py's config-2 workload mapped by gb_map_batch_device, records left in HBM."""
    import torch
    import bench
    g, index = bench.make_graph_and_index()
    d = capi.Device(index, 0)
    n, L = 20000, bench.READ_LEN
    d_reads, d_quals = bench.simulate_pairs_torch(g, n // 2, 22, torch.device("cuda", 0))
    d_off = torch.arange(n + 1, dtype=torch.int64, device="cuda") * L
    d_aln = torch.zeros((n, 32), dtype=torch.uint8, device="cuda")
    d_maps = torch.zeros((n * 14, 8), dtype=torch.uint8, device="cuda")
    d_edits = torch.zeros(n * 20, dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_tot = torch.zeros(2, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    vp = lambda t: C.c_void_p(t.data_ptr())
    rc = _lib().gb_map_batch_device(d.handle, C.byref(H.paired_params(bench.FRAG_MEAN, bench.FRAG_SD)), 1, n, vp(d_reads), vp(d_quals), vp(d_off), L,
                                    vp(d_aln), vp(d_maps), n * 14, vp(d_edits), n * 20, vp(d_status), vp(d_tot))
    assert rc == capi.GB_OK
    out = {k: d.emit_device(k, d_aln, d_maps, d_edits, d_reads, d_off, d_quals) for k in ("gam", "gaf")}
    yield d, out
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["gam", "gaf"])
def test_emitter_output_round_trips_and_compresses(mapped_config2, kind):
    d, out = mapped_config2
    emitted = out[kind]
    plain = emitted.cpu().numpy().tobytes()
    raw = d.bgzf_compress_device(emitted).cpu().numpy().tobytes()
    inflated = gzip.decompress(raw)
    assert inflated == plain
    if kind == "gam":
        got, _ = read_stream(inflated)
        want, _ = read_stream(plain)
        assert len(got) == len(want) >= 20000 * 0.9
        assert [decode_alignment(m) for m in got[:500]] == [decode_alignment(m) for m in want[:500]]
    else:
        assert inflated.decode().count("\n") == plain.decode().count("\n") >= 20000 * 0.9
    z1 = _zlib_level1_size(plain)
    assert len(raw) <= 1.10 * z1, f"{kind}: {len(raw)} bytes on the device, {z1} with zlib level 1 (ratio {len(plain) / len(raw):.2f} vs {len(plain) / z1:.2f})"
    for (off, bsize), (_, _, pay) in list(zip(_members(raw), _bgzf_blocks(raw)))[:2]:
        assert strict_inflate(raw[off + 18:off + bsize - 8]) == pay
