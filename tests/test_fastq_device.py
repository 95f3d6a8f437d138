"""FASTQ input on the GPU: gb_bgzf_decompress_device (BGZF members in HBM inflated on the device) and gb_fastq_parse_device
(FASTQ text in HBM parsed into the mapper's input arrays).

The inflater is held to zlib: a member is accepted exactly when zlib's raw inflate accepts its payload with nothing left
over and the trailer matches, and then its bytes are zlib's.  The parser is held to oracle/fastq.cpp, a restatement of vg's
FASTQ reader, which is itself checked here on hand-written records and on the reference's FASTQ files."""
import ctypes as C
import gzip
import random
import struct
import zlib
from pathlib import Path

import numpy as np
import pytest

import helpers as H
from vg_b200 import capi, synth

GOLD = Path(__file__).resolve().parent / "golden"
FIXTURES = sorted((GOLD / "fastq").glob("*.f*q"))
PAIRED_FIXTURES = {"grch38_lrc_kir_paired.fq", "xy2.matchpaired.fq"}
EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


# ---- the oracle -----------------------------------------------------------------------------------------------------------
def oracle_parse(texts, interleaved=False, strict=True):
    """oracle_fastq_parse over whole inputs: {"reads": [bytes], "quals": [bytes], "names": [bytes], "max_read_len"} or
    ("error", input, record, kind)."""
    lib = H.oracle_lib()
    fn = lib.oracle_fastq_parse
    fn.restype = C.c_int
    vp, u64 = C.c_void_p, C.c_uint64
    fn.argtypes = [C.c_uint32, vp, vp, C.c_uint32, C.c_int, u64, vp, vp, vp, vp, vp, vp, vp, vp]
    bufs = [np.frombuffer(t + b"\0", dtype=np.uint8) for t in texts]
    ptrs = (C.c_void_p * len(texts))(*[b.ctypes.data for b in bufs])
    sizes = (C.c_uint64 * len(texts))(*[len(t) for t in texts])
    total = sum(len(t) for t in texts) + 1
    max_rec = total // 3 + 2
    reads, quals, names = (np.zeros(total, np.uint8) for _ in range(3))
    roff, noff = np.zeros(max_rec + 1, np.uint64), np.zeros(max_rec + 1, np.uint64)
    n, mx, err = C.c_uint32(), C.c_uint32(), (C.c_int64 * 3)()
    rc = fn(len(texts), ptrs, sizes, capi.GB_FASTQ_INTERLEAVED if interleaved else 0, 1 if strict else 0, max_rec,
            reads.ctypes.data, quals.ctypes.data, roff.ctypes.data, names.ctypes.data, noff.ctypes.data, C.byref(n), C.byref(mx), err)
    if rc == capi.GB_ERR_FORMAT:
        return ("error", err[0], err[1], err[2])
    assert rc == 0
    k = n.value
    cut = lambda buf, off: [buf[int(off[i]): int(off[i + 1])].tobytes() for i in range(k)]
    return {"reads": cut(reads, roff), "quals": cut(quals, roff), "names": cut(names, noff), "max_read_len": mx.value}


def python_parse(text):
    """An independent reading of the same rules for well-formed files: 4 lines per record."""
    lines = text.split(b"\n")
    assert lines[-1] == b""
    out = {"reads": [], "quals": [], "names": []}
    for r in range(0, len(lines) - 1, 4):
        h, s, _, q = lines[r: r + 4]
        name = h[1:]
        for i, c in enumerate(name):
            if c in b" \t\v\f\r":
                name = name[:i]
                break
        out["names"].append(name)
        out["reads"].append(s.upper())
        out["quals"].append(bytes(c - 33 for c in q))
    return out


# ---- CPU: the oracle against hand-written records and the fixtures ------------------------------------------------------------
def test_oracle_rules_on_hand_written_records():
    got = oracle_parse([b"@r1 comment here\nacgtNn\n+r1\nIIII#!\n@\tx\nRYKM\n+\n~~~~\n@r/2\n\n+\n\n"])
    assert got["names"] == [b"r1", b"", b"r/2"]
    assert got["reads"] == [b"ACGTNN", b"RYKM", b""]
    assert got["quals"] == [bytes([40, 40, 40, 40, 2, 0]), bytes([93] * 4), b""]
    assert got["max_read_len"] == 6
    # vg's own rules (strict off) and the divergences (strict on)
    assert oracle_parse([b"@a\nACGT\n+\n\n"], strict=False)["reads"] == [b"ACGT"]           # vg accepts an empty quality
    assert oracle_parse([b"@a\nACGT\n+\n\n"]) == ("error", 0, 0, 4)
    assert oracle_parse([b"@a\nAC\r\n+\nII\r\n"], strict=False)["reads"] == [b"AC\r"]     # CRLF goes into the read in vg
    assert oracle_parse([b"@a\nAC\r\n+\nII\r\n"]) == ("error", 0, 0, 2)
    assert oracle_parse([b"@a\nAC\n-\nII\n"], strict=False)["reads"] == [b"AC"]            # vg does not look at the separator
    assert oracle_parse([b"@a\nAC\n-\nII\n"]) == ("error", 0, 0, 3)
    ok = b"@a\nAC\n+\nII\n"
    assert oracle_parse([ok + b">b\nAC\n+\nII\n"], strict=False) == ("error", 0, 1, 1)
    assert oracle_parse([ok + b"@b\nAC\n+\nI\n"], strict=False) == ("error", 0, 1, 4)
    assert oracle_parse([ok + b"@b\nAC\n+\nI\x00\n"]) == ("error", 0, 1, 5)
    assert oracle_parse([ok + b"@b\nAC\n+\nII"], strict=False) == ("error", 0, 1, 4)          # last byte chopped, then too short
    assert oracle_parse([ok + b"@b\nAC\n"]) == ("error", 0, 1, 6)
    # pairs: a mate without its partner is dropped
    two = oracle_parse([ok * 3, ok * 2])
    assert len(two["reads"]) == 4
    assert len(oracle_parse([ok * 3], interleaved=True)["reads"]) == 2


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: p.name)
def test_oracle_on_the_reference_fixtures(path):
    text = path.read_bytes()
    got = oracle_parse([text])
    want = python_parse(text)
    assert got["reads"] == want["reads"] and got["quals"] == want["quals"] and got["names"] == want["names"]
    if path.name in PAIRED_FIXTURES:
        assert len(oracle_parse([text], interleaved=True)["reads"]) == len(want["reads"]) // 2 * 2
    if path.name == "1mb1kgp_longread.fq":
        assert max(len(r) for r in got["reads"]) > 512
    if path.name == "cactus-BRCA2.fastq":
        assert len(got["reads"]) == 1000


def test_oracle_reads_the_giraffe_t_read():
    got = oracle_parse([(GOLD / "vcf" / "small.middle.ref.fq").read_bytes()])
    assert len(got["reads"]) == 1 and len(got["reads"][0]) == 63


# ---- a model of the inflater: the member walk and zlib ------------------------------------------------------------------------
class Refused(Exception):
    pass


def model_decompress(data, final=True):
    """(bytes, in_used) as gb_bgzf_decompress_device must give them, or Refused."""
    out, p = [], 0
    while p < len(data):
        b = data[p:]
        if b[:3] != b"\x1f\x8b\x08"[: len(b[:3])]:
            raise Refused(p)
        if len(b) >= 4 and b[3] != 4:
            raise Refused(p)
        if len(b) < 12 or len(b) < 12 + struct.unpack_from("<H", b, 10)[0]:
            break
        xlen = struct.unpack_from("<H", b, 10)[0]
        q, bsize = 12, None
        while q + 4 <= 12 + xlen:
            slen = struct.unpack_from("<H", b, q + 2)[0]
            if q + 4 + slen > 12 + xlen:
                break
            if bsize is None and b[q: q + 2] == b"BC" and slen == 2:
                bsize = struct.unpack_from("<H", b, q + 4)[0]
            q += 4 + slen
        if q != 12 + xlen or bsize is None or bsize + 1 < 12 + xlen + 8:
            raise Refused(p)
        mlen = bsize + 1
        if mlen > len(b):
            break
        crc, isize = struct.unpack_from("<II", b, mlen - 8)
        if isize > 65536:
            raise Refused(p)
        d = zlib.decompressobj(-15)
        try:
            got = d.decompress(b[12 + xlen: mlen - 8])
        except zlib.error:
            raise Refused(p)
        if not d.eof or d.unused_data or len(got) != isize or zlib.crc32(got) != crc:
            raise Refused(p)
        out.append(got)
        p += mlen
    if p < len(data) and final:
        raise Refused(p)
    return b"".join(out), p


def member(payload_raw, extra_before=b"", isize=None, crc=None, strategy=None, level=6):
    """One BGZF member of `payload_raw` (compressed by zlib unless it is given as ("raw", deflate bytes))."""
    if isinstance(payload_raw, tuple):
        data, deflated = payload_raw[1], payload_raw[2]
    else:
        data = payload_raw
        c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy if strategy is not None else zlib.Z_DEFAULT_STRATEGY)
        deflated = c.compress(data) + c.flush()
    extra = extra_before + b"BC" + struct.pack("<HH", 2, 0)
    hdr = b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff" + struct.pack("<H", len(extra)) + extra
    total = len(hdr) + len(deflated) + 8
    bc = len(hdr) - 2
    hdr = hdr[:bc] + struct.pack("<H", total - 1)
    trailer = struct.pack("<II", zlib.crc32(data) if crc is None else crc, len(data) if isize is None else isize)
    return hdr + deflated + trailer


def corpus(n=200_000, seed=5):
    rng = np.random.default_rng(seed)
    parts = [bytes(rng.integers(0, 256, 5000, dtype=np.uint8)), b"A" * 70000, b"ACGT" * 9000,
             bytes(rng.choice(np.frombuffer(b"ACGTN\n@+", np.uint8), n))]
    return b"".join(parts)


@pytest.fixture(scope="module")
def dev():
    g = synth.make_tiny_graph()
    d = capi.Device(g.build_index(), 0)
    yield d
    d.close()


def _t(b, offset=0):
    import torch
    buf = torch.zeros(len(b) + offset + 1, dtype=torch.uint8, device="cuda")
    if len(b):
        buf[offset: offset + len(b)] = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    return buf[offset: offset + len(b)]


def inflate(dev, data, final=True, offset=0):
    out, used = dev.bgzf_decompress_device(_t(data, offset), final=final)
    return out.cpu().numpy().tobytes(), used


def verdict(dev, data, final=True):
    try:
        return inflate(dev, data, final)
    except capi.GbError as e:
        assert e.code == capi.GB_ERR_FORMAT, e
        return "refused"


def model_verdict(data, final=True):
    try:
        return model_decompress(data, final)
    except Refused:
        return "refused"


# ---- GPU: inflate ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_inflate_equals_zlib_on_host_and_device_bgzf(dev):
    data = corpus()
    for level in (0, 1, 6, 9):
        z = capi.bgzf_compress(data, level)
        assert inflate(dev, z) == (data, len(z)), level
    fixed = b"".join(member(data[i: i + 0xff00], strategy=zlib.Z_FIXED) for i in range(0, len(data), 0xff00)) + EOF_BLOCK
    assert model_decompress(fixed) == (data, len(fixed))
    assert inflate(dev, fixed) == (data, len(fixed))
    z = dev.bgzf_compress_device(_t(data))
    assert inflate(dev, z.cpu().numpy().tobytes())[0] == data
    for gam in sorted((GOLD / "gam").glob("*.gam")):
        raw = gam.read_bytes()
        assert inflate(dev, raw) == (gzip.decompress(raw), len(raw)), gam.name


@pytest.mark.gpu
def test_inflate_edge_cases(dev):
    assert inflate(dev, b"") == (b"", 0)
    assert inflate(dev, EOF_BLOCK) == (b"", 28)
    a, b = b"hello " * 3000, bytes(range(256)) * 200
    s = member(a) + EOF_BLOCK + EOF_BLOCK + member(b) + EOF_BLOCK
    assert inflate(dev, s) == (a + b, len(s))
    s = member(a, extra_before=b"XY" + struct.pack("<H", 3) + b"abc") + member(b, extra_before=b"ZZ\x00\x00")
    assert model_decompress(s)[0] == a + b and inflate(dev, s) == (a + b, len(s))
    rng = np.random.default_rng(3)
    for n in (0, 0xff00, 65536):
        d = bytes(rng.integers(0, 4, n, dtype=np.uint8) + 65)
        for level in ((0, 6) if n <= 0xff00 else (6,)):        # a stored 64 KiB block does not fit a 64 KiB member
            m = member(d, level=level)
            assert inflate(dev, m) == (d, len(m)), (n, level)
    # length-258 matches, distance-32768 matches, distance-1 runs
    blk = bytes(rng.integers(0, 256, 32768, dtype=np.uint8))
    for d in (b"\x00" * 65536, blk + blk[:30000], b"x" + b"y" * 60000 + b"xz" * 2000):
        m = member(d, level=9)
        assert inflate(dev, m) == (d, len(m))
    z = capi.bgzf_compress(corpus(100_000), 6)
    for off in range(16):
        assert inflate(dev, z, offset=off) == (corpus(100_000), len(z)), off


@pytest.mark.gpu
def test_inflate_streaming_at_every_cut(dev):
    data = b"".join(member(x) for x in (b"abc" * 50, b"", b"ACGT" * 40, bytes(range(200)))) + EOF_BLOCK
    want = model_decompress(data)[0]
    for cut in range(len(data) + 1):
        first, used = inflate(dev, data[:cut], final=False)
        assert (first, used) == model_decompress(data[:cut], final=False)
        rest, used2 = inflate(dev, data[used:], final=True)
        assert first + rest == want and used + used2 == len(data), cut
        if cut < len(data) and used < cut:
            assert verdict(dev, data[:cut], final=True) == "refused"


class Bits:
    """LSB-first deflate bit writer: put() for header fields, huff() for Huffman codes (written MSB first)."""
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, x, k):
        self.v |= x << self.n
        self.n += k
        return self

    def huff(self, code, k):
        return self.put(int(format(code, "0%db" % k)[::-1], 2), k)

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def _stored(data, nlen=None):
    return bytes([1]) + struct.pack("<HH", len(data), (~len(data) & 0xffff) if nlen is None else nlen) + data


@pytest.mark.gpu
def test_inflate_refusals(dev):
    good = member(b"ACGT" * 1000)
    cases = {
        "bad crc": member(b"ACGT" * 1000, crc=1),
        "bad isize": member(b"ACGT" * 1000, isize=3999),
        "isize above 65536": member(("raw", b"", _stored(b"")), isize=70000),
        "bad bsize": good[:16] + struct.pack("<H", 20) + good[18:],
        "truncated": good[:-1],
        "plain gzip": gzip.compress(b"ACGT" * 100),
        "btype 11": member(("raw", b"", b"\x07\x00")),
        "stored len/nlen": member(("raw", b"abc", _stored(b"abc", nlen=0))),
        # dynamic block whose code-length code gives three symbols one bit each
        "over-subscribed": member(("raw", b"", Bits().put(1, 1).put(2, 2).put(0, 5).put(0, 5).put(0, 4)
                                   .put(1, 3).put(1, 3).put(1, 3).put(0, 3).bytes())),
        # fixed block: literal 'a', then a match of length 3 at distance 2, which reaches before the member's first byte
        "distance too far": member(("raw", b"aaaa", Bits().put(1, 1).put(1, 2).huff(0x30 + 97, 8).huff(1, 7).huff(1, 5)
                                    .huff(0, 7).bytes())),
        "trailing bytes in payload": member(("raw", b"", b"\x03\x00\x00")),
    }
    for name, data in cases.items():
        assert model_verdict(data) == "refused", name
        assert verdict(dev, data) == "refused", name
        assert verdict(dev, good + data) == "refused", name
    with pytest.raises(capi.GbError, match="byte 0") as e:
        inflate(dev, gzip.compress(b"x"))
    assert e.value.code == capi.GB_ERR_FORMAT


@pytest.mark.gpu
def test_inflate_single_bit_flips_agree_with_zlib(dev):
    rng = random.Random(11)
    data = capi.bgzf_compress(corpus(150_000, seed=9), 6)[:60_000]
    data = data[: model_decompress(data, final=False)[1]] + EOF_BLOCK
    fixed = member(b"GATTACA" * 300, strategy=zlib.Z_FIXED) + member(b"x" * 5000, level=0)
    accepted = 0
    for src in (data, fixed):
        for k in range(150 if src is data else 100):
            i = rng.randrange(len(src) * 8) if k % 5 else rng.randrange(18 * 8)     # every fifth in the first header
            flipped = bytearray(src)
            flipped[i // 8] ^= 1 << (i % 8)
            want = model_verdict(bytes(flipped))
            assert verdict(dev, bytes(flipped)) == want, i
            accepted += want != "refused"
    assert accepted > 0


@pytest.mark.gpu
def test_inflate_capacity_edge(dev):
    import torch
    data = capi.bgzf_compress(corpus(80_000), 6)
    need = len(corpus(80_000))
    lib = capi.load_library()
    src = _t(data)
    used, in_used = C.c_uint64(), C.c_uint64()
    out = torch.full((need,), 7, dtype=torch.uint8, device="cuda")
    rc = lib.gb_bgzf_decompress_device(dev.handle, C.c_void_p(src.data_ptr()), len(data), 1, C.c_void_p(out.data_ptr()), need - 1,
                                       C.byref(used), C.byref(in_used))
    assert rc == capi.GB_ERR_CAPACITY and used.value == need
    assert bool((out == 7).all())                                  # nothing written
    rc = lib.gb_bgzf_decompress_device(dev.handle, C.c_void_p(src.data_ptr()), len(data), 1, C.c_void_p(out.data_ptr()), need,
                                       C.byref(used), C.byref(in_used))
    assert rc == capi.GB_OK and used.value == need and in_used.value == len(data)
    assert out.cpu().numpy().tobytes() == corpus(80_000)


# ---- GPU: parse ---------------------------------------------------------------------------------------------------------------
def parse(dev, texts, **kw):
    got = dev.fastq_parse_device([_t(t) for t in texts], **kw)
    ro, no = got["read_off"].cpu().numpy(), got["name_off"].cpu().numpy()
    reads, quals, names = (got[k].cpu().numpy().tobytes() for k in ("reads", "quals", "names"))
    n = got["n_reads"]
    return {"reads": [reads[ro[i]: ro[i + 1]] for i in range(n)], "quals": [quals[ro[i]: ro[i + 1]] for i in range(n)],
            "names": [names[no[i]: no[i + 1]] for i in range(n)], "max_read_len": got["max_read_len"], "text_used": got["text_used"]}


def same(got, want):
    return all(got[k] == want[k] for k in ("reads", "quals", "names", "max_read_len"))


def generated(n=600, seed=1):
    rng = random.Random(seed)
    alphabet = b"ACGTNacgtnRYKMSWBDHVryk"
    recs = []
    for i in range(n):
        L = i + 1
        name = rng.choice([b"", b"r%d" % i, b"r%d/1" % i, b"read:%d#0" % i])
        tail = rng.choice([b"", b" comment", b"\tx y", b" ", b"\x0bz", b"\rq"])
        seq = bytes(rng.choice(alphabet) for _ in range(L))
        qual = bytes(33 + (j + i) % 94 for j in range(L))
        recs.append(b"@" + name + tail + b"\n" + seq + b"\n+" + rng.choice([b"", name]) + b"\n" + qual + b"\n")
    return b"".join(recs)


@pytest.mark.gpu
def test_parse_equals_the_oracle(dev):
    for path in FIXTURES:
        text = path.read_bytes()
        assert same(parse(dev, [text]), oracle_parse([text])), path.name
        if path.name in PAIRED_FIXTURES:
            assert same(parse(dev, [text], interleaved=True), oracle_parse([text], interleaved=True)), path.name
    text = generated()
    got, want = parse(dev, [text]), oracle_parse([text])
    assert same(got, want) and got["max_read_len"] == 600 and got["text_used"] == [len(text)]
    assert parse(dev, [(GOLD / "vcf" / "small.middle.ref.fq").read_bytes()])["max_read_len"] == 63


@pytest.mark.gpu
def test_parse_at_every_cut(dev):
    text = (GOLD / "fastq" / "small.middle.ref.indel.multi.fq").read_bytes()
    want = oracle_parse([text])
    for cut in range(len(text) + 1):
        a = parse(dev, [text[:cut]], final=False)
        b = parse(dev, [text[a["text_used"][0]:]], final=True)
        assert [a[k] + b[k] for k in ("reads", "quals", "names")] == [want[k] for k in ("reads", "quals", "names")], cut
        whole = text[:cut].count(b"\n") % 4 == 0 and (cut == 0 or text[cut - 1] == 10)
        if whole:
            assert parse(dev, [text[:cut]], final=True)["reads"] == want["reads"][: text[:cut].count(b"\n") // 4]
        else:
            with pytest.raises(capi.GbError) as e:
                parse(dev, [text[:cut]], final=True)
            assert e.value.code == capi.GB_ERR_FORMAT


@pytest.mark.gpu
def test_parse_capacity_stops(dev):
    text = generated(60, seed=4)
    want = oracle_parse([text])
    lens = np.cumsum([0] + [len(r) for r in want["reads"]])
    nlens = np.cumsum([0] + [len(r) for r in want["names"]])
    for k in (1, 7, 30, 59):
        assert len(parse(dev, [text], final=False, max_reads=k)["reads"]) == k
        got = parse(dev, [text], final=False, bases_cap=int(lens[k]) + (1 if k < 59 else 0))
        assert len(got["reads"]) == k
        got = parse(dev, [text], final=False, names_cap=int(nlens[k]))
        assert len(got["reads"]) == max(i for i in range(61) if nlens[i] <= nlens[k])
    for kw in (dict(max_reads=0), dict(bases_cap=0)):
        with pytest.raises(capi.GbError) as e:
            parse(dev, [text], final=False, **kw)
        assert e.value.code == capi.GB_ERR_CAPACITY


@pytest.mark.gpu
def test_parse_pairs(dev):
    a, b = generated(9, seed=5), generated(12, seed=6)
    got, want = parse(dev, [a, b]), oracle_parse([a, b])
    assert same(got, want) and len(got["reads"]) == 18
    assert got["text_used"] == [len(a), len(b"\n".join(b.split(b"\n")[:36]) + b"\n")]
    odd = generated(7, seed=7)
    got = parse(dev, [odd], interleaved=True)
    assert same(got, oracle_parse([odd], interleaved=True)) and len(got["reads"]) == 6
    assert got["text_used"] == [len(b"\n".join(odd.split(b"\n")[:24]) + b"\n")]


@pytest.mark.gpu
def test_parse_refusals(dev):
    ok = b"@a x\nACGT\n+\nIIII\n"
    for bad, kind in ((b">b\nACGT\n+\nIIII\n", 1), (b"@b\nACGT\n-\nIIII\n", 3), (b"@b\nACGT\n+\nIII\n", 4),
                      (b"@b\nAC\rT\n+\nIIII\n", 2), (b"@b\nACGT\n+\nII\x00I\n", 5), (b"@b\nACGT\n+\n\n", 4),
                      (b"@b\nAC T\n+\nIIII\n", 2)):
        text = ok * 3 + bad + ok
        assert oracle_parse([text])[1:] == (0, 3, kind)
        with pytest.raises(capi.GbError, match="input 0, record 3, byte") as e:
            parse(dev, [text])
        assert e.value.code == capi.GB_ERR_FORMAT
        with pytest.raises(capi.GbError, match="input 1, record 3, byte"):
            parse(dev, [ok * 5, text])
    for tail in (b"@a\nAC\n+\nII", b"\n", b"@a\n"):
        with pytest.raises(capi.GbError, match="ends inside a record"):
            parse(dev, [ok * 2 + tail])
        assert len(parse(dev, [ok * 2 + tail], final=False)["reads"]) == 2


# ---- GPU: end to end ----------------------------------------------------------------------------------------------------------
def fastq_of(reads, quals, mate):
    return b"".join(b"@p%d/%d extra\n" % (i, mate) + bytes(r) + b"\n+\n" + bytes(q + 33) + b"\n" for i, (r, q) in enumerate(zip(reads, quals)))


@pytest.mark.gpu
def test_end_to_end_fastq_gz_to_gam(dev):
    import torch
    g = synth.make_variant_graph(length=30000, n_snp=48, n_ins=6, n_del=6, n_haps=4, seed=3)
    index = g.build_index()
    d = capi.Device(index, 0)
    rs = synth.simulate_pairs(g, 200, sub_rate=0.002, seed=8, indel_rate=0.0002)
    rng = np.random.default_rng(2)
    quals = rng.choice(np.array([2, 12, 23, 37], np.uint8), size=rs.reads.shape, p=[0.02, 0.08, 0.2, 0.7])
    r1, r2 = (fastq_of(rs.reads[m::2], quals[m::2], m + 1) for m in (0, 1))
    z1, z2 = capi.bgzf_compress(r1, 6), capi.bgzf_compress(r2, 6)
    t1, _ = d.bgzf_decompress_device(_t(z1))
    t2, _ = d.bgzf_decompress_device(_t(z2))
    p = d.fastq_parse_device([t1, t2])
    n = p["n_reads"]
    host = oracle_parse([r1, r2])
    assert n == rs.n and host["reads"] == [bytes(x) for x in rs.reads]
    params = H.paired_params()
    MAP_PER, EDIT_PER = 24, 64
    d_aln = torch.zeros((n, 32), dtype=torch.uint8, device="cuda")
    d_maps = torch.zeros((n * MAP_PER, 8), dtype=torch.uint8, device="cuda")
    d_edits = torch.zeros(n * EDIT_PER, dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_tot = torch.zeros(2, dtype=torch.int64, device="cuda")
    vp = lambda t: C.c_void_p(t.data_ptr())
    lib = capi.load_library()
    rc = lib.gb_map_batch_device(d.handle, C.byref(params), 1, n, vp(p["reads"]), vp(p["quals"]), vp(p["read_off"]), p["max_read_len"],
                                 vp(d_aln), vp(d_maps), n * MAP_PER, vp(d_edits), n * EDIT_PER, vp(d_status), vp(d_tot))
    assert rc == capi.GB_OK
    lib.gb_device_synchronize(d.handle)
    gam = d.emit_device("gam", d_aln, d_maps, d_edits, p["reads"], p["read_off"], p["quals"], p["names"], p["name_off"])
    gam = gam.cpu().numpy().tobytes()
    rbuf = np.frombuffer(b"".join(host["reads"]), np.uint8).copy()
    qbuf = np.frombuffer(b"".join(host["quals"]), np.uint8).copy()
    roff = np.concatenate([[0], np.cumsum([len(x) for x in host["reads"]])]).astype(np.uint64)
    aln, maps, edits, _ = d.map_arrays(rbuf, qbuf, roff, params, paired=True)
    want = capi.emit_text("gam", index.view, aln, maps, edits, rbuf, qbuf, roff, names=[x.decode() for x in host["names"]])
    assert gam == want
    d.close()
    # the 50_vg_giraffe.t pin through the device reader: score 73 for small.middle.ref.fq
    import vcf_graph as V
    gx, _ = V.small_x()
    ix = gx.build_index()
    dx = capi.Device(ix, scores=capi.Scores(1, 4, 6, 1, 5))
    z = capi.bgzf_compress((GOLD / "vcf" / "small.middle.ref.fq").read_bytes(), 6)
    text, _ = dx.bgzf_decompress_device(_t(z))
    p = dx.fastq_parse_device([text])
    reads = p["reads"].cpu().numpy()[None, :].copy()
    got = H.gpu_map(dx, reads, p["quals"].cpu().numpy()[None, :].copy())
    assert int(got[0][0]["score"]) == 73
    dx.close()
    ix.close()
