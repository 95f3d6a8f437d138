#!/usr/bin/env python
"""bench_input.py — FASTQ input on the GPU (gb_bgzf_decompress_device + gb_fastq_parse_device) against the host, on
bench.py's workload.

  python scripts/bench_input.py [--reads 1000000] [--warmup 2] [--reps 5]

bench.py's configs[1] read pairs (150 bp), written as two FASTQ files (-f r1 -f r2) with Illumina-style names and a seeded
binned quality model (4 bins, as NovaSeq writes them; a constant quality would compress unrealistically well), each
compressed to BGZF at zlib level 6.  Times, with the host clock around the call and a device synchronise:
  inflate   gb_bgzf_decompress_device on both files (GB/s of output and of input)
  parse     gb_fastq_parse_device on both inflated files (M records/s)
  chain     compressed FASTQ in pinned host memory -> H2D -> inflate -> parse -> gb_map_batch_device (paired) ->
            gb_emit_gam_device -> gb_bgzf_compress_device -> D2H, beside the same chain started from parsed host arrays
            (reads, qualities, names and offsets in pinned memory -> H2D -> map -> GAM -> BGZF -> D2H)
  host      zlib inflate of the same members and the oracle's FASTQ reader (oracle/fastq.cpp), each on one core
Median of --reps after --warmup.  Prints one JSON line with the GPU name and power limit; exits non-zero when the parsed
reads differ from the oracle's or the GAM differs from the run on host-parsed arrays.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import struct
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "scripts"))

QUAL_BINS = np.array([2, 12, 23, 37], dtype=np.uint8)
QUAL_P = [0.01, 0.04, 0.10, 0.85]


def bgzf_level6(data: bytes) -> bytes:
    """BGZF members of 0xff00 input bytes at zlib level 6 (the cuts gb_bgzf_compress makes), compressed on all host cores."""
    def one(at):
        chunk = data[at: at + 0xff00]
        c = zlib.compressobj(6, zlib.DEFLATED, -15)
        body = c.compress(chunk) + c.flush()
        return (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", 18 + len(body) + 8 - 1) + body +
                struct.pack("<II", zlib.crc32(chunk), len(chunk)))
    with ThreadPoolExecutor() as ex:
        members = list(ex.map(one, range(0, len(data), 0xff00)))
    return b"".join(members) + bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def fastq_text(reads: np.ndarray, quals: np.ndarray, mate: int) -> bytes:
    n, L = reads.shape
    out = []
    for i in range(n):
        tile, x, y = 1101 + (i // 400_000) % 80, 1000 + (i * 7919) % 31000, 1000 + (i * 104729) % 37000
        out.append(b"@A00123:8:H5KJLDSXX:1:%d:%d:%d %d:N:0:ATCACGTT\n" % (tile, x, y, mate))
        out.append(reads[i].tobytes())
        out.append(b"\n+\n")
        out.append((quals[i] + 33).tobytes())
        out.append(b"\n")
    return b"".join(out)


def timed(fn, warmup, reps, sync):
    times = []
    for rep in range(warmup + reps):
        t0 = time.perf_counter()
        fn()
        sync()
        t1 = time.perf_counter()
        if rep >= warmup:
            times.append(t1 - t0)
    return statistics.median(times), times


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch
    import bench
    import helpers as H
    from bench_emit import gpu_identity
    from vg_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_input.py: no CUDA device")
    device = torch.device("cuda", 0)
    g, index = bench.make_graph_and_index()
    dev = capi.Device(index, 0)
    lib = capi.load_library()
    stream = torch.cuda.Stream(device=device)
    torch.cuda.set_stream(stream)
    lib.gb_device_set_stream(dev.handle, C.c_void_p(stream.cuda_stream))
    vp = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    sync = lambda: lib.gb_device_synchronize(dev.handle)

    n = args.reads - args.reads % 2
    L = bench.READ_LEN
    d_reads, _ = bench.simulate_pairs_torch(g, n // 2, 22, device)
    reads = d_reads.view(n, L).cpu().numpy()
    quals = np.random.default_rng(7).choice(QUAL_BINS, size=(n, L), p=QUAL_P).astype(np.uint8)
    texts = [fastq_text(reads[m::2], quals[m::2], m + 1) for m in (0, 1)]
    gz = [bgzf_level6(t) for t in texts]
    fq_bytes, gz_bytes = sum(len(t) for t in texts), sum(len(z) for z in gz)

    # ---- host baseline (one core each): zlib inflate of the same members, the oracle reader ----
    t0 = time.perf_counter()
    for z in gz:                                          # member by member, as the BSIZE walk finds them
        at = 0
        while at < len(z):
            end = at + struct.unpack_from("<H", z, at + 16)[0] + 1
            zlib.decompress(z[at + 18: end - 8], -15)
            at = end
    host_inflate = time.perf_counter() - t0
    olib = H.oracle_lib()
    olib.oracle_fastq_parse.restype = C.c_int
    obufs = [np.frombuffer(t, np.uint8) for t in texts]
    o_r, o_q, o_n = (np.zeros(fq_bytes, np.uint8) for _ in range(3))
    o_roff, o_noff = np.zeros(n + 1, np.uint64), np.zeros(n + 1, np.uint64)
    o_cnt, o_mx, o_err = C.c_uint32(), C.c_uint32(), (C.c_int64 * 3)()
    t0 = time.perf_counter()
    rc = olib.oracle_fastq_parse(C.c_uint32(2), (C.c_void_p * 2)(*[b.ctypes.data for b in obufs]), (C.c_uint64 * 2)(*[len(t) for t in texts]),
                                 C.c_uint32(0), C.c_int(1), C.c_uint64(n), *(C.c_void_p(a.ctypes.data) for a in (o_r, o_q, o_roff, o_n, o_noff)),
                                 C.byref(o_cnt), C.byref(o_mx), o_err)
    host_parse = time.perf_counter() - t0
    assert rc == 0 and o_cnt.value == n, (rc, o_cnt.value)

    # ---- device: inflate and parse ----
    d_gz = [torch.from_numpy(np.frombuffer(z, np.uint8).copy()).to(device) for z in gz]
    d_txt = [torch.empty(len(t), dtype=torch.uint8, device=device) for t in texts]
    used, in_used = C.c_uint64(), C.c_uint64()

    def inflate():
        for z, t in zip(d_gz, d_txt):
            rc = lib.gb_bgzf_decompress_device(dev.handle, vp(z), z.numel(), 1, vp(t), t.numel(), C.byref(used), C.byref(in_used))
            assert rc == capi.GB_OK and used.value == t.numel(), rc
    inflate_s, inflate_times = timed(inflate, args.warmup, args.reps, sync)
    inflated_ok = all(bytes(t.cpu().numpy().tobytes()) == x for t, x in zip(d_txt, texts))

    d_r = torch.empty(n * L, dtype=torch.uint8, device=device)
    d_q = torch.empty(n * L, dtype=torch.uint8, device=device)
    d_n = torch.empty(n * 64, dtype=torch.uint8, device=device)
    d_roff = torch.empty(n + 1, dtype=torch.int64, device=device)
    d_noff = torch.empty(n + 1, dtype=torch.int64, device=device)
    ptrs = (C.c_void_p * 2)(*[t.data_ptr() for t in d_txt])
    sizes = (C.c_uint64 * 2)(*[t.numel() for t in d_txt])
    tused = (C.c_uint64 * 2)()
    nr, mx = C.c_uint32(), C.c_uint32()

    def parse():
        rc = lib.gb_fastq_parse_device(dev.handle, 2, ptrs, sizes, 0, 1, n, vp(d_r), vp(d_q), n * L, vp(d_roff), vp(d_n), n * 64,
                                       vp(d_noff), C.byref(nr), C.byref(mx), tused)
        assert rc == capi.GB_OK and nr.value == n, (rc, nr.value)
    parse_s, parse_times = timed(parse, args.warmup, args.reps, sync)
    roff = d_roff.cpu().numpy()
    noff = d_noff.cpu().numpy()
    rb, qb, nb = d_r.cpu().numpy().tobytes(), d_q.cpu().numpy().tobytes(), d_n.cpu().numpy().tobytes()
    nbases, nnames = int(roff[n]), int(noff[n])
    parsed_ok = (mx.value == o_mx.value and np.array_equal(roff.astype(np.uint64), o_roff) and np.array_equal(noff.astype(np.uint64), o_noff)
                 and rb[:nbases] == o_r[:nbases].tobytes() and qb[:nbases] == o_q[:nbases].tobytes() and nb[:nnames] == o_n[:nnames].tobytes())

    # ---- the chain, from compressed FASTQ and from parsed host arrays ----
    params = H.paired_params(bench.FRAG_MEAN, bench.FRAG_SD)
    MAP_PER, EDIT_PER = 14, 20
    d_aln = torch.zeros((n, 32), dtype=torch.uint8, device=device)
    d_maps = torch.zeros((n * MAP_PER, 8), dtype=torch.uint8, device=device)
    d_edits = torch.zeros(n * EDIT_PER, dtype=torch.int32, device=device)
    d_status = torch.zeros(n, dtype=torch.uint8, device=device)
    d_tot = torch.zeros(2, dtype=torch.int64, device=device)
    d_gam = torch.empty(n * 1024, dtype=torch.uint8, device=device)
    d_bgzf = torch.empty(n * 1024 // 3, dtype=torch.uint8, device=device)
    h_gz = [torch.from_numpy(np.frombuffer(z, np.uint8).copy()).pin_memory() for z in gz]
    h_arrays = [torch.from_numpy(np.frombuffer(b, np.uint8).copy()).pin_memory() for b in (rb[: roff[n]], qb[: roff[n]], nb[: noff[n]])]
    h_offs = [torch.from_numpy(o[: n + 1].astype(np.int64)).pin_memory() for o in (roff, noff)]
    h_out = torch.empty(d_bgzf.numel(), dtype=torch.uint8).pin_memory()
    gam_used, bgzf_used = C.c_uint64(), C.c_uint64()

    def map_emit_compress(r, q, ro, nm, no, max_len):
        rc = lib.gb_map_batch_device(dev.handle, C.byref(params), 1, n, vp(r), vp(q), vp(ro), max_len, vp(d_aln), vp(d_maps), n * MAP_PER,
                                     vp(d_edits), n * EDIT_PER, vp(d_status), vp(d_tot))
        assert rc == capi.GB_OK, rc
        rc = lib.gb_emit_gam_device(dev.handle, n, vp(d_aln), vp(d_maps), n * MAP_PER, vp(d_edits), n * EDIT_PER, n, vp(r), vp(q), vp(ro),
                                    vp(nm), vp(no), vp(d_gam), d_gam.numel(), C.byref(gam_used))
        assert rc == capi.GB_OK, rc
        rc = lib.gb_bgzf_compress_device(dev.handle, vp(d_gam), gam_used.value, vp(d_bgzf), d_bgzf.numel(), C.byref(bgzf_used))
        assert rc == capi.GB_OK, rc
        h_out[: bgzf_used.value].copy_(d_bgzf[: bgzf_used.value], non_blocking=True)

    def chain_fastq():
        for h, z in zip(h_gz, d_gz):
            z.copy_(h, non_blocking=True)
        inflate()
        parse()
        map_emit_compress(d_r, d_q, d_roff, d_n, d_noff, mx.value)

    d_r2, d_q2, d_n2 = (torch.empty(h.numel(), dtype=torch.uint8, device=device) for h in h_arrays)
    d_roff2, d_noff2 = (torch.empty(n + 1, dtype=torch.int64, device=device) for _ in range(2))

    def chain_arrays():
        for h, d in zip(h_arrays + h_offs, (d_r2, d_q2, d_n2, d_roff2, d_noff2)):
            d.copy_(h, non_blocking=True)
        map_emit_compress(d_r2, d_q2, d_roff2, d_n2, d_noff2, L)

    chain_fastq_s, chain_fastq_times = timed(chain_fastq, args.warmup, args.reps, sync)
    gam_fastq = d_gam[: gam_used.value].cpu().numpy().tobytes()
    chain_arrays_s, chain_arrays_times = timed(chain_arrays, args.warmup, args.reps, sync)
    gam_arrays = d_gam[: gam_used.value].cpu().numpy().tobytes()
    gam_ok = gam_fastq == gam_arrays

    name, power = gpu_identity()
    result = {
        "metric": "FASTQ input on the GPU: BGZF inflate and FASTQ parse", "gpu": name, "power_limit": power, "reads": n,
        "workload": bench.WORKLOAD + "; Illumina-style names, 4-bin qualities, two BGZF FASTQ files at zlib level 6",
        "fastq_bytes": fq_bytes, "bgzf_bytes": gz_bytes, "compression_ratio": fq_bytes / gz_bytes,
        "inflate": {"output_gb_per_s": fq_bytes / inflate_s / 1e9, "input_gb_per_s": gz_bytes / inflate_s / 1e9, "ms": inflate_s * 1e3,
                    "ms_min": min(inflate_times) * 1e3, "ms_max": max(inflate_times) * 1e3},
        "parse": {"m_records_per_s": n / parse_s / 1e6, "gb_per_s": fq_bytes / parse_s / 1e9, "ms": parse_s * 1e3,
                  "ms_min": min(parse_times) * 1e3, "ms_max": max(parse_times) * 1e3},
        "chain_from_bgzf_fastq": {"reads_per_s": n / chain_fastq_s, "ms": chain_fastq_s * 1e3, "h2d_bytes": gz_bytes},
        "chain_from_parsed_host_arrays": {"reads_per_s": n / chain_arrays_s, "ms": chain_arrays_s * 1e3,
                                          "h2d_bytes": int(sum(h.numel() for h in h_arrays) + 16 * (n + 1))},
        "host_one_core": {"zlib_inflate_ms": host_inflate * 1e3, "zlib_inflate_output_mb_per_s": fq_bytes / host_inflate / 1e6,
                          "oracle_parse_ms": host_parse * 1e3, "oracle_parse_m_records_per_s": n / host_parse / 1e6},
        "speedup_inflate_vs_host_core": host_inflate / inflate_s, "speedup_parse_vs_host_core": host_parse / parse_s,
        "inflated_equal_to_fastq": inflated_ok, "parsed_equal_to_oracle": parsed_ok, "gam_equal_to_host_parsed_run": gam_ok,
        "method": f"host clock + device synchronise, median of {args.reps} after {args.warmup} warm-ups",
    }
    print(json.dumps(result))
    dev.close()
    return 0 if inflated_ok and parsed_ok and gam_ok else 1


if __name__ == "__main__":
    sys.exit(main())
