#!/usr/bin/env python
"""bench_surject.py — surjection and SAM output rate on the GPU, on bench.py's workload.

  python scripts/bench_surject.py [--reads 1000000] [--warmup 2] [--reps 5] [--check 20000]

Maps the reads (bench.py's configs[1] generator, 150 bp pairs, one gb_map_batch_device call) and surjects the records in
HBM onto haplotype 0, the reference path.  Times gb_surject_device and gb_emit_sam_device (host clock around the call and
a device synchronise, median of --reps after --warmup calls), reports the records on the direct route and those deferred
to the realigning route, and checks the first --check records (whole pairs) field for field and the SAM text byte for byte
against the host restatement in tests/surject_oracle.py, timing that on one host core.  Prints one JSON line with the GPU
name and power limit; exits non-zero when anything differs.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "scripts"))


def timed(lib, dev, call, args):
    times = []
    for rep in range(args.warmup + args.reps):
        t0 = time.perf_counter()
        rc = call()
        lib.gb_device_synchronize(dev.handle)
        t1 = time.perf_counter()
        assert rc == 0, rc
        if rep >= args.warmup:
            times.append(t1 - t0)
    return statistics.median(times), min(times), max(times)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--check", type=int, default=20_000)
    args = ap.parse_args()

    import torch
    import bench
    import helpers as H
    import surject_oracle as O
    from bench_emit import gpu_identity
    from vg_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_surject.py: no CUDA device")
    device = torch.device("cuda", 0)
    g, index = bench.make_graph_and_index()
    dev = capi.Device(index, 0)
    lib = capi.load_library()
    vp = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    paths = [("ref", g.paths[0])]
    rp = capi.RefPaths(index.view, paths)
    dev.set_ref_paths(rp)

    n = args.reads - args.reads % 2
    L = bench.READ_LEN
    d_reads, d_quals = bench.simulate_pairs_torch(g, n // 2, 22, device)
    d_off = torch.arange(n + 1, dtype=torch.int64, device=device) * L
    MAP_PER, EDIT_PER = 14, 20
    d_aln = torch.zeros((n, 32), dtype=torch.uint8, device=device)
    d_maps = torch.zeros((n * MAP_PER, 8), dtype=torch.uint8, device=device)
    d_edits = torch.zeros(n * EDIT_PER, dtype=torch.int32, device=device)
    d_status = torch.zeros(n, dtype=torch.uint8, device=device)
    d_tot = torch.zeros(2, dtype=torch.int64, device=device)
    params = H.paired_params(bench.FRAG_MEAN, bench.FRAG_SD)
    tlen_max = int(bench.FRAG_MEAN + 6 * bench.FRAG_SD)
    torch.cuda.synchronize()
    rc = lib.gb_map_batch_device(dev.handle, C.byref(params), 1, n, vp(d_reads), vp(d_quals), vp(d_off), L, vp(d_aln), vp(d_maps), n * MAP_PER,
                                 vp(d_edits), n * EDIT_PER, vp(d_status), vp(d_tot))
    if rc != capi.GB_OK:
        raise capi.GbError(rc, "gb_map_batch_device")
    lib.gb_device_synchronize(dev.handle)
    tot = [int(x) for x in d_tot.cpu()]

    d_rec = torch.empty(n * 40, dtype=torch.uint8, device=device)
    used, n_realign = C.c_uint64(), C.c_uint32()
    surject = lambda cig, cap: lib.gb_surject_device(dev.handle, n, vp(d_aln), vp(d_maps), tot[0], vp(d_edits), tot[1], n, vp(d_off), tlen_max,
                                                     vp(d_rec), vp(cig), cap, C.byref(used), C.byref(n_realign))
    probe = torch.empty(1, dtype=torch.int32, device=device)
    assert surject(probe, 0) == capi.GB_ERR_CAPACITY
    d_cig = torch.empty(max(1, used.value), dtype=torch.int32, device=device)
    s_sec, s_min, s_max = timed(lib, dev, lambda: surject(d_cig, d_cig.numel()), args)
    ops = used.value

    sused = C.c_uint64()
    emit = lambda out, cap: lib.gb_emit_sam_device(dev.handle, n, vp(d_rec), vp(d_cig), ops, n, vp(d_reads), vp(d_quals), vp(d_off),
                                                   None, None, vp(out), cap, C.byref(sused))
    assert emit(torch.empty(1, dtype=torch.uint8, device=device), 0) == capi.GB_ERR_CAPACITY
    d_sam = torch.empty(sused.value, dtype=torch.uint8, device=device)
    e_sec, e_min, e_max = timed(lib, dev, lambda: emit(d_sam, d_sam.numel()), args)
    sam_bytes = sused.value

    recs = np.frombuffer(d_rec.cpu().numpy().tobytes(), dtype=capi.sam_record_dt)
    routes = np.bincount(recs["route"], minlength=4)

    # the oracle on the first records (whole pairs), on one host core
    k = min(n, args.check - args.check % 2)
    aln = d_aln.cpu().numpy().view(capi.alignment_dt).reshape(-1)[:k]
    maps = d_maps[: tot[0] + 1].cpu().numpy().view(capi.mapping_dt).reshape(-1)
    edits = d_edits[: tot[1] + 1].cpu().numpy().view(np.uint32)
    reads = [bytes(r).decode() for r in d_reads.cpu().numpy().reshape(n, L)[:k]]
    quals = list(d_quals.cpu().numpy().reshape(n, L)[:k])
    node_len = index.array("nodes")["len"].astype(np.int64)
    t0 = time.perf_counter()
    want = O.surject(aln, maps, edits, paths, node_len, tlen_max=tlen_max)
    want_text = O.sam_text(want, None, reads, quals, ["ref"])
    host_sec = time.perf_counter() - t0
    got = O.decode_device(d_rec[: k * 40].cpu().numpy().tobytes(), d_cig.cpu().numpy().view(np.uint32))
    bad_fields = sum(1 for a, b in zip(got, want) if a != {x: v for x, v in b.items() if x != "rev"})
    got_text = d_sam.cpu().numpy().tobytes().decode()
    got_lines = got_text[: sum(len(l) for l in want_text.splitlines(keepends=True))]
    text_equal = got_lines == want_text

    name, power = gpu_identity()
    result = {"metric": "surjection onto haplotype 0 and SAM output of alignment records in HBM", "reads": n, "workload": bench.WORKLOAD,
              "tlen_max": tlen_max,
              "routes": {"direct": int(routes[0]), "unmapped": int(routes[1]), "realign_deferred": int(routes[2]), "absent": int(routes[3])},
              "direct_fraction": float(routes[0]) / n, "realign_deferred_fraction": float(routes[2]) / n,
              "realign_deferred_reported": n_realign.value,
              "surject": {"records_per_s": n / s_sec, "ms_per_call": s_sec * 1e3, "ms_min": s_min * 1e3, "ms_max": s_max * 1e3, "cigar_ops": ops},
              "emit_sam": {"records_per_s": n / e_sec, "ms_per_call": e_sec * 1e3, "ms_min": e_min * 1e3, "ms_max": e_max * 1e3,
                           "bytes": sam_bytes, "output_gb_per_s": sam_bytes / e_sec / 1e9},
              "surject_plus_sam_records_per_s": n / (s_sec + e_sec),
              "oracle_check": {"records": k, "records_differing": bad_fields, "sam_text_equal": text_equal,
                               "host_records_per_s_one_core": k / host_sec},
              "gpu": name, "power_limit": power,
              "timing": f"host clock around the call + gb_device_synchronize, median of {args.reps} after {args.warmup} warm-up calls"}
    print(json.dumps(result))
    rp.close(); dev.close()
    return 0 if bad_fields == 0 and text_equal and n_realign.value == int(routes[2]) else 1


if __name__ == "__main__":
    sys.exit(main())
