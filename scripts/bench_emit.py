#!/usr/bin/env python
"""bench_emit.py — GAF / GAM emission rate on the GPU against the host emitters, on bench.py's workload.

  python scripts/bench_emit.py [--reads 1000000] [--warmup 2] [--reps 5]

Maps the reads (bench.py's configs[1] generator, 150 bp pairs) with gb_map_batch_device, then times gb_emit_gaf_device and
gb_emit_gam_device on the records in HBM (host clock around the call and a device synchronise, so the sizing pass, its
one wait and the fill are all inside), downloads the records, times gb_emit_gaf / gb_emit_gam on one host core and
compares the two outputs byte for byte over the whole batch.  Then it times gb_bgzf_compress_device on each device output
(same clock), inflates the result and compares it with the host emitter's bytes, and sets its size against gb_bgzf_compress
at level 6 (timed on one host core) and zlib level 1 on the same 0xff00-byte cuts.  Prints one JSON line with the GPU
name and power limit; exits non-zero when any byte differs.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
import time
import zlib
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def gpu_identity():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = (s.strip() for s in out.split(",", 1))
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def bgzf(lib, dev, d_plain, host_plain, args):
    """gb_bgzf_compress_device on the device bytes, against gb_bgzf_compress level 6 and zlib level 1 on the same bytes."""
    import torch
    from vg_b200 import capi
    n_in = d_plain.numel()
    used = C.c_uint64()
    probe = torch.empty(1, dtype=torch.uint8, device=d_plain.device)
    rc = lib.gb_bgzf_compress_device(dev.handle, C.c_void_p(d_plain.data_ptr()), n_in, C.c_void_p(probe.data_ptr()), 0, C.byref(used))
    assert rc == capi.GB_ERR_CAPACITY, rc
    need = used.value
    out = torch.empty(need, dtype=torch.uint8, device=d_plain.device)
    times = []
    for rep in range(args.warmup + args.reps):
        t0 = time.perf_counter()
        rc = lib.gb_bgzf_compress_device(dev.handle, C.c_void_p(d_plain.data_ptr()), n_in, C.c_void_p(out.data_ptr()), need, C.byref(used))
        lib.gb_device_synchronize(dev.handle)
        t1 = time.perf_counter()
        assert rc == capi.GB_OK and used.value == need, rc
        if rep >= args.warmup:
            times.append(t1 - t0)
    sec = statistics.median(times)
    raw = out.cpu().numpy().tobytes()
    rest, parts = raw, []
    while rest:
        d = zlib.decompressobj(31); parts.append(d.decompress(rest)); rest = d.unused_data
    inflated = b"".join(parts)
    m = min(len(inflated), len(host_plain))
    differ = int((np.frombuffer(inflated[:m], np.uint8) != np.frombuffer(host_plain[:m], np.uint8)).sum()) + abs(len(inflated) - len(host_plain))
    src = np.frombuffer(host_plain, dtype=np.uint8)
    cap = len(host_plain) + 128 * (len(host_plain) // 0xff00 + 2)
    hout = np.empty(cap, dtype=np.uint8); hused = C.c_uint64()
    t0 = time.perf_counter()
    rc = lib.gb_bgzf_compress(capi.ptr(src), len(host_plain), 6, capi.ptr(hout), cap, C.byref(hused))
    host_sec = time.perf_counter() - t0
    assert rc == capi.GB_OK, rc
    z1 = 28
    for at in range(0, len(host_plain), 0xff00):
        c = zlib.compressobj(1, zlib.DEFLATED, -15)
        z1 += 26 + len(c.compress(host_plain[at:at + 0xff00]) + c.flush())
    return {"input_gb_per_s": n_in / sec / 1e9, "ms_per_call": sec * 1e3, "ms_min": min(times) * 1e3, "ms_max": max(times) * 1e3,
            "compressed_bytes": need, "ratio": n_in / need, "host_level6_bytes": hused.value, "host_level6_ratio": n_in / hused.value,
            "zlib_level1_bytes": z1, "zlib_level1_ratio": n_in / z1, "size_vs_level6": need / hused.value, "size_vs_level1": need / z1,
            "host_level6_ms_one_core": host_sec * 1e3, "host_level6_mb_per_s": n_in / host_sec / 1e6, "speedup_vs_host_level6": host_sec / sec,
            "bytes_differing": differ}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch
    import bench
    import helpers as H
    from vg_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_emit.py: no CUDA device")
    device = torch.device("cuda", 0)
    g, index = bench.make_graph_and_index()
    dev = capi.Device(index, 0)
    lib = capi.load_library()
    stream = torch.cuda.Stream(device=device)
    torch.cuda.set_stream(stream)
    lib.gb_device_set_stream(dev.handle, C.c_void_p(stream.cuda_stream))
    vp = lambda t: None if t is None else C.c_void_p(t.data_ptr())

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
    torch.cuda.synchronize()
    rc = lib.gb_map_batch_device(dev.handle, C.byref(params), 1, n, vp(d_reads), vp(d_quals), vp(d_off), L, vp(d_aln), vp(d_maps), n * MAP_PER,
                                 vp(d_edits), n * EDIT_PER, vp(d_status), vp(d_tot))
    if rc != capi.GB_OK:
        raise capi.GbError(rc, "gb_map_batch_device")
    lib.gb_device_synchronize(dev.handle)
    tot = [int(x) for x in d_tot.cpu()]

    result = {"metric": "device emission and BGZF compression of alignment records", "reads": n, "workload": bench.WORKLOAD,
              "mapped_fraction": float(((d_aln.view(-1, 32)[:, 9] & 1) != 0).float().mean().item())}
    for kind, fn, host_fn in (("gaf", lib.gb_emit_gaf_device, lib.gb_emit_gaf), ("gam", lib.gb_emit_gam_device, lib.gb_emit_gam)):
        used = C.c_uint64()
        probe = torch.empty(1, dtype=torch.uint8, device=device)
        call = lambda out, cap: fn(dev.handle, n, vp(d_aln), vp(d_maps), tot[0], vp(d_edits), tot[1], n, vp(d_reads), vp(d_quals), vp(d_off),
                                   None, None, vp(out), cap, C.byref(used))
        rc = call(probe, 0)
        assert rc == capi.GB_ERR_CAPACITY, rc
        need = used.value
        out = torch.empty(need, dtype=torch.uint8, device=device)
        times = []
        for rep in range(args.warmup + args.reps):
            t0 = time.perf_counter()
            rc = call(out, need)
            lib.gb_device_synchronize(dev.handle)
            t1 = time.perf_counter()
            assert rc == capi.GB_OK and used.value == need, rc
            if rep >= args.warmup:
                times.append(t1 - t0)
        sec = statistics.median(times)
        dev_bytes = out.cpu().numpy()

        # the host emitter on the same records, downloaded
        aln = d_aln.cpu().numpy().view(capi.alignment_dt).reshape(-1)
        maps = d_maps[: tot[0] + 1].cpu().numpy().view(capi.mapping_dt).reshape(-1)
        edits = d_edits[: tot[1] + 1].cpu().numpy().view(np.uint32)
        rbuf = d_reads.cpu().numpy().reshape(-1); qbuf = d_quals.cpu().numpy().reshape(-1)
        read_off = np.arange(n + 1, dtype=np.uint64) * np.uint64(L)
        host_out = np.zeros(need + (1 << 20), dtype=np.uint8); hused = C.c_uint64()
        t0 = time.perf_counter()
        rc = host_fn(C.byref(index.view), n, capi.ptr(aln), capi.ptr(maps), tot[0], capi.ptr(edits), tot[1], n, capi.ptr(rbuf), capi.ptr(qbuf),
                     capi.ptr(read_off), None, None, capi.ptr(host_out), len(host_out), C.byref(hused))
        host_sec = time.perf_counter() - t0
        assert rc == capi.GB_OK, rc
        host_bytes = host_out[: hused.value]
        m = min(len(host_bytes), len(dev_bytes))
        differ = int((host_bytes[:m] != dev_bytes[:m]).sum()) + abs(len(host_bytes) - len(dev_bytes))
        result[kind] = {"records_per_s": n / sec, "output_gb_per_s": need / sec / 1e9, "ms_per_call": sec * 1e3,
                        "ms_min": min(times) * 1e3, "ms_max": max(times) * 1e3, "bytes": need, "bytes_per_record": need / n,
                        "host_records_per_s": n / host_sec, "speedup_vs_host_core": host_sec / sec,
                        "bytes_differing_from_host": differ}
        result[kind]["bgzf"] = bgzf(lib, dev, out, host_bytes.tobytes(), args)
    name, power = gpu_identity()
    result["gpu"] = name
    result["power_limit"] = power
    result["timing"] = f"host clock around the call + gb_device_synchronize, median of {args.reps} after {args.warmup} warm-up calls"
    print(json.dumps(result))
    dev.close()
    return 0 if all(result[k]["bytes_differing_from_host"] == 0 and result[k]["bgzf"]["bytes_differing"] == 0 for k in ("gaf", "gam")) else 1


if __name__ == "__main__":
    sys.exit(main())
