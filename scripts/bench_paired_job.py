#!/usr/bin/env python
"""bench_paired_job.py — the paired job with a learned fragment-length distribution, on reads in host memory and in HBM.

  python scripts/bench_paired_job.py [--pairs 1000000] [--warmup 1] [--reps 5] [--windows 2048]

bench.py's configs[1] graph and read pairs (its generator and seeds), mapped without a forced distribution.  Times, with
the host clock around the call and a device synchronise:
  host_job     gb_map_paired_job from pinned host buffers (uploads, training windows, downloads)
  device_job   gb_map_paired_job_device on the same reads already in HBM, per training window in --windows
  forced       gb_map_batch_device(paired) on the reads in HBM with the distribution device_job learned, forced
Each call starts from a fresh distribution.  Also reports device_job's training windows and their host-clocked time, and
the GPU name and power limit read in the same run.  Median of --reps after --warmup.  Prints one JSON line; exits non-zero
when the two jobs' records, pools, routes or distributions differ.
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


def timed(fn, warmup, reps, sync):
    for _ in range(warmup):
        fn()
    sync()
    times = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        sync()
        times.append(time.perf_counter() - t)
    return statistics.median(times), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--windows", default="2048")
    args = ap.parse_args()

    import torch
    import bench
    from bench_emit import gpu_identity
    from vg_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_paired_job.py: no CUDA device")
    device = torch.device("cuda", 0)
    g, index = bench.make_graph_and_index()
    dev = capi.Device(index, 0)
    lib = capi.load_library()
    sync = lambda: (torch.cuda.synchronize(), lib.gb_device_synchronize(dev.handle))
    n_pairs = args.pairs
    n = 2 * n_pairs
    L = bench.READ_LEN
    d_reads, d_quals = bench.simulate_pairs_torch(g, n_pairs, 22, device)
    d_reads, d_quals = d_reads.reshape(-1).contiguous(), d_quals.reshape(-1).contiguous()
    d_off = torch.arange(n + 1, dtype=torch.int64, device=device) * L
    h_reads, h_quals, h_off = (t.cpu().pin_memory() for t in (d_reads, d_quals, d_off))
    p = capi.default_map_params()
    p.fragment_mean = 0.0; p.fragment_stdev = 0.0
    map_cap, edit_cap = n * 24, n * 64
    # host job outputs (pinned)
    h_aln = torch.zeros(n * 32, dtype=torch.uint8).pin_memory()
    h_maps = torch.zeros(map_cap * 8, dtype=torch.uint8).pin_memory()
    h_edits = torch.zeros(edit_cap * 4, dtype=torch.uint8).pin_memory()
    h_status = torch.zeros(n, dtype=torch.uint8).pin_memory()
    h_route = torch.zeros(n_pairs, dtype=torch.uint8).pin_memory()
    d_aln = torch.zeros(n * 32, dtype=torch.uint8, device=device)
    d_maps = torch.zeros(map_cap * 8, dtype=torch.uint8, device=device)
    d_edits = torch.zeros(edit_cap * 4, dtype=torch.uint8, device=device)
    d_status = torch.zeros(n, dtype=torch.uint8, device=device)
    d_route = torch.zeros(n_pairs, dtype=torch.uint8, device=device)
    d_tot = torch.zeros(2, dtype=torch.int64, device=device)
    vp = lambda t: C.c_void_p(t.data_ptr())
    state = {}

    def host_job():
        f = capi.FragmentDistribution()
        used = (C.c_uint64(), C.c_uint64())
        rc = lib.gb_map_paired_job(dev.handle, C.byref(p), f._h, 0, n, vp(h_reads), vp(h_quals), vp(h_off), vp(h_aln), vp(h_maps), map_cap,
                                   vp(h_edits), edit_cap, vp(h_status), vp(h_route), C.byref(used[0]), C.byref(used[1]))
        assert rc == capi.GB_OK, lib.gb_last_error()
        state["host"] = (used[0].value, used[1].value, (f.mean(), f.std_dev(), f.curr_sample_size()))
        f.close()

    def device_job(window):
        def run():
            f = capi.FragmentDistribution()
            rc, nm, ne = dev.map_paired_job_device(f, n, d_reads.data_ptr(), d_quals.data_ptr(), d_off.data_ptr(), L, d_aln.data_ptr(),
                                                   d_maps.data_ptr(), map_cap, d_edits.data_ptr(), edit_cap, d_status.data_ptr(),
                                                   d_route.data_ptr(), params=p, training_window=window)
            assert rc == capi.GB_OK, lib.gb_last_error()
            state["device"] = (nm, ne, (f.mean(), f.std_dev(), f.curr_sample_size()))
            state["stats"] = dev.paired_job_stats()
            f.close()
        return run

    host_s, host_t = timed(host_job, args.warmup, args.reps, sync)
    windows = [int(w) for w in args.windows.split(",")]
    dev_results = {}
    for w in windows:
        s, t = timed(device_job(w), args.warmup, args.reps, sync)
        nwin, train_ms = state["stats"]
        dev_results[w] = {"s": s, "ms_min": min(t) * 1e3, "ms_max": max(t) * 1e3, "training_windows": nwin, "training_ms": train_ms}
    nm_h, ne_h, f_h = state["host"]
    nm_d, ne_d, f_d = state["device"]
    same = (f_h == f_d and nm_h == nm_d and ne_h == ne_d and torch.equal(h_aln, d_aln.cpu()) and torch.equal(h_status, d_status.cpu()) and
            torch.equal(h_route, d_route.cpu()) and torch.equal(h_maps[: nm_h * 8], d_maps[: nm_d * 8].cpu()) and
            torch.equal(h_edits[: ne_h * 4], d_edits[: ne_d * 4].cpu()))

    pf = capi.default_map_params()
    pf.fragment_mean, pf.fragment_stdev = f_d[0], f_d[1]

    def forced():
        rc = lib.gb_map_batch_device(dev.handle, C.byref(pf), 1, n, vp(d_reads), vp(d_quals), vp(d_off), L, vp(d_aln), vp(d_maps), map_cap,
                                     vp(d_edits), edit_cap, vp(d_status), vp(d_tot))
        assert rc == capi.GB_OK, lib.gb_last_error()

    forced_s, forced_t = timed(forced, args.warmup, args.reps, sync)
    name, power = gpu_identity()
    w0 = windows[0]
    result = {
        "metric": "paired job with a learned fragment-length distribution: host buffers vs reads in HBM", "gpu": name, "power_limit": power,
        "pairs": n_pairs, "workload": bench.WORKLOAD + "; fragment distribution learned (1000 samples), not forced",
        "host_job_ms": host_s * 1e3, "host_job_ms_min": min(host_t) * 1e3, "host_job_ms_max": max(host_t) * 1e3,
        "device_job_ms": dev_results[w0]["s"] * 1e3,
        "device_job": {str(w): {"ms": r["s"] * 1e3, "ms_min": r["ms_min"], "ms_max": r["ms_max"], "training_windows": r["training_windows"],
                                "training_ms": r["training_ms"]} for w, r in dev_results.items()},
        "forced_device_ms": forced_s * 1e3, "forced_device_ms_min": min(forced_t) * 1e3, "forced_device_ms_max": max(forced_t) * 1e3,
        "learned": {"mean": f_d[0], "stdev": f_d[1], "samples": f_d[2]},
        "host_and_device_jobs_identical": bool(same), "reps": args.reps, "warmup": args.warmup,
    }
    print(json.dumps(result))
    dev.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
