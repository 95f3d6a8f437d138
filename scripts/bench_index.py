#!/usr/bin/env python
"""bench_index.py — the flat-index build on the host against the build with its minimizer step on the GPU.

  python scripts/bench_index.py [--length 20000000] [--haps 32] [--reps 3] [--out FILE]

Builds one seeded synthetic graph sized like a chromosome arm (vg_b200/synth.py: random backbone, one SNP / insertion /
deletion site per kbp as in config 2, nodes <= 32 bp), takes the flat GBWT of its path-built index, and feeds that GBWT with
the node sequences to gb_index_build_from_gbwt (host) and gb_index_build_from_gbwt_device (GPU 0), alternating, after one
warm-up call of each.  No distance payload is passed, so both routes derive it.  Each call is timed on the host clock
(both calls are synchronous); the builder's own step split (gb_index_build_timing) gives the minimizer step of each route and
how the host route divides between sequences, distance model, GBWT, minimizers and table placement.  The two indexes are
compared array by array and through gb_index_save's file.  Then the reference's y.giraffe.gbz goes end to end through
gb_index_from_gbz and gb_index_from_gbz_device.  Prints one JSON line with the GPU name and power limit; exits non-zero
when any byte differs.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

ARRAYS = ("nodes", "seq", "gbwt", "dist", "slots", "site_dist", "table", "hits")


def gpu_identity():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip()
    name, power = (s.strip() for s in out.split(",", 1))
    return name, power


def identical(a, b, tmp):
    same = all(a.array(n).tobytes() == b.array(n).tobytes() for n in ARRAYS)
    same &= all(getattr(a.view, f) == getattr(b.view, f) for f in ("n_nodes", "k", "w", "n_paths"))
    a.save(tmp / "a.gbflat"); b.save(tmp / "b.gbflat")
    return bool(same and (tmp / "a.gbflat").read_bytes() == (tmp / "b.gbflat").read_bytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--length", type=int, default=20_000_000)
    ap.add_argument("--haps", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=17)
    ap.add_argument("--out", type=Path, default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_index.py measures the device builder: no CUDA device")
    name, power = gpu_identity()
    from vg_b200 import capi, synth

    t0 = time.perf_counter()
    n_var = args.length // 1000
    g = synth.make_variant_graph(length=args.length, n_snp=n_var * 8 // 10, n_ins=n_var // 10, n_del=n_var // 10,
                                 n_haps=args.haps, seed=args.seed)
    ref = capi.HostIndex(g.node_seqs, g.paths, g.dist)
    words, rec_off = ref.array("gbwt").copy(), ref.array("nodes")["rec_off"].copy()
    n_paths = len(g.paths)
    ref.close()
    setup_s = time.perf_counter() - t0

    def call(device):
        t = time.perf_counter()
        ix = capi.HostIndex.from_gbwt(g.node_seqs, n_paths, words, rec_off, None, device=device)
        return time.perf_counter() - t, ix

    for device in (None, 0):                         # warm-up: first CUDA context, module load, allocator
        call(device)[1].close()
    runs = {"host": [], "device": []}
    last = {}
    for _ in range(args.reps):
        for label, device in (("host", None), ("device", 0)):
            s, ix = call(device)
            runs[label].append((s, ix.timing()))
            if label in last:
                last[label].close()
            last[label] = ix
    with tempfile.TemporaryDirectory() as d:
        same = identical(last["host"], last["device"], Path(d))
        gbz = ROOT / "tests" / "golden" / "gbz" / "y.giraffe.gbz"
        yh, yd = capi.HostIndex.from_gbz(gbz, k=29, w=11), capi.HostIndex.from_gbz(gbz, k=29, w=11, device=0)
        y_same = identical(yh, yd, Path(d))
        yh.close(); yd.close()
    counts = {c: int(runs["device"][-1][1][c]) for c in ("start_nodes", "continuations", "raw_pairs", "unique_pairs")}
    counts_agree = all(int(t[c]) == counts[c] for r in runs.values() for _, t in r for c in counts)
    med = lambda xs: round(statistics.median(xs), 4)
    result = {
        "workload": f"synthetic {args.length / 1e6:g} Mbp graph, {n_var} SNP/indel sites, {args.haps} haplotypes, nodes <= 32 bp, "
                    f"k=29 w=11, flat GBWT -> gb_index_build_from_gbwt(_device), distance model derived",
        "gpu": name, "power_limit": power,
        "graph": {"node_ids": len(g.node_seqs), "bases": int(sum(len(s) for s in g.node_seqs)), "gbwt_words": int(len(words))},
        **counts,
        "host_call_s": med([s for s, _ in runs["host"]]),
        "device_call_s": med([s for s, _ in runs["device"]]),
        "host_minimizers_s": med([t["minimizers_s"] for _, t in runs["host"]]),
        "device_minimizers_s": med([t["minimizers_s"] for _, t in runs["device"]]),
        "host_steps_s": {k: med([t[k] for _, t in runs["host"]]) for k in ("sequences_s", "distance_s", "gbwt_s", "minimizers_s", "table_s")},
        "device_steps_s": {k: med([t[k] for _, t in runs["device"]]) for k in ("sequences_s", "distance_s", "gbwt_s", "minimizers_s", "table_s")},
        "host_calls_s": [round(s, 4) for s, _ in runs["host"]],
        "device_calls_s": [round(s, 4) for s, _ in runs["device"]],
        "reps": args.reps, "setup_s": round(setup_s, 1),
        "byte_identical": same, "counts_agree": counts_agree, "y_gbz_byte_identical": y_same,
    }
    for ix in last.values():
        ix.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")
    sys.exit(0 if same and y_same and counts_agree else 1)


if __name__ == "__main__":
    main()
