"""Shared test plumbing: the oracle's ctypes bindings and converters.

The oracle (oracle/liboracle.so) is TEST INFRASTRUCTURE: it is loaded here, by
__graft_entry__.smoke() and by bench.py's CPU legs only.
"""
from __future__ import annotations

import ctypes as C
import json
from pathlib import Path

import numpy as np

from vg_b200 import capi

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"

_oracle = None


def oracle_lib_configure(lib):
    vp, u32 = C.c_void_p, C.c_uint32
    lib.oracle_extend.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), vp, u32, vp, u32, u32,
                                  C.c_double, C.c_int, vp, u32, vp, u32, vp, u32]
    lib.oracle_extend.restype = C.c_int
    lib.oracle_extend_limits.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), vp, u32, vp, u32, u32,
                                         C.c_double, C.c_int, u32, u32, u32, u32, u32, vp, vp]
    lib.oracle_extend_limits.restype = C.c_int
    lib.oracle_bd_state.argtypes = [C.POINTER(capi.FlatIndex), u32, vp]
    lib.oracle_bd_state.restype = C.c_int
    lib.oracle_follow_paths.argtypes = [C.POINTER(capi.FlatIndex), vp, C.c_int, vp, C.c_int]
    lib.oracle_follow_paths.restype = C.c_int
    lib.oracle_xdrop_pinned.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), vp, vp, u32, u32, vp, u32, u32, vp,
                                        vp, u32, vp, vp, u32, vp]
    lib.oracle_xdrop_pinned.restype = C.c_int
    return lib


def oracle_lib() -> C.CDLL:
    global _oracle
    if _oracle is None:
        path = ROOT / "oracle" / "liboracle.so"
        if not path.exists():
            from vg_b200 import build
            build.build_oracle()
        _oracle = oracle_lib_configure(C.CDLL(str(path)))
    return _oracle


def enc(node_id: int, rev: bool) -> int:
    """gbwt::Node::encode."""
    return 2 * node_id + (1 if rev else 0)


def oracle_extend(index: capi.HostIndex, read, seeds, max_mismatches=4, overlap_threshold=0.8, trim=True,
                  scores=None, max_ext=64, path_cap=2048, mism_cap=1024):
    """seeds: iterable of (node, diag).  Returns list of dict extensions (paths/mismatches expanded)."""
    lib = oracle_lib()
    scores = scores or capi.DEFAULT_SCORES
    rb = read.encode() if isinstance(read, str) else bytes(read)
    rbuf = np.frombuffer(rb + b"\0", dtype=np.uint8).copy()
    sd = np.zeros(max(1, len(seeds)), dtype=capi.seed_dt)
    for i, (node, diag) in enumerate(seeds):
        sd[i] = (node, diag)
    ext = np.zeros(max_ext, dtype=capi.extension_dt)
    pp = np.zeros(path_cap, dtype=np.uint32)
    mp = np.zeros(mism_cap, dtype=np.uint32)
    n = lib.oracle_extend(C.byref(index.view), C.byref(scores), capi.ptr(rbuf), len(rb), capi.ptr(sd), len(seeds),
                          max_mismatches, overlap_threshold, 1 if trim else 0, capi.ptr(ext), max_ext,
                          capi.ptr(pp), path_cap, capi.ptr(mp), mism_cap)
    assert n >= 0, "oracle output capacity too small"
    return [expand_extension(ext[i], pp, mp) for i in range(n)]


EXTEND_NEEDS = ("records", "path_nodes", "mismatches", "frontier", "arena")


def oracle_extend_limits(index: capi.HostIndex, read, seeds, q_cap=0xFFFFFFFF, a_cap=0xFFFFFFFF, max_ext=0xFFFFFFFF,
                         path_cap=0xFFFFFFFF, mism_cap=0xFFFFFFFF, max_mismatches=4, overlap_threshold=0.8, trim=True,
                         scores=None):
    """oracle_extend_limits: (GB_ITEM_* status under these capacities, needs dict keyed by EXTEND_NEEDS,
    per-input-seed skip codes: 0 extended, 1 inside the exact full-length extension, 2 invalid)."""
    lib = oracle_lib()
    scores = scores or capi.DEFAULT_SCORES
    rb = read.encode() if isinstance(read, str) else bytes(read)
    rbuf = np.frombuffer(rb + b"\0", dtype=np.uint8).copy()
    sd = np.zeros(max(1, len(seeds)), dtype=capi.seed_dt)
    for i, (node, diag) in enumerate(seeds):
        sd[i] = (node, diag)
    needs = np.zeros(len(EXTEND_NEEDS), dtype=np.uint64)
    skip = np.zeros(max(1, len(seeds)), dtype=np.uint8)
    status = lib.oracle_extend_limits(C.byref(index.view), C.byref(scores), capi.ptr(rbuf), len(rb), capi.ptr(sd), len(seeds),
                                      max_mismatches, overlap_threshold, 1 if trim else 0, q_cap, a_cap, max_ext, path_cap,
                                      mism_cap, capi.ptr(needs), capi.ptr(skip))
    return int(status), dict(zip(EXTEND_NEEDS, (int(x) for x in needs))), skip[:len(seeds)].tolist()


def expand_extension(e, path_pool, mism_pool) -> dict:
    return {
        "path": [int(x) for x in path_pool[int(e["path_off"]): int(e["path_off"]) + int(e["path_len"])]],
        "mismatches": [int(x) for x in mism_pool[int(e["mism_off"]): int(e["mism_off"]) + int(e["mism_len"])]],
        "offset": int(e["offset"]), "read_lo": int(e["read_lo"]), "read_hi": int(e["read_hi"]),
        "score": int(e["score"]), "left_full": bool(e["flags"] & 1), "right_full": bool(e["flags"] & 2),
        "state": tuple(int(e[f]) for f in ("fwd_node", "fwd_lo", "fwd_hi", "bwd_node", "bwd_lo", "bwd_hi")),
        "mismatch_count": int(e["mismatches"]),
    }


def gpu_extensions(ext_count, status, ext, path_pool, mism_pool, max_ext, with_status=False):
    """Expand gb_extend_batch outputs into per-item lists of dict extensions, every status asserted GB_ITEM_OK;
    with_status=True returns per-item (status, extensions) instead, refused items included as they came back."""
    out = []
    for i in range(len(ext_count)):
        if not with_status:
            assert status[i] == capi.GB_ITEM_OK, f"item {i} status {status[i]}"
        exts = [expand_extension(ext[i * max_ext + j], path_pool, mism_pool) for j in range(int(ext_count[i]))]
        out.append((int(status[i]), exts) if with_status else exts)
    return out


def extension_to_mappings(e: dict, node_len, read: str):
    """GaplessExtension::to_path (gbwt_extender.cpp:119-156) as [(node, offset, [(from,to,seq)...])]."""
    res = []
    mm = list(e["mismatches"])
    mi = 0
    read_offset, node_offset = e["read_lo"], e["offset"]
    for h in e["path"]:
        limit = min(read_offset + node_len(h) - node_offset, e["read_hi"])
        edits = []
        while mi < len(mm) and mm[mi] < limit:
            if read_offset < mm[mi]:
                edits.append((mm[mi] - read_offset, mm[mi] - read_offset, ""))
            edits.append((1, 1, read[mm[mi]]))
            read_offset = mm[mi] + 1
            mi += 1
        if read_offset < limit:
            edits.append((limit - read_offset, limit - read_offset, ""))
            read_offset = limit
        res.append((h, node_offset, edits))
        node_offset = 0
    return res


def parse_edit_string(s: str):
    """The reference unit tests' edit syntax (src/unittest/gbwt_extender.cpp:454-496)."""
    edits = []
    i = 0
    while i < len(s):
        c = s[i]
        if "1" <= c <= "9":
            edits.append((int(c), int(c), ""))
        elif c == "-":
            i += 1
            edits.append((int(s[i]), 0, ""))
        elif c == "+":
            i += 1
            n = int(s[i])
            edits.append((0, n, s[i + 1: i + 1 + n]))
            i += n
        else:
            edits.append((1, 1, c))
        i += 1
    return edits


def golden_graph_index(spec, k=29, w=11) -> capi.HostIndex:
    ids = sorted(int(i) for i in spec["nodes"])
    assert ids == list(range(1, len(ids) + 1))
    seqs = [spec["nodes"][str(i)] for i in ids]
    paths = [[enc(n, r) for n, r in thread] for thread in spec["threads"]]
    return capi.HostIndex(seqs, paths, None, k=k, w=w)


def to_seed(node_id, rev, offset, read_offset):
    """GaplessExtender::to_seed (gbwt_extender.hpp:159-162)."""
    return (enc(node_id, rev), int(read_offset) - int(offset))


def load_golden(name):
    return json.loads((GOLDEN / name).read_text())


# ---------------------------------------------------------------------------------------
# mapper-level plumbing
# ---------------------------------------------------------------------------------------
alignment_dt = capi.alignment_dt
mapping_dt = capi.mapping_dt
MapParams = capi.MapParams


COUNTER_NAMES = ["reads", "minimizers", "seeds", "clusters", "extend_calls", "direct", "tail_dps", "tail_cells",
                 "tail_nodes", "tail_bases", "path_nodes", "edits", "rescues"]


def default_map_params() -> MapParams:
    return capi.default_map_params()


def pack_reads(reads, quals=None):
    """reads: uint8 [n, L] array or list of bytes -> (buffer, qual buffer or None, read_off)."""
    if isinstance(reads, np.ndarray) and reads.ndim == 2:
        n, L = reads.shape
        read_off = (np.arange(n + 1, dtype=np.uint64) * np.uint64(L))
        rbuf = np.ascontiguousarray(reads).reshape(-1)
        qbuf = None if quals is None else np.ascontiguousarray(quals).reshape(-1)
        return rbuf, qbuf, read_off
    enc = [r.encode() if isinstance(r, str) else bytes(r) for r in reads]
    read_off = np.zeros(len(enc) + 1, dtype=np.uint64)
    read_off[1:] = np.cumsum([len(r) for r in enc])
    rbuf = np.frombuffer(b"".join(enc) + b"\0", dtype=np.uint8).copy()
    qbuf = None
    if quals is not None:
        qbuf = np.frombuffer(b"".join(bytes(q) for q in quals) + b"\0", dtype=np.uint8).copy()
    return rbuf, qbuf, read_off


def oracle_map(index, reads, quals=None, params=None, scores=None, threads=1):
    lib = oracle_lib()
    lib.oracle_map_batch.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), C.POINTER(MapParams), C.c_uint32,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_int, C.c_void_p]
    lib.oracle_map_batch.restype = C.c_int
    p = params or default_map_params()
    scores = scores or capi.DEFAULT_SCORES
    rbuf, qbuf, read_off = pack_reads(reads, quals)
    n = len(read_off) - 1
    k = max(1, int(p.max_multimaps))
    aln = np.zeros(n * k, dtype=alignment_dt)
    maps = np.zeros(n * k * p.mapping_cap_per_read, dtype=mapping_dt)
    edits = np.zeros(n * k * p.edit_cap_per_read, dtype=np.uint32)
    status = np.zeros(n, dtype=np.uint8)
    counters = np.zeros(len(COUNTER_NAMES), dtype=np.uint64)
    rc = lib.oracle_map_batch(C.byref(index.view), C.byref(scores), C.byref(p), n, capi.ptr(rbuf),
                              capi.ptr(qbuf) if qbuf is not None else None, capi.ptr(read_off), capi.ptr(aln),
                              capi.ptr(maps), capi.ptr(edits), capi.ptr(status), threads, capi.ptr(counters))
    assert rc == 0, "oracle_map_batch: output capacity too small"
    return aln, maps, edits, status, dict(zip(COUNTER_NAMES, (int(c) for c in counters)))


def decode_alignment(a, maps, edits):
    """-> (score, mapq, [(node, offset, [(op, length, base)...])...])"""
    path = []
    e = int(a["edit_off"])
    for i in range(int(a["n_mappings"])):
        m = maps[int(a["mapping_off"]) + i]
        ed = []
        for _ in range(int(m["n_edits"])):
            w = int(edits[e]); e += 1
            ed.append(("MSID"[w & 3], w >> 4, "ACGT"[(w >> 2) & 3] if (w & 3) == 1 else ""))
        path.append((int(m["node"]), int(m["offset"]), ed))
    return int(a["score"]), int(a["mapq"]), path


def gpu_map(dev, reads, quals=None, params=None, paired=False):
    rbuf, qbuf, read_off = pack_reads(reads, quals)
    return dev.map_arrays(rbuf, qbuf, read_off, params, paired=paired)


def compare_alignments(got, want, n, mapq_tol=1, indices=None, k=1):
    """got / want = (aln, maps, edits, status[, counters]).  Scores, paths and edits must be
    identical; MAPQ within +-mapq_tol (FP64 libm differences, BASELINE.json north_star).
    k = max_multimaps: the n * k rank-major records are all compared, and so are their mapped / secondary / absent flags."""
    ga, gm, ge, gs = got[:4]
    wa, wm, we, ws = want[:4]
    bad = []
    which = 1 if k == 1 else (1 | 2 | 16)
    for i in (range(n * k) if indices is None else indices):
        assert gs[i % n] == 0, f"read {i % n}: GPU status {gs[i % n]}"
        assert ws[i % n] == 0
        gd = decode_alignment(ga[i], gm, ge)
        wd = decode_alignment(wa[i], wm, we)
        if gd[0] != wd[0] or gd[2] != wd[2] or abs(gd[1] - wd[1]) > mapq_tol or (ga[i]["flags"] & which) != (wa[i]["flags"] & which) or \
                (k > 1 and int(ga[i]["read_id"]) != int(wa[i]["read_id"])):
            bad.append((i, gd, wd))
    return bad


def oracle_out_buffers(n, p):
    """Pre-touched output buffers for oracle_map*/oracle_map_paired (reusable across calls so a timed
    CPU run does not pay first-touch page faults)."""
    k = max(1, int(p.max_multimaps))
    aln = np.zeros(n * k, dtype=alignment_dt)
    maps = np.zeros(n * k * p.mapping_cap_per_read, dtype=mapping_dt)
    edits = np.zeros(n * k * p.edit_cap_per_read, dtype=np.uint32)
    status = np.zeros(n, dtype=np.uint8)
    for a in (aln, maps, edits, status):
        a.view(np.uint8).reshape(-1)[::4096] = 0
    return aln, maps, edits, status


def oracle_map_paired(index, reads, quals=None, params=None, scores=None, threads=1, out=None):
    """reads interleaved (2i = mate 1, 2i+1 = mate 2)."""
    lib = oracle_lib()
    lib.oracle_map_paired_batch.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), C.POINTER(MapParams), C.c_uint32,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_int, C.c_void_p]
    lib.oracle_map_paired_batch.restype = C.c_int
    p = params
    scores = scores or capi.DEFAULT_SCORES
    rbuf, qbuf, read_off = pack_reads(reads, quals)
    n = len(read_off) - 1
    aln, maps, edits, status = out if out is not None else oracle_out_buffers(n, p)
    counters = np.zeros(len(COUNTER_NAMES), dtype=np.uint64)
    rc = lib.oracle_map_paired_batch(C.byref(index.view), C.byref(scores), C.byref(p), n, capi.ptr(rbuf),
                                     capi.ptr(qbuf) if qbuf is not None else None, capi.ptr(read_off), capi.ptr(aln),
                                     capi.ptr(maps), capi.ptr(edits), capi.ptr(status), threads, capi.ptr(counters))
    assert rc == 0, f"oracle_map_paired_batch rc {rc}"
    return aln[:n * max(1, int(p.max_multimaps))], maps, edits, status[:n], dict(zip(COUNTER_NAMES, (int(c) for c in counters)))


def paired_params(mean=400.0, stdev=50.0):
    p = default_map_params()
    p.fragment_mean = mean
    p.fragment_stdev = stdev
    p.max_rescue_attempts = 0
    return p


def oracle_fragment_estimate(lengths, maximum_sample_size=1000, reestimation_frequency=1000, fraction=0.95):
    """Register `lengths` in order in the oracle's FragmentLengthDistribution; (mean, stdev, finalized, samples)."""
    lib = oracle_lib()
    lib.oracle_fragment_estimate.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_double, C.POINTER(C.c_double),
                                             C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
    lib.oracle_fragment_estimate.restype = None
    arr = np.ascontiguousarray(lengths, dtype=np.int64)
    mean, sd, fin, n = C.c_double(), C.c_double(), C.c_int(), C.c_uint64()
    lib.oracle_fragment_estimate(capi.ptr(arr), len(arr), maximum_sample_size, reestimation_frequency, fraction,
                                 C.byref(mean), C.byref(sd), C.byref(fin), C.byref(n))
    return mean.value, sd.value, bool(fin.value), int(n.value)


def oracle_map_paired_job(index, reads, quals, params, maximum_sample_size=1000, reestimation_frequency=1000, fraction=0.95, threads=1):
    """giraffe_main's paired job on the CPU: training, map_paired, ambiguous buffer.
    Returns (aln, maps, edits, status, route, (mean, stdev, samples))."""
    lib = oracle_lib()
    lib.oracle_map_paired_job.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), C.POINTER(MapParams), C.c_uint64, C.c_uint64,
                                          C.c_double, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.oracle_map_paired_job.restype = C.c_int
    p = params
    rbuf, qbuf, read_off = pack_reads(reads, quals)
    n = len(read_off) - 1
    aln, maps, edits, status = oracle_out_buffers(n, p)
    route = np.zeros(n // 2, dtype=np.uint8)
    frag = np.zeros(3, dtype=np.float64)
    rc = lib.oracle_map_paired_job(C.byref(index.view), C.byref(capi.DEFAULT_SCORES), C.byref(p), maximum_sample_size, reestimation_frequency, fraction,
                                   n, capi.ptr(rbuf), capi.ptr(qbuf) if qbuf is not None else None, capi.ptr(read_off), capi.ptr(aln),
                                   capi.ptr(maps), capi.ptr(edits), capi.ptr(status), capi.ptr(route), threads, capi.ptr(frag))
    assert rc == 0, f"oracle_map_paired_job rc {rc}"
    return aln, maps, edits, status, route, (float(frag[0]), float(frag[1]), int(frag[2]))


def oracle_seed_stage(index, reads, quals=None, params=None, paired=False, scores=None):
    """The oracle's stage dump (oracle_seed_stage in oracle/mapper_paired.cpp), same layout as Device.seed_stage."""
    lib = oracle_lib()
    vp, u64 = C.c_void_p, C.c_uint64
    lib.oracle_seed_stage.argtypes = [C.POINTER(capi.FlatIndex), C.POINTER(capi.Scores), C.POINTER(MapParams), C.c_int, C.c_uint32, vp, vp, vp,
                                      vp, vp, u64, vp, u64, vp, u64, vp, u64, vp, u64]
    lib.oracle_seed_stage.restype = C.c_int
    p = params or default_map_params()
    scores = scores or capi.DEFAULT_SCORES
    rbuf, qbuf, read_off = pack_reads(reads, quals)
    n = len(read_off) - 1
    outs = capi.stage_buffers(n)
    rc = lib.oracle_seed_stage(C.byref(index.view), C.byref(scores), C.byref(p), 1 if paired else 0, n, capi.ptr(rbuf), capi.ptr(qbuf) if qbuf is not None else None,
                               capi.ptr(read_off), capi.ptr(outs[0]), capi.ptr(outs[1]), len(outs[1]), capi.ptr(outs[2]), len(outs[2]), capi.ptr(outs[3]), len(outs[3]),
                               capi.ptr(outs[4]), len(outs[4]), capi.ptr(outs[5]), len(outs[5]))
    assert rc == 0, "oracle stage dump: capacity"
    return outs


def compare_stage_dumps(got, want, n):
    """Field-by-field, bit-exact (scores and coverages are IEEE doubles built from the same host tables).
    Returns a list of (read, stage, detail) for the first difference of each read."""
    bad = []
    gr, gm, gs, gc, gi, ge = got
    wr, wm, ws, wc, wi, we = want
    for r in range(n):
        a, b = gr[r], wr[r]
        if int(a["status"]) != 0:
            bad.append((r, "status", int(a["status"]))); continue
        deferred = int(a["reserved"][0]) > 1          # mate 2 with tied clusters: selection happens in the align stage (see giraffe_b200.h)
        for stage, cnt in (("a1 minimizer count", "min_cnt"), ("a3 seed count", "seed_cnt"), ("a4 cluster count", "cluster_cnt"), ("a6 item count", "item_cnt")):
            if deferred and cnt == "item_cnt":
                continue
            if int(a[cnt]) != int(b[cnt]):
                bad.append((r, stage, (int(a[cnt]), int(b[cnt])))); break
        else:
            x = gm[int(a["min_off"]): int(a["min_off"]) + int(a["min_cnt"])]; y = wm[int(b["min_off"]): int(b["min_off"]) + int(b["min_cnt"])]
            if x.tobytes() != y.tobytes():
                # a1 = which minimizers (as a set), a2 = their order after the score sort and tie shuffle
                same_set = sorted(x.tolist()) == sorted(y.tolist())
                bad.append((r, "a2 minimizer order" if same_set else "a1 minimizers", None)); continue
            x = gs[int(a["seed_off"]): int(a["seed_off"]) + int(a["seed_cnt"])]; y = ws[int(b["seed_off"]): int(b["seed_off"]) + int(b["seed_cnt"])]
            if any(x[f].tobytes() != y[f].tobytes() for f in ("node", "offset", "source")):
                bad.append((r, "a3 seeds", None)); continue
            if (x["cluster"] != y["cluster"]).any():
                bad.append((r, "a4 cluster membership", None)); continue
            x = gc[int(a["cluster_off"]): int(a["cluster_off"]) + int(a["cluster_cnt"])]; y = wc[int(b["cluster_off"]): int(b["cluster_off"]) + int(b["cluster_cnt"])]
            if any(x[f].tobytes() != y[f].tobytes() for f in ("score", "coverage", "first_seed", "n_seeds")):
                bad.append((r, "a5 cluster score / coverage", (x.tolist(), y.tolist()))); continue
            if (x["fragment"] != y["fragment"]).any():
                bad.append((r, "a19 fragment clusters", (x["fragment"].tolist(), y["fragment"].tolist()))); continue
            if deferred:
                # every cluster is listed once, in comparator order; the clusters the oracle kept are among them
                if sorted(x["kept_rank"].tolist()) != list(range(len(x))) or int(a["item_cnt"]) != len(x):
                    bad.append((r, "a6 deferred selection lists every cluster", x["kept_rank"].tolist()))
                continue
            if (x["kept_rank"] != y["kept_rank"]).any():
                bad.append((r, "a6 cluster selection / order", (x["kept_rank"].tolist(), y["kept_rank"].tolist()))); continue
            x = gi[int(a["item_off"]): int(a["item_off"]) + int(a["item_cnt"])]; y = wi[int(b["item_off"]): int(b["item_off"]) + int(b["item_cnt"])]
            if (x["cluster"] != y["cluster"]).any() or (x["fragment"] != y["fragment"]).any() or (x["seed_cnt"] != y["seed_cnt"]).any():
                bad.append((r, "a7 work items", None)); continue
            for t in range(len(x)):
                sx = ge[int(x[t]["seed_off"]): int(x[t]["seed_off"]) + int(x[t]["seed_cnt"])]; sy = we[int(y[t]["seed_off"]): int(y[t]["seed_off"]) + int(y[t]["seed_cnt"])]
                if sx.tobytes() != sy.tobytes():
                    bad.append((r, "a7 item seeds (node, diagonal)", t)); break
    return bad
