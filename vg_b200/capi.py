"""ctypes bindings for libgiraffe_b200.so (include/giraffe_b200.h).

Python is used here the way torch is used in this repo: plumbing for tests, the benchmark
and data generation.  The product is the shared library; this module only calls it.
There is no Python or CPU implementation of any hot-path stage in this package.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
LIB_PATH = ROOT / "vg_b200" / "libgiraffe_b200.so"

GB_OK = 0
GB_ERR_ARG, GB_ERR_CUDA, GB_ERR_NO_DEVICE, GB_ERR_CAPACITY, GB_ERR_FORMAT = -1, -2, -3, -4, -5
GB_ITEM_OK, GB_ITEM_QUEUE_FULL, GB_ITEM_OUT_FULL, GB_ITEM_DP_REFUSED = 0, 1, 2, 3
GB_ITEM_NO_BAND = 4
GB_EXT_LEFT_FULL, GB_EXT_RIGHT_FULL = 1, 2
GB_ALN_MAPPED, GB_ALN_SECONDARY, GB_ALN_PAIRED, GB_ALN_RESCUED, GB_ALN_ABSENT = 1, 2, 4, 8, 16
GB_MAX_MULTIMAPS = 8

# numpy mirrors of the ABI structs
node_rec_dt = np.dtype([("seq_off", "<u4"), ("rec_off", "<u4"), ("len", "<u4"), ("size", "<u4")])
dist_dt = np.dtype([("x_in", "<i4"), ("x_out", "<i4"), ("slot", "<u4"), ("allele", "<u2"), ("component", "<u2")])
min_cell_dt = np.dtype([("key", "<u8"), ("hit_off", "<u4"), ("hit_cnt", "<u4")])
hit_dt = np.dtype([("pos", "<u8"), ("payload", dist_dt)])
slot_dt = np.dtype([("table_off", "<u4"), ("n", "<u4")])
seed_dt = np.dtype([("node", "<u4"), ("diag", "<i4")])
extension_dt = np.dtype([
    ("path_off", "<u4"), ("path_len", "<u4"), ("mism_off", "<u4"), ("mism_len", "<u4"),
    ("offset", "<u4"), ("read_lo", "<u4"), ("read_hi", "<u4"), ("score", "<i4"), ("flags", "<u4"),
    ("fwd_node", "<u4"), ("fwd_lo", "<u4"), ("fwd_hi", "<u4"),
    ("bwd_node", "<u4"), ("bwd_lo", "<u4"), ("bwd_hi", "<u4"), ("mismatches", "<u4"),
])
assert node_rec_dt.itemsize == 16 and dist_dt.itemsize == 16 and min_cell_dt.itemsize == 16
assert hit_dt.itemsize == 24 and seed_dt.itemsize == 8 and extension_dt.itemsize == 64


class FlatIndex(C.Structure):
    _fields_ = [
        ("n_nodes", C.c_uint32), ("k", C.c_uint32), ("w", C.c_uint32), ("n_paths", C.c_uint32),
        ("nodes", C.c_void_p),
        ("seq", C.c_void_p), ("seq_bytes", C.c_uint64),
        ("gbwt", C.c_void_p), ("gbwt_words", C.c_uint64),
        ("dist", C.c_void_p),
        ("table", C.c_void_p), ("table_cells", C.c_uint64),
        ("hits", C.c_void_p), ("n_hits", C.c_uint64),
        ("slots", C.c_void_p), ("n_slots", C.c_uint64),
        ("site_dist", C.c_void_p), ("site_dist_len", C.c_uint64),
    ]


class Scores(C.Structure):
    _fields_ = [("match", C.c_int8), ("mismatch", C.c_int8), ("gap_open", C.c_int8),
                ("gap_extend", C.c_int8), ("full_length_bonus", C.c_int8)]


class ChainParams(C.Structure):
    _fields_ = [("item_bonus", C.c_int32), ("recombination_penalty", C.c_int32), ("consistency_bonus", C.c_int32),
                ("max_chains", C.c_uint32), ("gap_scale", C.c_double), ("max_indel_bases", C.c_uint64),
                ("max_read_lookback_bases", C.c_uint64)]


chain_anchor_dt = np.dtype([("read_start", "<u4"), ("length", "<u4"), ("margin_before", "<u4"), ("margin_after", "<u4"),
                            ("score", "<i4"), ("start_hint_offset", "<u4"), ("end_hint_offset", "<u4"), ("base_seed_length", "<u4"),
                            ("start_paths", "<u8"), ("end_paths", "<u8")])
chain_candidate_dt = np.dtype([("from", "<u4"), ("to", "<u4"), ("graph_distance", "<u8")])


class ExtendParams(C.Structure):
    _fields_ = [("max_mismatches", C.c_uint32), ("overlap_threshold", C.c_double), ("trim", C.c_uint32),
                ("max_ext_per_item", C.c_uint32), ("path_cap_per_item", C.c_uint32),
                ("mism_cap_per_item", C.c_uint32)]


DEFAULT_SCORES = Scores(1, 4, 6, 1, 5)

alignment_dt = np.dtype([("read_id", "<u4"), ("score", "<i4"), ("mapq", "u1"), ("flags", "u1"), ("n_mappings", "<u2"),
                         ("mapping_off", "<u4"), ("edit_off", "<u4"), ("n_edits", "<u4"),
                         ("mapq_uncapped", "<f4"), ("mapq_explored_cap", "<f4")])
mapping_dt = np.dtype([("node", "<u4"), ("offset", "<u2"), ("n_edits", "<u2")])
# gb_debug_seed_stage records
stage_minimizer_dt = np.dtype([("hash", "<u8"), ("score", "<f8"), ("fwd_offset", "<u4"), ("agg_start", "<u4"), ("agg_len", "<u4"), ("is_reverse", "<u4"), ("hits", "<u4"), ("reserved", "<u4")])
stage_seed_dt = np.dtype([("node", "<u4"), ("offset", "<u4"), ("source", "<u4"), ("cluster", "<u4")])
stage_cluster_dt = np.dtype([("score", "<f8"), ("coverage", "<f8"), ("first_seed", "<u4"), ("n_seeds", "<u4"), ("fragment", "<u4"), ("kept_rank", "<u4")])
stage_item_dt = np.dtype([("cluster", "<u4"), ("fragment", "<u4"), ("seed_off", "<u4"), ("seed_cnt", "<u4")])
stage_read_dt = np.dtype([("min_off", "<u4"), ("min_cnt", "<u4"), ("seed_off", "<u4"), ("seed_cnt", "<u4"), ("cluster_off", "<u4"), ("cluster_cnt", "<u4"),
                          ("item_off", "<u4"), ("item_cnt", "<u4"), ("status", "<u4"), ("reserved", "<u4", (3,))])
assert alignment_dt.itemsize == 32 and mapping_dt.itemsize == 8


class MapParams(C.Structure):
    """gb_map_params (include/giraffe_b200.h)."""
    _fields_ = [
        ("hit_cap", C.c_uint32), ("hard_hit_cap", C.c_uint32), ("minimizer_score_fraction", C.c_double),
        ("minimizer_coverage_flank", C.c_uint32), ("max_unique_min", C.c_uint32), ("num_bp_per_min", C.c_uint32),
        ("distance_limit", C.c_uint32), ("min_extensions", C.c_uint32), ("max_extensions", C.c_uint32),
        ("cluster_score_threshold", C.c_double), ("pad_cluster_score_threshold", C.c_double),
        ("cluster_coverage_threshold", C.c_double), ("extension_set_score_threshold", C.c_double),
        ("extension_score_threshold", C.c_int32), ("min_extension_sets", C.c_int32),
        ("extension_set_min_score", C.c_int32), ("max_alignments", C.c_uint32),
        ("max_extension_mismatches", C.c_uint32), ("max_multimaps", C.c_uint32), ("max_dozeu_cells", C.c_uint32),
        ("do_dp", C.c_uint32),
        ("fragment_mean", C.c_double), ("fragment_stdev", C.c_double), ("paired_distance_stdevs", C.c_double),
        ("paired_rescue_score_limit", C.c_double), ("rescue_subgraph_stdevs", C.c_double),
        ("max_rescue_attempts", C.c_uint32), ("max_fragment_length", C.c_uint32),
        ("rescue_seed_limit", C.c_uint32), ("reserved0", C.c_uint32), ("rescue_likelihood_limit", C.c_double),
        ("mapping_cap_per_read", C.c_uint32), ("edit_cap_per_read", C.c_uint32),
    ]


def default_map_params() -> "MapParams":
    p = MapParams()
    load_library().gb_map_params_default(C.byref(p))
    return p


_lib = None


def load_library() -> C.CDLL:
    """Load libgiraffe_b200.so; raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("GIRAFFE_B200_LIB", LIB_PATH))      # another build of the same library (kernel A/B runs)
    if not path.exists():
        raise RuntimeError(f"{path} is missing: run `python -m vg_b200.build` (there is no fallback path)")
    lib = C.CDLL(str(path))
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    lib.gb_index_build.argtypes = [u32, vp, vp, u32, vp, vp, vp, u32, u32, C.POINTER(vp)]
    lib.gb_index_build.restype = C.c_int
    lib.gb_index_free.argtypes = [vp]
    lib.gb_index_free.restype = None
    lib.gb_index_view.argtypes = [vp, C.POINTER(FlatIndex)]
    lib.gb_index_view.restype = C.c_int
    lib.gb_device_create.argtypes = [C.POINTER(FlatIndex), C.c_int, C.POINTER(vp)]
    lib.gb_device_create.restype = C.c_int
    lib.gb_device_destroy.argtypes = [vp]
    lib.gb_device_destroy.restype = None
    lib.gb_last_error.argtypes = []
    lib.gb_last_error.restype = C.c_char_p
    lib.gb_index_from_gbz.argtypes = [C.c_char_p, u32, u32, vp]
    lib.gb_index_from_gbz.restype = C.c_int
    lib.gb_index_from_gbz_min.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, vp]
    lib.gb_index_from_gbz_min.restype = C.c_int
    lib.gb_index_build_with_hits.argtypes = [u32, vp, vp, u32, vp, vp, vp, u32, u32, u64, vp, vp, vp]
    lib.gb_index_build_with_hits.restype = C.c_int
    lib.gb_index_build_from_gbwt.argtypes = [u32, vp, vp, u32, vp, u64, vp, vp, u32, u32, u64, vp, vp, vp]
    lib.gb_index_build_from_gbwt.restype = C.c_int
    lib.gb_index_save.argtypes = [C.POINTER(FlatIndex), C.c_char_p]
    lib.gb_index_save.restype = C.c_int
    lib.gb_index_load.argtypes = [C.c_char_p, vp]
    lib.gb_index_load.restype = C.c_int
    lib.gb_set_scores.argtypes = [vp, C.POINTER(Scores)]
    lib.gb_set_scores.restype = C.c_int
    lib.gb_extend_batch.argtypes = [vp, C.POINTER(ExtendParams), u32, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.gb_extend_batch.restype = C.c_int
    lib.gb_map_params_default.argtypes = [C.POINTER(MapParams)]
    lib.gb_map_params_default.restype = None
    lib.gb_map_batch.argtypes = [vp, C.POINTER(MapParams), u32, vp, vp, vp, vp, vp, u64, vp, u64, vp, vp, vp]
    lib.gb_map_batch.restype = C.c_int
    lib.gb_map_paired_batch.argtypes = [vp, C.POINTER(MapParams), u32, vp, vp, vp, vp, vp, u64, vp, u64, vp, vp, vp]
    lib.gb_map_batch_device.argtypes = [vp, C.POINTER(MapParams), C.c_int, u32, vp, vp, vp, u32, vp, vp, u64, vp, u64, vp, vp]
    lib.gb_map_batch_device.restype = C.c_int
    lib.gb_device_set_stream.argtypes = [vp, vp]
    lib.gb_device_set_stream.restype = C.c_int
    lib.gb_device_synchronize.argtypes = [vp]
    lib.gb_device_synchronize.restype = C.c_int
    lib.gb_stage_times.argtypes = [vp, vp]
    lib.gb_stage_times.restype = C.c_int
    lib.gb_map_paired_batch.restype = C.c_int
    lib.gb_xdrop_pinned_batch.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp, vp, u32, u32, vp, vp, vp, vp, vp, vp]
    lib.gb_xdrop_pinned_batch.restype = C.c_int
    lib.gb_sw_batch.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp, u32, u32, vp, vp, vp, vp, vp, vp]
    lib.gb_sw_batch.restype = C.c_int
    lib.gb_banded_global_batch.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp, vp, vp, u32, u32, vp, vp, vp, vp, vp, vp]
    lib.gb_banded_global_batch.restype = C.c_int
    lib.gb_xdrop_dag_batch.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp, vp, vp, u32, u32, vp, vp, vp, vp, vp, vp]
    lib.gb_xdrop_dag_batch.restype = C.c_int
    lib.gb_wfa_batch.argtypes = [vp, u32, vp, vp, vp, vp, vp, u32, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.gb_wfa_batch.restype = C.c_int
    lib.gb_chain_params_default.argtypes = [C.POINTER(ChainParams)]
    lib.gb_chain_params_default.restype = None
    lib.gb_chain_batch.argtypes = [vp, C.POINTER(ChainParams), u32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.gb_chain_batch.restype = C.c_int
    lib.gb_chain_batch_transitions.argtypes = [vp, C.POINTER(ChainParams), u32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.gb_chain_batch_transitions.restype = C.c_int
    lib.gb_chain_anchors.argtypes = [C.POINTER(FlatIndex), C.POINTER(Scores), u32, vp, vp, vp, vp, vp, vp]
    lib.gb_chain_anchors.restype = C.c_int
    lib.gb_chain_candidates_batch.argtypes = [vp, u32, vp, vp, u64, vp, u64, vp]
    lib.gb_chain_candidates_batch.restype = C.c_int
    lib.gb_fragment_create.argtypes = [u64, u64, C.c_double]
    lib.gb_fragment_create.restype = vp
    lib.gb_fragment_destroy.argtypes = [vp]
    lib.gb_fragment_destroy.restype = None
    lib.gb_fragment_force.argtypes = [vp, C.c_double, C.c_double]
    lib.gb_fragment_force.restype = None
    lib.gb_fragment_register.argtypes = [vp, C.c_int64]
    lib.gb_fragment_register.restype = None
    lib.gb_fragment_finalize.argtypes = [vp]
    lib.gb_fragment_finalize.restype = None
    lib.gb_fragment_mean.argtypes = [vp]
    lib.gb_fragment_mean.restype = C.c_double
    lib.gb_fragment_stdev.argtypes = [vp]
    lib.gb_fragment_stdev.restype = C.c_double
    lib.gb_fragment_is_finalized.argtypes = [vp]
    lib.gb_fragment_is_finalized.restype = C.c_int
    lib.gb_fragment_sample_size.argtypes = [vp]
    lib.gb_fragment_sample_size.restype = u64
    lib.gb_map_paired_job.argtypes = [vp, C.POINTER(MapParams), vp, u32, u32, vp, vp, vp, vp, vp, u64, vp, u64, vp, vp, vp, vp]
    lib.gb_map_paired_job.restype = C.c_int
    for fn in (lib.gb_emit_gaf, lib.gb_emit_json, lib.gb_emit_gam):
        fn.argtypes = [C.POINTER(FlatIndex), u32, vp, vp, u64, vp, u64, u32, vp, vp, vp, vp, vp, vp, u64, vp]
        fn.restype = C.c_int
    lib.gb_debug_seed_stage.argtypes = [vp, C.POINTER(MapParams), C.c_int, u32, vp, vp, vp, vp, vp, u64, vp, u64, vp, u64, vp, u64, vp, u64]
    lib.gb_debug_seed_stage.restype = C.c_int
    lib.gb_device_pool_overflow.argtypes = [vp, C.POINTER(C.c_int)]
    lib.gb_device_pool_overflow.restype = C.c_int
    lib.gb_kernel_times.argtypes = [vp, u32, vp, vp, vp]
    lib.gb_kernel_times.restype = C.c_int
    lib.gb_device_set_output_mirror.argtypes = [vp, vp, vp, u64, vp, u64]
    lib.gb_device_set_output_mirror.restype = C.c_int
    lib.gb_plan_stats.argtypes = [vp, vp]
    lib.gb_plan_stats.restype = C.c_int
    lib.gb_bgzf_compress.argtypes = [vp, u64, C.c_int, vp, u64, vp]
    lib.gb_bgzf_compress.restype = C.c_int
    lib.gb_last_kernel_ms.argtypes = [vp]
    lib.gb_last_kernel_ms.restype = C.c_float
    lib.gb_launch_count.argtypes = [vp]
    lib.gb_launch_count.restype = C.c_uint64
    _lib = lib
    return lib


def ptr(a: np.ndarray) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data)


def decode_path(maps, edits, n_maps, node_offset=0):
    """The first n_maps mappings of maps and their edit words, which start at edits[0], as
    [[node + node_offset, offset, [[op, length, base], ...]], ...] (base only on substitutions)."""
    path, e = [], 0
    for k in range(int(n_maps)):
        m = maps[k]
        ed = []
        for _ in range(int(m["n_edits"])):
            w = int(edits[e]); e += 1
            ed.append(["MSID"[w & 3], w >> 4, "ACGT"[(w >> 2) & 3] if (w & 3) == 1 else ""])
        path.append([int(m["node"]) + node_offset, int(m["offset"]), ed])
    return path


def _pack_dags(problems):
    """DAG problems (nodes, preds, query bytes, ...) as the seams' CSR arrays: node, node_off, pred, pred_off, query, query_off."""
    n = len(problems)
    node_off = np.zeros(n + 1, dtype=np.uint64)
    node_off[1:] = np.cumsum([len(p[0]) for p in problems])
    query_off = np.zeros(n + 1, dtype=np.uint64)
    query_off[1:] = np.cumsum([len(p[2]) for p in problems])
    nodes = np.concatenate([np.asarray(p[0], dtype=np.uint32) for p in problems])
    pred = np.asarray([x for p in problems for ps in p[1] for x in ps] + [0], dtype=np.uint32)
    pred_off = np.zeros(len(nodes) + 1, dtype=np.uint64)
    pred_off[1:] = np.cumsum([len(ps) for p in problems for ps in p[1]])
    q = np.frombuffer(b"".join(bytes(p[2]) for p in problems) + b"\0", dtype=np.uint8).copy()
    return nodes, node_off, pred, pred_off, q, query_off


def _seam_outputs(n, map_cap, edit_cap):
    """The output arrays of a batched alignment seam: score, maps, edits, n_maps, n_edits, status."""
    return (np.zeros(n, dtype=np.int32), np.zeros(n * map_cap, dtype=mapping_dt), np.zeros(n * edit_cap, dtype=np.uint32),
            np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8))


def _dag_seam_results(outs, map_cap, with_status):
    """The per-problem (score, path) of gb_sw_batch / gb_xdrop_dag_batch, every status asserted GB_ITEM_OK, or with
    with_status (status, score, path) with the path decoded from the returned counts whatever the status."""
    score, maps, edits, nm, _, status = outs
    edit_cap = len(edits) // len(score)
    res = []
    for i in range(len(score)):
        path = decode_path(maps[i * map_cap:], edits[i * edit_cap:], min(int(nm[i]), map_cap))
        if with_status:
            res.append((int(status[i]), int(score[i]), path))
        else:
            assert status[i] == GB_ITEM_OK, f"problem {i}: status {status[i]}"
            res.append((int(score[i]), path))
    return res


class GbError(RuntimeError):
    def __init__(self, code: int, what: str):
        msg = load_library().gb_last_error()
        super().__init__(f"{what} failed with status {code}: {msg.decode() if msg else ''}")
        self.code = code


class HostIndex:
    """Owns a gb_host_index built by the library from node sequences and haplotype paths."""

    def __init__(self, node_seqs, paths, dist=None, k=29, w=11, hits=None):
        """hits = (keys, positions): the minimizer table is taken from the caller (gb_index_build_with_hits)."""
        lib = load_library()
        n = len(node_seqs)
        node_off = np.zeros(n + 1, dtype=np.uint64)
        node_off[1:] = np.cumsum([len(s) for s in node_seqs])
        seq = np.frombuffer("".join(node_seqs).encode(), dtype=np.uint8).copy() if n else np.zeros(1, np.uint8)
        path_off = np.zeros(len(paths) + 1, dtype=np.uint64)
        path_off[1:] = np.cumsum([len(p) for p in paths])
        flat = np.concatenate([np.asarray(p, dtype=np.uint32) for p in paths]) if paths else np.zeros(1, np.uint32)
        flat = np.ascontiguousarray(flat, dtype=np.uint32)
        dptr = None
        if dist is not None:
            dist = np.ascontiguousarray(dist, dtype=dist_dt)
            assert len(dist) == n + 1, "dist payload is indexed by node id (entry 0 unused)"
            dptr = ptr(dist)
        h = C.c_void_p()
        if hits is None:
            rc = lib.gb_index_build(n, ptr(seq), ptr(node_off), len(paths), ptr(flat), ptr(path_off), dptr, k, w, C.byref(h))
        else:
            hk, hp = (np.ascontiguousarray(a, dtype=np.uint64) for a in hits)
            assert len(hk) == len(hp)
            rc = lib.gb_index_build_with_hits(n, ptr(seq), ptr(node_off), len(paths), ptr(flat), ptr(path_off), dptr, k, w,
                                              len(hk), ptr(hk), ptr(hp), C.byref(h))
        if rc != GB_OK:
            raise GbError(rc, "gb_index_build")
        self._h = h
        self.view = FlatIndex()
        rc = lib.gb_index_view(h, C.byref(self.view))
        if rc != GB_OK:
            raise GbError(rc, "gb_index_view")
        self.node_seqs = list(node_seqs)
        self.paths = [list(p) for p in paths]
        self.k, self.w = k, w

    def save(self, path):
        """gb_index_save: the flat index as one file."""
        rc = load_library().gb_index_save(C.byref(self.view), str(path).encode())
        if rc != GB_OK:
            raise GbError(rc, "gb_index_save")

    @classmethod
    def from_gbz(cls, path, k=29, w=11):
        """gb_index_from_gbz: the flat index of a GBZ file (graphs that are chains of bubbles)."""
        lib = load_library()
        h = C.c_void_p()
        rc = lib.gb_index_from_gbz(str(path).encode(), k, w, C.byref(h))
        if rc != GB_OK:
            raise GbError(rc, "gb_index_from_gbz")
        self = cls.__new__(cls)
        self._h = h
        self.view = FlatIndex()
        rc = lib.gb_index_view(h, C.byref(self.view))
        if rc != GB_OK:
            raise GbError(rc, "gb_index_view")
        self.node_seqs, self.paths = None, None
        self.k, self.w = k, w
        return self

    @classmethod
    def from_gbwt(cls, node_seqs, n_paths, gbwt_words, rec_off, dist=None, k=29, w=11, hits=None):
        """gb_index_build_from_gbwt: node sequences + a flat GBWT (gb_flat_index blob layout) instead of haplotype paths."""
        lib = load_library()
        n = len(node_seqs)
        node_off = np.zeros(n + 1, dtype=np.uint64)
        node_off[1:] = np.cumsum([len(s) for s in node_seqs])
        seq = np.frombuffer("".join(node_seqs).encode(), dtype=np.uint8).copy() if n else np.zeros(1, np.uint8)
        words = np.ascontiguousarray(gbwt_words, dtype=np.uint32); ro = np.ascontiguousarray(rec_off, dtype=np.uint32)
        dptr = None
        if dist is not None:
            dist = np.ascontiguousarray(dist, dtype=dist_dt); dptr = ptr(dist)
        hk = hp = None
        if hits is not None:
            hk, hp = (np.ascontiguousarray(a, dtype=np.uint64) for a in hits)
        h = C.c_void_p()
        rc = lib.gb_index_build_from_gbwt(n, ptr(seq), ptr(node_off), n_paths, ptr(words), len(words), ptr(ro), dptr, k, w,
                                          0 if hk is None else len(hk), None if hk is None else ptr(hk), None if hp is None else ptr(hp), C.byref(h))
        if rc != GB_OK:
            raise GbError(rc, "gb_index_build_from_gbwt")
        self = cls.__new__(cls)
        self._h = h
        self.view = FlatIndex()
        rc = lib.gb_index_view(h, C.byref(self.view))
        if rc != GB_OK:
            raise GbError(rc, "gb_index_view")
        self.node_seqs, self.paths = list(node_seqs), None
        self.k, self.w = k, w
        return self

    @classmethod
    def from_gbz_min(cls, gbz, min_path, zipcodes=None):
        """gb_index_from_gbz_min: GBZ + the .min (and .zipcodes) files giraffe loads beside it; k and w come from the .min."""
        lib = load_library()
        h = C.c_void_p()
        rc = lib.gb_index_from_gbz_min(str(gbz).encode(), str(min_path).encode(), str(zipcodes).encode() if zipcodes else None, C.byref(h))
        if rc != GB_OK:
            raise GbError(rc, "gb_index_from_gbz_min")
        self = cls.__new__(cls)
        self._h = h
        self.view = FlatIndex()
        rc = lib.gb_index_view(h, C.byref(self.view))
        if rc != GB_OK:
            raise GbError(rc, "gb_index_view")
        self.node_seqs, self.paths = None, None
        self.k, self.w = int(self.view.k), int(self.view.w)
        return self

    @classmethod
    def load(cls, path):
        """gb_index_load: an index written by save()."""
        lib = load_library()
        h = C.c_void_p()
        rc = lib.gb_index_load(str(path).encode(), C.byref(h))
        if rc != GB_OK:
            raise GbError(rc, "gb_index_load")
        self = cls.__new__(cls)
        self._h = h
        self.view = FlatIndex()
        rc = lib.gb_index_view(h, C.byref(self.view))
        if rc != GB_OK:
            raise GbError(rc, "gb_index_view")
        self.node_seqs, self.paths = None, None
        self.k, self.w = int(self.view.k), int(self.view.w)
        return self

    def array(self, name: str) -> np.ndarray:
        v = self.view
        spec = {
            "nodes": (v.nodes, v.n_nodes, node_rec_dt), "seq": (v.seq, v.seq_bytes, np.uint8),
            "gbwt": (v.gbwt, v.gbwt_words, np.uint32), "dist": (v.dist, v.n_nodes // 2, dist_dt),
            "table": (v.table, v.table_cells, min_cell_dt), "hits": (v.hits, v.n_hits, hit_dt),
            "slots": (v.slots, v.n_slots, slot_dt), "site_dist": (v.site_dist, v.site_dist_len, np.uint16),
        }[name]
        addr, n, dt = spec
        dt = np.dtype(dt)
        if n == 0:
            return np.zeros(0, dtype=dt)
        buf = (C.c_uint8 * (n * dt.itemsize)).from_address(addr)
        return np.frombuffer(buf, dtype=dt)

    def close(self):
        if getattr(self, "_h", None):
            load_library().gb_index_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


GB_PAIR_PAIRED, GB_PAIR_TRAINING, GB_PAIR_BUFFERED = 0, 1, 2


def chain_anchors(index, seeds, min_offset, min_is_reverse, min_length, paths=None, scores=None):
    """gb_chain_anchors (MinimizerMapper::to_anchor): seeds = [(oriented node, offset)], per-seed minimizer pin offset, strand, length."""
    lib = load_library()
    n = len(seeds)
    pos = np.ascontiguousarray(np.array(list(seeds) + [(0, 0)], dtype=np.uint32).reshape(-1))
    mo = np.ascontiguousarray(list(min_offset) + [0], dtype=np.uint32); mr = np.ascontiguousarray(list(min_is_reverse) + [0], dtype=np.uint8)
    ml = np.ascontiguousarray(list(min_length) + [0], dtype=np.uint32)
    pa = None if paths is None else np.ascontiguousarray(list(paths) + [0], dtype=np.uint64)
    out = np.zeros(n + 1, dtype=chain_anchor_dt)
    sc = scores or DEFAULT_SCORES
    rc = lib.gb_chain_anchors(C.byref(index.view), C.byref(sc), n, ptr(pos), ptr(mo), ptr(mr), ptr(ml), None if pa is None else ptr(pa), ptr(out))
    if rc != GB_OK:
        raise GbError(rc, "gb_chain_anchors")
    return out[:n]


def emit_text(kind, flat_index, aln, maps, edits, rbuf, qbuf, read_off, names=None):
    """gb_emit_gaf / gb_emit_json / gb_emit_gam (kind = "gaf" | "json" | "gam") over records `aln`; returns the text (bytes for GAM).
    names: optional list of read names (str)."""
    lib = load_library()
    fn = {"gaf": lib.gb_emit_gaf, "json": lib.gb_emit_json, "gam": lib.gb_emit_gam}[kind]
    nbuf = noff = None
    if names is not None:
        enc = [s.encode() for s in names]
        noff = np.zeros(len(enc) + 1, dtype=np.uint64)
        noff[1:] = np.cumsum([len(b) for b in enc])
        nbuf = np.frombuffer(b"".join(enc) + b"\0", dtype=np.uint8).copy()
    aln = np.ascontiguousarray(aln)
    cap = 4096 + len(aln) * 4096
    out = np.zeros(cap, dtype=np.uint8)
    used = C.c_uint64()
    rc = fn(C.byref(flat_index), len(aln), ptr(aln), ptr(maps), len(maps), ptr(edits), len(edits), len(read_off) - 1, ptr(rbuf),
            ptr(qbuf) if qbuf is not None else None, ptr(read_off), ptr(nbuf) if nbuf is not None else None, ptr(noff) if noff is not None else None,
            ptr(out), cap, C.byref(used))
    if rc != GB_OK:
        raise GbError(rc, "gb_emit_" + kind)
    data = out[: used.value].tobytes()
    return data if kind == "gam" else data.decode()


def bgzf_compress(data: bytes, level: int = 6) -> bytes:
    """gb_bgzf_compress: the BGZF container vg::io writes GAM streams in."""
    lib = load_library()
    src = np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
    cap = len(data) + 128 * (len(data) // 0xff00 + 2)
    out = np.zeros(cap, dtype=np.uint8)
    used = C.c_uint64()
    rc = lib.gb_bgzf_compress(ptr(src), len(data), level, ptr(out), cap, C.byref(used))
    if rc != GB_OK:
        raise GbError(rc, "gb_bgzf_compress")
    return out[: used.value].tobytes()


def stage_buffers(n, per_read=(160, 1024, 64, 64, 1024)):
    """Output arrays of gb_debug_seed_stage / the oracle's twin for n reads."""
    return (np.zeros(n, dtype=stage_read_dt), np.zeros(n * per_read[0] + 16, dtype=stage_minimizer_dt), np.zeros(n * per_read[1] + 16, dtype=stage_seed_dt),
            np.zeros(n * per_read[2] + 16, dtype=stage_cluster_dt), np.zeros(n * per_read[3] + 16, dtype=stage_item_dt), np.zeros(n * per_read[4] + 16, dtype=seed_dt))


class FragmentDistribution:
    """FragmentLengthDistribution (mapper.hpp:83-139) behind gb_fragment_*; MinimizerMapper's own is
    (1000, 1000, 0.95) (minimizer_mapper.cpp:72).  Host-side state: usable without a GPU."""

    def __init__(self, maximum_sample_size=1000, reestimation_frequency=1000, robust_estimation_fraction=0.95):
        self._h = load_library().gb_fragment_create(maximum_sample_size, reestimation_frequency, robust_estimation_fraction)
        if not self._h:
            raise GbError(GB_ERR_ARG, "gb_fragment_create")

    def register_fragment_length(self, length):
        load_library().gb_fragment_register(self._h, int(length))

    def force_parameters(self, mean, stdev):
        load_library().gb_fragment_force(self._h, mean, stdev)

    def finalize(self):
        load_library().gb_fragment_finalize(self._h)

    def mean(self):
        return load_library().gb_fragment_mean(self._h)

    def std_dev(self):
        return load_library().gb_fragment_stdev(self._h)

    def is_finalized(self):
        return bool(load_library().gb_fragment_is_finalized(self._h))

    def curr_sample_size(self):
        return int(load_library().gb_fragment_sample_size(self._h))

    def close(self):
        if getattr(self, "_h", None):
            load_library().gb_fragment_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Device:
    """gb_device handle on one GPU.  Raises GbError(GB_ERR_NO_DEVICE) when there is no GPU."""

    def __init__(self, index: HostIndex, ordinal: int = 0, scores: Scores | None = None):
        lib = load_library()
        h = C.c_void_p()
        rc = lib.gb_device_create(C.byref(index.view), ordinal, C.byref(h))
        if rc != GB_OK:
            raise GbError(rc, "gb_device_create")
        self._h = h
        self.index = index
        if scores is not None:
            lib.gb_set_scores(h, C.byref(scores))

    @property
    def handle(self):
        return self._h

    def kernel_ms(self) -> float:
        return float(load_library().gb_last_kernel_ms(self._h))

    def launches(self) -> int:
        return int(load_library().gb_launch_count(self._h))

    def extend_batch(self, reads, items, max_mismatches=4, overlap_threshold=0.8, trim=True,
                     max_ext=16, path_cap=256, mism_cap=128):
        """reads: list of bytes/str; items: list of (read_index, [(node, diag), ...]).

        Returns (ext_count, status, ext, path_pool, mism_pool) as numpy arrays."""
        lib = load_library()
        enc = [r.encode() if isinstance(r, str) else bytes(r) for r in reads]
        read_off = np.zeros(len(enc) + 1, dtype=np.uint64)
        read_off[1:] = np.cumsum([len(r) for r in enc])
        rbuf = np.frombuffer(b"".join(enc) + b"\0", dtype=np.uint8).copy()
        n_items = len(items)
        item_read = np.array([it[0] for it in items], dtype=np.uint32)
        seed_off = np.zeros(n_items + 1, dtype=np.uint64)
        seed_off[1:] = np.cumsum([len(it[1]) for it in items])
        seeds = np.zeros(max(1, int(seed_off[-1])), dtype=seed_dt)
        j = 0
        for it in items:
            for node, diag in it[1]:
                seeds[j] = (node, diag)
                j += 1
        return self.extend_arrays(rbuf, read_off, item_read, seeds, seed_off, max_mismatches, overlap_threshold,
                                  trim, max_ext, path_cap, mism_cap)

    def extend_arrays(self, rbuf, read_off, item_read, seeds, seed_off, max_mismatches=4, overlap_threshold=0.8,
                      trim=True, max_ext=16, path_cap=256, mism_cap=128):
        lib = load_library()
        n_items = len(item_read)
        p = ExtendParams(max_mismatches, overlap_threshold, 1 if trim else 0, max_ext, path_cap, mism_cap)
        ext_count = np.zeros(n_items, dtype=np.uint32)
        status = np.zeros(n_items, dtype=np.uint8)
        ext = np.zeros(n_items * max_ext, dtype=extension_dt)
        path_pool = np.zeros(n_items * path_cap, dtype=np.uint32)
        mism_pool = np.zeros(n_items * mism_cap, dtype=np.uint32)
        rc = lib.gb_extend_batch(self._h, C.byref(p), len(read_off) - 1, ptr(rbuf), ptr(read_off), n_items,
                                 ptr(item_read), ptr(seeds), ptr(seed_off), ptr(ext_count), ptr(status), ptr(ext),
                                 ptr(path_pool), ptr(mism_pool))
        if rc != GB_OK:
            raise GbError(rc, "gb_extend_batch")
        return ext_count, status, ext, path_pool, mism_pool

    def xdrop_pinned_batch(self, problems, map_cap=256, edit_cap=1024, with_status=False):
        """problems: list of (parents, nodes, root_trim, query bytes, max_gap).
        Returns list of (score, [[tree_index + 1, offset, [[op, len, base], ...]], ...]), every status
        asserted GB_ITEM_OK; with_status=True returns (status, score, path) instead, path empty unless
        status is GB_ITEM_OK."""
        lib = load_library()
        n = len(problems)
        tree_off = np.zeros(n + 1, dtype=np.uint64)
        tree_off[1:] = np.cumsum([len(p[0]) for p in problems])
        query_off = np.zeros(n + 1, dtype=np.uint64)
        query_off[1:] = np.cumsum([len(p[3]) for p in problems])
        par = np.concatenate([np.asarray(p[0], dtype=np.int32) for p in problems])
        nodes = np.concatenate([np.asarray(p[1], dtype=np.uint32) for p in problems])
        trim = np.array([p[2] for p in problems], dtype=np.uint32)
        q = np.frombuffer(b"".join(bytes(p[3]) for p in problems) + b"\0", dtype=np.uint8).copy()
        gap = np.array([p[4] for p in problems], dtype=np.uint32)
        score, maps, edits, nm, _, status = outs = _seam_outputs(n, map_cap, edit_cap)
        rc = lib.gb_xdrop_pinned_batch(self._h, n, ptr(par), ptr(nodes), ptr(tree_off), ptr(trim), ptr(q), ptr(query_off),
                                       ptr(gap), map_cap, edit_cap, *map(ptr, outs))
        if rc != GB_OK:
            raise GbError(rc, "gb_xdrop_pinned_batch")
        if with_status:
            return [(int(status[i]), int(score[i]),
                     decode_path(maps[i * map_cap:], edits[i * edit_cap:], nm[i], node_offset=1) if status[i] == GB_ITEM_OK else [])
                    for i in range(n)]
        out = []
        for i in range(n):
            assert status[i] == GB_ITEM_OK, f"problem {i}: status {status[i]}"
            out.append((int(score[i]), decode_path(maps[i * map_cap:], edits[i * edit_cap:], nm[i], node_offset=1)))
        return out

    def sw_batch(self, problems, map_cap=512, edit_cap=2048, with_status=False):
        """gb_sw_batch.  problems: list of (nodes, preds, query bytes) with nodes = oriented node ids in
        topological order and preds = per-node lists of predecessor indices.
        Returns list of (score, [[problem_index, offset, [[op, len, base], ...]], ...]), every status
        asserted GB_ITEM_OK; with_status=True returns (status, score, path) instead, path decoded from the
        returned counts whatever the status."""
        lib = load_library()
        n = len(problems)
        dags = _pack_dags(problems)
        outs = _seam_outputs(n, map_cap, edit_cap)
        rc = lib.gb_sw_batch(self._h, n, *map(ptr, dags), map_cap, edit_cap, *map(ptr, outs))
        if rc != GB_OK:
            raise GbError(rc, "gb_sw_batch")
        return _dag_seam_results(outs, map_cap, with_status)

    def banded_global_batch(self, problems, map_cap=512, edit_cap=2048):
        """gb_banded_global_batch.  problems: list of (nodes, preds, query bytes, band_padding, permissive)
        posed like sw_batch.  Returns list of (status, score, path) with path as in sw_batch (empty
        unless status is GB_ITEM_OK)."""
        lib = load_library()
        n = len(problems)
        pad = np.asarray([p[3] for p in problems], dtype=np.int32)
        permissive = np.asarray([1 if p[4] else 0 for p in problems], dtype=np.uint8)
        dags = _pack_dags(problems)
        score, maps, edits, nm, _, status = outs = _seam_outputs(n, map_cap, edit_cap)
        rc = lib.gb_banded_global_batch(self._h, n, *map(ptr, dags), ptr(pad), ptr(permissive), map_cap, edit_cap,
                                        *map(ptr, outs))
        if rc != GB_OK:
            raise GbError(rc, "gb_banded_global_batch")
        return [(int(status[i]), int(score[i]), decode_path(maps[i * map_cap:], edits[i * edit_cap:], nm[i])) for i in range(n)]

    def xdrop_dag_batch(self, problems, map_cap=512, edit_cap=2048, with_status=False):
        """gb_xdrop_dag_batch.  problems: list of (nodes, preds, query bytes, seed or None, max_gap) with
        seed = (node index, node offset, query offset).  Returns list of (score, path) like sw_batch, and
        with_status=True (status, score, path) like sw_batch."""
        lib = load_library()
        n = len(problems)
        seed = np.array([(0xFFFFFFFF, 0, 0) if p[3] is None else p[3] for p in problems], dtype=np.uint32).reshape(-1)
        gap = np.array([p[4] for p in problems], dtype=np.uint32)
        dags = _pack_dags(problems)
        outs = _seam_outputs(n, map_cap, edit_cap)
        rc = lib.gb_xdrop_dag_batch(self._h, n, *map(ptr, dags), ptr(seed), ptr(gap), map_cap, edit_cap,
                                    *map(ptr, outs))
        if rc != GB_OK:
            raise GbError(rc, "gb_xdrop_dag_batch")
        return _dag_seam_results(outs, map_cap, with_status)

    def chain_candidates_batch(self, problems, limit=2 ** 64 - 1, cap=None):
        """gb_chain_candidates_batch.  problems: list of seed lists [(oriented node, offset), ...].
        Returns per problem a chain_candidate_dt array sorted by (to, from)."""
        lib = load_library()
        n = len(problems)
        off = np.zeros(n + 1, dtype=np.uint64); off[1:] = np.cumsum([len(p) for p in problems])
        pos = np.ascontiguousarray(np.array([x for p in problems for x in p] + [(0, 0)], dtype=np.uint32).reshape(-1))
        coff = np.zeros(n + 1, dtype=np.uint64)
        if cap is None:
            rc = lib.gb_chain_candidates_batch(self._h, n, ptr(pos), ptr(off), limit, None, 0, ptr(coff))      # sizes first
            if rc not in (GB_OK, GB_ERR_CAPACITY):
                raise GbError(rc, "gb_chain_candidates_batch")
            cap = int(coff[n])
        out = np.zeros(cap + 1, dtype=chain_candidate_dt)
        rc = lib.gb_chain_candidates_batch(self._h, n, ptr(pos), ptr(off), limit, ptr(out), cap, ptr(coff))
        if rc != GB_OK:
            raise GbError(rc, "gb_chain_candidates_batch")
        return [out[int(coff[p]): int(coff[p + 1])].copy() for p in range(n)]

    def chain_batch(self, problems, params=None, transitions=False):
        """gb_chain_batch.  problems: list of (anchors, candidates) structured arrays (chain_anchor_dt sorted by read_start,
        chain_candidate_dt).  Returns per problem {"dp": [(score, source, paths, rec)], "chains": [(score, [anchor indices])]};
        transitions=True (gb_chain_batch_transitions) adds "transitions": {(from, to): indel} of the legal candidates."""
        lib = load_library()
        if params is None:
            params = ChainParams(); lib.gb_chain_params_default(C.byref(params))
        n = len(problems)
        aoff = np.zeros(n + 1, dtype=np.uint64); coff = np.zeros(n + 1, dtype=np.uint64)
        aoff[1:] = np.cumsum([len(a) for a, _ in problems]); coff[1:] = np.cumsum([len(c) for _, c in problems])
        anchors = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=chain_anchor_dt) for a, _ in problems] + [np.zeros(1, chain_anchor_dt)]))
        cands = np.ascontiguousarray(np.concatenate([np.asarray(c, dtype=chain_candidate_dt) for _, c in problems] + [np.zeros(1, chain_candidate_dt)]))
        ta = int(aoff[-1]); k = int(params.max_chains)
        dps = np.zeros(ta + 1, np.int32); dpsrc = np.zeros(ta + 1, np.uint32); dpp = np.zeros(ta + 1, np.uint64); dpr = np.zeros(ta + 1, np.uint32)
        nch = np.zeros(n, np.uint32); cs = np.zeros(n * k, np.int32); cb = np.zeros(n * k, np.uint32); cc = np.zeros(n * k, np.uint32)
        items = np.zeros(ta + 1, np.uint32)
        indel = np.zeros(int(coff[-1]) + 1, np.uint32)
        if transitions:
            rc = lib.gb_chain_batch_transitions(self._h, C.byref(params), n, ptr(anchors), ptr(aoff), ptr(cands), ptr(coff),
                                                ptr(dps), ptr(dpsrc), ptr(dpp), ptr(dpr), ptr(nch), ptr(cs), ptr(cb), ptr(cc), ptr(items), ptr(indel))
        else:
            rc = lib.gb_chain_batch(self._h, C.byref(params), n, ptr(anchors), ptr(aoff), ptr(cands), ptr(coff),
                                    ptr(dps), ptr(dpsrc), ptr(dpp), ptr(dpr), ptr(nch), ptr(cs), ptr(cb), ptr(cc), ptr(items))
        if rc != GB_OK:
            raise GbError(rc, "gb_chain_batch")
        out = []
        for p in range(n):
            a0, a1 = int(aoff[p]), int(aoff[p + 1])
            if transitions:
                c0, c1 = int(coff[p]), int(coff[p + 1])
                tr = {(int(x["from"]), int(x["to"])): int(i) for x, i in zip(cands[c0:c1], indel[c0:c1]) if i != 0xffffffff}
            out.append({**({"transitions": tr} if transitions else {}),"dp": [(int(dps[i]), int(dpsrc[i]), int(dpp[i]), int(dpr[i])) for i in range(a0, a1)],
                        "chains": [(int(cs[p * k + c]), [int(x) for x in items[int(cb[p * k + c]): int(cb[p * k + c]) + int(cc[p * k + c])]])
                                   for c in range(int(nch[p]))]})
        return out

    def wfa_batch(self, problems, error_model=None, path_cap=512, edit_cap=512, with_status=False):
        """gb_wfa_batch.  problems: list of (mode, sequence bytes, (from node, from offset) or None,
        (to node, to offset) or None) with mode 0 connect / 1 suffix / 2 prefix and oriented nodes.
        Returns list of dicts with the WFAAlignment fields (edits as (op letter, length), ops "MXID"),
        every problem asserted to fit the workspace and caps; with_status=True returns "ok" as the
        kernel's -1 / 0 / 1 instead."""
        lib = load_library()
        n = len(problems)
        seq_off = np.zeros(n + 1, dtype=np.uint64)
        seq_off[1:] = np.cumsum([len(p[1]) for p in problems])
        seq = np.frombuffer(b"".join(bytes(p[1]) for p in problems) + b"\0", dtype=np.uint8).copy()
        mode = np.array([p[0] for p in problems], dtype=np.uint32)
        pos = np.array([list(p[2] or (0, 0)) + list(p[3] or (0, 0)) for p in problems], dtype=np.uint32).reshape(-1)
        em = None if error_model is None else np.asarray(error_model, dtype=np.float64)
        ok = np.zeros(n, dtype=np.int32); score = np.zeros(n, dtype=np.int32)
        noff, soff, length, npath, nedits = (np.zeros(n, dtype=np.uint32) for _ in range(5))
        path = np.zeros(n * path_cap, dtype=np.uint32); edits = np.zeros(n * edit_cap, dtype=np.uint32)
        rc = lib.gb_wfa_batch(self._h, n, ptr(seq), ptr(seq_off), ptr(mode), ptr(pos), None if em is None else ptr(em), path_cap, edit_cap,
                              ptr(ok), ptr(score), ptr(noff), ptr(soff), ptr(length), ptr(path), ptr(npath), ptr(edits), ptr(nedits))
        if rc != GB_OK:
            raise GbError(rc, "gb_wfa_batch")
        out = []
        for i in range(n):
            assert with_status or ok[i] >= 0, f"problem {i}: workspace capacity exceeded"
            out.append({"ok": int(ok[i]) if with_status else bool(ok[i]), "score": int(score[i]), "node_offset": int(noff[i]), "seq_offset": int(soff[i]), "length": int(length[i]),
                        "path": [int(x) for x in path[i * path_cap: i * path_cap + int(npath[i])]],
                        "edits": [("MXID"[int(w) & 3], int(w) >> 2) for w in edits[i * edit_cap: i * edit_cap + int(nedits[i])]]})
        return out

    def map_arrays(self, rbuf, qbuf, read_off, params=None, paired=False, out=None):
        """gb_map_batch / gb_map_paired_batch on packed host arrays.
        Returns (aln, mappings, edits, status); mappings / edits are dense pools."""
        lib = load_library()
        p = params or default_map_params()
        n = len(read_off) - 1
        k = max(1, int(p.max_multimaps))              # aln holds n * max_multimaps records, rank-major (record j * n + read)
        if out is None:
            aln = np.zeros(n * k, dtype=alignment_dt)
            maps = np.zeros(n * k * 24 + 1024, dtype=mapping_dt)
            edits = np.zeros(n * k * 32 + 1024, dtype=np.uint32)
            status = np.zeros(n, dtype=np.uint8)
        else:
            aln, maps, edits, status = out
        used = (C.c_uint64(), C.c_uint64())
        fn = lib.gb_map_paired_batch if paired else lib.gb_map_batch
        rc = fn(self._h, C.byref(p), n, ptr(rbuf), ptr(qbuf) if qbuf is not None else None, ptr(read_off), ptr(aln),
                ptr(maps), len(maps), ptr(edits), len(edits), ptr(status), C.byref(used[0]), C.byref(used[1]))
        if rc == GB_ERR_CAPACITY and out is None:
            maps = np.zeros(n * k * p.mapping_cap_per_read, dtype=mapping_dt)
            edits = np.zeros(n * k * p.edit_cap_per_read, dtype=np.uint32)
            rc = fn(self._h, C.byref(p), n, ptr(rbuf), ptr(qbuf) if qbuf is not None else None, ptr(read_off), ptr(aln),
                    ptr(maps), len(maps), ptr(edits), len(edits), ptr(status), C.byref(used[0]), C.byref(used[1]))
        if rc != GB_OK:
            raise GbError(rc, "gb_map_paired_batch" if paired else "gb_map_batch")
        self.last_used = (used[0].value, used[1].value)
        return aln, maps, edits, status

    def map_paired_job(self, rbuf, qbuf, read_off, distribution, params=None, training_window=0):
        """gb_map_paired_job: fragment-length training + map_paired + the ambiguous buffer.
        Returns (aln, mappings, edits, status, pair_route)."""
        lib = load_library()
        p = params or default_map_params()
        n = len(read_off) - 1
        aln = np.zeros(n, dtype=alignment_dt)
        maps = np.zeros(n * p.mapping_cap_per_read, dtype=mapping_dt)
        edits = np.zeros(n * p.edit_cap_per_read, dtype=np.uint32)
        status = np.zeros(n, dtype=np.uint8)
        route = np.zeros(n // 2, dtype=np.uint8)
        used = (C.c_uint64(), C.c_uint64())
        rc = lib.gb_map_paired_job(self._h, C.byref(p), distribution._h, training_window, n, ptr(rbuf), ptr(qbuf) if qbuf is not None else None,
                                   ptr(read_off), ptr(aln), ptr(maps), len(maps), ptr(edits), len(edits), ptr(status), ptr(route),
                                   C.byref(used[0]), C.byref(used[1]))
        if rc != GB_OK:
            raise GbError(rc, "gb_map_paired_job")
        self.last_used = (used[0].value, used[1].value)
        return aln, maps, edits, status, route

    def seed_stage(self, rbuf, qbuf, read_off, params=None, paired=False, per_read=(160, 1024, 64, 64, 1024)):
        """gb_debug_seed_stage: (reads, minimizers, seeds, clusters, items, item_seeds) as structured arrays."""
        lib = load_library()
        p = params or default_map_params()
        n = len(read_off) - 1
        outs = stage_buffers(n, per_read)
        rc = lib.gb_debug_seed_stage(self._h, C.byref(p), 1 if paired else 0, n, ptr(rbuf), ptr(qbuf) if qbuf is not None else None, ptr(read_off),
                                     ptr(outs[0]), ptr(outs[1]), len(outs[1]), ptr(outs[2]), len(outs[2]), ptr(outs[3]), len(outs[3]),
                                     ptr(outs[4]), len(outs[4]), ptr(outs[5]), len(outs[5]))
        if rc != GB_OK:
            raise GbError(rc, "gb_debug_seed_stage")
        return outs

    def pool_overflow(self) -> bool:
        flag = C.c_int()
        rc = load_library().gb_device_pool_overflow(self._h, C.byref(flag))
        if rc != GB_OK:
            raise GbError(rc, "gb_device_pool_overflow")
        return bool(flag.value)

    def kernel_times(self):
        """Per-kernel device time of the last mapping call's last chunk: list of (kernel name, ms)."""
        cap = 48
        names = C.create_string_buffer(cap * 48); ms = (C.c_float * cap)(); n = C.c_uint32()
        rc = load_library().gb_kernel_times(self._h, cap, names, ms, C.byref(n))
        if rc != GB_OK:
            raise GbError(rc, "gb_kernel_times")
        return [(names.raw[i * 48:(i + 1) * 48].split(b"\0")[0].decode(), float(ms[i])) for i in range(n.value)]

    def plan_stats(self):
        out = (C.c_uint64 * 4)()
        rc = load_library().gb_plan_stats(self._h, out)
        if rc != GB_OK:
            raise GbError(rc, "gb_plan_stats")
        return {"tails": int(out[0]), "trees": int(out[1]), "in_place": int(out[2]), "cells": int(out[3])}

    def stage_times(self):
        ms = (C.c_float * 4)()
        rc = load_library().gb_stage_times(self._h, ms)
        if rc != GB_OK:
            raise GbError(rc, "gb_stage_times")
        return [float(x) for x in ms]

    def close(self):
        if getattr(self, "_h", None):
            load_library().gb_device_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
