"""What the DAG alignment seams gb_sw_batch, gb_xdrop_dag_batch and gb_banded_global_batch refuse: the
return code of each refused batch, and that a refused batch launches nothing.  The max_gap limit is checked on
gb_xdrop_pinned_batch as well."""
import ctypes as C

import numpy as np
import pytest

from vg_b200 import capi

SEQS = ["ACGTTGCAGGCTAACGTTAGCCATGCAATCGG", "TTGACCGATGCATGGCTAACGGTACCATGAAC", "GGCATTACGCATCCGATAGCTTGACGAACTGA"]
# id 4 has no sequence (an id a GBZ graph does not use), ids 5 and 6 are one base long
INDEX_SEQS = SEQS + ["", "C", "A"]
EMPTY_IDS = (8, 9)
NODES = [2, 4, 6]
CHAIN = [[], [0], [1]]
READ = (SEQS[0] + SEQS[1] + SEQS[2]).encode()


def _sw(dev, nodes, preds, q, pad=8):
    return dev.sw_batch([(nodes, preds, q)])


def _xdrop_dag(dev, nodes, preds, q, pad=8, seed=None, gap=30):
    return dev.xdrop_dag_batch([(nodes, preds, q, seed, gap)])


def _banded_global(dev, nodes, preds, q, pad=8):
    return dev.banded_global_batch([(nodes, preds, q, pad, False)])


SEAMS = {"sw": (_sw, "gb_sw_batch"), "xdrop_dag": (_xdrop_dag, "gb_xdrop_dag_batch"),
         "banded_global": (_banded_global, "gb_banded_global_batch")}


@pytest.fixture(scope="module")
def dev():
    index = capi.HostIndex(INDEX_SEQS, [NODES, [10, 12]], None, k=5, w=3)
    d = capi.Device(index)
    yield d
    d.close()


def refused(dev, call, code, *args, **kw):
    before = dev.launches()
    with pytest.raises(capi.GbError) as e:
        call(dev, *args, **kw)
    assert e.value.code == code
    assert dev.launches() == before


@pytest.mark.gpu
@pytest.mark.parametrize("seam", SEAMS)
def test_dag_seam_refuses_malformed_graphs(dev, seam):
    call = SEAMS[seam][0]
    for bad in (0, 1, *EMPTY_IDS, dev.index.view.n_nodes, dev.index.view.n_nodes + 1):
        refused(dev, call, capi.GB_ERR_ARG, [2, bad, 6], CHAIN, READ)
    refused(dev, call, capi.GB_ERR_ARG, [2, 4], [[], [0] * 256], READ)
    refused(dev, call, capi.GB_ERR_ARG, NODES, [[], [1], [1]], READ)
    refused(dev, call, capi.GB_ERR_ARG, NODES, [[], [2], [1]], READ)
    # the accepted neighbours of the refused shapes
    before = dev.launches()
    call(dev, [2, 4], [[], [0] * 255], READ)
    call(dev, NODES, CHAIN, READ)
    assert dev.launches() == before + 2


@pytest.mark.gpu
@pytest.mark.parametrize("seam", SEAMS)
def test_dag_seam_query_width_limit(dev, seam):
    call = SEAMS[seam][0]
    refused(dev, call, capi.GB_ERR_ARG, NODES, CHAIN, (READ * 11)[:1025])
    before = dev.launches()
    call(dev, NODES, CHAIN, (READ * 11)[:1024])
    assert dev.launches() == before + 1


@pytest.mark.gpu
@pytest.mark.parametrize("seam", SEAMS)
def test_dag_seam_refuses_more_than_8_gib_of_traceback(dev, seam):
    # 270 000 x 32 bases x 1001 query prefixes > 2^33 traceback bytes
    n = 270_000
    preds = [[]] + [[i] for i in range(n - 1)]
    refused(dev, SEAMS[seam][0], capi.GB_ERR_CAPACITY, [2] * n, preds, READ * 10 + READ[:40])


@pytest.mark.gpu
def test_banded_global_refuses_negative_padding(dev):
    refused(dev, _banded_global, capi.GB_ERR_ARG, NODES, CHAIN, READ, pad=-1)


@pytest.mark.gpu
def test_xdrop_dag_refuses_more_than_255_successors(dev):
    refused(dev, _xdrop_dag, capi.GB_ERR_ARG, [2] + [4] * 256, [[]] + [[0]] * 256, READ)
    before = dev.launches()
    _xdrop_dag(dev, [2] + [4] * 255, [[]] + [[0]] * 255, READ)
    assert dev.launches() == before + 1


def _raw_call(dev, seam, n, map_cap):
    """The seam's C entry point on zero-filled arrays (ctypes: the Python packers need a non-empty batch)."""
    lib = capi.load_library()
    u32 = np.zeros(16, dtype=np.uint32); off = np.zeros(16, dtype=np.uint64); q = np.zeros(16, dtype=np.uint8)
    score = np.zeros(16, dtype=np.int32); maps = np.zeros(16, dtype=capi.mapping_dt); edits = np.zeros(16, dtype=np.uint32)
    nm = np.zeros(16, dtype=np.uint32); ne = np.zeros(16, dtype=np.uint32); status = np.zeros(16, dtype=np.uint8)
    extra = {"sw": [], "xdrop_dag": [u32, u32], "banded_global": [np.zeros(16, dtype=np.int32), q]}[seam]
    args = [u32, off, u32, off, q, off, *extra]
    return getattr(lib, SEAMS[seam][1])(dev.handle, n, *map(capi.ptr, args), map_cap, 16,
                                        *map(capi.ptr, [score, maps, edits, nm, ne, status]))


@pytest.mark.gpu
@pytest.mark.parametrize("seam", SEAMS)
def test_dag_seam_empty_batch_and_zero_capacity(dev, seam):
    before = dev.launches()
    assert _raw_call(dev, seam, 0, 16) == capi.GB_OK
    assert _raw_call(dev, seam, 1, 0) == capi.GB_ERR_ARG
    assert dev.launches() == before


def _raw_dag_call(dev, seam, node, node_off, pred, pred_off, q, query_off):
    """The seam's C entry point on the caller's CSR arrays, one output slot per problem."""
    n = len(node_off) - 1
    outs = capi._seam_outputs(n, 16, 16)
    extra = {"sw": [], "xdrop_dag": [np.full(3 * n, 0xFFFFFFFF, dtype=np.uint32), np.full(n, 30, dtype=np.uint32)],
             "banded_global": [np.full(n, 8, dtype=np.int32), np.zeros(n, dtype=np.uint8)]}[seam]
    args = [node, node_off, pred, pred_off, q, query_off, *extra]
    return getattr(capi.load_library(), SEAMS[seam][1])(dev.handle, n, *map(capi.ptr, args), 16, 16, *map(capi.ptr, outs))


@pytest.mark.gpu
@pytest.mark.parametrize("seam", SEAMS)
def test_dag_seam_refuses_2_24_nodes(dev, seam):
    # traceback steps carry the node index in 24 bits: 2^24 one-base nodes (a problem may repeat an id) are refused on
    # the host, before anything is uploaded
    n = 1 << 24
    node = np.full(n, 10, dtype=np.uint32)
    node[-1] = 12
    pred_off = np.zeros(n + 1, dtype=np.uint64)
    q = np.frombuffer(b"A\0", dtype=np.uint8).copy()
    before = dev.launches()
    rc = _raw_dag_call(dev, seam, node, np.array([0, n], dtype=np.uint64), np.zeros(1, dtype=np.uint32), pred_off, q,
                       np.array([0, 1], dtype=np.uint64))
    assert rc == capi.GB_ERR_ARG
    assert b"2^24" in capi.load_library().gb_last_error()
    assert dev.launches() == before


@pytest.mark.gpu
def test_xdrop_dag_refuses_seeds_outside_the_problem(dev):
    m = len(READ)
    for seed in ((3, 0, 0), (0xFFFFFFFE, 0, 0), (2, 33, 0), (0, 0, m + 1), (1, 1 << 31, 0)):
        refused(dev, _xdrop_dag, capi.GB_ERR_ARG, NODES, CHAIN, READ, seed=seed)
    # the accepted neighbours: the last node, an offset equal to the node's length, a query offset equal to m
    before = dev.launches()
    for seed in ((2, 0, 64), (2, 32, 96), (0, 0, m), (2, 32, m), (0, 0, 0)):
        _xdrop_dag(dev, NODES, CHAIN, READ, seed=seed)
    assert dev.launches() == before + 5


@pytest.mark.gpu
def test_xdrop_seams_refuse_max_gap_above_65535(dev):
    # vg's max_gap is a uint16_t; a larger one would wrap the int32 X-drop threshold go + ge * (max_gap - 1)
    refused(dev, _xdrop_dag, capi.GB_ERR_ARG, NODES, CHAIN, READ, gap=65536)
    refused(dev, _xdrop_dag, capi.GB_ERR_ARG, NODES, CHAIN, READ, gap=0xFFFFFFFF)
    pinned = lambda d, gap: d.xdrop_pinned_batch([([-1, 0, 1], NODES, 0, READ, gap)])
    refused(dev, pinned, capi.GB_ERR_ARG, 65536)
    before = dev.launches()
    _xdrop_dag(dev, NODES, CHAIN, READ, gap=65535)
    _xdrop_dag(dev, NODES, CHAIN, READ, gap=0)
    pinned(dev, 65535)
    assert dev.launches() >= before + 3
