// xdrop_dag.cu — B3 stage seam: Aligner::align_xdrop(alignment, graph, order, mems, rc = false, max_gap)
// (aligner.cpp:833-855 -> DozeuInterface::align, dozeu_interface.cpp:608-685), the seeded two-pass
// X-drop alignment vg giraffe uses for mate rescue (minimizer_mapper.cpp:3385):
//   pass 1  from the seed, extend the query suffix to the right and take the best end as the "head"
//           (no seed: scan the last 15 query bases over the subgraph for their best local match);
//   pass 2  from the head, extend the query prefix to the LEFT with traceback; the query right of the
//           head is a soft clip.
// Cell rules: those of the pinned aligner (tail.cuh) extended to DAGs as oracle/xdrop_dag.cpp states.
//
// One warp per problem.  Pass 2 runs on the mirrored problem without materialising it: pass order t
// maps to node N - 1 - t, pass column c to base len - 1 - c, predecessors are the successors.
#include <cub/cub.cuh>
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "dag_dp.cuh"
#include "seam_batch.cuh"

namespace gb {

constexpr int XD_WARPS = 4;

struct XdBatch {
    DagDev dag;
    SeamOut out;
    const uint32_t* succ; const uint64_t* succ_off;         // forward successors, ascending (pred: forward predecessors, ascending)
    const uint32_t* seed;                                   // 3 per problem: node index (0xffffffff: none), node offset, query offset
    const uint32_t* max_gap;
    int32_t* lastH; int32_t* lastE; uint8_t* argH; uint8_t* argE;
    uint32_t* col_start; uint32_t* seq_off; uint32_t* seq_len; XdNode* nstate;
    uint32_t* work_counter;
};

__global__ void __launch_bounds__(XD_WARPS * 32)
xdrop_dag_kernel(DevIndex ix, DevScores sc, XdBatch b) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* q;
    const DpSmem dps = dp_smem_carve(smem, warp, b.dag.Lc, q);
    while (true) {
        uint32_t p = 0;
        if (lane == 0) p = atomicAdd(b.work_counter, 1u);
        p = __shfl_sync(FULL, p, 0);
        if (p >= b.dag.n) break;
        uint32_t status = GB_ITEM_OK; int32_t score = 0;
        PathBuf out = b.out.path(p);
        {
            DagView v;
            const uint64_t n0 = b.dag.view(p, v), c0 = b.dag.col_off[p];
            v.succ = b.succ; v.succ_off = b.succ_off + n0;
            v.col_start = b.col_start + n0; v.seq_off = b.seq_off + n0; v.seq_len = b.seq_len + n0; v.nstate = b.nstate + n0;
            v.lastH = b.lastH + c0; v.lastE = b.lastE + c0; v.argH = b.argH + c0; v.argE = b.argE + c0;
            uint32_t m;
            const uint8_t* read = b.dag.read(p, m);
            xd_align(ix, sc, v, read, m, b.seed[3 * p], b.seed[3 * p + 1], b.seed[3 * p + 2], b.max_gap[p],
                     q, dps, score, out, status);
        }
        if (status != GB_ITEM_OK || score <= 0) { score = 0; out.n_maps = 0; out.n_edits = 0; }
        b.out.store(p, score, out.n_maps, out.n_edits, status);
        __syncwarp();
    }
}

} // namespace gb

using namespace gb;

extern "C" int gb_xdrop_dag_batch(gb_device* d, uint32_t n,
                                  const uint32_t* node, const uint64_t* node_off, const uint32_t* pred, const uint64_t* pred_off,
                                  const uint8_t* query, const uint64_t* query_off, const uint32_t* seed, const uint32_t* max_gap,
                                  uint32_t map_cap, uint32_t edit_cap,
                                  int32_t* score, gb_mapping* maps, uint32_t* edits, uint32_t* n_maps, uint32_t* n_edits, uint8_t* status) {
    if (!d || !node || !node_off || !pred || !pred_off || !query || !query_off || !seed || !max_gap || !score || !maps || !edits ||
        !n_maps || !n_edits || !status || map_cap == 0 || edit_cap == 0) return GB_ERR_ARG;
    if (n == 0) return GB_OK;
    GB_CUDA(cudaSetDevice(d->device));
    DagProblems dag(n, node, node_off, pred, pred_off, query, query_off);
    int rc;
    if ((rc = dag.validate(d, "gb_xdrop_dag_batch"))) return rc;
    for (uint32_t p = 0; p < n; p++) {
        // vg's max_gap is a uint16_t (DozeuInterface::align), and the X-drop threshold go + ge * (max_gap - 1) is int32
        if (max_gap[p] > 65535) return DagProblems::fail("gb_xdrop_dag_batch", ": max_gap above 65535");
        // a seed lies in its problem: a node of the list, an offset up to that node's length, a query offset up to m
        const uint32_t su = seed[3 * p], so = seed[3 * p + 1], sq = seed[3 * p + 2];
        if (su == 0xffffffffu) continue;
        if (su >= dag.N[p]) return DagProblems::fail("gb_xdrop_dag_batch", ": seed node outside the problem");
        if (so > d->h_node_len[node[node_off[p] + su]]) return DagProblems::fail("gb_xdrop_dag_batch", ": seed offset past the seed node");
        if (sq > dag.m[p]) return DagProblems::fail("gb_xdrop_dag_batch", ": seed query offset past the query");
    }
    // successor CSR, ascending (nodes are visited in ascending order), at most 255 successors per node
    const uint64_t total_pred = pred_off[dag.total_nodes];
    std::vector<uint64_t> succ_off(dag.total_nodes + 1, 0);
    std::vector<uint32_t> succ(total_pred ? total_pred : 1);
    for (uint32_t p = 0; p < n; p++) {
        const uint64_t n0 = node_off[p], N = dag.N[p];
        std::vector<uint32_t> deg(N, 0);
        for (uint64_t e = pred_off[n0]; e < pred_off[n0 + N]; e++) deg[pred[e]]++;
        for (uint64_t u = 0; u < N; u++) {
            if (deg[u] > 255) { g_last_error = "gb_xdrop_dag_batch: more than 255 successors"; return GB_ERR_ARG; }
            succ_off[n0 + u + 1] = succ_off[n0 + u] + deg[u];
        }
        std::vector<uint32_t> fill(N, 0);
        for (uint64_t u = 0; u < N; u++)
            for (uint64_t e = pred_off[n0 + u]; e < pred_off[n0 + u + 1]; e++) { const uint32_t pu = pred[e]; succ[succ_off[n0 + pu] + fill[pu]++] = (uint32_t)u; }
    }
    XdBatch b;
    if ((rc = dag.check_limits("gb_xdrop_dag_batch")) || (rc = dag.upload(d->stream, b.dag))) return rc;
    SeamOutBufs out;
    DevBuf<uint32_t> d_succ, d_seed, d_gap, d_colstart, d_seqoff, d_seqlen; DevBuf<uint64_t> d_soff;
    DevBuf<int32_t> d_lastH, d_lastE; DevBuf<uint8_t> d_argH, d_argE; DevBuf<XdNode> d_nstate;
    const uint64_t cols = dag.col_off[n] + 1, nodes = dag.total_nodes + 1;
    if ((rc = d_succ.upload(succ.data(), total_pred ? total_pred : 1, d->stream, total_pred))) return rc;
    if ((rc = d_soff.upload(succ_off.data(), dag.total_nodes + 1, d->stream))) return rc;
    if ((rc = d_seed.upload(seed, 3 * (size_t)n, d->stream))) return rc;
    if ((rc = d_gap.upload(max_gap, n, d->stream))) return rc;
    if ((rc = out.reserve(n, map_cap, edit_cap))) return rc;
    if ((rc = d_lastH.reserve(cols)) || (rc = d_lastE.reserve(cols)) || (rc = d_argH.reserve(cols)) || (rc = d_argE.reserve(cols))) return rc;
    if ((rc = d_colstart.reserve(nodes)) || (rc = d_seqoff.reserve(nodes)) || (rc = d_seqlen.reserve(nodes)) || (rc = d_nstate.reserve(nodes))) return rc;
    b.out = out.view;
    b.succ = d_succ.ptr; b.succ_off = d_soff.ptr; b.seed = d_seed.ptr; b.max_gap = d_gap.ptr;
    b.lastH = d_lastH.ptr; b.lastE = d_lastE.ptr; b.argH = d_argH.ptr; b.argE = d_argE.ptr;
    b.col_start = d_colstart.ptr; b.seq_off = d_seqoff.ptr; b.seq_len = d_seqlen.ptr; b.nstate = d_nstate.ptr;
    if ((rc = launch_warp_per_problem(d, xdrop_dag_kernel, b, XD_WARPS, dp_smem_per_warp(dag.Lc) * XD_WARPS))) return rc;
    return out.download(d, n, score, maps, edits, n_maps, n_edits, status);
}
