// full_dp.cu — B3 stage seam: Aligner::align(alignment, graph, topological_order), the full
// (unbanded) local alignment of a read against a DAG that vg runs through GSSW
// (aligner.cpp:571-626 -> align_internal :344-564 -> gssw_graph_fill_pinned / gssw_graph_trace_back).
// vg giraffe reaches it as the rescue fallback (fix_dozeu_score, minimizer_mapper.cpp:3502-3517)
// and with --rescue-algorithm gssw (:3390).  The recurrence, end-cell and traceback rules are the
// ones stated in oracle/full_dp.cpp (gssw itself is absent from the reference tree).
//
// One warp per problem.  A DP column is swept in 32-cell chunks along the query (lane = query
// offset), the insertion chain by a max-plus prefix scan over shuffles; the two live columns sit in
// shared memory, every node's last column (for its successors), the predecessor choices of first
// columns and one traceback byte per cell in a per-problem HBM workspace whose size the host knows.
#include <cub/cub.cuh>
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "dag_dp.cuh"
#include "seam_batch.cuh"

namespace gb {

constexpr int SW_WARPS = 4;

struct SwBatch {
    DagDev dag;
    SeamOut out;
    // per-node workspaces, offset by the problem's first global node: node-granular columns at col_off[p] + u * (m + 1)
    int32_t* lastH; int32_t* lastE; uint8_t* argH; uint8_t* argE;
    uint32_t* col_start; uint32_t* seq_off; uint32_t* seq_len;   // per global node: first traceback column, sequence
    uint32_t* work_counter;
};

__global__ void __launch_bounds__(SW_WARPS * 32)
sw_kernel(DevIndex ix, DevScores sc, SwBatch b) {
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
            v.succ = nullptr; v.succ_off = nullptr;
            v.col_start = b.col_start + n0; v.seq_off = b.seq_off + n0; v.seq_len = b.seq_len + n0; v.nstate = nullptr;
            v.lastH = b.lastH + c0; v.lastE = b.lastE + c0; v.argH = b.argH + c0; v.argE = b.argE + c0;
            uint32_t m;
            const uint8_t* read = b.dag.read(p, m);
            sw_align(ix, sc, v, read, m, q, dps, score, out, status);
        }
        const bool ok = status == GB_ITEM_OK;
        b.out.store(p, ok ? score : 0, ok ? out.n_maps : 0, ok ? out.n_edits : 0, status);
        __syncwarp();
    }
}

} // namespace gb

using namespace gb;

extern "C" int gb_sw_batch(gb_device* d, uint32_t n,
                           const uint32_t* node, const uint64_t* node_off, const uint32_t* pred, const uint64_t* pred_off,
                           const uint8_t* query, const uint64_t* query_off, uint32_t map_cap, uint32_t edit_cap,
                           int32_t* score, gb_mapping* maps, uint32_t* edits, uint32_t* n_maps, uint32_t* n_edits, uint8_t* status) {
    if (!d || !node || !node_off || !pred || !pred_off || !query || !query_off || !score || !maps || !edits || !n_maps || !n_edits ||
        !status || map_cap == 0 || edit_cap == 0) return GB_ERR_ARG;
    if (n == 0) return GB_OK;
    GB_CUDA(cudaSetDevice(d->device));
    DagProblems dag(n, node, node_off, pred, pred_off, query, query_off);
    SeamOutBufs out;
    DevBuf<int32_t> d_lastH, d_lastE; DevBuf<uint8_t> d_argH, d_argE; DevBuf<uint32_t> d_colstart, d_seqoff, d_seqlen;
    SwBatch b;
    int rc;
    if ((rc = dag.validate(d, "gb_sw_batch")) || (rc = dag.check_limits("gb_sw_batch")) || (rc = dag.upload(d->stream, b.dag))) return rc;
    const uint64_t cols = dag.col_off[n] + 1, nodes = dag.total_nodes + 1;
    if ((rc = out.reserve(n, map_cap, edit_cap))) return rc;
    if ((rc = d_lastH.reserve(cols)) || (rc = d_lastE.reserve(cols)) || (rc = d_argH.reserve(cols)) || (rc = d_argE.reserve(cols))) return rc;
    if ((rc = d_colstart.reserve(nodes)) || (rc = d_seqoff.reserve(nodes)) || (rc = d_seqlen.reserve(nodes))) return rc;
    b.out = out.view;
    b.lastH = d_lastH.ptr; b.lastE = d_lastE.ptr; b.argH = d_argH.ptr; b.argE = d_argE.ptr;
    b.col_start = d_colstart.ptr; b.seq_off = d_seqoff.ptr; b.seq_len = d_seqlen.ptr;
    if ((rc = launch_warp_per_problem(d, sw_kernel, b, SW_WARPS, dp_smem_per_warp(dag.Lc) * SW_WARPS))) return rc;
    return out.download(d, n, score, maps, edits, n_maps, n_edits, status);
}
