// banded_global.cu — stage seam gb_banded_global_batch: Aligner::align_global_banded on a batch of DAG
// problems posed like gb_sw_batch, plus the band padding and permissive flag of each.  The DP itself is
// banded_global.cuh; this file sizes the workspaces, launches one warp per problem and copies back.
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "banded_global.cuh"

#include <algorithm>
#include <vector>

namespace gb {

constexpr int BG_WARPS = 4;

struct BgBatch {
    const uint32_t* node; const uint64_t* node_off;
    const uint32_t* pred; const uint64_t* pred_off;
    const uint8_t* query; const uint64_t* query_off;
    const int32_t* pad; const uint8_t* permissive;
    uint32_t n; uint32_t Lc;
    int32_t* score; gb_mapping* maps; uint32_t* edits; uint32_t* n_maps; uint32_t* n_edits; uint8_t* status;
    uint32_t map_cap, edit_cap;
    BgNode* nd; int64_t* sts; int64_t* lts;                          // per global node
    int32_t* lastM; int32_t* lastI; int32_t* lastD; uint8_t* argd; uint8_t* argh; const uint64_t* col_off;
    uint8_t* tb; const uint64_t* tb_off;
    uint32_t* steps; const uint64_t* step_off;
    uint32_t* work_counter;
};

__host__ __device__ inline size_t bg_smem_per_warp(uint32_t Lc) {
    const size_t W = (size_t)Lc + 1, Wb = (W + 15) & ~(size_t)15;
    return (((size_t)Lc + 15) & ~(size_t)15) + W * 4 * 8 + 2 * Wb + 64;
}

__global__ void __launch_bounds__(BG_WARPS * 32)
banded_global_kernel(DevIndex ix, DevScores sc, BgBatch b) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t W = (size_t)b.Lc + 1, Wb = (W + 15) & ~(size_t)15;
    uint8_t* base = smem + (size_t)warp * bg_smem_per_warp(b.Lc);
    uint8_t* q = base;
    int32_t* rows = reinterpret_cast<int32_t*>(base + (((size_t)b.Lc + 15) & ~(size_t)15));
    uint8_t* brows = reinterpret_cast<uint8_t*>(rows + 8 * W);
    while (true) {
        uint32_t p = 0;
        if (lane == 0) p = atomicAdd(b.work_counter, 1u);
        p = __shfl_sync(FULL, p, 0);
        if (p >= b.n) break;
        uint32_t status = GB_ITEM_OK; int32_t score = 0;
        PathBuf out; out.maps = b.maps + (size_t)p * b.map_cap; out.edits = b.edits + (size_t)p * b.edit_cap;
        out.map_cap = b.map_cap; out.edit_cap = b.edit_cap; pb_reset(out);
        {
            BgSmem s;
            s.pM = rows; s.pI = rows + W; s.pD = rows + 2 * W; s.cM = rows + 3 * W; s.cI = rows + 4 * W; s.cD = rows + 5 * W;
            s.xd = rows + 6 * W; s.xh = rows + 7 * W; s.sd = brows; s.sh = brows + Wb;
            const uint64_t n0 = b.node_off[p];
            BgView v;
            v.N = (uint32_t)(b.node_off[p + 1] - n0); v.node = b.node + n0;
            v.pred = b.pred; v.pred_off = b.pred_off + n0;
            v.nd = b.nd + n0; v.sts = b.sts + n0; v.lts = b.lts + n0;
            v.lastM = b.lastM + b.col_off[p]; v.lastI = b.lastI + b.col_off[p]; v.lastD = b.lastD + b.col_off[p];
            v.argd = b.argd + b.col_off[p]; v.argh = b.argh + b.col_off[p];
            v.tb = b.tb + b.tb_off[p]; v.steps = b.steps + b.step_off[p];
            const uint64_t q0 = b.query_off[p];
            bg_align(ix, sc, v, b.query + q0, (uint32_t)(b.query_off[p + 1] - q0), b.pad[p], b.permissive[p] != 0, q, s, score, out, status);
        }
        if (lane == 0) {
            const bool ok = status == GB_ITEM_OK;
            b.score[p] = ok ? score : 0; b.n_maps[p] = ok ? out.n_maps : 0; b.n_edits[p] = ok ? out.n_edits : 0; b.status[p] = (uint8_t)status;
        }
        __syncwarp();
    }
}

} // namespace gb

using namespace gb;

extern "C" int gb_banded_global_batch(gb_device* d, uint32_t n,
                                      const uint32_t* node, const uint64_t* node_off, const uint32_t* pred, const uint64_t* pred_off,
                                      const uint8_t* query, const uint64_t* query_off, const int32_t* band_padding, const uint8_t* permissive,
                                      uint32_t map_cap, uint32_t edit_cap,
                                      int32_t* score, gb_mapping* maps, uint32_t* edits, uint32_t* n_maps, uint32_t* n_edits, uint8_t* status) {
    if (!d || !node || !node_off || !pred || !pred_off || !query || !query_off || !band_padding || !permissive || !score || !maps ||
        !edits || !n_maps || !n_edits || !status || map_cap == 0 || edit_cap == 0) return GB_ERR_ARG;
    if (n == 0) return GB_OK;
    GB_CUDA(cudaSetDevice(d->device));
    const uint64_t total_nodes = node_off[n], total_pred = pred_off[total_nodes], total_q = query_off[n];
    // validate the DAG shape (predecessors precede, known non-empty nodes, at most 255 predecessors) and size the workspaces
    uint32_t max_q = 0;
    std::vector<uint64_t> col_off(n + 1, 0), tb_off(n + 1, 0), step_off(n + 1, 0);
    std::vector<int32_t> pad(n);
    for (uint32_t p = 0; p < n; p++) {
        const uint32_t m = (uint32_t)(query_off[p + 1] - query_off[p]);
        max_q = std::max(max_q, m);
        if (band_padding[p] < 0) { g_last_error = "gb_banded_global_batch: negative band padding"; return GB_ERR_ARG; }
        uint64_t bases = 0;
        const uint64_t N = node_off[p + 1] - node_off[p];
        // traceback steps carry the node index in 24 bits
        if (N >= (1u << 24)) { g_last_error = "gb_banded_global_batch: more than 2^24 - 1 nodes in a problem"; return GB_ERR_ARG; }
        for (uint64_t u = 0; u < N; u++) {
            const uint32_t v = node[node_off[p] + u];
            if (v < 2 || v >= d->ix.n_nodes || d->h_node_len[v] == 0) { g_last_error = "gb_banded_global_batch: unknown node"; return GB_ERR_ARG; }
            const uint64_t g = node_off[p] + u;
            if (pred_off[g + 1] - pred_off[g] > 255) { g_last_error = "gb_banded_global_batch: more than 255 predecessors"; return GB_ERR_ARG; }
            for (uint64_t e = pred_off[g]; e < pred_off[g + 1]; e++)
                if (pred[e] >= u) { g_last_error = "gb_banded_global_batch: nodes are not in topological order"; return GB_ERR_ARG; }
            bases += d->h_node_len[v];
        }
        // bands are int32 on the device: keep every diagonal within 2 * (m + bases) + 1
        if (bases > (1u << 28)) { g_last_error = "gb_banded_global_batch: more than 2^28 bases in a problem"; return GB_ERR_ARG; }
        // a padding of m + bases + 1 already puts every cell in the band, permissive or not, and masks no node;
        // a wider one gives the same alignment
        pad[p] = (int32_t)std::min<int64_t>(band_padding[p], (int64_t)m + (int64_t)bases + 1);
        col_off[p + 1] = col_off[p] + N * (uint64_t)(m + 1);
        tb_off[p + 1] = tb_off[p] + bases * (uint64_t)(m + 1);
        step_off[p + 1] = step_off[p] + bases + m + 2;
    }
    const uint32_t Lc = std::max<uint32_t>(32u, (max_q + 15u) & ~15u);
    if (Lc > 1024) { g_last_error = "query too long"; return GB_ERR_ARG; }
    if (tb_off[n] > (uint64_t)8 << 30) { g_last_error = "gb_banded_global_batch: batch needs more than 8 GiB of traceback"; return GB_ERR_CAPACITY; }
    DevBuf<uint32_t> d_node, d_pred, d_edits, d_nm, d_ne, d_counter, d_steps;
    DevBuf<uint64_t> d_noff, d_poff, d_qoff, d_coloff, d_tboff, d_stepoff;
    DevBuf<int32_t> d_score, d_pad, d_lastM, d_lastI, d_lastD; DevBuf<int64_t> d_sts, d_lts;
    DevBuf<uint8_t> d_q, d_perm, d_status, d_argd, d_argh, d_tb; DevBuf<gb_mapping> d_maps; DevBuf<BgNode> d_nd;
    int rc;
    if ((rc = d_node.upload(node, total_nodes ? total_nodes : 1, d->stream, total_nodes))) return rc;
    if ((rc = d_pred.upload(pred, total_pred ? total_pred : 1, d->stream, total_pred))) return rc;
    if ((rc = d_noff.upload(node_off, n + 1, d->stream))) return rc;
    if ((rc = d_poff.upload(pred_off, total_nodes + 1, d->stream))) return rc;
    if ((rc = d_q.upload(query, total_q ? total_q : 1, d->stream, total_q))) return rc;
    if ((rc = d_qoff.upload(query_off, n + 1, d->stream))) return rc;
    if ((rc = d_pad.upload(pad.data(), n, d->stream))) return rc;
    if ((rc = d_perm.upload(permissive, n, d->stream))) return rc;
    if ((rc = d_coloff.upload(col_off.data(), n + 1, d->stream))) return rc;
    if ((rc = d_tboff.upload(tb_off.data(), n + 1, d->stream))) return rc;
    if ((rc = d_stepoff.upload(step_off.data(), n + 1, d->stream))) return rc;
    if ((rc = d_score.reserve(n)) || (rc = d_nm.reserve(n)) || (rc = d_ne.reserve(n)) || (rc = d_status.reserve(n))) return rc;
    if ((rc = d_maps.reserve((size_t)n * map_cap)) || (rc = d_edits.reserve((size_t)n * edit_cap))) return rc;
    if ((rc = d_lastM.reserve(col_off[n] + 1)) || (rc = d_lastI.reserve(col_off[n] + 1)) || (rc = d_lastD.reserve(col_off[n] + 1))) return rc;
    if ((rc = d_argd.reserve(col_off[n] + 1)) || (rc = d_argh.reserve(col_off[n] + 1))) return rc;
    if ((rc = d_tb.reserve(tb_off[n] + 1)) || (rc = d_steps.reserve(step_off[n] + 1))) return rc;
    if ((rc = d_nd.reserve(total_nodes + 1)) || (rc = d_sts.reserve(total_nodes + 1)) || (rc = d_lts.reserve(total_nodes + 1))) return rc;
    if ((rc = d_counter.reserve(4))) return rc;
    GB_CUDA(cudaMemsetAsync(d_counter.ptr, 0, 16, d->stream));
    const size_t smem = bg_smem_per_warp(Lc) * BG_WARPS;
    if (smem > 48 * 1024) GB_CUDA(cudaFuncSetAttribute(banded_global_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int bps = 0;
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, banded_global_kernel, BG_WARPS * 32, smem));
    if (bps < 1) bps = 1;
    const uint32_t grid = std::max<uint32_t>(1u, std::min<uint32_t>((uint32_t)d->n_sms * bps, (n + BG_WARPS - 1) / BG_WARPS));
    BgBatch b;
    b.node = d_node.ptr; b.node_off = d_noff.ptr; b.pred = d_pred.ptr; b.pred_off = d_poff.ptr; b.query = d_q.ptr; b.query_off = d_qoff.ptr;
    b.pad = d_pad.ptr; b.permissive = d_perm.ptr;
    b.n = n; b.Lc = Lc; b.score = d_score.ptr; b.maps = d_maps.ptr; b.edits = d_edits.ptr; b.n_maps = d_nm.ptr; b.n_edits = d_ne.ptr;
    b.status = d_status.ptr; b.map_cap = map_cap; b.edit_cap = edit_cap;
    b.nd = d_nd.ptr; b.sts = d_sts.ptr; b.lts = d_lts.ptr;
    b.lastM = d_lastM.ptr; b.lastI = d_lastI.ptr; b.lastD = d_lastD.ptr; b.argd = d_argd.ptr; b.argh = d_argh.ptr; b.col_off = d_coloff.ptr;
    b.tb = d_tb.ptr; b.tb_off = d_tboff.ptr; b.steps = d_steps.ptr; b.step_off = d_stepoff.ptr; b.work_counter = d_counter.ptr;
    GB_CUDA(cudaEventRecord(d->ev0, d->stream));
    banded_global_kernel<<<grid, BG_WARPS * 32, smem, d->stream>>>(d->ix, d->sc, b);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaEventRecord(d->ev1, d->stream));
    GB_CUDA(cudaMemcpyAsync(score, d_score.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(n_maps, d_nm.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(n_edits, d_ne.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(status, d_status.ptr, n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(maps, d_maps.ptr, sizeof(gb_mapping) * (size_t)n * map_cap, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(edits, d_edits.ptr, 4 * (size_t)n * edit_cap, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));
    GB_CUDA(cudaEventElapsedTime(&d->last_kernel_ms, d->ev0, d->ev1));
    return GB_OK;
}
