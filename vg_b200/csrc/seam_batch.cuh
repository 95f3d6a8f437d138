// seam_batch.cuh — what the batched alignment seams (gb_sw_batch, gb_xdrop_dag_batch, gb_banded_global_batch,
// gb_xdrop_pinned_batch) have in common: the per-problem output arrays, the query-width rule, and for the three
// DAG seams the validation, workspace sizing and upload of the problems and the launch of a persistent
// one-warp-per-problem kernel.  What differs between the seams stays in their own files.
#pragma once
#include "device_state.cuh"

#include <algorithm>
#include <string>
#include <vector>

namespace gb {

// Per-problem outputs: score, status and counts per problem, map_cap mappings and edit_cap edit words per problem.
struct SeamOut {
    int32_t* score; gb_mapping* maps; uint32_t* edits; uint32_t* n_maps; uint32_t* n_edits; uint8_t* status;
    uint32_t map_cap, edit_cap;

    // problem p's output path, empty
    __device__ PathBuf path(uint32_t p) const {
        PathBuf o; o.maps = maps + (size_t)p * map_cap; o.edits = edits + (size_t)p * edit_cap;
        o.map_cap = map_cap; o.edit_cap = edit_cap; pb_reset(o);
        return o;
    }
    // lane 0 writes problem p's per-problem values
    __device__ void store(uint32_t p, int32_t s, uint32_t nm, uint32_t ne, uint32_t st) const {
        if ((threadIdx.x & 31) == 0) { score[p] = s; n_maps[p] = nm; n_edits[p] = ne; status[p] = (uint8_t)st; }
    }
};

// The device arrays behind a SeamOut.
struct SeamOutBufs {
    DevBuf<int32_t> score; DevBuf<gb_mapping> maps; DevBuf<uint32_t> edits, n_maps, n_edits; DevBuf<uint8_t> status;
    SeamOut view{};

    int reserve(uint32_t n, uint32_t map_cap, uint32_t edit_cap) {
        int rc;
        if ((rc = score.reserve(n)) || (rc = n_maps.reserve(n)) || (rc = n_edits.reserve(n)) || (rc = status.reserve(n))) return rc;
        if ((rc = maps.reserve((size_t)n * map_cap)) || (rc = edits.reserve((size_t)n * edit_cap))) return rc;
        view = SeamOut{score.ptr, maps.ptr, edits.ptr, n_maps.ptr, n_edits.ptr, status.ptr, map_cap, edit_cap};
        return GB_OK;
    }
    // copies the outputs of n problems into the caller's arrays, waits for the stream and records the time
    // between d->ev0 and d->ev1 as last_kernel_ms
    int download(gb_device* d, uint32_t n, int32_t* h_score, gb_mapping* h_maps, uint32_t* h_edits, uint32_t* h_n_maps,
                 uint32_t* h_n_edits, uint8_t* h_status) {
        GB_CUDA(cudaMemcpyAsync(h_score, score.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(h_n_maps, n_maps.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(h_n_edits, n_edits.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(h_status, status.ptr, n, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(h_maps, maps.ptr, sizeof(gb_mapping) * (size_t)n * view.map_cap, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(h_edits, edits.ptr, 4 * (size_t)n * view.edit_cap, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaStreamSynchronize(d->stream));
        GB_CUDA(cudaEventElapsedTime(&d->last_kernel_ms, d->ev0, d->ev1));
        return GB_OK;
    }
};

// Query columns of the per-warp DP buffers: the longest query rounded up to 16, at least 32.  The one-warp
// kernels hold at most 1024.
inline int query_columns(uint32_t max_q, uint32_t& Lc) {
    Lc = std::max<uint32_t>(32u, (max_q + 15u) & ~15u);
    if (Lc > 1024) { g_last_error = "query too long"; return GB_ERR_ARG; }
    return GB_OK;
}

// Device view of a batch of DAG problems.  Problem p: nodes node_off[p] .. node_off[p + 1] in topological order,
// their predecessors as a CSR over the global node index whose entries are positions within the problem, query
// query_off[p] .. query_off[p + 1].  Its workspaces start at col_off[p] (N * (m + 1) cells), tb_off[p] (one
// traceback byte per base and query prefix) and step_off[p] (bases + m + 2 traceback steps).
struct DagDev {
    const uint32_t* node; const uint64_t* node_off;
    const uint32_t* pred; const uint64_t* pred_off;
    const uint8_t* query; const uint64_t* query_off;
    const uint64_t* col_off;
    uint8_t* tb; const uint64_t* tb_off;
    uint32_t* steps; const uint64_t* step_off;
    uint32_t n, Lc;

    // fills the fields of problem p's DagView or BgView that come from here; returns the problem's first global node
    template <class View> __device__ uint64_t view(uint32_t p, View& v) const {
        const uint64_t n0 = node_off[p];
        v.N = (uint32_t)(node_off[p + 1] - n0); v.node = node + n0;
        v.pred = pred; v.pred_off = pred_off + n0;
        v.tb = tb + tb_off[p]; v.steps = steps + step_off[p];
        return n0;
    }
    __device__ const uint8_t* read(uint32_t p, uint32_t& m) const {
        const uint64_t q0 = query_off[p];
        m = (uint32_t)(query_off[p + 1] - q0);
        return query + q0;
    }
};

// The host side of a DagDev: the caller's arrays, what validate() derives from them, and their device copies.
struct DagProblems {
    uint32_t n; const uint32_t* node; const uint64_t* node_off; const uint32_t* pred; const uint64_t* pred_off;
    const uint8_t* query; const uint64_t* query_off;
    uint64_t total_nodes = 0;
    std::vector<uint32_t> m;                                  // per problem: query length,
    std::vector<uint64_t> N, bases;                           // node count and bases
    std::vector<uint64_t> col_off, tb_off, step_off;          // [n + 1] workspace offsets
    uint32_t max_q = 0, Lc = 0;
    DevBuf<uint32_t> d_node, d_pred, d_steps; DevBuf<uint64_t> d_noff, d_poff, d_qoff, d_coloff, d_tboff, d_stepoff;
    DevBuf<uint8_t> d_q, d_tb;

    DagProblems(uint32_t n_, const uint32_t* node_, const uint64_t* node_off_, const uint32_t* pred_, const uint64_t* pred_off_,
                const uint8_t* query_, const uint64_t* query_off_)
        : n(n_), node(node_), node_off(node_off_), pred(pred_), pred_off(pred_off_), query(query_), query_off(query_off_) {}

    // Refuses unknown nodes, nodes with more than 255 predecessors and predecessors that do not precede their
    // node; sizes the workspaces.
    int validate(const gb_device* d, const char* who) {
        total_nodes = node_off[n];
        m.assign(n, 0); N.assign(n, 0); bases.assign(n, 0);
        col_off.assign(n + 1, 0); tb_off.assign(n + 1, 0); step_off.assign(n + 1, 0);
        for (uint32_t p = 0; p < n; p++) {
            m[p] = (uint32_t)(query_off[p + 1] - query_off[p]);
            max_q = std::max(max_q, m[p]);
            N[p] = node_off[p + 1] - node_off[p];
            for (uint64_t u = 0; u < N[p]; u++) {
                const uint64_t g = node_off[p] + u;
                const uint32_t v = node[g];
                if (v < 2 || v >= d->ix.n_nodes) return fail(who, ": unknown node");
                if (pred_off[g + 1] - pred_off[g] > 255) return fail(who, ": more than 255 predecessors");
                for (uint64_t e = pred_off[g]; e < pred_off[g + 1]; e++)
                    if (pred[e] >= u) return fail(who, ": nodes are not in topological order");
                bases[p] += d->h_node_len[v];
            }
            col_off[p + 1] = col_off[p] + N[p] * (uint64_t)(m[p] + 1);
            tb_off[p + 1] = tb_off[p] + bases[p] * (uint64_t)(m[p] + 1);
            step_off[p + 1] = step_off[p] + bases[p] + m[p] + 2;
        }
        return GB_OK;
    }
    // The batch-wide limits, checked after validate() and the seam's own checks: the query width and 8 GiB of traceback.
    int check_limits(const char* who) {
        int rc;
        if ((rc = query_columns(max_q, Lc))) return rc;
        if (tb_off[n] > (uint64_t)8 << 30) { g_last_error = std::string(who) + ": batch needs more than 8 GiB of traceback"; return GB_ERR_CAPACITY; }
        return GB_OK;
    }
    int upload(cudaStream_t s, DagDev& v) {
        const uint64_t total_pred = pred_off[total_nodes], total_q = query_off[n];
        int rc;
        if ((rc = d_node.upload(node, total_nodes ? total_nodes : 1, s, total_nodes))) return rc;
        if ((rc = d_pred.upload(pred, total_pred ? total_pred : 1, s, total_pred))) return rc;
        if ((rc = d_noff.upload(node_off, n + 1, s))) return rc;
        if ((rc = d_poff.upload(pred_off, total_nodes + 1, s))) return rc;
        if ((rc = d_q.upload(query, total_q ? total_q : 1, s, total_q))) return rc;
        if ((rc = d_qoff.upload(query_off, n + 1, s))) return rc;
        if ((rc = d_coloff.upload(col_off.data(), n + 1, s))) return rc;
        if ((rc = d_tboff.upload(tb_off.data(), n + 1, s))) return rc;
        if ((rc = d_stepoff.upload(step_off.data(), n + 1, s))) return rc;
        if ((rc = d_tb.reserve(tb_off[n] + 1)) || (rc = d_steps.reserve(step_off[n] + 1))) return rc;
        v = DagDev{d_node.ptr, d_noff.ptr, d_pred.ptr, d_poff.ptr, d_q.ptr, d_qoff.ptr, d_coloff.ptr,
                   d_tb.ptr, d_tboff.ptr, d_steps.ptr, d_stepoff.ptr, n, Lc};
        return GB_OK;
    }
    static int fail(const char* who, const char* what) { g_last_error = std::string(who) + what; return GB_ERR_ARG; }
};

// Launches a persistent kernel that runs one warp per problem, `warps` warps per block, over b.n problems:
// as many blocks as are resident at once, at most one warp per problem.  d->work_counter hands out the
// problems; ev0 / ev1 bracket the launch alone.
template <class Batch>
int launch_warp_per_problem(gb_device* d, void (*kernel)(DevIndex, DevScores, Batch), Batch b, int warps, size_t smem) {
    if (smem > 48 * 1024) GB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int bps = 0;
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, kernel, warps * 32, smem));
    if (bps < 1) bps = 1;
    const uint32_t grid = std::max<uint32_t>(1u, std::min<uint32_t>((uint32_t)d->n_sms * bps, (b.dag.n + warps - 1) / warps));
    b.work_counter = d->work_counter;
    GB_CUDA(cudaMemsetAsync(d->work_counter, 0, sizeof(uint32_t), d->stream));
    GB_CUDA(cudaEventRecord(d->ev0, d->stream));
    kernel<<<grid, warps * 32, smem, d->stream>>>(d->ix, d->sc, b);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaEventRecord(d->ev1, d->stream));
    return GB_OK;
}

} // namespace gb
