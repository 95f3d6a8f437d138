// banded_global.cu — stage seam gb_banded_global_batch: Aligner::align_global_banded on a batch of DAG
// problems posed like gb_sw_batch, plus the band padding and permissive flag of each.  The DP itself is
// banded_global.cuh; this file runs it one warp per problem, with the checks and workspaces only this seam has
// (the host side the DAG seams share is seam_batch.cuh).
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "banded_global.cuh"
#include "seam_batch.cuh"

namespace gb {

constexpr int BG_WARPS = 4;

struct BgBatch {
    DagDev dag;
    SeamOut out;
    const int32_t* pad; const uint8_t* permissive;
    BgNode* nd; int64_t* sts; int64_t* lts;                          // per global node
    int32_t* lastM; int32_t* lastI; int32_t* lastD; uint8_t* argd; uint8_t* argh;
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
    const size_t W = (size_t)b.dag.Lc + 1, Wb = (W + 15) & ~(size_t)15;
    uint8_t* base = smem + (size_t)warp * bg_smem_per_warp(b.dag.Lc);
    uint8_t* q = base;
    int32_t* rows = reinterpret_cast<int32_t*>(base + (((size_t)b.dag.Lc + 15) & ~(size_t)15));
    uint8_t* brows = reinterpret_cast<uint8_t*>(rows + 8 * W);
    while (true) {
        uint32_t p = 0;
        if (lane == 0) p = atomicAdd(b.work_counter, 1u);
        p = __shfl_sync(FULL, p, 0);
        if (p >= b.dag.n) break;
        uint32_t status = GB_ITEM_OK; int32_t score = 0;
        PathBuf out = b.out.path(p);
        {
            BgSmem s;
            s.pM = rows; s.pI = rows + W; s.pD = rows + 2 * W; s.cM = rows + 3 * W; s.cI = rows + 4 * W; s.cD = rows + 5 * W;
            s.xd = rows + 6 * W; s.xh = rows + 7 * W; s.sd = brows; s.sh = brows + Wb;
            BgView v;
            const uint64_t n0 = b.dag.view(p, v), c0 = b.dag.col_off[p];
            v.nd = b.nd + n0; v.sts = b.sts + n0; v.lts = b.lts + n0;
            v.lastM = b.lastM + c0; v.lastI = b.lastI + c0; v.lastD = b.lastD + c0;
            v.argd = b.argd + c0; v.argh = b.argh + c0;
            uint32_t m;
            const uint8_t* read = b.dag.read(p, m);
            bg_align(ix, sc, v, read, m, b.pad[p], b.permissive[p] != 0, q, s, score, out, status);
        }
        const bool ok = status == GB_ITEM_OK;
        b.out.store(p, ok ? score : 0, ok ? out.n_maps : 0, ok ? out.n_edits : 0, status);
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
    return gb::guarded("gb_banded_global_batch", [&] {
        if (!d || !node || !node_off || !pred || !pred_off || !query || !query_off || !band_padding || !permissive || !score || !maps ||
            !edits || !n_maps || !n_edits || !status || map_cap == 0 || edit_cap == 0) return GB_ERR_ARG;
        if (n == 0) return GB_OK;
        GB_CUDA(cudaSetDevice(d->device));
        DagProblems dag(n, node, node_off, pred, pred_off, query, query_off);
        int rc;
        if ((rc = dag.validate(d, "gb_banded_global_batch"))) return rc;
        std::vector<int32_t> pad(n);
        for (uint32_t p = 0; p < n; p++) {
            if (band_padding[p] < 0) { g_last_error = "gb_banded_global_batch: negative band padding"; return GB_ERR_ARG; }
            // bands are int32 on the device: keep every diagonal within 2 * (m + bases) + 1
            if (dag.bases[p] > (1u << 28)) { g_last_error = "gb_banded_global_batch: more than 2^28 bases in a problem"; return GB_ERR_ARG; }
            // a padding of m + bases + 1 already puts every cell in the band, permissive or not, and masks no node;
            // a wider one gives the same alignment
            pad[p] = (int32_t)std::min<int64_t>(band_padding[p], (int64_t)dag.m[p] + (int64_t)dag.bases[p] + 1);
        }
        BgBatch b;
        if ((rc = dag.check_limits("gb_banded_global_batch")) || (rc = dag.upload(d->stream, b.dag))) return rc;
        SeamOutBufs out;
        DevBuf<int32_t> d_pad, d_lastM, d_lastI, d_lastD; DevBuf<int64_t> d_sts, d_lts;
        DevBuf<uint8_t> d_perm, d_argd, d_argh; DevBuf<BgNode> d_nd;
        const uint64_t cols = dag.col_off[n] + 1, nodes = dag.total_nodes + 1;
        if ((rc = d_pad.upload(pad.data(), n, d->stream)) || (rc = d_perm.upload(permissive, n, d->stream))) return rc;
        if ((rc = out.reserve(n, map_cap, edit_cap))) return rc;
        if ((rc = d_lastM.reserve(cols)) || (rc = d_lastI.reserve(cols)) || (rc = d_lastD.reserve(cols))) return rc;
        if ((rc = d_argd.reserve(cols)) || (rc = d_argh.reserve(cols))) return rc;
        if ((rc = d_nd.reserve(nodes)) || (rc = d_sts.reserve(nodes)) || (rc = d_lts.reserve(nodes))) return rc;
        b.out = out.view;
        b.pad = d_pad.ptr; b.permissive = d_perm.ptr;
        b.nd = d_nd.ptr; b.sts = d_sts.ptr; b.lts = d_lts.ptr;
        b.lastM = d_lastM.ptr; b.lastI = d_lastI.ptr; b.lastD = d_lastD.ptr; b.argd = d_argd.ptr; b.argh = d_argh.ptr;
        if ((rc = launch_warp_per_problem(d, banded_global_kernel, b, BG_WARPS, bg_smem_per_warp(dag.Lc) * BG_WARPS))) return rc;
        return out.download(d, n, score, maps, edits, n_maps, n_edits, status);
    });
}
