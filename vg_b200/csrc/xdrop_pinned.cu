// xdrop_pinned.cu — B3 stage seam: Aligner::align_pinned(xdrop = true), batched over explicit haplotype trees
// (aligner.cpp:628-686 -> DozeuInterface::align_pinned dozeu_interface.cpp:724-766).
//
// Problems the int16 tile kernel can hold are packed into tiles and run on xdrop_tile_kernel (xdrop_tile.cuh, the
// production path of the mapping tails); the rest, and the tiles that outgrow the tile's path capacities, run on the
// int32 column sweep of tail.cuh, one warp per problem.  Both compute the same function.
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "seam_batch.cuh"

#include <algorithm>
#include <string>
#include <vector>

namespace gb {

constexpr int XP_WARPS = 4;

struct XdropBatch {
    const int32_t* tree_parent; const uint32_t* tree_node; const uint64_t* tree_off; const uint32_t* root_trim;
    const uint8_t* query; const uint64_t* query_off; const uint32_t* max_gap;
    uint32_t n; uint32_t Lc;
    SeamOut out;
    uint8_t* ws_base; size_t ws_stride; uint32_t tb_cells;
    uint32_t* work_counter;
    uint8_t* skip;                   // [n] 1: the problem ran on xdrop_tile_kernel instead
};

// ---- tiles from explicit trees ---------------------------------------------------------------------------------------
struct PackBatch {
    const int32_t* tree_parent; const uint32_t* tree_node; const uint64_t* tree_off; const uint32_t* root_trim;
    const uint8_t* query; const uint64_t* query_off; const uint32_t* max_gap; uint32_t n;
    uint8_t* tiles; const uint32_t* tile_off;      // precomputed on the host
    uint32_t* lists[TILE_CLASSES]; uint32_t* list_count;      // [TILE_CLASSES]
    uint8_t* eligible;                              // [n] 0: not a tile problem (host falls back to the int32 kernel)
};
__global__ void pack_tiles_kernel(DevIndex ix, DevScores sc, PackBatch b) {
    const uint32_t p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (p >= b.n || !b.eligible[p]) return;
    const uint64_t t0 = b.tree_off[p]; const uint32_t nt = (uint32_t)(b.tree_off[p + 1] - t0);
    const uint64_t q0 = b.query_off[p]; const uint32_t m = (uint32_t)(b.query_off[p + 1] - q0);
    uint8_t* tile = b.tiles + (size_t)b.tile_off[p] * 16;
    TileNode* nodes = reinterpret_cast<TileNode*>(tile + 32);
    uint32_t n_bases = 0;
    for (uint32_t i = 0; i < nt; i++) {                       // sequential prefix (small trees; the stage seam is not a hot path)
        const uint32_t v = b.tree_node[t0 + i];
        const gb_node_rec nr = load_node(ix, v);
        const uint32_t trim = b.tree_parent[t0 + i] < 0 ? b.root_trim[p] : 0u;
        if (lane == 0) { TileNode tn; tn.parent = b.tree_parent[t0 + i] < 0 ? 0xffffu : (uint16_t)b.tree_parent[t0 + i]; tn.len = (uint16_t)(nr.len - trim); tn.node = v; nodes[i] = tn; }
        n_bases += nr.len - trim;
    }
    uint8_t* bases = tile + 32 + 8 * ((nt + 1u) & ~1u);
    uint32_t at = 0;
    for (uint32_t i = 0; i < nt; i++) {
        const uint32_t v = b.tree_node[t0 + i];
        const gb_node_rec nr = load_node(ix, v);
        const uint32_t trim = b.tree_parent[t0 + i] < 0 ? b.root_trim[p] : 0u;
        for (uint32_t x = lane; x < nr.len - trim; x += 32) bases[at + x] = __ldg(ix.seq + nr.seq_off + trim + x);
        at += nr.len - trim;
    }
    uint8_t* q = bases + ((n_bases + 15u) & ~15u);
    for (uint32_t x = lane; x < m; x += 32) q[x] = dp_query_base(b.query[q0 + x]);
    if (lane == 0) {
        TileHeader hd; hd.m = m; hd.n_nodes = nt; hd.n_bases = n_bases; hd.max_gap = max(b.max_gap[p], 1u); hd.flags = GB_TILE_TREE_SPACE;
        hd.root_trim = b.root_trim[p]; hd.bytes = tile_bytes(nt, n_bases, m); hd.result = p;
        *reinterpret_cast<TileHeader*>(tile) = hd;
        const int cls = tile_class(m);
        b.lists[cls][atomicAdd(&b.list_count[cls], 1u)] = p;
    }
}

// Counters of the tile route: per size class the list count and the work counter, and the result path cursor.
struct TileCounters {
    uint32_t list_count[TILE_CLASSES];
    uint32_t work[TILE_CLASSES];
    uint32_t path_words;
};

// results of the tile kernel -> the seam's output arrays.  A tile that outgrew the tile's own path capacities
// (TILE_MAP_CAP / TILE_EDIT_CAP / TILE_STEP_CAP) gives its problem back to xdrop_kernel, which aligns it within the
// caller's map_cap / edit_cap: the seam's answer does not depend on which kernel a problem was routed to.
__global__ void unpack_tile_results_kernel(XdropBatch b, const TileResult* results, const uint32_t* path_pool) {
    const uint32_t p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (p >= b.n || !b.skip[p]) return;
    const TileResult tr = results[p];
    if (tr.status != GB_TILE_ST_OK) {
        if (lane == 0) b.skip[p] = 0;
        return;
    }
    uint32_t status = GB_ITEM_OK;
    if (tr.n_maps > b.out.map_cap || tr.n_edits > b.out.edit_cap) status = GB_ITEM_OUT_FULL;
    if (status == GB_ITEM_OK) {
        const gb_mapping* gm = reinterpret_cast<const gb_mapping*>(path_pool + tr.path_off);
        const uint32_t* ge = path_pool + tr.path_off + 2 * tr.n_maps;
        for (uint32_t i = lane; i < tr.n_maps; i += 32) b.out.maps[(size_t)p * b.out.map_cap + i] = gm[i];
        for (uint32_t i = lane; i < tr.n_edits; i += 32) b.out.edits[(size_t)p * b.out.edit_cap + i] = ge[i];
    }
    const bool ok = status == GB_ITEM_OK;
    b.out.store(p, ok ? tr.score : 0, ok ? tr.n_maps : 0, ok ? tr.n_edits : 0, status);
}

__global__ void __launch_bounds__(XP_WARPS * 32, 4)
xdrop_kernel(DevIndex ix, DevScores sc, XdropBatch b) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t gwarp = blockIdx.x * XP_WARPS + warp;
    uint8_t* q;
    const DpSmem dps = dp_smem_carve(smem, warp, b.Lc, q);
    const TailWs ws = carve_tail_ws(b.ws_base + (size_t)gwarp * b.ws_stride, b.Lc, b.tb_cells);
    while (true) {
        uint32_t p = 0;
        if (lane == 0) p = atomicAdd(b.work_counter, 1u);
        p = __shfl_sync(FULL, p, 0);
        if (p >= b.n) break;
        if (b.skip && b.skip[p]) continue;
        const uint64_t t_begin = b.tree_off[p]; const uint32_t nt = (uint32_t)(b.tree_off[p + 1] - t_begin);
        const uint64_t q_begin = b.query_off[p]; const uint32_t m = (uint32_t)(b.query_off[p + 1] - q_begin);
        uint32_t status = GB_ITEM_OK; int32_t score = 0;
        PathBuf out = b.out.path(p);
        if (nt == 0 || nt > TAIL_T_CAP || m > b.Lc) status = GB_ITEM_OUT_FULL;
        else {
            for (uint32_t i = lane; i < m; i += 32) q[i] = dp_query_base(b.query[q_begin + i]);
            // materialise the tree (depths from parents)
            if (lane == 0) {
                for (uint32_t i = 0; i < nt; i++) {
                    TreeNode t; t.parent = b.tree_parent[t_begin + i]; t.node = b.tree_node[t_begin + i];
                    const gb_node_rec nr = load_node(ix, t.node);
                    const uint32_t trim = t.parent < 0 ? b.root_trim[p] : 0u;
                    t.seq_off = nr.seq_off + trim; t.len = nr.len - trim;
                    t.depth = t.parent < 0 ? 0u : ws.tree[t.parent].depth + 1;
                    t.tb_col = 0; t.lineage_max = 0; t.computed = 0;
                    ws.tree[i] = t;
                }
            }
            __syncwarp();
            bool ovf = false;
            score = xdrop_tree(ix, sc, ws, dps, 0, nt, q, m, max(b.max_gap[p], 1u), out, ovf);
            if (ovf || out.overflow) status = GB_ITEM_OUT_FULL;
        }
        b.out.store(p, score, out.n_maps, out.n_edits, status);
        __syncwarp();
    }
}

} // namespace gb

using namespace gb;

extern "C" int gb_xdrop_pinned_batch(gb_device* d, uint32_t n,
                                     const int32_t* tree_parent, const uint32_t* tree_node, const uint64_t* tree_off,
                                     const uint32_t* root_trim, const uint8_t* query, const uint64_t* query_off,
                                     const uint32_t* max_gap, uint32_t map_cap, uint32_t edit_cap,
                                     int32_t* score, gb_mapping* maps, uint32_t* edits, uint32_t* n_maps, uint32_t* n_edits,
                                     uint8_t* status) {
    return gb::guarded("gb_xdrop_pinned_batch", [&] {
        if (!d || !tree_parent || !tree_node || !tree_off || !root_trim || !query || !query_off || !max_gap || !score || !maps ||
            !edits || !n_maps || !n_edits || !status || map_cap == 0 || edit_cap == 0) return GB_ERR_ARG;
        if (n == 0) return GB_OK;
        // ---- validation, before anything reaches the device: known nodes; one root, first; the nodes in DFS visit order (both
        // kernels keep one DP column per tree level, which a node's parent must still own); the root trim leaves a base; fewer
        // than TAIL_D_CAP levels ----
        std::vector<uint64_t> prob_bases(n, 0); std::vector<uint32_t> prob_depth(n, 0), lineage;
        uint32_t max_q = 0, Lc;
        auto fail = [](const char* what) { g_last_error = std::string("gb_xdrop_pinned_batch: ") + what; return GB_ERR_ARG; };
        for (uint32_t i = 0; i < n; i++) {
            max_q = std::max<uint32_t>(max_q, (uint32_t)(query_off[i + 1] - query_off[i]));
            const uint64_t t0 = tree_off[i]; const uint32_t ntree = (uint32_t)(tree_off[i + 1] - t0);
            if (ntree == 0) return fail("empty tree");
            if (max_gap[i] > 65535) return fail("max_gap above 65535");      // vg's max_gap is a uint16_t
            lineage.clear();                     // root .. previous node
            for (uint32_t x = 0; x < ntree; x++) {
                const uint32_t v = tree_node[t0 + x]; const int32_t par = tree_parent[t0 + x];
                if (v < 2 || v >= d->ix.n_nodes || d->h_node_len[v] == 0) return fail("unknown node");
                if (x == 0 && par >= 0) return fail("the first tree node is not a root");
                if (x > 0 && par < 0) return fail("more than one root");
                if (par >= (int32_t)x) return fail("a parent does not precede its child");
                while (par >= 0 && !lineage.empty() && lineage.back() != (uint32_t)par) lineage.pop_back();
                if (par >= 0 && lineage.empty()) return fail("tree nodes are not in DFS visit order");
                lineage.push_back(x);
                const uint32_t len = d->h_node_len[v];
                if (par < 0) {
                    if (root_trim[i] >= len) return fail("root_trim leaves no base of the root");
                    prob_bases[i] += len - root_trim[i];
                } else prob_bases[i] += len;
                if (lineage.size() > TAIL_D_CAP) return fail("tree deeper than 511 levels");
                prob_depth[i] = std::max<uint32_t>(prob_depth[i], (uint32_t)lineage.size() - 1);
            }
        }
        int rc;
        if ((rc = query_columns(max_q, Lc))) return rc;
        GB_CUDA(cudaSetDevice(d->device));
        DevBuf<int32_t> d_par; DevBuf<uint32_t> d_node, d_trim, d_gap, d_counter; DevBuf<uint64_t> d_toff, d_qoff;
        DevBuf<uint8_t> d_q, d_ws; SeamOutBufs out;
        const uint64_t nt = tree_off[n], nq = query_off[n];
        if ((rc = d_par.upload(tree_parent, nt ? nt : 1, d->stream, nt))) return rc;
        if ((rc = d_node.upload(tree_node, nt ? nt : 1, d->stream, nt))) return rc;
        if ((rc = d_toff.upload(tree_off, n + 1, d->stream))) return rc;
        if ((rc = d_trim.upload(root_trim, n, d->stream))) return rc;
        if ((rc = d_gap.upload(max_gap, n, d->stream))) return rc;
        if ((rc = d_q.upload(query, nq ? nq : 1, d->stream, nq))) return rc;
        if ((rc = d_qoff.upload(query_off, n + 1, d->stream))) return rc;
        if ((rc = out.reserve(n, map_cap, edit_cap))) return rc;
        if ((rc = d_counter.reserve(4))) return rc;
        GB_CUDA(cudaMemsetAsync(d_counter.ptr, 0, 16, d->stream));
        const size_t smem = dp_smem_per_warp(Lc) * XP_WARPS;
        if (smem > 48 * 1024) GB_CUDA(cudaFuncSetAttribute(xdrop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        uint32_t grid = std::min<uint32_t>((uint32_t)d->n_sms * 2, (n + XP_WARPS - 1) / XP_WARPS);
        const uint32_t tb_cells = 2 * 1024 * 1024;
        const size_t ws_stride = tail_ws_bytes(Lc, tb_cells);
        if ((rc = d_ws.reserve(ws_stride * grid * XP_WARPS))) return rc;
        XdropBatch b;
        b.tree_parent = d_par.ptr; b.tree_node = d_node.ptr; b.tree_off = d_toff.ptr; b.root_trim = d_trim.ptr;
        b.query = d_q.ptr; b.query_off = d_qoff.ptr; b.max_gap = d_gap.ptr; b.n = n; b.Lc = Lc; b.out = out.view;
        b.ws_base = d_ws.ptr; b.ws_stride = ws_stride; b.tb_cells = tb_cells;
        b.work_counter = d_counter.ptr;
        // ---- problems the int16 tile kernel can hold run there (the production path of the tails); the rest on the int32 sweep ----
        std::vector<uint8_t> elig(n, 0); std::vector<uint32_t> toff(n, 0);
        uint64_t units = 0; uint32_t n_elig = 0;
        if (d->use_tiles) {
            for (uint32_t i = 0; i < n; i++) {
                const uint32_t ntree = (uint32_t)(tree_off[i + 1] - tree_off[i]), m = (uint32_t)(query_off[i + 1] - query_off[i]);
                const uint32_t bases = (uint32_t)std::min<uint64_t>(prob_bases[i], 0xffffffffu);
                if (!tile_eligible(d->sc, m, std::max(max_gap[i], 1u), ntree, bases, prob_depth[i])) continue;
                elig[i] = 1; toff[i] = (uint32_t)units; units += tile_bytes(ntree, bases, m) / 16; n_elig++;
            }
        }
        DevBuf<uint8_t> d_elig, d_tiles; DevBuf<uint32_t> d_tileoff, d_lists, d_paths; DevBuf<TileCounters> d_tc; DevBuf<TileResult> d_res;
        GB_CUDA(cudaEventRecord(d->ev0, d->stream));
        if (n_elig) {
            const uint32_t path_cap = (uint32_t)std::min<uint64_t>((uint64_t)n * (2 * TILE_MAP_CAP + TILE_EDIT_CAP), 0xfffffff0ull);
            if ((rc = d_elig.upload(elig.data(), n, d->stream)) || (rc = d_tileoff.upload(toff.data(), n, d->stream)) || (rc = d_tiles.reserve(units * 16 + 16)) ||
                (rc = d_lists.reserve(TILE_CLASSES * (size_t)n)) || (rc = d_tc.reserve(1)) || (rc = d_res.reserve(n)) || (rc = d_paths.reserve(path_cap))) return rc;
            GB_CUDA(cudaMemsetAsync(d_tc.ptr, 0, sizeof(TileCounters), d->stream));
            GB_CUDA(cudaMemsetAsync(d_res.ptr, 0xff, sizeof(TileResult) * (size_t)n, d->stream));
            PackBatch pk;
            pk.tree_parent = d_par.ptr; pk.tree_node = d_node.ptr; pk.tree_off = d_toff.ptr; pk.root_trim = d_trim.ptr;
            pk.query = d_q.ptr; pk.query_off = d_qoff.ptr; pk.max_gap = d_gap.ptr; pk.n = n; pk.tiles = d_tiles.ptr; pk.tile_off = d_tileoff.ptr;
            for (int c = 0; c < TILE_CLASSES; c++) pk.lists[c] = d_lists.ptr + (size_t)c * n;
            pk.list_count = d_tc.ptr->list_count; pk.eligible = d_elig.ptr;
            pack_tiles_kernel<<<(n + 7) / 8, 256, 0, d->stream>>>(d->ix, d->sc, pk);
            d->launches++;
            GB_CUDA(cudaGetLastError());
            d->kt_reset();
            if ((rc = launch_tile_kernels(d, d_tiles.ptr, d_tileoff.ptr, d_lists.ptr, n, d_tc.ptr->list_count, d_tc.ptr->work, d_res.ptr, d_paths.ptr,
                                          path_cap, &d_tc.ptr->path_words))) return rc;
            b.skip = d_elig.ptr;
            unpack_tile_results_kernel<<<(n + 7) / 8, 256, 0, d->stream>>>(b, d_res.ptr, d_paths.ptr);
            d->launches++;
            GB_CUDA(cudaGetLastError());
        } else b.skip = nullptr;
        // the int32 sweep takes the problems not eligible for a tile and those whose tile ended FULL; the latter are known only
        // on the device, so it runs after the tiles too and skips the problems they finished
        xdrop_kernel<<<grid, XP_WARPS * 32, smem, d->stream>>>(d->ix, d->sc, b);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        d->last_tile_problems = n_elig;
        GB_CUDA(cudaEventRecord(d->ev1, d->stream));
        return out.download(d, n, score, maps, edits, n_maps, n_edits, status);
    });
}
