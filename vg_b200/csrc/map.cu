// map.cu — gb_map_batch: the single-end Giraffe hot path on the GPU.
//   seed_kernel -> extend_kernel -> align_kernel, all persistent warp-per-unit kernels pulling
//   work from atomic counters; intermediate records stay in HBM (map_state.cuh).
// No CPU fallback: every stage is a CUDA kernel; the host only moves buffers and launches.
#include <cub/cub.cuh>
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "seed.cuh"
#include "align.cuh"
#include "extend.cuh"
#include "dag_dp.cuh"
#include "seam_batch.cuh"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

namespace gb {

int launch_extend_device(gb_device* d, const ExtendParams& p, const uint8_t* reads, const uint64_t* read_off,
                         const uint32_t* item_read, const gb_seed* seeds, const uint64_t* seed_off,
                         const DevItem* items, const uint32_t* n_items_dev, uint32_t n_items_max,
                         uint32_t* ext_count, uint8_t* status, gb_extension* ext, uint32_t* path_pool, uint32_t* mism_pool,
                         uint32_t max_read_len, const ExtendBig* big);

constexpr int SEED_WARPS = 16;          // warps per block of the seeding kernels (block-synchronised rounds)
constexpr int SEED_BLOCKS_PER_SM = 2;
constexpr int ALIGN_WARPS = 4;

struct MapBatch {
    const uint8_t* reads; const uint8_t* quals; const uint64_t* read_off; uint32_t n_reads;
    ReadState* states;
    uint32_t* work_counter;
    uint32_t Lc;
    // seeding passes: units (reads or pairs) come from in_list when set; units that overflow the
    // first pass's small shared tables (Mc, Cc) are appended to retry_list
    const uint32_t* in_list; const uint32_t* in_count;
    uint32_t* retry_list; uint32_t* retry_count;
    uint32_t Mc, Cc, Ns;
};

// ---------------------------------------------------------------------------------------
// K1
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SEED_WARPS * 32, SEED_BLOCKS_PER_SM)
seed_kernel(DevIndex ix, MapParamsDev P, MapBatch b, SeedPools pools) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ uint32_t s_base;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const SeedSmem sm = carve_seed_smem(smem + (size_t)warp * seed_smem_bytes(b.Lc, b.Mc, b.Cc), b.Lc, b.Mc, b.Cc);
    const uint32_t limit = b.in_list ? min(*b.in_count, b.n_reads) : b.n_reads;
    while (true) {
        // block-synchronised rounds, see seed_kernel_pe
        __syncthreads();
        if (threadIdx.x == 0) s_base = atomicAdd(b.work_counter, blockDim.x >> 5);
        __syncthreads();
        const uint32_t base = s_base;
        if (base >= limit) break;
        const bool active = base + warp < limit;
        const uint32_t r = !active ? 0u : (b.in_list ? b.in_list[base + warp] : base + warp);
        ReadState rs;
        memset(&rs, 0, sizeof(rs));
        uint32_t status = GB_ITEM_OK;
        uint32_t L = 0; uint64_t rb = 0;
        if (active) { rb = b.read_off[r]; L = (uint32_t)(b.read_off[r + 1] - rb); if (L > b.Lc) status = GB_ITEM_OUT_FULL; }
        const bool work = active && status == GB_ITEM_OK;
        DevRng rng; rng.inited = 0; rng.state = 0; rng.seed = 0;
        if (work) {
            for (uint32_t i = lane; i < L; i += 32) sm.read[i] = b.reads[rb + i];
            __syncwarp();
            rng.seed = fold_seed(0u, sm.read, L);                     // LazyRNG seed: the read sequence (:620-622)
            status = seed_phase_a(ix, P, sm, L, pools, rng, rs);
        }
        __syncthreads();
        if (work && status == GB_ITEM_OK) status = cluster_phase_se(ix, P, sm, L, r, pools, rng, rs);
        if (!active) continue;
        if (status == GB_ITEM_RETRY) {
            if (lane == 0) b.retry_list[atomicAdd(b.retry_count, 1u)] = r;
            continue;
        }
        rs.rng = rng;
        rs.status = status;
        if (status != GB_ITEM_OK) { rs.item_cnt = 0; }
        if (lane == 0) b.states[r] = rs;
    }
}

// ---------------------------------------------------------------------------------------
// K3
// ---------------------------------------------------------------------------------------
#include "align_read.cuh"

__global__ void __launch_bounds__(ALIGN_WARPS * 32, 4)
align_kernel(DevIndex ix, MapParamsDev P, DevScores sc, MapBatch b, AlignArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t gwarp = blockIdx.x * ALIGN_WARPS + warp;
    const uint32_t W = b.Lc + 1;
    // shared per warp: read, qual, query buffer, 4 DP columns
    const size_t per_warp = ((size_t)b.Lc * 3 + 15 & ~(size_t)15) + (size_t)W * 4 * 4 + 64 + a.tmp_bytes;
    uint8_t* base = smem + (size_t)warp * per_warp;
    uint8_t* stmp = a.tmp_bytes ? base + (((size_t)b.Lc * 3 + 15) & ~(size_t)15) + (size_t)W * 4 * 4 + 64 : nullptr;
    uint8_t* sread = base; uint8_t* squal = base + b.Lc; uint8_t* qbuf = base + 2 * (size_t)b.Lc;
    int32_t* cols = reinterpret_cast<int32_t*>(base + (((size_t)b.Lc * 3 + 15) & ~(size_t)15));
    DpSmem dps; dps.Hp = cols; dps.Ep = cols + W; dps.Hc = cols + 2 * W; dps.Ec = cols + 3 * W;
    const TailWs ws = carve_tail_ws(a.ws_base + (size_t)gwarp * a.ws_stride, b.Lc, a.tb_cells);
    uint8_t* cand_base = a.cand_base + (size_t)gwarp * a.cand_stride;

    while (true) {
        uint32_t r = 0;
        if (lane == 0) {
            r = atomicAdd(b.work_counter, 1u);
            if (a.slow_list) r = r < *a.slow_count ? a.slow_list[r] : 0xffffffffu;
        }
        r = __shfl_sync(FULL, r, 0);
        if (r >= b.n_reads) break;
        const uint64_t rb = b.read_off[r];
        const uint32_t L = (uint32_t)(b.read_off[r + 1] - rb);
        const ReadState rs = b.states[r];
        uint32_t status = rs.status;
        gb_alignment out;
        memset(&out, 0, sizeof(out));
        out.read_id = r;
        gb_mapping* out_maps = a.maps + (size_t)r * P.mapping_cap;
        uint32_t* out_edits = a.edits + (size_t)r * P.edit_cap;
        if (status == GB_ITEM_OK) {
            for (uint32_t i = lane; i < L; i += 32) { sread[i] = b.reads[rb + i]; if (b.quals) squal[i] = b.quals[rb + i]; }
            __syncwarp();
            status = align_read(ix, P, sc, rs, a, sread, b.quals ? squal : nullptr, L, r, ws, dps, qbuf, cand_base, out, out_maps, out_edits, stmp);
        }
        out.mapping_off = r * P.mapping_cap; out.edit_off = r * P.edit_cap;
        if (status != GB_ITEM_OK) { out.score = 0; out.flags = 0; out.n_mappings = 0; out.n_edits = 0; out.mapq = 0; }
        if (lane == 0) { a.aln[r] = out; a.status[r] = (uint8_t)status; }
        __syncwarp();
    }
}

#include "rescue.cuh"
#include "map_paired.cuh"
#include "align_fast.cuh"
#include "tail_plan.cuh"
#include "compact.cuh"

// AlignmentScorer::recover_log_base (alignment_scorer.cpp:30-99), gc 0.5, tol 1e-12.
static double recover_log_base(const DevScores& s) {
    auto partition = [&](double lambda) {
        double p = 0;
        for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) p += 0.25 * 0.25 * std::exp(lambda * (i == j ? (double)s.match : -(double)s.mismatch));
        return p;
    };
    double lower, upper, lambda = 1.0, part = partition(lambda);
    if (part < 1.0) { lower = lambda; while (part <= 1.0) { lower = lambda; lambda *= 2.0; part = partition(lambda); } upper = lambda; }
    else { upper = lambda; while (part >= 1.0) { upper = lambda; lambda /= 2.0; part = partition(lambda); } lower = lambda; }
    while (upper / lower - 1.0 > 1e-12) { lambda = 0.5 * (lower + upper); if (partition(lambda) < 1.0) lower = lambda; else upper = lambda; }
    return 0.5 * (lower + upper);
}

} // namespace gb

using namespace gb;

extern "C" void gb_map_params_default(gb_map_params* p) {
    memset(p, 0, sizeof(*p));
    p->hit_cap = 10; p->hard_hit_cap = 500; p->minimizer_score_fraction = 0.9; p->minimizer_coverage_flank = 250;
    p->max_unique_min = 500; p->num_bp_per_min = 1000; p->distance_limit = 200; p->min_extensions = 2; p->max_extensions = 800;
    p->cluster_score_threshold = 50; p->pad_cluster_score_threshold = 20; p->cluster_coverage_threshold = 0.3;
    p->extension_set_score_threshold = 20; p->extension_score_threshold = 1; p->min_extension_sets = 2;
    p->extension_set_min_score = 20; p->max_alignments = 8; p->max_extension_mismatches = 4; p->max_multimaps = 1;
    p->max_dozeu_cells = (uint32_t)(1.5 * 1024 * 1024); p->do_dp = 1;
    p->paired_distance_stdevs = 2.0; p->paired_rescue_score_limit = 0.9; p->rescue_subgraph_stdevs = 4.0;
    p->max_rescue_attempts = 15; p->max_fragment_length = 2000;
    p->rescue_seed_limit = 100; p->reserved0 = 0; p->rescue_likelihood_limit = 0.05;
    p->mapping_cap_per_read = 96; p->edit_cap_per_read = 160;
}

namespace gb {

// The three size classes of xdrop_tile_kernel over their work lists (lists[c * list_cap ..], counts on the device).
template <int R>
static int launch_tile_class(gb_device* d, int cls, const uint8_t* tiles, const uint32_t* tile_off, const uint32_t* lists, size_t list_cap,
                             const uint32_t* list_count, uint32_t* work, TileResult* results, uint32_t* paths, uint32_t path_cap, uint32_t* path_cursor) {
    const size_t smem = tile_smem_per_warp<R>() * TILE_WARPS;
    GB_CUDA(cudaFuncSetAttribute(xdrop_tile_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int bps = 0;
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, xdrop_tile_kernel<R>, TILE_WARPS * 32, smem));
    bps = std::max(1, std::min(bps, 2));
    const uint32_t grid = (uint32_t)(d->n_sms * bps);
    int rc;
    if ((rc = d->ws_tile.reserve(tile_ws_bytes() * (size_t)d->n_sms * 2 * TILE_WARPS))) return rc;
    TileBatch tb;
    tb.tiles = tiles; tb.tile_off = tile_off; tb.list = lists + (size_t)cls * list_cap; tb.list_count = list_count + cls; tb.list_cap = (uint32_t)list_cap;
    tb.work_counter = work + cls; tb.results = results; tb.path_pool = paths; tb.path_cap = path_cap; tb.path_cursor = path_cursor;
    tb.ws_base = d->ws_tile.ptr; tb.ws_stride = tile_ws_bytes();
    xdrop_tile_kernel<R><<<grid, TILE_WARPS * 32, smem, d->stream>>>(d->sc, tb);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    return d->kt_mark(R == 2 ? "xdrop_tile_kernel<2>" : R == 4 ? "xdrop_tile_kernel<4>" : R == 6 ? "xdrop_tile_kernel<6>" : R == 8 ? "xdrop_tile_kernel<8>" : R == 12 ? "xdrop_tile_kernel<12>" : "xdrop_tile_kernel<16>");
}
int launch_tile_kernels(gb_device* d, const uint8_t* tiles, const uint32_t* tile_off, const uint32_t* lists, size_t list_cap,
                        const uint32_t* list_count, uint32_t* work, TileResult* results, uint32_t* paths, uint32_t path_cap, uint32_t* path_cursor) {
    int rc;
    if ((rc = launch_tile_class<2>(d, 0, tiles, tile_off, lists, list_cap, list_count, work, results, paths, path_cap, path_cursor))) return rc;
    if ((rc = launch_tile_class<4>(d, 1, tiles, tile_off, lists, list_cap, list_count, work, results, paths, path_cap, path_cursor))) return rc;
    if ((rc = launch_tile_class<6>(d, 2, tiles, tile_off, lists, list_cap, list_count, work, results, paths, path_cap, path_cursor))) return rc;
    if ((rc = launch_tile_class<8>(d, 3, tiles, tile_off, lists, list_cap, list_count, work, results, paths, path_cap, path_cursor))) return rc;
    if ((rc = launch_tile_class<12>(d, 4, tiles, tile_off, lists, list_cap, list_count, work, results, paths, path_cap, path_cursor))) return rc;
    return launch_tile_class<16>(d, 5, tiles, tile_off, lists, list_cap, list_count, work, results, paths, path_cap, path_cursor);
}

// Device-resident mapping of a batch whose reads are already in HBM.
int map_device(gb_device* d, const gb_map_params* hp, uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals,
               const uint64_t* d_read_off, uint32_t max_len, uint64_t total_bases,
               gb_alignment* d_aln, uint8_t* d_status, bool paired,
               gb_mapping* out_maps, uint64_t out_map_cap, uint32_t* out_edits, uint64_t out_edit_cap,
               const uint64_t* d_run_base, uint32_t read_base, uint64_t* d_totals, uint32_t* d_overflow) {
    int rc0;
    if (hp->max_multimaps == 0 || hp->max_multimaps > GB_MAX_MULTIMAPS) { g_last_error = "max_multimaps must be 1 .. GB_MAX_MULTIMAPS"; return GB_ERR_ARG; }
    // the seeding kernels pack (node id << 10 | offset) into 32 bits (DevSeed.id_off): node ids stop at 2^22 - 1
    if (d->ix.n_nodes > (1u << 23)) { g_last_error = "the mapping kernels address node ids below 2^22 (4 194 303); split the graph (the stage seams have no such limit)"; return GB_ERR_CAPACITY; }
    const uint32_t K = hp->max_multimaps;            // records per read, rank-major: record j * n_reads + read
    if ((uint64_t)n_reads * K * std::max(hp->mapping_cap_per_read, hp->edit_cap_per_read) > 0xffffffffull) { g_last_error = "chunk too large for 32-bit record offsets (reads x max_multimaps x cap)"; return GB_ERR_ARG; }
    if ((rc0 = d->pad_maps.reserve((size_t)n_reads * K * hp->mapping_cap_per_read))) return rc0;
    if ((rc0 = d->pad_edits.reserve((size_t)n_reads * K * hp->edit_cap_per_read))) return rc0;
    gb_mapping* d_maps = d->pad_maps.ptr; uint32_t* d_edits = d->pad_edits.ptr;
    if (paired) {
        if (n_reads % 2 != 0) { g_last_error = "paired mapping needs an even number of reads"; return GB_ERR_ARG; }
        if (hp->max_rescue_attempts != 0 && hp->rescue_seed_limit >= RESCUE_SEEDS) { g_last_error = "rescue_seed_limit must be below 128"; return GB_ERR_ARG; }
        if (!(hp->fragment_stdev > 0)) { g_last_error = "paired mapping needs a forced fragment length distribution"; return GB_ERR_ARG; }
    }
    const uint32_t Lc = std::max<uint32_t>(32u, (max_len + 15u) & ~15u);
    if (Lc > 512) { g_last_error = "reads longer than 512 bp are not supported by the short-read path"; return GB_ERR_ARG; }
    int rc;
    // ---- parameter tables (host libm, so scores are bit-identical to a CPU run) ----
    if (!d->tables_ready || d->tables_hard_hit_cap != hp->hard_hit_cap) {
        std::vector<double> hit(hp->hard_hit_cap + 1, 0.0);
        const double base_score = 1.0 + std::log((double)hp->hard_hit_cap);
        for (uint32_t h = 1; h <= hp->hard_hit_cap; h++) hit[h] = base_score - std::log((double)h);
        std::vector<double> plo((32 + 1) * 256, 0.0);
        for (size_t n = 1; n <= 32; n++) for (size_t p = 0; p < 256; p++) plo[(n << 8) + p] = 1.0 - std::pow(1.0 - (2 * p + 1) / (2.0 * 256), (double)n);
        std::vector<double> pp(256);
        for (int i = 0; i < 256; i++) pp[i] = std::pow(10, -((double)i) / 10);
        if ((rc = d->t_hit.upload(hit.data(), hit.size(), d->stream))) return rc;
        if ((rc = d->t_plo.upload(plo.data(), plo.size(), d->stream))) return rc;
        if ((rc = d->t_phred.upload(pp.data(), pp.size(), d->stream))) return rc;
        GB_CUDA(cudaStreamSynchronize(d->stream));
        d->tables_ready = true; d->tables_hard_hit_cap = hp->hard_hit_cap;
    }
    MapParamsDev P;
    P.hit_cap = hp->hit_cap; P.hard_hit_cap = hp->hard_hit_cap; P.minimizer_score_fraction = hp->minimizer_score_fraction;
    P.minimizer_coverage_flank = hp->minimizer_coverage_flank; P.max_unique_min = hp->max_unique_min; P.num_bp_per_min = hp->num_bp_per_min;
    P.distance_limit = hp->distance_limit; P.min_extensions = hp->min_extensions; P.max_extensions = hp->max_extensions;
    P.cluster_score_threshold = hp->cluster_score_threshold; P.pad_cluster_score_threshold = hp->pad_cluster_score_threshold;
    P.cluster_coverage_threshold = hp->cluster_coverage_threshold; P.extension_set_score_threshold = hp->extension_set_score_threshold;
    P.extension_score_threshold = hp->extension_score_threshold; P.min_extension_sets = hp->min_extension_sets;
    P.extension_set_min_score = hp->extension_set_min_score; P.max_alignments = hp->max_alignments;
    P.max_extension_mismatches = hp->max_extension_mismatches; P.max_dozeu_cells = hp->max_dozeu_cells; P.do_dp = hp->do_dp;
    P.mapping_cap = hp->mapping_cap_per_read; P.edit_cap = hp->edit_cap_per_read;
    P.max_multimaps = K; P.out_stride = n_reads;
    P.log_base = recover_log_base(d->sc);
    P.max_rescue_attempts = paired ? hp->max_rescue_attempts : 0; P.rescue_seed_limit = hp->rescue_seed_limit;
    P.paired_rescue_score_limit = hp->paired_rescue_score_limit; P.rescue_subgraph_stdevs = hp->rescue_subgraph_stdevs;
    P.rescue_likelihood_limit = hp->rescue_likelihood_limit;
    P.hit_score_table = d->t_hit.ptr; P.prob_at_least_one = d->t_plo.ptr; P.phred_prob = d->t_phred.ptr;

    // ---- pools ----
    // Sized from per-read averages (48 minimizers, 64 seeds, 3 kept clusters) times d->pool_scale.  A chunk that needs
    // more sets the sticky overflow word (cursor 13); the host-buffer entry points then double the scale and rerun the
    // chunk (map_batch_host), gb_map_batch_device reports it through gb_device_pool_overflow.  Capacities stay below
    // 2^32 records (the cursors are 32-bit; pool_claim never lets one wrap).
    const double ps = d->pool_scale;
    const size_t min_cap = std::min<size_t>((size_t)((double)n_reads * 48 * ps) + 1024, 0xfffffff0u), seed_cap = std::min<size_t>((size_t)((double)n_reads * 64 * ps) + 4096, 0xfffffff0u);
    const size_t item_cap = std::min<size_t>((size_t)((double)n_reads * 3 * ps) + 1024, 0x7ffffff0u / 48), ext_cap = seed_cap;
    if ((rc = d->p_states.reserve(n_reads))) return rc;
    if ((rc = d->p_min.reserve(min_cap))) return rc;
    if ((rc = d->p_seeds.reserve(seed_cap))) return rc;
    if ((rc = d->p_items.reserve(item_cap))) return rc;
    if ((rc = d->p_ext_seeds.reserve(ext_cap))) return rc;
    if ((rc = d->p_cursors.reserve(48))) return rc;
    GB_CUDA(cudaMemsetAsync(d->p_cursors.ptr, 0, 48 * sizeof(uint32_t), d->stream));
    // 0 seed work, 1 min, 2 seed, 3 item, 4 ext, 5 extend work, 6 align work, 7 slow count, 8-10 seeding retry, 11-12 rescue, 13 pool overflow,
    // 14 plan work, 15 big extension items, 16 tiles, 17 tile bytes / 16, 18-29 tile list counts (2 waves x 6 classes),
    // 30 result path words, 31 decide work, 32-43 tile work
    uint32_t* cur = d->p_cursors.ptr;
    d->kt_reset();
    if (K > 1) {
        init_absent_kernel<<<d->n_sms * 4, 256, 0, d->stream>>>(d_aln, n_reads, n_reads * K, hp->mapping_cap_per_read, hp->edit_cap_per_read);
        d->launches++;
        GB_CUDA(cudaGetLastError());
    }

    int32_t fragment_limit = 0;
    if (paired) {
        // rightward working copy of the reads (mate 2 reverse-complemented), :1503-1506
        int rcw;
        if ((rcw = d->w_reads.reserve(total_bases ? total_bases : 1))) return rcw;
        if (d_quals) { if ((rcw = d->w_quals.reserve(total_bases ? total_bases : 1))) return rcw; }
        prep_pairs_kernel<<<d->n_sms * 8, 256, 0, d->stream>>>(d_reads, d_quals, d_read_off, n_reads, d->w_reads.ptr, d_quals ? d->w_quals.ptr : nullptr);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        d_reads = d->w_reads.ptr; if (d_quals) d_quals = d->w_quals.ptr;
        fragment_limit = (int32_t)(int64_t)(hp->fragment_mean + hp->paired_distance_stdevs * hp->fragment_stdev);   // :1470
        const uint32_t read_limit = std::max<uint32_t>(hp->distance_limit, max_len + 50);
        if (fragment_limit < (int32_t)read_limit) { g_last_error = "fragment distance limit smaller than the read distance limit (the reference falls back to single-end, :1471)"; return GB_ERR_ARG; }
        if ((rcw = d->p_pairs.reserve(n_reads / 2))) return rcw;
    }
    MapBatch b; b.reads = d_reads; b.quals = d_quals; b.read_off = d_read_off; b.n_reads = n_reads;
    b.states = d->p_states.ptr; b.work_counter = cur + 0; b.Lc = Lc;
    b.in_list = nullptr; b.in_count = nullptr; b.retry_list = nullptr; b.retry_count = nullptr; b.Mc = MAX_MINIMIZERS; b.Cc = MAX_CLUSTERS; b.Ns = d->seed_ns;
    SeedPools pools;
    pools.dbg_clusters = d->dbg_clusters; pools.overflow = cur + 13;
    pools.minimizers = d->p_min.ptr; pools.min_cap = (uint32_t)min_cap; pools.min_cursor = cur + 1;
    pools.seeds = d->p_seeds.ptr; pools.seed_cap = (uint32_t)seed_cap; pools.seed_cursor = cur + 2;
    pools.items = d->p_items.ptr; pools.item_cap = (uint32_t)item_cap; pools.item_cursor = cur + 3;
    pools.ext_seeds = d->p_ext_seeds.ptr; pools.ext_cap = (uint32_t)ext_cap; pools.ext_cursor = cur + 4;

    GB_CUDA(cudaEventRecord(d->ev_stage[0], d->stream));
    if ((rc = d->kt_mark("start"))) return rc;
    // ---- K1: a first pass with small shared tables (8 blocks per SM), then the units that did not
    // fit (many minimizers or clusters) once more at the maximum table sizes ----
    {
        const uint32_t n_units = paired ? n_reads / 2 : n_reads;
        if ((rc = d->p_retry.reserve(n_units + 1))) return rc;
        for (int pass = 0; pass < 2; pass++) {
            MapBatch bp = b;
            bp.Mc = pass == 0 ? d->seed_mc : MAX_MINIMIZERS; bp.Cc = pass == 0 ? d->seed_cc : MAX_CLUSTERS;
            bp.work_counter = pass == 0 ? cur + 0 : cur + 9;
            bp.in_list = pass == 0 ? nullptr : d->p_retry.ptr; bp.in_count = pass == 0 ? nullptr : cur + 8;
            bp.retry_list = d->p_retry.ptr; bp.retry_count = pass == 0 ? cur + 8 : cur + 10;
            // the cluster phases carve their scratch from the arrays that are dead after phase A
            while (seed_dead_bytes(Lc, bp.Mc) < cluster_scratch_bytes(bp.Cc) && bp.Mc < MAX_MINIMIZERS) bp.Mc += 8;
            uint32_t warps = SEED_WARPS;
            while (warps > 1 && seed_smem_bytes(Lc, bp.Mc, bp.Cc) * warps > 200 * 1024) warps >>= 1;
            const size_t smem = seed_smem_bytes(Lc, bp.Mc, bp.Cc) * warps;
            const bool fixed_layout = paired && Lc == 160 && bp.Mc == 64 && bp.Cc == 16;
            if (smem > 48 * 1024) {
                GB_CUDA(cudaFuncSetAttribute(seed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                GB_CUDA(cudaFuncSetAttribute(seed_kernel_pe<0, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                GB_CUDA(cudaFuncSetAttribute(seed_kernel_pe<160, 64, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            }
            int bps = 0;
            if (paired && fixed_layout) GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, seed_kernel_pe<160, 64, 16>, warps * 32, smem));
            else if (paired) GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, seed_kernel_pe<0, 0, 0>, warps * 32, smem));
            else GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, seed_kernel, warps * 32, smem));
            if (bps < 1) bps = 1;
            uint32_t grid = std::min<uint32_t>((uint32_t)(d->n_sms * bps), (n_units + warps - 1) / warps);
            if (grid == 0) grid = 1;
            if (paired) { PairBatch pbatch; pbatch.pairs = d->p_pairs.ptr; pbatch.fragment_limit = fragment_limit;
                          if (fixed_layout) seed_kernel_pe<160, 64, 16><<<grid, warps * 32, smem, d->stream>>>(d->ix, P, bp, pools, pbatch);
                          else seed_kernel_pe<0, 0, 0><<<grid, warps * 32, smem, d->stream>>>(d->ix, P, bp, pools, pbatch); }
            else seed_kernel<<<grid, warps * 32, smem, d->stream>>>(d->ix, P, bp, pools);
            d->launches++;
            GB_CUDA(cudaGetLastError());
            if ((rc = d->kt_mark(pass == 0 ? (paired ? "seed_kernel_pe" : "seed_kernel") : "seed_kernel(retry tables)"))) return rc;
        }
    }
    GB_CUDA(cudaEventRecord(d->ev_stage[1], d->stream));
    if (d->debug_stop_after_seed) return GB_OK;              // gb_debug_seed_stage reads the pools as the seeding kernels left them
    // ---- K2: extension over the items produced on the device ----
    const uint32_t max_ext = 48, path_cap = 384, mism_cap = 192;
    if ((rc = d->p_ext_count.reserve(item_cap))) return rc;
    if ((rc = d->p_ext_status.reserve(item_cap))) return rc;
    if ((rc = d->p_ext.reserve(item_cap * max_ext))) return rc;
    if ((rc = d->p_path.reserve(item_cap * path_cap))) return rc;
    if ((rc = d->p_mism.reserve(item_cap * mism_cap))) return rc;
    // clusters whose seeds yield more extensions than those strides hold (repeats: a hundred seeds in one cluster, one
    // extension per seed before GaplessExtender::extend removes duplicates) are redone with large strides
    ExtendBig big;
    big.cap = n_reads / 128 + 256; big.max_ext = 512; big.path_cap = 512 * 24; big.mism_cap = 512 * 4;
    if ((rc = d->p_big_list.reserve(big.cap)) || (rc = d->p_big_of.reserve(item_cap)) || (rc = d->p_big_ext.reserve((size_t)big.cap * big.max_ext)) ||
        (rc = d->p_big_path.reserve((size_t)big.cap * big.path_cap)) || (rc = d->p_big_mism.reserve((size_t)big.cap * big.mism_cap))) return rc;
    GB_CUDA(cudaMemsetAsync(d->p_big_of.ptr, 0xff, sizeof(uint32_t) * item_cap, d->stream));
    big.list = d->p_big_list.ptr; big.count = cur + 15; big.big_of = d->p_big_of.ptr;
    big.ext = d->p_big_ext.ptr; big.path = d->p_big_path.ptr; big.mism = d->p_big_mism.ptr;
    {
        ExtendParams ep;
        ep.sc = d->sc; ep.max_mismatches = hp->max_extension_mismatches; ep.overlap_threshold = 0.8; ep.overlap_threshold_unused = 0.f;
        ep.trim = 1; ep.max_ext = max_ext; ep.path_cap = path_cap; ep.mism_cap = mism_cap;
        if ((rc = launch_extend_device(d, ep, d_reads, d_read_off, nullptr, d->p_ext_seeds.ptr, nullptr, d->p_items.ptr, cur + 3,
                                       (uint32_t)item_cap, d->p_ext_count.ptr, d->p_ext_status.ptr, d->p_ext.ptr, d->p_path.ptr,
                                       d->p_mism.ptr, Lc, &big))) return rc;
    }
    GB_CUDA(cudaEventRecord(d->ev_stage[2], d->stream));
    // ---- K3 ----
    {
        const uint32_t W = Lc + 1;
        // the five temporary path buffers of a warp go to shared memory when they fit beside the DP columns
        const size_t slot_bytes = (size_t)hp->mapping_cap_per_read * sizeof(gb_mapping) + (size_t)hp->edit_cap_per_read * 4;
        const uint32_t tmp_bytes = N_TEMP_SLOTS * slot_bytes <= 12 * 1024 ? (uint32_t)(N_TEMP_SLOTS * slot_bytes) : 0u;
        const size_t per_warp = (((size_t)Lc * (paired ? 5 : 3) + 15) & ~(size_t)15) + (size_t)W * 4 * 4 + 64 + tmp_bytes;
        const size_t smem = per_warp * ALIGN_WARPS;
        if (smem > 48 * 1024) {
            GB_CUDA(cudaFuncSetAttribute(align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            GB_CUDA(cudaFuncSetAttribute(align_kernel_pe<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            GB_CUDA(cudaFuncSetAttribute(align_kernel_pe<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        }
        int bps = 0;
        const bool rescue = paired && hp->max_rescue_attempts != 0;
        int bps_rescue = 0;
        if (rescue) GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps_rescue, align_kernel_pe<true>, ALIGN_WARPS * 32, smem));
        if (paired) GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, align_kernel_pe<false>, ALIGN_WARPS * 32, smem));
        else GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, align_kernel, ALIGN_WARPS * 32, smem));
        if (bps < 1) bps = 1;
        if (bps > 4) bps = 4;          // bounds the per-warp tail workspaces (about 2 MB each)
        uint32_t grid_plain = std::min<uint32_t>((uint32_t)(d->n_sms * bps), (n_reads + ALIGN_WARPS - 1) / ALIGN_WARPS);
        if (grid_plain == 0) grid_plain = 1;
        bps_rescue = std::max(1, std::min(bps_rescue, 2));     // + the rescue workspaces (about 2 MB each)
        uint32_t grid = rescue ? std::min<uint32_t>((uint32_t)(d->n_sms * bps_rescue), grid_plain) : grid_plain;
        const size_t n_warps = (size_t)grid_plain * ALIGN_WARPS;
        const uint32_t tb_cells = hp->max_dozeu_cells + hp->max_dozeu_cells / 4 + 4096;
        const size_t ws_stride = tail_ws_bytes(Lc, tb_cells);
        const size_t cand_stride = (((size_t)hp->mapping_cap_per_read * sizeof(gb_mapping) + (size_t)hp->edit_cap_per_read * 4) * (N_SLOTS + N_TEMP_SLOTS) + 255) & ~(size_t)255;
        if ((rc = d->ws_tail.reserve(ws_stride * n_warps))) return rc;
        if ((rc = d->ws_cand.reserve(cand_stride * n_warps))) return rc;
        AlignArgs a;
        a.plan.entries = nullptr; a.plan.unit_base = nullptr; a.plan.unit_count = nullptr; a.plan.tile_off = nullptr; a.plan.results = nullptr; a.plan.path_pool = nullptr; a.plan.stats = nullptr;
        a.rescue_base = nullptr; a.rescue_stride = 0; a.tmp_bytes = tmp_bytes;
        if (rescue) {
            a.rescue_stride = (rescue_ws_bytes(Lc) + 255) & ~(size_t)255;
            if ((rc = d->ws_rescue.reserve(a.rescue_stride * (size_t)grid * ALIGN_WARPS))) return rc;
            if ((rc = d->p_rescue.reserve(n_reads / 2 + 1))) return rc;
            a.rescue_base = d->ws_rescue.ptr;
        }
        a.items = d->p_items.ptr; a.minimizers = d->p_min.ptr;
        a.ev.ext_count = d->p_ext_count.ptr; a.ev.ext_status = d->p_ext_status.ptr; a.ev.ext = d->p_ext.ptr;
        a.ev.path_pool = d->p_path.ptr; a.ev.mism_pool = d->p_mism.ptr; a.ev.max_ext = max_ext; a.ev.path_cap = path_cap; a.ev.mism_cap = mism_cap;
        a.ev.big_of = d->p_big_of.ptr; a.ev.big_ext = d->p_big_ext.ptr; a.ev.big_path = d->p_big_path.ptr; a.ev.big_mism = d->p_big_mism.ptr;
        a.ev.big_max_ext = big.max_ext; a.ev.big_path_cap = big.path_cap; a.ev.big_mism_cap = big.mism_cap;
        a.ws_base = d->ws_tail.ptr; a.ws_stride = ws_stride; a.cand_base = d->ws_cand.ptr; a.cand_stride = cand_stride;
        a.aln = d_aln; a.maps = d_maps; a.edits = d_edits; a.status = d_status; a.tb_cells = tb_cells;
        a.pairs = paired ? d->p_pairs.ptr : nullptr; a.frag_mean = hp->fragment_mean; a.frag_sd = hp->fragment_stdev;
        MapBatch b3 = b; b3.work_counter = cur + 6;
        // thread-per-unit fast path first; whatever it cannot finish goes to the warp-per-unit kernel
        const uint32_t n_units = paired ? n_reads / 2 : n_reads;
        if ((rc = d->p_slow.reserve(n_units + 1))) return rc;
        FastArgs fa; fa.slow_list = d->p_slow.ptr; fa.slow_count = cur + 7;
        const uint32_t fgrid = std::max<uint32_t>(1u, std::min<uint32_t>((n_units + 127) / 128, (uint32_t)d->n_sms * 16));
        a.slow_list = nullptr; a.slow_count = nullptr;
        if (paired) {
            if (d->fast_minb == 12) align_fast_kernel_pe<12><<<fgrid, 128, 0, d->stream>>>(d->ix, P, d->sc, b3, a, fa);
            else if (d->fast_minb == 16) align_fast_kernel_pe<16><<<fgrid, 128, 0, d->stream>>>(d->ix, P, d->sc, b3, a, fa);
            else align_fast_kernel_pe<0><<<fgrid, 128, 0, d->stream>>>(d->ix, P, d->sc, b3, a, fa);
        }
        else align_fast_kernel<<<fgrid, 128, 0, d->stream>>>(d->ix, P, d->sc, b3, a, fa);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        if ((rc = d->kt_mark(paired ? "align_fast_kernel_pe" : "align_fast_kernel"))) return rc;
        a.slow_list = d->p_slow.ptr; a.slow_count = cur + 7;
        // ---- tails of the slow units: plan (forests -> tiles), then the DP of every tile in its own compact kernel ----
        if (hp->do_dp && d->use_tiles) {
            const size_t tile_cap = (size_t)n_reads * 4 + 4096;
            const size_t unit_cap = std::min<size_t>((size_t)n_reads * 128 + (1u << 20), 0xfffffff0u);
            const size_t path_cap = std::min<size_t>(tile_cap * 32, 0xfffffff0u);
            if ((rc = d->pl_entries.reserve((size_t)n_units * PLAN_PER_UNIT)) || (rc = d->pl_unit_base.reserve(n_units)) || (rc = d->pl_unit_count.reserve(n_units)) ||
                (rc = d->pl_tiles.reserve(unit_cap * 16)) || (rc = d->pl_tile_off.reserve(tile_cap)) || (rc = d->pl_results.reserve(tile_cap)) ||
                (rc = d->pl_lists.reserve(2 * TILE_CLASSES * tile_cap)) || (rc = d->pl_paths.reserve(path_cap)) || (rc = d->pl_stats.reserve(4))) return rc;
            GB_CUDA(cudaMemsetAsync(d->pl_stats.ptr, 0, 4 * sizeof(uint64_t), d->stream));
            PlanPools pp;
            pp.entries = d->pl_entries.ptr; pp.unit_base = d->pl_unit_base.ptr; pp.unit_count = d->pl_unit_count.ptr;
            pp.tiles = d->pl_tiles.ptr; pp.tile_units_cap = (uint32_t)unit_cap; pp.tile_units_cursor = cur + 17;
            pp.tile_off = d->pl_tile_off.ptr; pp.tile_cap = (uint32_t)tile_cap; pp.tile_cursor = cur + 16;
            pp.results = d->pl_results.ptr;
            for (int c = 0; c < 2 * TILE_CLASSES; c++) pp.lists[c] = d->pl_lists.ptr + (size_t)c * tile_cap;
            pp.list_count = cur + 18; pp.stats = d->pl_stats.ptr;
            MapBatch bpl = b3; bpl.work_counter = cur + 14;
            if (paired) tail_plan_kernel<true><<<grid_plain, ALIGN_WARPS * 32, 0, d->stream>>>(d->ix, P, d->sc, bpl, a, pp);
            else tail_plan_kernel<false><<<grid_plain, ALIGN_WARPS * 32, 0, d->stream>>>(d->ix, P, d->sc, bpl, a, pp);
            d->launches++;
            GB_CUDA(cudaGetLastError());
            if ((rc = d->kt_mark("tail_plan_kernel"))) return rc;
            // wave 0: the tails that are always aligned; the decide pass cancels what the reference would skip; wave 1: the rest
            if ((rc = launch_tile_kernels(d, d->pl_tiles.ptr, d->pl_tile_off.ptr, d->pl_lists.ptr, tile_cap, cur + 18, cur + 32, d->pl_results.ptr,
                                          d->pl_paths.ptr, (uint32_t)path_cap, cur + 30))) return rc;
            MapBatch bdc = b3; bdc.work_counter = cur + 31;
            if (paired) tail_decide_kernel<true><<<grid_plain, ALIGN_WARPS * 32, 0, d->stream>>>(d->ix, P, d->sc, bdc, a, pp);
            else tail_decide_kernel<false><<<grid_plain, ALIGN_WARPS * 32, 0, d->stream>>>(d->ix, P, d->sc, bdc, a, pp);
            d->launches++;
            GB_CUDA(cudaGetLastError());
            if ((rc = d->kt_mark("tail_decide_kernel"))) return rc;
            if ((rc = launch_tile_kernels(d, d->pl_tiles.ptr, d->pl_tile_off.ptr, d->pl_lists.ptr + (size_t)TILE_CLASSES * tile_cap, tile_cap, cur + 18 + TILE_CLASSES,
                                          cur + 32 + TILE_CLASSES, d->pl_results.ptr, d->pl_paths.ptr, (uint32_t)path_cap, cur + 30))) return rc;
            a.plan.entries = d->pl_entries.ptr; a.plan.unit_base = d->pl_unit_base.ptr; a.plan.unit_count = d->pl_unit_count.ptr;
            a.plan.tile_off = d->pl_tile_off.ptr; a.plan.results = d->pl_results.ptr; a.plan.path_pool = d->pl_paths.ptr; a.plan.stats = d->pl_stats.ptr;
        }
        if (paired) {
            // the plain kernel takes every listed pair; with rescue enabled it defers the pairs that turn out to have
            // unpaired alignments to a second list, which the (larger, lower-occupancy) rescue instantiation redoes
            a.rescue_list = d->p_rescue.ptr; a.rescue_count = cur + 11;
            align_kernel_pe<false><<<grid_plain, ALIGN_WARPS * 32, smem, d->stream>>>(d->ix, P, d->sc, b3, a);
            if (rescue) {
                d->launches++;
                GB_CUDA(cudaGetLastError());
                if ((rc = d->kt_mark("align_kernel_pe"))) return rc;
                b3.work_counter = cur + 12;
                a.slow_list = d->p_rescue.ptr; a.slow_count = cur + 11;
                align_kernel_pe<true><<<grid, ALIGN_WARPS * 32, smem, d->stream>>>(d->ix, P, d->sc, b3, a);
            }
        }
        else align_kernel<<<grid, ALIGN_WARPS * 32, smem, d->stream>>>(d->ix, P, d->sc, b3, a);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        if ((rc = d->kt_mark(!paired ? "align_kernel" : (rescue ? "align_kernel_pe<rescue>" : "align_kernel_pe")))) return rc;
    }
    GB_CUDA(cudaEventRecord(d->ev_stage[3], d->stream));
    if ((rc = compact_outputs(d, n_reads * K, n_reads, d_aln, d_maps, d_edits, hp->mapping_cap_per_read, hp->edit_cap_per_read,
                              out_maps, out_map_cap, out_edits, out_edit_cap, d_run_base, read_base, d_totals, d_status))) return rc;
    if ((rc = d->kt_mark("compact (2 scans + gather)"))) return rc;
    if (d_overflow) GB_CUDA(cudaMemcpyAsync(d_overflow, cur + 13, sizeof(uint32_t), cudaMemcpyDeviceToDevice, d->stream));
    GB_CUDA(cudaEventRecord(d->ev_stage[4], d->stream));
    return GB_OK;
}

} // namespace gb

// Host-buffer entry: chunks of <= map_chunk reads are copied in, mapped, compacted and copied out,
// double-buffered over three streams: while chunk i computes, chunk i+1 uploads and chunk i-1
// downloads.  Output offsets are global (running totals kept on the device).
static int map_batch_host(gb_device* d, const gb_map_params* hp, bool paired,
                          uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                          gb_alignment* aln, gb_mapping* mappings, uint64_t mapping_pool_cap, uint32_t* edits, uint64_t edit_pool_cap,
                          uint8_t* status, uint64_t* n_mappings_used, uint64_t* n_edits_used) {
    if (!d || !hp || !reads || !read_off || !aln || !mappings || !edits || !status) return GB_ERR_ARG;
    if (n_mappings_used) *n_mappings_used = 0;
    if (n_edits_used) *n_edits_used = 0;
    if (n_reads == 0) return GB_OK;
    if (hp->max_multimaps == 0 || hp->max_multimaps > GB_MAX_MULTIMAPS) { g_last_error = "max_multimaps must be 1 .. GB_MAX_MULTIMAPS"; return GB_ERR_ARG; }
    const uint32_t K = hp->max_multimaps;
    if (paired && n_reads % 2 == 0) {
        // A distribution the clusterer cannot use (fragment limit below the read limit): the reference maps both
        // ends single-ended and emits them as a pair (minimizer_mapper.cpp:1469-1496).  The test is per pair
        // (get_distance_limit of read 1); a batch where only some pairs fail it is refused.
        const int64_t fragment_limit = (int64_t)(hp->fragment_mean + hp->paired_distance_stdevs * hp->fragment_stdev);
        uint32_t fallback = 0;
        for (uint32_t p = 0; p < n_reads / 2; p++) {
            const int64_t L1 = (int64_t)(read_off[2 * (size_t)p + 1] - read_off[2 * (size_t)p]);
            fallback += fragment_limit < std::max<int64_t>(hp->distance_limit, L1 + 50);
        }
        if (fallback == n_reads / 2) {
            const int rcs = map_batch_host(d, hp, false, n_reads, reads, quals, read_off, aln, mappings, mapping_pool_cap, edits, edit_pool_cap,
                                           status, n_mappings_used, n_edits_used);
            if (rcs == GB_OK) for (size_t r = 0; r < (size_t)n_reads * K; r++) if (!(aln[r].flags & GB_ALN_ABSENT)) aln[r].flags |= GB_ALN_PAIRED;
            return rcs;
        }
        if (fallback != 0) { g_last_error = "fragment distance limit below the read distance limit for some pairs only (mixed single-end fallback, minimizer_mapper.cpp:1471, is not supported in one batch)"; return GB_ERR_ARG; }
    }
    GB_CUDA(cudaSetDevice(d->device));
    const uint32_t chunk = d->map_chunk;
    uint64_t map_used = 0, edit_used = 0;
    float kernel_ms = 0.f;
    int rc;
    if ((rc = d->c_run.reserve(2))) return rc;
    GB_CUDA(cudaMemsetAsync(d->c_run.ptr, 0, 2 * sizeof(uint64_t), d->stream));
    const uint32_t n_chunks = (n_reads + chunk - 1) / chunk;
    bool used[2] = {false, false};
    constexpr int RERUN = 1000;                   // internal: the chunk overflowed the intermediate pools

    // download the dense mappings / edits of a chunk whose header copy has been queued
    auto finish = [&](uint32_t ci) -> int {
        gb_device::IoSet& io = d->io[ci & 1];
        GB_CUDA(cudaEventSynchronize(io.ev_hdr));
        const uint64_t tm = d->h_totals[3 * (ci & 1)], te = d->h_totals[3 * (ci & 1) + 1];
        if (d->h_totals[3 * (ci & 1) + 2] != 0) return RERUN;
        if (map_used + tm > mapping_pool_cap || edit_used + te > edit_pool_cap) {
            g_last_error = "output pool capacity too small";
            return GB_ERR_CAPACITY;
        }
        if (tm) GB_CUDA(cudaMemcpyAsync(mappings + map_used, io.maps.ptr, sizeof(gb_mapping) * tm, cudaMemcpyDeviceToHost, d->s_out));
        if (te) GB_CUDA(cudaMemcpyAsync(edits + edit_used, io.edits.ptr, 4 * te, cudaMemcpyDeviceToHost, d->s_out));
        if (d->mirror_aln) {
            // the same records stay in HBM for the caller's emission gather (gb_device_set_output_mirror)
            if (map_used + tm > d->mirror_map_cap || edit_used + te > d->mirror_edit_cap) { g_last_error = "output mirror too small"; return GB_ERR_CAPACITY; }
            if (tm) GB_CUDA(cudaMemcpyAsync(d->mirror_maps + map_used, io.maps.ptr, sizeof(gb_mapping) * tm, cudaMemcpyDeviceToDevice, d->s_out));
            if (te) GB_CUDA(cudaMemcpyAsync(d->mirror_edits + edit_used, io.edits.ptr, 4 * te, cudaMemcpyDeviceToDevice, d->s_out));
        }
        GB_CUDA(cudaEventRecord(io.ev_out, d->s_out));
        float ms = 0.f;
        GB_CUDA(cudaEventElapsedTime(&ms, io.ev_k0, io.ev_k1));
        kernel_ms += ms;
        map_used += tm; edit_used += te;
        return GB_OK;
    };
    auto drain = [&]() { cudaStreamSynchronize(d->s_in); cudaStreamSynchronize(d->stream); cudaStreamSynchronize(d->s_out); };

    auto launch = [&](uint32_t ci) -> int {
        const uint32_t c0 = ci * chunk;
        const uint32_t cn = std::min<uint32_t>(chunk, n_reads - c0);
        gb_device::IoSet& io = d->io[ci & 1];
        const uint64_t b0 = read_off[c0], b1 = read_off[c0 + cn], total = b1 - b0;
        uint32_t max_len = 0;
        for (uint32_t r = 0; r < cn; r++) max_len = std::max<uint32_t>(max_len, (uint32_t)(read_off[c0 + r + 1] - read_off[c0 + r]));
        const uint64_t chunk_map_cap = (uint64_t)cn * K * hp->mapping_cap_per_read, chunk_edit_cap = (uint64_t)cn * K * hp->edit_cap_per_read;
        if (used[ci & 1]) {
            // this set's inputs were read by chunk ci-2's kernels; its outputs must have left the device
            GB_CUDA(cudaStreamWaitEvent(d->s_in, io.ev_done, 0));
            GB_CUDA(cudaStreamWaitEvent(d->stream, io.ev_out, 0));
        }
        if ((rc = io.reads.reserve(total ? total : 1)) || (quals && (rc = io.quals.reserve(total ? total : 1))) || (rc = io.read_off.reserve(cn + 1)) ||
            (rc = io.aln.reserve((size_t)cn * K)) || (rc = io.status.reserve(cn)) || (rc = io.totals.reserve(3)) ||
            (rc = io.maps.reserve(chunk_map_cap)) || (rc = io.edits.reserve(chunk_edit_cap))) return rc;
        if (total) GB_CUDA(cudaMemcpyAsync(io.reads.ptr, reads + b0, total, cudaMemcpyHostToDevice, d->s_in));
        if (quals && total) GB_CUDA(cudaMemcpyAsync(io.quals.ptr, quals + b0, total, cudaMemcpyHostToDevice, d->s_in));
        GB_CUDA(cudaMemcpyAsync(io.read_off.ptr, read_off + c0, sizeof(uint64_t) * (cn + 1), cudaMemcpyHostToDevice, d->s_in));
        GB_CUDA(cudaEventRecord(io.ev_in, d->s_in));
        GB_CUDA(cudaStreamWaitEvent(d->stream, io.ev_in, 0));
        if (b0) gb::rebase_offsets_kernel<<<(cn + 256) / 256, 256, 0, d->stream>>>(io.read_off.ptr, cn + 1, b0);
        GB_CUDA(cudaEventRecord(io.ev_k0, d->stream));
        GB_CUDA(cudaMemsetAsync(io.totals.ptr + 2, 0, sizeof(uint64_t), d->stream));
        if ((rc = gb::map_device(d, hp, cn, io.reads.ptr, quals ? io.quals.ptr : nullptr, io.read_off.ptr, max_len, total,
                                 io.aln.ptr, io.status.ptr, paired, io.maps.ptr, chunk_map_cap, io.edits.ptr, chunk_edit_cap,
                                 d->c_run.ptr, c0, io.totals.ptr, reinterpret_cast<uint32_t*>(io.totals.ptr + 2)))) return rc;
        gb::advance_run_kernel<<<1, 1, 0, d->stream>>>(d->c_run.ptr, io.totals.ptr);
        GB_CUDA(cudaEventRecord(io.ev_k1, d->stream));
        GB_CUDA(cudaEventRecord(io.ev_done, d->stream));
        used[ci & 1] = true;
        // headers + totals of this chunk leave as soon as it is done
        GB_CUDA(cudaStreamWaitEvent(d->s_out, io.ev_done, 0));
        GB_CUDA(cudaMemcpyAsync(d->h_totals + 3 * (ci & 1), io.totals.ptr, 3 * sizeof(uint64_t), cudaMemcpyDeviceToHost, d->s_out));
        // rank j of the chunk's reads goes to rank j of the batch (record j * n_reads + read)
        for (uint32_t j = 0; j < K; j++) {
            GB_CUDA(cudaMemcpyAsync(aln + (size_t)j * n_reads + c0, io.aln.ptr + (size_t)j * cn, sizeof(gb_alignment) * cn, cudaMemcpyDeviceToHost, d->s_out));
            if (d->mirror_aln) GB_CUDA(cudaMemcpyAsync(d->mirror_aln + (size_t)j * n_reads + c0, io.aln.ptr + (size_t)j * cn, sizeof(gb_alignment) * cn, cudaMemcpyDeviceToDevice, d->s_out));
        }
        GB_CUDA(cudaMemcpyAsync(status + c0, io.status.ptr, cn, cudaMemcpyDeviceToHost, d->s_out));
        GB_CUDA(cudaEventRecord(io.ev_hdr, d->s_out));
        return GB_OK;
    };

    // chunk ci computes while chunk ci-1's dense pools are sized and fetched; a chunk that ran out of intermediate pool
    // space is redone (it and everything queued behind it) with the pools doubled, so capacity never shows in a result
    uint32_t next = 0, finished = 0;
    while (finished < n_chunks) {
        if (next < n_chunks) { if ((rc = launch(next))) { drain(); return rc; } next++; }
        if (next - finished == 2 || next == n_chunks) {
            rc = finish(finished);
            if (rc == RERUN) {
                drain();
                if (d->pool_scale >= 1024.0) { g_last_error = "intermediate pools overflow even at 1024x the per-read averages; use a smaller GIRAFFE_B200_MAP_CHUNK"; return GB_ERR_CAPACITY; }
                d->pool_scale *= 2.0; d->pool_reruns++;
                const uint64_t run[2] = {map_used, edit_used};
                GB_CUDA(cudaMemcpy(d->c_run.ptr, run, sizeof run, cudaMemcpyHostToDevice));
                used[0] = used[1] = false;
                next = finished;
                continue;
            }
            if (rc) { drain(); return rc; }
            finished++;
        }
    }
    GB_CUDA(cudaStreamSynchronize(d->s_out));
    GB_CUDA(cudaStreamSynchronize(d->stream));
    d->last_kernel_ms = kernel_ms;
    if (n_mappings_used) *n_mappings_used = map_used;
    if (n_edits_used) *n_edits_used = edit_used;
    return GB_OK;
}

extern "C" int gb_map_batch(gb_device* d, const gb_map_params* hp,
                            uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                            gb_alignment* aln, gb_mapping* mappings, uint64_t mapping_pool_cap, uint32_t* edits, uint64_t edit_pool_cap,
                            uint8_t* status, uint64_t* n_mappings_used, uint64_t* n_edits_used) {
    return map_batch_host(d, hp, false, n_reads, reads, quals, read_off, aln, mappings, mapping_pool_cap, edits, edit_pool_cap, status, n_mappings_used, n_edits_used);
}

extern "C" int gb_map_paired_batch(gb_device* d, const gb_map_params* hp,
                                   uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                                   gb_alignment* aln, gb_mapping* mappings, uint64_t mapping_pool_cap, uint32_t* edits, uint64_t edit_pool_cap,
                                   uint8_t* status, uint64_t* n_mappings_used, uint64_t* n_edits_used) {
    return map_batch_host(d, hp, true, n_reads, reads, quals, read_off, aln, mappings, mapping_pool_cap, edits, edit_pool_cap, status, n_mappings_used, n_edits_used);
}

// Device-pointer entry: inputs already in HBM, outputs stay in HBM; asynchronous on the handle's stream.
extern "C" int gb_map_batch_device(gb_device* d, const gb_map_params* hp, int paired, uint32_t n_reads,
                                   const uint8_t* d_reads, const uint8_t* d_quals, const uint64_t* d_read_off, uint32_t max_read_len,
                                   gb_alignment* d_aln, gb_mapping* d_mappings, uint64_t mapping_pool_cap, uint32_t* d_edits, uint64_t edit_pool_cap,
                                   uint8_t* d_status, uint64_t* d_totals) {
    if (!d || !hp || !d_reads || !d_read_off || !d_aln || !d_mappings || !d_edits || !d_status || !d_totals) return GB_ERR_ARG;
    if (n_reads == 0) return GB_OK;
    GB_CUDA(cudaSetDevice(d->device));
    return map_device(d, hp, n_reads, d_reads, d_quals, d_read_off, max_read_len, (uint64_t)n_reads * max_read_len, d_aln, d_status, paired != 0,
                      d_mappings, mapping_pool_cap, d_edits, edit_pool_cap, nullptr, 0, d_totals, nullptr);
}

// gb_map_batch_device cannot rerun a batch by itself (it only enqueues work): after synchronising, this tells whether the
// last batch ran out of intermediate pool space (reads then carry GB_ITEM_OUT_FULL) and, if so, doubles the pools for the
// next call, so the caller simply submits the batch again.
extern "C" int gb_device_pool_overflow(gb_device* d, int* overflowed) {
    if (!d || !overflowed) return GB_ERR_ARG;
    *overflowed = 0;
    if (!d->p_cursors.ptr) return GB_OK;
    GB_CUDA(cudaSetDevice(d->device));
    GB_CUDA(cudaStreamSynchronize(d->stream));
    uint32_t flag = 0;
    GB_CUDA(cudaMemcpy(&flag, d->p_cursors.ptr + 13, sizeof flag, cudaMemcpyDeviceToHost));
    if (flag) { *overflowed = 1; if (d->pool_scale < 1024.0) d->pool_scale *= 2.0; d->pool_reruns++; }
    return GB_OK;
}

// Stage dump for the parity tests: the seeding kernels only, then the pools as they left them, converted on the host.
extern "C" int gb_debug_seed_stage(gb_device* d, const gb_map_params* hp, int paired,
                                   uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                                   gb_stage_read* out_reads, gb_stage_minimizer* mins, uint64_t min_cap, gb_stage_seed* seeds, uint64_t seed_cap,
                                   gb_stage_cluster* clusters, uint64_t cluster_cap, gb_stage_item* items, uint64_t item_cap,
                                   gb_seed* item_seeds, uint64_t item_seed_cap) {
    if (!d || !hp || !reads || !read_off || !out_reads || !mins || !seeds || !clusters || !items || !item_seeds) return GB_ERR_ARG;
    if (n_reads == 0) return GB_OK;
    try {
        GB_CUDA(cudaSetDevice(d->device));
        const uint64_t total = read_off[n_reads];
        uint32_t max_len = 0;
        for (uint32_t r = 0; r < n_reads; r++) max_len = std::max<uint32_t>(max_len, (uint32_t)(read_off[r + 1] - read_off[r]));
        DevBuf<uint8_t> d_reads, d_quals, d_status; DevBuf<uint64_t> d_off, d_totals; DevBuf<gb_alignment> d_aln; DevBuf<DbgCluster> d_dbg;
        int rc;
        if ((rc = d_reads.upload(reads, total + 16, d->stream, total)) || (quals && (rc = d_quals.upload(quals, total + 16, d->stream, total))) ||
            (rc = d_off.upload(read_off, n_reads + 1, d->stream)) || (rc = d_status.reserve(n_reads)) || (rc = d_totals.reserve(2)) ||
            (rc = d_aln.reserve((size_t)n_reads * std::max<uint32_t>(hp->max_multimaps, 1u))) || (rc = d_dbg.reserve((size_t)n_reads * MAX_CLUSTERS))) return rc;
        GB_CUDA(cudaMemsetAsync(d_dbg.ptr, 0, sizeof(DbgCluster) * (size_t)n_reads * MAX_CLUSTERS, d->stream));
        std::vector<ReadState> st(n_reads);
        uint32_t cursors[16];
        for (int attempt = 0;; attempt++) {
            d->dbg_clusters = d_dbg.ptr; d->debug_stop_after_seed = true;
            rc = map_device(d, hp, n_reads, d_reads.ptr, quals ? d_quals.ptr : nullptr, d_off.ptr, max_len, total, d_aln.ptr, d_status.ptr, paired != 0,
                            nullptr, 0, nullptr, 0, nullptr, 0, d_totals.ptr, nullptr);
            d->dbg_clusters = nullptr; d->debug_stop_after_seed = false;
            if (rc) return rc;
            GB_CUDA(cudaStreamSynchronize(d->stream));
            GB_CUDA(cudaMemcpy(cursors, d->p_cursors.ptr, sizeof cursors, cudaMemcpyDeviceToHost));
            if (!cursors[13]) break;
            if (attempt >= 10) { g_last_error = "seed stage: pools overflow"; return GB_ERR_CAPACITY; }
            d->pool_scale *= 2.0; d->pool_reruns++;
        }
        GB_CUDA(cudaMemcpy(st.data(), d->p_states.ptr, sizeof(ReadState) * n_reads, cudaMemcpyDeviceToHost));
        std::vector<DevMinimizer> hm(cursors[1]); std::vector<DevSeed> hs(cursors[2]); std::vector<DevItem> hi(cursors[3]); std::vector<gb_seed> he(cursors[4]);
        std::vector<DbgCluster> hc((size_t)n_reads * MAX_CLUSTERS);
        if (!hm.empty()) GB_CUDA(cudaMemcpy(hm.data(), d->p_min.ptr, sizeof(DevMinimizer) * hm.size(), cudaMemcpyDeviceToHost));
        if (!hs.empty()) GB_CUDA(cudaMemcpy(hs.data(), d->p_seeds.ptr, sizeof(DevSeed) * hs.size(), cudaMemcpyDeviceToHost));
        if (!hi.empty()) GB_CUDA(cudaMemcpy(hi.data(), d->p_items.ptr, sizeof(DevItem) * hi.size(), cudaMemcpyDeviceToHost));
        if (!he.empty()) GB_CUDA(cudaMemcpy(he.data(), d->p_ext_seeds.ptr, sizeof(gb_seed) * he.size(), cudaMemcpyDeviceToHost));
        GB_CUDA(cudaMemcpy(hc.data(), d_dbg.ptr, sizeof(DbgCluster) * hc.size(), cudaMemcpyDeviceToHost));
        uint64_t nm = 0, ns = 0, nc = 0, ni = 0, ne = 0;
        for (uint32_t r = 0; r < n_reads; r++) {
            const ReadState& rs = st[r];
            gb_stage_read& o = out_reads[r];
            memset(&o, 0, sizeof o);
            o.status = rs.status;
            o.min_off = (uint32_t)nm; o.seed_off = (uint32_t)ns; o.cluster_off = (uint32_t)nc; o.item_off = (uint32_t)ni;
            if (rs.status != GB_ITEM_OK) continue;
            if (nm + rs.min_cnt > min_cap || ns + rs.seed_cnt > seed_cap || nc + rs.n_clusters > cluster_cap || ni + rs.item_cnt > item_cap) { g_last_error = "stage dump: output too small"; return GB_ERR_CAPACITY; }
            for (uint32_t i = 0; i < rs.min_cnt; i++) {
                const DevMinimizer& m = hm[rs.min_off + i];
                mins[nm + i] = gb_stage_minimizer{m.hash, m.score, m.fwd_offset, m.agg_start, m.agg_len, m.is_reverse, m.pad[1], 0};
            }
            // clusters in order of their first seed; a seed's label is the index of the first seed of its cluster
            std::vector<uint32_t> cluster_of_label(rs.seed_cnt, 0xffffffffu);
            for (uint32_t c = 0; c < rs.n_clusters; c++) {
                const DbgCluster& dc = hc[(size_t)r * MAX_CLUSTERS + c];
                if (!dc.valid || dc.first_seed >= rs.seed_cnt) { g_last_error = "stage dump: cluster record missing"; return GB_ERR_CUDA; }
                clusters[nc + c] = gb_stage_cluster{dc.score, dc.coverage, dc.first_seed, 0, dc.fragment, dc.kept_rank};
                cluster_of_label[dc.first_seed] = c;
            }
            for (uint32_t i = 0; i < rs.seed_cnt; i++) {
                const DevSeed& sd = hs[rs.seed_off + i];
                const uint32_t c = sd.label < rs.seed_cnt ? cluster_of_label[sd.label] : 0xffffffffu;
                seeds[ns + i] = gb_stage_seed{sd.node, sd.offset, sd.source, c};
                if (c != 0xffffffffu) clusters[nc + c].n_seeds++;
            }
            for (uint32_t t = 0; t < rs.item_cnt; t++) {
                const DevItem& it = hi[rs.item_off + t];
                if (ne + it.seed_cnt > item_seed_cap) { g_last_error = "stage dump: output too small"; return GB_ERR_CAPACITY; }
                uint32_t cl = 0xffffffffu;
                for (uint32_t c = 0; c < rs.n_clusters; c++) if (clusters[nc + c].kept_rank == t) cl = c;
                items[ni + t] = gb_stage_item{cl, it.fragment, (uint32_t)ne, it.seed_cnt};
                for (uint32_t x = 0; x < it.seed_cnt; x++) item_seeds[ne + x] = he[it.seed_off + x];
                ne += it.seed_cnt;
            }
            o.min_cnt = rs.min_cnt; o.seed_cnt = rs.seed_cnt; o.cluster_cnt = rs.n_clusters; o.item_cnt = rs.item_cnt;
            o.reserved[0] = rs.pad[0];          // > 1: cluster selection of this read (mate 2) is deferred to the align stage; items = all clusters in comparator order
            nm += rs.min_cnt; ns += rs.seed_cnt; nc += rs.n_clusters; ni += rs.item_cnt;
        }
        return GB_OK;
    } catch (...) { g_last_error = "stage dump: out of host memory"; return GB_ERR_CAPACITY; }
}

// Multi-GPU emission: gb_map_batch / gb_map_paired_batch additionally leave the records of the whole call in the caller's
// DEVICE buffers (same layout and offsets as the host outputs), so an NCCL gather can ship them without a second trip over
// PCIe.  NULL d_aln switches the mirror off.
extern "C" int gb_device_set_output_mirror(gb_device* d, gb_alignment* d_aln, gb_mapping* d_maps, uint64_t map_cap, uint32_t* d_edits, uint64_t edit_cap) {
    if (!d || (d_aln && (!d_maps || !d_edits))) return GB_ERR_ARG;
    d->mirror_aln = d_aln; d->mirror_maps = d_maps; d->mirror_edits = d_edits; d->mirror_map_cap = map_cap; d->mirror_edit_cap = edit_cap;
    return GB_OK;
}

extern "C" int gb_device_set_stream(gb_device* d, void* cuda_stream) {
    if (!d) return GB_ERR_ARG;
    d->stream = cuda_stream ? (cudaStream_t)cuda_stream : d->own_stream;
    return GB_OK;
}

extern "C" int gb_device_synchronize(gb_device* d) {
    if (!d) return GB_ERR_ARG;
    GB_CUDA(cudaSetDevice(d->device));
    GB_CUDA(cudaStreamSynchronize(d->stream));
    return GB_OK;
}

// Stage times of the last map_device call on this handle: seed, extend, align, compact (ms).
extern "C" int gb_stage_times(gb_device* d, float* ms4) {
    if (!d || !ms4) return GB_ERR_ARG;
    GB_CUDA(cudaSetDevice(d->device));
    GB_CUDA(cudaEventSynchronize(d->ev_stage[4]));
    for (int i = 0; i < 4; i++) GB_CUDA(cudaEventElapsedTime(&ms4[i], d->ev_stage[i], d->ev_stage[i + 1]));
    return GB_OK;
}

// Counters of the tail plan of the last mapping call (its last chunk): tails planned, trees, tails aligned in place by the
// align kernels although the unit had a plan (not planned, cancelled, or not tileable), DP cells of the tiles.
extern "C" int gb_plan_stats(gb_device* d, uint64_t* out4) {
    if (!d || !out4) return GB_ERR_ARG;
    for (int i = 0; i < 4; i++) out4[i] = 0;
    if (!d->pl_stats.ptr) return GB_OK;
    GB_CUDA(cudaSetDevice(d->device));
    GB_CUDA(cudaStreamSynchronize(d->stream));
    GB_CUDA(cudaMemcpy(out4, d->pl_stats.ptr, 4 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    return GB_OK;
}

// Device time of every kernel of the last mapping call on this handle (one chunk; CUDA events between the launches).
extern "C" int gb_kernel_times(gb_device* d, uint32_t cap, char* names, float* ms, uint32_t* n_out) {
    if (!d || !names || !ms || !n_out) return GB_ERR_ARG;
    GB_CUDA(cudaSetDevice(d->device));
    *n_out = 0;
    if (d->kt_n < 2) return GB_OK;
    GB_CUDA(cudaEventSynchronize(d->kt_ev[d->kt_n - 1]));
    for (int i = 1; i < d->kt_n && *n_out < cap; i++) {
        GB_CUDA(cudaEventElapsedTime(&ms[*n_out], d->kt_ev[i - 1], d->kt_ev[i]));
        std::strncpy(names + (size_t)*n_out * 48, d->kt_name[i], 47); names[(size_t)*n_out * 48 + 47] = 0;
        (*n_out)++;
    }
    return GB_OK;
}

// ---------------------------------------------------------------------------------------
// B3 stage seam: Aligner::align_pinned(xdrop = true), batched over explicit haplotype trees
// (aligner.cpp:628-686 -> DozeuInterface::align_pinned dozeu_interface.cpp:724-766).
// ---------------------------------------------------------------------------------------
namespace gb {

struct XdropBatch {
    const int32_t* tree_parent; const uint32_t* tree_node; const uint64_t* tree_off; const uint32_t* root_trim;
    const uint8_t* query; const uint64_t* query_off; const uint32_t* max_gap;
    uint32_t n; uint32_t Lc;
    SeamOut out;
    uint8_t* ws_base; size_t ws_stride; uint32_t tb_cells;
    uint32_t* work_counter;
    uint8_t* skip;                   // [n] 1: the problem ran on xdrop_tile_kernel instead
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

__global__ void __launch_bounds__(ALIGN_WARPS * 32, 4)
xdrop_kernel(DevIndex ix, DevScores sc, XdropBatch b) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t gwarp = blockIdx.x * ALIGN_WARPS + warp;
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

extern "C" int gb_xdrop_pinned_batch(gb_device* d, uint32_t n,
                                     const int32_t* tree_parent, const uint32_t* tree_node, const uint64_t* tree_off,
                                     const uint32_t* root_trim, const uint8_t* query, const uint64_t* query_off,
                                     const uint32_t* max_gap, uint32_t map_cap, uint32_t edit_cap,
                                     int32_t* score, gb_mapping* maps, uint32_t* edits, uint32_t* n_maps, uint32_t* n_edits,
                                     uint8_t* status) {
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
        lineage.clear();                      // root .. previous node
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
    const size_t smem = dp_smem_per_warp(Lc) * ALIGN_WARPS;
    if (smem > 48 * 1024) GB_CUDA(cudaFuncSetAttribute(xdrop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    uint32_t grid = std::min<uint32_t>((uint32_t)d->n_sms * 2, (n + ALIGN_WARPS - 1) / ALIGN_WARPS);
    const uint32_t tb_cells = 2 * 1024 * 1024;
    const size_t ws_stride = tail_ws_bytes(Lc, tb_cells);
    if ((rc = d_ws.reserve(ws_stride * grid * ALIGN_WARPS))) return rc;
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
    DevBuf<uint8_t> d_elig, d_tiles; DevBuf<uint32_t> d_tileoff, d_lists, d_tc, d_paths; DevBuf<TileResult> d_res;
    GB_CUDA(cudaEventRecord(d->ev0, d->stream));
    if (n_elig) {
        const uint32_t path_cap = (uint32_t)std::min<uint64_t>((uint64_t)n * (2 * TILE_MAP_CAP + TILE_EDIT_CAP), 0xfffffff0ull);
        if ((rc = d_elig.upload(elig.data(), n, d->stream)) || (rc = d_tileoff.upload(toff.data(), n, d->stream)) || (rc = d_tiles.reserve(units * 16 + 16)) ||
            (rc = d_lists.reserve(TILE_CLASSES * (size_t)n)) || (rc = d_tc.reserve(32)) || (rc = d_res.reserve(n)) || (rc = d_paths.reserve(path_cap))) return rc;
        GB_CUDA(cudaMemsetAsync(d_tc.ptr, 0, 128, d->stream));
        GB_CUDA(cudaMemsetAsync(d_res.ptr, 0xff, sizeof(TileResult) * (size_t)n, d->stream));
        PackBatch pk;
        pk.tree_parent = d_par.ptr; pk.tree_node = d_node.ptr; pk.tree_off = d_toff.ptr; pk.root_trim = d_trim.ptr;
        pk.query = d_q.ptr; pk.query_off = d_qoff.ptr; pk.max_gap = d_gap.ptr; pk.n = n; pk.tiles = d_tiles.ptr; pk.tile_off = d_tileoff.ptr;
        for (int c = 0; c < TILE_CLASSES; c++) pk.lists[c] = d_lists.ptr + (size_t)c * n;
        pk.list_count = d_tc.ptr; pk.eligible = d_elig.ptr;
        pack_tiles_kernel<<<(n + 7) / 8, 256, 0, d->stream>>>(d->ix, d->sc, pk);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        d->kt_reset();
        if ((rc = launch_tile_kernels(d, d_tiles.ptr, d_tileoff.ptr, d_lists.ptr, n, d_tc.ptr, d_tc.ptr + 8, d_res.ptr, d_paths.ptr, path_cap, d_tc.ptr + 16))) return rc;
        b.skip = d_elig.ptr;
        unpack_tile_results_kernel<<<(n + 7) / 8, 256, 0, d->stream>>>(b, d_res.ptr, d_paths.ptr);
        d->launches++;
        GB_CUDA(cudaGetLastError());
    } else b.skip = nullptr;
    // the int32 sweep takes the problems not eligible for a tile and those whose tile ended FULL; the latter are known only
    // on the device, so it runs after the tiles too and skips the problems they finished
    xdrop_kernel<<<grid, ALIGN_WARPS * 32, smem, d->stream>>>(d->ix, d->sc, b);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    d->last_tile_problems = n_elig;
    GB_CUDA(cudaEventRecord(d->ev1, d->stream));
    return out.download(d, n, score, maps, edits, n_maps, n_edits, status);
}
