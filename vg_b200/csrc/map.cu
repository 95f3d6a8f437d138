// map.cu — gb_map_batch / gb_map_paired_batch: the single- and paired-end Giraffe hot path on the GPU.
//   map_device runs the stages of one batch (a chunk of the host-buffer entry points):
//     seeding       seed_kernel / seed_kernel_pe (map_paired.cuh), then a second pass at the maximum table sizes
//     extension     extend_kernel + extend_finish_kernel (capi.cu), then the repeats again with large strides
//     align         align_fast_kernel(_pe) (align_fast.cuh), thread per unit; the units it cannot finish go on to
//     tails         tail_plan_kernel, xdrop_tile_kernel per size class, tail_decide_kernel, tiles again (tail_plan.cuh)
//                   and align_kernel / align_kernel_pe (+ its rescue build), warp per unit
//     compaction    compact.cuh: the records packed into the caller's pools
//   The persistent kernels pull work from the counters of MapCursors; intermediate records stay in HBM (map_state.cuh).
// No CPU fallback: every stage is a CUDA kernel; the host only moves buffers and launches.
#include <cub/cub.cuh>
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "seed.cuh"
#include "align.cuh"
#include "extend.cuh"
#include "dag_dp.cuh"

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
            stage_read(sm.read, b.reads + rb, L);
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
    const AlignSmem sm = align_smem_carve(smem, warp, b.Lc, 1, a.tmp_bytes);
    uint8_t* sread = sm.read[0]; uint8_t* squal = sm.qual[0]; uint8_t* qbuf = sm.qbuf; uint8_t* stmp = sm.tmp;
    const DpSmem dps = sm.dps;
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

// xdrop_tile_kernel per size class c, which runs R = tile_class_rows(c) rows per lane.
struct TileClassKernel { void (*kernel)(DevScores, TileBatch); size_t smem; const char* name; };
static_assert(tile_class_rows(0) == 2 && tile_class_rows(1) == 4 && tile_class_rows(2) == 6 && tile_class_rows(3) == 8 &&
              tile_class_rows(4) == 12 && tile_class_rows(5) == 16, "TILE_CLASS_KERNELS follows tile_class_rows");
static const TileClassKernel TILE_CLASS_KERNELS[TILE_CLASSES] = {
    {xdrop_tile_kernel<2>, tile_smem_per_warp<2>() * TILE_WARPS, "xdrop_tile_kernel<2>"},
    {xdrop_tile_kernel<4>, tile_smem_per_warp<4>() * TILE_WARPS, "xdrop_tile_kernel<4>"},
    {xdrop_tile_kernel<6>, tile_smem_per_warp<6>() * TILE_WARPS, "xdrop_tile_kernel<6>"},
    {xdrop_tile_kernel<8>, tile_smem_per_warp<8>() * TILE_WARPS, "xdrop_tile_kernel<8>"},
    {xdrop_tile_kernel<12>, tile_smem_per_warp<12>() * TILE_WARPS, "xdrop_tile_kernel<12>"},
    {xdrop_tile_kernel<16>, tile_smem_per_warp<16>() * TILE_WARPS, "xdrop_tile_kernel<16>"},
};

int launch_tile_kernels(gb_device* d, const uint8_t* tiles, const uint32_t* tile_off, const uint32_t* lists, size_t list_cap,
                        const uint32_t* list_count, uint32_t* work, TileResult* results, uint32_t* paths, uint32_t path_cap, uint32_t* path_cursor) {
    int rc;
    if ((rc = d->ws_tile.reserve(tile_ws_bytes() * (size_t)d->n_sms * 2 * TILE_WARPS))) return rc;
    for (int cls = 0; cls < TILE_CLASSES; cls++) {
        const TileClassKernel& k = TILE_CLASS_KERNELS[cls];
        GB_CUDA(cudaFuncSetAttribute(k.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem));
        int bps = 0;
        GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, k.kernel, TILE_WARPS * 32, k.smem));
        bps = std::max(1, std::min(bps, 2));
        TileBatch tb;
        tb.tiles = tiles; tb.tile_off = tile_off; tb.list = lists + (size_t)cls * list_cap; tb.list_count = list_count + cls; tb.list_cap = (uint32_t)list_cap;
        tb.work_counter = work + cls; tb.results = results; tb.path_pool = paths; tb.path_cap = path_cap; tb.path_cursor = path_cursor;
        tb.ws_base = d->ws_tile.ptr; tb.ws_stride = tile_ws_bytes();
        k.kernel<<<(uint32_t)(d->n_sms * bps), TILE_WARPS * 32, k.smem, d->stream>>>(d->sc, tb);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        if ((rc = d->kt_mark(k.name))) return rc;
    }
    return GB_OK;
}

// What the stages of one map_device call share.
struct MapRun {
    gb_device* d; const gb_map_params* hp;
    uint32_t n_reads, n_units, K, Lc;          // n_units: reads, or pairs when paired
    bool paired, rescue;
    MapParamsDev P;
    MapCursors* cur;
    MapBatch b;                                // the reads as the kernels see them (paired: mate 2 rightward)
    SeedPools pools;
    size_t item_cap;
    int32_t fragment_limit;
    AlignArgs a;                               // ev from the extension stage, plan from the tail stage
    // the warp-per-unit align kernels: the plain build (align_kernel or align_kernel_pe<false>), its grid, the grid of
    // the rescue build, their dynamic shared memory
    void (*align)(DevIndex, MapParamsDev, DevScores, MapBatch, AlignArgs);
    uint32_t grid_plain, grid_rescue;
    size_t align_smem;
};

static MapBatch with_work(const MapBatch& b, uint32_t* work_counter) {
    MapBatch x = b;
    x.work_counter = work_counter;
    return x;
}

// Parameter tables (host libm, so scores are bit-identical to a CPU run) and the device copy of the parameters.
static int map_params(gb_device* d, const gb_map_params* hp, uint32_t n_reads, bool paired, MapParamsDev& P) {
    int rc;
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
    P.hit_cap = hp->hit_cap; P.hard_hit_cap = hp->hard_hit_cap; P.minimizer_score_fraction = hp->minimizer_score_fraction;
    P.minimizer_coverage_flank = hp->minimizer_coverage_flank; P.max_unique_min = hp->max_unique_min; P.num_bp_per_min = hp->num_bp_per_min;
    P.distance_limit = hp->distance_limit; P.min_extensions = hp->min_extensions; P.max_extensions = hp->max_extensions;
    P.cluster_score_threshold = hp->cluster_score_threshold; P.pad_cluster_score_threshold = hp->pad_cluster_score_threshold;
    P.cluster_coverage_threshold = hp->cluster_coverage_threshold; P.extension_set_score_threshold = hp->extension_set_score_threshold;
    P.extension_score_threshold = hp->extension_score_threshold; P.min_extension_sets = hp->min_extension_sets;
    P.extension_set_min_score = hp->extension_set_min_score; P.max_alignments = hp->max_alignments;
    P.max_extension_mismatches = hp->max_extension_mismatches; P.max_dozeu_cells = hp->max_dozeu_cells; P.do_dp = hp->do_dp;
    P.mapping_cap = hp->mapping_cap_per_read; P.edit_cap = hp->edit_cap_per_read;
    P.max_multimaps = hp->max_multimaps; P.out_stride = n_reads;
    P.log_base = recover_log_base(d->sc);
    P.max_rescue_attempts = paired ? hp->max_rescue_attempts : 0; P.rescue_seed_limit = hp->rescue_seed_limit;
    P.paired_rescue_score_limit = hp->paired_rescue_score_limit; P.rescue_subgraph_stdevs = hp->rescue_subgraph_stdevs;
    P.rescue_likelihood_limit = hp->rescue_likelihood_limit;
    P.hit_score_table = d->t_hit.ptr; P.prob_at_least_one = d->t_plo.ptr; P.phred_prob = d->t_phred.ptr;
    return GB_OK;
}

// K1: a first pass with small shared tables (8 blocks per SM), then the units that did not fit (many minimizers or
// clusters) once more at the maximum table sizes.
static int map_seed(MapRun& r) {
    gb_device* d = r.d;
    int rc;
    if ((rc = d->p_retry.reserve(r.n_units + 1))) return rc;
    for (int pass = 0; pass < 2; pass++) {
        MapBatch bp = r.b;
        bp.Mc = pass == 0 ? d->seed_mc : MAX_MINIMIZERS; bp.Cc = pass == 0 ? d->seed_cc : MAX_CLUSTERS;
        bp.work_counter = pass == 0 ? &r.cur->seed_work : &r.cur->seed_retry_work;
        bp.in_list = pass == 0 ? nullptr : d->p_retry.ptr; bp.in_count = pass == 0 ? nullptr : &r.cur->seed_retry_count;
        bp.retry_list = d->p_retry.ptr; bp.retry_count = pass == 0 ? &r.cur->seed_retry_count : &r.cur->seed_retry_again;
        // the cluster phases carve their scratch from the arrays that are dead after phase A
        while (seed_dead_bytes(r.Lc, bp.Mc) < cluster_scratch_bytes(bp.Cc) && bp.Mc < MAX_MINIMIZERS) bp.Mc += 8;
        uint32_t warps = SEED_WARPS;
        while (warps > 1 && seed_smem_bytes(r.Lc, bp.Mc, bp.Cc) * warps > 200 * 1024) warps >>= 1;
        const size_t smem = seed_smem_bytes(r.Lc, bp.Mc, bp.Cc) * warps;
        const bool fixed_layout = r.Lc == 160 && bp.Mc == 64 && bp.Cc == 16;
        auto seed_pe = fixed_layout ? seed_kernel_pe<160, 64, 16> : seed_kernel_pe<0, 0, 0>;
        const void* kern = r.paired ? (const void*)seed_pe : (const void*)seed_kernel;
        if (smem > 48 * 1024) GB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int bps = 0;
        GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, kern, warps * 32, smem));
        if (bps < 1) bps = 1;
        uint32_t grid = std::min<uint32_t>((uint32_t)(d->n_sms * bps), (r.n_units + warps - 1) / warps);
        if (grid == 0) grid = 1;
        if (r.paired) seed_pe<<<grid, warps * 32, smem, d->stream>>>(d->ix, r.P, bp, r.pools, PairBatch{d->p_pairs.ptr, r.fragment_limit});
        else seed_kernel<<<grid, warps * 32, smem, d->stream>>>(d->ix, r.P, bp, r.pools);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        if ((rc = d->kt_mark(pass == 0 ? (r.paired ? "seed_kernel_pe" : "seed_kernel") : "seed_kernel(retry tables)"))) return rc;
    }
    return GB_OK;
}

// K2: extension over the items produced on the device.
static int map_extend(MapRun& r) {
    gb_device* d = r.d;
    const size_t item_cap = r.item_cap;
    const uint32_t max_ext = 48, path_cap = 384, mism_cap = 192;
    int rc;
    if ((rc = d->p_ext_count.reserve(item_cap))) return rc;
    if ((rc = d->p_ext_status.reserve(item_cap))) return rc;
    if ((rc = d->p_ext.reserve(item_cap * max_ext))) return rc;
    if ((rc = d->p_path.reserve(item_cap * path_cap))) return rc;
    if ((rc = d->p_mism.reserve(item_cap * mism_cap))) return rc;
    // clusters whose seeds yield more extensions than those strides hold (repeats: a hundred seeds in one cluster, one
    // extension per seed before GaplessExtender::extend removes duplicates) are redone with large strides
    ExtendBig big;
    big.cap = r.n_reads / 128 + 256; big.max_ext = 512; big.path_cap = 512 * 24; big.mism_cap = 512 * 4;
    if ((rc = d->p_big_list.reserve(big.cap)) || (rc = d->p_big_of.reserve(item_cap)) || (rc = d->p_big_ext.reserve((size_t)big.cap * big.max_ext)) ||
        (rc = d->p_big_path.reserve((size_t)big.cap * big.path_cap)) || (rc = d->p_big_mism.reserve((size_t)big.cap * big.mism_cap))) return rc;
    GB_CUDA(cudaMemsetAsync(d->p_big_of.ptr, 0xff, sizeof(uint32_t) * item_cap, d->stream));
    big.list = d->p_big_list.ptr; big.count = &r.cur->big_ext_count; big.big_of = d->p_big_of.ptr;
    big.ext = d->p_big_ext.ptr; big.path = d->p_big_path.ptr; big.mism = d->p_big_mism.ptr;
    ExtendParams ep;
    ep.sc = d->sc; ep.max_mismatches = r.hp->max_extension_mismatches; ep.overlap_threshold = 0.8; ep.overlap_threshold_unused = 0.f;
    ep.trim = 1; ep.max_ext = max_ext; ep.path_cap = path_cap; ep.mism_cap = mism_cap;
    if ((rc = launch_extend_device(d, ep, r.b.reads, r.b.read_off, nullptr, d->p_ext_seeds.ptr, nullptr, d->p_items.ptr, &r.cur->item_cursor,
                                   (uint32_t)item_cap, d->p_ext_count.ptr, d->p_ext_status.ptr, d->p_ext.ptr, d->p_path.ptr,
                                   d->p_mism.ptr, r.Lc, &big))) return rc;
    ExtView& ev = r.a.ev;
    ev.ext_count = d->p_ext_count.ptr; ev.ext_status = d->p_ext_status.ptr; ev.ext = d->p_ext.ptr;
    ev.path_pool = d->p_path.ptr; ev.mism_pool = d->p_mism.ptr; ev.max_ext = max_ext; ev.path_cap = path_cap; ev.mism_cap = mism_cap;
    ev.big_of = d->p_big_of.ptr; ev.big_ext = d->p_big_ext.ptr; ev.big_path = d->p_big_path.ptr; ev.big_mism = d->p_big_mism.ptr;
    ev.big_max_ext = big.max_ext; ev.big_path_cap = big.path_cap; ev.big_mism_cap = big.mism_cap;
    return GB_OK;
}

// K3 setup: the warp-per-unit kernels' builds, grids and shared memory, their per-warp workspaces, the AlignArgs.
static int setup_align(MapRun& r) {
    gb_device* d = r.d; const gb_map_params* hp = r.hp;
    // the five temporary path buffers of a warp go to shared memory when they fit beside the DP columns
    const size_t slot_bytes = (size_t)hp->mapping_cap_per_read * sizeof(gb_mapping) + (size_t)hp->edit_cap_per_read * 4;
    const uint32_t tmp_bytes = N_TEMP_SLOTS * slot_bytes <= 12 * 1024 ? (uint32_t)(N_TEMP_SLOTS * slot_bytes) : 0u;
    const size_t smem = align_smem_per_warp(r.Lc, r.paired ? 2 : 1, tmp_bytes) * ALIGN_WARPS;
    r.align = r.paired ? align_kernel_pe<false> : align_kernel;
    if (smem > 48 * 1024) {
        GB_CUDA(cudaFuncSetAttribute(r.align, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (r.rescue) GB_CUDA(cudaFuncSetAttribute(align_kernel_pe<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    int bps = 0, bps_rescue = 0;
    if (r.rescue) GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps_rescue, align_kernel_pe<true>, ALIGN_WARPS * 32, smem));
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, r.align, ALIGN_WARPS * 32, smem));
    bps = std::max(1, std::min(bps, 4));                  // 4 bounds the per-warp tail workspaces (about 2 MB each)
    r.grid_plain = std::max<uint32_t>(1u, std::min<uint32_t>((uint32_t)(d->n_sms * bps), (r.n_reads + ALIGN_WARPS - 1) / ALIGN_WARPS));
    bps_rescue = std::max(1, std::min(bps_rescue, 2));    // + the rescue workspaces (about 2 MB each)
    r.grid_rescue = r.rescue ? std::min<uint32_t>((uint32_t)(d->n_sms * bps_rescue), r.grid_plain) : r.grid_plain;
    r.align_smem = smem;
    const size_t n_warps = (size_t)r.grid_plain * ALIGN_WARPS;
    const uint32_t tb_cells = hp->max_dozeu_cells + hp->max_dozeu_cells / 4 + 4096;
    const size_t ws_stride = tail_ws_bytes(r.Lc, tb_cells);
    const size_t cand_stride = (((size_t)hp->mapping_cap_per_read * sizeof(gb_mapping) + (size_t)hp->edit_cap_per_read * 4) * (N_SLOTS + N_TEMP_SLOTS) + 255) & ~(size_t)255;
    int rc;
    if ((rc = d->ws_tail.reserve(ws_stride * n_warps))) return rc;
    if ((rc = d->ws_cand.reserve(cand_stride * n_warps))) return rc;
    AlignArgs& a = r.a;
    a.tmp_bytes = tmp_bytes;
    if (r.rescue) {
        a.rescue_stride = (rescue_ws_bytes(r.Lc) + 255) & ~(size_t)255;
        if ((rc = d->ws_rescue.reserve(a.rescue_stride * (size_t)r.grid_rescue * ALIGN_WARPS))) return rc;
        if ((rc = d->p_rescue.reserve(r.n_reads / 2 + 1))) return rc;
        a.rescue_base = d->ws_rescue.ptr;
    }
    a.items = d->p_items.ptr; a.minimizers = d->p_min.ptr;
    a.ws_base = d->ws_tail.ptr; a.ws_stride = ws_stride; a.cand_base = d->ws_cand.ptr; a.cand_stride = cand_stride;
    a.tb_cells = tb_cells;
    a.pairs = r.paired ? d->p_pairs.ptr : nullptr; a.frag_mean = hp->fragment_mean; a.frag_sd = hp->fragment_stdev;
    return d->p_slow.reserve(r.n_units + 1);
}

// Thread-per-unit fast path; whatever it cannot finish goes to the slow list of the warp-per-unit kernels.
static int map_align_fast(MapRun& r) {
    gb_device* d = r.d;
    FastArgs fa; fa.slow_list = d->p_slow.ptr; fa.slow_count = &r.cur->slow_count;
    const uint32_t fgrid = std::max<uint32_t>(1u, std::min<uint32_t>((r.n_units + 127) / 128, (uint32_t)d->n_sms * 16));
    auto fast = r.paired ? align_fast_kernel_pe : align_fast_kernel;
    fast<<<fgrid, 128, 0, d->stream>>>(d->ix, r.P, d->sc, with_work(r.b, &r.cur->align_work), r.a, fa);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    int rc;
    if ((rc = d->kt_mark(r.paired ? "align_fast_kernel_pe" : "align_fast_kernel"))) return rc;
    r.a.slow_list = d->p_slow.ptr; r.a.slow_count = &r.cur->slow_count;
    return GB_OK;
}

// Tails of the slow units: the plan (forests -> tiles), then the DP of every tile in its own compact kernel.  Wave 0: the
// tails that are always aligned; the decide pass cancels what the reference would skip; wave 1: the rest.
static int map_tails(MapRun& r) {
    gb_device* d = r.d; MapCursors* cur = r.cur;
    const size_t tile_cap = (size_t)r.n_reads * 4 + 4096;
    const size_t unit_cap = std::min<size_t>((size_t)r.n_reads * 128 + (1u << 20), 0xfffffff0u);
    const size_t path_cap = std::min<size_t>(tile_cap * 32, 0xfffffff0u);
    int rc;
    if ((rc = d->pl_entries.reserve((size_t)r.n_units * PLAN_PER_UNIT)) || (rc = d->pl_unit_base.reserve(r.n_units)) || (rc = d->pl_unit_count.reserve(r.n_units)) ||
        (rc = d->pl_tiles.reserve(unit_cap * 16)) || (rc = d->pl_tile_off.reserve(tile_cap)) || (rc = d->pl_results.reserve(tile_cap)) ||
        (rc = d->pl_lists.reserve(2 * TILE_CLASSES * tile_cap)) || (rc = d->pl_paths.reserve(path_cap)) || (rc = d->pl_stats.reserve(4))) return rc;
    GB_CUDA(cudaMemsetAsync(d->pl_stats.ptr, 0, 4 * sizeof(uint64_t), d->stream));
    PlanPools pp;
    pp.entries = d->pl_entries.ptr; pp.unit_base = d->pl_unit_base.ptr; pp.unit_count = d->pl_unit_count.ptr;
    pp.tiles = d->pl_tiles.ptr; pp.tile_units_cap = (uint32_t)unit_cap; pp.tile_units_cursor = &cur->tile_units;
    pp.tile_off = d->pl_tile_off.ptr; pp.tile_cap = (uint32_t)tile_cap; pp.tile_cursor = &cur->tile_count;
    pp.results = d->pl_results.ptr;
    for (int c = 0; c < 2 * TILE_CLASSES; c++) pp.lists[c] = d->pl_lists.ptr + (size_t)c * tile_cap;
    pp.list_count = cur->tile_list_count; pp.stats = d->pl_stats.ptr;
    auto wave = [&](int w) {
        return launch_tile_kernels(d, d->pl_tiles.ptr, d->pl_tile_off.ptr, d->pl_lists.ptr + (size_t)w * TILE_CLASSES * tile_cap, tile_cap,
                                   cur->tile_list_count + w * TILE_CLASSES, cur->tile_work + w * TILE_CLASSES, d->pl_results.ptr,
                                   d->pl_paths.ptr, (uint32_t)path_cap, &cur->tile_path_words);
    };
    auto plan = r.paired ? tail_plan_kernel<true> : tail_plan_kernel<false>;
    plan<<<r.grid_plain, ALIGN_WARPS * 32, 0, d->stream>>>(d->ix, r.P, d->sc, with_work(r.b, &cur->plan_work), r.a, pp);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    if ((rc = d->kt_mark("tail_plan_kernel")) || (rc = wave(0))) return rc;
    auto decide = r.paired ? tail_decide_kernel<true> : tail_decide_kernel<false>;
    decide<<<r.grid_plain, ALIGN_WARPS * 32, 0, d->stream>>>(d->ix, r.P, d->sc, with_work(r.b, &cur->decide_work), r.a, pp);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    if ((rc = d->kt_mark("tail_decide_kernel")) || (rc = wave(1))) return rc;
    PlanView& pv = r.a.plan;
    pv.entries = d->pl_entries.ptr; pv.unit_base = d->pl_unit_base.ptr; pv.unit_count = d->pl_unit_count.ptr;
    pv.tile_off = d->pl_tile_off.ptr; pv.results = d->pl_results.ptr; pv.path_pool = d->pl_paths.ptr; pv.stats = d->pl_stats.ptr;
    return GB_OK;
}

// The warp-per-unit align kernel over the slow list.  Paired with rescue enabled, it defers the pairs that turn out to
// have unpaired alignments to a second list, which the (larger, lower-occupancy) rescue build then redoes.
static int map_align_warp(MapRun& r) {
    gb_device* d = r.d; MapCursors* cur = r.cur;
    if (r.paired) { r.a.rescue_list = d->p_rescue.ptr; r.a.rescue_count = &cur->rescue_count; }
    r.align<<<r.grid_plain, ALIGN_WARPS * 32, r.align_smem, d->stream>>>(d->ix, r.P, d->sc, with_work(r.b, &cur->align_work), r.a);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    if (!r.rescue) return d->kt_mark(r.paired ? "align_kernel_pe" : "align_kernel");
    int rc;
    if ((rc = d->kt_mark("align_kernel_pe"))) return rc;
    AlignArgs a = r.a;
    a.slow_list = d->p_rescue.ptr; a.slow_count = &cur->rescue_count;
    align_kernel_pe<true><<<r.grid_rescue, ALIGN_WARPS * 32, r.align_smem, d->stream>>>(d->ix, r.P, d->sc, with_work(r.b, &cur->rescue_work), a);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    return d->kt_mark("align_kernel_pe<rescue>");
}

// Device-resident mapping of a batch whose reads are already in HBM.
int map_device(gb_device* d, const gb_map_params* hp, uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals,
               const uint64_t* d_read_off, uint32_t max_len, uint64_t total_bases,
               gb_alignment* d_aln, uint8_t* d_status, bool paired,
               gb_mapping* out_maps, uint64_t out_map_cap, uint32_t* out_edits, uint64_t out_edit_cap,
               const uint64_t* d_run_base, uint32_t read_base, uint64_t* d_totals, uint32_t* d_overflow) {
    int rc;
    if (hp->max_multimaps == 0 || hp->max_multimaps > GB_MAX_MULTIMAPS) { g_last_error = "max_multimaps must be 1 .. GB_MAX_MULTIMAPS"; return GB_ERR_ARG; }
    // node ids are those of the 32-bit n_nodes (below 2^31 - 1); chain coordinates must fit the seeds' int32 c_in / c_out
    if (!d->chain_coords_fit) { g_last_error = "the index's chain coordinates do not fit 32 bits (x_in + node length above 2^31 - 1, or x_out - node length below -2^31)"; return GB_ERR_CAPACITY; }
    const uint32_t K = hp->max_multimaps;            // records per read, rank-major: record j * n_reads + read
    if ((uint64_t)n_reads * K * std::max(hp->mapping_cap_per_read, hp->edit_cap_per_read) > 0xffffffffull) { g_last_error = "chunk too large for 32-bit record offsets (reads x max_multimaps x cap)"; return GB_ERR_ARG; }
    if ((rc = d->pad_maps.reserve((size_t)n_reads * K * hp->mapping_cap_per_read))) return rc;
    if ((rc = d->pad_edits.reserve((size_t)n_reads * K * hp->edit_cap_per_read))) return rc;
    if (paired) {
        if (n_reads % 2 != 0) { g_last_error = "paired mapping needs an even number of reads"; return GB_ERR_ARG; }
        if (hp->max_rescue_attempts != 0 && hp->rescue_seed_limit >= RESCUE_SEEDS) { g_last_error = "rescue_seed_limit must be below 128"; return GB_ERR_ARG; }
        if (!(hp->fragment_stdev > 0)) { g_last_error = "paired mapping needs a forced fragment length distribution"; return GB_ERR_ARG; }
    }
    const uint32_t Lc = std::max<uint32_t>(32u, (max_len + 15u) & ~15u);
    if (Lc > 512) { g_last_error = "reads longer than 512 bp are not supported by the short-read path"; return GB_ERR_ARG; }
    MapRun r{};
    r.d = d; r.hp = hp; r.n_reads = n_reads; r.n_units = paired ? n_reads / 2 : n_reads; r.K = K; r.Lc = Lc;
    r.paired = paired; r.rescue = paired && hp->max_rescue_attempts != 0;
    if ((rc = map_params(d, hp, n_reads, paired, r.P))) return rc;

    // ---- pools ----
    // Sized from per-read averages (48 minimizers, 64 seeds, 3 kept clusters) times d->pool_scale.  A chunk that needs
    // more sets the sticky MapCursors::pool_overflow; the host-buffer entry points then double the scale and rerun the
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
    if ((rc = d->p_cursors.reserve(1))) return rc;
    GB_CUDA(cudaMemsetAsync(d->p_cursors.ptr, 0, sizeof(MapCursors), d->stream));
    MapCursors* cur = r.cur = d->p_cursors.ptr;
    r.item_cap = item_cap;
    d->kt_reset();
    if (K > 1) {
        init_absent_kernel<<<d->n_sms * 4, 256, 0, d->stream>>>(d_aln, n_reads, n_reads * K, hp->mapping_cap_per_read, hp->edit_cap_per_read);
        d->launches++;
        GB_CUDA(cudaGetLastError());
    }
    if (paired) {
        // rightward working copy of the reads (mate 2 reverse-complemented), :1503-1506
        if ((rc = d->w_reads.reserve(total_bases ? total_bases : 1))) return rc;
        if (d_quals) { if ((rc = d->w_quals.reserve(total_bases ? total_bases : 1))) return rc; }
        prep_pairs_kernel<<<d->n_sms * 8, 256, 0, d->stream>>>(d_reads, d_quals, d_read_off, n_reads, d->w_reads.ptr, d_quals ? d->w_quals.ptr : nullptr);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        d_reads = d->w_reads.ptr; if (d_quals) d_quals = d->w_quals.ptr;
        r.fragment_limit = (int32_t)(int64_t)(hp->fragment_mean + hp->paired_distance_stdevs * hp->fragment_stdev);   // :1470
        const uint32_t read_limit = std::max<uint32_t>(hp->distance_limit, max_len + 50);
        if (r.fragment_limit < (int32_t)read_limit) { g_last_error = "fragment distance limit smaller than the read distance limit (the reference falls back to single-end, :1471)"; return GB_ERR_ARG; }
        if ((rc = d->p_pairs.reserve(n_reads / 2))) return rc;
    }
    MapBatch& b = r.b;
    b.reads = d_reads; b.quals = d_quals; b.read_off = d_read_off; b.n_reads = n_reads;
    b.states = d->p_states.ptr; b.work_counter = &cur->seed_work; b.Lc = Lc;
    b.in_list = nullptr; b.in_count = nullptr; b.retry_list = nullptr; b.retry_count = nullptr; b.Mc = MAX_MINIMIZERS; b.Cc = MAX_CLUSTERS; b.Ns = d->seed_ns;
    SeedPools& pools = r.pools;
    pools.dbg_clusters = d->dbg_clusters; pools.overflow = &cur->pool_overflow;
    pools.minimizers = d->p_min.ptr; pools.min_cap = (uint32_t)min_cap; pools.min_cursor = &cur->min_cursor;
    pools.seeds = d->p_seeds.ptr; pools.seed_cap = (uint32_t)seed_cap; pools.seed_cursor = &cur->seed_cursor;
    pools.items = d->p_items.ptr; pools.item_cap = (uint32_t)item_cap; pools.item_cursor = &cur->item_cursor;
    pools.ext_seeds = d->p_ext_seeds.ptr; pools.ext_cap = (uint32_t)ext_cap; pools.ext_cursor = &cur->ext_cursor;
    r.a.aln = d_aln; r.a.maps = d->pad_maps.ptr; r.a.edits = d->pad_edits.ptr; r.a.status = d_status;

    GB_CUDA(cudaEventRecord(d->ev_stage[0], d->stream));
    if ((rc = d->kt_mark("start")) || (rc = map_seed(r))) return rc;
    GB_CUDA(cudaEventRecord(d->ev_stage[1], d->stream));
    if (d->debug_stop_after_seed) return GB_OK;              // gb_debug_seed_stage reads the pools as the seeding kernels left them
    if ((rc = map_extend(r))) return rc;
    GB_CUDA(cudaEventRecord(d->ev_stage[2], d->stream));
    if ((rc = setup_align(r)) || (rc = map_align_fast(r))) return rc;
    if (hp->do_dp && d->use_tiles && (rc = map_tails(r))) return rc;
    if ((rc = map_align_warp(r))) return rc;
    GB_CUDA(cudaEventRecord(d->ev_stage[3], d->stream));
    if ((rc = compact_outputs(d, n_reads * K, n_reads, d_aln, d->pad_maps.ptr, d->pad_edits.ptr, hp->mapping_cap_per_read, hp->edit_cap_per_read,
                              out_maps, out_map_cap, out_edits, out_edit_cap, d_run_base, read_base, d_totals, d_status))) return rc;
    if ((rc = d->kt_mark("compact (2 scans + gather)"))) return rc;
    if (d_overflow) GB_CUDA(cudaMemcpyAsync(d_overflow, &cur->pool_overflow, sizeof(uint32_t), cudaMemcpyDeviceToDevice, d->stream));
    GB_CUDA(cudaEventRecord(d->ev_stage[4], d->stream));
    return GB_OK;
}

int grow_pools_for_rerun(gb_device* d) {
    if (d->pool_scale >= 1024.0) { g_last_error = "intermediate pools overflow even at 1024x the per-read averages; use a smaller GIRAFFE_B200_MAP_CHUNK"; return GB_ERR_CAPACITY; }
    d->pool_scale *= 2.0; d->pool_reruns++;
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
        for (uint32_t p = 0; p < n_reads / 2; p++)
            fallback += gb::single_end_fallback(fragment_limit, hp->distance_limit, (int64_t)(read_off[2 * (size_t)p + 1] - read_off[2 * (size_t)p]));
        if (fallback == n_reads / 2) {
            const int rcs = map_batch_host(d, hp, false, n_reads, reads, quals, read_off, aln, mappings, mapping_pool_cap, edits, edit_pool_cap,
                                           status, n_mappings_used, n_edits_used);
            if (rcs == GB_OK) for (size_t r = 0; r < (size_t)n_reads * K; r++) if (!(aln[r].flags & GB_ALN_ABSENT)) aln[r].flags |= GB_ALN_PAIRED;
            return rcs;
        }
        if (fallback != 0) { g_last_error = gb::MIXED_FALLBACK_REFUSAL; return GB_ERR_ARG; }
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
                if ((rc = gb::grow_pools_for_rerun(d))) return rc;
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
    return gb::guarded("gb_map_batch", [&] {
        return map_batch_host(d, hp, false, n_reads, reads, quals, read_off, aln, mappings, mapping_pool_cap, edits, edit_pool_cap, status, n_mappings_used, n_edits_used);
    });
}

extern "C" int gb_map_paired_batch(gb_device* d, const gb_map_params* hp,
                                   uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                                   gb_alignment* aln, gb_mapping* mappings, uint64_t mapping_pool_cap, uint32_t* edits, uint64_t edit_pool_cap,
                                   uint8_t* status, uint64_t* n_mappings_used, uint64_t* n_edits_used) {
    return gb::guarded("gb_map_paired_batch", [&] {
        return map_batch_host(d, hp, true, n_reads, reads, quals, read_off, aln, mappings, mapping_pool_cap, edits, edit_pool_cap, status, n_mappings_used, n_edits_used);
    });
}

// Device-pointer entry: inputs already in HBM, outputs stay in HBM; asynchronous on the handle's stream.
extern "C" int gb_map_batch_device(gb_device* d, const gb_map_params* hp, int paired, uint32_t n_reads,
                                   const uint8_t* d_reads, const uint8_t* d_quals, const uint64_t* d_read_off, uint32_t max_read_len,
                                   gb_alignment* d_aln, gb_mapping* d_mappings, uint64_t mapping_pool_cap, uint32_t* d_edits, uint64_t edit_pool_cap,
                                   uint8_t* d_status, uint64_t* d_totals) {
    return gb::guarded("gb_map_batch_device", [&] {
        if (!d || !hp || !d_reads || !d_read_off || !d_aln || !d_mappings || !d_edits || !d_status || !d_totals) return GB_ERR_ARG;
        if (n_reads == 0) return GB_OK;
        GB_CUDA(cudaSetDevice(d->device));
        return map_device(d, hp, n_reads, d_reads, d_quals, d_read_off, max_read_len, (uint64_t)n_reads * max_read_len, d_aln, d_status, paired != 0,
                          d_mappings, mapping_pool_cap, d_edits, edit_pool_cap, nullptr, 0, d_totals, nullptr);
    });
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
    GB_CUDA(cudaMemcpy(&flag, &d->p_cursors.ptr->pool_overflow, sizeof flag, cudaMemcpyDeviceToHost));
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
    return gb::guarded("gb_debug_seed_stage", [&] {
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
        MapCursors cursors;
        for (int attempt = 0;; attempt++) {
            d->dbg_clusters = d_dbg.ptr; d->debug_stop_after_seed = true;
            rc = map_device(d, hp, n_reads, d_reads.ptr, quals ? d_quals.ptr : nullptr, d_off.ptr, max_len, total, d_aln.ptr, d_status.ptr, paired != 0,
                            nullptr, 0, nullptr, 0, nullptr, 0, d_totals.ptr, nullptr);
            d->dbg_clusters = nullptr; d->debug_stop_after_seed = false;
            if (rc) return rc;
            GB_CUDA(cudaStreamSynchronize(d->stream));
            GB_CUDA(cudaMemcpy(&cursors, d->p_cursors.ptr, sizeof cursors, cudaMemcpyDeviceToHost));
            if (!cursors.pool_overflow) break;
            if (attempt >= 10) { g_last_error = "seed stage: pools overflow"; return GB_ERR_CAPACITY; }
            d->pool_scale *= 2.0; d->pool_reruns++;
        }
        GB_CUDA(cudaMemcpy(st.data(), d->p_states.ptr, sizeof(ReadState) * n_reads, cudaMemcpyDeviceToHost));
        std::vector<DevMinimizer> hm(cursors.min_cursor); std::vector<DevSeed> hs(cursors.seed_cursor); std::vector<DevItem> hi(cursors.item_cursor);
        std::vector<gb_seed> he(cursors.ext_cursor);
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
    });
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
