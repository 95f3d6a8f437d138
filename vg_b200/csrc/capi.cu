// capi.cu — C-ABI entry points of libgiraffe_b200.so (see include/giraffe_b200.h) and the
// kernels' launch wrappers.  There is no CPU fallback anywhere in this file: without a
// CUDA device every compute entry point returns GB_ERR_NO_DEVICE.
#include <cstdlib>
#include <cstdio>
#include <algorithm>
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "extend.cuh"

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace gb {

int fail_cuda(cudaError_t e, const char* what) {
    set_last_error(what, ": ", cudaGetErrorString(e));
    return (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) ? GB_ERR_NO_DEVICE : GB_ERR_CUDA;
}

// ---------------------------------------------------------------------------------------
// extend kernel: persistent warps pulling work items from a global counter
// ---------------------------------------------------------------------------------------
struct ExtendBatch {
    const uint8_t* reads; const uint64_t* read_off;
    const uint32_t* item_read;
    const gb_seed* seeds; const uint64_t* seed_off;
    uint32_t n_items;
    uint32_t* ext_count; uint8_t* status;
    gb_extension* ext; uint32_t* path_pool; uint32_t* mism_pool;
    uint32_t read_cap;          // bytes of shared memory per warp for the masked read
    uint32_t* work_counter;
    // device-produced work list (mapping pipeline): when `items` is set, item i is
    // items[i] and the item count is read from *n_items_dev (capped by n_items).
    const DevItem* items; const uint32_t* n_items_dev;
    // clusters with more seeds than the per-item output strides hold (repeats): the first launch lists them, a second
    // launch redoes them with large strides; item i of that launch is in_list[i], its outputs live in slot i of the large
    // pools and big_of[item] = i tells the align stage where (ExtView)
    uint32_t* retry_list; uint32_t* retry_count; uint32_t retry_cap;
    const uint32_t* in_list; const uint32_t* in_count; uint32_t* big_of;
    // items extend_kernel leaves for extend_finish_kernel (anything but one exact full-length extension)
    uint32_t* post_list; uint32_t* post_count; uint32_t* post_work;
};

// Four resident blocks per SM (a 64-register budget).  Measured on an H100 (DESIGN.md §5): 3 blocks 7.2 ms, 4 blocks 7.0 ms,
// 5 blocks 11.8 ms.
__global__ void __launch_bounds__(EXTEND_WARPS * 32, 4)
extend_kernel(DevIndex ix, ExtendParams p, ExtendBatch b, ExtendWorkspace ws) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp_in_block = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const uint32_t gwarp = blockIdx.x * EXTEND_WARPS + warp_in_block;
    uint8_t* sread = smem + (size_t)warp_in_block * b.read_cap;
    QEntry* queue = ws.queue + (size_t)gwarp * ws.q_cap;
    ArenaNode* arena = ws.arena + (size_t)gwarp * ws.a_cap;

    const uint32_t n_items = b.in_list ? min(*b.in_count, b.retry_cap) : (b.items ? min(b.n_items, *b.n_items_dev) : b.n_items);
    while (true) {
        uint32_t item = 0;
        if (lane == 0) item = atomicAdd(b.work_counter, 1u);
        item = __shfl_sync(FULL, item, 0);
        if (item >= n_items) break;
        const uint32_t out_slot = item;                       // where this item's outputs go
        if (b.in_list) item = b.in_list[item];

        uint32_t r; uint64_t sb; uint32_t n_seeds;
        if (b.items) { const DevItem it = b.items[item]; r = it.read; sb = it.seed_off; n_seeds = it.seed_cnt; }
        else { r = b.item_read[item]; sb = b.seed_off[item]; n_seeds = (uint32_t)(b.seed_off[item + 1] - sb); }
        const uint64_t rb = b.read_off[r];
        const uint32_t read_len = (uint32_t)(b.read_off[r + 1] - rb);
        uint32_t status = GB_ITEM_OK, n = 0;
        if (read_len > b.read_cap) {
            status = GB_ITEM_OUT_FULL;
        } else {
            // stage + mask the read (ReadMasker: anything but ACGT becomes 'X')
            for (uint32_t i = lane; i < read_len; i += 32) {
                uint8_t c = b.reads[rb + i];
                if (c != 'A' && c != 'C' && c != 'G' && c != 'T') c = 'X';
                sread[i] = c;
            }
            __syncwarp();
            n = extend_search(ix, p, sread, read_len, b.seeds + sb, n_seeds,
                              queue, ws.q_cap, arena, ws.a_cap,
                              b.ext + (size_t)out_slot * p.max_ext,
                              b.path_pool + (size_t)out_slot * p.path_cap, &status);
        }
        // everything but a single exact full-length extension goes on to extend_finish_kernel
        const bool unfinished = status == GB_ITEM_OK && !extend_result_is_final(b.ext + (size_t)out_slot * p.max_ext, n);
        if (lane == 0) {
            if (status == GB_ITEM_OUT_FULL && b.retry_list && read_len <= b.read_cap) {
                const uint32_t pos = atomicAdd(b.retry_count, 1u);
                if (pos < b.retry_cap) b.retry_list[pos] = item;
            }
            if (b.big_of) b.big_of[item] = out_slot;
            b.ext_count[item] = n; b.status[item] = (uint8_t)status;
            if (unfinished) b.post_list[atomicAdd(b.post_count, 1u)] = item;
        }
        __syncwarp();
    }
}

// Second half of GaplessExtender::extend (extend.cuh: extend_finish) for the items extend_kernel listed.
__global__ void __launch_bounds__(EXTEND_WARPS * 32)
extend_finish_kernel(DevIndex ix, ExtendParams p, ExtendBatch b) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp_in_block = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    uint8_t* sread = smem + (size_t)warp_in_block * b.read_cap;
    const uint32_t n_listed = *b.post_count;
    while (true) {
        uint32_t i = 0;
        if (lane == 0) i = atomicAdd(b.post_work, 1u);
        i = __shfl_sync(FULL, i, 0);
        if (i >= n_listed) break;
        const uint32_t item = b.post_list[i];
        const uint32_t out_slot = b.in_list ? b.big_of[item] : item;
        const uint32_t r = b.items ? b.items[item].read : b.item_read[item];
        const uint64_t rb = b.read_off[r];
        const uint32_t read_len = (uint32_t)(b.read_off[r + 1] - rb);
        for (uint32_t k = lane; k < read_len; k += 32) {
            uint8_t c = b.reads[rb + k];
            if (c != 'A' && c != 'C' && c != 'G' && c != 'T') c = 'X';
            sread[k] = c;
        }
        __syncwarp();
        uint32_t status = GB_ITEM_OK;
        const uint32_t n = extend_finish(ix, p, sread, b.ext + (size_t)out_slot * p.max_ext, b.ext_count[item],
                                         b.path_pool + (size_t)out_slot * p.path_cap, b.mism_pool + (size_t)out_slot * p.mism_cap, &status);
        if (lane == 0) {
            if (status == GB_ITEM_OUT_FULL && b.retry_list) {
                const uint32_t pos = atomicAdd(b.retry_count, 1u);
                if (pos < b.retry_cap) b.retry_list[pos] = item;
            }
            b.ext_count[item] = n; b.status[item] = (uint8_t)status;
        }
        __syncwarp();
    }
}

} // namespace gb

using namespace gb;

extern "C" const char* gb_last_error(void) { return g_last_error.c_str(); }

extern "C" int gb_device_create(const gb_flat_index* ix, int device_ordinal, gb_device** out) {
    return gb::guarded("gb_device_create", [&] {
        if (!ix || !out) return GB_ERR_ARG;
        int ndev = 0;
        cudaError_t e = cudaGetDeviceCount(&ndev);
        if (e != cudaSuccess || ndev == 0) {
            g_last_error = "no CUDA device available (libgiraffe_b200 has no CPU fallback)";
            return GB_ERR_NO_DEVICE;
        }
        if (device_ordinal < 0 || device_ordinal >= ndev) return GB_ERR_ARG;
        if ((ix->table_cells & (ix->table_cells - 1)) != 0) return GB_ERR_FORMAT;
        GB_CUDA(cudaSetDevice(device_ordinal));
        auto* d = new gb_device();
        d->device = device_ordinal;
        cudaDeviceProp prop;
        GB_CUDA(cudaGetDeviceProperties(&prop, device_ordinal));
        d->n_sms = prop.multiProcessorCount;
        if (const char* env = std::getenv("GIRAFFE_B200_MAP_CHUNK")) {
            const unsigned long v = std::strtoul(env, nullptr, 10);
            if (v >= 2 && v <= (1ul << 24)) d->map_chunk = (uint32_t)(v & ~1ul);
        }
        if (const char* env = std::getenv("GIRAFFE_B200_TILES")) d->use_tiles = std::atoi(env) != 0;
        if (const char* env = std::getenv("GIRAFFE_B200_POOL_SCALE")) {
            const double v = std::strtod(env, nullptr);
            if (v > 0.0 && v <= 1024.0) d->pool_scale = v;
        }
        if (const char* env = std::getenv("GIRAFFE_B200_SEED_TABLES")) {
            unsigned mc = 0, cc = 0, ns = 64;
            if (std::sscanf(env, "%u,%u,%u", &mc, &cc, &ns) >= 2 && mc >= 2 && cc >= 1) {
                d->seed_mc = std::max<uint32_t>(16u, std::min<uint32_t>(gb::MAX_MINIMIZERS, (mc + 7u) & ~7u));
                d->seed_cc = std::min<uint32_t>(64u, cc);
                d->seed_ns = std::min<uint32_t>(64u, ns);
            }
        }
        GB_CUDA(cudaStreamCreateWithFlags(&d->own_stream, cudaStreamNonBlocking));
        d->stream = d->own_stream;
        for (int i = 0; i < 5; i++) GB_CUDA(cudaEventCreate(&d->ev_stage[i]));
        GB_CUDA(cudaEventCreate(&d->ev0)); GB_CUDA(cudaEventCreate(&d->ev1));
        GB_CUDA(cudaStreamCreateWithFlags(&d->s_in, cudaStreamNonBlocking));
        GB_CUDA(cudaStreamCreateWithFlags(&d->s_out, cudaStreamNonBlocking));
        for (int i = 0; i < 2; i++) {
            GB_CUDA(cudaEventCreateWithFlags(&d->io[i].ev_in, cudaEventDisableTiming));
            GB_CUDA(cudaEventCreateWithFlags(&d->io[i].ev_done, cudaEventDisableTiming));
            GB_CUDA(cudaEventCreateWithFlags(&d->io[i].ev_hdr, cudaEventDisableTiming));
            GB_CUDA(cudaEventCreateWithFlags(&d->io[i].ev_out, cudaEventDisableTiming));
            GB_CUDA(cudaEventCreate(&d->io[i].ev_k0)); GB_CUDA(cudaEventCreate(&d->io[i].ev_k1));
        }
        GB_CUDA(cudaMallocHost(&d->h_totals, 6 * sizeof(uint64_t)));
        int rc;
        if ((rc = d->nodes.upload(ix->nodes, ix->n_nodes, d->stream))) return rc;
        if ((rc = d->seq.upload(ix->seq, ix->seq_bytes, d->stream))) return rc;
        if ((rc = d->gbwt.upload(ix->gbwt, ix->gbwt_words, d->stream))) return rc;
        if ((rc = d->dist.upload(ix->dist, ix->n_nodes / 2, d->stream))) return rc;
        if ((rc = d->table.upload(ix->table, ix->table_cells, d->stream))) return rc;
        if ((rc = d->hits.upload(ix->hits, ix->n_hits ? ix->n_hits : 1, d->stream, ix->n_hits))) return rc;
        GB_CUDA(cudaStreamSynchronize(d->stream));
        {
            // ids in chain order (the rescue subgraph is cut from it, minimizer_mapper.cpp:3364)
            std::vector<uint32_t> order;
            for (uint32_t id = 1; id < ix->n_nodes / 2; id++) if (ix->nodes[2 * id].len > 0) order.push_back(id);
            std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
                const gb_dist_payload& pa = ix->dist[a]; const gb_dist_payload& pb = ix->dist[b];
                if (pa.component != pb.component) return pa.component < pb.component;
                if (pa.slot != pb.slot) return pa.slot < pb.slot;
                if (pa.allele != pb.allele) return pa.allele < pb.allele;      // place inside the site = topological
                return a < b;
            });
            if ((rc = d->slot_order.upload(order.data(), order.size() ? order.size() : 1, d->stream, order.size()))) return rc;
            GB_CUDA(cudaStreamSynchronize(d->stream));
            d->ix.slot_order = d->slot_order.ptr; d->ix.n_ids = (uint32_t)order.size();
        }
        if (ix->n_slots) {
            if ((rc = d->slots.upload(ix->slots, ix->n_slots, d->stream))) return rc;
            if ((rc = d->site_dist.upload(ix->site_dist, ix->site_dist_len ? ix->site_dist_len : 1, d->stream, ix->site_dist_len))) return rc;
            GB_CUDA(cudaStreamSynchronize(d->stream));
        }
        d->ix.slots = ix->n_slots ? d->slots.ptr : nullptr; d->ix.n_slots = (uint32_t)ix->n_slots; d->ix.site_dist = ix->n_slots ? d->site_dist.ptr : nullptr;
        d->h_node_len.resize(ix->n_nodes);
        for (uint32_t v = 0; v < ix->n_nodes; v++) d->h_node_len[v] = ix->nodes[v].len;
        // c_in = x_in + offset and c_out = x_out - (length - offset) are int32 in the seeding kernels.  A derived payload
        // always fits (x_in + length is at most the graph's sequence, below 2^31 by the 32-bit seq_off); a hand-made one may not.
        for (uint32_t id = 1; id < ix->n_nodes / 2; id++) {
            const uint32_t len = ix->nodes[2 * id].len;
            if (len == 0) continue;
            const gb_dist_payload& p = ix->dist[id];
            if ((uint64_t)p.x_in + len > (uint64_t)INT32_MAX || (int64_t)(int32_t)p.x_out - len < (int64_t)INT32_MIN) { d->chain_coords_fit = false; break; }
        }
        d->ix.nodes = d->nodes.ptr; d->ix.seq = d->seq.ptr; d->ix.gbwt = d->gbwt.ptr; d->ix.dist = d->dist.ptr;
        d->ix.table = d->table.ptr; d->ix.hits = d->hits.ptr;
        d->ix.table_mask = ix->table_cells - 1; d->ix.n_nodes = ix->n_nodes; d->ix.k = ix->k; d->ix.w = ix->w;
        d->sc = DevScores{1, 4, 6, 1, 5};
        GB_CUDA(cudaMalloc(&d->work_counter, 64));
        *out = d;
        return GB_OK;
    });
}

extern "C" void gb_device_destroy(gb_device* d) {
    if (!d) return;
    cudaSetDevice(d->device);
    cudaStreamSynchronize(d->stream);
    for (int i = 0; i < 5; i++) cudaEventDestroy(d->ev_stage[i]);
    cudaFree(d->work_counter);
    cudaEventDestroy(d->ev0); cudaEventDestroy(d->ev1);
    for (int i = 0; i < 2; i++) {
        cudaEventDestroy(d->io[i].ev_in); cudaEventDestroy(d->io[i].ev_done); cudaEventDestroy(d->io[i].ev_hdr);
        cudaEventDestroy(d->io[i].ev_out); cudaEventDestroy(d->io[i].ev_k0); cudaEventDestroy(d->io[i].ev_k1);
    }
    for (cudaEvent_t ev : d->kt_ev) if (ev) cudaEventDestroy(ev);
    cudaFreeHost(d->h_totals);
    cudaStreamDestroy(d->s_in); cudaStreamDestroy(d->s_out);
    cudaStreamDestroy(d->own_stream);
    delete d;                              // the DevBuf destructors free the device memory
}

extern "C" int gb_set_scores(gb_device* d, const gb_scores* s) {
    if (!d || !s) return GB_ERR_ARG;
    d->sc = DevScores{s->match, s->mismatch, s->gap_open, s->gap_extend, s->full_length_bonus};
    return GB_OK;
}

extern "C" float gb_last_kernel_ms(const gb_device* d) { return d ? d->last_kernel_ms : 0.f; }
extern "C" uint64_t gb_launch_count(const gb_device* d) { return d ? d->launches : 0; }

namespace gb {

// Device-resident launch used by both the host-buffer entry point and the mapping pipeline.
int launch_extend(gb_device* d, const ExtendParams& p, const ExtendBatch& b_in, uint32_t max_read_len, bool mark = false) {
    ExtendBatch b = b_in;
    b.read_cap = (max_read_len + 15u) & ~15u;
    if (b.read_cap == 0) b.read_cap = 16;
    const size_t smem = (size_t)EXTEND_WARPS * b.read_cap;
    if (smem > 200 * 1024) { g_last_error = "read too long for the extension kernel"; return GB_ERR_ARG; }
    if (smem > 48 * 1024) {
        GB_CUDA(cudaFuncSetAttribute(extend_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        GB_CUDA(cudaFuncSetAttribute(extend_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    int blocks_per_sm = 0;
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, extend_kernel, EXTEND_WARPS * 32, smem));
    if (blocks_per_sm < 1) blocks_per_sm = 1;
    uint32_t grid = (uint32_t)(d->n_sms * blocks_per_sm);
    const uint32_t needed = (b.n_items + EXTEND_WARPS - 1) / EXTEND_WARPS;
    if (grid > needed) grid = needed ? needed : 1;
    const size_t n_warps = (size_t)grid * EXTEND_WARPS;
    int rc;
    if ((rc = d->ws_queue.reserve(n_warps * EXTEND_Q_CAP))) return rc;
    if ((rc = d->ws_arena.reserve(n_warps * EXTEND_A_CAP))) return rc;
    if ((rc = d->p_post.reserve(b.n_items ? b.n_items : 1))) return rc;
    ExtendWorkspace ws{d->ws_queue.ptr, d->ws_arena.ptr, EXTEND_Q_CAP, EXTEND_A_CAP};
    b.work_counter = d->work_counter; b.post_list = d->p_post.ptr; b.post_count = d->work_counter + 1; b.post_work = d->work_counter + 2;
    GB_CUDA(cudaMemsetAsync(d->work_counter, 0, 4 * sizeof(uint32_t), d->stream));
    extend_kernel<<<grid, EXTEND_WARPS * 32, smem, d->stream>>>(d->ix, p, b, ws);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    if (mark && (rc = d->kt_mark(b.in_list ? "extend_kernel(large strides)" : "extend_kernel"))) return rc;
    // post-processing of the items the search left unfinished (its own kernel: the search loop stays instruction-cache resident)
    int fin_blocks = 0;
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fin_blocks, extend_finish_kernel, EXTEND_WARPS * 32, smem));
    if (fin_blocks < 1) fin_blocks = 1;
    uint32_t fgrid = (uint32_t)(d->n_sms * fin_blocks);
    if (fgrid > needed) fgrid = needed ? needed : 1;
    extend_finish_kernel<<<fgrid, EXTEND_WARPS * 32, smem, d->stream>>>(d->ix, p, b);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    if (mark && (rc = d->kt_mark(b.in_list ? "extend_finish_kernel(large strides)" : "extend_finish_kernel"))) return rc;
    return GB_OK;
}

int launch_extend_device(gb_device* d, const ExtendParams& p, const uint8_t* reads, const uint64_t* read_off,
                         const uint32_t* item_read, const gb_seed* seeds, const uint64_t* seed_off,
                         const DevItem* items, const uint32_t* n_items_dev, uint32_t n_items_max,
                         uint32_t* ext_count, uint8_t* status, gb_extension* ext, uint32_t* path_pool, uint32_t* mism_pool,
                         uint32_t max_read_len, const ExtendBig* big) {
    const bool mark = big != nullptr;          // the mapping pipeline times its kernels
    ExtendBatch b{};
    b.reads = reads; b.read_off = read_off; b.item_read = item_read; b.seeds = seeds; b.seed_off = seed_off;
    b.n_items = n_items_max; b.items = items; b.n_items_dev = n_items_dev;
    b.ext_count = ext_count; b.status = status; b.ext = ext; b.path_pool = path_pool; b.mism_pool = mism_pool;
    if (big) { b.retry_list = big->list; b.retry_count = big->count; b.retry_cap = big->cap; }
    int rc = launch_extend(d, p, b, max_read_len, mark);
    if (rc || !big) return rc;
    // second launch: the listed items with the large strides
    ExtendParams pb = p; pb.max_ext = big->max_ext; pb.path_cap = big->path_cap; pb.mism_cap = big->mism_cap;
    ExtendBatch b2 = b;
    b2.retry_list = nullptr; b2.retry_count = nullptr; b2.in_list = big->list; b2.in_count = big->count; b2.retry_cap = big->cap; b2.big_of = big->big_of;
    b2.ext = big->ext; b2.path_pool = big->path; b2.mism_pool = big->mism;
    return launch_extend(d, pb, b2, max_read_len, mark);
}

} // namespace gb

extern "C" int gb_extend_batch(gb_device* d, const gb_extend_params* hp,
                               uint32_t n_reads, const uint8_t* reads, const uint64_t* read_off,
                               uint32_t n_items, const uint32_t* item_read,
                               const gb_seed* seeds, const uint64_t* seed_off,
                               uint32_t* ext_count, uint8_t* status,
                               gb_extension* ext, uint32_t* path_pool, uint32_t* mism_pool) {
    return gb::guarded("gb_extend_batch", [&] {
        if (!d || !hp || !reads || !read_off || !item_read || !seeds || !seed_off || !ext_count || !status || !ext ||
            !path_pool || !mism_pool) return GB_ERR_ARG;
        if (hp->max_ext_per_item == 0 || hp->path_cap_per_item == 0 || hp->mism_cap_per_item == 0) return GB_ERR_ARG;
        if (n_items == 0) return GB_OK;
        GB_CUDA(cudaSetDevice(d->device));
        uint32_t max_len = 0;
        for (uint32_t r = 0; r < n_reads; r++) max_len = std::max<uint32_t>(max_len, (uint32_t)(read_off[r + 1] - read_off[r]));
        for (uint32_t i = 0; i < n_items; i++) if (item_read[i] >= n_reads) return GB_ERR_ARG;
        const uint64_t n_seeds = seed_off[n_items];

        DevBuf<uint8_t> d_reads; DevBuf<uint64_t> d_read_off, d_seed_off; DevBuf<uint32_t> d_item_read; DevBuf<gb_seed> d_seeds;
        DevBuf<uint32_t> d_cnt, d_path, d_mism; DevBuf<uint8_t> d_status; DevBuf<gb_extension> d_ext;
        int rc;
        if ((rc = d_reads.upload(reads, read_off[n_reads] ? read_off[n_reads] : 1, d->stream, read_off[n_reads]))) return rc;
        if ((rc = d_read_off.upload(read_off, n_reads + 1, d->stream))) return rc;
        if ((rc = d_item_read.upload(item_read, n_items, d->stream))) return rc;
        if ((rc = d_seeds.upload(seeds, n_seeds ? n_seeds : 1, d->stream, n_seeds))) return rc;
        if ((rc = d_seed_off.upload(seed_off, n_items + 1, d->stream))) return rc;
        if ((rc = d_cnt.reserve(n_items))) return rc;
        if ((rc = d_status.reserve(n_items))) return rc;
        if ((rc = d_ext.reserve((size_t)n_items * hp->max_ext_per_item))) return rc;
        if ((rc = d_path.reserve((size_t)n_items * hp->path_cap_per_item))) return rc;
        if ((rc = d_mism.reserve((size_t)n_items * hp->mism_cap_per_item))) return rc;

        ExtendParams p;
        p.sc = d->sc; p.max_mismatches = hp->max_mismatches; p.overlap_threshold = hp->overlap_threshold;
        p.overlap_threshold_unused = 0.f; p.trim = hp->trim;
        p.max_ext = hp->max_ext_per_item; p.path_cap = hp->path_cap_per_item; p.mism_cap = hp->mism_cap_per_item;
        ExtendBatch b{};
        b.reads = d_reads.ptr; b.read_off = d_read_off.ptr; b.item_read = d_item_read.ptr;
        b.seeds = d_seeds.ptr; b.seed_off = d_seed_off.ptr; b.n_items = n_items;
        b.ext_count = d_cnt.ptr; b.status = d_status.ptr; b.ext = d_ext.ptr; b.path_pool = d_path.ptr; b.mism_pool = d_mism.ptr;

        GB_CUDA(cudaEventRecord(d->ev0, d->stream));
        if ((rc = launch_extend(d, p, b, max_len))) return rc;
        GB_CUDA(cudaEventRecord(d->ev1, d->stream));

        GB_CUDA(cudaMemcpyAsync(ext_count, d_cnt.ptr, sizeof(uint32_t) * n_items, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(status, d_status.ptr, n_items, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(ext, d_ext.ptr, sizeof(gb_extension) * (size_t)n_items * hp->max_ext_per_item, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(path_pool, d_path.ptr, sizeof(uint32_t) * (size_t)n_items * hp->path_cap_per_item, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(mism_pool, d_mism.ptr, sizeof(uint32_t) * (size_t)n_items * hp->mism_cap_per_item, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaStreamSynchronize(d->stream));
        GB_CUDA(cudaEventElapsedTime(&d->last_kernel_ms, d->ev0, d->ev1));
        // make pool offsets absolute
        for (uint32_t i = 0; i < n_items; i++) {
            for (uint32_t j = 0; j < ext_count[i]; j++) {
                gb_extension& e = ext[(size_t)i * hp->max_ext_per_item + j];
                e.path_off += i * hp->path_cap_per_item;
                e.mism_off += i * hp->mism_cap_per_item;
            }
        }
        return GB_OK;
    });
}
