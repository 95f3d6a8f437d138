// paired_job_device.cu — gb_map_paired_job_device: the paired job of paired_job.cu (fragment-length training, map_paired
// with the learned distribution, the ambiguous-pair buffer) for reads that are already in HBM.
//   pair_stats_kernel       thread per pair: single-end fallback count and the longest read of every sub-batch
//   train_classify_kernel   thread per pair: the training rule of map_paired (minimizer_mapper.cpp:1316-1336)
//   train_cut_kernel        thread per pair: which pairs a window consumes, their routes, the lengths to register, the buffer
//   gather_pairs_kernel     warp per read: a sub-batch's pairs as contiguous, zero-based reads and qualities
//   record_append_kernel    warp per record: a sub-batch's records into the caller's pools at the running totals
// Every mapping pass is map_device.  The distribution stays on the host: each training window copies back its cut and the
// lengths to register, and every sub-batch its totals, so the job synchronises a few times per window and per sub-batch.
#include <cub/cub.cuh>
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "fragment_distribution.h"

#include <algorithm>
#include <chrono>
#include <vector>

using gb::g_last_error;

namespace gb {

// The pairs a pass works on: list[i] when there is a list (the buffered pairs), first + i otherwise.
struct PairSet {
    const uint32_t* list; uint32_t first;
    __host__ __device__ uint32_t pair(uint32_t i) const { return list ? list[i] : first + i; }
    PairSet from(uint32_t i) const { return PairSet{list ? list + i : nullptr, first + i}; }
};

// Length of read i of a set (reads 2i and 2i + 1 are the mates of its pair i) in the caller's offsets; 0 for i >= n, so that
// an exclusive scan over n + 1 items ends with the total.
struct SetReadLen {
    const uint64_t* off; PairSet s; uint32_t n;
    __host__ __device__ uint64_t operator()(uint32_t i) const {
        if (i >= n) return 0;
        const uint64_t r = 2 * (uint64_t)s.pair(i >> 1) + (i & 1u);
        return off[r + 1] - off[r];
    }
};

// Mappings (edits when `edits`) of record i of a sub-batch when its pair is kept (keep == nullptr: every pair); 0 for i >= n.
struct KeptCount {
    const gb_alignment* aln; const uint32_t* keep; uint32_t n; bool edits;
    __host__ __device__ uint64_t operator()(uint32_t i) const {
        if (i >= n || (keep && !keep[i >> 1])) return 0;
        return edits ? aln[i].n_edits : aln[i].n_mappings;
    }
};

// stats[0] = pairs whose read 1 fails the paired distance limit (the single-end fallback of map_paired,
// minimizer_mapper.cpp:1469-1471, decided per pair as map_batch_host does); stats[1 + c] = longest read of sub-batch c.
__global__ void pair_stats_kernel(PairSet s, uint32_t n_pairs, uint32_t chunk_pairs, const uint64_t* off, int64_t fragment_limit,
                                  int64_t distance_limit, unsigned long long* stats) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pairs; i += gridDim.x * blockDim.x) {
        const uint64_t r = 2 * (uint64_t)s.pair(i);
        const uint64_t L1 = off[r + 1] - off[r], L2 = off[r + 2] - off[r + 1];
        if (fragment_limit < max(distance_limit, (int64_t)L1 + 50)) atomicAdd(stats, 1ull);
        atomicMax(stats + 1 + i / chunk_pairs, (unsigned long long)max(L1, L2));
    }
}

// The training rule, per pair of a window mapped single-ended (paired_job.cu restates it on the host): both ends mapped
// with status OK, MAPQ 60 and score >= 0.85 * match * length, and the distance from the first mapping of read 1 to the
// flipped first mapping of read 2 below max_fragment_length.  Unreachable is -1 (size_t max stored into an int64_t,
// minimizer_mapper.cpp:3879-3884), which passes that test and is registered, as the reference does.
__global__ void train_classify_kernel(DevIndex ix, uint32_t n_pairs, const gb_alignment* aln, const uint8_t* status, const gb_mapping* maps,
                                      const uint64_t* read_off, int match, int64_t max_fragment_length, uint32_t* elig, int64_t* len) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pairs; i += gridDim.x * blockDim.x) {
        bool both_perfect_unique = true;
#pragma unroll
        for (uint32_t r = 0; r < 2; r++) {
            const gb_alignment a = aln[2 * i + r];
            const int64_t L = (int64_t)(read_off[2 * i + r + 1] - read_off[2 * i + r]);
            const double max_score_aln = (double)(match * L);
            both_perfect_unique = both_perfect_unique && status[2 * i + r] == GB_ITEM_OK && (a.flags & GB_ALN_MAPPED) && a.mapq == 60 &&
                                  (double)a.score >= max_score_aln * 0.85;
        }
        uint32_t keep = 0; int64_t dist = 0;
        if (both_perfect_unique) {
            const gb_mapping first1 = maps[aln[2 * i].mapping_off], first2 = maps[aln[2 * i + 1].mapping_off];
            dist = oriented_distance(ix, first1.node, first1.offset, first2.node ^ 1u, load_node(ix, first2.node).len - (uint32_t)first2.offset);
            keep = !(dist == INT64_MAX || dist >= max_fragment_length);
        }
        elig[i] = keep; len[i] = dist;
    }
}

// incl = inclusive scan of elig.  A pair is consumed while fewer than `budget` eligible pairs precede it: the pair that
// brings the sample to maximum_sample_size finalizes the distribution and the pairs behind it are left for the paired pass.
// out[0] = pairs consumed, out[1] = eligible pairs consumed, out[2 ...] = their lengths in pair order.  Consumed pairs
// that are not eligible are appended to the buffer (after the n_buffered already there) in pair order.
__global__ void train_cut_kernel(uint32_t n_pairs, uint32_t first_pair, const uint32_t* elig, const uint32_t* incl, const int64_t* len,
                                 uint64_t budget, uint32_t* keep, uint32_t* buffered, uint32_t n_buffered, uint8_t* pair_route, int64_t* out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pairs; i += gridDim.x * blockDim.x) {
        const uint64_t before = incl[i] - elig[i];
        const bool consumed = before < budget;
        keep[i] = consumed && elig[i];
        if (consumed) {
            if (elig[i]) out[2 + before] = len[i];
            else buffered[n_buffered + i - before] = first_pair + i;
            if (pair_route) pair_route[first_pair + i] = elig[i] ? GB_PAIR_TRAINING : GB_PAIR_BUFFERED;
        }
        if (elig[i] && incl[i] == budget) out[0] = i + 1;
        if (i == n_pairs - 1) {
            if (incl[i] < budget) out[0] = n_pairs;
            out[1] = (int64_t)min((uint64_t)incl[i], budget);
        }
    }
}

// Read i of the set to dst_reads + dst_off[i] (dst_off: exclusive scan of the set's read lengths).
__global__ void gather_pairs_kernel(PairSet s, uint32_t n_reads, const uint64_t* off, const uint8_t* reads, const uint8_t* quals,
                                    const uint64_t* dst_off, uint8_t* dst_reads, uint8_t* dst_quals) {
    const uint32_t warps_per_block = blockDim.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t i = blockIdx.x * warps_per_block + (threadIdx.x >> 5); i < n_reads; i += gridDim.x * warps_per_block) {
        const uint64_t r = 2 * (uint64_t)s.pair(i >> 1) + (i & 1u);
        const uint64_t src = off[r], L = off[r + 1] - src, dst = dst_off[i];
        for (uint64_t k = lane; k < L; k += 32) {
            dst_reads[dst + k] = reads[src + k];
            if (quals) dst_quals[dst + k] = quals[src + k];
        }
    }
}

// Record i of a sub-batch (pair i / 2 of the set, mate i % 2) whose pair is kept goes to read 2 * pair + mate of the caller's
// outputs, its mappings and edits to map_base + map_off[i] / edit_base + edit_off[i] (exclusive scans of the kept counts).
__global__ void record_append_kernel(PairSet s, uint32_t n_reads, const uint32_t* keep, const gb_alignment* aln, const uint8_t* status,
                                     const gb_mapping* maps, const uint32_t* edits, const uint64_t* map_off, const uint64_t* edit_off,
                                     uint64_t map_base, uint64_t edit_base, uint8_t extra_flags,
                                     gb_alignment* out_aln, uint8_t* out_status, gb_mapping* out_maps, uint32_t* out_edits) {
    const uint32_t warps_per_block = blockDim.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t i = blockIdx.x * warps_per_block + (threadIdx.x >> 5); i < n_reads; i += gridDim.x * warps_per_block) {
        if (keep && !keep[i >> 1]) continue;
        gb_alignment a = aln[i];
        const uint64_t mo = map_base + map_off[i], eo = edit_base + edit_off[i];
        for (uint32_t k = lane; k < a.n_mappings; k += 32) out_maps[mo + k] = maps[a.mapping_off + k];
        for (uint32_t k = lane; k < a.n_edits; k += 32) out_edits[eo + k] = edits[a.edit_off + k];
        if (lane == 0) {
            const uint32_t dst = 2 * s.pair(i >> 1) + (i & 1u);
            a.read_id = dst; a.mapping_off = (uint32_t)mo; a.edit_off = (uint32_t)eo; a.flags |= extra_flags;
            out_aln[dst] = a; out_status[dst] = status[i];
        }
    }
}

namespace {

// The caller's arguments and the job's running state.
struct Job {
    gb_device* d; const gb_map_params* hp;
    const uint8_t* reads; const uint8_t* quals; const uint64_t* read_off; uint32_t max_read_len;
    gb_alignment* aln; gb_mapping* maps; uint64_t map_cap; uint32_t* edits; uint64_t edit_cap; uint8_t* status; uint8_t* route;
    uint64_t nm = 0, ne = 0;                  // mappings / edits appended so far
};

uint32_t grid_for(const gb_device* d, uint64_t items, uint32_t per_block) {
    return (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((items + per_block - 1) / per_block, (uint64_t)d->n_sms * 8));
}

template <typename In, typename Out>
int exclusive_scan(gb_device* d, In in, Out out, uint32_t n) {
    size_t bytes = 0;
    GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int)n, d->stream));
    if (int rc = d->pj.scan_tmp.reserve(bytes)) return rc;
    GB_CUDA(cub::DeviceScan::ExclusiveSum(d->pj.scan_tmp.ptr, bytes, in, out, (int)n, d->stream));
    d->launches++;
    return GB_OK;
}

// Sub-batch buffers for n reads.  Reserved before anything is enqueued that reads them (a reserve may reallocate).
int reserve_sub(gb_device* d, const gb_map_params* hp, uint32_t n) {
    auto& w = d->pj;
    int rc;
    if ((rc = w.aln.reserve(n)) || (rc = w.status.reserve(n)) || (rc = w.maps.reserve((size_t)n * hp->mapping_cap_per_read)) ||
        (rc = w.edits.reserve((size_t)n * hp->edit_cap_per_read)) || (rc = w.totals.reserve(3)) || (rc = w.append_off.reserve(2 * ((size_t)n + 1))))
        return rc;
    return GB_OK;
}

// map_device into the sub-batch buffers, redone with doubled intermediate pools until it does not overflow them.
int map_sub(gb_device* d, const gb_map_params* P, uint32_t n, const uint8_t* reads, const uint8_t* quals, const uint64_t* off,
            uint32_t max_len, bool paired) {
    auto& w = d->pj;
    for (;;) {
        GB_CUDA(cudaMemsetAsync(w.totals.ptr, 0, 3 * sizeof(uint64_t), d->stream));
        if (int rc = map_device(d, P, n, reads, quals, off, max_len, (uint64_t)n * max_len, w.aln.ptr, w.status.ptr, paired,
                                w.maps.ptr, (uint64_t)n * P->mapping_cap_per_read, w.edits.ptr, (uint64_t)n * P->edit_cap_per_read,
                                nullptr, 0, w.totals.ptr, reinterpret_cast<uint32_t*>(w.totals.ptr + 2))) return rc;
        uint64_t overflow = 0;
        GB_CUDA(cudaMemcpyAsync(&overflow, w.totals.ptr + 2, sizeof overflow, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaStreamSynchronize(d->stream));
        if (!overflow) return GB_OK;
        if (int rc = grow_pools_for_rerun(d)) return rc;
    }
}

// The sub-batch's records of the kept pairs (keep == nullptr: all) into the caller's outputs at the running totals: sizes
// and a scan first, then the copy, so nothing is written past the caller's capacities.
int append(Job& J, PairSet s, uint32_t n, const uint32_t* keep, uint8_t extra_flags) {
    gb_device* d = J.d; auto& w = d->pj;
    uint64_t* map_off = w.append_off.ptr; uint64_t* edit_off = w.append_off.ptr + n + 1;
    cub::CountingInputIterator<uint32_t> counting(0);
    int rc;
    if ((rc = exclusive_scan(d, cub::TransformInputIterator<uint64_t, KeptCount, cub::CountingInputIterator<uint32_t>>(counting, KeptCount{w.aln.ptr, keep, n, false}), map_off, n + 1)) ||
        (rc = exclusive_scan(d, cub::TransformInputIterator<uint64_t, KeptCount, cub::CountingInputIterator<uint32_t>>(counting, KeptCount{w.aln.ptr, keep, n, true}), edit_off, n + 1)))
        return rc;
    uint64_t tm = 0, te = 0;
    GB_CUDA(cudaMemcpyAsync(&tm, map_off + n, sizeof tm, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(&te, edit_off + n, sizeof te, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));
    if (J.nm + tm > J.map_cap || J.ne + te > J.edit_cap) { g_last_error = "gb_map_paired_job_device: output pool too small"; return GB_ERR_CAPACITY; }
    record_append_kernel<<<grid_for(d, n, 8), 256, 0, d->stream>>>(s, n, keep, w.aln.ptr, w.status.ptr, w.maps.ptr, w.edits.ptr, map_off, edit_off,
                                                                  J.nm, J.ne, extra_flags, J.aln, J.status, J.maps, J.edits);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    J.nm += tm; J.ne += te;
    return GB_OK;
}

// pair_stats_kernel over n_pairs pairs of a set in sub-batches of chunk_pairs: {fallback count, longest read per sub-batch}.
int pair_stats(Job& J, PairSet s, uint32_t n_pairs, uint32_t chunk_pairs, int64_t fragment_limit, std::vector<uint64_t>& stats) {
    gb_device* d = J.d; auto& w = d->pj;
    const uint32_t n_chunks = (n_pairs + chunk_pairs - 1) / chunk_pairs;
    int rc;
    if ((rc = w.out.reserve(1 + (size_t)n_chunks))) return rc;
    GB_CUDA(cudaMemsetAsync(w.out.ptr, 0, sizeof(int64_t) * (1 + (size_t)n_chunks), d->stream));
    pair_stats_kernel<<<grid_for(d, n_pairs, 256), 256, 0, d->stream>>>(s, n_pairs, chunk_pairs, J.read_off, fragment_limit, (int64_t)J.hp->distance_limit,
                                                                       reinterpret_cast<unsigned long long*>(w.out.ptr));
    d->launches++;
    GB_CUDA(cudaGetLastError());
    stats.assign(1 + (size_t)n_chunks, 0);
    GB_CUDA(cudaMemcpyAsync(stats.data(), w.out.ptr, sizeof(uint64_t) * stats.size(), cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));
    for (uint32_t c = 0; c < n_chunks; c++)
        if (stats[1 + c] > J.max_read_len) { g_last_error = "gb_map_paired_job_device: a read is longer than max_read_len"; return GB_ERR_ARG; }
    return GB_OK;
}

// The pairs of a set mapped paired with the finalized distribution in P (or, when every pair fails the paired distance
// limit, single-ended and flagged GB_ALN_PAIRED, as gb_map_paired_batch does): gathered per sub-batch of at most
// map_chunk reads into contiguous, zero-based arrays (map_device's paired working copy is addressed by the offsets).
int map_pairs(Job& J, const gb_map_params* P, PairSet s, uint32_t n_pairs) {
    gb_device* d = J.d; auto& w = d->pj;
    const uint32_t chunk_pairs = d->map_chunk / 2;
    const int64_t fragment_limit = (int64_t)(P->fragment_mean + P->paired_distance_stdevs * P->fragment_stdev);
    std::vector<uint64_t> stats;
    int rc;
    if ((rc = pair_stats(J, s, n_pairs, chunk_pairs, fragment_limit, stats))) return rc;
    const bool single_end = stats[0] == n_pairs;
    if (stats[0] != 0 && !single_end) { g_last_error = "fragment distance limit below the read distance limit for some pairs only (mixed single-end fallback, minimizer_mapper.cpp:1471, is not supported in one batch)"; return GB_ERR_ARG; }
    for (uint32_t c = 0; c * chunk_pairs < n_pairs; c++) {
        const uint32_t cpn = std::min(chunk_pairs, n_pairs - c * chunk_pairs), cn = 2 * cpn;
        const uint32_t max_len = (uint32_t)stats[1 + c];
        const PairSet sub = s.from(c * chunk_pairs);
        if ((rc = reserve_sub(d, P, cn)) || (rc = w.off.reserve((size_t)cn + 1)) || (rc = w.reads.reserve((size_t)cn * max_len + 16)) ||
            (J.quals && (rc = w.quals.reserve((size_t)cn * max_len + 16)))) return rc;
        cub::CountingInputIterator<uint32_t> counting(0);
        if ((rc = exclusive_scan(d, cub::TransformInputIterator<uint64_t, SetReadLen, cub::CountingInputIterator<uint32_t>>(counting, SetReadLen{J.read_off, sub, cn}),
                                 w.off.ptr, cn + 1))) return rc;
        gather_pairs_kernel<<<grid_for(d, cn, 8), 256, 0, d->stream>>>(sub, cn, J.read_off, J.reads, J.quals, w.off.ptr, w.reads.ptr, J.quals ? w.quals.ptr : nullptr);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        if ((rc = map_sub(d, P, cn, w.reads.ptr, J.quals ? w.quals.ptr : nullptr, w.off.ptr, max_len, !single_end)) ||
            (rc = append(J, sub, cn, nullptr, single_end ? (uint8_t)GB_ALN_PAIRED : (uint8_t)0))) return rc;
    }
    return GB_OK;
}

} // namespace
} // namespace gb

using namespace gb;

extern "C" int gb_map_paired_job_device(gb_device* d, const gb_map_params* hp, gb_fragment_distribution* f, uint32_t training_window,
                                        uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals, const uint64_t* d_read_off,
                                        uint32_t max_read_len, gb_alignment* d_aln, gb_mapping* d_mappings, uint64_t mapping_pool_cap,
                                        uint32_t* d_edits, uint64_t edit_pool_cap, uint8_t* d_status, uint8_t* d_pair_route,
                                        uint64_t* n_mappings_used, uint64_t* n_edits_used) {
    return gb::guarded("gb_map_paired_job_device", [&] {
        if (!d || !hp || !f || (n_reads && (!d_reads || !d_read_off || !d_aln || !d_mappings || !d_edits || !d_status))) {
            g_last_error = "gb_map_paired_job_device: null argument"; return GB_ERR_ARG;
        }
        if (n_reads % 2 != 0) { g_last_error = "paired mapping needs an even number of reads"; return GB_ERR_ARG; }
        if (hp->max_multimaps != 1) { g_last_error = "gb_map_paired_job_device reports one mapping per read (max_multimaps = 1); use gb_map_batch_device with a forced distribution for multi-mapping"; return GB_ERR_ARG; }
        if (max_read_len > 512) { g_last_error = "reads longer than 512 bp are not supported by the short-read path"; return GB_ERR_ARG; }
        if (training_window == 0) training_window = 2048;
        if (n_mappings_used) *n_mappings_used = 0;
        if (n_edits_used) *n_edits_used = 0;
        const uint32_t n_pairs = n_reads / 2;
        d->pj_windows = 0; d->pj_training_ms = 0.0;
        if (n_pairs == 0) return GB_OK;                  // nothing to map: the distribution stays as it is
        GB_CUDA(cudaSetDevice(d->device));
        auto& w = d->pj;
        Job J{d, hp, d_reads, d_quals, d_read_off, max_read_len, d_aln, d_mappings, mapping_pool_cap, d_edits, edit_pool_cap, d_status, d_pair_route};
        int rc;
        if ((rc = w.buffered.reserve(n_pairs))) return rc;
        uint32_t n_buffered = 0, next = 0;              // ambiguous_pair_buffer size; first pair not consumed yet

        // ---- training: windows of pairs mapped single-ended at the caller's offsets, in input order ----------------------
        const auto t0 = std::chrono::steady_clock::now();
        const uint32_t window_cap = std::min(training_window, d->map_chunk / 2);
        std::vector<uint64_t> stats;
        std::vector<int64_t> cut;
        while (!f->is_fixed && next < n_pairs) {
            const uint32_t wp = std::min(window_cap, n_pairs - next), wr = 2 * wp;
            const PairSet win{nullptr, next};
            const uint64_t* off = d_read_off + 2 * (uint64_t)next;
            if ((rc = pair_stats(J, win, wp, wp, 0, stats))) return rc;
            if ((rc = reserve_sub(d, hp, wr)) || (rc = w.pair.reserve(3 * (size_t)wp)) || (rc = w.out.reserve(3 + 2 * (size_t)wp))) return rc;
            if ((rc = map_sub(d, hp, wr, d_reads, d_quals, off, (uint32_t)stats[1], false))) return rc;
            uint32_t* elig = w.pair.ptr; uint32_t* incl = w.pair.ptr + wp; uint32_t* keep = w.pair.ptr + 2 * (size_t)wp;
            int64_t* len = w.out.ptr; int64_t* out = w.out.ptr + wp;
            train_classify_kernel<<<grid_for(d, wp, 128), 128, 0, d->stream>>>(d->ix, wp, w.aln.ptr, w.status.ptr, w.maps.ptr, off, d->sc.match,
                                                                               (int64_t)hp->max_fragment_length, elig, len);
            d->launches++;
            GB_CUDA(cudaGetLastError());
            size_t bytes = 0;
            GB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, bytes, elig, incl, (int)wp, d->stream));
            if ((rc = w.scan_tmp.reserve(bytes))) return rc;
            GB_CUDA(cub::DeviceScan::InclusiveSum(w.scan_tmp.ptr, bytes, elig, incl, (int)wp, d->stream));
            d->launches++;
            const uint64_t size = f->lengths.size();
            const uint64_t budget = f->maximum_sample_size > size ? f->maximum_sample_size - size : UINT64_MAX;     // add() never finalizes past it
            train_cut_kernel<<<grid_for(d, wp, 128), 128, 0, d->stream>>>(wp, next, elig, incl, len, budget, keep, w.buffered.ptr, n_buffered,
                                                                          d_pair_route, out);
            d->launches++;
            GB_CUDA(cudaGetLastError());
            cut.resize(2 + (size_t)std::min<uint64_t>(budget, wp));
            GB_CUDA(cudaMemcpyAsync(cut.data(), out, sizeof(int64_t) * cut.size(), cudaMemcpyDeviceToHost, d->stream));
            GB_CUDA(cudaStreamSynchronize(d->stream));
            const uint32_t consumed = (uint32_t)cut[0], n_kept = (uint32_t)cut[1];
            for (uint32_t i = 0; i < n_kept; i++) f->add(cut[2 + i]);
            // pair_all(mapped_pair) links the two single-ended records as mates (minimizer_mapper.cpp:1345-1350)
            if ((rc = append(J, win, wr, keep, (uint8_t)GB_ALN_PAIRED))) return rc;
            n_buffered += consumed - n_kept;
            next += consumed;
            d->pj_windows++;
        }
        d->pj_training_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        // end of input before the sample filled up: giraffe_main.cpp:2283-2296 finalizes with what there is
        f->is_fixed = true;
        gb_map_params P = *hp;
        P.fragment_mean = f->mu; P.fragment_stdev = f->sigma;

        // ---- the remaining pairs, then the ambiguous buffer (giraffe_main.cpp:2375-2396) ---------------------------------
        if (next < n_pairs) {
            if ((rc = map_pairs(J, &P, PairSet{nullptr, next}, n_pairs - next))) return rc;
            if (d_pair_route) GB_CUDA(cudaMemsetAsync(d_pair_route + next, GB_PAIR_PAIRED, n_pairs - next, d->stream));
        }
        if (n_buffered && (rc = map_pairs(J, &P, PairSet{w.buffered.ptr, 0}, n_buffered))) return rc;
        GB_CUDA(cudaStreamSynchronize(d->stream));
        if (n_mappings_used) *n_mappings_used = J.nm;
        if (n_edits_used) *n_edits_used = J.ne;
        return GB_OK;
    });
}

extern "C" int gb_paired_job_stats(const gb_device* d, uint32_t* training_windows, double* training_ms) {
    if (!d || !training_windows || !training_ms) return GB_ERR_ARG;
    *training_windows = d->pj_windows; *training_ms = d->pj_training_ms;
    return GB_OK;
}
