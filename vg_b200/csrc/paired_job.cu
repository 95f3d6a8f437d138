// paired_job.cu — the paired job of MinimizerMapper::map_paired(aln1, aln2, ambiguous_pair_buffer): the fragment length
// distribution, the training window both entry points map through, gb_map_paired_job (reads in host memory) and
// gb_map_paired_job_device (reads already in HBM).
//   FragmentLengthDistribution      mapper.hpp:83-139, mapper.cpp:5231-5333
//   Phi_inv / normal_pdf            statistics.cpp:49-113, statistics.hpp:181-188
//   map_paired (training branch)    minimizer_mapper.cpp:1303-1395
//   job driver                      giraffe_main.cpp:2246-2400
// Kernels:
//   pair_stats_kernel       thread per pair: single-end fallback count and the longest read of every sub-batch
//   train_classify_kernel   thread per pair: the training rule of map_paired (minimizer_mapper.cpp:1316-1336)
//   train_cut_kernel        thread per pair: which pairs a window consumes, their routes, the lengths to register, the buffer
//   gather_pairs_kernel     warp per read: a sub-batch's pairs as contiguous, zero-based reads and qualities
//   record_append_kernel    warp per record: a sub-batch's records into the caller's pools at the running totals
// Every mapping pass is map_device.  The distribution stays on the host, as the reference runs training single-threaded
// (giraffe_main.cpp:2253): each training window copies back its cut and the lengths to register.  The host job uploads
// each window, copies its records back and appends the kept pairs on the host, then maps the remaining and the buffered
// pairs with gb_map_paired_batch; the device job appends on the device and maps them per sub-batch, so it synchronises a
// few times per window and per sub-batch.
#include <cub/cub.cuh>
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "fragment_distribution.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

using gb::g_last_error;

namespace {

// AS 241 (Wichura 1988), PPND16: normal quantile by three rational approximations.
double phi_inv(double p) {
    static const double a[8] = {3.387132872796366608, 133.14166789178437745, 1971.5909503065514427, 13731.693765509461125,
                                45921.953931549871457, 67265.770927008700853, 33430.575583588128105, 2509.0809287301226727};
    static const double b[8] = {1.0, 42.313330701600911252, 687.1870074920579083, 5394.1960214247511077,
                                21213.794301586595867, 39307.89580009271061, 28729.085735721942674, 5226.495278852854561};
    static const double c[8] = {1.42343711074968357734, 4.6303378461565452959, 5.7694972214606914055, 3.64784832476320460504,
                                1.27045825245236838258, 0.24178072517745061177, 0.0227238449892691845833, 7.7454501427834140764e-4};
    static const double d[8] = {1.0, 2.05319162663775882187, 1.6763848301838038494, 0.68976733498510000455,
                                0.14810397642748007459, 0.0151986665636164571966, 5.475938084995344946e-4, 1.05075007164441684324e-9};
    static const double e[8] = {6.6579046435011037772, 5.4637849111641143699, 1.7848265399172913358, 0.29656057182850489123,
                                0.026532189526576123093, 0.0012426609473880784386, 2.71155556874348757815e-5, 2.01033439929228813265e-7};
    static const double f[8] = {1.0, 0.59983220655588793769, 0.13692988092273580531, 0.0148753612908506148525,
                                7.868691311456132591e-4, 1.8463183175100546818e-5, 1.4215117583164458887e-7, 2.04426310338993978564e-15};
    auto poly = [](const double* k, double r) { double v = k[7]; for (int i = 6; i >= 0; i--) v = v * r + k[i]; return v; };
    const double q = p - 0.5;
    if (std::fabs(q) <= 0.425) { const double r = 0.180625 - q * q; return q * poly(a, r) / poly(b, r); }
    double r = std::sqrt(-std::log(q > 0 ? 1.0 - p : p));
    double val;
    if (r <= 5.0) { r -= 1.6; val = poly(c, r) / poly(d, r); } else { r -= 5.0; val = poly(e, r) / poly(f, r); }
    return q < 0.0 ? -val : val;
}

} // namespace

void gb_fragment_distribution::estimate() {
    const size_t to_skip = (size_t)(lengths.size() * (1.0 - robust_estimation_fraction) * 0.5);
    auto begin = lengths.begin(); auto end = lengths.end();
    for (size_t i = 0; i < to_skip; i++) { ++begin; --end; }
    double count = 0.0, sum = 0.0, sum_of_sqs = 0.0;
    for (auto it = begin; it != end; ++it) { count += 1.0; sum += *it; sum_of_sqs += (*it) * (*it); }
    mu = sum / count;
    const double raw_var = sum_of_sqs / count - mu * mu;
    const double a = phi_inv(1.0 - 0.5 * (1.0 - robust_estimation_fraction));
    const double pdf_a = 0.3989422804014327 * std::exp(-0.5 * a * a);
    sigma = std::sqrt(raw_var / (1.0 - 2.0 * a * pdf_a));
}

extern "C" gb_fragment_distribution* gb_fragment_create(uint64_t maximum_sample_size, uint64_t reestimation_frequency, double robust_estimation_fraction) {
    if (!(robust_estimation_fraction > 0.0 && robust_estimation_fraction < 1.0) || reestimation_frequency == 0) {
        g_last_error = "gb_fragment_create: robust_estimation_fraction must be in (0, 1) and reestimation_frequency positive";
        return nullptr;
    }
    gb_fragment_distribution* f = new gb_fragment_distribution();
    f->maximum_sample_size = maximum_sample_size; f->reestimation_frequency = reestimation_frequency; f->robust_estimation_fraction = robust_estimation_fraction;
    return f;
}
extern "C" void gb_fragment_destroy(gb_fragment_distribution* f) { delete f; }
extern "C" void gb_fragment_force(gb_fragment_distribution* f, double mean, double stdev) { f->mu = mean; f->sigma = stdev; f->is_fixed = true; }
extern "C" void gb_fragment_register(gb_fragment_distribution* f, int64_t length) { f->add(length); }
extern "C" void gb_fragment_finalize(gb_fragment_distribution* f) { f->is_fixed = true; }
extern "C" double gb_fragment_mean(const gb_fragment_distribution* f) { return f->mu; }
extern "C" double gb_fragment_stdev(const gb_fragment_distribution* f) { return f->sigma; }
extern "C" int gb_fragment_is_finalized(const gb_fragment_distribution* f) { return f->is_fixed ? 1 : 0; }
extern "C" uint64_t gb_fragment_sample_size(const gb_fragment_distribution* f) { return f->lengths.size(); }

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

// stats[0] = pairs whose read 1 takes the single-end fallback of map_paired (decided per pair as map_batch_host does);
// stats[1 + c] = longest read of sub-batch c.
__global__ void pair_stats_kernel(PairSet s, uint32_t n_pairs, uint32_t chunk_pairs, const uint64_t* off, int64_t fragment_limit,
                                  int64_t distance_limit, unsigned long long* stats) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pairs; i += gridDim.x * blockDim.x) {
        const uint64_t r = 2 * (uint64_t)s.pair(i);
        const uint64_t L1 = off[r + 1] - off[r], L2 = off[r + 2] - off[r + 1];
        if (single_end_fallback(fragment_limit, distance_limit, (int64_t)L1)) atomicAdd(stats, 1ull);
        atomicMax(stats + 1 + i / chunk_pairs, (unsigned long long)max(L1, L2));
    }
}

// The training rule, per pair of a window mapped single-ended: both ends mapped with status OK, MAPQ 60 and score >= 0.85 *
// match * length, and the distance from the first mapping of read 1 to the flipped first mapping of read 2 below
// max_fragment_length.  Unreachable is -1 (size_t max stored into an int64_t, minimizer_mapper.cpp:3879-3884), which passes
// that test and is registered, as the reference does.
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

// The caller's arguments and the job's running state.  The arrays are host addresses for gb_map_paired_job and device
// addresses for gb_map_paired_job_device.
struct Job {
    gb_device* d; const gb_map_params* hp;
    const uint8_t* reads; const uint8_t* quals; const uint64_t* read_off; uint32_t max_read_len;
    gb_alignment* aln; gb_mapping* maps; uint64_t map_cap; uint32_t* edits; uint64_t edit_cap; uint8_t* status; uint8_t* route;
    uint64_t nm = 0, ne = 0;                  // mappings / edits appended so far
};

// The refusals and the default both entry points share; `multimap_entry` is the call to use for several mappings per read.
int check_job(const Job& J, const gb_fragment_distribution* f, uint32_t n_reads, const char* entry, const char* multimap_entry,
              uint32_t& training_window) {
    if (!J.d || !J.hp || !f || (n_reads && (!J.reads || !J.read_off || !J.aln || !J.maps || !J.edits || !J.status))) {
        g_last_error = std::string(entry) + ": null argument"; return GB_ERR_ARG;
    }
    if (n_reads % 2 != 0) { g_last_error = "paired mapping needs an even number of reads"; return GB_ERR_ARG; }
    if (J.hp->max_multimaps != 1) {
        g_last_error = std::string(entry) + " reports one mapping per read (max_multimaps = 1); use " + multimap_entry + " with a forced distribution for multi-mapping";
        return GB_ERR_ARG;
    }
    if (training_window == 0) training_window = 2048;
    return GB_OK;
}

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

// What a training window consumed: pairs, kept pairs, and the keep mask of its pairs (in d->pj).
struct WindowCut { uint32_t consumed, kept; const uint32_t* keep; };

// One training window: pairs [first, first + n_pairs), whose 2 * n_pairs reads are at reads + off[i] in HBM, mapped
// single-ended into d->pj's sub-batch buffers, classified, and cut where the sample fills; the kept lengths are
// registered with f in pair order.  Consumed pairs that are not kept go to d->pj.buffered after n_buffered, and to
// route (may be NULL).  Synchronous: the records and the keep mask are in place when it returns.
int train_window(gb_device* d, const gb_map_params* hp, gb_fragment_distribution* f, uint32_t first, uint32_t n_pairs,
                 const uint8_t* reads, const uint8_t* quals, const uint64_t* off, uint32_t max_len, uint32_t n_buffered,
                 uint8_t* route, WindowCut& cut) {
    auto& w = d->pj;
    const uint32_t wr = 2 * n_pairs;
    int rc;
    if ((rc = reserve_sub(d, hp, wr)) || (rc = w.pair.reserve(3 * (size_t)n_pairs)) || (rc = w.out.reserve(3 + 2 * (size_t)n_pairs))) return rc;
    if ((rc = map_sub(d, hp, wr, reads, quals, off, max_len, false))) return rc;
    uint32_t* elig = w.pair.ptr; uint32_t* incl = w.pair.ptr + n_pairs; uint32_t* keep = w.pair.ptr + 2 * (size_t)n_pairs;
    int64_t* len = w.out.ptr; int64_t* out = w.out.ptr + n_pairs;
    train_classify_kernel<<<grid_for(d, n_pairs, 128), 128, 0, d->stream>>>(d->ix, n_pairs, w.aln.ptr, w.status.ptr, w.maps.ptr, off, d->sc.match,
                                                                            (int64_t)hp->max_fragment_length, elig, len);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    size_t bytes = 0;
    GB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, bytes, elig, incl, (int)n_pairs, d->stream));
    if ((rc = w.scan_tmp.reserve(bytes))) return rc;
    GB_CUDA(cub::DeviceScan::InclusiveSum(w.scan_tmp.ptr, bytes, elig, incl, (int)n_pairs, d->stream));
    d->launches++;
    const uint64_t size = f->lengths.size();
    const uint64_t budget = f->maximum_sample_size > size ? f->maximum_sample_size - size : UINT64_MAX;     // add() never finalizes past it
    train_cut_kernel<<<grid_for(d, n_pairs, 128), 128, 0, d->stream>>>(n_pairs, first, elig, incl, len, budget, keep, w.buffered.ptr, n_buffered,
                                                                       route, out);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    std::vector<int64_t> h_out(2 + (size_t)std::min<uint64_t>(budget, n_pairs));
    GB_CUDA(cudaMemcpyAsync(h_out.data(), out, sizeof(int64_t) * h_out.size(), cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));
    cut = WindowCut{(uint32_t)h_out[0], (uint32_t)h_out[1], keep};
    for (uint32_t i = 0; i < cut.kept; i++) f->add(h_out[2 + i]);
    return GB_OK;
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
    if (stats[0] != 0 && !single_end) { g_last_error = MIXED_FALLBACK_REFUSAL; return GB_ERR_ARG; }
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

// Copy record `sub_index` of a sub-batch in host memory into the caller's pools at the running totals and store its header
// under the caller's read id.
int append_records(Job& J, const gb_alignment* sub_aln, const gb_mapping* sub_maps, const uint32_t* sub_edits, const uint8_t* sub_status,
                   uint32_t sub_index, uint32_t read_id, uint8_t extra_flags) {
    gb_alignment rec = sub_aln[sub_index];
    if (J.nm + rec.n_mappings > J.map_cap || J.ne + rec.n_edits > J.edit_cap) { g_last_error = "gb_map_paired_job: output pool too small"; return GB_ERR_CAPACITY; }
    if (rec.n_mappings) memcpy(J.maps + J.nm, sub_maps + rec.mapping_off, (size_t)rec.n_mappings * sizeof(gb_mapping));
    if (rec.n_edits) memcpy(J.edits + J.ne, sub_edits + rec.edit_off, (size_t)rec.n_edits * 4);
    rec.read_id = read_id; rec.mapping_off = (uint32_t)J.nm; rec.edit_off = (uint32_t)J.ne;
    rec.flags |= extra_flags;
    J.nm += rec.n_mappings; J.ne += rec.n_edits;
    J.aln[read_id] = rec; J.status[read_id] = sub_status[sub_index];
    return GB_OK;
}

} // namespace
} // namespace gb

using namespace gb;

extern "C" int gb_map_paired_job(gb_device* d, const gb_map_params* hp, gb_fragment_distribution* f, uint32_t training_window,
                                 uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                                 gb_alignment* aln, gb_mapping* mappings, uint64_t mapping_pool_cap, uint32_t* edits, uint64_t edit_pool_cap,
                                 uint8_t* status, uint8_t* pair_route, uint64_t* n_mappings_used, uint64_t* n_edits_used) {
    return gb::guarded("gb_map_paired_job", [&] {
        Job J{d, hp, reads, quals, read_off, 0, aln, mappings, mapping_pool_cap, edits, edit_pool_cap, status, pair_route};
        int rc;
        if ((rc = check_job(J, f, n_reads, "gb_map_paired_job", "gb_map_paired_batch", training_window))) return rc;
        const uint32_t n_pairs = n_reads / 2;
        if (n_pairs == 0) { if (n_mappings_used) *n_mappings_used = 0; if (n_edits_used) *n_edits_used = 0; return GB_OK; }     // nothing to map: the distribution stays as it is
        auto& w = d->pj;
        std::vector<uint32_t> buffered;               // ambiguous_pair_buffer (pair indices)
        uint32_t next = 0;                            // first pair not consumed yet

        // ---- training: each window uploaded, trained on the device, its kept records copied back in input order -------
        const uint32_t window_cap = std::min(training_window, d->map_chunk / 2);
        while (!f->is_fixed && next < n_pairs) {
            const uint32_t wp = std::min(window_cap, n_pairs - next), wr = 2 * wp;
            // the host copy of the window's records first: caps too large for host memory fail before any device work
            std::vector<gb_alignment> sa(wr); std::vector<uint8_t> ss(wr);
            std::vector<gb_mapping> sm((size_t)wr * hp->mapping_cap_per_read); std::vector<uint32_t> se((size_t)wr * hp->edit_cap_per_read);
            const uint64_t base = read_off[2 * (uint64_t)next], bases = read_off[2 * (uint64_t)next + wr] - base;
            std::vector<uint64_t> off(wr + 1);
            uint32_t max_len = 0;
            for (uint32_t i = 0; i <= wr; i++) off[i] = read_off[2 * (uint64_t)next + i] - base;
            for (uint32_t i = 0; i < wr; i++) max_len = std::max<uint32_t>(max_len, (uint32_t)(off[i + 1] - off[i]));
            GB_CUDA(cudaSetDevice(d->device));
            // train_cut_kernel lists the window's buffered pairs in w.buffered; this job keeps its buffer on the host
            if ((rc = w.reads.reserve(bases + 16)) || (quals && (rc = w.quals.reserve(bases + 16))) || (rc = w.off.reserve((size_t)wr + 1)) ||
                (rc = w.buffered.reserve(wp))) return rc;
            GB_CUDA(cudaMemcpyAsync(w.reads.ptr, reads + base, bases, cudaMemcpyHostToDevice, d->stream));
            if (quals) GB_CUDA(cudaMemcpyAsync(w.quals.ptr, quals + base, bases, cudaMemcpyHostToDevice, d->stream));
            GB_CUDA(cudaMemcpyAsync(w.off.ptr, off.data(), sizeof(uint64_t) * off.size(), cudaMemcpyHostToDevice, d->stream));
            WindowCut cut;
            if ((rc = train_window(d, hp, f, next, wp, w.reads.ptr, quals ? w.quals.ptr : nullptr, w.off.ptr, max_len, 0, nullptr, cut))) return rc;
            uint64_t used[2];
            GB_CUDA(cudaMemcpyAsync(used, w.totals.ptr, sizeof used, cudaMemcpyDeviceToHost, d->stream));
            GB_CUDA(cudaStreamSynchronize(d->stream));
            std::vector<uint32_t> keep(cut.consumed);
            GB_CUDA(cudaMemcpyAsync(keep.data(), cut.keep, sizeof(uint32_t) * keep.size(), cudaMemcpyDeviceToHost, d->stream));
            GB_CUDA(cudaMemcpyAsync(sa.data(), w.aln.ptr, sizeof(gb_alignment) * wr, cudaMemcpyDeviceToHost, d->stream));
            GB_CUDA(cudaMemcpyAsync(ss.data(), w.status.ptr, wr, cudaMemcpyDeviceToHost, d->stream));
            GB_CUDA(cudaMemcpyAsync(sm.data(), w.maps.ptr, sizeof(gb_mapping) * used[0], cudaMemcpyDeviceToHost, d->stream));
            GB_CUDA(cudaMemcpyAsync(se.data(), w.edits.ptr, sizeof(uint32_t) * used[1], cudaMemcpyDeviceToHost, d->stream));
            GB_CUDA(cudaStreamSynchronize(d->stream));
            for (uint32_t i = 0; i < cut.consumed; i++) {
                const uint32_t pair = next + i;
                if (keep[i]) {
                    for (uint32_t r = 0; r < 2; r++)
                        // pair_all(mapped_pair) links the two single-ended records as mates (minimizer_mapper.cpp:1345-1350)
                        if ((rc = append_records(J, sa.data(), sm.data(), se.data(), ss.data(), 2 * i + r, 2 * pair + r, GB_ALN_PAIRED))) return rc;
                    if (pair_route) pair_route[pair] = GB_PAIR_TRAINING;
                } else {
                    buffered.push_back(pair);
                    if (pair_route) pair_route[pair] = GB_PAIR_BUFFERED;
                }
            }
            next += cut.consumed;
        }
        // end of input before the sample filled up: giraffe_main.cpp:2283-2296 finalizes with what there is
        f->is_fixed = true;
        gb_map_params P = *hp;
        P.fragment_mean = f->mu; P.fragment_stdev = f->sigma;

        // ---- the remaining pairs, straight into the caller's pools ---------------------------------------------------
        if (next < n_pairs) {
            const uint32_t rr = 2 * (n_pairs - next);
            const uint64_t base = read_off[2 * (uint64_t)next];
            std::vector<uint64_t> off;
            const uint64_t* off_p = read_off + 2 * (uint64_t)next;
            if (base != 0) { off.resize(rr + 1); for (uint32_t i = 0; i <= rr; i++) off[i] = off_p[i] - base; off_p = off.data(); }
            uint64_t um = 0, ue = 0;
            if ((rc = gb_map_paired_batch(d, &P, rr, reads + base, quals ? quals + base : nullptr, off_p, aln + 2 * (size_t)next,
                                          mappings + J.nm, mapping_pool_cap - J.nm, edits + J.ne, edit_pool_cap - J.ne, status + 2 * (size_t)next, &um, &ue))) return rc;
            for (uint32_t i = 0; i < rr; i++) {
                gb_alignment& a = aln[2 * (size_t)next + i];
                a.read_id += 2 * next; a.mapping_off += (uint32_t)J.nm; a.edit_off += (uint32_t)J.ne;
            }
            J.nm += um; J.ne += ue;
            if (pair_route) for (uint32_t x = next; x < n_pairs; x++) pair_route[x] = GB_PAIR_PAIRED;
        }
        // ---- the ambiguous buffer, mapped paired last (giraffe_main.cpp:2375-2396) -----------------------------------
        if (!buffered.empty()) {
            const uint32_t br = 2 * (uint32_t)buffered.size();
            std::vector<uint64_t> off(br + 1, 0);
            for (uint32_t i = 0; i < buffered.size(); i++) for (uint32_t r = 0; r < 2; r++) {
                const uint64_t ri = 2 * (uint64_t)buffered[i] + r;
                off[2 * i + r + 1] = off[2 * i + r] + (read_off[ri + 1] - read_off[ri]);
            }
            std::vector<uint8_t> br_reads(off[br] + 16), br_quals(quals ? off[br] + 16 : 0);
            for (uint32_t i = 0; i < buffered.size(); i++) for (uint32_t r = 0; r < 2; r++) {
                const uint64_t ri = 2 * (uint64_t)buffered[i] + r, len = read_off[ri + 1] - read_off[ri];
                memcpy(br_reads.data() + off[2 * i + r], reads + read_off[ri], len);
                if (quals) memcpy(br_quals.data() + off[2 * i + r], quals + read_off[ri], len);
            }
            std::vector<gb_alignment> sa(br); std::vector<uint8_t> ss(br);
            std::vector<gb_mapping> sm((size_t)br * hp->mapping_cap_per_read); std::vector<uint32_t> se((size_t)br * hp->edit_cap_per_read);
            uint64_t um = 0, ue = 0;
            if ((rc = gb_map_paired_batch(d, &P, br, br_reads.data(), quals ? br_quals.data() : nullptr, off.data(), sa.data(), sm.data(), sm.size(),
                                          se.data(), se.size(), ss.data(), &um, &ue))) return rc;
            for (uint32_t i = 0; i < buffered.size(); i++) for (uint32_t r = 0; r < 2; r++)
                if ((rc = append_records(J, sa.data(), sm.data(), se.data(), ss.data(), 2 * i + r, 2 * buffered[i] + r, 0))) return rc;
        }
        if (n_mappings_used) *n_mappings_used = J.nm;
        if (n_edits_used) *n_edits_used = J.ne;
        return GB_OK;
    });
}

extern "C" int gb_map_paired_job_device(gb_device* d, const gb_map_params* hp, gb_fragment_distribution* f, uint32_t training_window,
                                        uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals, const uint64_t* d_read_off,
                                        uint32_t max_read_len, gb_alignment* d_aln, gb_mapping* d_mappings, uint64_t mapping_pool_cap,
                                        uint32_t* d_edits, uint64_t edit_pool_cap, uint8_t* d_status, uint8_t* d_pair_route,
                                        uint64_t* n_mappings_used, uint64_t* n_edits_used) {
    return gb::guarded("gb_map_paired_job_device", [&] {
        Job J{d, hp, d_reads, d_quals, d_read_off, max_read_len, d_aln, d_mappings, mapping_pool_cap, d_edits, edit_pool_cap, d_status, d_pair_route};
        int rc;
        if ((rc = check_job(J, f, n_reads, "gb_map_paired_job_device", "gb_map_batch_device", training_window))) return rc;
        if (max_read_len > 512) { g_last_error = "reads longer than 512 bp are not supported by the short-read path"; return GB_ERR_ARG; }
        if (n_mappings_used) *n_mappings_used = 0;
        if (n_edits_used) *n_edits_used = 0;
        const uint32_t n_pairs = n_reads / 2;
        d->pj_windows = 0; d->pj_training_ms = 0.0;
        if (n_pairs == 0) return GB_OK;                  // nothing to map: the distribution stays as it is
        GB_CUDA(cudaSetDevice(d->device));
        auto& w = d->pj;
        if ((rc = w.buffered.reserve(n_pairs))) return rc;
        uint32_t n_buffered = 0, next = 0;              // ambiguous_pair_buffer size; first pair not consumed yet

        // ---- training: windows of pairs mapped single-ended at the caller's offsets, in input order ----------------------
        const auto t0 = std::chrono::steady_clock::now();
        const uint32_t window_cap = std::min(training_window, d->map_chunk / 2);
        std::vector<uint64_t> stats;
        while (!f->is_fixed && next < n_pairs) {
            const uint32_t wp = std::min(window_cap, n_pairs - next);
            const PairSet win{nullptr, next};
            WindowCut cut;
            if ((rc = pair_stats(J, win, wp, wp, 0, stats)) ||
                (rc = train_window(d, hp, f, next, wp, d_reads, d_quals, d_read_off + 2 * (uint64_t)next, (uint32_t)stats[1], n_buffered, d_pair_route, cut)) ||
                // pair_all(mapped_pair) links the two single-ended records as mates (minimizer_mapper.cpp:1345-1350)
                (rc = append(J, win, 2 * wp, cut.keep, (uint8_t)GB_ALN_PAIRED))) return rc;
            n_buffered += cut.consumed - cut.kept;
            next += cut.consumed;
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
