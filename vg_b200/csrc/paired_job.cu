// paired_job.cu — host side of the paired job: the fragment length distribution and the training phase
// of MinimizerMapper::map_paired(aln1, aln2, ambiguous_pair_buffer).
//   FragmentLengthDistribution      mapper.hpp:83-139, mapper.cpp:5231-5333
//   Phi_inv / normal_pdf            statistics.cpp:49-113, statistics.hpp:181-188
//   map_paired (training branch)    minimizer_mapper.cpp:1303-1395
//   job driver                      giraffe_main.cpp:2246-2400
// All mapping work goes through gb_map_batch / gb_map_paired_batch (GPU); what is here is the sequential
// bookkeeping the reference also runs single-threaded (giraffe_main.cpp:2253), one window of pairs at a time.
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "fragment_distribution.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
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

namespace {

// minimum_distance(pos1, pos2), oriented, through the chain payload (the host twin of oriented_distance in
// align_read.cuh); unreachable is size_t max, which vg stores into an int64_t (minimizer_mapper.cpp:3879-3884).
int64_t host_oriented_distance(const gb_device* d, uint32_t node_a, uint32_t off_a, uint32_t node_b, uint32_t off_b) {
    const int64_t UNREACHABLE = -1;
    if ((node_a & 1u) != (node_b & 1u)) return UNREACHABLE;
    uint32_t src = node_a, dst = node_b; int64_t src_off = off_a, dst_off = off_b;
    if (node_a & 1u) {
        src = node_b; dst = node_a;
        src_off = (int64_t)d->h_node_len[node_b] - (int64_t)off_b;
        dst_off = (int64_t)d->h_node_len[node_a] - (int64_t)off_a;
    }
    const int64_t src_len = d->h_node_len[src];
    const gb_dist_payload& ps = d->h_dist[src >> 1]; const gb_dist_payload& pd = d->h_dist[dst >> 1];
    if (ps.component != pd.component) return UNREACHABLE;
    if ((src >> 1) == (dst >> 1)) return dst_off >= src_off ? dst_off - src_off : UNREACHABLE;
    if (ps.slot < pd.slot) return (src_len - src_off) + ((int64_t)(int32_t)pd.x_in - (int64_t)(int32_t)ps.x_out) + dst_off;
    if (ps.slot == pd.slot && ps.slot < d->h_slots.size()) {
        const gb_slot_rec& sr = d->h_slots[ps.slot];
        if (sr.table_off != 0xFFFFFFFFu && ps.allele < sr.n && pd.allele < sr.n) {
            const uint16_t t = d->h_site_dist[sr.table_off + (size_t)ps.allele * sr.n + pd.allele];
            if (t != 0xFFFF) return (src_len - src_off) + (int64_t)t + dst_off;
        }
    }
    return UNREACHABLE;
}

// Copy the records of reads [first, first + count) of a sub-batch into the caller's pools at the running
// totals and store their headers under the caller's read ids.
int append_records(const gb_alignment* sub_aln, const gb_mapping* sub_maps, const uint32_t* sub_edits, const uint8_t* sub_status,
                   uint32_t sub_index, uint32_t read_id, uint8_t extra_flags, gb_alignment* aln, gb_mapping* mappings, uint64_t mapping_pool_cap,
                   uint32_t* edits, uint64_t edit_pool_cap, uint8_t* status, uint64_t& nm, uint64_t& ne) {
    gb_alignment rec = sub_aln[sub_index];
    if (nm + rec.n_mappings > mapping_pool_cap || ne + rec.n_edits > edit_pool_cap) { g_last_error = "gb_map_paired_job: output pool too small"; return GB_ERR_CAPACITY; }
    if (rec.n_mappings) memcpy(mappings + nm, sub_maps + rec.mapping_off, (size_t)rec.n_mappings * sizeof(gb_mapping));
    if (rec.n_edits) memcpy(edits + ne, sub_edits + rec.edit_off, (size_t)rec.n_edits * 4);
    rec.read_id = read_id; rec.mapping_off = (uint32_t)nm; rec.edit_off = (uint32_t)ne;
    rec.flags |= extra_flags;
    nm += rec.n_mappings; ne += rec.n_edits;
    aln[read_id] = rec; status[read_id] = sub_status[sub_index];
    return GB_OK;
}

} // namespace

extern "C" int gb_map_paired_job(gb_device* d, const gb_map_params* hp, gb_fragment_distribution* f, uint32_t training_window,
                                 uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                                 gb_alignment* aln, gb_mapping* mappings, uint64_t mapping_pool_cap, uint32_t* edits, uint64_t edit_pool_cap,
                                 uint8_t* status, uint8_t* pair_route, uint64_t* n_mappings_used, uint64_t* n_edits_used) {
    return gb::guarded("gb_map_paired_job", [&] {
        if (!d || !hp || !f) { g_last_error = "gb_map_paired_job: null argument"; return GB_ERR_ARG; }
        if (n_reads % 2 != 0) { g_last_error = "paired mapping needs an even number of reads"; return GB_ERR_ARG; }
        if (hp->max_multimaps != 1) { g_last_error = "gb_map_paired_job reports one mapping per read (max_multimaps = 1); use gb_map_paired_batch with a forced distribution for multi-mapping"; return GB_ERR_ARG; }
        if (training_window == 0) training_window = 2048;
        const uint32_t n_pairs = n_reads / 2;
        if (n_pairs == 0) { if (n_mappings_used) *n_mappings_used = 0; if (n_edits_used) *n_edits_used = 0; return GB_OK; }     // nothing to map: the distribution stays as it is
        uint64_t nm = 0, ne = 0;
        int rc;
        std::vector<uint32_t> buffered;               // ambiguous_pair_buffer (pair indices)
        uint32_t next = 0;                            // first pair not consumed yet

        // ---- training: map(aln1), map(aln2), register unambiguous distances, in input order ------------------------
        while (!f->is_fixed && next < n_pairs) {
            const uint32_t wp = std::min(training_window, n_pairs - next), wr = 2 * wp;
            const uint64_t base = read_off[2 * (uint64_t)next];
            std::vector<uint64_t> off(wr + 1);
            for (uint32_t i = 0; i <= wr; i++) off[i] = read_off[2 * (uint64_t)next + i] - base;
            std::vector<gb_alignment> sa(wr); std::vector<uint8_t> ss(wr);
            std::vector<gb_mapping> sm((size_t)wr * hp->mapping_cap_per_read); std::vector<uint32_t> se((size_t)wr * hp->edit_cap_per_read);
            uint64_t um = 0, ue = 0;
            if ((rc = gb_map_batch(d, hp, wr, reads + base, quals ? quals + base : nullptr, off.data(), sa.data(), sm.data(), sm.size(),
                                   se.data(), se.size(), ss.data(), &um, &ue))) return rc;
            uint32_t consumed = 0;
            for (uint32_t i = 0; i < wp && !f->is_fixed; i++, consumed++) {
                const uint32_t pair = next + i;
                bool both_perfect_unique = true;
                for (uint32_t r = 0; r < 2; r++) {
                    const gb_alignment& a = sa[2 * i + r];
                    const int64_t L = (int64_t)(off[2 * i + r + 1] - off[2 * i + r]);
                    const double max_score_aln = (double)(d->sc.match * L);                      // score_exact_match (alignment_scorer.cpp:321)
                    both_perfect_unique = both_perfect_unique && ss[2 * i + r] == GB_ITEM_OK && (a.flags & GB_ALN_MAPPED) && a.mapq == 60 && (double)a.score >= max_score_aln * 0.85;
                }
                bool keep = false;
                if (both_perfect_unique) {
                    // initial_position(aln1) -> final_position(reverse complement of aln2) = the flipped start of aln2
                    const gb_mapping first1 = sm[sa[2 * i].mapping_off], first2 = sm[sa[2 * i + 1].mapping_off];
                    const int64_t dist = host_oriented_distance(d, first1.node, first1.offset, first2.node ^ 1u,
                                                                d->h_node_len[first2.node] - (uint32_t)first2.offset);
                    if (!(dist == std::numeric_limits<int64_t>::max() || dist >= (int64_t)hp->max_fragment_length)) { f->add(dist); keep = true; }
                }
                if (keep) {
                    for (uint32_t r = 0; r < 2; r++)
                        // pair_all(mapped_pair) links the two single-ended records as mates (minimizer_mapper.cpp:1345-1350)
                        if ((rc = append_records(sa.data(), sm.data(), se.data(), ss.data(), 2 * i + r, 2 * pair + r, GB_ALN_PAIRED, aln, mappings, mapping_pool_cap,
                                                 edits, edit_pool_cap, status, nm, ne))) return rc;
                    if (pair_route) pair_route[pair] = GB_PAIR_TRAINING;
                } else {
                    buffered.push_back(pair);
                    if (pair_route) pair_route[pair] = GB_PAIR_BUFFERED;
                }
            }
            next += consumed;
        }
        // end of input before the sample filled up: giraffe_main.cpp:2283-2296 finalizes with what there is
        if (!f->is_fixed) f->is_fixed = true;
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
                                          mappings + nm, mapping_pool_cap - nm, edits + ne, edit_pool_cap - ne, status + 2 * (size_t)next, &um, &ue))) return rc;
            for (uint32_t i = 0; i < rr; i++) {
                gb_alignment& a = aln[2 * (size_t)next + i];
                a.read_id += 2 * next; a.mapping_off += (uint32_t)nm; a.edit_off += (uint32_t)ne;
            }
            nm += um; ne += ue;
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
                if ((rc = append_records(sa.data(), sm.data(), se.data(), ss.data(), 2 * i + r, 2 * buffered[i] + r, 0, aln, mappings, mapping_pool_cap,
                                         edits, edit_pool_cap, status, nm, ne))) return rc;
        }
        if (n_mappings_used) *n_mappings_used = nm;
        if (n_edits_used) *n_edits_used = ne;
        return GB_OK;
    });
}
