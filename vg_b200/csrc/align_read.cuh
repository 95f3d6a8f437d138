// align_read.cuh — per-read / per-pair alignment logic of the align kernels (included by map.cu
// inside namespace gb).
//   extension-set selection      single-end minimizer_mapper.cpp:886-1063, paired-end :1904-2040
//   winner + MAPQ                single-end :1087-1188, paired-end :2505-2777
//   pairing                      :2108-2208, score_alignment_pair :6017-6028, distance_between :3879-3903
//   faster_cap                   :2946-3260
#pragma once

struct AlignArgs {
    const DevItem* items;
    const DevMinimizer* minimizers;
    ExtView ev;
    uint8_t* ws_base; size_t ws_stride;        // per-warp tail workspace
    uint8_t* cand_base; size_t cand_stride;    // per-warp candidate buffers
    gb_alignment* aln; gb_mapping* maps; uint32_t* edits; uint8_t* status;
    uint32_t tb_cells;
    // paired-end
    const PairState* pairs; double frag_mean, frag_sd;
    // work list written by the thread-per-pair fast path (nullptr: every pair)
    const uint32_t* slow_list; const uint32_t* slow_count;
    // mate rescue (max_rescue_attempts != 0): per-warp workspace; pairs found to need it by the plain kernel
    uint8_t* rescue_base; size_t rescue_stride;
    uint32_t* rescue_list; uint32_t* rescue_count;
    // tails whose DPs ran in xdrop_tile_kernel (entries == nullptr: none, every tail is aligned in place)
    PlanView plan;
    // bytes of shared memory per warp for the five temporary path buffers (0: they live in the HBM candidate workspace).
    // Paths are assembled by one lane with read-modify-write steps (the edit count of the open mapping): in HBM every step
    // is an L2 round trip, in shared memory it is a few cycles; the finished path is then copied to its slot by the warp.
    uint32_t tmp_bytes;
};

constexpr uint32_t N_SLOTS = 2 * MAX_CANDS + 8 + 32;   // candidate path slots per warp (both mates of a pair, + rescued alignments)
constexpr uint32_t N_TEMP_SLOTS = 5;              // res_left, res_right, scratch, middle, assembly

// Dynamic shared memory per warp of the warp-per-unit align kernels (align_kernel: 1 mate, align_kernel_pe: 2): the reads
// of the unit's mates, their qualities and the query buffer (Lc bytes each, rounded up to 16 together), the four DP
// columns of Lc + 1 cells and 64 spare bytes, then tmp_bytes for the temporary path slots.  Lc is a multiple of 16, so
// from the query buffer on this is the layout of dp_smem_per_warp(Lc).
__host__ __device__ inline size_t align_bytes_part(uint32_t Lc, uint32_t mates) { return ((size_t)(2 * mates + 1) * Lc + 15) & ~(size_t)15; }
__host__ __device__ inline size_t align_smem_per_warp(uint32_t Lc, uint32_t mates, uint32_t tmp_bytes) {
    return align_bytes_part(Lc, mates) + (size_t)(Lc + 1) * 4 * 4 + 64 + tmp_bytes;
}
struct AlignSmem {
    uint8_t* tmp;                                  // nullptr when tmp_bytes is 0
    uint8_t* read[2]; uint8_t* qual[2];            // [mate]
    uint8_t* qbuf;
    DpSmem dps;
};
__device__ inline AlignSmem align_smem_carve(uint8_t* smem, int warp, uint32_t Lc, uint32_t mates, uint32_t tmp_bytes) {
    uint8_t* base = smem + (size_t)warp * align_smem_per_warp(Lc, mates, tmp_bytes);
    AlignSmem s;
    s.tmp = tmp_bytes ? base + align_bytes_part(Lc, mates) + (size_t)(Lc + 1) * 4 * 4 + 64 : nullptr;
    s.read[0] = base; s.read[1] = base + Lc;                                 // read[1], qual[1]: two mates only
    s.qual[0] = base + (size_t)mates * Lc; s.qual[1] = base + (size_t)(mates + 1) * Lc;
    s.qbuf = base + 2 * (size_t)mates * Lc;
    s.dps = dp_cols_carve(reinterpret_cast<int32_t*>(base + align_bytes_part(Lc, mates)), Lc);
    return s;
}

// (real calls: the FP64 log1p / exp bodies are several hundred instructions and the align kernels are instruction-fetch bound)
static __device__ __noinline__ double d_add_log(double x, double y) { return x > y ? x + log1p(exp(y - x)) : y + log1p(exp(x - y)); }
static __device__ __noinline__ double d_subtract_log(double x, double y) { return x + log1p(-exp(y - x)); }

__device__ inline PathBuf slot_buf(uint8_t* cand_base, uint32_t slot, uint32_t map_cap, uint32_t edit_cap) {
    PathBuf p;
    const size_t per = (size_t)map_cap * sizeof(gb_mapping) + (size_t)edit_cap * 4;
    p.maps = (gb_mapping*)(cand_base + per * slot);
    p.edits = (uint32_t*)(cand_base + per * slot + (size_t)map_cap * sizeof(gb_mapping));
    p.n_maps = 0; p.n_edits = 0; p.map_cap = map_cap; p.edit_cap = edit_cap; p.overflow = false;
    return p;
}
// the mapping/edit counts of a finished slot live in the last two words of its mapping array
__device__ __forceinline__ uint32_t& slot_nm(const PathBuf& pb) { return ((uint32_t*)pb.maps)[2 * pb.map_cap - 2]; }
__device__ __forceinline__ uint32_t& slot_ne(const PathBuf& pb) { return ((uint32_t*)pb.maps)[2 * pb.map_cap - 1]; }

// faster_cap (minimizer_mapper.cpp:2946-3260); sequential FP64 (one thread).  The explored
// minimizers are packed into one 64-bit word each, sorted by (agglomeration end, start):
//   bits 0-15 agg_start, 16-31 agg_end, 32-47 forward_offset, 48-55 top byte of the hash
// `mp` needs room for the explored minimizers, `c` for one more double than that.
__device__ inline double faster_cap(const MapParamsDev& P, const DevMinimizer* mins, uint32_t k, const uint32_t* explored_mask, uint32_t M,
                                    const uint8_t* qual, uint32_t L, uint64_t* mp, double* c) {
    if (qual == nullptr) return INFINITY;
    uint32_t n = 0;
    for (uint32_t i = 0; i < M; i++) if (explored_mask[i >> 5] & (1u << (i & 31))) {
        // stable insertion by (agglomeration end, agglomeration start)
        const DevMinimizer dm = mins[i];
        const uint32_t as = dm.agg_start, ae = (uint32_t)dm.agg_start + dm.agg_len;
        const uint64_t wd = (uint64_t)as | ((uint64_t)ae << 16) | ((uint64_t)dm.fwd_offset << 32) | ((dm.hash >> 56) << 48);
        const uint32_t key = (ae << 16) | as;
        uint32_t j = n;
        while (j > 0) {
            const uint64_t o = mp[j - 1];
            const uint32_t okey = ((uint32_t)(o >> 16) << 16) | (uint32_t)(o & 0xffffu);
            if (key < okey) { mp[j] = o; j--; } else break;
        }
        mp[j] = wd; n++;
    }
    for (uint32_t i = 0; i <= n; i++) c[i] = -INFINITY;
    c[0] = 0.0;
    if (n == 0) return -c[n] * 10;
    auto column_prob = [&](uint32_t begin, uint32_t end, uint32_t index) {
        double p = P.phred_prob[qual[index]];
        for (uint32_t it = begin; it != end; ++it) {
            const uint64_t wd = mp[it];
            const uint32_t as = (uint32_t)wd & 0xffffu, ae = (uint32_t)(wd >> 16) & 0xffffu, fwd = (uint32_t)(wd >> 32) & 0xffffu;
            if (index - fwd >= k) {                                     // not inside the minimizer itself (unsigned: index < fwd wraps)
                const uint32_t possible = min(k, min(index - as + 1, ae - index));
                p *= P.prob_at_least_one[(possible << 8) + (uint32_t)(wd >> 48)];
            }
        }
        return p;
    };
    // for_each_agglomeration_interval (:3088-3161) turned inside out: the sweep ("stack" = window
    // [front, back) of mp) hands out one interval (left, right, bottom, top) at a time and the loop below
    // evaluates ONE read column per trip, so that the threads of a warp that run this for different reads
    // stay in step (the nested sweep / interval / column loops of the reference diverge badly under SIMT).
    // The floating-point operations and their order are those of the nested form.
    auto agg_start_of = [&](uint32_t it) { return (uint32_t)mp[it] & 0xffffu; };
    auto agg_end_of = [&](uint32_t it) { return (uint32_t)(mp[it] >> 16) & 0xffffu; };
    uint32_t front = 0, back = 1, left = agg_start_of(0), bottom = 0, it = 1;
    bool final_phase = n == 1;
    uint32_t pending_right = final_phase ? L : agg_start_of(1);       // emit_preceding(pending_right) in progress
    uint32_t col = 0, right = 0, ib = 0, itop = 0;
    double p = 0.0;
    bool open = false, first = true, done = false;
    auto close_interval = [&](double p_here) {
        const double pv = c[ib] + p_here;
        for (uint32_t i = ib + 1; i < itop + 1; i++) if (c[i] < pv) c[i] = pv;
    };
    while (true) {
        while (!open && !done) {
            if (left < pending_right) {
                const uint32_t stack_size = back - front, stack_top_end = agg_end_of(front);
                ib = bottom; itop = bottom + stack_size; col = left;
                if (stack_top_end <= pending_right) {
                    right = stack_top_end;
                    left = stack_size == 1 ? pending_right : stack_top_end;
                    bottom += 1; front++;
                } else { right = pending_right; left = pending_right; }
                if (col == right) close_interval(0.0);                 // empty interval (two agglomerations ending together)
                else { open = true; first = true; }
            } else if (final_phase) done = true;
            else {
                back++; it++;
                if (it < n) pending_right = agg_start_of(it); else { pending_right = L; final_phase = true; }
            }
        }
        if (done) break;
        const double col_p = column_prob(ib, itop, col);
        p = first ? col_p : (p + col_p - (p * col_p));
        first = false;
        col++;
        if (col == right) { close_interval(log10(p)); open = false; }
    }
    return -c[n] * 10;
}

// faster_cap for the warp-per-read kernels: the same sweep, all lanes in step (mp / c in shared memory),
// with the column probabilities of an interval evaluated 32 columns at a time and folded in column
// order (p + q - p q is not associative, so the fold stays sequential: every lane folds the shuffled
// values itself and all lanes hold the same p).  Bit-identical to faster_cap.
__device__ inline double faster_cap_warp(const MapParamsDev& P, const DevMinimizer* mins, uint32_t k, const uint32_t* explored_mask, uint32_t M,
                                         const uint8_t* qual, uint32_t L, uint64_t* mp, double* c) {
    if (qual == nullptr) return INFINITY;
    const int lane = lane_id();
    uint32_t n = 0;
    __syncwarp();                                  // mp / c reuse the DP columns: every lane is done with them
    if (lane == 0) {
#pragma unroll 1
        for (uint32_t i = 0; i < M; i++) if (explored_mask[i >> 5] & (1u << (i & 31))) {
            const DevMinimizer dm = mins[i];
            const uint32_t as = dm.agg_start, ae = (uint32_t)dm.agg_start + dm.agg_len;
            const uint64_t wd = (uint64_t)as | ((uint64_t)ae << 16) | ((uint64_t)dm.fwd_offset << 32) | ((dm.hash >> 56) << 48);
            const uint32_t key = (ae << 16) | as;
            uint32_t j = n;
#pragma unroll 1
            while (j > 0) {
                const uint64_t o = mp[j - 1];
                const uint32_t okey = ((uint32_t)(o >> 16) << 16) | (uint32_t)(o & 0xffffu);
                if (key < okey) { mp[j] = o; j--; } else break;
            }
            mp[j] = wd; n++;
        }
    }
    __syncwarp();                                  // lane 0's sorted words are visible to the warp
    n = __shfl_sync(FULL, n, 0);
#pragma unroll 1
    for (uint32_t i = lane; i <= n; i += 32) c[i] = i == 0 ? 0.0 : -INFINITY;
    __syncwarp();
    if (n == 0) { const double r0 = -c[n] * 10; __syncwarp(); return r0; }
    auto column_prob = [&](uint32_t begin, uint32_t end, uint32_t index) {
        double p = P.phred_prob[qual[index]];
#pragma unroll 1
        for (uint32_t it = begin; it != end; ++it) {
            const uint64_t wd = mp[it];
            const uint32_t as = (uint32_t)wd & 0xffffu, ae = (uint32_t)(wd >> 16) & 0xffffu, fwd = (uint32_t)(wd >> 32) & 0xffffu;
            if (index - fwd >= k) {
                const uint32_t possible = min(k, min(index - as + 1, ae - index));
                p *= P.prob_at_least_one[(possible << 8) + (uint32_t)(wd >> 48)];
            }
        }
        return p;
    };
    auto agg_start_of = [&](uint32_t it) { return (uint32_t)mp[it] & 0xffffu; };
    auto agg_end_of = [&](uint32_t it) { return (uint32_t)(mp[it] >> 16) & 0xffffu; };
    uint32_t front = 0, back = 1, left = agg_start_of(0), bottom = 0, it = 1;
    bool final_phase = n == 1;
    uint32_t pending_right = final_phase ? L : agg_start_of(1);
    // all lanes walk the sweep identically; lane 0 applies the updates of c
    auto close_interval = [&](uint32_t ib, uint32_t itop, double p_here) {
        __syncwarp();
        if (lane == 0) {
            const double pv = c[ib] + p_here;
#pragma unroll 1
            for (uint32_t i = ib + 1; i < itop + 1; i++) if (c[i] < pv) c[i] = pv;
        }
        __syncwarp();
    };
#pragma unroll 1
    while (true) {
        if (left < pending_right) {
            const uint32_t stack_size = back - front, stack_top_end = agg_end_of(front);
            const uint32_t ib = bottom, itop = bottom + stack_size, col0 = left;
            uint32_t right;
            if (stack_top_end <= pending_right) {
                right = stack_top_end;
                left = stack_size == 1 ? pending_right : stack_top_end;
                bottom += 1; front++;
            } else { right = pending_right; left = pending_right; }
            if (col0 == right) { close_interval(ib, itop, 0.0); continue; }
            double p = 0.0; bool first = true;
#pragma unroll 1
            for (uint32_t base = col0; base < right; base += 32) {
                const uint32_t idx = base + lane;
                const double cp = idx < right ? column_prob(ib, itop, idx) : 0.0;
                const uint32_t cnt = min(32u, right - base);
#pragma unroll 1
                for (uint32_t x = 0; x < cnt; x++) {
                    const double col_p = __shfl_sync(FULL, cp, x);
                    p = first ? col_p : (p + col_p - (p * col_p));
                    first = false;
                }
            }
            close_interval(ib, itop, log10(p));
        } else if (final_phase) break;
        else {
            back++; it++;
            if (it < n) pending_right = agg_start_of(it); else { pending_right = L; final_phase = true; }
        }
    }
    __syncwarp();
    const double result = -c[n] * 10;
    __syncwarp();                                  // the next call (the mate) rewrites mp / c
    return result;
}

// MappingQualityCalculator::compute_max_mapping_quality (exact), mapping_quality_calculator.cpp:26-67, :355-364, with
// the multiplicities of the scores when `mult` is given.  Returns the int32-truncated value as double.
__device__ inline double max_mapping_quality(const double* scores, uint32_t n, double log_base, const double* mult = nullptr) {
    const double quality_scale_factor = 10.0 / log(10.0);
    double log_sum_exp = -DBL_MAX, to_score = -DBL_MAX;
#pragma unroll 1
    for (int64_t i = (int64_t)n - 1; i >= 0; --i) {
        double score = log_base * scores[i];
        if (score >= to_score) to_score = score;
        if (mult && mult[i] > 1.0) score += log(mult[i]);
        log_sum_exp = d_add_log(log_sum_exp, score);
    }
    if (n == 1 && (!mult || mult[0] <= 1.0)) log_sum_exp = d_add_log(log_sum_exp, 0.0);
    const double direct = -quality_scale_factor * d_subtract_log(0.0, to_score - log_sum_exp);
    const double mq = isinf(direct) ? 2147483647.0 : direct;
    return (double)(int32_t)mq;
}

// Single-end MAPQ (:1146-1188): the explored cap (doubled past the escape threshold) and 60 bound the uncapped MAPQ.
// Fills the MAPQ fields of the primary record.
__device__ __forceinline__ void single_end_mapq(double mapq, double explored_cap, gb_alignment& out) {
    const double escape_bonus = mapq < 2147483647.0 ? 1.0 : 2.0;
    const double cap = escape_bonus * explored_cap;
    const double capped = round(fmin(cap, fmin(mapq, 60.0)));
    out.mapq = (uint8_t)fmax(fmin(capped, 60.0), 0.0);
    out.mapq_uncapped = (float)mapq; out.mapq_explored_cap = (float)cap;
}

// distance_between(aln1, aln2) (:3895-3903) of two finished candidate slots: initial_position(p0) -> final_position(p1)
__device__ __forceinline__ int64_t distance_between(const DevIndex& ix, const PathBuf& p0, const PathBuf& p1) {
    const gb_mapping first = p0.maps[0];
    const uint32_t nm1 = slot_nm(p1), ne1 = slot_ne(p1);
    const gb_mapping last = p1.maps[nm1 - 1];
    uint32_t used = 0;
#pragma unroll 1
    for (uint32_t x = ne1 - last.n_edits; x < ne1; x++) { const uint32_t wd = p1.edits[x]; const uint32_t op = wd & 3u; if (op != GB_EDIT_INS) used += (op == GB_EDIT_SUB) ? 1u : (wd >> 4); }
    return oriented_distance(ix, first.node, first.offset, last.node, (uint32_t)last.offset + used);
}

// score_alignment_pair (:6017-6028): both scores plus the fragment-length log-likelihood, never below the worse score
__device__ __forceinline__ double score_alignment_pair(int32_t s0, int32_t s1, int64_t dist, double frag_mean, double frag_sd, double log_base) {
    const double dev = (double)dist - frag_mean;
    const double ll = (-dev * dev / (2.0 * frag_sd * frag_sd)) / log_base;
    return fmax((double)s0 + (double)s1 + ll, fmin((double)s0, (double)s1));
}

// The fragment loop of map_paired (:2108-2208).  Candidates c < n have fragment frag(c), read read(c) (0 or 1) and score
// score(c).  In each fragment f < n_frag that holds both reads, every (read 0, read 1) combination becomes a pair, scored at
// distance dist(c0, c1); the candidates of the other fragments go to `unpaired`, read 0 first.  Returns false when the
// pairs do not fit in MAX_PAIRS.
template <uint32_t MAX_PAIRS, typename Frag, typename Read, typename Score, typename Dist>
__device__ __forceinline__ bool collect_pairs(uint32_t n, uint32_t n_frag, Frag frag, Read read, Score score, Dist dist,
                                              const uint8_t* better_cluster_count, double frag_mean, double frag_sd, double log_base,
                                              double* pair_score, int64_t* pair_dist, uint8_t* pair_c0, uint8_t* pair_c1, uint8_t* pair_better,
                                              uint32_t& n_pairs, bool& found_pair, uint8_t* unpaired, uint32_t& n_unpaired) {
    n_pairs = 0; found_pair = false; n_unpaired = 0;
#pragma unroll 1
    for (uint32_t f = 0; f < n_frag; f++) {
        bool has0 = false, has1 = false;
#pragma unroll 1
        for (uint32_t c = 0; c < n; c++) if (frag(c) == f) { if (read(c) == 0) has0 = true; else has1 = true; }
        if (has0 && has1) {
            found_pair = true;
#pragma unroll 1
            for (uint32_t c0 = 0; c0 < n; c0++) {
                if (frag(c0) != f || read(c0) != 0) continue;
#pragma unroll 1
                for (uint32_t c1 = 0; c1 < n; c1++) {
                    if (frag(c1) != f || read(c1) != 1) continue;
                    if (n_pairs >= MAX_PAIRS) return false;
                    const int64_t d = dist(c0, c1);
                    pair_score[n_pairs] = score_alignment_pair(score(c0), score(c1), d, frag_mean, frag_sd, log_base); pair_dist[n_pairs] = d;
                    pair_c0[n_pairs] = (uint8_t)c0; pair_c1[n_pairs] = (uint8_t)c1; pair_better[n_pairs] = better_cluster_count[f];
                    n_pairs++;
                }
            }
        } else {
#pragma unroll 1
            for (uint32_t r = 0; r < 2; r++)
#pragma unroll 1
                for (uint32_t c = 0; c < n; c++) if (frag(c) == f && read(c) == r) unpaired[n_unpaired++] = (uint8_t)c;
        }
    }
    return true;
}

// The best unpaired alignment of each end when no fragment holds a pair (:2216-2236): a LazyRNG coin flip decides a tie
// with the best so far.  best_c[r] = -1 when end r has none.
template <typename Read, typename Score>
__device__ __forceinline__ void best_unpaired_per_end(const uint8_t* unpaired, uint32_t n_unpaired, Read read, Score score, DevRng& rng,
                                                      int (&best_c)[2], int32_t (&best_score)[2]) {
    best_c[0] = best_c[1] = -1; best_score[0] = best_score[1] = 0;
#pragma unroll 1
    for (uint32_t u = 0; u < n_unpaired; u++) {
        const uint32_t c = unpaired[u], r = read(c);
        bool beats = score(c) > best_score[r];
        if (!beats && score(c) == best_score[r]) beats = (rng_next(rng) % 2) != 0;
        if (beats) { best_c[r] = (int)c; best_score[r] = score(c); }
    }
}

// MAPQ cap from the number of fragment clusters at least as good as the winning pair's, its own included (:2692-2697)
__device__ __forceinline__ double fragment_cluster_cap(uint32_t better_cluster_count) {
    return better_cluster_count > 1 ? -10.0 * log10(1.0 - (1.0 / (double)better_cluster_count)) : INFINITY;
}

// MAPQ of one read of the winning pair (:2727-2762): the fragment-cluster cap, the sum of both reads' explored caps
// (doubled past the escape threshold) and extra_cap (INFINITY: none) bound the pair's uncapped MAPQ, which is halved when
// the mates cannot reach each other and then split between the reads.  Fills the MAPQ fields of out once its flags are
// set: a read without GB_ALN_MAPPED gets 0.
__device__ __forceinline__ void pair_read_mapq(double uncapped, double cluster_cap, double caps_sum, bool unreachable, double extra_cap,
                                               gb_alignment& out) {
    const double escape_bonus = uncapped < 2147483647.0 ? 1.0 : 2.0;
    const double mapq_cap = fmin(fmin(cluster_cap, caps_sum * escape_bonus), extra_cap);
    double capped = fmin(mapq_cap, uncapped);
    if (unreachable) capped = capped / 2.0;
    const double read_mapq = (out.flags & GB_ALN_MAPPED) ? fmax(fmin(capped, 120.0) / 2.0, 0.0) : 0.0;
    out.mapq = (uint8_t)(int32_t)read_mapq;
    out.mapq_uncapped = (float)uncapped; out.mapq_explored_cap = (float)mapq_cap;
}

// Deferred cluster selection of read 2 of a pair (see cluster_phase_pe): the seeding kernel left every cluster of the read
// as a work item in comparator order with the keep-decision inputs in DevItem::fragment bits 8-10 and the length of the
// tied prefix in ReadState::pad[0].  Here, at the point of the per-read loop where the reference does it
// (minimizer_mapper.cpp:1780-1883, after read 1's alignments), the tied prefix is shuffled with the pair's LazyRNG and the
// order-dependent keep loop (process_until_threshold_c with its kept_cluster_count tests) picks the items.
// Returns false when the read is not deferred (sel untouched).
__device__ inline bool deferred_cluster_selection(const MapParamsDev& P, const ReadState& rs, const DevItem* items, DevRng& rng, uint8_t* sel, uint32_t& S) {
    const uint32_t ties = rs.pad[0];
    if (ties <= 1) return false;
    const uint32_t Cr = rs.item_cnt;
    uint8_t order[MAX_SETS];
#pragma unroll 1
    for (uint32_t i = 0; i < Cr; i++) order[i] = (uint8_t)i;
#pragma unroll 1
    for (uint32_t i = 1; i < ties && i < Cr; i++) { const uint32_t j = rng_next(rng) % (i + 1); const uint8_t t = order[j]; order[j] = order[i]; order[i] = t; }
    uint32_t unskipped = 0, kept_cluster_count = 0, nk = 0;
#pragma unroll 1
    for (uint32_t i = 0; i < Cr; i++) {
        if (unskipped >= P.max_extensions) continue;
        const uint32_t fl = items[rs.item_off + order[i]].fragment >> 8;
        bool keep = (fl & 1u) != 0;
        if (keep && (fl & 2u) && kept_cluster_count >= P.min_extensions) keep = false;
        else if (keep && (fl & 4u) && kept_cluster_count >= P.min_extensions) keep = false;
        if (keep) { sel[nk++] = order[i]; kept_cluster_count++; unskipped++; }
    }
    S = nk;
    return true;
}

struct CandList {
    int32_t score[2 * MAX_CANDS + 32];       // + rescued alignments
    uint8_t slot[2 * MAX_CANDS + 32];
    uint8_t frag[2 * MAX_CANDS + 32];
    uint8_t read[2 * MAX_CANDS + 32];
    uint32_t n;
};

// Turn the extension sets of one read into candidate alignments (appended to `cl`).
// paired = false: single-end rules (min_extension_sets, extension_set_min_score);
// paired = true:  process_until_threshold_b(..., 2, max_alignments) and fragment bookkeeping.
__device__ inline uint32_t align_sets(const DevIndex& ix, const MapParamsDev& P, const DevScores& sc, const ReadState& rs,
                                      const AlignArgs& a, const uint8_t* sread, uint32_t L, const TailWs& ws, DpSmem dps, uint8_t* qbuf,
                                      uint8_t* cand_base, bool* slot_used, DevRng& rng, bool paired, uint32_t read_num,
                                      CandList& cl, uint32_t* explored, uint32_t unit, uint8_t* stmp) {
    const int lane = lane_id();
    uint32_t status = GB_ITEM_OK;
    uint32_t S = rs.item_cnt;
    TailLookup tl; tl.pv = nullptr; tl.base = tl.count = tl.key = 0;
    if (a.plan.entries) { const uint32_t pb0 = a.plan.unit_base[unit]; if (pb0 != 0xffffffffu) { tl.pv = &a.plan; tl.base = pb0; tl.count = a.plan.unit_count[unit]; } }
    if (S > MAX_SETS) return GB_ITEM_OUT_FULL;
    uint8_t sel[MAX_SETS];                        // work items of this read in processing order (indices into its item list)
    if (!deferred_cluster_selection(P, rs, a.items, rng, sel, S)) for (uint32_t s = 0; s < S; s++) sel[s] = (uint8_t)s;
    const uint32_t map_cap = P.mapping_cap, edit_cap = P.edit_cap;
    auto alloc_slot = [&]() -> uint32_t {
#pragma unroll 1
        for (uint32_t i = 0; i < N_SLOTS; i++) if (!slot_used[i]) { slot_used[i] = true; return i; }
        return 0xffffffffu;
    };
#pragma unroll
    for (uint32_t x = 0; x < PRESENT_WORDS; x++) explored[x] = 0;

    int set_score[MAX_SETS]; uint8_t set_order[MAX_SETS];
#pragma unroll 1
    for (uint32_t s = 0; s < S; s++) {
        const uint32_t item = rs.item_off + sel[s];
        if (a.ev.ext_status[item] != GB_ITEM_OK) return a.ev.ext_status[item];
        set_score[s] = score_extension_group(ev_ext(a.ev, item), a.ev.ext_count[item], L, sc.gap_open, sc.gap_extend);
    }
    sort_shuffling_ties(S, [&](uint32_t x, uint32_t y) { return set_score[x] > set_score[y]; }, set_order, rng);
    const double set_cutoff = S == 0 ? 0.0 : (double)set_score[set_order[0]] - P.extension_set_score_threshold;
    const uint32_t min_sets = paired ? 2u : (uint32_t)P.min_extension_sets;
    uint32_t unskipped = 0;

    auto tmp_buf = [&](uint32_t k) { return stmp ? slot_buf(stmp, k, map_cap, edit_cap) : slot_buf(cand_base, N_SLOTS + k, map_cap, edit_cap); };
    PathBuf res_left = tmp_buf(0), res_right = tmp_buf(1), scratch = tmp_buf(2), middle = tmp_buf(3), asmb = tmp_buf(4);
    // a finished path leaves the assembly buffer for its candidate slot (the whole warp copies)
    auto store_slot = [&](PathBuf& dst, const PathBuf& src, uint32_t nm, uint32_t ne) {
#pragma unroll 1
        for (uint32_t i = lane; i < nm; i += 32) dst.maps[i] = src.maps[i];
#pragma unroll 1
        for (uint32_t i = lane; i < ne; i += 32) dst.edits[i] = src.edits[i];
        if (lane == 0) { slot_nm(dst) = nm; slot_ne(dst) = ne; }
        __syncwarp();
    };

#pragma unroll 1
    for (uint32_t oi = 0; oi < S && status == GB_ITEM_OK; oi++) {
        const uint32_t s = set_order[oi];
        bool process;
        if (P.extension_set_score_threshold != 0 && (double)set_score[s] <= set_cutoff) process = unskipped < min_sets;
        else process = unskipped < P.max_alignments;
        if (!process) continue;
        if (!paired && set_score[s] < P.extension_set_min_score) continue;           // single-end only (:912-916)
        unskipped++;
        const uint32_t item = rs.item_off + sel[s];
        const gb_extension* ext = ev_ext(a.ev, item);
        const uint32_t n_ext = a.ev.ext_count[item];
        const uint32_t* path_pool = ev_path(a.ev, item);
        const uint32_t* mism_pool = ev_mism(a.ev, item);
        const DevItem it = a.items[item];

        int32_t ba_score[50]; uint32_t ba_slot[50]; uint32_t n_ba = 0;
        if (n_ext > 0 && ext_full(ext[0]) && ext[0].mismatches <= 4) {
#pragma unroll 1
            for (uint32_t j = 0; j < n_ext && (j == 0 || ext_full(ext[j])) && n_ba < 49; j++) {
                const uint32_t slot = alloc_slot();
                if (slot == 0xffffffffu) { status = GB_ITEM_OUT_FULL; break; }
                PathBuf pb = slot_buf(cand_base, slot, map_cap, edit_cap);
                pb_reset(asmb);
                if (lane == 0) extension_to_path(ix, ext[j], path_pool, mism_pool, sread, asmb);
                __syncwarp();
                const uint32_t nm = __shfl_sync(FULL, asmb.n_maps, 0), ne = __shfl_sync(FULL, asmb.n_edits, 0);
                if (__shfl_sync(FULL, (int)asmb.overflow, 0) || nm + 1 > map_cap) { status = GB_ITEM_OUT_FULL; break; }
                store_slot(pb, asmb, nm, ne);
                ba_score[n_ba] = ext[j].score; ba_slot[n_ba] = slot; n_ba++;
            }
        } else if (P.do_dp) {
            // ---- find_optimal_tail_alignments (:5369-5622) -----------------------------------------
            uint32_t min_tails = 1;
#pragma unroll 1
            for (uint32_t j = 0; j < n_ext; j++) if (ext_full(ext[j])) min_tails++;
            if (min_tails < 2) min_tails = 2;
            Pareto lf[136], rf[136]; uint32_t nl = 0, nr = 0;
#pragma unroll 1
            for (uint32_t j = 0; j < n_ext && nl + 3 < 136; j++) {
                const gb_extension& e = ext[j];
                if (ext_full(e)) continue;
                const int32_t left_penalty = gap_penalty1(e.read_lo, sc);
                const int32_t mid_penalty = (int32_t)e.mism_len * (sc.match + sc.mismatch);
                const int32_t right_penalty = gap_penalty1(L - e.read_hi, sc);
                lf[nl++] = Pareto{e.read_hi, mid_penalty + left_penalty};
                rf[nr++] = Pareto{L - e.read_lo, mid_penalty + right_penalty};
                if (e.mism_len > 0) {
                    lf[nl++] = Pareto{mism_pool[e.mism_off], left_penalty};
                    rf[nr++] = Pareto{L - mism_pool[e.mism_off + e.mism_len - 1] - 1, right_penalty};
                }
            }
            lf[nl++] = Pareto{ix.k + ix.w - 2, 0}; rf[nr++] = Pareto{ix.k + ix.w - 2, 0};
            nl = find_pareto_frontier(lf, nl); nr = find_pareto_frontier(rf, nr);

            uint8_t eo[64]; const uint32_t ne_ = min(n_ext, 64u);
            sort_shuffling_ties(ne_, [&](uint32_t x, uint32_t y) { return ext[x].score > ext[y].score; }, eo, rng);
            const double ecut = ne_ == 0 ? 0.0 : (double)ext[eo[0]].score - (double)P.extension_score_threshold;
            uint32_t e_unskipped = 0;
            uint32_t win_slot = 0xffffffffu, sec_slot = 0xffffffffu;
            int32_t winning_score = 0, second_score = 0;
            int64_t winning_start = 0, winning_end = 0;
            bool partial_extension_aligned = false; int32_t threshold = -1;
#pragma unroll 1
            for (uint32_t xi = 0; xi < ne_ && status == GB_ITEM_OK; xi++) {
                const gb_extension& e = ext[eo[xi]];
                bool eproc;
                if (P.extension_score_threshold != 0 && (double)e.score <= ecut) eproc = e_unskipped < min_tails;
                else eproc = true;                                   // max_local_extensions = SIZE_MAX
                if (!eproc) continue;
                e_unskipped++;
                if (threshold < 0) threshold = e.score - P.extension_score_threshold;
                if (!ext_full(e)) {
                    if (partial_extension_aligned && e.score <= threshold) {
                        int32_t estimate = (int32_t)L * sc.match + 2 * sc.full_length_bonus - (int32_t)e.mism_len * (sc.match + sc.mismatch);
                        if (!(e.flags & GB_EXT_LEFT_FULL)) estimate -= flank_penalty(e.read_lo, lf, nl, sc);
                        if (!(e.flags & GB_EXT_RIGHT_FULL)) estimate -= flank_penalty(L - e.read_hi, rf, nr, sc);
                        if (estimate <= winning_score) continue;
                    }
                    partial_extension_aligned = true;
                }
                int32_t left_score = 0, right_score = 0;
                pb_reset(res_left); pb_reset(res_right);
                // one call site for both tails (left first): the forest / DP / traceback code exists once per kernel, so
                // warps working on different tails share the instruction cache (the align kernels are fetch-bound)
#pragma unroll 1
                for (uint32_t side = 0; side < 2 && status == GB_ITEM_OK; side++) {
                    const bool left_tail = side == 0;
                    if (e.flags & (left_tail ? GB_EXT_LEFT_FULL : GB_EXT_RIGHT_FULL)) continue;
                    PathBuf* res = left_tail ? &res_left : &res_right;
                    tl.key = tail_key(sel[s], read_num, eo[xi], left_tail);
                    const int32_t tail_score = align_tail(ix, P, sc, ws, dps, e, path_pool, sread, L, left_tail, qbuf, rng, *res, scratch, status, tl);
                    if (left_tail) left_score = tail_score; else right_score = tail_score;
                }
                if (status != GB_ITEM_OK) break;
                const int32_t total_score = e.score + left_score + right_score;
                const uint32_t first_node = path_pool[e.path_off], last_node = path_pool[e.path_off + e.path_len - 1];
                uint32_t ls = 0, re = 0;
                if (lane == 0) { ls = res_left.n_maps ? res_left.maps[0].node : first_node; re = res_right.n_maps ? res_right.maps[res_right.n_maps - 1].node : last_node; }
                ls = __shfl_sync(FULL, ls, 0); re = __shfl_sync(FULL, re, 0);
                const int64_t current_start = ls >> 1, current_end = re >> 1;
                const int64_t w_start = winning_score == 0 ? 0 : winning_start, w_end = winning_score == 0 ? 0 : winning_end;
                const bool different_left = w_start != current_start, different_right = w_end != current_end;
                int target = 0;      // 1: becomes winner, 2: becomes second
                if (total_score > winning_score || winning_score == 0) {
                    if (winning_score != 0 && different_left && different_right) {
                        if (sec_slot != 0xffffffffu) slot_used[sec_slot] = false;
                        second_score = winning_score; sec_slot = win_slot; win_slot = 0xffffffffu;
                    }
                    target = 1;
                } else if ((total_score > second_score || second_score == 0) && different_left && different_right) {
                    target = 2;
                }
                if (target) {
                    uint32_t& dst = target == 1 ? win_slot : sec_slot;
                    if (dst != 0xffffffffu) slot_used[dst] = false;
                    dst = alloc_slot();
                    if (dst == 0xffffffffu) { status = GB_ITEM_OUT_FULL; break; }
                    PathBuf pb = slot_buf(cand_base, dst, map_cap, edit_cap);
                    pb_reset(asmb);
                    if (lane == 0) {
                        pb_reset(middle);
                        extension_to_path(ix, e, path_pool, mism_pool, sread, middle);
                        add_to_path(asmb, res_left.maps, res_left.edits, res_left.n_maps);
                        add_to_path(asmb, middle.maps, middle.edits, middle.n_maps);
                        add_to_path(asmb, res_right.maps, res_right.edits, res_right.n_maps);
                        if (middle.overflow || asmb.n_maps + 1 > map_cap) asmb.overflow = true;
                    }
                    __syncwarp();
                    if (__shfl_sync(FULL, (int)asmb.overflow, 0)) { status = GB_ITEM_OUT_FULL; break; }
                    store_slot(pb, asmb, __shfl_sync(FULL, asmb.n_maps, 0), __shfl_sync(FULL, asmb.n_edits, 0));
                    if (target == 1) { winning_score = total_score; winning_start = current_start; winning_end = current_end; }
                    else second_score = total_score;
                }
            }
            if (status != GB_ITEM_OK) break;
            ba_score[0] = winning_score; ba_slot[0] = win_slot; ba_score[1] = second_score; ba_slot[1] = sec_slot; n_ba = 2;
        }
        if (status != GB_ITEM_OK) break;
        // keep alignments with score != 0 and >= 0.8 * best (:1025-1028, :2008-2011)
        bool keep = true;
#pragma unroll 1
        for (uint32_t j = 0; j < n_ba; j++) {
            if (keep && ba_score[j] != 0 && (double)ba_score[j] >= (double)ba_score[0] * 0.8) {
                if (cl.n >= 2 * MAX_CANDS || (cl.n >= MAX_CANDS && !paired)) { status = GB_ITEM_OUT_FULL; break; }
                cl.score[cl.n] = ba_score[j]; cl.slot[cl.n] = (uint8_t)ba_slot[j]; cl.frag[cl.n] = (uint8_t)it.fragment; cl.read[cl.n] = (uint8_t)read_num;
                cl.n++;
            } else {
                keep = false;
                if (ba_slot[j] != 0xffffffffu) slot_used[ba_slot[j]] = false;
            }
        }
#pragma unroll
        for (uint32_t x = 0; x < PRESENT_WORDS; x++) explored[x] |= it.present[x];
    }
    return status;
}

// Copy a finished candidate to the output pools.  Substitution bases are (re)read from the read
// so both strands follow the Edit.sequence rule.  rc = true applies
// reverse_complement_alignment_in_place (alignment.cpp:3338) for mate 2: `sread` is then the
// rightward (reverse-complemented) read the path was computed on.
__device__ inline void write_alignment(const DevIndex& ix, const PathBuf& pb, uint32_t nm, uint32_t ne, const uint8_t* sread, uint32_t L, bool rc,
                                       gb_mapping* out_maps, uint32_t* out_edits) {
    if (!rc) {
        uint32_t qoff = 0, e = 0;
#pragma unroll 1
        for (uint32_t i = 0; i < nm; i++) {
            out_maps[i] = pb.maps[i];
#pragma unroll 1
            for (uint32_t x = 0; x < pb.maps[i].n_edits; x++, e++) {
                uint32_t wd = pb.edits[e]; const uint32_t op = wd & 3u, len = wd >> 4;
                if (op == GB_EDIT_SUB) { wd = (1u << 4) | (base2(sread[qoff]) << 2) | GB_EDIT_SUB; qoff += 1; }
                else if (op == GB_EDIT_MATCH || op == GB_EDIT_INS) qoff += len;
                out_edits[e] = wd;
            }
        }
    } else {
        // walk mappings backwards; query offsets count from the end of the rightward read
        uint32_t e_end = ne, qend = L, w = 0;
        // total query length consumed equals L (softclips included)
#pragma unroll 1
        for (int64_t i = (int64_t)nm - 1; i >= 0; i--) {
            const gb_mapping m = pb.maps[i];
            const uint32_t e_begin = e_end - m.n_edits;
            uint32_t used = 0;
#pragma unroll 1
            for (uint32_t x = e_begin; x < e_end; x++) { const uint32_t wd = pb.edits[x]; const uint32_t op = wd & 3u; if (op != GB_EDIT_INS) used += (op == GB_EDIT_SUB) ? 1u : (wd >> 4); }
            gb_mapping o; o.node = m.node ^ 1u; o.offset = (uint16_t)(load_node(ix, m.node).len - used - m.offset); o.n_edits = m.n_edits;
            out_maps[nm - 1 - (uint32_t)i] = o;
#pragma unroll 1
            for (int64_t x = (int64_t)e_end - 1; x >= (int64_t)e_begin; x--) {
                uint32_t wd = pb.edits[x]; const uint32_t op = wd & 3u, len = wd >> 4;
                if (op == GB_EDIT_SUB) {
                    // the substituted base in input orientation = complement of the rightward read base
                    const uint8_t c = sread[qend - 1];
                    wd = (1u << 4) | (base2(comp_base(c)) << 2) | GB_EDIT_SUB; qend -= 1;
                    if (!is_acgt(c)) wd = (1u << 4) | GB_EDIT_SUB;
                } else if (op == GB_EDIT_MATCH || op == GB_EDIT_INS) qend -= len;
                out_edits[w++] = wd;
            }
            e_end = e_begin;
        }
    }
}

// ---- single-end: winner (process_until_threshold_a, :1095), MAPQ (:1146-1188), record -------------------
__device__ inline uint32_t finalize_se(const DevIndex& ix, const MapParamsDev& P, const ReadState& rs, const AlignArgs& a,
                                       const CandList& cl, const uint32_t* explored, DevRng& rng, const uint8_t* sread, const uint8_t* qual,
                                       uint32_t L, uint32_t read_idx, DpSmem dps, uint8_t* cand_base,
                                       gb_alignment& out, gb_mapping* out_maps, uint32_t* out_edits) {
    const int lane = lane_id();
    const uint32_t map_cap = P.mapping_cap, edit_cap = P.edit_cap;
    double scores_sorted[MAX_CANDS + 1];
    uint32_t n_scores = 0; uint32_t win = 0xffffffffu;
    uint8_t co[MAX_CANDS];
    if (cl.n == 0) { scores_sorted[0] = 0.0; n_scores = 1; }
    else {
        sort_shuffling_ties(cl.n, [&](uint32_t x, uint32_t y) { return cl.score[x] > cl.score[y]; }, co, rng);
#pragma unroll 1
        for (uint32_t c = 0; c < cl.n; c++) scores_sorted[c] = (double)cl.score[co[c]];
        n_scores = cl.n; win = co[0];
    }
    double mapq = 0.0;
    if (win != 0xffffffffu) mapq = max_mapping_quality(scores_sorted, n_scores, P.log_base);
    double* cbuf = reinterpret_cast<double*>(dps.Hp);       // DP columns are free here (Hp|Ep and Hc|Ec)
    uint64_t* ordbuf = reinterpret_cast<uint64_t*>(dps.Hc);
    const double cap = faster_cap_warp(P, a.minimizers + rs.min_off, ix.k, explored, rs.min_cnt, qual, L, ordbuf, cbuf);

    out.read_id = read_idx; out.score = 0; out.flags = 0; out.n_mappings = 0; out.n_edits = 0;
    single_end_mapq(mapq, cap, out);
    if (win != 0xffffffffu) {
        PathBuf pb = slot_buf(cand_base, cl.slot[win], map_cap, edit_cap);
        const uint32_t nm = slot_nm(pb), ne = slot_ne(pb);
        if (nm + 1 > map_cap || ne > edit_cap) return GB_ITEM_OUT_FULL;
        out.score = cl.score[win]; out.flags = nm ? GB_ALN_MAPPED : 0; out.n_mappings = (uint16_t)nm; out.n_edits = ne;
        if (lane == 0) write_alignment(ix, pb, nm, ne, sread, L, false, out_maps, out_edits);
    }
    // mappings 1 .. max_multimaps - 1 in the same order (:1095-1130, :1199-1206): secondaries, no MAPQ of their own
#pragma unroll 1
    for (uint32_t j = 1; j < P.max_multimaps && j < cl.n; j++) {
        const uint32_t c = co[j];
        PathBuf pb = slot_buf(cand_base, cl.slot[c], map_cap, edit_cap);
        const uint32_t nm = slot_nm(pb), ne = slot_ne(pb);
        if (nm + 1 > map_cap || ne > edit_cap) return GB_ITEM_OUT_FULL;
        const size_t R = (size_t)j * P.out_stride + read_idx;
        if (lane == 0) {
            gb_alignment sec;
            sec.read_id = read_idx; sec.score = cl.score[c]; sec.mapq = 0; sec.flags = (nm ? GB_ALN_MAPPED : 0) | GB_ALN_SECONDARY;
            sec.n_mappings = (uint16_t)nm; sec.n_edits = ne; sec.mapping_off = (uint32_t)(R * map_cap); sec.edit_off = (uint32_t)(R * edit_cap);
            sec.mapq_uncapped = 0.f; sec.mapq_explored_cap = 0.f;
            write_alignment(ix, pb, nm, ne, sread, L, false, a.maps + R * map_cap, a.edits + R * edit_cap);
            a.aln[R] = sec;
        }
    }
    __syncwarp();
    return GB_ITEM_OK;
}

// Pairs 1 .. max_multimaps - 1 of a pair in output order (:2505-2598): both reads of such a pair are secondary
// (:2552-2557) and carry no MAPQ.  Records of rank j live at j * P.out_stride + read.  rescue_frag = the fragment slot of
// rescued alignments (0xffffffff: none).  Capacities are checked before anything is written.
__device__ inline uint32_t write_secondary_pairs(const DevIndex& ix, const MapParamsDev& P, const AlignArgs& a, const CandList& cl,
                                                 const uint8_t* po, uint32_t n_pairs, const uint8_t* pair_c0, const uint8_t* pair_c1, uint32_t rescue_frag,
                                                 const uint8_t* const* sread, const uint32_t* L, uint32_t read_idx0, uint8_t* cand_base) {
    const int lane = lane_id();
    const uint32_t map_cap = P.mapping_cap, edit_cap = P.edit_cap;
    const uint32_t n_out = min(P.max_multimaps, n_pairs);
#pragma unroll 1
    for (uint32_t pass = 0; pass < 2; pass++) {
#pragma unroll 1
        for (uint32_t j = 1; j < n_out; j++) {
#pragma unroll 1
            for (uint32_t r = 0; r < 2; r++) {
                const uint32_t c = r == 0 ? pair_c0[po[j]] : pair_c1[po[j]];
                PathBuf pb = slot_buf(cand_base, cl.slot[c], map_cap, edit_cap);
                const uint32_t nm = slot_nm(pb), ne = slot_ne(pb);
                if (pass == 0) { if (nm + 1 > map_cap || ne > edit_cap) return GB_ITEM_OUT_FULL; continue; }
                const size_t R = (size_t)j * P.out_stride + read_idx0 + r;
                if (lane == 0) {
                    gb_alignment sec;
                    sec.read_id = read_idx0 + r; sec.score = cl.score[c]; sec.mapq = 0;
                    sec.flags = GB_ALN_PAIRED | GB_ALN_SECONDARY | (nm ? GB_ALN_MAPPED : 0) | (cl.frag[c] == rescue_frag ? GB_ALN_RESCUED : 0);
                    sec.n_mappings = (uint16_t)nm; sec.n_edits = ne; sec.mapping_off = (uint32_t)(R * map_cap); sec.edit_off = (uint32_t)(R * edit_cap);
                    sec.mapq_uncapped = 0.f; sec.mapq_explored_cap = 0.f;
                    if (nm) write_alignment(ix, pb, nm, ne, sread[r], L[r], r == 1, a.maps + R * map_cap, a.edits + R * edit_cap);
                    a.aln[R] = sec;
                }
            }
        }
    }
    __syncwarp();
    return GB_ITEM_OK;
}

// ---- paired-end: pairing, winner, MAPQ, two records (max_rescue_attempts = 0) ------------------------------------
__device__ inline uint32_t finalize_pe(const DevIndex& ix, const MapParamsDev& P, const ReadState* rs /*[2]*/, const PairState& ps,
                                       const AlignArgs& a, const CandList& cl, const uint32_t (*explored)[PRESENT_WORDS], DevRng& rng,
                                       const uint8_t* const* sread, const uint8_t* const* qual, const uint32_t* L, uint32_t read_idx0,
                                       DpSmem dps, uint8_t* cand_base, gb_alignment* out /*[2]*/, gb_mapping* const* out_maps, uint32_t* const* out_edits) {
    const int lane = lane_id();
    const uint32_t map_cap = P.mapping_cap, edit_cap = P.edit_cap;
#pragma unroll 1
    for (uint32_t r = 0; r < 2; r++) {
        out[r].read_id = read_idx0 + r; out[r].score = 0; out[r].mapq = 0; out[r].flags = GB_ALN_PAIRED; out[r].n_mappings = 0; out[r].n_edits = 0;
        out[r].mapq_uncapped = 0.f; out[r].mapq_explored_cap = 0.f;
    }
    // alignments[fragment][read] in insertion order == candidate order filtered by (fragment, read)
    const uint32_t n_frag_slots = ps.n_fragments + 1;     // + the (empty, no rescue) extra entry
    constexpr uint32_t MAX_PAIRS = 64;
    double pair_score[MAX_PAIRS]; int64_t pair_dist[MAX_PAIRS]; uint8_t pair_c0[MAX_PAIRS], pair_c1[MAX_PAIRS], pair_better[MAX_PAIRS];
    uint32_t n_pairs, n_unpaired; bool found_pair;
    uint8_t unpaired[2 * MAX_CANDS];
    auto frag_of = [&](uint32_t c) { return (uint32_t)cl.frag[c]; };
    auto read_of = [&](uint32_t c) { return (uint32_t)cl.read[c]; };
    auto score_of = [&](uint32_t c) { return cl.score[c]; };
    auto dist_of = [&](uint32_t c0, uint32_t c1) {
        return distance_between(ix, slot_buf(cand_base, cl.slot[c0], map_cap, edit_cap), slot_buf(cand_base, cl.slot[c1], map_cap, edit_cap));
    };
    if (!collect_pairs<MAX_PAIRS>(cl.n, n_frag_slots, frag_of, read_of, score_of, dist_of, ps.better_cluster_count, a.frag_mean, a.frag_sd, P.log_base,
                                  pair_score, pair_dist, pair_c0, pair_c1, pair_better, n_pairs, found_pair, unpaired, n_unpaired))
        return GB_ITEM_OUT_FULL;
    if (n_unpaired > 0 && P.max_rescue_attempts != 0) return GB_ITEM_RETRY;     // needs mate rescue: the rescue kernel redoes this pair

    if (n_unpaired > 0 && !found_pair) {
        // max_rescue_attempts == 0 (:2237-2287): best alignment of each end, MAPQ 1
        int best_c[2]; int32_t best_score[2];
        best_unpaired_per_end(unpaired, n_unpaired, read_of, score_of, rng, best_c, best_score);
#pragma unroll 1
        for (uint32_t r = 0; r < 2; r++) {
            out[r].mapq = 1;
            if (best_c[r] >= 0) {
                PathBuf pb = slot_buf(cand_base, cl.slot[best_c[r]], map_cap, edit_cap);
                const uint32_t nm = slot_nm(pb), ne = slot_ne(pb);
                out[r].score = cl.score[best_c[r]]; out[r].flags |= nm ? GB_ALN_MAPPED : 0; out[r].n_mappings = (uint16_t)nm; out[r].n_edits = ne;
                if (lane == 0) write_alignment(ix, pb, nm, ne, sread[r], L[r], r == 1, out_maps[r], out_edits[r]);
            }
        }
        __syncwarp();
        return GB_ITEM_OK;
    }
    if (n_pairs == 0) return GB_ITEM_OK;     // both unmapped

    // winner (:2505-2598)
    uint8_t po[MAX_PAIRS];
    sort_shuffling_ties(n_pairs, [&](uint32_t x, uint32_t y) { return pair_score[x] > pair_score[y]; }, po, rng);
    double scores_sorted[MAX_PAIRS];
#pragma unroll 1
    for (uint32_t p = 0; p < n_pairs; p++) scores_sorted[p] = pair_score[po[p]];
    const uint32_t wp = po[0];
    const double uncapped_mapq = scores_sorted[0] == 0 ? 0.0 : max_mapping_quality(scores_sorted, n_pairs, P.log_base);
    const double cluster_cap = fragment_cluster_cap(pair_better[wp]);
    double caps[2] = {0.0, 0.0};
    double* cbuf = reinterpret_cast<double*>(dps.Hp);
    uint64_t* ordbuf = reinterpret_cast<uint64_t*>(dps.Hc);
#pragma unroll 1
    for (uint32_t r = 0; r < 2; r++) caps[r] = faster_cap_warp(P, a.minimizers + rs[r].min_off, ix.k, explored[r], rs[r].min_cnt, qual[r], L[r], ordbuf, cbuf);
    const uint32_t cwin[2] = {pair_c0[wp], pair_c1[wp]};
#pragma unroll 1
    for (uint32_t r = 0; r < 2; r++) {
        PathBuf pb = slot_buf(cand_base, cl.slot[cwin[r]], map_cap, edit_cap);
        const uint32_t nm = slot_nm(pb), ne = slot_ne(pb);
        out[r].score = cl.score[cwin[r]]; out[r].flags |= nm ? GB_ALN_MAPPED : 0; out[r].n_mappings = (uint16_t)nm; out[r].n_edits = ne;
        pair_read_mapq(uncapped_mapq, cluster_cap, caps[0] + caps[1], pair_dist[wp] == INT64_MAX, INFINITY, out[r]);
        if (lane == 0) write_alignment(ix, pb, nm, ne, sread[r], L[r], r == 1, out_maps[r], out_edits[r]);
    }
    __syncwarp();
    if (P.max_multimaps > 1) return write_secondary_pairs(ix, P, a, cl, po, n_pairs, pair_c0, pair_c1, 0xffffffffu, sread, L, read_idx0, cand_base);
    return GB_ITEM_OK;
}

// single-end driver kept for the SE align kernel
__device__ inline uint32_t align_read(const DevIndex& ix, const MapParamsDev& P, const DevScores& sc, ReadState rs,
                                      const AlignArgs& a, const uint8_t* sread, const uint8_t* qual, uint32_t L, uint32_t read_idx,
                                      const TailWs& ws, DpSmem dps, uint8_t* qbuf, uint8_t* cand_base,
                                      gb_alignment& out, gb_mapping* out_maps, uint32_t* out_edits, uint8_t* stmp) {
    DevRng rng = rs.rng;
    bool slot_used[N_SLOTS];
#pragma unroll 1
    for (uint32_t i = 0; i < N_SLOTS; i++) slot_used[i] = false;
    CandList cl; cl.n = 0;
    uint32_t explored[PRESENT_WORDS];
    uint32_t status = align_sets(ix, P, sc, rs, a, sread, L, ws, dps, qbuf, cand_base, slot_used, rng, false, 0, cl, explored, read_idx, stmp);
    if (status != GB_ITEM_OK) return status;
    return finalize_se(ix, P, rs, a, cl, explored, rng, sread, qual, L, read_idx, dps, cand_base, out, out_maps, out_edits);
}
