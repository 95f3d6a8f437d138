// align_fast.cuh — thread-per-pair fast path of the paired-end align stage (included by map.cu
// inside namespace gb).
//
// On clean short reads almost every extension set is a full-length gapless extension, so the
// align stage is pure bookkeeping (set selection, to_path, pairing, FP64 MAPQ + explored cap):
// sequential per pair, identical across pairs.  One THREAD per pair runs it here, so a warp retires
// 32 pairs in lock step instead of idling 31 lanes; any pair that needs tail alignment (a non
// full-length set is selected) or exceeds the small per-thread tables is appended to a work list
// and handled, from scratch, by the warp-per-pair kernel (align_kernel_pe), which produces the
// same bits (both follow minimizer_mapper.cpp:1904-2777 and share their helper functions).
#pragma once

constexpr uint32_t FAST_MAX_SETS = 8;
constexpr uint32_t FAST_MAX_CANDS = 12;     // per pair (both mates)
constexpr uint32_t FAST_MAX_PAIRS = 16;
constexpr uint32_t FAST_MAX_EXPLORED = 64;

struct FastCand { int32_t score; uint32_t item; uint8_t ext_j, frag, read; };

// Write a full-length extension as the output alignment of a read (thread-level to_path +
// optional reverse_complement_alignment_in_place for mate 2).  `read` is the rightward read.
__device__ inline bool extension_to_output(const DevIndex& ix, const gb_extension& e, const uint32_t* path_pool, const uint32_t* mism_pool,
                                           const uint8_t* read, uint32_t L, bool rc, gb_mapping* out_maps, uint32_t* out_edits,
                                           uint32_t map_cap, uint32_t edit_cap, uint32_t& nm_out, uint32_t& ne_out) {
    // forward pass over the path: per mapping (node, offset, edit run); edits: match runs + 1-bp subs
    if (e.path_len + 1 > map_cap) return false;
    uint32_t nm = 0, ne = 0;
    if (!rc) {
        uint32_t mi = 0, read_offset = e.read_lo, node_offset = e.offset;
        for (uint32_t i = 0; i < e.path_len; i++) {
            const uint32_t h = path_pool[e.path_off + i];
            const uint32_t nlen = load_node(ix, h).len;
            const uint32_t limit = min(read_offset + nlen - node_offset, e.read_hi);
            gb_mapping m; m.node = h; m.offset = (uint16_t)node_offset; m.n_edits = 0;
            while (mi < e.mism_len && mism_pool[e.mism_off + mi] < limit) {
                const uint32_t mp = mism_pool[e.mism_off + mi];
                if (ne + 2 > edit_cap) return false;
                if (read_offset < mp) { out_edits[ne++] = edit_word(GB_EDIT_MATCH, mp - read_offset, 0); m.n_edits++; }
                out_edits[ne++] = edit_word(GB_EDIT_SUB, 1, base2(read[mp])); m.n_edits++;
                read_offset = mp + 1; mi++;
            }
            if (read_offset < limit) { if (ne + 1 > edit_cap) return false; out_edits[ne++] = edit_word(GB_EDIT_MATCH, limit - read_offset, 0); m.n_edits++; read_offset = limit; }
            out_maps[nm++] = m;
            node_offset = 0;
        }
    } else {
        // reversed: last path node first, offsets measured from the other node end, edits reversed,
        // substituted bases complemented (input orientation of mate 2)
        const uint32_t span = e.read_hi - e.read_lo;
        uint32_t before_last = 0;
        for (uint32_t i = 0; i + 1 < e.path_len; i++) before_last += load_node(ix, path_pool[e.path_off + i]).len - (i == 0 ? e.offset : 0u);
        uint32_t re = e.read_hi;
        int64_t x = (int64_t)e.mism_len - 1;
        for (int64_t i = (int64_t)e.path_len - 1; i >= 0; i--) {
            const uint32_t h = path_pool[e.path_off + i];
            const uint32_t nlen = load_node(ix, h).len;
            const uint32_t no = i == 0 ? e.offset : 0u;
            const uint32_t used = (uint32_t)i + 1 == e.path_len ? span - before_last : nlen - no;
            const uint32_t rb = re - used;
            gb_mapping m; m.node = h ^ 1u; m.offset = (uint16_t)(nlen - used - no); m.n_edits = 0;
            uint32_t cursor = re;
            while (x >= 0 && mism_pool[e.mism_off + x] >= rb) {
                const uint32_t mp = mism_pool[e.mism_off + x];
                if (ne + 2 > edit_cap) return false;
                if (mp + 1 < cursor) { out_edits[ne++] = edit_word(GB_EDIT_MATCH, cursor - (mp + 1), 0); m.n_edits++; }
                const uint8_t c = read[mp];
                out_edits[ne++] = is_acgt(c) ? edit_word(GB_EDIT_SUB, 1, base2(comp_base(c))) : edit_word(GB_EDIT_SUB, 1, 0); m.n_edits++;
                cursor = mp; x--;
            }
            if (rb < cursor) { if (ne + 1 > edit_cap) return false; out_edits[ne++] = edit_word(GB_EDIT_MATCH, cursor - rb, 0); m.n_edits++; }
            out_maps[nm++] = m;
            re = rb;
        }
    }
    nm_out = nm; ne_out = ne;
    return true;
}

// initial_position / final_position of a full-length extension (path.cpp:2466-2487)
__device__ inline void extension_ends(const DevIndex& ix, const gb_extension& e, const uint32_t* path_pool,
                                      uint32_t& first_node, uint32_t& first_off, uint32_t& last_node, uint32_t& last_end) {
    first_node = path_pool[e.path_off]; first_off = e.offset;
    uint32_t tail = e.offset + (e.read_hi - e.read_lo);
    for (uint32_t i = 0; i + 1 < e.path_len; i++) tail -= load_node(ix, path_pool[e.path_off + i]).len;
    last_node = path_pool[e.path_off + e.path_len - 1]; last_end = tail;
}

// Returns true when the pair was fully handled (outputs written), false when it must go to the
// warp-per-pair kernel.
__device__ inline bool fast_pair(const DevIndex& ix, const MapParamsDev& P, const DevScores& sc, const MapBatch& b, const AlignArgs& a, uint32_t p) {
    const ReadState rs0 = b.states[2 * p], rs1 = b.states[2 * p + 1];
    const ReadState* rsp[2] = {&rs0, &rs1};
    if (rs0.status != GB_ITEM_OK) return false;                 // let the slow kernel report it
    if (P.max_multimaps > 1) return false;                      // secondaries are written by the warp kernels only
    if (rs1.pad[0] > 1) return false;                           // deferred cluster selection of read 2 (rare: tied clusters): warp kernel
    const PairState ps = a.pairs[p];
    if (ps.n_fragments + 1 > MAX_FRAGMENTS) return false;
    DevRng rng = rs0.rng;
    FastCand cand[FAST_MAX_CANDS]; uint32_t n_cand = 0;
    uint32_t explored[2][PRESENT_WORDS];
    uint32_t L[2];
    const uint8_t* reads[2]; const uint8_t* quals[2];
    for (uint32_t r = 0; r < 2; r++) {
        const uint64_t rb = b.read_off[2 * p + r];
        L[r] = (uint32_t)(b.read_off[2 * p + r + 1] - rb);
        reads[r] = b.reads + rb; quals[r] = b.quals ? b.quals + rb : nullptr;
#pragma unroll
        for (uint32_t x = 0; x < PRESENT_WORDS; x++) explored[r][x] = 0;
    }
    for (uint32_t r = 0; r < 2; r++) {
        const ReadState& rs = *rsp[r];
        const uint32_t S = rs.item_cnt;
        if (S > FAST_MAX_SETS) return false;
        int set_score[FAST_MAX_SETS]; uint8_t set_order[FAST_MAX_SETS];
        for (uint32_t s = 0; s < S; s++) {
            const uint32_t item = rs.item_off + s;
            if (a.ev.ext_status[item] != GB_ITEM_OK) return false;
            const gb_extension* ext = ev_ext(a.ev, item);
            const uint32_t n_ext = a.ev.ext_count[item];
            // full-length sets carry their own score; anything else needs the sweep estimate (rare)
            if (n_ext > 0 && ext_full(ext[0]) && ext[0].mismatches <= 4) set_score[s] = ext[0].score;
            else set_score[s] = score_extension_group(ext, n_ext, L[r], sc.gap_open, sc.gap_extend);
        }
        sort_shuffling_ties(S, [&](uint32_t x, uint32_t y) { return set_score[x] > set_score[y]; }, set_order, rng);
        const double set_cutoff = S == 0 ? 0.0 : (double)set_score[set_order[0]] - P.extension_set_score_threshold;
        uint32_t unskipped = 0;
        for (uint32_t oi = 0; oi < S; oi++) {
            const uint32_t s = set_order[oi];
            bool process;
            if (P.extension_set_score_threshold != 0 && (double)set_score[s] <= set_cutoff) process = unskipped < 2u;
            else process = unskipped < P.max_alignments;
            if (!process) continue;
            unskipped++;
            const uint32_t item = rs.item_off + s;
            const gb_extension* ext = ev_ext(a.ev, item);
            const uint32_t n_ext = a.ev.ext_count[item];
            if (!(n_ext > 0 && ext_full(ext[0]) && ext[0].mismatches <= 4)) return false;     // tail alignment needed
            const DevItem it = a.items[item];
            const int32_t best0 = ext[0].score;
            bool keep = true;
            for (uint32_t j = 0; j < n_ext && (j == 0 || ext_full(ext[j])); j++) {
                if (keep && ext[j].score != 0 && (double)ext[j].score >= (double)best0 * 0.8) {
                    if (n_cand >= FAST_MAX_CANDS) return false;
                    cand[n_cand++] = FastCand{ext[j].score, item, (uint8_t)j, (uint8_t)it.fragment, (uint8_t)r};
                } else keep = false;
            }
#pragma unroll
            for (uint32_t x = 0; x < PRESENT_WORDS; x++) explored[r][x] |= it.present[x];
        }
    }

    // ---- pairing (:2108-2208) -----------------------------------------------------------------------
    gb_alignment out[2];
    for (uint32_t r = 0; r < 2; r++) {
        const uint32_t ri = 2 * p + r;
        out[r].read_id = ri; out[r].score = 0; out[r].mapq = 0; out[r].flags = GB_ALN_PAIRED; out[r].n_mappings = 0; out[r].n_edits = 0;
        out[r].mapping_off = ri * P.mapping_cap; out[r].edit_off = ri * P.edit_cap; out[r].mapq_uncapped = 0.f; out[r].mapq_explored_cap = 0.f;
    }
    gb_mapping* out_maps[2] = {a.maps + (size_t)(2 * p) * P.mapping_cap, a.maps + (size_t)(2 * p + 1) * P.mapping_cap};
    uint32_t* out_edits[2] = {a.edits + (size_t)(2 * p) * P.edit_cap, a.edits + (size_t)(2 * p + 1) * P.edit_cap};
    auto ext_of = [&](const FastCand& c) -> const gb_extension& { return ev_ext(a.ev, c.item)[c.ext_j]; };
    auto write_cand = [&](uint32_t r, const FastCand& c) -> bool {
        uint32_t nm = 0, ne = 0;
        const bool ok = extension_to_output(ix, ext_of(c), ev_path(a.ev, c.item), ev_mism(a.ev, c.item),
                                            reads[r], L[r], r == 1, out_maps[r], out_edits[r], P.mapping_cap, P.edit_cap, nm, ne);
        if (!ok) return false;
        out[r].score = c.score; out[r].flags |= nm ? GB_ALN_MAPPED : 0; out[r].n_mappings = (uint16_t)nm; out[r].n_edits = ne;
        return true;
    };
    double pair_score[FAST_MAX_PAIRS]; int64_t pair_dist[FAST_MAX_PAIRS]; uint8_t pair_c0[FAST_MAX_PAIRS], pair_c1[FAST_MAX_PAIRS], pair_better[FAST_MAX_PAIRS];
    uint32_t n_pairs, n_unpaired; bool found_pair;
    uint8_t unpaired[FAST_MAX_CANDS];
    auto frag_of = [&](uint32_t c) { return (uint32_t)cand[c].frag; };
    auto read_of = [&](uint32_t c) { return (uint32_t)cand[c].read; };
    auto score_of = [&](uint32_t c) { return cand[c].score; };
    auto dist_of = [&](uint32_t c0, uint32_t c1) {
        uint32_t fn, fo, ln, le, x0, x1, x2, x3;
        extension_ends(ix, ext_of(cand[c0]), ev_path(a.ev, cand[c0].item), fn, fo, x0, x1);
        extension_ends(ix, ext_of(cand[c1]), ev_path(a.ev, cand[c1].item), x2, x3, ln, le);
        return oriented_distance(ix, fn, fo, ln, le);
    };
    if (!collect_pairs<FAST_MAX_PAIRS>(n_cand, ps.n_fragments + 1, frag_of, read_of, score_of, dist_of, ps.better_cluster_count, a.frag_mean, a.frag_sd,
                                       P.log_base, pair_score, pair_dist, pair_c0, pair_c1, pair_better, n_pairs, found_pair, unpaired, n_unpaired))
        return false;
    bool done = false;
    if (n_unpaired > 0 && P.max_rescue_attempts != 0) return false;     // mate rescue is warp work
    if (n_unpaired > 0 && !found_pair) {
        int best_c[2]; int32_t best_score[2];
        best_unpaired_per_end(unpaired, n_unpaired, read_of, score_of, rng, best_c, best_score);
        for (uint32_t r = 0; r < 2; r++) {
            out[r].mapq = 1;
            if (best_c[r] >= 0 && !write_cand(r, cand[best_c[r]])) return false;
        }
        done = true;
    } else if (n_pairs > 0) {
        uint8_t po[FAST_MAX_PAIRS];
        sort_shuffling_ties(n_pairs, [&](uint32_t x, uint32_t y) { return pair_score[x] > pair_score[y]; }, po, rng);
        double scores_sorted[FAST_MAX_PAIRS];
        for (uint32_t q = 0; q < n_pairs; q++) scores_sorted[q] = pair_score[po[q]];
        const uint32_t wp = po[0];
        const double uncapped_mapq = scores_sorted[0] == 0 ? 0.0 : max_mapping_quality(scores_sorted, n_pairs, P.log_base);
        const double cluster_cap = fragment_cluster_cap(pair_better[wp]);
        double caps[2];
        for (uint32_t r = 0; r < 2; r++) {
            // explored-minimizer count bound for the per-thread tables
            uint32_t n_exp = 0;
#pragma unroll
            for (uint32_t x = 0; x < PRESENT_WORDS; x++) n_exp += __popc(explored[r][x]);
            if (n_exp > FAST_MAX_EXPLORED) return false;
            uint64_t mp[FAST_MAX_EXPLORED]; double cbuf[FAST_MAX_EXPLORED + 1];
            caps[r] = faster_cap(P, a.minimizers + rsp[r]->min_off, ix.k, explored[r], rsp[r]->min_cnt, quals[r], L[r], mp, cbuf);
        }
        const uint32_t cwin[2] = {pair_c0[wp], pair_c1[wp]};
        for (uint32_t r = 0; r < 2; r++) {
            if (!write_cand(r, cand[cwin[r]])) return false;
            pair_read_mapq(uncapped_mapq, cluster_cap, caps[0] + caps[1], pair_dist[wp] == INT64_MAX, INFINITY, out[r]);
        }
        done = true;
    } else {
        done = true;      // both unmapped
    }
    if (done) {
        a.aln[2 * p] = out[0]; a.aln[2 * p + 1] = out[1];
        a.status[2 * p] = GB_ITEM_OK; a.status[2 * p + 1] = GB_ITEM_OK;
    }
    return done;
}

// Single-end twin of fast_pair: one thread per read (minimizer_mapper.cpp:886-1188 restricted to
// full-length extension sets).  Returns false when the read must go to the warp-per-read kernel.
__device__ inline bool fast_read(const DevIndex& ix, const MapParamsDev& P, const DevScores& sc, const MapBatch& b, const AlignArgs& a, uint32_t r) {
    const ReadState rs = b.states[r];
    if (rs.status != GB_ITEM_OK) return false;
    if (P.max_multimaps > 1) return false;                      // secondaries are written by the warp kernels only
    DevRng rng = rs.rng;
    const uint64_t rb = b.read_off[r];
    const uint32_t L = (uint32_t)(b.read_off[r + 1] - rb);
    const uint8_t* read = b.reads + rb; const uint8_t* qual = b.quals ? b.quals + rb : nullptr;
    FastCand cand[FAST_MAX_CANDS]; uint32_t n_cand = 0;
    uint32_t explored[PRESENT_WORDS];
#pragma unroll
    for (uint32_t x = 0; x < PRESENT_WORDS; x++) explored[x] = 0;
    const uint32_t S = rs.item_cnt;
    if (S > FAST_MAX_SETS) return false;
    int set_score[FAST_MAX_SETS]; uint8_t set_order[FAST_MAX_SETS];
    for (uint32_t s = 0; s < S; s++) {
        const uint32_t item = rs.item_off + s;
        if (a.ev.ext_status[item] != GB_ITEM_OK) return false;
        const gb_extension* ext = ev_ext(a.ev, item);
        const uint32_t n_ext = a.ev.ext_count[item];
        if (n_ext > 0 && ext_full(ext[0]) && ext[0].mismatches <= 4) set_score[s] = ext[0].score;
        else set_score[s] = score_extension_group(ext, n_ext, L, sc.gap_open, sc.gap_extend);
    }
    sort_shuffling_ties(S, [&](uint32_t x, uint32_t y) { return set_score[x] > set_score[y]; }, set_order, rng);
    const double set_cutoff = S == 0 ? 0.0 : (double)set_score[set_order[0]] - P.extension_set_score_threshold;
    uint32_t unskipped = 0;
    for (uint32_t oi = 0; oi < S; oi++) {
        const uint32_t s = set_order[oi];
        bool process;
        if (P.extension_set_score_threshold != 0 && (double)set_score[s] <= set_cutoff) process = unskipped < (uint32_t)P.min_extension_sets;
        else process = unskipped < P.max_alignments;
        if (!process) continue;
        if (set_score[s] < P.extension_set_min_score) continue;                    // :912-916
        unskipped++;
        const uint32_t item = rs.item_off + s;
        const gb_extension* ext = ev_ext(a.ev, item);
        const uint32_t n_ext = a.ev.ext_count[item];
        if (!(n_ext > 0 && ext_full(ext[0]) && ext[0].mismatches <= 4)) return false;     // tail alignment needed
        const DevItem it = a.items[item];
        const int32_t best0 = ext[0].score;
        bool keep = true;
        for (uint32_t j = 0; j < n_ext && (j == 0 || ext_full(ext[j])); j++) {
            if (keep && ext[j].score != 0 && (double)ext[j].score >= (double)best0 * 0.8) {
                if (n_cand >= FAST_MAX_CANDS) return false;
                cand[n_cand++] = FastCand{ext[j].score, item, (uint8_t)j, 0, 0};
            } else keep = false;
        }
#pragma unroll
        for (uint32_t x = 0; x < PRESENT_WORDS; x++) explored[x] |= it.present[x];
    }
    // winner (process_until_threshold_a, :1095), MAPQ (:1146-1188)
    double scores_sorted[FAST_MAX_CANDS + 1]; uint32_t n_scores = 0; int win = -1;
    if (n_cand == 0) { scores_sorted[0] = 0.0; n_scores = 1; }
    else {
        uint8_t co[FAST_MAX_CANDS];
        sort_shuffling_ties(n_cand, [&](uint32_t x, uint32_t y) { return cand[x].score > cand[y].score; }, co, rng);
        for (uint32_t c = 0; c < n_cand; c++) scores_sorted[c] = (double)cand[co[c]].score;
        n_scores = n_cand; win = co[0];
    }
    const double mapq = win >= 0 ? max_mapping_quality(scores_sorted, n_scores, P.log_base) : 0.0;
    uint32_t n_exp = 0;
#pragma unroll
    for (uint32_t x = 0; x < PRESENT_WORDS; x++) n_exp += __popc(explored[x]);
    if (n_exp > FAST_MAX_EXPLORED) return false;
    uint64_t mp[FAST_MAX_EXPLORED]; double cbuf[FAST_MAX_EXPLORED + 1];
    const double cap = faster_cap(P, a.minimizers + rs.min_off, ix.k, explored, rs.min_cnt, qual, L, mp, cbuf);
    gb_alignment out;
    out.read_id = r; out.score = 0; out.flags = 0; out.n_mappings = 0; out.n_edits = 0;
    out.mapping_off = r * P.mapping_cap; out.edit_off = r * P.edit_cap;
    single_end_mapq(mapq, cap, out);
    if (win >= 0) {
        const FastCand& c = cand[win];
        uint32_t nm = 0, ne = 0;
        if (!extension_to_output(ix, ev_ext(a.ev, c.item)[c.ext_j], ev_path(a.ev, c.item),
                                 ev_mism(a.ev, c.item), read, L, false,
                                 a.maps + (size_t)r * P.mapping_cap, a.edits + (size_t)r * P.edit_cap, P.mapping_cap, P.edit_cap, nm, ne)) return false;
        out.score = c.score; out.flags = nm ? GB_ALN_MAPPED : 0; out.n_mappings = (uint16_t)nm; out.n_edits = ne;
    }
    a.aln[r] = out; a.status[r] = GB_ITEM_OK;
    return true;
}

struct FastArgs { uint32_t* slow_list; uint32_t* slow_count; };

// Registers uncapped: a cap for 12 or 16 resident blocks per SM makes the kernel spill to local memory.  Measured on an
// H100 SXM at a 400 W power limit, per 1 M reads (500 k pairs) of config 2: uncapped 7.4 ms, 12 blocks 16.4 ms, 16 blocks 18.7 ms.
__global__ void __launch_bounds__(128, 1)
align_fast_kernel_pe(DevIndex ix, MapParamsDev P, DevScores sc, MapBatch b, AlignArgs a, FastArgs fa) {
    const uint32_t n_pairs = b.n_reads / 2;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n_pairs; p += gridDim.x * blockDim.x) {
        if (!fast_pair(ix, P, sc, b, a, p)) {
            const uint32_t slot = atomicAdd(fa.slow_count, 1u);
            fa.slow_list[slot] = p;
        }
    }
}

__global__ void __launch_bounds__(128)
align_fast_kernel(DevIndex ix, MapParamsDev P, DevScores sc, MapBatch b, AlignArgs a, FastArgs fa) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < b.n_reads; r += gridDim.x * blockDim.x) {
        if (!fast_read(ix, P, sc, b, a, r)) {
            const uint32_t slot = atomicAdd(fa.slow_count, 1u);
            fa.slow_list[slot] = r;
        }
    }
}
