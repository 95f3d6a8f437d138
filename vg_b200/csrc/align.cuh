// align.cuh — align_kernel: one warp per read turns the read's gapless-extension sets into
// the output alignment record:
//   score_extension_group          minimizer_mapper.cpp:5022-5203
//   extension-set selection        :886-1063  (process_until_threshold_d)
//   extension_to_alignment         :3905-3914 / GaplessExtension::to_path gbwt_extender.cpp:119-156
//   find_optimal_tail_alignments   :5369-5622 (+ tail.cuh)
//   winner + MAPQ                  :1087-1188, mapping_quality_calculator.cpp:26-67, :355-364
//   faster_cap                     :2946-3260
#pragma once
#include "map_state.cuh"
#include "tail.cuh"
#include "xdrop_tile.cuh"

namespace gb {

constexpr uint32_t MAX_SETS = 64;          // extension sets (kept clusters) per read handled here
constexpr uint32_t MAX_CANDS = 24;         // candidate alignments per read

struct ExtView {                           // outputs of the extension kernel
    const uint32_t* ext_count; const uint8_t* ext_status;
    const gb_extension* ext; const uint32_t* path_pool; const uint32_t* mism_pool;
    uint32_t max_ext, path_cap, mism_cap;
    // items redone with large strides (ExtendBig): big_of[item] != 0xffffffff selects the large pools
    const uint32_t* big_of; const gb_extension* big_ext; const uint32_t* big_path; const uint32_t* big_mism;
    uint32_t big_max_ext, big_path_cap, big_mism_cap;
};
__device__ __forceinline__ const gb_extension* ev_ext(const ExtView& ev, uint32_t item) {
    const uint32_t s = ev.big_of ? ev.big_of[item] : 0xffffffffu;
    return s == 0xffffffffu ? ev.ext + (size_t)item * ev.max_ext : ev.big_ext + (size_t)s * ev.big_max_ext;
}
__device__ __forceinline__ const uint32_t* ev_path(const ExtView& ev, uint32_t item) {
    const uint32_t s = ev.big_of ? ev.big_of[item] : 0xffffffffu;
    return s == 0xffffffffu ? ev.path_pool + (size_t)item * ev.path_cap : ev.big_path + (size_t)s * ev.big_path_cap;
}
__device__ __forceinline__ const uint32_t* ev_mism(const ExtView& ev, uint32_t item) {
    const uint32_t s = ev.big_of ? ev.big_of[item] : 0xffffffffu;
    return s == 0xffffffffu ? ev.mism_pool + (size_t)item * ev.mism_cap : ev.big_mism + (size_t)s * ev.big_mism_cap;
}

struct CandBuf {                           // per-warp scratch for candidate alignments
    gb_mapping* maps; uint32_t* edits;     // [MAX_CANDS][map_cap] / [MAX_CANDS][edit_cap]
    uint32_t map_cap, edit_cap;
};

__device__ __forceinline__ bool ext_full(const gb_extension& e) { return (e.flags & 3u) == 3u; }

// score_extension_group for a non-full-length set (sweep line; heaps replaced by scans over
// the handful of extensions, which compute the same maxima).
__device__ inline int score_extension_group(const gb_extension* ext, uint32_t n, uint32_t seq_len, int go, int ge) {
    if (n == 0) return 0;
    if (ext_full(ext[0]) && ext[0].mismatches <= 4) return ext[0].score;
    if (seq_len == 0) return 0;
    // extensions are sorted by read interval (remove_duplicates), so entering order = index order
    int best_chain[64];
    bool active[64];
    const uint32_t nn = min(n, 64u);
#pragma unroll 1
    for (uint32_t i = 0; i < nn; i++) { best_chain[i] = 0; active[i] = false; }
    int overlap_enc[64]; bool overlap_live[64];
#pragma unroll 1
    for (uint32_t i = 0; i < nn; i++) overlap_live[i] = false;
    int64_t sweep_line = 0, last_sweep_line = 0;
    uint32_t unentered = 0;
    int best_gap_score = 0, best_past_ending_score_ever = 0, overlap_score_offset = 0;
#pragma unroll 1
    while (last_sweep_line <= (int64_t)seq_len) {
        int64_t next_seed_start = INT64_MAX, next_seed_end = INT64_MAX;
        if (unentered < nn) next_seed_start = ext[unentered].read_lo;
#pragma unroll 1
        for (uint32_t i = 0; i < nn; i++) if (active[i]) next_seed_end = min(next_seed_end, (int64_t)ext[i].read_hi);
        sweep_line = min(min(next_seed_end, next_seed_start), (int64_t)seq_len);
        const int sweep_distance = (int)(sweep_line - last_sweep_line + 1);
        int best_past_ending_score_here = 0;
#pragma unroll 1
        for (uint32_t i = 0; i < nn; i++) if (active[i] && (int64_t)ext[i].read_hi == sweep_line) {
            best_past_ending_score_here = max(best_past_ending_score_here, best_chain[i]);
            active[i] = false;
        }
        best_past_ending_score_ever = max(best_past_ending_score_ever, best_past_ending_score_here);
        if (sweep_line == (int64_t)seq_len) break;
        overlap_score_offset += sweep_distance * ge;
        int best_overlap_score = 0;
        {
            // top of the max-heap over (encoded score, past-end) among entries not yet passed
            bool any = false; int best_enc = 0; uint32_t best_end = 0;
#pragma unroll 1
            for (uint32_t i = 0; i < nn; i++) {
                if (!overlap_live[i]) continue;
                if ((int64_t)ext[i].read_hi <= sweep_line) continue;
                if (!any || overlap_enc[i] > best_enc || (overlap_enc[i] == best_enc && ext[i].read_hi > best_end)) { any = true; best_enc = overlap_enc[i]; best_end = ext[i].read_hi; }
            }
            if (any) best_overlap_score = best_enc + overlap_score_offset;
        }
        if (best_gap_score != 0) best_gap_score -= sweep_distance * ge;
        best_gap_score = max(0, max(best_gap_score, best_past_ending_score_here - (go - ge)));
#pragma unroll 1
        while (unentered < nn && (int64_t)ext[unentered].read_lo == sweep_line) {
            best_chain[unentered] = max(best_overlap_score, max(best_gap_score, best_past_ending_score_here)) + ext[unentered].score;
            const int extension_length = (int)(ext[unentered].read_hi - ext[unentered].read_lo);
            const int raw_overlap_score = best_chain[unentered] - go - ge * extension_length;
            overlap_enc[unentered] = raw_overlap_score - overlap_score_offset; overlap_live[unentered] = true;
            active[unentered] = true;
            unentered++;
        }
        last_sweep_line = sweep_line + 1;
    }
    return best_past_ending_score_ever;
}

// GaplessExtension::to_path appended to a PathBuf (lane 0 only).
__device__ inline void extension_to_path(const DevIndex& ix, const gb_extension& e, const uint32_t* path_pool, const uint32_t* mism_pool,
                                         const uint8_t* read, PathBuf& pb) {
    uint32_t mi = 0;
    uint32_t read_offset = e.read_lo, node_offset = e.offset;
#pragma unroll 1
    for (uint32_t i = 0; i < e.path_len; i++) {
        const uint32_t h = path_pool[e.path_off + i];
        const uint32_t nlen = load_node(ix, h).len;
        const uint32_t limit = min(read_offset + nlen - node_offset, e.read_hi);
        pb_add_mapping(pb, h, node_offset);
#pragma unroll 1
        while (mi < e.mism_len && mism_pool[e.mism_off + mi] < limit) {
            const uint32_t mp = mism_pool[e.mism_off + mi];
            if (read_offset < mp) pb_add_edit(pb, edit_word(GB_EDIT_MATCH, mp - read_offset, 0));
            pb_add_edit(pb, edit_word(GB_EDIT_SUB, 1, base2(read[mp])));
            read_offset = mp + 1; mi++;
        }
        if (read_offset < limit) { pb_add_edit(pb, edit_word(GB_EDIT_MATCH, limit - read_offset, 0)); read_offset = limit; }
        node_offset = 0;
    }
}

__device__ __forceinline__ bool mapping_is_total_insertion(const PathBuf& p, uint32_t mi, uint32_t first_edit) {
    return p.maps[mi].n_edits == 1 && (p.edits[first_edit] & 3u) == GB_EDIT_INS && (p.edits[first_edit] >> 4) > 0;
}

// add_to_path (minimizer_mapper.cpp:5318-5367): append `src` mappings to `dst` (lane 0 only).
__device__ inline void add_to_path(PathBuf& dst, const gb_mapping* src_maps, const uint32_t* src_edits, uint32_t n_maps) {
    uint32_t se = 0;
#pragma unroll 1
    for (uint32_t i = 0; i < n_maps; i++) {
        const gb_mapping m = src_maps[i];
        bool combined = false;
        if (dst.n_maps > 0) {
            gb_mapping& prev = dst.maps[dst.n_maps - 1];
            if ((m.node >> 1) == (prev.node >> 1)) {
                bool can_combine = false;
                if (m.offset != 0) can_combine = true;
                else {
                    const uint32_t prev_first = dst.n_edits - prev.n_edits;
                    const bool prev_ti = prev.n_edits == 1 && (dst.edits[prev_first] & 3u) == GB_EDIT_INS && (dst.edits[prev_first] >> 4) > 0;
                    const bool ti = m.n_edits == 1 && (src_edits[se] & 3u) == GB_EDIT_INS && (src_edits[se] >> 4) > 0;
                    if (prev_ti || ti) {
                        can_combine = true;
                        if (prev_ti) { prev.node = m.node; prev.offset = m.offset; }
                    }
                }
                if (can_combine) {
#pragma unroll 1
                    for (uint32_t x = 0; x < m.n_edits; x++) pb_add_edit(dst, src_edits[se + x]);
                    combined = true;
                }
            }
        }
        if (!combined) {
            pb_add_mapping(dst, m.node, m.offset);
#pragma unroll 1
            for (uint32_t x = 0; x < m.n_edits; x++) pb_add_edit(dst, src_edits[se + x]);
        }
        se += m.n_edits;
    }
}

// pareto frontier helpers, minimizer_mapper.cpp:5263-5311
struct Pareto { uint32_t first; int32_t second; };
__device__ inline uint32_t find_pareto_frontier(Pareto* v, uint32_t n) {
    if (n == 0) return 0;
    // sort by (second asc, first desc)
#pragma unroll 1
    for (uint32_t i = 1; i < n; i++) { Pareto key = v[i]; uint32_t j = i;
#pragma unroll 1
        while (j > 0 && (key.second < v[j - 1].second || (key.second == v[j - 1].second && key.first > v[j - 1].first))) { v[j] = v[j - 1]; j--; }
        v[j] = key; }
    uint32_t tail = 1;
#pragma unroll 1
    for (uint32_t i = 1; i < n; i++) { if (v[i].first <= v[tail - 1].first) continue; v[tail] = v[i]; tail++; }
    n = tail;
#pragma unroll 1
    for (uint32_t i = 1; i < n; i++) { Pareto key = v[i]; uint32_t j = i;
#pragma unroll 1
        while (j > 0 && (key.first < v[j - 1].first || (key.first == v[j - 1].first && key.second < v[j - 1].second))) { v[j] = v[j - 1]; j--; }
        v[j] = key; }
    return n;
}
__device__ __forceinline__ int32_t gap_penalty1(uint32_t length, const DevScores& s) { return length == 0 ? 0 : s.gap_open + ((int32_t)length - 1) * s.gap_extend; }
__device__ __forceinline__ int32_t gap_penalty2(uint32_t start, uint32_t limit, const DevScores& s) {
    return start >= limit ? s.gap_open : s.gap_open + ((int32_t)(limit - start) - 1) * s.gap_extend;
}
__device__ inline int32_t flank_penalty(uint32_t length, const Pareto* f, uint32_t n, const DevScores& s) {
    int32_t result = gap_penalty1(length, s);
#pragma unroll 1
    for (uint32_t i = 0; i < n; i++) {
        result = min(result, f[i].second + gap_penalty2(f[i].first, length, s));
        if (f[i].first >= length) break;
    }
    return result;
}

// One tail (left or right) of one extension: forest + best alignment against any tree.
// Result path (graph space) is written to `res`; returns the score.
// get_best_alignment_against_any_tree, minimizer_mapper.cpp:5626-5743.
__device__ inline int32_t align_tail(const DevIndex& ix, const MapParamsDev& P, const DevScores& sc, const TailWs& ws, DpSmem dps,
                                     const gb_extension& e, const uint32_t* path_pool, const uint8_t* read, uint32_t L,
                                     bool left_tail, uint8_t* qbuf, DevRng& rng, PathBuf& res, PathBuf& scratch, uint32_t& status,
                                     const TailLookup& tl) {
    const int lane = lane_id();
    uint32_t from_node, from_offset, tail_length; int32_t lo, hi;
    const uint32_t first = path_pool[e.path_off], last = path_pool[e.path_off + e.path_len - 1];
    uint32_t default_node, default_offset;
    if (left_tail) {
        from_node = first ^ 1u;
        from_offset = load_node(ix, first).len - e.offset;       // reverse(Position, node_length)
        lo = (int32_t)e.bwd_lo; hi = (int32_t)e.bwd_hi;
        tail_length = e.read_lo;
        default_node = first; default_offset = e.offset;         // starting_position
    } else {
        from_node = last;
        uint32_t tail_off = e.offset + (e.read_hi - e.read_lo);
#pragma unroll 1
        for (uint32_t i = 0; i + 1 < e.path_len; i++) tail_off -= load_node(ix, path_pool[e.path_off + i]).len;
        from_offset = tail_off;
        lo = (int32_t)e.fwd_lo; hi = (int32_t)e.fwd_hi;
        tail_length = L - e.read_hi;
        default_node = last; default_offset = tail_off;          // tail_position
    }
    pb_reset(res);
    if (tail_length == 0) return 0;
    // ---- planned tail: its DPs already ran in xdrop_tile_kernel; pick the winner among the trees in the same order, with
    // the same LazyRNG draws on ties, as the in-place loop below (get_best_alignment_against_any_tree, :5626-5743)
    if (tl.pv) {
        const TailPlanEntry* pe = nullptr;
#pragma unroll 1
        for (uint32_t x = 0; x < tl.count; x++) if (tl.pv->entries[tl.base + x].key == tl.key) { pe = tl.pv->entries + tl.base + x; break; }
        // a cancelled tail (the decide pass judged that the reference skips it, :5478-5492) is never asked for; should the
        // walk here disagree, the tail is simply aligned in place.  So is a tail with a tile that ran out of the tile's
        // fixed path capacities (TILE_MAP_CAP / TILE_EDIT_CAP / TILE_STEP_CAP): the in-place sweep writes into the
        // read's own buffers, whose caps the caller sets.  The check comes before any RNG draw, so the draw order is
        // the in-place loop's either way.
        if (pe) for (uint32_t t = 0; t < pe->n_trees; t++) {
            const uint32_t ti = pe->first_tile + t;
            if (tl.pv->tile_off[ti] != TILE_REFUSED && tl.pv->results[ti].status != GB_TILE_ST_OK) { pe = nullptr; break; }
        }
        if (pe) {
            int32_t best_score = 0;
            if (lane == 0) { pb_add_mapping(res, default_node, default_offset); pb_add_edit(res, edit_word(GB_EDIT_INS, tail_length, 0)); }
            __syncwarp();
            res.n_maps = 1; res.n_edits = 1;
#pragma unroll 1
            for (uint32_t t = 0; t < pe->n_trees; t++) {
                const uint32_t ti = pe->first_tile + t;
                if (tl.pv->tile_off[ti] == TILE_REFUSED) continue;            // subgraph too large for max_dozeu_cells (:5694-5701)
                const TileResult tr = tl.pv->results[ti];
                bool beats = false;
                if (tr.score > best_score) beats = true;
                else if (tr.score == best_score) beats = (rng_next(rng) % 2) != 0;
                if (beats) {
                    best_score = tr.score;
                    if (tr.n_maps > res.map_cap || tr.n_edits > res.edit_cap) { status = GB_ITEM_OUT_FULL; return 0; }
                    const gb_mapping* gm = reinterpret_cast<const gb_mapping*>(tl.pv->path_pool + tr.path_off);
                    const uint32_t* gedits = tl.pv->path_pool + tr.path_off + 2 * tr.n_maps;
#pragma unroll 1
                    for (uint32_t i = lane; i < tr.n_maps; i += 32) res.maps[i] = gm[i];
#pragma unroll 1
                    for (uint32_t i = lane; i < tr.n_edits; i += 32) res.edits[i] = gedits[i];
                    __syncwarp();
                    res.n_maps = tr.n_maps; res.n_edits = tr.n_edits; res.overflow = false;
                }
            }
            return best_score;
        }
        if (lane == 0 && tl.pv->stats) atomicAdd((unsigned long long*)&tl.pv->stats[2], 1ull);
    }
    const uint32_t gap = longest_detectable_gap(sc, L, tail_length);
    // query: the tail itself (right tail) or its reverse complement (left tail)
#pragma unroll 1
    for (uint32_t i = lane; i < tail_length; i += 32)
        qbuf[i] = dp_query_base(left_tail ? comp_base(read[tail_length - 1 - i]) : read[e.read_hi + i]);
    __syncwarp();

    // default: pure softclip on the node we are going to
    int32_t best_score = 0;
    if (lane == 0) { pb_add_mapping(res, default_node, default_offset); pb_add_edit(res, edit_word(GB_EDIT_INS, tail_length, 0)); }
    __syncwarp();
    res.n_maps = 1; res.n_edits = 1;

    uint32_t root_trim = 0;
    const uint32_t n_forest = build_tail_forest(ix, ws, from_node, lo, hi, from_offset, gap + tail_length, root_trim);
    if (n_forest == 0xffffffffu) { status = GB_ITEM_OUT_FULL; return 0; }
    uint32_t t0 = 0;
#pragma unroll 1
    while (t0 < n_forest) {
        uint32_t t1 = t0 + 1;
#pragma unroll 1
        while (t1 < n_forest && ws.tree[t1].parent >= 0) t1++;
        // subgraph size check (:5694-5701)
        uint32_t bases = 0;
#pragma unroll 1
        for (uint32_t i = t0 + lane; i < t1; i += 32) bases += ws.tree[i].len;
        bases = (uint32_t)warp_sum((int)bases);
        if ((uint64_t)bases * tail_length <= P.max_dozeu_cells) {
            bool ovf = false;
            const uint32_t g = max(gap, 1u);
            const int32_t score = xdrop_tree(ix, sc, ws, dps, t0, t1, qbuf, tail_length, g, scratch, ovf);
            if (ovf || scratch.overflow) { status = GB_ITEM_OUT_FULL; return 0; }
            bool beats = false;
            if (scratch.n_maps > 0) {
                // deterministic_beats(score, best_score, rng)
                if (score > best_score) beats = true;
                else if (score == best_score) beats = (rng_next(rng) % 2) != 0;
            }
            if (beats) {
                best_score = score;
                if (lane == 0) {
                    pb_reset(res);
                    if (!left_tail) {
                        // translate_down (tree_subgraph.cpp:172-195)
                        uint32_t se = 0;
#pragma unroll 1
                        for (uint32_t i = 0; i < scratch.n_maps; i++) {
                            const gb_mapping m = scratch.maps[i];
                            const TreeNode tn = ws.tree[m.node];
                            uint32_t off = m.offset;
                            if (m.node == t0 && root_trim != 0) off += root_trim;    // trimmed root, forward strand
                            pb_add_mapping(res, tn.node, off);
#pragma unroll 1
                            for (uint32_t x = 0; x < m.n_edits; x++) pb_add_edit(res, scratch.edits[se + x]);
                            se += m.n_edits;
                        }
                    } else {
                        // reverse_complement_path (path.cpp:1791-1882) then translate_down
                        uint32_t ends[1];
                        (void)ends;
                        // edit start offsets per mapping
                        uint32_t se_end = scratch.n_edits;
#pragma unroll 1
                        for (int64_t i = (int64_t)scratch.n_maps - 1; i >= 0; i--) {
                            const gb_mapping m = scratch.maps[i];
                            const uint32_t se_begin = se_end - m.n_edits;
                            const TreeNode tn = ws.tree[m.node];
                            uint32_t used = 0;
#pragma unroll 1
                            for (uint32_t x = se_begin; x < se_end; x++) { const uint32_t wd = scratch.edits[x]; const uint32_t op = wd & 3u; if (op != GB_EDIT_INS) used += (op == GB_EDIT_SUB) ? 1u : (wd >> 4); }
                            const uint32_t new_off = tn.len - used - m.offset;
                            pb_add_mapping(res, tn.node ^ 1u, new_off);
#pragma unroll 1
                            for (int64_t x = (int64_t)se_end - 1; x >= (int64_t)se_begin; x--) {
                                uint32_t wd = scratch.edits[x];
                                if ((wd & 3u) == GB_EDIT_SUB) wd = (wd & ~0xCu) | ((3u - ((wd >> 2) & 3u)) << 2);   // complement the base
                                pb_add_edit(res, wd);
                            }
                            se_end = se_begin;
                        }
                    }
                }
                __syncwarp();
                res.n_maps = __shfl_sync(FULL, res.n_maps, 0); res.n_edits = __shfl_sync(FULL, res.n_edits, 0);
                res.overflow = __shfl_sync(FULL, (int)res.overflow, 0) != 0;
                if (res.overflow) { status = GB_ITEM_OUT_FULL; return 0; }
            }
        }
        t0 = t1;
    }
    return best_score;
}

} // namespace gb
