// rescue.cuh — mate rescue on the device (included by map.cu inside namespace gb):
//   MinimizerMapper::attempt_rescue            minimizer_mapper.cpp:3264-3482
//   seeds_in_subgraph                          :3484-3500
//   fix_dozeu_score / fix_dozeu_end_deletions  :3502-3565
//   subgraph_in_distance_range                 snarl_distance_index.cpp:1875 (contract, through the distance payload)
// One warp rescues one mate: the subgraph is cut from the chain order by a range test on the payload
// coordinates, the mate's minimizer hits inside it seed a gapless extension (extend_item), and unless
// that is full length the seeded two-pass X-drop aligner (xd_align) runs on the subgraph, with the full
// local DP (sw_align) as the fallback vg uses when the rescored path is not positive.
// Semantics statement by statement: oracle/rescue.cpp.
#pragma once

constexpr uint32_t RESCUE_IDS = 320;        // node ids in a rescue subgraph
constexpr uint32_t RESCUE_BASES = 6144;     // bases of both orientations
constexpr uint32_t RESCUE_RAW = 2048;       // hits collected before deduplication
constexpr uint32_t RESCUE_SEEDS = 128;      // distinct seeds kept (rescue_seed_limit <= 127)
constexpr uint32_t RESCUE_DEG = 8;          // edges per oriented node kept
constexpr uint32_t RESCUE_MAX_EXT = 48, RESCUE_PATH_CAP = 384, RESCUE_MISM_CAP = 192;

struct RescueWs {
    uint32_t* ids; unsigned long long* raw; gb_seed* seeds;
    QEntry* queue; ArenaNode* arena; gb_extension* ext; uint32_t* path_pool; uint32_t* mism_pool;
    uint32_t* nodes; uint32_t* esrc; uint32_t* edst; uint32_t* pred; uint32_t* succ; uint64_t* pred_off; uint64_t* succ_off; uint32_t* cnt;
    uint32_t* col_start; uint32_t* seq_off; uint32_t* seq_len; XdNode* nstate;
    int32_t* lastH; int32_t* lastE; uint8_t* argH; uint8_t* argE; uint8_t* tb; uint32_t* steps;
};
__host__ __device__ inline size_t rescue_align16(size_t x) { return (x + 15) & ~(size_t)15; }
__host__ __device__ inline size_t rescue_ws_bytes(uint32_t Lc) {
    const size_t W = Lc + 1, NN = 2 * RESCUE_IDS;
    size_t b = 0;
    b += rescue_align16(RESCUE_IDS * 4) + rescue_align16(RESCUE_RAW * 8) + rescue_align16(RESCUE_SEEDS * sizeof(gb_seed));
    b += rescue_align16(EXTEND_Q_CAP * sizeof(QEntry)) + rescue_align16(EXTEND_A_CAP * sizeof(ArenaNode));
    b += rescue_align16(RESCUE_MAX_EXT * sizeof(gb_extension)) + rescue_align16(RESCUE_PATH_CAP * 4) + rescue_align16(RESCUE_MISM_CAP * 4);
    b += rescue_align16(NN * 4) + 4 * rescue_align16(NN * RESCUE_DEG * 4) + 2 * rescue_align16((NN + 1) * 8) + rescue_align16((NN + 1) * 4);
    b += 3 * rescue_align16(NN * 4) + rescue_align16(NN * sizeof(XdNode));
    b += 2 * rescue_align16(NN * W * 4) + 2 * rescue_align16(NN * W) + rescue_align16((size_t)RESCUE_BASES * W) + rescue_align16((RESCUE_BASES + W + 2) * 4);
    return b;
}
__device__ inline RescueWs carve_rescue_ws(uint8_t* p, uint32_t Lc) {
    const size_t W = Lc + 1, NN = 2 * RESCUE_IDS;
    RescueWs w;
    auto take = [&](size_t bytes) { uint8_t* r = p; p += rescue_align16(bytes); return r; };
    w.ids = (uint32_t*)take(RESCUE_IDS * 4); w.raw = (unsigned long long*)take(RESCUE_RAW * 8); w.seeds = (gb_seed*)take(RESCUE_SEEDS * sizeof(gb_seed));
    w.queue = (QEntry*)take(EXTEND_Q_CAP * sizeof(QEntry)); w.arena = (ArenaNode*)take(EXTEND_A_CAP * sizeof(ArenaNode));
    w.ext = (gb_extension*)take(RESCUE_MAX_EXT * sizeof(gb_extension)); w.path_pool = (uint32_t*)take(RESCUE_PATH_CAP * 4); w.mism_pool = (uint32_t*)take(RESCUE_MISM_CAP * 4);
    w.nodes = (uint32_t*)take(NN * 4);
    w.esrc = (uint32_t*)take(NN * RESCUE_DEG * 4); w.edst = (uint32_t*)take(NN * RESCUE_DEG * 4); w.pred = (uint32_t*)take(NN * RESCUE_DEG * 4); w.succ = (uint32_t*)take(NN * RESCUE_DEG * 4);
    w.pred_off = (uint64_t*)take((NN + 1) * 8); w.succ_off = (uint64_t*)take((NN + 1) * 8); w.cnt = (uint32_t*)take((NN + 1) * 4);
    w.col_start = (uint32_t*)take(NN * 4); w.seq_off = (uint32_t*)take(NN * 4); w.seq_len = (uint32_t*)take(NN * 4); w.nstate = (XdNode*)take(NN * sizeof(XdNode));
    w.lastH = (int32_t*)take(NN * W * 4); w.lastE = (int32_t*)take(NN * W * 4); w.argH = take(NN * W); w.argE = take(NN * W);
    w.tb = take((size_t)RESCUE_BASES * W); w.steps = (uint32_t*)take((RESCUE_BASES + W + 2) * 4);
    return w;
}

// Is node `id` inside the distance range of the walk that starts `to_end` bases before the end of `start`?
// (oracle/rescue.cpp subgraph_in_distance_range)
__device__ __forceinline__ bool rescue_in_range(const DevIndex& ix, uint32_t id, uint32_t start_node, int64_t to_end, int64_t min_distance, int64_t max_distance) {
    const uint32_t start_id = start_node >> 1;
    if (id == start_id) return to_end > min_distance;
    const uint4 ps = __ldg(reinterpret_cast<const uint4*>(ix.dist) + start_id);      // x_in, x_out, slot, allele | component << 16
    const uint4 pv = __ldg(reinterpret_cast<const uint4*>(ix.dist) + id);
    if ((ps.w >> 16) != (pv.w >> 16)) return false;
    int64_t d0;
    if (!(start_node & 1u)) {
        if (ps.z < pv.z) d0 = to_end + ((int64_t)(int32_t)pv.x - (int64_t)(int32_t)ps.y);
        else if (ps.z == pv.z) { const int64_t t = site_distance(ix, ps, pv); if (t < 0) return false; d0 = to_end + t; }
        else return false;
    } else {
        if (pv.z < ps.z) d0 = to_end + ((int64_t)(int32_t)ps.x - (int64_t)(int32_t)pv.y);
        else if (ps.z == pv.z) { const int64_t t = site_distance(ix, pv, ps); if (t < 0) return false; d0 = to_end + t; }
        else return false;
    }
    const int64_t len = load_node(ix, 2 * id).len;
    return d0 <= max_distance && d0 + len > min_distance;
}
__device__ __forceinline__ bool rescue_slot_less(const DevIndex& ix, uint32_t a, uint32_t b) {
    const uint4 pa = __ldg(reinterpret_cast<const uint4*>(ix.dist) + a), pb = __ldg(reinterpret_cast<const uint4*>(ix.dist) + b);
    if ((pa.w >> 16) != (pb.w >> 16)) return (pa.w >> 16) < (pb.w >> 16);
    if (pa.z != pb.z) return pa.z < pb.z;
    if ((pa.w & 0xFFFFu) != (pb.w & 0xFFFFu)) return (pa.w & 0xFFFFu) < (pb.w & 0xFFFFu);     // place inside the site = topological
    return a < b;
}

// score_contiguous_alignment with both bonuses allowed (alignment_scorer.cpp:154-246); one lane
__device__ inline int32_t rescue_rescore(const DevScores& sc, const PathBuf& pb) {
    int32_t score = 0; bool last_was_deletion = false;
    uint32_t e = 0;
#pragma unroll 1
    for (uint32_t i = 0; i < pb.n_maps; i++) {
#pragma unroll 1
        for (uint32_t j = 0; j < pb.maps[i].n_edits; j++, e++) {
            const uint32_t wd = pb.edits[e], op = wd & 3u, len = wd >> 4;
            if (op == GB_EDIT_MATCH) { score += sc.match * (int32_t)len; last_was_deletion = false; }
            else if (op == GB_EDIT_SUB) { score -= sc.mismatch * (int32_t)len; last_was_deletion = false; }
            else if (op == GB_EDIT_DEL) {
                if (last_was_deletion) score -= (int32_t)len * sc.gap_extend;
                else score -= len ? sc.gap_open + ((int32_t)len - 1) * sc.gap_extend : 0;
                if (len) last_was_deletion = true;
            } else if (!((i == 0 && j == 0) || (i + 1 == pb.n_maps && j + 1 == pb.maps[i].n_edits))) {
                score -= len ? sc.gap_open + ((int32_t)len - 1) * sc.gap_extend : 0;
                last_was_deletion = false;
            } else last_was_deletion = false;
        }
    }
    const bool clip_start = pb.n_maps > 0 && pb.maps[0].n_edits > 0 && (pb.edits[0] & 3u) == GB_EDIT_INS && (pb.edits[0] >> 4) > 0;
    const bool clip_end = pb.n_maps > 0 && pb.maps[pb.n_maps - 1].n_edits > 0 && (pb.edits[pb.n_edits - 1] & 3u) == GB_EDIT_INS && (pb.edits[pb.n_edits - 1] >> 4) > 0;
    if (!clip_start) score += sc.full_length_bonus;
    if (!clip_end) score += sc.full_length_bonus;
    return score;
}

// fix_dozeu_end_deletions (:3519-3565); one lane, in place
__device__ inline void rescue_fix_end_deletions(PathBuf& pb) {
    // leading mappings / edits that consume no read
    uint32_t i = 0, j = 0, e = 0;
#pragma unroll 1
    for (; i < pb.n_maps; i++) {
#pragma unroll 1
        for (j = 0; j < pb.maps[i].n_edits; j++) { const uint32_t wd = pb.edits[e + j]; if ((wd & 3u) != GB_EDIT_DEL && (wd >> 4) != 0) break; }
        if (j != pb.maps[i].n_edits) break;
        e += pb.maps[i].n_edits;
    }
    if (i == pb.n_maps) { pb.n_maps = 0; pb.n_edits = 0; return; }
    if (i != 0 || j != 0) {
        uint32_t removed = 0;
#pragma unroll 1
        for (uint32_t k = 0; k < j; k++) removed += pb.edits[e + k] >> 4;          // deletions: from_length
        const uint32_t drop_edits = e + j;
#pragma unroll 1
        for (uint32_t x = drop_edits; x < pb.n_edits; x++) pb.edits[x - drop_edits] = pb.edits[x];
        pb.n_edits -= drop_edits;
        gb_mapping first = pb.maps[i]; first.n_edits = (uint16_t)(first.n_edits - j); first.offset = (uint16_t)(first.offset + removed);
#pragma unroll 1
        for (uint32_t x = i; x < pb.n_maps; x++) pb.maps[x - i] = pb.maps[x];
        pb.n_maps -= i; pb.maps[0] = first;
    }
    // trailing deletions
#pragma unroll 1
    while (pb.n_maps > 0) {
        gb_mapping& m = pb.maps[pb.n_maps - 1];
#pragma unroll 1
        while (m.n_edits > 0 && (pb.edits[pb.n_edits - 1] & 3u) == GB_EDIT_DEL) { m.n_edits--; pb.n_edits--; }
        if (m.n_edits == 0) pb.n_maps--; else break;
    }
}

// position of oriented node v in the rescue DAG (forward half in chain order, mirrored half after it)
__device__ inline uint32_t rescue_index_of(const RescueWs& rw, uint32_t n_ids, uint32_t v) {
    const uint32_t id = v >> 1;
#pragma unroll 1
    for (uint32_t x = 0; x < n_ids; x++) if (rw.ids[x] == id) return (v & 1u) ? 2 * n_ids - 1 - x : x;
    return 0xffffffffu;
}

// attempt_rescue.  anchor: the mapped mate's path (rightward orientation); sread/L: the mate to rescue;
// mins/M: its minimizers (score order, all of them).  The rescued path is written to `out` (graph space);
// returns its score (0: nothing found).  status reports capacity problems.
__device__ inline int32_t attempt_rescue(const DevIndex& ix, const MapParamsDev& P, const DevScores& sc, const RescueWs& rw,
                                         const PathBuf& anchor, uint32_t anchor_nm, uint32_t anchor_ne,
                                         const uint8_t* sread, uint32_t L, const DevMinimizer* mins, uint32_t M, bool rescue_forward,
                                         double frag_mean, double frag_sd, uint8_t* qbuf, DpSmem dps, uint32_t Lc, PathBuf& out, uint32_t& status) {
    const int lane = lane_id();
    pb_reset(out);
    if (anchor_nm == 0 || L == 0) return 0;
    const int64_t min_distance = (int64_t)fmax(0.0, frag_mean - (double)L - P.rescue_subgraph_stdevs * frag_sd);
    const int64_t max_distance = (int64_t)(frag_mean + P.rescue_subgraph_stdevs * frag_sd);
    uint32_t start_node; int64_t to_end;
    if (rescue_forward) { const gb_mapping m0 = anchor.maps[0]; start_node = m0.node; to_end = (int64_t)load_node(ix, m0.node).len - (int64_t)m0.offset; }
    else {
        const gb_mapping last = anchor.maps[anchor_nm - 1];
        uint32_t used = 0;
#pragma unroll 1
        for (uint32_t x = anchor_ne - last.n_edits; x < anchor_ne; x++) { const uint32_t wd = anchor.edits[x]; const uint32_t op = wd & 3u; if (op != GB_EDIT_INS) used += (op == GB_EDIT_SUB) ? 1u : (wd >> 4); }
        start_node = last.node ^ 1u; to_end = (int64_t)(last.offset + used) + 1;
    }
    // ---- subgraph ids in chain order ---------------------------------------------------------------------
    uint32_t n_ids = 0;
#pragma unroll 1
    for (uint32_t base = 0; base < ix.n_ids; base += 32) {
        const uint32_t x = base + lane;
        uint32_t id = 0; bool in = false;
        if (x < ix.n_ids) { id = __ldg(ix.slot_order + x); in = rescue_in_range(ix, id, start_node, to_end, min_distance, max_distance); }
        const uint32_t bal = __ballot_sync(FULL, in);
        if (n_ids + __popc(bal) > RESCUE_IDS) { status = GB_ITEM_OUT_FULL; return 0; }
        if (in) rw.ids[n_ids + __popc(bal & ((1u << lane) - 1u))] = id;
        n_ids += __popc(bal);
    }
    __syncwarp();
    if (n_ids == 0) return 0;
    // ---- seeds_in_subgraph: distinct (handle, read offset - node offset) of the hits on subgraph nodes -------
    uint32_t n_raw = 0; bool raw_full = false;
#pragma unroll 1
    for (uint32_t mi = 0; mi < M && !raw_full; mi++) {
        const DevMinimizer dm = mins[mi];
        const uint32_t hoff = dm.pad[0], hits = dm.pad[1];
        const int32_t pin = (int32_t)dm.fwd_offset + (dm.is_reverse ? (int32_t)ix.k - 1 : 0);
#pragma unroll 1
        for (uint32_t hb = 0; hb < hits; hb += 32) {
            const uint32_t j = hb + lane;
            bool in = false; unsigned long long key = 0;
            if (j < hits) {
                const uint2 pw = __ldg(reinterpret_cast<const uint2*>(ix.hits + hoff + j));
                const uint64_t pos = ((uint64_t)pw.y << 32) | pw.x;
                uint32_t node = (uint32_t)(pos >> 10), off = (uint32_t)(pos & 1023u);
                if (rescue_in_range(ix, node >> 1, start_node, to_end, min_distance, max_distance)) {
                    if (dm.is_reverse) { const uint32_t nlen = load_node(ix, node).len; node ^= 1u; off = nlen - off - 1; }
                    in = true; key = ((unsigned long long)node << 32) | (uint32_t)((pin - (int32_t)off) ^ 0x80000000);
                }
            }
            const uint32_t bal = __ballot_sync(FULL, in);
            if (n_raw + __popc(bal) > RESCUE_RAW) { raw_full = true; break; }
            if (in) rw.raw[n_raw + __popc(bal & ((1u << lane) - 1u))] = key;
            n_raw += __popc(bal);
        }
    }
    __syncwarp();
    if (raw_full) { status = GB_ITEM_OUT_FULL; return 0; }
    uint32_t n_seeds = 0;
    if (lane == 0) {
        // sorted distinct keys (ascending node, diagonal)
        unsigned long long* keys = rw.raw;       // in-place insertion: distinct prefix grows from the front
#pragma unroll 1
        for (uint32_t x = 0; x < n_raw; x++) {
            const unsigned long long key = keys[x];
            uint32_t lo = 0; while (lo < n_seeds && keys[lo] < key) lo++;
            if (lo < n_seeds && keys[lo] == key) continue;
            if (n_seeds > P.rescue_seed_limit) { n_seeds = P.rescue_seed_limit + 1; break; }
#pragma unroll 1
            for (uint32_t y = n_seeds; y > lo; y--) keys[y] = keys[y - 1];
            keys[lo] = key; n_seeds++;
            if (n_seeds > P.rescue_seed_limit) break;
        }
        if (n_seeds <= P.rescue_seed_limit && n_seeds <= RESCUE_SEEDS)
#pragma unroll 1
            for (uint32_t x = 0; x < n_seeds; x++) { gb_seed g; g.node = (uint32_t)(keys[x] >> 32); g.diag = (int32_t)((uint32_t)keys[x] ^ 0x80000000u); rw.seeds[x] = g; }
    }
    n_seeds = __shfl_sync(FULL, n_seeds, 0);
    __syncwarp();
    if (n_seeds > P.rescue_seed_limit) return 0;
    if (n_seeds > RESCUE_SEEDS) { status = GB_ITEM_OUT_FULL; return 0; }
    // ---- gapless extension of the seeds (masked read in the query buffer) -------------------------------------
#pragma unroll 1
    for (uint32_t i = lane; i < L; i += 32) { const uint8_t c = sread[i]; qbuf[i] = is_acgt(c) ? c : (uint8_t)'X'; }
    __syncwarp();
    ExtendParams ep; ep.sc = sc; ep.max_mismatches = 4; ep.overlap_threshold = 0.8; ep.overlap_threshold_unused = 0.f; ep.trim = 1;
    ep.max_ext = RESCUE_MAX_EXT; ep.path_cap = RESCUE_PATH_CAP; ep.mism_cap = RESCUE_MISM_CAP;
    uint32_t ext_status = GB_ITEM_OK;
    const uint32_t n_ext = extend_item(ix, ep, qbuf, L, rw.seeds, n_seeds, rw.queue, EXTEND_Q_CAP, rw.arena, EXTEND_A_CAP, rw.ext, rw.path_pool, rw.mism_pool, &ext_status);
    __syncwarp();
    if (ext_status != GB_ITEM_OK) { status = ext_status; return 0; }
    if (n_ext > 0 && ext_full(rw.ext[0]) && rw.ext[0].mismatches <= 4) {
        if (lane == 0) extension_to_path(ix, rw.ext[0], rw.path_pool, rw.mism_pool, sread, out);
        out.n_maps = __shfl_sync(FULL, out.n_maps, 0); out.n_edits = __shfl_sync(FULL, out.n_edits, 0);
        out.overflow = __shfl_sync(FULL, (int)out.overflow, 0) != 0;
        if (out.overflow || out.n_maps + 1 > out.map_cap) { status = GB_ITEM_OUT_FULL; return 0; }
        __syncwarp();
        return rw.ext[0].score;
    }
    uint32_t best = n_ext;
#pragma unroll 1
    for (uint32_t i = 0; i < n_ext; i++) if (best >= n_ext || rw.ext[i].score > rw.ext[best].score) best = i;
    // the best extension's nodes join the subgraph (:3347-3349)
    if (best < n_ext) {
        if (lane == 0) {
            const gb_extension e = rw.ext[best];
#pragma unroll 1
            for (uint32_t x = 0; x < e.path_len; x++) {
                const uint32_t id = rw.path_pool[e.path_off + x] >> 1;
                uint32_t lo = 0; while (lo < n_ids && rescue_slot_less(ix, rw.ids[lo], id)) lo++;
                if (lo < n_ids && rw.ids[lo] == id) continue;
                if (n_ids >= RESCUE_IDS) { n_ids = RESCUE_IDS + 1; break; }
#pragma unroll 1
                for (uint32_t y = n_ids; y > lo; y--) rw.ids[y] = rw.ids[y - 1];
                rw.ids[lo] = id; n_ids++;
            }
        }
        n_ids = __shfl_sync(FULL, n_ids, 0);
        __syncwarp();
        if (n_ids > RESCUE_IDS) { status = GB_ITEM_OUT_FULL; return 0; }
    }
    // ---- the DAG: both orientations in chain order, edges among them ---------------------------------------------
    const uint32_t N = 2 * n_ids;
    uint32_t bases = 0;
#pragma unroll 1
    for (uint32_t x = lane; x < n_ids; x += 32) { const uint32_t id = rw.ids[x]; rw.nodes[x] = 2 * id; rw.nodes[N - 1 - x] = 2 * id + 1; bases += 2 * load_node(ix, 2 * id).len; }
    bases = (uint32_t)warp_sum((int)bases);
    __syncwarp();
    if ((uint64_t)bases * L > P.max_dozeu_cells) return 0;                     // :3371-3381
    if (bases > RESCUE_BASES || L > Lc) { status = GB_ITEM_OUT_FULL; return 0; }
    // edges i -> j (j > i), collected per source, then CSR by target and by source (lists ascending, distinct)
#pragma unroll 1
    for (uint32_t x = lane; x <= N; x += 32) rw.cnt[x] = 0;
    __syncwarp();
    uint32_t n_edges = 0; bool deg_full = false;
#pragma unroll 1
    for (uint32_t ib = 0; ib < N; ib += 32) {
        const uint32_t i = ib + lane;
        uint32_t tgt[RESCUE_DEG]; uint32_t nt = 0;
        if (i < N) {
            const gb_node_rec nr = load_node(ix, rw.nodes[i]);
            if (nr.size != 0) {
                const uint32_t* rec = ix.gbwt + nr.rec_off;
                const uint32_t ne = __ldg(rec);
#pragma unroll 1
                for (uint32_t e = 0; e < ne; e++) {
                    const uint32_t to = __ldg(rec + 2 + 2 * e);
                    if (to == 0) continue;
                    const uint32_t j = rescue_index_of(rw, n_ids, to);
                    if (j == 0xffffffffu || j <= i) continue;
                    bool dup = false;
#pragma unroll 1
                    for (uint32_t y = 0; y < nt; y++) dup |= tgt[y] == j;
                    if (dup) continue;
                    if (nt >= RESCUE_DEG) { deg_full = true; break; }
                    tgt[nt++] = j;
                }
            }
        }
        // this chunk's edges, in source order
        const uint32_t incl = (uint32_t)warp_incl_scan((int)nt);
        const uint32_t basee = n_edges + incl - nt;
#pragma unroll 1
        for (uint32_t y = 0; y < nt; y++) { rw.esrc[basee + y] = i; rw.edst[basee + y] = tgt[y]; }
        n_edges += __shfl_sync(FULL, incl, 31);
    }
    __syncwarp();
    if (__any_sync(FULL, deg_full)) { status = GB_ITEM_OUT_FULL; return 0; }
    if (lane == 0) {
        // CSR by target (sources ascending because edges are in source order), then by source (targets sorted)
#pragma unroll 1
        for (uint32_t x = 0; x <= N; x++) rw.cnt[x] = 0;
#pragma unroll 1
        for (uint32_t x = 0; x < n_edges; x++) rw.cnt[rw.edst[x] + 1]++;
        rw.pred_off[0] = 0; for (uint32_t x = 0; x < N; x++) rw.pred_off[x + 1] = rw.pred_off[x] + rw.cnt[x + 1];
#pragma unroll 1
        for (uint32_t x = 0; x <= N; x++) rw.cnt[x] = 0;
#pragma unroll 1
        for (uint32_t x = 0; x < n_edges; x++) { const uint32_t d = rw.edst[x]; rw.pred[rw.pred_off[d] + rw.cnt[d]++] = rw.esrc[x]; }
#pragma unroll 1
        for (uint32_t x = 0; x <= N; x++) rw.cnt[x] = 0;
#pragma unroll 1
        for (uint32_t x = 0; x < n_edges; x++) rw.cnt[rw.esrc[x] + 1]++;
        rw.succ_off[0] = 0; for (uint32_t x = 0; x < N; x++) rw.succ_off[x + 1] = rw.succ_off[x] + rw.cnt[x + 1];
#pragma unroll 1
        for (uint32_t x = 0; x <= N; x++) rw.cnt[x] = 0;
#pragma unroll 1
        for (uint32_t x = 0; x < n_edges; x++) {
            const uint32_t s = rw.esrc[x], d = rw.edst[x];
            uint32_t pos = rw.cnt[s]++; const uint64_t b0 = rw.succ_off[s];
#pragma unroll 1
            while (pos > 0 && rw.succ[b0 + pos - 1] > d) { rw.succ[b0 + pos] = rw.succ[b0 + pos - 1]; pos--; }
            rw.succ[b0 + pos] = d;
        }
    }
    __syncwarp();
    DagView v;
    v.N = N; v.node = rw.nodes; v.pred = rw.pred; v.pred_off = rw.pred_off; v.succ = rw.succ; v.succ_off = rw.succ_off;
    v.col_start = rw.col_start; v.seq_off = rw.seq_off; v.seq_len = rw.seq_len; v.nstate = rw.nstate;
    v.lastH = rw.lastH; v.lastE = rw.lastE; v.argH = rw.argH; v.argE = rw.argE; v.tb = rw.tb; v.steps = rw.steps;
    uint32_t seed_u = 0xffffffffu, seed_o = 0, seed_q = 0;
    if (best < n_ext) { const gb_extension e = rw.ext[best]; seed_u = rescue_index_of(rw, n_ids, rw.path_pool[e.path_off]); seed_o = e.offset; seed_q = e.read_lo; }
    const uint32_t gap_limit = longest_detectable_gap(sc, L, L / 2);
    int32_t score = 0;
    xd_align(ix, sc, v, sread, L, seed_u, seed_o, seed_q, gap_limit, qbuf, dps, score, out, status);
    if (status != GB_ITEM_OK) return 0;
    if (score <= 0) { out.n_maps = 0; out.n_edits = 0; }
    if (lane == 0) for (uint32_t x = 0; x < out.n_maps; x++) out.maps[x].node = rw.nodes[out.maps[x].node];
    __syncwarp();
    // fix_dozeu_score (:3502-3517)
    int32_t rescored = 0;
    if (lane == 0 && out.n_maps > 0) rescored = rescue_rescore(sc, out);
    rescored = __shfl_sync(FULL, rescored, 0);
    if (rescored > 0) score = rescored;
    else {
        sw_align(ix, sc, v, sread, L, qbuf, dps, score, out, status);
        if (status != GB_ITEM_OK) return 0;
        if (lane == 0) for (uint32_t x = 0; x < out.n_maps; x++) out.maps[x].node = rw.nodes[out.maps[x].node];
        __syncwarp();
    }
    if (lane == 0) rescue_fix_end_deletions(out);
    out.n_maps = __shfl_sync(FULL, out.n_maps, 0); out.n_edits = __shfl_sync(FULL, out.n_edits, 0);
    __syncwarp();
    if (out.n_maps == 0) score = 0;
    // chance filter (:3451-3481)
    const int64_t effective_matches = score / sc.match;
    const int64_t subgraph_size = bases;
    if (effective_matches <= (int64_t)L && effective_matches <= subgraph_size) {
        const double by_chance = 1.0 - pow(1.0 - pow(0.25, (double)effective_matches), (double)(((int64_t)L - effective_matches + 1) * (subgraph_size - effective_matches + 1)));
        if (by_chance > P.rescue_likelihood_limit) { out.n_maps = 0; out.n_edits = 0; score = 0; }
    }
    if (out.n_maps + 1 > out.map_cap) { status = GB_ITEM_OUT_FULL; return 0; }
    return score;
}

constexpr uint32_t RESCUE_MAX_PAIRS = 96;
enum : uint8_t { PT_PAIRED = 0, PT_UNPAIRED = 1, PT_RESCUED_FROM_FIRST = 2, PT_RESCUED_FROM_SECOND = 3 };

// Pairing, rescue, winner and MAPQ of one pair when max_rescue_attempts != 0 (minimizer_mapper.cpp:2046-2777;
// oracle/mapper_paired.cpp).  `cl` grows by the rescued alignments (fragment id = the extra last fragment).
__device__ inline uint32_t finalize_pe_rescue(const DevIndex& ix, const MapParamsDev& P, const DevScores& sc, const ReadState* rs /*[2]*/, const PairState& ps,
                                              const AlignArgs& a, CandList& cl, const uint32_t (*explored)[PRESENT_WORDS], DevRng& rng,
                                              const uint8_t* const* sread, const uint8_t* const* qual, const uint32_t* L, uint32_t read_idx0,
                                              DpSmem dps, uint8_t* qbuf, uint8_t* cand_base, bool* slot_used, const RescueWs& rw, uint32_t Lc,
                                              gb_alignment* out /*[2]*/, gb_mapping* const* out_maps, uint32_t* const* out_edits) {
    const int lane = lane_id();
    const uint32_t map_cap = P.mapping_cap, edit_cap = P.edit_cap;
#pragma unroll 1
    for (uint32_t r = 0; r < 2; r++) {
        out[r].read_id = read_idx0 + r; out[r].score = 0; out[r].mapq = 0; out[r].flags = GB_ALN_PAIRED; out[r].n_mappings = 0; out[r].n_edits = 0;
        out[r].mapq_uncapped = 0.f; out[r].mapq_explored_cap = 0.f;
    }
    const uint32_t rescue_frag = ps.n_fragments;               // alignments.back(): the fragment that collects rescued alignments
    double pair_score[RESCUE_MAX_PAIRS]; int64_t pair_dist[RESCUE_MAX_PAIRS];
    uint8_t pair_c0[RESCUE_MAX_PAIRS], pair_c1[RESCUE_MAX_PAIRS], pair_better[RESCUE_MAX_PAIRS], pair_type[RESCUE_MAX_PAIRS];
    uint32_t n_pairs, n_unpaired; bool found_pair;
    uint8_t unpaired[2 * MAX_CANDS];
    uint32_t status = GB_ITEM_OK;
    int32_t best_alignment_scores[2] = {0, 0};
#pragma unroll 1
    for (uint32_t c = 0; c < cl.n; c++) best_alignment_scores[cl.read[c]] = max(best_alignment_scores[cl.read[c]], cl.score[c]);
    auto frag_of = [&](uint32_t c) { return (uint32_t)cl.frag[c]; };
    auto read_of = [&](uint32_t c) { return (uint32_t)cl.read[c]; };
    auto score_of = [&](uint32_t c) { return cl.score[c]; };
    // distance_between(first mate's alignment c0, second mate's alignment c1)
    auto dist_of = [&](uint32_t c0, uint32_t c1) {
        return distance_between(ix, slot_buf(cand_base, cl.slot[c0], map_cap, edit_cap), slot_buf(cand_base, cl.slot[c1], map_cap, edit_cap));
    };
    // the fragments of the clusters: rescue_frag is still empty
    if (!collect_pairs<RESCUE_MAX_PAIRS>(cl.n, rescue_frag, frag_of, read_of, score_of, dist_of, ps.better_cluster_count, a.frag_mean, a.frag_sd, P.log_base,
                                         pair_score, pair_dist, pair_c0, pair_c1, pair_better, n_pairs, found_pair, unpaired, n_unpaired))
        return GB_ITEM_OUT_FULL;
#pragma unroll 1
    for (uint32_t p = 0; p < n_pairs; p++) pair_type[p] = PT_PAIRED;
    // per end: the unpaired alignments and their scores (the MAPQ cap of an unpaired winner)
    uint32_t unpaired_count[2] = {0, 0}, rescued_count[2] = {0, 0};
    double unpaired_scores[2][2 * MAX_CANDS];
#pragma unroll 1
    for (uint32_t u = 0; u < n_unpaired; u++) { const uint32_t c = unpaired[u], r = cl.read[c]; unpaired_scores[r][unpaired_count[r]++] = (double)cl.score[c]; }

    if (n_unpaired > 0) {
        if (!found_pair) {
            int best_c[2]; int32_t best_score[2];
            best_unpaired_per_end(unpaired, n_unpaired, read_of, score_of, rng, best_c, best_score);
            if (best_score[0] != 0 && best_score[1] != 0) {
                // the best alignments of the two ends as an (unpaired) pair at "infinite" distance (:2288-2334)
                pair_score[n_pairs] = score_alignment_pair(cl.score[best_c[0]], cl.score[best_c[1]], INT64_MAX, a.frag_mean, a.frag_sd, P.log_base);
                pair_dist[n_pairs] = INT64_MAX;
                pair_c0[n_pairs] = (uint8_t)best_c[0]; pair_c1[n_pairs] = (uint8_t)best_c[1]; pair_better[n_pairs] = 0; pair_type[n_pairs] = PT_UNPAIRED;
                n_pairs++;
            }
        }
        // rescue from the unpaired alignments, best first (:2338-2457)
        uint8_t uo[2 * MAX_CANDS];
        sort_shuffling_ties(n_unpaired, [&](uint32_t x, uint32_t y) { return cl.score[unpaired[x]] > cl.score[unpaired[y]]; }, uo, rng);
        uint32_t unskipped = 0;
#pragma unroll 1
        for (uint32_t oi = 0; oi < n_unpaired && status == GB_ITEM_OK; oi++) {
            if (unskipped >= P.max_rescue_attempts) continue;
            unskipped++;
            const uint32_t c = unpaired[uo[oi]]; const uint32_t r = cl.read[c], other = 1 - r;
            if (found_pair && (double)cl.score[c] < (double)best_alignment_scores[r] * P.paired_rescue_score_limit) continue;
            if (cl.n >= 2 * MAX_CANDS + 32 || n_pairs >= RESCUE_MAX_PAIRS) { status = GB_ITEM_OUT_FULL; break; }
            uint32_t slot = 0xffffffffu;
#pragma unroll 1
            for (uint32_t i = 0; i < N_SLOTS; i++) if (!slot_used[i]) { slot_used[i] = true; slot = i; break; }
            if (slot == 0xffffffffu) { status = GB_ITEM_OUT_FULL; break; }
            const PathBuf anchor = slot_buf(cand_base, cl.slot[c], map_cap, edit_cap);
            PathBuf pb = slot_buf(cand_base, slot, map_cap, edit_cap);
            const int32_t rescued_score = attempt_rescue(ix, P, sc, rw, anchor, slot_nm(anchor), slot_ne(anchor), sread[other], L[other],
                                                         a.minimizers + rs[other].min_off, rs[other].min_cnt, r == 0, a.frag_mean, a.frag_sd,
                                                         qbuf, dps, Lc, pb, status);
            if (status != GB_ITEM_OK) break;
            if (lane == 0) { slot_nm(pb) = pb.n_maps; slot_ne(pb) = pb.n_edits; }
            __syncwarp();
            const uint32_t cr = cl.n;
            cl.score[cr] = rescued_score; cl.slot[cr] = (uint8_t)slot; cl.frag[cr] = (uint8_t)rescue_frag; cl.read[cr] = (uint8_t)other; cl.n++;
            int64_t dist; double score;
            if (pb.n_maps != 0) {
                dist = r == 0 ? dist_of(c, cr) : dist_of(cr, c);
                score = score_alignment_pair(cl.score[c], rescued_score, dist, a.frag_mean, a.frag_sd, P.log_base);
            }
            else { score = (double)cl.score[c]; dist = INT64_MAX; }
            pair_score[n_pairs] = score; pair_dist[n_pairs] = dist;
            pair_c0[n_pairs] = (uint8_t)(r == 0 ? c : cr); pair_c1[n_pairs] = (uint8_t)(r == 0 ? cr : c);
            pair_better[n_pairs] = ps.better_cluster_count[cl.frag[c]]; pair_type[n_pairs] = r == 0 ? PT_RESCUED_FROM_FIRST : PT_RESCUED_FROM_SECOND;
            n_pairs++; rescued_count[r]++;
        }
        if (status != GB_ITEM_OK) return status;
    }
    if (n_pairs == 0) return GB_ITEM_OK;

    // winner (:2505-2598)
    uint8_t po[RESCUE_MAX_PAIRS];
    sort_shuffling_ties(n_pairs, [&](uint32_t x, uint32_t y) { return pair_score[x] > pair_score[y]; }, po, rng);
    double scores_sorted[RESCUE_MAX_PAIRS], mult[RESCUE_MAX_PAIRS];
    double est_mult[2];
#pragma unroll 1
    for (uint32_t r = 0; r < 2; r++) est_mult[r] = unpaired_count[r] > 0 ? (double)unpaired_count[r] / (double)min(rescued_count[r], P.max_rescue_attempts) : 1.0;
    bool all_rescued = true;
#pragma unroll 1
    for (uint32_t p = 0; p < n_pairs; p++) {
        scores_sorted[p] = pair_score[po[p]];
        const uint8_t t = pair_type[po[p]];
        if (t == PT_PAIRED) { mult[p] = 1.0; all_rescued = false; }
        else if (t == PT_UNPAIRED) mult[p] = 1.0;
        else mult[p] = est_mult[t == PT_RESCUED_FROM_FIRST ? 0 : 1];
    }
    const uint32_t wp = po[0];
    const double uncapped_mapq = scores_sorted[0] == 0 ? 0.0 : max_mapping_quality(scores_sorted, n_pairs, P.log_base, all_rescued ? mult : nullptr);
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
        if (cl.frag[cwin[r]] == rescue_frag) out[r].flags |= GB_ALN_RESCUED;
        const double unpaired_cap = pair_type[wp] == PT_UNPAIRED ? max_mapping_quality(unpaired_scores[r], unpaired_count[r], P.log_base) : INFINITY;   // :2735-2739
        pair_read_mapq(uncapped_mapq, cluster_cap, caps[0] + caps[1], pair_dist[wp] == INT64_MAX, unpaired_cap, out[r]);
        if (lane == 0 && nm) write_alignment(ix, pb, nm, ne, sread[r], L[r], r == 1, out_maps[r], out_edits[r]);
    }
    __syncwarp();
    if (P.max_multimaps > 1) return write_secondary_pairs(ix, P, a, cl, po, n_pairs, pair_c0, pair_c1, rescue_frag, sread, L, read_idx0, cand_base);
    return GB_ITEM_OK;
}
