// tail.cuh — haplotype tail forest + pinned X-drop alignment, one warp per problem.
//
//   get_tail_forest / dfs_gbwt                 minimizer_mapper.cpp:5745-6013
//   get_best_alignment_against_any_tree        minimizer_mapper.cpp:5626-5743
//   Aligner::align_pinned (xdrop)              aligner.cpp:628-686
//   DozeuInterface::align_pinned / do_poa      dozeu_interface.cpp:210-307, :724-766
//   traceback -> Path                          dozeu_interface.cpp:338-572
//   dz_extend / dz_trace                       vgteam/dozeu @ d0e9ba6 (ABSENT; semantics as
//                                              stated in oracle/tail_align.cpp, the contract)
//
// The DP is a warp-synchronous column sweep: the 32 lanes hold 32 consecutive query offsets
// of a column; the in-column insertion dependency is resolved with a max-plus prefix scan over
// the lanes (shuffles), the X-drop test and the column maximum with warp reductions, and every
// cell leaves one traceback byte in HBM.  Integer arithmetic only (int32).
#pragma once
#include "map_state.cuh"

namespace gb {

constexpr int32_t DP_NEG = INT_MIN / 4;
constexpr uint32_t TAIL_T_CAP = 2048;     // tree nodes per forest
constexpr uint32_t TAIL_S_CAP = 2048;     // DFS stack frames
constexpr uint32_t TAIL_D_CAP = 512;      // tree depth
constexpr uint32_t TAIL_STEP_CAP = 4096;  // traceback steps (TILE_STEP_CAP of xdrop_tile.cuh: a path fits both kernels or neither)

struct TreeNode {
    int32_t parent;        // index in the forest array, -1 for a tree root
    uint32_t node;         // oriented graph node
    uint32_t seq_off;      // sequence start (root: already trimmed)
    uint32_t len;          // bases used (root: trimmed length)
    uint32_t depth;
    uint32_t tb_col;       // first traceback column of this node
    int32_t lineage_max;
    uint16_t computed;
    uint8_t band_lo, band_hi;   // live 32-cell chunks [lo, hi) of the node's last DP column
};

struct DfsFrame { uint32_t node; int32_t lo, hi; uint32_t used; uint32_t visit; };

// Per-warp HBM workspace for tail alignment.
struct TailWs {
    TreeNode* tree;        // [TAIL_T_CAP]
    DfsFrame* stack;       // [TAIL_S_CAP]
    uint32_t* pstack;      // [TAIL_D_CAP]
    int32_t* colH;         // [TAIL_D_CAP][Lc + 1]   last column of the node at each depth
    int32_t* colE;
    uint8_t* tb;           // [tb_cells]             one byte per DP cell
    uint32_t* steps;       // [TAIL_STEP_CAP]        (tree node << 8) | op
    uint32_t tb_cells;
    uint32_t Lc;
};

__host__ __device__ inline size_t tail_ws_bytes(uint32_t Lc, uint32_t tb_cells) {
    size_t b = 0;
    b += sizeof(TreeNode) * TAIL_T_CAP;
    b += sizeof(DfsFrame) * TAIL_S_CAP;
    b += 4 * TAIL_D_CAP;
    b += (size_t)4 * TAIL_D_CAP * (Lc + 1) * 2;
    b += 4 * TAIL_STEP_CAP;
    b += tb_cells;
    return (b + 255) & ~(size_t)255;
}

__device__ inline TailWs carve_tail_ws(uint8_t* base, uint32_t Lc, uint32_t tb_cells) {
    TailWs w; uint8_t* p = base;
    w.tree = (TreeNode*)p; p += sizeof(TreeNode) * TAIL_T_CAP;
    w.stack = (DfsFrame*)p; p += sizeof(DfsFrame) * TAIL_S_CAP;
    w.pstack = (uint32_t*)p; p += 4 * TAIL_D_CAP;
    w.colH = (int32_t*)p; p += (size_t)4 * TAIL_D_CAP * (Lc + 1);
    w.colE = (int32_t*)p; p += (size_t)4 * TAIL_D_CAP * (Lc + 1);
    w.steps = (uint32_t*)p; p += 4 * TAIL_STEP_CAP;
    w.tb = p;
    w.tb_cells = tb_cells; w.Lc = Lc;
    return w;
}

// A path under construction: mappings + edits in two flat arrays (device-side Path).
struct PathBuf {
    gb_mapping* maps; uint32_t* edits;
    uint32_t n_maps, n_edits, map_cap, edit_cap;
    bool overflow;
};
__device__ __forceinline__ void pb_reset(PathBuf& p) { p.n_maps = 0; p.n_edits = 0; p.overflow = false; }
__device__ __forceinline__ void pb_add_mapping(PathBuf& p, uint32_t node, uint32_t offset) {
    if (p.n_maps >= p.map_cap) { p.overflow = true; return; }
    gb_mapping m; m.node = node; m.offset = (uint16_t)offset; m.n_edits = 0;
    p.maps[p.n_maps++] = m;
}
__device__ __forceinline__ void pb_add_edit(PathBuf& p, uint32_t word) {
    if (p.n_edits >= p.edit_cap || p.n_maps == 0) { p.overflow = true; return; }
    p.edits[p.n_edits++] = word;
    p.maps[p.n_maps - 1].n_edits++;
}
__device__ __forceinline__ uint32_t edit_word(uint32_t op, uint32_t len, uint32_t base) { return (len << 4) | (base << 2) | op; }
__device__ __forceinline__ uint32_t base2(uint8_t c) { return c == 'C' ? 1u : (c == 'G' ? 2u : (c == 'T' ? 3u : 0u)); }
__device__ __forceinline__ uint8_t comp_base(uint8_t c) { return c == 'A' ? 'T' : (c == 'C' ? 'G' : (c == 'G' ? 'C' : (c == 'T' ? 'A' : 'N'))); }
__device__ __forceinline__ bool is_acgt(uint8_t c) { return c == 'A' || c == 'C' || c == 'G' || c == 'T'; }
// DP queries are staged with every non-ACGT byte replaced by 0, which equals no graph base: the
// "non-ACGT never matches" rule then costs nothing in the inner loop.
__device__ __forceinline__ uint8_t dp_query_base(uint8_t c) { return is_acgt(c) ? c : (uint8_t)0; }

// EditAlignmentScorer::longest_detectable_gap(read_length, read_pos), alignment_scorer.cpp:264-271
__device__ __forceinline__ uint32_t longest_detectable_gap(const DevScores& s, uint32_t read_length, uint32_t read_pos) {
    const int64_t overhang = min(read_pos, read_length - read_pos);
    const int64_t numer = (int64_t)s.match * overhang + s.full_length_bonus;
    const int64_t gap = (numer - s.gap_open) / s.gap_extend + 1;
    return (gap >= 0 && overhang > 0) ? (uint32_t)gap : 0u;
}

// -----------------------------------------------------------------------------------------
// Haplotype DFS (dfs_gbwt) building the forest in ws.tree; returns number of forest nodes, or
// 0xffffffff on workspace overflow.  root_trim receives the offset trimmed from each root.
// -----------------------------------------------------------------------------------------
__device__ inline uint32_t build_tail_forest(const DevIndex& ix, const TailWs& ws, uint32_t start_node, int32_t lo, int32_t hi,
                                             uint32_t from_offset, uint32_t walk_distance, uint32_t& root_trim) {
    const int lane = lane_id();
    if (lo > hi) return 0;
    const gb_node_rec start_rec = load_node(ix, start_node);
    const uint32_t remaining_root = start_rec.len - from_offset;
    const bool start_included = from_offset < start_rec.len;
    root_trim = start_included ? from_offset : 0u;
    uint32_t sp = 0, n_tree = 0, pdepth = 0;
    if (lane == 0) ws.stack[0] = DfsFrame{start_node, lo, hi, 0u, 0u};
    sp = 1;
    __syncwarp();
#pragma unroll 1
    while (sp > 0) {
        const DfsFrame f = ws.stack[sp - 1];
        const bool is_root = (sp == 1);
        const bool hidden = is_root && remaining_root == 0;
        const gb_node_rec nr = load_node(ix, f.node);
        if (!f.visit) {
            if (!hidden) {
                if (n_tree >= TAIL_T_CAP || pdepth >= TAIL_D_CAP) return 0xffffffffu;
                if (lane == 0) {
                    TreeNode t;
                    t.parent = pdepth == 0 ? -1 : (int32_t)ws.pstack[pdepth - 1];
                    t.node = f.node;
                    const bool trimmed_root = is_root;       // only the DFS root is trimmed
                    t.seq_off = nr.seq_off + (trimmed_root ? from_offset : 0u);
                    t.len = trimmed_root ? remaining_root : nr.len;
                    t.depth = pdepth; t.tb_col = 0; t.lineage_max = 0; t.computed = 0;
                    ws.tree[n_tree] = t;
                    ws.pstack[pdepth] = n_tree;
                }
                n_tree++; pdepth++;
            }
            const uint32_t node_length = is_root ? remaining_root : nr.len;
            const uint32_t used = f.used + node_length;
            if (lane == 0) { ws.stack[sp - 1].visit = 1; ws.stack[sp - 1].used = used; }
            __syncwarp();
            if (used < walk_distance) {
                const EdgeFan fan = record_fan(ix, nr, f.lo, f.hi);
                bool pushed_any = false;
#pragma unroll 1
                for (uint32_t e = 0; e < fan.n_edges; e++) {
                    uint32_t to; int32_t first, cnt, rev;
                    if (fan.n_edges <= 32) {
                        to = __shfl_sync(FULL, fan.to, e); first = __shfl_sync(FULL, fan.first, e); cnt = __shfl_sync(FULL, fan.cnt, e);
                    } else {
                        record_edge_generic(ix, nr, f.lo, f.hi, e, to, first, cnt, rev);
                    }
                    if (to == 0 || cnt <= 0) continue;
                    if (sp >= TAIL_S_CAP) return 0xffffffffu;
                    if (lane == 0) ws.stack[sp] = DfsFrame{to, first, first + cnt - 1, used, 0u};
                    sp++; pushed_any = true;
                }
                __syncwarp();
                (void)pushed_any;
                continue;
            }
        }
        if (!hidden) pdepth--;
        sp--;
    }
    __syncwarp();
    return n_tree;
}

// -----------------------------------------------------------------------------------------
// Pinned X-drop DP over trees [t0, t1) of the forest (one tree), query q[0..m) in shared memory.
// sH/sE/sHc/sEc: per-warp shared columns of m+1 ints.  Writes the alignment (tree space:
// mapping.node = forest index) into `out`; returns the score (0 = softclip on the tree root).
// -----------------------------------------------------------------------------------------
struct DpSmem { int32_t *Hp, *Ep, *Hc, *Ec; };

// Dynamic shared memory per warp of the one-warp DP kernels (sw_kernel, xdrop_dag_kernel, xdrop_kernel):
// the staged query (Lc bytes, rounded up to 16), then the four DP columns of Lc + 1 cells, then 64 spare bytes.
__host__ __device__ inline size_t dp_smem_per_warp(uint32_t Lc) {
    return (((size_t)Lc + 15) & ~(size_t)15) + ((size_t)Lc + 1) * 4 * 4 + 64;
}
// the four DP columns at `cols`
__device__ inline DpSmem dp_cols_carve(int32_t* cols, uint32_t Lc) {
    const uint32_t W = Lc + 1;
    DpSmem dps; dps.Hp = cols; dps.Ep = cols + W; dps.Hc = cols + 2 * W; dps.Ec = cols + 3 * W;
    return dps;
}
// warp `warp`'s query buffer (q) and DP columns within that layout
__device__ inline DpSmem dp_smem_carve(uint8_t* smem, int warp, uint32_t Lc, uint8_t*& q) {
    uint8_t* base = smem + (size_t)warp * dp_smem_per_warp(Lc);
    q = base;
    return dp_cols_carve(reinterpret_cast<int32_t*>(base + (((size_t)Lc + 15) & ~(size_t)15)), Lc);
}

__device__ inline int32_t xdrop_tree(const DevIndex& ix, const DevScores& sc, const TailWs& ws, DpSmem dps,
                                     uint32_t t0, uint32_t t1, const uint8_t* q, uint32_t m, uint32_t max_gap,
                                     PathBuf& out, bool& overflow) {
    const int lane = lane_id();
    const int32_t go = sc.gap_open, ge = sc.gap_extend;
    const int32_t xt = go + ge * ((int32_t)max_gap - 1);
    const uint32_t W = m + 1;
    pb_reset(out);
    overflow = false;

    int32_t best = 0; uint32_t best_node = 0, best_col = 0, best_j = 0; bool have_best = false;
    uint32_t tb_cols = 0;
    const uint32_t n_chunks = (W + 31) >> 5;
#pragma unroll 1
    for (uint32_t i = t0; i < t1; i++) {
        TreeNode tn = ws.tree[i];
        int32_t run_max;
        // Cells outside the live chunk range [plo, phi) of the previous column are dead by definition
        // and are never read; the X-drop keeps that range a narrow band around the best diagonal.
        uint32_t plo, phi;
        if (tn.parent < 0) {
#pragma unroll 1
            for (uint32_t j = lane; j < W; j += 32) {
                int32_t h = DP_NEG;
                if (j == 0) h = 0; else if (j <= max_gap) h = -(go + (int32_t)(j - 1) * ge);
                dps.Hp[j] = h; dps.Ep[j] = DP_NEG;
            }
            plo = 0; phi = min(n_chunks, (min(max_gap, m) >> 5) + 1);
            run_max = 0;
        } else {
            const TreeNode par = ws.tree[tn.parent];
            if (!par.computed || par.band_lo >= par.band_hi) { continue; }
            plo = par.band_lo; phi = par.band_hi;
            const int32_t* cH = ws.colH + (size_t)par.depth * (ws.Lc + 1);
            const int32_t* cE = ws.colE + (size_t)par.depth * (ws.Lc + 1);
#pragma unroll 1
            for (uint32_t j = plo * 32 + lane; j < min(W, phi * 32); j += 32) { dps.Hp[j] = cH[j]; dps.Ep[j] = cE[j]; }
            run_max = par.lineage_max;
        }
        __syncwarp();
        if ((uint64_t)(tb_cols + tn.len) * W > ws.tb_cells) { overflow = true; return 0; }
        tn.tb_col = tb_cols; tn.computed = 1;
        // this lane's best cell of the node: first column, then smallest j, on ties (strict > below)
        int32_t lane_best = DP_NEG; uint32_t lane_col = 0, lane_j = 0;
#pragma unroll 1
        for (uint32_t c = 0; c < tn.len && plo < phi; c++) {
            const uint8_t r = __ldg(ix.seq + tn.seq_off + c);
            uint8_t* tbcol = ws.tb + (size_t)(tb_cols + c) * W;
            int32_t carry = INT_MIN;          // running max of (H'[i] + i*ge) over i < chunk start
            int32_t prevH_last = DP_NEG;      // H of the last cell of the previous chunk (for f_open)
            int32_t prev_ph_last = DP_NEG;    // previous column's H of the last cell of the previous chunk (diagonal)
            int32_t col_max = DP_NEG;
            uint32_t clo = n_chunks, chi = 0;
#pragma unroll 1
            for (uint32_t ch = plo; ch < n_chunks; ch++) {
                const uint32_t j = ch * 32 + lane;
                const bool in = j < W;
                const bool pin = in && ch < phi;                  // previous column has this chunk
                int32_t ph = DP_NEG, pe = DP_NEG;
                if (pin) { ph = dps.Hp[j]; pe = dps.Ep[j]; }
                int32_t phm1 = __shfl_up_sync(FULL, ph, 1);
                if (lane == 0) phm1 = prev_ph_last;
                prev_ph_last = __shfl_sync(FULL, ph, 31);
                int32_t e = DP_NEG;
                if (ph > DP_NEG) e = ph - go;
                if (pe > DP_NEG) e = max(e, pe - ge);
                int32_t d = DP_NEG;
                if (in && j > 0 && phm1 > DP_NEG) {
                    const uint8_t qc = q[j - 1];
                    int32_t s = (qc == r) ? sc.match : -sc.mismatch;
                    if (j == m) s += sc.full_length_bonus;
                    d = phm1 + s;
                }
                const int32_t hprime = max(d, e);
                // insertion chain: F[j] = max_{i<j, H'[i] live} (H'[i] + i*ge) - go - (j-1)*ge
                int32_t g = (in && hprime > DP_NEG) ? hprime + (int32_t)j * ge : INT_MIN;
                int32_t incl = g;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int32_t t = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl = max(incl, t); }
                int32_t excl = __shfl_up_sync(FULL, incl, 1);
                if (lane == 0) excl = INT_MIN;
                excl = max(excl, carry);
                carry = max(carry, __shfl_sync(FULL, incl, 31));
                int32_t f = DP_NEG;
                if (in && j > 0 && excl > INT_MIN) f = excl - go - (int32_t)(j - 1) * ge;
                int32_t h = max(hprime, f);
                // traceback byte: bits 0-1 source (0 diag, 1 E, 2 F), bit 2 E opened, bit 3 F opened
                int32_t hm1 = __shfl_up_sync(FULL, h, 1);
                if (lane == 0) hm1 = prevH_last;
                prevH_last = __shfl_sync(FULL, h, 31);
                uint8_t tbv = 0;
                if (in) {
                    if (d > DP_NEG && d == h) tbv = 0; else if (e > DP_NEG && e == h) tbv = 1; else tbv = 2;
                    if (ph > DP_NEG && e == ph - go) tbv |= 4;
                    if (j > 0 && hm1 > DP_NEG && f == hm1 - go) tbv |= 8;
                }
                // X-drop against the best of the earlier columns
                if (in && h > DP_NEG && h < run_max - xt) { h = DP_NEG; e = DP_NEG; }
                if (in) { dps.Hc[j] = h; dps.Ec[j] = e; tbcol[j] = tbv; }
                const bool alive = in && h > DP_NEG;
                if (alive) {
                    col_max = max(col_max, h);
                    if (h > lane_best) { lane_best = h; lane_col = c; lane_j = j; }
                }
                if (__any_sync(FULL, alive || (in && e > DP_NEG))) { clo = min(clo, ch); chi = ch + 1; }
                else if (ch >= phi) break;                // past the previous band (+1 chunk for the diagonal) and the insertion chain died
            }
            __syncwarp();
            col_max = __reduce_max_sync(FULL, col_max);
            if (col_max > run_max) run_max = col_max;
            // swap columns
            int32_t* t1p = dps.Hp; dps.Hp = dps.Hc; dps.Hc = t1p;
            int32_t* t2p = dps.Ep; dps.Ep = dps.Ec; dps.Ec = t2p;
            plo = clo; phi = chi;
        }
        // node maximum across lanes: highest score, then first column, then smallest query offset
        int32_t node_best = lane_best; uint32_t node_col = lane_col, node_j = lane_j;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const int32_t oh = __shfl_xor_sync(FULL, node_best, o);
            const uint32_t oc = __shfl_xor_sync(FULL, node_col, o), oj = __shfl_xor_sync(FULL, node_j, o);
            if (oh > node_best || (oh == node_best && (oc < node_col || (oc == node_col && oj < node_j)))) { node_best = oh; node_col = oc; node_j = oj; }
        }
        // keep this node's last column (its live band) for its children
        if (plo < phi) {
            int32_t* cH = ws.colH + (size_t)tn.depth * (ws.Lc + 1);
            int32_t* cE = ws.colE + (size_t)tn.depth * (ws.Lc + 1);
#pragma unroll 1
            for (uint32_t j = plo * 32 + lane; j < min(W, phi * 32); j += 32) { cH[j] = dps.Hp[j]; cE[j] = dps.Ep[j]; }
        }
        tn.band_lo = (uint8_t)min(plo, 255u); tn.band_hi = (uint8_t)(plo < phi ? phi : min(plo, 255u));
        tn.lineage_max = run_max;
        if (lane == 0) ws.tree[i] = tn;
        tb_cols += tn.len;
        if (node_best > best) { best = node_best; best_node = i; best_col = node_col; best_j = node_j; have_best = true; }
        __syncwarp();
    }

    if (!have_best || best <= 0) {
        // full-length insertion on the head node (dozeu_interface.cpp:344-360)
        if (lane == 0) { pb_add_mapping(out, t0, 0); pb_add_edit(out, edit_word(GB_EDIT_INS, m, 0)); }
        __syncwarp();
        out.n_maps = __shfl_sync(FULL, out.n_maps, 0); out.n_edits = __shfl_sync(FULL, out.n_edits, 0);
        out.overflow = __shfl_sync(FULL, (int)out.overflow, 0) != 0;
        return 0;
    }

    // ---- traceback (uniform; every lane walks the same bytes) --------------------------------
    // steps are recorded end -> start as (forest node << 8) | op, op: 0 M, 1 X, 2 I, 3 D
    uint32_t n_steps = 0;
    {
        uint32_t node = best_node, col = best_col, j = best_j;
        int state = 0;   // 0 H, 1 E, 2 F
        bool at_virtual = false;
#pragma unroll 1
        while (true) {
            if (at_virtual) {
#pragma unroll 1
                for (; j > 0; j--) { if (n_steps >= TAIL_STEP_CAP) { overflow = true; return 0; } if (lane == 0) ws.steps[n_steps] = (t0 << 8) | 2u; n_steps++; }
                break;
            }
            const TreeNode tn = ws.tree[node];
            const uint8_t tbv = ws.tb[(size_t)(tn.tb_col + col) * W + j];
            // predecessor column
            uint32_t pnode = node, pcol = 0; bool p_virtual = false;
            if (col > 0) pcol = col - 1;
            else if (tn.parent < 0) p_virtual = true;
            else { pnode = (uint32_t)tn.parent; pcol = ws.tree[pnode].len - 1; }
            if (n_steps >= TAIL_STEP_CAP) { overflow = true; return 0; }
            if (state == 0) {
                const uint32_t src = tbv & 3u;
                if (src == 0) {
                    if (j == 0) { overflow = true; return 0; }          // corrupt traceback: refuse, never walk off the matrix
                    const uint8_t qc = q[j - 1], r = __ldg(ix.seq + tn.seq_off + col);
                    if (lane == 0) ws.steps[n_steps] = (node << 8) | ((qc == r) ? 0u : 1u);
                    n_steps++;
                    j--; node = pnode; col = pcol; at_virtual = p_virtual;
                    if (at_virtual && j == 0) break;
                    continue;
                }
                state = src == 1 ? 1 : 2;
                continue;
            }
            if (state == 1) {
                if (lane == 0) ws.steps[n_steps] = (node << 8) | 3u;
                n_steps++;
                const bool open = (tbv & 4u) != 0;
                node = pnode; col = pcol; at_virtual = p_virtual;
                state = open ? 0 : 1;
                if (at_virtual && j == 0 && state == 0) break;
                continue;
            }
            if (lane == 0) ws.steps[n_steps] = (node << 8) | 2u;
            n_steps++;
            const bool open = (tbv & 8u) != 0;
            if (j == 0) { overflow = true; return 0; }
            j--;
            state = open ? 0 : 2;
        }
    }
    __syncwarp();

    // ---- steps -> mappings (calculate_and_save_alignment, dozeu_interface.cpp:493-533) ----------
    if (lane == 0) {
        uint32_t query_offset = 0;
        int64_t si = (int64_t)n_steps - 1;
#pragma unroll 1
        while (si >= 0) {
            const uint32_t nd = ws.steps[si] >> 8;
            pb_add_mapping(out, nd, 0);
            uint32_t cur = 0xff, run = 0;
            auto flush = [&]() {
                if (cur == 1) { for (uint32_t x = 0; x < run; x++) { pb_add_edit(out, edit_word(GB_EDIT_SUB, 1, base2(q[query_offset]))); query_offset++; } }
                else if (run > 0) {
                    if (cur == 0) { pb_add_edit(out, edit_word(GB_EDIT_MATCH, run, 0)); query_offset += run; }
                    else if (cur == 2) { pb_add_edit(out, edit_word(GB_EDIT_INS, run, 0)); query_offset += run; }
                    else if (cur == 3) { pb_add_edit(out, edit_word(GB_EDIT_DEL, run, 0)); }
                }
            };
#pragma unroll 1
            while (si >= 0 && (ws.steps[si] >> 8) == nd) {
                const uint32_t op = ws.steps[si] & 0xffu;
                if (op == cur) run++; else { if (cur != 0xff) flush(); cur = op; run = 1; }
                si--;
            }
            if (cur != 0xff) flush();
        }
        if (out.n_maps > 0 && query_offset != m) pb_add_edit(out, edit_word(GB_EDIT_INS, m - query_offset, 0));
    }
    __syncwarp();
    out.n_maps = __shfl_sync(FULL, out.n_maps, 0); out.n_edits = __shfl_sync(FULL, out.n_edits, 0);
    out.overflow = __shfl_sync(FULL, (int)out.overflow, 0) != 0;
    return best;
}

} // namespace gb
