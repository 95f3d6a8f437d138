// dag_dp.cuh — read-vs-DAG dynamic programming shared by the stage seams (full_dp.cu, xdrop_dag.cu) and the
// rescue path of the paired-end align kernel: the full local DP (GSSW replacement) and the seeded two-pass
// X-drop alignment (align_xdrop).  One warp per problem; the problem is described by a DagView whose
// workspaces the caller owns.  Rules: oracle/full_dp.cpp, oracle/xdrop_dag.cpp.
#pragma once
#include "align.cuh"

namespace gb {

struct XdNode { int32_t lineage_max; uint32_t first_col; uint8_t computed, live, band_lo, band_hi; };


// A DAG problem and its workspaces.  pred_off / succ_off are indexed by the node's position in the
// problem and index into pred / succ, whose entries are positions in the problem as well.
struct DagView {
    uint32_t N; const uint32_t* node;
    const uint32_t* pred; const uint64_t* pred_off;
    const uint32_t* succ; const uint64_t* succ_off;           // only the X-drop passes need successors
    uint32_t* col_start; uint32_t* seq_off; uint32_t* seq_len; XdNode* nstate;      // [N]
    int32_t* lastH; int32_t* lastE; uint8_t* argH; uint8_t* argE;                 // [N * (m + 1)]
    uint8_t* tb;                                                                  // [bases * (m + 1)]
    uint32_t* steps;                                                              // [bases + m + 2]
};

struct XdBest { int32_t best; uint32_t t, c, j; };

// One pinned X-drop pass over the (possibly mirrored) problem, starting before pass column `o` of pass
// node `s`, query q[0..m) in shared memory.  TB: write traceback bytes.
template <bool MIRROR, bool TB>
__device__ inline XdBest xd_pass(const DevIndex& ix, const DevScores& sc, const DagView& v,
                                 const uint8_t* q, uint32_t m, uint32_t s, uint32_t o, uint32_t max_gap, DpSmem dps) {
    const int lane = lane_id();
    const uint32_t W = m + 1, n_chunks = (W + 31) >> 5;
    const int32_t go = sc.gap_open, ge = sc.gap_extend;
    const int32_t xt = go + ge * ((int32_t)max_gap - 1);
    int32_t* lastH = v.lastH; int32_t* lastE = v.lastE;
    uint8_t* argH = v.argH; uint8_t* argE = v.argE;
    uint8_t* tb = v.tb;
    XdNode* ns = v.nstate; const uint32_t N = v.N;
    // the workspace rows are addressed by pass node index t with this pass's W
    for (uint32_t t = lane; t < N; t += 32) { XdNode z; z.lineage_max = 0; z.first_col = 0; z.computed = 0; z.live = 0; z.band_lo = 0; z.band_hi = 0; ns[t] = z; }
    __syncwarp();
    int32_t lane_best = DP_NEG; uint32_t lane_t = 0, lane_c = 0, lane_j = 0;
    for (uint32_t t = s; t < N; t++) {
        const uint32_t u = MIRROR ? N - 1 - t : t;
        const uint32_t len = v.seq_len[u], soff = v.seq_off[u];
        uint32_t plo, phi, first_col = 0; int32_t run_max;
        if (t == s) {
            for (uint32_t j = lane; j < W; j += 32) {
                int32_t h = DP_NEG;
                if (j == 0) h = 0; else if (j <= max_gap) h = -(go + (int32_t)(j - 1) * ge);
                dps.Hp[j] = h; dps.Ep[j] = DP_NEG;
            }
            plo = 0; phi = min(n_chunks, (min(max_gap, m) >> 5) + 1);
            run_max = 0; first_col = o;
        } else {
            // merge the last columns of the computed, live predecessors (pass order)
            const uint64_t e0 = MIRROR ? v.succ_off[u] : v.pred_off[u];
            const uint32_t ne = (uint32_t)((MIRROR ? v.succ_off[u + 1] : v.pred_off[u + 1]) - e0);
            plo = n_chunks; phi = 0; run_max = INT_MIN;
            bool any = false;
            for (uint32_t pi = 0; pi < ne; pi++) {
                const uint32_t pu = MIRROR ? v.succ[e0 + pi] : v.pred[e0 + pi];
                const uint32_t pt = MIRROR ? N - 1 - pu : pu;
                if (pt < s) continue;
                const XdNode pn = ns[pt];
                if (!pn.computed || !pn.live) continue;
                any = true;
                plo = min(plo, (uint32_t)pn.band_lo); phi = max(phi, (uint32_t)pn.band_hi);
                run_max = max(run_max, pn.lineage_max);
            }
            if (!any) continue;
            for (uint32_t j = plo * 32 + lane; j < min(W, phi * 32); j += 32) {
                int32_t h = DP_NEG, e = DP_NEG; uint32_t ah = 0xff, ae = 0xff;
                for (uint32_t pi = 0; pi < ne; pi++) {
                    const uint32_t pu = MIRROR ? v.succ[e0 + pi] : v.pred[e0 + pi];
                    const uint32_t pt = MIRROR ? N - 1 - pu : pu;
                    if (pt < s) continue;
                    const XdNode pn = ns[pt];
                    if (!pn.computed || !pn.live) continue;
                    if ((j >> 5) < pn.band_lo || (j >> 5) >= pn.band_hi) continue;
                    const int32_t ph = lastH[(size_t)pt * W + j], pe = lastE[(size_t)pt * W + j];
                    if (ph > h) { h = ph; ah = pi; }
                    if (pe > e) { e = pe; ae = pi; }
                }
                dps.Hp[j] = h; dps.Ep[j] = e;
                if (TB) { argH[(size_t)t * W + j] = (uint8_t)ah; argE[(size_t)t * W + j] = (uint8_t)ae; }
            }
        }
        __syncwarp();
        for (uint32_t c = first_col; c < len && plo < phi; c++) {
            const uint8_t r = __ldg(ix.seq + soff + (MIRROR ? len - 1 - c : c));
            uint8_t* tbcol = tb + (size_t)(v.col_start[u] + c) * W;
            int32_t carry = INT_MIN, prevH_last = DP_NEG, prev_ph_last = DP_NEG, col_max = DP_NEG;
            uint32_t clo = n_chunks, chi = 0;
            for (uint32_t ch = plo; ch < n_chunks; ch++) {
                const uint32_t j = ch * 32 + lane;
                const bool in = j < W;
                const bool pin = in && ch < phi;
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
                    int32_t sub = (qc == r) ? sc.match : -sc.mismatch;
                    if (j == m) sub += sc.full_length_bonus;
                    d = phm1 + sub;
                }
                const int32_t hprime = max(d, e);
                int32_t g = (in && hprime > DP_NEG) ? hprime + (int32_t)j * ge : INT_MIN;
                int32_t incl = g;
#pragma unroll
                for (int ofs = 1; ofs < 32; ofs <<= 1) { const int32_t tt = __shfl_up_sync(FULL, incl, ofs); if (lane >= ofs) incl = max(incl, tt); }
                int32_t excl = __shfl_up_sync(FULL, incl, 1);
                if (lane == 0) excl = INT_MIN;
                excl = max(excl, carry);
                carry = max(carry, __shfl_sync(FULL, incl, 31));
                int32_t f = DP_NEG;
                if (in && j > 0 && excl > INT_MIN) f = excl - go - (int32_t)(j - 1) * ge;
                int32_t h = max(hprime, f);
                int32_t hm1 = __shfl_up_sync(FULL, h, 1);
                if (lane == 0) hm1 = prevH_last;
                prevH_last = __shfl_sync(FULL, h, 31);
                uint8_t tbv = 0;
                if (TB && in) {
                    if (d > DP_NEG && d == h) tbv = 0; else if (e > DP_NEG && e == h) tbv = 1; else tbv = 2;
                    if (ph > DP_NEG && e == ph - go) tbv |= 4;
                    if (j > 0 && hm1 > DP_NEG && f == hm1 - go) tbv |= 8;
                }
                if (in && h > DP_NEG && h < run_max - xt) { h = DP_NEG; e = DP_NEG; }
                if (in) { dps.Hc[j] = h; dps.Ec[j] = e; if (TB) tbcol[j] = tbv; }
                const bool alive = in && h > DP_NEG;
                if (alive) {
                    col_max = max(col_max, h);
                    if (h > lane_best) { lane_best = h; lane_t = t; lane_c = c; lane_j = j; }
                }
                if (__any_sync(FULL, alive)) { clo = min(clo, ch); chi = ch + 1; }
                else if (ch >= phi) break;
            }
            __syncwarp();
            col_max = __reduce_max_sync(FULL, col_max);
            if (col_max > run_max) run_max = col_max;
            int32_t* t1p = dps.Hp; dps.Hp = dps.Hc; dps.Hc = t1p;
            int32_t* t2p = dps.Ep; dps.Ep = dps.Ec; dps.Ec = t2p;
            plo = clo; phi = chi;
        }
        if (plo < phi) for (uint32_t j = plo * 32 + lane; j < min(W, phi * 32); j += 32) { lastH[(size_t)t * W + j] = dps.Hp[j]; lastE[(size_t)t * W + j] = dps.Ep[j]; }
        if (lane == 0) {
            XdNode z; z.lineage_max = run_max; z.first_col = first_col; z.computed = 1; z.live = plo < phi ? 1 : 0;
            z.band_lo = (uint8_t)min(plo, 255u); z.band_hi = (uint8_t)(plo < phi ? phi : min(plo, 255u));
            ns[t] = z;
        }
        __syncwarp();
    }
    XdBest r; r.best = lane_best; r.t = lane_t; r.c = lane_c; r.j = lane_j;
#pragma unroll
    for (int ofs = 16; ofs > 0; ofs >>= 1) {
        const int32_t ob = __shfl_xor_sync(FULL, r.best, ofs);
        const uint32_t ot = __shfl_xor_sync(FULL, r.t, ofs), oc = __shfl_xor_sync(FULL, r.c, ofs), oj = __shfl_xor_sync(FULL, r.j, ofs);
        const bool take = ob > r.best || (ob == r.best && (ot < r.t || (ot == r.t && (oc < r.c || (oc == r.c && oj < r.j)))));
        if (take) { r.best = ob; r.t = ot; r.c = oc; r.j = oj; }
    }
    return r;
}

// Local scan of a short query (bonus at its right end only): best end cell; columns in shared memory,
// last columns per node in the workspace (oracle/xdrop_dag.cpp scan_local).
__device__ inline XdBest xd_scan(const DevIndex& ix, const DevScores& sc, const DagView& v,
                                 const uint8_t* q, uint32_t m, DpSmem dps) {
    const int lane = lane_id();
    const uint32_t W = m + 1;         // m <= 15: a single chunk
    const int32_t go = sc.gap_open, ge = sc.gap_extend, bonus = sc.full_length_bonus;
    int32_t* lastH = v.lastH; int32_t* lastE = v.lastE;
    const uint32_t N = v.N;
    int32_t lane_best = 0; uint32_t lane_t = 0, lane_c = 0, lane_j = 0;
    const uint32_t j = lane; const bool in = j < W;
    for (uint32_t u = 0; u < N; u++) {
        const uint32_t len = v.seq_len[u], soff = v.seq_off[u];
        int32_t ph = DP_NEG, pe = DP_NEG;
        const uint64_t e0 = v.pred_off[u]; const uint32_t ne = (uint32_t)(v.pred_off[u + 1] - e0);
        if (in) for (uint32_t pi = 0; pi < ne; pi++) { const uint32_t pu = v.pred[e0 + pi]; ph = max(ph, lastH[(size_t)pu * W + j]); pe = max(pe, lastE[(size_t)pu * W + j]); }
        for (uint32_t c = 0; c < len; c++) {
            const uint8_t r = __ldg(ix.seq + soff + c);
            const int32_t phm1 = __shfl_up_sync(FULL, ph, 1);
            int32_t d = DP_NEG, e = DP_NEG;
            if (in && j > 0) {
                const uint8_t qc = q[j - 1];
                const int32_t sub = (!is_acgt(r) || !is_acgt(qc)) ? 0 : (qc == r ? sc.match : -sc.mismatch);
                d = max(phm1, 0) + sub;
                if (ph > 0) e = ph - go;
                if (pe > DP_NEG) e = max(e, pe - ge);
                if (e <= 0) e = DP_NEG;
            }
            const int32_t hprime = max(d, e);
            int32_t incl = (in && j > 0 && hprime > 0) ? hprime + (int32_t)j * ge : INT_MIN;
#pragma unroll
            for (int ofs = 1; ofs < 32; ofs <<= 1) { const int32_t tt = __shfl_up_sync(FULL, incl, ofs); if (lane >= ofs) incl = max(incl, tt); }
            int32_t excl = __shfl_up_sync(FULL, incl, 1);
            if (lane == 0) excl = INT_MIN;
            int32_t f = DP_NEG;
            if (in && j > 0 && excl > INT_MIN) f = excl - go - (int32_t)(j - 1) * ge;
            if (f <= 0) f = DP_NEG;
            int32_t h = 0;
            if (in && j > 0) h = max(max(d, 0), max(e, f));
            if (in && j > 0) {
                int32_t cand = h;
                if (j == m && d + bonus >= h) cand = d + bonus;
                if (cand > lane_best) { lane_best = cand; lane_t = u; lane_c = c; lane_j = j; }
            }
            ph = in ? h : DP_NEG; pe = e;
        }
        if (in) { lastH[(size_t)u * W + j] = ph; lastE[(size_t)u * W + j] = pe; }
        __syncwarp();
    }
    XdBest r; r.best = lane_best; r.t = lane_t; r.c = lane_c; r.j = lane_j;
#pragma unroll
    for (int ofs = 16; ofs > 0; ofs >>= 1) {
        const int32_t ob = __shfl_xor_sync(FULL, r.best, ofs);
        const uint32_t ot = __shfl_xor_sync(FULL, r.t, ofs), oc = __shfl_xor_sync(FULL, r.c, ofs), oj = __shfl_xor_sync(FULL, r.j, ofs);
        const bool take = ob > r.best || (ob == r.best && (ot < r.t || (ot == r.t && (oc < r.c || (oc == r.c && oj < r.j)))));
        if (take) { r.best = ob; r.t = ot; r.c = oc; r.j = oj; }
    }
    (void)dps;
    return r;
}

// Two-pass seeded X-drop alignment of query[0..m) against the DAG view (oracle/xdrop_dag.cpp align_xdrop_dag).
// q: shared query buffer of the warp (>= m bytes).  seed_u == 0xffffffff: seedless scan.
__device__ inline void xd_align(const DevIndex& ix, const DevScores& sc, const DagView& v, const uint8_t* query, uint32_t m,
                                uint32_t seed_u, uint32_t seed_o, uint32_t seed_q, uint32_t max_gap_in,
                                uint8_t* q, DpSmem dps, int32_t& score_out, PathBuf& out, uint32_t& status) {
    const int lane = lane_id();
    const uint32_t N = v.N;
    score_out = 0; pb_reset(out);
    if (N == 0 || m == 0) return;
    const uint32_t max_gap = max(max_gap_in, 1u);
    if (lane == 0) {
        uint32_t cols = 0;
        for (uint32_t u = 0; u < N; u++) {
            const gb_node_rec nr = load_node(ix, v.node[u]);
            v.seq_off[u] = nr.seq_off; v.seq_len[u] = nr.len; v.col_start[u] = cols;
            cols += nr.len;
        }
    }
    __syncwarp();
    // ---- pass 1: the head ---------------------------------------------------------------------------
    uint32_t head_u, head_off, head_q;
    if (seed_u != 0xffffffffu) {
        const uint32_t m1 = m - seed_q;
        for (uint32_t i = lane; i < m1; i += 32) q[i] = dp_query_base(query[seed_q + i]);
        __syncwarp();
        const XdBest r = xd_pass<false, false>(ix, sc, v, q, m1, seed_u, seed_o, max_gap, dps);
        if (r.best > 0) { head_u = r.t; head_off = r.c + 1; head_q = seed_q + r.j; }
        else { head_u = seed_u; head_off = seed_o; head_q = seed_q; }
    } else {
        const uint32_t scan_len = min(m, 15u);
        for (uint32_t i = lane; i < scan_len; i += 32) q[i] = query[m - scan_len + i];
        __syncwarp();
        const XdBest r = xd_scan(ix, sc, v, q, scan_len, dps);
        if (r.best <= 0) return;
        head_u = r.t; head_off = r.c + 1; head_q = (m - scan_len) + r.j;
    }
    __syncwarp();
    if (head_q == 0) return;
    // ---- pass 2: leftwards from the head (mirrored problem) -------------------------------------------
    const uint32_t m2 = head_q;
    for (uint32_t i = lane; i < m2; i += 32) q[i] = dp_query_base(query[head_q - 1 - i]);
    __syncwarp();
    const uint32_t rs = N - 1 - head_u, ro = v.seq_len[head_u] - head_off;
    const XdBest r2 = xd_pass<true, true>(ix, sc, v, q, m2, rs, ro, max_gap, dps);
    if (r2.best <= 0) return;
    score_out = r2.best;

    // ---- traceback in mirrored space: recorded end -> start = forward alignment start -> head ------------
    const uint32_t W = m2 + 1;
    const uint8_t* argH = v.argH; const uint8_t* argE = v.argE;
    const uint8_t* tb = v.tb;
    const XdNode* ns = v.nstate;
    uint32_t* steps = v.steps;
    uint32_t n_steps = 0;
    {
        uint32_t t = r2.t, c = r2.c, j = r2.j;
        int state = 0; bool at_virtual = false;
        while (true) {
            if (at_virtual) { for (; j > 0; j--) { if (lane == 0) steps[n_steps] = (rs << 8) | 2u; n_steps++; } break; }
            const uint32_t u = N - 1 - t;
            const uint8_t tbv = tb[(size_t)(v.col_start[u] + c) * W + j];
            const bool first = c == ns[t].first_col;
            // previous column for query offset jj, through E or not
            auto go_prev = [&](uint32_t jj, bool via_E) {
                if (!first) { c--; return; }
                if (t == rs) { at_virtual = true; return; }
                uint32_t tt = t;
                while (true) {
                    const uint32_t uu = N - 1 - tt;
                    const uint32_t pi = via_E ? argE[(size_t)tt * W + jj] : argH[(size_t)tt * W + jj];
                    const uint32_t pu = v.succ[v.succ_off[uu] + pi];
                    const uint32_t pt = N - 1 - pu;
                    if (v.seq_len[pu] > ns[pt].first_col) { t = pt; c = v.seq_len[pu] - 1; return; }
                    if (pt == rs) { t = rs; at_virtual = true; return; }
                    tt = pt;
                }
            };
            if (state == 0) {
                const uint32_t src = tbv & 3u;
                if (src == 0) {
                    const uint8_t qc = q[j - 1], r = __ldg(ix.seq + v.seq_off[u] + (v.seq_len[u] - 1 - c));
                    if (lane == 0) steps[n_steps] = (t << 8) | (qc == r ? 0u : 1u);
                    n_steps++;
                    j--; go_prev(j, false);
                    if (at_virtual && j == 0) break;
                    continue;
                }
                state = src == 1 ? 1 : 2;
                continue;
            }
            if (state == 1) {
                if (lane == 0) steps[n_steps] = (t << 8) | 3u;
                n_steps++;
                const bool open = (tbv & 4u) != 0;
                go_prev(j, !open);
                state = open ? 0 : 1;
                if (at_virtual && j == 0 && state == 0) break;
                continue;
            }
            if (lane == 0) steps[n_steps] = (t << 8) | 2u;
            n_steps++;
            const bool open = (tbv & 8u) != 0;
            j--;
            state = open ? 0 : 2;
        }
    }
    __syncwarp();

    // ---- steps -> mappings in forward order -------------------------------------------------------------
    if (lane == 0) {
        uint32_t aligned_q = 0;
        for (uint32_t i = 0; i < n_steps; i++) aligned_q += (steps[i] & 0xffu) != 3u ? 1u : 0u;
        uint32_t qpos = head_q - aligned_q;
        const uint8_t* qf = query;                  // forward query (raw bytes) for substitution bases
        uint32_t i = 0;
        while (i < n_steps) {
            const uint32_t t = steps[i] >> 8, u = N - 1 - t;
            uint32_t k = i, cols = 0;
            while (k < n_steps && (steps[k] >> 8) == t) { if ((steps[k] & 0xffu) != 2u) cols++; k++; }
            const uint32_t end = (u == head_u) ? head_off : v.seq_len[u];
            pb_add_mapping(out, u, end - cols);
            if (i == 0 && qpos > 0) pb_add_edit(out, edit_word(GB_EDIT_INS, qpos, 0));
            uint32_t cur = 0xff, run = 0;
            auto flush = [&]() {
                if (cur == 1) { for (uint32_t x = 0; x < run; x++) { pb_add_edit(out, edit_word(GB_EDIT_SUB, 1, base2(qf[qpos]))); qpos++; } }
                else if (run > 0) {
                    if (cur == 0) { pb_add_edit(out, edit_word(GB_EDIT_MATCH, run, 0)); qpos += run; }
                    else if (cur == 2) {
                        // an insertion next to an insertion edit of this mapping (the leading soft clip) extends it
                        if (!out.overflow && out.maps[out.n_maps - 1].n_edits > 0 && (out.edits[out.n_edits - 1] & 3u) == GB_EDIT_INS) out.edits[out.n_edits - 1] += run << 4;
                        else pb_add_edit(out, edit_word(GB_EDIT_INS, run, 0));
                        qpos += run;
                    }
                    else pb_add_edit(out, edit_word(GB_EDIT_DEL, run, 0));
                }
            };
            for (uint32_t x = i; x < k; x++) {
                const uint32_t op = steps[x] & 0xffu;
                if (op == cur) run++; else { if (cur != 0xff) flush(); cur = op; run = 1; }
            }
            if (cur != 0xff) flush();
            i = k;
        }
        if (out.n_maps > 0 && head_q < m && !out.overflow) {
            if (out.maps[out.n_maps - 1].n_edits > 0 && (out.edits[out.n_edits - 1] & 3u) == GB_EDIT_INS) out.edits[out.n_edits - 1] += (m - head_q) << 4;
            else pb_add_edit(out, edit_word(GB_EDIT_INS, m - head_q, 0));
        }
    }
    __syncwarp();
    out.n_maps = __shfl_sync(FULL, out.n_maps, 0); out.n_edits = __shfl_sync(FULL, out.n_edits, 0);
    out.overflow = __shfl_sync(FULL, (int)out.overflow, 0) != 0;
    if (out.overflow) status = GB_ITEM_OUT_FULL;
}

// tb byte: bits 0-1 source of H (0 diagonal, 1 deletion, 2 insertion, 3 none: H == 0),
//          bit 2 deletion opened here, bit 3 insertion opened here, bit 4 the diagonal starts the alignment
__device__ inline void sw_align(const DevIndex& ix, const DevScores& sc, const DagView& v, const uint8_t* query, uint32_t m,
                                uint8_t* q, DpSmem dps, int32_t& score_out, PathBuf& out, uint32_t& status) {
    const int lane = lane_id();
    const uint32_t N = v.N;
    const uint32_t W = m + 1;
    const int32_t go = sc.gap_open, ge = sc.gap_extend, bonus = sc.full_length_bonus;
    score_out = 0; pb_reset(out);
    if (N == 0 || m == 0) return;
    for (uint32_t i = lane; i < m; i += 32) q[i] = query[i];
    // node table: sequence and first traceback column
    if (lane == 0) {
        uint32_t cols = 0;
        for (uint32_t u = 0; u < N; u++) {
            const gb_node_rec nr = load_node(ix, v.node[u]);
            v.seq_off[u] = nr.seq_off; v.seq_len[u] = nr.len; v.col_start[u] = cols;
            cols += nr.len;
        }
    }
    __syncwarp();
    int32_t* lastH = v.lastH; int32_t* lastE = v.lastE;
    uint8_t* argH = v.argH; uint8_t* argE = v.argE;
    uint8_t* tb = v.tb;

    // this lane's best end cell: (candidate score, node, column, query offset, attached right end)
    int32_t lane_best = 0; uint32_t lane_u = 0, lane_c = 0, lane_j = 0; bool lane_end = false;
    for (uint32_t u = 0; u < N; u++) {
        const uint32_t len = v.seq_len[u], soff = v.seq_off[u];
        // merged incoming column
        const uint64_t pb0 = v.pred_off[u]; const uint32_t np = (uint32_t)(v.pred_off[u + 1] - pb0);
        for (uint32_t j = lane; j < W; j += 32) {
            int32_t h = DP_NEG, e = DP_NEG; uint32_t ah = 0xff, ae = 0xff;
            for (uint32_t pi = 0; pi < np; pi++) {
                const uint32_t pu = v.pred[pb0 + pi];
                const int32_t ph = lastH[(size_t)pu * W + j], pe = lastE[(size_t)pu * W + j];
                if (ph > h) { h = ph; ah = pi; }
                if (pe > e) { e = pe; ae = pi; }
            }
            dps.Hp[j] = h; dps.Ep[j] = e; argH[(size_t)u * W + j] = (uint8_t)ah; argE[(size_t)u * W + j] = (uint8_t)ae;
        }
        __syncwarp();
        for (uint32_t c = 0; c < len; c++) {
            const uint8_t r = __ldg(ix.seq + soff + c);
            const bool r_ok = is_acgt(r);
            uint8_t* tbcol = tb + (size_t)(v.col_start[u] + c) * W;
            int32_t carry = INT_MIN, prevH_last = DP_NEG, prev_ph_last = DP_NEG;
            for (uint32_t jb = 0; jb < W; jb += 32) {
                const uint32_t j = jb + lane;
                const bool in = j < W;
                int32_t ph = DP_NEG, pe = DP_NEG;
                if (in) { ph = dps.Hp[j]; pe = dps.Ep[j]; }
                int32_t phm1 = __shfl_up_sync(FULL, ph, 1);
                if (lane == 0) phm1 = prev_ph_last;
                prev_ph_last = __shfl_sync(FULL, ph, 31);
                int32_t d = DP_NEG, e = DP_NEG;
                bool fresh = false;
                if (in && j > 0) {
                    const uint8_t qc = q[j - 1];
                    const int32_t s = (!r_ok || !is_acgt(qc)) ? 0 : (qc == r ? sc.match : -sc.mismatch);
                    fresh = j == 1 || !(phm1 > 0);
                    d = (j == 1 ? bonus : max(phm1, 0)) + s;
                    if (ph > 0) e = ph - go;
                    if (pe > DP_NEG) e = max(e, pe - ge);
                    if (e <= 0) e = DP_NEG;
                }
                const int32_t hprime = max(d, e);
                // insertion chain over the cells worth keeping (H' > 0)
                int32_t g = (in && j > 0 && hprime > 0) ? hprime + (int32_t)j * ge : INT_MIN;
                int32_t incl = g;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int32_t t = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl = max(incl, t); }
                int32_t excl = __shfl_up_sync(FULL, incl, 1);
                if (lane == 0) excl = INT_MIN;
                excl = max(excl, carry);
                carry = max(carry, __shfl_sync(FULL, incl, 31));
                int32_t f = DP_NEG;
                if (in && j > 0 && excl > INT_MIN) f = excl - go - (int32_t)(j - 1) * ge;
                if (f <= 0) f = DP_NEG;
                int32_t h = 0;
                if (in && j > 0) h = max(max(d, 0), max(e, f));
                int32_t hm1 = __shfl_up_sync(FULL, h, 1);
                if (lane == 0) hm1 = prevH_last;
                prevH_last = __shfl_sync(FULL, h, 31);
                if (in) {
                    uint8_t tbv;
                    if (h <= 0) tbv = 3; else if (d == h) tbv = 0; else if (e == h) tbv = 1; else tbv = 2;
                    if (ph > 0 && e == ph - go) tbv |= 4;
                    if (j > 0 && hm1 > 0 && f == hm1 - go) tbv |= 8;
                    if (fresh) tbv |= 16;
                    dps.Hc[j] = h; dps.Ec[j] = e; tbcol[j] = tbv;
                    if (j > 0) {
                        int32_t cand = h; bool end_diag = false;
                        if (j == m && d + bonus >= h) { cand = d + bonus; end_diag = true; }
                        if (cand > lane_best) { lane_best = cand; lane_u = u; lane_c = c; lane_j = j; lane_end = end_diag; }
                    }
                }
            }
            __syncwarp();
            int32_t* t1p = dps.Hp; dps.Hp = dps.Hc; dps.Hc = t1p;
            int32_t* t2p = dps.Ep; dps.Ep = dps.Ec; dps.Ec = t2p;
        }
        for (uint32_t j = lane; j < W; j += 32) { lastH[(size_t)u * W + j] = dps.Hp[j]; lastE[(size_t)u * W + j] = dps.Ep[j]; }
        __syncwarp();
    }
    // first maximum in (node, column, query offset) order
    int32_t best = lane_best; uint32_t bu = lane_u, bc = lane_c, bj = lane_j; uint32_t bend = lane_end ? 1u : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const int32_t ob = __shfl_xor_sync(FULL, best, o);
        const uint32_t ou = __shfl_xor_sync(FULL, bu, o), oc = __shfl_xor_sync(FULL, bc, o), oj = __shfl_xor_sync(FULL, bj, o), oe = __shfl_xor_sync(FULL, bend, o);
        const bool take = ob > best || (ob == best && (ou < bu || (ou == bu && (oc < bc || (oc == bc && oj < bj)))));
        if (take) { best = ob; bu = ou; bc = oc; bj = oj; bend = oe; }
    }
    if (best <= 0) return;
    score_out = best;

    // ---- traceback (uniform): steps end -> start as (node << 8) | op, op 0 match, 1 mismatch, 2 insertion, 3 deletion
    uint32_t* steps = v.steps;
    uint32_t n_steps = 0, start_j = 0;
    {
        uint32_t u = bu, c = bc, j = bj;
        int state = bend ? 3 : 0;
        while (true) {
            const uint8_t tbv = tb[(size_t)(v.col_start[u] + c) * W + j];
            if (state == 0) {
                const uint32_t src = tbv & 3u;
                if (src == 3) { start_j = j; break; }
                state = src == 0 ? 3 : (src == 1 ? 1 : 2);
                continue;
            }
            if (state == 3) {
                const uint8_t qc = q[j - 1], r = __ldg(ix.seq + v.seq_off[u] + c);
                if (lane == 0) steps[n_steps] = (u << 8) | (qc == r ? 0u : 1u);
                n_steps++;
                j--;
                if (tbv & 16u) { start_j = j; break; }
                if (c > 0) c--; else { u = v.pred[v.pred_off[u] + argH[(size_t)u * W + j]]; c = v.seq_len[u] - 1; }
                state = 0;
                continue;
            }
            if (state == 1) {
                if (lane == 0) steps[n_steps] = (u << 8) | 3u;
                n_steps++;
                const bool open = (tbv & 4u) != 0;
                if (c > 0) c--; else { u = v.pred[v.pred_off[u] + (open ? argH[(size_t)u * W + j] : argE[(size_t)u * W + j])]; c = v.seq_len[u] - 1; }
                state = open ? 0 : 1;
                continue;
            }
            if (lane == 0) steps[n_steps] = (u << 8) | 2u;
            n_steps++;
            const bool open = (tbv & 8u) != 0;
            j--;
            state = open ? 0 : 2;
        }
    }
    __syncwarp();

    // ---- steps -> mappings; soft clips as insertion edits on the first / last mapping (aligner.cpp:150-241)
    if (lane == 0) {
        uint32_t query_offset = start_j;
        int64_t si = (int64_t)n_steps - 1;
        bool first = true;
        while (si >= 0) {
            const uint32_t nd = steps[si] >> 8;
            // columns this mapping consumes, to place its offset
            uint32_t cols = 0; int64_t k = si;
            while (k >= 0 && (steps[k] >> 8) == nd) { if ((steps[k] & 0xffu) != 2u) cols++; k--; }
            const uint32_t end_col = k < 0 ? bc + 1 : v.seq_len[nd];
            pb_add_mapping(out, nd, end_col - cols);
            if (first && start_j > 0) pb_add_edit(out, edit_word(GB_EDIT_INS, start_j, 0));
            first = false;
            uint32_t cur = 0xff, run = 0;
            auto flush = [&]() {
                if (cur == 1) { for (uint32_t x = 0; x < run; x++) { pb_add_edit(out, edit_word(GB_EDIT_SUB, 1, base2(q[query_offset]))); query_offset++; } }
                else if (run > 0) {
                    if (cur == 0) { pb_add_edit(out, edit_word(GB_EDIT_MATCH, run, 0)); query_offset += run; }
                    else if (cur == 2) { pb_add_edit(out, edit_word(GB_EDIT_INS, run, 0)); query_offset += run; }
                    else if (cur == 3) { pb_add_edit(out, edit_word(GB_EDIT_DEL, run, 0)); }
                }
            };
            while (si > k) {
                const uint32_t op = steps[si] & 0xffu;
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
    if (out.overflow) status = GB_ITEM_OUT_FULL;
}


} // namespace gb
