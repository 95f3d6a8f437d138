// banded_global.cuh — Aligner::align_global_banded (aligner.cpp:699-761, banded_global_aligner.cpp): global
// alignment of a read against a DAG from a source to a sink, inside vg's per-node diagonal band, regular
// scoring.  The rules (band, recurrences, boundary moves, ties, the empty read) are stated in
// oracle/banded_global.cpp and followed here cell for cell.
//
// One warp per problem.  Lane 0 sets up the node table and the bands (an O(nodes + edges) pass); each
// DP column is then swept over its band rows only, 32 rows per step (lane = row), the insertion chain
// by a max-plus prefix scan over shuffles.  The two live columns and the merged predecessor column sit
// in shared memory; every node's last column, the predecessor choices of first columns and the
// traceback bytes go to a per-problem workspace the host sizes: one traceback byte per (base, query
// prefix) pair, of which only the band rows are written.  Lane 0 traces back and writes the path.
// Scores are int32 throughout.
#pragma once
#include "align.cuh"

namespace gb {

struct BgNode { int32_t top, bot; uint32_t len, seq_off, col_start; uint8_t source, sink, masked; };

struct BgView {
    uint32_t N; const uint32_t* node;
    const uint32_t* pred; const uint64_t* pred_off;          // pred_off indexed by the node's position in the problem
    BgNode* nd; int64_t* sts; int64_t* lts;                  // [N]
    int32_t* lastM; int32_t* lastI; int32_t* lastD;          // [N * (m + 1)]
    uint8_t* argd; uint8_t* argh;                            // [N * (m + 1)]
    uint8_t* tb;                                             // [bases * (m + 1)]
    uint32_t* steps;                                         // [bases + m + 2]
};

// per-warp shared memory: 8 int32 rows and 2 byte rows of m + 1 entries
struct BgSmem { int32_t *pM, *pI, *pD, *cM, *cI, *cD, *xd, *xh; uint8_t *sd, *sh; };

__device__ __forceinline__ bool bg_alive(int32_t x) { return x > DP_NEG / 2; }
__device__ __forceinline__ int32_t bg_sub(int32_t x, int32_t y) { return bg_alive(x) ? x - y : DP_NEG; }
__device__ __forceinline__ uint32_t bg_best3(int32_t a, int32_t b, int32_t c, int32_t& v) {
    v = a; uint32_t s = 0;
    if (b > v) { v = b; s = 1; }
    if (c > v) { v = c; s = 2; }
    if (!bg_alive(v)) v = DP_NEG;
    return s;
}
__device__ __forceinline__ int64_t bg_row_lo(const BgNode& n, int64_t c) { return (c == 0 && n.source) ? 0 : max((int64_t)0, (int64_t)n.top + c + 1); }
__device__ __forceinline__ int64_t bg_row_hi(const BgNode& n, int64_t c, int64_t m) { return min(m, (int64_t)n.bot + c + 1); }

// status: GB_ITEM_OK, GB_ITEM_NO_BAND (no global alignment inside the band) or GB_ITEM_OUT_FULL
__device__ inline void bg_align(const DevIndex& ix, const DevScores& sc, const BgView& v, const uint8_t* query, uint32_t m,
                                int32_t pad, bool permissive, uint8_t* q, BgSmem s, int32_t& score_out, PathBuf& out, uint32_t& status) {
    const int lane = lane_id();
    const uint32_t N = v.N, W = m + 1;
    const int32_t go = sc.gap_open, ge = sc.gap_extend;
    const int64_t M64 = m;
    score_out = 0; pb_reset(out);
    if (N == 0) { status = GB_ITEM_NO_BAND; return; }
    for (uint32_t i = lane; i < m; i += 32) q[i] = query[i];
    // ---- node table and bands (find_banded_paths) -------------------------------------------------------
    if (lane == 0) {
        uint32_t cols = 0;
        for (uint32_t u = 0; u < N; u++) {
            const gb_node_rec nr = load_node(ix, v.node[u]);
            BgNode z; z.len = nr.len; z.seq_off = nr.seq_off; z.col_start = cols; z.top = 0; z.bot = 0;
            z.source = v.pred_off[u + 1] == v.pred_off[u]; z.sink = 1; z.masked = 0;
            v.nd[u] = z; cols += nr.len;
            for (uint64_t e = v.pred_off[u]; e < v.pred_off[u + 1]; e++) v.nd[v.pred[e]].sink = 0;
        }
        for (uint32_t u = 0; u < N; u++) { v.sts[u] = v.nd[u].sink ? 0 : INT64_MAX; v.lts[u] = 0; }
        for (uint32_t i = N; i-- > 0;) {
            const int64_t L = v.nd[i].len;
            for (uint64_t e = v.pred_off[i]; e < v.pred_off[i + 1]; e++) {
                const uint32_t p = v.pred[e];
                v.lts[p] = max(v.lts[p], v.lts[i] + L);
                if (v.sts[i] != INT64_MAX) v.sts[p] = min(v.sts[p], v.sts[i] + L);
            }
        }
        if (m > 0) {
            for (uint32_t u = 0; u < N; u++) {
                BgNode n = v.nd[u];
                const int64_t L = n.len;
                int64_t top = INT64_MAX, bot = INT64_MIN;
                if (n.source) {
                    if (permissive) { top = min((int64_t)-pad, M64 - (L + v.lts[u]) - pad); bot = max((int64_t)pad, M64 - (L + v.sts[u]) + pad); }
                    else { top = -pad; bot = pad; }
                } else {
                    for (uint64_t e = v.pred_off[u]; e < v.pred_off[u + 1]; e++) {
                        const BgNode& p = v.nd[v.pred[e]];
                        if (p.masked) continue;
                        top = min(top, (int64_t)p.top + p.len); bot = max(bot, (int64_t)p.bot + p.len);
                    }
                }
                n.masked = (top > bot || top + L + v.sts[u] > M64 || bot + L + v.lts[u] < M64) ? 1 : 0;
                if (!n.masked) { n.top = (int32_t)top; n.bot = (int32_t)bot; }
                v.nd[u] = n;
            }
        }
    }
    __syncwarp();
    if (m == 0) {
        // the empty read: delete the shortest source-to-sink path (sts reused as distance, steps as the back link)
        if (lane == 0) {
            int64_t best = INT64_MAX; uint32_t bu = 0;
            for (uint32_t u = 0; u < N; u++) {
                int64_t d = 0; uint32_t from = 0xffffffffu;
                if (!v.nd[u].source) {
                    d = INT64_MAX;
                    for (uint64_t e = v.pred_off[u]; e < v.pred_off[u + 1]; e++) if (v.sts[v.pred[e]] < d) { d = v.sts[v.pred[e]]; from = v.pred[e]; }
                }
                v.sts[u] = d + v.nd[u].len; v.steps[u] = from;
            }
            for (uint32_t u = 0; u < N; u++) if (v.nd[u].sink && v.sts[u] < best) { best = v.sts[u]; bu = u; }
            uint32_t n_walk = 0;
            for (uint32_t u = bu; u != 0xffffffffu; u = v.steps[u]) v.lts[n_walk++] = u;
            for (uint32_t i = n_walk; i-- > 0;) { const uint32_t u = (uint32_t)v.lts[i]; pb_add_mapping(out, u, 0); pb_add_edit(out, edit_word(GB_EDIT_DEL, v.nd[u].len, 0)); }
            score_out = -(go + (int32_t)(best - 1) * ge);
        }
        __syncwarp();
        score_out = __shfl_sync(FULL, score_out, 0);
        out.n_maps = __shfl_sync(FULL, out.n_maps, 0); out.n_edits = __shfl_sync(FULL, out.n_edits, 0);
        out.overflow = __shfl_sync(FULL, (int)out.overflow, 0) != 0;
        if (out.overflow) status = GB_ITEM_OUT_FULL;
        return;
    }
    // ---- fill -------------------------------------------------------------------------------------------
    for (uint32_t u = 0; u < N; u++) {
        const BgNode n = v.nd[u];
        if (n.masked) continue;
        const int64_t L = n.len;
        const int64_t lo0 = bg_row_lo(n, 0), hi0 = bg_row_hi(n, 0, M64);
        // merged incoming column: diagonal source at row j (for M at j + 1), horizontal source at row j (for D at j)
        for (int64_t j = max((int64_t)0, lo0 - 1) + lane; j <= hi0; j += 32) {
            int32_t xd = DP_NEG, xh = DP_NEG; uint32_t sd = 0, sh = 0, ad = 0, ah = 0;
            if (n.source) {
                const int32_t iv = j == 0 ? DP_NEG : -(go + (int32_t)(j - 1) * ge);
                if (j == 0) { xd = 0; sd = 0; xh = -go; sh = 0; }
                else { xd = iv; sd = 1; if (j < min((int64_t)n.bot + 1, M64)) { xh = iv - go; sh = 1; } }
            } else {
                const uint64_t e0 = v.pred_off[u]; const uint32_t np = (uint32_t)(v.pred_off[u + 1] - e0);
                for (uint32_t pi = 0; pi < np; pi++) {
                    const uint32_t p = v.pred[e0 + pi];
                    const BgNode pn = v.nd[p];
                    if (pn.masked) continue;
                    const int64_t snt = (int64_t)pn.top + pn.len;
                    if (j < max((int64_t)0, snt) || j > bg_row_hi(pn, (int64_t)pn.len - 1, M64)) continue;
                    const size_t k = (size_t)p * W + j;
                    const int32_t pm = v.lastM[k], pI = v.lastI[k], pd = v.lastD[k];
                    int32_t val; uint32_t st = bg_best3(pm, pI, pd, val);
                    if (val > xd) { xd = val; sd = st; ad = pi; }
                    if (j - 1 >= snt) {
                        st = bg_best3(bg_sub(pm, go), bg_sub(pI, go), bg_sub(pd, ge), val);
                        if (val > xh) { xh = val; sh = st; ah = pi; }
                    }
                }
            }
            s.xd[j] = xd; s.xh[j] = xh; s.sd[j] = (uint8_t)sd; s.sh[j] = (uint8_t)sh;
            v.argd[(size_t)u * W + j] = (uint8_t)ad; v.argh[(size_t)u * W + j] = (uint8_t)ah;
        }
        __syncwarp();
        int64_t plo = 0, phi = -1;
        for (int64_t c = 0; c < L; c++) {
            const uint8_t r = __ldg(ix.seq + n.seq_off + c);
            const bool r_ok = is_acgt(r);
            const int64_t lo = bg_row_lo(n, c), hi = bg_row_hi(n, c, M64);
            uint8_t* tbcol = v.tb + (size_t)(n.col_start + c) * W;
            int32_t carry = INT_MIN, prevM = DP_NEG, prevI = DP_NEG, prevD = DP_NEG;
            for (int64_t jb = lo; jb <= hi; jb += 32) {
                const int64_t j = jb + lane;
                const bool in = j <= hi;
                int32_t mv = DP_NEG, dv = DP_NEG; uint32_t ms = 0, ds = 0;
                if (in) {
                    if (j >= 1) {
                        int32_t src = DP_NEG;
                        if (c == 0) { src = s.xd[j - 1]; ms = s.sd[j - 1]; }
                        else if (j - 1 >= plo && j - 1 <= phi) ms = bg_best3(s.pM[j - 1], s.pI[j - 1], s.pD[j - 1], src);
                        if (bg_alive(src)) { const uint8_t qc = q[j - 1]; mv = src + ((r_ok && is_acgt(qc)) ? (qc == r ? sc.match : -sc.mismatch) : 0); }
                    }
                    if (c == 0) { dv = s.xh[j]; ds = s.sh[j]; }
                    else if (j >= plo && j <= phi) ds = bg_best3(bg_sub(s.pM[j], go), bg_sub(s.pI[j], go), bg_sub(s.pD[j], ge), dv);
                }
                // insertion chain: I(j) = max over lo <= k < j of max(M, D)(k) - go - (j - 1 - k) * ge
                const int32_t md = max(mv, dv);
                int32_t incl = (in && bg_alive(md)) ? md + (int32_t)j * ge : INT_MIN;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int32_t t = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl = max(incl, t); }
                int32_t excl = __shfl_up_sync(FULL, incl, 1);
                if (lane == 0) excl = INT_MIN;
                excl = max(excl, carry);
                carry = max(carry, __shfl_sync(FULL, incl, 31));
                int32_t iv = DP_NEG;
                if (in && excl > INT_MIN) iv = excl - go - (int32_t)(j - 1) * ge;
                // the insertion's source state at j - 1 (M > I > D on ties)
                int32_t um = __shfl_up_sync(FULL, mv, 1), ui = __shfl_up_sync(FULL, iv, 1), ud = __shfl_up_sync(FULL, dv, 1);
                if (lane == 0) { um = prevM; ui = prevI; ud = prevD; }
                prevM = __shfl_sync(FULL, mv, 31); prevI = __shfl_sync(FULL, iv, 31); prevD = __shfl_sync(FULL, dv, 31);
                int32_t chk; const uint32_t is = bg_best3(bg_sub(um, go), bg_sub(ui, ge), bg_sub(ud, go), chk);
                if (in) {
                    s.cM[j] = mv; s.cI[j] = iv; s.cD[j] = dv;
                    tbcol[j] = (uint8_t)(ms | (ds << 2) | (is << 4));
                }
            }
            __syncwarp();
            int32_t* t;
            t = s.pM; s.pM = s.cM; s.cM = t;
            t = s.pI; s.pI = s.cI; s.cI = t;
            t = s.pD; s.pD = s.cD; s.cD = t;
            plo = lo; phi = hi;
        }
        for (int64_t j = plo + lane; j <= phi; j += 32) {
            const size_t k = (size_t)u * W + j;
            v.lastM[k] = s.pM[j]; v.lastI[k] = s.pI[j]; v.lastD[k] = s.pD[j];
        }
        __syncwarp();
    }
    // ---- end cell, traceback and path (lane 0) -------------------------------------------------------------
    if (lane == 0) {
        int32_t best = DP_NEG; int64_t bu = -1; uint32_t bst = 0;
        for (uint32_t u = 0; u < N; u++) {
            const BgNode n = v.nd[u];
            if (!n.sink || n.masked) continue;
            if (M64 < bg_row_lo(n, n.len - 1) || M64 > bg_row_hi(n, n.len - 1, M64)) continue;
            const size_t k = (size_t)u * W + m;
            int32_t val; const uint32_t st = bg_best3(v.lastM[k], v.lastI[k], v.lastD[k], val);
            if (bg_alive(val) && (bu < 0 || val > best)) { best = val; bu = u; bst = st; }
        }
        if (bu < 0) status = GB_ITEM_NO_BAND;
        else {
            score_out = best;
            // steps end -> start as (node << 8) | op, op 0 match, 1 mismatch, 2 insertion, 3 deletion
            uint32_t n_steps = 0;
            uint32_t u = (uint32_t)bu; int64_t c = v.nd[u].len - 1, j = m; uint32_t st = bst;
            while (true) {
                const BgNode n = v.nd[u];
                const uint8_t tb = v.tb[(size_t)(n.col_start + c) * W + j];
                if (st == 2) {
                    v.steps[n_steps++] = (u << 8) | 3u;
                    const uint32_t src = (tb >> 2) & 3u;
                    if (c > 0) { c--; st = src; continue; }
                    if (n.source) { for (int64_t x = 0; x < j; x++) v.steps[n_steps++] = (u << 8) | 2u; break; }
                    u = v.pred[v.pred_off[u] + v.argh[(size_t)u * W + j]]; c = v.nd[u].len - 1; st = src; continue;
                }
                if (st == 1) { v.steps[n_steps++] = (u << 8) | 2u; st = (tb >> 4) & 3u; j--; continue; }
                const uint8_t rb = __ldg(ix.seq + n.seq_off + c);
                v.steps[n_steps++] = (u << 8) | (q[j - 1] == rb ? 0u : 1u);
                const uint32_t src = tb & 3u;
                j--;
                if (c > 0) { c--; st = src; continue; }
                if (n.source) { for (int64_t x = 0; x < j; x++) v.steps[n_steps++] = (u << 8) | 2u; break; }
                u = v.pred[v.pred_off[u] + v.argd[(size_t)u * W + j]]; c = v.nd[u].len - 1; st = src;
            }
            // steps -> mappings (every mapping starts at offset 0)
            uint32_t qpos = 0, cur_node = 0xffffffu, last_op = 0xff;
            for (uint32_t x = n_steps; x-- > 0;) {
                const uint32_t nd = v.steps[x] >> 8, op = v.steps[x] & 0xffu;
                if (nd != cur_node) { pb_add_mapping(out, nd, 0); cur_node = nd; last_op = 0xff; }
                const bool extend = !out.overflow && last_op == op && op != 1u;
                if (extend) out.edits[out.n_edits - 1] += 1u << 4;
                else if (op == 0) pb_add_edit(out, edit_word(GB_EDIT_MATCH, 1, 0));
                else if (op == 1) pb_add_edit(out, edit_word(GB_EDIT_SUB, 1, base2(q[qpos])));
                else if (op == 2) pb_add_edit(out, edit_word(GB_EDIT_INS, 1, 0));
                else pb_add_edit(out, edit_word(GB_EDIT_DEL, 1, 0));
                if (op != 3) qpos++;
                last_op = op;
            }
        }
    }
    __syncwarp();
    score_out = __shfl_sync(FULL, score_out, 0);
    status = __shfl_sync(FULL, status, 0);
    out.n_maps = __shfl_sync(FULL, out.n_maps, 0); out.n_edits = __shfl_sync(FULL, out.n_edits, 0);
    out.overflow = __shfl_sync(FULL, (int)out.overflow, 0) != 0;
    if (out.overflow) status = GB_ITEM_OUT_FULL;
}

} // namespace gb
