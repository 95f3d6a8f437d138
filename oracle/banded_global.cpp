// ORACLE — TEST INFRASTRUCTURE ONLY.  Banded global alignment of a read against a DAG, from a source
// to a sink, with regular (not quality-adjusted) scoring:
//   Aligner::align_global_banded                                     aligner.cpp:699-761
//   BandedGlobalAligner::BandedGlobalAligner / find_banded_paths      banded_global_aligner.cpp:1961-2266
//   BandedGlobalAligner::path_lengths_to_sinks                        :2122-2169
//   BAMatrix::fill_matrix                                             :251-742
//   deletion aligner for the empty read                               aligner.cpp:703-706
// The chaining route reaches it as the DP fallback for chain middles (find_chain_alignment,
// minimizer_mapper_from_chains.cpp:2532-3332).
//
// Graph: nodes in topological order with per-node predecessor lists (indices into the problem), every
// node non-empty.  Sources have no predecessor, sinks no successor inside the problem.
//
// Band (find_banded_paths): node u gets diagonals [top_u, bot_u], a diagonal being (read index) -
// (node column).  Sources start at [-pad, pad], or with permissive banding at
// [min(-pad, m - len - longest_to_sink - pad), max(pad, m - len - shortest_to_sink + pad)]; a node is
// masked when its extended band cannot reach the read end along its shortest / longest path to a
// sink; unmasked nodes push [top + len, bot + len] into their successors (min / max).
//
// DP: cell (u, c, j) = node u, column c, query prefix j (0 <= j <= m, read index j - 1; row j = 0 is
// vg's implied "top edge" above the read).  A cell exists when its diagonal j - 1 - c lies in u's band.
// Three states: M (q[j-1] against base c), I (q[j-1] inserted), D (base c deleted).  A gap of length n
// costs gap_open + (n - 1) * gap_extend, a gap next to a gap of the other kind opens anew; a pair with
// a non-ACGT base scores 0, otherwise match / -mismatch (no full-length bonus: the alignment is global).
//   M(c, j) = s + best(M, I, D)(c - 1, j - 1)
//   D(c, j) = best(M - go, I - go, D - ge)(c - 1, j)
//   I(c, j) = best(M - go, I - ge, D - go)(c, j - 1)
// Column c - 1 of column 0 is, for a non-source node, the last column of each unmasked predecessor p;
// a move from p may only land on a diagonal of p's extended band [top_p + len_p, bot_p + len_p]
// (fill_matrix :403-543), which forbids the deletion move out of p's top band cell.  For a source it
// is the virtual column of lead insertions: row 0 the start (value 0), row j >= 1 an insertion of j
// bases; a deletion move from it is not taken into the last row of column 0 (:604-605), and the
// source's top-edge cell (0, 0) always exists with -gap_open (:577-579).
// The alignment ends at (last column, m) of a sink.
//
// Where the reference's vectors leave a choice open, this file DEFINES (the GPU kernel follows it):
//   * ties between states prefer M, then I, then D, everywhere (end cell, each recurrence);
//   * the merged predecessor column takes the first predecessor in list order on equal values;
//   * the end is the first sink in topological order with the maximal score;
//   * lead deletions follow top-edge cells (row 0) through the band like any other deletion; vg
//     instead prices them by the shortest source path regardless of band and masking
//     (cumulative_seq_len, :645, :659).  The two agree unless that shortest path leaves the band;
//   * an empty read is deleted along the shortest source-to-sink path (first predecessor on ties),
//     score -(gap_open + (L - 1) * gap_extend);
//   * mismatches are one edit per base; every mapping starts at offset 0 (global alignment);
//   * no cell of any sink in band (vg: NoAlignmentInBandException) -> status "no alignment".
#include "tail_align.hpp"
#include <climits>

namespace oracle {

namespace {
constexpr int32_t NEG = INT_MIN / 4;
inline bool alive(int32_t x) { return x > NEG / 2; }
inline bool is_acgt(char c) { return c == 'A' || c == 'C' || c == 'G' || c == 'T'; }
// best of three candidates with M > I > D preference; returns the state (0 M, 1 I, 2 D)
inline int best3(int32_t a, int32_t b, int32_t c, int32_t& v) {
    v = a; int s = 0;
    if (b > v) { v = b; s = 1; }
    if (c > v) { v = c; s = 2; }
    if (!alive(v)) v = NEG;
    return s;
}
inline int32_t sub(int32_t x, int32_t y) { return alive(x) ? x - y : NEG; }
}

struct BandedResult { int status = 0; int32_t score = 0; std::vector<Mapping> path; };

BandedResult banded_global_dag(const Graph& g, const gb_scores& sc, const DagProblem& P, const std::string& q,
                               int64_t pad, bool permissive, uint64_t* cells) {
    const size_t N = P.node.size(), m = q.size(), W = m + 1;
    const int32_t go = sc.gap_open, ge = sc.gap_extend;
    BandedResult out;
    std::vector<int64_t> len(N);
    std::vector<char> has_succ(N, 0);
    for (size_t u = 0; u < N; u++) { len[u] = g.get_length(P.node[u]); for (uint32_t p : P.pred[u]) has_succ[p] = 1; }
    if (N == 0) { out.status = 1; return out; }
    if (m == 0) {
        // shortest source-to-sink path, deleted whole
        std::vector<int64_t> dist(N); std::vector<int64_t> from(N, -1);
        for (size_t u = 0; u < N; u++) {
            int64_t d = 0;
            if (!P.pred[u].empty()) {
                d = INT64_MAX;
                for (uint32_t p : P.pred[u]) if (dist[p] < d) { d = dist[p]; from[u] = p; }
            }
            dist[u] = d + len[u];
        }
        int64_t best = INT64_MAX, bu = -1;
        for (size_t u = 0; u < N; u++) if (!has_succ[u] && dist[u] < best) { best = dist[u]; bu = (int64_t)u; }
        std::vector<uint32_t> walk;
        for (int64_t u = bu; u >= 0; u = from[u]) walk.push_back((uint32_t)u);
        std::reverse(walk.begin(), walk.end());
        for (uint32_t u : walk) { Mapping mp; mp.node = u; Edit e; e.from_length = (uint32_t)len[u]; mp.edits.push_back(e); out.path.push_back(mp); }
        out.score = -(go + (int32_t)(best - 1) * ge);
        return out;
    }
    // ---- bands (path_lengths_to_sinks, find_banded_paths) ----------------------------------------------
    std::vector<int64_t> sts(N, INT64_MAX), lts(N, 0);
    for (size_t u = 0; u < N; u++) if (!has_succ[u]) sts[u] = 0;
    for (size_t i = N; i-- > 0;) {
        for (uint32_t p : P.pred[i]) {
            lts[p] = std::max(lts[p], lts[i] + len[i]);
            if (sts[i] != INT64_MAX) sts[p] = std::min(sts[p], sts[i] + len[i]);
        }
    }
    const int64_t M64 = (int64_t)m;
    std::vector<int64_t> top(N, INT64_MAX), bot(N, INT64_MIN);
    std::vector<char> masked(N, 0);
    for (size_t u = 0; u < N; u++) {
        if (P.pred[u].empty()) {
            if (permissive) { top[u] = std::min(-pad, M64 - (len[u] + lts[u]) - pad); bot[u] = std::max(pad, M64 - (len[u] + sts[u]) + pad); }
            else { top[u] = -pad; bot[u] = pad; }
        } else {
            for (uint32_t p : P.pred[u]) if (!masked[p]) { top[u] = std::min(top[u], top[p] + len[p]); bot[u] = std::max(bot[u], bot[p] + len[p]); }
        }
        if (top[u] > bot[u] || top[u] + len[u] + sts[u] > M64 || bot[u] + len[u] + lts[u] < M64) masked[u] = 1;
    }
    // ---- fill ---------------------------------------------------------------------------------------------
    struct NodeDP { std::vector<int32_t> M, I, D; std::vector<uint8_t> tb; std::vector<uint8_t> argd, argh; };
    std::vector<NodeDP> dp(N);
    // the source's top-edge cell (0, 0) exists regardless of the band (fill_matrix :577-579)
    auto row_lo = [&](size_t u, int64_t c) { return (c == 0 && P.pred[u].empty()) ? 0 : std::max<int64_t>(0, top[u] + c + 1); };
    auto row_hi = [&](size_t u, int64_t c) { return std::min<int64_t>(M64, bot[u] + c + 1); };
    auto in_band = [&](size_t u, int64_t c, int64_t j) { return j >= row_lo(u, c) && j <= row_hi(u, c); };
    for (size_t u = 0; u < N; u++) {
        if (masked[u]) continue;
        NodeDP& n = dp[u];
        const std::string_view seq = g.get_sequence_view(P.node[u]);
        const int64_t L = len[u];
        n.M.assign(L * W, NEG); n.I.assign(L * W, NEG); n.D.assign(L * W, NEG); n.tb.assign(L * W, 0);
        n.argd.assign(W, 0); n.argh.assign(W, 0);
        const bool source = P.pred[u].empty();
        // incoming column: diagonal source value at row j (for M at j + 1) and horizontal value at row j (for D at j)
        std::vector<int32_t> xd(W, NEG), xh(W, NEG); std::vector<uint8_t> sd(W, 0), sh(W, 0);
        if (source) {
            for (size_t j = 0; j < W; j++) {
                const int32_t iv = j == 0 ? NEG : -(go + (int32_t)(j - 1) * ge);
                if (j == 0) { xd[0] = 0; sd[0] = 0; } else { xd[j] = iv; sd[j] = 1; }
                if (j == 0) { xh[0] = -go; sh[0] = 0; }
                else if ((int64_t)j < std::min<int64_t>(bot[u] + 1, M64)) { xh[j] = iv - go; sh[j] = 1; }
            }
        } else {
            for (size_t pi = 0; pi < P.pred[u].size(); pi++) {
                const uint32_t p = P.pred[u][pi];
                if (masked[p]) continue;
                const NodeDP& pn = dp[p];
                const int64_t pl = len[p], snt = top[p] + pl;
                for (int64_t j = std::max<int64_t>(0, snt); j <= row_hi(p, pl - 1); j++) {
                    const size_t k = (pl - 1) * W + j;
                    int32_t v; int s = best3(pn.M[k], pn.I[k], pn.D[k], v);
                    if (v > xd[j]) { xd[j] = v; sd[j] = (uint8_t)s; n.argd[j] = (uint8_t)pi; }
                    if (j - 1 >= snt) {
                        s = best3(sub(pn.M[k], go), sub(pn.I[k], go), sub(pn.D[k], ge), v);
                        if (v > xh[j]) { xh[j] = v; sh[j] = (uint8_t)s; n.argh[j] = (uint8_t)pi; }
                    }
                }
            }
        }
        for (int64_t c = 0; c < L; c++) {
            const char r = seq[c];
            const int64_t lo = row_lo(u, c), hi = row_hi(u, c);
            for (int64_t j = lo; j <= hi; j++) {
                if (cells) (*cells)++;
                const size_t k = c * W + j;
                int32_t mv = NEG, dv = NEG, iv = NEG; int ms = 0, ds = 0, is = 0;
                if (j >= 1) {
                    int32_t src = NEG;
                    if (c == 0) { src = xd[j - 1]; ms = sd[j - 1]; }
                    else if (in_band(u, c - 1, j - 1)) { const size_t kp = (c - 1) * W + j - 1; ms = best3(n.M[kp], n.I[kp], n.D[kp], src); }
                    if (alive(src)) mv = src + ((is_acgt(q[j - 1]) && is_acgt(r)) ? (q[j - 1] == r ? (int32_t)sc.match : -(int32_t)sc.mismatch) : 0);
                }
                if (c == 0) { dv = xh[j]; ds = sh[j]; }
                else if (in_band(u, c - 1, j)) { const size_t kp = (c - 1) * W + j; ds = best3(sub(n.M[kp], go), sub(n.I[kp], go), sub(n.D[kp], ge), dv); }
                if (j >= 1 && j - 1 >= lo) { const size_t kp = k - 1; is = best3(sub(n.M[kp], go), sub(n.I[kp], ge), sub(n.D[kp], go), iv); }
                n.M[k] = mv; n.D[k] = dv; n.I[k] = iv;
                n.tb[k] = (uint8_t)(ms | (ds << 2) | (is << 4));
            }
        }
    }
    // ---- end cell -----------------------------------------------------------------------------------------
    int32_t best = NEG; int64_t bu = -1; int bst = 0;
    for (size_t u = 0; u < N; u++) {
        if (has_succ[u] || masked[u] || !in_band(u, len[u] - 1, M64)) continue;
        const size_t k = (len[u] - 1) * W + m;
        int32_t v; const int s = best3(dp[u].M[k], dp[u].I[k], dp[u].D[k], v);
        if (alive(v) && (bu < 0 || v > best)) { best = v; bu = (int64_t)u; bst = s; }
    }
    if (bu < 0) { out.status = 1; return out; }
    out.score = best;
    // ---- traceback: steps end -> start as (node, op) --------------------------------------------------------
    struct Step { uint32_t u; char op; };
    std::vector<Step> steps;
    int64_t u = bu, c = len[bu] - 1, j = (int64_t)m; int st = bst;
    while (true) {
        const NodeDP& n = dp[u];
        const uint8_t tb = n.tb[c * W + j];
        if (st == 2) {
            steps.push_back({(uint32_t)u, 'D'});
            const int src = (tb >> 2) & 3;
            if (c > 0) { c--; st = src; continue; }
            if (P.pred[u].empty()) { for (int64_t x = 0; x < j; x++) steps.push_back({(uint32_t)u, 'I'}); break; }
            u = P.pred[u][n.argh[j]]; c = len[u] - 1; st = src; continue;
        }
        if (st == 1) { steps.push_back({(uint32_t)u, 'I'}); st = (tb >> 4) & 3; j--; continue; }
        steps.push_back({(uint32_t)u, q[j - 1] == g.get_sequence_view(P.node[u])[c] ? 'M' : 'X'});
        const int src = tb & 3;
        j--;
        if (c > 0) { c--; st = src; continue; }
        if (P.pred[u].empty()) { for (int64_t x = 0; x < j; x++) steps.push_back({(uint32_t)u, 'I'}); break; }
        u = P.pred[u][n.argd[j]]; c = len[u] - 1; st = src;
    }
    std::reverse(steps.begin(), steps.end());
    // ---- steps -> mappings ------------------------------------------------------------------------------
    size_t qpos = 0;
    for (size_t i = 0; i < steps.size();) {
        Mapping mp; mp.node = steps[i].u; mp.offset = 0;
        size_t k = i;
        for (; k < steps.size() && steps[k].u == mp.node; k++) {
            const char op = steps[k].op;
            Edit* last = mp.edits.empty() ? nullptr : &mp.edits.back();
            if (op == 'M') {
                if (last && last->from_length == last->to_length && last->sequence.empty() && last->from_length > 0) { last->from_length++; last->to_length++; }
                else { Edit e; e.from_length = e.to_length = 1; mp.edits.push_back(e); }
                qpos++;
            } else if (op == 'X') {
                Edit e; e.from_length = e.to_length = 1; e.sequence = std::string(1, q[qpos]); mp.edits.push_back(e); qpos++;
            } else if (op == 'I') {
                if (last && last->from_length == 0) { last->to_length++; last->sequence.push_back(q[qpos]); }
                else { Edit e; e.to_length = 1; e.sequence = std::string(1, q[qpos]); mp.edits.push_back(e); }
                qpos++;
            } else {
                if (last && last->to_length == 0) last->from_length++;
                else { Edit e; e.from_length = 1; mp.edits.push_back(e); }
            }
        }
        out.path.push_back(std::move(mp));
        i = k;
    }
    return out;
}

} // namespace oracle

// C entry for the parity tests: one problem, posed like oracle_sw_local, plus the band padding and the
// permissive flag.  Returns 0, or 1 when no global alignment fits the band (nothing written then).
extern "C" int oracle_banded_global(const gb_flat_index* ix, const gb_scores* scores,
                                    const uint32_t* node, uint32_t n_nodes, const uint32_t* pred, const uint32_t* pred_off,
                                    const uint8_t* query, uint32_t qlen, int32_t band_padding, int permissive,
                                    int32_t* score_out, gb_mapping* mappings, uint32_t mapping_cap, uint32_t* n_mappings,
                                    uint32_t* edits, uint32_t edit_cap, uint32_t* n_edits, uint64_t* cells_out) {
    oracle::Graph g(ix);
    oracle::DagProblem P;
    P.node.assign(node, node + n_nodes); P.pred.resize(n_nodes);
    for (uint32_t u = 0; u < n_nodes; u++) P.pred[u].assign(pred + pred_off[u], pred + pred_off[u + 1]);
    uint64_t cells = 0;
    oracle::BandedResult a = oracle::banded_global_dag(g, *scores, P, std::string((const char*)query, qlen), band_padding, permissive != 0, &cells);
    if (cells_out) *cells_out = cells;
    *score_out = a.score; *n_mappings = 0; *n_edits = 0;
    if (a.status) return 1;
    if (a.path.size() > mapping_cap) return -1;
    uint32_t ne = 0;
    for (size_t i = 0; i < a.path.size(); i++) {
        mappings[i].node = a.path[i].node; mappings[i].offset = (uint16_t)a.path[i].offset; mappings[i].n_edits = (uint16_t)a.path[i].edits.size();
        for (const oracle::Edit& e : a.path[i].edits) {
            if (ne >= edit_cap) return -1;
            uint32_t word;
            if (e.from_length == e.to_length && e.sequence.empty()) word = (e.from_length << 4) | GB_EDIT_MATCH;
            else if (e.from_length == e.to_length) {
                uint32_t b = 0; switch (e.sequence[0]) { case 'C': b = 1; break; case 'G': b = 2; break; case 'T': b = 3; break; default: b = 0; }
                word = (e.from_length << 4) | (b << 2) | GB_EDIT_SUB;
            } else if (e.from_length == 0) word = (e.to_length << 4) | GB_EDIT_INS;
            else word = (e.from_length << 4) | GB_EDIT_DEL;
            edits[ne++] = word;
        }
    }
    *n_mappings = (uint32_t)a.path.size(); *n_edits = ne;
    return 0;
}
