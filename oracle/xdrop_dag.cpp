// ORACLE — TEST INFRASTRUCTURE ONLY.  Seeded two-pass X-drop alignment of a read against a DAG:
//   Aligner::align_xdrop(Alignment&, const HandleGraph&, const vector<handle_t>& order,
//                        const vector<MaximalExactMatch>& mems, bool rc, uint16_t max_gap)      aligner.cpp:833-855
//   DozeuInterface::align (two passes)                                                          dozeu_interface.cpp:608-685
//     calculate_seed_position :75-112, scan_seed_position :143-208, do_poa :210-307,
//     calculate_max_position :114-141, align_downward :687-722, calculate_and_save_alignment :338-572
// vg giraffe calls it from attempt_rescue (minimizer_mapper.cpp:3385) with the best gapless extension
// as the only "MEM" (:3345-3358), or with no seed at all when the subgraph holds no seed.
//
// The pass structure below is vg's (dozeu_interface.cpp is part of the reference tree):
//   pass 1  from the seed position, the query suffix that starts at the seed is extended to the right
//           (left-to-right over the topological order) and the best-scoring end position is taken as the
//           "head" (:651-665); without a seed the last 15 query bases are scanned over the whole subgraph
//           for their best local match, whose end is the head (:143-208); no positive match: unaligned;
//   pass 2  from the head, the query prefix that ends at the head is extended to the LEFT and traced back;
//           the query right of the head is reported as a soft clip (:667, :687-722).
// PARITY UNPINNED: the DP inside each pass is vgteam/dozeu @ d0e9ba6 (ABSENT).  Each pass uses the
// cell rules this oracle already defines for the pinned aligner (tail_align.cpp: semi-global affine DP
// pinned at the start, leading insertion <= max_gap, cell-granular X-drop with xt = go + ge * (max_gap - 1),
// first maximum in (node, column, query offset), traceback diagonal > deletion > insertion, open > extend,
// full-length bonus on the last query base of the pass), extended to DAGs by merging the last columns of
// the computed predecessors element-wise (first predecessor on ties; the X-drop reference of a node is the
// largest lineage maximum among them).  On a tree-shaped DAG started at a root this is exactly xdrop_pinned
// (tests/test_xdrop_dag.py checks that).  The scan of pass 1 without a seed is the local DP of full_dp.cpp
// with the bonus at the right end only.
#include "tail_align.hpp"
#include <cassert>
#include <climits>

namespace oracle {

namespace xd {
constexpr int32_t NEG = INT_MIN / 4;
inline bool acgt(char c) { return c == 'A' || c == 'C' || c == 'G' || c == 'T'; }

struct OrientedDag {
    std::vector<std::string> seq;                 // node sequences in the direction of the pass
    std::vector<std::vector<uint32_t>> pred;      // predecessor indices (< own index)
};

struct Step { uint32_t node; char op; };          // 'M' match, 'X' mismatch, 'I' insertion, 'D' deletion

struct PassResult {
    int32_t best = 0; bool have = false;
    uint32_t u = 0, c = 0, j = 0;                 // best cell: node, column, query bases consumed
    std::vector<Step> steps;                      // start -> end (only when traceback was requested)
};

// Pinned X-drop DP over `dag`, starting before base `o` of node `s` with an empty query prefix.
PassResult xdrop_dag_pass(const OrientedDag& dag, const gb_scores& sc, const std::string& query, uint32_t s, uint32_t o,
                          uint32_t max_gap, bool traceback, uint64_t* cells) {
    PassResult out;
    const size_t N = dag.seq.size(), m = query.size(), W = m + 1;
    const int32_t go = sc.gap_open, ge = sc.gap_extend;
    max_gap = std::max<uint32_t>(max_gap, 1);                       // a max_gap of 0 means 1, as in the kernels
    const int32_t xt = go + ge * ((int32_t)max_gap - 1);
    struct NodeDP { std::vector<int32_t> H, E, F, inH, inE; std::vector<int32_t> argH, argE; int32_t lineage_max = 0; bool computed = false; bool live = false; uint32_t first_col = 0; };
    std::vector<NodeDP> dp(N);
    std::vector<int32_t> H0(W, NEG), E0(W, NEG);
    H0[0] = 0;
    for (size_t j = 1; j <= m && j <= max_gap; j++) H0[j] = -(go + (int32_t)(j - 1) * ge);
    for (size_t u = s; u < N; u++) {
        NodeDP& nd = dp[u];
        const std::string& seq = dag.seq[u];
        const size_t len = seq.size();
        int32_t run_max = 0;
        nd.inH.assign(W, NEG); nd.inE.assign(W, NEG); nd.argH.assign(W, -1); nd.argE.assign(W, -1);
        if (u == s) {
            nd.inH = H0; nd.inE = E0; nd.first_col = o; run_max = 0;
        } else {
            bool any = false; run_max = INT_MIN;
            for (size_t pi = 0; pi < dag.pred[u].size(); pi++) {
                const uint32_t p = dag.pred[u][pi];
                if (p < s || !dp[p].computed || !dp[p].live) continue;
                any = true;
                run_max = std::max(run_max, dp[p].lineage_max);
                const NodeDP& pd = dp[p];
                const size_t plen = dag.seq[p].size();
                const int32_t* lh = (plen > pd.first_col) ? &pd.H[(plen - 1) * W] : pd.inH.data();
                const int32_t* le = (plen > pd.first_col) ? &pd.E[(plen - 1) * W] : pd.inE.data();
                for (size_t j = 0; j < W; j++) {
                    if (lh[j] > nd.inH[j]) { nd.inH[j] = lh[j]; nd.argH[j] = (int32_t)pi; }
                    if (le[j] > nd.inE[j]) { nd.inE[j] = le[j]; nd.argE[j] = (int32_t)pi; }
                }
            }
            if (!any) continue;
            nd.first_col = 0;
        }
        nd.computed = true;
        nd.H.assign(len * W, NEG); nd.E.assign(len * W, NEG); nd.F.assign(len * W, NEG);
        const int32_t* pH = nd.inH.data(); const int32_t* pE = nd.inE.data();
        int32_t node_best = NEG; uint32_t node_col = 0, node_j = 0;
        bool last_live = false;
        for (size_t j = 0; j < W; j++) if (pH[j] > NEG) last_live = true;
        for (size_t c = nd.first_col; c < len; c++) {
            int32_t* H = &nd.H[c * W]; int32_t* E = &nd.E[c * W]; int32_t* F = &nd.F[c * W];
            const char r = seq[c];
            for (size_t j = 0; j < W; j++) {
                int32_t e = NEG, f = NEG, d = NEG;
                if (pH[j] > NEG) e = pH[j] - go;
                if (pE[j] > NEG) e = std::max(e, pE[j] - ge);
                if (j > 0) {
                    if (H[j - 1] > NEG) f = H[j - 1] - go;
                    if (F[j - 1] > NEG) f = std::max(f, F[j - 1] - ge);
                    if (pH[j - 1] > NEG) {
                        const char q = query[j - 1];
                        int32_t sub = (q == r && acgt(q)) ? sc.match : -(int32_t)sc.mismatch;
                        if (j == m) sub += sc.full_length_bonus;
                        d = pH[j - 1] + sub;
                    }
                }
                E[j] = e; F[j] = f; H[j] = std::max(d, std::max(e, f));
            }
            if (cells) *cells += W;
            int32_t col_max = NEG; last_live = false;
            for (size_t j = 0; j < W; j++) {
                if (H[j] > NEG && H[j] < run_max - xt) { H[j] = NEG; E[j] = NEG; F[j] = NEG; }
                if (H[j] > col_max) col_max = H[j];
                if (H[j] > NEG) last_live = true;
            }
            for (size_t j = 0; j < W; j++) if (H[j] > node_best) { node_best = H[j]; node_col = (uint32_t)c; node_j = (uint32_t)j; }
            if (col_max > run_max) run_max = col_max;
            pH = H; pE = E;
        }
        nd.live = last_live;
        nd.lineage_max = run_max;
        if (node_best > out.best) { out.best = node_best; out.u = (uint32_t)u; out.c = node_col; out.j = node_j; out.have = true; }
    }
    if (!traceback || !out.have || out.best <= 0) return out;

    // ---- traceback (diagonal > deletion > insertion, open > extend, first predecessor on ties) ----
    uint32_t u = out.u, c = out.c, j = out.j;
    int state = 0;      // 0 H, 1 E, 2 F
    bool at_virtual = false;
    std::vector<Step> steps;
    while (true) {
        if (at_virtual) { for (; j > 0; j--) steps.push_back({s, 'I'}); break; }
        const NodeDP& nd = dp[u];
        const int32_t* H = &nd.H[c * W]; const int32_t* E = &nd.E[c * W]; const int32_t* F = &nd.F[c * W];
        const bool first = c == nd.first_col;
        const int32_t* pH = first ? nd.inH.data() : &nd.H[(c - 1) * W];
        const int32_t* pE = first ? nd.inE.data() : &nd.E[(c - 1) * W];
        // where "the previous column" is, given the query offset jj it is entered at and whether through E
        auto go_prev = [&](uint32_t jj, bool via_E) {
            if (!first) { c--; return; }
            if (u == s) { at_virtual = true; return; }
            uint32_t p = dag.pred[u][via_E ? nd.argE[jj] : nd.argH[jj]];
            // a predecessor without columns of its own (the seed node entered at its end) hands over the virtual column
            while (true) {
                const NodeDP& pd = dp[p];
                if (dag.seq[p].size() > pd.first_col) { u = p; c = (uint32_t)dag.seq[p].size() - 1; return; }
                if (p == s) { u = s; at_virtual = true; return; }
                p = dag.pred[p][via_E ? pd.argE[jj] : pd.argH[jj]];
            }
        };
        if (state == 0) {
            int32_t d = NEG;
            if (j > 0 && pH[j - 1] > NEG) {
                const char q = query[j - 1], r = dag.seq[u][c];
                int32_t sub = (q == r && acgt(q)) ? sc.match : -(int32_t)sc.mismatch;
                if (j == m) sub += sc.full_length_bonus;
                d = pH[j - 1] + sub;
            }
            if (d == H[j]) {
                const char q = query[j - 1], r = dag.seq[u][c];
                steps.push_back({u, (q == r && acgt(q)) ? 'M' : 'X'});
                j--; go_prev(j, false);
                if (at_virtual && j == 0) break;
                continue;
            }
            if (E[j] == H[j]) { state = 1; continue; }
            assert(F[j] == H[j]);
            state = 2; continue;
        }
        if (state == 1) {
            steps.push_back({u, 'D'});
            const bool open = pH[j] > NEG && E[j] == pH[j] - go;
            go_prev(j, !open);
            state = open ? 0 : 1;
            if (at_virtual && j == 0 && state == 0) break;
            continue;
        }
        steps.push_back({u, 'I'});
        const bool open = H[j - 1] > NEG && F[j] == H[j - 1] - go;
        j--;
        state = open ? 0 : 2;
    }
    std::reverse(steps.begin(), steps.end());
    out.steps = std::move(steps);
    return out;
}

// local scan of a short query with the bonus at its right end only: best end cell (full_dp.cpp recurrence)
PassResult scan_local(const OrientedDag& dag, const gb_scores& sc, const std::string& q, uint64_t* cells) {
    PassResult out;
    const size_t N = dag.seq.size(), m = q.size(), W = m + 1;
    const int32_t go = sc.gap_open, ge = sc.gap_extend, bonus = sc.full_length_bonus;
    auto subst = [&](char a, char b) -> int32_t { if (!acgt(a) || !acgt(b)) return 0; return a == b ? (int32_t)sc.match : -(int32_t)sc.mismatch; };
    std::vector<std::vector<int32_t>> lastH(N), lastE(N);
    for (size_t u = 0; u < N; u++) {
        std::vector<int32_t> pH(W, NEG), pE(W, NEG);
        for (uint32_t p : dag.pred[u]) for (size_t j = 0; j < W; j++) { pH[j] = std::max(pH[j], lastH[p][j]); pE[j] = std::max(pE[j], lastE[p][j]); }
        std::vector<int32_t> H(W), E(W), F(W);
        for (size_t c = 0; c < dag.seq[u].size(); c++) {
            H[0] = 0; E[0] = NEG; F[0] = NEG;
            for (size_t j = 1; j < W; j++) {
                if (cells) (*cells)++;
                const int32_t d = std::max(pH[j - 1], 0) + subst(q[j - 1], dag.seq[u][c]);
                int32_t e = NEG;
                if (pH[j] > 0) e = pH[j] - go;
                if (pE[j] > NEG) e = std::max(e, pE[j] - ge);
                if (e <= 0) e = NEG;
                int32_t f = NEG;
                if (H[j - 1] > 0) f = H[j - 1] - go;
                if (F[j - 1] > NEG) f = std::max(f, F[j - 1] - ge);
                if (f <= 0) f = NEG;
                H[j] = std::max(std::max(d, 0), std::max(e, f)); E[j] = e; F[j] = f;
                int32_t cand = H[j];
                if (j == m && d + bonus >= H[j]) cand = d + bonus;
                if (cand > out.best) { out.best = cand; out.u = (uint32_t)u; out.c = (uint32_t)c; out.j = (uint32_t)j; out.have = true; }
            }
            pH = H; pE = E;
        }
        lastH[u] = pH; lastE[u] = pE;
    }
    return out;
}
} // namespace xd
using namespace xd;


// Returns score 0 and an empty path when nothing aligns.
LocalAlignmentResult align_xdrop_dag(const Graph& g, const gb_scores& sc, const DagProblem& P, const std::string& query,
                                     bool has_seed, uint32_t seed_u, uint32_t seed_o, uint32_t seed_q, uint32_t max_gap, uint64_t* cells) {
    LocalAlignmentResult out;
    const size_t N = P.node.size(), m = query.size();
    if (N == 0 || m == 0) return out;
    OrientedDag fwd; fwd.seq.resize(N); fwd.pred = P.pred;
    for (size_t u = 0; u < N; u++) fwd.seq[u] = std::string(g.get_sequence_view(P.node[u]));
    // ---- pass 1: the head -------------------------------------------------------------------------
    uint32_t head_u, head_off, head_q;     // cut after `head_off` bases of node head_u, after head_q query bases
    if (has_seed) {
        PassResult p1 = xdrop_dag_pass(fwd, sc, query.substr(seed_q), seed_u, seed_o, max_gap, false, cells);
        if (p1.have && p1.best > 0) { head_u = p1.u; head_off = p1.c + 1; head_q = seed_q + p1.j; }
        else { head_u = seed_u; head_off = seed_o; head_q = seed_q; }
    } else {
        const size_t scan_len = std::min<size_t>(m, 15);
        PassResult p1 = scan_local(fwd, sc, query.substr(m - scan_len), cells);
        if (!p1.have || p1.best <= 0) return out;
        head_u = p1.u; head_off = p1.c + 1; head_q = (uint32_t)(m - scan_len) + p1.j;
    }
    if (head_q == 0) return out;           // nothing left of the head to align
    // ---- pass 2: leftwards from the head, on the mirrored problem -------------------------------------
    OrientedDag rev; rev.seq.resize(N); rev.pred.resize(N);
    for (size_t u = 0; u < N; u++) { rev.seq[N - 1 - u] = std::string(fwd.seq[u].rbegin(), fwd.seq[u].rend()); }
    for (size_t u = 0; u < N; u++) for (uint32_t p : fwd.pred[u]) rev.pred[N - 1 - p].push_back((uint32_t)(N - 1 - u));
    for (auto& v : rev.pred) std::sort(v.begin(), v.end(), std::greater<uint32_t>());      // successors in forward topological order
    std::string rq(query.rend() - head_q, query.rend());                                  // reversed prefix
    const uint32_t rs = (uint32_t)(N - 1 - head_u), ro = (uint32_t)(fwd.seq[head_u].size() - head_off);
    PassResult p2 = xdrop_dag_pass(rev, sc, rq, rs, ro, max_gap, true, cells);
    if (!p2.have || p2.best <= 0) return out;
    out.score = p2.best;
    // steps are start -> end in mirrored space = head -> alignment start; turn them around
    std::vector<Step> steps(p2.steps.rbegin(), p2.steps.rend());
    const uint32_t aligned_q = (uint32_t)std::count_if(steps.begin(), steps.end(), [](const Step& s) { return s.op != 'D'; });
    size_t qpos = head_q - aligned_q;      // leading soft clip
    size_t i = 0;
    while (i < steps.size()) {
        const uint32_t ru = steps[i].node, u = (uint32_t)(N - 1 - ru);
        size_t k = i, cols = 0;
        while (k < steps.size() && steps[k].node == ru) { if (steps[k].op != 'I') cols++; k++; }
        Mapping mp; mp.node = u;
        const size_t end = (u == head_u) ? head_off : fwd.seq[u].size();
        mp.offset = (uint32_t)(end - cols);
        if (i == 0 && qpos > 0) mp.edits.push_back(Edit{0, (uint32_t)qpos, query.substr(0, qpos)});
        char cur = 0; size_t run = 0;
        auto flush = [&]() {
            if (cur == 'X') { for (size_t x = 0; x < run; x++) { mp.edits.push_back(Edit{1, 1, std::string(1, query[qpos])}); qpos++; } }
            else if (run > 0) {
                if (cur == 'M') { mp.edits.push_back(Edit{(uint32_t)run, (uint32_t)run, ""}); qpos += run; }
                else if (cur == 'I') {
                    if (!mp.edits.empty() && mp.edits.back().from_length == 0) { mp.edits.back().to_length += (uint32_t)run; mp.edits.back().sequence += query.substr(qpos, run); }
                    else mp.edits.push_back(Edit{0, (uint32_t)run, query.substr(qpos, run)});
                    qpos += run;
                }
                else mp.edits.push_back(Edit{(uint32_t)run, 0, ""});
            }
        };
        for (size_t x = i; x < k; x++) {
            if (steps[x].op == cur) run++; else { if (cur) flush(); cur = steps[x].op; run = 1; }
        }
        if (cur) flush();
        out.path.push_back(std::move(mp));
        i = k;
    }
    if (!out.path.empty() && head_q < m) {
        Edit& last = out.path.back().edits.back();
        if (last.from_length == 0) { last.to_length += (uint32_t)(m - head_q); last.sequence += query.substr(head_q); }
        else out.path.back().edits.push_back(Edit{0, (uint32_t)(m - head_q), query.substr(head_q)});
    }
    return out;
}

} // namespace oracle

// Test hook: ONE pass (left to right, with traceback) from (start_u, start_o); on a tree started at its
// root this must reproduce oracle_xdrop_pinned.  Mappings in problem space, offsets = first column used.
extern "C" int oracle_xdrop_dag_pass(const gb_flat_index* ix, const gb_scores* scores,
                                     const uint32_t* node, uint32_t n_nodes, const uint32_t* pred, const uint32_t* pred_off,
                                     const uint8_t* query, uint32_t qlen, uint32_t start_u, uint32_t start_o, uint32_t max_gap,
                                     int32_t* score_out, uint32_t* ops_out, uint32_t ops_cap, uint32_t* n_ops) {
    oracle::Graph g(ix);
    oracle::OrientedDag dag; dag.seq.resize(n_nodes); dag.pred.resize(n_nodes);
    for (uint32_t u = 0; u < n_nodes; u++) {
        dag.seq[u] = std::string(g.get_sequence_view(node[u]));
        dag.pred[u].assign(pred + pred_off[u], pred + pred_off[u + 1]);
    }
    oracle::PassResult r = oracle::xdrop_dag_pass(dag, *scores, std::string((const char*)query, qlen), start_u, start_o, max_gap, true, nullptr);
    *score_out = (r.have && r.best > 0) ? r.best : 0;
    *n_ops = 0;
    if (r.steps.size() > ops_cap) return -1;
    for (const auto& st : r.steps) ops_out[(*n_ops)++] = (st.node << 8) | (uint32_t)st.op;
    return 0;
}

// C entry: one problem; seed_u = 0xffffffff selects the seedless scan.  Mappings in PROBLEM space.
extern "C" int oracle_xdrop_dag(const gb_flat_index* ix, const gb_scores* scores,
                                const uint32_t* node, uint32_t n_nodes, const uint32_t* pred, const uint32_t* pred_off,
                                const uint8_t* query, uint32_t qlen, uint32_t seed_u, uint32_t seed_o, uint32_t seed_q, uint32_t max_gap,
                                int32_t* score_out, gb_mapping* mappings, uint32_t mapping_cap, uint32_t* n_mappings,
                                uint32_t* edits, uint32_t edit_cap, uint32_t* n_edits, uint64_t* cells_out) {
    oracle::Graph g(ix);
    oracle::DagProblem P;
    P.node.assign(node, node + n_nodes); P.pred.resize(n_nodes);
    for (uint32_t u = 0; u < n_nodes; u++) P.pred[u].assign(pred + pred_off[u], pred + pred_off[u + 1]);
    uint64_t cells = 0;
    oracle::LocalAlignmentResult a = oracle::align_xdrop_dag(g, *scores, P, std::string((const char*)query, qlen), seed_u != 0xffffffffu,
                                                            seed_u, seed_o, seed_q, max_gap, &cells);
    if (cells_out) *cells_out = cells;
    *score_out = a.score;
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
