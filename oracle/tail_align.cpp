// ORACLE — TEST INFRASTRUCTURE ONLY.  See tail_align.hpp for the reference lines restated.
//
// ---- The X-drop DP contract (parity UNPINNED against vgteam/dozeu @ d0e9ba6) -----------
// dozeu's source is not in /root/reference (deps/dozeu is empty), so its band-pruning
// granularity (8-lane SSE blocks) and traceback tie-breaks cannot be restated.  This file
// DEFINES the semantics our CUDA kernel is held to, chosen to reproduce everything the
// reference's own tests pin (src/unittest/xdrop_aligner.cpp:267-686, transcribed in
// tests/golden/xdrop_pinned.json) and vg's call-site contract (dozeu_interface.cpp:210-572):
//   * semi-global affine-gap DP, pinned at (tree root start, query start), free at the other
//     end; a gap of n bases costs gap_open + (n-1)*gap_extend; the full-length bonus is
//     added to the substitution score of the LAST query base (dz_pack_query_forward,
//     xdrop_aligner.cpp:86-94);
//   * leading insertions are allowed up to max_gap_length bases (dz_align_init root column);
//   * X-drop at CELL granularity: after a column is filled, a cell whose H is below
//     (best H in any earlier column of this root-to-node lineage) - xt is dead, with
//     xt = gap_open + gap_extend * (max_gap_length - 1), the cost of the longest allowed gap
//     (consistent with the title of xdrop_aligner.cpp:819); a node is only entered if its parent's
//     last column has a live cell (fr.epos > fr.spos, dozeu_interface.cpp:264);
//   * the reported cell is the maximum H: first node in tree order (= lazy topological order
//     of a DFS-numbered tree) that strictly improves (dozeu_interface.cpp:287), inside it
//     the first column, inside that the smallest query offset; max 0 -> pure softclip
//     (dozeu_interface.cpp:344-360);
//   * traceback preference at a cell: substitution/match, then deletion, then insertion;
//     inside a gap, "open" is preferred over "extend";
//   * non-ACGT bases never match.
#include "tail_align.hpp"

#include <algorithm>
#include <cassert>
#include <limits>
#include <list>
#include <stack>

namespace oracle {

namespace {

const int32_t NEG = std::numeric_limits<int32_t>::min() / 4;

inline bool is_acgt(char c) { return c == 'A' || c == 'C' || c == 'G' || c == 'T'; }

std::string tree_node_sequence(const Graph& g, const TailTree& t, size_t i) {
    std::string_view v = g.get_sequence_view(t.nodes[i].second);
    if (i == 0) v = v.substr(t.root_trim);
    return std::string(v);
}

char complement(char c) {
    switch (c) { case 'A': return 'T'; case 'C': return 'G'; case 'G': return 'C'; case 'T': return 'A'; default: return 'N'; }
}
std::string reverse_complement(const std::string& s) {
    std::string r(s.rbegin(), s.rend());
    for (char& c : r) c = complement(c);
    return r;
}

} // namespace

// EditAlignmentScorer::longest_detectable_gap(read_length, read_pos), alignment_scorer.cpp:264-271
size_t longest_detectable_gap(const gb_scores& s, size_t read_length, size_t read_pos) {
    int64_t overhang_length = std::min(read_pos, read_length - read_pos);
    int64_t numer = (int64_t)s.match * overhang_length + s.full_length_bonus;
    int64_t gap_length = (numer - s.gap_open) / s.gap_extend + 1;
    return gap_length >= 0 && overhang_length > 0 ? (size_t)gap_length : 0;
}

// ---------------------------------------------------------------------------------------
// xdrop_pinned
// ---------------------------------------------------------------------------------------
PinnedAlignment xdrop_pinned(const Graph& g, const gb_scores& sc, const TailTree& tree,
                             const std::string& query, uint32_t max_gap_length, uint64_t* cells) {
    PinnedAlignment out;
    const size_t m = query.size(), n_nodes = tree.nodes.size();
    const int32_t go = sc.gap_open, ge = sc.gap_extend;
    max_gap_length = std::max<uint32_t>(max_gap_length, 1);         // a max_gap of 0 means 1, as in the kernels
    const int32_t xt = go + ge * ((int32_t)max_gap_length - 1);   // cost of the longest allowed gap
    struct NodeDP {
        std::string seq;
        std::vector<int32_t> H, E, F;      // [len][m+1]
        int32_t lineage_max = 0;           // best H in columns up to and including this node
        bool computed = false;
    };
    std::vector<NodeDP> dp(n_nodes);
    // virtual column before the root
    std::vector<int32_t> H0(m + 1, NEG), E0(m + 1, NEG), F0(m + 1, NEG);
    H0[0] = 0;
    for (size_t j = 1; j <= m && j <= max_gap_length; j++) { F0[j] = -(go + (int32_t)(j - 1) * ge); H0[j] = F0[j]; }

    int32_t best = 0; size_t best_node = 0, best_col = 0, best_j = 0; bool have_best = false;
    for (size_t i = 0; i < n_nodes; i++) {
        NodeDP& nd = dp[i];
        nd.seq = tree_node_sequence(g, tree, i);
        const size_t len = nd.seq.size();
        const int32_t *pH, *pE;
        int32_t run_max;
        if (tree.nodes[i].first < 0) { pH = H0.data(); pE = E0.data(); run_max = 0; }
        else {
            const NodeDP& par = dp[(size_t)tree.nodes[i].first];
            if (!par.computed) continue;
            const size_t plen = par.seq.size();
            pH = par.H.data() + (plen - 1) * (m + 1); pE = par.E.data() + (plen - 1) * (m + 1);
            bool live = false;
            for (size_t j = 0; j <= m; j++) if (pH[j] > NEG) { live = true; break; }
            if (!live) continue;
            run_max = par.lineage_max;
        }
        nd.H.assign(len * (m + 1), NEG); nd.E.assign(len * (m + 1), NEG); nd.F.assign(len * (m + 1), NEG);
        nd.computed = true;
        int32_t node_best = NEG; size_t node_col = 0, node_j = 0;
        for (size_t c = 0; c < len; c++) {
            int32_t* H = nd.H.data() + c * (m + 1); int32_t* E = nd.E.data() + c * (m + 1); int32_t* F = nd.F.data() + c * (m + 1);
            const char r = nd.seq[c];
            for (size_t j = 0; j <= m; j++) {
                int32_t e = NEG, f = NEG, d = NEG;
                if (pH[j] > NEG) e = pH[j] - go;
                if (pE[j] > NEG) e = std::max(e, pE[j] - ge);
                if (j > 0) {
                    if (H[j - 1] > NEG) f = H[j - 1] - go;
                    if (F[j - 1] > NEG) f = std::max(f, F[j - 1] - ge);
                    if (pH[j - 1] > NEG) {
                        const char q = query[j - 1];
                        int32_t s = (q == r && is_acgt(q)) ? sc.match : -(int32_t)sc.mismatch;
                        if (j == m) s += sc.full_length_bonus;
                        d = pH[j - 1] + s;
                    }
                }
                E[j] = e; F[j] = f;
                H[j] = std::max(d, std::max(e, f));
            }
            if (cells) *cells += m + 1;
            // X-drop against the best of the earlier columns, then fold this column in
            int32_t col_max = NEG;
            for (size_t j = 0; j <= m; j++) {
                if (H[j] > NEG && H[j] < run_max - xt) { H[j] = NEG; E[j] = NEG; F[j] = NEG; }
                if (H[j] > col_max) col_max = H[j];
            }
            for (size_t j = 0; j <= m; j++) if (H[j] > node_best) { node_best = H[j]; node_col = c; node_j = j; }
            if (col_max > run_max) run_max = col_max;
            pH = H; pE = E;
        }
        nd.lineage_max = run_max;
        if (node_best > best) { best = node_best; best_node = i; best_col = node_col; best_j = node_j; have_best = true; }
    }

    out.score = best;
    auto softclip = [&]() {
        // full-length insertion on the head node (dozeu_interface.cpp:344-360)
        Mapping mp; mp.node = 1; mp.offset = 0;
        mp.edits.push_back(Edit{0, (uint32_t)m, query});
        out.path.push_back(std::move(mp));
        out.score = 0;
    };
    if (!have_best || best <= 0) { softclip(); return out; }

    // ---- traceback -------------------------------------------------------------------------
    // ops per node in reverse order: 'M' match, 'X' mismatch, 'I' insertion, 'D' deletion
    struct Step { size_t node; char op; };
    std::vector<Step> steps;
    size_t node = best_node, col = best_col, j = best_j;
    enum { ST_H, ST_E, ST_F } state = ST_H;
    bool at_virtual = false;
    while (true) {
        if (at_virtual) {
            // leading insertion in the virtual column: j query bases before any graph base
            for (; j > 0; j--) steps.push_back(Step{0, 'I'});
            break;
        }
        const NodeDP& nd = dp[node];
        const int32_t* H = nd.H.data() + col * (m + 1); const int32_t* E = nd.E.data() + col * (m + 1); const int32_t* F = nd.F.data() + col * (m + 1);
        // previous column
        const int32_t *pH, *pE; size_t pnode = node, pcol = 0; bool p_virtual = false;
        if (col > 0) { pH = nd.H.data() + (col - 1) * (m + 1); pE = nd.E.data() + (col - 1) * (m + 1); pcol = col - 1; }
        else if (tree.nodes[node].first < 0) { pH = H0.data(); pE = E0.data(); p_virtual = true; }
        else {
            pnode = (size_t)tree.nodes[node].first;
            const NodeDP& par = dp[pnode];
            pcol = par.seq.size() - 1;
            pH = par.H.data() + pcol * (m + 1); pE = par.E.data() + pcol * (m + 1);
        }
        if (state == ST_H) {
            int32_t d = NEG;
            if (j > 0 && pH[j - 1] > NEG) {
                const char q = query[j - 1], r = nd.seq[col];
                int32_t s = (q == r && is_acgt(q)) ? sc.match : -(int32_t)sc.mismatch;
                if (j == m) s += sc.full_length_bonus;
                d = pH[j - 1] + s;
            }
            if (d == H[j]) {
                const char q = query[j - 1], r = nd.seq[col];
                steps.push_back(Step{node, (q == r && is_acgt(q)) ? 'M' : 'X'});
                j--; node = pnode; col = pcol; at_virtual = p_virtual;
                if (at_virtual && j == 0) break;
                continue;
            }
            if (E[j] == H[j]) { state = ST_E; continue; }
            assert(F[j] == H[j]);
            state = ST_F; continue;
        }
        if (state == ST_E) {
            steps.push_back(Step{node, 'D'});
            const bool open = pH[j] > NEG && E[j] == pH[j] - go;
            node = pnode; col = pcol; at_virtual = p_virtual;
            state = open ? ST_H : ST_E;
            if (at_virtual && j == 0 && state == ST_H) break;
            continue;
        }
        // ST_F
        steps.push_back(Step{node, 'I'});
        const bool open = H[j - 1] > NEG && F[j] == H[j - 1] - go;
        j--;
        state = open ? ST_H : ST_F;
    }
    std::reverse(steps.begin(), steps.end());

    // ---- ops -> Mappings (calculate_and_save_alignment, dozeu_interface.cpp:493-533) ---------
    size_t query_offset = 0;
    auto flush = [&](Mapping& mp, char op, size_t len) {
        if (op == 'X') { for (size_t x = 0; x < len; x++) { mp.edits.push_back(Edit{1, 1, std::string(1, query[query_offset])}); query_offset++; } }
        else if (len > 0) {
            if (op == 'M') { mp.edits.push_back(Edit{(uint32_t)len, (uint32_t)len, ""}); query_offset += len; }
            else if (op == 'I') { mp.edits.push_back(Edit{0, (uint32_t)len, query.substr(query_offset, len)}); query_offset += len; }
            else { mp.edits.push_back(Edit{(uint32_t)len, 0, ""}); }
        }
    };
    size_t si = 0;
    while (si < steps.size()) {
        const size_t nd_i = steps[si].node;
        Mapping mp; mp.node = (uint32_t)nd_i + 1; mp.offset = 0;
        char cur = 0; size_t run = 0;
        while (si < steps.size() && steps[si].node == nd_i) {
            if (steps[si].op == cur) run++;
            else { if (cur) flush(mp, cur, run); cur = steps[si].op; run = 1; }
            si++;
        }
        if (cur) flush(mp, cur, run);
        out.path.push_back(std::move(mp));
    }
    if (!out.path.empty() && query_offset != m) {
        // trailing bases dozeu did not align: trailing insert (softclip) on the last mapping
        out.path.back().edits.push_back(Edit{0, (uint32_t)(m - query_offset), query.substr(query_offset)});
    }
    return out;
}

// ---------------------------------------------------------------------------------------
// get_tail_forest + dfs_gbwt, minimizer_mapper.cpp:5745-6013
// ---------------------------------------------------------------------------------------
static void dfs_gbwt(const Graph& g, const SearchState& start_state, size_t from_offset, size_t walk_distance,
                     const std::function<void(uint32_t)>& enter_handle, const std::function<void(void)>& exit_handle) {
    if (start_state.empty()) return;
    size_t remaining_root = g.get_length(start_state.node) - from_offset;
    struct Frame { SearchState here_state; size_t used_distance; bool visit; };
    std::vector<Frame> stack;
    stack.push_back({start_state, 0, false});
    while (!stack.empty()) {
        const size_t top = stack.size() - 1;
        const uint32_t here_handle = stack[top].here_state.node;
        bool is_root = (stack.size() == 1);
        bool is_hidden_root = (is_root && remaining_root == 0);
        if (stack[top].visit == false) {
            stack[top].visit = true;
            if (!is_hidden_root) enter_handle(here_handle);
            size_t node_length = is_root ? remaining_root : g.get_length(here_handle);
            stack[top].used_distance += node_length;
            if (stack[top].used_distance < walk_distance) {
                const SearchState here = stack[top].here_state;
                const size_t used = stack[top].used_distance;
                g.follow_paths(here, [&](const SearchState& there) -> bool { stack.push_back({there, used, false}); return true; });
                continue;
            }
        }
        if (!is_hidden_root) exit_handle();
        stack.pop_back();
    }
}

std::vector<TailTree> get_tail_forest(const Graph& g, const gb_scores& scores, const GaplessExtension& ext,
                                      size_t read_length, bool left_tails, size_t* longest_gap) {
    std::vector<TailTree> to_return;
    uint32_t from_node; size_t from_offset; size_t tail_length; const SearchState* base_state;
    if (left_tails) {
        // starting_position reversed: reverse(Position, node_length), position.cpp:41-46
        const auto start = ext.starting_position(g);
        from_node = start.first ^ 1u;
        from_offset = g.get_length(start.first) - start.second;
        base_state = &ext.state.backward;
        tail_length = ext.read_interval.first;
    } else {
        // tail_position, gbwt_extender.cpp:68-87
        const auto tail = ext.tail_position(g);
        from_node = tail.first;
        from_offset = tail.second;
        base_state = &ext.state.forward;
        tail_length = read_length - ext.read_interval.second;
    }
    if (tail_length == 0) return to_return;
    (void)from_node;
    std::vector<std::pair<int64_t, uint32_t>> tree;
    std::vector<int64_t> parent_stack;
    bool start_included = from_offset < g.get_length(from_node);
    size_t gap = longest_detectable_gap(scores, read_length, tail_length);
    if (longest_gap) *longest_gap = gap;
    size_t search_limit = gap + tail_length;
    dfs_gbwt(g, *base_state, from_offset, search_limit, [&](uint32_t entered) {
        if (parent_stack.empty()) {
            if (!tree.empty()) { to_return.push_back(TailTree{std::move(tree), start_included ? from_offset : 0}); tree.clear(); }
            tree.emplace_back(-1, entered);
        } else {
            tree.emplace_back(parent_stack.back(), entered);
        }
        parent_stack.push_back((int64_t)tree.size() - 1);
    }, [&]() { parent_stack.pop_back(); });
    if (!tree.empty()) to_return.push_back(TailTree{std::move(tree), start_included ? from_offset : 0});
    return to_return;
}

// ---------------------------------------------------------------------------------------
// get_best_alignment_against_any_tree, minimizer_mapper.cpp:5626-5743
// ---------------------------------------------------------------------------------------
static size_t tree_node_length(const Graph& g, const TailTree& t, size_t i) {
    size_t l = g.get_length(t.nodes[i].second);
    return i == 0 ? l - t.root_trim : l;
}

// reverse_complement_path (path.cpp:1791-1882) on tree-space mappings
static std::vector<Mapping> reverse_complement_path(const std::vector<Mapping>& path, const Graph& g, const TailTree& t,
                                                    std::vector<bool>& is_reverse_out) {
    std::vector<Mapping> reversed;
    for (int64_t i = (int64_t)path.size() - 1; i >= 0; i--) {
        const Mapping& m = path[i];
        Mapping r; r.node = m.node;
        size_t used = 0; for (const Edit& e : m.edits) used += e.from_length;
        size_t node_length = tree_node_length(g, t, m.node - 1);
        r.offset = (uint32_t)(node_length - used - m.offset);
        for (int64_t k = (int64_t)m.edits.size() - 1; k >= 0; k--) {
            Edit e = m.edits[k];
            e.sequence = reverse_complement(e.sequence);
            r.edits.push_back(std::move(e));
        }
        reversed.push_back(std::move(r));
    }
    is_reverse_out.assign(reversed.size(), true);
    return reversed;
}

static std::pair<std::vector<Mapping>, int32_t>
get_best_alignment_against_any_tree(const Graph& g, const gb_scores& scores, const gb_map_params& P,
                                    const std::vector<TailTree>& trees, const std::string& sequence,
                                    uint32_t default_node, uint32_t default_offset, bool pin_left,
                                    size_t longest_gap, LazyRNG& rng, MapCounters* counters) {
    std::vector<Mapping> best_path;
    int32_t best_score = 0;
    if (!sequence.empty()) {
        Mapping m; m.node = default_node; m.offset = default_offset;
        m.edits.push_back(Edit{0, (uint32_t)sequence.size(), sequence});
        best_path.push_back(std::move(m));
    }
    for (const TailTree& tree : trees) {
        if (tree.nodes.empty()) continue;
        std::string aln_seq = pin_left ? sequence : reverse_complement(sequence);
        size_t tail_subgraph_bases = 0;
        for (size_t i = 0; i < tree.nodes.size(); i++) tail_subgraph_bases += tree_node_length(g, tree, i);
        PinnedAlignment cur;
        bool aligned = false;
        if (tail_subgraph_bases * sequence.size() > P.max_dozeu_cells) {
            // refused: no path, score 0
        } else {
            uint32_t gap = (uint32_t)std::max<size_t>(longest_gap, 1);   // aligner.cpp:638; uint16_t in the reference
            gap = std::min<uint32_t>(gap, 65535u);
            uint64_t cells = 0;
            cur = xdrop_pinned(g, scores, tree, aln_seq, gap, &cells);
            aligned = true;
            if (counters) { counters->tail_dps++; counters->tail_cells += cells; counters->tail_nodes += tree.nodes.size(); counters->tail_bases += tail_subgraph_bases; }
        }
        if (aligned && !cur.path.empty() && deterministic_beats(cur.score, best_score, rng)) {
            std::vector<Mapping> path = cur.path;
            std::vector<bool> rev(path.size(), false);
            if (!pin_left) path = reverse_complement_path(path, g, tree, rev);
            // translate_down, tree_subgraph.cpp:172-195
            for (size_t i = 0; i < path.size(); i++) {
                const size_t ti = path[i].node - 1;
                uint32_t underlying = tree.nodes[ti].second;
                if (rev[i]) underlying ^= 1u;
                if (ti == 0 && !rev[i] && tree.root_trim != 0) path[i].offset += (uint32_t)tree.root_trim;
                path[i].node = underlying;
            }
            best_path = std::move(path);
            best_score = cur.score;
        }
    }
    return {best_path, best_score};
}

// ---------------------------------------------------------------------------------------
// find_optimal_tail_alignments, minimizer_mapper.cpp:5266-5622
// ---------------------------------------------------------------------------------------
typedef std::pair<uint32_t, int32_t> pareto_point;

static void find_pareto_frontier(std::vector<pareto_point>& v) {
    if (v.empty()) return;
    std::sort(v.begin(), v.end(), [](pareto_point a, pareto_point b) { return (a.second < b.second || (a.second == b.second && a.first > b.first)); });
    size_t tail = 1;
    for (size_t i = 1; i < v.size(); i++) {
        if (v[i].first <= v[tail - 1].first) continue;
        v[tail] = v[i]; tail++;
    }
    v.resize(tail);
    std::sort(v.begin(), v.end());
}
static int32_t gap_penalty(size_t length, const gb_scores& s) { return length == 0 ? 0 : s.gap_open + ((int32_t)length - 1) * s.gap_extend; }
static int32_t mismatch_penalty(size_t n, const gb_scores& s) { return (int32_t)n * (s.match + s.mismatch); }
static int32_t gap_penalty(size_t start, size_t limit, const gb_scores& s) {
    return start >= limit ? s.gap_open : s.gap_open + ((int32_t)(limit - start) - 1) * s.gap_extend;
}
static int32_t flank_penalty(size_t length, const std::vector<pareto_point>& frontier, const gb_scores& s) {
    int32_t result = gap_penalty(length, s);
    for (size_t i = 0; i < frontier.size(); i++) {
        int32_t candidate = frontier[i].second + gap_penalty(frontier[i].first, length, s);
        result = std::min(result, candidate);
        if (frontier[i].first >= length) break;
    }
    return result;
}

static bool mapping_is_total_insertion(const Mapping& m) { return m.edits.size() == 1 && m.edits[0].from_length == 0 && m.edits[0].to_length > 0; }

// add_to_path, minimizer_mapper.cpp:5318-5367
static void add_to_path(std::vector<Mapping>& target, std::vector<Mapping>& to_append) {
    for (Mapping& mapping : to_append) {
        if (!target.empty()) {
            Mapping& prev = target.back();
            if ((mapping.node >> 1) == (prev.node >> 1)) {
                bool can_combine = false;
                if (mapping.offset != 0) can_combine = true;
                else {
                    bool prev_ti = mapping_is_total_insertion(prev), ti = mapping_is_total_insertion(mapping);
                    if (prev_ti || ti) {
                        can_combine = true;
                        if (prev_ti) { prev.node = mapping.node; prev.offset = mapping.offset; }
                    }
                }
                if (can_combine) { for (Edit& e : mapping.edits) prev.edits.push_back(std::move(e)); continue; }
            }
        }
        target.push_back(std::move(mapping));
    }
}

double path_identity(const std::vector<Mapping>& path) {
    // identity(const Path&), path.cpp:2316-2335
    size_t total_length = 0, matched_length = 0;
    for (const Mapping& m : path) for (const Edit& e : m.edits) total_length += e.to_length;
    for (size_t i = 0; i < path.size(); i++)
        for (size_t j = 0; j < path[i].edits.size(); j++) {
            const Edit& e = path[i].edits[j];
            if (e.from_length == e.to_length && e.sequence.empty()) matched_length += e.from_length;
            else if (e.from_length == 0 && e.to_length > 0) {
                bool first = (i == 0 && j == 0), last = (i == path.size() - 1 && j == path[i].edits.size() - 1);
                if (first || last) total_length -= e.to_length;
            }
        }
    return total_length == 0 ? 0.0 : (double)matched_length / (double)total_length;
}

void find_optimal_tail_alignments(const Graph& g, const gb_scores& scores, const gb_map_params& P,
                                  const std::string& sequence, const std::vector<GaplessExtension>& extended_seeds,
                                  LazyRNG& rng, Alignment& best, Alignment& second_best, MapCounters* counters) {
    size_t min_tails = 1;
    for (const GaplessExtension& e : extended_seeds) if (e.full()) min_tails++;
    if (min_tails < 2) min_tails = 2;

    std::vector<pareto_point> left_frontier, right_frontier;
    {
        size_t seq_len = sequence.length();
        for (const GaplessExtension& e : extended_seeds) {
            if (e.full()) continue;
            int32_t left_penalty = gap_penalty(e.read_interval.first, scores);
            int32_t mid_penalty = mismatch_penalty(e.mismatch_positions.size(), scores);
            int32_t right_penalty = gap_penalty(seq_len - e.read_interval.second, scores);
            left_frontier.push_back(pareto_point((uint32_t)e.read_interval.second, mid_penalty + left_penalty));
            right_frontier.push_back(pareto_point((uint32_t)(seq_len - e.read_interval.first), mid_penalty + right_penalty));
            if (!e.mismatch_positions.empty()) {
                left_frontier.push_back(pareto_point((uint32_t)e.mismatch_positions.front(), left_penalty));
                right_frontier.push_back(pareto_point((uint32_t)(seq_len - e.mismatch_positions.back() - 1), right_penalty));
            }
        }
        size_t window_length = (size_t)g.ix->k + g.ix->w - 1;
        left_frontier.push_back(pareto_point((uint32_t)window_length - 1, 0));
        right_frontier.push_back(pareto_point((uint32_t)window_length - 1, 0));
    }
    find_pareto_frontier(left_frontier);
    find_pareto_frontier(right_frontier);

    std::vector<Mapping> winning_left, winning_middle, winning_right, second_left, second_middle, second_right;
    int32_t winning_score = 0, second_score = 0;
    bool partial_extension_aligned = false;
    int32_t threshold = -1;

    process_until_threshold_e<double>(extended_seeds.size(),
        [&](size_t i) -> double { return (double)extended_seeds[i].score; },
        [&](size_t a, size_t b) -> bool { return extended_seeds[a].score > extended_seeds[b].score; },
        [&](size_t) -> bool { return false; },
        P.extension_score_threshold, min_tails, std::numeric_limits<size_t>::max(), rng,
        [&](size_t extended_seed_num, size_t, bool) -> bool {
            const GaplessExtension& extension = extended_seeds[extended_seed_num];
            if (threshold < 0) threshold = extension.score - P.extension_score_threshold;
            if (!extension.full()) {
                if (partial_extension_aligned && extension.score <= threshold) {
                    int32_t score_estimate = (int32_t)sequence.length() * scores.match + 2 * scores.full_length_bonus -
                                             mismatch_penalty(extension.mismatch_positions.size(), scores);
                    if (!extension.left_full) score_estimate -= flank_penalty(extension.read_interval.first, left_frontier, scores);
                    if (!extension.right_full) score_estimate -= flank_penalty(sequence.length() - extension.read_interval.second, right_frontier, scores);
                    if (score_estimate <= winning_score) return true;
                }
                partial_extension_aligned = true;
            }
            std::pair<std::vector<Mapping>, int32_t> left_tail_result{{}, 0}, right_tail_result{{}, 0};
            if (!extension.left_full) {
                size_t gap;
                auto forest = get_tail_forest(g, scores, extension, sequence.size(), true, &gap);
                std::string before_sequence = sequence.substr(0, extension.read_interval.first);
                left_tail_result = get_best_alignment_against_any_tree(g, scores, P, forest, before_sequence,
                    extension.path.front(), (uint32_t)extension.offset, false, gap, rng, counters);
            }
            if (!extension.right_full) {
                size_t gap;
                auto forest = get_tail_forest(g, scores, extension, sequence.size(), false, &gap);
                std::string trailing_sequence = sequence.substr(extension.read_interval.second);
                size_t tail_off = extension.offset + extension.length();
                for (size_t i = 0; i + 1 < extension.path.size(); i++) tail_off -= g.get_length(extension.path[i]);
                right_tail_result = get_best_alignment_against_any_tree(g, scores, P, forest, trailing_sequence,
                    extension.path.back(), (uint32_t)tail_off, true, gap, rng, counters);
            }
            int32_t total_score = extension.score + left_tail_result.second + right_tail_result.second;

            auto node_id = [](uint32_t v) { return (int64_t)(v >> 1); };
            int64_t winning_start = winning_score == 0 ? 0 : (winning_left.empty() ? node_id(winning_middle.front().node) : node_id(winning_left.front().node));
            int64_t current_start = left_tail_result.first.empty() ? node_id(extension.path.front()) : node_id(left_tail_result.first.front().node);
            int64_t winning_end = winning_score == 0 ? 0 : (winning_right.empty() ? node_id(winning_middle.back().node) : node_id(winning_right.back().node));
            int64_t current_end = right_tail_result.first.empty() ? node_id(extension.path.back()) : node_id(right_tail_result.first.back().node);
            bool different_left = winning_start != current_start;
            bool different_right = winning_end != current_end;

            if (total_score > winning_score || winning_score == 0) {
                if (winning_score != 0 && different_left && different_right) {
                    second_score = winning_score;
                    second_left = std::move(winning_left); second_middle = std::move(winning_middle); second_right = std::move(winning_right);
                }
                winning_score = total_score;
                winning_left = std::move(left_tail_result.first);
                winning_middle = extension_to_path(g, extension, sequence);
                winning_right = std::move(right_tail_result.first);
            } else if ((total_score > second_score || second_score == 0) && different_left && different_right) {
                second_score = total_score;
                second_left = std::move(left_tail_result.first);
                second_middle = extension_to_path(g, extension, sequence);
                second_right = std::move(right_tail_result.first);
            }
            return true;
        },
        [&](size_t) {}, [&](size_t) {});

    best.score = winning_score;
    second_best.score = second_score;
    best.path = std::move(winning_left);
    add_to_path(best.path, winning_middle);
    add_to_path(best.path, winning_right);
    best.identity = path_identity(best.path);
    second_best.path = std::move(second_left);
    add_to_path(second_best.path, second_middle);
    add_to_path(second_best.path, second_right);
    second_best.identity = path_identity(second_best.path);
}

} // namespace oracle

// C entry for the stage-level parity tests of the pinned X-drop aligner: one tree.
// tree_parent[i] (-1 for the root) / tree_node[i] oriented nodes in DFS visit order.
// Output: score; mappings in TREE space (node = tree index + 1) packed like gb_alignment.
extern "C" int oracle_xdrop_pinned(const gb_flat_index* ix, const gb_scores* scores,
                                   const int32_t* tree_parent, const uint32_t* tree_node, uint32_t n_tree, uint32_t root_trim,
                                   const uint8_t* query, uint32_t qlen, uint32_t max_gap,
                                   int32_t* score_out, gb_mapping* mappings, uint32_t mapping_cap, uint32_t* n_mappings,
                                   uint32_t* edits, uint32_t edit_cap, uint32_t* n_edits) {
    oracle::Graph g(ix);
    oracle::TailTree t; t.root_trim = root_trim;
    for (uint32_t i = 0; i < n_tree; i++) t.nodes.emplace_back((int64_t)tree_parent[i], tree_node[i]);
    oracle::PinnedAlignment a = oracle::xdrop_pinned(g, *scores, t, std::string((const char*)query, qlen), max_gap);
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
