// ORACLE — TEST INFRASTRUCTURE ONLY.  Haplotype-consistent gap-affine wavefront alignment:
//   WFAExtender::connect / prefix / suffix      gbwt_extender.cpp:2052-2263
//   WFATree                                     gbwt_extender.cpp:1567-2046
//   WFANode                                     gbwt_extender.cpp:1434-1557
//   MatchPos, WFAPoint                          gbwt_extender.cpp:1262-1420
//   WFAAlignment::append / flip / final_offset  gbwt_extender.cpp:821-860
//   ErrorModel                                  gbwt_extender.hpp:340-385
// Everything here is vg's own code path (no absent dependency besides the GBWT search state, which
// oracle/gbwt_view.hpp restates), so parity is pinned by the reference's unit vectors
// (src/unittest/gbwt_extender.cpp:1531-2650 -> tests/golden/wfa.json).  One point is NOT pinned:
// WFATree::trim (best partial alignment when nothing full-length fits the score bound) scans
// hash maps in unspecified order (gbwt_extender.cpp:1880 "TODO: Does iteration order matter?");
// here wavefronts are ordered maps, so ties go to the smallest (tree node, score, diagonal).
#include "tail_align.hpp"
#include <climits>
#include <map>

namespace oracle {
namespace wfa {

enum EditOp : uint32_t { MATCH = 0, MISMATCH = 1, INSERTION = 2, DELETION = 3 };
constexpr uint32_t NO_TARGET = 0xffffffffu;

struct ErrorEvent { double per_base; int32_t min, max; int32_t evaluate(size_t length) const { return std::min(max, (int32_t)(per_base * length) + min); } };
struct ErrorModel { ErrorEvent mismatches, gaps, gap_length, distance; };

struct Pos {
    uint32_t seq_offset = 0, node_offset = 0;
    std::vector<uint32_t> path;              // tree offsets from a leaf (front) to the relevant node (back)
    bool empty() const { return path.empty(); }
    bool at_last_node() const { return path.size() == 1; }
    uint32_t node() const { return path.back(); }
    void pop() { path.pop_back(); }
    int32_t distance(int32_t diagonal) const { return 2 * (int32_t)seq_offset - diagonal; }
};
// MatchPos::operator< : positions are ordered by sequence offsets, empty ones first
static inline bool pos_less(const Pos& a, const Pos& b) {
    if (a.empty()) return !b.empty();
    if (b.empty()) return false;
    return a.seq_offset < b.seq_offset;
}

struct Point {
    int32_t score, diagonal; uint32_t seq_offset, node_offset;
    int32_t target_offset() const { return (int32_t)seq_offset - diagonal; }
    int32_t alignment_score(int32_t match, uint32_t final_insertion = 0) const {
        return (match * ((int32_t)(seq_offset + final_insertion) + target_offset()) - score) / 2;
    }
};

struct Node {
    std::vector<uint32_t> path;              // oriented graph nodes
    SearchState state;
    std::string seq;
    uint32_t parent = 0;
    std::vector<uint32_t> children;
    uint32_t target_offset = NO_TARGET;
    bool dead_end = false;
    std::map<std::pair<int32_t, int32_t>, std::pair<uint32_t, uint32_t>> wf[3];   // MATCHES, INSERTIONS, DELETIONS
    size_t length() const { return seq.size(); }
    bool is_leaf() const { return children.empty() || dead_end; }
    bool expanded() const { return !children.empty() || dead_end; }
};
constexpr size_t TARGET_LENGTH = 1024;
enum { MATCHES = 0, INSERTIONS = 1, DELETIONS = 2 };

struct Tree {
    const Graph& graph; const std::string& sequence;
    uint32_t to_node; uint32_t to_offset; bool has_to;
    std::vector<Node> nodes;
    Point candidate_point{INT_MAX, 0, 0, 0}; uint32_t candidate_node = 0;
    int32_t mismatch, gap_open, gap_extend, score_bound = 0, max_distance = 0, min_distance = 0;
    struct ScoreProperties { int32_t min_diagonal, max_diagonal; bool reachable_with_gap; };
    std::map<int32_t, ScoreProperties> possible_scores;
    // what gb_wfa_batch's fixed per-problem workspace would have needed (oracle_wfa_workspace)
    uint32_t max_successors = 0; int32_t max_point_score = 0, min_point_diagonal = 0, max_point_diagonal = 0;
    uint32_t max_point_seq_offset = 0, max_point_node_offset = 0;

    // WFANode::append_node
    bool append_node(Node& n, const SearchState& next) {
        n.state = next;
        n.path.push_back(next.node);
        std::string_view view = graph.get_sequence_view(next.node);
        n.seq.append(view.data(), view.size());
        if (has_to && to_node == next.node) { n.target_offset = (uint32_t)(n.seq.length() - (view.size() - to_offset)); return true; }
        return false;
    }
    // WFANode constructor
    Node make_node(const SearchState& state, uint32_t parent) {
        Node n; n.parent = parent;
        if (append_node(n, state)) return n;
        while (n.seq.length() < TARGET_LENGTH) {
            size_t successors = 0; SearchState next_state;
            graph.follow_paths(n.state, [&](const SearchState& next) { successors++; next_state = next; return true; });
            if (successors == 0) { n.dead_end = true; break; }
            else if (successors > 1) break;
            if (append_node(n, next_state)) break;
        }
        return n;
    }

    Tree(const Graph& g, const std::string& seq, uint32_t from_node, uint32_t from_offset, bool has_to_, uint32_t to_node_, uint32_t to_offset_,
         const gb_scores& sc, const ErrorModel& em)
        : graph(g), sequence(seq), to_node(to_node_), to_offset(to_offset_), has_to(has_to_),
          mismatch(2 * (sc.match + sc.mismatch)), gap_open(2 * (sc.gap_open - sc.gap_extend)), gap_extend(2 * sc.gap_extend + sc.match) {
        SearchState st; st.node = from_node; st.lo = 0; st.hi = (int64_t)g.record_size(from_node) - 1;
        nodes.push_back(make_node(st, 0));
        update(nodes[0], MATCHES, 0, 0, 0u, from_offset + 1);
        const int32_t max_mismatches = em.mismatches.evaluate(seq.length());
        const int32_t max_gaps = em.gaps.evaluate(seq.length());
        const int32_t max_gap_length = em.gap_length.evaluate(seq.length());
        score_bound = max_mismatches * mismatch + max_gaps * gap_open + max_gap_length * gap_extend;
        possible_scores[0] = {0, 0, false};
    }

    uint32_t size() const { return (uint32_t)nodes.size(); }
    int32_t gap_extend_penalty(uint32_t length) const { return (int32_t)length * gap_extend; }
    int32_t gap_penalty(uint32_t length) const { return gap_open + gap_extend_penalty(length); }

    void update(Node& n, int type, int32_t score, int32_t diagonal, uint32_t seq_offset, uint32_t node_offset) {
        n.wf[type][{score, diagonal}] = {seq_offset, node_offset};
        max_point_score = std::max(max_point_score, score);
        min_point_diagonal = std::min(min_point_diagonal, diagonal); max_point_diagonal = std::max(max_point_diagonal, diagonal);
        max_point_seq_offset = std::max(max_point_seq_offset, seq_offset); max_point_node_offset = std::max(max_point_node_offset, node_offset);
    }
    void update(int type, int32_t score, int32_t diagonal, const Pos& p) { update(nodes[p.node()], type, score, diagonal, p.seq_offset, p.node_offset); }

    std::vector<uint32_t> get_leaves() const { std::vector<uint32_t> l; for (uint32_t i = 0; i < size(); i++) if (nodes[i].is_leaf()) l.push_back(i); return l; }
    bool at_dead_end(const Pos& p) const { return nodes[p.node()].dead_end && p.node_offset >= nodes[p.node()].length(); }

    // WFATree::find_pos
    Pos find_pos(int type, uint32_t node, int32_t score, int32_t diagonal, bool extendable_seq, bool extendable_graph) const {
        if (score < 0) return Pos();
        std::vector<uint32_t> path;
        while (true) {
            path.push_back(node);
            auto it = nodes[node].wf[type].find({score, diagonal});
            if (it != nodes[node].wf[type].end()) {
                Pos p; p.seq_offset = it->second.first; p.node_offset = it->second.second; p.path = path;
                if (extendable_seq && p.seq_offset >= sequence.length()) return Pos();
                if (extendable_graph && at_dead_end(p)) return Pos();
                return p;
            }
            if (node == 0) return Pos();
            node = nodes[node].parent;
        }
    }

    void expand_if_necessary(const Pos& pos) {
        const uint32_t node = pos.node();
        if (nodes[node].expanded() || pos.node_offset < nodes[node].length()) return;
        bool found = false;
        std::vector<SearchState> kids;
        graph.follow_paths(nodes[node].state, [&](const SearchState& child) -> bool { kids.push_back(child); return true; });
        max_successors = std::max(max_successors, (uint32_t)kids.size());
        for (const SearchState& child : kids) {
            nodes[node].children.push_back(size());
            Node n = make_node(child, node);
            nodes.push_back(std::move(n));
            found = true;
        }
        if (!found) nodes[node].dead_end = true;
    }

    void successor_offset(Pos& pos) const {
        if (pos.node_offset >= nodes[pos.node()].length()) { pos.pop(); pos.node_offset = 0; }
        pos.node_offset++;
    }
    void predecessor_offset(uint32_t& node, uint32_t& offset) const {
        if (offset > 0) offset--;
        else { node = nodes[node].parent; offset = (uint32_t)nodes[node].length() - 1; }
    }

    void match_forward(const Node& n, Pos& pos) const {
        while (pos.seq_offset < sequence.length() && pos.node_offset < n.seq.length() && sequence[pos.seq_offset] == n.seq[pos.node_offset]) { pos.seq_offset++; pos.node_offset++; }
    }

    // wf_extend
    void extend_over(int32_t score, int32_t diagonal, const std::vector<uint32_t>& leaves) {
        for (uint32_t leaf : leaves) {
            Pos pos = find_pos(MATCHES, leaf, score, diagonal, false, false);
            if (pos.empty()) continue;
            while (true) {
                const uint32_t ni = pos.node();
                bool may_reach_target = nodes[ni].target_offset != NO_TARGET && nodes[ni].target_offset >= pos.node_offset && nodes[ni].target_offset < nodes[ni].length();
                match_forward(nodes[ni], pos);
                if ((may_reach_target && pos.node_offset >= nodes[ni].target_offset) || (!has_to && pos.seq_offset >= sequence.length())) {
                    const uint32_t overshoot = !has_to ? 0u : pos.node_offset - nodes[ni].target_offset;
                    const uint32_t gap_length = (uint32_t)(sequence.length() - pos.seq_offset) + overshoot;
                    int32_t gap_score = 0;
                    if (gap_length > 0) gap_score = gap_penalty(gap_length);
                    if (score + gap_score < candidate_point.score) {
                        candidate_point = {score + gap_score, diagonal, pos.seq_offset - overshoot, nodes[ni].target_offset};
                        candidate_node = ni;
                    }
                }
                max_distance = std::max(max_distance, pos.distance(diagonal));
                update(MATCHES, score, diagonal, pos);
                if (pos.node_offset < nodes[ni].length()) break;
                expand_if_necessary(pos);
                if (pos.at_last_node()) {
                    std::vector<uint32_t> new_leaves = nodes[pos.node()].children;
                    extend_over(score, diagonal, new_leaves);
                    break;
                }
                pos.pop(); pos.node_offset = 0;
            }
        }
    }
    void extend(int32_t score) {
        auto it = possible_scores.find(score);
        if (it == possible_scores.end()) return;
        const int32_t lo = it->second.min_diagonal, hi = it->second.max_diagonal;
        for (int32_t diagonal = lo; diagonal <= hi; diagonal++) { std::vector<uint32_t> leaves = get_leaves(); extend_over(score, diagonal, leaves); }
    }

    int32_t next_score(int32_t match_score) {
        const int32_t mismatch_score = match_score + mismatch;
        if (possible_scores.find(mismatch_score) == possible_scores.end()) possible_scores[mismatch_score] = {0, 0, false};
        auto match_iter = possible_scores.find(match_score);
        if (match_iter->second.reachable_with_gap) {
            const int32_t extend_score = match_score + gap_extend;
            auto e = possible_scores.find(extend_score);
            if (e != possible_scores.end()) e->second.reachable_with_gap = true; else possible_scores[extend_score] = {0, 0, true};
        }
        const int32_t open_score = match_score + gap_open + gap_extend;
        auto o = possible_scores.find(open_score);
        if (o != possible_scores.end()) o->second.reachable_with_gap = true; else possible_scores[open_score] = {0, 0, true};
        match_iter = possible_scores.find(match_score);
        ++match_iter;
        return match_iter->first;
    }

    std::pair<int32_t, int32_t> update_diagonal_range(std::pair<int32_t, int32_t> range, int32_t score) const {
        if (score >= 0) {
            auto it = possible_scores.find(score);
            if (it != possible_scores.end()) { range.first = std::min(range.first, it->second.min_diagonal); range.second = std::max(range.second, it->second.max_diagonal); }
        }
        return range;
    }
    std::pair<int32_t, int32_t> get_diagonals(int32_t score) const {
        std::pair<int32_t, int32_t> range{INT_MAX, INT_MIN};
        range = update_diagonal_range(range, score - mismatch);
        range = update_diagonal_range(range, score - gap_open - gap_extend);
        range = update_diagonal_range(range, score - gap_extend);
        if (range.first > range.second) return range;
        range.first--; range.second++;
        return range;
    }

    std::pair<Pos, EditOp> ins_predecessor(uint32_t node, int32_t score, int32_t diagonal) const {
        Pos open = find_pos(MATCHES, node, score - gap_open - gap_extend, diagonal - 1, true, false);
        Pos ext = find_pos(INSERTIONS, node, score - gap_extend, diagonal - 1, true, false);
        return pos_less(open, ext) ? std::make_pair(ext, INSERTION) : std::make_pair(open, MATCH);
    }
    std::pair<Pos, EditOp> del_predecessor(uint32_t node, int32_t score, int32_t diagonal) const {
        Pos open = find_pos(MATCHES, node, score - gap_open - gap_extend, diagonal + 1, false, true);
        Pos ext = find_pos(DELETIONS, node, score - gap_extend, diagonal + 1, false, true);
        return pos_less(open, ext) ? std::make_pair(ext, DELETION) : std::make_pair(open, MATCH);
    }
    std::pair<Pos, EditOp> match_predecessor(uint32_t node, int32_t score, int32_t diagonal) const {
        Pos ins = find_pos(INSERTIONS, node, score, diagonal, false, false);
        Pos del = find_pos(DELETIONS, node, score, diagonal, false, false);
        Pos subst = find_pos(MATCHES, node, score - mismatch, diagonal, false, false);
        if (!subst.empty()) { subst.seq_offset++; subst.node_offset++; }
        if (pos_less(ins, del)) return pos_less(del, subst) ? std::make_pair(subst, MISMATCH) : std::make_pair(del, DELETION);
        else return pos_less(ins, subst) ? std::make_pair(subst, MISMATCH) : std::make_pair(ins, INSERTION);
    }

    // wf_next
    void next(int32_t score) {
        const std::pair<int32_t, int32_t> diagonal_range = get_diagonals(score);
        std::pair<int32_t, int32_t> actual_range{INT_MAX, INT_MIN};
        auto adjust = [&](int32_t d) { actual_range.first = std::min(actual_range.first, d); actual_range.second = std::max(actual_range.second, d); };
        for (int64_t diagonal64 = diagonal_range.first; diagonal64 <= (int64_t)diagonal_range.second; diagonal64++) {
            const int32_t diagonal = (int32_t)diagonal64;
            std::vector<uint32_t> leaves = get_leaves();
            for (uint32_t leaf : leaves) {
                Pos ins = ins_predecessor(leaf, score, diagonal).first;
                if (!ins.empty()) {
                    ins.seq_offset++;
                    if (ins.distance(diagonal) >= min_distance) { update(INSERTIONS, score, diagonal, ins); adjust(diagonal); }
                }
                Pos del = del_predecessor(leaf, score, diagonal).first;
                if (!del.empty()) {
                    successor_offset(del);
                    if (del.distance(diagonal) >= min_distance) { update(DELETIONS, score, diagonal, del); adjust(diagonal); }
                    expand_if_necessary(del);
                }
                Pos subst = find_pos(MATCHES, leaf, score - mismatch, diagonal, true, true);
                if (!subst.empty()) { subst.seq_offset++; successor_offset(subst); expand_if_necessary(subst); }
                if (pos_less(subst, ins)) subst = std::move(ins);
                if (pos_less(subst, del)) subst = std::move(del);
                if (!subst.empty()) {
                    const uint32_t ni = subst.node();
                    if (subst.node_offset == nodes[ni].target_offset) {
                        const uint32_t gap_length = (uint32_t)(sequence.length() - subst.seq_offset);
                        int32_t gap_score = 0;
                        if (gap_length > 0) gap_score = gap_penalty(gap_length);
                        if (score + gap_score < candidate_point.score) { candidate_point = {score + gap_score, diagonal, subst.seq_offset, subst.node_offset}; candidate_node = ni; }
                    }
                    if (subst.distance(diagonal) >= min_distance) { update(MATCHES, score, diagonal, subst); adjust(diagonal); }
                }
            }
            if (diagonal == INT_MAX) break;
        }
        auto it = possible_scores.find(score);
        if (it != possible_scores.end()) { it->second.min_diagonal = actual_range.first; it->second.max_diagonal = actual_range.second; }
    }

    void trim(int32_t match) {
        candidate_point = {0, 0, 0, 0}; candidate_node = 0;
        int32_t best_score = 0;
        for (uint32_t node = 0; node < size(); node++) {
            for (const auto& entry : nodes[node].wf[MATCHES]) {
                Point point{entry.first.first, entry.first.second, entry.second.first, entry.second.second};
                const int32_t alignment_score = point.alignment_score(match);
                if (alignment_score > best_score) { candidate_point = point; candidate_node = node; best_score = alignment_score; }
            }
        }
    }
};

struct Alignment {
    std::vector<uint32_t> path;                          // oriented graph nodes
    std::vector<std::pair<EditOp, uint32_t>> edits;
    uint32_t node_offset = 0, seq_offset = 0, length = 0;
    int32_t score = 0;
    bool ok = false;
    void append(EditOp e, uint32_t len) { if (len == 0) return; if (edits.empty() || edits.back().first != e) edits.push_back({e, len}); else edits.back().second += len; }
    int64_t final_offset(const Graph& g) const {
        int64_t fo = node_offset;
        for (auto& e : edits) if (e.first != INSERTION) fo += e.second;
        for (size_t i = 0; i + 1 < path.size(); i++) fo -= g.get_length(path[i]);
        return fo;
    }
    void flip(const Graph& g, size_t seq_len) {
        seq_offset = (uint32_t)(seq_len - seq_offset - length);
        if (path.empty()) return;
        node_offset = (uint32_t)(g.get_length(path.back()) - final_offset(g));
        std::reverse(path.begin(), path.end());
        for (auto& h : path) h ^= 1u;
        std::reverse(edits.begin(), edits.end());
    }
};

static void mask(std::string& s) { for (char& c : s) if (c != 'A' && c != 'C' && c != 'G' && c != 'T') c = 'X'; }

// What one problem needs of gb_wfa_batch's per-problem workspace, measured when the wavefront loop stops (the kernel
// follows the same trajectory, so these are the maxima it meets).  Order of the fields: oracle_wfa_workspace.
struct Workspace {
    uint32_t trie_nodes = 0, seq_bytes = 0, path_entries = 0, points = 0, scores = 0;
    int32_t max_score = 0, min_diagonal = 0, max_diagonal = 0;
    uint32_t max_seq_offset = 0, max_node_offset = 0, max_successors = 0;
};
static void report(const Tree& t, Workspace& w) {
    w.trie_nodes = t.size();
    for (const Node& n : t.nodes) {
        w.seq_bytes += (uint32_t)n.seq.size(); w.path_entries += (uint32_t)n.path.size();
        for (int k = 0; k < 3; k++) w.points += (uint32_t)n.wf[k].size();
    }
    w.scores = (uint32_t)t.possible_scores.size();
    w.max_score = t.max_point_score; w.min_diagonal = t.min_point_diagonal; w.max_diagonal = t.max_point_diagonal;
    w.max_seq_offset = t.max_point_seq_offset; w.max_node_offset = t.max_point_node_offset; w.max_successors = t.max_successors;
}

// WFAExtender::connect (to_node == 0: no destination)
Alignment connect(const Graph& g, const gb_scores& sc, const ErrorModel& em, std::string sequence,
                  uint32_t from_node, uint32_t from_offset, uint32_t to_node, uint32_t to_offset, Workspace* ws = nullptr) {
    Alignment fail;
    if (!g.has_node(from_node)) return fail;
    mask(sequence);
    const bool has_to = to_node != 0;
    Tree tree(g, sequence, from_node, from_offset, has_to, to_node, to_offset, sc, em);
    int32_t score = 0;
    while (true) {
        tree.extend(score);
        const int32_t distance_band = em.distance.evaluate(sequence.length());
        if (distance_band < tree.max_distance) tree.min_distance = tree.max_distance - distance_band;
        if (tree.candidate_point.score <= score) break;
        score = tree.next_score(score);
        if (score > tree.score_bound) break;
        tree.next(score);
    }
    if (ws) report(tree, *ws);
    bool full_length = true;
    uint32_t unaligned_tail = (uint32_t)(sequence.length() - tree.candidate_point.seq_offset);
    if (tree.candidate_point.score > tree.score_bound) {
        unaligned_tail = 0;
        if (!has_to) { tree.trim(sc.match); full_length = false; }
        else return fail;
    }
    (void)full_length;
    Alignment result;
    result.node_offset = from_offset + 1; result.seq_offset = 0;
    result.length = tree.candidate_point.seq_offset + unaligned_tail;
    result.score = tree.candidate_point.alignment_score(sc.match, unaligned_tail);
    result.ok = true;
    uint32_t node = tree.candidate_node;
    while (true) {
        for (auto it = tree.nodes[node].path.rbegin(); it != tree.nodes[node].path.rend(); ++it) result.path.push_back(*it);
        if (node == 0) break;
        node = tree.nodes[node].parent;
    }
    std::reverse(result.path.begin(), result.path.end());
    Point point = tree.candidate_point;
    node = tree.candidate_node;
    if (unaligned_tail > 0) {
        const uint32_t final_insertion = (uint32_t)(sequence.length() - tree.candidate_point.seq_offset);
        result.append(INSERTION, final_insertion);
        point.score -= tree.gap_penalty(unaligned_tail);
    }
    EditOp edit = MATCH;
    while (point.seq_offset > 0 || point.diagonal != 0) {
        std::pair<Pos, EditOp> predecessor;
        switch (edit) {
        case MATCH:
            predecessor = tree.match_predecessor(node, point.score, point.diagonal);
            result.append(MATCH, point.seq_offset - predecessor.first.seq_offset);
            point.seq_offset = predecessor.first.seq_offset;
            point.node_offset = predecessor.first.node_offset;
            if (!predecessor.first.empty()) node = predecessor.first.node();
            edit = predecessor.second;
            break;
        case MISMATCH:
            result.append(MISMATCH, 1);
            point.seq_offset--;
            tree.predecessor_offset(node, point.node_offset);
            point.score -= tree.mismatch;
            edit = MATCH;
            break;
        case INSERTION:
            predecessor = tree.ins_predecessor(node, point.score, point.diagonal);
            result.append(INSERTION, 1);
            point.seq_offset--;
            if (predecessor.second == INSERTION) point.score -= tree.gap_extend; else point.score -= tree.gap_open + tree.gap_extend;
            point.diagonal--;
            edit = predecessor.second;
            break;
        case DELETION:
            predecessor = tree.del_predecessor(node, point.score, point.diagonal);
            result.append(DELETION, 1);
            tree.predecessor_offset(node, point.node_offset);
            if (predecessor.second == DELETION) point.score -= tree.gap_extend; else point.score -= tree.gap_open + tree.gap_extend;
            point.diagonal++;
            edit = predecessor.second;
            break;
        }
    }
    std::reverse(result.edits.begin(), result.edits.end());
    if (!result.path.empty() && result.node_offset >= g.get_length(result.path.front())) { result.path.erase(result.path.begin()); result.node_offset = 0; }
    int64_t final_offset = result.final_offset(g);
    while ((result.path.size() == 1 && final_offset == (int64_t)result.node_offset) || (result.path.size() > 1 && final_offset <= 0)) {
        result.path.pop_back();
        if (!result.path.empty()) final_offset += g.get_length(result.path.back());
    }
    return result;
}

Alignment suffix(const Graph& g, const gb_scores& sc, const ErrorModel& em, const std::string& sequence, uint32_t from_node, uint32_t from_offset,
                 Workspace* ws = nullptr) {
    Alignment r = connect(g, sc, em, sequence, from_node, from_offset, 0, 0, ws);
    if (!r.edits.empty() && r.length == sequence.length() && (r.edits.back().first == MATCH || r.edits.back().first == MISMATCH)) r.score += sc.full_length_bonus;
    return r;
}

static std::string revcomp(const std::string& s) {
    std::string r(s.rbegin(), s.rend());
    for (char& c : r) { switch (c) { case 'A': c = 'T'; break; case 'C': c = 'G'; break; case 'G': c = 'C'; break; case 'T': c = 'A'; break; default: c = 'N'; } }
    return r;
}

Alignment prefix(const Graph& g, const gb_scores& sc, const ErrorModel& em, const std::string& sequence, uint32_t to_node, uint32_t to_offset,
                 Workspace* ws = nullptr) {
    if (!g.has_node(to_node)) return Alignment();
    // reverse_base_pos: the same base on the other strand
    const uint32_t rnode = to_node ^ 1u, roff = g.get_length(to_node) - 1 - to_offset;
    Alignment r = connect(g, sc, em, revcomp(sequence), rnode, roff, 0, 0, ws);
    r.flip(g, sequence.length());
    if (!r.edits.empty() && r.length == sequence.length() && (r.edits.front().first == MATCH || r.edits.front().first == MISMATCH)) r.score += sc.full_length_bonus;
    return r;
}

} // namespace wfa
} // namespace oracle

// C entry.  mode: 0 connect(from, to), 1 suffix(from), 2 prefix(to).  Positions are (oriented node,
// offset); error_model = 12 numbers {per_base, min, max} x {mismatches, gaps, gap_length, distance}
// (nullptr: WFAExtender::ErrorModel defaults, gbwt_extender.hpp:372-381).
// Output: ok flag, score, node_offset, seq_offset, length, path (oriented nodes), edits as (length << 2) | op.
static oracle::wfa::Alignment run_wfa(const oracle::Graph& g, const gb_scores* scores, const double* error_model, int mode,
                                      const uint8_t* seq, uint32_t seq_len, uint32_t from_node, uint32_t from_offset, uint32_t to_node, uint32_t to_offset,
                                      oracle::wfa::Workspace* ws) {
    using namespace oracle::wfa;
    ErrorModel em{{0.03, 1, 6}, {0.05, 1, 10}, {0.1, 1, 20}, {0.1, 10, 200}};
    if (error_model) {
        const double* e = error_model;
        em = ErrorModel{{e[0], (int32_t)e[1], (int32_t)e[2]}, {e[3], (int32_t)e[4], (int32_t)e[5]}, {e[6], (int32_t)e[7], (int32_t)e[8]}, {e[9], (int32_t)e[10], (int32_t)e[11]}};
    }
    const std::string s((const char*)seq, seq_len);
    if (mode == 0) return connect(g, *scores, em, s, from_node, from_offset, to_node, to_offset, ws);
    if (mode == 1) return suffix(g, *scores, em, s, from_node, from_offset, ws);
    return prefix(g, *scores, em, s, to_node, to_offset, ws);
}

// C entry.  mode: 0 connect(from, to), 1 suffix(from), 2 prefix(to).  Positions are (oriented node,
// offset); error_model = 12 numbers {per_base, min, max} x {mismatches, gaps, gap_length, distance}
// (nullptr: WFAExtender::ErrorModel defaults, gbwt_extender.hpp:372-381).
// Output: ok flag, score, node_offset, seq_offset, length, path (oriented nodes), edits as (length << 2) | op.
extern "C" int oracle_wfa(const gb_flat_index* ix, const gb_scores* scores, const double* error_model, int mode,
                          const uint8_t* seq, uint32_t seq_len, uint32_t from_node, uint32_t from_offset, uint32_t to_node, uint32_t to_offset,
                          int32_t* ok, int32_t* score, uint32_t* node_offset, uint32_t* seq_offset, uint32_t* length,
                          uint32_t* path, uint32_t path_cap, uint32_t* n_path, uint32_t* edits, uint32_t edit_cap, uint32_t* n_edits) {
    oracle::Graph g(ix);
    const oracle::wfa::Alignment a = run_wfa(g, scores, error_model, mode, seq, seq_len, from_node, from_offset, to_node, to_offset, nullptr);
    *ok = a.ok ? 1 : 0; *score = a.score; *node_offset = a.node_offset; *seq_offset = a.seq_offset; *length = a.length;
    if (a.path.size() > path_cap || a.edits.size() > edit_cap) return -1;
    for (size_t i = 0; i < a.path.size(); i++) path[i] = a.path[i];
    for (size_t i = 0; i < a.edits.size(); i++) edits[i] = (a.edits[i].second << 2) | (uint32_t)a.edits[i].first;
    *n_path = (uint32_t)a.path.size(); *n_edits = (uint32_t)a.edits.size();
    return 0;
}

// The same problem as oracle_wfa, reporting what gb_wfa_batch's per-problem workspace needs for it.  out[11]:
// trie nodes, sequence bytes, path entries, wavefront points (all matrices and trie nodes), distinct possible scores,
// largest point score, smallest and largest point diagonal, largest point seq offset and node offset, most successors
// met in one expansion.  All zero when the start position is not in the graph (nothing is aligned).
extern "C" void oracle_wfa_workspace(const gb_flat_index* ix, const gb_scores* scores, const double* error_model, int mode,
                                     const uint8_t* seq, uint32_t seq_len, uint32_t from_node, uint32_t from_offset, uint32_t to_node, uint32_t to_offset,
                                     int32_t* out) {
    oracle::Graph g(ix);
    oracle::wfa::Workspace w;
    run_wfa(g, scores, error_model, mode, seq, seq_len, from_node, from_offset, to_node, to_offset, &w);
    const int32_t v[11] = {(int32_t)w.trie_nodes, (int32_t)w.seq_bytes, (int32_t)w.path_entries, (int32_t)w.points, (int32_t)w.scores,
                           w.max_score, w.min_diagonal, w.max_diagonal, (int32_t)w.max_seq_offset, (int32_t)w.max_node_offset, (int32_t)w.max_successors};
    for (int i = 0; i < 11; i++) out[i] = v[i];
}
