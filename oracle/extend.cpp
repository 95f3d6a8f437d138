// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/README.md).  CPU restatement of
// vg::GaplessExtender::extend and its helpers, src/gbwt_extender.cpp:186-737 @ fd49b9a9.
// Pinned by the reference's own unit vectors (src/unittest/gbwt_extender.cpp:868-1156),
// transcribed in tests/golden/gapless_extender.json.
//
// Canonicalisation of the two determinism hazards of the reference:
//   * the reference iterates an unordered hash set of seeds (gbwt_extender.cpp:550);
//     here seeds are visited in ascending (node, diag) order;
//   * std::sort with ties in handle_full_length (gbwt_extender.cpp:302) is replaced by a
//     stable sort (ties keep seed order).
#include "oracle.h"
#include "gbwt_view.hpp"
#include "extension.hpp"

#include <algorithm>
#include <cstring>
#include <limits>
#include <queue>
#include <set>
#include <string>

namespace oracle {

namespace {

// gbwt_extender.cpp:201-209
void set_score(GaplessExtension& e, const gb_scores& s) {
    e.score = (int32_t)((e.read_interval.second - e.read_interval.first) * s.match);
    e.score -= (int32_t)(e.internal_score * (s.match + s.mismatch));
    e.score += (int32_t)(e.left_full * s.full_length_bonus);
    e.score += (int32_t)(e.right_full * s.full_length_bonus);
}

// gbwt_extender.cpp:213-236 (byte-wise; the reference's 8-byte blocks count the same mismatches)
void match_initial(GaplessExtension& m, const std::string& seq, std::string_view target) {
    size_t node_offset = m.offset;
    size_t left = std::min(seq.length() - m.read_interval.second, target.size() - node_offset);
    while (left > 0) {
        if (seq[m.read_interval.second] != target[node_offset]) m.internal_score++;
        m.read_interval.second++; node_offset++; left--;
    }
    m.old_score = m.internal_score;
}

// gbwt_extender.cpp:241-267
size_t match_forward(GaplessExtension& m, const std::string& seq, std::string_view target, uint32_t mismatch_limit) {
    size_t node_offset = 0;
    size_t left = std::min(seq.length() - m.read_interval.second, target.size() - node_offset);
    while (left > 0) {
        if (seq[m.read_interval.second] != target[node_offset]) {
            if (m.internal_score + 1 >= mismatch_limit) return node_offset;
            m.internal_score++;
        }
        m.read_interval.second++; node_offset++; left--;
    }
    return node_offset;
}

// gbwt_extender.cpp:272-296
void match_backward(GaplessExtension& m, const std::string& seq, std::string_view target, uint32_t mismatch_limit) {
    size_t left = std::min(m.read_interval.first, m.offset);
    while (left > 0) {
        if (seq[m.read_interval.first - 1] != target[m.offset - 1]) {
            if (m.internal_score + 1 >= mismatch_limit) return;
            m.internal_score++;
        }
        m.read_interval.first--; m.offset--; left--;
    }
}

// gbwt_extender.cpp:301-329 (stable sort: canonical tie order)
void handle_full_length(const Graph& g, std::vector<GaplessExtension>& result, double overlap_threshold) {
    std::stable_sort(result.begin(), result.end(), [](const GaplessExtension& a, const GaplessExtension& b) {
        if (a.full() && b.full()) return a.internal_score < b.internal_score;
        return a.full() && !b.full();
    });
    size_t tail = 0;
    for (size_t i = 0; i < result.size(); i++) {
        if (!result[i].full()) break;
        bool overlap = false;
        for (size_t prev = 0; prev < tail; prev++) {
            if (result[i].overlap(g, result[prev]) > overlap_threshold * result[prev].length()) { overlap = true; break; }
        }
        if (overlap) continue;
        if (i > tail) result[tail] = std::move(result[i]);
        tail++;
    }
    result.resize(tail);
}

// gbwt_extender.cpp:332-365
void remove_duplicates(std::vector<GaplessExtension>& result) {
    auto sort_order = [](const GaplessExtension& a, const GaplessExtension& b) {
        if (a.read_interval != b.read_interval) return a.read_interval < b.read_interval;
        if (a.state.backward.node != b.state.backward.node) return a.state.backward.node < b.state.backward.node;
        if (a.state.forward.node != b.state.forward.node) return a.state.forward.node < b.state.forward.node;
        auto abr = std::make_pair(a.state.backward.lo, a.state.backward.hi), bbr = std::make_pair(b.state.backward.lo, b.state.backward.hi);
        if (abr != bbr) return abr < bbr;
        auto afr = std::make_pair(a.state.forward.lo, a.state.forward.hi), bfr = std::make_pair(b.state.forward.lo, b.state.forward.hi);
        if (afr != bfr) return afr < bfr;
        return a.offset < b.offset;
    };
    std::stable_sort(result.begin(), result.end(), sort_order);
    size_t tail = 0;
    for (size_t i = 0; i < result.size(); i++) {
        if (result[i].empty()) continue;
        if (tail == 0 || result[i] != result[tail - 1]) {
            if (i > tail) result[tail] = std::move(result[i]);
            tail++;
        }
    }
    result.resize(tail);
}

// gbwt_extender.cpp:368-387
void find_mismatches(const std::string& seq, const Graph& g, std::vector<GaplessExtension>& result) {
    for (GaplessExtension& e : result) {
        if (e.internal_score == 0) continue;
        size_t node_offset = e.offset, read_offset = e.read_interval.first;
        for (uint32_t h : e.path) {
            std::string_view target = g.get_sequence_view(h);
            while (node_offset < target.size() && read_offset < e.read_interval.second) {
                if (target[node_offset] != seq[read_offset]) e.mismatch_positions.push_back(read_offset);
                node_offset++; read_offset++;
            }
            node_offset = 0;
        }
    }
}

size_t interval_length(std::pair<size_t, size_t> iv) { return iv.second - iv.first; }

// gbwt_extender.cpp:421-529
bool trim_mismatches(GaplessExtension& e, const Graph& g, const gb_scores& s) {
    if (e.exact()) return false;
    auto mismatch = e.mismatch_positions.begin();
    std::pair<size_t, size_t> current(e.read_interval.first, *mismatch);
    int32_t current_score = (int32_t)interval_length(current) * s.match;
    if (e.left_full) current_score += s.full_length_bonus;
    std::pair<size_t, size_t> best = current;
    int32_t best_score = current_score;
    while (mismatch != e.mismatch_positions.end()) {
        if (current_score >= s.mismatch) { current.second++; current_score -= s.mismatch; }
        else { current.first = current.second = *mismatch + 1; current_score = 0; }
        ++mismatch;
        if (mismatch == e.mismatch_positions.end()) {
            size_t length = e.read_interval.second - current.second;
            current.second = e.read_interval.second;
            current_score += (int32_t)length * s.match;
            if (e.right_full) current_score += s.full_length_bonus;
        } else {
            size_t length = *mismatch - current.second;
            current.second = *mismatch;
            current_score += (int32_t)length * s.match;
        }
        if (current_score > best_score ||
            (current_score > 0 && current_score == best_score && interval_length(current) > interval_length(best))) {
            best = current; best_score = current_score;
        }
    }
    if (best == e.read_interval) return false;
    if (interval_length(best) == 0) {
        e.path.clear(); e.read_interval = best; e.mismatch_positions.clear();
        e.score = 0; e.left_full = e.right_full = false;
        return true;
    }
    if (best.first > e.read_interval.first) e.left_full = false;
    if (best.second < e.read_interval.second) e.right_full = false;
    size_t node_offset = e.offset, read_offset = e.read_interval.first;
    e.read_interval = best;
    e.score = best_score;
    size_t head = 0;
    while (head < e.path.size()) {
        size_t node_length = g.get_length(e.path[head]);
        read_offset += node_length - node_offset;
        node_offset = 0;
        if (read_offset > e.read_interval.first) {
            e.offset = node_length - (read_offset - e.read_interval.first);
            break;
        }
        head++;
    }
    size_t tail = head + 1;
    while (read_offset < e.read_interval.second) { read_offset += g.get_length(e.path[tail]); tail++; }
    if (head > 0 || tail < e.path.size()) {
        std::vector<uint32_t> sub(e.path.begin() + head, e.path.begin() + tail);
        e.path.swap(sub);
        e.state = g.bd_find(e.path);
    }
    std::vector<size_t> mm;
    for (size_t p : e.mismatch_positions) if (p >= e.read_interval.first && p < e.read_interval.second) mm.push_back(p);
    e.mismatch_positions.swap(mm);
    return true;
}

} // namespace

// What one call asks of the extension kernel's fixed resources (extend.cuh), and the GB_ITEM_* status the capacities
// below give it.  Each capacity is checked where the kernel checks it, so the first one exceeded decides the status:
//   frontier / arena   before every push of the search (extend.cuh extend_search: qn + 1 >= q_cap, an >= a_cap)
//   records / paths    when a seed's best match is added to the result
//   mismatch pool      after the full-length or duplicate filter, before trimming (extend_finish)
struct ExtendTrace {
    uint64_t q_cap = UINT64_MAX, a_cap = UINT64_MAX, max_ext = UINT64_MAX, path_cap = UINT64_MAX, mism_cap = UINT64_MAX;
    int status = GB_ITEM_OK;
    uint64_t records = 0, path_nodes = 0, mismatches = 0, peak_frontier = 0, peak_arena = 0;
    std::set<std::pair<uint32_t, int64_t>> contained, invalid;    // seeds skipped, by reason
    void fail(int s) { if (status == GB_ITEM_OK) status = s; }
};

// gbwt_extender.cpp:533-737.  Seeds the reference would read out of bounds with (a node that is not in the graph or
// is empty, a read offset past the read, a node offset past the node) are skipped, as in extend.cuh.
std::vector<GaplessExtension> extend(const Graph& g, const gb_scores& scores,
                                     const std::vector<std::pair<uint32_t, int64_t>>& cluster_in,
                                     std::string sequence, size_t max_mismatches,
                                     double overlap_threshold, bool trim, ExtendTrace* trace) {
    std::vector<GaplessExtension> result;
    if (cluster_in.empty() || sequence.empty()) return result;
    // ReadMasker("ACGT"), gbwt_extender.cpp:160-170
    for (char& c : sequence) if (c != 'A' && c != 'C' && c != 'G' && c != 'T') c = 'X';
    std::set<std::pair<uint32_t, int64_t>> cluster(cluster_in.begin(), cluster_in.end());
    result.reserve(cluster.size());

    size_t best_alignment = std::numeric_limits<size_t>::max();
    for (auto seed : cluster) {
        {
            const size_t read_offset = seed.second < 0 ? 0 : (size_t)seed.second;
            const size_t node_offset = seed.second < 0 ? (size_t)(-seed.second) : 0;
            if (!g.has_node(seed.first) || read_offset > sequence.length() || node_offset > g.get_length(seed.first)) {
                if (trace) trace->invalid.insert(seed);
                continue;
            }
        }
        if (best_alignment < result.size() && result[best_alignment].internal_score == 0) {
            if (result[best_alignment].contains(g, seed.first, seed.second)) {
                if (trace) trace->contained.insert(seed);
                continue;
            }
        }
        GaplessExtension best_match;
        best_match.score = std::numeric_limits<int32_t>::min();
        best_match.internal_score = std::numeric_limits<uint32_t>::max();
        best_match.old_score = std::numeric_limits<uint32_t>::max();

        typedef std::pair<GaplessExtension, size_t> queue_item;
        auto cmp = [](const queue_item& a, const queue_item& b) {
            // std::pair operator< over (GaplessExtension::operator<, size_t)
            if (a.first.score != b.first.score) return a.first.score < b.first.score;
            return a.second < b.second;
        };
        std::priority_queue<queue_item, std::vector<queue_item>, decltype(cmp)> extensions(cmp);
        size_t extension_number = 0;
        uint64_t arena = 0;              // extensions pushed for this seed: the kernel's parent-pointer arena
        // the kernel's check before pushing a new extension (arena node + frontier entry) or a re-pushed one (entry only)
        auto before_push = [&](bool new_node) {
            if (!trace) return;
            if ((new_node && arena >= trace->a_cap) || extensions.size() + 1 >= trace->q_cap) trace->fail(GB_ITEM_QUEUE_FULL);
            arena += new_node;
            trace->peak_arena = std::max(trace->peak_arena, arena);
            trace->peak_frontier = std::max<uint64_t>(trace->peak_frontier, extensions.size() + 1);
        };
        {
            size_t read_offset = seed.second < 0 ? 0 : (size_t)seed.second;
            size_t node_offset = seed.second < 0 ? (size_t)(-seed.second) : 0;
            GaplessExtension match;
            match.path = {seed.first};
            match.offset = node_offset;
            match.state = g.get_bd_state(seed.first);
            match.read_interval = {read_offset, read_offset};
            match_initial(match, sequence, g.get_sequence_view(seed.first));
            if (match.read_interval.first == 0) { match.left_full = true; match.left_maximal = true; }
            if (match.read_interval.second >= sequence.length()) { match.right_full = true; match.right_maximal = true; }
            set_score(match, scores);
            extensions.emplace(std::move(match), extension_number++);
            if (trace) trace->peak_frontier = std::max<uint64_t>(trace->peak_frontier, 1);
        }
        while (!extensions.empty()) {
            GaplessExtension curr = extensions.top().first;
            extensions.pop();
            if (!curr.right_maximal) {
                size_t num_extensions = 0;
                uint32_t mismatch_limit = std::max<uint32_t>((uint32_t)(max_mismatches + 1),
                                                             (uint32_t)(max_mismatches / 2 + curr.old_score + 1));
                g.follow_paths(curr.state, false, [&](const BidirectionalState& next_state) -> bool {
                    uint32_t handle = next_state.forward.node;
                    GaplessExtension next;
                    next.offset = curr.offset; next.state = next_state;
                    next.read_interval = curr.read_interval;
                    next.score = curr.score; next.left_full = curr.left_full; next.right_full = curr.right_full;
                    next.left_maximal = curr.left_maximal; next.right_maximal = curr.right_maximal;
                    next.internal_score = curr.internal_score; next.old_score = curr.old_score;
                    size_t node_offset = match_forward(next, sequence, g.get_sequence_view(handle), mismatch_limit);
                    if (node_offset == 0) return true;
                    next.path = curr.path; next.path.push_back(handle);
                    if (next.read_interval.second >= sequence.length()) {
                        next.right_full = true; next.right_maximal = true; next.old_score = next.internal_score;
                    } else if (node_offset < g.get_length(handle)) {
                        next.right_maximal = true; next.old_score = next.internal_score;
                    }
                    set_score(next, scores);
                    num_extensions += next.state.size();
                    before_push(true);
                    extensions.emplace(std::move(next), extension_number++);
                    return true;
                });
                if (num_extensions < curr.state.size()) {
                    curr.right_maximal = true;
                    curr.old_score = curr.internal_score;
                    before_push(false);
                    extensions.emplace(std::move(curr), extension_number++);
                }
                continue;
            }
            if (!curr.left_maximal) {
                bool found_extension = false;
                uint32_t mismatch_limit = std::max<uint32_t>((uint32_t)(max_mismatches + 1),
                                                             (uint32_t)(max_mismatches / 2 + curr.old_score + 1));
                g.follow_paths(curr.state, true, [&](const BidirectionalState& next_state) -> bool {
                    uint32_t handle = next_state.backward.node ^ 1u;
                    size_t node_length = g.get_length(handle);
                    GaplessExtension next;
                    next.offset = node_length; next.state = next_state;
                    next.read_interval = curr.read_interval;
                    next.score = curr.score; next.left_full = curr.left_full; next.right_full = curr.right_full;
                    next.left_maximal = curr.left_maximal; next.right_maximal = curr.right_maximal;
                    next.internal_score = curr.internal_score; next.old_score = curr.old_score;
                    match_backward(next, sequence, g.get_sequence_view(handle), mismatch_limit);
                    if (next.offset >= node_length) return true;
                    next.path.push_back(handle);
                    next.path.insert(next.path.end(), curr.path.begin(), curr.path.end());
                    if (next.read_interval.first == 0) { next.left_full = true; next.left_maximal = true; }
                    else if (next.offset > 0) { next.left_maximal = true; }
                    set_score(next, scores);
                    before_push(true);
                    extensions.emplace(std::move(next), extension_number++);
                    found_extension = true;
                    return true;
                });
                if (!found_extension) curr.left_maximal = true;
                else continue;
            }
            if (best_match < curr) best_match = std::move(curr);
        }
        if (!best_match.empty()) {
            if (trace) {
                if (result.size() >= trace->max_ext || trace->path_nodes + best_match.path.size() > trace->path_cap) trace->fail(GB_ITEM_OUT_FULL);
                trace->records++; trace->path_nodes += best_match.path.size();
            }
            if (best_match.full() && (best_alignment >= result.size() ||
                                      best_match.internal_score < result[best_alignment].internal_score)) {
                best_alignment = result.size();
            }
            result.emplace_back(std::move(best_match));
        }
    }

    auto count_mismatches = [&]() {
        if (!trace) return;
        for (const GaplessExtension& e : result) trace->mismatches += e.mismatch_positions.size();
        if (trace->mismatches > trace->mism_cap) trace->fail(GB_ITEM_OUT_FULL);
    };
    if (best_alignment < result.size() && result[best_alignment].internal_score <= max_mismatches) {
        handle_full_length(g, result, overlap_threshold);
        find_mismatches(sequence, g, result);
        count_mismatches();
    } else {
        remove_duplicates(result);
        find_mismatches(sequence, g, result);
        count_mismatches();
        if (trim) {
            bool trimmed = false;
            for (GaplessExtension& e : result) trimmed |= trim_mismatches(e, g, scores);
            if (trimmed) remove_duplicates(result);
        }
    }
    return result;
}

} // namespace oracle

extern "C" int oracle_extend(const gb_flat_index* ix, const gb_scores* scores,
                             const uint8_t* read, uint32_t read_len,
                             const gb_seed* seeds, uint32_t n_seeds,
                             uint32_t max_mismatches, double overlap_threshold, int trim,
                             gb_extension* ext_out, uint32_t max_ext,
                             uint32_t* path_pool, uint32_t path_cap,
                             uint32_t* mism_pool, uint32_t mism_cap) {
    oracle::Graph g(ix);
    std::vector<std::pair<uint32_t, int64_t>> cluster;
    for (uint32_t i = 0; i < n_seeds; i++) cluster.emplace_back(seeds[i].node, (int64_t)seeds[i].diag);
    auto result = oracle::extend(g, *scores, cluster, std::string((const char*)read, read_len),
                                 max_mismatches, overlap_threshold, trim != 0, nullptr);
    if (result.size() > max_ext) return -1;
    uint32_t pp = 0, mp = 0;
    for (size_t i = 0; i < result.size(); i++) {
        const auto& e = result[i];
        if (pp + e.path.size() > path_cap || mp + e.mismatch_positions.size() > mism_cap) return -1;
        gb_extension& o = ext_out[i];
        o.path_off = pp; o.path_len = (uint32_t)e.path.size();
        for (uint32_t h : e.path) path_pool[pp++] = h;
        o.mism_off = mp; o.mism_len = (uint32_t)e.mismatch_positions.size();
        for (size_t p : e.mismatch_positions) mism_pool[mp++] = (uint32_t)p;
        o.offset = (uint32_t)e.offset;
        o.read_lo = (uint32_t)e.read_interval.first; o.read_hi = (uint32_t)e.read_interval.second;
        o.score = e.score;
        o.flags = (e.left_full ? GB_EXT_LEFT_FULL : 0) | (e.right_full ? GB_EXT_RIGHT_FULL : 0);
        o.fwd_node = e.state.forward.node; o.fwd_lo = (uint32_t)e.state.forward.lo; o.fwd_hi = (uint32_t)e.state.forward.hi;
        o.bwd_node = e.state.backward.node; o.bwd_lo = (uint32_t)e.state.backward.lo; o.bwd_hi = (uint32_t)e.state.backward.hi;
        o.mismatches = (uint32_t)e.mismatch_positions.size();
    }
    return (int)result.size();
}

extern "C" int oracle_extend_limits(const gb_flat_index* ix, const gb_scores* scores,
                                    const uint8_t* read, uint32_t read_len,
                                    const gb_seed* seeds, uint32_t n_seeds,
                                    uint32_t max_mismatches, double overlap_threshold, int trim,
                                    uint32_t q_cap, uint32_t a_cap, uint32_t max_ext, uint32_t path_cap, uint32_t mism_cap,
                                    uint64_t* needs_out, uint8_t* seed_skip) {
    oracle::Graph g(ix);
    std::vector<std::pair<uint32_t, int64_t>> cluster;
    for (uint32_t i = 0; i < n_seeds; i++) cluster.emplace_back(seeds[i].node, (int64_t)seeds[i].diag);
    oracle::ExtendTrace t;
    t.q_cap = q_cap; t.a_cap = a_cap; t.max_ext = max_ext; t.path_cap = path_cap; t.mism_cap = mism_cap;
    oracle::extend(g, *scores, cluster, std::string((const char*)read, read_len), max_mismatches, overlap_threshold,
                   trim != 0, &t);
    if (needs_out) {
        needs_out[0] = t.records; needs_out[1] = t.path_nodes; needs_out[2] = t.mismatches;
        needs_out[3] = t.peak_frontier; needs_out[4] = t.peak_arena;
    }
    if (seed_skip) {
        for (uint32_t i = 0; i < n_seeds; i++) {
            const auto s = cluster[i];
            seed_skip[i] = t.invalid.count(s) ? 2 : t.contained.count(s) ? 1 : 0;
        }
    }
    return t.status;
}

// GaplessExtension helpers on hand-built extensions (test entries for unittest/gbwt_extender.cpp:576-820).
static oracle::GaplessExtension make_test_extension(const uint32_t* path, uint32_t n, uint32_t offset, uint32_t read_lo, uint32_t read_hi) {
    oracle::GaplessExtension e;
    e.path.assign(path, path + n); e.offset = offset; e.read_interval = {read_lo, read_hi};
    return e;
}
extern "C" uint64_t oracle_extension_overlap(const gb_flat_index* ix, const uint32_t* path_a, uint32_t n_a, uint32_t offset_a, uint32_t lo_a, uint32_t hi_a,
                                             const uint32_t* path_b, uint32_t n_b, uint32_t offset_b, uint32_t lo_b, uint32_t hi_b) {
    oracle::Graph g(ix);
    return make_test_extension(path_a, n_a, offset_a, lo_a, hi_a).overlap(g, make_test_extension(path_b, n_b, offset_b, lo_b, hi_b));
}
// out = {start node, start offset, tail node, tail offset}
extern "C" void oracle_extension_positions(const gb_flat_index* ix, const uint32_t* path, uint32_t n, uint32_t offset, uint32_t read_lo, uint32_t read_hi, uint32_t* out) {
    oracle::Graph g(ix);
    const oracle::GaplessExtension e = make_test_extension(path, n, offset, read_lo, read_hi);
    const auto s = e.starting_position(g), t = e.tail_position(g);
    out[0] = s.first; out[1] = (uint32_t)s.second; out[2] = t.first; out[3] = (uint32_t)t.second;
}
