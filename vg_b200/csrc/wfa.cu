// wfa.cu — B2 stage seam: WFAExtender::connect / suffix / prefix (gbwt_extender.hpp:386-470,
// gbwt_extender.cpp:2052-2263), the haplotype-consistent gap-affine wavefront alignment vg's chaining
// route uses between and beyond seeds (minimizer_mapper_from_chains.cpp:2574, :2625, :2955, :3169).
//
// One THREAD per problem: the algorithm is a chain of small dependent decisions over a lazily grown
// haplotype trie (WFATree), with tiny wavefronts (the error model bounds the score), so many
// independent problems side by side is the parallelism there is.  Every thread owns a workspace in
// HBM: trie nodes (GBWT search state, concatenated node sequence, graph path), the wavefront points in
// an open-addressing hash table keyed (trie node, matrix, score, diagonal), and the sorted set of
// possible scores.  Control flow follows oracle/wfa.cpp statement by statement (same iteration
// orders: leaves by trie index, diagonals ascending, GBWT successors in record order).
#include <cub/cub.cuh>
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "align.cuh"

#include <algorithm>
#include <cstdlib>
#include <vector>

namespace gb {

constexpr uint32_t WFA_NODES = 64;          // trie nodes per problem
constexpr uint32_t WFA_SEQ_POOL = 24576;    // bytes of concatenated node sequence per problem
constexpr uint32_t WFA_PATH_POOL = 2048;    // graph nodes over all trie nodes
constexpr uint32_t WFA_HASH = 4096;         // wavefront points (power of two)
constexpr uint32_t WFA_HASH_SMALL = 256;    // first attempt
constexpr uint32_t WFA_SCORES = 512;        // distinct possible scores
constexpr uint32_t WFA_STACK = 64;          // MatchPos path depth / traversal stack
constexpr uint32_t WFA_TARGET_LENGTH = 1024;
constexpr uint32_t WFA_NO_TARGET = 0xffffffffu;
constexpr uint32_t WFA_THREADS = 32;

enum : uint32_t { W_MATCH = 0, W_MISMATCH = 1, W_INSERTION = 2, W_DELETION = 3 };
enum : uint32_t { WF_MATCHES = 0, WF_INSERTIONS = 1, WF_DELETIONS = 2 };

struct WfaNode {
    uint32_t parent, child_begin, child_count;
    uint32_t g_node; int32_t lo, hi;            // GBWT search state at the end of the path
    uint32_t seq_off, seq_len;                  // in the sequence pool
    uint32_t path_off, path_len;                // in the path pool
    uint32_t target_offset;
    uint32_t dead_end;
};
struct WfaScore { int32_t score, min_diagonal, max_diagonal; uint32_t reachable_with_gap; };

struct WfaWs {
    WfaNode* nodes; uint8_t* seq; uint32_t* path; uint64_t* hash; WfaScore* scores;
    uint32_t n_nodes, seq_used, path_used, n_scores;
    uint32_t hash_mask;         // table size in use - 1: problems start with WFA_HASH_SMALL cells (clearing the table is most of a
                                // small problem's memory traffic) and are redone with all WFA_HASH cells when that fills up
    bool overflow, hash_full;
};

struct WfaPos {            // MatchPos: offsets + the trie path from a leaf (bottom) to the node (top)
    uint32_t seq_offset, node_offset;
    uint32_t path[WFA_STACK]; uint32_t depth;
    __device__ bool empty() const { return depth == 0; }
    __device__ uint32_t node() const { return path[depth - 1]; }
    __device__ int32_t distance(int32_t diagonal) const { return 2 * (int32_t)seq_offset - diagonal; }
};
__device__ __forceinline__ bool wfa_pos_less(const WfaPos& a, const WfaPos& b) {
    if (a.empty()) return !b.empty();
    if (b.empty()) return false;
    return a.seq_offset < b.seq_offset;
}

struct WfaProblem {
    const uint8_t* seq; uint32_t seq_len;       // masked sequence (non-ACGT -> 'X')
    uint32_t to_node, to_offset; bool has_to;
    int32_t mismatch, gap_open, gap_extend, score_bound, max_distance, min_distance;
    int32_t cand_score, cand_diagonal; uint32_t cand_seq_offset, cand_node_offset, cand_node;
};

// ---- wavefront points: open addressing, key = node | type | score | diagonal --------------------------
__device__ __forceinline__ uint32_t wfa_key(uint32_t type, uint32_t node, int32_t score, int32_t diagonal) {
    return (node << 26) | (type << 24) | ((uint32_t)score << 11) | (uint32_t)(diagonal + 1024);
}
__device__ inline bool wfa_find(const WfaWs& ws, uint32_t type, uint32_t node, int32_t score, int32_t diagonal, uint32_t& seq_offset, uint32_t& node_offset) {
    const uint32_t key = wfa_key(type, node, score, diagonal);
    uint32_t h = (key * 2654435761u) & ws.hash_mask;
    while (true) {
        const uint64_t e = ws.hash[h];
        if (e == ~0ull) return false;
        if ((uint32_t)(e >> 32) == key) { seq_offset = (uint32_t)e >> 16; node_offset = (uint32_t)e & 0xffffu; return true; }
        h = (h + 1) & ws.hash_mask;
    }
}
__device__ inline void wfa_update(WfaWs& ws, uint32_t type, uint32_t node, int32_t score, int32_t diagonal, uint32_t seq_offset, uint32_t node_offset, uint32_t& n_points) {
    if (score < 0 || score >= 8192 || diagonal < -1024 || diagonal >= 1024 || seq_offset > 0xffffu || node_offset > 0xffffu) { ws.overflow = true; return; }
    const uint32_t key = wfa_key(type, node, score, diagonal);
    uint32_t h = (key * 2654435761u) & ws.hash_mask;
    while (true) {
        const uint64_t e = ws.hash[h];
        if (e == ~0ull) {
            if (n_points + 1 >= (ws.hash_mask + 1) * 3 / 4) { ws.overflow = true; ws.hash_full = true; return; }
            n_points++;
            break;
        }
        if ((uint32_t)(e >> 32) == key) break;
        h = (h + 1) & ws.hash_mask;
    }
    ws.hash[h] = ((uint64_t)key << 32) | (seq_offset << 16) | node_offset;
}

// ---- possible scores: sorted array ------------------------------------------------------------------------
__device__ inline int32_t wfa_score_index(const WfaWs& ws, int32_t score) {
    int32_t lo = 0, hi = (int32_t)ws.n_scores - 1;
    while (lo <= hi) { const int32_t mid = (lo + hi) >> 1; const int32_t s = ws.scores[mid].score; if (s == score) return mid; if (s < score) lo = mid + 1; else hi = mid - 1; }
    return -1;
}
__device__ inline void wfa_score_insert(WfaWs& ws, int32_t score, bool reachable_with_gap) {
    if (ws.n_scores >= WFA_SCORES) { ws.overflow = true; return; }
    uint32_t i = ws.n_scores;
    while (i > 0 && ws.scores[i - 1].score > score) { ws.scores[i] = ws.scores[i - 1]; i--; }
    ws.scores[i] = WfaScore{score, 0, 0, reachable_with_gap ? 1u : 0u};
    ws.n_scores++;
}

// ---- trie nodes (WFANode) -----------------------------------------------------------------------------------
__device__ inline bool wfa_append_node(const DevIndex& ix, WfaWs& ws, const WfaProblem& P, WfaNode& n, uint32_t g_node, int32_t lo, int32_t hi) {
    n.g_node = g_node; n.lo = lo; n.hi = hi;
    const gb_node_rec nr = load_node(ix, g_node);
    if (ws.path_used + 1 > WFA_PATH_POOL || ws.seq_used + nr.len > WFA_SEQ_POOL) { ws.overflow = true; return true; }
    ws.path[ws.path_used++] = g_node; n.path_len++;
    for (uint32_t i = 0; i < nr.len; i++) ws.seq[ws.seq_used + i] = __ldg(ix.seq + nr.seq_off + i);
    ws.seq_used += nr.len; n.seq_len += nr.len;
    if (P.has_to && P.to_node == g_node) { n.target_offset = n.seq_len - (nr.len - P.to_offset); return true; }
    return false;
}
// occurrences of outrank e before `lo` and inside [lo, hi] of a record body (one thread; the warp version is record_edge_query)
__device__ inline void wfa_edge_query(const uint32_t* rec, uint32_t n_edges, uint32_t n_runs, int32_t lo, int32_t hi, uint32_t e, int32_t& below, int32_t& cnt) {
    const uint32_t* runs = rec + 2 + 2 * n_edges;
    int32_t pos = 0; below = 0; cnt = 0;
    for (uint32_t r = 0; r < n_runs; r++) {
        const uint32_t w = __ldg(runs + r);
        const int32_t len = (int32_t)(w >> 10), start = pos, end = pos + len;
        if ((w & 1023u) == e) { below += min(max(lo - start, 0), len); cnt += max(min(end, hi + 1) - max(start, lo), 0); }
        pos = end;
        if (pos > hi) break;
    }
}
// successors of a search state in record order (Graph::follow_paths, oracle/gbwt_view.hpp)
__device__ inline uint32_t wfa_successors(const DevIndex& ix, uint32_t g_node, int32_t lo, int32_t hi, uint32_t* to, int32_t* nlo, int32_t* nhi, uint32_t cap, bool& overflow) {
    const gb_node_rec nr = load_node(ix, g_node);
    if (nr.size == 0) return 0;
    const uint32_t* rec = ix.gbwt + nr.rec_off;
    const uint32_t n_edges = __ldg(rec), n_runs = __ldg(rec + 1);
    uint32_t count = 0;
    for (uint32_t e = 0; e < n_edges; e++) {
        const uint32_t t = __ldg(rec + 2 + 2 * e);
        if (t == 0) continue;
        int32_t below, cnt;
        wfa_edge_query(rec, n_edges, n_runs, lo, hi, e, below, cnt);
        if (cnt <= 0) continue;
        if (count >= cap) { overflow = true; return count; }
        const int32_t first = (int32_t)__ldg(rec + 3 + 2 * e) + below;
        to[count] = t; nlo[count] = first; nhi[count] = first + cnt - 1; count++;
    }
    return count;
}
__device__ inline uint32_t wfa_make_node(const DevIndex& ix, WfaWs& ws, const WfaProblem& P, uint32_t g_node, int32_t lo, int32_t hi, uint32_t parent) {
    if (ws.n_nodes >= WFA_NODES) { ws.overflow = true; return 0; }
    const uint32_t id = ws.n_nodes++;
    WfaNode n; n.parent = parent; n.child_begin = 0; n.child_count = 0; n.seq_off = ws.seq_used; n.seq_len = 0; n.path_off = ws.path_used; n.path_len = 0;
    n.target_offset = WFA_NO_TARGET; n.dead_end = 0;
    if (!wfa_append_node(ix, ws, P, n, g_node, lo, hi)) {
        while (n.seq_len < WFA_TARGET_LENGTH && !ws.overflow) {
            uint32_t to[2]; int32_t nlo[2], nhi[2]; bool many = false;
            const uint32_t successors = wfa_successors(ix, n.g_node, n.lo, n.hi, to, nlo, nhi, 2, many);
            if (successors == 0) { n.dead_end = 1; break; }
            if (successors > 1 || many) break;
            if (wfa_append_node(ix, ws, P, n, to[0], nlo[0], nhi[0])) break;
        }
    }
    ws.nodes[id] = n;
    return id;
}
__device__ __forceinline__ bool wfa_is_leaf(const WfaNode& n) { return n.child_count == 0 || n.dead_end; }
__device__ __forceinline__ bool wfa_expanded(const WfaNode& n) { return n.child_count != 0 || n.dead_end; }

__device__ inline void wfa_expand_if_necessary(const DevIndex& ix, WfaWs& ws, const WfaProblem& P, uint32_t node, uint32_t node_offset) {
    const WfaNode n = ws.nodes[node];
    if (wfa_expanded(n) || node_offset < n.seq_len) return;
    uint32_t to[32]; int32_t nlo[32], nhi[32]; bool ovf = false;
    const uint32_t cnt = wfa_successors(ix, n.g_node, n.lo, n.hi, to, nlo, nhi, 32, ovf);
    if (ovf) { ws.overflow = true; return; }
    if (cnt == 0) { ws.nodes[node].dead_end = 1; return; }
    ws.nodes[node].child_begin = ws.n_nodes; ws.nodes[node].child_count = cnt;
    for (uint32_t i = 0; i < cnt && !ws.overflow; i++) wfa_make_node(ix, ws, P, to[i], nlo[i], nhi[i], node);
}

// WFATree::find_pos
__device__ inline void wfa_find_pos(const WfaWs& ws, const WfaProblem& P, uint32_t type, uint32_t node, int32_t score, int32_t diagonal,
                                    bool extendable_seq, bool extendable_graph, WfaPos& pos) {
    pos.depth = 0; pos.seq_offset = 0; pos.node_offset = 0;
    if (score < 0) return;
    uint32_t depth = 0;
    while (true) {
        if (depth >= WFA_STACK) { pos.depth = 0; return; }
        pos.path[depth++] = node;
        uint32_t so, no;
        if (wfa_find(ws, type, node, score, diagonal, so, no)) {
            if (extendable_seq && so >= P.seq_len) return;
            if (extendable_graph && ws.nodes[node].dead_end && no >= ws.nodes[node].seq_len) return;
            pos.seq_offset = so; pos.node_offset = no; pos.depth = depth;
            return;
        }
        if (node == 0) return;
        node = ws.nodes[node].parent;
    }
}
__device__ inline void wfa_successor_offset(const WfaWs& ws, WfaPos& pos) {
    if (pos.node_offset >= ws.nodes[pos.node()].seq_len) { pos.depth--; pos.node_offset = 0; }
    pos.node_offset++;
}

struct WfaPred { WfaPos pos; uint32_t edit; };
__device__ inline void wfa_ins_predecessor(const WfaWs& ws, const WfaProblem& P, uint32_t node, int32_t score, int32_t diagonal, WfaPos& out, uint32_t& edit) {
    WfaPos open, ext;
    wfa_find_pos(ws, P, WF_MATCHES, node, score - P.gap_open - P.gap_extend, diagonal - 1, true, false, open);
    wfa_find_pos(ws, P, WF_INSERTIONS, node, score - P.gap_extend, diagonal - 1, true, false, ext);
    if (wfa_pos_less(open, ext)) { out = ext; edit = W_INSERTION; } else { out = open; edit = W_MATCH; }
}
__device__ inline void wfa_del_predecessor(const WfaWs& ws, const WfaProblem& P, uint32_t node, int32_t score, int32_t diagonal, WfaPos& out, uint32_t& edit) {
    WfaPos open, ext;
    wfa_find_pos(ws, P, WF_MATCHES, node, score - P.gap_open - P.gap_extend, diagonal + 1, false, true, open);
    wfa_find_pos(ws, P, WF_DELETIONS, node, score - P.gap_extend, diagonal + 1, false, true, ext);
    if (wfa_pos_less(open, ext)) { out = ext; edit = W_DELETION; } else { out = open; edit = W_MATCH; }
}
__device__ inline void wfa_match_predecessor(const WfaWs& ws, const WfaProblem& P, uint32_t node, int32_t score, int32_t diagonal, WfaPos& out, uint32_t& edit) {
    WfaPos ins, del, subst;
    wfa_find_pos(ws, P, WF_INSERTIONS, node, score, diagonal, false, false, ins);
    wfa_find_pos(ws, P, WF_DELETIONS, node, score, diagonal, false, false, del);
    wfa_find_pos(ws, P, WF_MATCHES, node, score - P.mismatch, diagonal, false, false, subst);
    if (!subst.empty()) { subst.seq_offset++; subst.node_offset++; }
    if (wfa_pos_less(ins, del)) { if (wfa_pos_less(del, subst)) { out = subst; edit = W_MISMATCH; } else { out = del; edit = W_DELETION; } }
    else { if (wfa_pos_less(ins, subst)) { out = subst; edit = W_MISMATCH; } else { out = ins; edit = W_INSERTION; } }
}

__device__ __forceinline__ int32_t wfa_gap_penalty(const WfaProblem& P, uint32_t length) { return P.gap_open + (int32_t)length * P.gap_extend; }

// wf_extend over one (score, diagonal): depth-first over the leaves, children as they appear
__device__ inline void wfa_extend_diagonal(const DevIndex& ix, WfaWs& ws, WfaProblem& P, int32_t score, int32_t diagonal, uint32_t& n_points) {
    // frames: [begin, end) ranges of trie nodes to visit; the first frame is the snapshot of all nodes (leaves only)
    uint32_t fb[WFA_STACK], fe[WFA_STACK]; bool leaves_only[WFA_STACK]; uint32_t sp = 0;
    fb[0] = 0; fe[0] = ws.n_nodes; leaves_only[0] = true; sp = 1;
    WfaPos pos;
    while (sp > 0 && !ws.overflow) {
        if (fb[sp - 1] >= fe[sp - 1]) { sp--; continue; }
        const uint32_t leaf = fb[sp - 1]++;
        if (leaves_only[sp - 1] && !wfa_is_leaf(ws.nodes[leaf])) continue;
        wfa_find_pos(ws, P, WF_MATCHES, leaf, score, diagonal, false, false, pos);
        if (pos.empty()) continue;
        while (!ws.overflow) {
            const uint32_t ni = pos.node();
            const WfaNode n = ws.nodes[ni];
            const bool may_reach_target = n.target_offset != WFA_NO_TARGET && n.target_offset >= pos.node_offset && n.target_offset < n.seq_len;
            // match_forward
            const uint8_t* ns = ws.seq + n.seq_off;
            while (pos.seq_offset < P.seq_len && pos.node_offset < n.seq_len && P.seq[pos.seq_offset] == ns[pos.node_offset]) { pos.seq_offset++; pos.node_offset++; }
            if ((may_reach_target && pos.node_offset >= n.target_offset) || (!P.has_to && pos.seq_offset >= P.seq_len)) {
                const uint32_t overshoot = !P.has_to ? 0u : pos.node_offset - n.target_offset;
                const uint32_t gap_length = (P.seq_len - pos.seq_offset) + overshoot;
                const int32_t gap_score = gap_length > 0 ? wfa_gap_penalty(P, gap_length) : 0;
                if (score + gap_score < P.cand_score) {
                    P.cand_score = score + gap_score; P.cand_diagonal = diagonal; P.cand_seq_offset = pos.seq_offset - overshoot; P.cand_node_offset = n.target_offset; P.cand_node = ni;
                }
            }
            P.max_distance = max(P.max_distance, pos.distance(diagonal));
            wfa_update(ws, WF_MATCHES, ni, score, diagonal, pos.seq_offset, pos.node_offset, n_points);
            if (pos.node_offset < n.seq_len) break;
            wfa_expand_if_necessary(ix, ws, P, ni, pos.node_offset);
            if (pos.depth == 1) {
                const WfaNode nn = ws.nodes[ni];
                if (nn.child_count > 0) {
                    if (sp >= WFA_STACK) { ws.overflow = true; break; }
                    fb[sp] = nn.child_begin; fe[sp] = nn.child_begin + nn.child_count; leaves_only[sp] = false; sp++;
                }
                break;
            }
            pos.depth--; pos.node_offset = 0;
        }
    }
}

struct WfaOut { int32_t ok, score; uint32_t node_offset, seq_offset, length, n_path, n_edits; };

// WFAExtender::connect; edits are written end -> start into `edits` then reversed in place
__device__ inline void wfa_connect(const DevIndex& ix, const DevScores& sc, const double* em, WfaWs& ws, const uint8_t* seq, uint32_t seq_len,
                                   uint32_t from_node, uint32_t from_offset, uint32_t to_node, uint32_t to_offset,
                                   uint32_t* out_path, uint32_t path_cap, uint32_t* out_edits, uint32_t edit_cap, WfaOut& out) {
    out.ok = 0; out.score = 0; out.node_offset = 0; out.seq_offset = 0; out.length = 0; out.n_path = 0; out.n_edits = 0;
    if (from_node < 2 || from_node >= ix.n_nodes || load_node(ix, from_node).len == 0) return;
    WfaProblem P;
    P.seq = seq; P.seq_len = seq_len; P.to_node = to_node; P.to_offset = to_offset; P.has_to = to_node != 0;
    P.mismatch = 2 * (sc.match + sc.mismatch); P.gap_open = 2 * (sc.gap_open - sc.gap_extend); P.gap_extend = 2 * sc.gap_extend + sc.match;
    P.max_distance = 0; P.min_distance = 0;
    P.cand_score = INT_MAX; P.cand_diagonal = 0; P.cand_seq_offset = 0; P.cand_node_offset = 0; P.cand_node = 0;
    auto evaluate = [&](int e) { return min((int32_t)em[3 * e + 2], (int32_t)(em[3 * e] * (double)seq_len) + (int32_t)em[3 * e + 1]); };
    P.score_bound = evaluate(0) * P.mismatch + evaluate(1) * P.gap_open + evaluate(2) * P.gap_extend;
    const int32_t distance_band = evaluate(3);
    ws.n_nodes = 0; ws.seq_used = 0; ws.path_used = 0; ws.n_scores = 0; ws.overflow = false; ws.hash_full = false;
    for (uint32_t i = 0; i <= ws.hash_mask; i++) ws.hash[i] = ~0ull;
    uint32_t n_points = 0;
    wfa_make_node(ix, ws, P, from_node, 0, (int32_t)load_node(ix, from_node).size - 1, 0);
    wfa_update(ws, WF_MATCHES, 0, 0, 0, 0, from_offset + 1, n_points);
    wfa_score_insert(ws, 0, false);

    int32_t score = 0;
    while (!ws.overflow) {
        // extend(score)
        const int32_t si = wfa_score_index(ws, score);
        if (si >= 0) {
            const int32_t lo = ws.scores[si].min_diagonal, hi = ws.scores[si].max_diagonal;
            for (int32_t diagonal = lo; diagonal <= hi && !ws.overflow; diagonal++) wfa_extend_diagonal(ix, ws, P, score, diagonal, n_points);
        }
        if (distance_band < P.max_distance) P.min_distance = P.max_distance - distance_band;
        if (P.cand_score <= score) break;
        // next_score(score)
        {
            const int32_t mismatch_score = score + P.mismatch;
            if (wfa_score_index(ws, mismatch_score) < 0) wfa_score_insert(ws, mismatch_score, false);
            int32_t mi = wfa_score_index(ws, score);
            if (ws.scores[mi].reachable_with_gap) {
                const int32_t extend_score = score + P.gap_extend;
                const int32_t ei = wfa_score_index(ws, extend_score);
                if (ei >= 0) ws.scores[ei].reachable_with_gap = 1; else wfa_score_insert(ws, extend_score, true);
            }
            const int32_t open_score = score + P.gap_open + P.gap_extend;
            const int32_t oi = wfa_score_index(ws, open_score);
            if (oi >= 0) ws.scores[oi].reachable_with_gap = 1; else wfa_score_insert(ws, open_score, true);
            if (ws.overflow) break;
            mi = wfa_score_index(ws, score);
            score = ws.scores[mi + 1].score;
        }
        if (score > P.score_bound) break;
        // next(score)
        {
            int32_t rlo = INT_MAX, rhi = INT_MIN;
            auto widen = [&](int32_t s) { if (s >= 0) { const int32_t k = wfa_score_index(ws, s); if (k >= 0) { rlo = min(rlo, ws.scores[k].min_diagonal); rhi = max(rhi, ws.scores[k].max_diagonal); } } };
            widen(score - P.mismatch); widen(score - P.gap_open - P.gap_extend); widen(score - P.gap_extend);
            int32_t alo = INT_MAX, ahi = INT_MIN;
            if (rlo <= rhi) {
                rlo--; rhi++;
                WfaPos ins, del, subst; uint32_t dummy;
                for (int32_t diagonal = rlo; diagonal <= rhi && !ws.overflow; diagonal++) {
                    const uint32_t snapshot = ws.n_nodes;
                    for (uint32_t leaf = 0; leaf < snapshot && !ws.overflow; leaf++) {
                        if (!wfa_is_leaf(ws.nodes[leaf])) continue;
                        wfa_ins_predecessor(ws, P, leaf, score, diagonal, ins, dummy);
                        if (!ins.empty()) {
                            ins.seq_offset++;
                            if (ins.distance(diagonal) >= P.min_distance) { wfa_update(ws, WF_INSERTIONS, ins.node(), score, diagonal, ins.seq_offset, ins.node_offset, n_points); alo = min(alo, diagonal); ahi = max(ahi, diagonal); }
                        }
                        wfa_del_predecessor(ws, P, leaf, score, diagonal, del, dummy);
                        if (!del.empty()) {
                            wfa_successor_offset(ws, del);
                            if (del.distance(diagonal) >= P.min_distance) { wfa_update(ws, WF_DELETIONS, del.node(), score, diagonal, del.seq_offset, del.node_offset, n_points); alo = min(alo, diagonal); ahi = max(ahi, diagonal); }
                            wfa_expand_if_necessary(ix, ws, P, del.node(), del.node_offset);
                        }
                        wfa_find_pos(ws, P, WF_MATCHES, leaf, score - P.mismatch, diagonal, true, true, subst);
                        if (!subst.empty()) { subst.seq_offset++; wfa_successor_offset(ws, subst); wfa_expand_if_necessary(ix, ws, P, subst.node(), subst.node_offset); }
                        if (wfa_pos_less(subst, ins)) subst = ins;
                        if (wfa_pos_less(subst, del)) subst = del;
                        if (!subst.empty()) {
                            const uint32_t ni = subst.node();
                            if (subst.node_offset == ws.nodes[ni].target_offset) {
                                const uint32_t gap_length = P.seq_len - subst.seq_offset;
                                const int32_t gap_score = gap_length > 0 ? wfa_gap_penalty(P, gap_length) : 0;
                                if (score + gap_score < P.cand_score) { P.cand_score = score + gap_score; P.cand_diagonal = diagonal; P.cand_seq_offset = subst.seq_offset; P.cand_node_offset = subst.node_offset; P.cand_node = ni; }
                            }
                            if (subst.distance(diagonal) >= P.min_distance) { wfa_update(ws, WF_MATCHES, ni, score, diagonal, subst.seq_offset, subst.node_offset, n_points); alo = min(alo, diagonal); ahi = max(ahi, diagonal); }
                        }
                    }
                }
            }
            const int32_t k = wfa_score_index(ws, score);
            if (k >= 0) { ws.scores[k].min_diagonal = alo; ws.scores[k].max_diagonal = ahi; }
        }
    }
    if (ws.overflow) { out.ok = -1; return; }

    uint32_t unaligned_tail = seq_len - P.cand_seq_offset;
    if (P.cand_score > P.score_bound) {
        unaligned_tail = 0;
        if (P.has_to) return;
        // trim: best partial alignment; ties to the smallest (trie node, score, diagonal) as in the oracle
        P.cand_score = 0; P.cand_diagonal = 0; P.cand_seq_offset = 0; P.cand_node_offset = 0; P.cand_node = 0;
        int32_t best_score = 0; uint64_t best_key = ~0ull;
        for (uint32_t h = 0; h <= ws.hash_mask; h++) {
            const uint64_t e = ws.hash[h];
            if (e == ~0ull) continue;
            const uint32_t key = (uint32_t)(e >> 32);
            if (((key >> 24) & 3u) != WF_MATCHES) continue;
            const uint32_t node = key >> 26; const int32_t s = (int32_t)((key >> 11) & 0x1fffu); const int32_t d = (int32_t)(key & 0x7ffu) - 1024;
            const uint32_t so = (uint32_t)e >> 16, no = (uint32_t)e & 0xffffu;
            const int32_t alignment_score = (sc.match * ((int32_t)so + ((int32_t)so - d)) - s) / 2;
            const uint64_t order = ((uint64_t)node << 40) | ((uint64_t)(uint32_t)s << 16) | (uint32_t)(d + 1024);
            if (alignment_score > best_score || (alignment_score == best_score && alignment_score > 0 && order < best_key)) {
                best_score = alignment_score; best_key = order;
                P.cand_score = s; P.cand_diagonal = d; P.cand_seq_offset = so; P.cand_node_offset = no; P.cand_node = node;
            }
        }
    }
    out.ok = 1;
    out.node_offset = from_offset + 1; out.seq_offset = 0;
    out.length = P.cand_seq_offset + unaligned_tail;
    out.score = (sc.match * ((int32_t)(P.cand_seq_offset + unaligned_tail) + ((int32_t)P.cand_seq_offset - P.cand_diagonal)) - P.cand_score) / 2;
    // backtrace; edits appended (merged) in reverse order
    uint32_t ne = 0;
    auto append = [&](uint32_t op, uint32_t len) {
        if (len == 0) return;
        if (ne > 0 && (out_edits[ne - 1] & 3u) == op) { out_edits[ne - 1] += len << 2; return; }
        if (ne >= edit_cap) { out.ok = -1; return; }
        out_edits[ne++] = (len << 2) | op;
    };
    int32_t pscore = P.cand_score, pdiag = P.cand_diagonal; uint32_t pseq = P.cand_seq_offset, pnode_off = P.cand_node_offset;
    uint32_t node = P.cand_node;
    if (unaligned_tail > 0) { append(W_INSERTION, seq_len - P.cand_seq_offset); pscore -= wfa_gap_penalty(P, unaligned_tail); }
    uint32_t edit = W_MATCH;
    WfaPos pred; uint32_t ptype;
    uint32_t guard = 0;
    while ((pseq > 0 || pdiag != 0) && out.ok == 1) {
        if (++guard > 100000) { out.ok = -1; break; }
        if (edit == W_MATCH) {
            wfa_match_predecessor(ws, P, node, pscore, pdiag, pred, ptype);
            append(W_MATCH, pseq - pred.seq_offset);
            pseq = pred.seq_offset; pnode_off = pred.node_offset;
            if (!pred.empty()) node = pred.node();
            edit = ptype;
        } else if (edit == W_MISMATCH) {
            append(W_MISMATCH, 1);
            pseq--;
            if (pnode_off > 0) pnode_off--; else { node = ws.nodes[node].parent; pnode_off = ws.nodes[node].seq_len - 1; }
            pscore -= P.mismatch;
            edit = W_MATCH;
        } else if (edit == W_INSERTION) {
            wfa_ins_predecessor(ws, P, node, pscore, pdiag, pred, ptype);
            append(W_INSERTION, 1);
            pseq--;
            pscore -= ptype == W_INSERTION ? P.gap_extend : P.gap_open + P.gap_extend;
            pdiag--;
            edit = ptype;
        } else {
            wfa_del_predecessor(ws, P, node, pscore, pdiag, pred, ptype);
            append(W_DELETION, 1);
            if (pnode_off > 0) pnode_off--; else { node = ws.nodes[node].parent; pnode_off = ws.nodes[node].seq_len - 1; }
            pscore -= ptype == W_DELETION ? P.gap_extend : P.gap_open + P.gap_extend;
            pdiag++;
            edit = ptype;
        }
    }
    if (out.ok != 1) return;
    for (uint32_t i = 0; i < ne / 2; i++) { const uint32_t t = out_edits[i]; out_edits[i] = out_edits[ne - 1 - i]; out_edits[ne - 1 - i] = t; }
    out.n_edits = ne;
    // The graph path is the candidate's trie branch, root first, without an unused first node and unused trailing
    // nodes (gbwt_extender.cpp:2191-2212).  A trie node grows along a non-branching haplotype up to WFA_TARGET_LENGTH
    // bases, so the branch can run far past the alignment: the kept range [p0, pn) is found first, walking the branch
    // from its end, and only that range has to fit path_cap.
    uint32_t total = 0; int64_t branch_len = 0;
    for (uint32_t node = P.cand_node;; node = ws.nodes[node].parent) {
        total += ws.nodes[node].path_len; branch_len += ws.nodes[node].seq_len;
        if (node == 0) break;
    }
    const uint32_t from_len = load_node(ix, from_node).len;          // the root's first graph node
    const uint32_t p0 = out.node_offset >= from_len ? 1u : 0u;
    if (p0) out.node_offset = 0;
    uint32_t pn = total;
    uint32_t c = P.cand_node, ci = ws.nodes[c].path_len;              // cursor: entry ci - 1 of trie node c is branch entry pn - 1
    auto step_back = [&]() { if (--ci == 0 && c != 0) { c = ws.nodes[c].parent; ci = ws.nodes[c].path_len; } };
    auto entry = [&]() { return ws.path[ws.nodes[c].path_off + ci - 1]; };
    if (pn > p0) {
        int64_t final_offset = out.node_offset;
        for (uint32_t i = 0; i < ne; i++) if ((out_edits[i] & 3u) != W_INSERTION) final_offset += out_edits[i] >> 2;
        final_offset -= branch_len - (p0 ? from_len : 0u) - load_node(ix, entry()).len;
        while ((pn - p0 == 1 && final_offset == (int64_t)out.node_offset) || (pn - p0 > 1 && final_offset <= 0)) {
            pn--; step_back();
            if (pn > p0) final_offset += load_node(ix, entry()).len;
        }
    }
    if (pn - p0 > path_cap) { out.ok = -1; return; }
    for (uint32_t i = pn; i > p0; i--, step_back()) out_path[i - 1 - p0] = entry();
    out.n_path = pn - p0;
}

struct WfaBatch {
    uint32_t n;
    const uint8_t* seq; const uint64_t* seq_off; const uint32_t* mode; const uint32_t* pos;     // pos: from node, from offset, to node, to offset
    const double* error_model;
    int32_t* ok; int32_t* score; uint32_t* node_offset; uint32_t* seq_offset; uint32_t* length; uint32_t* n_path; uint32_t* n_edits;
    uint32_t* path; uint32_t* edits; uint32_t path_cap, edit_cap;
    uint8_t* work_seq;                          // masked (and for prefix: reverse-complemented) copies
    WfaNode* nodes; uint8_t* seq_pool; uint32_t* path_pool; uint64_t* hash; WfaScore* scores;
    uint32_t* work_counter;
    uint32_t first_hash_mask;                   // WFA_HASH_SMALL - 1, or WFA_HASH - 1 with GIRAFFE_B200_WFA_SMALL_TABLE=0
};

__global__ void __launch_bounds__(WFA_THREADS)
wfa_kernel(DevIndex ix, DevScores sc, WfaBatch b) {
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    WfaWs ws;
    ws.nodes = b.nodes + tid * WFA_NODES; ws.seq = b.seq_pool + tid * WFA_SEQ_POOL; ws.path = b.path_pool + tid * WFA_PATH_POOL;
    ws.hash = b.hash + tid * WFA_HASH; ws.scores = b.scores + tid * WFA_SCORES;
    while (true) {
        const uint32_t p = atomicAdd(b.work_counter, 1u);
        if (p >= b.n) break;
        const uint64_t s0 = b.seq_off[p]; const uint32_t L = (uint32_t)(b.seq_off[p + 1] - s0);
        const uint32_t mode = b.mode[p];
        uint32_t from_node = b.pos[4 * p], from_offset = b.pos[4 * p + 1], to_node = b.pos[4 * p + 2], to_offset = b.pos[4 * p + 3];
        uint8_t* wseq = b.work_seq + s0;
        WfaOut out;
        uint32_t* opath = b.path + (size_t)p * b.path_cap; uint32_t* oedits = b.edits + (size_t)p * b.edit_cap;
        bool run = true;
        if (mode == 2) {
            // prefix: flip the position, align the reverse complement forward, flip the result (:2243-2259)
            if (to_node < 2 || to_node >= ix.n_nodes || load_node(ix, to_node).len == 0) { out.ok = 0; out.score = 0; out.node_offset = out.seq_offset = out.length = out.n_path = out.n_edits = 0; run = false; }
            else {
                for (uint32_t i = 0; i < L; i++) { const uint8_t c = b.seq[s0 + L - 1 - i]; wseq[i] = c == 'A' ? 'T' : (c == 'C' ? 'G' : (c == 'G' ? 'C' : (c == 'T' ? 'A' : 'X'))); }
                from_node = to_node ^ 1u; from_offset = load_node(ix, to_node).len - 1 - to_offset; to_node = 0; to_offset = 0;
            }
        } else {
            for (uint32_t i = 0; i < L; i++) { const uint8_t c = b.seq[s0 + i]; wseq[i] = (c == 'A' || c == 'C' || c == 'G' || c == 'T') ? c : (uint8_t)'X'; }
            if (mode == 1) { to_node = 0; to_offset = 0; }
        }
        if (run) {
            ws.hash_mask = b.first_hash_mask;
            wfa_connect(ix, sc, b.error_model, ws, wseq, L, from_node, from_offset, to_node, to_offset, opath, b.path_cap, oedits, b.edit_cap, out);
            if (out.ok == -1 && ws.hash_full && ws.hash_mask != WFA_HASH - 1) {          // the small table filled up: the same problem with the whole table
                ws.hash_mask = WFA_HASH - 1;
                wfa_connect(ix, sc, b.error_model, ws, wseq, L, from_node, from_offset, to_node, to_offset, opath, b.path_cap, oedits, b.edit_cap, out);
            }
        }
        if (run && out.ok == 1 && mode == 1) {
            if (out.n_edits > 0 && out.length == L && ((oedits[out.n_edits - 1] & 3u) == W_MATCH || (oedits[out.n_edits - 1] & 3u) == W_MISMATCH)) out.score += sc.full_length_bonus;
        }
        if (run && out.ok == 1 && mode == 2) {
            // WFAAlignment::flip (:834-848)
            out.seq_offset = L - out.seq_offset - out.length;
            if (out.n_path > 0) {
                int64_t final_offset = out.node_offset;
                for (uint32_t i = 0; i < out.n_edits; i++) if ((oedits[i] & 3u) != W_INSERTION) final_offset += oedits[i] >> 2;
                for (uint32_t i = 0; i + 1 < out.n_path; i++) final_offset -= load_node(ix, opath[i]).len;
                out.node_offset = (uint32_t)((int64_t)load_node(ix, opath[out.n_path - 1]).len - final_offset);
                for (uint32_t i = 0; i < out.n_path / 2; i++) { const uint32_t t = opath[i]; opath[i] = opath[out.n_path - 1 - i]; opath[out.n_path - 1 - i] = t; }
                for (uint32_t i = 0; i < out.n_path; i++) opath[i] ^= 1u;
                for (uint32_t i = 0; i < out.n_edits / 2; i++) { const uint32_t t = oedits[i]; oedits[i] = oedits[out.n_edits - 1 - i]; oedits[out.n_edits - 1 - i] = t; }
            }
            if (out.n_edits > 0 && out.length == L && ((oedits[0] & 3u) == W_MATCH || (oedits[0] & 3u) == W_MISMATCH)) out.score += sc.full_length_bonus;
        }
        b.ok[p] = out.ok; b.score[p] = out.ok == 1 ? out.score : 0; b.node_offset[p] = out.node_offset; b.seq_offset[p] = out.seq_offset;
        b.length[p] = out.length; b.n_path[p] = out.ok == 1 ? out.n_path : 0; b.n_edits[p] = out.ok == 1 ? out.n_edits : 0;
    }
}

} // namespace gb

using namespace gb;

extern "C" int gb_wfa_batch(gb_device* d, uint32_t n, const uint8_t* seq, const uint64_t* seq_off, const uint32_t* mode,
                            const uint32_t* pos, const double* error_model, uint32_t path_cap, uint32_t edit_cap,
                            int32_t* ok, int32_t* score, uint32_t* node_offset, uint32_t* seq_offset, uint32_t* length,
                            uint32_t* path, uint32_t* n_path, uint32_t* edits, uint32_t* n_edits) {
    if (!d || !seq || !seq_off || !mode || !pos || !ok || !score || !node_offset || !seq_offset || !length || !path || !n_path ||
        !edits || !n_edits || path_cap == 0 || edit_cap == 0) return GB_ERR_ARG;
    if (n == 0) return GB_OK;
    GB_CUDA(cudaSetDevice(d->device));
    static const double default_model[12] = {0.03, 1, 6, 0.05, 1, 10, 0.1, 1, 20, 0.1, 10, 200};     // gbwt_extender.hpp:372-381
    const double* em = error_model ? error_model : default_model;
    for (uint32_t i = 0; i < n; i++) {
        if (mode[i] > 2) return GB_ERR_ARG;
        if (seq_off[i + 1] - seq_off[i] > 60000) { g_last_error = "gb_wfa_batch: sequence too long"; return GB_ERR_ARG; }
    }
    const uint64_t total = seq_off[n];
    const uint32_t grid = std::max<uint32_t>(1u, std::min<uint32_t>((uint32_t)d->n_sms * 4, (n + WFA_THREADS - 1) / WFA_THREADS));
    const size_t threads = (size_t)grid * WFA_THREADS;
    DevBuf<uint8_t> d_seq, d_work, d_pool; DevBuf<uint64_t> d_soff, d_hash; DevBuf<uint32_t> d_mode, d_pos, d_noff, d_sqoff, d_len, d_np, d_ne, d_path, d_edits, d_ppool, d_counter;
    DevBuf<int32_t> d_ok, d_score; DevBuf<double> d_em; DevBuf<WfaNode> d_nodes; DevBuf<WfaScore> d_scores;
    int rc;
    if ((rc = d_seq.upload(seq, total ? total : 1, d->stream, total)) || (rc = d_work.reserve(total ? total : 1))) return rc;
    if ((rc = d_soff.upload(seq_off, n + 1, d->stream)) || (rc = d_mode.upload(mode, n, d->stream)) || (rc = d_pos.upload(pos, 4 * (size_t)n, d->stream))) return rc;
    if ((rc = d_em.upload(em, 12, d->stream))) return rc;
    if ((rc = d_ok.reserve(n)) || (rc = d_score.reserve(n)) || (rc = d_noff.reserve(n)) || (rc = d_sqoff.reserve(n)) || (rc = d_len.reserve(n)) ||
        (rc = d_np.reserve(n)) || (rc = d_ne.reserve(n))) return rc;
    if ((rc = d_path.reserve((size_t)n * path_cap)) || (rc = d_edits.reserve((size_t)n * edit_cap))) return rc;
    if ((rc = d_nodes.reserve(threads * WFA_NODES)) || (rc = d_pool.reserve(threads * WFA_SEQ_POOL)) || (rc = d_ppool.reserve(threads * WFA_PATH_POOL)) ||
        (rc = d_hash.reserve(threads * WFA_HASH)) || (rc = d_scores.reserve(threads * WFA_SCORES)) || (rc = d_counter.reserve(4))) return rc;
    GB_CUDA(cudaMemsetAsync(d_counter.ptr, 0, 16, d->stream));
    WfaBatch b;
    b.n = n; b.seq = d_seq.ptr; b.seq_off = d_soff.ptr; b.mode = d_mode.ptr; b.pos = d_pos.ptr; b.error_model = d_em.ptr;
    b.ok = d_ok.ptr; b.score = d_score.ptr; b.node_offset = d_noff.ptr; b.seq_offset = d_sqoff.ptr; b.length = d_len.ptr; b.n_path = d_np.ptr; b.n_edits = d_ne.ptr;
    b.path = d_path.ptr; b.edits = d_edits.ptr; b.path_cap = path_cap; b.edit_cap = edit_cap; b.work_seq = d_work.ptr;
    b.nodes = d_nodes.ptr; b.seq_pool = d_pool.ptr; b.path_pool = d_ppool.ptr; b.hash = d_hash.ptr; b.scores = d_scores.ptr; b.work_counter = d_counter.ptr;
    { const char* env = std::getenv("GIRAFFE_B200_WFA_SMALL_TABLE"); b.first_hash_mask = (env && std::atoi(env) == 0) ? WFA_HASH - 1 : WFA_HASH_SMALL - 1; }
    GB_CUDA(cudaEventRecord(d->ev0, d->stream));
    wfa_kernel<<<grid, WFA_THREADS, 0, d->stream>>>(d->ix, d->sc, b);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaEventRecord(d->ev1, d->stream));
    GB_CUDA(cudaMemcpyAsync(ok, d_ok.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(score, d_score.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(node_offset, d_noff.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(seq_offset, d_sqoff.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(length, d_len.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(n_path, d_np.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(n_edits, d_ne.ptr, 4 * (size_t)n, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(path, d_path.ptr, 4 * (size_t)n * path_cap, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(edits, d_edits.ptr, 4 * (size_t)n * edit_cap, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));
    GB_CUDA(cudaEventElapsedTime(&d->last_kernel_ms, d->ev0, d->ev1));
    return GB_OK;
}
