// index_builder.cpp — host-side construction of the flat ("GBZ-flat") index.
//
// Builds, from node sequences + haplotype paths:
//   * both-orientation node sequences, 1 B/base
//   * a bidirectional GBWT as flat record blobs (each path inserted forward and reverse,
//     like gbwt::GBWTBuilder::insert(path, true) — vg call site gbwt_helper.cpp:702-719)
//   * the (k,w)-minimizer hash table over all haplotypes with 16-B distance payloads
//     (vg: gbwtgraph::index_haplotypes via gbwtgraph_helper.cpp:511-630)
//
// This is offline indexing (out of the measured hot path); it exists so the synthetic
// BASELINE.json configs and the reference's unit-test graphs can be loaded into HBM.

#include "giraffe_b200.h"
#include "entry_guard.h"
#include "index_build.h"
#include "minimizer_common.h"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <array>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <new>
#include <numeric>
#include <string>
#include <unordered_map>
#include <vector>

struct gb_host_index {
    uint32_t n_nodes = 0, k = 0, w = 0, n_paths = 0;
    std::vector<gb_node_rec> nodes;
    std::vector<uint8_t> seq;
    std::vector<uint32_t> gbwt;
    std::vector<gb_dist_payload> dist;
    std::vector<gb_min_cell> table;
    std::vector<gb_hit> hits;
    std::vector<gb_slot_rec> slots;
    std::vector<uint16_t> site_dist;
    bool model_ok = true;            // the distance payload is valid (given by the caller or derived)
    gb_index_timing timing{};        // how the build spent its time (gb_index_build_timing)
};

namespace {

inline uint8_t comp(uint8_t c) {
    switch (c) {
        case 'A': return 'T'; case 'C': return 'G'; case 'G': return 'C'; case 'T': return 'A';
        default: return 'N';
    }
}

// Order all path visits by their reversed prefix (v_{i-1}, v_{i-2}, ..., v_0, $seq) using
// prefix doubling; this is the order of visits inside each GBWT record.
void gbwt_visit_order(const std::vector<std::vector<uint32_t>>& seqs,
                      std::vector<uint32_t>& rank_out /* per global visit */,
                      std::vector<uint64_t>& seq_start) {
    size_t n = 0;
    seq_start.resize(seqs.size() + 1);
    for (size_t s = 0; s < seqs.size(); s++) { seq_start[s] = n; n += seqs[s].size(); }
    seq_start[seqs.size()] = n;
    std::vector<uint32_t> pos_in_seq(n), seq_of(n);
    for (size_t s = 0; s < seqs.size(); s++)
        for (size_t i = 0; i < seqs[s].size(); i++) { pos_in_seq[seq_start[s] + i] = (uint32_t)i; seq_of[seq_start[s] + i] = (uint32_t)s; }

    // Initial key: (own node, predecessor node); visits with no predecessor are unique by seq id.
    // rank[p] is the rank of the reversed prefix of length h (starting at the predecessor).
    std::vector<uint64_t> key(n);
    std::vector<uint32_t> rank(n), tmp(n), order(n);
    // First element of the key is the predecessor node (0 = endmarker); ties among
    // endmarker predecessors are broken by sequence id which makes them final.
    // We use 64-bit keys: (pred_node << 32) | (pred is endmarker ? seq id : 0).
    for (size_t p = 0; p < n; p++) {
        uint32_t s = seq_of[p], i = pos_in_seq[p];
        if (i == 0) key[p] = (uint64_t)s;                         // (0, s)
        else key[p] = ((uint64_t)seqs[s][i - 1] << 32);
    }
    std::iota(order.begin(), order.end(), 0u);
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
    bool all_unique = true;
    {
        uint32_t r = 0;
        for (size_t j = 0; j < n; j++) {
            if (j > 0 && key[order[j]] != key[order[j - 1]]) r = (uint32_t)j;
            if (j > 0 && key[order[j]] == key[order[j - 1]]) all_unique = false;
            rank[order[j]] = r;
        }
    }
    // Doubling: rank_h covers h predecessors; combine with rank_h of the visit h steps back.
    for (size_t h = 1; !all_unique; h *= 2) {
        for (size_t p = 0; p < n; p++) {
            uint32_t i = pos_in_seq[p];
            // The visit h steps back; if it does not exist the key is already unique.
            uint64_t second = (i >= h) ? (uint64_t)rank[p - h] + 1 : 0;
            key[p] = ((uint64_t)rank[p] << 32) | second;
        }
        std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
        all_unique = true;
        uint32_t r = 0;
        for (size_t j = 0; j < n; j++) {
            if (j > 0 && key[order[j]] != key[order[j - 1]]) r = (uint32_t)j;
            else if (j > 0) all_unique = false;
            tmp[order[j]] = r;
        }
        rank.swap(tmp);
        if (h > n) break;
    }
    rank_out = rank;
}

// ---- distance payload from the graph itself -------------------------------------------------------------------------
// (what vg's SnarlDistanceIndex + zipcodes give the clusterer, snarl_seed_clusterer.cpp / zip_code.cpp, for DAGs.)
// The graph is the forward-strand edges the haplotype paths use.  Per connected component: topological order; cut nodes
// (every walk from a source to a sink passes them) split the order into slots — a cut node, or the site between two
// consecutive cut nodes; x_in = minimum distance from the component's sources to the node start; x_out = x_in of the next
// cut node minus the minimum distance from the node's end to it; per site the all-pairs table end(u) -> start(v).
// Returns false for anything outside that model (a reverse step, a cycle, an oversized site).
constexpr uint32_t MAX_SITE_NODES = 4096;

// The forward-strand graph of a set of haplotype paths: node ids in use and (id, id) edges; false when a haplotype steps onto a
// reverse strand.
bool forward_graph_of_paths(uint32_t n_node_ids, const std::vector<std::vector<uint32_t>>& fwd_paths, std::vector<bool>& used,
                            std::vector<std::pair<uint32_t, uint32_t>>& edges) {
    used.assign(n_node_ids + 1, false); edges.clear();
    for (const auto& p : fwd_paths) {
        for (size_t i = 0; i < p.size(); i++) {
            if (p[i] & 1u) return false;
            used[p[i] >> 1] = true;
            if (i) edges.emplace_back(p[i - 1] >> 1, p[i] >> 1);
        }
    }
    return true;
}

bool derive_distance_payload(uint32_t n_node_ids, const std::vector<uint32_t>& len /* by id */, const std::vector<bool>& used_in,
                             std::vector<std::pair<uint32_t, uint32_t>> edges,
                             std::vector<gb_dist_payload>& dist, std::vector<gb_slot_rec>& slots, std::vector<uint16_t>& site_dist) {
    const uint32_t N = n_node_ids + 1;
    std::vector<std::vector<uint32_t>> succ(N), pred(N);
    std::vector<bool> used = used_in;
    {
        std::sort(edges.begin(), edges.end());
        edges.erase(std::unique(edges.begin(), edges.end()), edges.end());
        for (const auto& e : edges) { succ[e.first].push_back(e.second); pred[e.second].push_back(e.first); }
    }
    dist.assign(N, gb_dist_payload{0, 0, 0, 0xFFFF, 0});
    slots.clear(); site_dist.clear();
    // components (undirected)
    std::vector<int32_t> comp(N, -1);
    uint32_t n_comp = 0;
    for (uint32_t s = 1; s < N; s++) {
        if (!used[s] || comp[s] >= 0) continue;
        std::vector<uint32_t> stack{s}; comp[s] = (int32_t)n_comp;
        while (!stack.empty()) {
            const uint32_t v = stack.back(); stack.pop_back();
            for (uint32_t w : succ[v]) if (comp[w] < 0) { comp[w] = (int32_t)n_comp; stack.push_back(w); }
            for (uint32_t w : pred[v]) if (comp[w] < 0) { comp[w] = (int32_t)n_comp; stack.push_back(w); }
        }
        n_comp++;
    }
    if (n_comp > 0xFFFF) return false;
    // one topological order over everything (Kahn, smallest id first: deterministic)
    std::vector<uint32_t> indeg(N, 0), order;
    for (uint32_t v = 1; v < N; v++) indeg[v] = (uint32_t)pred[v].size();
    {
        std::vector<uint32_t> ready;
        for (uint32_t v = N; v-- > 1;) if (used[v] && indeg[v] == 0) ready.push_back(v);       // descending: pop_back yields the smallest
        while (!ready.empty()) {
            const uint32_t v = ready.back(); ready.pop_back();
            order.push_back(v);
            bool pushed = false;
            for (uint32_t w : succ[v]) if (--indeg[w] == 0) { ready.push_back(w); pushed = true; }
            if (pushed) std::sort(ready.begin(), ready.end(), std::greater<uint32_t>());
        }
        size_t n_used = 0; for (uint32_t v = 1; v < N; v++) n_used += used[v];
        if (order.size() != n_used) return false;                 // a cycle
    }
    // per component: the nodes in topological order
    std::vector<std::vector<uint32_t>> comp_order(n_comp);
    for (uint32_t v : order) comp_order[(size_t)comp[v]].push_back(v);
    const uint64_t INF = ~0ull;
    std::vector<uint64_t> dS(N, INF);          // min distance from the component's sources to the node start
    std::vector<uint64_t> dX(N, 0);
    for (uint32_t c = 0; c < n_comp; c++) {
        const auto& ord = comp_order[c];
        for (uint32_t v : ord) {
            if (pred[v].empty()) dS[v] = 0;
            for (uint32_t p : pred[v]) dS[v] = std::min(dS[v], dS[p] + len[p]);
            if (dS[v] > 0x7FFFFFF0ull) return false;               // coordinates are read as int32
        }
        // cut nodes: every walk from a source to a sink passes them.  Sweep the order counting open edges (tail placed, head
        // not), with one virtual edge into every source and one out of every sink: v is a cut node exactly when all open
        // edges point at v as it comes up (an earlier sink keeps its virtual edge open for good, a waiting source too).
        std::vector<bool> is_cut(ord.size(), false);
        {
            uint64_t open = 0;
            for (uint32_t v : ord) open += pred[v].empty();
            for (size_t i = 0; i < ord.size(); i++) {
                const uint32_t v = ord[i];
                const uint64_t into_v = pred[v].empty() ? 1 : pred[v].size();
                is_cut[i] = (open == into_v);
                open -= into_v;
                open += succ[v].empty() ? 1 : succ[v].size();
            }
        }
        // slots along the chain
        size_t i = 0;
        while (i < ord.size()) {
            const uint32_t slot = (uint32_t)slots.size();
            if (is_cut[i]) {
                const uint32_t v = ord[i];
                dist[v] = gb_dist_payload{(uint32_t)dS[v], (uint32_t)(dS[v] + len[v]), slot, 0xFFFF, (uint16_t)c};
                slots.push_back(gb_slot_rec{0xFFFFFFFFu, 1u});
                i++;
                continue;
            }
            size_t j = i;
            while (j < ord.size() && !is_cut[j]) j++;
            const uint32_t n = (uint32_t)(j - i);
            if (n > MAX_SITE_NODES) return false;
            // exit coordinate: the next cut node's start, or (no cut node behind the site) the end of the chain
            uint64_t exit_coord;
            if (j < ord.size()) exit_coord = dS[ord[j]];
            else { exit_coord = 0; bool any = false; for (size_t x = i; x < j; x++) if (succ[ord[x]].empty()) { const uint64_t e = dS[ord[x]] + len[ord[x]]; exit_coord = any ? std::min(exit_coord, e) : e; any = true; } }
            // distance from each node's end to the exit (reverse order); nodes that cannot reach it keep INF
            std::vector<uint64_t> to_exit(n, INF);
            std::vector<uint32_t> local(n);
            std::map<uint32_t, uint32_t> li_of;
            for (uint32_t x = 0; x < n; x++) { local[x] = ord[i + x]; li_of[local[x]] = x; }
            for (uint32_t x = n; x-- > 0;) {
                const uint32_t v = local[x];
                if (succ[v].empty()) { to_exit[x] = 0; continue; }                 // ends the chain here
                for (uint32_t w : succ[v]) {
                    if (j < ord.size() && w == ord[j]) to_exit[x] = 0;
                    else { auto it = li_of.find(w); if (it != li_of.end() && to_exit[it->second] != INF) to_exit[x] = std::min(to_exit[x], to_exit[it->second] + len[w]); }
                }
            }
            const uint32_t table_off = (uint32_t)site_dist.size();
            if ((uint64_t)table_off + (uint64_t)n * n > 0xFFFFFFF0ull) return false;
            site_dist.resize((size_t)table_off + (size_t)n * n, 0xFFFF);
            for (uint32_t a = 0; a < n; a++) {
                // D[a][b]: min distance from the end of a to the start of b, forward in topological order
                std::vector<uint64_t> row(n, INF);
                for (uint32_t b = a + 1; b < n; b++) {
                    for (uint32_t p : pred[local[b]]) {
                        auto it = li_of.find(p);
                        if (it == li_of.end()) continue;
                        const uint32_t pl = it->second;
                        if (pl == a) row[b] = 0;
                        else if (pl > a && row[pl] != INF) row[b] = std::min(row[b], row[pl] + len[p]);
                    }
                    if (row[b] != INF) { if (row[b] >= 0xFFFF) return false; site_dist[(size_t)table_off + (size_t)a * n + b] = (uint16_t)row[b]; }
                }
            }
            for (uint32_t x = 0; x < n; x++) {
                const uint32_t v = local[x];
                // x_out is SIGNED (two's complement in the 32-bit field): when a shorter route bypasses the site (a deletion
                // spanning it), the way from this node to the exit is longer than the exit's own chain coordinate
                const int64_t xo = to_exit[x] == INF ? (int64_t)(dS[v] + len[v]) : (int64_t)exit_coord - (int64_t)to_exit[x];
                if (xo < -(int64_t)0x7ffffff0 || xo > (int64_t)0x7ffffff0) return false;
                dist[v] = gb_dist_payload{(uint32_t)dS[v], (uint32_t)(int32_t)xo, slot, (uint16_t)x, (uint16_t)c};
            }
            slots.push_back(gb_slot_rec{table_off, n});
            i = j;
        }
    }
    return true;
}

} // namespace

// A GBWT node record handed to the builder instead of haplotype paths (GBZ files, gb_index_build_from_gbwt): edges sorted by
// successor (oriented node, 0 = endmarker) with the offset of this node's visits in the successor's record, and the body as runs.
struct GbwtRecordIn { std::vector<std::pair<uint32_t, uint32_t>> edges; std::vector<std::pair<uint32_t, uint64_t>> runs; };

static int index_build_impl(uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off,
                            uint32_t n_paths, const uint32_t* path_nodes, const uint64_t* path_off,
                            const gb_dist_payload* dist, uint32_t k, uint32_t w,
                            gb_host_index** out,
                            uint64_t n_ext_hits = 0, const uint64_t* ext_keys = nullptr, const uint64_t* ext_pos = nullptr,
                            const std::vector<GbwtRecordIn>* records = nullptr, int device = -1) {
    if (!node_seq || !node_off || !out || (!records && n_paths && (!path_nodes || !path_off))) return GB_ERR_ARG;
    if (records && records->size() != 2 * ((size_t)n_node_ids + 1)) return GB_ERR_ARG;
    const bool external = ext_keys != nullptr || ext_pos != nullptr;
    if (external && (!ext_keys || !ext_pos)) return GB_ERR_ARG;
    if (k == 0 || k > 31 || w == 0) return GB_ERR_ARG;
    // offsets into seq / gbwt / hits are 32-bit (gb_node_rec, gb_min_cell): both orientations at 1 B/base bound the
    // graph at 2 Gbp; larger inputs are refused instead of wrapping
    if (n_node_ids >= 0x7ffffff0u || 2 * node_off[n_node_ids] + 64 > 0xffffffffull) return GB_ERR_FORMAT;
    auto* ix = new gb_host_index();
    ix->k = k; ix->w = w; ix->n_paths = n_paths;
    auto clock = std::chrono::steady_clock::now();
    auto lap = [&](double& seconds) {
        const auto now = std::chrono::steady_clock::now();
        seconds = std::chrono::duration<double>(now - clock).count(); clock = now;
    };
    ix->n_nodes = 2 * (n_node_ids + 1);
    ix->nodes.assign(ix->n_nodes, gb_node_rec{0, 0, 0, 0});

    // --- sequences, both orientations ---
    uint64_t total = node_off[n_node_ids];
    ix->seq.reserve(2 * total + 64);
    for (uint32_t id = 1; id <= n_node_ids; id++) {
        uint64_t b = node_off[id - 1], e = node_off[id];
        uint32_t len = (uint32_t)(e - b);
        if (len > 1024) { delete ix; return GB_ERR_FORMAT; }
        if (len == 0) continue;                       // an id the graph does not use (a GBZ whose ids do not start at 1): no sequence, and no path or record may name it
        uint32_t vf = 2 * id, vr = 2 * id + 1;
        ix->nodes[vf].seq_off = (uint32_t)ix->seq.size(); ix->nodes[vf].len = len;
        for (uint64_t i = b; i < e; i++) ix->seq.push_back(node_seq[i]);
        ix->nodes[vr].seq_off = (uint32_t)ix->seq.size(); ix->nodes[vr].len = len;
        for (uint64_t i = e; i > b; i--) ix->seq.push_back(comp(node_seq[i - 1]));
    }
    ix->seq.resize(ix->seq.size() + 64, 0);
    lap(ix->timing.sequences_s);

    ix->dist.assign(n_node_ids + 1, gb_dist_payload{0, 0, 0, 0xFFFF, 0});
    if (dist) for (uint32_t id = 1; id <= n_node_ids; id++) ix->dist[id] = dist[id];
    else {
        std::vector<uint32_t> len_by_id(n_node_ids + 1, 0);
        for (uint32_t id = 1; id <= n_node_ids; id++) len_by_id[id] = (uint32_t)(node_off[id] - node_off[id - 1]);
        std::vector<bool> used; std::vector<std::pair<uint32_t, uint32_t>> edges; bool forward = true;
        if (records) {
            // the forward-strand graph straight from the records of the forward nodes
            used.assign(n_node_ids + 1, false);
            for (uint32_t v = 2; v < ix->n_nodes && forward; v += 2) {
                const GbwtRecordIn& rc = (*records)[v];
                if (rc.runs.empty()) continue;
                used[v >> 1] = true;
                for (const auto& e : rc.edges) {
                    if (e.first == 0) continue;
                    if (e.first >= ix->n_nodes) { delete ix; return GB_ERR_FORMAT; }
                    if (e.first & 1u) { forward = false; break; }
                    edges.emplace_back(v >> 1, e.first >> 1);
                }
            }
        } else {
            std::vector<std::vector<uint32_t>> fwd(n_paths);
            for (uint32_t p = 0; p < n_paths; p++) fwd[p].assign(path_nodes + path_off[p], path_nodes + path_off[p + 1]);
            for (const auto& f : fwd) for (uint32_t v : f) if (v < 2 || v >= ix->n_nodes || ix->nodes[v].len == 0) { delete ix; return GB_ERR_FORMAT; }
            forward = forward_graph_of_paths(n_node_ids, fwd, used, edges);
        }
        if (!forward || !derive_distance_payload(n_node_ids, len_by_id, used, std::move(edges), ix->dist, ix->slots, ix->site_dist)) {
            // outside the chain model (a cycle, a reversing haplotype, an oversized site): the graph, GBWT and minimizers are
            // still built, so the stage seams work on it (the reference's cyclic WFA test graphs), but there is no
            // distance payload: gb_index_has_distance_model() says so and gb_index_from_gbz refuses such a file
            ix->dist.assign(n_node_ids + 1, gb_dist_payload{0, 0, 0, 0xFFFF, 0});
            ix->slots.clear(); ix->site_dist.clear(); ix->model_ok = false;
        }
    }
    lap(ix->timing.distance_s);

    // --- bidirectional GBWT ---
    std::vector<std::vector<uint32_t>> seqs(records ? 0 : 2 * (size_t)n_paths);
    if (!records) {
        for (uint32_t p = 0; p < n_paths; p++) {
            uint64_t b = path_off[p], e = path_off[p + 1];
            auto& f = seqs[2 * p]; auto& r = seqs[2 * p + 1];
            f.assign(path_nodes + b, path_nodes + e);
            r.resize(e - b);
            for (uint64_t i = 0; i < e - b; i++) r[i] = path_nodes[e - 1 - i] ^ 1u;
            for (uint32_t v : f) if (v < 2 || v >= ix->n_nodes || ix->nodes[v].len == 0) { delete ix; return GB_ERR_FORMAT; }
        }
        std::vector<uint32_t> vrank; std::vector<uint64_t> seq_start;
        gbwt_visit_order(seqs, vrank, seq_start);
        size_t nvis = vrank.size();
        // group visits per node in record order
        struct Visit { uint32_t node, rank, pred, succ; };
        std::vector<Visit> visits(nvis);
        for (size_t s = 0; s < seqs.size(); s++) {
            for (size_t i = 0; i < seqs[s].size(); i++) {
                size_t p = seq_start[s] + i;
                visits[p] = Visit{seqs[s][i], vrank[p], i ? seqs[s][i - 1] : 0u,
                                  i + 1 < seqs[s].size() ? seqs[s][i + 1] : 0u};
            }
        }
        std::sort(visits.begin(), visits.end(), [](const Visit& a, const Visit& b) {
            if (a.node != b.node) return a.node < b.node;
            return a.rank < b.rank;
        });
        // record start per node
        std::vector<size_t> rec_begin(ix->n_nodes + 1, 0);
        for (auto& vis : visits) rec_begin[vis.node + 1]++;
        for (uint32_t v = 0; v < ix->n_nodes; v++) rec_begin[v + 1] += rec_begin[v];

        ix->gbwt.clear();
        ix->gbwt.push_back(0); ix->gbwt.push_back(0);   // offset 0 = "no record" sentinel (0 edges, 0 runs)
        for (uint32_t v = 2; v < ix->n_nodes; v++) {
            size_t b = rec_begin[v], e = rec_begin[v + 1];
            ix->nodes[v].size = (uint32_t)(e - b);
            if (e == b) { ix->nodes[v].rec_off = 0; continue; }
            // distinct successors, ascending
            std::vector<uint32_t> succ;
            for (size_t i = b; i < e; i++) succ.push_back(visits[i].succ);
            std::sort(succ.begin(), succ.end());
            succ.erase(std::unique(succ.begin(), succ.end()), succ.end());
            if (succ.size() >= 1024) { delete ix; return GB_ERR_FORMAT; }
            if (ix->gbwt.size() & 1) ix->gbwt.push_back(0);   // 8-byte align the edge pairs
            if (ix->gbwt.size() > 0xfffffff0ull) { delete ix; return GB_ERR_FORMAT; }
            ix->nodes[v].rec_off = (uint32_t)ix->gbwt.size();
            ix->gbwt.push_back((uint32_t)succ.size());
            size_t nruns_at = ix->gbwt.size();
            ix->gbwt.push_back(0);
            for (uint32_t wnode : succ) {
                uint32_t off = 0;
                if (wnode != 0) {
                    // number of visits in record(w) whose predecessor is smaller than v
                    size_t wb = rec_begin[wnode], we = rec_begin[wnode + 1];
                    // visits in a record are sorted by predecessor first
                    size_t lo = wb, hi = we;
                    while (lo < hi) { size_t mid = (lo + hi) / 2; if (visits[mid].pred < v) lo = mid + 1; else hi = mid; }
                    off = (uint32_t)(lo - wb);
                }
                ix->gbwt.push_back(wnode);
                ix->gbwt.push_back(off);
            }
            uint32_t nruns = 0;
            size_t i = b;
            while (i < e) {
                size_t j = i;
                while (j < e && visits[j].succ == visits[i].succ && (j - i) < ((1u << 22) - 1)) j++;
                uint32_t outrank = (uint32_t)(std::lower_bound(succ.begin(), succ.end(), visits[i].succ) - succ.begin());
                ix->gbwt.push_back(((uint32_t)(j - i) << 10) | outrank);
                nruns++;
                i = j;
            }
            ix->gbwt[nruns_at] = nruns;
        }
    } else {
        // the records as given: same blob layout, same normalisation as above (edges ascending by successor, the endmarker edge with
        // offset 0, maximal runs cut at 2^22 - 1), so an index built from the records of a GBWT equals the one built from its paths
        ix->gbwt.clear();
        ix->gbwt.push_back(0); ix->gbwt.push_back(0);
        std::vector<uint64_t> rec_size(ix->n_nodes, 0);
        for (uint32_t v = 2; v < ix->n_nodes; v++) for (const auto& r : (*records)[v].runs) rec_size[v] += r.second;
        for (uint32_t v = 2; v < ix->n_nodes; v++) {
            const GbwtRecordIn& rc = (*records)[v];
            if (rec_size[v] == 0) { ix->nodes[v].rec_off = 0; ix->nodes[v].size = 0; continue; }
            if (rec_size[v] > 0xfffffff0ull || rc.edges.empty() || rc.edges.size() >= 1024 || ix->nodes[v].len == 0) { delete ix; return GB_ERR_FORMAT; }
            ix->nodes[v].size = (uint32_t)rec_size[v];
            // every visit leaves through an edge; the offsets must lie inside the successor's record
            std::vector<uint64_t> through(rc.edges.size(), 0);
            for (const auto& r : rc.runs) { if (r.first >= rc.edges.size() || r.second == 0) { delete ix; return GB_ERR_FORMAT; } through[r.first] += r.second; }
            for (size_t e = 0; e < rc.edges.size(); e++) {
                const uint32_t to = rc.edges[e].first;
                if (e && to <= rc.edges[e - 1].first) { delete ix; return GB_ERR_FORMAT; }
                if (to == 0) continue;
                if (to < 2 || to >= ix->n_nodes || (uint64_t)rc.edges[e].second + through[e] > rec_size[to]) { delete ix; return GB_ERR_FORMAT; }
            }
            if (ix->gbwt.size() & 1) ix->gbwt.push_back(0);
            if (ix->gbwt.size() > 0xfffffff0ull) { delete ix; return GB_ERR_FORMAT; }
            ix->nodes[v].rec_off = (uint32_t)ix->gbwt.size();
            ix->gbwt.push_back((uint32_t)rc.edges.size());
            const size_t nruns_at = ix->gbwt.size();
            ix->gbwt.push_back(0);
            for (const auto& e : rc.edges) { ix->gbwt.push_back(e.first); ix->gbwt.push_back(e.first == 0 ? 0u : e.second); }
            uint32_t nruns = 0;
            for (size_t i = 0; i < rc.runs.size();) {
                uint64_t len = 0; size_t j = i;
                while (j < rc.runs.size() && rc.runs[j].first == rc.runs[i].first) { len += rc.runs[j].second; j++; }
                while (len > 0) {
                    const uint64_t piece = std::min<uint64_t>(len, (1u << 22) - 1);
                    ix->gbwt.push_back(((uint32_t)piece << 10) | rc.runs[i].first);
                    nruns++; len -= piece;
                }
                i = j;
            }
            ix->gbwt[nruns_at] = nruns;
        }
    }
    ix->gbwt.resize(ix->gbwt.size() + 64, 0);
    lap(ix->timing.gbwt_s);

    // --- minimizer index over forward haplotypes ---
    using KP = gb::KeyPos;
    std::vector<KP> kps;
    gb::WindowCounts counts;
    bool sorted = false;                              // kps is already sorted and unique (the device route)
    std::string hap; std::vector<uint32_t> base_node; std::vector<uint32_t> base_off;
    std::vector<gbmin::Minimizer> mins;
    if (external) {
        // the minimizer table comes from the caller (what a gbwtgraph .min file holds, giraffe_main.cpp:1825-1881):
        // (key, position) pairs, position = id << 11 | is_reverse << 10 | offset, the first base of the canonical k-mer
        // on that oriented node.  Each is checked against the graph: the node exists, the offset lies inside it, and the
        // bases of the k-mer that fall on this node spell the leading bases of the key — a table that belongs to
        // another graph is GB_ERR_FORMAT, not a silent source of wrong seeds.
        kps.reserve(n_ext_hits);
        for (uint64_t i = 0; i < n_ext_hits; i++) {
            const uint64_t pos = ext_pos[i], v = pos >> 10; const uint32_t o = (uint32_t)(pos & 1023u);
            if (v < 2 || v >= ix->n_nodes || (k < 32 && (ext_keys[i] >> (2 * k)) != 0)) { delete ix; return GB_ERR_FORMAT; }
            const gb_node_rec& nr = ix->nodes[v];
            if (nr.len == 0 || o >= nr.len) { delete ix; return GB_ERR_FORMAT; }
            const uint32_t on_node = std::min<uint32_t>(k, nr.len - o);
            for (uint32_t j = 0; j < on_node; j++) {
                const uint32_t c = gbmin::base_code(ix->seq[nr.seq_off + o + j]);
                if (c != ((ext_keys[i] >> (2 * (k - 1 - j))) & 3u)) { delete ix; return GB_ERR_FORMAT; }
            }
            kps.push_back(KP{ext_keys[i], pos});
        }
    }
    // Two ways to the same set of (key, position) pairs.  The scan below walks every haplotype from end to end: work ~ haplotypes x
    // genome.  The window enumeration is what gbwtgraph's index construction does (index_haplotypes over for_each_haplotype_window,
    // gbwtgraph @ e27bc43, absent): every haplotype-consistent window of k + w - 1 bases is visited ONCE, however many haplotypes
    // share it, by following GBWT search states from every start position — work ~ graph x local diversity.  The minimizers of a
    // sequence are the union of the minimizers of its windows, so both give the same table (tests/test_gbz.py builds both).
    // Chosen by the haplotype count (more than 32: windows); GIRAFFE_B200_WINDOW_BUILDER=0|1 forces one.  A device build
    // (device >= 0, always from records) enumerates the windows on the GPU: only the sorted pair list comes from elsewhere.
    bool use_windows = n_paths > 32;
    if (const char* env = std::getenv("GIRAFFE_B200_WINDOW_BUILDER")) use_windows = std::atoi(env) != 0;
    if (records) use_windows = true;                   // there are no paths to scan
    const uint32_t W = k + w - 1;
    bool forward_only = true;                          // every haplotype stays on forward strands: forward starts cover every window
    if (use_windows && !external) {
        if (records) { for (uint32_t v = 2; v < ix->n_nodes && forward_only; v += 2) for (const auto& e : (*records)[v].edges) if (e.first & 1u) { forward_only = false; break; } }
        else for (uint32_t p = 0; p < n_paths && forward_only; p++) for (uint32_t v : seqs[2 * p]) if (v & 1u) { forward_only = false; break; }
    }
    if (use_windows && !external && device >= 0) {
        const int rc = gb::window_pairs_device(device, ix->nodes, ix->seq, ix->gbwt, k, w, forward_only, kps, counts);
        if (rc != GB_OK) { delete ix; return rc; }
        sorted = true;
    } else if (use_windows && !external) {
        // successors of a GBWT search state (node, [lo, hi]) in record order
        auto follow = [&](uint32_t v, int64_t lo, int64_t hi, std::vector<std::array<int64_t, 3>>& out) {
            out.clear();
            const gb_node_rec& nr = ix->nodes[v];
            if (nr.size == 0) return;
            const uint32_t* rec = ix->gbwt.data() + nr.rec_off;
            const uint32_t n_edges = rec[0], n_runs = rec[1];
            const uint32_t* runs = rec + 2 + 2 * n_edges;
            std::vector<int64_t> below(n_edges, 0), cnt(n_edges, 0);
            int64_t pos = 0;
            for (uint32_t r = 0; r < n_runs && pos <= hi; r++) {
                const int64_t len = runs[r] >> 10; const uint32_t e = runs[r] & 1023u;
                const int64_t b = pos, en = pos + len;
                below[e] += std::min<int64_t>(std::max<int64_t>(lo - b, 0), len);
                cnt[e] += std::max<int64_t>(std::min<int64_t>(en, hi + 1) - std::max<int64_t>(b, lo), 0);
                pos = en;
            }
            for (uint32_t e = 0; e < n_edges; e++) {
                const uint32_t to = rec[2 + 2 * e];
                if (to == 0 || cnt[e] <= 0) continue;
                const int64_t first = (int64_t)rec[3 + 2 * e] + below[e];
                out.push_back({(int64_t)to, first, first + cnt[e] - 1});
            }
        };
        std::string win; std::vector<uint32_t> wnode, woff;
        struct Frame { uint32_t node; int64_t lo, hi; size_t restore; };
        std::vector<Frame> stack; std::vector<std::array<int64_t, 3>> next;
        // Per start node: every haplotype-consistent continuation of W - 1 bases behind it.  The string node + continuation holds
        // exactly the windows that start on the node along that walk; its minimizers are computed once with the rolling hash.
        auto process = [&](size_t len) {
            mins.clear();
            gbmin::minimizers((const uint8_t*)win.data(), len, k, w, mins, nullptr);
            counts.continuations++; counts.raw_pairs += mins.size();
            for (const auto& m : mins) {
                uint32_t v = wnode[m.offset], o = woff[m.offset];
                if (m.is_reverse) { o = ix->nodes[v].len - 1 - o; v ^= 1u; }
                kps.push_back(KP{m.key, ((uint64_t)v << 10) | o});
            }
        };
        for (uint32_t v0 = 2; v0 < ix->n_nodes; v0++) {
            if (ix->nodes[v0].size == 0 || (forward_only && (v0 & 1u))) continue;
            counts.start_nodes++;
            const size_t need = (size_t)ix->nodes[v0].len + W - 1;
            stack.clear();
            stack.push_back(Frame{v0, 0, (int64_t)ix->nodes[v0].size - 1, 0});
            while (!stack.empty()) {
                const Frame f = stack.back(); stack.pop_back();
                win.resize(f.restore); wnode.resize(f.restore); woff.resize(f.restore);
                const gb_node_rec& nr = ix->nodes[f.node];
                for (uint32_t o = 0; o < nr.len && win.size() < need; o++) { win.push_back((char)ix->seq[nr.seq_off + o]); wnode.push_back(f.node); woff.push_back(o); }
                if (win.size() == need) { process(need); continue; }
                follow(f.node, f.lo, f.hi, next);
                if (next.empty()) { if (win.size() >= W) process(win.size()); continue; }          // the haplotypes end here
                for (size_t x = next.size(); x-- > 0;) stack.push_back(Frame{(uint32_t)next[x][0], next[x][1], next[x][2], win.size()});
            }
            if (kps.size() > (1ull << 26)) {      // keep the pair list bounded while it is full of duplicates
                std::sort(kps.begin(), kps.end(), [](const KP& a, const KP& b) { return a.key != b.key ? a.key < b.key : a.pos < b.pos; });
                kps.erase(std::unique(kps.begin(), kps.end(), [](const KP& a, const KP& b) { return a.key == b.key && a.pos == b.pos; }), kps.end());
            }
        }
    }
    for (uint32_t p = 0; p < n_paths && !external && !use_windows; p++) {
        hap.clear(); base_node.clear(); base_off.clear();
        for (uint32_t v : seqs[2 * p]) {
            const gb_node_rec& nr = ix->nodes[v];
            for (uint32_t o = 0; o < nr.len; o++) {
                hap.push_back((char)ix->seq[nr.seq_off + o]);
                base_node.push_back(v); base_off.push_back(o);
            }
        }
        mins.clear();
        gbmin::minimizers((const uint8_t*)hap.data(), hap.size(), k, w, mins, nullptr);
        counts.raw_pairs += mins.size();
        for (const auto& m : mins) {
            uint32_t v = base_node[m.offset], o = base_off[m.offset];
            if (m.is_reverse) { o = ix->nodes[v].len - 1 - o; v ^= 1u; }
            kps.push_back(KP{m.key, ((uint64_t)v << 10) | o});
        }
    }
    if (!sorted) {
        std::sort(kps.begin(), kps.end(), [](const KP& a, const KP& b) { return a.key != b.key ? a.key < b.key : a.pos < b.pos; });
        kps.erase(std::unique(kps.begin(), kps.end(), [](const KP& a, const KP& b) { return a.key == b.key && a.pos == b.pos; }), kps.end());
    }
    lap(ix->timing.minimizers_s);
    ix->timing.start_nodes = counts.start_nodes; ix->timing.continuations = counts.continuations;
    ix->timing.raw_pairs = external ? n_ext_hits : counts.raw_pairs; ix->timing.unique_pairs = kps.size();
    if (kps.size() > 0xfffffff0ull) { delete ix; return GB_ERR_FORMAT; }          // hit_off / hit_cnt are 32-bit
    size_t nkeys = 0;
    for (size_t i = 0; i < kps.size(); i++) if (i == 0 || kps[i].key != kps[i - 1].key) nkeys++;
    uint64_t cells = 16; while (cells < 2 * nkeys + 1) cells *= 2;
    ix->table.assign(cells, gb_min_cell{GB_NO_KEY, 0, 0});
    ix->hits.resize(kps.size());
    for (size_t i = 0; i < kps.size(); i++) {
        uint32_t v = (uint32_t)(kps[i].pos >> 10);
        ix->hits[i].pos = kps[i].pos;
        ix->hits[i].payload = ix->dist[v >> 1];
    }
    for (size_t i = 0; i < kps.size();) {
        size_t j = i; while (j < kps.size() && kps[j].key == kps[i].key) j++;
        uint64_t h = gbmin::hash64(kps[i].key) & (cells - 1);
        while (ix->table[h].key != GB_NO_KEY) h = (h + 1) & (cells - 1);
        ix->table[h] = gb_min_cell{kps[i].key, (uint32_t)i, (uint32_t)(j - i)};
        i = j;
    }
    lap(ix->timing.table_s);
    *out = ix;
    return GB_OK;
}

extern "C" int gb_index_build(uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off,
                              uint32_t n_paths, const uint32_t* path_nodes, const uint64_t* path_off,
                              const gb_dist_payload* dist, uint32_t k, uint32_t w,
                              gb_host_index** out) {
    return gb::guarded("gb_index_build", [&] { return index_build_impl(n_node_ids, node_seq, node_off, n_paths, path_nodes, path_off, dist, k, w, out); });
}

extern "C" int gb_index_build_with_hits(uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off,
                                        uint32_t n_paths, const uint32_t* path_nodes, const uint64_t* path_off,
                                        const gb_dist_payload* dist, uint32_t k, uint32_t w,
                                        uint64_t n_hits, const uint64_t* keys, const uint64_t* positions,
                                        gb_host_index** out) {
    static const uint64_t none = 0;
    if (n_hits == 0) { keys = keys ? keys : &none; positions = positions ? positions : &none; }
    return gb::guarded("gb_index_build_with_hits", [&] {
        return index_build_impl(n_node_ids, node_seq, node_off, n_paths, path_nodes, path_off, dist, k, w, out, n_hits, keys, positions);
    });
}

// The index from node sequences and a flat GBWT (the blob layout of gb_flat_index.gbwt) instead of haplotype paths: nothing here
// walks a haplotype, so the work follows the size of the graph, not haplotypes x genome.
int gb::index_build_from_gbwt(int device, uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off, uint32_t n_paths,
                              const uint32_t* gbwt_words, uint64_t n_words, const uint32_t* rec_off, const gb_dist_payload* dist,
                              uint32_t k, uint32_t w, uint64_t n_hits, const uint64_t* keys, const uint64_t* positions, gb_host_index** out) {
    if (!gbwt_words || !rec_off || !out || n_node_ids >= 0x7ffffff0u) return GB_ERR_ARG;
    if (device >= 0) {
        // the arguments index_build_impl refuses, before the device is touched
        if (!node_seq || !node_off || k == 0 || k > 31 || w == 0) return GB_ERR_ARG;
        if (const int rc = gb::device_ready(device)) return rc;
    }
    const size_t n_nodes = 2 * ((size_t)n_node_ids + 1);
    std::vector<GbwtRecordIn> records(n_nodes);
    for (size_t v = 2; v < n_nodes; v++) {
        const uint64_t off = rec_off[v];
        if (off == 0) continue;
        if (off + 2 > n_words) return GB_ERR_FORMAT;
        const uint64_t n_edges = gbwt_words[off], n_runs = gbwt_words[off + 1];
        if (n_edges >= 1024 || off + 2 + 2 * n_edges + n_runs > n_words) return GB_ERR_FORMAT;
        GbwtRecordIn& rc = records[v];
        for (uint64_t e = 0; e < n_edges; e++) rc.edges.push_back({gbwt_words[off + 2 + 2 * e], gbwt_words[off + 3 + 2 * e]});
        for (uint64_t r = 0; r < n_runs; r++) { const uint32_t wd = gbwt_words[off + 2 + 2 * n_edges + r]; rc.runs.push_back({wd & 1023u, (uint64_t)(wd >> 10)}); }
    }
    static const uint64_t none = 0;
    const bool ext = keys || positions;
    if (ext && n_hits == 0) { keys = keys ? keys : &none; positions = positions ? positions : &none; }
    return index_build_impl(n_node_ids, node_seq, node_off, n_paths, nullptr, nullptr, dist, k, w, out, n_hits, keys, positions, &records, device);
}

extern "C" int gb_index_build_from_gbwt(uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off, uint32_t n_paths,
                                        const uint32_t* gbwt_words, uint64_t n_words, const uint32_t* rec_off,
                                        const gb_dist_payload* dist, uint32_t k, uint32_t w,
                                        uint64_t n_hits, const uint64_t* keys, const uint64_t* positions, gb_host_index** out) {
    return gb::guarded("gb_index_build_from_gbwt", [&] {
        return gb::index_build_from_gbwt(-1, n_node_ids, node_seq, node_off, n_paths, gbwt_words, n_words, rec_off, dist, k, w, n_hits, keys, positions, out);
    });
}

extern "C" int gb_index_build_from_gbwt_device(uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off, uint32_t n_paths,
                                               const uint32_t* gbwt_words, uint64_t n_words, const uint32_t* rec_off,
                                               const gb_dist_payload* dist, uint32_t k, uint32_t w,
                                               uint64_t n_hits, const uint64_t* keys, const uint64_t* positions,
                                               int device_ordinal, gb_host_index** out) {
    return gb::guarded("gb_index_build_from_gbwt_device", [&] {
        if (device_ordinal < 0) return GB_ERR_ARG;
        return gb::index_build_from_gbwt(device_ordinal, n_node_ids, node_seq, node_off, n_paths, gbwt_words, n_words, rec_off, dist, k, w, n_hits, keys, positions, out);
    });
}

extern "C" int gb_index_build_timing(const gb_host_index* ix, gb_index_timing* out) {
    if (!ix || !out) return GB_ERR_ARG;
    *out = ix->timing;
    return GB_OK;
}

extern "C" void gb_index_free(gb_host_index* ix) { delete ix; }
extern "C" int gb_index_has_distance_model(const gb_host_index* ix) { return ix && ix->model_ok ? 1 : 0; }

extern "C" int gb_index_view(const gb_host_index* ix, gb_flat_index* out) {
    if (!ix || !out) return GB_ERR_ARG;
    out->n_nodes = ix->n_nodes; out->k = ix->k; out->w = ix->w; out->n_paths = ix->n_paths;
    out->nodes = ix->nodes.data();
    out->seq = ix->seq.data(); out->seq_bytes = ix->seq.size();
    out->gbwt = ix->gbwt.data(); out->gbwt_words = ix->gbwt.size();
    out->dist = ix->dist.data();
    out->table = ix->table.data(); out->table_cells = ix->table.size();
    out->hits = ix->hits.data(); out->n_hits = ix->hits.size();
    out->slots = ix->slots.data(); out->n_slots = ix->slots.size();
    out->site_dist = ix->site_dist.data(); out->site_dist_len = ix->site_dist.size();
    return GB_OK;
}

// ---- the flat index on disk ("GBZ-flat" file) ----------------------------------------------------------------
// What giraffe_main.cpp:1825-1881 does for GBZ / .min / .dist files, for the library's own layout: one file,
// a 64-byte header and the six arrays of gb_flat_index back to back, each padded to 16 bytes.  Little endian.
//   header: magic "GBFLAT2\0", n_nodes, k, w, n_paths (u32 each), seq_bytes, gbwt_words, table_cells, n_hits (u64 each), 8 B zero,
//           n_slots, site_dist_len (u64 each); then nodes, seq, gbwt, dist, table, hits, slots, site_dist
namespace {

struct FlatFileHeader {
    char magic[8];
    uint32_t n_nodes, k, w, n_paths;
    uint64_t seq_bytes, gbwt_words, table_cells, n_hits;
    uint64_t reserved;
    uint64_t n_slots, site_dist_len;
};
static_assert(sizeof(FlatFileHeader) == 80, "flat file header is 80 bytes");

bool write_padded(FILE* f, const void* p, size_t bytes) {
    static const char zero[16] = {0};
    if (bytes && fwrite(p, 1, bytes, f) != bytes) return false;
    const size_t pad = (16 - bytes % 16) % 16;
    return pad == 0 || fwrite(zero, 1, pad, f) == pad;
}
template <class T> bool read_padded(FILE* f, std::vector<T>& v, size_t count) {
    v.resize(count);
    const size_t bytes = count * sizeof(T);
    if (bytes && fread(v.data(), 1, bytes, f) != bytes) return false;
    const size_t pad = (16 - bytes % 16) % 16;
    char skip[16];
    return pad == 0 || fread(skip, 1, pad, f) == pad;
}

} // namespace

extern "C" int gb_index_save(const gb_flat_index* ix, const char* path) {
    if (!ix || !path) return GB_ERR_ARG;
    FILE* f = fopen(path, "wb");
    if (!f) return GB_ERR_FORMAT;
    FlatFileHeader h; memset(&h, 0, sizeof h);
    memcpy(h.magic, "GBFLAT2", 8);
    h.n_nodes = ix->n_nodes; h.k = ix->k; h.w = ix->w; h.n_paths = ix->n_paths;
    h.seq_bytes = ix->seq_bytes; h.gbwt_words = ix->gbwt_words; h.table_cells = ix->table_cells; h.n_hits = ix->n_hits;
    h.n_slots = ix->n_slots; h.site_dist_len = ix->site_dist_len;
    bool ok = fwrite(&h, 1, sizeof h, f) == sizeof h
        && write_padded(f, ix->nodes, (size_t)ix->n_nodes * sizeof(gb_node_rec))
        && write_padded(f, ix->seq, ix->seq_bytes)
        && write_padded(f, ix->gbwt, ix->gbwt_words * 4)
        && write_padded(f, ix->dist, (size_t)(ix->n_nodes / 2) * sizeof(gb_dist_payload))
        && write_padded(f, ix->table, ix->table_cells * sizeof(gb_min_cell))
        && write_padded(f, ix->hits, ix->n_hits * sizeof(gb_hit))
        && write_padded(f, ix->slots, ix->n_slots * sizeof(gb_slot_rec))
        && write_padded(f, ix->site_dist, ix->site_dist_len * sizeof(uint16_t));
    ok = (fclose(f) == 0) && ok;
    return ok ? GB_OK : GB_ERR_FORMAT;
}

static int index_load_impl(const char* path, gb_host_index** out) {
    if (!path || !out) return GB_ERR_ARG;
    *out = nullptr;
    FILE* f = fopen(path, "rb");
    if (!f) return GB_ERR_FORMAT;
    FlatFileHeader h;
    if (fread(&h, 1, sizeof h, f) != sizeof h || memcmp(h.magic, "GBFLAT2", 8) != 0) { fclose(f); return GB_ERR_FORMAT; }
    // plausibility before allocating: a power-of-two table, an even number of oriented nodes, sizes the file can hold
    fseek(f, 0, SEEK_END); const uint64_t file_bytes = (uint64_t)ftell(f); fseek(f, (long)sizeof h, SEEK_SET);
    // every count is bounded by the file size on its own first (a crafted header must not wrap the sum), then the sum
    const bool counts_ok = h.seq_bytes <= file_bytes && h.gbwt_words <= file_bytes / 4 && h.table_cells <= file_bytes / sizeof(gb_min_cell)
                        && h.n_hits <= file_bytes / sizeof(gb_hit) && (uint64_t)h.n_nodes <= file_bytes / sizeof(gb_node_rec)
                        && h.n_slots <= file_bytes / sizeof(gb_slot_rec) && h.site_dist_len <= file_bytes / sizeof(uint16_t);
    const uint64_t need = !counts_ok ? ~0ull : (uint64_t)h.n_nodes * sizeof(gb_node_rec) + h.seq_bytes + h.gbwt_words * 4 + (uint64_t)(h.n_nodes / 2) * sizeof(gb_dist_payload)
                        + h.table_cells * sizeof(gb_min_cell) + h.n_hits * sizeof(gb_hit) + h.n_slots * sizeof(gb_slot_rec) + h.site_dist_len * sizeof(uint16_t);
    if (!counts_ok || h.n_nodes % 2 != 0 || h.n_nodes < 2 || h.table_cells == 0 || (h.table_cells & (h.table_cells - 1)) != 0 || h.k == 0 || h.k > 31 || h.w == 0
        || h.seq_bytes < 16 || h.seq_bytes > 0xffffffffull || h.gbwt_words > 0xffffffffull || h.n_hits > 0xffffffffull || need > file_bytes) { fclose(f); return GB_ERR_FORMAT; }
    gb_host_index* ix = new gb_host_index();
    ix->n_nodes = h.n_nodes; ix->k = h.k; ix->w = h.w; ix->n_paths = h.n_paths;
    const bool ok = read_padded(f, ix->nodes, h.n_nodes) && read_padded(f, ix->seq, h.seq_bytes) && read_padded(f, ix->gbwt, h.gbwt_words)
                 && read_padded(f, ix->dist, h.n_nodes / 2) && read_padded(f, ix->table, h.table_cells) && read_padded(f, ix->hits, h.n_hits)
                 && read_padded(f, ix->slots, h.n_slots) && read_padded(f, ix->site_dist, h.site_dist_len);
    fclose(f);
    if (!ok) { delete ix; return GB_ERR_FORMAT; }
    // offsets must stay inside the arrays (a truncated or foreign file must not make the kernels read out of bounds)
    // the kernels read 16 bytes past a node's last base (vector loads): the sequence keeps >= 16 zero bytes of tail padding
    for (uint64_t i = h.seq_bytes - 16; i < h.seq_bytes; i++) if (ix->seq[i] != 0) { delete ix; return GB_ERR_FORMAT; }
    for (const gb_node_rec& r : ix->nodes) {
        if ((uint64_t)r.seq_off + r.len + 16 > h.seq_bytes || r.len > 1024) { delete ix; return GB_ERR_FORMAT; }
        if (r.size == 0) continue;
        // GBWT record: n_edges, n_runs, n_edges x {to, offset}, n_runs x {(len << 10) | outrank}; everything inside the blob
        if ((uint64_t)r.rec_off + 2 > h.gbwt_words) { delete ix; return GB_ERR_FORMAT; }
        const uint32_t* rec = ix->gbwt.data() + r.rec_off;
        const uint64_t n_edges = rec[0], n_runs = rec[1];
        if ((uint64_t)r.rec_off + 2 + 2 * n_edges + n_runs > h.gbwt_words) { delete ix; return GB_ERR_FORMAT; }
        for (uint64_t e = 0; e < n_edges; e++) if (rec[2 + 2 * e] >= h.n_nodes) { delete ix; return GB_ERR_FORMAT; }
        for (uint64_t t = 0; t < n_runs; t++) if ((rec[2 + 2 * n_edges + t] & 1023u) >= n_edges) { delete ix; return GB_ERR_FORMAT; }
    }
    // a hit carries its node's distance payload (the seeding kernels take two seeds on one node to share x_in)
    for (const gb_hit& hit : ix->hits)
        if ((hit.pos >> 10) >= h.n_nodes || memcmp(&hit.payload, &ix->dist[hit.pos >> 11], sizeof(gb_dist_payload)) != 0) { delete ix; return GB_ERR_FORMAT; }
    // slot tables stay inside site_dist, and a node that claims a place in a site table really has one
    for (const gb_slot_rec& sr : ix->slots)
        if (sr.table_off != 0xFFFFFFFFu && (uint64_t)sr.table_off + (uint64_t)sr.n * sr.n > h.site_dist_len) { delete ix; return GB_ERR_FORMAT; }
    if (h.n_slots) for (const gb_dist_payload& dp : ix->dist)
        if (dp.allele != 0xFFFF && dp.slot < h.n_slots && ix->slots[dp.slot].table_off != 0xFFFFFFFFu && dp.allele >= ix->slots[dp.slot].n) { delete ix; return GB_ERR_FORMAT; }
    for (const gb_min_cell& c : ix->table)
        if (c.key != GB_NO_KEY && (uint64_t)c.hit_off + c.hit_cnt > h.n_hits) { delete ix; return GB_ERR_FORMAT; }
    *out = ix;
    return GB_OK;
}

extern "C" int gb_index_load(const char* path, gb_host_index** out) {
    return gb::guarded("gb_index_load", GB_ERR_FORMAT, [&] { return index_load_impl(path, out); }, [&] { if (out) *out = nullptr; });
}
