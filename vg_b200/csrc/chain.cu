// chain.cu — stage seam of the chaining route: algorithms::find_best_chains (algorithms/chain_items.hpp:576,
// chain_items.cpp:733-900) = add_transition_if_legal (:262-355) + chain_items_dp (:384-640) + chain_items_traceback
// (:642-735), called by minimizer_mapper_from_chains.cpp:1201 (fragments) and :1933 (chains).
//
// One WARP per chaining problem, problems taken from a work counter (sizes vary by orders of magnitude).
//   1. candidates -> transitions: the lanes filter the candidates (read distance, exclusion zones, hint offsets, indel
//      bound) and a counting sort groups the survivors by DESTINATION anchor (count, warp prefix sum, scatter).
//   2. the DP, destinations in read order.  The reference walks one sorted transition list and updates
//      chain_scores[to] whenever (evaluation value, score, source) grows lexicographically (:541-552; TracedScore's
//      operator> is (score, source), chain_items.hpp:338).  All sources of a destination start earlier in the read,
//      so their cells are final when the destination is reached, and a running lexicographic maximum does not depend
//      on the order of its operands: the lanes evaluate 32 incoming transitions at a time, a shuffle reduction picks
//      the maximum (with "from nowhere" as one more operand, source = +infinity), one lane writes the cell.
//   3. best cell (first maximum, TracedScore::max_in :47-56), traceback starts ordered by (score, source) descending
//      (rank sort across the lanes), the pointer walk of chain_items_traceback on one lane (it is a chain of
//      dependent loads over every anchor exactly once), then max_chains selections of the smallest penalty.
// The minimap2-style gap cost (:364-372) is evaluated in FP64 exactly as the host does: 0.5 * log2(d) comes from a
// table built with the host libm, the product and the sum are separate IEEE operations (no FMA contraction).
#include <cub/cub.cuh>
#include "giraffe_b200.h"
#include "device_state.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <new>
#include <vector>

namespace gb {

constexpr uint32_t CHAIN_NOWHERE = 0xffffffffu;
constexpr uint32_t CHAIN_WARPS = 4;
constexpr unsigned CH_FULL = 0xffffffffu;

struct ChainBatch {
    uint32_t n_problems;
    const gb_chain_anchor* anchors; const uint64_t* anchor_off;
    const gb_chain_candidate* cands; const uint64_t* cand_off;
    const double* half_log2;            // [max_indel_bases + 1], host libm
    int32_t item_bonus, recombination_penalty, consistency_bonus; uint32_t max_chains;
    double gap_scale; uint64_t max_indel_bases, max_read_lookback_bases;
    // per anchor
    int32_t* dp_score; uint32_t* dp_source; uint64_t* dp_paths; uint32_t* dp_rec;
    uint32_t* in_begin; uint32_t* in_cursor;         // transitions into the anchor: [in_begin[i], in_begin[i + 1]) after step 1
    uint32_t* order;                                 // traceback starts in score order
    uint32_t* tb_items; uint32_t* tb_begin; uint32_t* tb_count; int32_t* tb_penalty;   // tracebacks (right to left), by creation order
    uint8_t* used;
    // per candidate
    uint32_t* legal_indel;                           // indel of a legal candidate, 0xffffffff otherwise
    uint32_t* t_from; uint32_t* t_indel;             // transitions grouped by destination
    // outputs
    uint32_t* n_chains; int32_t* chain_score; uint32_t* chain_begin; uint32_t* chain_count; uint32_t* chain_items;
    uint32_t* work_counter;
};

__device__ __forceinline__ int chain_gap(const ChainBatch& b, uint32_t indel, uint64_t base_seed_length) {
    if (indel == 0) return 0;
    const double prod = __dmul_rn(__dmul_rn(0.01, (double)base_seed_length), (double)indel);
    return (int)__dadd_rn(prod, b.half_log2[indel]);
}

__global__ void __launch_bounds__(CHAIN_WARPS * 32) chain_kernel(ChainBatch b) {
    const int lane = threadIdx.x & 31;
    while (true) {
        uint32_t p = 0;
        if (lane == 0) p = atomicAdd(b.work_counter, 1u);
        p = __shfl_sync(CH_FULL, p, 0);
        if (p >= b.n_problems) return;
        const uint64_t a0 = b.anchor_off[p], c0 = b.cand_off[p];
        const uint32_t n = (uint32_t)(b.anchor_off[p + 1] - a0);
        const uint64_t m = b.cand_off[p + 1] - c0;
        const gb_chain_anchor* A = b.anchors + a0;
        const gb_chain_candidate* C = b.cands + c0;
        if (n == 0) { if (lane == 0) b.n_chains[p] = 0; continue; }

        // ---- base seed length (:408-412), incoming-transition counts ----
        uint64_t bsl = 0;
        for (uint32_t i = lane; i < n; i += 32) { bsl += A[i].base_seed_length; b.in_cursor[a0 + i] = 0; b.used[a0 + i] = 0; }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) bsl += __shfl_xor_sync(CH_FULL, bsl, d);
        bsl /= n;
        __syncwarp();
        // ---- add_transition_if_legal (:262-355) ----
        for (uint64_t c = lane; c < m; c += 32) {
            const gb_chain_candidate cd = C[c];
            const gb_chain_anchor s = A[cd.from], t = A[cd.to];
            uint32_t indel = 0xffffffffu;
            const uint64_t s_end = (uint64_t)s.read_start + s.length;
            if (t.read_start >= s_end) {
                const uint64_t read_distance = t.read_start - s_end;
                const uint64_t remove = (uint64_t)t.start_hint_offset + s.end_hint_offset;
                if (read_distance <= b.max_read_lookback_bases &&
                    s_end + s.margin_after <= (uint64_t)t.read_start - t.margin_before &&
                    remove <= cd.graph_distance) {
                    const uint64_t g = cd.graph_distance - remove;
                    const uint64_t diff = read_distance > g ? read_distance - g : g - read_distance;
                    if (diff <= b.max_indel_bases) { indel = (uint32_t)diff; atomicAdd(&b.in_cursor[a0 + cd.to], 1u); }
                }
            }
            b.legal_indel[c0 + c] = indel;
        }
        __syncwarp();
        // ---- exclusive prefix sum of the counts -> group starts ----
        uint32_t carry = 0;
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t i = base + lane;
            const uint32_t cnt = i < n ? b.in_cursor[a0 + i] : 0u;
            uint32_t incl = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t up = __shfl_up_sync(CH_FULL, incl, d); if (lane >= d) incl += up; }
            if (i < n) { b.in_begin[a0 + i] = carry + incl - cnt; b.in_cursor[a0 + i] = carry + incl - cnt; }
            carry += __shfl_sync(CH_FULL, incl, 31);
        }
        const uint32_t n_trans = carry;
        __syncwarp();
        for (uint64_t c = lane; c < m; c += 32) {
            const uint32_t indel = b.legal_indel[c0 + c];
            if (indel != 0xffffffffu) {
                const gb_chain_candidate cd = C[c];
                const uint32_t slot = atomicAdd(&b.in_cursor[a0 + cd.to], 1u);
                b.t_from[c0 + slot] = cd.from; b.t_indel[c0 + slot] = indel;
            }
        }
        __syncwarp();

        // ---- chain_items_dp (:384-640): destinations in read order ----
        for (uint32_t i = 0; i < n; i++) {
            const gb_chain_anchor here = A[i];
            const int item_points = here.score + b.item_bonus;
            // every lane starts from "from nowhere" (:414-418, :441-456)
            int best_eval = item_points + b.consistency_bonus, best_score = item_points;
            uint32_t best_source = CHAIN_NOWHERE, best_rec = 0; uint64_t best_paths = here.end_paths;
            const uint32_t tb = b.in_begin[a0 + i], te = (i + 1 < n) ? b.in_begin[a0 + i + 1] : n_trans;
            for (uint32_t t = tb + lane; t < te; t += 32) {
                const uint32_t from = b.t_from[c0 + t];
                const int s_score = b.dp_score[a0 + from]; const uint64_t s_paths = b.dp_paths[a0 + from]; const uint32_t s_rec = b.dp_rec[a0 + from];
                int jump_points = (int)((double)(-chain_gap(b, b.t_indel[c0 + t], bsl)) * b.gap_scale);
                if ((s_paths & here.start_paths) == 0) jump_points -= b.recombination_penalty;          // check_recombination :376-382
                const int score = s_score + jump_points + item_points;
                uint64_t paths; uint32_t rec = s_rec;                                                    // set_shared_paths :69-96
                if (here.start_paths == here.end_paths) {
                    if ((s_paths & here.start_paths) == 0) { paths = here.start_paths; rec++; }
                    else paths = s_paths & here.start_paths;
                } else paths = here.end_paths;
                int bonus = 0;
                if (b.consistency_bonus > 0) {
                    const int pre = __popcll(s_paths);
                    if (pre > 0 && (s_paths & here.start_paths) != 0) bonus = (b.consistency_bonus * __popcll(paths)) / pre;
                }
                const int ev = score + bonus;
                if (ev > best_eval || (ev == best_eval && (score > best_score || (score == best_score && from > best_source)))) {
                    best_eval = ev; best_score = score; best_source = from; best_paths = paths; best_rec = rec;
                }
            }
            // lexicographic maximum of (eval, score, source) over the lanes
            int r_eval = best_eval, r_score = best_score; uint32_t r_source = best_source;
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) {
                const int oe = __shfl_xor_sync(CH_FULL, r_eval, d), os = __shfl_xor_sync(CH_FULL, r_score, d);
                const uint32_t osrc = __shfl_xor_sync(CH_FULL, r_source, d);
                if (oe > r_eval || (oe == r_eval && (os > r_score || (os == r_score && osrc > r_source)))) { r_eval = oe; r_score = os; r_source = osrc; }
            }
            const unsigned holders = __ballot_sync(CH_FULL, best_eval == r_eval && best_score == r_score && best_source == r_source);
            if (lane == __ffs(holders) - 1) {
                b.dp_score[a0 + i] = best_score; b.dp_source[a0 + i] = best_source; b.dp_paths[a0 + i] = best_paths; b.dp_rec[a0 + i] = best_rec;
            }
            __syncwarp();
        }

        // ---- best cell: the first maximum (TracedScore::max_in :47-56) ----
        int top = INT_MIN; uint32_t top_i = 0xffffffffu;
        for (uint32_t i = lane; i < n; i += 32) { const int s = b.dp_score[a0 + i]; if (s > top) { top = s; top_i = i; } }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const int os = __shfl_xor_sync(CH_FULL, top, d); const uint32_t oi = __shfl_xor_sync(CH_FULL, top_i, d);
            if (os > top || (os == top && oi < top_i)) { top = os; top_i = oi; }
        }
        const int best_total = top;

        // ---- traceback starts by (score, source) descending, index ascending (rank sort) ----
        for (uint32_t i = lane; i < n; i += 32) {
            const int si = b.dp_score[a0 + i]; const uint32_t ri = b.dp_source[a0 + i];
            uint32_t rank = 0;
            for (uint32_t j = 0; j < n; j++) {
                const int sj = b.dp_score[a0 + j]; const uint32_t rj = b.dp_source[a0 + j];
                const bool j_first = sj > si || (sj == si && (rj > ri || (rj == ri && j < i)));
                rank += j_first ? 1u : 0u;
            }
            b.order[a0 + rank] = i;
        }
        __syncwarp();

        // ---- chain_items_traceback (:642-735): one lane, every anchor visited once ----
        uint32_t n_tb = 0;
        if (lane == 0) {
            uint32_t w = 0;
            for (uint32_t k = 0; k < n; k++) {
                const uint32_t trace_from = b.order[a0 + k];
                if (b.used[a0 + trace_from]) continue;
                const uint32_t begin = w;
                b.tb_items[a0 + w++] = trace_from;
                int penalty = best_total - b.dp_score[a0 + trace_from];
                uint32_t here = trace_from;
                while (here != CHAIN_NOWHERE) {
                    b.used[a0 + here] = 1;
                    const uint32_t next = b.dp_source[a0 + here];
                    if (next != CHAIN_NOWHERE) {
                        if (b.used[a0 + next]) {
                            penalty += b.dp_score[a0 + here];
                            penalty -= A[here].score + b.item_bonus;
                            break;
                        }
                        b.tb_items[a0 + w++] = next;
                    }
                    here = next;
                }
                b.tb_begin[a0 + n_tb] = begin; b.tb_count[a0 + n_tb] = w - begin; b.tb_penalty[a0 + n_tb] = penalty;
                n_tb++;
            }
        }
        n_tb = __shfl_sync(CH_FULL, n_tb, 0);
        __syncwarp();

        // ---- the max_chains smallest penalties, earlier traceback first among equals; score = best - penalty (:780-800) ----
        const uint32_t n_out = min(n_tb, b.max_chains);
        uint32_t w_out = 0;
        for (uint32_t c = 0; c < n_out; c++) {
            int pen = INT_MAX; uint32_t which = 0xffffffffu;
            for (uint32_t t = lane; t < n_tb; t += 32) {
                const uint32_t cnt = b.tb_count[a0 + t];
                if (cnt & 0x80000000u) continue;                                   // already taken
                const int q = b.tb_penalty[a0 + t];
                if (q < pen) { pen = q; which = t; }
            }
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) {
                const int oq = __shfl_xor_sync(CH_FULL, pen, d); const uint32_t ot = __shfl_xor_sync(CH_FULL, which, d);
                if (oq < pen || (oq == pen && ot < which)) { pen = oq; which = ot; }
            }
            const uint32_t begin = b.tb_begin[a0 + which], cnt = b.tb_count[a0 + which];
            __syncwarp();
            for (uint32_t x = lane; x < cnt; x += 32) b.chain_items[a0 + w_out + x] = b.tb_items[a0 + begin + cnt - 1 - x];     // left to right
            if (lane == 0) {
                const size_t o = (size_t)p * b.max_chains + c;
                b.chain_score[o] = best_total - pen; b.chain_begin[o] = (uint32_t)(a0 + w_out); b.chain_count[o] = cnt;
                b.tb_count[a0 + which] = cnt | 0x80000000u;
            }
            w_out += cnt;
            __syncwarp();
        }
        if (lane == 0) b.n_chains[p] = n_out;
    }
}

// ---- candidates: every (source, destination) pair of seeds within the lookback, with its minimum graph distance -------------
// One warp per DESTINATION seed; the lanes take the sources of the same problem 32 at a time.  Two passes: count, then (after
// an exclusive scan over all seeds) fill — so the output is dense and sorted by (destination, source) without atomics.
struct CandBatch {
    uint32_t n_seeds; const uint32_t* pos; const uint32_t* prob_begin; const uint32_t* prob_end;    // per seed: its problem's seed range
    uint64_t limit; uint64_t* count; const uint64_t* offset; gb_chain_candidate* out;
};
template <bool FILL>
__global__ void __launch_bounds__(128) chain_candidates_kernel(DevIndex ix, CandBatch b) {
    const int lane = threadIdx.x & 31;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < b.n_seeds; j += warps) {
        const uint32_t a0 = b.prob_begin[j], a1 = b.prob_end[j];
        const uint32_t nj = b.pos[2 * j], oj = b.pos[2 * j + 1];
        uint64_t n = 0;
        const uint64_t base = FILL ? b.offset[j] : 0;
        for (uint32_t i0 = a0; i0 < a1; i0 += 32) {
            const uint32_t i = i0 + lane;
            int64_t d = -1;
            if (i < a1 && i != j) d = oriented_distance(ix, b.pos[2 * i], b.pos[2 * i + 1], nj, oj);
            const bool hit = d >= 0 && (uint64_t)d <= b.limit;
            const unsigned m = __ballot_sync(0xffffffffu, hit);
            if (FILL && hit) {
                gb_chain_candidate c; c.from = i - a0; c.to = j - a0; c.graph_distance = (uint64_t)d;
                b.out[base + n + __popc(m & ((1u << lane) - 1u))] = c;
            }
            n += __popc(m);
        }
        if (!FILL && lane == 0) b.count[j] = n;
    }
}

} // namespace gb

using namespace gb;

extern "C" void gb_chain_params_default(gb_chain_params* p) {
    if (!p) return;
    p->item_bonus = 0; p->recombination_penalty = 0; p->consistency_bonus = 0; p->max_chains = 1; p->gap_scale = 1.0;
    p->max_indel_bases = 100; p->max_read_lookback_bases = ~0ull;                  // chain_items.hpp:407-418, :583-584
}

static int chain_batch_impl(gb_device* d, const gb_chain_params* P, uint32_t n_problems,
                            const gb_chain_anchor* anchors, const uint64_t* anchor_off,
                            const gb_chain_candidate* cands, const uint64_t* cand_off,
                            int32_t* dp_score, uint32_t* dp_source, uint64_t* dp_paths, uint32_t* dp_rec,
                            uint32_t* n_chains, int32_t* chain_score, uint32_t* chain_begin, uint32_t* chain_count, uint32_t* chain_items,
                            uint32_t* candidate_indel) {
    if (!d || !P || !anchor_off || !cand_off || !n_chains || !chain_score || !chain_begin || !chain_count) return GB_ERR_ARG;
    if (P->max_chains == 0 || P->max_indel_bases > 65535 || P->recombination_penalty < 0 || P->consistency_bonus < 0) { g_last_error = "gb_chain_batch: parameters out of range"; return GB_ERR_ARG; }
    if (n_problems == 0) return GB_OK;
    const uint64_t total_a = anchor_off[n_problems], total_c = cand_off[n_problems];
    if (total_a >= 0xfffffff0ull || total_c >= 0xfffffff0ull) return GB_ERR_ARG;
    if (total_a && (!anchors || !dp_score || !dp_source || !dp_paths || !dp_rec || !chain_items)) return GB_ERR_ARG;
    if (total_c && !cands) return GB_ERR_ARG;
    for (uint32_t p = 0; p < n_problems; p++) {
        if (anchor_off[p + 1] < anchor_off[p] || cand_off[p + 1] < cand_off[p]) return GB_ERR_ARG;
        const uint64_t a0 = anchor_off[p], n = anchor_off[p + 1] - a0;
        // the traceback starts are ordered by a rank sort (n^2 / 32 steps per warp): bound the problem so one call cannot run for minutes
        if (n > GB_CHAIN_MAX_ANCHORS) { g_last_error = "gb_chain_batch: more than GB_CHAIN_MAX_ANCHORS anchors in one problem"; return GB_ERR_ARG; }
        for (uint64_t i = 0; i < n; i++) {
            const gb_chain_anchor& a = anchors[a0 + i];
            // the DP visits destinations in index order: anchors must come sorted by read start, and an anchor covers >= 1 base
            if (a.length == 0 || a.margin_before > a.read_start || (i && a.read_start < anchors[a0 + i - 1].read_start)) {
                g_last_error = "gb_chain_batch: anchors must be sorted by read_start, non-empty, with margins inside the read"; return GB_ERR_ARG;
            }
        }
        for (uint64_t c = cand_off[p]; c < cand_off[p + 1]; c++)
            if (cands[c].from >= n || cands[c].to >= n) { g_last_error = "gb_chain_batch: candidate names an anchor outside its problem"; return GB_ERR_ARG; }
    }
    GB_CUDA(cudaSetDevice(d->device));
    std::vector<double> hl(P->max_indel_bases + 1, 0.0);
    for (uint64_t x = 1; x <= P->max_indel_bases; x++) hl[x] = 0.5 * std::log2((double)x);
    const size_t na = total_a ? total_a : 1, nc = total_c ? total_c : 1, nk = (size_t)n_problems * P->max_chains;
    DevBuf<gb_chain_anchor> d_anch; DevBuf<gb_chain_candidate> d_cand; DevBuf<uint64_t> d_aoff, d_coff, d_paths; DevBuf<double> d_hl;
    DevBuf<int32_t> d_score, d_pen, d_cscore; DevBuf<uint32_t> d_source, d_rec, d_begin, d_cursor, d_order, d_items, d_tbb, d_tbc, d_legal, d_from, d_indel, d_nch, d_cbegin, d_ccount, d_citems, d_counter;
    DevBuf<uint8_t> d_used;
    int rc;
    if ((rc = d_anch.upload(anchors, na, d->stream, total_a)) || (rc = d_cand.upload(cands, nc, d->stream, total_c)) ||
        (rc = d_aoff.upload(anchor_off, n_problems + 1, d->stream)) || (rc = d_coff.upload(cand_off, n_problems + 1, d->stream)) ||
        (rc = d_hl.upload(hl.data(), hl.size(), d->stream))) return rc;
    if ((rc = d_score.reserve(na)) || (rc = d_source.reserve(na)) || (rc = d_paths.reserve(na)) || (rc = d_rec.reserve(na)) || (rc = d_begin.reserve(na)) ||
        (rc = d_cursor.reserve(na)) || (rc = d_order.reserve(na)) || (rc = d_items.reserve(na)) || (rc = d_tbb.reserve(na)) || (rc = d_tbc.reserve(na)) ||
        (rc = d_pen.reserve(na)) || (rc = d_used.reserve(na)) || (rc = d_citems.reserve(na)) ||
        (rc = d_legal.reserve(nc)) || (rc = d_from.reserve(nc)) || (rc = d_indel.reserve(nc)) ||
        (rc = d_nch.reserve(n_problems)) || (rc = d_cscore.reserve(nk)) || (rc = d_cbegin.reserve(nk)) || (rc = d_ccount.reserve(nk)) || (rc = d_counter.reserve(4))) return rc;
    GB_CUDA(cudaMemsetAsync(d_counter.ptr, 0, 16, d->stream));
    GB_CUDA(cudaMemsetAsync(d_cscore.ptr, 0, 4 * nk, d->stream));
    GB_CUDA(cudaMemsetAsync(d_cbegin.ptr, 0, 4 * nk, d->stream));
    GB_CUDA(cudaMemsetAsync(d_ccount.ptr, 0, 4 * nk, d->stream));
    GB_CUDA(cudaMemsetAsync(d_citems.ptr, 0, 4 * na, d->stream));
    ChainBatch b;
    b.n_problems = n_problems; b.anchors = d_anch.ptr; b.anchor_off = d_aoff.ptr; b.cands = d_cand.ptr; b.cand_off = d_coff.ptr; b.half_log2 = d_hl.ptr;
    b.item_bonus = P->item_bonus; b.recombination_penalty = P->recombination_penalty; b.consistency_bonus = P->consistency_bonus; b.max_chains = P->max_chains;
    b.gap_scale = P->gap_scale; b.max_indel_bases = P->max_indel_bases; b.max_read_lookback_bases = P->max_read_lookback_bases;
    b.dp_score = d_score.ptr; b.dp_source = d_source.ptr; b.dp_paths = d_paths.ptr; b.dp_rec = d_rec.ptr; b.in_begin = d_begin.ptr; b.in_cursor = d_cursor.ptr;
    b.order = d_order.ptr; b.tb_items = d_items.ptr; b.tb_begin = d_tbb.ptr; b.tb_count = d_tbc.ptr; b.tb_penalty = d_pen.ptr; b.used = d_used.ptr;
    b.legal_indel = d_legal.ptr; b.t_from = d_from.ptr; b.t_indel = d_indel.ptr;
    b.n_chains = d_nch.ptr; b.chain_score = d_cscore.ptr; b.chain_begin = d_cbegin.ptr; b.chain_count = d_ccount.ptr; b.chain_items = d_citems.ptr;
    b.work_counter = d_counter.ptr;
    const uint32_t grid = std::max<uint32_t>(1u, std::min<uint32_t>((uint32_t)d->n_sms * 8, (n_problems + CHAIN_WARPS - 1) / CHAIN_WARPS));
    GB_CUDA(cudaEventRecord(d->ev0, d->stream));
    chain_kernel<<<grid, CHAIN_WARPS * 32, 0, d->stream>>>(b);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaEventRecord(d->ev1, d->stream));
    if (total_a) {
        GB_CUDA(cudaMemcpyAsync(dp_score, d_score.ptr, 4 * total_a, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(dp_source, d_source.ptr, 4 * total_a, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(dp_paths, d_paths.ptr, 8 * total_a, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(dp_rec, d_rec.ptr, 4 * total_a, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaMemcpyAsync(chain_items, d_citems.ptr, 4 * total_a, cudaMemcpyDeviceToHost, d->stream));
    }
    if (candidate_indel && total_c) GB_CUDA(cudaMemcpyAsync(candidate_indel, d_legal.ptr, 4 * total_c, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(n_chains, d_nch.ptr, 4 * (size_t)n_problems, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(chain_score, d_cscore.ptr, 4 * nk, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(chain_begin, d_cbegin.ptr, 4 * nk, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaMemcpyAsync(chain_count, d_ccount.ptr, 4 * nk, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));
    GB_CUDA(cudaEventElapsedTime(&d->last_kernel_ms, d->ev0, d->ev1));
    return GB_OK;
}

extern "C" int gb_chain_batch(gb_device* d, const gb_chain_params* P, uint32_t n_problems,
                              const gb_chain_anchor* anchors, const uint64_t* anchor_off,
                              const gb_chain_candidate* cands, const uint64_t* cand_off,
                              int32_t* dp_score, uint32_t* dp_source, uint64_t* dp_paths, uint32_t* dp_rec,
                              uint32_t* n_chains, int32_t* chain_score, uint32_t* chain_begin, uint32_t* chain_count, uint32_t* chain_items) {
    return gb::guarded("gb_chain_batch", [&] {
        return chain_batch_impl(d, P, n_problems, anchors, anchor_off, cands, cand_off, dp_score, dp_source, dp_paths, dp_rec,
                                n_chains, chain_score, chain_begin, chain_count, chain_items, nullptr);
    });
}

extern "C" int gb_chain_batch_transitions(gb_device* d, const gb_chain_params* P, uint32_t n_problems,
                                          const gb_chain_anchor* anchors, const uint64_t* anchor_off,
                                          const gb_chain_candidate* cands, const uint64_t* cand_off,
                                          int32_t* dp_score, uint32_t* dp_source, uint64_t* dp_paths, uint32_t* dp_rec,
                                          uint32_t* n_chains, int32_t* chain_score, uint32_t* chain_begin, uint32_t* chain_count, uint32_t* chain_items,
                                          uint32_t* candidate_indel) {
    return gb::guarded("gb_chain_batch_transitions", [&] {
        return chain_batch_impl(d, P, n_problems, anchors, anchor_off, cands, cand_off, dp_score, dp_source, dp_paths, dp_rec,
                                n_chains, chain_score, chain_begin, chain_count, chain_items, candidate_indel);
    });
}

// MinimizerMapper::to_anchor, minimizer_mapper_from_chains.cpp:3978-4038 (host side: a few integer operations per seed)
extern "C" int gb_chain_anchors(const gb_flat_index* ix, const gb_scores* scores, uint32_t n, const uint32_t* seed_pos,
                                const uint32_t* min_offset, const uint8_t* min_is_reverse, const uint32_t* min_length,
                                const uint64_t* paths, gb_chain_anchor* out) {
    return gb::guarded("gb_chain_anchors", [&] {
        if (!ix || !scores || (n && (!seed_pos || !min_offset || !min_is_reverse || !min_length || !out))) return GB_ERR_ARG;
        for (uint32_t i = 0; i < n; i++) {
            const uint32_t v = seed_pos[2 * i], off = seed_pos[2 * i + 1], mlen = min_length[i];
            if (v < 2 || v >= ix->n_nodes || ix->nodes[v].len == 0 || off >= ix->nodes[v].len || mlen == 0) { g_last_error = "gb_chain_anchors: seed outside the graph or empty minimizer"; return GB_ERR_ARG; }
            uint32_t length, margin_left, margin_right, read_start, hint_start;
            if (min_is_reverse[i]) {
                const uint32_t end = off + 1;                              // the seed is the final base of the match: past-end position
                length = std::min(mlen, end);                              // how much of the node lies before it
                margin_left = mlen - length; margin_right = 0;
                if (min_offset[i] + 1 < length) { g_last_error = "gb_chain_anchors: reverse minimizer runs off the read start"; return GB_ERR_ARG; }
                read_start = min_offset[i] + 1 - length;
                hint_start = length - 1;                                   // the seed is the last 1 bp interval
            } else {
                length = std::min(mlen, ix->nodes[v].len - off);           // how much of the node lies behind the seed
                margin_left = 0; margin_right = mlen - length;
                read_start = min_offset[i];
                hint_start = 0;
            }
            gb_chain_anchor a;
            a.read_start = read_start; a.length = length; a.margin_before = margin_left; a.margin_after = margin_right;
            a.score = (int32_t)scores->match * (int32_t)(margin_left + length + margin_right);        // score_exact_match over the whole minimizer
            a.start_hint_offset = hint_start; a.end_hint_offset = length - hint_start; a.base_seed_length = margin_left + length + margin_right;
            a.start_paths = a.end_paths = paths ? paths[i] : 0;
            out[i] = a;
        }
        return GB_OK;
    });
}

extern "C" int gb_chain_candidates_batch(gb_device* d, uint32_t n_problems, const uint32_t* seed_pos, const uint64_t* seed_off,
                                         uint64_t limit, gb_chain_candidate* candidates, uint64_t candidate_cap, uint64_t* cand_off) {
    return gb::guarded("gb_chain_candidates_batch", [&] {
        if (!d || !seed_off || !cand_off || (candidate_cap && !candidates)) return GB_ERR_ARG;
        for (uint32_t p = 0; p <= n_problems; p++) cand_off[p] = 0;
        if (n_problems == 0) return GB_OK;
        const uint64_t total = seed_off[n_problems];
        if (total >= 0x7ffffff0ull || (total && !seed_pos)) return GB_ERR_ARG;
        if (total == 0) return GB_OK;
        std::vector<uint32_t> pb(total), pe(total);
        for (uint32_t p = 0; p < n_problems; p++) {
            if (seed_off[p + 1] < seed_off[p]) return GB_ERR_ARG;
            if (seed_off[p + 1] - seed_off[p] > GB_CHAIN_MAX_ANCHORS) { g_last_error = "gb_chain_candidates_batch: more than GB_CHAIN_MAX_ANCHORS seeds in one problem"; return GB_ERR_ARG; }
            for (uint64_t i = seed_off[p]; i < seed_off[p + 1]; i++) {
                const uint32_t v = seed_pos[2 * i], o = seed_pos[2 * i + 1];
                if (v < 2 || v >= d->h_node_len.size() || d->h_node_len[v] == 0 || o >= d->h_node_len[v]) { g_last_error = "gb_chain_candidates_batch: seed position outside the graph"; return GB_ERR_ARG; }
                pb[i] = (uint32_t)seed_off[p]; pe[i] = (uint32_t)seed_off[p + 1];
            }
        }
        GB_CUDA(cudaSetDevice(d->device));
        DevBuf<uint32_t> d_pos, d_pb, d_pe; DevBuf<uint64_t> d_count, d_offset; DevBuf<uint8_t> d_tmp; DevBuf<gb_chain_candidate> d_out;
        int rc;
        if ((rc = d_pos.upload(seed_pos, 2 * total, d->stream)) || (rc = d_pb.upload(pb.data(), total, d->stream)) || (rc = d_pe.upload(pe.data(), total, d->stream)) ||
            (rc = d_count.reserve(total + 1)) || (rc = d_offset.reserve(total + 1))) return rc;
        GB_CUDA(cudaMemsetAsync(d_count.ptr + total, 0, sizeof(uint64_t), d->stream));
        CandBatch b; b.n_seeds = (uint32_t)total; b.pos = d_pos.ptr; b.prob_begin = d_pb.ptr; b.prob_end = d_pe.ptr; b.limit = limit;
        b.count = d_count.ptr; b.offset = d_offset.ptr; b.out = nullptr;
        const uint32_t grid = std::max<uint32_t>(1u, std::min<uint32_t>((uint32_t)d->n_sms * 16, (uint32_t)((total + 3) / 4)));
        GB_CUDA(cudaEventRecord(d->ev0, d->stream));
        chain_candidates_kernel<false><<<grid, 128, 0, d->stream>>>(d->ix, b);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        size_t tmp_bytes = 0;
        GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_count.ptr, d_offset.ptr, (int)(total + 1), d->stream));
        if ((rc = d_tmp.reserve(tmp_bytes + 256))) return rc;
        size_t tb = d_tmp.cap;
        GB_CUDA(cub::DeviceScan::ExclusiveSum(d_tmp.ptr, tb, d_count.ptr, d_offset.ptr, (int)(total + 1), d->stream));
        d->launches++;
        std::vector<uint64_t> h_off(total + 1);
        GB_CUDA(cudaMemcpyAsync(h_off.data(), d_offset.ptr, sizeof(uint64_t) * (total + 1), cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaStreamSynchronize(d->stream));
        for (uint32_t p = 0; p <= n_problems; p++) cand_off[p] = h_off[seed_off[p]];
        const uint64_t n_out = h_off[total];
        if (n_out > candidate_cap) { g_last_error = "gb_chain_candidates_batch: candidate capacity too small (cand_off holds the sizes needed)"; return GB_ERR_CAPACITY; }
        if (n_out) {
            if ((rc = d_out.reserve(n_out))) return rc;
            b.out = d_out.ptr;
            chain_candidates_kernel<true><<<grid, 128, 0, d->stream>>>(d->ix, b);
            d->launches++;
            GB_CUDA(cudaGetLastError());
            GB_CUDA(cudaEventRecord(d->ev1, d->stream));
            GB_CUDA(cudaMemcpyAsync(candidates, d_out.ptr, sizeof(gb_chain_candidate) * n_out, cudaMemcpyDeviceToHost, d->stream));
        } else GB_CUDA(cudaEventRecord(d->ev1, d->stream));
        GB_CUDA(cudaStreamSynchronize(d->stream));
        GB_CUDA(cudaEventElapsedTime(&d->last_kernel_ms, d->ev0, d->ev1));
        return GB_OK;
    });
}
