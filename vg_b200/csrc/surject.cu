// surject.cu — reference paths (gb_ref_paths_build, gb_sam_header, gb_device_set_ref_paths) and gb_surject_device:
// Surjector::surject (surjector.cpp:223-630) for records in HBM, with giraffe's defaults, then the pair fields
// HTSAlignmentEmitter::convert_paired adds (hts_alignment_emitter.cpp:799-836).
//
// Kernels, one thread per record (the records are independent until the pair pass):
//   validate   record_valid (the GAF / GAM emitters' check) and the mate layout of paired records, one flag for the batch
//   count      the raw CIGAR op count of each record: its region of the cigar pool (simplification only shrinks it), and
//              the records left to the realigning route
//   scan       region offsets; the one wait: the pool size decides whether the fill runs
//   fill       placement on the paths, score, CIGAR, flags of each record
//   pair       a thread per pair: mate fields, TLEN and the pair flags of both records
// A record that leaves the reference path needs vg's realigning route, which is not built here.  It is not guessed at: the
// record, and its mate when paired (whose mate fields and flags depend on it), get GB_SURJ_REALIGN and no SAM line, so every
// line gb_emit_sam_device writes is the one vg writes, and the caller surjects the deferred records with vg.
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "emit_format.h"

#include <cub/cub.cuh>

#include <algorithm>
#include <string>
#include <vector>

struct gb_ref_paths {
    uint32_t n_nodes = 0;                  // gb_flat_index.n_nodes of the graph the paths were built on
    std::vector<uint32_t> node;            // 2 per node id, the layout of gb_device::ref_node
    std::vector<uint64_t> length;
    std::string names;
    std::vector<uint64_t> name_off;
};

namespace gb {
namespace {

constexpr uint32_t NO_REF = 0xffffffffu;
constexpr uint32_t SURJ_BLOCK = 128;
constexpr uint32_t BAM_M = 0, BAM_I = 1, BAM_D = 2, BAM_S = 4;

// The Surjector is an AlignerClient with vg's default scores (surjector.cpp:45-57): SurjectingAlignmentEmitter does not hand
// it giraffe's --match / --mismatch / ... (surjecting_alignment_emitter.cpp:18-26), so AS uses these, not gb_set_scores'.
constexpr DevScores SURJECT_SCORES{1, 4, 6, 1, 5};

struct SurjArgs {
    EmitArgs E;                            // records, pools, read offsets, graph (reads and names unused)
    const uint32_t* ref_node;
    DevScores sc;
    int64_t tlen_max;
};

__device__ bool surj_valid(const SurjArgs& S, uint32_t x) {
    const gb_alignment a = S.E.aln[x];
    if (!record_valid(S.E, a)) return false;
    if (!(a.flags & GB_ALN_PAIRED)) return true;
    const uint32_t y = x ^ 1u;
    return y < S.E.n && (S.E.aln[y].flags & GB_ALN_PAIRED) && S.E.aln[y].read_id == (a.read_id ^ 1u);
}

// Where the record lies on the reference paths (extract_overlapping_paths, surjector.cpp:4109-4260, for a path whose nodes
// are each on at most one reference path): every mapping on consecutive steps of one path strand is one chunk covering the
// whole read, the direct route (:3235-3253).  pos is the leftmost reference base on the path's forward strand.
struct Placement { int32_t ref, pos; bool rev; uint32_t route; };

__device__ Placement place(const SurjArgs& S, const gb_alignment& a) {
    Placement P{-1, -1, false, GB_SURJ_UNMAPPED};
    if (a.flags & GB_ALN_ABSENT) { P.route = GB_SURJ_ABSENT; return P; }
    if (!(a.flags & GB_ALN_MAPPED) || a.n_mappings == 0) return P;
    const gb_mapping* m = S.E.maps + a.mapping_off;
    const uint32_t* e = S.E.edits + a.edit_off;
    bool any = false, one = true, rev = false;
    uint32_t path = 0, prev_off = 0, prev_len = 0, ei = 0;
    int64_t first = 0, last = 0;
    for (uint32_t i = 0; i < a.n_mappings; i++) {
        const gb_mapping mi = m[i];
        uint32_t from = 0;
        for (uint32_t j = 0; j < mi.n_edits; j++, ei++) if ((e[ei] & 3u) != GB_EDIT_INS) from += edit_len(e[ei]);
        const uint32_t pr = S.ref_node[2 * (mi.node >> 1)], off = S.ref_node[2 * (mi.node >> 1) + 1], len = S.E.nodes[mi.node].len;
        if (pr == NO_REF) { one = false; continue; }
        const bool r = ((mi.node ^ pr) & 1u) != 0;          // the read walks the node against the path: the path's reverse strand
        if (!any) { path = pr >> 1; rev = r; }
        else if ((pr >> 1) != path || r != rev || (!rev ? off != prev_off + prev_len : off + len != prev_off)) one = false;
        any = true;
        prev_off = off; prev_len = len;
        if (i == 0) first = (int64_t)off + mi.offset;
        if (i + 1 == a.n_mappings) last = (int64_t)off + len - mi.offset - from;
    }
    if (!any) return P;
    if (!one) { P.route = GB_SURJ_REALIGN; return P; }
    P.ref = (int32_t)path; P.rev = rev; P.pos = (int32_t)(rev ? last : first); P.route = GB_SURJ_DIRECT;
    return P;
}

// place() with the pair rule: a paired record whose mate needs the realigning route is deferred with it.
__device__ Placement place_record(const SurjArgs& S, uint32_t x) {
    const gb_alignment a = S.E.aln[x];
    Placement P = place(S, a);
    if ((a.flags & GB_ALN_PAIRED) && P.route != GB_SURJ_ABSENT && P.route != GB_SURJ_REALIGN &&
        place(S, S.E.aln[x ^ 1u]).route == GB_SURJ_REALIGN)
        P = Placement{-1, -1, false, GB_SURJ_REALIGN};
    return P;
}

// EditAlignmentScorer::score_contiguous_alignment (alignment_scorer.cpp:159-245) with both bonuses allowed.
__device__ int32_t contiguous_score(const SurjArgs& S, const gb_alignment& a) {
    const gb_mapping* m = S.E.maps + a.mapping_off;
    const uint32_t* e = S.E.edits + a.edit_off;
    const DevScores& c = S.sc;
    int32_t score = 0;
    bool last_del = false;
    for (uint32_t i = 0, ei = 0; i < a.n_mappings; i++) {
        const uint32_t ne = m[i].n_edits;
        for (uint32_t j = 0; j < ne; j++, ei++) {
            const uint32_t op = e[ei] & 3u, len = edit_len(e[ei]);
            if (op == GB_EDIT_MATCH) { score += c.match * (int32_t)len; last_del = false; }
            else if (op == GB_EDIT_SUB) { score -= c.mismatch * (int32_t)len; last_del = false; }
            else if (op == GB_EDIT_DEL) { score -= last_del ? (int32_t)len * c.gap_extend : c.gap_open + ((int32_t)len - 1) * c.gap_extend; last_del = true; }
            else {
                const bool end = (i == 0 && j == 0) || (i + 1 == a.n_mappings && j + 1 == ne);
                if (!end) score -= c.gap_open + ((int32_t)len - 1) * c.gap_extend;
                last_del = false;
            }
        }
    }
    // softclip_start / softclip_end: the first edit of the first mapping, the last of the last, is an insertion
    const bool clip_start = m[0].n_edits && (e[0] & 3u) == GB_EDIT_INS;
    const uint32_t last_ne = m[a.n_mappings - 1].n_edits;
    const bool clip_end = last_ne && (e[a.n_edits - 1] & 3u) == GB_EDIT_INS;
    if (!clip_start) score += c.full_length_bonus;
    if (!clip_end) score += c.full_length_bonus;
    return score;
}

// The raw CIGAR of mapping_cigar over every mapping (alignment.cpp:1253-1283: matches and substitutions are M), adjacent
// equal ops merged (append_cigar_operation), in reverse order on the reverse strand (cigar_against_path, :1350-1353).
// out == NULL counts.
__device__ uint32_t raw_cigar(const SurjArgs& S, const gb_alignment& a, bool rev, uint32_t* out) {
    const uint32_t* e = S.E.edits + a.edit_off;
    uint32_t n = 0, cur_op = 0xffu, cur_len = 0;
    for (uint32_t k = 0; k < a.n_edits; k++) {
        const uint32_t wd = e[rev ? a.n_edits - 1 - k : k], op = wd & 3u, len = edit_len(wd);
        const uint32_t bop = op == GB_EDIT_INS ? BAM_I : op == GB_EDIT_DEL ? BAM_D : BAM_M;
        if (bop == cur_op) { cur_len += len; continue; }
        if (cur_op != 0xffu) { if (out) out[n] = cur_len << 4 | cur_op; n++; }
        cur_op = bop; cur_len = len;
    }
    if (cur_op != 0xffu) { if (out) out[n] = cur_len << 4 | cur_op; n++; }
    return n;
}

__device__ __forceinline__ uint32_t cop(uint32_t c) { return c & 15u; }
__device__ __forceinline__ uint32_t clen(uint32_t c) { return c >> 4; }

// The end handling and simplify_cigar of cigar_against_path (alignment.cpp:1355-1390, :1518-1570), in place; returns the
// op count.  An insertion behind an end deletion moves outside it, an end insertion becomes a soft clip, a run of two or
// more I / D ops becomes one D and one I, empty ops go, adjacent equal ops merge.
__device__ uint32_t finish_cigar(uint32_t* c, uint32_t n) {
    if (n == 0) return 0;
    if (n > 1 && cop(c[n - 1]) == BAM_D && cop(c[n - 2]) == BAM_I) { const uint32_t t = c[n - 1]; c[n - 1] = c[n - 2]; c[n - 2] = t; }
    if (cop(c[n - 1]) == BAM_I) c[n - 1] = clen(c[n - 1]) << 4 | BAM_S;
    if (n > 1 && cop(c[0]) == BAM_D && cop(c[1]) == BAM_I) { const uint32_t t = c[0]; c[0] = c[1]; c[1] = t; }
    if (cop(c[0]) == BAM_I) c[0] = clen(c[0]) << 4 | BAM_S;
    // runs of I / D
    uint32_t w = 0;
    for (uint32_t i = 0; i < n;) {
        const uint32_t o = cop(c[i]);
        if (o != BAM_I && o != BAM_D) { c[w++] = c[i++]; continue; }
        uint32_t j = i, d = 0, ins = 0;
        for (; j < n && (cop(c[j]) == BAM_I || cop(c[j]) == BAM_D); j++) (cop(c[j]) == BAM_D ? d : ins) += clen(c[j]);
        if (j - i >= 2) { c[w++] = d << 4 | BAM_D; c[w++] = ins << 4 | BAM_I; }
        else c[w++] = c[i];
        i = j;
    }
    // empty ops, adjacent equal ops
    uint32_t v = 0;
    for (uint32_t i = 0; i < w; i++) {
        if (clen(c[i]) == 0) continue;
        if (v && cop(c[v - 1]) == cop(c[i])) c[v - 1] += clen(c[i]) << 4;
        else c[v++] = c[i];
    }
    return v;
}

__global__ void surj_validate_kernel(SurjArgs S, uint32_t* bad) {
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < S.E.n; x += gridDim.x * blockDim.x)
        if (!surj_valid(S, x)) *bad = 1u;
}

__global__ void surj_count_kernel(SurjArgs S, const uint32_t* bad, uint64_t* ops, unsigned long long* n_realign) {
    const bool refused = *bad != 0;
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x <= S.E.n; x += gridDim.x * blockDim.x) {
        uint64_t k = 0;
        if (x < S.E.n && !refused) {
            const Placement P = place_record(S, x);
            if (P.route == GB_SURJ_DIRECT) k = raw_cigar(S, S.E.aln[x], P.rev, nullptr);
            if (P.route == GB_SURJ_REALIGN) atomicAdd(n_realign, 1ull);
        }
        ops[x] = k;
    }
}

__global__ void surj_fill_kernel(SurjArgs S, const uint64_t* off, gb_sam_record* out, uint32_t* cigar) {
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < S.E.n; x += gridDim.x * blockDim.x) {
        const gb_alignment a = S.E.aln[x];
        const Placement P = place_record(S, x);
        gb_sam_record r;
        r.read_id = a.read_id; r.route = (uint8_t)P.route;
        r.ref = P.ref; r.pos = P.pos; r.mate_ref = -1; r.mate_pos = -1; r.tlen = 0;
        r.cigar_off = (uint32_t)off[x]; r.n_cigar = 0;
        const bool mapped = P.route == GB_SURJ_DIRECT;
        r.mapq = mapped ? a.mapq : 0;
        r.score = mapped ? contiguous_score(S, a) : 0;
        if (mapped) r.n_cigar = finish_cigar(cigar + off[x], raw_cigar(S, a, P.rev, cigar + off[x]));
        uint32_t f = 0;                                   // sam_flag, alignment.cpp:2898-2931
        if (!mapped) f |= 0x4u;
        if (P.rev) f |= 0x10u;
        if (a.flags & GB_ALN_SECONDARY) f |= 0x100u;
        r.flag = (uint16_t)f;
        out[x] = r;
    }
}

// find_bounds of compute_template_lengths (alignment.cpp:2848-2875): the outermost M bases; none: (INT64_MAX, INT64_MIN).
__device__ void bounds(const gb_sam_record& r, const uint32_t* cigar, int64_t& lo, int64_t& hi) {
    lo = INT64_MAX; hi = INT64_MIN;
    int64_t here = r.pos;
    if (r.ref < 0) return;
    for (uint32_t i = 0; i < r.n_cigar; i++) {
        const uint32_t c = cigar[r.cigar_off + i];
        if (cop(c) == BAM_M) { lo = min(lo, here); hi = max(hi, here + (int64_t)clen(c)); }
        if (cop(c) == BAM_M || cop(c) == BAM_D) here += clen(c);
    }
}

// determine_flag's pair part (alignment.cpp:719-751) for record r with mate m.
__device__ uint16_t pair_flag(const gb_sam_record& r, const gb_sam_record& m, int64_t tlen_max) {
    uint32_t f = r.flag | 0x1u | ((r.read_id & 1u) ? 0x80u : 0x40u);
    const bool rev = (r.flag & 0x10u) != 0, mrev = (m.flag & 0x10u) != 0;
    if (r.ref >= 0 && m.ref == r.ref) {
        const bool facing = (r.pos <= m.pos && !rev && mrev) || (m.pos <= r.pos && rev && !mrev);
        const int64_t t = r.tlen < 0 ? -(int64_t)r.tlen : r.tlen;
        if (facing && (tlen_max == 0 || t <= tlen_max)) f |= 0x2u;
    }
    if (m.ref < 0) f |= 0x8u;
    if (mrev) f |= 0x20u;
    return (uint16_t)f;
}

__global__ void surj_pair_kernel(SurjArgs S, gb_sam_record* out, const uint32_t* cigar) {
    for (uint32_t x = 2 * (blockIdx.x * blockDim.x + threadIdx.x); x + 1 < S.E.n; x += 2 * gridDim.x * blockDim.x) {
        if (!(S.E.aln[x].flags & GB_ALN_PAIRED)) continue;
        const uint32_t x1 = (S.E.aln[x].read_id & 1u) ? x + 1 : x, x2 = x1 ^ 1u;      // x1: mate 1 (the even read)
        gb_sam_record r1 = out[x1], r2 = out[x2];
        if (r1.route == GB_SURJ_REALIGN) continue;                 // deferred with its mate: no pair fields
        int64_t lo1, hi1, lo2, hi2;
        bounds(r1, cigar, lo1, hi1); bounds(r2, cigar, lo2, hi2);
        // int32_t dist = max_end - min_start, in the reference's int64 arithmetic (wrapping when neither mate has M bases)
        const int32_t dist = (int32_t)(uint64_t)((uint64_t)max(hi1, hi2) - (uint64_t)min(lo1, lo2));
        const bool first = lo1 < lo2 || (lo1 == lo2 && hi1 < hi2);
        r1.tlen = first ? dist : -dist; r2.tlen = first ? -dist : dist;
        r1.mate_ref = r2.ref; r1.mate_pos = r2.pos; r2.mate_ref = r1.ref; r2.mate_pos = r1.pos;
        const uint16_t f1 = pair_flag(r1, r2, S.tlen_max), f2 = pair_flag(r2, r1, S.tlen_max);
        r1.flag = f1; r2.flag = f2;
        out[x1] = r1; out[x2] = r2;
    }
}

int surject_device(gb_device* d, uint32_t n, const gb_alignment* d_aln, const gb_mapping* d_mappings, uint64_t mapping_pool_len,
                   const uint32_t* d_edits, uint64_t edit_pool_len, uint32_t n_reads, const uint64_t* d_read_off, int64_t tlen_max,
                   gb_sam_record* d_out, uint32_t* d_cigar, uint64_t cigar_cap, uint64_t* cigar_used, uint32_t* n_realign) {
    if (!d || !d_aln || !d_read_off || !d_out || !cigar_used || n == 0xffffffffu || tlen_max < 0) return GB_ERR_ARG;
    if (!d->ref_ready) { g_last_error = "gb_surject_device: no reference paths on the handle (gb_device_set_ref_paths)"; return GB_ERR_ARG; }
    GB_CUDA(cudaSetDevice(d->device));
    SurjArgs S;
    EmitArgs& A = S.E;
    A.n = n; A.aln = d_aln; A.maps = d_mappings; A.map_len = mapping_pool_len; A.edits = d_edits; A.edit_len = edit_pool_len;
    A.n_reads = n_reads; A.reads = nullptr; A.quals = nullptr; A.read_off = d_read_off; A.names = nullptr; A.name_off = nullptr;
    A.nodes = d->ix.nodes; A.seq = d->ix.seq; A.n_nodes = d->ix.n_nodes;
    S.ref_node = d->ref_node.ptr; S.sc = SURJECT_SCORES; S.tlen_max = tlen_max;

    const size_t m = (size_t)n + 1;
    size_t tb = 0;
    GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t)m, d->stream));
    uint64_t *status, *ops, *off;
    void* tmp;
    int rc = carve(d->surj_ws, [&](Carve& c) { status = c.take<uint64_t>(3); ops = c.take<uint64_t>(m); off = c.take<uint64_t>(m); tmp = c.take<uint8_t>(tb); });
    if (rc) return rc;
    const uint32_t grid = (uint32_t)std::min<uint64_t>((m + SURJ_BLOCK - 1) / SURJ_BLOCK, (uint64_t)d->n_sms * 64);
    // status: {refused, pool size, records left to the realigning route}
    GB_CUDA(cudaMemsetAsync(status, 0, 3 * sizeof(uint64_t), d->stream));
    surj_validate_kernel<<<grid, SURJ_BLOCK, 0, d->stream>>>(S, (uint32_t*)status);
    surj_count_kernel<<<grid, SURJ_BLOCK, 0, d->stream>>>(S, (const uint32_t*)status, ops, (unsigned long long*)(status + 2));
    d->launches += 2;
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, ops, off, (int64_t)m, d->stream));
    d->launches++;
    GB_CUDA(cudaMemcpyAsync(status + 1, off + n, sizeof(uint64_t), cudaMemcpyDeviceToDevice, d->stream));
    uint64_t h_status[3];
    GB_CUDA(cudaMemcpyAsync(h_status, status, sizeof h_status, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));              // the one wait: the pool size decides whether the fill runs
    if (h_status[0] & 0xffffffffull) {
        g_last_error = "gb_surject_device: a record points outside its read, pools or the graph, or a paired record's mate is not at x ^ 1";
        return GB_ERR_ARG;
    }
    *cigar_used = h_status[1];
    if (n_realign) *n_realign = (uint32_t)h_status[2];
    if (h_status[1] > 0xffffffffull) { g_last_error = "gb_surject_device: the cigar pool would pass 2^32 ops (gb_sam_record.cigar_off is 32-bit): split the batch"; return GB_ERR_CAPACITY; }
    if (h_status[1] > cigar_cap) { g_last_error = "gb_surject_device: cigar pool too small (*cigar_used holds the ops needed)"; return GB_ERR_CAPACITY; }
    if (h_status[1] && !d_cigar) return GB_ERR_ARG;
    if (n) {
        surj_fill_kernel<<<grid, SURJ_BLOCK, 0, d->stream>>>(S, off, d_out, d_cigar);
        surj_pair_kernel<<<grid, SURJ_BLOCK, 0, d->stream>>>(S, d_out, d_cigar);
        d->launches += 2;
        GB_CUDA(cudaGetLastError());
    }
    return GB_OK;
}

bool sam_name_ok(const uint8_t* p, uint64_t k) {
    if (k == 0) return false;
    for (uint64_t i = 0; i < k; i++) if (p[i] < '!' || p[i] > '~') return false;
    return true;
}

int ref_paths_build(const gb_flat_index* ix, uint32_t n_paths, const uint8_t* names, const uint64_t* name_off,
                    const uint32_t* path_nodes, const uint64_t* path_off, gb_ref_paths** out) {
    if (!out) return GB_ERR_ARG;
    *out = nullptr;
    if (!ix || !ix->nodes || !names || !name_off || !path_off || (!path_nodes && path_off[n_paths] > path_off[0])) return GB_ERR_ARG;
    for (uint32_t p = 0; p < n_paths; p++)
        if (name_off[p + 1] < name_off[p] || path_off[p + 1] < path_off[p]) return GB_ERR_ARG;
    auto rp = std::make_unique<gb_ref_paths>();
    const uint32_t n_ids = ix->n_nodes / 2;
    rp->n_nodes = ix->n_nodes;
    rp->node.assign(2 * (size_t)n_ids, NO_REF);
    rp->name_off.push_back(0);
    for (uint32_t p = 0; p < n_paths; p++) {
        const uint8_t* nm = names + name_off[p];
        const uint64_t nk = name_off[p + 1] - name_off[p];
        if (!sam_name_ok(nm, nk)) { set_last_error("gb_ref_paths_build: ", "a path name is empty or holds a byte outside '!'..'~'"); return GB_ERR_FORMAT; }
        if (path_off[p + 1] == path_off[p]) { set_last_error("gb_ref_paths_build: ", "an empty path"); return GB_ERR_FORMAT; }
        uint64_t len = 0;
        for (uint64_t i = path_off[p]; i < path_off[p + 1]; i++) {
            const uint32_t v = path_nodes[i], id = v >> 1;
            if (id >= n_ids || ix->nodes[v].len == 0) { set_last_error("gb_ref_paths_build: ", "a node the graph does not have"); return GB_ERR_FORMAT; }
            if (rp->node[2 * (size_t)id] != NO_REF) { set_last_error("gb_ref_paths_build: ", "a node occurs more than once across the reference paths"); return GB_ERR_FORMAT; }
            if (len + ix->nodes[v].len >= (1ull << 31)) { set_last_error("gb_ref_paths_build: ", "a path of 2^31 bases or more"); return GB_ERR_FORMAT; }
            rp->node[2 * (size_t)id] = p << 1 | (v & 1u);
            rp->node[2 * (size_t)id + 1] = (uint32_t)len;
            len += ix->nodes[v].len;
        }
        rp->length.push_back(len);
        rp->names.append((const char*)nm, nk);
        rp->name_off.push_back(rp->names.size());
    }
    *out = rp.release();
    return GB_OK;
}

int sam_header(const gb_ref_paths* rp, char* out, uint64_t out_cap, uint64_t* out_used) {
    if (!rp || !out_used || (!out && out_cap)) return GB_ERR_ARG;
    std::string h = "@HD\tVN:1.5\tSO:unknown\n";
    for (size_t p = 0; p < rp->length.size(); p++)
        h.append("@SQ\tSN:").append(rp->names, rp->name_off[p], rp->name_off[p + 1] - rp->name_off[p])
         .append("\tLN:").append(std::to_string(rp->length[p])).append("\n");
    *out_used = h.size();
    if (h.size() > out_cap) { g_last_error = "gb_sam_header: output capacity too small (*out_used holds the bytes needed)"; return GB_ERR_CAPACITY; }
    std::copy(h.begin(), h.end(), out);
    return GB_OK;
}

int set_ref_paths(gb_device* d, const gb_ref_paths* rp) {
    if (!d || !rp) return GB_ERR_ARG;
    if (rp->n_nodes != d->ix.n_nodes) { g_last_error = "gb_device_set_ref_paths: the paths were built for another graph"; return GB_ERR_ARG; }
    GB_CUDA(cudaSetDevice(d->device));
    d->ref_ready = false;
    if (int rc = d->ref_node.upload(rp->node.data(), rp->node.size(), d->stream)) return rc;
    if (int rc = d->ref_names.upload((const uint8_t*)rp->names.data(), rp->names.size(), d->stream)) return rc;
    if (int rc = d->ref_name_off.upload(rp->name_off.data(), rp->name_off.size(), d->stream)) return rc;
    GB_CUDA(cudaStreamSynchronize(d->stream));              // the host vectors may go away after the call
    d->n_ref_paths = (uint32_t)rp->length.size();
    d->ref_ready = true;
    return GB_OK;
}

} // namespace
} // namespace gb

extern "C" int gb_ref_paths_build(const gb_flat_index* ix, uint32_t n_paths, const uint8_t* names, const uint64_t* name_off,
                                  const uint32_t* path_nodes, const uint64_t* path_off, gb_ref_paths** out) {
    return gb::guarded("gb_ref_paths_build", [&] { return gb::ref_paths_build(ix, n_paths, names, name_off, path_nodes, path_off, out); });
}
extern "C" void gb_ref_paths_free(gb_ref_paths* rp) { delete rp; }
extern "C" int gb_sam_header(const gb_ref_paths* rp, char* out, uint64_t out_cap, uint64_t* out_used) {
    return gb::guarded("gb_sam_header", [&] { return gb::sam_header(rp, out, out_cap, out_used); });
}
extern "C" int gb_device_set_ref_paths(gb_device* dev, const gb_ref_paths* rp) {
    return gb::guarded("gb_device_set_ref_paths", [&] { return gb::set_ref_paths(dev, rp); });
}
extern "C" int gb_surject_device(gb_device* dev, uint32_t n, const gb_alignment* d_aln, const gb_mapping* d_mappings, uint64_t mapping_pool_len,
                                 const uint32_t* d_edits, uint64_t edit_pool_len, uint32_t n_reads, const uint64_t* d_read_off, int64_t tlen_max,
                                 gb_sam_record* d_out, uint32_t* d_cigar, uint64_t cigar_cap, uint64_t* cigar_used, uint32_t* n_realign) {
    return gb::guarded("gb_surject_device", [&] { return gb::surject_device(dev, n, d_aln, d_mappings, mapping_pool_len, d_edits, edit_pool_len,
                                                                            n_reads, d_read_off, tlen_max, d_out, d_cigar, cigar_cap, cigar_used, n_realign); });
}
