// seed.cuh — seeding stage, one warp per read (single-end) or per read pair (paired-end):
//   find_minimizers            minimizer_mapper.cpp:3918-3974  (gbwtgraph minimizer_regions + find)
//   sort_minimizers_by_score   :4074-4107  (LazyRNG tie shuffle, utility.hpp:771-794)
//   find_seeds                 :4109-4517  (filter cascade with running state)
//   cluster_seeds              snarl_seed_clusterer.cpp:28-63 / :65-145 (connected components under
//                              the unoriented minimum distance, via the 16-byte distance payload)
//   score_cluster              :4738-4780
//   cluster selection          single-end :655-832, paired-end :1568-1883
//   extend_seed_group packing  :4784-4850  ((handle, read_offset - node_offset) seeds)
// and leaves DevMinimizer / DevSeed / DevItem records in HBM for the next kernels.
//
// Phase A (per read) needs the k-mer scratch in shared memory; phase B (clusters) works on the
// HBM records plus a small shared cluster table, so a pair reuses one shared scratch.
#pragma once
#include "map_state.cuh"
#include "minimizer_common.h"

namespace gb {

constexpr uint32_t MAX_CLUSTERS = 64;     // read clusters per read kept in shared memory (second-pass capacity)
constexpr uint32_t GB_ITEM_RETRY = 100;   // internal: did not fit the small first-pass tables

// Stage-parity debugging (gb_debug_seed_stage): every cluster of every read with its score, coverage,
// fragment and rank among the read's work items; [n_reads * MAX_CLUSTERS], null in production runs.
struct DbgCluster { double score, coverage; uint32_t first_seed, fragment, kept_rank, valid; };

struct SeedPools {
    DbgCluster* dbg_clusters;
    uint32_t* overflow;       // sticky: a pool ran out; the host grows the pools and reruns the chunk
    DevMinimizer* minimizers; uint32_t min_cap;  uint32_t* min_cursor;
    DevSeed* seeds;           uint32_t seed_cap; uint32_t* seed_cursor;
    DevItem* items;           uint32_t item_cap; uint32_t* item_cursor;
    gb_seed* ext_seeds;       uint32_t ext_cap;  uint32_t* ext_cursor;
};

// Per-warp shared memory carve-up.
struct SeedSmem {
    uint8_t*  read;        // [Lc]
    uint64_t* khash;       // [Lc]  canonical hash per k-mer start (scratch after compaction)
    uint64_t* kkey;        // [Lc]  canonical key
    uint8_t*  kflag;       // [Lc]  bit0 valid, bit1 reverse
    uint64_t* m_key;       // [MAX_MINIMIZERS]
    uint64_t* m_hash;
    double*   m_score;
    uint32_t* m_hit_off;
    uint32_t* m_hit_cnt;
    uint16_t* m_fwd;
    uint16_t* m_agg_start;
    uint16_t* m_agg_len;
    uint8_t*  m_rev;
    uint8_t*  m_order;     // score order -> read order index
    uint8_t*  m_pass;      // per score-order minimizer: passed the filters
    // clusters (two reads' worth)
    double*   c_score;     // [2 * MAX_CLUSTERS]
    double*   c_cov;
    uint32_t* c_label;
    uint32_t* c_present;   // [2 * MAX_CLUSTERS * PRESENT_WORDS]
    uint8_t*  c_order;     // [2 * MAX_CLUSTERS] processing order
    uint8_t*  c_frag;      // [2 * MAX_CLUSTERS] fragment id of each read cluster
    uint8_t*  scratch;     // [2 * Cc + Mc]
    // capacities of this launch: Mc minimizers per read, Cc clusters per read.  The first launch uses
    // small tables (occupancy); units that do not fit are retried by a second launch at the maxima.
    uint32_t Mc, Cc, Lc;
    uint32_t ns_max;       // largest pair seed set clustered in shared memory (<= 64)
};

__host__ __device__ inline size_t seed_smem_bytes(uint32_t Lc, uint32_t Mc, uint32_t Cc) {
    size_t b = 0;
    b += (size_t)Lc * 8 * 2;                            // khash, kkey
    b += (size_t)Mc * (8 + 8 + 8);                      // m_key, m_hash, m_score
    b += (size_t)2 * Cc * (8 + 8);                      // c_score, c_cov
    b += (size_t)Mc * (4 + 4);                          // hit_off, hit_cnt
    b += (size_t)2 * Cc * 4 * (1 + PRESENT_WORDS);
    b += (size_t)Mc * (2 + 2 + 2);                      // fwd, agg_start, agg_len
    b += (size_t)Lc * 2;                                // read, kflag
    b += (size_t)Mc * 3;                                // rev, order, pass
    b += (size_t)2 * Cc * 2;                            // c_order, c_frag
    b += (size_t)2 * Cc + Mc;                           // scratch
    return (b + 15) & ~(size_t)15;
}

// Lc, Mc, Cc are multiples of 8, so every array below stays naturally aligned.
__device__ __forceinline__ SeedSmem carve_seed_smem(uint8_t* base, uint32_t Lc, uint32_t Mc, uint32_t Cc, uint32_t ns_max = 64) {
    SeedSmem s;
    uint8_t* p = base;
    s.Mc = Mc; s.Cc = Cc; s.Lc = Lc; s.ns_max = ns_max;
    s.khash = (uint64_t*)p; p += (size_t)Lc * 8;
    s.kkey = (uint64_t*)p; p += (size_t)Lc * 8;
    s.m_key = (uint64_t*)p; p += Mc * 8;
    s.m_hash = (uint64_t*)p; p += Mc * 8;
    s.m_score = (double*)p; p += Mc * 8;
    s.c_score = (double*)p; p += 2 * Cc * 8;
    s.c_cov = (double*)p; p += 2 * Cc * 8;
    s.m_hit_off = (uint32_t*)p; p += Mc * 4;
    s.m_hit_cnt = (uint32_t*)p; p += Mc * 4;
    s.c_label = (uint32_t*)p; p += 2 * Cc * 4;
    s.c_present = (uint32_t*)p; p += 2 * Cc * 4 * PRESENT_WORDS;
    s.m_fwd = (uint16_t*)p; p += Mc * 2;
    s.m_agg_start = (uint16_t*)p; p += Mc * 2;
    s.m_agg_len = (uint16_t*)p; p += Mc * 2;
    s.read = p; p += Lc;
    s.kflag = p; p += Lc;
    s.m_rev = p; p += Mc;
    s.m_order = p; p += Mc;
    s.m_pass = p; p += Mc;
    s.c_order = p; p += 2 * Cc;
    s.c_frag = p; p += 2 * Cc;
    s.scratch = p; p += 2 * Cc + Mc;
    return s;
}
__device__ __forceinline__ uint32_t table_full(uint32_t have, uint32_t max_cap) { return have < max_cap ? GB_ITEM_RETRY : (uint32_t)GB_ITEM_OUT_FULL; }

// Claim `n` records of an HBM pool (warp-uniform).  Once any pool has run out the sticky flag stops every later
// claim before it touches the cursor, so a cursor can never wrap; the host sees the flag, grows the pools and
// reruns the whole chunk (map.cu), so which reads happened to fail never shows in a result.
__device__ __forceinline__ bool pool_claim(uint32_t* cursor, uint32_t n, uint32_t cap, uint32_t* overflow, uint32_t& off) {
    uint32_t o = 0xffffffffu;
    if (lane_id() == 0) {
        if (*(volatile uint32_t*)overflow == 0) {
            o = atomicAdd(cursor, n);
            if (o > cap || n > cap - o) { atomicExch(overflow, 1u); o = 0xffffffffu; }
        }
    }
    off = __shfl_sync(FULL, o, 0);
    return off != 0xffffffffu;
}

// dump the cluster table of one read for the stage-parity tests
__device__ __forceinline__ void dbg_dump_clusters(const SeedPools& pools, const SeedSmem& sm, uint32_t read_idx, uint32_t cbase, uint32_t Cn,
                                                  const uint8_t* kept, uint32_t n_kept, bool deferred = false) {
    if (!pools.dbg_clusters) return;
#pragma unroll 1
    for (uint32_t c = lane_id(); c < Cn; c += 32) {
        DbgCluster dc; dc.score = sm.c_score[cbase + c]; dc.coverage = sm.c_cov[cbase + c]; dc.first_seed = sm.c_label[cbase + c];
        dc.fragment = sm.c_frag[cbase + c]; dc.kept_rank = 0xffffffffu; dc.valid = deferred ? 2u : 1u;
#pragma unroll 1
        for (uint32_t t = 0; t < n_kept; t++) if (kept[t] == c) dc.kept_rank = t;
        pools.dbg_clusters[(size_t)read_idx * MAX_CLUSTERS + c] = dc;
    }
}

__device__ __forceinline__ uint32_t pow13(uint32_t e) {
    uint32_t r = 1, b = 13;
    while (e) { if (e & 1) r *= b; b *= b; e >>= 1; }
    return r;
}

// seedNumber = fold(seed * 13 + byte) over `bytes` (utility.cpp:911-927), continuing from `seed`: byte i weighs 13^(L-1-i).
// Lane q takes the bytes q, q + 32, ... places from the end (Horner in 13^32, then times 13^q), so its loads are
// independent of each other and `bytes` can be the read in HBM.
__device__ inline uint32_t fold_seed(uint32_t seed, const uint8_t* bytes, uint32_t L) {
    const uint32_t lane = lane_id();
    constexpr uint32_t P32 = 0x6a265881u;                        // 13^32 mod 2^32
    const int32_t n = L > lane ? (int32_t)((L - 1 - lane) >> 5) + 1 : 0;
    uint32_t acc = 0;
#pragma unroll 4
    for (int32_t j = n - 1; j >= 0; j--) acc = acc * P32 + bytes[L - 1 - lane - 32 * (uint32_t)j];
    uint32_t term = acc * pow13(lane);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) term += __shfl_xor_sync(FULL, term, o);
    return seed * pow13(L) + term;
}

// Copy a read of L bytes to shared memory with up to 256 bytes of loads in flight per round trip (L <= 256 takes one).
__device__ __forceinline__ void stage_read(uint8_t* dst, const uint8_t* src, uint32_t L) {
    const uint32_t lane = lane_id();
#pragma unroll 1
    for (uint32_t base = 0; base < L; base += 256) {
        uint32_t v[8];
#pragma unroll
        for (uint32_t k = 0; k < 8; k++) { const uint32_t i = base + lane + 32 * k; v[k] = i < L ? src[i] : 0u; }
#pragma unroll
        for (uint32_t k = 0; k < 8; k++) { const uint32_t i = base + lane + 32 * k; if (i < L) dst[i] = (uint8_t)v[k]; }
    }
}

// set bits [lo, hi) of a bitmap made of 32-bit words
__device__ __forceinline__ void set_bit_range(uint32_t* words, uint32_t lo, uint32_t hi) {
    if (lo >= hi) return;
    const uint32_t w0 = lo >> 5, w1 = (hi - 1) >> 5;
    const uint32_t m0 = 0xffffffffu << (lo & 31), m1 = 0xffffffffu >> (31 - ((hi - 1) & 31));
    if (w0 == w1) { words[w0] |= (m0 & m1); return; }
    words[w0] |= m0;
#pragma unroll 1
    for (uint32_t w = w0 + 1; w < w1; w++) words[w] = 0xffffffffu;
    words[w1] |= m1;
}
__device__ __forceinline__ bool any_bit_in_range(const uint32_t* words, uint32_t lo, uint32_t hi) {
    if (lo >= hi) return false;
    const uint32_t w0 = lo >> 5, w1 = (hi - 1) >> 5;
    const uint32_t m0 = 0xffffffffu << (lo & 31), m1 = 0xffffffffu >> (31 - ((hi - 1) & 31));
    if (w0 == w1) return (words[w0] & m0 & m1) != 0;
    if (words[w0] & m0) return true;
#pragma unroll 1
    for (uint32_t w = w0 + 1; w < w1; w++) if (words[w]) return true;
    return (words[w1] & m1) != 0;
}

// unoriented minimum graph distance <= limit between two seeds (see gb_dist_payload)
// Two different nodes of one site: distance through the site's table (either direction), INT_MAX when unreachable.
// c_in = x_in + offset, c_out = x_out - (length - offset), offsets on the forward strand.
__device__ __noinline__ int32_t same_site_distance(const DevIndex& ix, uint32_t id_a, int32_t c_in_a, int32_t c_out_a, uint32_t id_b, int32_t c_in_b, int32_t c_out_b) {
    if (ix.n_slots == 0) return INT_MAX;
    const uint4 pa = __ldg(reinterpret_cast<const uint4*>(ix.dist) + id_a), pb = __ldg(reinterpret_cast<const uint4*>(ix.dist) + id_b);
    int64_t best = -1;
    int64_t t = site_distance(ix, pa, pb);                       // a -> b: rest of a + table + offset in b
    if (t >= 0) best = ((int64_t)(int32_t)pa.y - c_out_a) + t + ((int64_t)c_in_b - (int64_t)(int32_t)pb.x);
    t = site_distance(ix, pb, pa);
    if (t >= 0) { const int64_t d = ((int64_t)(int32_t)pb.y - c_out_b) + t + ((int64_t)c_in_a - (int64_t)(int32_t)pa.x); if (best < 0 || d < best) best = d; }
    return best < 0 || best > INT_MAX - 1 ? INT_MAX : (int32_t)best;
}

__device__ __forceinline__ bool seeds_within(const DevIndex& ix, const DevSeed& a, const DevSeed& b, int32_t limit) {
    const uint32_t ida = a.node >> 1, idb = b.node >> 1;
    if (ida == idb) {
        const int32_t d = b.c_in - a.c_in;                        // one node, one x_in: the forward offsets' difference
        return (d >= 0 ? d : -d) <= limit;
    }
    if (a.slot < b.slot) return (b.c_in - a.c_out) <= limit;
    if (b.slot < a.slot) return (a.c_in - b.c_out) <= limit;
    return same_site_distance(ix, ida, a.c_in, a.c_out, idb, b.c_in, b.c_out) <= limit;
}

// -----------------------------------------------------------------------------------------
// Phase A: minimizers -> score order -> filter cascade -> DevMinimizer + DevSeed records.
// `sm.read` must already hold the read.  rng is advanced by the tie shuffle.
// -----------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t seed_phase_a(const DevIndex& ix, const MapParamsDev& P, const SeedSmem& sm, uint32_t L,
                                        const SeedPools& pools, DevRng& rng, ReadState& rs) {
    const int lane = lane_id();
    const uint32_t k = ix.k, w = ix.w;
    const uint32_t window_bp = k + w - 1;
    rs.min_off = rs.min_cnt = rs.item_off = rs.item_cnt = rs.seed_off = rs.seed_cnt = 0; rs.n_clusters = 0;
    if (L > 512) return GB_ITEM_OUT_FULL;          // short-read path: coverage bitmaps are 512 bits
    if (L < window_bp) return GB_ITEM_OK;          // no minimizers -> no seeds

    // ---- canonical k-mer hashes ------------------------------------------------------------
    // The read is packed 2 bits per base (first base in the top bits) with one warp vote per 32
    // bases; lane s then cuts k-mer s out of two packed words, so no lane rolls through k - 1
    // warm-up bases.  Encoding and canonical choice as gbwtgraph's minimizer key (minimizer_common.h).
    const uint32_t nk = L - k + 1;
    {
        uint64_t* packed = sm.m_key;                                    // [n_blocks + 1]; m_key is filled later
        uint32_t* invalid = reinterpret_cast<uint32_t*>(sm.m_key + 17);  // [n_blocks]  (Mc >= 16: 24 * Mc bytes follow m_key)
        const uint32_t n_blocks = (L + 31) >> 5;
#pragma unroll 1
        for (uint32_t t = 0; t < n_blocks; t++) {
            const uint32_t pos = t * 32 + lane;
            const uint32_t ch = pos < L ? sm.read[pos] : 0u;
            const uint32_t idx = (ch & 0xDFu) - 0x41u;                     // 'A' = 0, 'C' = 2, 'G' = 6, 'T' = 19
            const bool ok = idx < 32u && ((0x00080045u >> idx) & 1u);
            uint32_t code = (ch >> 1) & 3u; code ^= code >> 1;             // A 0, C 1, G 2, T 3
            const uint32_t v = ok ? code : 0u;
            const uint32_t hi = __reduce_or_sync(FULL, lane < 16 ? v << (30 - 2 * lane) : 0u);
            const uint32_t lo = __reduce_or_sync(FULL, lane >= 16 ? v << (62 - 2 * lane) : 0u);
            const uint32_t bad = __ballot_sync(FULL, !ok && pos < L);
            if (lane == 0) { packed[t] = ((uint64_t)hi << 32) | lo; invalid[t] = bad; }
        }
        if (lane == 0) packed[n_blocks] = 0;
        __syncwarp();
#pragma unroll 1
        for (uint32_t s = lane; s < nk; s += 32) {
            const uint32_t wd = s >> 5, sh = 2 * (s & 31);
            const uint64_t x = sh ? (packed[wd] << sh) | (packed[wd + 1] >> (64 - sh)) : packed[wd];
            uint8_t flag = 0; uint64_t h = ~0ull, key = 0;
            if (!any_bit_in_range(invalid, s, s + k)) {
                const uint64_t fk = x >> (64 - 2 * k);
                uint64_t rv = __brevll((~x) >> (64 - 2 * k));              // reversed groups, bits swapped inside each group
                rv = ((rv & 0xAAAAAAAAAAAAAAAAull) >> 1) | ((rv & 0x5555555555555555ull) << 1);
                const uint64_t rk = rv >> (64 - 2 * k);
                const uint64_t hf = gbmin::hash64(fk), hr = gbmin::hash64(rk);
                if (hr < hf) { h = hr; key = rk; flag = 3; } else { h = hf; key = fk; flag = 1; }
            }
            sm.khash[s] = h; sm.kkey[s] = key; sm.kflag[s] = flag;
        }
    }
    __syncwarp();
    // ---- window minima -> minimizers in read order ---------------------------------------------
    // (invalid k-mers carry hash ~0, so they never beat a valid one)
    uint32_t M = 0;
    {
        const int32_t last_window = (int32_t)(L - window_bp);
#pragma unroll 1
        for (uint32_t base = 0; base < nk; base += 32) {
            const uint32_t s = base + lane;
            bool is_min = false; int32_t lo = 0, hi = -1;
            if (s < nk && (sm.kflag[s] & 1)) {
                const uint64_t h = sm.khash[s];
                int32_t l = -1000000, r = 1000000;
                for (int32_t d = 1; d < (int32_t)w; d++) {
                    const int32_t tl = (int32_t)s - d, tr = (int32_t)s + d;
                    if (l < 0 && tl >= 0 && sm.khash[tl] < h) l = tl;
                    if (r == 1000000 && tr < (int32_t)nk && sm.khash[tr] < h) r = tr;
                }
                lo = max(max((int32_t)s - (int32_t)w + 1, l + 1), 0);
                hi = min(min((int32_t)s, r - (int32_t)w), last_window);
                is_min = lo <= hi;
            }
            const uint32_t bal = __ballot_sync(FULL, is_min);
            const uint32_t cnt = __popc(bal);
            if (M + cnt > sm.Mc) return table_full(sm.Mc, MAX_MINIMIZERS);
            if (is_min) {
                const uint32_t idx = M + __popc(bal & ((1u << lane) - 1u));
                sm.m_key[idx] = sm.kkey[s]; sm.m_hash[idx] = sm.khash[s];
                sm.m_fwd[idx] = (uint16_t)s; sm.m_rev[idx] = (sm.kflag[s] >> 1) & 1;
                sm.m_agg_start[idx] = (uint16_t)lo; sm.m_agg_len[idx] = (uint16_t)(hi - lo + (int32_t)window_bp);
            }
            M += cnt;
        }
    }
    __syncwarp();
    if (M == 0) return GB_ITEM_OK;

    // ---- index lookup + score ----------------------------------------------------------------------
#pragma unroll 1
    for (uint32_t a = lane; a < M; a += 32) {
        const uint64_t key = sm.m_key[a];
        uint64_t h = gbmin::hash64(key) & ix.table_mask;
        uint32_t off = 0, cnt = 0;
#pragma unroll 1
        while (true) {
            const uint4 cell = __ldg(reinterpret_cast<const uint4*>(ix.table) + h);
            const uint64_t ckey = ((uint64_t)cell.y << 32) | cell.x;
            if (ckey == GB_NO_KEY) break;
            if (ckey == key) { off = cell.z; cnt = cell.w; break; }
            h = (h + 1) & ix.table_mask;
        }
        sm.m_hit_off[a] = off; sm.m_hit_cnt[a] = cnt;
        sm.m_score[a] = cnt == 0 ? 0.0 : (cnt <= P.hard_hit_cap ? P.hit_score_table[cnt] : 1.0);
    }
    __syncwarp();

    // ---- score order (stable rank sort on (score desc, key asc)) -----------------------------------
#pragma unroll 1
    for (uint32_t a = lane; a < M; a += 32) {
        const double sa = sm.m_score[a]; const uint64_t ka = sm.m_key[a];
        uint32_t rank = 0;
        for (uint32_t b = 0; b < M; b++) {
            const double sb = sm.m_score[b]; const uint64_t kb = sm.m_key[b];
            const bool before = sb > sa || (sb == sa && (kb < ka || (kb == ka && b < a)));
            rank += before ? 1u : 0u;
        }
        sm.m_order[rank] = (uint8_t)a;
    }
    __syncwarp();

    // ---- shuffle the runs tied at the top score (sort_shuffling_ties over runs) ----------------------
    // Runs (equal keys, adjacent after the sort) and the top-score prefix are found by the whole warp;
    // only the Fisher-Yates draws themselves are sequential.
    uint8_t* run_begin = reinterpret_cast<uint8_t*>(sm.khash);          // khash/kkey are dead: scratch
    uint8_t* run_len = run_begin + sm.Mc;
    uint8_t* tmp_order = run_len + sm.Mc;
    auto run_start_words = [&](uint32_t* rsw) {
#pragma unroll
        for (uint32_t t = 0; t < PRESENT_WORDS; t++) {
            const uint32_t i = lane + 32 * t;
            bool rs = false;
            if (i < M) rs = i == 0 || sm.m_key[sm.m_order[i - 1]] != sm.m_key[sm.m_order[i]];
            rsw[t] = __ballot_sync(FULL, rs);
        }
    };
    // first run start after position i (or `end`)
    auto next_run_start = [&](const uint32_t* rsw, uint32_t i, uint32_t end) {
        uint32_t nxt = end;
        bool found = false;
#pragma unroll
        for (uint32_t t = 0; t < PRESENT_WORDS; t++) {
            uint32_t m = rsw[t];
            if (t < (i >> 5)) m = 0;
            else if (t == (i >> 5)) m &= ~((2u << (i & 31)) - 1u);
            if (!found && m) { nxt = 32 * t + (uint32_t)__ffs(m) - 1; found = true; }
        }
        return min(nxt, end);
    };
    uint32_t rsw[PRESENT_WORDS];
    run_start_words(rsw);
    {
        const double top = sm.m_score[sm.m_order[0]];
        uint32_t tied_end = 0, T = 0;
        uint32_t tiew[PRESENT_WORDS];
#pragma unroll
        for (uint32_t t = 0; t < PRESENT_WORDS; t++) {
            const uint32_t i = lane + 32 * t;
            tiew[t] = __ballot_sync(FULL, i < M && sm.m_score[sm.m_order[i]] == top);
            tied_end += __popc(tiew[t]); T += __popc(tiew[t] & rsw[t]);
        }
        if (T > 1) {
            uint32_t before = 0;
#pragma unroll
            for (uint32_t t = 0; t < PRESENT_WORDS; t++) {
                const uint32_t i = lane + 32 * t;
                const uint32_t starts = tiew[t] & rsw[t];
                if ((starts >> lane) & 1u) {
                    const uint32_t q = before + __popc(starts & ((1u << lane) - 1u));
                    run_begin[q] = (uint8_t)i; run_len[q] = (uint8_t)(next_run_start(rsw, i, tied_end) - i);
                }
                before += __popc(starts);
            }
            __syncwarp();
            // Knuth shuffle, swap(i, rng() % (i + 1)) for i = 1 .. T-1 (utility.hpp:722-728): the T - 1 draws are taken by the
            // lanes in parallel (draw i is 48271^i away from the state), only the swaps themselves stay in order
            {
                uint8_t* draw_j = tmp_order;                                   // [T] scratch until the runs are laid out below
#pragma unroll 1
                for (uint32_t i = 1 + lane; i < T; i += 32) draw_j[i] = (uint8_t)(rng_peek(rng, i) % (i + 1));
                __syncwarp();
                if (lane == 0) {
#pragma unroll 1
                    for (uint32_t i = 1; i < T; i++) {
                        const uint32_t j = draw_j[i];
                        const uint8_t tb = run_begin[j], tl = run_len[j];
                        run_begin[j] = run_begin[i]; run_len[j] = run_len[i];
                        run_begin[i] = tb; run_len[i] = tl;
                    }
                }
                rng_skip(rng, T - 1);
            }
            __syncwarp();
            uint32_t carry = 0;
#pragma unroll 1
            for (uint32_t qb = 0; qb < T; qb += 32) {
                const uint32_t q = qb + lane;
                const uint32_t len = q < T ? run_len[q] : 0u;
                const uint32_t incl = (uint32_t)warp_incl_scan((int)len);
                const uint32_t wstart = carry + incl - len;
                if (q < T) for (uint32_t x = 0; x < len; x++) tmp_order[wstart + x] = sm.m_order[run_begin[q] + x];
                carry += __shfl_sync(FULL, incl, 31);
            }
            __syncwarp();
#pragma unroll 1
            for (uint32_t x = lane; x < tied_end; x += 32) sm.m_order[x] = tmp_order[x];
            __syncwarp();
            run_start_words(rsw);                      // runs moved as blocks: new start positions
        }
    }
    rng.state = __shfl_sync(FULL, rng.state, 0); rng.inited = __shfl_sync(FULL, rng.inited, 0);
    __syncwarp();

    // ---- find_seeds filter cascade ------------------------------------------------------------------------
    const uint32_t num_min_by_read_len_ = L / P.num_bp_per_min;
    const bool track_cov_ = P.max_unique_min != 0 && M > max(P.max_unique_min, num_min_by_read_len_);
    uint32_t total_hits = 0;
    if (!track_cov_) {
        // The read-coverage stage cannot reject anything while fewer than max(max_unique_min, L / num_bp_per_min)
        // minimizers have passed, i.e. for every read the tables can hold with default parameters.  Per-position
        // inputs (hits, score, run hits, run start) are staged by the warp; the running-score chain stays sequential.
        uint32_t* s_hits = reinterpret_cast<uint32_t*>(sm.khash);           // [M]
        uint32_t* s_runhits = s_hits + M;                                    // [M]  bit 31 = run start
        double* s_score = reinterpret_cast<double*>(sm.kkey);                // [M]
#pragma unroll 1
        for (uint32_t i = lane; i < M; i += 32) { const uint32_t a = sm.m_order[i]; s_hits[i] = sm.m_hit_cnt[a]; s_score[i] = sm.m_score[a]; }
        __syncwarp();
#pragma unroll
        for (uint32_t t = 0; t < PRESENT_WORDS; t++) {
            const uint32_t i = lane + 32 * t;
            if ((rsw[t] >> lane) & 1u) {
                const uint32_t e = next_run_start(rsw, i, M);
                uint32_t sum = 0;
                for (uint32_t j = i; j < e; j++) sum += s_hits[j];
                for (uint32_t j = i; j < e; j++) s_runhits[j] = sum | (j == i ? 0x80000000u : 0u);
            }
        }
        __syncwarp();
        // When no minimizer has more than hit_cap hits, the hit-cap||score-fraction clause passes every minimizer that
        // reaches it, so the target score is never lowered and the running state cannot change a decision: passing is
        // hits > 0 && run hits <= hard_hit_cap, one position per lane.
        const bool use_fraction = (P.hit_cap != 0 || P.minimizer_score_fraction != 1.0);
        bool over_cap = false;
#pragma unroll 1
        for (uint32_t i = lane; i < M; i += 32) over_cap |= s_hits[i] > P.hit_cap;
        if (!use_fraction || !__any_sync(FULL, over_cap)) {
            uint32_t hits_sum = 0;
#pragma unroll 1
            for (uint32_t i = lane; i < M; i += 32) {
                const uint32_t hits = s_hits[i];
                const bool passing = hits > 0 && (s_runhits[i] & 0x7fffffffu) <= P.hard_hit_cap;
                sm.m_pass[i] = passing ? 1 : 0;
                hits_sum += passing ? hits : 0u;
            }
            total_hits = (uint32_t)warp_sum((int)hits_sum);
        } else if (lane == 0) {
            double base_target_score = 0.0, target_score = 0.0, selected_score = 0.0;
            if (use_fraction) {
                for (uint32_t i = 0; i < M; i++) base_target_score += s_score[i];
                target_score = (base_target_score * P.minimizer_score_fraction) + 0.000001;
            }
            bool taking_run = false;
            for (uint32_t i = 0; i < M; i++) {
                const uint32_t hits = s_hits[i], rh = s_runhits[i], run_hits = rh & 0x7fffffffu;
                if (rh >> 31) taking_run = false;
                bool passing = hits > 0 && run_hits <= P.hard_hit_cap;             // any-hits, hard-hit-cap
                if (passing && use_fraction) {                                      // hit-cap||score-fraction
                    const double score = s_score[i];
                    passing = (hits <= P.hit_cap) || (run_hits <= P.hard_hit_cap && selected_score + score <= target_score) || taking_run;
                    if (passing) selected_score += score; else target_score = selected_score;
                }
                sm.m_pass[i] = passing ? 1 : 0;
                if (passing) { taking_run = true; total_hits += hits; }
            }
        }
        total_hits = __shfl_sync(FULL, total_hits, 0);
        __syncwarp();
    } else {
        // general path (coverage vector in use): sequential running state on lane 0
    if (lane == 0) {
        double base_target_score = 0.0, target_score = 0.0, selected_score = 0.0;
        const bool use_fraction = (P.hit_cap != 0 || P.minimizer_score_fraction != 1.0);
        if (use_fraction) {
#pragma unroll 1
            for (uint32_t i = 0; i < M; i++) base_target_score += sm.m_score[sm.m_order[i]];
            target_score = (base_target_score * P.minimizer_score_fraction) + 0.000001;
        }
        uint32_t limit = 0, run_hits = 0; bool taking_run = false;
        uint32_t num_minimizers = 0, worst_kept_hits = 0;
        const uint32_t num_min_by_read_len = L / P.num_bp_per_min;
        uint32_t* cov = reinterpret_cast<uint32_t*>(sm.kkey);          // read_coverage bit vector
        const uint32_t cov_words = (L + 31) / 32;
        // the coverage vector is only consulted once num_minimizers reaches the cap below, which the
        // M minimizers of this read cannot do when M <= cap: skip its upkeep then
        const uint32_t unique_cap = max(P.max_unique_min, num_min_by_read_len);
        const bool track_cov = M > unique_cap;
        if (track_cov) for (uint32_t x = 0; x < cov_words; x++) cov[x] = 0;
#pragma unroll 1
        for (uint32_t i = 0; i < M; i++) {
            const uint32_t a = sm.m_order[i];
            if (i >= limit) {
                limit = i + 1; run_hits = sm.m_hit_cnt[a];
#pragma unroll 1
                for (uint32_t j = i + 1; j < M && sm.m_key[sm.m_order[j]] == sm.m_key[a]; j++) { limit++; run_hits += sm.m_hit_cnt[sm.m_order[j]]; }
                taking_run = false;
            }
            const uint32_t hits = sm.m_hit_cnt[a];
            const double score = sm.m_score[a];
            bool passing = hits > 0;                                        // any-hits
            if (passing) passing = run_hits <= P.hard_hit_cap;             // hard-hit-cap
            if (passing && P.max_unique_min != 0) {                        // max-min||num-bp-per-min
                const uint32_t fwd = sm.m_fwd[a];
                const uint32_t cs = fwd < P.minimizer_coverage_flank ? 0 : fwd - P.minimizer_coverage_flank;
                const uint32_t ce = min(L, fwd + k + P.minimizer_coverage_flank);
                if (num_minimizers < unique_cap) {
                    if (track_cov) set_bit_range(cov, cs, ce);
                    worst_kept_hits = max(hits, worst_kept_hits);
                } else if (hits > worst_kept_hits) {
                    passing = false;
                } else {
                    if (any_bit_in_range(cov, cs, ce)) passing = false;
                    else set_bit_range(cov, cs, ce);
                }
            }
            if (passing && use_fraction) {                                  // hit-cap||score-fraction
                passing = (hits <= P.hit_cap) || (run_hits <= P.hard_hit_cap && selected_score + score <= target_score) || taking_run;
                if (passing) selected_score += score; else target_score = selected_score;
            }
            sm.m_pass[i] = passing ? 1 : 0;
            if (passing) { taking_run = true; num_minimizers++; total_hits += hits; }
        }
    }
    total_hits = __shfl_sync(FULL, total_hits, 0);
    __syncwarp();

    }

    // ---- minimizer records (score order) -------------------------------------------------------------------
    uint32_t min_off = 0;
    if (!pool_claim(pools.min_cursor, M, pools.min_cap, pools.overflow, min_off)) return GB_ITEM_OUT_FULL;
#pragma unroll 1
    for (uint32_t i = lane; i < M; i += 32) {
        const uint32_t a = sm.m_order[i];
        DevMinimizer dm; dm.hash = sm.m_hash[a]; dm.score = sm.m_score[a]; dm.fwd_offset = sm.m_fwd[a];
        dm.agg_start = sm.m_agg_start[a]; dm.agg_len = sm.m_agg_len[a]; dm.is_reverse = sm.m_rev[a]; dm.pad[0] = sm.m_hit_off[a]; dm.pad[1] = sm.m_hit_cnt[a];     // hit list (seeds_in_subgraph of mate rescue)
        pools.minimizers[min_off + i] = dm;
    }
    rs.min_off = min_off; rs.min_cnt = M;
    if (total_hits == 0) return GB_ITEM_OK;

    // ---- seeds ----------------------------------------------------------------------------------------------
    uint32_t seed_off = 0;
    if (!pool_claim(pools.seed_cursor, total_hits, pools.seed_cap, pools.overflow, seed_off)) return GB_ITEM_OUT_FULL;
    DevSeed* seeds = pools.seeds + seed_off;
    {
        // one lane per (minimizer, hit): exclusive prefix of the passing minimizers' hit counts, then
        // each seed index finds its minimizer by binary search (seed order = score order, hit order)
        uint32_t* pre = reinterpret_cast<uint32_t*>(sm.khash);             // [M + 1]
        uint32_t carry = 0;
#pragma unroll 1
        for (uint32_t base = 0; base < M; base += 32) {
            const uint32_t i = base + lane;
            const uint32_t h = (i < M && sm.m_pass[i]) ? sm.m_hit_cnt[sm.m_order[i]] : 0u;
            const uint32_t incl = (uint32_t)warp_incl_scan((int)h);
            if (i < M) pre[i] = carry + incl - h;
            carry += __shfl_sync(FULL, incl, 31);
        }
        if (lane == 0) pre[M] = carry;
        __syncwarp();
#pragma unroll 1
        for (uint32_t idx = lane; idx < total_hits; idx += 32) {
            uint32_t lo = 0, hi = M;                                         // last i with pre[i] <= idx
#pragma unroll 1
            while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (pre[mid] <= idx) lo = mid; else hi = mid; }
            const uint32_t i = lo, j = idx - pre[lo];
            const uint32_t a = sm.m_order[i];
            const bool rev = sm.m_rev[a];
            const gb_hit* hp = ix.hits + sm.m_hit_off[a] + j;
            // gb_hit is 24 bytes (8-byte aligned): three 64-bit loads
            const uint2 pw = __ldg(reinterpret_cast<const uint2*>(hp));
            const uint2 p1 = __ldg(reinterpret_cast<const uint2*>(hp) + 1);
            const uint2 p2 = __ldg(reinterpret_cast<const uint2*>(hp) + 2);
            const uint64_t pos = ((uint64_t)pw.y << 32) | pw.x;
            uint32_t node = (uint32_t)(pos >> 10), off = (uint32_t)(pos & 1023u);
            const uint32_t nlen = load_node(ix, node).len;
            if (rev) { node ^= 1u; off = nlen - off - 1; }          // reverse_base_pos, :4462-4465
            const uint32_t off_f = (node & 1u) ? nlen - 1 - off : off;
            DevSeed sd;
            sd.node = node; sd.offset = off; sd.source = i; sd.label = idx;
            sd.c_in = (int32_t)p1.x + (int32_t)off_f;
            sd.c_out = (int32_t)p1.y - (int32_t)(nlen - off_f);
            sd.slot = p2.x;
            seeds[idx] = sd;
        }
    }
    rs.seed_off = seed_off; rs.seed_cnt = total_hits;
    __syncwarp();
    return GB_ITEM_OK;
}

// Label propagation: every seed's label becomes the smallest label reachable within `limit`.
__device__ __forceinline__ void propagate_labels(const DevIndex& ix, DevSeed* seeds_a, uint32_t na, DevSeed* seeds_b, uint32_t nb, int32_t limit) {
    const int lane = lane_id();
    const uint32_t n = na + nb;
#pragma unroll 1
    while (true) {
        bool changed = false;
#pragma unroll 1
        for (uint32_t i = lane; i < n; i += 32) {
            DevSeed* pi = i < na ? seeds_a + i : seeds_b + (i - na);
            const DevSeed si = *pi;
            uint32_t best = si.label;
            for (uint32_t j = 0; j < n; j++) {
                if (j == i) continue;
                const DevSeed* pj = j < na ? seeds_a + j : seeds_b + (j - na);
                const uint32_t lj = pj->label;
                if (lj < best && seeds_within(ix, si, *pj, limit)) best = lj;
            }
            if (best != si.label) { pi->label = best; changed = true; }
        }
        __syncwarp();
        if (!__any_sync(FULL, changed)) break;
    }
}

// Scratch of the cluster phases, carved from the shared arrays that are dead once phase A has
// written its records (khash .. m_score are contiguous: Lc * 16 + Mc * 24 bytes).
struct ClusterScratch {
    uint32_t* startbits;   // [16]   k-mer start bitmap of one cluster (coverage)
    double* fs0; double* fs1; double* fc0; double* fc1;   // [F] per-fragment best score / coverage per read
    uint32_t* side;        // [2 * Cc] fragment label of each read cluster
    uint8_t* fo;           // [F]
    uint8_t* has_pair;     // [F]
    uint32_t F;
    // joint clustering of small seed sets in shared memory (whatever is left of the dead arrays)
    uint4* seedbuf;        // [ns_cap]  (node id, c_in, c_out, slot)
    uint8_t* lab_frag;     // [ns_cap]  fragment label (index in the concatenation of both reads)
    uint8_t* lab_read;     // [ns_cap]  read-cluster label (same index space)
    uint32_t ns_cap;       // <= 64
};
__host__ __device__ inline uint32_t cluster_scratch_fragments(uint32_t Cc) { return 2 * Cc < MAX_FRAGMENTS ? 2 * Cc : MAX_FRAGMENTS; }
__host__ __device__ inline size_t cluster_scratch_bytes(uint32_t Cc) { const size_t F = cluster_scratch_fragments(Cc); return 64 + 32 * F + 8 * (size_t)Cc + 2 * F; }
__host__ __device__ inline size_t seed_dead_bytes(uint32_t Lc, uint32_t Mc) { return (size_t)Lc * 16 + (size_t)Mc * 24; }
__device__ __forceinline__ ClusterScratch carve_cluster_scratch(const SeedSmem& sm) {
    ClusterScratch cs;
    uint8_t* p = reinterpret_cast<uint8_t*>(sm.khash);
    cs.F = cluster_scratch_fragments(sm.Cc);
    cs.startbits = (uint32_t*)p; p += 64;
    cs.fs0 = (double*)p; p += 8 * cs.F; cs.fs1 = (double*)p; p += 8 * cs.F;
    cs.fc0 = (double*)p; p += 8 * cs.F; cs.fc1 = (double*)p; p += 8 * cs.F;
    cs.side = (uint32_t*)p; p += 8 * sm.Cc;
    cs.fo = p; p += cs.F; cs.has_pair = p; p += cs.F;
    const size_t used = ((size_t)(p - reinterpret_cast<uint8_t*>(sm.khash)) + 15) & ~(size_t)15;
    const size_t dead = seed_dead_bytes(sm.Lc, sm.Mc);
    cs.ns_cap = dead > used ? (uint32_t)min((size_t)min(64u, sm.ns_max), (dead - used) / 18) : 0u;
    cs.seedbuf = reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(sm.khash) + used);
    cs.lab_frag = reinterpret_cast<uint8_t*>(cs.seedbuf + cs.ns_cap); cs.lab_read = cs.lab_frag + cs.ns_cap;
    return cs;
}

// Clusters of one read in order of their first seed + score_cluster (:4738-4780), one cluster at
// a time with the warp sharing the work.  Cluster c of this read is stored at table index
// cbase + c.  Returns C, or 0xffffffff on overflow.
__device__ __forceinline__ uint32_t collect_clusters(const SeedSmem& sm, const ClusterScratch& cs, const DevSeed* seeds, uint32_t H,
                                                     const DevMinimizer* mins, uint32_t M, uint32_t k, uint32_t L, uint32_t cbase) {
    const int lane = lane_id();
    uint32_t Cn = 0;
#pragma unroll 1
    for (uint32_t base = 0; base < H; base += 32) {
        const uint32_t i = base + lane;
        const bool root = i < H && seeds[i].label == i;
        const uint32_t bal = __ballot_sync(FULL, root);
        if (Cn + __popc(bal) > sm.Cc) return 0xffffffffu;
        if (root) sm.c_label[cbase + Cn + __popc(bal & ((1u << lane) - 1u))] = i;
        Cn += __popc(bal);
    }
    __syncwarp();
    // this lane's share of the minimizer records (score order): score and forward offset
    double mscore[PRESENT_WORDS]; uint32_t mfwd[PRESENT_WORDS];
#pragma unroll
    for (uint32_t t = 0; t < PRESENT_WORDS; t++) {
        const uint32_t j = lane + 32 * t;
        mscore[t] = 0.0; mfwd[t] = 0;
        if (j < M) { const DevMinimizer dm = mins[j]; mscore[t] = dm.score; mfwd[t] = dm.fwd_offset; }
    }
    const uint32_t n_words = (L + 31) >> 5;
#pragma unroll 1
    for (uint32_t c = 0; c < Cn; c++) {
        const uint32_t label = sm.c_label[cbase + c];
        uint32_t present[PRESENT_WORDS];
#pragma unroll
        for (uint32_t x = 0; x < PRESENT_WORDS; x++) present[x] = 0;
#pragma unroll 1
        for (uint32_t i = lane; i < H; i += 32) {
            const DevSeed sd = seeds[i];
            if (sd.label == label) {
                const uint32_t bit = 1u << (sd.source & 31), wd = sd.source >> 5;
#pragma unroll
                for (uint32_t x = 0; x < PRESENT_WORDS; x++) present[x] |= wd == x ? bit : 0u;
            }
        }
#pragma unroll
        for (uint32_t x = 0; x < PRESENT_WORDS; x++) present[x] = __reduce_or_sync(FULL, present[x]);
        // score: minimizer scores summed in score order (same order as the sequential loop of the reference)
        double score = 0.0;
#pragma unroll
        for (uint32_t x = 0; x < PRESENT_WORDS; x++) {
            uint32_t bits = present[x];
#pragma unroll 1
            while (bits) { const int bpos = __ffs(bits) - 1; bits &= bits - 1; score += __shfl_sync(FULL, mscore[x], bpos); }
        }
        // coverage: a base is covered when a present minimizer's k-mer starts in (pos - k, pos]
        if (lane < 16) cs.startbits[lane] = 0;
        __syncwarp();
#pragma unroll
        for (uint32_t x = 0; x < PRESENT_WORDS; x++)
            if ((present[x] >> lane) & 1u) atomicOr(&cs.startbits[mfwd[x] >> 5], 1u << (mfwd[x] & 31));
        __syncwarp();
        uint32_t cnt = 0;
#pragma unroll 1
        for (uint32_t wd = 0; wd < n_words; wd++) {
            const uint32_t pos = wd * 32 + lane;
            const bool covered = pos < L && any_bit_in_range(cs.startbits, pos + 1 > k ? pos + 1 - k : 0u, pos + 1);
            cnt += __popc(__ballot_sync(FULL, covered));
        }
        if (lane == 0) {
            sm.c_score[cbase + c] = score;
            sm.c_cov[cbase + c] = (double)cnt / (double)L;
#pragma unroll
            for (uint32_t x = 0; x < PRESENT_WORDS; x++) sm.c_present[(cbase + c) * PRESENT_WORDS + x] = present[x];
        }
        __syncwarp();
    }
    return Cn;
}

// Emit the work items of one read for the kept clusters kept[0..n_kept) (table indices cbase + c).
__device__ __forceinline__ uint32_t emit_items(const DevIndex& ix, const SeedSmem& sm, const SeedPools& pools, const DevSeed* seeds, uint32_t H,
                                               const DevMinimizer* mins, uint32_t read_idx, const uint8_t* kept, uint32_t n_kept, uint32_t cbase,
                                               uint32_t& item_off_out, const uint8_t* cflags = nullptr) {
    const int lane = lane_id();
    item_off_out = 0;
    if (n_kept == 0) return GB_ITEM_OK;
    uint32_t item_off = 0;
    if (!pool_claim(pools.item_cursor, n_kept, pools.item_cap, pools.overflow, item_off)) return GB_ITEM_OUT_FULL;
    // one ext_seeds range for the whole read, the items' seeds back to back in kept order
    uint32_t total = 0;
#pragma unroll 1
    for (uint32_t t = 0; t < n_kept; t++) {
        const uint32_t label = sm.c_label[cbase + kept[t]];
#pragma unroll 1
        for (uint32_t i = lane; i < H; i += 32) total += seeds[i].label == label ? 1u : 0u;
    }
    total = (uint32_t)warp_sum((int)total);
    uint32_t eoff = 0;
    if (!pool_claim(pools.ext_cursor, total, pools.ext_cap, pools.overflow, eoff)) return GB_ITEM_OUT_FULL;
#pragma unroll 1
    for (uint32_t t = 0; t < n_kept; t++) {
        const uint32_t c = kept[t];
        const uint32_t label = sm.c_label[cbase + c];
        uint32_t wpos = 0;
#pragma unroll 1
        for (uint32_t base = 0; base < H; base += 32) {
            const uint32_t i = base + lane;
            const bool mine = i < H && seeds[i].label == label;
            const uint32_t bal = __ballot_sync(FULL, mine);
            if (mine) {
                const DevSeed s = seeds[i];
                const DevMinimizer dm = mins[s.source];
                const int32_t pin = (int32_t)dm.fwd_offset + (dm.is_reverse ? (int32_t)ix.k - 1 : 0);   // value.offset
                gb_seed g; g.node = s.node; g.diag = pin - (int32_t)s.offset;                      // to_seed, gbwt_extender.hpp:159
                pools.ext_seeds[eoff + wpos + __popc(bal & ((1u << lane) - 1u))] = g;
            }
            wpos += __popc(bal);
        }
        if (lane == 0) {
            DevItem it; it.read = read_idx; it.seed_off = eoff; it.seed_cnt = wpos;
            it.fragment = sm.c_frag[cbase + c] | (cflags ? (uint32_t)cflags[c] << 8 : 0u);         // deferred selection flags, see cluster_phase_pe
#pragma unroll
            for (uint32_t x = 0; x < PRESENT_WORDS; x++) it.present[x] = sm.c_present[(cbase + c) * PRESENT_WORDS + x];
            pools.items[item_off + t] = it;
        }
        eoff += wpos;
    }
    item_off_out = item_off;
    return GB_ITEM_OK;
}

// -----------------------------------------------------------------------------------------
// Phase B, single-end: clusters, selection (minimizer_mapper.cpp:640-832), items.
// -----------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_phase_se(const DevIndex& ix, const MapParamsDev& P, const SeedSmem& sm, uint32_t L, uint32_t read_idx,
                                                     const SeedPools& pools, DevRng& rng, ReadState& rs) {
    const int lane = lane_id();
    const uint32_t H = rs.seed_cnt, M = rs.min_cnt;
    if (H == 0) return GB_ITEM_OK;
    DevSeed* seeds = pools.seeds + rs.seed_off;
    const DevMinimizer* mins = pools.minimizers + rs.min_off;
    const ClusterScratch cs = carve_cluster_scratch(sm);
    const int32_t limit = (int32_t)max(P.distance_limit, L + 50);      // get_distance_limit, minimizer_mapper.hpp:554
    propagate_labels(ix, seeds, H, seeds, 0, limit);
    const uint32_t Cn = collect_clusters(sm, cs, seeds, H, mins, M, ix.k, L, 0);
    if (Cn == 0xffffffffu) return table_full(sm.Cc, MAX_CLUSTERS);
    rs.n_clusters = Cn;
#pragma unroll 1
    for (uint32_t c = lane; c < Cn; c += 32) sm.c_frag[c] = 0;

    uint32_t n_kept = 0;
    uint8_t* kept = sm.scratch;
    if (lane == 0) {
        double best_cluster_score = 0.0, second_best_cluster_score = 0.0;
#pragma unroll 1
        for (uint32_t c = 0; c < Cn; c++) {
            const double sc = sm.c_score[c];
            if (sc > best_cluster_score) { second_best_cluster_score = best_cluster_score; best_cluster_score = sc; }
            else if (sc > second_best_cluster_score) second_best_cluster_score = sc;
        }
        double cluster_score_cutoff = best_cluster_score - P.cluster_score_threshold;
        if (cluster_score_cutoff - P.pad_cluster_score_threshold < second_best_cluster_score)
            cluster_score_cutoff = min(cluster_score_cutoff, second_best_cluster_score);
        auto comes_before = [&](uint32_t a, uint32_t b) {
            return (sm.c_cov[a] > sm.c_cov[b]) || (sm.c_cov[a] == sm.c_cov[b] && sm.c_score[a] > sm.c_score[b]);
        };
        sort_shuffling_ties(Cn, comes_before, sm.c_order, rng);
        const double cutoff = Cn == 0 ? 0.0 : sm.c_cov[sm.c_order[0]] - P.cluster_coverage_threshold;
        uint32_t unskipped = 0, kept_cluster_count = 0;
#pragma unroll 1
        for (uint32_t i = 0; i < Cn; i++) {
            const uint32_t c = sm.c_order[i];
            bool process;
            if (P.cluster_coverage_threshold != 0 && sm.c_cov[c] <= cutoff) process = unskipped < P.min_extensions;
            else process = unskipped < P.max_extensions;
            if (!process) continue;
            if (P.cluster_score_threshold != 0 && sm.c_score[c] < cluster_score_cutoff && kept_cluster_count >= P.min_extensions) continue;
            kept[n_kept++] = (uint8_t)c;
            kept_cluster_count++; unskipped++;
        }
    }
    n_kept = __shfl_sync(FULL, n_kept, 0);
    rng.state = __shfl_sync(FULL, rng.state, 0); rng.inited = __shfl_sync(FULL, rng.inited, 0);
    __syncwarp();
    dbg_dump_clusters(pools, sm, read_idx, 0, Cn, kept, n_kept);
    uint32_t item_off = 0;
    const uint32_t st = emit_items(ix, sm, pools, seeds, H, mins, read_idx, kept, n_kept, 0, item_off);
    if (st == GB_ITEM_OK) { rs.item_off = item_off; rs.item_cnt = n_kept; }
    return st;
}

// -----------------------------------------------------------------------------------------
// Phase B, paired-end: joint clustering (snarl_seed_clusterer.cpp:65-145), fragment bookkeeping
// and per-read selection (minimizer_mapper.cpp:1561-1883).  `gps` is the pair's record in HBM.
// Everything that exists once per read runs in a two-trip loop with a single call site, so the
// (large) helpers are instantiated once.
// -----------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_phase_pe(const DevIndex& ix, const MapParamsDev& P, const SeedSmem& sm,
                                                     uint32_t L0, uint32_t L1, uint32_t read_idx0, int32_t fragment_limit,
                                                     const SeedPools& pools, DevRng& rng, ReadState& rs0, ReadState& rs1, PairState* gps,
                                                     uint32_t& n_fragments_out) {
    const int lane = lane_id();
    // the records' bases are read again from the states at each use rather than held in registers through the phase
    auto seeds_of = [&](uint32_t r) { return pools.seeds + (r ? rs1.seed_off : rs0.seed_off); };
    const uint32_t H0 = rs0.seed_cnt, H1 = rs1.seed_cnt;
    auto mins_of = [&](uint32_t r) -> const DevMinimizer* { return pools.minimizers + (r ? rs1.min_off : rs0.min_off); };
    n_fragments_out = 0;
    if (H0 + H1 == 0) return GB_ITEM_OK;
    const int32_t read_limit = (int32_t)max(P.distance_limit, L0 + 50);
    const ClusterScratch cs = carve_cluster_scratch(sm);

    uint32_t Cn[2] = {0, 0};
    uint32_t overflow = 0;
    const uint32_t n_all = H0 + H1;
    if (n_all <= cs.ns_cap) {
        // ---- small seed sets (the usual case): one pass builds both adjacency relations as 64-bit
        // masks in registers (lane owns seeds lane and lane + 32), components by min-label sweeps
        // over the masks; labels live in shared memory.
#pragma unroll 1
        for (uint32_t i = lane; i < n_all; i += 32) {
            const DevSeed sd = i < H0 ? seeds_of(0)[i] : seeds_of(1)[i - H0];
            cs.seedbuf[i] = make_uint4(sd.node >> 1, (uint32_t)sd.c_in, (uint32_t)sd.c_out, sd.slot);
        }
        __syncwarp();
        bool has[2]; uint64_t adj_f[2] = {0, 0}, adj_r[2] = {0, 0};
#pragma unroll
        for (uint32_t q = 0; q < 2; q++) has[q] = lane + 32 * q < n_all;
        // The distance is unoriented, so the relations are symmetric: lane q walks row q over every column and row q + 32
        // over the columns >= 32; the columns < 32 of rows >= 32 are read back from the first rows by vote.  Pairs of
        // different nodes in one site need the site table (same_site_distance, out of line): they are set aside in
        // `pend` and resolved after the walk, so the call and the registers it saves stay off the row loop.
        auto add_edge = [&](uint32_t row, uint32_t j, int32_t d, uint64_t& af, uint64_t& ar) {
            if (d <= fragment_limit) af |= 1ull << j;
            if (d <= read_limit && (row < H0) == (j < H0)) ar |= 1ull << j;
        };
        auto walk_row = [&](uint32_t row, uint32_t j0, uint64_t& af, uint64_t& ar) {
            const uint4 a = row < n_all ? cs.seedbuf[row] : make_uint4(0, 0, 0, 0);
            uint64_t pend = 0;
#pragma unroll 1
            for (uint32_t j = j0; j < n_all; j++) {
                const uint4 c = cs.seedbuf[j];
                if (row >= n_all || row == j) continue;
                int32_t d;
                if (a.x == c.x) { d = (int32_t)c.y - (int32_t)a.y; d = d >= 0 ? d : -d; }
                else if (a.w < c.w) d = (int32_t)c.y - (int32_t)a.z;
                else if (c.w < a.w) d = (int32_t)a.y - (int32_t)c.z;
                else { pend |= 1ull << j; continue; }
                add_edge(row, j, d, af, ar);
            }
#pragma unroll 1
            while (pend) {
                const uint32_t j = (uint32_t)(__ffsll((long long)pend) - 1); pend &= pend - 1;
                const uint4 c = cs.seedbuf[j];
                const int32_t d = same_site_distance(ix, a.x, (int32_t)a.y, (int32_t)a.z, c.x, (int32_t)c.y, (int32_t)c.z);
                if (d != INT_MAX) add_edge(row, j, d, af, ar);
            }
        };
        walk_row(lane, 0, adj_f[0], adj_r[0]);
        if (n_all > 32) walk_row(lane + 32, 32, adj_f[1], adj_r[1]);
#pragma unroll 1
        for (uint32_t i = 32; i < n_all; i++) {
            const uint32_t lo_f = __ballot_sync(FULL, (adj_f[0] >> i) & 1ull), lo_r = __ballot_sync(FULL, (adj_r[0] >> i) & 1ull);
            if ((uint32_t)lane + 32 == i) { adj_f[1] |= lo_f; adj_r[1] |= lo_r; }
        }
#pragma unroll 1
        for (uint32_t level = 0; level < 2; level++) {
            uint8_t* lab = level == 0 ? cs.lab_frag : cs.lab_read;
            // Components by min-label sweeps on the masks.  A label starts as the smallest index among the
            // seed and its neighbours; a sweep then lets every seed take the smallest label found among its
            // neighbours, label by label: one pair of warp votes tells which seeds carry label L, and a seed
            // adopts the first (smallest) L whose carriers intersect its row.  Same fixed point as seed-by-seed
            // propagation (the smallest index of the component), in a handful of votes for the usual 1-3 clusters.
            uint32_t mine[2];
#pragma unroll
            for (uint32_t q = 0; q < 2; q++) {
                const uint64_t row = level == 0 ? adj_f[q] : adj_r[q];
                const uint32_t i = lane + 32 * q;
                mine[q] = row ? min(i, (uint32_t)(__ffsll((long long)row) - 1)) : i;
            }
#pragma unroll 1
            while (true) {
                const uint32_t p_lo = __reduce_or_sync(FULL, (has[0] && mine[0] < 32 ? 1u << mine[0] : 0u) | (has[1] && mine[1] < 32 ? 1u << mine[1] : 0u));
                const uint32_t p_hi = __reduce_or_sync(FULL, (has[0] && mine[0] >= 32 ? 1u << (mine[0] - 32) : 0u) | (has[1] && mine[1] >= 32 ? 1u << (mine[1] - 32) : 0u));
                uint64_t present = ((uint64_t)p_hi << 32) | p_lo;
                uint32_t next[2] = {mine[0], mine[1]};
                bool changed = false;
#pragma unroll 1
                while (present) {
                    const uint32_t L = (uint32_t)(__ffsll((long long)present) - 1); present &= present - 1;
                    const uint64_t carriers = (uint64_t)__ballot_sync(FULL, has[0] && mine[0] == L) | ((uint64_t)__ballot_sync(FULL, has[1] && mine[1] == L) << 32);
#pragma unroll
                    for (uint32_t q = 0; q < 2; q++) {
                        const uint64_t row = level == 0 ? adj_f[q] : adj_r[q];
                        if (has[q] && L < next[q] && (row & carriers)) { next[q] = L; changed = true; }
                    }
                }
                mine[0] = next[0]; mine[1] = next[1];
                if (!__any_sync(FULL, changed)) break;
            }
#pragma unroll
            for (uint32_t q = 0; q < 2; q++) if (has[q]) lab[lane + 32 * q] = (uint8_t)mine[q];
            __syncwarp();
        }
        // read-cluster labels back to the records (local index space of each read)
#pragma unroll 1
        for (uint32_t i = lane; i < n_all; i += 32) {
            if (i < H0) seeds_of(0)[i].label = cs.lab_read[i]; else seeds_of(1)[i - H0].label = (uint32_t)cs.lab_read[i] - H0;
        }
        __syncwarp();
#pragma unroll 1
        for (uint32_t r = 0; r < 2; r++) {
            const uint32_t Hr = r ? H1 : H0, g0 = r ? H0 : 0u;
            uint32_t n_roots = 0;
#pragma unroll 1
            for (uint32_t base = 0; base < Hr && !overflow; base += 32) {
                const uint32_t i = base + lane;
                const bool root = i < Hr && cs.lab_read[g0 + i] == g0 + i;
                const uint32_t bal = __ballot_sync(FULL, root);
                if (n_roots + __popc(bal) > sm.Cc) { overflow = 1; break; }
                if (root) cs.side[r * sm.Cc + n_roots + __popc(bal & ((1u << lane) - 1u))] = cs.lab_frag[g0 + i];
                n_roots += __popc(bal);
            }
        }
        __syncwarp();
    } else {
        // ---- large seed sets: label propagation over the records in HBM.
        // pass 0: fragment components over both reads (labels = index in the concatenation), stashed in
        // the upper bits of `source` (source < 128); passes 1, 2: the read clusters of each read.
#pragma unroll 1
        for (uint32_t pass = 0; pass < 3; pass++) {
            DevSeed* sa = seeds_of(pass == 2); const uint32_t na = pass == 2 ? H1 : H0;
            const uint32_t nb = pass == 0 ? H1 : 0u;
#pragma unroll 1
            for (uint32_t i = lane; i < na; i += 32) sa[i].label = i;
#pragma unroll 1
            for (uint32_t i = lane; i < nb; i += 32) seeds_of(1)[i].label = na + i;
            __syncwarp();
            propagate_labels(ix, sa, na, seeds_of(1), nb, pass == 0 ? fragment_limit : read_limit);
            if (pass == 0) {
#pragma unroll 1
                for (uint32_t i = lane; i < H0; i += 32) seeds_of(0)[i].source |= seeds_of(0)[i].label << 8;
#pragma unroll 1
                for (uint32_t i = lane; i < H1; i += 32) seeds_of(1)[i].source |= seeds_of(1)[i].label << 8;
            }
            __syncwarp();
        }
        // the fragment label of each read-cluster root goes to the side table, then `source` is restored
#pragma unroll 1
        for (uint32_t r = 0; r < 2; r++) {
            DevSeed* sr = seeds_of(r); const uint32_t Hr = r ? H1 : H0;
            uint32_t n_roots = 0;
#pragma unroll 1
            for (uint32_t base = 0; base < Hr && !overflow; base += 32) {
                const uint32_t i = base + lane;
                const bool root = i < Hr && sr[i].label == i;
                const uint32_t bal = __ballot_sync(FULL, root);
                if (n_roots + __popc(bal) > sm.Cc) { overflow = 1; break; }
                if (root) cs.side[r * sm.Cc + n_roots + __popc(bal & ((1u << lane) - 1u))] = sr[i].source >> 8;
                n_roots += __popc(bal);
            }
            __syncwarp();
#pragma unroll 1
            for (uint32_t i = lane; i < Hr; i += 32) sr[i].source &= 0xffu;
            __syncwarp();
        }
    }
#pragma unroll 1
    for (uint32_t r = 0; r < 2 && !overflow; r++) {
        const uint32_t cn = collect_clusters(sm, cs, seeds_of(r), r ? H1 : H0, mins_of(r), r ? rs1.min_cnt : rs0.min_cnt, ix.k, r ? L1 : L0, r * sm.Cc);
        if (cn == 0xffffffffu) overflow = 1;
        else if (r) Cn[1] = cn; else Cn[0] = cn;
    }
    if (overflow) return table_full(sm.Cc, MAX_CLUSTERS);
    rs0.n_clusters = Cn[0]; rs1.n_clusters = Cn[1];

    // ---- fragment ids in order of first appearance; per-fragment bests; better_cluster_count --------------
    uint8_t* kept0 = sm.scratch; uint8_t* kept1 = sm.scratch + sm.Cc;
    uint8_t* cflags1 = sm.scratch + 2 * sm.Cc;                   // [Cc <= Mc] keep-decision flags of read 2's clusters (deferred selection)
    uint32_t n_kept0 = 0, n_kept1 = 0, defer_ties = 0;
    uint32_t status = GB_ITEM_OK;
    uint32_t n_frag = 0;
    {
        // fragment renumbering (:129-141 of the clusterer wrapper): fragments are numbered in order of first appearance
        // over read 1's clusters, then read 2's.  Lane g takes cluster g of that concatenation (n_cl <= 2 * Cc <= 32 *
        // PRESENT_WORDS); its fragment id is the number of first appearances before its head's first cluster.
        const uint32_t n_cl = Cn[0] + Cn[1];
        auto slot = [&](uint32_t g) { return g < Cn[0] ? g : sm.Cc + g - Cn[0]; };
        uint32_t first_pos[PRESENT_WORDS], firstw[PRESENT_WORDS];
#pragma unroll
        for (uint32_t t = 0; t < PRESENT_WORDS; t++) {
            const uint32_t g = lane + 32 * t;
            uint32_t fp = g;
            if (g < n_cl) {
                const uint32_t head = cs.side[slot(g)];
#pragma unroll 1
                for (uint32_t x = 0; x < g; x++) if (cs.side[slot(x)] == head) { fp = x; break; }
            }
            first_pos[t] = fp;
            firstw[t] = __ballot_sync(FULL, g < n_cl && fp == g);
            n_frag += __popc(firstw[t]);
        }
#pragma unroll
        for (uint32_t t = 0; t < PRESENT_WORDS; t++) {
            const uint32_t g = lane + 32 * t, fp = first_pos[t];
            if (g < n_cl) {
                uint32_t f = 0;
#pragma unroll
                for (uint32_t x = 0; x < PRESENT_WORDS; x++)
                    f += __popc(firstw[x] & (x < (fp >> 5) ? 0xffffffffu : x == (fp >> 5) ? (1u << (fp & 31)) - 1u : 0u));
                sm.c_frag[slot(g)] = (uint8_t)f;
            }
        }
        __syncwarp();
    }
    if (n_frag > cs.F) status = table_full(sm.Cc, MAX_CLUSTERS);
    else {
        // per-fragment best score and coverage of each read, and whether both reads have a cluster in it: lane f scans the clusters
        bool any_pair = false;
#pragma unroll 1
        for (uint32_t f = lane; f < n_frag; f += 32) {
            bool hf = false, hp = false;
            double bs0 = 0.0, bs1 = 0.0, bc0 = 0.0, bc1 = 0.0;
#pragma unroll 1
            for (uint32_t c = 0; c < Cn[0]; c++) if (sm.c_frag[c] == f) { hf = true; bs0 = max(bs0, sm.c_score[c]); bc0 = max(bc0, sm.c_cov[c]); }
#pragma unroll 1
            for (uint32_t c = sm.Cc; c < sm.Cc + Cn[1]; c++) if (sm.c_frag[c] == f) { hp = hf; bs1 = max(bs1, sm.c_score[c]); bc1 = max(bc1, sm.c_cov[c]); }
            cs.has_pair[f] = hp;
            cs.fs0[f] = bs0; cs.fs1[f] = bs1; cs.fc0[f] = bc0; cs.fc1[f] = bc1;
            any_pair |= hp;
        }
        const bool found_paired_cluster = __any_sync(FULL, any_pair);
        __syncwarp();
        if (lane == 0) {
            double* const fs[2] = {cs.fs0, cs.fs1}; double* const fc[2] = {cs.fc0, cs.fc1};
            uint8_t* has_pair = cs.has_pair; uint8_t* fo = cs.fo;
            // better_cluster_count (:1657-1690)
            auto total = [&](uint32_t f) { return (fc[0][f] + fc[1][f]) + (fs[0][f] + fs[1][f]); };
            sort_shuffling_ties(n_frag, [&](uint32_t x, uint32_t y) { return total(x) > total(y); }, fo, rng);
            double prev_score_sum = 0.0;
            uint8_t* better = gps->better_cluster_count;
#pragma unroll 1
            for (int rank = (int)n_frag - 1; rank >= 0; rank--) {
                const uint32_t f = fo[rank];
                if (rank == (int)n_frag - 1) better[f] = (uint8_t)(rank + 1);
                else {
                    const double curr = total(f);
                    if (curr == prev_score_sum) better[f] = better[fo[rank + 1]];
                    else { better[f] = (uint8_t)(rank + 1); prev_score_sum = curr; }
                }
            }
            gps->n_fragments = n_frag; gps->found_paired_cluster = found_paired_cluster ? 1u : 0u;

            // ---- per-read selection (:1723-1883) ------------------------------------------------------------------
#pragma unroll 1
            for (uint32_t r = 0; r < 2; r++) {
                const uint32_t cb = r * sm.Cc, Cr = r ? Cn[1] : Cn[0];
                double cluster_score_cutoff = 0.0, cluster_coverage_cutoff = 0.0, second_best = 0.0;
                double best_cov = 0.0, best_cov_score = 0.0;
#pragma unroll 1
                for (uint32_t c = 0; c < Cr; c++) {
                    const double cov = sm.c_cov[cb + c], sc = sm.c_score[cb + c];
                    if (cov > best_cov) { best_cov = cov; best_cov_score = sc; }
                    else if (cov == best_cov) best_cov_score = max(best_cov_score, sc);
                    cluster_coverage_cutoff = max(cluster_coverage_cutoff, cov);
                    if (sc > cluster_score_cutoff) { second_best = cluster_score_cutoff; cluster_score_cutoff = sc; }
                    else if (sc > second_best) second_best = sc;
                }
                cluster_score_cutoff -= P.cluster_score_threshold;
                cluster_coverage_cutoff -= P.cluster_coverage_threshold;
                if (cluster_score_cutoff - P.pad_cluster_score_threshold < second_best) cluster_score_cutoff = min(cluster_score_cutoff, second_best);
                auto comes_before = [&](uint32_t a, uint32_t b) {
                    const uint32_t fa = sm.c_frag[cb + a], fb = sm.c_frag[cb + b];
                    const double coverage_a = fc[0][fa] + fc[1][fa], coverage_b = fc[0][fb] + fc[1][fb];
                    const double score_a = fs[0][fa] + fs[1][fa], score_b = fs[0][fb] + fs[1][fb];
                    if (has_pair[fa] != has_pair[fb]) return has_pair[fa] != 0;
                    else if (coverage_a != coverage_b) return coverage_a > coverage_b;
                    else if (score_a != score_b) return score_a > score_b;
                    else if (sm.c_cov[cb + a] != sm.c_cov[cb + b]) return sm.c_cov[cb + a] > sm.c_cov[cb + b];
                    else return sm.c_score[cb + a] > sm.c_score[cb + b];
                };
                uint8_t* order = sm.c_order + cb;
#pragma unroll 1
                for (uint32_t c = 0; c < Cr; c++) { uint32_t j = c; while (j > 0 && comes_before(c, order[j - 1])) { order[j] = order[j - 1]; j--; } order[j] = (uint8_t)c; }
                uint32_t ties = 0;
#pragma unroll 1
                while (ties < Cr && !comes_before(order[0], order[ties])) ties++;
                uint8_t* kept = r == 0 ? kept0 : kept1;
                if (r == 1 && ties > 1) {
                    // The reference draws the tie shuffle of read 2's clusters from the pair's LazyRNG only AFTER read 1's
                    // extension sets and tails have drawn theirs (the per-read loop, :1723-2043).  The draws of that stage
                    // are not known here, so the shuffle and the order-dependent keep loop move to the align stage: every
                    // cluster becomes a work item, in comparator order, carrying the order-independent inputs of the keep
                    // decision as flags (bit 0 eligible, bit 1 below the coverage cutoff, bit 2 below the score cutoff).
#pragma unroll 1
                    for (uint32_t i = 0; i < Cr; i++) {
                        const uint32_t c = order[i];
                        const uint32_t f = sm.c_frag[cb + c];
                        const double cov = sm.c_cov[cb + c], sc = sm.c_score[cb + c];
                        uint8_t fl = 0;
                        if (!found_paired_cluster || has_pair[f] || (cov == best_cov && sc == best_cov_score)) fl |= 1;
                        if (P.cluster_coverage_threshold != 0 && cov < cluster_coverage_cutoff) fl |= 2;
                        if (P.cluster_score_threshold != 0 && sc < cluster_score_cutoff) fl |= 4;
                        cflags1[c] = fl; kept[i] = (uint8_t)c;
                    }
                    n_kept1 = Cr; defer_ties = ties;
                    continue;
                }
#pragma unroll 1
                for (uint32_t i = 1; i < ties; i++) { const uint32_t j = rng_next(rng) % (i + 1); const uint8_t t = order[j]; order[j] = order[i]; order[i] = t; }
                // process_until_threshold_c with threshold 0: everything is "good enough", max_extensions caps
                uint32_t unskipped = 0, kept_cluster_count = 0, nk = 0;
#pragma unroll 1
                for (uint32_t i = 0; i < Cr; i++) {
                    const uint32_t c = order[i];
                    if (unskipped >= P.max_extensions) continue;
                    const uint32_t f = sm.c_frag[cb + c];
                    const double cov = sm.c_cov[cb + c], sc = sm.c_score[cb + c];
                    bool keep = false;
                    if (!found_paired_cluster || has_pair[f] || (cov == best_cov && sc == best_cov_score)) {
                        keep = true;
                        if (P.cluster_coverage_threshold != 0 && cov < cluster_coverage_cutoff && kept_cluster_count >= P.min_extensions) keep = false;
                        else if (P.cluster_score_threshold != 0 && sc < cluster_score_cutoff && kept_cluster_count >= P.min_extensions) keep = false;
                    }
                    if (keep) { kept[nk++] = (uint8_t)c; kept_cluster_count++; unskipped++; }
                }
                if (r == 0) n_kept0 = nk; else n_kept1 = nk;
            }
        }
    }
    status = __shfl_sync(FULL, status, 0);
    n_kept0 = __shfl_sync(FULL, n_kept0, 0); n_kept1 = __shfl_sync(FULL, n_kept1, 0); defer_ties = __shfl_sync(FULL, defer_ties, 0);
    rng.state = __shfl_sync(FULL, rng.state, 0); rng.inited = __shfl_sync(FULL, rng.inited, 0);
    n_fragments_out = __shfl_sync(FULL, n_frag, 0);
    rs1.pad[0] = defer_ties;
    __syncwarp();
    if (status != GB_ITEM_OK) return status;
#pragma unroll 1
    for (uint32_t r = 0; r < 2; r++) {
        uint32_t item_off = 0;
        const uint32_t nk = r ? n_kept1 : n_kept0;
        dbg_dump_clusters(pools, sm, read_idx0 + r, r * sm.Cc, r ? Cn[1] : Cn[0], r ? kept1 : kept0, nk, r && defer_ties);
        const uint32_t st = emit_items(ix, sm, pools, seeds_of(r), r ? H1 : H0, mins_of(r), read_idx0 + r, r ? kept1 : kept0, nk, r * sm.Cc, item_off,
                                       r && defer_ties ? cflags1 : nullptr);
        if (st != GB_ITEM_OK) return st;
        if (r) { rs1.item_off = item_off; rs1.item_cnt = nk; } else { rs0.item_off = item_off; rs0.item_cnt = nk; }
    }
    return GB_ITEM_OK;
}

} // namespace gb
