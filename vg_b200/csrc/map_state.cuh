// map_state.cuh — HBM-resident intermediate records passed between the mapping kernels.
//
//   seed_kernel   (one warp / read): minimizers -> seeds -> clusters -> ordered work items
//   extend_kernel (one warp / item): GaplessExtender::extend
//   align_kernel  (one warp / read): extension scoring, tail alignment, winner, MAPQ, records
//
// Everything is integer except the minimizer / cluster scores and MAPQ (FP64), exactly the
// places where the reference uses double.
#pragma once
#include "device_index.cuh"

namespace gb {

constexpr uint32_t MAX_MINIMIZERS = 128;          // per read (short-read path)
constexpr uint32_t PRESENT_WORDS = MAX_MINIMIZERS / 32;

// LazyRNG (utility.cpp:907-931): std::minstd_rand seeded lazily from the read sequence.
struct DevRng {
    uint32_t state;       // current minstd state (valid when inited)
    uint32_t inited;
    uint32_t seed;        // seedNumber folded from the sequence (always available)
};

__device__ __forceinline__ uint32_t rng_next(DevRng& r) {
    if (!r.inited) {
        // std::minstd_rand(seed): x = seed % 2147483647, 0 -> 1
        uint32_t x = r.seed % 2147483647u;
        r.state = x == 0 ? 1u : x;
        r.inited = 1;
    }
    // x * 48271 mod (2^31 - 1) without a 64-bit division: 2^31 = 1 (mod M), so the product folds as low 31 bits + the rest
    const uint64_t p = (uint64_t)r.state * 48271ull;                 // < 2^47
    uint32_t s = (uint32_t)(p & 0x7fffffffu) + (uint32_t)(p >> 31);  // < 2^31 + 2^16
    if (s >= 2147483647u) s -= 2147483647u;
    r.state = s;
    return r.state;
}

// minstd_rand is a pure multiplicative generator, x_n = 48271^n x_0 mod (2^31 - 1): draw n of a batch is one modular power
// away from the state, so the lanes of a warp can take the next 32 draws at once (tie shuffles) instead of lane 0 walking them.
__device__ __forceinline__ uint32_t minstd_mulmod(uint32_t a, uint32_t b) {
    const uint64_t p = (uint64_t)a * b;                                     // < 2^62
    uint64_t s = (p & 0x7fffffffull) + (p >> 31);                           // < 2^32
    s = (s & 0x7fffffffull) + (s >> 31);
    return s >= 2147483647ull ? (uint32_t)(s - 2147483647ull) : (uint32_t)s;
}
__device__ __forceinline__ uint32_t minstd_pow(uint32_t e) {               // 48271^e mod (2^31 - 1)
    uint32_t r = 1, b = 48271u;
    while (e) { if (e & 1u) r = minstd_mulmod(r, b); b = minstd_mulmod(b, b); e >>= 1; }
    return r;
}
// The n-th next draw (n >= 1) without advancing; rng_skip(r, n) then moves the state past n draws.
__device__ __forceinline__ uint32_t rng_peek(DevRng r, uint32_t n) {
    if (!r.inited) { const uint32_t x = r.seed % 2147483647u; r.state = x == 0 ? 1u : x; }
    return minstd_mulmod(r.state, minstd_pow(n));
}
__device__ __forceinline__ void rng_skip(DevRng& r, uint32_t n) {
    if (n == 0) return;
    if (!r.inited) { const uint32_t x = r.seed % 2147483647u; r.state = x == 0 ? 1u : x; r.inited = 1; }
    r.state = minstd_mulmod(r.state, minstd_pow(n));
}

// sort_shuffling_ties (utility.hpp:770-793): order = 0 .. n - 1 stably sorted by `before(a, b)` (a goes first), then the
// items tied with the first are shuffled with the LazyRNG (deterministic_shuffle: one draw per tied item after the first).
template <typename Before>
__device__ __forceinline__ void sort_shuffling_ties(uint32_t n, Before before, uint8_t* order, DevRng& rng) {
#pragma unroll 1
    for (uint32_t c = 0; c < n; c++) {
        uint32_t j = c;
#pragma unroll 1
        while (j > 0 && before(c, order[j - 1])) { order[j] = order[j - 1]; j--; }
        order[j] = (uint8_t)c;
    }
    uint32_t ties = 0;
#pragma unroll 1
    while (ties < n && !before(order[0], order[ties])) ties++;
#pragma unroll 1
    for (uint32_t i = 1; i < ties; i++) { const uint32_t j = rng_next(rng) % (i + 1); const uint8_t t = order[j]; order[j] = order[i]; order[i] = t; }
}

// One minimizer of the read in SCORE order (MinimizerMapper::Minimizer, minimizer_mapper.hpp:565).
struct __align__(16) DevMinimizer {
    uint64_t hash;
    double   score;
    uint16_t fwd_offset;      // forward_offset()
    uint16_t agg_start;
    uint16_t agg_len;
    uint16_t is_reverse;
    uint32_t pad[2];
};
static_assert(sizeof(DevMinimizer) == 32, "DevMinimizer must be 32 bytes");

// One seed (SnarlDistanceIndexClusterer::Seed) plus its chain coordinates.
struct __align__(16) DevSeed {
    uint32_t node;            // oriented node of pos
    uint32_t offset;          // offset of pos
    uint32_t source;          // minimizer index (score order)
    uint32_t label;           // cluster label = smallest seed index in the component
    int32_t  c_out;           // x_out - (len - off_fwd): coordinate when the seed is the source
    int32_t  c_in;            // x_in + off_fwd:          coordinate when the seed is the target
    uint32_t slot;
};
// A hit's payload is the distance payload of its node id (gb_hit), so two seeds on one node share x_in and their c_in
// differ by their forward offsets: the seed needs no packed (id, offset) word, and node ids keep all 31 bits.
static_assert(sizeof(DevSeed) == 32, "DevSeed must be 32 bytes");

// One (read, cluster) work item for the extension kernel, in processing order.
struct __align__(16) DevItem {
    uint32_t read;
    uint32_t seed_off, seed_cnt;          // gb_seed pool
    uint32_t present[PRESENT_WORDS];      // minimizers with a hit in the cluster
    uint32_t fragment;                    // paired-end: fragment cluster of this read cluster
};

// Per-read state carried from seed_kernel to align_kernel.
struct __align__(16) ReadState {
    DevRng rng;
    uint32_t min_off, min_cnt;            // DevMinimizer pool
    uint32_t item_off, item_cnt;          // DevItem pool (contiguous, processing order)
    uint32_t seed_off, seed_cnt;          // DevSeed pool
    uint32_t status;
    uint32_t n_clusters;
    uint32_t pad[4];
};

// Paired-end: per-pair state (fragment clusters), minimizer_mapper.cpp:1568-1690.
constexpr uint32_t MAX_FRAGMENTS = 64;
struct __align__(16) PairState {
    uint32_t n_fragments;                 // max_fragment_num + 1 (0 when there are no clusters)
    uint32_t found_paired_cluster;
    uint32_t pad[2];
    uint8_t  better_cluster_count[MAX_FRAGMENTS];
};

struct MapParamsDev {
    uint32_t hit_cap, hard_hit_cap;
    double   minimizer_score_fraction;
    uint32_t minimizer_coverage_flank, max_unique_min, num_bp_per_min, distance_limit;
    uint32_t min_extensions, max_extensions;
    double   cluster_score_threshold, pad_cluster_score_threshold, cluster_coverage_threshold;
    double   extension_set_score_threshold;
    int32_t  extension_score_threshold, min_extension_sets, extension_set_min_score;
    uint32_t max_alignments, max_extension_mismatches, max_dozeu_cells, do_dp;
    uint32_t mapping_cap, edit_cap;
    uint32_t max_multimaps, out_stride;   // mappings reported per read; records of rank j live at j * out_stride + read (out_stride = reads of the chunk)
    uint32_t max_rescue_attempts, rescue_seed_limit;
    double   paired_rescue_score_limit, rescue_subgraph_stdevs, rescue_likelihood_limit;
    double   log_base;
    const double* hit_score_table;        // [hard_hit_cap + 1]: score for a hit count (host libm)
    const double* prob_at_least_one;      // [(32 + 1) * 256]   (statistics.cpp:525-560)
    const double* phred_prob;             // [256]              (statistics.cpp:471-484)
};

} // namespace gb
