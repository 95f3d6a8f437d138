// ORACLE — TEST INFRASTRUCTURE ONLY.  Shared types of the mapper restatement.
#pragma once
#include "oracle.h"
#include "gbwt_view.hpp"

#include <cmath>
#include <cstdint>
#include <functional>
#include <memory>
#include <random>
#include <string>
#include <vector>

namespace oracle {

// ---- GaplessExtension (oracle/extend.cpp) ---------------------------------------------
} // namespace oracle
#include "extension.hpp"
namespace oracle {
struct ExtendTrace;
std::vector<GaplessExtension> extend(const Graph& g, const gb_scores& scores,
                                     const std::vector<std::pair<uint32_t, int64_t>>& cluster,
                                     std::string sequence, size_t max_mismatches,
                                     double overlap_threshold, bool trim, ExtendTrace* trace = nullptr);

// ---- LazyRNG, utility.cpp:907-931 / utility.hpp:698-794 -------------------------------
class LazyRNG {
public:
    explicit LazyRNG(std::function<std::string(void)> get_seed) : get_seed(std::move(get_seed)) {}
    std::minstd_rand::result_type operator()() {
        if (!rng) {
            std::string seed = get_seed();
            uint32_t seedNumber = 0;
            for (uint8_t byte : seed) seedNumber = seedNumber * 13 + byte;
            rng = std::make_unique<std::minstd_rand>(seedNumber);
        }
        return (*rng)();
    }
private:
    std::function<std::string(void)> get_seed;
    std::unique_ptr<std::minstd_rand> rng;
};

inline bool deterministic_flip(LazyRNG& rng) { return rng() % 2; }

template <class RandomIt>
void deterministic_shuffle(RandomIt begin, RandomIt end, LazyRNG& rng) {
    int64_t width = end - begin;
    for (int64_t i = 1; i < width; i++) std::swap(*(begin + (rng() % (i + 1))), *(begin + i));
}

template <typename Number>
bool deterministic_beats(const Number& a, const Number& b, LazyRNG& rng) {
    return (a > b || (a == b && deterministic_flip(rng)));
}

template <class RandomIt, class Compare>
void sort_shuffling_ties(RandomIt begin, RandomIt end, Compare comp, LazyRNG& rng) {
    std::stable_sort(begin, end, comp);
    RandomIt ties_end = begin;
    while (ties_end != end && !comp(*begin, *ties_end)) ++ties_end;
    if (begin != ties_end) deterministic_shuffle(begin, ties_end, rng);
}

// ---- process_until_threshold_e, minimizer_mapper.hpp:1580-1659 ------------------------
template <typename Score>
void process_until_threshold_e(size_t items, const std::function<Score(size_t)>& get_score,
                               const std::function<bool(size_t, size_t)>& comparator,
                               const std::function<bool(size_t)>& threshold_escape,
                               double threshold, size_t min_count, size_t max_count, LazyRNG& rng,
                               const std::function<bool(size_t, size_t, bool)>& process_item,
                               const std::function<void(size_t)>& discard_item_by_count,
                               const std::function<void(size_t)>& discard_item_by_score) {
    std::vector<size_t> indexes_in_order;
    indexes_in_order.reserve(items);
    for (size_t i = 0; i < items; i++) indexes_in_order.push_back(i);
    sort_shuffling_ties(indexes_in_order.begin(), indexes_in_order.end(), comparator, rng);
    std::vector<size_t> better_or_equal_count(items, items);
    for (int i = (int)items - 2; i >= 0; --i) {
        if (comparator(indexes_in_order[i], indexes_in_order[i + 1])) better_or_equal_count[i] = i + 1;
        else better_or_equal_count[i] = better_or_equal_count[i + 1];
    }
    double cutoff = items == 0 ? 0 : get_score(indexes_in_order[0]) - threshold;
    size_t unskipped = 0;
    for (size_t i = 0; i < indexes_in_order.size(); i++) {
        size_t item_num = indexes_in_order[i];
        if (threshold != 0 && get_score(item_num) <= cutoff) {
            bool escape = false;
            if (unskipped < min_count || (escape = threshold_escape(item_num))) {
                unskipped += (size_t)process_item(item_num, better_or_equal_count[i], escape);
            } else {
                discard_item_by_score(item_num);
            }
        } else {
            if (unskipped < max_count) unskipped += (size_t)process_item(item_num, better_or_equal_count[i], false);
            else discard_item_by_count(item_num);
        }
    }
}

// ---- alignment records ----------------------------------------------------------------
struct Edit { uint32_t from_length = 0, to_length = 0; std::string sequence; };
struct Mapping { uint32_t node = 0; uint32_t offset = 0; std::vector<Edit> edits; };
struct Alignment {
    std::vector<Mapping> path;
    int32_t score = 0;
    double identity = 0;
    double mapq = 0;
    double mapq_uncapped = 0, mapq_explored_cap = 0;
    bool rescued = false;
    bool secondary = false;                    // set_is_secondary (:1205, :2555)
    std::vector<Alignment> secondaries;        // on a primary: mappings 1 .. max_multimaps - 1 in output order
};

// MinimizerMapper::Minimizer, minimizer_mapper.hpp:565-621
struct Minimizer {
    uint64_t key = 0, hash = 0;
    uint32_t offset = 0;          // value.offset (pin offset)
    bool is_reverse = false;
    size_t agglomeration_start = 0, agglomeration_length = 0;
    uint32_t hit_off = 0, hit_cnt = 0;
    int32_t length = 0, candidates_per_window = 0;
    double score = 0;
    size_t hits() const { return hit_cnt; }
    size_t forward_offset() const { return is_reverse ? offset - (length - 1) : offset; }
    bool operator<(const Minimizer& o) const { return score > o.score || (score == o.score && key < o.key); }
};

struct Seed { uint32_t node; uint32_t offset; size_t source; gb_dist_payload payload; };   // pos_t + source + zipcode
struct Cluster { std::vector<size_t> seeds; size_t fragment = 0; double score = 0, coverage = 0; };

// Minimum distance from the END of node a to the START of node b inside one site (gb_dist_payload); -1: not reachable or
// no table (hand-made payloads: parallel single-node alleles).
inline int64_t site_distance(const gb_flat_index* ix, const gb_dist_payload& pa, const gb_dist_payload& pb) {
    if (pa.slot != pb.slot || pa.slot >= ix->n_slots) return -1;
    const gb_slot_rec& sr = ix->slots[pa.slot];
    if (sr.table_off == 0xFFFFFFFFu || pa.allele >= sr.n || pb.allele >= sr.n) return -1;
    const uint16_t t = ix->site_dist[sr.table_off + (size_t)pa.allele * sr.n + pb.allele];
    return t == 0xFFFF ? -1 : (int64_t)t;
}

// Stage trace for the stage-level parity tests (oracle_seed_stage): when the thread-local pointer is set, map_from_extensions
// / map_paired record what they computed up to the extension calls, per read of the unit.
struct StageTrace {
    struct Item { size_t cluster, fragment; std::vector<std::pair<uint32_t, int64_t>> seeds; };
    struct Read { std::vector<Minimizer> minimizers; std::vector<Seed> seeds; std::vector<Cluster> clusters; std::vector<Item> items; };
    Read reads[2];
};
extern thread_local StageTrace* g_stage_trace;

} // namespace oracle
