/* ORACLE — TEST INFRASTRUCTURE ONLY.
 * C entry points of liboracle.so: the CPU restatement of the reference algorithms
 * (vg @ fd49b9a9) that the CUDA path is checked against.  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may load it.
 * The product (vg_b200/, libgiraffe_b200.so) never includes or links this.
 */
#ifndef GB_ORACLE_H
#define GB_ORACLE_H
#include "../include/giraffe_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* GaplessExtender::extend (gbwt_extender.cpp:533-737).  Returns the number of extensions,
 * or -1 when an output capacity is too small.  path_off / mism_off are relative to the
 * pools passed in. */
int oracle_extend(const gb_flat_index* ix, const gb_scores* scores,
                  const uint8_t* read, uint32_t read_len,
                  const gb_seed* seeds, uint32_t n_seeds,
                  uint32_t max_mismatches, double overlap_threshold, int trim,
                  gb_extension* ext_out, uint32_t max_ext,
                  uint32_t* path_pool, uint32_t path_cap,
                  uint32_t* mism_pool, uint32_t mism_cap);

/* The GB_ITEM_* status gb_extend_batch gives the same call when its warp has a q_cap-entry frontier and an
 * a_cap-node path arena (extend.cuh: EXTEND_Q_CAP, EXTEND_A_CAP) and the item has max_ext / path_cap / mism_cap output
 * strides.  Each capacity is checked where the kernel checks it (frontier and arena before every push of the search,
 * records and path nodes when a seed's best match is added, the mismatch pool after the full-length or duplicate
 * filter, before trimming); the first one exceeded decides.  needs_out[5] (may be NULL): raw records, raw path nodes,
 * pre-trim mismatches, peak frontier entries, peak arena nodes of one seed.  seed_skip[n_seeds] (may be NULL):
 * 0 extended, 1 skipped because an exact full-length extension contains it, 2 skipped as invalid (see
 * gb_extend_batch). */
int oracle_extend_limits(const gb_flat_index* ix, const gb_scores* scores,
                         const uint8_t* read, uint32_t read_len,
                         const gb_seed* seeds, uint32_t n_seeds,
                         uint32_t max_mismatches, double overlap_threshold, int trim,
                         uint32_t q_cap, uint32_t a_cap, uint32_t max_ext, uint32_t path_cap, uint32_t mism_cap,
                         uint64_t* needs_out, uint8_t* seed_skip);

/* Haplotype-consistency primitives, exposed so tests can cross-check the flat GBWT
 * against brute-force path scanning.  state = {fwd_node,fwd_lo,fwd_hi,bwd_node,bwd_lo,bwd_hi}
 * (closed ranges as int64).  Returns number of successor states written (each 6 int64). */
int oracle_bd_state(const gb_flat_index* ix, uint32_t node, int64_t* state6);
int oracle_follow_paths(const gb_flat_index* ix, const int64_t* state6, int backward,
                        int64_t* out_states, int max_out);


/* MinimizerMapper::map (single-end), minimizer_mapper.cpp:608-1284.  Output layout as
 * gb_map_batch.  counters_out (13 x uint64, may be NULL): reads, minimizers, seeds, clusters,
 * extend calls, direct (full-length) alignments, tail DPs, tail DP cells, tail tree nodes,
 * tail tree bases, path nodes, edits, rescues.  n_threads = OpenMP threads over reads
 * (the reference's own parallelisation, giraffe_main.cpp:2471). */
void oracle_map_params_default(gb_map_params* p);
int oracle_map_batch(const gb_flat_index* ix, const gb_scores* scores, const gb_map_params* p,
                     uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                     gb_alignment* aln, gb_mapping* mappings, uint32_t* edits, uint8_t* status,
                     int n_threads, uint64_t* counters_out);

/* Pinned X-drop alignment of a query against one haplotype tree (Aligner::align_pinned with
 * xdrop=true, aligner.cpp:628-686).  Mappings are in TREE space: node = tree index + 1. */
int oracle_xdrop_pinned(const gb_flat_index* ix, const gb_scores* scores,
                        const int32_t* tree_parent, const uint32_t* tree_node, uint32_t n_tree, uint32_t root_trim,
                        const uint8_t* query, uint32_t qlen, uint32_t max_gap,
                        int32_t* score_out, gb_mapping* mappings, uint32_t mapping_cap, uint32_t* n_mappings,
                        uint32_t* edits, uint32_t edit_cap, uint32_t* n_edits);

/* MinimizerMapper::map_paired with a forced fragment distribution and max_rescue_attempts = 0
 * (minimizer_mapper.cpp:1462-2942 without the rescue branch).  Reads are interleaved
 * (2i = mate 1, 2i+1 = mate 2, both in input orientation).  Returns -2 if p->max_rescue_attempts != 0. */
int oracle_map_paired_batch(const gb_flat_index* ix, const gb_scores* scores, const gb_map_params* p,
                            uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                            gb_alignment* aln, gb_mapping* mappings, uint32_t* edits, uint8_t* status,
                            int n_threads, uint64_t* counters_out);

/* algorithms::find_best_chains for one problem (chain_items.cpp:733-800) with the candidate list standing in for the
 * zip-code-tree iterator; outputs as gb_chain_batch (chain_begin relative to chain_items).  -1: a candidate names an
 * anchor that does not exist. */
int oracle_chain(const gb_chain_params* P, uint32_t n_anchors, const gb_chain_anchor* anchors,
                 uint64_t n_candidates, const gb_chain_candidate* candidates,
                 int32_t* dp_score, uint32_t* dp_source, uint64_t* dp_paths, uint32_t* dp_rec,
                 uint32_t* n_chains, int32_t* chain_score, uint32_t* chain_begin, uint32_t* chain_count,
                 uint32_t* chain_items, uint32_t* candidate_indel /* may be NULL */);
void oracle_to_anchor(const gb_scores* scores, uint32_t node_len, uint32_t seed_offset, uint32_t min_offset, int min_is_reverse,
                      uint32_t min_length, uint64_t paths, gb_chain_anchor* out);

#ifdef __cplusplus
}
#endif
#endif
