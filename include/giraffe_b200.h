/*
 * giraffe_b200.h — C ABI of libgiraffe_b200.so, the H100-native (sm_90a) replacement for the
 * short-read `vg giraffe` hot path (minimizer lookup -> seed clustering -> gapless
 * extension -> X-drop tail alignment -> MAPQ).
 *
 * Plain C: pointers and sizes only.  No torch / C++ types cross this boundary.
 * Every entry point cites the reference seam it replaces (paths relative to the vg tree,
 * commit fd49b9a9).  Errors are integer status codes (no exceptions cross the ABI) plus a
 * per-item status byte where a batch can partially fail.
 *
 * Ownership: the caller owns every input/output buffer; the library owns device state
 * behind the opaque handles.  Threading: one gb_device handle per GPU; calls on a handle
 * are serialised on that handle's CUDA stream.
 */
#ifndef GIRAFFE_B200_H
#define GIRAFFE_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------
 * Status codes
 * ---------------------------------------------------------------------------------- */
#define GB_OK                 0
#define GB_ERR_ARG           -1   /* bad argument (null pointer, inconsistent sizes)        */
#define GB_ERR_CUDA          -2   /* CUDA runtime error; see gb_last_error()                */
#define GB_ERR_NO_DEVICE     -3   /* no CUDA device: the product path has NO CPU fallback   */
#define GB_ERR_CAPACITY      -4   /* an output capacity given by the caller was too small   */
#define GB_ERR_FORMAT        -5   /* flat index failed validation                           */

/* No C++ exception leaves an entry point that returns a status: one that escapes its body becomes a status code, and
 * gb_last_error() says why.
 *   out of host memory (std::bad_alloc)  GB_ERR_CAPACITY, "<entry point>: out of host memory"
 *   any other exception                  GB_ERR_ARG, or GB_ERR_FORMAT from the readers of GBZ, .min and flat index files
 *                                        (gb_index_from_gbz, gb_index_from_gbz_min, gb_index_load), with the
 *                                        exception's message; the readers also set *out to NULL
 * Entry points that return void or a pointer (gb_fragment_create, gb_fragment_register) have no status to report one
 * with and are not covered. */

/* per-item status byte */
#define GB_ITEM_OK            0
#define GB_ITEM_QUEUE_FULL    1   /* best-first frontier exceeded the per-warp workspace    */
#define GB_ITEM_OUT_FULL      2   /* more extensions / path nodes / mismatches than capacity*/
#define GB_ITEM_DP_REFUSED    3   /* tail DP refused (cells > max_dozeu_cells), softclipped */
#define GB_ITEM_NO_BAND       4   /* banded global DP: no global alignment fits inside the band */

/* ------------------------------------------------------------------------------------
 * Flat ("GBZ-flat") index: what GBZ + .min + distance payload become in HBM.
 *
 * Oriented node handle = GBWT node number  v = 2*id + is_reverse   (gbwt::Node::encode;
 * used by vg at gbwt_extender.hpp:159-162).  ids are 1..max_id, so v in [2, n_nodes).
 * Both orientations of every node sequence are stored explicitly, 1 byte per base
 * (ASCII upper-case ACGTN), so a strand walk never complements on the fly.
 * ---------------------------------------------------------------------------------- */

/* 16-byte node record, one per oriented node (vg: GBWTGraph::get_sequence_view /
 * get_length / CachedGBWTGraph record lookup, gbwt_extender.cpp:582,616,654). */
typedef struct gb_node_rec {
    uint32_t seq_off;   /* byte offset of this orientation's sequence in gb_flat_index.seq */
    uint32_t rec_off;   /* word offset of the GBWT record in gb_flat_index.gbwt            */
    uint32_t len;       /* node length in bp (<= 1024)                                     */
    uint32_t size;      /* number of haplotype visits (GBWT record size); 0 = no record    */
} gb_node_rec;

/* GBWT record blob at gbwt[rec_off]:
 *   word 0: n_edges      word 1: n_runs
 *   n_edges x { to (oriented node, 0 = endmarker), offset (start of our visits in to's record) }
 *   n_runs  x { (run_len << 10) | outrank }          outrank < 1024, run_len < 2^22
 * Edges are sorted by `to`.  LF(i, r) = edge[r].offset + |{ j < i : body[j] == r }|.
 * (restates jltsiren/gbwt @ c2e0199 CompressedRecord; absent from /root/reference) */

/* Distance payload (16 B) — what the clusterer needs of the snarl-tree distance index, flattened
 * (vg: ZipCode::payload_type, zip_code.hpp:74-75, consumed by snarl_seed_clusterer.cpp; minimum_distance
 * minimizer_mapper.cpp:3879-3903).  Every connected component of the graph is a chain of SLOTS: a slot is a cut node
 * (every source-to-sink walk of the component passes through it: the backbone) or a SITE, the subgraph between two
 * consecutive cut nodes — any DAG: nested bubbles, alleles of several nodes, adjacent or overlapping variants.
 *   x_in  = minimum distance from the chain start to the first base of the node
 *   x_out = x_in of the cut node behind the node's slot - minimum distance from the node's end to that cut node
 *           (a cut node: x_in + its length).  SIGNED, two's complement in the 32-bit field: a route that bypasses the
 *           site (a deletion spanning it) makes the cut node's coordinate smaller than the way out of the site
 *   slot  = index of the slot along the chain;  allele = index of the node inside its site in topological order
 *           (0xFFFF: cut node);  component = the chain
 * For u before v in different slots:  d(end of u -> start of v) = x_in[v] - x_out[u]  (every walk crosses the cut nodes
 * between them).  Inside one site the minimum distance from the end of u to the start of v is the site's table entry
 * site_dist[slots[slot].table_off + allele_u * slots[slot].n + allele_v] (0xFFFF: not reachable).
 * Hand-made payloads (gb_index_build with dist != NULL, the synthetic benchmark graphs) may leave a multi-node slot
 * without a table (table_off 0xFFFFFFFF): its nodes are then parallel single-node alleles, reachable only from
 * themselves, and consecutive slots count as fully connected. */
typedef struct gb_dist_payload {
    uint32_t x_in;
    uint32_t x_out;
    uint32_t slot;
    uint16_t allele;
    uint16_t component;
} gb_dist_payload;

/* Minimizer hash-table cell (16 B): open addressing, linear probing, capacity power of 2.
 * key = 2-bit packed k-mer (A0 C1 G2 T3, first base most significant); GB_NO_KEY = empty.
 * (restates gbwtgraph @ e27bc43 MinimizerIndex; call sites minimizer_mapper.cpp:3930-3933) */
#define GB_NO_KEY 0xFFFFFFFFFFFFFFFFull
typedef struct gb_min_cell {
    uint64_t key;
    uint32_t hit_off;   /* first hit in gb_flat_index.hits */
    uint32_t hit_cnt;
} gb_min_cell;

/* One located minimizer occurrence (24 B): packed position + payload
 * (vg: MinimizerIndex::get_value, minimizer_mapper.cpp:4458-4473).
 * pos = (v << 10) | offset, v = oriented node of the k-mer's first base in the k-mer's
 * own orientation (gbwtgraph Position::encode).  payload = dist[v >> 1], the payload of the hit's node (the builders
 * write it so; gb_index_load refuses a file where it differs). */
typedef struct gb_hit {
    uint64_t pos;
    gb_dist_payload payload;
} gb_hit;

typedef struct gb_slot_rec {         /* one slot of a chain (see gb_dist_payload)           */
    uint32_t table_off;              /* first entry of the site's n x n table in site_dist; 0xFFFFFFFF: no table */
    uint32_t n;                      /* nodes in the slot (1 for a cut node)                */
} gb_slot_rec;

typedef struct gb_flat_index {
    uint32_t n_nodes;                /* number of oriented-node slots = 2*(max_id+1)        */
    uint32_t k, w;                   /* minimizer parameters (vg default 29 / 11)           */
    uint32_t n_paths;                /* haplotype paths (each inserted in both orientations)*/
    const gb_node_rec* nodes;        /* [n_nodes]                                           */
    const uint8_t* seq;  uint64_t seq_bytes;     /* padded with >= 16 zero bytes           */
    const uint32_t* gbwt; uint64_t gbwt_words;
    const gb_dist_payload* dist;     /* [n_nodes/2], indexed by node id                     */
    const gb_min_cell* table; uint64_t table_cells;  /* power of two                       */
    const gb_hit* hits;   uint64_t n_hits;
    const gb_slot_rec* slots; uint64_t n_slots;      /* slots of all chains, indexed by gb_dist_payload.slot (may be empty: no tables) */
    const uint16_t* site_dist; uint64_t site_dist_len;   /* site tables, see gb_dist_payload */
} gb_flat_index;

/* ------------------------------------------------------------------------------------
 * Host-side index construction (replaces, for synthetic inputs, what `vg autoindex`
 * produces: index_registry.cpp:100-119, gbwtgraph_helper.cpp:511-630, and
 * get_gbwt() gbwt_helper.cpp:702-719 for the unit-test graphs).
 * ---------------------------------------------------------------------------------- */
typedef struct gb_host_index gb_host_index;

/* node i (1-based id) has forward sequence node_seq[node_off[i-1] .. node_off[i]); an EMPTY sequence marks an id the graph
 * does not use (ids need not start at 1: outputs always carry the caller's ids) — no path or record may name it.
 * path p is path_nodes[path_off[p] .. path_off[p+1]) in GBWT node encoding.
 * dist == NULL: the builder derives the distance payload and the site tables itself from the graph the paths span
 * (chains of cut nodes and sites, see gb_dist_payload) — any graph whose haplotypes walk forward through a DAG;
 * a cycle, a reversing step or a site of more than 4096 nodes leaves the index WITHOUT a distance model
 * (gb_index_has_distance_model() == 0: extension / DP / WFA seams work on it, mapping needs the model).
 * dist != NULL: a hand-made payload indexed by node id (slots without tables).
 * The minimizer table is found either by scanning every haplotype end to end or — with more than 32 haplotypes, or
 * GIRAFFE_B200_WINDOW_BUILDER=1 — by visiting every haplotype-consistent window of k + w - 1 bases once through GBWT
 * search states (gbwtgraph's index_haplotypes); both give the same table. */
int gb_index_build(uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off,
                   uint32_t n_paths, const uint32_t* path_nodes, const uint64_t* path_off,
                   const gb_dist_payload* dist, uint32_t k, uint32_t w,
                   gb_host_index** out);
void gb_index_free(gb_host_index* ix);
int gb_index_has_distance_model(const gb_host_index* ix);
/* Borrowed view; valid until gb_index_free. */
int gb_index_view(const gb_host_index* ix, gb_flat_index* out);
/* The flat index as one file (what giraffe_main.cpp:1825-1881 does for GBZ / .min / .dist): a 64-byte header
 * ("GBFLAT2", n_nodes, k, w, n_paths, seq_bytes, gbwt_words, table_cells, n_hits, then n_slots, site_dist_len in a second 16-byte line) and the eight arrays of gb_flat_index
 * back to back, each padded to 16 bytes, little endian.  gb_index_load checks sizes and offsets and returns
 * GB_ERR_FORMAT for anything that is not such a file; the result is freed with gb_index_free. */
/* Build the flat index from a GBZ file (gbwtgraph::GBZ, what `vg giraffe -Z` loads, giraffe_main.cpp:1825-1881): node
 * sequences from the GBWTGraph, the GBWT records re-laid as they are (no haplotype is walked: gb_index_build_from_gbwt), the
 * distance payload from the chain decomposition of the graph the forward records span, minimizers (k, w) by window
 * enumeration over GBWT search states.  GBZ version 1 /
 * GBWT version 5 / GBWTGraph version 3 in simple-sds serialization.  GB_ERR_FORMAT for anything else, and for graphs
 * outside the index model (haplotypes that step onto a reverse strand, cycles, a site of more than 4096 nodes). */
int gb_index_from_gbz(const char* path, uint32_t k, uint32_t w, gb_host_index** out);
/* The same with the minimizer table READ from the gbwtgraph .min file giraffe loads beside the GBZ (`-m`,
 * giraffe_main.cpp:1825-1881) instead of re-derived by scanning every haplotype: k, w, keys and positions come from the
 * file (minimizer index version 10, 16-byte payloads), every position is checked against the graph (node, offset, the
 * bases of the k-mer on that node), and zipcodes_path (may be NULL; `-z`, zip_code.cpp:2111-2170) must hold every
 * oversized zipcode the table points at.  The distance payload is still the library's own chain model derived from the
 * graph (vg's zipcodes are a different encoding of the same coordinates: tests/test_gbz.py pins the prefix sums); `.dist`
 * is not needed.  Limit, stated rather than guessed: a .min whose keys have several occurrences stores them after the table
 * in a layout the reference's only .min fixture (test/primers/y.min) does not show — from such a file only k and w are
 * taken, and the minimizers are found on the graph by window enumeration (the same set: that is what a .min holds). */
int gb_index_from_gbz_min(const char* gbz_path, const char* min_path, const char* zipcodes_path, gb_host_index** out);
/* gb_index_build with the minimizer hits given by the caller: hit i = (keys[i], positions[i]), position =
 * id << 11 | is_reverse << 10 | offset of the first base of the canonical k-mer on that oriented node (gbwtgraph's
 * Position encoding).  Hits that do not lie on the graph or do not spell their key are GB_ERR_FORMAT. */
/* The same from a GBWT instead of haplotype paths: gbwt_words / rec_off in the blob layout of gb_flat_index (record of oriented
 * node v at gbwt_words[rec_off[v]], rec_off[v] == 0: no record; rec_off has 2 * (n_node_ids + 1) entries).  This is what a
 * caller holding vg's gbwt::GBWT hands over after flattening its records, and what gb_index_from_gbz does with the GBZ's own
 * records: no haplotype is walked, the distance model comes from the edges of the forward records, the minimizers from the
 * window enumeration (or from keys / positions when given, as gb_index_build_with_hits).  Records are validated (edges
 * ascending, ranks inside the edge list, offsets inside the successor's record): GB_ERR_FORMAT otherwise. */
int gb_index_build_from_gbwt(uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off, uint32_t n_paths,
                             const uint32_t* gbwt_words, uint64_t n_words, const uint32_t* rec_off,
                             const gb_dist_payload* dist, uint32_t k, uint32_t w,
                             uint64_t n_hits, const uint64_t* keys, const uint64_t* positions, gb_host_index** out);
int gb_index_build_with_hits(uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off,
                             uint32_t n_paths, const uint32_t* path_nodes, const uint64_t* path_off,
                             const gb_dist_payload* dist, uint32_t k, uint32_t w,
                             uint64_t n_hits, const uint64_t* keys, const uint64_t* positions,
                             gb_host_index** out);
/* gb_index_from_gbz and gb_index_build_from_gbwt with the minimizer step on CUDA device `device_ordinal`: the same GBZ reader,
 * record validation, sequences, distance payload, GBWT blob and table placement on the host; on the GPU one warp per start node
 * follows the GBWT search states to every haplotype-consistent continuation of k + w - 2 bases, computes the minimizers of each
 * start node + continuation string, and radix-sorts and de-duplicates the (key, position) pairs.  The result is byte-identical to
 * the host entry point's: every gb_index_view array, k, w, n_paths, gb_index_save's file, gb_index_has_distance_model.
 * Synchronous; every device allocation is freed before the call returns.  Argument checks come first and return the host entry
 * point's codes (GB_ERR_ARG for NULL path / out / node arrays, k == 0, k > 31, w == 0, and for device_ordinal < 0 or out of
 * range); then GB_ERR_NO_DEVICE without a GPU (there is no host fallback: the host entry points are the CPU route); then the
 * host entry point's GB_ERR_FORMAT for a damaged file or record.  With keys / positions given, gb_index_build_from_gbwt_device
 * takes the table from them as the host call does and enumerates nothing.  GB_ERR_CAPACITY, beyond the host's cases, when a
 * GBWT record has more than 2^31 - 1 visits, when the longest node + k + w - 2 bases (16 B each) do not fit one warp's shared
 * memory, or when one start node has more minimizers than the pair pool holds.
 * HBM: the node records (32 B per node id), both sequence orientations (2 B per base), the GBWT blob, 20 B per start node,
 * the warps' search-state stacks (16 B per warp x the largest GBWT record, about the haplotype count; at most 256 MiB) and the
 * pair pool with its sort buffers (56 B per pair, at most 2 GiB: min(2 GiB, 56 B x the pairs before de-duplication)).
 * Start nodes are processed in batches whose pairs fit the pool; GIRAFFE_B200_INDEX_POOL_PAIRS (a pair count; for tests
 * only) shrinks the pool so that a small graph needs several batches. */
int gb_index_from_gbz_device(const char* path, uint32_t k, uint32_t w, int device_ordinal, gb_host_index** out);
int gb_index_build_from_gbwt_device(uint32_t n_node_ids, const uint8_t* node_seq, const uint64_t* node_off, uint32_t n_paths,
                                    const uint32_t* gbwt_words, uint64_t n_words, const uint32_t* rec_off,
                                    const gb_dist_payload* dist, uint32_t k, uint32_t w,
                                    uint64_t n_hits, const uint64_t* keys, const uint64_t* positions,
                                    int device_ordinal, gb_host_index** out);
/* How a build spent its time, host-clocked (seconds), and what its minimizer step visited: start nodes and continuations of the
 * window enumeration (0 for the haplotype scan and for a table given by the caller), (key, position) pairs before and after
 * de-duplication.  All zero for an index read by gb_index_load. */
typedef struct gb_index_timing {
    double sequences_s, distance_s, gbwt_s, minimizers_s, table_s;
    uint64_t start_nodes, continuations, raw_pairs, unique_pairs;
} gb_index_timing;
int gb_index_build_timing(const gb_host_index* ix, gb_index_timing* out);
int gb_index_save(const gb_flat_index* ix, const char* path);
int gb_index_load(const char* path, gb_host_index** out);

/* ------------------------------------------------------------------------------------
 * Device handle
 * ---------------------------------------------------------------------------------- */
typedef struct gb_device gb_device;

/* Copies the flat index into HBM of CUDA device `device_ordinal`.
 * Fails with GB_ERR_NO_DEVICE when there is no GPU (no CPU fallback exists). */
int gb_device_create(const gb_flat_index* ix, int device_ordinal, gb_device** out);
void gb_device_destroy(gb_device* dev);
const char* gb_last_error(void);

/* Scoring (vg: MinimizerMapper::set_alignment_scores minimizer_mapper.cpp:77 ->
 * Aligner ctor aligner.cpp:1417; defaults alignment_scorer.hpp:18-28: 1/4/6/1/5). */
typedef struct gb_scores {
    int8_t match, mismatch, gap_open, gap_extend, full_length_bonus;
} gb_scores;
int gb_set_scores(gb_device* dev, const gb_scores* s);

/* ------------------------------------------------------------------------------------
 * B2: GaplessExtender::extend, batched
 *   vector<GaplessExtension> GaplessExtender::extend(cluster_type&, std::string sequence,
 *       const CachedGBWTGraph*, size_t max_mismatches = 4, double overlap_threshold = 0.8,
 *       bool trim = true) const                     gbwt_extender.hpp:205, .cpp:533-737
 * One work item = one (read, cluster) call of the reference.
 * ---------------------------------------------------------------------------------- */
typedef struct gb_seed {          /* GaplessExtension::seed_type, gbwt_extender.hpp:32    */
    uint32_t node;                /* oriented node v                                        */
    int32_t  diag;                /* read_offset - node_offset                              */
} gb_seed;

#define GB_EXT_LEFT_FULL   1u
#define GB_EXT_RIGHT_FULL  2u

typedef struct gb_extension {     /* GaplessExtension, gbwt_extender.hpp:30-109             */
    uint32_t path_off, path_len;  /* into the path pool (oriented nodes)                    */
    uint32_t mism_off, mism_len;  /* into the mismatch pool (read offsets, ascending)       */
    uint32_t offset;              /* offset in path[0]                                      */
    uint32_t read_lo, read_hi;    /* read_interval                                          */
    int32_t  score;
    uint32_t flags;               /* GB_EXT_LEFT_FULL | GB_EXT_RIGHT_FULL                   */
    uint32_t fwd_node, fwd_lo, fwd_hi;   /* gbwt::BidirectionalState forward  (closed range)*/
    uint32_t bwd_node, bwd_lo, bwd_hi;   /*                           backward              */
    uint32_t mismatches;          /* internal_score                                         */
} gb_extension;                   /* 64 bytes                                               */

typedef struct gb_extend_params {
    uint32_t max_mismatches;      /* reference default 4  (GaplessExtender::MAX_MISMATCHES) */
    double   overlap_threshold;   /* reference default 0.8                                  */
    uint32_t trim;                /* reference default 1                                    */
    uint32_t max_ext_per_item;    /* output capacity per work item                          */
    uint32_t path_cap_per_item;   /* path-pool capacity per work item (nodes)               */
    uint32_t mism_cap_per_item;   /* mismatch-pool capacity per work item                   */
} gb_extend_params;

/* reads: concatenated read bytes (ASCII); read_off[n_reads+1].
 * item_read[n_items]: which read each work item extends.
 * seeds / seed_off[n_items+1]: the cluster of each item (duplicates allowed; they collapse,
 * as in the reference's hash set).
 * Outputs (host): ext_count[n_items], status[n_items],
 *   ext[n_items * max_ext_per_item], path_pool[n_items * path_cap_per_item],
 *   mism_pool[n_items * mism_cap_per_item]; gb_extension.path_off / mism_off are absolute
 *   indices into those pools.
 * Canonical order (the reference iterates an unordered set, gbwt_extender.cpp:550): seeds
 * are processed in ascending (node, diag) order and ties in the full-length sort
 * (gbwt_extender.cpp:302) keep that order (stable).
 * Seeds the reference would read out of bounds with are skipped: a node v outside [2, n_nodes) or of length 0, a
 * read offset max(diag, 0) past the end of the read, or a node offset max(-diag, 0) past the end of the node.  Offsets
 * equal to the read or node length are valid (an empty initial match).
 * Limits: reads of up to 25600 bases (8 warps x read length of shared memory, at most 200 KiB; a longer read returns
 * GB_ERR_ARG before anything is launched); per warp, a best-first frontier of 511 entries and 4096 path-arena nodes
 * per seed (GB_ITEM_QUEUE_FULL past either); per item, max_ext_per_item raw records (one per extended seed, before
 * duplicates are removed), path_cap_per_item nodes over those records and mism_cap_per_item mismatches over the
 * records left after the full-length or duplicate filter, before trimming (GB_ITEM_OUT_FULL past any).  An item
 * refused this way has ext_count 0. */
int gb_extend_batch(gb_device* dev, const gb_extend_params* p,
                    uint32_t n_reads, const uint8_t* reads, const uint64_t* read_off,
                    uint32_t n_items, const uint32_t* item_read,
                    const gb_seed* seeds, const uint64_t* seed_off,
                    uint32_t* ext_count, uint8_t* status,
                    gb_extension* ext, uint32_t* path_pool, uint32_t* mism_pool);

/* ------------------------------------------------------------------------------------
 * B1: MinimizerMapper::map / map_paired, batched
 *   vector<Alignment> MinimizerMapper::map(Alignment&)           minimizer_mapper.hpp:44-100,
 *   map_from_extensions                                          minimizer_mapper.cpp:608-1284
 * Output is the GAM-equivalent record: the fields of vg.proto Alignment / Path / Mapping /
 * Edit that the reference fills on this path (gbwt_extender.cpp:119-156,
 * dozeu_interface.cpp:310-336, minimizer_mapper.cpp:1146-1216).
 * ---------------------------------------------------------------------------------- */
typedef struct gb_mapping {       /* one Mapping: position + run of edits (8 B)              */
    uint32_t node;                /* oriented node v = 2*id + is_reverse                     */
    uint16_t offset;              /* Position.offset                                         */
    uint16_t n_edits;             /* edits follow each other in the edit pool                */
} gb_mapping;

/* One Edit (4 B): (length << 4) | (base << 2) | op.
 * MATCH: from=to=length.  SUB: from=to=1, sequence = base (A0 C1 G2 T3; N is reported as the
 * read base itself, look it up by query offset).  INS: from=0,to=length (sequence = the read
 * bases at the current query offset; softclips are insertions at the ends).  DEL: from=length,to=0. */
#define GB_EDIT_MATCH 0u
#define GB_EDIT_SUB   1u
#define GB_EDIT_INS   2u
#define GB_EDIT_DEL   3u

#define GB_ALN_MAPPED     1u      /* path is non-empty                                       */
#define GB_ALN_SECONDARY  2u
#define GB_ALN_PAIRED     4u      /* produced by map_paired                                  */
#define GB_ALN_RESCUED    8u
#define GB_ALN_ABSENT     16u     /* max_multimaps > 1: this rank of this read has no mapping (skip the record)   */
#define GB_MAX_MULTIMAPS  8u

typedef struct gb_alignment {     /* 32 B header per output alignment                        */
    uint32_t read_id;             /* index of the read in the batch                          */
    int32_t  score;               /* Alignment.score                                         */
    uint8_t  mapq;                /* Alignment.mapping_quality                               */
    uint8_t  flags;
    uint16_t n_mappings;
    uint32_t mapping_off;         /* into the mapping pool                                   */
    uint32_t edit_off;            /* into the edit pool                                      */
    uint32_t n_edits;
    float    mapq_uncapped;       /* annotation mapq_uncapped (minimizer_mapper.cpp:1173)    */
    float    mapq_explored_cap;   /* annotation mapq_explored_cap (:1174)                    */
} gb_alignment;

/* MinimizerMapper settings on this path; defaults = minimizer_mapper.hpp:108-521. */
typedef struct gb_map_params {
    uint32_t hit_cap;                    /* 10   */
    uint32_t hard_hit_cap;               /* 500  */
    double   minimizer_score_fraction;   /* 0.9  */
    uint32_t minimizer_coverage_flank;   /* 250  */
    uint32_t max_unique_min;             /* 500  */
    uint32_t num_bp_per_min;             /* 1000 */
    uint32_t distance_limit;             /* 200  */
    uint32_t min_extensions;             /* 2    */
    uint32_t max_extensions;             /* 800  */
    double   cluster_score_threshold;    /* 50   */
    double   pad_cluster_score_threshold;/* 20   */
    double   cluster_coverage_threshold; /* 0.3  */
    double   extension_set_score_threshold; /* 20 */
    int32_t  extension_score_threshold;  /* 1    */
    int32_t  min_extension_sets;         /* 2    */
    int32_t  extension_set_min_score;    /* 20   */
    uint32_t max_alignments;             /* 8    */
    uint32_t max_extension_mismatches;   /* 4    */
    uint32_t max_multimaps;              /* 1 .. GB_MAX_MULTIMAPS: mappings reported per read (or pairs per pair)   */
    uint32_t max_dozeu_cells;            /* 1.5 * 1024 * 1024                                */
    uint32_t do_dp;                      /* 1    */
    /* paired-end (map_paired, minimizer_mapper.cpp:1462) */
    double   fragment_mean, fragment_stdev;      /* forced distribution (--fragment-mean/-stdev) */
    double   paired_distance_stdevs;     /* 2.0  */
    double   paired_rescue_score_limit;  /* 0.9  */
    double   rescue_subgraph_stdevs;     /* 4.0  */
    uint32_t max_rescue_attempts;        /* 15   */
    uint32_t max_fragment_length;        /* 2000 */
    uint32_t rescue_seed_limit;          /* 100  (minimizer_mapper.hpp:459)                  */
    uint32_t reserved0;
    double   rescue_likelihood_limit;    /* 0.05 (minimizer_mapper.hpp:475)                  */
    /* output capacities per read */
    uint32_t mapping_cap_per_read;
    uint32_t edit_cap_per_read;
} gb_map_params;

void gb_map_params_default(gb_map_params* p);

/* Single-end batch.  reads/quals are concatenated bytes addressed by read_off[n_reads+1]
 * (quals = raw Phred bytes, may be NULL: then the explored-minimizer cap is +inf as in
 * minimizer_mapper.cpp:2950).  aln[n_reads * max_multimaps] and status[n_reads]: record j * n_reads + r is
 * mapping j of read r in output order (minimizer_mapper.cpp:1087-1206; map_paired: pair j of the pair, :2505-2598) —
 * j = 0 the primary, which alone carries the MAPQ; j >= 1 secondaries (GB_ALN_SECONDARY), or GB_ALN_ABSENT when the
 * read has fewer mappings.  With max_multimaps = 1 (the default) that is one record per read.
 * Limits of the mapping entry points: reads up to 512 bp.  Index limits, the same for every mapping entry point:
 *   node ids below 2^31 - 1 (n_nodes = 2 * (max_id + 1) is a uint32_t; tested past 2^22 with more than 2^22 real nodes
 *   and with ids shifted up to 2^24);
 *   sequence below 2^31 - 32 bp: both orientations are addressed by the 32-bit gb_node_rec.seq_off;
 *   chain coordinates: x_in + length <= 2^31 - 1 and (int32) x_out - length >= -2^31 for every node with a sequence
 *   (a payload the builder derives always fits; GB_ERR_CAPACITY from the mapping entry points for one that does not);
 *   memory: nodes (16 B per oriented node) and dist (16 B per id) are dense over the ids: 48 B of HBM per id, used or not.
 * mappings / edits are DENSE pools of the given capacities
 * (gb_alignment.mapping_off / edit_off index into them); the elements used are returned
 * through n_mappings_used / n_edits_used (may be NULL).  GB_ERR_CAPACITY if a pool is too
 * small.  Internally the batch is processed in chunks of 2^20 reads. */
int gb_map_batch(gb_device* dev, const gb_map_params* p,
                 uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                 gb_alignment* aln, gb_mapping* mappings, uint64_t mapping_pool_cap, uint32_t* edits, uint64_t edit_pool_cap,
                 uint8_t* status, uint64_t* n_mappings_used, uint64_t* n_edits_used);

/* Paired-end batch: MinimizerMapper::map_paired(aln1, aln2) with a finalized (forced)
 * fragment length distribution, minimizer_mapper.hpp:100, minimizer_mapper.cpp:1462-2942
 * (`vg giraffe --fragment-mean M --fragment-stdev S`).  Reads are interleaved: read 2i is
 * mate 1 and read 2i+1 mate 2 of pair i, both in sequencer (inward) orientation; outputs are
 * per read as in gb_map_batch, mate 2 reported in its input orientation, flags |= GB_ALN_PAIRED.
 * p->max_rescue_attempts == 0 takes the reference branch :2238-2287; otherwise unpaired
 * alignments rescue their mates (attempt_rescue :3264-3565 with rescue_algorithm dozeu and the
 * full-DP fallback of fix_dozeu_score; pairing / multiplicities / caps :2288-2777) and rescued
 * records carry GB_ALN_RESCUED.  A rescue subgraph larger than the per-warp workspace (320 nodes,
 * 6144 bases of both orientations, 127 seeds) sets status GB_ITEM_OUT_FULL for both mates of that
 * pair; rescue_seed_limit must be below 128. */
int gb_map_paired_batch(gb_device* dev, const gb_map_params* p,
                        uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                        gb_alignment* aln, gb_mapping* mappings, uint64_t mapping_pool_cap, uint32_t* edits, uint64_t edit_pool_cap,
                        uint8_t* status, uint64_t* n_mappings_used, uint64_t* n_edits_used);

/* ---- fragment length distribution and the whole paired job --------------------------------
 * FragmentLengthDistribution (mapper.hpp:83-139, mapper.cpp:5231-5333): robust running estimate
 * of the fragment length; MinimizerMapper owns one as fragment_length_distr(1000, 1000, 0.95)
 * (minimizer_mapper.cpp:72).  Host-side state, no device work. */
typedef struct gb_fragment_distribution gb_fragment_distribution;
gb_fragment_distribution* gb_fragment_create(uint64_t maximum_sample_size, uint64_t reestimation_frequency,
                                             double robust_estimation_fraction);
void     gb_fragment_destroy(gb_fragment_distribution* f);
void     gb_fragment_force(gb_fragment_distribution* f, double mean, double stdev);   /* force_parameters, mapper.cpp:5250 */
void     gb_fragment_register(gb_fragment_distribution* f, int64_t length);           /* register_fragment_length, :5256  */
void     gb_fragment_finalize(gb_fragment_distribution* f);     /* finalize_fragment_length_distr, minimizer_mapper.hpp:539 */
double   gb_fragment_mean(const gb_fragment_distribution* f);
double   gb_fragment_stdev(const gb_fragment_distribution* f);
int      gb_fragment_is_finalized(const gb_fragment_distribution* f);
uint64_t gb_fragment_sample_size(const gb_fragment_distribution* f);

#define GB_PAIR_PAIRED   0u   /* map_paired with the finalized distribution                              */
#define GB_PAIR_TRAINING 1u   /* both ends mapped single-ended, their distance registered (:1303-1386)   */
#define GB_PAIR_BUFFERED 2u   /* ambiguous while training (ambiguous_pair_buffer), mapped paired at end  */

/* The paired job as `vg giraffe` runs it without --fragment-mean/--fragment-stdev
 * (giraffe_main.cpp:2246-2400): while `f` is not finalized, pairs are taken in input order through
 * MinimizerMapper::map_paired(aln1, aln2, ambiguous_pair_buffer) (minimizer_mapper.cpp:1303-1395) —
 * both ends mapped single-ended on the GPU (windows of training_window pairs, at most half the map chunk,
 * each uploaded and trained by the same step as gb_map_paired_job_device; pairs of a window behind the
 * finalizing pair are not consumed), pairs whose ends are both MAPQ 60 with score >=
 * 0.85 * match * length and whose distance is below max_fragment_length register it and keep their
 * single-ended records, every other pair is buffered; once finalized (or, at the end of the input,
 * finalized by force as giraffe_main.cpp:2283-2296 does) all remaining and all buffered pairs go through
 * gb_map_paired_batch with the estimated mean / stdev (p->fragment_mean / p->fragment_stdev are
 * ignored; `f` carries the distribution across calls).  Outputs as gb_map_paired_batch;
 * pair_route[n_reads / 2] receives GB_PAIR_* (may be NULL).  training_window 0 selects 2048.  Refused with
 * GB_ERR_ARG: a NULL p or f, a NULL required array when n_reads > 0, an odd n_reads, max_multimaps != 1.
 * Workspace on the handle: gb_map_paired_job_device's for one training window, plus its reads and qualities. */
int gb_map_paired_job(gb_device* dev, const gb_map_params* p, gb_fragment_distribution* f, uint32_t training_window,
                      uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                      gb_alignment* aln, gb_mapping* mappings, uint64_t mapping_pool_cap, uint32_t* edits, uint64_t edit_pool_cap,
                      uint8_t* status, uint8_t* pair_route, uint64_t* n_mappings_used, uint64_t* n_edits_used);

/* gb_map_paired_job for reads already in HBM: d_reads, d_quals (may be NULL), d_read_off, d_aln, d_mappings, d_edits,
 * d_status and d_pair_route (may be NULL) are DEVICE addresses; p, f and the two counts are on the host.  For the same reads,
 * parameters and distribution state the outputs are exactly gb_map_paired_job's: every record field, the pools up to the
 * used counts in the same order (training pairs in input order, then the remaining pairs, then the buffered pairs in
 * buffer order), status, routes and the state of f afterwards.  d_read_off may start at any value and may leave gaps
 * between reads; every read is at most max_read_len <= 512 long (a longer one is GB_ERR_ARG).  Refused with GB_ERR_ARG
 * before any work: a NULL p or f, a NULL required array when n_reads > 0, an odd n_reads, max_multimaps != 1,
 * max_read_len > 512.  n_reads == 0 returns GB_OK and leaves f as it is.  GB_ERR_CAPACITY when a pool is too small: every
 * sub-batch is sized before it is copied, so nothing is written past mapping_pool_cap / edit_pool_cap.  One call is one
 * input: when the pairs run out before the sample fills, f is finalized with what it has (the 0 +- 1 it starts with when
 * nothing was registered, whose pairs then take map_paired's single-end fallback), so a streaming caller's later calls map
 * fully paired; the ambiguous buffer does not outlive the call.
 * The call is synchronous (it runs on the handle's stream and returns with the records in place): each training window
 * (training_window pairs, 0 selects 2048, at most half the map chunk) is mapped single-ended, classified on the device and
 * copied back once (the cut and the lengths to register); the remaining and the buffered pairs are gathered into
 * zero-based sub-batches of at most the map chunk (GIRAFFE_B200_MAP_CHUNK, 2^20 reads) and mapped paired.  A sub-batch
 * that overflows the intermediate pools is redone with them doubled, as in gb_map_batch.  Workspace on the handle (kept,
 * grown on demand), per read of the largest sub-batch: 8 * mapping_cap_per_read + 4 * edit_cap_per_read + 57 bytes (1.5 KB
 * with the default caps) plus 2 * max_read_len for the gathered reads and qualities; 4 bytes per pair of the call for the
 * buffer; 28 bytes per pair of a training window. */
int gb_map_paired_job_device(gb_device* dev, const gb_map_params* p, gb_fragment_distribution* f, uint32_t training_window,
                             uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals, const uint64_t* d_read_off,
                             uint32_t max_read_len,
                             gb_alignment* d_aln, gb_mapping* d_mappings, uint64_t mapping_pool_cap,
                             uint32_t* d_edits, uint64_t edit_pool_cap, uint8_t* d_status, uint8_t* d_pair_route,
                             uint64_t* n_mappings_used, uint64_t* n_edits_used);
/* The training windows of the last gb_map_paired_job_device call on this handle and the host-clocked time they took (ms). */
int gb_paired_job_stats(const gb_device* dev, uint32_t* training_windows, double* training_ms);

/* ---- emission (host side, no device work) ---------------------------------------------------
 * giraffe_main.cpp:2209-2226 hands alignments to a vg::io::AlignmentEmitter (libvgio @ d029989,
 * absent from the reference tree).  These two write the same information as text, one line per
 * record, into `out` (GB_ERR_CAPACITY if it does not fit; *out_used = bytes written):
 *   gb_emit_gaf   GAF: name, length, query start / end (the whole read: soft clips are insertions in cs),
 *                 '+', path as >id / <id steps (mappings that only carry an insertion are left out), path
 *                 length, start / end on the path, matches, block length, MAPQ, then AS:i, bq:Z (when quals),
 *                 cs:Z (":n" "*RQ" "+Q" "-R", match runs merged across mappings), dv:f, fn:Z / fp:Z for
 *                 mates; unaligned reads: empty path ('*') and cs "+<read>" — the conventions the reference's
 *                 own tests fix (unittest/alignment.cpp:398-470, :793-820)
 *   gb_emit_json  one protobuf-JSON Alignment per line with vg.proto's field names, as `vg view -aj`
 *                 prints them (64-bit integers as strings, default values omitted, quality base64)
 * names / name_off may be NULL (reads are then called read<i>); records may be any subset / order
 * (read_id selects the read among n_reads).  Records are validated against mapping_pool_len / edit_pool_len / n_reads,
 * the graph and the read length before anything is written: GB_ERR_ARG for a record that points outside them. */
int gb_emit_gaf(const gb_flat_index* ix, uint32_t n, const gb_alignment* aln, const gb_mapping* mappings, uint64_t mapping_pool_len,
                const uint32_t* edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                const uint8_t* names, const uint64_t* name_off, char* out, uint64_t out_cap, uint64_t* out_used);
int gb_emit_json(const gb_flat_index* ix, uint32_t n, const gb_alignment* aln, const gb_mapping* mappings, uint64_t mapping_pool_len,
                 const uint32_t* edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                 const uint8_t* names, const uint64_t* name_off, char* out, uint64_t out_cap, uint64_t* out_used);
/* GAM: the same records as vg.proto Alignment messages in vg::io's type-tagged group framing (uncompressed; vg reads
 * plain, gzip and BGZF streams).  libvgio is absent from the reference tree: field numbers and framing are read off GAM
 * files written by vg itself (reference test data, tests/golden/gam/): sequence 1, path 2 {mapping 2 {position 1
 * {node_id 1, offset 2, is_reverse 4}, edit 2 {from_length 1, to_length 2, sequence 3}, rank 5}}, name 3, quality 4,
 * mapping_quality 5, score 6, fragment_prev 11 / fragment_next 12, identity 16, annotation 100 (Struct). */
int gb_emit_gam(const gb_flat_index* ix, uint32_t n, const gb_alignment* aln, const gb_mapping* mappings, uint64_t mapping_pool_len,
                const uint32_t* edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                const uint8_t* names, const uint64_t* name_off, char* out, uint64_t out_cap, uint64_t* out_used);

/* BGZF, the blocked gzip container vg::io's emitters write GAM in (giraffe_main.cpp:2209-2226; libvgio's
 * BlockedGzipOutputStream over htslib bgzf): `in` is cut into blocks of at most 0xff00 bytes, each a complete gzip
 * member carrying the 'BC' extra subfield (block size - 1), followed by the 28-byte empty EOF block.  level 0-9 (zlib).
 * GB_ERR_CAPACITY when `out` is too small (in_bytes + 128 * (in_bytes / 0xff00 + 2) always suffices). */
int gb_bgzf_compress(const void* in, uint64_t in_bytes, int level, void* out, uint64_t out_cap, uint64_t* out_used);

/* GAF and GAM formatted on the GPU: gb_emit_gaf / gb_emit_gam for records that are already in HBM (gb_map_batch_device's
 * outputs, or any records copied there).  Every array is a DEVICE address; node lengths and reference bases come from the
 * handle's copy of the graph.  For the same records the bytes written to d_out are exactly those the host emitter writes:
 * any subset or order of records (read_id selects the read), GB_ALN_ABSENT ranks skipped, read<i> names when d_names is
 * NULL, bq:Z and the GAM quality field only when d_quals is non-NULL, GAM groups of 1000 present records.
 *   GB_ERR_ARG       a record the host emitter refuses (decided on the device; nothing is written)
 *   GB_ERR_CAPACITY  out_cap is too small: nothing is written and *out_used is the number of bytes needed, so the caller
 *                    can resize and call again.  On success *out_used is the number of bytes written.
 * The call runs on the handle's stream and synchronises once, after sizing every record: the total decides whether the
 * fill runs.  The fill itself is left enqueued on the stream; work ordered after it there (a copy of d_out to the host,
 * gb_device_synchronize) sees the bytes.  The output is uncompressed: gb_bgzf_compress_device compresses it without leaving HBM
 * (or gb_bgzf_compress once it is copied to the host). */
int gb_emit_gaf_device(gb_device* dev, uint32_t n, const gb_alignment* d_aln, const gb_mapping* d_mappings, uint64_t mapping_pool_len,
                       const uint32_t* d_edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals,
                       const uint64_t* d_read_off, const uint8_t* d_names, const uint64_t* d_name_off,
                       char* d_out, uint64_t out_cap, uint64_t* out_used);
int gb_emit_gam_device(gb_device* dev, uint32_t n, const gb_alignment* d_aln, const gb_mapping* d_mappings, uint64_t mapping_pool_len,
                       const uint32_t* d_edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals,
                       const uint64_t* d_read_off, const uint8_t* d_names, const uint64_t* d_name_off,
                       char* d_out, uint64_t out_cap, uint64_t* out_used);

/* BGZF on the GPU: the container gb_bgzf_compress writes, for bytes already in HBM (gb_emit_gam_device / gb_emit_gaf_device
 * output, or any other bytes).  d_in and d_out are DEVICE addresses; d_in may start at any byte.  The input is cut every
 * 0xff00 bytes exactly as gb_bgzf_compress cuts it (so BGZF virtual offsets agree); every block is one gzip member with the
 * host's 16 header bytes, BSIZE - 1, a raw deflate payload, CRC32 and ISIZE, and the stream ends with the same 28-byte EOF
 * block (an empty input gives only that block).  The payload is the device's own: one dynamic-Huffman deflate block per
 * BGZF block, or a stored block when that would not be smaller, so it is not zlib's bytes, but any inflater reads it and
 * the same input gives the same bytes on every call.  There is no level: the device has one compressor.
 *   GB_ERR_ARG       dev or out_used is NULL, d_out is NULL, or d_in is NULL with in_bytes > 0
 *   GB_ERR_CAPACITY  out_cap is too small: nothing is written to d_out and *out_used is the number of bytes needed.
 *                    in_bytes + 128 * (in_bytes / 0xff00 + 2), gb_bgzf_compress's bound, always suffices.
 * The call runs on the handle's stream and synchronises once, for the total size; the gather into d_out is left enqueued
 * there, like the fill of gb_emit_*_device.  Workspace on the handle (kept between calls, grown on demand): 64 KiB per
 * input block (about 1.004 x in_bytes) plus 255 KiB per SM for the parsed tokens (34 MB on a 132-SM H100). */
int gb_bgzf_compress_device(gb_device* dev, const void* d_in, uint64_t in_bytes, void* d_out, uint64_t out_cap, uint64_t* out_used);

/* BGZF inflated on the GPU, the inverse of gb_bgzf_compress_device: the whole BGZF members at the start of d_in (a DEVICE
 * address, any byte alignment) are inflated into d_out (DEVICE), one after the other.  A member is a gzip header whose FLG is
 * FEXTRA alone (FNAME, FCOMMENT and FHCRC are refused) with a 'BC' subfield of SLEN 2 anywhere among its XLEN bytes; BSIZE
 * gives its length; its raw deflate payload (stored, fixed and dynamic blocks) must end with its BFINAL block in the
 * payload's last byte; CRC32 and ISIZE must match the inflated bytes and ISIZE must be at most 65536; back-references may not
 * reach before the member's own output.  A member is accepted exactly when zlib's raw inflate accepts its payload with
 * nothing left over and the trailer matches, and the output is then zlib's bytes.  Empty members (the 28-byte EOF block) are
 * accepted anywhere, so concatenated bgzip files work.
 *   final == 0  a member that runs past in_bytes ends the call without error: *in_used is its first byte, and the caller
 *               passes the bytes from there again, followed by more input, in its next call
 *   final != 0  such a member is GB_ERR_FORMAT
 *   GB_ERR_FORMAT    not BGZF (gb_last_error() names the byte offset), including single-member gzip without the 'BC'
 *                    subfield (plain `gzip` output), which cannot be split into blocks: inflate such a file on the host.
 *                    After it, the contents of d_out are unspecified.
 *   GB_ERR_CAPACITY  out_cap is below the sum of the ISIZEs (read from the trailers before anything is inflated): nothing is
 *                    written and *out_used is the number of bytes needed.
 * On success *out_used is the number of bytes written and *in_used the bytes of d_in consumed.  The call runs on the
 * handle's stream and waits twice: once for the member walk (count, sizes, where it stopped), once for the inflate status.
 * Workspace on the handle (kept, grown on demand): 32 bytes per 26 input bytes in the worst case (the member list). */
int gb_bgzf_decompress_device(gb_device* dev, const void* d_in, uint64_t in_bytes, int final,
                              void* d_out, uint64_t out_cap, uint64_t* out_used, uint64_t* in_used);

/* FASTQ parsed on the GPU into the arrays gb_map_batch_device and gb_emit_{gaf,gam}_device take: bases and qualities
 * concatenated and addressed by d_read_off[n + 1], names concatenated and addressed by d_name_off[n + 1] (all DEVICE).
 * d_text is a HOST array of n_inputs DEVICE pointers, each starting at a record boundary:
 *   n_inputs 1              single-end: record i is read i
 *   n_inputs 1, flags GB_FASTQ_INTERLEAVED   records 2i and 2i + 1 are mates 1 and 2 (vg giraffe -i)
 *   n_inputs 2              record i of input 0 is read 2i, record i of input 1 read 2i + 1 (vg giraffe -f r1 -f r2): the
 *                           mate order gb_map_batch_device(paired = 1) expects
 * Per record, vg's reader (get_next_alignment_from_fastq, src/alignment.cpp:159-250; giraffe_main.cpp:2319, :2433):
 *   name       the bytes after '@' up to the first of " \t\v\f\r" or the line end (the comment is dropped, /1 and /2 are
 *              kept; may be empty)
 *   sequence   the second line (one line); 'a'..'z' uppercased, every other byte unchanged
 *   separator  the third line, which must start with '+' (its rest is not looked at)
 *   quality    the fourth line, each byte - 33 (raw Phred, as vg's Alignment.quality holds it); d_quals may be NULL
 * The call takes whole records (whole pairs when paired) in input order and stops, without error, at the first that is not
 * complete in the text or does not fit max_reads, bases_cap or names_cap.  *n_reads, *max_read_len (the longest read taken)
 * and text_used[n_inputs] (bytes consumed per input) say how far it got; the caller passes the rest again, followed by more
 * text, in its next call.  GB_ERR_CAPACITY when a complete record (pair) is present but none fits.
 * With final != 0 the text is the end of the input: an input whose whole records were all taken must end with the last of
 * them (bytes that do not form a complete record, such as a last line without '\n', are GB_ERR_FORMAT; vg refuses such a
 * file too).  With two inputs the longer one's surplus records, and the odd last record of an interleaved input, are left
 * unconsumed (text_used shows them; vg drops them silently, alignment.cpp:252-258).
 * GB_ERR_FORMAT, with the input, record index and byte offset in gb_last_error(), for a record the call reaches whose
 *   - header does not start with '@' (including FASTA's '>': FASTA input is not supported)
 *   - separator line does not start with '+'
 *   - quality length differs from the sequence length (divergence: vg also accepts an empty quality line)
 *   - sequence or quality line holds a byte outside '!'..'~' (divergence: this refuses CRLF files and NULs, which vg passes
 *     into the read as '\r' and as a negative quality)
 * After GB_ERR_FORMAT the contents of the output arrays are unspecified.
 * Not supported: multi-line FASTQ, FASTA, --comments-as-tags.  The call runs on the handle's stream and waits once, for the
 * counts.  Workspace on the handle (kept, grown on demand): 32 bytes per line the call may look at (4 * max_reads + 8 lines)
 * plus 40 bytes per read of max_reads. */
#define GB_FASTQ_INTERLEAVED 1u
int gb_fastq_parse_device(gb_device* dev, uint32_t n_inputs, const uint8_t* const* d_text, const uint64_t* text_bytes,
                          uint32_t flags, int final, uint32_t max_reads, uint8_t* d_reads, uint8_t* d_quals, uint64_t bases_cap,
                          uint64_t* d_read_off, uint8_t* d_names, uint64_t names_cap, uint64_t* d_name_off,
                          uint32_t* n_reads, uint32_t* max_read_len, uint64_t* text_used);

/* Device-pointer variant of both (paired != 0 selects map_paired): every pointer is a DEVICE
 * address (inputs already resident in HBM, outputs stay in HBM); all reads are at most
 * max_read_len long; d_aln holds n_reads * p->max_multimaps records (rank-major, as gb_map_batch);
 * d_totals[2] (device) receives {mappings used, edits used}.  With paired != 0, d_read_off[0] must be 0 and
 * d_read_off[n_reads] <= n_reads * max_read_len (the paired working copy of the reads is addressed by them).  The call only
 * enqueues work on the handle's stream (gb_device_set_stream) and returns; use
 * gb_device_synchronize or stream ordering before reading the outputs. */
int gb_map_batch_device(gb_device* dev, const gb_map_params* p, int paired, uint32_t n_reads,
                        const uint8_t* d_reads, const uint8_t* d_quals, const uint64_t* d_read_off, uint32_t max_read_len,
                        gb_alignment* d_aln, gb_mapping* d_mappings, uint64_t mapping_pool_cap, uint32_t* d_edits, uint64_t edit_pool_cap,
                        uint8_t* d_status, uint64_t* d_totals);

/* Intermediate pools (minimizer, seed, work-item records between the kernels) are sized from per-read averages
 * (48 minimizers, 64 seeds, 3 kept clusters per read) times a scale that starts at 1 (GIRAFFE_B200_POOL_SCALE overrides).
 * gb_map_batch / gb_map_paired_batch / gb_map_paired_job notice a chunk that ran out, double the scale and redo that
 * chunk, so the limit never shows in their results.  gb_map_batch_device only enqueues work: after it, this call
 * synchronises and reports whether the batch overflowed (its reads then carry GB_ITEM_OUT_FULL); if so the scale has
 * been doubled and the caller submits the batch again. */
int gb_device_pool_overflow(gb_device* dev, int* overflowed);

/* ---- stage-level dump for parity tests -------------------------------------------------------------------------
 * Runs only the seeding stage (find_minimizers / sort_minimizers_by_score / find_seeds / cluster_seeds / score_cluster /
 * cluster selection / extend_seed_group packing; minimizer_mapper.cpp:3918-4517, :4738-4850, :655-832, :1568-1883,
 * snarl_seed_clusterer.cpp:28-145) on host buffers and returns what the seeding kernels hand to the extension kernel,
 * per read, so tests can compare every intermediate with the oracle's.  paired != 0: reads are interleaved mates and
 * mate 2 is seeded on its reverse complement, as map_paired does (:1503-1506).
 *   minimizers  in score order (after the tie shuffle); seeds in (minimizer, hit) order, each with the index of its
 *   read cluster; clusters in order of their first seed; items = kept clusters in processing order, each with its
 *   (node, read_offset - node_offset) seeds in item_seeds.
 * gb_stage_read.reserved[0] > 1 marks a mate 2 whose clusters tie at the top of the processing order: the reference
 * shuffles them with the pair's LazyRNG after mate 1's alignments have drawn from it (minimizer_mapper.cpp:1723-2043), so
 * the align stage does that shuffle and the keep loop; such a read lists ALL its clusters as items, in comparator order
 * before the shuffle, and reserved[0] is the length of the tied prefix.
 * Offsets in gb_stage_read index the flat output arrays; GB_ERR_CAPACITY when one is too small. */
typedef struct gb_stage_minimizer { uint64_t hash; double score; uint32_t fwd_offset, agg_start, agg_len, is_reverse, hits, reserved; } gb_stage_minimizer;
typedef struct gb_stage_seed { uint32_t node, offset, source, cluster; } gb_stage_seed;
typedef struct gb_stage_cluster { double score, coverage; uint32_t first_seed, n_seeds, fragment, kept_rank; } gb_stage_cluster;   /* kept_rank 0xffffffff: not kept */
typedef struct gb_stage_item { uint32_t cluster, fragment, seed_off, seed_cnt; } gb_stage_item;
typedef struct gb_stage_read { uint32_t min_off, min_cnt, seed_off, seed_cnt, cluster_off, cluster_cnt, item_off, item_cnt, status, reserved[3]; } gb_stage_read;
int gb_debug_seed_stage(gb_device* dev, const gb_map_params* p, int paired,
                        uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                        gb_stage_read* out_reads, gb_stage_minimizer* mins, uint64_t min_cap, gb_stage_seed* seeds, uint64_t seed_cap,
                        gb_stage_cluster* clusters, uint64_t cluster_cap, gb_stage_item* items, uint64_t item_cap,
                        gb_seed* item_seeds, uint64_t item_seed_cap);

/* Multi-GPU emission (SURVEY §8(e), giraffe_main.cpp:2209-2226 on rank 0): after this call gb_map_batch /
 * gb_map_paired_batch also leave the records of every call in the caller's DEVICE buffers — headers d_aln[n_reads], dense
 * mappings / edits with the same offsets as the host outputs — so the ranks can gather whole records over NCCL / NVLink
 * without a second PCIe trip.  The copies are ordered before the call returns.  d_aln = NULL switches it off. */
int gb_device_set_output_mirror(gb_device* dev, gb_alignment* d_aln, gb_mapping* d_maps, uint64_t map_cap, uint32_t* d_edits, uint64_t edit_cap);

/* Run this handle's work on the caller's CUDA stream (cudaStream_t; NULL = the handle's own). */
int gb_device_set_stream(gb_device* dev, void* cuda_stream);
int gb_device_synchronize(gb_device* dev);
/* Device time of the four stages of the last mapping call (seed+cluster, extend, align, compact), ms. */
int gb_stage_times(gb_device* dev, float* ms4);
/* Device time of every kernel of the last mapping call (its last chunk), in launch order: names[i * 48 ..] (NUL
 * terminated) and ms[i]; at most cap entries, *n receives the count.  CUDA events recorded between the launches. */
int gb_kernel_times(gb_device* dev, uint32_t cap, char* names, float* ms, uint32_t* n);
/* Counters of the tail plan of the last mapping call (its last chunk): out4 = tails planned, haplotype trees, tails the
 * align kernels aligned in place (int32 sweep) although their read had a plan, DP cells (columns x rows) handed to
 * xdrop_tile_kernel. */
int gb_plan_stats(gb_device* dev, uint64_t* out4);

/* ------------------------------------------------------------------------------------
 * B3: Aligner::align_pinned(alignment, graph, pin_left = true, xdrop = true, max_gap),
 * batched over explicit haplotype trees      aligner.hpp:183, aligner.cpp:628-686,
 *                                             DozeuInterface::align_pinned dozeu_interface.cpp:724
 * Problem i: tree nodes tree_off[i] .. tree_off[i+1] as (parent index within the tree or -1,
 * oriented node) in DFS visit order (the TreeSubgraph numbering of
 * MinimizerMapper::get_tail_forest, minimizer_mapper.cpp:5838-5845), the root's first
 * root_trim[i] bases cut off; query i = query[query_off[i] .. query_off[i+1]).
 * Outputs per problem: score, mappings (node = tree index, offsets in trimmed coordinates),
 * edits, counts.  Right-pinned problems are posed, as the reference does
 * (minimizer_mapper.cpp:5663-5665), on the reverse-complemented query and reverse tree.
 * A problem's status is GB_ITEM_OUT_FULL when its path needs more than map_cap mappings or
 * edit_cap edits, more than 4096 traceback steps (query bases plus deleted bases), or, on the
 * int32 sweep, more than 2048 tree nodes or 2^21 traceback cells.  A problem the int16 tile
 * kernel can hold never exceeds the sweep's node and cell limits, and a tile that outgrows its
 * own path buffers is recomputed on the sweep, so which kernel ran it does not change the answer.
 * Returns GB_ERR_ARG, before anything is uploaded, when map_cap or edit_cap is 0, a query is
 * longer than 1024 bases, or a tree is malformed: no nodes, a node id below 2 or not in the
 * index, a first node whose parent is not negative, a later node whose parent is negative (a
 * second root), not below its own index or not on the path from the root to the node before
 * it (not DFS visit order), a root_trim not below the root's length, or a node 512 or more
 * levels below the root; or when a max_gap is above 65535 (vg's max_gap is a uint16_t).
 * A max_gap of 0 is taken as 1: the leading insertion may then be one base long and the
 * X-drop threshold is gap_open.
 * ---------------------------------------------------------------------------------- */
int gb_xdrop_pinned_batch(gb_device* dev, uint32_t n,
                          const int32_t* tree_parent, const uint32_t* tree_node, const uint64_t* tree_off,
                          const uint32_t* root_trim, const uint8_t* query, const uint64_t* query_off,
                          const uint32_t* max_gap, uint32_t map_cap, uint32_t edit_cap,
                          int32_t* score, gb_mapping* maps, uint32_t* edits, uint32_t* n_maps, uint32_t* n_edits,
                          uint8_t* status);

/* ------------------------------------------------------------------------------------
 * B3: Aligner::align(alignment, graph, topological_order) — the full (unbanded) local alignment
 * vg runs through GSSW                        aligner.hpp:180, aligner.cpp:571-626, :344-564
 * (rescue fallback fix_dozeu_score minimizer_mapper.cpp:3502-3517; --rescue-algorithm gssw :3390).
 * Problem i: oriented nodes node[node_off[i] .. node_off[i+1]) in topological order; the
 * predecessors of the problem's u-th node are pred[pred_off[g] .. pred_off[g+1]) with
 * g = node_off[i] + u, each an index < u into the same problem (graph edges restricted to the
 * subgraph, at most 255 per node); query i = query[query_off[i] .. query_off[i+1]).
 * Scoring: gb_set_scores; a pair with a non-ACGT base on either side scores 0; the full-length
 * bonus is granted at each read end that is aligned rather than soft clipped.
 * Outputs per problem: score (0 and no mappings when nothing scores > 0), mappings
 * (node = index into the problem's node list), edits (soft clips are insertions on the first /
 * last mapping), counts, status: GB_ITEM_OUT_FULL when the path exceeds map_cap / edit_cap,
 * with score 0 and both counts 0.
 * The three DAG seams (gb_sw_batch, gb_banded_global_batch, gb_xdrop_dag_batch) return
 * GB_ERR_ARG, before anything is uploaded, when map_cap or edit_cap is 0, a query is longer
 * than 1024 bases, a problem has 2^24 or more nodes (traceback steps carry the node index in
 * 24 bits), a node id is below 2, not in the index or has no sequence, a node has more than 255
 * predecessors, or a predecessor index is not below its node's; and GB_ERR_CAPACITY when the
 * batch needs more than 8 GiB of traceback (one byte per base and query prefix).
 * ---------------------------------------------------------------------------------- */
int gb_sw_batch(gb_device* dev, uint32_t n,
                const uint32_t* node, const uint64_t* node_off, const uint32_t* pred, const uint64_t* pred_off,
                const uint8_t* query, const uint64_t* query_off, uint32_t map_cap, uint32_t edit_cap,
                int32_t* score, gb_mapping* maps, uint32_t* edits, uint32_t* n_maps, uint32_t* n_edits,
                uint8_t* status);

/* ------------------------------------------------------------------------------------
 * B3: Aligner::align_global_banded(alignment, graph, band_padding, permissive_banding) — global
 * alignment from a source to a sink inside vg's per-node diagonal band, regular scoring
 *                    aligner.cpp:699-761, banded_global_aligner.cpp:251-742, :1961-2266
 * (the DP fallback for chain middles, minimizer_mapper_from_chains.cpp:2532-3332).
 * Problems are posed like gb_sw_batch (nodes in topological order + predecessor CSR; sources are the
 * nodes without predecessors, sinks the nodes without successors in the problem), with
 * band_padding[i] >= 0 and permissive[i] != 0 for vg's permissive banding.  Queries up to 1024 bases.
 * Scoring: gb_set_scores without the full-length bonus; a pair with a non-ACGT base scores 0.
 * Outputs per problem: score, mappings (node = index into the problem's node list, every offset 0),
 * edits, counts, status: GB_ITEM_NO_BAND when no global alignment fits the band (nothing written),
 * GB_ITEM_OUT_FULL when the path exceeds map_cap / edit_cap (score 0 and both counts 0; the input
 * checks are those of gb_sw_batch, plus band_padding >= 0).  An empty query is a deletion of the
 * shortest source-to-sink path.  Rules and tie-breaking: oracle/banded_global.cpp.
 * ---------------------------------------------------------------------------------- */
int gb_banded_global_batch(gb_device* dev, uint32_t n,
                           const uint32_t* node, const uint64_t* node_off, const uint32_t* pred, const uint64_t* pred_off,
                           const uint8_t* query, const uint64_t* query_off, const int32_t* band_padding, const uint8_t* permissive,
                           uint32_t map_cap, uint32_t edit_cap,
                           int32_t* score, gb_mapping* maps, uint32_t* edits, uint32_t* n_maps, uint32_t* n_edits,
                           uint8_t* status);

/* ------------------------------------------------------------------------------------
 * B3: Aligner::align_xdrop(alignment, graph, order, mems, reverse_complemented = false, max_gap)
 * — the seeded two-pass X-drop alignment of mate rescue     aligner.hpp:200, aligner.cpp:833-855,
 *                                                           DozeuInterface::align dozeu_interface.cpp:608-685
 * Problems are posed like gb_sw_batch (nodes in topological order + predecessor CSR).  seed holds
 * three words per problem: the index of the seed node in the problem's list (0xffffffff: no seed,
 * the last 15 query bases are scanned for their best local match instead, dozeu_interface.cpp:143-208),
 * the offset in that node and the query offset where the seed match begins (the best gapless
 * extension in attempt_rescue, minimizer_mapper.cpp:3345-3358).  Pass 1 extends the query suffix to
 * the right of the seed and fixes the head; pass 2 aligns the query prefix leftwards from the head
 * with traceback; the query right of the head is a soft clip.  score is the score of pass 2 (vg
 * rescores the path afterwards, fix_dozeu_score minimizer_mapper.cpp:3502).  A max_gap of 0 is
 * taken as 1, as in gb_xdrop_pinned_batch.  Status GB_ITEM_OUT_FULL when the path exceeds
 * map_cap / edit_cap, with score 0 and both counts 0.
 * Besides the checks of gb_sw_batch, returns GB_ERR_ARG before anything is uploaded when a max_gap
 * is above 65535 (vg's max_gap is a uint16_t), a node has more than 255 successors, or a seed
 * lies outside its problem: a seed node index not below the node count, a seed offset above the
 * seed node's length or a seed query offset above the query length (an offset equal to the
 * length is a seed at the end).
 * ---------------------------------------------------------------------------------- */
int gb_xdrop_dag_batch(gb_device* dev, uint32_t n,
                       const uint32_t* node, const uint64_t* node_off, const uint32_t* pred, const uint64_t* pred_off,
                       const uint8_t* query, const uint64_t* query_off, const uint32_t* seed, const uint32_t* max_gap,
                       uint32_t map_cap, uint32_t edit_cap,
                       int32_t* score, gb_mapping* maps, uint32_t* edits, uint32_t* n_maps, uint32_t* n_edits,
                       uint8_t* status);

/* ------------------------------------------------------------------------------------
 * B2: WFAExtender::connect / suffix / prefix      gbwt_extender.hpp:386-470, gbwt_extender.cpp:2052-2263
 * (haplotype-consistent gap-affine wavefront alignment; called by the chaining route,
 * minimizer_mapper_from_chains.cpp:2574, :2625, :2955, :3169).
 * Problem i: sequence seq[seq_off[i] .. seq_off[i+1]); mode[i] = 0 connect(from, to), 1 suffix(from),
 * 2 prefix(to); pos holds 4 words per problem: from node, from offset, to node, to offset (oriented
 * nodes; the unused end is ignored).  error_model: 12 numbers {per_base, min, max} for mismatches,
 * gaps, gap length, distance (WFAExtender::ErrorModel, gbwt_extender.hpp:340-385), NULL = defaults.
 * Outputs per problem, as the fields of WFAAlignment (gbwt_extender.hpp:233-307): ok (0: no
 * alignment, 1: alignment, -1: see below), score, node_offset, seq_offset, length, path (oriented
 * nodes, at most path_cap), edits as (length << 2) | op with op 0 match, 1 mismatch, 2 insertion,
 * 3 deletion (at most edit_cap).
 * Each problem runs in a fixed workspace.  ok is -1, with score and counts 0, exactly when the
 * problem needs more than one of: 64 haplotype-trie nodes, 24 576 bytes of trie node sequence,
 * 2 048 graph nodes over all trie nodes, 3 071 stored wavefront points (over the three matrices
 * and all trie nodes), 512 distinct possible scores, 32 successors of one trie node; or stores a
 * point with score 8192 or more, a diagonal outside [-1024, 1024), or a sequence or node offset
 * above 65 535; or when the returned path (after its unused first and trailing nodes are dropped)
 * has more than path_cap nodes or its edits more than edit_cap runs.  A trie node grows along a
 * non-branching haplotype until it holds 1 024 bases, so the trie can hold far more graph nodes
 * than the returned path.  The kernel first tries a 256-cell point table (191 points) and redoes a
 * problem that fills it with the whole table; GIRAFFE_B200_WFA_SMALL_TABLE=0, read on every call,
 * starts with the whole table.  Returns GB_ERR_ARG when path_cap or edit_cap is 0, a mode is above
 * 2 or a sequence is longer than 60 000 bases; n = 0 returns GB_OK without a launch.
 * ---------------------------------------------------------------------------------- */
int gb_wfa_batch(gb_device* dev, uint32_t n, const uint8_t* seq, const uint64_t* seq_off, const uint32_t* mode,
                 const uint32_t* pos, const double* error_model, uint32_t path_cap, uint32_t edit_cap,
                 int32_t* ok, int32_t* score, uint32_t* node_offset, uint32_t* seq_offset, uint32_t* length,
                 uint32_t* path, uint32_t* n_path, uint32_t* edits, uint32_t* n_edits);

/* ------------------------------------------------------------------------------------
 * Chaining route, stage seam: algorithms::find_best_chains  (algorithms/chain_items.hpp:576, chain_items.cpp:733-900)
 * = add_transition_if_legal (:262-355) + chain_items_dp (:395-640) + chain_items_traceback (:642-735), the anchor
 * chaining DP of minimizer_mapper_from_chains.cpp:1201 (fragments) and :1933 (chains).  The zip-code tree that
 * enumerates candidate (source, destination, graph distance) triples (zip_code_tree.cpp; generate_zip_tree_transitions
 * chain_items.cpp:157-260) stays on the caller's side: it is the iterator argument of the reference function.
 *
 * Problem p: anchors[anchor_off[p] .. anchor_off[p+1]) sorted by read_start (ties: longer first, sort_anchor_indexes :102),
 * candidates[cand_off[p] .. cand_off[p+1]) in any order; from / to are anchor indices inside the problem and
 * graph_distance is what the zip-code tree measured between the two hint positions.  A candidate becomes a transition
 * when the read distance exists and is <= max_read_lookback_bases, the exclusion zones do not overlap, the hint offsets
 * fit into graph_distance and the indel |read - graph| is <= max_indel_bases.
 * Outputs: dp_score / dp_source per anchor (the TracedScore table; source 0xffffffff = nowhere), dp_paths / dp_rec per
 * anchor (supported haplotype flags, recombinations so far); per problem up to max_chains chains in the reference's
 * order (penalty ascending): chain_score[p * max_chains + c], chain_begin / chain_count into chain_items (anchor
 * indices left to right; chain_items is laid out like anchors: a problem's chains share its anchor range).
 * n_chains[p] = chains written (0 for a problem without anchors: the reference returns one empty chain of score 0).
 * Where the reference leaves the order open (std::sort of equal keys in the traceback starts and in the final
 * penalty sort) the lower anchor index / the earlier traceback comes first.
 * ---------------------------------------------------------------------------------- */
typedef struct {
    uint32_t read_start, length;               /* Anchor::read_start(), length()                                        */
    uint32_t margin_before, margin_after;      /* read_exclusion_start = read_start - margin_before, ..._end = read_end + margin_after */
    int32_t  score;                            /* Anchor::score()                                                       */
    uint32_t start_hint_offset, end_hint_offset;
    uint32_t base_seed_length;
    uint64_t start_paths, end_paths;           /* anchor_start_paths(), anchor_end_paths() (path_flags_t)               */
} gb_chain_anchor;                             /* 48 bytes */
typedef struct { uint32_t from, to; uint64_t graph_distance; } gb_chain_candidate;     /* 16 bytes */
#define GB_CHAIN_MAX_ANCHORS 65535u            /* anchors (seeds) per problem: both kernels do all-pairs work inside a problem */
typedef struct {
    int32_t  item_bonus;                       /* ChainScoringScheme, chain_items.hpp:407-418 */
    int32_t  recombination_penalty, consistency_bonus;
    uint32_t max_chains;                       /* >= 1 */
    double   gap_scale;
    uint64_t max_indel_bases;                  /* <= 65535 */
    uint64_t max_read_lookback_bases;
} gb_chain_params;
void gb_chain_params_default(gb_chain_params* p);      /* 0, 0, 0, 1 chain, 1.0, 100, unlimited */
int gb_chain_batch(gb_device* dev, const gb_chain_params* params, uint32_t n_problems,
                   const gb_chain_anchor* anchors, const uint64_t* anchor_off,
                   const gb_chain_candidate* candidates, const uint64_t* cand_off,
                   int32_t* dp_score, uint32_t* dp_source, uint64_t* dp_paths, uint32_t* dp_rec,
                   uint32_t* n_chains, int32_t* chain_score, uint32_t* chain_begin, uint32_t* chain_count,
                   uint32_t* chain_items);
/* The same, also returning what add_transition_if_legal made of every candidate: candidate_indel[c] = the indel size of the
 * transition, 0xffffffff for a candidate that is not one (candidate_indel may be NULL). */
int gb_chain_batch_transitions(gb_device* dev, const gb_chain_params* params, uint32_t n_problems,
                               const gb_chain_anchor* anchors, const uint64_t* anchor_off,
                               const gb_chain_candidate* candidates, const uint64_t* cand_off,
                               int32_t* dp_score, uint32_t* dp_source, uint64_t* dp_paths, uint32_t* dp_rec,
                               uint32_t* n_chains, int32_t* chain_score, uint32_t* chain_begin, uint32_t* chain_count,
                               uint32_t* chain_items, uint32_t* candidate_indel);
/* MinimizerMapper::to_anchor (minimizer_mapper_from_chains.cpp:3978-4038), host side: seed i = position seed_pos[2i],
 * seed_pos[2i + 1] (oriented node, offset: the FIRST graph base of a forward-read-strand minimizer's match, the LAST base of a
 * reverse-read-strand one, as the seeds of find_seeds carry them) of a minimizer with pin offset min_offset[i]
 * (Minimizer::value.offset), strand min_is_reverse[i] and length min_length[i].  The anchor is the part of the match on the
 * seed's node (margins record what was cut off, the hint offsets where the seed position lies inside the anchor), scored as an
 * exact match of the whole minimizer.  paths (may be NULL) = Seed::paths.  Pinned by unittest/minimizer_mapper.cpp:882-1048. */
int gb_chain_anchors(const gb_flat_index* ix, const gb_scores* scores, uint32_t n, const uint32_t* seed_pos,
                     const uint32_t* min_offset, const uint8_t* min_is_reverse, const uint32_t* min_length,
                     const uint64_t* paths, gb_chain_anchor* out);

/* The candidate side of the same seam: what zip_tree_transition_iterator enumerates for find_best_chains
 * (chain_items.cpp:116-260 over ZipCodeTree::find_distances, zip_code_tree.cpp): for every destination seed the seeds it
 * can be reached FROM within max_graph_lookback_bases, with the minimum graph distance between the two positions (the
 * number of bases walked from the source position to the destination position; positions on different strands, on
 * parallel alleles or in different components do not see each other).  The reference reads those distances off its
 * zip-code tree; this library has no snarl tree, the distances come from its own distance model (gb_dist_payload: chains
 * of cut nodes and sites with all-pairs tables), which answers the same minimum-distance query — pinned by the
 * "Check iterator" expectations of the reference's zip-code-tree tests on DAGs (unittest/zip_code_tree.cpp).  The
 * iteration ORDER of the tree is not reproduced: the chaining DP does not depend on it (gb_chain_batch).
 * Problem p: seeds seed_pos[2 * i], seed_pos[2 * i + 1] = oriented node, offset for i in seed_off[p] .. seed_off[p+1].
 * Output: candidates of problem p at cand_off[p] .. cand_off[p+1], sorted by (destination, source), from / to = seed
 * indices inside the problem; two seeds at the same position see each other in both directions at distance 0 (the tree
 * offers one of the two; the read-order test of add_transition_if_legal keeps at most one).  cand_off is always filled;
 * GB_ERR_CAPACITY when cand_off[n_problems] > candidate_cap (nothing is written then).  Needs an index with a distance
 * model. */
int gb_chain_candidates_batch(gb_device* dev, uint32_t n_problems, const uint32_t* seed_pos, const uint64_t* seed_off,
                              uint64_t max_graph_lookback_bases, gb_chain_candidate* candidates, uint64_t candidate_cap,
                              uint64_t* cand_off);

/* ------------------------------------------------------------------------------------
 * Surjection onto reference paths and SAM output (`vg giraffe -o SAM`, giraffe_main.cpp:2164-2215):
 * SurjectingAlignmentEmitter (surjecting_alignment_emitter.cpp:28-60) calls Surjector::surject (surjector.cpp:223-630)
 * for every alignment, then HTSAlignmentEmitter writes alignment_to_sam_internal (alignment.cpp:607-754).
 * Giraffe's defaults only: no --prune-low-cplx, no supplementaries (SA), no left-align, no GR / NR / SS tags.
 * Not built here: the realigning route of realigning_surject (surjector.cpp:3255-3560, an alignment that leaves the
 * reference path: gb_surject_device defers such records to the caller rather than write anything vg would not), spliced
 * surjection, BAM and CRAM, @RG / RG, --comments-as-tags, @SQ M5, @PG, and
 * reference paths read from GBZ metadata.
 * ---------------------------------------------------------------------------------- */
typedef struct gb_ref_paths gb_ref_paths;

/* Reference paths in the caller's order (the --ref-paths / sequence-dictionary order, and the order of the @SQ lines):
 * path p is named names[name_off[p] .. name_off[p+1]) and walks the oriented nodes path_nodes[path_off[p] .. path_off[p+1])
 * in GBWT encoding (v = 2 * id + is_reverse), as a vg shim reads them off its PathPositionHandleGraph.  The result is a
 * dense per-node-id record (path, strand, base offset of the node on the path) and each path's length.
 *   GB_ERR_ARG     NULL arrays or out, decreasing offsets
 *   GB_ERR_FORMAT  a node the graph does not have (id past the index, or an id without sequence); a node that occurs more
 *                  than once across all reference paths (LIMIT: every node is on at most one reference path, once, so a
 *                  read's path has one place on the references); a path of 2^31 bases or more (SAM / BAM positions are
 *                  32-bit); an empty path; a name that is empty or holds a byte outside '!'..'~'
 * Freed with gb_ref_paths_free. */
int gb_ref_paths_build(const gb_flat_index* ix, uint32_t n_paths, const uint8_t* names, const uint64_t* name_off,
                       const uint32_t* path_nodes, const uint64_t* path_off, gb_ref_paths** out);
void gb_ref_paths_free(gb_ref_paths* rp);
/* The SAM header HTSAlignmentEmitter writes for these paths with giraffe's defaults: "@HD\tVN:1.5\tSO:unknown" and one
 * "@SQ\tSN:<name>\tLN:<length>" per path in the caller's order, each line ending in '\n'.  No M5 and no @PG (vg adds them
 * from data this library does not hold).  GB_ERR_CAPACITY when out_cap is too small (*out_used = bytes needed). */
int gb_sam_header(const gb_ref_paths* rp, char* out, uint64_t out_cap, uint64_t* out_used);
/* Copies the reference paths to the handle's HBM (8 B per node id plus the names); they replace earlier ones.  GB_ERR_ARG
 * when rp was built for a graph with a different node count than the handle's. */
int gb_device_set_ref_paths(gb_device* dev, const gb_ref_paths* rp);

/* One surjected record (40 B): what HTSAlignmentEmitter writes for one Alignment.  The CIGAR is ops cigar[cigar_off ..
 * cigar_off + n_cigar) of the cigar pool in BAM encoding, length << 4 | op (M 0, I 1, D 2, S 4). */
typedef struct gb_sam_record {
    uint32_t read_id;
    uint16_t flag;                /* SAM FLAG                                                               */
    uint8_t  mapq;                /* MAPQ carried over from the input record; 0 when unmapped               */
    uint8_t  route;               /* GB_SURJ_*                                                              */
    int32_t  ref;                 /* reference path index, -1 unmapped                                      */
    int32_t  pos;                 /* 0-based leftmost reference base, -1 unmapped                           */
    int32_t  score;               /* AS: score_contiguous_alignment of the surjected path (0 when unmapped) */
    int32_t  mate_ref, mate_pos;  /* paired: the mate's ref / pos (-1 unmapped); unpaired: -1, -1           */
    int32_t  tlen;                /* compute_template_lengths (hts_alignment_emitter.cpp:812); unpaired: 0  */
    uint32_t cigar_off, n_cigar;
} gb_sam_record;

#define GB_SURJ_DIRECT    0u      /* one path chunk covers the whole read (surjector.cpp:3235-3253): copied over        */
#define GB_SURJ_UNMAPPED  1u      /* unmapped input, or no node of the read's path is on a reference path              */
#define GB_SURJ_REALIGN   2u      /* deferred: the read, or its mate, leaves the reference path and needs vg's realigning
                                     route, which is not built here.  No SAM line is written for it; the caller surjects
                                     these records (and, paired, their mates: both carry this route) with vg's Surjector */
#define GB_SURJ_ABSENT    3u      /* GB_ALN_ABSENT input rank: no record (the SAM emitter skips it)                    */

/* Surjector::surject for records already in HBM (gb_map_batch_device / gb_map_paired_job_device outputs, or any records
 * copied there); every array is a DEVICE address.  Record x of d_aln gives d_out[x].  Per record, on the paths set by
 * gb_device_set_ref_paths:
 *   - the read's path is cut into chunks as extract_overlapping_paths does (surjector.cpp:4109): consecutive mappings
 *     on consecutive steps of one path strand.  One chunk over all mappings is the direct route: the path is copied, POS is
 *     its leftmost reference base, CIGAR is cigar_against_path (alignment.cpp:1339: M for matches and substitutions,
 *     reversed on the reverse strand, end insertions as S, simplify_cigar), the score is score_contiguous_alignment
 *     (alignment_scorer.cpp:159-245) with vg's default scores 1/4/6/1/5 whatever gb_set_scores set: vg's Surjector keeps
 *     its own default aligner (surjector.cpp:45-57), MAPQ is carried over.
 *   - no mapping on a reference path: unmapped (surjector.cpp:436-480); a read with several chunks, and its mate when
 *     paired: GB_SURJ_REALIGN, deferred (ref / pos -1, no CIGAR, no SAM line; *n_realign counts them, may be NULL).
 *   - flags: sam_flag / determine_flag (alignment.cpp:697-754, :2898): 0x10 reverse, 0x4 unmapped, 0x100 for GB_ALN_SECONDARY.
 * Paired records (GB_ALN_PAIRED) must come as the mappers lay them out: the mate of record x is record x ^ 1 (read_id ^ 1).
 * They get 0x1, 0x40 / 0x80 (even / odd read), the mate's ref / pos, 0x8 / 0x20 from the mate, TLEN from
 * compute_template_lengths, and 0x2 when both lie on one path facing each other and |TLEN| <= tlen_max (tlen_max 0: no
 * limit; giraffe passes mean + 6 stdev of a finalized fragment distribution, giraffe_main.cpp:2334-2339).
 *   GB_ERR_ARG       no reference paths on the handle, NULL arrays, a record gb_emit_gaf_device would refuse, a paired
 *                    record whose mate is not at x ^ 1 (decided on the device; nothing is written)
 *   GB_ERR_CAPACITY  cigar_cap is too small: *cigar_used is the pool size needed, nothing is written; also when the pool
 *                    would pass 2^32 ops (cigar_off is 32-bit: split the batch)
 * On success *cigar_used is the extent of the cigar pool used (a record's region is sized by its raw op count, so the
 * pool may hold gaps).  The call synchronises once, for the pool size; the fill is left enqueued on the handle's stream. */
int gb_surject_device(gb_device* dev, uint32_t n, const gb_alignment* d_aln, const gb_mapping* d_mappings, uint64_t mapping_pool_len,
                      const uint32_t* d_edits, uint64_t edit_pool_len, uint32_t n_reads, const uint64_t* d_read_off, int64_t tlen_max,
                      gb_sam_record* d_out, uint32_t* d_cigar, uint64_t cigar_cap, uint64_t* cigar_used, uint32_t* n_realign);

/* SAM alignment lines of surjected records, formatted on the GPU (alignment_to_sam_internal, alignment.cpp:607-695): QNAME
 * (names, or read<i> when d_names is NULL; paired records lose a trailing [/_][12]; '*' when empty), FLAG, RNAME, 1-based
 * POS, MAPQ, CIGAR, RNEXT ('=' on the same path, '*' without a mate location), PNEXT, TLEN, SEQ and QUAL reverse-complemented
 * / reversed on the reverse strand (QUAL '*' when d_quals is NULL), then AS:i.  An unmapped paired record takes its mate's
 * RNAME and POS (SAMv1 §2.4.1).  GB_SURJ_ABSENT and GB_SURJ_REALIGN records are skipped.  The header is gb_sam_header's.  The contract of
 * gb_emit_gaf_device: GB_ERR_ARG for a record outside its read, cigar pool or paths (decided on the device), GB_ERR_CAPACITY
 * with *out_used = bytes needed, one synchronisation, the fill left enqueued. */
int gb_emit_sam_device(gb_device* dev, uint32_t n, const gb_sam_record* d_rec, const uint32_t* d_cigar, uint64_t cigar_len,
                       uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals, const uint64_t* d_read_off,
                       const uint8_t* d_names, const uint64_t* d_name_off, char* d_out, uint64_t out_cap, uint64_t* out_used);

/* Kernel-only timing of the last gb_*_batch call on this handle, milliseconds
 * (CUDA events on the handle's stream around the kernels, copies excluded). */
float gb_last_kernel_ms(const gb_device* dev);
/* Number of kernels this library launched on the handle since creation. */
uint64_t gb_launch_count(const gb_device* dev);

#ifdef __cplusplus
}
#endif
#endif /* GIRAFFE_B200_H */
