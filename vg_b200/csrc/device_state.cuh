// device_state.cuh — the opaque gb_device handle: HBM-resident index, stream, workspaces.
#pragma once
#include "giraffe_b200.h"
#include "entry_guard.h"
#include "device_index.cuh"
#include "extend.cuh"
#include "map_state.cuh"
#include "xdrop_tile.cuh"
namespace gb { struct DbgCluster; }

#include <cuda_runtime.h>
#include <cstddef>
#include <string>
#include <vector>

namespace gb {

constexpr int EXTEND_WARPS = 8;           // warps per CTA of the extension kernel
constexpr uint32_t EXTEND_Q_CAP = 512;    // frontier entries per warp (64 B each)
constexpr uint32_t EXTEND_A_CAP = 4096;   // path-arena nodes per warp (8 B each)

int fail_cuda(cudaError_t e, const char* what);

#define GB_CUDA(call)                                                        \
    do {                                                                     \
        cudaError_t _e = (call);                                             \
        if (_e != cudaSuccess) return ::gb::fail_cuda(_e, #call);            \
    } while (0)

// Growable device buffer (cudaMalloc on demand, never shrinks).
template <typename T>
struct DevBuf {
    T* ptr = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    void release() { if (ptr) cudaFree(ptr); ptr = nullptr; cap = 0; }
    int reserve(size_t n) {
        if (n <= cap && ptr) return GB_OK;
        if (ptr) { cudaFree(ptr); ptr = nullptr; cap = 0; }
        if (n == 0) n = 1;
        cudaError_t e = cudaMalloc(&ptr, n * sizeof(T));
        if (e != cudaSuccess) { ptr = nullptr; return fail_cuda(e, "cudaMalloc"); }
        cap = n;
        return GB_OK;
    }
    // allocate `n` elements, copy `n_copy` (default n) from host
    int upload(const T* host, size_t n, cudaStream_t s, size_t n_copy = (size_t)-1) {
        int rc = reserve(n);
        if (rc) return rc;
        if (n_copy == (size_t)-1) n_copy = n;
        if (n_copy && host) {
            cudaError_t e = cudaMemcpyAsync(ptr, host, n_copy * sizeof(T), cudaMemcpyHostToDevice, s);
            if (e != cudaSuccess) return fail_cuda(e, "cudaMemcpyAsync H2D");
        }
        return GB_OK;
    }
};

// Typed slices of one workspace, each starting on a 256-byte boundary (CUB's temp storage is one more slice).  Without a
// base it only adds up the bytes, so carve() below runs the same layout once to size the buffer and once to bind it.
struct Carve {
    uint8_t* base;
    size_t bytes = 0;
    template <typename T> T* take(size_t n) {
        T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
        bytes += (n * sizeof(T) + 255) & ~(size_t)255;
        return p;
    }
};

// Reserves `ws` for the slices `layout(Carve&)` takes, then binds them to it (the pattern of cub::AliasTemporaries).
template <typename Layout>
int carve(DevBuf<uint8_t>& ws, Layout&& layout) {
    Carve size{nullptr};
    layout(size);
    if (int rc = ws.reserve(size.bytes)) return rc;
    Carve bind{ws.ptr};
    layout(bind);
    return GB_OK;
}

// The mapping pipeline's device counters, zeroed at the start of every map_device call: work counters that hand units
// to the persistent kernels, and the cursors and counts of what the kernels appended to the pools and lists.  The
// extension launches count on d->work_counter, so they have no field here.
struct MapCursors {
    uint32_t seed_work;                              // seeding, first pass
    uint32_t min_cursor, seed_cursor, item_cursor, ext_cursor;      // SeedPools
    uint32_t align_work;                             // align fast path, then the warp-per-unit align kernel
    uint32_t slow_count;                             // units the fast path leaves to the warp-per-unit kernels
    uint32_t seed_retry_count;                       // units the first seeding pass could not fit
    uint32_t seed_retry_work;                        // seeding, second pass
    uint32_t seed_retry_again;                       // units the second pass lists again (not read)
    uint32_t rescue_count, rescue_work;              // pairs deferred to the rescue build of align_kernel_pe
    uint32_t pool_overflow;                          // sticky: a pool ran out (the host doubles the pools and reruns)
    uint32_t plan_work;                              // tail_plan_kernel
    uint32_t big_ext_count;                          // items redone with the large extension strides
    uint32_t tile_count, tile_units;                 // tiles, tile bytes / 16
    uint32_t tile_list_count[2 * TILE_CLASSES];      // [wave][class]: tail_plan_kernel indexes it as one array
    uint32_t tile_path_words;                        // result path pool of the tiles
    uint32_t decide_work;                            // tail_decide_kernel
    uint32_t tile_work[2 * TILE_CLASSES];            // [wave][class]
};
static_assert(sizeof(MapCursors) == 43 * sizeof(uint32_t), "MapCursors is 43 packed 32-bit counters");
static_assert(offsetof(MapCursors, tile_path_words) == offsetof(MapCursors, tile_list_count) + 2 * TILE_CLASSES * sizeof(uint32_t),
              "the two waves' tile list counts are contiguous");

} // namespace gb

struct gb_device;
namespace gb {

// map.cu: one batch of reads already in HBM through every stage, records compacted into out_maps / out_edits (paired:
// d_read_off[0] == 0 and d_read_off[n_reads] <= total_bases, the size of the working copy of the reads).
int map_device(gb_device* d, const gb_map_params* hp, uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals,
               const uint64_t* d_read_off, uint32_t max_len, uint64_t total_bases,
               gb_alignment* d_aln, uint8_t* d_status, bool paired,
               gb_mapping* out_maps, uint64_t out_map_cap, uint32_t* out_edits, uint64_t out_edit_cap,
               const uint64_t* d_run_base, uint32_t read_base, uint64_t* d_totals, uint32_t* d_overflow);

// A batch that set MapCursors::pool_overflow is redone with the intermediate pools doubled: this doubles them, or
// refuses (GB_ERR_CAPACITY) once they are at 1024x the per-read averages.
int grow_pools_for_rerun(gb_device* d);

// Read 1 of a pair, L1 bases long, takes map_paired's single-end fallback when the fragment limit (mean +
// paired_distance_stdevs * stdev) is below its distance limit (minimizer_mapper.cpp:1469-1471).
__host__ __device__ inline bool single_end_fallback(int64_t fragment_limit, int64_t distance_limit, int64_t L1) {
    const int64_t read_limit = L1 + 50;
    return fragment_limit < (distance_limit > read_limit ? distance_limit : read_limit);
}
// The refusal of a paired batch in which only some pairs take the fallback.
inline constexpr char MIXED_FALLBACK_REFUSAL[] = "fragment distance limit below the read distance limit for some pairs only (mixed single-end "
                                                 "fallback, minimizer_mapper.cpp:1471, is not supported in one batch)";

} // namespace gb

struct gb_device {
    int device = 0;
    int n_sms = 0;
    std::vector<uint32_t> h_node_len;      // host copy of the node lengths (workspace sizing of the DP seams)
    bool chain_coords_fit = true;          // every used node's chain coordinates fit the mapping kernels' int32 c_in / c_out
    // first-pass seeding table sizes (minimizers, clusters per read); GIRAFFE_B200_SEED_TABLES="Mc,Cc" overrides
    uint32_t seed_mc = 64, seed_cc = 16, seed_ns = 64;
    cudaStream_t stream = nullptr, own_stream = nullptr;
    cudaEvent_t ev_stage[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    gb::DevIndex ix{};
    gb::DevScores sc{1, 4, 6, 1, 5};
    gb::DevBuf<gb_node_rec> nodes;
    gb::DevBuf<uint8_t> seq;
    gb::DevBuf<uint32_t> gbwt;
    gb::DevBuf<gb_dist_payload> dist;
    gb::DevBuf<gb_min_cell> table;
    gb::DevBuf<gb_hit> hits;
    gb::DevBuf<uint32_t> slot_order;
    gb::DevBuf<gb_slot_rec> slots; gb::DevBuf<uint16_t> site_dist;
    gb::DevBuf<gb::QEntry> ws_queue;
    gb::DevBuf<gb::ArenaNode> ws_arena;
    gb::DevBuf<uint32_t> p_post;                     // items extend_kernel hands to extend_finish_kernel
    uint32_t* work_counter = nullptr;
    float last_kernel_ms = 0.f;
    uint64_t launches = 0;
    // mapping pipeline: parameter tables, intermediate pools, workspaces, I/O staging
    bool tables_ready = false; uint32_t tables_hard_hit_cap = 0;
    gb::DevBuf<double> t_hit, t_plo, t_phred;
    gb::DevBuf<gb::ReadState> p_states;
    gb::DevBuf<gb::DevMinimizer> p_min;
    gb::DevBuf<gb::DevSeed> p_seeds;
    gb::DevBuf<gb::DevItem> p_items;
    gb::DevBuf<gb_seed> p_ext_seeds;
    gb::DevBuf<gb::MapCursors> p_cursors;
    gb::DevBuf<uint32_t> p_ext_count, p_path, p_mism;
    gb::DevBuf<uint8_t> p_ext_status;
    gb::DevBuf<uint32_t> p_big_list, p_big_of, p_big_path, p_big_mism; gb::DevBuf<gb_extension> p_big_ext;      // ExtendBig
    gb::DevBuf<gb_extension> p_ext;
    gb::DevBuf<uint8_t> ws_tail, ws_cand, w_reads, w_quals, ws_rescue;
    gb::DevBuf<gb::PairState> p_pairs;
    gb::DevBuf<uint32_t> p_retry;         // units the first seeding pass could not fit
    gb::DevBuf<uint32_t> p_slow;          // pairs routed to the warp-per-pair align kernel
    gb::DevBuf<uint32_t> p_rescue;        // pairs the plain kernel defers to the rescue instantiation
    gb::DevBuf<gb_mapping> pad_maps;
    gb::DevBuf<uint32_t> pad_edits;
    gb::DevBuf<uint64_t> c_map_off, c_edit_off, c_totals;
    gb::DevBuf<uint8_t> c_tmp;
    // host-buffer entry points: two staging sets so chunk i+1 uploads and chunk i-1 downloads while
    // chunk i computes (streams s_in / stream / s_out)
    struct IoSet {
        gb::DevBuf<uint8_t> reads, quals, status;
        gb::DevBuf<uint64_t> read_off, totals;
        gb::DevBuf<gb_alignment> aln;
        gb::DevBuf<gb_mapping> maps;
        gb::DevBuf<uint32_t> edits;
        cudaEvent_t ev_in = nullptr, ev_done = nullptr, ev_hdr = nullptr, ev_out = nullptr, ev_k0 = nullptr, ev_k1 = nullptr;
    } io[2];
    cudaStream_t s_in = nullptr, s_out = nullptr;
    uint64_t* h_totals = nullptr;          // pinned, 3 per set: mappings, edits, pool-overflow flag
    double pool_scale = 1.0;               // intermediate pools = per-read averages x this; doubled when a chunk overflows (GIRAFFE_B200_POOL_SCALE)
    uint32_t pool_reruns = 0;              // chunks redone because of it
    gb::DbgCluster* dbg_clusters = nullptr; bool debug_stop_after_seed = false;     // gb_debug_seed_stage
    // tail plan + DP tiles (xdrop_tile.cuh); GIRAFFE_B200_TILES=0 keeps every tail DP in the align kernels (int32 sweep)
    bool use_tiles = true; uint32_t last_tile_problems = 0;
    gb_alignment* mirror_aln = nullptr; gb_mapping* mirror_maps = nullptr; uint32_t* mirror_edits = nullptr; uint64_t mirror_map_cap = 0, mirror_edit_cap = 0;
    gb::DevBuf<gb::TailPlanEntry> pl_entries;
    gb::DevBuf<uint32_t> pl_unit_base, pl_unit_count, pl_tile_off, pl_lists, pl_paths;
    gb::DevBuf<uint8_t> pl_tiles, ws_tile;
    gb::DevBuf<gb::TileResult> pl_results;
    gb::DevBuf<uint64_t> pl_stats;
    // per-kernel device times of the last map_device call (events between the launches)
    static constexpr int KT_MAX = 48;
    cudaEvent_t kt_ev[KT_MAX] = {}; const char* kt_name[KT_MAX] = {}; int kt_n = 0;
    void kt_reset() { kt_n = 0; }
    int kt_mark(const char* name) {
        if (kt_n >= KT_MAX) return GB_OK;
        if (!kt_ev[kt_n]) { cudaError_t e = cudaEventCreate(&kt_ev[kt_n]); if (e != cudaSuccess) return gb::fail_cuda(e, "cudaEventCreate"); }
        cudaError_t e = cudaEventRecord(kt_ev[kt_n], stream);
        if (e != cudaSuccess) return gb::fail_cuda(e, "cudaEventRecord");
        kt_name[kt_n++] = name;
        return GB_OK;
    }
    gb::DevBuf<uint64_t> c_run;            // running mapping / edit totals of a host-buffer call
    uint32_t map_chunk = 1u << 20;         // reads per chunk; GIRAFFE_B200_MAP_CHUNK overrides
    gb::DevBuf<uint8_t> emit_ws;           // gb_emit_*_device: per-record sizes, offsets, scan temporaries
    gb::DevBuf<uint8_t> bgzf_ws;           // gb_bgzf_compress_device: member slots, token slots, member sizes and offsets
    gb::DevBuf<uint8_t> inflate_ws;        // gb_bgzf_decompress_device: the member list and the walk's summary
    gb::DevBuf<uint8_t> fastq_ws;          // gb_fastq_parse_device: line ends, per-read lengths and offsets, scan temporaries
    // the paired jobs: one sub-batch's records, its gathered or uploaded reads, the per-pair training arrays, the buffered pairs
    struct PairedJobWs {
        gb::DevBuf<gb_alignment> aln;
        gb::DevBuf<uint8_t> status, reads, quals, scan_tmp;
        gb::DevBuf<gb_mapping> maps;
        gb::DevBuf<uint32_t> edits, pair, buffered;
        gb::DevBuf<uint64_t> off, totals, append_off;
        gb::DevBuf<int64_t> out;
    } pj;
    uint32_t pj_windows = 0; double pj_training_ms = 0.0;      // training windows of the last such call and their host-clocked time
    // gb_device_set_ref_paths: per node id {path << 1 | the path walks the node reversed (0xFFFFFFFF: on no path), base offset
    // of the node on the path}, and the path names addressed by ref_name_off[n_ref_paths + 1]
    bool ref_ready = false; uint32_t n_ref_paths = 0;
    gb::DevBuf<uint32_t> ref_node;
    gb::DevBuf<uint8_t> ref_names; gb::DevBuf<uint64_t> ref_name_off;
    gb::DevBuf<uint8_t> surj_ws;           // gb_surject_device: validation flag, per-record op counts, offsets, scan temporaries
};
