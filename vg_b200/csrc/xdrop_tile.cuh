// xdrop_tile.cuh — the pinned X-drop tail DP as its own compact kernel, fed from a device work list.
//
//   Aligner::align_pinned (xdrop)              aligner.cpp:628-686
//   DozeuInterface::align_pinned / do_poa      dozeu_interface.cpp:210-307, :724-766
//   traceback -> Path                          dozeu_interface.cpp:338-572
//   dz_extend / dz_trace                       vgteam/dozeu @ d0e9ba6 (ABSENT; the contract is oracle/tail_align.cpp)
//
// A *tile* is everything one DP problem needs, contiguous in HBM (written by the planning kernel, tail_plan.cuh, or by
// pack_tiles_kernel for the stage seam): a 32-byte header, the haplotype tree (8 B per node), the subgraph bases of the
// tree in node order (1 B/base) and the query.  A warp stages its tile into shared memory with ONE bulk asynchronous
// copy (cp.async.bulk global -> shared, completion on an mbarrier), prefetching the next tile of its list while it works
// on the current one, then runs the DP entirely out of registers and shared memory:
//
//   * cells are int16, two per 32-bit register (dozeu itself is int16); a column of 32 R rows is held by the warp as
//     R/2 packed registers per lane: lane l owns rows [l R/2, (l+1) R/2) in the low halves and the same rows + 16 R in
//     the high halves, so the whole recurrence runs on DPX / packed video instructions (VIADDMNMX.S16x2, VIMNMX.S16x2,
//     VIADD.16x2) with no shared-memory traffic for H / E;
//   * substitution scores come from a query profile in shared memory (one packed word per register and reference base,
//     the full-length bonus folded into row m), the reference base of a column is warp-uniform;
//   * the in-column insertion chain F[j] = max_{i<j}(H'[i] + i ge) - go - (j-1) ge is a running maximum inside the lane
//     (R/2 steps, both halves at once) plus ONE 5-step max-scan over the lanes per column, instead of one scan per
//     32 cells;
//   * X-drop exactly as the contract states it (cell granular, against the best H of the earlier columns of the
//     root-to-node lineage): dead cells are the constant NEG16 and every live value stays above ALIVE_FLOOR, which
//     the eligibility test (tile_scores_fit_int16) guarantees from the scoring parameters and the query length;
//   * traceback flags are 4 bits per cell, packed 2 cells per byte, one coalesced store per lane and column;
//   * the best cell (first node, first column, smallest row on ties) is tracked per row in registers.
// Problems the int16 ranges cannot hold, or whose tile / traceback exceed the per-warp budgets, never reach this kernel:
// they stay on the int32 column sweep of tail.cuh, which computes the same function.
#pragma once
#include "tail.cuh"
#include <cstdio>

namespace gb {

constexpr int32_t NEG16 = -16384;                 // dead cell
constexpr int32_t ALIVE_FLOOR = -8192;            // every live value is above this, every dead-derived value below
constexpr uint32_t NEG16x2 = 0xC000C000u;
constexpr uint32_t TILE_SMEM_BYTES = 4096;        // tiles up to this size are staged by the bulk copy (larger ones are read in place)
constexpr uint32_t TILE_MAX_NODES = 1024;
constexpr uint32_t TILE_MAX_ROWS = 512;           // m + 1 <= 512
constexpr uint32_t TILE_TB_BYTES = 512 * 1024;    // per-warp traceback workspace
constexpr uint32_t TILE_STEP_CAP = 4096;          // traceback steps
constexpr uint32_t TILE_MAP_CAP = 96, TILE_EDIT_CAP = 192;    // result path of one tail (mappings / edits)
constexpr int TILE_WARPS = 8;

#define GB_TILE_LEFT        1u     // result is reported on the reverse strand (left tail: reverse_complement_path + translate_down)
#define GB_TILE_TREE_SPACE  2u     // stage seam: mappings keep tree indices (no translation)
#define GB_TILE_ST_OK       0u
#define GB_TILE_ST_FULL     1u     // a result / traceback capacity was exceeded
#define GB_TILE_ST_CANCELLED 2u    // second-wave tile whose tail the reference would not align (tail_decide_kernel)
#define GB_TILE_ST_PENDING  0xffu

struct __align__(16) TileHeader {
    uint32_t m;            // query length
    uint32_t n_nodes;
    uint32_t n_bases;      // sum of node lengths (root already trimmed)
    uint32_t max_gap;      // >= 1
    uint32_t flags;        // GB_TILE_*
    uint32_t root_trim;    // offset trimmed from the root node
    uint32_t bytes;        // whole tile, multiple of 16
    uint32_t result;       // index of the TileResult record
};
struct TileNode { uint16_t parent; uint16_t len; uint32_t node; };      // parent 0xffff: root; node: oriented graph node
// tile = TileHeader | TileNode[n_nodes rounded up to even] | bases[n_bases rounded to 16] | query[m rounded to 16]
__host__ __device__ inline uint32_t tile_bytes(uint32_t n_nodes, uint32_t n_bases, uint32_t m) {
    return 32u + 8u * ((n_nodes + 1u) & ~1u) + ((n_bases + 15u) & ~15u) + ((m + 15u) & ~15u);
}

struct __align__(16) TileResult {
    int32_t score; uint32_t status;        // GB_TILE_ST_*
    uint32_t n_maps, n_edits;
    uint32_t path_off;                     // into the result path pool (32-bit words): n_maps x gb_mapping, then n_edits words
    uint32_t cells_lo, cells_hi, pad;      // DP cells computed (profiling)
};

// rows per lane needed for a query of length m
constexpr int TILE_CLASSES = 6;
__host__ __device__ inline int tile_class(uint32_t m) {                    // R = 2, 4, 6, 8, 12, 16 rows per lane
    const uint32_t rows = m + 1;
    return rows <= 64 ? 0 : (rows <= 128 ? 1 : (rows <= 192 ? 2 : (rows <= 256 ? 3 : (rows <= 384 ? 4 : 5))));
}
__host__ __device__ constexpr int tile_class_rows(int cls) { return cls == 0 ? 2 : (cls == 1 ? 4 : (cls == 2 ? 6 : (cls == 3 ? 8 : (cls == 4 ? 12 : 16)))); }
// traceback bytes per lane and column for P = R / 2 packed registers (padded so one store serves a lane)
__host__ __device__ constexpr int tile_tb_stride(int P) { return P == 1 ? 1 : (P == 2 ? 2 : (P <= 4 ? 4 : 8)); }

// The int16 ranges hold for these scores and this query length (see the header comment).
__host__ __device__ inline bool tile_scores_fit_int16(const DevScores& s, uint32_t m, uint32_t max_gap) {
    if (m == 0 || m + 1 > TILE_MAX_ROWS) return false;
    const int64_t ge = s.gap_extend, go = s.gap_open;
    if (s.match < 0 || s.mismatch < 0 || ge < 0 || go < ge || s.full_length_bonus < 0) return false;
    const int64_t xt = go + ge * ((int64_t)max_gap - 1);
    const int64_t top = (int64_t)m * s.match + s.full_length_bonus;            // largest score
    const int64_t drop = xt + go + (int64_t)(m + 1) * ge + s.mismatch + s.match + s.full_length_bonus;   // how far below run_max a live value can sit inside a column
    return top < 12000 && drop < 7000 && top + (int64_t)(m + 1) * ge < 24000;
}

#ifdef GB_TILE_DEBUG
#define TILE_FAIL(code) do { if (lane_id() == 0) printf("tile fail %d: m=%d nodes=%u bases=%u best=%d node=%u col=%u row=%u steps=%u\n", code, m, hd.n_nodes, hd.n_bases, best, best_node, best_col, best_row, n_steps); status_out = GB_TILE_ST_FULL; return 0; } while (0)
#else
#define TILE_FAIL(code) do { status_out = GB_TILE_ST_FULL; return 0; } while (0)
#endif

// ---- packed helpers ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pk2(int lo, int hi) { return ((uint32_t)lo & 0xffffu) | ((uint32_t)hi << 16); }
__device__ __forceinline__ uint32_t pk1(int v) { return pk2(v, v); }
__device__ __forceinline__ int lo16(uint32_t x) { return (int)(int16_t)(x & 0xffffu); }
__device__ __forceinline__ int hi16(uint32_t x) { return (int)(int16_t)(x >> 16); }
// 0xffff in each half whose signed value is negative
// (PTX prmt in its default mode replicates the sign of the selected byte when bit 3 of the selector nibble is set; the
// __byte_perm intrinsic ignores that bit)
__device__ __forceinline__ uint32_t sign_mask2(uint32_t x) { uint32_t r; asm("prmt.b32 %0, %1, %1, 0xbb99;" : "=r"(r) : "r"(x)); return r; }

// ---- bulk copy + mbarrier (PTX) ----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- per-warp workspaces -----------------------------------------------------------------------------------------
struct TileWs {
    uint8_t* tb;          // [TILE_TB_BYTES]   packed traceback flags, column-major, one word of 2R bytes... (R/2 bytes per lane and column)
    uint32_t* cols;       // [TILE_D_CAP][2][32 * P_MAX]  last column (H, E) of the node at each depth
    uint32_t* node_col;   // [TILE_MAX_NODES]  first traceback column of each node
    uint8_t* node_live;   // [TILE_MAX_NODES]  1: computed and its last column has a live cell
    int32_t* node_lin;    // [TILE_MAX_NODES]  lineage maximum after the node
    uint16_t* node_depth; // [TILE_MAX_NODES]
};
constexpr uint32_t TILE_D_CAP = 256;
__host__ __device__ inline size_t tile_ws_bytes() {
    return (size_t)TILE_TB_BYTES + (size_t)TILE_D_CAP * 2 * 32 * 8 * 4 + (size_t)TILE_MAX_NODES * (4 + 1 + 4 + 2) + 256;
}
__device__ inline TileWs carve_tile_ws(uint8_t* base) {
    TileWs w; uint8_t* p = base;
    w.tb = p; p += TILE_TB_BYTES;
    w.cols = (uint32_t*)p; p += (size_t)TILE_D_CAP * 2 * 32 * 8 * 4;
    w.node_col = (uint32_t*)p; p += (size_t)TILE_MAX_NODES * 4;
    w.node_lin = (int32_t*)p; p += (size_t)TILE_MAX_NODES * 4;
    w.node_depth = (uint16_t*)p; p += (size_t)TILE_MAX_NODES * 2;
    w.node_live = p;
    return w;
}

// Can this problem run on the tile kernel?  (everything else stays on tail.cuh's int32 sweep)
__host__ __device__ inline bool tile_eligible(const DevScores& s, uint32_t m, uint32_t max_gap, uint32_t n_nodes, uint32_t n_bases, uint32_t max_depth) {
    if (!tile_scores_fit_int16(s, m, max_gap)) return false;
    if (n_nodes == 0 || n_nodes > TILE_MAX_NODES || max_depth >= TILE_D_CAP || n_bases == 0 || n_bases > 0xffffu) return false;
    const int R = tile_class_rows(tile_class(m));
    return (uint64_t)n_bases * 32u * (uint32_t)tile_tb_stride(R / 2) <= TILE_TB_BYTES;
}

// -----------------------------------------------------------------------------------------------------------------
// The DP of one tile.  `tile` points at the staged (or in-place) tile; prof is the warp's profile area
// [5][32 * P] words; out_maps / out_edits are the warp's result scratch.  Returns the score; n_maps / n_edits / status out.
// -----------------------------------------------------------------------------------------------------------------
template <int R>
__device__ __noinline__ int32_t xdrop_tile_dp(const DevScores& sc, const uint8_t* tile, const TileWs& ws, uint32_t* prof,
                                              gb_mapping* out_maps, uint32_t* out_edits, uint32_t& n_maps_out, uint32_t& n_edits_out,
                                              uint32_t& map_base_out, uint32_t& edit_base_out, uint32_t& status_out, uint64_t& cells_out) {
    constexpr int P = R / 2;
    constexpr int HALF = 16 * R;
    constexpr int TBS = tile_tb_stride(P);
    const int lane = lane_id();
    const TileHeader hd = *reinterpret_cast<const TileHeader*>(tile);
    const TileNode* nodes = reinterpret_cast<const TileNode*>(tile + 32);
    const uint8_t* bases = tile + 32 + 8 * ((hd.n_nodes + 1u) & ~1u);
    const uint8_t* q = bases + ((hd.n_bases + 15u) & ~15u);
    const int m = (int)hd.m;
    const int go = sc.gap_open, ge = sc.gap_extend;
    const int xt = go + ge * ((int)hd.max_gap - 1);
    status_out = GB_TILE_ST_OK; n_maps_out = 0; n_edits_out = 0;
    uint64_t cells = 0;

    // ---- query profile: prof[b][lane * P + i] = packed substitution scores of the lane's rows against base b --------
    // row j scores query base j - 1; the full-length bonus rides on row m; rows 0 and > m get the mismatch score (never used)
    {
        const int mm = -sc.mismatch;
#pragma unroll
        for (int i = 0; i < P; i++) {
            const int jl = lane * P + i, jh = HALF + lane * P + i;
            const uint8_t ql = (jl >= 1 && jl <= m) ? q[jl - 1] : (uint8_t)0, qh = (jh >= 1 && jh <= m) ? q[jh - 1] : (uint8_t)0;
            const int bl = jl == m ? sc.full_length_bonus : 0, bh = jh == m ? sc.full_length_bonus : 0;
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const uint8_t rb = (uint8_t)("ACGT"[b]);
                prof[b * 32 * P + lane * P + i] = pk2((ql == rb ? sc.match : mm) + bl, (qh == rb ? sc.match : mm) + bh);
            }
            prof[4 * 32 * P + lane * P + i] = pk2(mm + bl, mm + bh);
        }
    }
    // rows beyond the query are not cells
    uint32_t inval[P];
#pragma unroll
    for (int i = 0; i < P; i++) inval[i] = ((lane * P + i > m) ? 0x0000ffffu : 0u) | ((HALF + lane * P + i > m) ? 0xffff0000u : 0u);
    // per-register constants of the insertion chain: jge = row * ge, cf = jge + (go - ge)
    uint32_t jge[P];
#pragma unroll
    for (int i = 0; i < P; i++) jge[i] = pk2((lane * P + i) * ge, (HALF + lane * P + i) * ge);
    const uint32_t gmg2 = pk1(go - ge), ngo2 = pk1(-go), nge2 = pk1(-ge);
    __syncwarp();

    int32_t best = 0; uint32_t best_node = 0, best_col = 0, best_row = 0; bool have_best = false;
    uint32_t n_steps = 0;
    uint32_t tb_cols = 0;
    uint8_t* const tb = ws.tb;

    for (uint32_t ni = 0, base_off = 0; ni < hd.n_nodes; base_off += nodes[ni].len, ni++) {
        const TileNode tn = nodes[ni];
        uint32_t Hp[P], Ep[P];
        int run_max; uint32_t depth;
        if (tn.parent == 0xffffu) {
            // virtual column before the root: H0[0] = 0, H0[j] = -(go + (j-1) ge) for j <= max_gap
#pragma unroll
            for (int i = 0; i < P; i++) {
                const int jl = lane * P + i, jh = HALF + lane * P + i;
                const int hl = jl == 0 ? 0 : ((jl <= m && (uint32_t)jl <= hd.max_gap) ? -(go + (jl - 1) * ge) : NEG16);
                const int hh = (jh <= m && (uint32_t)jh <= hd.max_gap) ? -(go + (jh - 1) * ge) : NEG16;
                Hp[i] = pk2(hl, hh); Ep[i] = NEG16x2;
            }
            run_max = 0; depth = 0;
        } else {
            if (!ws.node_live[tn.parent]) { if (lane == 0) ws.node_live[ni] = 0; __syncwarp(); continue; }
            depth = (uint32_t)ws.node_depth[tn.parent] + 1u;
            const uint32_t* pc = ws.cols + (size_t)(depth - 1) * 2 * 32 * 8;
#pragma unroll
            for (int i = 0; i < P; i++) { Hp[i] = pc[i * 32 + lane]; Ep[i] = pc[(8 + i) * 32 + lane]; }
            run_max = ws.node_lin[tn.parent];
        }
        if (lane == 0) { ws.node_col[ni] = tb_cols; ws.node_depth[ni] = (uint16_t)depth; }
        // best cell of the node: the first column whose maximum beats every earlier column of the node, kept as a snapshot
        uint32_t snap[P]; int node_best = NEG16; uint32_t node_best_col = 0;
#pragma unroll
        for (int i = 0; i < P; i++) snap[i] = NEG16x2;
        // diagonal feed of the first register: previous lane's last register (rows wrap from the low half into the high half)
        uint32_t up = __shfl_sync(FULL, Hp[P - 1], (lane + 31) & 31);
        if (lane == 0) up = (up << 16) | 0xC000u;
        int col_max_prev = 0x7fffffff;            // maximum of the previous column (pending fold into run_max)
        bool alive_prev = true;
        uint32_t c = 0;
        for (; c < tn.len; c++) {
            // fold the previous column's maximum into the lineage maximum (the X-drop looks at EARLIER columns only)
            if (col_max_prev != 0x7fffffff) {
                if (col_max_prev > node_best) {   // Hp still holds that column
                    node_best = col_max_prev; node_best_col = c - 1;
#pragma unroll
                    for (int i = 0; i < P; i++) snap[i] = Hp[i];
                }
                if (col_max_prev > run_max) run_max = col_max_prev;
                alive_prev = col_max_prev > ALIVE_FLOOR;
            }
            if (!alive_prev) break;               // a dead column stays dead: nothing below it can score
            const uint8_t rbase = bases[base_off + c];
            const uint32_t bcode = rbase == 'A' ? 0u : (rbase == 'C' ? 1u : (rbase == 'G' ? 2u : (rbase == 'T' ? 3u : 4u)));
            const uint32_t* pr = prof + bcode * 32 * P + lane * P;
            uint32_t s[P];
#pragma unroll
            for (int i = 0; i < P; i++) s[i] = pr[i];
            uint32_t e[P], d[P], hp[P], ex[P], h[P], f[P], t1[P];
            uint32_t run = NEG16x2;
#pragma unroll
            for (int i = 0; i < P; i++) {
                t1[i] = __vadd2(Hp[i], ngo2);                                   // open a deletion
                e[i] = __viaddmax_s16x2(Ep[i], nge2, t1[i]);                    // max(E - ge, H - go)
                d[i] = __vadd2(i == 0 ? up : Hp[i - 1], s[i]);
                hp[i] = __vmaxs2(d[i], e[i]);
                ex[i] = run;                                                    // best H' + row ge among the lane's earlier rows
                run = __viaddmax_s16x2(hp[i], jge[i], run);
            }
            // one max-scan over the lanes (both halves at once), the low half's total feeds the high half
            uint32_t incl = run;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl = __vmaxs2(incl, t); }
            uint32_t excl = __shfl_up_sync(FULL, incl, 1);
            const uint32_t tot = __shfl_sync(FULL, incl, 31);
            if (lane == 0) excl = NEG16x2;
            excl = __vmaxs2(excl, (tot << 16) | 0xC000u);
            const int thr = max(run_max - xt, ALIVE_FLOOR);
            const uint32_t thr2 = pk1(thr);
            uint32_t cm = NEG16x2;
#pragma unroll
            for (int i = 0; i < P; i++) {
                f[i] = __vsub2(__vsub2(__vmaxs2(ex[i], excl), jge[i]), gmg2);   // F = best - go - (row - 1) ge
                h[i] = __vmaxs2(hp[i], f[i]);
            }
            // X-drop + rows beyond the query: dead cells become NEG16 (H and E)
#pragma unroll
            for (int i = 0; i < P; i++) {
                const uint32_t dead = sign_mask2(__vsub2(h[i], thr2)) | inval[i];
                Hp[i] = (h[i] & ~dead) | (NEG16x2 & dead);
                Ep[i] = (e[i] & ~dead) | (NEG16x2 & dead);
                cm = __vmaxs2(cm, Hp[i]);
            }
#ifdef GB_TILE_DEBUG
#pragma unroll
            for (int i = 0; i < P; i++) if (lo16(Hp[i]) > 12000 || hi16(Hp[i]) > 12000)
                printf("BIG c=%u lane=%d i=%d Hp=%08x h=%08x hp=%08x d=%08x e=%08x f=%08x ex=%08x excl=%08x jge=%08x s=%08x t1=%08x up=%08x thr=%d run_max=%d\n", c, lane, i, Hp[i], h[i], hp[i], d[i], e[i], f[i], ex[i], excl, jge[i], s[i], t1[i], up, thr, run_max);
#endif
            up = __shfl_sync(FULL, Hp[P - 1], (lane + 31) & 31);
            if (lane == 0) up = (up << 16) | 0xC000u;
            // traceback flags from sign bits (no packed compares): per cell
            //   bit 0: d < h (not a diagonal step)   bit 1: e < h (not a deletion)
            //   bit 2: H'(col-1) - go < e (deletion extended)   bit 3: H(row-1) - go < f (insertion extended)
            uint32_t tbw[(P + 3) / 4];
#pragma unroll
            for (int i = 0; i < (P + 3) / 4; i++) tbw[i] = 0;
#pragma unroll
            for (int i = 0; i < P; i++) {
                const uint32_t a = __vsub2(d[i], h[i]), b = __vsub2(e[i], h[i]), cx = __vsub2(t1[i], e[i]);
                const uint32_t hm1 = i == 0 ? up : Hp[i - 1];
                const uint32_t dx = __vsub2(__vadd2(hm1, ngo2), f[i]);
                uint32_t t = ((a >> 3) & 0x10001000u) | ((b >> 2) & 0x20002000u) | ((cx >> 1) & 0x40004000u) | (dx & 0x80008000u);
                t = (t | (t >> 20)) & 0x0000ff00u;                 // byte 1: low-half cell in bits 12-15, high-half cell in bits 8-11
                tbw[i / 4] |= (t >> 8) << (8 * (i % 4));
            }
            // one store per lane and column: P bytes (padded to TBS) at tb[(col * 32 + lane) * TBS]
            {
                uint8_t* dst = tb + ((size_t)(tb_cols + c) * 32 + lane) * TBS;
                if constexpr (TBS == 1) *dst = (uint8_t)tbw[0];
                else if constexpr (TBS == 2) *reinterpret_cast<uint16_t*>(dst) = (uint16_t)tbw[0];
                else if constexpr (TBS == 4) *reinterpret_cast<uint32_t*>(dst) = tbw[0];
                else *reinterpret_cast<uint2*>(dst) = make_uint2(tbw[0], tbw[1]);
            }
            col_max_prev = __reduce_max_sync(FULL, max(lo16(cm), hi16(cm)));
        }
        cells += (uint64_t)c * (uint64_t)(m + 1);
        if (col_max_prev != 0x7fffffff) {
            if (col_max_prev > node_best) {
                node_best = col_max_prev; node_best_col = c - 1;
#pragma unroll
                for (int i = 0; i < P; i++) snap[i] = Hp[i];
            }
            if (col_max_prev > run_max) run_max = col_max_prev;
            alive_prev = col_max_prev > ALIVE_FLOOR;
        }
        // node maximum: highest score, then first column (the snapshot), then smallest row (rows live in (lane, register, half))
        if (node_best > best) {
            uint32_t key = 0xffffffffu;
#pragma unroll
            for (int i = 0; i < P; i++) {
                if (lo16(snap[i]) == node_best) key = min(key, (uint32_t)(lane * P + i));
                if (hi16(snap[i]) == node_best) key = min(key, (uint32_t)(HALF + lane * P + i));
            }
            key = __reduce_min_sync(FULL, key);
            best = node_best; best_node = ni; best_col = node_best_col; best_row = key; have_best = true;
        }
        // the node's last column for its children
        const bool live = alive_prev && c == tn.len;
        if (live) {
            uint32_t* pc = ws.cols + (size_t)depth * 2 * 32 * 8;
#pragma unroll
            for (int i = 0; i < P; i++) { pc[i * 32 + lane] = Hp[i]; pc[(8 + i) * 32 + lane] = Ep[i]; }
        }
        if (lane == 0) { ws.node_live[ni] = live ? 1 : 0; ws.node_lin[ni] = run_max; }
        tb_cols += tn.len;
        __syncwarp();
    }
    cells_out = cells;

#ifdef GB_TILE_DEBUG
    if (lane == 0) printf("tile dp: m=%d nodes=%u bases=%u gap=%u best=%d have=%d node=%u col=%u row=%u cells=%llu\n", m, hd.n_nodes, hd.n_bases, hd.max_gap, best, (int)have_best, best_node, best_col, best_row, (unsigned long long)cells);
#endif
    // ---- result path in tree space: mappings (node = tree index), edits -----------------------------------------------
    // The traceback walks from the best cell to the pin, so mappings and edits come out last to first: they are written
    // from the back of the result scratch (map_base / edit_base say where the path starts).  Merging rules of
    // calculate_and_save_alignment (dozeu_interface.cpp:493-533): one mapping per run of steps on a node, matches /
    // insertions / deletions merged into runs, one edit per mismatch, the unaligned query suffix as a trailing insertion.
    map_base_out = 0; edit_base_out = 0;
    if (!have_best || best <= 0) {
        // full-length insertion on the head node (dozeu_interface.cpp:344-360)
        if (lane == 0) { gb_mapping mp; mp.node = 0; mp.offset = 0; mp.n_edits = 1; out_maps[0] = mp; out_edits[0] = edit_word(GB_EDIT_INS, (uint32_t)m, 0); }
        __syncwarp();
        n_maps_out = 1; n_edits_out = 1;
        return 0;
    }
    uint32_t em = TILE_MAP_CAP, ee = TILE_EDIT_CAP;
    uint32_t cur_node = best_node, cur_edits = 0, run_op = 0xffu, run_len = 0;
    bool ovf = false;
    auto emit_edit = [&](uint32_t word) { if (ee == 0) { ovf = true; return; } ee--; if (lane == 0) out_edits[ee] = word; cur_edits++; };
    auto flush_run = [&]() {
        if (run_len) emit_edit(edit_word(run_op == 0 ? GB_EDIT_MATCH : (run_op == 2 ? GB_EDIT_INS : GB_EDIT_DEL), run_len, 0));
        run_len = 0; run_op = 0xffu;
    };
    auto close_mapping = [&]() {
        flush_run();
        if (em == 0) { ovf = true; return; }
        em--;
        if (lane == 0) { gb_mapping mp; mp.node = cur_node; mp.offset = 0; mp.n_edits = (uint16_t)cur_edits; out_maps[em] = mp; }
        cur_edits = 0;
    };
    // op: 0 M, 1 X, 2 I, 3 D; qidx: query base of an X
    auto step = [&](uint32_t node, uint32_t op, uint32_t qidx) {
        if (node != cur_node) { close_mapping(); cur_node = node; }
        if (op == 1u) { flush_run(); emit_edit(edit_word(GB_EDIT_SUB, 1, base2(q[qidx]))); }
        else if (op == run_op) run_len++;
        else { flush_run(); run_op = op; run_len = 1; }
        n_steps++;
    };
    if (best_row < (uint32_t)m) emit_edit(edit_word(GB_EDIT_INS, (uint32_t)m - best_row, 0));     // query past the best cell: soft clip
    {
        uint32_t node = best_node, col = best_col, j = best_row;
        int state = 0;   // 0 H, 1 E, 2 F
        bool at_virtual = false;
        uint32_t node_base = 0;                    // offset of the node's bases
        for (uint32_t x = 0; x < node; x++) node_base += nodes[x].len;
        // flags of up to 32 cells down the diagonal from (pf_col, pf_j) of node pf_node, one per lane (one L2 round trip
        // serves a whole run of matches instead of one per step)
        uint32_t pf_node = 0xffffffffu, pf_col = 0, pf_j = 0, pf_byte = 0;
        while (!ovf) {
            if (at_virtual) {
                for (; j > 0; j--) {                                 // leading insertion in the virtual column, on the root
                    if (n_steps >= TILE_STEP_CAP) TILE_FAIL(6);      // the same step count as the int32 sweep's TAIL_STEP_CAP
                    step(0, 2u, 0);
                }
                break;
            }
            const TileNode tn = nodes[node];
            uint32_t byte;
            {
                const uint32_t k = pf_col - col;
                if (node == pf_node && col <= pf_col && k < 32u && pf_j - j == k) byte = __shfl_sync(FULL, pf_byte, k);
                else {
                    pf_node = node; pf_col = col; pf_j = j;
                    pf_byte = 0;
                    if ((uint32_t)lane <= col && (uint32_t)lane <= j) {
                        const uint32_t jl = j - lane, hl = jl >= (uint32_t)HALF ? 1u : 0u, jj = jl - hl * HALF;
                        pf_byte = tb[((size_t)(ws.node_col[node] + col - lane) * 32 + jj / P) * TBS + jj % P];
                    }
                    byte = __shfl_sync(FULL, pf_byte, 0);
                }
            }
            const uint32_t nib = j >= (uint32_t)HALF ? (byte & 15u) : (byte >> 4);
            uint32_t pnode = node, pcol = 0, pbase = node_base; bool p_virtual = false;
            if (col > 0) pcol = col - 1;
            else if (tn.parent == 0xffffu) p_virtual = true;
            else { pnode = tn.parent; pcol = nodes[pnode].len - 1; pbase = 0; for (uint32_t x = 0; x < pnode; x++) pbase += nodes[x].len; }
            if (n_steps >= TILE_STEP_CAP) TILE_FAIL(2);
            if (state == 0) {
                if (!(nib & 1u)) {                                   // diagonal
                    if (j == 0) TILE_FAIL(3);      // never walk off the matrix
                    const uint8_t qc = q[j - 1], r = bases[node_base + col];
                    step(node, (qc == r) ? 0u : 1u, j - 1);
                    j--; node = pnode; col = pcol; node_base = pbase; at_virtual = p_virtual;
                    if (at_virtual && j == 0) break;
                    continue;
                }
                state = !(nib & 2u) ? 1 : 2;
                continue;
            }
            if (state == 1) {
                step(node, 3u, 0);
                const bool open = !(nib & 4u);
                node = pnode; col = pcol; node_base = pbase; at_virtual = p_virtual;
                state = open ? 0 : 1;
                if (at_virtual && j == 0 && state == 0) break;
                continue;
            }
            step(node, 2u, 0);
            const bool open = !(nib & 8u);
            if (j == 0) TILE_FAIL(4);
            j--;
            state = open ? 0 : 2;
        }
    }
    close_mapping();
    __syncwarp();
    if (ovf) TILE_FAIL(5);
    map_base_out = em; edit_base_out = ee;
    n_maps_out = TILE_MAP_CAP - em; n_edits_out = TILE_EDIT_CAP - ee;
    return best;
}

// -----------------------------------------------------------------------------------------------------------------
// The kernel: persistent warps, each pulling tile indices of ONE size class from a device work list.
// -----------------------------------------------------------------------------------------------------------------
struct TileBatch {
    const uint8_t* tiles;            // tile pool
    const uint32_t* tile_off;        // [n_tiles] byte offset / 16 of each tile
    const uint32_t* list;            // tile indices of this class
    const uint32_t* list_count;      // device count (clamped to list_cap)
    uint32_t list_cap;
    uint32_t* work_counter;
    TileResult* results;             // [n_tiles]
    uint32_t* path_pool; uint32_t path_cap; uint32_t* path_cursor;     // result paths (32-bit words)
    uint8_t* ws_base; size_t ws_stride;
};

// smem per warp: 2 tile buffers + profile [5][32 P] words + result scratch + 2 mbarriers
template <int R> __host__ __device__ constexpr size_t tile_smem_per_warp() {
    return 2 * (size_t)TILE_SMEM_BYTES + 5 * 32 * (R / 2) * 4 + TILE_MAP_CAP * 8 + TILE_EDIT_CAP * 4 + 16;
}

template <int R>
__global__ void __launch_bounds__(TILE_WARPS * 32, 1)
xdrop_tile_kernel(DevScores sc, TileBatch b) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* my = smem + (size_t)warp * tile_smem_per_warp<R>();
    uint8_t* buf[2] = {my, my + TILE_SMEM_BYTES};
    uint32_t* prof = reinterpret_cast<uint32_t*>(my + 2 * TILE_SMEM_BYTES);
    gb_mapping* smaps_all = reinterpret_cast<gb_mapping*>(prof + 5 * 32 * (R / 2));
    uint32_t* sedits_all = reinterpret_cast<uint32_t*>(smaps_all + TILE_MAP_CAP);
    uint64_t* bar = reinterpret_cast<uint64_t*>(sedits_all + TILE_EDIT_CAP);
    const TileWs ws = carve_tile_ws(b.ws_base + (size_t)(blockIdx.x * TILE_WARPS + warp) * b.ws_stride);
    const uint32_t n = min(*b.list_count, b.list_cap);
    if (lane == 0) { mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();

    // claim + stage: returns the claimed list position (or >= n)
    auto claim = [&]() -> uint32_t { uint32_t p = 0; if (lane == 0) p = atomicAdd(b.work_counter, 1u); return __shfl_sync(FULL, p, 0); };
    auto tile_ptr = [&](uint32_t pos) -> const uint8_t* { return b.tiles + (size_t)b.tile_off[b.list[pos]] * 16; };
    auto stage = [&](uint32_t pos, int which) -> bool {          // true: staged into shared memory (wait on the barrier)
        const uint8_t* src = tile_ptr(pos);
        const uint32_t bytes = reinterpret_cast<const TileHeader*>(src)->bytes;
        if (bytes > TILE_SMEM_BYTES) return false;
        if (lane == 0) { fence_proxy_async(); mbar_expect_tx(&bar[which], bytes); bulk_copy_g2s(buf[which], src, bytes, &bar[which]); }
        return true;
    };
    uint32_t phase[2] = {0, 0};
    uint32_t cur = claim();
    bool cur_staged = cur < n ? stage(cur, 0) : false;
    int which = 0;
    while (cur < n) {
        const uint32_t nxt = claim();
        __syncwarp();                                             // everyone is done reading the other buffer
        const bool nxt_staged = nxt < n ? stage(nxt, which ^ 1) : false;
        const uint8_t* tile = tile_ptr(cur);
        if (cur_staged) { mbar_wait(&bar[which], phase[which]); phase[which] ^= 1u; tile = buf[which]; }
        const uint32_t ti = b.list[cur];
        if (b.results[ti].status == GB_TILE_ST_CANCELLED) { __syncwarp(); cur = nxt; cur_staged = nxt_staged; which ^= 1; continue; }
        uint32_t nm = 0, ne = 0, mb = 0, eb = 0, st = GB_TILE_ST_OK; uint64_t cells = 0;
        const int32_t score = xdrop_tile_dp<R>(sc, tile, ws, prof, smaps_all, sedits_all, nm, ne, mb, eb, st, cells);
        const gb_mapping* smaps = smaps_all + mb; const uint32_t* sedits = sedits_all + eb;
        __syncwarp();
        // ---- result: translate to graph space, write to the result pool ------------------------------------------------
        const TileHeader hd = *reinterpret_cast<const TileHeader*>(tile);
        const TileNode* nodes = reinterpret_cast<const TileNode*>(tile + 32);
        TileResult res; res.score = score; res.status = st; res.n_maps = nm; res.n_edits = ne; res.path_off = 0;
        res.cells_lo = (uint32_t)cells; res.cells_hi = (uint32_t)(cells >> 32); res.pad = 0;
        if (st == GB_TILE_ST_OK) {
            uint32_t off = 0;
            if (lane == 0) {
                off = atomicAdd(b.path_cursor, 2 * nm + ne);
                if (off > b.path_cap || 2 * nm + ne > b.path_cap - off) off = 0xffffffffu;
            }
            off = __shfl_sync(FULL, off, 0);
            if (off == 0xffffffffu) res.status = GB_TILE_ST_FULL;
            else {
                res.path_off = off;
                gb_mapping* gm = reinterpret_cast<gb_mapping*>(b.path_pool + off);
                uint32_t* gedits = b.path_pool + off + 2 * nm;
                if (lane == 0) {
                    if (hd.flags & GB_TILE_TREE_SPACE) {
                        for (uint32_t i = 0; i < nm; i++) gm[i] = smaps[i];
                        for (uint32_t i = 0; i < ne; i++) gedits[i] = sedits[i];
                    } else if (!(hd.flags & GB_TILE_LEFT)) {
                        // translate_down (tree_subgraph.cpp:172-195)
                        for (uint32_t i = 0; i < nm; i++) {
                            gb_mapping mp = smaps[i];
                            const uint32_t tnode = mp.node;
                            if (tnode == 0 && hd.root_trim != 0) mp.offset = (uint16_t)(mp.offset + hd.root_trim);
                            mp.node = nodes[tnode].node;
                            gm[i] = mp;
                        }
                        for (uint32_t i = 0; i < ne; i++) gedits[i] = sedits[i];
                    } else {
                        // reverse_complement_path (path.cpp:1791-1882) then translate_down
                        uint32_t se_end = ne, w = 0;
                        for (int64_t i = (int64_t)nm - 1; i >= 0; i--) {
                            const gb_mapping mp = smaps[i];
                            const uint32_t se_begin = se_end - mp.n_edits;
                            uint32_t used = 0;
                            for (uint32_t x = se_begin; x < se_end; x++) { const uint32_t wd = sedits[x]; const uint32_t op = wd & 3u; if (op != GB_EDIT_INS) used += (op == GB_EDIT_SUB) ? 1u : (wd >> 4); }
                            gb_mapping o; o.node = nodes[mp.node].node ^ 1u; o.offset = (uint16_t)(nodes[mp.node].len - used - mp.offset); o.n_edits = mp.n_edits;
                            gm[nm - 1 - (uint32_t)i] = o;
                            for (int64_t x = (int64_t)se_end - 1; x >= (int64_t)se_begin; x--) {
                                uint32_t wd = sedits[x];
                                if ((wd & 3u) == GB_EDIT_SUB) wd = (wd & ~0xCu) | ((3u - ((wd >> 2) & 3u)) << 2);   // complement the base
                                gedits[w++] = wd;
                            }
                            se_end = se_begin;
                        }
                    }
                }
            }
        }
        if (lane == 0) b.results[ti] = res;
        __syncwarp();
        cur = nxt; cur_staged = nxt_staged; which ^= 1;
    }
}

// ---- the plan: which tails of which reads have tiles -----------------------------------------------------------------
// The planning kernel (tail_plan_kernel, map.cu) walks the slow units' extension sets the way align_sets will, builds the
// haplotype forest of every tail that can be asked for and leaves one entry per tail: the key (work item, extension, side)
// and the run of tile indices of its trees (tile_off 0xffffffff: tree refused by max_dozeu_cells).  align_tail looks the
// tail up; a tail without an entry (plan capacity, tile budgets, scores outside int16) is aligned in place by the int32
// sweep, so the plan only ever decides where a DP runs, never what it returns.
constexpr uint32_t PLAN_PER_UNIT = 32;
constexpr uint32_t TILE_REFUSED = 0xffffffffu;
struct TailPlanEntry { uint32_t key, first_tile, n_trees, wave; };     // wave 1: its tiles wait for tail_decide_kernel
__device__ __forceinline__ uint32_t tail_key(uint32_t item_local, uint32_t read_num, uint32_t ext, bool left) { return (read_num << 30) | (item_local << 9) | (ext << 1) | (left ? 1u : 0u); }
struct PlanView {
    const TailPlanEntry* entries;      // [n_units * PLAN_PER_UNIT], unit = position in the slow list
    const uint32_t* unit_base;         // [n_units] first entry of a unit (indexed by read / pair number), 0xffffffff: not planned
    const uint32_t* unit_count;        // [n_units]
    const uint32_t* tile_off;
    const TileResult* results;
    const uint32_t* path_pool;
    uint64_t* stats;                   // plan counters (gb_plan_stats); [2] counts tails of planned units that were aligned in place
};
struct TailLookup { const PlanView* pv; uint32_t base, count, key; };     // pv == nullptr: no plan (always in place)

// Runs xdrop_tile_kernel over one wave of tiles: one launch per size class c over lists[c * list_cap ..], with its list
// count at list_count[c] and its work counter at work[c] (map.cu, the only file that instantiates the kernel).
int launch_tile_kernels(gb_device* d, const uint8_t* tiles, const uint32_t* tile_off, const uint32_t* lists, size_t list_cap,
                        const uint32_t* list_count, uint32_t* work, TileResult* results, uint32_t* paths, uint32_t path_cap, uint32_t* path_cursor);

} // namespace gb
