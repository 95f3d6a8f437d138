// map_paired.cuh — paired-end kernels (included by map.cu inside namespace gb).
//   MinimizerMapper::map_paired, minimizer_mapper.cpp:1462-2942, forced fragment distribution.  With
//   max_rescue_attempts != 0, pairs left with unpaired alignments go to the rescue build of align_kernel_pe
//   (rescue.cuh, SURVEY.md §8 a17).
#pragma once

// Mate 2 is mapped "rightward": reverse-complemented sequence, reversed qualities (:1503-1506).
__global__ void prep_pairs_kernel(const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off, uint32_t n_reads,
                                  uint8_t* w_reads, uint8_t* w_quals) {
    const uint32_t warps_per_block = blockDim.x >> 5;
    const uint32_t lane = threadIdx.x & 31;
#pragma unroll 1
    for (uint32_t r = blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < n_reads; r += gridDim.x * warps_per_block) {
        const uint64_t b = read_off[r]; const uint32_t L = (uint32_t)(read_off[r + 1] - b);
        if ((r & 1u) == 0) {
#pragma unroll 1
            for (uint32_t i = lane; i < L; i += 32) { w_reads[b + i] = reads[b + i]; if (quals) w_quals[b + i] = quals[b + i]; }
        } else {
#pragma unroll 1
            for (uint32_t i = lane; i < L; i += 32) {
                w_reads[b + i] = comp_base(reads[b + L - 1 - i]);
                if (quals) w_quals[b + i] = quals[b + L - 1 - i];
            }
        }
    }
}

struct PairBatch {
    PairState* pairs;
    int32_t fragment_limit;
};

// The warps of a block take SEED_WARPS consecutive pairs per round and meet at a block barrier
// between phases: the kernel's code is far larger than the instruction caches, and warps that
// drift apart each stream it from L2 on their own (ncu: "no instruction" was the top stall).
// LC / MC / CC != 0 fix the shared-memory layout at compile time (the usual launch: 150 bp reads, first-pass tables), so the
// twenty table pointers are immediates on one base register instead of being rebuilt from (Lc, Mc, Cc) at every use (the
// 64-register budget cannot hold them; ncu attributed 8 % of the kernel's instructions to that arithmetic).
template <int LC, int MC, int CC>
__global__ void __launch_bounds__(SEED_WARPS * 32, SEED_BLOCKS_PER_SM)
seed_kernel_pe(DevIndex ix, MapParamsDev P, MapBatch b, SeedPools pools, PairBatch pb) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ uint32_t s_base;
    // The two reads' states live from phase A to the end of the round: in registers they would take 32 of the 64.
    __shared__ ReadState s_rs[SEED_WARPS][2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    ReadState& rs0 = s_rs[warp][0];
    ReadState& rs1 = s_rs[warp][1];
    const uint32_t lay_L = LC ? (uint32_t)LC : b.Lc, lay_M = MC ? (uint32_t)MC : b.Mc, lay_C = CC ? (uint32_t)CC : b.Cc;
    const SeedSmem sm = carve_seed_smem(smem + (size_t)warp * seed_smem_bytes(lay_L, lay_M, lay_C), lay_L, lay_M, lay_C, b.Ns);
    const uint32_t n_pairs = b.n_reads / 2;
    const uint32_t limit = b.in_list ? min(*b.in_count, n_pairs) : n_pairs;
#pragma unroll 1
    while (true) {
        __syncthreads();
        if (threadIdx.x == 0) s_base = atomicAdd(b.work_counter, blockDim.x >> 5);
        __syncthreads();
        const uint32_t base = s_base;
        if (base >= limit) break;
        const bool active = base + warp < limit;
        const uint32_t p = !active ? 0u : (b.in_list ? b.in_list[base + warp] : base + warp);
        if (lane < 2 * sizeof(ReadState) / 4) reinterpret_cast<uint32_t*>(s_rs[warp])[lane] = 0;
        __syncwarp();
        uint32_t n_fragments = 0;
        uint32_t status = GB_ITEM_OK;
        // read offsets and lengths are loaded again where they are used (L1 hits) rather than held through the phases
        auto read_len = [&](uint32_t r) { return (uint32_t)(b.read_off[2 * p + r + 1] - b.read_off[2 * p + r]); };
        DevRng rng; rng.inited = 0; rng.state = 0; rng.seed = 0;
        if (active) {
            const uint64_t rb0 = b.read_off[2 * p], rb1 = b.read_off[2 * p + 1];
            const uint32_t L0 = (uint32_t)(rb1 - rb0), L1 = (uint32_t)(b.read_off[2 * p + 2] - rb1);
            if (L0 > b.Lc || L1 > b.Lc) status = GB_ITEM_OUT_FULL;
            // LazyRNG seed: aln1.sequence() + aln2.sequence() with mate 2 already rightward (:1529-1531)
            else rng.seed = fold_seed(fold_seed(0u, b.reads + rb0, L0), b.reads + rb1, L1);
        }
        const bool work = active && status == GB_ITEM_OK;
#pragma unroll 1
        for (uint32_t r = 0; r < 2; r++) {
            __syncthreads();
            if (work && status == GB_ITEM_OK) {
                const uint32_t Lr = read_len(r);
                stage_read(sm.read, b.reads + b.read_off[2 * p + r], Lr);
                __syncwarp();
                status = seed_phase_a(ix, P, sm, Lr, pools, rng, s_rs[warp][r]);
                __syncwarp();
            }
        }
        __syncthreads();
        if (work && status == GB_ITEM_OK)
            status = cluster_phase_pe(ix, P, sm, read_len(0), read_len(1), 2 * p, pb.fragment_limit, pools, rng, rs0, rs1, pb.pairs + p, n_fragments);
        if (!active) continue;
        if (status == GB_ITEM_RETRY) {
            if (lane == 0) b.retry_list[atomicAdd(b.retry_count, 1u)] = p;
            continue;
        }
        if (lane == 0) {
            rs0.rng = rng; rs1.rng = rng;
            rs0.status = rs1.status = status;
            if (status != GB_ITEM_OK) { rs0.item_cnt = rs1.item_cnt = 0; }
            b.states[2 * p] = rs0; b.states[2 * p + 1] = rs1;
            // cluster_phase_pe fills the record when the pair has clusters
            if (status != GB_ITEM_OK || n_fragments == 0) { pb.pairs[p].n_fragments = 0; pb.pairs[p].found_paired_cluster = 0; }
        }
    }
}

template <bool RESCUE>
__global__ void __launch_bounds__(ALIGN_WARPS * 32, RESCUE ? 2 : 4)
align_kernel_pe(DevIndex ix, MapParamsDev P, DevScores sc, MapBatch b, AlignArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t gwarp = blockIdx.x * ALIGN_WARPS + warp;
    const AlignSmem sm = align_smem_carve(smem, warp, b.Lc, 2, a.tmp_bytes);
    uint8_t* sread[2] = {sm.read[0], sm.read[1]};
    uint8_t* squal[2] = {sm.qual[0], sm.qual[1]};
    uint8_t* qbuf = sm.qbuf; uint8_t* stmp = sm.tmp;
    const DpSmem dps = sm.dps;
    const TailWs ws = carve_tail_ws(a.ws_base + (size_t)gwarp * a.ws_stride, b.Lc, a.tb_cells);
    uint8_t* cand_base = a.cand_base + (size_t)gwarp * a.cand_stride;
    const uint32_t n_pairs = b.n_reads / 2;

#pragma unroll 1
    while (true) {
        uint32_t p = 0;
        if (lane == 0) {
            p = atomicAdd(b.work_counter, 1u);
            if (a.slow_list) p = p < *a.slow_count ? a.slow_list[p] : 0xffffffffu;
        }
        p = __shfl_sync(FULL, p, 0);
        if (p >= n_pairs) break;
        ReadState rs[2] = {b.states[2 * p], b.states[2 * p + 1]};
        const PairState ps = a.pairs[p];
        uint32_t status = rs[0].status;
        gb_alignment out[2];
        memset(&out[0], 0, sizeof(gb_alignment)); memset(&out[1], 0, sizeof(gb_alignment));
        uint32_t L[2];
        gb_mapping* out_maps[2]; uint32_t* out_edits[2];
#pragma unroll 1
        for (uint32_t r = 0; r < 2; r++) {
            const uint32_t ri = 2 * p + r;
            L[r] = (uint32_t)(b.read_off[ri + 1] - b.read_off[ri]);
            out_maps[r] = a.maps + (size_t)ri * P.mapping_cap; out_edits[r] = a.edits + (size_t)ri * P.edit_cap;
            out[r].read_id = ri; out[r].flags = GB_ALN_PAIRED;
        }
        if (status == GB_ITEM_OK) {
#pragma unroll 1
            for (uint32_t r = 0; r < 2; r++) {
                const uint64_t rb = b.read_off[2 * p + r];
#pragma unroll 1
                for (uint32_t i = lane; i < L[r]; i += 32) { sread[r][i] = b.reads[rb + i]; if (b.quals) squal[r][i] = b.quals[rb + i]; }
            }
            __syncwarp();
            DevRng rng = rs[0].rng;
            bool slot_used[N_SLOTS];
#pragma unroll 1
            for (uint32_t i = 0; i < N_SLOTS; i++) slot_used[i] = false;
            CandList cl; cl.n = 0;
            uint32_t explored[2][PRESENT_WORDS];
#pragma unroll 1
            for (uint32_t r = 0; r < 2 && status == GB_ITEM_OK; r++)          // one copy of align_sets per kernel (instruction cache)
                status = align_sets(ix, P, sc, rs[r], a, sread[r], L[r], ws, dps, qbuf, cand_base, slot_used, rng, true, r, cl, explored[r], p, stmp);
            if (status == GB_ITEM_OK) {
                const uint8_t* sr[2] = {sread[0], sread[1]};
                const uint8_t* sq[2] = {b.quals ? squal[0] : nullptr, b.quals ? squal[1] : nullptr};
                if constexpr (RESCUE) {
                    const RescueWs rw = carve_rescue_ws(a.rescue_base + (size_t)gwarp * a.rescue_stride, b.Lc);
                    status = finalize_pe_rescue(ix, P, sc, rs, ps, a, cl, explored, rng, sr, sq, L, 2 * p, dps, qbuf, cand_base, slot_used, rw, b.Lc, out, out_maps, out_edits);
                } else
                    status = finalize_pe(ix, P, rs, ps, a, cl, explored, rng, sr, sq, L, 2 * p, dps, cand_base, out, out_maps, out_edits);
            }
        }
        if (!RESCUE && status == GB_ITEM_RETRY) {
            // unpaired alignments and rescue enabled: hand the pair to the rescue instantiation of this kernel
            if (lane == 0) a.rescue_list[atomicAdd(a.rescue_count, 1u)] = p;
            __syncwarp();
            continue;
        }
#pragma unroll 1
        for (uint32_t r = 0; r < 2; r++) {
            const uint32_t ri = 2 * p + r;
            out[r].mapping_off = ri * P.mapping_cap; out[r].edit_off = ri * P.edit_cap;
            if (status != GB_ITEM_OK) { out[r].score = 0; out[r].flags = GB_ALN_PAIRED; out[r].n_mappings = 0; out[r].n_edits = 0; out[r].mapq = 0; }
            if (lane == 0) { a.aln[ri] = out[r]; a.status[ri] = (uint8_t)status; }
        }
        __syncwarp();
    }
}
