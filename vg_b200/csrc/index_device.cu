// index_device.cu — the minimizer step of the flat-index builder on the GPU (gb_index_from_gbz_device,
// gb_index_build_from_gbwt_device).
//
// The host builder (index_builder.cpp) makes the sequences, the distance payload and the GBWT blob, and places the table;
// this unit only turns those into the sorted, unique (key, position) list the host window enumeration would give:
//   1. window_kernel<false>: one warp per start oriented node follows GBWT search states (node, lo, hi) depth first to every
//      haplotype-consistent continuation of W - 1 = k + w - 2 bases, and counts the minimizers of every string start node +
//      continuation (or of a shorter string where the haplotypes end, when it still holds a whole window);
//   2. the host cuts the start nodes into batches whose pairs fit the pair pool;
//   3. window_kernel<true> redoes each batch and writes the pairs at the counted offsets;
//   4. two stable CUB radix sorts (position, then key) and a flag / scan / scatter drop the duplicates;
//   5. the unique pairs of every batch go back to the host, which merges batches when there is more than one.
// Counting first and filling second enumerates everything twice but needs no retry: a batch can never overflow.
#include <cub/cub.cuh>

#include "device_state.cuh"
#include "index_build.h"
#include "minimizer_common.h"

#include <algorithm>
#include <cstdlib>
#include <string>
#include <vector>

namespace gb {

int device_ready(int device) {
    int ndev = 0;
    const cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        set_last_error("no CUDA device available (libgiraffe_b200 has no CPU fallback)", "");
        return GB_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= ndev) { set_last_error("device ordinal out of range", ""); return GB_ERR_ARG; }
    return GB_OK;
}

namespace {

constexpr int WIN_WARPS = 4;                           // warps per block of window_kernel
constexpr size_t SMEM_PER_BASE = 16;                   // hash 8, node 4, offset 2, base 1, k-mer flags 1
constexpr size_t STACK_BYTES = 256ull << 20;           // all warps' search-state stacks together
constexpr size_t POOL_BYTES = 2ull << 30;              // pair pool of one batch, with its sort buffers
constexpr size_t BYTES_PER_PAIR = 56;                  // key, position, their sort alternates, flag, index, output pair

struct Frame { uint32_t node; int32_t lo, hi; uint32_t len; };      // search state + length of the string before the node

struct WinArgs {
    DevIndex ix;                                        // nodes, seq, gbwt
    uint32_t k, w, lcap;                                // lcap: bases per warp in shared memory (longest node + W - 1)
    const uint32_t* starts; uint32_t first, last;       // start oriented nodes [first, last)
    Frame* stacks; uint32_t stack_cap;
    uint32_t* work; unsigned long long* continuations; uint32_t* stack_overflow;
    uint64_t* counts;                                   // count pass: pairs per start node
    const uint64_t* offsets; uint64_t base;             // fill pass: start node i writes at offsets[i] - base
    uint64_t* out_key; uint64_t* out_pos;
};

__device__ __forceinline__ void kmer_of(const uint8_t* chr, uint32_t s, uint32_t k, uint64_t& fk, uint64_t& rk, bool& valid) {
    fk = 0; rk = 0; valid = true;
    for (uint32_t j = 0; j < k; j++) {
        const uint32_t c = gbmin::base_code(chr[s + j]);
        valid &= c < 4;
        fk = (fk << 2) | (c & 3u);
        rk |= (uint64_t)(3u - (c & 3u)) << (2 * j);
    }
}

// The minimizers of the string chr[0, len) (gbmin::minimizers: a valid k-mer is reported when some window of w k-mers holds
// it and no strictly smaller hash), counted; with FILL also written from out[at] on.  Warp-uniform; returns the count.
template <bool FILL>
__device__ __forceinline__ uint32_t select_minimizers(const WinArgs& a, uint32_t len, const uint64_t* hsh, const uint32_t* bnode,
                                                      const uint16_t* boff, const uint8_t* chr, const uint8_t* flg, uint64_t at) {
    const int lane = threadIdx.x & 31;
    const int k = (int)a.k, w = (int)a.w;
    const int nk = (int)len - k + 1, last_window = (int)len - (int)(a.k + a.w - 1);
    uint32_t n = 0;
    for (int c = 0; c < nk; c += 32) {
        const int s = c + lane;
        bool rep = false;
        if (s < nk && (flg[s] & 1u)) {
            const uint64_t h = hsh[s];
            int lo = max(s - w + 1, 0), hi = min(s, last_window);
            for (int j = s - 1; j >= lo; j--) if ((flg[j] & 1u) && hsh[j] < h) { lo = j + 1; break; }
            const int rmax = min(s + w - 1, nk - 1);
            for (int j = s + 1; j <= rmax; j++) if ((flg[j] & 1u) && hsh[j] < h) { hi = min(hi, j - w); break; }
            rep = lo <= hi;
        }
        const unsigned mask = __ballot_sync(FULL, rep);
        if (FILL && rep) {
            uint64_t fk, rk; bool valid;
            kmer_of(chr, (uint32_t)s, a.k, fk, rk, valid);
            const bool rev = flg[s] & 2u;
            const uint32_t at_base = rev ? (uint32_t)s + a.k - 1 : (uint32_t)s;
            uint32_t v = bnode[at_base], o = boff[at_base];
            if (rev) { o = load_node(a.ix, v).len - 1 - o; v ^= 1u; }
            const uint64_t i = at + n + __popc(mask & ((1u << lane) - 1u));
            a.out_key[i] = rev ? rk : fk;
            a.out_pos[i] = ((uint64_t)v << 10) | o;
        }
        n += __popc(mask);
    }
    return n;
}

template <bool FILL>
__global__ void __launch_bounds__(WIN_WARPS * 32) window_kernel(WinArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint32_t gwarp = blockIdx.x * (blockDim.x >> 5) + wib;
    uint8_t* mine = smem + (size_t)wib * a.lcap * SMEM_PER_BASE;
    uint64_t* hsh = reinterpret_cast<uint64_t*>(mine);                       // hash of the canonical k-mer starting at each base
    uint32_t* bnode = reinterpret_cast<uint32_t*>(mine + 8 * (size_t)a.lcap);  // oriented node of each base
    uint16_t* boff = reinterpret_cast<uint16_t*>(mine + 12 * (size_t)a.lcap);  // its offset in that node
    uint8_t* chr = mine + 14 * (size_t)a.lcap;
    uint8_t* flg = mine + 15 * (size_t)a.lcap;                                 // bit 0: valid k-mer, bit 1: reverse strand
    Frame* stack = a.stacks + (size_t)gwarp * a.stack_cap;
    const uint32_t W = a.k + a.w - 1;
    unsigned long long n_cont = 0;
    while (true) {
        uint32_t i = 0;
        if (lane == 0) i = atomicAdd(a.work, 1u);
        i = __shfl_sync(FULL, i, 0) + a.first;
        if (i >= a.last) break;
        const uint32_t v0 = a.starts[i];
        const gb_node_rec n0 = load_node(a.ix, v0);
        const uint32_t need = n0.len + W - 1;
        const uint64_t at = FILL ? a.offsets[i] - a.base : 0;
        uint64_t found = 0;
        if (lane == 0) stack[0] = Frame{v0, 0, (int32_t)n0.size - 1, 0};
        uint32_t sp = 1;
        __syncwarp();
        while (sp > 0) {
            const Frame f = stack[--sp];
            const gb_node_rec nr = load_node(a.ix, f.node);
            const uint32_t take = min(nr.len, need - f.len), len = f.len + take;
            for (uint32_t o = lane; o < take; o += 32) {
                chr[f.len + o] = a.ix.seq[nr.seq_off + o]; bnode[f.len + o] = f.node; boff[f.len + o] = (uint16_t)o;
            }
            __syncwarp();
            // the k-mers that end on the new bases; those inside the prefix were computed when it was laid down
            for (uint32_t e = max(f.len, a.k - 1) + lane; e < len; e += 32) {
                const uint32_t s = e + 1 - a.k;
                uint64_t fk, rk; bool valid;
                kmer_of(chr, s, a.k, fk, rk, valid);
                const uint64_t hf = gbmin::hash64(fk), hr = gbmin::hash64(rk);
                hsh[s] = hr < hf ? hr : hf;
                flg[s] = valid ? (hr < hf ? 3u : 1u) : 0u;
            }
            __syncwarp();
            bool leaf = len == need;
            if (!leaf) {
                // successors in the GBWT: what the host's `follow` gives, one lane per edge
                uint32_t pushed = 0;
                if (nr.size != 0) {
                    const uint32_t* rec = a.ix.gbwt + nr.rec_off;
                    const uint32_t n_edges = __ldg(rec);
                    if (n_edges <= 32) {
                        const EdgeFan fan = record_fan(a.ix, nr, f.lo, f.hi);
                        const bool ok = (uint32_t)lane < fan.n_edges && fan.to != 0 && fan.cnt > 0;
                        const unsigned mask = __ballot_sync(FULL, ok);
                        pushed = __popc(mask);
                        if (sp + pushed > a.stack_cap) { if (lane == 0) atomicExch(a.stack_overflow, 1u); sp = 0; break; }
                        if (ok) stack[sp + __popc(mask & ((1u << lane) - 1u))] = Frame{fan.to, fan.first, fan.first + fan.cnt - 1, len};
                    } else {
                        const uint32_t n_runs = __ldg(rec + 1);
                        for (uint32_t e = 0; e < n_edges; e++) {
                            int32_t below, cnt;
                            record_edge_query(rec, n_edges, n_runs, f.lo, f.hi, e, below, cnt);
                            const uint32_t to = __ldg(rec + 2 + 2 * e);
                            if (to == 0 || cnt <= 0) continue;
                            if (sp + pushed >= a.stack_cap) { if (lane == 0) atomicExch(a.stack_overflow, 1u); break; }
                            const int32_t first = (int32_t)__ldg(rec + 3 + 2 * e) + below;
                            if (lane == 0) stack[sp + pushed] = Frame{to, first, first + cnt - 1, len};
                            pushed++;
                        }
                    }
                }
                __syncwarp();
                sp += pushed;
                if (pushed == 0) leaf = len >= W;                   // the haplotypes end here: a whole window or nothing
                else continue;
            }
            if (leaf) {
                found += select_minimizers<FILL>(a, len, hsh, bnode, boff, chr, flg, at + found);
                n_cont++;
            }
            __syncwarp();
        }
        if (!FILL && lane == 0) a.counts[i] = found;
    }
    if (!FILL && lane == 0 && n_cont) atomicAdd(a.continuations, n_cont);
}

// flags[i] = pair i differs from pair i - 1 (the input is sorted)
__global__ void mark_unique(const uint64_t* key, const uint64_t* pos, uint64_t n, uint32_t* flags) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        flags[i] = i == 0 || key[i] != key[i - 1] || pos[i] != pos[i - 1];
}

__global__ void gather_unique(const uint64_t* key, const uint64_t* pos, const uint32_t* flags, const uint32_t* idx, uint64_t n, KeyPos* out) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        if (flags[i]) out[idx[i]] = KeyPos{key[i], pos[i]};
}

struct StreamHolder {
    cudaStream_t s = nullptr;
    ~StreamHolder() { if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); } }
};

uint32_t bits_for(uint64_t max_value) { uint32_t b = 0; while (b < 64 && (max_value >> b) != 0) b++; return b; }

} // namespace

int window_pairs_device(int device, const std::vector<gb_node_rec>& nodes, const std::vector<uint8_t>& seq,
                        const std::vector<uint32_t>& gbwt, uint32_t k, uint32_t w, bool forward_only,
                        std::vector<KeyPos>& out, WindowCounts& counts) {
    out.clear();
    counts = WindowCounts{};
    // start nodes, the longest node and the largest start record (a bound on the pending search states of one start node: the
    // states on a warp's stack hold disjoint sets of that node's visits)
    std::vector<uint32_t> starts;
    uint32_t max_len = 1, stack_cap = 1;
    for (uint32_t v = 2; v < (uint32_t)nodes.size(); v++) {
        max_len = std::max(max_len, nodes[v].len);
        if (nodes[v].size == 0 || (forward_only && (v & 1u))) continue;
        if (nodes[v].size > 0x7fffffffu) { set_last_error("gb_index_*_device: a GBWT record of more than 2^31 - 1 visits", ""); return GB_ERR_CAPACITY; }
        starts.push_back(v);
        stack_cap = std::max(stack_cap, nodes[v].size);
    }
    counts.start_nodes = starts.size();
    if (starts.empty()) return GB_OK;

    GB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    GB_CUDA(cudaGetDeviceProperties(&prop, device));
    const uint32_t W = k + w - 1;
    const uint32_t lcap = (max_len + W - 1 + 7) & ~7u;
    const size_t smem_warp = (size_t)lcap * SMEM_PER_BASE;
    const int warps_per_block = (int)std::min<size_t>(WIN_WARPS, prop.sharedMemPerBlockOptin / smem_warp);
    if (warps_per_block < 1) { set_last_error("gb_index_*_device: the longest node + k + w - 2 bases do not fit one warp's shared memory", ""); return GB_ERR_CAPACITY; }
    const size_t smem = smem_warp * warps_per_block;
    GB_CUDA(cudaFuncSetAttribute(window_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    GB_CUDA(cudaFuncSetAttribute(window_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, window_kernel<true>, warps_per_block * 32, smem));
    size_t blocks = (size_t)std::max(per_sm, 1) * prop.multiProcessorCount;
    blocks = std::min(blocks, std::max<size_t>(1, STACK_BYTES / ((size_t)stack_cap * sizeof(Frame) * warps_per_block)));
    blocks = std::min(blocks, (starts.size() + warps_per_block - 1) / warps_per_block);
    // the pair pool: GIRAFFE_B200_INDEX_POOL_PAIRS (test-only) makes it small enough to need several batches on a small graph
    uint64_t pool = POOL_BYTES / BYTES_PER_PAIR;
    if (const char* env = std::getenv("GIRAFFE_B200_INDEX_POOL_PAIRS")) {
        const unsigned long long v = std::strtoull(env, nullptr, 10);
        if (v >= 1 && v < pool) pool = v;
    }

    StreamHolder st;
    GB_CUDA(cudaStreamCreateWithFlags(&st.s, cudaStreamNonBlocking));
    DevBuf<gb_node_rec> d_nodes; DevBuf<uint8_t> d_seq; DevBuf<uint32_t> d_gbwt, d_starts, d_counters;
    DevBuf<Frame> d_stacks; DevBuf<uint64_t> d_counts, d_offsets;
    int rc;
    if ((rc = d_nodes.upload(nodes.data(), nodes.size(), st.s))) return rc;
    if ((rc = d_seq.upload(seq.data(), seq.size(), st.s))) return rc;
    if ((rc = d_gbwt.upload(gbwt.data(), gbwt.size(), st.s))) return rc;
    if ((rc = d_starts.upload(starts.data(), starts.size(), st.s))) return rc;
    if ((rc = d_stacks.reserve(blocks * warps_per_block * (size_t)stack_cap))) return rc;
    if ((rc = d_counts.reserve(starts.size()))) return rc;
    if ((rc = d_offsets.reserve(starts.size()))) return rc;
    if ((rc = d_counters.reserve(4))) return rc;                      // work, stack overflow, continuations (64-bit)
    GB_CUDA(cudaMemsetAsync(d_counters.ptr, 0, 4 * sizeof(uint32_t), st.s));

    WinArgs a{};
    a.ix.nodes = d_nodes.ptr; a.ix.seq = d_seq.ptr; a.ix.gbwt = d_gbwt.ptr; a.ix.n_nodes = (uint32_t)nodes.size(); a.ix.k = k; a.ix.w = w;
    a.k = k; a.w = w; a.lcap = lcap;
    a.starts = d_starts.ptr; a.first = 0; a.last = (uint32_t)starts.size();
    a.stacks = d_stacks.ptr; a.stack_cap = stack_cap;
    a.work = d_counters.ptr; a.stack_overflow = d_counters.ptr + 1;
    a.continuations = reinterpret_cast<unsigned long long*>(d_counters.ptr + 2);
    a.counts = d_counts.ptr; a.offsets = d_offsets.ptr;
    window_kernel<false><<<(unsigned)blocks, warps_per_block * 32, smem, st.s>>>(a);
    GB_CUDA(cudaGetLastError());
    std::vector<uint64_t> h_counts(starts.size());
    uint32_t h_counters[4];
    GB_CUDA(cudaMemcpyAsync(h_counts.data(), d_counts.ptr, h_counts.size() * sizeof(uint64_t), cudaMemcpyDeviceToHost, st.s));
    GB_CUDA(cudaMemcpyAsync(h_counters, d_counters.ptr, sizeof h_counters, cudaMemcpyDeviceToHost, st.s));
    GB_CUDA(cudaStreamSynchronize(st.s));
    if (h_counters[1]) { set_last_error("gb_index_*_device: GBWT search states beyond the visits of their start node (inconsistent records)", ""); return GB_ERR_FORMAT; }
    counts.continuations = (uint64_t)h_counters[2] | ((uint64_t)h_counters[3] << 32);
    std::vector<uint64_t> h_off(starts.size());
    uint64_t total = 0, largest = 0;
    for (size_t i = 0; i < starts.size(); i++) { h_off[i] = total; total += h_counts[i]; largest = std::max(largest, h_counts[i]); }
    counts.raw_pairs = total;
    if (total == 0) return GB_OK;
    if (largest > pool) { set_last_error("gb_index_*_device: one start node has more minimizers than the pair pool holds", ""); return GB_ERR_CAPACITY; }
    if ((rc = d_offsets.upload(h_off.data(), h_off.size(), st.s))) return rc;

    // the pool of one batch and its sort / unique buffers
    const uint64_t cap = std::min<uint64_t>(pool, total);
    DevBuf<uint64_t> key0, pos0, key1, pos1; DevBuf<uint32_t> flags, idx; DevBuf<KeyPos> uniq; DevBuf<uint8_t> tmp;
    if ((rc = key0.reserve(cap)) || (rc = pos0.reserve(cap)) || (rc = key1.reserve(cap)) || (rc = pos1.reserve(cap)) ||
        (rc = flags.reserve(cap)) || (rc = idx.reserve(cap)) || (rc = uniq.reserve(cap))) return rc;
    const int key_bits = (int)(2 * k), pos_bits = (int)(10 + bits_for(nodes.size() - 1));
    size_t sort_bytes = 0, key_sort_bytes = 0, scan_bytes = 0;         // temporaries grow with the bits sorted
    {
        cub::DoubleBuffer<uint64_t> kb(key0.ptr, key1.ptr), pb(pos0.ptr, pos1.ptr);
        GB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, pb, kb, (int)cap, 0, pos_bits, st.s));
        GB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, key_sort_bytes, kb, pb, (int)cap, 0, key_bits, st.s));
        GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, flags.ptr, idx.ptr, (int)cap, st.s));
    }
    sort_bytes = std::max(sort_bytes, key_sort_bytes);
    if ((rc = tmp.reserve(std::max(sort_bytes, scan_bytes)))) return rc;

    std::vector<size_t> run_begin;
    for (size_t b = 0; b < starts.size();) {
        size_t e = b; uint64_t n = 0;
        while (e < starts.size() && n + h_counts[e] <= cap) n += h_counts[e++];
        if (n > 0) {
            a.first = (uint32_t)b; a.last = (uint32_t)e; a.base = h_off[b];
            a.out_key = key0.ptr; a.out_pos = pos0.ptr;
            GB_CUDA(cudaMemsetAsync(d_counters.ptr, 0, sizeof(uint32_t), st.s));
            const size_t fill_blocks = std::min(blocks, (e - b + warps_per_block - 1) / warps_per_block);
            window_kernel<true><<<(unsigned)fill_blocks, warps_per_block * 32, smem, st.s>>>(a);
            GB_CUDA(cudaGetLastError());
            cub::DoubleBuffer<uint64_t> kb(key0.ptr, key1.ptr), pb(pos0.ptr, pos1.ptr);
            size_t bytes = sort_bytes;
            GB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.ptr, bytes, pb, kb, (int)n, 0, pos_bits, st.s));
            bytes = sort_bytes;
            GB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.ptr, bytes, kb, pb, (int)n, 0, key_bits, st.s));
            const unsigned grid = (unsigned)std::min<uint64_t>((n + 255) / 256, 4096);
            mark_unique<<<grid, 256, 0, st.s>>>(kb.Current(), pb.Current(), n, flags.ptr);
            GB_CUDA(cudaGetLastError());
            bytes = scan_bytes;
            GB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.ptr, bytes, flags.ptr, idx.ptr, (int)n, st.s));
            gather_unique<<<grid, 256, 0, st.s>>>(kb.Current(), pb.Current(), flags.ptr, idx.ptr, n, uniq.ptr);
            GB_CUDA(cudaGetLastError());
            uint32_t last_idx = 0, last_flag = 0;
            GB_CUDA(cudaMemcpyAsync(&last_idx, idx.ptr + n - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st.s));
            GB_CUDA(cudaMemcpyAsync(&last_flag, flags.ptr + n - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st.s));
            GB_CUDA(cudaStreamSynchronize(st.s));
            const size_t n_unique = (size_t)last_idx + last_flag;
            run_begin.push_back(out.size());
            out.resize(out.size() + n_unique);
            GB_CUDA(cudaMemcpyAsync(out.data() + run_begin.back(), uniq.ptr, n_unique * sizeof(KeyPos), cudaMemcpyDeviceToHost, st.s));
            GB_CUDA(cudaStreamSynchronize(st.s));
        }
        b = e;
    }
    // several batches: merge their sorted runs pairwise, then drop the pairs two batches share
    if (run_begin.size() > 1) {
        auto less = [](const KeyPos& x, const KeyPos& y) { return x.key != y.key ? x.key < y.key : x.pos < y.pos; };
        run_begin.push_back(out.size());
        while (run_begin.size() > 2) {
            std::vector<size_t> next;
            for (size_t r = 0; r + 2 < run_begin.size(); r += 2) {
                std::inplace_merge(out.begin() + run_begin[r], out.begin() + run_begin[r + 1], out.begin() + run_begin[r + 2], less);
                next.push_back(run_begin[r]);
            }
            if ((run_begin.size() - 1) % 2) next.push_back(run_begin[run_begin.size() - 2]);
            next.push_back(out.size());
            run_begin.swap(next);
        }
        out.erase(std::unique(out.begin(), out.end(), [](const KeyPos& x, const KeyPos& y) { return x.key == y.key && x.pos == y.pos; }), out.end());
    }
    return GB_OK;
}

} // namespace gb
