// bgzf_device.cu — gb_bgzf_compress_device: the BGZF container of gb_bgzf_compress (emit.cpp), compressed on the GPU from
// bytes already in HBM (gb_emit_gam_device / gb_emit_gaf_device output, or any other bytes).
//
// The input is cut every 0xff00 bytes exactly as on the host, so block k holds the same bytes in both and BGZF virtual
// offsets agree.  One CTA compresses one block at a time (a persistent grid walks the blocks), entirely in shared memory:
//   stage     the block's bytes into smem (16-byte aligned loads, so the input may start at any byte)
//   crc       CRC-32 of each thread's slice by table, the slices combined in a tree with zlib's crc32_combine algebra
//             (multiplication by x^(8 len) mod P in GF(2))
//   chains    prev[p] = the distance to an earlier position with the same 3-byte hash, built in rounds of one position
//             per thread: a position takes the nearest earlier lane of its warp with the same hash (__match_any_sync),
//             otherwise the head table as the previous rounds left it; then the last lane of each hash raises the head
//             with atomicMax.  The result depends on nothing but the input, whatever order the atomics run in.
//   parse     BGZF_SEGS threads parse one segment each, greedily: the longest match among the first BGZF_CHAIN candidates
//             of the chain (3..258 bytes, distance <= 32768, possibly reaching back into earlier segments, never past
//             the segment's own end).  Tokens go to the CTA's token slot in HBM, symbol counts to smem (atomicAdd:
//             integer sums, so order does not matter).
//   huffman   one dynamic block: counting sort by (count, symbol), Moffat–Katajainen code lengths, limited to 15 bits
//             (7 for the code-length code) by the JPEG Annex K.3 adjustment, canonical codes, the 16/17/18 RLE header.
//             Trees with fewer than two used symbols get a second one, so every code is complete.
//   pack      each segment's bit count, a block scan, then every thread ORs its bits into smem words.  The dynamic
//             block is kept only when it is smaller than the stored form (5 + len bytes); otherwise the block is stored.
//   member    the gzip member (the host's 18-byte header, the payload, CRC32 and ISIZE) to the block's 64 KiB slot.
// A CUB scan over the member sizes gives their offsets, the host waits once for the total, and bgzf_gather_kernel
// copies the members to d_out and appends the 28-byte EOF block.  Every step is a function of the block's bytes alone,
// so the output is the same on every call.
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "crc32.cuh"

#include <cub/cub.cuh>

#include <algorithm>

namespace gb {
namespace {

constexpr uint32_t BGZF_BLOCK = 0xff00;          // input bytes per BGZF block (emit.cpp, htslib)
constexpr uint32_t BGZF_SLOT = 0x10000;          // workspace bytes per compressed member (a member never exceeds 64 KiB)
constexpr uint32_t BGZF_THREADS = 512;
constexpr uint32_t BGZF_SEGS = 256;              // parse segments per block (threads 0..255)
constexpr uint32_t BGZF_CHAIN = 8;               // chain candidates tried per parse step
constexpr uint32_t BGZF_NICE = 128;              // a match this long ends the chain walk
constexpr uint32_t HASH_BITS = 13;
constexpr uint32_t WINDOW = 32768;
constexpr uint32_t CRC_LEVELS = 9;               // log2(BGZF_THREADS): levels of the CRC combine tree
static_assert(1u << CRC_LEVELS == BGZF_THREADS, "one CRC slice per thread");

// shared memory: input (+16 for the word reads past the end), prev chain (u16 distances; reused as the bit buffer), the
// head table (reused for the CRC slices, then for counts and codes); the CRC tables are static and built once per CTA
constexpr uint32_t SM_IN = 0, SM_PREV = BGZF_BLOCK + 16, SM_H = SM_PREV + 2 * BGZF_BLOCK, SM_BYTES = SM_H + 4 * (1u << HASH_BITS);
static_assert(SM_PREV % 16 == 0 && SM_H % 16 == 0, "aligned regions");

// words of the H region after the chains are built
constexpr uint32_t H_LFREQ = 0, H_DFREQ = 288, H_CFREQ = 320, H_LCODE = 352, H_DCODE = 640, H_CCODE = 672,
                   H_LSORT = 704, H_DSORT = 992, H_CSORT = 1024, H_LWORK = 1056, H_DWORK = 1344, H_RLE = 1376,
                   H_NTOK = 1696, H_SEGBITS = H_NTOK + BGZF_SEGS, H_END = H_SEGBITS + BGZF_SEGS / 32;
static_assert(H_END <= (1u << HASH_BITS), "the H region holds the Huffman tables");
// slots of the small static smem array `misc`
constexpr uint32_t M_NRLE = 0, M_HLIT = 1, M_HDIST = 2, M_HCLEN = 3, M_HDRBITS = 4, M_TOTBITS = 5, M_CRC = 6, M_STORED = 7;

__constant__ uint8_t c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
__constant__ uint8_t c_eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};

// ---- deflate symbols ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ilog2(uint32_t v) { return 31 - __clz(v); }
// length 3..258 -> (symbol 257..285, extra bits, extra value)
__device__ __forceinline__ void len_sym(uint32_t len, uint32_t& sym, uint32_t& nb, uint32_t& ev) {
    const uint32_t l = len - 3;
    if (len == 258) { sym = 285; nb = 0; ev = 0; }
    else if (l < 8) { sym = 257 + l; nb = 0; ev = 0; }
    else { nb = ilog2(l) - 2; sym = 257 + 4 * (nb + 1) + ((l >> nb) - 4); ev = l & ((1u << nb) - 1); }
}
// distance 1..32768 -> (symbol 0..29, extra bits, extra value)
__device__ __forceinline__ void dist_sym(uint32_t dist, uint32_t& sym, uint32_t& nb, uint32_t& ev) {
    const uint32_t d = dist - 1;
    if (d < 4) { sym = d; nb = 0; ev = 0; }
    else { nb = ilog2(d) - 1; sym = 2 * (nb + 1) + ((d >> nb) & 1); ev = d & ((1u << nb) - 1); }
}

// ---- Huffman code lengths ----------------------------------------------------------------------------------------------
// Counting-sort rank of every used symbol by (count, symbol), parallel over the calling threads (t = 0..n-1 of them).
__device__ void rank_symbols(const uint32_t* freq, uint32_t n, uint32_t* sorted, uint32_t t) {
    if (t >= n || freq[t] == 0) return;
    const uint32_t f = freq[t];
    uint32_t r = 0;
    for (uint32_t j = 0; j < n; j++) {
        const uint32_t g = freq[j];
        r += g != 0 && (g < f || (g == f && j < t));
    }
    sorted[r] = t;
}

// One thread: code[s] = length << 16 for the used symbols sorted[0..k), ascending by count; limit = the longest code
// allowed.  Needs k >= 2.  A = k words of scratch.
__device__ void code_lengths(const uint32_t* freq, const uint32_t* sorted, uint32_t k, uint32_t limit, uint32_t* A, uint32_t* code) {
    for (uint32_t i = 0; i < k; i++) A[i] = freq[sorted[i]];
    // Moffat & Katajainen, in place: internal node weights, then parent indices, then depths
    A[0] += A[1];
    uint32_t root = 0, leaf = 2;
    for (uint32_t next = 1; next + 1 < k; next++) {
        if (leaf >= k || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = next; }
        else A[next] = A[leaf++];
        if (leaf >= k || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = next; }
        else A[next] += A[leaf++];
    }
    A[k - 2] = 0;
    for (int next = (int)k - 3; next >= 0; next--) A[next] = A[A[next]] + 1;
    int avail = 1, used = 0, depth = 0, r = (int)k - 2, nx = (int)k - 1;
    while (avail > 0) {
        while (r >= 0 && (int)A[r] == depth) { used++; r--; }
        while (avail > used) { A[nx--] = depth; avail--; }
        avail = 2 * used; depth++; used = 0;
    }
    // A[i] = depth of the i-th leaf (non-increasing).  Count per depth and fold the deep ones up to `limit`.
    uint32_t cnt[48];
    for (uint32_t i = 0; i < 48; i++) cnt[i] = 0;
    uint32_t maxd = 0;
    for (uint32_t i = 0; i < k; i++) { cnt[A[i]]++; maxd = max(maxd, A[i]); }
    for (uint32_t i = maxd; i > limit; i--) {
        while (cnt[i] > 0) {
            uint32_t j = i - 2;
            while (cnt[j] == 0) j--;
            cnt[i] -= 2; cnt[i - 1] += 1; cnt[j + 1] += 2; cnt[j] -= 1;
        }
    }
    // the rarest symbols take the longest codes
    uint32_t idx = 0;
    for (uint32_t len = min(maxd, limit); len >= 1; len--)
        for (uint32_t c = 0; c < cnt[len]; c++) code[sorted[idx++]] = len << 16;
}

// Canonical codes (RFC 1951 3.2.2), bit-reversed for LSB-first output: code[s] = reversed code | len << 16.
__device__ void canonical(uint32_t* code, uint32_t n) {
    uint32_t bl[16] = {0}, next[16];
    for (uint32_t s = 0; s < n; s++) bl[code[s] >> 16]++;
    bl[0] = 0;
    uint32_t c = 0;
    for (uint32_t b = 1; b < 16; b++) { c = (c + bl[b - 1]) << 1; next[b] = c; }
    for (uint32_t s = 0; s < n; s++) {
        const uint32_t len = code[s] >> 16;
        if (len) code[s] = (__brev(next[len]++) >> (32 - len)) | (len << 16);
    }
}

// Used-symbol count of a tree, with a second symbol added when fewer than two are used (a complete code either way).
__device__ uint32_t pad_used(uint32_t* freq, uint32_t n) {
    uint32_t k = 0;
    for (uint32_t s = 0; s < n; s++) k += freq[s] != 0;
    for (uint32_t s = 0; k < 2 && s < n; s++)
        if (freq[s] == 0) { freq[s] = 1; k++; }
    return k;
}

// ---- bit output --------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void put_bits(uint32_t* W, uint32_t pos, uint32_t v, uint32_t n) {  // n <= 32
    if (!n) return;
    const uint32_t w = pos >> 5, sh = pos & 31;
    atomicOr(&W[w], v << sh);
    if (sh + n > 32) atomicOr(&W[w + 1], v >> (32 - sh));
}

__device__ __forceinline__ uint32_t load32(const uint8_t* in, uint32_t i) {    // 4 bytes at any offset (little-endian)
    const uint32_t* w = (const uint32_t*)in;
    return __funnelshift_r(w[i >> 2], w[(i >> 2) + 1], (i & 3) * 8);
}

__device__ __forceinline__ uint32_t hash3(const uint8_t* in, uint32_t p) {
    return ((load32(in, p) & 0xffffffu) * 2654435761u) >> (32 - HASH_BITS);
}

// the match length of p against c < p, at most `limit`
__device__ __forceinline__ uint32_t match_len(const uint8_t* in, uint32_t c, uint32_t p, uint32_t limit) {
    uint32_t l = 0;
    while (l < limit) {
        const uint32_t x = load32(in, c + l) ^ load32(in, p + l);
        if (x) { l += (__ffs(x) - 1) >> 3; break; }
        l += 4;
    }
    return min(l, limit);
}

__global__ void __launch_bounds__(BGZF_THREADS, 1)
bgzf_block_kernel(const uint8_t* __restrict__ src, uint64_t in_bytes, uint64_t n_blocks, uint8_t* __restrict__ slots,
                  uint32_t* __restrict__ token_ws, uint64_t* __restrict__ member_bytes) {
    extern __shared__ __align__(16) uint8_t sm[];
    uint8_t* in = sm + SM_IN;
    uint16_t* prev = (uint16_t*)(sm + SM_PREV);
    uint32_t* W = (uint32_t*)(sm + SM_PREV);
    uint32_t* H = (uint32_t*)(sm + SM_H);
    __shared__ uint32_t misc[8];
    uint32_t* tokens = token_ws + (uint64_t)blockIdx.x * BGZF_BLOCK;
    const uint32_t t = threadIdx.x, lane = t & 31;
    // the CRC table and x^(2^k) mod P, once per CTA
    __shared__ uint32_t crc_tab[256], x2n[32], level_op[CRC_LEVELS];
    crc32_tables(crc_tab, x2n, t, BGZF_THREADS);

    for (uint64_t b = blockIdx.x; b < n_blocks; b += gridDim.x) {
        const uint64_t at = b * BGZF_BLOCK;
        const uint32_t len = (uint32_t)min((uint64_t)BGZF_BLOCK, in_bytes - at);
        __syncthreads();                                      // the previous block's member is out of smem

        // ---- stage: aligned 16-byte loads covering [at, at + len); bytes outside it are not kept
        {
            const uint8_t* p0 = src + at;
            const uintptr_t a0 = (uintptr_t)p0 & ~(uintptr_t)15;
            const uint32_t nv = (uint32_t)(((uintptr_t)p0 + len - a0 + 15) >> 4);
            for (uint32_t v = t; v < nv; v += BGZF_THREADS) {
                const uint4 q = *(const uint4*)(a0 + 16 * (uintptr_t)v);
                const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
                const int64_t base = (int64_t)(a0 + 16 * (uintptr_t)v) - (int64_t)(uintptr_t)p0;
#pragma unroll
                for (int k = 0; k < 16; k++) {
                    const int64_t i = base + k;
                    if (i >= 0 && i < len) in[i] = (uint8_t)(w4[k >> 2] >> (8 * (k & 3)));
                }
            }
            if (t < 16) in[len + t] = 0;
        }
        // x^(8 S 2^k) mod P: the shift of a whole right-hand subtree at tree level k (only the tail's subtrees are shorter)
        const uint32_t S = (len + BGZF_THREADS - 1) / BGZF_THREADS;
        if (t < CRC_LEVELS) level_op[t] = x8nmodp((uint64_t)S << t, x2n);
        __syncthreads();

        // ---- crc: slices of S bytes, combined pairwise in a tree
        {
            const uint32_t lo = min(len, t * S), hi = min(len, lo + S);
            uint32_t c = 0xffffffffu;
            for (uint32_t i = lo; i < hi; i++) c = crc_tab[(c ^ in[i]) & 0xff] ^ (c >> 8);
            uint32_t* part = H;
            part[t] = hi > lo ? ~c : 0u;
            __syncthreads();
            for (uint32_t step = 1, k = 0; step < BGZF_THREADS; step *= 2, k++) {
                if (t % (2 * step) == 0) {
                    const uint32_t l2 = min(len, (t + 2 * step) * S) - min(len, (t + step) * S);
                    if (l2) part[t] = multmodp(l2 == S * step ? level_op[k] : x8nmodp(l2, x2n), part[t]) ^ part[t + step];
                }
                __syncthreads();
            }
            const uint32_t crc = part[0];
            __syncthreads();
            if (t == 0) misc[M_CRC] = crc;
        }

        // ---- chains
        uint32_t* head = H;                                  // head[h] = the last position so far with hash h, + 1
        for (uint32_t i = t; i < (1u << HASH_BITS); i += BGZF_THREADS) head[i] = 0;
        __syncthreads();
        for (uint32_t r0 = 0; r0 < len; r0 += BGZF_THREADS) {
            const uint32_t p = r0 + t;
            const bool ok = p + 2 < len;
            const uint32_t h = ok ? hash3(in, p) : 0x10000u + lane;
            const uint32_t same = __match_any_sync(0xffffffffu, h);
            const uint32_t before = same & ((1u << lane) - 1);
            if (ok) {
                uint32_t d = 0;
                if (before) d = lane - (31 - __clz(before));
                else { const uint32_t q = head[h]; if (q && p - (q - 1) <= WINDOW) d = p - (q - 1); }
                prev[p] = (uint16_t)d;                    // 0 = no earlier position; WINDOW fits u16
            }
            __syncthreads();
            if (ok && (same >> lane) == 1u) atomicMax(&head[h], p + 1);
            __syncthreads();
        }

        // ---- parse
        for (uint32_t i = t; i < H_END; i += BGZF_THREADS) H[i] = 0;
        __syncthreads();
        uint32_t* lfreq = H + H_LFREQ; uint32_t* dfreq = H + H_DFREQ;
        const uint32_t seg = (len + BGZF_SEGS - 1) / BGZF_SEGS;
        if (t < BGZF_SEGS) {
            const uint32_t s0 = min(len, t * seg), s1 = min(len, s0 + seg);
            uint32_t* tk = tokens + s0;
            uint32_t nt = 0, p = s0;
            while (p < s1) {
                const uint32_t limit = min(258u, s1 - p);
                uint32_t best = 0, bdist = 0;
                if (limit >= 3) {
                    uint32_t c = p, d = prev[p];
                    for (uint32_t k = 0; k < BGZF_CHAIN && d; k++) {
                        if (p - c + d > WINDOW) break;
                        c -= d;
                        const uint32_t l = match_len(in, c, p, limit);
                        if (l > best) { best = l; bdist = p - c; if (l >= min(limit, BGZF_NICE)) break; }
                        d = prev[c];
                    }
                }
                if (best >= 3) {
                    tk[nt++] = (best << 16) | bdist;
                    uint32_t sym, nb, ev;
                    len_sym(best, sym, nb, ev); atomicAdd(&lfreq[sym], 1u);
                    dist_sym(bdist, sym, nb, ev); atomicAdd(&dfreq[sym], 1u);
                    p += best;
                } else {
                    tk[nt++] = in[p];
                    atomicAdd(&lfreq[in[p]], 1u);
                    p++;
                }
            }
            H[H_NTOK + t] = nt;
        }
        if (t == 0) lfreq[256] = 1;                    // end of block
        __syncthreads();

        // ---- huffman: litlen and distance trees by warps 0 and 1, then the code-length code by thread 0
        uint32_t* lcode = H + H_LCODE; uint32_t* dcode = H + H_DCODE; uint32_t* ccode = H + H_CCODE;
        if (t == 0) misc[M_HLIT] = pad_used(lfreq, 286);
        if (t == 32) misc[M_HDIST] = pad_used(dfreq, 30);
        __syncthreads();
        rank_symbols(lfreq, 286, H + H_LSORT, t);
        if (t >= 288 && t < 318) rank_symbols(dfreq, 30, H + H_DSORT, t - 288);
        __syncthreads();
        if (t == 0) code_lengths(lfreq, H + H_LSORT, misc[M_HLIT], 15, H + H_LWORK, lcode);
        if (t == 32) code_lengths(dfreq, H + H_DSORT, misc[M_HDIST], 15, H + H_DWORK, dcode);
        __syncthreads();
        if (t == 0) {
            canonical(lcode, 286);
            canonical(dcode, 30);
            uint32_t hlit = 286, hdist = 30;
            while (hlit > 257 && (lcode[hlit - 1] >> 16) == 0) hlit--;
            while (hdist > 1 && (dcode[hdist - 1] >> 16) == 0) hdist--;
            // RLE of the hlit + hdist lengths as one sequence: rle[] = symbol | extra value << 8
            uint32_t* rle = H + H_RLE; uint32_t* cfreq = H + H_CFREQ;
            uint32_t nr = 0;
            const uint32_t total = hlit + hdist;
            auto L = [&](uint32_t i) { return i < hlit ? lcode[i] >> 16 : dcode[i - hlit] >> 16; };
            for (uint32_t i = 0; i < total;) {
                const uint32_t v = L(i);
                uint32_t run = 1;
                while (i + run < total && L(i + run) == v) run++;
                uint32_t r = run;
                if (v == 0) {
                    while (r >= 11) { const uint32_t n = min(r, 138u); rle[nr++] = 18 | (n - 11) << 8; r -= n; }
                    if (r >= 3) { rle[nr++] = 17 | (r - 3) << 8; r = 0; }
                } else {
                    rle[nr++] = v; r--;
                    while (r >= 3) { const uint32_t n = min(r, 6u); rle[nr++] = 16 | (n - 3) << 8; r -= n; }
                }
                while (r > 0) { rle[nr++] = v; r--; }
                i += run;
            }
            for (uint32_t i = 0; i < nr; i++) cfreq[rle[i] & 0xff]++;
            const uint32_t kc = pad_used(cfreq, 19);
            uint32_t* csort = H + H_CSORT;
            for (uint32_t s = 0; s < 19; s++) rank_symbols(cfreq, 19, csort, s);
            code_lengths(cfreq, csort, kc, 7, H + H_LWORK, ccode);
            canonical(ccode, 19);
            uint32_t hclen = 19;
            while (hclen > 4 && (ccode[c_cl_order[hclen - 1]] >> 16) == 0) hclen--;
            uint32_t bits = 3 + 5 + 5 + 4 + 3 * hclen;
            for (uint32_t i = 0; i < nr; i++) {
                const uint32_t s = rle[i] & 0xff;
                bits += (ccode[s] >> 16) + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
            }
            misc[M_NRLE] = nr; misc[M_HLIT] = hlit; misc[M_HDIST] = hdist; misc[M_HCLEN] = hclen; misc[M_HDRBITS] = bits;
        }
        __syncthreads();

        // ---- pack: bits per segment, scan, decide, write
        uint32_t mybits = 0, nt = 0;
        const uint32_t s0 = min(len, t * seg);
        if (t < BGZF_SEGS) {
            nt = H[H_NTOK + t];
            for (uint32_t i = 0; i < nt; i++) {
                const uint32_t x = tokens[s0 + i];
                if (x < 256) { mybits += lcode[x] >> 16; continue; }
                uint32_t sym, nb, ev;
                len_sym(x >> 16, sym, nb, ev); mybits += (lcode[sym] >> 16) + nb;
                dist_sym(x & 0xffff, sym, nb, ev); mybits += (dcode[sym] >> 16) + nb;
            }
        }
        uint32_t incl = mybits;                        // warp-inclusive scan; BGZF_SEGS threads = 4 warps
#pragma unroll
        for (int o = 1; o < 32; o *= 2) { const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += y; }
        if (t < BGZF_SEGS && lane == 31) H[H_SEGBITS + (t >> 5)] = incl;
        __syncthreads();
        uint32_t wbase = misc[M_HDRBITS];
        for (uint32_t w = 0; w < (t >> 5) && w < BGZF_SEGS / 32; w++) wbase += H[H_SEGBITS + w];
        const uint32_t my0 = wbase + incl - mybits;   // this segment's first bit
        if (t == BGZF_SEGS - 1) {
            const uint32_t tot = my0 + mybits + (lcode[256] >> 16);
            misc[M_TOTBITS] = tot;
            misc[M_STORED] = (tot + 7) / 8 >= len + 5;
        }
        __syncthreads();
        const bool stored = misc[M_STORED] != 0;
        const uint32_t pay = stored ? len + 5 : (misc[M_TOTBITS] + 7) / 8;
        if (!stored) {
            const uint32_t nw = (pay + 3) / 4 + 1;
            for (uint32_t i = t; i < nw; i += BGZF_THREADS) W[i] = 0;
            __syncthreads();
            if (t == 0) {                              // block header: BFINAL 1, BTYPE 10, HLIT, HDIST, HCLEN, code lengths
                uint32_t pos = 0;
                const uint32_t hlit = misc[M_HLIT], hdist = misc[M_HDIST], hclen = misc[M_HCLEN], nr = misc[M_NRLE];
                put_bits(W, pos, 1 | 2 << 1 | (hlit - 257) << 3 | (hdist - 1) << 8 | (hclen - 4) << 13, 17); pos += 17;
                for (uint32_t i = 0; i < hclen; i++) { put_bits(W, pos, ccode[c_cl_order[i]] >> 16, 3); pos += 3; }
                const uint32_t* rle = H + H_RLE;
                for (uint32_t i = 0; i < nr; i++) {
                    const uint32_t s = rle[i] & 0xff, c = ccode[s];
                    const uint32_t nb = s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0;
                    put_bits(W, pos, (c & 0xffff) | (rle[i] >> 8) << (c >> 16), (c >> 16) + nb); pos += (c >> 16) + nb;
                }
                const uint32_t e = lcode[256];
                put_bits(W, misc[M_TOTBITS] - (e >> 16), e & 0xffff, e >> 16);
            }
            if (t < BGZF_SEGS) {
                uint32_t pos = my0;
                for (uint32_t i = 0; i < nt; i++) {
                    const uint32_t x = tokens[s0 + i];
                    if (x < 256) { const uint32_t c = lcode[x]; put_bits(W, pos, c & 0xffff, c >> 16); pos += c >> 16; continue; }
                    uint32_t sym, nb, ev;
                    len_sym(x >> 16, sym, nb, ev);
                    uint32_t c = lcode[sym];
                    put_bits(W, pos, (c & 0xffff) | ev << (c >> 16), (c >> 16) + nb); pos += (c >> 16) + nb;
                    dist_sym(x & 0xffff, sym, nb, ev);
                    c = dcode[sym];
                    put_bits(W, pos, (c & 0xffff) | ev << (c >> 16), (c >> 16) + nb); pos += (c >> 16) + nb;
                }
            }
            __syncthreads();
        }

        // ---- member: header, payload, CRC32, ISIZE into the block's slot
        uint8_t* out = slots + b * BGZF_SLOT;
        const uint32_t total = 18 + pay + 8;
        const uint8_t* wb = (const uint8_t*)W;
        for (uint32_t i = t; i < total; i += BGZF_THREADS) {
            uint8_t v;
            if (i < 16) v = c_eof[i];
            else if (i == 16) v = (uint8_t)((total - 1) & 0xff);
            else if (i == 17) v = (uint8_t)((total - 1) >> 8);
            else if (i < 18 + pay) {
                const uint32_t j = i - 18;
                if (!stored) v = wb[j];
                else if (j == 0) v = 1;                                // BFINAL 1, BTYPE 00
                else if (j < 5) v = (uint8_t)(((j < 3 ? len : ~len) >> (8 * ((j - 1) & 1))) & 0xff);
                else v = in[j - 5];
            } else {
                const uint32_t j = i - 18 - pay;
                v = (uint8_t)((j < 4 ? misc[M_CRC] : len) >> (8 * (j & 3)));
            }
            out[i] = v;
        }
        if (t == 0) member_bytes[b] = total;
    }
}

// Members to their scanned offsets, then the EOF block: CTA b < n_blocks copies member b, CTA n_blocks the EOF block.
__global__ void bgzf_gather_kernel(const uint8_t* __restrict__ slots, const uint64_t* __restrict__ member_bytes,
                                   const uint64_t* __restrict__ off, uint64_t n_blocks, uint8_t* __restrict__ out) {
    for (uint64_t b = blockIdx.x; b <= n_blocks; b += gridDim.x) {
        if (b == n_blocks) {
            if (threadIdx.x < 28) out[off[b] + threadIdx.x] = c_eof[threadIdx.x];
            continue;
        }
        const uint8_t* s = slots + b * BGZF_SLOT;
        uint8_t* d = out + off[b];
        const uint32_t n = (uint32_t)member_bytes[b];
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) d[i] = s[i];
    }
}

int bgzf_compress_device(gb_device* d, const void* d_in, uint64_t in_bytes, void* d_out, uint64_t out_cap, uint64_t* out_used) {
    if (!d || !out_used || (!d_in && in_bytes) || !d_out) return GB_ERR_ARG;
    GB_CUDA(cudaSetDevice(d->device));
    const uint64_t nb = (in_bytes + BGZF_BLOCK - 1) / BGZF_BLOCK;
    const uint32_t grid = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(nb, 1), (uint64_t)d->n_sms);
    size_t scan = 0;
    GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t)(nb + 1), d->stream));
    // workspace: total (not read: the host takes it from off[nb]), member_bytes[nb + 1], off[nb + 1], scan temp, token slots
    // (one block of u32 per CTA), member slots
    uint64_t *sizes, *off;
    uint32_t* tok;
    uint8_t *tmp, *slots;
    int rc = carve(d->bgzf_ws, [&](Carve& c) {
        c.take<uint64_t>(1); sizes = c.take<uint64_t>(nb + 1); off = c.take<uint64_t>(nb + 1); tmp = c.take<uint8_t>(scan);
        tok = c.take<uint32_t>((size_t)grid * BGZF_BLOCK); slots = c.take<uint8_t>((size_t)nb * BGZF_SLOT);
    });
    if (rc) return rc;
    GB_CUDA(cudaFuncSetAttribute(bgzf_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SM_BYTES));
    GB_CUDA(cudaMemsetAsync(sizes + nb, 0, sizeof(uint64_t), d->stream));
    if (nb) {
        bgzf_block_kernel<<<grid, BGZF_THREADS, SM_BYTES, d->stream>>>((const uint8_t*)d_in, in_bytes, nb, slots, tok, sizes);
        d->launches++;
        GB_CUDA(cudaGetLastError());
    }
    GB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, scan, sizes, off, (int64_t)(nb + 1), d->stream));
    d->launches++;
    uint64_t h_total = 0;
    GB_CUDA(cudaMemcpyAsync(&h_total, off + nb, sizeof h_total, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));              // the one wait: the total decides whether the gather runs
    const uint64_t total = h_total + 28;
    *out_used = total;
    if (total > out_cap) { g_last_error = "gb_bgzf_compress_device: output capacity too small (*out_used holds the bytes needed)"; return GB_ERR_CAPACITY; }
    const uint32_t ggrid = (uint32_t)std::min<uint64_t>(nb + 1, (uint64_t)d->n_sms * 16);
    bgzf_gather_kernel<<<ggrid, 256, 0, d->stream>>>(slots, sizes, off, nb, (uint8_t*)d_out);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    return GB_OK;
}

} // namespace
} // namespace gb

extern "C" int gb_bgzf_compress_device(gb_device* dev, const void* d_in, uint64_t in_bytes, void* d_out, uint64_t out_cap, uint64_t* out_used) {
    return gb::guarded("gb_bgzf_compress_device", [&] { return gb::bgzf_compress_device(dev, d_in, in_bytes, d_out, out_cap, out_used); });
}
