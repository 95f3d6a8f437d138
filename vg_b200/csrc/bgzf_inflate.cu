// bgzf_inflate.cu — gb_bgzf_decompress_device: BGZF members already in HBM inflated on the GPU, the inverse of
// gb_bgzf_compress_device (and of gb_bgzf_compress, bgzip, htslib, vg::io).
//
//   walk      one thread follows BSIZE from member to member, checks each gzip header (FLG = FEXTRA, a 'BC' subfield of
//             SLEN 2 among the XLEN bytes) and reads CRC32 / ISIZE from the trailer; the output offset of every member is
//             the running sum of the ISIZEs.  The host waits once for the count, the total and where the walk stopped.
//   inflate   one warp per member (INF_WARPS per CTA).  The payload is staged through a per-warp window in shared
//             memory; every lane holds the same bit buffer and decodes the same symbol (a deflate block is serial), so
//             the control flow stays warp-uniform.  Litlen / distance codes decode through a 10-bit / 8-bit table in
//             shared memory with a canonical walk for longer codes; the code-length code through the canonical walk.
//             Literals are stored by lane 0; a match is copied by all lanes, byte i from out[pos - dist + i % dist], so
//             a match that overlaps its source needs no ordering inside the copy.  Back-references read d_out (written
//             by this warp, ordered by __syncwarp).  Every read is bounded by the member's payload and every write by its
//             ISIZE slot.  The code tables follow zlib's rules (over-subscribed codes refused, incomplete ones only for a
//             single one-bit litlen / distance code), so a member is accepted exactly when zlib's raw inflate accepts
//             its payload with nothing left over, and the output is then zlib's bytes.
//   crc       the lanes compute CRC-32 over slices of the member's output and combine them (crc32.cuh); CRC and
//             ISIZE must match the trailer.  A failing member lowers one device word to its offset; the host waits
//             for it once.
#include "giraffe_b200.h"
#include "device_state.cuh"
#include "crc32.cuh"

#include <algorithm>
#include <string>

namespace gb {
namespace {

constexpr uint32_t INF_WARPS = 8;                 // warps (members in flight) per CTA
constexpr uint32_t WIN_WORDS = 512;               // payload window per warp: 2 KiB
constexpr uint32_t LBITS = 10, DBITS = 8;         // first-level table bits of the litlen / distance codes
constexpr uint32_t MIN_MEMBER = 26;               // 12-byte header + a 6-byte BC subfield + the 8-byte trailer
constexpr uint64_t NONE = ~0ull;

enum WalkStatus : uint32_t { W_END = 0, W_TRUNC = 1, W_NOT_GZIP = 2, W_FLAGS = 3, W_EXTRA = 4, W_NO_BC = 5, W_BSIZE = 6, W_ISIZE = 7 };

struct Member {
    uint64_t at;          // first byte of the member in d_in
    uint64_t out;         // first byte of its output in d_out
    uint32_t pay, plen;   // payload offset inside the member, payload bytes
    uint32_t isize, crc;
};
struct WalkSum {
    uint64_t n, stop, total;     // members, where the walk stopped, sum of ISIZE
    uint32_t status, pad;
    unsigned long long bad_at;   // offset of the first member that does not inflate (NONE: all did)
};

// ---- walk ---------------------------------------------------------------------------------------------------------------
__global__ void bgzf_walk_kernel(const uint8_t* __restrict__ in, uint64_t in_bytes, uint64_t cap, Member* __restrict__ mem,
                                 WalkSum* __restrict__ sum) {
    uint64_t p = 0, n = 0, total = 0;
    uint32_t status = W_END;
    while (p < in_bytes) {
        const uint8_t* b = in + p;
        const uint64_t avail = in_bytes - p;
        bool ok = b[0] == 0x1f;
        if (avail > 1) ok &= b[1] == 0x8b;
        if (avail > 2) ok &= b[2] == 8;
        if (!ok) { status = W_NOT_GZIP; break; }
        if (avail >= 4 && !(b[3] & 4)) { status = W_NO_BC; break; }     // no extra field: plain gzip
        if (avail >= 4 && b[3] != 4) { status = W_FLAGS; break; }
        if (avail < 12) { status = W_TRUNC; break; }
        const uint32_t xlen = b[10] | (uint32_t)b[11] << 8;
        if (avail < 12 + xlen) { status = W_TRUNC; break; }
        uint32_t q = 12, bsize = 0;
        bool found = false;
        while (q + 4 <= 12 + xlen) {
            const uint32_t slen = b[q + 2] | (uint32_t)b[q + 3] << 8;
            if (q + 4 + slen > 12 + xlen) break;
            if (!found && b[q] == 'B' && b[q + 1] == 'C' && slen == 2) { bsize = b[q + 4] | (uint32_t)b[q + 5] << 8; found = true; }
            q += 4 + slen;
        }
        if (q != 12 + xlen) { status = W_EXTRA; break; }
        if (!found) { status = W_NO_BC; break; }
        const uint64_t mlen = (uint64_t)bsize + 1;
        if (mlen < 12 + xlen + 8) { status = W_BSIZE; break; }
        if (mlen > avail) { status = W_TRUNC; break; }
        const uint8_t* t = b + mlen - 8;
        const uint32_t crc = t[0] | (uint32_t)t[1] << 8 | (uint32_t)t[2] << 16 | (uint32_t)t[3] << 24;
        const uint32_t isize = t[4] | (uint32_t)t[5] << 8 | (uint32_t)t[6] << 16 | (uint32_t)t[7] << 24;
        if (isize > 65536) { status = W_ISIZE; break; }
        if (n == cap) { status = W_BSIZE; break; }        // cannot happen: every member is at least MIN_MEMBER bytes
        mem[n] = Member{p, total, 12 + xlen, (uint32_t)(mlen - 12 - xlen - 8), isize, crc};
        n++; total += isize; p += mlen;
    }
    *sum = WalkSum{n, p, total, status, 0, NONE};
}

// ---- inflate ------------------------------------------------------------------------------------------------------------
__constant__ uint16_t c_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                     131, 163, 195, 227, 258};
__constant__ uint8_t c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                     2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// Per warp: the payload window, and each code as counts per length, symbols sorted by (length, symbol) and a
// first-level table indexed by the next stream bits holding (length << 9 | symbol), 0 when the code is longer or absent.
struct WarpSmem {
    uint32_t win[WIN_WORDS + 2];
    uint16_t llut[1u << LBITS], dlut[1u << DBITS];
    uint16_t lcnt[16], dcnt[16], lsym[288], dsym[32];
    uint8_t lens[288 + 32];
    uint16_t offs[16];                            // build_code's scratch
    uint8_t cl[19];
    uint8_t ok;
};

// Builds the code of lens[0..n) (warp-cooperative).  zlib's inflate_table rules: over-subscribed is refused; incomplete
// is refused for the code-length code and for any code whose longest length is not 1; no symbols at all is accepted
// (every lookup then fails).
__device__ bool build_code(const uint8_t* lens, uint32_t n, uint16_t* cnt, uint16_t* sym, uint16_t* lut, uint32_t bits,
                           bool codelen, uint16_t* offs, uint8_t* okp, uint32_t lane) {
    __syncwarp();
    if (lane == 0) {
        for (int l = 0; l < 16; l++) cnt[l] = 0;
        for (uint32_t s = 0; s < n; s++) cnt[lens[s]]++;
        cnt[0] = 0;
        int left = 1, maxl = 0;
        bool ok = true;
        for (int l = 1; l < 16; l++) { left <<= 1; left -= cnt[l]; if (left < 0) ok = false; if (cnt[l]) maxl = l; }
        if (ok && maxl && left > 0 && (codelen || maxl != 1)) ok = false;
        if (ok) {
            offs[1] = 0;
            for (int l = 1; l < 15; l++) offs[l + 1] = offs[l] + cnt[l];
            for (uint32_t s = 0; s < n; s++) if (lens[s]) sym[offs[lens[s]]++] = (uint16_t)s;
        }
        *okp = ok;
    }
    __syncwarp();
    if (!*okp) return false;
    if (lut) {
        for (uint32_t i = lane; i < (1u << bits); i += 32) lut[i] = 0;
        __syncwarp();
        // sorted index i has length l and code first[l] + (i - start[l])
        uint32_t total = 0;
        for (int l = 1; l < 16; l++) total += cnt[l];
        for (uint32_t i = lane; i < total; i += 32) {
            uint32_t start = 0, code = 0, l = 1;
            for (; l < 16; l++) {
                if (i < start + cnt[l]) break;
                start += cnt[l];
                code = (code + cnt[l]) << 1;
            }
            if (l > bits) continue;
            code += i - start;
            const uint32_t rev = __brev(code) >> (32 - l);
            for (uint32_t k = 0; k < (1u << (bits - l)); k++) lut[rev | k << l] = (uint16_t)(l << 9 | sym[i]);
        }
        __syncwarp();
    }
    return true;
}

struct BitReader {
    const uint8_t* P;     // payload
    uint32_t plen;
    uint64_t buf;
    uint32_t nb;          // valid bits in buf
    uint32_t ip;          // next payload byte to append to buf
    uint64_t wa;          // window base address (4-aligned)
    uint32_t wend;        // payload index below which 4 bytes can be read from the window

    __device__ void load_window(uint32_t* win, uint32_t lane) {
        __syncwarp();
        const uint64_t pa = (uint64_t)(uintptr_t)P;
        wa = (pa + ip) & ~3ull;
        for (uint32_t k = lane; k < WIN_WORDS + 2; k += 32) {
            const uint64_t a = wa + 4ull * k;
            win[k] = (a + 4 > pa && a < pa + plen) ? *(const uint32_t*)(uintptr_t)a : 0u;
        }
        wend = (uint32_t)(wa + 4ull * WIN_WORDS - pa);
        __syncwarp();
    }
    // at least 33 valid bits afterwards; false once the reader is more than 8 bytes past the payload
    __device__ bool refill(uint32_t* win, uint32_t lane) {
        if (nb > 32) return true;
        if (ip > plen + 8) return false;
        if (ip + 4 > wend) load_window(win, lane);
        const uint32_t r = (uint32_t)((uint64_t)(uintptr_t)P + ip - wa);
        const uint32_t w = __funnelshift_r(win[r >> 2], win[(r >> 2) + 1], (r & 3) * 8);
        buf |= (uint64_t)w << nb;
        nb += 32; ip += 4;
        return true;
    }
    __device__ uint32_t bits(uint32_t n) {
        const uint32_t v = (uint32_t)buf & ((1u << n) - 1);
        buf >>= n; nb -= n;
        return v;
    }
    __device__ uint64_t consumed() const { return 8ull * ip - nb; }
};

// Next symbol of a code, or -1 for a bit pattern that is no code.
__device__ __forceinline__ int decode(BitReader& br, const uint16_t* lut, uint32_t lbits, const uint16_t* cnt, const uint16_t* sym) {
    if (lut) {
        const uint32_t e = lut[br.buf & ((1u << lbits) - 1)];
        if (e) { br.bits(e >> 9); return (int)(e & 511); }
    }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; l++) {
        code |= (int)((br.buf >> (l - 1)) & 1);
        const int count = cnt[l];
        if (code - count < first) { br.bits(l); return sym[index + (code - first)]; }
        index += count; first += count;
        first <<= 1; code <<= 1;
    }
    return -1;
}

__global__ void __launch_bounds__(INF_WARPS * 32, 4)
bgzf_inflate_kernel(const uint8_t* __restrict__ in, const Member* __restrict__ mem, uint64_t n_members, uint8_t* out_base,
                    WalkSum* sum) {
    __shared__ WarpSmem wsm[INF_WARPS];
    __shared__ uint32_t crc_tab[256], x2n[32];
    crc32_tables(crc_tab, x2n, threadIdx.x, blockDim.x);
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    WarpSmem& S = wsm[w];
    for (uint64_t m = (uint64_t)blockIdx.x * INF_WARPS + w; m < n_members; m += (uint64_t)gridDim.x * INF_WARPS) {
        const Member M = mem[m];
        uint8_t* out = out_base + M.out;
        const uint32_t osz = M.isize;
        BitReader br{in + M.at + M.pay, M.plen, 0, 0, 0, 0, 0};
        br.load_window(S.win, lane);
        uint32_t op = 0;
        bool ok = true, last = false;
        while (ok && !last) {
            if (!br.refill(S.win, lane)) { ok = false; break; }
            last = br.bits(1);
            const uint32_t type = br.bits(2);
            if (type == 0) {                                      // stored
                br.bits(br.nb & 7);
                if (!br.refill(S.win, lane)) { ok = false; break; }
                const uint32_t len = br.bits(16), nlen = br.bits(16);
                const uint32_t at = br.ip - br.nb / 8;
                if ((len ^ 0xffffu) != nlen || at + len > br.plen || op + len > osz) { ok = false; break; }
                for (uint32_t i = lane; i < len; i += 32) out[op + i] = br.P[at + i];
                op += len;
                br.ip = at + len; br.buf = 0; br.nb = 0;
                continue;
            }
            if (type == 3) { ok = false; break; }
            uint32_t hlit = 288, hdist = 32;
            if (type == 1) {                                      // fixed
                for (uint32_t s = lane; s < 320; s += 32)
                    S.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
            } else {                                              // dynamic
                if (!br.refill(S.win, lane)) { ok = false; break; }
                hlit = br.bits(5) + 257; hdist = br.bits(5) + 1;
                const uint32_t hclen = br.bits(4) + 4;
                if (hlit > 286 || hdist > 30) { ok = false; break; }
                for (uint32_t i = lane; i < 19; i += 32) S.cl[i] = 0;
                __syncwarp();
                for (uint32_t i = 0; i < hclen; i++) {
                    if (!br.refill(S.win, lane)) { ok = false; break; }
                    const uint32_t v = br.bits(3);
                    if (lane == 0) S.cl[c_cl_order[i]] = (uint8_t)v;
                }
                if (!ok) break;
                __syncwarp();
                if (!build_code(S.cl, 19, S.lcnt, S.lsym, nullptr, 0, true, S.offs, &S.ok, lane)) { ok = false; break; }
                const uint32_t total = hlit + hdist;
                for (uint32_t i = 0; i < total && ok;) {
                    if (!br.refill(S.win, lane)) { ok = false; break; }
                    const int s = decode(br, nullptr, 0, S.lcnt, S.lsym);
                    uint32_t v = 0, rep = 1;
                    if (s < 0) { ok = false; break; }
                    if (s < 16) v = (uint32_t)s;
                    else if (s == 16) { if (i == 0) { ok = false; break; } v = S.lens[i - 1]; rep = 3 + br.bits(2); }
                    else if (s == 17) rep = 3 + br.bits(3);
                    else rep = 11 + br.bits(7);
                    if (i + rep > total) { ok = false; break; }
                    __syncwarp();
                    for (uint32_t k = lane; k < rep; k += 32) S.lens[i + k] = (uint8_t)v;
                    __syncwarp();
                    i += rep;
                }
                if (!ok) break;
                const uint8_t dl = lane < hdist ? S.lens[hlit + lane] : 0;     // distances to [288, 320) (hdist <= 30)
                __syncwarp();
                if (lane < hdist) S.lens[288 + lane] = dl;
                for (uint32_t s = hlit + lane; s < 288; s += 32) S.lens[s] = 0;
                __syncwarp();
                if (S.lens[256] == 0) { ok = false; break; }
            }
            if (!build_code(S.lens, hlit, S.lcnt, S.lsym, S.llut, LBITS, false, S.offs, &S.ok, lane) ||
                !build_code(S.lens + 288, hdist, S.dcnt, S.dsym, S.dlut, DBITS, false, S.offs, &S.ok, lane)) { ok = false; break; }
            for (;;) {                                            // the block's symbols
                if (!br.refill(S.win, lane)) { ok = false; break; }
                const int s = decode(br, S.llut, LBITS, S.lcnt, S.lsym);
                if (s < 0 || s > 285) { ok = false; break; }
                if (s < 256) {
                    if (op >= osz) { ok = false; break; }
                    if (lane == 0) out[op] = (uint8_t)s;
                    op++;
                    continue;
                }
                if (s == 256) break;
                const uint32_t len = c_lbase[s - 257] + br.bits(c_lext[s - 257]);
                if (!br.refill(S.win, lane)) { ok = false; break; }
                const int ds = decode(br, S.dlut, DBITS, S.dcnt, S.dsym);
                if (ds < 0 || ds > 29) { ok = false; break; }
                const uint32_t dist = c_dbase[ds] + br.bits(c_dext[ds]);
                if (dist > op || op + len > osz) { ok = false; break; }
                __syncwarp();                                     // earlier literals and copies are visible to every lane
                const uint8_t* src = out + op - dist;
                if (dist >= len) { for (uint32_t i = lane; i < len; i += 32) out[op + i] = src[i]; }
                else { for (uint32_t i = lane; i < len; i += 32) out[op + i] = src[i % dist]; }
                op += len;
            }
        }
        // nothing left over: the last block ends in the payload's last byte; the member's size and CRC match the trailer
        ok = ok && (br.consumed() + 7) / 8 == br.plen && op == osz;
        if (ok) {
            __syncwarp();
            const uint32_t sl = (osz + 31) / 32, lo = min(osz, lane * sl), hi = min(osz, lo + sl);
            uint32_t c = 0xffffffffu;
            for (uint32_t i = lo; i < hi; i++) c = crc_tab[(c ^ out[i]) & 0xff] ^ (c >> 8);
            c = ~c;
            uint32_t len = hi - lo;
            for (uint32_t step = 1; step < 32; step *= 2) {
                const uint32_t oc = __shfl_down_sync(0xffffffffu, c, step), ol = __shfl_down_sync(0xffffffffu, len, step);
                if (lane % (2 * step) == 0 && lane + step < 32) { c = crc32_combine(c, oc, ol, x2n); len += ol; }
            }
            ok = __shfl_sync(0xffffffffu, c, 0) == M.crc;
        }
        if (!ok && lane == 0) atomicMin(&sum->bad_at, (unsigned long long)M.at);
        __syncwarp();
    }
}

int bgzf_decompress_device(gb_device* d, const void* d_in, uint64_t in_bytes, int final, void* d_out, uint64_t out_cap,
                           uint64_t* out_used, uint64_t* in_used) {
    if (!d || !out_used || !in_used || (!d_in && in_bytes) || (!d_out && out_cap)) return GB_ERR_ARG;
    *out_used = 0; *in_used = 0;
    GB_CUDA(cudaSetDevice(d->device));
    const uint64_t cap = in_bytes / MIN_MEMBER + 1;
    WalkSum* sum;
    Member* mem;
    if (int rc = carve(d->inflate_ws, [&](Carve& c) { sum = c.take<WalkSum>(1); mem = c.take<Member>(cap); })) return rc;
    bgzf_walk_kernel<<<1, 1, 0, d->stream>>>((const uint8_t*)d_in, in_bytes, cap, mem, sum);
    d->launches++;
    GB_CUDA(cudaGetLastError());
    WalkSum h{};
    GB_CUDA(cudaMemcpyAsync(&h, sum, sizeof h, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));              // wait 1: the members, their total and where the walk stopped
    if (h.status > W_TRUNC || (h.status == W_TRUNC && final)) {
        static const char* what[] = {"", "a member runs past the end of the input", "not a gzip member (no 1f 8b 08 magic)",
                                     "the gzip flags are not FEXTRA alone (FNAME, FCOMMENT and FHCRC are not supported)",
                                     "the gzip extra field's subfields do not add up to XLEN",
                                     "no 'BC' subfield: plain gzip is not BGZF and cannot be inflated by blocks; inflate it on the host",
                                     "BSIZE is smaller than the member's header and trailer", "ISIZE is above 65536"};
        g_last_error = "gb_bgzf_decompress_device: byte " + std::to_string(h.stop) + ": " + what[h.status];
        return GB_ERR_FORMAT;
    }
    if (h.total > out_cap) {
        *out_used = h.total;
        g_last_error = "gb_bgzf_decompress_device: output capacity too small (*out_used holds the bytes needed)";
        return GB_ERR_CAPACITY;
    }
    if (h.n) {
        const uint32_t grid = (uint32_t)std::min<uint64_t>((h.n + INF_WARPS - 1) / INF_WARPS, (uint64_t)d->n_sms * 4);
        bgzf_inflate_kernel<<<grid, INF_WARPS * 32, 0, d->stream>>>((const uint8_t*)d_in, mem, h.n, (uint8_t*)d_out, sum);
        d->launches++;
        GB_CUDA(cudaGetLastError());
        unsigned long long bad = 0;
        GB_CUDA(cudaMemcpyAsync(&bad, &sum->bad_at, sizeof bad, cudaMemcpyDeviceToHost, d->stream));
        GB_CUDA(cudaStreamSynchronize(d->stream));          // wait 2: did every member inflate
        if (bad != NONE) {
            g_last_error = "gb_bgzf_decompress_device: the BGZF member at byte " + std::to_string(bad) +
                           " does not inflate to its trailer's CRC32 and ISIZE";
            return GB_ERR_FORMAT;
        }
    }
    *out_used = h.total;
    *in_used = h.stop;
    return GB_OK;
}

} // namespace
} // namespace gb

extern "C" int gb_bgzf_decompress_device(gb_device* dev, const void* d_in, uint64_t in_bytes, int final, void* d_out,
                                         uint64_t out_cap, uint64_t* out_used, uint64_t* in_used) {
    return gb::guarded("gb_bgzf_decompress_device",
                       [&] { return gb::bgzf_decompress_device(dev, d_in, in_bytes, final, d_out, out_cap, out_used, in_used); });
}
