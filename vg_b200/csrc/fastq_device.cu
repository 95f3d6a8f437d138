// fastq_device.cu — gb_fastq_parse_device: FASTQ text already in HBM (gb_bgzf_decompress_device output) parsed into the
// arrays gb_map_batch_device and gb_emit_*_device take: reads / quals addressed by read_off, names by name_off.
//
// Per input:
//   lines     CTAs of 256 threads count the '\n' bytes of 4 KiB tiles (16-byte aligned loads, so the text may start at
//             any byte), a CUB scan gives every tile's first line index, and a second pass writes the position of
//             every '\n' (the first 4 * records_needed of them).  The caller's text begins at a record boundary, so
//             record r is lines 4r .. 4r + 3.
//   records   one warp per record checks the header ('@'), finds the end of the name (the first of " \t\v\f\r", by
//             ballot), checks the sequence and quality bytes ('!'..'~'), the separator ('+') and the quality length,
//             and writes the read's sequence and name lengths in output order (pairs interleaved: mate 1, mate 2).
// Then CUB scans of the lengths give the candidate offsets; one thread finds the longest prefix of whole records (pairs)
// that fits max_reads, bases_cap and names_cap and decides the status; a reduction takes the longest read of that
// prefix; one warp per read copies the name, uppercases the bases and subtracts 33 from the qualities.  The host
// waits once, for the summary.
#include "giraffe_b200.h"
#include "device_state.cuh"

#include <cub/cub.cuh>

#include <algorithm>
#include <string>

namespace gb {
namespace {

constexpr uint32_t NL_THREADS = 256;                // threads per line-finding CTA, 16 bytes each
constexpr uint32_t REC_WARPS = 8;

enum FqErr : uint32_t { FQ_OK = 0, FQ_HEADER = 1, FQ_SEQ_BYTE = 2, FQ_SEPARATOR = 3, FQ_QUAL_LEN = 4, FQ_QUAL_BYTE = 5 };

struct FqSum {
    uint64_t n_lines[2];          // '\n' bytes of each input (all of them, not only those stored)
    uint64_t text_used[2];
    uint64_t err_off;             // byte offset of the refused record's fault in its input
    uint32_t first_bad;           // smallest read index of a refused record (0xffffffff: none)
    uint32_t err_kind, n_take, max_len, status;     // status: 0 ok, 1 refused record, 2 capacity (nothing fits)
    uint32_t need_kind;           // capacity: 0 max_reads, 1 bases_cap, 2 names_cap
    uint64_t need;                // capacity: what the first record (pair) needs of it
};

struct Input {
    const uint8_t* text;
    uint64_t bytes;
    const uint64_t* nl;           // line ends (positions of '\n'), the first line_cap of them
};

// The 16 bytes of vector v (aligned addresses from a0) that lie in [text, text + n), as a mask of '\n' bytes.
__device__ __forceinline__ uint32_t nl_mask(const uint8_t* text, uint64_t n, uintptr_t a0, uint64_t v) {
    const uintptr_t a = a0 + 16 * v;
    const uintptr_t lo = (uintptr_t)text, hi = lo + n;
    if (a + 16 <= lo || a >= hi) return 0;
    const uint4 q = *(const uint4*)a;
    const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const uintptr_t p = a + k;
        if (p >= lo && p < hi && ((w4[k >> 2] >> (8 * (k & 3))) & 0xff) == '\n') m |= 1u << k;
    }
    return m;
}

__global__ void __launch_bounds__(NL_THREADS) nl_count_kernel(const uint8_t* text, uint64_t n, uintptr_t a0, uint64_t n_vec,
                                                              uint64_t* tile_count) {
    const uint64_t v = (uint64_t)blockIdx.x * NL_THREADS + threadIdx.x;
    const uint32_t c = v < n_vec ? __popc(nl_mask(text, n, a0, v)) : 0;
    typedef cub::BlockReduce<uint32_t, NL_THREADS> R;
    __shared__ typename R::TempStorage tmp;
    const uint32_t s = R(tmp).Sum(c);
    if (threadIdx.x == 0) tile_count[blockIdx.x] = s;
}

__global__ void __launch_bounds__(NL_THREADS) nl_write_kernel(const uint8_t* text, uint64_t n, uintptr_t a0, uint64_t n_vec,
                                                              const uint64_t* tile_off, uint64_t line_cap, uint64_t* nl) {
    const uint64_t v = (uint64_t)blockIdx.x * NL_THREADS + threadIdx.x;
    uint32_t m = v < n_vec ? nl_mask(text, n, a0, v) : 0;
    typedef cub::BlockScan<uint32_t, NL_THREADS> S;
    __shared__ typename S::TempStorage tmp;
    uint32_t before;
    S(tmp).ExclusiveSum(__popc(m), before);
    uint64_t idx = tile_off[blockIdx.x] + before;
    const int64_t base = (int64_t)(a0 + 16 * v) - (int64_t)(uintptr_t)text;
    for (; m && idx < line_cap; m &= m - 1, idx++) nl[idx] = (uint64_t)(base + __ffs(m) - 1);
}

__device__ __forceinline__ bool bad_byte(uint8_t c) { return c < '!' || c > '~'; }

// First position in [lo, hi) whose byte fails `bad` (hi when none), warp-cooperative.
template <typename F>
__device__ uint64_t warp_find(const uint8_t* t, uint64_t lo, uint64_t hi, uint32_t lane, F bad) {
    for (uint64_t b = lo; b < hi; b += 32) {
        const uint64_t p = b + lane;
        const uint32_t m = __ballot_sync(0xffffffffu, p < hi && bad(t[p]));
        if (m) return b + __ffs(m) - 1;
    }
    return hi;
}

// mode: 0 single, 1 interleaved, 2 two inputs (input `which` gives the reads 2r + which)
__global__ void __launch_bounds__(REC_WARPS * 32) fq_record_kernel(Input in, uint32_t which, uint32_t mode, uint64_t rec_cap,
                                                                   uint32_t max_reads, FqSum* sum, uint64_t* slen,
                                                                   uint64_t* nlen, uint64_t* err) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_rec = min(sum->n_lines[which] / 4, rec_cap);
    for (uint64_t r = (uint64_t)blockIdx.x * REC_WARPS + (threadIdx.x >> 5); r < n_rec; r += (uint64_t)gridDim.x * REC_WARPS) {
        const uint64_t read = mode == 2 ? 2 * r + which : r;
        if (read >= max_reads) continue;
        const uint8_t* t = in.text;
        const uint64_t s0 = r ? in.nl[4 * r - 1] + 1 : 0, e0 = in.nl[4 * r], e1 = in.nl[4 * r + 1], e2 = in.nl[4 * r + 2],
                       e3 = in.nl[4 * r + 3];
        uint32_t kind = FQ_OK;
        uint64_t at = 0;
        if (e0 == s0 || t[s0] != '@') { kind = FQ_HEADER; at = s0; }
        const uint64_t name_end = warp_find(t, s0 + 1, e0, lane,
                                            [](uint8_t c) { return c == ' ' || c == '\t' || c == '\v' || c == '\f' || c == '\r'; });
        if (!kind) { at = warp_find(t, e0 + 1, e1, lane, bad_byte); if (at < e1) kind = FQ_SEQ_BYTE; }
        if (!kind && (e2 == e1 + 1 || t[e1 + 1] != '+')) { kind = FQ_SEPARATOR; at = e1 + 1; }
        if (!kind && e3 - e2 != e1 - e0) { kind = FQ_QUAL_LEN; at = e2 + 1; }
        if (!kind) { at = warp_find(t, e2 + 1, e3, lane, bad_byte); if (at < e3) kind = FQ_QUAL_BYTE; }
        if (lane == 0) {
            slen[read] = e1 - e0 - 1;
            nlen[read] = kind == FQ_HEADER ? 0 : name_end - s0 - 1;
            if (kind) { err[read] = (uint64_t)kind << 56 | at; atomicMin(&sum->first_bad, (uint32_t)read); }
        }
    }
}

__device__ uint64_t records_of(const FqSum* s, uint32_t t, uint64_t rec_cap) { return min(s->n_lines[t] / 4, rec_cap); }

// The longest prefix of whole groups that fits, the status, and text_used.
__global__ void fq_finalize_kernel(Input in0, Input in1, uint32_t mode, uint64_t rec_cap, uint32_t max_reads, uint64_t bases_cap,
                                   uint64_t names_cap, const uint64_t* roff, const uint64_t* noff, const uint64_t* err, FqSum* s) {
    const uint32_t group = mode ? 2 : 1;
    const uint64_t c0 = records_of(s, 0, rec_cap), c1 = mode == 2 ? records_of(s, 1, rec_cap) : 0;
    const uint64_t reads_present = mode == 0 ? c0 : mode == 1 ? c0 & ~1ull : 2 * min(c0, c1);
    const uint64_t n_cand = min(reads_present, (uint64_t)(max_reads / group * group));
    uint64_t lo = 0, hi = n_cand / group;                  // groups: the largest k <= hi whose prefix fits
    while (lo < hi) {
        const uint64_t mid = (lo + hi + 1) / 2, n = mid * group;
        if (roff[n] <= bases_cap && noff[n] <= names_cap) lo = mid; else hi = mid - 1;
    }
    const uint64_t n_take = lo * group;
    s->status = 0;
    if (s->first_bad < n_cand && s->first_bad / group <= lo) {
        s->status = 1;
        s->err_kind = (uint32_t)(err[s->first_bad] >> 56);
        s->err_off = err[s->first_bad] & ((1ull << 56) - 1);
    } else if (n_take == 0 && reads_present > 0) {
        s->status = 2;
        if (max_reads < group) { s->need_kind = 0; s->need = group; }
        else if (roff[group] > bases_cap) { s->need_kind = 1; s->need = roff[group]; }
        else { s->need_kind = 2; s->need = noff[group]; }
    }
    s->n_take = (uint32_t)n_take;
    const uint64_t k = mode == 2 ? n_take / 2 : n_take;
    s->text_used[0] = k ? in0.nl[4 * k - 1] + 1 : 0;
    s->text_used[1] = mode == 2 && k ? in1.nl[4 * k - 1] + 1 : 0;
}

__global__ void fq_maxlen_kernel(const uint64_t* slen, FqSum* s) {
    const uint32_t n = s->n_take;
    uint32_t m = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        m = max(m, (uint32_t)slen[i]);
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0 && m) atomicMax(&s->max_len, m);
}

__global__ void __launch_bounds__(REC_WARPS * 32) fq_fill_kernel(Input in0, Input in1, uint32_t mode, const uint64_t* roff,
                                                                 const uint64_t* noff, const FqSum* s, uint8_t* reads, uint8_t* quals,
                                                                 uint64_t* read_off, uint8_t* names, uint64_t* name_off) {
    const uint32_t lane = threadIdx.x & 31, n = s->n_take;
    for (uint64_t i = (uint64_t)blockIdx.x * REC_WARPS + (threadIdx.x >> 5); i < n; i += (uint64_t)gridDim.x * REC_WARPS) {
        const Input& in = mode == 2 && (i & 1) ? in1 : in0;
        const uint64_t r = mode == 2 ? i / 2 : i;
        const uint8_t* t = in.text;
        const uint64_t s0 = r ? in.nl[4 * r - 1] + 1 : 0, e0 = in.nl[4 * r], e2 = in.nl[4 * r + 2];
        const uint64_t ro = roff[i], len = roff[i + 1] - ro, no = noff[i], nl = noff[i + 1] - no;
        for (uint64_t k = lane; k < nl; k += 32) names[no + k] = t[s0 + 1 + k];
        for (uint64_t k = lane; k < len; k += 32) {
            const uint8_t c = t[e0 + 1 + k];
            reads[ro + k] = c >= 'a' && c <= 'z' ? c - 32 : c;
            if (quals) quals[ro + k] = t[e2 + 1 + k] - 33;
        }
        if (lane == 0) {
            read_off[i] = ro; name_off[i] = no;
            if (i + 1 == n) { read_off[n] = roff[n]; name_off[n] = noff[n]; }
        }
    }
}

int fastq_parse_device(gb_device* d, uint32_t n_inputs, const uint8_t* const* d_text, const uint64_t* text_bytes, uint32_t flags,
                       int final, uint32_t max_reads, uint8_t* d_reads, uint8_t* d_quals, uint64_t bases_cap, uint64_t* d_read_off,
                       uint8_t* d_names, uint64_t names_cap, uint64_t* d_name_off, uint32_t* n_reads, uint32_t* max_read_len,
                       uint64_t* text_used) {
    if (!d || !d_text || !text_bytes || !n_reads || !max_read_len || !text_used || !d_read_off || !d_name_off ||
        (n_inputs != 1 && n_inputs != 2) || (flags & ~GB_FASTQ_INTERLEAVED) || (n_inputs == 2 && (flags & GB_FASTQ_INTERLEAVED)) ||
        (!d_reads && bases_cap) || (!d_names && names_cap) || max_reads == 0xffffffffu)
        return GB_ERR_ARG;
    for (uint32_t t = 0; t < n_inputs; t++)
        if (!d_text[t] && text_bytes[t]) return GB_ERR_ARG;
    *n_reads = 0; *max_read_len = 0;
    for (uint32_t t = 0; t < n_inputs; t++) text_used[t] = 0;
    GB_CUDA(cudaSetDevice(d->device));
    const uint32_t mode = n_inputs == 2 ? 2 : (flags & GB_FASTQ_INTERLEAVED) ? 1 : 0;
    // records of one input the call can look at: every one it could take, and the next (to report it when it is refused)
    const uint64_t rec_cap = mode == 2 ? max_reads / 2 + 1 : (uint64_t)max_reads + 2, line_cap = 4 * rec_cap;
    const uint64_t nr = (uint64_t)max_reads + 1;
    uint64_t n_tiles[2] = {0, 0};
    size_t scan_tiles = 0, scan_reads = 0;
    for (uint32_t t = 0; t < n_inputs; t++) {
        const uintptr_t a0 = (uintptr_t)d_text[t] & ~(uintptr_t)15;
        const uint64_t n_vec = text_bytes[t] ? ((uintptr_t)d_text[t] + text_bytes[t] - a0 + 15) / 16 : 0;
        n_tiles[t] = (n_vec + NL_THREADS - 1) / NL_THREADS;
        size_t b = 0;
        GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t)(n_tiles[t] + 1), d->stream));
        scan_tiles = std::max(scan_tiles, b);
    }
    GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_reads, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t)nr, d->stream));
    // workspace: summary, per input {tile counts, tile offsets, line ends}, per read {seq len, name len, error, offsets}, temp
    FqSum* sum;
    uint64_t *tc[2], *to[2], *nl[2], *slen, *nlen, *err, *roff, *noff;
    void* tmp;
    int rc = carve(d->fastq_ws, [&](Carve& c) {
        sum = c.take<FqSum>(1);
        for (uint32_t t = 0; t < 2; t++) {
            tc[t] = c.take<uint64_t>(n_tiles[t] + 1); to[t] = c.take<uint64_t>(n_tiles[t] + 1);
            nl[t] = t < n_inputs ? c.take<uint64_t>(line_cap) : nullptr;
        }
        slen = c.take<uint64_t>(nr); nlen = c.take<uint64_t>(nr); err = c.take<uint64_t>(nr); roff = c.take<uint64_t>(nr); noff = c.take<uint64_t>(nr);
        tmp = c.take<uint8_t>(std::max(scan_tiles, scan_reads));
    });
    if (rc) return rc;
    GB_CUDA(cudaMemsetAsync(sum, 0, sizeof(FqSum), d->stream));
    GB_CUDA(cudaMemsetAsync(&sum->first_bad, 0xff, sizeof(uint32_t), d->stream));
    GB_CUDA(cudaMemsetAsync(slen, 0, 8 * nr, d->stream));            // reads without a record scan as length 0
    GB_CUDA(cudaMemsetAsync(nlen, 0, 8 * nr, d->stream));
    Input in[2] = {};
    for (uint32_t t = 0; t < n_inputs; t++) {
        in[t] = Input{d_text[t], text_bytes[t], nl[t]};
        const uintptr_t a0 = (uintptr_t)d_text[t] & ~(uintptr_t)15;
        const uint64_t n_vec = text_bytes[t] ? ((uintptr_t)d_text[t] + text_bytes[t] - a0 + 15) / 16 : 0;
        GB_CUDA(cudaMemsetAsync(tc[t] + n_tiles[t], 0, 8, d->stream));
        if (n_tiles[t]) {
            nl_count_kernel<<<(uint32_t)n_tiles[t], NL_THREADS, 0, d->stream>>>(d_text[t], text_bytes[t], a0, n_vec, tc[t]);
            d->launches++;
            GB_CUDA(cudaGetLastError());
        }
        GB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, scan_tiles, tc[t], to[t], (int64_t)(n_tiles[t] + 1), d->stream));
        d->launches++;
        GB_CUDA(cudaMemcpyAsync(&sum->n_lines[t], to[t] + n_tiles[t], 8, cudaMemcpyDeviceToDevice, d->stream));
        if (n_tiles[t]) {
            nl_write_kernel<<<(uint32_t)n_tiles[t], NL_THREADS, 0, d->stream>>>(d_text[t], text_bytes[t], a0, n_vec, to[t], line_cap, nl[t]);
            d->launches++;
            GB_CUDA(cudaGetLastError());
        }
        const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((rec_cap + REC_WARPS - 1) / REC_WARPS, (uint64_t)d->n_sms * 8));
        fq_record_kernel<<<grid, REC_WARPS * 32, 0, d->stream>>>(in[t], t, mode, rec_cap, max_reads, sum, slen, nlen, err);
        d->launches++;
        GB_CUDA(cudaGetLastError());
    }
    GB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, scan_reads, slen, roff, (int64_t)nr, d->stream));
    GB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, scan_reads, nlen, noff, (int64_t)nr, d->stream));
    d->launches += 2;
    fq_finalize_kernel<<<1, 1, 0, d->stream>>>(in[0], in[1], mode, rec_cap, max_reads, bases_cap, names_cap, roff, noff, err, sum);
    const uint32_t rgrid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((nr + REC_WARPS - 1) / REC_WARPS, (uint64_t)d->n_sms * 8));
    fq_maxlen_kernel<<<(uint32_t)std::min<uint64_t>((nr + 255) / 256, (uint64_t)d->n_sms * 4), 256, 0, d->stream>>>(slen, sum);
    fq_fill_kernel<<<rgrid, REC_WARPS * 32, 0, d->stream>>>(in[0], in[1], mode, roff, noff, sum, d_reads, d_quals, d_read_off,
                                                            d_names, d_name_off);
    d->launches += 3;
    GB_CUDA(cudaGetLastError());
    FqSum h{};
    GB_CUDA(cudaMemcpyAsync(&h, sum, sizeof h, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));              // the one wait: how far the call got
    if (h.status == 1) {
        const uint32_t t = mode == 2 ? h.first_bad & 1 : 0;
        const uint64_t rec = mode == 2 ? h.first_bad / 2 : h.first_bad;
        static const char* what[] = {"", "the header does not start with '@'", "a sequence byte is outside '!'..'~'",
                                     "the separator line does not start with '+'",
                                     "the quality line's length differs from the sequence's", "a quality byte is outside '!'..'~'"};
        g_last_error = "gb_fastq_parse_device: input " + std::to_string(t) + ", record " + std::to_string(rec) + ", byte " +
                       std::to_string(h.err_off) + ": " + what[h.err_kind];
        return GB_ERR_FORMAT;
    }
    if (h.status == 2) {
        static const char* cap[] = {"max_reads", "bases_cap", "names_cap"};
        g_last_error = std::string("gb_fastq_parse_device: the first record") + (mode ? " pair" : "") + " needs " + cap[h.need_kind] +
                       " >= " + std::to_string(h.need);
        return GB_ERR_CAPACITY;
    }
    const uint64_t k = mode == 2 ? h.n_take / 2 : h.n_take;
    if (final) {
        // an input whose whole records were all taken must end with the last of them
        for (uint32_t t = 0; t < n_inputs; t++)
            if (k == h.n_lines[t] / 4 && h.text_used[t] < text_bytes[t]) {
                g_last_error = "gb_fastq_parse_device: input " + std::to_string(t) + ", record " + std::to_string(k) + ", byte " +
                               std::to_string(h.text_used[t]) + ": the input ends inside a record (every line must end with '\\n')";
                return GB_ERR_FORMAT;
            }
    }
    if (h.n_take == 0) {
        GB_CUDA(cudaMemsetAsync(d_read_off, 0, 8, d->stream));
        GB_CUDA(cudaMemsetAsync(d_name_off, 0, 8, d->stream));
    }
    *n_reads = h.n_take;
    *max_read_len = h.max_len;
    for (uint32_t t = 0; t < n_inputs; t++) text_used[t] = h.text_used[t];
    return GB_OK;
}

} // namespace
} // namespace gb

extern "C" int gb_fastq_parse_device(gb_device* dev, uint32_t n_inputs, const uint8_t* const* d_text, const uint64_t* text_bytes,
                                     uint32_t flags, int final, uint32_t max_reads, uint8_t* d_reads, uint8_t* d_quals,
                                     uint64_t bases_cap, uint64_t* d_read_off, uint8_t* d_names, uint64_t names_cap,
                                     uint64_t* d_name_off, uint32_t* n_reads, uint32_t* max_read_len, uint64_t* text_used) {
    return gb::guarded("gb_fastq_parse_device", [&] {
        return gb::fastq_parse_device(dev, n_inputs, d_text, text_bytes, flags, final, max_reads, d_reads, d_quals, bases_cap,
                                      d_read_off, d_names, names_cap, d_name_off, n_reads, max_read_len, text_used);
    });
}
