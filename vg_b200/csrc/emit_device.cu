// emit_device.cu — gb_emit_gaf_device / gb_emit_gam_device: GAF lines and GAM messages formatted on the GPU from records
// that are already in HBM, byte for byte what the host emitters in emit.cpp write for the same records.
//
// Count / scan / fill, one thread per record:
//   validate   every record against the rules of emit.cpp's records_valid, one flag for the whole batch
//   size       the exact bytes of each record (GAF: the line; GAM: the Alignment message)
//   scan       GAM: present records -> message index (group of 1000 and the place of its header); bytes -> offsets
//   fill       the bytes at the scanned offsets
// Sizing and filling run the SAME formatting code over two sinks (Count adds lengths, Write stores bytes), so the sizes
// cannot disagree with what is written.  GAM's nested length prefixes are found the same way: a sub-message's body is
// run over a Count sink before its tag and length are written (Edit -> Mapping -> Path -> Alignment, then the Struct).
// A thread formats its record straight into the output with byte stores; the lines are a few hundred bytes and the
// stores of a warp land in L2, which merges them before they reach HBM.
#include "giraffe_b200.h"
#include "device_state.cuh"

#include <cub/cub.cuh>

#include <algorithm>

namespace gb {
namespace {

constexpr uint32_t EMIT_BLOCK = 128;
constexpr uint32_t GAM_GROUP = 1000;             // messages per GAM group (emit.cpp)

struct EmitArgs {
    uint32_t n; const gb_alignment* aln;
    const gb_mapping* maps; uint64_t map_len; const uint32_t* edits; uint64_t edit_len;
    uint32_t n_reads; const uint8_t* reads; const uint8_t* quals; const uint64_t* read_off;
    const uint8_t* names; const uint64_t* name_off;          // names == NULL: read<i>
    const gb_node_rec* nodes; const uint8_t* seq; uint32_t n_nodes;
};

struct Count {
    static constexpr bool counting = true;
    uint64_t n = 0;
    __device__ void ch(char) { n++; }
    __device__ void put(const void*, uint64_t k) { n += k; }
};

struct Write {
    static constexpr bool counting = false;
    char* p;
    __device__ void ch(char c) { *p++ = c; }
    __device__ void put(const void* s, uint64_t k) { const char* c = (const char*)s; for (uint64_t i = 0; i < k; i++) p[i] = c[i]; p += k; }
};

template <class S, size_t N> __device__ __forceinline__ void lit(S& s, const char (&t)[N]) { s.put(t, N - 1); }

template <class S> __device__ void unum(S& s, uint64_t v) {
    char t[20]; int k = 0;
    do { t[k++] = (char)('0' + v % 10); v /= 10; } while (v);
    if constexpr (S::counting) s.n += k;
    else while (k) s.ch(t[--k]);
}
template <class S> __device__ void snum(S& s, int64_t v) {
    if (v < 0) s.ch('-');
    unum(s, v < 0 ? 0 - (uint64_t)v : (uint64_t)v);
}

__device__ __forceinline__ uint32_t varint_len(uint64_t v) { uint32_t k = 1; while (v >= 0x80) { v >>= 7; k++; } return k; }
template <class S> __device__ void varint(S& s, uint64_t v) {
    if constexpr (S::counting) s.n += varint_len(v);
    else { while (v >= 0x80) { s.ch((char)(v | 0x80)); v >>= 7; } s.ch((char)v); }
}

__device__ __forceinline__ uint32_t edit_len(uint32_t wd) { return (wd & 3u) == GB_EDIT_SUB ? 1u : wd >> 4; }

// ---- glibc "%.6g" of a double in [0, 1], exactly --------------------------------------------------------------------
// v = M / 2^sh with M < 2^53.  The digits are round-half-even(v * 10^k) for the k that leaves six of them, computed in
// 128-bit integers: no rounding happens before the one the format asks for.  The GAF dv values are 1 - m / b of
// doubles, which lie on the 2^-53 grid (x >= 0.5: 1 - x is exact; x < 0.5: v >= 0.5), so sh <= 106 and v * 10^k, k <= 21,
// stays below 2^124.
template <class S> __device__ void g6(S& s, double v) {
    if (v == 0.0) { s.ch('0'); return; }
    int e;
    const double f = frexp(v, &e);
    const uint64_t M = (uint64_t)ldexp(f, 53);
    const int sh = 53 - e;
    typedef unsigned __int128 u128;
    u128 p10 = 100000; int k = 5;
    while ((((u128)M * p10) >> sh) < 100000) { p10 *= 10; k++; }
    const u128 N = (u128)M * p10;
    uint64_t D = (uint64_t)(N >> sh);
    const u128 rem = N & ((((u128)1) << sh) - 1), half = ((u128)1) << (sh - 1);
    if (rem > half || (rem == half && (D & 1))) D++;
    if (D == 1000000) { D = 100000; k--; }
    const int X = 5 - k;                                 // decimal exponent of the first digit
    char dg[6];
    for (int i = 5; i >= 0; i--) { dg[i] = (char)('0' + D % 10); D /= 10; }
    int nd = 6;
    while (nd > 1 && dg[nd - 1] == '0') nd--;           // %g drops trailing zeros (and a bare point)
    if (X < -4 || X >= 6) {
        s.ch(dg[0]);
        if (nd > 1) { s.ch('.'); s.put(dg + 1, nd - 1); }
        s.ch('e'); s.ch(X < 0 ? '-' : '+');
        const int ax = X < 0 ? -X : X;
        if (ax < 10) s.ch('0');
        unum(s, (uint64_t)ax);
    } else if (X >= 0) {
        s.put(dg, X + 1);
        if (nd > X + 1) { s.ch('.'); s.put(dg + X + 1, nd - X - 1); }
    } else {
        s.ch('0'); s.ch('.');
        for (int i = 0; i < -X - 1; i++) s.ch('0');
        s.put(dg, nd);
    }
}

// ---- records --------------------------------------------------------------------------------------------------------
__device__ bool record_valid(const EmitArgs& A, const gb_alignment& a) {
    if (a.read_id >= A.n_reads || A.read_off[a.read_id + 1] < A.read_off[a.read_id]) return false;
    if ((a.flags & GB_ALN_PAIRED) && (a.read_id ^ 1u) >= A.n_reads) return false;
    if (!(a.flags & GB_ALN_MAPPED) || a.n_mappings == 0) return true;
    if (!A.maps || !A.edits || (uint64_t)a.mapping_off + a.n_mappings > A.map_len || (uint64_t)a.edit_off + a.n_edits > A.edit_len) return false;
    const uint64_t L = A.read_off[a.read_id + 1] - A.read_off[a.read_id];
    uint64_t ei = 0, q = 0;
    for (uint32_t i = 0; i < a.n_mappings; i++) {
        const gb_mapping m = A.maps[a.mapping_off + i];
        if (m.node >= A.n_nodes || ei + m.n_edits > a.n_edits) return false;
        uint64_t off = m.offset;
        for (uint32_t j = 0; j < m.n_edits; j++, ei++) {
            const uint32_t wd = A.edits[a.edit_off + ei], op = wd & 3u, len = edit_len(wd);
            if (op != GB_EDIT_DEL) q += len;
            if (op != GB_EDIT_INS) off += len;
        }
        if (off > A.nodes[m.node].len || q > L) return false;
    }
    return ei == a.n_edits && q == L;
}

__device__ __forceinline__ bool use_names(const EmitArgs& A) { return A.names && A.name_off; }
__device__ uint64_t name_len(const EmitArgs& A, uint32_t r) {
    if (use_names(A)) return A.name_off[r + 1] - A.name_off[r];
    Count c; unum(c, r); return 4 + c.n;
}
template <class S> __device__ void name(S& s, const EmitArgs& A, uint32_t r) {
    if (use_names(A)) s.put(A.names + A.name_off[r], A.name_off[r + 1] - A.name_off[r]);
    else { lit(s, "read"); unum(s, r); }
}

// One GAF line (emit.cpp gb_emit_gaf_impl).
template <class S> __device__ void gaf_record(S& s, const EmitArgs& A, const gb_alignment& a) {
    const uint32_t r = a.read_id;
    const uint8_t* seq = A.reads + A.read_off[r];
    const uint32_t L = (uint32_t)(A.read_off[r + 1] - A.read_off[r]);
    name(s, A, r); s.ch('\t'); unum(s, L); s.ch('\t');
    if (!(a.flags & GB_ALN_MAPPED) || a.n_mappings == 0) {
        lit(s, "0\t"); unum(s, L); lit(s, "\t*\t*\t*\t*\t*\t*\t*\t255");
        lit(s, "\tcs:Z:+"); s.put(seq, L);
    } else {
        const gb_mapping* m = A.maps + a.mapping_off;
        const uint32_t* e = A.edits + a.edit_off;
        uint64_t path_len = 0, matches = 0, block = 0, ref_used = 0, pstart = 0;
        bool have_start = false;
        for (uint32_t i = 0, ei = 0; i < a.n_mappings; i++) {
            const gb_mapping mi = m[i];
            bool uses_node = false;
            for (uint32_t j = 0; j < mi.n_edits; j++, ei++) {
                const uint32_t wd = e[ei], op = wd & 3u, len = edit_len(wd);
                uses_node |= op != GB_EDIT_INS;
                if (op == GB_EDIT_MATCH) matches += len;
                block += len;
                if (op != GB_EDIT_INS) ref_used += len;
            }
            if (uses_node) {
                path_len += A.nodes[mi.node].len;
                if (!have_start) { pstart = mi.offset; have_start = true; }
            }
        }
        lit(s, "0\t"); unum(s, L); lit(s, "\t+\t");
        if (!have_start) s.ch('*');
        else for (uint32_t i = 0, ei = 0; i < a.n_mappings; i++) {          // mappings that only insert are left out
            const gb_mapping mi = m[i];
            bool uses_node = false;
            for (uint32_t j = 0; j < mi.n_edits; j++, ei++) uses_node |= (e[ei] & 3u) != GB_EDIT_INS;
            if (uses_node) { s.ch((mi.node & 1u) ? '<' : '>'); unum(s, mi.node >> 1); }
        }
        s.ch('\t'); unum(s, path_len); s.ch('\t'); unum(s, pstart); s.ch('\t'); unum(s, pstart + ref_used); s.ch('\t');
        unum(s, matches); s.ch('\t'); unum(s, block); s.ch('\t'); unum(s, a.mapq);
        lit(s, "\tAS:i:"); snum(s, a.score);
        if (A.quals) {
            lit(s, "\tbq:Z:");
            const uint8_t* qv = A.quals + A.read_off[r];
            if constexpr (S::counting) s.n += L;
            else for (uint32_t t = 0; t < L; t++) s.ch((char)(qv[t] + 33));
        }
        lit(s, "\tcs:Z:");
        uint32_t q = 0, run = 0;
        for (uint32_t i = 0, ei = 0; i < a.n_mappings; i++) {
            const gb_mapping mi = m[i];
            const uint8_t* ref = A.seq + A.nodes[mi.node].seq_off;
            uint32_t off = mi.offset;
            for (uint32_t j = 0; j < mi.n_edits; j++, ei++) {
                const uint32_t wd = e[ei], op = wd & 3u, len = edit_len(wd);
                if (op == GB_EDIT_MATCH) { run += len; q += len; off += len; continue; }
                if (run) { s.ch(':'); unum(s, run); run = 0; }             // match runs merge across edits and mappings
                if (op == GB_EDIT_SUB) { s.ch('*'); s.ch((char)ref[off]); s.ch((char)seq[q]); q += 1; off += 1; }
                else if (op == GB_EDIT_INS) { s.ch('+'); s.put(seq + q, len); q += len; }
                else { s.ch('-'); s.put(ref + off, len); off += len; }
            }
        }
        if (run) { s.ch(':'); unum(s, run); }
        lit(s, "\tdv:f:");
        // 1.0 - matches / block in IEEE double, each operation rounded on its own (no contraction)
        g6(s, block ? __dsub_rn(1.0, __ddiv_rn((double)matches, (double)block)) : 0.0);
    }
    if (a.flags & GB_ALN_PAIRED) {
        if ((r & 1u) == 0) { lit(s, "\tfn:Z:"); name(s, A, r + 1); }
        else { lit(s, "\tfp:Z:"); name(s, A, r - 1); }
    }
    s.ch('\n');
}

// ---- protobuf (emit.cpp pb_*): proto3, zero / false fields are not written ------------------------------------------
template <class S> __device__ __forceinline__ void pb_tag(S& s, uint32_t field, uint32_t wire) { varint(s, ((uint64_t)field << 3) | wire); }
template <class S> __device__ void pb_uint(S& s, uint32_t field, uint64_t v) { if (v) { pb_tag(s, field, 0); varint(s, v); } }
template <class S> __device__ void pb_bytes(S& s, uint32_t field, const void* p, uint64_t n) { pb_tag(s, field, 2); varint(s, n); s.put(p, n); }
template <class S> __device__ void pb_double(S& s, uint32_t field, double v) {
    pb_tag(s, field, 1);
    const uint64_t b = (uint64_t)__double_as_longlong(v);
    if constexpr (S::counting) s.n += 8;
    else for (int i = 0; i < 8; i++) s.ch((char)(b >> (8 * i)));
}
// a length-delimited sub-message: its body runs over a Count sink for the length, then over s
template <class S, class F> __device__ void pb_msg(S& s, uint32_t field, const F& body) {
    Count c; body(c);
    pb_tag(s, field, 2); varint(s, c.n);
    if constexpr (S::counting) s.n += c.n;
    else body(s);
}
template <class S, class F> __device__ void pb_annotation(S& st, const char* key, uint32_t key_len, const F& value) {
    pb_msg(st, 1, [&](auto& entry) { pb_bytes(entry, 1, key, key_len); pb_msg(entry, 2, value); });
}

// One vg.proto Alignment message (emit.cpp gb_emit_gam_impl), without its length prefix.
template <class S> __device__ void gam_message(S& s, const EmitArgs& A, const gb_alignment& a) {
    const uint32_t r = a.read_id;
    const uint8_t* seq = A.reads + A.read_off[r];
    const uint32_t L = (uint32_t)(A.read_off[r + 1] - A.read_off[r]);
    pb_bytes(s, 1, seq, L);
    uint64_t matches = 0;
    if ((a.flags & GB_ALN_MAPPED) && a.n_mappings) {
        const gb_mapping* m = A.maps + a.mapping_off;
        const uint32_t* e = A.edits + a.edit_off;
        for (uint32_t k = 0; k < a.n_edits; k++) if ((e[k] & 3u) == GB_EDIT_MATCH) matches += e[k] >> 4;
        pb_msg(s, 2, [&](auto& path) {
            uint32_t q = 0, ei = 0;
            for (uint32_t i = 0; i < a.n_mappings; i++) {
                const gb_mapping mi = m[i];
                const uint32_t* me = e + ei;
                const uint8_t* mq = seq + q;
                pb_msg(path, 2, [&](auto& mp) {
                    pb_msg(mp, 1, [&](auto& pos) { pb_uint(pos, 1, mi.node >> 1); pb_uint(pos, 2, mi.offset); pb_uint(pos, 4, mi.node & 1u); });
                    uint32_t mq_off = 0;
                    for (uint32_t j = 0; j < mi.n_edits; j++) {
                        const uint32_t wd = me[j], op = wd & 3u, len = edit_len(wd);
                        const uint8_t* eq = mq + mq_off;
                        pb_msg(mp, 2, [&](auto& ed) {
                            if (op == GB_EDIT_MATCH) { pb_uint(ed, 1, len); pb_uint(ed, 2, len); }
                            else if (op == GB_EDIT_SUB) { pb_uint(ed, 1, 1); pb_uint(ed, 2, 1); pb_bytes(ed, 3, eq, 1); }
                            else if (op == GB_EDIT_INS) { pb_uint(ed, 2, len); pb_bytes(ed, 3, eq, len); }
                            else pb_uint(ed, 1, len);
                        });
                        if (op != GB_EDIT_DEL) mq_off += len;
                    }
                    pb_uint(mp, 5, i + 1);
                });
                for (uint32_t j = 0; j < mi.n_edits; j++, ei++) if ((e[ei] & 3u) != GB_EDIT_DEL) q += edit_len(e[ei]);
            }
        });
    }
    pb_tag(s, 3, 2); varint(s, name_len(A, r)); name(s, A, r);
    if (A.quals && L) pb_bytes(s, 4, A.quals + A.read_off[r], L);
    pb_uint(s, 5, a.mapq);
    pb_uint(s, 6, (uint64_t)(int64_t)a.score);                 // a negative int32 is a sign-extended 10-byte varint
    if (a.flags & GB_ALN_PAIRED) {
        const uint32_t mate = r ^ 1u;
        pb_msg(s, (r & 1u) ? 11 : 12, [&](auto& frag) { pb_tag(frag, 3, 2); varint(frag, name_len(A, mate)); name(frag, A, mate); });
    }
    if (a.flags & GB_ALN_SECONDARY) pb_uint(s, 15, 1);
    if ((a.flags & GB_ALN_MAPPED) && L) pb_double(s, 16, __ddiv_rn((double)matches, (double)L));
    const double uncapped = a.mapq_uncapped, cap = a.mapq_explored_cap;
    const bool rescued = (a.flags & GB_ALN_RESCUED) != 0;
    pb_msg(s, 100, [&](auto& st) {
        pb_annotation(st, "mapq_uncapped", 13, [&](auto& v) { pb_double(v, 2, uncapped); });
        pb_annotation(st, "mapq_explored_cap", 17, [&](auto& v) { pb_double(v, 2, cap); });
        if (rescued) pb_annotation(st, "rescued", 7, [&](auto& v) { pb_tag(v, 4, 0); varint(v, 1); });
    });
}

// varint(n + 1) varint(3) "GAM": the header of a group of n messages
__device__ __forceinline__ uint64_t gam_header_len(uint32_t n) { return varint_len((uint64_t)n + 1) + 1 + 3; }

// ---- kernels --------------------------------------------------------------------------------------------------------
__global__ void emit_validate_kernel(EmitArgs A, uint32_t* bad) {
    const uint32_t total = max(A.n, A.n_reads);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        bool ok = true;
        if (i < A.n_reads && use_names(A) && A.name_off[i + 1] < A.name_off[i]) ok = false;      // names are addressed like reads
        if (ok && i < A.n) ok = record_valid(A, A.aln[i]);
        if (!ok) *bad = 1u;
    }
}

// bytes[x] = the record's line (GAF) or message (GAM), 0 for an absent rank; present[x] (GAM) = 1 for a written record.
// Nothing is formatted when the batch was refused: the records may point anywhere.
template <bool GAM>
__global__ void emit_size_kernel(EmitArgs A, const uint32_t* bad, uint64_t* bytes, uint32_t* present) {
    const bool refused = *bad != 0;
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x <= A.n; x += gridDim.x * blockDim.x) {
        uint64_t sz = 0; uint32_t pr = 0;
        if (x < A.n && !refused) {
            const gb_alignment a = A.aln[x];
            if (!(a.flags & GB_ALN_ABSENT)) {
                Count c;
                if (GAM) gam_message(c, A, a); else gaf_record(c, A, a);
                sz = c.n; pr = 1;
            }
        }
        bytes[x] = sz;
        if (GAM) present[x] = pr;
    }
}

// GAM: a record's bytes in the stream = its group header when it opens a group + varint(message length) + message.
__global__ void gam_frame_kernel(uint32_t n, const uint64_t* msg, const uint32_t* pidx, uint64_t* framed) {
    const uint32_t np = pidx[n];
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x <= n; x += gridDim.x * blockDim.x) {
        uint64_t t = 0;
        if (x < n && pidx[x + 1] > pidx[x]) {
            const uint32_t p = pidx[x];
            t = varint_len(msg[x]) + msg[x];
            if (p % GAM_GROUP == 0) t += gam_header_len(min(GAM_GROUP, np - p));
        }
        framed[x] = t;
    }
}

template <bool GAM>
__global__ void emit_fill_kernel(EmitArgs A, const uint64_t* msg, const uint32_t* pidx, const uint64_t* off, char* out) {
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < A.n; x += gridDim.x * blockDim.x) {
        const gb_alignment a = A.aln[x];
        if (a.flags & GB_ALN_ABSENT) continue;
        Write w{out + off[x]};
        if (GAM) {
            const uint32_t p = pidx[x];
            if (p % GAM_GROUP == 0) { varint(w, (uint64_t)min(GAM_GROUP, pidx[A.n] - p) + 1); varint(w, 3); lit(w, "GAM"); }
            varint(w, msg[x]);
            gam_message(w, A, a);
        } else {
            gaf_record(w, A, a);
        }
    }
}

template <bool GAM>
int emit_device(gb_device* d, uint32_t n, const gb_alignment* d_aln, const gb_mapping* d_mappings, uint64_t mapping_pool_len,
                const uint32_t* d_edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals,
                const uint64_t* d_read_off, const uint8_t* d_names, const uint64_t* d_name_off, char* d_out, uint64_t out_cap, uint64_t* out_used) {
    if (!d || !d_aln || !d_reads || !d_read_off || !d_out || !out_used) return GB_ERR_ARG;
    if (n == 0xffffffffu) return GB_ERR_ARG;                 // the scans run over n + 1 entries
    GB_CUDA(cudaSetDevice(d->device));
    EmitArgs A;
    A.n = n; A.aln = d_aln; A.maps = d_mappings; A.map_len = mapping_pool_len; A.edits = d_edits; A.edit_len = edit_pool_len;
    A.n_reads = n_reads; A.reads = d_reads; A.quals = d_quals; A.read_off = d_read_off; A.names = d_names; A.name_off = d_name_off;
    A.nodes = d->ix.nodes; A.seq = d->ix.seq; A.n_nodes = d->ix.n_nodes;

    // workspace: status {refused, total bytes}, bytes[n + 1], framed[n + 1] (GAM), off[n + 1], present / pidx[n + 1] (GAM), scan temp
    const size_t m = (size_t)n + 1;
    size_t scan64 = 0, scan32 = 0;
    GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan64, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t)m, d->stream));
    GB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan32, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)m, d->stream));
    size_t tb = std::max(scan64, scan32);
    uint64_t *status, *bytes, *framed, *off;
    uint32_t *present, *pidx;
    void* tmp;
    int rc = carve(d->emit_ws, [&](Carve& c) {
        status = c.take<uint64_t>(2); bytes = c.take<uint64_t>(m); framed = GAM ? c.take<uint64_t>(m) : bytes; off = c.take<uint64_t>(m);
        present = GAM ? c.take<uint32_t>(m) : nullptr; pidx = GAM ? c.take<uint32_t>(m) : nullptr; tmp = c.take<uint8_t>(tb);
    });
    if (rc) return rc;

    const uint32_t grid = (uint32_t)std::min<uint64_t>((m + EMIT_BLOCK - 1) / EMIT_BLOCK, (uint64_t)d->n_sms * 64);
    const uint32_t vgrid = (uint32_t)std::min<uint64_t>(((uint64_t)std::max(n, n_reads) + EMIT_BLOCK) / EMIT_BLOCK, (uint64_t)d->n_sms * 64);
    GB_CUDA(cudaMemsetAsync(status, 0, 2 * sizeof(uint64_t), d->stream));
    emit_validate_kernel<<<vgrid, EMIT_BLOCK, 0, d->stream>>>(A, (uint32_t*)status);
    emit_size_kernel<GAM><<<grid, EMIT_BLOCK, 0, d->stream>>>(A, (const uint32_t*)status, bytes, present);
    d->launches += 2;
    GB_CUDA(cudaGetLastError());
    if (GAM) {
        GB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, present, pidx, (int64_t)m, d->stream));
        gam_frame_kernel<<<grid, EMIT_BLOCK, 0, d->stream>>>(n, bytes, pidx, framed);
        d->launches += 2;
        GB_CUDA(cudaGetLastError());
    }
    GB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, framed, off, (int64_t)m, d->stream));
    d->launches++;
    GB_CUDA(cudaMemcpyAsync(status + 1, off + n, sizeof(uint64_t), cudaMemcpyDeviceToDevice, d->stream));
    uint64_t h_status[2];
    GB_CUDA(cudaMemcpyAsync(h_status, status, sizeof h_status, cudaMemcpyDeviceToHost, d->stream));
    GB_CUDA(cudaStreamSynchronize(d->stream));              // the one wait: the total decides whether the fill runs
    if (h_status[0] & 0xffffffffull) { g_last_error = GAM ? "gb_emit_gam_device: a record points outside its read, pools or the graph"
                                                          : "gb_emit_gaf_device: a record points outside its read, pools or the graph"; return GB_ERR_ARG; }
    const uint64_t total = h_status[1];
    *out_used = total;
    if (total > out_cap) { g_last_error = "gb_emit_*_device: output capacity too small (*out_used holds the bytes needed)"; return GB_ERR_CAPACITY; }
    if (n) {
        emit_fill_kernel<GAM><<<grid, EMIT_BLOCK, 0, d->stream>>>(A, bytes, pidx, off, d_out);
        d->launches++;
        GB_CUDA(cudaGetLastError());
    }
    return GB_OK;
}

} // namespace
} // namespace gb

#define GB_EMIT_DEVICE_ENTRY(NAME, GAM)                                                                                            \
    extern "C" int NAME(gb_device* dev, uint32_t n, const gb_alignment* d_aln, const gb_mapping* d_mappings, uint64_t mapping_pool_len, \
                        const uint32_t* d_edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* d_reads, const uint8_t* d_quals,  \
                        const uint64_t* d_read_off, const uint8_t* d_names, const uint64_t* d_name_off, char* d_out, uint64_t out_cap,        \
                        uint64_t* out_used) {                                                                                              \
        return gb::guarded(#NAME, [&] { return gb::emit_device<GAM>(dev, n, d_aln, d_mappings, mapping_pool_len, d_edits, edit_pool_len, n_reads, \
                                                                    d_reads, d_quals, d_read_off, d_names, d_name_off, d_out, out_cap, out_used); }); \
    }
GB_EMIT_DEVICE_ENTRY(gb_emit_gaf_device, false)
GB_EMIT_DEVICE_ENTRY(gb_emit_gam_device, true)
