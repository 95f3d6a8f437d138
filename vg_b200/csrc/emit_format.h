// emit_format.h — the GAF line and the GAM message of one alignment record, and the check a record must pass before either
// is formatted.  emit.cpp (gb_emit_gaf / gb_emit_gam, plain C++) and emit_device.cu (gb_emit_gaf_device / gb_emit_gam_device)
// both run this code, so the host and the device write the same bytes for the same records.
//
// Every formatter runs over a sink: Count adds up lengths, Write stores bytes.  A caller counts a record first and writes it
// where it fits, so a size cannot disagree with what is written.  GAM's nested length prefixes are found the same way: a
// sub-message's body runs over a Count sink before its tag and length are written.
//
// GAF: the text format `vg giraffe -o gaf` writes (alignment_to_gaf lives in libvgio @ d029989, ABSENT from the reference
// tree).  Columns follow the published GAF specification and minimap2's cs difference string: ":n" matches, "*RQ"
// substitution, "+Q" insertion, "-R" deletion.  The conventions the reference's own tests fix (unittest/alignment.cpp:398-470,
// :793-820) are followed: the query interval is the whole read (soft clips stay in cs as insertions), cs bases are upper case,
// match runs merge across edits and mappings, a mapping that only carries an insertion (a soft clip parked on an unused node)
// is left out of the path, and an unaligned read has an empty path ('*') and cs "+<read>".
//
// GAM: vg.proto Alignment messages in vg::io's group framing.  libvgio is absent from the reference tree; the wire layout is
// read off GAM files vg itself wrote, kept as fixtures in tests/golden/gam/ (test/surject/perpendicular.gam is Giraffe output):
//   stream    groups of [varint n] [varint 3]["GAM"] then n-1 x [varint len][Alignment]      (type-tagged groups)
//   Alignment 1 sequence, 2 path, 3 name, 4 quality (raw phred bytes), 5 mapping_quality, 6 score,
//             11 fragment_prev / 12 fragment_next (an Alignment carrying only 3 name), 15 is_secondary, 16 identity (double),
//             100 annotation (google.protobuf.Struct: 1 fields{1 key, 2 Value{2 number_value, 4 bool_value}})
//   Path      2 mapping;   Mapping 1 position, 2 edit, 5 rank;   Position 1 node_id, 2 offset, 4 is_reverse;
//   Edit      1 from_length, 2 to_length, 3 sequence.   proto3: zero / false / empty fields are not written.
// The stream is written uncompressed: vg::io's BlockedGzipInputStream reads uncompressed, gzip and BGZF data alike
// (unittest/blocked_gzip_input_stream.cpp:136, :364, :400).
//
// Plain C++ without CUDA as well: the host sanitizer build compiles emit.cpp with g++ alone.  Everything here has internal
// linkage, so the g++ and the nvcc copies of a function never meet at link time.
#pragma once
#include "giraffe_b200.h"

#include <cmath>
#include <cstdint>
#include <cstring>

#ifdef __CUDACC__
#define GB_FMT __host__ __device__
#define GB_FMT_INLINE __host__ __device__ __forceinline__
#else
#define GB_FMT inline
#define GB_FMT_INLINE inline
#endif

namespace gb {
namespace {

constexpr uint32_t GAM_GROUP = 1000;             // messages per GAM group

// One call's records, reads, names and graph, all in the memory of the side that formats them.
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
    GB_FMT void ch(char) { n++; }
    GB_FMT void put(const void*, uint64_t k) { n += k; }
};

struct Write {
    static constexpr bool counting = false;
    char* p;
    GB_FMT void ch(char c) { *p++ = c; }
    GB_FMT void put(const void* s, uint64_t k) { const char* c = (const char*)s; for (uint64_t i = 0; i < k; i++) p[i] = c[i]; p += k; }
};

template <class S, size_t N> GB_FMT_INLINE void lit(S& s, const char (&t)[N]) { s.put(t, N - 1); }

template <class S> GB_FMT void unum(S& s, uint64_t v) {
    char t[20]; int k = 0;
    do { t[k++] = (char)('0' + v % 10); v /= 10; } while (v);
    if constexpr (S::counting) s.n += k;
    else while (k) s.ch(t[--k]);
}
template <class S> GB_FMT void snum(S& s, int64_t v) {
    if (v < 0) s.ch('-');
    unum(s, v < 0 ? 0 - (uint64_t)v : (uint64_t)v);
}

GB_FMT_INLINE uint32_t varint_len(uint64_t v) { uint32_t k = 1; while (v >= 0x80) { v >>= 7; k++; } return k; }
template <class S> GB_FMT void varint(S& s, uint64_t v) {
    if constexpr (S::counting) s.n += varint_len(v);
    else { while (v >= 0x80) { s.ch((char)(v | 0x80)); v >>= 7; } s.ch((char)v); }
}

GB_FMT_INLINE uint32_t edit_len(uint32_t wd) { return (wd & 3u) == GB_EDIT_SUB ? 1u : wd >> 4; }

// ---- glibc "%.6g" of a double in [0, 1], exactly --------------------------------------------------------------------
// v = M / 2^sh with M < 2^53.  The digits are round-half-even(v * 10^k) for the k that leaves six of them, computed in
// 128-bit integers: no rounding happens before the one the format asks for.  The GAF dv values are 1 - m / b of
// doubles, which lie on the 2^-53 grid (x >= 0.5: 1 - x is exact; x < 0.5: v >= 0.5), so sh <= 106 and v * 10^k, k <= 21,
// stays below 2^124.
template <class S> GB_FMT void g6(S& s, double v) {
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

// ---- the record check -----------------------------------------------------------------------------------------------
// Every record must stay inside what the caller handed over: its read, its slice of the two pools, the graph, and the
// read length its edits consume.  The formatters index with these fields, so a batch with one damaged record is refused.
GB_FMT bool record_valid(const EmitArgs& A, const gb_alignment& a) {
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

GB_FMT_INLINE bool use_names(const EmitArgs& A) { return A.names && A.name_off; }
// names are addressed like reads: n_reads + 1 non-decreasing offsets
GB_FMT_INLINE bool name_valid(const EmitArgs& A, uint32_t r) { return !use_names(A) || A.name_off[r + 1] >= A.name_off[r]; }

GB_FMT uint64_t name_len(const EmitArgs& A, uint32_t r) {
    if (use_names(A)) return A.name_off[r + 1] - A.name_off[r];
    Count c; unum(c, r); return 4 + c.n;
}
template <class S> GB_FMT void name(S& s, const EmitArgs& A, uint32_t r) {
    if (use_names(A)) s.put(A.names + A.name_off[r], A.name_off[r + 1] - A.name_off[r]);
    else { lit(s, "read"); unum(s, r); }
}

// ---- GAF ------------------------------------------------------------------------------------------------------------
// One GAF line, its newline included.
template <class S> GB_FMT void gaf_record(S& s, const EmitArgs& A, const gb_alignment& a) {
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
        // IEEE double, each operation rounded on its own: a subtraction of a quotient cannot be contracted
        g6(s, block ? 1.0 - (double)matches / (double)block : 0.0);
    }
    if (a.flags & GB_ALN_PAIRED) {
        // mates are interleaved: fragment_next on mate 1, fragment_prev on mate 2 (pair_all, minimizer_mapper.cpp:1280-1300)
        if ((r & 1u) == 0) { lit(s, "\tfn:Z:"); name(s, A, r + 1); }
        else { lit(s, "\tfp:Z:"); name(s, A, r - 1); }
    }
    s.ch('\n');
}

// ---- GAM ------------------------------------------------------------------------------------------------------------
template <class S> GB_FMT_INLINE void pb_tag(S& s, uint32_t field, uint32_t wire) { varint(s, ((uint64_t)field << 3) | wire); }
template <class S> GB_FMT void pb_uint(S& s, uint32_t field, uint64_t v) { if (v) { pb_tag(s, field, 0); varint(s, v); } }
template <class S> GB_FMT void pb_bytes(S& s, uint32_t field, const void* p, uint64_t n) { pb_tag(s, field, 2); varint(s, n); s.put(p, n); }
template <class S> GB_FMT void pb_double(S& s, uint32_t field, double v) {
    pb_tag(s, field, 1);
    uint64_t b;
    memcpy(&b, &v, 8);
    if constexpr (S::counting) s.n += 8;
    else for (int i = 0; i < 8; i++) s.ch((char)(b >> (8 * i)));
}
// a length-delimited sub-message: its body runs over a Count sink for the length, then over s
template <class S, class F> GB_FMT void pb_msg(S& s, uint32_t field, const F& body) {
    Count c; body(c);
    pb_tag(s, field, 2); varint(s, c.n);
    if constexpr (S::counting) s.n += c.n;
    else body(s);
}
template <class S, class F> GB_FMT void pb_annotation(S& st, const char* key, uint32_t key_len, const F& value) {
    pb_msg(st, 1, [&](auto& entry) { pb_bytes(entry, 1, key, key_len); pb_msg(entry, 2, value); });
}

// One vg.proto Alignment message, without its length prefix.
template <class S> GB_FMT void gam_message(S& s, const EmitArgs& A, const gb_alignment& a) {
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
    pb_uint(s, 6, (uint64_t)(int64_t)a.score);                 // proto3 int32: a negative value is a sign-extended 10-byte varint
    if (a.flags & GB_ALN_PAIRED) {
        const uint32_t mate = r ^ 1u;
        pb_msg(s, (r & 1u) ? 11 : 12, [&](auto& frag) { pb_tag(frag, 3, 2); varint(frag, name_len(A, mate)); name(frag, A, mate); });
    }
    if (a.flags & GB_ALN_SECONDARY) pb_uint(s, 15, 1);
    if ((a.flags & GB_ALN_MAPPED) && L) pb_double(s, 16, (double)matches / (double)L);
    const double uncapped = a.mapq_uncapped, cap = a.mapq_explored_cap;
    const bool rescued = (a.flags & GB_ALN_RESCUED) != 0;
    pb_msg(s, 100, [&](auto& st) {
        pb_annotation(st, "mapq_uncapped", 13, [&](auto& v) { pb_double(v, 2, uncapped); });
        pb_annotation(st, "mapq_explored_cap", 17, [&](auto& v) { pb_double(v, 2, cap); });
        if (rescued) pb_annotation(st, "rescued", 7, [&](auto& v) { pb_tag(v, 4, 0); varint(v, 1); });
    });
}

// varint(n + 1) varint(3) "GAM": the header of a group of n messages
GB_FMT_INLINE uint64_t gam_header_len(uint32_t n) { return varint_len((uint64_t)n + 1) + 1 + 3; }
template <class S> GB_FMT_INLINE void gam_header(S& s, uint32_t n) { varint(s, (uint64_t)n + 1); varint(s, 3); lit(s, "GAM"); }

} // namespace
} // namespace gb
