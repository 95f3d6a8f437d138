// emit.cpp — host-side emission of alignment records (no device work):
//   GAF lines   the text format `vg giraffe -o gaf` writes (alignment_to_gaf lives in libvgio @ d029989,
//               ABSENT from the reference tree; columns follow the published GAF specification and the
//               cs difference string of minimap2: ":n" matches, "*RQ" substitution, "+Q" insertion, "-R" deletion; the
//               conventions the reference's tests fix, unittest/alignment.cpp:398-470 and :793-820, are followed)
//   JSON lines  the protobuf JSON of vg.proto's Alignment as `vg view -aj` prints it (field names as used at
//               gbwt_extender.cpp:119-156, aligner.cpp:120-241, minimizer_mapper.cpp:1146-1216: sequence, path.mapping[]
//               {position{node_id, offset, is_reverse}, edit[]{from_length, to_length, sequence}, rank}, name, quality
//               (base64), mapping_quality, score, identity, fragment_next / fragment_prev, annotation)
// giraffe_main.cpp:2209-2226 hands alignments to an AlignmentEmitter; this is the stand-in until the shim converts
// records to vg::Alignment itself (INTEGRATION.md §2).  PARITY UNPINNED: no libvgio here to compare bytes with.
#include "giraffe_b200.h"
#include "entry_guard.h"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace {

struct Out {
    char* buf; uint64_t cap; uint64_t n; bool overflow;
    void put(const char* s, size_t len) { if (n + len > cap) { overflow = true; return; } memcpy(buf + n, s, len); n += len; }
    void str(const char* s) { put(s, strlen(s)); }
    void str(const std::string& s) { put(s.data(), s.size()); }
    void ch(char c) { put(&c, 1); }
    void num(long long v) { char t[32]; const int k = snprintf(t, sizeof t, "%lld", v); put(t, (size_t)k); }
    void real(double v) { char t[40]; const int k = snprintf(t, sizeof t, "%.6g", v); put(t, (size_t)k); }
};


// base i of oriented node v (gb_flat_index stores the sequence of both orientations)
inline char node_base(const gb_flat_index* ix, uint32_t v, uint32_t i) {
    const gb_node_rec& r = ix->nodes[v];
    return (char)ix->seq[r.seq_off + i];
}

std::string read_name(const uint8_t* names, const uint64_t* name_off, uint32_t r) {
    if (names && name_off) return std::string((const char*)names + name_off[r], (size_t)(name_off[r + 1] - name_off[r]));
    return "read" + std::to_string(r);
}

void base64(Out& o, const uint8_t* p, size_t n) {
    static const char* T = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    for (size_t i = 0; i < n; i += 3) {
        const uint32_t a = p[i], b = i + 1 < n ? p[i + 1] : 0, c = i + 2 < n ? p[i + 2] : 0;
        o.ch(T[a >> 2]); o.ch(T[((a & 3) << 4) | (b >> 4)]);
        o.ch(i + 1 < n ? T[((b & 15) << 2) | (c >> 6)] : '=');
        o.ch(i + 2 < n ? T[c & 63] : '=');
    }
}

void json_string(Out& o, const std::string& s) {
    o.ch('"');
    for (char c : s) {
        if (c == '"' || c == '\\') { o.ch('\\'); o.ch(c); }
        else if ((unsigned char)c < 0x20) { char t[8]; snprintf(t, sizeof t, "\\u%04x", c); o.str(t); }
        else o.ch(c);
    }
    o.ch('"');
}

// Every record must stay inside what the caller handed over: its read, its slice of the two pools, the graph, and the
// read length its edits consume.  The emitters index with these fields, so a damaged record is refused here.
bool records_valid(const gb_flat_index* ix, uint32_t n, const gb_alignment* aln, const gb_mapping* mappings, uint64_t mapping_pool_len,
                   const uint32_t* edits, uint64_t edit_pool_len, uint32_t n_reads, const uint64_t* read_off,
                   const uint8_t* names, const uint64_t* name_off) {
    // names are addressed like reads: n_reads + 1 non-decreasing offsets
    if (names && name_off) for (uint32_t r = 0; r < n_reads; r++) if (name_off[r + 1] < name_off[r]) return false;
    for (uint32_t x = 0; x < n; x++) {
        const gb_alignment& a = aln[x];
        if (a.read_id >= n_reads || read_off[a.read_id + 1] < read_off[a.read_id]) return false;
        if ((a.flags & GB_ALN_PAIRED) && (a.read_id ^ 1u) >= n_reads) return false;
        if (!(a.flags & GB_ALN_MAPPED) || a.n_mappings == 0) continue;
        if (!mappings || !edits || (uint64_t)a.mapping_off + a.n_mappings > mapping_pool_len || (uint64_t)a.edit_off + a.n_edits > edit_pool_len) return false;
        const uint64_t L = read_off[a.read_id + 1] - read_off[a.read_id];
        uint64_t ei = 0, q = 0;
        for (uint32_t i = 0; i < a.n_mappings; i++) {
            const gb_mapping& m = mappings[a.mapping_off + i];
            if (m.node >= ix->n_nodes || ei + m.n_edits > a.n_edits) return false;
            uint64_t off = m.offset;
            for (uint32_t j = 0; j < m.n_edits; j++, ei++) {
                const uint32_t wd = edits[a.edit_off + ei], op = wd & 3u, len = op == GB_EDIT_SUB ? 1u : wd >> 4;
                if (op != GB_EDIT_DEL) q += len;
                if (op != GB_EDIT_INS) off += len;
            }
            if (off > ix->nodes[m.node].len || q > L) return false;
        }
        if (ei != a.n_edits || q != L) return false;
    }
    return true;
}

} // namespace

static int gb_emit_gaf_impl(const gb_flat_index* ix, uint32_t n, const gb_alignment* aln, const gb_mapping* mappings, uint64_t mapping_pool_len,
                           const uint32_t* edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                           const uint8_t* names, const uint64_t* name_off, char* out, uint64_t out_cap, uint64_t* out_used) {
    if (!ix || !aln || !reads || !read_off || !out || !out_used) return GB_ERR_ARG;
    if (!records_valid(ix, n, aln, mappings, mapping_pool_len, edits, edit_pool_len, n_reads, read_off, names, name_off)) return GB_ERR_ARG;
    Out o{out, out_cap, 0, false};
    for (uint32_t x = 0; x < n; x++) {
        const gb_alignment& a = aln[x];
        if (a.flags & GB_ALN_ABSENT) continue;                   // max_multimaps > 1: this read has fewer mappings than ranks
        const uint32_t r = a.read_id;
        const uint8_t* seq = reads + read_off[r];
        const uint32_t L = (uint32_t)(read_off[r + 1] - read_off[r]);
        o.str(read_name(names, name_off, r)); o.ch('\t'); o.num(L); o.ch('\t');
        // Conventions pinned by the reference's own GAF tests (unittest/alignment.cpp:398-470, :793-820): the query
        // interval is the whole read (soft clips stay in the difference string as insertions), cs bases are upper
        // case, match runs merge across edits and mappings, a mapping that only carries an insertion (a soft clip
        // parked on an unused node) is left out of the path, an unaligned read has an empty path and cs "+<read>".
        if (!(a.flags & GB_ALN_MAPPED) || a.n_mappings == 0) {
            o.num(0); o.ch('\t'); o.num(L); o.str("\t*\t*\t*\t*\t*\t*\t*\t255");
            o.str("\tcs:Z:+"); o.put((const char*)seq, L);
        } else {
            const gb_mapping* m = mappings + a.mapping_off;
            const uint32_t* e = edits + a.edit_off;
            std::string path, cs;
            uint64_t path_len = 0, matches = 0, block = 0, ref_used_total = 0, pstart = 0;
            uint32_t q = 0, ei = 0, run = 0;
            bool have_start = false;
            auto flush_run = [&]() { if (run) { cs += ':'; cs += std::to_string(run); run = 0; } };
            for (uint32_t i = 0; i < a.n_mappings; i++) {
                const uint32_t v = m[i].node;
                bool uses_node = false;
                for (uint32_t j = 0; j < m[i].n_edits; j++) uses_node |= (e[ei + j] & 3u) != GB_EDIT_INS;
                if (uses_node) {
                    path += (v & 1u) ? '<' : '>'; path += std::to_string(v >> 1);
                    path_len += ix->nodes[v].len;
                    if (!have_start) { pstart = m[i].offset; have_start = true; }
                }
                uint32_t off = m[i].offset;
                for (uint32_t j = 0; j < m[i].n_edits; j++, ei++) {
                    const uint32_t wd = e[ei], op = wd & 3u, len = op == GB_EDIT_SUB ? 1u : wd >> 4;
                    if (op == GB_EDIT_MATCH) { run += len; matches += len; block += len; q += len; off += len; ref_used_total += len; }
                    else if (op == GB_EDIT_SUB) { flush_run(); cs += '*'; cs += node_base(ix, v, off); cs += (char)seq[q]; block += 1; q += 1; off += 1; ref_used_total += 1; }
                    else if (op == GB_EDIT_INS) { flush_run(); cs += '+'; cs.append((const char*)seq + q, len); block += len; q += len; }
                    else { flush_run(); cs += '-'; for (uint32_t t = 0; t < len; t++) cs += node_base(ix, v, off + t); block += len; off += len; ref_used_total += len; }
                }
            }
            flush_run();
            o.num(0); o.ch('\t'); o.num(L); o.str("\t+\t"); o.str(path.empty() ? std::string("*") : path); o.ch('\t'); o.num((long long)path_len); o.ch('\t');
            o.num((long long)pstart); o.ch('\t'); o.num((long long)(pstart + ref_used_total)); o.ch('\t');
            o.num((long long)matches); o.ch('\t'); o.num((long long)block); o.ch('\t'); o.num(a.mapq);
            o.str("\tAS:i:"); o.num(a.score);
            if (quals) { o.str("\tbq:Z:"); for (uint32_t t = 0; t < L; t++) o.ch((char)(quals[read_off[r] + t] + 33)); }
            o.str("\tcs:Z:"); o.str(cs);
            o.str("\tdv:f:"); o.real(block ? 1.0 - (double)matches / (double)block : 0.0);
        }
        if (a.flags & GB_ALN_PAIRED) {
            // mates are interleaved: fragment_next on mate 1, fragment_prev on mate 2 (pair_all, minimizer_mapper.cpp:1280-1300)
            if ((r & 1u) == 0) { o.str("\tfn:Z:"); o.str(read_name(names, name_off, r + 1)); }
            else { o.str("\tfp:Z:"); o.str(read_name(names, name_off, r - 1)); }
        }
        o.ch('\n');
    }
    *out_used = o.n;
    return o.overflow ? GB_ERR_CAPACITY : GB_OK;
}

static int gb_emit_json_impl(const gb_flat_index* ix, uint32_t n, const gb_alignment* aln, const gb_mapping* mappings, uint64_t mapping_pool_len,
                            const uint32_t* edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                            const uint8_t* names, const uint64_t* name_off, char* out, uint64_t out_cap, uint64_t* out_used) {
    if (!ix || !aln || !reads || !read_off || !out || !out_used) return GB_ERR_ARG;
    if (!records_valid(ix, n, aln, mappings, mapping_pool_len, edits, edit_pool_len, n_reads, read_off, names, name_off)) return GB_ERR_ARG;
    Out o{out, out_cap, 0, false};
    for (uint32_t x = 0; x < n; x++) {
        const gb_alignment& a = aln[x];
        if (a.flags & GB_ALN_ABSENT) continue;
        const uint32_t r = a.read_id;
        const uint8_t* seq = reads + read_off[r];
        const uint32_t L = (uint32_t)(read_off[r + 1] - read_off[r]);
        o.str("{\"sequence\": "); json_string(o, std::string((const char*)seq, L));
        uint64_t matches = 0;
        if ((a.flags & GB_ALN_MAPPED) && a.n_mappings) {
            const gb_mapping* m = mappings + a.mapping_off;
            const uint32_t* e = edits + a.edit_off;
            o.str(", \"path\": {\"mapping\": [");
            uint32_t q = 0, ei = 0;
            for (uint32_t i = 0; i < a.n_mappings; i++) {
                if (i) o.str(", ");
                o.str("{\"position\": {\"node_id\": \""); o.num(m[i].node >> 1); o.ch('"');
                if (m[i].offset) { o.str(", \"offset\": \""); o.num(m[i].offset); o.ch('"'); }
                if (m[i].node & 1u) o.str(", \"is_reverse\": true");
                o.str("}, \"edit\": [");
                for (uint32_t j = 0; j < m[i].n_edits; j++, ei++) {
                    const uint32_t wd = e[ei], op = wd & 3u, len = op == GB_EDIT_SUB ? 1u : wd >> 4;
                    if (j) o.str(", ");
                    if (op == GB_EDIT_MATCH) { o.str("{\"from_length\": "); o.num(len); o.str(", \"to_length\": "); o.num(len); o.ch('}'); matches += len; q += len; }
                    else if (op == GB_EDIT_SUB) { o.str("{\"from_length\": 1, \"to_length\": 1, \"sequence\": "); json_string(o, std::string(1, (char)seq[q])); o.ch('}'); q += 1; }
                    else if (op == GB_EDIT_INS) { o.str("{\"to_length\": "); o.num(len); o.str(", \"sequence\": "); json_string(o, std::string((const char*)seq + q, len)); o.ch('}'); q += len; }
                    else { o.str("{\"from_length\": "); o.num(len); o.ch('}'); }
                }
                o.str("], \"rank\": \""); o.num(i + 1); o.str("\"}");
            }
            o.str("]}");
        }
        o.str(", \"name\": "); json_string(o, read_name(names, name_off, r));
        if (quals) { o.str(", \"quality\": \""); base64(o, quals + read_off[r], L); o.ch('"'); }
        if (a.mapq) { o.str(", \"mapping_quality\": "); o.num(a.mapq); }
        if (a.score) { o.str(", \"score\": "); o.num(a.score); }
        if (a.flags & GB_ALN_SECONDARY) o.str(", \"is_secondary\": true");        // set_is_secondary, minimizer_mapper.cpp:1205, :2555
        if ((a.flags & GB_ALN_MAPPED) && L) { o.str(", \"identity\": "); o.real((double)matches / (double)L); }      // identity(path), alignment.cpp
        if (a.flags & GB_ALN_PAIRED) {
            if ((r & 1u) == 0) { o.str(", \"fragment_next\": {\"name\": "); json_string(o, read_name(names, name_off, r + 1)); o.ch('}'); }
            else { o.str(", \"fragment_prev\": {\"name\": "); json_string(o, read_name(names, name_off, r - 1)); o.ch('}'); }
        }
        o.str(", \"annotation\": {\"mapq_uncapped\": "); o.real(a.mapq_uncapped); o.str(", \"mapq_explored_cap\": ");
        if (a.mapq_explored_cap > 1e30f) o.str("\"Infinity\""); else o.real(a.mapq_explored_cap);
        if (a.flags & GB_ALN_RESCUED) o.str(", \"rescued\": true");
        o.str("}}\n");
    }
    *out_used = o.n;
    return o.overflow ? GB_ERR_CAPACITY : GB_OK;
}

// ---- GAM: vg.proto Alignment messages in vg::io's group framing -------------------------------------------------
// libvgio (vg.proto, the stream framing) is absent from the reference tree; the wire layout is read off GAM files vg
// itself wrote, kept as fixtures in tests/golden/gam/ (test/surject/perpendicular.gam is Giraffe output):
//   stream    groups of [varint n] [varint 3]["GAM"] then n-1 x [varint len][Alignment]      (type-tagged groups)
//   Alignment 1 sequence, 2 path, 3 name, 4 quality (raw phred bytes), 5 mapping_quality, 6 score,
//             11 fragment_prev / 12 fragment_next (an Alignment carrying only 3 name), 16 identity (double),
//             100 annotation (google.protobuf.Struct: 1 fields{1 key, 2 Value{2 number_value, 4 bool_value}})
//   Path      2 mapping;   Mapping 1 position, 2 edit, 5 rank;   Position 1 node_id, 2 offset, 4 is_reverse;
//   Edit      1 from_length, 2 to_length, 3 sequence.   proto3: zero / false / empty fields are not written.
// The stream is written uncompressed: vg::io's BlockedGzipInputStream reads uncompressed, gzip and BGZF data alike
// (unittest/blocked_gzip_input_stream.cpp:136, :364, :400).
namespace {

void pb_varint(std::string& s, uint64_t v) { while (v >= 0x80) { s.push_back((char)(v | 0x80)); v >>= 7; } s.push_back((char)v); }
void pb_tag(std::string& s, uint32_t field, uint32_t wire) { pb_varint(s, ((uint64_t)field << 3) | wire); }
void pb_uint(std::string& s, uint32_t field, uint64_t v) { if (v) { pb_tag(s, field, 0); pb_varint(s, v); } }
void pb_bytes(std::string& s, uint32_t field, const char* p, size_t n) { pb_tag(s, field, 2); pb_varint(s, n); s.append(p, n); }
void pb_msg(std::string& s, uint32_t field, const std::string& m) { pb_bytes(s, field, m.data(), m.size()); }
void pb_double(std::string& s, uint32_t field, double v) { pb_tag(s, field, 1); char b[8]; memcpy(b, &v, 8); s.append(b, 8); }
void pb_annotation(std::string& st, const char* key, const std::string& value_msg) {
    std::string entry; pb_bytes(entry, 1, key, strlen(key)); pb_msg(entry, 2, value_msg);
    pb_msg(st, 1, entry);
}

} // namespace

static int gb_emit_gam_impl(const gb_flat_index* ix, uint32_t n, const gb_alignment* aln, const gb_mapping* mappings, uint64_t mapping_pool_len,
                           const uint32_t* edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* reads, const uint8_t* quals, const uint64_t* read_off,
                           const uint8_t* names, const uint64_t* name_off, char* out, uint64_t out_cap, uint64_t* out_used) {
    if (!ix || !aln || !reads || !read_off || !out || !out_used) return GB_ERR_ARG;
    if (!records_valid(ix, n, aln, mappings, mapping_pool_len, edits, edit_pool_len, n_reads, read_off, names, name_off)) return GB_ERR_ARG;
    Out o{out, out_cap, 0, false};
    const uint32_t GROUP = 1000;                 // messages per group
    std::vector<uint32_t> present;               // max_multimaps > 1: ranks a read does not have are skipped
    present.reserve(n);
    for (uint32_t x = 0; x < n; x++) if (!(aln[x].flags & GB_ALN_ABSENT)) present.push_back(x);
    const uint32_t np = (uint32_t)present.size();
    for (uint32_t g0 = 0; g0 < np; g0 += GROUP) {
        const uint32_t gn = std::min(GROUP, np - g0);
        std::string group;
        pb_varint(group, (uint64_t)gn + 1); pb_varint(group, 3); group += "GAM";
        for (uint32_t y = g0; y < g0 + gn; y++) {
            const gb_alignment& a = aln[present[y]];
            const uint32_t r = a.read_id;
            const char* seq = (const char*)reads + read_off[r];
            const uint32_t L = (uint32_t)(read_off[r + 1] - read_off[r]);
            std::string msg;
            pb_bytes(msg, 1, seq, L);
            uint64_t matches = 0;
            if ((a.flags & GB_ALN_MAPPED) && a.n_mappings) {
                const gb_mapping* m = mappings + a.mapping_off;
                const uint32_t* e = edits + a.edit_off;
                std::string path;
                uint32_t q = 0, ei = 0;
                for (uint32_t i = 0; i < a.n_mappings; i++) {
                    std::string mp, pos;
                    pb_uint(pos, 1, m[i].node >> 1); pb_uint(pos, 2, m[i].offset); pb_uint(pos, 4, m[i].node & 1u);
                    pb_msg(mp, 1, pos);
                    for (uint32_t j = 0; j < m[i].n_edits; j++, ei++) {
                        const uint32_t wd = e[ei], op = wd & 3u, len = op == GB_EDIT_SUB ? 1u : wd >> 4;
                        std::string ed;
                        if (op == GB_EDIT_MATCH) { pb_uint(ed, 1, len); pb_uint(ed, 2, len); matches += len; q += len; }
                        else if (op == GB_EDIT_SUB) { pb_uint(ed, 1, 1); pb_uint(ed, 2, 1); pb_bytes(ed, 3, seq + q, 1); q += 1; }
                        else if (op == GB_EDIT_INS) { pb_uint(ed, 2, len); pb_bytes(ed, 3, seq + q, len); q += len; }
                        else pb_uint(ed, 1, len);
                        pb_msg(mp, 2, ed);
                    }
                    pb_uint(mp, 5, i + 1);
                    pb_msg(path, 2, mp);
                }
                pb_msg(msg, 2, path);
            }
            const std::string nm = read_name(names, name_off, r);
            pb_bytes(msg, 3, nm.data(), nm.size());
            if (quals && L) pb_bytes(msg, 4, (const char*)quals + read_off[r], L);
            pb_uint(msg, 5, a.mapq);
            pb_uint(msg, 6, (uint64_t)(int64_t)a.score);           // proto3 int32: a negative value is a sign-extended 10-byte varint
            if (a.flags & GB_ALN_PAIRED) {
                const std::string mate = read_name(names, name_off, r ^ 1u);
                std::string frag; pb_bytes(frag, 3, mate.data(), mate.size());
                pb_msg(msg, (r & 1u) ? 11 : 12, frag);
            }
            if (a.flags & GB_ALN_SECONDARY) pb_uint(msg, 15, 1);           // vg.proto Alignment.is_secondary = 15
            if ((a.flags & GB_ALN_MAPPED) && L) pb_double(msg, 16, (double)matches / (double)L);
            std::string st, v;
            v.clear(); pb_double(v, 2, (double)a.mapq_uncapped); pb_annotation(st, "mapq_uncapped", v);
            v.clear(); pb_double(v, 2, (double)a.mapq_explored_cap); pb_annotation(st, "mapq_explored_cap", v);
            if (a.flags & GB_ALN_RESCUED) { v.clear(); pb_tag(v, 4, 0); pb_varint(v, 1); pb_annotation(st, "rescued", v); }
            pb_msg(msg, 100, st);
            pb_varint(group, msg.size()); group += msg;
        }
        o.put(group.data(), group.size());
    }
    *out_used = o.n;
    return o.overflow ? GB_ERR_CAPACITY : GB_OK;
}


// ---- the C ABI: no exception leaves the library (std::string growth can throw) -----------------------------------
#define GB_EMIT_ENTRY(NAME)                                                                                                        \
    extern "C" int NAME(const gb_flat_index* ix, uint32_t n, const gb_alignment* aln, const gb_mapping* mappings, uint64_t mapping_pool_len, \
                        const uint32_t* edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* reads, const uint8_t* quals,         \
                        const uint64_t* read_off, const uint8_t* names, const uint64_t* name_off, char* out, uint64_t out_cap, uint64_t* out_used) { \
        return gb::guarded(#NAME, [&] { return NAME##_impl(ix, n, aln, mappings, mapping_pool_len, edits, edit_pool_len, n_reads, reads, quals, \
                                                           read_off, names, name_off, out, out_cap, out_used); });                  \
    }
GB_EMIT_ENTRY(gb_emit_gaf)
GB_EMIT_ENTRY(gb_emit_json)
GB_EMIT_ENTRY(gb_emit_gam)

// ---- BGZF: the blocked gzip container vg::io writes GAM in (giraffe_main.cpp:2209-2226 -> vg::io::ProtobufEmitter over a
// BlockedGzipOutputStream; htslib's bgzf.c layout).  Every block is a complete gzip member of at most 64 KiB with the
// extra subfield 'B','C' = total block size - 1, so readers can seek by (block offset, offset in block); the stream ends
// with the 28-byte empty block.  Input is cut every 0xff00 bytes as htslib does.
#include <zlib.h>
extern "C" int gb_bgzf_compress(const void* in, uint64_t in_bytes, int level, void* out, uint64_t out_cap, uint64_t* out_used) {
    if ((!in && in_bytes) || !out || !out_used || level < 0 || level > 9) return GB_ERR_ARG;
    const uint8_t* src = (const uint8_t*)in; uint8_t* dst = (uint8_t*)out;
    uint64_t o = 0;
    const uint64_t BLOCK = 0xff00;
    auto block = [&](const uint8_t* p, uint32_t len) -> int {
        uint8_t buf[0x10000];
        z_stream zs; memset(&zs, 0, sizeof zs);
        if (deflateInit2(&zs, len ? level : Z_DEFAULT_COMPRESSION, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) return GB_ERR_ARG;
        zs.next_in = const_cast<uint8_t*>(p); zs.avail_in = len; zs.next_out = buf + 18; zs.avail_out = sizeof buf - 18 - 8;
        int zr = deflate(&zs, Z_FINISH);
        if (zr != Z_STREAM_END) {                       // incompressible data at this level: store it (always fits: 0xff00 + 5)
            deflateEnd(&zs);
            memset(&zs, 0, sizeof zs);
            if (deflateInit2(&zs, 0, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) return GB_ERR_ARG;
            zs.next_in = const_cast<uint8_t*>(p); zs.avail_in = len; zs.next_out = buf + 18; zs.avail_out = sizeof buf - 18 - 8;
            zr = deflate(&zs, Z_FINISH);
            if (zr != Z_STREAM_END) { deflateEnd(&zs); return GB_ERR_ARG; }
        }
        const uint32_t clen = (uint32_t)zs.total_out;
        deflateEnd(&zs);
        const uint32_t total = 18 + clen + 8;
        static const uint8_t head[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
        memcpy(buf, head, 16);
        buf[16] = (uint8_t)((total - 1) & 0xff); buf[17] = (uint8_t)((total - 1) >> 8);
        const uint32_t crc = (uint32_t)crc32(crc32(0L, Z_NULL, 0), p, len);
        for (int i = 0; i < 4; i++) { buf[18 + clen + i] = (uint8_t)(crc >> (8 * i)); buf[22 + clen + i] = (uint8_t)(len >> (8 * i)); }
        if (o + total > out_cap) return GB_ERR_CAPACITY;
        memcpy(dst + o, buf, total); o += total;
        return GB_OK;
    };
    for (uint64_t at = 0; at < in_bytes; at += BLOCK) {
        const int rc = block(src + at, (uint32_t)std::min<uint64_t>(BLOCK, in_bytes - at));
        if (rc) return rc;
    }
    const int rc = block(src, 0);                       // the EOF marker block
    if (rc) return rc;
    *out_used = o;
    return GB_OK;
}
