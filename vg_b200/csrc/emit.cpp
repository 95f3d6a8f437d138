// emit.cpp — host-side emission of alignment records (no device work):
//   GAF, GAM    gb_emit_gaf / gb_emit_gam run the formatter and record check of emit_format.h, as the device emitters do
//   JSON lines  the protobuf JSON of vg.proto's Alignment as `vg view -aj` prints it (field names as used at
//               gbwt_extender.cpp:119-156, aligner.cpp:120-241, minimizer_mapper.cpp:1146-1216: sequence, path.mapping[]
//               {position{node_id, offset, is_reverse}, edit[]{from_length, to_length, sequence}, rank}, name, quality
//               (base64), mapping_quality, score, identity, fragment_next / fragment_prev, annotation)
//   BGZF        gb_bgzf_compress: the container vg::io writes GAM in
// Each record (for GAM, each group of GAM_GROUP messages with its header) is counted first and written only when it fits,
// so after GB_ERR_CAPACITY the output ends at a whole record or group.
// giraffe_main.cpp:2209-2226 hands alignments to an AlignmentEmitter; this is the stand-in until the shim converts
// records to vg::Alignment itself (INTEGRATION.md §2).  PARITY UNPINNED: no libvgio here to compare bytes with.
#include "giraffe_b200.h"
#include "entry_guard.h"
#include "emit_format.h"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

namespace gb {
namespace {

bool batch_valid(const EmitArgs& A) {
    for (uint32_t r = 0; r < A.n_reads; r++) if (!name_valid(A, r)) return false;
    for (uint32_t x = 0; x < A.n; x++) if (!record_valid(A, A.aln[x])) return false;
    return true;
}

// One line per present record: record(sink, a) formats it.
template <class Record>
int emit_lines(const EmitArgs& A, char* out, uint64_t out_cap, uint64_t* out_used, const Record& record) {
    *out_used = 0;
    for (uint32_t x = 0; x < A.n; x++) {
        const gb_alignment& a = A.aln[x];
        if (a.flags & GB_ALN_ABSENT) continue;                   // max_multimaps > 1: this read has fewer mappings than ranks
        Count c; record(c, a);
        if (c.n > out_cap - *out_used) return GB_ERR_CAPACITY;
        Write w{out + *out_used}; record(w, a);
        *out_used += c.n;
    }
    return GB_OK;
}

int emit_gaf(const EmitArgs& A, char* out, uint64_t out_cap, uint64_t* out_used) {
    return emit_lines(A, out, out_cap, out_used, [&](auto& s, const gb_alignment& a) { gaf_record(s, A, a); });
}

int emit_gam(const EmitArgs& A, char* out, uint64_t out_cap, uint64_t* out_used) {
    std::vector<uint32_t> present;               // max_multimaps > 1: ranks a read does not have are skipped
    for (uint32_t x = 0; x < A.n; x++) if (!(A.aln[x].flags & GB_ALN_ABSENT)) present.push_back(x);
    const size_t np = present.size();
    std::vector<uint64_t> len(std::min<size_t>(np, GAM_GROUP));
    *out_used = 0;
    for (size_t g0 = 0; g0 < np; g0 += GAM_GROUP) {
        const uint32_t gn = (uint32_t)std::min<size_t>(GAM_GROUP, np - g0);
        uint64_t need = gam_header_len(gn);
        for (uint32_t y = 0; y < gn; y++) {
            Count c; gam_message(c, A, A.aln[present[g0 + y]]);
            len[y] = c.n; need += varint_len(c.n) + c.n;
        }
        if (need > out_cap - *out_used) return GB_ERR_CAPACITY;
        Write w{out + *out_used};
        gam_header(w, gn);
        for (uint32_t y = 0; y < gn; y++) { varint(w, len[y]); gam_message(w, A, A.aln[present[g0 + y]]); }
        *out_used += need;
    }
    return GB_OK;
}

// ---- JSON: host only --------------------------------------------------------------------------------------------------
template <class S> void json_string(S& s, const uint8_t* p, uint64_t n) {
    s.ch('"');
    for (uint64_t i = 0; i < n; i++) {
        const char c = (char)p[i];
        if (c == '"' || c == '\\') { s.ch('\\'); s.ch(c); }
        else if ((unsigned char)c < 0x20) { char t[8]; s.put(t, snprintf(t, sizeof t, "\\u%04x", c)); }
        else s.ch(c);
    }
    s.ch('"');
}

template <class S> void json_name(S& s, const EmitArgs& A, uint32_t r) {
    if (use_names(A)) json_string(s, A.names + A.name_off[r], A.name_off[r + 1] - A.name_off[r]);
    else { s.ch('"'); name(s, A, r); s.ch('"'); }          // read<r> needs no escaping
}

template <class S> void base64(S& s, const uint8_t* p, size_t n) {
    static const char* T = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    for (size_t i = 0; i < n; i += 3) {
        const uint32_t a = p[i], b = i + 1 < n ? p[i + 1] : 0, c = i + 2 < n ? p[i + 2] : 0;
        s.ch(T[a >> 2]); s.ch(T[((a & 3) << 4) | (b >> 4)]);
        s.ch(i + 1 < n ? T[((b & 15) << 2) | (c >> 6)] : '=');
        s.ch(i + 2 < n ? T[c & 63] : '=');
    }
}

// printf's "%.6g": the annotations are not in [0, 1], where g6 is exact
template <class S> void real(S& s, double v) { char t[40]; s.put(t, snprintf(t, sizeof t, "%.6g", v)); }

template <class S> void json_record(S& s, const EmitArgs& A, const gb_alignment& a) {
    const uint32_t r = a.read_id;
    const uint8_t* seq = A.reads + A.read_off[r];
    const uint32_t L = (uint32_t)(A.read_off[r + 1] - A.read_off[r]);
    lit(s, "{\"sequence\": "); json_string(s, seq, L);
    uint64_t matches = 0;
    if ((a.flags & GB_ALN_MAPPED) && a.n_mappings) {
        const gb_mapping* m = A.maps + a.mapping_off;
        const uint32_t* e = A.edits + a.edit_off;
        lit(s, ", \"path\": {\"mapping\": [");
        uint32_t q = 0, ei = 0;
        for (uint32_t i = 0; i < a.n_mappings; i++) {
            if (i) lit(s, ", ");
            lit(s, "{\"position\": {\"node_id\": \""); unum(s, m[i].node >> 1); s.ch('"');
            if (m[i].offset) { lit(s, ", \"offset\": \""); unum(s, m[i].offset); s.ch('"'); }
            if (m[i].node & 1u) lit(s, ", \"is_reverse\": true");
            lit(s, "}, \"edit\": [");
            for (uint32_t j = 0; j < m[i].n_edits; j++, ei++) {
                const uint32_t wd = e[ei], op = wd & 3u, len = edit_len(wd);
                if (j) lit(s, ", ");
                if (op == GB_EDIT_MATCH) { lit(s, "{\"from_length\": "); unum(s, len); lit(s, ", \"to_length\": "); unum(s, len); s.ch('}'); matches += len; q += len; }
                else if (op == GB_EDIT_SUB) { lit(s, "{\"from_length\": 1, \"to_length\": 1, \"sequence\": "); json_string(s, seq + q, 1); s.ch('}'); q += 1; }
                else if (op == GB_EDIT_INS) { lit(s, "{\"to_length\": "); unum(s, len); lit(s, ", \"sequence\": "); json_string(s, seq + q, len); s.ch('}'); q += len; }
                else { lit(s, "{\"from_length\": "); unum(s, len); s.ch('}'); }
            }
            lit(s, "], \"rank\": \""); unum(s, i + 1); lit(s, "\"}");
        }
        lit(s, "]}");
    }
    lit(s, ", \"name\": "); json_name(s, A, r);
    if (A.quals) { lit(s, ", \"quality\": \""); base64(s, A.quals + A.read_off[r], L); s.ch('"'); }
    if (a.mapq) { lit(s, ", \"mapping_quality\": "); unum(s, a.mapq); }
    if (a.score) { lit(s, ", \"score\": "); snum(s, a.score); }
    if (a.flags & GB_ALN_SECONDARY) lit(s, ", \"is_secondary\": true");        // set_is_secondary, minimizer_mapper.cpp:1205, :2555
    if ((a.flags & GB_ALN_MAPPED) && L) { lit(s, ", \"identity\": "); real(s, (double)matches / (double)L); }      // identity(path), alignment.cpp
    if (a.flags & GB_ALN_PAIRED) {
        if ((r & 1u) == 0) { lit(s, ", \"fragment_next\": {\"name\": "); json_name(s, A, r + 1); s.ch('}'); }
        else { lit(s, ", \"fragment_prev\": {\"name\": "); json_name(s, A, r - 1); s.ch('}'); }
    }
    lit(s, ", \"annotation\": {\"mapq_uncapped\": "); real(s, a.mapq_uncapped); lit(s, ", \"mapq_explored_cap\": ");
    if (a.mapq_explored_cap > 1e30f) lit(s, "\"Infinity\""); else real(s, a.mapq_explored_cap);
    if (a.flags & GB_ALN_RESCUED) lit(s, ", \"rescued\": true");
    lit(s, "}}\n");
}

int emit_json(const EmitArgs& A, char* out, uint64_t out_cap, uint64_t* out_used) {
    return emit_lines(A, out, out_cap, out_used, [&](auto& s, const gb_alignment& a) { json_record(s, A, a); });
}

} // namespace
} // namespace gb

// ---- the C ABI: no exception leaves the library (gb_emit_gam's record lists can fail to allocate) ----------------------
#define GB_EMIT_ENTRY(NAME, EMIT)                                                                                                  \
    extern "C" int NAME(const gb_flat_index* ix, uint32_t n, const gb_alignment* aln, const gb_mapping* mappings, uint64_t mapping_pool_len, \
                        const uint32_t* edits, uint64_t edit_pool_len, uint32_t n_reads, const uint8_t* reads, const uint8_t* quals,         \
                        const uint64_t* read_off, const uint8_t* names, const uint64_t* name_off, char* out, uint64_t out_cap, uint64_t* out_used) { \
        return gb::guarded(#NAME, [&] {                                                                                            \
            if (!ix || !aln || !reads || !read_off || !out || !out_used) return GB_ERR_ARG;                                        \
            const gb::EmitArgs A{n, aln, mappings, mapping_pool_len, edits, edit_pool_len, n_reads, reads, quals, read_off, names, name_off, \
                                 ix->nodes, ix->seq, ix->n_nodes};                                                                 \
            return gb::batch_valid(A) ? EMIT(A, out, out_cap, out_used) : GB_ERR_ARG;                                              \
        });                                                                                                                        \
    }
GB_EMIT_ENTRY(gb_emit_gaf, gb::emit_gaf)
GB_EMIT_ENTRY(gb_emit_json, gb::emit_json)
GB_EMIT_ENTRY(gb_emit_gam, gb::emit_gam)

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
