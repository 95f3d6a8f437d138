// gbz_reader.cpp — read a GBZ file (what `vg giraffe -Z` loads, giraffe_main.cpp:1825-1881) and build the flat index
// from it: node sequences from the GBWTGraph, the GBWT records decoded and handed to the builder in its blob layout
// (gb_index_build_from_gbwt: no haplotype is walked, so the work follows the graph, not haplotypes x genome); the distance
// payload (chains of cut nodes and sites) and the minimizers come from the library's own index builder.
//
// gbwt (jltsiren/gbwt @ c2e0199), gbwtgraph (@ e27bc43) and simple-sds are ABSENT from the reference tree; the layout
// below is their published serialization format, checked against the GBZ the reference ships as test data
// (test/primers/y.giraffe.gbz, kept as tests/golden/gbz/y.giraffe.gbz): 66 nodes, 1012 bp, 3 haplotypes, BWT size 322.
//   simple-sds      little-endian 64-bit elements; Vector<T> = len + items padded to 8 B; RawVector = bit length +
//                   Vector<u64>; BitVector = ones + RawVector + 3 optional supports (each: size in elements + data);
//                   IntVector = len + width + RawVector; SparseVector (Elias-Fano) = len + high BitVector + low
//                   IntVector, value i = ((position of the i-th one - i) << width) | low[i];
//                   StringArray = SparseVector of string starts + alphabet Vector<u8> + IntVector of alphabet ranks
//   GBZ             tag "GBZ " / version 1, flags, Tags (StringArray), GBWT, GBWTGraph
//   GBWT            tag 0x6B376B37 / version 5, sequences, size, offset, alphabet size, flags; Tags; BWT = SparseVector
//                   of record starts + Vector<u8>; optional DA samples; optional metadata
//   GBWT record     ByteCode outdegree, outdegree x (ByteCode successor delta, ByteCode offset), runs: for outdegree
//                   sigma < 255 one byte c = rank + sigma (len - 1), len == 256 / sigma continues with a ByteCode;
//                   otherwise ByteCode rank + ByteCode (len - 1)
//   GBWTGraph       tag 0x6B3764AF / version 3, nodes, flags, forward sequences (StringArray), node-to-segment translation
// Only what this path needs is kept; anything the reader does not understand is GB_ERR_FORMAT, never a guess.
#include "giraffe_b200.h"
#include "entry_guard.h"
#include "index_build.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

namespace {

struct Reader {
    const std::vector<uint64_t>& w; const std::vector<uint8_t>& bytes; size_t i = 0; bool ok = true;
    uint64_t u() { if (i >= w.size()) { ok = false; return 0; } return w[i++]; }
    void skip(uint64_t n) { if (n > w.size() - i) { ok = false; i = w.size(); } else i += n; }
};

bool raw_vector(Reader& r, uint64_t& bits, std::vector<uint64_t>& words) {
    bits = r.u(); const uint64_t n = r.u();
    if (!r.ok || n > r.w.size() - r.i || bits > n * 64) return r.ok = false;
    words.assign(r.w.begin() + r.i, r.w.begin() + r.i + n); r.i += n;
    return true;
}
void skip_optional(Reader& r) { r.skip(r.u()); }

bool int_vector(Reader& r, std::vector<uint64_t>& out, uint64_t* width_out = nullptr) {
    const uint64_t n = r.u(), width = r.u();
    uint64_t bits; std::vector<uint64_t> words;
    if (!raw_vector(r, bits, words) || width == 0 || width > 64 || n > bits / width + 1 || n * width > bits) return r.ok = false;
    out.resize(n);
    for (uint64_t k = 0; k < n; k++) {
        const uint64_t b = k * width, wd = b >> 6, sh = b & 63;
        uint64_t v = words[wd] >> sh;
        if (sh + width > 64) v |= words[wd + 1] << (64 - sh);
        out[k] = width == 64 ? v : v & ((1ull << width) - 1);
    }
    if (width_out) *width_out = width;
    return true;
}

bool sparse_values(Reader& r, std::vector<uint64_t>& values, uint64_t& universe) {
    universe = r.u();
    const uint64_t ones = r.u();
    uint64_t bits; std::vector<uint64_t> words;
    if (!raw_vector(r, bits, words)) return false;
    skip_optional(r); skip_optional(r); skip_optional(r);
    std::vector<uint64_t> low; uint64_t width = 0;
    if (!r.ok || !int_vector(r, low, &width) || low.size() != ones) return r.ok = false;
    values.clear();
    for (uint64_t p = 0; p < bits; p++) if ((words[p >> 6] >> (p & 63)) & 1) {
        const uint64_t idx = values.size();
        if (idx >= ones || p < idx) return r.ok = false;
        values.push_back(((p - idx) << width) | low[idx]);
    }
    return values.size() == ones ? true : (r.ok = false);
}

bool vector_u8(Reader& r, std::vector<uint8_t>& out) {
    const uint64_t n = r.u();
    const uint64_t start = (uint64_t)r.i * 8;
    if (!r.ok || n > r.bytes.size() - start) return r.ok = false;
    out.assign(r.bytes.begin() + start, r.bytes.begin() + start + n);
    r.skip((n + 7) / 8);
    return r.ok;
}

bool string_array(Reader& r, std::vector<std::string>& out) {
    std::vector<uint64_t> starts, ranks; uint64_t universe; std::vector<uint8_t> alphabet;
    if (!sparse_values(r, starts, universe) || !vector_u8(r, alphabet) || !int_vector(r, ranks)) return false;
    std::string all(ranks.size(), '\0');
    for (size_t k = 0; k < ranks.size(); k++) { if (ranks[k] >= alphabet.size()) return r.ok = false; all[k] = (char)alphabet[ranks[k]]; }
    out.clear();
    for (size_t s = 0; s < starts.size(); s++) {
        const uint64_t a = starts[s], b = s + 1 < starts.size() ? starts[s + 1] : all.size();
        if (a > b || b > all.size()) return r.ok = false;
        out.push_back(all.substr(a, b - a));
    }
    return true;
}

uint64_t bytecode(const std::vector<uint8_t>& b, size_t& i, size_t end, bool& ok) {
    uint64_t v = 0; int shift = 0;
    while (true) {
        if (i >= end || shift > 56) { ok = false; return 0; }
        const uint8_t c = b[i++]; v |= (uint64_t)(c & 0x7F) << shift; shift += 7;
        if (!(c & 0x80)) return v;
    }
}

struct Record { std::vector<std::pair<uint64_t, uint64_t>> edges; std::vector<std::pair<uint32_t, uint64_t>> runs; };

int fail(const char* why) { if (getenv("GB_GBZ_DEBUG")) fprintf(stderr, "gbz reader: %s\n", why); return GB_ERR_FORMAT; }

} // namespace

// The minimizer table of a gbwtgraph .min file (what `vg giraffe -m` loads, giraffe_main.cpp:1825-1881; written by
// gbwtgraph::DefaultMinimizerIndex::serialize, gbwtgraph @ e27bc43 — absent from the reference tree).  Layout as found in
// the file the reference ships for its test GBZ (test/primers/y.min, kept as tests/golden/gbz/y.min) and checked there
// cell by cell against this library's own minimizer scan (tests/test_gbz.py):
//   9-word header  tag 0x31513151 | version 10 << 32, k, w, keys, (unused), max_keys, values, unique, flags
//                  (flags 0x40 in that file: bits 0-7 the key size in bits, 64; bit 8 = syncmers, refused)
//   word 9         capacity, then capacity 32-byte cells: key, position, payload[2]; the empty key is 2^63 - 1
//   after the table one 64-bit count of multi-occurrence values: 0 in that file.
// Keys with SEVERAL occurrences (key bit 63 set; values == unique is false) are laid out after the table in a way that
// file cannot show, so the table of such a file is not read rather than guessed at: k and w are taken from its header and
// the minimizers are found on the graph by window enumeration — the same set, since a .min is exactly that.
struct MinFile { uint32_t k = 0, w = 0; bool multi = false; std::vector<uint64_t> keys, pos, payload0, payload1; };
static int read_min_file(const char* path, MinFile& m) {
    FILE* f = fopen(path, "rb");
    if (!f) return fail("open .min");
    std::vector<uint8_t> bytes;
    { uint8_t buf[65536]; size_t n; while ((n = fread(buf, 1, sizeof buf, f)) > 0) bytes.insert(bytes.end(), buf, buf + n); }
    fclose(f);
    if (bytes.size() < 88 || bytes.size() % 8 != 0) return fail(".min size");
    std::vector<uint64_t> W(bytes.size() / 8);
    memcpy(W.data(), bytes.data(), bytes.size());
    if ((uint32_t)W[0] != 0x31513151u || (W[0] >> 32) != 10) return fail("not a minimizer index version 10");
    const uint64_t k = W[1], w = W[2], keys = W[3], values = W[6], unique = W[7], flags = W[8], capacity = W[9];
    if (k == 0 || k > 31 || w == 0 || w > 4096) return fail(".min k / w");
    // flags: bits 0-7 = key size in bits (64: Key64, the only key type giraffe uses), bit 8 = syncmers; anything else
    // (weighted minimizers, further bits) is refused.  The 16-byte payload shows in the 32-byte cells below.
    if ((flags & 0xFFu) != 64) return fail(".min keys are not 64-bit");
    if ((flags & 0x100u) != 0) return fail(".min holds syncmers, not minimizers");
    if ((flags & ~0x1FFull) != 0) return fail(".min carries flags this reader does not know");
    if (capacity == 0 || (capacity & (capacity - 1)) != 0 || capacity > (W.size() - 10) / 4) return fail(".min capacity");
    m.k = (uint32_t)k; m.w = (uint32_t)w;
    if (keys > capacity) return fail(".min key count");
    if (values != keys || unique != keys) { m.multi = true; return GB_OK; }      // several occurrences per key: only k and w are taken from this file
    if (W.size() != 10 + 4 * capacity + 1 || W.back() != 0) return fail(".min tail");
    m.k = (uint32_t)k; m.w = (uint32_t)w;
    for (uint64_t c = 0; c < capacity; c++) {
        const uint64_t* cell = &W[10 + 4 * c];
        if (cell[0] == 0x7FFFFFFFFFFFFFFFull) continue;
        if (cell[0] >> 63) return fail(".min pointer cell");
        m.keys.push_back(cell[0]); m.pos.push_back(cell[1]); m.payload0.push_back(cell[2]); m.payload1.push_back(cell[3]);
    }
    if (m.keys.size() != keys) return fail(".min key count");
    return GB_OK;
}
// The oversized zipcodes of a .zipcodes file ("SPIZ", zip_code.cpp:2111-2170): only counted here — a cell whose payload is
// (0, i) points at zipcode i of this file, and the three files must agree on that (zip_code.cpp:2018-2058).
static int count_zipcodes(const char* path, uint64_t& count) {
    FILE* f = fopen(path, "rb");
    if (!f) return fail("open .zipcodes");
    std::vector<uint8_t> z;
    { uint8_t buf[65536]; size_t n; while ((n = fread(buf, 1, sizeof buf, f)) > 0) z.insert(z.end(), buf, buf + n); }
    fclose(f);
    if (z.size() < 8 || memcmp(z.data(), "SPIZ", 4) != 0) return fail("not a zipcode file");
    size_t i = 8; count = 0;
    auto varint = [&](uint64_t& v) { v = 0; for (unsigned sh = 0; sh < 64; sh += 7) { if (i >= z.size()) return false; const uint8_t c = z[i++]; v |= (uint64_t)(c & 0x7F) << sh; if (!(c & 0x80)) return true; } return false; };
    while (i < z.size()) {
        uint64_t n;
        if (!varint(n) || n > z.size() - i) return fail("zipcode length"); i += n;        // the zipcode's varints
        if (!varint(n) || n > z.size() - i) return fail("decoder length"); i += n;        // its decoder
        count++;
    }
    return GB_OK;
}

// device < 0: the whole build on the host; device >= 0: the minimizers are enumerated on that GPU (gb_index_from_gbz_device).
static int index_from_gbz_impl(const char* path, uint32_t k, uint32_t w, gb_host_index** out, const MinFile* min = nullptr, int device = -1) {
    if (!path || !out) return GB_ERR_ARG;
    *out = nullptr;
    if (device >= 0) {
        if (k == 0 || k > 31 || w == 0) return GB_ERR_ARG;
        if (const int rc = gb::device_ready(device)) return rc;
    }
    FILE* f = fopen(path, "rb");
    if (!f) return fail("open");
    std::vector<uint8_t> bytes;
    { uint8_t buf[65536]; size_t n; while ((n = fread(buf, 1, sizeof buf, f)) > 0) bytes.insert(bytes.end(), buf, buf + n); }
    fclose(f);
    if (bytes.size() < 64 || bytes.size() % 8 != 0) return fail("size");
    std::vector<uint64_t> words(bytes.size() / 8);
    memcpy(words.data(), bytes.data(), bytes.size());
    Reader r{words, bytes};

    // ---- GBZ header, tags ----
    const uint64_t h0 = r.u(); r.u();
    if ((uint32_t)h0 != 0x205A4247u || (h0 >> 32) != 1) return fail("not a GBZ version 1 file");
    std::vector<std::string> tags;
    if (!string_array(r, tags)) return fail("gbz tags");
    // ---- GBWT ----
    const uint64_t g0 = r.u();
    if ((uint32_t)g0 != 0x6B376B37u || (g0 >> 32) != 5) return fail("gbwt header");
    const uint64_t sequences = r.u(), size = r.u(), offset = r.u(), alphabet_size = r.u(), gflags = r.u();
    if (!r.ok || !(gflags & 1) || !(gflags & 4) || alphabet_size <= offset + 1 || sequences % 2 != 0) return fail("gbwt must be bidirectional simple-sds");
    if (sequences > size) return fail("gbwt sizes");
    if (!string_array(r, tags)) return fail("gbwt tags");
    std::vector<uint64_t> rec_start; uint64_t universe; std::vector<uint8_t> data;
    if (!sparse_values(r, rec_start, universe) || !vector_u8(r, data) || universe != data.size() || rec_start.size() != alphabet_size - offset) return fail("bwt");
    skip_optional(r); skip_optional(r);          // document-array samples, metadata
    // ---- GBWTGraph ----
    const uint64_t gg = r.u(), n_graph_nodes = r.u(); r.u();
    if (!r.ok || (uint32_t)gg != 0x6B3764AFu || (gg >> 32) != 3) return fail("gbwtgraph header");
    std::vector<std::string> seqs;
    if (!string_array(r, seqs) || seqs.size() != n_graph_nodes) return fail("sequences");

    // ---- records ----
    std::vector<Record> records(rec_start.size());
    for (size_t c = 0; c < rec_start.size(); c++) {
        size_t i = rec_start[c]; const size_t end = c + 1 < rec_start.size() ? rec_start[c + 1] : data.size();
        if (i > end || end > data.size()) return fail("record bounds");
        if (i == end) continue;
        bool ok = true;
        const uint64_t sigma = bytecode(data, i, end, ok);
        uint64_t prev = 0;
        for (uint64_t e = 0; e < sigma && ok; e++) { prev += bytecode(data, i, end, ok); const uint64_t o = bytecode(data, i, end, ok); records[c].edges.push_back({prev, o}); }
        if (!ok) return fail("record edges");
        const uint64_t run_continues = sigma && sigma < 255 ? 256 / sigma : 0;
        while (i < end && sigma) {
            uint64_t rank, len;
            if (sigma >= 255) { rank = bytecode(data, i, end, ok); len = bytecode(data, i, end, ok) + 1; }
            else { const uint8_t cb = data[i++]; rank = cb % sigma; len = cb / sigma + 1; if (len == run_continues) len += bytecode(data, i, end, ok); }
            if (!ok || rank >= sigma) return fail("record runs");
            records[c].runs.push_back({(uint32_t)rank, len});
        }
    }
    // ---- the records in the library's blob layout: nothing below walks a haplotype (work ~ graph, not haplotypes x genome) ----
    // GBWT node = 2 * id + orientation; record c belongs to node c + offset; graph sequence s belongs to id first_id + s
    const uint64_t first_id = (offset + 1) / 2;
    const uint64_t n_ids = first_id + n_graph_nodes - 1;               // ids 1 .. n_ids are addressable; those below first_id stay empty
    if (n_ids == 0 || n_ids > (1u << 26)) return fail("node ids");
    std::vector<uint32_t> blob{0, 0}, rec_off(2 * (n_ids + 1), 0);
    for (size_t c = 1; c < records.size(); c++) {
        const Record& rc = records[c];
        if (rc.runs.empty()) continue;
        const uint64_t v = c + offset;
        if (v < 2 || (v >> 1) > n_ids || rc.edges.empty() || rc.edges.size() >= 1024) return fail("record node");
        if (blob.size() & 1) blob.push_back(0);
        if (blob.size() > 0xfffffff0ull) return fail("gbwt too large for 32-bit record offsets");
        rec_off[v] = (uint32_t)blob.size();
        blob.push_back((uint32_t)rc.edges.size());
        const size_t n_runs_at = blob.size(); blob.push_back(0);
        for (const auto& e : rc.edges) {
            if (e.first >= alphabet_size || (e.first != 0 && e.first <= offset) || e.second > 0xfffffff0ull) return fail("record edge");
            blob.push_back((uint32_t)e.first); blob.push_back((uint32_t)e.second);
        }
        uint32_t n_runs = 0;
        for (const auto& run : rc.runs) {
            for (uint64_t left = run.second; left > 0;) {                 // a run word holds up to 2^22 - 1 visits
                const uint64_t piece = std::min<uint64_t>(left, (1u << 22) - 1);
                blob.push_back(((uint32_t)piece << 10) | run.first); n_runs++; left -= piece;
            }
        }
        blob[n_runs_at] = n_runs;
    }
    // ---- node sequences ----
    std::vector<uint8_t> node_seq; std::vector<uint64_t> node_off(n_ids + 1, 0);
    std::vector<uint32_t> len(n_ids + 1, 0);
    for (uint64_t id = 1; id <= n_ids; id++) {
        if (id >= first_id) { const std::string& s = seqs[id - first_id]; node_seq.insert(node_seq.end(), s.begin(), s.end()); len[id] = (uint32_t)s.size(); }
        node_off[id] = node_seq.size();
    }
    // ---- build: distance payload derived from the edges of the forward records (chains of cut nodes and sites with all-pairs
    // tables, see gb_dist_payload: nested bubbles, multi-node alleles and adjacent variants are all fine), minimizers by window
    // enumeration over GBWT search states, or taken from the .min file ----
    if (node_seq.empty()) node_seq.push_back(0);
    const int rc = gb::guarded("gb_index_build_from_gbwt", [&] {
        return gb::index_build_from_gbwt(device, (uint32_t)n_ids, node_seq.data(), node_off.data(), (uint32_t)(sequences / 2), blob.data(), blob.size(),
                                         rec_off.data(), nullptr, k, w, min ? min->keys.size() : 0, min ? min->keys.data() : nullptr,
                                         min ? min->pos.data() : nullptr, out);
    });
    if (rc == GB_OK && !gb_index_has_distance_model(*out)) { gb_index_free(*out); *out = nullptr; return fail("graph outside the chain model (cycle, reversing haplotype or oversized site)"); }
    return rc;
}

extern "C" int gb_index_from_gbz(const char* path, uint32_t k, uint32_t w, gb_host_index** out) {
    return gb::guarded("gb_index_from_gbz", GB_ERR_FORMAT, [&] { return index_from_gbz_impl(path, k, w, out); }, [&] { if (out) *out = nullptr; });
}

extern "C" int gb_index_from_gbz_device(const char* path, uint32_t k, uint32_t w, int device_ordinal, gb_host_index** out) {
    return gb::guarded("gb_index_from_gbz_device", GB_ERR_FORMAT, [&] {
        if (device_ordinal < 0) { if (out) *out = nullptr; return GB_ERR_ARG; }
        return index_from_gbz_impl(path, k, w, out, nullptr, device_ordinal);
    }, [&] { if (out) *out = nullptr; });
}

extern "C" int gb_index_from_gbz_min(const char* gbz_path, const char* min_path, const char* zipcodes_path, gb_host_index** out) {
    return gb::guarded("gb_index_from_gbz_min", GB_ERR_FORMAT, [&] {
        if (!gbz_path || !min_path || !out) return GB_ERR_ARG;
        *out = nullptr;
        MinFile m;
        int rc = read_min_file(min_path, m);
        if (rc != GB_OK) return rc;
        if (m.multi) {
            // keys with several occurrences: their layout after the table is not known to this reader (see above), so the
            // table is not read — k and w come from the file, the minimizers are found on the graph (the same set: a .min IS
            // the minimizers of the haplotypes), the zipcode file is still checked for being one
            if (zipcodes_path) { uint64_t n = 0; rc = count_zipcodes(zipcodes_path, n); if (rc != GB_OK) return rc; }
            return index_from_gbz_impl(gbz_path, m.k, m.w, out, nullptr);
        }
        uint64_t oversized = 0;
        for (size_t i = 0; i < m.keys.size(); i++) if ((m.payload0[i] & 0xFF) == 0) oversized = std::max<uint64_t>(oversized, m.payload1[i] + 1);
        if (zipcodes_path) {
            uint64_t n = 0;
            rc = count_zipcodes(zipcodes_path, n);
            if (rc != GB_OK) return rc;
            if (oversized > n) return fail(".min points past the end of .zipcodes");
        }
        return index_from_gbz_impl(gbz_path, m.k, m.w, out, &m);
    }, [&] { if (out) *out = nullptr; });
}
