// fastq.cpp — ORACLE (test infrastructure): vg's FASTQ reader over an in-memory buffer, the parity reference of
// gb_fastq_parse_device and the host baseline of scripts/bench_input.py.
//
// Restates vgteam/vg @ fd49b9a9:
//   get_next_alignment_from_fastq                 src/alignment.cpp:159-250 (FASTQ branch: one sequence line)
//   get_next_interleaved_alignment_pair_from_fastq src/alignment.cpp:252-254
//   get_next_alignment_pair_from_fastqs           src/alignment.cpp:256-258
//   check_quality_length                          src/alignment.cpp:4548
//   toUppercaseInPlace of every read              src/subcommand/giraffe_main.cpp:2319-2320, :2433
//   whitespace = " \t\n\v\f\r"                     src/utility.hpp:56
// gzgets is read as "the next line, with its '\n' when there is one"; vg's fixed line buffer and C-string handling of
// NUL bytes are not modelled.  strict != 0 adds the refusals where gb_fastq_parse_device diverges from vg on purpose:
// a separator line not starting with '+', a quality length that differs from the sequence's (vg also accepts an empty
// quality line), a byte outside '!'..'~' in a sequence or quality line, and a last line without '\n'.
#include <cstdint>
#include <cstring>
#include <string>

#include "../include/giraffe_b200.h"

namespace {

enum : int { FQ_HEADER = 1, FQ_SEQ_BYTE = 2, FQ_SEPARATOR = 3, FQ_QUAL_LEN = 4, FQ_QUAL_BYTE = 5, FQ_INCOMPLETE = 6 };

struct Reader {
    const uint8_t* p;
    uint64_t n, pos = 0;
    bool gets(std::string& line) {                     // gzgets: 0 at the end of the input
        if (pos >= n) return false;
        const void* e = std::memchr(p + pos, '\n', n - pos);
        const uint64_t end = e ? (uint64_t)((const uint8_t*)e - p) + 1 : n;
        line.assign((const char*)p + pos, end - pos);
        pos = end;
        return true;
    }
};

struct Record { std::string name, seq, qual; };

bool printable(const std::string& s) {
    for (unsigned char c : s) if (c < '!' || c > '~') return false;
    return true;
}

// 1: a record, 0: the end of the input, < 0: -(the refusal)
int next_record(Reader& r, Record& rec, bool strict) {
    std::string line;
    if (!r.gets(line)) return 0;                                    // :164, no more to get
    std::string name_line = line.substr(0, line.size() - 1);       // :165, buffer[strlen(buffer) - 1] = '\0'
    if (name_line.empty() || name_line[0] != '@') return -FQ_HEADER;   // :167-173 ('>' is FASTA: not restated)
    const size_t div = name_line.find_first_of(" \t\n\v\f\r");     // :175-176
    rec.name = name_line.substr(1, div == std::string::npos ? std::string::npos : div - 1);
    if (!r.gets(line)) return -FQ_INCOMPLETE;                       // :190-194, there was no sequence
    rec.seq = line;                                                 // :199-206, one line; the '\n' dropped
    if (!rec.seq.empty() && rec.seq.back() == '\n') rec.seq.pop_back();
    std::string sep;
    if (!r.gets(sep)) return -FQ_INCOMPLETE;                        // :233-235
    if (!r.gets(line)) return -FQ_INCOMPLETE;                       // :237-244
    const bool terminated = !line.empty() && line.back() == '\n';
    const std::string q = line.substr(0, line.size() - 1);         // :238, the last byte chopped whatever it is
    if (strict) {
        if (!printable(rec.seq)) return -FQ_SEQ_BYTE;
        if (sep.empty() || sep[0] != '+') return -FQ_SEPARATOR;
        if (!terminated) return -FQ_INCOMPLETE;
        if (q.size() != rec.seq.size()) return -FQ_QUAL_LEN;
        if (!printable(q)) return -FQ_QUAL_BYTE;
    } else if (!q.empty() && q.size() != rec.seq.size()) {
        return -FQ_QUAL_LEN;                                        // check_quality_length, :4548
    }
    rec.qual = q;
    for (char& c : rec.qual) c = (char)(c - 33);                    // string_quality_char_to_short
    for (char& c : rec.seq) if (c >= 'a' && c <= 'z') c = (char)(c - 32);   // toUppercaseInPlace
    return 1;
}

} // namespace

/* The whole input, as vg giraffe reads it: n_inputs 1 (single-end, or interleaved pairs with GB_FASTQ_INTERLEAVED) or 2
 * (record i of each input makes pair i: reads 2i and 2i + 1).  Outputs as gb_fastq_parse_device; the buffers hold what the
 * caller sized them for (reads / quals / names: the total text bytes; read_off / name_off: max_records + 1).  Returns 0,
 * GB_ERR_CAPACITY when there are more than max_records reads, or GB_ERR_FORMAT with err = {input, record, kind}
 * (kind 1 header, 2 sequence byte, 3 separator, 4 quality length, 5 quality byte, 6 incomplete record). */
extern "C" int oracle_fastq_parse(uint32_t n_inputs, const uint8_t* const* text, const uint64_t* text_bytes, uint32_t flags, int strict,
                                  uint64_t max_records, uint8_t* reads, uint8_t* quals, uint64_t* read_off, uint8_t* names,
                                  uint64_t* name_off, uint32_t* n_reads, uint32_t* max_read_len, int64_t* err) {
    Reader in[2] = {{text[0], text_bytes[0]}, {n_inputs > 1 ? text[1] : nullptr, n_inputs > 1 ? text_bytes[1] : 0}};
    const bool paired = n_inputs == 2 || (flags & GB_FASTQ_INTERLEAVED);
    uint64_t n = 0, rec_index[2] = {0, 0};
    uint32_t mx = 0;
    read_off[0] = name_off[0] = 0;
    Record rec[2];
    for (;;) {
        const int k = paired ? 2 : 1;
        int got = 1;
        for (int m = 0; m < k && got == 1; m++) {
            const uint32_t t = n_inputs == 2 ? (uint32_t)m : 0;
            got = next_record(in[t], rec[m], strict != 0);
            if (got < 0) { err[0] = t; err[1] = (int64_t)rec_index[t]; err[2] = -got; return GB_ERR_FORMAT; }
            if (got == 1) rec_index[t]++;
        }
        if (got == 0) break;                                        // a mate without its partner is dropped (:252-258)
        for (int m = 0; m < k; m++) {
            if (n == max_records) return GB_ERR_CAPACITY;
            const Record& r = rec[m];
            std::memcpy(reads + read_off[n], r.seq.data(), r.seq.size());
            if (!r.qual.empty()) std::memcpy(quals + read_off[n], r.qual.data(), r.qual.size());
            else std::memset(quals + read_off[n], 0, r.seq.size());
            std::memcpy(names + name_off[n], r.name.data(), r.name.size());
            read_off[n + 1] = read_off[n] + r.seq.size();
            name_off[n + 1] = name_off[n] + r.name.size();
            if (r.seq.size() > mx) mx = (uint32_t)r.seq.size();
            n++;
        }
    }
    *n_reads = (uint32_t)n;
    *max_read_len = mx;
    return 0;
}
