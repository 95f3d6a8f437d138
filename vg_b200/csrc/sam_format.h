// sam_format.h — the SAM alignment line of one surjected record (gb_sam_record), and the check a record must pass before it
// is formatted.  emit_device.cu drives it with the Count / Write sinks of emit_format.h, as it drives GAF and GAM.
//
// The line is alignment_to_sam_internal (alignment.cpp:607-695) field for field:
//   QNAME  the read's name; paired records (FLAG 0x1) lose a trailing [/_][12] (alignment.cpp:626-629); '*' when empty
//   FLAG   as gb_surject_device set it
//   RNAME  the path's name when mapped; an unmapped paired record with a mapped mate takes the mate's (SAMv1 §2.4.1,
//          alignment.cpp:646-659); '*' otherwise
//   POS    1-based: pos + 1, or mate_pos + 1 in the mate-location case (so 0 when unmapped)
//   MAPQ, CIGAR   '0' and '*' when unmapped
//   RNEXT  '*' without a mate location, '=' when it is RNAME's path (compared with the record's own ref), else its name
//   PNEXT  mate_pos + 1;  TLEN
//   SEQ    reverse-complemented when FLAG has 0x10; QUAL reversed then, raw Phred + 33, '*' without qualities
//   AS:i:score
// No RG, SS, GR or NR tags (giraffe's defaults write none).
#pragma once
#include "emit_format.h"

namespace gb {
namespace {

struct SamArgs {
    uint32_t n; const gb_sam_record* rec;
    const uint32_t* cigar; uint64_t cigar_len;
    uint32_t n_reads; const uint8_t* reads; const uint8_t* quals; const uint64_t* read_off;
    const uint8_t* names; const uint64_t* name_off;                      // names == NULL: read<i>
    uint32_t n_paths; const uint8_t* path_names; const uint64_t* path_name_off;
};

constexpr uint32_t BAM_CMATCH = 0, BAM_CINS = 1, BAM_CDEL = 2, BAM_CSOFT_CLIP = 4;

// Absent ranks have no record; records left to the realigning route are surjected by the caller.
GB_FMT_INLINE bool sam_present(const gb_sam_record& r) { return r.route != GB_SURJ_ABSENT && r.route != GB_SURJ_REALIGN; }

GB_FMT_INLINE bool sam_name_valid(const SamArgs& A, uint32_t i) {
    return !(A.names && A.name_off) || A.name_off[i + 1] >= A.name_off[i];
}

// A record must stay inside its read, the cigar pool and the paths, and its CIGAR must consume the read.
GB_FMT bool sam_record_valid(const SamArgs& A, const gb_sam_record& r) {
    if (!sam_present(r)) return true;
    if (r.read_id >= A.n_reads || A.read_off[r.read_id + 1] < A.read_off[r.read_id]) return false;
    if (r.ref < -1 || r.ref >= (int64_t)A.n_paths || r.mate_ref < -1 || r.mate_ref >= (int64_t)A.n_paths) return false;
    if (r.ref < 0) return true;
    if (!A.cigar || (uint64_t)r.cigar_off + r.n_cigar > A.cigar_len || r.n_cigar == 0) return false;
    uint64_t q = 0;
    for (uint32_t i = 0; i < r.n_cigar; i++) {
        const uint32_t op = A.cigar[r.cigar_off + i] & 15u;
        if (op != BAM_CMATCH && op != BAM_CINS && op != BAM_CDEL && op != BAM_CSOFT_CLIP) return false;
        if (op != BAM_CDEL) q += A.cigar[r.cigar_off + i] >> 4;
    }
    return q == A.read_off[r.read_id + 1] - A.read_off[r.read_id];
}

template <class S> GB_FMT void path_name(S& s, const SamArgs& A, int32_t p) {
    s.put(A.path_names + A.path_name_off[p], A.path_name_off[p + 1] - A.path_name_off[p]);
}

GB_FMT_INLINE char complement(char c) {
    switch (c) { case 'A': return 'T'; case 'C': return 'G'; case 'G': return 'C'; case 'T': return 'A';
                 case 'a': return 't'; case 'c': return 'g'; case 'g': return 'c'; case 't': return 'a'; default: return c; }
}

// One SAM line, its newline included.
template <class S> GB_FMT void sam_line(S& s, const SamArgs& A, const gb_sam_record& r) {
    const uint32_t id = r.read_id;
    const uint8_t* seq = A.reads + A.read_off[id];
    const uint32_t L = (uint32_t)(A.read_off[id + 1] - A.read_off[id]);
    const bool mapped = r.ref >= 0, rev = (r.flag & 0x10u) != 0, paired = (r.flag & 0x1u) != 0;
    // QNAME
    if (A.names && A.name_off) {
        const uint8_t* nm = A.names + A.name_off[id];
        uint64_t k = A.name_off[id + 1] - A.name_off[id];
        if (paired && k >= 2 && (nm[k - 1] == '1' || nm[k - 1] == '2') && (nm[k - 2] == '/' || nm[k - 2] == '_')) k -= 2;
        if (k) s.put(nm, k); else s.ch('*');
    } else {
        lit(s, "read"); unum(s, id);
    }
    s.ch('\t'); unum(s, r.flag); s.ch('\t');
    const bool use_mate_loc = !mapped && paired && r.mate_ref >= 0;
    if (mapped) path_name(s, A, r.ref); else if (use_mate_loc) path_name(s, A, r.mate_ref); else s.ch('*');
    s.ch('\t'); snum(s, (int64_t)(use_mate_loc ? r.mate_pos : r.pos) + 1);
    s.ch('\t'); unum(s, mapped ? r.mapq : 0); s.ch('\t');
    if (mapped) {
        for (uint32_t i = 0; i < r.n_cigar; i++) {
            const uint32_t c = A.cigar[r.cigar_off + i];
            unum(s, c >> 4); s.ch("MIDNSHP=X"[c & 15u]);
        }
    } else {
        s.ch('*');
    }
    s.ch('\t');
    if (r.mate_ref < 0) s.ch('*'); else if (r.mate_ref == r.ref) s.ch('='); else path_name(s, A, r.mate_ref);
    s.ch('\t'); snum(s, (int64_t)r.mate_pos + 1); s.ch('\t'); snum(s, r.tlen); s.ch('\t');
    if (!L) s.ch('*');
    else if (!rev) s.put(seq, L);
    else if constexpr (S::counting) s.n += L;
    else for (uint32_t i = L; i-- > 0;) s.ch(complement((char)seq[i]));
    s.ch('\t');
    if (!A.quals || !L) s.ch('*');
    else if constexpr (S::counting) s.n += L;
    else {
        const uint8_t* qv = A.quals + A.read_off[id];
        for (uint32_t i = 0; i < L; i++) s.ch((char)(qv[rev ? L - 1 - i : i] + 33));
    }
    lit(s, "\tAS:i:"); snum(s, r.score);
    s.ch('\n');
}

} // namespace
} // namespace gb
