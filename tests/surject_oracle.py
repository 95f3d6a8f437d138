"""Host restatement of gb_surject_device and gb_emit_sam_device, written from vg's sources independently of the CUDA code
(surject.cu, sam_format.h), so the device is checked against a second implementation.

  chunks        Surjector::extract_overlapping_paths (surjector.cpp:4109-4260): a mapping extends the chunk of the previous
                mapping when its step is the next step of the same path strand
  route         realigning_surject (:3223-3253): no chunk -> unmapped; one chunk over the whole read -> copied over;
                anything else is vg's realigning route, which this library does not build: the record, and its mate when
                paired, are deferred (route 2) and get no SAM line
  score         EditAlignmentScorer::score_contiguous_alignment (alignment_scorer.cpp:159-245)
  CIGAR         cigar_against_path / mapping_cigar / simplify_cigar (alignment.cpp:1253-1283, :1339-1391, :1518-1570)
  pairs         compute_template_lengths (alignment.cpp:2838-2896), determine_flag / sam_flag (:697-754, :2898-2931)
  SAM line      alignment_to_sam_internal (alignment.cpp:607-695)

What cannot be pinned without the vg binary: the TLEN of a pair with no mapped mate (compute_template_lengths then
subtracts INT64_MAX from INT64_MIN; restated here with the wrap-around a two's-complement build gives).  The choices vg
makes only on the realigning route (tie order among equal-scoring path strands in choose_primary_strand, co-optimal
banded-global paths) do not arise: a direct-route read has a place on one path strand only, and its path is copied.

The oracle is Python beside the tests rather than C++ in oracle/: that library restates the mapper, and surjection needs
nothing from it but the records; in Python the restatement reads line for line against vg's C++ and shares no code, not
even a language, with surject.cu and sam_format.h."""
import numpy as np

import helpers as H


def ref_index(paths, node_len):
    """paths: [(name, [oriented node, ...])] -> ({node id: (path, walks reversed, offset, step)}, [lengths])."""
    where, lengths = {}, []
    for p, (_, nodes) in enumerate(paths):
        off = 0
        for step, v in enumerate(nodes):
            where[v >> 1] = (p, v & 1, off, step)
            off += node_len[v]
        lengths.append(off)
    return where, lengths


def _chunks(path, where):
    """[(path, strand, first mapping, last mapping)] in the order extract_overlapping_paths opens them."""
    out, prev = [], None                      # prev = (path, strand, step, chunk index) of the previous mapping
    for i, (node, _, _) in enumerate(path):
        w = where.get(node >> 1)
        if w is None:
            prev = None
            continue
        p, walk_rev, _, step = w
        strand = (node & 1) ^ walk_rev
        want = None if prev is None else prev[2] + (1 if strand == 0 else -1)
        if prev is not None and prev[0] == p and prev[1] == strand and step == want:
            c = prev[3]
            out[c] = (p, strand, out[c][2], i)
        else:
            c = len(out)
            out.append((p, strand, i, i))
        prev = (p, strand, step, c)
    return out


def _score(path, sc):
    match, mismatch, gap_open, gap_extend, bonus = sc
    score, last_del = 0, False
    for i, (_, _, edits) in enumerate(path):
        for j, (op, ln, _) in enumerate(edits):
            if op == "M":
                score += match * ln; last_del = False
            elif op == "S":
                score -= mismatch * ln; last_del = False
            elif op == "D":
                score -= ln * gap_extend if last_del else gap_open + (ln - 1) * gap_extend
                last_del = True
            else:
                if not ((i == 0 and j == 0) or (i == len(path) - 1 and j == len(edits) - 1)):
                    score -= gap_open + (ln - 1) * gap_extend
                last_del = False
    clip_start = bool(path[0][2]) and path[0][2][0][0] == "I"
    clip_end = bool(path[-1][2]) and path[-1][2][-1][0] == "I"
    return score + (0 if clip_start else bonus) + (0 if clip_end else bonus)


def _append(cigar, n, op):
    if cigar and cigar[-1][1] == op:
        cigar[-1][0] += n
    else:
        cigar.append([n, op])


def _simplify(cigar):
    out, i = [], 0
    while i < len(cigar):
        if cigar[i][1] not in "ID":
            out.append(cigar[i]); i += 1
            continue
        j = i
        while j < len(cigar) and cigar[j][1] in "ID":
            j += 1
        if j - i >= 2:
            out += [[sum(c[0] for c in cigar[i:j] if c[1] == "D"), "D"], [sum(c[0] for c in cigar[i:j] if c[1] == "I"), "I"]]
        else:
            out.append(cigar[i])
        i = j
    res = []
    for c in out:
        if c[0] == 0:
            continue
        if res and res[-1][1] == c[1]:
            res[-1][0] += c[0]
        else:
            res.append(list(c))
    return res


def cigar_against_path(path, rev):
    cigar = []
    for _, _, edits in path:
        for op, ln, _ in edits:
            _append(cigar, ln, {"M": "M", "S": "M", "I": "I", "D": "D"}[op])
    if rev:
        cigar.reverse()
    if len(cigar) > 1 and cigar[-1][1] == "D" and cigar[-2][1] == "I":
        cigar[-1], cigar[-2] = cigar[-2], cigar[-1]
    if cigar[-1][1] == "I":
        cigar[-1][1] = "S"
    if len(cigar) > 1 and cigar[0][1] == "D" and cigar[1][1] == "I":
        cigar[0], cigar[1] = cigar[1], cigar[0]
    if cigar[0][1] == "I":
        cigar[0][1] = "S"
    return [tuple(c) for c in _simplify(cigar)]


def surject_one(flags, score_mapq_path, where, node_len, sc):
    """One record -> dict(ref, pos, rev, route, score, mapq, cigar, flag)."""
    _, mapq, path = score_mapq_path
    r = dict(ref=-1, pos=-1, rev=False, route=1, score=0, mapq=0, cigar=[], flag=0x4)
    if flags & 2:
        r["flag"] |= 0x100
    if flags & 16:
        r["route"] = 3
        return r
    if not (flags & 1) or not path:
        return r
    chunks = _chunks(path, where)
    if not chunks:
        return r
    if len(chunks) != 1 or chunks[0][2] != 0 or chunks[0][3] != len(path) - 1:
        r["route"] = 2
        return r
    p, strand = chunks[0][0], chunks[0][1]
    if strand == 0:
        node, off, _ = path[0]
        pos = where[node >> 1][2] + off
    else:
        node, off, edits = path[-1]
        from_len = sum(ln for op, ln, _ in edits if op != "I")
        pos = where[node >> 1][2] + node_len[node] - off - from_len
    return dict(ref=p, pos=pos, rev=bool(strand), route=0, score=_score(path, sc), mapq=mapq,
                cigar=cigar_against_path(path, bool(strand)), flag=(0x10 if strand else 0) | (r["flag"] & 0x100))


def _bounds(rec):
    lo, hi = 2 ** 63 - 1, -2 ** 63
    here = rec["pos"]
    if rec["ref"] < 0:
        return lo, hi
    for n, op in rec["cigar"]:
        if op == "M":
            lo, hi = min(lo, here), max(hi, here + n)
        if op in "MD":
            here += n
    return lo, hi


def _wrap32(v):
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= 1 << 31 else v


def template_lengths(r1, r2):
    (lo1, hi1), (lo2, hi2) = _bounds(r1), _bounds(r2)
    dist = _wrap32(max(hi1, hi2) - min(lo1, lo2))
    return (dist, -dist) if (lo1 < lo2 or (lo1 == lo2 and hi1 < hi2)) else (-dist, dist)


def surject(aln, maps, edits, paths, node_len, sc=(1, 4, 6, 1, 5), tlen_max=0):
    """All records (the layout gb_surject_device takes) -> list of dicts with the gb_sam_record fields and the CIGAR."""
    where, _ = ref_index(paths, node_len)
    out = []
    for a in aln:
        d = surject_one(int(a["flags"]), H.decode_alignment(a, maps, edits), where, node_len, sc)
        d.update(read_id=int(a["read_id"]), mate_ref=-1, mate_pos=-1, tlen=0)
        out.append(d)
    for x in range(0, len(aln) - 1, 2):
        if not (int(aln[x]["flags"]) & 4):
            continue
        i1 = x if int(aln[x]["read_id"]) % 2 == 0 else x + 1
        r1, r2 = out[i1], out[i1 ^ 1]
        if 2 in (r1["route"], r2["route"]):                   # deferred together: the mate fields depend on both
            for r in (r1, r2):
                if r["route"] != 3:
                    r.update(ref=-1, pos=-1, rev=False, route=2, score=0, mapq=0, cigar=[], flag=0x4 | (r["flag"] & 0x100))
            continue
        r1["tlen"], r2["tlen"] = template_lengths(r1, r2)
        r1["mate_ref"], r1["mate_pos"], r2["mate_ref"], r2["mate_pos"] = r2["ref"], r2["pos"], r1["ref"], r1["pos"]
        for r, m in ((r1, r2), (r2, r1)):
            f = r["flag"] | 0x1 | (0x80 if r["read_id"] % 2 else 0x40)
            if r["ref"] >= 0 and m["ref"] == r["ref"]:
                facing = (r["pos"] <= m["pos"] and not r["rev"] and m["rev"]) or (m["pos"] <= r["pos"] and r["rev"] and not m["rev"])
                if facing and (tlen_max == 0 or abs(r["tlen"]) <= tlen_max):
                    f |= 0x2
            if m["ref"] < 0:
                f |= 0x8
            if m["rev"]:
                f |= 0x20
            r["pflag"] = f
        r1["flag"], r2["flag"] = r1.pop("pflag"), r2.pop("pflag")
    return out


_COMP = str.maketrans("ACGTacgt", "TGCAtgca")


def sam_line(r, names, reads, quals, path_names):
    """alignment_to_sam_internal for one surjected record (names / quals may be None)."""
    rid = r["read_id"]
    paired = bool(r["flag"] & 1)
    name = names[rid] if names is not None else f"read{rid}"
    if paired and len(name) >= 2 and name[-1] in "12" and name[-2] in "/_":
        name = name[:-2]
    mapped = r["ref"] >= 0
    rev = bool(r["flag"] & 0x10)
    use_mate_loc = not mapped and paired and r["mate_ref"] >= 0
    seq = reads[rid]
    qual = None if quals is None else quals[rid]
    cols = [name or "*", str(r["flag"]),
            path_names[r["ref"]] if mapped else (path_names[r["mate_ref"]] if use_mate_loc else "*"),
            str((r["mate_pos"] if use_mate_loc else r["pos"]) + 1),
            str(r["mapq"] if mapped else 0),
            "".join(f"{n}{op}" for n, op in r["cigar"]) if mapped else "*",
            "*" if r["mate_ref"] < 0 else ("=" if r["mate_ref"] == r["ref"] else path_names[r["mate_ref"]]),
            str(r["mate_pos"] + 1), str(r["tlen"]),
            (seq[::-1].translate(_COMP) if rev else seq) if seq else "*",
            "".join(chr(q + 33) for q in (qual[::-1] if rev else qual)) if qual is not None and len(qual) else "*"]
    return "\t".join(cols) + f"\tAS:i:{r['score']}\n"


def sam_text(recs, names, reads, quals, path_names):
    return "".join(sam_line(r, names, reads, quals, path_names) for r in recs if r["route"] not in (2, 3))


def decode_device(rec_bytes, cigar):
    """gb_sam_record bytes + cigar pool -> the dicts surject() returns (without the oracle's 'rev')."""
    from vg_b200 import capi
    recs = np.frombuffer(rec_bytes, dtype=capi.sam_record_dt)
    out = []
    for r in recs:
        c = [(int(w) >> 4, "MIDNSHP=X"[int(w) & 15]) for w in cigar[int(r["cigar_off"]): int(r["cigar_off"]) + int(r["n_cigar"])]]
        out.append(dict(read_id=int(r["read_id"]), flag=int(r["flag"]), mapq=int(r["mapq"]), route=int(r["route"]), ref=int(r["ref"]),
                        pos=int(r["pos"]), score=int(r["score"]), mate_ref=int(r["mate_ref"]), mate_pos=int(r["mate_pos"]),
                        tlen=int(r["tlen"]), cigar=c))
    return out
