"""Plain restatement of the per-record filters of the ingest and of CleanSam, written from the reference's Go source:

  RemoveUnmappedReads / RemoveUnmappedReadsStrict           filters/simple-filters.go:71-83
  RemoveNonExactMappingReads (nonExactMappingOperator)      filters/simple-filters.go:85-99
  RemoveNonExactMappingReadsStrict                          filters/simple-filters.go:115-136 (TAGS.Get: utils.SmallMap, first entry)
  RemoveDuplicateReads                                      filters/simple-filters.go:138-140
  CleanSam                                                  filters/simple-filters.go:292-306
  RemoveNonOverlappingReads                                 filters/simple-filters.go:310-328, intervals.Overlap intervals/intervals.go:146-161
  RemoveMappingQualityLessThan                              filters/simple-filters.go:332-347
  softClipEndOfRead / elementStradlessClippedRead           filters/utils.go:81-119
  Alignment.End / ReadLengthFromCigar                       sam/sam-types.go:750-775 (int32 arithmetic: it wraps)
  parseBamAlignment and its optional-field table            sam/bam-files.go:130-283, 317-400

Two inputs: ``Rec`` (the parsed fields the filters look at; CIGARs are lists of (op code 0..8 of "MIDNSHP=X", length)) and the raw bytes
of one BAM record with its block_size (``parse_bam``).  Nothing here imports the oracle or the CUDA library: the tests compare both with it.

One stated deviation: RemoveNonExactMappingReadsStrict asserts ``x0.(int64)``, which panics when X0/X1/XM/XO/XG holds an f, A, Z, H or B
value.  The device treats such a value as a mismatch (the read is dropped); ``non_exact_strict`` does the same and says so, rather than
claiming that the reference does it.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field

import knownsites_ref as ks

OPS = "MIDNSHP=X"
CONSUMES_READ = (0, 1, 4, 7, 8)            # sam.CigarOperatorConsumesReadBases: M I S = X
CONSUMES_REF = (0, 2, 3, 7, 8)             # CigarOperatorConsumesReferenceBases: M D N = X
NON_EXACT = (1, 2, 3, 5, 6, 7, 8)          # nonExactMappingOperator: I D N H P X = (simple-filters.go:85)
F_UNMAPPED, F_DUPLICATE = 0x4, 0x400
INT_TYPES = "cCsSiI"
STRICT_WANT = ((b"X0", 1), (b"X1", 0), (b"XM", 0), (b"XO", 0), (b"XG", 0))   # simple-filters.go:117-131, in that order


def i32(x):
    """int32 arithmetic of Go: wraps"""
    return ((int(x) + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def parse_cigar(s):
    return [(OPS.index(op), n) for op, n in ks.parse_cigar(s)]


def cigar_words(c):
    """(op, length) list -> BAM u32 words; a negative length wraps as uint32(length) << 4 does in Go"""
    return [((ln << 4) | op) & 0xFFFFFFFF for op, ln in c]


def cigar_from_words(words):
    return [(int(w) & 15, int(w) >> 4) for w in words]


@dataclass
class Rec:
    refid: int                              # -1: RNAME "*"
    pos: int                                # 1-based POS
    flag: int = 0
    mapq: int = 0
    cigar: list = field(default_factory=list)
    lseq: int = 0
    qname: bytes = b"r"
    tags: list = field(default_factory=list)    # [(tag bytes, type char, value)] in record order; duplicates kept (parseBamAlignment appends)


def read_length(c):
    """sam.ReadLengthFromCigar (sam-types.go:750-756), int32"""
    n = 0
    for op, ln in c:
        n = i32(n + (ln if op in CONSUMES_READ else 0))
    return n


def ref_length(c):
    n = 0
    for op, ln in c:
        n = i32(n + (ln if op in CONSUMES_REF else 0))
    return n


def end(r):
    """Alignment.End (sam-types.go:769-775): POS + reference length - 1, int32"""
    return i32(r.pos + ref_length(r.cigar) - 1)


# ---------------------------------------------------------------- parseBamAlignment
class Malformed(ValueError):
    """a record the reference cannot parse (an index past the record, an unknown type byte) -- the device's ELP_EBAM"""


_SIZE = {"A": 1, "c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4}
_FMT = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I", "f": "<f"}


def parse_bam(raw):
    """the bytes of one record (block_size first) -> Rec.  Raises Malformed where parseBamAlignment would index past the record or find
    no parser for a type byte, and for bytes left over after the last field (the device refuses those too)."""
    raw = bytes(raw)
    if len(raw) < 36 or struct.unpack_from("<I", raw, 0)[0] + 4 != len(raw):
        raise Malformed("block_size")
    refid, pos0, l_name, mapq, _bin, n_cig, flag, l_seq = struct.unpack_from("<iiBBHHHi", raw, 4)
    if l_name < 1 or l_seq < 0:
        raise Malformed("l_read_name / l_seq")
    x = 36
    if x + l_name + 4 * n_cig + (l_seq + 1) // 2 + l_seq > len(raw):
        raise Malformed("variable part past block_size")
    qname = raw[x:x + l_name - 1]
    x += l_name
    cig = cigar_from_words(struct.unpack_from("<%dI" % n_cig, raw, x))
    x += 4 * n_cig + (l_seq + 1) // 2 + l_seq
    tags = []
    while x + 3 <= len(raw):
        tag, ty = raw[x:x + 2], chr(raw[x + 2])
        x += 3
        if ty in _SIZE:
            if x + _SIZE[ty] > len(raw):
                raise Malformed("field past block_size")
            v = raw[x] if ty == "A" else struct.unpack_from(_FMT[ty], raw, x)[0]
            x += _SIZE[ty]
        elif ty in "ZH":
            e = raw.find(b"\0", x)
            if e < 0:
                raise Malformed("string without NUL")
            v, x = raw[x:e], e + 1
        elif ty == "B":
            if x + 5 > len(raw) or chr(raw[x]) not in "cCsSiIf":
                raise Malformed("B array")
            sub, cnt = chr(raw[x]), struct.unpack_from("<I", raw, x + 1)[0]
            if x + 5 + cnt * _SIZE[sub] > len(raw):
                raise Malformed("B array past block_size")
            v = list(struct.unpack_from("<%d%s" % (cnt, _FMT[sub][1]), raw, x + 5))
            x += 5 + cnt * _SIZE[sub]
            ty = "B" + sub
        else:
            raise Malformed("unknown type %r" % ty)
        tags.append((tag, ty, v))
    if x != len(raw):
        raise Malformed("bytes after the last field")
    return Rec(refid=-1 if refid < 0 else refid, pos=i32(pos0 + 1), flag=flag, mapq=mapq, cigar=cig, lseq=l_seq, qname=qname, tags=tags)


# ---------------------------------------------------------------- the filters (True: the read stays)
def remove_unmapped(r):
    """RemoveUnmappedReads (simple-filters.go:73-75)"""
    return (r.flag & F_UNMAPPED) == 0


def remove_unmapped_strict(r):
    """RemoveUnmappedReadsStrict (:79-83): FLAG 0x4, POS 0 or RNAME *"""
    return (r.flag & F_UNMAPPED) == 0 and r.pos != 0 and r.refid >= 0


def remove_non_exact(r):
    """RemoveNonExactMappingReads (:90-99): any operation of nonExactMappingOperator drops the read"""
    return not any(op in NON_EXACT for op, _ in r.cigar)


def remove_duplicates(r):
    """RemoveDuplicateReads (:138-140): the FLAG the record comes in with"""
    return (r.flag & F_DUPLICATE) == 0


def mapq_filter(mq):
    """RemoveMappingQualityLessThan(mq int) (:332-347) -> predicate, or None (0: no filter)"""
    if mq == 0:
        return None
    if mq > 255:
        return lambda r: False
    m = int(mq) & 255                                       # byte(mq)
    return lambda r: r.mapq >= m


def tags_get(r, tag):
    """SmallMap.Get: the first entry with that key -> (type, value) or None"""
    for t, ty, v in r.tags:
        if t == tag:
            return ty, v
    return None


def non_exact_strict(r):
    """RemoveNonExactMappingReadsStrict (:115-136): X0 == 1, X1 == XM == XO == XG == 0, each present.  A non-integer value is a mismatch
    (the stated deviation: the Go type assertion panics there)."""
    for tag, want in STRICT_WANT:
        e = tags_get(r, tag)
        if e is None or e[0] not in INT_TYPES or e[1] != want:
            return False
    return True


def flatten_regions(pairs):
    """ParallelSortByStart + ParallelFlatten of one contig's regions (:311-315), as knownsites_ref restates them"""
    return [tuple(map(int, p)) for p in ks.sort_and_flatten(pairs)]


def overlap(iv, start, end_):
    """intervals.Overlap (intervals.go:146-161) over flattened, start-sorted (start, end) pairs; end - 1 and start - 1 in int32"""
    left, right = 0, len(iv) - 1
    e1, s1 = i32(end_ - 1), i32(start - 1)
    while left <= right:
        mid = (left + right) // 2
        if iv[mid][0] > e1:
            right = mid - 1
        elif iv[mid][1] <= s1:
            left = mid + 1
        else:
            return True
    return False


def aln_span(r):
    """[alnStart, alnEnd] of RemoveNonOverlappingReads (:318-324): End() only for a mapped read with read bases in its CIGAR"""
    e = r.pos
    if not r.flag & F_UNMAPPED and read_length(r.cigar) > 0:
        e = end(r)
    return r.pos, e


def remove_non_overlapping(flat):
    """RemoveNonOverlappingReads over {refid: flattened pairs}: ivals[RNAME] of a contig without regions (or "*") is nil, and Overlap(nil)
    is false"""
    def keep(r):
        s, e = aln_span(r)
        return overlap(flat.get(r.refid, []) if r.refid >= 0 else [], s, e)
    return keep


# ---------------------------------------------------------------- CleanSam
class CleanSamPanic(AssertionError):
    pass


PANIC_TEXT = "Unexpected non-0 relative clipping position in CleanSam."


def _stradless(new, op, rel, clipped):
    """elementStradlessClippedRead (utils.go:81-100)"""
    if op in CONSUMES_READ:
        if op in CONSUMES_REF:
            if rel > 0:
                new.append((op, rel))
        else:
            clipped = i32(clipped + rel)
    elif rel != 0:
        raise CleanSamPanic(PANIC_TEXT)
    new.append((4, clipped))
    return new


def soft_clip_end_of_read(clip_from, cigar):
    """softClipEndOfRead (utils.go:102-119), its arithmetic kept: `pos += endPos`, the clipped length ReadLengthFromCigar + clipFrom"""
    pos = 0
    clip_from = i32(clip_from - 1)
    new = []
    for op, ln in cigar:
        end_pos = i32(pos + (ln if op in CONSUMES_READ else 0))
        if end_pos < clip_from:
            new.append((op, ln))
        else:
            return _stradless(new, op, i32(clip_from - pos), i32(read_length(cigar) + clip_from))
        pos = i32(pos + end_pos)
    return new


def clean_sam(r, contig_lengths):
    """CleanSam (:292-306) on one read -> (CIGAR, MAPQ, rewritten).  rewritten: the CIGAR was replaced (a mapped read with End() > the
    length of its RNAME, 0 for "*"), even when the replacement equals it -- what elp_clean_sam counts.  Raises CleanSamPanic."""
    if r.flag & F_UNMAPPED:
        return list(r.cigar), 0, False
    length = contig_lengths[r.refid] if 0 <= r.refid < len(contig_lengths) else 0
    if end(r) > length:
        return soft_clip_end_of_read(i32(length - r.pos + 1), r.cigar), r.mapq, True
    return list(r.cigar), r.mapq, False


def clean_cigar(words, pos, length, unmapped):
    """CleanSam's CIGAR rewrite on BAM u32 words (the form the device arena and AlignmentBatch hold)"""
    if unmapped:
        return list(words)
    r = Rec(refid=0, pos=pos, flag=0, cigar=cigar_from_words(words))
    if end(r) > length:
        return cigar_words(soft_clip_end_of_read(i32(length - pos + 1), r.cigar))
    return list(words)
