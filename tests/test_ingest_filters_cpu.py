"""Pins tests/ingestfilter_ref.py (the restated ingest filters and CleanSam) with hand-derived answers, each citing the Go line it follows,
then checks the column predicates of elprep_b200/filters.py and the oracle's orc_overlap against it on a seeded grid.  No GPU."""
import ctypes as C
import struct

import numpy as np
import pytest

import ingestfilter_ref as R
from ingestfilter_ref import Rec, parse_cigar as pc

INT32_MAX = (1 << 31) - 1


# ---- RemoveNonOverlappingReads (simple-filters.go:318-324) and intervals.Overlap (intervals.go:146-161) ----
@pytest.mark.parametrize("pos,cigar,expect", [
    # region [100, 200].  Overlap keeps a read iff Start <= End() - 1 and End >= POS (`intervalStart > end-1`, `intervalEnd <= start-1`):
    # the read must reach one base past the region start, and may start on the region end
    (90, "10M", False),      # ends at 99 = region start - 1
    (91, "10M", False),      # ends at 100 = region start: 100 > 100 - 1
    (92, "10M", True),       # ends at 101
    (199, "10M", True),      # starts at region end - 1
    (200, "10M", True),      # starts at region end: 200 <= 200 - 1 is false
    (201, "10M", False),     # starts at region end + 1
    (100, "1M", False),      # one base on the region start: [100, 100], 100 > 99
    (101, "1M", True),
    (200, "1M", True),
    (201, "1M", False),
])
def test_region_boundaries(pos, cigar, expect):
    flat = {0: R.flatten_regions([[100, 200]])}
    assert R.remove_non_overlapping(flat)(Rec(refid=0, pos=pos, cigar=pc(cigar))) == expect


def test_region_span_rules():
    keep = R.remove_non_overlapping({0: [(100, 200)]})
    # unmapped reads placed at their mate use [POS, POS] whatever their CIGAR says (:320-321)
    assert keep(Rec(refid=0, pos=150, flag=4, cigar=pc("500M")))
    assert not keep(Rec(refid=0, pos=50, flag=4, cigar=pc("500M")))
    # a mapped read without CIGAR operations: ReadLengthFromCigar is 0, so [POS, POS]
    assert keep(Rec(refid=0, pos=101)) and not keep(Rec(refid=0, pos=100))
    # I/S only: rl > 0, fl = 0, so End() = POS - 1 and the span is [POS, POS - 1]
    r = Rec(refid=0, pos=100, cigar=pc("5S3I"))
    assert R.read_length(r.cigar) == 8 and R.end(r) == 99 and R.aln_span(r) == (100, 99)
    assert not keep(r)                                          # Overlap(100, 99): start 100 > end - 1 = 98
    assert not keep(Rec(refid=0, pos=101, cigar=pc("5S3I")))    # [101, 100]: 100 > 99
    assert keep(Rec(refid=0, pos=102, cigar=pc("5S3I")))        # [102, 101]: 100 > 100 fails, 200 <= 101 fails -> overlaps
    # POS 0 (BAM pos -1): [0, -1 + ref length]
    assert not keep(Rec(refid=0, pos=0, cigar=pc("100M")))      # [0, 99]
    assert not keep(Rec(refid=0, pos=0, cigar=pc("101M")))      # [0, 100]
    assert keep(Rec(refid=0, pos=0, cigar=pc("102M")))          # [0, 101]
    # RNAME * and a contig without regions: ivals[RNAME] is nil
    assert not keep(Rec(refid=-1, pos=150, cigar=pc("10M")))
    assert not keep(Rec(refid=1, pos=150, cigar=pc("10M")))


def test_end_wraps_in_int32():
    r = Rec(refid=0, pos=INT32_MAX - 5, cigar=pc("10M"))
    assert R.end(r) == -(1 << 31) + 3                           # POS + 10 - 1 past 2^31 - 1 wraps
    assert R.aln_span(r) == (INT32_MAX - 5, -(1 << 31) + 3)
    assert not R.remove_non_overlapping({0: [(INT32_MAX - 100, INT32_MAX)]})(r)
    # intervals.Overlap with start = INT32_MIN: start - 1 wraps to INT32_MAX, nothing ends above it
    assert not R.overlap([(0, 10)], -(1 << 31), 5)


def test_region_flatten():
    # ParallelSortByStart + ParallelFlatten: unsorted, duplicated, contained, touching (end == next start) and adjacent intervals
    assert R.flatten_regions([[50, 60], [10, 20], [10, 20], [12, 15], [20, 30], [31, 40]]) == [(10, 30), (31, 40), (50, 60)]


# ---- RemoveMappingQualityLessThan (simple-filters.go:332-347) ----
@pytest.mark.parametrize("mq,kept", [
    (0, None), (1, [1, 254, 255]), (254, [254, 255]), (255, [255]), (256, []), (INT32_MAX, []),
    (-1, [255]), (-255, [1, 254, 255]), (-256, [0, 1, 254, 255]),
])
def test_mapq_threshold(mq, kept):
    f = R.mapq_filter(mq)
    if kept is None:
        assert f is None
    else:
        assert [q for q in (0, 1, 254, 255) if f(Rec(refid=0, pos=1, mapq=q))] == kept


# ---- RemoveNonExactMappingReads (simple-filters.go:85-99) ----
def test_non_exact_ops():
    for op in range(9):
        assert R.remove_non_exact(Rec(refid=0, pos=1, cigar=[(op, 5)])) == (op in (0, 4)), "MIDNSHP=X"[op]
    assert R.remove_non_exact(Rec(refid=0, pos=1, cigar=pc("5S90M5S")))
    assert not R.remove_non_exact(Rec(refid=0, pos=1, cigar=pc("5S45M1X44M5S")))


# ---- RemoveUnmappedReads(Strict) (simple-filters.go:73-83) and RemoveDuplicateReads (:138-140) ----
def test_unmapped_clauses():
    for flag, pos, refid, loose, strict in ((0, 5, 0, True, True), (4, 5, 0, False, False), (0, 0, 0, True, False), (0, 5, -1, True, False),
                                           (4, 0, -1, False, False), (0x400, 5, 0, True, True)):
        r = Rec(refid=refid, pos=pos, flag=flag)
        assert R.remove_unmapped(r) == loose and R.remove_unmapped_strict(r) == strict
    assert not R.remove_duplicates(Rec(refid=0, pos=1, flag=0x400)) and R.remove_duplicates(Rec(refid=0, pos=1, flag=0x4))


# ---- RemoveNonExactMappingReadsStrict (simple-filters.go:115-136) ----
GOOD = [(b"X0", "C", 1), (b"X1", "C", 0), (b"XM", "C", 0), (b"XO", "C", 0), (b"XG", "C", 0)]


def test_strict_tags():
    assert R.non_exact_strict(Rec(refid=0, pos=1, tags=GOOD))
    for k in range(5):                                          # each tag missing (`!ok`)
        assert not R.non_exact_strict(Rec(refid=0, pos=1, tags=GOOD[:k] + GOOD[k + 1:]))
    # TAGS.Get returns the first entry: good then bad keeps, bad then good drops
    assert R.non_exact_strict(Rec(refid=0, pos=1, tags=GOOD + [(b"X0", "C", 2)]))
    assert not R.non_exact_strict(Rec(refid=0, pos=1, tags=[(b"X0", "C", 2)] + GOOD))
    # every integer type compares as int64: X1 as I 2^32 - 1 is no 0, X0 as c -1 is no 1
    assert not R.non_exact_strict(Rec(refid=0, pos=1, tags=[(b"X0", "c", -1)] + GOOD[1:]))
    assert not R.non_exact_strict(Rec(refid=0, pos=1, tags=GOOD[:1] + [(b"X1", "I", (1 << 32) - 1)] + GOOD[2:]))
    # the stated deviation: a non-integer value is a mismatch (the reference's x0.(int64) would panic)
    for ty, v in (("f", 1.0), ("A", ord("1")), ("Z", b"1"), ("H", b"01"), ("Bc", [1])):
        assert not R.non_exact_strict(Rec(refid=0, pos=1, tags=[(b"X0", ty, v)] + GOOD[1:]))
    # case matters: x0 is another tag
    assert not R.non_exact_strict(Rec(refid=0, pos=1, tags=[(b"x0", "C", 1)] + GOOD[1:]))


def _bam(tags_bytes, cigar="10M", lseq=10, l_name=2, refid=0, pos0=99, mapq=30, flag=0):
    body = struct.pack("<iiBBHHHiiii", refid, pos0, l_name, mapq, 0, len(pc(cigar)), flag, lseq, -1, -1, 0) + b"r" * (l_name - 1) + b"\0"
    body += b"".join(struct.pack("<I", w) for w in R.cigar_words(pc(cigar))) + b"\0" * ((lseq + 1) // 2) + b"\x1e" * lseq + tags_bytes
    return struct.pack("<I", len(body)) + body


def test_parse_bam_tag_walk():
    t = b"MDZ10\0" + b"XXH0A1B\0" + b"ZBBs" + struct.pack("<I", 2) + struct.pack("<2h", 1, -1) + b"X0c\xff" + b"X0I" + struct.pack("<I", 7)
    r = R.parse_bam(_bam(t))
    assert r.pos == 100 and r.cigar == [(0, 10)] and r.lseq == 10
    assert [(tag, ty) for tag, ty, _ in r.tags] == [(b"MD", "Z"), (b"XX", "H"), (b"ZB", "Bs"), (b"X0", "c"), (b"X0", "I")]
    assert R.tags_get(r, b"X0") == ("c", -1)
    for bad in (b"X0C", b"ZBBs" + struct.pack("<I", 3) + struct.pack("<2h", 1, -1), b"X0q\x01", b"MDZ10"):
        with pytest.raises(R.Malformed):
            R.parse_bam(_bam(bad))
    raw = bytearray(_bam(b""))
    raw[20:24] = struct.pack("<i", 1000)                        # l_seq past block_size
    with pytest.raises(R.Malformed):
        R.parse_bam(bytes(raw))


# ---- CleanSam (simple-filters.go:292-306), softClipEndOfRead (utils.go:102-119), elementStradlessClippedRead (utils.go:81-100) ----
def clean(cigar, pos, length=1000, flag=0, refid=0, mapq=30):
    cg, mq, rw = R.clean_sam(Rec(refid=refid, pos=pos, flag=flag, mapq=mapq, cigar=pc(cigar)), [length])
    return R.ks.cigar_str([("MIDNSHP=X"[o], n) for o, n in cg]), mq, rw


def test_clean_sam_clip_points():
    # End() = 1050 > 1000: clipFrom = 1000 - 951 + 1 = 50, decremented to 49; 100M: endPos 100 >= 49 -> 49M, S of 100 + 49 (utils.go:109-113)
    assert clean("100M", 951) == ("49M149S", 30, True)
    # End() == length: no clip; length + 1: clipFrom 99 -> 98
    assert clean("100M", 901) == ("100M", 30, False)
    assert clean("100M", 902) == ("98M198S", 30, True)
    # clip point inside I: End() 1007, clipFrom 13 -> 12; 10M endPos 10 < 12 kept, pos = 10; 20I endPos 30 >= 12: rel 2, I consumes read
    # bases only, so the S grows by rel: 40 + 12 + 2 = 54 (utils.go:91-92)
    assert clean("10M20I10M", 988) == ("10M54S", 30, True)
    # clip point inside S: 5S then 100M; 5S endPos 5 < 49 kept, pos = 5; 100M: endPos 5 + 100 >= 49, rel 44 -> 44M, S 105 + 49
    assert clean("5S100M", 951) == ("5S44M154S", 30, True)
    # clip inside the leading S: clipFrom 5 -> 4: 5S endPos 5 >= 4: rel 4, S consumes read bases only: 105 + 4 + 4
    assert clean("5S100M", 996) == ("113S", 30, True)
    # on an M/I boundary: 10M20I70M, clipFrom 11 -> 10: 10M endPos 10 >= 10: rel 10 -> 10M, S 100 + 10
    assert clean("10M20I70M", 990) == ("10M110S", 30, True)
    # inside = and X
    assert clean("100=", 951) == ("49=149S", 30, True)
    assert clean("30M70X", 951) == ("30M19X149S", 30, True)


def test_clean_sam_pos_plus_end_pos():
    # `pos += endPos` (utils.go:117) adds the running end to the running position: after op k, pos = pos + endPos, not endPos.
    # 10M10I10M10I10M at 975: End() 1004, clipFrom 26 -> 25.  10M endPos 10 (pos 10); 10I endPos 20 (pos 30); 10M endPos 40 >= 25:
    # rel 25 - 30 = -5, no M; S 50 + 25.  A running sum would give 10M10I5M75S.
    assert clean("10M10I10M10I10M", 975) == ("10M10I75S", 30, True)
    # 10M10D10M10I10M at 965: End() 1004, clipFrom 36 -> 35.  endPos 10 (pos 10), 10 (pos 20), 30 (pos 50), then 10I endPos 60 >= 35:
    # rel 35 - 50 = -15, I: S 40 + 35 - 15.  A running sum would give 10M10D10M10I5M75S.
    assert clean("10M10D10M10I10M", 965) == ("10M10D10M60S", 30, True)


def test_clean_sam_d_n_panic_and_no_panic():
    # 50M10D50M at 949: clipFrom 52 -> 51: 50M endPos 50 (pos 50); 10D endPos 50 (pos 100); 50M endPos 150: rel -49, no M, S 100 + 51
    assert clean("50M10D50M", 949) == ("50M10D151S", 30, True)
    # the panic (utils.go:94-95) needs a D/N reached with rel != 0: through `pos += endPos` -- 10M10I then D at 975: clipFrom 26 -> 25,
    # endPos 10 (pos 10), 20 (pos 30), D endPos 30 >= 25, rel -5 -- or with POS past the contig end (clipFrom - 1 < 0, rel < 0 at once)
    for cigar, pos in (("10M10I10D100M", 975), ("10M10I10N100M", 975), ("10D100M", 1100), ("10N100M", 1100)):
        with pytest.raises(R.CleanSamPanic, match="Unexpected non-0 relative clipping position in CleanSam."):
            clean(cigar, pos)
    # rel 0 at the D does not panic: 10M10I10D100M at 970, clipFrom 31 -> 30: D endPos 30 >= 30, rel 0 -> only the S of 120 + 30
    assert clean("10M10I10D100M", 970) == ("10M10I150S", 30, True)
    # a leading D at clipFrom 1 -> 0: endPos 0 >= 0, rel 0 -> S of 100 + 0
    assert clean("5D100M", 1000) == ("100S", 30, True)
    # one base further in, the D is kept (endPos 0 < 1) and the clip falls in the M: rel 1
    assert clean("5D100M", 999) == ("5D1M101S", 30, True)


def test_clean_sam_past_contig_and_star():
    # POS past the end: clipFrom = 1000 - 1100 + 1 = -99 -> -100; the first operation clips with rel -100: no M, S of 100 - 100 = 0
    assert clean("100M", 1100) == ("0S", 30, True)
    # further out the S length goes negative (it is written as uint32(length) << 4)
    cg, _, _ = R.clean_sam(Rec(refid=0, pos=1200, cigar=pc("100M")), [1000])     # clipFrom -199 -> -200: S 100 - 200
    assert cg == [(4, -100)] and R.cigar_words(cg) == [((-100 << 4) | 4) & 0xFFFFFFFF]
    # RNAME * with FLAG 0x4 clear: referenceSequenceTable["*"] is 0, so End() > 0 clips from 1 - POS
    assert clean("10M", 5, refid=-1) == ("5S", 30, True)        # clipFrom -4 -> -5: rel -5, no M; S 10 - 5
    # unmapped: MAPQ 0, CIGAR untouched
    assert clean("100M", 1100, flag=4, mapq=7) == ("100M", 0, False)
    assert clean("100M", 1, flag=4, mapq=255) == ("100M", 0, False)


def test_clean_cigar_words_matches_records():
    rng = np.random.default_rng(5)
    for _ in range(500):
        ops = [(int(rng.choice([0, 1, 4, 7, 8])), int(rng.integers(1, 40))) for _ in range(int(rng.integers(1, 6)))]
        pos = int(rng.integers(800, 1100))
        w = R.cigar_words(ops)
        assert R.clean_cigar(w, pos, 1000, False) == R.cigar_words(R.clean_sam(Rec(refid=0, pos=pos, cigar=ops), [1000])[0])


# ---- the column predicates of elprep_b200/filters.py and the oracle's orc_overlap, against the restatement ----
def _grid(seed, n=4000):
    from elprep_b200 import sam
    rng = np.random.default_rng(seed)
    recs, rs = [], []
    for i in range(n):
        ops = [(int(rng.integers(0, 9)), int(rng.integers(1, 30))) for _ in range(int(rng.integers(0, 4)))]
        flag = int(rng.choice([0, 4, 0x400, 0x404, 16]))
        refid = int(rng.integers(-1, 3))
        pos = int(rng.integers(0, 400))
        mapq = int(rng.choice([0, 1, 30, 254, 255]))
        rs.append(Rec(refid=refid, pos=pos, flag=flag, mapq=mapq, cigar=ops))
        recs.append(dict(QNAME=f"q{i}", FLAG=flag, RNAME=("*", "c0", "c1", "c2")[refid + 1], POS=pos, MAPQ=mapq,
                         CIGAR="".join(f"{ln}{'MIDNSHP=X'[o]}" for o, ln in ops) or "*"))
    h = sam.Header(sq=[{"SN": "c0", "LN": 500}, {"SN": "c1", "LN": 500}, {"SN": "c2", "LN": 500}])
    return h, sam.AlignmentBatch.from_records(h, recs), rs


def _kept(flt, batch):
    t = batch.copy()
    t.tlen = np.arange(batch.n, dtype=np.int32)
    return sorted(int(x) for x in flt(t).tlen)


def test_column_filters_match_restatement():
    from elprep_b200 import filters
    h, b, rs = _grid(11)
    for flt, pred in ((filters.RemoveUnmappedReads(h), R.remove_unmapped), (filters.RemoveUnmappedReadsStrict(h), R.remove_unmapped_strict),
                      (filters.RemoveNonExactMappingReads(h), R.remove_non_exact), (filters.RemoveDuplicateReads(h), R.remove_duplicates)):
        assert _kept(flt, b) == [i for i, r in enumerate(rs) if pred(r)]
    for mq in (1, 30, 254, 255, 256, INT32_MAX, -1, -255, -256, -257):
        assert _kept(filters.RemoveMappingQualityLessThan(mq)(h), b) == [i for i, r in enumerate(rs) if R.mapq_filter(mq)(r)], mq
    assert filters.RemoveMappingQualityLessThan(0) is None
    regions = [np.array([[50, 60], [10, 20], [20, 30], [200, 210], [205, 300]]), np.array([[0, 1], [399, 400]]), np.zeros((0, 2))]
    flat = {k: R.flatten_regions(iv) for k, iv in enumerate(regions)}
    assert _kept(filters.RemoveNonOverlappingReads(regions)(h), b) == [i for i, r in enumerate(rs) if R.remove_non_overlapping(flat)(r)]


def test_orc_overlap_matches_restatement(orc):
    L = orc.lib()
    rng = np.random.default_rng(12)
    for _ in range(200):
        iv = R.flatten_regions(rng.integers(-20, 200, size=(int(rng.integers(0, 12)), 2)).cumsum(axis=1))
        a = np.array(iv, dtype=np.int32).reshape(-1)
        for _ in range(20):
            s = int(rng.integers(-30, 260))
            e = s + int(rng.integers(-3, 40))
            got = bool(L.orc_overlap(a.ctypes.data_as(C.c_void_p) if a.size else None, C.c_int64(len(iv)), C.c_int32(s), C.c_int32(e)))
            assert got == R.overlap(iv, s, e), (iv, s, e)
    for s, e in ((-(1 << 31), 5), (INT32_MAX, -(1 << 31)), (INT32_MAX - 1, INT32_MAX)):
        iv = [(-5, 10), (INT32_MAX - 3, INT32_MAX)]
        a = np.array(iv, dtype=np.int32).reshape(-1)
        assert bool(L.orc_overlap(a.ctypes.data_as(C.c_void_p), C.c_int64(2), C.c_int32(s), C.c_int32(e))) == R.overlap(iv, s, e)
