"""The expected results of elp_filter_target_regions (tests/targetregions_ref.py) pinned on hand-built reads: which reads the
RemoveNonOverlappingReads predicate keeps at a region's edges, and a pair whose FLAGs differ between the reference order (mark every read,
then filter) and the ingest-filter order (filter, then mark)."""
import numpy as np

import targetregions_ref as T
from elprep_b200 import sam

H = sam.Header(sq=[{"SN": "c0", "LN": 10000}, {"SN": "c1", "LN": 10000}], rg=[{"ID": "g1", "LB": "l1"}])


def rec(name, pos, cigar="10M", flag=0, rname="c0", mapq=60, q=30, rnext="*", pnext=0):
    n = sum(int(x) for x in __import__("re").findall(r"(\d+)[MIS=X]", cigar)) if cigar != "*" else 10
    return dict(QNAME=name, FLAG=flag, RNAME=rname, POS=pos, MAPQ=mapq, CIGAR=cigar, RNEXT=rnext, PNEXT=pnext, SEQ="ACGT" * (n // 4) + "ACGT"[:n % 4],
                QUAL=[q] * n, RG="g1")


def test_keep_set_at_region_edges():
    # region [100, 200] on c0; a read [POS, alnEnd] overlaps iff 100 < alnEnd + 1 - 1 ... i.e. start <= alnEnd - 1 and end >= POS
    # (intervals.Overlap compares with end - 1 and start - 1)
    cases = [
        (rec("a", 90), False),               # [90, 99]: ends before the start
        (rec("b", 91), False),               # [91, 100]: ends ON the start -- Overlap needs start <= alnEnd - 1
        (rec("c", 92), True),                # [92, 101]
        (rec("d", 200), True),               # starts on the end
        (rec("e", 201), False),              # starts after it
        (rec("f", 150, flag=4), True),       # unmapped at its mate's position: [150, 150]
        (rec("g", 100, flag=4), False),      # unmapped: [100, 100] ends on the start
        (rec("h", 100, flag=4, cigar="20M"), False),   # an unmapped read's CIGAR does not count
        (rec("i", 150, rname="*"), False),   # RNAME *
        (rec("j", 150, cigar="*"), True),    # no read bases: [POS, POS]
        (rec("k", 150, cigar="5H"), True),   # hard clips only: no read bases either
        (rec("l", 95, cigar="2S3M20D3M"), True),   # End() counts M D N = X: [95, 120]
        (rec("m", 150, rname="c1"), False),  # a contig without regions
    ]
    b = sam.AlignmentBatch.from_records(H, [r for r, _ in cases])
    got = T.keep_mask(b, {0: [(100, 200)]})
    assert got.tolist() == [k for _, k in cases]
    # the same reads through the reference order without marking and in arrival order
    res = T.mark_then_filter(None, {0: [(100, 200)]}, sort="keep", markdup=False, bqsr=False, batch=b)
    assert res["perm"].tolist() == [i for i, (_, k) in enumerate(cases) if k]
    assert res["n_removed"] == sum(1 for _, k in cases if not k)


def test_unsorted_overlapping_regions_flatten():
    b = sam.AlignmentBatch.from_records(H, [rec("a", 305), rec("b", 350), rec("c", 412)])
    # (400, 420) and (300, 310) unsorted; (305, 401) bridges them into one region [300, 420]
    assert T.keep_mask(b, {0: [(400, 420), (300, 310), (305, 401)]}).tolist() == [True, True, True]
    assert T.keep_mask(b, {0: [(400, 420), (300, 310)]}).tolist() == [True, False, True]


def _pairs():
    """pair A (QUAL 30) and pair B (QUAL 20) with the same unclipped 5' ends: B loses the pair group.  Their second mates lie at 5000,
    outside the region [50, 400].  Fragment F shares A's first mate's 5' end."""
    recs = []
    for name, q in (("A", 30), ("B", 20)):
        recs.append(rec(name, 100, flag=0x1 | 0x2 | 0x20 | 0x40, q=q, rnext="=", pnext=5000))
        recs.append(rec(name, 5000, flag=0x1 | 0x2 | 0x10 | 0x80, q=q, rnext="=", pnext=100))
    recs.append(rec("F", 100, q=40))
    return sam.AlignmentBatch.from_records(H, recs)


def test_marking_before_filtering_differs_from_ingest_filter():
    import oracle
    oracle.build()
    b = _pairs()
    regions = {0: [(50, 400)]}
    w = type("W", (), {"header": H})()
    ref = T.mark_then_filter(w, regions, bqsr=False, batch=b)
    # reference order: B's first mate stays a duplicate of pair A, and fragment F is a duplicate because pairs shadow fragments
    assert ref["perm"].tolist() == [0, 2, 4]
    assert [int(f) & 0x400 for f in ref["flag"]] == [0, 0x400, 0x400]
    assert ref["n_removed"] == 2
    # ingest-filter order: without their mates A and B never complete a pair group, so B's first mate is no longer a duplicate
    # (F is still shadowed by them)
    idx, flag = T.ingest_then_mark(H, b, regions)
    assert idx.tolist() == [0, 2, 4]
    assert [int(f) & 0x400 for f in flag] == [0, 0, 0x400]
