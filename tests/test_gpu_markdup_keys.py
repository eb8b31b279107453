"""Duplicate marking and the coordinate sort's long-tie rounds on the key layouts the radix sorts specialise on.

The fragment sort orders by the group bits only and the winner is found from the score bits in the group walk; the pair sort
orders by the signature alone (64-bit keys when it fits, else 128-bit) with the pair scores kept beside it; the long-tie rounds
skip chunks that are equal on every long-run element and sort the others over their differing bits only.  Every case compares
FLAG, output order and the duplication metrics bit for bit with the oracle, and checks from kernel_stats() which sort widths
ran and how many digit passes each took (markdup_check.py restates the key widths)."""
import pytest

from elprep_b200 import sam, synth
from markdup_check import check as _check

pytestmark = pytest.mark.gpu

H = sam.Header(sq=[{"SN": "chr1", "LN": 100000}, {"SN": "chr2", "LN": 50000}],
               rg=[{"ID": "rg1", "LB": "libA"}, {"ID": "rg2", "LB": "libA"}, {"ID": "rg3", "LB": "libB"}])


def R(q, flag, pos, score, rg="rg1", rname="chr1", cigar="4M", mapq=60, **kw):
    return dict(QNAME=q, FLAG=flag, RNAME=rname, POS=pos, MAPQ=mapq, CIGAR=cigar, SEQ="ACGT", QUAL=[score] * 4, RG=rg, **kw)


def pair(q, p1, p2, s1, s2=None, flags=(99, 147), rg="rg1"):
    return [R(q, flags[0], p1, s1, RNEXT="=", PNEXT=p2, rg=rg), R(q, flags[1], p2, s1 if s2 is None else s2, RNEXT="=", PNEXT=p1, rg=rg)]


def _dups(flag, recs, name):
    return [bool(flag[i] & 0x400) for i, r in enumerate(recs) if r["QNAME"] == name]


def test_fragment_ties_later_arrival_survives():
    recs = [R("fb", 0, 100, 30), R("fa", 0, 100, 40), R("fa", 0, 100, 40), R("fc", 0, 100, 40), R("fa", 0, 100, 20),   # max 40: smallest QNAME fa, later of the two
            R("g2", 16, 100, 30), R("g1", 16, 100, 30), R("g1", 16, 100, 30),                                          # reverse strand: its own group
            R("h", 0, 200, 35, rg="rg3"), R("h", 0, 200, 35),                                                          # two libraries: two groups
            R("s", 0, 300, 25, cigar="1S3M"), R("t", 0, 299, 25)]                                                      # same unclipped position
    flag, _ = _check(sam.AlignmentBatch.from_records(H, recs), H)
    assert _dups(flag, recs, "fa") == [True, False, True] and _dups(flag, recs, "fb") == [True] and _dups(flag, recs, "fc") == [True]
    assert _dups(flag, recs, "g1") == [True, False] and _dups(flag, recs, "g2") == [True]
    assert _dups(flag, recs, "h") == [False, False]
    assert _dups(flag, recs, "s") == [False] and _dups(flag, recs, "t") == [True]


def test_groups_mixing_pair_and_fragment_reads():
    recs = ([R("f1", 0, 100, 40), R("f2", 0, 100, 45)] + pair("p1", 100, 400, 10) +              # a pair read in the group: both fragments lose
            [R("f3", 0, 500, 40), R("f4", 0, 500, 40)] +                                           # fragments only
            [R("m1", 0x1 | 0x8 | 0x40, 600, 30), R("f5", 0, 600, 50)] +                          # mate unmapped: a fragment, not a pair read
            pair("p2", 700, 900, 20) + [R("f6", 16, 900, 60)])                                   # the pair's reverse read shares the group
    flag, _ = _check(sam.AlignmentBatch.from_records(H, recs), H)
    assert _dups(flag, recs, "f1") == [True] and _dups(flag, recs, "f2") == [True] and _dups(flag, recs, "p1") == [False, False]
    assert _dups(flag, recs, "f3") == [False] and _dups(flag, recs, "f4") == [True]
    assert _dups(flag, recs, "m1") == [True] and _dups(flag, recs, "f5") == [False]
    assert _dups(flag, recs, "f6") == [True] and _dups(flag, recs, "p2") == [False, False]


def test_pair_groups_with_score_ties():
    recs = (pair("b", 100, 300, 30) + pair("a", 100, 300, 20, 40) + pair("c", 100, 300, 35, 25) + pair("a", 100, 300, 30) +   # sum 60 x4: smallest QNAME a, later pair
            pair("z", 1000, 1200, 10) + pair("y", 1000, 1200, 40) + pair("x", 1000, 1200, 10) +                                   # max score arrives in the middle
            pair("q", 2000, 2100, 30, flags=(83, 163)) + pair("q", 2000, 2100, 30, flags=(99, 147)) +                           # strands differ: two groups
            pair("r", 3000, 3100, 30, rg="rg3") + pair("r", 3000, 3100, 30))                                                    # libraries differ
    flag, _ = _check(sam.AlignmentBatch.from_records(H, recs), H)
    assert _dups(flag, recs, "a") == [True, True, False, False] and _dups(flag, recs, "b") == [True, True] and _dups(flag, recs, "c") == [True, True]
    assert _dups(flag, recs, "y") == [False, False] and _dups(flag, recs, "z") == [True, True] and _dups(flag, recs, "x") == [True, True]
    assert not any(_dups(flag, recs, "q")) and not any(_dups(flag, recs, "r"))


@pytest.mark.parametrize("seed,kw", [(1, dict(dup_frac=0.3, optical_frac=0.4)), (2, dict(dup_frac=0.5, optical_frac=0.5, unmapped_frac=0.1, mate_unmapped_frac=0.05))])
def test_synthetic_u64_pair_keys(seed, kw):
    w = synth.make_workload(20_000, [("chr20", 600_000), ("chr21", 300_000)], seed=seed, want_reference=False, **kw)
    _, stats = _check(w.batch, w.header)
    assert "radix_onesweep_u128" not in stats


def test_many_contigs_take_the_u128_pair_keys():
    contigs = [("chr1", 3_000_000)] + [(f"c{i}", 1_500) for i in range(4000)]
    w = synth.make_workload(20_000, contigs, seed=7, want_reference=False, dup_frac=0.3, optical_frac=0.4, cross_contig_frac=0.2)
    _, stats = _check(w.batch, w.header)
    assert stats["radix_onesweep_u128"]["launches"] > 0


def test_long_tie_runs_with_partly_constant_chunks():
    recs = []
    # run 1: prefix QNAMEs ("r", "r1", "r12", ...), MAPQ and TLEN constant, fragments
    for k in range(60):
        recs.append(R("r" + "123456789abcdefghij"[:k % 20], 0, 100, 30))
    # run 2: equal 16-byte prefix, differing third chunk, MAPQ varying, pairs with a distant mate
    for k in range(50):
        recs += pair(f"sameprefix16byte{(k * 7919) % 50:03d}", 500, 5000 + 10 * (k % 5), 30)
    for r in recs[60:]:
        if r["POS"] == 500:
            r["MAPQ"] = (int(r["QNAME"][-3:]) * 13) % 61
    # run 3: the reverse strand at the same position, identical names (arrival order decides)
    for k in range(40):
        recs.append(R("dup", 16, 100, 20 + k % 3))
    # an unmapped block: refid -1, TLEN 0, no mate information
    for k in range(120):
        recs.append(dict(QNAME=f"U:{(k * 31) % 120:04d}", FLAG=4, RNAME="*", POS=0, MAPQ=0, CIGAR="*", SEQ="ACGT", QUAL=[30] * 4, RG="rg2"))
    _check(sam.AlignmentBatch.from_records(H, recs), H)


def test_long_tie_runs_synthetic_unmapped_block():
    w = synth.make_workload(6_000, [("chr20", 3_000)], seed=31, unmapped_frac=0.4, dup_frac=0.6, want_reference=False)
    _check(w.batch, w.header)
