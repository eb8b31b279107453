"""The known-sites masking of BQSR on the CPU: the restatement in knownsites_ref.py against brute-force definitions, and the oracle (the
CPU restatement of the reference that the device tests compare with) against the restatement: read coordinates over a grid of CIGARs,
Flatten / ParallelFlatten over awkward interval lists, and the bases bqsr_gather counts on hand-made single reads."""
import ctypes as C

import numpy as np
import pytest

import knownsites_cases as kc
import knownsites_ref as ks
from elprep_b200 import sam

SOFT_START = 1000

CIGARS = ["60M", "5S55M", "55M5S", "5S50M5S", "5H55M", "55M5H", "3H5S50M5S2H",
          "3I57M", "30M3I27M", "57M3I", "2S3I55M",
          "3D60M", "30M3D30M", "60M3D", "30M3N30M",
          "30M2I3D28M", "30M3D2I28M", "1M1I58M", "58M1I1M", "1M1D59M", "59M1D1M",
          "5H3I52M", "5S3I52M", "2S10M2D10M2I10M2D10M2I14M", "10M1I1D1I48M"]


def _probe(orc, c, ref, tail):
    a = np.array(sam.encode_cigar(ks.cigar_str(c)), dtype=np.uint32)
    ok = C.c_int()
    rb = orc.lib().orc_probe_readcoord(a.ctypes.data_as(C.c_void_p), C.c_int32(len(a)), C.c_int(SOFT_START), C.c_int(ref), C.c_int(tail), C.byref(ok))
    return rb, bool(ok.value)


@pytest.mark.parametrize("cigar", CIGARS)
def test_read_coordinate_grid(orc, cigar):
    """every reference coordinate from softStart - 2 to softEnd + 2, both tails"""
    c = ks.parse_cigar(cigar)
    pos = SOFT_START + sum(n for op, n in c[:next(i for i, (op, _) in enumerate(c) if op not in "HS")] if op == "S")
    assert ks.soft_start(pos, c) == SOFT_START
    end = ks.soft_end(pos, c)
    seen_fail = seen_ok = 0
    for ref in range(SOFT_START - 2, end + 3):
        for tail in (0, 1):
            rb, ok = ks.get_read_coord(c, SOFT_START, ref, tail_right=bool(tail))
            orb, ook = _probe(orc, c, ref, tail)
            assert ok == ook, (cigar, ref, tail)
            if ok:
                assert rb == orb, (cigar, ref, tail, rb, orb)
                seen_ok += 1
            else:
                seen_fail += 1
    assert seen_ok and seen_fail          # the range reaches both failures (before softStart) and successes


def test_read_coordinate_quirks():
    """hand-derived values of the quirks the masking depends on"""
    g = lambda cg, ref, tail=False: ks.get_read_coord(ks.parse_cigar(cg), 1000, ref, tail)
    assert g("10M5D140M", 1012) == (9, True) and g("10M5D140M", 1012, True) == (10, True)     # inside a deletion
    assert g("10M5D140M", 1010) == (9, True) and g("10M5D140M", 1010, True) == (10, True)     # first deleted base: ends just before
    assert g("10M5D140M", 1009) == (9, True) and g("10M5D140M", 1009, True) == (9, True)      # last base before the deletion
    assert g("10M5D140M", 1015) == (10, True)                                                  # first base after it
    assert g("10M3I47M", 1010) == (13, True)                                                   # first base after an insertion
    assert g("5H3I52M", 1000) == (3, True) and g("5H3I52M", 1000, True) == (0, True)          # readStartsWithInsertion (left tail only)
    assert g("3I57M", 1000) == (3, True)
    assert g("60M", 999) == (-1, False) and g("60M", 1059) == (59, True) and g("60M", 1060) == (-1, False)
    assert g("57M3I", 1056) == (56, True) and g("57M3I", 1057) == (-1, False)                # the insertion ends the CIGAR


# ---------------------------------------------------------------- Flatten / ParallelFlatten
def _brute(pairs):
    """union of closed intervals: doubled coordinates make touching intervals ([5,5] + [5,9]) share a point and adjacent ones ([5,5] +
    [6,6]) stay apart; maximal runs of the doubled set are the flattened intervals"""
    p = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    if not p.size:
        return []
    lo = int(p.min())
    mark = np.zeros(2 * (int(p.max()) - lo) + 2, dtype=bool)
    for s, e in p:
        mark[2 * (s - lo):2 * (e - lo) + 1] = True
    d = np.diff(np.concatenate([[0], mark.astype(np.int8), [0]]))
    starts, ends = np.nonzero(d == 1)[0], np.nonzero(d == -1)[0] - 1
    return [[int(s) // 2 + lo, int(e) // 2 + lo] for s, e in zip(starts, ends)]


def _awkward(n, seed):
    """n intervals: random short ones plus duplicates, contained, touching and adjacent neighbours, in random order"""
    rng = np.random.default_rng(seed)
    out = []
    x = 100
    while len(out) < n:
        kind = int(rng.integers(0, 6))
        s = x + int(rng.integers(0, 30))
        e = s + int(rng.integers(0, 12))
        out.append([s, e])
        if kind == 1:
            out.append([s, e])                                   # duplicate
        elif kind == 2:
            out.append([s + (e - s) // 2, s + (e - s) // 2])     # contained
        elif kind == 3:
            out.append([e, e + int(rng.integers(0, 5))])         # touching: merges
        elif kind == 4:
            out.append([e + 1, e + 1 + int(rng.integers(0, 5))])  # adjacent: stays apart
        x = e + int(rng.integers(-8, 20))
    out = out[:n]
    rng.shuffle(out)
    return out


def test_flatten_touching_and_adjacent():
    assert ks.flatten([[5, 5], [5, 9]]) == [[5, 9]]
    assert ks.flatten([[5, 5], [6, 6]]) == [[5, 5], [6, 6]]
    assert ks.flatten([[1, 10], [2, 3], [10, 12], [13, 13]]) == [[1, 12], [13, 13]]
    assert _brute([[5, 5], [5, 9]]) == [[5, 9]] and _brute([[5, 5], [6, 6]]) == [[5, 5], [6, 6]]


@pytest.mark.parametrize("n", [1, 2, 7, 500, 4095, 4096, 4097, 8191, 8192, 8193, 20000])
def test_flatten_matches_union(orc, n):
    raw = _awkward(n, seed=n)
    srt = sorted(raw, key=lambda x: x[0])                        # stable, as ParallelSortByStart
    want = _brute(raw)
    assert ks.flatten([list(x) for x in srt]) == want
    assert ks.parallel_flatten([list(x) for x in srt]) == want
    assert ks.sort_and_flatten(np.array(raw, np.int32)).tolist() == want
    a = np.array(srt, dtype=np.int32).reshape(-1)
    m = orc.lib().orc_flatten(a.ctypes.data_as(C.c_void_p), C.c_int64(len(srt)))
    assert a[:2 * m].reshape(-1, 2).tolist() == want


def test_parallel_flatten_left_swallows_right():
    """ParallelFlatten indexes right[0] after each merge: a left half whose last interval covers the whole right half panics in Go"""
    iv = [[1, 10 ** 6]] + [[10 * k, 10 * k] for k in range(1, ks.GRAIN)]
    with pytest.raises(IndexError):
        ks.parallel_flatten(iv)
    assert ks.flatten([list(x) for x in iv]) == [[1, 10 ** 6]]


def test_intersect():
    iv = np.array([[5, 5], [7, 9], [12, 20]], np.int32)
    assert ks.intersect(iv, 6, 6) == (1, 1)
    assert ks.intersect(iv, 5, 7) == (0, 2)
    assert ks.intersect(iv, 9, 12) == (1, 3)
    assert ks.intersect(iv, 21, 30) == (3, 3)
    assert ks.intersect(iv, 0, 4) == (0, 0)


# ---------------------------------------------------------------- the oracle's mask on single reads
def _unpaired(cases):
    return [c for c in cases if c[3] == "plain"]


CASE_GROUPS = {"count151": kc.count_cases(151), "count32": kc.count_cases(32), "count33": kc.count_cases(33), "handoff": kc.handoff_cases(151),
               "overflow": kc.overflow_cases(151), "overflow512": kc.overflow_cases(512), "quirks": kc.quirk_cases()}


def _clipped(b, i):
    cg = ks.parse_cigar(sam.decode_cigar(b.cigar[int(b.cigar_off[i]):int(b.cigar_off[i + 1])]))
    return ks.hard_clip_soft_clips(int(b.pos[i]), cg)


@pytest.mark.parametrize("group", sorted(CASE_GROUPS))
def test_oracle_mask_single_reads(orc, group):
    """one unpaired read per workload (hardClipAdaptorSequence leaves it alone; soft clips become H): the oracle's total of observations
    equals the ACGT bases with QUAL >= 6 that the restatement's skip slice leaves unmasked"""
    import oracle
    cases = _unpaired(CASE_GROUPS[group])
    counted = masked = 0
    for case in cases:
        w, _ = kc.build([case], quals=(2, 12, 30), n_rg=1, seed=len(case[0]))
        b = w.batch
        for i in range(b.n):
            if b.flag[i] & 1:
                continue                                         # the unmatched second-of-pair copies: same mask, not needed here
            one = b.take(np.array([i]))
            pos, c, s0 = _clipped(one, 0)
            skip = ks.skip_slice(pos, c, w.sites[0])
            L = ks.read_length(c)
            seq = sam.decode_seq(one.seq, int(one.lseq[0]))[s0:s0 + L]
            q = one.qual[s0:s0 + L]
            want = sum(1 for k in range(L) if not skip[k] and seq[k] in "ACGT" and q[k] >= 6)
            ref = oracle.Reference(w.header, w.contig_bases, w.sites)
            t = oracle.bqsr_gather(one, w.header, ref, max_cycle=600, n_threads=1)
            assert int(t.q_obs.sum()) == want, (case[0], int(one.flag[0]), int(t.q_obs.sum()), want)
            counted += want
            masked += int(skip.sum())
    assert counted and masked


def test_case_range_counts():
    """the hand cases reach the range counts their groups are named for (on the clipped alignment, after flattening)"""
    def counts(cases):
        w, names = kc.build(_unpaired(cases), quals=(2, 30), n_rg=1)
        out = {}
        for i in range(w.batch.n):
            pos, c, _ = _clipped(w.batch, i)
            out.setdefault(names[i], set()).add(ks.n_ranges(pos, c, w.sites[0]))
        return out
    for L in (32, 33, 64, 151, 1024):
        assert max(max(v) for v in counts(kc.count_cases(L)).values()) <= 2
    h = counts(kc.handoff_cases(151))
    assert h["three"] == {3} and h["four"] == {4} and h["four_wide"] == {4}
    assert all(v == {1} for k, v in h.items() if k.startswith(("ins", "del")) and not k.endswith("none"))
    o = counts(kc.overflow_cases(512))
    assert min(min(v) for v in o.values()) >= 5
    assert o["seventeen"] == {17} and o["every_other_base"] == {256}
    q = counts(kc.quirk_cases())
    assert q["many_around_deletion"] == {6}
