"""Hand-made reads that pin the CIGAR geometry of the BQSR gather, grouped into families by what they aim at.  Shared by the CPU checks of
the case set against the oracle (test_gather_cigar_cases_cpu.py) and the device parity tests (test_gpu_gather_cigar_edges.py).

  indel              one I {1, 2, 15, 16, 17, 31, 32, 33, 255} or D {1, 16, 17, 4095}: the count kernel's indel records, 32-base lanes and
                     two reference windows (fast alphabet), the chunk kernel's per-lane CIGAR walk over 16-base chunks (general alphabet)
  indel_over_record  I = 256 or D = 4096: past the indel record's fields, so bqsr_prep2_kernel hands the read to the general kernels
  complex            shapes closed_form_clip rejects: two indels, adjacent I D / D I, leading and trailing I, =/X runs, P, > 9 and 64 operations,
                     a leading D that a clip on the right folds into H while POS stays put (the reference then reads the reference from POS)
  adaptor            the adaptor boundary (TLEN of forward reads, PNEXT of reverse reads) swept from POS - 1 to the alignment end + 1; a
                     boundary the clipping cannot map to a read base is ELP_ECLIP
  contig_end         the kept alignment ends on the contig's last base, or one base past it with that base counted or not

The indel family places the indel after every number of aligned bases for 48, 64 and 100 aligned bases, and 16k-1, 16k, 16k+1, 32k-1, 32k,
32k+1 bases from either end for 151 and 300; leading / trailing soft clips of 0, 1, 15, 16, 17 bases, hard clips, strand and mate are drawn
per read from a seeded generator.  Every read of a family sits on its own stretch of the contig (no two share a duplicate-marking key);
contig-end reads each get a contig of their own.

A family is (workload of the reads every path must accept, their names, error reads).  An error read is (name, one-read workload, oracle
error code or None, device error code): the reads the oracle or the device refuse, each to be run in a context of its own."""
from __future__ import annotations

import ctypes as C

import numpy as np

from elprep_b200 import sam, synth
from knownsites_ref import parse_cigar

FAST = (2, 5, 14, 30, 40)                        # bqsr_count_kernel S = 3, classifier shift 2; 5 is below the first slot
GENERAL = (2, 5, 6, 15, 22, 27, 33, 37, 40)      # seven values >= 6: the general kernels
INS = (1, 2, 15, 16, 17, 31, 32, 33, 255, 256)
DEL = (1, 16, 17, 4095, 4096)
CLIPS = (0, 1, 15, 16, 17)
FAMILIES = ("indel", "indel_over_record", "complex", "adaptor", "contig_end")

ORACLE_ECLIP = (-3, -4)      # "reference coordinate matches a non-existing base in read", "clip out of range"
ORACLE_EREFEND = -6          # "read extends past contig end"
ELP_ECLIP, ELP_EREFEND, ELP_ELIMIT = -13, -14, -15

FLAGS = {"fwd": 0, "rev": 0x10, "first_fwd": 0x1 | 0x20 | 0x40, "first_rev": 0x1 | 0x10 | 0x40,
         "second_fwd": 0x1 | 0x20 | 0x80, "second_rev": 0x1 | 0x10 | 0x80}


def ref_span(cigar):
    return sum(n for op, n in parse_cigar(cigar) if op in "MDN=X")


def read_len(cigar):
    return sum(n for op, n in parse_cigar(cigar) if op in "MIS=X")


def boundary_offsets(L):
    """16k-1, 16k, 16k+1, 32k-1, 32k, 32k+1 aligned bases from either end of an L-base alignment"""
    xs = {b * k + d for b in (16, 32) for k in range(1, L // b + 1) for d in (-1, 0, 1)}
    return sorted(x for x in xs | {L - x for x in xs} if 1 <= x <= L - 1)


def indel_offsets(L):
    return list(range(1, L)) if L <= 100 else boundary_offsets(L)


def _case(name, cigar, flag="fwd", tlen=0, pnext=None, **kw):
    """pnext: offset from POS (paired reads; None = POS itself); kw: contig_end (bases past the contig end of the last aligned base, the
    read then sits on a contig of its own), qual / seq {read index: value} overrides, sites [[start, end]] as offsets from POS"""
    return dict(name=name, cigar=cigar, flag=FLAGS[flag], tlen=tlen, pnext=pnext, **kw)


def indel_cases(over_record=False, seed=1):
    rng = np.random.default_rng(seed)
    out = []
    for L in (48, 64, 100, 151, 300):
        for op, n in [("I", n) for n in INS] + [("D", n) for n in DEL]:
            if (n == 256 if op == "I" else n == 4096) != over_record or (op == "I" and n >= 255 and L > 151):   # (<= 441 bases with clips)
                continue
            for m1 in indel_offsets(L):
                a, b = CLIPS[int(rng.integers(0, 5))], CLIPS[int(rng.integers(0, 5))]
                h = int(rng.integers(0, 4))
                cg = ("4H" if h & 1 else "") + (f"{a}S" if a else "") + f"{m1}M{n}{op}{L - m1}M" + (f"{b}S" if b else "") + ("3H" if h & 2 else "")
                flag = str(rng.choice(["first_fwd", "first_rev", "second_fwd", "second_rev", "fwd", "rev"], p=[.23, .23, .23, .23, .04, .04]))
                out.append(_case(f"{op}{n}_L{L}_at{m1}", cg, flag))
    return out


def _ops64():
    """2S (3M 1D) x 30 3M 1I 4M: 64 operations, 100 bases"""
    return "2S" + "3M1D" * 30 + "3M1I4M"


def complex_cases():
    c = [("two_indels", "20M2I10M3D28M"), ("del_then_ins", "10M5D10M5I40M"), ("adjacent_ID", "30M2I2D28M"), ("adjacent_DI", "30M2D2I28M"),
         ("leading_I", "3I57M"), ("leading_I_after_S", "4S3I53M"), ("leading_I_after_HS", "2H4S3I53M"), ("trailing_I", "57M3I"),
         ("trailing_I_before_S", "52M3I5S"), ("eq_x_runs", "20=1X39="), ("m_eq_x", "10M2X5=43M"), ("x_first", "1X59M"),
         ("padding", "20M2P40M"), ("padding_in_insertion", "10M1I2P1I48M"), ("ten_ops", "3S5M1I5M1D5M1I5M1D34M"),
         ("leading_D_right_clip", "2D56M4S"), ("leading_D_indel_right_clip", "3H2D20M2I34M4S"),   # clip on the right: the D folds into H, POS stays
         ("many_indels", "2S" + "4M1I3M1D" * 6 + "10M2S"), ("ops64", _ops64())]
    out = [_case(n, cg, f) for n, cg in c for f in ("fwd", "rev", "second_fwd", "second_rev")]
    for n, cg in c[4:7]:                        # readStartsWithInsertion: a known site at POS maps to the read start
        out.append(_case(n + "_site_at_pos", cg, "rev", sites=[[0, 0]]))
    # 64 operations whose adaptor clip splits an operation (the middle base of the 16th 3M, 61 reference bases after POS): the clipped
    # CIGAR has one operation more than the stored one before clean_hard_clipped merges the hard clips
    out += [_case("ops64_adaptor_fwd", _ops64(), "first_fwd", tlen=61), _case("ops64_adaptor_rev", _ops64(), "second_rev", tlen=-150, pnext=62),
            _case("ops64_adaptor_fwd_in_del", _ops64(), "first_fwd", tlen=63), _case("ops64_adaptor_rev_in_del", _ops64(), "second_rev", tlen=-150, pnext=64)]
    # 64 operations without soft clips: the reverse read's clip splits the first operation, so the clipped CIGAR has 65
    ops = "3M1D" * 31 + "3M1I"
    out += [_case("ops64_split_first_rev", ops, "second_rev", tlen=-200, pnext=2), _case("ops64_split_last_fwd", ops, "first_fwd", tlen=125)]
    # 65 operations: past MAXC of bqsr_prep_kernel, refused as ELP_ELIMIT (the oracle accepts the read)
    out += [_case("ops65", _ops64() + "2S", "fwd", limit=True), _case("ops65_rev", _ops64() + "2S", "second_rev", limit=True)]
    return out


ADAPTOR_CIGARS = ("10S30M5I30M5S", "40M10D40M", "5H3S20M2I2D20M3S", "1M1I58M", "58M1D1M", "5S50M5S", "2D58M")   # 2D58M: the oracle refuses
                                                                                                                # a boundary on POS + 1


def adaptor_cases():
    """forward reads: boundary = POS + |TLEN| for TLEN = 1 .. span + 1 (POS + 1 .. alignment end + 2); reverse reads: boundary = PNEXT - 1
    for PNEXT = POS .. alignment end + 2 (POS - 1: no clip, .. alignment end + 1); first and second of pair alternate"""
    out = []
    for cg in ADAPTOR_CIGARS:
        R = ref_span(cg)
        for t in range(1, R + 2):
            out.append(_case(f"{cg}_fwd_b{t}", cg, "first_fwd" if t % 2 else "second_fwd", tlen=t))
        for p in range(0, R + 2):
            out.append(_case(f"{cg}_rev_b{p - 1}", cg, "second_rev" if p % 2 else "first_rev", tlen=-(R + 50), pnext=p))
    return out


def contig_end_cases():
    """contig_end: how far past the contig end the last aligned base lies (0: on the contig's last base); the QUAL / SEQ overrides are
    read indices of the 60-base reads (59: the last base)"""
    last, tail2 = {59: 5}, {58: 2, 59: 2}
    c = [("ends_on_last_base", "60M", 0, {}, {}, None), ("ends_on_last_base_rev", "60M", 0, {}, {}, None, "rev"),
         ("soft_clip_past_end", "58M2S", 0, {}, {}, None), ("trailing_deletion_past_end", "60M5D", 0, {}, {}, None),
         ("past_counted", "60M", 1, {}, {}, None), ("past_counted_rev", "60M", 1, {}, {}, None, "second_rev"),
         ("past_qual_below_6", "60M", 1, last, {}, None), ("past_qual_below_6_rev", "60M", 1, last, {}, None, "second_rev"),
         ("past_n", "60M", 1, {}, {59: "N"}, None), ("past_low_quality_tail", "60M", 1, tail2, {}, None),
         ("past_known_site", "60M", 1, {}, {}, [[58, 70]]), ("past_two_uncounted", "60M", 2, {58: 5, 59: 3}, {}, None),
         ("past_after_deletion", "40M5D20M", 1, {}, {}, None), ("past_after_deletion_uncounted", "40M5D20M", 1, last, {}, None),
         ("past_after_insertion_uncounted", "40M3I17M", 1, last, {}, None), ("past_clipped_s_uncounted", "3S57M", 1, last, {}, None)]
    out = []
    for name, cg, end, q, s, sites, *fl in c:
        out.append(_case(name, cg, fl[0] if fl else "fwd", contig_end=end, qual=q, seq=s, sites=sites or []))
    return out


CASES = {"indel": lambda: indel_cases(False), "indel_over_record": lambda: indel_cases(True), "complex": complex_cases,
         "adaptor": adaptor_cases, "contig_end": contig_end_cases}


def build(cases, quals, n_rg=4, seed=0):
    """-> (Workload of all the cases, names in input order).  Aligned bases copy the reference with 5 % other bases and 1 % N; QUAL is drawn
    from ``quals``, every third read starting and every fifth ending in a low-quality tail (QUAL 2)"""
    rng = np.random.default_rng(seed)
    quals = sorted(set(int(q) for q in quals))
    main = 1000 + sum(ref_span(c["cigar"]) + read_len(c["cigar"]) + 100 for c in cases if "contig_end" not in c) + 1000
    n_end = sum(1 for c in cases if "contig_end" in c)
    contigs = [("chr20", main)] + [(f"end{k}", 2000) for k in range(n_end)]
    base = synth.make_workload(1, contigs, seed=seed + 11, n_rg=n_rg)
    recs, names, sites = [], [], [[] for _ in contigs]
    p, e = 1000, 0
    for c in cases:
        cg, ops = c["cigar"], parse_cigar(c["cigar"])
        lead = sum(n for op, n in ops[:2] if op == "S") if ops[0][0] in "SH" else 0
        at_end = "contig_end" in c
        if at_end:
            e += 1
            ci = e
            last_m = max(i for i, (op, _) in enumerate(ops) if op in "M=X")
            pos = contigs[ci][1] - sum(n for op, n in ops[:last_m + 1] if op in "MDN=X") + 1 + c["contig_end"]
        else:
            ci = 0
            pos = p + 50 + lead
            p += ref_span(cg) + read_len(cg) + 100
        ref = base.contig_bases[ci]
        seq, past, j = [], [], pos - 1
        for op, n in ops:
            if op in "M=X":
                for _ in range(n):
                    if j >= len(ref):
                        past.append(len(seq))
                        seq.append("ACGT"[int(rng.integers(0, 4))])
                    else:
                        r = rng.random()
                        b = chr(ref[j]) if r > 0.05 else ("N" if r < 0.01 else "ACGT"[int(rng.integers(0, 4))])
                        seq.append(b if b in "ACGTN" else "A")
                    j += 1
            elif op in "IS":
                seq += ["ACGT"[int(x)] for x in rng.integers(0, 4, size=n)]
            elif op in "DN":
                j += n
        q = rng.choice(quals, size=len(seq))
        k = len(recs)
        if at_end:
            q[past] = quals[-1]                     # counted unless the case says otherwise
        else:
            if k % 3 == 0:
                q[:3] = 2
            if k % 5 == 0:
                q[-4:] = 2
        for i, v in c.get("qual", {}).items():
            q[i] = v
        for i, v in c.get("seq", {}).items():
            seq[i] = v
        paired = bool(c["flag"] & 1)
        pnext = pos + (c["pnext"] or 0)
        recs.append(dict(QNAME=f"cg{k:05d}", FLAG=c["flag"], RNAME=contigs[ci][0], POS=pos, MAPQ=60, CIGAR=cg, RNEXT="=" if paired else "*",
                         PNEXT=pnext if paired else 0, TLEN=c["tlen"], SEQ="".join(seq), QUAL=[int(x) for x in q], RG=f"rg{k % n_rg + 1}"))
        sites[ci] += [[pos + s0, pos + s1] for s0, s1 in c.get("sites", [])]
        names.append(c["name"])
    batch = sam.AlignmentBatch.from_records(base.header, recs)
    flat = [np.array(sorted(s), dtype=np.int32).reshape(-1, 2) for s in sites]
    return synth.Workload(base.header, batch, base.contig_bases, flat, {}), names


def probe_clip(b, i):
    """the oracle's hardClipAdaptorSequence + hardClipSoftClippedBases of read i -> (rc, kept [lo, hi), POS after clipping, clipped CIGAR
    words); rc < 0: the oracle's error code, -1: clipped away"""
    import oracle
    co = b.cigar_off.astype(np.int64)
    cg = np.ascontiguousarray(b.cigar[co[i]:co[i + 1]])
    lo, hi, npos = C.c_int32(), C.c_int32(), C.c_int32()
    out = np.zeros(256, np.uint32)
    rc = oracle.lib().orc_probe_clip(C.c_int32(int(b.pos[i])), C.c_uint16(int(b.flag[i])), C.c_int32(int(b.pnext[i])), C.c_int32(int(b.tlen[i])),
                                     C.c_int32(int(b.refid[i])), C.c_int32(int(b.nref[i])), cg.ctypes.data_as(C.c_void_p), C.c_int32(len(cg)),
                                     C.c_int32(int(b.lseq[i])), C.byref(lo), C.byref(hi), C.byref(npos), out.ctypes.data_as(C.c_void_p), C.c_int(256))
    return rc, lo.value, hi.value, npos.value, out[:max(rc, 0)].copy()


class Family:
    """good: Workload of the reads every path accepts, names: theirs; errors: [(name, one-read Workload, oracle code or None, device code)]"""

    def __init__(self, good, names, errors):
        self.good, self.names, self.errors = good, names, errors


def expected_error(case, b, i):
    """(oracle error code or None, device error code) of read i built from ``case``, or None when both accept it"""
    if case.get("limit"):
        return None, ELP_ELIMIT
    if case.get("contig_end", 0) > 0:
        return ORACLE_EREFEND, ELP_EREFEND
    rc = probe_clip(b, i)[0]
    return (rc, ELP_ECLIP) if rc in ORACLE_ECLIP else None


def family(name, quals, seed=0):
    cases = CASES[name]()
    w, names = build(cases, quals, seed=seed)
    b = w.batch
    good, errors = [], []
    for i, c in enumerate(cases):
        e = expected_error(c, b, i)
        if e is None:
            good.append(i)
        else:
            errors.append((names[i], synth.Workload(w.header, b.take([i]), w.contig_bases, w.sites, {}), e[0], e[1]))
    return Family(synth.Workload(w.header, b.take(good), w.contig_bases, w.sites, {}), [names[i] for i in good], errors)


def cap_cycles(w, max_cycle):
    """QUAL 2 on every stored base whose cycle (prepareCycleCovariates, bqsr.go:376-383: 1-based position in sequencing order) is beyond
    ``max_cycle``: BQSR then accepts reads longer than max_cycle, whose kept bases the gather kernels take one warp per read"""
    b = w.batch.copy()
    qo = b.qual_off.astype(np.int64)
    for i in range(b.n):
        L = int(b.lseq[i])
        if L > max_cycle:
            q = b.qual[qo[i]:qo[i] + L]
            if b.flag[i] & 0x10:
                q[:L - max_cycle] = 2
            else:
                q[max_cycle:] = 2
    return synth.Workload(w.header, b, w.contig_bases, w.sites, w.params)


def oracle_dense(w, max_cycle=500):
    """the oracle's dense table counters [n_cov][94][ncols][2] of the reads of ``w`` as they stand (no duplicate marking)"""
    import oracle
    from util import oracle_tables_dense
    t = oracle.bqsr_gather(w.batch, w.header, oracle.Reference(w.header, w.contig_bases, w.sites), max_cycle=max_cycle, n_threads=1)
    return oracle_tables_dense(t, max_cycle)[0]


def contributions(w, max_cycle=500, reads=None):
    """read index -> its dense table counters alone, for ``reads`` (default: all) of ``w``"""
    out = {}
    for i in (range(w.batch.n) if reads is None else reads):
        out[i] = oracle_dense(synth.Workload(w.header, w.batch.take([i]), w.contig_bases, w.sites, {}), max_cycle)
    return out
