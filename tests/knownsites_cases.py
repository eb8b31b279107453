"""Hand-made reads with known sites placed on them, grouped by the device path their number of site ranges selects (bqsr_prep2_kernel's
two record slots, ReadDesc.skip[4] of bqsr_prep_kernel, or the 512-bit overflow masks).  Shared by the CPU checks of the oracle's masking
(test_known_sites_cpu.py) and the device parity tests (test_gpu_known_sites.py).

A case is (name, CIGAR, sites, mode): sites are [start, end] offsets from POS (the first aligned base; negative offsets lie before it,
in a leading soft clip), mode is "plain" (unpaired and unmatched second-of-pair reads on both strands, no adaptor clipping) or
("fwd" | "rev", b): a pair whose adaptor boundary lies b bases after POS, so hardClipAdaptorSequence keeps [POS, POS + b) of a forward
read and [POS + b + 1, end] of a reverse one."""
from __future__ import annotations

import numpy as np

from elprep_b200 import sam, synth
from knownsites_ref import parse_cigar, sort_and_flatten

CONTIG = "chr20"


def count_cases(L):
    """0-2 ranges on reads without an indel: all of them stay in bqsr_count_kernel"""
    M, Lm = f"{L}M", L - 10
    S = f"5S{Lm}M5S"
    c = [("none", M, []), ("base0", M, [[0, 0]]), ("base_last", M, [[L - 1, L - 1]]), ("whole_and_beyond", M, [[-5, L + 5]])]
    for a, b in ((31, 32), (32, 32), (30, 33), (63, 64)):
        if a < L:
            c.append((f"lanes_{a}_{b}", M, [[a, b]]))
    c += [("adjacent_1bp", M, [[10, 10], [11, 11]]), ("two_in_one_lane", M, [[3, 5], [8, 9]]), ("first_and_last_lane", M, [[1, 2], [L - 3, L - 2]]),
          ("into_left_clip", S, [[-3, 2]]), ("into_right_clip", S, [[Lm - 3, Lm + 2]]), ("inside_left_clip", S, [[-4, -2]]),
          ("inside_right_clip", S, [[Lm + 1, Lm + 3], [Lm - 1, Lm - 1]])]
    return [(n, cg, s, "plain") for n, cg, s in c]


def adaptor_cases(L):
    """adaptor-clipped pairs (closed form in bqsr_prep2_kernel: hi = rc forward, lo = rc + 1 and cpos = boundary + 1 reverse) with one 1-bp
    site just inside, on and just outside the boundary"""
    b, M = L // 2, f"{L}M"
    out = []
    for side, where in (("fwd", {"inside": b - 1, "on": b, "outside": b + 1}), ("rev", {"inside": b + 1, "on": b, "outside": b - 1})):
        for w, x in where.items():
            out.append((f"adaptor_{side}_{w}", M, [[x, x]], (side, b)))
        out.append((f"adaptor_{side}_two", M, [[b - 3, b - 2], [b + 2, b + 3]], (side, b)))
    return out


def handoff_cases(L):
    """3 and 4 ranges (ReadDesc.skip[4] of the general kernels), and 1-bp sites before, on and after an indel (any site on an indel read
    leaves the count kernel)"""
    M = f"{L}M"
    c = [("three", M, [[2, 2], [10, 12], [20, 20]]), ("four", M, [[2, 2], [10, 12], [20, 20], [L - 3, L - 1]]),
         ("four_wide", M, [[-2, 0], [31, 32], [63, 64], [L - 1, L + 3]])]
    for n in (1, 5):
        ins = f"30M{n}I{L - 30 - n}M"
        c += [(f"ins{n}_none", ins, []), (f"ins{n}_before", ins, [[28, 28]]), (f"ins{n}_on", ins, [[29, 29]]), (f"ins{n}_after", ins, [[30, 30]])]
        dl = f"30M{n}D{L - 30}M"
        c += [(f"del{n}_none", dl, []), (f"del{n}_before", dl, [[29, 29]]), (f"del{n}_on", dl, [[30, 30]]), (f"del{n}_after", dl, [[30 + n, 30 + n]])]
    return [(n, cg, s, "plain") for n, cg, s in c]


def overflow_cases(L):
    """more than four ranges: the 512-bit masks of bqsr_prep_kernel, read by bqsr_general_kernel"""
    M = f"{L}M"
    five = [[1, 1], [5, 5], [9, 9], [13, 13], [17, 17]]
    c = [("five", M, five), ("six", M, five + [[40, 45]]), ("seventeen", M, [[3 * k, 3 * k] for k in range(17)]),
         ("every_other_base", M, [[k, k] for k in range(0, L, 2)]),
         ("ins_six", f"30M2I{L - 32}M", [[5, 5], [10, 10], [29, 29], [30, 30], [31, 31], [60, 62]]),
         ("del_six", f"30M3D{L - 30}M", [[5, 5], [28, 28], [29, 29], [31, 31], [33, 33], [40, 40]]),
         ("clipped_six", f"4S{L - 8}M4S", [[-4, -3], [0, 0], [7, 7], [15, 16], [L - 12, L - 12], [L - 9, L - 5]])]
    if L >= 512:
        c += [("last_word", M, [[100, 100], [480, 481], [485, 485], [490, 495], [500, 500], [505, 511]]),
              ("last_word_every_other", M, [[k, k] for k in range(480, 512, 2)]),
              ("last_word_past_end", M, [[470, 470], [479, 480], [495, 495], [499, 500], [508, 520]])]
    return [(n, cg, s, "plain") for n, cg, s in c]


def quirk_cases(L=60):
    """getReadCoordinateForReferenceCoordinate's quirks, on reads the general kernels take"""
    c = [("starts_in_deletion", "30M5D30M", [[32, 40]]), ("ends_in_deletion", "30M5D30M", [[25, 32]]),
         ("before_deletion", "30M5D30M", [[29, 29]]), ("first_after_insertion", "30M3I27M", [[30, 30]]),
         ("insertion_after_clip_at_pos", "5S3I52M", [[0, 0]]), ("insertion_after_clip_into_clip", "5S3I52M", [[-3, 1]]),
         ("insertion_first_at_pos", "3I57M", [[0, 0]]), ("past_read_end", "30M2D30M", [[L - 1, L + 10]]),
         ("whole_deletion", "30M5D30M", [[30, 34]]), ("many_around_deletion", "30M5D30M", [[3, 3], [27, 27], [29, 31], [34, 35], [40, 40], [50, 52]])]
    return [(n, cg, s, "plain") for n, cg, s in c]


def _flags(mode):
    if mode == "plain":
        return [(0, 0), (0x10, 0), (0x1 | 0x20 | 0x80, 0), (0x1 | 0x10 | 0x80, 0)]
    side, b = mode
    if side == "fwd":
        return [(0x1 | 0x20 | 0x40, b), (0x1 | 0x20 | 0x80, b)]
    return [(0x1 | 0x10 | 0x80, -(b + 50)), (0x1 | 0x10 | 0x40, -(b + 50))]


def build(cases, quals, n_rg=4, seed=0, low_tails=True):
    """-> Workload with one read per (case, flag variant), each on its own stretch of the contig, and the flattened site list of all of
    them; plus the list of (case name, read index) in input order"""
    rng = np.random.default_rng(seed)
    quals = sorted(set(int(q) for q in quals))
    maxlen = max(sum(n for op, n in parse_cigar(cg) if op in "MIDNS=X") for _, cg, _, _ in cases)
    span = maxlen + 400
    n_reads = sum(len(_flags(m)) for *_, m in cases)
    contig_len = 1000 + span * n_reads + 2000
    base = synth.make_workload(1, [(CONTIG, contig_len)], seed=seed + 11, n_rg=n_rg)
    ref = base.contig_bases[0]
    recs, sites, names = [], [], []
    p = 1000
    for name, cg, rel, mode in cases:
        ops = parse_cigar(cg)
        for flag, tlen in _flags(mode):
            pos = p + 100
            p += span
            seq, j = [], pos - 1
            for op, n in ops:
                if op in "M=X":
                    for _ in range(n):
                        r = rng.random()
                        b = chr(ref[j]) if r > 0.05 else ("N" if r < 0.01 else "ACGT"[int(rng.integers(0, 4))])
                        seq.append(b if b in "ACGTN" else "A")
                        j += 1
                elif op in "IS":
                    seq += ["ACGT"[int(x)] for x in rng.integers(0, 4, size=n)]
                elif op in "DN":
                    j += n
            L = len(seq)
            q = rng.choice(quals, size=L)
            k = len(recs)
            if low_tails and k % 3 == 0:
                q[:3] = quals[0]
            if low_tails and k % 5 == 0:
                q[-4:] = quals[0]
            paired = bool(flag & 1)
            if mode == "plain":
                pnext = pos
            else:
                side, bnd = mode
                pnext = pos if side == "fwd" else pos + bnd + 1
            recs.append(dict(QNAME=f"ks{k:05d}", FLAG=flag, RNAME=CONTIG, POS=pos, MAPQ=60, CIGAR=cg, RNEXT="=" if paired else "*",
                             PNEXT=pnext if paired else 0, TLEN=tlen, SEQ="".join(seq), QUAL=[int(x) for x in q], RG=f"rg{k % n_rg + 1}"))
            sites += [[pos + s, pos + e] for s, e in rel]
            names.append(name)
    batch = sam.AlignmentBatch.from_records(base.header, recs)
    flat = sort_and_flatten(np.array(sites, dtype=np.int32).reshape(-1, 2))
    return synth.Workload(base.header, batch, base.contig_bases, [flat], {}), names
