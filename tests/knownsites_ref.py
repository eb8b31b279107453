"""Plain restatement of the known-sites masking of BQSR, written from the reference's Go source:

  Extend / Flatten / ParallelFlatten / Intersect          intervals/intervals.go:88-173 (and ParallelSortByStart :76-80, a stable sort)
  computeReadCoordinateForReferenceCoordinate,
  getReadCoordinateForReferenceCoordinate                  filters/utils.go:267-349
  readStartsWithInsertion                                  filters/bqsr.go:287-299
  calculateSkipSlice                                       filters/bqsr.go:389-414

Intervals are [start, end] pairs, both ends inclusive (1-based reference positions).  CIGARs are lists of (op, length) with op one of
"MIDNSHP=X"; ``parse_cigar`` reads the SAM text form.  Nothing here imports the oracle or the CUDA library: the tests compare both with it.
"""
from __future__ import annotations

import re

import numpy as np

CONSUMES_REF = set("MDN=X")
CONSUMES_READ = set("MIS=X")
GRAIN = 0x1000                      # parallelFlattenGrainSize


def parse_cigar(s):
    return [(op, int(n)) for n, op in re.findall(r"(\d+)([MIDNSHP=X])", s)]


def cigar_str(c):
    return "".join(f"{n}{op}" for op, n in c)


def read_length(c):
    """sam.ReadLengthFromCigar"""
    return sum(n for op, n in c if op in CONSUMES_READ)


def ref_length(c):
    return sum(n for op, n in c if op in CONSUMES_REF)


# ---------------------------------------------------------------- intervals
def extend(a, b):
    """Interval.Extend: grows ``a`` (a mutable [start, end]) when ``b`` overlaps or touches it; b.start >= a.start is a precondition"""
    if b[0] > a[1]:
        return False
    if b[1] > a[1]:
        a[1] = b[1]
    return True


def flatten(iv):
    """Flatten over a start-sorted list of [start, end] lists, in place, returning the prefix that holds the result"""
    i, n = 0, len(iv) - 1
    while i < n:
        if extend(iv[i], iv[i + 1]):
            n += 1
            for j in range(i + 1, n):
                if not extend(iv[i], iv[j]):
                    i += 1
                    iv[i] = list(iv[j])
            return iv[:i + 1]
        i += 1
    return iv


def parallel_flatten(iv):
    """ParallelFlatten: halves below the grain size are flattened serially, then the halves are joined.  Go indexes right[0] after every
    merge, so a left interval that swallows the whole right half panics there; that surfaces as IndexError."""
    if len(iv) < GRAIN:
        return flatten(iv)
    half = len(iv) >> 1
    left, right = parallel_flatten(iv[:half]), parallel_flatten(iv[half:])
    while extend(left[-1], right[0]):
        right = right[1:]
    return left + right


def sort_and_flatten(pairs):
    """what NewBaseRecalibrator does to a contig's known sites: a stable sort by start, then ParallelFlatten -> int32 array [k, 2]"""
    iv = sorted(([int(s), int(e)] for s, e in np.asarray(pairs).reshape(-1, 2)), key=lambda x: x[0])
    out = parallel_flatten(iv) if iv else []
    return np.array(out, dtype=np.int32).reshape(-1, 2)


def intersect(iv, start, end):
    """Intersect: the slice of a flattened, sorted interval list that overlaps [start, end] -> (lo, hi) indices"""
    iv = np.asarray(iv).reshape(-1, 2)
    lo = int(np.searchsorted(iv[:, 1], start, side="left"))      # first i with End >= start
    hi = int(np.searchsorted(iv[:, 0], end, side="right"))       # first i with Start > end
    return lo, max(lo, hi)


# ---------------------------------------------------------------- read coordinates
def compute_read_coord(c, soft_start, ref_index):
    """computeReadCoordinateForReferenceCoordinate -> (readBases, fallsInsideOrJustBeforeDeletionOrSkippedRegion); (-1, False) on failure"""
    goal = ref_index - soft_start
    if goal < 0:
        return -1, False
    read_bases = ref_bases = 0
    falls_inside = ends_just_before = fob = False
    index = 0
    while ref_bases != goal and index < len(c):
        op, ln = c[index]
        index += 1
        shift = 0
        if op in CONSUMES_REF or op == "S":
            shift = ln if ref_bases + ln < goal else goal - ref_bases
            ref_bases += shift
        if ref_bases != goal:
            read_bases += ln if op in CONSUMES_READ else 0
        else:
            if shift >= ln and index == len(c):
                return -1, False
            nxt = None
            if shift < ln:
                falls_inside = op in "DN"
            else:
                nxt = c[index]
                index += 1
                if nxt[0] == "I":
                    read_bases += nxt[1]
                    if index == len(c):
                        return -1, False
                    nxt = c[index]
                    index += 1
                ends_just_before = nxt[0] in "DN"
            fob = ends_just_before or falls_inside
            cr = 1 if op in CONSUMES_READ else 0
            if not fob:
                read_bases += cr * shift
            elif ends_just_before:
                read_bases += cr * (shift - 1)
            elif falls_inside or (ends_just_before and nxt is not None and nxt[0] in "DN"):
                read_bases -= 1
    if ref_bases != goal:
        return -1, False
    return read_bases, fob


def read_starts_with_insertion(c):
    """readStartsWithInsertion -> (length, True) for the first I behind leading H / S, else (-1, False)"""
    for op, ln in c:
        if op == "I":
            return ln, True
        if op in "HS":
            continue
        return -1, False
    return -1, False


def get_read_coord(c, soft_start, ref_index, tail_right=False):
    """getReadCoordinateForReferenceCoordinate -> (read coordinate, ok)"""
    rb, fob = compute_read_coord(c, soft_start, ref_index)
    if rb == -1:
        return -1, False
    if tail_right and fob:
        rb += 1
    if not tail_right and rb == 0:
        fl, first = read_starts_with_insertion(c)
        if first:
            rb = min(fl, read_length(c) - 1)
    return rb, True


def soft_start(pos, c):
    s = pos
    for op, ln in c:
        if op == "S":
            s -= ln
        elif op != "H":
            break
    return s


def soft_end(pos, c):
    end = pos + ref_length(c) - 1
    se = end
    for op, ln in reversed(c):
        if op == "S":
            se += ln
        elif op != "H":
            return se
    return end


# ---------------------------------------------------------------- calculateSkipSlice
def hard_clip_soft_clips(pos, c):
    """hardClipSoftClippedBases (filters/utils.go:506-534) for an alignment whose soft clips touch an M, I, = or X operation: the clips
    become H (merged with any H beside them) and POS stays.  -> (pos, clipped CIGAR, first kept base of the stored read)"""
    src = list(c)
    left_h = left_s = right_h = right_s = 0
    i = 0
    while i < len(src) and src[i][0] in "HS":
        left_h += src[i][1] if src[i][0] == "H" else 0
        left_s += src[i][1] if src[i][0] == "S" else 0
        i += 1
    j = len(src)
    while j > i and src[j - 1][0] in "HS":
        right_h += src[j - 1][1] if src[j - 1][0] == "H" else 0
        right_s += src[j - 1][1] if src[j - 1][0] == "S" else 0
        j -= 1
    mid = src[i:j]
    if mid and (mid[0][0] in "DN" or mid[-1][0] in "DN"):
        raise NotImplementedError("a deletion beside a clip is folded into the hard clip; this restatement does not cover it")
    out = ([("H", left_h + left_s)] if left_h + left_s else []) + mid + ([("H", right_h + right_s)] if right_h + right_s else [])
    return pos, out, left_s


def skip_slice(pos, c, sites):
    """calculateSkipSlice over a clipped alignment (POS ``pos``, CIGAR ``c`` without S) and a flattened, sorted site list -> bool [L]"""
    L = read_length(c)
    ss, se = soft_start(pos, c), soft_end(pos, c)
    skip = np.zeros(L, dtype=bool)
    sites = np.asarray(sites).reshape(-1, 2)
    lo, hi = intersect(sites, ss, se)
    for s, e in sites[lo:hi]:
        fs, ok = get_read_coord(c, ss, int(s))
        if not ok or fs < 0:
            fs = 0
        fe, ok = get_read_coord(c, ss, int(e))
        if not ok or fe > L - 1:
            fe = L - 1
        skip[fs:fe + 1] = True
    return skip


def n_ranges(pos, c, sites):
    """site ranges (flattened intervals) the clipped alignment overlaps: what decides the device path of a read"""
    lo, hi = intersect(sites, soft_start(pos, c), soft_end(pos, c))
    return hi - lo
