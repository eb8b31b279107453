"""Plain restatement of the --known-sites input, written from the reference's Go source:

  intervals.FromElsitesFile            intervals/intervals.go:199-254 (the header, then bufio.Scanner lines split at the first two tabs)
  bufio.ScanLines / MaxScanTokenSize   a line ends at '\\n', one '\\r' before it is dropped, the last line may lack its '\\n'; a line of
                                       65536 bytes or more stops the scanner (ErrTooLong)
  strconv.ParseInt(s, 10, 32)          an optional sign, then decimal digits only, inside int32
  NewBaseRecalibrator                  filters/bqsr.go:424-443: the files' intervals appended per chromosome, then sorted and flattened

Sorting and flattening reuse knownsites_ref.  Where ParallelFlatten would panic (knownsites_ref raises IndexError) the serial Flatten
result is used, as elp_set_known_sites and elp_load_known_sites do.  Nothing here imports the CUDA library."""
from __future__ import annotations

import numpy as np

import knownsites_ref as ks

HEADER = b"# elsites format version 1.0\n"     # intervals.ElsitesHeader (intervals.go:176)
MAX_TOKEN = 65536                              # bufio.MaxScanTokenSize

# reasons, as elp_last_error words them
HEADER_BAD, FIELDS, START, END, LONG = "header", "invalid sites line", "start", "end", "too long"


class ElsitesError(ValueError):
    def __init__(self, file, line, reason):
        super().__init__(f"file {file}, line {line}: {reason}")
        self.file, self.line, self.reason = file, line, reason


def parse_int32(s: bytes) -> int:
    """strconv.ParseInt(s, 10, 32); ValueError when it fails"""
    t, neg = s, False
    if t[:1] in (b"+", b"-"):
        neg, t = t[:1] == b"-", t[1:]
    if not t or any(c < 0x30 or c > 0x39 for c in t):
        raise ValueError(s)
    v = -int(t) if neg else int(t)
    if not -(1 << 31) <= v < (1 << 31):
        raise ValueError(s)
    return v


def scan_lines(body: bytes):
    """bufio.ScanLines over the bytes after the header -> [(raw length before '\\n', line without '\\n' and one '\\r')]"""
    out, i = [], 0
    while i < len(body):
        j = body.find(b"\n", i)
        tok = body[i:] if j < 0 else body[i:j]
        i = len(body) if j < 0 else j + 1
        out.append((len(tok), tok[:-1] if tok.endswith(b"\r") else tok))
    return out


def from_elsites(data: bytes, file=0):
    """FromElsitesFile -> [(chromosome bytes, start, end)] in file order; ElsitesError(file, line, reason) at the first rejected line
    (line numbers 0-based, the header is line 0)"""
    nl = data.find(b"\n")
    if nl < 0 or data[:nl + 1] != HEADER:
        raise ElsitesError(file, 0, HEADER_BAD)
    out = []
    for k, (raw, s) in enumerate(scan_lines(data[nl + 1:]), start=1):
        if raw >= MAX_TOKEN:
            raise ElsitesError(file, k, LONG)
        i = s.find(b"\t")
        if i <= 0:
            raise ElsitesError(file, k, FIELDS)
        j = s.find(b"\t", i + 1)
        if j < 0:
            raise ElsitesError(file, k, FIELDS)
        try:
            st = parse_int32(s[i + 1:j])
        except ValueError:
            raise ElsitesError(file, k, START) from None
        try:
            en = parse_int32(s[j + 1:])
        except ValueError:
            raise ElsitesError(file, k, END) from None
        out.append((s[:i], st, en))
    return out


def sort_flatten(pairs):
    """a contig's list as the device keeps it: knownsites_ref.sort_and_flatten, or the serial Flatten where ParallelFlatten panics"""
    try:
        return ks.sort_and_flatten(pairs)
    except IndexError:
        iv = sorted(([int(s), int(e)] for s, e in np.asarray(pairs).reshape(-1, 2)), key=lambda x: x[0])
        return np.array(ks.flatten(iv), dtype=np.int32).reshape(-1, 2)


def sort_flatten_fast(pairs):
    """the same list as sort_flatten for large inputs, vectorised: after a stable sort by start, interval i opens a group iff its start
    lies above every earlier end (a closed group ended below the start of the group after it), and a group keeps the max of its ends"""
    p = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    if not len(p):
        return np.zeros((0, 2), np.int32)
    o = np.argsort(p[:, 0], kind="stable")
    s, e = p[o, 0], p[o, 1]
    prev = np.concatenate([[-(1 << 31) - 1], np.maximum.accumulate(e)[:-1]])
    heads = np.flatnonzero(s > prev)
    return np.stack([s[heads], np.maximum.reduceat(e, heads)], axis=1).astype(np.int32)


def load(files, contig_names):
    """elp_load_known_sites over file contents -> (per-contig (k, 2) int32 lists, lines whose chromosome is "*" or no @SQ SN).
    Every contig whose SN equals a line's chromosome gets the interval."""
    names = [n.encode() if isinstance(n, str) else n for n in contig_names]
    per_name = {}
    unmatched = 0
    for f, data in enumerate(files):
        for chrom, st, en in from_elsites(data, f):
            if chrom == b"*" or chrom not in names:
                unmatched += 1
            else:
                per_name.setdefault(chrom, []).append((st, en))
    tables = [sort_flatten(np.array(per_name.get(n, []) if n != b"*" else [], dtype=np.int64).reshape(-1, 2)) for n in names]
    return tables, unmatched


def write(chroms_starts_ends, crlf=False, final_newline=True):
    """an .elsites file from (chromosome, start, end) rows"""
    eol = b"\r\n" if crlf else b"\n"
    rows = [b"%s\t%d\t%d" % (c.encode() if isinstance(c, str) else c, s, e) for c, s, e in chroms_starts_ends]
    body = eol.join(rows) + (eol if final_newline and rows else b"")
    return HEADER + body
